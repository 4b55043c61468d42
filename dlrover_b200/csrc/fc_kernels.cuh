// fc_kernels.cuh — the three copy kernels of the Flash Checkpoint path (sm_90a),
// all templated on direction (0 = gather/pack: tensors -> arena, 1 = scatter):
//   fc_copy_lsu        128-bit LDG/STG, any alignment (heads, tails, small ranges,
//                      table slices of the windowed / hybrid saves)
//   fc_copy_tma        cp.async.bulk global->shared->global ring, 16-B congruent bodies
//   fc_copy_tma_shift  TMA in, funnel shift shared->shared, TMA out: ranges whose
//                      source and destination are not congruent mod 16
// Pure byte copies; bound: HBM bandwidth, 2 bytes of traffic per checkpoint byte.
// And the two gather-compare kernels of the incremental save (end of the file):
//   fc_delta_tma       16-B congruent bodies: TMA loads of the source tile AND of the
//                      arena tile it replaces, compare in shared memory, TMA store
//                      only of the tiles that differ
//   fc_delta_lsu       everything else (heads, tails, shifted ranges, small pieces):
//                      copy_range with a compare, stores only the vectors that differ
// Both write `seq` into dirty[item.pad0] when any byte of the item differs.
// Traffic: 2 bytes read per checkpoint byte + 1 byte written per dirty byte.
// Included by flashckpt.cu only.
#pragma once

#include <cuda_runtime.h>

#include "fc_items.h"

// ------------------------------------------------------------ device helpers --

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ uint4 ldg_cached(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ void stg_stream(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// 16 output bytes starting r bytes into the 32-byte little-endian pair (lo,hi).
// q = r>>2 selects the first 32-bit word, sh = 8*(r&3) the bit shift.
template <int Q>
__device__ __forceinline__ uint4 funnel16(const uint4& lo, const uint4& hi, uint32_t sh) {
  const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  uint4 o;
  o.x = __funnelshift_r(w[Q + 0], w[Q + 1], sh);
  o.y = __funnelshift_r(w[Q + 1], w[Q + 2], sh);
  o.z = __funnelshift_r(w[Q + 2], w[Q + 3], sh);
  o.w = __funnelshift_r(w[Q + 3], w[Q + 4], sh);
  return o;
}

__device__ __forceinline__ uint4 shfl_down1(const uint4& v) {
  uint4 o;
  o.x = __shfl_down_sync(0xffffffffu, v.x, 1);
  o.y = __shfl_down_sync(0xffffffffu, v.y, 1);
  o.z = __shfl_down_sync(0xffffffffu, v.z, 1);
  o.w = __shfl_down_sync(0xffffffffu, v.w, 1);
  return o;
}

// Copy nvec 16-B vectors: dst is 16-B aligned, src = abase + r (abase aligned).
// Output vector i needs the aligned words W[i] and W[i+1].  Every lane loads
// its W[i] ONCE (coalesced 512 B per warp) and takes W[i+1] from its right
// neighbour with a shuffle; only lane 31 loads the extra halo word.  (Loading
// both words per lane fetches every straddled sector twice.)
template <int Q>
__device__ __forceinline__ void copy_shifted(const uint4* __restrict__ abase,
                                             uint4* __restrict__ dst, uint32_t nvec,
                                             uint32_t sh) {
  constexpr int T = kLsuThreads, U = kLsuUnroll;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t wbase = threadIdx.x - lane;  // first vector of this warp in the block row
  // W[nvec] (the halo of the last vector) shares a 16-B word with valid source
  // bytes, so indices <= nvec are readable.
  for (uint32_t base = wbase; base < nvec; base += U * T) {  // warp-uniform bounds
    uint4 lo[U], hi[U];
    // all global loads first (body + lane-31 halos), so one memory latency is
    // exposed per iteration, not two
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint32_t idx = base + j * T + lane;
      lo[j] = idx <= nvec ? ldg_stream(abase + idx) : make_uint4(0, 0, 0, 0);
      hi[j] = (lane == 31u && idx < nvec) ? ldg_cached(abase + idx + 1) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint4 nb = shfl_down1(lo[j]);
      if (lane != 31u) hi[j] = nb;
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint32_t idx = base + j * T + lane;
      if (idx < nvec) stg_stream(dst + idx, funnel16<Q>(lo[j], hi[j], sh));
    }
  }
}

// CTA-wide copy of n bytes, any alignment on either side.
__device__ __forceinline__ void copy_range(const uint8_t* __restrict__ src,
                                           uint8_t* __restrict__ dst, uint32_t n) {
  constexpr int T = kLsuThreads, U = kLsuUnroll;
  // head: bring dst to 16-B alignment
  uint32_t head = (uint32_t)((16u - ((uintptr_t)dst & 15u)) & 15u);
  if (head > n) head = n;
  if (threadIdx.x < head) dst[threadIdx.x] = src[threadIdx.x];
  src += head;
  dst += head;
  n -= head;
  const uint32_t nvec = n >> 4;
  const uint32_t tail = n & 15u;
  if (threadIdx.x < tail) {
    const uint32_t o = (nvec << 4) + threadIdx.x;
    dst[o] = src[o];
  }
  if (nvec == 0) return;
  const uint32_t r = (uint32_t)((uintptr_t)src & 15u);
  uint4* __restrict__ d = reinterpret_cast<uint4*>(dst);
  if (r == 0) {
    const uint4* __restrict__ s = reinterpret_cast<const uint4*>(src);
    uint32_t i = threadIdx.x;
    for (; i + (U - 1) * T < nvec; i += U * T) {
      uint4 v[U];
#pragma unroll
      for (int j = 0; j < U; ++j) v[j] = ldg_stream(s + i + j * T);
#pragma unroll
      for (int j = 0; j < U; ++j) stg_stream(d + i + j * T, v[j]);
    }
    for (; i < nvec; i += T) stg_stream(d + i, ldg_stream(s + i));
  } else {
    // The two aligned words that straddle each output vector: the first starts
    // r bytes before src, the last ends (16-r) bytes after the body; both share
    // a 16-B word with at least one valid source byte, so no page is touched
    // that the source range does not already touch.
    const uint4* __restrict__ ab = reinterpret_cast<const uint4*>(src - r);
    const uint32_t sh = (r & 3u) * 8u;
    switch (r >> 2) {
      case 0: copy_shifted<0>(ab, d, nvec, sh); break;
      case 1: copy_shifted<1>(ab, d, nvec, sh); break;
      case 2: copy_shifted<2>(ab, d, nvec, sh); break;
      default: copy_shifted<3>(ab, d, nvec, sh); break;
    }
  }
}

// DIR 0: tensors -> arena (pack).  DIR 1: arena -> tensors (unpack).
template <int DIR>
__global__ void __launch_bounds__(kLsuThreads)
fc_copy_lsu(const FcItem* __restrict__ items, uint32_t n_items, uint8_t* __restrict__ arena) {
  for (uint32_t c = blockIdx.x; c < n_items; c += gridDim.x) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(items + c));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(items + c) + 1);
    uint8_t* t = reinterpret_cast<uint8_t*>(((uint64_t)a.y << 32) | a.x);
    uint8_t* ar = arena + (((uint64_t)a.w << 32) | a.z);
    const uint32_t n = b.x;
    if (DIR == 0)
      copy_range(t, ar, n);
    else
      copy_range(ar, t, n);
  }
}

// ---------------------------------------------------------------- TMA kernel --

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "FC_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra FC_DONE_%=;\n"
      "bra FC_WAIT_%=;\n"
      "FC_DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes,
                                         uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_dst),
      "l"(gsrc), "r"(bytes), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, uint32_t smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Walks the tiles of the items owned by this CTA (items blockIdx.x, +gridDim.x, ...).
struct TileCursor {
  const FcItem* items;
  uint32_t n_items, item, off, n;
  uint32_t idx;  // FcItem.pad0: index of the item's `all` entry (gather-compare only)
  uint64_t tptr, aoff;
  __device__ __forceinline__ void fetch() {
    if (item < n_items) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(items + item));
      const uint4 b = __ldg(reinterpret_cast<const uint4*>(items + item) + 1);
      tptr = ((uint64_t)a.y << 32) | a.x;
      aoff = ((uint64_t)a.w << 32) | a.z;
      n = b.x;
      idx = b.y;
    }
  }
  __device__ __forceinline__ void init(const FcItem* it, uint32_t cnt) {
    items = it;
    n_items = cnt;
    item = blockIdx.x;
    off = 0;
    fetch();
  }
  __device__ __forceinline__ bool valid() const { return item < n_items; }
  __device__ __forceinline__ uint32_t bytes(uint32_t tile) const {
    const uint32_t left = n - off;
    return left < tile ? left : tile;
  }
  __device__ __forceinline__ void advance(uint32_t tile) {
    off += tile;
    if (off >= n) {
      item += gridDim.x;
      off = 0;
      fetch();
    }
  }
};

// Every item handed to this kernel has tptr, aoff (and the arena base) 16-B
// aligned and nbytes a multiple of 16 — the plan builder guarantees it.
template <int DIR>
__global__ void __launch_bounds__(32)
fc_copy_tma(const FcItem* __restrict__ items, uint32_t n_items, uint8_t* __restrict__ arena,
            uint32_t tile, uint32_t stages) {
  extern __shared__ __align__(128) uint8_t fc_smem[];
  if (threadIdx.x != 0) return;
  const uint32_t smem_base = smem_u32(fc_smem);
  const uint32_t bar_base = smem_base + stages * tile;
  for (uint32_t s = 0; s < stages; ++s) mbar_init(bar_base + 8 * s, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

  TileCursor ld, st;
  ld.init(items, n_items);
  st.init(items, n_items);

  auto issue_load = [&](uint32_t stage) {
    const uint32_t nb = ld.bytes(tile);
    const void* g = DIR == 0 ? reinterpret_cast<const void*>(ld.tptr + ld.off)
                             : reinterpret_cast<const void*>(arena + ld.aoff + ld.off);
    mbar_expect_tx(bar_base + 8 * stage, nb);
    bulk_g2s(smem_base + stage * tile, g, nb, bar_base + 8 * stage);
    ld.advance(tile);
  };

  uint32_t primed = 0;
  while (primed < stages && ld.valid()) issue_load(primed++);

  for (uint32_t k = 0; st.valid(); ++k) {
    const uint32_t stage = k % stages;
    mbar_wait(bar_base + 8 * stage, (k / stages) & 1u);
    const uint32_t nb = st.bytes(tile);
    void* g = DIR == 0 ? reinterpret_cast<void*>(arena + st.aoff + st.off)
                       : reinterpret_cast<void*>(st.tptr + st.off);
    bulk_s2g(g, smem_base + stage * tile, nb);
    bulk_commit();
    st.advance(tile);
    if (k >= 1 && ld.valid()) {
      bulk_wait_read<1>();  // store k-1 (and older) no longer reads its stage
      issue_load((k - 1) % stages);
    }
  }
  bulk_wait_all();
}

// ---- TMA-fed byte-shift kernel ------------------------------------------------
// For ranges whose source and destination are NOT congruent mod 16 (everything
// behind a 4-byte optimizer `step` scalar in the reference's unpadded layout).
// Global traffic is all bulk-async and fully sector-efficient: the aligned
// source span of each 16 KiB destination tile (+ one 16-B halo word) is
// TMA-loaded into a shared-memory ring, 128 threads funnel-shift it from shared
// to shared (two LDS.128 + four SHF + one STS.128 per 16 B), and the aligned
// result is TMA-stored.  The LSU shifted path re-reads straddled sectors; this
// one does not.
constexpr int kShiftThreads = 256;
// shared memory: in_stages x (tile + 128 B halo slot) input ring, 2 x tile
// output double buffer, in_stages mbarriers
static inline size_t shift_smem_bytes(uint32_t tile, uint32_t in_stages) {
  return (size_t)in_stages * (tile + 128u) + 2u * (size_t)tile + 8u * in_stages;
}

struct ShiftCursor {
  const FcItem* items;
  uint32_t n_items, item, voff;  // voff: vectors of the body already consumed
  // per item (after the destination-aligning peel)
  const uint8_t* src;  // first body byte (r = src & 15)
  uint8_t* dst;        // 16-B aligned
  uint32_t nvec, r;
};

template <int DIR>
__device__ __forceinline__ void shift_fetch(ShiftCursor& c, uint8_t* arena) {
  while (c.item < c.n_items) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(c.items + c.item));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(c.items + c.item) + 1);
    uint8_t* t = reinterpret_cast<uint8_t*>(((uint64_t)a.y << 32) | a.x);
    uint8_t* ar = arena + (((uint64_t)a.w << 32) | a.z);
    const uint8_t* s = DIR == 0 ? t : ar;
    uint8_t* d = DIR == 0 ? ar : t;
    uint32_t n = b.x;
    uint32_t head = (uint32_t)((16u - ((uintptr_t)d & 15u)) & 15u);
    if (head > n) head = n;
    c.src = s + head;
    c.dst = d + head;
    c.nvec = (n - head) >> 4;
    c.r = (uint32_t)((uintptr_t)c.src & 15u);
    c.voff = 0;
    if (c.nvec) return;
    c.item += gridDim.x;  // nothing but peel bytes: the consumer side copies them
  }
}

// Head (< 16 B before the aligned body) and tail (< 16 B after it) of an item.
template <int DIR>
__device__ __forceinline__ void shift_peel(const FcItem* items, uint32_t item, uint8_t* arena) {
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(items + item));
  const uint4 b = __ldg(reinterpret_cast<const uint4*>(items + item) + 1);
  uint8_t* t = reinterpret_cast<uint8_t*>(((uint64_t)a.y << 32) | a.x);
  uint8_t* ar = arena + (((uint64_t)a.w << 32) | a.z);
  const uint8_t* s = DIR == 0 ? t : ar;
  uint8_t* d = DIR == 0 ? ar : t;
  const uint32_t n = b.x;
  uint32_t head = (uint32_t)((16u - ((uintptr_t)d & 15u)) & 15u);
  if (head > n) head = n;
  const uint32_t body = (n - head) & ~15u;
  const uint32_t tail = n - head - body;
  if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
  if (threadIdx.x >= 16 && threadIdx.x - 16 < tail) {
    const uint32_t o = head + body + threadIdx.x - 16;
    d[o] = s[o];
  }
}

template <int Q>
__device__ __forceinline__ void shift_tile(const uint8_t* in, uint8_t* out, uint32_t nv,
                                           uint32_t sh) {
  const uint4* __restrict__ w = reinterpret_cast<const uint4*>(in);
  uint4* __restrict__ o = reinterpret_cast<uint4*>(out);
  for (uint32_t i = threadIdx.x; i < nv; i += kShiftThreads) o[i] = funnel16<Q>(w[i], w[i + 1], sh);
}

template <int DIR>
__global__ void __launch_bounds__(kShiftThreads)
fc_copy_tma_shift(const FcItem* __restrict__ items, uint32_t n_items,
                  uint8_t* __restrict__ arena, uint32_t kShiftTile, uint32_t kShiftStages) {
  extern __shared__ __align__(128) uint8_t fc_smem[];
  const uint32_t kShiftInStride = kShiftTile + 128u;
  uint8_t* in_base = fc_smem;
  uint8_t* out_base = fc_smem + kShiftStages * kShiftInStride;
  const uint32_t bar_base = smem_u32(out_base + 2u * kShiftTile);
  const uint32_t kTileVec = kShiftTile / 16;
  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < kShiftStages; ++s) mbar_init(bar_base + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // Peel bytes of every item this CTA owns (tiny, done up front).
  for (uint32_t it = blockIdx.x; it < n_items; it += gridDim.x) shift_peel<DIR>(items, it, arena);

  // Load cursor lives in thread 0 only; the consume cursor is replicated.
  ShiftCursor ld, cs;
  cs.items = items; cs.n_items = n_items; cs.item = blockIdx.x;
  shift_fetch<DIR>(cs, arena);
  ld = cs;

  auto tile_vecs = [&](const ShiftCursor& c) {
    const uint32_t left = c.nvec - c.voff;
    return left < kTileVec ? left : kTileVec;
  };
  auto advance = [&](ShiftCursor& c) {
    c.voff += kTileVec;
    if (c.voff >= c.nvec) {
      c.item += gridDim.x;
      shift_fetch<DIR>(c, arena);
    }
  };
  auto issue_load = [&](uint32_t stage) {  // thread 0
    const uint32_t nv = tile_vecs(ld);
    const uint32_t nb = nv * 16u + (ld.r ? 16u : 0u);  // + halo word
    const void* g = ld.src - ld.r + (size_t)ld.voff * 16u;
    mbar_expect_tx(bar_base + 8 * stage, nb);
    bulk_g2s(smem_u32(in_base + stage * kShiftInStride), g, nb, bar_base + 8 * stage);
    advance(ld);
  };

  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < kShiftStages && ld.item < n_items; ++s) issue_load(s);
  }

  for (uint32_t k = 0; cs.item < n_items; ++k) {
    const uint32_t stage = k % kShiftStages;
    mbar_wait(bar_base + 8 * stage, (k / kShiftStages) & 1u);
    const uint32_t nv = tile_vecs(cs);
    const uint8_t* in = in_base + stage * kShiftInStride;
    uint8_t* out = out_base + (k & 1u) * kShiftTile;
    const uint32_t sh = (cs.r & 3u) * 8u;
    switch (cs.r >> 2) {
      case 0: shift_tile<0>(in, out, nv, sh); break;
      case 1: shift_tile<1>(in, out, nv, sh); break;
      case 2: shift_tile<2>(in, out, nv, sh); break;
      default: shift_tile<3>(in, out, nv, sh); break;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // STS -> bulk store
    __syncthreads();  // tile shifted; input stage fully read
    if (threadIdx.x == 0) {
      bulk_s2g(cs.dst + (size_t)cs.voff * 16u, smem_u32(out), nv * 16u);
      bulk_commit();
      if (ld.item < n_items) issue_load(stage);  // refill the stage just consumed
      bulk_wait_read<1>();  // store k-1 done reading: out[(k+1)&1] is free again
    }
    advance(cs);
    __syncthreads();
  }
  if (threadIdx.x == 0) bulk_wait_all();
}

// ---- gather-compare kernels (incremental save) -----------------------------------
// The arena still holds the image the previous save drained to the segment.  These
// kernels write into it only the bytes that differ from the new source bytes and mark
// every `all` item that had any difference: dirty[item.pad0] = seq.  The host then
// drains only the marked items.  A mark is the save's sequence number, so the marks
// need no clearing between saves.

// Plain (coherent) 128-bit load of arena bytes that this kernel may store to later.
__device__ __forceinline__ uint4 ld_arena(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ bool differ(const uint4& a, const uint4& b) {
  return ((a.x ^ b.x) | (a.y ^ b.y) | (a.z ^ b.z) | (a.w ^ b.w)) != 0u;
}

// copy_shifted with a compare: the old vector is loaded with the source words and the
// shifted result is stored only where it differs.  Returns this thread's "differs".
template <int Q>
__device__ __forceinline__ bool delta_shifted(const uint4* __restrict__ abase,
                                              uint4* __restrict__ dst, uint32_t nvec,
                                              uint32_t sh) {
  constexpr int T = kLsuThreads, U = kLsuUnroll;
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t wbase = threadIdx.x - lane;
  bool d = false;
  for (uint32_t base = wbase; base < nvec; base += U * T) {  // warp-uniform bounds
    uint4 lo[U], hi[U], old[U];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint32_t idx = base + j * T + lane;
      lo[j] = idx <= nvec ? ldg_stream(abase + idx) : make_uint4(0, 0, 0, 0);
      hi[j] = (lane == 31u && idx < nvec) ? ldg_cached(abase + idx + 1) : make_uint4(0, 0, 0, 0);
      old[j] = idx < nvec ? ld_arena(dst + idx) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint4 nb = shfl_down1(lo[j]);
      if (lane != 31u) hi[j] = nb;
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint32_t idx = base + j * T + lane;
      if (idx < nvec) {
        const uint4 v = funnel16<Q>(lo[j], hi[j], sh);
        if (differ(v, old[j])) {
          stg_stream(dst + idx, v);
          d = true;
        }
      }
    }
  }
  return d;
}

// copy_range with a compare (any alignment on either side).  Every thread of the CTA
// must call it; returns this thread's "differs".
__device__ __forceinline__ bool delta_range(const uint8_t* __restrict__ src,
                                            uint8_t* __restrict__ dst, uint32_t n) {
  constexpr int T = kLsuThreads, U = kLsuUnroll;
  bool d = false;
  uint32_t head = (uint32_t)((16u - ((uintptr_t)dst & 15u)) & 15u);
  if (head > n) head = n;
  if (threadIdx.x < head) {
    const uint8_t v = src[threadIdx.x];
    if (dst[threadIdx.x] != v) {
      dst[threadIdx.x] = v;
      d = true;
    }
  }
  src += head;
  dst += head;
  n -= head;
  const uint32_t nvec = n >> 4;
  const uint32_t tail = n & 15u;
  if (threadIdx.x < tail) {
    const uint32_t o = (nvec << 4) + threadIdx.x;
    const uint8_t v = src[o];
    if (dst[o] != v) {
      dst[o] = v;
      d = true;
    }
  }
  if (nvec == 0) return d;
  const uint32_t r = (uint32_t)((uintptr_t)src & 15u);
  uint4* __restrict__ dv = reinterpret_cast<uint4*>(dst);
  if (r == 0) {
    const uint4* __restrict__ s = reinterpret_cast<const uint4*>(src);
    uint32_t i = threadIdx.x;
    for (; i + (U - 1) * T < nvec; i += U * T) {
      uint4 v[U], o[U];
#pragma unroll
      for (int j = 0; j < U; ++j) {
        v[j] = ldg_stream(s + i + j * T);
        o[j] = ld_arena(dv + i + j * T);
      }
#pragma unroll
      for (int j = 0; j < U; ++j)
        if (differ(v[j], o[j])) {
          stg_stream(dv + i + j * T, v[j]);
          d = true;
        }
    }
    for (; i < nvec; i += T) {
      const uint4 v = ldg_stream(s + i);
      if (differ(v, ld_arena(dv + i))) {
        stg_stream(dv + i, v);
        d = true;
      }
    }
    return d;
  }
  const uint4* __restrict__ ab = reinterpret_cast<const uint4*>(src - r);
  const uint32_t sh = (r & 3u) * 8u;
  switch (r >> 2) {
    case 0: return delta_shifted<0>(ab, dv, nvec, sh) || d;
    case 1: return delta_shifted<1>(ab, dv, nvec, sh) || d;
    case 2: return delta_shifted<2>(ab, dv, nvec, sh) || d;
    default: return delta_shifted<3>(ab, dv, nvec, sh) || d;
  }
}

// Gather-compare for any item (residues, shifted ranges, pieces under 4 KiB; every item
// under FC_VARIANT_LSU).  One CTA per item; a warp that saw a difference marks it.
__global__ void __launch_bounds__(kLsuThreads)
fc_delta_lsu(const FcItem* __restrict__ items, uint32_t n_items, uint8_t* __restrict__ arena,
             uint32_t* __restrict__ dirty, uint32_t seq) {
  for (uint32_t c = blockIdx.x; c < n_items; c += gridDim.x) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(items + c));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(items + c) + 1);
    const uint8_t* t = reinterpret_cast<const uint8_t*>(((uint64_t)a.y << 32) | a.x);
    uint8_t* ar = arena + (((uint64_t)a.w << 32) | a.z);
    const bool d = delta_range(t, ar, b.x);
    if (__any_sync(0xffffffffu, d) && (threadIdx.x & 31u) == 0u) dirty[b.y] = seq;
  }
}

// Gather-compare for the 16-B congruent bodies.  A stage holds the source tile and the
// arena tile it replaces, both TMA-loaded on one mbarrier; the CTA compares them with
// 128-bit shared-memory loads, and thread 0 TMA-stores the source tile only if it
// differs.  Shared memory: stages x 2 x tile + one mbarrier per stage.
constexpr int kDeltaThreads = 256;
static inline size_t delta_smem_bytes(uint32_t tile, uint32_t stages) {
  return (size_t)stages * 2u * tile + 8u * stages;
}

__global__ void __launch_bounds__(kDeltaThreads)
fc_delta_tma(const FcItem* __restrict__ items, uint32_t n_items, uint8_t* __restrict__ arena,
             uint32_t* __restrict__ dirty, uint32_t seq, uint32_t tile, uint32_t stages) {
  extern __shared__ __align__(128) uint8_t fc_smem[];
  const uint32_t smem_base = smem_u32(fc_smem);
  const uint32_t bar_base = smem_base + stages * 2u * tile;
  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < stages; ++s) mbar_init(bar_base + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // the load cursor is used by thread 0 only; the consume cursor is replicated
  TileCursor ld, st;
  ld.init(items, n_items);
  st.init(items, n_items);

  auto issue_load = [&](uint32_t stage) {  // thread 0
    const uint32_t nb = ld.bytes(tile);
    const uint32_t bar = bar_base + 8 * stage;
    const uint32_t s_new = smem_base + stage * 2u * tile;
    mbar_expect_tx(bar, 2u * nb);
    bulk_g2s(s_new, reinterpret_cast<const void*>(ld.tptr + ld.off), nb, bar);
    bulk_g2s(s_new + tile, arena + ld.aoff + ld.off, nb, bar);
    ld.advance(tile);
  };

  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < stages && ld.valid(); ++s) issue_load(s);
  }

  for (uint32_t k = 0; st.valid(); ++k) {
    const uint32_t stage = k % stages;
    mbar_wait(bar_base + 8 * stage, (k / stages) & 1u);
    const uint32_t nb = st.bytes(tile);
    const uint4* nw = reinterpret_cast<const uint4*>(fc_smem + (size_t)stage * 2u * tile);
    const uint4* od = nw + tile / 16u;
    bool d = false;
    for (uint32_t i = threadIdx.x; i < nb / 16u; i += kDeltaThreads) d |= differ(nw[i], od[i]);
    // every thread is done reading the stage (and the one before it) past this point
    const bool tile_dirty = __syncthreads_or(d) != 0;
    if (threadIdx.x == 0) {
      if (tile_dirty) {
        bulk_s2g(arena + st.aoff + st.off, smem_base + stage * 2u * tile, nb);
        bulk_commit();
        dirty[st.idx] = seq;
      }
      if (k >= 1 && ld.valid()) {
        // refill the stage consumed at k-1 once its store (if any) has read it out;
        // only committed stores count as groups
        if (tile_dirty)
          bulk_wait_read<1>();
        else
          bulk_wait_read<0>();
        issue_load((k - 1) % stages);
      }
    }
    st.advance(tile);
  }
  if (threadIdx.x == 0) bulk_wait_all();
}

// ------------------------------------------------------------- non-finite scan --
// fc_scan_nonfinite: read-only scan of the source bytes of a plan that counts the
// elements whose exponent field is all ones (NaN or +-Inf).  float8_e4m3fn has no Inf:
// only its NaN patterns (0x7F, 0xFF) count.  Complex kinds are scanned as their float
// components.  Its own item table: FcItem.tptr = element-aligned source address,
// .nbytes = whole elements (<= kDefaultChunk), .aoff = kind (FC_KIND_*), .pad0 = index of
// the input range.  Bodies: 128-bit non-allocating loads, 4x unrolled as in copy_range;
// 16-B heads and tails: element loads.  Traffic: 1 byte read per scanned byte; clean
// data writes nothing, an item with a hit costs one atomic per warp per output.
enum : uint32_t {
  kScanF16 = 1,
  kScanBF16 = 2,
  kScanF32 = 3,
  kScanF64 = 4,
  kScanE5M2 = 5,
  kScanE4M3 = 6
};

// hits in one 32-bit word (F64: the word holding an element's exponent)
template <uint32_t K>
__device__ __forceinline__ uint32_t bad_word(uint32_t w) {
  if (K == kScanF64) return (w & 0x7FF00000u) == 0x7FF00000u;
  if (K == kScanF32) return (w & 0x7F800000u) == 0x7F800000u;
  if (K == kScanF16) return __popc(__vcmpeq2(w & 0x7C007C00u, 0x7C007C00u)) >> 4;
  if (K == kScanBF16) return __popc(__vcmpeq2(w & 0x7F807F80u, 0x7F807F80u)) >> 4;
  if (K == kScanE5M2) return __popc(__vcmpeq4(w & 0x7C7C7C7Cu, 0x7C7C7C7Cu)) >> 3;
  return __popc(__vcmpeq4(w & 0x7F7F7F7Fu, 0x7F7F7F7Fu)) >> 3;  // e4m3fn: S.1111.111
}

template <uint32_t K>
__device__ __forceinline__ uint32_t bad_vec(const uint4& v) {
  // a 16-B aligned vector holds whole elements; a float64's exponent is in its high word
  if (K == kScanF64) return bad_word<K>(v.y) + bad_word<K>(v.w);
  return bad_word<K>(v.x) + bad_word<K>(v.y) + bad_word<K>(v.z) + bad_word<K>(v.w);
}

// one element of ES bytes, zero-extended (the upper lanes of the word then never match)
template <uint32_t K, uint32_t ES>
__device__ __forceinline__ uint32_t bad_elem(const uint8_t* p) {
  if (ES == 8) return bad_word<K>(__ldg(reinterpret_cast<const uint32_t*>(p) + 1));
  if (ES == 4) return bad_word<K>(__ldg(reinterpret_cast<const uint32_t*>(p)));
  if (ES == 2) return bad_word<K>(__ldg(reinterpret_cast<const unsigned short*>(p)));
  return bad_word<K>(__ldg(reinterpret_cast<const unsigned char*>(p)));
}

// this thread's hits among the n bytes at p (p and n multiples of ES)
template <uint32_t K, uint32_t ES>
__device__ __forceinline__ uint32_t scan_range(const uint8_t* __restrict__ p, uint32_t n) {
  constexpr int T = kLsuThreads, U = kLsuUnroll;
  uint32_t head = (uint32_t)((16u - ((uintptr_t)p & 15u)) & 15u);
  if (head > n) head = n;
  const uint32_t body = (n - head) & ~15u;
  const uint32_t nhead = head / ES, ntail = (n - head - body) / ES;
  uint32_t bad = 0;
  if (threadIdx.x < nhead)
    bad += bad_elem<K, ES>(p + threadIdx.x * ES);
  else if (threadIdx.x < nhead + ntail)
    bad += bad_elem<K, ES>(p + head + body + (threadIdx.x - nhead) * ES);
  const uint4* __restrict__ s = reinterpret_cast<const uint4*>(p + head);
  const uint32_t nvec = body >> 4;
  uint32_t i = threadIdx.x;
  for (; i + (U - 1) * T < nvec; i += U * T) {
    uint4 v[U];
#pragma unroll
    for (int j = 0; j < U; ++j) v[j] = ldg_stream(s + i + j * T);
#pragma unroll
    for (int j = 0; j < U; ++j) bad += bad_vec<K>(v[j]);
  }
  for (; i < nvec; i += T) bad += bad_vec<K>(ldg_stream(s + i));
  return bad;
}

__device__ __forceinline__ void add_saturating(uint32_t* c, uint32_t v) {
  const uint32_t old = atomicAdd(c, v);
  if (old + v < old) atomicMax(c, 0xFFFFFFFFu);  // every wrap is followed by its own max
}

// counts[range] += hits of the item (saturating), *total += hits.
__global__ void __launch_bounds__(kLsuThreads)
fc_scan_nonfinite(const FcItem* __restrict__ items, uint32_t n_items, uint32_t* counts,
                  unsigned long long* total) {
  for (uint32_t c = blockIdx.x; c < n_items; c += gridDim.x) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(items + c));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(items + c) + 1);
    const uint8_t* p = reinterpret_cast<const uint8_t*>(((uint64_t)a.y << 32) | a.x);
    const uint32_t n = b.x;
    uint32_t bad = 0;
    switch (a.z) {  // uniform per item
      case kScanF16: bad = scan_range<kScanF16, 2>(p, n); break;
      case kScanBF16: bad = scan_range<kScanBF16, 2>(p, n); break;
      case kScanF32: bad = scan_range<kScanF32, 4>(p, n); break;
      case kScanF64: bad = scan_range<kScanF64, 8>(p, n); break;
      case kScanE5M2: bad = scan_range<kScanE5M2, 1>(p, n); break;
      case kScanE4M3: bad = scan_range<kScanE4M3, 1>(p, n); break;
      default: break;
    }
    bad = __reduce_add_sync(0xffffffffu, bad);
    if ((threadIdx.x & 31u) == 0 && bad) {
      add_saturating(counts + b.y, bad);
      atomicAdd(total, (unsigned long long)bad);
    }
  }
}
