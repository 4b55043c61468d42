// flashckpt.cu — device engine of the H100 Flash Checkpoint path (sm_90a only).
//
// What the reference does on this path (dlrover @ 468d632):
//   ckpt_saver.py:198-231   per leaf: torch.frombuffer(shm).copy_(gpu_tensor)
//                           -> one blocking pageable cudaMemcpy per tensor.
// What this file does instead:
//   1. a cached descriptor table ("plan") maps every leaf tensor to its byte
//      offset in the checkpoint segment (reference layout: running sum of
//      numel*element_size, no padding; ckpt_saver.py:286-301);
//   2. ONE persistent gather kernel copies all leaves into a contiguous HBM
//      arena that is a byte image of the segment (pack), HBM-bandwidth bound:
//      algorithmic traffic 2*S bytes per save;
//   3. the arena is drained to the (pinned, NUMA-local) POSIX shm segment by DMA
//      on a side stream gated by an event — the training stream only ever waits
//      for (2).  A pump thread feeds the copy engine one kDrainPiece (16 MiB)
//      piece at a time (fc_set_drain) so the drain does not starve the
//      application's own D2H copies;
//   4. restore is the inverse: DMA fill + scatter kernel;
//   5. if the state does not fit in HBM a second time it is drained IN PLACE (DMA
//      straight from the tensors, optionally with a snapshot of the tail that fits:
//      fc_save_direct_async / fc_save_hybrid_async); a forced arena cap streams it
//      window by window through a bounded arena instead (blocking, PCIe speed).
//
// Three kernels (fc_kernels.cuh), all templated on direction (0 = gather/pack, 1 = scatter):
//   fc_copy_tma       one elected thread per CTA drives a ring of cp.async.bulk
//                     global->shared (mbarrier complete_tx) and shared->global
//                     (bulk_group) transfers: the 16-B congruent bodies.
//                     Default: one CTA per SM (132 on H100 SXM) x 2 stages x
//                     96 KiB, 192 KiB of the 227 KB of shared memory a block may use.
//   fc_copy_tma_shift ranges whose source and destination are NOT congruent
//                     mod 16: TMA in, funnel shift shared->shared, TMA out.
//   fc_copy_lsu       256-thread CTAs, 128-bit LDG/STG, 4-way unrolled: heads,
//                     tails, tiny ranges, and everything when FC_VARIANT_LSU is
//                     selected.
// and, for the opt-in incremental save (fc_save_delta_async), their gather-compare
// twins fc_delta_tma / fc_delta_lsu: they write only the bytes that differ from the
// arena's previous image and mark the work items to drain.
//
// No torch types here; see include/flashckpt.h for the ABI contract.

#include "../../include/flashckpt.h"

#include <cuda_runtime.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <errno.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

// ------------------------------------------------------------------ errors --

static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, const char* a = "", const char* b = "") {
  snprintf(g_err, sizeof(g_err), fmt, a, b);
  return code;
}

#define FC_CUDA(call)                                                          \
  do {                                                                         \
    cudaError_t _e = (call);                                                   \
    if (_e != cudaSuccess) return fail(FC_ECUDA, "%s: %s", #call, cudaGetErrorString(_e)); \
  } while (0)

extern "C" int fc_version(void) { return FC_VERSION; }

extern "C" const char* fc_strerror(int code) {
  switch (code) {
    case FC_OK: return "ok";
    case FC_EINVAL: return "invalid argument";
    case FC_ECUDA: return "CUDA runtime error";
    case FC_ENOMEM: return "out of memory";
    case FC_EBUSY: return "a save/restore is still in flight";
    case FC_ENOIMAGE: return "the arena holds no image of the segment for this plan";
    case FC_EIO: return "reading the source file failed";
    case FC_ENOTREADY: return "not ready";
    default: return "unknown flashckpt error";
  }
}

extern "C" const char* fc_last_error(void) { return g_err; }

#include "fc_items.h"
#include "fc_kernels.cuh"

// ----------------------------------------------------------------- host side --

// What the drain of an incremental save needs to turn dirty marks into DMA runs: the
// extent of every `all` item (ascending arena offset) and the plan's runs (arena offset
// -> segment offset).  Built once per plan fill and shared with the queued drain jobs,
// so a plan update or destroy never pulls it from under a drain.
struct DeltaMap {
  std::vector<uint64_t> aoff;
  std::vector<uint32_t> len;
  std::vector<FcRun> runs;
  bool same_extents(const DeltaMap& o) const {
    if (aoff != o.aoff || len != o.len || runs.size() != o.runs.size()) return false;
    for (size_t i = 0; i < runs.size(); ++i)
      if (runs[i].off != o.runs[i].off || runs[i].len != o.runs[i].len ||
          runs[i].hoff != o.runs[i].hoff)
        return false;
    return true;
  }
};

// One part of a transfer between the device and the host: len bytes at device address dev,
// at offset off of the host mapping (or of the file a restore reads).
struct Seg {
  uint8_t* dev;
  uint64_t off;
  uint64_t len;
};

struct fc_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t copy_stream = nullptr;
  cudaStream_t copy_stream2 = nullptr;  // second leg of the ping-pong drain
  uint8_t* arena = nullptr;
  uint64_t arena_bytes = 0;
  uint64_t arena_cap = 0;  // 0 = unlimited; else fc_arena_reserve never allocates more
  // tuning (launch shapes of the three copy kernels)
  int variant = FC_VARIANT_TMA;
  int lsu_ctas_per_sm = 2;
  int tma_ctas_per_sm = 1;
  int tma_stages = 2;
  int tma_tile = 96 << 10;
  int shift_ctas_per_sm = 2;
  int shift_tile = 16 << 10;
  int shift_stages = 2;
  // save pipeline state (one in flight)
  cudaEvent_t ev_pack_start = nullptr, ev_pack_end = nullptr, ev_drain_start = nullptr,
              ev_drain_end = nullptr;
  uint64_t ticket = 0;        // last issued
  bool save_inflight = false; // until observed complete
  // restore pipeline state
  cudaEvent_t ev_fill_start = nullptr, ev_fill_end = nullptr, ev_scatter_end = nullptr;
  bool restore_inflight = false;
  // host ranges pinned for DMA: one entry per fc_host_register* call; a background
  // registration pins slice by slice on its own thread
  struct HostReg {
    uint8_t* base = nullptr;
    uint64_t bytes = 0;
    uint64_t slice = 0;             // 0: one cudaHostRegister call for the whole range
    std::vector<void*> done;        // registered slice starts
    std::thread th;
    std::atomic<bool> cancel{false};
    std::atomic<int> state{0};      // 0 in progress, 1 complete, -1 failed
  };
  std::vector<std::unique_ptr<HostReg>> regs;
  // bounce slots of the staged transfers (segment not registered yet)
  struct StageWorker {
    cudaStream_t stream = nullptr;
    uint8_t* slot[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
  };
  std::vector<StageWorker> stage;
  uint64_t stage_slot = 8ull << 20;
  int stage_threads = 8;
  // evidence counters: kernels launched / DMA copies enqueued by this context
  uint64_t n_kernels = 0, n_memcpys = 0;
  // drain pump (one thread per context, started lazily)
  std::thread pump;
  std::mutex mu;
  std::condition_variable cv;
  struct DrainJob {
    int staged_threads = 0;  // > 0: host range not registered, go through the bounce slots
    uint8_t* host = nullptr;
    std::vector<Seg> spans;  // in-place part: DMA straight from the tensors, drained first
    std::vector<Seg> runs;   // arena part
    bool direct = false;     // in-place form: report the in-place part (inplace_done_ticket)
    uint64_t ticket = 0;
    // incremental save: `runs` is built by the pump from the items marked `seq`
    std::shared_ptr<const DeltaMap> delta;
    uint32_t seq = 0;
  };
  uint64_t direct_ticket = 0;  // last ticket with an in-place part (sources frozen until drained)
  uint64_t inplace_done_ticket = 0;  // last ticket whose in-place part has left the tensors
  uint64_t held_ticket = 0;  // the pump must not start the drain of this ticket yet
  std::deque<DrainJob> jobs;
  bool pump_stop = false;
  uint64_t drained_ticket = 0;  // last ticket whose bytes are all in host memory
  int drain_rc = FC_OK;         // sticky error of the pump
  std::string drain_err;
  cudaEvent_t ring[kDrainRing] = {};
  cudaEvent_t ring_pp[kDrainRing] = {};  // ping-pong mode: blocking-sync events
  int drain_mode = FC_DRAIN_HOST_PACED;
  // device/pinned buffers whose cudaFree (a device-wide sync) is deferred to a
  // moment that synchronises anyway
  std::vector<void*> dead_dev, dead_pinned;
  uint64_t drain_piece = kDrainPiece;
  int drain_depth = kDrainDepth;
  // Incremental saves (fc_save_delta_async).  The baseline is the (plan, host_base) of
  // the last delta save that drained without error: the arena then is a byte image of
  // what the segment holds for that plan.  Every other operation that writes the arena
  // or the segment through this context forgets it (delta_forget).  Guarded by `mu`.
  const fc_plan* base_plan = nullptr;
  const uint8_t* base_host = nullptr;
  bool base_valid = false;
  uint64_t base_ticket = 0;  // the delta save that becomes the baseline once drained
  // Arena image (fc_restore_from_image_async): for every run of img_map, arena byte `off`
  // equals segment byte `hoff` at img_host.  Set by a full-arena fc_save_async* or an
  // fc_save_delta_async once it has drained without error, kept by the rollback, forgotten
  // by everything that forgets the baseline.  Guarded by `mu`.
  std::shared_ptr<const DeltaMap> img_map;
  const fc_plan* img_plan = nullptr;
  const uint8_t* img_host = nullptr;
  bool img_valid = false;
  uint64_t img_ticket = 0;  // the save that sets the image once drained
  // dirty marks: one entry per `all` item of the plan being saved, = the save's seq
  uint32_t* dirty = nullptr;
  uint32_t* dirty_pinned = nullptr;
  uint32_t dirty_cap = 0;
  uint32_t delta_seq = 0;
  // what the drain of ticket stat_ticket moved
  uint64_t stat_ticket = 0, stat_bytes = 0;
  int stat_delta = 0;
};

static void baseline_forget_locked(fc_ctx* c) {
  c->base_valid = false;
  c->base_ticket = 0;
}

static void image_forget_locked(fc_ctx* c) {
  c->img_valid = false;
  c->img_ticket = 0;
}

// The arena or the segment may no longer hold the image: forget the incremental baseline
// and the arena image.
static void delta_forget_locked(fc_ctx* c) {
  baseline_forget_locked(c);
  image_forget_locked(c);
}

// A save that leaves the arena a byte image of the segment for plan p (full-arena gather,
// then a drain of every run it changed): the image is valid once ticket has drained.
static void image_expect_locked(fc_ctx* c, const fc_plan* p, const uint8_t* host,
                                uint64_t ticket);

static void delta_forget(fc_ctx* c) {
  std::lock_guard<std::mutex> lk(c->mu);
  delta_forget_locked(c);
}

static fc_ctx::HostReg* reg_covering(fc_ctx* c, const uint8_t* p, uint64_t len);

// A host range pinned slice by slice is a row of separate registrations to CUDA, and
// a cudaMemcpy that straddles two of them fails with "invalid argument": every DMA
// the library issues is cut at the slice boundaries of the range it touches.
struct SliceClip {
  const uint8_t* base = nullptr;
  uint64_t slice = 0;
  SliceClip(fc_ctx* c, const uint8_t* some_byte) {
    std::lock_guard<std::mutex> lk(c->mu);
    if (fc_ctx::HostReg* r = reg_covering(c, some_byte, 1)) {
      base = r->base;
      slice = r->slice;
    }
  }
  uint64_t operator()(const uint8_t* p, uint64_t len) const {
    if (!slice) return len;
    const uint64_t in = (uint64_t)(p - base) % slice;
    return std::min<uint64_t>(len, slice - in);
  }
};

// ---- staged transfers ---------------------------------------------------------
// A host range that is not (yet) cudaHostRegister-ed — the segment a restarted
// trainer has just attached to, or a brand-new one whose registration (3-6 s for
// 16 GB) has been moved to the background — is moved through pinned bounce slots:
// T host threads, each with its own stream and two slots, memcpy between the
// segment and a slot while the DMA of their other slot is in flight.  The
// reference does the same thing implicitly (a pageable cudaMemcpy is staged by the
// driver through one small pinned buffer, 11-18 GB/s); this reaches PCIe speed.
struct StagePiece {
  uint8_t* dev;
  uint8_t* host;
  uint64_t len;
  uint64_t foff;  // offset in the files' virtual concatenation (StageFile), else unused
};

// Cuts every segment into slot-sized pieces, and at every offset of `cuts` (sorted; the
// file boundaries of a multi-file source).  host == nullptr: the segments' offsets are
// file offsets.
static std::vector<StagePiece> stage_pieces(const std::vector<Seg>& segs, uint8_t* host,
                                            uint64_t slot,
                                            const std::vector<uint64_t>* cuts = nullptr) {
  std::vector<StagePiece> out;
  for (const Seg& g : segs)
    for (uint64_t o = 0, len = 0; o < g.len; o += len) {
      len = std::min<uint64_t>(slot, g.len - o);
      if (cuts) {
        auto it = std::upper_bound(cuts->begin(), cuts->end(), g.off + o);
        if (it != cuts->end()) len = std::min<uint64_t>(len, *it - (g.off + o));
      }
      out.push_back({g.dev + o, host ? host + g.off + o : nullptr, len, g.off + o});
    }
  return out;
}

// Files as the source of a staged fill (fc_restore_files_async): the workers pread each
// piece's bytes into their slot instead of a memcpy from a host mapping.  The pieces'
// offsets lie in the virtual concatenation of the files: file k owns [bases[k],
// bases[k+1]), and no piece crosses a base.  The first short read or I/O error stops every
// worker and is remembered here.
struct StageFile {
  std::vector<int> fds;
  std::vector<uint64_t> bases;
  std::atomic<bool> failed{false};
  std::mutex mu;
  uint32_t bad_file = 0;  // index of the file that could not be read
  uint64_t bad_off = 0;   // offset in that file of the first byte that could not be read
  int err_no = 0;         // 0: end of file (short read)
  // the file holding virtual offset `off` (bases[0] <= off)
  uint32_t file_of(uint64_t off) const {
    return (uint32_t)(std::upper_bound(bases.begin(), bases.end(), off) - bases.begin() - 1);
  }
  bool read(uint8_t* dst, uint64_t len, uint64_t off) {
    const uint32_t k = file_of(off);
    off -= bases[k];
    for (uint64_t got = 0; got < len;) {
      const ssize_t r = pread(fds[k], dst + got, len - got, (off_t)(off + got));
      if (r > 0) {
        got += (uint64_t)r;
        continue;
      }
      if (r < 0 && errno == EINTR) continue;
      std::lock_guard<std::mutex> lk(mu);
      if (!failed.load()) {
        bad_file = k;
        bad_off = off + got;
        err_no = r < 0 ? errno : 0;
        failed.store(true);
      }
      return false;
    }
    return true;
  }
};

// Prefix of the errors about file k of an n-file restore: the one-file call names no index.
static void file_who(char* out, size_t cap, size_t n, uint32_t k) {
  if (n == 1)
    snprintf(out, cap, "fc_restore_file_async");
  else
    snprintf(out, cap, "fc_restore_files_async: file %u", k);
}

static cudaError_t stage_worker_init(fc_ctx* c, fc_ctx::StageWorker& w) {
  cudaError_t e = cudaSuccess;
  if (!w.stream) e = cudaStreamCreateWithFlags(&w.stream, cudaStreamNonBlocking);
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    if (!w.slot[i]) e = cudaHostAlloc((void**)&w.slot[i], c->stage_slot, cudaHostAllocDefault);
    if (e == cudaSuccess && !w.ev[i])
      e = cudaEventCreateWithFlags(&w.ev[i], cudaEventDisableTiming | cudaEventBlockingSync);
  }
  return e;
}

// to_host=false: host -> slot (memcpy, or pread from `file`) -> device (DMA).  true: the
// inverse.
static void stage_worker(fc_ctx* c, int wi, const std::vector<StagePiece>* pieces,
                         std::atomic<size_t>* next, bool to_host, cudaEvent_t gate,
                         std::atomic<int>* err, StageFile* file) {
  cudaSetDevice(c->device);
  fc_ctx::StageWorker& w = c->stage[wi];
  cudaError_t e = stage_worker_init(c, w);
  if (e == cudaSuccess && gate) e = cudaStreamWaitEvent(w.stream, gate, 0);
  const size_t n = pieces->size();
  if (!to_host) {
    bool used[2] = {false, false};
    for (int j = 0; e == cudaSuccess; ++j) {
      const size_t i = next->fetch_add(1);
      if (i >= n) break;
      const StagePiece& pc = (*pieces)[i];
      const int sl = j & 1;
      if (used[sl]) e = cudaEventSynchronize(w.ev[sl]);  // the DMA out of this slot is done
      if (e != cudaSuccess) break;
      if (file) {
        if (file->failed.load() || !file->read(w.slot[sl], pc.len, pc.foff)) break;
      } else {
        memcpy(w.slot[sl], pc.host, pc.len);
      }
      e = cudaMemcpyAsync(pc.dev, w.slot[sl], pc.len, cudaMemcpyHostToDevice, w.stream);
      if (e == cudaSuccess) e = cudaEventRecord(w.ev[sl], w.stream);
      used[sl] = true;
    }
  } else {
    // software pipeline: the DMA of piece n+1 runs while piece n is copied out
    size_t cur = next->fetch_add(1);
    int sl = 0;
    if (cur < n && e == cudaSuccess) {
      e = cudaMemcpyAsync(w.slot[0], (*pieces)[cur].dev, (*pieces)[cur].len,
                          cudaMemcpyDeviceToHost, w.stream);
      if (e == cudaSuccess) e = cudaEventRecord(w.ev[0], w.stream);
    }
    while (cur < n && e == cudaSuccess) {
      const size_t nxt = next->fetch_add(1);
      if (nxt < n) {
        e = cudaMemcpyAsync(w.slot[sl ^ 1], (*pieces)[nxt].dev, (*pieces)[nxt].len,
                            cudaMemcpyDeviceToHost, w.stream);
        if (e == cudaSuccess) e = cudaEventRecord(w.ev[sl ^ 1], w.stream);
      }
      if (e == cudaSuccess) e = cudaEventSynchronize(w.ev[sl]);
      if (e != cudaSuccess) break;
      memcpy((*pieces)[cur].host, w.slot[sl], (*pieces)[cur].len);
      cur = nxt;
      sl ^= 1;
    }
  }
  if (w.stream) {
    cudaError_t e2 = cudaStreamSynchronize(w.stream);
    if (e == cudaSuccess) e = e2;
  }
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    err->store((int)e);
  }
}

// Runs the pieces over `threads` workers (the caller is one of them); blocks.  With a
// `file`, the caller checks file->failed as well: an I/O error is no CUDA error.
static cudaError_t stage_run(fc_ctx* c, const std::vector<StagePiece>& pieces, bool to_host,
                             cudaEvent_t gate, int threads, StageFile* file = nullptr) {
  if (pieces.empty()) return cudaSuccess;
  int nt = std::max(1, std::min(threads, 32));
  nt = (int)std::min<size_t>((size_t)nt, pieces.size());
  if ((int)c->stage.size() < nt) c->stage.resize(nt);
  std::atomic<size_t> next{0};
  std::atomic<int> err{0};
  std::vector<std::thread> th;
  for (int i = 1; i < nt; ++i)
    th.emplace_back(stage_worker, c, i, &pieces, &next, to_host, gate, &err, file);
  stage_worker(c, 0, &pieces, &next, to_host, gate, &err, file);
  for (auto& t : th) t.join();
  return (cudaError_t)err.load();
}

// Incremental save: fetch the dirty marks once the gather-compare kernels are done and
// turn the items marked job.seq into runs, merged where both the arena and the segment
// continue.  Item i lies inside one plan run, which maps its arena offset to the segment.
static cudaError_t delta_runs(fc_ctx* c, fc_ctx::DrainJob& job) {
  const DeltaMap& m = *job.delta;
  const size_t n = m.aoff.size();
  job.runs.clear();
  if (n == 0) return cudaSuccess;
  cudaError_t e = cudaMemcpyAsync(c->dirty_pinned, c->dirty, n * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost, c->copy_stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->copy_stream);
  if (e != cudaSuccess) return e;
  size_t r = 0;
  for (size_t i = 0; i < n; ++i) {
    if (c->dirty_pinned[i] != job.seq) continue;
    while (m.runs[r].off + m.runs[r].len <= m.aoff[i]) ++r;
    const uint64_t hoff = m.runs[r].hoff + (m.aoff[i] - m.runs[r].off);
    uint8_t* dev = c->arena + m.aoff[i];
    if (!job.runs.empty()) {
      Seg& last = job.runs.back();
      if (last.dev + last.len == dev && last.off + last.len == hoff) {
        last.len += m.len[i];
        continue;
      }
    }
    job.runs.push_back({dev, hoff, m.len[i]});
  }
  return cudaSuccess;
}

// Calls put(host destination, device source, length) for every piece of segs: at most
// drain_piece bytes, never across a slice boundary of the host range.  Stops at the first
// error.
template <class Put>
static cudaError_t for_pieces(fc_ctx* c, uint8_t* host, const std::vector<Seg>& segs,
                              const SliceClip& clip, Put put) {
  cudaError_t e = cudaSuccess;
  for (const Seg& g : segs)
    for (uint64_t o = 0, len = 0; o < g.len && e == cudaSuccess; o += len) {
      len = clip(host + g.off + o, std::min<uint64_t>(c->drain_piece, g.len - o));
      e = put(host + g.off + o, g.dev + o, len);
    }
  return e;
}

// The in-place part: one batch (<= drain_piece bytes, <= 64 copies) in flight, then wait:
// the pacing rule of the arena part, and small tensors share a batch.
static cudaError_t drain_spans(fc_ctx* c, uint8_t* host, const std::vector<Seg>& segs,
                               const SliceClip& clip, uint64_t* copies) {
  uint64_t batch_bytes = 0;
  int batch_n = 0;
  auto flush = [&] {
    batch_bytes = 0;
    batch_n = 0;
    cudaError_t e = cudaEventRecord(c->ring[0], c->copy_stream);
    return e == cudaSuccess ? cudaEventSynchronize(c->ring[0]) : e;
  };
  auto put = [&](uint8_t* dst, const uint8_t* src, uint64_t len) {
    cudaError_t e = cudaMemcpyAsync(dst, src, len, cudaMemcpyDeviceToHost, c->copy_stream);
    ++*copies;
    batch_bytes += len;
    if (e == cudaSuccess && (batch_bytes >= c->drain_piece || ++batch_n >= 64)) e = flush();
    return e;
  };
  cudaError_t e = for_pieces(c, host, segs, clip, put);
  if (e == cudaSuccess && batch_bytes) e = flush();
  return e;
}

// The arena part: host-paced (piece k is submitted once piece k - drain_depth has
// completed) or chained on the device (ping-pong mode).  On return copy_stream is ordered
// after the last piece.
static cudaError_t drain_runs(fc_ctx* c, uint8_t* host, const std::vector<Seg>& segs,
                              const SliceClip& clip, uint64_t* copies) {
  const int depth = std::max(1, std::min(c->drain_depth, kDrainRing));
  const bool pingpong = c->drain_mode == FC_DRAIN_PINGPONG && c->copy_stream2 != nullptr;
  cudaStream_t last_stream = c->copy_stream;
  uint64_t k = 0;
  auto put = [&](uint8_t* dst, const uint8_t* src, uint64_t len) {
    cudaError_t e = cudaSuccess;
    if (pingpong) {
      // Piece k goes to stream k&1 and waits ON THE DEVICE for piece k-1 (the other
      // stream): neither stream ever has a second copy queued behind the one in
      // flight, so the copy engine arbitrates between our next piece and a
      // foreign copy after every piece — and there is no host round trip between
      // two pieces.  The host only keeps two pieces submitted.
      cudaStream_t sk = (k & 1) ? c->copy_stream2 : c->copy_stream;
      if (k >= 2) e = cudaEventSynchronize(c->ring_pp[(k - 2) % kDrainRing]);
      if (e == cudaSuccess && k >= 1)
        e = cudaStreamWaitEvent(sk, c->ring_pp[(k - 1) % kDrainRing], 0);
      if (e == cudaSuccess) e = cudaMemcpyAsync(dst, src, len, cudaMemcpyDeviceToHost, sk);
      if (e == cudaSuccess) e = cudaEventRecord(c->ring_pp[k % kDrainRing], sk);
      last_stream = sk;
    } else {
      if (k >= (uint64_t)depth) e = cudaEventSynchronize(c->ring[k % depth]);  // piece k-depth
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(dst, src, len, cudaMemcpyDeviceToHost, c->copy_stream);
      if (e == cudaSuccess) e = cudaEventRecord(c->ring[k % depth], c->copy_stream);
    }
    ++k;
    ++*copies;
    return e;
  };
  cudaError_t e = for_pieces(c, host, segs, clip, put);
  if (e == cudaSuccess && last_stream != c->copy_stream)
    e = cudaStreamWaitEvent(c->copy_stream, c->ring_pp[(k - 1) % kDrainRing], 0);
  return e;
}

// One part of a drain job: through the bounce slots when the host range is not
// page-locked, else by DMA under the part's pacing rule (drain_spans or drain_runs).
using DmaDrain = cudaError_t (*)(fc_ctx*, uint8_t*, const std::vector<Seg>&, const SliceClip&,
                                 uint64_t*);
static cudaError_t drain_part(fc_ctx* c, const fc_ctx::DrainJob& job, const std::vector<Seg>& segs,
                              DmaDrain dma, uint64_t* copies) {
  if (job.staged_threads > 0) {
    const std::vector<StagePiece> pieces = stage_pieces(segs, job.host, c->stage_slot);
    *copies += pieces.size();
    return stage_run(c, pieces, true, c->ev_pack_end, job.staged_threads);
  }
  // a range registered slice by slice: no DMA may straddle two slices
  const SliceClip clip(c, job.host + (segs.empty() ? 0 : segs.front().off));
  return dma(c, job.host, segs, clip, copies);
}

// Drains one save once its gather has completed: the in-place part first (then the
// tensors are free again), then the arena part; ev_drain_start / ev_drain_end bracket it.
static cudaError_t drain_job(fc_ctx* c, fc_ctx::DrainJob& job, uint64_t* copies) {
  cudaError_t e = cudaStreamWaitEvent(c->copy_stream, c->ev_pack_end, 0);
  if (e == cudaSuccess) e = cudaEventRecord(c->ev_drain_start, c->copy_stream);
  if (job.delta && e == cudaSuccess) e = delta_runs(c, job);
  if (e == cudaSuccess) e = drain_part(c, job, job.spans, drain_spans, copies);
  if (job.direct) {
    {
      // the tensors are free again (on error too: nothing reads them any more)
      std::lock_guard<std::mutex> lk(c->mu);
      c->inplace_done_ticket = job.ticket;
    }
    c->cv.notify_all();
  }
  if (e == cudaSuccess) e = drain_part(c, job, job.runs, drain_runs, copies);
  if (e == cudaSuccess) e = cudaEventRecord(c->ev_drain_end, c->copy_stream);
  if (e == cudaSuccess) e = cudaEventSynchronize(c->ev_drain_end);
  return e;
}

static void pump_main(fc_ctx* c) {
  cudaSetDevice(c->device);
  for (;;) {
    fc_ctx::DrainJob job;
    {
      std::unique_lock<std::mutex> lk(c->mu);
      c->cv.wait(lk, [&] {
        return c->pump_stop || (!c->jobs.empty() && c->jobs.front().ticket != c->held_ticket);
      });
      if (c->jobs.empty()) return;  // stop requested and nothing queued
      if (c->jobs.front().ticket == c->held_ticket) c->held_ticket = 0;  // stopping: drain anyway
      job = std::move(c->jobs.front());
      c->jobs.pop_front();
    }
    uint64_t copies = 0;
    const cudaError_t e = drain_job(c, job, &copies);
    uint64_t drained = 0;
    for (const Seg& g : job.spans) drained += g.len;
    for (const Seg& g : job.runs) drained += g.len;
    {
      std::lock_guard<std::mutex> lk(c->mu);
      c->n_memcpys += copies;
      if (e != cudaSuccess) {
        c->drain_rc = FC_ECUDA;
        c->drain_err = std::string("drain pump: ") + cudaGetErrorString(e);
        (void)cudaGetLastError();
        delta_forget_locked(c);
      } else {
        // the segment now holds the arena's image of this plan
        if (job.ticket == c->base_ticket) c->base_valid = true;
        if (job.ticket == c->img_ticket) c->img_valid = true;
      }
      c->stat_ticket = job.ticket;
      c->stat_bytes = drained;
      c->stat_delta = job.delta ? 1 : 0;
      c->drained_ticket = job.ticket;
    }
    c->cv.notify_all();
  }
}

// One device-resident work table + its pinned staging copy (grow-only).
struct FcTable {
  FcItem* dev = nullptr;
  FcItem* pinned = nullptr;
  uint32_t cap = 0;
  uint32_t n = 0;
};

struct fc_plan {
  fc_ctx* ctx = nullptr;
  FcTable all;    // every byte, <= chunk pieces (LSU variant)
  FcTable bulk;   // 16-B congruent bodies (TMA variant)
  FcTable resid;  // heads and tails of congruent ranges (TMA variant)
  FcTable shift;  // ranges not congruent mod 16 (TMA variant: fc_copy_tma_shift)
  uint64_t payload = 0, arena_end = 0;
  // extent of the plan in the host segment; identity: segment offset == arena offset for
  // every range (the arena is a byte image of the segment).  A compacting plan
  // (fc_plan_create_mapped) packs ranges that are scattered over the segment into a
  // small arena; hybrid / bounded-arena saves need the identity.
  uint64_t host_lo = 0, host_hi = 0;
  bool identity = true;
  uint32_t chunk = kDefaultChunk;
  std::vector<FcRun> runs;
  std::vector<FcItem> h_all;  // host copy of `all`, ascending arena offset
  // bulk/resid/shift are derived from `all` item by item, in the same (ascending
  // offset) order: pos_x[i] = number of x-items derived from all[0..i), so the
  // item range [i0,i1) of `all` is bulk[pos_bulk[i0]..pos_bulk[i1]) etc.  Hybrid
  // and windowed saves launch the TMA kernels over such slices.
  std::vector<uint32_t> pos_bulk, pos_resid, pos_shift;
  std::vector<FcSpan> spans;  // source ranges by arena offset (in-place save / restore)
  std::shared_ptr<const DeltaMap> dmap;  // item extents + runs for the incremental drain
  cudaEvent_t ev_upload = nullptr;  // last table upload
  cudaEvent_t ev_last_use = nullptr;  // last kernel that read the tables
  // non-finite scan: the input ranges as given (empty ones included), one kind byte
  // each, the scan's own item table (rebuilt on the next scan after a create / update /
  // kind change) and its result buffers (n uint32 counts + a uint64 total)
  std::vector<FcSpan> inputs;  // tptr, len (off unused)
  std::vector<uint8_t> kinds;
  FcTable scan;
  bool scan_stale = true;
  bool scan_enqueued = false;
  uint8_t* scan_dev = nullptr;
  uint8_t* scan_host = nullptr;
  size_t scan_cap = 0;
  cudaEvent_t ev_scan = nullptr;  // the last scan's result has reached scan_host
};

static void image_expect_locked(fc_ctx* c, const fc_plan* p, const uint8_t* host,
                                uint64_t ticket) {
  c->img_map = p->dmap;
  c->img_plan = p;
  c->img_host = host;
  c->img_valid = false;
  c->img_ticket = ticket;
}

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) ok = cudaSetDevice(dev) == cudaSuccess;
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};

#define FC_GUARD(ctx)                                                      \
  DeviceGuard _guard((ctx)->device);                                       \
  if (!_guard.ok) return fail(FC_ECUDA, "cudaSetDevice failed%s%s")

extern "C" int fc_ctx_create(int device, fc_ctx** out) {
  if (!out || device < 0) return fail(FC_EINVAL, "fc_ctx_create: bad argument%s%s");
  fc_ctx* c = new (std::nothrow) fc_ctx();
  if (!c) return fail(FC_ENOMEM, "fc_ctx_create: host alloc%s%s");
  c->device = device;
  DeviceGuard g(device);
  if (!g.ok) {
    delete c;
    return fail(FC_ECUDA, "cudaSetDevice failed%s%s");
  }
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) {
    delete c;
    return fail(FC_ECUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
  }
  c->sm_count = prop.multiProcessorCount;
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  e = cudaStreamCreateWithPriority(&c->copy_stream, cudaStreamNonBlocking, hi);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&c->copy_stream2, cudaStreamNonBlocking, hi);
  cudaEvent_t* evs[] = {&c->ev_pack_start, &c->ev_pack_end,  &c->ev_drain_start, &c->ev_drain_end,
                        &c->ev_fill_start, &c->ev_fill_end,  &c->ev_scatter_end};
  for (cudaEvent_t* ev : evs)
    if (e == cudaSuccess) e = cudaEventCreate(ev);
  // The host-paced pump waits for piece k before it submits piece k+1, so its wake-up
  // latency is on the critical path: a spinning wait drains faster than a blocking one.
  // Spinning costs one busy
  // host core while a checkpoint drains (~0.3 s) — nothing on a 128-core GPU host, a lot
  // in an 8-vCPU container.  Default: spin when the machine has more than 16 hardware
  // threads; otherwise sleep in a blocking wait AND chain the pieces on the device
  // (ping-pong mode: no host round trip between pieces).
  // FC_DRAIN_SPIN=0/1 and FC_DRAIN_MODE=0/1 override.
  const char* spin_env = getenv("FC_DRAIN_SPIN");
  const bool many_cores = std::thread::hardware_concurrency() > 16;
  const bool drain_spin = spin_env ? spin_env[0] != '0' : many_cores;
  if (!drain_spin) c->drain_mode = FC_DRAIN_PINGPONG;
  for (int i = 0; i < kDrainRing; ++i)
    if (e == cudaSuccess)
      e = cudaEventCreateWithFlags(
          &c->ring[i], cudaEventDisableTiming | (drain_spin ? 0 : cudaEventBlockingSync));
  for (int i = 0; i < kDrainRing; ++i)
    if (e == cudaSuccess)
      e = cudaEventCreateWithFlags(&c->ring_pp[i], cudaEventDisableTiming | cudaEventBlockingSync);
  if (const char* m = getenv("FC_DRAIN_MODE")) c->drain_mode = atoi(m) ? FC_DRAIN_PINGPONG : FC_DRAIN_HOST_PACED;
  if (e != cudaSuccess) {
    fc_ctx_destroy(c);
    return fail(FC_ECUDA, "fc_ctx_create: %s", cudaGetErrorString(e));
  }
  *out = c;
  return FC_OK;
}

extern "C" int fc_ctx_destroy(fc_ctx* c) {
  if (!c) return FC_OK;
  DeviceGuard g(c->device);
  if (c->pump.joinable()) {
    {
      std::lock_guard<std::mutex> lk(c->mu);
      c->pump_stop = true;
    }
    c->cv.notify_all();
    c->pump.join();
  }
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  if (c->copy_stream2) cudaStreamSynchronize(c->copy_stream2);
  for (int i = 0; i < kDrainRing; ++i) {
    if (c->ring[i]) cudaEventDestroy(c->ring[i]);
    if (c->ring_pp[i]) cudaEventDestroy(c->ring_pp[i]);
  }
  for (auto& r : c->regs) {
    r->cancel = true;
    if (r->th.joinable()) r->th.join();
    for (void* q : r->done) cudaHostUnregister(q);
  }
  c->regs.clear();
  for (auto& w : c->stage) {
    if (w.stream) cudaStreamSynchronize(w.stream);
    for (int i = 0; i < 2; ++i) {
      if (w.ev[i]) cudaEventDestroy(w.ev[i]);
      if (w.slot[i]) cudaFreeHost(w.slot[i]);
    }
    if (w.stream) cudaStreamDestroy(w.stream);
  }
  c->stage.clear();
  cudaEvent_t evs[] = {c->ev_pack_start, c->ev_pack_end, c->ev_drain_start, c->ev_drain_end,
                       c->ev_fill_start, c->ev_fill_end, c->ev_scatter_end};
  for (cudaEvent_t ev : evs)
    if (ev) cudaEventDestroy(ev);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->copy_stream2) cudaStreamDestroy(c->copy_stream2);
  if (c->arena) cudaFree(c->arena);
  if (c->dirty) cudaFree(c->dirty);
  if (c->dirty_pinned) cudaFreeHost(c->dirty_pinned);
  for (void* q : c->dead_dev) cudaFree(q);
  for (void* q : c->dead_pinned) cudaFreeHost(q);
  delete c;
  return FC_OK;
}

static int refresh_inflight(fc_ctx* c) {
  if (c->save_inflight) {
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->drained_ticket >= c->ticket) c->save_inflight = false;
  }
  if (c->restore_inflight) {
    cudaError_t e = cudaEventQuery(c->ev_scatter_end);
    if (e == cudaSuccess)
      c->restore_inflight = false;
    else if (e != cudaErrorNotReady)
      return fail(FC_ECUDA, "cudaEventQuery(scatter): %s", cudaGetErrorString(e));
  }
  return FC_OK;
}

extern "C" int fc_arena_reserve(fc_ctx* c, uint64_t bytes) {
  if (!c) return fail(FC_EINVAL, "fc_arena_reserve: null ctx%s%s");
  FC_GUARD(c);
  if (c->arena_cap && bytes > c->arena_cap) bytes = c->arena_cap;
  if (bytes <= c->arena_bytes) return FC_OK;
  int rc = refresh_inflight(c);
  if (rc) return rc;
  if (c->save_inflight || c->restore_inflight)
    return fail(FC_EBUSY, "fc_arena_reserve: arena in use%s%s");
  delta_forget(c);  // the new arena holds no image of the segment
  if (c->arena) {
    FC_CUDA(cudaFree(c->arena));
    c->arena = nullptr;
    c->arena_bytes = 0;
  }
  for (void* q : c->dead_dev) cudaFree(q);  // cudaFree above synchronised already
  for (void* q : c->dead_pinned) cudaFreeHost(q);
  c->dead_dev.clear();
  c->dead_pinned.clear();
  // +32: the shifted load path may read one aligned 16-B word past the end.
  uint64_t want = ((bytes + 32 + 511) / 512) * 512;
  cudaError_t e = cudaMalloc(&c->arena, want);
  if (e != cudaSuccess) {
    c->arena = nullptr;
    (void)cudaGetLastError();
    return fail(FC_ENOMEM, "cudaMalloc(arena): %s", cudaGetErrorString(e));
  }
  c->arena_bytes = bytes;
  return FC_OK;
}

extern "C" int fc_set_arena_limit(fc_ctx* c, uint64_t bytes) {
  if (!c) return fail(FC_EINVAL, "fc_set_arena_limit: null ctx%s%s");
  if (bytes && bytes < (8ull << 20))
    return fail(FC_EINVAL, "fc_set_arena_limit: at least 8 MiB%s%s");
  c->arena_cap = bytes;
  return FC_OK;
}

extern "C" int fc_arena_info(fc_ctx* c, void** dev_ptr, uint64_t* bytes) {
  if (!c) return fail(FC_EINVAL, "fc_arena_info: null ctx%s%s");
  if (dev_ptr) *dev_ptr = c->arena;
  if (bytes) *bytes = c->arena_bytes;
  return FC_OK;
}

// NUMA node the GPU's PCIe root hangs off (-1 if unknown / single node).
static int gpu_numa_node(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) {
    (void)cudaGetLastError();
    return -1;
  }
  for (char* q = bus; *q; ++q)
    if (*q >= 'A' && *q <= 'Z') *q = (char)(*q - 'A' + 'a');
  char path[128];
  snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
  FILE* f = fopen(path, "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}

// Ask the kernel to back [host, host+bytes) with pages of `node` (the DMA
// target should be local to the GPU's socket: with 8 ranks draining at once
// the inter-socket link would otherwise carry half of the 440 GB/s).  Applies
// to pages not faulted in yet; best effort, failures are ignored.
static void mbind_preferred(uintptr_t lo, uintptr_t hi, int node) {
#if defined(SYS_mbind)
  if (node < 0 || node >= 1024 || hi <= lo) return;
  unsigned long mask[16] = {0};
  mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
  const int kMpolPreferred = 1;
  (void)syscall(SYS_mbind, (void*)lo, (unsigned long)(hi - lo), kMpolPreferred, mask,
                (unsigned long)(8 * sizeof(mask)), 0u);
#else
  (void)lo; (void)hi; (void)node;
#endif
}

// remote_per256 > 0: of every 256 consecutive 2-MiB blocks that many (spread evenly)
// are bound to `remote` instead of `node` — when more GPUs of one socket drain at
// once than its memory controllers absorb and the other socket is idle, a share of
// the DMA writes goes over the inter-socket link.
static void prefer_numa_node(void* host, uint64_t bytes, int node, int remote = -1,
                             int remote_per256 = 0) {
  if (node < 0) return;
  const uintptr_t pg = (uintptr_t)sysconf(_SC_PAGESIZE);
  const uintptr_t lo = (uintptr_t)host & ~(pg - 1);
  const uintptr_t hi = ((uintptr_t)host + bytes + pg - 1) & ~(pg - 1);
  mbind_preferred(lo, hi, node);
  if (remote < 0 || remote == node || remote_per256 <= 0) return;
  if (remote_per256 > 256) remote_per256 = 256;
  const uintptr_t blk = 2ull << 20;
  // block k is remote iff floor((k+1)*r/256) > floor(k*r/256): evenly spread;
  // indexed from the block number of the ADDRESS so sub-ranges registered by
  // different processes agree on the pattern
  for (uintptr_t a = lo & ~(blk - 1); a < hi; a += blk) {
    const uint64_t k = (uint64_t)(a / blk);
    if (((k + 1) * (uint64_t)remote_per256) / 256 > (k * (uint64_t)remote_per256) / 256)
      mbind_preferred(std::max(a, lo), std::min(a + blk, hi), remote);
  }
}

static int numa_node_count() {
  int n = 0;
  char path[96];
  for (; n < 64; ++n) {
    snprintf(path, sizeof(path), "/sys/devices/system/node/node%d", n);
    if (access(path, F_OK) != 0) break;
  }
  return n;
}

extern "C" int fc_device_numa_node(int device, int* node, int* n_nodes) {
  if (node) *node = gpu_numa_node(device);
  if (n_nodes) *n_nodes = numa_node_count();
  return FC_OK;
}

extern "C" int fc_host_bind_numa(fc_ctx* c, void* host, uint64_t bytes, int remote_per256) {
  if (!c || !host || bytes == 0) return fail(FC_EINVAL, "fc_host_bind_numa: bad argument%s%s");
  if (getenv("FC_NO_NUMA")) return FC_OK;
  const int node = gpu_numa_node(c->device);
  const int nn = numa_node_count();
  int remote = -1;
  if (remote_per256 > 0 && node >= 0 && nn == 2) remote = 1 - node;
  prefer_numa_node(host, bytes, node, remote, remote_per256);
  return FC_OK;
}

struct PrefaultJob {
  uint8_t* p;
  size_t n;
};

static void* prefault_worker(void* arg) {
  PrefaultJob* j = static_cast<PrefaultJob*>(arg);
#ifdef MADV_POPULATE_WRITE
  if (madvise(j->p, j->n, MADV_POPULATE_WRITE) == 0) return nullptr;
#endif
  // Fallback: read-touch every page (never modifies an attached segment).
  const long pg = sysconf(_SC_PAGESIZE);
  volatile uint8_t sink = 0;
  for (size_t o = 0; o < j->n; o += (size_t)pg) sink ^= j->p[o];
  (void)sink;
  return nullptr;
}

static void prefault_range(void* host, uint64_t bytes, int prefault_threads) {
  const long pg = sysconf(_SC_PAGESIZE);
  int nt = std::max(1, std::min(prefault_threads, 64));
  uint64_t per = ((bytes / nt + pg - 1) / pg) * pg;
  if (per == 0) per = pg;
  std::vector<pthread_t> th;
  std::vector<PrefaultJob> jobs;
  jobs.reserve(nt);
  // mmap'd segments are page aligned; tolerate an unaligned start anyway
  uint8_t* base = static_cast<uint8_t*>(host);
  for (uint64_t o = 0; o < bytes; o += per)
    jobs.push_back({base + o, (size_t)std::min<uint64_t>(per, bytes - o)});
  th.resize(jobs.size());
  for (size_t i = 0; i < jobs.size(); ++i)
    if (pthread_create(&th[i], nullptr, prefault_worker, &jobs[i]) != 0) {
      prefault_worker(&jobs[i]);
      th[i] = 0;
    }
  for (size_t i = 0; i < jobs.size(); ++i)
    if (th[i]) pthread_join(th[i], nullptr);
}

static fc_ctx::HostReg* find_reg(fc_ctx* c, const void* host) {
  for (auto& r : c->regs)
    if (r->base == host) return r.get();
  return nullptr;
}

// The registration covering [p, p+len), or nullptr.
static fc_ctx::HostReg* reg_covering(fc_ctx* c, const uint8_t* p, uint64_t len) {
  for (auto& r : c->regs)
    if (p >= r->base && p + len <= r->base + r->bytes) return r.get();
  return nullptr;
}

static bool is_pinned_host(const void* q) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, q) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeHost;
}

// 0 when [p, p+len) is page-locked for CUDA (a completed fc_host_register*, or memory
// the caller pinned itself, e.g. cudaHostAlloc): plain DMA.  Else the number of host
// threads the staged path should use.
static int staged_threads_for(fc_ctx* c, const uint8_t* p, uint64_t len) {
  if (len == 0 || getenv("FC_NO_STAGING")) return 0;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    for (auto& r : c->regs) {
      const bool overlaps = p < r->base + r->bytes && r->base < p + len;
      if (overlaps && r->state != 1) return std::max(1, c->stage_threads);  // still pinning
    }
  }
  if (is_pinned_host(p) && is_pinned_host(p + len - 1)) return 0;
  return std::max(1, c->stage_threads);
}

static void register_slices(fc_ctx* c, fc_ctx::HostReg* r) {
  cudaSetDevice(c->device);
  for (uint64_t o = 0; o < r->bytes && !r->cancel; o += r->slice) {
    const uint64_t len = std::min<uint64_t>(r->slice, r->bytes - o);
    cudaError_t e = cudaHostRegister(r->base + o, len, cudaHostRegisterPortable);
    if (e == cudaErrorHostMemoryAlreadyRegistered) {
      (void)cudaGetLastError();
      continue;
    }
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      r->state = -1;
      return;
    }
    {
      std::lock_guard<std::mutex> lk(c->mu);
      r->done.push_back(r->base + o);
    }
    // cudaHostRegister holds a driver lock every other CUDA call of the process needs
    // (measured: a kernel launch issued during a 16 GB registration waits for all of
    // it, 0.87 s): give the training thread a window after every slice
    usleep(500);
  }
  if (!r->cancel) r->state = 1;
}

static void madvise_hugepage(void* host, uint64_t bytes) {
#ifdef MADV_HUGEPAGE
  // 2 MiB pages where the host allows them for this mapping (tmpfs: only with
  // transparent_hugepage/shmem_enabled = advise|always): fewer IOMMU / page-table
  // entries under the DMA.  Advice only; a refusal changes nothing.
  if (!getenv("FC_NO_HUGEPAGE")) {
    const uintptr_t pg = (uintptr_t)sysconf(_SC_PAGESIZE);
    uintptr_t lo = ((uintptr_t)host + pg - 1) & ~(pg - 1);
    uintptr_t hi = ((uintptr_t)host + bytes) & ~(pg - 1);
    if (hi > lo) (void)madvise((void*)lo, hi - lo, MADV_HUGEPAGE);
  }
#else
  (void)host; (void)bytes;
#endif
}

extern "C" int fc_host_register(fc_ctx* c, void* host, uint64_t bytes, int prefault_threads) {
  if (!c || !host || bytes == 0) return fail(FC_EINVAL, "fc_host_register: bad argument%s%s");
  FC_GUARD(c);
  if (fc_ctx::HostReg* old = find_reg(c, host)) {
    if (old->th.joinable()) old->th.join();  // a background registration: let it finish
    if (old->state == 1 && old->bytes >= bytes) return FC_OK;
    return fail(FC_EINVAL, "fc_host_register: range already known with another size%s%s");
  }
  if (!getenv("FC_NO_NUMA")) prefer_numa_node(host, bytes, gpu_numa_node(c->device));
  madvise_hugepage(host, bytes);
  if (prefault_threads > 0) prefault_range(host, bytes, prefault_threads);
  cudaError_t e = cudaHostRegister(host, bytes, cudaHostRegisterPortable);
  if (e == cudaErrorHostMemoryAlreadyRegistered) {
    (void)cudaGetLastError();
    return FC_OK;
  }
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(FC_ECUDA, "cudaHostRegister: %s", cudaGetErrorString(e));
  }
  std::unique_ptr<fc_ctx::HostReg> r(new fc_ctx::HostReg());
  r->base = static_cast<uint8_t*>(host);
  r->bytes = bytes;
  r->done.push_back(host);
  r->state = 1;
  std::lock_guard<std::mutex> lk(c->mu);
  c->regs.push_back(std::move(r));
  return FC_OK;
}

extern "C" int fc_host_register_background(fc_ctx* c, void* host, uint64_t bytes,
                                           uint64_t slice_bytes) {
  if (!c || !host || bytes == 0)
    return fail(FC_EINVAL, "fc_host_register_background: bad argument%s%s");
  if (find_reg(c, host)) return FC_OK;  // known: in progress or done
  const uint64_t pg = (uint64_t)sysconf(_SC_PAGESIZE);
  if (slice_bytes == 0) slice_bytes = 256ull << 20;
  slice_bytes = std::max<uint64_t>((slice_bytes + pg - 1) / pg * pg, 2ull << 20);
  std::unique_ptr<fc_ctx::HostReg> r(new fc_ctx::HostReg());
  r->base = static_cast<uint8_t*>(host);
  r->bytes = bytes;
  r->slice = slice_bytes;
  fc_ctx::HostReg* raw = r.get();
  {
    std::lock_guard<std::mutex> lk(c->mu);
    c->regs.push_back(std::move(r));
  }
  raw->th = std::thread(register_slices, c, raw);
  return FC_OK;
}

extern "C" int fc_host_ready(fc_ctx* c, const void* host) {
  if (!c || !host) return fail(FC_EINVAL, "fc_host_ready: bad argument%s%s");
  fc_ctx::HostReg* r = find_reg(c, host);
  if (!r) return fail(FC_EINVAL, "fc_host_ready: unknown host range%s%s");
  const int st = r->state;
  if (st == 1) return FC_OK;
  if (st == 0) return FC_ENOTREADY;
  return fail(FC_ECUDA, "background cudaHostRegister failed%s%s");
}

extern "C" int fc_host_unregister(fc_ctx* c, void* host) {
  if (!c || !host) return fail(FC_EINVAL, "fc_host_unregister: bad argument%s%s");
  FC_GUARD(c);
  fc_ctx::HostReg* r = find_reg(c, host);
  if (!r) return FC_OK;
  r->cancel = true;
  if (r->th.joinable()) r->th.join();
  // no DMA may still target the range: let the pump finish, then the stream
  {
    std::unique_lock<std::mutex> lk(c->mu);
    c->cv.wait(lk, [&] { return c->drained_ticket >= c->ticket; });
  }
  FC_CUDA(cudaStreamSynchronize(c->copy_stream));
  if (c->copy_stream2) FC_CUDA(cudaStreamSynchronize(c->copy_stream2));
  cudaError_t first = cudaSuccess;
  for (void* q : r->done) {
    cudaError_t e = cudaHostUnregister(q);
    if (e != cudaSuccess && first == cudaSuccess) first = e;
  }
  {
    std::lock_guard<std::mutex> lk(c->mu);
    for (auto it = c->regs.begin(); it != c->regs.end(); ++it)
      if (it->get() == r) {
        c->regs.erase(it);
        break;
      }
  }
  if (first != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(FC_ECUDA, "cudaHostUnregister: %s", cudaGetErrorString(first));
  }
  return FC_OK;
}

// Split [off, off+n) so interior boundaries are 128-B aligned in arena space.
static void split_range(std::vector<FcItem>& out, uint64_t tptr, uint64_t off, uint64_t n,
                        uint32_t chunk) {
  uint64_t first = chunk - (off & 127u);
  while (n > 0) {
    uint64_t len = std::min<uint64_t>(n, first);
    FcItem it;
    it.tptr = tptr;
    it.aoff = off;
    it.nbytes = (uint32_t)len;
    it.pad0 = 0;
    it.pad1 = 0;
    out.push_back(it);
    tptr += len;
    off += len;
    n -= len;
    first = chunk;
  }
}

// Put `v` into table `t` (device copy ordered on `s`).  sync=true: blocking
// cudaMemcpy from the vector (plan creation).  sync=false: staged through the
// table's pinned buffer and cudaMemcpyAsync on `s`, never a device-wide sync.
static int table_set(fc_ctx* c, FcTable& t, const std::vector<FcItem>& v, cudaStream_t s,
                     bool sync) {
  t.n = (uint32_t)v.size();
  if (v.empty()) return FC_OK;
  if (v.size() > t.cap) {
    uint32_t cap = (uint32_t)std::min<uint64_t>(0xFFFFFFF0ull, v.size() + v.size() / 4 + 16);
    FcItem* nd = nullptr;
    FcItem* np = nullptr;
    cudaError_t e = cudaMalloc(&nd, (size_t)cap * sizeof(FcItem));
    if (e == cudaSuccess) e = cudaHostAlloc(&np, (size_t)cap * sizeof(FcItem), cudaHostAllocDefault);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      if (nd) c->dead_dev.push_back(nd);
      return fail(FC_ENOMEM, "plan table alloc: %s", cudaGetErrorString(e));
    }
    if (t.dev) c->dead_dev.push_back(t.dev);  // may still be read by a queued kernel
    if (t.pinned) c->dead_pinned.push_back(t.pinned);
    t.dev = nd;
    t.pinned = np;
    t.cap = cap;
  }
  const size_t bytes = v.size() * sizeof(FcItem);
  if (sync) {
    FC_CUDA(cudaMemcpy(t.dev, v.data(), bytes, cudaMemcpyHostToDevice));
  } else {
    memcpy(t.pinned, v.data(), bytes);
    FC_CUDA(cudaMemcpyAsync(t.dev, t.pinned, bytes, cudaMemcpyHostToDevice, s));
  }
  return FC_OK;
}

// (Re)build the plan's runs and work tables from n ranges.
static int plan_fill(fc_plan* p, uint32_t n, const void* const* dev_ptrs,
                     const uint64_t* arena_off, const uint64_t* nbytes, cudaStream_t s,
                     bool sync, const uint64_t* host_off = nullptr) {
  fc_ctx* c = p->ctx;
  const uint32_t chunk_bytes = p->chunk;
  uint64_t payload = 0, arena_end = 0, host_lo = ~0ull, host_hi = 0;
  bool identity = true;
  std::vector<FcRun> ranges, runs;
  std::vector<FcSpan> spans;
  ranges.reserve(n);
  spans.reserve(n);
  for (uint32_t i = 0; i < n; ++i) {
    if (nbytes[i] == 0) continue;
    if (!dev_ptrs[i])
      return fail(FC_EINVAL, "plan: null device pointer for a non-empty tensor%s%s");
    if (arena_off[i] + nbytes[i] < arena_off[i]) return fail(FC_EINVAL, "plan: offset overflow%s%s");
    const uint64_t hoff = host_off ? host_off[i] : arena_off[i];
    if (hoff + nbytes[i] < hoff) return fail(FC_EINVAL, "plan: offset overflow%s%s");
    ranges.push_back({arena_off[i], nbytes[i], hoff});
    spans.push_back({(uint64_t)(uintptr_t)dev_ptrs[i], hoff, nbytes[i]});
    payload += nbytes[i];
    arena_end = std::max(arena_end, arena_off[i] + nbytes[i]);
    host_lo = std::min(host_lo, hoff);
    host_hi = std::max(host_hi, hoff + nbytes[i]);
    if (hoff != arena_off[i]) identity = false;
  }
  if (ranges.empty()) host_lo = 0;
  std::sort(ranges.begin(), ranges.end(),
            [](const FcRun& a, const FcRun& b) { return a.off < b.off; });
  for (const FcRun& r : ranges) {
    if (!runs.empty()) {
      FcRun& last = runs.back();
      if (r.off < last.off + last.len)
        return fail(FC_EINVAL, "plan: tensors overlap in the arena%s%s");
      if (r.off == last.off + last.len && r.hoff == last.hoff + last.len) {
        last.len += r.len;
        continue;
      }
    }
    runs.push_back(r);
  }

  std::vector<FcItem> all, bulk, resid, shift;
  for (uint32_t i = 0; i < n; ++i) {
    if (nbytes[i] == 0) continue;
    split_range(all, (uint64_t)(uintptr_t)dev_ptrs[i], arena_off[i], nbytes[i], chunk_bytes);
  }
  if (all.size() > 0xFFFFFFF0ull) return fail(FC_EINVAL, "plan: too many work items%s%s");
  std::stable_sort(all.begin(), all.end(),
                   [](const FcItem& a, const FcItem& b) { return a.aoff < b.aoff; });
  // every item, and every piece derived from it below, carries the index of its `all`
  // entry: the gather-compare kernels mark dirty[pad0]; the copy kernels ignore it
  for (size_t k = 0; k < all.size(); ++k) all[k].pad0 = (uint32_t)k;
  // Derive the TMA-variant tables from `all`, item by item.  Interior item
  // boundaries are 128-B aligned in arena space, so a head (< 16 B) only exists at
  // the start of a range and a tail only at its end.
  std::vector<uint32_t> pos_bulk(all.size() + 1), pos_resid(all.size() + 1),
      pos_shift(all.size() + 1);
  for (size_t k = 0; k < all.size(); ++k) {
    pos_bulk[k] = (uint32_t)bulk.size();
    pos_resid[k] = (uint32_t)resid.size();
    pos_shift[k] = (uint32_t)shift.size();
    const FcItem& it = all[k];
    const uint64_t tp = it.tptr, off = it.aoff, nb = it.nbytes;
    if (((tp - off) & 15u) != 0) {  // not congruent mod 16: byte-shift path
      // pieces too small for a TMA tile go to the LSU kernel
      (nb < 4096 ? resid : shift).push_back(it);
      continue;
    }
    const uint64_t head = std::min<uint64_t>((16u - (off & 15u)) & 15u, nb);
    const uint64_t body = (nb - head) & ~15ull;
    const uint64_t tail = nb - head - body;
    FcItem piece = it;
    if (head) {
      piece.nbytes = (uint32_t)head;
      resid.push_back(piece);
    }
    if (body) {
      piece.tptr = tp + head;
      piece.aoff = off + head;
      piece.nbytes = (uint32_t)body;
      bulk.push_back(piece);
    }
    if (tail) {
      piece.tptr = tp + head + body;
      piece.aoff = off + head + body;
      piece.nbytes = (uint32_t)tail;
      resid.push_back(piece);
    }
  }
  pos_bulk[all.size()] = (uint32_t)bulk.size();
  pos_resid[all.size()] = (uint32_t)resid.size();
  pos_shift[all.size()] = (uint32_t)shift.size();
  int rc = table_set(c, p->all, all, s, sync);
  if (!rc) rc = table_set(c, p->bulk, bulk, s, sync);
  if (!rc) rc = table_set(c, p->resid, resid, s, sync);
  if (!rc) rc = table_set(c, p->shift, shift, s, sync);
  if (rc) return rc;
  p->payload = payload;
  p->arena_end = arena_end;
  p->host_lo = host_lo;
  p->host_hi = host_hi;
  p->identity = identity;
  if (!identity) {
    // host ranges must not overlap either
    std::vector<FcSpan> by_host(spans);
    std::sort(by_host.begin(), by_host.end(),
              [](const FcSpan& a, const FcSpan& b) { return a.off < b.off; });
    for (size_t i = 1; i < by_host.size(); ++i)
      if (by_host[i].off < by_host[i - 1].off + by_host[i - 1].len)
        return fail(FC_EINVAL, "plan: tensors overlap in the segment%s%s");
  }
  std::shared_ptr<DeltaMap> dmap = std::make_shared<DeltaMap>();
  dmap->aoff.reserve(all.size());
  dmap->len.reserve(all.size());
  for (const FcItem& it : all) {
    dmap->aoff.push_back(it.aoff);
    dmap->len.push_back(it.nbytes);
  }
  dmap->runs = runs;
  // re-targeting the tensors (same extents) keeps an incremental baseline; anything
  // that moves a byte of the image does not
  if (!p->dmap || !p->dmap->same_extents(*dmap)) {
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->base_plan == p) baseline_forget_locked(c);
    if (c->img_plan == p) image_forget_locked(c);
  }
  p->dmap = std::move(dmap);
  p->runs.swap(runs);
  p->h_all.swap(all);
  p->pos_bulk.swap(pos_bulk);
  p->pos_resid.swap(pos_resid);
  p->pos_shift.swap(pos_shift);
  std::sort(spans.begin(), spans.end(),
            [](const FcSpan& a, const FcSpan& b) { return a.off < b.off; });
  // NOT merged even where tensor and arena addresses both continue: two tensors may
  // sit in adjacent but separate device allocations, and a cudaMemcpy must not
  // straddle allocations (kernels do not care, the copy API does).
  p->spans.swap(spans);
  if (p->kinds.size() != n) p->kinds.assign(n, (uint8_t)FC_KIND_NONE);
  p->inputs.resize(n);
  for (uint32_t i = 0; i < n; ++i)
    p->inputs[i] = {(uint64_t)(uintptr_t)dev_ptrs[i], 0, nbytes[i]};
  p->scan_stale = true;
  return FC_OK;
}

extern "C" int fc_plan_create(fc_ctx* c, uint32_t n, const void* const* dev_ptrs,
                              const uint64_t* arena_off, const uint64_t* nbytes,
                              uint32_t chunk_bytes, fc_plan** out) {
  if (!c || !out || (n && (!dev_ptrs || !arena_off || !nbytes)))
    return fail(FC_EINVAL, "fc_plan_create: null argument%s%s");
  if (chunk_bytes == 0) chunk_bytes = kDefaultChunk;
  if (chunk_bytes < 4096 || (chunk_bytes & 127u) || chunk_bytes > (1u << 30))
    return fail(FC_EINVAL, "fc_plan_create: chunk_bytes must be a multiple of 128 in [4 KiB, 1 GiB]%s%s");
  FC_GUARD(c);
  fc_plan* p = new (std::nothrow) fc_plan();
  if (!p) return fail(FC_ENOMEM, "fc_plan_create: host alloc%s%s");
  p->ctx = c;
  p->chunk = chunk_bytes;
  cudaError_t e = cudaEventCreateWithFlags(&p->ev_upload, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_last_use, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_scan, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    fc_plan_destroy(p);
    return fail(FC_ECUDA, "fc_plan_create: %s", cudaGetErrorString(e));
  }
  int rc = plan_fill(p, n, dev_ptrs, arena_off, nbytes, nullptr, /*sync=*/true);
  if (rc) {
    fc_plan_destroy(p);
    return rc;
  }
  *out = p;
  return FC_OK;
}

extern "C" int fc_plan_update(fc_plan* p, uint32_t n, const void* const* dev_ptrs,
                              const uint64_t* arena_off, const uint64_t* nbytes, void* stream) {
  if (!p || (n && (!dev_ptrs || !arena_off || !nbytes)))
    return fail(FC_EINVAL, "fc_plan_update: null argument%s%s");
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  int rc = refresh_inflight(c);
  if (rc) return rc;
  if (c->save_inflight || c->restore_inflight)
    return fail(FC_EBUSY, "fc_plan_update: a save/restore is still in flight%s%s");
  // the staging buffers are reused: the previous upload must have executed
  FC_CUDA(cudaEventSynchronize(p->ev_upload));
  cudaStream_t s = (cudaStream_t)stream;
  // a kernel of this plan queued on ANOTHER stream must not see the new table
  FC_CUDA(cudaStreamWaitEvent(s, p->ev_last_use, 0));
  rc = plan_fill(p, n, dev_ptrs, arena_off, nbytes, s, /*sync=*/false);
  if (rc) return rc;
  FC_CUDA(cudaEventRecord(p->ev_upload, s));
  return FC_OK;
}

extern "C" int fc_plan_create_mapped(fc_ctx* c, uint32_t n, const void* const* dev_ptrs,
                                     const uint64_t* arena_off, const uint64_t* host_off,
                                     const uint64_t* nbytes, uint32_t chunk_bytes,
                                     fc_plan** out) {
  if (!host_off && n) return fail(FC_EINVAL, "fc_plan_create_mapped: null host_off%s%s");
  int rc = fc_plan_create(c, 0, nullptr, nullptr, nullptr, chunk_bytes, out);
  if (rc) return rc;
  FC_GUARD(c);
  rc = plan_fill(*out, n, dev_ptrs, arena_off, nbytes, nullptr, /*sync=*/true, host_off);
  if (rc) {
    fc_plan_destroy(*out);
    *out = nullptr;
  }
  return rc;
}

extern "C" int fc_plan_update_mapped(fc_plan* p, uint32_t n, const void* const* dev_ptrs,
                                     const uint64_t* arena_off, const uint64_t* host_off,
                                     const uint64_t* nbytes, void* stream) {
  if (!p || (n && (!dev_ptrs || !arena_off || !host_off || !nbytes)))
    return fail(FC_EINVAL, "fc_plan_update_mapped: null argument%s%s");
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  int rc = refresh_inflight(c);
  if (rc) return rc;
  if (c->save_inflight || c->restore_inflight)
    return fail(FC_EBUSY, "fc_plan_update_mapped: a save/restore is still in flight%s%s");
  FC_CUDA(cudaEventSynchronize(p->ev_upload));
  cudaStream_t s = (cudaStream_t)stream;
  FC_CUDA(cudaStreamWaitEvent(s, p->ev_last_use, 0));
  rc = plan_fill(p, n, dev_ptrs, arena_off, nbytes, s, /*sync=*/false, host_off);
  if (rc) return rc;
  FC_CUDA(cudaEventRecord(p->ev_upload, s));
  return FC_OK;
}

extern "C" int fc_plan_destroy(fc_plan* p) {
  if (!p) return FC_OK;
  fc_ctx* c = p->ctx;
  DeviceGuard g(c->device);
  // Queued kernels may still read the tables: wait for the last one (not for
  // the whole device) and defer the cudaFree (which would sync everything).
  if (p->ev_last_use) cudaEventSynchronize(p->ev_last_use);
  if (p->ev_upload) cudaEventSynchronize(p->ev_upload);
  if (p->ev_scan) cudaEventSynchronize(p->ev_scan);
  {
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->base_plan == p) {
      baseline_forget_locked(c);
      c->base_plan = nullptr;  // a later plan may be allocated at the same address
    }
    if (c->img_plan == p) {
      image_forget_locked(c);
      c->img_plan = nullptr;
      c->img_map.reset();
    }
  }
  for (FcTable* t : {&p->all, &p->bulk, &p->resid, &p->shift, &p->scan}) {
    if (t->dev) c->dead_dev.push_back(t->dev);
    if (t->pinned) c->dead_pinned.push_back(t->pinned);
  }
  if (p->scan_dev) c->dead_dev.push_back(p->scan_dev);
  if (p->scan_host) c->dead_pinned.push_back(p->scan_host);
  if (p->ev_upload) cudaEventDestroy(p->ev_upload);
  if (p->ev_last_use) cudaEventDestroy(p->ev_last_use);
  if (p->ev_scan) cudaEventDestroy(p->ev_scan);
  delete p;
  return FC_OK;
}

extern "C" int fc_plan_spans(const fc_plan* p, uint32_t* n_spans) {
  if (!p || !n_spans) return fail(FC_EINVAL, "fc_plan_spans: null argument%s%s");
  *n_spans = (uint32_t)p->spans.size();
  return FC_OK;
}

extern "C" int fc_plan_info(const fc_plan* p, uint64_t* payload_bytes, uint32_t* n_items,
                            uint32_t* n_runs, uint64_t* arena_end) {
  if (!p) return fail(FC_EINVAL, "fc_plan_info: null plan%s%s");
  if (payload_bytes) *payload_bytes = p->payload;
  if (n_items) *n_items = p->all.n;
  if (n_runs) *n_runs = (uint32_t)p->runs.size();
  if (arena_end) *arena_end = p->arena_end;
  return FC_OK;
}

extern "C" int fc_launch_count(fc_ctx* c, uint64_t* kernels, uint64_t* memcpys) {
  if (!c) return fail(FC_EINVAL, "fc_launch_count: null ctx%s%s");
  if (kernels) *kernels = c->n_kernels;
  if (memcpys) *memcpys = c->n_memcpys;
  return FC_OK;
}

extern "C" int fc_set_variant(fc_ctx* c, int variant) {
  if (!c || variant < FC_VARIANT_AUTO || variant > FC_VARIANT_TMA)
    return fail(FC_EINVAL, "fc_set_variant: bad argument%s%s");
  c->variant = variant == FC_VARIANT_AUTO ? FC_VARIANT_TMA : variant;
  return FC_OK;
}

extern "C" int fc_set_launch(fc_ctx* c, int lsu_ctas_per_sm, int tma_ctas_per_sm, int tma_stages,
                             int tma_tile_bytes) {
  if (!c) return fail(FC_EINVAL, "fc_set_launch: null ctx%s%s");
  if (lsu_ctas_per_sm < 0 || lsu_ctas_per_sm > 8 || tma_ctas_per_sm < 0 || tma_ctas_per_sm > 16 ||
      tma_stages < 0 || tma_stages == 1 || tma_stages > 32 || tma_tile_bytes < 0 ||
      (tma_tile_bytes & 15) || tma_tile_bytes > (128 << 10))
    return fail(FC_EINVAL, "fc_set_launch: out of range%s%s");
  int stages = tma_stages ? tma_stages : c->tma_stages;
  int tile = tma_tile_bytes ? tma_tile_bytes : c->tma_tile;
  if ((uint64_t)stages * tile + 8ull * stages > (227u << 10))
    return fail(FC_EINVAL, "fc_set_launch: ring exceeds 227 KB of shared memory%s%s");
  if (lsu_ctas_per_sm) c->lsu_ctas_per_sm = lsu_ctas_per_sm;
  if (tma_ctas_per_sm) c->tma_ctas_per_sm = tma_ctas_per_sm;
  c->tma_stages = stages;
  c->tma_tile = tile;
  return FC_OK;
}

template <int DIR>
static int launch_lsu(fc_ctx* c, const FcItem* items, uint32_t n, uint8_t* arena, cudaStream_t s) {
  if (n == 0) return FC_OK;
  uint32_t grid = std::min<uint32_t>(n, (uint32_t)(c->sm_count * c->lsu_ctas_per_sm));
  fc_copy_lsu<DIR><<<grid, kLsuThreads, 0, s>>>(items, n, arena);
  FC_CUDA(cudaGetLastError());
  c->n_kernels += 1;
  return FC_OK;
}

template <int DIR>
static int launch_tma(fc_ctx* c, const FcItem* items, uint32_t n, uint8_t* arena, cudaStream_t s) {
  if (n == 0) return FC_OK;
  const size_t smem = (size_t)c->tma_stages * c->tma_tile + 8u * c->tma_stages;
  FC_CUDA(cudaFuncSetAttribute(fc_copy_tma<DIR>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)smem));
  uint32_t grid = std::min<uint32_t>(n, (uint32_t)(c->sm_count * c->tma_ctas_per_sm));
  fc_copy_tma<DIR><<<grid, 32, smem, s>>>(items, n, arena, (uint32_t)c->tma_tile,
                                           (uint32_t)c->tma_stages);
  FC_CUDA(cudaGetLastError());
  c->n_kernels += 1;
  return FC_OK;
}

template <int DIR>
static int launch_shift(fc_ctx* c, const FcItem* items, uint32_t n, uint8_t* arena,
                        cudaStream_t s) {
  if (n == 0) return FC_OK;
  const size_t smem = shift_smem_bytes((uint32_t)c->shift_tile, (uint32_t)c->shift_stages);
  FC_CUDA(cudaFuncSetAttribute(fc_copy_tma_shift<DIR>,
                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  uint32_t grid = std::min<uint32_t>(n, (uint32_t)(c->sm_count * c->shift_ctas_per_sm));
  fc_copy_tma_shift<DIR><<<grid, kShiftThreads, smem, s>>>(
      items, n, arena, (uint32_t)c->shift_tile, (uint32_t)c->shift_stages);
  FC_CUDA(cudaGetLastError());
  c->n_kernels += 1;
  return FC_OK;
}

// Where arena byte 0 stands when only the part of a plan at and above segment offset
// `lo` is staged: rounded down to 128 B so that every item keeps its alignment class
// (mod 16 congruence, 128-B interior boundaries) and the same tables apply.
static inline uint64_t arena_base_for(uint64_t lo) { return lo & ~127ull; }

// Copy the items [i0, i1) of the offset-sorted `all` table (both directions), the
// arena's byte 0 standing for segment offset `base` (a multiple of 128).
template <int DIR>
static int launch_slice(fc_plan* p, cudaStream_t s, int variant, uint32_t i0, uint32_t i1,
                        uint64_t base) {
  fc_ctx* c = p->ctx;
  if (i1 <= i0) return FC_OK;
  if (variant == FC_VARIANT_AUTO) variant = c->variant;
  uint8_t* arena = c->arena - base;  // the kernels add the item's absolute offset
  int rc;
  if (variant == FC_VARIANT_TMA) {
    rc = launch_tma<DIR>(c, p->bulk.dev + p->pos_bulk[i0], p->pos_bulk[i1] - p->pos_bulk[i0],
                         arena, s);
    if (!rc)
      rc = launch_shift<DIR>(c, p->shift.dev + p->pos_shift[i0],
                             p->pos_shift[i1] - p->pos_shift[i0], arena, s);
    if (!rc)
      rc = launch_lsu<DIR>(c, p->resid.dev + p->pos_resid[i0],
                           p->pos_resid[i1] - p->pos_resid[i0], arena, s);
  } else {
    rc = launch_lsu<DIR>(c, p->all.dev + i0, i1 - i0, arena, s);
  }
  return rc;
}

template <int DIR>
static int launch_copy(fc_plan* p, cudaStream_t s, int variant) {
  fc_ctx* c = p->ctx;
  if (p->arena_end > c->arena_bytes)
    return fail(FC_EINVAL, "arena smaller than the plan: call fc_arena_reserve first%s%s");
  // tables may have been (re)uploaded on another stream
  FC_CUDA(cudaStreamWaitEvent(s, p->ev_upload, 0));
  int rc = launch_slice<DIR>(p, s, variant, 0, p->all.n, 0);
  if (rc) return rc;
  FC_CUDA(cudaEventRecord(p->ev_last_use, s));
  return FC_OK;
}

extern "C" int fc_pack_async(fc_plan* p, void* stream, int variant) {
  if (!p) return fail(FC_EINVAL, "fc_pack_async: null plan%s%s");
  FC_GUARD(p->ctx);
  delta_forget(p->ctx);
  return launch_copy<0>(p, (cudaStream_t)stream, variant);
}

extern "C" int fc_unpack_async(fc_plan* p, void* stream, int variant) {
  if (!p) return fail(FC_EINVAL, "fc_unpack_async: null plan%s%s");
  FC_GUARD(p->ctx);
  delta_forget(p->ctx);
  return launch_copy<1>(p, (cudaStream_t)stream, variant);
}

// ---- bounded arena ("windowed") mode ---------------------------------------------
// When the state does not fit a second time in HBM (arena smaller than the
// plan: fc_set_arena_limit, or the full-size cudaMalloc failed) the checkpoint is
// streamed through the arena window by window: gather the items of one window
// (the plan's kernels over a slice of the offset-sorted table), DMA the window's
// bytes, next window.  The tensors must not change until the LAST window has been
// gathered, so this mode blocks the caller for the whole checkpoint — the
// reference's behaviour, at PCIe instead of pageable-copy speed.  Restores stream
// the same windows the other way.
struct Window {
  uint32_t i0, i1;      // item index range in h_all / d_all
  uint64_t base, end;   // segment byte range covered
  uint64_t abase;       // segment offset arena byte 0 stands for (base rounded down to 128)
};

static std::vector<Window> make_windows(const fc_plan* p, uint64_t arena_bytes) {
  std::vector<Window> w;
  const std::vector<FcItem>& it = p->h_all;
  uint32_t i = 0, n = (uint32_t)it.size();
  while (i < n) {
    Window cur{i, i, it[i].aoff, it[i].aoff, arena_base_for(it[i].aoff)};
    while (cur.i1 < n && it[cur.i1].aoff + it[cur.i1].nbytes - cur.abase <= arena_bytes) {
      cur.end = std::max<uint64_t>(cur.end, it[cur.i1].aoff + it[cur.i1].nbytes);
      ++cur.i1;
    }
    if (cur.i1 == cur.i0) return {};  // one item larger than the arena
    w.push_back(cur);
    i = cur.i1;
  }
  return w;
}

// ---- restores ---------------------------------------------------------------------
// Every restore refuses while the context is busy, moves the checkpoint's bytes from one
// source into the arena or the tensors (the fill) and, through the arena, enqueues the
// plan's unpack kernels on the caller's stream.

// FC_EBUSY with the message `busy` while a save or a restore is in flight.  forget: the
// restore overwrites what the incremental baseline and the arena image describe.
static int restore_begin(fc_ctx* c, const char* busy, bool forget = true) {
  int rc = refresh_inflight(c);
  if (rc) return rc;
  if (c->save_inflight || c->restore_inflight) return fail(FC_EBUSY, "%s%s", busy);
  if (forget) delta_forget(c);
  return FC_OK;
}

// Where a fill reads: the host mapping `host`, or the file `file` (host unused).
struct FillSource {
  const uint8_t* host;
  StageFile* file;
  const char* what;  // prefix of the error a failed staged copy returns
};

// Moves every segment's bytes from src (Seg::off: offset in the source).  A file, or a
// host range that is not page-locked, goes through the bounce slots (the stage workers
// start once `gate`, if any, has completed) and is on the device on return.  A page-locked
// range is queued on the copy stream in kDmaPiece pieces cut at slice boundaries.
static int restore_fill(fc_ctx* c, const std::vector<Seg>& segs, const FillSource& src,
                        cudaEvent_t gate) {
  if (segs.empty()) return FC_OK;
  uint64_t lo = ~0ull, hi = 0;
  for (const Seg& g : segs) {
    lo = std::min(lo, g.off);
    hi = std::max(hi, g.off + g.len);
  }
  uint8_t* host = const_cast<uint8_t*>(src.host);
  const int staged = src.file ? c->stage_threads : staged_threads_for(c, host + lo, hi - lo);
  if (staged > 0) {
    const std::vector<StagePiece> pieces = stage_pieces(
        segs, src.file ? nullptr : host, c->stage_slot, src.file ? &src.file->bases : nullptr);
    cudaError_t e = stage_run(c, pieces, false, gate, staged, src.file);
    if (src.file && src.file->failed.load()) {
      char who[64], at[160];
      file_who(who, sizeof(who), src.file->fds.size(), src.file->bad_file);
      snprintf(at, sizeof(at), "%s: read failed at file offset %llu", who,
               (unsigned long long)src.file->bad_off);
      return fail(FC_EIO, "%s: %s", at,
                  src.file->err_no ? strerror(src.file->err_no) : "unexpected end of file");
    }
    if (e != cudaSuccess) return fail(FC_ECUDA, "%s: %s", src.what, cudaGetErrorString(e));
    c->n_memcpys += pieces.size();
    return FC_OK;
  }
  const SliceClip clip(c, host + lo);
  for (const Seg& g : segs)
    for (uint64_t o = 0, len = 0; o < g.len; o += len) {
      len = clip(host + g.off + o, std::min<uint64_t>(kDmaPiece, g.len - o));
      FC_CUDA(cudaMemcpyAsync(g.dev + o, host + g.off + o, len, cudaMemcpyHostToDevice,
                              c->copy_stream));
      c->n_memcpys += 1;
    }
  return FC_OK;
}

// A fill into memory that work queued on `s` may still use (the tensors of an in-place
// restore, the arena of fc_arena_fill): it starts once `s` has reached this point, and
// `s` continues once the bytes are in place.
static int restore_fill_gated(fc_ctx* c, cudaStream_t s, const std::vector<Seg>& segs,
                              const FillSource& src) {
  FC_CUDA(cudaEventRecord(c->ev_scatter_end, s));
  FC_CUDA(cudaStreamWaitEvent(c->copy_stream, c->ev_scatter_end, 0));
  FC_CUDA(cudaEventRecord(c->ev_fill_start, c->copy_stream));
  int rc = restore_fill(c, segs, src, c->ev_scatter_end);
  if (rc) return rc;
  FC_CUDA(cudaEventRecord(c->ev_fill_end, c->copy_stream));
  FC_CUDA(cudaStreamWaitEvent(s, c->ev_fill_end, 0));
  return FC_OK;
}

// The plan's runs inside arena range [lo, hi), into an arena whose byte 0 stands for offset ab.
static std::vector<Seg> run_segs(const fc_plan* p, uint64_t lo, uint64_t hi, uint64_t ab) {
  std::vector<Seg> segs;
  for (const FcRun& r : p->runs) {
    const uint64_t a = std::max(lo, r.off), b = std::min(hi, r.off + r.len);
    if (a < b) segs.push_back({p->ctx->arena + (a - ab), r.hoff + (a - r.off), b - a});
  }
  return segs;
}

// A plan larger than the arena: fill and scatter one window after the other; returns once
// the last window's scatter is enqueued.
static int restore_windowed(fc_plan* p, cudaStream_t s, const FillSource& src) {
  fc_ctx* c = p->ctx;
  std::vector<Window> wins = make_windows(p, c->arena_bytes);
  if (wins.empty() && !p->h_all.empty())
    return fail(FC_EINVAL, "arena window too small for a work item%s%s");
  FC_CUDA(cudaStreamWaitEvent(s, p->ev_upload, 0));
  FC_CUDA(cudaEventRecord(c->ev_fill_start, c->copy_stream));
  for (const Window& w : wins) {
    int rc = restore_fill(c, run_segs(p, w.base, w.end, w.abase), src, nullptr);
    if (rc) return rc;
    FC_CUDA(cudaEventRecord(c->ev_fill_end, c->copy_stream));
    FC_CUDA(cudaStreamWaitEvent(s, c->ev_fill_end, 0));
    rc = launch_slice<1>(p, s, FC_VARIANT_AUTO, w.i0, w.i1, w.abase);
    if (rc) return rc;
    FC_CUDA(cudaEventRecord(c->ev_scatter_end, s));
    FC_CUDA(cudaEventSynchronize(c->ev_scatter_end));  // window is reused by the next fill
  }
  FC_CUDA(cudaEventRecord(c->ev_fill_end, c->copy_stream));
  FC_CUDA(cudaEventRecord(p->ev_last_use, s));
  FC_CUDA(cudaEventRecord(c->ev_scatter_end, s));
  return FC_OK;
}

// A restore through the arena: fill it from src (window by window when the plan is larger
// than the arena), then scatter on `s`.  src == nullptr: the arena already holds the bytes
// (rollback); both fill events go on `s`, so fc_restore_timings reports the scatter alone.
// The next save, restore or fill refuses (FC_EBUSY) until the scatter has read the arena.
static int restore_arena(fc_plan* p, cudaStream_t s, const FillSource* src) {
  fc_ctx* c = p->ctx;
  if (src && p->arena_end > c->arena_bytes) {
    int rc = restore_windowed(p, s, *src);
    if (rc) return rc;
  } else {
    cudaStream_t fs = src ? c->copy_stream : s;
    FC_CUDA(cudaEventRecord(c->ev_fill_start, fs));
    if (src) {
      int rc = restore_fill(c, run_segs(p, 0, p->arena_end, 0), *src, nullptr);
      if (rc) return rc;
    }
    FC_CUDA(cudaEventRecord(c->ev_fill_end, fs));
    FC_CUDA(cudaStreamWaitEvent(s, c->ev_fill_end, 0));
    int rc = launch_copy<1>(p, s, FC_VARIANT_AUTO);
    if (rc) return rc;
    FC_CUDA(cudaEventRecord(c->ev_scatter_end, s));
  }
  c->restore_inflight = true;
  return FC_OK;
}

// ---- saves ------------------------------------------------------------------------
// Every save is one form of the same thing: the plan's ranges below segment offset `cut`
// drain in place (DMA straight from the tensors, first), the ranges from the cut on are
// gathered into the arena, whose byte 0 stands for the cut rounded down to 128 B, and
// drained from there.  cut = 0 snapshots everything (fc_save_async, fc_save_delta_async),
// cut = ~0 drains everything in place (fc_save_direct_async), anything else is a hybrid
// (fc_save_hybrid_async).  Each save runs the same checks (save_begin), one gather
// (save_gather) and one enqueue (save_enqueue); the pump drains it (drain_job).  A save
// through a bounded arena is drained window by window on the caller's thread instead
// (save_windowed).
struct SaveForm {
  const char* who;   // prefix of the refusals
  uint64_t cut;
  bool in_place;     // fc_save_hybrid_async / fc_save_direct_async: identity and cut rules,
                     // the sources stay frozen until the in-place part drained, no image
  bool incremental;  // fc_save_delta_async: compare with the baseline, then become it
  bool hold;         // the drain waits for fc_save_release
};

static int launch_delta_lsu(fc_ctx* c, const FcItem* items, uint32_t n, cudaStream_t s,
                            uint32_t seq) {
  if (n == 0) return FC_OK;
  uint32_t grid = std::min<uint32_t>(n, (uint32_t)(c->sm_count * c->lsu_ctas_per_sm));
  fc_delta_lsu<<<grid, kLsuThreads, 0, s>>>(items, n, c->arena, c->dirty, seq);
  FC_CUDA(cudaGetLastError());
  c->n_kernels += 1;
  return FC_OK;
}

// The ring takes the copy ring's shared memory (fc_set_launch): a stage holds a source
// and an old tile of half the copy tile each (default 2 stages x 2 x 48 KiB).
static int launch_delta_tma(fc_ctx* c, const FcItem* items, uint32_t n, cudaStream_t s,
                            uint32_t seq) {
  if (n == 0) return FC_OK;
  const uint32_t tile = std::max<uint32_t>(128u, ((uint32_t)c->tma_tile / 2u) & ~127u);
  const uint32_t stages = (uint32_t)c->tma_stages;
  const size_t smem = delta_smem_bytes(tile, stages);
  FC_CUDA(cudaFuncSetAttribute(fc_delta_tma, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)smem));
  uint32_t grid = std::min<uint32_t>(n, (uint32_t)(c->sm_count * c->tma_ctas_per_sm));
  fc_delta_tma<<<grid, kDeltaThreads, smem, s>>>(items, n, c->arena, c->dirty, seq, tile, stages);
  FC_CUDA(cudaGetLastError());
  c->n_kernels += 1;
  return FC_OK;
}

// Gather-compare over the whole plan: bulk bodies through the TMA ring, shifted ranges
// and residues through the LSU kernel (FC_VARIANT_LSU: every item through the LSU kernel).
static int launch_delta(fc_plan* p, cudaStream_t s, uint32_t seq) {
  fc_ctx* c = p->ctx;
  if (c->variant != FC_VARIANT_TMA) return launch_delta_lsu(c, p->all.dev, p->all.n, s, seq);
  int rc = launch_delta_tma(c, p->bulk.dev, p->bulk.n, s, seq);
  if (!rc) rc = launch_delta_lsu(c, p->shift.dev, p->shift.n, s, seq);
  if (!rc) rc = launch_delta_lsu(c, p->resid.dev, p->resid.n, s, seq);
  return rc;
}

// What a save covers once its checks have passed.
struct SaveScope {
  uint32_t i0 = 0;          // first item of the arena part
  uint64_t abase = 0;       // segment offset arena byte 0 stands for
  std::vector<Window> wins; // a bounded-arena save: its windows
};

// The checks of a save after the null argument, in a fixed order: the busy rule, the
// form's own rules, the sticky drain error.  Nothing is forgotten or written before all of
// them have passed.
static int save_begin(fc_plan* p, const SaveForm& f, SaveScope* s) {
  fc_ctx* c = p->ctx;
  int rc = refresh_inflight(c);
  if (rc) return rc;
  if (c->save_inflight || c->restore_inflight)
    return fail(FC_EBUSY, "%s: previous save/restore still draining%s", f.who);
  if (f.in_place) {
    if (!p->identity && f.cut != ~0ull)
      return fail(FC_EINVAL, "fc_save_hybrid_async: needs a plan whose arena is an image of "
                             "the segment%s%s");
    const std::vector<FcItem>& it = p->h_all;
    s->i0 = (uint32_t)(std::lower_bound(it.begin(), it.end(), f.cut,
                                        [](const FcItem& a, uint64_t v) { return a.aoff < v; }) -
                       it.begin());
    if (s->i0 > 0 && it[s->i0 - 1].aoff + it[s->i0 - 1].nbytes > f.cut)
      return fail(FC_EINVAL, "fc_save_hybrid_async: cut is not a tensor boundary%s%s");
    s->abase = arena_base_for(std::min(f.cut, p->arena_end));
    if (s->i0 < it.size() && p->arena_end - s->abase > c->arena_bytes)
      return fail(FC_EINVAL, "fc_save_hybrid_async: arena smaller than the snapshot part%s%s");
  } else if (p->arena_end > c->arena_bytes) {
    if (f.incremental)
      return fail(FC_EINVAL, "fc_save_delta_async: the arena must hold the whole plan (no "
                             "incremental bounded-arena save)%s%s");
    if (c->arena_bytes < (8ull << 20) || !p->identity)
      return fail(FC_EINVAL, "arena smaller than the plan: call fc_arena_reserve first%s%s");
    s->wins = make_windows(p, c->arena_bytes);
    if (s->wins.empty()) return fail(FC_EINVAL, "arena window too small for a work item%s%s");
  }
  // a sticky drain error must surface BEFORE the arena is overwritten
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->drain_rc != FC_OK) return fail(c->drain_rc, "%s", c->drain_err.c_str());
  return FC_OK;
}

// The gather of a save on the caller's stream, between ev_pack_start and ev_pack_end: the
// copy kernels over the items from i0 on, or (compare) the gather-compare kernels over
// the whole plan.  With no item the pair of events still orders the drain after
// everything already queued on the stream (the optimizer step that produced the values).
static int save_gather(fc_plan* p, cudaStream_t cs, const SaveScope& s, bool compare) {
  fc_ctx* c = p->ctx;
  const uint32_t n = p->all.n;
  if (compare) {
    bool reset = false;
    if (n > c->dirty_cap) {
      const uint32_t cap = (uint32_t)std::min<uint64_t>(0xFFFFFFF0ull, n + n / 4 + 16);
      uint32_t* nd = nullptr;
      uint32_t* np = nullptr;
      cudaError_t e = cudaMalloc(&nd, (size_t)cap * sizeof(uint32_t));
      if (e == cudaSuccess)
        e = cudaHostAlloc(&np, (size_t)cap * sizeof(uint32_t), cudaHostAllocDefault);
      if (e != cudaSuccess) {
        (void)cudaGetLastError();
        if (nd) c->dead_dev.push_back(nd);
        return fail(FC_ENOMEM, "dirty marks alloc: %s", cudaGetErrorString(e));
      }
      if (c->dirty) c->dead_dev.push_back(c->dirty);  // no save is in flight: nothing reads them
      if (c->dirty_pinned) c->dead_pinned.push_back(c->dirty_pinned);
      c->dirty = nd;
      c->dirty_pinned = np;
      c->dirty_cap = cap;
      reset = true;
    }
    // marks are sequence numbers: cleared only for a fresh array or when seq wraps
    if (++c->delta_seq == 0) reset = true;
    if (reset) {
      FC_CUDA(cudaMemsetAsync(c->dirty, 0, (size_t)c->dirty_cap * sizeof(uint32_t), cs));
      c->delta_seq = 1;
    }
  }
  FC_CUDA(cudaEventRecord(c->ev_pack_start, cs));
  if (s.i0 < n) {
    FC_CUDA(cudaStreamWaitEvent(cs, p->ev_upload, 0));  // tables may come from another stream
    int rc = compare ? launch_delta(p, cs, c->delta_seq)
                     : launch_slice<0>(p, cs, FC_VARIANT_AUTO, s.i0, n, s.abase);
    if (rc) return rc;
    FC_CUDA(cudaEventRecord(p->ev_last_use, cs));
  }
  FC_CUDA(cudaEventRecord(c->ev_pack_end, cs));
  return FC_OK;
}

// Under mu: refuses while a drain error is pending, else issues the next save ticket.
static int next_ticket_locked(fc_ctx* c, uint64_t* ticket) {
  if (c->drain_rc != FC_OK) return fail(c->drain_rc, "%s", c->drain_err.c_str());
  c->ticket += 1;
  if (ticket) *ticket = c->ticket;
  return FC_OK;
}

// A bounded-arena save: gather and drain one window after the other on the caller's
// thread, each window's runs under the pacing of the arena part (drain_runs).  Complete
// on return, with its ticket drained; fc_save_timings spans the first gather to the last
// drain.
static int save_windowed(fc_plan* p, const std::vector<Window>& wins, uint8_t* host,
                         cudaStream_t cs, uint64_t* ticket) {
  fc_ctx* c = p->ctx;
  const SliceClip clip(c, host + p->host_lo);
  FC_CUDA(cudaStreamWaitEvent(cs, p->ev_upload, 0));
  FC_CUDA(cudaEventRecord(c->ev_pack_start, cs));
  for (size_t i = 0; i < wins.size(); ++i) {
    const Window& w = wins[i];
    int rc = launch_slice<0>(p, cs, FC_VARIANT_AUTO, w.i0, w.i1, w.abase);
    if (rc) return rc;
    FC_CUDA(cudaEventRecord(c->ev_pack_end, cs));
    FC_CUDA(cudaStreamWaitEvent(c->copy_stream, c->ev_pack_end, 0));
    if (i == 0) FC_CUDA(cudaEventRecord(c->ev_drain_start, c->copy_stream));
    const cudaError_t e =
        drain_runs(c, host, run_segs(p, w.base, w.end, w.abase), clip, &c->n_memcpys);
    if (e != cudaSuccess)
      return fail(FC_ECUDA, "bounded-arena drain: %s%s", cudaGetErrorString(e));
    // the next gather overwrites the window: it must wait for this drain
    FC_CUDA(cudaEventRecord(c->ev_drain_end, c->copy_stream));
    FC_CUDA(cudaStreamWaitEvent(cs, c->ev_drain_end, 0));
  }
  FC_CUDA(cudaEventRecord(c->ev_pack_end, cs));
  FC_CUDA(cudaEventRecord(p->ev_last_use, cs));
  FC_CUDA(cudaEventRecord(c->ev_drain_end, c->copy_stream));
  FC_CUDA(cudaEventSynchronize(c->ev_drain_end));
  FC_CUDA(cudaEventSynchronize(c->ev_pack_end));
  std::lock_guard<std::mutex> lk(c->mu);
  int rc = next_ticket_locked(c, ticket);
  if (rc) return rc;
  c->stat_ticket = c->ticket;
  c->stat_bytes = p->payload;
  c->stat_delta = 0;
  c->drained_ticket = c->ticket;
  return FC_OK;
}

// Issues the save's ticket and hands its drain to the pump, with the records the form sets.
static int save_enqueue(fc_plan* p, const SaveForm& f, uint8_t* host, fc_ctx::DrainJob& job,
                        uint64_t* ticket) {
  fc_ctx* c = p->ctx;
  {
    std::lock_guard<std::mutex> lk(c->mu);
    int rc = next_ticket_locked(c, ticket);
    if (rc) return rc;
    if (!c->pump.joinable()) c->pump = std::thread(pump_main, c);
    job.ticket = c->ticket;
    if (f.hold) c->held_ticket = c->ticket;
    if (f.in_place) c->direct_ticket = c->ticket;
    c->jobs.push_back(std::move(job));
    c->save_inflight = true;
    if (f.incremental) {
      c->base_plan = p;
      c->base_host = host;
      c->base_ticket = c->ticket;
    }
    if (!f.in_place) image_expect_locked(c, p, host, c->ticket);
  }
  c->cv.notify_all();
  return FC_OK;
}

static int save(fc_plan* p, void* host_base, void* compute_stream, uint64_t* ticket,
                const SaveForm& f) {
  if (!p || (!host_base && p->payload)) return fail(FC_EINVAL, "%s: null argument%s", f.who);
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  SaveScope s;
  int rc = save_begin(p, f, &s);
  if (rc) return rc;
  uint8_t* host = static_cast<uint8_t*>(host_base);
  cudaStream_t cs = (cudaStream_t)compute_stream;
  bool compare;
  {
    // the arena changes now; an incremental save's baseline is valid again once it drained
    std::lock_guard<std::mutex> lk(c->mu);
    compare = f.incremental && c->base_valid && c->base_plan == p && c->base_host == host;
    delta_forget_locked(c);
  }
  if (!s.wins.empty()) return save_windowed(p, s.wins, host, cs, ticket);
  rc = save_gather(p, cs, s, compare);
  if (rc) return rc;
  fc_ctx::DrainJob job;
  job.host = host;
  job.direct = f.in_place;
  for (const FcSpan& sp : p->spans)
    if (sp.off < f.cut) job.spans.push_back({(uint8_t*)(uintptr_t)sp.tptr, sp.off, sp.len});
  if (compare) {
    job.delta = p->dmap;
    job.seq = c->delta_seq;
  } else {
    job.runs = run_segs(p, f.cut, ~0ull, s.abase);
  }
  job.staged_threads =
      p->runs.empty() ? 0 : staged_threads_for(c, host + p->host_lo, p->host_hi - p->host_lo);
  return save_enqueue(p, f, host, job, ticket);
}

//                                                        who, cut, in_place, incremental, hold
extern "C" int fc_save_async(fc_plan* p, void* host_base, void* compute_stream, uint64_t* ticket) {
  return save(p, host_base, compute_stream, ticket, {"fc_save_async", 0, false, false, false});
}

extern "C" int fc_save_async_held(fc_plan* p, void* host_base, void* compute_stream,
                                  uint64_t* ticket) {
  return save(p, host_base, compute_stream, ticket, {"fc_save_async", 0, false, false, true});
}

extern "C" int fc_save_hybrid_async(fc_plan* p, void* host_base, void* compute_stream,
                                    uint64_t cut, int hold, uint64_t* ticket) {
  return save(p, host_base, compute_stream, ticket,
              {"fc_save_hybrid_async", cut, true, false, hold != 0});
}

extern "C" int fc_save_direct_async(fc_plan* p, void* host_base, void* compute_stream, int hold,
                                    uint64_t* ticket) {
  return save(p, host_base, compute_stream, ticket,
              {"fc_save_hybrid_async", ~0ull, true, false, hold != 0});
}

extern "C" int fc_save_delta_async(fc_plan* p, void* host_base, void* compute_stream, int hold,
                                   uint64_t* ticket) {
  return save(p, host_base, compute_stream, ticket,
              {"fc_save_delta_async", 0, false, true, hold != 0});
}

extern "C" int fc_save_release(fc_ctx* c, uint64_t ticket) {
  if (!c) return fail(FC_EINVAL, "fc_save_release: null ctx%s%s");
  {
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->held_ticket == ticket) c->held_ticket = 0;
  }
  c->cv.notify_all();
  return FC_OK;
}

extern "C" int fc_save_cancel(fc_ctx* c, uint64_t ticket) {
  if (!c) return fail(FC_EINVAL, "fc_save_cancel: null ctx%s%s");
  {
    std::lock_guard<std::mutex> lk(c->mu);
    if (c->held_ticket != ticket || ticket == 0)
      return fail(FC_EBUSY, "fc_save_cancel: the drain is not held (any more)%s%s");
    for (auto it = c->jobs.begin(); it != c->jobs.end(); ++it)
      if (it->ticket == ticket) {
        c->jobs.erase(it);
        break;
      }
    // the gather has changed the arena, the segment keeps the previous image
    delta_forget_locked(c);
    c->stat_ticket = ticket;
    c->stat_bytes = 0;
    c->stat_delta = 0;
    c->held_ticket = 0;
    c->drained_ticket = std::max(c->drained_ticket, ticket);  // nothing will be written
    if (c->direct_ticket == ticket) c->inplace_done_ticket = ticket;
  }
  c->cv.notify_all();
  return FC_OK;
}

static int check_ticket(fc_ctx* c, uint64_t ticket, const char* who);

extern "C" int fc_save_delta_stats(fc_ctx* c, uint64_t ticket, uint64_t* drained_bytes,
                                   int* delta) {
  int rc = check_ticket(c, ticket, "fc_save_delta_stats");
  if (rc) return rc;
  std::lock_guard<std::mutex> lk(c->mu);
  if (c->drained_ticket < ticket) return FC_ENOTREADY;
  if (c->stat_ticket != ticket) return fail(FC_EINVAL, "fc_save_delta_stats: no statistics%s%s");
  if (drained_bytes) *drained_bytes = c->stat_bytes;
  if (delta) *delta = c->stat_delta;
  return FC_OK;
}

extern "C" int fc_delta_invalidate(fc_ctx* c) {
  if (!c) return fail(FC_EINVAL, "fc_delta_invalidate: null ctx%s%s");
  delta_forget(c);
  return FC_OK;
}

extern "C" int fc_restore_direct_async(fc_plan* p, const void* host_base, void* stream) {
  if (!p || (!host_base && p->payload))
    return fail(FC_EINVAL, "fc_restore_direct_async: null argument%s%s");
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  int rc = restore_begin(c, "fc_restore_direct_async: context busy");
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<Seg> segs;
  for (const FcSpan& sp : p->spans) segs.push_back({(uint8_t*)(uintptr_t)sp.tptr, sp.off, sp.len});
  const FillSource src{static_cast<const uint8_t*>(host_base), nullptr, "staged restore"};
  rc = restore_fill_gated(c, s, segs, src);
  if (rc) return rc;
  FC_CUDA(cudaEventRecord(c->ev_scatter_end, s));
  c->restore_inflight = true;
  return FC_OK;
}

static int check_ticket(fc_ctx* c, uint64_t ticket, const char* who) {
  if (!c) return fail(FC_EINVAL, "%s: null ctx", who);
  if (ticket == 0 || ticket != c->ticket) return fail(FC_EINVAL, "%s: unknown ticket", who);
  return FC_OK;
}

static int drain_status(fc_ctx* c, uint64_t ticket, bool wait);

// FC_OK once nothing of save `ticket` reads the source tensors any more: its gather
// kernel (if any) has finished and its in-place part (if any) has been drained.
static int sources_status(fc_ctx* c, uint64_t ticket, bool wait) {
  {
    std::unique_lock<std::mutex> lk(c->mu);
    if (ticket == c->direct_ticket) {
      if (wait)
        c->cv.wait(lk, [&] { return c->inplace_done_ticket >= ticket || c->drain_rc != FC_OK; });
      if (c->drain_rc != FC_OK) return fail(c->drain_rc, "%s", c->drain_err.c_str());
      if (c->inplace_done_ticket < ticket) return FC_ENOTREADY;
    }
  }
  DeviceGuard g(c->device);
  if (!g.ok) return fail(FC_ECUDA, "cudaSetDevice failed%s%s");
  cudaError_t e = wait ? cudaEventSynchronize(c->ev_pack_end) : cudaEventQuery(c->ev_pack_end);
  if (e == cudaSuccess) return FC_OK;
  if (e == cudaErrorNotReady) return FC_ENOTREADY;
  return fail(FC_ECUDA, "cudaEvent(pack): %s", cudaGetErrorString(e));
}

extern "C" int fc_save_pack_done(fc_ctx* c, uint64_t ticket) {
  int rc = check_ticket(c, ticket, "fc_save_pack_done");
  if (rc) return rc;
  return sources_status(c, ticket, false);
}

extern "C" int fc_save_sources_wait(fc_ctx* c, uint64_t ticket) {
  int rc = check_ticket(c, ticket, "fc_save_sources_wait");
  if (rc) return rc;
  return sources_status(c, ticket, true);
}

static int drain_status(fc_ctx* c, uint64_t ticket, bool wait) {
  std::unique_lock<std::mutex> lk(c->mu);
  if (wait) c->cv.wait(lk, [&] { return c->drained_ticket >= ticket; });
  if (c->drained_ticket < ticket) return FC_ENOTREADY;
  if (c->drain_rc != FC_OK) return fail(c->drain_rc, "%s", c->drain_err.c_str());
  c->save_inflight = false;
  return FC_OK;
}

extern "C" int fc_save_poll(fc_ctx* c, uint64_t ticket) {
  int rc = check_ticket(c, ticket, "fc_save_poll");
  if (rc) return rc;
  return drain_status(c, ticket, false);
}

extern "C" int fc_save_wait(fc_ctx* c, uint64_t ticket) {
  int rc = check_ticket(c, ticket, "fc_save_wait");
  if (rc) return rc;
  return drain_status(c, ticket, true);
}

extern "C" int fc_save_timings(fc_ctx* c, uint64_t ticket, float* pack_ms, float* drain_ms,
                               float* total_ms) {
  int rc = check_ticket(c, ticket, "fc_save_timings");
  if (rc) return rc;
  rc = drain_status(c, ticket, true);
  if (rc) return rc;
  FC_GUARD(c);
  float t = 0.f;
  if (pack_ms) {
    FC_CUDA(cudaEventElapsedTime(&t, c->ev_pack_start, c->ev_pack_end));
    *pack_ms = t;
  }
  if (drain_ms) {
    FC_CUDA(cudaEventElapsedTime(&t, c->ev_drain_start, c->ev_drain_end));
    *drain_ms = t;
  }
  if (total_ms) {
    FC_CUDA(cudaEventElapsedTime(&t, c->ev_pack_start, c->ev_drain_end));
    *total_ms = t;
  }
  return FC_OK;
}

extern "C" int fc_set_shift_launch(fc_ctx* c, int ctas_per_sm, int in_stages, int tile_bytes) {
  if (!c) return fail(FC_EINVAL, "fc_set_shift_launch: null ctx%s%s");
  int cps = ctas_per_sm ? ctas_per_sm : c->shift_ctas_per_sm;
  int st = in_stages ? in_stages : c->shift_stages;
  int tile = tile_bytes ? tile_bytes : c->shift_tile;
  if (cps < 1 || cps > 8 || st < 2 || st > 8 || tile < 4096 || (tile & 127) ||
      shift_smem_bytes((uint32_t)tile, (uint32_t)st) > (227u << 10))
    return fail(FC_EINVAL, "fc_set_shift_launch: out of range%s%s");
  c->shift_ctas_per_sm = cps;
  c->shift_stages = st;
  c->shift_tile = tile;
  return FC_OK;
}

extern "C" int fc_set_drain(fc_ctx* c, uint64_t piece_bytes, int depth) {
  if (!c) return fail(FC_EINVAL, "fc_set_drain: null ctx%s%s");
  if ((piece_bytes && piece_bytes < (64u << 10)) || depth < 0 || depth > kDrainRing)
    return fail(FC_EINVAL, "fc_set_drain: piece >= 64 KiB, depth in [1, 8]%s%s");
  std::lock_guard<std::mutex> lk(c->mu);
  if (piece_bytes) c->drain_piece = piece_bytes;
  if (depth) c->drain_depth = depth;
  return FC_OK;
}

extern "C" int fc_set_stage(fc_ctx* c, int threads, uint64_t slot_bytes) {
  if (!c || threads < 0 || threads > 32 || (slot_bytes && slot_bytes < (256u << 10)) ||
      slot_bytes > (256ull << 20))
    return fail(FC_EINVAL, "fc_set_stage: threads in [1, 32], slot in [256 KiB, 256 MiB]%s%s");
  std::lock_guard<std::mutex> lk(c->mu);
  if (threads) c->stage_threads = threads;
  if (slot_bytes && slot_bytes != c->stage_slot) {
    if (!c->stage.empty()) return fail(FC_EBUSY, "fc_set_stage: slots already allocated%s%s");
    c->stage_slot = slot_bytes;
  }
  return FC_OK;
}

extern "C" int fc_set_drain_mode(fc_ctx* c, int mode) {
  if (!c || (mode != FC_DRAIN_HOST_PACED && mode != FC_DRAIN_PINGPONG))
    return fail(FC_EINVAL, "fc_set_drain_mode: bad argument%s%s");
  std::lock_guard<std::mutex> lk(c->mu);
  c->drain_mode = mode;
  return FC_OK;
}

// ---- host-resident leaves ---------------------------------------------------
// CPU tensors inside a state_dict (optimizer step counters, RNG state, a whole
// CPU model in the gloo/CPU configuration) are already in host memory: they go
// straight into the segment with a (multi-threaded) memcpy, no device hop.

struct HostJob {
  uint8_t* dst;             // segment base (the "packed" side)
  const void* const* src;   // the ranges (the "tensor" side)
  const uint64_t* off;
  const uint64_t* nbytes;
  uint64_t first, last;
  uint64_t skip_first, trim_last;  // byte sub-range of the first / last range
  bool unpack;              // false: ranges -> segment, true: segment -> ranges
};

static void* host_pack_worker(void* arg) {
  HostJob* j = static_cast<HostJob*>(arg);
  for (uint64_t i = j->first; i < j->last; ++i) {
    uint64_t lo = (i == j->first) ? j->skip_first : 0;
    uint64_t hi = (i + 1 == j->last) ? j->trim_last : j->nbytes[i];
    if (hi <= lo) continue;
    uint8_t* packed = j->dst + j->off[i] + lo;
    uint8_t* range = static_cast<uint8_t*>(const_cast<void*>(j->src[i])) + lo;
    if (j->unpack)
      memcpy(range, packed, hi - lo);
    else
      memcpy(packed, range, hi - lo);
  }
  return nullptr;
}

static int host_copy(void* base, uint32_t n, const void* const* ranges, const uint64_t* off,
                     const uint64_t* nbytes, int threads, bool unpack, const char* who);

extern "C" int fc_host_pack(void* dst_base, uint32_t n, const void* const* src,
                            const uint64_t* off, const uint64_t* nbytes, int threads) {
  return host_copy(dst_base, n, src, off, nbytes, threads, false, "fc_host_pack");
}

extern "C" int fc_host_unpack(const void* src_base, uint32_t n, void* const* dst,
                              const uint64_t* off, const uint64_t* nbytes, int threads) {
  return host_copy(const_cast<void*>(src_base), n, dst, off, nbytes, threads, true,
                   "fc_host_unpack");
}

static int host_copy(void* dst_base, uint32_t n, const void* const* src, const uint64_t* off,
                     const uint64_t* nbytes, int threads, bool unpack, const char* who) {
  if (!dst_base || (n && (!src || !off || !nbytes))) return fail(FC_EINVAL, "%s: null argument%s", who);
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (nbytes[i] && !src[i]) return fail(FC_EINVAL, "%s: null range%s", who);
    total += nbytes[i];
  }
  if (total == 0) return FC_OK;
  int nt = std::max(1, std::min(threads, 64));
  if (total < (8ull << 20)) nt = 1;  // not worth a thread
  // equal BYTE shares: a worker may start/stop in the middle of a range
  std::vector<HostJob> jobs;
  uint64_t share = (total + nt - 1) / nt;
  uint32_t i = 0;
  uint64_t inner = 0;  // bytes of range i already assigned
  while (i < n) {
    HostJob j{static_cast<uint8_t*>(dst_base), src, off, nbytes, i, i, inner, 0, unpack};
    uint64_t need = share;
    while (i < n && need > 0) {
      uint64_t left = nbytes[i] - inner;
      if (left <= need) {
        need -= left;
        j.trim_last = nbytes[i];
        ++i;
        inner = 0;
      } else {
        inner += need;
        j.trim_last = inner;
        need = 0;
        j.last = i + 1;
        break;
      }
      j.last = i;
    }
    if (j.last > j.first) jobs.push_back(j);
  }
  std::vector<pthread_t> th(jobs.size());
  for (size_t k = 0; k < jobs.size(); ++k) {
    if (k + 1 == jobs.size() || pthread_create(&th[k], nullptr, host_pack_worker, &jobs[k]) != 0) {
      host_pack_worker(&jobs[k]);
      th[k] = 0;
    }
  }
  for (size_t k = 0; k < jobs.size(); ++k)
    if (th[k]) pthread_join(th[k], nullptr);
  return FC_OK;
}

extern "C" int fc_restore_async(fc_plan* p, const void* host_base, void* stream) {
  if (!p || (!host_base && p->payload)) return fail(FC_EINVAL, "fc_restore_async: null argument%s%s");
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  int rc = restore_begin(c, "fc_restore_async: arena busy");
  if (rc) return rc;
  if (p->arena_end > c->arena_bytes && (c->arena_bytes < (8ull << 20) || !p->identity))
    return fail(FC_EINVAL, "arena smaller than the plan: call fc_arena_reserve first%s%s");
  const FillSource src{static_cast<const uint8_t*>(host_base), nullptr, "staged restore"};
  return restore_arena(p, (cudaStream_t)stream, &src);
}

// ---- restore from a file ------------------------------------------------------------
// The plan's host offsets are file offsets.  The stage workers pread every run into their
// pinned bounce slots and DMA each slot into the arena; the scatter is enqueued only once
// every byte has arrived, so a short read or an I/O error changes no target tensor (in
// the windowed mode: none after the first window, whose scatter has already run).
// Several files: the plan's host offsets lie in their virtual concatenation (file k owns
// [bases[k], bases[k+1])).  One fill reads every file, then one scatter runs.
static int restore_files(fc_plan* p, uint32_t n, const int* fds, const uint64_t* bases,
                         void* stream) {
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  char who[64], at[160], end[64];
  int rc = restore_begin(c, n == 1 ? "fc_restore_file_async: arena busy"
                                   : "fc_restore_files_async: arena busy");
  if (rc) return rc;
  StageFile file;
  file.fds.assign(fds, fds + n);
  file.bases.assign(bases, bases + n);
  // the highest byte the plan reads in each file, in that file's own offsets
  std::vector<uint64_t> need(n, 0);
  for (const FcRun& r : p->runs) {
    if (r.len == 0) continue;
    if (r.hoff < bases[0])
      return fail(FC_EINVAL, "fc_restore_files_async: the plan reads below the first file's base%s%s");
    for (uint32_t k = file.file_of(r.hoff); k < n && bases[k] < r.hoff + r.len; ++k) {
      const uint64_t hi = k + 1 < n ? std::min(r.hoff + r.len, bases[k + 1]) : r.hoff + r.len;
      need[k] = std::max(need[k], hi - bases[k]);
    }
  }
  // a truncated file: refuse before any byte moves, in every mode
  for (uint32_t k = 0; k < n; ++k) {
    file_who(who, sizeof(who), n, k);
    struct stat st;
    if (fstat(fds[k], &st) != 0) {
      snprintf(at, sizeof(at), "%s: fstat", who);
      return fail(FC_EIO, "%s: %s", at, strerror(errno));
    }
    if ((uint64_t)st.st_size < need[k]) {
      snprintf(at, sizeof(at), "%s: the plan reads up to file offset %llu", who,
               (unsigned long long)need[k]);
      snprintf(end, sizeof(end), "%llu", (unsigned long long)st.st_size);
      return fail(FC_EIO, "%s, the file ends at %s", at, end);
    }
  }
  if (p->arena_end > c->arena_bytes && c->arena_bytes < (8ull << 20))
    return fail(FC_EINVAL, "arena smaller than the plan: call fc_arena_reserve first%s%s");
  const FillSource src{nullptr, &file, "file restore"};
  return restore_arena(p, (cudaStream_t)stream, &src);
}

extern "C" int fc_restore_file_async(fc_plan* p, int fd, void* stream) {
  if (!p || fd < 0) return fail(FC_EINVAL, "fc_restore_file_async: null plan or bad fd%s%s");
  const uint64_t base = 0;
  return restore_files(p, 1, &fd, &base, stream);
}

extern "C" int fc_restore_files_async(fc_plan* p, uint32_t n, const int* fds,
                                      const uint64_t* bases, void* stream) {
  if (!p || n == 0 || !fds || !bases)
    return fail(FC_EINVAL, "fc_restore_files_async: null plan, no files or null array%s%s");
  for (uint32_t k = 0; k < n; ++k)
    if (fds[k] < 0 || (k > 0 && bases[k] <= bases[k - 1]))
      return fail(FC_EINVAL, "fc_restore_files_async: bad fd or bases not strictly increasing%s%s");
  return restore_files(p, n, fds, bases, stream);
}

// ---- rollback from the arena image ----------------------------------------------
// Every run of `p`, as (arena off, segment hoff, len), must lie inside one run of the
// image map at the same offset on both sides: then the arena holds, at p's arena offsets,
// exactly the bytes fc_restore_async would fetch from host_base.  The image runs are
// sorted by arena offset and do not overlap: one binary search per run of p.
static bool image_covers_locked(const fc_ctx* c, const fc_plan* p, const uint8_t* host) {
  if (!c->img_valid || !c->img_map || c->img_host != host) return false;
  if (p->arena_end > c->arena_bytes) return false;
  const std::vector<FcRun>& img = c->img_map->runs;
  for (const FcRun& r : p->runs) {
    auto it = std::upper_bound(img.begin(), img.end(), r.off,
                               [](uint64_t v, const FcRun& m) { return v < m.off; });
    if (it == img.begin()) return false;
    const FcRun& m = *(it - 1);
    const uint64_t in = r.off - m.off;
    if (in + r.len > m.len || r.hoff < m.hoff || r.hoff - m.hoff != in) return false;
  }
  return true;
}

extern "C" int fc_image_covers(const fc_plan* p, const void* host_base) {
  if (!p || (!host_base && p->payload)) return fail(FC_EINVAL, "fc_image_covers: null argument%s%s");
  fc_ctx* c = p->ctx;
  std::lock_guard<std::mutex> lk(c->mu);
  return image_covers_locked(c, p, static_cast<const uint8_t*>(host_base)) ? FC_OK : FC_ENOIMAGE;
}

extern "C" int fc_restore_from_image_async(fc_plan* p, const void* host_base, void* stream) {
  if (!p || (!host_base && p->payload))
    return fail(FC_EINVAL, "fc_restore_from_image_async: null argument%s%s");
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  int rc = restore_begin(c, "fc_restore_from_image_async: context busy", false);
  if (rc) return rc;
  {
    // nothing runs between this check and the scatter's enqueue that could change the
    // record: saves, restores and plan updates of this context refuse while it is busy,
    // and the pump has drained every ticket (save_inflight is false)
    std::lock_guard<std::mutex> lk(c->mu);
    if (!image_covers_locked(c, p, static_cast<const uint8_t*>(host_base)))
      return fail(FC_ENOIMAGE, "fc_restore_from_image_async: no arena image covers the plan%s%s");
  }
  return restore_arena(p, (cudaStream_t)stream, nullptr);
}

extern "C" int fc_arena_fill(fc_ctx* c, const void* host_base, uint64_t lo, uint64_t hi,
                             void* stream) {
  if (!c || !host_base || hi < lo) return fail(FC_EINVAL, "fc_arena_fill: bad argument%s%s");
  FC_GUARD(c);
  int rc = restore_begin(c, "fc_arena_fill: arena busy");
  if (rc) return rc;
  if (hi > c->arena_bytes) return fail(FC_EINVAL, "fc_arena_fill: arena too small%s%s");
  if (hi == lo) return FC_OK;
  const FillSource src{static_cast<const uint8_t*>(host_base), nullptr, "fc_arena_fill (staged)"};
  return restore_fill_gated(c, (cudaStream_t)stream, {{c->arena + lo, lo, hi - lo}}, src);
}

extern "C" int fc_restore_wait(fc_ctx* c) {
  if (!c) return fail(FC_EINVAL, "fc_restore_wait: null ctx%s%s");
  FC_GUARD(c);
  FC_CUDA(cudaEventSynchronize(c->ev_scatter_end));
  c->restore_inflight = false;
  return FC_OK;
}

extern "C" int fc_restore_timings(fc_ctx* c, float* fill_ms, float* scatter_ms, float* total_ms) {
  if (!c) return fail(FC_EINVAL, "fc_restore_timings: null ctx%s%s");
  FC_GUARD(c);
  FC_CUDA(cudaEventSynchronize(c->ev_scatter_end));
  c->restore_inflight = false;
  float t = 0.f;
  if (fill_ms) {
    FC_CUDA(cudaEventElapsedTime(&t, c->ev_fill_start, c->ev_fill_end));
    *fill_ms = t;
  }
  if (scatter_ms) {
    FC_CUDA(cudaEventElapsedTime(&t, c->ev_fill_end, c->ev_scatter_end));
    *scatter_ms = t;
  }
  if (total_ms) {
    FC_CUDA(cudaEventElapsedTime(&t, c->ev_fill_start, c->ev_scatter_end));
    *total_ms = t;
  }
  return FC_OK;
}

// ---- non-finite scan --------------------------------------------------------------
static_assert((int)FC_KIND_F16 == (int)kScanF16 && (int)FC_KIND_BF16 == (int)kScanBF16 &&
                  (int)FC_KIND_F32 == (int)kScanF32 && (int)FC_KIND_F64 == (int)kScanF64 &&
                  (int)FC_KIND_E5M2 == (int)kScanE5M2 && (int)FC_KIND_E4M3FN == (int)kScanE4M3,
              "kind codes of the header and the kernel differ");

static uint32_t kind_bytes(uint8_t kind) {
  switch (kind) {
    case FC_KIND_F16: case FC_KIND_BF16: return 2;
    case FC_KIND_F32: return 4;
    case FC_KIND_F64: return 8;
    case FC_KIND_E5M2: case FC_KIND_E4M3FN: return 1;
    default: return 0;
  }
}

extern "C" int fc_plan_set_kinds(fc_plan* p, uint32_t n, const uint8_t* kinds) {
  if (!p || (n && !kinds)) return fail(FC_EINVAL, "fc_plan_set_kinds: null argument%s%s");
  if (n != p->inputs.size())
    return fail(FC_EINVAL, "fc_plan_set_kinds: n differs from the plan's number of ranges%s%s");
  for (uint32_t i = 0; i < n; ++i)
    if (kinds[i] > FC_KIND_E4M3FN) return fail(FC_EINVAL, "fc_plan_set_kinds: unknown kind%s%s");
  if (!std::equal(kinds, kinds + n, p->kinds.begin())) {
    p->kinds.assign(kinds, kinds + n);
    p->scan_stale = true;
  }
  return FC_OK;
}

extern "C" int fc_scan_nonfinite_async(fc_plan* p, void* stream) {
  if (!p) return fail(FC_EINVAL, "fc_scan_nonfinite_async: null plan%s%s");
  fc_ctx* c = p->ctx;
  FC_GUARD(c);
  cudaStream_t s = (cudaStream_t)stream;
  const uint32_t n = (uint32_t)p->inputs.size();
  // the previous scan may still read the item table and write the result buffers
  if (p->scan_enqueued) FC_CUDA(cudaEventSynchronize(p->ev_scan));
  if (p->scan_stale) {
    // whole elements only: a range clipped inside an element (a window of the segment
    // cut at any byte) is widened by rounding its address.  Tensor data is
    // element-aligned, so the widened range stays inside the tensor.
    std::vector<FcItem> items;
    for (uint32_t i = 0; i < n; ++i) {
      const uint32_t es = kind_bytes(p->kinds[i]);
      const FcSpan& r = p->inputs[i];
      if (!es || !r.len) continue;
      uint64_t a = r.tptr & ~(uint64_t)(es - 1);
      const uint64_t end = (r.tptr + r.len + es - 1) & ~(uint64_t)(es - 1);
      while (a < end) {
        // kDefaultChunk is a multiple of every element size: cuts stay on elements
        const uint64_t len = std::min<uint64_t>(end - a, kDefaultChunk);
        FcItem it;
        it.tptr = a;
        it.aoff = p->kinds[i];
        it.nbytes = (uint32_t)len;
        it.pad0 = i;
        it.pad1 = 0;
        items.push_back(it);
        a += len;
      }
    }
    if (items.size() > 0xFFFFFFF0ull) return fail(FC_EINVAL, "scan: too many work items%s%s");
    int rc = table_set(c, p->scan, items, s, /*sync=*/false);
    if (rc) return rc;
    p->scan_stale = false;
  }
  const size_t total_at = ((size_t)n * 4 + 7) & ~(size_t)7;  // counts, then the total
  const size_t bytes = total_at + 8;
  if (bytes > p->scan_cap) {
    uint8_t* nd = nullptr;
    uint8_t* np = nullptr;
    cudaError_t e = cudaMalloc(&nd, bytes);
    if (e == cudaSuccess) e = cudaHostAlloc(&np, bytes, cudaHostAllocDefault);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      if (nd) c->dead_dev.push_back(nd);
      return fail(FC_ENOMEM, "scan buffers: %s", cudaGetErrorString(e));
    }
    if (p->scan_dev) c->dead_dev.push_back(p->scan_dev);
    if (p->scan_host) c->dead_pinned.push_back(p->scan_host);
    p->scan_dev = nd;
    p->scan_host = np;
    p->scan_cap = bytes;
  }
  FC_CUDA(cudaMemsetAsync(p->scan_dev, 0, bytes, s));
  if (p->scan.n) {
    const uint32_t grid =
        std::min<uint32_t>(p->scan.n, (uint32_t)c->sm_count * (2048u / kLsuThreads));
    fc_scan_nonfinite<<<grid, kLsuThreads, 0, s>>>(
        p->scan.dev, p->scan.n, reinterpret_cast<uint32_t*>(p->scan_dev),
        reinterpret_cast<unsigned long long*>(p->scan_dev + total_at));
    FC_CUDA(cudaGetLastError());
    c->n_kernels += 1;
  }
  FC_CUDA(cudaMemcpyAsync(p->scan_host, p->scan_dev, bytes, cudaMemcpyDeviceToHost, s));
  FC_CUDA(cudaEventRecord(p->ev_scan, s));
  p->scan_enqueued = true;
  return FC_OK;
}

extern "C" int fc_scan_wait(fc_plan* p, uint64_t* total, uint32_t* counts, uint32_t n) {
  if (!p) return fail(FC_EINVAL, "fc_scan_wait: null plan%s%s");
  if (!p->scan_enqueued) return fail(FC_EINVAL, "fc_scan_wait: no scan was enqueued%s%s");
  if (counts && n != p->inputs.size())
    return fail(FC_EINVAL, "fc_scan_wait: n differs from the plan's number of ranges%s%s");
  FC_GUARD(p->ctx);
  FC_CUDA(cudaEventSynchronize(p->ev_scan));
  const size_t nn = p->inputs.size();
  const size_t total_at = (nn * 4 + 7) & ~(size_t)7;
  if (counts) memcpy(counts, p->scan_host, nn * 4);
  if (total) memcpy(total, p->scan_host + total_at, 8);
  return FC_OK;
}
