/*
 * flashckpt.h — C-ABI of libflashckpt.so, the H100 (sm_90a) device engine that
 * sits UNDER the Flash Checkpoint shared-memory handler.
 *
 * The reference (dlrover @ 468d632) has no native boundary on this path: the
 * whole "serialise a state_dict into host shared memory" step is a Python loop
 * of blocking per-tensor device->pageable-host copies
 *   dlrover/python/elastic_agent/torch/ckpt_saver.py:198-231
 *     (_traverse_copy_to_shm / _write_shared_memory: frombuffer(...).copy_(t))
 *   dlrover/trainer/torch/flash_checkpoint/fsdp_engine.py:133-155 (_write_item)
 * and the inverse on restore
 *   dlrover/python/elastic_agent/torch/ckpt_saver.py:144-161 (_read_tensor_from_buf)
 *   dlrover/trainer/torch/flash_checkpoint/fsdp_engine.py:250-308 (read_data)
 *   dlrover/trainer/torch/flash_checkpoint/megatron_dist_ckpt.py:654-683.
 * Every entry point below replaces (part of) that loop; the comment on each
 * says which lines.  A reference maintainer binds them with ctypes (see
 * INTEGRATION.md); no torch / C++ types cross this boundary.
 *
 * Conventions
 *   - every function returns FC_OK (0) or a negative FC_E* code; nothing throws;
 *     fc_last_error() gives the thread-local detail string (CUDA error text...).
 *   - the caller owns the tensors and must keep them alive and unmodified until
 *     the pack kernel of a save has finished (fc_save_pack_done / stream order);
 *     the library owns the staging arena, its streams/events and host
 *     registrations.
 *   - "arena offset" == byte offset inside the checkpoint shared-memory segment
 *     == TensorMeta.offset of the reference (ckpt_saver.py:286-301): running sum
 *     of numel*element_size, NO padding.  The arena is a byte image of the
 *     segment, so the drain is a plain DMA.
 *   - streams are passed as void* (a cudaStream_t / CUstream, e.g.
 *     torch.cuda.current_stream().cuda_stream); NULL = legacy default stream.
 */
#ifndef FLASHCKPT_H_
#define FLASHCKPT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FC_VERSION 200 /* 0.2.0 */

enum {
  FC_OK = 0,
  FC_EINVAL = -1,  /* bad argument (null handle, overlapping/oversized range...) */
  FC_ECUDA = -2,   /* a CUDA runtime call failed; see fc_last_error()            */
  FC_ENOMEM = -3,  /* host or device allocation failed                           */
  FC_EBUSY = -4,   /* a save/restore is still in flight on this context          */
  FC_ENOIMAGE = -5, /* the arena holds no image of the segment for this plan     */
  FC_EIO = -6,     /* reading the source file failed (short read, I/O error)     */
  FC_ENOTREADY = 1 /* poll: work still pending (not an error)                    */
};

/* kernel variants (fc_set_variant / fc_pack_async 'variant' argument) */
enum {
  FC_VARIANT_AUTO = 0, /* library default (FC_VARIANT_TMA) */
  FC_VARIANT_LSU = 1,  /* 128-bit LDG/STG register path for everything         */
  FC_VARIANT_TMA = 2   /* cp.async.bulk global->smem->global ring for the 16-B
                          congruent bodies + LSU kernel for heads/tails/shifted */
};

typedef struct fc_ctx fc_ctx;   /* one per (process, device)                    */
typedef struct fc_plan fc_plan; /* cached descriptor table of one state_dict    */

int fc_version(void);
const char* fc_strerror(int code);
const char* fc_last_error(void);

/* ---- context, staging arena, host segment ------------------------------- */

/* Creates the side (copy) stream + events on `device`. */
int fc_ctx_create(int device, fc_ctx** out);
int fc_ctx_destroy(fc_ctx* ctx);

/* Grow-only device staging arena (HBM image of the SHM segment).
 * Replaces nothing in the reference: it is what lets the training stream
 * resume after an HBM-speed snapshot instead of after the PCIe copy. */
int fc_arena_reserve(fc_ctx* ctx, uint64_t bytes);
int fc_arena_info(fc_ctx* ctx, void** dev_ptr, uint64_t* bytes);
/* Cap the arena (0 = no cap, minimum 8 MiB).  A plan larger than the arena is
 * then streamed through it window by window by fc_save_async/fc_restore_async
 * (gather window -> DMA -> next window).  The tensors must stay unchanged until
 * the last window is gathered, so in this mode fc_save_async returns only when
 * the whole checkpoint is in host memory (the reference's blocking behaviour,
 * at PCIe speed).  Each window drains under the context's drain pacing
 * (fc_set_drain, fc_set_drain_mode).  Use when the state does not fit in HBM a
 * second time. */
int fc_set_arena_limit(fc_ctx* ctx, uint64_t bytes);

/* Pin (cudaHostRegister) a host range the CALLER mapped — the POSIX shm
 * segment of multi_process.py:696-734 / ckpt_saver.py:164-195 — so the drain
 * is a true async DMA.  prefault_threads>0 first touches the pages from that
 * many threads (the reference pays this page-fault cost inside its first
 * copy_ loop).  Registration is per process; the agent never needs it. */
int fc_host_register(fc_ctx* ctx, void* host, uint64_t bytes, int prefault_threads);
int fc_host_unregister(fc_ctx* ctx, void* host);
/* The same pinning, off the caller's thread: a library thread registers the range
 * slice by slice (slice_bytes, 0 = 256 MiB, a pause after each so that the caller's own
 * CUDA calls get the driver lock in between; no DMA of this library ever straddles two
 * slices) and the call returns at once.  Until fc_host_ready() answers FC_OK, saves
 * and restores that touch the range go through the staged path below — so neither the
 * first save of a run nor the restore of a restarted trainer waits 3-6 s for
 * cudaHostRegister of a 16 GB segment (the reference never pins: every one of its
 * copies is a pageable cudaMemcpy, ckpt_saver.py:221-231, :144-161).
 * fc_host_ready: FC_OK pinned, FC_ENOTREADY in progress, < 0 failed / unknown range. */
int fc_host_register_background(fc_ctx* ctx, void* host, uint64_t bytes, uint64_t slice_bytes);
int fc_host_ready(fc_ctx* ctx, const void* host);
/* NUMA placement of a range that has not been touched yet (the pages of the segment
 * are faulted in by whoever writes them first): prefer the node of the context's GPU;
 * remote_per256 > 0 on a two-socket host binds that many of every 256 consecutive
 * 2-MiB blocks to the OTHER socket instead (when more GPUs of one socket drain at once
 * than its memory absorbs and the other socket is idle).  fc_host_register applies the
 * all-local policy by itself.  Best effort. */
int fc_host_bind_numa(fc_ctx* ctx, void* host, uint64_t bytes, int remote_per256);
/* NUMA node of a CUDA device (-1 unknown) and the number of nodes of the host. */
int fc_device_numa_node(int device, int* node, int* n_nodes);
/* Staged path for host ranges that are not (completely) registered: `threads` host
 * threads (default 8), each with its own stream and two pinned bounce slots of
 * slot_bytes (default 8 MiB), memcpy between segment and slot while the DMA of their
 * other slot is in flight.  Chosen automatically by fc_save_* / fc_restore_*; a
 * staged restore returns when the data is on the device.  0 keeps a value. */
int fc_set_stage(fc_ctx* ctx, int threads, uint64_t slot_bytes);

/* ---- plan: the on-device "serialisation header" -------------------------- */

/* Build the descriptor table for n device tensors (contiguous byte ranges):
 * tensor i lives at dev_ptrs[i] (nbytes[i] bytes) and is serialised at
 * arena_off[i].  Ranges must not overlap in the arena.  The table is split
 * into <= chunk_bytes work items whose interior boundaries are 128-B aligned
 * in arena space, uploaded once, and reused by every later save/restore of
 * the same state_dict structure (the reference re-walks the dict and re-plans
 * nothing either: ckpt_saver.py:307-313).  chunk_bytes==0 -> default. */
int fc_plan_create(fc_ctx* ctx, uint32_t n, const void* const* dev_ptrs,
                   const uint64_t* arena_off, const uint64_t* nbytes,
                   uint32_t chunk_bytes, fc_plan** out);
/* Re-target an existing plan at a new set of ranges (frameworks that hand out
 * fresh tensors on every state_dict() call, e.g. FSDP): the tables are rebuilt
 * on the host, staged in pinned memory and uploaded with cudaMemcpyAsync on
 * `stream` — ordered before the next kernel of this plan, never a device-wide
 * synchronisation.  FC_EBUSY while a save/restore of the context is in flight. */
int fc_plan_update(fc_plan* plan, uint32_t n, const void* const* dev_ptrs,
                   const uint64_t* arena_off, const uint64_t* nbytes, void* stream);
/* The same with the arena offset of a range independent from its offset in the host
 * segment (host_off[i]): ranges that are scattered over a large segment — one rank's
 * shards of a FULL state dict that several ranks assemble in one segment — are packed
 * into a small arena, and the drain copies arena_off -> host_off range by range (runs
 * are merged where both sides continue).  Choosing arena_off[i] congruent to dev_ptrs[i]
 * mod 16 sends every range through the bulk (TMA ring) kernel.  Ranges must not overlap
 * in the arena nor in the segment.  Hybrid and bounded-arena saves need the identity
 * mapping of fc_plan_create.  Replaces, for such a rank, the all-gather of the full
 * tensors + the saving rank's copy loop (fsdp.py:238-262, ckpt_saver.py:198-231). */
int fc_plan_create_mapped(fc_ctx* ctx, uint32_t n, const void* const* dev_ptrs,
                          const uint64_t* arena_off, const uint64_t* host_off,
                          const uint64_t* nbytes, uint32_t chunk_bytes, fc_plan** out);
int fc_plan_update_mapped(fc_plan* plan, uint32_t n, const void* const* dev_ptrs,
                          const uint64_t* arena_off, const uint64_t* host_off,
                          const uint64_t* nbytes, void* stream);
int fc_plan_destroy(fc_plan* plan);
/* total payload bytes, number of work items, number of merged arena runs,
 * end offset (max arena_off+nbytes) */
int fc_plan_info(const fc_plan* plan, uint64_t* payload_bytes, uint32_t* n_items,
                 uint32_t* n_runs, uint64_t* arena_end);
/* number of source spans (= non-empty input ranges; never merged, a DMA must not
 * straddle two device allocations): the minimum DMA count of the in-place save /
 * restore below */
int fc_plan_spans(const fc_plan* plan, uint32_t* n_spans);

/* ---- device kernels alone (tests, ncu, roofline) ------------------------- */

/* tensors -> arena.  Replaces the body of _write_shared_memory
 * (ckpt_saver.py:221-231) for all leaves at once, at HBM speed. */
int fc_pack_async(fc_plan* plan, void* stream, int variant);
/* arena -> tensors.  Replaces the per-parameter copy_ of the restore paths
 * (ckpt_saver.py:152-158 + user load_state_dict; fsdp_engine.py:303;
 * megatron_dist_ckpt.py:683). */
int fc_unpack_async(fc_plan* plan, void* stream, int variant);
/* how many of this library's kernels / DMA copies the context has enqueued
 * since creation (bench.py reports the delta over its timed region). */
int fc_launch_count(fc_ctx* ctx, uint64_t* kernels, uint64_t* memcpys);
int fc_set_variant(fc_ctx* ctx, int variant);
/* tuning knobs for the sweep in bench/ncu runs; 0 keeps the current value */
int fc_set_launch(fc_ctx* ctx, int lsu_ctas_per_sm, int tma_ctas_per_sm,
                  int tma_stages, int tma_tile_bytes);

/* same for the byte-shift kernel (ranges not congruent mod 16) */
int fc_set_shift_launch(fc_ctx* ctx, int ctas_per_sm, int in_stages, int tile_bytes);

/* ---- save: snapshot + drain ---------------------------------------------- */

/* Enqueue the pack kernel on `compute_stream` (the ONLY work the training
 * stream waits for), then on the context's copy stream — gated by an event,
 * never by a host sync — DMA every arena run to host_base+offset in
 * <= drain_piece pieces (fc_set_drain).  host_base should be
 * fc_host_register()-ed; if it is not, the copies go through the context's
 * pinned bounce slots (fc_set_stage).  One save may be in flight per context
 * (FC_EBUSY otherwise).  Replaces _traverse_copy_to_shm (ckpt_saver.py:198-218). */
int fc_save_async(fc_plan* plan, void* host_base, void* compute_stream,
                  uint64_t* ticket);
/* Same, but the drain does not start until fc_save_release(ticket): lets the
 * caller publish "segment is being written" to its peer from another thread,
 * off the training thread, before the first byte of the segment changes.
 * (In the bounded-arena mode the save is complete on return; release is a no-op.) */
int fc_save_async_held(fc_plan* plan, void* host_base, void* compute_stream, uint64_t* ticket);
int fc_save_release(fc_ctx* ctx, uint64_t ticket);
/* Drop a held save instead of releasing it (the peer could not be told that the
 * segment is about to change): no byte of the segment is touched, the ticket counts
 * as complete.  FC_EBUSY if the drain is not held any more.  Mirrors the reference
 * raising "Fail to set metadata!" (multi_process.py:648-649) from save_state_dict
 * (ckpt_saver.py:315-318) BEFORE its copy loop starts. */
int fc_save_cancel(fc_ctx* ctx, uint64_t ticket);
/* In-place save, no snapshot and no arena: the drain DMAs every span straight
 * from the source tensors into host_base+offset (paced like fc_save_async; small
 * spans share a batch).  Nothing runs on `compute_stream` — the drain is only
 * ordered after the work already queued there — so the exposed cost is the call
 * itself, but the caller must keep the tensors UNCHANGED until fc_save_poll /
 * fc_save_wait report the ticket drained (fc_save_pack_done answers the same for
 * such a ticket).  For states that do not fit in HBM twice (weights + fp32 Adam
 * moments of an 8B model: 112 GB): parameters and optimizer state are not written
 * between two optimizer steps, so a guard in front of the next step is enough.
 * hold != 0: as fc_save_async_held.  This is the asynchronous form of the
 * reference's loop (ckpt_saver.py:198-231), which blocks for the same copies. */
int fc_save_direct_async(fc_plan* plan, void* host_base, void* compute_stream, int hold,
                         uint64_t* ticket);
/* Hybrid of the two: tensors whose segment offset is >= `cut` (a tensor boundary)
 * are snapshotted into the arena (which must hold arena_end - (cut & ~127) bytes; its
 * byte 0 stands for offset `cut` rounded down to 128 B, so every range keeps its
 * alignment class and goes through the same bulk / shift kernels as a full save),
 * the tensors below `cut` are drained in place — first, so
 * that they are released as early as possible.  Spends whatever HBM is to spare on
 * shortening the time the sources stay frozen: (bytes below cut) / PCIe rate.
 * (The reference keeps the sources frozen for the whole copy, ckpt_saver.py:198-231.) */
int fc_save_hybrid_async(fc_plan* plan, void* host_base, void* compute_stream, uint64_t cut,
                         int hold, uint64_t* ticket);
/* Incremental save (opt-in).  After a save has drained, the arena is a byte image of
 * the segment; the next save of the same plan to the same host_base compares every new
 * byte with the arena byte it replaces (gather-compare kernels: 2 bytes read per
 * checkpoint byte + 1 written per changed byte), writes only what differs and drains
 * only the work items (<= chunk_bytes each) that had a difference.  The segment ends up
 * byte-identical to what fc_save_async writes.
 * The comparison is against a BASELINE: the (plan, host_base) of the last delta save
 * that drained without error.  Without a baseline the call is a normal full gather +
 * drain, which then becomes the baseline.  The library forgets the baseline whenever
 * the arena or the segment may no longer hold that image: arena reallocation, any
 * other save / restore / pack / unpack / fc_arena_fill, fc_save_cancel, a drain error,
 * fc_plan_destroy of the baseline plan, and an fc_plan_update* that changes the
 * (arena offset, segment offset, length) of any range (re-targeting the tensor
 * pointers alone keeps it).  A writer of the segment outside this context must call
 * fc_delta_invalidate.  The arena must hold the whole plan (no bounded-arena mode:
 * FC_EINVAL).  hold != 0: as fc_save_async_held. */
int fc_save_delta_async(fc_plan* plan, void* host_base, void* compute_stream, int hold,
                        uint64_t* ticket);
/* Once `ticket` has drained (FC_ENOTREADY before): the bytes its drain moved and
 * whether it was an incremental save (1) or a full one (0). */
int fc_save_delta_stats(fc_ctx* ctx, uint64_t ticket, uint64_t* drained_bytes, int* delta);
/* Forget the baseline (the next fc_save_delta_async is a full save) and the arena image
 * (the next fc_restore_from_image_async answers FC_ENOIMAGE). */
int fc_delta_invalidate(fc_ctx* ctx);

/* FC_OK once nothing of save `ticket` reads the source tensors any more (they may
 * change): its gather kernel, if any, has finished and its in-place part, if any,
 * has been drained; FC_ENOTREADY before.  fc_save_sources_wait blocks the calling
 * host thread until then. */
int fc_save_pack_done(fc_ctx* ctx, uint64_t ticket);
int fc_save_sources_wait(fc_ctx* ctx, uint64_t ticket);
/* FC_OK when all bytes are in host memory, FC_ENOTREADY while pending. */
int fc_save_poll(fc_ctx* ctx, uint64_t ticket);
int fc_save_wait(fc_ctx* ctx, uint64_t ticket);
/* device-side times of the last completed save: pack kernel, drain DMA, and
 * first-kernel-start -> last-byte-landed. */
int fc_save_timings(fc_ctx* ctx, uint64_t ticket, float* pack_ms, float* drain_ms,
                    float* total_ms);

/* Drain pacing.  While a stream has another D2H copy queued behind the one in
 * flight the copy engine keeps serving it, and every other D2H copy of the
 * process (e.g. `loss.item()`) starves until the whole checkpoint has left the
 * device.  The drain is therefore fed by a library thread that submits piece
 * k+1 only after piece k completed (default: depth 1 x 16 MiB; a foreign copy
 * then waits at most one piece, ~0.3 ms; 32 MiB pieces: +1.8 % throughput, +2 ms of
 * exposed stall per checkpoint).  0 keeps the current value. */
int fc_set_drain(fc_ctx* ctx, uint64_t piece_bytes, int depth);
/* How the pump (and the bounded-arena save, window by window) keeps "one piece in
 * flight":
 *   FC_DRAIN_HOST_PACED  the host submits piece k+1 after piece k completed (one host
 *                        round trip between two pieces; a spinning wait hides most of it);
 *   FC_DRAIN_PINGPONG    pieces alternate between two copy streams, piece k waiting on
 *                        the DEVICE for piece k-1: no stream ever has a second copy
 *                        queued, no host round trip between pieces, the host thread
 *                        sleeps in a blocking wait.  Small pieces then cost no
 *                        throughput. */
enum { FC_DRAIN_HOST_PACED = 0, FC_DRAIN_PINGPONG = 1 };
int fc_set_drain_mode(fc_ctx* ctx, int mode);

/* ---- host-resident leaves --------------------------------------------------- */

/* CPU tensors of a state_dict (optimizer step scalars, RNG state, or the whole
 * model in the CPU/gloo configuration): range i (nbytes[i] bytes at src[i]) is
 * memcpy'd to dst_base+off[i], split in equal byte shares over `threads` host
 * threads.  Needs no GPU.  Replaces the CPU-tensor case of
 * _write_shared_memory (ckpt_saver.py:221-231). */
int fc_host_pack(void* dst_base, uint32_t n, const void* const* src, const uint64_t* off,
                 const uint64_t* nbytes, int threads);
/* The inverse for CPU targets: nbytes[i] bytes at src_base+off[i] are memcpy'd to
 * dst[i] with the same byte-balanced threading.  Replaces the per-tensor
 * `param.copy_(view_on_the_segment)` loop a user runs after load_state_dict
 * (ckpt_saver.py:144-161 hands out the views) in the CPU/gloo configuration. */
int fc_host_unpack(const void* src_base, uint32_t n, void* const* dst, const uint64_t* off,
                   const uint64_t* nbytes, int threads);

/* ---- restore: fill + scatter ---------------------------------------------- */

/* DMA host_base+offset -> arena on the copy stream, then scatter
 * arena -> tensors on `stream` (gated by an event).  Inverse of fc_save_async. */
int fc_restore_async(fc_plan* plan, const void* host_base, void* stream);
/* In-place restore: H2D DMA of every span straight into the target tensors (no
 * arena, no scatter kernel); `stream` waits for the last copy.  Preferable for
 * few large spans or when HBM has no room for the arena; fc_restore_wait /
 * fc_restore_timings apply (scatter time = 0). */
int fc_restore_direct_async(fc_plan* plan, const void* host_base, void* stream);
/* Cooperative restore of a REPLICATED state (every local rank needs the whole image):
 * fill only the arena bytes [lo, hi) from host_base+[lo, hi) (plain DMA when the range
 * is page-locked, bounce slots when it is not — then the call returns with the data on
 * the device), `stream` waits for it.  The caller exchanges the slices between the local
 * ranks' arenas over NVLink (NCCL all-gather, in place) and scatters with
 * fc_unpack_async: each rank reads 1/n of the image from host memory instead of all of
 * it (the reference: every rank copies every tensor from shared memory itself,
 * ckpt_saver.py:144-161 + load_state_dict). */
int fc_arena_fill(fc_ctx* ctx, const void* host_base, uint64_t lo, uint64_t hi, void* stream);
int fc_restore_wait(fc_ctx* ctx);
int fc_restore_timings(fc_ctx* ctx, float* fill_ms, float* scatter_ms, float* total_ms);

/* ---- restore from a file ---------------------------------------------------- */

/* Restore straight from a file (a torch.save archive the agent persisted): `plan` is a
 * mapped plan (fc_plan_create_mapped) whose host offsets are FILE offsets into `fd`.  The
 * stage workers (fc_set_stage) pread each run's bytes into their pinned bounce slots and
 * DMA every slot into the arena; once all bytes are there, the plan's unpack kernels are
 * enqueued on `stream`, gated by an event.  No mmap of the file, no cudaHostRegister.
 * The call returns when the data is on the device; fc_restore_wait / fc_restore_timings
 * apply (fill = read + DMA).  When the arena is smaller than the plan (>= 8 MiB, a state
 * that does not fit in HBM twice) the plan is streamed through it window by window, as
 * fc_restore_async does.  Forgets the incremental baseline and the arena image like every
 * restore; FC_EBUSY while a save/restore is in flight.
 * FC_EIO when the file ends before the plan's last byte (checked before anything moves) or
 * a read fails; fc_last_error() names the file offset.  No scatter is enqueued then, so no
 * target tensor has changed (windowed mode: a read error after the first window leaves the
 * earlier windows restored).
 * Replaces torch.load(path, map_location="cpu") + the per-tensor pageable copy_ of
 * load_state_dict (reference full_ckpt_engine.py _load_from_storage). */
int fc_restore_file_async(fc_plan* plan, int fd, void* stream);

/* Restore from n open files in one fill and one scatter: the checkpoint of a resharded
 * job, whose shards a rank reads from several files.  The plan is a mapped plan
 * (fc_plan_create_mapped) whose host offsets lie in the virtual concatenation of the
 * files: file k owns [bases[k], bases[k+1]) and is read at offset - bases[k]; bases is
 * strictly increasing, so the files' offset 0 do not collide and the mapped plan's overlap
 * rule applies as usual.  The stage workers' pieces are cut at every base, so no pread
 * crosses a file.  An arena smaller than the plan streams it window by window, as
 * fc_restore_file_async does.  Before anything moves, every file is checked (fstat)
 * against the highest plan byte inside its range: FC_EIO when one is short, and
 * fc_last_error() names the file index and offset.  A failed read returns FC_EIO too,
 * stops every worker and enqueues no scatter.  FC_EINVAL for no files, a negative fd,
 * bases that do not increase, or a plan byte below bases[0].  FC_EBUSY and the forgotten
 * incremental baseline and image as in fc_restore_file_async, which is the call with
 * n = 1 and base 0. */
int fc_restore_files_async(fc_plan* plan, uint32_t n, const int* fds, const uint64_t* bases,
                           void* stream);

/* ---- rollback: restore from the arena image ------------------------------- */

/* After a save has drained, the arena still holds a byte image of what it wrote to the
 * segment.  The context records it: the plan's runs (arena offset -> segment offset) and
 * host_base of the last full-arena fc_save_async / fc_save_async_held or
 * fc_save_delta_async (full or incremental) that drained without error.  A rollback keeps
 * the record, and so does an fc_plan_update* that only re-targets the tensor pointers of
 * that plan.  Every event that forgets the incremental baseline forgets it too (the other
 * saves, every restore, pack / unpack, fc_arena_fill, arena reallocation, fc_save_cancel,
 * a drain error, fc_plan_destroy of that plan, an update that moves a range,
 * fc_delta_invalidate).  Bounded-arena, in-place and hybrid saves never set it.
 *
 * Restore from the arena image: if the context's arena holds, for host_base, the bytes
 * every range of `plan` restores from, enqueue the scatter arena -> tensors on `stream`
 * (the plan's unpack kernels, no DMA) and return FC_OK; fc_restore_wait /
 * fc_restore_timings apply (fill 0).  FC_ENOIMAGE when there is no image or it does not
 * cover the plan: nothing is enqueued, nothing is forgotten, the caller restores from
 * host memory.  FC_EBUSY while a save/restore is in flight.  Keeps the image and the
 * incremental baseline.
 * Coverage: every run of `plan`, as (arena offset, segment offset, length), lies inside
 * one run of the image at the same offset into that run on both sides.  A restore plan
 * over a subset of the saved ranges is covered. */
int fc_restore_from_image_async(fc_plan* plan, const void* host_base, void* stream);
/* The coverage test alone, nothing enqueued: FC_OK when the image covers `plan` for
 * host_base, FC_ENOIMAGE when not (also while the save that would set it has not drained). */
int fc_image_covers(const fc_plan* plan, const void* host_base);

/* ---- non-finite scan: refuse to overwrite a good checkpoint --------------- */

/* Element kinds of the scan.  A kind names how the exponent field sits in the bytes:
 * complex64 / complex128 are scanned as FC_KIND_F32 / FC_KIND_F64 components.
 * FC_KIND_NONE (integers, bool, the float8 kinds not listed) is not scanned. */
enum {
  FC_KIND_NONE = 0,
  FC_KIND_F16 = 1,
  FC_KIND_BF16 = 2,
  FC_KIND_F32 = 3,
  FC_KIND_F64 = 4,
  FC_KIND_E5M2 = 5,  /* float8_e5m2                                      */
  FC_KIND_E4M3FN = 6 /* float8_e4m3fn: no Inf, NaN = 0x7F / 0xFF          */
};
/* One kind byte per input range of `plan` (n = the n of its last create / update, empty
 * ranges included).  The kinds survive an fc_plan_update* with the same n (another n
 * resets them to FC_KIND_NONE).  The scan's item table is built on the next scan after a
 * create, an update or a change of kinds, and reused by every scan after that. */
int fc_plan_set_kinds(fc_plan* plan, uint32_t n, const uint8_t* kinds);
/* Enqueue on `stream` a read-only scan of the plan's source bytes (the tensors, never the
 * arena) that counts, per input range, the elements whose exponent field is all ones:
 * NaN or +-Inf (FC_KIND_E4M3FN: its NaN patterns).  A range that starts or ends inside an
 * element (a slice of the segment cut at any byte) is widened to whole elements by
 * rounding its address, so an element cut in two is counted by both halves.  No
 * device-wide synchronisation; the arena, the incremental baseline and the image record
 * are untouched, and a save may be in flight.  One scan per plan at a time: a second call
 * first waits for the previous one.  The reference has no such check: its save copies
 * whatever the tensors hold (ckpt_saver.py:198-231). */
int fc_scan_nonfinite_async(fc_plan* plan, void* stream);
/* Block the calling host thread until the plan's last scan has finished (that scan's
 * event only), then return the total number of hits and, when counts != NULL, one
 * saturating uint32 count per input range (n must then be the plan's n).  FC_EINVAL when
 * no scan was enqueued. */
int fc_scan_wait(fc_plan* plan, uint64_t* total, uint32_t* counts, uint32_t n);

#ifdef __cplusplus
}
#endif
#endif /* FLASHCKPT_H_ */
