// fc_items.h — work-item / range types and pacing constants shared by the kernels
// (fc_kernels.cuh) and the host side (flashckpt.cu).
#pragma once

#include <stdint.h>

// --------------------------------------------------------------- work items --

// One work item = one contiguous byte range of one tensor, <= chunk_bytes.
// 32 bytes so a CTA fetches it with two 16-B loads.
struct __align__(16) FcItem {
  uint64_t tptr;    // device address inside the tensor
  uint64_t aoff;    // byte offset inside the arena (== offset in the shm segment)
  uint32_t nbytes;  // > 0
  uint32_t pad0;
  uint64_t pad1;
};
static_assert(sizeof(FcItem) == 32, "FcItem must be 32 bytes");

struct FcRun {  // merged range, contiguous in the arena AND in the segment (DMA granularity)
  uint64_t off;   // arena offset
  uint64_t len;
  uint64_t hoff;  // offset in the host segment (== off unless the plan compacts the arena)
};

struct FcSpan {  // one input range (a tensor's bytes), ascending SEGMENT offset
  uint64_t tptr;
  uint64_t off;   // offset in the host segment
  uint64_t len;
};

constexpr int kLsuThreads = 256;
constexpr int kLsuUnroll = 4;
constexpr uint32_t kDefaultChunk = 256u << 10;      // work-item size
constexpr uint64_t kDmaPiece = 256ull << 20;        // restore fill memcpy size
// Drain pacing (tools/d2h_probe2.py shows it): while a stream has ANOTHER D2H
// copy queued behind the one in flight, the copy engine keeps serving that
// stream, and a small D2H copy from any other stream of the process (a
// `loss.item()`!) starves until the whole checkpoint has left the device.  With
// exactly ONE piece in flight the engine's queue empties for a moment after every piece and the foreign copy
// goes through after at most one piece.  The pump thread therefore submits piece
// k+1 only after piece k completed.
// Piece size: each `.item()` a training loop issues during the drain waits for
// the piece in flight, so smaller pieces lose less of the step and a little
// checkpoint throughput; the default favours the stall.  fc_set_drain /
// DLROVER_B200_DRAIN_PIECE_MB change it.
constexpr uint64_t kDrainPiece = 16ull << 20;
constexpr int kDrainDepth = 1;
constexpr int kDrainRing = 8;
