// inflate.cuh -- the GPU zlib decoder and the batch pipeline that brings compressed segments of a
// file to the device (both in inflate.cu).  Users: geotiff.cu (GeoTIFF segments) and decode.cu
// (cutout chunks).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <vector>

namespace atl {

constexpr int64_t SEG_ALIGN = 16;  // segment starts in the batch buffers
inline int64_t seg_align_up(int64_t v) { return (v + SEG_ALIGN - 1) / SEG_ALIGN * SEG_ALIGN; }

// Where one zlib stream sits: its compressed bytes in the input buffer and its decoded span in the
// output buffer (starts SEG_ALIGN-aligned).
struct InflSpan {
  int64_t in_off, in_bytes, out_off, out_bytes;
};

// Inflate n streams with one warp each: stream k is described by the InflSpan at the start of
// spans + k * stride (a device array of the caller's descriptors that begin with one), and
// status[k] gets its ATL_INFLATE_* status.
cudaError_t launch_inflate(const uint8_t* in, uint8_t* out, const void* spans, size_t stride, int n,
                           int32_t* status, cudaStream_t st);
const char* inflate_status_text(int status);

// Segments of one file brought to the device batch by batch: the segments of a batch are read with
// parallel pread into a pinned buffer, copied on a copy stream while the previous batch's kernels
// run, and then handed to the caller's kernels on the caller's stream.
struct SegmentBatches {
  const int64_t* file_offset = nullptr;  // per segment k: where its bytes start in the file,
  const int64_t* read_bytes = nullptr;   // how many are read,
  const int64_t* xfer_off = nullptr;     // and where they go in their batch's transfer buffer
  std::vector<int64_t> batch_start;      // batch b = segments [batch_start[b], batch_start[b + 1])
  int64_t max_xfer = 0;                  // transfer bytes of the largest batch
  const void* desc = nullptr;            // per-segment descriptors (desc_bytes each) that go with
  size_t desc_bytes = 0;                 //   every batch to the device
  int n_threads = 0;                     // readers (0: one per CPU, at most 64)
};

// launch(slot, k0, n, xfer_dev, desc_dev, status_dev): enqueue the kernels of segments [k0, k0 + n)
// on the stream; slot (0 or 1) names the double buffer the batch is in, so the caller can keep
// per-slot device scratch.  status_dev points at the n statuses of the batch (zeroed).
using SegmentLaunch = std::function<cudaError_t(int, int64_t, int, const uint8_t*, const void*, int32_t*)>;

// Runs every batch and returns ATL_OK with status[k] for every segment (read back once, after the
// last batch), ATL_ERR_INVALID with *bad_k = k when the file ends inside segment k (no message
// set: the caller names the segment) or -1 when the file cannot be opened, or a CUDA error.
int run_segment_batches(int device, const char* path, const SegmentBatches& S, cudaStream_t st,
                        const SegmentLaunch& launch, std::vector<int32_t>& status, int64_t* bad_k);

}  // namespace atl
