// Device-resident step state of a training loop replayed from a CUDA graph (kgrec_b200.GraphedTrainLoop).
//
// A captured launch keeps the by-value arguments it was captured with, so everything that changes from one step to
// the next lives in a kgrec_step_state in device memory: the step count (Adam's t, and the offset of the Gumbel and
// sampler seeds), the epoch mark and the learning rate.  A step begins with
//   k_batch_gather   the batch's id columns from the shuffled visiting order at the batch cursor (DeviceTrainIterator)
//   k_step_advance   step += 1, epoch += 1, cursor += batch
// and the `_dev` entry points of the samplers, the loss steps and the sparse-row optimizer read the state after that.
#include "common.cuh"

namespace kgrec {

constexpr int kMaxGatherCols = 4;

struct GatherArgs {
  const int64_t* order;
  int64_t n_order;
  const int64_t* cursor;
  const void* src[kMaxGatherCols];
  void* dst[kMaxGatherCols];
  int n_cols;
  int is64;
  int64_t n_rows, batch;
  int32_t* status;
};

__global__ void k_step_advance(kgrec_step_state* state, int64_t* cursor, int64_t batch) {
  state->step += 1;
  state->epoch += 1;
  if (cursor) *cursor += batch;
}

__global__ void __launch_bounds__(256) k_batch_gather(const GatherArgs A) {
  const int64_t c0 = __ldg(A.cursor);
  bool bad = false;
  for (int64_t j = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; j < A.batch;
       j += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t p = c0 + j;
    int64_t row = 0;
    if (p >= 0 && p < A.n_order) row = __ldg(A.order + p);
    else bad = true;
    if (static_cast<uint64_t>(row) >= static_cast<uint64_t>(A.n_rows)) { bad = true; row = 0; }
#pragma unroll
    for (int c = 0; c < kMaxGatherCols; ++c) {
      if (c >= A.n_cols) break;
      if (A.is64) static_cast<int64_t*>(A.dst[c])[j] = __ldg(static_cast<const int64_t*>(A.src[c]) + row);
      else static_cast<int32_t*>(A.dst[c])[j] = __ldg(static_cast<const int32_t*>(A.src[c]) + row);
    }
  }
  if (bad && A.status) *A.status = 1;
}

}  // namespace kgrec

using namespace kgrec;

extern "C" int kgrec_step_advance(kgrec_step_state* state, int64_t* cursor, int64_t batch, kgrec_stream_t stream) {
  if (!state || batch < 0) { set_error("kgrec_step_advance: NULL state or negative batch"); return KGREC_ERR_INVALID; }
  k_step_advance<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(state, cursor, batch);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}

extern "C" int kgrec_batch_gather(const int64_t* order, int64_t n_order, const int64_t* cursor, const void* const* cols,
                                  void* const* out, int n_cols, int idx_bytes, int64_t n_rows, int64_t batch,
                                  int32_t* status, kgrec_stream_t stream) {
  if (!order || !cursor || !cols || !out || n_cols < 1 || n_cols > kMaxGatherCols || (idx_bytes != 4 && idx_bytes != 8) ||
      n_order < 1 || n_rows < 1 || batch < 0) {
    set_error("kgrec_batch_gather: bad arguments (1..%d columns of 4- or 8-byte ids)", kMaxGatherCols);
    return KGREC_ERR_INVALID;
  }
  GatherArgs A{};
  A.order = order; A.n_order = n_order; A.cursor = cursor; A.n_cols = n_cols; A.is64 = idx_bytes == 8;
  A.n_rows = n_rows; A.batch = batch; A.status = status;
  for (int c = 0; c < n_cols; ++c) {
    if (!cols[c] || !out[c]) { set_error("kgrec_batch_gather: column %d is NULL", c); return KGREC_ERR_INVALID; }
    A.src[c] = cols[c];
    A.dst[c] = out[c];
  }
  if (batch == 0) return KGREC_OK;
  const int64_t blocks = (batch + 255) / 256, cap = static_cast<int64_t>(sm_count()) * 4;
  k_batch_gather<<<static_cast<int>(blocks < cap ? blocks : cap), 256, 0, static_cast<cudaStream_t>(stream)>>>(A);
  KGREC_CUDA_OK(cudaGetLastError());
  return KGREC_OK;
}
