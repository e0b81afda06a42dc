// SPDX-License-Identifier: Apache-2.0
//
// action_delay.cu -- the handle-side kernels of action-delay randomisation (upkie_b200_set_action_delay; the step
// kernels apply the delay inside their ticks, step_kernel.cuh). In a translation unit of their own, so that the kernels
// of upkie_b200.cu (k_reset among them) keep their code whether or not a handle ever sets a spec: an explicit
// upkie_b200_reset draws and stops the previous commands in k_action_delay_reset, launched right before k_reset on the
// same stream.
#include "kernel_common.cuh"

namespace upkie_b200 {
namespace {

// the envs the reset takes (mask, NULL = all) draw their next delay and hold the stop row
__global__ void k_action_delay_reset(const ActionDelay* __restrict__ A, int n, const uint8_t* __restrict__ mask,
                                     uint64_t seed, uint64_t env_offset) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  action_delay_reset(*A, seed, env_offset + uint64_t(i), i);
  action_delay_fill_history(*A, i);
}

// command rows [n][UPKIE_ACT_DIM] of the columns [UPKIE_ACT_DIM][stride] (cols null: stop rows)
__global__ void k_command_rows(const float* __restrict__ cols, int n, int stride, float* __restrict__ rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int c = 0; c < UPKIE_ACT_DIM; ++c)
    rows[size_t(i) * UPKIE_ACT_DIM + c] = cols ? cols[size_t(c) * stride + i] : action_delay_stop_value(c);
}

// the columns of command rows (rows null: stop rows)
__global__ void k_command_cols(const float* __restrict__ rows, int n, int stride, float* __restrict__ cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int c = 0; c < UPKIE_ACT_DIM; ++c)
    cols[size_t(c) * stride + i] = rows ? rows[size_t(i) * UPKIE_ACT_DIM + c] : action_delay_stop_value(c);
}

int grid_of(int n) { return (n + 127) / 128; }

// rows [ages][n][dim] <-> ages 0 .. ages - 1 of the rings [K][dim][stride] (head null: row 0 is the next write)
__global__ void k_ring_copy(float* __restrict__ ring, const uint32_t* __restrict__ head, int ticks, int dim, int n,
                            int stride, int ages, float* __restrict__ rows, int to_rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = head ? head[i] : 0u;
  for (int a = 0; a < ages; ++a) {
    float* const col = ring + size_t(delay_ring_row(h, uint32_t(ticks), uint32_t(a))) * dim * stride + size_t(i);
    float* const row = rows + (size_t(a) * n + i) * dim;
    for (int k = 0; k < dim; ++k) {
      if (to_rows) row[k] = col[size_t(k) * stride];
      else col[size_t(k) * stride] = row[k];
    }
  }
}

// the rings `src` [K_src][dim][stride] (next write head[i], null: 0) into `dst` [K_dst][dim][stride] in age order, with
// row 0 of dst the next write: the ages beyond K_src are stop rows (stop) or copies of the oldest; columns = a mask of
// the columns copied (bit k, 64 bits at most), all of them for ~0
__global__ void k_ring_resize(const float* __restrict__ src, const uint32_t* __restrict__ head, int src_ticks,
                              float* __restrict__ dst, int dst_ticks, int dim, int n, int stride, int stop,
                              uint64_t columns) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = head ? head[i] : 0u;
  for (int a = 0; a < dst_ticks; ++a) {
    const int sa = a < src_ticks ? a : src_ticks - 1;
    const float* const s = src + size_t(delay_ring_row(h, uint32_t(src_ticks), uint32_t(sa))) * dim * stride + i;
    float* const d = dst + size_t(delay_ring_row(0u, uint32_t(dst_ticks), uint32_t(a))) * dim * stride + i;
    for (int k = 0; k < dim; ++k)
      if ((columns >> k) & 1u) d[size_t(k) * stride] = (stop && a >= src_ticks) ? action_delay_stop_value(k) : s[size_t(k) * stride];
  }
}

}  // namespace

cudaError_t launch_action_delay_reset(const ActionDelay* A, int n, const uint8_t* mask, uint64_t seed,
                                      uint64_t env_offset, cudaStream_t stream) {
  k_action_delay_reset<<<grid_of(n), 128, 0, stream>>>(A, n, mask, seed, env_offset);
  return cudaGetLastError();
}

cudaError_t launch_command_rows(const float* cols, int n, int stride, float* rows, cudaStream_t stream) {
  k_command_rows<<<grid_of(n), 128, 0, stream>>>(cols, n, stride, rows);
  return cudaGetLastError();
}

cudaError_t launch_command_cols(const float* rows, int n, int stride, float* cols, cudaStream_t stream) {
  k_command_cols<<<grid_of(n), 128, 0, stream>>>(rows, n, stride, cols);
  return cudaGetLastError();
}

cudaError_t launch_ring_rows(const float* ring, const uint32_t* head, int ticks, int dim, int n, int stride, int ages,
                             float* rows, cudaStream_t stream) {
  k_ring_copy<<<grid_of(n), 128, 0, stream>>>(const_cast<float*>(ring), head, ticks, dim, n, stride, ages, rows, 1);
  return cudaGetLastError();
}

cudaError_t launch_ring_cols(const float* rows, const uint32_t* head, int ticks, int dim, int n, int stride, int ages,
                             float* ring, cudaStream_t stream) {
  k_ring_copy<<<grid_of(n), 128, 0, stream>>>(ring, head, ticks, dim, n, stride, ages, const_cast<float*>(rows), 0);
  return cudaGetLastError();
}

cudaError_t launch_ring_resize(const float* src, const uint32_t* head, int src_ticks, float* dst, int dst_ticks,
                               int dim, int n, int stride, int stop, uint64_t columns, cudaStream_t stream) {
  k_ring_resize<<<grid_of(n), 128, 0, stream>>>(src, head, src_ticks, dst, dst_ticks, dim, n, stride, stop, columns);
  return cudaGetLastError();
}

}  // namespace upkie_b200
