// SPDX-License-Identifier: Apache-2.0
// One translation unit of step kernels, compiled once per row of build.py's unit table: the explicit instantiations of
// launch_step for one TILE (UPKIE_STEP_TILE) and one or two families (UPKIE_STEP_FAMILY0, UPKIE_STEP_FAMILY1), with
// UPKIE_BODY_CONTACTS_BUILD set to their `body` trait. See step_family.h and DESIGN.md section 4.
#include "step_kernel.cuh"

namespace upkie_b200 {

#if UPKIE_STEP_TILE == 2 && UPKIE_STEP_FAMILY0 == 0  // FAM_PLAIN
// NVSwitch-multicast instantiations (TILE=2): the TILE=1 tile path whose compact observation rows and `terminated`
// words leave through multimem.st to the multicast address of a symmetric rollout buffer, so that every GPU's buffer
// receives them without a collective. The last rows of a rollout have no later launch to ride on: a small kernel of
// their own.
namespace {
__global__ void k_push_rows(const __grid_constant__ PeerPtrs pp, int n) {
  const int wb = (blockIdx.x * blockDim.x + threadIdx.x) & ~31;
  if (wb + 32 <= n) push_rows(pp, wb, threadIdx.x & 31);
}
}  // namespace

cudaError_t launch_push_rows(const PeerPtrs& pp, int n, cudaStream_t stream) {
  k_push_rows<<<(n + 127) / 128, 128, 0, stream>>>(pp, n);
  return cudaGetLastError();
}
#endif

template cudaError_t launch_step<UPKIE_STEP_TILE, UPKIE_STEP_FAMILY0>(const StepArgs&);
#ifdef UPKIE_STEP_FAMILY1
template cudaError_t launch_step<UPKIE_STEP_TILE, UPKIE_STEP_FAMILY1>(const StepArgs&);
#endif
#ifdef UPKIE_STEP_FAMILY2
#error "a step unit holds one or two families"
#endif

}  // namespace upkie_b200
