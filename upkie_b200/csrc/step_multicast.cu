// SPDX-License-Identifier: Apache-2.0
// NVSwitch-multicast instantiations of the env-step kernel (TILE=2): the TILE=1 tile path whose compact observation
// rows and `terminated` words leave through multimem.st to the multicast address of a symmetric rollout buffer, so
// that every GPU's buffer receives them without a collective: the plain and extras families, UpkieServos only.
// See step_family.h.
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
namespace {
// the last rows of a rollout have no later launch to ride on: a small kernel of their own
__global__ void k_push_rows(const __grid_constant__ PeerPtrs pp, int n) {
  const int wb = (blockIdx.x * blockDim.x + threadIdx.x) & ~31;
  if (wb + 32 <= n) push_rows(pp, wb, threadIdx.x & 31);
}
}  // namespace

cudaError_t launch_push_rows(const PeerPtrs& pp, int n, cudaStream_t stream) {
  k_push_rows<<<(n + 127) / 128, 128, 0, stream>>>(pp, n);
  return cudaGetLastError();
}

template cudaError_t launch_step<2, FAM_PLAIN>(const StepArgs&);
template cudaError_t launch_step<2, FAM_EXTRAS>(const StepArgs&);
}  // namespace upkie_b200
