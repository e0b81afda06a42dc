// SPDX-License-Identifier: Apache-2.0
// Host-buffer / coalesced-tile instantiations of the env-step kernel (TILE=1), see kernel_common.cuh.
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_host(const StepArgs& a) {
  if (a.noise == 4) return launch_step_host_body(a);  // step_host_body.cu
  if (a.noise == 6) return launch_step_host_push(a);  // step_host_push.cu
  if (a.noise == 7) return launch_step_host_body_push(a);  // step_host_body_push.cu
  if (a.noise == 3) return launch_step_host_spine(a);  // step_host_spine.cu
  if (a.noise == 5) return launch_step_host_table(a);  // step_host_table.cu
  if (a.noise == 2) return launch_step_host_limits(a);  // step_host_limits.cu
  return launch_step_kernels<1>(a);
}
}  // namespace upkie_b200
