// SPDX-License-Identifier: Apache-2.0
// Device-buffer instantiations of the env-step kernel (TILE=0), see kernel_common.cuh.
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_device(const StepArgs& a) {
  if (a.noise == 4) return launch_step_device_body(a);  // step_device_body.cu
  if (a.noise == 6) return launch_step_device_push(a);  // step_device_push.cu
  if (a.noise == 7) return launch_step_device_body_push(a);  // step_device_body_push.cu
  if (a.noise == 3) return launch_step_device_spine(a);  // step_device_spine.cu
  if (a.noise == 5) return launch_step_device_table(a);  // step_device_table.cu
  if (a.noise == 2) return launch_step_device_limits(a);  // step_device_limits.cu
  return launch_step_kernels<0>(a);
}
}  // namespace upkie_b200
