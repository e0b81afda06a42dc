// SPDX-License-Identifier: Apache-2.0
// TILE=1 instantiations of the body-contact family with the push randomisation (NOISE=7), see
// step_device_body_push.cu.
#define UPKIE_STEP_PUSH_TU 7
#define UPKIE_BODY_CONTACTS_BUILD 1
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_host_body_push(const StepArgs& a) { return launch_step_kernels<1>(a); }
}  // namespace upkie_b200
