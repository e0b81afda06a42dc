// SPDX-License-Identifier: Apache-2.0
// TILE=0 instantiations of the body-contact family with the push randomisation (NOISE=7: joint-limit rows,
// body-ground contact rows, pushes). Their own translation unit, so that the NOISE=4 kernels keep their code. See
// kernel_common.cuh.
#define UPKIE_STEP_PUSH_TU 7
#define UPKIE_BODY_CONTACTS_BUILD 1
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_device_body_push(const StepArgs& a) { return launch_step_kernels<0>(a); }
}  // namespace upkie_b200
