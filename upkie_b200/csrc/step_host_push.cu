// SPDX-License-Identifier: Apache-2.0
// TILE=1 instantiations of the table family with the push randomisation (NOISE=6), see step_device_push.cu.
#define UPKIE_STEP_PUSH_TU 6
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_host_push(const StepArgs& a) { return launch_step_kernels<1>(a); }
}  // namespace upkie_b200
