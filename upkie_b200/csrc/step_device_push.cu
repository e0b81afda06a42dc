// SPDX-License-Identifier: Apache-2.0
// TILE=0 instantiations of the table family with the push randomisation (NOISE=6: joint-limit rows, per-env table
// reads, pushes; upkie_b200_set_push_randomization). Their own translation unit, so that the NOISE=5 kernels keep the
// code, and the arithmetic, they had before pushes existed. See kernel_common.cuh.
#define UPKIE_STEP_PUSH_TU 6
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_device_push(const StepArgs& a) { return launch_step_kernels<0>(a); }
}  // namespace upkie_b200
