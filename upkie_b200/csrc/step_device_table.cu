// SPDX-License-Identifier: Apache-2.0
// TILE=0 instantiations with joint-limit rows and the reads of the per-env parameter table (NOISE=5): the NOISE=2
// kernels with a table set (upkie_b200_set_env_params), see kernel_common.cuh.
#define UPKIE_STEP_TABLE_TU 1
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_device_table(const StepArgs& a) { return launch_step_kernels<0>(a); }
}  // namespace upkie_b200
