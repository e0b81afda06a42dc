// SPDX-License-Identifier: Apache-2.0
// TILE=1 instantiations with joint-limit rows and the reads of the per-env parameter table (NOISE=5), see
// step_device_table.cu.
#define UPKIE_STEP_TABLE_TU 1
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
cudaError_t launch_step_host_table(const StepArgs& a) { return launch_step_kernels<1>(a); }
}  // namespace upkie_b200
