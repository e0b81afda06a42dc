// SPDX-License-Identifier: Apache-2.0
// In-kernel rollout transport step kernels (TILE=2) of the joint-limit family. See step_family.h.
#define UPKIE_BODY_CONTACTS_BUILD 0
#include "step_kernel.cuh"

namespace upkie_b200 {
template cudaError_t launch_step<2, FAM_LIMITS>(const StepArgs&);
}  // namespace upkie_b200
