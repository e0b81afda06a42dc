// SPDX-License-Identifier: Apache-2.0
// Host-buffer tile step kernels (TILE=1) of the body-contact family with pushes and the action delay. See step_family.h.
#define UPKIE_BODY_CONTACTS_BUILD 1
#include "step_kernel.cuh"

namespace upkie_b200 {
template cudaError_t launch_step<1, FAM_BODY_DELAY>(const StepArgs&);
}  // namespace upkie_b200
