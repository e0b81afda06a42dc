// SPDX-License-Identifier: Apache-2.0
// Device-buffer step kernels (TILE=0) of the spine-timing family. See step_family.h.
#define UPKIE_BODY_CONTACTS_BUILD 1
#include "step_kernel.cuh"

namespace upkie_b200 {
template cudaError_t launch_step<0, FAM_SPINE>(const StepArgs&);
}  // namespace upkie_b200
