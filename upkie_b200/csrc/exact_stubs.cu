// SPDX-License-Identifier: Apache-2.0
// Exact-arithmetic companion library (build.py: build_exact): only the device-buffer kernels are instantiated there;
// the launchers of the other families report that they are absent.
#include "kernel_common.cuh"

namespace upkie_b200 {
cudaError_t launch_step_host(const StepArgs&) { return cudaErrorNotSupported; }
cudaError_t launch_step_multicast(const StepArgs&) { return cudaErrorNotSupported; }
cudaError_t launch_push_rows(const PeerPtrs&, int, cudaStream_t) { return cudaErrorNotSupported; }
cudaError_t launch_step_device_spine(const StepArgs&) { return cudaErrorNotSupported; }
cudaError_t launch_step_device_body(const StepArgs&) { return cudaErrorNotSupported; }
cudaError_t launch_step_device_table(const StepArgs&) { return cudaErrorNotSupported; }
cudaError_t launch_step_device_push(const StepArgs&) { return cudaErrorNotSupported; }
cudaError_t launch_step_device_body_push(const StepArgs&) { return cudaErrorNotSupported; }
}  // namespace upkie_b200
