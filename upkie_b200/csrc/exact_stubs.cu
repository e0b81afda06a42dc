// SPDX-License-Identifier: Apache-2.0
// Exact-arithmetic companion library (build.py: build_exact): it holds the device-buffer step kernels of families 0-2
// only (the dispatch of upkie_b200.cu narrows to them), and no flush of the in-kernel rollout transport.
#include "kernel_common.cuh"

namespace upkie_b200 {
cudaError_t launch_push_rows(const PeerPtrs&, int, cudaStream_t) { return cudaErrorNotSupported; }
}  // namespace upkie_b200
