// Microbenchmark (round 2, VERDICT item 3 "measure, don't estimate"): the articulated-body passes 1-2 of one substep
// - the largest paired-leg stretch of k_step - in the two thread mappings:
//   A  lane = robot: base_inertia_bias + legs_pass12 (both legs as pairs, sim_pair.cuh), what
//      the kernels run;
//   B  lane = leg: two adjacent lanes per robot, each runs base_inertia_bias (redundantly) and the scalar leg_pass12 of
//      sim_core.cuh on its own leg, then the two halves of the base's articulated inertia / bias force (27 words) are
//      combined with __shfl_xor. OPTIMISTIC for B: every lane uses the compile-time constants of the left leg (a real
//      lane-per-leg kernel would select its leg's constants at run time: one more instruction per constant operand).
// Both run `REPS` dependent repetitions per launch (a tick has 5 substeps) and fold every output into a checksum.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --use_fast_math -o lane_per_leg_bench lane_per_leg_bench.cu
//   python -c "...write /tmp/pgs_model.bin (UpkieModel + UpkieSimConfig), see tools/r02/body_gate_stats.cpp" ; ./lane_per_leg_bench
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../upkie_b200/csrc/params.h"
using namespace upkie_b200;

constexpr int REPS = 5;

__global__ void __launch_bounds__(256) k_robot_per_lane(const __grid_constant__ SimParams P, int n, const float* __restrict__ in,
                                                        float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float q[6], qd[6], tau[6], V0[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    q[k] = in[(0 * 6 + k) * n + i]; qd[k] = in[(1 * 6 + k) * n + i]; tau[k] = in[(2 * 6 + k) * n + i]; V0[k] = in[(3 * 6 + k) * n + i];
  }
  float acc = 0.f;
  for (int r = 0; r < REPS; ++r) {
    float IA0[21], pA0[6];
    base_inertia_bias(P, V0, IA0, pA0);
    LegCache2 lc;
    f2 cc[3][6], uu[3];
    legs_pass12(P, q, qd, tau, V0, nullptr, lc, cc, uu, IA0, pA0, false);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 21; ++k) s += IA0[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) s += pA0[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      s += uu[k].x + uu[k].y + lc.invD[k].x + lc.invD[k].y;
#pragma unroll
      for (int c = 0; c < 6; ++c) s += cc[k][c].x + cc[k][c].y + lc.U[k][c].x + lc.U[k][c].y;
    }
    acc += s;
#pragma unroll
    for (int k = 0; k < 6; ++k) { q[k] += 1e-7f * s; qd[k] += 1e-6f * s; }  // the next repetition depends on this one
  }
  out[i] = acc;
}

__global__ void __launch_bounds__(256) k_leg_per_lane(const __grid_constant__ SimParams P, int n, const float* __restrict__ in,
                                                      float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = t >> 1, leg = t & 1;
  if (i >= n) return;
  // this lane's leg in the slots of the LEFT leg (compile-time constants, see the header)
  float q[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, qd[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, tau[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, V0[6];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    q[k] = in[(0 * 6 + 3 * leg + k) * n + i]; qd[k] = in[(1 * 6 + 3 * leg + k) * n + i]; tau[k] = in[(2 * 6 + 3 * leg + k) * n + i];
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) V0[k] = in[(3 * 6 + k) * n + i];
  float acc = 0.f;
  for (int r = 0; r < REPS; ++r) {
    float IA0[21], pA0[6];
    base_inertia_bias(P, V0, IA0, pA0);  // both lanes (a real kernel could halve this too)
    float IAl[21], pAl[6];
#pragma unroll
    for (int k = 0; k < 21; ++k) IAl[k] = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) pAl[k] = 0.f;
    LegCache lc;
    float cc[3][6], uu[3];
    leg_pass12<0>(P, q, qd, tau, V0, nullptr, lc, cc, uu, IAl, pAl);
    // the other leg's contribution to the base
#pragma unroll
    for (int k = 0; k < 21; ++k) IA0[k] += IAl[k] + __shfl_xor_sync(0xffffffffu, IAl[k], 1);
#pragma unroll
    for (int k = 0; k < 6; ++k) pA0[k] += pAl[k] + __shfl_xor_sync(0xffffffffu, pAl[k], 1);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 21; ++k) s += IA0[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) s += pA0[k];
    float sl = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      sl += uu[k] + lc.invD[k];
#pragma unroll
      for (int c = 0; c < 6; ++c) sl += cc[k][c] + lc.U[k][c];
    }
    s += sl + __shfl_xor_sync(0xffffffffu, sl, 1);
    acc += s;
#pragma unroll
    for (int k = 0; k < 3; ++k) { q[k] += 1e-7f * s; qd[k] += 1e-6f * s; }
  }
  if (leg == 0) out[i] = acc;
}

template <typename F>
static float time_ms(F launch, int iters) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int k = 0; k < 5; ++k) launch();
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  for (int k = 0; k < iters; ++k) launch();
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  return ms / iters;
}

int main() {
  UpkieModel m; UpkieSimConfig c;
  FILE* f = fopen("/tmp/pgs_model.bin", "rb");
  if (!f || fread(&m, sizeof(m), 1, f) != 1 || fread(&c, sizeof(c), 1, f) != 1) { fprintf(stderr, "no /tmp/pgs_model.bin\n"); return 1; }
  fclose(f);
  SimParams P; std::memset(&P, 0, sizeof(P)); std::string err;
  if (make_sim_params(m, c, P, err)) { fprintf(stderr, "%s\n", err.c_str()); return 1; }
  cudaFuncAttributes fa, fb;
  cudaFuncGetAttributes(&fa, k_robot_per_lane);
  cudaFuncGetAttributes(&fb, k_leg_per_lane);
  printf("registers / thread: lane = robot %d, lane = leg %d; local bytes %zu / %zu\n", fa.numRegs, fb.numRegs, fa.localSizeBytes, fb.localSizeBytes);
  for (int n : {4096, 16384, 65536, 262144}) {
    std::vector<float> h(size_t(24) * n);
    unsigned s = 12345u;
    for (auto& x : h) { s = s * 1664525u + 1013904223u; x = (float(s >> 8) / 16777216.f - 0.5f) * 1.2f; }
    float *in, *outA, *outB;
    cudaMalloc(&in, h.size() * 4); cudaMalloc(&outA, size_t(n) * 4); cudaMalloc(&outB, size_t(n) * 4);
    cudaMemcpy(in, h.data(), h.size() * 4, cudaMemcpyHostToDevice);
    for (int block : {128, 256}) {
      const float a = time_ms([&] { k_robot_per_lane<<<(n + block - 1) / block, block>>>(P, n, in, outA); }, 50);
      const float b = time_ms([&] { k_leg_per_lane<<<(2 * n + block - 1) / block, block>>>(P, n, in, outB); }, 50);
      std::vector<float> ra(n), rb(n);
      cudaMemcpy(ra.data(), outA, size_t(n) * 4, cudaMemcpyDeviceToHost);
      cudaMemcpy(rb.data(), outB, size_t(n) * 4, cudaMemcpyDeviceToHost);
      printf("n %7d block %3d: lane = robot %.4f ms (%.2f ns / robot-pass), lane = leg %.4f ms (%.2f ns / robot-pass)  [checksums %g %g]\n", n, block,
             a, 1e6 * a / n / REPS, b, 1e6 * b / n / REPS, ra[n / 2], rb[n / 2]);
    }
    cudaFree(in); cudaFree(outA); cudaFree(outB);
  }
  return 0;
}
