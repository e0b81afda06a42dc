// SPDX-License-Identifier: Apache-2.0
//
// mpc.cuh -- batched MPC balancer: kernel + handle management.
// One thread = one robot's horizon-N box-constrained LQ problem; the per-step
// Riccati gains (5 N floats per robot) live in shared memory laid out
// [5 N][blockDim] (conflict-free: consecutive robots hit consecutive banks),
// followed by the handle's free-tail tables (20 N floats, mpc_core.cuh), which
// every block copies from global memory once.
#pragma once

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <new>
#include <string>

#include "../../include/upkie_b200.h"
#include "mpc_core.cuh"

namespace upkie_b200 {

template <typename Real>
inline int make_mpc_params(const UpkieMpcConfig& c, MpcParams<Real>& M, std::string& err) {
  if (c.nb_timesteps < 1 || c.nb_timesteps > 64) {
    err = "mpc: nb_timesteps must be in [1, 64]";
    return UPKIE_B200_EINVAL;
  }
  if (!(c.leg_length > 0) || !(c.sampling_period > 0) || !(c.max_ground_accel > 0)) {
    err = "mpc: leg_length, sampling_period and max_ground_accel must be positive";
    return UPKIE_B200_EINVAL;
  }
  // qpmpc WheeledInvertedPendulum discretisation (third-party, restated; see oracle/upkie_oracle.cpp MpcOracle)
  const double Ts = c.sampling_period, g = c.gravity;
  const double om = std::sqrt(g / c.leg_length);
  const double ch = std::cosh(Ts * om), sh = std::sinh(Ts * om);
  M.Ts = Real(Ts);
  M.ch = Real(ch);
  M.sho = Real(sh / om);
  M.osh = Real(om * sh);
  M.b0 = Real(Ts * Ts / 2.0);
  M.b1 = Real(-ch / g + 1.0 / g);
  M.b2 = Real(Ts);
  M.b3 = Real(-om * sh / g);
  M.w_u = Real(c.stage_input_cost_weight);
  M.w_x = Real(c.stage_state_cost_weight);
  M.w_T = Real(c.terminal_cost_weight);
  M.a_max = Real(c.max_ground_accel);
  M.v_max = Real(c.max_ground_velocity);
  M.fall_pitch = Real(c.fall_pitch);
  M.N = c.nb_timesteps;
  M.max_iterations = c.max_iterations > 0 ? c.max_iterations : 30;
  return 0;
}

struct MpcHandle {
  uint32_t magic;
  int n, device, block;
  MpcParams<float> M;
  float* plan = nullptr;      // [N][n] last optimal input sequence
  float* tab = nullptr;       // [N][kMpcTabRow] free-tail tables (mpc_core.cuh), built in double precision at create
  uint64_t* active = nullptr;  // [2][n] warm-start active sets (upper, lower)
  size_t smem;
};
constexpr uint32_t kMpcMagic = 0x55504D43u;

__global__ void k_mpc_step(const __grid_constant__ MpcParams<float> M, int n, const float* __restrict__ x0_all,
                           const float* __restrict__ v_target, const uint8_t* __restrict__ floor_contact, float dt,
                           float* __restrict__ v_cmd, float* __restrict__ first_input, uint8_t* __restrict__ found,
                           float* __restrict__ plan, uint64_t* __restrict__ active, const float* __restrict__ tab_g) {
  extern __shared__ float smem[];
  float* tab = smem + size_t(5) * M.N * blockDim.x;
  {
    // 20 N floats = 5 N float4 (both 16 B aligned): all loads of a lane are issued before the first store, so the copy
    // costs one L2 round trip instead of one per element (ncu: the dependent LDG -> STS pairs of the scalar loop were
    // a quarter of the kernel's stall samples)
    const float4* src = reinterpret_cast<const float4*>(tab_g);
    float4* dst = reinterpret_cast<float4*>(tab);
    const int n4 = M.N * (kMpcTabRow / 4);
#pragma unroll 4
    for (int k = threadIdx.x; k < n4; k += blockDim.x) dst[k] = __ldg(src + k);
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  MpcScratch<float> sc{smem + threadIdx.x, int(blockDim.x)};
  const float4 xv = __ldg(reinterpret_cast<const float4*>(x0_all) + i);
  const float x0[4] = {xv.x, xv.y, xv.z, xv.w};
  // warm start: previous tick's active set (the receding horizon barely moves at 200 Hz)
  uint64_t up = active[i], lo = active[size_t(n) + i];
  float u0 = 0.f;
  const bool ok = mpc_solve(M, tab, x0, v_target[i], sc, u0, up, lo);
  active[i] = ok ? up : 0ull;
  active[size_t(n) + i] = ok ? lo : 0ull;
  for (int k = 0; k < M.N; ++k) plan[size_t(k) * n + i] = fminf(fmaxf(sc.at(k, 4), -M.a_max), M.a_max);
  const bool contact = floor_contact ? floor_contact[i] != 0 : true;
  v_cmd[i] = mpc_command_update(M, v_cmd[i], x0[1], contact, ok, u0, dt);
  if (first_input) first_input[i] = u0;
  if (found) found[i] = ok ? 1 : 0;
}

__global__ void k_mpc_reset(int n, const uint8_t* __restrict__ mask, uint64_t* __restrict__ active) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (mask && !mask[i]) return;
  active[i] = 0ull;
  active[size_t(n) + i] = 0ull;
}

__global__ void k_mpc_plan(int n, int N, const float* __restrict__ plan, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < N; ++k) out[size_t(i) * N + k] = plan[size_t(k) * n + i];
}

inline MpcHandle* as_mpc(void* p) {
  MpcHandle* h = static_cast<MpcHandle*>(p);
  return (h && h->magic == kMpcMagic) ? h : nullptr;
}

inline void mpc_destroy_impl(void* p) {
  MpcHandle* h = as_mpc(p);
  if (!h) return;
  cudaSetDevice(h->device);
  cudaFree(h->plan);
  cudaFree(h->active);
  cudaFree(h->tab);
  h->magic = 0;
  delete h;
}

inline int mpc_create_impl(const UpkieMpcConfig& c, int n, int device, void** out, std::string& err) {
  if (n < 1) { err = "mpc_create: n_robots must be >= 1"; return UPKIE_B200_EINVAL; }
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) {
    err = "mpc_create: no CUDA device available (this library has no CPU path)";
    return UPKIE_B200_ECUDA;
  }
  if (device < 0 || device >= count) { err = "mpc_create: invalid device index"; return UPKIE_B200_EINVAL; }
  MpcHandle* h = new (std::nothrow) MpcHandle();
  if (!h) { err = "mpc_create: out of host memory"; return UPKIE_B200_ENOMEM; }
  int rc = make_mpc_params(c, h->M, err);
  if (rc) { delete h; return rc; }
  h->magic = kMpcMagic;
  h->n = n;
  h->device = device;
  // 5 N floats of gains per robot in shared memory; keep blocks small so that
  // several fit per SM (227 KB) and N = 4096 spreads over 128 of the H100's 132 SMs
  h->block = 32;
  h->smem = (size_t(5) * h->M.N * h->block + size_t(h->M.N) * kMpcTabRow) * sizeof(float);
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess && h->smem > 48 * 1024)
    e = cudaFuncSetAttribute(k_mpc_step, cudaFuncAttributeMaxDynamicSharedMemorySize, int(h->smem));
  if (e == cudaSuccess) e = cudaMalloc(&h->plan, size_t(h->M.N) * n * sizeof(float));
  if (e == cudaSuccess) e = cudaMalloc(&h->active, size_t(2) * n * sizeof(uint64_t));
  if (e == cudaSuccess) e = cudaMemset(h->plan, 0, size_t(h->M.N) * n * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(h->active, 0, size_t(2) * n * sizeof(uint64_t));
  if (e == cudaSuccess) e = cudaMalloc(&h->tab, size_t(h->M.N) * kMpcTabRow * sizeof(float));
  if (e == cudaSuccess) {
    MpcParams<double> Md;
    std::string e2;
    make_mpc_params(c, Md, e2);
    float host_tab[64 * kMpcTabRow];
    mpc_build_tables(Md, host_tab);
    e = cudaMemcpy(h->tab, host_tab, size_t(h->M.N) * kMpcTabRow * sizeof(float), cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    err = std::string("mpc_create: ") + cudaGetErrorString(e);
    mpc_destroy_impl(h);
    return UPKIE_B200_ECUDA;
  }
  *out = h;
  return 0;
}

inline int mpc_reset_impl(void* p, const uint8_t* mask, cudaStream_t s, std::string& err) {
  MpcHandle* h = as_mpc(p);
  if (!h) { err = "invalid mpc handle"; return UPKIE_B200_EINVAL; }
  cudaSetDevice(h->device);
  k_mpc_reset<<<(h->n + 127) / 128, 128, 0, s>>>(h->n, mask, h->active);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { err = cudaGetErrorString(e); return UPKIE_B200_ECUDA; }
  return 0;
}

inline int mpc_step_impl(void* p, const float* x0, const float* v_target, const uint8_t* contact, float dt, float* v_cmd,
                         float* first_input, uint8_t* found, cudaStream_t s, std::string& err) {
  MpcHandle* h = as_mpc(p);
  if (!h) { err = "invalid mpc handle"; return UPKIE_B200_EINVAL; }
  if (!x0 || !v_target || !v_cmd) { err = "mpc_step: null buffer"; return UPKIE_B200_EINVAL; }
  cudaSetDevice(h->device);
  const int grid = (h->n + h->block - 1) / h->block;
  k_mpc_step<<<grid, h->block, h->smem, s>>>(h->M, h->n, x0, v_target, contact, dt, v_cmd, first_input, found,
                                             h->plan, h->active, h->tab);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { err = cudaGetErrorString(e); return UPKIE_B200_ECUDA; }
  return 0;
}

inline int mpc_plan_impl(void* p, float* out, cudaStream_t s, std::string& err) {
  MpcHandle* h = as_mpc(p);
  if (!h || !out) { err = "mpc_plan: invalid argument"; return UPKIE_B200_EINVAL; }
  cudaSetDevice(h->device);
  k_mpc_plan<<<(h->n + 127) / 128, 128, 0, s>>>(h->n, h->M.N, h->plan, out);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { err = cudaGetErrorString(e); return UPKIE_B200_ECUDA; }
  return 0;
}

}  // namespace upkie_b200
