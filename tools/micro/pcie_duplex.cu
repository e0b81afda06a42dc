// SPDX-License-Identifier: Apache-2.0
// Developer microbenchmark: what the host<->device leg of one env step can reach on this box.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pcie_duplex pcie_duplex.cu && ./pcie_duplex
// Measures pinned H2D (9.4 MB = 65536 x 144 B) and D2H (8.3 MB = 65536 x 126 B) alone, concurrently on two streams
// (full duplex), chunked, and through zero-copy (SM loads/stores on mapped pinned memory).
#include <chrono>
#include <cstdio>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

__global__ void zc_read(const float4* __restrict__ src, float4* __restrict__ dst, size_t n) {
  for (size_t i = blockIdx.x * size_t(blockDim.x) + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) dst[i] = src[i];
}
// one thread = one env: 9 x float4 in (144 B), then 30 floats out as 15 float2 (like k_step)
__global__ void zc_env(const float4* __restrict__ act, float2* __restrict__ obs, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { const float4 v = act[size_t(i) * 9 + k]; s += v.x + v.y + v.z + v.w; }
#pragma unroll
  for (int k = 0; k < 15; ++k) obs[size_t(i) * 15 + k] = make_float2(s, s + k);
}


// Persistent-block pipeline shaped like k_step<TILE=1>: cp.async prefetch of the next tile's action rows, a spin of
// `delay` cycles standing in for the physics, coalesced observation rows out. mode bit0 = read actions from `act`
// (else skip), bit1 = write observations.
__device__ __forceinline__ void cpa16(void* d, const void* s) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(uint32_t(__cvta_generic_to_shared(d))), "l"(s) : "memory");
}
__global__ void zc_pipeline(const float4* __restrict__ act, float4* __restrict__ obs, int n, long long delay, int mode) {
  extern __shared__ float4 sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float4* buf[2] = {sm + warp * 288, sm + (nw + warp) * 288};
  const int ntiles = n / blockDim.x;
  auto prefetch = [&](int t, float4* dst) {
    if (mode & 1) {
      const float4* src = act + size_t(t * blockDim.x + warp * 32) * 9;
      for (int k = 0; k < 9; ++k) cpa16(dst + k * 32 + lane, src + k * 32 + lane);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  int t = blockIdx.x, it = 0;
  if (t < ntiles) prefetch(t, buf[0]);
  for (; t < ntiles; t += gridDim.x, ++it) {
    const int nt = t + gridDim.x;
    if (nt < ntiles) { prefetch(nt, buf[(it + 1) & 1]); asm volatile("cp.async.wait_group 1;" ::: "memory"); }
    else asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    float4* b = buf[it & 1];
    float s = 0.f;
    for (int k = 0; k < 9; ++k) { const float4 v = b[lane * 9 + k]; s += v.x + v.y + v.z + v.w; }
    const long long t0 = clock64();
    while (clock64() - t0 < delay) {}
    __syncwarp();
    float2* t2 = reinterpret_cast<float2*>(b) + lane * 15;
    for (int k = 0; k < 15; ++k) t2[k] = make_float2(s, s + k);
    __syncwarp();
    if (mode & 2) {
      float4* dst = obs + size_t(t * blockDim.x + warp * 32) * 30 / 4;
      for (int k = 0; k < 8; ++k) { const int idx = k * 32 + lane; if (idx < 240) dst[idx] = b[idx]; }
    }
    __syncwarp();
  }
}

template <typename F>
double wall_ms(F f, int reps) {
  for (int i = 0; i < 3; ++i) f();
  cudaDeviceSynchronize();
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < reps; ++i) f();
  cudaDeviceSynchronize();
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / reps;
}

int main() {
  const int n = 65536;
  const size_t ab = size_t(n) * 144, ob = size_t(n) * 126;
  char *ha, *ho, *da, *dob;
  CK(cudaHostAlloc(&ha, ab, cudaHostAllocMapped));
  CK(cudaHostAlloc(&ho, ob, cudaHostAllocMapped));
  CK(cudaMalloc(&da, ab));
  CK(cudaMalloc(&dob, ob));
  cudaStream_t s1, s2, s3;
  CK(cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s3, cudaStreamNonBlocking));
  const int R = 100;
  double t;
  t = wall_ms([&] { cudaMemcpyAsync(da, ha, ab, cudaMemcpyHostToDevice, s1); cudaStreamSynchronize(s1); }, R);
  printf("H2D %.2f MB alone + sync: %.4f ms (%.1f GB/s)\n", ab / 1e6, t, ab / t / 1e6);
  t = wall_ms([&] { cudaMemcpyAsync(ho, dob, ob, cudaMemcpyDeviceToHost, s2); cudaStreamSynchronize(s2); }, R);
  printf("D2H %.2f MB alone + sync: %.4f ms (%.1f GB/s)\n", ob / 1e6, t, ob / t / 1e6);
  t = wall_ms([&] {
    cudaMemcpyAsync(da, ha, ab, cudaMemcpyHostToDevice, s1);
    cudaMemcpyAsync(ho, dob, ob, cudaMemcpyDeviceToHost, s2);
    cudaStreamSynchronize(s1); cudaStreamSynchronize(s2);
  }, R);
  printf("H2D + D2H concurrently (2 streams): %.4f ms\n", t);
  t = wall_ms([&] {
    cudaMemcpyAsync(da, ha, ab, cudaMemcpyHostToDevice, s1);
    cudaMemcpyAsync(ho, dob, ob, cudaMemcpyDeviceToHost, s1);
    cudaStreamSynchronize(s1);
  }, R);
  printf("H2D then D2H (1 stream): %.4f ms\n", t);
  for (int c : {2, 4, 8, 16}) {
    t = wall_ms([&] {
      for (int k = 0; k < c; ++k) cudaMemcpyAsync(da + k * (ab / c), ha + k * (ab / c), ab / c, cudaMemcpyHostToDevice, s1);
      cudaStreamSynchronize(s1);
    }, R);
    printf("H2D in %d chunks (1 stream): %.4f ms\n", c, t);
    t = wall_ms([&] {
      for (int k = 0; k < c; ++k) {
        cudaMemcpyAsync(da + k * (ab / c), ha + k * (ab / c), ab / c, cudaMemcpyHostToDevice, s1);
        cudaMemcpyAsync(ho + k * (ob / c), dob + k * (ob / c), ob / c, cudaMemcpyDeviceToHost, s2);
      }
      cudaStreamSynchronize(s1); cudaStreamSynchronize(s2);
    }, R);
    printf("H2D + D2H concurrently in %d chunks each: %.4f ms\n", c, t);
  }
  // zero-copy
  float4 *zha; float2* zho;
  CK(cudaHostGetDevicePointer(&zha, ha, 0));
  CK(cudaHostGetDevicePointer(&zho, ho, 0));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  for (int grid : {sms, 2 * sms, 4 * sms, 8 * sms}) {
    t = wall_ms([&] { zc_read<<<grid, 256, 0, s1>>>(zha, reinterpret_cast<float4*>(da), ab / 16); cudaStreamSynchronize(s1); }, R);
    printf("zero-copy read 9.4 MB, grid %d x 256: %.4f ms (%.1f GB/s)\n", grid, t, ab / t / 1e6);
    t = wall_ms([&] { zc_read<<<grid, 256, 0, s1>>>(reinterpret_cast<const float4*>(dob), reinterpret_cast<float4*>(ho), ob / 16); cudaStreamSynchronize(s1); }, R);
    printf("zero-copy write 8.3 MB, grid %d x 256: %.4f ms (%.1f GB/s)\n", grid, t, ob / t / 1e6);
  }
  t = wall_ms([&] { zc_env<<<n / 224 + 1, 224, 0, s1>>>(zha, zho, n); cudaStreamSynchronize(s1); }, R);
  printf("zero-copy env-shaped kernel (144 B in, 120 B out per thread, 65536 threads): %.4f ms\n", t);
  t = wall_ms([&] { zc_env<<<n / 224 + 1, 224, 0, s1>>>(reinterpret_cast<float4*>(da), reinterpret_cast<float2*>(dob), n); cudaStreamSynchronize(s1); }, R);
  printf("same kernel on device memory: %.4f ms\n", t);
  // launch + sync floor
  t = wall_ms([&] { zc_env<<<1, 32, 0, s1>>>(reinterpret_cast<float4*>(da), reinterpret_cast<float2*>(dob), 32); cudaStreamSynchronize(s1); }, R);
  printf("empty launch + stream sync: %.4f ms\n", t);
  // pipeline model of the zero-copy step kernel
  for (int block : {128, 64}) {
    for (long long delay : {0LL, 35000LL, 70000LL}) {  // cycles at ~1.9 GHz: 0, ~18 us, ~37 us
      for (int mode : {1, 2, 3}) {
        t = wall_ms([&] { zc_pipeline<<<sms, block, 2 * (block / 32) * 4608, s1>>>(zha, reinterpret_cast<float4*>(zho), n, delay, mode); cudaStreamSynchronize(s1); }, R);
        printf("zc_pipeline %d x %d, delay %lld cycles, %s: %.4f ms\n", sms, block, delay, mode == 1 ? "read only" : mode == 2 ? "write only" : "read+write", t);
      }
    }
  }
  return 0;
}
