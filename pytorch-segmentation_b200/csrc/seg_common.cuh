// seg_common.cuh — shared helpers for the sm_90a segmentation kernels (error plumbing, bf16 vector helpers,
// launch accounting).  Internal header; the public C ABI is include/seg_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include "../../include/seg_b200.h"

namespace seg {

void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;

inline int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return 1;
  }
  return 0;
}

#define SEG_REQUIRE(cond, ...)        \
  do {                                \
    if (!(cond)) {                    \
      seg::set_error(__VA_ARGS__);    \
      return 1;                       \
    }                                 \
  } while (0)

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---- bf16x8 (16-byte) vector helpers ----
struct __align__(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void unpack8(const bf16x8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float* f) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}
__device__ __forceinline__ float bf2f(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ __nv_bfloat16 f2bf(float x) { return __float2bfloat16_rn(x); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// counter-based RNG for dropout: splitmix64 finaliser over (seed, element index) -> uniform [0,1)
__device__ __forceinline__ float hash_uniform(uint64_t seed, uint64_t idx) {
  uint64_t z = seed + idx * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

// ---- programmatic dependent launch (PDL) -------------------------------------------------------------------------
// The hot kernels of the train step are launched with the programmatic-stream-serialization attribute: their CTAs may be
// scheduled, and run their prologue, while the previous kernel in the stream drains.  Every such kernel executes
// pdl_wait() before its first global-memory access (it returns once the previous grid has COMPLETED and flushed), so the
// data flow is unchanged; pdl_trigger() at the top lets the next kernel do the same with this one.  Both instructions
// are no-ops in a kernel launched the ordinary way.  Inside the CUDA-graph replay of the step the launch gaps are already
// hidden, so it is OFF by default; SEG_PDL=1 in the environment turns it on.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("SEG_PDL");
    v = e ? atoi(e) : 0;
  }
  return v != 0;
}

template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace seg
