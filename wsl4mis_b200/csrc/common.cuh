// Shared helpers for the wsl4mis_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#define WSL_API extern "C" __attribute__((visibility("default")))

// error plumbing (abi.cu)
void wsl_set_error(const char* fmt, ...);
int  wsl_check_launch(const char* what);

#define WSL_REQUIRE(cond, ...)                                  \
  do {                                                          \
    if (!(cond)) { wsl_set_error(__VA_ARGS__); return -1; }     \
  } while (0)

// SMs of the current device (132 on an H100 SXM, 114 on an H100 PCIe, fewer on a MIG slice): grids are sized in waves of
// resident CTAs over them.  Queried once per device.
inline int wsl_num_sms() {
  static int cache[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cache[dev] == 0) {
    int n = 0;
    cache[dev] = (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) ? n : 132;
  }
  return cache[dev];
}
constexpr int WSL_MAX_PARTIAL_BLOCKS = 2048;   // every reduction kernel launches <= this many CTAs
constexpr int WSL_WS_FLOATS = 1 << 20;  // per-call workspace (floats, 4 MiB), zero-initialised once; [0,64) tickets, rest partials

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Deterministic two-level reduction.  Every block reduces K per-thread values, writes them to
// partials[block*K + k]; the last block to finish (ticket) sums all partials in a fixed order into
// `result[k]` (double) and returns true on that block (all its threads).  The ticket is reset so the
// workspace can be reused by the next launch on the same stream.
template <int K, int THREADS>
__device__ bool block_reduce_final(float (&v)[K], float* partials, unsigned* ticket, double* result /*smem[K]*/) {
  __shared__ float s_w[THREADS / 32][K];
  __shared__ double s_d[THREADS / 32][K];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    float r = warp_sum(v[k]);
    if (lane == 0) s_w[warp][k] = r;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    float r = 0.f;
    for (int w = 0; w < THREADS / 32; ++w) r += s_w[w][threadIdx.x];
    partials[(size_t)blockIdx.x * K + threadIdx.x] = r;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = atomicAdd(ticket, 1u);
    s_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return false;
  __threadfence();
  double acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += THREADS) {
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] += (double)__ldcg(&partials[(size_t)b * K + k]);
  }
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double r = acc[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if (lane == 0) s_d[warp][k] = r;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double r = 0.0;
    for (int w = 0; w < THREADS / 32; ++w) r += s_d[w][threadIdx.x];
    result[threadIdx.x] = r;
  }
  if (threadIdx.x == 0) *ticket = 0u;
  __syncthreads();
  return true;
}

__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
// 8 bf16 <-> 8 floats (one 16-byte vector)
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16(f[0], f[1]); u.y = pack_bf16(f[2], f[3]);
  u.z = pack_bf16(f[4], f[5]); u.w = pack_bf16(f[6], f[7]);
  return u;
}

// fp16 twins (storage dtype code 2: kind::f16 tensor-core operands with an 11-bit mantissa)
__device__ __forceinline__ uint32_t pack_f16(float a, float b) {
  __half2 t = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ void unpack8h(const uint4& u, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { const float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
}
__device__ __forceinline__ uint4 pack8h(const float (&f)[8]) {
  uint4 u;
  u.x = pack_f16(f[0], f[1]); u.y = pack_f16(f[2], f[3]);
  u.z = pack_f16(f[4], f[5]); u.w = pack_f16(f[6], f[7]);
  return u;
}
// run-time 16-bit storage type (warp-uniform flag): 0 = bf16, 2 = fp16
__device__ __forceinline__ uint4 pack8_dt(const float (&f)[8], int dt) { return dt == 2 ? pack8h(f) : pack8(f); }
__device__ __forceinline__ void unpack8_dt(const uint4& u, float (&f)[8], int dt) {
  if (dt == 2) unpack8h(u, f); else unpack8(u, f);
}

// counter-based RNG for dropout (graph-capture safe: state lives in arguments, not in a generator)
__device__ __forceinline__ uint32_t wsl_hash32(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
  return (uint32_t)x;
}
__device__ __forceinline__ float wsl_uniform(uint64_t seed, uint64_t idx) {
  return (wsl_hash32(seed * 0x9E3779B97F4A7C15ULL + idx) >> 8) * (1.0f / 16777216.0f);
}

// 8 x 16 random bits for one 8-element vector (two splitmix64 rounds): dropout keeps element j when r16_j >= p*65536.
__device__ __forceinline__ uint64_t wsl_splitmix64(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
__device__ __forceinline__ void wsl_rand8x16(uint64_t seed, uint32_t vec, uint32_t (&r)[8]) {
  const uint64_t a = wsl_splitmix64(seed + (uint64_t)vec * 0x9E3779B97F4A7C15ULL);
  const uint64_t b = wsl_splitmix64(a + 0xD1B54A32D192ED03ULL);
  r[0] = (uint32_t)(a & 0xffff); r[1] = (uint32_t)((a >> 16) & 0xffff); r[2] = (uint32_t)((a >> 32) & 0xffff); r[3] = (uint32_t)(a >> 48);
  r[4] = (uint32_t)(b & 0xffff); r[5] = (uint32_t)((b >> 16) & 0xffff); r[6] = (uint32_t)((b >> 32) & 0xffff); r[7] = (uint32_t)(b >> 48);
}
