// wgmma implicit-GEMM convolution for sm_90a (3x3 pad 1 / 1x1) on channels-last bf16 activations.
//
//   D[128 pixels, NT couts] (fp32, registers) = sum_{tap} sum_{kblock} A_tap[128 x KBLK] * B_tap[KBLK x NT]
//
//   * A: one TMA 4-D box (KBLK channels x 16 w x 8 h x 1 image) per (tap, k-block) at the tap-shifted pixel
//     coordinate; TMA's out-of-bounds zero fill IS the convolution's zero padding (im2col-free).
//   * B: packed weights [tap][Cout][Cin] bf16 (K-major), one 3-D box (KBLK x NT x 1) per (tap, k-block).
//   * both land in 128B/64B/32B-swizzled shared memory (swizzle span = KBLK*2 bytes) and are consumed by
//     wgmma.mma_async (M = 64, N = NT, K = 16) straight from shared memory; fp32 accumulators in registers.
//   * thread roles (every kernel in this file): warpgroups 0 and 1 = consumers, each owning accumulator rows
//     64*h .. 64*h+63 of the 128-row tile (MMA issue + epilogue from its registers); warpgroup 2 = producer (warp 8 issues TMA).
//   * mbarrier ring (full/empty) of STAGES stages between TMA and the consumers; every consumer warp releases a stage
//     once its wgmma group has retired.
//
// The same kernel is the data-gradient (dgrad) kernel when fed tap-flipped, transposed weights, and the 1x1
// convolution with TAPS = 1.  Two source tensors model torch.cat([skip, up], 1) without materialising it.
// Reference call sites: networks/unet.py:19,23 (3x3), :55 (1x1), :67 (concat), :120 (out_conv).
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <mutex>
#include <unordered_map>
#include <string>
#include <type_traits>
#include <string.h>
#include <stdlib.h>

namespace {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must abort the kernel (trap -> launch error), never hang the GPU.  No printf here: any
// function call inside a wgmma kernel makes ptxas serialise every wgmma.mma_async of that kernel.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
    if (spin > (1u << 24)) __trap();
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// TMA tensor store from shared memory, tracked by the issuing thread's bulk async-groups; out-of-bounds parts of the box
// are not written.  Shared-memory writes of other threads must be made visible to the async proxy first (fence_proxy_async
// by every writer, then a barrier).  These run only where `on` is set, as predicated instructions: a branch on the thread
// index while an MMA group is in flight makes ptxas serialise every wgmma of the kernel (C7518).
__device__ __forceinline__ void tma_store_4d(bool on, const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %0, 0;\n\t"
               "@p cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%1, {%3, %4, %5, %6}], [%2];\n\t}"
               ::"r"((uint32_t)on), "l"((uint64_t)map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit(bool on) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %0, 0;\n\t@p cp.async.bulk.commit_group;\n\t}" ::"r"((uint32_t)on) : "memory");
}
// every committed store has finished reading its shared-memory source (the buffer may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all(bool on) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %0, 0;\n\t@p cp.async.bulk.wait_group.read 0;\n\t}" ::"r"((uint32_t)on) : "memory");
}
// every committed store has completed
__device__ __forceinline__ void bulk_wait_all(bool on) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %0, 0;\n\t@p cp.async.bulk.wait_group 0;\n\t}" ::"r"((uint32_t)on) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}
__device__ __forceinline__ uint32_t elect_one() {
  uint32_t e;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(e));
  return e;
}
__device__ __forceinline__ uint32_t uniform(uint32_t v) { return __shfl_sync(0xffffffffu, v, 0); }

// wgmma shared-memory descriptor of a swizzled operand (swizzle span SW = 32/64/128 bytes, the TMA box's swizzle):
//   K-major:  8-row groups SBO bytes apart (LBO unused);
//   MN-major: SW-byte wide groups along M/N LBO bytes apart, 8-row groups along K SBO bytes apart.
// Several kernels view one TMA tile through descriptors whose start is shifted by whole rows (the taps of a 3x3 halo):
// the tensor core takes the swizzle phase from the absolute shared-memory address, as TMA does, so base_offset stays 0.
template <int SW>
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  constexpr uint64_t layout = (SW == 128) ? 1 : (SW == 64) ? 2 : 3;
  return (uint64_t)((saddr & 0x3ffff) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32) | (layout << 62);
}

// Fragment coordinates of a consumer thread (t = thread index inside its warpgroup): accumulator element
// acc[4*j + 2*i + b] is row frag_row(t) + 8*i of the warpgroup's 64 rows, column 8*j + frag_col(t) + b.
__device__ __forceinline__ int frag_row(int t) { return 16 * (t >> 5) + ((t & 31) >> 2); }
__device__ __forceinline__ int frag_col(int t) { return 2 * (t & 3); }

// Two consumer warpgroups and one producer warpgroup (only its first warp issues TMA).  Registers are allocated per warpgroup, so
// the producer warpgroup hands its share to the consumers: 40 + 2 x 232 registers per thread-slot of a warpgroup fill the file.
constexpr int CONSUMER_WARPS = 8, CONSUMERS = 32 * CONSUMER_WARPS, NUM_THREADS = CONSUMERS + 128, PRODUCER_WARP = CONSUMER_WARPS;
__device__ __forceinline__ void producer_regs() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory"); }
__device__ __forceinline__ void consumer_regs() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory"); }
// consumer warp retired its wgmma group: one arrival per warp (empty barriers count CONSUMER_WARPS)
__device__ __forceinline__ void release_stage(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// Stores two adjacent output channels (c, c + 1) of one pixel.  out_mode 0: 16-bit NHWC, 1: fp32 NCHW, 2: fp32 NHWC.
__device__ __forceinline__ void store_pair(void* out, int out_mode, int dt, int CoutStore, int H, int W, int n, int gy, int gx,
                                           int c, float v0, float v1) {
  if (out_mode == 0) {
    if (c < CoutStore) {
      uint32_t* o = reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(out) + (((long long)n * H + gy) * W + gx) * CoutStore + c);
      *o = dt == 2 ? pack_f16(v0, v1) : pack_bf16(v0, v1);
    }
  } else if (out_mode == 2) {
    float* o = reinterpret_cast<float*>(out) + (((long long)n * H + gy) * W + gx) * CoutStore + c;
    if (c + 1 < CoutStore) *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
    else if (c < CoutStore) o[0] = v0;
  } else {
    float* o = reinterpret_cast<float*>(out);
    if (c < CoutStore) o[(((long long)n * CoutStore + c) * H + gy) * W + gx] = v0;
    if (c + 1 < CoutStore) o[(((long long)n * CoutStore + c + 1) * H + gy) * W + gx] = v1;
  }
}

struct ConvTcParams {
  int N, H, W;
  int C0, C1;        // channels of source 0 / source 1 (C1 may be 0)
  int CoutP;         // padded output channels (rows of the packed weight)
  int CoutStore;     // channels stored per pixel (bf16 NHWC) or real channels (fp32 NCHW)
  int taps, ks;
  int tiles_x, tiles_y;
  int out_mode;       // 0: 16-bit NHWC, 1: fp32 NCHW, 2: fp32 NHWC
  int dt;             // 16-bit operand / storage type: 0 bf16, 2 fp16
  int dil;            // dilation (PNet2D's blocks, networks/pnet.py:25-28): tap (dy, dx) reads pixel (y + dil*dy, x + dil*dx)
  const float* bias;
  const float* out_scale;   // optional device scalar multiplied into the accumulator before the bias (split mode: 2^-k of the staged operand)
  void* out;
};

constexpr int TILE_W = 16, TILE_H = 8, TILE_M = 128;

template <int KBLK, int NT, int STAGES>
struct ConvSmem {
  static constexpr int A_BYTES = TILE_M * KBLK * 2;
  static constexpr int B_BYTES = NT * KBLK * 2;
  static constexpr int STAGE_BYTES = ((A_BYTES + B_BYTES + 1023) / 1024) * 1024;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

template <int KBLK, int NT, int STAGES, int DT>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_tc_kernel(const __grid_constant__ CUtensorMap map_a0,
                                                                 const __grid_constant__ CUtensorMap map_a1,
                                                                 const __grid_constant__ CUtensorMap map_b, const ConvTcParams p) {
  using S = ConvSmem<KBLK, NT, STAGES>;
  constexpr int SW = KBLK * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;
  const int n = tile / (p.tiles_x * p.tiles_y);
  const int tr = tile - n * p.tiles_x * p.tiles_y;
  const int y0 = (tr / p.tiles_x) * TILE_H, x0 = (tr % p.tiles_x) * TILE_W;
  const int n0 = blockIdx.y * NT;
  const int pad = p.ks >> 1;
  const int kb0 = p.C0 / KBLK, kb1 = p.C1 / KBLK;
  const int iters = p.taps * (kb0 + kb1);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
    fence_barrier_init();
    prefetch_tmap(&map_a0);
    prefetch_tmap(&map_b);
    if (kb1) prefetch_tmap(&map_a1);
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    producer_regs();
    if (warp != PRODUCER_WARP) return;
    // ===================== TMA producer =====================
    if (lane == 0) {
      int it = 0;
      for (int t = 0; t < p.taps; ++t) {
        const int dy = (t / p.ks - pad) * p.dil, dx = (t % p.ks - pad) * p.dil;
        for (int kb = 0; kb < kb0 + kb1; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          mbar_wait(&empty_bar[s], ph ^ 1);
          uint8_t* a_dst = smem + s * S::STAGE_BYTES;
          uint8_t* b_dst = a_dst + S::A_BYTES;
          mbar_expect_tx(&full_bar[s], S::A_BYTES + S::B_BYTES);
          if (kb < kb0) tma_load_4d(&map_a0, &full_bar[s], a_dst, kb * KBLK, x0 + dx, y0 + dy, n);
          else          tma_load_4d(&map_a1, &full_bar[s], a_dst, (kb - kb0) * KBLK, x0 + dx, y0 + dy, n);
          tma_load_3d(&map_b, &full_bar[s], b_dst, kb * KBLK, n0, t);
        }
      }
    }
    return;
  }
  consumer_regs();
  // ===================== consumers: warpgroup h owns pixel rows 64h .. 64h+63 =====================
  const int h = threadIdx.x >> 7, t = threadIdx.x & 127;
  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
  for (int it = 0; it < iters; ++it) {
    const int s = it % STAGES;
    mbar_wait(&full_bar[s], (it / STAGES) & 1);
    const uint32_t a_addr = smem_u32(smem + s * S::STAGE_BYTES) + (uint32_t)(h * 64 * SW);
    const uint32_t b_addr = smem_u32(smem + s * S::STAGE_BYTES + S::A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KBLK / 16; ++k)   // 16 elements (32 bytes) along K inside the swizzle span
      Wgmma<NT>::template mma<0, 0, DT>(acc, gmma_desc<SW>(a_addr + 32 * k, 16, 8 * SW), gmma_desc<SW>(b_addr + 32 * k, 16, 8 * SW),
                                        (it > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    release_stage(&empty_bar[s]);
  }
  wgmma_fence_regs(acc);
  // ===================== epilogue from registers =====================
  const float sc = p.out_scale ? *p.out_scale : 1.f;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = 64 * h + frag_row(t) + 8 * i;   // pixel index inside the tile
    const int gy = y0 + m / TILE_W, gx = x0 + m % TILE_W;
    if (gy >= p.H || gx >= p.W) continue;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      const int c = n0 + 8 * j + frag_col(t);
      float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
      if (p.out_scale) { v0 *= sc; v1 *= sc; }
      if (p.bias) { v0 += p.bias[c]; v1 += p.bias[c + 1]; }
      store_pair(p.out, p.out_mode, DT, p.CoutStore, p.H, p.W, n, gy, gx, c, v0, v1);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host: tensor maps
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(f);
  });
  return fn;
}

CUtensorMapSwizzle swizzle_for(int kblk) {
  return kblk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : kblk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}

struct MapKey {
  const void* ptr; long long d[4]; int b[4]; int rank; int sw; int dt; int pitch;
  bool operator==(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    const uint64_t* w = reinterpret_cast<const uint64_t*>(&k);
    uint64_t h = 1469598103934665603ULL;
    for (size_t i = 0; i < sizeof(MapKey) / 8; ++i) { h ^= w[i]; h *= 1099511628211ULL; }
    return (size_t)h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// 16-bit tensor (dt 0 = bf16, 2 = fp16), dims innermost-first; strides derived (dense) unless `pitch` (elements between
// consecutive indices of dimension 1, i.e. the channel pitch of a channels-last tensor) is given: a channel-range view of a
// wider tensor.  Cached by (ptr, dims, box, swizzle, type, pitch).
int get_map(const void* ptr, int rank, const long long* dims, const int* box, int kblk, CUtensorMap* out, int dt = 0, int pitch = 0) {
  MapKey key;
  memset(&key, 0, sizeof(key));
  key.ptr = ptr; key.rank = rank; key.sw = kblk; key.dt = dt; key.pitch = pitch;
  for (int i = 0; i < rank; ++i) { key.d[i] = dims[i]; key.b[i] = box[i]; }
  {
    std::lock_guard<std::mutex> g(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return 0; }
  }
  PFN_encodeTiled enc = get_encode();
  if (!enc) { wsl_set_error("cuTensorMapEncodeTiled unavailable (driver too old?)"); return -3; }
  cuuint64_t gdim[4], gstride[3];
  cuuint32_t bdim[4], estr[4];
  unsigned long long stride = 2;
  for (int i = 0; i < rank; ++i) {
    gdim[i] = (cuuint64_t)dims[i];
    bdim[i] = (cuuint32_t)box[i];
    estr[i] = 1;
    stride *= (unsigned long long)((i == 0 && pitch > 0) ? pitch : dims[i]);
    if (i < rank - 1) gstride[i] = stride;
  }
  CUresult r = enc(out, dt == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), gdim, gstride, bdim, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(kblk), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { wsl_set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return -4; }
  std::lock_guard<std::mutex> g(g_map_mu);
  if (g_maps.size() > 4096) g_maps.clear();
  g_maps[key] = *out;
  return 0;
}

// Calls f(std::integral_constant<int, DT>) with the 16-bit operand type dt (0 bf16, 2 fp16) as a compile-time constant.
template <class F>
int with_dt(int dt, F&& f) {
  return dt == 2 ? f(std::integral_constant<int, 2>{}) : f(std::integral_constant<int, 0>{});
}

template <int KBLK, int NT, int STAGES, int DT>
int launch_conv(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const ConvTcParams& p, cudaStream_t stream) {
  using S = ConvSmem<KBLK, NT, STAGES>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<KBLK, NT, STAGES, DT>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL);
    if (e != cudaSuccess) { wsl_set_error("conv_tc: cudaFuncSetAttribute: %s", cudaGetErrorString(e)); return -5; }
    attr = true;
  }
  dim3 grid(p.N * p.tiles_x * p.tiles_y, p.CoutP / NT);
  conv_tc_kernel<KBLK, NT, STAGES, DT><<<grid, NUM_THREADS, S::TOTAL, stream>>>(a0, a1, b, p);
  return wsl_check_launch("conv_tc");
}

template <int KBLK>
int dispatch_nt(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const ConvTcParams& p, int nt, cudaStream_t stream) {
  return with_dt(p.dt, [&](auto dt) {
    constexpr int DT = decltype(dt)::value;
    switch (nt) {
      case 16:  return launch_conv<KBLK, 16, 6, DT>(a0, a1, b, p, stream);
      case 32:  return launch_conv<KBLK, 32, 6, DT>(a0, a1, b, p, stream);
      case 64:  return launch_conv<KBLK, 64, 6, DT>(a0, a1, b, p, stream);
      case 128: return launch_conv<KBLK, 128, 5, DT>(a0, a1, b, p, stream);
    }
    wsl_set_error("conv_tc: unsupported N tile %d", nt);
    return -1;
  });
}


// ================================================================================================
// conv_tc v2: persistent, weights resident in shared memory, ONE halo load per (tile, k-block)
//
//   * pixel tile = 8 w x (16*MT) h  (MT accumulators of M = 128 rows, row m = h*8 + w);
//   * A: one TMA box (KBLK channels x 10 w x (16*MT+2) h) per k-block -- the 3x3 halo.  The nine taps are NOT
//     reloaded: tap (dy,dx) of sub-tile j is the same shared-memory tile viewed through a wgmma descriptor whose
//     start address is shifted by ((16*j+dy)*10 + dx) rows and whose 8-row-group stride (SBO) is one halo row
//     (10 pixels).  The 128B/64B/32B swizzle is a function of the absolute shared-memory address (TMA writes and
//     wgmma reads agree), so a row-shifted start keeps the pattern consistent.
//   * B: the CTA's whole weight slice [taps][k-blocks][NT x KBLK] is loaded once (it fits: NT is chosen on the
//     host so that taps*Cin*NT*2 <= ~148 KB) and stays resident while the CTA walks its pixel tiles.
//   * accumulators: MT x NT fp32 per 128 rows, i.e. MT*NT/2 registers per consumer thread (the host keeps MT*NT <= 128).
// L2->SM traffic per output pixel drops from 9*(Cin + NT)*2 B (v1) to ~1.4*Cin*2 B.
// ================================================================================================
struct ConvV2Params {
  int N, H, W;
  int C0, C1;
  int CoutP, CoutStore;
  int tiles_x, tiles_y, ntiles;
  int out_mode;
  int dt;                 // 16-bit operand / storage type: 0 bf16, 2 fp16
  const float* bias;
  void* out;
  float* stat_partials;   // optional [gridDim.x][2][CoutP]: per-CTA sum / sum of squares of the stored (16-bit-rounded) outputs
};

template <int KS, int KBLK, int NT, int MT>
struct ConvV2Cfg {
  static constexpr int PAD = KS / 2;
  static constexpr int TW = 8, TH = 16 * MT;
  static constexpr int HW_ = TW + 2 * PAD, HH_ = TH + 2 * PAD;
  static constexpr int ROWB = KBLK * 2;
  static constexpr int HALO_BYTES = HW_ * HH_ * ROWB;
  static constexpr int A_STAGE = ((HALO_BYTES + 1023) / 1024) * 1024;
  static constexpr int W_SUB = NT * ROWB;                  // one (tap, k-block) weight tile
  // 16-bit output tile staged for the TMA store: OUT_BOXES boxes of OUT_CH channels x 8 w x TH h, each in the swizzle of
  // its OUT_CH * 2-byte rows (so the epilogue's writes, 8 pixels x 4 channel pairs per warp instruction, hit 32 banks)
  static constexpr int OUT_CH = NT < 64 ? NT : 64, OUT_BOXES = NT / OUT_CH;
  static constexpr int OUT_BOX_BYTES = TW * TH * OUT_CH * 2, OUT_BYTES = OUT_BOXES * OUT_BOX_BYTES;
};

// Byte offset of (pixel px of the tile, channel c of the N tile) in the staged output tile: box c / OUT_CH, row px, in the
// TMA swizzle of the box (16-byte chunk index XOR row-of-128-bytes index, over OUT_CH * 2 / 16 chunks).
template <int OUT_CH, int OUT_BOX_BYTES>
__device__ __forceinline__ uint32_t out_stage_offset(int px, int c) {
  constexpr uint32_t ROWB = OUT_CH * 2, CHUNK_MASK = ROWB / 16 - 1;
  const uint32_t o = (uint32_t)px * ROWB + (uint32_t)(c % OUT_CH) * 2;
  return (uint32_t)(c / OUT_CH) * OUT_BOX_BYTES + (o ^ (((o >> 7) & CHUNK_MASK) << 4));
}

// The MMAs of k-block kb of one tile (MT sub-tiles x T taps x KBLK/16 k-steps) as one commit group.  The first MMA of each
// sub-tile at kb = 0 has scale-d = 0, so acc needs no zero fill: no other instruction writes accumulator registers while the
// previous tile's epilogue runs under this group.
template <int KS, int KBLK, int NT, int MT, int DT>
__device__ __forceinline__ void tile_mma(float (&acc)[MT][NT / 2], uint32_t a_base, uint32_t w_base, int kb, int nkb) {
  using Cfg = ConvV2Cfg<KS, KBLK, NT, MT>;
  constexpr int SW = KBLK * 2, T = KS * KS;
  // The next tile's first group reads the loop-invariant weight slice: without this, ptxas hoists its T * KBLK / 16 64-bit
  // descriptors out of the tile loop and keeps them live (spilling) across the whole epilogue.
  asm volatile("" : "+r"(w_base));
  wgmma_fence();
#pragma unroll
  for (int j = 0; j < MT; ++j) {
#pragma unroll
    for (int tap = 0; tap < T; ++tap) {
      const int dy = tap / KS, dx = tap % KS;
#pragma unroll
      for (int k = 0; k < KBLK / 16; ++k)
        Wgmma<NT>::template mma<0, 0, DT>(acc[j],
                                          gmma_desc<SW>(a_base + (uint32_t)(((16 * j + dy) * Cfg::HW_ + dx) * Cfg::ROWB + 32 * k), 16, Cfg::HW_ * Cfg::ROWB),
                                          gmma_desc<SW>(w_base + (uint32_t)(tap * nkb * Cfg::W_SUB + 32 * k), 16, 8 * SW),
                                          (kb > 0 || tap > 0 || k > 0) ? 1u : 0u);
    }
  }
  wgmma_commit();
}

// Per-thread running BatchNorm sums (NT/4 channels per thread: column 8*j + frag_col + b) -> this CTA's row of
// stat_partials: the lanes holding the same channels are summed with shuffles, then the eight consumer warps in a
// fixed order.  Consumer threads only (named barrier 1); s_stat is shared-memory scratch of the caller.
template <int NT>
__device__ __forceinline__ void write_stat_partials(float (&rs)[NT / 4], float (&rq)[NT / 4], float* stat_partials, int CoutP, int n0,
                                                    float (*s_stat)[2][NT]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < NT / 4; ++k) {
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      rs[k] += __shfl_xor_sync(0xffffffffu, rs[k], o);
      rq[k] += __shfl_xor_sync(0xffffffffu, rq[k], o);
    }
  }
  if (lane < 4) {
#pragma unroll
    for (int k = 0; k < NT / 4; ++k) {
      const int ch = 8 * (k >> 1) + 2 * lane + (k & 1);
      s_stat[warp][0][ch] = rs[k];
      s_stat[warp][1][ch] = rq[k];
    }
  }
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
  for (int c = threadIdx.x; c < 2 * NT; c += CONSUMERS) {
    const int which = c / NT, ch = c % NT;
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < CONSUMER_WARPS; ++w) a += s_stat[w][which][ch];
    stat_partials[((size_t)blockIdx.x * 2 + which) * CoutP + n0 + ch] = a;
  }
}

template <int KS, int KBLK, int NT, int MT, int STAGES, int DT>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_tc2_kernel(const __grid_constant__ CUtensorMap map_a0,
                                                                  const __grid_constant__ CUtensorMap map_a1,
                                                                  const __grid_constant__ CUtensorMap map_b,
                                                                  const __grid_constant__ CUtensorMap map_o, const ConvV2Params p,
                                                                  const int w_bytes) {
  using Cfg = ConvV2Cfg<KS, KBLK, NT, MT>;
  constexpr int T = KS * KS;
  static_assert(MT * NT <= 128, "accumulator registers");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* w_smem = smem;
  uint8_t* a_smem = smem + w_bytes;                         // w_bytes is a multiple of 1024
  uint8_t* o_smem = a_smem + STAGES * Cfg::A_STAGE;         // staged 16-bit output tile (1024-aligned: the swizzle atom)
  uint64_t* bars = reinterpret_cast<uint64_t*>(o_smem + Cfg::OUT_BYTES);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + STAGES;
  uint64_t* w_bar = bars + 2 * STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.y * NT;
  const int kb0 = p.C0 / KBLK, nkb = kb0 + p.C1 / KBLK;
  const int my_tiles = (p.ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], CONSUMER_WARPS); }
    mbar_init(w_bar, 1);
    fence_barrier_init();
    prefetch_tmap(&map_a0);
    prefetch_tmap(&map_b);
    if (p.out_mode == 0) prefetch_tmap(&map_o);
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    producer_regs();
    if (warp != PRODUCER_WARP) return;
    if (lane == 0) {
      mbar_expect_tx(w_bar, (uint32_t)(T * nkb * Cfg::W_SUB));
      for (int t = 0; t < T; ++t)
        for (int kb = 0; kb < nkb; ++kb) tma_load_3d(&map_b, w_bar, w_smem + (t * nkb + kb) * Cfg::W_SUB, kb * KBLK, n0, t);
      int it = 0;
      for (int i = 0; i < my_tiles; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        const int n = tile / (p.tiles_x * p.tiles_y);
        const int tr = tile - n * p.tiles_x * p.tiles_y;
        const int y0 = (tr / p.tiles_x) * Cfg::TH, x0 = (tr % p.tiles_x) * Cfg::TW;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&a_empty[s], ((it / STAGES) & 1) ^ 1);
          mbar_expect_tx(&a_full[s], Cfg::HALO_BYTES);
          if (kb < kb0) tma_load_4d(&map_a0, &a_full[s], a_smem + s * Cfg::A_STAGE, kb * KBLK, x0 - Cfg::PAD, y0 - Cfg::PAD, n);
          else          tma_load_4d(&map_a1, &a_full[s], a_smem + s * Cfg::A_STAGE, (kb - kb0) * KBLK, x0 - Cfg::PAD, y0 - Cfg::PAD, n);
        }
      }
    }
    return;
  }
  consumer_regs();
  const int h = threadIdx.x >> 7, t = threadIdx.x & 127;
  const uint32_t a_u = smem_u32(a_smem), w_u = smem_u32(w_smem);
  float rs[NT / 4], rq[NT / 4];          // running per-channel sum / sum of squares of this thread's pixels
#pragma unroll
  for (int k = 0; k < NT / 4; ++k) rs[k] = rq[k] = 0.f;
  __shared__ float s_bias[NT];
  if (threadIdx.x < NT) s_bias[threadIdx.x] = p.bias ? p.bias[n0 + threadIdx.x] : 0.f;
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
  const bool store_thread = threadIdx.x == 0;   // issues (and waits for) the TMA stores of the output tiles
  const bool stats = p.out_mode == 0 && p.stat_partials;
  mbar_wait(w_bar, 0);
  // One MMA group in flight: group `it` reads A stage it % STAGES and is released once the next group has been issued and
  // it has retired (the same stage order as a serial tile loop).  Tile i + 1's first group is issued as soon as tile i's
  // accumulator is rounded into registers, so tile i's BatchNorm sums and stores run under it.  Rows 64h.. of a sub-tile
  // start 8h halo rows further down.
  const uint32_t a_h = a_u + (uint32_t)(8 * h * Cfg::HW_ * Cfg::ROWB);
  float acc[MT][NT / 2];
  // 16-bit NHWC epilogue.  stage_tile rounds each channel pair (c, c + 1) of pixel m to the 16-bit type (value(j, ii, jj)),
  // accumulates the BatchNorm sums of the rounded values and writes them to the staging buffer; store_tile hands the buffer
  // to TMA.  When the registers allow, the tile is first rounded into pk (registers no MMA writes) and both run under the
  // next tile's first MMA group: pk (a quarter of MT * NT) and the running sums (NT / 2) then live beside the in-flight
  // accumulator (MT * NT / 2).  ptxas allocates the 168 registers of a 384-thread CTA (the setmaxnreg raise to 232 does not
  // enter its allocation), so larger tiles are staged straight from the accumulator before the group is issued and only the
  // store overlaps.
  constexpr bool STAGE_UNDER_MMA = 3 * MT * NT / 4 + NT / 2 <= 64;
  // staging offset of this thread's first pair: pixel 64h + frag_row, channel frag_col
  const uint32_t o_thr = out_stage_offset<Cfg::OUT_CH, Cfg::OUT_BOX_BYTES>(64 * h + frag_row(t), frag_col(t));
  auto stage_tile = [&](auto&& value) {
    bulk_wait_read_all(store_thread);       // the previous tile's store has read the staging buffer
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
#pragma unroll
    for (int j = 0; j < MT; ++j)
#pragma unroll
      for (int ii = 0; ii < 2; ++ii)
#pragma unroll
        for (int jj = 0; jj < NT / 8; ++jj) {
          const uint32_t u = value(j, ii, jj);
          if (stats) {                      // BatchNorm statistics of the values exactly as stored
            float2 r;
            if (DT == 2) r = __half22float2(*reinterpret_cast<const __half2*>(&u));
            else r = make_float2(bf16_lo(u), bf16_hi(u));
            rs[2 * jj] += r.x;     rq[2 * jj] += r.x * r.x;
            rs[2 * jj + 1] += r.y; rq[2 * jj + 1] += r.y * r.y;
          }
          // pixel 128 j + 8 ii further on is a multiple of 256 bytes further on, which keeps the swizzle phase: the 16-byte
          // chunk of channel group jj is an XOR of the thread's base offset (one live register, no per-chunk addresses)
          constexpr int CG = Cfg::OUT_CH / 8;
          const uint32_t off = (o_thr + (uint32_t)((jj / CG) * Cfg::OUT_BOX_BYTES + (128 * j + 8 * ii) * Cfg::OUT_CH * 2)) ^ (uint32_t)((jj % CG) << 4);
          *reinterpret_cast<uint32_t*>(o_smem + off) = u;
        }
    fence_proxy_async();
  };
  auto store_tile = [&](int n, int y0, int x0) {
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
#pragma unroll
    for (int b = 0; b < Cfg::OUT_BOXES; ++b)
      tma_store_4d(store_thread, &map_o, o_smem + b * Cfg::OUT_BOX_BYTES, n0 + b * Cfg::OUT_CH, x0, y0, n);
    bulk_commit(store_thread);
  };
  auto from_acc = [&](int j, int ii, int jj) -> uint32_t {
    const int c = 8 * jj + frag_col(t);
    float v0 = acc[j][4 * jj + 2 * ii], v1 = acc[j][4 * jj + 2 * ii + 1];
    if (p.bias) { v0 += s_bias[c]; v1 += s_bias[c + 1]; }
    return DT == 2 ? pack_f16(v0, v1) : pack_bf16(v0, v1);
  };
  // Every CTA has at least one tile (the host keeps the grid <= ntiles), so the first group is issued unconditionally: the
  // MMAs are issued on paths that never join one without a group in flight (a join of the two makes ptxas serialise, C7518).
  mbar_wait(&a_full[0], 0);
  tile_mma<KS, KBLK, NT, MT, DT>(acc, a_h, w_u, 0, nkb);
  int it = 1;
  for (int i = 0;; ++i) {
    const int tile = blockIdx.x + i * gridDim.x;
    const int n = tile / (p.tiles_x * p.tiles_y);
    const int tr = tile - n * p.tiles_x * p.tiles_y;
    const int y0 = (tr / p.tiles_x) * Cfg::TH, x0 = (tr % p.tiles_x) * Cfg::TW;
    for (int kb = 1; kb < nkb; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(&a_full[s], (it / STAGES) & 1);
      tile_mma<KS, KBLK, NT, MT, DT>(acc, a_h + (uint32_t)(s * Cfg::A_STAGE), w_u + (uint32_t)(kb * Cfg::W_SUB), kb, nkb);
      wgmma_wait<1>();                     // the previous k-block's group has retired: its stage can be refilled
      release_stage(&a_empty[(it + STAGES - 1) % STAGES]);
    }
    wgmma_wait<0>();
    release_stage(&a_empty[(it + STAGES - 1) % STAGES]);
#pragma unroll
    for (int j = 0; j < MT; ++j) wgmma_fence_regs(acc[j]);
    uint32_t pk[MT][2][NT / 8];
    if (p.out_mode == 0) {
      if constexpr (STAGE_UNDER_MMA) {
#pragma unroll
        for (int j = 0; j < MT; ++j)
#pragma unroll
          for (int ii = 0; ii < 2; ++ii)
#pragma unroll
            for (int jj = 0; jj < NT / 8; ++jj) pk[j][ii][jj] = from_acc(j, ii, jj);
      } else {
        stage_tile(from_acc);
      }
    } else {                                // fp32 NCHW (the logits): stored from the accumulator before the next group
#pragma unroll
      for (int j = 0; j < MT; ++j)
#pragma unroll
        for (int ii = 0; ii < 2; ++ii) {
          const int m = 64 * h + frag_row(t) + 8 * ii;
          const int gy = y0 + 16 * j + m / 8, gx = x0 + (m & 7);
#pragma unroll
          for (int jj = 0; jj < NT / 8; ++jj) {
            const int c = 8 * jj + frag_col(t);
            float v0 = acc[j][4 * jj + 2 * ii], v1 = acc[j][4 * jj + 2 * ii + 1];
            if (p.bias) { v0 += s_bias[c]; v1 += s_bias[c + 1]; }
            store_pair(p.out, 1, DT, p.CoutStore, p.H, p.W, n, gy, gx, n0 + c, v0, v1);
          }
        }
    }
#pragma unroll
    for (int j = 0; j < MT; ++j) wgmma_discard_regs(acc[j]);
    auto finish_tile = [&]() {
      if (p.out_mode == 0) {
        if constexpr (STAGE_UNDER_MMA) stage_tile([&](int j, int ii, int jj) { return pk[j][ii][jj]; });
        store_tile(n, y0, x0);
      }
    };
    if (i + 1 == my_tiles) {                // last tile: no next group to overlap
      finish_tile();
      break;
    }
    mbar_wait(&a_full[it % STAGES], (it / STAGES) & 1);
    tile_mma<KS, KBLK, NT, MT, DT>(acc, a_h + (uint32_t)((it % STAGES) * Cfg::A_STAGE), w_u, 0, nkb);
    ++it;
    finish_tile();
  }
  bulk_wait_all(store_thread);
  if (stats) {                              // the staging buffer is free: it holds the cross-warp combine
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    write_stat_partials<NT>(rs, rq, p.stat_partials, p.CoutP, n0, reinterpret_cast<float (*)[2][NT]>(o_smem));
  }
}

// ================================================================================================
// wgmma weight gradient:  dW[co][ci][t] += sum_{pixels} dY[p][co] * X[p + tap_t][ci]
//
//   D_t[M = 128 couts, N = CWB cins] (fp32, registers) += A^T[K = 128 pixels x M] * B_t[K = 128 pixels x N]
//
// Both operands are "MN-major" for the tensor core: K (pixels) indexes shared-memory rows, the channel (M or N)
// is contiguous inside a row -- exactly what a channels-last TMA box (channels x 16 w x 8 h) produces.  A (dY) is
// loaded once per 128-pixel chunk, B (the tap-shifted X box, TMA zero fill = padding) once per tap of the CTA's
// tap group; each CTA owns (Cout tile of 128) x (Cin block of CWB) x (TG taps), loops over its share of the
// N*H*W/128 pixel chunks (split-K), keeps TG accumulators in registers and finally adds them into the fp32
// torch-layout gradient with red.global.add.f32.
//   CWA/CWB = channels per A/B box (16/32/64 -> swizzle 32/64/128 B), NA = A boxes per stage (1 or 2).
// Consumer warpgroup h owns couts 64h..64h+63 of the tile and skips its MMAs when they are all padding.  When Cout < 64
// the M = 64 MMA still reads the missing channel groups from whatever shared memory follows the A box; those
// accumulator rows are never stored.
// ================================================================================================
struct WgradTcParams {
  int N, H, W;
  int C0, C1;          // source channels
  int CoutP, CoutReal;
  int taps, ks;
  int tiles_x, tiles_y, nchunks;
  int n_tiles0, n_tiles1;   // Cin blocks in source 0 / 1
  int tap_groups;
  int dt;               // 16-bit operand type: 0 bf16, 2 fp16
  const float* scale_a;  // optional device scalars multiplied into the result (split mode: 2^-k of the staged dY / X)
  const float* scale_b;
  float* dw;
  float* partials;       // optional [gridDim.y][gridDim.x][TG*CWB][128]: per-CTA partial tiles for the fixed-order finalize
  int dil;               // dilation of the convolution
};

template <int CWA, int NA, int CWB, int TG, int STAGES>
struct WgradSmem {
  static constexpr int A_BOX = TILE_M * CWA * 2;
  static constexpr int B_BOX = TILE_M * CWB * 2;
  static constexpr int STAGE_BYTES = ((NA * A_BOX + TG * B_BOX + 1023) / 1024) * 1024;
  static constexpr int SLACK = (64 / CWA) * A_BOX;    // aliased channel groups of the last stage stay inside the allocation
  static constexpr int TOTAL = STAGES * STAGE_BYTES + SLACK + 1024 + 256;
};

template <int CWA, int NA, int CWB, int TG, int STAGES, int DT>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_dy,
                                                                  const __grid_constant__ CUtensorMap map_x0,
                                                                  const __grid_constant__ CUtensorMap map_x1, const WgradTcParams p) {
  using S = WgradSmem<CWA, NA, CWB, TG, STAGES>;
  constexpr int SWA = CWA * 2, SWB = CWB * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES + S::SLACK);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // blockIdx.y -> (m tile, n tile, tap group)
  int by = blockIdx.y;
  const int tg = by % p.tap_groups; by /= p.tap_groups;
  const int n_tiles = p.n_tiles0 + p.n_tiles1;
  const int nt = by % n_tiles;
  const int mt = by / n_tiles;
  const int m0 = mt * 128;
  const bool src1 = nt >= p.n_tiles0;
  const int cb0 = (src1 ? nt - p.n_tiles0 : nt) * CWB;             // channel offset inside the source tensor
  const int ci_global = (src1 ? p.C0 : 0) + cb0;                   // channel offset in the concatenated input
  const int pad = p.ks >> 1;
  const int my_chunks = (p.nchunks - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
    fence_barrier_init();
    prefetch_tmap(&map_dy);
    prefetch_tmap(src1 ? &map_x1 : &map_x0);
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    producer_regs();
    if (warp != PRODUCER_WARP) return;
    if (lane == 0) {
      const CUtensorMap* mx = src1 ? &map_x1 : &map_x0;
      for (int it = 0; it < my_chunks; ++it) {
        const int chunk = blockIdx.x + it * gridDim.x;
        const int n = chunk / (p.tiles_x * p.tiles_y);
        const int tr = chunk - n * p.tiles_x * p.tiles_y;
        const int y0 = (tr / p.tiles_x) * TILE_H, x0 = (tr % p.tiles_x) * TILE_W;
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        mbar_wait(&empty_bar[s], ph ^ 1);
        uint8_t* a_dst = smem + s * S::STAGE_BYTES;
        uint8_t* b_dst = a_dst + NA * S::A_BOX;
        mbar_expect_tx(&full_bar[s], NA * S::A_BOX + TG * S::B_BOX);
#pragma unroll
        for (int i = 0; i < NA; ++i) tma_load_4d(&map_dy, &full_bar[s], a_dst + i * S::A_BOX, m0 + i * CWA, x0, y0, n);
#pragma unroll
        for (int tl = 0; tl < TG; ++tl) {
          const int t = tg * TG + tl;
          const int dy = (t / p.ks - pad) * p.dil, dx = (t % p.ks - pad) * p.dil;
          tma_load_4d(mx, &full_bar[s], b_dst + tl * S::B_BOX, cb0, x0 + dx, y0 + dy, n);
        }
      }
    }
    return;
  }
  consumer_regs();
  const int h = threadIdx.x >> 7, t = threadIdx.x & 127;
  const bool active = m0 + 64 * h < p.CoutP;
  float acc[TG][CWB / 2];
#pragma unroll
  for (int tl = 0; tl < TG; ++tl)
#pragma unroll
    for (int e = 0; e < CWB / 2; ++e) acc[tl][e] = 0.f;
  for (int it = 0; it < my_chunks; ++it) {
    const int s = it % STAGES;
    mbar_wait(&full_bar[s], (it / STAGES) & 1);
    if (active) {
      const uint32_t a_addr = smem_u32(smem + s * S::STAGE_BYTES) + (uint32_t)((64 * h / CWA) * S::A_BOX);
      const uint32_t b_addr = smem_u32(smem + s * S::STAGE_BYTES + NA * S::A_BOX);
      wgmma_fence();
#pragma unroll
      for (int tl = 0; tl < TG; ++tl) {
#pragma unroll
        for (int k = 0; k < TILE_M / 16; ++k)   // 16 pixels (rows) per MMA: advance both operands by 16 rows
          Wgmma<CWB>::template mma<1, 1, DT>(acc[tl], gmma_desc<SWA>(a_addr + (uint32_t)(k * 16 * SWA), S::A_BOX, 8 * SWA),
                                             gmma_desc<SWB>(b_addr + (uint32_t)(tl * S::B_BOX + k * 16 * SWB), S::B_BOX, 8 * SWB),
                                             (it > 0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
    }
    release_stage(&empty_bar[s]);
  }
  if (my_chunks == 0 || !active) return;
  const int CinTot = p.C0 + p.C1;
  const float osc = (p.scale_a ? *p.scale_a : 1.f) * (p.scale_b ? *p.scale_b : 1.f);
#pragma unroll
  for (int tl = 0; tl < TG; ++tl) {
    wgmma_fence_regs(acc[tl]);
#pragma unroll
    for (int ii = 0; ii < 2; ++ii) {
      const int r = 64 * h + frag_row(t) + 8 * ii, row = m0 + r;   // output channel
#pragma unroll
      for (int e = 0; e < CWB / 4; ++e) {
        const int c = 8 * (e >> 1) + frag_col(t) + (e & 1);          // input channel inside the block
        const float v = acc[tl][4 * (e >> 1) + 2 * ii + (e & 1)] * osc;
        if (p.partials != nullptr)          // deterministic split-K (see wgrad1_finalize_kernel)
          p.partials[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (size_t)(TG * CWB * 128) + (size_t)(tl * CWB + c) * 128 + r] = v;
        else if (row < p.CoutReal)
          atomicAdd(p.dw + ((size_t)row * CinTot + ci_global + c) * p.taps + tg * TG + tl, v);
      }
    }
  }
}

// ================================================================================================
// wgrad v3 (3x3): taps in the M dimension, filter rows in the N dimension.
//
//   A := X rows (MN-major).  An M = 64 operand is 64/CWB channel groups spaced LBO apart; with LBO = ONE PIXEL
//        (CWB*2 bytes) group g is the same tile viewed g pixels further right, i.e. filter column dx = g.  One MMA
//        therefore accumulates dx = 0,1,2 of the filter at once (groups >= 3 are don't-care rows of D; warpgroup 1,
//        holding groups 64/CWB.., only runs when CWB = 32).
//   B := dY tile (MN-major) loaded with one halo row above and below (18 x 8 pixels); N-group g of the B operand is
//        the dY tile viewed g - 1 rows further down (LBO = one tile row), while A is the un-shifted X row block
//        (16 x 10 pixels).  X[p + (1 - g) rows + dx] * dY[p] lands in column group g, i.e. dy = 2 - g; the products
//        that fall outside the chunk's rows are exactly those against the zero padding (TMA zero fill).
//   D[(dx, ci)][(dy, co)]: one accumulator of N = 3*NTILE columns (NTILE = Cout tile <= 64).
// ================================================================================================
template <int CWB, int NTILE, int STAGES>
struct Wgrad3Smem {
  static constexpr int ROWB = CWB * 2;
  static constexpr int N_BOX = 18 * 8 * NTILE * 2;
  static constexpr int A_OFF = ((N_BOX + 1023) / 1024) * 1024;
  static constexpr int A_BYTES = 10 * 16 * ROWB;
  static constexpr int STAGE_BYTES = ((A_OFF + A_BYTES + 1023) / 1024) * 1024;
  static constexpr int SLACK = 2048;
  static constexpr int TOTAL = STAGES * STAGE_BYTES + SLACK + 1024 + 256;
};

struct Wgrad3Params {
  int N, H, W;
  int C0, C1;
  int CoutReal;
  int tiles_x, tiles_y, nchunks;
  int k_tiles0, k_tiles1;     // Cin blocks (of CWB channels) in source 0 / 1
  int dt;                     // 16-bit operand type: 0 bf16, 2 fp16
  float* dw;
  float* partials;            // optional [gridDim.y][gridDim.x][3*NTILE][128]: per-CTA partial tiles for the fixed-order finalize
};

template <int CWB, int NTILE, int STAGES, int DT>
__global__ void __launch_bounds__(NUM_THREADS, 1) wgrad_tc3_kernel(const __grid_constant__ CUtensorMap map_dy,
                                                                   const __grid_constant__ CUtensorMap map_x0,
                                                                   const __grid_constant__ CUtensorMap map_x1, const Wgrad3Params p) {
  using S = Wgrad3Smem<CWB, NTILE, STAGES>;
  constexpr int SWX = CWB * 2, SWN = NTILE * 2, NG = 3 * NTILE;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * S::STAGE_BYTES + S::SLACK);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k_tiles = p.k_tiles0 + p.k_tiles1;
  const int kt = blockIdx.y % k_tiles;          // Cin block
  const int nt = blockIdx.y / k_tiles;          // Cout tile
  const int n0 = nt * NTILE;
  const bool src1 = kt >= p.k_tiles0;
  const int cb0 = (src1 ? kt - p.k_tiles0 : kt) * CWB;
  const int ci_global = (src1 ? p.C0 : 0) + cb0;
  const int my_chunks = (p.nchunks - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CONSUMER_WARPS); }
    fence_barrier_init();
    prefetch_tmap(&map_dy);
    prefetch_tmap(src1 ? &map_x1 : &map_x0);
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    producer_regs();
    if (warp != PRODUCER_WARP) return;
    if (lane == 0) {
      const CUtensorMap* mx = src1 ? &map_x1 : &map_x0;
      for (int it = 0; it < my_chunks; ++it) {
        const int chunk = blockIdx.x + it * gridDim.x;
        const int n = chunk / (p.tiles_x * p.tiles_y);
        const int tr = chunk - n * p.tiles_x * p.tiles_y;
        const int y0 = (tr / p.tiles_x) * 16, x0 = (tr % p.tiles_x) * 8;
        const int s = it % STAGES;
        mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
        uint8_t* b_dst = smem + s * S::STAGE_BYTES;          // dY box
        uint8_t* a_dst = b_dst + S::A_OFF;                   // X block
        mbar_expect_tx(&full_bar[s], S::N_BOX + S::A_BYTES);
        tma_load_4d(&map_dy, &full_bar[s], b_dst, n0, x0, y0 - 1, n);
        tma_load_4d(mx, &full_bar[s], a_dst, cb0, x0 - 1, y0, n);
      }
    }
    return;
  }
  consumer_regs();
  const int h = threadIdx.x >> 7, t = threadIdx.x & 127;
  const bool active = 64 * h < 3 * CWB;       // warpgroup 1 holds filter columns only when the Cin block is 32 wide
  float acc[NG / 2];
#pragma unroll
  for (int e = 0; e < NG / 2; ++e) acc[e] = 0.f;
  for (int it = 0; it < my_chunks; ++it) {
    const int s = it % STAGES;
    mbar_wait(&full_bar[s], (it / STAGES) & 1);
    if (active) {
      const uint32_t b_addr = smem_u32(smem + s * S::STAGE_BYTES);
      const uint32_t a_addr = b_addr + (uint32_t)(S::A_OFF + (64 * h / CWB) * S::ROWB);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k)      // k-step = 16 pixels = chunk rows 2k, 2k+1
        Wgmma<NG>::template mma<1, 1, DT>(acc, gmma_desc<SWX>(a_addr + (uint32_t)(k * 2 * 10 * S::ROWB), S::ROWB, 10 * S::ROWB),
                                          gmma_desc<SWN>(b_addr + (uint32_t)(k * 16 * SWN), 8 * SWN, 8 * SWN), (it > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    release_stage(&empty_bar[s]);
  }
  if (my_chunks == 0 || !active) return;
  wgmma_fence_regs(acc);
  const int CinTot = p.C0 + p.C1;
#pragma unroll
  for (int ii = 0; ii < 2; ++ii) {
    const int m = 64 * h + frag_row(t) + 8 * ii;
    const int g = m / CWB, ci = m % CWB;        // filter column dx, input channel inside the block
#pragma unroll
    for (int e = 0; e < NG / 4; ++e) {
      const int col = 8 * (e >> 1) + frag_col(t) + (e & 1);
      const float v = acc[4 * (e >> 1) + 2 * ii + (e & 1)];
      if (p.partials != nullptr) {
        // deterministic split-K: this CTA's partial tile goes to its own slot; wgrad3_finalize_kernel sums the slots of an
        // output tile in split order and adds the result into dw
        p.partials[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * (size_t)(NG * 128) + (size_t)col * 128 + m] = v;
      } else {
        const int grp = col / NTILE, co = n0 + col % NTILE, dy = 2 - grp;   // column group -> filter row
        if (g < 3 && co < p.CoutReal) atomicAdd(p.dw + ((size_t)co * CinTot + ci_global + ci) * 9 + dy * 3 + g, v);
      }
    }
  }
}

// Fixed-order reduction of the per-CTA partial tiles of one wgrad_tc3 launch: element e = (grp * NTILE + col) * 128 + m of output tile
// blockIdx.y is summed over the `splits` slots in index order (independent of which CTA finished when) and ADDED to the torch-layout
// gradient (accumulation semantics are kept: a second backward through shared weights adds on top).
__global__ void __launch_bounds__(256) wgrad3_finalize_kernel(const float* __restrict__ partials, int splits, int ntile, int cwb, int dyn,
                                                              int k_tiles0, int k_tiles, int C0, int CinTot, int CoutReal,
                                                              float* __restrict__ dw) {
  const int E = 3 * ntile * 128;
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= E) return;
  const int m = e & 127, col = (e >> 7) % ntile, grp = (e >> 7) / ntile;
  const int g = m / cwb, ci = m % cwb;
  const int kt = blockIdx.y % k_tiles, nt = blockIdx.y / k_tiles;
  const int co = nt * ntile + col;
  if (g >= 3 || co >= CoutReal) return;
  const bool src1 = kt >= k_tiles0;
  const int ci_global = (src1 ? C0 : 0) + (src1 ? kt - k_tiles0 : kt) * cwb;
  const float* src = partials + (size_t)blockIdx.y * splits * E + e;
  float acc = 0.f;
  int s = 0;
  for (; s + 8 <= splits; s += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldcg(src + (size_t)(s + u) * E);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += v[u];
  }
  for (; s < splits; ++s) acc += __ldcg(src + (size_t)s * E);
  const int dy = dyn ? 2 - grp : grp;
  dw[((size_t)co * CinTot + ci_global + ci) * 9 + dy * 3 + g] += acc;
}

template <int CWB, int NTILE, int DT>
int launch_wgrad3(const CUtensorMap& mdy, const CUtensorMap& mx0, const CUtensorMap& mx1, Wgrad3Params p, int n_tiles,
                  float* partial_ws, long long partial_floats, cudaStream_t stream) {
  constexpr int per_stage = TILE_M * NTILE * 2 + 12 * 1024;
  constexpr int STAGES = per_stage >= 40 * 1024 ? 3 : 4;
  using S = Wgrad3Smem<CWB, NTILE, STAGES>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_tc3_kernel<CWB, NTILE, STAGES, DT>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL);
    if (e != cudaSuccess) { wsl_set_error("wgrad_tc3: cudaFuncSetAttribute(%d bytes): %s", S::TOTAL, cudaGetErrorString(e)); return -5; }
    attr = true;
  }
  const int gy = n_tiles * (p.k_tiles0 + p.k_tiles1);
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wgrad_tc3_kernel<CWB, NTILE, STAGES, DT>, NUM_THREADS, S::TOTAL);
  if (per_sm < 1) per_sm = 1;
  if (per_sm > 2) per_sm = 2;
  int splits = (wsl_num_sms() * per_sm + gy - 1) / gy;
  if (splits > p.nchunks) splits = p.nchunks;
  if (splits < 1) splits = 1;
  dim3 grid(splits, gy);
  const long long need = (long long)splits * gy * 3 * NTILE * 128;
  p.partials = (partial_ws != nullptr && need <= partial_floats) ? partial_ws : nullptr;     // too small a workspace: atomics
  wgrad_tc3_kernel<CWB, NTILE, STAGES, DT><<<grid, NUM_THREADS, S::TOTAL, stream>>>(mdy, mx0, mx1, p);
  int rc = wsl_check_launch("wgrad_tc3");
  if (rc || p.partials == nullptr) return rc;
  wgrad3_finalize_kernel<<<dim3((3 * NTILE * 128 + 255) / 256, gy), 256, 0, stream>>>(p.partials, splits, NTILE, CWB, 1, p.k_tiles0,
                                                                                     p.k_tiles0 + p.k_tiles1, p.C0, p.C0 + p.C1, p.CoutReal, p.dw);
  return wsl_check_launch("wgrad3_finalize");
}

// fixed-order reduction of wgrad_tc_kernel's per-CTA partial tiles: element e = (tl * CWB + c) * 128 + lane of output tile blockIdx.y
__global__ void __launch_bounds__(256) wgrad1_finalize_kernel(const float* __restrict__ partials, int splits, int tg_size, int cwb,
                                                              int tap_groups, int n_tiles0, int n_tiles, int C0, int CinTot,
                                                              int CoutReal, int taps, float* __restrict__ dw) {
  const int E = tg_size * cwb * 128;
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= E) return;
  const int lane = e & 127, c = (e >> 7) % cwb, tl = (e >> 7) / cwb;
  int by = blockIdx.y;
  const int tg = by % tap_groups; by /= tap_groups;
  const int nt = by % n_tiles, mt = by / n_tiles;
  const int row = mt * 128 + lane;
  if (row >= CoutReal) return;
  const bool src1 = nt >= n_tiles0;
  const int ci = (src1 ? C0 : 0) + (src1 ? nt - n_tiles0 : nt) * cwb + c;
  const float* src = partials + (size_t)blockIdx.y * splits * E + e;
  float acc = 0.f;
  int s = 0;
  for (; s + 8 <= splits; s += 8) {            // eight loads in flight, fixed summation order
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldcg(src + (size_t)(s + u) * E);
#pragma unroll
    for (int u = 0; u < 8; ++u) acc += v[u];
  }
  for (; s < splits; ++s) acc += __ldcg(src + (size_t)s * E);
  dw[((size_t)row * CinTot + ci) * taps + tg * tg_size + tl] += acc;
}

static thread_local float* g_wgrad1_ws = nullptr;        // set by the entry point for the launch helpers below
static thread_local long long g_wgrad1_ws_floats = 0;

template <int CWA, int NA, int CWB, int TG, int DT>
int launch_wgrad(const CUtensorMap& mdy, const CUtensorMap& mx0, const CUtensorMap& mx1, WgradTcParams p, int m_tiles,
                 cudaStream_t stream) {
  constexpr int per_stage = NA * TILE_M * CWA * 2 + TG * TILE_M * CWB * 2;
  constexpr int STAGES = per_stage >= 80 * 1024 ? 2 : per_stage >= 48 * 1024 ? 3 : 4;
  using S = WgradSmem<CWA, NA, CWB, TG, STAGES>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_tc_kernel<CWA, NA, CWB, TG, STAGES, DT>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::TOTAL);
    if (e != cudaSuccess) { wsl_set_error("wgrad_tc: cudaFuncSetAttribute(%d bytes): %s", S::TOTAL, cudaGetErrorString(e)); return -5; }
    attr = true;
  }
  const int gy = m_tiles * (p.n_tiles0 + p.n_tiles1) * p.tap_groups;
  int splits = (wsl_num_sms() * 2 + gy - 1) / gy;
  if (splits > p.nchunks) splits = p.nchunks;
  if (splits < 1) splits = 1;
  dim3 grid(splits, gy);
  const long long need = (long long)splits * gy * TG * CWB * 128;
  p.partials = (g_wgrad1_ws != nullptr && need <= g_wgrad1_ws_floats) ? g_wgrad1_ws : nullptr;
  wgrad_tc_kernel<CWA, NA, CWB, TG, STAGES, DT><<<grid, NUM_THREADS, S::TOTAL, stream>>>(mdy, mx0, mx1, p);
  int rc = wsl_check_launch("wgrad_tc");
  if (rc || p.partials == nullptr) return rc;
  wgrad1_finalize_kernel<<<dim3((TG * CWB * 128 + 255) / 256, gy), 256, 0, stream>>>(p.partials, splits, TG, CWB, p.tap_groups, p.n_tiles0,
                                                                                   p.n_tiles0 + p.n_tiles1, p.C0, p.C0 + p.C1, p.CoutReal,
                                                                                   p.taps, p.dw);
  return wsl_check_launch("wgrad1_finalize");
}

template <int CWA, int NA, int CWB>
int wgrad_dispatch_tg(const CUtensorMap& a, const CUtensorMap& b0, const CUtensorMap& b1, const WgradTcParams& p, int m_tiles, cudaStream_t st) {
  return with_dt(p.dt, [&](auto dt) {
    constexpr int DT = decltype(dt)::value;
    if (p.ks == 3) return launch_wgrad<CWA, NA, CWB, 3, DT>(a, b0, b1, p, m_tiles, st);
    return launch_wgrad<CWA, NA, CWB, 1, DT>(a, b0, b1, p, m_tiles, st);
  });
}
template <int CWA, int NA>
int wgrad_dispatch_b(int cwb, const CUtensorMap& a, const CUtensorMap& b0, const CUtensorMap& b1, const WgradTcParams& p, int m_tiles, cudaStream_t st) {
  switch (cwb) {
    case 64: return wgrad_dispatch_tg<CWA, NA, 64>(a, b0, b1, p, m_tiles, st);
    case 32: return wgrad_dispatch_tg<CWA, NA, 32>(a, b0, b1, p, m_tiles, st);
    default: return wgrad_dispatch_tg<CWA, NA, 16>(a, b0, b1, p, m_tiles, st);
  }
}

// per-channel sum of a channels-last bf16 tensor, added into out[C] (bias gradients of conv1x1 / out_conv)
template <typename T, bool HALF = false>
__global__ void __launch_bounds__(256) channel_sum_kernel(const T* __restrict__ x, long long P, int C, int Creal,
                                                          float* __restrict__ out, float* __restrict__ ws) {
  extern __shared__ float s_red[];
  const int cg = C >> 3, rows = 256 / cg;
  const int g = threadIdx.x % cg, r = threadIdx.x / cg;
  float sum[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sum[j] = 0.f;
  for (long long q = (long long)blockIdx.x * rows + r; r < rows && q < P; q += (long long)gridDim.x * rows) {   // threads beyond rows*cg idle
    float v[8];
    if constexpr (sizeof(T) == 2) {
      unpack8_dt(*reinterpret_cast<const uint4*>(x + q * C + g * 8), v, HALF ? 2 : 0);
    } else {
      const float4 a = reinterpret_cast<const float4*>(x + q * C + g * 8)[0], b = reinterpret_cast<const float4*>(x + q * C + g * 8)[1];
      v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sum[j] += v[j];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) s_red[threadIdx.x * 8 + j] = sum[j];
  __syncthreads();
  if (ws == nullptr) {
    for (int c = threadIdx.x; c < Creal; c += 256) {
      float a = 0.f;
      for (int rr = 0; rr < rows; ++rr) a += s_red[(rr * cg + (c >> 3)) * 8 + (c & 7)];
      atomicAdd(out + c, a);
    }
    return;
  }
  // deterministic: per-block rows, the last block to finish (ticket in ws[0]) adds them up in block order
  for (int c = threadIdx.x; c < Creal; c += 256) {
    float a = 0.f;
    for (int rr = 0; rr < rows; ++rr) a += s_red[(rr * cg + (c >> 3)) * 8 + (c & 7)];
    ws[64 + (size_t)blockIdx.x * Creal + c] = a;
  }
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(reinterpret_cast<unsigned*>(ws), 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // all 256 threads: `parts` threads per channel walk interleaved block subsets (8 loads in flight), then a fixed-order combine;
  // more than 256 channels (PNet2D's 320-channel concat head) go in slabs of 256
  __shared__ float s_fin[256];
  for (int cb = 0; cb < Creal; cb += 256) {
    const int cn = Creal - cb < 256 ? Creal - cb : 256;
    const int parts = 256 / cn;
    const int c = cb + threadIdx.x % cn, part = threadIdx.x / cn;
    float a = 0.f;
    if (part < parts) {
      int b = part;
      for (; b + 7 * parts < (int)gridDim.x; b += 8 * parts) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = __ldcg(&ws[64 + (size_t)(b + u * parts) * Creal + c]);
#pragma unroll
        for (int u = 0; u < 8; ++u) a += v[u];
      }
      for (; b < (int)gridDim.x; b += parts) a += __ldcg(&ws[64 + (size_t)b * Creal + c]);
    }
    s_fin[threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.x < cn) {
      float t = 0.f;
      for (int q = 0; q < parts; ++q) t += s_fin[q * cn + threadIdx.x];
      out[cb + threadIdx.x] += t;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *reinterpret_cast<unsigned*>(ws) = 0u;
}


static int g_conv2_last_rows = 0;   // gridDim.x of the most recent conv_tc2 launch (rows of stat_partials)

template <int KS, int KBLK, int NT, int MT, int DT>
int launch_conv2(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& o, const ConvV2Params& p,
                 cudaStream_t stream) {
  using Cfg = ConvV2Cfg<KS, KBLK, NT, MT>;
  constexpr int STAGES = (Cfg::A_STAGE <= 8 * 1024) ? 4 : (Cfg::A_STAGE <= 13 * 1024) ? 3 : 2;
  const int T = KS * KS;
  const int nkb = (p.C0 + p.C1) / KBLK;
  const int w_bytes = ((T * nkb * Cfg::W_SUB + 1023) / 1024) * 1024;
  const int smem = w_bytes + STAGES * Cfg::A_STAGE + Cfg::OUT_BYTES + 1024 + 256;
  if (smem > 227 * 1024) { wsl_set_error("conv_tc2: %d bytes of shared memory needed", smem); return -6; }
  static int attr_bytes = 0;
  if (smem > attr_bytes) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc2_kernel<KS, KBLK, NT, MT, STAGES, DT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { wsl_set_error("conv_tc2: cudaFuncSetAttribute(%d): %s", smem, cudaGetErrorString(e)); return -5; }
    attr_bytes = smem;
  }
  const int n_tiles = p.CoutP / NT;
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, conv_tc2_kernel<KS, KBLK, NT, MT, STAGES, DT>, NUM_THREADS, smem);
  if (occ < 1) occ = 1;
  int gx = (wsl_num_sms() * occ) / n_tiles;
  if (gx < 1) gx = 1;
  if (gx > p.ntiles) gx = p.ntiles;
  dim3 grid(gx, n_tiles);
  g_conv2_last_rows = gx;
  conv_tc2_kernel<KS, KBLK, NT, MT, STAGES, DT><<<grid, NUM_THREADS, smem, stream>>>(a0, a1, b, o, p, w_bytes);
  return wsl_check_launch("conv_tc2");
}

template <int KS, int KBLK, int MT>
int conv2_dispatch_nt(int nt, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& o, const ConvV2Params& p,
                      cudaStream_t st) {
  return with_dt(p.dt, [&](auto dt) {
    constexpr int DT = decltype(dt)::value;
    switch (nt) {
      case 16:  return launch_conv2<KS, KBLK, 16, MT, DT>(a0, a1, b, o, p, st);
      case 32:  return launch_conv2<KS, KBLK, 32, MT, DT>(a0, a1, b, o, p, st);
      case 64:  if constexpr (MT <= 2) return launch_conv2<KS, KBLK, 64, MT, DT>(a0, a1, b, o, p, st); else break;
      case 128: if constexpr (MT == 1) return launch_conv2<KS, KBLK, 128, MT, DT>(a0, a1, b, o, p, st); else break;
    }
    wsl_set_error("conv_tc2: unsupported N tile %d", nt);
    return -1;
  });
}

// ================================================================================================
// conv_row: 3x3 convolution for narrow outputs (CoutP = 16 or 32) with the filter ROWS in the MMA's N dimension.
//
// With N = Cout = 16 or 32 an MMA is bound by reading its A operand, and conv_tc2 issues nine of them per 128 pixels.
// Here the work unit is one INPUT row of 128 pixels:
//     E_i[c][(dy, co)] = sum_{dx, ci} X[row i][c + dx - 1][ci] * W[dy][dx][co][ci]
// i.e. 3 MMAs per 16 input channels (dx = pixel-shifted views of ONE row buffer), each with N = 3*Cout; an output row is
//     out[r][c] = E_r[c][dy=0] + E_{r+1}[c][dy=1] + E_{r+2}[c][dy=2]
// summed in registers by the thread that owns pixel c (a rolling pair of partial rows): no cross-thread traffic.
//   warp 8: TMA producer (one [KBW ch x 130 px] box per input row and channel block; OOB zero fill = padding)
//   warpgroup h: pixels 64h .. 64h+63 of the strip (MMA issue + epilogue).  The MMAs of input row i + 1 are issued before
//   the output row that row i completes is stored, so the tensor core works through the stores.  16-bit output rows leave
//   through TMA tensor stores from swizzled shared-memory slots; nothing in the epilogue branches on the thread index (such
//   a branch while a group is in flight makes ptxas serialise every wgmma of the kernel, C7518).
// Work item = (image, 128-pixel column strip, segment of RS output rows); persistent CTAs walk the items.
// ================================================================================================
constexpr int ROW_PX = 128;
// bytes of one input-row buffer: 130 halo pixels x KBW channels, padded to a multiple of the 8-row swizzle atom
__host__ __device__ constexpr int row_abytes(int kbw) { return ((130 * kbw * 2 + 255) / 256) * 256; }

// The MMAs of one input row (KB channel blocks x KBW/16 k-steps x 3 pixel shifts) into acc as one commit group.  The first
// has scale-d = 0, so acc needs no zero fill: no other instruction writes accumulator registers while a group is in flight.
template <int NT, int KBW, int KB, int DT>
__device__ __forceinline__ void row_mma(float (&acc)[3 * NT / 2], uint32_t a_row, uint32_t w_u) {
  constexpr int NG = 3 * NT, SWB = KBW * 2, ROW_ABYTES = row_abytes(KBW);
  // the weights are loop-invariant: without this, ptxas hoists their descriptors out of the row loop and keeps them live
  asm volatile("" : "+r"(w_u));
  wgmma_fence();
#pragma unroll
  for (int kb = 0; kb < KB; ++kb) {
#pragma unroll
    for (int ks = 0; ks < KBW / 16; ++ks) {
#pragma unroll
      for (int dx = 0; dx < 3; ++dx)
        Wgmma<NG>::template mma<0, 0, DT>(acc, gmma_desc<SWB>(a_row + (uint32_t)(kb * ROW_ABYTES + dx * SWB + 32 * ks), 16, 8 * SWB),
                                          gmma_desc<SWB>(w_u + (uint32_t)((kb * 3 + dx) * NG * SWB + 32 * ks), 16, 8 * SWB),
                                          (kb > 0 || ks > 0 || dx > 0) ? 1u : 0u);
    }
  }
  wgmma_commit();
}

// fp32 global store where `on` is set, as a predicated instruction (see tma_store_4d: no branch on the thread index while an
// MMA group is in flight)
__device__ __forceinline__ void st_f32_if(bool on, float* ptr, float v) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %0, 0;\n\t@p st.global.f32 [%1], %2;\n\t}" ::"r"((uint32_t)on), "l"(ptr), "f"(v)
               : "memory");
}

// Staged 16-bit output rows: per consumer warpgroup ROW_OUT_SLOTS slots of 64 pixels x NT channels, each the swizzled box of
// the output tensor map; consecutive stored rows alternate slots.
constexpr int ROW_OUT_SLOTS = 2;
__host__ __device__ constexpr int row_out_bytes(int nt) { return 2 * ROW_OUT_SLOTS * 64 * nt * 2; }

// OM: output mode as a template parameter (0: 16-bit NHWC through TMA stores, 1: fp32 NCHW logits stored directly).
template <int NT, int KBW, int KB, int DT, int OM>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_row_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
                                                                  const __grid_constant__ CUtensorMap map_b,
                                                                  const __grid_constant__ CUtensorMap map_o, const ConvV2Params p,
                                                                  const int RS, const int w_bytes, const int STAGES) {
  constexpr int NG = 3 * NT;                              // accumulator columns of one input row (three filter rows)
  constexpr int SWB = KBW * 2, ROW_ABYTES = row_abytes(KBW);   // channel block = swizzle span: 32 B (16 ch) or 64 B (32 ch)
  constexpr int SLOT_BYTES = 64 * NT * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* w_smem = smem;                                 // [KB][dx][3*NT rows x SWB]
  uint8_t* o_smem = smem + w_bytes;                       // [warpgroup][slot] staged output rows (w_bytes is a multiple of 1024)
  uint8_t* a_smem = o_smem + row_out_bytes(NT);
  uint64_t* bars = reinterpret_cast<uint64_t*>(a_smem + (size_t)STAGES * KB * ROW_ABYTES);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + STAGES;
  uint64_t* w_bar = bars + 2 * STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kb0 = p.C0 / KBW;
  const int strips = p.W / ROW_PX, segs = p.H / RS;
  const int items = p.N * strips * segs;
  const int my_items = (items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int rows_in = RS + 2;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], CONSUMER_WARPS); }
    mbar_init(w_bar, 1);
    fence_barrier_init();
    prefetch_tmap(&map_a0);
    prefetch_tmap(&map_b);
    if (OM == 0) prefetch_tmap(&map_o);
  }
  __syncthreads();

  if (warp >= PRODUCER_WARP) {
    producer_regs();
    if (warp != PRODUCER_WARP) return;
    if (lane == 0) {
      mbar_expect_tx(w_bar, (uint32_t)(KB * 9 * NT * SWB));
      for (int kb = 0; kb < KB; ++kb)
        for (int dx = 0; dx < 3; ++dx)
          for (int dy = 0; dy < 3; ++dy)
            tma_load_3d(&map_b, w_bar, w_smem + (((kb * 3 + dx) * 3 + dy) * NT) * SWB, kb * KBW, 0, dy * 3 + dx);
    }
    __syncwarp();
    // row loop: the warp stays converged, one elected lane issues with warp-uniform operands
    const uint32_t elected = elect_one();
    const uint32_t a_u = uniform(smem_u32(a_smem)), full_u = uniform(smem_u32(a_full));
    int s = 0;
    uint32_t sph = 1;                    // parity to wait for on a_empty[s] (fresh barrier: passes)
    for (int it = 0; it < my_items; ++it) {
      const int item = blockIdx.x + it * gridDim.x;
      const int seg = item % segs, t1 = item / segs, strip = t1 % strips, n = t1 / strips;
      const int y0 = seg * RS, x0 = strip * ROW_PX;
      for (int i = 0; i < rows_in; ++i) {
        mbar_wait(&a_empty[s], sph);
        if (elected) {
          const uint32_t bar = full_u + (uint32_t)(s * 8);
          asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((uint32_t)(KB * 130 * SWB)) : "memory");
          for (int kb = 0; kb < KB; ++kb) {
            const uint32_t dst = a_u + (uint32_t)((s * KB + kb) * ROW_ABYTES);
            const CUtensorMap* mp = (kb < kb0) ? &map_a0 : &map_a1;
            const int c0 = (kb < kb0 ? kb : kb - kb0) * KBW;
            asm volatile(
                "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                ::"r"(dst), "l"((uint64_t)mp), "r"(bar), "r"(c0), "r"(x0 - 1), "r"(y0 - 1 + i), "r"(n)
                : "memory");
          }
        }
        __syncwarp();
        if (++s == STAGES) { s = 0; sph ^= 1u; }
      }
    }
    return;
  }
  consumer_regs();
  // consumers: bias from shared memory, BatchNorm partial sums accumulated per thread and combined once at the end
  __shared__ float s_bias[NT];
  const int h = threadIdx.x >> 7, t = threadIdx.x & 127;
  if (threadIdx.x < NT) s_bias[threadIdx.x] = p.bias ? p.bias[threadIdx.x] : 0.f;
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
  const uint32_t a_u = smem_u32(a_smem) + (uint32_t)(64 * h * SWB), w_u = smem_u32(w_smem);
  float ls[NT / 4], lq[NT / 4];
#pragma unroll
  for (int k = 0; k < NT / 4; ++k) ls[k] = lq[k] = 0.f;
  mbar_wait(w_bar, 0);
  // The CTA walks R = my_items * (RS + 2) input rows in the producer's order (row r sits in stage r % STAGES); every CTA has
  // at least one item (the host keeps the grid <= items).
  const int R = my_items * rows_in;
  const bool store_thread = t == 0;     // issues (and waits for) the TMA stores of its warpgroup's 64 pixels
  const bool stats = OM == 0 && p.stat_partials != nullptr;
  uint8_t* o_wg = o_smem + h * ROW_OUT_SLOTS * SLOT_BYTES;
  // staging offset of this thread's first pair: pixel frag_row, channel frag_col of its warpgroup's box
  const uint32_t o_thr = out_stage_offset<NT, SLOT_BYTES>(frag_row(t), frag_col(t));
  float pa[NT / 2], pb[NT / 2];         // partial output rows i-2 (dy 0 + 1 summed) and i-1 (dy 0)
  float o[NT / 2];                      // output row i - 2 of the last folded row i, before rounding to the storage type
#pragma unroll
  for (int e = 0; e < NT / 2; ++e) pa[e] = pb[e] = 0.f;

  int s_iss = 0, s_rel = 0;             // stage of the next row to issue / of the row whose group retires next
  uint32_t ph_iss = 0;
  auto issue = [&](float (&acc)[NG / 2]) {
    mbar_wait(&a_full[s_iss], ph_iss);
    row_mma<NT, KBW, KB, DT>(acc, a_u + (uint32_t)(s_iss * KB * ROW_ABYTES), w_u);
    if (++s_iss == STAGES) { s_iss = 0; ph_iss ^= 1u; }
  };
  // acc holds the retired group of row r: free its stage and fold it into o and the partial rows.  The partial rows need no
  // reset between items: what they hold at an item's first row reaches only the outputs of rows 0 and 1, which are not stored.
  auto fold = [&](float (&acc)[NG / 2]) {
    release_stage(&a_empty[s_rel]);
    if (++s_rel == STAGES) s_rel = 0;
    wgmma_fence_regs(acc);
    // column 8*j + frag_col + b of E: filter row j / (NT/8), output channel 8*(j % (NT/8)) + frag_col + b
#pragma unroll
    for (int ii = 0; ii < 2; ++ii)
#pragma unroll
      for (int jj = 0; jj < NT / 8; ++jj)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int e = 4 * jj + 2 * ii + b;
          o[e] = (pa[e] + acc[4 * (2 * NT / 8 + jj) + 2 * ii + b]) + s_bias[8 * jj + frag_col(t) + b];
          pa[e] = pb[e] + acc[4 * (NT / 8 + jj) + 2 * ii + b];   // output row i - 1: + filter row 1
          pb[e] = acc[4 * jj + 2 * ii + b];                       // output row i: filter row 0
        }
    wgmma_discard_regs(acc);
  };
  // output row i - 2 of the current item, complete once its row i >= 2 (the CTA's row r) is folded
  int i = 0, n = 0, strip = 0, y0 = 0;
  auto start_item = [&](int it) {
    const int item = blockIdx.x + it * (int)gridDim.x;
    const int seg = item % segs, t1 = item / segs;
    strip = t1 % strips; n = t1 / strips; y0 = seg * RS;
  };
  auto store_row = [&](int r) {
    if (i < 2) return;
    const int gy = y0 + i - 2;
    if constexpr (OM == 0) {
      // Consecutive stored rows alternate slots (an item's rows 0 and 1 store nothing, which keeps the alternation), and the
      // wait before the barrier of one row frees the slot the next row writes.
      const uint32_t slot = (uint32_t)((r & 1) * SLOT_BYTES);
#pragma unroll
      for (int ii = 0; ii < 2; ++ii)
#pragma unroll
        for (int jj = 0; jj < NT / 8; ++jj) {
          const int e = 4 * jj + 2 * ii;
          const uint32_t u = DT == 2 ? pack_f16(o[e], o[e + 1]) : pack_bf16(o[e], o[e + 1]);
          if (stats) {                   // statistics of the values exactly as stored (rounded to the 16-bit type)
            float2 v;
            if (DT == 2) v = __half22float2(*reinterpret_cast<const __half2*>(&u));
            else v = make_float2(bf16_lo(u), bf16_hi(u));
            ls[2 * jj] += v.x;     lq[2 * jj] = fmaf(v.x, v.x, lq[2 * jj]);
            ls[2 * jj + 1] += v.y; lq[2 * jj + 1] = fmaf(v.y, v.y, lq[2 * jj + 1]);
          }
          // pixel + 8 is NT * 16 bytes further on, which keeps the swizzle phase: channel group jj is an XOR of the base offset
          *reinterpret_cast<uint32_t*>(o_wg + ((o_thr + slot + (uint32_t)(8 * ii * NT * 2)) ^ (uint32_t)(jj << 4))) = u;
        }
      fence_proxy_async();
      bulk_wait_read_all(store_thread);  // the previous row's store has read the other slot
      asm volatile("bar.sync %0, 128;" ::"r"(2 + h) : "memory");
      tma_store_4d(store_thread, &map_o, o_wg + slot, 0, strip * ROW_PX + 64 * h, gy, n);
      bulk_commit(store_thread);
    } else {
      float* out = reinterpret_cast<float*>(p.out);
#pragma unroll
      for (int ii = 0; ii < 2; ++ii) {
        const int gx = strip * ROW_PX + 64 * h + frag_row(t) + 8 * ii;
#pragma unroll
        for (int jj = 0; jj < NT / 8; ++jj)
#pragma unroll
          for (int b = 0; b < 2; ++b) {
            const int c = 8 * jj + frag_col(t) + b;
            st_f32_if(c < p.CoutStore, out + (((long long)n * p.CoutStore + c) * p.H + gy) * p.W + gx, o[4 * jj + 2 * ii + b]);
          }
      }
    }
  };

  // One accumulator: row r is folded as soon as its group retires, then row r + 1's group is issued and runs while row r's
  // output row is rounded, staged and stored.  A second accumulator would let row r + 1's group run under the fold as well,
  // but ptxas then reports too few registers for the wgmma pipeline (C7511, at NT = 16 too) and serialises every MMA.  The
  // last row is peeled: no MMA is issued on a path that joins one without a group in flight.
  float acc[NG / 2];
  issue(acc);
  start_item(0);
  for (int r = 0, it = 0;; ++r) {
    wgmma_wait<0>();
    fold(acc);
    if (r + 1 == R) {
      store_row(r);
      break;
    }
    issue(acc);
    store_row(r);
    if (++i == rows_in) { i = 0; start_item(++it); }
  }
  bulk_wait_all(store_thread);
  __shared__ float s_stat[CONSUMER_WARPS][2][NT];
  if (stats) write_stat_partials<NT>(ls, lq, p.stat_partials, p.CoutP, 0, s_stat);
}

template <int NT, int KBW, int KB, int DT, int OM>
int launch_conv_row(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& o, const ConvV2Params& p,
                    int RS, cudaStream_t stream) {
  // Row buffers in flight: ~80 KB per SM cover the HBM latency.
  const int STAGES = KB == 1 ? 12 : KB == 2 ? 8 : 6;
  const int w_bytes = ((KB * 9 * NT * KBW * 2 + 1023) / 1024) * 1024;
  const int smem = w_bytes + row_out_bytes(NT) + STAGES * KB * row_abytes(KBW) + 1024 + 256;
  if (smem > 220 * 1024) { wsl_set_error("conv_row: %d bytes of shared memory needed", smem); return -6; }
  static int attr_bytes = 0;
  if (smem > attr_bytes) {
    cudaError_t e = cudaFuncSetAttribute(conv_row_kernel<NT, KBW, KB, DT, OM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { wsl_set_error("conv_row: cudaFuncSetAttribute(%d): %s", smem, cudaGetErrorString(e)); return -5; }
    attr_bytes = smem;
  }
  const int items = p.N * (p.W / ROW_PX) * (p.H / RS);
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, conv_row_kernel<NT, KBW, KB, DT, OM>, NUM_THREADS, smem);
  if (occ < 1) occ = 1;
  int gx = wsl_num_sms() * occ;
  if (gx > items) gx = items;
  g_conv2_last_rows = gx;
  conv_row_kernel<NT, KBW, KB, DT, OM><<<gx, NUM_THREADS, smem, stream>>>(a0, a1, b, o, p, RS, w_bytes, STAGES);
  return wsl_check_launch("conv_row");
}

// KB = (C0 + C1) / KBW channel blocks: 1-4 at KBW = 16, 1-2 at KBW = 32 (the caller keeps C0 + C1 <= 64)
template <int NT, int KBW, int DT, int OM>
int conv_row_dispatch_kb(int KB, const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& b, const CUtensorMap& o,
                         const ConvV2Params& p, int RS, cudaStream_t stream) {
  switch (KB) {
    case 1: return launch_conv_row<NT, KBW, 1, DT, OM>(a0, a1, b, o, p, RS, stream);
    case 2: return launch_conv_row<NT, KBW, 2, DT, OM>(a0, a1, b, o, p, RS, stream);
    case 3: if constexpr (KBW == 16) return launch_conv_row<NT, KBW, 3, DT, OM>(a0, a1, b, o, p, RS, stream); else break;
    case 4: if constexpr (KBW == 16) return launch_conv_row<NT, KBW, 4, DT, OM>(a0, a1, b, o, p, RS, stream); else break;
  }
  wsl_set_error("conv_row: unsupported channel block count %d", KB);
  return -1;
}

}  // namespace

WSL_API int wsl_tc_available(void) { return get_encode() != nullptr ? 1 : 0; }

static int conv_tc_impl(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias, void* out,
                        int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype, int dilation,
                        cudaStream_t stream) {
  WSL_REQUIRE(ksize == 3 || ksize == 1, "wsl_conv_tc: ksize must be 1 or 3");
  WSL_REQUIRE(dilation >= 1 && dilation <= 64, "wsl_conv_tc: dilation must be in 1..64 (got %d)", dilation);
  WSL_REQUIRE(dtype == 0 || dtype == 2, "wsl_conv_tc: dtype must be 0 (bf16) or 2 (fp16)");
  WSL_REQUIRE(C0 % 16 == 0 && C1 % 16 == 0 && C0 > 0, "wsl_conv_tc: source channels must be multiples of 16 (got %d,%d)", C0, C1);
  WSL_REQUIRE(CoutP % 16 == 0, "wsl_conv_tc: CoutP must be a multiple of 16");
  WSL_REQUIRE(W % TILE_W == 0 && H % TILE_H == 0, "wsl_conv_tc: H,W must be multiples of the 8x16 pixel tile (got %dx%d)", H, W);
  // k-block = largest of 64/32/16 dividing both sources' channel counts
  int kblk = 64;
  while (kblk > 16 && (C0 % kblk != 0 || (C1 > 0 && C1 % kblk != 0))) kblk >>= 1;
  int nt = CoutP >= 128 ? 128 : CoutP;
  while (nt > 16 && CoutP % nt != 0) nt >>= 1;          // e.g. CoutP = 320 (PNet2D's concat block): five tiles of 64
  WSL_REQUIRE(CoutP % nt == 0 && (nt == 16 || nt == 32 || nt == 64 || nt == 128), "wsl_conv_tc: unsupported CoutP %d", CoutP);
  const int CinP = C0 + C1, T = ksize * ksize;
  CUtensorMap a0, a1, b;
  {
    long long d[4] = {C0, W, H, N};
    int bx[4] = {kblk, TILE_W, TILE_H, 1};
    int rc = get_map(src0, 4, d, bx, kblk, &a0, dtype);
    if (rc) return rc;
  }
  if (C1 > 0) {
    long long d[4] = {C1, W, H, N};
    int bx[4] = {kblk, TILE_W, TILE_H, 1};
    int rc = get_map(src1, 4, d, bx, kblk, &a1, dtype);
    if (rc) return rc;
  } else {
    a1 = a0;
  }
  {
    long long d[3] = {CinP, CoutP, T};
    int bx[3] = {kblk, nt, 1};
    int rc = get_map(wpk_bf16, 3, d, bx, kblk, &b, dtype);
    if (rc) return rc;
  }
  ConvTcParams p;
  p.N = N; p.H = H; p.W = W; p.C0 = C0; p.C1 = C1; p.CoutP = CoutP; p.CoutStore = CoutStore; p.taps = T; p.ks = ksize;
  p.tiles_x = W / TILE_W; p.tiles_y = H / TILE_H; p.out_mode = out_mode; p.dt = dtype; p.dil = dilation; p.bias = bias; p.out_scale = nullptr; p.out = out;
  switch (kblk) {
    case 64: return dispatch_nt<64>(a0, a1, b, p, nt, stream);
    case 32: return dispatch_nt<32>(a0, a1, b, p, nt, stream);
    default: return dispatch_nt<16>(a0, a1, b, p, nt, stream);
  }
}

WSL_API int wsl_conv_tc(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias, void* out,
                        int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype, cudaStream_t stream) {
  return conv_tc_impl(src0, C0, src1, C1, wpk_bf16, bias, out, out_mode, N, H, W, CoutP, CoutStore, ksize, dtype, 1, stream);
}

// dilated 3x3 convolution (PNet2D, networks/pnet.py:25-28): same kernel, tap coordinates scaled by the dilation (TMA zero fill = padding)
WSL_API int wsl_conv_tc_dil(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias, void* out,
                            int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype, int dilation,
                            cudaStream_t stream) {
  return conv_tc_impl(src0, C0, src1, C1, wpk_bf16, bias, out, out_mode, N, H, W, CoutP, CoutStore, ksize, dtype, dilation, stream);
}

// pitch_x / pitch_dy > 0: the operands are channel-range views of wider channels-last tensors (fp16 hi/lo split planes)
static int wgrad_tc_impl(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                         int W, int CoutReal, int ksize, int dtype, int pitch_x, int pitch_dy, const float* scale_a,
                         const float* scale_b, cudaStream_t stream, float* partial_ws = nullptr, long long partial_floats = 0,
                         int dilation = 1) {
  g_wgrad1_ws = partial_ws;
  g_wgrad1_ws_floats = partial_floats;
  WSL_REQUIRE(ksize == 3 || ksize == 1, "wsl_wgrad_tc: ksize must be 1 or 3");
  WSL_REQUIRE(dtype == 0 || dtype == 2, "wsl_wgrad_tc: dtype must be 0 (bf16) or 2 (fp16)");
  WSL_REQUIRE(C0 % 16 == 0 && C1 % 16 == 0 && C0 > 0, "wsl_wgrad_tc: source channels must be multiples of 16 (got %d,%d)", C0, C1);
  WSL_REQUIRE(CoutP % 16 == 0, "wsl_wgrad_tc: CoutP must be a multiple of 16");
  WSL_REQUIRE(W % TILE_W == 0 && H % TILE_H == 0, "wsl_wgrad_tc: H,W must be multiples of the 8x16 pixel tile (got %dx%d)", H, W);
  const int cwa = CoutP >= 64 ? 64 : CoutP;       // 16 / 32 / 64
  WSL_REQUIRE(cwa == 16 || cwa == 32 || cwa == 64, "wsl_wgrad_tc: unsupported CoutP %d", CoutP);
  WSL_REQUIRE(CoutP <= 64 || CoutP % 64 == 0, "wsl_wgrad_tc: CoutP above 64 must be a multiple of 64 (got %d)", CoutP);   // one dY box per 64 couts
  int cwb = 64;
  while (cwb > 16 && (C0 % cwb != 0 || (C1 > 0 && C1 % cwb != 0))) cwb >>= 1;
  const int na = CoutP >= 128 ? 2 : 1;
  const int m_tiles = CoutP >= 128 ? (CoutP + 127) / 128 : 1;
  CUtensorMap mdy, mx0, mx1;
  {
    long long d[4] = {CoutP, W, H, N};
    int bx[4] = {cwa, TILE_W, TILE_H, 1};
    int rc = get_map(dy, 4, d, bx, cwa, &mdy, dtype, pitch_dy);
    if (rc) return rc;
  }
  {
    long long d[4] = {C0, W, H, N};
    int bx[4] = {cwb, TILE_W, TILE_H, 1};
    int rc = get_map(src0, 4, d, bx, cwb, &mx0, dtype, pitch_x);
    if (rc) return rc;
  }
  if (C1 > 0) {
    long long d[4] = {C1, W, H, N};
    int bx[4] = {cwb, TILE_W, TILE_H, 1};
    int rc = get_map(src1, 4, d, bx, cwb, &mx1, dtype, pitch_x);
    if (rc) return rc;
  } else {
    mx1 = mx0;
  }
  WgradTcParams p;
  p.N = N; p.H = H; p.W = W; p.C0 = C0; p.C1 = C1; p.CoutP = CoutP; p.CoutReal = CoutReal; p.taps = ksize * ksize; p.ks = ksize;
  p.tiles_x = W / TILE_W; p.tiles_y = H / TILE_H; p.nchunks = N * p.tiles_x * p.tiles_y;
  p.n_tiles0 = C0 / cwb; p.n_tiles1 = C1 / cwb; p.tap_groups = ksize == 3 ? 3 : 1; p.dt = dtype; p.scale_a = scale_a; p.scale_b = scale_b; p.dw = dw; p.partials = nullptr; p.dil = dilation;
  if (cwa == 64 && na == 2) return wgrad_dispatch_b<64, 2>(cwb, mdy, mx0, mx1, p, m_tiles, stream);
  if (cwa == 64) return wgrad_dispatch_b<64, 1>(cwb, mdy, mx0, mx1, p, m_tiles, stream);
  if (cwa == 32) return wgrad_dispatch_b<32, 1>(cwb, mdy, mx0, mx1, p, m_tiles, stream);
  return wgrad_dispatch_b<16, 1>(cwb, mdy, mx0, mx1, p, m_tiles, stream);
}

WSL_API int wsl_wgrad_tc(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                         int W, int CoutReal, int ksize, int dtype, float* partial_ws, long long partial_floats, cudaStream_t stream) {
  return wgrad_tc_impl(src0, C0, src1, C1, dy, CoutP, dw, N, H, W, CoutReal, ksize, dtype, 0, 0, nullptr, nullptr, stream, partial_ws,
                       partial_floats);
}

WSL_API int wsl_wgrad_tc_dil(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                             int W, int CoutReal, int ksize, int dtype, int dilation, float* partial_ws, long long partial_floats,
                             cudaStream_t stream) {
  WSL_REQUIRE(dilation >= 1 && dilation <= 64, "wsl_wgrad_tc_dil: dilation must be in 1..64 (got %d)", dilation);
  return wgrad_tc_impl(src0, C0, src1, C1, dy, CoutP, dw, N, H, W, CoutReal, ksize, dtype, 0, 0, nullptr, nullptr, stream, partial_ws,
                       partial_floats, dilation);
}

// ---- fp16 hi/lo split ("fp16x3") tensor-core parity mode ------------------------------------------------------------
// An fp32 value v is carried as hi = fp16(v), lo = fp16(v - hi) (22 significant bits); a product a*b is evaluated as
// a_hi*b_hi + a_lo*b_hi + a_hi*b_lo on kind::f16 with fp32 accumulation (the dropped lo*lo term is ~2^-22 relative).
// Staged operands are channels-last fp16 [P][2C] = (hi plane | lo plane), produced by wsl_split_f32 (net_ops.cu).
//   forward / data gradient: K = 3*Cin: source 0 = the whole staged tensor (hi | lo) against (w_hi | w_hi), source 1 = its hi
//   plane again (channel-range view, pitch 2*Cin) against w_lo; weights fp16 [T][CoutP][3*Cin] from wsl_pack_split_weights.
//   weight gradient: three accumulating launches (dy_hi,x_hi), (dy_hi,x_lo), (dy_lo,x_hi).
// out_mode 2: fp32 NHWC [P][CoutStore]; 1: fp32 NCHW.
WSL_API int wsl_conv_tc_split(const void* staged, int Cin, const float* inv_scale, const void* wpk3, const float* bias, float* out,
                              int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dilation, cudaStream_t stream) {
  WSL_REQUIRE(dilation >= 1 && dilation <= 64, "wsl_conv_tc_split: dilation must be in 1..64 (got %d)", dilation);
  WSL_REQUIRE(ksize == 3 || ksize == 1, "wsl_conv_tc_split: ksize must be 1 or 3");
  WSL_REQUIRE(Cin % 16 == 0 && Cin > 0 && CoutP % 16 == 0, "wsl_conv_tc_split: channel counts must be multiples of 16 (got %d,%d)", Cin, CoutP);
  WSL_REQUIRE(W % TILE_W == 0 && H % TILE_H == 0, "wsl_conv_tc_split: H,W must be multiples of the 8x16 pixel tile (got %dx%d)", H, W);
  WSL_REQUIRE(out_mode == 1 || out_mode == 2, "wsl_conv_tc_split: out_mode must be 1 (fp32 NCHW) or 2 (fp32 NHWC)");
  int kblk = 64;
  while (kblk > 16 && Cin % kblk != 0) kblk >>= 1;
  int nt = CoutP >= 128 ? 128 : CoutP;
  while (nt > 16 && CoutP % nt != 0) nt >>= 1;
  WSL_REQUIRE(CoutP % nt == 0 && (nt == 16 || nt == 32 || nt == 64 || nt == 128), "wsl_conv_tc_split: unsupported CoutP %d", CoutP);
  const int T = ksize * ksize;
  CUtensorMap a0, a1, b;
  {
    long long d[4] = {2LL * Cin, W, H, N};
    int bx[4] = {kblk, TILE_W, TILE_H, 1};
    int rc = get_map(staged, 4, d, bx, kblk, &a0, 2);
    if (rc) return rc;
  }
  {
    long long d[4] = {Cin, W, H, N};
    int bx[4] = {kblk, TILE_W, TILE_H, 1};
    int rc = get_map(staged, 4, d, bx, kblk, &a1, 2, 2 * Cin);
    if (rc) return rc;
  }
  {
    long long d[3] = {3LL * Cin, CoutP, T};
    int bx[3] = {kblk, nt, 1};
    int rc = get_map(wpk3, 3, d, bx, kblk, &b, 2);
    if (rc) return rc;
  }
  ConvTcParams p;
  p.N = N; p.H = H; p.W = W; p.C0 = 2 * Cin; p.C1 = Cin; p.CoutP = CoutP; p.CoutStore = CoutStore; p.taps = T; p.ks = ksize;
  p.tiles_x = W / TILE_W; p.tiles_y = H / TILE_H; p.out_mode = out_mode; p.dt = 2; p.dil = dilation; p.bias = bias; p.out_scale = inv_scale; p.out = out;
  switch (kblk) {
    case 64: return dispatch_nt<64>(a0, a1, b, p, nt, stream);
    case 32: return dispatch_nt<32>(a0, a1, b, p, nt, stream);
    default: return dispatch_nt<16>(a0, a1, b, p, nt, stream);
  }
}

WSL_API int wsl_wgrad_tc_split(const void* x_staged, int Cin, const float* x_inv_scale, const void* dy_staged, int CoutP,
                               const float* dy_inv_scale, float* dw, int N, int H, int W, int CoutReal, int ksize, int dilation,
                               cudaStream_t stream) {
  WSL_REQUIRE(Cin % 16 == 0 && Cin > 0, "wsl_wgrad_tc_split: Cin must be a multiple of 16 (got %d)", Cin);
  const __half* x = reinterpret_cast<const __half*>(x_staged);
  const __half* g = reinterpret_cast<const __half*>(dy_staged);
  int rc = wgrad_tc_impl(x, Cin, nullptr, 0, g, CoutP, dw, N, H, W, CoutReal, ksize, 2, 2 * Cin, 2 * CoutP, dy_inv_scale, x_inv_scale, stream, nullptr, 0, dilation);
  if (rc) return rc;
  rc = wgrad_tc_impl(x + Cin, Cin, nullptr, 0, g, CoutP, dw, N, H, W, CoutReal, ksize, 2, 2 * Cin, 2 * CoutP, dy_inv_scale, x_inv_scale, stream, nullptr, 0, dilation);
  if (rc) return rc;
  return wgrad_tc_impl(x, Cin, nullptr, 0, g + CoutP, CoutP, dw, N, H, W, CoutReal, ksize, 2, 2 * Cin, 2 * CoutP, dy_inv_scale, x_inv_scale, stream, nullptr, 0, dilation);
}

WSL_API int wsl_channel_sum(const void* x, int dtype, long long P, int C, int Creal, float* out, float* ws, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0 && C / 8 <= 256 && Creal <= C, "wsl_channel_sum: unsupported channel count %d", C);
  const int rows = 256 / (C / 8);
  long long b = (P + rows * 16 - 1) / (rows * 16);
  if (b > wsl_num_sms() * 2) b = wsl_num_sms() * 2;
  if (b < 1) b = 1;
  if (dtype == 1) channel_sum_kernel<float><<<(int)b, 256, 256 * 8 * sizeof(float), stream>>>((const float*)x, P, C, Creal, out, ws);
  else if (dtype == 2) channel_sum_kernel<__nv_bfloat16, true><<<(int)b, 256, 256 * 8 * sizeof(float), stream>>>((const __nv_bfloat16*)x, P, C, Creal, out, ws);
  else channel_sum_kernel<__nv_bfloat16><<<(int)b, 256, 256 * 8 * sizeof(float), stream>>>((const __nv_bfloat16*)x, P, C, Creal, out, ws);
  return wsl_check_launch("channel_sum");
}

// conv_tc v2 entry point (same contract as wsl_conv_tc; needs W % 8 == 0 and H % (16*MT) == 0)
WSL_API int wsl_conv_tc2(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias, void* out,
                         int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype, float* stat_partials,
                         int* stat_rows_host, cudaStream_t stream) {
  WSL_REQUIRE(ksize == 3 || ksize == 1, "wsl_conv_tc2: ksize must be 1 or 3");
  WSL_REQUIRE(dtype == 0 || dtype == 2, "wsl_conv_tc2: dtype must be 0 (bf16) or 2 (fp16)");
  // both epilogues store 16-bit NHWC or fp32 NCHW only (store_pair(..., out_mode == 0 ? 0 : 1, ...))
  WSL_REQUIRE(out_mode == 0 || out_mode == 1, "wsl_conv_tc2: out_mode must be 0 (16-bit NHWC) or 1 (fp32 NCHW), got %d", out_mode);
  WSL_REQUIRE(C0 % 16 == 0 && C1 % 16 == 0 && C0 > 0, "wsl_conv_tc2: source channels must be multiples of 16 (got %d,%d)", C0, C1);
  WSL_REQUIRE(CoutP % 16 == 0, "wsl_conv_tc2: CoutP must be a multiple of 16");
  // 16-bit outputs leave through TMA stores, whose global row pitch must be a multiple of 16 bytes
  WSL_REQUIRE(out_mode != 0 || CoutStore % 8 == 0, "wsl_conv_tc2: 16-bit outputs need CoutStore %% 8 == 0 (got %d)", CoutStore);
  {   // narrow outputs at >= 128-pixel rows: the row kernel (filter rows in N) is 1.8-2.3x faster per pixel
    // channel block per TMA box / swizzle span: 32 channels (64 B) when every source allows it and the output is 32 wide
    const int kbw = (CoutP == 32 && C0 % 32 == 0 && C1 % 32 == 0) ? 32 : 16;
    const int KB = (C0 + C1) / kbw;
    // row segments of 32 output rows (6 % halo re-reads) unless that leaves fewer than ~4 work items per SM
    const int RS = (H % 32 == 0 && (long long)N * (W / ROW_PX) * (H / 32) >= 4 * wsl_num_sms()) ? 32 : 16;
    if (ksize == 3 && (CoutP == 16 || CoutP == 32) && W % ROW_PX == 0 && H % 16 == 0 && (C0 + C1) <= 64) {
      CUtensorMap a0, a1, b;
      {
        long long d[4] = {C0, W, H, N};
        int bx[4] = {kbw, 130, 1, 1};
        int rc = get_map(src0, 4, d, bx, kbw, &a0, dtype);
        if (rc) return rc;
      }
      if (C1 > 0) {
        long long d[4] = {C1, W, H, N};
        int bx[4] = {kbw, 130, 1, 1};
        int rc = get_map(src1, 4, d, bx, kbw, &a1, dtype);
        if (rc) return rc;
      } else {
        a1 = a0;
      }
      {
        long long d[3] = {C0 + C1, CoutP, 9};
        int bx[3] = {kbw, CoutP, 1};
        int rc = get_map(wpk_bf16, 3, d, bx, kbw, &b, dtype);
        if (rc) return rc;
      }
      CUtensorMap o;
      if (out_mode == 0) {   // one box per warpgroup: CoutP channels x 64 pixels of one row; TMA clips channels >= CoutStore
        long long d[4] = {CoutStore, W, H, N};
        int bx[4] = {CoutP, 64, 1, 1};
        int rc = get_map(out, 4, d, bx, CoutP, &o, dtype);
        if (rc) return rc;
      } else {
        o = a0;
      }
      ConvV2Params p;
      p.N = N; p.H = H; p.W = W; p.C0 = C0; p.C1 = C1; p.CoutP = CoutP; p.CoutStore = CoutStore;
      p.tiles_x = 0; p.tiles_y = 0; p.ntiles = 0;
      p.out_mode = out_mode; p.dt = dtype; p.bias = bias; p.out = out;
      p.stat_partials = (out_mode == 0) ? stat_partials : nullptr;
      auto by_nt = [&](auto om) {
        constexpr int OM = decltype(om)::value;
        return with_dt(dtype, [&](auto dt) {
          constexpr int DT = decltype(dt)::value;
          return (CoutP == 16) ? conv_row_dispatch_kb<16, 16, DT, OM>(KB, a0, a1, b, o, p, RS, stream)
                 : (kbw == 32) ? conv_row_dispatch_kb<32, 32, DT, OM>(KB, a0, a1, b, o, p, RS, stream)
                               : conv_row_dispatch_kb<32, 16, DT, OM>(KB, a0, a1, b, o, p, RS, stream);
        });
      };
      const int rc = out_mode == 0 ? by_nt(std::integral_constant<int, 0>{}) : by_nt(std::integral_constant<int, 1>{});
      if (stat_rows_host) *stat_rows_host = g_conv2_last_rows;
      return rc;
    }
  }
  int kblk = 64;
  while (kblk > 16 && (C0 % kblk != 0 || (C1 > 0 && C1 % kblk != 0))) kblk >>= 1;
  int mt = kblk == 64 ? 1 : kblk == 32 ? 2 : 4;
  while (mt > 1 && H % (16 * mt) != 0) mt >>= 1;
  WSL_REQUIRE(W % 8 == 0 && H % (16 * mt) == 0, "wsl_conv_tc2: H,W must be multiples of the 16x8 pixel tile (got %dx%d)", H, W);
  const int CinP = C0 + C1, T = ksize * ksize;
  // N tile: largest of 128/64/32/16 dividing CoutP whose resident weight slice fits (~148 KB) and whose accumulators
  // fit the registers (MT*NT <= 128: 64 fp32 per consumer thread)
  int nt = CoutP >= 128 ? 128 : CoutP;
  while (nt > 16 && (CoutP % nt != 0 || (long long)T * CinP * nt * 2 > 148 * 1024 || mt * nt > 128)) nt >>= 1;
  WSL_REQUIRE(CoutP % nt == 0 && (long long)T * CinP * nt * 2 <= 152 * 1024, "wsl_conv_tc2: weights do not fit (Cin %d, NT %d)", CinP, nt);
  const int pad = ksize / 2;
  CUtensorMap a0, a1, b, o;
  {
    long long d[4] = {C0, W, H, N};
    int bx[4] = {kblk, 8 + 2 * pad, 16 * mt + 2 * pad, 1};
    int rc = get_map(src0, 4, d, bx, kblk, &a0, dtype);
    if (rc) return rc;
  }
  if (C1 > 0) {
    long long d[4] = {C1, W, H, N};
    int bx[4] = {kblk, 8 + 2 * pad, 16 * mt + 2 * pad, 1};
    int rc = get_map(src1, 4, d, bx, kblk, &a1, dtype);
    if (rc) return rc;
  } else {
    a1 = a0;
  }
  {
    long long d[3] = {CinP, CoutP, T};
    int bx[3] = {kblk, nt, 1};
    int rc = get_map(wpk_bf16, 3, d, bx, kblk, &b, dtype);
    if (rc) return rc;
  }
  if (out_mode == 0) {   // one box per 64 channels of the N tile (ConvV2Cfg::OUT_CH); TMA clips channels >= CoutStore
    long long d[4] = {CoutStore, W, H, N};
    const int och = nt < 64 ? nt : 64;
    int bx[4] = {och, 8, 16 * mt, 1};
    int rc = get_map(out, 4, d, bx, och, &o, dtype);
    if (rc) return rc;
  } else {
    o = a0;
  }
  ConvV2Params p;
  p.N = N; p.H = H; p.W = W; p.C0 = C0; p.C1 = C1; p.CoutP = CoutP; p.CoutStore = CoutStore;
  p.tiles_x = W / 8; p.tiles_y = H / (16 * mt); p.ntiles = N * p.tiles_x * p.tiles_y;
  p.out_mode = out_mode; p.dt = dtype; p.bias = bias; p.out = out;
  p.stat_partials = (out_mode == 0) ? stat_partials : nullptr;
#define WSL_C2(KS_, KB_, MT_)                                                   \
  do {                                                                         \
    int rc_ = conv2_dispatch_nt<KS_, KB_, MT_>(nt, a0, a1, b, o, p, stream);   \
    if (stat_rows_host) *stat_rows_host = g_conv2_last_rows;                   \
    return rc_;                                                                \
  } while (0)
  if (ksize == 3) {
    if (kblk == 64) WSL_C2(3, 64, 1);
    if (kblk == 32) { if (mt == 2) WSL_C2(3, 32, 2); WSL_C2(3, 32, 1); }
    if (mt == 4) WSL_C2(3, 16, 4);
    if (mt == 2) WSL_C2(3, 16, 2);
    WSL_C2(3, 16, 1);
  } else {
    if (kblk == 64) WSL_C2(1, 64, 1);
    if (kblk == 32) { if (mt == 2) WSL_C2(1, 32, 2); WSL_C2(1, 32, 1); }
    if (mt == 4) WSL_C2(1, 16, 4);
    if (mt == 2) WSL_C2(1, 16, 2);
    WSL_C2(1, 16, 1);
  }
#undef WSL_C2
}

// 3x3 weight gradient, v3 (filter columns in the MMA's M dimension).  Same contract as wsl_wgrad_tc; needs W % 8 == 0 and H % 16 == 0.
WSL_API int wsl_wgrad_tc3(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                          int W, int CoutReal, int ksize, int dtype, float* partial_ws, long long partial_floats, cudaStream_t stream) {
  WSL_REQUIRE(ksize == 3, "wsl_wgrad_tc3: 3x3 only");
  WSL_REQUIRE(dtype == 0 || dtype == 2, "wsl_wgrad_tc3: dtype must be 0 (bf16) or 2 (fp16)");
  WSL_REQUIRE(C0 % 16 == 0 && C1 % 16 == 0 && C0 > 0, "wsl_wgrad_tc3: source channels must be multiples of 16 (got %d,%d)", C0, C1);
  WSL_REQUIRE(CoutP % 16 == 0 && (CoutP <= 64 || CoutP % 128 == 0), "wsl_wgrad_tc3: unsupported CoutP %d", CoutP);
  WSL_REQUIRE(CoutP == 16 || CoutP == 32 || CoutP >= 64, "wsl_wgrad_tc3: unsupported CoutP %d", CoutP);
  WSL_REQUIRE(W % 8 == 0 && H % 16 == 0, "wsl_wgrad_tc3: H,W must be multiples of the 16x8 pixel chunk (got %dx%d)", H, W);
  const int cwb = (C0 % 32 == 0 && (C1 == 0 || C1 % 32 == 0)) ? 32 : 16;
  const int cwn = CoutP >= 64 ? 64 : CoutP;
  const int ntile = CoutP >= 64 ? 64 : CoutP;     // N = 3*ntile <= 192 accumulator columns per consumer thread pair
  const int n_tiles = CoutP / ntile;
  CUtensorMap mdy, mx0, mx1;
  {
    long long d[4] = {CoutP, W, H, N};
    int bx[4] = {cwn, 8, 18, 1};         // one halo row above and below: filter rows in the MMA's N dimension
    int rc = get_map(dy, 4, d, bx, cwn, &mdy, dtype);
    if (rc) return rc;
  }
  {
    long long d[4] = {C0, W, H, N};
    int bx[4] = {cwb, 10, 16, 1};
    int rc = get_map(src0, 4, d, bx, cwb, &mx0, dtype);
    if (rc) return rc;
  }
  if (C1 > 0) {
    long long d[4] = {C1, W, H, N};
    int bx[4] = {cwb, 10, 16, 1};
    int rc = get_map(src1, 4, d, bx, cwb, &mx1, dtype);
    if (rc) return rc;
  } else {
    mx1 = mx0;
  }
  Wgrad3Params p;
  p.N = N; p.H = H; p.W = W; p.C0 = C0; p.C1 = C1; p.CoutReal = CoutReal;
  p.tiles_x = W / 8; p.tiles_y = H / 16; p.nchunks = N * p.tiles_x * p.tiles_y;
  p.k_tiles0 = C0 / cwb; p.k_tiles1 = C1 / cwb; p.dt = dtype; p.dw = dw; p.partials = nullptr;
  return with_dt(dtype, [&](auto dt) {
    constexpr int DT = decltype(dt)::value;
#define WSL_W3(CWB_) \
    if (ntile == 64) return launch_wgrad3<CWB_, 64, DT>(mdy, mx0, mx1, p, n_tiles, partial_ws, partial_floats, stream);  \
    if (ntile == 32) return launch_wgrad3<CWB_, 32, DT>(mdy, mx0, mx1, p, n_tiles, partial_ws, partial_floats, stream);  \
    return launch_wgrad3<CWB_, 16, DT>(mdy, mx0, mx1, p, n_tiles, partial_ws, partial_floats, stream);
    if (cwb == 32) { WSL_W3(32) }
    WSL_W3(16)
#undef WSL_W3
  });
}

