// Network operators for the U-Net hot path on channels-last (NHWC) bf16 activations:
//   * direct (CUDA-core) convolution forward / data-gradient / weight-gradient -- used for the layers that do
//     not map to wgmma tiles (Cin = 1, tiny problems) and as the on-device cross-check of conv_tc.cu;
//   * training-mode BatchNorm statistics, normalise + LeakyReLU + dropout (+ fused 2x2 max-pool), and the
//     matching backward (reference: networks/unet.py:18-26,38);
//   * bilinear x2 upsample (align_corners=True, networks/unet.py:56-57) forward / backward;
//   * channel dropout of the aux branch (networks/unet.py:254-256,344);
//   * weight packing, fused SGD (train_weakly_supervised_pCE_2D.py:79-80,104).
#include "common.cuh"

namespace {

constexpr int TPB = 256;

// Storage type of activations / activation gradients: bf16 (fast path, tensor cores) or fp32 (the reference-accurate
// "parity" mode that runs the CUDA-core direct convolutions) or fp16 (same tensor-core rate as bf16, 11-bit mantissa; needs
// a scaled loss so that gradients stay in range).  dtype codes in the C ABI: 0 = bf16, 1 = fp32, 2 = fp16.
using bf16 = __nv_bfloat16;
template <typename T> __device__ __forceinline__ void ld8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void ld8<bf16>(const bf16* p, float (&v)[8]) { unpack8(*reinterpret_cast<const uint4*>(p), v); }
template <> __device__ __forceinline__ void ld8<__half>(const __half* p, float (&v)[8]) { unpack8h(*reinterpret_cast<const uint4*>(p), v); }
template <> __device__ __forceinline__ void ld8<float>(const float* p, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <typename T> __device__ __forceinline__ void st8(T* p, const float (&v)[8]);
template <> __device__ __forceinline__ void st8<bf16>(bf16* p, const float (&v)[8]) { *reinterpret_cast<uint4*>(p) = pack8(v); }
template <> __device__ __forceinline__ void st8<__half>(__half* p, const float (&v)[8]) { *reinterpret_cast<uint4*>(p) = pack8h(v); }
template <> __device__ __forceinline__ void st8<float>(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
// value as it will be read back from storage
template <typename T> __device__ __forceinline__ void round8(float (&v)[8]);
template <> __device__ __forceinline__ void round8<bf16>(float (&v)[8]) { const uint4 u = pack8(v); unpack8(u, v); }
template <> __device__ __forceinline__ void round8<__half>(float (&v)[8]) { const uint4 u = pack8h(v); unpack8h(u, v); }
template <> __device__ __forceinline__ void round8<float>(float (&v)[8]) {}
// generic source element loader for the direct convolutions (dtype code at run time)
__device__ __forceinline__ void ld8_dyn(const void* base, long long elem_off, int dt, float (&v)[8]) {
  if (dt == 1) ld8(reinterpret_cast<const float*>(base) + elem_off, v);
  else if (dt == 2) ld8(reinterpret_cast<const __half*>(base) + elem_off, v);
  else ld8(reinterpret_cast<const bf16*>(base) + elem_off, v);
}
constexpr float BN_EPS_DEFAULT = 1e-5f;

// ================================================================================================
// direct convolution (forward and, with flipped/transposed packed weights, data gradient)
// ================================================================================================
// Source: up to two channels-last tensors concatenated along C (torch.cat([x2, x1], 1), unet.py:67) or one
// fp32 single-channel image.  Weights: fp32 [taps][CinP][CoutP] (CinP, CoutP multiples of 16, zero padded).
// CTA = 16x16 pixels x 16 output channels, 128 threads, each thread 2 pixels (rows py, py+8) x 16 channels.
template <int KS>
__global__ void __launch_bounds__(128) conv_direct_kernel(
    const void* __restrict__ src0, int C0, const void* __restrict__ src1, int C1, int src_f32,
    const float* __restrict__ wpk, const float* __restrict__ bias, void* __restrict__ out, int out_mode,
    int N, int H, int W, int CinP, int CoutP, int CoutStore, int tiles_x, int tiles_y) {
  constexpr int PAD = KS / 2, HT = 16 + 2 * PAD, TAPS = KS * KS;
  __shared__ float s_in[16][HT][HT + 1];
  __shared__ __align__(16) float s_w[TAPS][16][16];
  const int tile = blockIdx.x;
  const int n = tile / (tiles_x * tiles_y);
  const int tr = tile - n * tiles_x * tiles_y;
  const int y0 = (tr / tiles_x) * 16, x0 = (tr % tiles_x) * 16;
  const int cob = blockIdx.y * 16;
  const int px = threadIdx.x & 15, py = threadIdx.x >> 4;
  float acc[2][16];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < 16; ++c) acc[r][c] = 0.f;
  const int Cin = C0 + C1;
  for (int c0 = 0; c0 < CinP; c0 += 16) {
    __syncthreads();
    // ---- input halo tile -> smem (fp32, channel-planar) ----
    for (int i = threadIdx.x; i < HT * HT * 2; i += 128) {
      const int half = i & 1, p = i >> 1;
      const int hy = p / HT, hx = p - hy * HT;
      const int gy = y0 + hy - PAD, gx = x0 + hx - PAD;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        const long long pix = ((long long)n * H + gy) * W + gx;
        const int c = c0 + half * 8;
        if (src_f32 == 1 && (C0 % 8) != 0) {          // single-channel image
          if (c < Cin) {
            const float* s = reinterpret_cast<const float*>(src0) + pix * C0 + c;
            for (int j = 0; j < 8 && c + j < Cin; ++j) v[j] = s[j];
          }
        } else if (c < C0) {
          ld8_dyn(src0, pix * C0 + c, src_f32, v);
        } else if (c < Cin) {
          ld8_dyn(src1, pix * C1 + (c - C0), src_f32, v);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s_in[half * 8 + j][hy][hx] = v[j];
    }
    // ---- weights chunk -> smem ----
    for (int i = threadIdx.x; i < TAPS * 16 * 16; i += 128) {
      const int co = i & 15, ci = (i >> 4) & 15, t = i >> 8;
      s_w[t][ci][co] = wpk[((size_t)t * CinP + c0 + ci) * CoutP + cob + co];
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < 16; ++ci) {
#pragma unroll
      for (int t = 0; t < TAPS; ++t) {
        const int dy = t / KS, dx = t % KS;
        const float a0 = s_in[ci][py + dy][px + dx];
        const float a1 = s_in[ci][py + 8 + dy][px + dx];
        const float4* wv = reinterpret_cast<const float4*>(&s_w[t][ci][0]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 w = wv[q];
          acc[0][q * 4 + 0] = fmaf(a0, w.x, acc[0][q * 4 + 0]); acc[1][q * 4 + 0] = fmaf(a1, w.x, acc[1][q * 4 + 0]);
          acc[0][q * 4 + 1] = fmaf(a0, w.y, acc[0][q * 4 + 1]); acc[1][q * 4 + 1] = fmaf(a1, w.y, acc[1][q * 4 + 1]);
          acc[0][q * 4 + 2] = fmaf(a0, w.z, acc[0][q * 4 + 2]); acc[1][q * 4 + 2] = fmaf(a1, w.z, acc[1][q * 4 + 2]);
          acc[0][q * 4 + 3] = fmaf(a0, w.w, acc[0][q * 4 + 3]); acc[1][q * 4 + 3] = fmaf(a1, w.w, acc[1][q * 4 + 3]);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int gy = y0 + py + r * 8, gx = x0 + px;
    if (gy >= H || gx >= W) continue;
    float v[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) v[c] = acc[r][c] + (bias ? bias[cob + c] : 0.f);
    if (out_mode == 0 || out_mode == 3) {   // 16-bit NHWC: 0 = bf16, 3 = fp16
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out) + (((long long)n * H + gy) * W + gx) * CoutStore + cob;
      float lo[8], hi[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) { lo[c] = v[c]; hi[c] = v[8 + c]; }
      if (cob + 8 <= CoutStore) reinterpret_cast<uint4*>(o)[0] = pack8_dt(lo, out_mode == 3 ? 2 : 0);
      if (cob + 16 <= CoutStore) reinterpret_cast<uint4*>(o)[1] = pack8_dt(hi, out_mode == 3 ? 2 : 0);
    } else if (out_mode == 2) {  // fp32 NHWC with CoutStore channels (parity mode activations)
      float* o = reinterpret_cast<float*>(out) + (((long long)n * H + gy) * W + gx) * CoutStore + cob;
#pragma unroll
      for (int c = 0; c < 16; ++c)
        if (cob + c < CoutStore) o[c] = v[c];
    } else {  // fp32 NCHW with CoutStore real channels
      float* o = reinterpret_cast<float*>(out);
#pragma unroll
      for (int c = 0; c < 16; ++c)
        if (cob + c < CoutStore) o[(((long long)n * CoutStore + cob + c) * H + gy) * W + gx] = v[c];
    }
  }
}


// ================================================================================================
// first layer (Cin = 1, unet.py:81 in_conv): x fp32 [N,H,W] -> y bf16 [N,H,W,16]; HBM-bound (36 B/pixel)
// ================================================================================================
// Two horizontally adjacent pixels x eight channels per thread: the 3 x 4 input window is loaded once, every tap's weights are read
// from shared memory as 16-byte vectors and used for both pixels (the one-pixel form issued 144 scalar shared-memory loads per pixel and
// was bound by the LDS pipe: 85 us for 64 x 256 x 256 against the 23 us its 150 MB of traffic need).  Optional fused BatchNorm
// statistics: per-CTA rows {sum, sum of squares} of the values as stored, finalised by bn_finalize_kernel like conv_tc2's.
__device__ __forceinline__ float4 lds128_volatile(const float* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"((uint32_t)__cvta_generic_to_shared(p)));
  return v;
}

template <typename T>
__global__ void __launch_bounds__(TPB, 4) conv_first_kernel(const float* __restrict__ x, const float* __restrict__ w /*[16][9]*/,
                                                         const float* __restrict__ bias, T* __restrict__ y,
                                                         int N, int H, int W, float* __restrict__ stat_partials) {
  __shared__ __align__(16) float s_w[9][16];
  __shared__ __align__(16) float s_b[16];
  __shared__ float s_stat[TPB / 32][32];
  if (threadIdx.x < 144) s_w[threadIdx.x % 9][threadIdx.x / 9] = w[threadIdx.x];
  if (threadIdx.x < 16) s_b[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  // thread = (pixel pair, channel half): lanes 2k / 2k+1 own channels 0-7 / 8-15 of the same two pixels, so a pair of lanes
  // stores one full 32-byte pixel and the input window is a broadcast load
  const int half = threadIdx.x & 1;
  const int PW = (W + 1) >> 1;                                   // pixel pairs per row
  const int total = N * H * PW;                                    // 32-bit indexing (64-bit div / mod dominated the loop)
  float ssum[8], ssq[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) ssum[c] = ssq[c] = 0.f;
  const float4 bl = reinterpret_cast<const float4*>(s_b)[half * 2], bh = reinterpret_cast<const float4*>(s_b)[half * 2 + 1];
  for (int i = (blockIdx.x * TPB + threadIdx.x) >> 1; i < total; i += (gridDim.x * TPB) >> 1) {
    const int xp = i % PW, q_ = i / PW, yy = q_ % H;
    const long long n = q_ / H;
    const int xx = xp * 2;
    const bool two = xx + 1 < W;
    const float* img = x + n * (long long)H * W;
    float v[3][4];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int gy = yy + a - 1;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int gx = xx + b - 1;
        v[a][b] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? img[(long long)gy * W + gx] : 0.f;
      }
    }
    float o0[8] = {bl.x, bl.y, bl.z, bl.w, bh.x, bh.y, bh.z, bh.w}, o1[8] = {bl.x, bl.y, bl.z, bl.w, bh.x, bh.y, bh.z, bh.w};
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float a0 = v[t / 3][t % 3], a1 = v[t / 3][t % 3 + 1];
      // volatile shared-memory loads: as plain loads the compiler hoists all 72 loop-invariant weights out of the pixel loop
      // and spills them (272 bytes of stack per thread, 141 us)
      const float4 wl = lds128_volatile(&s_w[t][half * 8]), wh = lds128_volatile(&s_w[t][half * 8 + 4]);
      o0[0] = fmaf(a0, wl.x, o0[0]); o0[1] = fmaf(a0, wl.y, o0[1]); o0[2] = fmaf(a0, wl.z, o0[2]); o0[3] = fmaf(a0, wl.w, o0[3]);
      o0[4] = fmaf(a0, wh.x, o0[4]); o0[5] = fmaf(a0, wh.y, o0[5]); o0[6] = fmaf(a0, wh.z, o0[6]); o0[7] = fmaf(a0, wh.w, o0[7]);
      o1[0] = fmaf(a1, wl.x, o1[0]); o1[1] = fmaf(a1, wl.y, o1[1]); o1[2] = fmaf(a1, wl.z, o1[2]); o1[3] = fmaf(a1, wl.w, o1[3]);
      o1[4] = fmaf(a1, wh.x, o1[4]); o1[5] = fmaf(a1, wh.y, o1[5]); o1[6] = fmaf(a1, wh.z, o1[6]); o1[7] = fmaf(a1, wh.w, o1[7]);
    }
    const long long pix = (n * H + yy) * (long long)W + xx;
    st8(y + pix * 16 + half * 8, o0);
    if (two) st8(y + (pix + 1) * 16 + half * 8, o1);
    if (stat_partials) {
      round8<T>(o0);
      round8<T>(o1);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        ssum[c] += o0[c];
        ssq[c] = fmaf(o0[c], o0[c], ssq[c]);
        if (two) { ssum[c] += o1[c]; ssq[c] = fmaf(o1[c], o1[c], ssq[c]); }
      }
    }
  }
  if (stat_partials) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      float a = ssum[c], b = ssq[c];
#pragma unroll
      for (int o = 16; o > 1; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }   // lanes of equal parity
      if (lane < 2) { s_stat[warp][lane * 8 + c] = a; s_stat[warp][16 + lane * 8 + c] = b; }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      float a = 0.f;
#pragma unroll
      for (int wv = 0; wv < TPB / 32; ++wv) a += s_stat[wv][threadIdx.x];
      stat_partials[(size_t)blockIdx.x * 32 + threadIdx.x] = a;      // row layout [2][16], like the conv_tc2 epilogue rows
    }
  }
}

// dW[co][t] += sum_p dY[p][co] * x[p + tap_t]: every thread walks pixels with an 8x9 register tile (blockIdx.y picks
// the channel half; 72 FMAs per 10 loads), then warp-shuffle + one atomicAdd per warp and entry.
template <typename T>
__global__ void __launch_bounds__(256, 2) wgrad_first_kernel(const float* __restrict__ x, const T* __restrict__ dy,
                                                             float* __restrict__ dw /*[16][9]*/, int N, int H, int W) {
  float acc[8][9];
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[c][t] = 0.f;
  const int half = blockIdx.y;
  const long long total = (long long)N * H * W;
#pragma unroll 2
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int xx = (int)(i % W), yy = (int)((i / W) % H);
    const float* base = x + (i - (long long)yy * W - xx);
    float v[9], g[8];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int gy = yy + t / 3 - 1, gx = xx + t % 3 - 1;
      v[t] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? base[(long long)gy * W + gx] : 0.f;
    }
    ld8(dy + i * 16 + half * 8, g);
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int t = 0; t < 9; ++t) acc[c][t] = fmaf(g[c], v[t], acc[c][t]);
  }
  // block reduction (fixed order inside the block), then ONE atomic per value and block: 72 same-address atomics per warp
  // of 1184 blocks used to serialise in L2 for ~0.25 ms.
  __shared__ float s_red[8][72];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const float r = warp_sum(acc[c][t]);
      if (lane == 0) s_red[warp][c * 9 + t] = r;
    }
  __syncthreads();
  if (threadIdx.x < 72) {
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) r += s_red[w][threadIdx.x];
    atomicAdd(dw + half * 72 + threadIdx.x, r);
  }
}

// ================================================================================================
// direct weight gradient:  dW[co][ci][dy][dx] = sum_{n,y,x} dY[n,y,x,co] * X[n,y+dy-P,x+dx-P,ci]
// CTA = 16 co x 16 ci x all taps, 256 threads (co = t%16, ci = t/16); loops over 8x16 pixel tiles of its split,
// accumulates in registers, then atomically adds into the (pre-zeroed) fp32 torch-layout gradient.
// ================================================================================================
template <int KS>
__global__ void __launch_bounds__(256) wgrad_direct_kernel(
    const void* __restrict__ src0, int C0, const void* __restrict__ src1, int C1, int src_f32,
    const void* __restrict__ dy, int dy_f32, int CoutP, float* __restrict__ dw, float* __restrict__ dbias,
    int N, int H, int W, int CoutReal, int tiles_x, int tiles_y) {
  constexpr int PAD = KS / 2, TH = 8, TW = 16, HH = TH + 2 * PAD, HWD = TW + 2 * PAD, TAPS = KS * KS;
  __shared__ float s_g[TH * TW][16];
  __shared__ float s_x[HH * HWD][17];
  const int Cin = C0 + C1;
  const int ci_blocks = (Cin + 15) / 16;
  const int cob = (blockIdx.x / ci_blocks) * 16, cib = (blockIdx.x % ci_blocks) * 16;
  const int co = threadIdx.x & 15, ci = threadIdx.x >> 4;
  float acc[TAPS];
#pragma unroll
  for (int t = 0; t < TAPS; ++t) acc[t] = 0.f;
  float bsum = 0.f;
  const int ntiles = N * tiles_x * tiles_y;
  for (int tile = blockIdx.y; tile < ntiles; tile += gridDim.y) {
    const int n = tile / (tiles_x * tiles_y);
    const int tr = tile - n * tiles_x * tiles_y;
    const int y0 = (tr / tiles_x) * TH, x0 = (tr % tiles_x) * TW;
    __syncthreads();
    {  // dY tile: 128 px x 16 co, one 16-byte vector per thread
      const int p = threadIdx.x >> 1, half = threadIdx.x & 1;
      const int gy = y0 + p / TW, gx = x0 + p % TW;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
      if (gy < H && gx < W) ld8_dyn(dy, (((long long)n * H + gy) * W + gx) * CoutP + cob + half * 8, dy_f32, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) s_g[p][half * 8 + j] = v[j];
    }
    for (int i = threadIdx.x; i < HH * HWD * 2; i += 256) {
      const int half = i & 1, p = i >> 1;
      const int hy = p / HWD, hx = p - hy * HWD;
      const int gy = y0 + hy - PAD, gx = x0 + hx - PAD;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        const long long pix = ((long long)n * H + gy) * W + gx;
        const int c = cib + half * 8;
        if (src_f32 == 1 && (C0 % 8) != 0) {          // single-channel image
          if (c < Cin) {
            const float* s = reinterpret_cast<const float*>(src0) + pix * C0 + c;
            for (int j = 0; j < 8 && c + j < Cin; ++j) v[j] = s[j];
          }
        } else if (c < C0) {
          ld8_dyn(src0, pix * C0 + c, src_f32, v);
        } else if (c < Cin) {
          ld8_dyn(src1, pix * C1 + (c - C0), src_f32, v);
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) s_x[p][half * 8 + j] = v[j];
    }
    __syncthreads();
#pragma unroll 4
    for (int p = 0; p < TH * TW; ++p) {
      const float g = s_g[p][co];
      const int py = p / TW, pxx = p % TW;
      bsum += g;
#pragma unroll
      for (int t = 0; t < TAPS; ++t) acc[t] = fmaf(g, s_x[(py + t / KS) * HWD + pxx + t % KS][ci], acc[t]);
    }
  }
  if (cob + co < CoutReal && cib + ci < Cin) {
#pragma unroll
    for (int t = 0; t < TAPS; ++t) atomicAdd(dw + ((size_t)(cob + co) * Cin + cib + ci) * TAPS + t, acc[t]);
  }
  if (dbias != nullptr && cib == 0 && ci == 0 && cob + co < CoutReal) atomicAdd(dbias + cob + co, bsum);
}


// Fixed-order sum of per-block partials [nblocks][2][C] for all channels with all 256 threads:
// thread t handles channel t % CP (CP = C rounded up to a power of two <= 256) and block subset t / CP.
// Results (double) land in s_fin[2][C].
__device__ __forceinline__ void bn_finalize_partials(const float* partials, int nblocks, int C, double* s_fin /*[2*C]*/,
                                                     double* s_part /*[TPB*2]*/) {
  for (int cbase = 0; cbase < C; cbase += TPB) {
    const int cw = min(C - cbase, TPB);
    int parts = TPB / cw;                       // threads per channel
    const int c = cbase + (int)(threadIdx.x % cw);
    const int part = threadIdx.x / cw;
    double a = 0.0, b = 0.0;
    if (part < parts) {
      int bl = part;
      for (; bl + 7 * parts < nblocks; bl += 8 * parts) {   // 16 independent loads in flight, fixed summation order
        float va[8], vb[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          va[u] = __ldcg(&partials[((size_t)(bl + u * parts) * 2 + 0) * C + c]);
          vb[u] = __ldcg(&partials[((size_t)(bl + u * parts) * 2 + 1) * C + c]);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) { a += (double)va[u]; b += (double)vb[u]; }
      }
      for (; bl < nblocks; bl += parts) {
        a += (double)__ldcg(&partials[((size_t)bl * 2 + 0) * C + c]);
        b += (double)__ldcg(&partials[((size_t)bl * 2 + 1) * C + c]);
      }
    }
    s_part[threadIdx.x * 2 + 0] = a;
    s_part[threadIdx.x * 2 + 1] = b;
    __syncthreads();
    if (threadIdx.x < cw) {
      double x = 0.0, y = 0.0;
      for (int q = 0; q < parts; ++q) { x += s_part[(q * cw + threadIdx.x) * 2]; y += s_part[(q * cw + threadIdx.x) * 2 + 1]; }
      s_fin[c] = x;
      s_fin[C + c] = y;
    }
    __syncthreads();
  }
}

// ================================================================================================
// BatchNorm (training): per-channel statistics over N*H*W of a channels-last bf16 tensor
// ================================================================================================
// thread (row r = t / cg, group g = t % cg) owns 8 channels; rows stride over pixels.
// Partials [block][2][C]; the last block finalises in fixed order (deterministic):
//   save[0:C] = mean, save[C:2C] = invstd; ss[0:C] = gamma*invstd, ss[C:2C] = beta - mean*scale;
//   running_mean/var updated with momentum (unbiased variance), num_batches_tracked += 1.
template <typename T>
__global__ void __launch_bounds__(TPB) bn_stats_kernel(
    const T* __restrict__ y, long long P, int C, const float* __restrict__ gamma,
    const float* __restrict__ beta, float* running_mean, float* running_var, long long* nbt, float momentum,
    float eps, float* __restrict__ save, float* __restrict__ ss, float* partials, unsigned* ticket, float* raw_sums) {
  extern __shared__ float s_red[];  // [TPB][16]
  const int cg = C >> 3, rows = TPB / cg;
  const int g = threadIdx.x % cg, r = threadIdx.x / cg;
  float sum[8], sq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sum[j] = sq[j] = 0.f;
  if (r < rows) {
    for (long long p = (long long)blockIdx.x * rows + r; p < P; p += (long long)gridDim.x * rows) {
      float v[8];
      ld8(y + p * C + g * 8, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) { sum[j] += v[j]; sq[j] = fmaf(v[j], v[j], sq[j]); }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { s_red[threadIdx.x * 16 + j] = sum[j]; s_red[threadIdx.x * 16 + 8 + j] = sq[j]; }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += TPB) {
    const int gg = c >> 3, j = c & 7;
    float a = 0.f, b = 0.f;
    for (int rr = 0; rr < rows; ++rr) { a += s_red[(rr * cg + gg) * 16 + j]; b += s_red[(rr * cg + gg) * 16 + 8 + j]; }
    partials[((size_t)blockIdx.x * 2 + 0) * C + c] = a;
    partials[((size_t)blockIdx.x * 2 + 1) * C + c] = b;
  }
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  __shared__ double s_fin[2 * 256];
  __shared__ double s_part[TPB * 2];
  bn_finalize_partials(partials, gridDim.x, C, s_fin, s_part);
  if (raw_sums != nullptr) {       // synchronised BatchNorm: hand out {sum, sum of squares}; the caller all-reduces and finalises
    for (int c = threadIdx.x; c < 2 * C; c += TPB) raw_sums[c] = (float)s_fin[c];
    if (threadIdx.x == 0) *ticket = 0u;
    return;
  }
  for (int c = threadIdx.x; c < C; c += TPB) {
    const double a = s_fin[c], b = s_fin[C + c];
    const double mean = a / (double)P;
    double var = b / (double)P - mean * mean;
    if (var < 0.0) var = 0.0;
    const float invstd = (float)(1.0 / sqrt(var + (double)eps));
    save[c] = (float)mean;
    save[C + c] = invstd;
    const float sc = gamma[c] * invstd;
    ss[c] = sc;
    ss[C + c] = beta[c] - (float)mean * sc;
    if (running_mean) {
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
      const double unb = (P > 1) ? var * (double)P / (double)(P - 1) : var;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
    }
  }
  if (threadIdx.x == 0) {
    if (nbt) *nbt += 1;
    *ticket = 0u;
  }
}

// finalize-only variant: partial rows [nrows][2][C] produced by the convolution epilogue (conv_tc.cu)
// One block per 16 channels, 16 threads per channel walking the partial rows (fixed order -> deterministic); a single block
// for all channels took 12 us per layer on the forward critical path.
__global__ void __launch_bounds__(TPB) bn_finalize_kernel(const float* __restrict__ partials, int nrows, long long P, int C,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          float* running_mean, float* running_var, long long* nbt, float momentum,
                                                          float eps, float* __restrict__ save, float* __restrict__ ss) {
  constexpr int CB = 16, PARTS = TPB / CB;
  __shared__ double s_part[TPB * 2];
  const int cl = threadIdx.x % CB, part = threadIdx.x / CB;
  const int c = blockIdx.x * CB + cl;
  double a = 0.0, b = 0.0;
  if (c < C) {
    int bl = part;
    for (; bl + 7 * PARTS < nrows; bl += 8 * PARTS) {
      float va[8], vb[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        va[u] = __ldcg(&partials[((size_t)(bl + u * PARTS) * 2 + 0) * C + c]);
        vb[u] = __ldcg(&partials[((size_t)(bl + u * PARTS) * 2 + 1) * C + c]);
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) { a += (double)va[u]; b += (double)vb[u]; }
    }
    for (; bl < nrows; bl += PARTS) {
      a += (double)__ldcg(&partials[((size_t)bl * 2 + 0) * C + c]);
      b += (double)__ldcg(&partials[((size_t)bl * 2 + 1) * C + c]);
    }
  }
  s_part[threadIdx.x * 2 + 0] = a;
  s_part[threadIdx.x * 2 + 1] = b;
  __syncthreads();
  if (threadIdx.x < CB && c < C) {
    double x = 0.0, y = 0.0;
    for (int q = 0; q < PARTS; ++q) { x += s_part[(q * CB + cl) * 2]; y += s_part[(q * CB + cl) * 2 + 1]; }
    const double mean = x / (double)P;
    double var = y / (double)P - mean * mean;
    if (var < 0.0) var = 0.0;
    const float invstd = (float)(1.0 / sqrt(var + (double)eps));
    save[c] = (float)mean;
    save[C + c] = invstd;
    const float sc = gamma[c] * invstd;
    ss[c] = sc;
    ss[C + c] = beta[c] - (float)mean * sc;
    if (running_mean) {
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
      const double unb = (P > 1) ? var * (double)P / (double)(P - 1) : var;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && nbt) *nbt += 1;
}

// ---- per-sample BatchNorm (training statistics of every image on its own) ---------------------------------------------
// For the Scribble2Label ensemble refresh (train_s2l.py:221-228): B batch-1 training forwards in one batched pass.  Pass 1: grid
// (blocks per image, N), the layout of bn_stats_kernel restricted to one image's HW pixels, partials [N][nblk][2][C].  Pass 2:
// one thread per channel walks the images in order (fixed-order double sums as bn_finalize_kernel), writes {mean, invstd} and
// {scale, shift} per image, and applies the N running-statistics updates in slice order (unbiased variance with n = HW).
template <typename T>
__global__ void __launch_bounds__(TPB) bn_stats_ps_kernel(const T* __restrict__ y, int HW, int C, float* __restrict__ partials) {
  extern __shared__ float s_red[];  // [TPB][16]
  const int cg = C >> 3, rows = TPB / cg;
  const int g = threadIdx.x % cg, r = threadIdx.x / cg;
  const T* yn = y + (size_t)blockIdx.y * HW * C;
  float sum[8], sq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sum[j] = sq[j] = 0.f;
  for (int p = blockIdx.x * rows + r; p < HW; p += gridDim.x * rows) {
    float v[8];
    ld8(yn + (size_t)p * C + g * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) { sum[j] += v[j]; sq[j] = fmaf(v[j], v[j], sq[j]); }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { s_red[threadIdx.x * 16 + j] = sum[j]; s_red[threadIdx.x * 16 + 8 + j] = sq[j]; }
  __syncthreads();
  float* part = partials + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2 * C;
  for (int c = threadIdx.x; c < C; c += TPB) {
    const int gg = c >> 3, j = c & 7;
    float a = 0.f, b = 0.f;
    for (int rr = 0; rr < rows; ++rr) { a += s_red[(rr * cg + gg) * 16 + j]; b += s_red[(rr * cg + gg) * 16 + 8 + j]; }
    part[c] = a;
    part[C + c] = b;
  }
}

__global__ void __launch_bounds__(TPB) bn_finalize_ps_kernel(const float* __restrict__ partials, int nblk, int N, int HW, int C,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             float* running_mean, float* running_var, long long* nbt, float momentum,
                                                             float eps, float* __restrict__ save, float* __restrict__ ss) {
  const int c = blockIdx.x * TPB + threadIdx.x;
  if (c < C) {
    float rm = running_mean ? running_mean[c] : 0.f, rv = running_var ? running_var[c] : 0.f;
    for (int n = 0; n < N; ++n) {
      const float* part = partials + (size_t)n * nblk * 2 * C;
      double a = 0.0, b = 0.0;
      for (int bl = 0; bl < nblk; ++bl) { a += (double)part[(size_t)bl * 2 * C + c]; b += (double)part[(size_t)bl * 2 * C + C + c]; }
      const double mean = a / (double)HW;
      double var = b / (double)HW - mean * mean;
      if (var < 0.0) var = 0.0;
      const float invstd = (float)(1.0 / sqrt(var + (double)eps));
      const float sc = gamma[c] * invstd;
      save[(size_t)n * 2 * C + c] = (float)mean;
      save[(size_t)n * 2 * C + C + c] = invstd;
      ss[(size_t)n * 2 * C + c] = sc;
      ss[(size_t)n * 2 * C + C + c] = beta[c] - (float)mean * sc;
      const double unb = (HW > 1) ? var * (double)HW / (double)(HW - 1) : var;
      rm = (1.f - momentum) * rm + momentum * (float)mean;
      rv = (1.f - momentum) * rv + momentum * (float)unb;
    }
    if (running_mean) { running_mean[c] = rm; running_var[c] = rv; }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && nbt) *nbt += N;
}

// eval mode: scale/shift from running statistics
__global__ void bn_eval_prepare_kernel(const float* gamma, const float* beta, const float* rm, const float* rv,
                                       float eps, int C, float* ss) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    const float sc = gamma[c] * rsqrtf(rv[c] + eps);
    ss[c] = sc;
    ss[C + c] = beta[c] - rm[c] * sc;
  }
}

// ---- shared per-thread machinery of the BN forward/backward elementwise kernels ---------------------------------
// Thread t owns channel group g = t % (C/8) for its whole life (per-channel constants live in registers) and walks
// pixels p = block*rows + t/(C/8), p += grid*rows: a warp reads 512 contiguous bytes per tensor and iteration.
struct DropCtx {
  const uint8_t* mask;      // optional explicit keep mask (NHWC uint8)
  unsigned long long seed;
  uint32_t thresh;          // drop when r16 < thresh
  float inv_keep;
  bool on;
};

__device__ __forceinline__ uint32_t keep_bits8(const DropCtx& d, long long eidx, uint32_t vec) {
  // bit j set -> element j is kept
  if (!d.on) return 0xffu;
  uint32_t bits = 0;
  if (d.mask) {
    const uint2 mk = *reinterpret_cast<const uint2*>(d.mask + eidx);
#pragma unroll
    for (int j = 0; j < 8; ++j) bits |= ((((j < 4 ? (mk.x >> (8 * j)) : (mk.y >> (8 * (j - 4)))) & 0xffu) != 0) ? 1u : 0u) << j;
  } else {
    uint32_t r[8];
    wsl_rand8x16(d.seed, vec, r);
#pragma unroll
    for (int j = 0; j < 8; ++j) bits |= (r[j] >= d.thresh ? 1u : 0u) << j;
  }
  return bits;
}

__device__ __forceinline__ DropCtx make_drop(float p, const uint8_t* mask, unsigned long long seed, const unsigned long long* seed_ptr) {
  DropCtx d;
  d.on = p > 0.f;
  d.mask = mask;
  d.seed = seed + (seed_ptr ? *seed_ptr : 0ULL);
  d.thresh = (uint32_t)(p * 65536.0f);
  d.inv_keep = d.on ? 1.f / (1.f - p) : 1.f;
  return d;
}

// Statistics finalisation folded into the consumer (narrow layers, C <= 32): every block re-derives {scale, shift} from the convolution
// epilogue's partial rows [nrows][2][C] (<= 296 x 64 floats, L2-resident) instead of waiting for a separate bn_finalize launch on the
// forward critical path; block 0 also publishes save / ss / running statistics exactly like bn_finalize_kernel (same double sums, same
// values up to the last bit of the double sums).
struct BnFin {
  const float* partials;   // null -> scale / shift are read from ss
  int nrows;
  long long P;
  const float* gamma; const float* beta;
  float* running_mean; float* running_var; long long* nbt;
  float momentum, eps;
  float* save; float* ss_out;
};

// A = dropout(leaky_relu(y*scale + shift)); optional fused 2x2 max-pool of A (DownBlock, unet.py:38).
// PER_SAMPLE: ss holds {scale, shift} per image, [N][2][C] (per-sample BatchNorm, bn_stats_ps_kernel); reloaded when the pixel's image changes.
template <typename T, bool PER_SAMPLE = false>
__global__ void __launch_bounds__(TPB) bn_act_fwd_kernel(
    const T* __restrict__ y, const float* __restrict__ ss, int N, int H, int W, int C, float slope,
    float drop_p, const uint8_t* __restrict__ mask, unsigned long long seed, const unsigned long long* seed_ptr,
    T* __restrict__ act, T* __restrict__ pooled, uint8_t* __restrict__ pool_idx, const BnFin fin) {
  const int cg = C >> 3, rows = TPB / cg;
  const int g = threadIdx.x % cg, r = threadIdx.x / cg, c0 = g * 8;
  const DropCtx dc = make_drop(drop_p, mask, seed, seed_ptr);
  float sc[8], sh[8];
  if (fin.partials != nullptr) {
    __shared__ double s_sum[64];          // [2][C], C <= 32
    __shared__ float s_ss[64];
    // TPB / (2C) threads per statistic walk interleaved row subsets, then a fixed-order combine (as bn_finalize_kernel: 16 parts)
    __shared__ double s_part[TPB];
    const int nstat = 2 * C, parts = TPB / nstat;           // 8 (C = 16) or 4 (C = 32) threads per statistic
    const int st = threadIdx.x % nstat, part = threadIdx.x / nstat;
    double a = 0.0;
    if (part < parts) {
      const int which = st / C, c = st % C;
      for (int bl = part; bl < fin.nrows; bl += parts) a += (double)__ldcg(&fin.partials[((size_t)bl * 2 + which) * C + c]);
    }
    s_part[threadIdx.x] = a;
    __syncthreads();
    if (threadIdx.x < nstat) {
      double t = 0.0;
      for (int q = 0; q < parts; ++q) t += s_part[q * nstat + threadIdx.x];
      s_sum[threadIdx.x] = t;
    }
    __syncthreads();
    if (threadIdx.x < C) {
      const int c = threadIdx.x;
      const double mean = s_sum[c] / (double)fin.P;
      double var = s_sum[C + c] / (double)fin.P - mean * mean;
      if (var < 0.0) var = 0.0;
      const float invstd = (float)(1.0 / sqrt(var + (double)fin.eps));
      const float scl = fin.gamma[c] * invstd, shf = fin.beta[c] - (float)mean * scl;
      s_ss[c] = scl;
      s_ss[C + c] = shf;
      if (blockIdx.x == 0) {
        fin.save[c] = (float)mean;
        fin.save[C + c] = invstd;
        fin.ss_out[c] = scl;
        fin.ss_out[C + c] = shf;
        if (fin.running_mean) {
          fin.running_mean[c] = (1.f - fin.momentum) * fin.running_mean[c] + fin.momentum * (float)mean;
          const double unb = (fin.P > 1) ? var * (double)fin.P / (double)(fin.P - 1) : var;
          fin.running_var[c] = (1.f - fin.momentum) * fin.running_var[c] + fin.momentum * (float)unb;
        }
        if (c == 0 && fin.nbt) *fin.nbt += 1;
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = s_ss[c0 + j]; sh[j] = s_ss[C + c0 + j]; }
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = ss[c0 + j]; sh[j] = ss[C + c0 + j]; }
  }
  // loads are issued for all pixels of an iteration before the first use (the dropout branch would otherwise serialise them)
  int cur_n = 0;
  auto act8 = [&](int p, const float (&v)[8], float (&o)[8]) {
    if constexpr (PER_SAMPLE) {
      const int n = p / (H * W);
      if (n != cur_n) {
        cur_n = n;
#pragma unroll
        for (int j = 0; j < 8; ++j) { sc[j] = ss[(size_t)n * 2 * C + c0 + j]; sh[j] = ss[(size_t)n * 2 * C + C + c0 + j]; }
      }
    }
    const uint32_t kb = keep_bits8(dc, (long long)p * C + c0, (uint32_t)p * cg + g);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float z = fmaf(v[j], sc[j], sh[j]);
      z = z > 0.f ? z : z * slope;
      o[j] = ((kb >> j) & 1u) ? z * dc.inv_keep : 0.f;
    }
  };
  if (pooled == nullptr) {
    const int P = N * H * W, stride = gridDim.x * rows;
    int p = blockIdx.x * rows + r;
    for (; p + stride < P; p += 2 * stride) {
      float v0[8], v1[8], o0[8], o1[8];
      ld8(y + (long long)p * C + c0, v0);
      ld8(y + (long long)(p + stride) * C + c0, v1);
      act8(p, v0, o0);
      act8(p + stride, v1, o1);
      st8(act + (long long)p * C + c0, o0);
      st8(act + (long long)(p + stride) * C + c0, o1);
    }
    if (p < P) {
      float v[8], o[8];
      ld8(y + (long long)p * C + c0, v);
      act8(p, v, o);
      st8(act + (long long)p * C + c0, o);
    }
  } else {
    const int Hp = H >> 1, Wp = W >> 1, Q = N * Hp * Wp;
    for (int q = blockIdx.x * rows + r; q < Q; q += gridDim.x * rows) {
      const int xp = q % Wp, t = q / Wp, yp = t % Hp, n = t / Hp;
      float best[8], v[4][8];
      int arg[8];
#pragma unroll
      for (int k = 0; k < 4; ++k) ld8(y + (long long)((n * H + yp * 2 + (k >> 1)) * W + xp * 2 + (k & 1)) * C + c0, v[k]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int p = (n * H + yp * 2 + (k >> 1)) * W + xp * 2 + (k & 1);
        float o[8];
        act8(p, v[k], o);
        st8(act + (long long)p * C + c0, o);
        round8<T>(o);     // pool over the activations exactly as stored
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (k == 0 || o[j] > best[j]) { best[j] = o[j]; arg[j] = k; }  // first maximum wins (torch)
      }
      st8(pooled + (long long)q * C + c0, best);
      uint2 ai;
      ai.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
      ai.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | (arg[7] << 24);
      *reinterpret_cast<uint2*>(pool_idx + (long long)q * C + c0) = ai;
    }
  }
}

// ---- BatchNorm backward -------------------------------------------------------------------------
// dA(p,c) = g0[p,c] + cs1[n,c]*g1[p,c] + (pool_idx[q,c]==k ? gp[q,c] : 0)         (any of the three may be absent)
// dz      = dA * dropout_factor * leaky'(z),   z = y*scale+shift,  xhat = (y-mean)*invstd
// reduce : sum dz, sum dz*xhat  -> dbeta, dgamma, c1 = sum dz / P, c2 = sum dz*xhat / P
// apply  : dY = scale * (dz - c1 - xhat*c2)
template <typename T>
struct BnBwdArgs {
  const T* y;
  const float* ss;     // scale, shift
  const float* save;   // mean, invstd
  const T* g0;
  const T* g1;
  const float* cs1;    // [N][C] channel scale for g1 (nullable -> 1)
  const T* gp;
  const uint8_t* pool_idx;
  const uint8_t* mask;
  unsigned long long seed;
  const unsigned long long* seed_ptr;
  float drop_p, slope;
  int N, H, W, C;
};

struct BnBwdThread {
  float sc[8], sh[8];    // z = y*sc + sh (only its sign is needed)
  int c0, g, cg;
  DropCtx dc;
};

template <typename T>
__device__ __forceinline__ BnBwdThread bn_bwd_thread(const BnBwdArgs<T>& a) {
  BnBwdThread t;
  t.cg = a.C >> 3;
  t.g = threadIdx.x % t.cg;
  t.c0 = t.g * 8;
#pragma unroll
  for (int j = 0; j < 8; ++j) { t.sc[j] = a.ss[t.c0 + j]; t.sh[j] = a.ss[a.C + t.c0 + j]; }
  t.dc = make_drop(a.drop_p, a.mask, a.seed, a.seed_ptr);
  return t;
}

// summed incoming gradient g and the raw conv output y of 8 channels of pixel p.
// MODE bit 0: g1 present (channel-scaled by cs1 when given), bit 1: pooled gradient present; g0 is required -> straight-line
// code, so the two-pixel unrolled callers get every load of both pixels in flight before the first use.
// MODE 4: any combination including a missing g0 (uniform runtime branches).
template <int MODE, typename T>
__device__ __forceinline__ void bn_bwd_gather8(const BnBwdArgs<T>& a, const BnBwdThread& t, int p, float (&g)[8], float (&yv)[8]) {
  const long long off = (long long)p * a.C + t.c0;
  ld8(a.y + off, yv);
  if (MODE < 4) {
    ld8(a.g0 + off, g);
    if (MODE != 0) {
      const int x = p % a.W, r = p / a.W, yy = r % a.H, n = r / a.H;
      float v1[8], vp[8];
      float4 s0 = make_float4(1.f, 1.f, 1.f, 1.f), s1 = s0;
      uint2 ai = make_uint2(0u, 0u);
      const long long q = ((long long)(n * (a.H >> 1) + (yy >> 1)) * (a.W >> 1) + (x >> 1)) * a.C + t.c0;
      if (MODE & 1) {
        ld8(a.g1 + off, v1);
        if (a.cs1) {
          s0 = *reinterpret_cast<const float4*>(a.cs1 + (long long)n * a.C + t.c0);
          s1 = *reinterpret_cast<const float4*>(a.cs1 + (long long)n * a.C + t.c0 + 4);
        }
      }
      if (MODE & 2) {
        ai = *reinterpret_cast<const uint2*>(a.pool_idx + q);
        ld8(a.gp + q, vp);
      }
      if (MODE & 1) {
        g[0] = fmaf(v1[0], s0.x, g[0]); g[1] = fmaf(v1[1], s0.y, g[1]); g[2] = fmaf(v1[2], s0.z, g[2]); g[3] = fmaf(v1[3], s0.w, g[3]);
        g[4] = fmaf(v1[4], s1.x, g[4]); g[5] = fmaf(v1[5], s1.y, g[5]); g[6] = fmaf(v1[6], s1.z, g[6]); g[7] = fmaf(v1[7], s1.w, g[7]);
      }
      if (MODE & 2) {
        const int k = ((yy & 1) << 1) | (x & 1);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int aj = (j < 4 ? (ai.x >> (8 * j)) : (ai.y >> (8 * (j - 4)))) & 0xff;
          if (aj == k) g[j] += vp[j];
        }
      }
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) g[j] = 0.f;
  if (a.g0) {
    float v[8];
    ld8(a.g0 + off, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] += v[j];
  }
  if (a.g1 || a.gp) {
    const int x = p % a.W, r = p / a.W, yy = r % a.H, n = r / a.H;
    if (a.g1) {
      float v[8];
      ld8(a.g1 + off, v);
      if (a.cs1) {
        const float4 s0 = *reinterpret_cast<const float4*>(a.cs1 + (long long)n * a.C + t.c0);
        const float4 s1 = *reinterpret_cast<const float4*>(a.cs1 + (long long)n * a.C + t.c0 + 4);
        g[0] = fmaf(v[0], s0.x, g[0]); g[1] = fmaf(v[1], s0.y, g[1]); g[2] = fmaf(v[2], s0.z, g[2]); g[3] = fmaf(v[3], s0.w, g[3]);
        g[4] = fmaf(v[4], s1.x, g[4]); g[5] = fmaf(v[5], s1.y, g[5]); g[6] = fmaf(v[6], s1.z, g[6]); g[7] = fmaf(v[7], s1.w, g[7]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) g[j] += v[j];
      }
    }
    if (a.gp) {
      const long long q = ((long long)(n * (a.H >> 1) + (yy >> 1)) * (a.W >> 1) + (x >> 1)) * a.C + t.c0;
      const int k = ((yy & 1) << 1) | (x & 1);
      const uint2 ai = *reinterpret_cast<const uint2*>(a.pool_idx + q);
      float v[8];
      ld8(a.gp + q, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int aj = (j < 4 ? (ai.x >> (8 * j)) : (ai.y >> (8 * (j - 4)))) & 0xff;
        if (aj == k) g[j] += v[j];
      }
    }
  }
}

// summed incoming gradient g -> dz: dropout mask (regenerated) and LeakyReLU derivative; in place.
// KEEP_Z: yv is overwritten with the normalised value z = y*scale + shift (= gamma*xhat + beta).  The reduction accumulates
// sum(dz*z) instead of sum(dz*y): sum(dz*xhat) = (sum(dz*z) - beta*sum(dz)) / gamma then cancels against beta*sum(dz) (beta is
// O(0.1)) rather than against mean*sum(dz) on the raw convolution output, whose mean can be many standard deviations (measured
// at 4 x 256 x 256: 1e-2 relative error on dgamma / 8e-3 on the following weight gradient in fp32 storage with the raw form).
template <bool KEEP_Z = false, typename T>
__device__ __forceinline__ void bn_bwd_finish8(const BnBwdArgs<T>& a, const BnBwdThread& t, int p, float (&g)[8], float (&yv)[8]) {
  const uint32_t kb = keep_bits8(t.dc, (long long)p * a.C + t.c0, (uint32_t)p * t.cg + t.g);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float z = fmaf(yv[j], t.sc[j], t.sh[j]);
    const float d = g[j] * (z > 0.f ? 1.f : a.slope);
    g[j] = ((kb >> j) & 1u) ? d * t.dc.inv_keep : 0.f;
    if (KEEP_Z) yv[j] = z;
  }
}

template <int MODE, typename T>
__global__ void __launch_bounds__(TPB, (MODE == 0 || MODE == 4) ? 3 : 2) bn_bwd_reduce_kernel(BnBwdArgs<T> a, float* __restrict__ dgamma,
                                                               float* __restrict__ dbeta, float* __restrict__ coef /*[2C]*/,
                                                               float* partials, unsigned* ticket, int accumulate, float* raw_sums = nullptr) {
  extern __shared__ float s_red[];
  const BnBwdThread t = bn_bwd_thread(a);
  const int C = a.C, cg = t.cg, rows = TPB / cg;
  const int P = a.N * a.H * a.W;
  const int r = threadIdx.x / cg;
  // accumulate sum(dz) and sum(dz*z), z = the normalised value the LeakyReLU sign test computes anyway (no extra registers);
  // sum(dz*xhat) = (sum(dz*z) - beta*sum(dz)) / gamma is formed per block below
  float s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s1[j] = s2[j] = 0.f;
  const int stride = gridDim.x * rows;
  int p = blockIdx.x * rows + r;
  for (; p + stride < P; p += 2 * stride) {
    float dz0[8], y0[8], dz1[8], y1[8];
    bn_bwd_gather8<MODE>(a, t, p, dz0, y0);            // all loads of both pixels are issued before the first use
    bn_bwd_gather8<MODE>(a, t, p + stride, dz1, y1);
    bn_bwd_finish8<true>(a, t, p, dz0, y0);
    bn_bwd_finish8<true>(a, t, p + stride, dz1, y1);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] += dz0[j]; s2[j] = fmaf(dz0[j], y0[j], s2[j]); }
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] += dz1[j]; s2[j] = fmaf(dz1[j], y1[j], s2[j]); }
  }
  if (p < P) {
    float dz[8], yv[8];
    bn_bwd_gather8<MODE>(a, t, p, dz, yv);
    bn_bwd_finish8<true>(a, t, p, dz, yv);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s1[j] += dz[j]; s2[j] = fmaf(dz[j], yv[j], s2[j]); }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { s_red[threadIdx.x * 16 + j] = s1[j]; s_red[threadIdx.x * 16 + 8 + j] = s2[j]; }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += TPB) {
    const int gg = c >> 3, j = c & 7;
    float x = 0.f, y = 0.f;
    for (int rr = 0; rr < rows; ++rr) { x += s_red[(rr * cg + gg) * 16 + j]; y += s_red[(rr * cg + gg) * 16 + 8 + j]; }
    partials[((size_t)blockIdx.x * 2 + 0) * C + c] = x;
    // sum(dz * xhat): gamma = scale / invstd, beta = shift + mean * scale (gamma == 0 would make xhat unobservable through z;
    // BatchNorm weights start at 1 and an exact zero is a measure-zero event, the term is then reported as 0)
    const float gam = a.ss[c] / a.save[C + c], bet = fmaf(a.save[c], a.ss[c], a.ss[C + c]);
    partials[((size_t)blockIdx.x * 2 + 1) * C + c] = gam != 0.f ? (y - bet * x) / gam : 0.f;
  }
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  __shared__ double s_fin[2 * 256];
  __shared__ double s_part[TPB * 2];
  bn_finalize_partials(partials, gridDim.x, C, s_fin, s_part);
  for (int c = threadIdx.x; c < C; c += TPB) {
    const double x = s_fin[c], y = s_fin[C + c];
    dbeta[c] = accumulate ? dbeta[c] + (float)x : (float)x;      // accumulate: second backward through shared weights
    dgamma[c] = accumulate ? dgamma[c] + (float)y : (float)y;
    if (raw_sums != nullptr) { raw_sums[c] = (float)x; raw_sums[C + c] = (float)y; }   // synchronised BatchNorm: all-reduced by the caller
    // apply-pass constants: dY = dz*A + y*B + D with A = scale, B = -scale*c2*invstd, D = -scale*c1 + scale*c2*mean*invstd
    const double c1 = x / (double)P, c2 = y / (double)P;
    const double sc = (double)a.ss[c], istd = (double)a.save[C + c], mean = (double)a.save[c];
    coef[c] = (float)(-sc * c2 * istd);
    coef[C + c] = (float)(-sc * c1 + sc * c2 * mean * istd);
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

template <int MODE, typename T>
__global__ void __launch_bounds__(TPB, (MODE == 0 || MODE == 4) ? 3 : 2) bn_bwd_apply_kernel(BnBwdArgs<T> a, const float* __restrict__ coef,
                                                              T* __restrict__ dy) {
  const BnBwdThread t = bn_bwd_thread(a);
  const int C = a.C, rows = TPB / t.cg;
  const int P = a.N * a.H * a.W;
  const int r = threadIdx.x / t.cg;
  float kb_[8], kd_[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { kb_[j] = coef[t.c0 + j]; kd_[j] = coef[C + t.c0 + j]; }
  const int stride = gridDim.x * rows;
  int p = blockIdx.x * rows + r;
  for (; p + stride < P; p += 2 * stride) {
    float dz0[8], y0[8], dz1[8], y1[8], o0[8], o1[8];
    bn_bwd_gather8<MODE>(a, t, p, dz0, y0);
    bn_bwd_gather8<MODE>(a, t, p + stride, dz1, y1);
    bn_bwd_finish8(a, t, p, dz0, y0);
    bn_bwd_finish8(a, t, p + stride, dz1, y1);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o0[j] = fmaf(dz0[j], t.sc[j], fmaf(y0[j], kb_[j], kd_[j]));
      o1[j] = fmaf(dz1[j], t.sc[j], fmaf(y1[j], kb_[j], kd_[j]));
    }
    st8(dy + (long long)p * C + t.c0, o0);
    st8(dy + (long long)(p + stride) * C + t.c0, o1);
  }
  if (p < P) {
    float dz[8], yv[8], o[8];
    bn_bwd_gather8<MODE>(a, t, p, dz, yv);
    bn_bwd_finish8(a, t, p, dz, yv);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = fmaf(dz[j], t.sc[j], fmaf(yv[j], kb_[j], kd_[j]));
    st8(dy + (long long)p * C + t.c0, o);
  }
}

// First layer (Cin = 1 -> 16, unet.py:81): the BatchNorm-backward apply pass and the weight gradient in ONE kernel.  dY of the first
// layer has no other consumer (there is no data gradient towards the image), so it is formed in registers,
//   dY = dz*scale + y*B + D,   dW[co][t] += sum_p dY[p][co] * x[p + tap_t],
// and never written: replaces bn_bwd_apply (read 2, write 1 activation-sized tensors) + wgrad_first (read 1) by one pass that reads 2.
// Thread = (pixel, channel half); two pixels in flight; 8 x 9 accumulators per thread, reduced over the warp / block, one atomicAdd per
// value and block.
template <typename T>
__global__ void __launch_bounds__(TPB, 1) bn_bwd_apply_first_kernel(BnBwdArgs<T> a, const float* __restrict__ coef, const float* __restrict__ x,
                                                                    float* __restrict__ dw /*[16][9]*/, float* __restrict__ ws) {
  // (a channel-QUARTER mapping with 36 accumulators and two blocks per SM was measured slower, 240 vs 177 us: the bytes in flight per
  // SM are what bounds this kernel, and halving the bytes per thread cancels the doubled thread count)
  const BnBwdThread t = bn_bwd_thread(a);          // C == 16: cg == 2, t.g = channel half
  const int C = 16, rows = TPB / 2;
  const int P = a.N * a.H * a.W;
  const int r = threadIdx.x >> 1;
  float kb_[8], kd_[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { kb_[j] = coef[t.c0 + j]; kd_[j] = coef[C + t.c0 + j]; }
  float acc[8][9];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int k = 0; k < 9; ++k) acc[j][k] = 0.f;
  auto window = [&](int p, float (&v)[9]) {
    const int xx = p % a.W, q = p / a.W, yy = q % a.H;
    const float* base = x + (long long)(p - yy * a.W - xx);
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int gy = yy + k / 3 - 1, gx = xx + k % 3 - 1;
      v[k] = (gy >= 0 && gy < a.H && gx >= 0 && gx < a.W) ? base[(long long)gy * a.W + gx] : 0.f;
    }
  };
  auto accumulate = [&](const float (&dz)[8], const float (&yv)[8], const float (&v)[9]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float o = fmaf(dz[j], t.sc[j], fmaf(yv[j], kb_[j], kd_[j]));
#pragma unroll
      for (int k = 0; k < 9; ++k) acc[j][k] = fmaf(o, v[k], acc[j][k]);
    }
  };
  const int stride = gridDim.x * rows;
  int p = blockIdx.x * rows + r;
  for (; p + stride < P; p += 2 * stride) {
    float dz0[8], y0[8], dz1[8], y1[8], v0[9], v1[9];
    bn_bwd_gather8<0>(a, t, p, dz0, y0);
    bn_bwd_gather8<0>(a, t, p + stride, dz1, y1);
    window(p, v0);
    window(p + stride, v1);
    bn_bwd_finish8(a, t, p, dz0, y0);
    bn_bwd_finish8(a, t, p + stride, dz1, y1);
    accumulate(dz0, y0, v0);
    accumulate(dz1, y1, v1);
  }
  if (p < P) {
    float dz[8], yv[8], v[9];
    bn_bwd_gather8<0>(a, t, p, dz, yv);
    window(p, v);
    bn_bwd_finish8(a, t, p, dz, yv);
    accumulate(dz, yv, v);
  }
  __shared__ float s_red[TPB / 32][2][72];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      float v = acc[j][k];
#pragma unroll
      for (int o = 16; o > 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);       // lanes of equal parity = same channel half
      if (lane < 2) s_red[warp][lane][j * 9 + k] = v;
    }
  __syncthreads();
  // deterministic: one row of 144 values per block in the workspace, the last block (ticket) adds the rows in block order into dw
  if (threadIdx.x < 144) {
    const int half = threadIdx.x / 72, e = threadIdx.x % 72;
    float v = 0.f;
#pragma unroll
    for (int wv = 0; wv < TPB / 32; ++wv) v += s_red[wv][half][e];
    ws[64 + (size_t)blockIdx.x * 144 + threadIdx.x] = v;                            // index = co*9 + t with co = half*8 + j
  }
  __shared__ bool s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(reinterpret_cast<unsigned*>(ws) + 1, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (threadIdx.x < 144) {
    float v = 0.f;
    int b = 0;
    for (; b + 8 <= (int)gridDim.x; b += 8) {
      float u[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) u[k] = __ldcg(&ws[64 + (size_t)(b + k) * 144 + threadIdx.x]);
#pragma unroll
      for (int k = 0; k < 8; ++k) v += u[k];
    }
    for (; b < (int)gridDim.x; ++b) v += __ldcg(&ws[64 + (size_t)b * 144 + threadIdx.x]);
    dw[threadIdx.x] += v;
  }
  if (threadIdx.x == 0) reinterpret_cast<unsigned*>(ws)[1] = 0u;
}

// ================================================================================================
// bilinear x2 upsample, align_corners=True (nn.Upsample(scale_factor=2, mode='bilinear'), unet.py:56-57)
// index arithmetic follows ATen's area_pixel_compute_source_index for align_corners: src = dst*(in-1)/(out-1)
// ================================================================================================
// With align_corners=True and out = 2*in, src(Y) = Y*(in-1)/(2*in-1): output rows 2i and 2i+1 interpolate between source rows
// (i-1, i) and (i, i+1) respectively (src(2i) = i - i/(2in-1), src(2i+1) = i + (in-1-i)/(2in-1)), and likewise for columns.  So a
// 2 x 2 block of output pixels needs exactly the 3 x 3 source neighbourhood of (i, j): nine 16-byte loads for four stores instead
// of sixteen (the old one-pixel-per-thread form was bound by L2 read bandwidth: 4 loads per stored vector).
// Weight of the upper / left source of output index Y = 2i + a: lam = clamp(src(Y) - (i - 1 + a), 0, 1) (clamped border rows coincide).
__device__ __forceinline__ float up_lam(int Y, int i_base, float ratio) {
  return fminf(fmaxf(ratio * (float)Y - (float)i_base, 0.f), 1.f);
}

template <typename T>
__global__ void __launch_bounds__(TPB) upsample2x_fwd_kernel(const T* __restrict__ t, int N, int h, int w, int C,
                                                             T* __restrict__ u) {
  const int cg = C >> 3, H = 2 * h, W = 2 * w;
  const float ry = (H > 1) ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = (W > 1) ? (float)(w - 1) / (float)(W - 1) : 0.f;
  const int total = N * h * w * cg;                    // 32-bit index arithmetic (checked on the host)
  for (int idx = blockIdx.x * TPB + threadIdx.x; idx < total; idx += gridDim.x * TPB) {
    const int g = idx % cg;
    const int p = idx / cg;
    const int j = p % w, q_ = p / w, i = q_ % h;
    const long long n = q_ / h;
    const int c0 = g * 8;
    const int ys[3] = {max(i - 1, 0), i, min(i + 1, h - 1)}, xs[3] = {max(j - 1, 0), j, min(j + 1, w - 1)};
    const T* base = t + n * (long long)h * w * C + c0;
    float v[3][3][8];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) ld8(base + ((long long)ys[a] * w + xs[b]) * C, v[a][b]);
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const float ly = up_lam(2 * i + a, i - 1 + a, ry);
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const float lx = up_lam(2 * j + b, j - 1 + b, rx);
        float o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k)
          o[k] = (1.f - ly) * ((1.f - lx) * v[a][b][k] + lx * v[a][b + 1][k]) + ly * ((1.f - lx) * v[a + 1][b][k] + lx * v[a + 1][b + 1][k]);
        st8(u + ((n * H + 2 * i + a) * (long long)W + 2 * j + b) * C + c0, o);
      }
    }
  }
}

// transpose of the above in gather form (deterministic): source row i receives from output rows 2i-1, 2i (as the LOWER source,
// weight lam) and 2i+1, 2i+2 (as the UPPER source, weight 1 - lam); the same for columns -> a 4 x 4 window of du per low-res pixel
// with closed-form weights.
template <typename T>
__global__ void __launch_bounds__(TPB) upsample2x_bwd_kernel(const T* __restrict__ du, int N, int h, int w, int C,
                                                             T* __restrict__ dt) {
  const int cg = C >> 3, H = 2 * h, W = 2 * w;
  const float ry = (H > 1) ? (float)(h - 1) / (float)(H - 1) : 0.f, rx = (W > 1) ? (float)(w - 1) / (float)(W - 1) : 0.f;
  const int total = N * h * w * cg;                    // 32-bit index arithmetic (checked on the host)
  for (int idx = blockIdx.x * TPB + threadIdx.x; idx < total; idx += gridDim.x * TPB) {
    const int g = idx % cg;
    const int p = idx / cg;
    const int j = p % w, q_ = p / w, i = q_ % h;
    const long long n = q_ / h;
    const int c0 = g * 8;
    // window rows Y = 2i-1+d, d = 0..3: d < 2 -> this pixel is the lower source (base row i-1 ... i), else the upper one
    float wy[4], wx[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int Y = 2 * i - 1 + d, X = 2 * j - 1 + d;
      const int iy = (Y >> 1), ay = Y & 1, ix = (X >> 1), ax = X & 1;      // Y = 2*iy + ay (Y >= 0 where used)
      const float ly = up_lam(Y, iy - 1 + ay, ry), lx = up_lam(X, ix - 1 + ax, rx);
      // upper source of Y is clamp(iy - 1 + ay), lower is clamp(iy + ay): pixel i may be either or (at clamped borders) both
      float a = 0.f, b = 0.f;
      if (Y >= 0 && Y < H) {
        if (max(iy - 1 + ay, 0) == i) a += 1.f - ly;
        if (min(iy + ay, h - 1) == i) a += ly;
      }
      if (X >= 0 && X < W) {
        if (max(ix - 1 + ax, 0) == j) b += 1.f - lx;
        if (min(ix + ax, w - 1) == j) b += lx;
      }
      wy[d] = a;
      wx[d] = b;
    }
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    const T* base = du + n * (long long)H * W * C + c0;
#pragma unroll
    for (int dy = 0; dy < 4; ++dy) {
      const int Y = min(max(2 * i - 1 + dy, 0), H - 1);                  // weight is 0 where clamped
      float gv[4][8];
#pragma unroll
      for (int d = 0; d < 4; ++d) ld8(base + ((long long)Y * W + min(max(2 * j - 1 + d, 0), W - 1)) * C, gv[d]);
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        const float ww = wy[dy] * wx[d];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = fmaf(ww, gv[d][k], acc[k]);
      }
    }
    st8(dt + (long long)p * C + c0, acc);
  }
}

// ================================================================================================
// channel dropout (aux branch), misc elementwise
// ================================================================================================
__global__ void chan_mask_gen_kernel(unsigned long long seed, const unsigned long long* seed_ptr, int n, float p, float* cs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (seed_ptr) seed += *seed_ptr;
  if (i < n) cs[i] = (wsl_uniform(seed, (unsigned long long)i) >= p) ? 1.f / (1.f - p) : 0.f;
}

// FeatureNoise of the third head of UNet_CCT_3H (unet.py:270-283, :369): out = f * z + f with one noise tensor z[H][W][C] shared by
// the batch; backward d f = d out * (1 + z), optionally added onto another gradient of the same feature.
__global__ void uniform_fill_kernel(unsigned long long seed, const unsigned long long* seed_ptr, long long n, float lo, float hi, float* out) {
  if (seed_ptr) seed += *seed_ptr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = lo + (hi - lo) * wsl_uniform(seed, (unsigned long long)i);
}

template <typename T>
__global__ void __launch_bounds__(TPB) feat_noise_kernel(const T* __restrict__ f, const float* __restrict__ z, long long total_vec,
                                                         long long hwc_vec, const T* __restrict__ acc, T* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total_vec; i += (long long)gridDim.x * TPB) {
    const long long zi = (i % hwc_vec) * 8;
    float v[8], a[8];
    ld8(f + i * 8, v);
    const float4 z0 = *reinterpret_cast<const float4*>(z + zi), z1 = *reinterpret_cast<const float4*>(z + zi + 4);
    const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j], zz[j], v[j]);
    if (acc) {
      ld8(acc + i * 8, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += a[j];
    }
    st8(out + i * 8, v);
  }
}

// LeakyReLU backward without BatchNorm (PNet2D's 1x1 heads, networks/pnet.py:54-59,75-81): out = g * (y > 0 ? 1 : slope), y = the stored
// pre-activation
template <typename T>
__global__ void __launch_bounds__(TPB) lrelu_bwd_kernel(const T* __restrict__ y, const T* __restrict__ g, float slope, long long total_vec,
                                                        T* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total_vec; i += (long long)gridDim.x * TPB) {
    float yv[8], gv[8];
    ld8(y + i * 8, yv);
    ld8(g + i * 8, gv);
#pragma unroll
    for (int j = 0; j < 8; ++j) gv[j] *= (yv[j] > 0.f ? 1.f : slope);
    st8(out + i * 8, gv);
  }
}

template <typename T>
__global__ void __launch_bounds__(TPB) lrelu_fwd_kernel(const T* __restrict__ y, float slope, long long total_vec, T* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total_vec; i += (long long)gridDim.x * TPB) {
    float v[8];
    ld8(y + i * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = v[j] > 0.f ? v[j] : v[j] * slope;
    st8(out + i * 8, v);
  }
}

template <typename T>
__global__ void __launch_bounds__(TPB) chan_scale_kernel(const T* __restrict__ a, const float* __restrict__ cs,
                                                         long long HW, int C, long long total_vec, T* __restrict__ d) {
  const int cg = C >> 3, hw = (int)HW, tv = (int)total_vec;       // 32-bit index arithmetic (checked on the host)
  for (int i = blockIdx.x * TPB + threadIdx.x; i < tv; i += gridDim.x * TPB) {
    const int p = i / cg;
    const int c0 = (i - p * cg) * 8;
    const long long n = p / hw;
    float v[8];
    ld8(a + (long long)p * C + c0, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] *= cs[n * C + c0 + j];
    st8(d + (long long)p * C + c0, v);
  }
}

// fp32 NCHW [N,Creal,H,W] -> bf16 NHWC [N,H,W,CP] (zero padded channels); used for dlogits
template <typename T>
__global__ void __launch_bounds__(TPB) nchw_f32_to_nhwc_bf16_kernel(const float* __restrict__ src, int Creal, int CP, long long HW,
                                                                    long long npix, float scale, T* __restrict__ dst) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < npix; i += (long long)gridDim.x * TPB) {
    const long long n = i / HW, o = i - n * HW;
    for (int c0 = 0; c0 < CP; c0 += 8) {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = (c0 + j < Creal) ? src[(n * Creal + c0 + j) * HW + o] * scale : 0.f;
      st8(dst + i * CP + c0, v);
    }
  }
}

// bf16 NHWC -> fp32 NCHW (feature export for tests / API)
template <typename T>
__global__ void __launch_bounds__(TPB) nhwc_bf16_to_nchw_f32_kernel(const T* __restrict__ src, int C, long long HW,
                                                                    long long total, float* __restrict__ dst) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const long long p = i / C;
    const int c = (int)(i - p * C);
    const long long n = p / HW, o = p - n * HW;
    dst[(n * C + c) * HW + o] = (float)src[i];
  }
}

// ================================================================================================
// weight packing and SGD
// ================================================================================================
// w: fp32 [Cout][Cin][KS][KS] (torch layout).  Outputs (any may be null):
//   wf  fp32 [T][CinP][CoutP]      forward operand of conv_direct
//   bf  bf16 [T][CoutP][CinP]      wgmma B operand, forward  (K-major: Cin contiguous)
// and, for the input-channel slice [ci_begin, ci_begin+ci_count) (one slice per concatenated source), SliceP =
// ci_count rounded up to 16:
//   wd  fp32 [T][CoutP][SliceP]    dgrad operand of conv_direct (tap flipped, roles swapped)
//   bd  bf16 [T][SliceP][CoutP]    wgmma B operand, dgrad    (K-major: Cout contiguous), tap flipped
// one 16-bit element: bf16 or (half16) fp16 bits in the same slot
__device__ __forceinline__ void st16(__nv_bfloat16* dst, float v, int half16) {
  if (half16) *reinterpret_cast<__half*>(dst) = __float2half_rn(v);
  else *dst = __float2bfloat16(v);
}

__global__ void __launch_bounds__(TPB) pack_weights_kernel(const float* __restrict__ w, int Cout, int Cin, int T, int CoutP,
                                                           int CinP, int ci_begin, int ci_count, float* wf, float* wd,
                                                           __nv_bfloat16* bf, __nv_bfloat16* bd, int half16) {
  const long long total = (long long)T * CoutP * CinP;
  const int SliceP = (ci_count + 15) & ~15;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int ci = (int)(i % CinP), co = (int)((i / CinP) % CoutP), t = (int)(i / ((long long)CinP * CoutP));
    const float v = (co < Cout && ci < Cin) ? w[((size_t)co * Cin + ci) * T + t] : 0.f;
    if (wf) wf[((size_t)t * CinP + ci) * CoutP + co] = v;
    if (bf) st16(bf + ((size_t)t * CoutP + co) * CinP + ci, v, half16);
    const int cs = ci - ci_begin;
    if (cs >= 0 && cs < SliceP) {
      const float vs = (cs < ci_count) ? v : 0.f;
      if (wd) wd[((size_t)(T - 1 - t) * CoutP + co) * SliceP + cs] = vs;
      if (bd) st16(bd + ((size_t)(T - 1 - t) * SliceP + cs) * CoutP + co, vs, half16);
    }
  }
}

// Batched form: ONE launch packs every layer.  table[e] = 13 int64: {w, wf, wd, bf, bd, Cout, Cin, T, CoutP, CinP, ci_begin,
// ci_count, first_item}; items of entry e are [first_item(e), first_item(e+1)).
__global__ void __launch_bounds__(TPB) pack_weights_batched_kernel(const long long* __restrict__ table, int n_entries, long long total,
                                                                   int half16) {
  __shared__ long long s_first[129];
  for (int e = threadIdx.x; e <= n_entries; e += TPB) s_first[e] = (e < n_entries) ? table[e * 13 + 12] : total;
  __syncthreads();
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    int lo = 0, hi = n_entries - 1;
    while (lo < hi) {                     // last entry whose first_item <= i
      const int mid = (lo + hi + 1) >> 1;
      if (s_first[mid] <= i) lo = mid; else hi = mid - 1;
    }
    const long long* t = table + lo * 13;
    const float* w = reinterpret_cast<const float*>(t[0]);
    float* wf = reinterpret_cast<float*>(t[1]);
    float* wd = reinterpret_cast<float*>(t[2]);
    __nv_bfloat16* bf = reinterpret_cast<__nv_bfloat16*>(t[3]);
    __nv_bfloat16* bd = reinterpret_cast<__nv_bfloat16*>(t[4]);
    const int Cout = (int)t[5], Cin = (int)t[6], T = (int)t[7], CoutP = (int)t[8], CinP = (int)t[9], ci_begin = (int)t[10],
              ci_count = (int)t[11];
    const long long j = i - s_first[lo];
    const int SliceP = (ci_count + 15) & ~15;
    const int ci = (int)(j % CinP), co = (int)((j / CinP) % CoutP), tt = (int)(j / ((long long)CinP * CoutP));
    const float v = (co < Cout && ci < Cin) ? w[((size_t)co * Cin + ci) * T + tt] : 0.f;
    if (wf) wf[((size_t)tt * CinP + ci) * CoutP + co] = v;
    if (bf) st16(bf + ((size_t)tt * CoutP + co) * CinP + ci, v, half16);
    const int cs = ci - ci_begin;
    if (cs >= 0 && cs < SliceP) {
      const float vs = (cs < ci_count) ? v : 0.f;
      if (wd) wd[((size_t)(T - 1 - tt) * CoutP + co) * SliceP + cs] = vs;
      if (bd) st16(bd + ((size_t)(T - 1 - tt) * SliceP + cs) * CoutP + co, vs, half16);
    }
  }
}

// torch.optim.SGD(momentum, weight_decay), dampening 0, no nesterov: g += wd*p; buf = mu*buf + g; p -= lr*buf
// (zero-initialised buf reproduces torch's first-step "buf = g").
__global__ void __launch_bounds__(TPB) sgd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                  long long n, const float* lr_ptr, float lr, float mu, float wd, float gscale) {
  const float l = lr_ptr ? *lr_ptr : lr;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < n; i += (long long)gridDim.x * TPB) {
    const float gg = fmaf(wd, p[i], g[i] * gscale);
    const float b = fmaf(mu, m[i], gg);
    m[i] = b;
    p[i] = p[i] - l * b;
  }
}

// torch.optim.Adam (weight_decay 0, amsgrad off), one step over a flat buffer, rounded where torch's multi-tensor path rounds:
// each foreach op stores its result, and `a + s * b` compiles to one fma there as here.  w1 = 1 - beta1, w2 = 1 - beta2, eps and
// the two t-dependent scalars are the fp32 values of torch's Python doubles; scal_ptr (device) = {lr / (1 - beta1^t),
// sqrt(1 - beta2^t)} replaces the by-value pair so a captured CUDA graph follows t.
__global__ void __launch_bounds__(TPB) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, long long n, const float* scal_ptr, float step_size,
                                                   float bc2_sqrt, float w1, float b2, float w2, float eps) {
  const float ss = scal_ptr ? scal_ptr[0] : step_size;
  const float bc = scal_ptr ? scal_ptr[1] : bc2_sqrt;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < n; i += (long long)gridDim.x * TPB) {
    const float gi = g[i];
    const float mi = fmaf(w1, gi - m[i], m[i]);             // exp_avg.lerp_(g, 1 - beta1): weight < 0.5 branch of at::lerp
    float vi = v[i] * b2;                                   // exp_avg_sq.mul_(beta2)
    vi = fmaf(w2, gi * gi, vi);                             //           .addcmul_(g, g, value=1 - beta2)
    const float denom = sqrtf(vi) / bc + eps;               // (exp_avg_sq.sqrt() / sqrt(1 - beta2^t)).add_(eps)
    m[i] = mi;
    v[i] = vi;
    p[i] = fmaf(-ss, mi / denom, p[i]);                     // param.addcdiv_(exp_avg, denom, value=-step_size)
  }
}

// ---- fp16 hi/lo split operands of the "fp16x3" tensor-core parity mode (conv_tc.cu: wsl_conv_tc_split) -------------
// fp32 channels-last [P][C0] (and optionally [P][C1], concatenated along C) -> fp16 [P][2*(C0+C1)] = (hi plane | lo plane),
// hi = fp16(v), lo = fp16(v - hi): v is carried with 22 significant bits.
// Every staged tensor carries its own power-of-two scale (2^k with max|v| * 2^k in [2^13, 2^14)): fp16 has a 5-bit exponent, and
// the lo plane sits 11 binades below the hi plane, so without it small activations / gradients would lose their lo bits to
// underflow (measured: 8e-3 relative error on first-layer weight gradients with a single global loss scale).  scale2 = {2^k, 2^-k}
// is written for the consumers, which multiply their fp32 results by 2^-k (exact).
__global__ void __launch_bounds__(TPB) absmax_kernel(const float* __restrict__ s0, long long n0, const float* __restrict__ s1, long long n1,
                                                     unsigned* __restrict__ amax_bits) {
  float m = 0.f;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < n0 + n1; i += (long long)gridDim.x * TPB)
    m = fmaxf(m, fabsf(i < n0 ? s0[i] : s1[i - n0]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax_bits, __float_as_uint(m));     // non-negative floats order like their bits
}

__global__ void __launch_bounds__(TPB) split_f32_kernel(const float* __restrict__ s0, int C0, const float* __restrict__ s1, int C1,
                                                        long long P, __half* __restrict__ dst, const unsigned* __restrict__ amax_bits,
                                                        float* __restrict__ scale2) {
  const int C = C0 + C1, cg = C >> 3;
  const long long total = P * cg;
  const float amax = __uint_as_float(*amax_bits);
  int e = 0;
  if (amax > 0.f && amax < 3.0e38f) frexpf(amax, &e);            // amax = f * 2^e, f in [0.5, 1)
  const float sc = (amax > 0.f) ? ldexpf(1.f, 14 - e) : 1.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) { scale2[0] = sc; scale2[1] = 1.f / sc; }
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const long long p = i / cg;
    const int c = (int)(i - p * cg) * 8;
    float v[8], hi[8], lo[8];
    if (c < C0) ld8(s0 + p * C0 + c, v); else ld8(s1 + p * C1 + (c - C0), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      v[j] *= sc;
      hi[j] = __half2float(__float2half_rn(v[j]));
      lo[j] = v[j] - hi[j];
    }
    st8(dst + p * 2 * C + c, hi);
    st8(dst + p * 2 * C + C + c, lo);
  }
}

// w: fp32 torch layout [Cout][Cin][T].  f3: fp16 [T][CoutP][3*CinP] = (w_hi | w_hi | w_lo) along K (forward B operand);
// d3 for the input-channel slice [ci_begin, ci_begin + ci_count): fp16 [T][SliceP][3*CoutP], taps flipped (dgrad B operand).
__global__ void __launch_bounds__(TPB) pack_split_weights_kernel(const float* __restrict__ w, int Cout, int Cin, int T, int CoutP,
                                                                 int CinP, int ci_begin, int ci_count, __half* f3, __half* d3) {
  const long long total = (long long)T * CoutP * CinP;
  const int SliceP = (ci_count + 15) & ~15;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int ci = (int)(i % CinP), co = (int)((i / CinP) % CoutP), t = (int)(i / ((long long)CinP * CoutP));
    const float v = (co < Cout && ci < Cin) ? w[((size_t)co * Cin + ci) * T + t] : 0.f;
    const __half h = __float2half_rn(v);
    const __half l = __float2half_rn(v - __half2float(h));
    if (f3) {
      __half* o = f3 + ((size_t)t * CoutP + co) * 3 * CinP;
      o[ci] = h; o[CinP + ci] = h; o[2 * CinP + ci] = l;
    }
    const int cs = ci - ci_begin;
    if (d3 && cs >= 0 && cs < SliceP) {
      const bool real = cs < ci_count;
      __half* o = d3 + ((size_t)(T - 1 - t) * SliceP + cs) * 3 * CoutP;
      o[co] = real ? h : __half(0.f); o[CoutP + co] = real ? h : __half(0.f); o[2 * CoutP + co] = real ? l : __half(0.f);
    }
  }
}

inline int grid_for(long long items) {
  long long b = (items + TPB - 1) / TPB;
  if (b < 1) b = 1;
  if (b > wsl_num_sms() * 8) b = wsl_num_sms() * 8;
  return (int)b;
}

inline int bn_grid(long long P, int C, int per_sm = 3) {
  // every block should stream >= ~96 KB so that the fixed-order finalize (one pass over all partials) stays negligible
  long long b = (P * C * 2 + 96 * 1024 - 1) / (96 * 1024);
  if (b < 1) b = 1;
  if (b > wsl_num_sms() * per_sm) b = wsl_num_sms() * per_sm;      // one full wave: 3 resident blocks / SM at 80 registers, 2 for the multi-source variants
  return (int)b;
}

}  // namespace

// run `expr` with T = bf16 (dtype 0) or float (dtype 1)
#define WSL_DISPATCH_T(dtype, ...)                             \
  do {                                                         \
    if ((dtype) == 1) { using T = float; __VA_ARGS__; }        \
    else if ((dtype) == 2) { using T = __half; __VA_ARGS__; }  \
    else { using T = bf16; __VA_ARGS__; }                      \
  } while (0)

// ================================================================================================
// C ABI
// ================================================================================================
WSL_API int wsl_conv_direct(const void* src0, int C0, const void* src1, int C1, int src_f32, const float* wpk,
                            const float* bias, void* out, int out_mode, int N, int H, int W, int CinP, int CoutP,
                            int CoutStore, int ksize, cudaStream_t stream) {
  WSL_REQUIRE(ksize == 3 || ksize == 1, "wsl_conv_direct: ksize must be 1 or 3");
  WSL_REQUIRE(CinP % 16 == 0 && CoutP % 16 == 0, "wsl_conv_direct: padded channel counts must be multiples of 16");
  WSL_REQUIRE((src_f32 == 1 && C1 == 0) || (C0 % 8 == 0 && C1 % 8 == 0), "wsl_conv_direct: multi-channel sources need C %% 8 == 0");
  const int tx = (W + 15) / 16, ty = (H + 15) / 16;
  dim3 grid(N * tx * ty, CoutP / 16);
  if (ksize == 3)
    conv_direct_kernel<3><<<grid, 128, 0, stream>>>(src0, C0, src1, C1, src_f32, wpk, bias, out, out_mode, N, H, W, CinP, CoutP, CoutStore, tx, ty);
  else
    conv_direct_kernel<1><<<grid, 128, 0, stream>>>(src0, C0, src1, C1, src_f32, wpk, bias, out, out_mode, N, H, W, CinP, CoutP, CoutStore, tx, ty);
  return wsl_check_launch("conv_direct");
}

WSL_API int wsl_wgrad_direct(const void* src0, int C0, const void* src1, int C1, int src_f32, const void* dy, int dy_f32,
                             int CoutP, float* dw, float* dbias, int N, int H, int W, int CoutReal, int ksize,
                             cudaStream_t stream) {
  WSL_REQUIRE(ksize == 3 || ksize == 1, "wsl_wgrad_direct: ksize must be 1 or 3");
  WSL_REQUIRE(CoutP % 16 == 0, "wsl_wgrad_direct: CoutP must be a multiple of 16");
  const int Cin = C0 + C1;
  const int tx = (W + 15) / 16, ty = (H + 7) / 8;
  const int ob = (CoutP / 16) * ((Cin + 15) / 16);
  int splits = (wsl_num_sms() * 6 + ob - 1) / ob;
  const int ntiles = N * tx * ty;
  if (splits > ntiles) splits = ntiles;
  if (splits < 1) splits = 1;
  dim3 grid(ob, splits);
  if (ksize == 3)
    wgrad_direct_kernel<3><<<grid, 256, 0, stream>>>(src0, C0, src1, C1, src_f32, dy, dy_f32, CoutP, dw, dbias, N, H, W, CoutReal, tx, ty);
  else
    wgrad_direct_kernel<1><<<grid, 256, 0, stream>>>(src0, C0, src1, C1, src_f32, dy, dy_f32, CoutP, dw, dbias, N, H, W, CoutReal, tx, ty);
  return wsl_check_launch("wgrad_direct");
}

WSL_API int wsl_bn_stats(const void* y, int dtype, long long P, int C, const float* gamma, const float* beta, float* running_mean,
                         float* running_var, long long* num_batches_tracked, float momentum, float eps, float* save,
                         float* ss, float* ws, float* raw_sums, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0 && C <= 256 && TPB % (C / 8) == 0, "wsl_bn_stats: unsupported channel count %d", C);
  const int grid = bn_grid(P, C);
  WSL_REQUIRE((long long)grid * 2 * C + 64 <= WSL_WS_FLOATS, "wsl_bn_stats: workspace too small");
  WSL_DISPATCH_T(dtype, bn_stats_kernel<T><<<grid, TPB, TPB * 16 * sizeof(float), stream>>>(
                            (const T*)y, P, C, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, save, ss,
                            ws + 64, reinterpret_cast<unsigned*>(ws), raw_sums));
  return wsl_check_launch("bn_stats");
}

WSL_API int wsl_bn_eval_prepare(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                                float eps, int C, float* ss, cudaStream_t stream) {
  bn_eval_prepare_kernel<<<(C + 127) / 128, 128, 0, stream>>>(gamma, beta, running_mean, running_var, eps, C, ss);
  return wsl_check_launch("bn_eval_prepare");
}

static int bn_act_launch(const void* y, int dtype, const float* ss, int N, int H, int W, int C, float slope, float drop_p,
                         const uint8_t* mask, unsigned long long seed, const unsigned long long* seed_ptr, void* act,
                         void* pooled, uint8_t* pool_idx, const BnFin& fin, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0, "wsl_bn_act_fwd: C %% 8 != 0");
  WSL_REQUIRE(pooled == nullptr || (H % 2 == 0 && W % 2 == 0), "wsl_bn_act_fwd: pooling needs even H, W");
  WSL_REQUIRE(TPB % (C / 8) == 0 && (long long)N * H * W < (1LL << 31), "wsl_bn_act_fwd: unsupported C=%d or too many pixels", C);
  const long long items = (long long)N * H * W * (C / 8) / (pooled ? 4 : 1);
  WSL_DISPATCH_T(dtype, bn_act_fwd_kernel<T><<<grid_for((items + 1) / 2), TPB, 0, stream>>>(
                            (const T*)y, ss, N, H, W, C, slope, drop_p, mask, seed, seed_ptr, (T*)act, (T*)pooled, pool_idx, fin));
  return wsl_check_launch("bn_act_fwd");
}

WSL_API int wsl_bn_act_fwd(const void* y, int dtype, const float* ss, int N, int H, int W, int C, float slope, float drop_p,
                           const uint8_t* mask, unsigned long long seed, const unsigned long long* seed_ptr, void* act,
                           void* pooled, uint8_t* pool_idx, cudaStream_t stream) {
  BnFin fin;
  fin.partials = nullptr; fin.nrows = 0; fin.P = 0; fin.gamma = fin.beta = nullptr; fin.running_mean = fin.running_var = nullptr;
  fin.nbt = nullptr; fin.momentum = 0.f; fin.eps = 0.f; fin.save = fin.ss_out = nullptr;
  return bn_act_launch(y, dtype, ss, N, H, W, C, slope, drop_p, mask, seed, seed_ptr, act, pooled, pool_idx, fin, stream);
}

WSL_API int wsl_bn_finalize_act_fwd(const void* y, int dtype, const float* partials, int nrows, const float* gamma, const float* beta,
                                    float* running_mean, float* running_var, long long* num_batches_tracked, float momentum, float eps,
                                    float* save, float* ss, int N, int H, int W, int C, float slope, float drop_p, const uint8_t* mask,
                                    unsigned long long seed, const unsigned long long* seed_ptr, void* act, void* pooled,
                                    uint8_t* pool_idx, cudaStream_t stream) {
  WSL_REQUIRE(C <= 32 && partials != nullptr && nrows >= 1, "wsl_bn_finalize_act_fwd: C <= 32 and partial rows are required (got C=%d)", C);
  BnFin fin;
  fin.partials = partials; fin.nrows = nrows; fin.P = (long long)N * H * W; fin.gamma = gamma; fin.beta = beta;
  fin.running_mean = running_mean; fin.running_var = running_var; fin.nbt = num_batches_tracked; fin.momentum = momentum; fin.eps = eps;
  fin.save = save; fin.ss_out = ss;
  return bn_act_launch(y, dtype, ss, N, H, W, C, slope, drop_p, mask, seed, seed_ptr, act, pooled, pool_idx, fin, stream);
}

template <typename T>
static int bn_bwd_launch(const void* y, const float* ss, const float* save, const void* g0, const void* g1, const float* cs1,
                         const void* gpool, const uint8_t* pool_idx, const uint8_t* mask, unsigned long long seed,
                         const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W, int C, float* dgamma,
                         float* dbeta, float* coef, void* dy, float* ws, int accumulate, cudaStream_t stream, int phase = 0,
                         float* raw_sums = nullptr) {
  BnBwdArgs<T> a;
  a.y = (const T*)y; a.ss = ss; a.save = save; a.g0 = (const T*)g0; a.g1 = (const T*)g1;
  a.cs1 = cs1; a.gp = (const T*)gpool; a.pool_idx = pool_idx; a.mask = mask; a.seed = seed; a.seed_ptr = seed_ptr; a.drop_p = drop_p;
  a.slope = slope; a.N = N; a.H = H; a.W = W; a.C = C;
  const long long P = (long long)N * H * W;
  const int mode = (g0 == nullptr) ? 4 : ((g1 ? 1 : 0) | (gpool ? 2 : 0));
  const int grid = bn_grid(P, C, (mode == 0 || mode == 4) ? 3 : 2);
  unsigned* ticket = reinterpret_cast<unsigned*>(ws);
#define WSL_BN_RED(M) bn_bwd_reduce_kernel<M, T><<<grid, TPB, TPB * 16 * sizeof(float), stream>>>(a, dgamma, dbeta, coef, ws + 64, ticket, accumulate, raw_sums)
#define WSL_BN_APP(M) bn_bwd_apply_kernel<M, T><<<grid, TPB, 0, stream>>>(a, coef, (T*)dy)
  int rc = 0;
  if (phase != 2) {
    switch (mode) {
      case 0: WSL_BN_RED(0); break;
      case 1: WSL_BN_RED(1); break;
      case 2: WSL_BN_RED(2); break;
      case 3: WSL_BN_RED(3); break;
      default: WSL_BN_RED(4); break;
    }
    rc = wsl_check_launch("bn_bwd_reduce");
    if (rc || phase == 1) return rc;
  }
  switch (mode) {
    case 0: WSL_BN_APP(0); break;
    case 1: WSL_BN_APP(1); break;
    case 2: WSL_BN_APP(2); break;
    case 3: WSL_BN_APP(3); break;
    default: WSL_BN_APP(4); break;
  }
#undef WSL_BN_RED
#undef WSL_BN_APP
  return wsl_check_launch("bn_bwd_apply");
}

WSL_API int wsl_bn_bwd(const void* y, int dtype, const float* ss, const float* save, const void* g0, const void* g1, const float* cs1,
                       const void* gpool, const uint8_t* pool_idx, const uint8_t* mask, unsigned long long seed,
                       const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W, int C, float* dgamma, float* dbeta, float* coef, void* dy, float* ws, int accumulate,
                       cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0 && C <= 256 && TPB % (C / 8) == 0, "wsl_bn_bwd: unsupported channel count %d", C);
  const long long P = (long long)N * H * W;
  WSL_REQUIRE((long long)bn_grid(P, C) * 2 * C + 64 <= WSL_WS_FLOATS && P < (1LL << 31), "wsl_bn_bwd: workspace too small / too many pixels");
  if (dtype == 1)
    return bn_bwd_launch<float>(y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, seed, seed_ptr, drop_p, slope, N, H, W, C, dgamma, dbeta, coef, dy, ws, accumulate, stream);
  if (dtype == 2)
    return bn_bwd_launch<__half>(y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, seed, seed_ptr, drop_p, slope, N, H, W, C, dgamma, dbeta, coef, dy, ws, accumulate, stream);
  return bn_bwd_launch<bf16>(y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, seed, seed_ptr, drop_p, slope, N, H, W, C, dgamma, dbeta, coef, dy, ws, accumulate, stream);
}

// Synchronised BatchNorm (global-batch statistics across data-parallel ranks): phase 1 = reduction only (local dgamma / dbeta and the raw
// sums {sum dz, sum dz*xhat}), the caller all-reduces raw_sums, wsl_bn_bwd_coef turns the GLOBAL sums into the apply constants, phase 2 =
// apply only.
WSL_API int wsl_bn_bwd_phase(const void* y, int dtype, const float* ss, const float* save, const void* g0, const void* g1, const float* cs1,
                             const void* gpool, const uint8_t* pool_idx, const uint8_t* mask, unsigned long long seed,
                             const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W, int C, float* dgamma,
                             float* dbeta, float* coef, void* dy, float* ws, int accumulate, int phase, float* raw_sums, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0 && C <= 256 && TPB % (C / 8) == 0, "wsl_bn_bwd_phase: unsupported channel count %d", C);
  WSL_REQUIRE(phase == 1 || phase == 2, "wsl_bn_bwd_phase: phase must be 1 (reduce) or 2 (apply)");
  if (dtype == 1)
    return bn_bwd_launch<float>(y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, seed, seed_ptr, drop_p, slope, N, H, W, C, dgamma, dbeta, coef, dy, ws, accumulate, stream, phase, raw_sums);
  if (dtype == 2)
    return bn_bwd_launch<__half>(y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, seed, seed_ptr, drop_p, slope, N, H, W, C, dgamma, dbeta, coef, dy, ws, accumulate, stream, phase, raw_sums);
  return bn_bwd_launch<bf16>(y, ss, save, g0, g1, cs1, gpool, pool_idx, mask, seed, seed_ptr, drop_p, slope, N, H, W, C, dgamma, dbeta, coef, dy, ws, accumulate, stream, phase, raw_sums);
}

__global__ void bn_bwd_coef_kernel(const float* __restrict__ raw_sums, double P, const float* __restrict__ ss, const float* __restrict__ save,
                                   int C, float* __restrict__ coef) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double c1 = (double)raw_sums[c] / P, c2 = (double)raw_sums[C + c] / P;
  const double sc = (double)ss[c], istd = (double)save[C + c], mean = (double)save[c];
  coef[c] = (float)(-sc * c2 * istd);
  coef[C + c] = (float)(-sc * c1 + sc * c2 * mean * istd);
}

WSL_API int wsl_bn_bwd_coef(const float* raw_sums, long long P_global, const float* ss, const float* save, int C, float* coef,
                            cudaStream_t stream) {
  bn_bwd_coef_kernel<<<(C + 127) / 128, 128, 0, stream>>>(raw_sums, (double)P_global, ss, save, C, coef);
  return wsl_check_launch("bn_bwd_coef");
}

WSL_API int wsl_bn_bwd_first(const void* y, int dtype, const float* ss, const float* save, const void* g0, const uint8_t* mask,
                             unsigned long long seed, const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W,
                             float* dgamma, float* dbeta, float* coef, const float* image, float* dw, float* ws, int accumulate,
                             cudaStream_t stream) {
  const int C = 16;
  const long long P = (long long)N * H * W;
  WSL_REQUIRE(g0 != nullptr && image != nullptr && dw != nullptr, "wsl_bn_bwd_first: g0, image and dw are required");
  WSL_REQUIRE((long long)bn_grid(P, C) * 2 * C + 64 <= WSL_WS_FLOATS && P < (1LL << 31), "wsl_bn_bwd_first: workspace too small / too many pixels");
  unsigned* ticket = reinterpret_cast<unsigned*>(ws);
  const int grid = bn_grid(P, C, 3);
  int grid2 = (int)((P * 2 + TPB - 1) / TPB);
  if (grid2 > wsl_num_sms()) grid2 = wsl_num_sms();
  if (grid2 < 1) grid2 = 1;
  WSL_DISPATCH_T(dtype, {
    BnBwdArgs<T> a;
    a.y = (const T*)y; a.ss = ss; a.save = save; a.g0 = (const T*)g0; a.g1 = nullptr; a.cs1 = nullptr; a.gp = nullptr; a.pool_idx = nullptr;
    a.mask = mask; a.seed = seed; a.seed_ptr = seed_ptr; a.drop_p = drop_p; a.slope = slope; a.N = N; a.H = H; a.W = W; a.C = C;
    bn_bwd_reduce_kernel<0, T><<<grid, TPB, TPB * 16 * sizeof(float), stream>>>(a, dgamma, dbeta, coef, ws + 64, ticket, accumulate);
    bn_bwd_apply_first_kernel<T><<<grid2, TPB, 0, stream>>>(a, coef, image, dw, ws);   // reuses ws after the reduce kernel (same stream)
  });
  return wsl_check_launch("bn_bwd_first");
}

WSL_API int wsl_upsample2x_fwd(const void* t, int dtype, int N, int h, int w, int C, void* u, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0, "wsl_upsample2x_fwd: C %% 8 != 0");
  WSL_REQUIRE(TPB % (C / 8) == 0, "wsl_upsample2x_fwd: unsupported C=%d", C);
  WSL_REQUIRE((long long)N * h * w * (C / 8) < (1LL << 31), "wsl_upsample2x_fwd: too many elements for 32-bit indexing");
  WSL_DISPATCH_T(dtype, upsample2x_fwd_kernel<T><<<grid_for((long long)N * h * w * (C / 8)), TPB, 0, stream>>>((const T*)t, N, h, w, C, (T*)u));
  return wsl_check_launch("upsample2x_fwd");
}

WSL_API int wsl_upsample2x_bwd(const void* du, int dtype, int N, int h, int w, int C, void* dt, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0, "wsl_upsample2x_bwd: C %% 8 != 0");
  WSL_REQUIRE((long long)N * h * w * (C / 8) < (1LL << 31), "wsl_upsample2x_bwd: too many elements for 32-bit indexing");
  WSL_DISPATCH_T(dtype, upsample2x_bwd_kernel<T><<<grid_for((long long)N * h * w * (C / 8)), TPB, 0, stream>>>((const T*)du, N, h, w, C, (T*)dt));
  return wsl_check_launch("upsample2x_bwd");
}

WSL_API int wsl_chan_mask_gen(unsigned long long seed, const unsigned long long* seed_ptr, int n, float p, float* cs,
                              cudaStream_t stream) {
  chan_mask_gen_kernel<<<(n + 255) / 256, 256, 0, stream>>>(seed, seed_ptr, n, p, cs);
  return wsl_check_launch("chan_mask_gen");
}

WSL_API int wsl_uniform_fill(unsigned long long seed, const unsigned long long* seed_ptr, long long n, float lo, float hi, float* out,
                             cudaStream_t stream) {
  uniform_fill_kernel<<<grid_for(n), 256, 0, stream>>>(seed, seed_ptr, n, lo, hi, out);
  return wsl_check_launch("uniform_fill");
}

WSL_API int wsl_feat_noise_fwd(const void* f, int dtype, const float* z, int N, long long hwc, void* out, cudaStream_t stream) {
  WSL_REQUIRE(hwc % 8 == 0, "wsl_feat_noise_fwd: H*W*C must be a multiple of 8");
  WSL_DISPATCH_T(dtype, feat_noise_kernel<T><<<grid_for(N * hwc / 8), TPB, 0, stream>>>((const T*)f, z, N * hwc / 8, hwc / 8, nullptr, (T*)out));
  return wsl_check_launch("feat_noise_fwd");
}

WSL_API int wsl_feat_noise_bwd(const void* g, int dtype, const float* z, int N, long long hwc, void* acc, void* out, cudaStream_t stream) {
  WSL_REQUIRE(hwc % 8 == 0, "wsl_feat_noise_bwd: H*W*C must be a multiple of 8");
  // acc != NULL: acc += g * (1 + z) (in place); else out = g * (1 + z) (out may alias g)
  WSL_DISPATCH_T(dtype, feat_noise_kernel<T><<<grid_for(N * hwc / 8), TPB, 0, stream>>>((const T*)g, z, N * hwc / 8, hwc / 8, (const T*)acc,
                                                                                    (T*)(acc ? acc : out)));
  return wsl_check_launch("feat_noise_bwd");
}

WSL_API int wsl_lrelu_fwd(const void* y, int dtype, float slope, long long n, void* out, cudaStream_t stream) {
  WSL_REQUIRE(n % 8 == 0, "wsl_lrelu_fwd: element count must be a multiple of 8");
  WSL_DISPATCH_T(dtype, lrelu_fwd_kernel<T><<<grid_for(n / 8), TPB, 0, stream>>>((const T*)y, slope, n / 8, (T*)out));
  return wsl_check_launch("lrelu_fwd");
}

WSL_API int wsl_lrelu_bwd(const void* y, int dtype, const void* g, float slope, long long n, void* out, cudaStream_t stream) {
  WSL_REQUIRE(n % 8 == 0, "wsl_lrelu_bwd: element count must be a multiple of 8");
  WSL_DISPATCH_T(dtype, lrelu_bwd_kernel<T><<<grid_for(n / 8), TPB, 0, stream>>>((const T*)y, (const T*)g, slope, n / 8, (T*)out));
  return wsl_check_launch("lrelu_bwd");
}

WSL_API int wsl_chan_scale(const void* a, int dtype, const float* cs, int N, int H, int W, int C, void* d, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0, "wsl_chan_scale: C %% 8 != 0");
  const long long tv = (long long)N * H * W * (C / 8);
  WSL_REQUIRE(tv < (1LL << 31), "wsl_chan_scale: too many elements for 32-bit indexing");
  WSL_DISPATCH_T(dtype, chan_scale_kernel<T><<<grid_for(tv), TPB, 0, stream>>>((const T*)a, cs, (long long)H * W, C, tv, (T*)d));
  return wsl_check_launch("chan_scale");
}

WSL_API int wsl_nchw_f32_to_nhwc(const float* src, int N, int Creal, int H, int W, int CP, void* dst, int dtype, float scale,
                                 cudaStream_t stream) {
  WSL_REQUIRE(CP % 8 == 0 && CP >= Creal, "wsl_nchw_f32_to_nhwc: bad padded channel count");
  const long long npix = (long long)N * H * W;
  WSL_DISPATCH_T(dtype, nchw_f32_to_nhwc_bf16_kernel<T><<<grid_for(npix), TPB, 0, stream>>>(src, Creal, CP, (long long)H * W, npix, scale, (T*)dst));
  return wsl_check_launch("nchw_f32_to_nhwc");
}

WSL_API int wsl_nhwc_to_nchw_f32(const void* src, int dtype, int N, int C, int H, int W, float* dst, cudaStream_t stream) {
  const long long total = (long long)N * H * W * C;
  WSL_DISPATCH_T(dtype, nhwc_bf16_to_nchw_f32_kernel<T><<<grid_for(total), TPB, 0, stream>>>((const T*)src, C, (long long)H * W, total, dst));
  return wsl_check_launch("nhwc_to_nchw_f32");
}

WSL_API int wsl_pack_conv_weights(const float* w, int Cout, int Cin, int ksize, int CoutP, int CinP, int ci_begin,
                                  int ci_count, float* wf, float* wd, void* bf, void* bd, int dtype16, cudaStream_t stream) {
  const int T = ksize * ksize;
  WSL_REQUIRE(ci_begin % 16 == 0 || ci_count == 0, "wsl_pack_conv_weights: slice start must be a multiple of 16");
  WSL_REQUIRE(ci_begin + ((ci_count + 15) & ~15) <= CinP || ci_count == 0, "wsl_pack_conv_weights: slice exceeds CinP");
  pack_weights_kernel<<<grid_for((long long)T * CoutP * CinP), TPB, 0, stream>>>(w, Cout, Cin, T, CoutP, CinP, ci_begin, ci_count,
                                                                                 wf, wd, (__nv_bfloat16*)bf, (__nv_bfloat16*)bd, dtype16 == 2);
  return wsl_check_launch("pack_conv_weights");
}

WSL_API int wsl_split_f32(const float* src0, int C0, const float* src1, int C1, long long P, void* dst, float* scale3,
                          cudaStream_t stream) {
  WSL_REQUIRE(C0 % 8 == 0 && C1 % 8 == 0 && C0 > 0, "wsl_split_f32: channel counts must be multiples of 8 (got %d,%d)", C0, C1);
  // scale3 = {2^k, 2^-k, scratch}: the third word holds the bit pattern of max|v| between the two kernels
  unsigned* amax = reinterpret_cast<unsigned*>(scale3 + 2);
  cudaMemsetAsync(amax, 0, sizeof(unsigned), stream);
  absmax_kernel<<<grid_for(P * (C0 + C1) / 4), TPB, 0, stream>>>(src0, P * C0, src1, P * C1, amax);
  split_f32_kernel<<<grid_for(P * ((C0 + C1) / 8)), TPB, 0, stream>>>(src0, C0, src1, C1, P, (__half*)dst, amax, scale3);
  return wsl_check_launch("split_f32");
}

WSL_API int wsl_pack_split_weights(const float* w, int Cout, int Cin, int ksize, int CoutP, int CinP, int ci_begin, int ci_count,
                                   void* f3, void* d3, cudaStream_t stream) {
  const int T = ksize * ksize;
  WSL_REQUIRE(ci_begin % 16 == 0 || ci_count == 0, "wsl_pack_split_weights: slice start must be a multiple of 16");
  pack_split_weights_kernel<<<grid_for((long long)T * CoutP * CinP), TPB, 0, stream>>>(w, Cout, Cin, T, CoutP, CinP, ci_begin, ci_count,
                                                                                       (__half*)f3, (__half*)d3);
  return wsl_check_launch("pack_split_weights");
}

WSL_API int wsl_sgd_step(float* param, const float* grad, float* mom, long long n, const float* lr_ptr, float lr,
                         float momentum, float weight_decay, float grad_scale, cudaStream_t stream) {
  sgd_kernel<<<grid_for(n), TPB, 0, stream>>>(param, grad, mom, n, lr_ptr, lr, momentum, weight_decay, grad_scale);
  return wsl_check_launch("sgd_step");
}

WSL_API int wsl_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, const float* scalars_ptr,
                          double step_size, double bc2_sqrt, double beta1, double beta2, double eps, cudaStream_t stream) {
  WSL_REQUIRE(n >= 0 && beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0, "wsl_adam_step: bad betas (%g, %g)", beta1, beta2);
  if (n == 0) return 0;
  adam_kernel<<<grid_for(n), TPB, 0, stream>>>(param, grad, exp_avg, exp_avg_sq, n, scalars_ptr, (float)step_size, (float)bc2_sqrt,
                                               (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps);
  return wsl_check_launch("adam_step");
}

WSL_API int wsl_conv_first(const float* x, const float* w, const float* bias, void* y, int dtype, int N, int H, int W, int Cout,
                           float* stat_partials, int* stat_rows_host, cudaStream_t stream) {
  WSL_REQUIRE(Cout == 16, "wsl_conv_first: compiled for 1 -> 16 channels (got Cout=%d)", Cout);
  WSL_REQUIRE((long long)N * H * W < (1LL << 30), "wsl_conv_first: too many pixels for 32-bit indexing");
  long long b = ((long long)N * H * ((W + 1) / 2) * 2 + TPB - 1) / TPB;
  if (b > wsl_num_sms() * 4) b = wsl_num_sms() * 4;                  // one wave: four resident blocks per SM
  if (b < 1) b = 1;
  WSL_DISPATCH_T(dtype, conv_first_kernel<T><<<(int)b, TPB, 0, stream>>>(x, w, bias, (T*)y, N, H, W, stat_partials));
  if (stat_rows_host) *stat_rows_host = (int)b;
  return wsl_check_launch("conv_first");
}

WSL_API int wsl_wgrad_first(const float* x, const void* dy, int dtype, float* dw, int N, int H, int W, int Cout, cudaStream_t stream) {
  WSL_REQUIRE(Cout == 16, "wsl_wgrad_first: compiled for 1 -> 16 channels (got Cout=%d)", Cout);
  long long b = ((long long)N * H * W + 256 * 16 - 1) / (256 * 16);
  if (b > wsl_num_sms()) b = wsl_num_sms();                      // x 2 channel halves x 2 resident blocks per SM = one wave
  if (b < 1) b = 1;
  WSL_DISPATCH_T(dtype, wgrad_first_kernel<T><<<dim3((int)b, 2), 256, 0, stream>>>(x, (const T*)dy, dw, N, H, W));
  return wsl_check_launch("wgrad_first");
}

WSL_API int wsl_pack_conv_weights_batched(const long long* table, int n_entries, long long total_items, int dtype16, cudaStream_t stream) {
  WSL_REQUIRE(n_entries >= 1 && n_entries <= 128, "wsl_pack_conv_weights_batched: 1..128 entries (got %d)", n_entries);
  pack_weights_batched_kernel<<<grid_for(total_items), TPB, 0, stream>>>(table, n_entries, total_items, dtype16 == 2);
  return wsl_check_launch("pack_conv_weights_batched");
}

WSL_API int wsl_bn_finalize(const float* partials, int nrows, long long P, int C, const float* gamma, const float* beta,
                            float* running_mean, float* running_var, long long* num_batches_tracked, float momentum, float eps,
                            float* save, float* ss, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0 && C <= 256, "wsl_bn_finalize: unsupported channel count %d", C);
  bn_finalize_kernel<<<(C + 15) / 16, TPB, 0, stream>>>(partials, nrows, P, C, gamma, beta, running_mean, running_var, num_batches_tracked,
                                            momentum, eps, save, ss);
  return wsl_check_launch("bn_finalize");
}

WSL_API int wsl_bn_stats_ps(const void* y, int dtype, int N, int HW, int C, const float* gamma, const float* beta, float* running_mean,
                            float* running_var, long long* num_batches_tracked, float momentum, float eps, float* save, float* ss, float* ws,
                            cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0 && C <= 256 && TPB % (C / 8) == 0, "wsl_bn_stats_ps: unsupported channel count %d", C);
  WSL_REQUIRE(N > 0 && N <= 65535 && HW > 0, "wsl_bn_stats_ps: bad shape (N=%d, HW=%d)", N, HW);
  long long nblk = ((long long)HW * C + 65535) / 65536;      // ~64 K elements per block
  if (nblk > 32) nblk = 32;
  if (nblk < 1) nblk = 1;
  WSL_REQUIRE((long long)N * nblk * 2 * C <= WSL_WS_FLOATS, "wsl_bn_stats_ps: workspace too small for N=%d, C=%d", N, C);
  WSL_DISPATCH_T(dtype, bn_stats_ps_kernel<T><<<dim3((unsigned)nblk, (unsigned)N), TPB, TPB * 16 * sizeof(float), stream>>>((const T*)y, HW, C, ws));
  if (const int rc = wsl_check_launch("bn_stats_ps")) return rc;
  bn_finalize_ps_kernel<<<(C + TPB - 1) / TPB, TPB, 0, stream>>>(ws, (int)nblk, N, HW, C, gamma, beta, running_mean, running_var,
                                                                 num_batches_tracked, momentum, eps, save, ss);
  return wsl_check_launch("bn_finalize_ps");
}

WSL_API int wsl_bn_act_fwd_ps(const void* y, int dtype, const float* ss, int N, int H, int W, int C, float slope, float drop_p,
                              const uint8_t* mask, unsigned long long seed, const unsigned long long* seed_ptr, void* act,
                              void* pooled, uint8_t* pool_idx, cudaStream_t stream) {
  WSL_REQUIRE(C % 8 == 0, "wsl_bn_act_fwd_ps: C %% 8 != 0");
  WSL_REQUIRE(pooled == nullptr || (H % 2 == 0 && W % 2 == 0), "wsl_bn_act_fwd_ps: pooling needs even H, W");
  WSL_REQUIRE(TPB % (C / 8) == 0 && (long long)N * H * W < (1LL << 31), "wsl_bn_act_fwd_ps: unsupported C=%d or too many pixels", C);
  BnFin fin;
  fin.partials = nullptr; fin.nrows = 0; fin.P = 0; fin.gamma = fin.beta = nullptr; fin.running_mean = fin.running_var = nullptr;
  fin.nbt = nullptr; fin.momentum = 0.f; fin.eps = 0.f; fin.save = fin.ss_out = nullptr;
  const long long items = (long long)N * H * W * (C / 8) / (pooled ? 4 : 1);
  WSL_DISPATCH_T(dtype, (bn_act_fwd_kernel<T, true><<<grid_for((items + 1) / 2), TPB, 0, stream>>>(
                            (const T*)y, ss, N, H, W, C, slope, drop_p, mask, seed, seed_ptr, (T*)act, (T*)pooled, pool_idx, fin)));
  return wsl_check_launch("bn_act_fwd_ps");
}
