// FCDiscriminator (networks/discriminator.py:58-101) around the existing 3x3 tensor-core convolutions.
//
// A 4x4 / stride-2 / pad-1 convolution is a 3x3 / stride-1 / pad-1 convolution over the space-to-depth tensor
//   T[n, Y, X, (a*2 + b)*Cin + c] = x[n, 2Y + a, 2X + b, c]          (a, b in {0, 1}; half resolution, 4*Cin channels)
// with a structured weight: filter tap k (0..3) of an axis lands in 3x3 tap t = (k + 1) >> 1 at phase a = (k + 1) & 1, so each
// of the 16 taps fills one of the 36 (tap, phase) slots and the other 20 are zero.  The zero fill of T's rows / columns -1 and
// H/2 is exactly the padding.  The kernels below are the data movement around that plan: the input packer, the
// LeakyReLU x Dropout2d scale fused with space-to-depth (and its transpose), the weight scatter / gradient gather and the head
// (LeakyReLU -> AvgPool2d(7) -> Linear).  Storage type: dtype 0 = bf16, 1 = fp32.
#include "common.cuh"

namespace {

constexpr int DTPB = 256;

inline int dgrid(long long items) {
  long long b = (items + DTPB - 1) / DTPB;
  if (b < 1) b = 1;
  if (b > wsl_num_sms() * 16) b = wsl_num_sms() * 16;
  return (int)b;
}

__device__ __forceinline__ float ld1(const float* p, long long i) { return p[i]; }
__device__ __forceinline__ float ld1(const __nv_bfloat16* p, long long i) { return __bfloat162float(p[i]); }
__device__ __forceinline__ void st1(float* p, long long i, float v) { p[i] = v; }
__device__ __forceinline__ void st1(__nv_bfloat16* p, long long i, float v) { p[i] = __float2bfloat16_rn(v); }

// 8 consecutive elements (16-byte aligned for bf16, 32-byte for fp32)
__device__ __forceinline__ void ld8v(const float* p, float (&f)[8]) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void ld8v(const __nv_bfloat16* p, float (&f)[8]) { unpack8(*reinterpret_cast<const uint4*>(p), f); }
__device__ __forceinline__ void st8v(float* p, const float (&f)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(f[0], f[1], f[2], f[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(f[4], f[5], f[6], f[7]);
}
__device__ __forceinline__ void st8v(__nv_bfloat16* p, const float (&f)[8]) { *reinterpret_cast<uint4*>(p) = pack8(f); }

// map [N][C0][H][W] and feature [N][C1][H][W] (fp32) -> T [N][H/2][W/2][CP], channel (a*2+b)*(C0+C1) + c, zero above 4*(C0+C1)
template <typename T>
__global__ void __launch_bounds__(DTPB) pack_input_kernel(const float* __restrict__ map, int C0, const float* __restrict__ feat, int C1,
                                                          int N, int H, int W, int CP, T* __restrict__ out) {
  const int h = H >> 1, w = W >> 1, C = C0 + C1;
  const long long total = (long long)N * h * w * CP;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int k = (int)(i % CP);
    const long long pix = i / CP;
    const int X = (int)(pix % w), Y = (int)((pix / w) % h), n = (int)(pix / ((long long)w * h));
    float v = 0.f;
    if (k < 4 * C) {
      const int q = k / C, c = k - q * C;
      const int y = 2 * Y + (q >> 1), x = 2 * X + (q & 1);
      v = c < C0 ? map[(((long long)n * C0 + c) * H + y) * W + x] : feat[(((long long)n * C1 + (c - C0)) * H + y) * W + x];
    }
    st1(out, i, v);
  }
}

// dT [N][H/2][W/2][CP] -> d map [N][C0][H][W], d feature [N][C1][H][W] (fp32; either may be NULL)
template <typename T>
__global__ void __launch_bounds__(DTPB) unpack_input_grad_kernel(const T* __restrict__ dT, int N, int H, int W, int CP, int C0, int C1,
                                                                 float* __restrict__ dmap, float* __restrict__ dfeat) {
  const int C = C0 + C1, h = H >> 1, w = W >> 1;
  const long long total = (long long)N * C * H * W;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const long long nc = i / ((long long)W * H);
    const int c = (int)(nc % C), n = (int)(nc / C);
    const int k = ((y & 1) * 2 + (x & 1)) * C + c;
    const float v = ld1(dT, (((long long)n * h + (y >> 1)) * w + (x >> 1)) * CP + k);
    if (c < C0) {
      if (dmap) dmap[(((long long)n * C0 + c) * H + y) * W + x] = v;
    } else if (dfeat) {
      dfeat[(((long long)n * C1 + (c - C0)) * H + y) * W + x] = v;
    }
  }
}

// y [N][h][w][C] -> T [N][h/2][w/2][4C]: T = LeakyReLU(slope)(y) * cs[n][c] (cs NULL: 1)
template <typename T>
__global__ void __launch_bounds__(DTPB) s2d_act_kernel(const T* __restrict__ y, int N, int h, int w, int C, float slope,
                                                       const float* __restrict__ cs, T* __restrict__ out) {
  const int cg = C >> 3;
  const long long total = (long long)N * h * w * cg;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int c = (int)(i % cg) * 8;
    const long long pix = i / cg;
    const int x = (int)(pix % w), yy = (int)((pix / w) % h), n = (int)(pix / ((long long)w * h));
    float f[8];
    ld8v(y + pix * C + c, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = f[j] > 0.f ? f[j] : f[j] * slope;
      if (cs) v *= cs[(long long)n * C + c + j];
      f[j] = v;
    }
    const long long o = (((long long)n * (h >> 1) + (yy >> 1)) * (w >> 1) + (x >> 1)) * 4 * C + ((yy & 1) * 2 + (x & 1)) * C + c;
    st8v(out + o, f);
  }
}

// dT [N][h/2][w/2][4C] -> dy [N][h][w][C] = depth-to-space(dT) * cs[n][c] * (y > 0 ? 1 : slope)  (y may be NULL when slope == 1)
template <typename T>
__global__ void __launch_bounds__(DTPB) d2s_act_bwd_kernel(const T* __restrict__ dT, const T* __restrict__ y, int N, int h, int w, int C,
                                                           float slope, const float* __restrict__ cs, T* __restrict__ dy) {
  const int cg = C >> 3;
  const long long total = (long long)N * h * w * cg;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int c = (int)(i % cg) * 8;
    const long long pix = i / cg;
    const int x = (int)(pix % w), yy = (int)((pix / w) % h), n = (int)(pix / ((long long)w * h));
    const long long o = (((long long)n * (h >> 1) + (yy >> 1)) * (w >> 1) + (x >> 1)) * 4 * C + ((yy & 1) * 2 + (x & 1)) * C + c;
    float g[8], v[8];
    ld8v(dT + o, g);
    if (y) ld8v(y + pix * C + c, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float r = g[j];
      if (cs) r *= cs[(long long)n * C + c + j];
      if (y && !(v[j] > 0.f)) r *= slope;
      g[j] = r;
    }
    st8v(dy + pix * C + c, g);
  }
}

// 4x4 torch-layout weights w0 [Cout][C0][4][4] (+ w1 [Cout][C1][4][4]) -> structured 3x3 torch layout w3 [Cout][CP][3][3];
// bias_out = b0 (+ b1) when given
__global__ void __launch_bounds__(DTPB) scatter_weights_kernel(const float* __restrict__ w0, const float* __restrict__ b0, int C0,
                                                               const float* __restrict__ w1, const float* __restrict__ b1, int C1,
                                                               int Cout, int CP, float* __restrict__ w3, float* __restrict__ bias_out) {
  const int C = C0 + C1;
  const long long total = (long long)Cout * CP * 9;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int tx = (int)(i % 3), ty = (int)((i / 3) % 3), k = (int)((i / 9) % CP), co = (int)(i / (9LL * CP));
    float v = 0.f;
    if (k < 4 * C) {
      const int q = k / C, c = k - q * C;
      const int ky = 2 * ty + (q >> 1) - 1, kx = 2 * tx + (q & 1) - 1;
      if (ky >= 0 && ky < 4 && kx >= 0 && kx < 4)
        v = c < C0 ? w0[(((long long)co * C0 + c) * 4 + ky) * 4 + kx] : w1[(((long long)co * C1 + (c - C0)) * 4 + ky) * 4 + kx];
    }
    w3[i] = v;
    if (bias_out && i < Cout) bias_out[i] = b0[i] + (b1 ? b1[i] : 0.f);
  }
}

// structured 3x3 weight gradient dw3 [Cout][CP][3][3] -> dw0 [Cout][C0][4][4] (and dw1 [Cout][C1][4][4])
__global__ void __launch_bounds__(DTPB) gather_wgrad_kernel(const float* __restrict__ dw3, int Cout, int CP, int C0, int C1,
                                                            float* __restrict__ dw0, float* __restrict__ dw1) {
  const int C = C0 + C1;
  const long long total = (long long)Cout * C * 16;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int kx = (int)(i & 3), ky = (int)((i >> 2) & 3), c = (int)((i >> 4) % C), co = (int)(i / (16LL * C));
    const int ty = (ky + 1) >> 1, a = (ky + 1) & 1, tx = (kx + 1) >> 1, b = (kx + 1) & 1;
    const float v = dw3[(((long long)co * CP + (a * 2 + b) * C + c) * 3 + ty) * 3 + tx];
    if (c < C0) dw0[(((long long)co * C0 + c) * 4 + ky) * 4 + kx] = v;
    else if (dw1) dw1[(((long long)co * C1 + (c - C0)) * 4 + ky) * 4 + kx] = v;
  }
}

// head forward, part 1: pooled[n][c*4 + i*2 + j] = mean over rows 7i..7i+6, columns 7j..7j+6 of LeakyReLU(y) (16 x 16 map).
// Block (n, 32-channel group): thread t -> channel c = 32*blockIdx.y + (t & 31), quadrant t >> 5; fixed summation order.
template <typename T>
__global__ void __launch_bounds__(128) head_pool_kernel(const T* __restrict__ y, int C, float slope, float* __restrict__ pooled) {
  const int n = blockIdx.x, c = blockIdx.y * 32 + (threadIdx.x & 31), q = threadIdx.x >> 5;
  const int i = q >> 1, j = q & 1;
  if (c >= C) return;
  float s = 0.f;
  for (int r = 0; r < 7; ++r)
    for (int x = 0; x < 7; ++x) {
      const float v = ld1(y, (((long long)n * 16 + 7 * i + r) * 16 + 7 * j + x) * C + c);
      s += v > 0.f ? v : v * slope;
    }
  pooled[(long long)n * 4 * C + c * 4 + q] = s * (1.f / 49.f);
}

// head forward, part 2: logits[n][o] = bc[o] + sum_k wc[o][k] * pooled[n][k], K = 4C (one block per image, fixed order)
__global__ void __launch_bounds__(DTPB) head_linear_kernel(const float* __restrict__ pooled, int K, const float* __restrict__ wc,
                                                           const float* __restrict__ bc, float* __restrict__ logits) {
  __shared__ float s_red[2][DTPB / 32];
  const int n = blockIdx.x;
  float a0 = 0.f, a1 = 0.f;
  for (int k = threadIdx.x; k < K; k += DTPB) {
    const float p = pooled[(long long)n * K + k];
    a0 = fmaf(wc[k], p, a0);
    a1 = fmaf(wc[K + k], p, a1);
  }
  a0 = warp_sum(a0);
  a1 = warp_sum(a1);
  if ((threadIdx.x & 31) == 0) { s_red[0][threadIdx.x >> 5] = a0; s_red[1][threadIdx.x >> 5] = a1; }
  __syncthreads();
  if (threadIdx.x < 2) {
    float s = 0.f;
    for (int wv = 0; wv < DTPB / 32; ++wv) s += s_red[threadIdx.x][wv];
    logits[n * 2 + threadIdx.x] = s + bc[threadIdx.x];
  }
}

// head backward: dy[n][y][x][c] = (y, x < 14) ? (sum_o dl[n][o] wc[o][c*4 + (y/7)*2 + x/7]) / 49 * LeakyReLU'(y) : 0
template <typename T>
__global__ void __launch_bounds__(DTPB) head_bwd_act_kernel(const float* __restrict__ dl, const T* __restrict__ y, int N, int C, float slope,
                                                            const float* __restrict__ wc, T* __restrict__ dy) {
  const long long total = (long long)N * 256 * C;
  const int K = 4 * C;
  for (long long i = blockIdx.x * (long long)DTPB + threadIdx.x; i < total; i += (long long)gridDim.x * DTPB) {
    const int c = (int)(i % C);
    const int pix = (int)((i / C) % 256), n = (int)(i / (256LL * C));
    const int yy = pix >> 4, x = pix & 15;
    float g = 0.f;
    if (yy < 14 && x < 14) {
      const int k = c * 4 + (yy / 7) * 2 + x / 7;
      g = (dl[2 * n] * wc[k] + dl[2 * n + 1] * wc[K + k]) * (1.f / 49.f);
      if (!(ld1(y, i) > 0.f)) g *= slope;
    }
    st1(dy, i, g);
  }
}

// classifier gradients: dwc[o][k] = sum_n dl[n][o] pooled[n][k], dbc[o] = sum_n dl[n][o] (batch order, deterministic)
__global__ void __launch_bounds__(DTPB) head_bwd_param_kernel(const float* __restrict__ dl, const float* __restrict__ pooled, int N, int K,
                                                              float* __restrict__ dwc, float* __restrict__ dbc) {
  const int i = blockIdx.x * DTPB + threadIdx.x;
  if (i < 2 * K) {
    const int o = i / K, k = i - o * K;
    float s = 0.f;
    for (int n = 0; n < N; ++n) s = fmaf(dl[2 * n + o], pooled[(long long)n * K + k], s);
    dwc[i] = s;
  } else if (i < 2 * K + 2) {
    const int o = i - 2 * K;
    float s = 0.f;
    for (int n = 0; n < N; ++n) s += dl[2 * n + o];
    dbc[o] = s;
  }
}

// 2-class cross entropy of logits [N][2] against targets 1 for rows < n_ones, 0 after (one warp, fixed summation order):
// loss[0] = mean NLL; dl[n][c] = (softmax - onehot) * weight / N with weight = *weight_ptr when given
__global__ void __launch_bounds__(32) disc_ce_kernel(const float* __restrict__ logits, int N, int n_ones, const float* weight_ptr,
                                                     float weight, float* __restrict__ loss, float* __restrict__ dl) {
  const float w = (weight_ptr ? *weight_ptr : weight) / (float)N;
  float s = 0.f;
  for (int n = threadIdx.x; n < N; n += 32) {
    const float z0 = logits[2 * n], z1 = logits[2 * n + 1];
    const float m = fmaxf(z0, z1);
    const float e0 = expf(z0 - m), e1 = expf(z1 - m), se = e0 + e1;
    const int t = n < n_ones ? 1 : 0;
    s += logf(se) - ((t ? z1 : z0) - m);
    dl[2 * n] = (e0 / se - (t ? 0.f : 1.f)) * w;
    dl[2 * n + 1] = (e1 / se - (t ? 1.f : 0.f)) * w;
  }
  s = warp_sum(s);
  if (threadIdx.x == 0) loss[0] = s / (float)N;
}

}  // namespace

#define WSL_DISC_T(dtype, ...)                                   \
  do {                                                           \
    if ((dtype) == 1) { using T = float; __VA_ARGS__; }          \
    else { using T = __nv_bfloat16; __VA_ARGS__; }               \
  } while (0)

#define WSL_DISC_DTYPE(fn, dtype) WSL_REQUIRE((dtype) == 0 || (dtype) == 1, fn ": dtype must be 0 (bf16) or 1 (fp32), got %d", (dtype))

WSL_API int wsl_disc_pack_input(const float* map, int C0, const float* feature, int C1, int N, int H, int W, int CP, void* out, int dtype,
                                cudaStream_t stream) {
  WSL_DISC_DTYPE("wsl_disc_pack_input", dtype);
  WSL_REQUIRE(H % 2 == 0 && W % 2 == 0 && CP >= 4 * (C0 + C1) && C0 > 0 && C1 >= 0, "wsl_disc_pack_input: bad shape");
  const long long items = (long long)N * (H / 2) * (W / 2) * CP;
  WSL_DISC_T(dtype, pack_input_kernel<T><<<dgrid(items), DTPB, 0, stream>>>(map, C0, feature, C1, N, H, W, CP, (T*)out));
  return wsl_check_launch("disc_pack_input");
}

WSL_API int wsl_disc_unpack_input_grad(const void* dT, int dtype, int N, int H, int W, int CP, int C0, int C1, float* dmap, float* dfeature,
                                       cudaStream_t stream) {
  WSL_DISC_DTYPE("wsl_disc_unpack_input_grad", dtype);
  WSL_REQUIRE(H % 2 == 0 && W % 2 == 0 && CP >= 4 * (C0 + C1), "wsl_disc_unpack_input_grad: bad shape");
  const long long items = (long long)N * (C0 + C1) * H * W;
  WSL_DISC_T(dtype, unpack_input_grad_kernel<T><<<dgrid(items), DTPB, 0, stream>>>((const T*)dT, N, H, W, CP, C0, C1, dmap, dfeature));
  return wsl_check_launch("disc_unpack_input_grad");
}

WSL_API int wsl_s2d_act_fwd(const void* y, int dtype, int N, int H, int W, int C, float slope, const float* cs, void* out,
                            cudaStream_t stream) {
  WSL_DISC_DTYPE("wsl_s2d_act_fwd", dtype);
  WSL_REQUIRE(C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "wsl_s2d_act_fwd: needs C %% 8 == 0 and even H, W (got C=%d, %dx%d)", C, H, W);
  WSL_DISC_T(dtype, s2d_act_kernel<T><<<dgrid((long long)N * H * W * (C / 8)), DTPB, 0, stream>>>((const T*)y, N, H, W, C, slope, cs, (T*)out));
  return wsl_check_launch("s2d_act_fwd");
}

WSL_API int wsl_d2s_act_bwd(const void* dT, const void* y, int dtype, int N, int H, int W, int C, float slope, const float* cs, void* dy,
                            cudaStream_t stream) {
  WSL_DISC_DTYPE("wsl_d2s_act_bwd", dtype);
  WSL_REQUIRE(C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "wsl_d2s_act_bwd: needs C %% 8 == 0 and even H, W (got C=%d, %dx%d)", C, H, W);
  WSL_REQUIRE(y != nullptr || slope == 1.f, "wsl_d2s_act_bwd: the pre-activation is required unless slope == 1");
  WSL_DISC_T(dtype, d2s_act_bwd_kernel<T><<<dgrid((long long)N * H * W * (C / 8)), DTPB, 0, stream>>>((const T*)dT, (const T*)y, N, H, W, C,
                                                                                                    slope, cs, (T*)dy));
  return wsl_check_launch("d2s_act_bwd");
}

WSL_API int wsl_disc_scatter_weights(const float* w0, const float* b0, int C0, const float* w1, const float* b1, int C1, int Cout, int CP,
                                     float* w3, float* bias_out, cudaStream_t stream) {
  WSL_REQUIRE(CP >= 4 * (C0 + C1) && C0 > 0 && (C1 == 0 || w1 != nullptr), "wsl_disc_scatter_weights: bad shape");
  WSL_REQUIRE(bias_out == nullptr || b0 != nullptr, "wsl_disc_scatter_weights: bias_out needs b0");
  scatter_weights_kernel<<<dgrid((long long)Cout * CP * 9), DTPB, 0, stream>>>(w0, b0, C0, w1, b1, C1, Cout, CP, w3, bias_out);
  return wsl_check_launch("disc_scatter_weights");
}

WSL_API int wsl_disc_gather_wgrad(const float* dw3, int Cout, int CP, int C0, int C1, float* dw0, float* dw1, cudaStream_t stream) {
  WSL_REQUIRE(CP >= 4 * (C0 + C1) && C0 > 0 && (C1 == 0 || dw1 != nullptr), "wsl_disc_gather_wgrad: bad shape");
  gather_wgrad_kernel<<<dgrid((long long)Cout * (C0 + C1) * 16), DTPB, 0, stream>>>(dw3, Cout, CP, C0, C1, dw0, dw1);
  return wsl_check_launch("disc_gather_wgrad");
}

WSL_API int wsl_disc_head_fwd(const void* y, int dtype, int N, int C, float slope, const float* wc, const float* bc, float* pooled,
                              float* logits, cudaStream_t stream) {
  WSL_DISC_DTYPE("wsl_disc_head_fwd", dtype);
  WSL_REQUIRE(C % 32 == 0 && N > 0, "wsl_disc_head_fwd: C must be a multiple of 32 (got %d)", C);
  WSL_DISC_T(dtype, head_pool_kernel<T><<<dim3(N, C / 32), 128, 0, stream>>>((const T*)y, C, slope, pooled));
  int rc = wsl_check_launch("disc_head_pool");
  if (rc) return rc;
  head_linear_kernel<<<N, DTPB, 0, stream>>>(pooled, 4 * C, wc, bc, logits);
  return wsl_check_launch("disc_head_linear");
}

WSL_API int wsl_disc_head_bwd(const float* dlogits, const float* pooled, const void* y, int dtype, int N, int C, float slope, const float* wc,
                              float* dwc, float* dbc, void* dy, cudaStream_t stream) {
  WSL_DISC_DTYPE("wsl_disc_head_bwd", dtype);
  WSL_REQUIRE(C % 8 == 0 && N > 0, "wsl_disc_head_bwd: bad channel count %d", C);
  WSL_DISC_T(dtype, head_bwd_act_kernel<T><<<dgrid((long long)N * 256 * C), DTPB, 0, stream>>>(dlogits, (const T*)y, N, C, slope, wc, (T*)dy));
  int rc = wsl_check_launch("disc_head_bwd_act");
  if (rc) return rc;
  WSL_REQUIRE((dwc == nullptr) == (dbc == nullptr), "wsl_disc_head_bwd: dwc and dbc are both given or both NULL");
  if (dwc == nullptr) return 0;                    // map gradient only: no classifier gradients
  head_bwd_param_kernel<<<(8 * C + 2 + DTPB - 1) / DTPB, DTPB, 0, stream>>>(dlogits, pooled, N, 4 * C, dwc, dbc);
  return wsl_check_launch("disc_head_bwd_param");
}

WSL_API int wsl_disc_ce(const float* logits, int N, int n_ones, const float* weight_ptr, float weight, float* loss, float* dlogits,
                        cudaStream_t stream) {
  WSL_REQUIRE(N > 0 && n_ones >= 0 && n_ones <= N, "wsl_disc_ce: bad N=%d / n_ones=%d", N, n_ones);
  disc_ce_kernel<<<1, 32, 0, stream>>>(logits, N, n_ones, weight_ptr, weight, loss, dlogits);
  return wsl_check_launch("disc_ce");
}
