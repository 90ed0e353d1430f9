// Random-walker pseudo labels from scribbles (dataloaders/acdc_pseudo_label_random_walker.py:9-26, i.e. skimage's
// random_walker(rescale_intensity(image, (-0.35, 1.35), (-1, 1)), markers, beta=100, mode='bf') per slice) for a whole ragged
// slice store in one launch.
//
// One persistent CTA owns one slice at a time: it takes the next slice id from an atomic work counter (the caller orders the
// ids by descending pixel count, so the last wave is short), builds the 4-neighbour edge weights in its workspace slot and runs
// Jacobi-preconditioned conjugate gradients on the Laplacian system L_UU x_l = -L_UM m_l of all label columns at once (one
// float4 per pixel, column l in component l) until max_l ||r_l|| / ||b_l|| <= tol, with no host round trip.  Vectors are fp32;
// every dot product is accumulated in fp64 per thread in a fixed pixel order and combined in a fixed warp / block order, so a
// slice's result is bit-identical run to run and does not depend on which CTA solved it or which slices shared the launch.
//
// Matrix-free form: seeds are not unknowns.  Their x / r / p entries stay 0, so the stencil sum over all neighbours is the sum
// over unknown neighbours; deg_i (over ALL incident edges) is the diagonal of L_UU, and the right-hand side of an unknown pixel is
// the sum of the weights of its edges to seeds, put in the seed's label column.
#include "common.cuh"

namespace {

constexpr int RW_TPB = 512;
constexpr int RW_WARPS = RW_TPB / 32;
constexpr long long RW_HEADER_FLOATS = 64;       // [0]: the work counter (reset by the launcher)
constexpr int RW_FLOATS_PER_PX = 4 * 4 + 3;      // x, r, p, Ap (float4) + right / down edge weight + degree

__host__ __device__ inline long long rw_slot_stride(long long slot_px) {
  const long long p = (slot_px + 63) / 64 * 64;
  return p * RW_FLOATS_PER_PX;
}

// sum of K per-thread fp64 values over the block, fixed order; result in out[0..K) (shared) for every thread on return
template <int K>
__device__ __forceinline__ void rw_block_sum(double (&v)[K], double (*red)[K], double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double r = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    if (lane == 0) red[warp][k] = r;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double r = 0.0;
    for (int w = 0; w < RW_WARPS; ++w) r += red[w][threadIdx.x];
    out[threadIdx.x] = r;
  }
  __syncthreads();
}

__device__ __forceinline__ double rw_rescale(float v) {      // rescale_intensity(in_range=(-0.35, 1.35), out_range=(-1, 1))
  double d = (double)v;
  d = d < -0.35 ? -0.35 : (d > 1.35 ? 1.35 : d);
  return (d + 0.35) / 1.7 * 2.0 - 1.0;
}

__device__ __forceinline__ float comp(const float4& v, int l) { return l == 0 ? v.x : (l == 1 ? v.y : (l == 2 ? v.z : v.w)); }

__global__ void __launch_bounds__(RW_TPB, 2) random_walker_kernel(
    const float* __restrict__ images, const uint8_t* __restrict__ scribbles, const long long* __restrict__ offs,
    const int* __restrict__ shapes, const int* __restrict__ order, int n_slices, float beta, float tol, int max_iter,
    float* __restrict__ ws, long long slot_px, uint8_t* __restrict__ labels, float4* __restrict__ probs, int* __restrict__ iters,
    float* __restrict__ resid) {
  __shared__ double red[RW_WARPS][8];
  __shared__ double sh[8];
  __shared__ double s_alpha[4], s_beta[4], s_rz[4], s_bn[4];
  __shared__ double s_res;
  __shared__ int s_job, s_present;
  __shared__ uint8_t s_remap[5];
  __shared__ int s_K;
  unsigned* counter = reinterpret_cast<unsigned*>(ws);
  float* slot = ws + RW_HEADER_FLOATS + (long long)blockIdx.x * rw_slot_stride(slot_px);
  const long long P4 = (slot_px + 63) / 64 * 64;
  float4* X = reinterpret_cast<float4*>(slot);
  float4* R = X + P4;
  float4* Pv = R + P4;
  float4* AP = Pv + P4;
  float* WR = reinterpret_cast<float*>(AP + P4);
  float* WD = WR + P4;
  float* DEG = WD + P4;
  const int tid = threadIdx.x;

  for (;;) {
    if (tid == 0) { s_job = (int)atomicAdd(counter, 1u); s_present = 0; }
    __syncthreads();
    const int job = s_job;
    if (job >= n_slices) break;
    const int sl = order[job];
    const int h = shapes[2 * sl], w = shapes[2 * sl + 1];
    const long long P = (long long)h * w, off = offs[sl];
    const float* img = images + off;
    const uint8_t* scr = scribbles + off;
    if (P > slot_px) {                           // the caller sized the workspace for smaller slices: report, solve nothing
      if (tid == 0) { iters[sl] = -1; resid[sl] = __int_as_float(0x7fc00000); }
      __syncthreads();
      continue;
    }
    // ---- prologue: class presence, fp64 mean / std of the rescaled slice ----
    int present = 0;
    double acc1[1] = {0.0};
    for (long long i = tid; i < P; i += RW_TPB) {
      const int s = scr[i];
      if (s < 4) present |= 1 << s;
      acc1[0] += rw_rescale(img[i]);
    }
    present = __reduce_or_sync(0xffffffffu, present);
    if ((tid & 31) == 0) atomicOr(&s_present, present);
    rw_block_sum<1>(acc1, reinterpret_cast<double (*)[1]>(red), sh);
    const double mean = sh[0] / (double)P;
    const int pres = s_present;
    if ((pres & 0xE) != 0xE) {                   // a class of 1, 2, 3 has no scribble: the pseudo label is all zeros (:12-13)
      for (long long i = tid; i < P; i += RW_TPB) {
        labels[off + i] = 0;
        if (probs) probs[off + i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (tid == 0) { iters[sl] = 0; resid[sl] = 0.f; }
      __syncthreads();
      continue;
    }
    double acc2[1] = {0.0};
    for (long long i = tid; i < P; i += RW_TPB) {
      const double dv = rw_rescale(img[i]) - mean;
      acc2[0] += dv * dv;
    }
    rw_block_sum<1>(acc2, reinterpret_cast<double (*)[1]>(red), sh);
    if (tid == 0) {
      // markers 1..4 of the present classes renumbered by rank (skimage relabels non-consecutive markers and keeps the relabelled
      // output, DESIGN F17): without a background scribble, classes 1..3 become labels 0..2
      int k = 0;
      for (int c = 0; c < 4; ++c) s_remap[c] = (pres >> c & 1) ? (uint8_t)k++ : (uint8_t)0;
      s_remap[4] = 0;
      s_K = k;
    }
    const double sd = sqrt(sh[0] / (double)P);
    const double scale = sd > 0.0 ? -(double)beta / (10.0 * sd) : 0.0;    // a constant slice has no contrast: uniform weights
    __syncthreads();
    // ---- edge weights w = exp(scale * (d_i - d_j)^2) + 1e-10 (skimage _compute_weights_3d, eps 1e-10) ----
    for (long long i = tid; i < P; i += RW_TPB) {
      const int y = (int)(i / w), x = (int)(i - (long long)y * w);
      const double di = rw_rescale(img[i]);
      float wr = 0.f, wd = 0.f;
      if (x + 1 < w) { const double g = di - rw_rescale(img[i + 1]); wr = (float)(exp(scale * g * g) + 1e-10); }
      if (y + 1 < h) { const double g = di - rw_rescale(img[i + w]); wd = (float)(exp(scale * g * g) + 1e-10); }
      WR[i] = wr;
      WD[i] = wd;
    }
    __syncthreads();
    // ---- degree (0 marks a seed), right-hand side, x = 0, r = b, p = z = D^-1 r ----
    double acc8[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (long long i = tid; i < P; i += RW_TPB) {
      const int y = (int)(i / w), x = (int)(i - (long long)y * w);
      const bool seed = scr[i] < 4;
      float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
      float deg = 0.f;
      if (!seed) {
        const float wn[4] = {WR[i], x > 0 ? WR[i - 1] : 0.f, WD[i], y > 0 ? WD[i - w] : 0.f};
        const long long nj[4] = {i + 1, i - 1, i + w, i - w};
        float bb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (wn[e] == 0.f) continue;            // no neighbour on this side
          deg += wn[e];
          const int sj = scr[nj[e]];
          if (sj < 4) bb[s_remap[sj]] += wn[e];
        }
        b = make_float4(bb[0], bb[1], bb[2], bb[3]);
      }
      DEG[i] = deg;
      const float inv = seed ? 0.f : 1.0f / deg;
      const float4 z = make_float4(b.x * inv, b.y * inv, b.z * inv, b.w * inv);
      X[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      R[i] = b;
      Pv[i] = z;
      acc8[0] += (double)b.x * z.x; acc8[1] += (double)b.y * z.y; acc8[2] += (double)b.z * z.z; acc8[3] += (double)b.w * z.w;
      acc8[4] += (double)b.x * b.x; acc8[5] += (double)b.y * b.y; acc8[6] += (double)b.z * b.z; acc8[7] += (double)b.w * b.w;
    }
    rw_block_sum<8>(acc8, red, sh);
    if (tid < 4) { s_rz[tid] = sh[tid]; s_bn[tid] = sqrt(sh[4 + tid]); }
    if (tid == 0) s_res = 0.0;
    __syncthreads();
    if (tid == 0) {
      double res = 0.0;
      for (int l = 0; l < 4; ++l) if (s_bn[l] > 0.0) res = fmax(res, 1.0);     // r = b at the start
      s_res = res;
    }
    __syncthreads();
    int it = 0;
    while (s_res > (double)tol && it < max_iter) {
      // Ap = L_UU p and p.Ap per column
      double a4[4] = {0.0, 0.0, 0.0, 0.0};
      for (long long i = tid; i < P; i += RW_TPB) {
        const float deg = DEG[i];
        float4 ap = make_float4(0.f, 0.f, 0.f, 0.f);
        if (deg != 0.f) {
          const int y = (int)(i / w), x = (int)(i - (long long)y * w);
          const float4 pi = Pv[i];
          float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
          const float w0 = WR[i];
          if (x + 1 < w) { const float4 q = Pv[i + 1]; s.x += w0 * q.x; s.y += w0 * q.y; s.z += w0 * q.z; s.w += w0 * q.w; }
          if (x > 0) { const float w1 = WR[i - 1]; const float4 q = Pv[i - 1]; s.x += w1 * q.x; s.y += w1 * q.y; s.z += w1 * q.z; s.w += w1 * q.w; }
          const float w2 = WD[i];
          if (y + 1 < h) { const float4 q = Pv[i + w]; s.x += w2 * q.x; s.y += w2 * q.y; s.z += w2 * q.z; s.w += w2 * q.w; }
          if (y > 0) { const float w3 = WD[i - w]; const float4 q = Pv[i - w]; s.x += w3 * q.x; s.y += w3 * q.y; s.z += w3 * q.z; s.w += w3 * q.w; }
          ap = make_float4(deg * pi.x - s.x, deg * pi.y - s.y, deg * pi.z - s.z, deg * pi.w - s.w);
          a4[0] += (double)pi.x * ap.x; a4[1] += (double)pi.y * ap.y; a4[2] += (double)pi.z * ap.z; a4[3] += (double)pi.w * ap.w;
        }
        AP[i] = ap;
      }
      rw_block_sum<4>(a4, reinterpret_cast<double (*)[4]>(red), sh);
      if (tid < 4) s_alpha[tid] = sh[tid] > 0.0 ? s_rz[tid] / sh[tid] : 0.0;
      __syncthreads();
      const float al[4] = {(float)s_alpha[0], (float)s_alpha[1], (float)s_alpha[2], (float)s_alpha[3]};
      // x += alpha p, r -= alpha Ap, r.z and r.r per column
      for (int k = 0; k < 8; ++k) acc8[k] = 0.0;
      for (long long i = tid; i < P; i += RW_TPB) {
        const float deg = DEG[i];
        if (deg == 0.f) continue;
        const float4 p = Pv[i], ap = AP[i];
        float4 x = X[i], r = R[i];
        x.x += al[0] * p.x; x.y += al[1] * p.y; x.z += al[2] * p.z; x.w += al[3] * p.w;
        r.x -= al[0] * ap.x; r.y -= al[1] * ap.y; r.z -= al[2] * ap.z; r.w -= al[3] * ap.w;
        X[i] = x;
        R[i] = r;
        const float inv = 1.0f / deg;
        acc8[0] += (double)r.x * (r.x * inv); acc8[1] += (double)r.y * (r.y * inv);
        acc8[2] += (double)r.z * (r.z * inv); acc8[3] += (double)r.w * (r.w * inv);
        acc8[4] += (double)r.x * r.x; acc8[5] += (double)r.y * r.y; acc8[6] += (double)r.z * r.z; acc8[7] += (double)r.w * r.w;
      }
      rw_block_sum<8>(acc8, red, sh);
      if (tid < 4) {
        s_beta[tid] = s_rz[tid] > 0.0 ? sh[tid] / s_rz[tid] : 0.0;
        s_rz[tid] = sh[tid];
      }
      if (tid == 0) {
        double res = 0.0;
        for (int l = 0; l < 4; ++l) if (s_bn[l] > 0.0) res = fmax(res, sqrt(sh[4 + l]) / s_bn[l]);
        s_res = res;
      }
      __syncthreads();
      ++it;
      if (s_res <= (double)tol) break;
      const float be[4] = {(float)s_beta[0], (float)s_beta[1], (float)s_beta[2], (float)s_beta[3]};
      // p = D^-1 r + beta p
      for (long long i = tid; i < P; i += RW_TPB) {
        const float deg = DEG[i];
        if (deg == 0.f) continue;
        const float inv = 1.0f / deg;
        const float4 r = R[i];
        float4 p = Pv[i];
        p.x = r.x * inv + be[0] * p.x; p.y = r.y * inv + be[1] * p.y; p.z = r.z * inv + be[2] * p.z; p.w = r.w * inv + be[3] * p.w;
        Pv[i] = p;
      }
      __syncthreads();
    }
    // ---- epilogue: label = argmax over the K label columns (first maximum wins, as np.argmax); seeds keep their marker ----
    const int K = s_K;
    for (long long i = tid; i < P; i += RW_TPB) {
      const int s = scr[i];
      float4 pr;
      uint8_t lab;
      if (s < 4) {
        lab = s_remap[s];
        pr = make_float4(lab == 0, lab == 1, lab == 2, lab == 3);
      } else {
        pr = X[i];
        lab = 0;
        float best = pr.x;
        for (int l = 1; l < K; ++l) if (comp(pr, l) > best) { best = comp(pr, l); lab = (uint8_t)l; }
      }
      labels[off + i] = lab;
      if (probs) probs[off + i] = pr;
    }
    if (tid == 0) { iters[sl] = it; resid[sl] = (float)s_res; }
    __syncthreads();
  }
}

int rw_resident_ctas() {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, random_walker_kernel, RW_TPB, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  return per_sm * wsl_num_sms();
}

}  // namespace

WSL_API int wsl_random_walker_workspace(int ctas, long long max_px, long long* out2) {
  WSL_REQUIRE(out2 != nullptr && max_px > 0, "wsl_random_walker_workspace: out2 must be given and max_px > 0");
  if (ctas <= 0) ctas = rw_resident_ctas();
  out2[0] = ctas;
  out2[1] = RW_HEADER_FLOATS + (long long)ctas * rw_slot_stride(max_px);
  return 0;
}

WSL_API int wsl_random_walker(const float* images, const uint8_t* scribbles, const long long* offs, const int* shapes, const int* order,
                              int n_slices, float beta, float tol, int max_iter, float* ws, int ctas, long long slot_px, uint8_t* labels,
                              float* probs, int* iters, float* resid, cudaStream_t stream) {
  WSL_REQUIRE(n_slices > 0 && ctas > 0 && slot_px > 0 && max_iter >= 0, "wsl_random_walker: empty launch (n_slices=%d, ctas=%d)", n_slices, ctas);
  WSL_REQUIRE(((uintptr_t)ws & 15) == 0 && ((uintptr_t)probs & 15) == 0, "wsl_random_walker: workspace and probabilities must be 16-byte aligned");
  WSL_REQUIRE(beta > 0.f && tol >= 0.f, "wsl_random_walker: beta must be > 0 and tol >= 0");
  if (cudaMemsetAsync(ws, 0, sizeof(unsigned), stream) != cudaSuccess) return wsl_check_launch("random_walker counter reset");
  random_walker_kernel<<<ctas, RW_TPB, 0, stream>>>(images, scribbles, offs, shapes, order, n_slices, beta, tol, max_iter, ws, slot_px,
                                                    labels, reinterpret_cast<float4*>(probs), iters, resid);
  return wsl_check_launch("random_walker");
}
