// Surface-distance metrics of label volumes (medpy.metric.binary's dc / jc / hd95 / asd and its __surface_distances with
// voxelspacing and connectivity 1, as val_2D.py:7-15, test_2D_fully.py:74-80 and utils/metrics.py:19-25 call them) for every
// foreground class of a [S,H,W] (rank 3) or [H,W] (rank 2) pair of uint8 label maps.
//
// Per call: one pass marks the surface voxels of both maps (a mask voxel whose face neighbour is outside the mask or outside the
// array: mask ^ binary_erosion(mask, generate_binary_structure(ndim, 1)) with border_value 0) and counts the overlaps.  Then per
// class, the exact anisotropic Euclidean distance transform of ~surface (scipy's distance_transform_edt(~border, sampling)) is
// built separably for both surfaces at once:
//   z: distance to the nearest feature of the column, f1 = (dz*sz)^2;
//   y: f2(y) = min_j f1(j) + ((y-j)*sy)^2, one thread per voxel scanning outwards from y until (r*sy)^2 >= best (an x-plane
//      without features is +inf throughout);
//   x: d^2 = min_j f2(j) + ((x-j)*sx)^2 the same way, only at the query voxels (the other map's surface).
// Every product and sum is rounded separately (no FMA contraction) in scipy's order, ((dz*sz)^2 + (dy*sy)^2) + (dx*sx)^2, so the
// minimum equals scipy's value at its nearest feature: exactly for integer spacings, to an ulp of near-ties otherwise.
// The two order statistics np.percentile(.., 95) interpolates are found by an 8-pass radix select on the fp64 bit patterns
// (distances are >= 0, so the bits order like the values).  Sums are taken in a fixed order: results are bit-identical run to run.
// A class whose prediction or label is empty has no distances: its kernels return at once and its distance fields stay 0.
#include "common.cuh"

#include <math.h>

#include <algorithm>

namespace {

constexpr int SM_TPB = 256;
constexpr int SM_XTPB = 128;
constexpr int SM_MAX_CLASSES = 16;
constexpr int SM_OUT = 12;                       // doubles per class in `out`, see the header
constexpr int SM_MAX_W = 4096;                   // one x-row of fp64 in shared memory
constexpr int SM_RADIX_PASSES = 8;
constexpr size_t SM_HEADER_BYTES = 4096;
constexpr size_t SM_ZEROED_BYTES = SM_HEADER_BYTES + 2 * SM_MAX_W;  // header + per-x-plane feature flags

struct SmHeader {                                // ws[0..4096): zeroed at the start of every call
  unsigned long long cnt[SM_MAX_CLASSES][5];     // |P&G|, |P|, |G|, #pred-surface, #gt-surface voxels per class
  unsigned long long prefix[2], rank[2];         // radix-select state of the two order statistics
  unsigned int hist[2][256];
  unsigned int ticket;
};
static_assert(sizeof(SmHeader) <= SM_HEADER_BYTES, "surface-metrics header too large");

struct SmLayout {
  long long n, rows;
  size_t plane, surf, f1, f2, part, total;
};

inline size_t sm_align(size_t b) { return (b + 255) / 256 * 256; }

SmLayout sm_layout(int S, int H, int W) {
  SmLayout l;
  l.n = (long long)S * H * W;
  l.rows = (long long)S * H;
  size_t off = SM_HEADER_BYTES;
  l.plane = off; off += 2 * SM_MAX_W;                                // set * SM_MAX_W + x: == c when plane x has a feature
  l.surf = off; off += sm_align((size_t)l.n);                      // pred-surface class | gt-surface class << 4
  l.f1 = off;   off += sm_align(2 * (size_t)l.n * sizeof(double));  // z pass, then the distances at the query voxels
  l.f2 = off;   off += sm_align(2 * (size_t)l.n * sizeof(double));  // y pass
  l.part = off; off += sm_align(2 * (size_t)l.rows * 2 * sizeof(double));  // per (set, x-row): {sum, max}
  l.total = off;
  return l;
}

__device__ __forceinline__ double sm_inf() { return __longlong_as_double(0x7ff0000000000000LL); }
__device__ __forceinline__ double sm_sq(double d, double s) { const double t = __dmul_rn(d, s); return __dmul_rn(t, t); }

__device__ __forceinline__ bool sm_on_surface(const uint8_t* __restrict__ lab, long long v, int c, int x, int y, int z, int S, int H,
                                              int W, long long HW, int rank3) {
  if (x == 0 || x == W - 1 || y == 0 || y == H - 1) return true;
  if (lab[v - 1] != c || lab[v + 1] != c || lab[v - W] != c || lab[v + W] != c) return true;
  if (rank3) {
    if (z == 0 || z == S - 1) return true;
    if (lab[v - HW] != c || lab[v + HW] != c) return true;
  }
  return false;
}

__global__ void __launch_bounds__(SM_TPB) sm_surface_kernel(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ gt, int rank3,
                                                            int S, int H, int W, int classes, uint8_t* __restrict__ surf,
                                                            SmHeader* __restrict__ hdr) {
  __shared__ unsigned cnt[SM_MAX_CLASSES][5];
  for (int i = threadIdx.x; i < SM_MAX_CLASSES * 5; i += blockDim.x) (&cnt[0][0])[i] = 0u;
  __syncthreads();
  const long long HW = (long long)H * W, n = HW * S;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(v % W), y = (int)((v / W) % H), z = (int)(v / HW);
    const int p = pred[v], g = gt[v];
    int ps = 0, gs = 0;
    if (p > 0 && p < classes) {
      atomicAdd(&cnt[p][1], 1u);
      if (sm_on_surface(pred, v, p, x, y, z, S, H, W, HW, rank3)) { ps = p; atomicAdd(&cnt[p][3], 1u); }
      if (g == p) atomicAdd(&cnt[p][0], 1u);
    }
    if (g > 0 && g < classes) {
      atomicAdd(&cnt[g][2], 1u);
      if (sm_on_surface(gt, v, g, x, y, z, S, H, W, HW, rank3)) { gs = g; atomicAdd(&cnt[g][4], 1u); }
    }
    surf[v] = (uint8_t)(ps | (gs << 4));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SM_MAX_CLASSES * 5; i += blockDim.x) {
    const unsigned k = (&cnt[0][0])[i];
    if (k) atomicAdd(&hdr->cnt[0][0] + i, (unsigned long long)k);
  }
}

// Set 0: features = gt surface of class c (its distances are read at the pred surface: pred -> gt); set 1 the other way round.
__device__ __forceinline__ bool sm_is_feature(uint8_t s, int set, int c) { return ((set == 0 ? s >> 4 : s & 15)) == c; }
__device__ __forceinline__ bool sm_is_query(uint8_t s, int set, int c) { return ((set == 0 ? s & 15 : s >> 4)) == c; }
__device__ __forceinline__ bool sm_class_empty(const SmHeader* hdr, int c) { return hdr->cnt[c][3] == 0ull || hdr->cnt[c][4] == 0ull; }

__global__ void __launch_bounds__(SM_XTPB) sm_edt_z_kernel(const uint8_t* __restrict__ surf, int c, int S, long long HW, int W, double sz,
                                                           const SmHeader* __restrict__ hdr, uint8_t* __restrict__ plane,
                                                           double* __restrict__ f1) {
  const long long col = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (col >= HW || sm_class_empty(hdr, c)) return;
  const int set = blockIdx.y;
  double* f = f1 + set * (long long)S * HW + col;
  const uint8_t* s = surf + col;
  int last = -1;
  for (int z = 0; z < S; ++z) {                   // distance to the nearest feature at or before z (-1: none)
    if (sm_is_feature(s[z * HW], set, c)) last = z;
    f[z * HW] = last < 0 ? -1.0 : (double)(z - last);
  }
  int next = -1;
  for (int z = S - 1; z >= 0; --z) {
    if (sm_is_feature(s[z * HW], set, c)) next = z;
    double d = f[z * HW];
    if (next >= 0 && (d < 0.0 || (double)(next - z) < d)) d = (double)(next - z);
    f[z * HW] = d < 0.0 ? sm_inf() : sm_sq(d, sz);
  }
  if (next >= 0) plane[set * SM_MAX_W + col % W] = (uint8_t)c;
}

__global__ void __launch_bounds__(SM_XTPB) sm_edt_y_kernel(const double* __restrict__ f1, const uint8_t* __restrict__ plane, int c,
                                                           long long n, int H, int W, double sy, const SmHeader* __restrict__ hdr,
                                                           double* __restrict__ f2) {
  const long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (v >= n || sm_class_empty(hdr, c)) return;
  const int set = blockIdx.y;
  const int x = (int)(v % W), y = (int)((v / W) % H);
  const double* g = f1 + set * n + (v - (long long)y * W);   // the y-line through v
  double best = sm_inf();
  if (plane[set * SM_MAX_W + x] == c) {
    best = g[(long long)y * W];
    for (int r = 1;; ++r) {
      const bool lo = y - r >= 0, hi = y + r < H;
      const double q = sm_sq((double)r, sy);
      if ((!lo && !hi) || !(q < best)) break;    // every later candidate is >= q
      if (lo) best = fmin(best, __dadd_rn(g[(long long)(y - r) * W], q));
      if (hi) best = fmin(best, __dadd_rn(g[(long long)(y + r) * W], q));
    }
  }
  f2[set * n + v] = best;
}

// One CTA per (x-row, set): distances at the row's query voxels, and the row's {sum (fixed order), max} of them.
__global__ void __launch_bounds__(SM_XTPB) sm_edt_x_kernel(const double* __restrict__ f2, const uint8_t* __restrict__ surf, int c,
                                                           long long n, long long rows, int W, double sx, const SmHeader* __restrict__ hdr,
                                                           double* __restrict__ dist, double* __restrict__ part) {
  extern __shared__ double row[];
  if (sm_class_empty(hdr, c)) return;
  __shared__ double red[2][SM_XTPB / 32];
  const long long r = blockIdx.x;
  const int set = blockIdx.y;
  const long long base = r * W;
  bool has = false;
  for (int x = threadIdx.x; x < W; x += SM_XTPB) has |= sm_is_query(surf[base + x], set, c);
  double sum = 0.0, mx = 0.0;
  if (__syncthreads_or(has)) {
    const double* g = f2 + set * n + base;
    for (int x = threadIdx.x; x < W; x += SM_XTPB) row[x] = g[x];
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += SM_XTPB) {
      if (!sm_is_query(surf[base + x], set, c)) continue;
      double best = row[x];
      for (int k = 1;; ++k) {
        const bool lo = x - k >= 0, hi = x + k < W;
        const double q = sm_sq((double)k, sx);
        if ((!lo && !hi) || !(q < best)) break;
        if (lo) best = fmin(best, __dadd_rn(row[x - k], q));
        if (hi) best = fmin(best, __dadd_rn(row[x + k], q));
      }
      const double d = __dsqrt_rn(best);
      dist[set * n + base + x] = d;
      sum = __dadd_rn(sum, d);
      mx = fmax(mx, d);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum = __dadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { red[0][warp] = sum; red[1][warp] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0, m = 0.0;
    for (int w = 0; w < SM_XTPB / 32; ++w) { s = __dadd_rn(s, red[0][w]); m = fmax(m, red[1][w]); }
    part[(set * rows + r) * 2] = s;
    part[(set * rows + r) * 2 + 1] = m;
  }
}

// One CTA: the class's counts, the per-direction sums (rows in a fixed order) and maxima into out, and the two ranks that
// np.percentile(.., 95) interpolates between (its 'linear' virtual index (n-1) * 0.95).
__global__ void __launch_bounds__(SM_TPB) sm_finalize_kernel(const double* __restrict__ part, long long rows, int c,
                                                             SmHeader* __restrict__ hdr, double* __restrict__ out) {
  __shared__ double red[4][SM_TPB / 32];
  double v[4] = {0.0, 0.0, 0.0, 0.0};            // sum A, sum B, max A, max B
  const bool empty = sm_class_empty(hdr, c);
  for (long long r = threadIdx.x; r < rows && !empty; r += SM_TPB) {
#pragma unroll
    for (int set = 0; set < 2; ++set) {
      v[set] = __dadd_rn(v[set], part[(set * rows + r) * 2]);
      v[2 + set] = fmax(v[2 + set], part[(set * rows + r) * 2 + 1]);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      v[k] = __dadd_rn(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
      v[2 + k] = fmax(v[2 + k], __shfl_xor_sync(0xffffffffu, v[2 + k], o));
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) for (int k = 0; k < 4; ++k) red[k][warp] = v[k];
  __syncthreads();
  if (threadIdx.x != 0) return;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int w = 0; w < SM_TPB / 32; ++w) {
    s[0] = __dadd_rn(s[0], red[0][w]); s[1] = __dadd_rn(s[1], red[1][w]);
    s[2] = fmax(s[2], red[2][w]);      s[3] = fmax(s[3], red[3][w]);
  }
  const unsigned long long* k = hdr->cnt[c];
  double* o = out + (long long)(c - 1) * SM_OUT;
  o[0] = (double)k[0]; o[1] = (double)k[1]; o[2] = (double)k[2]; o[3] = (double)(k[1] + k[2] - k[0]);
  o[4] = (double)k[3]; o[5] = (double)k[4];
  o[6] = s[0]; o[7] = s[1]; o[8] = s[2]; o[9] = s[3];
  o[10] = o[11] = 0.0;
  const unsigned long long nn = k[3] + k[4];
  unsigned long long lo = 0, hi = 0;
  if (!empty) {
    const double vi = __dmul_rn((double)(nn - 1), 0.95);
    if (vi >= (double)(nn - 1)) lo = hi = nn - 1;
    else { lo = (unsigned long long)floor(vi); hi = lo + 1; }
  }
  hdr->prefix[0] = hdr->prefix[1] = 0ull;
  hdr->rank[0] = lo;
  hdr->rank[1] = hi;
}

// One radix digit (8 bits, most significant first) of both order statistics over the distances of both directions.  Counts are
// integers, so the atomics leave the result order-independent; the last CTA picks the digits and resets histogram and ticket.
__global__ void __launch_bounds__(SM_TPB) sm_select_kernel(const double* __restrict__ dist, const uint8_t* __restrict__ surf, int c,
                                                           long long n, int pass, SmHeader* __restrict__ hdr, double* __restrict__ out) {
  __shared__ unsigned h[2][256];
  __shared__ bool last;
  if (sm_class_empty(hdr, c)) return;
  for (int i = threadIdx.x; i < 512; i += SM_TPB) (&h[0][0])[i] = 0u;
  __syncthreads();
  const int shift = 56 - 8 * pass;
  const unsigned long long mask = pass == 0 ? 0ull : (~0ull << (64 - 8 * pass));
  const unsigned long long p0 = hdr->prefix[0], p1 = hdr->prefix[1];
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    const uint8_t s = surf[v];
#pragma unroll
    for (int set = 0; set < 2; ++set) {
      if (!sm_is_query(s, set, c)) continue;
      const unsigned long long b = (unsigned long long)__double_as_longlong(dist[set * n + v]);
      const unsigned d = (unsigned)(b >> shift) & 255u;
      if ((b & mask) == p0) atomicAdd(&h[0][d], 1u);
      if ((b & mask) == p1) atomicAdd(&h[1][d], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 512; i += SM_TPB) {
    const unsigned k = (&h[0][0])[i];
    if (k) atomicAdd(&hdr->hist[0][0] + i, k);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&hdr->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x < 2) {
    unsigned long long k = hdr->rank[threadIdx.x], pre = hdr->prefix[threadIdx.x];
    for (int b = 0; b < 256; ++b) {
      const unsigned cb = __ldcg(&hdr->hist[threadIdx.x][b]);
      if (k < cb) { pre |= (unsigned long long)b << shift; break; }
      k -= cb;
    }
    hdr->rank[threadIdx.x] = k;
    hdr->prefix[threadIdx.x] = pre;
    if (pass == SM_RADIX_PASSES - 1) out[(long long)(c - 1) * SM_OUT + 10 + threadIdx.x] = __longlong_as_double((long long)pre);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 512; i += SM_TPB) (&hdr->hist[0][0])[i] = 0u;
  if (threadIdx.x == 0) hdr->ticket = 0u;
}

int sm_check_shape(const char* what, int ndim, int S, int H, int W, int classes) {
  WSL_REQUIRE(ndim == 2 || ndim == 3, "%s: ndim must be 2 or 3 (got %d)", what, ndim);
  WSL_REQUIRE(ndim == 3 || S == 1, "%s: a rank-2 volume has S == 1 (got %d)", what, S);
  WSL_REQUIRE(S >= 1 && H >= 1 && W >= 1 && W <= SM_MAX_W, "%s: shape [%d,%d,%d] out of range (1 <= W <= %d)", what, S, H, W, SM_MAX_W);
  // <= 2^30 voxels: the 2n distances fit the 32-bit radix histograms and S*H x-rows fit gridDim.x
  WSL_REQUIRE((long long)S * H * W <= (1ll << 30), "%s: volume of %lld voxels is too large (at most 2^30)", what, (long long)S * H * W);
  WSL_REQUIRE(classes >= 2 && classes <= SM_MAX_CLASSES, "%s: classes must be in 2..%d (got %d)", what, SM_MAX_CLASSES, classes);
  return 0;
}

}  // namespace

WSL_API int wsl_surface_metrics_workspace(int ndim, int S, int H, int W, int classes, long long* out_bytes) {
  WSL_REQUIRE(out_bytes != nullptr, "wsl_surface_metrics_workspace: out_bytes must be given");
  if (sm_check_shape("wsl_surface_metrics_workspace", ndim, S, H, W, classes)) return -1;
  *out_bytes = (long long)sm_layout(S, H, W).total;
  return 0;
}

WSL_API int wsl_surface_metrics(const uint8_t* pred, const uint8_t* gt, int ndim, int S, int H, int W, int classes, double sz, double sy,
                                double sx, void* ws, double* out, cudaStream_t stream) {
  if (sm_check_shape("wsl_surface_metrics", ndim, S, H, W, classes)) return -1;
  WSL_REQUIRE(pred && gt && out && ws && ((uintptr_t)ws & 255) == 0, "wsl_surface_metrics: null pointer or workspace not 256-byte aligned");
  WSL_REQUIRE(isfinite(sz) && isfinite(sy) && isfinite(sx) && sz > 0.0 && sy > 0.0 && sx > 0.0,
              "wsl_surface_metrics: voxel spacing must be finite and > 0 (got %g, %g, %g)", sz, sy, sx);
  const SmLayout l = sm_layout(S, H, W);
  char* base = static_cast<char*>(ws);
  SmHeader* hdr = reinterpret_cast<SmHeader*>(base);
  uint8_t* surf = reinterpret_cast<uint8_t*>(base + l.surf);
  double* f1 = reinterpret_cast<double*>(base + l.f1);
  double* f2 = reinterpret_cast<double*>(base + l.f2);
  double* part = reinterpret_cast<double*>(base + l.part);
  const long long HW = (long long)H * W;
  uint8_t* plane = reinterpret_cast<uint8_t*>(base + l.plane);
  if (cudaMemsetAsync(hdr, 0, SM_ZEROED_BYTES, stream) != cudaSuccess) return wsl_check_launch("surface_metrics header reset");
  const int grid = (int)std::min<long long>((l.n + SM_TPB - 1) / SM_TPB, 8ll * wsl_num_sms());
  sm_surface_kernel<<<grid, SM_TPB, 0, stream>>>(pred, gt, ndim == 3, S, H, W, classes, surf, hdr);
  if (int rc = wsl_check_launch("surface_metrics surface")) return rc;
  const dim3 gz((unsigned)((HW + SM_XTPB - 1) / SM_XTPB), 2), gy((unsigned)((l.n + SM_XTPB - 1) / SM_XTPB), 2);
  const dim3 gx((unsigned)l.rows, 2);
  for (int c = 1; c < classes; ++c) {
    sm_edt_z_kernel<<<gz, SM_XTPB, 0, stream>>>(surf, c, S, HW, W, sz, hdr, plane, f1);
    sm_edt_y_kernel<<<gy, SM_XTPB, 0, stream>>>(f1, plane, c, l.n, H, W, sy, hdr, f2);
    sm_edt_x_kernel<<<gx, SM_XTPB, W * sizeof(double), stream>>>(f2, surf, c, l.n, l.rows, W, sx, hdr, f1, part);
    sm_finalize_kernel<<<1, SM_TPB, 0, stream>>>(part, l.rows, c, hdr, out);
    for (int pass = 0; pass < SM_RADIX_PASSES; ++pass)
      sm_select_kernel<<<grid, SM_TPB, 0, stream>>>(f1, surf, c, l.n, pass, hdr, out);
    if (int rc = wsl_check_launch("surface_metrics class")) return rc;
  }
  return 0;
}
