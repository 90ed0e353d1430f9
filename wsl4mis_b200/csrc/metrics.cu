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
//
// Batched form: V volumes of their own shapes, packed back to back, are scored in ONE launch sequence per class.  A device
// table (SmVol) gives each volume's first voxel, first x-row and first (y, x) column in the packed set, its shape and spacing.
// The line and row work items of all volumes share one grid and find their volume by binary search over those prefixes; the
// grid-stride passes (surface marking, radix select) take one grid row per volume.  Every (volume, class) keeps its own header,
// plane flags and sums, and each sum is taken in the same fixed order as for a lone volume, so the batched results are
// bit-identical to V separate calls.  The single-volume entry point is the V = 1 case of the same kernels.
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
constexpr size_t SM_ZEROED_BYTES = SM_HEADER_BYTES + 2 * SM_MAX_W;  // per volume: header + per-x-plane feature flags
constexpr long long SM_MAX_VOXELS = 1ll << 30;   // per volume: the 2n distances fit the 32-bit radix histograms
constexpr int SM_MAX_VOLUMES = 65535;            // one grid row per volume in the grid-stride passes

struct SmHeader {                                // one per volume, zeroed at the start of every call
  unsigned long long cnt[SM_MAX_CLASSES][5];     // |P&G|, |P|, |G|, #pred-surface, #gt-surface voxels per class
  unsigned long long prefix[2], rank[2];         // radix-select state of the two order statistics
  unsigned int hist[2][256];
  unsigned int ticket;
};
static_assert(sizeof(SmHeader) <= SM_HEADER_BYTES, "surface-metrics header too large");

struct SmVol {                                   // one row of the volume table (wsl_surface_metrics_volume_bytes() bytes)
  long long voff, roff, coff;                    // first voxel, first x-row (of S*H) and first (y, x) column (of H*W) in the set
  int S, H, W, rank3;
  double sz, sy, sx;
};
static_assert(sizeof(SmVol) == 64, "SmVol layout");

struct SmLayout {
  size_t plane, surf, f1, f2, part, tab, total;
};

inline size_t sm_align(size_t b) { return (b + 255) / 256 * 256; }

// V headers, then V pairs of plane-flag rows (together the zeroed prefix), then the per-voxel and per-row arrays of the whole set;
// within them volume v starts at its voff / roff (f1, f2: the two sets of volume v back to back at 2 * voff).
SmLayout sm_layout(int V, long long n, long long rows) {
  SmLayout l;
  size_t off = (size_t)V * SM_HEADER_BYTES;
  l.plane = off; off += (size_t)V * 2 * SM_MAX_W;                   // set * SM_MAX_W + x: == c when plane x has a feature
  l.surf = off;  off += sm_align((size_t)n);                        // pred-surface class | gt-surface class << 4
  l.f1 = off;    off += sm_align(2 * (size_t)n * sizeof(double));   // z pass, then the distances at the query voxels
  l.f2 = off;    off += sm_align(2 * (size_t)n * sizeof(double));   // y pass
  l.part = off;  off += sm_align(2 * (size_t)rows * 2 * sizeof(double));  // per (volume, set, x-row): {sum, max}
  l.tab = off;   off += sm_align(sizeof(SmVol));                    // the single-volume entry point's one-row table
  l.total = off;
  return l;
}

__host__ __device__ __forceinline__ SmHeader* sm_hdr(void* base, int v) {
  return reinterpret_cast<SmHeader*>(static_cast<char*>(base) + (size_t)v * SM_HEADER_BYTES);
}
__host__ __device__ __forceinline__ const SmHeader* sm_hdr(const void* base, int v) {
  return reinterpret_cast<const SmHeader*>(static_cast<const char*>(base) + (size_t)v * SM_HEADER_BYTES);
}

// the volume whose range [start, next start) holds global index i; field 0: voxels, 1: x-rows, 2: columns
__device__ __forceinline__ int sm_volume_of(const SmVol* __restrict__ tab, int V, long long i, int field) {
  int lo = 0, hi = V - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const long long st = field == 0 ? tab[mid].voff : (field == 1 ? tab[mid].roff : tab[mid].coff);
    if (st <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
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

__global__ void sm_table_kernel(SmVol* tab, int S, int H, int W, int rank3, double sz, double sy, double sx) {
  tab->voff = tab->roff = tab->coff = 0;
  tab->S = S; tab->H = H; tab->W = W; tab->rank3 = rank3;
  tab->sz = sz; tab->sy = sy; tab->sx = sx;
}

// grid (x, V): grid row v strides over volume v
__global__ void __launch_bounds__(SM_TPB) sm_surface_kernel(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ gt,
                                                            const SmVol* __restrict__ tab, int classes, uint8_t* __restrict__ surf,
                                                            void* __restrict__ hdrs) {
  __shared__ unsigned cnt[SM_MAX_CLASSES][5];
  for (int i = threadIdx.x; i < SM_MAX_CLASSES * 5; i += blockDim.x) (&cnt[0][0])[i] = 0u;
  __syncthreads();
  const SmVol t = tab[blockIdx.y];
  const int S = t.S, H = t.H, W = t.W;
  pred += t.voff; gt += t.voff; surf += t.voff;
  const long long HW = (long long)H * W, n = HW * S;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(v % W), y = (int)((v / W) % H), z = (int)(v / HW);
    const int p = pred[v], g = gt[v];
    int ps = 0, gs = 0;
    if (p > 0 && p < classes) {
      atomicAdd(&cnt[p][1], 1u);
      if (sm_on_surface(pred, v, p, x, y, z, S, H, W, HW, t.rank3)) { ps = p; atomicAdd(&cnt[p][3], 1u); }
      if (g == p) atomicAdd(&cnt[p][0], 1u);
    }
    if (g > 0 && g < classes) {
      atomicAdd(&cnt[g][2], 1u);
      if (sm_on_surface(gt, v, g, x, y, z, S, H, W, HW, t.rank3)) { gs = g; atomicAdd(&cnt[g][4], 1u); }
    }
    surf[v] = (uint8_t)(ps | (gs << 4));
  }
  __syncthreads();
  SmHeader* hdr = sm_hdr(hdrs, blockIdx.y);
  for (int i = threadIdx.x; i < SM_MAX_CLASSES * 5; i += blockDim.x) {
    const unsigned k = (&cnt[0][0])[i];
    if (k) atomicAdd(&hdr->cnt[0][0] + i, (unsigned long long)k);
  }
}

// Set 0: features = gt surface of class c (its distances are read at the pred surface: pred -> gt); set 1 the other way round.
__device__ __forceinline__ bool sm_is_feature(uint8_t s, int set, int c) { return ((set == 0 ? s >> 4 : s & 15)) == c; }
__device__ __forceinline__ bool sm_is_query(uint8_t s, int set, int c) { return ((set == 0 ? s & 15 : s >> 4)) == c; }
__device__ __forceinline__ bool sm_class_empty(const SmHeader* hdr, int c) { return hdr->cnt[c][3] == 0ull || hdr->cnt[c][4] == 0ull; }

// one thread per (y, x) column of the set (all volumes' columns in one grid), blockIdx.y = set
__global__ void __launch_bounds__(SM_XTPB) sm_edt_z_kernel(const uint8_t* __restrict__ surf, int c, const SmVol* __restrict__ tab, int V,
                                                           long long cols, const void* __restrict__ hdrs, uint8_t* __restrict__ planes,
                                                           double* __restrict__ f1) {
  const long long gcol = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (gcol >= cols) return;
  const int vol = sm_volume_of(tab, V, gcol, 2);
  if (sm_class_empty(sm_hdr(hdrs, vol), c)) return;
  const SmVol t = tab[vol];
  const long long HW = (long long)t.H * t.W, n = HW * t.S, col = gcol - t.coff;
  const int set = blockIdx.y, S = t.S;
  double* f = f1 + 2 * t.voff + set * n + col;
  const uint8_t* s = surf + t.voff + col;
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
    f[z * HW] = d < 0.0 ? sm_inf() : sm_sq(d, t.sz);
  }
  if (next >= 0) planes[(2 * (long long)vol + set) * SM_MAX_W + col % t.W] = (uint8_t)c;
}

// one thread per voxel of the set, blockIdx.y = set
__global__ void __launch_bounds__(SM_XTPB) sm_edt_y_kernel(const double* __restrict__ f1, const uint8_t* __restrict__ planes, int c,
                                                           const SmVol* __restrict__ tab, int V, long long n_total,
                                                           const void* __restrict__ hdrs, double* __restrict__ f2) {
  const long long gv = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (gv >= n_total) return;
  const int vol = sm_volume_of(tab, V, gv, 0);
  if (sm_class_empty(sm_hdr(hdrs, vol), c)) return;
  const SmVol t = tab[vol];
  const int H = t.H, W = t.W;
  const long long n = (long long)t.S * H * W, v = gv - t.voff;
  const int set = blockIdx.y;
  const int x = (int)(v % W), y = (int)((v / W) % H);
  const double* g = f1 + 2 * t.voff + set * n + (v - (long long)y * W);   // the y-line through v
  double best = sm_inf();
  if (planes[(2 * (long long)vol + set) * SM_MAX_W + x] == c) {
    best = g[(long long)y * W];
    for (int r = 1;; ++r) {
      const bool lo = y - r >= 0, hi = y + r < H;
      const double q = sm_sq((double)r, t.sy);
      if ((!lo && !hi) || !(q < best)) break;    // every later candidate is >= q
      if (lo) best = fmin(best, __dadd_rn(g[(long long)(y - r) * W], q));
      if (hi) best = fmin(best, __dadd_rn(g[(long long)(y + r) * W], q));
    }
  }
  f2[2 * t.voff + set * n + v] = best;
}

// One CTA per (x-row of the set, set): distances at the row's query voxels, and the row's {sum (fixed order), max} of them.
__global__ void __launch_bounds__(SM_XTPB) sm_edt_x_kernel(const double* __restrict__ f2, const uint8_t* __restrict__ surf, int c,
                                                           const SmVol* __restrict__ tab, int V, const void* __restrict__ hdrs,
                                                           double* __restrict__ dist, double* __restrict__ part) {
  extern __shared__ double row[];
  const int vol = sm_volume_of(tab, V, blockIdx.x, 1);
  if (sm_class_empty(sm_hdr(hdrs, vol), c)) return;
  __shared__ double red[2][SM_XTPB / 32];
  const SmVol t = tab[vol];
  const int W = t.W;
  const long long rows = (long long)t.S * t.H, n = rows * W, r = blockIdx.x - t.roff;
  const int set = blockIdx.y;
  const long long base = r * W;
  surf += t.voff;
  bool has = false;
  for (int x = threadIdx.x; x < W; x += SM_XTPB) has |= sm_is_query(surf[base + x], set, c);
  double sum = 0.0, mx = 0.0;
  if (__syncthreads_or(has)) {
    const double* g = f2 + 2 * t.voff + set * n + base;
    for (int x = threadIdx.x; x < W; x += SM_XTPB) row[x] = g[x];
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += SM_XTPB) {
      if (!sm_is_query(surf[base + x], set, c)) continue;
      double best = row[x];
      for (int k = 1;; ++k) {
        const bool lo = x - k >= 0, hi = x + k < W;
        const double q = sm_sq((double)k, t.sx);
        if ((!lo && !hi) || !(q < best)) break;
        if (lo) best = fmin(best, __dadd_rn(row[x - k], q));
        if (hi) best = fmin(best, __dadd_rn(row[x + k], q));
      }
      const double d = __dsqrt_rn(best);
      dist[2 * t.voff + set * n + base + x] = d;
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
    double* p = part + (2 * t.roff + set * rows + r) * 2;
    p[0] = s;
    p[1] = m;
  }
}

// One CTA per volume: the class's counts, the per-direction sums (rows in a fixed order) and maxima into out, and the two ranks
// that np.percentile(.., 95) interpolates between (its 'linear' virtual index (n-1) * 0.95).
__global__ void __launch_bounds__(SM_TPB) sm_finalize_kernel(const double* __restrict__ part, const SmVol* __restrict__ tab, int c,
                                                             int classes, void* __restrict__ hdrs, double* __restrict__ out) {
  __shared__ double red[4][SM_TPB / 32];
  const int vol = blockIdx.x;
  const SmVol t = tab[vol];
  SmHeader* hdr = sm_hdr(hdrs, vol);
  const long long rows = (long long)t.S * t.H;
  part += 2 * t.roff * 2;
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
  double* o = out + ((long long)vol * (classes - 1) + (c - 1)) * SM_OUT;
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

// One radix digit (8 bits, most significant first) of both order statistics over the distances of both directions; grid row v
// strides over volume v.  Counts are integers, so the atomics leave the result order-independent; the last CTA of a volume picks
// its digits and resets that volume's histogram and ticket.
__global__ void __launch_bounds__(SM_TPB) sm_select_kernel(const double* __restrict__ dist, const uint8_t* __restrict__ surf, int c,
                                                           const SmVol* __restrict__ tab, int classes, int pass, void* __restrict__ hdrs,
                                                           double* __restrict__ out) {
  __shared__ unsigned h[2][256];
  __shared__ bool last;
  const int vol = blockIdx.y;
  SmHeader* hdr = sm_hdr(hdrs, vol);
  if (sm_class_empty(hdr, c)) return;
  const SmVol t = tab[vol];
  const long long n = (long long)t.S * t.H * t.W;
  dist += 2 * t.voff;
  surf += t.voff;
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
    if (pass == SM_RADIX_PASSES - 1)
      out[((long long)vol * (classes - 1) + (c - 1)) * SM_OUT + 10 + threadIdx.x] = __longlong_as_double((long long)pre);
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
  WSL_REQUIRE((long long)S * H * W <= SM_MAX_VOXELS, "%s: volume of %lld voxels is too large (at most 2^30)", what, (long long)S * H * W);
  WSL_REQUIRE(classes >= 2 && classes <= SM_MAX_CLASSES, "%s: classes must be in 2..%d (got %d)", what, SM_MAX_CLASSES, classes);
  return 0;
}

int sm_check_set(const char* what, int V, long long n, long long rows, long long cols, long long max_n, int max_w, int classes) {
  WSL_REQUIRE(V >= 1 && V <= SM_MAX_VOLUMES, "%s: V must be in 1..%d (got %d)", what, SM_MAX_VOLUMES, V);
  WSL_REQUIRE(max_w >= 1 && max_w <= SM_MAX_W, "%s: max_w must be in 1..%d (got %d)", what, SM_MAX_W, max_w);
  WSL_REQUIRE(max_n >= 1 && max_n <= SM_MAX_VOXELS, "%s: max_n must be in 1..2^30 (got %lld)", what, max_n);
  WSL_REQUIRE(n >= V && rows >= V && cols >= V && max_n <= n && rows <= n && cols <= n && rows < (1ll << 31),
              "%s: inconsistent totals (V %d, voxels %lld, rows %lld, columns %lld)", what, V, n, rows, cols);
  WSL_REQUIRE(classes >= 2 && classes <= SM_MAX_CLASSES, "%s: classes must be in 2..%d (got %d)", what, SM_MAX_CLASSES, classes);
  return 0;
}

int sm_run(const uint8_t* pred, const uint8_t* gt, const SmVol* tab, int V, long long n, long long rows, long long cols, long long max_n,
           int max_w, int classes, void* ws, double* out, cudaStream_t stream) {
  const SmLayout l = sm_layout(V, n, rows);
  char* base = static_cast<char*>(ws);
  uint8_t* planes = reinterpret_cast<uint8_t*>(base + l.plane);
  uint8_t* surf = reinterpret_cast<uint8_t*>(base + l.surf);
  double* f1 = reinterpret_cast<double*>(base + l.f1);
  double* f2 = reinterpret_cast<double*>(base + l.f2);
  double* part = reinterpret_cast<double*>(base + l.part);
  if (cudaMemsetAsync(base, 0, (size_t)V * SM_ZEROED_BYTES, stream) != cudaSuccess) return wsl_check_launch("surface_metrics header reset");
  // grid-stride passes: about 8 waves of CTAs over the SMs in all, split evenly over the volumes
  const int gx = (int)std::min<long long>((max_n + SM_TPB - 1) / SM_TPB, std::max(1, 8 * wsl_num_sms() / V));
  const dim3 gs((unsigned)gx, (unsigned)V);
  sm_surface_kernel<<<gs, SM_TPB, 0, stream>>>(pred, gt, tab, classes, surf, base);
  if (int rc = wsl_check_launch("surface_metrics surface")) return rc;
  const dim3 gz((unsigned)((cols + SM_XTPB - 1) / SM_XTPB), 2), gy((unsigned)((n + SM_XTPB - 1) / SM_XTPB), 2);
  const dim3 gxr((unsigned)rows, 2);
  for (int c = 1; c < classes; ++c) {
    sm_edt_z_kernel<<<gz, SM_XTPB, 0, stream>>>(surf, c, tab, V, cols, base, planes, f1);
    sm_edt_y_kernel<<<gy, SM_XTPB, 0, stream>>>(f1, planes, c, tab, V, n, base, f2);
    sm_edt_x_kernel<<<gxr, SM_XTPB, max_w * sizeof(double), stream>>>(f2, surf, c, tab, V, base, f1, part);
    sm_finalize_kernel<<<V, SM_TPB, 0, stream>>>(part, tab, c, classes, base, out);
    for (int pass = 0; pass < SM_RADIX_PASSES; ++pass)
      sm_select_kernel<<<gs, SM_TPB, 0, stream>>>(f1, surf, c, tab, classes, pass, base, out);
    if (int rc = wsl_check_launch("surface_metrics class")) return rc;
  }
  return 0;
}

}  // namespace

WSL_API int wsl_surface_metrics_workspace(int ndim, int S, int H, int W, int classes, long long* out_bytes) {
  WSL_REQUIRE(out_bytes != nullptr, "wsl_surface_metrics_workspace: out_bytes must be given");
  if (sm_check_shape("wsl_surface_metrics_workspace", ndim, S, H, W, classes)) return -1;
  *out_bytes = (long long)sm_layout(1, (long long)S * H * W, (long long)S * H).total;
  return 0;
}

WSL_API int wsl_surface_metrics(const uint8_t* pred, const uint8_t* gt, int ndim, int S, int H, int W, int classes, double sz, double sy,
                                double sx, void* ws, double* out, cudaStream_t stream) {
  if (sm_check_shape("wsl_surface_metrics", ndim, S, H, W, classes)) return -1;
  WSL_REQUIRE(pred && gt && out && ws && ((uintptr_t)ws & 255) == 0, "wsl_surface_metrics: null pointer or workspace not 256-byte aligned");
  WSL_REQUIRE(isfinite(sz) && isfinite(sy) && isfinite(sx) && sz > 0.0 && sy > 0.0 && sx > 0.0,
              "wsl_surface_metrics: voxel spacing must be finite and > 0 (got %g, %g, %g)", sz, sy, sx);
  const long long n = (long long)S * H * W, rows = (long long)S * H;
  SmVol* tab = reinterpret_cast<SmVol*>(static_cast<char*>(ws) + sm_layout(1, n, rows).tab);
  sm_table_kernel<<<1, 1, 0, stream>>>(tab, S, H, W, ndim == 3, sz, sy, sx);
  if (int rc = wsl_check_launch("surface_metrics table")) return rc;
  return sm_run(pred, gt, tab, 1, n, rows, (long long)H * W, n, W, classes, ws, out, stream);
}

WSL_API int wsl_surface_metrics_volume_bytes(void) { return (int)sizeof(SmVol); }

WSL_API int wsl_surface_metrics_batched_workspace(int V, long long n_total, long long rows_total, int classes, long long* out_bytes) {
  WSL_REQUIRE(out_bytes != nullptr, "wsl_surface_metrics_batched_workspace: out_bytes must be given");
  if (sm_check_set("wsl_surface_metrics_batched_workspace", V, n_total, rows_total, rows_total, 1, 1, classes)) return -1;
  *out_bytes = (long long)sm_layout(V, n_total, rows_total).total;
  return 0;
}

WSL_API int wsl_surface_metrics_batched(const uint8_t* pred, const uint8_t* gt, const void* vols, int V, long long n_total,
                                        long long rows_total, long long cols_total, long long max_n, int max_w, int classes, void* ws,
                                        double* out, cudaStream_t stream) {
  if (sm_check_set("wsl_surface_metrics_batched", V, n_total, rows_total, cols_total, max_n, max_w, classes)) return -1;
  WSL_REQUIRE(pred && gt && vols && out && ws && ((uintptr_t)ws & 255) == 0 && ((uintptr_t)vols & 7) == 0,
              "wsl_surface_metrics_batched: null pointer, workspace not 256-byte aligned or table not 8-byte aligned");
  return sm_run(pred, gt, static_cast<const SmVol*>(vols), V, n_total, rows_total, cols_total, max_n, max_w, classes, ws, out, stream);
}
