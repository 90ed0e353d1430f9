// Input pipeline on the GPU (SURVEY 8(f) rank 2): the per-sample augmentation of dataloaders/dataset_semi.py:126-171
// (RandomGenerator: rot90+flip | small-angle rotate, then scipy.ndimage.zoom(order=0) to the network size) for a whole
// batch in one launch, reading the training slices from a resident ragged store.  Every stage is nearest-neighbour, so
// the composition is a pure index map: out[o] = aug[zoom(o)], aug[a] = slice[rot(a)] or the constant fill.  Coordinates
// are evaluated in double with SciPy's operation order (NI_GeometricTransform / NI_ZoomShift: shift + o0*m0 + o1*m1,
// mode='constant': a coordinate outside [0, len-1] reads cval, index = floor(cc + 0.5)); no FMA contraction.
#include "common.cuh"

namespace {

constexpr int TPB = 256;

struct AugSample {           // one row per output sample (host-filled table in device memory)
  long long off;             // element offset of the slice inside the ragged stores
  int h, w;                  // slice shape
  int mode;                  // 0: none, 1: rot90(k) + flip(axis), 2: rotate(matrix, offset)
  int k, axis;
  int lab_cval;              // fill value of the rotated label map (4 when the scribble map holds "unlabelled", else 0)
  double m00, m01, m10, m11, o0, o1;   // input coordinate = M * output index + o   (scipy.ndimage.rotate, reshape=False)
};

__device__ __forceinline__ int zoom0(int o, int n_in, int n_out, bool& oob) {
  const double scale = (n_out > 1) ? (double)(n_in - 1) / (double)(n_out - 1) : 0.0;
  const double cc = __dmul_rn((double)o, scale);
  oob = (cc < 0.0) || (cc > (double)(n_in - 1));
  const int i = (int)floor(cc + 0.5);
  return i < 0 ? 0 : (i > n_in - 1 ? n_in - 1 : i);
}

// Source of output pixel (oy, ox) of sample s: element offset inside the ragged stores, or AUG_ZOOM_FILL (zoom's own constant
// fill, 0 for every array) / AUG_ROT_FILL (outside the rotated slice: 0 for the image, lab_cval for the label map).
constexpr long long AUG_ZOOM_FILL = -1, AUG_ROT_FILL = -2;

__device__ __forceinline__ long long aug_source(const AugSample& s, int oy, int ox, int OH, int OW) {
  const bool swap = (s.mode == 1) && (s.k & 1);
  const int ah = swap ? s.w : s.h, aw = swap ? s.h : s.w;       // shape of the augmented slice
  bool by, bx;
  int ay = zoom0(oy, ah, OH, by), ax = zoom0(ox, aw, OW, bx);
  if (by || bx) return AUG_ZOOM_FILL;
  int sy = ay, sx = ax;
  if (s.mode == 1) {
    if (s.axis == 0) ay = ah - 1 - ay; else ax = aw - 1 - ax;   // np.flip(axis) of the rot90 result
    switch (s.k & 3) {                                          // np.rot90(m, k): source index of element (ay, ax)
      case 1: sy = ax; sx = s.w - 1 - ay; break;
      case 2: sy = s.h - 1 - ay; sx = s.w - 1 - ax; break;
      case 3: sy = s.h - 1 - ax; sx = ay; break;
      default: sy = ay; sx = ax; break;
    }
  } else if (s.mode == 2) {
    const double c0 = __dadd_rn(__dadd_rn(s.o0, __dmul_rn((double)ay, s.m00)), __dmul_rn((double)ax, s.m01));
    const double c1 = __dadd_rn(__dadd_rn(s.o1, __dmul_rn((double)ay, s.m10)), __dmul_rn((double)ax, s.m11));
    if ((c0 < 0.0) || (c0 > (double)(s.h - 1)) || (c1 < 0.0) || (c1 > (double)(s.w - 1))) return AUG_ROT_FILL;
    sy = (int)floor(c0 + 0.5);
    sx = (int)floor(c1 + 0.5);
  }
  return s.off + (long long)sy * s.w + sx;
}

__global__ void __launch_bounds__(TPB) augment_batch_kernel(const float* __restrict__ images, const uint8_t* __restrict__ labels,
                                                            const AugSample* __restrict__ tab, int B, int OH, int OW,
                                                            float* __restrict__ out_img, uint8_t* __restrict__ out_lab) {
  const long long total = (long long)B * OH * OW;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int ox = (int)(i % OW), oy = (int)((i / OW) % OH), b = (int)(i / ((long long)OW * OH));
    const AugSample s = tab[b];
    const long long src = aug_source(s, oy, ox, OH, OW);
    out_img[i] = src >= 0 ? images[src] : 0.f;
    out_lab[i] = (uint8_t)(src >= 0 ? labels[src] : (src == AUG_ROT_FILL ? s.lab_cval : 0));
  }
}

// Scribble2Label sample transform (dataset_s2l.py:103-153): the same index map applied to the image, the scribble (rotated with
// scipy's default cval 0, SURVEY F15 -- the caller puts 0 in lab_cval) and the [h,w,4] prediction memory, whose rot90 / flip /
// rotate act on the first two axes and whose zoom factor on the class axis is 1: every channel follows its pixel.  The memory is
// a ragged channels-last store (4 floats per pixel at 4*off) and lands as [B,OH,OW,4], the reference's weight_batch layout.
__global__ void __launch_bounds__(TPB) augment_batch_s2l_kernel(const float* __restrict__ images, const uint8_t* __restrict__ scribbles,
                                                                const float4* __restrict__ weights, const AugSample* __restrict__ tab,
                                                                int B, int OH, int OW, float* __restrict__ out_img,
                                                                uint8_t* __restrict__ out_scr, float4* __restrict__ out_w) {
  const long long total = (long long)B * OH * OW;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int ox = (int)(i % OW), oy = (int)((i / OW) % OH), b = (int)(i / ((long long)OW * OH));
    const AugSample s = tab[b];
    const long long src = aug_source(s, oy, ox, OH, OW);
    out_img[i] = src >= 0 ? images[src] : 0.f;
    out_scr[i] = (uint8_t)(src >= 0 ? scribbles[src] : (src == AUG_ROT_FILL ? s.lab_cval : 0));
    out_w[i] = src >= 0 ? weights[src] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// Ensemble refresh of train_s2l.py:221-243 for a chunk of slices whose SxS logits come from one batched forward: every native
// pixel (y, x) of slice b reads the zoom(order 0) source pixel (zoom0(y, S, h), zoom0(x, S, w)) of softmax(logits[b]) -- the
// channel axis has zoom factor 1 -- and folds it into the memory: w = alpha*p + (1-alpha)*w in fp32, no contraction (:235-242).
__global__ void __launch_bounds__(TPB) s2l_refresh_kernel(const float* __restrict__ logits, const AugSample* __restrict__ tab, int B,
                                                          int S, long long max_hw, float alpha, float one_minus_alpha,
                                                          float4* __restrict__ weights) {
  const long long total = (long long)B * max_hw;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int b = (int)(i / max_hw);
    const long long j = i - (long long)b * max_hw;
    const AugSample s = tab[b];
    if (j >= (long long)s.h * s.w) continue;
    const int y = (int)(j / s.w), x = (int)(j % s.w);
    bool oy, ox;
    // the last row / column of some sizes maps just past S-1 in double arithmetic (h = 216 among ACDC's shapes): scipy reads
    // its cval there, so that pixel folds a zero prediction into the memory (SURVEY F16 notes the quirk)
    const int sy = zoom0(y, S, s.h, oy), sx = zoom0(x, S, s.w, ox);
    float p0 = 0.f, p1 = 0.f, p2 = 0.f, p3 = 0.f;
    if (!(oy || ox)) {
      const float* l = logits + (long long)b * 4 * S * S + (long long)sy * S + sx;
      const long long plane = (long long)S * S;
      const float x0 = l[0], x1 = l[plane], x2 = l[2 * plane], x3 = l[3 * plane];
      const float m = fmaxf(fmaxf(x0, x1), fmaxf(x2, x3));
      const float e0 = expf(x0 - m), e1 = expf(x1 - m), e2 = expf(x2 - m), e3 = expf(x3 - m);
      const float inv = 1.0f / (e0 + e1 + e2 + e3);
      p0 = e0 * inv; p1 = e1 * inv; p2 = e2 * inv; p3 = e3 * inv;
    }
    float4 w = weights[s.off + j];
    w.x = __fadd_rn(__fmul_rn(alpha, p0), __fmul_rn(one_minus_alpha, w.x));
    w.y = __fadd_rn(__fmul_rn(alpha, p1), __fmul_rn(one_minus_alpha, w.y));
    w.z = __fadd_rn(__fmul_rn(alpha, p2), __fmul_rn(one_minus_alpha, w.z));
    w.w = __fadd_rn(__fmul_rn(alpha, p3), __fmul_rn(one_minus_alpha, w.w));
    weights[s.off + j] = w;
  }
}

inline int aug_grid(long long total) {
  long long blocks = (total + TPB * 4 - 1) / (TPB * 4);
  if (blocks > wsl_num_sms() * 8) blocks = wsl_num_sms() * 8;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace

WSL_API int wsl_augment_sample_bytes(void) { return (int)sizeof(AugSample); }

WSL_API int wsl_augment_batch(const float* images, const uint8_t* labels, const void* table, int B, int OH, int OW, float* out_img,
                              uint8_t* out_lab, cudaStream_t stream) {
  WSL_REQUIRE(B > 0 && OH > 0 && OW > 0, "wsl_augment_batch: empty batch or output (B=%d, %dx%d)", B, OH, OW);
  augment_batch_kernel<<<aug_grid((long long)B * OH * OW), TPB, 0, stream>>>(images, labels, reinterpret_cast<const AugSample*>(table), B,
                                                                             OH, OW, out_img, out_lab);
  return wsl_check_launch("augment_batch");
}

WSL_API int wsl_augment_batch_s2l(const float* images, const uint8_t* scribbles, const float* weights, const void* table, int B, int OH,
                                  int OW, float* out_img, uint8_t* out_scr, float* out_weight, cudaStream_t stream) {
  WSL_REQUIRE(B > 0 && OH > 0 && OW > 0, "wsl_augment_batch_s2l: empty batch or output (B=%d, %dx%d)", B, OH, OW);
  WSL_REQUIRE(((uintptr_t)weights & 15) == 0 && ((uintptr_t)out_weight & 15) == 0, "wsl_augment_batch_s2l: weight stores must be 16-byte aligned");
  augment_batch_s2l_kernel<<<aug_grid((long long)B * OH * OW), TPB, 0, stream>>>(
      images, scribbles, reinterpret_cast<const float4*>(weights), reinterpret_cast<const AugSample*>(table), B, OH, OW, out_img, out_scr,
      reinterpret_cast<float4*>(out_weight));
  return wsl_check_launch("augment_batch_s2l");
}

WSL_API int wsl_s2l_refresh(const float* logits, const void* table, int B, int S, long long max_hw, float alpha, float one_minus_alpha,
                            float* weights, cudaStream_t stream) {
  WSL_REQUIRE(B > 0 && S > 1 && max_hw > 0, "wsl_s2l_refresh: empty chunk (B=%d, S=%d)", B, S);
  WSL_REQUIRE(((uintptr_t)weights & 15) == 0, "wsl_s2l_refresh: the memory must be 16-byte aligned");
  s2l_refresh_kernel<<<aug_grid((long long)B * max_hw), TPB, 0, stream>>>(logits, reinterpret_cast<const AugSample*>(table), B, S, max_hw,
                                                                          alpha, one_minus_alpha, reinterpret_cast<float4*>(weights));
  return wsl_check_launch("s2l_refresh");
}
