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

__global__ void __launch_bounds__(TPB) augment_batch_kernel(const float* __restrict__ images, const uint8_t* __restrict__ labels,
                                                            const AugSample* __restrict__ tab, int B, int OH, int OW,
                                                            float* __restrict__ out_img, uint8_t* __restrict__ out_lab) {
  const long long total = (long long)B * OH * OW;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int ox = (int)(i % OW), oy = (int)((i / OW) % OH), b = (int)(i / ((long long)OW * OH));
    const AugSample s = tab[b];
    const bool swap = (s.mode == 1) && (s.k & 1);
    const int ah = swap ? s.w : s.h, aw = swap ? s.h : s.w;       // shape of the augmented slice
    bool by, bx;
    int ay = zoom0(oy, ah, OH, by), ax = zoom0(ox, aw, OW, bx);
    float v = 0.f;                                                 // zoom's own constant fill is 0 for image and label
    int l = 0;
    if (!(by || bx)) {
      int sy = ay, sx = ax;
      bool fill = false;
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
        fill = (c0 < 0.0) || (c0 > (double)(s.h - 1)) || (c1 < 0.0) || (c1 > (double)(s.w - 1));
        sy = (int)floor(c0 + 0.5);
        sx = (int)floor(c1 + 0.5);
      }
      if (fill) {
        v = 0.f;
        l = s.lab_cval;
      } else {
        const long long src = s.off + (long long)sy * s.w + sx;
        v = images[src];
        l = labels[src];
      }
    }
    out_img[i] = v;
    out_lab[i] = (uint8_t)l;
  }
}

}  // namespace

WSL_API int wsl_augment_sample_bytes(void) { return (int)sizeof(AugSample); }

WSL_API int wsl_augment_batch(const float* images, const uint8_t* labels, const void* table, int B, int OH, int OW, float* out_img,
                              uint8_t* out_lab, cudaStream_t stream) {
  WSL_REQUIRE(B > 0 && OH > 0 && OW > 0, "wsl_augment_batch: empty batch or output (B=%d, %dx%d)", B, OH, OW);
  const long long total = (long long)B * OH * OW;
  long long blocks = (total + TPB * 4 - 1) / (TPB * 4);
  if (blocks > wsl_num_sms() * 8) blocks = wsl_num_sms() * 8;
  augment_batch_kernel<<<(int)blocks, TPB, 0, stream>>>(images, labels, reinterpret_cast<const AugSample*>(table), B, OH, OW, out_img,
                                                        out_lab);
  return wsl_check_launch("augment_batch");
}
