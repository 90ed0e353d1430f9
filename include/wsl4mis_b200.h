/*
 * wsl4mis_b200 -- C ABI of the H100 (sm_90a) kernels behind the WSL4MIS segmentation-training hot path.
 *
 * The reference (HiLab-git/WSL4MIS) has no native code and no FFI: every operation below is, in the reference,
 * a stock PyTorch call made from Python.  Each entry point therefore cites the reference *Python* call site
 * (paths relative to /root/reference/code) whose arithmetic it replaces; INTEGRATION.md shows the ctypes
 * binding a maintainer adds on the reference side.
 *
 * Conventions
 *   - plain pointers + sizes, no torch types; all pointers are DEVICE pointers unless stated otherwise;
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*-compatible handle), never
 *     allocates, never synchronises; the caller owns all buffers;
 *   - return 0 on success, negative on error; wsl_last_error() returns a thread-local message;
 *   - "act" tensors are channels-last (NHWC); their storage type is bf16 (`dtype` 0, the fast tensor-core path),
 *     fp32 (`dtype` 1: the reference-accurate parity modes -- CUDA-core direct convolutions, or the fp16 hi/lo split
 *     tensor-core convolutions wsl_conv_tc_split / wsl_wgrad_tc_split) or fp16 (`dtype` 2: same wgmma rate as
 *     bf16 with an 11-bit mantissa; gradients then travel multiplied by a power-of-two loss scale chosen by the caller);
 *     logits / probabilities / losses are fp32 NCHW;
 *   - `ws` is a caller-provided workspace of wsl_workspace_floats() floats, zero-initialised ONCE by the
 *     caller (kernels leave its ticket words zero again); one workspace must not be shared by two kernels
 *     that may run concurrently.
 */
#ifndef WSL4MIS_B200_H
#define WSL4MIS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* cudaStream_t;

/* ---- library ------------------------------------------------------------------------------------------- */
const char* wsl_last_error(void);
int wsl_abi_version(void);
int wsl_workspace_floats(void);

/* ---- losses (utils/losses.py, utils/gate_crf_loss.py, torch CrossEntropyLoss) ---------------------------- */

/* torch.softmax(outputs,1) + CrossEntropyLoss(ignore_index)(outputs,label.long()):
 * train_weakly_supervised_pCE_2D.py:81,98,100.  probs may be NULL.  out2 = {loss, labelled-pixel count}. */
int wsl_softmax_pce_fwd(const float* logits, const uint8_t* label, float* probs, int N, int C, int H, int W,
                        int ignore_index, float* out2, float* ws, cudaStream_t stream);

/* Scribble2Label step head (train_s2l.py:123-147): softmax once, u-labels where scribble == 4 and weight[..., c] > thr_conf (the
 * last qualifying class wins, :133-145; map written to ulab), both masked NLL means.  ctrl = {thr_conf, w_u} in device memory
 * (w_u = 0 before thr_iter, 0.5 after).  out5 = {pCE, #labelled, CE_u, #u-labelled, loss}, loss = pCE (w_u == 0) or
 * pCE + w_u * CE_u (NaN when no pixel qualifies, as torch).  weight: [N,H,W,4] fp32.  wsl_s2l_head_bwd: dlogits of that loss
 * times `scale` (an empty u-support adds nothing), fp32 NCHW and / or NHWC-16 bf16 / fp16 as wsl_head_bwd. */
int wsl_s2l_fwd(const float* logits, const uint8_t* scribble, const float* weight, const float* ctrl, int N, int C, int H, int W,
                float* probs, uint8_t* ulab, float* out5, float* ws, cudaStream_t stream);
int wsl_s2l_head_bwd(const float* probs, const uint8_t* scribble, const uint8_t* ulab, const float* stats5, const float* ctrl,
                     float scale, int N, int C, int H, int W, float* dlogits, void* dlogits_nhwc16, int dtype16, cudaStream_t stream);

/* d(w_ce*pCE + <gprobs*gprobs_scale, softmax(logits)>)/dlogits, times *grad_out (NULL -> 1).
 * Replaces autograd through softmax / log_softmax+nll_loss.  label/gprobs may be NULL.  Either output may be NULL:
 * dlogits = fp32 NCHW (API layout), dlogits_nhwc16 = channels-last bf16 / fp16 (dtype16 0 / 2) padded to 16 channels (the
 * layout the out_conv gradient kernels consume; saves a conversion pass in the fused step). */
int wsl_head_bwd(const float* probs, const uint8_t* label, const float* ce_stats, const float* grad_out,
                 float w_ce, const float* gprobs, float gprobs_scale, int N, int C, int H, int W,
                 int ignore_index, float* dlogits, void* dlogits_nhwc16, int dtype16, cudaStream_t stream);

/* ModelLossSemsegGatedCRF.forward(y, [{'weight':w,'xy':sxy,'rgb':srgb}], radius, image, H, W)['loss']:
 * utils/gate_crf_loss.py:20-117 (fast path: no masks, Potts).  Also emits d loss / d y into gprobs (may be
 * NULL).  out2 = {loss, kernels.sum()}. */
int wsl_gatedcrf_fwd(const float* probs, const float* image, float* gprobs, int N, int C, int H, int W,
                     int radius, float sigma_xy, float sigma_rgb, float weight, float* out2, float* ws,
                     cudaStream_t stream);

/* MumfordShah_Loss()(image, prediction): utils/losses.py:275-309.  centroids: [N*C] scratch kept for bwd. */
int wsl_mumford_shah_fwd(const float* image, const float* probs, int N, int C, int H, int W, float* out1,
                         float* centroids, float* ws, cudaStream_t stream);
int wsl_mumford_shah_bwd(const float* image, const float* probs, const float* centroids, int N, int C, int H,
                         int W, float scale, int accumulate, float* gprobs, cudaStream_t stream);

/* argmax(beta*p1 + (1-beta)*p2, dim=1): train_weakly_supervised_segmentation_pCE_ours_proposed.py:117-120.
 * p2 may be NULL (plain argmax).  beta_ptr (optional, device {beta, 1-beta}) overrides the scalars so that a captured
 * CUDA graph follows the script's per-step `random.random()` (:117). */
int wsl_mix_argmax(const float* p1, const float* p2, float beta, float one_minus_beta, const float* beta_ptr, int N, int C,
                   int H, int W, uint8_t* out, cudaStream_t stream);

/* batch-summed ignore mask of pDLoss (utils/losses.py:219-220 + the [N,1,H,W] broadcast at :209-211). */
int wsl_mask_count(const uint8_t* target, int N, int H, int W, int ignore_index, float* msum, cudaStream_t stream);

/* pDLoss(n_classes=4, ignore_index)(probs, target): utils/losses.py:195-232.  msum NULL -> constant mconst.
 * out13 = {loss, I[4], Y[4], Z[4]} (kept for the backward). */
int wsl_pdice_fwd(const float* probs, const uint8_t* target, const float* msum, float mconst, int N, int C, int H,
                  int W, float* out13, float* ws, cudaStream_t stream);
int wsl_pdice_bwd(const float* probs, const uint8_t* target, const float* msum, float mconst, const float* sums13,
                  int N, int C, int H, int W, float scale, int accumulate, float* gprobs, cudaStream_t stream);

/* tv_loss(pred): train_weakly_supervised_pCE_TV_2D.py:58-65.  planes = N'*C.  gprobs_zeroed may be NULL;
 * when given it must be zero-filled and receives grad_scale * d loss / d pred. */
int wsl_tv_loss(const float* probs, int planes, int H, int W, float grad_scale, float* gprobs_zeroed, float* out1,
                float* ws, cudaStream_t stream);

/* losses.entropy_loss(p, C) (utils/losses.py:30-36; train_weakly_supervised_pCE_Entropy_Mini_2D.py:99-102) and its gradient
 * (gprobs (+)= scale * d/dp). */
int wsl_entropy_fwd(const float* probs, int N, int C, int H, int W, float* out1, float* ws, cudaStream_t stream);
int wsl_entropy_bwd(const float* probs, int N, int C, int H, int W, float scale, int accumulate, float* gprobs,
                    cudaStream_t stream);
/* inter_class_variance - intra_class_variance (train_weakly_supervised_pCE_Inter&Intra_Class_2D.py:30-36,114).
 * out3 = {inter - intra, inter, intra}; stats = [N*4*2 + N*2] scratch kept for the backward. */
int wsl_class_variance_fwd(const float* image, const float* probs, int N, int C, int H, int W, float* out3, float* stats,
                           float* ws, cudaStream_t stream);
int wsl_class_variance_bwd(const float* image, const float* probs, const float* stats, int N, int C, int H, int W,
                           float scale, int accumulate, float* gprobs, cudaStream_t stream);

/* Mean-teacher consistency between softmax(student) and softmax(teacher) (utils/losses.py:65-82, softmax_mse_loss), two modes:
 * T >= 2 (even), uncertainty-aware (train_uncertainty_aware_mean_teacher_2D.py:164-188): mean softmax of the T stochastic
 *   teacher passes (mc_logits [T*B,4,H,W], script layout) -> entropy -> mask (u8 [B,H,W]) -> masked squared distance summed
 *   / (2*sum(mask)+1e-16); out3 = {sum, sum(mask), loss}.
 * T = 0, unmasked (train_mean_teacher_2D.py:169-170): torch.mean of the squared distance over B*C*H*W; mc_logits and mask
 *   may be NULL (the backward takes mask = NULL); out3 = {sum, B*C*H*W, loss}.
 * threshold / weight are read from device memory when the *_ptr is non-NULL (graph-capture friendly ramps). */
int wsl_uamt_consistency_fwd(const float* student, const float* teacher, const float* mc_logits, int T, int B, int C, int H,
                             int W, const float* threshold_ptr, float threshold, uint8_t* mask, float* out3, float* ws,
                             cudaStream_t stream);
int wsl_uamt_consistency_bwd(const float* student, const float* teacher, const uint8_t* mask, const float* stats3,
                             const float* weight_ptr, float weight, int B, int C, int H, int W, float* dlogits,
                             cudaStream_t stream);
/* out[r*n + i] = x[i] + clamp(sigma*N(0,1), -clamp, clamp)  (:147-149,167-169), counter RNG, r < reps */
int wsl_add_clamped_noise(const float* x, long long n, int reps, float sigma, float clamp, unsigned long long seed,
                          const unsigned long long* seed_ptr, float* out, cudaStream_t stream);

/* Validation path (val_2D.py:18-50): scipy.ndimage.zoom(order=0) semantics on S slices ([S,h,w] -> [S,H,W], fp32 images
 * or uint8 label maps, including SciPy's cval=0 read when rounding pushes the last coordinate past in-1) and per-class
 * overlap counts {|P&G|, |P|, |G|} (index c*3+k, classes 1..classes-1) for medpy-style Dice. */
int wsl_zoom_nearest(const void* src, int is_u8, int S, int h, int w, int H, int W, void* dst, cudaStream_t stream);
int wsl_overlap_counts(const uint8_t* pred, const uint8_t* gt, long long n, int classes, unsigned long long* counts_zeroed,
                       cudaStream_t stream);

/* torch.rot90(x, k, [2,3]) of square fp32 maps ([planes,S,S]; dst (+)= rot(src)) and the mean-teacher EMA update
 * ema = alpha*ema + (1-alpha)*param (train_weakly_supervised_ustm_2D.py:61-65,124-125,150,163). */
int wsl_rot90(const float* src, long long planes, int S, int k, int accumulate, float* dst, cudaStream_t stream);
int wsl_ema_update(float* ema, const float* param, long long n, float alpha, cudaStream_t stream);

/* Deep-supervision heads (Decoder_DS.forward, networks/unet.py:177,181,185): F.interpolate(x, size) in its default nearest
 * mode on fp32 [planes,h,w] -> [planes,H,W] maps, and its transpose for the backward pass. */
int wsl_nearest_resize_fwd(const float* src, long long planes, int h, int w, int H, int W, float* dst, cudaStream_t stream);
int wsl_nearest_resize_bwd(const float* gdst, long long planes, int h, int w, int H, int W, float* gsrc, cudaStream_t stream);

/* Input pipeline (dataloaders/dataset_semi.py:126-171, RandomGenerator): rot90+flip | rotate(order 0) followed by
 * zoom(order 0) to OH x OW for B samples read from a resident ragged slice store; `table` holds B rows of
 * wsl_augment_sample_bytes() bytes: {int64 off; int32 h, w, mode, k, axis, lab_cval; double m00, m01, m10, m11, o0, o1}. */
int wsl_augment_sample_bytes(void);
int wsl_augment_batch(const float* images, const uint8_t* labels, const void* table, int B, int OH, int OW, float* out_img,
                      uint8_t* out_lab, cudaStream_t stream);
/* Scribble2Label sample transform (dataloaders/dataset_s2l.py:103-153, RandomGenerator_s2l): the same index map applied to the
 * image, the scribble (rotation fill = lab_cval; the reference's scipy default is 0, SURVEY F15) and the [h,w,4] fp32 prediction
 * memory, read from a ragged channels-last store (4 floats per pixel at element 4*off) and written as [B,OH,OW,4]. */
int wsl_augment_batch_s2l(const float* images, const uint8_t* scribbles, const float* weights, const void* table, int B, int OH,
                          int OW, float* out_img, uint8_t* out_scr, float* out_weight, cudaStream_t stream);
/* Scribble2Label ensemble refresh (train_s2l.py:221-243) for B slices (table rows: off, h, w) whose [B,4,S,S] fp32 logits come
 * from one batched forward: softmax at the zoom(order 0) source pixel of every native pixel (zoom's out-of-range fill reads 0),
 * then weights = alpha * p + one_minus_alpha * weights in fp32 (ragged channels-last memory, updated in place). */
int wsl_s2l_refresh(const float* logits, const void* table, int B, int S, long long max_hw, float alpha, float one_minus_alpha,
                    float* weights, cudaStream_t stream);

/* Random-walker pseudo labels (dataloaders/acdc_pseudo_label_random_walker.py:9-26, pseudo_label_generator_acdc, and the per-slice
 * loop :50-55; skimage random_walker(rescale_intensity(image, (-0.35, 1.35), (-1, 1)), markers, beta, mode='bf')) for n_slices
 * ragged slices of a resident store (fp32 images and u8 scribbles at element offs[s], shapes[s] = {h, w}; scribble 0..3 = class,
 * 4 = unlabelled).  A slice lacking a scribble of class 1, 2 or 3 gets all-zero labels and probabilities (:12-13).  Otherwise one
 * persistent CTA solves L_UU x_l = -L_UM m_l for every label column by Jacobi-preconditioned CG (fp32 vectors, fp64 dot products
 * in a fixed order) until max_l ||r_l|| / ||b_l|| <= tol or max_iter iterations; labels = argmax (seeds keep theirs), written as
 * the pseudo label (label - 1, markers renumbered by rank when the background scribble is missing: DESIGN F17).  Slices are taken
 * in the order given by `order` (descending pixel count keeps the last wave short).  probs ([px, 4] fp32, may be NULL) holds the
 * per-column probabilities; iters / resid ([n_slices], indexed by slice id) the iteration count and final relative residual
 * (iters = -1: the slice does not fit slot_px).  Results are bit-identical run to run and independent of the other slices.
 * ws: caller-owned, wsl_random_walker_workspace() floats for `ctas` CTAs and slices of at most slot_px pixels (no zeroing needed).
 * wsl_random_walker_workspace: ctas <= 0 picks the resident CTA count of the device; out2 is a HOST pointer receiving
 * {ctas, workspace floats}. */
int wsl_random_walker_workspace(int ctas, long long max_px, long long* out2);
int wsl_random_walker(const float* images, const uint8_t* scribbles, const long long* offs, const int* shapes, const int* order,
                      int n_slices, float beta, float tol, int max_iter, float* ws, int ctas, long long slot_px, uint8_t* labels,
                      float* probs, int* iters, float* resid, cudaStream_t stream);

/* Surface metrics of two uint8 label volumes pred / gt, [S,H,W] (ndim 3) or [H,W] (ndim 2, S = 1), for classes 1..classes-1
 * (2 <= classes <= 16, W <= 4096, at most 2^30 voxels): medpy.metric.binary dc / jc / hd95 / asd with voxelspacing (sz, sy, sx; sz unused for ndim 2)
 * and connectivity 1, i.e. its __surface_distances as val_2D.py:7-15 (calculate_metric_percase), test_2D_fully.py:74-80 and
 * utils/metrics.py:19-25 call it: surface = mask ^ binary_erosion(mask, generate_binary_structure(ndim, 1)) (border voxels are
 * surface, so a [1,H,W] volume differs from its [H,W] slice), distances = distance_transform_edt(~surface, sampling) at the other
 * surface, exact, fp64, evaluated as scipy does.  out: (classes-1) rows of 12 doubles,
 *   {|P&G|, |P|, |G|, |P|G|, nA, nB, sumA, sumB, maxA, maxB, x[lo], x[hi]},
 * A = pred-surface -> gt-surface distances (asd = sumA / nA), B = gt -> pred, x[lo] / x[hi] the order statistics at
 * lo = floor((n-1)*0.95), hi = lo + 1 (both n-1 at the top) of the n = nA + nB distances of both directions, which
 * np.percentile(.., 95) interpolates.  A class whose pred or gt mask is empty keeps 0 in fields 6..11.  Sums are in a fixed
 * order (bit-identical run to run).  ws: wsl_surface_metrics_workspace() bytes, 256-byte aligned, no zeroing needed; out_bytes is a HOST pointer. */
int wsl_surface_metrics_workspace(int ndim, int S, int H, int W, int classes, long long* out_bytes);
int wsl_surface_metrics(const uint8_t* pred, const uint8_t* gt, int ndim, int S, int H, int W, int classes, double sz, double sy,
                        double sx, void* ws, double* out, cudaStream_t stream);

/* ---- network operators (networks/unet.py) ---------------------------------------------------------------- */

/* nn.Conv2d(k=3,pad=1)/(k=1) forward on CUDA cores (unet.py:19,23,55,120); with dgrad-packed weights also the
 * data gradient.  Two channels-last sources model torch.cat([x2,x1],1) (unet.py:67).
 * out_mode 0: bf16 NHWC with CoutStore channels; 1: fp32 NCHW with CoutStore channels; 2: fp32 NHWC; 3: fp16 NHWC.
 * src_f32 (a dtype code): 1 = sources are fp32 (a single-channel image, or fp32 NHWC activations with C %% 8 == 0),
 * 0 = bf16, 2 = fp16; likewise dy_f32 of the weight gradient. */
int wsl_conv_direct(const void* src0, int C0, const void* src1, int C1, int src_f32, const float* wpk,
                    const float* bias, void* out, int out_mode, int N, int H, int W, int CinP, int CoutP,
                    int CoutStore, int ksize, cudaStream_t stream);

/* weight (+bias) gradient of the same convolutions, accumulated into zero-filled fp32 torch-layout grads. */
int wsl_wgrad_direct(const void* src0, int C0, const void* src1, int C1, int src_f32, const void* dy, int dy_f32,
                     int CoutP, float* dw, float* dbias, int N, int H, int W, int CoutReal, int ksize, cudaStream_t stream);

/* first layer (Cin = 1 -> 16, unet.py:81): x fp32 [N,H,W], w fp32 torch layout [16][1][3][3], y bf16 NHWC; and its
 * weight gradient (dw accumulated, zero-filled by the caller; the bias feeds BatchNorm -> zero gradient). */
int wsl_conv_first(const float* x, const float* w, const float* bias, void* y, int dtype, int N, int H, int W, int Cout,
                   float* stat_partials, int* stat_rows_host, cudaStream_t stream);   /* stat_*: as for wsl_conv_tc2 (optional) */
int wsl_wgrad_first(const float* x, const void* dy, int dtype, float* dw, int N, int H, int W, int Cout,
                    cudaStream_t stream);

/* wgmma implicit-GEMM convolution (conv_tc.cu): same contract as wsl_conv_direct for 16-bit NHWC sources (dtype 0 = bf16,
 * 2 = fp16: operands, packed weights and out_mode-0 outputs all have that type) with channel counts that are multiples
 * of 16.  wpk_bf16: [taps][CoutP][CinP] (K-major).  Requires wsl_tc_available(). */
int wsl_tc_available(void);
int wsl_conv_tc(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias,
                void* out, int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype,
                cudaStream_t stream);
/* v2 of the same convolution: persistent CTAs, weights resident in shared memory, one halo load per pixel tile whose
 * nine taps are row-shifted wgmma descriptor views (no reload).  Same contract, except that out_mode must be 0 (16-bit NHWC)
 * or 1 (fp32 NCHW); needs W % 8 == 0 and H % 16 == 0. */
int wsl_conv_tc2(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias,
                 void* out, int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype,
                 float* stat_partials, int* stat_rows_host, cudaStream_t stream);
/* stat_partials (optional, device, >= 592*2*CoutP floats): per-CTA sum / sum-of-squares rows of the stored outputs for the
 * following BatchNorm; *stat_rows_host (optional, HOST int) receives the number of rows written.  wsl_bn_finalize turns
 * the rows into {mean, invstd, scale, shift} and updates the running statistics exactly like wsl_bn_stats. */
int wsl_bn_finalize(const float* partials, int nrows, long long P, int C, const float* gamma, const float* beta,
                    float* running_mean, float* running_var, long long* num_batches_tracked, float momentum, float eps,
                    float* save, float* ss, cudaStream_t stream);
/* wgmma weight gradient (conv_tc.cu): dw (fp32, torch layout [CoutReal][C0+C1][k][k]) += dY^T * X over all pixels.
 * Bias gradients are NOT produced here (see wsl_channel_sum). */
int wsl_wgrad_tc(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                 int W, int CoutReal, int ksize, int dtype, float* partial_ws, long long partial_floats, cudaStream_t stream);
/* v2 of the 3x3 weight gradient: one halo load of X per 16x8 pixel chunk, nine row-shifted descriptor views. */
int wsl_wgrad_tc2(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                  int W, int CoutReal, int ksize, int dtype, cudaStream_t stream);
/* v3: filter columns ride in the MMA's M dimension (A = X halo with one-pixel group stride, B = dY, N = Cout tile). */
int wsl_wgrad_tc3(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                  int W, int CoutReal, int ksize, int dtype, float* partial_ws, long long partial_floats, cudaStream_t stream);
/* partial_ws (optional, partial_floats floats): split-K partial tiles go there and a fixed-order finalize adds them into dw -> the
 * weight gradient is bit-stable run to run; NULL (or too small): fp32 red.global.add, order-dependent in the last bits. */

/* fp16 hi/lo split ("fp16x3") tensor-core parity mode: the reference computes in fp32 (unet.py:18-26); here an fp32 value
 * travels as hi = fp16(v), lo = fp16(v - hi) and a product is a_hi*b_hi + a_lo*b_hi + a_hi*b_lo on kind::f16 with fp32
 * accumulation (22 significant bits).  wsl_split_f32: fp32 NHWC [P][C0] (+ [P][C1] concatenated) -> fp16 [P][2*(C0+C1)]
 * (hi plane | lo plane) of v * 2^k, k chosen per call so that max|v| * 2^k lies in [2^13, 2^14) (fp16's exponent range would
 * otherwise cost small values their lo bits); consumers take &scale3[1] = 2^-k as inv_scale.  wsl_pack_split_weights: torch-layout fp32 weight -> f3 = fp16 [T][CoutP][3*CinP] (hi|hi|lo along
 * K, forward) and, for the input-channel slice, d3 = fp16 [T][SliceP][3*CoutP] (taps flipped, data gradient).
 * wsl_conv_tc_split: conv of a staged tensor with such weights, out fp32 NHWC (out_mode 2) or NCHW (1); needs W %% 16 == 0,
 * H %% 8 == 0.  wsl_wgrad_tc_split: dw += three accumulating weight-gradient launches on the staged X / dY planes. */
int wsl_split_f32(const float* src0, int C0, const float* src1, int C1, long long P, void* dst, float* scale3,
                  cudaStream_t stream);   /* scale3 (3 floats): receives {2^k, 2^-k, scratch}; dst holds the planes of v * 2^k */
int wsl_pack_split_weights(const float* w, int Cout, int Cin, int ksize, int CoutP, int CinP, int ci_begin, int ci_count,
                           void* f3, void* d3, cudaStream_t stream);
int wsl_conv_tc_split(const void* staged, int Cin, const float* inv_scale, const void* wpk3, const float* bias, float* out,
                      int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dilation, cudaStream_t stream);
int wsl_wgrad_tc_split(const void* x_staged, int Cin, const float* x_inv_scale, const void* dy_staged, int CoutP,
                       const float* dy_inv_scale, float* dw, int N, int H, int W, int CoutReal, int ksize, int dilation,
                       cudaStream_t stream);

/* dilated 3x3 convolution of PNet2D's blocks (networks/pnet.py:25-28, dilation = padding = 1, 2, 4, 8, 16) on the per-tap wgmma
 * kernel: tap (dy, dx) is the TMA box at (y0 + dilation*dy, x0 + dilation*dx), out-of-bounds zero fill = the padding; with the flipped /
 * transposed pack it is the data gradient; wsl_wgrad_tc_dil is the matching weight gradient.  LeakyReLU backward without BatchNorm for the
 * 1x1 heads (pnet.py:54-59,75-81). */
int wsl_conv_tc_dil(const void* src0, int C0, const void* src1, int C1, const void* wpk_bf16, const float* bias, void* out,
                    int out_mode, int N, int H, int W, int CoutP, int CoutStore, int ksize, int dtype, int dilation,
                    cudaStream_t stream);
int wsl_wgrad_tc_dil(const void* src0, int C0, const void* src1, int C1, const void* dy, int CoutP, float* dw, int N, int H,
                     int W, int CoutReal, int ksize, int dtype, int dilation, float* partial_ws, long long partial_floats,
                     cudaStream_t stream);
/* nn.LeakyReLU without a BatchNorm in front (pnet.py:60-61,94-95): out = y > 0 ? y : slope*y over n elements of any layout;
 * wsl_lrelu_bwd: out = g * (y > 0 ? 1 : slope) with y the PRE-activation */
int wsl_lrelu_fwd(const void* y, int dtype, float slope, long long n, void* out, cudaStream_t stream);
int wsl_lrelu_bwd(const void* y, int dtype, const void* g, float slope, long long n, void* out, cudaStream_t stream);
/* out[c] += sum over the P pixels of a channels-last bf16 tensor (bias gradient of convs not followed by BN). */
int wsl_channel_sum(const void* x, int dtype, long long P, int C, int Creal, float* out, float* ws, cudaStream_t stream);
/* ws (optional zero-initialised workspace): per-block rows + fixed-order sum by the last block -> bit-stable; NULL: atomicAdd */

/* nn.BatchNorm2d training statistics (unet.py:20,24): save = {mean[C], invstd[C]}, ss = {scale[C], shift[C]};
 * running stats / num_batches_tracked updated in place when non-NULL. */
int wsl_bn_stats(const void* y, int dtype, long long P, int C, const float* gamma, const float* beta, float* running_mean,
                 float* running_var, long long* num_batches_tracked, float momentum, float eps, float* save,
                 float* ss, float* ws, float* raw_sums, cudaStream_t stream);
/* raw_sums (optional, 2C floats): write {sum, sum of squares} there and stop (no save / ss / running update): synchronised BatchNorm
 * all-reduces them over the data-parallel ranks and finalises with wsl_bn_finalize(raw_sums, 1, P_global, ...). */
int wsl_bn_eval_prepare(const float* gamma, const float* beta, const float* running_mean, const float* running_var,
                        float eps, int C, float* ss, cudaStream_t stream);
/* Per-sample BatchNorm training statistics (the batch-1 train-mode forwards of train_s2l.py:221-228 run as one batch): every
 * image of [N][HW][C] gets its own {mean, invstd} -> save [N][2C] and {scale, shift} -> ss [N][2C]; running statistics take the
 * N sequential momentum updates in image order (unbiased variance, n = HW) and num_batches_tracked += N.  Two deterministic
 * launches (per-image partial rows in ws, fixed-order double sums). */
int wsl_bn_stats_ps(const void* y, int dtype, int N, int HW, int C, const float* gamma, const float* beta, float* running_mean,
                    float* running_var, long long* num_batches_tracked, float momentum, float eps, float* save, float* ss, float* ws,
                    cudaStream_t stream);
/* wsl_bn_act_fwd with ss = per-image {scale, shift} [N][2C] from wsl_bn_stats_ps. */
int wsl_bn_act_fwd_ps(const void* y, int dtype, const float* ss, int N, int H, int W, int C, float slope, float drop_p,
                      const uint8_t* mask, unsigned long long seed, const unsigned long long* seed_ptr, void* act,
                      void* pooled, uint8_t* pool_idx, cudaStream_t stream);

/* BN-affine + LeakyReLU(slope) + Dropout(p) (unet.py:20-22) and, when pooled != NULL, MaxPool2d(2) (unet.py:38)
 * of the result.  mask: optional uint8 keep mask (NHWC); NULL -> counter RNG on `seed` (+ *seed_ptr when non-NULL, so a
 * captured CUDA graph draws fresh masks every replay). */
int wsl_bn_act_fwd(const void* y, int dtype, const float* ss, int N, int H, int W, int C, float slope, float drop_p,
                   const uint8_t* mask, unsigned long long seed, const unsigned long long* seed_ptr, void* act,
                   void* pooled, uint8_t* pool_idx, cudaStream_t stream);

/* the same with wsl_bn_finalize folded in (C <= 32): every block derives {scale, shift} from the convolution epilogue's partial rows,
 * block 0 publishes save / ss / running statistics; one launch less on the forward critical path of the full-resolution layers. */
int wsl_bn_finalize_act_fwd(const void* y, int dtype, const float* partials, int nrows, const float* gamma, const float* beta,
                            float* running_mean, float* running_var, long long* num_batches_tracked, float momentum, float eps,
                            float* save, float* ss, int N, int H, int W, int C, float slope, float drop_p, const uint8_t* mask,
                            unsigned long long seed, const unsigned long long* seed_ptr, void* act, void* pooled,
                            uint8_t* pool_idx, cudaStream_t stream);

/* backward of the same chain: dA = g0 + cs1*g1 + maxpool-routed gpool (each optional) -> dY, dgamma, dbeta (added to the
 * existing values when accumulate != 0: a second backward through shared weights, e.g. the mean-teacher student). */
int wsl_bn_bwd(const void* y, int dtype, const float* ss, const float* save, const void* g0, const void* g1, const float* cs1,
               const void* gpool, const uint8_t* pool_idx, const uint8_t* mask, unsigned long long seed,
               const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W, int C, float* dgamma, float* dbeta, float* coef, void* dy, float* ws, int accumulate,
               cudaStream_t stream);

/* synchronised BatchNorm backward: phase 1 = reduction only (local dgamma / dbeta + raw_sums {sum dz, sum dz*xhat}); the caller
 * all-reduces raw_sums; wsl_bn_bwd_coef forms the apply constants from the GLOBAL sums and pixel count; phase 2 = apply only. */
int wsl_bn_bwd_phase(const void* y, int dtype, const float* ss, const float* save, const void* g0, const void* g1, const float* cs1,
                     const void* gpool, const uint8_t* pool_idx, const uint8_t* mask, unsigned long long seed,
                     const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W, int C, float* dgamma,
                     float* dbeta, float* coef, void* dy, float* ws, int accumulate, int phase, float* raw_sums, cudaStream_t stream);
int wsl_bn_bwd_coef(const float* raw_sums, long long P_global, const float* ss, const float* save, int C, float* coef,
                    cudaStream_t stream);

/* first layer (1 -> 16 channels, unet.py:81 in_conv): BatchNorm backward + the convolution's weight gradient in one pass -- dY is
 * formed in registers and never stored (the image needs no data gradient): dgamma / dbeta as wsl_bn_bwd, dw[16][1][3][3] += dY^T * x. */
int wsl_bn_bwd_first(const void* y, int dtype, const float* ss, const float* save, const void* g0, const uint8_t* mask,
                     unsigned long long seed, const unsigned long long* seed_ptr, float drop_p, float slope, int N, int H, int W,
                     float* dgamma, float* dbeta, float* coef, const float* image, float* dw, float* ws, int accumulate,
                     cudaStream_t stream);

/* nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True) (unet.py:56-57) and its transpose. */
int wsl_upsample2x_fwd(const void* t, int dtype, int N, int h, int w, int C, void* u, cudaStream_t stream);
int wsl_upsample2x_bwd(const void* du, int dtype, int N, int h, int w, int C, void* dt, cudaStream_t stream);

/* F.dropout2d(x, 0.5) of the aux branch (unet.py:254-256,344): cs[N*C] in {0, 1/(1-p)}. */
int wsl_chan_mask_gen(unsigned long long seed, const unsigned long long* seed_ptr, int n, float p, float* cs,
                      cudaStream_t stream);
int wsl_chan_scale(const void* a, int dtype, const float* cs, int N, int H, int W, int C, void* d, cudaStream_t stream);

/* FeatureNoise of UNet_CCT_3H's third head (unet.py:270-283, :369): z = uniform(lo, hi) of the feature's [H][W][C] shape (one tensor
 * for the whole batch), out = f * z + f; backward: acc += g * (1 + z) when acc != NULL, else out = g * (1 + z). */
int wsl_uniform_fill(unsigned long long seed, const unsigned long long* seed_ptr, long long n, float lo, float hi, float* out,
                     cudaStream_t stream);
int wsl_feat_noise_fwd(const void* f, int dtype, const float* z, int N, long long hwc, void* out, cudaStream_t stream);
int wsl_feat_noise_bwd(const void* g, int dtype, const float* z, int N, long long hwc, void* acc, void* out, cudaStream_t stream);

/* FCDiscriminator (networks/discriminator.py:58-101; trained by train_deep_adversarial_network_2D.py:107-178), disc_ops.cu.
 * Every nn.Conv2d(k=4, stride=2, padding=1) runs as a 3x3 / stride-1 / pad-1 convolution (wsl_conv_tc, wsl_conv_direct, their
 * dgrad packs and the 3x3 weight gradients) over the space-to-depth tensor T[n, Y, X, (a*2+b)*Cin + c] = x[n, 2Y+a, 2X+b, c] with a
 * structured weight: 4x4 tap k of an axis sits at 3x3 tap (k+1)>>1, phase (k+1)&1; the other slots are zero.  dtype: 0 bf16, 1 fp32.
 * wsl_disc_pack_input: map [N,C0,H,W] and feature [N,C1,H,W] fp32 (conv0 / conv1 inputs, :80-81) -> T [N,H/2,W/2,CP], CP >= 4(C0+C1),
 * channels above 4(C0+C1) zero; wsl_disc_unpack_input_grad: its transpose (dmap / dfeature fp32 NCHW, either may be NULL). */
int wsl_disc_pack_input(const float* map, int C0, const float* feature, int C1, int N, int H, int W, int CP, void* out, int dtype,
                        cudaStream_t stream);
int wsl_disc_unpack_input_grad(const void* dT, int dtype, int N, int H, int W, int CP, int C0, int C1, float* dmap, float* dfeature,
                               cudaStream_t stream);
/* LeakyReLU(slope) then Dropout2d (:86-87, :90-91; cs [N*C] in {0, 2} or NULL) fused with space-to-depth: y [N,H,W,C] -> T [N,H/2,W/2,4C];
 * slope 1 and cs NULL is the plain repacking of conv0 + conv1, which has no activation (:83-85).  wsl_d2s_act_bwd: depth-to-space of
 * dT times cs times LeakyReLU'(y) (y = the pre-activation; NULL allowed when slope == 1). */
int wsl_s2d_act_fwd(const void* y, int dtype, int N, int H, int W, int C, float slope, const float* cs, void* out, cudaStream_t stream);
int wsl_d2s_act_bwd(const void* dT, const void* y, int dtype, int N, int H, int W, int C, float slope, const float* cs, void* dy,
                    cudaStream_t stream);
/* 4x4 torch-layout weights w0 [Cout,C0,4,4] (+ w1 [Cout,C1,4,4], the second source of the first layer) -> structured 3x3 torch layout
 * w3 [Cout,CP,3,3] for wsl_pack_conv_weights; bias_out (optional) = b0 (+ b1): conv0 + conv1 as one convolution.  wsl_disc_gather_wgrad:
 * the 16 used slots of a 3x3 weight gradient dw3 [Cout,CP,3,3] -> dw0 (and dw1), written, not accumulated. */
int wsl_disc_scatter_weights(const float* w0, const float* b0, int C0, const float* w1, const float* b1, int C1, int Cout, int CP,
                             float* w3, float* bias_out, cudaStream_t stream);
int wsl_disc_gather_wgrad(const float* dw3, int Cout, int CP, int C0, int C1, float* dw0, float* dw1, cudaStream_t stream);
/* Head (:94-97): LeakyReLU(slope) -> AvgPool2d(7) of the 16x16 conv4 map y [N,16,16,C] (rows / columns 0..13) -> flatten in NCHW
 * order (c*4 + i*2 + j) -> Linear(4C, 2): pooled [N,4C] (kept for the backward), logits [N,2] fp32.  wsl_disc_head_bwd: dy [N,16,16,C]
 * (zero at rows / columns 14, 15) and the classifier gradients dwc [2,4C], dbc [2] (written; batch sums in a fixed order; both NULL: dy
 * only, as in the DAN script's phase 1, whose discriminator gradients train_deep_adversarial_network_2D.py:176 discards). */
int wsl_disc_head_fwd(const void* y, int dtype, int N, int C, float slope, const float* wc, const float* bc, float* pooled, float* logits,
                      cudaStream_t stream);
int wsl_disc_head_bwd(const float* dlogits, const float* pooled, const void* y, int dtype, int N, int C, float slope, const float* wc,
                      float* dwc, float* dbc, void* dy, cudaStream_t stream);
/* F.cross_entropy of the discriminator's logits [N,2] (train_deep_adversarial_network_2D.py:155-156 and :175): target 1 for the first
 * n_ones rows, 0 for the rest (DAN_target, :135-137).  loss[0] = mean NLL (unweighted); dlogits [N,2] = (softmax - onehot) / N * weight,
 * weight read from weight_ptr (device) when non-NULL, so a captured graph follows the ramped consistency weight (:151-152). */
int wsl_disc_ce(const float* logits, int N, int n_ones, const float* weight_ptr, float weight, float* loss, float* dlogits,
                cudaStream_t stream);

/* layout helpers at the API boundary */
int wsl_nchw_f32_to_nhwc(const float* src, int N, int Creal, int H, int W, int CP, void* dst, int dtype, float scale,
                         cudaStream_t stream);   /* dst = scale * src (the loss scale of the fp16 modes; 1 otherwise) */
int wsl_nhwc_to_nchw_f32(const void* src, int dtype, int N, int C, int H, int W, float* dst, cudaStream_t stream);

/* fp32 torch-layout conv weight -> packed operands (any output may be NULL), see net_ops.cu */
int wsl_pack_conv_weights(const float* w, int Cout, int Cin, int ksize, int CoutP, int CinP, int ci_begin,
                          int ci_count, float* wf, float* wd, void* bf, void* bd, int dtype16, cudaStream_t stream);

/* all layers in one launch: table = n_entries x 13 int64 {w, wf, wd, bf, bd, Cout, Cin, T, CoutP, CinP, ci_begin,
 * ci_count, first_item} in device memory (pointers as integers), items = T*CoutP*CinP per entry */
int wsl_pack_conv_weights_batched(const long long* table, int n_entries, long long total_items, int dtype16,
                                  cudaStream_t stream);   /* dtype16: 0 = bf16, 2 = fp16 for the 16-bit packs bf / bd */

/* optim.SGD(lr, momentum, weight_decay).step() over a flat fp32 buffer (train_weakly_supervised_pCE_2D.py:79-80,104);
 * lr is read from lr_ptr (device) when non-NULL so a captured CUDA graph follows the poly schedule (:106-108);
 * grad_scale = 1/world_size turns the all-reduced gradient sum into DDP's mean. */
int wsl_sgd_step(float* param, const float* grad, float* mom, long long n, const float* lr_ptr, float lr,
                 float momentum, float weight_decay, float grad_scale, cudaStream_t stream);

/* optim.Adam(lr, betas, eps, weight_decay=0).step() over a flat fp32 buffer (train_deep_adversarial_network_2D.py:112-113,178), in
 * the order and rounding of torch's multi-tensor path: exp_avg.lerp_(g, 1-beta1); exp_avg_sq.mul_(beta2).addcmul_(g, g, 1-beta2);
 * denom = sqrt(exp_avg_sq) / bc2_sqrt + eps; param -= step_size * exp_avg / denom, with step_size = lr / (1 - beta1^t) and
 * bc2_sqrt = sqrt(1 - beta2^t) for the step count t (after its increment).  The doubles are rounded to fp32 as torch rounds its
 * Python scalars; scalars_ptr (device, {step_size, bc2_sqrt} in fp32) replaces the by-value pair so a captured graph follows t. */
int wsl_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, long long n, const float* scalars_ptr,
                  double step_size, double bc2_sqrt, double beta1, double beta2, double eps, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* WSL4MIS_B200_H */
