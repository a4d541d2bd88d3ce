/*
 * frl_b200.h — C ABI of the H100 (sm_90a) data-parallel training-step kernels.
 *
 * The reference (facebookresearch/FRL-Distributed-ML-Scaffold) has no native boundary of its
 * own: its step arithmetic runs inside PyTorch.  Each entry point below replaces the PyTorch
 * call the reference makes at the cited line; the reference-side binding is the ctypes stub in
 * INTEGRATION.md.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (the library never allocates or
 *     frees caller-visible memory) unless the parameter name ends in `_host`;
 *     `*_mapped` pointers may be pinned, device-mapped host memory;
 *   - every function enqueues work on `stream` (a cudaStream_t passed as void*) and returns
 *     immediately; nothing synchronises;
 *   - return value: 0 = ok, negative = argument error (FRL_E_*), positive = cudaError_t of
 *     the launch; `frl_last_error()` gives a thread-local message;
 *   - no exceptions, no longjmp, no global mutable state except the launch counter.
 *   - dtype codes: FRL_F32 = 0, FRL_BF16 = 1, FRL_U8 = 2, FRL_I64 = 3.
 */
#ifndef FRL_B200_H
#define FRL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FRL_ABI_VERSION 1

enum { FRL_F32 = 0, FRL_BF16 = 1, FRL_U8 = 2, FRL_I64 = 3 };
enum { FRL_E_ARG = -1, FRL_E_ALIGN = -2, FRL_E_DTYPE = -3, FRL_E_TOO_MANY = -4 };

int          frl_abi_version(void);
const char*  frl_last_error(void);
/* number of kernels this library has launched since load / since the last reset */
uint64_t     frl_launch_count(void);
void         frl_launch_count_reset(void);
/* SM count and sm arch (major*10+minor) of the current device; <0 on error */
int          frl_device_sm_count(void);
int          frl_device_arch(void);

/* ------------------------------------------------------------------------------------------
 * K2 — fused optimizer update over a flat bucket of the parameter arena.
 * Replaces torch.optim.{SGD,Adam,RMSprop}.step() (reference solver.py:162-188, called at
 * solver_worker.py:592) AND the DDP reducer's scale / copy-out passes (reference
 * solver.py:287-289): the reduced gradient is read once, straight from the bucket.
 *
 *   p        fp32 master weights [n]           (read + written)
 *   g        gradient bucket [n], dtype g_dtype (FRL_F32 or FRL_BF16), read once
 *   p_lp     optional bf16 shadow weights [n] (written), NULL when the model runs in fp32
 *   grad_scale      host scalar multiplied into g (1/world_size for the DDP mean)
 *   grad_scale_dev  optional device scalar multiplied in as well (clip coefficient written
 *                   by frl_grad_sumsq_clip), NULL = 1
 * All arrays must be 16-byte aligned; n is arbitrary (scalar tail).
 * Hyper-parameters are doubles (Python floats): derived constants such as 1-beta2 or the
 * Adam bias corrections are formed in double and rounded to fp32 once, exactly as torch does
 * when it hands Python scalars to fp32 tensor ops.
 *   dyn      optional DEVICE array of per-step scalars that override the by-value arguments,
 *            so a CUDA graph that captured the launch stays valid while they change:
 *            SGD / RMSprop: dyn[0] = lr ;  Adam: dyn[0] = -lr/(1-beta1^t), dyn[1] = sqrt(1-beta2^t).
 * Update rules are torch 2.11's (L2-coupled weight decay: g += wd * p first).
 * ---------------------------------------------------------------------------------------- */

/* SGD: buf = first_step ? g : mu*buf + (1-dampening)*g ; p -= lr*buf.   mu == 0: buf may be NULL. */
int frl_sgd_momentum(float* p, const void* g, float* buf, void* p_lp, int64_t n,
                     double lr, double mu, double dampening, double wd,
                     double grad_scale, const float* grad_scale_dev, const float* dyn,
                     int first_step, int g_dtype, void* stream);

/* Adam (coupled L2, optional amsgrad when vmax != NULL).  `step` is the 1-based step count
 * used for the bias corrections (computed in double on the host side of the call). */
int frl_adam(float* p, const void* g, float* m, float* v, float* vmax, void* p_lp, int64_t n,
             double lr, double beta1, double beta2, double eps, double wd, int64_t step,
             double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
             void* stream);

/* RMSprop (not centered): sq = alpha*sq + (1-alpha)*g^2 ; avg = sqrt(sq)+eps ;
 * mu > 0: buf = mu*buf + g/avg ; p -= lr*buf     else: p -= lr*g/avg  (buf may be NULL). */
int frl_rmsprop(float* p, const void* g, float* sq, float* buf, void* p_lp, int64_t n,
                double lr, double alpha, double eps, double wd, double mu,
                double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
             void* stream);

/* ------------------------------------------------------------------------------------------
 * K12 — weight-gradient GEMM gw = dz^T x on the tensor cores (persistent, TMA + WGMMA), with
 * an optional SGD update of the same weights in its epilogue.
 *   dz [rows, out] (leading dimension ld_dz), x [rows, in] (ld_x): row-major bf16;
 *   gw [out, in]: contiguous bf16, written in both forms (fp32 accumulation, rounded once).
 *   out % 128 == 0, in % 256 == 0, rows % 64 == 0 (FRL_E_ARG); every pointer 16-byte aligned
 *   and ld_dz, ld_x multiples of 8 (FRL_E_ALIGN / FRL_E_ARG).
 * frl_dw_gemm     : gw only (what torch.mm(dz.t(), x, out=gw) computes).
 * frl_dw_gemm_sgd : gw, then frl_sgd_momentum's update of p / buf / p_lp ([out, in], contiguous)
 *                   applied to exactly the bf16 gw just written: bit-identical to frl_dw_gemm
 *                   followed by frl_sgd_momentum(g_dtype = FRL_BF16) over the slice.
 * ---------------------------------------------------------------------------------------- */
int frl_dw_gemm(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                int64_t out, int64_t in, void* gw, void* stream);
int frl_dw_gemm_sgd(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                    int64_t out, int64_t in, void* gw, float* p, float* buf, void* p_lp,
                    double lr, double mu, double dampening, double wd, double grad_scale,
                    const float* dyn, int first_step, void* stream);

/* ------------------------------------------------------------------------------------------
 * K2-mt / K1 — multi-tensor forms of the update and the bucket flatten.
 * Replaces the DDP reducer's per-tensor bucket copy-in / copy-out (reference solver.py:287-289 ->
 * torch Reducer) for parameters whose gradients autograd allocates itself (convolutions,
 * normalisation layers): a SEGMENT TABLE in device memory names, per parameter tensor, where its
 * gradient lies, its dtype, its arena offset (a multiple of 8 elements) and its length.
 *   tile_prefix_dev[s] = number of tiles of segments 0..s-1 (int64, n_segs + 1 entries), a tile
 *   being frl_mt_tile_elems() arena elements of ONE segment; n_tiles = tile_prefix_dev[n_segs];
 *   tile_seg_dev[t] = segment index of tile t (int32, n_tiles entries).
 *   Gradient pointers must be 16-byte aligned; tensors contiguous in the parameter's layout.
 * frl_flatten_grads : arena_grad[arena_off + i] = cast(g[i] * scale) for every segment, one launch.
 * frl_*_mt          : the K2 update of the listed segments reading g in place; p / state / p_lp
 *                     are the ARENA BASE pointers (offset 0), other arguments as in K2.
 * ---------------------------------------------------------------------------------------- */
typedef struct frl_grad_seg {
    const void* g;          /* device pointer of the gradient tensor (g_dtype elements) */
    int64_t     arena_off;  /* first arena element of the parameter */
    int64_t     numel;      /* elements of the parameter */
    int32_t     g_dtype;    /* FRL_F32 | FRL_BF16 */
    int32_t     _pad;
} frl_grad_seg;

int64_t frl_mt_tile_elems(void);

int frl_flatten_grads(const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                      const int32_t* tile_seg_dev, int64_t n_tiles, void* arena_grad, int dst_dtype,
                      double scale, void* stream);

int frl_sgd_momentum_mt(float* p, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                        const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                        double lr, double mu, double dampening, double wd, double grad_scale,
                        const float* grad_scale_dev, const float* dyn, int first_step, void* stream);

int frl_adam_mt(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double beta1,
                double beta2, double eps, double wd, int64_t step, double grad_scale,
                const float* grad_scale_dev, const float* dyn, void* stream);

int frl_rmsprop_mt(float* p, float* sq, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                   const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double alpha,
                   double eps, double wd, double mu, double grad_scale, const float* grad_scale_dev,
                   const float* dyn, void* stream);

/* ------------------------------------------------------------------------------------------
 * K2-lw — layer-wise adaptive updates over a segment table (an extension: the reference offers
 * SGD, Adam and RMSprop only).  LARS (You et al. 2017) is layer adaptation on the SGD rule, LAMB
 * (You et al. 2019) on the Adam rule.  Segment table, p / state / p_lp and the other arguments
 * as in frl_*_mt; additionally
 *   n_segs         segments in the table
 *   seg_flags_dev  int32 [n_segs]: FRL_LW_ADAPTED = the tensor is adapted (2 or more dimensions:
 *                  Linear / conv weights, embeddings; 0-/1-D tensors such as biases, normalisation
 *                  affine and criterion parameters get ratio 1 and no weight decay);
 *                  FRL_LW_CLIPPED = grad_scale_dev multiplies this segment's gradient (model
 *                  parameters under global-norm clipping; criterion parameters are not clipped)
 *   ratio_dev      fp32 [n_segs], written: the trust ratio each tensor was updated with
 *   scratch        frl_layerwise_scratch_bytes(n_tiles, n_segs) bytes, zero-initialised once
 * Per segment, fp32, with g^ = g * grad_scale (* *grad_scale_dev if FRL_LW_CLIPPED), w the master
 * weights before the update, lr the scheduled rate:
 *   LARS (trust coefficient eta = 0.001, fixed; mu = momentum; no dampening):
 *     adapted:     ratio = eta*||w|| / (||g^|| + wd*||w||) if ||w|| > 0 and ||g^|| > 0, else 1;
 *                  d = ratio * (g^ + wd*w)
 *     not adapted: d = g^   (ratio 1, no weight decay)
 *     buf = first_step ? d : mu*buf + d ; w -= lr*buf        (mu == 0: w -= lr*d, buf may be NULL)
 *   LAMB (lam = wd if adapted else 0; t = step, >= 1):
 *     m = m + (1-beta1)*(g^ - m) ; v = beta2*v + (1-beta2)*g^^2
 *     u = (m / bc1) / (sqrt(v) / sqrt(bc2) + eps) + lam*w     bc_i = 1 - beta_i^t
 *     ratio = ||w|| / ||u|| if adapted and ||w|| > 0 and ||u|| > 0, else 1 ;  w -= lr*ratio*u
 *     The weight decay is DECOUPLED (part of u), unlike frl_adam's L2-coupled decay.
 * A non-finite gradient yields non-finite weights (a NaN norm takes the ratio-1 branch, which
 * passes the NaN on).  Norms: fp32 per tile, folded per tensor in double in tile order (no float
 * atomics, deterministic).  Two launches: stats (LAMB writes m, v here) and apply.
 *   dyn  LARS: dyn[0] = lr ;  LAMB: dyn[0] = lr, dyn[1] = 1/(1-beta1^t), dyn[2] = sqrt(1-beta2^t).
 * ---------------------------------------------------------------------------------------- */
enum { FRL_LW_ADAPTED = 1, FRL_LW_CLIPPED = 2 };
int64_t frl_layerwise_scratch_bytes(int64_t n_tiles, int64_t n_segs);
int frl_lars_mt(float* p, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                int64_t n_segs, const int32_t* seg_flags_dev, float* ratio_dev, void* scratch,
                double lr, double mu, double wd, double grad_scale, const float* grad_scale_dev,
                const float* dyn, int first_step, void* stream);
int frl_lamb_mt(float* p, float* m, float* v, void* p_lp, const frl_grad_seg* segs_dev,
                const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                int64_t n_segs, const int32_t* seg_flags_dev, float* ratio_dev, void* scratch,
                double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream);

/* ------------------------------------------------------------------------------------------
 * K10 — gradient accumulation (an extension: the reference has no accumulation).  Several
 * microbatches per optimizer update: after each microbatch's backward, one launch folds every
 * gradient of a K2-mt segment table into an fp32 accumulator.
 *   acc[seg.arena_off + i] = (first ? 0 : acc[seg.arena_off + i]) + w * g[i]   for every segment,
 *   fp32, computed as fmaf(w, g, base); a segment with g == NULL contributes 0 (so `first`
 *   zeroes it, and without `first` it is not touched).
 * acc: fp32 arena-shaped vector, 16-byte aligned, covering every segment's arena_off + numel
 * rounded up to 4; segment table as in K2-mt (any mix of FRL_F32 / FRL_BF16 gradients,
 * arena-resident or read in place).  Elements outside every segment are untouched.
 * dyn: optional device fp32[2] overriding the by-value arguments: dyn[0] = w, dyn[1] != 0 -> first.
 * Graph-capturable: no host reads, no allocation.  n_tiles == 0: returns 0, launches nothing.
 * ---------------------------------------------------------------------------------------- */
int frl_grad_accumulate_mt(float* acc, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                           const int32_t* tile_seg_dev, int64_t n_tiles, double w, int first,
                           const float* dyn, void* stream);

/* ------------------------------------------------------------------------------------------
 * K11 — weight EMA (an extension: the reference has no EMA).  Replaces the
 * torch.optim.swa_utils.AveragedModel(..., multi_avg_fn=get_ema_multi_avg_fn(decay))
 * .update_parameters(model) call a user would add after optimizer.step() (reference
 * solver_worker.py:592): one streaming pass over the model range of the fp32 master weights,
 *   ema[i] = lerp(ema[i], p[i], (float)w)   for i < n,
 * with torch's lerp formula  |w| < 0.5 ? e + w*(p - e) : p - (p - e)*(1 - w),  each branch one
 * fmaf.  The caller passes w = 1 - decay (formed in double).  12 B per element.
 * ema, p: fp32, 16-byte aligned (FRL_E_ALIGN); n >= 0 and 0 <= w <= 1 (FRL_E_ARG); every check
 * is made before any launch.  Graph-capturable: no host reads, no allocation.  n == 0: returns 0,
 * launches nothing.
 * ---------------------------------------------------------------------------------------- */
int frl_weight_ema(float* ema, const float* p, int64_t n, double w, void* stream);

/* ------------------------------------------------------------------------------------------
 * K3 — global gradient norm for clipping.
 * Replaces torch.nn.utils.clip_grad_norm_ (reference solver_worker.py:588-591): one pass
 * over the model-parameter range of the gradient arena.
 *   out[0] = sum(g^2) * pre_scale^2,  out[1] = sqrt(out[0]),
 *   out[2] = min(1, max_norm / (out[1] + 1e-6))   (the coefficient K2 reads)
 * As in clip_grad_norm_ (clamp(max=1)), a NaN gradient makes out[2] NaN, so every clipped
 * gradient becomes NaN; an inf gradient makes it 0 (NaN only where the gradient was inf).
 * scratch: >= frl_reduce_scratch_floats() floats + 1 uint32 ticket, zero-initialised once.
 * Deterministic: fixed-order two-stage reduction.
 * ---------------------------------------------------------------------------------------- */
int64_t frl_reduce_scratch_bytes(void);
int frl_grad_sumsq_clip(const void* g, int64_t n, int g_dtype, float pre_scale, float max_norm,
                        float* out3, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * K4 — fused multitask criterion.
 * Replaces ParallelCriterion.compute_split_loss/forward (reference criteria.py:42-61), the
 * nn.MSELoss / nn.CrossEntropyLoss kernels underneath, MaskedLoss's gather
 * (criteria.py:267-287) and the isnan()/item() syncs of the loop (solver_worker.py:486-487,
 * 569).
 * A task whose mask selects nothing gives the reference's inner(out - out, tgt - tgt): 0 for MSE,
 * log C for CE, or NaN for CE with ignore_index == 0 (every label of tgt - tgt is 0, so every
 * row is ignored), eps * log C for CE_PROB, with a zero gradient.  Two differences remain, both
 * only with non-finite outputs: the reference's out - out is NaN where an output is inf or NaN,
 * which makes that loss NaN, but the kernels never read a masked-out output, so they still give
 * 0 / log C; and torch's gradient of a NaN row whose label is ignore_index is NaN, where the
 * kernels write 0.
 * Cross-entropy with label smoothing eps (torch's F.cross_entropy, mean reduction; x a row's
 * logits, lse its log-sum-exp, C = cols):
 *   FRL_LOSS_CE, class index y:  row loss = lse - (1-eps) x_y - (eps/C) sum_c x_c, summed over the
 *     selected rows whose label is not ignore_index and divided by their count;
 *     gradient = (softmax - (1-eps) e_y - eps/C) * coef.
 *   FRL_LOSS_CE_PROB, probabilities q (rows not renormalised), q' = (1-eps) q + eps/C:
 *     row loss = sum_c q'_c (lse - x_c), divided by the number of selected rows;
 *     gradient = (softmax * sum_c q'_c - q') * coef.
 *   With eps == 0 and class indices the kernels compute what they computed before soft targets.
 * Left to the caller's composed torch ops: class weights, and per-position probability targets.
 * ---------------------------------------------------------------------------------------- */
#define FRL_MAX_TASKS 8
enum { FRL_LOSS_MSE = 0, FRL_LOSS_CE = 1, FRL_LOSS_CE_PROB = 2 };

typedef struct frl_task_desc {
    int32_t     kind;         /* FRL_LOSS_MSE | FRL_LOSS_CE | FRL_LOSS_CE_PROB */
    int32_t     out_dtype;    /* FRL_F32 | FRL_BF16 : dtype of `out` (and of `dout`) */
    int32_t     tgt_dtype;    /* MSE, CE_PROB: FRL_F32 | FRL_BF16 ; CE: FRL_I64 */
    int32_t     ignore_index; /* CE only (torch default -100) */
    const void* out;          /* model output  [rows, cols] row-major contiguous */
    const void* tgt;          /* MSE, CE_PROB: [rows, cols] ; CE: int64 class index [rows] */
    const uint8_t* mask;      /* optional (MaskedLoss): nonzero = use ; numel = rows*cols/mask_inner
                                 (CE / CE_PROB: one entry per row) */
    void*       dout;         /* backward only: gradient wrt out, same shape/dtype as out */
    int64_t     rows;
    int64_t     cols;
    int64_t     mask_inner;   /* elements of `out` covered by one mask entry (1 or cols ...) */
    float       weight;       /* loss weight w_i */
    float       label_smoothing;  /* eps in [0, 1], CE / CE_PROB only (0 for MSE) */
} frl_task_desc;

/* scratch bytes for T tasks (partials + ticket); zero-initialise once */
int64_t frl_criteria_scratch_bytes(int n_tasks);

/* forward: losses[0] = sum_i w_i*L_i (left-to-right), losses[1+i] = w_i*L_i.
 *   aux[i]      = 1/count_i (0 if nothing selected) for the backward
 *   lse[...]    = per-row slots of every CE / CE_PROB task, in task order: rows floats (the
 *                 log-sum-exp) for a CE task, 2 * rows for a CE_PROB task (the log-sum-exp of
 *                 every row, then sum_c q'_c of every row); sum(rows) + sum(rows of CE_PROB) in all
 *   sink_mapped = optional second destination of losses[0..T] (e.g. a row of a pinned loss
 *                 log), nan_flag_mapped = optional int set to 1 when losses[0] is NaN.
 * Argument errors (before any launch): a kind other than the three, eps outside [0, 1], eps != 0
 * on an MSE task, a CE_PROB target that is not FRL_F32 / FRL_BF16, a CE / CE_PROB mask that is
 * not per row. */
int frl_criteria_forward(const frl_task_desc* tasks_host, int n_tasks,
                         float* losses, float* aux, float* lse,
                         float* sink_mapped, int32_t* nan_flag_mapped,
                         void* scratch, void* stream);

/* backward: dout_i = (gl[0] + gl[1+i]) * w_i * dL_i/dout_i, gl = gradient wrt losses[0..T]
 * (device, fp32 [1+T]); reads aux / lse written by the forward. */
int frl_criteria_backward(const frl_task_desc* tasks_host, int n_tasks,
                          const float* grad_losses, const float* aux, const float* lse,
                          void* stream);

/* ------------------------------------------------------------------------------------------
 * K5 — device-side batch preprocessing.
 * Batched replacement of the per-sample MultifieldTransform arithmetic (reference
 * transform.py:25-38, multitask_problem.py:56-71): dst = (src * scale[c] + bias[c]), with
 * c = (i / inner) % channels, converting FRL_U8|FRL_F32|FRL_BF16 -> FRL_F32|FRL_BF16.
 * scale/bias: device fp32 [channels]; NULL scale = 1, NULL bias = 0.
 * ---------------------------------------------------------------------------------------- */
int frl_preproc_affine(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n,
                       int64_t inner, int64_t channels, const float* scale, const float* bias,
                       void* stream);

/* ------------------------------------------------------------------------------------------
 * K5a — on-device image augmentation: crop box + bilinear resize + horizontal flip + per-channel
 * affine in one pass (an extension: the reference's Problems augment per sample on the host,
 * inside their MultifieldTransform).
 *   src        uint8 [B, C, H, W] contiguous, 1 <= C <= 4
 *   idx        int64 [B] (device): the dataset row of each image, keys its random draws
 *   seed, epoch  the rest of the key; nothing else (batch size, order, rank) enters the draws
 *   mode       FRL_AUG_RRC         random resized crop, area share in [smin, smax], aspect in [rmin, rmax]
 *              FRL_AUG_PAD_CROP    random out_h x out_w crop of the image zero-padded by `pad` per side
 *              FRL_AUG_CENTER_RESIZE  centred round(H*eval_crop) x round(W*eval_crop) box, resized
 *              FRL_AUG_CENTER_CROP    centred out_h x out_w box (zero fill outside the image)
 *   flip       0/1: mirror with p = 1/2 (never in the two CENTER modes)
 *   scale/bias device fp32 [C]; NULL scale = 1, NULL bias = 0
 *   dst        [B, C, out_h, out_w] of dst_dtype (FRL_F32 | FRL_BF16)
 *   params_out optional int32 [B, 5]: (top, left, h, w, flipped) of each sample's box
 *
 * Sample parameters (oracle/augment_np.py restates them):
 *   draws: Philox4x32-10, key (lo32(seed), hi32(seed)), counter (lo32(i), hi32(i), epoch, j) for
 *     block j of sample i = idx[b]; each block gives words w0..w3.
 *     u(w) = (w >> 8) * 2^-24;  an integer in [0, n) is (uint64(w) * n) >> 32.
 *   RRC (torchvision RandomResizedCrop.get_params), in double: attempt t = 0..9 uses block t:
 *     area = H*W * (smin + u(w0)*(smax - smin)); aspect = exp(log rmin + u(w1)*(log rmax - log rmin))
 *     w = rint(sqrt(area*aspect)), h = rint(sqrt(area/aspect))  (rint: half to even, Python's round)
 *     accepted if 0 < w <= W and 0 < h <= H: top = int(w2, H-h+1), left = int(w3, W-w+1).
 *     No attempt accepted: the ratio-clamped centre crop, r = W/H:
 *       r < rmin: w = W, h = rint(W/rmin); r > rmax: h = H, w = rint(H*rmax); else h = H, w = W;
 *       h, w at least 1; top = (H-h)/2, left = (W-w)/2 (floor).
 *   PAD_CROP: block 0: top = int(w0, H+2p-out_h+1) - p, left = int(w1, W+2p-out_w+1) - p; h = out_h, w = out_w.
 *   CENTER_RESIZE: h = rint(H*eval_crop), w = rint(W*eval_crop); CENTER_CROP: h = out_h, w = out_w;
 *     both: top = rint((H-h)/2), left = rint((W-w)/2) (torchvision center_crop).
 *   flip (RRC / PAD_CROP with flip != 0): block 10, flipped = w0 >> 31.
 * Pixels: bilinear, align_corners=False, no antialiasing (torch interpolate on the crop): per axis
 *   s = (float)crop / (float)out, src = max(fmaf(s, o + 0.5f, -0.5f), 0) in fp32, taps i0 = (int)src and
 *   min(i0 + 1, crop - 1), blend in fp32; crop pixels outside the image read 0 (so the normalised
 *   fill is bias[c]).  A crop the size of the output is an exact copy.  A flipped sample's output
 *   column x takes the resized column out_w-1-x.  dst = round_nearest(fmaf(v, scale[c], bias[c])).
 * Graph-capturable: no host reads, no allocation.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_AUG_RRC = 0, FRL_AUG_PAD_CROP = 1, FRL_AUG_CENTER_RESIZE = 2, FRL_AUG_CENTER_CROP = 3 };
int frl_augment_images(const void* src, int64_t batch, int channels, int height, int width,
                       const int64_t* idx, uint64_t seed, int epoch, int mode,
                       double smin, double smax, double rmin, double rmax, double eval_crop, int pad,
                       int flip, const float* scale, const float* bias, void* dst, int dst_dtype,
                       int out_h, int out_w, int32_t* params_out, void* stream);

/* K5a with Mixup / CutMix in the same pass (an extension: the usual large-batch ImageNet recipe,
 * Zhang et al. 2018 / Yun et al. 2019).  Arguments as frl_augment_images, plus
 *   mix_mode   FRL_MIX_MIXUP or FRL_MIX_CUTMIX;  lam in [0, 1];  lam1 = 1 - (double)lam rounded once
 *              to fp32
 *   box_*      CutMix box [box_y0, box_y1) x [box_x0, box_x1) on the output image (inside it;
 *              ignored by Mixup)
 * Sample p is paired with sample j = B-1-p.  With a_p, a_j the fp32 values K5a would round to the
 * output dtype for the same pixel (the same boxes, drawn as K5a draws them):
 *   Mixup:  out_p = __fadd_rn(__fmul_rn(lam, a_p), __fmul_rn(lam1, a_j))
 *   CutMix: out_p = a_j inside the box, a_p outside
 * and only that final store rounds.  The middle sample of an odd batch, and params_out, are
 * written exactly as by frl_augment_images.  Grid (ceil(B/2), ceil(out_h/8)): one CTA per pair.
 *
 * frl_mix_targets: the target fields of the same batch, one launch per field, partner j = B-1-i.
 *   src_dtype FRL_I64: src int64 [B] labels of n_classes >= 2 classes (inner must be 1); dst fp32
 *     [B, n_classes] = lam at y_i plus lam1 at y_j (fp32 adds onto 0); a row whose y_i or y_j lies
 *     outside [0, n_classes) is NaN, so a NaN-loss check fires without a host read.
 *   src_dtype FRL_F32 | FRL_BF16: src [B, inner], dst of the same dtype and shape =
 *     round(__fadd_rn(__fmul_rn(lam, t_i), __fmul_rn(lam1, t_j))).
 *   lam = 1 gives one-hot rows (labels) and t_i (finite values): the targets of an unmixed batch.
 * Graph-capturable: no host reads, no allocation.  Every argument check comes before any launch.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_MIX_MIXUP = 1, FRL_MIX_CUTMIX = 2 };
int frl_augment_mix_images(const void* src, int64_t batch, int channels, int height, int width,
                           const int64_t* idx, uint64_t seed, int epoch, int mode,
                           double smin, double smax, double rmin, double rmax, double eval_crop, int pad,
                           int flip, const float* scale, const float* bias, void* dst, int dst_dtype,
                           int out_h, int out_w, int32_t* params_out, int mix_mode, float lam,
                           int box_y0, int box_y1, int box_x0, int box_x1, void* stream);
int frl_mix_targets(const void* src, int src_dtype, int64_t batch, int64_t inner, int n_classes, float lam,
                    void* dst, void* stream);

/* dtype conversion / scaled copy used by the arena (master -> shadow refresh after a
 * checkpoint load, gradient flatten for modules the arena cannot write into directly):
 * dst = src * scale. */
int frl_cast_scale(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n,
                   float scale, void* stream);

/* ------------------------------------------------------------------------------------------
 * K6 — column sum: out[c] (+)= sum_r x[r, c], x row-major [rows, cols].
 * The bias gradient of a linear layer, written straight into the gradient arena; replaces the
 * generic reduction autograd runs inside `total_loss.backward()` (reference
 * solver_worker.py:586).  accumulate != 0 adds to `out` (a layer applied twice in one step).
 * rows == 0 (an empty batch; the matrices may then be null) stores 0, or leaves `out` as it is
 * when accumulating.
 * scratch: frl_colsum_scratch_bytes(rows, cols) bytes, zero-initialised once; deterministic.
 * ---------------------------------------------------------------------------------------- */
int64_t frl_colsum_scratch_bytes(int64_t rows, int64_t cols);
int frl_colsum(const void* x, int x_dtype, int64_t rows, int64_t cols, void* out, int out_dtype,
               int accumulate, void* scratch, void* stream);
/* K6b — the same pass with ReLU's backward folded in, for a Linear+ReLU pair: dz[r,c] =
 * threshold_backward(dy, act, 0)[r,c] = act[r,c] <= 0 ? 0 : dy[r,c], so a NaN activation passes dy
 * through as torch's ReLU backward does (act = the layer's forward output; dy, act, dz share dtype
 * and the [rows, cols] layout; dz may alias dy) and out[c] (+)= sum_r dz[r,c].  Replaces autograd's
 * threshold_backward kernel plus the bias-gradient reduction (reference solver_worker.py:586). */
int frl_drelu_colsum(const void* dy, const void* act, void* dz, int dtype, int64_t rows, int64_t cols,
                     void* out, int out_dtype, int accumulate, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------
 * K7 — fused gradient all-reduce + optimizer update + weight broadcast over NVSwitch multicast
 * (world_size > 1).  Replaces, per gradient bucket, the DDP reducer's ncclAllReduce
 * (reference solver.py:287-289, run inside solver_worker.py:586) AND optimizer.step()
 * (solver_worker.py:592) with one kernel: barrier | g = multimem.ld_reduce over all ranks'
 * bucket copies | update this rank's 1/world shard | multimem.st the new weights into every
 * replica | barrier.
 *
 *   p, state...        LOCAL fp32 master / optimizer-state slices of the bucket [n]
 *   mc_g               MULTICAST address of the bucket's gradient slice (symmetric allocation)
 *   mc_out             MULTICAST address of the slice every rank's module reads its weights
 *                      from: bf16 shadow weights (g_dtype FRL_BF16) or the fp32 master
 *                      (g_dtype FRL_F32, where p is that same memory, locally addressed)
 *   signal_pads_dev    device array [world] of pointers to each rank's uint32 signal pad;
 *                      slots [pad_base, pad_base + 64) are used
 *   local_scratch      rank-local uint32[8 + max_blocks], zero-initialised once
 *   max_blocks         grid size (1..1024; with in-kernel barriers all blocks must be co-resident)
 *   flags              0: the kernel carries both barriers itself.
 *                      FRL_NVLS_EXTERNAL_SYNC: no barrier inside; the caller issues, on the same
 *                      stream, frl_nvls_barrier(slot 0) before and frl_nvls_barrier(slot 1) after.
 *                      A rank that waits for slower peers then holds one warp instead of a grid
 *                      of spinning CTAs (which would keep its own backward GEMMs off the SMs).
 * n must be a multiple of 8; launch order must be identical on all ranks.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_NVLS_EXTERNAL_SYNC = 1 };
/* 1-CTA cross-GPU rendezvous over the signal pads (slots [32*pad_slot, 32*pad_slot + world)). */
int frl_nvls_barrier(void* const* signal_pads_dev, int rank, int world, int pad_slot, void* stream);
int frl_nvls_sgd(float* p, float* buf, const void* mc_g, void* mc_out, int64_t n, int rank,
                 int world, void* const* signal_pads_dev, int pad_base, void* local_scratch,
                 int max_blocks, double lr, double mu, double dampening, double wd, double grad_scale,
                 const float* dyn, int first_step, int g_dtype, int flags, void* stream);
int frl_nvls_adam(float* p, float* m, float* v, float* vmax, const void* mc_g, void* mc_out,
                  int64_t n, int rank, int world, void* const* signal_pads_dev, int pad_base,
                  void* local_scratch, int max_blocks, double lr, double beta1, double beta2,
                  double eps, double wd,
                  int64_t step, double grad_scale, const float* dyn, int g_dtype, int flags, void* stream);
int frl_nvls_rmsprop(float* p, float* sq, float* buf, const void* mc_g, void* mc_out, int64_t n,
                     int rank, int world, void* const* signal_pads_dev, int pad_base,
                     void* local_scratch, int max_blocks, double lr, double alpha, double eps,
                     double wd, double mu,
                     double grad_scale, const float* dyn, int g_dtype, int flags, void* stream);

/* ------------------------------------------------------------------------------------------
 * K8 — gather the rows of a minibatch from a pinned, device-mapped host dataset into HBM:
 * dst[i, :] = src[idx[i], :].  Replaces the per-sample __getitem__/collate/H2D sequence of the
 * loop (reference solver_worker.py:462-469): the kernel's PCIe reads are the transfer.
 * src_mapped: host pointer valid on the device (cudaHostAlloc / torch pin_memory); idx_dev:
 * int64 [n_rows] (device or mapped).  Rows that are multiples of 16 bytes take the wide path,
 * narrower rows (labels) an element-wise one.  max_blocks <= 0 -> 64 CTAs.
 * ---------------------------------------------------------------------------------------- */
int frl_gather_rows(const void* src_mapped, int64_t src_rows, const int64_t* idx_dev, void* dst,
                    int64_t n_rows, int64_t row_bytes, int max_blocks, void* stream);
/* K8w — rows of a window of retained minibatches (device tensors that are NOT contiguous with
 * one another): window row w lives in batch b at row w - sum(batch_rows[:b]).  dst[i, :] = that
 * row for w = idx_dev[i]; rows whose index is outside the window are left untouched.  Replaces
 * the per-sample slicing of retained minibatches in the loop's SamplerState (reference
 * solver_worker.py:254-262, 321-351: random picks and the worst-k heap keep data[i] slices)
 * where the indices only exist on the device.  batch_ptrs / batch_rows are HOST arrays (copied
 * into the kernel's parameter block, 64 batches per launch); idx_dev int64 [n_rows] on the device. */
int frl_gather_window_rows(const void* const* batch_ptrs, const int64_t* batch_rows, int n_batches,
                           const int64_t* idx_dev, void* dst, int64_t n_rows, int64_t row_bytes,
                           void* stream);
/* Same contract, moved by the SMs' bulk-copy engine (cp.async.bulk: host -> shared memory -> HBM,
 * one elected thread per CTA, 8 x 16 KB stages in flight).  Rows and pointers must be multiples
 * of 16 bytes.  max_blocks <= 0 -> one CTA per SM. */
int frl_gather_rows_tma(const void* src_mapped, int64_t src_rows, const int64_t* idx_dev, void* dst,
                        int64_t n_rows, int64_t row_bytes, int max_blocks, void* stream);
/* K8t — padded lines of a newline-separated text corpus in pinned, device-mapped host memory.
 * Replaces the per-sample TextDataset.get_raw_item + transform + default_collate of the loop
 * (reference text_dataset.py, solver_worker.py:462-469).  For row r, with i = idx_dev[r]
 * (an index outside [0, n_lines) reads line 0):
 *   lo = starts_dev[i], len = clamp(starts_dev[i+1] - 1 - lo, 0, row_len), at most corpus_bytes - lo;
 *   dst[r, j] = corpus[lo + j] for j < len, else pad.
 * corpus_mapped: 16-byte aligned, corpus_alloc_bytes >= corpus_bytes rounded up to 16 (the
 * kernel reads only aligned 16-byte units, each once).  starts_dev: int64 [n_lines + 1] on the
 * device; dst: uint8 [n_rows, row_len], contiguous, any alignment.  max_blocks <= 0 -> 8 CTAs. */
int frl_gather_lines(const void* corpus_mapped, int64_t corpus_bytes, int64_t corpus_alloc_bytes,
                     const int64_t* starts_dev, int64_t n_lines, const int64_t* idx_dev,
                     void* dst, int64_t n_rows, int64_t row_len, int pad, int max_blocks, void* stream);

/* ------------------------------------------------------------------------------------------
 * K9 — FP8 operands with current per-tensor scaling, for the Hopper FP8 tensor-core GEMMs of the
 * FP8 training precision (an extension: the reference trains in fp32 only).  Nothing is kept
 * between calls: the scale is derived on the device from the tensor being quantised.
 *
 * frl_fp8_amax: amax_out[0] = max |src[i]| over n elements of src_dtype (FRL_F32 | FRL_BF16);
 *   NaN anywhere gives NaN.  The function zeroes amax_out itself on `stream` before the
 *   reduction (capturable).  src 16-byte aligned, n >= 1.
 * frl_fp8_quantize: src is row-major [rows, cols] of src_dtype; amax a device scalar (as written
 *   by frl_fp8_amax).  With FP8_MAX = 448 (FRL_FP8_E4M3, e4m3fn) or 57344 (FRL_FP8_E5M2):
 *     scale = 2^k, k = floor(log2(FP8_MAX / amax)) clamped to [-126, 126]; scale = 1 if amax == 0;
 *     scale = NaN if amax is not finite (every code NaN, inv_scale_out NaN);
 *     q = saturate(round_to_nearest_even(src * scale)), bit for bit torch's
 *         (x.float() * scale).clamp(-FP8_MAX, FP8_MAX).to(float8);
 *     dst   [rows, cols] row-major codes, dst_t [cols, rows] (the transposed copy), either may
 *           be NULL but not both; inv_scale_out[0] = 1 / scale (the dequantisation scale).
 *   One read of src makes both copies.  Any rows, cols >= 1; src, dst, dst_t 16-byte aligned.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_FP8_E4M3 = 0, FRL_FP8_E5M2 = 1 };
int frl_fp8_amax(const void* src, int64_t n, int src_dtype, float* amax_out, void* stream);
int frl_fp8_quantize(const void* src, int64_t rows, int64_t cols, int src_dtype, const float* amax,
                     int fmt, void* dst, void* dst_t, float* inv_scale_out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Host gather pool — the host half of the input path (no CUDA calls inside).
 * Replaces the reference's per-sample __getitem__ + transform + default_collate on the host
 * (reference solver_worker.py:805-832, transform.py:25-38) with native worker threads that copy
 * the raw rows of a minibatch, dst[i, :] = src[idx[i], :], into a pinned staging buffer with
 * non-temporal stores; the caller then moves the staging buffer to HBM with one DMA and runs the
 * per-sample arithmetic on the device (K5).
 *   create(n_threads)            -> pool or NULL (frl_last_error)
 *   submit(...)                  -> ticket >= 1, or a negative FRL_E_* code; returns immediately;
 *                                   idx is copied, src/dst must stay valid until the job completes;
 *                                   an index outside [0, src_rows) rejects the whole job
 *   wait(pool, ticket)           -> blocks until every job up to and including `ticket` is done
 *                                   and its stores are globally visible (sfence)
 * Thread-safe; jobs run FIFO.
 * ---------------------------------------------------------------------------------------- */
typedef struct frl_gather_pool frl_gather_pool;
frl_gather_pool* frl_gather_pool_create(int n_threads);
void frl_gather_pool_destroy(frl_gather_pool* pool);
int frl_gather_pool_threads(const frl_gather_pool* pool);
int64_t frl_gather_pool_submit(frl_gather_pool* pool, const void* src_host, int64_t src_rows,
                               const int64_t* idx_host, void* dst_host, int64_t n_rows,
                               int64_t row_bytes);
/* Same gather with the PCIe hop in bf16: src rows are fp32 [row_elems], dst rows bf16 [row_elems],
 * converted round-to-nearest-even (NaN -> quiet NaN), bit-identical to the device cast, while the
 * worker threads touch the bytes anyway.  Halves the H2D payload of a bf16-compute run. */
int64_t frl_gather_pool_submit_f32_to_bf16(frl_gather_pool* pool, const void* src_host,
                                           int64_t src_rows, const int64_t* idx_host, void* dst_host,
                                           int64_t n_rows, int64_t row_elems);
int frl_gather_pool_wait(frl_gather_pool* pool, int64_t ticket);

#ifdef __cplusplus
}
#endif
#endif /* FRL_B200_H */
