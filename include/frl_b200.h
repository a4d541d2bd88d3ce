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
 *            SGD / RMSprop: dyn[0] = lr ;  Adam: dyn[0] = -lr/(1-beta1^t), dyn[1] = sqrt(1-beta2^t);
 *            AdamW: Adam's two, then dyn[2] = fp32(1 - lr*wd);  Lion: dyn[0] = lr, dyn[1] = fp32(1 - lr*wd).
 * Update rules are torch 2.11's (L2-coupled weight decay: g += wd * p first), except AdamW's
 * decoupled decay (frl_adamw*).
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

/* AdamW — torch 2.11's Adam(decoupled_weight_decay=True), which torch.optim.AdamW is.  Four entry
 * points, each with exactly the arguments of its Adam form: frl_adamw (K2, frl_adam's),
 * frl_adamw_mt (K2-mt, frl_adam_mt's), frl_adamw8_mt (K2-q8, frl_adam8_mt's) and frl_nvls_adamw
 * (K7, frl_nvls_adam's).  Per element, with g the scaled gradient:
 *     p  = p * fp32(1 - lr*wd)             its own fp32 multiply, before anything else
 *                                         (1 - lr*wd formed in double, rounded once to fp32)
 *     m  = lerp(m, g, 1-beta1) ; v = beta2*v + (1-beta2)*g^2 ; vmax = max(vmax, v) (amsgrad)
 *     p += -lr/(1-beta1^t) * m / (sqrt(v or vmax)/sqrt(1-beta2^t) + eps)
 * The gradient carries no decay term; with wd == 0 the result is frl_adam's, bit for bit.
 * dyn (may be NULL): dyn[0] = -lr/(1-beta1^t), dyn[1] = sqrt(1-beta2^t), dyn[2] = fp32(1 - lr*wd),
 * so a captured CUDA graph follows a scheduled lr in the decay as well.  Graph-capturable.  Every
 * argument check is made before any launch, as in the Adam forms; frl_abi_version() stays 1. */
int frl_adamw(float* p, const void* g, float* m, float* v, float* vmax, void* p_lp, int64_t n,
              double lr, double beta1, double beta2, double eps, double wd, int64_t step,
              double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
              void* stream);

/* Lion (Chen et al. 2023, Symbolic Discovery of Optimization Algorithms, Algorithm 2), with one
 * state m = exp_avg (non-NULL; it starts at zero and there is no first-step special case).  Seven
 * entry points, each with its SGD form's arguments with (beta1, beta2) in place of (mu, dampening)
 * and no first_step: frl_lion (K2), frl_lion_mt (K2-mt), frl_lion_sr / frl_lion_mt_sr (K2-sr),
 * frl_nvls_lion (K7), frl_dw_gemm_lion / frl_dw_gemm_lion_sr (K12).  Per element, in fp32, with g
 * the scaled gradient:
 *     p = p * fp32(1 - lr*wd)              its own fp32 multiply (1 - lr*wd formed in double,
 *                                          rounded once), as AdamW's
 *     c = fmaf(1-beta1, g - m, m)          lerp(m, g, 1-beta1)
 *     p = fmaf(-lr, sign(c), p)            sign: +1 / -1 / 0, and NaN for a NaN c
 *     m = fmaf(1-beta2, g - m, m)          lerp(m, g, 1-beta2)
 * 20 B per parameter with an fp32 gradient and no shadow, as SGD with momentum.  beta1 and beta2
 * must lie in [0, 1) (FRL_E_ARG).  dyn (may be NULL): dyn[0] = lr, dyn[1] = fp32(1 - lr*wd), and
 * for the _sr forms dyn[3] = t.  Every argument check is made before any launch; graph-capturable. */
int frl_lion(float* p, const void* g, float* m, void* p_lp, int64_t n, double lr, double beta1, double beta2,
             double wd, double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
             void* stream);

/* RMSprop (not centered): sq = alpha*sq + (1-alpha)*g^2 ; avg = sqrt(sq)+eps ;
 * mu > 0: buf = mu*buf + g/avg ; p -= lr*buf     else: p -= lr*g/avg  (buf may be NULL). */
int frl_rmsprop(float* p, const void* g, float* sq, float* buf, void* p_lp, int64_t n,
                double lr, double alpha, double eps, double wd, double mu,
                double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
             void* stream);

/* ------------------------------------------------------------------------------------------
 * K12 — weight-gradient GEMM gw = dz^T x on the tensor cores (persistent, TMA + WGMMA), with
 * an optional SGD or Lion update of the same weights in its epilogue.
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
/* frl_dw_gemm_sgd_sr: frl_dw_gemm_sgd for bf16 master weights (K2-sr below): p is the slice's bf16
 * weights (no shadow), arena_off the arena index of p's element 0 (a multiple of 4), seed and t as in
 * frl_sgd_momentum_sr, dyn[3] = t's bits under replay.  Bit-identical to frl_dw_gemm followed by
 * frl_sgd_momentum_sr(g_dtype = FRL_BF16) over the slice. */
int frl_dw_gemm_sgd_sr(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                       int64_t out, int64_t in, void* gw, void* p, float* buf, int64_t arena_off, uint64_t seed,
                       int64_t t, double lr, double mu, double dampening, double wd, double grad_scale,
                       const float* dyn, int first_step, void* stream);

/* frl_dw_gemm_lion / frl_dw_gemm_lion_sr: frl_dw_gemm_sgd / frl_dw_gemm_sgd_sr with frl_lion's rule
 * (m = exp_avg of the slice, non-NULL): bit-identical to frl_dw_gemm followed by frl_lion /
 * frl_lion_sr (g_dtype = FRL_BF16) over the slice. */
int frl_dw_gemm_lion(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                     int64_t out, int64_t in, void* gw, float* p, float* m, void* p_lp, double lr, double beta1,
                     double beta2, double wd, double grad_scale, const float* dyn, void* stream);
int frl_dw_gemm_lion_sr(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                        int64_t out, int64_t in, void* gw, void* p, float* m, int64_t arena_off, uint64_t seed,
                        int64_t t, double lr, double beta1, double beta2, double wd, double grad_scale,
                        const float* dyn, void* stream);

/* ------------------------------------------------------------------------------------------
 * K13 — data-gradient GEMM of an upper Linear layer with the lower Linear+ReLU unit's backward in
 * its epilogue (persistent, TMA + WGMMA):
 *   dz[r, c]  = act[r, c] <= 0 ? 0 : bf16((dz_up w)[r, c])    (fp32 accumulation, rounded once;
 *               a NaN activation passes the gradient through, as threshold_backward does)
 *   db[c]   (+)= sum_r dz[r, c]                                 (fp32 sums, stored as bf16)
 *   dz_up [rows, k] (ld_dz_up), w [k, cols] (ld_w), act / dz [rows, cols] (ld_act / ld_dz): row-major
 *   bf16; db [cols] bf16.  rows % 128 == 0, cols % 256 == 0, k % 8 == 0, every pointer except db
 *   16-byte aligned and every leading dimension a multiple of 8, else FRL_E_ARG.  scratch: at least
 *   frl_dx_drelu_scratch_bytes(rows, cols) bytes, zeroed before the first launch and left zeroed by
 *   every launch; launches sharing it must be stream-ordered.  Deterministic: no float atomics.
 * ---------------------------------------------------------------------------------------- */
int64_t frl_dx_drelu_scratch_bytes(int64_t rows, int64_t cols);
int frl_dx_gemm_drelu(const void* dz_up, int64_t ld_dz_up, const void* w, int64_t ld_w, const void* act,
                      int64_t ld_act, void* dz, int64_t ld_dz, void* db, int64_t rows, int64_t k,
                      int64_t cols, int accumulate, void* scratch, void* stream);

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

/* K2-mt AdamW: frl_adam_mt's arguments, frl_adamw's rule and dyn layout. */
int frl_adamw_mt(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                 const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double beta1,
                 double beta2, double eps, double wd, int64_t step, double grad_scale,
                 const float* grad_scale_dev, const float* dyn, void* stream);

/* K2-mt Lion: frl_sgd_momentum_mt's arguments, frl_lion's rule and dyn layout. */
int frl_lion_mt(float* p, float* m, void* p_lp, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double beta1, double beta2, double wd,
                double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream);

int frl_rmsprop_mt(float* p, float* sq, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                   const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double alpha,
                   double eps, double wd, double mu, double grad_scale, const float* grad_scale_dev,
                   const float* dyn, void* stream);

/* ------------------------------------------------------------------------------------------
 * K2-sr / K2-mt-sr — the K2 / K2-mt update on bf16 master weights with stochastic rounding
 * (an extension, types.MasterWeights.BF16: no fp32 copy of the model's weights exists).
 * Arguments: those of the fp32 form, except that p is the bf16 weight vector (there is no
 * separate p_lp), plus arena_off (flat forms: the arena index of p's element 0, a multiple of 4),
 * seed and t.  The _mt_sr forms take p as the ARENA BASE of the bf16 weights and list model slots.
 * Per element: widen the bf16 weight to fp32, apply the fp32 form's rule unchanged, store
 *     bf16 bits = (bits(x) + r) >> 16          (x NaN: 0x7FC0)
 * where r, the 16 random bits of arena element i at update t (the optimizer's 1-based update
 * count; the Adam forms use their step), are the low 16 bits of word (i & 3) of
 *     Philox4x32-10(counter = (lo32(i >> 2), hi32(i >> 2), t, 0x53520000),
 *                   key     = (lo32(seed), hi32(seed))).
 * That rounds the magnitude up with probability (discarded fraction) / 2^16, so the expected
 * stored value is x: +-inf and bf16-exact values never change, a finite value reaches inf only
 * by carrying out of 0x7F7F.  dyn: the fp32 form's layout, and dyn[3] holds t as a uint32 bit
 * pattern (it then replaces the t argument).  Graph-capturable.
 * frl_weight_ema_bf16: frl_weight_ema with p a bf16 vector (10 B per element instead of 12).
 * ---------------------------------------------------------------------------------------- */
int frl_sgd_momentum_sr(void* p, const void* g, float* buf, int64_t n, int64_t arena_off, uint64_t seed,
                        int64_t t, double lr, double mu, double dampening, double wd, double grad_scale,
                        const float* grad_scale_dev, const float* dyn, int first_step, int g_dtype, void* stream);
int frl_adam_sr(void* p, const void* g, float* m, float* v, float* vmax, int64_t n, int64_t arena_off,
                uint64_t seed, double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype, void* stream);
int frl_adamw_sr(void* p, const void* g, float* m, float* v, float* vmax, int64_t n, int64_t arena_off,
                 uint64_t seed, double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                 double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype, void* stream);
int frl_lion_sr(void* p, const void* g, float* m, int64_t n, int64_t arena_off, uint64_t seed, int64_t t,
                double lr, double beta1, double beta2, double wd, double grad_scale, const float* grad_scale_dev,
                const float* dyn, int g_dtype, void* stream);
int frl_rmsprop_sr(void* p, const void* g, float* sq, float* buf, int64_t n, int64_t arena_off, uint64_t seed,
                   int64_t t, double lr, double alpha, double eps, double wd, double mu, double grad_scale,
                   const float* grad_scale_dev, const float* dyn, int g_dtype, void* stream);
int frl_sgd_momentum_mt_sr(void* p, float* buf, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                           const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed, int64_t t, double lr,
                           double mu, double dampening, double wd, double grad_scale, const float* grad_scale_dev,
                           const float* dyn, int first_step, void* stream);
int frl_adam_mt_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                   const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed,
                   double lr, double beta1, double beta2, double eps, double wd, int64_t step, double grad_scale,
                   const float* grad_scale_dev, const float* dyn, void* stream);
int frl_adamw_mt_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                    const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed,
                    double lr, double beta1, double beta2, double eps, double wd, int64_t step, double grad_scale,
                    const float* grad_scale_dev, const float* dyn, void* stream);
int frl_lion_mt_sr(void* p, float* m, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                   const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed, int64_t t, double lr, double beta1,
                   double beta2, double wd, double grad_scale, const float* grad_scale_dev, const float* dyn,
                   void* stream);
int frl_rmsprop_mt_sr(void* p, float* sq, float* buf, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                      const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed, int64_t t, double lr,
                      double alpha, double eps, double wd, double mu, double grad_scale,
                      const float* grad_scale_dev, const float* dyn, void* stream);
int frl_weight_ema_bf16(float* ema, const void* p, int64_t n, double w, void* stream);

/* ------------------------------------------------------------------------------------------
 * K2-mt grouped / K2-mt-sr grouped — parameter groups (torch.optim's param_groups): a learning
 * rate and a weight decay per group, in the segment-table update of SGD (with or without
 * momentum), Adam, AdamW, RMSprop and Lion.  Arguments: those of the frl_*_mt / frl_*_mt_sr form
 * without lr, wd, dyn and t / step, and after n_tiles
 *   seg_group_dev  int32 [n_segs]: the group of each segment, in [0, n_groups) (the caller
 *                  validates it when it builds the table: the kernel does not read it back first)
 *   seg_flags_dev  int32 [n_segs]: FRL_LW_CLIPPED = grad_scale_dev multiplies this segment's
 *                  gradient (model parameters under clipping), as in K2-lw; other bits ignored
 *   group_dyn      fp32 [n_groups][FRL_GROUP_DYN_COLS], 16-byte aligned, read at every launch
 *                  (eager or replayed from a CUDA graph), one row per group g with lr_g, wd_g:
 *     col 0-3  the ungrouped form's dyn layout for lr_g / wd_g, so a row pointer is a valid dyn
 *              for K12 and the SR forms:
 *                SGD, RMSprop   (lr_g, -, -, t)
 *                Adam           (-lr_g / (1 - beta1^t), sqrt(1 - beta2^t), -, t)
 *                AdamW          (-lr_g / (1 - beta1^t), sqrt(1 - beta2^t), fp32(1 - lr_g*wd_g), t)
 *                Lion           (lr_g, fp32(1 - lr_g*wd_g), -, t)
 *              t: the 1-based update count as uint32 bits (read by the _sr forms only)
 *     col 4    wd_g, the L2-coupled decay of SGD, Adam and RMSprop
 *   n_groups       rows of group_dyn, >= 1
 * Per element of a segment of group g, the ungrouped rule with lr = lr_g and wd = wd_g:
 *   SGD      d = g^ + wd_g*w ; buf = first_step ? d : mu*buf + (1-dampening)*d ; w -= lr_g*buf
 *   Adam     the frl_adam rule on g^ + wd_g*w, step size lr_g / bc1
 *   AdamW    w *= fp32(1 - lr_g*wd_g), then frl_adam's rule with no decay term
 *   RMSprop  the frl_rmsprop rule on g^ + wd_g*w, lr_g
 *   Lion     w *= fp32(1 - lr_g*wd_g) ; w -= lr_g*sign(lerp(m, g^, 1-beta1)) ; m = lerp(m, g^, 1-beta2)
 * with g^ = g * grad_scale (* *grad_scale_dev if the segment has FRL_LW_CLIPPED).  Bytes per
 * parameter are the ungrouped form's: a tile reads its segment's row once.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_GROUP_DYN_COLS = 8 };
int frl_sgd_momentum_mt_grouped(float* p, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                                const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                                int n_groups, double mu, double dampening, double grad_scale,
                                const float* grad_scale_dev, int first_step, void* stream);
int frl_adam_mt_grouped(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                        const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                        const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                        int n_groups, double beta1, double beta2, double eps, double grad_scale,
                        const float* grad_scale_dev, void* stream);
int frl_adamw_mt_grouped(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                         const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                         const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                         int n_groups, double beta1, double beta2, double eps, double grad_scale,
                         const float* grad_scale_dev, void* stream);
int frl_lion_mt_grouped(float* p, float* m, void* p_lp, const frl_grad_seg* segs_dev,
                        const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                        const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                        int n_groups, double beta1, double beta2, double grad_scale, const float* grad_scale_dev,
                        void* stream);
int frl_rmsprop_mt_grouped(float* p, float* sq, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                           const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                           int n_groups, double alpha, double eps, double mu, double grad_scale,
                           const float* grad_scale_dev, void* stream);
int frl_sgd_momentum_mt_grouped_sr(void* p, float* buf, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                   const int32_t* tile_seg_dev, int64_t n_tiles, const int32_t* seg_group_dev,
                                   const int32_t* seg_flags_dev, const float* group_dyn, int n_groups, uint64_t seed,
                                   double mu, double dampening, double grad_scale, const float* grad_scale_dev,
                                   int first_step, void* stream);
int frl_adam_mt_grouped_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                           const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                           int n_groups, uint64_t seed, double beta1, double beta2, double eps, double grad_scale,
                           const float* grad_scale_dev, void* stream);
int frl_adamw_mt_grouped_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                            const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                            const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                            int n_groups, uint64_t seed, double beta1, double beta2, double eps, double grad_scale,
                            const float* grad_scale_dev, void* stream);
int frl_lion_mt_grouped_sr(void* p, float* m, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                           const int32_t* tile_seg_dev, int64_t n_tiles, const int32_t* seg_group_dev,
                           const int32_t* seg_flags_dev, const float* group_dyn, int n_groups, uint64_t seed,
                           double beta1, double beta2, double grad_scale, const float* grad_scale_dev, void* stream);
int frl_rmsprop_mt_grouped_sr(void* p, float* sq, float* buf, const frl_grad_seg* segs_dev,
                              const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                              const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                              int n_groups, uint64_t seed, double alpha, double eps, double mu, double grad_scale,
                              const float* grad_scale_dev, void* stream);

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
 * passes the NaN on).  Norms: squares and per-tile sums in double (no overflow or underflow for
 * any finite fp32 gradient), folded per tensor in tile order (no float atomics, deterministic).
 * Two launches: stats (LAMB writes m, v here) and apply.
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
 * K2-q8 — Adam with 8-bit block-wise optimizer state (an extension: Dettmers et al., "8-bit
 * Optimizers via Block-wise Quantization", ICLR 2022).  exp_avg and exp_avg_sq are stored as one
 * byte per arena element plus one fp32 absmax per block:
 *   blocks    each segment (parameter tensor) is cut into blocks of FRL_Q8_BLOCK = 256
 *             consecutive elements starting at its first element; the last may be short; no block
 *             spans two segments.  Block b of segment s has the global index qbase_dev[s] + b
 *             (qbase: a prefix sum of ceil(numel / 256) over every arena slot in arena order).
 *   absmax    per state and block: max |x| over the block, NaN if the block holds a NaN.
 *   exp_avg   code c = sign bit of the fp32 value << 7 | k, decodes to +-MAG7[k] * absmax.
 *   exp_avg_sq code k, decodes to MAG8[k] * absmax.
 *   tables    each entry computed in double and rounded once to fp32, increasing:
 *             MAG7 = 0, then for i = 0..6, j = 0..2^i - 1: 10^(i-6) * (0.1 + 0.9*(j + 0.5)/2^i)
 *                    (127 values), the largest of them (0.99296875) replaced by 1.0: 128 entries;
 *             MAG8 = 0, then for i = 0..6, j = 0..2^(i+1) - 1: 10^(i-6) * (0.1 + 0.9*(j + 0.5)/2^(i+1))
 *                    (254 values), then 1.0: 256 entries.
 *   encoding  r = |x| / absmax (IEEE fp32 division; r = 0 if absmax == 0), the code is the index
 *             of the table entry nearest to r, ties to the smaller index (a NaN r gives index 0).
 *             Both tables hold 0 and 1, so decoding a block and encoding it again returns the same
 *             bytes and absmax.
 *   Code arrays are arena-shaped (one byte per arena element, 16-byte aligned); elements outside
 *   every segment (padding) are never written.
 * frl_adam8_mt: arguments of frl_adam_mt (no amsgrad) plus the code and absmax arrays, n_segs,
 *   qbase_dev (int64 [n_segs]) and seg_flags_dev (int32 [n_segs]; FRL_LW_CLIPPED: grad_scale_dev
 *   multiplies this segment's gradient, as in K2-lw).  Per element of a listed segment:
 *   decode m and v; apply frl_adam_mt's fp32 rule exactly (L2-coupled wd, lerp for m, dyn);
 *   write the master and, with p_lp, the bf16 shadow from this step's fp32 m and v; reduce the
 *   block's new absmax of m and of v; encode.  A non-finite gradient therefore gives the weights
 *   frl_adam_mt gives from the same decoded state.  dyn as for frl_adam_mt.  Graph-capturable.
 * frl_q8_encode_mt / frl_q8_decode_mt: fp32 arena-shaped state x <-> codes and absmax of the
 *   listed segments, for `state` FRL_Q8_EXP_AVG or FRL_Q8_EXP_AVG_SQ (the segment table's
 *   gradient pointers are not read).  Decoding writes 0 to the padding of a segment's last
 *   vector of 4.  Same encoder and decoder as frl_adam8_mt.
 * frl_q8_tables: host copy of MAG7 (128 floats) and MAG8 (256 floats); either may be NULL.
 * Every argument check is made before any launch; n_tiles == 0 launches nothing.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_Q8_BLOCK = 256, FRL_Q8_EXP_AVG = 0, FRL_Q8_EXP_AVG_SQ = 1 };
void frl_q8_tables(float* mag7, float* mag8);
int frl_adam8_mt(float* p, uint8_t* m_q, uint8_t* v_q, float* m_absmax, float* v_absmax, void* p_lp,
                 const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev,
                 int64_t n_tiles, int64_t n_segs, const int64_t* qbase_dev, const int32_t* seg_flags_dev,
                 double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                 double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream);
/* K2-q8 AdamW: frl_adam8_mt's arguments, encoder and decoder; frl_adamw's rule (no amsgrad) and
 * dyn layout, applied to the decoded moments. */
int frl_adamw8_mt(float* p, uint8_t* m_q, uint8_t* v_q, float* m_absmax, float* v_absmax, void* p_lp,
                  const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev,
                  int64_t n_tiles, int64_t n_segs, const int64_t* qbase_dev, const int32_t* seg_flags_dev,
                  double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                  double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream);
int frl_q8_encode_mt(const float* x, uint8_t* q, float* absmax, int state, const frl_grad_seg* segs_dev,
                     const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                     int64_t n_segs, const int64_t* qbase_dev, void* stream);
int frl_q8_decode_mt(const uint8_t* q, const float* absmax, float* x, int state, const frl_grad_seg* segs_dev,
                     const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                     int64_t n_segs, const int64_t* qbase_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * K2-af — Adafactor (an extension: Shazeer & Stern, ICML 2018), the rule of
 * torch.optim.Adafactor with foreach=False and maximize=False.  No first moment; the second
 * moment of a tensor of 2 or more dimensions, viewed as [B, R, C] (B = product of the leading
 * dimensions), is factored into row_var [B, R] and col_var [B, C]; a 0-/1-D tensor keeps a full
 * variance.  Per segment s, fp32, with g^ = g * grad_scale (* *grad_scale_dev if FRL_LW_CLIPPED),
 * t = step (>= 1) and eps1 passed explicitly (torch's None is the fp32 epsilon 2^-23):
 *   w_t = t^beta2_decay ; rho = min(lr, 1/sqrt(t))                        (host, double)
 *   alpha = max(eps2, ||p|| / sqrt(numel)) * rho       (p before the decay; a NaN norm gives eps2)
 *   factored:   row_var[b,r] = lerp(row_var[b,r], sum_c g^^2 / C, w_t)
 *               col_var[b,c] = lerp(col_var[b,c], sum_r g^^2 / R, w_t)
 *               vhat = row_var[b,r] * col_var[b,c] / max(mean_r row_var[b,r], eps1)
 *   unfactored: variance = lerp(variance, g^^2, w_t) ; vhat = variance
 *   u = rsqrt(max(vhat, eps1^2)) * g^ ; denom = max(1, ||u|| / (sqrt(numel) * d))  (NaN gives 1)
 *   p = p * (1 - lr*wd) + (-alpha / denom) * u        (both factors formed in double, rounded once)
 * lerp is torch's fp32 formula (K11's).  Sums of squares and the norms are double, folded per
 * tensor in a fixed order: no float atomics, two launches give the same bytes.
 *   shape_dev      int64 [n_segs][3] = (B, R, C); R = 0 for an unfactored tensor (C = numel)
 *   state_off_dev  int64 [n_segs]: offset in `state` (one compact fp32 buffer) of the segment's
 *                  row_var then col_var, or of its variance
 *   seg_flags_dev  int32 [n_segs]: FRL_LW_CLIPPED as in K2-lw
 *   work_dev, n_work, seg_info_dev   the band table frl_adafactor_plan builds from the shapes
 *   scratch        frl_adafactor_scratch_bytes(shape, n_segs) bytes, zero-initialised once
 *   dyn            dyn[0] = lr, dyn[1] = w_t, dyn[2] = rho (replaces the by-value scalars)
 * frl_adafactor_plan: host; shape as shape_dev.  Writes work (int64 [n_work][4]) and seg_info
 *   (int64 [n_segs][3]) when they are not NULL and returns n_work, or -1 on a bad shape.
 * Three launches (stats, norm, apply); every argument check is made before any launch;
 * n_work == 0 launches nothing.  Graph-capturable.
 * ---------------------------------------------------------------------------------------- */
int64_t frl_adafactor_plan(const int64_t* shape, int64_t n_segs, int64_t* work, int64_t* seg_info);
int64_t frl_adafactor_scratch_bytes(const int64_t* shape, int64_t n_segs);
int frl_adafactor_mt(float* p, float* state, void* p_lp, const frl_grad_seg* segs_dev, int64_t n_segs,
                     const int64_t* shape_dev, const int64_t* state_off_dev, const int32_t* seg_flags_dev,
                     const int64_t* work_dev, int64_t n_work, const int64_t* seg_info_dev, void* scratch,
                     double lr, double beta2_decay, double eps1, double eps2, double d, double wd, int64_t step,
                     double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream);

/* ------------------------------------------------------------------------------------------
 * K14 — Muon (an extension: Jordan et al. 2024; torch.optim.Muon's rule) for the 2-D weights of
 * a segment table.  Per matrix p [R, C] (fp32 master), m = min(R, C), n = max(R, C), with
 * g^ = g * grad_scale (* *grad_scale_dev: every Muon matrix is a model parameter):
 *   buf = lerp(buf, g^, 1 - momentum)          buf: the matrix's range of exp_avg (fp32)
 *   u   = nesterov ? lerp(g^, buf, momentum) : buf
 *   X   = bf16(u) as [m, n] (transposed when R > C); X = bf16(X / max(bf16(||X||_F), bf16(eps)))
 *   ns_steps times:  A = bf16(X X^T);  B = bf16(b A + c A A);  X = bf16(a X + B X)
 *     (fp32 accumulation, one bf16 rounding per output element)
 *   p = p * (1 - lr*wd) - adj * float(O),  O = X transposed back when R > C;  p_lp = bf16(p)
 *   adj = lr * (adjust_lr ? 0.2 * sqrt(max(R, C)) : sqrt(max(1, R / C)))
 *     (adjust_lr 1 = "match_rms_adamw", 0 = "original" / None)
 * The NS iterates ping-pong in the matrix's range of the fp32 exp_avg_sq vector (two bf16
 * [m, n] matrices in its 4 bytes per element) when n is a multiple of 8, else in the workspace.
 * The workspace also holds A and B ([m, m] bf16, leading dimension rounded up to 8) per matrix,
 * laid out from its start in plan order: plans over subsets of the same matrices may share one
 * workspace sized for all of them, as long as their launches do not overlap.
 * frl_muon_plan_bytes: host; shape int64 [n_mat][4] = (segment index in the table, arena offset
 *   (a multiple of 8), R, C).  Returns the plan's size in bytes (-1 on a bad shape) and writes
 *   the scratch's size (tickets, norms, partials: one per plan) and the workspace's size where
 *   non-NULL.
 * frl_muon_plan: host; fills the plan (tensor maps, grouped tile tables) for the given
 *   exp_avg_sq base and workspace (128-byte aligned).  The caller copies it to the device
 *   (64-byte aligned) and keeps both copies while the buffers live.
 * frl_muon_mt: scratch as sized above, 16-byte aligned, zeroed once.  Every planned segment index
 *   must be < n_segs (FRL_E_ARG otherwise); that segment's numel must be R * C (the table lives on
 *   the device, so the caller checks this).
 * frl_muon_mt: prologue (momentum, iterate, per-matrix norm folded in tile order by the last
 *   CTA of each matrix), normalisation, then 3 * ns_steps persistent TMA + WGMMA launches
 *   (gram, poly, update) over every matrix at once; Gram and poly compute only tiles on or above
 *   the diagonal.  The last update writes p and p_lp directly.  No float atomics or split-K:
 *   repeated launches give the same bytes.  dyn: optional device fp32, dyn[2] = lr (replaces the
 *   by-value lr).  1 <= ns_steps < 100.  All checks run before the first launch; graph-capturable.
 * ---------------------------------------------------------------------------------------- */
int64_t frl_muon_plan_bytes(const int64_t* shape, int64_t n_mat, int64_t* scratch_bytes, int64_t* workspace_bytes);
int frl_muon_plan(const int64_t* shape, int64_t n_mat, const float* exp_avg_sq, void* workspace, void* plan);
int frl_muon_mt(float* p, float* exp_avg, void* p_lp, const frl_grad_seg* segs_dev, int64_t n_segs,
                const void* plan_host, const void* plan_dev, void* scratch, double lr, double wd,
                double momentum, int nesterov, double a, double b, double c, int ns_steps, double eps,
                int adjust_lr, double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream);

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

/* K5 into channels_last: src [batch, channels, hw] contiguous (an image batch [B, C, H, W],
 * hw = H * W, 1 <= channels <= 4; u8 / f32 / bf16) -> dst [batch, hw, channels] in memory (the
 * NHWC storage of a channels_last [B, C, H, W] tensor; f32 / bf16).  Values are frl_preproc_affine's
 * with inner = hw bit for bit: dst = fmaf(src, scale[c], bias[c]) (a NULL scale is 1, a NULL bias
 * 0), or src * 1 when both are NULL.  src and dst 16-byte aligned. */
int frl_preproc_affine_nhwc(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t batch,
                            int channels, int64_t hw, const float* scale, const float* bias, void* stream);

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
/* frl_augment_images with dst in [B, out_h, out_w, C] memory order (the NHWC storage of a
 * channels_last [B, C, out_h, out_w] tensor): the same values, permuted. */
int frl_augment_images_nhwc(const void* src, int64_t batch, int channels, int height, int width,
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
/* frl_augment_mix_images with dst in [B, out_h, out_w, C] memory order: the same values, permuted. */
int frl_augment_mix_images_nhwc(const void* src, int64_t batch, int channels, int height, int width,
                                const int64_t* idx, uint64_t seed, int epoch, int mode,
                                double smin, double smax, double rmin, double rmax, double eval_crop, int pad,
                                int flip, const float* scale, const float* bias, void* dst, int dst_dtype,
                                int out_h, int out_w, int32_t* params_out, int mix_mode, float lam,
                                int box_y0, int box_y1, int box_x0, int box_x1, void* stream);
int frl_mix_targets(const void* src, int src_dtype, int64_t batch, int64_t inner, int n_classes, float lam,
                    void* dst, void* stream);

/* ------------------------------------------------------------------------------------------
 * K5p — K5a's training crop and flip, then an automatic augmentation policy (TrivialAugmentWide,
 * Müller & Hutter 2021, or RandAugment, Cubuk et al. 2020), then the affine, then random erasing
 * (Zhong et al. 2020), as torchvision v2 does them on a uint8 image.  One CTA per sample stages its
 * crop in shared memory.
 *   src, idx, seed, epoch, smin..rmax, pad, flip, scale, bias, dst, out_h, out_w, params_out:
 *              as frl_augment_images; mode FRL_AUG_RRC or FRL_AUG_PAD_CROP only
 *   policy     FRL_POLICY_NONE (erasing alone), FRL_POLICY_TRIVIAL_AUGMENT (num_ops must be 1) or
 *              FRL_POLICY_RAND_AUGMENT (num_ops in [1, 4], magnitude in [0, num_bins)); a policy
 *              needs channels 1 or 3, K5p serves at most 3
 *   mags       device fp32 [14, num_bins], num_bins >= 2: the magnitude of op o at bin k (the
 *              unsigned table torchvision builds for the output size; Posterize's bits as floats;
 *              0 for the three ops without a magnitude)
 *   erase_p    probability of erasing, in [0, 1]; 0 turns erasing off.  erase_smin/smax: area share
 *              in [0, 1]; erase_rmin/rmax > 0: aspect range.  erase_random != 0: N(0, 1) values;
 *              else erase_value (device fp32 [C], NULL = 0), in the normalised domain
 *   policy_out optional int32 [B, 3*num_ops + 5] (num_ops 0 without a policy): (op, bin, sign) per
 *              op, then (erased, top, left, h, w)
 * channels * out_h * out_w must be at most FRL_AUGMENT_POLICY_SMEM_BYTES (FRL_E_ARG).
 *
 * Draws (Philox4x32-10 with K5a's key and counter (lo32(i), hi32(i), epoch, block); u(w) and
 * int(w, n) as K5a's; K5a's blocks 0..10 keep their meaning, so the box and flip do not depend on
 * the policy or erasing):
 *   op k (k < num_ops): block 11 + k: op = int(w0, 14) in torchvision's _AUGMENTATION_SPACE order
 *     (Identity, ShearX, ShearY, TranslateX, TranslateY, Rotate, Brightness, Color, Contrast,
 *     Sharpness, Posterize, Solarize, AutoContrast, Equalize); bin = int(w1, num_bins) for
 *     TrivialAugmentWide, `magnitude` for RandAugment; sign = -1 if w2 >> 31 for the nine signed
 *     ops (ShearX .. Sharpness), else +1.  Ops without a magnitude record bin 0.
 *     magnitude = sign * mags[op, bin].
 *   erasing: block 15: erase if u(w0) < erase_p.  Attempt t = 0..9 uses block 16 + t, in double:
 *     area = out_h*out_w * (smin + u(w0)*(smax - smin)); aspect = exp(log rmin + u(w1)*(log rmax -
 *     log rmin)); h = rint(sqrt(area*aspect)), w = rint(sqrt(area/aspect)) (h takes the product,
 *     the reverse of RRC); accepted if h < out_h and w < out_w: top = int(w2, out_h-h+1),
 *     left = int(w3, out_w-w+1).  No attempt accepted: nothing is erased.
 *   random values: element e = (c*h + y)*w + x of the box uses block 32 + e/4, pair j = (e/2) % 2:
 *     u1 = ((w_{2j} >> 8) + 1) * 2^-24, u2 = (w_{2j+1} >> 8) * 2^-24, r = sqrt(-2 ln u1),
 *     value = r cos(2 pi u2) for even e, r sin(2 pi u2) for odd e (fp32; not torch's stream).
 * Pixels:
 *   1. the crop: K5a's bilinear value v before the affine, rounded half to even to uint8
 *      (F.resized_crop(x.float(), antialias=False).round_()); flipped samples mirrored.
 *   2. each op on the uint8 image, uint8 after every op, as TrivialAugmentWide.
 *      _apply_image_or_video_transform does it: geometric ops with NEAREST and fill 0, their
 *      inverse matrix from torchvision's formula in double, the grid in fp32; colour ops in fp32
 *      with torch's roundings, then clamped to [0, 255] and truncated.
 *   3. dst = fmaf(v, scale[c], bias[c]) as K5a; inside the erased box the erasing value instead.
 * dst is also the CTA's scratch: it stages index-map op results in its own sample's region.
 * Graph-capturable: no host reads, no allocation.  Every argument check comes before any launch.
 * ---------------------------------------------------------------------------------------- */
enum { FRL_POLICY_NONE = 0, FRL_POLICY_TRIVIAL_AUGMENT = 1, FRL_POLICY_RAND_AUGMENT = 2 };
enum { FRL_AUGMENT_POLICY_SMEM_BYTES = 224256 };
int frl_augment_policy_images(const void* src, int64_t batch, int channels, int height, int width,
                              const int64_t* idx, uint64_t seed, int epoch, int mode,
                              double smin, double smax, double rmin, double rmax, int pad, int flip,
                              int policy, int num_ops, int magnitude, int num_bins, const float* mags,
                              double erase_p, double erase_smin, double erase_smax, double erase_rmin,
                              double erase_rmax, int erase_random, const float* erase_value,
                              const float* scale, const float* bias, void* dst, int dst_dtype,
                              int out_h, int out_w, int32_t* params_out, int32_t* policy_out, void* stream);
/* frl_augment_policy_images with dst in [B, out_h, out_w, C] memory order: the same values. */
int frl_augment_policy_images_nhwc(const void* src, int64_t batch, int channels, int height, int width,
                                   const int64_t* idx, uint64_t seed, int epoch, int mode,
                                   double smin, double smax, double rmin, double rmax, int pad, int flip,
                                   int policy, int num_ops, int magnitude, int num_bins, const float* mags,
                                   double erase_p, double erase_smin, double erase_smax, double erase_rmin,
                                   double erase_rmax, int erase_random, const float* erase_value,
                                   const float* scale, const float* bias, void* dst, int dst_dtype,
                                   int out_h, int out_w, int32_t* params_out, int32_t* policy_out,
                                   void* stream);

/* Mixup / CutMix of finished images in place: dst [B, C, out_h, out_w] (fp32 / bf16; the _nhwc
 * form: [B, out_h, out_w, C] in memory), sample p with sample j = B-1-p, p < B/2:
 *   Mixup:  out_p = round(__fadd_rn(__fmul_rn(lam, a_p), __fmul_rn(lam1, a_j))), lam1 as
 *           frl_augment_mix_images.  a_p is the stored value, so bf16 images round twice.
 *   CutMix: a_p and a_j swap inside [box_y0, box_y1) x [box_x0, box_x1) (exact).
 * The middle sample of an odd batch is left as it is.  Every argument check comes before any launch. */
int frl_mix_images(void* dst, int dst_dtype, int64_t batch, int channels, int out_h, int out_w, int mix_mode,
                   float lam, int box_y0, int box_y1, int box_x0, int box_x1, void* stream);
int frl_mix_images_nhwc(void* dst, int dst_dtype, int64_t batch, int channels, int out_h, int out_w,
                        int mix_mode, float lam, int box_y0, int box_y1, int box_x0, int box_x1, void* stream);

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
/* K7 AdamW: frl_nvls_adam's arguments, frl_adamw's rule and dyn layout. */
int frl_nvls_adamw(float* p, float* m, float* v, float* vmax, const void* mc_g, void* mc_out,
                   int64_t n, int rank, int world, void* const* signal_pads_dev, int pad_base,
                   void* local_scratch, int max_blocks, double lr, double beta1, double beta2,
                   double eps, double wd,
                   int64_t step, double grad_scale, const float* dyn, int g_dtype, int flags, void* stream);
/* K7 Lion: frl_nvls_sgd's arguments with (beta1, beta2) for (mu, dampening); frl_lion's rule and dyn. */
int frl_nvls_lion(float* p, float* m, const void* mc_g, void* mc_out, int64_t n, int rank, int world,
                  void* const* signal_pads_dev, int pad_base, void* local_scratch, int max_blocks, double lr,
                  double beta1, double beta2, double wd, double grad_scale, const float* dyn, int g_dtype, int flags,
                  void* stream);
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
