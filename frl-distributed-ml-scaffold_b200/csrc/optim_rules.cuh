// Update rules shared by the single-GPU update kernel (optim.cu) and the fused NVLS
// reduce + update + broadcast kernel (nvls.cu).  Scalar, fp32, torch 2.11 operation order.
#pragma once
#include "frl_common.cuh"

namespace frl {

// ---- update rules (scalar, fp32) ------------------------------------------------------------
// patch(dyn): the per-step scalars of the rule's dyn layout.  patch_group(row): the same from one
// row of a parameter-group table (FRL_GROUP_DYN_COLS floats: columns 0-3 the dyn layout for that
// group's lr / wd, column 4 the group's L2-coupled decay, read by the rules that have one).
struct SgdRule {
    float neg_lr, mu, one_minus_damp, wd;
    int first_step, has_buf;
    static constexpr int kStates = 1;
    __device__ __forceinline__ void patch(const float* dyn) { neg_lr = -__ldg(dyn); }
    __device__ __forceinline__ void patch_group(const float* row) { patch(row); wd = __ldg(row + 4); }
    __device__ __forceinline__ void operator()(float& p, float g, float& buf, float&, float&) const {
        g = fmaf(wd, p, g);
        if (has_buf) {
            buf = first_step ? g : fmaf(mu, buf, one_minus_damp * g);
            g = buf;
        }
        p = fmaf(neg_lr, g, p);
    }
};

// Adam's step after any weight decay: moments, amsgrad maximum, bias-corrected parameter update.
template <bool AMSGRAD>
__device__ __forceinline__ void adam_moments_and_param(float& p, float g, float& m, float& v, float& vmax,
                                                       float w1, float beta2, float w2, float eps,
                                                       float neg_step_size, float bc2_sqrt) {
    m = fmaf(w1, g - m, m);                       // exp_avg.lerp_(g, 1-beta1), weight < 0.5 branch
    v = fmaf(w2 * g, g, v * beta2);               // mul_(beta2).addcmul_(g, g, 1-beta2)
    float vv = v;
    if (AMSGRAD) {                                // torch.maximum: NaN in either operand wins
        vmax = (v > vmax || v != v) ? v : vmax;   // (fmaxf would drop it)
        vv = vmax;
    }
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    p = fmaf(neg_step_size, m / denom, p);        // addcdiv_(m, denom, -step_size)
}

template <bool AMSGRAD>
struct AdamRule {
    float w1;               // 1 - beta1   (lerp weight)
    float beta2, w2;        // beta2, 1 - beta2
    float eps, wd;
    float neg_step_size;    // -lr / (1 - beta1^t)
    float bc2_sqrt;         // sqrt(1 - beta2^t)
    static constexpr int kStates = AMSGRAD ? 3 : 2;
    __device__ __forceinline__ void patch(const float* dyn) {
        neg_step_size = __ldg(dyn);
        bc2_sqrt = __ldg(dyn + 1);
    }
    __device__ __forceinline__ void patch_group(const float* row) { patch(row); wd = __ldg(row + 4); }
    __device__ __forceinline__ void operator()(float& p, float g, float& m, float& v, float& vmax) const {
        g = fmaf(wd, p, g);                           // L2-coupled decay (torch Adam)
        adam_moments_and_param<AMSGRAD>(p, g, m, v, vmax, w1, beta2, w2, eps, neg_step_size, bc2_sqrt);
    }
};

// AdamW: torch 2.11's Adam(decoupled_weight_decay=True), i.e. torch.optim.AdamW.  The parameter is
// first scaled by its own fp32 multiply, p * fp32(1 - lr*wd) (torch: param.mul_(1 - lr*weight_decay)),
// then Adam's step runs with no decay term in the gradient.  dyn[2] carries the decay factor, so
// under CUDA-graph replay it follows the scheduled lr as the bias-corrected step size does.
template <bool AMSGRAD>
struct AdamWRule {
    float w1;               // 1 - beta1   (lerp weight)
    float beta2, w2;        // beta2, 1 - beta2
    float eps;
    float neg_step_size;    // -lr / (1 - beta1^t)
    float bc2_sqrt;         // sqrt(1 - beta2^t)
    float decay;            // fp32(1 - lr*wd), formed in double
    static constexpr int kStates = AMSGRAD ? 3 : 2;
    __device__ __forceinline__ void patch(const float* dyn) {
        neg_step_size = __ldg(dyn);
        bc2_sqrt = __ldg(dyn + 1);
        decay = __ldg(dyn + 2);
    }
    __device__ __forceinline__ void patch_group(const float* row) { patch(row); }
    __device__ __forceinline__ void operator()(float& p, float g, float& m, float& v, float& vmax) const {
        p = __fmul_rn(p, decay);                      // param.mul_(1 - lr*wd): its own rounding, never
                                                      // contracted into the update's FMA
        adam_moments_and_param<AMSGRAD>(p, g, m, v, vmax, w1, beta2, w2, eps, neg_step_size, bc2_sqrt);
    }
};

// Lion (Chen et al. 2023, Algorithm 2) with decoupled weight decay: one state, m = exp_avg.
//   p = p * fp32(1 - lr*wd)            its own multiply, as AdamWRule's
//   c = lerp(m, g, 1 - beta1)          the update direction's interpolation
//   p = p - lr * sign(c)               sign(NaN) is NaN, so a non-finite gradient reaches the weight
//   m = lerp(m, g, 1 - beta2)
// dyn[0] is lr and dyn[1] the decay factor, so a replayed graph follows the scheduled lr in both.
struct LionRule {
    float w1, w2;           // 1 - beta1, 1 - beta2   (lerp weights)
    float neg_lr;
    float decay;            // fp32(1 - lr*wd), formed in double
    static constexpr int kStates = 1;
    __device__ __forceinline__ void patch(const float* dyn) {
        neg_lr = -__ldg(dyn);
        decay = __ldg(dyn + 1);
    }
    __device__ __forceinline__ void patch_group(const float* row) { patch(row); }
    __device__ __forceinline__ void operator()(float& p, float g, float& m, float&, float&) const {
        p = __fmul_rn(p, decay);
        const float c = fmaf(w1, g - m, m);
        const float s = c > 0.f ? 1.f : c < 0.f ? -1.f : c == 0.f ? 0.f : c;     // NaN stays NaN
        p = fmaf(neg_lr, s, p);
        m = fmaf(w2, g - m, m);
    }
};

template <bool MOMENTUM>
struct RmspropRule {
    float alpha, one_minus_alpha, eps, wd, mu, neg_lr;
    static constexpr int kStates = MOMENTUM ? 2 : 1;
    __device__ __forceinline__ void patch(const float* dyn) { neg_lr = -__ldg(dyn); }
    __device__ __forceinline__ void patch_group(const float* row) { patch(row); wd = __ldg(row + 4); }
    __device__ __forceinline__ void operator()(float& p, float g, float& sq, float& buf, float&) const {
        g = fmaf(wd, p, g);
        sq = fmaf(one_minus_alpha * g, g, sq * alpha);
        const float avg = sqrtf(sq) + eps;
        float upd = g / avg;
        if (MOMENTUM) { buf = fmaf(mu, buf, upd); upd = buf; }
        p = fmaf(neg_lr, upd, p);
    }
};


// Parameter groups of a segment-table update (the _mt_grouped forms): per segment its group and
// its FRL_LW_CLIPPED flag, per group one row of FRL_GROUP_DYN_COLS floats.  Zero in the ungrouped
// instantiations, which never read it.
struct GroupTable {
    const int32_t* seg_group;
    const int32_t* seg_flags;
    const float* rows;
};

// the argument checks of a grouped launch (inside a function returning int); the group index of each
// segment is validated on the host when the table is built
#define FRL_CHECK_GROUPS(grp, n_groups, name)                                                            \
    do {                                                                                                 \
        FRL_REQUIRE((n_groups) >= 1, FRL_E_ARG, "%s: n_groups %d < 1", name, (n_groups));                 \
        FRL_REQUIRE((grp).seg_group && (grp).seg_flags && (grp).rows, FRL_E_ARG,                         \
                    "%s: null seg_group / seg_flags / group_dyn", name);                                 \
        FRL_REQUIRE(aligned16((grp).rows), FRL_E_ALIGN, "%s: group_dyn must be 16-byte aligned", name);  \
    } while (0)

// ---- host-side construction from the double-precision hyper-parameters -----------------------
static inline SgdRule make_sgd_rule(double lr, double mu, double dampening, double wd, int first_step) {
    return SgdRule{static_cast<float>(-lr), static_cast<float>(mu), static_cast<float>(1.0 - dampening),
                   static_cast<float>(wd), first_step ? 1 : 0, (mu != 0.0) ? 1 : 0};
}
template <bool AMS>
static inline AdamRule<AMS> make_adam_rule(double lr, double beta1, double beta2, double eps, double wd,
                                           int64_t step) {
    // bias corrections in double, as torch computes them from Python floats
    const double bc1 = 1.0 - pow(beta1, static_cast<double>(step));
    const double bc2 = 1.0 - pow(beta2, static_cast<double>(step));
    return AdamRule<AMS>{static_cast<float>(1.0 - beta1), static_cast<float>(beta2),
                         static_cast<float>(1.0 - beta2), static_cast<float>(eps), static_cast<float>(wd),
                         static_cast<float>(-(lr / bc1)), static_cast<float>(sqrt(bc2))};
}
template <bool AMS>
static inline AdamWRule<AMS> make_adamw_rule(double lr, double beta1, double beta2, double eps, double wd,
                                             int64_t step) {
    const double bc1 = 1.0 - pow(beta1, static_cast<double>(step));
    const double bc2 = 1.0 - pow(beta2, static_cast<double>(step));
    return AdamWRule<AMS>{static_cast<float>(1.0 - beta1), static_cast<float>(beta2),
                          static_cast<float>(1.0 - beta2), static_cast<float>(eps),
                          static_cast<float>(-(lr / bc1)), static_cast<float>(sqrt(bc2)),
                          static_cast<float>(1.0 - lr * wd)};
}
// the argument checks every Lion entry point makes before any launch (inside a function returning int)
#define FRL_CHECK_LION(beta1, beta2, m, name)                                                            \
    do {                                                                                                 \
        FRL_REQUIRE((m) != nullptr, FRL_E_ARG, "%s: null exp_avg", name);                                \
        FRL_REQUIRE((beta1) >= 0.0 && (beta1) < 1.0 && (beta2) >= 0.0 && (beta2) < 1.0, FRL_E_ARG,        \
                    "%s: betas (%g, %g) outside [0, 1)", name, (beta1), (beta2));                        \
    } while (0)
static inline LionRule make_lion_rule(double lr, double beta1, double beta2, double wd) {
    return LionRule{static_cast<float>(1.0 - beta1), static_cast<float>(1.0 - beta2), static_cast<float>(-lr),
                    static_cast<float>(1.0 - lr * wd)};
}
template <bool MOM>
static inline RmspropRule<MOM> make_rmsprop_rule(double lr, double alpha, double eps, double wd, double mu) {
    return RmspropRule<MOM>{static_cast<float>(alpha), static_cast<float>(1.0 - alpha), static_cast<float>(eps),
                            static_cast<float>(wd), static_cast<float>(mu), static_cast<float>(-lr)};
}

}  // namespace frl
