// activation.cuh -- the hidden-layer activations of ActorCritic (AC_Args.activation, actor_critic.py:149-166 of the reference):
// the one place that knows their formulas.  KIND is a Go1Activation (include/go1_b200.h); `crelu` is ReLU in the reference.
//
//   act_exact<KIND>(v)   f(v), libm-accurate: the exact-fp32 path (impl 0, the generic trailing-input kernel)
//   act_fast<KIND>(v)    f(v), branch-free, for the epilogues of the wgmma path (see the error bound below)
//   act_deriv<KIND>(y)   f'(v) written as a function of the SAVED OUTPUT y = f(v): every backward kernel keeps y only.  The values at
//                        the kink are torch autograd's (v = 0: relu 0, lrelu 0.01, elu / selu the left branch).
//   ActDeriv             the same derivatives as ONE branch-free expression with per-kind coefficients, for the kernels whose register
//                        budget has no room for a six-way switch around an unrolled loop (see gemm_tf32.cu)
//
// Error bound of act_fast: absolute error <= 1e-6 against the fp64 value for every kind over [-30, 30] (plus the fp32 rounding of the
// result itself, one ulp, where |f(v)| > 1: selu of a large v), so that the activation stays well below the TF32 operand rounding
// (5e-4 relative) of the product it feeds.  Established two ways:
//   * analysis: ex2.approx.ftz.f32 is accurate to 2 ulp (2.4e-7 relative) and its argument v log2(e), rounded to fp32, adds |v| 6e-8
//     relative.  elu / selu: below -0.35 the result e - 1 carries the absolute error of e <= 0.71, i.e. < 2e-7 (x lambda alpha = 1.76
//     for selu); above, the degree-7 Taylor polynomial truncates at 0.35^8 / 8! = 6e-9.  sigmoid = 1 / (1 + e^-v): an error eps relative
//     in e^-v moves the quotient by s (1 - s) eps <= eps / 4, the reciprocal (rcp.approx, 1 ulp) adds 6e-8.  tanh = 1 - 2 / (1 + e^2v)
//     outside (-0.25, 0.25): same argument, twice the sensitivity (< 4e-7); inside, the odd degree-9 Taylor polynomial, whose next term is
//     below 0.0089 x 0.25^11 = 2.2e-9, keeps the RELATIVE accuracy that the quotient form loses to cancellation near 0.
//   * measurement: tests/test_activations_gpu.py sweeps 2^20 points of [-30, 30] through a kernel that uses act_fast, against fp64, and
//     asserts this bound on an H100 (and 1e-6 RELATIVE for |v| < 0.2 for elu / selu / tanh).
#pragma once
#include "../../include/go1_b200.h"

#define GO1_ACT_DI __device__ __forceinline__

constexpr float GO1_SELU_LAMBDA = 1.0507009873554805f, GO1_SELU_ALPHA = 1.6732632423543772f;
constexpr float GO1_LRELU_SLOPE = 0.01f;      // nn.LeakyReLU() default

// Runs `...` with KD bound to the compile-time value of the (warp-uniform) runtime kind: the switch sits OUTSIDE the unrolled epilogue
// loops, so each loop body holds one activation's straight-line code.  The callers have validated the kind (go1_act_kind_ok).
#define GO1_ACT_SWITCH(kind, KD, ...)                                          \
    switch (kind) {                                                            \
    case GO1_ACT_SELU: { constexpr int KD = GO1_ACT_SELU; __VA_ARGS__ } break;         \
    case GO1_ACT_RELU: { constexpr int KD = GO1_ACT_RELU; __VA_ARGS__ } break;         \
    case GO1_ACT_LRELU: { constexpr int KD = GO1_ACT_LRELU; __VA_ARGS__ } break;       \
    case GO1_ACT_TANH: { constexpr int KD = GO1_ACT_TANH; __VA_ARGS__ } break;         \
    case GO1_ACT_SIGMOID: { constexpr int KD = GO1_ACT_SIGMOID; __VA_ARGS__ } break;   \
    default: { constexpr int KD = GO1_ACT_ELU; __VA_ARGS__ } break;                    \
    }

static inline bool go1_act_kind_ok(int kind) { return kind >= GO1_ACT_ELU && kind <= GO1_ACT_SIGMOID; }

GO1_ACT_DI float go1_ex2_approx(float x) {
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x));
    return e;
}

// expm1(v) for v <= 0, branch-free: a degree-7 Taylor polynomial on (-0.35, 0] (truncation error < 2e-8 relative) and
// ex2.approx(v log2 e) - 1 below it (absolute error ~1e-7 on a value >= 0.29); 13 instructions instead of expm1f's ~28 plus a
// divergent branch.
GO1_ACT_DI float go1_expm1_neg_fast(float v) {
    float p = fmaf(v, 1.f / 5040.f, 1.f / 720.f);
    p = fmaf(p, v, 1.f / 120.f); p = fmaf(p, v, 1.f / 24.f); p = fmaf(p, v, 1.f / 6.f); p = fmaf(p, v, 0.5f);
    p = fmaf(p * v, v, v);
    const float e = go1_ex2_approx(v * 1.4426950408889634f);
    return v > -0.35f ? p : e - 1.0f;
}

template <int KIND> GO1_ACT_DI float act_exact(float v) {
    if (KIND == GO1_ACT_SELU) return GO1_SELU_LAMBDA * (v > 0.f ? v : GO1_SELU_ALPHA * expm1f(v));
    if (KIND == GO1_ACT_RELU) return v > 0.f ? v : 0.f;
    if (KIND == GO1_ACT_LRELU) return v > 0.f ? v : GO1_LRELU_SLOPE * v;
    if (KIND == GO1_ACT_TANH) return tanhf(v);
    if (KIND == GO1_ACT_SIGMOID) return 1.0f / (1.0f + expf(-v));
    return v > 0.f ? v : expm1f(v);
}

template <int KIND> GO1_ACT_DI float act_fast(float v) {
    if (KIND == GO1_ACT_SELU) return GO1_SELU_LAMBDA * (v > 0.f ? v : GO1_SELU_ALPHA * go1_expm1_neg_fast(v));
    if (KIND == GO1_ACT_RELU) return v > 0.f ? v : 0.f;
    if (KIND == GO1_ACT_LRELU) return v > 0.f ? v : GO1_LRELU_SLOPE * v;
    if (KIND == GO1_ACT_TANH) {
        const float v2 = v * v;
        float p = fmaf(v2, 62.f / 2835.f, -17.f / 315.f);
        p = fmaf(p, v2, 2.f / 15.f); p = fmaf(p, v2, -1.f / 3.f);
        p = fmaf(p * v2, v, v);
        const float q = 1.0f - __fdividef(2.0f, 1.0f + go1_ex2_approx(v * 2.8853900817779268f));      // e^2v = inf: 1 - 0
        return fabsf(v) < 0.25f ? p : q;
    }
    if (KIND == GO1_ACT_SIGMOID) return __fdividef(1.0f, 1.0f + go1_ex2_approx(v * -1.4426950408889634f));
    const float n = go1_expm1_neg_fast(v);
    return v > 0.f ? v : n;
}

template <int KIND> GO1_ACT_DI float act_deriv(float y) {
    if (KIND == GO1_ACT_SELU) return y > 0.f ? GO1_SELU_LAMBDA : y + GO1_SELU_LAMBDA * GO1_SELU_ALPHA;
    if (KIND == GO1_ACT_RELU) return y > 0.f ? 1.0f : 0.f;
    if (KIND == GO1_ACT_LRELU) return y > 0.f ? 1.0f : GO1_LRELU_SLOPE;
    if (KIND == GO1_ACT_TANH) return fmaf(-y, y, 1.0f);
    if (KIND == GO1_ACT_SIGMOID) return y * (1.0f - y);
    return y > 0.f ? 1.0f : y + 1.0f;
}

// Every derivative above is (y > 0 ? a1 : a0) + (y > 0 ? b1 : b0) y + c y^2:
//   elu (1, 1, 0, 1, 0)   selu (lambda, lambda alpha, 0, 1, 0)   relu (1, 0, 0, 0, 0)   lrelu (1, 0.01, 0, 0, 0)   tanh (1, 1, 0, 0, -1)
//   sigmoid (0, 0, 1, 1, -1)
// evaluated as fma(y, fma(c, y, b), a), which rounds like act_deriv<KIND> for finite y (y + 1, 1 - y^2 and y (1 - y) are each one
// rounding on top of exact terms).
struct ActDeriv {
    float a1, a0, b1, b0, c;
    GO1_ACT_DI float operator()(float y) const { const bool pos = y > 0.f; return fmaf(y, fmaf(c, y, pos ? b1 : b0), pos ? a1 : a0); }
};
GO1_ACT_DI ActDeriv act_deriv_coefficients(int kind) {
    ActDeriv d = {1.f, 1.f, 0.f, 1.f, 0.f};
    if (kind == GO1_ACT_SELU) { d.a1 = GO1_SELU_LAMBDA; d.a0 = GO1_SELU_LAMBDA * GO1_SELU_ALPHA; }
    else if (kind == GO1_ACT_RELU) { d.a0 = 0.f; d.b0 = 0.f; }
    else if (kind == GO1_ACT_LRELU) { d.a0 = GO1_LRELU_SLOPE; d.b0 = 0.f; }
    else if (kind == GO1_ACT_TANH) { d.b0 = 0.f; d.c = -1.f; }
    else if (kind == GO1_ACT_SIGMOID) { d.a1 = 0.f; d.a0 = 0.f; d.b1 = 1.f; d.c = -1.f; }
    return d;
}
