// refine.cuh — device helpers shared by the camera refinement kernels: the rotation of extrinsics refinement
// (pose.cu, DESIGN.md §6i), which intrinsics refinement (camera.cu, §6l) chains its gradient through, and the Adam
// update both apply to their corrections.
#pragma once

#include "common.cuh"

namespace ngp {

// theta^2 below which Exp and J_l use their Taylor series (the closed forms cancel there); fp64, so the series'
// first omitted term (theta^6 / 5040 at most) stays far below fp32 precision
constexpr double kSeriesTheta2 = 1e-6;

// Exp(w) = I + A K + B K^2, K = [w]x, A = sin(t)/t, B = (1 - cos t)/t^2 = 2 sin^2(t/2)/t^2 (no cancellation).
// kSinPi: sin through sinpi(t / pi), whose argument reduction is exact and needs no stack frame (fp64 sin keeps its
// slow-path reduction on the stack); t / pi adds one fp64 rounding, far below the fp32 the rotation is rounded to.
template <bool kSinPi = false>
__device__ inline void so3_exp(const double w[3], double E[9]) {
    const double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    double A, B;
    if (t2 < kSeriesTheta2) {
        A = 1.0 - t2 / 6.0 + t2 * t2 / 120.0;
        B = 0.5 - t2 / 24.0 + t2 * t2 / 720.0;
    } else {
        const double t = sqrt(t2);
        double s, st;
        if constexpr (kSinPi) {
            const double tp = t * (1.0 / 3.141592653589793238462643383279502884);
            s = sinpi(0.5 * tp);
            st = sinpi(tp);
        } else {
            s = sin(0.5 * t);
            st = sin(t);
        }
        A = st / t;
        B = 2.0 * s * s / t2;
    }
    // K^2 = w w^T - t^2 I
    const double c = 1.0 - B * t2;
    E[0] = c + B * w[0] * w[0];
    E[4] = c + B * w[1] * w[1];
    E[8] = c + B * w[2] * w[2];
    E[1] = B * w[0] * w[1] - A * w[2];
    E[3] = B * w[0] * w[1] + A * w[2];
    E[2] = B * w[0] * w[2] + A * w[1];
    E[6] = B * w[0] * w[2] - A * w[1];
    E[5] = B * w[1] * w[2] - A * w[0];
    E[7] = B * w[1] * w[2] + A * w[0];
}

// The rotation R' = Exp(omega) R of image img's pose as ngp_pose_apply forms it (fp64, rounded once to fp32; omega = 0
// or no corrections keep R).  poses [n_img, 3, 4] row-major camera-to-world, corr [n_img, 8] or null.  kSinPi: see
// so3_exp.
template <bool kSinPi = false>
__device__ inline void corrected_rotation(const float* __restrict__ poses, const float* __restrict__ corr, int64_t img,
                                          float R[9]) {
    const float* P = poses + img * 12;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int k = 0; k < 3; ++k) R[a * 3 + k] = P[a * 4 + k];
    if (corr == nullptr) return;
    const float4 w4 = reinterpret_cast<const float4*>(corr)[img * 2 + 0];
    if (w4.x != 0.0f || w4.y != 0.0f || w4.z != 0.0f) {
        const double w[3] = {w4.x, w4.y, w4.z};
        double E[9];
        so3_exp<kSinPi>(w, E);
        float Rn[9];
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
            for (int k = 0; k < 3; ++k)
                Rn[a * 3 + k] = (float)(E[a * 3 + 0] * (double)R[k] + E[a * 3 + 1] * (double)R[3 + k] +
                                        E[a * 3 + 2] * (double)R[6 + k]);
#pragma unroll
        for (int k = 0; k < 9; ++k) R[k] = Rn[k];
    }
}

// Adam of ngp_adam_step_dyn (optim.cu, adam1), contractions spelled out the same way
__device__ __forceinline__ void refine_adam1(float& p, float g, float& m, float& v, float lr_over_bc1, float bc2_sqrt,
                                             float beta1, float beta2, float eps, float inv_scale) {
    const float gg = __fmul_rn(g, inv_scale);
    m = __fmaf_rn(__fsub_rn(gg, m), 1.0f - beta1, m);
    v = __fmaf_rn(v, beta2, __fmul_rn(__fmul_rn(1.0f - beta2, gg), gg));
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), bc2_sqrt), eps);
    p = __fmaf_rn(-lr_over_bc1, __fdiv_rn(m, denom), p);
}

}  // namespace ngp
