// pose.cu — camera extrinsics refinement (DESIGN.md §6i): per-image pose corrections (omega_i, tau_i) trained with the
// model.
//
// Corrections live in one fp32 buffer [n_img, 8] = (omega_x, omega_y, omega_z, 0, tau_x, tau_y, tau_z, 0); the gradient
// and the two Adam moments have the same layout, so every row is two float4.
//
//   ngp_pose_apply: R'_i = Exp(omega_i) R_i (Rodrigues), o'_i = o_i + tau_i, rays_d = R' c, rays_o = o'.
//   ngp_pose_grad:  per ray G_o = sum_s g_s, G_d = sum_s t_s g_s (g_s = dL/dx_s of the ray's samples); per image
//                   grad[i] += (d' x G_d, G_o).
//   ngp_pose_adam:  omega gradient through J_l(omega)^T, unscale, inf-skip, Adam, gradient zeroed.
#include "refine.cuh"

namespace {

using ngp::kSeriesTheta2;
using ngp::so3_exp;

__device__ __forceinline__ int64_t clamp_img(int64_t img, int64_t n_img) {
    return min(max(img, (int64_t)0), n_img - 1);
}

__global__ void __launch_bounds__(256) pose_apply_kernel(const float* __restrict__ dirs,
                                                         const int64_t* __restrict__ img_idxs,
                                                         const float* __restrict__ poses,
                                                         const float* __restrict__ corr, int64_t n_img,
                                                         float* __restrict__ rays_o, float* __restrict__ rays_d,
                                                         int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t img = clamp_img(img_idxs[i], n_img);
    const float* P = poses + img * 12;   // row-major [3][4] camera-to-world
    const float4 t4 = reinterpret_cast<const float4*>(corr)[img * 2 + 1];
    float R[9];
    ngp::corrected_rotation(poses, corr, img, R);   // omega = 0 keeps R (Exp(0) R is exactly R)
    const float d0 = dirs[i * 3 + 0], d1 = dirs[i * 3 + 1], d2 = dirs[i * 3 + 2];
    const float tau[3] = {t4.x, t4.y, t4.z};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        // the order of ngp_sample_ray_batch (rays.cu): sum_c d[c] * R[a][c], strict fp32 in source order
        rays_d[i * 3 + a] = f_add(f_add(f_mul(d0, R[a * 3 + 0]), f_mul(d1, R[a * 3 + 1])), f_mul(d2, R[a * 3 + 2]));
        const float o = P[a * 4 + 3];
        rays_o[i * 3 + a] = tau[a] != 0.0f ? f_add(o, tau[a]) : o;   // tau = 0 keeps o (and the sign of a zero)
    }
}

// One warp per ray, kPoseRaysPerWarp consecutive rays per warp.  Lanes stride over the ray's samples; the six sums are
// reduced with shuffles, so each ray's (G_o, d' x G_d) is formed in a fixed order.  Consecutive rays of one image are
// summed in registers and reach the [n_img, 8] buffer as one atomicAdd per component; contributions of different warps
// to one image meet in the atomics, in no fixed order.
constexpr int kPoseRaysPerWarp = 16;

__global__ void __launch_bounds__(256) pose_grad_kernel(const float* __restrict__ dx, const float* __restrict__ ts,
                                                        const int32_t* __restrict__ rays_a,
                                                        const int64_t* __restrict__ img_idxs,
                                                        const float* __restrict__ rays_d, int64_t n_max,
                                                        const int32_t* __restrict__ n_dev, int64_t n_rows,
                                                        int64_t n_img, float* __restrict__ grad,
                                                        int32_t* __restrict__ found_inf) {
    int64_t n = n_max;
    if (n_dev != nullptr) n = min(n, (int64_t)max(*n_dev, 0));
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t k0 = warp * kPoseRaysPerWarp;
    if (k0 >= n) return;
    const int64_t k1 = min(k0 + kPoseRaysPerWarp, n);
    int64_t cur = -1;       // image whose sums are being carried
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    bool bad = false;
    auto flush = [&]() {
        if (cur >= 0 && lane < 6) {
            // lane j adds component j: (omega-part 0..2, tau-part 4..6)
            float v = acc[0];
#pragma unroll
            for (int j = 1; j < 6; ++j)
                if (lane == j) v = acc[j];
            atomicAdd(grad + cur * 8 + (lane < 3 ? lane : lane + 1), v);
        }
    };
    for (int64_t k = k0; k < k1; ++k) {
        const int64_t ray = rays_a[k * 3 + 0];
        const int64_t start = rays_a[k * 3 + 1];
        int64_t cnt = rays_a[k * 3 + 2];
        cnt = min(cnt, n_rows - start);   // never read past the sample buffers
        if (cnt <= 0 || start < 0) continue;
        float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f};
        for (int64_t s = start + lane; s < start + cnt; s += 32) {
            const float t = ts[s];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float g = dx[s * 3 + c];
                go[c] += g;
                gd[c] = fmaf(t, g, gd[c]);
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            go[c] = warp_sum(go[c]);
            gd[c] = warp_sum(gd[c]);
        }
        const float d0 = rays_d[ray * 3 + 0], d1 = rays_d[ray * 3 + 1], d2 = rays_d[ray * 3 + 2];
        const float r[6] = {d1 * gd[2] - d2 * gd[1], d2 * gd[0] - d0 * gd[2], d0 * gd[1] - d1 * gd[0],
                            go[0], go[1], go[2]};
        const int64_t img = clamp_img(img_idxs[ray], n_img);
        if (img != cur) {
            flush();
            cur = img;
#pragma unroll
            for (int j = 0; j < 6; ++j) acc[j] = 0.f;
        }
#pragma unroll
        for (int j = 0; j < 6; ++j) {
            bad |= !isfinite(r[j]);
            acc[j] += r[j];
        }
    }
    flush();
    if (bad && lane == 0 && found_inf != nullptr) atomicExch(found_inf, 1);
}

// J_l(w) = I + B K + C K^2, B = (1 - cos t)/t^2, C = (t - sin t)/t^3; J_l^T = I - B K + C K^2
__device__ void so3_jl_transpose_apply(const double w[3], const double g[3], double out[3]) {
    const double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    double B, Cc;
    if (t2 < kSeriesTheta2) {
        B = 0.5 - t2 / 24.0 + t2 * t2 / 720.0;
        Cc = 1.0 / 6.0 - t2 / 120.0 + t2 * t2 / 5040.0;
    } else {
        const double t = sqrt(t2), s = sin(0.5 * t);
        B = 2.0 * s * s / t2;
        Cc = (t - sin(t)) / (t2 * t);
    }
    // K g = w x g; K^2 g = w (w.g) - t^2 g
    const double kg[3] = {w[1] * g[2] - w[2] * g[1], w[2] * g[0] - w[0] * g[2], w[0] * g[1] - w[1] * g[0]};
    const double wg = w[0] * g[0] + w[1] * g[1] + w[2] * g[2];
#pragma unroll
    for (int a = 0; a < 3; ++a) out[a] = g[a] - B * kg[a] + Cc * (w[a] * wg - t2 * g[a]);
}

__global__ void __launch_bounds__(128) pose_adam_kernel(float* __restrict__ corr, float* __restrict__ grad,
                                                        float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                        const int32_t* __restrict__ found_inf,
                                                        const float* __restrict__ hyper, float lr_ratio, float beta1,
                                                        float beta2, float eps, int64_t n_img) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_img) return;
    const bool skip = found_inf != nullptr && *found_inf != 0;
    float4* G = reinterpret_cast<float4*>(grad) + i * 2;
    if (!skip) {
        float4* P = reinterpret_cast<float4*>(corr) + i * 2;
        float4* M = reinterpret_cast<float4*>(exp_avg) + i * 2;
        float4* V = reinterpret_cast<float4*>(exp_avg_sq) + i * 2;
        float4 p0 = P[0], p1 = P[1], m0 = M[0], m1 = M[1], v0 = V[0], v1 = V[1];
        const float4 g0 = G[0], g1 = G[1];
        // the world-frame rotation gradient becomes the gradient of omega through the left Jacobian
        const double w[3] = {p0.x, p0.y, p0.z}, gw[3] = {g0.x, g0.y, g0.z};
        double gj[3];
        so3_jl_transpose_apply(w, gw, gj);
        const float lr = __fmul_rn(lr_ratio, hyper[0]), bc2 = hyper[1], inv = hyper[2];
        ngp::refine_adam1(p0.x, (float)gj[0], m0.x, v0.x, lr, bc2, beta1, beta2, eps, inv);
        ngp::refine_adam1(p0.y, (float)gj[1], m0.y, v0.y, lr, bc2, beta1, beta2, eps, inv);
        ngp::refine_adam1(p0.z, (float)gj[2], m0.z, v0.z, lr, bc2, beta1, beta2, eps, inv);
        ngp::refine_adam1(p1.x, g1.x, m1.x, v1.x, lr, bc2, beta1, beta2, eps, inv);
        ngp::refine_adam1(p1.y, g1.y, m1.y, v1.y, lr, bc2, beta1, beta2, eps, inv);
        ngp::refine_adam1(p1.z, g1.z, m1.z, v1.z, lr, bc2, beta1, beta2, eps, inv);
        P[0] = p0;
        P[1] = p1;
        M[0] = m0;
        M[1] = m1;
        V[0] = v0;
        V[1] = v1;
    }
    G[0] = G[1] = make_float4(0.f, 0.f, 0.f, 0.f);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int ngp_pose_apply(const float* directions, const int64_t* img_idxs, const float* poses, const float* corr,
                   int64_t n_img, float* rays_o, float* rays_d, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(n_img > 0, "n_img must be > 0");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(directions && img_idxs && poses && corr && rays_o && rays_d, "null pointer");
    NGP_REQUIRE(aligned16(corr), "corrections must be 16-byte aligned");
    pose_apply_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        directions, img_idxs, poses, corr, n_img, rays_o, rays_d, n_rays);
    NGP_LAUNCHED("pose_apply_kernel");
    return 0;
}

int ngp_pose_grad(const float* dx, const float* ts, const int32_t* rays_a, const int64_t* img_idxs,
                  const float* rays_d, int64_t n_rays, const int32_t* n_rays_dev, int64_t n_rows, int64_t n_img,
                  float* grad, int32_t* found_inf_or_null, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_rows >= 0, "negative n_rays / n_rows");
    NGP_REQUIRE(n_img > 0, "n_img must be > 0");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && img_idxs && rays_d && grad, "null pointer");
    NGP_REQUIRE(n_rows == 0 || (dx && ts), "null pointer");
    const int64_t warps = (n_rays + kPoseRaysPerWarp - 1) / kPoseRaysPerWarp;
    pose_grad_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        dx, ts, rays_a, img_idxs, rays_d, n_rays, n_rays_dev, n_rows, n_img, grad, found_inf_or_null);
    NGP_LAUNCHED("pose_grad_kernel");
    return 0;
}

int ngp_pose_adam(float* corr, float* grad, float* exp_avg, float* exp_avg_sq, const int32_t* found_inf_or_null,
                  const float* hyper_dev, float lr_ratio, float beta1, float beta2, float eps, int64_t n_img,
                  void* stream) {
    NGP_REQUIRE(n_img >= 0, "negative n_img");
    if (n_img == 0) return 0;
    NGP_REQUIRE(corr && grad && exp_avg && exp_avg_sq && hyper_dev, "null pointer");
    NGP_REQUIRE(aligned16(corr) && aligned16(grad) && aligned16(exp_avg) && aligned16(exp_avg_sq),
                "pose buffers must be 16-byte aligned");
    NGP_REQUIRE(lr_ratio >= 0.0f && lr_ratio < INFINITY, "lr_ratio must be finite and >= 0");
    pose_adam_kernel<<<(unsigned)((n_img + 127) / 128), 128, 0, ngp::as_stream(stream)>>>(
        corr, grad, exp_avg, exp_avg_sq, found_inf_or_null, hyper_dev, lr_ratio, beta1, beta2, eps, n_img);
    NGP_LAUNCHED("pose_adam_kernel");
    return 0;
}

}  // extern "C"
