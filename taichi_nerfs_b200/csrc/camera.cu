// camera.cu — camera intrinsics (DESIGN.md §6l): lens distortion and a learned focal length and principal point.
//
// Pixel p of a W x H image has u = p mod W, v = floor(p / W); its distorted normalised coordinates are
// x_d = (u - cx' + 0.5) / fx', y_d = (v - cy' + 0.5) / fy' in fp32 in the order of get_ray_directions, and its
// camera-frame direction is (x_u, y_u, 1) with (x_u, y_u) = U(x_d, y_d), U the inverse of the distortion map D
// (OPENCV form: radial 1 + k1 r^2 + k2 r^4, tangential p1, p2), found by Newton's method in fp64 and rounded once.
// Corrections (a, b_x, b_y, 0): fx' = fx e^a, fy' = fy e^a, cx' = cx + W b_x, cy' = cy + H b_y.
//
//   ngp_camera_unproject: directions of pixels (a list or the whole image) under the corrected intrinsics.
//   ngp_intrinsics_grad:  per ray, G_d = sum_s t_s g_s chained through R'^T, U and the pixel's coordinates.
//   ngp_intrinsics_adam:  fixed-order fp64 reduction of the per-ray gradients, then the model's Adam.
#include "refine.cuh"

namespace {

struct Camera {
    double fx, fy, cx, cy, k1, k2, p1, p2;
};

constexpr int kNewtonIters = 20;
// |D(x) - x_d| (infinity norm, normalised coordinates) at which Newton stops; fp64 evaluates D to ~1e-16 here
constexpr double kNewtonTol = 1e-13;

// D and its Jacobian J = [[j00, j01], [j10, j11]] at (x, y)
__device__ __forceinline__ void distort(const Camera& c, double x, double y, double& dx, double& dy, double J[4]) {
    const double r2 = x * x + y * y;
    const double rad = 1.0 + c.k1 * r2 + c.k2 * r2 * r2;
    const double q = 2.0 * c.k1 + 4.0 * c.k2 * r2;   // d rad / d(x, y) = q (x, y)
    dx = x * rad + 2.0 * c.p1 * x * y + c.p2 * (r2 + 2.0 * x * x);
    dy = y * rad + c.p1 * (r2 + 2.0 * y * y) + 2.0 * c.p2 * x * y;
    J[0] = rad + q * x * x + 2.0 * c.p1 * y + 6.0 * c.p2 * x;
    J[1] = q * x * y + 2.0 * c.p1 * x + 2.0 * c.p2 * y;
    J[2] = J[1];
    J[3] = rad + q * y * y + 6.0 * c.p1 * y + 2.0 * c.p2 * x;
}

// The corrected intrinsics, each formed in fp64 and rounded once (zero corrections give exactly fx, cx, ...)
struct Pinhole {
    float fx, fy, cx, cy;
};

__device__ __forceinline__ Pinhole corrected(const Camera& c, const float* corr, int64_t W, int64_t H) {
    double fx = c.fx, fy = c.fy, cx = c.cx, cy = c.cy;
    if (corr != nullptr) {
        const float4 k = *reinterpret_cast<const float4*>(corr);
        if (k.x != 0.0f) {
            const double e = exp((double)k.x);
            fx *= e;
            fy *= e;
        }
        if (k.y != 0.0f) cx += (double)W * (double)k.y;
        if (k.z != 0.0f) cy += (double)H * (double)k.z;
    }
    return {(float)fx, (float)fy, (float)cx, (float)cy};
}

// get_ray_directions' ((u - cx) + 0.5) / fx, strict fp32
__device__ __forceinline__ void pixel_xd(int64_t p, int64_t W, const Pinhole& k, float& xd, float& yd) {
    const float u = (float)(p % W), v = (float)(p / W);
    xd = f_div(f_add(f_sub(u, k.cx), 0.5f), k.fx);
    yd = f_div(f_add(f_sub(v, k.cy), 0.5f), k.fy);
}

__global__ void __launch_bounds__(256) unproject_kernel(const int64_t* __restrict__ pix, int64_t n, int64_t W,
                                                        int64_t H, Camera cam, const float* __restrict__ corr,
                                                        float* __restrict__ dirs, float4* __restrict__ grad_rows,
                                                        int32_t* __restrict__ n_bad, int32_t* __restrict__ found_inf) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (grad_rows != nullptr) grad_rows[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int64_t p = pix == nullptr ? i : min(max(pix[i], (int64_t)0), W * H - 1);
    const Pinhole k = corrected(cam, corr, W, H);
    float xdf, ydf;
    pixel_xd(p, W, k, xdf, ydf);
    const double xd = xdf, yd = ydf;
    double x = xd, y = yd, J[4];
    bool ok = false;
    for (int it = 0; it <= kNewtonIters; ++it) {
        double fx, fy;
        distort(cam, x, y, fx, fy, J);
        fx -= xd;
        fy -= yd;
        if (fabs(fx) <= kNewtonTol && fabs(fy) <= kNewtonTol) {
            ok = true;
            break;
        }
        if (it == kNewtonIters) break;
        const double det = J[0] * J[3] - J[1] * J[2];
        x -= (J[3] * fx - J[1] * fy) / det;
        y -= (J[0] * fy - J[2] * fx) / det;
    }
    // a root past the fold: det J_D <= 0, or a radial factor <= 0 (D has turned back through zero, so the root lies
    // across the centre, where det J_D can be positive again)
    const double r2 = x * x + y * y;
    ok = ok && (J[0] * J[3] - J[1] * J[2]) > 0.0 && 1.0 + cam.k1 * r2 + cam.k2 * r2 * r2 > 0.0 && isfinite(x) &&
         isfinite(y);
    if (!ok) {   // not invertible: keep the finite distorted coordinates, count the pixel
        x = xd;
        y = yd;
        if (n_bad != nullptr) atomicAdd(n_bad, 1);
        if (found_inf != nullptr) atomicExch(found_inf, 1);
    }
    dirs[i * 3 + 0] = (float)x;
    dirs[i * 3 + 1] = (float)y;
    dirs[i * 3 + 2] = 1.0f;
}

// One warp per rays_a row.  Lanes stride over the ray's samples and the three sums of G_d are reduced with shuffles
// in a fixed order; the ray's gradient goes to its own row grad_rays[ray], so no two rows meet in an atomic.
__global__ void __launch_bounds__(256) intrinsics_grad_kernel(
    const float* __restrict__ dx, const float* __restrict__ ts, const int32_t* __restrict__ rays_a, int64_t n_max,
    const int32_t* __restrict__ n_dev, int64_t n_rows, const int64_t* __restrict__ pix,
    const int64_t* __restrict__ img_idxs, const float* __restrict__ poses, const float* __restrict__ pose_corr,
    int64_t n_img, const float* __restrict__ cam_dirs, int64_t W, int64_t H, Camera cam,
    const float* __restrict__ corr, float4* __restrict__ grad_rays, int64_t max_rays, int32_t* __restrict__ found_inf) {
    int64_t n = n_max;
    if (n_dev != nullptr) n = min(n, (int64_t)max(*n_dev, 0));
    const int lane = threadIdx.x & 31;
    const int64_t k = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (k >= n) return;
    const int64_t ray = rays_a[k * 3 + 0];
    const int64_t start = rays_a[k * 3 + 1];
    int64_t cnt = rays_a[k * 3 + 2];
    cnt = min(cnt, n_rows - start);   // never read past the sample buffers
    if (cnt <= 0 || start < 0 || ray < 0 || ray >= max_rays) return;
    float gd[3] = {0.f, 0.f, 0.f};
    for (int64_t s = start + lane; s < start + cnt; s += 32) {
        const float t = ts[s];
#pragma unroll
        for (int c = 0; c < 3; ++c) gd[c] = fmaf(t, dx[s * 3 + c], gd[c]);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) gd[c] = warp_sum(gd[c]);
    if (lane != 0) return;
    const int64_t img = min(max(img_idxs[ray], (int64_t)0), n_img - 1);
    float R[9];
    ngp::corrected_rotation<true>(poses, pose_corr, img, R);   // (sinpi: no stack frame)
    // g_c = R'^T G_d (d = R' c), its first two components
    double gc[2];
#pragma unroll
    for (int c = 0; c < 2; ++c)
        gc[c] = (double)R[0 * 3 + c] * gd[0] + (double)R[1 * 3 + c] * gd[1] + (double)R[2 * 3 + c] * gd[2];
    const double xu = cam_dirs[ray * 3 + 0], yu = cam_dirs[ray * 3 + 1];
    double ddx, ddy, J[4];
    distort(cam, xu, yu, ddx, ddy, J);
    const double det = J[0] * J[3] - J[1] * J[2];
    // g_xd = J_D^{-T} g_c[0:2]
    const double g0 = (J[3] * gc[0] - J[2] * gc[1]) / det;
    const double g1 = (J[0] * gc[1] - J[1] * gc[0]) / det;
    const Pinhole kp = corrected(cam, corr, W, H);
    const int64_t p = min(max(pix[ray], (int64_t)0), W * H - 1);
    float xd, yd;
    pixel_xd(p, W, kp, xd, yd);
    const float4 r = make_float4((float)(-(g0 * xd + g1 * yd)), (float)(-((double)W / kp.fx) * g0),
                                 (float)(-((double)H / kp.fy) * g1), 0.f);
    grad_rays[ray] = r;
    if (!(isfinite(r.x) && isfinite(r.y) && isfinite(r.z)) && found_inf != nullptr) atomicExch(found_inf, 1);
}

constexpr int kAdamThreads = 256;
// launch limits: at most 2^31 - 1 blocks of 256 threads (unproject) or of 8 rays (gradient)
constexpr int64_t kMaxUnproject = ((int64_t)1 << 31) - 1;
constexpr int64_t kMaxGradRays = ((int64_t)1 << 31) - 1;

// One CTA: thread t sums rays t, t + 256, ... in fp64, then a fixed shared-memory tree; thread 0 runs the Adam.
__global__ void __launch_bounds__(kAdamThreads) intrinsics_adam_kernel(
    float4* __restrict__ corr, const float4* __restrict__ grad_rays, int64_t n, float4* __restrict__ exp_avg,
    float4* __restrict__ exp_avg_sq, const int32_t* __restrict__ found_inf, const float* __restrict__ hyper,
    float lr_ratio, float beta1, float beta2, float eps, float4* __restrict__ grad_out) {
    __shared__ double sh[3][kAdamThreads];
    const int t = threadIdx.x;
    double a = 0.0, bx = 0.0, by = 0.0;
    for (int64_t r = t; r < n; r += kAdamThreads) {
        const float4 g = grad_rays[r];
        a += g.x;
        bx += g.y;
        by += g.z;
    }
    sh[0][t] = a;
    sh[1][t] = bx;
    sh[2][t] = by;
    __syncthreads();
    for (int w = kAdamThreads / 2; w > 0; w >>= 1) {
        if (t < w) {
#pragma unroll
            for (int c = 0; c < 3; ++c) sh[c][t] += sh[c][t + w];
        }
        __syncthreads();
    }
    if (t != 0) return;
    const float g[3] = {(float)sh[0][0], (float)sh[1][0], (float)sh[2][0]};
    if (grad_out != nullptr) *grad_out = make_float4(g[0], g[1], g[2], 0.f);
    if (found_inf != nullptr && *found_inf != 0) return;
    float4 p = *corr, m = *exp_avg, v = *exp_avg_sq;
    const float lr = __fmul_rn(lr_ratio, hyper[0]), bc2 = hyper[1], inv = hyper[2];
    ngp::refine_adam1(p.x, g[0], m.x, v.x, lr, bc2, beta1, beta2, eps, inv);
    ngp::refine_adam1(p.y, g[1], m.y, v.y, lr, bc2, beta1, beta2, eps, inv);
    ngp::refine_adam1(p.z, g[2], m.z, v.z, lr, bc2, beta1, beta2, eps, inv);
    *corr = p;
    *exp_avg = m;
    *exp_avg_sq = v;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// model ids of include/ngp_b200.h: 0 PINHOLE, 1 SIMPLE_RADIAL (k1), 2 RADIAL (k1, k2), 3 OPENCV (k1, k2, p1, p2)
const char* camera_error(int model, const double* p, int64_t W, int64_t H) {
    if (W <= 0 || H <= 0 || W > (int64_t)1 << 24 || H > (int64_t)1 << 24) return "W and H must be in [1, 2^24]";
    if (p == nullptr) return "null camera parameters";
    if (model < 0 || model > 3) return "camera model must be 0 (PINHOLE), 1 (SIMPLE_RADIAL), 2 (RADIAL) or 3 (OPENCV)";
    for (int j = 0; j < 8; ++j)
        if (!isfinite(p[j])) return "camera parameters must be finite";
    if (!(p[0] > 0.0 && p[1] > 0.0)) return "focal lengths must be > 0";
    const int n_dist = model == 0 ? 0 : model == 1 ? 1 : model == 2 ? 2 : 4;
    for (int j = 4 + n_dist; j < 8; ++j)
        if (p[j] != 0.0) return "a distortion term the camera model does not have is non-zero";
    return nullptr;
}

Camera to_camera(const double* p) { return {p[0], p[1], p[2], p[3], p[4], p[5], p[6], p[7]}; }

}  // namespace

extern "C" {

int ngp_camera_unproject(const int64_t* pix_idxs_or_null, int64_t n, int64_t W, int64_t H, int model,
                         const double* params, const float* corr_or_null, float* dirs, float* grad_rows_or_null,
                         int32_t* n_bad_or_null, int32_t* found_inf_or_null, void* stream) {
    const char* e = camera_error(model, params, W, H);
    NGP_REQUIRE(e == nullptr, e);
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(n <= kMaxUnproject, "n must be < 2^31 pixels");
    NGP_REQUIRE(pix_idxs_or_null != nullptr || n == W * H, "without pixel indices n must be W * H");
    if (n == 0) return 0;
    NGP_REQUIRE(dirs, "null pointer");
    NGP_REQUIRE(corr_or_null == nullptr || aligned16(corr_or_null), "corrections must be 16-byte aligned");
    NGP_REQUIRE(grad_rows_or_null == nullptr || aligned16(grad_rows_or_null), "gradient rows must be 16-byte aligned");
    unproject_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        pix_idxs_or_null, n, W, H, to_camera(params), corr_or_null, dirs,
        reinterpret_cast<float4*>(grad_rows_or_null), n_bad_or_null, found_inf_or_null);
    NGP_LAUNCHED("unproject_kernel");
    return 0;
}

int ngp_intrinsics_grad(const float* dx, const float* ts, const int32_t* rays_a, int64_t n_rays,
                        const int32_t* n_rays_dev, int64_t n_rows, const int64_t* pix_idxs, const int64_t* img_idxs,
                        const float* poses, const float* pose_corr_or_null, int64_t n_img, const float* cam_dirs,
                        int64_t W, int64_t H, int model, const double* params, const float* corr, float* grad_rays,
                        int64_t max_rays, int32_t* found_inf_or_null, void* stream) {
    const char* e = camera_error(model, params, W, H);
    NGP_REQUIRE(e == nullptr, e);
    NGP_REQUIRE(n_rays >= 0 && n_rows >= 0 && max_rays >= 0, "negative n_rays / n_rows / max_rays");
    NGP_REQUIRE(n_img > 0, "n_img must be > 0");
    NGP_REQUIRE(n_rays <= kMaxGradRays && max_rays <= kMaxGradRays, "n_rays and max_rays must be < 2^31");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && pix_idxs && img_idxs && poses && cam_dirs && corr && grad_rays, "null pointer");
    NGP_REQUIRE(n_rows == 0 || (dx && ts), "null pointer");
    NGP_REQUIRE(aligned16(corr) && aligned16(grad_rays) &&
                    (pose_corr_or_null == nullptr || aligned16(pose_corr_or_null)),
                "corrections and gradient rows must be 16-byte aligned");
    intrinsics_grad_kernel<<<(unsigned)((n_rays * 32 + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        dx, ts, rays_a, n_rays, n_rays_dev, n_rows, pix_idxs, img_idxs, poses, pose_corr_or_null, n_img, cam_dirs, W,
        H, to_camera(params), corr, reinterpret_cast<float4*>(grad_rays), max_rays, found_inf_or_null);
    NGP_LAUNCHED("intrinsics_grad_kernel");
    return 0;
}

int ngp_intrinsics_adam(float* corr, const float* grad_rays, int64_t n_rays, float* exp_avg, float* exp_avg_sq,
                        const int32_t* found_inf_or_null, const float* hyper_dev, float lr_ratio, float beta1,
                        float beta2, float eps, float* grad_out_or_null, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(n_rays <= kMaxGradRays, "n_rays must be < 2^31");
    NGP_REQUIRE(corr && exp_avg && exp_avg_sq && hyper_dev, "null pointer");
    NGP_REQUIRE(n_rays == 0 || grad_rays, "null pointer");
    NGP_REQUIRE(aligned16(corr) && aligned16(exp_avg) && aligned16(exp_avg_sq) &&
                    (grad_rays == nullptr || aligned16(grad_rays)) &&
                    (grad_out_or_null == nullptr || aligned16(grad_out_or_null)),
                "intrinsics buffers must be 16-byte aligned");
    NGP_REQUIRE(lr_ratio >= 0.0f && lr_ratio < INFINITY, "lr_ratio must be finite and >= 0");
    intrinsics_adam_kernel<<<1, kAdamThreads, 0, ngp::as_stream(stream)>>>(
        reinterpret_cast<float4*>(corr), reinterpret_cast<const float4*>(grad_rays), n_rays,
        reinterpret_cast<float4*>(exp_avg), reinterpret_cast<float4*>(exp_avg_sq), found_inf_or_null, hyper_dev,
        lr_ratio, beta1, beta2, eps, reinterpret_cast<float4*>(grad_out_or_null));
    NGP_LAUNCHED("intrinsics_adam_kernel");
    return 0;
}

}  // extern "C"
