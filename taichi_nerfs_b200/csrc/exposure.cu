// exposure.cu — per-image exposure compensation (DESIGN.md §6k): a learned log2 gain e_i in R^3 for every training
// image, applied to the radiance of every sample of the image's rays, c' = 2^e_i * c (per channel).
//
// Exposures live in one fp32 buffer [n_img, 4] = (e_r, e_g, e_b, 0); the gradient and the two Adam moments have the
// same layout, so every row is one float4.  Gains are formed in fp64 (g = exp2((double)e)) and every product is rounded
// once to the row's dtype, so e = 0 gives g = 1 and c' = c, dL/dc = dL/dc' bit for bit.
//
//   ngp_exposure_apply: out[s] = g_img(ray) * rgbs[s] over each ray's rows (a separate buffer: the voxel backward
//                       re-reads rgbs for its sigmoid mask).
//   ngp_exposure_bwd:   per ray, G = ln2 * sum_s drgbs[s] * out[s] (drgbs = dL/dc', fp32 in a fixed order per ray), then
//                       drgbs[s] <- g * drgbs[s]; per image grad[i] += G over its rays (atomics).
//   ngp_exposure_adam:  one CTA: unscale, inf-skip, Adam, gradient zeroed, then e -= mean_i e per channel (fp64, fixed
//                       order).
#include "common.cuh"

namespace {

constexpr double kLn2 = 0.69314718055994530942;

// consecutive rays of one warp in the backward; their per-image sums are carried in registers between atomics (four, so
// that a batch of 8192 rays still gives 2048 warps)
constexpr int kExpRaysPerWarp = 4;
constexpr int kAdamThreads = 256;

__device__ __forceinline__ int64_t clamp_img(int64_t img, int64_t n_img) {
    return min(max(img, (int64_t)0), n_img - 1);
}

__device__ __forceinline__ int64_t row_bound(int64_t n_rows, const int32_t* n_rows_dev) {
    return n_rows_dev != nullptr ? min(n_rows, (int64_t)max(*n_rows_dev, 0)) : n_rows;
}

__device__ __forceinline__ void gains(const float* expo, int64_t img, double g[3]) {
    const float4 e = reinterpret_cast<const float4*>(expo)[img];
    g[0] = exp2((double)e.x);
    g[1] = exp2((double)e.y);
    g[2] = exp2((double)e.z);
}

template <typename T>
__device__ __forceinline__ void store_from_double(T* p, int64_t i, double v);
template <>
__device__ __forceinline__ void store_from_double<float>(float* p, int64_t i, double v) { p[i] = __double2float_rn(v); }
template <>
__device__ __forceinline__ void store_from_double<__half>(__half* p, int64_t i, double v) { p[i] = __double2half(v); }

// one warp per ray, lanes stride over its rows
template <typename T>
__global__ void __launch_bounds__(256) exposure_apply_kernel(const T* __restrict__ rgbs,
                                                             const int32_t* __restrict__ rays_a,
                                                             const int64_t* __restrict__ img_idxs,
                                                             const float* __restrict__ expo, int64_t n_img,
                                                             T* __restrict__ out, int64_t n_rays, int64_t n_rows,
                                                             const int32_t* __restrict__ n_rows_dev) {
    const int lane = threadIdx.x & 31;
    const int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (n >= n_rays) return;
    const int64_t rows = row_bound(n_rows, n_rows_dev);
    const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
    int64_t cnt = rays_a[n * 3 + 2];
    cnt = min(cnt, rows - start);   // never past the sample buffers
    if (cnt <= 0 || start < 0) return;
    double g[3];
    gains(expo, clamp_img(img_idxs[ray], n_img), g);
    for (int64_t s = start + lane; s < start + cnt; s += 32) {
#pragma unroll
        for (int c = 0; c < 3; ++c) store_from_double(out, s * 3 + c, g[c] * (double)load_as_float(rgbs, s * 3 + c));
    }
}

// kExpRaysPerWarp consecutive rays per warp.  Each ray's three sums are formed by the lanes and reduced with shuffles
// (a fixed order); consecutive rays of one image are summed in registers and reach grad as one atomicAdd per channel, so
// contributions of different warps to one image meet in the atomics, in no fixed order.
template <typename T>
__global__ void __launch_bounds__(256) exposure_bwd_kernel(const T* __restrict__ out, T* __restrict__ drgb,
                                                           const int32_t* __restrict__ rays_a,
                                                           const int64_t* __restrict__ img_idxs,
                                                           const float* __restrict__ expo, int64_t n_img,
                                                           float* __restrict__ grad, int32_t* __restrict__ found_inf,
                                                           int64_t n_rays, int64_t n_rows,
                                                           const int32_t* __restrict__ n_rows_dev) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t k0 = warp * kExpRaysPerWarp;
    if (k0 >= n_rays) return;
    const int64_t k1 = min(k0 + kExpRaysPerWarp, n_rays);
    const int64_t rows = row_bound(n_rows, n_rows_dev);
    int64_t cur = -1;   // image whose sums are being carried
    float acc[3] = {0.f, 0.f, 0.f};
    bool bad = false;
    auto flush = [&]() {
        if (cur >= 0 && lane < 3) atomicAdd(grad + cur * 4 + lane, lane == 0 ? acc[0] : lane == 1 ? acc[1] : acc[2]);
    };
    for (int64_t k = k0; k < k1; ++k) {
        const int64_t ray = rays_a[k * 3 + 0], start = rays_a[k * 3 + 1];
        int64_t cnt = rays_a[k * 3 + 2];
        cnt = min(cnt, rows - start);
        if (cnt <= 0 || start < 0) continue;
        const int64_t img = clamp_img(img_idxs[ray], n_img);
        double g[3];
        gains(expo, img, g);
        float sum[3] = {0.f, 0.f, 0.f};
        for (int64_t s = start + lane; s < start + cnt; s += 32) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float d = load_as_float(drgb, s * 3 + c);
                sum[c] = fmaf(d, load_as_float(out, s * 3 + c), sum[c]);
                store_from_double(drgb, s * 3 + c, g[c] * (double)d);
                bad |= !isfinite(load_as_float(drgb, s * 3 + c));   // the stored value: fp16 overflow included
            }
        }
        if (img != cur) {
            flush();
            cur = img;
            acc[0] = acc[1] = acc[2] = 0.f;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float r = (float)(kLn2 * (double)warp_sum(sum[c]));
            bad |= !isfinite(r);
            acc[c] += r;
        }
    }
    flush();
    if (found_inf != nullptr && __any_sync(0xffffffffu, bad) && lane == 0) atomicExch(found_inf, 1);
}

// Adam of ngp_adam_step_dyn (optim.cu, adam1), contractions spelled out the same way
__device__ __forceinline__ void exposure_adam1(float& p, float g, float& m, float& v, float lr_over_bc1, float bc2_sqrt,
                                               float beta1, float beta2, float eps, float inv_scale) {
    const float gg = __fmul_rn(g, inv_scale);
    m = __fmaf_rn(__fsub_rn(gg, m), 1.0f - beta1, m);
    v = __fmaf_rn(v, beta2, __fmul_rn(__fmul_rn(1.0f - beta2, gg), gg));
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), bc2_sqrt), eps);
    p = __fmaf_rn(-lr_over_bc1, __fdiv_rn(m, denom), p);
}

// One CTA.  Thread t owns images t, t + kAdamThreads, ...; its fp64 partial sums meet in a fixed tree, so the mean and
// the projected exposures do not depend on scheduling.
__global__ void __launch_bounds__(kAdamThreads) exposure_adam_kernel(float* __restrict__ expo, float* __restrict__ grad,
                                                                     float* __restrict__ exp_avg,
                                                                     float* __restrict__ exp_avg_sq,
                                                                     const int32_t* __restrict__ found_inf,
                                                                     const float* __restrict__ hyper, float lr_ratio,
                                                                     float beta1, float beta2, float eps,
                                                                     int64_t n_img) {
    __shared__ double red[3][kAdamThreads];
    const int t = threadIdx.x;
    const bool skip = found_inf != nullptr && *found_inf != 0;
    float4* P = reinterpret_cast<float4*>(expo);
    float4* G = reinterpret_cast<float4*>(grad);
    float4* M = reinterpret_cast<float4*>(exp_avg);
    float4* V = reinterpret_cast<float4*>(exp_avg_sq);
    const float lr = __fmul_rn(lr_ratio, hyper[0]), bc2 = hyper[1], inv = hyper[2];
    double s[3] = {0.0, 0.0, 0.0};
    for (int64_t i = t; i < n_img; i += kAdamThreads) {
        if (!skip) {
            float4 p = P[i], m = M[i], v = V[i];
            const float4 g = G[i];
            exposure_adam1(p.x, g.x, m.x, v.x, lr, bc2, beta1, beta2, eps, inv);
            exposure_adam1(p.y, g.y, m.y, v.y, lr, bc2, beta1, beta2, eps, inv);
            exposure_adam1(p.z, g.z, m.z, v.z, lr, bc2, beta1, beta2, eps, inv);
            P[i] = p;
            M[i] = m;
            V[i] = v;
            s[0] += (double)p.x;
            s[1] += (double)p.y;
            s[2] += (double)p.z;
        }
        G[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (skip) return;   // uniform over the CTA
#pragma unroll
    for (int c = 0; c < 3; ++c) red[c][t] = s[c];
    __syncthreads();
    for (int h = kAdamThreads / 2; h > 0; h >>= 1) {
        if (t < h)
#pragma unroll
            for (int c = 0; c < 3; ++c) red[c][t] += red[c][t + h];
        __syncthreads();
    }
    const double mean[3] = {red[0][0] / (double)n_img, red[1][0] / (double)n_img, red[2][0] / (double)n_img};
    for (int64_t i = t; i < n_img; i += kAdamThreads) {
        float4 p = P[i];
        p.x = __double2float_rn((double)p.x - mean[0]);
        p.y = __double2float_rn((double)p.y - mean[1]);
        p.z = __double2float_rn((double)p.z - mean[2]);
        P[i] = p;
    }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int ngp_exposure_apply(const void* rgbs, int rgbs_dtype, const int32_t* rays_a, const int64_t* img_idxs,
                       const float* expo, int64_t n_img, void* out, int64_t n_rays, int64_t n_rows,
                       const int32_t* n_rows_dev, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_rows >= 0, "negative n_rays / n_rows");
    NGP_REQUIRE(n_img > 0, "n_img must be > 0");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && img_idxs && expo, "null pointer");
    NGP_REQUIRE(n_rows == 0 || (rgbs && out), "null pointer");
    NGP_REQUIRE(aligned16(expo), "exposures must be 16-byte aligned");
    NGP_REQUIRE(rgbs != out || n_rows == 0, "out must not alias rgbs");
    const unsigned grid = (unsigned)((n_rays * 32 + 255) / 256);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        exposure_apply_kernel<__half><<<grid, 256, 0, st>>>((const __half*)rgbs, rays_a, img_idxs, expo, n_img,
                                                            (__half*)out, n_rays, n_rows, n_rows_dev);
    else
        exposure_apply_kernel<float><<<grid, 256, 0, st>>>((const float*)rgbs, rays_a, img_idxs, expo, n_img,
                                                           (float*)out, n_rays, n_rows, n_rows_dev);
    NGP_LAUNCHED("exposure_apply_kernel");
    return 0;
}

int ngp_exposure_bwd(const void* out, void* dL_drgbs, int rgbs_dtype, const int32_t* rays_a, const int64_t* img_idxs,
                     const float* expo, int64_t n_img, float* grad, int32_t* found_inf_or_null, int64_t n_rays,
                     int64_t n_rows, const int32_t* n_rows_dev, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_rows >= 0, "negative n_rays / n_rows");
    NGP_REQUIRE(n_img > 0, "n_img must be > 0");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && img_idxs && expo && grad, "null pointer");
    NGP_REQUIRE(n_rows == 0 || (out && dL_drgbs), "null pointer");
    NGP_REQUIRE(aligned16(expo), "exposures must be 16-byte aligned");
    const int64_t warps = (n_rays + kExpRaysPerWarp - 1) / kExpRaysPerWarp;
    const unsigned grid = (unsigned)((warps * 32 + 255) / 256);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        exposure_bwd_kernel<__half><<<grid, 256, 0, st>>>((const __half*)out, (__half*)dL_drgbs, rays_a, img_idxs,
                                                          expo, n_img, grad, found_inf_or_null, n_rays, n_rows,
                                                          n_rows_dev);
    else
        exposure_bwd_kernel<float><<<grid, 256, 0, st>>>((const float*)out, (float*)dL_drgbs, rays_a, img_idxs, expo,
                                                         n_img, grad, found_inf_or_null, n_rays, n_rows, n_rows_dev);
    NGP_LAUNCHED("exposure_bwd_kernel");
    return 0;
}

int ngp_exposure_adam(float* expo, float* grad, float* exp_avg, float* exp_avg_sq, const int32_t* found_inf_or_null,
                      const float* hyper_dev, float lr_ratio, float beta1, float beta2, float eps, int64_t n_img,
                      void* stream) {
    NGP_REQUIRE(n_img >= 0, "negative n_img");
    if (n_img == 0) return 0;
    NGP_REQUIRE(expo && grad && exp_avg && exp_avg_sq && hyper_dev, "null pointer");
    NGP_REQUIRE(aligned16(expo) && aligned16(grad) && aligned16(exp_avg) && aligned16(exp_avg_sq),
                "exposure buffers must be 16-byte aligned");
    NGP_REQUIRE(lr_ratio >= 0.0f && lr_ratio < INFINITY, "lr_ratio must be finite and >= 0");
    exposure_adam_kernel<<<1, kAdamThreads, 0, ngp::as_stream(stream)>>>(expo, grad, exp_avg, exp_avg_sq,
                                                                         found_inf_or_null, hyper_dev, lr_ratio,
                                                                         beta1, beta2, eps, n_img);
    NGP_LAUNCHED("exposure_adam_kernel");
    return 0;
}

}  // extern "C"
