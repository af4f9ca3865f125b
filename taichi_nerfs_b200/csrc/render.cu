// render.cu — SH direction encoding and volume-rendering compositing (train fwd/bwd, test).
//
// Semantics: modules/spherical_harmonics.py:16-42, modules/volume_train.py:22-48 (+ its Taichi
// autodiff transpose, volume_train.py:160-173) and modules/volume_render_test.py:19-54.
//
// GPU mapping.  The reference composites with one thread per ray walking up to 1024 samples
// serially through a global T scratch array.  Here one WARP owns a ray: lanes take consecutive
// samples (coalesced 128-byte loads), transmittance is a warp prefix product carried across
// 32-sample chunks, early termination is a ballot, and the per-ray sums are shuffle reductions.
// Streaming work: HBM/L2-bandwidth bound, ~22 B/sample forward and ~36 B/sample backward.
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kChunkCap = 128;  // chunk-start transmittances kept in smem per warp (4096 samples)

// ---- a6: SH degree 4 ---------------------------------------------------------------------------
__device__ __forceinline__ void sh16(float x, float y, float z, float* e) {
    const float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
    e[0] = 0.28209479177387814f;
    e[1] = -0.48860251190291987f * y;
    e[2] = 0.48860251190291987f * z;
    e[3] = -0.48860251190291987f * x;
    e[4] = 1.0925484305920792f * xy;
    e[5] = -1.0925484305920792f * yz;
    e[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
    e[7] = -1.0925484305920792f * xz;
    e[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
    e[9] = 0.59004358992664352f * y * (-3.0f * x2 + y2);
    e[10] = 2.8906114426405538f * xy * z;
    e[11] = 0.45704579946446572f * y * (1.0f - 5.0f * z2);
    e[12] = 0.3731763325901154f * z * (5.0f * z2 - 3.0f);
    e[13] = 0.45704579946446572f * x * (1.0f - 5.0f * z2);
    e[14] = 1.4453057213202769f * z * (x2 - y2);
    e[15] = 0.59004358992664352f * x * (-x2 + 3.0f * y2);
}

__global__ void __launch_bounds__(256) dir_encode_kernel(const float* __restrict__ dirs, float* __restrict__ out,
                                                         int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float e[16];
    sh16(dirs[i * 3 + 0], dirs[i * 3 + 1], dirs[i * 3 + 2], e);
    float4* o = reinterpret_cast<float4*>(out + i * 16);
#pragma unroll
    for (int k = 0; k < 4; ++k) o[k] = make_float4(e[4 * k], e[4 * k + 1], e[4 * k + 2], e[4 * k + 3]);
}

// ---- a8 forward ---------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
composite_train_fwd_kernel(const float* __restrict__ sigmas, const T* __restrict__ rgbs,
                           const float* __restrict__ deltas, const float* __restrict__ ts,
                           const int32_t* __restrict__ rays_a, float thr, int32_t* __restrict__ total_samples,
                           float* __restrict__ opacity, float* __restrict__ depth, float* __restrict__ rgb,
                           float* __restrict__ ws, int64_t n_rays) {
    const int lane = threadIdx.x & 31;
    const int64_t n = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (n >= n_rays) return;
    const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
    const int N = rays_a[n * 3 + 2];

    float r = 0.f, g = 0.f, b = 0.f, dep = 0.f, op = 0.f;
    float Tc = 1.0f;  // transmittance at the start of the chunk
    int cnt = 0;
    bool alive = true;
    for (int base = 0; base < N; base += 32) {
        const int k = base + lane;
        const bool valid = k < N;
        const int64_t s = start + k;
        if (!alive) {  // after early termination: only the (defined) zero weights remain
            if (valid) ws[s] = 0.0f;
            continue;
        }
        float a = 0.0f, c0 = 0.f, c1 = 0.f, c2 = 0.f, tm = 0.f;
        if (valid) {
            a = 1.0f - expf(-sigmas[s] * deltas[s]);  // volume_train.py:39
            c0 = load_as_float(rgbs, s * 3 + 0);
            c1 = load_as_float(rgbs, s * 3 + 1);
            c2 = load_as_float(rgbs, s * 3 + 2);
            tm = ts[s];
        }
        const float incl = warp_scan_mul(1.0f - a, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.0f;
        const float Tb = Tc * excl;                 // T before this sample
        const bool active = valid && Tb > thr;      // volume_train.py:38
        const float w = active ? a * Tb : 0.0f;
        r += w * c0;
        g += w * c1;
        b += w * c2;
        dep += w * tm;
        op += w;
        if (valid) ws[s] = w;
        const unsigned act = __ballot_sync(0xffffffffu, active);
        const unsigned val = __ballot_sync(0xffffffffu, valid);
        cnt += __popc(act);
        if (act != val) alive = false;              // some valid sample fell below the threshold
        Tc = Tc * __shfl_sync(0xffffffffu, incl, 31);
    }
    r = warp_sum(r);
    g = warp_sum(g);
    b = warp_sum(b);
    dep = warp_sum(dep);
    op = warp_sum(op);
    if (lane == 0) {
        rgb[ray * 3 + 0] = r;
        rgb[ray * 3 + 1] = g;
        rgb[ray * 3 + 2] = b;
        depth[ray] = dep;
        opacity[ray] = op;
        total_samples[ray] = cnt;
    }
}

// ---- a8 backward ---------------------------------------------------------------------------------
// dL/drgbs[s] = w_s * dL/drgb ;  dL/dsigma[s] = delta_s * (T_{s+1} * G_s - sum_{j>s} w_j G_j)
// with G_j = dL/drgb . c_j + dL/ddepth * t_j + dL/dopacity + dL/dws_j  (active samples only).
template <typename T>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
composite_train_bwd_kernel(const float* __restrict__ gop, const float* __restrict__ gdep,
                           const float* __restrict__ grgb, const float* __restrict__ gws,
                           const float* __restrict__ sigmas, const T* __restrict__ rgbs,
                           const float* __restrict__ deltas, const float* __restrict__ ts,
                           const int32_t* __restrict__ rays_a, float thr, float* __restrict__ dsigmas,
                           T* __restrict__ drgbs, int64_t n_rays) {
    __shared__ float Tstart_s[kWarpsPerBlock][kChunkCap];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t n = (int64_t)blockIdx.x * kWarpsPerBlock + wid;
    if (n >= n_rays) return;
    const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
    const int N = rays_a[n * 3 + 2];
    const float gr = grgb[ray * 3 + 0], gg = grgb[ray * 3 + 1], gb = grgb[ray * 3 + 2];
    const float gd = gdep[ray], go = gop[ray];
    float* Tstart = Tstart_s[wid];

    // pass 1 (forward): transmittance at every chunk start, index of the last active chunk
    const int n_chunks = (N + 31) >> 5;
    int last_chunk = -1;
    {
        float Tc = 1.0f;
        for (int c = 0; c < n_chunks; ++c) {
            const int k = c * 32 + lane;
            const bool valid = k < N;
            const int64_t s = start + k;
            const float a = valid ? 1.0f - expf(-sigmas[s] * deltas[s]) : 0.0f;
            const float incl = warp_scan_mul(1.0f - a, lane);
            float excl = __shfl_up_sync(0xffffffffu, incl, 1);
            if (lane == 0) excl = 1.0f;
            const bool active = valid && Tc * excl > thr;
            const unsigned act = __ballot_sync(0xffffffffu, active);
            const unsigned val = __ballot_sync(0xffffffffu, valid);
            if (lane == 0 && c < kChunkCap) Tstart[c] = Tc;
            if (act) last_chunk = c;
            if (act != val) {  // terminated inside this chunk: zero the tail's gradients
                for (int c2 = c; c2 < n_chunks; ++c2) {
                    const int k2 = c2 * 32 + lane;
                    if (k2 < N && !(c2 == c && active)) {
                        const int64_t s2 = start + k2;
                        dsigmas[s2] = 0.0f;
                        store_from_float(drgbs, s2 * 3 + 0, 0.0f);
                        store_from_float(drgbs, s2 * 3 + 1, 0.0f);
                        store_from_float(drgbs, s2 * 3 + 2, 0.0f);
                    }
                }
                break;
            }
            Tc = Tc * __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    __syncwarp();

    // pass 2 (reverse over chunks): exact suffix accumulation
    float suffix = 0.0f;  // sum_{j in later chunks} w_j G_j
    for (int c = last_chunk; c >= 0; --c) {
        float Tc;
        if (c < kChunkCap) {
            Tc = Tstart[c];
        } else {  // rare: > 4096 samples on one ray — recompute the chunk start
            Tc = Tstart[kChunkCap - 1];
            for (int c2 = kChunkCap - 1; c2 < c; ++c2) {
                const int k2 = c2 * 32 + lane;
                const float a2 = k2 < N ? 1.0f - expf(-sigmas[start + k2] * deltas[start + k2]) : 0.0f;
                const float in2 = warp_scan_mul(1.0f - a2, lane);
                Tc = Tc * __shfl_sync(0xffffffffu, in2, 31);
            }
        }
        const int k = c * 32 + lane;
        const bool valid = k < N;
        const int64_t s = start + k;
        float a = 0.f, dl = 0.f, c0 = 0.f, c1 = 0.f, c2v = 0.f, tm = 0.f, gw = 0.f;
        if (valid) {
            dl = deltas[s];
            a = 1.0f - expf(-sigmas[s] * dl);
            c0 = load_as_float(rgbs, s * 3 + 0);
            c1 = load_as_float(rgbs, s * 3 + 1);
            c2v = load_as_float(rgbs, s * 3 + 2);
            tm = ts[s];
            gw = gws ? gws[s] : 0.0f;
        }
        const float incl = warp_scan_mul(1.0f - a, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.0f;
        const float Tb = Tc * excl;
        const bool active = valid && Tb > thr;
        const float w = active ? a * Tb : 0.0f;
        const float G = gr * c0 + gg * c1 + gb * c2v + gd * tm + go + gw;
        const float wG = w * G;
        // reverse inclusive scan of wG within the warp
        float rs = wG;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float nb = __shfl_down_sync(0xffffffffu, rs, o);
            if (lane + o < 32) rs += nb;
        }
        const float later = suffix + (rs - wG);  // sum over j > s
        if (active) {
            const float Tnext = Tb * (1.0f - a);
            dsigmas[s] = dl * (Tnext * G - later);
            store_from_float(drgbs, s * 3 + 0, w * gr);
            store_from_float(drgbs, s * 3 + 1, w * gg);
            store_from_float(drgbs, s * 3 + 2, w * gb);
        }
        suffix += __shfl_sync(0xffffffffu, rs, 0);
    }
}

// ---- a9 -----------------------------------------------------------------------------------------
template <typename TRgb>
__global__ void __launch_bounds__(256)
composite_test_kernel(const float* __restrict__ sigmas, const TRgb* __restrict__ rgbs, const float* __restrict__ deltas,
                      const float* __restrict__ ts, const int64_t* __restrict__ pack_info,
                      int64_t* __restrict__ alive_indices, float thr, float* __restrict__ opacity,
                      float* __restrict__ depth, float* __restrict__ rgb, int64_t n_alive) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int64_t start = pack_info[n * 2 + 0], steps = pack_info[n * 2 + 1];
    const int64_t ray = alive_indices[n];
    if (steps == 0) {  // volume_render_test.py:24-25
        alive_indices[n] = -1;
        return;
    }
    float T = 1.0f - opacity[ray];
    float r = 0.f, g = 0.f, b = 0.f, dep = 0.f, op = 0.f;
    for (int64_t k = 0; k < steps; ++k) {
        const int64_t s = start + k;
        const float a = 1.0f - expf(-sigmas[s] * deltas[s]);
        const float w = a * T;
        r += w * load_as_float(rgbs, s * 3 + 0);
        g += w * load_as_float(rgbs, s * 3 + 1);
        b += w * load_as_float(rgbs, s * 3 + 2);
        dep += w * ts[s];
        op += w;
        T *= 1.0f - a;
        if (T <= thr) {  // volume_render_test.py:46-48
            alive_indices[n] = -1;
            break;
        }
    }
    rgb[ray * 3 + 0] += r;
    rgb[ray * 3 + 1] += g;
    rgb[ray * 3 + 2] += b;
    depth[ray] += dep;
    opacity[ray] += op;
}

// ---- per-ray loss head ------------------------------------------------------------------------------------
// out = rgb + bg (1 - opacity) (rendering.py:219-226); loss = mean((out - gt)^2) (train.py:193);
// gradients of loss*loss_scale wrt the compositing outputs, in one launch instead of ~8 torch ops.
__global__ void __launch_bounds__(256) mse_loss_grad_kernel(const float* __restrict__ rgb, const float* __restrict__ opacity,
                                                            const float* __restrict__ gt, float bg, float coef,
                                                            const float* __restrict__ scale_dev,
                                                            float* __restrict__ loss_sum, float* __restrict__ g_rgb,
                                                            float* __restrict__ g_op, int64_t n_rays) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (scale_dev != nullptr) coef *= *scale_dev;  // coef was built with scale 1
    float sq = 0.f;
    if (r < n_rays) {
        const float keep = bg * (1.0f - opacity[r]);
        float gsum = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float diff = rgb[r * 3 + c] + keep - gt[r * 3 + c];
            sq += diff * diff;
            const float g = coef * diff;  // coef = loss_scale * 2 / (3 n_rays)
            g_rgb[r * 3 + c] = g;
            gsum += g;
        }
        g_op[r] = -bg * gsum;
    }
    sq = warp_sum(sq);
    if ((threadIdx.x & 31) == 0 && sq != 0.f) atomicAdd(loss_sum, sq);
}

// ---- fused per-ray head for the graph-captured step: composite forward + MSE loss + composite backward ------
// One warp per ray does what composite_train_fwd_kernel, mse_loss_grad_kernel and composite_train_bwd_kernel do
// in three launches: the ray's samples are read from HBM once (the reverse pass hits L1/L2), and the
// per-sample ws / per-ray depth that the loss does not need are never written.
//
// kDist adds the distortion loss w_d * mean(distortion) (distortion_fwd_kernel / distortion_bwd_kernel) to the same
// launch.  With W_<k, WT_<k the exclusive prefix sums of w and w t along the ray and W_>k, WT_>k the suffix sums:
//   loss_ray = sum_k w_k (2 (t_k W_<k - WT_<k) + w_k delta_k / 3)
//   dL/dw_k  = coef_d (2 (t_k W_<k - WT_<k) + 2 (WT_>k - t_k W_>k) + 2/3 w_k delta_k),  coef_d = scale w_d / n_rays
// and dL/dw_k joins G_k, as dL_dws does in composite_train_bwd_kernel.  The prefix carries at every chunk start sit in
// shared memory beside Tstart (the reverse pass rescans each chunk); the suffixes are accumulated by the reverse walk.
//
// kRandBg (--random_bg, DESIGN.md §6f): the background is the ray's own colour c_r = bg_rgb[ray] instead of the
// constant bg; where the image had an alpha channel (alpha != nullptr) the target's loader background b_load is swapped
// for c_r: gt' = gt + (c_r - b_load)(1 - a).  dL/dopacity = -sum_c c_r,c g_c.
//
// kDepth (--depth_loss_w, DESIGN.md §6h) adds w_z (1 / n_rays) sum_r v_r (D_r - D^_r)^2 with D_r = sum_k w_k t_k the
// ray's expected depth and D^_r = depth_gt[ray]; v_r = 1 where D^_r is finite and > 0, else 0.  Its dL/dD_r =
// coef_z v_r (D_r - D^_r), coef_z = scale 2 w_z / n_rays, enters G_k as dL_ddepth t_k does in
// composite_train_bwd_kernel.
template <typename T, bool kDist, bool kRandBg = false, bool kDepth = false>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
ray_head_fused_kernel(const float* __restrict__ sigmas, const T* __restrict__ rgbs, const float* __restrict__ deltas,
                      const float* __restrict__ ts, const int32_t* __restrict__ rays_a, const float* __restrict__ gt,
                      float bg, float coef, float coef_d, float w_d, const float* __restrict__ scale_dev, float thr,
                      float* __restrict__ loss_sum, float* __restrict__ opacity_out, float* __restrict__ rgb_out,
                      float* __restrict__ dsigmas, T* __restrict__ drgbs, int64_t n_rays,
                      const float* __restrict__ bg_rgb = nullptr, const float* __restrict__ alpha = nullptr,
                      float b_load = 0.0f, const float* __restrict__ depth_gt = nullptr, float coef_z = 0.0f,
                      float w_z = 0.0f) {
    __shared__ float Tstart_s[kWarpsPerBlock][kChunkCap];
    __shared__ float Wstart_s[kDist ? kWarpsPerBlock : 1][kDist ? kChunkCap : 1];   // W_<k at every chunk start
    __shared__ float WTstart_s[kDist ? kWarpsPerBlock : 1][kDist ? kChunkCap : 1];  // WT_<k at every chunk start
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t n = (int64_t)blockIdx.x * kWarpsPerBlock + wid;
    if (n >= n_rays) return;
    if (scale_dev != nullptr) {
        coef *= *scale_dev;
        if constexpr (kDist) coef_d *= *scale_dev;
        if constexpr (kDepth) coef_z *= *scale_dev;
    }
    const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
    const int N = rays_a[n * 3 + 2];
    float* Tstart = Tstart_s[wid];
    float* Wstart = Wstart_s[kDist ? wid : 0];
    float* WTstart = WTstart_s[kDist ? wid : 0];

    // forward: colour / opacity sums, transmittance at every chunk start, last active chunk
    const int n_chunks = (N + 31) >> 5;
    int last_chunk = -1;
    float r = 0.f, g = 0.f, b = 0.f, op = 0.f;
    float dist = 0.f;  // kDist: this lane's share of loss_ray
    float dep = 0.f;   // kDepth: this lane's share of D
    {
        float Tc = 1.0f;
        float Wc = 0.f, WTc = 0.f;  // kDist: W_<k, WT_<k at the chunk start
        for (int c = 0; c < n_chunks; ++c) {
            const int k = c * 32 + lane;
            const bool valid = k < N;
            const int64_t s = start + k;
            float a = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f, dl = 0.f, tm = 0.f;
            if (valid) {
                if constexpr (kDist) {
                    dl = deltas[s];
                    tm = ts[s];
                    a = 1.0f - expf(-sigmas[s] * dl);
                } else {
                    a = 1.0f - expf(-sigmas[s] * deltas[s]);
                    if constexpr (kDepth) tm = ts[s];
                }
                c0 = load_as_float(rgbs, s * 3 + 0);
                c1 = load_as_float(rgbs, s * 3 + 1);
                c2 = load_as_float(rgbs, s * 3 + 2);
            }
            const float incl = warp_scan_mul(1.0f - a, lane);
            float excl = __shfl_up_sync(0xffffffffu, incl, 1);
            if (lane == 0) excl = 1.0f;
            const float Tb = Tc * excl;
            const bool active = valid && Tb > thr;
            const float w = active ? a * Tb : 0.0f;
            r += w * c0;
            g += w * c1;
            b += w * c2;
            op += w;
            if constexpr (kDepth) dep += w * tm;
            if constexpr (kDist) {
                const float wt = w * tm;
                const float wi = warp_scan_add(w, lane), wti = warp_scan_add(wt, lane);
                float we = __shfl_up_sync(0xffffffffu, wi, 1), wte = __shfl_up_sync(0xffffffffu, wti, 1);
                if (lane == 0) we = wte = 0.0f;
                dist += w * (2.0f * (tm * (Wc + we) - (WTc + wte)) + (1.0f / 3.0f) * w * dl);
                if (lane == 0 && c < kChunkCap) {
                    Wstart[c] = Wc;
                    WTstart[c] = WTc;
                }
                Wc += __shfl_sync(0xffffffffu, wi, 31);
                WTc += __shfl_sync(0xffffffffu, wti, 31);
            }
            const unsigned act = __ballot_sync(0xffffffffu, active);
            const unsigned val = __ballot_sync(0xffffffffu, valid);
            if (lane == 0 && c < kChunkCap) Tstart[c] = Tc;
            if (act) last_chunk = c;
            if (act != val) {  // terminated inside this chunk: zero the tail's gradients
                for (int c2i = c; c2i < n_chunks; ++c2i) {
                    const int k2 = c2i * 32 + lane;
                    if (k2 < N && !(c2i == c && active)) {
                        const int64_t s2 = start + k2;
                        dsigmas[s2] = 0.0f;
                        store_from_float(drgbs, s2 * 3 + 0, 0.0f);
                        store_from_float(drgbs, s2 * 3 + 1, 0.0f);
                        store_from_float(drgbs, s2 * 3 + 2, 0.0f);
                    }
                }
                break;
            }
            Tc = Tc * __shfl_sync(0xffffffffu, incl, 31);
        }
    }
    r = warp_sum(r);
    g = warp_sum(g);
    b = warp_sum(b);
    op = warp_sum(op);
    // loss head (rendering.py:219-226, train.py:193)
    float k0, k1, k2, t0 = gt[ray * 3 + 0], t1 = gt[ray * 3 + 1], t2 = gt[ray * 3 + 2];
    float bc0 = bg, bc1 = bg, bc2 = bg;
    if constexpr (kRandBg) {
        bc0 = bg_rgb[ray * 3 + 0];
        bc1 = bg_rgb[ray * 3 + 1];
        bc2 = bg_rgb[ray * 3 + 2];
        const float t = 1.0f - op;
        k0 = bc0 * t;
        k1 = bc1 * t;
        k2 = bc2 * t;
        if (alpha != nullptr) {
            const float ta = 1.0f - alpha[ray];
            t0 += (bc0 - b_load) * ta;
            t1 += (bc1 - b_load) * ta;
            t2 += (bc2 - b_load) * ta;
        }
    } else {
        k0 = k1 = k2 = bg * (1.0f - op);
    }
    const float d0 = r + k0 - t0, d1 = g + k1 - t1, d2 = b + k2 - t2;
    const float gr = coef * d0, gg = coef * d1, gb = coef * d2;
    float go;
    if constexpr (kRandBg) go = -(bc0 * gr + bc1 * gg + bc2 * gb);
    else go = -bg * (gr + gg + gb);
    if constexpr (kDist) dist = warp_sum(dist);
    float gz = 0.f, lz = 0.f;  // kDepth: dL/dD (scaled) and v (D - D^)^2
    if constexpr (kDepth) {
        dep = warp_sum(dep);
        const float dh = depth_gt[ray];
        if (dh > 0.0f && dh < INFINITY) {  // NaN fails both
            const float dd = dep - dh;
            lz = dd * dd;
            gz = coef_z * dd;
        }
    }
    if (lane == 0) {
        // kDist: loss_sum / (3 n_rays) = mse + w_d mean(loss_ray); kDepth adds w_z mean(v (D - D^)^2)
        float l;
        if constexpr (kDist) l = d0 * d0 + d1 * d1 + d2 * d2 + 3.0f * w_d * dist;
        else l = d0 * d0 + d1 * d1 + d2 * d2;
        if constexpr (kDepth) l += 3.0f * w_z * lz;
        atomicAdd(loss_sum, l);
        if (opacity_out) opacity_out[ray] = op;
        if (rgb_out) {
            rgb_out[ray * 3 + 0] = r + k0;
            rgb_out[ray * 3 + 1] = g + k1;
            rgb_out[ray * 3 + 2] = b + k2;
        }
    }
    __syncwarp();

    // backward: exact reverse suffix accumulation (same as composite_train_bwd_kernel with g_depth = 0 or the depth
    // term, and g_ws = 0 or the distortion term)
    float suffix = 0.0f;
    float sW = 0.f, sWT = 0.f;  // kDist: sums of w and w t over the later chunks
    for (int c = last_chunk; c >= 0; --c) {
        float Tc, Wc = 0.f, WTc = 0.f;
        if (c < kChunkCap) {
            Tc = Tstart[c];
            if constexpr (kDist) {
                Wc = Wstart[c];
                WTc = WTstart[c];
            }
        } else if constexpr (kDist) {  // rare: > 4096 samples on one ray — redo the forward carries from the last kept
            Tc = Tstart[kChunkCap - 1];
            Wc = Wstart[kChunkCap - 1];
            WTc = WTstart[kChunkCap - 1];
            for (int c2i = kChunkCap - 1; c2i < c; ++c2i) {
                const int k2 = c2i * 32 + lane;
                const bool v2 = k2 < N;
                const float dl2 = v2 ? deltas[start + k2] : 0.0f;
                const float a2 = v2 ? 1.0f - expf(-sigmas[start + k2] * dl2) : 0.0f;
                const float in2 = warp_scan_mul(1.0f - a2, lane);
                float ex2 = __shfl_up_sync(0xffffffffu, in2, 1);
                if (lane == 0) ex2 = 1.0f;
                const float Tb2 = Tc * ex2;
                const float w2 = v2 && Tb2 > thr ? a2 * Tb2 : 0.0f;
                const float wt2 = w2 * (v2 ? ts[start + k2] : 0.0f);
                Wc += __shfl_sync(0xffffffffu, warp_scan_add(w2, lane), 31);
                WTc += __shfl_sync(0xffffffffu, warp_scan_add(wt2, lane), 31);
                Tc = Tc * __shfl_sync(0xffffffffu, in2, 31);
            }
        } else {
            Tc = Tstart[kChunkCap - 1];
            for (int c2i = kChunkCap - 1; c2i < c; ++c2i) {
                const int k2 = c2i * 32 + lane;
                const float a2 = k2 < N ? 1.0f - expf(-sigmas[start + k2] * deltas[start + k2]) : 0.0f;
                const float in2 = warp_scan_mul(1.0f - a2, lane);
                Tc = Tc * __shfl_sync(0xffffffffu, in2, 31);
            }
        }
        const int k = c * 32 + lane;
        const bool valid = k < N;
        const int64_t s = start + k;
        float a = 0.f, dl = 0.f, c0 = 0.f, c1 = 0.f, c2v = 0.f, tm = 0.f;
        if (valid) {
            dl = deltas[s];
            a = 1.0f - expf(-sigmas[s] * dl);
            c0 = load_as_float(rgbs, s * 3 + 0);
            c1 = load_as_float(rgbs, s * 3 + 1);
            c2v = load_as_float(rgbs, s * 3 + 2);
            if constexpr (kDist || kDepth) tm = ts[s];
        }
        const float incl = warp_scan_mul(1.0f - a, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.0f;
        const float Tb = Tc * excl;
        const bool active = valid && Tb > thr;
        const float w = active ? a * Tb : 0.0f;
        float G = gr * c0 + gg * c1 + gb * c2v + go;
        if constexpr (kDist) {
            const float wt = w * tm;
            // prefix W_<k, WT_<k: the forward's own scan, from the same carries
            const float wi = warp_scan_add(w, lane), wti = warp_scan_add(wt, lane);
            float we = __shfl_up_sync(0xffffffffu, wi, 1), wte = __shfl_up_sync(0xffffffffu, wti, 1);
            if (lane == 0) we = wte = 0.0f;
            // suffix W_>k, WT_>k: reverse inclusive scan inside the chunk, shifted down one lane, plus the later chunks
            float rw = w, rwt = wt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float nw = __shfl_down_sync(0xffffffffu, rw, o), nwt = __shfl_down_sync(0xffffffffu, rwt, o);
                if (lane + o < 32) {
                    rw += nw;
                    rwt += nwt;
                }
            }
            float lw = __shfl_down_sync(0xffffffffu, rw, 1), lwt = __shfl_down_sync(0xffffffffu, rwt, 1);
            if (lane == 31) lw = lwt = 0.0f;
            const float sel = tm * (Wc + we) - (WTc + wte);       // distortion.py:110; 0 at k = 0
            const float later_d = (sWT + lwt) - tm * (sW + lw);
            G += coef_d * (2.0f * (sel + later_d) + (2.0f / 3.0f) * w * dl);
            sW += __shfl_sync(0xffffffffu, rw, 0);
            sWT += __shfl_sync(0xffffffffu, rwt, 0);
        }
        if constexpr (kDepth) G += gz * tm;
        const float wG = w * G;
        float rs = wG;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float nb = __shfl_down_sync(0xffffffffu, rs, o);
            if (lane + o < 32) rs += nb;
        }
        const float later = suffix + (rs - wG);
        if (active) {
            dsigmas[s] = dl * (Tb * (1.0f - a) * G - later);
            store_from_float(drgbs, s * 3 + 0, w * gr);
            store_from_float(drgbs, s * 3 + 1, w * gg);
            store_from_float(drgbs, s * 3 + 2, w * gb);
        }
        suffix += __shfl_sync(0xffffffffu, rs, 0);
    }
}

// ---- distortion loss (Mip-NeRF 360), modules/distortion.py:15-119 -----------------------------------
// warp per ray; per-ray scans of w and w*t are warp prefix sums carried across 32-sample chunks
// (the reference's TODO at distortion.py:4-6 asks for exactly this shared/warp scan).
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
distortion_fwd_kernel(const float* __restrict__ ws, const float* __restrict__ deltas, const float* __restrict__ ts,
                      const int32_t* __restrict__ rays_a, float* __restrict__ loss, int64_t n_rays) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (i >= n_rays) return;
    const int64_t ray = rays_a[i * 3 + 0], start = rays_a[i * 3 + 1];
    const int N = rays_a[i * 3 + 2];
    float cw = 0.f, cwt = 0.f, acc = 0.f;  // carries = scans up to the previous chunk
    for (int base = 0; base < N; base += 32) {
        const int k = base + lane;
        const bool valid = k < N;
        const float w = valid ? ws[start + k] : 0.f;
        const float t = valid ? ts[start + k] : 0.f;
        const float d = valid ? deltas[start + k] : 0.f;
        const float wt = w * t;
        const float w_inc = cw + warp_scan_add(w, lane), wt_inc = cwt + warp_scan_add(wt, lane);
        const float w_exc = w_inc - w, wt_exc = wt_inc - wt;
        if (valid) acc += 2.f * (wt_inc * w_exc - w_inc * wt_exc) + (1.f / 3.f) * w * w * d;
        cw = __shfl_sync(0xffffffffu, w_inc, 31);
        cwt = __shfl_sync(0xffffffffu, wt_inc, 31);
    }
    acc = warp_sum(acc);
    if (lane == 0) loss[ray] = acc;
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
distortion_bwd_kernel(const float* __restrict__ dL_dloss, const float* __restrict__ ws,
                      const float* __restrict__ deltas, const float* __restrict__ ts,
                      const int32_t* __restrict__ rays_a, float* __restrict__ dL_dws, int64_t n_rays) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
    if (i >= n_rays) return;
    const int64_t ray = rays_a[i * 3 + 0], start = rays_a[i * 3 + 1];
    const int N = rays_a[i * 3 + 2];
    float w_sum = 0.f, wt_sum = 0.f;
    for (int k = lane; k < N; k += 32) {
        const float w = ws[start + k];
        w_sum += w;
        wt_sum += w * ts[start + k];
    }
    w_sum = warp_sum(w_sum);
    wt_sum = warp_sum(wt_sum);
    const float g = dL_dloss[ray];
    float cw = 0.f, cwt = 0.f;
    for (int base = 0; base < N; base += 32) {
        const int k = base + lane;
        const bool valid = k < N;
        const float w = valid ? ws[start + k] : 0.f;
        const float t = valid ? ts[start + k] : 0.f;
        const float wt = w * t;
        const float w_inc = cw + warp_scan_add(w, lane), wt_inc = cwt + warp_scan_add(wt, lane);
        const float w_exc = w_inc - w, wt_exc = wt_inc - wt;
        if (valid) {
            const float selector = k == 0 ? 0.f : t * w_exc - wt_exc;  // distortion.py:110
            float d = g * 2.f * (selector + (wt_sum - wt_inc - t * (w_sum - w_inc)));
            d += g * (2.f / 3.f) * w * deltas[start + k];
            dL_dws[start + k] = d;
        }
        cw = __shfl_sync(0xffffffffu, w_inc, 31);
        cwt = __shfl_sync(0xffffffffu, wt_inc, 31);
    }
}

// =====================================================================================================
// Compacting test-time renderer (replaces the host-driven loop of modules/rendering.py:96-144 and its re-ordering
// kernels; the reference's own device-side variant is deployment/InstantNGP/taichi_ngp/kernels.py:225-260).
// A frame is a fixed sequence of ROUNDS; each round = [bookkeeping] -> march (csrc/march.cu, kMode 3: persistent warps
// over the list of live rays, <= limit samples per ray, resume point kept per ray) -> hash encode -> MLP -> this
// kernel: composite the round's samples onto the per-ray accumulators (volume_render_test.py:19-54) and COMPACT the
// rays that are still alive (T > threshold and not out of the box) into the next round's list, one atomic per block.
// Nothing is read back by the host between rounds: the live count and the row count stay in `state`.
//   state[0] rows written by this round's march   state[2] live rays of this round   state[3] live rays of the next
//   state[4] samples evaluated so far             state[1], state[5..7] spare
constexpr int kRoundWarps = 8;

__global__ void frame_begin_kernel(const float* __restrict__ hits_t, float* __restrict__ t_cur,
                                   int32_t* __restrict__ n_marched, int32_t* __restrict__ alive,
                                   int32_t* __restrict__ state,
                                   float* __restrict__ opacity, float* __restrict__ depth, float* __restrict__ rgb,
                                   int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        state[0] = state[1] = 0;
        state[2] = 0;
        state[3] = (int32_t)n;     // becomes the live count at the first round_begin
        state[4] = 0;
    }
    if (i >= n) return;
    const float t1 = hits_t[i * 2 + 0];
    t_cur[i] = 0.0f < t1 ? t1 : -1.0f;     // ray_march.py:226 (strict 0 < t); rays that miss the box never emit
    n_marched[i] = 0;
    alive[i] = (int32_t)i;
    opacity[i] = 0.0f;
    depth[i] = 0.0f;
    rgb[i * 3 + 0] = rgb[i * 3 + 1] = rgb[i * 3 + 2] = 0.0f;
}

__global__ void frame_round_begin_kernel(int32_t* __restrict__ state) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    state[4] += state[0];
    state[0] = 0;
    state[2] = state[3];
    state[3] = 0;
}

// G lanes per ray (G = 4, 8, 16 or 32, >= the round's sample budget when that is small): a warp composites 32 / G rays
// at once, so the early rounds (a handful of samples for each of ~10^5..10^6 live rays) are not latency-bound on
// one-ray-per-warp chains.
template <typename T, int G>
__global__ void __launch_bounds__(kRoundWarps * 32)
composite_round_kernel(const float* __restrict__ sigmas, const T* __restrict__ rgbs, const float* __restrict__ deltas,
                       const float* __restrict__ ts, const int32_t* __restrict__ rays_a,
                       int32_t* __restrict__ state, const float* __restrict__ t_cur,
                       const float* __restrict__ hits_t, float thr, float* __restrict__ opacity,
                       float* __restrict__ depth, float* __restrict__ rgb, int32_t* __restrict__ next_alive) {
    constexpr int kPerWarp = 32 / G;
    __shared__ int32_t s_keep[kRoundWarps];
    __shared__ int32_t s_base;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gi = lane / G, sub = lane % G;
    const unsigned gmask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
    const int64_t n_alive = state[2];
    const int64_t per_block = (int64_t)kRoundWarps * kPerWarp;
    const int64_t n_iter = (n_alive + per_block - 1) / per_block;   // block-uniform trip count
    for (int64_t it = blockIdx.x; it < n_iter; it += gridDim.x) {
        const int64_t slot = (it * kRoundWarps + warp) * kPerWarp + gi;
        int32_t ray = -1;
        bool keep = false;
        if (slot < n_alive) {
            ray = rays_a[slot * 3 + 0];
            const int64_t start = rays_a[slot * 3 + 1];
            const int N = rays_a[slot * 3 + 2];
            float r = 0.f, g = 0.f, b = 0.f, dep = 0.f, op = 0.f;
            float Tc = 1.0f - opacity[ray];     // volume_render_test.py:30
            bool alive = true;
            for (int base = 0; base < N && alive; base += G) {
                const int k = base + sub;
                const bool valid = k < N;
                const int64_t s = start + k;
                float a = 0.0f, c0 = 0.f, c1 = 0.f, c2 = 0.f, tm = 0.f;
                if (valid) {
                    a = 1.0f - expf(-sigmas[s] * deltas[s]);
                    c0 = load_as_float(rgbs, s * 3 + 0);
                    c1 = load_as_float(rgbs, s * 3 + 1);
                    c2 = load_as_float(rgbs, s * 3 + 2);
                    tm = ts[s];
                }
                float incl = 1.0f - a;            // inclusive prefix product inside the group
#pragma unroll
                for (int o = 1; o < G; o <<= 1) {
                    const float nb = __shfl_up_sync(gmask, incl, o, G);
                    if (sub >= o) incl *= nb;
                }
                float excl = __shfl_up_sync(gmask, incl, 1, G);
                if (sub == 0) excl = 1.0f;
                const float Tb = Tc * excl;               // T before this sample
                const bool active = valid && Tb > thr;    // the loop breaks once T <= threshold (:47-49)
                const float w = active ? a * Tb : 0.0f;
                r += w * c0;
                g += w * c1;
                b += w * c2;
                dep += w * tm;
                op += w;
                const unsigned act = __ballot_sync(gmask, active) & gmask;
                const unsigned val = __ballot_sync(gmask, valid) & gmask;
                if (act != val) alive = false;
                Tc = Tc * __shfl_sync(gmask, incl, G - 1, G);
            }
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) {
                r += __shfl_xor_sync(gmask, r, o, G);
                g += __shfl_xor_sync(gmask, g, o, G);
                b += __shfl_xor_sync(gmask, b, o, G);
                dep += __shfl_xor_sync(gmask, dep, o, G);
                op += __shfl_xor_sync(gmask, op, o, G);
            }
            if (sub == 0 && N > 0) {
                rgb[ray * 3 + 0] += r;
                rgb[ray * 3 + 1] += g;
                rgb[ray * 3 + 2] += b;
                depth[ray] += dep;
                opacity[ray] += op;
            }
            // still alive: transmittance above the threshold and the march has not left the box (:51-52: a ray with
            // no samples left or T <= threshold gets alive_indices = -1)
            keep = alive && Tc > thr && t_cur[ray] < hits_t[(int64_t)ray * 2 + 1];
        }
        // block-level compaction of the live rays: one atomic per block
        const unsigned kept = __ballot_sync(0xffffffffu, keep && sub == 0);
        if (lane == 0) s_keep[warp] = __popc(kept);
        __syncthreads();
        if (threadIdx.x == 0) {
            int c = 0;
#pragma unroll
            for (int w = 0; w < kRoundWarps; ++w) c += s_keep[w];
            s_base = c ? atomicAdd(&state[3], c) : 0;
        }
        __syncthreads();
        if (keep && sub == 0) {
            int off = __popc(kept & ((1u << lane) - 1u));
            for (int w = 0; w < warp; ++w) off += s_keep[w];
            next_alive[s_base + off] = ray;
        }
        __syncthreads();
    }
}

}  // namespace

// ---- --random_bg: one background colour per training ray (DESIGN.md §6f) ------------------------------------------
// c_r = (unit(v0), unit(v1), unit(v2)) of Philox4x32-10 with counter (r, r >> 32, step, kBgCounterWord) and key
// (seed, seed >> 32).  The batch sampler (rays.cu) draws with counter word 0, so the two streams never share a counter.
constexpr uint32_t kBgCounterWord = 0x62670001u;

__device__ __forceinline__ void random_bg_colour(uint64_t seed, uint32_t step, int64_t r, float* out) {
    const Philox4 v = philox4x32_10((uint32_t)r, (uint32_t)((uint64_t)r >> 32), step, kBgCounterWord, (uint32_t)seed,
                                    (uint32_t)(seed >> 32));
    out[0] = philox_unit(v.v[0]);
    out[1] = philox_unit(v.v[1]);
    out[2] = philox_unit(v.v[2]);
}

__global__ void __launch_bounds__(256) random_bg_kernel(uint64_t seed, const int32_t* __restrict__ step_dev,
                                                        int32_t step_host, float* __restrict__ out, int64_t n) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    random_bg_colour(seed, (uint32_t)(step_dev ? *step_dev : step_host), r, out + r * 3);
}

extern "C" {

int ngp_mse_loss_grad(const float* rgb, const float* opacity, const float* gt, float bg, float loss_scale,
                      float* loss_sum, float* g_rgb, float* g_opacity, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rgb && opacity && gt && loss_sum && g_rgb && g_opacity, "null pointer");
    const float coef = loss_scale * 2.0f / (3.0f * (float)n_rays);
    mse_loss_grad_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        rgb, opacity, gt, bg, coef, nullptr, loss_sum, g_rgb, g_opacity, n_rays);
    NGP_LAUNCHED("mse_loss_grad_kernel");
    return 0;
}

int ngp_mse_loss_grad_dyn(const float* rgb, const float* opacity, const float* gt, float bg, const float* scale_dev,
                          float* loss_sum, float* g_rgb, float* g_opacity, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rgb && opacity && gt && loss_sum && g_rgb && g_opacity && scale_dev, "null pointer");
    const float coef = 2.0f / (3.0f * (float)n_rays);
    mse_loss_grad_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        rgb, opacity, gt, bg, coef, scale_dev, loss_sum, g_rgb, g_opacity, n_rays);
    NGP_LAUNCHED("mse_loss_grad_kernel");
    return 0;
}

int ngp_ray_head_fused(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas, const int32_t* rays_a,
                       const float* gt, float bg, float loss_scale, const float* scale_dev, float T_threshold,
                       float* loss_sum, float* opacity_out, float* rgb_out, float* dL_dsigmas, void* dL_drgbs,
                       int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(sigmas && rgbs && deltas && rays_a && gt && loss_sum && dL_dsigmas && dL_drgbs, "null pointer");
    const float coef = (scale_dev ? 1.0f : loss_scale) * 2.0f / (3.0f * (float)n_rays);
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        ray_head_fused_kernel<__half, false><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const __half*)rgbs, deltas, nullptr, rays_a, gt, bg, coef, 0.0f, 0.0f, scale_dev, T_threshold,
            loss_sum, opacity_out, rgb_out, dL_dsigmas, (__half*)dL_drgbs, n_rays);
    else
        ray_head_fused_kernel<float, false><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const float*)rgbs, deltas, nullptr, rays_a, gt, bg, coef, 0.0f, 0.0f, scale_dev, T_threshold,
            loss_sum, opacity_out, rgb_out, dL_dsigmas, (float*)dL_drgbs, n_rays);
    NGP_LAUNCHED("ray_head_fused_kernel");
    return 0;
}

int ngp_ray_head_fused_distortion(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas,
                                  const float* ts, const int32_t* rays_a, const float* gt, float bg, float loss_scale,
                                  const float* scale_dev, float T_threshold, float distortion_w, float* loss_sum,
                                  float* opacity_out, float* rgb_out, float* dL_dsigmas, void* dL_drgbs, int64_t n_rays,
                                  void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    NGP_REQUIRE(distortion_w >= 0.0f && distortion_w < INFINITY, "distortion_w must be finite and >= 0");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(sigmas && rgbs && deltas && ts && rays_a && gt && loss_sum && dL_dsigmas && dL_drgbs, "null pointer");
    const float scale = scale_dev ? 1.0f : loss_scale;
    const float coef = scale * 2.0f / (3.0f * (float)n_rays);
    const float coef_d = scale * distortion_w / (float)n_rays;   // d(w_d mean(loss_ray)) / d loss_ray, scaled
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        ray_head_fused_kernel<__half, true><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const __half*)rgbs, deltas, ts, rays_a, gt, bg, coef, coef_d, distortion_w, scale_dev,
            T_threshold, loss_sum, opacity_out, rgb_out, dL_dsigmas, (__half*)dL_drgbs, n_rays);
    else
        ray_head_fused_kernel<float, true><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const float*)rgbs, deltas, ts, rays_a, gt, bg, coef, coef_d, distortion_w, scale_dev,
            T_threshold, loss_sum, opacity_out, rgb_out, dL_dsigmas, (float*)dL_drgbs, n_rays);
    NGP_LAUNCHED("ray_head_fused_kernel");
    return 0;
}

int ngp_random_bg(uint64_t seed, const int32_t* step_dev, int32_t step_host, float* out, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(out, "null pointer");
    random_bg_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(seed, step_dev, step_host,
                                                                                          out, n_rays);
    NGP_LAUNCHED("random_bg_kernel");
    return 0;
}

int ngp_ray_head_fused_random_bg(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas,
                                 const float* ts, const int32_t* rays_a, const float* gt, const float* bg_rgb,
                                 const float* alpha, float b_load, float loss_scale, const float* scale_dev,
                                 float T_threshold, float distortion_w, float* loss_sum, float* opacity_out,
                                 float* rgb_out, float* dL_dsigmas, void* dL_drgbs, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    NGP_REQUIRE(distortion_w >= 0.0f && distortion_w < INFINITY, "distortion_w must be finite and >= 0");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(sigmas && rgbs && deltas && rays_a && gt && bg_rgb && loss_sum && dL_dsigmas && dL_drgbs,
                "null pointer");
    const bool dist = distortion_w > 0.0f;
    NGP_REQUIRE(!dist || ts, "null pointer (ts, needed by the distortion loss)");
    const float scale = scale_dev ? 1.0f : loss_scale;
    const float coef = scale * 2.0f / (3.0f * (float)n_rays);
    const float coef_d = scale * distortion_w / (float)n_rays;
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    cudaStream_t st = ngp::as_stream(stream);
#define NGP_HEAD_RBG(TT, DD)                                                                                        \
    ray_head_fused_kernel<TT, DD, true><<<grid, kWarpsPerBlock * 32, 0, st>>>(                                      \
        sigmas, (const TT*)rgbs, deltas, ts, rays_a, gt, 0.0f, coef, coef_d, distortion_w, scale_dev, T_threshold,   \
        loss_sum, opacity_out, rgb_out, dL_dsigmas, (TT*)dL_drgbs, n_rays, bg_rgb, alpha, b_load)
    if (rgbs_dtype == NGP_F16) {
        if (dist) NGP_HEAD_RBG(__half, true);
        else NGP_HEAD_RBG(__half, false);
    } else {
        if (dist) NGP_HEAD_RBG(float, true);
        else NGP_HEAD_RBG(float, false);
    }
#undef NGP_HEAD_RBG
    NGP_LAUNCHED("ray_head_fused_kernel");
    return 0;
}

int ngp_ray_head_fused_depth(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas, const float* ts,
                             const int32_t* rays_a, const float* gt, float bg, const float* bg_rgb, const float* alpha,
                             float b_load, float loss_scale, const float* scale_dev, float T_threshold,
                             float distortion_w, const float* depth_gt, float depth_w, float* loss_sum,
                             float* opacity_out, float* rgb_out, float* dL_dsigmas, void* dL_drgbs, int64_t n_rays,
                             void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    NGP_REQUIRE(distortion_w >= 0.0f && distortion_w < INFINITY, "distortion_w must be finite and >= 0");
    NGP_REQUIRE(depth_w >= 0.0f && depth_w < INFINITY, "depth_w must be finite and >= 0");
    NGP_REQUIRE(bg_rgb || !alpha, "alpha is read with bg_rgb only");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(sigmas && rgbs && deltas && ts && rays_a && gt && depth_gt && loss_sum && dL_dsigmas && dL_drgbs,
                "null pointer");
    const float scale = scale_dev ? 1.0f : loss_scale;
    const float coef = scale * 2.0f / (3.0f * (float)n_rays);
    const float coef_d = scale * distortion_w / (float)n_rays;
    const float coef_z = scale * 2.0f * depth_w / (float)n_rays;   // d(w_z mean(v (D - D^)^2)) / d(D - D^) / v
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    cudaStream_t st = ngp::as_stream(stream);
    // depth_w == 0 runs the depth-free instantiation: the result of ngp_ray_head_fused_{distortion,random_bg}
    const bool dist = distortion_w > 0.0f, rbg = bg_rgb != nullptr, depth = depth_w > 0.0f;
#define NGP_HEAD_Z(TT, DD, RB, ZZ)                                                                                  \
    ray_head_fused_kernel<TT, DD, RB, ZZ><<<grid, kWarpsPerBlock * 32, 0, st>>>(                                    \
        sigmas, (const TT*)rgbs, deltas, ts, rays_a, gt, RB ? 0.0f : bg, coef, coef_d, distortion_w, scale_dev,      \
        T_threshold, loss_sum, opacity_out, rgb_out, dL_dsigmas, (TT*)dL_drgbs, n_rays, bg_rgb, alpha, b_load,      \
        depth_gt, coef_z, depth_w)
#define NGP_HEAD_Z_RB(TT, DD, ZZ)        \
    if (rbg) NGP_HEAD_Z(TT, DD, true, ZZ); \
    else NGP_HEAD_Z(TT, DD, false, ZZ)
#define NGP_HEAD_Z_DD(TT, ZZ)                  \
    if (dist) { NGP_HEAD_Z_RB(TT, true, ZZ); } \
    else { NGP_HEAD_Z_RB(TT, false, ZZ); }
    if (rgbs_dtype == NGP_F16) {
        if (depth) { NGP_HEAD_Z_DD(__half, true) }
        else { NGP_HEAD_Z_DD(__half, false) }
    } else {
        if (depth) { NGP_HEAD_Z_DD(float, true) }
        else { NGP_HEAD_Z_DD(float, false) }
    }
#undef NGP_HEAD_Z_DD
#undef NGP_HEAD_Z_RB
#undef NGP_HEAD_Z
    NGP_LAUNCHED("ray_head_fused_kernel");
    return 0;
}

int ngp_distortion_fwd(const float* ws, const float* deltas, const float* ts, const int32_t* rays_a, float* loss,
                       int64_t n_rays, int64_t n_samples, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_samples >= 0, "negative size");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && loss && (n_samples == 0 || (ws && deltas && ts)), "null pointer");
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    distortion_fwd_kernel<<<grid, kWarpsPerBlock * 32, 0, ngp::as_stream(stream)>>>(ws, deltas, ts, rays_a, loss, n_rays);
    NGP_LAUNCHED("distortion_fwd_kernel");
    return 0;
}

int ngp_distortion_bwd(const float* dL_dloss, const float* ws, const float* deltas, const float* ts,
                       const int32_t* rays_a, float* dL_dws, int64_t n_rays, int64_t n_samples, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_samples >= 0, "negative size");
    if (n_rays == 0 || n_samples == 0) return 0;
    NGP_REQUIRE(dL_dloss && ws && deltas && ts && rays_a && dL_dws, "null pointer");
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    distortion_bwd_kernel<<<grid, kWarpsPerBlock * 32, 0, ngp::as_stream(stream)>>>(dL_dloss, ws, deltas, ts, rays_a,
                                                                                     dL_dws, n_rays);
    NGP_LAUNCHED("distortion_bwd_kernel");
    return 0;
}

int ngp_dir_encode(const float* dirs, float* out, int64_t n, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    NGP_REQUIRE(dirs && out, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "out must be 16-byte aligned");
    dir_encode_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(dirs, out, n);
    NGP_LAUNCHED("dir_encode_kernel");
    return 0;
}

int ngp_composite_train_fwd(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas,
                            const float* ts, const int32_t* rays_a, float T_threshold, int32_t* total_samples,
                            float* opacity, float* depth, float* rgb, float* ws, int64_t n_rays,
                            int64_t n_samples, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_samples >= 0, "negative size");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && total_samples && opacity && depth && rgb, "null pointer");
    NGP_REQUIRE(n_samples == 0 || (sigmas && rgbs && deltas && ts && ws), "null sample pointer");
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        composite_train_fwd_kernel<__half><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const __half*)rgbs, deltas, ts, rays_a, T_threshold, total_samples, opacity, depth, rgb, ws, n_rays);
    else
        composite_train_fwd_kernel<float><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const float*)rgbs, deltas, ts, rays_a, T_threshold, total_samples, opacity, depth, rgb, ws, n_rays);
    NGP_LAUNCHED("composite_train_fwd_kernel");
    return 0;
}

int ngp_composite_train_bwd(const float* dL_dopacity, const float* dL_ddepth, const float* dL_drgb,
                            const float* dL_dws, const float* sigmas, const void* rgbs, int rgbs_dtype,
                            const float* deltas, const float* ts, const int32_t* rays_a, const float* opacity,
                            const float* depth, const float* rgb, float T_threshold, float* dL_dsigmas,
                            void* dL_drgbs, int64_t n_rays, int64_t n_samples, void* stream) {
    (void)opacity; (void)depth; (void)rgb;
    NGP_REQUIRE(n_rays >= 0 && n_samples >= 0, "negative size");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_rays == 0 || n_samples == 0) return 0;
    NGP_REQUIRE(dL_dopacity && dL_ddepth && dL_drgb && sigmas && rgbs && deltas && ts && rays_a && dL_dsigmas &&
                    dL_drgbs,
                "null pointer");
    const unsigned grid = (unsigned)((n_rays + kWarpsPerBlock - 1) / kWarpsPerBlock);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        composite_train_bwd_kernel<__half><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            dL_dopacity, dL_ddepth, dL_drgb, dL_dws, sigmas, (const __half*)rgbs, deltas, ts, rays_a, T_threshold,
            dL_dsigmas, (__half*)dL_drgbs, n_rays);
    else
        composite_train_bwd_kernel<float><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            dL_dopacity, dL_ddepth, dL_drgb, dL_dws, sigmas, (const float*)rgbs, deltas, ts, rays_a, T_threshold,
            dL_dsigmas, (float*)dL_drgbs, n_rays);
    NGP_LAUNCHED("composite_train_bwd_kernel");
    return 0;
}

int ngp_composite_test(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas, const float* ts,
                       const int64_t* pack_info, int64_t* alive_indices, float T_threshold, float* opacity,
                       float* depth, float* rgb, int64_t n_alive, void* stream) {
    NGP_REQUIRE(n_alive >= 0, "negative n_alive");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_alive == 0) return 0;
    NGP_REQUIRE(pack_info && alive_indices && opacity && depth && rgb, "null pointer");
    const unsigned grid = (unsigned)((n_alive + 255) / 256);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        composite_test_kernel<__half><<<grid, 256, 0, st>>>(sigmas, (const __half*)rgbs, deltas, ts, pack_info,
                                                            alive_indices, T_threshold, opacity, depth, rgb, n_alive);
    else
        composite_test_kernel<float><<<grid, 256, 0, st>>>(sigmas, (const float*)rgbs, deltas, ts, pack_info,
                                                           alive_indices, T_threshold, opacity, depth, rgb, n_alive);
    NGP_LAUNCHED("composite_test_kernel");
    return 0;
}

int ngp_frame_begin(const float* hits_t, float* t_cur, int32_t* n_marched, int32_t* alive, int32_t* state,
                    float* opacity, float* depth, float* rgb, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 1 && n_rays < (1ll << 31), "n_rays out of range");
    NGP_REQUIRE(hits_t && t_cur && n_marched && alive && state && opacity && depth && rgb, "null pointer");
    frame_begin_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        hits_t, t_cur, n_marched, alive, state, opacity, depth, rgb, n_rays);
    NGP_LAUNCHED("frame_begin_kernel");
    return 0;
}

int ngp_frame_round_begin(int32_t* state, void* stream) {
    NGP_REQUIRE(state != nullptr, "null pointer");
    frame_round_begin_kernel<<<1, 32, 0, ngp::as_stream(stream)>>>(state);
    NGP_LAUNCHED("frame_round_begin_kernel");
    return 0;
}

int ngp_composite_round(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas, const float* ts,
                        const int32_t* rays_a, int32_t* state, const float* t_cur, const float* hits_t,
                        float T_threshold, float* opacity, float* depth, float* rgb, int32_t* next_alive,
                        int64_t n_rays, int limit, void* stream) {
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    NGP_REQUIRE(n_rays >= 1 && limit >= 1, "n_rays / limit out of range");
    NGP_REQUIRE(sigmas && rgbs && deltas && ts && rays_a && state && t_cur && hits_t && opacity && depth && rgb &&
                    next_alive, "null pointer");
    const int G = limit <= 4 ? 4 : limit <= 8 ? 8 : limit <= 16 ? 16 : 32;   // lanes per ray
    const int64_t per_block = (int64_t)kRoundWarps * (32 / G);
    const int64_t want = (n_rays + per_block - 1) / per_block;
    const int64_t cap_ctas = (int64_t)ngp::sm_count() * 8;
    const unsigned grid = (unsigned)(want < cap_ctas ? want : cap_ctas);
    cudaStream_t st = ngp::as_stream(stream);
#define NGP_CR(TT, GG)                                                                                              \
    composite_round_kernel<TT, GG><<<grid, kRoundWarps * 32, 0, st>>>(sigmas, (const TT*)rgbs, deltas, ts, rays_a, state, \
                                                                      t_cur, hits_t, T_threshold, opacity, depth, rgb,   \
                                                                      next_alive)
#define NGP_CR_G(TT)               \
    do {                           \
        if (G == 4) NGP_CR(TT, 4); \
        else if (G == 8) NGP_CR(TT, 8); \
        else if (G == 16) NGP_CR(TT, 16); \
        else NGP_CR(TT, 32);       \
    } while (0)
    if (rgbs_dtype == NGP_F16) NGP_CR_G(__half);
    else NGP_CR_G(float);
#undef NGP_CR_G
#undef NGP_CR
    NGP_LAUNCHED("composite_round_kernel");
    return 0;
}

}  // extern "C"
