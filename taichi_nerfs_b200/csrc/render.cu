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
template <typename T>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
ray_head_fused_kernel(const float* __restrict__ sigmas, const T* __restrict__ rgbs, const float* __restrict__ deltas,
                      const int32_t* __restrict__ rays_a, const float* __restrict__ gt, float bg, float coef,
                      const float* __restrict__ scale_dev, float thr, float* __restrict__ loss_sum,
                      float* __restrict__ opacity_out, float* __restrict__ rgb_out, float* __restrict__ dsigmas,
                      T* __restrict__ drgbs, int64_t n_rays) {
    __shared__ float Tstart_s[kWarpsPerBlock][kChunkCap];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t n = (int64_t)blockIdx.x * kWarpsPerBlock + wid;
    if (n >= n_rays) return;
    if (scale_dev != nullptr) coef *= *scale_dev;
    const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
    const int N = rays_a[n * 3 + 2];
    float* Tstart = Tstart_s[wid];

    // forward: colour / opacity sums, transmittance at every chunk start, last active chunk
    const int n_chunks = (N + 31) >> 5;
    int last_chunk = -1;
    float r = 0.f, g = 0.f, b = 0.f, op = 0.f;
    {
        float Tc = 1.0f;
        for (int c = 0; c < n_chunks; ++c) {
            const int k = c * 32 + lane;
            const bool valid = k < N;
            const int64_t s = start + k;
            float a = 0.f, c0 = 0.f, c1 = 0.f, c2 = 0.f;
            if (valid) {
                a = 1.0f - expf(-sigmas[s] * deltas[s]);
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
    const float keep = bg * (1.0f - op);
    const float d0 = r + keep - gt[ray * 3 + 0], d1 = g + keep - gt[ray * 3 + 1], d2 = b + keep - gt[ray * 3 + 2];
    const float gr = coef * d0, gg = coef * d1, gb = coef * d2;
    const float go = -bg * (gr + gg + gb);
    if (lane == 0) {
        atomicAdd(loss_sum, d0 * d0 + d1 * d1 + d2 * d2);
        if (opacity_out) opacity_out[ray] = op;
        if (rgb_out) {
            rgb_out[ray * 3 + 0] = r + keep;
            rgb_out[ray * 3 + 1] = g + keep;
            rgb_out[ray * 3 + 2] = b + keep;
        }
    }
    __syncwarp();

    // backward: exact reverse suffix accumulation (same as composite_train_bwd_kernel with g_depth = g_ws = 0)
    float suffix = 0.0f;
    for (int c = last_chunk; c >= 0; --c) {
        float Tc;
        if (c < kChunkCap) {
            Tc = Tstart[c];
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
        float a = 0.f, dl = 0.f, c0 = 0.f, c1 = 0.f, c2v = 0.f;
        if (valid) {
            dl = deltas[s];
            a = 1.0f - expf(-sigmas[s] * dl);
            c0 = load_as_float(rgbs, s * 3 + 0);
            c1 = load_as_float(rgbs, s * 3 + 1);
            c2v = load_as_float(rgbs, s * 3 + 2);
        }
        const float incl = warp_scan_mul(1.0f - a, lane);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.0f;
        const float Tb = Tc * excl;
        const bool active = valid && Tb > thr;
        const float w = active ? a * Tb : 0.0f;
        const float G = gr * c0 + gg * c1 + gb * c2v + go;
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
        ray_head_fused_kernel<__half><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const __half*)rgbs, deltas, rays_a, gt, bg, coef, scale_dev, T_threshold, loss_sum, opacity_out,
            rgb_out, dL_dsigmas, (__half*)dL_drgbs, n_rays);
    else
        ray_head_fused_kernel<float><<<grid, kWarpsPerBlock * 32, 0, st>>>(
            sigmas, (const float*)rgbs, deltas, rays_a, gt, bg, coef, scale_dev, T_threshold, loss_sum, opacity_out,
            rgb_out, dL_dsigmas, (float*)dL_drgbs, n_rays);
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
