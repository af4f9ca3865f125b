// errmap.cu — error-map ray sampling (--ray_sampling_strategy error_map, DESIGN.md §6j): training pixels are drawn in
// proportion to their tile's recent error, and each ray's loss is weighted so that the objective stays the uniform one
// in expectation.
//
// Image i (W x H) is cut into R x R tiles; pixel (x, y) lies in tile (ty, tx) = (floor(y R / H), floor(x R / W)), and the
// tiles of every image form one flat array of T = n_img R^2 (t = i R^2 + ty R + tx).  Tile t has n_t = rows(ty) cols(tx)
// pixels, rows(ty) = ceil((ty+1) H / R) - ceil(ty H / R) (>= 1 for R <= H), cols likewise.  All map state is integer:
//   E   [T] uint64  per-tile error, fixed point 2^30 (EMA of the per-ray errors)
//   acc [T] uint64  sum of u_r = floor(min(e_r, 3) 2^30) of this interval's rays, e_r = sum_c (pred_c - target_c)^2
//   cnt [T] uint32  number of those rays
//   C   [T] uint64  inclusive prefix sum of the masses m_t = n_t (E'_t + c); M = C[T-1] < 2^53
//
//   ngp_error_map_accumulate: acc[t] += u_r, cnt[t] += 1 (integer atomics: the result does not depend on their order).
//   ngp_error_map_rebuild:    E += (acc / cnt - E) >> s where cnt > 0; acc = cnt = 0; E' = E >> k with k the least shift
//                             such that max E' <= lim (lim from n_img W H and the floor, so that M < 2^53);
//                             c = max(1, ceil(p S / ((q - p) N_pix))), S = sum_t n_t E'_t, alpha = p / q; C = scan(m).
//   ngp_error_map_sample:     Philox4x32-10 (ray, ray >> 32, step, kErrMapCounterWord), key seed: v = floor(((r0 << 32)
//                             | r1) M / 2^64), t = first tile with C[t] > v, pixel j = floor(r2 n_t / 2^32) of the tile in
//                             row-major order, w = (float)((double)M n_t / ((double)N_pix m_t)).
//   ngp_ray_grad_weight:      every per-sample gradient of ray r times w_r (the ray's whole loss is scaled by w_r).
#include "common.cuh"
#include "philox.cuh"

namespace {

// the counter's last word separates this stream from the batch sampler's (0) and the random background's
constexpr uint32_t kErrMapCounterWord = 0x656d0001u;
constexpr int kFixedShift = 30;                  // u = floor(e 2^30)
constexpr float kErrMax = 3.0f;
constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;
constexpr int kWsHeader = 8;                     // workspace words before the per-block sums

// workspace header words
enum { kWsEmax = 0, kWsS = 1, kWsM = 2, kWsStatus = 3, kWsShift = 4, kWsC = 5 };

struct Geom {
    int64_t n_img, W, H, R;
};

__device__ __forceinline__ int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// first row (col) of tile ty (tx) along an axis of `len` pixels cut into R parts
__device__ __forceinline__ int64_t tile_lo(int64_t k, int64_t len, int64_t R) { return ceil_div(k * len, R); }

__device__ __forceinline__ uint64_t tile_pixels(const Geom& g, int64_t t) {
    const int64_t l = t % (g.R * g.R), ty = l / g.R, tx = l % g.R;
    const int64_t h = tile_lo(ty + 1, g.H, g.R) - tile_lo(ty, g.H, g.R);
    const int64_t w = tile_lo(tx + 1, g.W, g.R) - tile_lo(tx, g.W, g.R);
    return (uint64_t)(h * w);
}

__device__ __forceinline__ int64_t clamp64(int64_t v, int64_t hi) { return min(max(v, (int64_t)0), hi - 1); }

__device__ __forceinline__ int shift_for(uint64_t emax, uint64_t lim) {
    int k = 0;
    while ((emax >> k) > lim) ++k;
    return k;
}

// ---- sampling ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) error_map_sample_kernel(const uint64_t* __restrict__ cdf, Geom g, int64_t T,
                                                               uint64_t seed, const int32_t* __restrict__ step_dev,
                                                               int32_t step_host, int64_t* __restrict__ img_out,
                                                               int64_t* __restrict__ pix_out,
                                                               float* __restrict__ w_out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t step = (uint32_t)(step_dev ? *step_dev : step_host);
    const Philox4 r = philox4x32_10((uint32_t)i, (uint32_t)((uint64_t)i >> 32), step, kErrMapCounterWord,
                                    (uint32_t)seed, (uint32_t)(seed >> 32));
    const uint64_t M = cdf[T - 1];
    const uint64_t v = __umul64hi(((uint64_t)r.v[0] << 32) | r.v[1], M);   // in [0, M)
    // first t with C[t] > v
    int64_t lo = 0, hi = T - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (cdf[mid] > v) hi = mid;
        else lo = mid + 1;
    }
    const int64_t t = lo;
    const uint64_t m_t = cdf[t] - (t > 0 ? cdf[t - 1] : 0ull);
    const int64_t img = t / (g.R * g.R), l = t % (g.R * g.R), ty = l / g.R, tx = l % g.R;
    const int64_t y0 = tile_lo(ty, g.H, g.R), x0 = tile_lo(tx, g.W, g.R);
    const int64_t tw = tile_lo(tx + 1, g.W, g.R) - x0;
    const int64_t n_t = (tile_lo(ty + 1, g.H, g.R) - y0) * tw;
    const int64_t j = (int64_t)(((uint64_t)r.v[2] * (uint64_t)n_t) >> 32);
    img_out[i] = img;
    pix_out[i] = (y0 + j / tw) * g.W + x0 + j % tw;
    const double n_pix = (double)(g.n_img * g.W * g.H);
    w_out[i] = __double2float_rn(__ddiv_rn(__dmul_rn((double)M, (double)n_t), __dmul_rn(n_pix, (double)m_t)));
}

// ---- accumulation --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) error_map_accumulate_kernel(
    const float* __restrict__ pred, const float* __restrict__ target, const float* __restrict__ bg_rgb,
    const float* __restrict__ alpha, float b_load, const int64_t* __restrict__ img_idxs,
    const int64_t* __restrict__ pix_idxs, Geom g, unsigned long long* __restrict__ acc, unsigned* __restrict__ cnt,
    int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float e = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float t = target[i * 3 + c];
        if (bg_rgb != nullptr && alpha != nullptr)   // the random-background head's target: gt + (c_r - b_load)(1 - a)
            t = f_add(t, f_mul(f_sub(bg_rgb[i * 3 + c], b_load), f_sub(1.0f, alpha[i])));
        const float d = f_sub(pred[i * 3 + c], t);
        e = f_add(e, f_mul(d, d));
    }
    e = e < kErrMax ? e : kErrMax;   // NaN and inf count as the largest error
    const uint64_t u = (uint64_t)f_mul(e, (float)(1u << kFixedShift));
    const int64_t img = clamp64(img_idxs[i], g.n_img);
    const int64_t pix = clamp64(pix_idxs[i], g.W * g.H);
    const int64_t y = pix / g.W, x = pix % g.W;
    const int64_t t = img * g.R * g.R + (y * g.R / g.H) * g.R + x * g.R / g.W;
    atomicAdd(acc + t, (unsigned long long)u);
    atomicAdd(cnt + t, 1u);
}

// ---- rebuild -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) error_map_ema_kernel(uint64_t* __restrict__ E, uint64_t* __restrict__ acc,
                                                            unsigned* __restrict__ cnt, int shift, int64_t T,
                                                            unsigned long long* __restrict__ ws) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t e = 0;
    if (t < T) {
        e = E[t];
        const unsigned c = cnt[t];
        if (c > 0) {
            const int64_t d = (int64_t)(acc[t] / c) - (int64_t)e;
            e = (uint64_t)((int64_t)e + (d >> shift));   // arithmetic shift: floor(d / 2^s)
            E[t] = e;
            acc[t] = 0;
            cnt[t] = 0;
        }
    }
    // block max, then one atomic per block
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e = max(e, (uint64_t)__shfl_xor_sync(0xffffffffu, (unsigned long long)e, o));
    if ((threadIdx.x & 31) == 0 && e > 0) atomicMax(ws + kWsEmax, (unsigned long long)e);
}

__device__ __forceinline__ uint64_t block_sum_u64(uint64_t v) {
    __shared__ unsigned long long part[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, (unsigned long long)v, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    uint64_t s = 0;
    if (threadIdx.x == 0)
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += part[k];
    return s;   // valid in thread 0
}

__global__ void __launch_bounds__(256) error_map_sum_kernel(const uint64_t* __restrict__ E, Geom g, int64_t T,
                                                            uint64_t lim, unsigned long long* __restrict__ ws) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int k = shift_for(ws[kWsEmax], lim);
    const uint64_t v = t < T ? tile_pixels(g, t) * (E[t] >> k) : 0ull;
    const uint64_t s = block_sum_u64(v);
    if (threadIdx.x == 0) {
        if (s) atomicAdd(ws + kWsS, (unsigned long long)s);
        if (blockIdx.x == 0) ws[kWsShift] = (unsigned long long)k;
    }
}

struct MassCtx {
    int k;
    uint64_t c;
};

__device__ __forceinline__ MassCtx mass_ctx(const unsigned long long* ws, uint64_t lim, uint64_t n_pix, uint64_t p,
                                            uint64_t q) {
    MassCtx m;
    m.k = shift_for(ws[kWsEmax], lim);
    const uint64_t d = (q - p) * n_pix;
    const uint64_t c = (p * ws[kWsS] + d - 1) / d;   // p S < 2^63: S < 2^53 and p <= 1024
    m.c = c > 0 ? c : 1;
    return m;
}

// each thread: kScanItems consecutive tiles; masses summed per thread, then per block
__global__ void __launch_bounds__(kScanThreads) error_map_mass_blocks_kernel(const uint64_t* __restrict__ E, Geom g,
                                                                             int64_t T, uint64_t lim, uint64_t p,
                                                                             uint64_t q,
                                                                             unsigned long long* __restrict__ ws) {
    const MassCtx mc = mass_ctx(ws, lim, (uint64_t)(g.n_img * g.W * g.H), p, q);
    const int64_t t0 = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    uint64_t s = 0;
    for (int k = 0; k < kScanItems; ++k) {
        const int64_t t = t0 + k;
        if (t < T) s += tile_pixels(g, t) * ((E[t] >> mc.k) + mc.c);
    }
    s = block_sum_u64(s);
    if (threadIdx.x == 0) {
        ws[kWsHeader + blockIdx.x] = s;
        if (blockIdx.x == 0) ws[kWsC] = mc.c;
    }
}

// inclusive warp scan of uint64
__device__ __forceinline__ uint64_t warp_scan_u64(uint64_t v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t n = __shfl_up_sync(0xffffffffu, (unsigned long long)v, o);
        if (lane >= o) v += n;
    }
    return v;
}

// exclusive block scan of uint64 (blockDim.x = kScanThreads); returns (exclusive prefix, block total)
__device__ __forceinline__ uint64_t block_exclusive_scan_u64(uint64_t v, uint64_t& total) {
    __shared__ unsigned long long wsum[kScanThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t incl = warp_scan_u64(v, lane);
    if (lane == 31) wsum[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint64_t w = lane < kScanThreads / 32 ? wsum[lane] : 0ull;
        w = warp_scan_u64(w, lane);
        if (lane < kScanThreads / 32) wsum[lane] = w;
    }
    __syncthreads();
    total = wsum[kScanThreads / 32 - 1];
    const uint64_t r = incl - v + (wid > 0 ? wsum[wid - 1] : 0ull);
    __syncthreads();
    return r;
}

// one block: exclusive scan of the per-block sums in place, in rounds of kScanThreads with a carry
__global__ void __launch_bounds__(kScanThreads) error_map_scan_blocks_kernel(unsigned long long* __restrict__ ws,
                                                                             int64_t n_blocks) {
    unsigned long long* b = ws + kWsHeader;
    uint64_t carry = 0;
    for (int64_t base = 0; base < n_blocks; base += kScanThreads) {
        const int64_t k = base + threadIdx.x;
        const uint64_t v = k < n_blocks ? b[k] : 0ull;
        uint64_t total;
        const uint64_t ex = block_exclusive_scan_u64(v, total);
        if (k < n_blocks) b[k] = carry + ex;
        carry += total;
    }
}

__global__ void __launch_bounds__(kScanThreads) error_map_cdf_kernel(const uint64_t* __restrict__ E, Geom g, int64_t T,
                                                                     uint64_t lim, uint64_t p, uint64_t q,
                                                                     unsigned long long* __restrict__ ws,
                                                                     uint64_t* __restrict__ cdf) {
    const MassCtx mc = mass_ctx(ws, lim, (uint64_t)(g.n_img * g.W * g.H), p, q);
    const int64_t t0 = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    uint64_t m[kScanItems], s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int64_t t = t0 + k;
        m[k] = t < T ? tile_pixels(g, t) * ((E[t] >> mc.k) + mc.c) : 0ull;
        s += m[k];
    }
    uint64_t total;
    uint64_t run = ws[kWsHeader + blockIdx.x] + block_exclusive_scan_u64(s, total);
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
        const int64_t t = t0 + k;
        run += m[k];
        if (t < T) cdf[t] = run;
        if (t == T - 1) {
            ws[kWsM] = run;
            ws[kWsStatus] = run < (1ull << 53) ? 0ull : 1ull;   // never set when lim holds: see ngp_error_map_rebuild
        }
    }
}

// ---- gradient weights ----------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) ray_grad_weight_kernel(const int32_t* __restrict__ rays_a,
                                                              const float* __restrict__ w, float* __restrict__ dsig,
                                                              T* __restrict__ drgb, int32_t* __restrict__ found_inf,
                                                              int64_t n_rays, int64_t n_rows) {
    const int lane = threadIdx.x & 31;
    const int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (n >= n_rays) return;
    const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
    int64_t cnt = rays_a[n * 3 + 2];
    cnt = min(cnt, n_rows - start);   // never past the sample buffers
    if (cnt <= 0 || start < 0) return;
    const float wr = w[ray];
    bool bad = false;
    for (int64_t s = start + lane; s < start + cnt; s += 32) {
        const float a = __fmul_rn(dsig[s], wr);
        dsig[s] = a;
        bad |= !isfinite(a);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v = __fmul_rn(load_as_float(drgb, s * 3 + c), wr);
            store_from_float(drgb, s * 3 + c, v);
            bad |= !isfinite(load_as_float(drgb, s * 3 + c));   // the stored value: fp16 overflow included
        }
    }
    if (found_inf != nullptr && __any_sync(0xffffffffu, bad) && lane == 0) atomicExch(found_inf, 1);
}

bool geom_ok(int64_t n_img, int64_t W, int64_t H, int64_t R) {
    return n_img > 0 && W > 0 && H > 0 && R > 0 && R <= W && R <= H && n_img * W * H < (1ll << 40) &&
           n_img * R * R < (1ll << 31);
}

}  // namespace

extern "C" {

int64_t ngp_error_map_workspace_bytes(int64_t n_tiles) {
    if (n_tiles <= 0) return 0;
    return (int64_t)sizeof(uint64_t) * (kWsHeader + (n_tiles + kScanTile - 1) / kScanTile);
}

int ngp_error_map_sample(const uint64_t* cdf, int64_t n_img, int64_t W, int64_t H, int64_t R, uint64_t seed,
                         const int32_t* step_dev, int32_t step_host, int64_t* img_out, int64_t* pix_out, float* w_out,
                         int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(geom_ok(n_img, W, H, R), "bad map geometry (need 0 < R <= min(W, H), n_img W H < 2^40)");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(cdf && img_out && pix_out && w_out, "null pointer");
    error_map_sample_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        cdf, Geom{n_img, W, H, R}, n_img * R * R, seed, step_dev, step_host, img_out, pix_out, w_out, n_rays);
    NGP_LAUNCHED("error_map_sample_kernel");
    return 0;
}

int ngp_error_map_accumulate(const float* pred, const float* target, const float* bg_rgb, const float* alpha,
                             float b_load, const int64_t* img_idxs, const int64_t* pix_idxs, int64_t n_img, int64_t W,
                             int64_t H, int64_t R, uint64_t* acc, uint32_t* cnt, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(geom_ok(n_img, W, H, R), "bad map geometry (need 0 < R <= min(W, H), n_img W H < 2^40)");
    NGP_REQUIRE(bg_rgb || !alpha, "alpha is read with bg_rgb only");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(pred && target && img_idxs && pix_idxs && acc && cnt, "null pointer");
    error_map_accumulate_kernel<<<(unsigned)((n_rays + 255) / 256), 256, 0, ngp::as_stream(stream)>>>(
        pred, target, bg_rgb, alpha, b_load, img_idxs, pix_idxs, Geom{n_img, W, H, R},
        reinterpret_cast<unsigned long long*>(acc), cnt, n_rays);
    NGP_LAUNCHED("error_map_accumulate_kernel");
    return 0;
}

int ngp_error_map_rebuild(uint64_t* E, uint64_t* acc, uint32_t* cnt, uint64_t* cdf, int64_t n_img, int64_t W,
                          int64_t H, int64_t R, int ema_shift, int floor_num, int floor_den, void* workspace,
                          int64_t workspace_bytes, void* stream) {
    NGP_REQUIRE(geom_ok(n_img, W, H, R), "bad map geometry (need 0 < R <= min(W, H), n_img W H < 2^40)");
    NGP_REQUIRE(ema_shift >= 0 && ema_shift < 32, "ema_shift must be in [0, 32)");
    NGP_REQUIRE(floor_den >= 2 && floor_den <= 1024 && floor_num >= 1 && floor_num < floor_den,
                "floor must be num / den with 1 <= num < den <= 1024");
    NGP_REQUIRE(E && acc && cnt && cdf && workspace, "null pointer");
    const int64_t T = n_img * R * R;
    NGP_REQUIRE(workspace_bytes >= ngp_error_map_workspace_bytes(T), "workspace too small");
    // lim: the largest E' for which M = S + c N <= N E'max q / (q - p) + N stays below 2^53
    const unsigned __int128 N = (unsigned __int128)(n_img * W * H), p = (unsigned)floor_num, q = (unsigned)floor_den;
    const unsigned __int128 lim128 = ((q - p) * (((unsigned __int128)1 << 53) - N) - 1) / (N * q);
    NGP_REQUIRE(lim128 >= 1, "map too large: the CDF would not fit 53 bits");
    const uint64_t lim = lim128 > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)lim128;
    cudaStream_t st = ngp::as_stream(stream);
    auto* ws = static_cast<unsigned long long*>(workspace);
    const cudaError_t e = cudaMemsetAsync(ws, 0, kWsHeader * sizeof(uint64_t), st);
    if (e != cudaSuccess) {
        ngp::set_error("ngp_error_map_rebuild: %s", cudaGetErrorString(e));
        return (int)e;
    }
    const Geom g{n_img, W, H, R};
    const unsigned tb = (unsigned)((T + 255) / 256);
    const int64_t nb = (T + kScanTile - 1) / kScanTile;
    error_map_ema_kernel<<<tb, 256, 0, st>>>(E, acc, cnt, ema_shift, T, ws);
    NGP_LAUNCHED("error_map_ema_kernel");
    error_map_sum_kernel<<<tb, 256, 0, st>>>(E, g, T, lim, ws);
    NGP_LAUNCHED("error_map_sum_kernel");
    error_map_mass_blocks_kernel<<<(unsigned)nb, kScanThreads, 0, st>>>(E, g, T, lim, p, q, ws);
    NGP_LAUNCHED("error_map_mass_blocks_kernel");
    error_map_scan_blocks_kernel<<<1, kScanThreads, 0, st>>>(ws, nb);
    NGP_LAUNCHED("error_map_scan_blocks_kernel");
    error_map_cdf_kernel<<<(unsigned)nb, kScanThreads, 0, st>>>(E, g, T, lim, p, q, ws, cdf);
    NGP_LAUNCHED("error_map_cdf_kernel");
    return 0;
}

int ngp_ray_grad_weight(const int32_t* rays_a, const float* w, float* dL_dsigmas, void* dL_drgbs, int rgbs_dtype,
                        int32_t* found_inf_or_null, int64_t n_rays, int64_t n_rows, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && n_rows >= 0, "negative n_rays / n_rows");
    NGP_REQUIRE(rgbs_dtype == NGP_F32 || rgbs_dtype == NGP_F16, "bad dtype");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_a && w, "null pointer");
    NGP_REQUIRE(n_rows == 0 || (dL_dsigmas && dL_drgbs), "null pointer");
    const unsigned grid = (unsigned)((n_rays * 32 + 255) / 256);
    cudaStream_t st = ngp::as_stream(stream);
    if (rgbs_dtype == NGP_F16)
        ray_grad_weight_kernel<__half><<<grid, 256, 0, st>>>(rays_a, w, dL_dsigmas, (__half*)dL_drgbs,
                                                             found_inf_or_null, n_rays, n_rows);
    else
        ray_grad_weight_kernel<float><<<grid, 256, 0, st>>>(rays_a, w, dL_dsigmas, (float*)dL_drgbs,
                                                            found_inf_or_null, n_rays, n_rows);
    NGP_LAUNCHED("ray_grad_weight_kernel");
    return 0;
}

}  // extern "C"
