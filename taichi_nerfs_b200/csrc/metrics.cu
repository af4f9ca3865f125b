// metrics.cu — test-time image metrics: SSIM over interleaved RGB images (DESIGN.md §6e).
//
// SSIM as torchmetrics' StructuralSimilarityIndexMeasure(data_range=1) defines it: Gaussian window sigma = 1.5 with
// 11 taps, k1 = 0.01, k2 = 0.03, the mean of the SSIM map over 3 channels x the (H-10) x (W-10) positions where the
// window lies inside the image (torchmetrics reflect-pads by 5 and crops 5 again, so the padding never reaches the
// mean).  Two launches, no atomics: ssim_rows_kernel writes one partial sum per (image, output row), ssim_mean_kernel
// sums each image's partials in a fixed order and divides, so the result is bit-reproducible.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kR = 5;                          // window radius
constexpr int kTaps = 2 * kR + 1;              // 11
constexpr int kTX = 96;                        // output columns per x-tile = threads per CTA
constexpr int kTY = 8;                         // output rows per CTA (its band)
constexpr int kInRows = kTY + 2 * kR;          // tile rows with the halo
constexpr int kInCols = (kTX + 2 * kR) * 3;    // interleaved floats per tile row
constexpr int kSumThreads = 256;
constexpr float kC1 = 1e-4f;                   // (k1 * data_range)^2
constexpr float kC2 = 9e-4f;                   // (k2 * data_range)^2

struct Window {
    float g[kTaps];
};

Window gaussian_window() {
    double e[kTaps], sum = 0.0;
    for (int i = 0; i < kTaps; ++i) {
        const double d = (i - kR) / 1.5;
        e[i] = exp(-0.5 * d * d);
        sum += e[i];
    }
    Window w;
    for (int i = 0; i < kTaps; ++i) w.g[i] = (float)(e[i] / sum);
    return w;
}

__device__ __forceinline__ float ssim_of(float mx, float my, float exx, float eyy, float exy) {
    const float mxx = mx * mx, myy = my * my, mxy = mx * my;
    const float vx = exx - mxx, vy = eyy - myy, cxy = exy - mxy;
    return ((2.0f * mxy + kC1) * (2.0f * cxy + kC2)) / ((mxx + myy + kC1) * (vx + vy + kC2));
}

// One CTA per (image, band of kTY output rows); it sweeps the band's x-tiles left to right.  Per tile the pred and
// target pixels of kInRows rows x (kTX + 10) columns go to shared memory as they lie in HBM (interleaved RGB).  Thread
// t owns output column t of the tile: per channel it runs the horizontal 11-tap pass of the five moments for each of
// the kInRows input rows and adds each result straight into the vertical sums of the kTY outputs that row reaches, so
// the vertical pass lives in registers.  row_sum[j] collects s over channels and tiles in a fixed order.
__global__ void __launch_bounds__(kTX) ssim_rows_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                        int H, int W, int n_bands, Window win,
                                                        float* __restrict__ partial) {
    __shared__ float sx[kInRows][kInCols];
    __shared__ float sy[kInRows][kInCols];
    __shared__ float red[kTY][kTX / 32];
    const int64_t img = blockIdx.x / n_bands;
    const int row0 = (int)(blockIdx.x - img * n_bands) * kTY;
    const int Ho = H - 2 * kR, Wo = W - 2 * kR;
    const int t = threadIdx.x;
    const int64_t base = img * H * W * 3;
    float row_sum[kTY];
#pragma unroll
    for (int j = 0; j < kTY; ++j) row_sum[j] = 0.0f;

    for (int col0 = 0; col0 < Wo; col0 += kTX) {
        __syncthreads();   // the previous tile's reads are done
        const int avail = min(kTX + 2 * kR, W - col0) * 3;
        for (int i = t; i < kInRows * kInCols; i += kTX) {
            const int r = i / kInCols, e = i - r * kInCols;
            float a = 0.0f, b = 0.0f;
            if (row0 + r < H && e < avail) {
                const int64_t off = base + ((int64_t)(row0 + r) * W + col0) * 3 + e;
                a = __ldg(pred + off);
                b = __ldg(target + off);
            }
            sx[r][e] = a;
            sy[r][e] = b;
        }
        __syncthreads();
        const bool col_ok = col0 + t < Wo;
        for (int ch = 0; ch < 3; ++ch) {
            float acc[kTY][5];
#pragma unroll
            for (int j = 0; j < kTY; ++j)
#pragma unroll
                for (int m = 0; m < 5; ++m) acc[j][m] = 0.0f;
#pragma unroll
            for (int i = 0; i < kInRows; ++i) {
                float hx = 0.0f, hy = 0.0f, hxx = 0.0f, hyy = 0.0f, hxy = 0.0f;
#pragma unroll
                for (int k = 0; k < kTaps; ++k) {
                    const float x = sx[i][(t + k) * 3 + ch], y = sy[i][(t + k) * 3 + ch];
                    const float gx = win.g[k] * x, gy = win.g[k] * y;
                    hx += gx;
                    hy += gy;
                    hxx += gx * x;
                    hyy += gy * y;
                    hxy += gx * y;
                }
#pragma unroll
                for (int j = 0; j < kTY; ++j) {
                    const int k = i - j;   // input row i is tap k of output row j
                    if (k >= 0 && k < kTaps) {
                        acc[j][0] += win.g[k] * hx;
                        acc[j][1] += win.g[k] * hy;
                        acc[j][2] += win.g[k] * hxx;
                        acc[j][3] += win.g[k] * hyy;
                        acc[j][4] += win.g[k] * hxy;
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < kTY; ++j) {
                const float s = ssim_of(acc[j][0], acc[j][1], acc[j][2], acc[j][3], acc[j][4]);
                row_sum[j] += (col_ok && row0 + j < Ho) ? s : 0.0f;   // a select: a masked NaN never enters
            }
        }
    }
    const int lane = t & 31, warp = t >> 5;
#pragma unroll
    for (int j = 0; j < kTY; ++j) {
        const float v = warp_sum(row_sum[j]);
        if (lane == 0) red[j][warp] = v;
    }
    __syncthreads();
    if (t < kTY && row0 + t < Ho) {
        float s = red[t][0];
#pragma unroll
        for (int w = 1; w < kTX / 32; ++w) s += red[t][w];
        partial[img * Ho + row0 + t] = s;
    }
}

// One CTA per image: thread t sums rows t, t + 256, ... in order, then a fixed-shape tree.
__global__ void __launch_bounds__(kSumThreads) ssim_mean_kernel(const float* __restrict__ partial, int Ho, int Wo,
                                                                float* __restrict__ out) {
    __shared__ float red[kSumThreads];
    const int64_t img = blockIdx.x;
    const int t = threadIdx.x;
    float s = 0.0f;
    for (int r = t; r < Ho; r += kSumThreads) s += partial[img * Ho + r];
    red[t] = s;
    __syncthreads();
#pragma unroll
    for (int h = kSumThreads / 2; h > 0; h >>= 1) {
        if (t < h) red[t] += red[t + h];
        __syncthreads();
    }
    if (t == 0) out[img] = (float)((double)red[0] / (3.0 * Ho * Wo));
}

}  // namespace

extern "C" {

int ngp_ssim(const float* pred, const float* target, int64_t n_images, int height, int width, float* partial,
             float* ssim_out, void* stream) {
    NGP_REQUIRE(n_images >= 0, "negative n_images");
    NGP_REQUIRE(height > 2 * kR && width > 2 * kR, "height and width must be >= 11 (the 11x11 window)");
    if (n_images == 0) return 0;
    NGP_REQUIRE(pred && target && partial && ssim_out, "null pointer");
    const int64_t n_bands = (height - 2 * kR + kTY - 1) / kTY;
    NGP_REQUIRE(n_images <= INT32_MAX / n_bands, "too many images for one launch");
    cudaStream_t st = ngp::as_stream(stream);
    ssim_rows_kernel<<<(unsigned)(n_images * n_bands), kTX, 0, st>>>(pred, target, height, width, (int)n_bands,
                                                                     gaussian_window(), partial);
    NGP_LAUNCHED("ssim_rows_kernel");
    ssim_mean_kernel<<<(unsigned)n_images, kSumThreads, 0, st>>>(partial, height - 2 * kR, width - 2 * kR, ssim_out);
    NGP_LAUNCHED("ssim_mean_kernel");
    return 0;
}

}  // extern "C"
