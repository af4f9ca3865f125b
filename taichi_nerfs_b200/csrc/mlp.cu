// mlp.cu — the fused NGP MLP (sigma net 32->64->16, SH, rgb net 32->64->64->3) on the Hopper warpgroup tensor
// cores: wgmma.mma_async with fp32 accumulators in registers, one 64-sample tile per warpgroup (CTA) iteration.
//
// Replaces, in the reference, five torch.nn.Linear (cuBLAS) calls under torch.autocast(fp16) plus
// ~10 elementwise/cat/cast kernels: modules/networks.py:136-166 (NGP.density/forward), :369-380
// (MLP.forward), :18-30 (TruncExp) and modules/spherical_harmonics.py:16-42 (SH is fused into the
// rgb-net input stage).  Numerics follow autocast: fp16 operands, fp32 accumulate, every layer
// output rounded to fp16, TruncExp / direction normalisation / SH in fp32.
//
// Data layout.  Weights (9,408 fp16 = 18.4 KB, W5 zero-padded to 16 rows) stay resident in shared memory for the
// lifetime of the persistent CTA, in the no-swizzle core-matrix layout (8x8 fp16 core matrices of 128 contiguous
// bytes): the forward reads them K-major (D = X W^T), the backward reads the same copy MN-major (dX = dY W).
// Forward: only the embedding tile goes through shared memory (layer 1 is an SS MMA); every later layer takes its A
// operand from registers — the previous layer's accumulators, converted to fp16 pairs in place (wgmma.cuh).
// Backward: the dX chain runs the same way from registers; the weight gradients dW = dY^T X (M = 64, K = the tile's
// 64 samples) read both operands MN-major from shared-memory copies of the activations and accumulate in registers
// across all tiles of the persistent CTA, flushed once at the end with fp32 atomics.
#include "wgmma.cuh"

namespace {
using namespace ngp_wg;

constexpr int kThreads = 128;   // one warpgroup
constexpr int kB64 = kTile * 64 * 2;   // one [64 x 64] fp16 operand buffer
constexpr int kB32 = kTile * 32 * 2;
constexpr int kB16 = kTile * 16 * 2;

// forward: the embedding tile
constexpr int kX = kAct;
constexpr int kSmemFwd = kX + kB32;           // 24,576 B
// backward: the activations the weight-gradient MMAs read
constexpr int kE = kAct;                       // X = emb            [64 x 32]
constexpr int kH1 = kE + kB32;                 // relu(X W1^T)       [64 x 64]
constexpr int kX3 = kH1 + kB64;                // [SH | h]           [64 x 32]
constexpr int kH3 = kX3 + kB32;                // relu(X3 W3^T)      [64 x 64]
constexpr int kH4 = kH3 + kB64;                // relu(H3 W4^T)      [64 x 64]
constexpr int kDO = kH4 + kB64;                // dL/do (3 of 16)    [64 x 16]
constexpr int kDH4 = kDO + kB16;               // dL/dH4             [64 x 64]
constexpr int kDH3 = kDH4 + kB64;              // dL/dH3             [64 x 64]
constexpr int kDH = kDH3 + kB64;               // dL/dh              [64 x 16]
constexpr int kDH1 = kDH + kB16;               // dL/dH1             [64 x 64]
constexpr int kSmemBwd = kDH1 + kB64;          // 81,920 B

// activations saved by the forward for the backward (ngp_mlp_save_bytes): [n_max x 16] fp16 h = sigma-net output,
// then [n_max x 4] fp16 rgb (the sigmoid output, as torch's sigmoid backward keeps it)
__device__ __forceinline__ const __half* save_rgb_ptr(const __half* save, int64_t n_max) { return save + n_max * 16; }
__device__ __forceinline__ __half* save_rgb_ptr(__half* save, int64_t n_max) { return save + n_max * 16; }

__device__ __forceinline__ float r16(float x) { return __half2float(__float2half_rn(x)); }

// the two 16-byte chunks of embedding row `row` that thread half `q2` (0/1) stages
template <typename TEmb>
__device__ __forceinline__ void load_emb(const TEmb* __restrict__ emb, int64_t row, bool valid, int q2, uint4 e[2]) {
    e[0] = e[1] = make_uint4(0, 0, 0, 0);
    if (!valid) return;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const int kc = q2 * 2 + q;
        if constexpr (sizeof(TEmb) == 2) {
            e[q] = __ldg(reinterpret_cast<const uint4*>(emb + row * 32) + kc);
        } else {
            const float4 a = __ldg(reinterpret_cast<const float4*>(emb + row * 32 + kc * 8));
            const float4 b = __ldg(reinterpret_cast<const float4*>(emb + row * 32 + kc * 8 + 4));
            e[q] = make_uint4(pack_h2(a.x, a.y), pack_h2(a.z, a.w), pack_h2(b.x, b.y), pack_h2(b.z, b.w));
        }
    }
}

// ---- register fragments (wgmma.cuh): a thread holds rows r0 = 16*warp + lane/4 and r1 = r0 + 8, column pairs
// 2t, 2t+1 (+8, +16, ...) with t = lane % 4.  Fragment kk of a [64 x K] operand covers columns 16kk..16kk+15.
__device__ __forceinline__ void relu_frags(const float* d, int nk, uint32_t (*f)[4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
        if (kk < nk)
#pragma unroll
            for (int q = 0; q < 4; ++q) f[kk][q] = pack_h2_relu(d[8 * kk + 2 * q], d[8 * kk + 2 * q + 1]);
}
// fragment kk -> the shared-memory operand layout of a [64 x K] buffer
__device__ __forceinline__ void store_frag(uint8_t* buf, int K, int kk, const uint32_t f[4], int r0, int t) {
    *reinterpret_cast<uint32_t*>(buf + chunk_off(r0, 2 * kk, K) + 4 * t) = f[0];
    *reinterpret_cast<uint32_t*>(buf + chunk_off(r0 + 8, 2 * kk, K) + 4 * t) = f[1];
    *reinterpret_cast<uint32_t*>(buf + chunk_off(r0, 2 * kk + 1, K) + 4 * t) = f[2];
    *reinterpret_cast<uint32_t*>(buf + chunk_off(r0 + 8, 2 * kk + 1, K) + 4 * t) = f[3];
}
__device__ __forceinline__ uint32_t load_pair(const uint8_t* buf, int K, int row, int col) {
    return *reinterpret_cast<const uint32_t*>(buf + chunk_off(row, col >> 3, K) + (col & 7) * 2);
}
// backward hidden epilogue: fp16(D) masked by relu'(act) (act = the post-ReLU forward activation, a [64 x 64]
// buffer), as select semantics like threshold_backward -> fragments + the dst buffer.  threshold_backward zeroes the
// gradient where act <= 0, so a NaN activation passes it (unordered compare), as in torch
__device__ __forceinline__ void relu_bwd_frags(const float* d, const uint8_t* act, uint8_t* dst, int r0, int t,
                                               uint32_t (*f)[4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint32_t a = load_pair(act, 64, r0 + 8 * (q & 1), 16 * kk + 8 * (q >> 1) + 2 * t);
            f[kk][q] = pack_h2(d[8 * kk + 2 * q], d[8 * kk + 2 * q + 1]) &
                       __hgtu2_mask(*reinterpret_cast<const __half2*>(&a), __float2half2_rn(0.0f));
        }
        store_frag(dst, 64, kk, f[kk], r0, t);
    }
}
// fp16 pair (e[2t], e[2t+1]) of a 16-vector without dynamic register indexing
__device__ __forceinline__ uint32_t pick_pair(const float* e, int t) {
    float a = e[0], b = e[1];
#pragma unroll
    for (int c = 1; c < 4; ++c)
        if (t == c) {
            a = e[2 * c];
            b = e[2 * c + 1];
        }
    return pack_h2(a, b);
}
// X3 fragment 0: SH16((d/|d| + 1)/2) of rows r0 (d0) and r1 (d1)  (networks.py:162-164)
__device__ __forceinline__ void sh_frag(const float* d0, const float* d1, int t, uint32_t f[4]) {
    float e[16];
    float inv = 1.0f / sqrtf(d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2]);
    sh16((d0[0] * inv + 1.0f) / 2.0f, (d0[1] * inv + 1.0f) / 2.0f, (d0[2] * inv + 1.0f) / 2.0f, e);
    f[0] = pick_pair(e, t);
    f[2] = pick_pair(e + 8, t);
    inv = 1.0f / sqrtf(d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]);
    sh16((d1[0] * inv + 1.0f) / 2.0f, (d1[1] * inv + 1.0f) / 2.0f, (d1[2] * inv + 1.0f) / 2.0f, e);
    f[1] = pick_pair(e, t);
    f[3] = pick_pair(e + 8, t);
}
__device__ __forceinline__ void load_dir(const float* __restrict__ dirs, int64_t i, bool valid, float d[3]) {
    d[0] = 0.f; d[1] = 0.f; d[2] = 1.f;
    if (valid) {
        d[0] = __ldg(dirs + i * 3 + 0);
        d[1] = __ldg(dirs + i * 3 + 1);
        d[2] = __ldg(dirs + i * 3 + 2);
    }
}

// fp32 atomics of a [64 x N] accumulator into grad_w (dst(m, col) -> address, or null to skip); element 4j + 2k + c
// of a thread is (row r0 + 8k, column 8j + 2t + c)
template <int N, typename F>
__device__ __forceinline__ void flush_acc(const float* d, int r0, int t, bool& bad, F dst) {
#pragma unroll
    for (int e = 0; e < N / 2; ++e) {
        const int j = e >> 2, k = (e >> 1) & 1, c = e & 1;
        bad = bad || !(fabsf(d[e]) < INFINITY);
        if (float* p = dst(r0 + 8 * k, 8 * j + 2 * t + c)) atomicAdd(p, d[e]);
    }
}

// per-CTA occupancy of a kernel on the current device, for the persistent grid
template <typename K>
int ctas_per_sm(K kernel, int smem) {
    int b = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, kernel, kThreads, smem) != cudaSuccess || b < 1) {
        cudaGetLastError();
        b = 1;
    }
    return b;
}

template <typename TEmb>
__global__ void __launch_bounds__(kThreads, 3) mlp_fwd_kernel(const TEmb* __restrict__ emb, const float* __restrict__ dirs,
                                                           ngp_mlp_weights w, float* __restrict__ sigmas,
                                                           __half* __restrict__ rgbs, __half* __restrict__ save,
                                                           int64_t n_max, const int32_t* __restrict__ n_dev) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int64_t n = n_dev ? min(n_max, max((int64_t)*n_dev, (int64_t)0)) : n_max;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, t = lane & 3;
    const int r0 = 16 * warp + (lane >> 2), srow = tid >> 1, q2 = tid & 1;
    stage_weights(smem, w);
    const uint32_t aX = smem_u32(smem + kX), aW1 = smem_u32(smem + kW1), aW2 = smem_u32(smem + kW2),
                   aW3 = smem_u32(smem + kW3), aW4 = smem_u32(smem + kW4), aW5 = smem_u32(smem + kW5);

    const int64_t n_tiles = (n + kTile - 1) / kTile;
    uint4 cur[2];
    load_emb(emb, (int64_t)blockIdx.x * kTile + srow, (int64_t)blockIdx.x * kTile + srow < n, q2, cur);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        // ---- stage X = emb[tile rows] as fp16 (K = 32 layout); inputs were fetched one tile ago
        *reinterpret_cast<uint4*>(smem + kX + chunk_off(srow, 2 * q2, 32)) = cur[0];
        *reinterpret_cast<uint4*>(smem + kX + chunk_off(srow, 2 * q2 + 1, 32)) = cur[1];
        {
            const int64_t in = (tile + gridDim.x) * kTile + srow;
            load_emb(emb, in, in < n, q2, cur);
        }
        const int64_t i0 = tile * kTile + r0, i1 = i0 + 8;
        const bool v0 = i0 < n, v1 = i1 < n;
        float d0[3], d1[3];
        load_dir(dirs, i0, v0, d0);
        load_dir(dirs, i1, v1, d1);
        fence_proxy_async();
        __syncthreads();   // also orders the weight staging before the first tile

        // ---- layer 1: H1 = relu(X W1^T)                       [64x32]x[32x64]
        float acc[32];
        uint32_t f[4][4];
        wgmma_fence();
        wgmma_ss_n64<0, 0>(acc, desc_kmajor(aX, 32, 0), desc_kmajor(aW1, 32, 0), 0u);
        wgmma_ss_n64<0, 0>(acc, desc_kmajor(aX, 32, 1), desc_kmajor(aW1, 32, 1), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_frags(acc, 4, f);

        // ---- layer 2: h = H1 W2^T                             [64x64]x[64x16]
        float h[8];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n16<0>(h, f[kk], desc_kmajor(aW2, 64, kk), kk > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        // sigma = TruncExp(h[:,0]) (networks.py:22-24, :146); X3 = [SH | h]
        if (t == 0) {
            if (v0) sigmas[i0] = expf(r16(h[0]));
            if (v1) sigmas[i1] = expf(r16(h[2]));
        }
        uint32_t x3[2][4];
        sh_frag(d0, d1, t, x3[0]);
        x3[1][0] = pack_h2(h[0], h[1]);
        x3[1][1] = pack_h2(h[2], h[3]);
        x3[1][2] = pack_h2(h[4], h[5]);
        x3[1][3] = pack_h2(h[6], h[7]);
        if (save != nullptr) {   // the backward restarts from h instead of recomputing layers 1-2
            if (v0) {
                reinterpret_cast<uint32_t*>(save + i0 * 16)[t] = x3[1][0];
                reinterpret_cast<uint32_t*>(save + i0 * 16)[4 + t] = x3[1][2];
            }
            if (v1) {
                reinterpret_cast<uint32_t*>(save + i1 * 16)[t] = x3[1][1];
                reinterpret_cast<uint32_t*>(save + i1 * 16)[4 + t] = x3[1][3];
            }
        }

        // ---- layer 3: H3 = relu(X3 W3^T)                      [64x32]x[32x64]
        wgmma_fence();
        wgmma_rs_n64<0>(acc, x3[0], desc_kmajor(aW3, 32, 0), 0u);
        wgmma_rs_n64<0>(acc, x3[1], desc_kmajor(aW3, 32, 1), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_frags(acc, 4, f);

        // ---- layer 4: H4 = relu(H3 W4^T)                      [64x64]x[64x64]
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n64<0>(acc, f[kk], desc_kmajor(aW4, 64, kk), kk > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        relu_frags(acc, 4, f);

        // ---- layer 5: rgb = sigmoid(H4 W5^T)                  [64x64]x[64x8 (3 used)]
        float o[4];
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n8<0>(o, f[kk], desc_kmajor(aW5, 64, kk), kk > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        if (t < 2) {   // t = 0: channels 0, 1; t = 1: channel 2 (column 3 is padding)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const int64_t i = k ? i1 : i0;
                if (!(k ? v1 : v0)) continue;
                const __half a = __float2half_rn(1.0f / (1.0f + expf(-r16(o[2 * k]))));
                const __half b = __float2half_rn(1.0f / (1.0f + expf(-r16(o[2 * k + 1]))));
                rgbs[i * 3 + 2 * t] = a;
                if (t == 0) rgbs[i * 3 + 1] = b;
                if (save != nullptr) {
                    const __half2 p = __halves2half2(a, t == 0 ? b : __float2half_rn(0.0f));
                    reinterpret_cast<__half2*>(save_rgb_ptr(save, n_max) + i * 4)[t] = p;
                }
            }
        }
    }
}

// =====================================================================================================
// Backward.  Replaces the autograd graph of the five nn.Linear layers (cuBLAS dX + dW GEMMs), ReLU /
// Sigmoid / TruncExp backward (modules/networks.py:26-30) under autocast.  Per 64-sample tile:
//   1. recompute the forward activations (with saved activations, layers 2 and 5 are skipped: h and rgb are read);
//   2. chain  dO -> dH4 -> dH3 -> dX3 -> dh -> dH1 -> dE  with  dX = dY W  as RS MMAs whose B operand is the SAME
//      shared-memory weight copy read MN-major;
//   3. weight gradients  dW = dY^T X  as SS MMAs (both operands MN-major from shared memory) issued together with the
//      round's dX MMA, accumulated in registers across all tiles of the persistent CTA.
// Gradient operands of invalid (tail) rows are zero, so they do not contribute to dW.
template <typename TEmb, bool kSaved>
__global__ void __launch_bounds__(kThreads, 2) mlp_bwd_kernel(const TEmb* __restrict__ emb, const float* __restrict__ dirs,
                                                           ngp_mlp_weights w, const __half* __restrict__ save,
                                                           const float* __restrict__ dsigmas,
                                                           const __half* __restrict__ drgbs, TEmb* __restrict__ demb,
                                                           float* __restrict__ grad_w, int64_t n_max,
                                                           const int32_t* __restrict__ n_dev,
                                                           int32_t* __restrict__ found_inf) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int64_t n = n_dev ? min(n_max, max((int64_t)*n_dev, (int64_t)0)) : n_max;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, t = lane & 3;
    const int r0 = 16 * warp + (lane >> 2), srow = tid >> 1, q2 = tid & 1;
    stage_weights(smem, w);
    const uint32_t aW1 = smem_u32(smem + kW1), aW2 = smem_u32(smem + kW2), aW3 = smem_u32(smem + kW3),
                   aW4 = smem_u32(smem + kW4), aW5 = smem_u32(smem + kW5);
    const uint32_t aE = smem_u32(smem + kE), aH1 = smem_u32(smem + kH1), aX3 = smem_u32(smem + kX3),
                   aH3 = smem_u32(smem + kH3), aH4 = smem_u32(smem + kH4), aDO = smem_u32(smem + kDO),
                   aDH4 = smem_u32(smem + kDH4), aDH3 = smem_u32(smem + kDH3), aDH = smem_u32(smem + kDH),
                   aDH1 = smem_u32(smem + kDH1);

    // weight-gradient accumulators: dW4 [64 out x 64 in], dW3 / dW1 [64 out x 32 in], dW2^T [64 in x 16 out],
    // dW5^T [64 in x 8 (3 used)]
    float gW4[32], gW3[16], gW1[16], gW2T[8], gW5T[4];
#pragma unroll
    for (int j = 0; j < 32; ++j) gW4[j] = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) gW3[j] = gW1[j] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) gW2T[j] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) gW5T[j] = 0.f;

    bool bad = false;   // a non-finite dL/demb or weight gradient (GradScaler's inf check, raised at the source)
    const int64_t n_tiles = (n + kTile - 1) / kTile;
    uint4 cur[2];
    load_emb(emb, (int64_t)blockIdx.x * kTile + srow, (int64_t)blockIdx.x * kTile + srow < n, q2, cur);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        *reinterpret_cast<uint4*>(smem + kE + chunk_off(srow, 2 * q2, 32)) = cur[0];
        *reinterpret_cast<uint4*>(smem + kE + chunk_off(srow, 2 * q2 + 1, 32)) = cur[1];
        {
            const int64_t in = (tile + gridDim.x) * kTile + srow;
            load_emb(emb, in, in < n, q2, cur);
        }
        // this thread's two rows: directions, upstream gradients, saved activations
        int64_t ii[2];
        bool vv[2];
        float dd[2][3], dsig[2], dr[2][3];
        uint32_t hs[2][2] = {{0u, 0u}, {0u, 0u}};
        uint2 rgb_saved[2] = {make_uint2(0, 0), make_uint2(0, 0)};
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            ii[k] = tile * kTile + r0 + 8 * k;
            vv[k] = ii[k] < n;
            load_dir(dirs, ii[k], vv[k], dd[k]);
            dsig[k] = vv[k] ? __ldg(dsigmas + ii[k]) : 0.f;
#pragma unroll
            for (int c = 0; c < 3; ++c) dr[k][c] = vv[k] ? __half2float(drgbs[ii[k] * 3 + c]) : 0.f;
            if constexpr (kSaved) {
                if (vv[k]) {
                    hs[k][0] = __ldg(reinterpret_cast<const uint32_t*>(save + ii[k] * 16) + t);
                    hs[k][1] = __ldg(reinterpret_cast<const uint32_t*>(save + ii[k] * 16) + 4 + t);
                    rgb_saved[k] = __ldg(reinterpret_cast<const uint2*>(save_rgb_ptr(save, n_max) + ii[k] * 4));
                }
            }
        }
        fence_proxy_async();
        __syncthreads();

        // ================= forward recompute =================
        float acc[32], a32[16];
        uint32_t f[4][4];
        wgmma_fence();                                                   // H1 = relu(E W1^T)
        wgmma_ss_n64<0, 0>(acc, desc_kmajor(aE, 32, 0), desc_kmajor(aW1, 32, 0), 0u);
        wgmma_ss_n64<0, 0>(acc, desc_kmajor(aE, 32, 1), desc_kmajor(aW1, 32, 1), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_frags(acc, 4, f);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) store_frag(smem + kH1, 64, kk, f[kk], r0, t);
        uint32_t x3[2][4];
        float h0[2];
        if constexpr (kSaved) {   // X3 = [SH | h] straight from the saved h
            x3[1][0] = hs[0][0];
            x3[1][1] = hs[1][0];
            x3[1][2] = hs[0][1];
            x3[1][3] = hs[1][1];
            h0[0] = __low2float(*reinterpret_cast<const __half2*>(&hs[0][0]));
            h0[1] = __low2float(*reinterpret_cast<const __half2*>(&hs[1][0]));
        } else {
            float h[8];
            wgmma_fence();                                               // h = H1 W2^T
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_rs_n16<0>(h, f[kk], desc_kmajor(aW2, 64, kk), kk > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait_all();
            h0[0] = r16(h[0]);
            h0[1] = r16(h[2]);
            x3[1][0] = pack_h2(h[0], h[1]);
            x3[1][1] = pack_h2(h[2], h[3]);
            x3[1][2] = pack_h2(h[4], h[5]);
            x3[1][3] = pack_h2(h[6], h[7]);
        }
        sh_frag(dd[0], dd[1], t, x3[0]);
        store_frag(smem + kX3, 32, 0, x3[0], r0, t);
        store_frag(smem + kX3, 32, 1, x3[1], r0, t);
        wgmma_fence();                                                   // H3 = relu(X3 W3^T)
        wgmma_rs_n64<0>(acc, x3[0], desc_kmajor(aW3, 32, 0), 0u);
        wgmma_rs_n64<0>(acc, x3[1], desc_kmajor(aW3, 32, 1), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_frags(acc, 4, f);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) store_frag(smem + kH3, 64, kk, f[kk], r0, t);
        wgmma_fence();                                                   // H4 = relu(H3 W4^T)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n64<0>(acc, f[kk], desc_kmajor(aW4, 64, kk), kk > 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        relu_frags(acc, 4, f);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) store_frag(smem + kH4, 64, kk, f[kk], r0, t);
        // rgb of this thread's columns 2t, 2t+1 (t < 2; channel 3 is padding)
        float rgbv[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
        if constexpr (kSaved) {   // torch's sigmoid backward also uses the saved fp16 output
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const uint32_t p = t == 0 ? rgb_saved[k].x : rgb_saved[k].y;
                rgbv[k][0] = __low2float(*reinterpret_cast<const __half2*>(&p));
                rgbv[k][1] = __high2float(*reinterpret_cast<const __half2*>(&p));
            }
        } else {
            float o[4];
            wgmma_fence();                                               // o = H4 W5^T
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) wgmma_rs_n8<0>(o, f[kk], desc_kmajor(aW5, 64, kk), kk > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait_all();
#pragma unroll
            for (int k = 0; k < 2; ++k)
#pragma unroll
                for (int c = 0; c < 2; ++c) rgbv[k][c] = r16(1.0f / (1.0f + expf(-r16(o[2 * k + c]))));
        }
        // dL/do = dL/drgb * rgb (1 - rgb), rounded to fp16 like the autocast graph; columns 3..15 are zero
        uint32_t dof[4] = {0u, 0u, 0u, 0u};
        if (t < 2) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float g0 = t == 0 ? dr[k][0] : dr[k][2];
                const float g1 = t == 0 ? dr[k][1] : 0.f;
                dof[k] = pack_h2(g0 * rgbv[k][0] * (1.0f - rgbv[k][0]), g1 * rgbv[k][1] * (1.0f - rgbv[k][1]));
            }
        }
        store_frag(smem + kDO, 16, 0, dof, r0, t);
        fence_proxy_async();
        __syncthreads();

        // ================= backward =================
        // R1: dH4pre = dO W5 ;  dW5^T += H4^T dO
        wgmma_fence();
        wgmma_rs_n64<1>(acc, dof, desc_mnmajor(aW5, 64, 0), 0u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss_n8<1, 1>(gW5T, desc_mnmajor(aH4, 64, kk), desc_mnmajor(aDO, 16, kk), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_bwd_frags(acc, smem + kH4, smem + kDH4, r0, t, f);
        fence_proxy_async();
        __syncthreads();
        // R2: dH3pre = dH4 W4 ;  dW4 += dH4^T H3
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n64<1>(acc, f[kk], desc_mnmajor(aW4, 64, kk), kk > 0 ? 1u : 0u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss_n64<1, 1>(gW4, desc_mnmajor(aDH4, 64, kk), desc_mnmajor(aH3, 64, kk), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_bwd_frags(acc, smem + kH3, smem + kDH3, r0, t, f);
        fence_proxy_async();
        __syncthreads();
        // R3: dX3 = dH3 W3 ;  dW3 += dH3^T X3
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n32<1>(a32, f[kk], desc_mnmajor(aW3, 32, kk), kk > 0 ? 1u : 0u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss_n32<1, 1>(gW3, desc_mnmajor(aDH3, 64, kk), desc_mnmajor(aX3, 32, kk), 1u);
        wgmma_commit();
        wgmma_wait_all();
        // dh = dX3[:, 16:32] (+ TruncExp backward on h[:,0], networks.py:26-30), fp16
        if (t == 0) {
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const float ds = r16(dsig[k] * expf(fminf(fmaxf(h0[k], -15.0f), 15.0f)));
                a32[8 + 2 * k] = r16(a32[8 + 2 * k]) + ds;
            }
        }
        uint32_t dhf[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) dhf[q] = pack_h2(a32[8 + 2 * q], a32[9 + 2 * q]);
        store_frag(smem + kDH, 16, 0, dhf, r0, t);
        fence_proxy_async();
        __syncthreads();
        // R4: dH1pre = dh W2 ;  dW2^T += H1^T dh
        wgmma_fence();
        wgmma_rs_n64<1>(acc, dhf, desc_mnmajor(aW2, 64, 0), 0u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss_n16<1, 1>(gW2T, desc_mnmajor(aH1, 64, kk), desc_mnmajor(aDH, 16, kk), 1u);
        wgmma_commit();
        wgmma_wait_all();
        relu_bwd_frags(acc, smem + kH1, smem + kDH1, r0, t, f);
        fence_proxy_async();
        __syncthreads();
        // R5: dE = dH1 W1 ;  dW1 += dH1^T E
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_rs_n32<1>(a32, f[kk], desc_mnmajor(aW1, 32, kk), kk > 0 ? 1u : 0u);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_ss_n32<1, 1>(gW1, desc_mnmajor(aDH1, 64, kk), desc_mnmajor(aE, 32, kk), 1u);
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            if (!vv[k]) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float a = a32[4 * j + 2 * k], b = a32[4 * j + 2 * k + 1];
                const uint32_t p = pack_h2(a, b);
                bad = bad || (p & 0x7c00u) == 0x7c00u || (p & 0x7c000000u) == 0x7c000000u;   // fp16 inf / NaN
                if constexpr (sizeof(TEmb) == 2) {
                    *reinterpret_cast<uint32_t*>(demb + ii[k] * 32 + 8 * j + 2 * t) = p;
                } else {   // fp16-rounded like the autocast graph, stored as fp32
                    *reinterpret_cast<float2*>(demb + ii[k] * 32 + 8 * j + 2 * t) = make_float2(r16(a), r16(b));
                }
            }
        }
        __syncthreads();   // every buffer is restaged by the next tile
    }

    // ---- flush the weight-gradient accumulators: thread element 4j + 2k + c is (row r0 + 8k, column 8j + 2t + c)
    if ((int64_t)blockIdx.x >= n_tiles) return;
    constexpr int o2 = NGP_MLP_W1, o3 = o2 + NGP_MLP_W2, o4 = o3 + NGP_MLP_W3, o5 = o4 + NGP_MLP_W4;
    flush_acc<64>(gW4, r0, t, bad, [&](int m, int c) { return grad_w + o4 + m * 64 + c; });
    flush_acc<32>(gW3, r0, t, bad, [&](int m, int c) { return grad_w + o3 + m * 32 + c; });
    flush_acc<32>(gW1, r0, t, bad, [&](int m, int c) { return grad_w + m * 32 + c; });
    flush_acc<16>(gW2T, r0, t, bad, [&](int m, int c) { return grad_w + o2 + c * 64 + m; });   // W2 is [16 out x 64 in]
    // W5 is [3 out x 64 in]; columns 3..7 hold products with the zero padding of dO: finite unless dO is not
    flush_acc<8>(gW5T, r0, t, bad, [&](int m, int c) { return c < 3 ? grad_w + o5 + c * 64 + m : (float*)nullptr; });
    if (bad && found_inf != nullptr) *found_inf = 1;
}

template <typename TEmb, bool kSaved>
int launch_bwd(const void* emb, const float* dirs, const ngp_mlp_weights* w, const void* save, const float* dsigmas,
               const void* drgbs, void* demb, float* grad_w, int64_t n, const int32_t* n_dev, int32_t* found_inf,
               cudaStream_t st) {
    auto kernel = mlp_bwd_kernel<TEmb, kSaved>;
    static int per_sm[64] = {};   // set up once per device of this process
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (per_sm[dev] == 0) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBwd);
        if (e != cudaSuccess) {
            ngp::set_error("mlp_bwd_kernel: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
            return (int)e;
        }
        per_sm[dev] = ctas_per_sm(kernel, kSmemBwd);
    }
    const int64_t n_tiles = (n + kTile - 1) / kTile;
    const int64_t max_ctas = (int64_t)ngp::sm_count() * per_sm[dev];
    const unsigned grid = (unsigned)(n_tiles < max_ctas ? n_tiles : max_ctas);
    kernel<<<grid, kThreads, kSmemBwd, st>>>((const TEmb*)emb, dirs, *w, (const __half*)save, dsigmas,
                                             (const __half*)drgbs, (TEmb*)demb, grad_w, n, n_dev, found_inf);
    NGP_LAUNCHED("mlp_bwd_kernel");
    return 0;
}

template <typename TEmb>
int launch_fwd(const void* emb, const float* dirs, const ngp_mlp_weights* w, float* sigmas, void* rgbs, void* save,
               int64_t n, const int32_t* n_dev, cudaStream_t st) {
    auto kernel = mlp_fwd_kernel<TEmb>;
    static int per_sm[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (per_sm[dev] == 0) per_sm[dev] = ctas_per_sm(kernel, kSmemFwd);
    const int64_t n_tiles = (n + kTile - 1) / kTile;
    const int64_t max_ctas = (int64_t)ngp::sm_count() * per_sm[dev];
    const unsigned grid = (unsigned)(n_tiles < max_ctas ? n_tiles : max_ctas);
    kernel<<<grid, kThreads, kSmemFwd, st>>>((const TEmb*)emb, dirs, *w, sigmas, (__half*)rgbs, (__half*)save, n, n_dev);
    NGP_LAUNCHED("mlp_fwd_kernel");
    return 0;
}

}  // namespace

extern "C" {

int64_t ngp_mlp_save_bytes(int64_t n) {
    // [n x 16] fp16 h (sigma-net output) + [n x 4] fp16 rgb (3 used): with them the backward skips layers 2 and 5
    return n > 0 ? n * 40 : 0;
}

static int check_mlp_args(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w) {
    NGP_REQUIRE(emb_dtype == NGP_F32 || emb_dtype == NGP_F16, "bad dtype");
    NGP_REQUIRE(emb && dirs && w, "null pointer");
    NGP_REQUIRE(w->w1 && w->w2 && w->w3 && w->w4 && w->w5, "null weight pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(emb) & 15) == 0, "emb must be 16-byte aligned");
    const uintptr_t wal = reinterpret_cast<uintptr_t>(w->w1) | reinterpret_cast<uintptr_t>(w->w2) |
                          reinterpret_cast<uintptr_t>(w->w3) | reinterpret_cast<uintptr_t>(w->w4) |
                          reinterpret_cast<uintptr_t>(w->w5);
    NGP_REQUIRE((wal & 15) == 0, "weights must be 16-byte aligned");
    return 0;
}

int ngp_mlp_fwd(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w, float* sigmas,
                void* rgbs_f16, void* save, int64_t n, void* stream) {
    return ngp_mlp_fwd_dyn(emb, emb_dtype, dirs, w, sigmas, rgbs_f16, save, n, nullptr, stream);
}

int ngp_mlp_fwd_dyn(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w, float* sigmas,
                    void* rgbs_f16, void* save, int64_t n, const int32_t* n_dev, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    if (int rc = check_mlp_args(emb, emb_dtype, dirs, w)) return rc;
    NGP_REQUIRE(sigmas && rgbs_f16, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(save) & 15) == 0, "save must be 16-byte aligned");
    cudaStream_t st = ngp::as_stream(stream);
    if (emb_dtype == NGP_F16) return launch_fwd<__half>(emb, dirs, w, sigmas, rgbs_f16, save, n, n_dev, st);
    return launch_fwd<float>(emb, dirs, w, sigmas, rgbs_f16, save, n, n_dev, st);
}

int ngp_mlp_bwd(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w, const void* save,
                const float* dsigmas, const void* drgbs_f16, void* demb, float* grad_w, int64_t n, void* stream) {
    return ngp_mlp_bwd_dyn(emb, emb_dtype, dirs, w, save, dsigmas, drgbs_f16, demb, grad_w, n, nullptr, nullptr, stream);
}

int ngp_mlp_bwd_dyn(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w, const void* save,
                    const float* dsigmas, const void* drgbs_f16, void* demb, float* grad_w, int64_t n,
                    const int32_t* n_dev, int32_t* found_inf_or_null, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    if (int rc = check_mlp_args(emb, emb_dtype, dirs, w)) return rc;
    NGP_REQUIRE(dsigmas && drgbs_f16 && demb && grad_w, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(demb) & 15) == 0, "demb must be 16-byte aligned");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(save) & 15) == 0, "save must be 16-byte aligned");
    cudaStream_t st = ngp::as_stream(stream);
    if (emb_dtype == NGP_F16)
        return save ? launch_bwd<__half, true>(emb, dirs, w, save, dsigmas, drgbs_f16, demb, grad_w, n, n_dev, found_inf_or_null, st)
                    : launch_bwd<__half, false>(emb, dirs, w, save, dsigmas, drgbs_f16, demb, grad_w, n, n_dev, found_inf_or_null, st);
    return save ? launch_bwd<float, true>(emb, dirs, w, save, dsigmas, drgbs_f16, demb, grad_w, n, n_dev, found_inf_or_null, st)
                : launch_bwd<float, false>(emb, dirs, w, save, dsigmas, drgbs_f16, demb, grad_w, n, n_dev, found_inf_or_null, st);
}

}  // extern "C"
