// voxel.cu — the voxel-grid model (`--model_name svox`): trilinear spherical-harmonics field, forward (full and
// density-only, static and device-counted rows), field backward and the gradient of the total-variation and sparsity
// regularisers.
//
// Semantics (DESIGN.md §6d): the reference's VoxelGrid (modules/networks.py:382-575) with its missing parts decided
// here.  Node (i,j,k) of the G^3 lattice sits at ((i,j,k) - ceil(G/2) + 1) * radius (networks.py:450-466); a world
// point maps to u = (x - c_min) / radius (:521-522) and is interpolated trilinearly over the nodes floor(u) and
// floor(u)+1 of every axis.  A corner outside [0, G) contributes zero (the reference's out-of-grid mask, :489-508,
// :552).  sigma = ReLU(interpolated density); rgb_c = sigmoid(sum_k Y_k(d/|d|) * sh[c*D + k]) with the real SH basis
// of degree <= 2 in the PlenOctree convention (D = (deg+1)^2 coefficients per colour).
//
// Field layout: sh [G,G,G,3D] and density [G,G,G] fp32, node (i,j,k) at ((i*G + j)*G + k); every byte offset is
// int64 (at G = 256, deg 2 the sh field takes 1.81 GB, a larger G passes 2^31 bytes).
//
// GPU mapping, forward and backward: C = 3D + 1 consecutive lanes of a warp own one sample, lane ch = channel ch
// (sh channels 0..3D-1, density last), 32/C samples per warp (deg 2: 1, deg 1: 2, deg 0: 8).  A corner's channels
// are contiguous, so each of the 8 corner gathers (forward) or scatters (backward) is one warp instruction over
// 4*3D contiguous bytes plus the density float.  The backward needs no gather: the ReLU and sigmoid masks come from
// the forward's outputs (sigma > 0, rgb*(1-rgb)), which autograd saves anyway.  Rows of 3D floats (27 at deg 2) are
// not 16-byte aligned, so the scatter is scalar red.global.add.f32; the lanes of one instruction still cover whole
// sectors.  The thread-per-sample backward (one thread issues all 8*C reds of its sample) is kept behind
// `mapping` = NGP_VOXEL_BWD_THREAD so the two can be compared (scripts/bench_voxel_grid.py).
//
// Arithmetic is fp32 with explicit round-to-nearest intrinsics, and the density of a sample is summed over the
// corners in the same order by the full and the density-only kernel, so their sigma is bit-identical.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// Real SH basis, degrees 0..2 (the convention of PlenOctrees' eval_sh):
//   Y0 = 1/(2 sqrt(pi)); Y1..3 = sqrt(3)/(2 sqrt(pi)) * (-y, z, -x);
//   Y4..8 = sqrt(15)/(2 sqrt(pi)) * (xy, -yz), sqrt(5)/(4 sqrt(pi)) * (2zz - xx - yy), -sqrt(15)/(2 sqrt(pi)) * xz,
//           sqrt(15)/(4 sqrt(pi)) * (xx - yy)
constexpr float kY0 = 0.28209479177387814f;
constexpr float kY1 = 0.4886025119029199f;
constexpr float kY2a = 1.0925484305920792f;
constexpr float kY2b = 0.31539156525252005f;
constexpr float kY2c = 0.5462742152960396f;

__device__ __forceinline__ float sh_basis(int k, const float d[3]) {
    const float x = d[0], y = d[1], z = d[2];
    switch (k) {
        case 0: return kY0;
        case 1: return -kY1 * y;
        case 2: return kY1 * z;
        case 3: return -kY1 * x;
        case 4: return kY2a * (x * y);
        case 5: return -kY2a * (y * z);
        case 6: return kY2b * (2.0f * (z * z) - x * x - y * y);
        case 7: return -kY2a * (x * z);
        default: return kY2c * (x * x - y * y);
    }
}

// d / |d|.  A direction whose largest component lies outside [2^-40, 2^40] is first scaled by 2^90 or 2^-90, so that
// its squares neither underflow (subnormal components: 0/0) nor overflow (components ~1e30: x/inf = 0).  The scaling is
// exact unless a component more than 2^-50 times smaller than the largest underflows, which is below the fp32
// resolution of d / |d|.  Every other direction takes the unscaled formula, bit for bit.  A zero direction stays 0/0 = NaN, as in the fp64 model.
__device__ __forceinline__ void unit_dir(const float* dirs, int64_t i, float d[3]) {
    float a = dirs[i * 3], b = dirs[i * 3 + 1], c = dirs[i * 3 + 2];
    const float m = fmaxf(fabsf(a), fmaxf(fabsf(b), fabsf(c)));
    if (m > 0x1p40f || (m < 0x1p-40f && m > 0.0f)) {
        const float s = m > 0x1p40f ? 0x1p-90f : 0x1p90f;
        a = f_mul(a, s);
        b = f_mul(b, s);
        c = f_mul(c, s);
    }
    const float norm = sqrtf(f_add(f_add(f_mul(a, a), f_mul(b, b)), f_mul(c, c)));
    d[0] = f_div(a, norm);
    d[1] = f_div(b, norm);
    d[2] = f_div(c, norm);
}

// The cell of a sample: lower corner per axis and the fraction within the cell.  Positions whose lower corner lies
// outside [-1, G) — far away, infinite or NaN — get lo = -2, so both corners of that axis fall outside the grid and
// are masked without converting an out-of-range float to int.
struct Cell {
    int lo[3];
    float fr[3];
};

__device__ __forceinline__ Cell sample_cell(const ngp_voxel_layout& lay, const float* xyz, int64_t i) {
    Cell c;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float u = f_div(f_sub(xyz[i * 3 + k], lay.c_min), lay.radius);
        const float fl = floorf(u);
        c.fr[k] = f_sub(u, fl);
        c.lo[k] = (fl >= -1.0f && fl < (float)lay.grid) ? (int)fl : -2;
    }
    return c;
}

// Corner q: bit 2 -> x + 1, bit 1 -> y + 1, bit 0 -> z + 1 (z fastest, the memory order).  Returns the node index
// or -1 when the corner lies outside the grid; w = ((w_x * w_y) * w_z).
__device__ __forceinline__ int64_t corner(const ngp_voxel_layout& lay, const Cell& c, int q, float& w) {
    const int a = (q >> 2) & 1, b = (q >> 1) & 1, e = q & 1;
    const int ix = c.lo[0] + a, iy = c.lo[1] + b, iz = c.lo[2] + e;
    const float wx = a ? c.fr[0] : f_sub(1.0f, c.fr[0]);
    const float wy = b ? c.fr[1] : f_sub(1.0f, c.fr[1]);
    const float wz = e ? c.fr[2] : f_sub(1.0f, c.fr[2]);
    w = f_mul(f_mul(wx, wy), wz);
    const uint32_t G = (uint32_t)lay.grid;
    if ((uint32_t)ix >= G || (uint32_t)iy >= G || (uint32_t)iz >= G) return -1;
    return ((int64_t)ix * G + iy) * G + iz;
}

__device__ __forceinline__ int64_t rows(int64_t n_max, const int32_t* n_dev) {
    if (n_dev == nullptr) return n_max;
    const int64_t v = (int64_t)*n_dev;
    return v < n_max ? (v < 0 ? 0 : v) : n_max;
}

__device__ __forceinline__ float relu(float v) { return v > 0.0f ? v : 0.0f; }

__device__ __forceinline__ float sigmoid(float z) { return f_div(1.0f, f_add(1.0f, expf(-z))); }

// Non-finite test that survives fast-math style folding: false for +-inf and NaN.
__device__ __forceinline__ bool finite(float v) { return fabsf(v) < INFINITY; }

template <int DEG>
struct Lanes {
    static constexpr int D = (DEG + 1) * (DEG + 1);   // SH coefficients per colour
    static constexpr int C = 3 * D + 1;               // channels per node: 3D sh + density
    static constexpr int SPW = 32 / C;                 // samples per warp
    static constexpr int SPB = SPW * kWarps;           // samples per block
};

template <int DEG>
__global__ void __launch_bounds__(kThreads) voxel_fwd_kernel(const float* __restrict__ xyz,
                                                             const float* __restrict__ dirs,
                                                             const float* __restrict__ sh,
                                                             const float* __restrict__ density,
                                                             const ngp_voxel_layout lay, float* __restrict__ sigma,
                                                             float* __restrict__ rgb, int64_t n_max,
                                                             const int32_t* __restrict__ n_dev) {
    using Lx = Lanes<DEG>;
    __shared__ float part[kThreads];
    const int64_t n = rows(n_max, n_dev);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / Lx::C, ch = lane - sub * Lx::C;
    const int64_t i = (int64_t)blockIdx.x * Lx::SPB + warp * Lx::SPW + sub;
    const bool active = sub < Lx::SPW && i < n;
    float v = 0.0f;
    if (active) {
        const Cell c = sample_cell(lay, xyz, i);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float w;
            const int64_t node = corner(lay, c, q, w);
            if (node < 0) continue;
            const float f = ch < 3 * Lx::D ? __ldg(sh + node * (3 * Lx::D) + ch) : __ldg(density + node);
            v = f_add(v, f_mul(w, f));
        }
        if (ch < 3 * Lx::D) {
            float d[3];
            unit_dir(dirs, i, d);
            part[threadIdx.x] = f_mul(sh_basis(ch % Lx::D, d), v);
        }
    }
    __syncwarp();
    if (!active) return;
    if (ch < 3) {   // lanes 0..2 of the sample sum colour ch over its D coefficients, k ascending
        const float* p = part + (threadIdx.x - ch) + ch * Lx::D;
        float z = 0.0f;
#pragma unroll
        for (int k = 0; k < Lx::D; ++k) z = f_add(z, p[k]);
        rgb[i * 3 + ch] = sigmoid(z);
    }
    if (ch == 3 * Lx::D) sigma[i] = relu(v);
}

// sigma only (NGP.density / the occupancy-grid update): one thread per sample, the corners in the forward's order.
__global__ void __launch_bounds__(kThreads) voxel_density_kernel(const float* __restrict__ xyz,
                                                                 const float* __restrict__ density,
                                                                 const ngp_voxel_layout lay,
                                                                 float* __restrict__ sigma, int64_t n_max,
                                                                 const int32_t* __restrict__ n_dev) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= rows(n_max, n_dev)) return;
    const Cell c = sample_cell(lay, xyz, i);
    float v = 0.0f;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        float w;
        const int64_t node = corner(lay, c, q, w);
        if (node < 0) continue;
        v = f_add(v, f_mul(w, __ldg(density + node)));
    }
    sigma[i] = relu(v);
}

// dL/d(interpolated channel ch) of sample i: dL/drgb_c * rgb_c(1 - rgb_c) * Y_k for sh channel c*D + k, dL/dsigma
// where sigma > 0 for the density.
template <int DEG>
__device__ __forceinline__ float channel_grad(int ch, int64_t i, const float* dirs, const float* sigma,
                                              const float* rgb, const float* dsigma, const float* drgb) {
    constexpr int D = Lanes<DEG>::D;
    if (ch == 3 * D) return sigma[i] > 0.0f ? dsigma[i] : 0.0f;
    const int col = ch / D;
    const float s = rgb[i * 3 + col];
    const float g = drgb[i * 3 + col] * f_mul(s, f_sub(1.0f, s));
    float d[3];
    unit_dir(dirs, i, d);
    return g * sh_basis(ch % D, d);
}

__device__ __forceinline__ float* channel_dst(float* dsh, float* ddensity, int64_t node, int ch, int D) {
    return ch < 3 * D ? dsh + node * (3 * D) + ch : ddensity + node;
}

template <int DEG>
__global__ void __launch_bounds__(kThreads) voxel_bwd_warp_kernel(
    const float* __restrict__ xyz, const float* __restrict__ dirs, const float* __restrict__ sigma,
    const float* __restrict__ rgb, const float* __restrict__ dsigma, const float* __restrict__ drgb,
    const ngp_voxel_layout lay, float* __restrict__ dsh, float* __restrict__ ddensity, int64_t n_max,
    const int32_t* __restrict__ n_dev, int32_t* __restrict__ found_inf) {
    using Lx = Lanes<DEG>;
    const int64_t n = rows(n_max, n_dev);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane / Lx::C, ch = lane - sub * Lx::C;
    const int64_t i = (int64_t)blockIdx.x * Lx::SPB + warp * Lx::SPW + sub;
    if (sub >= Lx::SPW || i >= n) return;
    const float g = channel_grad<DEG>(ch, i, dirs, sigma, rgb, dsigma, drgb);
    if (g == 0.0f) return;   // samples behind the termination point, masked channels: nothing to scatter
    const Cell c = sample_cell(lay, xyz, i);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        float w;
        const int64_t node = corner(lay, c, q, w);
        if (node < 0) continue;
        atomicAdd(channel_dst(dsh, ddensity, node, ch, Lx::D), w * g);   // red.global.add.f32
    }
    if (!finite(g) && found_inf != nullptr) *found_inf = 1;
}

template <int DEG>
__global__ void __launch_bounds__(kThreads) voxel_bwd_thread_kernel(
    const float* __restrict__ xyz, const float* __restrict__ dirs, const float* __restrict__ sigma,
    const float* __restrict__ rgb, const float* __restrict__ dsigma, const float* __restrict__ drgb,
    const ngp_voxel_layout lay, float* __restrict__ dsh, float* __restrict__ ddensity, int64_t n_max,
    const int32_t* __restrict__ n_dev, int32_t* __restrict__ found_inf) {
    using Lx = Lanes<DEG>;
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (i >= rows(n_max, n_dev)) return;
    float g[Lx::C];
    bool bad = false;
#pragma unroll
    for (int ch = 0; ch < Lx::C; ++ch) {
        g[ch] = channel_grad<DEG>(ch, i, dirs, sigma, rgb, dsigma, drgb);
        bad = bad || !finite(g[ch]);
    }
    const Cell c = sample_cell(lay, xyz, i);
#pragma unroll 1
    for (int q = 0; q < 8; ++q) {
        float w;
        const int64_t node = corner(lay, c, q, w);
        if (node < 0) continue;
#pragma unroll
        for (int ch = 0; ch < Lx::C; ++ch)
            if (g[ch] != 0.0f) atomicAdd(channel_dst(dsh, ddensity, node, ch, Lx::D), w * g[ch]);
    }
    if (bad && found_inf != nullptr) *found_inf = 1;
}

// ---- regularisers: total variation and density sparsity over the node block B (DESIGN.md §6d) ----------------------
// Gather, not scatter: the thread of (node v, channel ch) computes the whole gradient of that element from v's own
// term and the terms of its three backward neighbours v - e_a, so every gradient float is written by one thread with
// a plain read-modify-write: no atomics, bit-reproducible.  Mapping: blockIdx.y = the x-slice of B; the (y, z) plane
// of B times the C active channels is flattened, channel fastest, so C consecutive lanes own one node and a node's
// neighbour read is one coalesced row (the lane-per-channel mapping of the kernels above).
struct RegArgs {
    const float* sh;
    const float* density;
    float* dsh;
    float* ddensity;
    const float* scale_dev;
    float* loss;
    float loss_scale;
    float c_tv_sh;       // w_tv_sh / (|B| * 3D)
    float c_tv_sigma;    // w_tv_sigma / |B|
    float c_sparsity;    // w_sparsity / |B|
    int32_t grid;
    int32_t lo[3], hi[3];
    int32_t ny, nz;      // B's extent along y and z
};

constexpr float kRegEps = 1e-8f;

// sqrt(dx^2 + dy^2 + dz^2 + eps), in this order
__device__ __forceinline__ float tv_norm(float dx, float dy, float dz) {
    return sqrtf(f_add(f_add(f_add(f_mul(dx, dx), f_mul(dy, dy)), f_mul(dz, dz)), kRegEps));
}

template <int NSH, bool DEN>
__global__ void __launch_bounds__(kThreads) voxel_reg_kernel(const RegArgs a) {
    constexpr int C = NSH + (DEN ? 1 : 0);
    __shared__ float part[kWarps];
    const int e = blockIdx.x * kThreads + threadIdx.x;   // < ny * nz * C <= 2048^2 * 28
    float loss = 0.0f;
    if (e < a.ny * a.nz * C) {
        const int yz = e / C, ch = e - yz * C;
        const int i = a.lo[0] + (int)blockIdx.y, j = a.lo[1] + yz / a.nz, k = a.lo[2] + yz % a.nz;
        const bool den = DEN && ch == NSH;
        const float* f = den ? a.density : a.sh + ch;
        float* dst = den ? a.ddensity : a.dsh + ch;
        const int64_t stride = den ? 1 : NSH;   // floats per node
        const int64_t G = a.grid, sx = G * G, sy = G;
        const int64_t n0 = ((int64_t)i * G + j) * G + k;
        const bool px = i + 1 < a.hi[0], py = j + 1 < a.hi[1], pz = k + 1 < a.hi[2];
        const float v0 = __ldg(f + n0 * stride);
        const float c_tv = den ? a.c_tv_sigma : a.c_tv_sh;
        float g = 0.0f;
        if (c_tv != 0.0f) {
            // v's own term: d s(v) / d V(v) = -(dx + dy + dz) / s(v)
            const float dx = px ? f_sub(__ldg(f + (n0 + sx) * stride), v0) : 0.0f;
            const float dy = py ? f_sub(__ldg(f + (n0 + sy) * stride), v0) : 0.0f;
            const float dz = pz ? f_sub(__ldg(f + (n0 + 1) * stride), v0) : 0.0f;
            const float s = tv_norm(dx, dy, dz);
            float t = -f_div(f_add(f_add(dx, dy), dz), s);
            // backward neighbour w = v - e_a: d s(w) / d V(v) = Delta_a(w) / s(w); w's other two differences reach
            // w + e_b, which lies in B exactly when v + e_b does
            if (i > a.lo[0]) {
                const int64_t w = n0 - sx;
                const float b = __ldg(f + w * stride);
                const float ex = f_sub(v0, b);
                const float ey = py ? f_sub(__ldg(f + (w + sy) * stride), b) : 0.0f;
                const float ez = pz ? f_sub(__ldg(f + (w + 1) * stride), b) : 0.0f;
                t = f_add(t, f_div(ex, tv_norm(ex, ey, ez)));
            }
            if (j > a.lo[1]) {
                const int64_t w = n0 - sy;
                const float b = __ldg(f + w * stride);
                const float ex = px ? f_sub(__ldg(f + (w + sx) * stride), b) : 0.0f;
                const float ey = f_sub(v0, b);
                const float ez = pz ? f_sub(__ldg(f + (w + 1) * stride), b) : 0.0f;
                t = f_add(t, f_div(ey, tv_norm(ex, ey, ez)));
            }
            if (k > a.lo[2]) {
                const int64_t w = n0 - 1;
                const float b = __ldg(f + w * stride);
                const float ex = px ? f_sub(__ldg(f + (w + sx) * stride), b) : 0.0f;
                const float ey = py ? f_sub(__ldg(f + (w + sy) * stride), b) : 0.0f;
                const float ez = f_sub(v0, b);
                t = f_add(t, f_div(ez, tv_norm(ex, ey, ez)));
            }
            g = f_mul(c_tv, t);
            loss = f_mul(c_tv, s);
        }
        if (den && a.c_sparsity != 0.0f) {
            // log(1 + 2 r^2), r = ReLU(density); d/d density = 4 r / (1 + 2 r^2).  NaN stays NaN (not 0) so that the
            // finite check downstream sees it.
            const float r = v0 < 0.0f ? 0.0f : v0;
            const float q = f_add(1.0f, f_mul(2.0f, f_mul(r, r)));
            g = f_add(g, f_mul(a.c_sparsity, f_div(f_mul(4.0f, r), q)));
            loss = f_add(loss, f_mul(a.c_sparsity, logf(q)));
        }
        const float scale = a.scale_dev != nullptr ? *a.scale_dev : a.loss_scale;
        // a channel whose terms are all off is not written (DEN is false when both density weights are 0)
        if (den ? (c_tv != 0.0f || a.c_sparsity != 0.0f) : c_tv != 0.0f)
            dst[n0 * stride] = f_add(dst[n0 * stride], f_mul(scale, g));
    }
    if (a.loss == nullptr) return;   // uniform over the launch
    loss = warp_sum(loss);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float sum = 0.0f;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) sum += part[w];
        atomicAdd(a.loss, sum);
    }
}

template <int NSH, bool DEN>
void launch_reg(const RegArgs& a, int nx, cudaStream_t st) {
    constexpr int C = NSH + (DEN ? 1 : 0);
    const int plane = a.ny * a.nz * C;
    voxel_reg_kernel<NSH, DEN><<<dim3((unsigned)((plane + kThreads - 1) / kThreads), (unsigned)nx), kThreads, 0, st>>>(a);
}

template <int DEG>
void launch_reg_deg(const RegArgs& a, int nx, bool sh, bool den, cudaStream_t st) {
    constexpr int NSH = 3 * Lanes<DEG>::D;
    if (sh && den)
        launch_reg<NSH, true>(a, nx, st);
    else if (sh)
        launch_reg<NSH, false>(a, nx, st);
    else
        launch_reg<0, true>(a, nx, st);
}

int check_layout(const ngp_voxel_layout* lay) {
    NGP_REQUIRE(lay != nullptr, "null layout");
    NGP_REQUIRE(lay->grid >= 1 && lay->grid <= NGP_VOXEL_MAX_GRID, "grid must be in [1, 2048]");
    NGP_REQUIRE(lay->sh_degree >= 0 && lay->sh_degree <= 2, "sh_degree must be 0, 1 or 2");
    NGP_REQUIRE(lay->radius > 0.0f && lay->radius < INFINITY, "radius must be positive and finite");
    NGP_REQUIRE(fabsf(lay->c_min) < INFINITY, "c_min must be finite");
    return 0;
}

template <int DEG>
unsigned warp_blocks(int64_t n) {
    return (unsigned)((n + Lanes<DEG>::SPB - 1) / Lanes<DEG>::SPB);
}

unsigned thread_blocks(int64_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

template <int DEG>
void launch_fwd(const float* xyz, const float* dirs, const float* sh, const float* density,
                const ngp_voxel_layout& lay, float* sigma, float* rgb, int64_t n_max, const int32_t* n_dev,
                cudaStream_t st) {
    voxel_fwd_kernel<DEG><<<warp_blocks<DEG>(n_max), kThreads, 0, st>>>(xyz, dirs, sh, density, lay, sigma, rgb,
                                                                         n_max, n_dev);
}

template <int DEG>
void launch_bwd(int mapping, const float* xyz, const float* dirs, const float* sigma, const float* rgb,
                const float* dsigma, const float* drgb, const ngp_voxel_layout& lay, float* dsh, float* ddensity,
                int64_t n_max, const int32_t* n_dev, int32_t* found_inf, cudaStream_t st) {
    if (mapping == NGP_VOXEL_BWD_THREAD)
        voxel_bwd_thread_kernel<DEG><<<thread_blocks(n_max), kThreads, 0, st>>>(
            xyz, dirs, sigma, rgb, dsigma, drgb, lay, dsh, ddensity, n_max, n_dev, found_inf);
    else
        voxel_bwd_warp_kernel<DEG><<<warp_blocks<DEG>(n_max), kThreads, 0, st>>>(
            xyz, dirs, sigma, rgb, dsigma, drgb, lay, dsh, ddensity, n_max, n_dev, found_inf);
}

}  // namespace

extern "C" {

int ngp_voxel_fwd(const float* xyz, const float* dirs, const float* sh, const float* density,
                  const ngp_voxel_layout* layout, float* sigma, float* rgb, int64_t n, void* stream) {
    return ngp_voxel_fwd_dyn(xyz, dirs, sh, density, layout, sigma, rgb, n, nullptr, stream);
}

int ngp_voxel_fwd_dyn(const float* xyz, const float* dirs, const float* sh, const float* density,
                      const ngp_voxel_layout* layout, float* sigma, float* rgb, int64_t n_max, const int32_t* n_dev,
                      void* stream) {
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n_max >= 0, "negative n");
    if (n_max == 0) return 0;
    NGP_REQUIRE(xyz && density && sigma, "null pointer");
    cudaStream_t st = ngp::as_stream(stream);
    if (rgb == nullptr) {   // density-only mode
        voxel_density_kernel<<<thread_blocks(n_max), kThreads, 0, st>>>(xyz, density, *layout, sigma, n_max, n_dev);
        NGP_LAUNCHED("voxel_density_kernel");
        return 0;
    }
    NGP_REQUIRE(dirs && sh, "null pointer");
    switch (layout->sh_degree) {
        case 0: launch_fwd<0>(xyz, dirs, sh, density, *layout, sigma, rgb, n_max, n_dev, st); break;
        case 1: launch_fwd<1>(xyz, dirs, sh, density, *layout, sigma, rgb, n_max, n_dev, st); break;
        default: launch_fwd<2>(xyz, dirs, sh, density, *layout, sigma, rgb, n_max, n_dev, st); break;
    }
    NGP_LAUNCHED("voxel_fwd_kernel");
    return 0;
}

int ngp_voxel_bwd(const float* xyz, const float* dirs, const float* sigma, const float* rgb, const float* dsigma,
                  const float* drgb, const ngp_voxel_layout* layout, float* dsh, float* ddensity, int64_t n,
                  int32_t* found_inf_or_null, int mapping, void* stream) {
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(mapping == NGP_VOXEL_BWD_WARP || mapping == NGP_VOXEL_BWD_THREAD, "unknown mapping");
    if (n == 0) return 0;
    NGP_REQUIRE(xyz && dirs && sigma && rgb && dsigma && drgb && dsh && ddensity, "null pointer");
    cudaStream_t st = ngp::as_stream(stream);
    switch (layout->sh_degree) {
        case 0:
            launch_bwd<0>(mapping, xyz, dirs, sigma, rgb, dsigma, drgb, *layout, dsh, ddensity, n, nullptr,
                          found_inf_or_null, st);
            break;
        case 1:
            launch_bwd<1>(mapping, xyz, dirs, sigma, rgb, dsigma, drgb, *layout, dsh, ddensity, n, nullptr,
                          found_inf_or_null, st);
            break;
        default:
            launch_bwd<2>(mapping, xyz, dirs, sigma, rgb, dsigma, drgb, *layout, dsh, ddensity, n, nullptr,
                          found_inf_or_null, st);
            break;
    }
    NGP_LAUNCHED("voxel_bwd_kernel");
    return 0;
}

int ngp_voxel_reg(const float* sh, const float* density, const ngp_voxel_layout* layout, const int32_t* block6,
                  float w_tv_sigma, float w_tv_sh, float w_sparsity, float loss_scale, const float* scale_dev,
                  float* dsh, float* ddensity, float* loss_or_null, void* stream) {
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(block6 != nullptr, "null block");
    for (int a = 0; a < 3; ++a)
        NGP_REQUIRE(block6[a] >= 0 && block6[a] < block6[a + 3] && block6[a + 3] <= layout->grid,
                    "block bounds must satisfy 0 <= lo < hi <= grid on every axis");
    for (float w : {w_tv_sigma, w_tv_sh, w_sparsity})
        NGP_REQUIRE(w >= 0.0f && w < INFINITY, "weights must be finite and >= 0");
    NGP_REQUIRE(scale_dev != nullptr || fabsf(loss_scale) < INFINITY, "loss_scale must be finite");
    const bool sh_on = w_tv_sh != 0.0f, den_on = w_tv_sigma != 0.0f || w_sparsity != 0.0f;
    if (!sh_on && !den_on) return 0;
    NGP_REQUIRE(sh && density && dsh && ddensity, "null pointer");
    RegArgs a;
    a.sh = sh;
    a.density = density;
    a.dsh = dsh;
    a.ddensity = ddensity;
    a.scale_dev = scale_dev;
    a.loss = loss_or_null;
    a.loss_scale = loss_scale;
    a.grid = layout->grid;
    for (int k = 0; k < 3; ++k) {
        a.lo[k] = block6[k];
        a.hi[k] = block6[k + 3];
    }
    const int nx = a.hi[0] - a.lo[0];
    a.ny = a.hi[1] - a.lo[1];
    a.nz = a.hi[2] - a.lo[2];
    const double nodes = (double)nx * a.ny * a.nz, nsh = 3.0 * (layout->sh_degree + 1) * (layout->sh_degree + 1);
    a.c_tv_sh = (float)(w_tv_sh / (nodes * nsh));
    a.c_tv_sigma = (float)(w_tv_sigma / nodes);
    a.c_sparsity = (float)(w_sparsity / nodes);
    cudaStream_t st = ngp::as_stream(stream);
    switch (layout->sh_degree) {
        case 0: launch_reg_deg<0>(a, nx, sh_on, den_on, st); break;
        case 1: launch_reg_deg<1>(a, nx, sh_on, den_on, st); break;
        default: launch_reg_deg<2>(a, nx, sh_on, den_on, st); break;
    }
    NGP_LAUNCHED("voxel_reg_kernel");
    return 0;
}

}  // extern "C"
