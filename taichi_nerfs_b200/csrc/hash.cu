// hash.cu — multiresolution hash-grid encoding: forward, table backward, input backward.
//
// Semantics: modules/hash_encoder.py:43-143 (fp32) and modules/hash_encoder_half.py:112-213
// (fp16 table, fp16 accumulate) of the reference.  Per-level scale/resolution come from the
// host-built ngp_hash_layout (see include/ngp_b200.h) instead of a per-thread expf.
//
// GPU mapping.  The reference launches one thread per (sample, level) with the level as the
// fastest index and block_dim=16, so a warp touches 2 samples x 16 unrelated table regions and
// every thread pays 8 integer modulos.  Here a CTA owns 512 consecutive samples (xyz staged once in
// shared memory), WARP w handles LEVEL w and each lane walks a chunk of 16 consecutive samples.
// Consecutive samples of a ray are <= 1 finest-level cell apart, so (a) the forward re-gathers the
// 8 corners only when the cell changes (37x fewer loads at level 0, ~1x at the finest levels),
// (b) the backward accumulates w*dy in registers and issues its vector atomics only at cell
// changes, for the corners the new cell does not share with the old one, and (c) all lanes of a
// warp stay inside one level's table slab (L1/L2 locality).
// The fp32 gradient (43.6 MiB) and the streams of one launch exceed the H100's 50 MB L2, and the scatter is sensitive
// to that (scripts/hash_l2_probe.py: the same requests into an 8x smaller gradient run 1.58x faster; the forward's
// gathers only 1.04x).  So a large backward scatters one level group at a time, each group's gradient slice at most
// half the L2, with evict-first loads of dL/dout and evict-last atomics.  Results are staged in shared memory
// ([level][sample], chunk stride 17 words = conflict-free) and written with coalesced stores in
// the reference's [n, L*F] row-major layout.
#include <atomic>

#include "common.cuh"

namespace {

// Work decomposition (see file header): one CTA = 512 consecutive samples, warp w = level w,
// lane = a chunk of 16 consecutive samples processed serially with run-length reuse of the cell.
constexpr int kTile = 512;
constexpr int kChunk = 16;
constexpr int kThreads = 512;
constexpr int kRow = kTile + kTile / kChunk + 1;  // 545 words: chunk stride 17 (conflict-free), odd row stride
constexpr int kXChunk = kChunk + 1;               // xyz staged as float4, 17 float4 (272 B) per 16-sample chunk:
                                                  // one LDS.128 per sample, conflict-free per quarter warp
constexpr int kXWords = (kTile / kChunk) * kXChunk * 4;

// optional run-time extras: device-side row count and the world->[0,1] normalisation of NGP.density
struct Dyn {
    const int32_t* n_dev;  // rows = min(n, *n_dev) when non-null
    float lo[3], span[3];
    int normalize;
};
__device__ __forceinline__ int64_t effective_n(const Dyn& dyn, int64_t n) {
    if (dyn.n_dev == nullptr) return n;
    const int64_t v = (int64_t)*dyn.n_dev;
    return v < n ? (v < 0 ? 0 : v) : n;
}

struct LevelMeta {
    uint32_t offset;     // entries
    uint32_t size;       // entries
    uint32_t mask;       // size-1 if power of two else 0
    uint32_t res, res2;
    float scale;
    int dense;
};

__device__ __forceinline__ LevelMeta level_meta(const ngp_hash_layout& lay, int l) {
    LevelMeta m;
    m.offset = (uint32_t)lay.offsets[l];
    m.size = (uint32_t)lay.map_sizes[l];
    m.mask = (m.size & (m.size - 1)) == 0 ? m.size - 1 : 0u;
    m.res = lay.resolutions[l];
    m.res2 = m.res * m.res;
    m.scale = lay.scales[l];
    m.dense = l < lay.begin_fast_hash_level;
    return m;
}

// grid coordinate + fractional position of x at this level (hash_encoder.py:108-110)
template <bool kFracF16>
__device__ __forceinline__ void grid_pos(const float x[3], const LevelMeta& m, uint32_t g[3], float pos[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float p = f_add(f_mul(x[d], m.scale), 0.5f);
        const float fl = floorf(p);
        g[d] = (uint32_t)(int32_t)fl;
        // half kernel: pos -= cast(pos_grid, f16) (hash_encoder_half.py:132) — exact below 2048
        const float gf = kFracF16 ? __half2float(__float2half_rn((float)g[d])) : (float)g[d];
        pos[d] = f_sub(p, gf);
    }
}

// entry index of the 8 corners of cell g.  Same values as under_hash / fast_hash followed by
// `% map_size` (hash_encoder.py:43-71) but with the per-axis products hoisted out of the corner loop
// and the modulo replaced by a mask (power-of-two tables) or a conditional subtract (dense levels,
// where the linear index is < 2*size unless the coordinate wrapped).
__device__ __forceinline__ void corner_indices(const LevelMeta& m, const uint32_t g[3], uint32_t idx[8]) {
    if (m.dense) {
        const uint32_t base = g[0] + g[1] * m.res + g[2] * m.res2;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            uint32_t h = base + (c & 1) + ((c >> 1) & 1) * m.res + (c >> 2) * m.res2;
            if (h >= m.size) {
                h -= m.size;
                if (h >= m.size) h %= m.size;
            }
            idx[c] = m.offset + h;
        }
    } else {
        const uint32_t hy0 = g[1] * 2654435761u, hy1 = hy0 + 2654435761u;
        const uint32_t hz0 = g[2] * 805459861u, hz1 = hz0 + 805459861u;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const uint32_t h = (g[0] + (c & 1)) ^ ((c & 2) ? hy1 : hy0) ^ ((c & 4) ? hz1 : hz0);
            idx[c] = m.offset + (m.mask ? (h & m.mask) : (h % m.size));
        }
    }
}

// the 8 trilinear weights, w_c = ((1 * a_x) * a_y) * a_z exactly as hash_encoder.py:116-126
__device__ __forceinline__ void corner_weights(const float pos[3], float w[8]) {
    const float ax[2] = {f_sub(1.0f, pos[0]), pos[0]};
    const float ay[2] = {f_sub(1.0f, pos[1]), pos[1]};
    const float az[2] = {f_sub(1.0f, pos[2]), pos[2]};
    float axy[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) axy[c] = f_mul(ax[c & 1], ay[c >> 1]);
#pragma unroll
    for (int c = 0; c < 8; ++c) w[c] = f_mul(axy[c & 3], az[c >> 2]);
}

// Corner reuse between consecutive cells.  When a lane moves from cell pg to cell g and every per-axis offset
// g - pg is in {-1, 0, 1}, corner c' of g is corner c' + (g - pg) of pg whenever that lies in {0, 1}^3: the same grid
// coordinate, so the same table entry on dense and hashed levels alike.  Corner masks are 8-bit sets over c = x + 2y + 4z.
struct CellStep {
    uint32_t carried;  // corners of the new cell that are corners of the old one
    uint32_t stays;    // corners of the old cell that are corners of the new one (the others leave)
    int32_t d[3];
};

__device__ __forceinline__ CellStep cell_step(const uint32_t pg[3], const uint32_t g[3]) {
    constexpr uint32_t kLow[3] = {0x55u, 0x33u, 0x0Fu};  // corners with bit d clear; the complement has it set
    CellStep s;
    s.carried = s.stays = 0xFFu;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        s.d[d] = (int32_t)(g[d] - pg[d]);
        const uint32_t lo = kLow[d], hi = ~kLow[d] & 0xFFu;
        s.carried &= s.d[d] == 0 ? 0xFFu : s.d[d] == 1 ? lo : s.d[d] == -1 ? hi : 0u;
        s.stays &= s.d[d] == 0 ? 0xFFu : s.d[d] == 1 ? hi : s.d[d] == -1 ? lo : 0u;
    }
    return s;
}

// moves the carried corners' values to their places in the new cell, axis by axis (compile-time indices, selects);
// the slots of corners that are not carried are left holding stale values
__device__ __forceinline__ void shift_corners(float2 a[8], const CellStep& s) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (c & (1 << d)) continue;
            const float2 lo = a[c], hi = a[c | (1 << d)];
            a[c] = s.d[d] == 1 ? hi : lo;
            a[c | (1 << d)] = s.d[d] == -1 ? lo : hi;
        }
    }
}

// Per-instruction L2 eviction priorities (PTX createpolicy + .L2::cache_hint; no persisting-L2 set-aside is needed)
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_evict_last() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t l2_evict_normal() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint4 ldg_hint(const uint4* p, uint64_t pol) {
    uint4 v;
    asm("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
        : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
        : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void red_add_hint(float2* p, float2 v, uint64_t pol) {
    asm volatile("red.global.add.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(pol)
                 : "memory");
}
__device__ __forceinline__ void red_add_hint(float4* p, float4 v, uint64_t pol) {
    asm volatile("red.global.add.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w), "l"(pol)
                 : "memory");
}

template <typename T>
struct Vec2;
template <>
struct Vec2<float> { using type = float2; };
template <>
struct Vec2<__half> { using type = __half2; };

// two adjacent table entries as one vector load
template <typename V2>
struct Pair;
template <>
struct Pair<float2> {
    using type = float4;
    __device__ static __forceinline__ float2 lo(const float4& p) { return make_float2(p.x, p.y); }
    __device__ static __forceinline__ float2 hi(const float4& p) { return make_float2(p.z, p.w); }
};
template <>
struct Pair<__half2> {
    using type = uint2;
    __device__ static __forceinline__ __half2 lo(const uint2& p) { return *reinterpret_cast<const __half2*>(&p.x); }
    __device__ static __forceinline__ __half2 hi(const uint2& p) { return *reinterpret_cast<const __half2*>(&p.y); }
};

// ---- forward -------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) hash_fwd_kernel(const float* __restrict__ xyz,
                                                            const T* __restrict__ table,
                                                            const __grid_constant__ ngp_hash_layout lay,
                                                            T* __restrict__ out, int64_t n_max, const Dyn dyn) {
    using V2 = typename Vec2<T>::type;
    const int64_t n = effective_n(dyn, n_max);
    constexpr bool kHalf = sizeof(T) == 2;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    float* sx = reinterpret_cast<float*>(smem_raw);                         // [kTile*3]
    V2* tile = reinterpret_cast<V2*>(smem_raw + kXWords * sizeof(float));  // [L][kRow]

    const int L = lay.n_levels;
    const int64_t base = (int64_t)blockIdx.x * kTile;
    if (base >= n) return;
    const int rows = (int)min((int64_t)kTile, n - base);
    for (int r = threadIdx.x; r < rows; r += kThreads) {
        float v[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            v[k] = xyz[(base + r) * 3 + k];
            if (dyn.normalize) v[k] = f_div(f_sub(v[k], dyn.lo[k]), dyn.span[k]);  // networks.py:144
        }
        reinterpret_cast<float4*>(sx)[r + r / kChunk] = make_float4(v[0], v[1], v[2], 0.0f);
    }
    __syncthreads();

    const int level = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (level < L) {
        const LevelMeta m = level_meta(lay, level);
        const V2* tab = reinterpret_cast<const V2*>(table);
        uint32_t pg[3] = {0u, 0u, 0u};
        bool have = false;
        V2 v[8];
        V2* trow = tile + level * kRow + lane * (kChunk + 1);
#pragma unroll 4
        for (int j = 0; j < kChunk; ++j) {
            const int s = lane * kChunk + j;
            if (s >= rows) break;
            const float4 xv = reinterpret_cast<const float4*>(sx)[lane * kXChunk + j];
            const float x[3] = {xv.x, xv.y, xv.z};
            uint32_t g[3];
            float pos[3];
            grid_pos<kHalf>(x, m, g, pos);
            if (!have || g[0] != pg[0] || g[1] != pg[1] || g[2] != pg[2]) {  // new cell: gather its 8 corners
                have = true;
                uint32_t idx[8];
                corner_indices(m, g, idx);
                // the two x-neighbours (c, c+1) share one aligned 2-entry block whenever their indices
                // differ only in bit 0 (always on hashed levels with even gx: h(x+1) = h(x)^1): one load
#pragma unroll
                for (int c = 0; c < 8; c += 2) {
                    if ((idx[c] ^ idx[c + 1]) == 1u) {
                        using V4 = typename Pair<V2>::type;
                        const V4 pr = __ldg(reinterpret_cast<const V4*>(tab + (idx[c] & ~1u)));
                        const V2 lo = Pair<V2>::lo(pr), hi = Pair<V2>::hi(pr);
                        v[c] = (idx[c] & 1u) ? hi : lo;
                        v[c + 1] = (idx[c] & 1u) ? lo : hi;
                    } else {
                        v[c] = __ldg(tab + idx[c]);
                        v[c + 1] = __ldg(tab + idx[c + 1]);
                    }
                }
                pg[0] = g[0];
                pg[1] = g[1];
                pg[2] = g[2];
            }
            float w[8];
            corner_weights(pos, w);
            if constexpr (kHalf) {
                __half2 acc = __float2half2_rn(0.0f);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const float2 t = __half22float2(v[c]);
                    // local += cast(w * table[idx], f16); f16 accumulate (hash_encoder_half.py:159)
                    acc = __hadd2(acc, __floats2half2_rn(f_mul(w[c], t.x), f_mul(w[c], t.y)));
                }
                trow[j] = acc;
            } else {
                float2 acc = make_float2(0.0f, 0.0f);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    acc.x = f_add(acc.x, f_mul(w[c], v[c].x));
                    acc.y = f_add(acc.y, f_mul(w[c], v[c].y));
                }
                trow[j] = acc;
            }
        }
    }
    __syncthreads();
    // coalesced write-out of the [rows, L] result
    V2* o2 = reinterpret_cast<V2*>(out) + base * L;
    constexpr int kVec = 16 / sizeof(V2);  // entries per 16-byte store (4 for fp16, 2 for fp32)
    if (L % kVec == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
        const int groups = L / kVec;
        for (int k = threadIdx.x; k < rows * groups; k += kThreads) {
            const int r = k / groups, l0 = (k - r * groups) * kVec;
            V2 v[kVec];
#pragma unroll
            for (int q = 0; q < kVec; ++q) v[q] = tile[(l0 + q) * kRow + r + r / kChunk];
            *reinterpret_cast<uint4*>(o2 + (int64_t)r * L + l0) = *reinterpret_cast<const uint4*>(v);
        }
    } else {
        for (int k = threadIdx.x; k < rows * L; k += kThreads) {
            const int r = k / L, l = k - r * L;
            o2[k] = tile[l * kRow + r + r / kChunk];
        }
    }
}

// ---- backward wrt table ------------------------------------------------------------------------------
// Consecutive samples of a ray stay in the same cell for 1/(res*dt) steps (37 at level 0 down to ~1
// at the finest levels), so a lane accumulates w*dy for its 16-sample chunk in registers and issues
// the 8 vector atomics only when the cell changes: ~2.3x fewer L2 atomics on Lego-shape rays.  When the
// new cell is a neighbour of the old one, only the corners that leave are scattered and the shared ones
// keep accumulating (cell_step): another 25 % fewer atomics on the lego_half sample stream
// (scripts/hash_corner_reuse.py).  The forward does not carry corners: there it saved loads but not time.
// At most 56 registers (ptxas alone picks 63): the scatter waits on L2 atomics and loads, and what hides that latency
// is warps per SM.  56 lets three CTAs of the coarse level group (11 levels, 352 threads) fit per SM instead of two,
// and seven of the fine group (5 levels) instead of six; 48 would spill.  DESIGN.md §4 has the measurements.
template <typename T>
__global__ void __maxnreg__(56) hash_bwd_kernel(const float* __restrict__ xyz,
                                                const T* __restrict__ dout,
                                                const __grid_constant__ ngp_hash_layout lay,
                                                float* __restrict__ grad_table, int64_t n_max,
                                                const Dyn dyn, int level_begin, int level_end,
                                                int32_t* __restrict__ found_inf, int grouped) {
    // blockDim.x = 32 * (level_end - level_begin): warp w scatters level level_begin + w.  The host launches one level
    // group at a time (bwd_level_groups), so only the group's dL/dout columns are staged: tile row w = level
    // level_begin + w.
    using V2 = typename Vec2<T>::type;
    const int64_t n = effective_n(dyn, n_max);
    constexpr bool kHalf = sizeof(T) == 2;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    float* sx = reinterpret_cast<float*>(smem_raw);
    V2* tile = reinterpret_cast<V2*>(smem_raw + kXWords * sizeof(float));

    const int L = lay.n_levels;
    const int nthreads = blockDim.x;
    const int64_t base = (int64_t)blockIdx.x * kTile;
    if (base >= n) return;
    const int rows = (int)min((int64_t)kTile, n - base);
    for (int r = threadIdx.x; r < rows; r += nthreads) {
        float v[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            v[k] = xyz[(base + r) * 3 + k];
            if (dyn.normalize) v[k] = f_div(f_sub(v[k], dyn.lo[k]), dyn.span[k]);  // networks.py:144
        }
        reinterpret_cast<float4*>(sx)[r + r / kChunk] = make_float4(v[0], v[1], v[2], 0.0f);
    }
    // grouped launches: dL/dout is read once, evict-first, so that it does not push the gradient slice being
    // scattered out of L2.  A launch that is the only group keeps the default priorities: an evict-last gradient left
    // in L2 after it slowed the small-batch step more than the hints sped the launch up.
    const uint64_t stream_pol = grouped ? l2_evict_first() : l2_evict_normal();
    const V2* d2 = reinterpret_cast<const V2*>(dout) + base * L;
    constexpr int kVec = 16 / sizeof(V2);
    if (L % kVec == 0 && (reinterpret_cast<uintptr_t>(dout) & 15) == 0) {
        // 16-byte loads over the aligned column blocks that cover [level_begin, level_end)
        const int v0 = level_begin / kVec, groups = (level_end + kVec - 1) / kVec - v0;
        for (int k = threadIdx.x; k < rows * groups; k += nthreads) {
            const int r = k / groups, l0 = (v0 + k - r * groups) * kVec;
            const uint4 raw = ldg_hint(reinterpret_cast<const uint4*>(d2 + (int64_t)r * L + l0), stream_pol);
            const V2* v = reinterpret_cast<const V2*>(&raw);
#pragma unroll
            for (int q = 0; q < kVec; ++q)
                if (l0 + q >= level_begin && l0 + q < level_end) tile[(l0 + q - level_begin) * kRow + r + r / kChunk] = v[q];
        }
    } else {
        const int nl = level_end - level_begin;
        for (int k = threadIdx.x; k < rows * nl; k += nthreads) {
            const int r = k / nl, l = k - r * nl;
            tile[l * kRow + r + r / kChunk] = d2[(int64_t)r * L + level_begin + l];
        }
    }
    __syncthreads();

    const int level = level_begin + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (level >= L || level >= level_end) return;
    const LevelMeta m = level_meta(lay, level);
    float2* g2 = reinterpret_cast<float2*>(grad_table);
    const V2* trow = tile + (level - level_begin) * kRow + lane * (kChunk + 1);
    // the group's gradient slice is sized to stay in L2 for the whole launch (bwd_level_groups); evict-last keeps it
    // there against the streams
    const uint64_t grad_pol = grouped ? l2_evict_last() : l2_evict_normal();

    uint32_t pg[3] = {0u, 0u, 0u};
    float2 acc[8];
    bool pending = false;
    bool bad = false;   // a non-finite contribution: raised at the source, so that no separate pass over the 45 MB
                        // gradient buffer is needed for GradScaler's inf check (optional, found_inf may be NULL)
    // scatters the corners of cell pg in `leaving` (the others are carried into the next cell)
    auto flush = [&](uint32_t leaving) {
        uint32_t idx[8];
        corner_indices(m, pg, idx);
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if ((leaving >> c) & 1u) bad = bad || !(fabsf(acc[c].x) < INFINITY) || !(fabsf(acc[c].y) < INFINITY);
#pragma unroll
        for (int c = 0; c < 8; c += 2) {
            const bool out0 = (leaving >> c) & 1u, out1 = (leaving >> (c + 1)) & 1u;
            if (out0 && out1 && (idx[c] ^ idx[c + 1]) == 1u) {  // x-neighbours in one aligned 16-byte block: one L2 atomic
                const float2 lo = (idx[c] & 1u) ? acc[c + 1] : acc[c], hi = (idx[c] & 1u) ? acc[c] : acc[c + 1];
                red_add_hint(reinterpret_cast<float4*>(g2 + (idx[c] & ~1u)), make_float4(lo.x, lo.y, hi.x, hi.y), grad_pol);
            } else {
                if (out0) red_add_hint(g2 + idx[c], acc[c], grad_pol);
                if (out1) red_add_hint(g2 + idx[c + 1], acc[c + 1], grad_pol);
            }
        }
    };
#pragma unroll 2
    for (int j = 0; j < kChunk; ++j) {
        const int s = lane * kChunk + j;
        if (s >= rows) break;
        float2 dy;
        if constexpr (kHalf) dy = __half22float2(trow[j]);
        else dy = trow[j];
        if (dy.x == 0.0f && dy.y == 0.0f) continue;  // hash_encoder_half.py:210
        const float4 xv = reinterpret_cast<const float4*>(sx)[lane * kXChunk + j];
        const float x[3] = {xv.x, xv.y, xv.z};
        uint32_t g[3];
        float pos[3];
        grid_pos<kHalf>(x, m, g, pos);
        if (!pending || g[0] != pg[0] || g[1] != pg[1] || g[2] != pg[2]) {
            uint32_t carried = 0u;
            if (pending) {
                const CellStep st = cell_step(pg, g);
                flush(~st.stays & 0xFFu);
                shift_corners(acc, st);
                carried = st.carried;
            }
            pg[0] = g[0];
            pg[1] = g[1];
            pg[2] = g[2];
#pragma unroll
            for (int c = 0; c < 8; ++c)
                if (!((carried >> c) & 1u)) acc[c] = make_float2(0.0f, 0.0f);
            pending = true;
        }
        float w[8];
        corner_weights(pos, w);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            acc[c].x += w[c] * dy.x;
            acc[c].y += w[c] * dy.y;
        }
    }
    if (pending) flush(0xFFu);
    if (bad && found_inf != nullptr) *found_inf = 1;
}

// ---- generic feature width (F = 1..8, e.g. the reference's --deployment config L=4 F=4) -----------
// Plain thread-per-(sample, level) kernels; the tuned kernels above cover the stock F = 2.
template <typename T>
__global__ void __launch_bounds__(256) hash_fwd_generic_kernel(const float* __restrict__ xyz, const T* __restrict__ table,
                                                               const __grid_constant__ ngp_hash_layout lay,
                                                               T* __restrict__ out, int64_t n_max, const Dyn dyn) {
    constexpr bool kHalf = sizeof(T) == 2;
    const int64_t n = effective_n(dyn, n_max);
    const int L = lay.n_levels, F = lay.feat_dim;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n * L) return;
    const int64_t i = gid / L;
    const int level = (int)(gid - i * L);
    float x[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        x[k] = xyz[i * 3 + k];
        if (dyn.normalize) x[k] = f_div(f_sub(x[k], dyn.lo[k]), dyn.span[k]);
    }
    const LevelMeta m = level_meta(lay, level);
    uint32_t g[3], idx[8];
    float pos[3], w[8];
    grid_pos<kHalf>(x, m, g, pos);
    corner_indices(m, g, idx);
    corner_weights(pos, w);
    for (int f = 0; f < F; ++f) {
        if constexpr (kHalf) {
            __half acc = __float2half_rn(0.0f);
#pragma unroll
            for (int c = 0; c < 8; ++c)
                acc = __hadd(acc, __float2half_rn(f_mul(w[c], __half2float(table[(int64_t)idx[c] * F + f]))));
            out[i * L * F + level * F + f] = acc;
        } else {
            float acc = 0.0f;
#pragma unroll
            for (int c = 0; c < 8; ++c) acc = f_add(acc, f_mul(w[c], table[(int64_t)idx[c] * F + f]));
            out[i * L * F + level * F + f] = acc;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) hash_bwd_generic_kernel(const float* __restrict__ xyz, const T* __restrict__ dout,
                                                               const __grid_constant__ ngp_hash_layout lay,
                                                               float* __restrict__ grad_table, int64_t n_max,
                                                               const Dyn dyn) {
    constexpr bool kHalf = sizeof(T) == 2;
    const int64_t n = effective_n(dyn, n_max);
    const int L = lay.n_levels, F = lay.feat_dim;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= n * L) return;
    const int64_t i = gid / L;
    const int level = (int)(gid - i * L);
    float dy[8];
    bool any = false;
    for (int f = 0; f < F; ++f) {
        dy[f] = load_as_float(dout, i * L * F + level * F + f);
        any |= dy[f] != 0.0f;
    }
    if (!any) return;
    float x[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        x[k] = xyz[i * 3 + k];
        if (dyn.normalize) x[k] = f_div(f_sub(x[k], dyn.lo[k]), dyn.span[k]);
    }
    const LevelMeta m = level_meta(lay, level);
    uint32_t g[3], idx[8];
    float pos[3], w[8];
    grid_pos<kHalf>(x, m, g, pos);
    corner_indices(m, g, idx);
    corner_weights(pos, w);
#pragma unroll
    for (int c = 0; c < 8; ++c)
        for (int f = 0; f < F; ++f) atomicAdd(grad_table + (int64_t)idx[c] * F + f, w[c] * dy[f]);
}

__device__ __forceinline__ uint32_t corner_index(const LevelMeta& m, const uint32_t g[3], int c) {
    uint32_t idx[8];
    corner_indices(m, g, idx);
    return idx[c];
}

// ---- backward wrt input position ----------------------------------------------------------------
// The derivative of the forward inside the cell of x: the fp16 kernel takes it at the forward's fraction p - f16(g),
// which differs from p - g for odd g above 2048 (levels 14-15 at max_res 4096).  With the AABB fold (dyn.normalize) x
// is the world position, normalised as the forward does, and dx is the world gradient: the [0,1] gradient divided by
// the span, as autograd divides it through NGP.density's normalisation.
__device__ __forceinline__ void load_input_pos(const float* __restrict__ xyz, int64_t i, const Dyn& dyn, float x[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        x[k] = xyz[i * 3 + k];
        if (dyn.normalize) x[k] = f_div(f_sub(x[k], dyn.lo[k]), dyn.span[k]);
    }
}

__device__ __forceinline__ void store_input_grad(float* __restrict__ dx, int64_t i, const Dyn& dyn, float gx, float gy,
                                                 float gz) {
    if (dyn.normalize) {
        gx = f_div(gx, dyn.span[0]);
        gy = f_div(gy, dyn.span[1]);
        gz = f_div(gz, dyn.span[2]);
    }
    dx[i * 3 + 0] = gx;
    dx[i * 3 + 1] = gy;
    dx[i * 3 + 2] = gz;
}

template <typename T>
__global__ void __launch_bounds__(256) hash_bwd_input_kernel(const float* __restrict__ xyz,
                                                             const T* __restrict__ table,
                                                             const T* __restrict__ dout,
                                                             const __grid_constant__ ngp_hash_layout lay,
                                                             float* __restrict__ dx, int64_t n_max, const Dyn dyn) {
    using V2 = typename Vec2<T>::type;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= effective_n(dyn, n_max)) return;
    const int L = lay.n_levels;
    float x[3];
    load_input_pos(xyz, i, dyn, x);
    float gx = 0.f, gy = 0.f, gz = 0.f;
    for (int l = 0; l < L; ++l) {
        const LevelMeta m = level_meta(lay, l);
        uint32_t g[3];
        float pos[3];
        grid_pos<sizeof(T) == 2>(x, m, g, pos);
        const V2 dyv = reinterpret_cast<const V2*>(dout)[i * L + l];
        float2 dy;
        if constexpr (sizeof(T) == 2) dy = __half22float2(dyv);
        else dy = dyv;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const V2 tv = __ldg(reinterpret_cast<const V2*>(table) + corner_index(m, g, c));
            float2 t;
            if constexpr (sizeof(T) == 2) t = __half22float2(tv);
            else t = tv;
            const float v = (t.x * dy.x + t.y * dy.y) * m.scale;
            const float wx = (c & 1) ? pos[0] : 1.0f - pos[0];
            const float wy = (c & 2) ? pos[1] : 1.0f - pos[1];
            const float wz = (c & 4) ? pos[2] : 1.0f - pos[2];
            gx += ((c & 1) ? v : -v) * wy * wz;
            gy += ((c & 2) ? v : -v) * wx * wz;
            gz += ((c & 4) ? v : -v) * wx * wy;
        }
    }
    store_input_grad(dx, i, dyn, gx, gy, gz);
}

// any feature width in [1, 8] (the --deployment model has 4): the same terms, the feature sum in feature order
template <typename T>
__global__ void __launch_bounds__(256) hash_bwd_input_generic_kernel(const float* __restrict__ xyz,
                                                                     const T* __restrict__ table,
                                                                     const T* __restrict__ dout,
                                                                     const __grid_constant__ ngp_hash_layout lay,
                                                                     float* __restrict__ dx, int64_t n_max,
                                                                     const Dyn dyn) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= effective_n(dyn, n_max)) return;
    const int L = lay.n_levels, F = lay.feat_dim;
    float x[3];
    load_input_pos(xyz, i, dyn, x);
    float gx = 0.f, gy = 0.f, gz = 0.f;
    for (int l = 0; l < L; ++l) {
        const LevelMeta m = level_meta(lay, l);
        uint32_t g[3], idx[8];
        float pos[3];
        grid_pos<sizeof(T) == 2>(x, m, g, pos);
        corner_indices(m, g, idx);
        float dy[8];
        for (int f = 0; f < F; ++f) dy[f] = load_as_float(dout, (i * L + l) * F + f);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float dot = 0.0f;
            for (int f = 0; f < F; ++f) dot += load_as_float(table, (int64_t)idx[c] * F + f) * dy[f];
            const float v = dot * m.scale;
            const float wx = (c & 1) ? pos[0] : 1.0f - pos[0];
            const float wy = (c & 2) ? pos[1] : 1.0f - pos[1];
            const float wz = (c & 4) ? pos[2] : 1.0f - pos[2];
            gx += ((c & 1) ? v : -v) * wy * wz;
            gy += ((c & 2) ? v : -v) * wx * wz;
            gz += ((c & 4) ? v : -v) * wx * wy;
        }
    }
    store_input_grad(dx, i, dyn, gx, gy, gz);
}

size_t smem_bytes(int n_levels, int vec_bytes) {
    return (size_t)kXWords * sizeof(float) + (size_t)n_levels * kRow * vec_bytes;
}

// the fp32 tiles need more than the default 48 KB of dynamic shared memory (6 KB + 16*545*8 = 74 KB)
int configure_smem() {
    static bool done = false;
    if (done) return 0;
    const int big = (int)smem_bytes(NGP_MAX_LEVELS, 8);
    cudaError_t e = cudaFuncSetAttribute(hash_fwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, big);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(hash_bwd_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, big);
    if (e != cudaSuccess) {
        ngp::set_error("hash kernels: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        return (int)e;
    }
    done = true;
    return 0;
}

Dyn make_dyn(const int32_t* n_dev, const float* aabb6) {
    Dyn d;
    d.n_dev = n_dev;
    d.normalize = aabb6 != nullptr;
    for (int k = 0; k < 3; ++k) {
        d.lo[k] = aabb6 ? aabb6[k] : 0.0f;
        d.span[k] = aabb6 ? aabb6[3 + k] : 1.0f;
    }
    return d;
}

// Share of the L2 that one level group's fp32 gradient slice may fill.  The rest holds what streams through during the
// launch (dL/dout, xyz) and the lines in flight; DESIGN.md §4 has the measurements behind the value.
constexpr int64_t kL2BudgetNum = 1, kL2BudgetDen = 2;
// Launches of fewer rows stay one group: they scatter too few requests per gradient line for the residency to pay for
// the extra launches (measured: the 393 k-row lego_fp32_1024 step got slower grouped, the 3.1 M-row lego_half and
// 8.4 M-row garden16 steps faster).
constexpr int64_t kGroupMinRows = 1 << 20;

// L2 size of the current device, queried once per device.  Attribute queries are not stream operations, so this is
// legal while a stream is being captured.
int64_t device_l2_bytes() {
    constexpr int kMaxDevices = 64;
    static std::atomic<int> cached[kMaxDevices];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (dev < kMaxDevices && cached[dev].load(std::memory_order_relaxed) > 0) return cached[dev].load(std::memory_order_relaxed);
    int bytes = 0;
    if (cudaDeviceGetAttribute(&bytes, cudaDevAttrL2CacheSize, dev) != cudaSuccess || bytes <= 0) return 0;
    if (dev < kMaxDevices) cached[dev].store(bytes, std::memory_order_relaxed);
    return bytes;
}

int check_layout(const ngp_hash_layout* lay) {
    NGP_REQUIRE(lay != nullptr, "null layout");
    NGP_REQUIRE(lay->n_levels >= 1 && lay->n_levels <= NGP_MAX_LEVELS, "n_levels out of range");
    NGP_REQUIRE(lay->feat_dim >= 1 && lay->feat_dim <= 8, "feature_per_level must be in [1, 8]");
    return 0;
}

}  // namespace

extern "C" {

int ngp_hash_encode_fwd(const float* xyz, const void* table, const ngp_hash_layout* layout, void* out,
                        int dtype, int64_t n, void* stream) {
    return ngp_hash_encode_fwd_dyn(xyz, table, layout, out, dtype, n, nullptr, nullptr, stream);
}

int ngp_hash_encode_fwd_dyn(const float* xyz, const void* table, const ngp_hash_layout* layout, void* out,
                            int dtype, int64_t n, const int32_t* n_dev, const float* aabb6, void* stream) {
    const Dyn dyn = make_dyn(n_dev, aabb6);
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(dtype == NGP_F32 || dtype == NGP_F16, "bad dtype");
    if (n == 0) return 0;
    NGP_REQUIRE(xyz && table && out, "null pointer");
    cudaStream_t st = ngp::as_stream(stream);
    if (layout->feat_dim != 2) {  // generic feature width
        const unsigned gg = (unsigned)((n * layout->n_levels + 255) / 256);
        if (dtype == NGP_F16)
            hash_fwd_generic_kernel<__half><<<gg, 256, 0, st>>>(xyz, (const __half*)table, *layout, (__half*)out, n, dyn);
        else
            hash_fwd_generic_kernel<float><<<gg, 256, 0, st>>>(xyz, (const float*)table, *layout, (float*)out, n, dyn);
        NGP_LAUNCHED("hash_fwd_generic_kernel");
        return 0;
    }
    // the gather loads an x-pair of entries as one vector from tab + (idx & ~1), and every access to out is at least
    // one entry wide
    const uintptr_t entry = dtype == NGP_F16 ? 4 : 8;
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(table) & (2 * entry - 1)) == 0,
                "table must be aligned to two entries (16 bytes for fp32, 8 for fp16) when feature_per_level == 2");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(out) & (entry - 1)) == 0,
                "out must be aligned to one entry (8 bytes for fp32, 4 for fp16) when feature_per_level == 2");
    const unsigned grid = (unsigned)((n + kTile - 1) / kTile);
    if (int rc = configure_smem()) return rc;
    if (dtype == NGP_F16)
        hash_fwd_kernel<__half><<<grid, kThreads, smem_bytes(layout->n_levels, 4), st>>>(xyz, (const __half*)table, *layout, (__half*)out, n, dyn);
    else
        hash_fwd_kernel<float><<<grid, kThreads, smem_bytes(layout->n_levels, 8), st>>>(xyz, (const float*)table, *layout, (float*)out, n, dyn);
    NGP_LAUNCHED("hash_fwd_kernel");
    return 0;
}

int ngp_hash_encode_bwd(const float* xyz, const void* dout, int dout_dtype, const ngp_hash_layout* layout,
                        float* grad_table, int64_t n, void* stream) {
    return ngp_hash_encode_bwd_dyn(xyz, dout, dout_dtype, layout, grad_table, n, nullptr, nullptr, stream);
}

int ngp_hash_encode_bwd_dyn(const float* xyz, const void* dout, int dout_dtype, const ngp_hash_layout* layout,
                            float* grad_table, int64_t n, const int32_t* n_dev, const float* aabb6, void* stream) {
    return ngp_hash_encode_bwd_levels(xyz, dout, dout_dtype, layout, grad_table, n, n_dev, aabb6, 0,
                                      layout ? layout->n_levels : 0, nullptr, stream);
}

int ngp_hash_encode_bwd_levels(const float* xyz, const void* dout, int dout_dtype, const ngp_hash_layout* layout,
                               float* grad_table, int64_t n, const int32_t* n_dev, const float* aabb6, int level_begin,
                               int level_end, int32_t* found_inf_or_null, void* stream) {
    const Dyn dyn = make_dyn(n_dev, aabb6);
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(level_begin >= 0 && level_begin < level_end && level_end <= layout->n_levels, "bad level range");
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(dout_dtype == NGP_F32 || dout_dtype == NGP_F16, "bad dtype");
    if (n == 0) return 0;
    NGP_REQUIRE(xyz && dout && grad_table, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(grad_table) & 7) == 0, "grad_table must be 8-byte aligned");
    cudaStream_t st = ngp::as_stream(stream);
    if (layout->feat_dim != 2) {
        NGP_REQUIRE(level_begin == 0 && level_end == layout->n_levels, "level groups need feature_per_level == 2");
        const unsigned gg = (unsigned)((n * layout->n_levels + 255) / 256);
        if (dout_dtype == NGP_F16)
            hash_bwd_generic_kernel<__half><<<gg, 256, 0, st>>>(xyz, (const __half*)dout, *layout, grad_table, n, dyn);
        else
            hash_bwd_generic_kernel<float><<<gg, 256, 0, st>>>(xyz, (const float*)dout, *layout, grad_table, n, dyn);
        NGP_LAUNCHED("hash_bwd_generic_kernel");
        return 0;
    }
    // a flush scatters an x-pair of entries as one 16-byte reduction at g2 + (idx & ~1), and dL/dout is read at least
    // one entry at a time
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(grad_table) & 15) == 0,
                "grad_table must be 16-byte aligned when feature_per_level == 2");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(dout) & (dout_dtype == NGP_F16 ? 3 : 7)) == 0,
                "dout must be aligned to one entry (8 bytes for fp32, 4 for fp16) when feature_per_level == 2");
    const unsigned grid = (unsigned)((n + kTile - 1) / kTile);
    if (int rc = configure_smem()) return rc;
    // one launch per level group, in level order: each launch's scatter stays inside an L2-sized gradient slice
    int32_t bounds[NGP_MAX_LEVELS + 1];
    const int64_t l2 = n >= kGroupMinRows ? device_l2_bytes() : 0;
    const int n_groups = ngp_hash_bwd_level_groups(layout, level_begin, level_end, l2, bounds);
    for (int g = 0; g < n_groups; ++g) {
        const int a = bounds[g], b = bounds[g + 1];
        const unsigned threads = 32u * (unsigned)(b - a);
        if (dout_dtype == NGP_F16)
            hash_bwd_kernel<__half><<<grid, threads, smem_bytes(b - a, 4), st>>>(xyz, (const __half*)dout, *layout, grad_table, n, dyn, a, b, found_inf_or_null, n_groups > 1);
        else
            hash_bwd_kernel<float><<<grid, threads, smem_bytes(b - a, 8), st>>>(xyz, (const float*)dout, *layout, grad_table, n, dyn, a, b, found_inf_or_null, n_groups > 1);
        NGP_LAUNCHED("hash_bwd_kernel");
    }
    return 0;
}

int ngp_hash_bwd_level_groups(const ngp_hash_layout* layout, int level_begin, int level_end, int64_t l2_bytes,
                              int32_t* bounds) {
    // greedy: a group grows while its fp32 gradient slice stays within the budget; a level larger than the budget
    // is a group of its own; l2_bytes <= 0 (unknown) gives one group
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(level_begin >= 0 && level_begin < level_end && level_end <= layout->n_levels, "bad level range");
    NGP_REQUIRE(bounds != nullptr, "null pointer");
    const int64_t budget = l2_bytes * kL2BudgetNum / kL2BudgetDen;
    int n_groups = 0;
    int64_t used = 0;
    bounds[0] = level_begin;
    for (int l = level_begin; l < level_end; ++l) {
        const int64_t bytes = (int64_t)layout->map_sizes[l] * layout->feat_dim * (int64_t)sizeof(float);
        if (l > bounds[n_groups] && l2_bytes > 0 && used + bytes > budget) {
            bounds[++n_groups] = l;
            used = 0;
        }
        used += bytes;
    }
    bounds[++n_groups] = level_end;
    return n_groups;
}

int ngp_hash_encode_bwd_input(const float* xyz, const void* table, const void* dout, int dtype,
                              const ngp_hash_layout* layout, float* dx, int64_t n, void* stream) {
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(dtype == NGP_F32 || dtype == NGP_F16, "bad dtype");
    if (n == 0) return 0;
    NGP_REQUIRE(xyz && table && dout && dx, "null pointer");
    NGP_REQUIRE(layout->feat_dim == 2, "dL/dx is implemented for feature_per_level == 2");
    return ngp_hash_encode_bwd_input_dyn(xyz, table, dout, dtype, layout, dx, n, nullptr, nullptr, stream);
}

int ngp_hash_encode_bwd_input_dyn(const float* xyz, const void* table, const void* dout, int dtype,
                                  const ngp_hash_layout* layout, float* dx, int64_t n, const int32_t* n_dev,
                                  const float* aabb6, void* stream) {
    const Dyn dyn = make_dyn(n_dev, aabb6);
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(dtype == NGP_F32 || dtype == NGP_F16, "bad dtype");
    if (n == 0) return 0;
    NGP_REQUIRE(xyz && table && dout && dx, "null pointer");
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaStream_t st = ngp::as_stream(stream);
    if (layout->feat_dim != 2) {
        if (dtype == NGP_F16)
            hash_bwd_input_generic_kernel<__half><<<grid, 256, 0, st>>>(xyz, (const __half*)table, (const __half*)dout, *layout, dx, n, dyn);
        else
            hash_bwd_input_generic_kernel<float><<<grid, 256, 0, st>>>(xyz, (const float*)table, (const float*)dout, *layout, dx, n, dyn);
        NGP_LAUNCHED("hash_bwd_input_generic_kernel");
        return 0;
    }
    if (dtype == NGP_F16)
        hash_bwd_input_kernel<__half><<<grid, 256, 0, st>>>(xyz, (const __half*)table, (const __half*)dout, *layout, dx, n, dyn);
    else
        hash_bwd_input_kernel<float><<<grid, 256, 0, st>>>(xyz, (const float*)table, (const float*)dout, *layout, dx, n, dyn);
    NGP_LAUNCHED("hash_bwd_input_kernel");
    return 0;
}

}  // extern "C"
