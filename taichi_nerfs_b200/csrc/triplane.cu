// triplane.cu — tri-plane position encoding: forward (static and device-counted rows) and table backward.
//
// Semantics: triplane_encoder_kernel of the reference (modules/triplane.py:35-98) and its Taichi autodiff
// (:186-197).  Per-level scale/resolution come from the host-built ngp_triplane_layout (the same fp32
// derivation as the hash levels, taichi_nerfs_b200/layout.py).  Arithmetic is strict fp32 in the reference's
// source order (f_mul/f_add/... of common.cuh), so the forward is bit-identical to oracle/triplane.c.
//
// One deliberate deviation: the reference has no bounds check (commented out at triplane.py:88-89).  The
// max_res-grid coordinate is clamped to [0, max_res-1]; that is the identity for every position in [0, 1], and no
// finite, infinite or NaN position can read or write outside the table.  floor() and the cast to the max_res grid
// are saturating conversions (cvt.rmi / cvt.rzi: negative -> 0, NaN -> 0), which equal the reference's casts
// wherever those are defined.
//
// GPU mapping, forward.  One thread per (sample, level), level fastest.  A thread computes the sample's three axis
// coordinates at its level once (floor, fraction and both max_res-grid corners per axis: every axis is the first
// coordinate of one plane and the second of another), then gathers the 3 planes x 4 corners: the F features of an
// entry are contiguous, so each gather is one float4 (F = 4) or float2 (F = 2) load.  Output column j*L + level of
// row i (the reference's feature-major order, triplane.py:43-45) is written straight from registers: for fixed j the
// L level-threads of a sample store L consecutive floats, so at L >= 8 every store instruction covers whole 32-byte
// sectors and a shared-memory transpose would save nothing.
//
// Backward (one kernel for the static and the device-counted entry, see triplane_bwd_kernel): lf[.] (the three plane
// features) is recomputed, not saved by the forward.  Saving it costs 3*L*F*4 B per sample written by the forward and
// read back (384 B at L=8 F=4; 384 MB for a 1 M-sample batch, held from forward to backward); recomputing re-gathers
// 12*L*F*4 B (1536 B) per sample, of which the coarse levels are L2 hits.  Rows whose dL/dout is zero in all F columns
// of a level (samples behind the termination point) issue no atomics.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kBwdThreads = 128;   // the F = 4 backward holds 48 accumulators (168 registers): 3 blocks of 128 fit an SM
constexpr int kBwdRun = 8;         // consecutive rows one backward thread walks (16 measured 2-4 % slower)

struct Box {
    float lo[3], span[3];
    int normalize;
};

Box make_box(const float* aabb6) {
    Box b;
    b.normalize = aabb6 != nullptr;
    for (int k = 0; k < 3; ++k) {
        b.lo[k] = aabb6 ? aabb6[k] : 0.0f;
        b.span[k] = aabb6 ? aabb6[3 + k] : 1.0f;
    }
    return b;
}

template <int F>
struct Vec;
template <>
struct Vec<2> {
    using type = float2;
    __device__ static __forceinline__ float get(const float2& v, int j) { return j == 0 ? v.x : v.y; }
};
template <>
struct Vec<4> {
    using type = float4;
    __device__ static __forceinline__ float get(const float4& v, int j) {
        return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w;
    }
};

// Per-level geometry of one sample: for each axis the two max_res-grid coordinates and the two linear weights
// (1 - frac, frac).  triplane.py:51-76.
struct Axes {
    uint32_t ori[3][2];
    float a[3][2];
};

__device__ __forceinline__ Axes sample_axes(const ngp_triplane_layout& lay, int level, const float x[3]) {
    Axes ax;
    const uint32_t res = lay.resolutions[level];
    const float res_m1 = __uint2float_rn(res - 1u);
    const float res_f = __uint2float_rn(res);
    const uint32_t mr = (uint32_t)lay.max_res;
    const float mr_m1 = __uint2float_rn(mr - 1u);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float p = f_add(f_mul(x[k], res_m1), 0.5f);     // pos = xyz*(res-1) + 0.5            (:56)
        const uint32_t g = __float2uint_rd(p);                // pos_grid = u32(floor(pos))         (:57)
        const float fr = f_sub(p, __uint2float_rn(g));        // pos -= f32(pos_grid)               (:58)
        ax.a[k][0] = f_sub(1.0f, fr);                          // w *= 1 - pos | w *= pos            (:67,:70)
        ax.a[k][1] = fr;
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            // u32(f32(g_c / res) * (max_res-1)), clamped to the grid                               (:73-76)
            const uint32_t o = __float2uint_rz(f_mul(f_div(__uint2float_rn(g + (uint32_t)b), res_f), mr_m1));
            ax.ori[k][b] = o < mr - 1u ? o : mr - 1u;
        }
    }
    return ax;
}

// plane fd pairs axis fd (first coordinate, stride 1) with axis (fd+1)%3 (second, stride max_res):
// (x,y), (y,z), (z,x), triplane.py:46-50,78-87.  Corner c: bit 0 picks the first axis' g+1, bit 1 the second's.
__device__ __forceinline__ int64_t corner_entry(const ngp_triplane_layout& lay, const uint32_t ori[3][2], int fd,
                                                int c) {
    const int s = fd == 2 ? 0 : fd + 1;
    const int64_t mr = lay.max_res;
    const int64_t index = (int64_t)ori[fd][c & 1] + (int64_t)ori[s][c >> 1] * mr;
    return ((int64_t)fd * mr * mr + index) * lay.feat_dim;
}

__device__ __forceinline__ float corner_weight(const Axes& ax, int fd, int c) {
    const int s = fd == 2 ? 0 : fd + 1;
    return f_mul(ax.a[fd][c & 1], ax.a[s][c >> 1]);   // ((1 * a_d0) * a_d1), triplane.py:61-70
}

__device__ __forceinline__ void load_position(const float* xyz, int64_t i, const Box& box, float x[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        x[k] = xyz[i * 3 + k];
        if (box.normalize) x[k] = f_div(f_sub(x[k], box.lo[k]), box.span[k]);  // networks.py:144
    }
}

// lf[fd][j] = sum over corners 0..3 of w_c[fd] * table[entry + j], from 0 in corner order (triplane.py:90-92)
template <int F>
__device__ __forceinline__ void plane_features(const float* __restrict__ table, const ngp_triplane_layout& lay,
                                               const Axes& ax, float lf[3][F]) {
    using V = typename Vec<F>::type;
#pragma unroll
    for (int fd = 0; fd < 3; ++fd) {
#pragma unroll
        for (int j = 0; j < F; ++j) lf[fd][j] = 0.0f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const V t = __ldg(reinterpret_cast<const V*>(table + corner_entry(lay, ax.ori, fd, c)));
            const float w = corner_weight(ax, fd, c);
#pragma unroll
            for (int j = 0; j < F; ++j) lf[fd][j] = f_add(lf[fd][j], f_mul(w, Vec<F>::get(t, j)));
        }
    }
}

__device__ __forceinline__ int64_t rows(int64_t n_max, const int32_t* n_dev) {
    if (n_dev == nullptr) return n_max;
    const int64_t v = (int64_t)*n_dev;
    return v < n_max ? (v < 0 ? 0 : v) : n_max;
}

template <int F>
__global__ void __launch_bounds__(kThreads) triplane_fwd_kernel(const float* __restrict__ xyz,
                                                                const float* __restrict__ table,
                                                                const __grid_constant__ ngp_triplane_layout lay,
                                                                float* __restrict__ out, int64_t n_max,
                                                                const int32_t* __restrict__ n_dev, const Box box) {
    const int L = lay.n_levels;
    const int64_t n = rows(n_max, n_dev);
    const int64_t gid = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    const int64_t i = gid / L;
    if (i >= n) return;
    const int level = (int)(gid - i * L);
    float x[3];
    load_position(xyz, i, box, x);
    const Axes ax = sample_axes(lay, level, x);
    float lf[3][F];
    plane_features<F>(table, lay, ax, lf);
    float* o = out + i * (int64_t)(L * F) + level;
#pragma unroll
    for (int j = 0; j < F; ++j) o[j * L] = f_mul(f_mul(lf[0][j], lf[1][j]), lf[2][j]);  // ((1*lf0)*lf1)*lf2 (:94-98)
}

// Non-finite test that survives fast-math style folding: false for +-inf and NaN.
__device__ __forceinline__ bool finite(float v) { return fabsf(v) < INFINITY; }

// Table backward.  A thread owns one level of kBwdRun consecutive rows (level fastest, so the L level-threads of a
// chunk read L consecutive floats of dout per feature: whole 32-byte sectors at L >= 8).  Rows of one ray are
// consecutive in the march output, and at the coarse levels many of them fall into the same cell of a plane, so
// the finished per-corner contributions w_c * dlf are kept in registers while a plane's four entries do not
// change and are scattered once, when they change or the chunk ends (dlf differs from row to row - it holds the
// other two planes' features - so it is the contribution that is accumulated, not a weight sum).  "Do not
// change" is judged on the max_res-grid coordinates themselves, so two level cells that land on the same entries
// (possible at the finest level, where res == max_res) share one flush.
// Rows >= min(n_max, *n_dev) are never read; a chunk wholly beyond the count exits on the first comparison.
template <int F>
__global__ void __launch_bounds__(kBwdThreads) triplane_bwd_kernel(const float* __restrict__ xyz,
                                                                const float* __restrict__ table,
                                                                const float* __restrict__ dout,
                                                                const __grid_constant__ ngp_triplane_layout lay,
                                                                float* __restrict__ grad_table, int64_t n_max,
                                                                const int32_t* __restrict__ n_dev, const Box box,
                                                                int32_t* __restrict__ found_inf) {
    using V = typename Vec<F>::type;
    const int L = lay.n_levels;
    const int64_t n = rows(n_max, n_dev);
    const int64_t gid = (int64_t)blockIdx.x * kBwdThreads + threadIdx.x;
    const int64_t chunk = gid / L;
    const int64_t i0 = chunk * kBwdRun;
    if (i0 >= n) return;
    const int level = (int)(gid - chunk * L);
    const int64_t i1 = i0 + kBwdRun < n ? i0 + kBwdRun : n;

    uint32_t pori[3][2] = {};  // max_res-grid coordinates of the entries the accumulators belong to
    float acc[3][4][F];       // [plane][corner][feature]
    bool pending = false;
    bool bad = false;         // a non-finite value handed to a reduction: GradScaler's inf check at the source
    auto flush = [&](int fd) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            V g;
            float* gp = reinterpret_cast<float*>(&g);
#pragma unroll
            for (int j = 0; j < F; ++j) {
                gp[j] = acc[fd][c][j];
                bad = bad || !finite(gp[j]);
            }
            atomicAdd(reinterpret_cast<V*>(grad_table + corner_entry(lay, pori, fd, c)), g);  // red.global.add.v{2,4}.f32
        }
    };
#pragma unroll 1
    for (int64_t i = i0; i < i1; ++i) {
        float dy[F];
        bool any = false;
#pragma unroll
        for (int j = 0; j < F; ++j) {
            dy[j] = dout[i * (int64_t)(L * F) + j * L + level];
            any |= dy[j] != 0.0f;
        }
        if (!any) continue;   // samples behind the termination point: nothing gathered, nothing scattered
        float x[3];
        load_position(xyz, i, box, x);
        const Axes ax = sample_axes(lay, level, x);
        float lf[3][F];
        plane_features<F>(table, lay, ax, lf);
        // adjoints of out = ((1*lf0)*lf1)*lf2 in the order Taichi's reverse pass forms them (triplane.py:94-98)
        float dlf[3][F];
#pragma unroll
        for (int j = 0; j < F; ++j) {
            const float d2 = dy[j] * lf[2][j];
            dlf[2][j] = dy[j] * (lf[0][j] * lf[1][j]);
            dlf[1][j] = d2 * lf[0][j];
            dlf[0][j] = d2 * lf[1][j];
        }
        bool moved[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) moved[k] = ax.ori[k][0] != pori[k][0] || ax.ori[k][1] != pori[k][1];
#pragma unroll
        for (int fd = 0; fd < 3; ++fd) {
            const int s = fd == 2 ? 0 : fd + 1;
            const bool fresh = !pending || moved[fd] || moved[s];
            if (pending && fresh) flush(fd);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float w = corner_weight(ax, fd, c);
#pragma unroll
                for (int j = 0; j < F; ++j) acc[fd][c][j] = fresh ? w * dlf[fd][j] : acc[fd][c][j] + w * dlf[fd][j];
            }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            pori[k][0] = ax.ori[k][0];
            pori[k][1] = ax.ori[k][1];
        }
        pending = true;
    }
    if (pending) {
#pragma unroll
        for (int fd = 0; fd < 3; ++fd) flush(fd);
    }
    if (bad && found_inf != nullptr) *found_inf = 1;
}

int check_layout(const ngp_triplane_layout* lay) {
    NGP_REQUIRE(lay != nullptr, "null layout");
    NGP_REQUIRE(lay->n_levels >= 1 && lay->n_levels <= NGP_MAX_LEVELS, "n_levels must be in [1, 16]");
    NGP_REQUIRE(lay->feat_dim == 2 || lay->feat_dim == 4, "feature_per_level must be 2 or 4");
    NGP_REQUIRE(lay->max_res >= 2 && lay->max_res <= NGP_TRIPLANE_MAX_RES, "max_res must be in [2, 16384]");
    for (int l = 0; l < lay->n_levels; ++l)
        NGP_REQUIRE(lay->resolutions[l] >= 1u, "level resolution must be >= 1");
    return 0;
}

bool aligned(const void* p, int F) { return (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(4 * F - 1)) == 0; }

unsigned blocks(int64_t n, int L, int threads = kThreads) { return (unsigned)((n * L + threads - 1) / threads); }

}  // namespace

extern "C" {

int ngp_triplane_encode_fwd(const float* xyz, const float* table, const ngp_triplane_layout* layout, float* out,
                            int64_t n, const float* aabb6, void* stream) {
    return ngp_triplane_encode_fwd_dyn(xyz, table, layout, out, n, nullptr, aabb6, stream);
}

int ngp_triplane_encode_fwd_dyn(const float* xyz, const float* table, const ngp_triplane_layout* layout, float* out,
                                int64_t n_max, const int32_t* n_dev, const float* aabb6, void* stream) {
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n_max >= 0, "negative n");
    if (n_max == 0) return 0;
    NGP_REQUIRE(xyz && table && out, "null pointer");
    NGP_REQUIRE(aligned(table, layout->feat_dim), "table must be aligned to one entry (4*F bytes)");
    const Box box = make_box(aabb6);
    cudaStream_t st = ngp::as_stream(stream);
    const unsigned grid = blocks(n_max, layout->n_levels);
    if (layout->feat_dim == 4)
        triplane_fwd_kernel<4><<<grid, kThreads, 0, st>>>(xyz, table, *layout, out, n_max, n_dev, box);
    else
        triplane_fwd_kernel<2><<<grid, kThreads, 0, st>>>(xyz, table, *layout, out, n_max, n_dev, box);
    NGP_LAUNCHED("triplane_fwd_kernel");
    return 0;
}

int ngp_triplane_encode_bwd(const float* xyz, const float* table, const float* dout,
                            const ngp_triplane_layout* layout, float* grad_table, int64_t n, void* stream) {
    return ngp_triplane_encode_bwd_dyn(xyz, table, dout, layout, grad_table, n, nullptr, nullptr, nullptr, stream);
}

int ngp_triplane_encode_bwd_dyn(const float* xyz, const float* table, const float* dout,
                                const ngp_triplane_layout* layout, float* grad_table, int64_t n_max,
                                const int32_t* n_dev, const float* aabb6, int32_t* found_inf_or_null, void* stream) {
    if (int rc = check_layout(layout)) return rc;
    NGP_REQUIRE(n_max >= 0, "negative n");
    if (n_max == 0) return 0;
    NGP_REQUIRE(xyz && table && dout && grad_table, "null pointer");
    NGP_REQUIRE(aligned(table, layout->feat_dim) && aligned(grad_table, layout->feat_dim),
                "table and grad_table must be aligned to one entry (4*F bytes)");
    const Box box = make_box(aabb6);
    cudaStream_t st = ngp::as_stream(stream);
    const unsigned grid = blocks((n_max + kBwdRun - 1) / kBwdRun, layout->n_levels, kBwdThreads);
    if (layout->feat_dim == 4)
        triplane_bwd_kernel<4><<<grid, kBwdThreads, 0, st>>>(xyz, table, dout, *layout, grad_table, n_max, n_dev, box,
                                                          found_inf_or_null);
    else
        triplane_bwd_kernel<2><<<grid, kBwdThreads, 0, st>>>(xyz, table, dout, *layout, grad_table, n_max, n_dev, box,
                                                          found_inf_or_null);
    NGP_LAUNCHED("triplane_bwd_kernel");
    return 0;
}

}  // extern "C"
