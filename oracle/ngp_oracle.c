/*
 * ngp_oracle.c — CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * A plain-C, strict-fp32 restatement of the Instant-NGP hot path of
 * taichi-dev/taichi-nerfs.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / `--impl reference` legs may load this library; the product
 * path (taichi_nerfs_b200/ + modules/) never does and fails loudly without its
 * CUDA library.
 *
 * PARITY PIN STATUS: the reference ships NO tests, golden vectors or fixtures
 * for these kernels and its runtime (Taichi) cannot be imported in the build
 * container, so per-kernel parity is "unpinned by the reference".  What is
 * pinned: the hash layout constants printed in notebooks/pipeline.ipynb
 * (tests/test_layout.py) and an end-to-end render of the reference's shipped,
 * trained Lego deployment model through this oracle (oracle/kat_lego.py ->
 * tests/golden/lego_kat.png: the yellow bulldozer comes out; tests/test_kat_lego.py).
 *
 * Every function cites the reference file:line it follows.  Build:
 *   gcc -O2 -march=x86-64-v3 -ffp-contract=off -fopenmp -shared -fPIC
 * `-ffp-contract=off` matters: marching must be bit-reproducible on the GPU
 * (which uses __fmul_rn/__fadd_rn/__fdiv_rn), so no FMA contraction anywhere.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/ngp_b200.h"

typedef _Float16 f16;

static inline float rh(float x) { return (float)(f16)x; } /* round to fp16 and back */

/* ------------------------------------------------------------------------- */
/* a1  ray_aabb_intersect              modules/intersection.py:8-37           */
/* ------------------------------------------------------------------------- */
#define NEAR_DISTANCE 0.01f /* modules/utils.py:13 */

int ngp_ray_aabb_intersect_cpu(const float* rays_o, const float* rays_d, float scale,
                               float* hits_t, int64_t n_rays) {
    /* half_size = (xyz_max - xyz_min)/2 = scale ; center = 0  (intersection.py:15-18) */
    const float half = (scale - (-scale)) / 2.0f;
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < n_rays; ++r) {
        float t1 = -INFINITY, t2 = INFINITY;
        for (int k = 0; k < 3; ++k) {
            const float o = rays_o[r * 3 + k], d = rays_d[r * 3 + k];
            const float inv = 1.0f / d;                 /* :24 */
            const float tmin = (0.0f - half - o) * inv; /* :26 */
            const float tmax = (0.0f + half - o) * inv; /* :27 */
            const float lo = fminf(tmin, tmax), hi = fmaxf(tmin, tmax);
            t1 = fmaxf(t1, lo); /* :31 */
            t2 = fminf(t2, hi); /* :32 */
        }
        if (t2 > 0.0f && t2 < INFINITY) { /* :34; a ray with no finite far hit (zero or NaN direction) misses */
            hits_t[r * 2 + 0] = fmaxf(t1, NEAR_DISTANCE);
            hits_t[r * 2 + 1] = t2;
        } else {
            hits_t[r * 2 + 0] = -1.0f;
            hits_t[r * 2 + 1] = -1.0f;
        }
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* marching helpers                    modules/utils.py:12-117                */
/* ------------------------------------------------------------------------- */
#define SQRT3_MAX_SAMPLES ((float)(1.7320508075688772 / 1024)) /* utils.py:15 */
#define SQRT3_2 ((float)(1.7320508075688772 * 2))              /* utils.py:16 */

static inline float calc_dt(float t, float esf, int grid_size, float scale) { /* utils.py:54-57 */
    const float hi = SQRT3_2 * scale / (float)grid_size;
    const float v = t * esf;
    return fminf(fmaxf(v, SQRT3_MAX_SAMPLES), hi);
}

/* The next march position t + dt, or +inf when the add does not increase t: near t = dt * 2^24 the fp32 sum rounds
 * back to t, and a NaN t never compares greater.  Every march loop advances only through this, so each iteration
 * strictly increases a finite t or ends the ray (+inf fails `t < t2` and `tn < t_target`); fp32 has finitely many
 * values, so every loop ends.  The reference adds unconditionally and loops forever on such rays
 * (ray_march.py:64,72-74). */
static inline float march_advance(float t, float dt) {
    const float tn = t + dt;
    return tn > t ? tn : INFINITY;
}

static inline int frexp_bit(float x) { /* utils.py:60-75 */
    int exponent = 0;
    if (x != 0.0f) {
        uint32_t bits;
        memcpy(&bits, &x, 4);
        exponent = (int)((bits & 0x7f800000u) >> 23) - 127;
        bits &= 0x7fffffu;
        bits |= 0x3f800000u;
        float frac;
        memcpy(&frac, &bits, 4);
        if (frac < 0.5f) exponent -= 1;
        else if (frac > 1.0f) exponent += 1;
    }
    return exponent;
}

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

static inline int mip_from_pos(float x, float y, float z, int cascades) { /* utils.py:78-84 */
    const float mx = fmaxf(fmaxf(fabsf(x), fabsf(y)), fabsf(z));
    const int exponent = frexp_bit(mx) + 1;
    return imin(cascades - 1, imax(0, exponent));
}
static inline int mip_from_dt(float dt, int grid_size, int cascades) { /* utils.py:87-92 */
    const int exponent = frexp_bit(dt * (float)grid_size);
    return imin(cascades - 1, imax(0, exponent));
}
static inline uint32_t expand_bits(uint32_t v) { /* utils.py:95-100 */
    v = (v * 0x00010001u) & 0xFF0000FFu;
    v = (v * 0x00000101u) & 0x0F00F00Fu;
    v = (v * 0x00000011u) & 0xC30C30C3u;
    v = (v * 0x00000005u) & 0x49249249u;
    return v;
}
static inline uint32_t morton3d(uint32_t x, uint32_t y, uint32_t z) { /* utils.py:103-107 */
    return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2);
}
static inline int32_t morton3d_invert1(uint32_t x) { /* utils.py:110-117 */
    x = x & 0x49249249u;
    x = (x | (x >> 2)) & 0xc30c30c3u;
    x = (x | (x >> 4)) & 0x0f00f00fu;
    x = (x | (x >> 8)) & 0xff0000ffu;
    x = (x | (x >> 16)) & 0x0000ffffu;
    return (int32_t)x;
}
static inline float fsign(float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); }

typedef struct {
    float o[3], d[3], dinv[3];
    int cascades, grid_size;
    float scale, esf;
    const uint8_t* bits;
} march_ctx;

/* One iteration body shared by all marching loops (ray_march.py:45-74, 86-123, 226-266).
 * Returns 1 if the cell at t is occupied (then *dt_out is the step), else advances *t
 * to the first step past the cell exit and returns 0. */
static inline int march_step(const march_ctx* c, float* t, float* xyz, float* dt_out) {
    const int gs = c->grid_size;
    const float gsf = (float)gs;
    const float tt = *t;
    xyz[0] = c->o[0] + tt * c->d[0];
    xyz[1] = c->o[1] + tt * c->d[1];
    xyz[2] = c->o[2] + tt * c->d[2];
    const float dt = calc_dt(tt, c->esf, gs, c->scale);
    const int mip = imax(mip_from_pos(xyz[0], xyz[1], xyz[2], c->cascades),
                         mip_from_dt(dt, gs, c->cascades));
    const float mip_bound = fminf(ldexpf(1.0f, mip - 1), c->scale); /* pow(2, mip-1) */
    const float mip_bound_inv = 1.0f / mip_bound;
    float nxyz[3];
    uint32_t u[3];
    for (int k = 0; k < 3; ++k) {
        float v = 0.5f * (xyz[k] * mip_bound_inv + 1.0f) * gsf;
        v = fminf(fmaxf(v, 0.0f), gsf - 1.0f);
        nxyz[k] = v;
        u[k] = (uint32_t)v;
    }
    const uint32_t idx = (uint32_t)mip * (uint32_t)(gs * gs * gs) + morton3d(u[0], u[1], u[2]);
    const int occ = c->bits[idx >> 3] & (1u << (idx & 7u));
    *dt_out = dt;
    if (occ) return 1;
    const float gs_inv = 1.0f / gsf;
    float tmin = INFINITY;
    for (int k = 0; k < 3; ++k) {
        const float tx =
            (((nxyz[k] + 0.5f + 0.5f * fsign(c->d[k])) * gs_inv * 2.0f - 1.0f) * mip_bound - xyz[k]) *
            c->dinv[k];
        tmin = fminf(tmin, tx);
    }
    const float t_target = tt + fmaxf(0.0f, tmin);
    float tn = march_advance(tt, calc_dt(tt, c->esf, gs, c->scale));
    while (tn < t_target) tn = march_advance(tn, calc_dt(tn, c->esf, gs, c->scale));
    *t = tn;
    return 0;
}

static inline void march_ctx_init(march_ctx* c, const float* o, const float* d, int cascades,
                                  int grid_size, float scale, float esf, const uint8_t* bits) {
    for (int k = 0; k < 3; ++k) {
        c->o[k] = o[k];
        c->d[k] = d[k];
        c->dinv[k] = 1.0f / d[k];
    }
    c->cascades = cascades;
    c->grid_size = grid_size;
    c->scale = scale;
    c->esf = esf;
    c->bits = bits;
}

/* ------------------------------------------------------------------------- */
/* a2  raymarching_train_kernel        modules/ray_march.py:8-123             */
/* ------------------------------------------------------------------------- */
static inline float march_train_t0(const float* hits_t, const float* noise, int64_t r, float esf,
                                   int grid_size, float scale) {
    float t1 = hits_t[r * 2 + 0];
    if (t1 >= 0.0f) { /* :36-38 */
        const float dt = calc_dt(t1, esf, grid_size, scale);
        t1 += dt * noise[r];
    }
    return t1;
}

int ngp_raymarching_train_count_cpu(const float* rays_o, const float* rays_d, const float* hits_t,
                                    const uint8_t* density_bitfield, const float* noise,
                                    int cascades, int grid_size, float scale, float exp_step_factor,
                                    int max_samples, int32_t* counter, int32_t* rays_a,
                                    int64_t n_rays) {
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t r = 0; r < n_rays; ++r) {
        march_ctx c;
        march_ctx_init(&c, rays_o + r * 3, rays_d + r * 3, cascades, grid_size, scale,
                       exp_step_factor, density_bitfield);
        const float t2 = hits_t[r * 2 + 1];
        float t = march_train_t0(hits_t, noise, r, exp_step_factor, grid_size, scale);
        int n = 0;
        float xyz[3], dt;
        while (0.0f <= t && t < t2 && n < max_samples) { /* :43 */
            if (march_step(&c, &t, xyz, &dt)) {
                t = march_advance(t, dt);
                n += 1;
            }
        }
        rays_a[r * 3 + 0] = (int32_t)r;
        rays_a[r * 3 + 2] = n;
    }
    /* deterministic replacement of the atomics at :76-81: exclusive scan in ray order */
    int64_t total = 0;
    for (int64_t r = 0; r < n_rays; ++r) {
        rays_a[r * 3 + 1] = (int32_t)total;
        total += rays_a[r * 3 + 2];
    }
    counter[0] = (int32_t)total;
    counter[1] = (int32_t)n_rays;
    return 0;
}

int ngp_raymarching_train_write_cpu(const float* rays_o, const float* rays_d, const float* hits_t,
                                    const uint8_t* density_bitfield, const float* noise,
                                    int cascades, int grid_size, float scale, float exp_step_factor,
                                    int32_t* counter, int32_t* rays_a, float* xyzs, float* dirs,
                                    float* deltas, float* ts, int64_t n_rays, int64_t capacity) {
    /* rays that do not fit form a suffix (starts are monotone): clamp the total first */
    for (int64_t r = 0; r < n_rays; ++r)
        if ((int64_t)rays_a[r * 3 + 1] + rays_a[r * 3 + 2] > capacity) {
            if (rays_a[r * 3 + 1] < counter[0]) counter[0] = rays_a[r * 3 + 1];
            break;
        }
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t r = 0; r < n_rays; ++r) {
        const int64_t start = rays_a[r * 3 + 1];
        const int n = rays_a[r * 3 + 2];
        if (start + n > capacity) {
            rays_a[r * 3 + 2] = 0;
            continue;
        }
        march_ctx c;
        march_ctx_init(&c, rays_o + r * 3, rays_d + r * 3, cascades, grid_size, scale,
                       exp_step_factor, density_bitfield);
        const float t2 = hits_t[r * 2 + 1];
        float t = march_train_t0(hits_t, noise, r, exp_step_factor, grid_size, scale);
        int s = 0;
        float xyz[3], dt;
        while (t < t2 && s < n) { /* :86 */
            if (march_step(&c, &t, xyz, &dt)) {
                const int64_t i = start + s;
                xyzs[i * 3 + 0] = xyz[0];
                xyzs[i * 3 + 1] = xyz[1];
                xyzs[i * 3 + 2] = xyz[2];
                dirs[i * 3 + 0] = c.d[0];
                dirs[i * 3 + 1] = c.d[1];
                dirs[i * 3 + 2] = c.d[2];
                ts[i] = t;
                deltas[i] = dt;
                t = march_advance(t, dt);
                s += 1;
            }
        }
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a3  raymarching_test_kernel         modules/ray_march.py:197-268           */
/* ------------------------------------------------------------------------- */
int ngp_raymarching_test_cpu(const float* rays_o, const float* rays_d, float* hits_t,
                             const int64_t* alive_indices, const uint8_t* density_bitfield,
                             int cascades, int grid_size, float scale, float exp_step_factor,
                             int max_samples, int64_t* ray_indices, uint8_t* valid_mask,
                             float* deltas, float* ts, int32_t* samples_counter, int64_t n_alive) {
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t n = 0; n < n_alive; ++n) {
        const int64_t r = alive_indices[n];
        march_ctx c;
        march_ctx_init(&c, rays_o + r * 3, rays_d + r * 3, cascades, grid_size, scale,
                       exp_step_factor, density_bitfield);
        float t = hits_t[r * 2 + 0];
        const float t2 = hits_t[r * 2 + 1];
        int s = 0;
        const int64_t base = n * (int64_t)max_samples;
        float xyz[3], dt;
        while (0.0f < t && t < t2 && s < max_samples) { /* :226 (strict 0 < t) */
            if (march_step(&c, &t, xyz, &dt)) {
                const int64_t i = base + s;
                ray_indices[i] = r;
                valid_mask[i] = 1;
                ts[i] = t;
                deltas[i] = dt;
                t = march_advance(t, dt);
                hits_t[r * 2 + 0] = t; /* :257 */
                s += 1;
            }
        }
        samples_counter[n] = s;
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a4/a5  hash encoder   modules/hash_encoder.py:43-143, hash_encoder_half.py  */
/* ------------------------------------------------------------------------- */
static inline uint32_t fast_hash(const uint32_t p[3]) { /* hash_encoder.py:43-51 */
    return (p[0] * 1u) ^ (p[1] * 2654435761u) ^ (p[2] * 805459861u);
}
static inline uint32_t under_hash(const uint32_t p[3], uint32_t res) { /* hash_encoder.py:53-60 */
    uint32_t result = 0, stride = 1;
    for (int i = 0; i < 3; ++i) {
        result += p[i] * stride;
        stride *= res;
    }
    return result;
}

/* grid coordinate and fractional position of xyz at one level (hash_encoder.py:108-110) */
static inline void hash_cell(const float* xyz, float scale, int frac_f16, uint32_t g[3], float pos[3]) {
    for (int d = 0; d < 3; ++d) {
        const float p = xyz[d] * scale + 0.5f; /* hash_encoder.py:108 */
        const float fl = floorf(p);
        g[d] = (uint32_t)(int32_t)fl;
        /* :110  pos -= cast(pos_grid, data_type); the half kernel casts the grid coordinate
         * to f16 first (hash_encoder_half.py:132, data_type = f16) — exact below 2048. */
        const float gf = frac_f16 ? rh((float)g[d]) : (float)g[d];
        pos[d] = p - gf;
    }
}

/* entry index (level-local, + offset) of corner c of cell g: bit d of c selects g[d] + 1 (:116-126) */
static inline uint32_t corner_entry(const ngp_hash_layout* lay, int level, const uint32_t g[3], int c) {
    uint32_t p[3];
    for (int d = 0; d < 3; ++d) p[d] = g[d] + (uint32_t)((c >> d) & 1);
    const uint32_t h = level < lay->begin_fast_hash_level ? under_hash(p, lay->resolutions[level]) : fast_hash(p);
    return (uint32_t)lay->offsets[level] + h % (uint32_t)lay->map_sizes[level]; /* :71, :134 */
}

/* per (sample, level): the 8 corner entry indices (level-local, + offset) and weights */
static inline void hash_corners(const float* xyz, const ngp_hash_layout* lay, int level, int frac_f16,
                                uint32_t idx[8], float w[8]) {
    float pos[3];
    uint32_t g[3];
    hash_cell(xyz, lay->scales[level], frac_f16, g, pos);
    for (int c = 0; c < 8; ++c) { /* :116-126 */
        float ww = 1.0f;
        for (int d = 0; d < 3; ++d) ww *= (c & (1 << d)) ? pos[d] : 1.0f - pos[d];
        idx[c] = corner_entry(lay, level, g, c);
        w[c] = ww;
    }
}

int ngp_hash_encode_fwd_cpu(const float* xyz, const void* table, const ngp_hash_layout* lay,
                            void* out, int dtype, int64_t n) {
    const int L = lay->n_levels, F = lay->feat_dim;
    if (F > 8) return -1;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        for (int l = 0; l < L; ++l) {
            uint32_t idx[8];
            float w[8];
            hash_corners(xyz + i * 3, lay, l, dtype == NGP_F16, idx, w);
            if (dtype == NGP_F32) {
                const float* tab = (const float*)table;
                float acc[8] = {0};
                for (int c = 0; c < 8; ++c)
                    for (int f = 0; f < F; ++f) acc[f] += w[c] * tab[(int64_t)idx[c] * F + f];
                for (int f = 0; f < F; ++f) ((float*)out)[i * L * F + l * F + f] = acc[f];
            } else {
                /* hash_encoder_half.py:159: local += cast(w * table[idx], f16); f16 accumulate */
                const f16* tab = (const f16*)table;
                f16 acc[8] = {0};
                for (int c = 0; c < 8; ++c)
                    for (int f = 0; f < F; ++f) {
                        const float prod = w[c] * (float)tab[(int64_t)idx[c] * F + f];
                        const f16 ph = (f16)prod;
                        acc[f] = (f16)((double)acc[f] + (double)ph); /* correctly rounded f16 add */
                    }
                for (int f = 0; f < F; ++f) ((f16*)out)[i * L * F + l * F + f] = acc[f];
            }
        }
    }
    return 0;
}

/* modules/hash_encoder.py:265-277 (autodiff) / hash_encoder_half.py:164-213 */
int ngp_hash_encode_bwd_cpu(const float* xyz, const void* dout, int dout_dtype,
                            const ngp_hash_layout* lay, float* grad_table, int64_t n) {
    const int L = lay->n_levels, F = lay->feat_dim;
    /* parallel over levels: levels own disjoint table ranges, so no atomics are needed and
     * the accumulation order (sample order) is deterministic */
#pragma omp parallel for schedule(dynamic, 1)
    for (int l = 0; l < L; ++l) {
        for (int64_t i = 0; i < n; ++i) {
            float dy[8];
            int any = 0;
            for (int f = 0; f < F; ++f) {
                dy[f] = dout_dtype == NGP_F16 ? (float)((const f16*)dout)[i * L * F + l * F + f]
                                              : ((const float*)dout)[i * L * F + l * F + f];
                any |= dy[f] != 0.0f;
            }
            if (!any) continue; /* hash_encoder_half.py:210 */
            uint32_t idx[8];
            float w[8];
            hash_corners(xyz + i * 3, lay, l, dout_dtype == NGP_F16, idx, w);
            for (int c = 0; c < 8; ++c)
                for (int f = 0; f < F; ++f) grad_table[(int64_t)idx[c] * F + f] += w[c] * dy[f];
        }
    }
    return 0;
}

/* d out / d xyz  (notebooks/autodiff.ipynb cell 2 semantics; reference returns None): the derivative of the
 * forward inside the cell of x, so with the fp16 table it is taken at the fraction the half forward uses,
 * p - f16(g) (hash_encoder_half.py:132-133), not at p - g. */
int ngp_hash_encode_bwd_input_cpu(const float* xyz, const void* table, const void* dout, int dtype,
                                  const ngp_hash_layout* lay, float* dx, int64_t n) {
    const int L = lay->n_levels, F = lay->feat_dim;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        double g[3] = {0, 0, 0};
        for (int l = 0; l < L; ++l) {
            const float scale = lay->scales[l];
            uint32_t cell[3];
            float pos[3];
            hash_cell(xyz + i * 3, scale, dtype == NGP_F16, cell, pos);
            for (int c = 0; c < 8; ++c) {
                const uint32_t idx = corner_entry(lay, l, cell, c);
                double v = 0;
                for (int f = 0; f < F; ++f) {
                    const int64_t e = (int64_t)idx * F + f, o = i * L * F + l * F + f;
                    const float tv = dtype == NGP_F16 ? (float)((const f16*)table)[e] : ((const float*)table)[e];
                    const float dy = dtype == NGP_F16 ? (float)((const f16*)dout)[o] : ((const float*)dout)[o];
                    v += (double)tv * dy;
                }
                for (int d = 0; d < 3; ++d) {
                    double wd = (c & (1 << d)) ? 1.0 : -1.0;
                    for (int e = 0; e < 3; ++e)
                        if (e != d) wd *= (c & (1 << e)) ? pos[e] : 1.0f - pos[e];
                    g[d] += wd * scale * v;
                }
            }
        }
        for (int d = 0; d < 3; ++d) dx[i * 3 + d] = (float)g[d];
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a6  dir_encoder                     modules/spherical_harmonics.py:16-42   */
/* ------------------------------------------------------------------------- */
static inline void sh16(float x, float y, float z, float* e) {
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

int ngp_dir_encode_cpu(const float* dirs, float* out, int64_t n) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) sh16(dirs[i * 3], dirs[i * 3 + 1], dirs[i * 3 + 2], out + i * 16);
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a7  MLP under autocast(fp16)   modules/networks.py:18-30,136-166,369-380    */
/* ------------------------------------------------------------------------- */
/* torch.autocast semantics restated: every nn.Linear runs with fp16 inputs and an fp16 copy
 * of the fp32 master weight, accumulates in fp32 (cuBLAS) and rounds its output to fp16;
 * ReLU / Sigmoid act on fp16; TruncExp and the direction normalisation run in fp32. */
typedef struct {
    float e[32];  /* fp16-rounded embedding                      */
    float h1[64]; /* relu(W1 e)            fp16-rounded          */
    float h[16];  /* W2 h1                 fp16-rounded          */
    float x3[32]; /* [sh16 | h]            fp16-rounded          */
    float h3[64], h4[64];
    float rgb[3]; /* sigmoid, fp16-rounded                       */
} mlp_act;

static inline void linear_h(const float* wh, const float* x, float* y, int out, int in, int relu) {
    for (int o = 0; o < out; ++o) {
        float acc = 0.0f;
        const float* wr = wh + o * in;
        for (int k = 0; k < in; ++k) acc += wr[k] * x[k];
        acc = rh(acc);
        y[o] = relu ? fmaxf(acc, 0.0f) : acc;
    }
}

static void mlp_forward_one(const float* const wh[5], const float* emb, const float* dir, mlp_act* a,
                            float* sigma) {
    for (int k = 0; k < 32; ++k) a->e[k] = rh(emb[k]);
    linear_h(wh[0], a->e, a->h1, 64, 32, 1);
    linear_h(wh[1], a->h1, a->h, 16, 64, 0);
    *sigma = expf(a->h[0]); /* TruncExp.forward, networks.py:22-24 */
    /* networks.py:162-163: d/|d| then (d+1)/2, fp32 */
    const float nrm = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
    float sh[16];
    sh16((dir[0] / nrm + 1.0f) / 2.0f, (dir[1] / nrm + 1.0f) / 2.0f, (dir[2] / nrm + 1.0f) / 2.0f, sh);
    for (int k = 0; k < 16; ++k) a->x3[k] = rh(sh[k]);
    for (int k = 0; k < 16; ++k) a->x3[16 + k] = a->h[k];
    linear_h(wh[2], a->x3, a->h3, 64, 32, 1);
    linear_h(wh[3], a->h3, a->h4, 64, 64, 1);
    float o[3];
    linear_h(wh[4], a->h4, o, 3, 64, 0);
    for (int k = 0; k < 3; ++k) a->rgb[k] = rh(1.0f / (1.0f + expf(-o[k])));
}

static float* round_weights(const ngp_mlp_weights* w) {
    float* wh = (float*)malloc(sizeof(float) * NGP_MLP_PARAMS);
    const float* src[5] = {w->w1, w->w2, w->w3, w->w4, w->w5};
    const int cnt[5] = {NGP_MLP_W1, NGP_MLP_W2, NGP_MLP_W3, NGP_MLP_W4, NGP_MLP_W5};
    int off = 0;
    for (int i = 0; i < 5; ++i) {
        for (int k = 0; k < cnt[i]; ++k) wh[off + k] = rh(src[i][k]);
        off += cnt[i];
    }
    return wh;
}

static inline float load_emb(const void* emb, int dtype, int64_t i) {
    return dtype == NGP_F16 ? (float)((const f16*)emb)[i] : ((const float*)emb)[i];
}

int64_t ngp_mlp_save_bytes_cpu(int64_t n) { return n * (int64_t)sizeof(mlp_act); }

int ngp_mlp_fwd_cpu(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w,
                    float* sigmas, void* rgbs_f16, void* save, int64_t n) {
    float* whb = round_weights(w);
    const float* wh[5] = {whb, whb + NGP_MLP_W1, whb + NGP_MLP_W1 + NGP_MLP_W2,
                          whb + NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3,
                          whb + NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3 + NGP_MLP_W4};
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        mlp_act local;
        mlp_act* a = save ? ((mlp_act*)save) + i : &local;
        float e[32];
        for (int k = 0; k < 32; ++k) e[k] = load_emb(emb, emb_dtype, i * 32 + k);
        mlp_forward_one(wh, e, dirs + i * 3, a, sigmas + i);
        for (int k = 0; k < 3; ++k) ((f16*)rgbs_f16)[i * 3 + k] = (f16)a->rgb[k];
    }
    free(whb);
    return 0;
}

/* backward of the autocast graph; weight grads accumulate in fp32 (the reference rounds each
 * weight grad to fp16 before the fp32 master .grad — a <=2^-11 relative difference) */
int ngp_mlp_bwd_cpu(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w,
                    const void* save, const float* dsigmas, const void* drgbs_f16, void* demb,
                    float* grad_w, int64_t n) {
    float* whb = round_weights(w);
    const float* wh[5] = {whb, whb + NGP_MLP_W1, whb + NGP_MLP_W1 + NGP_MLP_W2,
                          whb + NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3,
                          whb + NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3 + NGP_MLP_W4};
    const int goff[5] = {0, NGP_MLP_W1, NGP_MLP_W1 + NGP_MLP_W2, NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3,
                         NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3 + NGP_MLP_W4};
    int nthreads = 1;
#ifdef _OPENMP
    extern int omp_get_max_threads(void);
    extern int omp_get_thread_num(void);
    nthreads = omp_get_max_threads();
#endif
    double* gacc = (double*)calloc((size_t)nthreads * NGP_MLP_PARAMS, sizeof(double));
#pragma omp parallel
    {
        int tid = 0;
#ifdef _OPENMP
        tid = omp_get_thread_num();
#endif
        double* g = gacc + (size_t)tid * NGP_MLP_PARAMS;
#pragma omp for schedule(static)
        for (int64_t i = 0; i < n; ++i) {
            mlp_act local;
            const mlp_act* a;
            if (save) {
                a = ((const mlp_act*)save) + i;
            } else {
                float e[32], sg;
                for (int k = 0; k < 32; ++k) e[k] = load_emb(emb, emb_dtype, i * 32 + k);
                mlp_forward_one(wh, e, dirs + i * 3, &local, &sg);
                a = &local;
            }
            /* sigmoid backward, fp16 */
            float d_o[3];
            for (int k = 0; k < 3; ++k) {
                const float dy = (float)((const f16*)drgbs_f16)[i * 3 + k];
                d_o[k] = rh(dy * a->rgb[k] * (1.0f - a->rgb[k]));
            }
            float dh4[64], dh3[64], dx3[32], dh[16], dh1[64], de[32];
            /* layer 5: o = W5 h4 */
            for (int j = 0; j < 64; ++j) {
                float acc = 0.0f;
                for (int k = 0; k < 3; ++k) acc += d_o[k] * wh[4][k * 64 + j];
                dh4[j] = a->h4[j] > 0.0f ? rh(acc) : 0.0f;
            }
            for (int k = 0; k < 3; ++k)
                for (int j = 0; j < 64; ++j) g[goff[4] + k * 64 + j] += (double)d_o[k] * a->h4[j];
            /* layer 4 */
            for (int j = 0; j < 64; ++j) {
                float acc = 0.0f;
                for (int k = 0; k < 64; ++k) acc += dh4[k] * wh[3][k * 64 + j];
                dh3[j] = a->h3[j] > 0.0f ? rh(acc) : 0.0f;
            }
            for (int k = 0; k < 64; ++k)
                if (dh4[k] != 0.0f)
                    for (int j = 0; j < 64; ++j) g[goff[3] + k * 64 + j] += (double)dh4[k] * a->h3[j];
            /* layer 3 */
            for (int j = 0; j < 32; ++j) {
                float acc = 0.0f;
                for (int k = 0; k < 64; ++k) acc += dh3[k] * wh[2][k * 32 + j];
                dx3[j] = rh(acc);
            }
            for (int k = 0; k < 64; ++k)
                if (dh3[k] != 0.0f)
                    for (int j = 0; j < 32; ++j) g[goff[2] + k * 32 + j] += (double)dh3[k] * a->x3[j];
            /* h = x3[16:32]; TruncExp backward (networks.py:26-30) on h[0] */
            for (int k = 0; k < 16; ++k) dh[k] = dx3[16 + k];
            {
                const float x = fminf(fmaxf(a->h[0], -15.0f), 15.0f);
                const float ds = rh(dsigmas[i] * expf(x)); /* fp32 grad cast to the fp16 h */
                dh[0] = rh(dh[0] + ds);
            }
            /* layer 2: h = W2 h1 */
            for (int j = 0; j < 64; ++j) {
                float acc = 0.0f;
                for (int k = 0; k < 16; ++k) acc += dh[k] * wh[1][k * 64 + j];
                dh1[j] = a->h1[j] > 0.0f ? rh(acc) : 0.0f;
            }
            for (int k = 0; k < 16; ++k)
                for (int j = 0; j < 64; ++j) g[goff[1] + k * 64 + j] += (double)dh[k] * a->h1[j];
            /* layer 1 */
            for (int j = 0; j < 32; ++j) {
                float acc = 0.0f;
                for (int k = 0; k < 64; ++k) acc += dh1[k] * wh[0][k * 32 + j];
                de[j] = rh(acc);
            }
            for (int k = 0; k < 64; ++k)
                if (dh1[k] != 0.0f)
                    for (int j = 0; j < 32; ++j) g[goff[0] + k * 32 + j] += (double)dh1[k] * a->e[j];
            for (int j = 0; j < 32; ++j) {
                if (emb_dtype == NGP_F16) ((f16*)demb)[i * 32 + j] = (f16)de[j];
                else ((float*)demb)[i * 32 + j] = de[j];
            }
        }
    }
    for (int t = 0; t < nthreads; ++t)
        for (int k = 0; k < NGP_MLP_PARAMS; ++k) grad_w[k] += (float)gacc[(size_t)t * NGP_MLP_PARAMS + k];
    free(gacc);
    free(whb);
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a8  volume_rendering_kernel         modules/volume_train.py:6-48           */
/* ------------------------------------------------------------------------- */
static inline float load_rgb(const void* rgbs, int dtype, int64_t i) {
    return dtype == NGP_F16 ? (float)((const f16*)rgbs)[i] : ((const float*)rgbs)[i];
}

int ngp_composite_train_fwd_cpu(const float* sigmas, const void* rgbs, int rgbs_dtype,
                                const float* deltas, const float* ts, const int32_t* rays_a,
                                float T_threshold, int32_t* total_samples, float* opacity,
                                float* depth, float* rgb, float* ws, int64_t n_rays,
                                int64_t n_samples) {
    (void)n_samples;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t n = 0; n < n_rays; ++n) {
        const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
        const int N = rays_a[n * 3 + 2];
        float r = 0, g = 0, b = 0, dep = 0, op = 0, T = 1.0f; /* :27-34 */
        int cnt = 0;
        for (int k = 0; k < N; ++k) {
            const int64_t s = start + k;
            if (T > T_threshold) { /* :38 */
                const float a = 1.0f - expf(-sigmas[s] * deltas[s]);
                const float w = a * T;
                r += w * load_rgb(rgbs, rgbs_dtype, s * 3 + 0);
                g += w * load_rgb(rgbs, rgbs_dtype, s * 3 + 1);
                b += w * load_rgb(rgbs, rgbs_dtype, s * 3 + 2);
                dep += w * ts[s];
                op += w;
                ws[s] = w;
                T = T * (1.0f - a);
                cnt += 1;
            } else {
                ws[s] = 0.0f; /* reference: uninitialised (volume_train.py:91-94) */
            }
        }
        rgb[ray * 3 + 0] = r;
        rgb[ray * 3 + 1] = g;
        rgb[ray * 3 + 2] = b;
        depth[ray] = dep;
        opacity[ray] = op;
        total_samples[ray] = cnt;
    }
    return 0;
}

/* reverse mode of the loop above (what Taichi autodiff generates, volume_train.py:160-173);
 * the `T > threshold` branch is a constant of the trace. */
int ngp_composite_train_bwd_cpu(const float* dL_dopacity, const float* dL_ddepth,
                                const float* dL_drgb, const float* dL_dws, const float* sigmas,
                                const void* rgbs, int rgbs_dtype, const float* deltas,
                                const float* ts, const int32_t* rays_a, const float* opacity,
                                const float* depth, const float* rgb, float T_threshold,
                                float* dL_dsigmas, void* dL_drgbs, int64_t n_rays,
                                int64_t n_samples) {
    (void)n_samples; (void)opacity; (void)depth; (void)rgb;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t n = 0; n < n_rays; ++n) {
        const int64_t ray = rays_a[n * 3 + 0], start = rays_a[n * 3 + 1];
        const int N = rays_a[n * 3 + 2];
        const float gr = dL_drgb[ray * 3 + 0], gg = dL_drgb[ray * 3 + 1], gb = dL_drgb[ray * 3 + 2];
        const float gd = dL_ddepth[ray], go = dL_dopacity[ray];
        /* forward replay to find the active prefix and T values (double for the oracle) */
        double T = 1.0;
        float Tf = 1.0f; /* fp32 replay decides the active prefix exactly like the forward */
        int active = 0;
        double* Ts = (double*)malloc(sizeof(double) * (size_t)(N + 1));
        Ts[0] = 1.0;
        for (int k = 0; k < N; ++k) {
            const int64_t s = start + k;
            if (Tf > T_threshold) {
                const float af = 1.0f - expf(-sigmas[s] * deltas[s]);
                Tf = Tf * (1.0f - af);
                const double a = 1.0 - exp(-(double)sigmas[s] * deltas[s]);
                T = T * (1.0 - a);
                active = k + 1;
            }
            Ts[k + 1] = T;
        }
        double suffix = 0.0; /* sum_{j>s} w_j G_j */
        for (int k = N - 1; k >= 0; --k) {
            const int64_t s = start + k;
            if (k >= active) {
                dL_dsigmas[s] = 0.0f;
                for (int c = 0; c < 3; ++c) {
                    if (rgbs_dtype == NGP_F16) ((f16*)dL_drgbs)[s * 3 + c] = (f16)0.0f;
                    else ((float*)dL_drgbs)[s * 3 + c] = 0.0f;
                }
                continue;
            }
            const double Tk = Ts[k], Tk1 = Ts[k + 1];
            const double w = Tk - Tk1; /* a*T */
            const double c0 = load_rgb(rgbs, rgbs_dtype, s * 3 + 0), c1 = load_rgb(rgbs, rgbs_dtype, s * 3 + 1),
                         c2 = load_rgb(rgbs, rgbs_dtype, s * 3 + 2);
            const double G = gr * c0 + gg * c1 + gb * c2 + gd * (double)ts[s] + go + (double)dL_dws[s];
            dL_dsigmas[s] = (float)((double)deltas[s] * (Tk1 * G - suffix));
            const double gc[3] = {w * gr, w * gg, w * gb};
            for (int c = 0; c < 3; ++c) {
                if (rgbs_dtype == NGP_F16) ((f16*)dL_drgbs)[s * 3 + c] = (f16)gc[c];
                else ((float*)dL_drgbs)[s * 3 + c] = (float)gc[c];
            }
            suffix += w * G;
        }
        free(Ts);
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a9  composite_test                  modules/volume_render_test.py:4-54     */
/* ------------------------------------------------------------------------- */
int ngp_composite_test_cpu(const float* sigmas, const void* rgbs, int rgbs_dtype,
                           const float* deltas, const float* ts, const int64_t* pack_info,
                           int64_t* alive_indices, float T_threshold, float* opacity,
                           float* depth, float* rgb, int64_t n_alive) {
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t n = 0; n < n_alive; ++n) {
        const int64_t start = pack_info[n * 2 + 0], steps = pack_info[n * 2 + 1];
        const int64_t ray = alive_indices[n];
        if (steps == 0) {
            alive_indices[n] = -1;
            continue;
        }
        float T = 1.0f - opacity[ray];
        float r = 0, g = 0, b = 0, dep = 0, op = 0;
        for (int64_t k = 0; k < steps; ++k) {
            const int64_t s = start + k;
            const float a = 1.0f - expf(-sigmas[s] * deltas[s]);
            const float w = a * T;
            r += w * load_rgb(rgbs, rgbs_dtype, s * 3 + 0);
            g += w * load_rgb(rgbs, rgbs_dtype, s * 3 + 1);
            b += w * load_rgb(rgbs, rgbs_dtype, s * 3 + 2);
            dep += w * ts[s];
            op += w;
            T *= 1.0f - a;
            if (T <= T_threshold) {
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
    return 0;
}

/* ------------------------------------------------------------------------- */
/* distortion loss                     modules/distortion.py:15-119           */
/* ------------------------------------------------------------------------- */
int ngp_distortion_fwd_cpu(const float* ws, const float* deltas, const float* ts, const int32_t* rays_a,
                           float* loss, int64_t n_rays, int64_t n_samples) {
    (void)n_samples;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < n_rays; ++i) {
        const int64_t ray = rays_a[i * 3 + 0], start = rays_a[i * 3 + 1];
        const int N = rays_a[i * 3 + 2];
        float ws_t = 0.f, wts_t = 0.f, acc = 0.f;
        for (int n = 0; n < N; ++n) { /* prefix_sums_kernel :28-44 fused with _loss_kernel :55-64 */
            const int64_t s = start + n;
            const float ws_exc = ws_t, wts_exc = wts_t;
            ws_t += ws[s];
            wts_t += ws[s] * ts[s];
            acc += 2.f * (wts_t * ws_exc - ws_t * wts_exc) + 1.f / 3.f * ws[s] * ws[s] * deltas[s];
        }
        loss[ray] = acc; /* :82 */
    }
    return 0;
}

int ngp_distortion_bwd_cpu(const float* dL_dloss, const float* ws, const float* deltas, const float* ts,
                           const int32_t* rays_a, float* dL_dws, int64_t n_rays, int64_t n_samples) {
    (void)n_samples;
#pragma omp parallel for schedule(dynamic, 64)
    for (int64_t i = 0; i < n_rays; ++i) {
        const int64_t ray = rays_a[i * 3 + 0], start = rays_a[i * 3 + 1];
        const int N = rays_a[i * 3 + 2];
        float ws_sum = 0.f, wts_sum = 0.f;
        for (int n = 0; n < N; ++n) {
            ws_sum += ws[start + n];
            wts_sum += ws[start + n] * ts[start + n];
        }
        float ws_inc = 0.f, wts_inc = 0.f;
        const float g = dL_dloss[ray];
        for (int n = 0; n < N; ++n) { /* :104-117 */
            const int64_t s = start + n;
            const float selector = n == 0 ? 0.f : ts[s] * ws_inc - wts_inc; /* scans up to s-1 */
            ws_inc += ws[s];
            wts_inc += ws[s] * ts[s];
            float d = g * 2.f * (selector + (wts_sum - wts_inc - ts[s] * (ws_sum - ws_inc)));
            d += g * 2.f / 3.f * ws[s] * deltas[s];
            dL_dws[s] = d;
        }
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* occupancy-grid helpers              modules/utils.py:120-169               */
/* ------------------------------------------------------------------------- */
int ngp_packbits_cpu(const float* density_grid, float density_threshold, uint8_t* density_bitfield,
                     int64_t n_bytes) {
#pragma omp parallel for schedule(static)
    for (int64_t n = 0; n < n_bytes; ++n) {
        uint8_t bits = 0;
        for (int i = 0; i < 8; ++i)
            bits |= (density_grid[8 * n + i] > density_threshold) ? (uint8_t)(1u << i) : 0;
        density_bitfield[n] = bits;
    }
    return 0;
}
int ngp_morton3d_cpu(const int32_t* coords, int32_t* indices, int64_t n) {
    for (int64_t i = 0; i < n; ++i)
        indices[i] = (int32_t)morton3d((uint32_t)coords[i * 3], (uint32_t)coords[i * 3 + 1],
                                       (uint32_t)coords[i * 3 + 2]);
    return 0;
}
int ngp_morton3d_invert_cpu(const int32_t* indices, int32_t* coords, int64_t n) {
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t ind = (uint32_t)indices[i];
        coords[i * 3 + 0] = morton3d_invert1(ind >> 0);
        coords[i * 3 + 1] = morton3d_invert1(ind >> 1);
        coords[i * 3 + 2] = morton3d_invert1(ind >> 2);
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a12  GradScaler.unscale_ + torch.optim.Adam(eps=1e-15)   train.py:137-201  */
/* ------------------------------------------------------------------------- */
int ngp_check_finite_cpu(const float* grad, int64_t n, int32_t* found_inf) {
    int bad = 0;
#pragma omp parallel for reduction(| : bad)
    for (int64_t i = 0; i < n; ++i) bad |= !isfinite(grad[i]);
    if (bad) *found_inf = 1;
    return 0;
}

int ngp_adam_step_cpu(float* param, float* grad, float* exp_avg, float* exp_avg_sq,
                      void* param_f16_or_null, const int32_t* found_inf_or_null, float lr,
                      float beta1, float beta2, float eps, float inv_scale, int32_t step,
                      int zero_grad, int64_t n) {
    const int skip = found_inf_or_null && *found_inf_or_null;
    /* torch/optim/adam.py _single_tensor_adam: bias corrections in double, then fp32 ops */
    const double bc1 = 1.0 - pow((double)beta1, (double)step);
    const double bc2 = 1.0 - pow((double)beta2, (double)step);
    const float step_size = (float)((double)lr / bc1);
    const float bc2_sqrt = (float)sqrt(bc2);
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        if (!skip) {
            const float g = grad[i] * inv_scale;
            const float m = exp_avg[i] + (g - exp_avg[i]) * (1.0f - beta1); /* lerp_ */
            const float v = exp_avg_sq[i] * beta2 + (1.0f - beta2) * g * g;
            exp_avg[i] = m;
            exp_avg_sq[i] = v;
            const float denom = sqrtf(v) / bc2_sqrt + eps;
            param[i] = param[i] - step_size * (m / denom);
            if (param_f16_or_null) ((f16*)param_f16_or_null)[i] = (f16)param[i];
        }
        if (zero_grad) grad[i] = 0.0f;
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* training ray batch sampling   datasets/base.py:34-61, ray_utils.py:51-80   */
/* ------------------------------------------------------------------------- */
/* Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11;
 * the generator behind torch's CUDA randint/rand).  Pinned against the Random123 known-answer
 * vectors in tests/test_oracle.py. */
void ngp_philox4x32_10_cpu(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
    uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3], k0 = key[0], k1 = key[1];
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
        const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        c0 = n0;
        c1 = (uint32_t)p1;
        c2 = n2;
        c3 = (uint32_t)p0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

/* The reference draws img/pix with torch.randint (base.py:38-52), gathers rays/poses/directions
 * (:53-60) and rotates directions by the pose (ray_utils.py:67-75); the index draw here is the
 * library's own Philox mapping (documented in include/ngp_b200.h), the rest follows the reference. */
int ngp_sample_ray_batch_cpu(const float* image_bank, int channels, const float* poses, const float* directions,
                             int64_t n_img, int64_t n_pix, const int64_t* img_idxs, const int64_t* pix_idxs,
                             int64_t fixed_img, uint64_t seed, int32_t step, float* rays_o, float* rays_d,
                             float* rgb, float* noise, int64_t* img_out, int64_t* pix_out, int64_t n_rays) {
    for (int64_t i = 0; i < n_rays; ++i) {
        const uint32_t ctr[4] = {(uint32_t)i, (uint32_t)((uint64_t)i >> 32), (uint32_t)step, 0u};
        const uint32_t key[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
        uint32_t r[4];
        ngp_philox4x32_10_cpu(ctr, key, r);
        int64_t img = img_idxs ? img_idxs[i]
                               : (fixed_img >= 0 ? fixed_img : (int64_t)(((uint64_t)r[0] * (uint64_t)n_img) >> 32));
        int64_t pix = pix_idxs ? pix_idxs[i] : (int64_t)(((uint64_t)r[1] * (uint64_t)n_pix) >> 32);
        if (img < 0) img = 0;
        if (img > n_img - 1) img = n_img - 1;
        if (pix < 0) pix = 0;
        if (pix > n_pix - 1) pix = n_pix - 1;
        const float* P = poses + img * 12;
        const float* d = directions + pix * 3;
        for (int a = 0; a < 3; ++a) {
            rays_d[i * 3 + a] = (d[0] * P[a * 4 + 0] + d[1] * P[a * 4 + 1]) + d[2] * P[a * 4 + 2];
            rays_o[i * 3 + a] = P[a * 4 + 3];
        }
        if (rgb)
            for (int c = 0; c < 3; ++c) rgb[i * 3 + c] = image_bank[(img * n_pix + pix) * channels + c];
        if (noise) noise[i] = (float)(r[2] >> 8) * 5.9604644775390625e-8f;
        if (img_out) img_out[i] = img;
        if (pix_out) pix_out[i] = pix;
    }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* Blueprint of the planned cell-stepping march (DESIGN.md §7, exp_step_factor == 0 only).              */
/* Same loop as march_step / ray_march.py:45-74, except that the inner `while t < t_target: t += dt`     */
/* is replaced by a closed-form jump: inside one fp32 binade every `t += dt` adds the same whole number  */
/* of ulps, so the first candidate position >= t_target follows from one integer division; only a step   */
/* that crosses into the next binade is taken with a real add.  Must emit bit-identical sample times     */
/* (tests/test_oracle.py::test_cellstep_march_equals_reference_march).                                   */
/* ------------------------------------------------------------------------- */
static inline uint32_t f2u(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
static inline float u2f(uint32_t u) { float x; memcpy(&x, &u, 4); return x; }

/* first position of the sequence t, t+dt, (t+dt)+dt, ... that is >= t_target, taking at least one step */
static inline float advance_const_dt(float t, float dt, float t_target, int64_t* real_adds) {
    float tn = march_advance(t, dt);
    *real_adds += 1;
    while (tn < t_target) {
        const uint32_t b = f2u(tn), e = b >> 23; /* tn > 0: no sign bit */
        const float t1 = tn + dt;
        const uint32_t b1 = f2u(t1);
        *real_adds += 1;
        if (!(t1 > tn)) return INFINITY; /* no progress: the ray ends (march_advance) */
        if ((b1 >> 23) != e) { /* this step leaves the binade */
            tn = t1;
            continue;
        }
        const uint32_t m = (b & 0x7FFFFFu) | 0x800000u;
        const uint32_t c = ((b1 & 0x7FFFFFu) | 0x800000u) - m; /* ulps per step in this binade */
        const uint32_t kmax = (0xFFFFFFu - m) / c;              /* steps that stay inside it */
        uint32_t k = kmax;
        const uint32_t bt = f2u(t_target);
        if ((bt >> 23) == e) { /* target in the same binade: a multiple of the same ulp */
            const uint32_t need = ((bt & 0x7FFFFFu) | 0x800000u) - m;
            const uint32_t kk = (need + c - 1) / c;
            if (kk < k) k = kk;
        }
        if (k == 0) { /* next step crosses (cannot happen after the exponent check, kept for safety) */
            tn = t1;
            continue;
        }
        tn = u2f((e << 23) | ((m + k * c) & 0x7FFFFFu));
    }
    return tn;
}

int ngp_raymarching_cellstep_cpu(const float* rays_o, const float* rays_d, const float* hits_t,
                                 const uint8_t* density_bitfield, const float* noise, int cascades,
                                 int grid_size, float scale, int max_samples, const int32_t* rays_a,
                                 float* ts, int32_t* counts, int64_t* stats /* [iterations, real adds] */,
                                 int64_t n_rays) {
    int64_t iters = 0, adds = 0;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : iters, adds)
    for (int64_t r = 0; r < n_rays; ++r) {
        march_ctx c;
        march_ctx_init(&c, rays_o + r * 3, rays_d + r * 3, cascades, grid_size, scale, 0.0f, density_bitfield);
        const int gs = grid_size;
        const float gsf = (float)gs, gs_inv = 1.0f / gsf;
        const float t2 = hits_t[r * 2 + 1];
        float t = march_train_t0(hits_t, noise, r, 0.0f, grid_size, scale);
        const float dt = calc_dt(t, 0.0f, gs, scale); /* constant for exp_step_factor == 0 */
        const int64_t start = rays_a[r * 3 + 1];
        int n = 0;
        uint32_t last_idx = 0xFFFFFFFFu;
        int last_occ = 0;
        while (0.0f <= t && t < t2 && n < max_samples) {
            iters += 1;
            float xyz[3], nxyz[3];
            uint32_t u[3];
            for (int k = 0; k < 3; ++k) xyz[k] = c.o[k] + t * c.d[k];
            const int mip = imax(mip_from_pos(xyz[0], xyz[1], xyz[2], cascades), mip_from_dt(dt, gs, cascades));
            const float mip_bound = fminf(ldexpf(1.0f, mip - 1), scale);
            const float mip_bound_inv = 1.0f / mip_bound;
            for (int k = 0; k < 3; ++k) {
                float v = 0.5f * (xyz[k] * mip_bound_inv + 1.0f) * gsf;
                v = fminf(fmaxf(v, 0.0f), gsf - 1.0f);
                nxyz[k] = v;
                u[k] = (uint32_t)v;
            }
            const uint32_t idx = (uint32_t)mip * (uint32_t)(gs * gs * gs) + morton3d(u[0], u[1], u[2]);
            if (idx != last_idx) { /* consecutive positions in one cell share the bitfield lookup */
                last_idx = idx;
                last_occ = (density_bitfield[idx >> 3] >> (idx & 7u)) & 1;
            }
            if (last_occ) {
                ts[start + n] = t;
                n += 1;
                t = march_advance(t, dt);
                adds += 1;
                continue;
            }
            float tmin = INFINITY;
            for (int k = 0; k < 3; ++k) {
                const float tx =
                    (((nxyz[k] + 0.5f + 0.5f * fsign(c.d[k])) * gs_inv * 2.0f - 1.0f) * mip_bound - xyz[k]) * c.dinv[k];
                tmin = fminf(tmin, tx);
            }
            t = advance_const_dt(t, dt, t + fmaxf(0.0f, tmin), &adds);
        }
        counts[r] = n;
    }
    stats[0] = iters;
    stats[1] = adds;
    return 0;
}

/* ------------------------------------------------------------------------- */
/* Lane-level emulation of the planned warp-per-ray marching fast path (DESIGN.md §7): 32 candidate       */
/* positions per chunk, lane k holds position k.  A chunk is REGULAR when every in-box lane is either      */
/* occupied or has an axis with d < -1e-3 whose grid coordinate is not clamped — then each visited          */
/* position's successor is the next position (exit quirk, see the tests) and emit = occupied lanes; any     */
/* other chunk, and any chunk entered with a pending jump, goes through the sequential reference loop.      */
/* Returns sample times in the layout of rays_a and the number of regular / general chunks.                 */
/* ------------------------------------------------------------------------- */
int ngp_raymarching_lanes_cpu(const float* rays_o, const float* rays_d, const float* hits_t,
                              const uint8_t* density_bitfield, const float* noise, int grid_size, float scale,
                              int max_samples, const int32_t* rays_a, float* ts, int32_t* counts,
                              int64_t* stats /* [regular chunks, general chunks] */, int64_t n_rays) {
    int64_t n_reg = 0, n_gen = 0;
    const int gs = grid_size;
    const float gsf = (float)gs;
#pragma omp parallel for schedule(dynamic, 64) reduction(+ : n_reg, n_gen)
    for (int64_t r = 0; r < n_rays; ++r) {
        march_ctx c;
        march_ctx_init(&c, rays_o + r * 3, rays_d + r * 3, 1, grid_size, scale, 0.0f, density_bitfield);
        const float t2 = hits_t[r * 2 + 1];
        float t = march_train_t0(hits_t, noise, r, 0.0f, grid_size, scale);
        const float dt = calc_dt(t, 0.0f, gs, scale);
        const float mip_bound = fminf(0.5f, scale), mip_bound_inv = 1.0f / mip_bound;
        const int64_t start = rays_a[r * 3 + 1];
        int n = 0;
        while (0.0f <= t && t < t2 && n < max_samples) {
            /* candidate positions of this chunk (the occupancy-independent sequence) */
            float pos[33];
            pos[0] = t;
            {
                /* lane k's position without the serial chain when the 33 positions share t's binade: k steps add
                 * k * c ulps (c = ulps per step in this binade); otherwise (a binade boundary inside the chunk,
                 * once or twice per ray) fall back to the sequential adds */
                const uint32_t b = f2u(t), e = b >> 23, m = (b & 0x7FFFFFu) | 0x800000u;
                const uint32_t b1 = f2u(t + dt);
                const uint32_t cstep = ((b1 & 0x7FFFFFu) | 0x800000u) - m;
                if ((b1 >> 23) == e && (uint64_t)m + 32ull * cstep <= 0xFFFFFFull) {
                    for (int k = 1; k <= 32; ++k) pos[k] = u2f((e << 23) | ((m + (uint32_t)k * cstep) & 0x7FFFFFu));
                } else {
                    for (int k = 1; k <= 32; ++k) pos[k] = pos[k - 1] + dt;
                }
            }
            int regular = 1, occ[32], valid[32];
            for (int k = 0; k < 32; ++k) {
                valid[k] = pos[k] < t2;
                occ[k] = 0;
                if (!valid[k]) continue;
                int ok = 0;
                uint32_t u[3];
                for (int a = 0; a < 3; ++a) {
                    const float x = c.o[a] + pos[k] * c.d[a];
                    const float raw = 0.5f * (x * mip_bound_inv + 1.0f) * gsf;
                    if (c.d[a] < -1e-3f && raw < gsf - 1.0f) ok = 1; /* exit distance ~0 along this axis */
                    u[a] = (uint32_t)fminf(fmaxf(raw, 0.0f), gsf - 1.0f);
                }
                const uint32_t idx = morton3d(u[0], u[1], u[2]);
                occ[k] = (density_bitfield[idx >> 3] >> (idx & 7u)) & 1;
                if (!occ[k] && !ok) regular = 0;
            }
            int stalled = 0; /* a step that does not advance ends the ray: the sequential loop below handles it */
            for (int k = 0; k < 32; ++k) stalled |= !(pos[k + 1] > pos[k]);
            if (stalled) regular = 0;
            if (regular) {
                n_reg += 1;
                int k = 0;
                for (; k < 32 && valid[k] && n < max_samples; ++k)
                    if (occ[k]) ts[start + n++] = pos[k];
                if (k < 32) break; /* left the box or hit the sample cap inside this chunk */
                t = pos[32];
            } else {
                /* general path: the reference loop over this chunk's span (may overshoot into the next span) */
                n_gen += 1;
                const float t_end = stalled ? INFINITY : pos[32];
                float xyz[3], dts;
                while (0.0f <= t && t < t2 && n < max_samples && t < t_end) {
                    float tt = t;
                    if (march_step(&c, &tt, xyz, &dts)) {
                        ts[start + n++] = t;
                        t = march_advance(t, dts);
                    } else {
                        t = tt;
                    }
                }
            }
        }
        counts[r] = n;
    }
    stats[0] = n_reg;
    stats[1] = n_gen;
    return 0;
}

/* ---- host thread control for the timed CPU arms (bench.py cpu_baseline / --impl reference) --------------------
 * torchrun exports OMP_NUM_THREADS=1 to its workers; the baseline must use the cores it reports. */
extern void omp_set_num_threads(int);
extern int omp_get_max_threads(void);
int ngp_oracle_set_threads(int n) {
    if (n > 0) omp_set_num_threads(n);
    return omp_get_max_threads();
}
int ngp_oracle_threads_used(void) {
    int n = 0;
#pragma omp parallel
    {
#pragma omp atomic
        n += 1;
    }
    return n;
}

