/*
 * triplane.c — CPU ORACLE of the tri-plane encoder (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * A plain-C, strict-fp32 restatement of triplane_encoder_kernel (modules/triplane.py:35-98 of
 * taichi-dev/taichi-nerfs) and of its Taichi autodiff (:186-197), in the reference's source order.
 * Built like ngp_oracle.c (gcc -O2 -march=x86-64-v3 -ffp-contract=off -fopenmp) into its own library
 * by oracle/triplane.py; `-ffp-contract=off` matters: the CUDA forward must equal it bit for bit.
 * Only tests/ load it.
 */
#include <math.h>
#include <stdint.h>

#include "../include/ngp_b200.h"

/* ------------------------------------------------------------------------- */
/* tri-plane encoder                   modules/triplane.py:35-98, :186-197    */
/* ------------------------------------------------------------------------- */
/* Taichi's casts as the GPU executes them (cvt.rmi/cvt.rzi.u32.f32 saturate; NaN -> 0): equal to C's casts
 * for every value the reference defines, and defined for the rest. */
static inline uint32_t u32_floor_sat(float p) {
    if (!(p > 0.0f)) return 0u;
    if (p >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)floorf(p);
}
static inline uint32_t u32_trunc_sat(float p) {
    if (!(p > 0.0f)) return 0u;
    if (p >= 4294967296.0f) return 0xFFFFFFFFu;
    return (uint32_t)p;
}

/* One level of one sample: for each axis the two max_res-grid coordinates and the weights (1-frac, frac).
 * Plane fd pairs axis fd (first coordinate) with axis (fd+1)%3 (second): the vector
 * [x,y, y,z, z,x] of :46-50 read with [d::2].  Note the inner `for i in ti.static(range(2))` at :80 reuses the
 * sample-index name `i`; Taichi scopes static-for targets, so the output row at :98 is still the sample. */
static void triplane_axes(const float x[3], const ngp_triplane_layout* lay, int level, uint32_t ori[3][2],
                          float a[3][2]) {
    const uint32_t res = lay->resolutions[level];
    const uint32_t mr = (uint32_t)lay->max_res;
    const float res_m1 = (float)(res - 1u), res_f = (float)res, mr_m1 = (float)(mr - 1u);
    for (int k = 0; k < 3; ++k) {
        const float p = x[k] * res_m1 + 0.5f;          /* pos = xyz * (resolution - 1) + 0.5       :56 */
        const uint32_t g = u32_floor_sat(p);           /* pos_grid = u32(floor(pos))                 :57 */
        const float fr = p - (float)g;                 /* pos -= f32(pos_grid)                       :58 */
        a[k][0] = 1.0f - fr;                           /* w *= 1 - pos                               :67 */
        a[k][1] = fr;                                  /* w *= pos                                   :70 */
        for (int b = 0; b < 2; ++b) {
            /* u32(f32(g_c) / f32(res) * (max_res - 1))                                               :73-76
             * clamped to [0, max_res-1]: the reference's bound check is commented out (:88-89); the clamp is
             * the identity for xyz in [0, 1] */
            const uint32_t o = u32_trunc_sat((float)(g + (uint32_t)b) / res_f * mr_m1);
            ori[k][b] = o < mr - 1u ? o : mr - 1u;
        }
    }
}

/* entry of corner c (bit d -> g+1 on the plane's d-th coordinate, :60-70) of plane fd: index = ori[first] +
 * ori[second] * max_res (:78-82); entry = fd*max_res^2*F + index*F (+ j) (:84-87) */
static inline int64_t triplane_entry(const ngp_triplane_layout* lay, uint32_t ori[3][2], int fd, int c) {
    const int s = (fd + 1) % 3;
    const int64_t mr = lay->max_res;
    return ((int64_t)fd * mr * mr + (int64_t)ori[fd][c & 1] + (int64_t)ori[s][c >> 1] * mr) * lay->feat_dim;
}
static inline float triplane_weight(float a[3][2], int fd, int c) {
    const float w0 = 1.0f * a[fd][c & 1];              /* w = 1; w *= a_d0; w *= a_d1              :61-70 */
    return w0 * a[(fd + 1) % 3][c >> 1];
}

static int triplane_check(const ngp_triplane_layout* lay) {
    if (!lay || lay->n_levels < 1 || lay->n_levels > NGP_MAX_LEVELS) return -1;
    if (lay->feat_dim != 2 && lay->feat_dim != 4) return -1;
    if (lay->max_res < 2 || lay->max_res > NGP_TRIPLANE_MAX_RES) return -1;
    return 0;
}

/* lf[fd][j] = sum_c w_c[fd] * table[entry_c + j] from 0, corners in order (:90-92) */
static void triplane_lf(const float* table, const ngp_triplane_layout* lay, uint32_t ori[3][2], float a[3][2],
                        float lf[3][4]) {
    const int F = lay->feat_dim;
    for (int fd = 0; fd < 3; ++fd) {
        for (int j = 0; j < F; ++j) lf[fd][j] = 0.0f;
        for (int c = 0; c < 4; ++c) {
            const float w = triplane_weight(a, fd, c);
            const int64_t e = triplane_entry(lay, ori, fd, c);
            for (int j = 0; j < F; ++j) lf[fd][j] = lf[fd][j] + w * table[e + j];
        }
    }
}

/* out[i, j*L + level] (sn = j*L + level: j = sn // levels, level = sn % levels, :43-45)
 *   = ((1 * lf[0][j]) * lf[1][j]) * lf[2][j]                                                          :94-98 */
int ngp_triplane_encode_fwd_cpu(const float* xyz, const float* table, const ngp_triplane_layout* lay, float* out,
                                int64_t n) {
    if (triplane_check(lay)) return -1;
    const int L = lay->n_levels, F = lay->feat_dim;
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < n; ++i) {
        for (int l = 0; l < L; ++l) {
            uint32_t ori[3][2];
            float a[3][2], lf[3][4];
            triplane_axes(xyz + i * 3, lay, l, ori, a);
            triplane_lf(table, lay, ori, a, lf);
            for (int j = 0; j < F; ++j) {
                float cp = 1.0f;
                for (int fd = 0; fd < 3; ++fd) cp = cp * lf[fd][j];
                out[i * L * F + j * L + l] = cp;
            }
        }
    }
    return 0;
}

/* Taichi autodiff of the kernel above (:186-197): with c1 = 1*lf0, c2 = c1*lf1, out = c2*lf2 the reverse pass
 * forms dlf2 = dy*c2, dlf1 = (dy*lf2)*c1, dlf0 = (dy*lf2)*lf1, then table[entry_c] += dlf[fd] * w_c[fd].
 * grad_table is accumulated into, one plane per thread (planes own disjoint ranges; sample order within). */
int ngp_triplane_encode_bwd_cpu(const float* xyz, const float* table, const float* dout,
                                const ngp_triplane_layout* lay, float* grad_table, int64_t n) {
    if (triplane_check(lay)) return -1;
    const int L = lay->n_levels, F = lay->feat_dim;
#pragma omp parallel for schedule(static, 1)
    for (int fd = 0; fd < 3; ++fd) {
        for (int64_t i = 0; i < n; ++i) {
            for (int l = 0; l < L; ++l) {
                uint32_t ori[3][2];
                float a[3][2], lf[3][4], dlf[4];
                int any = 0;
                for (int j = 0; j < F; ++j) any |= dout[i * L * F + j * L + l] != 0.0f;
                if (!any) continue;
                triplane_axes(xyz + i * 3, lay, l, ori, a);
                triplane_lf(table, lay, ori, a, lf);
                for (int j = 0; j < F; ++j) {
                    const float dy = dout[i * L * F + j * L + l];
                    const float c1 = 1.0f * lf[0][j], c2 = c1 * lf[1][j];
                    dlf[j] = fd == 2 ? dy * c2 : fd == 1 ? (dy * lf[2][j]) * c1 : (dy * lf[2][j]) * lf[1][j];
                }
                for (int c = 0; c < 4; ++c) {
                    const float w = triplane_weight(a, fd, c);
                    const int64_t e = triplane_entry(lay, ori, fd, c);
                    for (int j = 0; j < F; ++j) grad_table[e + j] += dlf[j] * w;
                }
            }
        }
    }
    return 0;
}
