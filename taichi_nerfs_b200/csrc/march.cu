// march.cu — ray/AABB intersection and occupancy-grid ray marching (train + test).
//
// Semantics follow modules/intersection.py:8-37, modules/ray_march.py:8-123,197-268 and the
// device helpers modules/utils.py:54-117 of the reference, in strict fp32 source order (every
// op an explicit *_rn intrinsic) so that sample positions are bit-identical to the CPU oracle.
//
// GPU notes: these kernels are latency-bound integer/fp32 work over a 256 KiB..1.5 MiB
// bitfield that lives in L1/L2 — there is nothing for tensor cores here.  Training march is
// count -> single-CTA scan -> write, giving a deterministic, ray-ordered sample layout without
// the global atomics (ray_march.py:76-81) or the n_rays*1024-row scratch (ray_march.py:149-168).
#include "common.cuh"
#include "occupancy.cuh"

namespace {

constexpr float kNear = 0.01f;                                      // utils.py:13
constexpr float kSqrt3MaxSamples = (float)(1.7320508075688772 / 1024);  // utils.py:15
constexpr float kSqrt3x2 = (float)(1.7320508075688772 * 2);             // utils.py:16

__device__ __forceinline__ float calc_dt(float t, float esf, float dt_max) {  // utils.py:54-57
    return fminf(fmaxf(f_mul(t, esf), kSqrt3MaxSamples), dt_max);
}

// The next march position t + dt, or +inf when the add does not increase t: near t = dt * 2^24 the fp32 sum rounds
// back to t, and a NaN t never compares greater.  Every march loop advances only through this (the warp march checks
// the same condition on its 32-position chain), so each iteration strictly increases a finite t or ends the ray (+inf
// fails `t < t2` and `tn < t_target`); fp32 has finitely many values, so every loop ends.  The reference adds
// unconditionally and loops forever on such rays (ray_march.py:64,72-74).
__device__ __forceinline__ float march_advance(float t, float dt) {
    const float tn = f_add(t, dt);
    return tn > t ? tn : INFINITY;
}

__device__ __forceinline__ float fsign(float v) { return v > 0.0f ? 1.0f : (v < 0.0f ? -1.0f : 0.0f); }

struct Ray {
    float o[3], d[3], dinv[3];
};

struct MarchParams {
    const uint8_t* __restrict__ bits;
    int cascades;
    int grid_size;
    float gsf;       // (float)grid_size
    float gs_inv;    // 1/gsf
    uint32_t gs3;    // grid_size^3
    float scale;
    float esf;
    float dt_max;    // SQRT3_2*scale/grid_size
};

__device__ __forceinline__ void load_ray(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                         int64_t r, Ray& ray) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        ray.o[k] = rays_o[r * 3 + k];
        ray.d[k] = rays_d[r * 3 + k];
        ray.dinv[k] = f_div(1.0f, ray.d[k]);
    }
}

// One loop iteration of ray_march.py:45-74.  Occupied: returns true with xyz/dt set.
// Empty: advances t past the cell exit (ray_march.py:66-74) and returns false.
__device__ __forceinline__ bool march_step(const MarchParams& p, const Ray& ray, float& t, float xyz[3], float& dt) {
    const float tt = t;
#pragma unroll
    for (int k = 0; k < 3; ++k) xyz[k] = f_add(ray.o[k], f_mul(tt, ray.d[k]));
    dt = calc_dt(tt, p.esf, p.dt_max);
    int mip = 0;
    if (p.cascades > 1) {
        const float mx = fmaxf(fmaxf(fabsf(xyz[0]), fabsf(xyz[1])), fabsf(xyz[2]));
        const int m_pos = min(p.cascades - 1, max(0, frexp_bit(mx) + 1));            // utils.py:78-84
        const int m_dt = min(p.cascades - 1, max(0, frexp_bit(f_mul(dt, p.gsf))));   // utils.py:87-92
        mip = max(m_pos, m_dt);
    }
    // pow(2, mip-1), exact
    const float mip_bound = fminf(__uint_as_float((uint32_t)(127 + mip - 1) << 23), p.scale);
    const float mip_bound_inv = f_div(1.0f, mip_bound);
    float nxyz[3];
    uint32_t u[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float v = f_mul(f_mul(0.5f, f_add(f_mul(xyz[k], mip_bound_inv), 1.0f)), p.gsf);
        v = fminf(fmaxf(v, 0.0f), f_sub(p.gsf, 1.0f));
        nxyz[k] = v;
        u[k] = __float2uint_rz(v);
    }
    const uint32_t idx = (uint32_t)mip * p.gs3 + morton3d(u[0], u[1], u[2]);
    const uint32_t occ = (uint32_t)__ldg(p.bits + (idx >> 3)) & (1u << (idx & 7u));
    if (occ) return true;
    float tmin = INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float a = f_add(f_add(nxyz[k], 0.5f), f_mul(0.5f, fsign(ray.d[k])));
        a = f_sub(f_mul(f_mul(a, p.gs_inv), 2.0f), 1.0f);
        a = f_mul(f_sub(f_mul(a, mip_bound), xyz[k]), ray.dinv[k]);
        tmin = fminf(tmin, a);
    }
    const float t_target = f_add(tt, fmaxf(0.0f, tmin));
    float tn = march_advance(tt, calc_dt(tt, p.esf, p.dt_max));
    while (tn < t_target) tn = march_advance(tn, calc_dt(tn, p.esf, p.dt_max));
    t = tn;
    return false;
}

__device__ __forceinline__ float train_t0(const float* __restrict__ hits_t, const float* __restrict__ noise,
                                          int64_t r, const MarchParams& p) {
    float t1 = hits_t[r * 2 + 0];
    if (t1 >= 0.0f) {  // ray_march.py:36-38
        const float dt = calc_dt(t1, p.esf, p.dt_max);
        t1 = f_add(t1, f_mul(dt, noise[r]));
    }
    return t1;
}

// ---- a1 ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ray_aabb_kernel(const float* __restrict__ rays_o,
                                                       const float* __restrict__ rays_d, float scale,
                                                       float* __restrict__ hits_t, int64_t n) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const float half = f_div(f_sub(scale, -scale), 2.0f);
    float t1 = -INFINITY, t2 = INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float o = rays_o[r * 3 + k], d = rays_d[r * 3 + k];
        const float inv = f_div(1.0f, d);
        const float tmin = f_mul(f_sub(f_sub(0.0f, half), o), inv);
        const float tmax = f_mul(f_sub(f_add(0.0f, half), o), inv);
        t1 = fmaxf(t1, fminf(tmin, tmax));
        t2 = fminf(t2, fmaxf(tmin, tmax));
    }
    float2 out;
    if (t2 > 0.0f && t2 < INFINITY) out = make_float2(fmaxf(t1, kNear), t2);
    else out = make_float2(-1.0f, -1.0f);
    reinterpret_cast<float2*>(hits_t)[r] = out;
}

// ---- a2: warp-per-ray marching ---------------------------------------------------------------------
// The reference walks each ray with one thread (ray_march.py:27, block_dim=128): ~530 dependent grid
// steps per Lego ray, with divergent inner while-loops.  The sequence of candidate positions
// t_0, t_{k+1} = t_k + calc_dt(t_k) does NOT depend on occupancy (both the occupied branch and the
// skip loop advance by calc_dt(t)), so a warp can take one ray: every lane recomputes the same
// 32-step t chain (cheap, keeps it bit-identical to the sequential fp32 recurrence), lane k tests
// position k against the bitfield, and the "which positions are actually visited" logic (emit if
// occupied, else jump to the first position >= the cell's exit time) is resolved with ballots and a
// short shuffle pointer walk.  Samples come out in the same order with the same bits.
struct CellTest {
    float xyz[3];
    float nxyz[3];   // clamped grid coordinate (kept un-floored: the reference's exit uses it as is)
    float mip_bound;
    float dt;
    bool occ;
    bool regular;    // some axis has d < -1e-3 with an unclamped coordinate: the exit distance along it is ~0, so
                     // the reference loop advances by exactly ONE step from here (tests/test_oracle.py, exit quirk)
};

__device__ __forceinline__ CellTest test_cell(const MarchParams& p, const Ray& ray, float tt, float dt) {
    CellTest c;
#pragma unroll
    for (int k = 0; k < 3; ++k) c.xyz[k] = f_add(ray.o[k], f_mul(tt, ray.d[k]));
    c.dt = dt;
    int mip = 0;
    if (p.cascades > 1) {
        const float mx = fmaxf(fmaxf(fabsf(c.xyz[0]), fabsf(c.xyz[1])), fabsf(c.xyz[2]));
        const int m_pos = min(p.cascades - 1, max(0, frexp_bit(mx) + 1));
        const int m_dt = min(p.cascades - 1, max(0, frexp_bit(f_mul(dt, p.gsf))));
        mip = max(m_pos, m_dt);
    }
    const float mip_bound = fminf(__uint_as_float((uint32_t)(127 + mip - 1) << 23), p.scale);
    const float mip_bound_inv = f_div(1.0f, mip_bound);
    uint32_t u[3];
    c.regular = false;
    c.mip_bound = mip_bound;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float raw = f_mul(f_mul(0.5f, f_add(f_mul(c.xyz[k], mip_bound_inv), 1.0f)), p.gsf);
        c.regular = c.regular || (ray.d[k] < -1e-3f && raw < f_sub(p.gsf, 1.0f));
        const float v = fminf(fmaxf(raw, 0.0f), f_sub(p.gsf, 1.0f));
        c.nxyz[k] = v;
        u[k] = __float2uint_rz(v);
    }
    const uint32_t idx = (uint32_t)mip * p.gs3 + morton3d(u[0], u[1], u[2]);
    c.occ = ((uint32_t)__ldg(p.bits + (idx >> 3)) & (1u << (idx & 7u))) != 0;
    return c;
}

// exit time of the (empty) cell, ray_march.py:66-71
__device__ __forceinline__ float cell_exit(const MarchParams& p, const Ray& ray, const CellTest& c, float tt) {
    float tmin = INFINITY;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float a = f_add(f_add(c.nxyz[k], 0.5f), f_mul(0.5f, fsign(ray.d[k])));
        a = f_sub(f_mul(f_mul(a, p.gs_inv), 2.0f), 1.0f);
        a = f_mul(f_sub(f_mul(a, c.mip_bound), c.xyz[k]), ray.dinv[k]);
        tmin = fminf(tmin, a);
    }
    return f_add(tt, fmaxf(0.0f, tmin));
}

constexpr int kRaysPerBlock = 4;

// kMode: 0 = count (pass 1), 1 = write (pass 2), 2 = single pass for test-time frames (sample times are
// buffered in shared memory, the ray reserves its rows with one atomicAdd, then writes them coalesced),
// 3 = one ROUND of the compacting test-time renderer (render.cu: persistent warps walk the list of live rays, every
// ray resumes at t_cur[ray], emits at most `limit` samples and leaves its resume point behind)
constexpr int kMaxFrameSamples = 1024;
struct RoundArgs {
    const int32_t* __restrict__ alive;      // live ray ids of this round
    const int32_t* __restrict__ n_alive;    // their number (device)
    float* __restrict__ t_cur;              // per ray: where the march resumes (in/out); +inf = left the box
    int32_t* __restrict__ n_marched;        // per ray: samples emitted in earlier rounds of the frame (in/out)
    int max_samples;                        // per-ray cap over the whole frame (the one-shot march's max_samples)
    int limit;                              // samples per ray this round (reduced so that all live rays fit `capacity`)
};

template <int kMode>
__device__ __forceinline__ void march_one_ray(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                              const float* __restrict__ hits_t, const float* __restrict__ noise,
                                              const MarchParams& p, int max_samples, int32_t* __restrict__ rays_a,
                                              int32_t* __restrict__ counter, float* __restrict__ xyzs,
                                              float* __restrict__ dirs, float* __restrict__ deltas,
                                              float* __restrict__ ts, int64_t r, int64_t slot, int64_t capacity,
                                              float* my_buf, const RoundArgs& round) {
    constexpr bool kWrite = kMode == 1;
    const int lane = threadIdx.x & 31;
    const unsigned full = 0xffffffffu;

    int limit = max_samples;
    int64_t start = 0;
    if (kWrite) {
        start = rays_a[r * 3 + 1];
        limit = rays_a[r * 3 + 2];
        if (start + limit > capacity) {  // does not fit: drop the ray's samples (dropped rays form a suffix)
            if (lane == 0) {
                rays_a[r * 3 + 2] = 0;
                atomicMin(&counter[0], (int32_t)start);
            }
            return;
        }
        if (limit == 0) return;
    }
    Ray ray;
    load_ray(rays_o, rays_d, r, ray);
    const float t2 = hits_t[r * 2 + 1];
    float t;
    float t_resume = INFINITY;   // kMode 3: where the next round continues; stays +inf when the ray leaves the box
    int marched_before = 0;
    if (kMode == 3) {
        t = round.t_cur[r];
        if (!(0.0f < t)) t = -1.0f;
        marched_before = round.n_marched[r];
        limit = max(0, min(limit, round.max_samples - marched_before));   // the frame's per-ray cap
    } else if (kMode == 2 && noise == nullptr) {  // test time: no jitter, strict 0 < t (ray_march.py:226)
        t = hits_t[r * 2 + 0];
        if (!(0.0f < t)) t = -1.0f;
    } else {
        t = train_t0(hits_t, noise, r, p);
    }
    int emitted = 0;
    float skip_until = -INFINITY;
    const bool const_dt = p.esf == 0.0f;
    const float dt0 = calc_dt(t, p.esf, p.dt_max);

    while (0.0f <= t && t < t2 && emitted < limit) {  // ray_march.py:43 / :86 (warp-uniform)
        // t chain: position k of this chunk, identical on every lane
        float tk = t, my_t = t, my_dt = dt0;
        if (const_dt) {
            // inside one binade every `t += dt` adds the same whole number of ulps (tests/test_oracle.py, closed form):
            // lane k's position is k steps away without the serial chain; a chunk that contains a binade boundary
            // (once or twice per ray) falls back to the sequential adds
            const uint32_t b = __float_as_uint(t), e = b >> 23, m = (b & 0x7fffffu) | 0x800000u;
            const uint32_t b1 = __float_as_uint(f_add(t, dt0));
            const uint32_t cs = ((b1 & 0x7fffffu) | 0x800000u) - m;
            if ((b1 >> 23) == e && m + 32u * cs <= 0xffffffu) {
                my_t = __uint_as_float((e << 23) | ((m + (uint32_t)lane * cs) & 0x7fffffu));
                tk = __uint_as_float((e << 23) | ((m + 32u * cs) & 0x7fffffu));
            } else {
#pragma unroll
                for (int k = 0; k < 32; ++k) {
                    if (k == lane) my_t = tk;
                    tk = f_add(tk, dt0);
                }
            }
        } else {
#pragma unroll 8
            for (int k = 0; k < 32; ++k) {
                const float dk = calc_dt(tk, p.esf, p.dt_max);
                if (k == lane) {
                    my_t = tk;
                    my_dt = dk;
                }
                tk = f_add(tk, dk);
            }
        }
        // progress: position k+1 is reached only if every step up to it increased t (a step that does not stays put
        // forever, so the positions after the first stall repeat it and are not on the ray: march_advance)
        const float t_down = __shfl_down_sync(full, my_t, 1);   // every lane takes part: outside the select below
        const float t_next = lane < 31 ? t_down : tk;
        const unsigned stall_mask = __ballot_sync(full, !(t_next > my_t));
        const unsigned reach = stall_mask ? (2u << (__ffs(stall_mask) - 1)) - 1u : full;
        const bool valid = my_t < t2 && ((reach >> lane) & 1u);
        const CellTest c = test_cell(p, ray, my_t, my_dt);
        const unsigned valid_mask = __ballot_sync(full, valid);
        const unsigned occ_mask = __ballot_sync(full, valid && c.occ);

        // Independent-positions fast path: if every in-box lane is occupied or "regular" (and no jump is pending from
        // the previous chunk) each visited position's successor is simply the next one, so the visited set is the
        // whole chunk and the emitted samples are its occupied lanes — no exit times, search or pointer walk.
        const bool chunk_regular = const_dt && p.cascades == 1 && skip_until == -INFINITY &&
                                   __all_sync(full, !valid || c.occ || c.regular);
        unsigned emit = 0;
        if (chunk_regular) {
            emit = occ_mask;
            const int room = limit - emitted;
            if (__popc(emit) > room) emit &= (1u << __fns(emit, 0, room + 1)) - 1u;  // max_samples cap
        } else {
        const float t_target = cell_exit(p, ray, c, my_t);
        // empty lanes: first position j > lane with t_j >= t_target (at least one step, ray_march.py:72-74)
        int lo = lane + 1, hi = 32;
#pragma unroll
        for (int it = 0; it < 5; ++it) {
            const int mid = (lo + hi) >> 1;
            const float tm = __shfl_sync(full, my_t, min(mid, 31));
            if (lo < hi) {
                if (tm < t_target) lo = mid + 1;
                else hi = mid;
            }
        }
        const int nxt = lo;

        // Which positions does the sequential loop actually visit?  successor(j) = j+1 if occupied, else the
        // jump target; positions at/after the box exit end the walk.  The orbit of the chunk's entry
        // position under `successor` is found by pointer doubling (5 shuffle rounds) instead of a serial walk.
        int F = valid ? (c.occ ? lane + 1 : nxt) : 32;
        unsigned M = 1u << lane;
#pragma unroll
        for (int it = 0; it < 5; ++it) {
            const int src = min(F, 31);
            const unsigned Mo = __shfl_sync(full, M, src);
            const int Fo = __shfl_sync(full, F, src);
            if (F < 32) {
                M |= Mo;
                F = Fo;
            }
        }
        // entry position: skip the positions still inside the cell left at the end of the previous chunk
        const int pos0 = __popc(__ballot_sync(full, my_t < skip_until));
        if (pos0 < 32) {
            const unsigned visited = __shfl_sync(full, M, pos0) & valid_mask;
            emit = visited & occ_mask;
            const int room = limit - emitted;
            if (__popc(emit) > room) emit &= (1u << __fns(emit, 0, room + 1)) - 1u;  // max_samples cap
            skip_until = -INFINITY;
            if (visited) {
                const int q = 31 - __clz(visited);  // last visited position
                const int nq = __shfl_sync(full, nxt, q);
                const float tq = __shfl_sync(full, t_target, q);
                if (!((occ_mask >> q) & 1u) && nq >= 32) skip_until = tq;  // cell extends into the next chunk
            }
        }
        }
        if (kWrite && ((emit >> lane) & 1u)) {
            const int64_t i = start + emitted + __popc(emit & ((1u << lane) - 1u));
            xyzs[i * 3 + 0] = c.xyz[0];
            xyzs[i * 3 + 1] = c.xyz[1];
            xyzs[i * 3 + 2] = c.xyz[2];
            dirs[i * 3 + 0] = ray.d[0];
            dirs[i * 3 + 1] = ray.d[1];
            dirs[i * 3 + 2] = ray.d[2];
            ts[i] = my_t;
            deltas[i] = c.dt;
        }
        if ((kMode == 2 || kMode == 3) && ((emit >> lane) & 1u)) my_buf[emitted + __popc(emit & ((1u << lane) - 1u))] = my_t;
        emitted += __popc(emit);
        if (kMode == 3 && emitted >= limit) {
            // budget of this round used up: the march resumes at the position after the last emitted sample
            // (occupied -> `t += dt`, ray_march.py:258-262), i.e. the next lane's position or the next chunk's first
            const int q = 31 - __clz(emit);
            const float nx = __shfl_sync(full, t_next, q);
            t_resume = ((stall_mask >> q) & 1u) ? INFINITY : nx;
            break;
        }
        if (valid_mask != full || stall_mask) break;  // the ray left the box or stopped advancing inside this chunk
        t = tk;
    }
    if (kMode == 0 && lane == 0) {
        rays_a[r * 3 + 0] = (int32_t)r;
        rays_a[r * 3 + 2] = emitted;
    }
    if (kMode == 3) {
        // rows always fit: limit <= capacity / n_alive.  rays_a is indexed by the live-list slot.
        int s0 = 0;
        if (lane == 0 && emitted > 0) s0 = atomicAdd(&counter[0], emitted);
        s0 = __shfl_sync(full, s0, 0);
        if (lane == 0) {
            rays_a[slot * 3 + 0] = (int32_t)r;
            rays_a[slot * 3 + 1] = s0;
            rays_a[slot * 3 + 2] = emitted;
            // a ray that has reached max_samples is done, like the one-shot march: +inf takes it off the live list
            const bool capped = marched_before + emitted >= round.max_samples;
            round.n_marched[r] = marched_before + emitted;
            round.t_cur[r] = capped ? INFINITY : t_resume;
        }
        __syncwarp();
        for (int k = lane; k < emitted; k += 32) {
            const float tt = my_buf[k];
            const int64_t i = (int64_t)s0 + k;
            xyzs[i * 3 + 0] = f_add(ray.o[0], f_mul(tt, ray.d[0]));
            xyzs[i * 3 + 1] = f_add(ray.o[1], f_mul(tt, ray.d[1]));
            xyzs[i * 3 + 2] = f_add(ray.o[2], f_mul(tt, ray.d[2]));
            dirs[i * 3 + 0] = ray.d[0];
            dirs[i * 3 + 1] = ray.d[1];
            dirs[i * 3 + 2] = ray.d[2];
            ts[i] = tt;
            deltas[i] = calc_dt(tt, p.esf, p.dt_max);
        }
        __syncwarp();   // my_buf is reused by this warp's next ray
    }
    if (kMode == 2) {
        int s0 = 0;
        if (lane == 0 && emitted > 0) s0 = atomicAdd(&counter[0], emitted);  // reserve a contiguous row range
        s0 = __shfl_sync(full, s0, 0);
        // Capacity overflow.  Rows are handed out in atomic order, so exactly ONE ray can straddle the end of the
        // buffers (s0 < capacity < s0 + emitted); every ray reserving after it starts beyond the capacity.  The
        // straddling ray keeps the samples that fit (it is rendered truncated), the later ones own no rows — so every
        // row below min(counter[0], capacity) is written by its owner and no stale row reaches the network kernels.
        const bool fits = (int64_t)s0 + emitted <= capacity;
        const int keep = fits ? emitted : (int)max((int64_t)0, min((int64_t)emitted, capacity - (int64_t)s0));
        if (lane == 0) {
            rays_a[r * 3 + 0] = (int32_t)r;
            rays_a[r * 3 + 1] = keep > 0 ? s0 : 0;
            rays_a[r * 3 + 2] = keep;
            if (!fits) atomicAdd(&counter[1], 1);  // number of rays truncated / dropped for lack of capacity
        }
        if (keep == 0) return;
        emitted = keep;
        __syncwarp();
        for (int k = lane; k < emitted; k += 32) {
            const float tt = my_buf[k];
            const int64_t i = (int64_t)s0 + k;
            xyzs[i * 3 + 0] = f_add(ray.o[0], f_mul(tt, ray.d[0]));
            xyzs[i * 3 + 1] = f_add(ray.o[1], f_mul(tt, ray.d[1]));
            xyzs[i * 3 + 2] = f_add(ray.o[2], f_mul(tt, ray.d[2]));
            dirs[i * 3 + 0] = ray.d[0];
            dirs[i * 3 + 1] = ray.d[1];
            dirs[i * 3 + 2] = ray.d[2];
            ts[i] = tt;
            deltas[i] = calc_dt(tt, p.esf, p.dt_max);
        }
    }
}

// The single-pass march (kMode 2: the graph-captured training step, render_frame) is held to 12 CTAs per SM, i.e. at
// most 40 registers; left to itself ptxas gives it 47 and 10 CTAs.  0 leaves the other modes unconstrained.
template <int kMode>
__global__ void __launch_bounds__(kRaysPerBlock * 32, kMode == 2 ? 12 : 0)
march_train_warp_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                        const float* __restrict__ hits_t, const float* __restrict__ noise, MarchParams p,
                        int max_samples, int32_t* __restrict__ rays_a, int32_t* __restrict__ counter,
                        float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas,
                        float* __restrict__ ts, int64_t n, int64_t capacity, RoundArgs round) {
    __shared__ float sbuf[kMode >= 2 ? kRaysPerBlock * kMaxFrameSamples : 1];
    float* my_buf = sbuf + (kMode >= 2 ? (threadIdx.x >> 5) * kMaxFrameSamples : 0);
    if (kMode == 3) {
        // persistent warps over the compacted list of live rays
        const int64_t n_alive = min((int64_t)max(*round.n_alive, 0), n);
        if (n_alive == 0) return;
        RoundArgs ra = round;
        ra.limit = (int)max((int64_t)1, min((int64_t)round.limit, capacity / n_alive));
        for (int64_t slot = (int64_t)blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5); slot < n_alive;
             slot += (int64_t)gridDim.x * kRaysPerBlock)
            march_one_ray<3>(rays_o, rays_d, hits_t, noise, p, ra.limit, rays_a, counter, xyzs, dirs, deltas, ts,
                             (int64_t)round.alive[slot], slot, capacity, my_buf, ra);
        return;
    }
    const int64_t r = (int64_t)blockIdx.x * kRaysPerBlock + (threadIdx.x >> 5);
    if (r >= n) return;
    march_one_ray<kMode>(rays_o, rays_d, hits_t, noise, p, max_samples, rays_a, counter, xyzs, dirs, deltas, ts, r, r,
                         capacity, my_buf, round);
}

// exclusive scan of rays_a[:,2] into rays_a[:,1] by one CTA; counter = (total, n_rays)
__global__ void __launch_bounds__(1024) march_scan_kernel(int32_t* __restrict__ rays_a,
                                                          int32_t* __restrict__ counter, int64_t n) {
    __shared__ int32_t warp_tot[32];
    __shared__ int32_t carry_s;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) carry_s = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += 1024) {
        const int64_t r = base + tid;
        const int32_t v = r < n ? rays_a[r * 3 + 2] : 0;
        int32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int32_t nb = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += nb;
        }
        if (lane == 31) warp_tot[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            int32_t w = warp_tot[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int32_t nb = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += nb;
            }
            warp_tot[lane] = w;  // inclusive over warps
        }
        __syncthreads();
        const int32_t carry = carry_s;
        const int32_t warp_off = wid == 0 ? 0 : warp_tot[wid - 1];
        if (r < n) rays_a[r * 3 + 1] = carry + warp_off + incl - v;
        __syncthreads();
        if (tid == 1023) carry_s = carry + warp_tot[31];
        __syncthreads();
    }
    if (tid == 0) {
        counter[0] = carry_s;
        counter[1] = (int32_t)n;
    }
}

// ---- a3 ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) march_test_kernel(const float* __restrict__ rays_o,
                                                         const float* __restrict__ rays_d,
                                                         float* __restrict__ hits_t,
                                                         const int64_t* __restrict__ alive, MarchParams p,
                                                         int max_samples, int64_t* __restrict__ ray_indices,
                                                         uint8_t* __restrict__ valid_mask,
                                                         float* __restrict__ deltas, float* __restrict__ ts,
                                                         int32_t* __restrict__ samples_counter, int64_t n_alive) {
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int64_t r = alive[n];
    Ray ray;
    load_ray(rays_o, rays_d, r, ray);
    float t = hits_t[r * 2 + 0];
    const float t2 = hits_t[r * 2 + 1];
    int s = 0;
    const int64_t base = n * (int64_t)max_samples;
    float xyz[3], dt;
    float t_resume = t;  // t right after the last emitted sample (ray_march.py:256-257)
    while (0.0f < t && t < t2 && s < max_samples) {  // ray_march.py:226 (strict 0 < t)
        if (march_step(p, ray, t, xyz, dt)) {
            const int64_t i = base + s;
            ray_indices[i] = r;
            valid_mask[i] = 1;
            ts[i] = t;
            deltas[i] = dt;
            t = march_advance(t, dt);
            t_resume = t;
            s += 1;
        }
    }
    if (s > 0) hits_t[r * 2 + 0] = t_resume;
    samples_counter[n] = s;
}

MarchParams make_params(const uint8_t* bits, int cascades, int grid_size, float scale, float esf) {
    MarchParams p;
    p.bits = bits;
    p.cascades = cascades;
    p.grid_size = grid_size;
    p.gsf = (float)grid_size;
    p.gs_inv = 1.0f / p.gsf;
    p.gs3 = (uint32_t)grid_size * (uint32_t)grid_size * (uint32_t)grid_size;
    p.scale = scale;
    p.esf = esf;
    // SQRT3_2 * scale / grid_size in fp32, mul then div (utils.py:56-57); host IEEE fp32
    volatile float m = kSqrt3x2 * scale;
    p.dt_max = m / p.gsf;
    return p;
}

}  // namespace

extern "C" {

int ngp_ray_aabb_intersect(const float* rays_o, const float* rays_d, float scale, float* hits_t,
                           int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_o && rays_d && hits_t, "null pointer");
    const int block = 256;
    ray_aabb_kernel<<<(unsigned)((n_rays + block - 1) / block), block, 0, ngp::as_stream(stream)>>>(
        rays_o, rays_d, scale, hits_t, n_rays);
    NGP_LAUNCHED("ray_aabb_kernel");
    return 0;
}

int ngp_raymarching_train_count(const float* rays_o, const float* rays_d, const float* hits_t,
                                const uint8_t* density_bitfield, const float* noise, int cascades,
                                int grid_size, float scale, float exp_step_factor, int max_samples,
                                int32_t* counter, int32_t* rays_a, int64_t n_rays, void* stream) {
    NGP_REQUIRE(n_rays >= 0, "negative n_rays");
    NGP_REQUIRE(counter && (n_rays == 0 || (rays_o && rays_d && hits_t && density_bitfield && noise && rays_a)),
                "null pointer");
    NGP_REQUIRE(cascades >= 1 && grid_size >= 1 && grid_size <= 1024, "bad grid");
    cudaStream_t st = ngp::as_stream(stream);
    const MarchParams p = make_params(density_bitfield, cascades, grid_size, scale, exp_step_factor);
    if (n_rays > 0) {
        const unsigned grid = (unsigned)((n_rays + kRaysPerBlock - 1) / kRaysPerBlock);
        march_train_warp_kernel<0><<<grid, kRaysPerBlock * 32, 0, st>>>(
            rays_o, rays_d, hits_t, noise, p, max_samples, rays_a, counter, nullptr, nullptr, nullptr, nullptr,
            n_rays, 0, RoundArgs{});
        NGP_LAUNCHED("march_train_warp_kernel<count>");
    }
    march_scan_kernel<<<1, 1024, 0, st>>>(rays_a, counter, n_rays);
    NGP_LAUNCHED("march_scan_kernel");
    return 0;
}

int ngp_raymarching_train_write(const float* rays_o, const float* rays_d, const float* hits_t,
                                const uint8_t* density_bitfield, const float* noise, int cascades,
                                int grid_size, float scale, float exp_step_factor, int32_t* counter,
                                int32_t* rays_a, float* xyzs, float* dirs, float* deltas, float* ts,
                                int64_t n_rays, int64_t capacity, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && capacity >= 0, "negative size");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_o && rays_d && hits_t && density_bitfield && noise && rays_a && counter, "null pointer");
    NGP_REQUIRE(capacity == 0 || (xyzs && dirs && deltas && ts), "null output");
    const MarchParams p = make_params(density_bitfield, cascades, grid_size, scale, exp_step_factor);
    const unsigned grid = (unsigned)((n_rays + kRaysPerBlock - 1) / kRaysPerBlock);
    march_train_warp_kernel<1><<<grid, kRaysPerBlock * 32, 0, ngp::as_stream(stream)>>>(
        rays_o, rays_d, hits_t, noise, p, 0, rays_a, counter, xyzs, dirs, deltas, ts, n_rays, capacity, RoundArgs{});
    NGP_LAUNCHED("march_train_warp_kernel<write>");
    return 0;
}

int ngp_raymarching_frame(const float* rays_o, const float* rays_d, const float* hits_t, const float* noise,
                          const uint8_t* density_bitfield, int cascades, int grid_size, float scale,
                          float exp_step_factor, int max_samples, int32_t* counter, int32_t* rays_a, float* xyzs,
                          float* dirs, float* deltas, float* ts, int64_t n_rays, int64_t capacity, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && capacity >= 0, "negative size");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_o && rays_d && hits_t && density_bitfield && counter && rays_a, "null pointer");
    NGP_REQUIRE(capacity == 0 || (xyzs && dirs && deltas && ts), "null output");
    NGP_REQUIRE(max_samples >= 1 && max_samples <= kMaxFrameSamples, "max_samples must be in [1, 1024]");
    const MarchParams p = make_params(density_bitfield, cascades, grid_size, scale, exp_step_factor);
    const unsigned grid = (unsigned)((n_rays + kRaysPerBlock - 1) / kRaysPerBlock);
    march_train_warp_kernel<2><<<grid, kRaysPerBlock * 32, 0, ngp::as_stream(stream)>>>(
        rays_o, rays_d, hits_t, noise, p, max_samples, rays_a, counter, xyzs, dirs, deltas, ts, n_rays, capacity,
        RoundArgs{});
    NGP_LAUNCHED("march_train_warp_kernel<frame>");
    return 0;
}


int ngp_raymarching_round(const float* rays_o, const float* rays_d, const float* hits_t,
                          const uint8_t* density_bitfield, int cascades, int grid_size, float scale,
                          float exp_step_factor, int limit, int max_samples, const int32_t* alive, int32_t* state,
                          float* t_cur, int32_t* n_marched, int32_t* rays_a, float* xyzs, float* dirs, float* deltas,
                          float* ts, int64_t n_rays, int64_t capacity, void* stream) {
    NGP_REQUIRE(n_rays >= 0 && capacity >= 1, "bad size");
    if (n_rays == 0) return 0;
    NGP_REQUIRE(rays_o && rays_d && hits_t && density_bitfield && alive && state && t_cur && n_marched && rays_a &&
                    xyzs && dirs && deltas && ts, "null pointer");
    NGP_REQUIRE(limit >= 1 && limit <= kMaxFrameSamples, "limit must be in [1, 1024]");
    NGP_REQUIRE(max_samples >= 1, "max_samples must be >= 1");
    const MarchParams p = make_params(density_bitfield, cascades, grid_size, scale, exp_step_factor);
    RoundArgs ra;
    ra.alive = alive;
    ra.n_alive = state + 2;
    ra.t_cur = t_cur;
    ra.n_marched = n_marched;
    ra.max_samples = max_samples;
    ra.limit = limit;
    // persistent warps: a few CTAs per SM walk the live list (16 KB of shared memory and 128 threads per CTA)
    const int64_t want = (n_rays + kRaysPerBlock - 1) / kRaysPerBlock;
    const int64_t cap_ctas = (int64_t)ngp::sm_count() * 12;
    const unsigned grid = (unsigned)(want < cap_ctas ? want : cap_ctas);
    march_train_warp_kernel<3><<<grid, kRaysPerBlock * 32, 0, ngp::as_stream(stream)>>>(
        rays_o, rays_d, hits_t, nullptr, p, limit, rays_a, state, xyzs, dirs, deltas, ts, n_rays, capacity, ra);
    NGP_LAUNCHED("march_train_warp_kernel<round>");
    return 0;
}

int ngp_raymarching_test(const float* rays_o, const float* rays_d, float* hits_t, const int64_t* alive_indices,
                         const uint8_t* density_bitfield, int cascades, int grid_size, float scale,
                         float exp_step_factor, int max_samples, int64_t* ray_indices, uint8_t* valid_mask,
                         float* deltas, float* ts, int32_t* samples_counter, int64_t n_alive, void* stream) {
    NGP_REQUIRE(n_alive >= 0, "negative n_alive");
    if (n_alive == 0) return 0;
    NGP_REQUIRE(rays_o && rays_d && hits_t && alive_indices && density_bitfield && ray_indices && valid_mask &&
                    deltas && ts && samples_counter,
                "null pointer");
    const MarchParams p = make_params(density_bitfield, cascades, grid_size, scale, exp_step_factor);
    const int block = 128;
    march_test_kernel<<<(unsigned)((n_alive + block - 1) / block), block, 0, ngp::as_stream(stream)>>>(
        rays_o, rays_d, hits_t, alive_indices, p, max_samples, ray_indices, valid_mask, deltas, ts,
        samples_counter, n_alive);
    NGP_LAUNCHED("march_test_kernel");
    return 0;
}

}  // extern "C"
