// optim.cu — fused optimizer pass: GradScaler unscale + inf-skip + Adam + fp16 shadow refresh +
// gradient zeroing in ONE read-modify-write sweep over the parameters.
//
// Replaces, for the hot path, the separate passes of the reference's step (train.py:197-201):
// optimizer.zero_grad (4 B/param write), GradScaler.unscale_ (8 B/param), torch.optim.Adam /
// apex FusedAdam (28 B/param) and the per-forward `hash_table.to(float16)` cast
// (modules/hash_encoder_half.py:367, 6 B/param).  Here: read p,g,m,v (16 B) + write p,m,v,g=0
// (16 B) + write fp16 shadow (2 B) = 34 B/param, a pure HBM-streaming kernel (roofline: HBM).
// Arithmetic follows torch/optim/adam.py::_single_tensor_adam.
#include "common.cuh"

namespace {

struct AdamArgs {
    float lr_over_bc1;   // lr / (1 - beta1^t)
    float bc2_sqrt;      // sqrt(1 - beta2^t)
    float beta1, beta2, eps, inv_scale;
    int zero_grad;
};

// The FMA contractions are spelled out: left to nvcc they differed between the fp32- and fp16-gradient instantiations
// (v * beta2 rounded first in one, ((1-beta2)*gg)*gg in the other), so the multi-GPU fp16 path drifted by an ulp from
// the single-GPU path on identical gradients.  These are the contractions the fp32 instantiation had.
__device__ __forceinline__ void adam1(float& p, float& g, float& m, float& v, const AdamArgs& a) {
    const float gg = __fmul_rn(g, a.inv_scale);
    m = __fmaf_rn(__fsub_rn(gg, m), 1.0f - a.beta1, m);                           // exp_avg.lerp_(grad, 1-beta1)
    v = __fmaf_rn(v, a.beta2, __fmul_rn(__fmul_rn(1.0f - a.beta2, gg), gg));       // .mul_(beta2).addcmul_(g,g,1-beta2)
    const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), a.bc2_sqrt), a.eps);
    p = __fmaf_rn(-a.lr_over_bc1, __fdiv_rn(m, denom), p);
}

// TGrad = float: the gradient is read from (and zeroed in) `grad`.  TGrad = __half: the gradient comes from the fp16
// transport buffer of the multi-GPU all-reduce (`grad_in`), the fp32 accumulation buffer `grad` is only zeroed.
template <typename TGrad>
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ param, float* __restrict__ grad,
                                                   const TGrad* __restrict__ grad_in,
                                                   float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                   __half* __restrict__ shadow, const int32_t* __restrict__ found_inf,
                                                   const float* __restrict__ hyper_dev, AdamArgs a, int64_t n) {
    const bool skip = found_inf != nullptr && *found_inf != 0;
    if (hyper_dev != nullptr) {  // per-step scalars from device memory (graph-captured step)
        a.lr_over_bc1 = hyper_dev[0];
        a.bc2_sqrt = hyper_dev[1];
        a.inv_scale = hyper_dev[2];
    }
    const int64_t n4 = n >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        if (!skip) {
            float4 p = reinterpret_cast<float4*>(param)[i];
            float4 g;
            if constexpr (sizeof(TGrad) == 4) {
                g = reinterpret_cast<const float4*>(grad_in)[i];
            } else {
                const uint2 raw = reinterpret_cast<const uint2*>(grad_in)[i];
                const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
                const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
                g = make_float4(lo.x, lo.y, hi.x, hi.y);
            }
            float4 m = reinterpret_cast<float4*>(exp_avg)[i];
            float4 v = reinterpret_cast<float4*>(exp_avg_sq)[i];
            adam1(p.x, g.x, m.x, v.x, a);
            adam1(p.y, g.y, m.y, v.y, a);
            adam1(p.z, g.z, m.z, v.z, a);
            adam1(p.w, g.w, m.w, v.w, a);
            reinterpret_cast<float4*>(param)[i] = p;
            reinterpret_cast<float4*>(exp_avg)[i] = m;
            reinterpret_cast<float4*>(exp_avg_sq)[i] = v;
            if (shadow) {
                __half2 lo = __floats2half2_rn(p.x, p.y), hi = __floats2half2_rn(p.z, p.w);
                uint2 pk;
                pk.x = *reinterpret_cast<uint32_t*>(&lo);
                pk.y = *reinterpret_cast<uint32_t*>(&hi);
                reinterpret_cast<uint2*>(shadow)[i] = pk;
            }
        }
        if (a.zero_grad && grad != nullptr) reinterpret_cast<float4*>(grad)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // tail (n not a multiple of 4)
    for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (!skip) {
            float p = param[i], g = load_as_float(grad_in, i), m = exp_avg[i], v = exp_avg_sq[i];
            adam1(p, g, m, v, a);
            param[i] = p;
            exp_avg[i] = m;
            exp_avg_sq[i] = v;
            if (shadow) shadow[i] = __float2half_rn(p);
        }
        if (a.zero_grad && grad != nullptr) grad[i] = 0.0f;
    }
}

// fp32 gradient -> fp16 transport buffer (the reference's own gradients are fp16 under autocast); a value that does not
// fit fp16 becomes inf and is caught by the finite check on the reduced buffer
__global__ void __launch_bounds__(256) grad_pack_f16_kernel(const float* __restrict__ grad, __half* __restrict__ out,
                                                            int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 g = reinterpret_cast<const float4*>(grad)[i];
        const __half2 lo = __floats2half2_rn(g.x, g.y), hi = __floats2half2_rn(g.z, g.w);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&lo);
        pk.y = *reinterpret_cast<const uint32_t*>(&hi);
        reinterpret_cast<uint2*>(out)[i] = pk;
    }
    for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        out[i] = __float2half_rn(grad[i]);
}

__global__ void __launch_bounds__(256) check_finite_f16_kernel(const __half* __restrict__ grad, int64_t n,
                                                               int32_t* __restrict__ found_inf) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    bool bad = false;
    const int64_t n8 = n >> 3;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) {
        const uint4 raw = reinterpret_cast<const uint4*>(grad)[i];
        const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int k = 0; k < 4; ++k)   // exponent all ones = inf or NaN, per half
            bad |= ((w[k] & 0x7c00u) == 0x7c00u) | ((w[k] & 0x7c000000u) == 0x7c000000u);
    }
    for (int64_t i = (n8 << 3) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        bad |= (__half_as_ushort(grad[i]) & 0x7c00u) == 0x7c00u;
    if (__syncthreads_or(bad) && threadIdx.x == 0) *found_inf = 1;
}

// hyper = [lr / bc1, sqrt(bc2), inv_scale, Adam step count t (int bits)].  The LR schedule follows the iteration count
// (scheduler.step() runs every iteration, train.py:199-201) while Adam's bias-correction count t only advances on steps
// that are applied: GradScaler.step skips optimizer.step() when the gradients hold an inf/NaN.
__global__ void adam_hyper_kernel(int32_t* __restrict__ step_dev, float lr0, float lr_min, int32_t max_steps, float beta1,
                                  float beta2, float inv_scale, const int32_t* __restrict__ found_inf,
                                  float* __restrict__ hyper) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int32_t s = *step_dev;  // 0-based index of the iteration being taken
    const double frac = (double)min(s, max_steps) / (double)max(max_steps, 1);
    const double lr = (double)lr_min + ((double)lr0 - (double)lr_min) * (1.0 + cos(3.14159265358979323846 * frac)) / 2.0;
    const bool skipped = found_inf != nullptr && *found_inf != 0;
    const int32_t t_applied = __float_as_int(hyper[3]) + (skipped ? 0 : 1);
    hyper[3] = __int_as_float(t_applied);
    const double t = (double)max(t_applied, 1);
    const double bc1 = 1.0 - pow((double)beta1, t), bc2 = 1.0 - pow((double)beta2, t);
    hyper[0] = (float)(lr / bc1);
    hyper[1] = (float)sqrt(bc2);
    if (inv_scale > 0.0f) hyper[2] = inv_scale;  // <= 0: leave the value maintained by ngp_loss_scale_update
    *step_dev = s + 1;
}

// per-step scalar housekeeping in one launch (each pointer optional)
__global__ void step_reset_kernel(int32_t* __restrict__ counter2, float* __restrict__ loss_sum,
                                  int32_t* __restrict__ found_inf, int32_t* __restrict__ batch_counter) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (counter2) counter2[0] = counter2[1] = 0;
    if (loss_sum) *loss_sum = 0.0f;
    if (found_inf) *found_inf = 0;
    if (batch_counter) *batch_counter += 1;
}

// GradScaler.update(): torch/amp/grad_scaler.py -> _amp_update_scale_
__global__ void loss_scale_update_kernel(float* __restrict__ state, int32_t* __restrict__ found_inf, float growth,
                                         float backoff, int32_t interval, float world, float* __restrict__ hyper,
                                         int clear_found_inf) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float scale = state[0];
    int32_t tracker = __float_as_int(state[1]);
    if (found_inf != nullptr && *found_inf != 0) {
        scale *= backoff;
        tracker = 0;
    } else {
        tracker += 1;
        if (tracker >= interval) {
            const float grown = scale * growth;
            if (grown < INFINITY) scale = grown;
            tracker = 0;
        }
    }
    state[0] = scale;
    state[1] = __int_as_float(tracker);
    if (hyper != nullptr) hyper[2] = 1.0f / (scale * world);
    // last reader of the step's flag: hand a clean one to the next backward (kernels that raise it at the source)
    if (clear_found_inf && found_inf != nullptr) *found_inf = 0;
}

__global__ void __launch_bounds__(256) check_finite_kernel(const float* __restrict__ grad, int64_t n,
                                                           int32_t* __restrict__ found_inf) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    bool bad = false;
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 g = reinterpret_cast<const float4*>(grad)[i];
        // |x| < inf is false for inf and NaN
        bad |= !(fabsf(g.x) < INFINITY) | !(fabsf(g.y) < INFINITY) | !(fabsf(g.z) < INFINITY) | !(fabsf(g.w) < INFINITY);
    }
    for (int64_t i = (n4 << 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
        bad |= !(fabsf(grad[i]) < INFINITY);
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicExch(found_inf, 1);
}

// ---- the node block B of a voxel field (DESIGN.md §6b) ------------------------------------------------------------
// A field [G, G, G, C] restricted to B = [lo, hi) per axis is nx * ny runs, one per (x, y), of nz * C contiguous
// floats.  One CTA walks one run at a time with scalar, coalesced accesses (a run starts at any float); the CTAs
// stride over the runs.  Offsets are int64: a degree-2 field passes 2^31 floats at G >= 431.
struct BlockRuns {
    int64_t G, C;
    int32_t lo_x, lo_y, lo_z, ny;
    int64_t runs, run_len;
};

__device__ __forceinline__ int64_t run_base(const BlockRuns& b, int64_t r) {
    const int64_t i = b.lo_x + r / b.ny, j = b.lo_y + r % b.ny;
    return ((i * b.G + j) * b.G + b.lo_z) * b.C;
}

__global__ void __launch_bounds__(256) adam_block_kernel(float* __restrict__ param, float* __restrict__ grad,
                                                         float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                         const int32_t* __restrict__ found_inf,
                                                         const float* __restrict__ hyper_dev, AdamArgs a,
                                                         const BlockRuns b) {
    const bool skip = found_inf != nullptr && *found_inf != 0;
    a.lr_over_bc1 = hyper_dev[0];
    a.bc2_sqrt = hyper_dev[1];
    a.inv_scale = hyper_dev[2];
    for (int64_t r = blockIdx.x; r < b.runs; r += gridDim.x) {
        const int64_t base = run_base(b, r);
        for (int64_t e = threadIdx.x; e < b.run_len; e += blockDim.x) {
            const int64_t k = base + e;
            if (!skip) {
                float p = param[k], g = grad[k], m = exp_avg[k], v = exp_avg_sq[k];
                adam1(p, g, m, v, a);
                param[k] = p;
                exp_avg[k] = m;
                exp_avg_sq[k] = v;
            }
            grad[k] = 0.0f;
        }
    }
}

__global__ void __launch_bounds__(256) check_finite_block_kernel(const float* __restrict__ grad, const BlockRuns b,
                                                                 int32_t* __restrict__ found_inf) {
    bool bad = false;
    for (int64_t r = blockIdx.x; r < b.runs; r += gridDim.x) {
        const int64_t base = run_base(b, r);
        for (int64_t e = threadIdx.x; e < b.run_len; e += blockDim.x) bad |= !(fabsf(grad[base + e]) < INFINITY);
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicExch(found_inf, 1);
}

int block_runs(int32_t grid, int32_t channels, const int32_t* block6, BlockRuns& b) {
    NGP_REQUIRE(grid >= 1, "grid must be >= 1");
    NGP_REQUIRE(channels >= 1, "channels must be >= 1");
    NGP_REQUIRE(block6 != nullptr, "null block");
    for (int k = 0; k < 3; ++k)
        NGP_REQUIRE(block6[k] >= 0 && block6[k] < block6[k + 3] && block6[k + 3] <= grid,
                    "block bounds must satisfy 0 <= lo < hi <= grid on every axis");
    b.G = grid;
    b.C = channels;
    b.lo_x = block6[0];
    b.lo_y = block6[1];
    b.lo_z = block6[2];
    b.ny = block6[4] - block6[1];
    b.runs = (int64_t)(block6[3] - block6[0]) * b.ny;
    b.run_len = (int64_t)(block6[5] - block6[2]) * channels;
    return 0;
}

unsigned block_grid(const BlockRuns& b) {   // one run per CTA (B has at most 2048^2 runs)
    return (unsigned)min(b.runs, (int64_t)INT32_MAX);
}

}  // namespace

extern "C" {

int ngp_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq, void* param_f16_or_null,
                  const int32_t* found_inf_or_null, float lr, float beta1, float beta2, float eps, float inv_scale,
                  int32_t step, int zero_grad, int64_t n, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    NGP_REQUIRE(step >= 1, "step is 1-based");
    if (n == 0) return 0;
    NGP_REQUIRE(param && grad && exp_avg && exp_avg_sq, "null pointer");
    const uintptr_t al = reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) |
                         reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq);
    NGP_REQUIRE((al & 15) == 0, "param/grad/state must be 16-byte aligned");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(param_f16_or_null) & 7) == 0, "fp16 shadow must be 8-byte aligned");
    AdamArgs a;
    const double bc1 = 1.0 - pow((double)beta1, (double)step);
    const double bc2 = 1.0 - pow((double)beta2, (double)step);
    a.lr_over_bc1 = (float)((double)lr / bc1);
    a.bc2_sqrt = (float)sqrt(bc2);
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.inv_scale = inv_scale;
    a.zero_grad = zero_grad;
    const int64_t work = (n + 3) / 4;
    const int64_t max_blocks = (int64_t)ngp::sm_count() * 8;
    const unsigned grid = (unsigned)min((work + 255) / 256, max_blocks);
    adam_kernel<float><<<grid, 256, 0, ngp::as_stream(stream)>>>(param, grad, grad, exp_avg, exp_avg_sq,
                                                                 (__half*)param_f16_or_null, found_inf_or_null, nullptr, a, n);
    NGP_LAUNCHED("adam_kernel");
    return 0;
}

int ngp_adam_step_dyn(float* param, float* grad, float* exp_avg, float* exp_avg_sq, void* param_f16_or_null,
                      const int32_t* found_inf_or_null, const float* hyper_dev, float beta1, float beta2, float eps,
                      int zero_grad, int64_t n, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    NGP_REQUIRE(param && grad && exp_avg && exp_avg_sq && hyper_dev, "null pointer");
    const uintptr_t al = reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) |
                         reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq);
    NGP_REQUIRE((al & 15) == 0, "param/grad/state must be 16-byte aligned");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(param_f16_or_null) & 7) == 0, "fp16 shadow must be 8-byte aligned");
    AdamArgs a;
    a.lr_over_bc1 = 0.f;
    a.bc2_sqrt = 1.f;
    a.inv_scale = 1.f;
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.zero_grad = zero_grad;
    const int64_t work = (n + 3) / 4;
    const int64_t max_blocks = (int64_t)ngp::sm_count() * 8;
    const unsigned grid = (unsigned)min((work + 255) / 256, max_blocks);
    adam_kernel<float><<<grid, 256, 0, ngp::as_stream(stream)>>>(param, grad, grad, exp_avg, exp_avg_sq,
                                                                 (__half*)param_f16_or_null, found_inf_or_null, hyper_dev, a, n);
    NGP_LAUNCHED("adam_kernel");
    return 0;
}

int ngp_adam_step_dyn_g16(float* param, const void* grad_f16, float* grad_f32_to_zero_or_null, float* exp_avg,
                          float* exp_avg_sq, void* param_f16_or_null, const int32_t* found_inf_or_null,
                          const float* hyper_dev, float beta1, float beta2, float eps, int64_t n, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    NGP_REQUIRE(param && grad_f16 && exp_avg && exp_avg_sq && hyper_dev, "null pointer");
    const uintptr_t al = reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad_f32_to_zero_or_null) |
                         reinterpret_cast<uintptr_t>(exp_avg) | reinterpret_cast<uintptr_t>(exp_avg_sq);
    NGP_REQUIRE((al & 15) == 0, "param/grad/state must be 16-byte aligned");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(grad_f16) & 7) == 0, "fp16 gradient must be 8-byte aligned");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(param_f16_or_null) & 7) == 0, "fp16 shadow must be 8-byte aligned");
    AdamArgs a;
    a.lr_over_bc1 = 0.f;
    a.bc2_sqrt = 1.f;
    a.inv_scale = 1.f;
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.zero_grad = 1;
    const int64_t work = (n + 3) / 4;
    const int64_t max_blocks = (int64_t)ngp::sm_count() * 8;
    const unsigned grid = (unsigned)min((work + 255) / 256, max_blocks);
    adam_kernel<__half><<<grid, 256, 0, ngp::as_stream(stream)>>>(param, grad_f32_to_zero_or_null, (const __half*)grad_f16,
                                                                  exp_avg, exp_avg_sq, (__half*)param_f16_or_null,
                                                                  found_inf_or_null, hyper_dev, a, n);
    NGP_LAUNCHED("adam_kernel<f16 grad>");
    return 0;
}

int ngp_grad_pack_f16(const float* grad, void* out_f16, int64_t n, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    NGP_REQUIRE(grad && out_f16, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(grad) & 15) == 0 && (reinterpret_cast<uintptr_t>(out_f16) & 7) == 0,
                "grad must be 16-byte, out 8-byte aligned");
    const int64_t work = (n + 3) / 4;
    const unsigned grid = (unsigned)min((work + 255) / 256, (int64_t)ngp::sm_count() * 8);
    grad_pack_f16_kernel<<<grid, 256, 0, ngp::as_stream(stream)>>>(grad, (__half*)out_f16, n);
    NGP_LAUNCHED("grad_pack_f16_kernel");
    return 0;
}

int ngp_check_finite_f16(const void* grad_f16, int64_t n, int32_t* found_inf, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    NGP_REQUIRE(grad_f16 && found_inf, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(grad_f16) & 15) == 0, "grad must be 16-byte aligned");
    const int64_t work = (n + 7) / 8;
    const unsigned grid = (unsigned)min((work + 255) / 256, (int64_t)ngp::sm_count() * 8);
    check_finite_f16_kernel<<<grid, 256, 0, ngp::as_stream(stream)>>>((const __half*)grad_f16, n, found_inf);
    NGP_LAUNCHED("check_finite_f16_kernel");
    return 0;
}

int ngp_adam_hyper_update(int32_t* step_dev, float lr0, float lr_min, int32_t max_steps, float beta1, float beta2,
                          float inv_scale, const int32_t* found_inf_or_null, float* hyper_dev, void* stream) {
    NGP_REQUIRE(step_dev && hyper_dev, "null pointer");
    adam_hyper_kernel<<<1, 32, 0, ngp::as_stream(stream)>>>(step_dev, lr0, lr_min, max_steps, beta1, beta2, inv_scale,
                                                            found_inf_or_null, hyper_dev);
    NGP_LAUNCHED("adam_hyper_kernel");
    return 0;
}

int ngp_loss_scale_update(float* state_dev, int32_t* found_inf, float growth, float backoff,
                          int32_t growth_interval, float world_size, float* hyper_dev, int clear_found_inf,
                          void* stream) {
    NGP_REQUIRE(state_dev != nullptr, "null pointer");
    NGP_REQUIRE(growth >= 1.0f && backoff > 0.0f && backoff <= 1.0f && growth_interval >= 1, "bad GradScaler constants");
    loss_scale_update_kernel<<<1, 32, 0, ngp::as_stream(stream)>>>(state_dev, found_inf, growth, backoff, growth_interval,
                                                                   world_size, hyper_dev, clear_found_inf);
    NGP_LAUNCHED("loss_scale_update_kernel");
    return 0;
}

int ngp_step_reset(int32_t* march_counter2, float* loss_sum, int32_t* found_inf, int32_t* batch_counter, void* stream) {
    step_reset_kernel<<<1, 32, 0, ngp::as_stream(stream)>>>(march_counter2, loss_sum, found_inf, batch_counter);
    NGP_LAUNCHED("step_reset_kernel");
    return 0;
}

int ngp_check_finite(const float* grad, int64_t n, int32_t* found_inf, void* stream) {
    NGP_REQUIRE(n >= 0, "negative n");
    if (n == 0) return 0;
    NGP_REQUIRE(grad && found_inf, "null pointer");
    NGP_REQUIRE((reinterpret_cast<uintptr_t>(grad) & 15) == 0, "grad must be 16-byte aligned");
    const int64_t work = (n + 3) / 4;
    const int64_t max_blocks = (int64_t)ngp::sm_count() * 8;
    const unsigned grid = (unsigned)min((work + 255) / 256, max_blocks);
    check_finite_kernel<<<grid, 256, 0, ngp::as_stream(stream)>>>(grad, n, found_inf);
    NGP_LAUNCHED("check_finite_kernel");
    return 0;
}

int ngp_check_finite_voxel_block(const float* grad, int32_t grid, int32_t channels, const int32_t* block6,
                                 int32_t* found_inf, void* stream) {
    BlockRuns b;
    if (int rc = block_runs(grid, channels, block6, b)) return rc;
    NGP_REQUIRE(grad && found_inf, "null pointer");
    check_finite_block_kernel<<<block_grid(b), 256, 0, ngp::as_stream(stream)>>>(grad, b, found_inf);
    NGP_LAUNCHED("check_finite_block_kernel");
    return 0;
}

int ngp_adam_step_voxel_block_dyn(float* param, float* grad, float* exp_avg, float* exp_avg_sq, int32_t grid,
                                  int32_t channels, const int32_t* block6, const int32_t* found_inf_or_null,
                                  const float* hyper_dev, float beta1, float beta2, float eps, void* stream) {
    BlockRuns b;
    if (int rc = block_runs(grid, channels, block6, b)) return rc;
    NGP_REQUIRE(param && grad && exp_avg && exp_avg_sq && hyper_dev, "null pointer");
    AdamArgs a;
    a.lr_over_bc1 = 0.f;
    a.bc2_sqrt = 1.f;
    a.inv_scale = 1.f;
    a.beta1 = beta1;
    a.beta2 = beta2;
    a.eps = eps;
    a.zero_grad = 1;
    adam_block_kernel<<<block_grid(b), 256, 0, ngp::as_stream(stream)>>>(param, grad, exp_avg, exp_avg_sq,
                                                                         found_inf_or_null, hyper_dev, a, b);
    NGP_LAUNCHED("adam_block_kernel");
    return 0;
}

}  // extern "C"
