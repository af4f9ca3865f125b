// wgmma.cuh — PTX wrappers for the Hopper warpgroup tensor-core MMA (wgmma.mma_async, sm_90a), the shared-memory
// matrix descriptor for the no-swizzle layout and the few device helpers shared by the fused MLP kernels (mlp.cu).
//
// A warpgroup (4 warps, 128 threads) computes D[64 x N] (+)= A[64 x 16] * B[16 x N] per instruction.  D is held in
// registers: warp w owns rows 16w..16w+15; with g = lane / 4 and t = lane % 4, thread element 4j+0/4j+1 is
// (row 16w+g, columns 8j+2t, 8j+2t+1) and 4j+2/4j+3 is the same pair on row 16w+g+8.  A may instead come from
// registers in the same arrangement (four fp16 pairs per 16-wide K step), so a layer's fp32 output converts in place
// into the next layer's A operand without a round trip through shared memory.
#pragma once
#include "common.cuh"

namespace ngp_wg {

constexpr int kTile = 64;   // sample rows per tile == wgmma M

// weights in shared memory (fp16, no-swizzle K-major layout), identical in every MLP kernel
constexpr int kW1 = 0;                       // [64 x 32]
constexpr int kW2 = kW1 + 64 * 32 * 2;       // [16 x 64]
constexpr int kW3 = kW2 + 16 * 64 * 2;       // [64 x 32]
constexpr int kW4 = kW3 + 64 * 32 * 2;       // [64 x 64]
constexpr int kW5 = kW4 + 64 * 64 * 2;       // [16 x 64] (rows 3..15 zero)
constexpr int kAct = kW5 + 16 * 64 * 2;      // 20480: first byte after the weights

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// shared-memory writes of the generic proxy become visible to wgmma (async proxy) after this + a barrier
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// ---- descriptors -------------------------------------------------------------------------------------
// shared-memory matrix descriptor, no swizzle (layout type 0): start address, LBO and SBO in 16-byte units.
// The operands are stored as 8x8 fp16 core matrices of 128 contiguous bytes (row stride 16 B).
__host__ __device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// byte offset of the 16-byte chunk (row r, k-chunk kc) inside an operand stored with K columns
__host__ __device__ __forceinline__ int chunk_off(int r, int kc, int K) { return (r >> 3) * (K * 16) + kc * 128 + (r & 7) * 16; }
// descriptor of K step k (16 wide) of an operand stored as [rows][K] and consumed K-major (rows = M or N):
// core matrices adjacent along K are 128 B apart (LBO), 8-row groups K*16 B apart (SBO)
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t addr, int K, int k) { return smem_desc(addr + k * 256, 128, K * 16); }
// the same storage consumed MN-major (transposed): MN = the stored columns, K = the stored rows.  8-row groups
// (along K) are K*16 B apart (LBO), column chunks (along MN) 128 B apart (SBO)
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t addr, int K, int k) { return smem_desc(addr + k * K * 32, K * 16, 128); }

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// relu fused into the conversion; low half = a
__device__ __forceinline__ uint32_t pack_h2_relu(float a, float b) {
    uint32_t r;
    asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
    return r;
}

// copy a row-major fp32 weight [rows x K] into the fp16 operand layout (rows_pad rows, zero padded)
__device__ __forceinline__ void stage_weight(uint8_t* smem, const float* __restrict__ w, int rows, int rows_pad, int K) {
    const int kchunks = K / 8;
    for (int c = threadIdx.x; c < rows_pad * kchunks; c += blockDim.x) {
        const int r = c / kchunks, kc = c % kchunks;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (r < rows) {
            const float4 a = __ldg(reinterpret_cast<const float4*>(w + r * K + kc * 8));
            const float4 b = __ldg(reinterpret_cast<const float4*>(w + r * K + kc * 8 + 4));
            v = make_uint4(pack_h2(a.x, a.y), pack_h2(a.z, a.w), pack_h2(b.x, b.y), pack_h2(b.z, b.w));
        }
        *reinterpret_cast<uint4*>(smem + chunk_off(r, kc, K)) = v;
    }
}
__device__ __forceinline__ void stage_weights(uint8_t* smem, const ngp_mlp_weights& w) {
    stage_weight(smem + kW1, w.w1, 64, 64, 32);
    stage_weight(smem + kW2, w.w2, 16, 16, 64);
    stage_weight(smem + kW3, w.w3, 64, 64, 32);
    stage_weight(smem + kW4, w.w4, 64, 64, 64);
    stage_weight(smem + kW5, w.w5, 3, 16, 64);
}

__device__ __forceinline__ void sh16(float x, float y, float z, float* e) {  // spherical_harmonics.py:16-42
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

// ---- wgmma m64nNk16, fp32 accumulate, fp16 operands.  SS: A and B from shared memory (TA / TB: 1 = MN-major);
// RS: A from registers (four fp16 pairs).  scale_d = 0 overwrites D, 1 accumulates.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n8(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n8(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, %10;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n16(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n16(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, %14;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n32(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n32(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, %22;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB)
        : "memory");
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n64(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB)
        : "memory");
}
template <int TB>
__device__ __forceinline__ void wgmma_rs_n64(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d), "n"(TB)
        : "memory");
}

}  // namespace ngp_wg
