// mesh.cu — mesh export: the density lattice's node positions and mask, and marching cubes over an fp32 lattice
// (DESIGN.md §6g).
//
// Lattice: N nodes per axis over [-b, b]^3, spacing s = f_div(2b, N - 1), node i at f_add(-b, f_mul((float)i, s)),
// stored [ix, iy, iz] with z fastest.  Marching cubes runs in four launches with no atomics, so the output is unique:
//   count  — per tile of kTile consecutive nodes: the vertices the tile's nodes own (one per crossing edge from the
//            node to its +x, +y, +z neighbour) and the triangles of the cells whose lowest node they are;
//   scan   — exclusive scan of the tile counts (one CTA per 1024 tiles, then one CTA over the block sums);
//   emit_vertices — vertices in edge-id order (node_linear * 3 + axis), and each owning node's first vertex id;
//   emit_faces    — triangles in cell order, then table order, each corner resolved through the owner's vertex id.
// Every kernel walks its tile in rounds of kThreads nodes, so consecutive threads read consecutive z.
#include <math.h>

#include "common.cuh"
#include "mc_table.cuh"
#include "occupancy.cuh"

namespace {

constexpr int kThreads = 256;                  // threads per CTA of the count / emit kernels
constexpr int kRounds = 4;                     // node rounds per tile
constexpr int kTile = kThreads * kRounds;      // nodes per tile
constexpr int kScanThreads = 1024;             // tiles per scan block; also the most scan blocks one CTA sums
constexpr int kMaxN = 1024;
constexpr int kPointThreads = 256;

// ---- lattice -------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lattice_spacing(float bound, int n) { return f_div(f_mul(2.0f, bound), (float)(n - 1)); }
__device__ __forceinline__ float node_coord(float bound, float s, int i) { return f_add(-bound, f_mul((float)i, s)); }

struct Occupancy {
    const uint8_t* __restrict__ bits;
    int cascades;
    int grid_size;
    float scale;
};

// march_step's cell test at a position (march.cu), without the dt term of the cascade choice
__device__ __forceinline__ bool occupied(const Occupancy& p, const float x[3]) {
    int mip = 0;
    if (p.cascades > 1) {
        const float mx = fmaxf(fmaxf(fabsf(x[0]), fabsf(x[1])), fabsf(x[2]));
        mip = min(p.cascades - 1, max(0, frexp_bit(mx) + 1));
    }
    const float gsf = (float)p.grid_size;
    const float mip_bound = fminf(__uint_as_float((uint32_t)(127 + mip - 1) << 23), p.scale);
    const float mip_bound_inv = f_div(1.0f, mip_bound);
    uint32_t u[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float v = f_mul(f_mul(0.5f, f_add(f_mul(x[k], mip_bound_inv), 1.0f)), gsf);
        v = fminf(fmaxf(v, 0.0f), f_sub(gsf, 1.0f));
        u[k] = __float2uint_rz(v);
    }
    const uint32_t gs3 = (uint32_t)p.grid_size * p.grid_size * p.grid_size;
    const uint32_t idx = (uint32_t)mip * gs3 + morton3d(u[0], u[1], u[2]);
    return (__ldg(p.bits + (idx >> 3)) >> (idx & 7u)) & 1u;
}

__global__ void __launch_bounds__(kPointThreads) mesh_points_kernel(int n, float bound, int64_t start, int64_t count,
                                                                    Occupancy occ_p, float* __restrict__ xyz,
                                                                    uint8_t* __restrict__ occ) {
    const int64_t j = (int64_t)blockIdx.x * kPointThreads + threadIdx.x;
    if (j >= count) return;
    const int64_t i = start + j;
    const int64_t nn = (int64_t)n * n;
    const int idx[3] = {(int)(i / nn), (int)((i / n) % n), (int)(i % n)};
    const float s = lattice_spacing(bound, n);
    float x[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        x[k] = node_coord(bound, s, idx[k]);
        xyz[j * 3 + k] = x[k];
    }
    occ[j] = occupied(occ_p, x) ? 1 : 0;
}

__global__ void __launch_bounds__(kPointThreads) mesh_store_kernel(const float* __restrict__ sigma,
                                                                   const uint8_t* __restrict__ occ, int64_t start,
                                                                   int64_t count, float* __restrict__ lattice) {
    const int64_t j = (int64_t)blockIdx.x * kPointThreads + threadIdx.x;
    if (j >= count) return;
    const float v = sigma[j];
    lattice[start + j] = (occ[j] && isfinite(v)) ? v : 0.0f;
}

// ---- marching cubes ------------------------------------------------------------------------------------------
struct Lattice {
    const float* __restrict__ v;
    int n;
    float tau;
    __device__ __forceinline__ float at(int x, int y, int z) const { return v[((int64_t)x * n + y) * n + z]; }
    __device__ __forceinline__ bool in(int x, int y, int z) const { return at(x, y, z) > tau; }
};

struct NodeInfo {
    int idx[3];
    uint32_t vmask;   // bit a: the edge to the +a neighbour crosses the surface
    int cube;         // case of the cell whose lowest node this is, -1 past the last cell
};

__device__ __forceinline__ NodeInfo node_info(const Lattice& L, int64_t i) {
    NodeInfo r;
    const int64_t nn = (int64_t)L.n * L.n;
    r.idx[0] = (int)(i / nn);
    r.idx[1] = (int)((i / L.n) % L.n);
    r.idx[2] = (int)(i % L.n);
    const int x = r.idx[0], y = r.idx[1], z = r.idx[2], m = L.n - 1;
    const bool c0 = L.in(x, y, z);
    const bool cx = x < m && L.in(x + 1, y, z);
    const bool cy = y < m && L.in(x, y + 1, z);
    const bool cz = z < m && L.in(x, y, z + 1);
    r.vmask = (x < m && cx != c0 ? 1u : 0u) | (y < m && cy != c0 ? 2u : 0u) | (z < m && cz != c0 ? 4u : 0u);
    r.cube = -1;
    if (x < m && y < m && z < m) {
        r.cube = (int)c0 | (int)cx << 1 | (int)cy << 2 | (int)L.in(x + 1, y + 1, z) << 3 | (int)cz << 4 |
                 (int)L.in(x + 1, y, z + 1) << 5 | (int)L.in(x, y + 1, z + 1) << 6 |
                 (int)L.in(x + 1, y + 1, z + 1) << 7;
    }
    return r;
}

__device__ __forceinline__ int tri_count(const NodeInfo& r) { return r.cube < 0 ? 0 : (int)kMcTriCount[r.cube]; }

// exclusive scan of (a, b) over the CTA (blockDim.x a multiple of 32, at most 1024); the CTA's totals go to *ta, *tb
__device__ __forceinline__ void block_exclusive_scan2(long long& a, long long& b, long long* ta, long long* tb) {
    __shared__ long long wa[32], wb[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    long long sa = a, sb = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long na = __shfl_up_sync(0xffffffffu, sa, o), nb = __shfl_up_sync(0xffffffffu, sb, o);
        if (lane >= o) {
            sa += na;
            sb += nb;
        }
    }
    __syncthreads();   // wa / wb of an earlier call have been read
    if (lane == 31) {
        wa[warp] = sa;
        wb[warp] = sb;
    }
    __syncthreads();
    if (warp == 0) {
        long long xa = lane < n_warps ? wa[lane] : 0, xb = lane < n_warps ? wb[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long na = __shfl_up_sync(0xffffffffu, xa, o), nb = __shfl_up_sync(0xffffffffu, xb, o);
            if (lane >= o) {
                xa += na;
                xb += nb;
            }
        }
        if (lane < n_warps) {
            wa[lane] = xa;
            wb[lane] = xb;
        }
    }
    __syncthreads();
    const long long pa = warp ? wa[warp - 1] : 0, pb = warp ? wb[warp - 1] : 0;
    a = pa + sa - a;
    b = pb + sb - b;
    *ta = wa[n_warps - 1];
    *tb = wb[n_warps - 1];
}

struct Workspace {
    int2* tile_counts;        // [tiles] (vertices, faces) of each tile
    longlong2* tile_off;      // [tiles] exclusive offsets within the tile's scan block
    longlong2* block_sum;     // [blocks]
    longlong2* block_off;     // [blocks] exclusive offsets of the scan blocks
    int64_t tiles, blocks, bytes;
};

Workspace workspace_layout(void* base, int64_t n) {
    Workspace w;
    const int64_t nodes = n * n * n;
    w.tiles = (nodes + kTile - 1) / kTile;
    w.blocks = (w.tiles + kScanThreads - 1) / kScanThreads;
    char* p = (char*)base;
    int64_t off = 0;
    auto take = [&](int64_t bytes) {
        char* q = p ? p + off : nullptr;
        off += (bytes + 255) / 256 * 256;
        return q;
    };
    w.tile_counts = (int2*)take(w.tiles * (int64_t)sizeof(int2));
    w.tile_off = (longlong2*)take(w.tiles * (int64_t)sizeof(longlong2));
    w.block_sum = (longlong2*)take(w.blocks * (int64_t)sizeof(longlong2));
    w.block_off = (longlong2*)take(w.blocks * (int64_t)sizeof(longlong2));
    w.bytes = off;
    return w;
}

__global__ void __launch_bounds__(kThreads) mc_count_kernel(Lattice L, int64_t nodes, int2* __restrict__ tile_counts) {
    const int64_t tile0 = (int64_t)blockIdx.x * kTile;
    int vc = 0, fc = 0;
#pragma unroll
    for (int k = 0; k < kRounds; ++k) {
        const int64_t i = tile0 + k * kThreads + threadIdx.x;
        if (i < nodes) {
            const NodeInfo r = node_info(L, i);
            vc += __popc(r.vmask);
            fc += tri_count(r);
        }
    }
    __shared__ int sv[kThreads / 32], sf[kThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        vc += __shfl_xor_sync(0xffffffffu, vc, o);
        fc += __shfl_xor_sync(0xffffffffu, fc, o);
    }
    if ((threadIdx.x & 31) == 0) {
        sv[threadIdx.x >> 5] = vc;
        sf[threadIdx.x >> 5] = fc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int a = 0, b = 0;
#pragma unroll
        for (int w = 0; w < kThreads / 32; ++w) {
            a += sv[w];
            b += sf[w];
        }
        tile_counts[blockIdx.x] = make_int2(a, b);
    }
}

__global__ void __launch_bounds__(kScanThreads) mc_scan_tiles_kernel(const int2* __restrict__ tile_counts,
                                                                     int64_t tiles, longlong2* __restrict__ tile_off,
                                                                     longlong2* __restrict__ block_sum) {
    const int64_t t = (int64_t)blockIdx.x * kScanThreads + threadIdx.x;
    const int2 c = t < tiles ? tile_counts[t] : make_int2(0, 0);
    long long a = c.x, b = c.y, ta, tb;
    block_exclusive_scan2(a, b, &ta, &tb);
    if (t < tiles) tile_off[t] = make_longlong2(a, b);
    if (threadIdx.x == 0) block_sum[blockIdx.x] = make_longlong2(ta, tb);
}

__global__ void __launch_bounds__(kScanThreads) mc_scan_blocks_kernel(const longlong2* __restrict__ block_sum,
                                                                      int64_t blocks, longlong2* __restrict__ block_off,
                                                                      int64_t* __restrict__ totals) {
    const int t = threadIdx.x;
    const longlong2 c = t < blocks ? block_sum[t] : make_longlong2(0, 0);
    long long a = c.x, b = c.y, ta, tb;
    block_exclusive_scan2(a, b, &ta, &tb);
    if (t < blocks) block_off[t] = make_longlong2(a, b);
    if (t == 0) {
        totals[0] = ta;
        totals[1] = tb;
    }
}

__device__ __forceinline__ long long tile_base_v(const Workspace& w, int64_t tile) {
    return w.block_off[tile / kScanThreads].x + w.tile_off[tile].x;
}
__device__ __forceinline__ long long tile_base_f(const Workspace& w, int64_t tile) {
    return w.block_off[tile / kScanThreads].y + w.tile_off[tile].y;
}

// density gradient component c at node p, in units of 1/spacing: central inside, one-sided on the border
__device__ __forceinline__ float grad_comp(const Lattice& L, const int p[3], int c) {
    int lo[3] = {p[0], p[1], p[2]}, hi[3] = {p[0], p[1], p[2]};
    const bool central = p[c] > 0 && p[c] < L.n - 1;
    if (central) {
        lo[c] -= 1;
        hi[c] += 1;
    } else if (p[c] == 0) {
        hi[c] += 1;
    } else {
        lo[c] -= 1;
    }
    const float d = f_sub(L.at(hi[0], hi[1], hi[2]), L.at(lo[0], lo[1], lo[2]));
    return central ? f_mul(d, 0.5f) : d;
}

__global__ void __launch_bounds__(kThreads) mc_emit_vertices_kernel(Lattice L, int64_t nodes, float bound, Workspace w,
                                                                    int32_t* __restrict__ vbase,
                                                                    float* __restrict__ vertices,
                                                                    float* __restrict__ normals) {
    const int64_t tile = blockIdx.x;
    long long running = tile_base_v(w, tile);
    const float s = lattice_spacing(bound, L.n);
    for (int k = 0; k < kRounds; ++k) {
        const int64_t i = tile * kTile + k * kThreads + threadIdx.x;
        NodeInfo r;
        r.vmask = 0;
        if (i < nodes) r = node_info(L, i);
        long long id = __popc(r.vmask), unused = 0, total, unused_t;
        block_exclusive_scan2(id, unused, &total, &unused_t);
        id += running;
        running += total;
        if (!r.vmask) continue;
        vbase[i] = (int32_t)id;
        float xa[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) xa[c] = node_coord(bound, s, r.idx[c]);
        const float va = L.at(r.idx[0], r.idx[1], r.idx[2]);
        float ga[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) ga[c] = grad_comp(L, r.idx, c);
        for (int axis = 0; axis < 3; ++axis) {
            if (!(r.vmask >> axis & 1u)) continue;
            int pb[3] = {r.idx[0], r.idx[1], r.idx[2]};
            pb[axis] += 1;
            const float vb = L.at(pb[0], pb[1], pb[2]);
            const float t = f_div(f_sub(L.tau, va), f_sub(vb, va));
            float m[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float gb = grad_comp(L, pb, c);
                m[c] = f_add(ga[c], f_mul(t, f_sub(gb, ga[c])));
                vertices[id * 3 + c] = c == axis ? f_add(xa[c], f_mul(t, s)) : xa[c];
            }
            const float len = __fsqrt_rn(f_add(f_add(f_mul(m[0], m[0]), f_mul(m[1], m[1])), f_mul(m[2], m[2])));
#pragma unroll
            for (int c = 0; c < 3; ++c) normals[id * 3 + c] = len == 0.0f ? (c == 2 ? 1.0f : 0.0f) : -f_div(m[c], len);
            ++id;
        }
    }
}

__global__ void __launch_bounds__(kThreads) mc_emit_faces_kernel(Lattice L, int64_t nodes, Workspace w,
                                                                 const int32_t* __restrict__ vbase,
                                                                 int32_t* __restrict__ faces) {
    const int64_t tile = blockIdx.x;
    long long running = tile_base_f(w, tile);
    const int64_t nn = (int64_t)L.n * L.n;
    for (int k = 0; k < kRounds; ++k) {
        const int64_t i = tile * kTile + k * kThreads + threadIdx.x;
        NodeInfo r;
        r.cube = -1;
        if (i < nodes) r = node_info(L, i);
        const int nt = tri_count(r);
        long long f = nt, unused = 0, total, unused_t;
        block_exclusive_scan2(f, unused, &total, &unused_t);
        f += running;
        running += total;
        for (int j = 0; j < 3 * nt; ++j) {
            const int e = kMcTriEdges[r.cube][j];
            const int c = kMcEdgeCorner[e], axis = kMcEdgeAxis[e];
            const int o[3] = {r.idx[0] + (c & 1), r.idx[1] + (c >> 1 & 1), r.idx[2] + (c >> 2 & 1)};
            // rank of this edge among the owner's crossing edges: count its crossing edges along lower axes
            const bool in_o = r.cube >> c & 1;
            int rank = 0;
            for (int a = 0; a < axis; ++a) {
                bool in_n;
                if (!(c >> a & 1)) {
                    in_n = r.cube >> (c | 1 << a) & 1;      // the neighbour is a corner of this cell
                } else {
                    if (o[a] + 1 >= L.n) continue;           // no edge past the border
                    int q[3] = {o[0], o[1], o[2]};
                    q[a] += 1;
                    in_n = L.in(q[0], q[1], q[2]);
                }
                rank += in_n != in_o;
            }
            faces[f * 3 + j] = vbase[(o[0] * nn + (int64_t)o[1] * L.n) + o[2]] + rank;
        }
    }
}

int check_lattice_args(int64_t n, float threshold, const char* fn) {
    if (n < 2 || n > kMaxN) {
        ngp::set_error("%s: lattice size n must be in [2, %d]", fn, kMaxN);
        return -1;
    }
    if (!isfinite(threshold)) {
        ngp::set_error("%s: threshold must be finite", fn);
        return -1;
    }
    return 0;
}

}  // namespace

extern "C" {

int ngp_mesh_lattice_points(int64_t n, float bound, int64_t start, int64_t count, const uint8_t* density_bitfield,
                            int cascades, int grid_size, float scale, float* xyz, uint8_t* occ, void* stream) {
    NGP_REQUIRE(n >= 2 && n <= kMaxN, "lattice size n must be in [2, 1024]");
    NGP_REQUIRE(isfinite(scale) && scale > 0.0f, "scale must be finite and > 0");
    NGP_REQUIRE(isfinite(bound) && bound > 0.0f && bound <= scale, "bound must lie in (0, scale]");
    NGP_REQUIRE(cascades >= 1 && grid_size >= 1 && grid_size <= 1024, "bad occupancy-grid shape");
    NGP_REQUIRE(start >= 0 && count >= 0 && start + count <= n * n * n, "node range outside the lattice");
    if (count == 0) return 0;
    NGP_REQUIRE(density_bitfield && xyz && occ, "null pointer");
    Occupancy p{density_bitfield, cascades, grid_size, scale};
    mesh_points_kernel<<<(unsigned)((count + kPointThreads - 1) / kPointThreads), kPointThreads, 0,
                         ngp::as_stream(stream)>>>((int)n, bound, start, count, p, xyz, occ);
    NGP_LAUNCHED("mesh_points_kernel");
    return 0;
}

int ngp_mesh_lattice_store(const float* sigma, const uint8_t* occ, int64_t start, int64_t count, float* lattice,
                           void* stream) {
    NGP_REQUIRE(start >= 0 && count >= 0, "negative node range");
    if (count == 0) return 0;
    NGP_REQUIRE(sigma && occ && lattice, "null pointer");
    mesh_store_kernel<<<(unsigned)((count + kPointThreads - 1) / kPointThreads), kPointThreads, 0,
                        ngp::as_stream(stream)>>>(sigma, occ, start, count, lattice);
    NGP_LAUNCHED("mesh_store_kernel");
    return 0;
}

int64_t ngp_mc_workspace_bytes(int64_t n) {
    if (n < 2 || n > kMaxN) {
        ngp::set_error("%s: lattice size n must be in [2, %d]", __func__, kMaxN);
        return -1;
    }
    return workspace_layout(nullptr, n).bytes;
}

int ngp_mc_count(const float* lattice, int64_t n, float threshold, void* workspace, void* stream) {
    if (check_lattice_args(n, threshold, __func__)) return -1;
    NGP_REQUIRE(lattice && workspace, "null pointer");
    const Workspace w = workspace_layout(workspace, n);
    mc_count_kernel<<<(unsigned)w.tiles, kThreads, 0, ngp::as_stream(stream)>>>(Lattice{lattice, (int)n, threshold},
                                                                                 n * n * n, w.tile_counts);
    NGP_LAUNCHED("mc_count_kernel");
    return 0;
}

int ngp_mc_scan(int64_t n, void* workspace, int64_t* totals, void* stream) {
    NGP_REQUIRE(n >= 2 && n <= kMaxN, "lattice size n must be in [2, 1024]");
    NGP_REQUIRE(workspace && totals, "null pointer");
    const Workspace w = workspace_layout(workspace, n);
    cudaStream_t st = ngp::as_stream(stream);
    mc_scan_tiles_kernel<<<(unsigned)w.blocks, kScanThreads, 0, st>>>(w.tile_counts, w.tiles, w.tile_off, w.block_sum);
    NGP_LAUNCHED("mc_scan_tiles_kernel");
    mc_scan_blocks_kernel<<<1, kScanThreads, 0, st>>>(w.block_sum, w.blocks, w.block_off, totals);
    NGP_LAUNCHED("mc_scan_blocks_kernel");
    return 0;
}

int ngp_mc_emit_vertices(const float* lattice, int64_t n, float threshold, float bound, void* workspace,
                         int64_t n_vertices, int32_t* vbase, float* vertices, float* normals, void* stream) {
    if (check_lattice_args(n, threshold, __func__)) return -1;
    NGP_REQUIRE(isfinite(bound) && bound > 0.0f, "bound must be finite and > 0");
    NGP_REQUIRE(n_vertices >= 0 && n_vertices < ((int64_t)1 << 31), "vertex count must be in [0, 2^31)");
    NGP_REQUIRE(lattice && workspace && vbase, "null pointer");
    if (n_vertices == 0) return 0;
    NGP_REQUIRE(vertices && normals, "null pointer");
    const Workspace w = workspace_layout(workspace, n);
    mc_emit_vertices_kernel<<<(unsigned)w.tiles, kThreads, 0, ngp::as_stream(stream)>>>(
        Lattice{lattice, (int)n, threshold}, n * n * n, bound, w, vbase, vertices, normals);
    NGP_LAUNCHED("mc_emit_vertices_kernel");
    return 0;
}

int ngp_mc_emit_faces(const float* lattice, int64_t n, float threshold, void* workspace, const int32_t* vbase,
                      int64_t n_faces, int32_t* faces, void* stream) {
    if (check_lattice_args(n, threshold, __func__)) return -1;
    NGP_REQUIRE(n_faces >= 0 && n_faces < ((int64_t)1 << 31), "face count must be in [0, 2^31)");
    NGP_REQUIRE(lattice && workspace && vbase, "null pointer");
    if (n_faces == 0) return 0;
    NGP_REQUIRE(faces, "null pointer");
    const Workspace w = workspace_layout(workspace, n);
    mc_emit_faces_kernel<<<(unsigned)w.tiles, kThreads, 0, ngp::as_stream(stream)>>>(
        Lattice{lattice, (int)n, threshold}, n * n * n, w, vbase, faces);
    NGP_LAUNCHED("mc_emit_faces_kernel");
    return 0;
}

}  // extern "C"
