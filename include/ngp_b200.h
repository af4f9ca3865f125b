/*
 * ngp_b200.h — C-ABI of the Instant-NGP hot path for the H100 (sm_90a).
 *
 * This header is the drop-in boundary.  Every entry point replaces one Taichi
 * kernel (or one torch op sequence) of taichi-dev/taichi-nerfs; the reference
 * interface each one stands in for is cited as `file:line` (relative to the
 * reference checkout).  The reference's "FFI" is Taichi's ndarray binding:
 * caller-allocated, contiguous torch tensors passed by raw device pointer on
 * the caller's CUDA stream; kernels return nothing and write into caller
 * buffers.  We keep exactly that contract:
 *
 *   - all buffers are caller-owned device memory (plain pointers + sizes);
 *   - every call is asynchronous on the `stream` argument (a cudaStream_t
 *     passed as void*); no call synchronises the device;
 *   - return value: 0 = ok, <0 = argument error, >0 = cudaError_t;
 *     `ngp_last_error()` holds a human readable message for the calling thread;
 *   - no torch / ATen types appear in any signature.
 *
 * The CPU oracle (oracle/ngp_oracle.c, TEST INFRASTRUCTURE ONLY) exports the
 * same signatures with a `_cpu` suffix and without the stream argument.
 */
#ifndef NGP_B200_H
#define NGP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NGP_MAX_LEVELS 16

/* dtype tags for `void*` tensor arguments */
#define NGP_F32 0
#define NGP_F16 1

/*
 * Multiresolution hash-grid layout.  Mirrors what HashEncoder.__init__ derives
 * (modules/hash_encoder.py:183-208 / modules/hash_encoder_half.py:256-284) plus
 * the per-level `scale`/`resolution` that the Taichi kernel recomputes per
 * thread in f32 (modules/hash_encoder.py:73-80,103-104).  They are computed
 * once on the host (f32 semantics) and handed to both the oracle and the CUDA
 * kernels so the two can never disagree on a knife-edge `expf`.
 */
typedef struct ngp_hash_layout {
    int32_t  n_levels;               /* L (<= NGP_MAX_LEVELS)                    */
    int32_t  feat_dim;               /* F: features per level (1..8)             */
    int32_t  begin_fast_hash_level;  /* first level indexed by the xor-prime hash */
    int32_t  reserved;
    int32_t  offsets[NGP_MAX_LEVELS];     /* first entry of each level (entries)   */
    int32_t  map_sizes[NGP_MAX_LEVELS];   /* entries per level                     */
    float    scales[NGP_MAX_LEVELS];      /* base_res*exp(l*log_b) - 1     (f32)   */
    uint32_t resolutions[NGP_MAX_LEVELS]; /* ceil(scale)+1                         */
} ngp_hash_layout;

/*
 * Tri-plane layout (modules/triplane.py of the reference): three max_res x max_res planes of F features,
 * plane fd starting at fd*max_res^2*F (triplane.py:24,85), entry (u, v) of a plane at (u + v*max_res)*F.
 * `scales`/`resolutions` are the per-level fp32 scale base_res*exp(l*log_b) - 1 and ceil(scale) + 1
 * (triplane.py:27-33), derived on the host exactly like the hash levels'.
 */
#define NGP_TRIPLANE_MAX_RES 16384
typedef struct ngp_triplane_layout {
    int32_t  n_levels;               /* L, 1..NGP_MAX_LEVELS                      */
    int32_t  feat_dim;               /* F: features per level, 2 or 4             */
    int32_t  max_res;                /* plane side, 2..NGP_TRIPLANE_MAX_RES       */
    int32_t  reserved;
    float    scales[NGP_MAX_LEVELS];      /* base_res*exp(l*log_b) - 1     (f32)   */
    uint32_t resolutions[NGP_MAX_LEVELS]; /* ceil(scale)+1                         */
} ngp_triplane_layout;

/*
 * Voxel-grid layout (`--model_name svox`, the reference's VoxelGrid, modules/networks.py:382-575): a G^3 lattice of
 * nodes ((i,j,k) - ceil(G/2) + 1) * radius (networks.py:450-466), i.e. node 0 at c_min = (1 - ceil(G/2)) * radius
 * on every axis (rounded to fp32 on the host).  sh field [G,G,G,3*(deg+1)^2] and density field [G,G,G], node
 * (i,j,k) at ((i*G + j)*G + k).
 */
#define NGP_VOXEL_MAX_GRID 2048
typedef struct ngp_voxel_layout {
    int32_t grid;        /* G, 1..NGP_VOXEL_MAX_GRID                        */
    int32_t sh_degree;   /* 0, 1 or 2                                       */
    float   radius;      /* node spacing                                    */
    float   c_min;       /* world coordinate of node 0 on every axis        */
} ngp_voxel_layout;

/* Weights of the tiny NGP MLP (modules/networks.py:111-132): no biases.
 * Row-major [out, in] exactly like torch.nn.Linear.weight, fp32 master copy. */
typedef struct ngp_mlp_weights {
    const float* w1;   /* xyz_encoder.hidden_layers.0.weight  [64,32] */
    const float* w2;   /* xyz_encoder.output_layer.weight     [16,64] */
    const float* w3;   /* rgb_net.hidden_layers.0.weight      [64,32] */
    const float* w4;   /* rgb_net.hidden_layers.1.weight      [64,64] */
    const float* w5;   /* rgb_net.output_layer.weight         [ 3,64] */
} ngp_mlp_weights;

#define NGP_MLP_W1 (64 * 32)
#define NGP_MLP_W2 (16 * 64)
#define NGP_MLP_W3 (64 * 32)
#define NGP_MLP_W4 (64 * 64)
#define NGP_MLP_W5 (3 * 64)
#define NGP_MLP_PARAMS (NGP_MLP_W1 + NGP_MLP_W2 + NGP_MLP_W3 + NGP_MLP_W4 + NGP_MLP_W5) /* 9408 */

/* ---- library ------------------------------------------------------------- */
int         ngp_version(void);
const char* ngp_last_error(void);
/* number of kernel launches this library has issued in the calling process */
int64_t     ngp_launch_count(void);

/* ---- a1: ray / AABB slab test ------------------------------------------- */
/* replaces ray_aabb_intersect, modules/intersection.py:8-37 (wrapper :40-55) */
int ngp_ray_aabb_intersect(const float* rays_o, const float* rays_d, float scale,
                           float* hits_t, int64_t n_rays, void* stream);

/* ---- a2: occupancy-grid ray marching, training -------------------------- */
/* replaces raymarching_train_kernel, modules/ray_march.py:8-123.
 * Split in two launches so the host wrapper (or a fused step) can size the
 * sample buffers from `counter[0]` instead of allocating n_rays*max_samples
 * rows (modules/ray_march.py:149-168):
 *   _count : pass 1 (ray_march.py:45-74) -> rays_a[r] = (r, exclusive-scan, n),
 *            counter[0] = total samples, counter[1] = n_rays.
 *            Layout is deterministic (ray order), unlike the atomics of :76-81.
 *   _write : pass 2 (ray_march.py:86-123) -> xyzs, dirs, deltas, ts.
 *            Rays whose segment would exceed `capacity` rows write nothing and
 *            get rays_a[r,2] = 0; counter[0] is clamped accordingly. */
int ngp_raymarching_train_count(const float* rays_o, const float* rays_d, const float* hits_t,
                                const uint8_t* density_bitfield, const float* noise,
                                int cascades, int grid_size, float scale, float exp_step_factor,
                                int max_samples, int32_t* counter, int32_t* rays_a,
                                int64_t n_rays, void* stream);
int ngp_raymarching_train_write(const float* rays_o, const float* rays_d, const float* hits_t,
                                const uint8_t* density_bitfield, const float* noise,
                                int cascades, int grid_size, float scale, float exp_step_factor,
                                int32_t* counter, int32_t* rays_a,
                                float* xyzs, float* dirs, float* deltas, float* ts,
                                int64_t n_rays, int64_t capacity, void* stream);

/* Single-pass variant.  noise == NULL: test-time semantics (no jitter, `0 < t` as ray_march.py:226);
 * noise != NULL: training semantics (ray_march.py:36-43).  Every ray marches
 * once, reserves its rows with one atomicAdd on counter[0] (caller zeroes counter[0..1]) and writes
 * rays_a[r] = (r, start, n) + its samples.  Row order across rays is arbitrary (as in the reference,
 * ray_march.py:76-81); the one ray that straddles the end of the
 * `capacity` buffers keeps the samples that fit (rendered truncated), rays reserving after it own no rows; both kinds
 * are counted in counter[1], and every row below min(counter[0], capacity) is written. */
int ngp_raymarching_frame(const float* rays_o, const float* rays_d, const float* hits_t, const float* noise,
                          const uint8_t* density_bitfield, int cascades, int grid_size, float scale,
                          float exp_step_factor, int max_samples, int32_t* counter, int32_t* rays_a,
                          float* xyzs, float* dirs, float* deltas, float* ts, int64_t n_rays,
                          int64_t capacity, void* stream);

/* ---- a3: occupancy-grid ray marching, test time -------------------------- */
/* replaces raymarching_test_kernel, modules/ray_march.py:197-268.
 * hits_t[r,0] is advanced in place (ray_march.py:257). */
int ngp_raymarching_test(const float* rays_o, const float* rays_d, float* hits_t,
                         const int64_t* alive_indices, const uint8_t* density_bitfield,
                         int cascades, int grid_size, float scale, float exp_step_factor,
                         int max_samples, int64_t* ray_indices, uint8_t* valid_mask,
                         float* deltas, float* ts, int32_t* samples_counter,
                         int64_t n_alive, void* stream);

/* ---- a4/a5: multiresolution hash-grid encoding --------------------------- */
/* forward: replaces hash_encoder_kernel, modules/hash_encoder.py:89-143 (fp32
 * table, fp32 out [n, L*F]) and modules/hash_encoder_half.py:112-161 (fp16 table,
 * fp16 accumulate, fp16 out [n, L, F]).  `dtype` selects NGP_F32 / NGP_F16 for
 * both `table` and `out`. */
int ngp_hash_encode_fwd(const float* xyz, const void* table, const ngp_hash_layout* layout,
                        void* out, int dtype, int64_t n, void* stream);
/* backward wrt the table: replaces hash_encoder_kernel.grad (Taichi autodiff,
 * modules/hash_encoder.py:265-277) and hash_encoder_backward_kernel
 * (modules/hash_encoder_half.py:164-213).  grad_table is fp32 [entries*F] and is
 * ACCUMULATED into (caller zeroes it, hash_encoder_half.py:350-352). */
int ngp_hash_encode_bwd(const float* xyz, const void* dout, int dout_dtype,
                        const ngp_hash_layout* layout, float* grad_table,
                        int64_t n, void* stream);
/* backward wrt the input position (the reference returns None here,
 * hash_encoder.py:277; semantics from notebooks/autodiff.ipynb cell 2):
 * dx[n,3] = d out / d xyz contracted with dout, the derivative of the forward inside the cell of xyz.
 * With an fp16 table it is taken at the fp16 forward's fraction, pos - f16(pos_grid)
 * (hash_encoder_half.py:132), which differs from pos - pos_grid for odd pos_grid above 2048.
 * feature_per_level must be 2. */
int ngp_hash_encode_bwd_input(const float* xyz, const void* table, const void* dout, int dtype,
                              const ngp_hash_layout* layout, float* dx,
                              int64_t n, void* stream);

/* ---- tri-plane encoding ---------------------------------------------------- */
/* forward: replaces triplane_encoder_kernel, modules/triplane.py:35-98.  xyz [n,3] in [0,1] ->
 * out fp32 [n, L*F], column j*L + level (feature-major, triplane.py:43-45).  The max_res-grid
 * coordinate is clamped to [0, max_res-1] (the reference's bounds check is commented out,
 * triplane.py:88-89); the clamp is the identity for positions in [0,1].
 * `aabb6` (HOST pointer, 6 floats: xyz_min[3], xyz_max-xyz_min[3]; may be NULL) folds NGP.density's
 * normalisation (modules/networks.py:144) into the load, bit-identical to normalising first.
 * `table` (and `grad_table`) must be aligned to one entry (4*F bytes). */
int ngp_triplane_encode_fwd(const float* xyz, const float* table, const ngp_triplane_layout* layout,
                            float* out, int64_t n, const float* aabb6, void* stream);
/* the same with the row count read on the device: rows [0, min(n_max, *n_dev)) (the compacting frame
 * renderer's round, see ngp_hash_encode_fwd_dyn); rows >= that count are not written. */
int ngp_triplane_encode_fwd_dyn(const float* xyz, const float* table, const ngp_triplane_layout* layout,
                                float* out, int64_t n_max, const int32_t* n_dev, const float* aabb6,
                                void* stream);
/* backward wrt the table: replaces triplane_encoder_kernel.grad (Taichi autodiff, triplane.py:186-197):
 * grad_table[entry(fd,c)] += dout * w_c[fd] * prod_{fd' != fd} lf[fd'], ACCUMULATED into the caller's fp32
 * buffer.  xyz in [0,1] (no aabb).  There is no dL/dxyz (the reference returns None, :197). */
int ngp_triplane_encode_bwd(const float* xyz, const float* table, const float* dout,
                            const ngp_triplane_layout* layout, float* grad_table, int64_t n, void* stream);
/* the same with the row count read on the device, for the graph-captured training step: rows
 * [0, min(n_max, max(*n_dev, 0))) (n_dev == NULL: n_max rows); rows at or beyond the count are never read.
 * `aabb6` as in the forward (world positions, normalised by the same arithmetic, so the geometry is the forward's bit
 * for bit).  found_inf_or_null: set to 1 when a non-finite value is handed to a reduction - GradScaler's inf check
 * raised at the source (see ngp_hash_encode_bwd_levels); a row whose dout is zero in all F columns of a level issues
 * no reduction and raises nothing.  ngp_triplane_encode_bwd is this call with n_dev = aabb6 = found_inf = NULL. */
int ngp_triplane_encode_bwd_dyn(const float* xyz, const float* table, const float* dout,
                                const ngp_triplane_layout* layout, float* grad_table, int64_t n_max,
                                const int32_t* n_dev, const float* aabb6, int32_t* found_inf_or_null, void* stream);

/* ---- voxel grid (`--model_name svox`) ---------------------------------------------------------- */
/* forward: the reference's VoxelGrid.forward / query_grids (modules/networks.py:521-575) with the semantics it leaves
 * undefined decided in DESIGN.md §6d.  xyz [n,3] world positions, dirs [n,3] (normalised in the kernel, as in
 * NGP.forward, networks.py:152-166) -> sigma [n] = ReLU(trilinear density), rgb [n,3] =
 * sigmoid(sum_k Y_k(d) * sh[c*D + k]) (real SH basis of modules/sh_utils.py:58-113, degree <= 2), all fp32.  Corners
 * outside [0, G) contribute zero (the out-of-grid mask, networks.py:489-508, :552).  rgb == NULL: density-only mode
 * (sh and dirs are not read); its sigma is bit-identical to the full forward's. */
int ngp_voxel_fwd(const float* xyz, const float* dirs, const float* sh, const float* density,
                  const ngp_voxel_layout* layout, float* sigma, float* rgb, int64_t n, void* stream);
/* the same with the row count read on the device: rows [0, min(n_max, max(*n_dev, 0))); rows beyond are not
 * written. */
int ngp_voxel_fwd_dyn(const float* xyz, const float* dirs, const float* sh, const float* density,
                      const ngp_voxel_layout* layout, float* sigma, float* rgb, int64_t n_max, const int32_t* n_dev,
                      void* stream);
/* backward wrt the fields: dsh += dL/dsh, ddensity += dL/ddensity, ACCUMULATED into the caller's fp32 buffers.
 * sigma and rgb are the forward's outputs (they give the ReLU mask sigma > 0 and the sigmoid derivative
 * rgb*(1-rgb)); dsigma [n], drgb [n,3] fp32.  No dL/dxyz, no dL/ddirs.  found_inf_or_null: set to 1 when a
 * non-finite value is handed to a reduction (GradScaler's inf check at the source).  mapping: NGP_VOXEL_BWD_WARP
 * (lanes walk one corner's channels: one coalesced scatter instruction per corner) or NGP_VOXEL_BWD_THREAD (one thread
 * per sample issues all 8 * (3D+1) reductions; kept for comparison). */
#define NGP_VOXEL_BWD_WARP 0
#define NGP_VOXEL_BWD_THREAD 1
int ngp_voxel_bwd(const float* xyz, const float* dirs, const float* sigma, const float* rgb, const float* dsigma,
                  const float* drgb, const ngp_voxel_layout* layout, float* dsh, float* ddensity, int64_t n,
                  int32_t* found_inf_or_null, int mapping, void* stream);
/* Regularisers of the voxel grid (DESIGN.md §6d) over the node block B = [lo, hi) per axis, block6 (HOST pointer) =
 * {lo_x, lo_y, lo_z, hi_x, hi_y, hi_z}, 0 <= lo < hi <= G.  For a channel of node v in B, with forward differences
 * Delta_a = V(v + e_a) - V(v) (0 when v + e_a lies outside B), s(v) = sqrt(Dx^2 + Dy^2 + Dz^2 + 1e-8):
 *   L_tv_sigma = mean over B of s (density), L_tv_sh = mean over B x the 3D sh channels of s,
 *   L_sparsity = mean over B of log(1 + 2 ReLU(density)^2).
 * dsh / ddensity += scale * (w_tv_sigma dL_tv_sigma + w_tv_sh dL_tv_sh + w_sparsity dL_sparsity), scale =
 * scale_dev[0] if scale_dev != NULL else loss_scale.  Each gradient float is computed and written by one thread (no
 * atomics): the result is bit-reproducible.  A weight of 0 skips its term (its channels are not written); all three 0:
 * no launch.  Weights must be finite and >= 0.  loss_or_null accumulates the unscaled weighted loss
 * w_tv_sigma L_tv_sigma + w_tv_sh L_tv_sh + w_sparsity L_sparsity (caller zeroes it; fp32 atomic sum). */
int ngp_voxel_reg(const float* sh, const float* density, const ngp_voxel_layout* layout, const int32_t* block6,
                  float w_tv_sigma, float w_tv_sh, float w_sparsity, float loss_scale, const float* scale_dev,
                  float* dsh, float* ddensity, float* loss_or_null, void* stream);

/* ---- sync-free ("_dyn") variants used by the graph-captured training step -------------------
 * Same kernels as above, but the number of valid rows is read ON THE DEVICE: rows [0, min(n_max,*n_dev))
 * are processed, so a step can be enqueued (or replayed as a CUDA graph) without the host read-back of
 * the sample counter that the reference performs at modules/ray_march.py:187-192.
 * `aabb6` (HOST pointer, 6 floats: xyz_min[3], xyz_max-xyz_min[3]; may be NULL) folds NGP.density's
 * normalisation x = (x - xyz_min)/(xyz_max - xyz_min) (modules/networks.py:144) into the gather. */
int ngp_hash_encode_fwd_dyn(const float* xyz, const void* table, const ngp_hash_layout* layout, void* out,
                            int dtype, int64_t n_max, const int32_t* n_dev, const float* aabb6, void* stream);
int ngp_hash_encode_bwd_dyn(const float* xyz, const void* dout, int dout_dtype, const ngp_hash_layout* layout,
                            float* grad_table, int64_t n_max, const int32_t* n_dev, const float* aabb6,
                            void* stream);
/* Same, restricted to the levels [level_begin, level_end): the levels own disjoint slices of grad_table, so a range
 * can be scattered on its own; inside the range the launch scatters one L2-sized level group at a time
 * (ngp_hash_bwd_level_groups below).  found_inf_or_null: set to 1 when a non-finite contribution is scattered -
 * GradScaler's inf check raised at the source instead of a separate pass over the gradient buffer
 * (ngp_check_finite). */
int ngp_hash_encode_bwd_levels(const float* xyz, const void* dout, int dout_dtype, const ngp_hash_layout* layout,
                               float* grad_table, int64_t n_max, const int32_t* n_dev, const float* aabb6,
                               int level_begin, int level_end, int32_t* found_inf_or_null, void* stream);
/* The level groups the F = 2 table backward above scatters one launch at a time, for an L2 of l2_bytes (the
 * backward passes the current device's when n_max >= 2^20 rows, else 0: one group): consecutive groups covering [level_begin, level_end), each one's fp32
 * gradient slice at most half of l2_bytes unless it is a single level.  Writes the group boundaries
 * bounds[0] = level_begin < ... < bounds[G] = level_end (room for NGP_MAX_LEVELS + 1) and returns G, or < 0. */
int ngp_hash_bwd_level_groups(const ngp_hash_layout* layout, int level_begin, int level_end, int64_t l2_bytes,
                              int32_t* bounds);
int ngp_mlp_fwd_dyn(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w, float* sigmas,
                    void* rgbs_f16, void* save, int64_t n_max, const int32_t* n_dev, void* stream);
int ngp_mlp_bwd_dyn(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w, const void* save,
                    const float* dsigmas, const void* drgbs_f16, void* demb, float* grad_w, int64_t n_max,
                    const int32_t* n_dev, int32_t* found_inf_or_null, void* stream);
/* Adam with the per-step scalars in device memory: hyper_dev[4] = {lr/(1-beta1^t), sqrt(1-beta2^t), inv_scale,
 * t (Adam's applied-step count, int bits)} (so the launch arguments are step-invariant and the launch can live in a
 * CUDA graph). */
int ngp_adam_step_dyn(float* param, float* grad, float* exp_avg, float* exp_avg_sq, void* param_f16_or_null,
                      const int32_t* found_inf_or_null, const float* hyper_dev, float beta1, float beta2,
                      float eps, int zero_grad, int64_t n, void* stream);
/* Advances the device-side iteration counter and writes hyper_dev for ngp_adam_step_dyn:
 * lr = cosine annealing from lr0 to lr_min over max_steps (train.py:159-163) evaluated at the 0-based iteration
 * (scheduler.step() runs every iteration, train.py:201); Adam bias corrections (train.py:143-156) for t = number of
 * APPLIED steps: t advances only when *found_inf == 0 (GradScaler.step skips optimizer.step() on inf/NaN, :199). */
int ngp_adam_hyper_update(int32_t* step_dev, float lr0, float lr_min, int32_t max_steps, float beta1,
                          float beta2, float inv_scale, const int32_t* found_inf_or_null, float* hyper_dev,
                          void* stream);
/* torch.cuda.amp.GradScaler.update() on the device (train.py:137-141,200): state_dev = {scale, growth_tracker};
 * found_inf != 0 -> scale *= backoff, tracker = 0; else tracker += 1 and, every growth_interval clean steps,
 * scale *= growth.  Also refreshes hyper_dev[2] = 1 / (scale * world_size) for the NEXT step's Adam. */
int ngp_loss_scale_update(float* state_dev, int32_t* found_inf, float growth, float backoff,
                          int32_t growth_interval, float world_size, float* hyper_dev, int clear_found_inf,
                          void* stream);
/* the scalar housekeeping the reference does with tensor ops every step, in one launch (each pointer may be
 * NULL): counter[0:2] = 0 (modules/ray_march.py:183 `counter.zero_()`), *loss_sum = 0, *found_inf = 0
 * (GradScaler's per-step found_inf tensor), *batch_counter += 1 (batches drawn by ngp_sample_ray_batch) */
int ngp_step_reset(int32_t* march_counter2, float* loss_sum, int32_t* found_inf, int32_t* batch_counter, void* stream);
/* per-ray loss head: out = rgb + bg*(1-opacity) (modules/rendering.py:219-226), loss = mean((out-gt)^2)
 * (train.py:193), and d(loss*loss_scale)/d rgb, /d opacity in one launch.  *loss_sum accumulates
 * sum((out-gt)^2) (caller zeroes it; divide by 3*n_rays). */
int ngp_mse_loss_grad(const float* rgb, const float* opacity, const float* gt, float bg, float loss_scale,
                      float* loss_sum, float* g_rgb, float* g_opacity, int64_t n_rays, void* stream);
/* same with the loss scale read from device memory (scale_dev[0]); loss_scale is ignored */
int ngp_mse_loss_grad_dyn(const float* rgb, const float* opacity, const float* gt, float bg,
                          const float* scale_dev, float* loss_sum, float* g_rgb, float* g_opacity,
                          int64_t n_rays, void* stream);

/* ---- a6: spherical-harmonics direction encoding -------------------------- */
/* replaces dir_encoder, modules/spherical_harmonics.py:7-42 */
int ngp_dir_encode(const float* dirs, float* out, int64_t n, void* stream);

/* ---- a7: fused NGP MLP (sigma net + SH + rgb net) ------------------------- */
/* replaces NGP.forward's network part, modules/networks.py:136-166 with
 * MLP.forward :369-380 under torch.autocast(fp16) (train.py:177):
 *   emb [n,32] (fp16 or fp32), dirs [n,3] fp32 (un-normalised)
 *   -> sigmas [n] fp32, rgbs [n,3] fp16, h [n,16] fp16 (geometry feature)
 * With `save` != NULL (ngp_mlp_save_bytes(n) = 40 n bytes, 16-byte aligned) the forward also stores what
 * torch.autograd would keep for the backward and is cheap to keep: h [n,16] fp16 and the fp16 sigmoid output
 * [n,4]; the backward given the same `save` then restarts from h (layers 2 and 5 are not recomputed) and
 * forms sigmoid' from the saved output exactly as torch's sigmoid_backward does.  save == NULL: the backward
 * recomputes everything from (emb, dirs). */
int64_t ngp_mlp_save_bytes(int64_t n);
int ngp_mlp_fwd(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w,
                float* sigmas, void* rgbs_f16, void* save, int64_t n, void* stream);
/* backward: dsigmas [n] fp32, drgbs [n,3] fp16 -> demb [n,32] (emb dtype) and
 * fp32 weight gradients ACCUMULATED into grad_w (NGP_MLP_PARAMS floats, order
 * w1|w2|w3|w4|w5). */
int ngp_mlp_bwd(const void* emb, int emb_dtype, const float* dirs, const ngp_mlp_weights* w,
                const void* save, const float* dsigmas, const void* drgbs_f16,
                void* demb, float* grad_w, int64_t n, void* stream);

/* ---- a8: volume-rendering compositing, training --------------------------- */
/* replaces volume_rendering_kernel, modules/volume_train.py:6-48.
 * rgbs may be fp16 (autocast) or fp32.  Outputs are indexed by ray id
 * (rays_a[n,0]).  ws is written for every sample (0 after early termination —
 * the reference leaves those uninitialised, volume_train.py:91-94). */
int ngp_composite_train_fwd(const float* sigmas, const void* rgbs, int rgbs_dtype,
                            const float* deltas, const float* ts, const int32_t* rays_a,
                            float T_threshold, int32_t* total_samples, float* opacity,
                            float* depth, float* rgb, float* ws,
                            int64_t n_rays, int64_t n_samples, void* stream);
/* replaces volume_rendering_kernel.grad (Taichi autodiff), volume_train.py:131-175 */
int ngp_composite_train_bwd(const float* dL_dopacity, const float* dL_ddepth,
                            const float* dL_drgb, const float* dL_dws,
                            const float* sigmas, const void* rgbs, int rgbs_dtype,
                            const float* deltas, const float* ts, const int32_t* rays_a,
                            const float* opacity, const float* depth, const float* rgb,
                            float T_threshold, float* dL_dsigmas, void* dL_drgbs,
                            int64_t n_rays, int64_t n_samples, void* stream);

/* ---- a9: incremental compositing, test time ------------------------------- */
/* replaces composite_test, modules/volume_render_test.py:4-54 (in place) */
int ngp_composite_test(const float* sigmas, const void* rgbs, int rgbs_dtype,
                       const float* deltas, const float* ts, const int64_t* pack_info,
                       int64_t* alive_indices, float T_threshold,
                       float* opacity, float* depth, float* rgb,
                       int64_t n_alive, void* stream);

/* Fused per-ray head used by the graph-captured step: composite forward (volume_train.py:6-48) + background +
 * MSE (rendering.py:219-226, train.py:193) + composite backward in ONE launch.  gt is indexed by ray id;
 * loss scale = scale_dev[0] if scale_dev != NULL else loss_scale; *loss_sum accumulates sum((out-gt)^2);
 * opacity_out / rgb_out may be NULL. */
int ngp_ray_head_fused(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas,
                       const int32_t* rays_a, const float* gt, float bg, float loss_scale,
                       const float* scale_dev, float T_threshold, float* loss_sum, float* opacity_out,
                       float* rgb_out, float* dL_dsigmas, void* dL_drgbs, int64_t n_rays, void* stream);
/* The same head with the distortion loss (modules/distortion.py, train.py:194-195) in the same launch: the loss is
 * mse + distortion_w * mean(loss_ray), loss_ray as in ngp_distortion_fwd over the composited weights.  Its dL/dw
 * (ngp_distortion_bwd with dL_dloss = distortion_w / n_rays, times the loss scale) enters the composite backward as
 * dL_dws does in ngp_composite_train_bwd.  *loss_sum accumulates sum((out-gt)^2) + 3 distortion_w sum(loss_ray), so
 * that loss_sum / (3 n_rays) is the total loss.  ts are the sample midpoints; distortion_w >= 0 (0 adds nothing). */
int ngp_ray_head_fused_distortion(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas,
                                  const float* ts, const int32_t* rays_a, const float* gt, float bg,
                                  float loss_scale, const float* scale_dev, float T_threshold,
                                  float distortion_w, float* loss_sum, float* opacity_out, float* rgb_out,
                                  float* dL_dsigmas, void* dL_drgbs, int64_t n_rays, void* stream);

/* ---- distortion loss (SURVEY §8f rank 3) -------------------------------------- */
/* replaces prefix_sums_kernel + _loss_kernel + distortion_loss_fw_kernel
 * (modules/distortion.py:15-84): loss[ray] = sum_s 2*(wts_inc*ws_exc - ws_inc*wts_exc) + w^2*delta/3
 * with per-ray inclusive/exclusive scans of w and w*t. */
int ngp_distortion_fwd(const float* ws, const float* deltas, const float* ts, const int32_t* rays_a,
                       float* loss, int64_t n_rays, int64_t n_samples, void* stream);
/* replaces distortion_loss_bw_kernel (modules/distortion.py:86-119) */
int ngp_distortion_bwd(const float* dL_dloss, const float* ws, const float* deltas, const float* ts,
                       const int32_t* rays_a, float* dL_dws, int64_t n_rays, int64_t n_samples,
                       void* stream);

/* ---- compacting test-time renderer (north_star: persistent warps + live-ray compaction) -----------------------
 * Replaces the host-driven loop of modules/rendering.py:96-144 (raymarching_test + boolean-mask compaction with host
 * syncs + composite_test per iteration; the reference's device-side re-ordering: deployment/InstantNGP/taichi_ngp/
 * kernels.py:225-260).  One frame = ngp_frame_begin, then per ROUND: ngp_frame_round_begin -> ngp_raymarching_round ->
 * ngp_hash_encode_fwd_dyn / ngp_mlp_fwd_dyn with n_dev = state -> ngp_composite_round.  `state` (int32[8], device):
 * [0] sample rows of the current round, [2] live rays of the current round, [3] live rays of the next round,
 * [4] samples evaluated so far.  `alive` / `next_alive` ping-pong between rounds.  No host read is needed until the
 * frame is complete (state[3] == 0). */
int ngp_frame_begin(const float* hits_t, float* t_cur, int32_t* n_marched, int32_t* alive, int32_t* state,
                    float* opacity, float* depth, float* rgb, int64_t n_rays, void* stream);
int ngp_frame_round_begin(int32_t* state, void* stream);
/* One round of marching (modules/ray_march.py:197-268 semantics: resume at t_cur[ray], strict 0 < t, no jitter):
 * persistent warps walk alive[0 .. state[2]); every live ray emits at most min(limit, capacity / state[2]) samples
 * (so the rows always fit), reserves them with one atomicAdd on state[0], writes rays_a[slot] = (ray, start, n) and
 * leaves its resume point in t_cur[ray] (+inf once it has left the box).  The cap over the frame: a live ray emits at
 * most max_samples - n_marched[ray] samples, adds what it emitted to n_marched[ray] (zeroed by ngp_frame_begin; must
 * not be NULL) and gets t_cur[ray] = +inf once it has max_samples, so that no ray gets more samples over the frame
 * than the one-shot march gives it. */
int ngp_raymarching_round(const float* rays_o, const float* rays_d, const float* hits_t,
                          const uint8_t* density_bitfield, int cascades, int grid_size, float scale,
                          float exp_step_factor, int limit, int max_samples, const int32_t* alive, int32_t* state,
                          float* t_cur, int32_t* n_marched, int32_t* rays_a, float* xyzs, float* dirs, float* deltas,
                          float* ts, int64_t n_rays, int64_t capacity, void* stream);
/* composite_test (modules/volume_render_test.py:4-54) for the round's samples, accumulating into opacity/depth/rgb
 * [n_rays], + block-level compaction of the rays that stay alive (T > T_threshold and still inside the box) into
 * next_alive[0 .. state[3]).  `limit` = the round's sample budget per ray (picks how many lanes share a ray). */
int ngp_composite_round(const float* sigmas, const void* rgbs, int rgbs_dtype, const float* deltas, const float* ts,
                        const int32_t* rays_a, int32_t* state, const float* t_cur, const float* hits_t,
                        float T_threshold, float* opacity, float* depth, float* rgb, int32_t* next_alive,
                        int64_t n_rays, int limit, void* stream);

/* ---- occupancy-grid helpers (SURVEY §8f rank 1) ---------------------------- */
/* replaces packbits, modules/utils.py:157-169 */
int ngp_packbits(const float* density_grid, float density_threshold,
                 uint8_t* density_bitfield, int64_t n_bytes, void* stream);
/* same, with the threshold min(*mean_density_dev, density_threshold) taken from device memory so
 * that NGP.update_density_grid (modules/networks.py:286-290) needs no `.item()` host sync */
int ngp_packbits_dev(const float* density_grid, const float* mean_density_dev, float density_threshold,
                     uint8_t* density_bitfield, int64_t n_bytes, void* stream);
/* replaces morton3D_kernel / morton3D_invert_kernel, modules/utils.py:120-154 */
int ngp_morton3d(const int32_t* coords, int32_t* indices, int64_t n, void* stream);
int ngp_morton3d_invert(const int32_t* indices, int32_t* coords, int64_t n, void* stream);

/* ---- fused occupancy-grid update (SURVEY §8f rank 1) ------------------------------------------------------
 * Stage 1 replaces NGP.get_all_cells / sample_uniform_and_occupied_cells (modules/networks.py:168-209: torch.randint,
 * torch.nonzero + len() host sync, morton3D[_invert] + ti.sync()) and the jittered positions of
 * update_density_grid (:263-271).  mode 0 (warm-up): every cell of every cascade once, slot i = Morton index i
 * (per cascade grid_size^3 slots).  mode 1: per cascade M uniformly drawn cells followed by M cells drawn uniformly
 * among those with density_grid > density_threshold (2M slots; cell_idx = -1 when no cell qualifies).  Randomness:
 * Philox4x32-10 keyed by `seed`, counter (slot, cascade, step, stream id) - identical on every rank for equal
 * (seed, step).  Outputs: cell_idx [cascades * slots] (Morton index inside the cascade), xyz [cascades * slots, 3]
 * world positions.  `workspace`: ngp_grid_workspace_bytes() bytes of caller-owned scratch, 16-byte aligned. */
int64_t ngp_grid_workspace_bytes(int cascades, int grid_size);
int ngp_grid_sample_cells(const float* density_grid, int cascades, int grid_size, float scale,
                          float density_threshold, int mode, int64_t M, uint64_t seed, uint32_t step,
                          void* workspace, int32_t* cell_idx, float* xyz, void* stream);
/* Stage 2 (after the caller evaluated `densities` at xyz with the hash + sigma-net kernels) replaces :272-290:
 * tmp[c, idx] = density (maximum over duplicate picks), density_grid = grid < 0 ? grid : max(grid * decay, tmp)
 * (count_grid != NULL: erode, decay_i = clamp(decay^(1/count_i), 0.1, 0.95)), *mean_out = mean of the positive cells
 * (deterministic two-level reduction, no .item()), density_bitfield = packbits(grid > min(mean, density_threshold)). */
int ngp_grid_update(float* density_grid, const int32_t* cell_idx, const float* densities, int64_t slots_per_cascade,
                    int cascades, int grid_size, const float* count_grid_or_null, float decay,
                    float density_threshold, void* workspace, float* mean_out, uint8_t* density_bitfield,
                    void* stream);

/* ---- training ray batch sampling (SURVEY §8f rank 2) ------------------------ */
/* replaces, per step: BaseDataset.__getitem__ (datasets/base.py:34-61: torch.randint x2 + gathers of
 * self.rays / self.poses / self.directions), get_rays (datasets/ray_utils.py:51-80:
 * rays_d = directions @ c2w[:, :3].T, rays_o = c2w[:, 3]) and the per-ray marching jitter
 * torch.rand_like (modules/ray_march.py:166), in one launch.
 *   image_bank [n_img, n_pix, channels] f32 (channels >= 3; may be NULL when rgb == NULL)
 *   poses [n_img, 3, 4] f32, directions [n_pix, 3] f32 (get_ray_directions, ray_utils.py:8-48)
 *   img_idxs / pix_idxs [n_rays] int64: the reference's sample['img_idxs'/'pix_idxs']; when NULL the
 *     index is drawn from Philox4x32-10 with counter (ray, ray>>32, step, 0) and key = seed:
 *     img = (r0 * n_img) >> 32 (or fixed_img when >= 0: ray_sampling_strategy 'same_image'),
 *     pix = (r1 * n_pix) >> 32, noise = (r2 >> 8) * 2^-24
 *   step: *step_dev when step_dev != NULL (CUDA-graph replayable), else step_host
 *   outputs rays_o / rays_d / rgb [n_rays, 3] f32, noise [n_rays] f32 (NULL = skip),
 *   img_out / pix_out [n_rays] int64 (NULL = skip) */
int ngp_sample_ray_batch(const float* image_bank, int channels, const float* poses, const float* directions,
                         int64_t n_img, int64_t n_pix, const int64_t* img_idxs, const int64_t* pix_idxs,
                         int64_t fixed_img, uint64_t seed, const int32_t* step_dev, int32_t step_host,
                         float* rays_o, float* rays_d, float* rgb, float* noise, int64_t* img_out,
                         int64_t* pix_out, int64_t n_rays, void* stream);

/* ---- a12: fused optimizer pass ---------------------------------------------- */
/* replaces GradScaler.unscale_ + inf check + torch.optim.Adam(eps=1e-15) step
 * (train.py:137-156,197-201) in ONE pass over the parameters:
 *   g = grad * inv_scale;  skip everything if *found_inf != 0;
 *   m,v update; p -= lr * mhat / (sqrt(vhat) + eps);
 *   optionally refresh the fp16 shadow copy (hash_encoder_half.py:367) and
 *   zero the gradient (optimizer.zero_grad, train.py:197).
 * `step` is the 1-based Adam step count used for bias correction. */
int ngp_adam_step(float* param, float* grad, float* exp_avg, float* exp_avg_sq,
                  void* param_f16_or_null, const int32_t* found_inf_or_null,
                  float lr, float beta1, float beta2, float eps, float inv_scale,
                  int32_t step, int zero_grad, int64_t n, void* stream);
/* sets *found_inf = 1 if any element of grad is non-finite (GradScaler check) */
int ngp_check_finite(const float* grad, int64_t n, int32_t* found_inf, void* stream);
/* Multi-GPU gradient transport in fp16 (what the reference's autocast backward produces for its parameters; the
 * loss scale keeps the values in range and a value that does not fit becomes inf, i.e. a skipped step + scale backoff
 * exactly as with GradScaler): pack the fp32 accumulation buffer, all-reduce the fp16 buffer (half the bytes), check
 * the REDUCED buffer (identical on every rank) and let Adam read it directly while zeroing the fp32 buffer. */
int ngp_grad_pack_f16(const float* grad, void* out_f16, int64_t n, void* stream);
int ngp_check_finite_f16(const void* grad_f16, int64_t n, int32_t* found_inf, void* stream);
int ngp_adam_step_dyn_g16(float* param, const void* grad_f16, float* grad_f32_to_zero_or_null, float* exp_avg,
                          float* exp_avg_sq, void* param_f16_or_null, const int32_t* found_inf_or_null,
                          const float* hyper_dev, float beta1, float beta2, float eps, int64_t n, void* stream);

/* ---- multi-GPU: gradient exchange fused into the optimizer over NVLink peer memory (csrc/p2p.cu) ----------
 * What the reference would get from DDP around train.py:197-201 (an NCCL all-reduce of every gradient, then
 * GradScaler.step / Adam on every rank) as ONE kernel per rank: rank r sums slice r of every rank's gradient buffer
 * with peer loads (reduce-scatter), runs Adam on that slice only, and stores the updated fp16 table slice into every
 * rank's shadow table with peer stores (all-gather); the replicated MLP weights are updated by every rank from the
 * same peer sums.  The buffers peers touch are allocated here and exported through CUDA IPC; the caller exchanges
 * the opaque handles (e.g. torch.distributed.all_gather_object) and opens its peers' buffers. */
#define NGP_MAX_PEERS 8
#define NGP_IPC_HANDLE_BYTES 64
int ngp_p2p_alloc(int64_t bytes, void** dev_ptr, uint8_t* handle64);   /* zero-filled, 256-byte aligned */
int ngp_p2p_open(const uint8_t* handle64, void** peer_ptr);            /* a peer's buffer in this process */
int ngp_p2p_close(void* peer_ptr);
int ngp_p2p_free(void* dev_ptr);
int64_t ngp_p2p_flag_bytes(void);                                       /* size of one rank's flag block */
/* Barrier across the ranks of one box, enqueued on `stream` (graph-capturable): flag_blocks[p] = rank p's flag block
 * (ngp_p2p_flag_bytes() zero-initialised bytes inside an IPC buffer), *epoch_dev = this rank's barrier count (device
 * memory, starts at 0, incremented by the kernel).  If found_inf != NULL it is this rank's GradScaler inf flag on entry
 * and the OR over all ranks on exit.  A rank that waits longer than ~20 s gives up and sets the sticky error word
 * (flag block word 2 * NGP_MAX_PEERS; later barriers do not wait) instead of hanging the GPU. */
int ngp_p2p_barrier(void* const* flag_blocks, int rank, int world, uint32_t* epoch_dev, int32_t* found_inf_or_null,
                    void* stream);
/* grad_peers[p] / shadow_peers[p]: rank p's flat fp32 gradient buffer / flat fp16 shadow buffer (same layout as
 * param).  Elements [own_begin, own_end) are this rank's optimizer shard (updated here, shadow broadcast to every
 * rank); [rep_begin, rep_end) are replicated parameters (updated by every rank, shadow written locally).  Nothing
 * happens when *found_inf != 0.  hyper_dev as ngp_adam_step_dyn.  The caller brackets the call with two
 * ngp_p2p_barrier and clears its gradient buffer after the second. */
int ngp_adam_step_p2p(float* param, void* const* grad_peers, float* exp_avg, float* exp_avg_sq,
                      void* const* shadow_peers, int rank, int world, const int32_t* found_inf, const float* hyper_dev,
                      float beta1, float beta2, float eps, int64_t own_begin, int64_t own_end, int64_t rep_begin,
                      int64_t rep_end, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NGP_B200_H */
