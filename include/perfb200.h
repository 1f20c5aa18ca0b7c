/*
 * perfb200.h -- C-ABI of libperfb200.so: the H100-native (sm_90a) implementation of PeRF's
 * per-ray hot path (equirect ray-gen -> fixed-S sampling -> hash-grid encode + 64-wide MLP ->
 * alpha composite, forward and backward, + fused Adam).
 *
 * Boundary rules (SURVEY.md section 8b):
 *   - extern "C", plain C types; no torch / pybind types cross this boundary.
 *   - Every pointer named d_* is a DEVICE pointer owned by the caller; h_* is a host pointer.
 *   - Every entry point enqueues work on `stream` (a cudaStream_t passed as void*) of the
 *     CURRENT device and returns without synchronising.  The library never allocates.
 *   - Return value: PERF_OK (0) or a negative PERF_E* code; perf_last_error() returns a
 *     thread-local human-readable message for the last failure.
 *   - Re-entrant across distinct streams / devices.
 *
 * Each function cites the reference interface it replaces (paths relative to the PeRF
 * repository, perf-project/PeRF @ 1431a35a).  The third-party modules the reference calls on
 * this path (tinycudann 1.7, nerfacc 0.5.3, torch_efficient_distloss 0.1.3) are not vendored;
 * the call sites are cited instead.
 */
#ifndef PERFB200_H
#define PERFB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PERF_ABI_VERSION 1

#define PERF_OK            0
#define PERF_EINVAL       -1   /* bad argument (null pointer, unsupported size, misaligned) */
#define PERF_EUNSUPPORTED -2   /* configuration outside what the kernels implement          */
#define PERF_ECUDA        -3   /* a CUDA runtime call failed (launch error, wrong arch ...)  */

#define PERF_MAX_LEVELS 16

/* encoding_config of tcnn.NetworkWithInputEncoding / tcnn.Encoding as the reference passes it
 * (modules/fields/ngp_nerf.py:99-106,119-126; modules/geo_predictors/pano_joint_predictor.py:30). */
typedef struct perf_grid_cfg {
    uint32_t n_levels;              /* <= PERF_MAX_LEVELS                       */
    uint32_t n_features_per_level;  /* must be 2                                */
    uint32_t log2_hashmap_size;
    uint32_t base_resolution;
    float    per_level_scale;
    uint32_t interpolation;         /* 0 = Linear, 1 = Smoothstep               */
} perf_grid_cfg;

typedef struct perf_level {
    float    scale;        /* exp2f(l*log2f(s))*base - 1                       */
    uint32_t resolution;   /* ceilf(scale) + 1                                 */
    uint32_t size;         /* entries in the level                             */
    uint32_t offset;       /* first entry of the level in the flat table       */
    uint32_t hashed;       /* 1: xor-prime hash, 0: dense x-fastest indexing   */
} perf_level;

/* network_config of tcnn FullyFusedMLP (ngp_nerf.py:107-113,127-133): bias-free, ReLU hidden. */
typedef struct perf_mlp_cfg {
    uint32_t n_in;               /* must be 32 (= 16 levels x 2 features)       */
    uint32_t n_out;              /* 1..16; last matrix is stored padded to 16 rows */
    uint32_t n_neurons;          /* must be 64                                  */
    uint32_t n_hidden_layers;    /* 1 or 2                                      */
    uint32_t output_activation;  /* 0 = None, 1 = Sigmoid                       */
} perf_mlp_cfg;

/* flags of the render / field entry points */
#define PERF_FLAG_TRAINING   1u   /* stratified jitter + training background rule        */
#define PERF_FLAG_SIMT_MLP   2u   /* debug only: MLP on CUDA cores instead of wgmma       */
#define PERF_FLAG_GENERIC_ADDR 8u  /* render: disable the specialised (4 dense + hashed pow2) addressing path */
#define PERF_FLAG_L0_SMEM 16u      /* render_pano (experimental variant): level 0 of the table staged into
                                      shared memory by one cp.async.bulk per CTA and read by its four
                                      warpgroups (the 132 KB shared-memory carveout instead of 100 KB) */
#define PERF_FLAG_SCAN_KERNEL 4u   /* render: samples-along-lanes kernel (warp-shuffle scan composite) instead of ray marching */

int         perf_abi_version(void);
const char* perf_last_error(void);
/* compute capability of the current device as major*10+minor (90 on H100), or <0 */
int         perf_device_arch(void);

/* Level/offset table of a grid config (tcnn GridEncodingTemplated ctor; SURVEY.md Appendix A).
 * h_levels: n_levels entries (may be NULL); h_n_entries: total table entries (may be NULL). */
int perf_grid_describe(const perf_grid_cfg* cfg, perf_level* h_levels, uint64_t* h_n_entries);
/* Length of the flat `params` vector of a network (MLP matrices, then the grid). */
int perf_network_param_count(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, uint64_t* h_count);

/* fp32 master params -> fp16 shadow, n elements (replaces the per-forward `params.to(half)` of
 * the tcnn torch binding; ngp_nerf.py:142,158 call sites). */
int perf_params_to_half(const float* d_params, void* d_params_half, uint64_t n, void* stream);

/* Interleave the two fp16 grid tables into one {geo.f0,geo.f1,app.f0,app.f1} table so one
 * 8-byte gather serves both fields.  d_*_params_half: full fp16 params of each network.
 * Layout of d_packed (8-byte entries, 16-byte aligned buffer): entries [0, n_entries) in parameter order,
 * followed by a cell-major copy of the leading dense levels (up to four; for each, res^3 cells x the 8 corner
 * entries of the cell = one 64-byte record per cell) which the fused field kernels read with four 16-byte
 * loads per sample and level.  perf_packed_table_entries gives the total entry count to allocate. */
int perf_packed_table_entries(const perf_grid_cfg* cfg, uint64_t* h_entries);
int perf_pack_tables(const perf_grid_cfg* grid, const perf_mlp_cfg* geo_mlp, const perf_mlp_cfg* app_mlp,
                     const void* d_geo_params_half, const void* d_app_params_half,
                     void* d_packed /* perf_packed_table_entries() * 8 bytes */, void* stream);

/* Equirect rays for image rows [row0,row0+rows) of an H x W panorama; h_pose: row-major 4x4
 * camera-to-world.  d_rays_o/d_rays_d: [rows*W,3] fp32.
 * Replaces utils/camera_utils.py:229-234 gen_pano_rays (+ :113-155). */
int perf_raygen_pano(const float* h_pose, int H, int W, int row0, int rows,
                     float* d_rays_o, float* d_rays_d, void* stream);

/* Perspective (OpenCV-style) rays of an H x W camera with vertical field of view `fovy` (radians).
 * Replaces utils/camera_utils.py:237-241 gen_pers_rays (+ :60-80 cam_rays_cam_space), the
 * cam_type != 'pano' branch of render_dense (core_exp_runner.py:234-235). */
int perf_raygen_pers(const float* h_pose, float fovy, int H, int W, float* d_rays_o, float* d_rays_d, void* stream);

/* Hash-grid encode forward: d_x01 [N,3] fp32 in [0,1] -> d_feat [N, L*2] fp16.
 * d_table: fp16 [n_entries,2].  Replaces tcnn kernel_grid (Encoding.forward). */
int perf_hashgrid_fwd(const perf_grid_cfg* cfg, const void* d_table, const float* d_x01,
                      uint64_t N, void* d_feat, void* stream);
/* Hash-grid backward w.r.t. the table: d_dtable [n_entries,2] fp32 += scatter(w * dfeat)
 * (caller zeroes it).  d_dfeat [N, L*2] fp32.  Replaces tcnn kernel_grid_backward. */
int perf_hashgrid_bwd(const perf_grid_cfg* cfg, const float* d_x01, const float* d_dfeat,
                      uint64_t N, float* d_dtable, void* stream);

/* Hash-grid backward w.r.t. the INPUT positions: d_dx [N,3] fp32 = sum_f dfeat_f * d feat_f / d x01
 * (Linear and Smoothstep).  d_table_half: fp16 [n_entries,2]; d_dfeat [N, L*2] fp32.
 * Replaces tcnn kernel_grid_backward_input, reached by tcnn.Encoding when its input requires grad
 * (modules/geo_predictors/pano_joint_predictor.py:30-41,48-52; pano_geo_refiner.py:19). */
int perf_hashgrid_bwd_input(const perf_grid_cfg* cfg, const void* d_table_half, const float* d_x01,
                            const float* d_dfeat, uint64_t N, float* d_dx, void* stream);
/* Double backward of perf_hashgrid_bwd_input: with d_ddx [N,3] = d(loss)/d(d_dx), writes the gradient
 * w.r.t. dfeat (d_ddfeat [N, L*2] fp32, overwritten), accumulates the gradient w.r.t. the table
 * (d_dtable [n_entries,2] fp32 +=, caller zeroes) and w.r.t. x01 (d_dx2 [N,3] fp32 +=, caller zeroes).
 * Any of the three outputs may be NULL.  Replaces tcnn kernel_grid_backward_input_backward_dLdoutput /
 * _backward_grid / _backward_input, i.e. what torch.autograd.grad(distance, directions,
 * create_graph=True) followed by loss.backward() runs (pano_joint_predictor.py:58-64). */
int perf_hashgrid_bwd_bwd_input(const perf_grid_cfg* cfg, const void* d_table_half, const float* d_x01,
                                const float* d_dfeat, const float* d_ddx, uint64_t N,
                                float* d_ddfeat, float* d_dtable, float* d_dx2, void* stream);

/* MLP backward from the saved fp16 activations, one wgmma kernel (tcnn FullyFusedMLP backward for the two
 * PeRF networks, ngp_nerf.py:107-113,127-133).  d_feat [N,32], d_h1 [N,64], d_h2 [N,64] (two hidden layers,
 * else NULL): fp16 saves of perf_network_fwd / perf_train_forward; d_dz [N,n_out] fp32 = gradient w.r.t. the
 * output pre-activation (n_out <= 3).  d_dweights: fp32 gradient of the flat MLP params, ACCUMULATED (caller
 * zeroes); d_dfeat [N,32] fp32 overwritten.  flags: PERF_FLAG_SIMT_MLP selects the CUDA-core twin.
 * The training steps call it (no library GEMM is left on that path). */
int perf_mlp_bwd(const perf_mlp_cfg* mlp, const void* d_weights_half, const void* d_feat, const void* d_h1, const void* d_h2,
                 const float* d_dz, uint64_t N, const int64_t* d_n_dev /* nullable: live row count in device memory, <= N */,
                 float* d_dweights, float* d_dfeat, uint32_t flags, void* stream);

/* Network forward = encode + MLP fused (tcnn NetworkWithInputEncoding.forward;
 * ngp_nerf.py:142,158).  d_x01 [N,3] fp32; d_params_half: fp16 flat params (MLP | grid);
 * d_out [N, n_out] fp16.  Optional saves for the backward pass (NULL to skip):
 * d_feat [N,32] fp16, d_h1 [N,64] fp16, d_h2 [N,64] fp16 (2-hidden-layer nets only). */
int perf_network_fwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* d_params_half,
                     const float* d_x01, uint64_t N, void* d_out,
                     void* d_feat, void* d_h1, void* d_h2, uint32_t flags, void* stream);

/* MLP forward alone on the tensor cores: d_in [N,32] fp16 -> d_out [N,n_out] fp16
 * (tcnn kernel_mlp_fused).  d_weights_half: the MLP part of the fp16 flat params. */
int perf_mlp_fwd(const perf_mlp_cfg* mlp, const void* d_weights_half, const void* d_in,
                 uint64_t N, void* d_out, void* d_h1, void* d_h2, uint32_t flags, void* stream);

/* Packed transmittance scan (nerfacc render_weight_from_density; nerf_renderer.py:170-171).
 * Samples sorted by ray; d_ray_indices int64 [N].  Outputs fp32 [N] (any may be NULL). */
int perf_weights_from_density(const float* d_t_starts, const float* d_t_ends, const float* d_sigmas,
                              const int64_t* d_ray_indices, uint64_t N, uint64_t n_rays,
                              float* d_weights, float* d_trans, float* d_alphas, void* stream);
/* Backward of the above w.r.t. sigmas given dL/dweights (and optional dL/dtrans). */
int perf_weights_from_density_bwd(const float* d_t_starts, const float* d_t_ends, const float* d_sigmas,
                                  const int64_t* d_ray_indices, uint64_t N, uint64_t n_rays,
                                  const float* d_weights, const float* d_trans,
                                  const float* d_grad_weights, const float* d_grad_trans /*nullable*/,
                                  float* d_grad_sigmas, void* stream);
/* out[r, :] = sum_{i in ray r} w_i * v_i[:]  (nerfacc accumulate_along_rays;
 * nerf_renderer.py:173,175,183).  d_values [N,D] fp32 or NULL (D=1, v=1).  d_out [n_rays,D]
 * is overwritten.  Deterministic (no atomics). */
int perf_accumulate_along_rays(const float* d_weights, const float* d_values, int D,
                               const int64_t* d_ray_indices, uint64_t N, uint64_t n_rays,
                               float* d_out, void* stream);

/* Arguments of the fused renderer (NeRFOCCRenderer.render, nerf_renderer.py:112-209, with the
 * fixed-S sampler; NeRFScene.render, nerf.py:74-99). */
typedef struct perf_render_args {
    perf_grid_cfg grid;           /* both fields use the same grid config (ngp_nerf.py:96-134) */
    const void*   d_packed_table; /* from perf_pack_tables (perf_packed_table_entries() * 8 bytes) */
    const void*   d_geo_mlp_half; /* fp16 MLP matrices of the density net (3072 values)         */
    const void*   d_app_mlp_half; /* fp16 MLP matrices of the colour net  (7168 values)         */
    float         aabb[6];        /* min xyz, max xyz (nerf.py:35)                              */
    uint32_t      n_samples;      /* S                                                          */
    float         near, far;      /* nerf.py:317-318: 1e-2, 1.0                                 */
    uint32_t      flags;          /* PERF_FLAG_*                                                */
    const float*  d_jitter;       /* [R] U[0,1) per-ray offset (training) or NULL               */
    const float*  d_bg_noise;     /* [R,4] training background rgb + distance noise or NULL     */
    float*        d_rgb;          /* [R,3]                                                      */
    float*        d_distance;     /* [R]                                                        */
    float*        d_opacity;      /* [R] or NULL                                                */
    uint32_t      image_width;    /* perf_render_rays only: >0 = the R rays are a row-major image of this
                                     width (locality hint: threads are tiled as 16x8 pixel patches); 0 = no structure */
} perf_render_args;

/* Render explicit rays: d_rays_o / d_rays_d [R,3] fp32. */
int perf_render_rays(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d,
                     uint64_t R, void* stream);
/* Render rays whose samples are given as packed intervals sorted by ray (the output of an occupancy
 * estimator, nerf_renderer.py:145-155): ray r owns samples [d_offsets[r], d_offsets[r+1]) of
 * d_t_starts / d_t_ends.  args->n_samples / near / far are ignored; eval-mode background rule. */
int perf_render_packed(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R,
                       const int64_t* d_offsets, const float* d_t_starts, const float* d_t_ends, void* stream);
/* Render rows [row0,row0+rows) of an H x W equirect panorama with ray generation fused in
 * (core_exp_runner.py:229-238 render_dense inner loop).  Outputs are [rows*W, .]. */
int perf_render_pano(const perf_render_args* args, const float* h_pose, int H, int W,
                     int row0, int rows, void* stream);

/* ---- surface normals: the three renders above (and perf_fields_packed) with a fourth output.
 * Definition, per sample at normalised position x01 (the renderer's own position, selector and fp16 features):
 *   h = W1 f (the density net's layer-1 pre-activation, fp32), m_j = [h_j > 0],
 *   g = W1^T (m . w_out) (fp16 weights as fp32; the forward's fp16 roundings count as identity),
 *   d raw / d x01_d = sum_levels sum_features g * scale * A_d (Linear interpolation; perf_hashgrid_bwd_input's arithmetic
 *   on the fp16 geo entries), raw = the density logit BEFORE trunc_exp (same direction: sigma = exp(raw)),
 *   grad_d = (d raw / d x01_d) / (aabb max_d - min_d),  n = -grad / |grad|;  n = 0 when the selector is false or |grad| = 0.
 * Per ray: d_normal [R,3] fp32 = sum_i w_i n_i with the weights that produce distance / opacity -- no background term, no
 * normalisation (|normal| <= opacity; normalise for display).  rgb / distance / opacity are the plain entry points' outputs.
 * Eval mode on the ray-marching wgmma kernel only: PERF_FLAG_SIMT_MLP, PERF_FLAG_SCAN_KERNEL, PERF_FLAG_L0_SMEM and
 * PERF_FLAG_TRAINING return PERF_EUNSUPPORTED. */
int perf_render_pano_normals(const perf_render_args* args, const float* h_pose, int H, int W, int row0, int rows,
                             float* d_normal, void* stream);
/* Explicit rays (args->image_width > 0: a row-major image, pixel-patch tiling as perf_render_rays). */
int perf_render_rays_normals(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, uint64_t R,
                             float* d_normal, void* stream);
/* perf_fields_packed, phase 0 (no saves), plus the sample normal n (definition above) d_normal [N,3] of every packed sample.
 * The occupancy render's ray normal is then perf_composite_packed_fwd (d_weights, with its early_stop_eps cut) followed by
 * perf_accumulate_along_rays(d_weights, d_normal, D = 3). */
int perf_fields_packed_normals(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, const int64_t* d_ray_indices,
                               const float* d_t_starts, const float* d_t_ends, uint64_t N, const int64_t* d_n_dev /* nullable */,
                               float* d_sigma, void* d_rgb_half4, float* d_x01, float* d_normal, void* stream);

/* ---- both fields off the rays: on a lattice and at arbitrary points (eval mode, the kernel body of perf_fields_packed
 * phase 0; the flags of the normals entry points above return PERF_EUNSUPPORTED).  args: grid / tables / weights / aabb.
 * Replaces NGPNeRF.query_density / query_rgb on torch-built positions (ngp_nerf.py:136-162) for mesh extraction. */
/* sigma [nx, ry, rz] fp32 at lattice nodes (i, j, k), i in [x0, x0 + nx), of the rx x ry x rz lattice spanning the box, faces
 * included: x01_d = i_d / (r_d - 1) (one fp32 division, no world round trip), selector 0 < x01 < 1 strict -- face nodes are
 * exactly 0.  d_sigma[((i - x0) * ry + j) * rz + k] (x slowest, the occupancy grid's layout).  r_d >= 2 and rx ry rz < 2^31,
 * else PERF_EINVAL. */
int perf_fields_lattice(const perf_render_args* args, const int* h_res3, int x0, int nx, float* d_sigma, void* stream);
/* d_x [N,3] world points: x01 = (x - aabb_min) / ext as perf_fields_packed normalises, the renderer's selector.
 * d_sigma [N], d_rgb_half4 [N,4] fp16 (4th lane unused), d_normal [N,3] (nullable) = the sample normal defined above. */
int perf_fields_points(const perf_render_args* args, const float* d_x, uint64_t N, float* d_sigma, void* d_rgb_half4,
                       float* d_normal /* nullable */, void* stream);

/* ---- surface extraction: marching tetrahedra on the Freudenthal decomposition of a density lattice d_sigma [rx, ry, rz] fp32
 * (x slowest; any grid of that layout, e.g. perf_fields_lattice's or the occupancy grid).  Node (i,j,k) is inside iff
 * sigma > threshold.  Each cube splits into the 6 tets 000, e_a, e_a + e_b, 111 (one per axis permutation (a, b, c), in the order
 * xyz xzy yxz yzx zxy zyx); each node owns the 7 positive edges e = +x +y +z +xy +xz +yz +xyz (0..6), and an edge crosses when
 * it lies in the lattice and exactly one end is inside.
 * perf_mesh_count: d_vcount [n] uint8 = crossing edges of the node (<= 7), d_fcount [n] uint8 = triangles of the cube whose
 * minimum corner is the node (<= 12; 0 on the far faces).  The caller builds exclusive int32 scans d_voff / d_foff of both
 * (totals V, F < 2^31) and allocates d_vertices [V,3] fp32 (world), d_faces [F,3] int32.
 * perf_mesh_write: vertex of edge (p, e) = d_voff[p] + popc(mask(p) & ((1 << e) - 1)); with b the edge's other end,
 *   t = (threshold - sigma_p) / (sigma_b - sigma_p), x01_d = i_d / (r_d - 1) (+ t * ((i_d + 1) / (r_d - 1) - x01_d) along
 *   the edge's axes), world_d = aabb_min_d + x01_d * (aabb_max_d - aabb_min_d), each step one rounded fp32 operation;
 * the cube's triangles from d_foff[p] on, tet by tet; each is oriented so that its normal (v1 - v0) x (v2 - v0) points from the
 * inside to the outside (along -grad sigma of the tet's linear interpolant: the rendered normal's sense); a quad case splits
 * along the diagonal between its edges (a,c) and (b,d) (inside a < b).  The output order is fixed by the scans: repeated runs
 * are byte-identical.  r_d >= 2 and rx ry rz < 2^31, else PERF_EINVAL. */
int perf_mesh_count(const float* d_sigma, const int* h_res3, float threshold, uint8_t* d_vcount, uint8_t* d_fcount, void* stream);
int perf_mesh_write(const float* d_sigma, const int* h_res3, float threshold, const float* h_aabb6, const int32_t* d_voff,
                    const int32_t* d_foff, float* d_vertices, int32_t* d_faces, void* stream);

/* ---- mesh decimation: quadric-error (Garland-Heckbert) edge collapse in rounds of independent collapses, down to a target
 * face count (ops.decimate drives the rounds; csrc/decimate.cu).
 * Input: d_vertices [V,3] fp32, d_faces [F,3] int32, a closed, consistently oriented, edge-manifold mesh: every directed edge
 * a -> b of a face appears exactly once, and so does b -> a (perf_decimate_check).  Half-edge (edge id) i = 3f + k runs from
 * faces[f][k] to faces[f][(k+1) % 3]; each undirected edge is visited once, as its half-edge with u = a < w = b.
 * Adjacency (rebuilt by the caller every round): d_adj [3F] int32 = the corners 3f + k sorted by vertex faces[f][k], stable
 * (so ascending face index per vertex), d_adj_off [V + 1] its offsets.  N(v) = the next vertices of v's corners.
 * Quadrics (fp64, entries 00 01 02 03 11 12 13 22 23 33 of the symmetric 4x4 Q): per face n = (p1 - p0) x (p2 - p0),
 *   e = (n / |n|, -(n / |n|) . p0), Q_f = (|n| / 2) e e^T (area-weighted; 0 when n . n = 0); Q_v = sum of Q_f over v's faces in
 *   ascending face index.  A collapse of w into u sets Q_u <- Q_u + Q_w; quadrics are never recomputed.
 * Placement, Q = Q_u + Q_w = [[A, b], [b^T, c]]: with adj(A) the cofactors, det = A00 adj00 + A01 adj01 + A02 adj02 and
 *   tr = A00 + A11 + A22, the system is well conditioned iff det > 1e-6 tr^3 (scale-free; a rank-deficient A -- all faces
 *   coplanar, or a crease -- fails it).  Then s = -adj(A) b / det, rounded to fp32, is used iff |s - m|^2 <= |u - w|^2 with m =
 *   0.5 (u + w) in fp64.  Otherwise the cheapest of u, w and fp32(m), first in that order on ties.  The error of p is
 *   (p, 1)^T Q (p, 1) evaluated at the fp32 point; cost = fp32(max(0, error)).  Every fp64 step is one rounded operation in the
 *   order csrc/decimate.cu writes (dec_place, dec_err), never contracted.
 * Validity (all must hold): |N(u) n N(w)| = 2; both vertices opposite the edge have valence (incident faces) > 3; no face of
 *   star(u) u star(w) that survives the collapse flips: its normals (p1 - p0) x (p2 - p0) before and after (u or w moved to
 *   the placement) have a positive dot product; faces with n . n = 0 before are exempt.
 * Selection: key = (fp32 bits of cost) << 32 | edge id (int64, >= 0; INT64_MAX = no candidate); m1[v] = min key over the
 *   candidate edges at v; m2[v] = min of m1 over v and N(v); edge selected iff key == m2[u] == m2[w].  Selected edges have
 *   pairwise non-adjacent endpoints, so their stars are disjoint.  Integer atomicMin only: order-independent.
 * Collapse: Q_u += Q_w, u moves to the placement, w dies, the two faces on the edge die, w is replaced by u in its other faces.
 *   Each collapse removes 2 faces; the caller applies at most ceil((F - target) / 2) collapses, those with the smallest keys.
 * Compaction keeps the live faces in order and the live vertices in ascending index.  Rounds end when F <= target or a
 *   round selects nothing.  All of it is deterministic: repeated runs are byte-identical.
 * V < 2^31 and 3F < 2^31, else PERF_EINVAL. */
/* d_flags [1] int32, zeroed by the caller, ORed with: 1 a face repeats a vertex, 2 a directed edge appears more than once,
 * 4 a directed edge has no opposite (open mesh).  Vertex indices must already lie in [0, V). */
int perf_decimate_check(const int32_t* d_faces, uint64_t F, uint64_t V, const int32_t* d_adj, const int32_t* d_adj_off, int32_t* d_flags,
                        void* stream);
/* d_quadrics [V,10] fp64 of the input mesh. */
int perf_decimate_quadrics(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_adj,
                           const int32_t* d_adj_off, double* d_quadrics, void* stream);
/* Per half-edge: d_key [3F] int64 (INT64_MAX unless a candidate with u < w), d_place [3F,3] fp32 (candidates only);
 * d_vmin [V] int64 = m1, filled by atomicMin into a caller-set INT64_MAX. */
int perf_decimate_edges(const float* d_vertices, const double* d_quadrics, uint64_t V, const int32_t* d_faces, uint64_t F,
                        const int32_t* d_adj, const int32_t* d_adj_off, int64_t* d_key, float* d_place, int64_t* d_vmin, void* stream);
/* d_vmin2 [V] = m2 (the caller copies m1 into it), d_selected [3F] uint8 = 1 for a selected edge (two launches). */
int perf_decimate_select(const int32_t* d_faces, uint64_t F, uint64_t V, const int64_t* d_key, const int64_t* d_vmin, int64_t* d_vmin2,
                         uint8_t* d_selected, void* stream);
/* Collapses the n selected edge ids d_edges in place: d_vertices, d_quadrics, d_faces; clears d_valive [V] / d_falive [F]
 * (uint8, set to 1 by the caller) of the dead vertices and faces.  n <= F / 2. */
int perf_decimate_collapse(const int64_t* d_edges, uint64_t n, float* d_vertices, double* d_quadrics, uint64_t V, int32_t* d_faces,
                           uint64_t F, const int32_t* d_adj, const int32_t* d_adj_off, const float* d_place, uint8_t* d_valive,
                           uint8_t* d_falive, void* stream);
/* d_voff / d_foff: exclusive int32 scans of d_valive / d_falive.  Writes the live vertices and quadrics at d_voff and the live
 * faces, renumbered by d_voff, at d_foff (two launches). */
int perf_decimate_compact(const float* d_vertices, const double* d_quadrics, uint64_t V, const uint8_t* d_valive, const int32_t* d_voff,
                          const int32_t* d_faces, uint64_t F, const uint8_t* d_falive, const int32_t* d_foff,
                          float* d_out_vertices, double* d_out_quadrics, int32_t* d_out_faces, void* stream);

/* ---- topological-noise removal for the decimation (opt-in: ops.decimate(max_cut=, min_component=); csrc/decimate.cu).  A
 * briefly fitted field leaves small handles through its walls and floaters in free space; the link condition keeps both, so
 * the collapse stalls.  Same input contract, half-edges and adjacency as the decimation above.
 * Components: vertices are connected when a face holds both; label(v) = the smallest vertex index of v's component, a
 *   face's label that of its vertex 0.  The label is unique, so any union-find gives it: hook (half-edge u -> w: atomicMin of
 *   label[label[u]] with label[w] when that is smaller), then pointer-jump each vertex to its root; passes until neither
 *   changes anything.  Box: per label, integer atomicMin/Max of the order-preserving int32 image of the fp32 coordinates
 *   (b >= 0 ? b : b ^ 0x7FFFFFFF of the bits).  Diagonal^2 = (dx dx + dy dy) + dz dz in fp64, d = fp64(hi) - fp64(lo), one
 *   rounded operation per step; a component is dropped iff diagonal^2 < min_component^2 (fp64).  Dropped vertices and faces
 *   are cleared in valive / falive and perf_decimate_compact removes them (order kept, vertices renumbered ascending).
 * Cut candidates: half-edge i = u -> w, u < w, link count > 2, opposite vertices o1 (of i) and o2 (of w -> u): the third
 *   vertices x in N(u) n N(w) \ {o1, o2} with x > w, so a 3-cycle {a < b < c} is found once, from edge (a, b).  Perimeter p =
 *   fp32((|u - w| + |w - x|) + |x - u|), |d| = sqrt((dx dx + dy dy) + dz dz), fp64 with rounded steps.  The candidate is the x
 *   of smallest (p, x) with p <= max_cut (fp32) and u, w, x vertex-manifold (the fan walk below from a vertex's first corner
 *   visits all its corners); key = fp32 bits(p) << 32 | i, INT64_MAX when there is none.
 * Selection: m1[v] = min key over the candidates at v in {u, w, x}; m2[v] = min of m1 over v and N(v); cycle selected iff
 *   key == m2[u] == m2[w] == m2[x].  Two selected cycles s, t (key_s < key_t) share no vertex and no edge between their
 *   vertices: a vertex b of t equal or adjacent to a vertex of s would have m2[b] <= key_s < key_t.  So their fans are
 *   disjoint and the cuts run in parallel without races.
 * Cut of selected cycle s (s-th in ascending half-edge order), u -> w -> x: fan step at v from corner c = v's corner whose
 *   next is c's prev.  The left arc of cycle vertex v runs from the face of its outgoing cycle half-edge (v's next is the
 *   next cycle vertex) by fan steps to, and including, the face of its incoming one (v's prev is the previous cycle vertex).
 *   New vertices u', w', x' at V + 3s + {0, 1, 2} copy position and quadric; v becomes v' in exactly its left arc's corners;
 *   all three arcs are walked before any corner is rewritten.  Caps (u, w, x) and (u', x', w') at F + 2s and F + 2s + 1 (no
 *   quadric).  Every directed edge still appears once with its opposite; the genus drops by 1 or the component count rises
 *   by 1: chi rises by 2.
 * Driver (ops.decimate): with min_component, drop before the first round; collapse rounds as above (bit-identical to a call
 *   without the new arguments up to the first stall when nothing is dropped); when a round selects nothing, F > target and
 *   max_cut is set: one cut round, the component drop, collapse rounds again; stop when F <= target or a cut round selects
 *   nothing. */
/* One union-find pass: hook over the half-edges, pointer jump over the vertices (two launches).  d_label [V] int32 = 0 .. V - 1
 * before the first pass; d_changed [1] int32, zeroed by the caller, becomes nonzero when the pass changed a label. */
int perf_decimate_components(const int32_t* d_faces, uint64_t F, uint64_t V, int32_t* d_label, int32_t* d_changed, void* stream);
/* d_box [V,6] int32 per label (min xyz, max xyz images), set by the caller to INT32_MAX x 3, INT32_MIN x 3; d_valive [V] /
 * d_falive [F] uint8 = 1 unless dropped (three launches). */
int perf_decimate_component_box(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_label,
                                double min_component, int32_t* d_box, uint8_t* d_valive, uint8_t* d_falive, void* stream);
/* Per half-edge: d_key [3F] int64, d_third [3F] int32 (x, candidates only); d_vmin [V] = m1 (caller-set INT64_MAX). */
int perf_decimate_cycles(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_adj,
                         const int32_t* d_adj_off, float max_cut, int64_t* d_key, int32_t* d_third, int64_t* d_vmin, void* stream);
/* d_vmin2 [V] = m2 (the caller copies m1 into it), d_selected [3F] uint8 (two launches). */
int perf_decimate_cycle_select(const int32_t* d_faces, uint64_t F, uint64_t V, const int64_t* d_key, const int32_t* d_third,
                               const int64_t* d_vmin, int64_t* d_vmin2, uint8_t* d_selected, void* stream);
/* Cuts the n selected cycles d_cycles (half-edge ids, ascending) in place: d_vertices [V + 3n, 3] and d_quadrics [V + 3n, 10]
 * hold the mesh's V rows first, d_faces [F + 2n, 3] its F faces; d_adj / d_adj_off are the F-face mesh's. */
int perf_decimate_cut(const int64_t* d_cycles, uint64_t n, const int32_t* d_third, float* d_vertices, double* d_quadrics, uint64_t V,
                      int32_t* d_faces, uint64_t F, const int32_t* d_adj, const int32_t* d_adj_off, void* stream);

/* ---- texture atlas of a triangle mesh (ops.texture_atlas drives it; csrc/texture.cu).  A T x T texture, T a power of two in
 * [256, 16384]; texel (x, y) (y up: image row T - 1 - y) covers [x, x + 1] x [y, y + 1] in texel units and has the Morton
 * index m = interleave(x in the even bits, y in the odd bits).
 * Charts: face f maps affinely onto a right isosceles triangle.  Its right-angle corner k0 is the corner opposite its longest
 *   edge (|p_{k+2} - p_{k+1}|^2 = (dx dx + dy dy) + dz dz in fp32; the lowest k on a tie); corners k0 + 1 and k0 + 2 (mod 3)
 *   follow along the legs, so every chart keeps the face's winding (positive signed area in UV, v up).
 * Cells: a cell is an aligned s x s square, s = 2^j >= 4, at Morton offset o (a multiple of s^2, lower-left corner
 *   (compact(o), compact(o >> 1))).  Its first face's chart has the right angle at the corner + (0.5, 0.5) and legs L = s - 3
 *   along +x (k0 + 1) and +y (k0 + 2); its second face's chart is that triangle rotated 180 degrees about the cell's centre.
 *   Bleed invariant: the 0.5-texel inset and the 4-texel gap between the hypotenuses make every texel whose centre lies within
 *   Chebyshev distance < 1 of a chart -- every texel a bilinear lookup on the chart reads -- a texel of the chart's face.
 * Size classes (caller): leg_f = sqrt(2 area_f) (perf_atlas_legs); with the density d (texels per world unit, fp32) the class
 *   of f is the smallest s = 2^j >= 4 with fp32(leg_f * d) <= s - 3.  Packing sorts the faces by class descending, then face
 *   index; consecutive faces of a class pair into cells (the last of an odd class alone); cell offsets are the exclusive scan
 *   of s^2 in that order, so every cell is aligned and the cells tile [0, used) of the Morton curve without gap or overlap.
 *   d is the result of a bisection over the bit patterns of the non-negative fp32 values, [0, +inf), that keeps "the cells
 *   fit in T^2 with no class above T" true at its lower end and false at its upper end.
 * Texels: texel m lies in the last cell whose offset is <= m (binary search); past the last cell it is unused (face -1,
 *   point 0).  In a chart's frame (right angle at the origin, legs along +a, +b) the texel centre is an integer point; its
 *   nearest chart point is found in integers (doubled coordinates), the nearer chart of the cell wins (the first on a tie),
 *   and with beta = fp32(2a' / 2L), gamma = fp32(2b' / 2L) the point is p = (p_k0 + beta (p_k0+1 - p_k0)) + gamma (p_k0+2 -
 *   p_k0), each step one rounded fp32 operation in that order.
 * F < 2^29 and V < 2^31, else PERF_EINVAL. */
/* d_legs [F] fp32: n = (p1 - p0) x (p2 - p0) in fp32, leg = sqrt(sqrt((nx nx + ny ny) + nz nz)), correctly rounded steps. */
int perf_atlas_legs(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, float* d_legs, void* stream);
/* d_order [F] int32: the faces in packing order.  h_classes [n_classes, 5] int32, descending side: (first position in d_order,
 * face count, first cell, Morton offset of the first cell, side), each class starting where the previous one ends.  Writes
 * d_uv [F,3,2] fp32 (u, v in [0, 1], v up), d_face_rec [F,4] int32 (cell offset, side, half 0/1, right-angle corner k0) and
 * d_cells [C,4] int32 (offset, side, first face, second face or -1), C = sum of ceil(count / 2). */
int perf_atlas_layout(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, int size, const int32_t* d_order,
                      const int32_t* h_classes, int n_classes, float* d_uv, int32_t* d_face_rec, int32_t* d_cells, void* stream);
/* Texels m in [m0, m0 + n) (m0 + n <= 2^28): d_face [n] int32 (-1 unused) and d_point [n,3] fp32 world sample points. */
int perf_atlas_texels(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_face_rec,
                      const int32_t* d_cells, uint64_t C, uint64_t m0, uint64_t n, int32_t* d_face, float* d_point, void* stream);

/* ---- chart texture atlas of a triangle mesh (ops.chart_atlas drives it; csrc/charts.cu).  Same texture as perf_atlas_*: T
 * a power of two in [256, 16384], texel (x, y) covers [x, x + 1] x [y, y + 1], y up; a texel's image index is
 * (T - 1 - y) T + x (row 0 at v = 1).  fp64 steps are one rounded operation each, in the order written; dot products are
 * (a0 b0 + a1 b1) + a2 b2.  Integer atomics only (min / max / add), so the result does not depend on arrival order.
 * Charts (rounds over the dual graph, the decimation's selection pattern):
 *   Start: chart f = face f, S_f = (p1 - p0) x (p2 - p0) in fp64 from the fp32 positions (twice the area-weighted normal),
 *   alpha_f = 0.  Axis n = S / |S|; a chart with S = 0 (zero-area faces only) has none.
 *   Dual edges (caller): an undirected edge {u, w} whose directed halves u -> w and w -> u each appear exactly once among the
 *   faces' half-edges (faces[f][k] -> faces[f][(k+1) % 3]); boundary and non-manifold edges are never crossed.  Listed in
 *   ascending order of the face corner 3f + k of their u < w half; edges [E,2] = the charts of the two faces.
 *   Merge of A and B: n_AB = normalise(S_A + S_B); alpha_AB = max over the parts X with S_X != 0 of alpha_X + ang(n_X . n_AB);
 *   0 when S_A = S_B = 0; not allowed when S_A + S_B = 0 otherwise.  ang(x) = sqrt(1 - x) P(x) + 1e-7 (Abramowitz & Stegun
 *   4.4.46, |error| <= 2e-8 on [0, 1], Horner from the top coefficient; x clamped to 1; x < 0 is not allowed).  The pad keeps
 *   the bound conservative: every face normal of a chart lies within alpha of its axis.  Allowed iff alpha_AB <= max_angle
 *   (radians, in (0, pi/2)).
 *   Selection: key = fp32 bits of alpha_AB << 32 | edge id (INT64_MAX when not allowed); cmin[c] = atomicMin over the allowed
 *   edges at c; an edge is selected iff key == cmin of both charts: a matching.  Merge: the lower chart id A absorbs B: S_A +=
 *   S_B, alpha_A = alpha_AB.  The caller relabels faces and edges (B -> A), drops the edges inside a chart (order kept) and
 *   stops when a round selects nothing.  Charts are then numbered 0 .. C - 1 in order of their lowest face.
 * Frames: n as above ((0, 0, 1) without one); b1, b2 of Duff et al. 2017: s = +1 if n.z >= 0 else -1, q = -1 / (s + n.z),
 *   b = (n.x n.y) q, b1 = (1 + ((s n.x) n.x) q, s b, -(s n.x)), b2 = (b, s + (n.y n.y) q, -n.y); b1 x b2 = n.  Vertex p of a
 *   chart: X = p . b1, Y = p . b2, and for k = 0 .. 7 with (c, s) = (cos, sin)(k pi / 16) (the fp64 constants in charts.cu):
 *   x = c X + s Y, y = c Y - s X.  Boxes per (chart, k): integer atomicMin / Max of the order-preserving int64 image of the
 *   fp64 bits.  The chart takes the k of smallest (x1 - x0)(y1 - y0), the first on a tie; when h = y1 - y0 > w = x1 - x0 it
 *   is turned by (x, y) -> (y, -x).  rot = k (+ 8 when turned), frame = (x0, y0, w, h) in the final coordinates.
 * Packing at density d (texels per world unit, fp32): cells = max(1, ceil(fp64(ext d))) per axis (capped at 2^24), the
 *   rectangle cells + 2g, g = 2.  The caller sorts the rectangles by (h desc, w desc, chart) and fills shelves of width T
 *   greedily: next[i] = the largest j with prefix[j] - prefix[i] <= T (binary search over the width prefix sums), shelf k
 *   starts at next^k(0) (binary lifting: level l of the table is next^(2^l)), its height is its first rectangle's.  They fit
 *   when every rectangle is <= T wide and tall and the shelf heights sum to <= T.  d is the bisection over the fp32 bit
 *   patterns of ops.texture_atlas.  Rectangle origin: (prefix[i] - prefix[start of its shelf], sum of the heights below).
 * UV: per corner in fixed point, 1/256 texel: per axis q = clamp(floor((local d) 256 + 0.5), 0, 256 cells), local = the
 *   corner's frame coordinate minus x0 / y0, U = 256 (origin + g) + q; uv = fp32(U) / fp32(256 T), exact.  Corners that share
 *   a vertex and a chart get identical bits.
 * Texels: texel centre P = (256 x + 128, 256 y + 128).  Face f's candidates are the texels with P in its fixed-point box
 *   widened by 256 g.  Face f contains P when its fixed-point doubled area is > 0 and each edge function (edge k+1 -> k+2)
 *   is > 0, or 0 on a top-left edge (dy < 0, or dy = 0 and dx < 0).  Otherwise d2 = the squared distance to the nearest of its
 *   edges 0-1, 1-2, 2-0 (fp64: s = clamp((r . e) / (e . e), 0, 1), 0 when e . e = 0; d2 = |r - s e|^2; strictly nearer wins),
 *   and f competes iff d2 <= (256 g)^2.  key = f when contained, else (fp32 bits of d2 + 1) << 32 | f; the texel takes the
 *   minimum key (INT64_MAX: unused).  Chart rectangles are disjoint and carry the g margin, so one chart competes per texel;
 *   since g > sqrt 2, every texel a bilinear lookup at a point of a face reads belongs to that face's chart.  inside[m] counts
 *   the faces that contain P: a texel with two marks its chart as overlapping (the caller splits such charts into single
 *   faces and lays out once more).  Texel point: contained -> b_k = fp32(w_k / area) (fp64 division), p = (p0 + b1 (p1 -
 *   p0)) + b2 (p2 - p0); else p = p_k + fp32(s) (p_k+1 - p_k) for the nearest edge k, fp32 steps.
 * F < 2^29 and V < 2^31, else PERF_EINVAL. */
/* d_sums [F,3] fp64 and d_alpha [F] (zero) of the single-face charts. */
int perf_chart_sums(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, double* d_sums, double* d_alpha, void* stream);
/* d_key [E] and d_cmin (per chart id, caller-set INT64_MAX, atomicMin) of the dual edges d_edges [E,2]. */
int perf_chart_edges(const int32_t* d_edges, uint64_t E, const double* d_sums, const double* d_alpha, double max_angle, int64_t* d_key,
                     int64_t* d_cmin, void* stream);
/* d_selected [E] uint8. */
int perf_chart_select(const int32_t* d_edges, uint64_t E, const int64_t* d_key, const int64_t* d_cmin, uint8_t* d_selected, void* stream);
/* Merges the n selected edges d_selected_ids: d_sums / d_alpha of the lower chart. */
int perf_chart_merge(const int32_t* d_edges, const int64_t* d_selected_ids, uint64_t n, double* d_sums, double* d_alpha, void* stream);
/* d_chart [F] in [0, C), d_sums [C,3]; d_box [C,8,4] int64 set by the caller to INT64_MAX, INT64_MIN, INT64_MAX, INT64_MIN;
 * writes d_rot [C] and d_frame [C,4] fp64 (two launches). */
int perf_chart_frames(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_chart, uint64_t C,
                      const double* d_sums, int64_t* d_box, int32_t* d_rot, double* d_frame, void* stream);
/* d_rect [C,4] int32: cells x, cells y, rectangle width, height at the density. */
int perf_chart_rects(const double* d_frame, uint64_t C, float density, int32_t* d_rect, void* stream);
/* n sorted rectangles: d_prefix [n + 1] int64 exclusive width prefix (prefix[n] = total), d_height [n]; every width <= size.
 * d_lift [levels, n + 1] (2^levels > n); writes d_start [n] (n past the last shelf) and d_shelf_h [n] (0 there);
 * levels + 1 launches. */
int perf_chart_shelves(const int64_t* d_prefix, const int32_t* d_height, uint64_t n, int size, int32_t* d_lift, int levels,
                       int32_t* d_start, int32_t* d_shelf_h, void* stream);
/* d_shelf_y [n] int64 exclusive prefix of d_shelf_h, d_order [n] the chart at each sorted position; writes d_origin [C,2]. */
int perf_chart_place(const int64_t* d_prefix, const int32_t* d_start, const int64_t* d_shelf_y, const int32_t* d_order, uint64_t n,
                     int32_t* d_origin, void* stream);
/* d_uvq [F,3,2] int32 fixed point and d_uv [F,3,2] fp32. */
int perf_chart_uv(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_chart, uint64_t C,
                  const double* d_sums, const int32_t* d_rot, const double* d_frame, const int32_t* d_rect, const int32_t* d_origin,
                  float density, int size, int32_t* d_uvq, float* d_uv, void* stream);
/* d_count [F] int64 candidate texels per face. */
int perf_chart_count(const int32_t* d_uvq, uint64_t F, int size, int64_t* d_count, void* stream);
/* d_offsets [F + 1] exclusive scan of the counts (d_offsets[F] = total).  d_key [T^2] int64 (caller-set INT64_MAX, atomicMin),
 * d_inside [T^2] int32 (zeroed, atomicAdd), both in image order. */
int perf_chart_raster(const int32_t* d_uvq, uint64_t F, int size, const int64_t* d_offsets, uint64_t total, int64_t* d_key,
                      int32_t* d_inside, void* stream);
/* The n used texels d_index [n] (image index) / d_face [n] (their key's face): d_point [n,3] fp32 world sample points. */
int perf_chart_texels(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_uvq, int size,
                      const int32_t* d_index, const int32_t* d_face, uint64_t n, float* d_point, void* stream);

/* ---- ray casting of a triangle mesh (ops.mesh_bvh / mesh_cast / mesh_shade drive it; csrc/raycast.cu).  d_vertices [V,3] fp32,
 * d_faces [F,3] int32 (any triangle soup; zero-area faces are never hit).  F < 2^30 and V < 2^31, else PERF_EINVAL.
 * BVH (Karras 2012 linear BVH, deterministic: two builds of one mesh are byte-identical):
 *   Codes: per face c = ((p0 + p1) + p2) / 3 in fp32; per axis with ext = hi - lo of the caller's box (the mesh's exact vertex
 *   min / max), u = fp32(fp32(c - lo) / ext) * 2^21, q = min(2^21 - 1, floor(max(u, 0))), q = 0 when ext = 0; code = the bits
 *   of qx at 3k, qy at 3k + 1, qz at 3k + 2 (63 bits, int64 >= 0).  The caller sorts (code, face) stably: d_order [F] int32 =
 *   the face at each leaf position, the sorted codes for the topology.
 *   Topology: delta(i, j) = clz64(code_i ^ code_j), or 64 + clz32(i ^ j) when the codes are equal, -1 for j outside [0, F);
 *   internal node i of F - 1 takes Karras's range and split (direction d = sign(delta(i, i+1) - delta(i, i-1)), binary
 *   searches for the range end and for the split gamma); children gamma and gamma + 1 are leaves when they end the range.
 *   F = 1: one leaf and no internal node; F = 0: nothing, every ray misses.
 *   Boxes: exact fp32 min / max, bottom-up, the second thread to reach a node (one atomic counter per node) unites its two
 *   child boxes, so the result does not depend on arrival order.
 * Node layout: d_nodes [F - 1, 16] 32-bit words, 64 bytes: words 0-5 the left child's box (lo xyz, hi xyz, fp32), 6-11 the
 *   right child's, 12 / 13 the left / right child link (c >= 0: internal node c; c < 0: leaf ~c), 14 the parent (-1 at the
 *   root, node 0), 15 zero.  One 64-byte read decides both children.  d_tris [F, 12] fp32, 48 bytes per leaf in leaf order:
 *   p0 xyz, the original face id (int32 bits), p1 xyz, 0, p2 xyz, 0 (the face's corners in its own order).
 *   d_leaf_parent [F] int32 (build only).  Bytes per face: 64 + 48 = 112 for the cast (+ 4 leaf parent, + 8 code and 4 order
 *   kept by ops.mesh_bvh).
 * Cast (closest hit): per ray a 16-byte record (t fp32, original face id int32 or -1 on a miss, b1 fp32, b2 fp32); the hit
 *   point is (1 - b1 - b2) p0 + b1 p1 + b2 p2.  On a miss t = +inf and b1 = b2 = 0.  Only t in [t_min, t_max] counts.  The
 *   result minimises (t, face id) lexicographically, independently of the traversal order.
 *   Triangle test: Woop, Benthin & Wald (JCGT 2013), two-sided: kz = the axis of the largest |d| (the first on a tie), kx =
 *   kz + 1, ky = kx + 1 (mod 3), swapped when d_kz < 0; Sx = d_kx / d_kz, Sy = d_ky / d_kz, Sz = 1 / d_kz; per vertex P = p - o,
 *   x = P_kx - Sx P_kz, y = P_ky - Sy P_kz; U = cx by - cy bx, V = ax cy - ay cx, W = bx ay - by ax, recomputed in fp64 (then
 *   rounded to fp32) when any of them is 0; a miss when they have mixed signs or det = (U + V) + W = 0; T = ((U Sz A_kz + V
 *   Sz B_kz) + W Sz C_kz); t = T / det, b1 = V / det, b2 = W / det.  Each step is one rounded fp32 operation in this order.
 *   Slab test (conservative; Ize 2013): per axis t0, t1 = (lo - o) / d, (hi - o) / d with the reciprocal 1 / d, widened by
 *   2^-16 (m / max |d| + |t|), m = the box's largest |lo - o|, |hi - o|; an axis with |d| < 2^-100 is parallel and culls
 *   only when o lies outside the slab by more than 2^-16 m.  A box is kept when its widened entry is <= the current best t
 *   (equality kept, for the face-id tie rule).  Traversal: ordered, nearer child first, per-thread stack of 96 entries: the
 *   common-prefix length delta grows strictly down a Karras tree and is at most 64 + 31.
 * Shade: from the records, d_rgb [R,3], d_distance [R], d_opacity [R], d_normal [R,3], d_back [R] uint8.  A hit has opacity 1,
 *   distance t, b0 = (1 - b1) - b2; normal = the blend b0 n0 + b1 n1 + b2 n2 of the vertex normals, normalised (the geometric
 *   normal (p1 - p0) x (p2 - p0) normalised without d_normals); colour = the blend of the uint8 vertex colours / 255, or with
 *   d_uv [F,3,2] and d_texture [T,T,3] uint8 (row 0 at v = 1) a bilinear lookup at the blended uv: x = u T - 0.5, y = (1 - v)
 *   T - 0.5 (texel (x, y) centred at integers), indices clamped to [0, T - 1].  back = d . n_geo > 0.  A miss has opacity 0,
 *   normal 0, colour 0 and distance 0 before the eval renders' background rule: distance += 5 (1 - opacity), rgb += 0.5 (1 -
 *   opacity). */
/* d_codes [F] int64.  h_lo3 / h_hi3: the code box (lo <= hi, finite). */
int perf_bvh_codes(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const float* h_lo3, const float* h_hi3,
                   int64_t* d_codes, void* stream);
/* From the sorted codes: links (words 12-15) of d_nodes [F - 1, 16] and d_leaf_parent [F]. */
int perf_bvh_topology(const int64_t* d_sorted_codes, uint64_t F, int32_t* d_nodes, int32_t* d_leaf_parent, void* stream);
/* Boxes (words 0-11) of d_nodes and d_tris [F, 12]; d_counters [F - 1] int32 zeroed by the caller. */
int perf_bvh_boxes(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const int32_t* d_order,
                   const int32_t* d_leaf_parent, int32_t* d_nodes, float* d_tris, int32_t* d_counters, void* stream);
/* d_hits [R, 16 bytes] for the rays d_rays_o / d_rays_d [R,3]. */
int perf_mesh_cast(const int32_t* d_nodes, const float* d_tris, uint64_t F, const float* d_rays_o, const float* d_rays_d, uint64_t R,
                   float t_min, float t_max, void* d_hits, void* stream);
/* d_hits [rows, W, 16 bytes] for the rays perf_raygen_pano generates for rows [row0, row0 + rows) of an H x W pano at h_pose;
 * a warp casts an 8 x 4 pixel patch. */
int perf_mesh_cast_pano(const int32_t* d_nodes, const float* d_tris, uint64_t F, const float* h_pose, int H, int W, int row0, int rows,
                        float t_min, float t_max, void* d_hits, void* stream);
/* d_rays_d [R,3]: the rays' directions (back-face test).  d_colors, d_normals, d_uv / d_texture nullable. */
int perf_mesh_shade(const void* d_hits, const float* d_rays_d, uint64_t R, const float* d_vertices, uint64_t V, const int32_t* d_faces,
                    uint64_t F, const uint8_t* d_colors, const float* d_normals, const float* d_uv, const uint8_t* d_texture, int T,
                    float* d_rgb, float* d_distance, float* d_opacity, float* d_normal, uint8_t* d_back, void* stream);

/* ---- normal texture of a decimated mesh (ops.bake_normal_texture / mesh_shade drive it; csrc/raycast.cu).  The low mesh
 * (d_vertices, d_faces, d_normals nullable, d_uv [F,3,2] its atlas, perf_atlas_layout) gets a tangent-space normal texture of
 * the high mesh (the full-resolution surface, d_hi_*, with its BVH from perf_bvh_*).  Each step is one rounded fp32 operation
 * in the order written; dot products are (a0 b0 + a1 b1) + a2 b2, cross products a x b = (a1 b2 - a2 b1, a2 b0 - a0 b2,
 * a0 b1 - a1 b0).
 *   Barycentrics of texel point p on its low face f: e1 = p1 - p0, e2 = p2 - p0, q = p - p0, g = e1 x e2, G = g . g;
 *   b1 = ((q x e2) . g) / G, b2 = ((e1 x q) . g) / G, b0 = (1 - b1) - b2.  G = 0: the flat texel, offset +inf.
 *   Casts: from p along +g^ and -g^ (g^ = g / sqrt(G)), t in [0, distance], the cast of perf_mesh_cast; the hit is the one of
 *   smaller t, +g^ on a tie; offset = +t or -t, +inf when neither ray hits (then the flat texel).
 *   High normal N at the hit: perf_mesh_shade's normal rule on the high mesh (blend of d_hi_normals normalised, else the
 *   geometric normal normalised).
 *   Frame (MikkTSpace for per-face charts: no corner is welded across faces): du_k = u_k - u0, dv_k = v_k - v0 (k = 1, 2),
 *   T_f = (dv2 e1 - dv1 e2) / (du1 dv2 - du2 dv1) per component; per corner n_k = the vertex normal (the unit geometric normal
 *   g^ without d_normals), t_k = T_f - n_k (n_k . T_f) normalised (0 when it is 0); n = (b0 n0 + b1 n1) + b2 n2 and t likewise,
 *   unnormalised; b = n x t (sign +1: every chart has positive signed area in uv).
 *   Encode: det = t . (b x n); flat when !(|det| > ((1e-12 |t|) |b|) |n|); c = (N . (b x n), t . (N x n), t . (b x N)) / det,
 *   normalised (flat when |c| = 0); texel = clamp(floor((c + 1) 127.5 + 0.5), 0, 255) per channel, RGB8 (+G = +v, OpenGL /
 *   glTF).  Flat texel: (128, 128, 255), also for an unused texel (d_face -1, offset +inf).
 *   Shade (perf_mesh_shade_normal_texture): perf_mesh_shade with, after the normal, a bilinear lookup of d_normal_texture
 *   [T,T,3] at the blended uv with the albedo's addressing, per channel on the bytes: top = (1 - fx) s00 + fx s10, bottom
 *   likewise, s = (1 - fy) top + fy bottom; c = s / 127.5 - 1; normal = ((c0 t + c1 b) + c2 n) normalised with the frame at the
 *   hit's barycentrics, or the normal without the texture when that vector is 0. */
/* d_texel [N,3] uint8 and d_offset [N] fp32 for the texels d_face [N] / d_point [N,3] of perf_atlas_texels; distance finite
 * and >= 0. */
int perf_normal_texture_bake(const int32_t* d_nodes, const float* d_tris, const float* d_hi_vertices, uint64_t hi_V,
                             const int32_t* d_hi_faces, uint64_t hi_F, const float* d_hi_normals, const float* d_vertices, uint64_t V,
                             const int32_t* d_faces, uint64_t F, const float* d_normals, const float* d_uv, const int32_t* d_face,
                             const float* d_point, uint64_t N, float distance, uint8_t* d_texel, float* d_offset, void* stream);
/* perf_mesh_shade's arguments plus d_normal_texture [T,T,3] uint8 (needs d_uv; d_texture nullable, of the same side T). */
int perf_mesh_shade_normal_texture(const void* d_hits, const float* d_rays_d, uint64_t R, const float* d_vertices, uint64_t V,
                                   const int32_t* d_faces, uint64_t F, const uint8_t* d_colors, const float* d_normals, const float* d_uv,
                                   const uint8_t* d_texture, const uint8_t* d_normal_texture, int T, float* d_rgb, float* d_distance,
                                   float* d_opacity, float* d_normal, uint8_t* d_back, void* stream);
/* d_tangents [F,3,3]: per face and corner the unit tangent t_k of the frame above (the one the normal texture is baked and
 * shaded with; 0 where T_f - n_k (n_k . T_f) is 0), from the low mesh (d_normals nullable) and its atlas d_uv [F,3,2].  A
 * glTF viewer's TBN with these tangents (w = +1), the interpolated vertex normals and B = N x T reproduces the frame at the
 * corners. */
int perf_mesh_corner_tangents(const float* d_vertices, uint64_t V, const int32_t* d_faces, uint64_t F, const float* d_normals,
                              const float* d_uv, float* d_tangents, void* stream);

/* ---- texture colour from registered panoramas (ops.texture_views drives it; csrc/texture_views.cu).  One thread per texel
 * point p of face f = d_face[i] (d_face -1: unused texel); d_face_normal [F,3] the unit geometric normals n (faces point into
 * free space).  d_views [n_views, H, W] float4 (16-byte aligned): r, g, b in [0, 1] and the distance D, 0 where the view did
 * not observe the pixel; h_poses [n_views, 16] row-major camera-to-world, rotation R, centre c.  n_views <= 64 (the 12 pose
 * floats of each view travel in the kernel arguments), else PERF_EINVAL.  Each step below is one rounded fp32 operation in
 * the order written; dot products are (a0 b0 + a1 b1) + a2 b2.
 *   Per view v, in registration order: q = p - c, dist2 = q . q; skip v when dist2 = 0; dist = sqrt(dist2).
 *   Grazing test: cos = -(n . q) / dist (= n . (c - p) / dist); skip v unless cos >= 0.15 (sup_info.py's normal_cos limit).
 *   Direction: e = (R^T q) / dist per component, e_k = ((R_0k q0 + R_1k q1) + R_2k q2) / dist.  alpha = atan2(e1, e0),
 *   beta = atan2(e2, sqrt(e0 e0 + e1 e1)); x = (0.5 - alpha * fp32(1 / 2pi)) * W - 0.5, y = (0.5 - beta * fp32(1 / pi)) * H
 *   - 0.5 (the inverse of common.cuh::pano_dir; pixel centres at integers).
 *   atan2: t = min(|x|, |y|) / max(|x|, |y|); when t > 0.41421356 (tan pi/8), t = (t - 1) / (t + 1) and pi/4 is added back;
 *   s = t t, q = ((c9 s + c7) s + c5) s + c3, r = t + (t s) q (c3..c9 in texture_views.cu); r = pi/2 - r when |y| > |x|,
 *   r = pi - r when x < 0, -r when y < 0; atan2(0, 0) = 0 (fp32 constants).  Max |error| against fp64 arctan2 of the same fp32
 *   inputs, over 2 M angles at three radii: 2.72e-7 rad (about one ulp of pi), so 1.8e-4 px of x at W = 2048.
 *   Taps: x0 = floor(x), y0 = floor(y), fx = x - x0, fy = y - y0; columns x0, x0 + 1 wrap modulo W (the seam is continuous on
 *   the sphere), rows y0, y0 + 1 clamp to [0, H - 1].  Tap weights (1 - fx)(1 - fy), fx (1 - fy), (1 - fx) fy, fx fy in that
 *   order.  A tap counts when its weight > 0, D > 0 and |dist - D| <= depth_tol (PeRF's visibility test made two-sided: a
 *   floater in front of an observed wall does not take the wall's colour).  With sw = the sum of the counting weights and
 *   s = the sum of weight * rgb over them (in tap order), view v counts when sw > 0, its colour rgb_v = s / sw (failed taps
 *   are dropped, not blended, so silhouettes do not bleed foreground colour onto the background).
 *   Blend: w_v = cos / dist2; over the views that count, in view order, acc += w_v rgb_v and wsum += w_v.
 *   Outputs: d_rgb [N,3] = acc / wsum (0 when wsum = 0), d_weight [N] = wsum, d_view [N] int32 = the view with the largest w_v
 *   (the first on a tie), -1 when no view counts, -2 for an unused texel (rgb and weight 0). */
int perf_texture_views(const float* d_points, const int32_t* d_face, uint64_t N, const float* d_face_normal, uint64_t F,
                       const float* d_views, int n_views, int H, int W, const float* h_poses, float depth_tol, float* d_rgb,
                       float* d_weight, int32_t* d_view, void* stream);

/* ---- pull-push fill of a texture's unused texels (ops.texture_fill drives it; csrc/texture_fill.cu).  d_image [T,T,3]
 * uint8 (rows in image order, row 0 at v = 1), d_used [T,T] uint8 (nonzero: used), T a power of two in [256, 16384];
 * h_empty 3 host bytes.  For each level l = 0 .. log2 T, block B_l(i, j) is the aligned square of texels [i 2^l, (i + 1) 2^l)
 * x [j 2^l, (j + 1) 2^l) in image coordinates (T is a power of two, so flipping the rows keeps 2^l alignment); count is the
 * number of used texels of the block and sum[c] the exact integer sum of channel c over them (int64: at 16384^2 the top sum
 * reaches 6.8e10).
 *   Output d_out [T,T,3]: a used texel is unchanged, byte for byte.  An unused texel p takes, per channel,
 *   (2 sum + count) / (2 count) (integer division: the mean rounded half up) of the smallest block with l >= 1 that contains
 *   p and has count > 0.  With no used texel at all, every texel is h_empty.
 *   Guarantee: for every level l and every block with count > 0, every filled texel of the block lies per channel in [min,
 *   max] of the block's used texels, so the box-filter mean over the block (a viewer's mip level l before its own rounding)
 *   does too: a mip block never takes a colour from outside itself and black is never introduced.  Neighbouring charts that
 *   share a block still mix: the fill does not make an atlas mip-safe between charts.  Base-level lookups that read only used
 *   texels do not change.
 * Integer arithmetic only, no atomics: the result does not depend on execution order.  d_out may be d_image (in place), no
 * other overlap.  d_image, d_used, d_out and d_workspace 16-byte aligned; d_workspace of at least
 * perf_texture_fill_workspace_bytes(T) bytes: 32 bytes per block of levels 5 .. log2 T, sum over l of (T >> l)^2 records, about
 * 4/3 T^2 / 1024 (2.8 MB at 8192^2); its contents on entry do not matter. */
uint64_t perf_texture_fill_workspace_bytes(int size);     /* 0 for a size outside the rule */
int perf_texture_fill(const uint8_t* d_image, const uint8_t* d_used, int size, const uint8_t* h_empty, void* d_workspace,
                      uint64_t workspace_bytes, uint8_t* d_out, void* stream);

/* ---- PNG encoder (ops.png_encode drives it; csrc/png.cu).  d_image [H,W,3] uint8 RGB, row 0 at the top; 1 <= H and
 * 1 <= W <= 21844 (a filtered row, 1 + 3 W bytes, fits a stored block), else PERF_EINVAL.  The file, byte for byte:
 *   Filter: each row takes the filter type f in {0 None, 1 Sub, 2 Up, 3 Average, 4 Paeth} (bpp 3; the row above row 0 and
 *   the bytes left of a row are 0) of the smallest sum over the row of |residual as int8|, the lower type on a tie (libpng's
 *   heuristic).  Filtered stream: per row f, then the 3 W residuals.
 *   Segments: consecutive whole rows, floor(65535 / (1 + 3 W)) per segment (the last may have fewer); each segment is
 *   compressed on its own, nothing refers back across a segment start.
 *   Tokens: per maximal run [rs, re) of equal bytes of a segment: byte rs is a literal; the remaining r = re - rs - 1 bytes
 *   are matches at distance 1 of min(258, left) while left >= 3, then 1-2 literals.
 *   Huffman codes (literal / length: symbols 0-285 with end-of-block 256 counted once; code lengths: symbols 0-18): the used
 *   symbols (fewer than two: the lowest unused symbols join with count 0) sorted by (count, symbol); the two-queue Huffman
 *   tree over them (of two smallest-weight candidates a leaf before an internal node of equal weight); leaf depths capped at
 *   the limit (15, code lengths 7); then, while the Kraft sum sum 2^(limit - len) exceeds 2^limit, one length count at the
 *   limit is dropped and one at the longest length l < limit that has any moves to l + 1 with a second added there (miniz's
 *   rule); the counts are handed out from the limit down to 1 in sorted order (the rarest symbols get the longest codes).
 *   Codes are the canonical codes of RFC 1951 3.2.2.  The distance code is two codes of length 1 (distance 1 is code 0).
 *   Block: BFINAL 0, BTYPE 2; HLIT = max(257, last used literal / length symbol + 1), HDIST = 2, HCLEN = max(4, the
 *   last nonzero code-length length in RFC order + 1).  The HLIT + 2 lengths as one sequence, per run of n equal values v:
 *   v = 0: 18 with min(n, 138) while n >= 11, then 17 with n if n >= 3, the rest literal 0s; v > 0: literal v, then 16 with
 *   min(left, 6) while left >= 3, the rest literal v.  Then the tokens, end-of-block, and an empty stored block (sync flush:
 *   3 zero bits, padding to a byte, 00 00 ff ff).  When that is more bytes than 5 + n (a stored block of the n bytes:
 *   00, LEN, NLEN little-endian, the bytes), the segment is that stored block instead.
 *   Stream: 78 01, the segments, the final empty fixed-Huffman block 03 00, the Adler-32 of the filtered stream
 *   (big-endian, combined from per-segment sums).
 *   File: the PNG signature, IHDR (W, H, 8, 2, 0, 0, 0), one IDAT per segment (the first starts with 78 01, the last ends
 *   with 03 00 and the Adler-32), IEND; every chunk with its CRC-32.
 * Integer arithmetic only; the bytes do not depend on execution order.
 * Calls, in order: perf_png_workspace_bytes(H, W) bytes of d_workspace (16-byte aligned; about H (1 + 3 W) + 65544 per
 * segment) and perf_png_max_bytes(H, W) bytes of d_out (every segment stored); perf_png_compress (3 launches: filter,
 * segments, finish) then perf_png_write (1 launch: the file into d_out, its size into d_file_bytes[0]).  The caller copies
 * the size, then that many bytes of d_out. */
uint64_t perf_png_workspace_bytes(int H, int W);           /* 0 outside the limits */
uint64_t perf_png_max_bytes(int H, int W);                 /* 0 outside the limits */
int perf_png_compress(const uint8_t* d_image, int H, int W, void* d_workspace, uint64_t workspace_bytes, void* stream);
int perf_png_write(const void* d_workspace, uint64_t workspace_bytes, int H, int W, uint8_t* d_out, uint64_t out_bytes,
                   uint64_t* d_file_bytes, void* stream);

/* ---- baseline JPEG encoder (ops.jpeg_encode drives it; csrc/jpeg.cu).  d_image [H,W,3] uint8 RGB, row 0 at the top;
 * 1 <= H, W <= 65535 and 1 <= quality <= 100, else PERF_EINVAL.  The file is libjpeg's (IJG / libjpeg-turbo, default ISLOW
 * path) for quality q, 4:4:4 sampling and a restart interval of ceil(W / 8) MCUs, byte for byte:
 *   Blocks: MX = ceil(W / 8) by MY = ceil(H / 8) MCUs, each one 8 x 8 block of Y, Cb and Cr; samples past the right or bottom
 *   edge repeat the last column or row.
 *   Colour: Y = (19595 R + 38470 G + 7471 B + 32768) >> 16, Cb = (-11059 R - 21709 G + 32768 B + 8421375) >> 16,
 *   Cr = (32768 R - 27439 G - 5329 B + 8421375) >> 16; the DCT input is the sample - 128.
 *   DCT: libjpeg's jpeg_fdct_islow (LL&M; CONST_BITS 13, PASS1_BITS 2; rows, then columns; DESCALE(x, n) = (x + 2^(n-1)) >> n,
 *   arithmetic), 32-bit integers; its outputs are 8 x the orthonormal DCT.
 *   Quantisers: with s = 5000 / q for q < 50 and 200 - 2 q otherwise, Q = clamp((K * s + 50) / 100, 1, 255) per entry K of
 *   the ITU-T T.81 Annex K.1 (luma) / K.2 (chroma) table.  Coefficient v -> sign(v) ((|v| + 4 Q) / (8 Q)), integer division
 *   (libjpeg-turbo's reciprocal form gives the same value for every |v| these DCTs produce).
 *   Entropy: the Annex K.3 / K.5 Huffman tables (DC 0 / AC 0 for Y, DC 1 / AC 1 for Cb and Cr); per block the DC difference
 *   to the same component of the MCU to the left (0 at the start of every MCU row), then the AC run-lengths in zigzag order
 *   with ZRL per 16 zeros before a nonzero coefficient and EOB when the block ends in zeros; magnitude bits of v < 0 are
 *   those of v - 1.  Each MCU row is one restart interval: its bits MSB first, padded with 1 bits to a byte, every FF
 *   followed by 00, then RST(r mod 8) after row r unless it is the last.
 *   File: SOI; APP0 JFIF 1.01, units 0, density 1:1, no thumbnail; DQT 0 (luma) and DQT 1 (chroma), 8-bit, zigzag order; SOF0
 *   (8-bit, H, W, components 1, 2, 3 at 1x1 with tables 0, 1, 1); DHT DC 0, AC 0, DC 1, AC 1; DRI MX; SOS (components 1, 2, 3
 *   with tables 0/0, 1/1, 1/1; 0, 63, 0); the rows; EOI.  629 bytes precede the entropy-coded data.
 * Integer arithmetic only; the only atomics are integer ORs, so the bytes do not depend on execution order.
 * Calls, in order: perf_jpeg_workspace_bytes(H, W) bytes of d_workspace (16-byte aligned; 16 bytes per MCU plus, per MCU row,
 * room for the row's unstuffed bits at the worst case of 4978 bits per MCU: about 10 bytes per pixel); perf_jpeg_compress (5
 * launches: bits, interval, emit, count, finish); then either perf_jpeg_file_bytes (the file's exact size into
 * d_file_bytes[0], a device-to-device copy) and, once the caller has read it, an output buffer of that size, or an output
 * buffer of perf_jpeg_max_bytes(H, W) bytes (every row at the worst case, every byte stuffed: about 19.5 bytes per pixel)
 * without the read; then perf_jpeg_write (1 launch): when the file fits the out_bytes of d_out, the file into d_out and its
 * size into d_file_bytes[0]; when it does not, nothing is written and d_file_bytes[0] = 0.  out_bytes below the smallest
 * file (631 bytes) is PERF_EINVAL.  The caller copies the size, then that many bytes of d_out. */
uint64_t perf_jpeg_workspace_bytes(int H, int W);          /* 0 outside the limits */
uint64_t perf_jpeg_max_bytes(int H, int W);                /* 0 outside the limits */
int perf_jpeg_compress(const uint8_t* d_image, int H, int W, int quality, void* d_workspace, uint64_t workspace_bytes,
                       void* stream);
int perf_jpeg_file_bytes(const void* d_workspace, uint64_t workspace_bytes, int H, int W, uint64_t* d_file_bytes, void* stream);
int perf_jpeg_write(const void* d_workspace, uint64_t workspace_bytes, int H, int W, uint8_t* d_out, uint64_t out_bytes,
                    uint64_t* d_file_bytes, void* stream);

/* ---- intra-only H.264 encoder (ops.h264_encode and perf_b200/video.py drive it; csrc/h264.cu).  d_frames [N,H,W,3] uint8
 * RGB, row 0 at the top; 1 <= N <= 65535, H and W even in [2, 16384], at most 139264 macroblocks a frame (MaxFS of level
 * 6.2), 0 <= qp <= 51, else PERF_EINVAL.  Every byte:
 *   Stream: H.264 Constrained Baseline (profile_idc 66, constraint_set0_flag and constraint_set1_flag set), 8-bit 4:2:0,
 *   CAVLC, one slice per picture.  Every frame is an IDR picture (nal_ref_idc 3), idr_pic_id = frame index & 1, frame_num 0,
 *   pic_order_cnt_type 2, max_num_ref_frames 0, so every frame is coded at once and every MP4 sample is a sync sample.
 *   Level: the smallest of Table A-1 (1 to 6.2, 1b skipped) whose MaxFS, MaxMBPS and sqrt(8 MaxFS) side bound admit the
 *   frame at the frame rate (perf_h264_level; 0, and PERF_EINVAL from perf_h264_parameter_sets, beyond 6.2).  The bit rate is
 *   not bounded by the level's MaxBR: constant QP decides it.
 *   Size: the picture is ceil(W / 16) x ceil(H / 16) macroblocks, padded by repeating the last RGB column and row, and cropped
 *   back with frame_cropping (right and bottom) in the SPS.
 *   Colour: BT.601 limited range, Y = ((66 R + 129 G + 25 B + 128) >> 8) + 16, Cb = ((-38 R - 74 G + 112 B + 128) >> 8) + 128,
 *   Cr = ((112 R - 94 G - 18 B + 128) >> 8) + 128 (arithmetic shifts), per pixel; each chroma sample is (s0 + s1 + s2 + s3 + 2)
 *   >> 2 of its 2 x 2 block.  The VUI carries video_full_range_flag 0, colour_primaries / transfer_characteristics /
 *   matrix_coefficients 6 / 6 / 6 and timing_info (num_units_in_tick fps_den, time_scale 2 fps_num, fixed_frame_rate_flag 1).
 *   PPS: CAVLC, pic_init_qp 26, chroma_qp_index_offset 0, deblocking_filter_control_present_flag 1.  Slice header:
 *   slice_type 7 (I), slice_qp_delta qp - 26, disable_deblocking_filter_idc 1, so the decoder's output is exactly the
 *   encoder's reconstruction (perf_h264_reconstruction).
 *   Macroblocks: Intra 16x16 or Intra 4x4.  Intra 16x16: the luma mode (vertical, horizontal, DC, plane; those whose
 *   neighbours exist) of least SATD + lambda bits(mb_type), SATD the sum over the 16 4x4 blocks of |Hadamard(source -
 *   prediction)| / 2, bits 3 for vertical / horizontal and 5 for DC / plane, lambda = round(0.85 2^((qp - 12) / 6)), at least
 *   1.  Intra 4x4: the blocks in decoding order, each the mode of the 9 (8.3.1.2; those whose neighbours exist, the top-right
 *   samples replaced by p[3, -1] where 6.4.11.4 makes them unavailable) of least SATD + lambda (1 when it is the most
 *   probable mode of 8.3.1.1, else 4), predicted from the reconstruction of the blocks before it; the macroblock's cost is
 *   their sum + lambda, and Intra 4x4 is chosen when that is below the Intra 16x16 cost.  Its 4x4 blocks are quantised
 *   whole (DC included) with the rounding term 2^qbits / 3; coded_block_pattern has one luma bit per 8x8 block with a
 *   nonzero level, coded by the Intra_4x4 column of Table 9-4; mb_qp_delta is present only when it is nonzero.  The
 *   chroma mode (DC,
 *   horizontal, vertical, plane) of least SATD(Cb) + SATD(Cr) + lambda bits(intra_chroma_pred_mode), bits 1, 3, 3, 5; ties
 *   go to the lower mode number.  Forward 4x4 core transform, quantised as sign(v) ((|v| MF + 2^qbits / 3) >> qbits), qbits
 *   15 + qp / 6, MF of qp % 6 and the position class {13107, 5243, 8066} ...; the luma DCs by the 4x4 Hadamard, halved
 *   (arithmetic shift), and the chroma DCs by the 2x2 one, both with MF of position 0, twice the rounding term and qbits + 1;
 *   chroma at QPc of Table 8-15.  coded_block_pattern: luma 15 when any AC level is nonzero, else 0; chroma 2 when any AC
 *   level, 1 when only DC levels are nonzero, else 0 (luma as above for Intra 16x16: 15 when any AC level is nonzero).  A macroblock whose CAVLC bits exceed 5934 (A.3.1: 128 + 3072 189 / 100)
 *   or one of whose levels would need level_prefix > 15 is coded I_PCM with the source samples.
 *   Integer arithmetic only; the only atomics are integer ORs, so the bytes do not depend on execution order.
 * Calls, in order: perf_h264_workspace_bytes(N, H, W) bytes of d_workspace (16-byte aligned; per frame 384 bytes of
 * reconstruction, 796 bytes of mode and levels and about 1.9 KB of slice data and staging per macroblock: about 11 bytes per
 * pixel); perf_h264_encode (one launch per wavefront t = x + 2 y that holds a macroblock, at most ceil(W / 16) + 2 ceil(H / 16)
 * - 2, then scan, emit, nal, finish); then
 * perf_h264_au_bytes (each frame's access-unit size into d_au_bytes[0..N-1], a device-to-device copy) and, once the caller
 * has read them, an output buffer of their sum; then perf_h264_write (1 launch and a copy): when the access units fit the
 * out_bytes of d_out, frame after frame into d_out, each as a 4-byte big-endian length and the IDR NAL unit (AVCC, emulation
 * prevention applied), and their total into d_total_bytes[0]; when they do not, nothing is written and d_total_bytes[0] is
 * the size they need.  perf_h264_reconstruction: the decoder's output, N frames of I420 (Y [H,W], Cb, Cr [H/2,W/2]), into
 * d_yuv.  perf_h264_mb_modes: per macroblock of every frame, raster order, 20 bytes: mode (0-3 the Intra 16x16 mode,
 * 4 I_PCM, 5 Intra 4x4), the chroma mode, the luma and chroma coded_block_pattern, and the 16 Intra4x4PredMode values in
 * raster order of the 4x4 blocks (2 outside Intra 4x4 macroblocks).  perf_h264_parameter_sets (host memory, no GPU): the SPS and PPS NAL units (header byte, no start code or length)
 * for the frame size and fps_num / fps_den frames a second, back to back into out, their sizes into sps_bytes, pps_bytes. */
int perf_h264_level(int H, int W, int fps_num, int fps_den);                  /* level_idc (10 .. 62), 0 outside the limits */
int perf_h264_parameter_sets(int H, int W, int fps_num, int fps_den, uint8_t* out, int out_bytes, int* sps_bytes, int* pps_bytes);
uint64_t perf_h264_workspace_bytes(int N, int H, int W);                      /* 0 outside the limits */
int perf_h264_encode(const uint8_t* d_frames, int N, int H, int W, int qp, void* d_workspace, uint64_t workspace_bytes, void* stream);
int perf_h264_au_bytes(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint64_t* d_au_bytes, void* stream);
int perf_h264_write(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint8_t* d_out, uint64_t out_bytes,
                    uint64_t* d_total_bytes, void* stream);
int perf_h264_reconstruction(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint8_t* d_yuv, void* stream);
int perf_h264_mb_modes(const void* d_workspace, uint64_t workspace_bytes, int N, int H, int W, uint8_t* d_modes, void* stream);

/* ---- fused training step (fixed-S sampler): forward with saves, composite backward, grid scatter ----
 * All per-sample buffers are SAMPLE-MAJOR: row = k * R + ray (k = sample index along the ray), so
 * that a warp of neighbouring rays reads/writes contiguous rows.  Replaces, for one optimisation
 * step, the call chain modules/scene/nerf.py:186-297 -> nerf_renderer.py:112-209 -> tcnn/nerfacc
 * forward + the autograd backward through them. */
#define PERF_PHASE_GEO 1   /* density net trained: nerf.py:186-257 (colour under no_grad)           */
#define PERF_PHASE_APP 2   /* colour net trained:  nerf.py:259-297 (density under no_grad)           */
typedef struct perf_train_buffers {
    float* d_sigma;      /* [S*R] density                                                   */
    float* d_weights;    /* [S*R] w = T * alpha                                             */
    float* d_trans;      /* [S*R] T                                                         */
    void*  d_rgb;        /* [S*R,4] fp16 sample colours (PHASE_APP only, 4th lane unused)   */
    void*  d_feat;       /* [S*R,32] fp16 features of the trained network                   */
    void*  d_h1;         /* [S*R,64] fp16 hidden 1                                          */
    void*  d_h2;         /* [S*R,64] fp16 hidden 2 (PHASE_APP only)                         */
    float* d_dist_acc;   /* [R] sum w*t_mid before the background rule                      */
    float* d_distloss;   /* [R] distortion-loss numerator per ray (flatten_eff_distloss * n_rays) */
    /* Ray splitting for small batches (optional, both NULL = off): the forward may cut every ray into
     * `segments` pieces handled by different threads; then d_weights / d_trans hold segment-LOCAL values
     * (T = 1 at the segment start) and d_seg_trans [PERF_MAX_SEGMENTS * R] the transmittance at each
     * segment start (row = segment * R + ray).  The forward writes the count it chose to *h_segments_out;
     * pass the same struct (and that count) to perf_train_backward_composite. */
    float*    d_seg_trans;
    uint32_t* h_segments_out;
} perf_train_buffers;
#define PERF_MAX_SEGMENTS 64

/* Forward of a training step: like perf_render_rays (PERF_FLAG_TRAINING semantics: jitter, training
 * background rule) and additionally fills `buf`. */
int perf_train_forward(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d,
                       uint64_t R, int phase, const perf_train_buffers* buf, void* stream);

/* Backward through the composite given per-ray gradients of the renderer outputs.
 * PHASE_GEO: d_out [S*R]   = dL/d(raw density logit)   (trunc_exp backward included)
 * PHASE_APP: d_out [S*R,3] = dL/d(colour pre-sigmoid)  (weights are detached, nerf_renderer.py:183)
 * d_g_* may be NULL (zero gradient).  d_distance_out: the forward's distance output (ReLU mask). */
int perf_train_backward_composite(int phase, uint32_t n_samples, uint32_t segments, float near, float far, uint64_t R,
                                  const float* d_jitter, const float* d_bg_noise, const perf_train_buffers* buf,
                                  const float* d_g_rgb, const float* d_g_distance, const float* d_g_opacity,
                                  const float* d_g_distloss, const float* d_distance_out, const float* d_opacity_out,
                                  float* d_out, void* stream);

/* The scalar losses of one training step and their gradients w.r.t. the renderer outputs in ONE launch
 * (nerf.py:208-238: smooth-L1 depth, beta 1e-2, + w_distloss * ratio * flatten_eff_distloss; nerf.py:281-287: smooth-L1
 * colour, beta 5e-2; torch `reduction='mean'`).  d_pred / d_gt [n] (n = R distances or 3 R colours); d_distloss [R] =
 * per-ray numerators from the forward or NULL; d_ratio: device scalar (the ramp min(2 progress, 1)) or NULL = 1;
 * d_inv_n_rays: device scalar 1 / (ray_id.max() + 1) or NULL = 1 / R.  d_loss3 = {total, mean smooth-L1, distortion
 * term}; d_g_pred [n], d_g_distloss [R] = d total / d input (NOT multiplied by the 2^7 loss scale). */
int perf_train_loss(const float* d_pred, const float* d_gt, uint64_t n, uint64_t R, float beta, float w_main,
                    const float* d_distloss, const float* d_ratio, const float* d_inv_n_rays, float w_distloss,
                    float* d_loss3, float* d_g_pred, float* d_g_distloss, void* stream);

/* Grid gradient for sample-major rows whose positions are recomputed from the rays:
 * d_dfeat [S*R, 32] fp32.  Same-cell neighbours inside a warp are merged before the atomics. */
int perf_hashgrid_bwd_rays(const perf_grid_cfg* cfg, const float* aabb6, const float* d_rays_o, const float* d_rays_d,
                           const float* d_jitter, uint64_t R, uint32_t n_samples, float near, float far,
                           const float* d_dfeat, float* d_dtable, void* stream);

/* The fixed-S training step's MLP backward WITH the fine-level grid scatter in its epilogue: perf_mlp_bwd on the R x S
 * sample-major rows (row = k * R + ray) of perf_train_forward; the thread that owns a row issues the reductions of levels
 * [8, 16) into d_dtable itself (positions recomputed from the rays as in perf_hashgrid_bwd_rays) and writes only the coarse
 * half of the feature gradient into d_dfeat (capacity >= 16 N floats) as eight LEVEL-MAJOR planes, plane l = float2 [N]
 * (what the march kernel reads coalesced).  Follow with perf_hashgrid_bwd_rays_coarse for levels [0, 8).  Together they
 * replace perf_mlp_bwd + perf_hashgrid_bwd_rays; the fine half of dfeat never reaches HBM and the L2-reduction-bound
 * scatter overlaps the latency-bound MMA phases. */
int perf_mlp_bwd_scatter(const perf_mlp_cfg* mlp, const void* d_weights_half, const void* d_feat, const void* d_h1, const void* d_h2,
                         const float* d_dz, uint64_t N, float* d_dweights, float* d_dfeat,
                         const perf_grid_cfg* grid, const float* aabb6, const float* d_rays_o, const float* d_rays_d, const float* d_jitter,
                         uint64_t R, uint32_t n_samples, float near, float far, float* d_dtable, void* stream);
int perf_hashgrid_bwd_rays_coarse(const perf_grid_cfg* cfg, const float* aabb6, const float* d_rays_o, const float* d_rays_d,
                                  const float* d_jitter, uint64_t R, uint32_t n_samples, float near, float far,
                                  const float* d_dfeat, float* d_dtable, void* stream);

/* Occupancy-grid interval sampler (nerfacc OccGridEstimator.sampling, levels=1, cone_angle=0;
 * nerf_renderer.py:145-155; SURVEY.md 8f row 1).  d_binaries: bool/uint8 [rx*ry*rz] (x slowest).
 * Pass 1 writes the per-ray sample counts; the caller exclusive-scans them into d_offsets and
 * allocates the packed outputs; pass 2 writes (ray_indices int64, t_starts, t_ends), sorted by ray. */
int perf_occ_count(const uint8_t* d_binaries, const int* h_res3, const float* h_aabb6, const float* d_rays_o, const float* d_rays_d,
                   const float* d_jitter, uint64_t R, float near, float far, float step, uint32_t pieces, int32_t* d_counts,
                   uint32_t* d_masks /* nullable, see below */, void* stream);
int perf_occ_write(const uint8_t* d_binaries, const int* h_res3, const float* h_aabb6, const float* d_rays_o, const float* d_rays_d,
                   const float* d_jitter, uint64_t R, float near, float far, float step, uint32_t pieces, const int64_t* d_offsets, uint64_t capacity,
                   const uint32_t* d_masks /* nullable */, int64_t* d_ray_indices, float* d_t_starts, float* d_t_ends, void* stream);
/* d_masks [R * pieces * 4] uint32 (optional, the same buffer in both passes): the count pass records WHICH lattice points of
 * every piece are samples (one bit each) and the write pass only expands those bits -- the grid is marched once, not twice.
 * Usable when a piece holds at most 128 lattice points, i.e. (far - near) / step / pieces + 1 <= 128 (else PERF_EINVAL). */
/* `pieces` (>= 1, the same in both passes): every ray's lattice range is cut into that many consecutive parts marched by
 * different threads -- a ray is a serial walk of up to (far - near) / step lattice points, and 8192 rays alone leave the GPU
 * empty.  d_counts and d_offsets then have R * pieces entries indexed [ray * pieces + piece] (exclusive scan over all of
 * them); the packed output is the same, sorted by ray and t.  A ray's range is d_offsets[ray * pieces] .. [(ray+1) * pieces]. */

/* ---- fused training step for PACKED samples (the occupancy sampler PeRF trains with, configs/nerf.yaml:25;
 * nerf_renderer.py:145-183, nerf.py:186-297): perf_occ_count/write -> perf_fields_packed ->
 * perf_composite_packed_fwd -> losses -> perf_composite_packed_bwd -> perf_mlp_bwd -> perf_hashgrid_bwd_merged.
 * All per-sample buffers are indexed by the packed sample number n (sorted by ray). */

/* Both fields at N packed samples in one launch: position o + d (ts+te)/2, aabb normalisation and selector
 * (ngp_nerf.py:136-162), encode of both grids, both MLPs.  args: only grid / tables / weights / aabb / flags are read.
 * d_sigma [N] fp32, d_rgb_half4 [N,4] fp16 (4th lane unused), d_x01 [N,3] fp32 (normalised position; masked-out
 * samples get the in-box stand-in their features were taken at).  phase 0: no saves; PERF_PHASE_GEO / _APP: also
 * d_feat [N,32], d_h1 [N,64] (and d_h2 [N,64] for _APP) fp16 of the trained network. */
int perf_fields_packed(const perf_render_args* args, const float* d_rays_o, const float* d_rays_d, const int64_t* d_ray_indices,
                       const float* d_t_starts, const float* d_t_ends, uint64_t N, const int64_t* d_n_dev /* nullable, see below */,
                       int phase, float* d_sigma, void* d_rgb_half4, float* d_x01, void* d_feat, void* d_h1, void* d_h2, void* stream);

/* Composite of packed samples, one warp per ray: w, T (nerfacc render_weight_from_density), opacity / distance /
 * colour (accumulate_along_rays), background rule (PERF_FLAG_TRAINING in flags: nerf_renderer.py:192-194, else
 * :195-197), distortion-loss numerator per ray (flatten_eff_distloss * n_rays).  Samples whose transmittance is below
 * early_stop_eps get weight 0 and T = 0 -- identical to nerfacc dropping them inside OccGridEstimator.sampling.
 * d_offsets int64 [R+1]; d_weights / d_trans [N]; d_rgb_out [R,3]; the others [R]. */
int perf_composite_packed_fwd(const int64_t* d_offsets, const float* d_t_starts, const float* d_t_ends, const float* d_sigma,
                              const void* d_rgb_half4, uint64_t R, float early_stop_eps, uint32_t flags, const float* d_bg_noise,
                              float* d_weights, float* d_trans, float* d_rgb_out, float* d_distance_out, float* d_opacity_out,
                              float* d_dist_acc, float* d_distloss, void* stream);
/* Its backward: d_dz [N] = dL/d(raw density logit) (PERF_PHASE_GEO, trunc_exp backward included) or [N,3] =
 * dL/d(colour pre-sigmoid) (PERF_PHASE_APP).  d_g_* [R,.] may be NULL. */
int perf_composite_packed_bwd(int phase, const int64_t* d_offsets, const float* d_t_starts, const float* d_t_ends, const float* d_sigma,
                              const void* d_rgb_half4, uint64_t R, const float* d_bg_noise, const float* d_weights, const float* d_trans,
                              const float* d_distance_out, const float* d_opacity_out, const float* d_dist_acc,
                              const float* d_g_rgb, const float* d_g_distance, const float* d_g_opacity, const float* d_g_distloss,
                              float* d_dz, void* stream);
/* perf_hashgrid_bwd with the number of levels whose same-cell runs of consecutive samples are merged before the
 * atomics chosen by the caller (packed samples are 5e-4 apart: runs exist up to resolution ~1000). */
int perf_hashgrid_bwd_merged(const perf_grid_cfg* cfg, const float* d_x01, const float* d_dfeat, uint64_t N, const int64_t* d_n_dev,
                             float* d_dtable, uint32_t n_merge_levels, void* stream);
/* d_n_dev (perf_fields_packed, perf_mlp_bwd, perf_hashgrid_bwd_merged): the sample count of a step is only known on the device
 * (it is the last entry of the offsets scan).  Passing N = the CAPACITY of the buffers and d_n_dev = a device int64 holding the
 * live count makes the launch sequence independent of the count -- the whole occupancy-sampler step can be captured into a CUDA
 * graph and replayed without a host read.  perf_occ_write's `capacity` (0 = unlimited) drops samples that would not fit; the
 * caller clamps the offsets and the count to it. */

/* ---- normal-consistency loss of the density phase (MonoSDF's L1 + angular normal loss against the supervision normals that
 * SupInfoPool.rand_ray_color_data returns, sup_info.py:236-259, and train_one_step_geo drops, nerf.py:193).  Definition, per sample i
 * of a density-phase training step at normalised position x01:
 *   h1 = the fp16 layer-1 activation the training forward saved, m = [h1 > 0] (the eval normals' m = [h > 0] on the fp32 h differs
 *   only where 0 < h < 2^-25, which rounds to an fp16 zero), g = W1^T (m . w_out) (fp16 shadow weights as fp32),
 *   grad01 = sum_levels of perf_hashgrid_bwd_input's arithmetic with dL/dfeature = g on the fp16 geo table, grad = grad01 / aabb extent,
 *   n_i = -grad / |grad|, and n_i = 0 when the selector is false, |grad| = 0, w_i = 0 or T_i = 0 (a dropped sample).
 * Ray normal N_r = sum_i sg(w_i) n_i (the weights are detached: the loss turns the density gradient where the surface already is).
 * Loss: g^_r = gt_r / |gt_r|; ray r is valid iff |gt_r| > 0.5 and |N_r| > 1e-6; N^_r = N_r / |N_r|;
 *   l_r = |N^_r - g^_r|_1 + (1 - N^_r . g^_r),  L_n = sum_valid l_r / max(#valid, 1),
 *   dl/dN = (I - N^ N^T)(sign(N^ - g^) - g^) / |N| with sign(0) = 0.
 * The supervision normals point toward the camera (the orientation of -grad raw); pools without a normal map hold zeros. */
typedef struct perf_sample_layout {
    uint64_t R;                    /* rays                                                                                   */
    uint64_t N;                    /* sample rows: R * n_samples (fixed-S) or the capacity of the packed buffers             */
    float    aabb[6];              /* the renderer's box (min xyz, max xyz)                                                  */
    /* packed (occupancy) layout, selected by d_x01 != NULL: samples sorted by ray, as perf_fields_packed saved them          */
    const float*   d_x01;          /* [N,3] perf_fields_packed's saved normalised positions                                   */
    const int64_t* d_offsets;      /* [R+1] per-ray ranges                                                                    */
    const int64_t* d_ray_indices;  /* [N] (perf_normals_train_bwd only)                                                       */
    const int64_t* d_n_dev;        /* nullable: live sample count in device memory (<= N), as perf_fields_packed             */
    /* fixed-S layout (d_x01 == NULL): sample-major rows k * R + ray, positions recomputed from the rays bit for bit as the forward */
    const float* d_rays_o;         /* [R,3]                                                                                   */
    const float* d_rays_d;         /* [R,3]                                                                                   */
    const float* d_jitter;         /* [R] or NULL                                                                             */
    uint32_t n_samples, segments;  /* S and the segment count perf_train_forward chose (perf_train_buffers)                   */
    float near, far;
    const float* d_seg_trans;      /* perf_train_buffers::d_seg_trans when segments > 1                                       */
} perf_sample_layout;
/* Sample normals and ray normals of a density-phase step.  d_params_half: the density net's fp16 flat params (MLP | grid; 16 levels,
 * 32 -> 64 -> 1, else PERF_EUNSUPPORTED); d_h1 [N,64] fp16, d_weights / d_trans [N]: the step's saves (perf_train_forward /
 * perf_fields_packed + perf_composite_packed_fwd).  Writes d_sample_normal [N,3] = n_i, d_inv_norm [N] = 1 / |grad| (0 where n_i = 0)
 * and d_ray_normal [R,3] = N_r (deterministic: a fixed summation order per ray, no atomics). */
int perf_normals_train_fwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* d_params_half, const perf_sample_layout* layout,
                           const void* d_h1, const float* d_weights, const float* d_trans,
                           float* d_sample_normal, float* d_inv_norm, float* d_ray_normal, void* stream);
/* The loss above in one launch: d_loss2 = {L_n, #valid}; d_g_ray_normal [R,3] = dL_n / dN_r (unscaled, 0 on invalid rays).
 * d_ray_normal / d_gt_normal [R,3] (NULL allowed when R = 0: d_loss2 = {0, 0}).  The valid count stays on the device. */
int perf_normal_loss(const float* d_ray_normal, const float* d_gt_normal, uint64_t R, float* d_loss2, float* d_g_ray_normal, void* stream);
/* Backward of the ray normals into the density net: with G_r = d_g_ray_normal [R,3] and u = -(I - n n^T)(w_i G_r) / |grad|,
 * v = u / aabb extent (= dL/d grad01), per level dg = sum_d v_d scale s' A_d (the dfeat branch of perf_hashgrid_bwd_bwd_input) and the
 * table term of the same function; P = sum_i m_i (x) dg_i (64 x 32), dW1 = diag(w_out) P, dw_out_j = sum_k W1_jk P_jk.
 * d_sample_normal / d_inv_norm: perf_normals_train_fwd's outputs.  d_dparams [n_mlp + 2 n_entries] fp32 in the flat parameter layout
 * (MLP | grid), ACCUMULATED (fp32 atomics; the caller zeroes it, or passes the step's gradient).  Samples with w_i |G_r| = 0 issue
 * nothing. */
int perf_normals_train_bwd(const perf_grid_cfg* grid, const perf_mlp_cfg* mlp, const void* d_params_half, const perf_sample_layout* layout,
                           const void* d_h1, const float* d_weights, const float* d_trans,
                           const float* d_sample_normal, const float* d_inv_norm, const float* d_g_ray_normal,
                           float* d_dparams, void* stream);

/* Batch draw (sup_info.py:253-259): dst_k[b, :] = src_k[idx[b], :] for up to 6 row-major fp32 arrays of row widths
 * h_width[k] in one launch.  h_src / h_dst: HOST arrays of device pointers. */
int perf_gather_rows(const int64_t* d_idx, uint64_t B, int n_arrays, const float* const* h_src, float* const* h_dst, const int* h_width, void* stream);

/* The whole batch draw in one launch: B SORTED uniform row indices in [0, M) from the running sums d_csum [B+1] (fp64) of i.i.d.
 * Exp(1) variates -- S_k / S_{B+1} are the order statistics of B uniforms, i.e. torch.randint followed by a sort, without the
 * sort -- and the gather of perf_gather_rows with them.  d_idx_out [B] int64 or NULL.  With the pool stored in Morton order
 * of its pixels a sorted batch is a spatially coherent one. */
int perf_draw_gather_rows(const double* d_csum, uint64_t B, uint64_t M, int64_t* d_idx_out, int n_arrays, const float* const* h_src,
                          float* const* h_dst, const int* h_width, void* stream);

/* Diagnostic (bench.py's train_roofline denominator): n_atomics reductions of `vec` (1, 2 or 4) floats at pseudo-random
 * vec-aligned slots of d_table [n_floats] -- the L2 atomic rate that bounds the grid-gradient scatter. */
int perf_debug_atomic_rate(float* d_table, uint64_t n_floats, uint64_t n_atomics, int vec, void* stream);

/* Occupancy-grid update (nerfacc OccGridEstimator.update_every_n_steps, levels = 1; nerf.py:159-168).
 * perf_occ_points: a uniformly jittered point inside each listed cell (d_cell_idx int64 [n], NULL = cells 0..n-1),
 * d_x [n,3]; the caller evaluates its occ_eval_fn there.  perf_occ_update: occs[c] = max(occs[c] * ema_decay, occ),
 * then binaries = occs > min(mean(occs), occ_thre) (deterministic two-stage mean).  d_workspace: 2 * PERF_OCC_PARTIALS doubles. */
#define PERF_OCC_PARTIALS 1024
int perf_occ_points(const int64_t* d_cell_idx, uint64_t n, const int* h_res3, const float* h_aabb6, uint64_t seed, float* d_x, void* stream);
int perf_occ_update(float* d_occs, uint64_t n_cells, const int64_t* d_cell_idx, const float* d_occ_new, uint64_t n, float ema_decay,
                    float occ_thre, uint8_t* d_binaries, double* d_workspace, void* stream);

/* MLP backward helpers on the saved fp16 activations (tcnn kernel_mlp_fused_backward pieces; the
 * matrix products themselves are plain GEMMs left to cuBLAS):
 *   perf_mlp_bwd_out: d_dh [N,64] fp16 = (d_dz [N,n_out] fp32 @ Wout[:n_out] fp16) * (d_h > 0)
 *   perf_relu_mask:   d_dh *= (d_h > 0), in place, n_values fp16 values each */
int perf_mlp_bwd_out(const float* d_dz, int n_out, const void* d_wout_half, const void* d_h, void* d_dh, uint64_t N, void* stream);
int perf_relu_mask(void* d_dh, const void* d_h, uint64_t n_values, void* stream);

/* Fused Adam on a flat fp32 parameter vector + refresh of its fp16 shadow
 * (torch.optim.Adam at nerf.py:171,180,253,293; betas/eps defaults).  grad_scale multiplies
 * the gradient first (the reference never unscales its 128x GradScaler; pass 1 to keep that). */
int perf_adam_step(float* d_params, const float* d_grads, float* d_exp_avg, float* d_exp_avg_sq,
                   void* d_params_half /*nullable*/, uint64_t n, float lr, float beta1, float beta2,
                   float eps, uint32_t step /*1-based*/, float grad_scale, void* stream);

/* d_dst[0..n) = h_values[0..n), n <= 8, stream-ordered; the values travel as kernel arguments, so the
 * host array may be reused immediately (feeds the device-side schedule of a replayed CUDA graph). */
int perf_set_scalars(float* d_dst, const float* h_values, int n, void* stream);

/* Same update with {lr, 1 - beta1^step, sqrt(1 - beta2^step)} read from DEVICE memory (d_hyper[3]) at
 * run time: the launch can live inside a captured CUDA graph and be replayed with a new schedule. */
int perf_adam_step_dev(float* d_params, const float* d_grads, float* d_exp_avg, float* d_exp_avg_sq,
                       void* d_params_half /*nullable*/, uint64_t n, const float* d_hyper, float beta1, float beta2,
                       float eps, float grad_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PERFB200_H */
