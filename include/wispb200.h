/*
 * wispb200.h -- C ABI of libwispb200.so: the H100 (sm_90a) volumetric render path that drops in behind
 * kaolin-wisp's Pipeline / BaseTracer / BLASGrid / BaseNeuralField API.
 *
 * Conventions (SURVEY.md 8(b)):
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch owns all tensors; the library borrows
 *     them for the duration of the call and allocates nothing persistent);
 *   - every entry point takes the cudaStream_t to launch on (as void*), never synchronises the host,
 *     and returns 0 on success or a negative wb_status; wb_last_error() describes the last failure of the
 *     calling thread.  The reference raises from AT_ERROR/AT_CUDA_CHECK instead
 *     (wisp/csrc/ops/hashgrid_interpolate.cpp:66-68, uniform_sample_cuda.cu:95);
 *   - layouts are the reference's: row-major, float32 unless stated, int64 ridx, bool(u8) masks;
 *   - every launch, copy and memset of a call goes to that stream, none to the legacy default stream; work the library forks onto
 *     its own side stream (the chunked precision-1 backward of wb_rf_shade_bwd) joins the caller's stream before the call returns;
 *   - entry points may be called concurrently from several host threads, on one device or on several: the library's shared state
 *     (per-device side streams and events, dynamic shared-memory limits, which are only ever raised) is guarded, the error text and
 *     the wb_rf_workspace_holds_ray_rows hint are per thread;
 *   - every stream-taking entry point can be captured into a CUDA graph (wb_sdf_trace's cooperative launch included) over buffers
 *     allocated before the capture; a count -> scan -> fill chain is captured with the fill's outputs sized to a capacity, since
 *     the caller reads the total on the host between the stages.  A captured wb_rf_shade_bwd never forks onto the shared side
 *     stream: it runs the one-stream schedule (the same sums up to the order of the atomic additions), so captures and eager calls
 *     of other threads cannot mix.  tests/test_gpu_stream_contract.py checks all of this per entry, the chunked backward included.
 *
 * Each group cites the reference interface it replaces (paths relative to the kaolin-wisp checkout).
 */
#ifndef WISPB200_H_
#define WISPB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* wb_stream;            /* cudaStream_t */

enum wb_status {
    WB_OK = 0,
    WB_ERR_INVALID = -1,            /* bad argument / unsupported configuration */
    WB_ERR_CUDA = -2,               /* a CUDA runtime call failed (message has the cudaError string) */
    WB_ERR_NODEVICE = -3            /* no sm_90 device: there is NO CPU fallback */
};

const char* wb_last_error(void);
int wb_version(void);
/* Device check used by the host shim at import: WB_OK only on compute capability 9.0. */
int wb_device_check(int device);
/* Number of kernels this library launched since load (bench.py's gpu_launches). */
int64_t wb_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Neural field descriptor (NeuralRadianceField + HashGrid + BasicDecoder x2 + PositionalEmbedder)
 *   wisp/models/nefs/nerf.py:30-173, wisp/models/grids/hash_grid.py:27-89, wisp/models/grids/utils.py:13-63
 * Plain C struct, passed by pointer (host memory); the pointers inside are device pointers.
 * ---------------------------------------------------------------------------------------------- */
#define WB_MAX_LODS 32
#define WB_MAX_LAYERS 8

typedef struct wb_nef_desc {
    /* hash grid */
    int32_t num_lods;                       /* L                                                     */
    int32_t feature_dim;                    /* F (even, ops/grid.py:83-84)                           */
    int32_t codebook_size;                  /* T = 2^codebook_bitwidth (hashgrid_interpolate.cpp:59) */
    int32_t multiscale;                     /* 0 'cat', 1 'sum' (hash_grid.py:226-231)               */
    int32_t lod_idx;                        /* 'cat': features of LODs >= lod_idx are zeroed         */
    int32_t resolutions[WB_MAX_LODS];       /* MultiTable.resolutions                                */
    int64_t begin_idxes[WB_MAX_LODS + 1];   /* MultiTable.begin_idxes (rows)                         */
    const float* table;                     /* MultiTable.feats [rows, F] fp32 master                */
    /* embedders: 0 none, 1 identity, 2 positional (no input), 3 positional + input                   */
    int32_t pos_mode, pos_freq;             /* nerf.py:103-104                                       */
    int32_t view_mode, view_freq;           /* nerf.py:105-106 (include_input=True => never 0/2)     */
    /* decoders: packed parameters [W0 (out x in, row-major like nn.Linear.weight), b0?, W1, b1?, ...] */
    int32_t has_bias;
    int32_t dens_layers;                    /* linear layers of decoder_density = num_layers + 1     */
    int32_t dens_dims[WB_MAX_LAYERS + 1];
    int32_t col_layers;                     /* linear layers of decoder_color   = num_layers + 2     */
    int32_t col_dims[WB_MAX_LAYERS + 1];
    const float* dens_params;
    const float* col_params;
    /* ---- feature grids other than the hash grid (fused path only; zero for the hash grid) ----
     * grid_kind 1 = TriplanarGrid (triplanar_grid.py:24-150): num_lods = LODs used (lod_idx + 1), feature_dim = 3 * fdim
     *   (the width of one LOD's [plane, fdim] block), resolutions[l] = 2^(log_base_resolution + l) (plane side - 1),
     *   grid_ptrs = 3*num_lods planes (fmx, fmy, fmz of LOD 0, LOD 1, ...), each [1, fdim, res+1, res+1] fp32.
     * grid_kind 2 = OctreeGrid (octree_grid.py:24-226): num_lods = LODs used, feature_dim = F, grid_ptrs = features[0..num_lods)
     *   each [pyramid_dual[0,l]+1, F] fp32; oct/points/trinkets/base_lod/half_round as in wb_octree_interp_fwd.
     * For both: lod_idx = num_lods (nothing is zeroed), table / resolutions-as-hash / begin_idxes / codebook_size unused.
     * grid_grads: same shapes as grid_ptrs, accumulated into by the backward entry points (their grad_table may be NULL).
     * grid_layout (grid_kind 1 only): 0 = the reference's plane layout [1, fdim, res+1, res+1]; 1 = channel-last [res+1, res+1, fdim]
     *   for grid_ptrs AND grid_grads (fdim == 4: one 16-byte load / one 16-byte reduction per texel instead of four 4-byte ones;
     *   wb_triplane_relayout converts between the two). */
    int32_t grid_kind;
    int32_t base_lod, half_round;
    const float* const* grid_ptrs;          /* HOST array of device pointers */
    float* const* grid_grads;               /* HOST array of device pointers (backward only) */
    const struct wb_octree* oct;            /* grid_kind 2 */
    const int16_t* points;
    const int32_t* trinkets;
    int32_t grid_layout;
} wb_nef_desc;

/* Rays (wisp/core/rays.py:19-36).  near/far: scalars, or per-ray arrays when near_v != NULL. */
typedef struct wb_rays {
    const float* origins;                   /* [R,3] */
    const float* dirs;                      /* [R,3] */
    int64_t num_rays;
    float dist_min, dist_max;
    const float* near_v;                    /* optional [R] */
    const float* far_v;                     /* optional [R] */
} wb_rays;

/* Occupancy structure (wisp/accelstructs/octree_as.py:43-62): the SPC tensors the reference keeps. */
typedef struct wb_octree {
    const uint8_t* octree;                  /* [nbytes] one byte per non-leaf node, breadth first   */
    const int32_t* prefix;                  /* [nbytes+1] exclusive sum of popcounts ("exsum")      */
    int64_t nbytes;
    int32_t max_level;
    const uint32_t* bits;                   /* optional dense bitmask of `bits_level` built by       */
    int32_t bits_level;                     /*   wb_octree_build_bits; NULL -> descend the bytes     */
    int32_t has_bbox;                       /* optional: bounding box (normalised [-1,1] coords) of  */
    float bbox_lo[3], bbox_hi[3];           /*   the occupied cells of the marched level; lets the   */
                                            /*   marcher skip candidates that cannot be occupied     */
    const uint32_t* coarse_bits;            /* optional: dilated occupancy of `coarse_level` built   */
    int32_t coarse_level;                   /*   by wb_octree_build_coarse from `bits`; lets the     */
} wb_octree;                                /*   marcher skip whole 32-candidate words. NULL -> off  */

/* ------------------------------------------------------------------------------------------------
 * SPC helpers  -- replace kaolin.ops.spc.unbatched_query; occupancy bitmasks for the marcher
 *   call sites: wisp/ops/spc/conversions.py:84-87, wisp/accelstructs/octree_as.py:146-163
 * ---------------------------------------------------------------------------------------------- */
/* bits: zero-initialised uint32 [(8^level + 31)/32]; bit (x<<2L | y<<L | z) set iff the level-L cell is occupied. */
int wb_octree_build_bits(const int16_t* level_points, int64_t num_points, int32_t level, uint32_t* bits, wb_stream s);
/* coarse_bits: zero-initialised uint32 [(8^coarse_level + 31)/32]; a bit is set iff the coarse cell or one of its 26
 * neighbours contains an occupied level-`level` cell (coarse_level < level <= 10).  No reference counterpart: it is an
 * exact (conservative) accelerator for wb_raymarch_ray_count, results are identical with and without it. */
int wb_octree_build_coarse(const int16_t* level_points, int64_t num_points, int32_t level, int32_t coarse_level,
                           uint32_t* coarse_bits, wb_stream s);
/* OctreeAS.query (octree_as.py:146-163): out int32 [N] or [N, level+1] (with_parents). */
int wb_query(const wb_octree* oct, const float* coords, int64_t N, int32_t level, int32_t with_parents,
             int32_t* out, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * OctreeAS._raymarch_ray  (wisp/accelstructs/octree_as.py:247-309)
 *   count -> (caller scans counts into offsets, reads the total) -> fill.
 *   jitter: explicit [R, n] tensor (the reference's torch.rand draw) or NULL for the counter-based stream
 *   keyed by (seed, ray, step) (see DESIGN.md "Jitter contract").
 *   hitmask: uint32 [R, (n+31)/32] written by count and consumed by fill.
 * ---------------------------------------------------------------------------------------------- */
int wb_raymarch_ray_count(const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t num_samples,
                          const float* jitter, uint32_t seed, uint32_t* hitmask, int32_t* counts, wb_stream s);
/* exclusive scan of counts -> offsets (int64 [R+1], offsets[R] = total).  workspace >= wb_scan_workspace_bytes(R). */
int64_t wb_scan_workspace_bytes(int64_t R);
int wb_scan_counts(const int32_t* counts, int64_t R, int64_t* offsets, void* workspace, int64_t workspace_bytes, wb_stream s);
/* ASRaymarchResults layout (base_as.py:57-84): ridx i64[S], samples f32[S,3], depth f32[S,1], deltas f32[S,1],
 * boundary u8[S].  Any output pointer may be NULL. */
int wb_raymarch_ray_fill(const wb_rays* rays, int32_t num_samples, const float* jitter, uint32_t seed,
                         const uint32_t* hitmask, const int64_t* offsets,
                         int64_t* ridx, float* samples, float* depth, float* deltas, uint8_t* boundary, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * OctreeAS.raytrace (octree_as.py:165-186 -> kaolin unbatched_raytrace, with_exit=True) and the samplers built on it:
 * _raymarch_voxel (octree_as.py:188-245) and _raymarch_uniform (octree_as.py:311-374 + wisp._C.ops.uniform_sample_cuda,
 * wisp/csrc/ops/uniform_sample.cpp:28-42).  count -> wb_scan_counts -> fill.  Nuggets: ridx/pidx int32 [Ng], depth f32 [Ng,2]
 * (entry, exit), ordered by ray then front to back.  Sample outputs use the ASRaymarchResults layout; any output pointer may
 * be NULL; rec_ray (int32 ray index per sample) is the extra record the fused path needs.
 * ---------------------------------------------------------------------------------------------- */
int wb_raytrace_count(const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t* counts, wb_stream s);
int wb_raytrace_fill(const wb_octree* oct, int32_t level, const wb_rays* rays, const int64_t* offsets,
                     int32_t* ridx, int32_t* pidx, float* depth, wb_stream s);
/* The same pair with ONE octree traversal: the count pass keeps the first cache_k nuggets of every ray in `cache`
 * (wb_raytrace_cache_bytes(R, cache_k) bytes), the fill copies them and re-traverses only rays with more than cache_k nuggets. */
int64_t wb_raytrace_cache_bytes(int64_t R, int32_t cache_k);
int wb_raytrace_count_cached(const wb_octree* oct, int32_t level, const wb_rays* rays, int32_t* counts, void* cache, int32_t cache_k, wb_stream s);
int wb_raytrace_fill_cached(const wb_octree* oct, int32_t level, const wb_rays* rays, const int64_t* offsets, const void* cache, int32_t cache_k,
                            int32_t* ridx, int32_t* pidx, float* depth, wb_stream s);
/* num_samples per nugget; jitter: explicit [Ng, num_samples] or NULL for the counter stream keyed by (seed, nugget, k). */
int wb_raymarch_voxel_fill(const wb_rays* rays, const int32_t* nug_ridx, const float* nug_depth, int64_t Ng, int32_t num_samples,
                           const float* jitter, uint32_t seed, int64_t* ridx, float* samples, float* depth, float* deltas,
                           uint8_t* boundary, int32_t* rec_ray, wb_stream s);
/* scale = ceil(1 / (2*sqrt(3)/num_samples)) (octree_as.py:336-338), computed by the caller. */
int wb_raymarch_uniform_count(const float* nug_depth, int64_t Ng, int32_t scale, int32_t* cnt, wb_stream s);
/* sample_offsets int64 [Ng+1] = scan of cnt; ray_nugget_offsets int64 [R+1] = scan of the raytrace counts. */
int wb_raymarch_uniform_fill(const wb_rays* rays, const int32_t* nug_ridx, const float* nug_depth, int64_t Ng, int32_t scale,
                             const int64_t* sample_offsets, const int64_t* ray_nugget_offsets,
                             int64_t* ridx, float* samples, float* depth, float* deltas, uint8_t* boundary, int32_t* rec_ray, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * HashGrid.interpolate kernels -- replace wisp._C.ops.hashgrid_interpolate_cuda / _backward_cuda
 *   (wisp/csrc/ops/hashgrid_interpolate.h:18-33, hashgrid_interpolate.cpp:46-105): all LODs in ONE launch.
 *   feats/grad_feats: [N, L*F] raw kernel output (the 'cat' zeroing / 'sum' reduction of hash_grid.py:224-233
 *   is applied by the host shim, as in the reference).  grad_table must be zero-initialised (cpp:85).
 * ---------------------------------------------------------------------------------------------- */
int wb_hashgrid_fwd(const float* coords, int64_t N, const wb_nef_desc* grid, float* feats, wb_stream s);
int wb_hashgrid_bwd(const float* coords, int64_t N, const wb_nef_desc* grid, const float* grad_feats,
                    float* grad_table, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * TriplanarGrid.interpolate (wisp/models/grids/triplanar_grid.py:98-143, 205-223): replaces 3 F.grid_sample launches per LOD
 * (align_corners=True, padding_mode='reflection') plus the stack/permute/cat copies.  res[l] = 2^(log_base_resolution + l);
 * planes: HOST array of 3*num_lods device pointers (fmx, fmy, fmz of LOD 0, then LOD 1, ...), each [1, fdim, res+1, res+1];
 * feats / grad_feats: [N, num_lods, 3, fdim] (the reference's cat layout; 'sum' is applied by the caller);
 * grad_planes: same shapes as planes, accumulated into (caller zeroes).
 * ---------------------------------------------------------------------------------------------- */
int wb_triplane_fwd(const float* coords, int64_t N, int32_t num_lods, int32_t fdim, const int32_t* res,
                    const float* const* planes, float* feats, wb_stream s);
int wb_triplane_bwd(const float* coords, int64_t N, int32_t num_lods, int32_t fdim, const int32_t* res,
                    const float* const* planes, const float* grad_feats, float* const* grad_planes, wb_stream s);
/* Plane layout conversion for the fused path (wb_nef_desc.grid_layout = 1), all planes in ONE launch: src / dst are HOST arrays of
 * n_planes device pointers, sizes[i] = plane side (res + 1).  to_channel_last != 0: [fdim, size, size] -> [size, size, fdim];
 * 0: the inverse (gradients back into the layout of the reference's nn.Parameter, triplanar_grid.py:178-180).  dst is overwritten. */
int wb_triplane_relayout(const float* const* src, float* const* dst, const int32_t* sizes, int32_t n_planes, int32_t fdim,
                         int32_t to_channel_last, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * OctreeGrid.interpolate (wisp/models/grids/octree_grid.py:130-219): replaces blas.query(with_parents=True) + one
 * kaolin unbatched_interpolate_trilinear launch per LOD + cat/sum.  points int16 [T,3] and trinkets int32 [T,8] are the
 * tensors the reference keeps (blas.points, grid.trinkets: LEVEL-LOCAL corner-feature indices); feats: HOST array of
 * num_lods_used device pointers (grid.features[0..lod_idx], each [pyramid_dual[0,l]+1, feature_dim] fp32).
 * out: [N, num_lods_used*feature_dim] ('cat', multiscale 0) or [N, feature_dim] ('sum', multiscale 1).
 * half_round != 0 reproduces the call site's feats.half() ... .float() rounding (octree_grid.py:147-149).
 * Backward accumulates into grad_feats (caller zeroes); no gradient flows to coords (as in Kaolin).
 * ---------------------------------------------------------------------------------------------- */
int wb_octree_interp_fwd(const wb_octree* oct, const int16_t* points, const int32_t* trinkets, const float* coords, int64_t N,
                         int32_t feature_dim, int32_t base_lod, int32_t num_lods_used, int32_t multiscale, int32_t half_round,
                         const float* const* feats, float* out, wb_stream s);
int wb_octree_interp_bwd(const wb_octree* oct, const int16_t* points, const int32_t* trinkets, const float* coords, int64_t N,
                         int32_t feature_dim, int32_t base_lod, int32_t num_lods_used, int32_t multiscale,
                         const float* const* feats, const float* grad_out, float* const* grad_feats, wb_stream s);
/* wisp._C.render.find_depth_bound_cuda(query f32[P,1], curr_idxes i32[P], depth f32[Ng,2]) -> i32[P]
 * (wisp/csrc/render/find_depth_bound.cpp:23-36, kernel find_depth_bound_cuda.cu:16-45), launched on the given stream. */
int wb_find_depth_bound(const float* query, const int32_t* curr_idxes, const float* depth, int64_t num_packs, int64_t num_nugs,
                        int32_t* out, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * NeuralSDF(OctreeGrid) and the sphere tracer of app/nglod (BASELINE config 3)
 *   wb_sdf_eval  replaces NeuralSDF.sdf (wisp/models/nefs/neural_sdf.py:120-155): OctreeGrid.interpolate
 *                (octree_grid.py:130-219) or HashGrid.interpolate (hash_grid.py:205-233, wb_sdf_desc.hash) + position
 *                embedding + BasicDecoder, one launch, fp32 decoder.  Octree 'cat' grids: lod_idx = num_lods-1 only; hash grids:
 *                any lod_idx.
 *   wb_sdf_trace replaces the whole loop of PackedSDFTracer.trace (wisp/tracers/packed_sdf_tracer.py:78-174) including
 *                wisp._C.render.find_depth_bound_cuda (find_depth_bound_cuda.cu:16-45) and finitediff_gradient
 *                (wisp/ops/differential/gradients.py:29-45): ONE persistent cooperative kernel.  Input: the nuggets of
 *                wb_raytrace_fill at level base_lod + lod_idx (raw depths: the kernel adds the reference's 1e-5 to the
 *                entries itself) and the per-ray nugget offsets of wb_scan_counts.  Outputs are per ray; the caller
 *                initialises them (zeros; rgb = 0.5 when want_normals, packed_sdf_tracer.py:168) and the kernel
 *                writes the rays that hit: xyz [R,3], depth [R], hit u8 [R], normal [R,3], rgb [R,3], alpha [R].
 * ---------------------------------------------------------------------------------------------- */
typedef struct wb_sdf_desc {
    /* OctreeGrid (octree_grid.py:58-104): level-local trinkets, one feature tensor per active LOD */
    const int16_t* points;                  /* blas.points int16 [T,3]                               */
    const int32_t* trinkets;                /* grid.trinkets int32 [T,8]                             */
    const float* const* feats;              /* HOST array of num_lods device pointers [rows_l, F] f32 */
    int32_t feature_dim, base_lod, num_lods;
    int32_t multiscale;                     /* 0 'cat', 1 'sum'                                      */
    int32_t half_round;                     /* feats.half() ... .float() of the call site (:147-149) */
    /* NeuralSDF (neural_sdf.py:30-99): position embedding FIRST, then grid features                   */
    int32_t pos_mode, pos_freq;             /* 0 none, 1 identity, 2 positional, 3 positional+input  */
    int32_t num_layers, hidden_dim;         /* BasicDecoder(bias=True): num_layers hidden layers, relu, 1 output */
    const float* params;                    /* packed [W0, b0, ..., Wout, bout], nn.Linear layout      */
    const wb_nef_desc* hash;  /* non-null: NeuralSDF(HashGrid); only the hash-grid fields are read; points/trinkets/feats/half_round unused */
} wb_sdf_desc;
/* A hash field (hash != NULL, HashGrid.interpolate, hash_grid.py:205-233): hash->feature_dim 4 or 8, 'cat' or 'sum', 3D; the
 * table is codebook.feats [rows, F] fp32 (16-byte aligned), LOD l at rows begin_idxes[l] ..; feature_dim, num_lods and multiscale
 * must equal the hash description's, base_lod is 0, and oct may be NULL.  'cat' features are L*F wide whatever lod_idx: the LODs
 * >= lod_idx are zero (the reference's in-place write); 'sum' adds all L LODs whatever lod_idx.  No occupancy test: coordinates
 * are clamped into each level's cells.  The table is read in fp32 (the reference's enable_amp fp16 table is not reproduced). */
int wb_sdf_eval(const wb_octree* oct, const wb_sdf_desc* nef, int32_t lod_idx, const float* coords, int64_t N, float* sdf, wb_stream s);
/* wb_sdf_train: one training launch of SDFTrainer.step (wisp/trainers/sdf_trainer.py:65-124) for the loss LOD lod_idx, over
 * NeuralSDF.sdf (wisp/models/nefs/neural_sdf.py:120-155): forward as wb_sdf_eval, loss and backward in the same kernel.
 *   coords f32 [N,3], sdf_gt f32 [N]; decoders with 1 to 4 hidden layers whose training footprint fits in shared memory
 *   (wb_sdf_train_smem_bytes(nef) >= 0; otherwise the call fails).
 *   *loss_out     += sum_i (y_i - gt_i)^2 * inv_count               (inv_count = 1 / batch size: `loss /= batch_size`)
 *   grad_params   += dL/d params, packed like nef->params [W0, b0, W1, b1, ..., Wout, bout] (nn.Linear layout: W_k [H, in])
 *   grad_feats[k] += dL/d feats[k] for k = 0 .. lod_idx (HOST array of device pointers, shapes of nef->feats), fp32, as
 *                    wb_octree_interp_bwd: no gradient to the coordinates, the fp16 rounding of the forward passed straight through.
 *   hash field:   grad_feats[0] += dL/d codebook.feats [rows, F] (16-byte aligned), fp32, as wb_hashgrid_bwd; the zeroed 'cat'
 *                    LODs receive nothing.
 * Everything accumulates: the caller zeroes loss_out and the gradients; a loss over several LODs is one call per LOD. */
int wb_sdf_train(const wb_octree* oct, const wb_sdf_desc* nef, int32_t lod_idx, const float* coords, const float* sdf_gt, int64_t N,
                 float inv_count, float* const* grad_feats, float* grad_params, float* loss_out, wb_stream s);
/* Dynamic shared memory (bytes) of a wb_sdf_train launch for this field, or < 0 when wb_sdf_train cannot train it (a description
 * wb_sdf_eval refuses, or a decoder with more than one hidden layer whose weights, weight-gradient accumulators and a 32-sample
 * tile exceed 227 KB).  Host only: no device is touched. */
int64_t wb_sdf_train_smem_bytes(const wb_sdf_desc* nef);
/* wb_sdf_train_tc: wb_sdf_train with the reference's enable_amp arithmetic (torch.cuda.amp.autocast around SDFTrainer.step,
 * wisp/trainers/base_trainer.py:338; sdf_trainer.py:65-124) on the tensor cores: every decoder nn.Linear takes fp16 inputs, weights
 * and biases, accumulates in fp32 and rounds its output (the prediction included) to fp16; the loss is fp32.  Same arguments and
 * accumulate-into semantics as wb_sdf_train, gradients in fp32.  Deviations: the hash table is read in fp32, the output gradient
 * carries a power-of-two loss scale (removed exactly in fp32), weight gradients accumulate in fp32 over the batch.  Decoders with
 * 1 to 4 hidden layers whose footprint fits (wb_sdf_train_tc_smem_bytes(nef) >= 0; otherwise the call fails). */
int wb_sdf_train_tc(const wb_octree* oct, const wb_sdf_desc* nef, int32_t lod_idx, const float* coords, const float* sdf_gt, int64_t N,
                    float inv_count, float* const* grad_feats, float* grad_params, float* loss_out, wb_stream s);
/* Dynamic shared memory (bytes) of a wb_sdf_train_tc launch: fp16 weight packs, fp32 weight-gradient accumulators and one 64-sample
 * tile; < 0 when that exceeds 227 KB or wb_sdf_eval refuses the description.  Host only. */
int64_t wb_sdf_train_tc_smem_bytes(const wb_sdf_desc* nef);
/* Per-pack state of the sphere tracer (pack = ray with >= 1 nugget).  All device pointers, allocated by the caller for R rays;
 * nothing needs initialising.  state bit 0 = alive (the reference's `mask`), bit 1 = hit. */
typedef struct wb_sdf_state {
    int32_t* flags;                         /* [R]    ray has nuggets                                  */
    int64_t* pack_off;                      /* [R+1]  exclusive scan of flags; pack_off[R] = #packs    */
    void* scan_ws; int64_t scan_ws_bytes;   /* wb_scan_workspace_bytes(R)                              */
    int32_t* pack_ray;                      /* [R]    ray of pack p                                    */
    float* t; float* dist; float* dist_prev;/* [R]    depth along the ray, last / previous sdf step    */
    float* x;                               /* [R,3]  current point                                    */
    int32_t* cursor0; int32_t* cursor1;     /* [R]    nugget cursor, double buffered                   */
    uint8_t* state;                         /* [R]                                                     */
    int32_t* iterflags;                     /* [2*num_steps+4] any-pack-alive flags of every iteration; [2*num_steps+2] = field evaluations of wb_sdf_trace */
} wb_sdf_state;
int wb_sdf_trace(const wb_octree* oct, const wb_sdf_desc* nef, int32_t lod_idx, const wb_rays* rays,
                 const float* nug_depth, int64_t Ng, const int64_t* ray_offsets,
                 int32_t num_steps, float step_size, double min_dis, int32_t want_normals, const wb_sdf_state* state,
                 float* xyz, float* depth, uint8_t* hit, float* normal, float* rgb, float* alpha, wb_stream s);
/* wb_sdf_trace takes octree fields only: a hash description returns WB_ERR_INVALID before anything is launched.
 * The same state machine one phase per launch, for fields wb_sdf_trace does not trace (NeuralSDF over a hash grid,
 * app/nglod/configs/nglod_hash.yaml, whose field the caller evaluates with wb_sdf_eval; or over a triplanar grid, evaluated outside
 * this library): the caller evaluates its field at state->x of the alive packs and writes state->dist between the phases.  phase 0: pack list (then read pack_off[R])  1: initial t, x, cursor, alive   2: step 1 of
 * iteration `iteration` (packed_sdf_tracer.py:120-131)   3: step 2 (:133-141)   4: outputs of the packs that hit.
 * iterflags[2*iteration + (phase == 3)] != 0 afterwards iff a pack is still alive (the loop's `break` tests). */
int wb_sdf_phase(int32_t phase, const wb_rays* rays, const float* nug_depth, int64_t Ng, const int64_t* ray_offsets,
                 int32_t num_steps, int32_t iteration, double min_dis, const wb_sdf_state* state,
                 float* xyz, float* depth, uint8_t* hit, float* alpha, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Packed compositing -- replaces kaolin.render.spc.{exponential_integration, sum_reduce} + the buffer
 *   scatter of PackedRFTracer.trace (wisp/tracers/packed_rf_tracer.py:136-165).
 *   shaded: float4 [S] = (r, g, b, sigma); offsets int64 [R+1]; depth/deltas [S].
 *   bg: HOST pointer to 3 floats (tracer.bg_color; a launch parameter, not a tensor).
 *   outputs: rgb [R,3], depth_out [R] (may be NULL), alpha [R], hit u8[R].
 * ---------------------------------------------------------------------------------------------- */
int wb_composite_fwd(const float* shaded, const float* depth, const float* deltas, const int64_t* offsets, int64_t R,
                     const float* bg, float* rgb, float* depth_out, float* alpha, uint8_t* hit, wb_stream s);
/* g_shaded float4 [S] = dL/d(r,g,b,sigma).  g_depth / g_alpha may be NULL.
 * absmax (may be NULL): device float, zero-initialised by the caller; receives max |g_shaded| (atomic max), from which the
 * caller derives the power-of-two loss scale of the fp16 decoder backward without another pass over g_shaded. */
int wb_composite_bwd(const float* shaded, const float* depth, const float* deltas, const int64_t* offsets, int64_t R,
                     const float* bg, const float* g_rgb, const float* g_depth, const float* g_alpha,
                     float* g_shaded, float* absmax, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Fused render path -- replaces PackedRFTracer.trace + NeuralRadianceField.rgba + HashGrid.interpolate
 *   (wisp/tracers/packed_rf_tracer.py:84-181, wisp/models/nefs/nerf.py:219-264).
 *   1. wb_raymarch_ray_count + wb_scan_counts            (sample culling, bit-exact with the reference)
 *   2. wb_rf_march_fill   : compact sample records (t, delta, ray) -- 12 B/sample instead of 29 B
 *   3. wb_rf_shade_fwd    : gather + decoders fused, one pass, (r,g,b,sigma) per sample
 *   4. wb_composite_fwd
 *   backward: wb_composite_bwd -> wb_rf_shade_bwd (recomputes the decoders, scatters table gradients).
 *   precision: 0 = fp32 SIMT decoders (reference autocast-off numerics),
 *              1 = fp16 tensor-core decoders with fp32 accumulation (reference autocast-on numerics).
 * ---------------------------------------------------------------------------------------------- */
int wb_rf_march_fill(const wb_rays* rays, int32_t num_samples, const float* jitter, uint32_t seed,
                     const uint32_t* hitmask, const int64_t* offsets,
                     float* rec_t, float* rec_delta, int32_t* rec_ray, wb_stream s);
/* Packs decoder parameters into the shared-memory image the shade kernels stage with one bulk (TMA) copy.
 * blob: float [wb_rf_param_blob_floats(nef)]. */
int64_t wb_rf_param_blob_floats(const wb_nef_desc* nef, int32_t precision);
/* 1 if the decoder configuration can run at `precision` (forward only, or forward + backward), else 0 with the reason in
 * wb_last_error().  precision 0 always can; precision 1 needs layers at most 128 wide and, for the backward, a decoder whose
 * activation tiles and weight-gradient accumulators fit in shared memory (decoders with up to one hidden density and two hidden
 * colour layers may split the accumulators over several passes).  Host-side query, no device work. */
int wb_rf_precision_supported(const wb_nef_desc* nef, int32_t precision, int32_t backward);
/* *shaped = 1 when the precision-1 forward (backward == 0), or the decoder backward with the fused hash-table scatter
 * (backward == 1), of this decoder runs a kernel instance compiled for its layer widths (the app/nerf 64-wide decoders), 0 when it
 * runs the instance that reads the widths at run time.  Host-side query, no device work. */
int wb_rf_tc_shaped(const wb_nef_desc* nef, int32_t backward, int32_t* shaped);
int wb_rf_pack_params(const wb_nef_desc* nef, int32_t precision, float* blob, wb_stream s);
/* precision 1 scratch: workspace = per-ray view-embedding rows (+ dL/dfeat planes when backward != 0);
 * feat = the gathered grid features the forward saves for the backward (2*Kp0 bytes per sample).  Both 0 for precision 0. */
int64_t wb_rf_workspace_bytes(const wb_nef_desc* nef, int32_t precision, int64_t R, int64_t S, int32_t backward);
int64_t wb_rf_feat_bytes(const wb_nef_desc* nef, int32_t precision, int64_t S);
/* feat_save: optional (NULL = inference, nothing saved); workspace: wb_rf_workspace_bytes(.., backward=0) bytes. */
int wb_rf_shade_fwd(const wb_nef_desc* nef, const float* blob, int32_t precision, const wb_rays* rays,
                    const float* rec_t, const int32_t* rec_ray, int64_t S, float* shaded, void* feat_save, void* workspace, wb_stream s);
/* grad_table [rows,F], grad_dens / grad_col (packed like the params) are ACCUMULATED into (caller zeroes).
 * loss_scale: device pointer to ONE float, a power of two by which precision 1 scales the incoming gradients while
 * they are carried in fp16 (unscaled again in fp32 before they leave the kernels); ignored (may be NULL) for precision 0.
 * feat_saved: what the forward wrote to feat_save; workspace: wb_rf_workspace_bytes(.., backward=1) bytes. */
int wb_rf_shade_bwd(const wb_nef_desc* nef, const float* blob, int32_t precision, const wb_rays* rays,
                    const float* rec_t, const int32_t* rec_ray, int64_t S, const float* g_shaded, const float* loss_scale,
                    const void* feat_saved, void* workspace,
                    float* grad_table, float* grad_dens, float* grad_col, wb_stream s);

/* Precision 1: wb_rf_shade_fwd writes the per-ray colour-input rows (view embedding) at the start of its workspace; a caller that hands
 * the SAME workspace (sized with backward = 1) and the same rays to the backward can say so right before that call and save the
 * launch that would rebuild them.  Applies to the next wb_rf_shade_bwd / wb_rf_decoder_bwd of the calling thread only, whatever
 * that call returns (also with S == 0, precision 0 or an argument error). */
int wb_rf_workspace_holds_ray_rows(int32_t yes);

/* scale = 2^clamp(floor(log2(64 / max(absmax, 1e-30))), -20, 60): the loss scale wb_rf_decoder_bwd / wb_rf_table_scatter expect,
 * derived on the device from wb_composite_bwd's absmax. */
int wb_rf_loss_scale(const float* absmax, float* scale, wb_stream s);

/* The two stages of the precision-1 backward, callable separately (wb_rf_shade_bwd runs them back to back):
 * wb_rf_decoder_bwd writes the weight gradients and leaves dL/dfeat (fp16 planes) in the workspace; wb_rf_table_scatter
 * turns those planes into hash-table updates with warp-level merging of samples that share a cell.
 * Workspace layout (bytes), R rays, S samples, Kc = width of the colour-decoder input rounded up to 16:
 *   [0, R * Kc * 2)                     per-ray colour-input rows, fp16 [R][Kc] (view embedding at features dout-1 .., zeros)
 *   [align256(R * Kc * 2), + P * S * F * 2)  dL/dfeat, fp16 [P][S][F], still multiplied by the loss scale; F = feature_dim,
 *                                       P = one plane per live LOD ('cat': min(lod_idx, num_lods)) or 1 ('sum').
 * feat_saved (wb_rf_shade_fwd's feat_save): the density-decoder input rows, fp16, chunk-major [Kp0 / 8][S] x 8 features
 *   (Kp0 = its width rounded up to 16): grid features, then the position embedding, then zeros. */
int wb_rf_decoder_bwd(const wb_nef_desc* nef, const float* blob, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray,
                      int64_t S, const float* g_shaded, const float* loss_scale, const void* feat_saved, void* workspace,
                      float* grad_dens, float* grad_col, wb_stream s);
int wb_rf_table_scatter(const wb_nef_desc* nef, const wb_rays* rays, const float* rec_t, const int32_t* rec_ray, int64_t S,
                        const float* loss_scale, void* workspace, float* grad_table, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * CodebookOctreeGrid (VQAD; wisp/models/grids/codebook_grid.py:103-172), row-wise: the softmax / straight-through selection of a
 * dictionary entry depends only on the corner row, so it runs once per row and LOD instead of once per (sample, corner):
 *   wb_codebook_rows_fwd : E[row] = sum_k keys[row,k] * dictionary[k]; training != 0: keys = (y_hard - y_soft) + y_soft (:117-123),
 *                          else one_hot(argmax) (:128-131).  logits [rows, K], dictionary [K, F], E [rows, F]; argmax_out optional.
 *   wb_codebook_rows_bwd : from dE [rows, F] (what wb_octree_interp_bwd accumulated): g_dictionary [K, F] accumulated into,
 *                          g_logits [rows, K] written for rows with a non-zero dE (caller zeroes both).
 * The per-sample blend is wb_octree_interp_fwd / _bwd over E (half_round = 0: the codebook grid blends in fp32, :164-165).
 * ---------------------------------------------------------------------------------------------- */
int wb_codebook_rows_fwd(const float* logits, const float* dictionary, int64_t rows, int32_t K, int32_t F, int32_t training,
                         float* E, int32_t* argmax_out, wb_stream s);
int wb_codebook_rows_bwd(const float* logits, const float* dictionary, const float* dE, int64_t rows, int32_t K, int32_t F,
                         float* g_logits, float* g_dictionary, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Trainer step glue (SURVEY.md 8(f) rank 2): MultiviewTrainer.step (wisp/trainers/multiview_trainer.py:111-180) and
 * BaseTrainer.init_optimizer (wisp/trainers/base_trainer.py:205-235).
 *   wb_composite_bwd_loss : wb_composite_bwd with the image loss and its gradient evaluated inside: rgb_pred = wb_composite_fwd's
 *       rgb, target = ground truth [R,3]; loss_type 0 = l2 (mse_loss), 1 = l1, 2 = huber (smooth_l1_loss), reduction =
 *       sum * inv_count; *loss_out (device float, zeroed by the caller) receives the loss value.
 *   wb_adam_step : torch.optim.Adam (amsgrad off) over up to 64 tensors in one launch; per-segment lr and weight decay carry the
 *       reference's parameter groups; grad_scale multiplies every gradient first (1/world after an all-reduce(sum)); zero_grad != 0
 *       clears each gradient as it is consumed.  The step's description (segments, bias corrections, scales) is passed to the
 *       kernel by value, so segs may be reused as soon as the call returns, however far the host runs ahead of the stream.
 *   wb_adamw_step : torch.optim.AdamW (amsgrad off; what apex FusedAdam computes by default) with wb_adam_step's contract and
 *       segments: p *= 1 - lr * weight_decay (the factor formed in double, one fp32 multiply), then Adam's moments and update
 *       without the L2 term.
 *   wb_rmsprop_step : torch.optim.RMSprop (centered off) with wb_adam_step's contract: g = grad * grad_scale (+ weight_decay * p);
 *       square_avg = alpha * square_avg + (1 - alpha) g^2; q = g / (sqrt(square_avg) + eps); momentum == 0: p -= lr * q, and
 *       momentum_buffer is neither read nor written (it may be null); momentum > 0: buf = momentum * buf + q, p -= lr * buf.
 *   Roundings of the two (ours, not torch's, which runs one kernel per operation): every product, quotient and square root is
 *   rounded once; the moment updates and the final parameter update are single fused multiply-adds (b * state + fl(..),
 *   p - lr * q); wb_optim.cu lists the chains.  fp32 parameters and state.
 * ---------------------------------------------------------------------------------------------- */
int wb_composite_bwd_loss(const float* shaded, const float* depth, const float* deltas, const int64_t* offsets, int64_t R,
                          const float* bg, const float* rgb_pred, const float* target, int32_t loss_type, float inv_count,
                          float* g_shaded, float* absmax, float* loss_out, wb_stream s);
typedef struct wb_adam_segment {
    float* param; float* grad; float* exp_avg; float* exp_avg_sq;
    int64_t numel;
    float lr, weight_decay;
} wb_adam_segment;
int wb_adam_step(const wb_adam_segment* segs, int32_t nseg, float beta1, float beta2, float eps, int32_t step, float grad_scale,
                 int32_t zero_grad, wb_stream s);
int wb_adamw_step(const wb_adam_segment* segs, int32_t nseg, float beta1, float beta2, float eps, int32_t step, float grad_scale,
                  int32_t zero_grad, wb_stream s);
typedef struct wb_rmsprop_segment {
    float* param; float* grad; float* square_avg; float* momentum_buffer;      /* momentum_buffer: null when momentum == 0 */
    int64_t numel;
    float lr, weight_decay;
} wb_rmsprop_segment;
int wb_rmsprop_step(const wb_rmsprop_segment* segs, int32_t nseg, float alpha, float eps, float momentum, float grad_scale,
                    int32_t zero_grad, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Ray generation (camera -> rays on the device); origin/view/right/up/cam_pos/rotation are HOST pointers (launch parameters).
 *   wb_raygen_lookat  : _look_at + _generate_rays (wisp/trainers/tracker/offline_renderer.py:23-89) over normalized_grid
 *                       (wisp/ops/geometric.py:65-99, use_aspect=True, no jitter); view/right/up are the normalised camera frame
 *                       the reference derives from (from, to); ortho != 0 selects mode='ortho'.  origins / dirs: [H*W, 3].
 *   wb_raygen_pinhole : generate_pinhole_rays (wisp/ops/raygen/raygen.py:40-85) with the pixel grid of
 *                       generate_centered_pixel_coords (:24-31); the Kaolin camera is passed as numbers: position, camera-to-world
 *                       rotation (row-major 3x3), principal point x0/y0, tan(fov/2) per axis, image size, ray-grid size.
 * ---------------------------------------------------------------------------------------------- */
int wb_raygen_lookat(const float* origin, const float* view, const float* right, const float* up, float tan_half_fov,
                     int32_t height, int32_t width, int32_t ortho, float* origins, float* dirs, wb_stream s);
int wb_raygen_pinhole(const float* cam_pos, const float* cam_to_world_rot, float x0, float y0, float tan_half_fov_h, float tan_half_fov_v,
                      int32_t img_height, int32_t img_width, int32_t res_y, int32_t res_x, float* origins, float* dirs, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * NeuralRadianceField.prune (wisp/models/nefs/nerf.py:175-212), the elementwise halves around the density probe:
 *   wb_prune_samples : one probe point per finest-level cell, samples = ((points + u) / 2^level) * 2 - 1 (:189-192) and a unit
 *                      direction; u = explicit [N,3] draw, or NULL for the counter stream keyed by (seed, cell, axis).  Also writes
 *                      rec_t = 0 and rec_ray = i so that wb_rf_shade_fwd evaluates the field at the probe points (rays of length 0).
 *   wb_prune_update  : occupancy = max(sigma, occupancy * decay) (:186,:196); keep = occupancy > min_density (:198);
 *                      shaded = float4 [N] written by wb_rf_shade_fwd (sigma in .w).
 * ---------------------------------------------------------------------------------------------- */
int wb_prune_samples(const int16_t* points, int64_t N, int32_t level, const float* u, uint32_t seed,
                     float* samples, float* dirs, float* rec_t, int32_t* rec_ray, wb_stream s);
int wb_prune_update(const float* shaded, int64_t N, float decay, float min_density, float* occupancy, uint8_t* keep, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * Diagnostics: one-tile wgmma GEMM that pins the shared-memory operand layouts of the tensor-core decoder
 * kernels (csrc/wb_tc.cuh).  a_img / b_img are byte images of the operand tiles (R = 128 sample rows, or 64 -- the
 * decoder kernels' tile -- when mode has bit 4 set); D is fp32, [R, N] for modes 0 / 1 and [128, N] for mode 2.
 * mode 0: D = A[RxK] . W[NxK]^T   mode 1: D = A[RxK] . W[KxN]   mode 2: D = A[Rx128]^T . B[RxN]
 * N = 8 or a multiple of 16 up to 128.
 * ---------------------------------------------------------------------------------------------- */
int wb_tc_selftest(const void* a_img, int a_bytes, const void* b_img, int b_bytes, float* D, int N, int K, int mode, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * HashGrid.interpolate over [N, 2] coordinates (app/image): wb_hashgrid_fwd / _bwd's contract and layouts, with the reference's 2-D
 * kernels (hashgrid_interpolate_2d_cuda_kernel and its backward, hashgrid_interpolate_cuda.cu:214-339, hash_index_2d in
 * hash_utils.cuh:65-84; the reference picks them from coords.size(1), :374): 4 corners per LOD, dense rows x + y*res
 * when res < T and res^2 < T, hashed rows (x ^ y*2654435761) & (T-1) otherwise.  Only the hash fields of `grid` are read.  Rows are
 * level-local from begin_idxes, so tables of min(res^3, T) rows per level (coord_dim = 3, what image_hash.yaml builds) and of
 * min(res^2, T) rows (coord_dim = 2) both work.  Deviation: on a dense level's last cell (res >= 258, coordinate +1) the weight-0 +1
 * corner keeps the cell's own row instead of the reference's row past the level.  No gradient to the coordinates. */
int wb_hashgrid2d_fwd(const float* coords, int64_t N, const wb_nef_desc* grid, float* feats, wb_stream s);
int wb_hashgrid2d_bwd(const float* coords, int64_t N, const wb_nef_desc* grid, const float* grad_feats,
                      float* grad_table, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * ImageNeuralField (wisp/models/nefs/image_nef.py:37-97) of app/image over a 2-D HashGrid, fp32 SIMT, one launch each:
 *   wb_image_eval  replaces ImageNeuralField.rgb: sigmoid(decoder(cat([HashGrid.interpolate(coords, lod_idx), embed(coords)]))),
 *                  embed = get_positional_embedder(3, include_input=True) on [N, 2]: [x, y, sin(x 2^k, y 2^k)_k, cos(...)_k], 14 wide.
 *                  'cat': features of LODs >= lod_idx are zero (hash_grid.py:228); 'sum' adds all LODs.  rgb f32 [N, 3].
 *   wb_image_train one ImageTrainer.step (wisp/trainers/image_trainer.py:51-80) without the optimiser: the forward of wb_image_eval,
 *                  F.mse_loss over [N, 3] and the backward.  Accumulates (the caller zeroes): *loss_out += sum (y - gt)^2 * inv_count
 *                  (inv_count = 1 / (3N): the mean), grad_table [rows, F] += dL/d codebook.feats (the zeroed 'cat' LODs get nothing),
 *                  grad_params += dL/d params.
 * grid: hash fields of a wb_nef_desc, feature_dim 2, 4 or 8, table 8-byte (F = 2) or 16-byte aligned, grad_table aligned alike.
 * Decoder: BasicDecoder(in, 3, relu, bias=True, num_layers=1, hidden_dim) with in = (L*F 'cat' | F 'sum') + 14 and hidden_dim a
 * multiple of 4 up to 128; params: HOST array of 4 device pointers W0 [H, in], b0 [H], Wout [3, H], bout [3] (nn.Linear layout);
 * grad_params packed [W0, b0, Wout, bout] in that order.  N >= 1.
 * Deviations: the table is read in fp32 (no enable_amp fp16 copy); embedder.bands is not trained (requires_grad=False in the
 * reference too) and is taken as 2^0, 2^1, 2^2. */
int wb_image_eval(const wb_nef_desc* grid, int32_t hidden_dim, const float* const* params, int32_t lod_idx, const float* coords,
                  int64_t N, float* rgb, wb_stream s);
int wb_image_train(const wb_nef_desc* grid, int32_t hidden_dim, const float* const* params, int32_t lod_idx, const float* coords,
                   const float* rgb_gt, int64_t N, float inv_count, float* grad_table, float* grad_params, float* loss_out, wb_stream s);
/* Dynamic shared memory (bytes) of a wb_image_eval (train = 0) or wb_image_train (train != 0) launch for this field, or < 0 when the
 * kernel does not take it (the reason in wb_last_error()).  Host only: no device is touched. */
int64_t wb_image_smem_bytes(const wb_nef_desc* grid, int32_t hidden_dim, int32_t train);

/* ------------------------------------------------------------------------------------------------
 * PackedSPCTracer.trace (wisp/tracers/packed_spc_tracer.py:50-90) over SPCField: the first nugget of every ray at `level`
 * (the nugget of wb_raytrace_fill: the cell of `level` whose slab interval is first in front of the origin), in ONE launch.
 * A hit writes depth[r] = its entry depth (the first depth[2 * offsets[r]] of wb_raytrace_fill), hit[r] = 1,
 * rgb[3r..3r+2] = colors[(pidx - point_offset) * color_stride + 0..2] (pidx: the cell's point index) and alpha[r] = 1;
 * a miss writes 0 to all four.  colors: f32, color_stride >= 3; the caller keeps pidx - point_offset inside the colour rows
 * (SPCField: point_offset = pyramid[1, max_level] and level = max_level).  depth / alpha f32 [R], hit uint8 [R], rgb f32 [R, 3].
 * level <= 15 and <= oct->max_level.  R = 0 launches nothing. */
int wb_spc_trace(const wb_octree* oct, int32_t level, const wb_rays* rays, const float* colors, int64_t color_stride, int64_t point_offset,
                 float* depth, uint8_t* hit, float* rgb, float* alpha, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * wisp.ops.mesh.compute_sdf (wisp/ops/mesh/compute_sdf.py; kernel wisp/csrc/external/mesh2sdf_kernel.cu:334-584, 844-903):
 * out[i] = the signed distance from points[i] to the triangle soup tris, with the reference's arithmetic and sign rule:
 * fp64 per pair except its fp32 roundings (idot2 = __frcp_rn, copysignf, the fminf-clamped edge parameter, the fminf minima),
 * sqrtf of the fp32 minimum, negated when all 13 stab directions have a hit with t >= 0 and one with t < 0 (|det| < 1e-8 skipped);
 * +inf when no triangle has a nonzero normal, and for a point with a NaN coordinate.
 * A bounding-volume hierarchy (LBVH over centroid Morton codes) is built per call in `workspace` and culls, conservatively,
 * the pairs that cannot set the fp32 minimum or a stab flag; the result is the reference's, not an approximation of it.
 * tris: f64 [T, 9] (V[F] row-major), points: f64 [N, 3], out: f64 [N].  T <= 2^29; T = 0 gives +inf.  N = 0 launches nothing.
 * Launches (wb_launch_count): 6 for T >= 2 (the CUB radix sort counted as one), 5 for T = 1, 1 for T = 0. */
/* Workspace bytes of a wb_mesh_sdf call over num_triangles triangles (any number of points); < 0 on a bad count or, for T >= 1, when
 * the radix sort's size query of the current device fails (reason in wb_last_error()).  Launches nothing. */
int64_t wb_mesh_sdf_workspace_bytes(int64_t num_triangles);
int wb_mesh_sdf(const double* tris, int64_t num_triangles, const double* points, int64_t num_points, void* workspace,
                int64_t workspace_bytes, double* out, wb_stream s);

/* ------------------------------------------------------------------------------------------------
 * wisp.ops.spc.mesh_to_octree (wisp/ops/spc/conversions.py:91-109; sampler wisp/ops/mesh/sample_surface.py): the occupancy of
 * num_samples area-weighted surface samples and their jittered copies at `level`, in ONE launch, no sample materialised.
 * Sample i (a 64-bit counter) draws a face by inverse CDF (the f with cdf[f] <= U * cdf[T] < cdf[f + 1], U a 53-bit uniform),
 * u = sqrtf(r1), v = r2, x = ((1-u) a + (u (1-v)) b) + (u v) c and xj = x + (r * 2 - 1) / 2^(level+1) per axis, all fp32 op by op;
 * x and xj are quantized as spc.quantize_points does (floor(clamp(2^level (p + 1) / 2, 0, 2^level - 1))) and their bits set.
 * Draws come from the counter-based stream keyed by (seed, sample, draw) (DESIGN.md "Sampling contract").
 * tris: f32 [T, 9] (V[F] row-major); cdf: f64 [T + 1], the exclusive prefix sum of the face areas with cdf[T] > 0 their total;
 * bits: uint32 [(8^level + 31)/32], ORed into (zero it first), the layout of wb_octree_build_bits (bit x<<2L | y<<L | z).
 * 1 <= level <= 10, T >= 1.  num_samples = 0 launches nothing. */
int wb_mesh_octree_bits(const float* tris, const double* cdf, int64_t num_triangles, int64_t num_samples, int32_t level,
                        uint32_t seed, uint32_t* bits, wb_stream s);

#ifdef __cplusplus
}
#endif
#endif /* WISPB200_H_ */
