/* libsstb200 - C ABI of the H100-native SST/FSD hot path.
 *
 * Drop-in boundary (SURVEY.md 8b).  The reference (tusen-ai/SST @ 7c95376) reaches its native code
 * through three extension modules; each entry point below names the reference interface it replaces:
 *
 *   pybind module `voxel_layer`          mmdet3d/ops/voxel/src/voxelization.cpp:6-11, voxelization.h:51-130
 *   torch_scatter.scatter / scatter_max   call sites mmdet3d/ops/sst/sst_ops.py:173-175
 *   TorchEx ingroup_indices.forward       call site  mmdet3d/ops/sst/sst_ops.py:246-264
 *
 * plus fused entry points for the parts of the path the reference runs as chains of ATen ops
 * (window partition / bucketing, the Sparse-Regional-Attention encoder layer, DynamicVFE, SIRLayer).
 *
 * Conventions
 *   - plain C types only: device pointers, sizes, a cudaStream_t passed as void*.  No torch types.
 *   - every function returns 0 on success, <0 on error; sstb200_last_error(ctx) describes it.
 *   - all work is enqueued on the context's stream (sstb200_set_stream); no function synchronises
 *     unless it has a `*_host` out-parameter that is non-NULL (documented per function).
 *   - outputs are caller-allocated.  Data-dependent row counts (number of voxels / windows) are
 *     returned in device memory (`*_dev`); capacity of such outputs is the worst case (= #inputs).
 *   - temporaries come from a per-context arena that grows on demand.
 *   - one context per (device, stream, thread).
 */
#ifndef SSTB200_H_
#define SSTB200_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct sstb200_ctx sstb200_ctx;

#define SSTB200_REDUCE_SUM 0
#define SSTB200_REDUCE_MEAN 1
#define SSTB200_REDUCE_MAX 2
#define SSTB200_PREC_FP32 0 /* fp32 tolerance: fp32 math, except that the SRA encoder layer runs its Linears as split-fp16 tensor-core GEMMs
                             * (as SSTB200_PREC_FP32_TC below) when d_model and dim_ff are multiples of 64, fp32 FFMA otherwise */
#define SSTB200_PREC_BF16 1 /* 16-bit tensor-core GEMMs, fp32 accumulate / softmax / LayerNorm / residual.  The SRA encoder uses
                             * IEEE fp16 operands (the reference's own mixed-precision mode, `fp16 = dict(loss_scale=32.0)`), the
                             * VFE / SIR tensor paths bf16; the API name of the mode stays 'bf16'. */
#define SSTB200_PREC_F16 1
#define SSTB200_PREC_FP32_TC 2 /* sstb200_spconv_forward only: fp32 tolerance on the tensor core - every operand carried as two fp16 numbers
                                * (hi + residue), three wgmma products per stage, fp32 accumulation.  22 significant bits for
                                * every element within 2^-16 of the largest one its output row gathers (see sstb200_spconv_forward) */

int sstb200_version(void);
sstb200_ctx* sstb200_create(int device);
void sstb200_destroy(sstb200_ctx* ctx);
int sstb200_set_stream(sstb200_ctx* ctx, void* cuda_stream);
const char* sstb200_last_error(sstb200_ctx* ctx);
int sstb200_num_sms(sstb200_ctx* ctx);

/* V1  voxel_layer.dynamic_voxelize(points, coors, voxel_size, coors_range, NDim=3)
 *     (voxelization.h:72-88, kernel voxelization_cuda.cu:25-65).  points [P,F] fp32 row-major,
 *     coors [P,3] int32 (z,y,x), clamped to the grid like this fork does.  No device sync
 *     (the reference's cudaDeviceSynchronize at voxelization_cuda.cu:371 is not reproduced). */
int sstb200_dynamic_voxelize(sstb200_ctx* ctx, const float* points, int num_points, int num_features,
                             const float voxel_size[3], const float coors_range[6], int32_t* coors);

/* V1' voxel_layer.hard_voxelize(points, voxels, coors, num_points_per_voxel, voxel_size, coors_range, max_points, max_voxels)
 *     (voxelization.h:51-70 -> voxelization_cpu.cpp:43-142 / voxelization_cuda.cu:68-330; SURVEY 8f next-4).  voxels
 *     [max_voxels, max_points, F], coors [max_voxels,3] (z,y,x), num_points_per_voxel [max_voxels] are caller-allocated AND
 *     zero-initialised, as ops/voxel/voxelize.py:46-53 does.  Voxels are numbered by first appearance in the point list; every
 *     voxel keeps its first max_points points in input order.  Returns the voxel count in device memory and, if
 *     voxel_num_host != NULL, on the host (one stream sync; the reference returns an int). */
int sstb200_hard_voxelize(sstb200_ctx* ctx, const float* points, int num_points, int num_features, const float voxel_size[3],
                          const float coors_range[6], int max_points, int max_voxels, float* voxels, int32_t* coors,
                          int32_t* num_points_per_voxel, int32_t* voxel_num_dev, int32_t* voxel_num_host);

/* V2  voxel_layer.dynamic_point_to_voxel_forward(feats, coors, reduce_type)
 *     (voxelization.h:96-108 -> scatter_points_cuda.cu:183-234).
 *     feats [P,C] fp32, coors [P,3] int32.  coor_lo/hi: inclusive bounds of the non-negative
 *     coordinates per column (the reference needs none because it sorts; this build ranks through a
 *     bitmap over the bounding grid).  Outputs (capacity P rows): reduced [.,C], out_coors [.,3],
 *     coors_map [P] (-1 = dropped), reduce_count [.].  num_voxels_dev: device int32.
 *     If num_voxels_host != NULL the call synchronises the stream and stores the count there; it then also fails
 *     (SSTB200 error, no silent result) if a row with non-negative coordinates lay outside coor_lo/hi.
 *     Reproduces the reference's unconditional removal of the first sorted row (:207-210). */
int sstb200_dynamic_point_to_voxel_forward(sstb200_ctx* ctx, const float* feats, const int32_t* coors,
                                           int num_points, int num_feats, int reduce_type,
                                           const int32_t coor_lo[3], const int32_t coor_hi[3],
                                           float* reduced, int32_t* out_coors, int32_t* coors_map,
                                           int32_t* reduce_count, int32_t* num_voxels_dev,
                                           int32_t* num_voxels_host);

/* V3  voxel_layer.dynamic_point_to_voxel_backward (voxelization.h:110-130 ->
 *     scatter_points_cuda.cu:236-303).  grad_feats [P,C] is fully written (zero where no grad). */
int sstb200_dynamic_point_to_voxel_backward(sstb200_ctx* ctx, float* grad_feats, const float* grad_reduced,
                                            const float* feats, const float* reduced,
                                            const int32_t* coors_map, const int32_t* reduce_count,
                                            int num_points, int num_voxels, int num_feats, int reduce_type);

/* V5a torch.unique(coors, dim=0, return_inverse=True, return_counts=True) on int64 rows
 *     (sst_ops.py:158-160,170; voxel_encoder.py:561; sir.py:70).  coors [P,ndim] int64, ndim<=4,
 *     every value inside [coor_lo, coor_hi].  Outputs: new_coors [.,ndim] (lexicographically sorted),
 *     inverse [P] int64, counts [.] int32 (may be NULL). */
int sstb200_unique_rows_i64(sstb200_ctx* ctx, const int64_t* coors, int num_rows, int ndim,
                            const int64_t* coor_lo, const int64_t* coor_hi, int64_t* new_coors,
                            int64_t* inverse, int32_t* counts, int32_t* num_unique_dev,
                            int32_t* num_unique_host);

/* V5b torch_scatter.scatter(src, index, dim=0, reduce=sum|mean) / scatter_max (sst_ops.py:173-175).
 *     src [P,C] fp32, index [P] int64, out [num_segments,C] (empty segments: 0).
 *     argmax (int64 [num_segments,C], may be NULL): lowest row attaining the max, P if empty.
 *     Rows whose index lies outside [0, num_segments) are dropped: they count towards no segment (nor a mean's divisor).  The call
 *     does not report them (it makes no host sync). */
int sstb200_segment_reduce(sstb200_ctx* ctx, const float* src, const int64_t* index, int num_rows,
                           int num_feats, int num_segments, int reduce_type, float* out, int64_t* argmax);

/* B2  ingroup_indices.forward(group_inds, out_inds) (sst_ops.py:246-264): rank of each element among
 *     the elements carrying the same id, in stable (input) order == get_inner_win_inds_slow
 *     (sst_input_layer.py:200-208).  group ids in [0, max_group_id]. */
int sstb200_ingroup_indices(sstb200_ctx* ctx, const int64_t* group_inds, int num, int64_t max_group_id,
                            int64_t* out_inds);

/* B1+B2+B3(levels)+B4  window partition and bucketing for ONE shift (do_shift = 0 | 1), fused.
 *   get_window_coors            ops/sst/sst_ops.py:266-314
 *   get_inner_win_inds          ops/sst/sst_ops.py:244-264 (stable order, sst_input_layer.py:200-208)
 *   level assignment            models/middle_encoders/sst_input_layer_v2.py:128-150
 *   make_continuous_inds + get_flat2win_inds   ops/sst/sst_ops.py:316-331, 27-64
 * coors [n,4] (b,z,y,x).  n may also be given on the device (n_dev != NULL, n = capacity).
 * token_level (int64 [n], may be NULL): drop level carried over from a preceding drop phase; when NULL the
 * level of a window follows from its token count.  All outputs caller-allocated with capacity n
 * (win_offsets n+1); pointers marked "opt" may be NULL. */
typedef struct {
  int32_t sparse_shape[3]; /* x, y, z */
  int32_t window_shape[3]; /* x, y, z (z = sparse z for 2-D windows) */
  int32_t batch_size;      /* upper bound of batch index + 1 */
  int32_t num_levels;      /* <= 8, in the iteration order of the reference's drop_info dict */
  int32_t level_id[8];     /* dict keys */
  int32_t level_lo[8];     /* drop_range[0] */
  int32_t level_hi[8];     /* drop_range[1] */
  int32_t level_max_tokens[8];
} sstb200_window_cfg;

typedef struct {
  int64_t* batch_win_inds; /* opt [n]   == get_window_coors()[0] */
  int64_t* coors_in_win;   /* opt [n,3] == get_window_coors()[1]  (z,y,x) */
  int64_t* drop_level;     /* opt [n]   dict key of the window's level */
  int64_t* flat2win_inds;  /* opt [n]   rank_in_level * max_tokens + inner */
  int32_t* pos_code;       /* opt [n]   x | y<<8 | z<<16 of coors_in_win */
  int32_t* tok_win;        /* [n]   compact window index (rank of the window id among non-empty windows) */
  int32_t* tok_inner;      /* [n]   stable rank of the token inside its window */
  int32_t* win_offsets;    /* [n+1] CSR offsets into tok_perm, R+1 entries valid */
  int32_t* tok_perm;       /* [n]   token indices grouped by window, stable order inside */
  int32_t* win_level;      /* [n]   level slot (0..num_levels-1) per window, R valid */
  int32_t* win_rank;       /* [n]   rank of the window among the windows of its level */
  int32_t* counters;       /* [20]  R, windows per level slot [8], tokens per level slot [8], number of window batches,
                            *       [18] status bits (bit0 token outside the window grid, bit1 window count not covered), [19] spare */
  int32_t* tok_slot;       /* opt [n] position of the token inside tok_perm (inverse permutation) */
  int32_t* win_batch;      /* opt [n+16], 16-byte aligned: one record of 4 ints per batch b = the windows whose first slot lies in
                              [112b, 112b+112): {first window, end window, first slot, end slot}; at most n/32 + 2 records (fits: 4 (n/32 + 2) <= n + 16) */
} sstb200_window_shift;

/* status_host (opt, int32[18]): if non-NULL the call synchronises and returns
 * [0] = bit0: token outside the window grid, bit1: window count not covered by any drop_range;
 * [1..17] = copy of counters[0..16]. */
int sstb200_window_plan(sstb200_ctx* ctx, const int64_t* coors, int n, const int32_t* n_dev,
                        const sstb200_window_cfg* cfg, int do_shift, const int64_t* token_level,
                        const sstb200_window_shift* out, int32_t* status_host);
int sstb200_window_plan_i32(sstb200_ctx* ctx, const int32_t* coors, int n, const int32_t* n_dev,
                            const sstb200_window_cfg* cfg, int do_shift, const sstb200_window_shift* out);

/* A1+A2+A3  one Sparse-Regional-Attention encoder layer (EncoderLayer.forward,
 * mmdet3d/models/sst/sst_basic_block_v2.py:77-126 with WindowAttention :41-75, nn.MultiheadAttention or
 * CosineMultiheadAttention models/sst/cosine_msa.py:449-536), eval mode (dropout = identity).
 * All weight pointers are device pointers in the reference's nn.Module layouts (row-major [out,in]). */
typedef struct {
  int32_t d_model, nhead, dim_ff;
  int32_t act;       /* 1 relu, 2 gelu(erf) */
  int32_t post_norm; /* layer_cfg['post_norm'] (default 1) */
  float norm_eps;    /* LayerNorm 1e-5 / BatchNorm 1e-5 */
  const float *in_proj_w, *in_proj_b;   /* [3d,d], [3d] */
  const float *out_proj_w, *out_proj_b; /* [d,d], [d] */
  const float *lin1_w, *lin1_b;         /* [ff,d], [ff] */
  const float *lin2_w, *lin2_b;         /* [d,ff], [d] */
  const float *norm1_w, *norm1_b, *norm2_w, *norm2_b;
  const float *norm1_mean, *norm1_var, *norm2_mean, *norm2_var; /* non-NULL: layer_cfg['use_bn'] (eval BN) */
  const float* tau; /* non-NULL: cosine attention; tau_n = 1 or nhead */
  int32_t tau_n;
  float tau_min;
  /* optional IEEE fp16 copies of the four weight matrices (tensor-core path); NULL -> fp32 path only */
  const void *in_proj_w_f16, *out_proj_w_f16, *lin1_w_f16, *lin2_w_f16;
} sstb200_sra_layer;

/* window CSR of one shift (produced by sstb200_window_plan) + positional-embedding table
 * (SSTInputLayerV2.get_pos_embed, sst_input_layer_v2.py:238-305: pos[t, axis*L + j] =
 * table[axis][coord_in_win(axis)][j], zero beyond ndim*L). */
typedef struct {
  const int32_t* win_offsets; /* [R+1] */
  const int32_t* tok_perm;    /* [n] */
  const int32_t* tok_win;     /* [n] */
  const int32_t* pos_code;    /* [n] */
  const int32_t* num_windows_dev; /* counters[0] */
  const float* pos_table;     /* [pos_ndim][pos_maxw][pos_L] fp32 */
  int32_t pos_L, pos_maxw, pos_ndim;
  int32_t max_window_tokens;  /* upper bound on tokens per window (e.g. 144) */
  const int32_t* tok_slot;    /* [n] inverse of tok_perm (needed by the bf16 path) */
  const int32_t* win_batch;   /* opt [.] window batches (see sstb200_window_shift); counters[17] = number of batches */
} sstb200_sra_plan;


/* x, y: [n, d_model] fp32 in flat voxel order (y may alias x only if precision == FP32 is not used).
 * n may be device-resident (n_dev).  */
int sstb200_sra_layer_forward(sstb200_ctx* ctx, const sstb200_sra_layer* layer, const sstb200_sra_plan* plan,
                              const float* x, float* y, int n, const int32_t* n_dev, int precision);

/* nn.Linear forward: out[M,N] = act(A[M,K] . W[N,K]^T + bias), fp32 (act: 0 none, 1 relu, 2 gelu-erf).
 * Used for SSTv2.linear0 (models/backbones/sst_v2.py:60-61,127-128) and as a building block. */
int sstb200_linear(sstb200_ctx* ctx, const float* A, const float* W, const float* bias, float* out,
                   int M, int N, int K, int act);

/* V4 DynamicVFE.forward / V6 DynamicScatterVFE.forward, eval-mode BatchNorm, <= 2 VFE layers
 * (mmdet3d/models/voxel_encoders/voxel_encoder.py:229-298 and :551-612; layers utils.py:107-144).
 * points [P,in_channels] fp32, coors [P,4] (b,z,y,x).  Output rows are the non-empty voxels sorted by
 * (b,z,y,x); capacity P.  drop_first_voxel_per_sample = 1 reproduces DynamicVFE's DynamicScatter behaviour
 * (scatter_points_cuda.cu:207-210 through the per-sample loop scatter_points.py:85-99): a sample loses its first
 * voxel unless one of its points has a negative z, y or x (then the removed row is that point's (-1,-1,-1) row).
 * Points with a negative or out-of-canvas coordinate belong to no voxel.  DynamicScatterVFE (torch.unique based)
 * keeps every voxel. */
typedef struct {
  int32_t in_channels;       /* raw point dims F (before decoration) */
  int32_t num_layers;        /* 1 or 2 */
  int32_t feat_channels[2];
  int32_t with_cluster_center, with_voxel_center, with_distance;
  int32_t mode_max;          /* 1: max pooling, 0: average */
  int32_t drop_first_voxel_per_sample;
  int32_t batch_size;
  int32_t grid_zyx[3];       /* canvas dims (voxel_encoder.py:199-204) */
  float voxel_size[3];       /* vx, vy, vz */
  float center_offset[3];    /* v/2 + range_min (voxel_encoder.py:160-162) */
  float rel_dist_scaler;     /* DynamicScatterVFE only, else 1 */
  float bn_eps;
  int32_t precision;         /* SSTB200_PREC_FP32: FFMA everywhere; SSTB200_PREC_BF16: layer 1 on wgmma (bf16 operands) */
  const float* weight[2];    /* vfe_layers.i.linear.weight  [C_i, in_i] */
  const float* bn_weight[2]; /* vfe_layers.i.norm.{weight,bias,running_mean,running_var} */
  const float* bn_bias[2];
  const float* bn_mean[2];
  const float* bn_var[2];
} sstb200_vfe_cfg;

int sstb200_dynamic_vfe_forward(sstb200_ctx* ctx, const sstb200_vfe_cfg* cfg, const float* points,
                                const int32_t* coors, int num_points, float* voxel_feats, int32_t* voxel_coors,
                                int32_t* num_voxels_dev, int32_t* num_voxels_host);
int sstb200_dynamic_scatter_vfe_forward(sstb200_ctx* ctx, const sstb200_vfe_cfg* cfg, const float* points,
                                        const int64_t* coors, int num_points, float* voxel_feats,
                                        int64_t* voxel_coors, int64_t* unq_inv, int32_t* num_voxels_dev,
                                        int32_t* num_voxels_host);

/* V1 (batched, sync-free form used by the frame engine): voxelise a batch of frames stored back to back.
 * points [capacity,F]; frame_offsets_dev: device int32 [num_frames+1] (row ranges of the frames, last entry =
 * number of valid rows).  coors4 [capacity,4] int32 = (b,z,y,x) like DynamicVoxelNet.voxelize
 * (mmdet3d/models/detectors/dynamic_voxelnet.py:49-71); rows beyond the last offset get (-1,-1,-1,-1) and are
 * ignored by every later stage. */
int sstb200_voxelize_frames(sstb200_ctx* ctx, const float* points, int capacity, int num_features,
                            const int32_t* frame_offsets_dev, int num_frames, const float voxel_size[3],
                            const float coors_range[6], int32_t* coors4);

/* C5  SingleStageFSDV2.voxelize_with_batch_idx (mmdet3d/models/detectors/single_stage_fsd_v2.py:108-123): virtual-voxel coordinates
 * of the concatenated real + virtual points.  points [n, ldp] fp32 (x,y,z first), batch_idx [n] int64 ->
 * coors [n,4] int64 (batch, z, y, x) = floor_div(p - range_lo, voxel_size) with torch.div(rounding_mode='floor') semantics, no clamp. */
int sstb200_voxelize_with_batch_idx(sstb200_ctx* ctx, const float* points, int n, int ldp, const int64_t* batch_idx,
                                    const float voxel_size[3], const float range_lo[3], int64_t* coors);

/* Fork / join of a side branch.  `side` is a second context (own stream, own workspace arena).  fork: side's stream waits for the
 * point of ctx's stream at which the last sstb200_dynamic_vfe_forward / sstb200_dynamic_scatter_vfe_forward call had produced
 * voxel_coors and num_dev (the VFE layers that follow in that call keep running on ctx's stream); join: ctx's stream waits for
 * everything enqueued on side's stream so far.  The engine runs the two sstb200_window_plan calls of a frame on the side branch,
 * next to the VFE layers.  Valid on plain streams and inside sstb200_graph_begin/end (the side stream joins the capture). */
int sstb200_branch_fork(sstb200_ctx* ctx, sstb200_ctx* side);
int sstb200_branch_join(sstb200_ctx* ctx, sstb200_ctx* side);

/* CUDA-graph helpers for callers that chain several entry points per frame (the reference has no
 * counterpart: it launches ~10^3 ATen kernels per frame with >= 8 host syncs, SURVEY.md 3.1).
 * begin: start capturing the context's stream; end: stop, instantiate, return an opaque handle and the number
 * of kernel / memset+memcpy nodes; launch: replay on the context's stream. */
int sstb200_graph_begin(sstb200_ctx* ctx);
int sstb200_graph_end(sstb200_ctx* ctx, void** graph_exec_out, int32_t* num_kernel_nodes, int32_t* num_other_nodes);
int sstb200_graph_launch(sstb200_ctx* ctx, void* graph_exec);
int sstb200_graph_destroy(sstb200_ctx* ctx, void* graph_exec);

/* S1-S3  SIRLayer.forward (mmdet3d/models/voxel_encoders/voxel_encoder.py:696-764; build_mlp ops/sst/sst_ops.py:334-361;
 * DynamicVFELayerV2 voxel_encoders/utils.py:147-189), LayerNorm norm, mode='max', with_rel_mlp=True.
 * in_feats [N,in_channels] = cat(points, feats) as SIR.forward builds it (models/backbones/sir.py:77), f_cluster [N,3]
 * (un-scaled; divided by rel_dist_scaler inside), group index inv [N] int64 in [0,G) (torch.unique inverse).
 * out_point [N, C_last]; out_group [G, C0+C1] = concatenated per-layer group max (voxel_encoder.py:751). */
typedef struct {
  int32_t in_channels;
  int32_t rel_in;          /* rel_mlp_in_channel (3) */
  int32_t num_rel;         /* number of rel-MLP layers (hidden dims + in_channels) */
  int32_t rel_dims[4];
  int32_t num_vfe;         /* 1 or 2 */
  int32_t feat_channels[2];
  int32_t act;             /* 1 relu, 2 gelu */
  int32_t mode_max;
  int32_t with_shortcut;
  float norm_eps;
  float xyz_normalizer[3];
  float rel_dist_scaler;
  const float* rel_w[4];    /* rel_mlp.i.0.weight [dims[i], in_i] */
  const float* rel_ln_w[4]; /* rel_mlp.i.1.weight */
  const float* rel_ln_b[4];
  const float* vfe_w[2];    /* vfe_layers.i.linear.weight  [C_i, in_i] (in_1 = 2*C0) */
  const float* vfe_ln_w[2];
  const float* vfe_ln_b[2];
} sstb200_sir_layer;

int sstb200_sir_layer_forward(sstb200_ctx* ctx, const sstb200_sir_layer* layer, const float* in_feats,
                              const float* f_cluster, const int64_t* inv, int num_points, int num_groups,
                              float* out_point, float* out_group);

/* S1' as above, plus: a cached group CSR (csr_offsets [G+1], csr_order [N] from sstb200_group_csr; both NULL = built inside),
 * `precision` (SSTB200_PREC_BF16: the rel-MLP's last layer and both VFE layers run as wgmma GEMMs with bf16 operands and fp32
 * accumulation - needs feat_channels [128,128], rel-MLP [16,32,cin], cin <= 192, else SSTB200 "unsupported" error) and a row
 * pitch for out_point (>= C_last; lets SIR.forward write block i's point features straight into block i+1's [points || feats]
 * input; bf16 path only, 0 = dense).  in_feats may likewise be a pitched matrix (in_ld floats per row, 0 = dense) whose columns
 * >= in_gap_at sit in_gap floats further right (the 16-byte aligned feature block of that hand-over buffer). */
int sstb200_sir_layer_forward_ex(sstb200_ctx* ctx, const sstb200_sir_layer* layer, const float* in_feats, int in_ld,
                                 int in_gap_at, int in_gap, const float* f_cluster, const int64_t* inv, int num_points, int num_groups,
                                 const int32_t* csr_offsets, const int32_t* csr_order, int precision, float* out_point,
                                 int out_point_ld, float* out_group);

/* S1 training (fp32, as the reference trains SIRLayer under @force_fp32).  Range: mode_max, rel-MLP present with rel_in <= 32 and
 * widths <= 256, 1-2 VFE layers with feat_channels multiples of 32 and <= 256, in_channels in [3, 256]; anything else is
 * SSTB_ERR_UNSUPPORTED.  num_points = 0 or num_groups = 0 launches nothing (and writes nothing).
 * forward_train: the inputs of sstb200_sir_layer_forward_ex on dense fp32 rows, the same outputs as the fp32 eval forward, and a
 * caller-owned `state` of sstb200_sir_layer_train_state_bytes() bytes (the pre-LayerNorm values of the VFE layers and the row of
 * each group max, the lowest point index attaining it) that the backward reads.  The state must outlive the backward call. */
size_t sstb200_sir_layer_train_state_bytes(const sstb200_sir_layer* layer, int num_points, int num_groups);
int sstb200_sir_layer_forward_train(sstb200_ctx* ctx, const sstb200_sir_layer* layer, const float* in_feats, const float* f_cluster,
                                    const int64_t* inv, int num_points, int num_groups, const int32_t* csr_offsets,
                                    const int32_t* csr_order, float* out_point, float* out_group, void* state, size_t state_bytes);
/* Parameter gradients in the layout of the parameters (rel_w[i] [dims[i], in_i], vfe_w[i] [C_i, in_i], ...); written, not added. */
typedef struct {
  float* rel_w[4];
  float* rel_ln_w[4];
  float* rel_ln_b[4];
  float* vfe_w[2];
  float* vfe_ln_w[2];
  float* vfe_ln_b[2];
} sstb200_sir_layer_grads;
/* backward of forward_train with the same layer, inputs, CSR and state: grad_point [N, C_last] (d loss / d out_point) and
 * grad_group [G, C0+C1] (d loss / d out_group), either NULL = zero.  Writes grad_in_feats [N, in_channels] and grad_f_cluster
 * [N, rel_in] (each NULL = skipped) and every gradient of `grads`.  No float atomics: two calls give the same bits. */
int sstb200_sir_layer_backward(sstb200_ctx* ctx, const sstb200_sir_layer* layer, const float* in_feats, const float* f_cluster,
                               const int64_t* inv, int num_points, int num_groups, const int32_t* csr_offsets, const int32_t* csr_order,
                               const void* state, size_t state_bytes, const float* grad_point, const float* grad_group,
                               float* grad_in_feats, float* grad_f_cluster, const sstb200_sir_layer_grads* grads);

/* Points grouped by `inv` (values in [0, num_groups)): offsets [num_groups+1] int32, order [num_points] int32 (order inside a
 * group unspecified).  What SIR.forward (models/backbones/sir.py:67-87, `unique_once`) shares between its blocks. */
int sstb200_group_csr(sstb200_ctx* ctx, const int64_t* inv, int num_points, int num_groups, int32_t* offsets, int32_t* order);

/* A4'  SSTv2.recover_bev (mmdet3d/models/backbones/sst_v2.py:161-196): voxel_feat [M,C] fp32 rows at coors [M,4] int64 (b,z,y,x)
 * -> canvas [B,C,ny,nx] fp32, empty cells 0 (the canvas need not be zeroed by the caller: every element is written once).
 * Synchronises the stream to report out-of-canvas coordinates as an error (the reference would raise an index error). */
int sstb200_recover_bev(sstb200_ctx* ctx, const float* voxel_feat, const int64_t* coors, int num_voxels, int channels,
                        int batch_size, int ny, int nx, float* canvas);

/* A4' backward: grad_feat[m, :] = grad_canvas[b_m, :, y_m, x_m] for every row m (rows that share a cell each receive that cell's
 * gradient, as torch's index_put backward gives them), a pure copy.  grad_canvas [B,C,ny,nx] fp32 contiguous, grad_feat [M,C] fp32.
 * Precondition: the coordinates passed sstb200_recover_bev (no check here, so no stream synchronisation); a row outside the
 * canvas gets zeros and nothing is read for it. */
int sstb200_recover_bev_backward(sstb200_ctx* ctx, const float* grad_canvas, const int64_t* coors, int num_voxels, int channels,
                                 int batch_size, int ny, int nx, float* grad_feat);

/* N1  Voxel2PointScatterNeck.forward (mmdet3d/models/necks/voxel2point_neck.py:28-62; SURVEY 8f next-2): points [N,Cp] fp32,
 * pts_coors [N,4] int64 (b,z,y,x), voxel_feats [M,C] fp32 (rows of dropped voxels hold `padding`), voxel2point_inds [N] int64.
 * out [<=N, C(+3)] receives, for every point whose voxel row is not all-padding and in input order, the voxel row followed (with_xyz)
 * by the point's offset from its voxel centre; mask_out [N] (1 = kept).  The call synchronises once to return the row count (the
 * reference's boolean indexing does the same) and to report out-of-range indices as an error. */
int sstb200_voxel2point(sstb200_ctx* ctx, const float* points, int point_dims, const int64_t* pts_coors, const float* voxel_feats,
                        int num_voxels, int channels, const int64_t* voxel2point_inds, int num_points, float padding,
                        const float voxel_size[3], const float pc_min[3], int with_xyz, int normalize_local_xyz, float* out,
                        uint8_t* mask_out, int32_t* num_out_dev, int32_t* num_out_host);

/* N1 backward (gradient w.r.t. voxel_feats only): grad_out [num_kept, C(+3 if with_xyz)] fp32 is the gradient of the forward's
 * `out`, mask [N] its mask_out and num_kept its row count.  grad_voxel [M,C] fp32 receives, for each voxel v, the sum of
 * grad_out[pos(p), 0:C] over the kept points p with voxel2point_inds[p] == v (pos = rank among the kept points); voxels no kept
 * point references (padded rows among them) get 0.  Summed in fp64 without float atomics, so two calls give the same bits.
 * No stream synchronisation; indices outside [0, M) are skipped. */
int sstb200_voxel2point_backward(sstb200_ctx* ctx, const float* grad_out, const uint8_t* mask, const int64_t* voxel2point_inds,
                                 int num_points, int num_kept, int num_voxels, int channels, int with_xyz, float* grad_voxel);

/* A4  the whole encoder stack (SSTv2.forward's block loop, mmdet3d/models/backbones/sst_v2.py:129-133 with
 * BasicShiftBlockV2.forward, models/sst/sst_basic_block_v2.py:144-169): layer l uses the windows of shift l % 2.
 * x [n,d] input (not modified), y [n,d] output, tmp [n,d] scratch; all fp32, distinct buffers.  With precision BF16 and the
 * SST-6 shape (d=128, h=8, ff=256, post-norm LayerNorm, GELU) this runs 2 launches per layer: ragged window attention and a
 * fused wgmma / TMA kernel (out-proj + LN1 + FFN + LN2 + the next layer's QKV); otherwise it loops sstb200_sra_layer_forward. */
int sstb200_sra_stack_forward(sstb200_ctx* ctx, const sstb200_sra_layer* layers, int num_layers,
                              const sstb200_sra_plan* plan_shift0, const sstb200_sra_plan* plan_shift1, const float* x,
                              float* y, float* tmp, int n, const int32_t* n_dev, int precision);

/* ---- training (BASELINE config 4): SSTv2's encoder stack with everything the backward pass needs kept in `workspace`, and the
 * backward pass (the autograd graph torch builds over sst_basic_block_v2.py:100-126 / backbones/sst_v2.py:129-133 in the reference).
 * Shape: d_model 128, 8 heads, dim_ff 256, post-norm LayerNorm, GELU, windows <= 144 tokens (all configs/sst_refactor models).
 * Attention: plain scaled dot product, or cosine attention (layer.tau non-NULL: tau_n 1 or 8 temperatures, tau_min > 0; the
 * gradient of tau is 0 where tau < tau_min, as torch's clamp(min=) gives it).  BatchNorm layers (norm1_mean non-NULL) are refused.
 * GEMM operands and saved activations are bf16, accumulation / softmax / LayerNorm / residual stream / gradients of the
 * parameters fp32.  For these two entry points the `*_w_f16` fields of sstb200_sra_layer hold BF16 copies of the weights. */
typedef struct {
  const void *in_proj_wt, *out_proj_wt, *lin1_wt, *lin2_wt; /* bf16 TRANSPOSED copies, [in, out] row-major */
} sstb200_sra_layer_wt;
typedef struct { /* fp32 accumulators in the layout of the parameters; the call ADDS to them */
  float *in_proj_w, *in_proj_b, *out_proj_w, *out_proj_b, *lin1_w, *lin1_b, *lin2_w, *lin2_b, *norm1_w, *norm1_b, *norm2_w, *norm2_b;
  float* tau; /* [tau_n] for a cosine-attention layer, NULL for plain attention */
} sstb200_sra_layer_grads;

size_t sstb200_sra_train_workspace_bytes(int n, int num_layers);
/* x [n,128] fp32 (not modified) -> y_out [n,128]; workspace: device buffer of sstb200_sra_train_workspace_bytes() */
int sstb200_sra_stack_forward_train(sstb200_ctx* ctx, const sstb200_sra_layer* layers, int num_layers,
                                    const sstb200_sra_plan* plan_shift0, const sstb200_sra_plan* plan_shift1, const float* x,
                                    float* y_out, void* workspace, int n);
/* dy [n,128] = d loss / d y_out  ->  dx [n,128] = d loss / d x, parameter gradients accumulated into `grads`.  Every reduction
 * runs in a fixed order without float atomics, so two calls give the same bits, and the result equals G0 + g bit for bit, where
 * G0 is what `grads` held and g what the call adds to zeroed buffers.  n == 0 touches neither dx nor `grads`. */
int sstb200_sra_stack_backward(sstb200_ctx* ctx, const sstb200_sra_layer* layers, const sstb200_sra_layer_wt* wt,
                               const sstb200_sra_layer_grads* grads, int num_layers, const sstb200_sra_plan* plan_shift0,
                               const sstb200_sra_plan* plan_shift1, const float* x, void* workspace, const float* dy, float* dx,
                               int n);
/* torch.optim.AdamW step over a flat fp32 buffer (decoupled weight decay, bias-corrected moments); the gradient is read as
 * grads[i] * grad_scale (1 / world_size after a summing all-reduce).  step counts from 1. */
int sstb200_adamw_step(sstb200_ctx* ctx, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                       float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale);

/* ---- next-1 (SURVEY 8f): sparse 3-D convolution of the reference's sparse U-Nets (SimpleSparseUNet / VirtualVoxelMixer,
 * mmdet3d/models/middle_encoders/sparse_unet.py:15-505; SparseBasicBlock / make_sparse_convmodule, mmdet3d/ops/sparse_block.py:81-289),
 * which the reference delegates to spconv.  The three entry points replace spconv's native interface as vendored in the tree
 * (mmdet3d/ops/spconv/src/all.cc:21-33): get_indice_pairs_3d (ops.py:47-107 -> include/spconv/spconv_ops.h:25-93, geometry.h:25-301)
 * and indice_conv_fp32 / fused_indice_conv_fp32 (ops.py:110-137 -> spconv_ops.h:95-260, fused_spconv_ops.h).
 * Coordinates are int32 rows (batch, z, y, x); spatial shapes / kernel sizes / strides / paddings are (z, y, x) triples; kernel
 * offset k = (dz * ky + dy) * kx + dx reads the input cell  out * stride - padding + (dz, dy, dx)  (geometry.h:60-67).
 * The rulebook is OUTPUT-STATIONARY: nbr[o][k] = input row feeding output row o through offset k, or -1. */

/* Active output cells of SparseConv3d (non-submanifold): every output cell with at least one active input in its receptive field,
 * emitted in lexicographic (b,z,y,x) order (spconv's order is hash-insertion order; features are compared per coordinate).
 * out_cap >= min(n_in * prod(ceil(k/s)), batch * prod(out_shape)).  num_out_host != NULL: one stream sync, and an input coordinate
 * outside batch_size / in_shape is reported as an error. */
int sstb200_spconv_out_coors(sstb200_ctx* ctx, const int32_t* in_coors, int n_in, int batch_size, const int32_t in_shape[3],
                             const int32_t out_shape[3], const int32_t ksize[3], const int32_t stride[3], const int32_t padding[3],
                             int32_t* out_coors, int out_cap, int32_t* num_out_dev, int32_t* num_out_host);

/* Neighbour tables between two coordinate sets (rows unique).  SubMConv3d: out_coors = in_coors, stride 1, out_shape = in_shape.
 * nbr [n_out, KV] (may be NULL): input row at  out * stride - padding + delta_k.  nbr_inv [n_in, KV] (may be NULL): the transposed
 * table = output row that input row i feeds through offset k - the table SparseInverseConv3d runs on (indice pairs of its couple
 * conv with in / out swapped, mmdet3d/ops/spconv/conv.py:147-153).  status_host != NULL: one stream sync, coordinates outside the
 * grids are an error. */
int sstb200_spconv_table(sstb200_ctx* ctx, const int32_t* in_coors, int n_in, const int32_t* out_coors, int n_out, int batch_size,
                         const int32_t in_shape[3], const int32_t out_shape[3], const int32_t ksize[3], const int32_t stride[3],
                         const int32_t padding[3], int32_t* nbr, int32_t* nbr_inv, int32_t* status_host);

/* out[o, :] = act( (sum_k feats[nbr[o][k], :] . W[k]) * scale + shift + residual[o, :] )   - one launch for conv + folded
 * BatchNorm1d (+ residual add) (+ ReLU).  feats [*, c_in] fp32, weight [KV, c_in, c_out] fp32 = the reference's parameter layout
 * (D,H,W,in,out; mmdet3d/ops/spconv/conv.py:97-98), scale / shift [c_out] or NULL (1 / 0), residual [n_out, c_out] or NULL.
 * n_in = rows of feats (every nbr entry is < n_in).
 * precision FP32: FFMA implicit GEMM (c_in, c_out multiples of 4).  precision BF16 (the name of the mode; the operands are IEEE
 * fp16, fp32 accumulation): wgmma implicit GEMM over weight_h16 = fp16 copy laid out [KV, c_out, c_in]; needs c_in, c_out multiples
 * of 64, KV <= 27.  precision FP32_TC: the same kernel in split mode; weight_h16 = [2][KV, c_out, c_in]: the fp16 copy followed by
 * the fp16 residue (w - float(half(w))).
 * Operand range of the two tensor-core modes.  fp16 keeps 11 bits only between 2^-14 and 65504, so neither operand is rounded as it
 * is.  feats: the call first gives every row of feats a power-of-two exponent (one extra small launch, n_in ints of the context's
 * arena); an output row's operand rows are scaled by the smallest exponent among the rows it gathers, which puts the largest
 * gathered |element| in [2^13, 2^14), and the accumulator row is scaled back.  weight_h16: the copy may carry one power of two per
 * output channel, w16[k][co][ci] = half(w[k][ci][co] * 2^e[co]); weight_h16_unscale [c_out] fp32 then holds 2^-e[co] (NULL: the copy
 * is unscaled, which is accurate only for |w| in about [2^-14, 65504]).  All of this is exact in fp32, so the result is homogeneous:
 * feats * 2^s or weight * 2^s gives out * 2^s with the same relative error, for any s that keeps out a normal fp32 number.  What
 * remains is relative to the largest element an output row gathers: elements below 2^-27 of it (BF16; 2^-16 for the
 * 22 bits of FP32_TC) are rounded with an absolute error of 2^-38 of it instead of a relative one. */
int sstb200_spconv_forward(sstb200_ctx* ctx, const float* feats, int n_in, int c_in, const int32_t* nbr, int n_out, int kernel_volume,
                           const float* weight, const void* weight_h16, const float* weight_h16_unscale, int c_out,
                           const float* scale, const float* shift, const float* residual, int relu, int precision, float* out);

/* Backward of sstb200_spconv_forward without epilogue (indice_conv_backward_fp32, mmdet3d/ops/spconv/src/all.cc:34-35 ->
 * spconv_ops.h:262-420).  The input gradient needs no entry point of its own: dX = sstb200_spconv_forward(dY, nbr_T, W^T) on the
 * TRANSPOSED table (nbr_inv of sstb200_spconv_table; the table SparseInverseConv3d runs on); the operand exponents described there
 * are what keeps it accurate for the 1e-5 ... 1e-8 rows of a mean-reduced loss's gradient.  This call computes the weight gradient
 * grad_weight [KV, c_in, c_out] fp32 (fully written) = sum over pairs of feats[nbr[o][k]]^T . grad_out[o]; fp32 atomics across row
 * chunks, so the last bits depend on the launch like the reference's backward. */
int sstb200_spconv_backward_weight(sstb200_ctx* ctx, const float* feats, int c_in, const int32_t* nbr, int n_out, int kernel_volume,
                                   const float* grad_out, int c_out, float* grad_weight);

/* ---- next-3 (SURVEY 8f): FSD instance grouping.  find_connected_componets / _single_batch / _gpu
 * (mmdet3d/models/detectors/single_stage_fsd.py:37-81; TorchEx connected_components at :20,39-45): two centres of the same sample are
 * adjacent when sqrt(dx^2 + dy^2) < dist (xy only, fp32); labels [n] = component number, components numbered sample by sample (batch
 * index ascending) and, inside a sample, by their first centre in input order - scipy.sparse.csgraph.connected_components' numbering
 * with the reference's running `base`.  centers [n, stride >= 2] fp32 (x, y first), batch_idx [n] int32 in [0, batch_size) or NULL
 * (one sample).  xy_min / xy_max bound the binning grid (centres outside are binned into the border cells: still exact).
 * num_components_host != NULL: one stream sync; a batch index outside [0, batch_size) is then reported as an error (label -1). */
int sstb200_connected_components(sstb200_ctx* ctx, const float* centers, int stride, const int32_t* batch_idx, int n, int batch_size,
                                 float dist, const float xy_min[2], const float xy_max[2], int32_t* labels,
                                 int32_t* num_components_dev, int32_t* num_components_host);

/* ---- next-3 (SURVEY 8f): FSD RoI point pooling.  dynamic_point_pool / dynamic_point_pool_mixed (mmdet3d/ops/dynamic_point_pool_op.py:9-113,
 * kernel in TorchEx's unvendored dynamic_point_pool_ext) as used by DynamicPointROIExtractor (models/roi_heads/roi_extractors/
 * dynamic_point_roi_extractor.py:32-136).  rois [num_rois, 7] fp32 = (x, y, z_bottom, w, l, h, rz) mmdet3d-0.15 LiDAR boxes; pts [num_pts, 3].
 * rois_batch / pts_batch: int32 batch ids (>= 0) or both NULL (one sample); a point pairs only with RoIs of its own batch id.
 * In-box test: check_pt_in_box3d of mmdet3d/ops/roiaware_pool3d/src/points_in_boxes_cuda.cu:24-49 as the same float expressions (centre
 * z = bottom + h/2, |z - cz| > h/2 rejects, angle rz + pi/2, strict |local x| < l/2, |local y| < w/2).
 * Output rows (pair = point inside the ENLARGED box): out_pts_idx int64, out_roi_idx int64, out_feats fp32 [., 13] = point xyz,
 * local xyz, boundary offsets [6], is_in_margin.  Pinned by the reference: the layout, off[0]+off[3] = l, off[1]+off[4] = w,
 * off[2]+off[5] = h, xyz = pts[idx], and one fake row (-1, -1, zeros) when nothing pairs.
 * Chosen here (TorchEx's source is not available; the offset order and the origin of local z feed FullySparseBboxHead's f_cluster and are
 * UNVERIFIED against TorchEx, so a checkpoint trained with it may see different features):
 *   - enlarged box: same centre and yaw, dims (w + e0, l + e1, h + e2), i.e. the box (x, y, z_bottom - e2/2, w + e0, l + e1, h + e2, rz);
 *   - is_in_margin = 1 inside the enlarged box but outside the original one, else 0;
 *   - local xyz = (local x, local y, z - centre z): local z from the box CENTRE;
 *   - offsets = (l/2 + lx, w/2 + ly, h/2 + lz, l/2 - lx, w/2 - ly, h/2 - lz) against the ORIGINAL box (negative in the margin);
 *   - rows sorted by RoI, then point index; every RoI keeps its first max_inbox_point (1..8192) points in input order.  Deterministic:
 *     two calls give bit-identical results (the reference assigns slots with atomics, so its choice and order vary from run to run);
 *   - capacity: pairs beyond max_all_pts (>= 1) are dropped in (RoI, point) order.  per_sample = 0: max_all_pts and the fake row apply
 *     to the whole call (outputs hold max_all_pts rows; no RoI at all gives no row).  per_sample = 1 (batch ids required, RoIs grouped by
 *     ascending batch id): they apply to every sample, i.e. every run of equal RoI batch ids, its fake row placed where its rows would
 *     be - the per-sample loop of DynamicPointROIExtractor in one call; outputs hold max_all_pts x (number of samples) rows.
 * num_out_dev: rows written.  num_pairs_host (int32[3]) != NULL: one stream sync, then [0] rows written, [1] pairs found (at most
 * max_inbox_point per RoI), [2] pairs written; a negative batch id, or RoIs not grouped in per-sample mode, is then an error. */
int sstb200_dynamic_point_pool(sstb200_ctx* ctx, const float* rois, const int32_t* rois_batch, int num_rois, const float* pts,
                               const int32_t* pts_batch, int num_pts, const float extra_wlh[3], int max_inbox_point, int max_all_pts,
                               int per_sample, int64_t* out_pts_idx, int64_t* out_roi_idx, float* out_feats, int32_t* num_out_dev,
                               int32_t* num_pairs_host);

/* ---- Rotated BEV overlap, IoU and NMS: mmdet3d/ops/iou3d (iou3d_utils.py, src/iou3d.cpp, src/iou3d_kernel.cu), used by
 * box3d_multiclass_nms (core/post_processing/box3d_nms.py:10-143), CenterHead / FullySparseBboxHead (nms_gpu) and
 * BaseInstance3DBoxes.overlaps (boxes_overlap_bev_gpu).
 * Boxes are fp32 [x1, y1, x2, y2, r] rows.  Corners (x1,y1), (x2,y1), (x2,y2), (x1,y2) are turned about the box centre by
 * (dx cos r + dy sin r, -dx sin r + dy cos r), the reference's convention.  Overlap = exact area of the two rectangles' intersection,
 * evaluated in fp32 relative to one box's centre (0 when the circumscribed circles are apart, 0 for a zero-area box, never NaN);
 * iou = overlap / max(sa + sb - overlap, 1e-8), s = (x2 - x1)(y2 - y1).
 *
 * sstb200_boxes_overlap_bev / sstb200_boxes_iou_bev: out [num_a, num_b] row-major (out[i * num_b + j] for a_i, b_j); every entry is
 * written.  num_a or num_b = 0 writes nothing; a negative size is SSTB_ERR_ARG; num_a > 65535 * 32 is SSTB_ERR_UNSUPPORTED.  No sync. */
int sstb200_boxes_overlap_bev(sstb200_ctx* ctx, const float* boxes_a, int num_a, const float* boxes_b, int num_b, float* overlap);
int sstb200_boxes_iou_bev(sstb200_ctx* ctx, const float* boxes_a, int num_a, const float* boxes_b, int num_b, float* iou);

/* Segmented greedy NMS (nms_gpu / nms_normal_gpu of iou3d_utils.py:31-56,106-124 over every segment of one call).
 * boxes [num, 5] are grouped into segments s = rows [seg_offsets[s], seg_offsets[s+1]), each sorted by descending score (the caller
 * sorts).  seg_offsets is a HOST int32 array of num_segs + 1 entries: seg_offsets[0] = 0, non-decreasing, seg_offsets[num_segs] = num;
 * thresh is a HOST float array of num_segs thresholds (INFINITY keeps every box of its segment).  Within a segment, box j is
 * suppressed by an earlier kept box i iff IoU(i, j) > thresh[s] (strict); rotated = 1 uses the rotated IoU, rotated = 0 the
 * axis-aligned IoU of nms_normal_gpu (r ignored).  The result equals the reference's 64-bit mask + greedy scan (iou3d.cpp:130-143)
 * run on each segment alone, up to fp32 rounding of IoUs that lie at the threshold.
 * keep_out (int64, capacity num): positions into `boxes` of the kept boxes, segment after segment, ascending within a segment;
 * num_keep_dev (device int32): their number; num_keep_host != NULL: one stream sync, then the same number on the host.
 * Workspace: caller-allocated device memory of at least sstb200_nms_bev_workspace_bytes(num, seg_offsets, num_segs) bytes (mask of
 * sum_s n_s * ceil(n_s / 64) 64-bit words, plus num + num_segs int32 and the segment table); the call allocates nothing and uses no
 * atomics, so results are deterministic.  Largest segment: 65536 boxes (SSTB_ERR_UNSUPPORTED beyond, from both functions).
 * Errors (SSTB_ERR_ARG, nothing enqueued): num or num_segs negative, seg_offsets NULL with num_segs > 0, num_segs = 0 with num > 0,
 * offsets not starting at 0, decreasing or not ending at num, boxes / keep_out / thresh NULL when needed, workspace NULL;
 * workspace_bytes below the query's value is SSTB_ERR_WORKSPACE. */
int sstb200_nms_bev_workspace_bytes(sstb200_ctx* ctx, int num, const int32_t* seg_offsets, int num_segs, int64_t* bytes);
int sstb200_nms_bev(sstb200_ctx* ctx, const float* boxes, int num, const int32_t* seg_offsets, int num_segs, const float* thresh,
                    int rotated, void* workspace, int64_t workspace_bytes, int64_t* keep_out, int32_t* num_keep_dev,
                    int32_t* num_keep_host);

/* ---- Points in boxes and RoI-aware pooling: mmdet3d/ops/roiaware_pool3d (points_in_boxes.py, roiaware_pool3d.py, src/).
 * Boxes / RoIs are fp32 rows (x, y, z_bottom, w, l, h, rz).  A point is inside when check_pt_in_box3d
 * (src/points_in_boxes_cuda.cu:24-49) says so, evaluated as the same float expressions: centre z = bottom + h/2, |z - cz| > h/2 rejects,
 * angle rz + pi/2, strict |local x| < l/2, |local y| < w/2.  Results are bit-identical to the reference kernels'.
 *
 * sstb200_points_in_boxes: pts [batch, num_pts, 3], boxes [batch, num_boxes, 7] (sample b's points against sample b's boxes).
 * mode SSTB200_PIB_FIRST (points_in_boxes_gpu): out int32 [batch, num_pts] = the LOWEST box index containing the point, else -1.
 * mode SSTB200_PIB_ALL (points_in_boxes_batch): out int32 [batch, num_pts, num_boxes] = 1 inside, else 0.
 * Every entry is written (no fill needed); zero-size boxes contain nothing.  No atomics, no sync.  Errors: negative sizes or an unknown
 * mode (SSTB_ERR_ARG); more than 786432 boxes per sample in ALL mode (SSTB_ERR_UNSUPPORTED). */
#define SSTB200_PIB_FIRST 0
#define SSTB200_PIB_ALL 1
int sstb200_points_in_boxes(sstb200_ctx* ctx, const float* pts, const float* boxes, int batch, int num_pts, int num_boxes, int mode,
                            int32_t* out);

/* RoIAwarePool3d (roiaware_pool3d.py:24-86, src/roiaware_pool3d_kernel.cu), in two calls on one context:
 *
 * sstb200_roiaware_pool3d_plan: rois [num_rois, 7], pts [num_pts, 3]; rois_batch / pts_batch int32 batch ids (>= 0) or both NULL (one
 * sample): a point pairs only with the RoIs of its own batch id, so one call covers every sample.  out_size = (ox, oy, oz), each in
 * [1, 255]; max_pts_per_voxel = m >= 1.  Finds the (RoI, point) pairs and syncs the stream once: *num_pairs_host = P, their number.
 * What it computed stays in the context's scratch arena for sstb200_roiaware_pool3d_forward, which must be the next call on the context.
 * Errors: negative sizes, out_size outside [1, 255], m < 1, a negative batch id (SSTB_ERR_ARG); RoI, voxel and point indices that do
 * not fit one 64-bit key, or P >= 2^31 (SSTB_ERR_UNSUPPORTED).
 *
 * sstb200_roiaware_pool3d_forward: pts_feature [num_pts, channels] fp32, mode SSTB200_POOL3D_MAX or _AVG.  A point inside RoI r falls in
 * voxel (x, y, z) = int((local x + l/2) / (l/ox)), int((local y + w/2) / (w/oy)), int((z - z_bottom) / (h/oz)) (fp32, each clamped to
 * [0, o - 1]); every voxel keeps its first m - 1 points in ascending point index (the reference's buffer holds a counter in slot 0).
 * max: from -inf, strict `>` in ascending point order (argmax = the first point reaching the maximum; NaN / -inf are never selected);
 * avg: sequential fp32 sum in ascending point order / count.  pooled [num_rois, ox, oy, oz, channels] is dense and fully written; a voxel
 * without a selected point writes 0.  The state the backward needs is compact, in caller buffers of capacity P (P + 1 offsets):
 *   voxel_slot int64   occupied voxels, ascending r * ox*oy*oz + (x * oy + y) * oz + z;
 *   voxel_offsets      int32 CSR over them into point_idx;
 *   point_idx int32    kept point indices, ascending within a voxel;
 *   argmax int32       [occupied, channels] (max mode only; NULL for avg), -1 where nothing was selected;
 *   counts_dev int32[2] (device): occupied voxels, kept points.
 * Deterministic; no sync.
 *
 * sstb200_roiaware_pool3d_backward: grad_out [num_rois, ox, oy, oz, channels] -> grad_in [num_pts, channels], fully written.  max: the
 * grad_out of every (voxel, channel) whose argmax is the point; avg: grad_out * (1 / max(count, 1)) of every voxel that kept the point.
 * Each point's terms are summed in (RoI, voxel) order without atomics, so two runs are bit-identical (the reference adds them with
 * float atomics).  num_pairs = the plan's P, with the state written by the forward.  No sync. */
#define SSTB200_POOL3D_MAX 0
#define SSTB200_POOL3D_AVG 1
int sstb200_roiaware_pool3d_plan(sstb200_ctx* ctx, const float* rois, const int32_t* rois_batch, int num_rois, const float* pts,
                                 const int32_t* pts_batch, int num_pts, const int32_t out_size[3], int max_pts_per_voxel,
                                 int64_t* num_pairs_host);
int sstb200_roiaware_pool3d_forward(sstb200_ctx* ctx, const float* pts_feature, int channels, int mode, float* pooled, int64_t* voxel_slot,
                                    int32_t* voxel_offsets, int32_t* point_idx, int32_t* argmax, int32_t* counts_dev);
int sstb200_roiaware_pool3d_backward(sstb200_ctx* ctx, int num_pts, int channels, int mode, int64_t num_pairs, const int64_t* voxel_slot,
                                     const int32_t* voxel_offsets, const int32_t* point_idx, const int32_t* argmax,
                                     const int32_t* counts_dev, const float* grad_out, float* grad_in);

/* ---- Deformable convolution: mmcv 1.3.8-1.4.0 deform_conv2d (DeformConv2d / DeformConv2dPack = 'DCN'), as CenterHead's DCNSeparateHead
 * (mmdet3d/models/dense_heads/centerpoint_head.py:124-238) runs it.  fp32 only, FFMA.
 * geom (15 int32) = N, Cin, H, W, Cout, kh, kw, stride h, stride w, pad h, pad w, dilation h, dilation w, groups, deform_groups.
 * x [N, Cin, H, W], offset [N, 2 dg kh kw, Ho, Wo], weight [Cout, Cin / groups, kh, kw], y / grad_y [N, Cout, Ho, Wo], all contiguous fp32,
 * Ho = (H + 2 ph - (dh (kh - 1) + 1)) / sh + 1 and the same for Wo.
 * y[n, o, ho, wo] = sum over c in o's group and taps (i, j) of W[o, c mod Cin/groups, i, j] * S(n, c, p), with
 *   p_h = (float)(ho sh - ph + i dh) + offset[n, 2K g + 2 (i kw + j), ho, wo],  p_w = (float)(wo sw - pw + j dw) + offset[.., + 1, ..],
 *   g = c / (Cin / dg), K = kh kw; S = 0 unless -1 < p_h < H and -1 < p_w < W, else the bilinear blend of the corners floor(p) and
 *   floor(p) + 1, a corner outside the image counting 0.  Zero offsets give a grouped conv2d.
 * sstb200_dcn_forward: y fully written; temporaries (x transposed to NHWC) from the context arena.  No sync.
 * sstb200_dcn_backward: grad_x = the transpose of the sampling, grad_offset = sum_c grad_col dS/dp with the corners held at floor(p) (the
 *   forward difference at an integer p; 0 outside the open domain), grad_weight = sum over (n, ho, wo) of grad_y S.  Any of the three may be
 *   NULL (not computed); the others are fully written.  Caller-owned workspace of sstb200_dcn_backward_workspace_bytes(geom) bytes; no
 *   float atomics, so two calls give bit-identical results.  No sync.
 * Errors: a size < 1, negative padding, Cin or Cout not divisible by groups, Cin not by dg, a kernel larger than the padded input
 * (SSTB_ERR_ARG); 4 N dg K Ho Wo reaching 2^32, N dg H W reaching 2^32 - 1, N > 65535, groups * ceil(Cin / groups * K / 16) or
 * groups * ceil(Cout / groups / 16) above 65535 (SSTB_ERR_UNSUPPORTED); a short workspace (SSTB_ERR_WORKSPACE).  The backward and its
 * workspace query sort the M = 4 N dg K Ho Wo sample corners with an int item count, so they also refuse M >= 2^31 (SSTB_ERR_UNSUPPORTED);
 * the forward does not sort and keeps the 2^32 limit. */
int sstb200_dcn_forward(sstb200_ctx* ctx, const int32_t geom[15], const float* x, const float* offset, const float* weight, float* y);
int sstb200_dcn_backward_workspace_bytes(sstb200_ctx* ctx, const int32_t geom[15], int64_t* bytes);
int sstb200_dcn_backward(sstb200_ctx* ctx, const int32_t geom[15], const float* x, const float* offset, const float* weight,
                         const float* grad_y, void* workspace, int64_t workspace_bytes, float* grad_x, float* grad_offset,
                         float* grad_weight);

/* ---- CenterHead training (mmdet3d/models/dense_heads/centerpoint_head.py:421-610), fp32, stream-ordered, no sync.
 *
 * sstb200_centerpoint_targets: CenterHead.get_targets for the whole batch and every task in three launches.
 *   boxes [N, box_dim] gravity-centred (x, y, z, dx, dy, dz, yaw[, vx, vy]), box_dim 7 or 9, labels int64 [N], the samples' boxes
 *   concatenated: sample b owns rows [sample_offsets[b], sample_offsets[b + 1]) (host, batch + 1 entries, sample_offsets[0] = 0).
 *   Task t owns the labels [task_label_offsets[t], task_label_offsets[t + 1]) (host, num_tasks + 1 entries, each range non-empty);
 *   other labels are ignored.  Geometry: pc_min (x, y), voxel_size (x, y), out_size_factor, the feature map width x height,
 *   gaussian_overlap, min_radius, max_objs, norm_bbox.  Outputs per task t (host arrays of num_tasks device pointers), fully written:
 *     heatmaps[t] f32 [batch, ncls_t, height, width], anno_boxes[t] f32 [batch, max_objs, 10], inds[t] int64 [batch, max_objs],
 *     masks[t] uint8 [batch, max_objs].
 *   A task's boxes take slots ordered by class within the task, then by input row; only the first max_objs are considered.  A box is
 *   skipped (its slot keeps ind 0, mask 0, anno_box 0) when dx / vx / osf <= 0 or dy / vy / osf <= 0 or trunc((x - pc_min) / voxel /
 *   osf) lies outside the map; every quantity is the reference's sequence of correctly rounded fp32 operations (gaussian_radius with
 *   the Python scalars 1 - o, 1 + o, -2 o, o - 1 and 4 (4 o) rounded to fp32), radius = max(min_radius, trunc(min(r1, r2, r3))).
 *   ind = cy * width + cx, anno_box = (x_map - cx, y_map - cy, z, log(dims) or dims, sin(yaw), cos(yaw), vx, vy), zeros for 7-dim boxes.
 *   The heatmap is the max over the drawn boxes of fp32(exp(-(dx^2 + dy^2) / (2 sigma^2))) in double, sigma = (2 r + 1) / 6, over the
 *   window clipped to the map; two calls give bit-identical results.  Temporaries (16 bytes per slot) from the context arena.
 *   Errors: box_dim not 7 or 9, a size < 1, non-monotone offsets, an empty task range, a NULL pointer (SSTB_ERR_ARG); more than 256
 *   samples or 16 tasks, height * width or batch * num_tasks * max_objs reaching 2^31 (SSTB_ERR_UNSUPPORTED).
 *
 * sstb200_gaussian_focal_loss_forward: mmdet 2.14 GaussianFocalLoss (alpha 2, gamma 4, reduction 'mean') on p = clamp(sigmoid(logits),
 *   1e-4, 1 - 1e-4) against target, both [n]: *loss = loss_weight * sum / max(num_pos, 1), *num_pos = the number of targets equal to 1
 *   (both device f32 scalars).  The clamp keeps NaN, as torch.clamp does: a NaN logit makes the loss NaN.  Block partials in double,
 *   then one block sums them in a fixed order: deterministic.  Two launches, partials from the context arena.
 * sstb200_gaussian_focal_loss_backward: grad_logits [n] = grad_loss[0] * loss_weight / max(num_pos[0], 1) * d loss / d logit, recomputed
 *   from (logits, target); the clamp passes the gradient where the sigmoid lies within its bounds inclusive (as torch.clamp), and a
 *   NaN logit gets a NaN gradient.  One launch.
 *   Errors (both): n < 1 or a NULL pointer (SSTB_ERR_ARG).
 *
 * sstb200_centerpoint_l1_loss_forward: mmdet 2.14 L1Loss (reduction 'mean') of CenterHead.loss: heads = (reg [B, 2, H, W], height
 *   [B, 1, H, W], dim [B, 3, H, W], rot [B, 2, H, W], vel [B, 2, H, W]) read in place at ind, against anno_box [B, max_objs, 10], weight
 *   mask * (target not NaN) * code_weights[c]; *loss = loss_weight * sum(|pred - target| weight) / (sum(mask) + 1e-4) (device f32,
 *   avg factor in fp32 on the device).  Every slot is gathered, as in the reference: a masked-out slot adds |pred - target| * 0, so a
 *   NaN prediction at its ind, or an ind outside [0, H W) of any slot, makes the loss NaN; a NaN target does too.  One launch.
 * sstb200_centerpoint_l1_loss_backward: grad_heads (same shapes as heads) fully written: zero, except at each masked cell the sum over
 *   the slots gathering it, in slot order, of grad_loss[0] * loss_weight / avg * weight * sign(pred - target) (0 for a NaN target or
 *   a NaN difference, as torch.sign).  No float atomics, two calls give bit-identical results.  Two launches.
 *   Errors (both): a size < 1 or a NULL pointer (SSTB_ERR_ARG); max_objs above 4096 (SSTB_ERR_UNSUPPORTED). */
int sstb200_centerpoint_targets(sstb200_ctx* ctx, const float* boxes, const int64_t* labels, int box_dim, const int32_t* sample_offsets,
                                int batch, const int32_t* task_label_offsets, int num_tasks, const float pc_min[2],
                                const float voxel_size[2], int out_size_factor, int width, int height, double gaussian_overlap,
                                int min_radius, int max_objs, int norm_bbox, float* const* heatmaps, float* const* anno_boxes,
                                int64_t* const* inds, uint8_t* const* masks);
int sstb200_gaussian_focal_loss_forward(sstb200_ctx* ctx, const float* logits, const float* target, int64_t n, float loss_weight,
                                        float* loss, float* num_pos);
int sstb200_gaussian_focal_loss_backward(sstb200_ctx* ctx, const float* logits, const float* target, int64_t n, float loss_weight,
                                         const float* num_pos, const float* grad_loss, float* grad_logits);
int sstb200_centerpoint_l1_loss_forward(sstb200_ctx* ctx, const float* const heads[5], int batch, int height, int width,
                                        const float* anno_box, const int64_t* ind, const uint8_t* mask, int max_objs,
                                        const float code_weights[10], float loss_weight, float* loss);
int sstb200_centerpoint_l1_loss_backward(sstb200_ctx* ctx, const float* const heads[5], int batch, int height, int width,
                                         const float* anno_box, const int64_t* ind, const uint8_t* mask, int max_objs,
                                         const float code_weights[10], float loss_weight, const float* grad_loss,
                                         float* const grad_heads[5]);

/* ---- Anchor3DHead training (mmdet3d/models/dense_heads/anchor3d_head.py:197-379, train_mixins.py), fp32, stream-ordered, no sync.
 *
 * sstb200_anchor3d_targets: anchor_target_3d of one level with one MaxIoUAssigner per anchor size (BboxOverlapsNearest3D,
 *   ignore_iof_thr -1, match_low_quality), PseudoSampler, DeltaXYZWLHRBBoxCoder (code_size 7) and get_direction_target, for every
 *   sample and size in a fixed number of launches (seven).
 *   Anchors (AlignedAnchor3DRangeGenerator, never materialised): anchor ((y W + x) S + s) R + r = (x_centers[x], y_centers[y],
 *   size_z[s], size_wlh[s][0..2], rotations[r]), device arrays [W], [H], [S], [S, 3], [R].  GT boxes [N, 7] bottom-centre (x, y, z, w,
 *   l, h, yaw) and labels int64 [N], the samples concatenated: sample b owns rows [sample_offsets[b], sample_offsets[b + 1]) (host,
 *   batch + 1 entries).  Per size s (host arrays): pos_iou_thr, neg_iou_thr, min_pos_iou (compared as fp32), gt_max_assign_all.
 *   assign_per_class: size s sees only the GTs labelled s.
 *   Assignment (mmdet 2.14 MaxIoUAssigner.assign_wrt_overlaps, IoU(gt, anchor)), per sample and size:
 *     - an anchor with max IoU >= 0 and < neg_iou_thr gets 0 (negative); every other anchor starts at -1 (ignored);
 *     - an anchor with max IoU >= pos_iou_thr gets argmax + 1, the argmax being the first GT on ties;
 *     - then for each GT i in order whose max IoU over the anchors is >= min_pos_iou, every anchor whose IoU with i equals that max gets
 *       i + 1 (only the first such anchor when gt_max_assign_all is 0).  Later GTs overwrite earlier ones; this overrides the first two
 *       rules.
 *     - with no GT (of its class, under assign_per_class) every anchor of the size is negative.
 *   IoU = mmdet bbox_overlaps of the nearest BEV boxes (lidar_box3d.py nearest_bev: w and l swapped when |limit_period(yaw, 0.5, pi)|
 *   > pi / 4), every operation a correctly rounded fp32 one with pi and pi / 4 rounded to fp32, no FMA contraction:
 *   overlap / max(area_gt + area_anchor - overlap, 1e-6).  Per-GT maxima combine by an integer max on the fp32 bits, so two calls give
 *   bit-identical results.  Boxes must be finite.
 *   Outputs [batch, A] in the anchor order above (A = H W S R), fully written:
 *     labels int64 (the GT's label for positives, num_classes otherwise), label_weights f32 (1 for positive and negative, 0 for
 *     ignored), bbox_targets / bbox_weights f32 [batch, A, 7] (encode(anchor, gt) and 1 for positives, else 0), dir_targets int64 /
 *     dir_weights f32 (clamp(floor(limit_period(rt + ra - dir_offset, 0, 2 pi) / pi), 0, 1) and 1 for positives, else 0), and the
 *     device scalar num_total_pos int64 = sum over samples of max(positives, 1).  Temporaries (12 bytes per anchor and sample, 8 per GT
 *     and size) from the context arena.
 *   Errors: a NULL pointer, a size < 1, non-monotone offsets (SSTB_ERR_ARG); more than 256 samples, 8 sizes or 8 rotations, more than
 *   4096 GTs in a sample, batch A reaching 2^28 (SSTB_ERR_UNSUPPORTED).
 *
 * sstb200_anchor_focal_loss_forward: mmdet 2.14 FocalLoss(use_sigmoid, gamma 2, alpha 0.25) of cls_score [B, A_loc C, H, W] (read in
 *   place; element (b, y, x, a, c) is channel a C + c, anchor (y W + x) A_loc + a) against one-hot(labels) [B, A] with background
 *   num_classes, weighted by label_weights [B, A]: *loss = loss_weight * sum / num_total_pos (device int64).  Log-sigmoid is the stable
 *   softplus form of mmdet's py_sigmoid_focal_loss: it stays exact for logits of any size, where mmcv's CUDA kernel clamps
 *   log(max(1 - p, FLT_MIN)) and so saturates near 87 for logits beyond about +-17.  A NaN logit makes the loss NaN.  An infinite logit
 *   follows the closed form: on its label's side (+inf for the target class, -inf otherwise) loss 0 and gradient 0, on the other side
 *   loss inf and gradient NaN; mmdet's Python path gives NaN for both.  Block partials in double summed in a fixed order:
 *   deterministic.  Two launches, partials from the context arena.
 * sstb200_anchor_focal_loss_backward: grad_cls_score (same shape) = grad_loss[0] * loss_weight / num_total_pos * label_weight * d loss /
 *   d logit, recomputed from the logits in one elementwise pass; NaN only at a NaN logit.
 *
 * sstb200_anchor_reg_dir_loss_forward: over the positives (0 <= label < num_classes) only.  bbox_pred [B, A_loc 7, H, W] and
 *   dir_cls_preds [B, A_loc 2, H, W] read in place.  loss_bbox = loss_weight_bbox * sum |pred - target| * bbox_weight * code_weight /
 *   num_total_pos, channel 6 compared as sin(p) cos(t) against cos(p) sin(t) (add_sin_difference); loss_dir = loss_weight_dir *
 *   sum dir_weight * (logsumexp(z) - z[dir_target]) / num_total_pos.  No positives: both 0.  Two launches.
 * sstb200_anchor_reg_dir_loss_backward: grad_losses = (d / d loss_bbox, d / d loss_dir) on the device; grad_bbox_pred / grad_dir_cls_preds
 *   fully written, zero off the positives: each positive owns its cells' channels, so there are no atomics.  sign(0) = sign(NaN) = 0, as
 *   torch.abs' gradient: a NaN box coordinate gets gradient 0.  The yaw channel's derivative goes through both sin(p) cos(t) and cos(p)
 *   sin(t), their products rounded apart as torch rounds them: a yaw equal to its target gets gradient 0, a NaN yaw a NaN gradient.  One
 *   launch.
 *   Errors (all four): a NULL pointer or a size < 1 (SSTB_ERR_ARG). */
int sstb200_anchor3d_targets(sstb200_ctx* ctx, const float* x_centers, int width, const float* y_centers, int height, const float* size_z,
                             const float* size_wlh, int num_sizes, const float* rotations, int num_rots, const float* gt_boxes,
                             const int64_t* gt_labels, const int32_t* sample_offsets, int batch, const float* pos_iou_thr,
                             const float* neg_iou_thr, const float* min_pos_iou, const int32_t* gt_max_assign_all, int assign_per_class,
                             int num_classes, float dir_offset, int64_t* labels, float* label_weights, float* bbox_targets,
                             float* bbox_weights, int64_t* dir_targets, float* dir_weights, int64_t* num_total_pos);
int sstb200_anchor_focal_loss_forward(sstb200_ctx* ctx, const float* cls_score, int batch, int num_anchors, int num_classes, int height,
                                      int width, const int64_t* labels, const float* label_weights, const int64_t* num_total_pos,
                                      float loss_weight, float* loss);
int sstb200_anchor_focal_loss_backward(sstb200_ctx* ctx, const float* cls_score, int batch, int num_anchors, int num_classes, int height,
                                       int width, const int64_t* labels, const float* label_weights, const int64_t* num_total_pos,
                                       float loss_weight, const float* grad_loss, float* grad_cls_score);
int sstb200_anchor_reg_dir_loss_forward(sstb200_ctx* ctx, const float* bbox_pred, const float* dir_cls_preds, int batch, int num_anchors,
                                        int num_classes, int height, int width, const int64_t* labels, const float* bbox_targets,
                                        const float* bbox_weights, const int64_t* dir_targets, const float* dir_weights,
                                        const float code_weight[7], const int64_t* num_total_pos, float loss_weight_bbox,
                                        float loss_weight_dir, float* loss_bbox, float* loss_dir);
int sstb200_anchor_reg_dir_loss_backward(sstb200_ctx* ctx, const float* bbox_pred, const float* dir_cls_preds, int batch, int num_anchors,
                                         int num_classes, int height, int width, const int64_t* labels, const float* bbox_targets,
                                         const float* bbox_weights, const int64_t* dir_targets, const float* dir_weights,
                                         const float code_weight[7], const int64_t* num_total_pos, float loss_weight_bbox,
                                         float loss_weight_dir, const float* grad_losses, float* grad_bbox_pred,
                                         float* grad_dir_cls_preds);

/* ---- VoteSegHead training (mmdet3d/models/decode_heads/segmentation_head.py), fp32, stream-ordered, no sync.
 *
 * sstb200_voteseg_targets: get_targets (lines 212-283, centroid_offset and extra_width unset) for the whole batch in one launch.
 *   points [N, >= 3] fp32 with row stride point_stride (floats), the samples concatenated: sample b owns rows
 *   [point_offsets[b], point_offsets[b + 1]).  gt_boxes [G, 7] bottom-centre LiDAR boxes and gt_labels int64 [G], sample b owning rows
 *   [gt_offsets[b], gt_offsets[b + 1]).  Both offset arrays are host arrays of batch + 1 entries.
 *   A point takes the label of the lowest-index box of its own sample that contains it, boxes with a negative label skipped (the
 *   reference's valid_gt_mask filter, line 229, then points_in_boxes_gpu's first hit).  The in-box test is sstb200_points_in_boxes'
 *   (box3d.cuh), so it is bit-identical to the reference kernel.  Its vote target is encode_vote_targets(gravity_center - point) with the
 *   reference's fp32 expressions: centre z = z + h * 0.5, the subtraction, then sign(d) * sqrt(|d|) with an IEEE square root; the
 *   results are bit-exact.  A point in no box (so every point of a sample with no valid GT, lines 231-234) gets bg_label (num_classes:
 *   the background column of a sigmoid head, the last of the num_classes + 1 logits of a softmax head), vote target 0 and mask 0.
 *   Outputs labels int64 [N], vote_targets f32 [N, 3] and vote_mask uint8 [N] (0 / 1), every entry written.  GTs are staged in shared
 *   memory 256 at a time and a point stops at its first hit.  No temporaries.
 *   Errors: a NULL pointer, batch < 1, stride < 3, offsets that do not start at 0 or decrease (SSTB_ERR_ARG); more than 256 samples or
 *   more than 4096 GTs in one sample (SSTB_ERR_UNSUPPORTED).
 *
 * sstb200_voteseg_loss_forward: `losses` (lines 107-173) in one read of every point's row.  seg_logits [N, C] (row stride logit_stride)
 *   and vote_preds [N, 3 C] (row stride vote_stride, class-major: class c owns channels 3 c .. 3 c + 2) are read in place; labels int64
 *   [N], vote_targets f32 [N, 3] contiguous, vote_mask uint8 [N].  Every logit is first multiplied by cfg->logit_scale (line 116).
 *   - use_softmax 0: mmdet 2.14 FocalLoss(use_sigmoid=True, gamma, alpha) against one-hot(label) without the background column
 *     (label C), reduction 'mean' without avg_factor: losses[0] = loss_weight * sum / (N C).  The log-sigmoid is the stable softplus form
 *     of py_sigmoid_focal_loss, exact for logits of any size; mmcv's CUDA kernel instead clamps log(max(1 - p, FLT_MIN)) and so saturates
 *     near 87 for logits beyond about +-17.  An infinite logit follows the closed form: on its label's side loss 0 and gradient 0, on
 *     the other loss inf and gradient NaN, where mmdet's Python path gives NaN for both.  gamma must be >= 1.
 *   - use_softmax 1: mmseg CrossEntropyLoss(use_sigmoid=False, class_weight): losses[0] = loss_weight * sum w[y] (logsumexp(x) - x[y]) / N,
 *     divided by N and not by the sum of the weights (F.cross_entropy(reduction='none') then weight_reduce_loss, mmseg 0.14.1 to 1.0,
 *     avg_non_ignore False).  class_weight: host [C], NULL for ones.  Labels come from get_targets and are never 255 or -100, so
 *     ignore_index plays no part.
 *   - vote loss: mmdet 2.14 L1Loss over the valid points (mask 1): losses[1] = loss_weight_vote * sum |vote_preds[i, 3 y + k] -
 *     vote_targets[i, k]| / (3 n_valid), n_valid counted and divided on the device and written to *num_valid (int64).  Only the three
 *     channels of a valid point's own class are read.  With no valid point losses[1] = vote_preds.sum() * 0 as in the reference (line
 *     142): 0, or NaN when any vote prediction is not finite (an fp32 overflow of the sum of finite predictions is not reproduced).  A
 *     third launch reads the device n_valid and scans the whole vote tensor for that only when n_valid is 0.
 *   - training-log counts (lines 146-171), int64 [2 E + 1]: tp[e] (E entries), real[e], then num_fg.  Group g predicts a point when
 *     its score exceeds group_thresh[g] (compared in fp32); the score is the sum over the classes in group_masks[g] (bit c = class c) of
 *     sigmoid(x) (use_softmax 0) or of the softmax probabilities (use_softmax 1).  tp[e] counts the points of class entry_class[e]
 *     that group entry_group[e] predicts, real[e] the points of class entry_class[e], num_fg the sum over groups of the points each
 *     predicts.  The recall quotients are left to the caller.  The reference's host asserts (lines 124-127, 134-135) are not made.
 *   - NaN: a NaN logit makes losses[0] NaN, and a NaN vote prediction that is read makes losses[1] NaN.  A label outside [0, C] (sigmoid)
 *     or [0, C) (softmax), or a valid point whose label is not below C, makes the loss NaN instead of reading out of bounds.
 *   Block partials (double sums, integer counts) summed in a fixed order: deterministic.  Three launches, partials from the context arena.
 * sstb200_voteseg_loss_backward: grad_losses (d / d losses[0], d / d losses[1], device) -> grad_logits [N, C] and grad_vote_preds
 *   [N, 3 C], both contiguous and fully written.  Each point writes only its own row, with no atomics: two calls are bit-identical.
 *   d logit = logit_scale * loss_weight / (N C) (sigmoid) or loss_weight w[y] / N (softmax) times the element's derivative, recomputed
 *   from the logits.  A NaN logit makes its own gradient NaN (its whole row in softmax mode) and no other.  The vote gradient is
 *   loss_weight_vote * sign(pred - target) / (3 n_valid) on the three channels of a valid point's own class, sign(0) = sign(NaN) = 0 as
 *   torch.abs' gradient, and 0 everywhere else; with no valid point it is all zeros.  One launch.
 *   Errors (both): a NULL pointer, N < 1, C < 1, a row stride below the row, a group or entry out of range (SSTB_ERR_ARG); more than 64
 *   classes, 64 groups or 64 entries, a focal gamma below 1 (SSTB_ERR_UNSUPPORTED). */
typedef struct {
  int32_t num_classes;           /* C: logit columns (num_classes + 1 for a softmax head) */
  int32_t use_softmax;           /* 0: sigmoid focal loss, 1: softmax cross-entropy */
  float gamma, alpha;            /* focal loss */
  float logit_scale;
  float loss_weight;             /* loss_decode */
  float loss_weight_vote;        /* loss_vote */
  const float* class_weight;     /* host [C] or NULL (softmax) */
  int32_t num_groups;            /* G <= 64 */
  const uint64_t* group_masks;   /* host [G] */
  const float* group_thresh;     /* host [G] */
  int32_t num_entries;           /* E <= 64 */
  const int32_t* entry_group;    /* host [E] */
  const int32_t* entry_class;    /* host [E] */
} sstb200_voteseg_cfg;
int sstb200_voteseg_targets(sstb200_ctx* ctx, const float* points, int64_t point_stride, const int32_t* point_offsets,
                            const float* gt_boxes, const int64_t* gt_labels, const int32_t* gt_offsets, int batch, int bg_label,
                            int64_t* labels, float* vote_targets, uint8_t* vote_mask);
int sstb200_voteseg_loss_forward(sstb200_ctx* ctx, const sstb200_voteseg_cfg* cfg, const float* seg_logits, int64_t logit_stride,
                                 const float* vote_preds, int64_t vote_stride, int64_t num_points, const int64_t* labels,
                                 const float* vote_targets, const uint8_t* vote_mask, float* losses, int64_t* num_valid, int64_t* counts);
int sstb200_voteseg_loss_backward(sstb200_ctx* ctx, const sstb200_voteseg_cfg* cfg, const float* seg_logits, int64_t logit_stride,
                                  const float* vote_preds, int64_t vote_stride, int64_t num_points, const int64_t* labels,
                                  const float* vote_targets, const uint8_t* vote_mask, const int64_t* num_valid, const float* grad_losses,
                                  float* grad_logits, float* grad_vote_preds);

/* ---- SparseClusterHeadV2 training (mmdet3d/models/dense_heads/sparse_cluster_head{,_v2}.py), fp32, stream-ordered, no sync.
 *
 * sstb200_cluster_head_targets: get_targets of every task (v2 lines 299-405 after modify_gt_for_single_task, assign_single of v1 lines
 *   364-397 with enlarge_width unset, assign_by_dist unset) for the whole batch in one launch.
 *   cluster_xyz [M, >= 3] fp32 with row stride xyz_stride (floats); batch_idx int64 [M] with element stride batch_stride (column 1 of
 *   cluster_inds [M, 3] is batch_idx = cluster_inds + 1, stride 3).  Clusters need not be sorted by sample.  gt_boxes [G, 7] bottom-centre
 *   LiDAR boxes and gt_labels int64 [G] (global class ids), sample b owning rows [gt_offsets[b], gt_offsets[b + 1]) (host, batch + 1).
 *   class_task / class_rank (host [num_classes]): the task of each global class and its position in that task's class list, task -1
 *   for a class in no task.  task_classes (host [num_tasks]): C_t.
 *   Per task t a cluster takes the GT of its own sample that contains it with the smallest (class rank, GT index): the first hit of
 *   points_in_boxes_gpu over modify_gt_for_single_task's list, which concatenates the task's classes in order and keeps the input order
 *   within a class.  A GT with a negative label or a class in no task takes part in no task.  The in-box test is sstb200_points_in_boxes'
 *   (box3d.cuh), bit-identical to the reference kernel.
 *   Outputs, per task t: labels[t] int64 [M] = the rank of the hit's class, C_t (background) without a hit; bbox_targets[t] f32 [M, 8] =
 *   BasePointBBoxCoder.encode (xyz - cluster xyz, exact in fp32; log(dims + 1e-6) with the addition in fp32; sin(yaw), cos(yaw)), the
 *   three transcendentals in double rounded once, zeros on negatives; num_pos int64 [T] (device) = the positives of each task.
 *   A cluster whose batch index is outside [0, batch) gets label -1 and NaN targets in every task (the reference's boolean split would
 *   give it no sample and a zero row), so the classification loss is NaN.  Every entry is written.
 *   Errors: a NULL pointer, batch < 1, a stride below the row, offsets that do not start at 0 or decrease, a class mapped outside its
 *   task (SSTB_ERR_ARG); more than 256 samples, 8 tasks, 64 classes or 4096 GTs in one sample (SSTB_ERR_UNSUPPORTED).
 *
 * sstb200_cluster_head_loss_forward: loss_single_task of every task (v2 lines 192-297) in one launch sequence.  Per task t,
 *   cls_logits[t] [M, C_t] and reg_preds[t] [M, 8] are read in place with row strides logit_strides[t] / reg_strides[t]; labels[t],
 *   bbox_targets[t] and num_pos from sstb200_cluster_head_targets; cls_avg_factor and reg_avg_factor fp32 [T] on the device.
 *   losses f32 [T, 4] = (cls, center, size, rot) with
 *   - cls: loss_weight_cls * sum focal / cls_avg_factor[t], mmdet 2.14 FocalLoss(use_sigmoid=True, gamma, alpha) against one-hot(label)
 *     without the background column C_t, label_weights all ones, in the stable softplus form (see sstb200_voteseg_loss_forward for the
 *     difference from mmcv's clamped CUDA kernel, and for its infinite logits).  A label outside [0, C_t] makes it NaN.  gamma must be >= 1.
 *   - center / size / rot: loss_weight_q * sum over the positives (0 <= label < C_t) of L1 |d| or, with smooth_l1, mmdet's SmoothL1
 *     (|d| < beta ? 0.5 d^2 / beta : |d| - 0.5 beta) on columns [0, 3), [3, 6), [6, 8), over reg_avg_factor[t].  When the local
 *     num_pos[t] is 0 they are exactly 0 whatever the factor (the reference's `num_pos > 0` branch takes pos_reg_preds.sum() * 0).
 *   Block partials in double summed in a fixed order: deterministic.  Two launches, partials from the context arena.
 * sstb200_cluster_head_loss_backward: grad_losses (device [T, 4]) -> grad_logits[t] [M, C_t] and grad_reg_preds[t] [M, 8], contiguous
 *   and fully written; each cluster writes only its own rows, with no atomics, so two calls are bit-identical.  A NaN logit makes its own
 *   gradient NaN and no other; the reg gradient is 0 off the positives and for a task with no local positive.  One launch.
 *   Errors (both): a NULL pointer, M < 1, a row stride below the row, C_t < 1, SmoothL1 with beta <= 0 (SSTB_ERR_ARG); more than 8
 *   tasks or 64 classes in a task, a gamma below 1 (SSTB_ERR_UNSUPPORTED). */
typedef struct {
  float gamma, alpha;                  /* focal loss */
  int32_t smooth_l1;                   /* 0: L1Loss, 1: SmoothL1Loss(beta) for center, size and rot */
  float beta;
  float loss_weight_cls, loss_weight_center, loss_weight_size, loss_weight_rot;
} sstb200_cluster_head_loss_cfg;
int sstb200_cluster_head_targets(sstb200_ctx* ctx, const float* cluster_xyz, int64_t xyz_stride, const int64_t* batch_idx,
                                 int64_t batch_stride, int64_t num_clusters, const float* gt_boxes, const int64_t* gt_labels,
                                 const int32_t* gt_offsets, int batch, int num_classes, const int32_t* class_task, const int32_t* class_rank,
                                 int num_tasks, const int32_t* task_classes, int64_t* const* labels, float* const* bbox_targets,
                                 int64_t* num_pos);
int sstb200_cluster_head_loss_forward(sstb200_ctx* ctx, const sstb200_cluster_head_loss_cfg* cfg, int num_tasks, int64_t num_clusters,
                                      const float* const* cls_logits, const int64_t* logit_strides, const int32_t* task_classes,
                                      const float* const* reg_preds, const int64_t* reg_strides, int64_t* const* labels,
                                      float* const* bbox_targets, const int64_t* num_pos, const float* cls_avg_factor,
                                      const float* reg_avg_factor, float* losses);
int sstb200_cluster_head_loss_backward(sstb200_ctx* ctx, const sstb200_cluster_head_loss_cfg* cfg, int num_tasks, int64_t num_clusters,
                                       const float* const* cls_logits, const int64_t* logit_strides, const int32_t* task_classes,
                                       const float* const* reg_preds, const int64_t* reg_strides, int64_t* const* labels,
                                       float* const* bbox_targets, const int64_t* num_pos, const float* cls_avg_factor,
                                       const float* reg_avg_factor, const float* grad_losses, float* const* grad_logits,
                                       float* const* grad_reg_preds);

/* ---- FSDV2Head training (mmdet3d/models/dense_heads/fsd_v2_head.py): the cluster-head kernels above with centroid assignment and
 * velocity.  The three functions above are these with assign_xyz NULL, gt_width 7 and code_size 8, and give the same results bit for bit.
 *
 * sstb200_cluster_head_targets_ex: sstb200_cluster_head_targets plus
 *   - assign_xyz (NULL, or [M, >= 3] fp32 with row stride assign_stride): the points of the in-box test, train_cfg centroid_assign's
 *     aux_xyz (lines 359-362); the encode still subtracts cluster_xyz (line 382).  NULL tests cluster_xyz.
 *   - gt_width: the row width of gt_boxes, 7, 9 (with velocity, columns 7-8) or 10 (plus the copy-paste flag, column 9).
 *   - code_size 8 or 10.  With 10, bbox_targets[t] is f32 [M, 11]: columns 0-7 as above, 8-9 = the hit's GT columns 7-8, and column 10 =
 *     the velocity loss weight, GT column 9 for gt_width 10 (lines 383-388) and 1 for gt_width 9; all 11 are 0 on negatives and NaN for
 *     an out-of-range batch index.  With 8, bbox_targets[t] is [M, 8].
 *   Errors: those of sstb200_cluster_head_targets; code_size other than 8 / 10, code_size 10 with gt_width 7 (the reference's encode
 *   has no velocity to copy), code_size 8 with gt_width 9 / 10 (its encode asserts code_size == 10), assign_stride < 3 (SSTB_ERR_ARG).
 *
 * sstb200_cluster_head_loss_forward_ex / _backward_ex: sstb200_cluster_head_loss_forward / _backward with cfg->code_size.  With 8 they
 *   are those functions.  With 10, reg_preds[t] is [M, >= 10], bbox_targets[t] [M, 11] from sstb200_cluster_head_targets_ex, and losses
 *   f32 [T, 5] = (cls, center, size, rot, vel) with
 *   - vel: loss_weight_vel * sum over the positives of the L1 / SmoothL1 element (the type and beta of the other three) of columns
 *     [8, 10) times the target's column 10, over 2 * num_pos[t], the local count: loss_vel is called without avg_factor (lines 243-248),
 *     mmdet's reduction 'mean' over the [num_pos, 2] elements.  Exactly 0 when num_pos[t] is 0.
 *   The backward takes grad_losses [T, 5] and writes grad_reg_preds[t] [M, 10], contiguous; columns 8-9 are 0 where the weight is 0.
 *   Block partials in double summed in a fixed order as above; no atomics; deterministic.
 *   Errors: those of the functions above, and code_size other than 8 / 10 or a reg row stride below code_size (SSTB_ERR_ARG). */
typedef struct {
  float gamma, alpha;                  /* focal loss */
  int32_t smooth_l1;                   /* 0: L1Loss, 1: SmoothL1Loss(beta) for center, size, rot and vel */
  float beta;
  float loss_weight_cls, loss_weight_center, loss_weight_size, loss_weight_rot;
  float loss_weight_vel;               /* code_size 10 only */
  int32_t code_size;                   /* 8 or 10 */
} sstb200_cluster_head_loss_cfg_ex;
int sstb200_cluster_head_targets_ex(sstb200_ctx* ctx, const float* cluster_xyz, int64_t xyz_stride, const float* assign_xyz,
                                    int64_t assign_stride, const int64_t* batch_idx, int64_t batch_stride, int64_t num_clusters,
                                    const float* gt_boxes, int gt_width, const int64_t* gt_labels, const int32_t* gt_offsets, int batch,
                                    int num_classes, const int32_t* class_task, const int32_t* class_rank, int num_tasks,
                                    const int32_t* task_classes, int code_size, int64_t* const* labels, float* const* bbox_targets,
                                    int64_t* num_pos);
int sstb200_cluster_head_loss_forward_ex(sstb200_ctx* ctx, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks, int64_t num_clusters,
                                         const float* const* cls_logits, const int64_t* logit_strides, const int32_t* task_classes,
                                         const float* const* reg_preds, const int64_t* reg_strides, int64_t* const* labels,
                                         float* const* bbox_targets, const int64_t* num_pos, const float* cls_avg_factor,
                                         const float* reg_avg_factor, float* losses);
int sstb200_cluster_head_loss_backward_ex(sstb200_ctx* ctx, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks,
                                          int64_t num_clusters, const float* const* cls_logits, const int64_t* logit_strides,
                                          const int32_t* task_classes, const float* const* reg_preds, const int64_t* reg_strides,
                                          int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                                          const float* cls_avg_factor, const float* reg_avg_factor, const float* grad_losses,
                                          float* const* grad_logits, float* const* grad_reg_preds);

/* ---- FSD's second stage (mmdet3d/models/roi_heads/fsd_roi_head.py, bbox_heads/fsd_bbox_head.py,
 * core/bbox/samplers/iou_neg_piecewise_sampler.py), fp32, stream-ordered, no host sync.
 *
 * sstb200_roi_assign_sample: GroupCorrectionHead._assign_and_sample for every sample in one launch (one CTA per sample).
 *   proposals [P, prop_width] (7 or 9 columns, LiDAR bottom-centre) with predicted labels int64 [P], sample b owning rows
 *   [prop_offsets[b], prop_offsets[b + 1]) (host, batch + 1; every sample needs a proposal: the caller adds the reference's fake box);
 *   keys fp32 [P], one per proposal; gt_boxes [G, gt_width] (7, 9 or 10; columns 0-6 are used) and gt_labels int64 [G] with host
 *   gt_offsets.  per_class: proposal i is matched only against the GTs labelled plab[i] by assigner plab[i] (a label outside
 *   [0, num_classes) leaves it negative with IoU 0); otherwise one assigner over every GT.  Each assigner is mmdet 2.14
 *   MaxIoUAssigner.assign_wrt_overlaps with match_low_quality and gt_max_assign_all, over the 3-D IoU of
 *   LiDARInstance3DBoxes.overlaps (fp32, the BEV overlap of sstb200_boxes_overlap_bev).  The sampler is IoUNegPiecewiseSampler with
 *   neg_pos_ub < 0 and no GT proposals: at most num_pos (= int(num * pos_fraction)) positives, then num - positives negatives split
 *   into IoU pieces [piece_thrs[q + 1], piece_thrs[q]) (the last [0, piece_thrs[last])) with the reference's carry-over.  Where the
 *   reference calls random_choice(gallery, k) this keeps the k members with the smallest keys, ties to the lower index.
 *   Outputs: sample b's rows at [b * num, b * num + counts[2 b + 1]), positives (counts[2 b] of them) by ascending proposal index, then
 *   negatives by ascending index: out_inds (global proposal row), out_iou (max_overlaps), out_gt (global GT row, -1 on negatives),
 *   out_labels (the GT's label, -1 on negatives); counts int32 [batch, 2] on the device.  Temporaries from the context arena.
 *   Errors: a NULL pointer, a width other than the above, offsets that do not start at 0 or decrease, a sample without proposals
 *   (SSTB_ERR_ARG); more than 4096 proposals or GTs in a sample, more than 8 assigners or IoU pieces (SSTB_ERR_UNSUPPORTED).
 *
 * sstb200_roi_head_targets: FullySparseBboxHead.get_targets for all num_rows sampled rows in one launch.  rois [R, roi_width] the
 *   sampled proposals, iou / gt_rows / labels the rows of sstb200_roi_assign_sample (gt_rows index gt_boxes).  Outputs per row:
 *   soft_labels fp32 (get_multi_class_soft_label with cls_pos_thr / cls_neg_thr, host double [num_classes]: the compares take them
 *   in fp32 and the divisor is (float)(pos - neg) formed in double, as torch does with Python floats; 0 on negatives), reg_mask int64
 *   (1 on positives), bbox_targets fp32 [R, 7] (the canonical transform into the RoI's frame and DeltaXYZWLHRBBoxCoder.encode against
 *   the zero-centred RoI, in double, rounded once; 0 on negatives) and pos_gt_bboxes fp32 [R, 7] (the GT's columns 0-6; 0 on negatives).
 *
 * sstb200_roi_head_loss_forward: FullySparseBboxHead.loss in one launch sequence.  cls_score [R] and bbox_pred [R, 7] read with row
 *   strides; nonempty uint8 [R]; the targets above; labels the rows' GT labels; rois [R, roi_width] without the batch column;
 *   cls_avg_factor / reg_avg_factor fp32 [1] on the device.  losses fp32 [3] = (cls, bbox, corner):
 *   - cls: loss_weight_cls * sum over non-empty rows of the sigmoid BCE against the soft label, over cls_avg_factor;
 *   - bbox: loss_weight_bbox * sum over positives on non-empty RoIs of L1 / SmoothL1(beta) times code_weights, over reg_avg_factor;
 *   - corner: corner_loss_weight * the mean over those positives (of class corner_class, or all with -1) and their 8 corners of the
 *     Huber (delta 1) distance from the prediction decoded against its RoI to the nearer of the GT's and the heading-flipped GT's.
 *   A term without rows is exactly 0.  counts fp32 [2] = (positives on non-empty RoIs, corner rows), for the backward.  Block partials
 *   in double summed in a fixed order: deterministic.  Two launches, partials from the context arena.
 * sstb200_roi_head_loss_backward: grad_losses (device [3]) -> grad_cls [R] and grad_pred [R, 7], contiguous, each row writing only its
 *   own entries (no atomics).  One launch.
 *   Errors (both): a NULL pointer, R < 1, a row stride below the row, roi_width other than 7 / 9, SmoothL1 with beta <= 0 (SSTB_ERR_ARG). */
typedef struct {
  int32_t per_class;                   /* 1: one assigner per predicted class; 0: one assigner over every GT */
  int32_t num_classes;                 /* assigners when per_class */
  float pos_iou_thr[8], neg_iou_thr[8], min_pos_iou[8];
  int32_t num, num_pos;                /* sampler num, int(num * pos_fraction) */
  int32_t num_pieces;
  double piece_fractions[8];
  float piece_thrs[8];
} sstb200_roi_sample_cfg;
typedef struct {
  int32_t smooth_l1;                   /* 0: L1Loss, 1: SmoothL1Loss(beta) */
  float beta;
  float loss_weight_cls, loss_weight_bbox;
  int32_t with_corner_loss;
  int32_t corner_class;                /* -1: every positive */
  float corner_loss_weight;
  float code_weights[7];
} sstb200_roi_loss_cfg;
int sstb200_roi_assign_sample(sstb200_ctx* ctx, const sstb200_roi_sample_cfg* cfg, const float* proposals, int prop_width,
                              const int64_t* prop_labels, const float* keys, const int32_t* prop_offsets, const float* gt_boxes,
                              int gt_width, const int64_t* gt_labels, const int32_t* gt_offsets, int batch, int64_t* out_inds,
                              float* out_iou, int64_t* out_gt, int64_t* out_labels, int32_t* counts);
int sstb200_roi_head_targets(sstb200_ctx* ctx, const float* rois, int roi_width, const float* iou, const int64_t* gt_rows,
                             const int64_t* labels, int64_t num_rows, const float* gt_boxes, int gt_width, int num_classes,
                             const double* cls_pos_thr, const double* cls_neg_thr, float* soft_labels, int64_t* reg_mask,
                             float* bbox_targets, float* pos_gt_bboxes);
int sstb200_roi_head_loss_forward(sstb200_ctx* ctx, const sstb200_roi_loss_cfg* cfg, const float* cls_score, int64_t cls_stride,
                                  const float* bbox_pred, int64_t pred_stride, const uint8_t* nonempty, const float* soft_labels,
                                  const int64_t* reg_mask, const float* bbox_targets, const float* pos_gt_bboxes, const int64_t* labels,
                                  const float* rois, int roi_width, int64_t num_rows, const float* cls_avg_factor,
                                  const float* reg_avg_factor, float* losses, float* counts);
int sstb200_roi_head_loss_backward(sstb200_ctx* ctx, const sstb200_roi_loss_cfg* cfg, const float* cls_score, int64_t cls_stride,
                                   const float* bbox_pred, int64_t pred_stride, const uint8_t* nonempty, const float* soft_labels,
                                   const int64_t* reg_mask, const float* bbox_targets, const float* pos_gt_bboxes, const int64_t* labels,
                                   const float* rois, int roi_width, int64_t num_rows, const float* cls_avg_factor,
                                   const float* reg_avg_factor, const float* counts, const float* grad_losses, float* grad_cls,
                                   float* grad_pred);

#ifdef __cplusplus
}
#endif
#endif
