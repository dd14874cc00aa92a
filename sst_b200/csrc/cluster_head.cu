// SparseClusterHeadV2 training path (mmdet3d/models/dense_heads/sparse_cluster_head{,_v2}.py): the per-task cluster labels and box
// targets of get_targets (v2 lines 299-405, v1 lines 364-397) for every task and sample of a batch in one launch, and the fused
// per-task losses of loss_single_task (v2 lines 192-297): sigmoid focal on the logits, L1 or SmoothL1 on the positives' center / size /
// rot columns, forward and backward.  fp32, stream-ordered, no host sync.
//
// Targets: one thread per cluster, one grid row per sample; a block row stages its sample's GTs in shared memory CH_CHUNK at a time and
// only the clusters whose batch index is that sample test them, with in_box.cuh's make_box / to_local / in_box (the test of
// points_in_boxes_gpu, so a hit is bit-identical to the reference's).  modify_gt_for_single_task orders a task's GTs class by class in
// the task's class order and by input index within a class, and points_in_boxes_gpu takes the first box of that list: so a cluster
// takes, per task, the hit with the smallest (class rank, GT index).  Every GT is tested once for all tasks.
//
// Losses: block partials in double, one block sums them in a fixed order; the backward writes each cluster's own logit and reg rows.
//
// FSDV2Head (fsd_v2_head.py) runs the same kernels with two additions, each a template parameter so that the SparseClusterHeadV2
// instantiation (code size 8, in-box test on cluster_xyz) is unchanged: ASSIGN tests a separate point per cluster (the voxel centroid
// of centroid_assign, lines 359-362) while the encode still subtracts cluster_xyz, and CODE 10 adds the velocity targets (GT columns
// 7-8, lines 381-388) and a fifth loss group, vel = columns [8, 10), weighted per cluster by the copy-paste flag and divided by
// 2 * num_pos (loss_vel is called without avg_factor, lines 243-248).
#include <stdarg.h>
#include <algorithm>
#include <climits>
#include <cmath>
#include "heads.cuh"
#include "in_box.cuh"

namespace {

#define CH_THREADS 256       // targets block
#define CH_CHUNK 256         // GTs staged in shared memory per step
#define CH_MAX_BATCH 256
#define CH_MAX_GT 4096       // GTs per sample
#define CH_MAX_TASKS 8
#define CH_MAX_CLASSES 64    // global classes, and classes per task

// code size 8 or 10: target row TS = CODE + its velocity weight column for 10, loss groups NQ = cls, center, size, rot (+ vel)
template <int CODE>
struct ChCode {
  static_assert(CODE == 8 || CODE == 10, "code size 8 or 10");
  static constexpr int TS = CODE == 10 ? 11 : 8;
  static constexpr int NQ = CODE == 10 ? 5 : 4;
};

struct ChTargetArgs {
  const float* xyz;  // [M, >= 3], row stride xs
  const int64_t* bidx;  // [M], element stride bs
  long long xs, bs, M;
  const float* gt;    // [G, 7] bottom-centre
  const int64_t* gl;  // [G] global labels
  int gt_off[CH_MAX_BATCH + 1];
  int B, T, K;
  int cls_code[CH_MAX_CLASSES];  // task | rank << 8, or -1 for a class in no task
  int C[CH_MAX_TASKS];
  int64_t* labels[CH_MAX_TASKS];  // [M]
  float* tg[CH_MAX_TASKS];        // [M, TS]
  unsigned long long* num_pos;    // [T], zeroed before the launch
  const float* axyz;  // ASSIGN: [M, >= 3] points of the in-box test, row stride as
  long long as;
  int gw;             // GT row width: 7 for CODE 8; 9 or 10 for CODE 10
};

template <int CODE, bool ASSIGN>
__global__ void __launch_bounds__(CH_THREADS) ch_targets_kernel(const __grid_constant__ ChTargetArgs a) {
  constexpr int TS = ChCode<CODE>::TS;
  const int gs = CODE == 8 ? 7 : a.gw;
  __shared__ Box sb[CH_CHUNK];
  __shared__ int sc[CH_CHUNK];
  const int b = blockIdx.y;
  const long long j = (long long)blockIdx.x * CH_THREADS + threadIdx.x;
  const bool live = j < a.M;
  const long long bi = live ? __ldg(a.bidx + j * a.bs) : -1;
  const bool mine = live && bi == b;
  const bool bad = live && b == 0 && (bi < 0 || bi >= a.B);  // written by the first block row
  if (!__syncthreads_or(mine || bad)) return;  // uniform over the block
  float x = 0.f, y = 0.f, z = 0.f, px = 0.f, py = 0.f, pz = 0.f;  // encode base, in-box point
  if (mine) {
    const float* p = a.xyz + j * a.xs;
    x = p[0], y = p[1], z = p[2];
    if (ASSIGN) {
      const float* q = a.axyz + j * a.as;
      px = q[0], py = q[1], pz = q[2];
    }
  }
  if (!ASSIGN) px = x, py = y, pz = z;
  int best[CH_MAX_TASKS];  // rank * CH_MAX_GT + GT index in the sample, INT_MAX for no hit
#pragma unroll
  for (int u = 0; u < CH_MAX_TASKS; u++) best[u] = INT_MAX;
  const int g0 = a.gt_off[b], g1 = a.gt_off[b + 1];
  for (int k0 = g0; k0 < g1; k0 += CH_CHUNK) {
    const int m = min(CH_CHUNK, g1 - k0);
    if (threadIdx.x < m) {
      const float* q = a.gt + (size_t)(k0 + threadIdx.x) * gs;
      sb[threadIdx.x] = make_box(q[0], q[1], q[2], q[3], q[4], q[5], q[6]);
      const int64_t l = a.gl[k0 + threadIdx.x];
      sc[threadIdx.x] = l >= 0 && l < a.K ? a.cls_code[l] : -1;
    }
    __syncthreads();
    if (mine)
      for (int k = 0; k < m; k++) {
        const int code = sc[k];
        if (code < 0) continue;  // uniform over the block
        float lx, ly;
        to_local(sb[k], px, py, lx, ly);
        if (in_box(sb[k], pz, lx, ly)) {
          const int t = code & 0xff, key = (code >> 8) * CH_MAX_GT + (k0 - g0 + k);
#pragma unroll
          for (int u = 0; u < CH_MAX_TASKS; u++)
            if (u == t) best[u] = min(best[u], key);
        }
      }
    __syncthreads();  // this chunk's reads before the next chunk's stores
  }
#pragma unroll
  for (int u = 0; u < CH_MAX_TASKS; u++) {
    if (u >= a.T) break;  // uniform
    const bool pos = mine && best[u] != INT_MAX;
    if (mine) {
      float* t = a.tg[u] + j * TS;
      if (pos) {
        const int k = best[u] % CH_MAX_GT;
        const float* q = a.gt + (size_t)(g0 + k) * gs;
        if (CODE == 10) {  // velocity, and its loss weight: the copy-paste flag of a 10-column GT, 1 otherwise (stored first: nothing
                           // of it stays live across the transcendentals' calls)
          t[8] = q[7];
          t[9] = q[8];
          t[10] = a.gw == 10 ? q[9] : 1.f;
        }
        // BasePointBBoxCoder.encode: bottom-centre xyz - cluster xyz, log(dims + 1e-6), sin(yaw), cos(yaw); the transcendentals in
        // double, rounded once
        t[0] = __fsub_rn(q[0], x);
        t[1] = __fsub_rn(q[1], y);
        t[2] = __fsub_rn(q[2], z);
        for (int d = 0; d < 3; d++) t[3 + d] = (float)log((double)__fadd_rn(q[3 + d], 1e-6f));
        t[6] = (float)sin((double)q[6]);
        t[7] = (float)cos((double)q[6]);
        a.labels[u][j] = best[u] / CH_MAX_GT;
      } else {
        for (int d = 0; d < TS; d++) t[d] = 0.f;
        a.labels[u][j] = a.C[u];
      }
    } else if (bad) {
      float* t = a.tg[u] + j * TS;
      for (int d = 0; d < TS; d++) t[d] = NAN;
      a.labels[u][j] = -1;
    }
    const unsigned cnt = __popc(__ballot_sync(0xffffffffu, pos));
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(a.num_pos + u, (unsigned long long)cnt);
  }
}

// ---- losses -------------------------------------------------------------------------------------------------------------------------
struct ChLossArgs {
  int T;
  long long M;
  const float* x[CH_MAX_TASKS];  // [M, C_t] logits, row stride xs
  const float* r[CH_MAX_TASKS];  // [M, 8] reg preds, row stride rs
  long long xs[CH_MAX_TASKS], rs[CH_MAX_TASKS];
  int C[CH_MAX_TASKS];
  const int64_t* labels[CH_MAX_TASKS];
  const float* tg[CH_MAX_TASKS];
  float gamma, alpha, beta;
  int smooth;
  float w[4];                // loss weights: cls, center, size, rot
  const float* cls_avg;      // [T] device
  const float* reg_avg;      // [T] device
  const int64_t* num_pos;    // [T] device, the local positives
  float wvel;                // CODE 10: loss weight of vel
};

// mmdet 2.14 l1_loss / smooth_l1_loss element of d = pred - target, and its derivative
__device__ __forceinline__ float ch_reg(const ChLossArgs& a, float d) {
  const float ad = fabsf(d);
  if (!a.smooth) return ad;
  return ad < a.beta ? 0.5f * ad * ad / a.beta : ad - 0.5f * a.beta;
}

__device__ __forceinline__ float ch_reg_grad(const ChLossArgs& a, float d) {
  const float sg = abs_grad(d);
  if (!a.smooth) return sg;
  const float ad = fabsf(d);
  return ad < a.beta ? ad / a.beta * sg : sg;
}

// column groups of the reg code: center [0, 3), size [3, 6), rot [6, 8) (vel [8, 10) is summed apart, with its weight)
__device__ __forceinline__ int ch_group(int k) { return k < 3 ? 1 : (k < 6 ? 2 : 3); }

template <int CODE>
__global__ void __launch_bounds__(LOSS_THREADS) ch_loss_forward_kernel(const __grid_constant__ ChLossArgs a, double* part, int nb) {
  constexpr int TS = ChCode<CODE>::TS, NQ = ChCode<CODE>::NQ;
  __shared__ double sh[LOSS_THREADS / 32];
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (int t = 0; t < a.T; t++) {
    double acc[NQ] = {};
    const int C = a.C[t];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.M; i += stride) {
      const float* xr = a.x[t] + i * a.xs[t];
      const int64_t y = __ldg(a.labels[t] + i);
      for (int c = 0; c < C; c++) acc[0] += (double)sigmoid_focal(__ldg(xr + c), y == c, a.alpha, a.gamma);
      if (!(y >= 0 && y <= C)) acc[0] += (double)NAN;  // an out-of-range batch index (label -1)
      if (y >= 0 && y < C) {
        const float* rr = a.r[t] + i * a.rs[t];
        const float* tr = a.tg[t] + i * TS;
        for (int k = 0; k < 8; k++) acc[ch_group(k)] += (double)ch_reg(a, __ldg(rr + k) - __ldg(tr + k));
        if (CODE == 10) {
          const float vw = __ldg(tr + 10);
          for (int k = 8; k < 10; k++) acc[NQ - 1] += (double)(ch_reg(a, __ldg(rr + k) - __ldg(tr + k)) * vw);
        }
      }
    }
    for (int q = 0; q < NQ; q++) {
      const double s = thread0_block_sum(acc[q], sh);
      if (threadIdx.x == 0) part[(size_t)(t * NQ + q) * nb + blockIdx.x] = s;
    }
  }
}

// fixed-order sums of the partials -> losses [T, NQ]
template <int CODE>
__global__ void __launch_bounds__(LOSS_THREADS) ch_loss_final_kernel(const __grid_constant__ ChLossArgs a, const double* part, int nb,
                                                                     float* losses) {
  constexpr int NQ = ChCode<CODE>::NQ;
  __shared__ double sh[LOSS_THREADS / 32];
  for (int k = 0; k < NQ * a.T; k++) {
    const double s = sum_partials(part, nb, k, sh);
    if (threadIdx.x == 0) {
      const int t = k / NQ, q = k % NQ;
      if (q == 0)
        losses[k] = (float)((double)a.w[0] * (s / (double)a.cls_avg[t]));
      else if (CODE == 10 && q == 4)  // mmdet's reduction 'mean' without avg_factor: over the 2 * num_pos local elements
        losses[k] = a.num_pos[t] > 0 ? (float)((double)a.wvel * (s / (2.0 * (double)a.num_pos[t]))) : 0.f;
      else  // the reference's `num_pos > 0` branch on the local count: pos_reg_preds.sum() * 0 otherwise
        losses[k] = a.num_pos[t] > 0 ? (float)((double)a.w[q] * (s / (double)a.reg_avg[t])) : 0.f;
    }
  }
}

struct ChGradPtrs {
  float* gx[CH_MAX_TASKS];  // [M, C_t] contiguous
  float* gr[CH_MAX_TASKS];  // [M, CODE] contiguous
};

template <int CODE>
__global__ void __launch_bounds__(LOSS_THREADS) ch_loss_backward_kernel(const __grid_constant__ ChLossArgs a, const float* grad_losses,
                                                                        const __grid_constant__ ChGradPtrs p) {
  constexpr int TS = ChCode<CODE>::TS, NQ = ChCode<CODE>::NQ;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (int t = 0; t < a.T; t++) {
    const int C = a.C[t];
    const float gc = (float)((double)grad_losses[NQ * t] * a.w[0] / (double)a.cls_avg[t]);
    float gq[NQ] = {};
    if (a.num_pos[t] > 0) {
      for (int q = 1; q < 4; q++) gq[q] = (float)((double)grad_losses[NQ * t + q] * a.w[q] / (double)a.reg_avg[t]);
      if (CODE == 10) gq[NQ - 1] = (float)((double)grad_losses[NQ * t + 4] * a.wvel / (2.0 * (double)a.num_pos[t]));
    }
    float* gxt = p.gx[t];
    float* grt = p.gr[t];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.M; i += stride) {
      const float* xr = a.x[t] + i * a.xs[t];
      const int64_t y = __ldg(a.labels[t] + i);
      const bool ok = y >= 0 && y <= C;
      for (int c = 0; c < C; c++) gxt[i * C + c] = ok ? gc * sigmoid_focal_grad(__ldg(xr + c), y == c, a.alpha, a.gamma) : NAN;
      float* g = grt + i * CODE;
      if (y >= 0 && y < C) {
        const float* rr = a.r[t] + i * a.rs[t];
        const float* tr = a.tg[t] + i * TS;
        for (int k = 0; k < 8; k++) g[k] = gq[ch_group(k)] * ch_reg_grad(a, __ldg(rr + k) - __ldg(tr + k));
        if (CODE == 10) {
          const float vw = __ldg(tr + 10);
          for (int k = 8; k < 10; k++) g[k] = gq[NQ - 1] * (ch_reg_grad(a, __ldg(rr + k) - __ldg(tr + k)) * vw);
        }
      } else {
        for (int k = 0; k < CODE; k++) g[k] = 0.f;
      }
    }
  }
}

sstb200_cluster_head_loss_cfg_ex cfg_ex(const sstb200_cluster_head_loss_cfg* cfg) {
  sstb200_cluster_head_loss_cfg_ex e{};
  if (cfg) {
    e.gamma = cfg->gamma, e.alpha = cfg->alpha, e.smooth_l1 = cfg->smooth_l1, e.beta = cfg->beta;
    e.loss_weight_cls = cfg->loss_weight_cls, e.loss_weight_center = cfg->loss_weight_center;
    e.loss_weight_size = cfg->loss_weight_size, e.loss_weight_rot = cfg->loss_weight_rot;
  }
  e.loss_weight_vel = 0.f, e.code_size = 8;
  return e;
}

int ch_loss_args(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks, int64_t num_clusters,
                 const float* const* cls_logits, const int64_t* logit_strides, const int32_t* task_classes, const float* const* reg_preds,
                 const int64_t* reg_strides, int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                 const float* cls_avg_factor, const float* reg_avg_factor, ChLossArgs& a) {
  CHECK_ARG(c, cfg && cls_logits && logit_strides && task_classes && reg_preds && reg_strides && labels && bbox_targets);
  CHECK_ARG(c, num_pos && cls_avg_factor && reg_avg_factor && num_clusters >= 1 && num_tasks >= 1);
  CHECK_ARG(c, cfg->code_size == 8 || cfg->code_size == 10);
  if (num_tasks > CH_MAX_TASKS)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "cluster_head_loss: %d tasks, at most %d", num_tasks, CH_MAX_TASKS);
  if (!(cfg->gamma >= 1.f)) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "cluster_head_loss: focal gamma %g, at least 1", (double)cfg->gamma);
  CHECK_ARG(c, !cfg->smooth_l1 || cfg->beta > 0.f);
  a.T = num_tasks, a.M = num_clusters;
  for (int t = 0; t < num_tasks; t++) {
    const int C = task_classes[t];
    CHECK_ARG(c, cls_logits[t] && reg_preds[t] && labels[t] && bbox_targets[t] && C >= 1);
    CHECK_ARG(c, logit_strides[t] >= C && reg_strides[t] >= cfg->code_size);
    if (C > CH_MAX_CLASSES) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "cluster_head_loss: %d classes in a task, at most %d", C, CH_MAX_CLASSES);
    a.x[t] = cls_logits[t], a.r[t] = reg_preds[t], a.xs[t] = logit_strides[t], a.rs[t] = reg_strides[t], a.C[t] = C;
    a.labels[t] = labels[t], a.tg[t] = bbox_targets[t];
  }
  a.gamma = cfg->gamma, a.alpha = cfg->alpha, a.beta = cfg->beta, a.smooth = cfg->smooth_l1 != 0;
  a.w[0] = cfg->loss_weight_cls, a.w[1] = cfg->loss_weight_center, a.w[2] = cfg->loss_weight_size, a.w[3] = cfg->loss_weight_rot;
  a.wvel = cfg->code_size == 10 ? cfg->loss_weight_vel : 0.f;
  a.cls_avg = cls_avg_factor, a.reg_avg = reg_avg_factor, a.num_pos = num_pos;
  return SSTB_OK;
}

int ch_targets(sstb200_ctx* c, const float* cluster_xyz, int64_t xyz_stride, const float* assign_xyz, int64_t assign_stride,
               const int64_t* batch_idx, int64_t batch_stride, int64_t num_clusters, const float* gt_boxes, int gt_width,
               const int64_t* gt_labels, const int32_t* gt_offsets, int batch, int num_classes, const int32_t* class_task,
               const int32_t* class_rank, int num_tasks, const int32_t* task_classes, int code_size, int64_t* const* labels,
               float* const* bbox_targets, int64_t* num_pos) {
  CHECK_ARG(c, gt_offsets && class_task && class_rank && task_classes && labels && bbox_targets && num_pos);
  CHECK_ARG(c, batch >= 1 && num_clusters >= 0 && xyz_stride >= 3 && batch_stride >= 1 && num_tasks >= 1 && num_classes >= 1);
  // code size 8 encodes 7-column boxes (BasePointBBoxCoder.encode asserts code_size == 10 on 9 / 10 columns); 10 needs the velocity
  CHECK_ARG(c, (code_size == 8 && gt_width == 7) || (code_size == 10 && (gt_width == 9 || gt_width == 10)));
  CHECK_ARG(c, !assign_xyz || assign_stride >= 3);
  if (batch > CH_MAX_BATCH) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "cluster_head_targets: %d samples, at most %d", batch, CH_MAX_BATCH);
  if (num_tasks > CH_MAX_TASKS || num_classes > CH_MAX_CLASSES)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "cluster_head_targets: %d tasks / %d classes, at most %d / %d", num_tasks, num_classes,
                     CH_MAX_TASKS, CH_MAX_CLASSES);
  const int rc = check_offsets(c, "cluster_head_targets", gt_offsets, batch, CH_MAX_GT);
  if (rc) return rc;
  ChTargetArgs a;
  for (int t = 0; t < num_tasks; t++) {
    CHECK_ARG(c, task_classes[t] >= 1 && task_classes[t] <= CH_MAX_CLASSES);
    CHECK_ARG(c, num_clusters == 0 || (labels[t] && bbox_targets[t]));
    a.C[t] = task_classes[t], a.labels[t] = labels[t], a.tg[t] = bbox_targets[t];
  }
  for (int k = 0; k < num_classes; k++) {
    const int t = class_task[k];
    CHECK_ARG(c, t < num_tasks && (t < 0 || (class_rank[k] >= 0 && class_rank[k] < task_classes[t])));
    a.cls_code[k] = t < 0 ? -1 : (t | class_rank[k] << 8);
  }
  const int G = gt_offsets[batch];
  CHECK_ARG(c, num_clusters == 0 || (cluster_xyz && batch_idx));
  CHECK_ARG(c, G == 0 || (gt_boxes && gt_labels));
  CUDA_TRY(c, cudaMemsetAsync(num_pos, 0, sizeof(int64_t) * num_tasks, c->stream));
  if (num_clusters == 0) return SSTB_OK;
  a.xyz = cluster_xyz, a.xs = xyz_stride, a.bidx = batch_idx, a.bs = batch_stride, a.M = num_clusters;
  a.gt = gt_boxes, a.gl = gt_labels, a.B = batch, a.T = num_tasks, a.K = num_classes;
  for (int b = 0; b <= batch; b++) a.gt_off[b] = gt_offsets[b];
  a.num_pos = (unsigned long long*)num_pos;
  a.gw = gt_width;
  // code size 10 without assignment points tests cluster_xyz itself through the ASSIGN instantiation
  a.axyz = assign_xyz ? assign_xyz : cluster_xyz, a.as = assign_xyz ? assign_stride : xyz_stride;
  const long long bx = (num_clusters + CH_THREADS - 1) / CH_THREADS;
  if (bx > 0x7fffffffLL) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "cluster_head_targets: %lld clusters", (long long)num_clusters);
  const dim3 grid((unsigned)bx, (unsigned)batch);
  if (code_size == 10)
    ch_targets_kernel<10, true><<<grid, CH_THREADS, 0, c->stream>>>(a);
  else if (assign_xyz)
    ch_targets_kernel<8, true><<<grid, CH_THREADS, 0, c->stream>>>(a);
  else
    ch_targets_kernel<8, false><<<grid, CH_THREADS, 0, c->stream>>>(a);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

int ch_loss_forward(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks, int64_t num_clusters,
                    const float* const* cls_logits, const int64_t* logit_strides, const int32_t* task_classes, const float* const* reg_preds,
                    const int64_t* reg_strides, int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                    const float* cls_avg_factor, const float* reg_avg_factor, float* losses) {
  ChLossArgs a;
  int rc = ch_loss_args(c, cfg, num_tasks, num_clusters, cls_logits, logit_strides, task_classes, reg_preds, reg_strides, labels,
                        bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, a);
  if (rc) return rc;
  CHECK_ARG(c, losses);
  const bool vel = cfg->code_size == 10;
  const int nq = vel ? ChCode<10>::NQ : ChCode<8>::NQ;
  const int nb = loss_grid(c, a.M);
  arena_reset(c);
  double* part;
  rc = arena_carve(c, [&](Carve& cv) { part = cv.take<double>((size_t)nq * num_tasks * nb); });
  if (rc) return rc;
  if (vel)
    ch_loss_forward_kernel<10><<<nb, LOSS_THREADS, 0, c->stream>>>(a, part, nb);
  else
    ch_loss_forward_kernel<8><<<nb, LOSS_THREADS, 0, c->stream>>>(a, part, nb);
  LAUNCH_CHECK(c);
  if (vel)
    ch_loss_final_kernel<10><<<1, LOSS_THREADS, 0, c->stream>>>(a, part, nb, losses);
  else
    ch_loss_final_kernel<8><<<1, LOSS_THREADS, 0, c->stream>>>(a, part, nb, losses);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

int ch_loss_backward(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks, int64_t num_clusters,
                     const float* const* cls_logits, const int64_t* logit_strides, const int32_t* task_classes, const float* const* reg_preds,
                     const int64_t* reg_strides, int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                     const float* cls_avg_factor, const float* reg_avg_factor, const float* grad_losses, float* const* grad_logits,
                     float* const* grad_reg_preds) {
  ChLossArgs a;
  int rc = ch_loss_args(c, cfg, num_tasks, num_clusters, cls_logits, logit_strides, task_classes, reg_preds, reg_strides, labels,
                        bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, a);
  if (rc) return rc;
  CHECK_ARG(c, grad_losses && grad_logits && grad_reg_preds);
  ChGradPtrs p;
  for (int t = 0; t < num_tasks; t++) {
    CHECK_ARG(c, grad_logits[t] && grad_reg_preds[t]);
    p.gx[t] = grad_logits[t], p.gr[t] = grad_reg_preds[t];
  }
  if (cfg->code_size == 10)
    ch_loss_backward_kernel<10><<<loss_grid(c, a.M), LOSS_THREADS, 0, c->stream>>>(a, grad_losses, p);
  else
    ch_loss_backward_kernel<8><<<loss_grid(c, a.M), LOSS_THREADS, 0, c->stream>>>(a, grad_losses, p);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

}  // namespace

extern "C" int sstb200_cluster_head_targets(sstb200_ctx* c, const float* cluster_xyz, int64_t xyz_stride, const int64_t* batch_idx,
                                            int64_t batch_stride, int64_t num_clusters, const float* gt_boxes, const int64_t* gt_labels,
                                            const int32_t* gt_offsets, int batch, int num_classes, const int32_t* class_task,
                                            const int32_t* class_rank, int num_tasks, const int32_t* task_classes, int64_t* const* labels,
                                            float* const* bbox_targets, int64_t* num_pos) {
  return ch_targets(c, cluster_xyz, xyz_stride, nullptr, 0, batch_idx, batch_stride, num_clusters, gt_boxes, 7, gt_labels, gt_offsets,
                    batch, num_classes, class_task, class_rank, num_tasks, task_classes, 8, labels, bbox_targets, num_pos);
}

extern "C" int sstb200_cluster_head_targets_ex(sstb200_ctx* c, const float* cluster_xyz, int64_t xyz_stride, const float* assign_xyz,
                                               int64_t assign_stride, const int64_t* batch_idx, int64_t batch_stride, int64_t num_clusters,
                                               const float* gt_boxes, int gt_width, const int64_t* gt_labels, const int32_t* gt_offsets,
                                               int batch, int num_classes, const int32_t* class_task, const int32_t* class_rank,
                                               int num_tasks, const int32_t* task_classes, int code_size, int64_t* const* labels,
                                               float* const* bbox_targets, int64_t* num_pos) {
  return ch_targets(c, cluster_xyz, xyz_stride, assign_xyz, assign_stride, batch_idx, batch_stride, num_clusters, gt_boxes, gt_width,
                    gt_labels, gt_offsets, batch, num_classes, class_task, class_rank, num_tasks, task_classes, code_size, labels,
                    bbox_targets, num_pos);
}

extern "C" int sstb200_cluster_head_loss_forward(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg* cfg, int num_tasks,
                                                 int64_t num_clusters, const float* const* cls_logits, const int64_t* logit_strides,
                                                 const int32_t* task_classes, const float* const* reg_preds, const int64_t* reg_strides,
                                                 int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                                                 const float* cls_avg_factor, const float* reg_avg_factor, float* losses) {
  CHECK_ARG(c, cfg);
  const sstb200_cluster_head_loss_cfg_ex e = cfg_ex(cfg);
  return ch_loss_forward(c, &e, num_tasks, num_clusters, cls_logits, logit_strides, task_classes, reg_preds, reg_strides, labels,
                         bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, losses);
}

extern "C" int sstb200_cluster_head_loss_forward_ex(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks,
                                                    int64_t num_clusters, const float* const* cls_logits, const int64_t* logit_strides,
                                                    const int32_t* task_classes, const float* const* reg_preds, const int64_t* reg_strides,
                                                    int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                                                    const float* cls_avg_factor, const float* reg_avg_factor, float* losses) {
  CHECK_ARG(c, cfg);
  return ch_loss_forward(c, cfg, num_tasks, num_clusters, cls_logits, logit_strides, task_classes, reg_preds, reg_strides, labels,
                         bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, losses);
}

extern "C" int sstb200_cluster_head_loss_backward(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg* cfg, int num_tasks,
                                                  int64_t num_clusters, const float* const* cls_logits, const int64_t* logit_strides,
                                                  const int32_t* task_classes, const float* const* reg_preds, const int64_t* reg_strides,
                                                  int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                                                  const float* cls_avg_factor, const float* reg_avg_factor, const float* grad_losses,
                                                  float* const* grad_logits, float* const* grad_reg_preds) {
  CHECK_ARG(c, cfg);
  const sstb200_cluster_head_loss_cfg_ex e = cfg_ex(cfg);
  return ch_loss_backward(c, &e, num_tasks, num_clusters, cls_logits, logit_strides, task_classes, reg_preds, reg_strides, labels,
                          bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, grad_losses, grad_logits, grad_reg_preds);
}

extern "C" int sstb200_cluster_head_loss_backward_ex(sstb200_ctx* c, const sstb200_cluster_head_loss_cfg_ex* cfg, int num_tasks,
                                                     int64_t num_clusters, const float* const* cls_logits, const int64_t* logit_strides,
                                                     const int32_t* task_classes, const float* const* reg_preds, const int64_t* reg_strides,
                                                     int64_t* const* labels, float* const* bbox_targets, const int64_t* num_pos,
                                                     const float* cls_avg_factor, const float* reg_avg_factor, const float* grad_losses,
                                                     float* const* grad_logits, float* const* grad_reg_preds) {
  CHECK_ARG(c, cfg);
  return ch_loss_backward(c, cfg, num_tasks, num_clusters, cls_logits, logit_strides, task_classes, reg_preds, reg_strides, labels,
                          bbox_targets, num_pos, cls_avg_factor, reg_avg_factor, grad_losses, grad_logits, grad_reg_preds);
}
