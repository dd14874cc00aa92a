// VoteSegHead training path (mmdet3d/models/decode_heads/segmentation_head.py): the per-point labels and vote targets of get_targets
// (lines 212-283) for a whole batch in one launch, and the fused segmentation + vote losses of `losses` (lines 107-173) with their
// training-log counts, forward and backward.  fp32, stream-ordered, no host sync.
//
// Targets: one thread per point, one grid row per sample.  The sample's GTs are staged in shared memory VS_CHUNK at a time and tested
// with in_box.cuh's make_box / to_local / in_box, the test sstb200_points_in_boxes uses, so the hit is bit-identical to the reference's
// points_in_boxes_gpu (first hit wins); a point stops scanning at its first hit.  GTs with a negative label are skipped, which is the
// reference's valid_gt_mask filter followed by points_in_boxes on the survivors.
//
// Losses: one read per direction of each point's logit row and of the three vote channels of its own class.  Forward = block partials
// (double for the sums, integers for the counts), one block sums them in a fixed order; the whole vote tensor is scanned only when no
// point is valid.  Backward = one pass in which every point writes only its own logits and vote channels.
#include <stdarg.h>
#include <algorithm>
#include <cmath>
#include "heads.cuh"
#include "in_box.cuh"

namespace {

#define VS_THREADS 256      // targets block
#define VS_CHUNK 256         // GTs staged in shared memory per step
#define VS_MAX_BATCH 256
#define VS_MAX_GT 4096       // GTs per sample
#define VS_MAX_CLASSES 64    // logit columns
#define VS_MAX_GROUPS 64
#define VS_MAX_ENTRIES 64

struct VsTargetArgs {
  const float* pts;  // [N, >= 3], row stride `stride`
  long long stride;
  const float* gt;      // [G, 7] bottom-centre
  const int64_t* gl;    // [G]
  int pt_off[VS_MAX_BATCH + 1];
  int gt_off[VS_MAX_BATCH + 1];
  int bg_label;
  int64_t* labels;  // [N]
  float* vt;        // [N, 3]
  uint8_t* mask;    // [N]
};

// encode_vote_targets: sign(d) * |d| ** 0.5 (torch's pow 0.5 is the IEEE square root)
__device__ __forceinline__ float vs_encode(float d) { return d == 0.f ? 0.f : copysignf(__fsqrt_rn(fabsf(d)), d); }

__global__ void __launch_bounds__(VS_THREADS) vs_targets_kernel(const __grid_constant__ VsTargetArgs a) {
  __shared__ Box sb[VS_CHUNK];
  __shared__ int sv[VS_CHUNK];
  const int b = blockIdx.y;
  const int p0 = a.pt_off[b], n = a.pt_off[b + 1] - p0;
  if ((int)(blockIdx.x * VS_THREADS) >= n) return;  // uniform over the block
  const int j = blockIdx.x * VS_THREADS + threadIdx.x;
  const bool live = j < n;
  const long long i = (long long)p0 + j;
  float x = 0.f, y = 0.f, z = 0.f;
  if (live) {
    const float* p = a.pts + i * a.stride;
    x = p[0], y = p[1], z = p[2];
  }
  int hit = -1;
  const int g0 = a.gt_off[b], g1 = a.gt_off[b + 1];
  for (int k0 = g0; k0 < g1; k0 += VS_CHUNK) {
    const int m = min(VS_CHUNK, g1 - k0);
    if (threadIdx.x < m) {
      const float* q = a.gt + (size_t)(k0 + threadIdx.x) * 7;
      sb[threadIdx.x] = make_box(q[0], q[1], q[2], q[3], q[4], q[5], q[6]);
      sv[threadIdx.x] = a.gl[k0 + threadIdx.x] >= 0;
    }
    __syncthreads();
    if (live && hit < 0)
      for (int k = 0; k < m; k++) {
        if (!sv[k]) continue;  // uniform over the block
        float lx, ly;
        to_local(sb[k], x, y, lx, ly);
        if (in_box(sb[k], z, lx, ly)) {
          hit = k0 + k;
          break;
        }
      }
    if (__syncthreads_and(!live || hit >= 0)) break;  // also orders this chunk's reads before the next chunk's stores
  }
  if (!live) return;
  float* t = a.vt + i * 3;
  if (hit >= 0) {
    // gravity_center (lidar_box3d.py:45-51): z + h * 0.5 in fp32; delta = centre - point (segmentation_head.py:276)
    const float* q = a.gt + (size_t)hit * 7;
    const float cz = __fadd_rn(q[2], __fmul_rn(q[5], 0.5f));
    t[0] = vs_encode(__fsub_rn(q[0], x));
    t[1] = vs_encode(__fsub_rn(q[1], y));
    t[2] = vs_encode(__fsub_rn(cz, z));
    a.labels[i] = a.gl[hit];
    a.mask[i] = 1;
  } else {
    t[0] = t[1] = t[2] = 0.f;
    a.labels[i] = a.bg_label;
    a.mask[i] = 0;
  }
}

// ---- losses -------------------------------------------------------------------------------------------------------------------------
struct VsLossArgs {
  const float* x;  // [N, C] logits, row stride xs
  const float* v;  // [N, 3 C] vote predictions, row stride vs
  long long xs, vs, n;
  const int64_t* labels;  // [N]
  const float* vt;        // [N, 3]
  const uint8_t* mask;    // [N]
  int C, softmax;
  float gamma, alpha, scale;
  float cw[VS_MAX_CLASSES];
  int G, E;
  unsigned long long gmask[VS_MAX_GROUPS];
  float thr[VS_MAX_GROUPS];
  int eg[VS_MAX_ENTRIES], ec[VS_MAX_ENTRIES];
};

__device__ __forceinline__ float logit(const VsLossArgs& a, const float* xr, int c) { return __fmul_rn(__ldg(xr + c), a.scale); }

// softmax statistics of a row: max and sum of exp(x - max); NaN anywhere in the row makes both NaN
__device__ __forceinline__ void row_softmax(const VsLossArgs& a, const float* xr, float& m, float& se) {
  m = -INFINITY;
  bool nan = false;
  for (int c = 0; c < a.C; c++) {
    const float xc = logit(a, xr, c);
    nan |= xc != xc;
    m = fmaxf(m, xc);
  }
  se = 0.f;
  for (int c = 0; c < a.C; c++) se += expf(logit(a, xr, c) - m);
  if (nan) m = se = NAN;
}

__device__ __forceinline__ bool label_ok(const VsLossArgs& a, int64_t y) { return y >= 0 && y < (a.softmax ? a.C : a.C + 1); }

// integer partials per block: n_valid, num_fg, then tp[E], real[E]
#define VS_NINT(E) (2 + 2 * (E))

__global__ void __launch_bounds__(LOSS_THREADS) vs_loss_forward_kernel(const __grid_constant__ VsLossArgs a, double* part, int* ipart,
                                                                        int nb) {
  __shared__ double sh[LOSS_THREADS / 32];
  __shared__ int scnt[VS_NINT(VS_MAX_ENTRIES)];
  const int K = VS_NINT(a.E);
  for (int k = threadIdx.x; k < K; k += blockDim.x) scnt[k] = 0;
  __syncthreads();
  double seg = 0.0, vote = 0.0;
  int nvalid = 0, fg = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    const float* xr = a.x + i * a.xs;
    const float* vr = a.v + i * a.vs;
    const int64_t y = __ldg(a.labels + i);
    const bool ok = label_ok(a, y);
    float m = 0.f, se = 1.f;
    // segmentation loss (lines 116-118)
    if (!a.softmax) {
      for (int c = 0; c < a.C; c++) seg += (double)sigmoid_focal(logit(a, xr, c), y == c, a.alpha, a.gamma);
    } else {
      row_softmax(a, xr, m, se);
      if (ok) seg += (double)(a.cw[y] * (m + logf(se) - logit(a, xr, (int)y)));
    }
    if (!ok) seg += (double)NAN;
    // vote loss (lines 122-142): only the three channels of a valid point's own class are read
    if (__ldg(a.mask + i)) {
      nvalid++;
      if (y >= 0 && y < a.C) {
        const float* t = a.vt + i * 3;
        for (int k = 0; k < 3; k++) vote += (double)fabsf(__ldg(vr + 3 * y + k) - __ldg(t + k));
      } else {
        vote += (double)NAN;
      }
    }
    // training-log counts (lines 146-171): group g predicts the point when its score (sigmoid, or the sum of the softmax
    // probabilities of its classes) exceeds thr[g]; entry e counts the points of class ec[e] that group eg[e] predicts
    for (int g = 0; g < a.G; g++) {
      float score = 0.f;
      for (int c = 0; c < a.C; c++)
        if (a.gmask[g] >> c & 1ull) {
          const float xc = logit(a, xr, c);
          score += a.softmax ? expf(xc - m) / se : sig(xc).s;
        }
      const bool pred = score > a.thr[g];
      fg += pred;
      if (pred)
        for (int e = 0; e < a.E; e++)
          if (a.eg[e] == g && y == a.ec[e]) atomicAdd(scnt + 2 + e, 1);
    }
    for (int e = 0; e < a.E; e++)
      if (y == a.ec[e]) atomicAdd(scnt + 2 + a.E + e, 1);
  }
  seg = thread0_block_sum(seg, sh);
  vote = thread0_block_sum(vote, sh);
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    nvalid += __shfl_xor_sync(0xffffffffu, nvalid, o);
    fg += __shfl_xor_sync(0xffffffffu, fg, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(scnt, nvalid);
    atomicAdd(scnt + 1, fg);
  }
  __syncthreads();
  if (threadIdx.x == 0) part[blockIdx.x] = seg, part[nb + blockIdx.x] = vote;
  for (int k = threadIdx.x; k < K; k += blockDim.x) ipart[(size_t)k * nb + blockIdx.x] = scnt[k];
}

// fixed-order sums of the partials -> losses[0..1], the device n_valid and the counts (tp[E], real[E], num_fg)
__global__ void __launch_bounds__(LOSS_THREADS) vs_loss_final_kernel(const double* part, const int* ipart, int nb, int E, long long n,
                                                                     int C, int softmax, float w_seg, float w_vote, float* losses,
                                                                     int64_t* num_valid, int64_t* counts) {
  __shared__ double sh[LOSS_THREADS / 32];
  double s[2];
  for (int k = 0; k < 2; k++) s[k] = sum_partials(part, nb, k, sh);
  // the integer partials: one warp per count, its lanes striding over the blocks (integer sums do not depend on the order)
  __shared__ long long v[VS_NINT(VS_MAX_ENTRIES)];
  const int lane = threadIdx.x & 31;
  for (int k = threadIdx.x >> 5; k < VS_NINT(E); k += blockDim.x >> 5) {
    long long t = 0;
    for (int i = lane; i < nb; i += 32) t += ipart[(size_t)k * nb + i];
#pragma unroll
    for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) v[k] = t;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    losses[0] = (float)((double)w_seg * (s[0] / (double)(softmax ? n : n * C)));
    // no valid point: vote_preds.sum() * 0, i.e. 0 here; vs_vote_nonfinite_kernel then makes it NaN when a prediction is not finite
    losses[1] = v[0] > 0 ? (float)((double)w_vote * (s[1] / (double)(3 * v[0]))) : 0.f;
    *num_valid = v[0];
    for (int e = 0; e < 2 * E; e++) counts[e] = v[2 + e];
    counts[2 * E] = v[1];
  }
}

// The no-valid-point case of the vote loss: vote_preds.sum() * 0 is NaN when any vote prediction is not finite.  Every block returns at
// once unless the device n_valid is 0, so the whole [N, 3 C] vote tensor is read only in that case.
__global__ void __launch_bounds__(LOSS_THREADS) vs_vote_nonfinite_kernel(const __grid_constant__ VsLossArgs a,
                                                                         const int64_t* num_valid, float* losses) {
  if (*num_valid > 0) return;
  const int W = 3 * a.C;
  bool bad = false;
  const long long stride = (long long)gridDim.x * blockDim.x, n = a.n * W;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n && !bad; j += stride) {
    const long long i = j / W;
    bad = !isfinite(__ldg(a.v + i * a.vs + (j - i * W)));
  }
  if (bad) losses[1] = NAN;  // every writer stores the same value
}

__global__ void __launch_bounds__(LOSS_THREADS) vs_loss_backward_kernel(const __grid_constant__ VsLossArgs a, float w_seg,
                                                                        float w_vote, const int64_t* num_valid, const float* grad_losses,
                                                                        float* gx, float* gv) {
  const float gs = (float)((double)grad_losses[0] * w_seg * a.scale / (double)(a.softmax ? a.n : a.n * a.C));
  const long long nv = *num_valid;
  const float gvs = nv > 0 ? (float)((double)grad_losses[1] * w_vote / (double)(3 * nv)) : 0.f;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    const float* xr = a.x + i * a.xs;
    const float* vr = a.v + i * a.vs;
    float* gxr = gx + i * a.C;
    float* gvr = gv + i * 3 * a.C;
    const int64_t y = __ldg(a.labels + i);
    const bool ok = label_ok(a, y);
    if (!a.softmax) {
      for (int c = 0; c < a.C; c++) gxr[c] = ok ? gs * sigmoid_focal_grad(logit(a, xr, c), y == c, a.alpha, a.gamma) : NAN;
    } else {
      float m, se;
      row_softmax(a, xr, m, se);
      const float w = ok ? gs * a.cw[y] : NAN;
      for (int c = 0; c < a.C; c++) gxr[c] = w * (expf(logit(a, xr, c) - m) / se - (c == y ? 1.f : 0.f));
    }
    const bool valid = __ldg(a.mask + i) != 0;
    for (int k = 0; k < 3 * a.C; k++) gvr[k] = valid && !(y >= 0 && y < a.C) ? NAN : 0.f;
    if (valid && y >= 0 && y < a.C) {
      const float* t = a.vt + i * 3;
      for (int k = 0; k < 3; k++) {
        const float d = __ldg(vr + 3 * y + k) - __ldg(t + k);
        gvr[3 * y + k] = gvs * abs_grad(d);
      }
    }
  }
}

int vs_loss_args(sstb200_ctx* c, const sstb200_voteseg_cfg* cfg, const float* seg_logits, int64_t logit_stride, const float* vote_preds,
                 int64_t vote_stride, int64_t num_points, const int64_t* labels, const float* vote_targets, const uint8_t* vote_mask,
                 VsLossArgs& a) {
  CHECK_ARG(c, cfg && seg_logits && vote_preds && labels && vote_targets && vote_mask);
  const int C = cfg->num_classes;
  CHECK_ARG(c, num_points >= 1 && C >= 1 && logit_stride >= C && vote_stride >= 3LL * C);
  CHECK_ARG(c, cfg->num_groups >= 0 && cfg->num_entries >= 0);
  CHECK_ARG(c, cfg->num_groups == 0 || (cfg->group_masks && cfg->group_thresh));
  CHECK_ARG(c, cfg->num_entries == 0 || (cfg->entry_group && cfg->entry_class));
  if (C > VS_MAX_CLASSES || cfg->num_groups > VS_MAX_GROUPS || cfg->num_entries > VS_MAX_ENTRIES)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "voteseg_loss: %d classes / %d groups / %d entries, at most %d / %d / %d", C,
                     cfg->num_groups, cfg->num_entries, VS_MAX_CLASSES, VS_MAX_GROUPS, VS_MAX_ENTRIES);
  if (!cfg->use_softmax && !(cfg->gamma >= 1.f))
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "voteseg_loss: focal gamma %g, at least 1", (double)cfg->gamma);
  a.x = seg_logits, a.v = vote_preds, a.xs = logit_stride, a.vs = vote_stride, a.n = num_points;
  a.labels = labels, a.vt = vote_targets, a.mask = vote_mask;
  a.C = C, a.softmax = cfg->use_softmax != 0;
  a.gamma = cfg->gamma, a.alpha = cfg->alpha, a.scale = cfg->logit_scale;
  for (int k = 0; k < C; k++) a.cw[k] = cfg->class_weight ? cfg->class_weight[k] : 1.f;
  a.G = cfg->num_groups, a.E = cfg->num_entries;
  for (int g = 0; g < a.G; g++) {
    CHECK_ARG(c, C == 64 || (cfg->group_masks[g] >> C) == 0);
    a.gmask[g] = cfg->group_masks[g], a.thr[g] = cfg->group_thresh[g];
  }
  for (int e = 0; e < a.E; e++) {
    CHECK_ARG(c, cfg->entry_group[e] >= 0 && cfg->entry_group[e] < a.G && cfg->entry_class[e] >= 0 && cfg->entry_class[e] < C);
    a.eg[e] = cfg->entry_group[e], a.ec[e] = cfg->entry_class[e];
  }
  return SSTB_OK;
}

}  // namespace

extern "C" int sstb200_voteseg_targets(sstb200_ctx* c, const float* points, int64_t point_stride, const int32_t* point_offsets,
                                       const float* gt_boxes, const int64_t* gt_labels, const int32_t* gt_offsets, int batch, int bg_label,
                                       int64_t* labels, float* vote_targets, uint8_t* vote_mask) {
  CHECK_ARG(c, point_offsets && gt_offsets && batch >= 1 && point_stride >= 3);
  if (batch > VS_MAX_BATCH) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "voteseg_targets: %d samples, at most %d", batch, VS_MAX_BATCH);
  int rc = check_offsets(c, "voteseg_targets", point_offsets, batch, INT_MAX);
  if (!rc) rc = check_offsets(c, "voteseg_targets", gt_offsets, batch, VS_MAX_GT);
  if (rc) return rc;
  int max_pts = 0;
  for (int b = 0; b < batch; b++) max_pts = std::max(max_pts, point_offsets[b + 1] - point_offsets[b]);
  const int N = point_offsets[batch], G = gt_offsets[batch];
  CHECK_ARG(c, N == 0 || (points && labels && vote_targets && vote_mask));
  CHECK_ARG(c, G == 0 || (gt_boxes && gt_labels));
  if (N == 0) return SSTB_OK;
  VsTargetArgs a;
  a.pts = points, a.stride = point_stride, a.gt = gt_boxes, a.gl = gt_labels, a.bg_label = bg_label;
  for (int b = 0; b <= batch; b++) a.pt_off[b] = point_offsets[b], a.gt_off[b] = gt_offsets[b];
  a.labels = labels, a.vt = vote_targets, a.mask = vote_mask;
  const dim3 grid((unsigned)((max_pts + VS_THREADS - 1) / VS_THREADS), (unsigned)batch);
  vs_targets_kernel<<<grid, VS_THREADS, 0, c->stream>>>(a);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_voteseg_loss_forward(sstb200_ctx* c, const sstb200_voteseg_cfg* cfg, const float* seg_logits, int64_t logit_stride,
                                            const float* vote_preds, int64_t vote_stride, int64_t num_points, const int64_t* labels,
                                            const float* vote_targets, const uint8_t* vote_mask, float* losses, int64_t* num_valid,
                                            int64_t* counts) {
  VsLossArgs a;
  int rc = vs_loss_args(c, cfg, seg_logits, logit_stride, vote_preds, vote_stride, num_points, labels, vote_targets, vote_mask, a);
  if (rc) return rc;
  CHECK_ARG(c, losses && num_valid && counts);
  const int nb = loss_grid(c, a.n);
  arena_reset(c);
  double* part;
  int* ipart;
  rc = arena_carve(c, [&](Carve& cv) {
    part = cv.take<double>(2 * (size_t)nb);
    ipart = cv.take<int>((size_t)VS_NINT(a.E) * nb);
  });
  if (rc) return rc;
  vs_loss_forward_kernel<<<nb, LOSS_THREADS, 0, c->stream>>>(a, part, ipart, nb);
  LAUNCH_CHECK(c);
  vs_loss_final_kernel<<<1, LOSS_THREADS, 0, c->stream>>>(part, ipart, nb, a.E, a.n, a.C, a.softmax, cfg->loss_weight,
                                                          cfg->loss_weight_vote, losses, num_valid, counts);
  LAUNCH_CHECK(c);
  vs_vote_nonfinite_kernel<<<loss_grid(c, a.n * 3 * a.C), LOSS_THREADS, 0, c->stream>>>(a, num_valid, losses);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_voteseg_loss_backward(sstb200_ctx* c, const sstb200_voteseg_cfg* cfg, const float* seg_logits, int64_t logit_stride,
                                             const float* vote_preds, int64_t vote_stride, int64_t num_points, const int64_t* labels,
                                             const float* vote_targets, const uint8_t* vote_mask, const int64_t* num_valid,
                                             const float* grad_losses, float* grad_logits, float* grad_vote_preds) {
  VsLossArgs a;
  int rc = vs_loss_args(c, cfg, seg_logits, logit_stride, vote_preds, vote_stride, num_points, labels, vote_targets, vote_mask, a);
  if (rc) return rc;
  CHECK_ARG(c, num_valid && grad_losses && grad_logits && grad_vote_preds);
  vs_loss_backward_kernel<<<loss_grid(c, a.n), LOSS_THREADS, 0, c->stream>>>(a, cfg->loss_weight, cfg->loss_weight_vote, num_valid,
                                                                             grad_losses, grad_logits, grad_vote_preds);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
