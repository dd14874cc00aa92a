// FSD's second stage, GroupCorrectionHead + FullySparseBboxHead (mmdet3d/models/roi_heads/fsd_roi_head.py, bbox_heads/fsd_bbox_head.py,
// core/bbox/samplers/iou_neg_piecewise_sampler.py): RoI assignment and sampling, the RoI targets and the fused RoI losses.  fp32 in and
// out, stream-ordered.
//
// Assignment and sampling, one CTA per sample (rs_assign_sample_kernel):
//   max     per proposal: the max 3-D IoU over the GTs its assigner sees and the first GT attaining it; per GT: the max over those
//           proposals (heads.cuh's warp_max_iou into shared memory, as anchor3d.cu's assigner)
//   lowq    per proposal: the last GT whose max it attains (match_low_quality with gt_max_assign_all)
//   assign  mmdet 2.14 assign_wrt_overlaps; then the sampler: the positives, then the negatives piece by piece.  Where the reference
//           draws random_choice(gallery, k) the kernel keeps the k members with the smallest caller-given keys (ties: lower index).
//   write   positives by ascending proposal index, then negatives by ascending index (the reference's two `unique` calls)
// The IoU is LiDARInstance3DBoxes.overlaps(gt, proposal): bev_overlap (bev_overlap.cuh, the kernel of boxes_overlap_bev) times the
// overlap of [z, z + h], over max(v_gt + v_proposal - overlap, 1e-8), each step a correctly rounded fp32 operation as in torch.
// It is recomputed per (proposal, GT) pair in both passes, never stored.
//
// Targets (rs_targets_kernel): one thread per sampled row: the soft label, the canonical transform and the encode in double, rounded once.
// Losses: forward = block partials in double, one block sums them in a fixed order; backward = one pass, each row writes its own
// gradient rows, no atomics.
#include <stdarg.h>
#include "bev_overlap.cuh"
#include "heads.cuh"

namespace {

#define RS_THREADS 512
#define RS_MAX_CLASSES 8
#define RS_MAX_PIECES 8
#define RS_MAX_PROPOSALS 4096  // per sample
#define RS_MAX_GT 4096         // per sample: the per-GT maxima live in shared memory

#define RS_PI 3.14159265358979323846
#define RS_2PI 6.28318530717958647692

struct Box3 {
  BevBox bev;
  float zb, zt, vol;
};

// LiDARInstance3DBoxes (x, y, z_bottom, w, l, h, yaw): xywhr2xyxyr(bev), bottom / top height and volume, in torch's fp32 order
__device__ __forceinline__ Box3 load_box3(const float* __restrict__ p) {
  const float hw = __fdiv_rn(p[3], 2.f), hl = __fdiv_rn(p[4], 2.f);
  const float q[5] = {__fsub_rn(p[0], hw), __fsub_rn(p[1], hl), __fadd_rn(p[0], hw), __fadd_rn(p[1], hl), p[6]};
  Box3 b;
  b.bev = make_bev(q);
  b.zb = p[2];
  b.zt = __fadd_rn(p[2], p[5]);
  b.vol = __fmul_rn(__fmul_rn(p[3], p[4]), p[5]);
  return b;
}

// base_box3d.py:396-450, mode 'iou', boxes1 = the GT (MaxIoUAssigner calls iou_calculator(gt_bboxes, bboxes))
__device__ __forceinline__ float iou3d(const Box3& g, const Box3& p) {
  const float ov_h = fmaxf(__fsub_rn(fminf(g.zt, p.zt), fmaxf(g.zb, p.zb)), 0.f);
  const float ov = __fmul_rn(bev_overlap(g.bev, p.bev), ov_h);
  return __fdiv_rn(ov, fmaxf(__fsub_rn(__fadd_rn(g.vol, p.vol), ov), 1e-8f));
}

struct RsArgs {
  const float* props;   // [P, pw]
  const int64_t* plab;  // [P]
  const float* keys;    // [P]
  const float* gt;      // [G, gw]
  const int64_t* glab;  // [G]
  const int32_t* poff;  // device [B + 1]
  const int32_t* goff;  // device [B + 1]
  int pw, gw, per_class, num_classes;
  float pos_thr[RS_MAX_CLASSES], neg_thr[RS_MAX_CLASSES], min_pos[RS_MAX_CLASSES];
  int num, num_pos, num_pieces;
  double piece_frac[RS_MAX_PIECES];
  float piece_thr[RS_MAX_PIECES];
  // temporaries [P]
  float* mo;
  int* gi;  // assigned GT, sample-local 1-based; 0 negative, -1 ignored
  int* sel; // 1 sampled positive, 2 sampled negative
  // outputs, sample b at rows [b * num, b * num + counts[2 b + 1])
  int64_t *out_idx, *out_gt, *out_label;
  float* out_iou;
  int32_t* counts;  // [B, 2]: sampled positives, sampled rows
};

__device__ __forceinline__ bool sees(const RsArgs& a, int c, int g) { return !a.per_class || a.glab[g] == (int64_t)c; }

// the assigner of proposal i: its predicted class, -1 when no assigner takes it
__device__ __forceinline__ int assigner_of(const RsArgs& a, int i) {
  if (!a.per_class) return 0;
  const int64_t c = a.plab[i];
  return c >= 0 && c < a.num_classes ? (int)c : -1;
}

// Marks with `mark` the k members of {i in [p0, p1): pred(i)} with the smallest (key, i), all of them when there are at most k.  n is
// the member count.  O(n^2 / threads): the samples hold hundreds of proposals.
template <typename Pred>
__device__ void select_smallest(const RsArgs& a, int p0, int p1, int n, int k, int mark, Pred pred) {
  for (int i = p0 + threadIdx.x; i < p1; i += blockDim.x) {
    if (!pred(i)) continue;
    bool take = n <= k;
    if (!take && k > 0) {
      const float ki = a.keys[i];
      int rank = 0;
      for (int j = p0; j < p1 && rank < k; j++)
        if (j != i && pred(j)) {
          const float kj = a.keys[j];
          rank += (kj < ki || (kj == ki && j < i));
        }
      take = rank < k;
    }
    if (take) a.sel[i] = mark;
  }
  __syncthreads();
}

template <typename Pred>
__device__ int block_count(int p0, int p1, Pred pred) {
  int n = 0;
  for (int base = p0; base < p1; base += blockDim.x) {
    const int i = base + threadIdx.x;
    n += __syncthreads_count(i < p1 && pred(i));
  }
  return n;
}

// writes the rows with sel == mark in ascending index from row `at`; returns the number written
__device__ int block_write(const RsArgs& a, int b, int p0, int p1, int at, int mark, int* warp_off) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int g0 = a.goff[b];
  for (int base = p0; base < p1; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const bool on = i < p1 && a.sel[i] == mark;
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if (lane == 0) warp_off[warp] = __popc(bal);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < nw; w++) {
      before += w < warp ? warp_off[w] : 0;
      tot += warp_off[w];
    }
    if (on) {
      const long long r = (long long)b * a.num + at + before + __popc(bal & ((1u << lane) - 1u));
      const int gi = a.gi[i];
      a.out_idx[r] = i;
      a.out_iou[r] = a.mo[i];
      a.out_gt[r] = gi > 0 ? g0 + gi - 1 : -1;
      a.out_label[r] = gi > 0 ? a.glab[g0 + gi - 1] : -1;
    }
    at += tot;
    __syncthreads();
  }
  return at;
}

__global__ void __launch_bounds__(RS_THREADS) rs_assign_sample_kernel(const __grid_constant__ RsArgs a) {
  __shared__ unsigned gmax[RS_MAX_GT];
  __shared__ int warp_off[RS_THREADS / 32];
  const int b = blockIdx.x;
  const int p0 = a.poff[b], p1 = a.poff[b + 1], g0 = a.goff[b], g1 = a.goff[b + 1];
  for (int g = threadIdx.x; g < g1 - g0; g += blockDim.x) gmax[g] = 0u;
  __syncthreads();
  // max: every thread of a warp walks the same GTs, so the warp max is uniform
  for (int base = p0; base < p1; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const bool live = i < p1;
    const int c = live ? assigner_of(a, i) : -1;
    Box3 p;
    if (c >= 0) p = load_box3(a.props + (size_t)i * a.pw);
    float best = -1.f;
    int arg = -1;
    for (int g = g0; g < g1; g++) {
      float iou = 0.f;
      if (c >= 0 && sees(a, c, g)) {
        iou = iou3d(load_box3(a.gt + (size_t)g * a.gw), p);
        if (iou > best) best = iou, arg = g - g0;
      }
      warp_max_iou(gmax + (g - g0), __float_as_uint(iou));
    }
    if (live) {
      a.mo[i] = best;
      a.gi[i] = arg;  // argmax, rewritten below
    }
  }
  __syncthreads();
  // lowq + assign
  for (int i = p0 + threadIdx.x; i < p1; i += blockDim.x) {
    const int c = assigner_of(a, i);
    const int arg = a.gi[i];
    int gi = 0;
    float mo = 0.f;  // no assigner, or no GT for it: negative with max_overlaps 0
    if (c >= 0 && arg >= 0) {
      mo = a.mo[i];
      const Box3 p = load_box3(a.props + (size_t)i * a.pw);
      int lq = 0;
      for (int g = g0; g < g1; g++) {
        if (!sees(a, c, g)) continue;
        const float m = __uint_as_float(gmax[g - g0]);
        if (m >= a.min_pos[c] && iou3d(load_box3(a.gt + (size_t)g * a.gw), p) == m) lq = g - g0 + 1;
      }
      gi = -1;
      if (mo >= 0.f && mo < a.neg_thr[c]) gi = 0;
      if (mo >= a.pos_thr[c]) gi = arg + 1;
      if (lq > 0) gi = lq;
    }
    a.mo[i] = mo;
    a.gi[i] = gi;
    a.sel[i] = 0;
  }
  __syncthreads();
  // IoUNegPiecewiseSampler.sample: positives
  const int npos = block_count(p0, p1, [&](int i) { return a.gi[i] > 0; });
  select_smallest(a, p0, p1, npos, a.num_pos, 1, [&](int i) { return a.gi[i] > 0; });
  const int npos_sel = min(npos, a.num_pos);
  // negatives
  const int nexp = a.num - npos_sel;
  const int nneg = block_count(p0, p1, [&](int i) { return a.gi[i] == 0; });
  if (nneg <= nexp) {
    select_smallest(a, p0, p1, nneg, nneg, 2, [&](int i) { return a.gi[i] == 0; });
  } else {
    int chosen = 0, extend = 0;
    for (int q = 0; q < a.num_pieces; q++) {
      const bool last = q == a.num_pieces - 1;
      const int want = last ? nexp - chosen : (int)((double)nexp * a.piece_frac[q]) + extend;
      const float lo = last ? 0.f : a.piece_thr[q + 1], hi = a.piece_thr[q];
      auto in_piece = [&](int i) { return a.gi[i] == 0 && a.mo[i] >= lo && a.mo[i] < hi; };
      const int n = block_count(p0, p1, in_piece);
      if (n < want) {
        select_smallest(a, p0, p1, n, n, 2, in_piece);
        extend += want - n;
        chosen += n;
      } else {
        select_smallest(a, p0, p1, n, want, 2, in_piece);
        extend = 0;
        chosen += want;
      }
    }
  }
  const int at = block_write(a, b, p0, p1, 0, 1, warp_off);
  const int total = block_write(a, b, p0, p1, at, 2, warp_off);
  if (threadIdx.x == 0) {
    a.counts[2 * b] = at;
    a.counts[2 * b + 1] = total;
  }
}

// ---- targets ---------------------------------------------------------------------------------------------------------------------
struct TgArgs {
  const float* rois;    // [R, rw]: the sampled proposals (7 or 9 columns)
  const float* iou;     // [R]
  const int64_t* gt_row;// [R], -1 on negatives
  const int64_t* label; // [R], -1 on negatives
  const float* gt;      // [G, gw]
  int rw, gw, num_classes;
  float pos_thr[RS_MAX_CLASSES], neg_thr[RS_MAX_CLASSES], span[RS_MAX_CLASSES];
  long long R;
  float* soft;          // [R]
  int64_t* reg_mask;    // [R]
  float* bbox_t;        // [R, 7], 0 on negatives
  float* pos_gt;        // [R, 7], 0 on negatives
};

__device__ __forceinline__ double pymod(double a, double m) { return a - floor(a / m) * m; }

__global__ void rs_targets_kernel(const __grid_constant__ TgArgs a) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= a.R) return;
  const long long g = a.gt_row[r];
  float* bt = a.bbox_t + r * 7;
  float* pg = a.pos_gt + r * 7;
  if (g < 0) {
    a.soft[r] = 0.f;
    a.reg_mask[r] = 0;
    for (int k = 0; k < 7; k++) bt[k] = 0.f, pg[k] = 0.f;
    return;
  }
  // get_multi_class_soft_label: fp32 compares and (iou - neg) / (pos - neg), the span formed in double from the thresholds as given
  const int c = (int)a.label[r];
  const float iou = a.iou[r];
  float s = 0.f;
  if (c >= 0 && c < a.num_classes) {
    if (iou > a.pos_thr[c]) s = 1.f;
    else if (!(iou < a.neg_thr[c])) s = __fdiv_rn(__fsub_rn(iou, a.neg_thr[c]), a.span[c]);
  } else {
    s = __int_as_float(0x7fffffff);  // a label outside the classes: the reference's masks leave no defined value
  }
  a.soft[r] = s;
  a.reg_mask[r] = 1;
  const float* p = a.rois + r * a.rw;
  const float* q = a.gt + g * a.gw;
  for (int k = 0; k < 7; k++) pg[k] = q[k];
  // _get_target_single: canonical transform into the RoI's frame, then DeltaXYZWLHRBBoxCoder.encode against the zero-centred RoI
  const double ry = pymod((double)p[6], RS_2PI);
  const double dx = (double)q[0] - p[0], dy = (double)q[1] - p[1], dz = (double)q[2] - p[2];
  double sa, ca;
  sincos(-(ry + 0.5 * RS_PI), &sa, &ca);
  const double lx = dx * ca + dy * sa, ly = -dx * sa + dy * ca;
  double yl = pymod((double)q[6] - ry, RS_2PI);
  if (yl > 0.5 * RS_PI && yl < 1.5 * RS_PI) yl = pymod(yl + RS_PI, RS_2PI);
  if (yl > RS_PI) yl -= RS_2PI;
  yl = fmin(fmax(yl, -0.5 * RS_PI), 0.5 * RS_PI);
  const double pw = p[3], pl = p[4], ph = p[5];
  const double diag = sqrt(pl * pl + pw * pw);
  bt[0] = (float)(lx / diag);
  bt[1] = (float)(ly / diag);
  bt[2] = (float)((dz + 0.5 * q[5] - 0.5 * ph) / ph);
  bt[3] = (float)log(q[3] / pw);
  bt[4] = (float)log(q[4] / pl);
  bt[5] = (float)log(q[5] / ph);
  bt[6] = (float)yl;
}

// ---- losses ----------------------------------------------------------------------------------------------------------------------
#define RL_NPART 5  // cls, bbox, corner sums; positive and corner-row counts

struct LsArgs {
  const float* cls;      // [R] (row stride cls_stride)
  const float* pred;     // [R, 7] (row stride pred_stride)
  long long cls_stride, pred_stride;
  const uint8_t* nonempty;   // [R]
  const float* soft;         // [R]
  const int64_t* reg_mask;   // [R]
  const float* bbox_t;       // [R, 7]
  const float* pos_gt;       // [R, 7]
  const int64_t* label;      // [R]
  const float* rois;         // [R, rw] (without the batch column)
  int rw;
  long long R;
  const float* cls_avg;      // device [1]
  const float* reg_avg;      // device [1]
  int smooth_l1, with_corner, car;  // car: the class of the corner loss, -1 for all
  float beta, w_cls, w_bbox, w_corner;
  float cw[7];
};

__device__ __forceinline__ bool reg_row(const LsArgs& a, long long r) { return a.reg_mask[r] > 0 && a.nonempty[r]; }
__device__ __forceinline__ bool corner_row(const LsArgs& a, long long r) {
  return a.with_corner && reg_row(a, r) && (a.car < 0 || a.label[r] == (int64_t)a.car);
}

__device__ __forceinline__ float reg_elem(const LsArgs& a, float d) {
  const float ad = fabsf(d);
  return a.smooth_l1 ? (ad < a.beta ? 0.5f * d * d / a.beta : ad - 0.5f * a.beta) : ad;
}
__device__ __forceinline__ float reg_grad(const LsArgs& a, float d) {
  return a.smooth_l1 && fabsf(d) < a.beta ? d / a.beta : abs_grad(d);
}

// get_corner_loss_lidar of one row: the prediction decoded against its RoI (decode, rotate by roi_yaw + pi / 2, shift), its corners
// against the nearer of the GT's and the heading-flipped GT's, Huber (delta 1), summed over the 8 corners.  With grad != nullptr, also
// d(sum) / d(bbox_pred row) into grad[7].  rotation_3d_in_axis(axis 2) maps (x, y) to (x cos + y sin, -x sin + y cos).
__device__ double corner_row_loss(const float* p, const float* roi, const float* gt, double* grad) {
  const double pw = roi[3], pl = roi[4], ph = roi[5], pr = roi[6];
  const double diag = sqrt(pl * pl + pw * pw);
  const double xl = p[0] * diag, yl = p[1] * diag;
  const double w = exp((double)p[3]) * pw, l = exp((double)p[4]) * pl, h = exp((double)p[5]) * ph;
  const double zc = p[2] * ph + 0.5 * ph - 0.5 * h;
  const double yaw = (double)p[6] + pr;
  double sa, ca, sy, cy, sg, cg;
  sincos(pr + 0.5 * RS_PI, &sa, &ca);
  sincos(yaw, &sy, &cy);
  sincos((double)gt[6], &sg, &cg);
  const double cx = xl * ca + yl * sa + roi[0], cyy = -xl * sa + yl * ca + roi[1], cz = zc + roi[2];
  double gcx = 0, gcy = 0, gcz = 0, gyaw = 0, gw = 0, gl = 0, gh = 0, loss = 0;
  for (int k = 0; k < 8; k++) {
    // corners_norm[[0, 1, 3, 2, 4, 5, 7, 6]] - (0.5, 0.5, 0)
    const int bits = (k & 4) | ((k & 2) ? ((k & 1) ? 2 : 3) : (k & 1));
    const double ux = ((bits >> 2) & 1) - 0.5, uy = ((bits >> 1) & 1) - 0.5, uz = bits & 1;
    const double ox = ux * w, oy = uy * l, oz = uz * h;
    const double X = ox * cy + oy * sy + cx, Y = -ox * sy + oy * cy + cyy, Z = oz + cz;
    const double gox = ux * gt[3], goy = uy * gt[4];
    const double GX = gox * cg + goy * sg + gt[0], GY = -gox * sg + goy * cg + gt[1], GZ = uz * gt[5] + gt[2];
    const double FX = -gox * cg - goy * sg + gt[0], FY = gox * sg - goy * cg + gt[1];  // yaw + pi
    const double ex = X - GX, ey = Y - GY, ez = Z - GZ, fx = X - FX, fy = Y - FY;
    const double d1 = sqrt(ex * ex + ey * ey + ez * ez), d2 = sqrt(fx * fx + fy * fy + ez * ez);
    const double d = fmin(d1, d2);
    const double qd = fmin(d, 1.0);
    loss += 0.5 * qd * qd + (d - qd);
    if (grad) {
      const double hg = d <= 1.0 ? d : 1.0;  // d huber / d d (0 at d = 0)
      // torch.min splits a tie's gradient in half; torch.norm's gradient is 0 at 0
      const double w1 = d1 < d2 ? 1.0 : (d1 == d2 ? 0.5 : 0.0), w2 = 1.0 - w1;
      const double a1 = d1 > 0 ? hg * w1 / d1 : 0.0, a2 = d2 > 0 ? hg * w2 / d2 : 0.0;
      const double gX = a1 * ex + a2 * fx, gY = a1 * ey + a2 * fy, gZ = (a1 + a2) * ez;
      gcx += gX;
      gcy += gY;
      gcz += gZ;
      gyaw += gX * (-ox * sy + oy * cy) + gY * (-ox * cy - oy * sy);
      gw += ux * (gX * cy - gY * sy);
      gl += uy * (gX * sy + gY * cy);
      gh += uz * gZ;
    }
  }
  if (grad) {
    grad[0] = diag * (gcx * ca - gcy * sa);
    grad[1] = diag * (gcx * sa + gcy * ca);
    grad[2] = gcz * ph;
    grad[3] = gw * w;
    grad[4] = gl * l;
    grad[5] = (gh - 0.5 * gcz) * h;
    grad[6] = gyaw;
  }
  return loss;
}

__global__ void __launch_bounds__(LOSS_THREADS) rl_forward_kernel(const LsArgs a, double* part) {
  __shared__ double sh[LOSS_THREADS / 32];
  double acc[RL_NPART] = {0, 0, 0, 0, 0};
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < a.R; r += (long long)gridDim.x * blockDim.x) {
    if (a.nonempty[r]) {
      const Sig g = sig(a.cls[r * a.cls_stride]);
      const float y = a.soft[r];
      acc[0] += (double)((1.f - y) * g.sp_pos + y * g.sp_neg);
    }
    if (!reg_row(a, r)) continue;
    const float* p = a.pred + r * a.pred_stride;
    float s = 0.f;
    for (int k = 0; k < 7; k++) s += reg_elem(a, p[k] - a.bbox_t[r * 7 + k]) * a.cw[k];
    acc[1] += (double)s;
    acc[3] += 1.0;
    if (corner_row(a, r)) {
      float pf[7];
      for (int k = 0; k < 7; k++) pf[k] = p[k];
      acc[2] += corner_row_loss(pf, a.rois + r * a.rw, a.pos_gt + r * 7, nullptr);
      acc[4] += 1.0;
    }
  }
  for (int k = 0; k < RL_NPART; k++) {
    const double s = thread0_block_sum(acc[k], sh);
    if (threadIdx.x == 0) part[(size_t)k * gridDim.x + blockIdx.x] = s;
  }
}

// losses [3] = (cls, bbox, corner); counts [2] = (positives on non-empty RoIs, corner rows), for the backward
__global__ void __launch_bounds__(LOSS_THREADS) rl_final_kernel(const LsArgs a, const double* part, int nb, float* losses, float* counts) {
  __shared__ double sh[LOSS_THREADS / 32];
  double s[RL_NPART];
  for (int k = 0; k < RL_NPART; k++) s[k] = sum_partials(part, nb, k, sh);
  if (threadIdx.x) return;
  losses[0] = (float)((double)a.w_cls * s[0] / (double)a.cls_avg[0]);
  losses[1] = s[3] > 0 ? (float)((double)a.w_bbox * s[1] / (double)a.reg_avg[0]) : 0.f;
  losses[2] = s[4] > 0 ? (float)((double)a.w_corner * s[2] / (8.0 * s[4])) : 0.f;
  counts[0] = (float)s[3];
  counts[1] = (float)s[4];
}

__global__ void __launch_bounds__(LOSS_THREADS) rl_backward_kernel(const LsArgs a, const float* counts, const float* grad_losses,
                                                                   float* grad_cls, float* grad_pred) {
  const float gc = grad_losses[0] * a.w_cls / a.cls_avg[0];
  const float gb = counts[0] > 0.f ? grad_losses[1] * a.w_bbox / a.reg_avg[0] : 0.f;
  const double gk = counts[1] > 0.f ? (double)grad_losses[2] * a.w_corner / (8.0 * counts[1]) : 0.0;
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < a.R; r += (long long)gridDim.x * blockDim.x) {
    float gx = 0.f;
    if (a.nonempty[r]) {
      const Sig g = sig(a.cls[r * a.cls_stride]);
      gx = gc * (g.s - a.soft[r]);
    }
    grad_cls[r] = gx;
    float* gp = grad_pred + r * 7;
    if (!reg_row(a, r)) {
      for (int k = 0; k < 7; k++) gp[k] = 0.f;
      continue;
    }
    const float* p = a.pred + r * a.pred_stride;
    float pf[7];
    for (int k = 0; k < 7; k++) pf[k] = p[k];
    double cg[7] = {0, 0, 0, 0, 0, 0, 0};
    if (corner_row(a, r)) corner_row_loss(pf, a.rois + r * a.rw, a.pos_gt + r * 7, cg);
    for (int k = 0; k < 7; k++) gp[k] = gb * a.cw[k] * reg_grad(a, pf[k] - a.bbox_t[r * 7 + k]) + (float)(gk * cg[k]);
  }
}

int check_loss(sstb200_ctx* c, const sstb200_roi_loss_cfg* cfg, const float* cls, int64_t cls_stride, const float* pred,
               int64_t pred_stride, const uint8_t* nonempty, const float* soft, const int64_t* reg_mask, const float* bbox_t,
               const float* pos_gt, const int64_t* label, const float* rois, int roi_width, int64_t R, const float* cls_avg,
               const float* reg_avg) {
  CHECK_ARG(c, c && cfg && R >= 1 && cls && pred && nonempty && soft && reg_mask && bbox_t && pos_gt && label && rois && cls_avg && reg_avg);
  CHECK_ARG(c, cls_stride >= 1 && pred_stride >= 7 && (roi_width == 7 || roi_width == 9));
  if (cfg->smooth_l1 && !(cfg->beta > 0.f)) return sstb_fail(c, SSTB_ERR_ARG, "roi_head_loss: SmoothL1 beta must be > 0, got %g", cfg->beta);
  return SSTB_OK;
}

LsArgs loss_args(const sstb200_roi_loss_cfg* cfg, const float* cls, int64_t cls_stride, const float* pred, int64_t pred_stride,
                 const uint8_t* nonempty, const float* soft, const int64_t* reg_mask, const float* bbox_t, const float* pos_gt,
                 const int64_t* label, const float* rois, int roi_width, int64_t R, const float* cls_avg, const float* reg_avg) {
  LsArgs a;
  a.cls = cls, a.pred = pred, a.cls_stride = cls_stride, a.pred_stride = pred_stride, a.nonempty = nonempty, a.soft = soft;
  a.reg_mask = reg_mask, a.bbox_t = bbox_t, a.pos_gt = pos_gt, a.label = label, a.rois = rois, a.rw = roi_width, a.R = R;
  a.cls_avg = cls_avg, a.reg_avg = reg_avg;
  a.smooth_l1 = cfg->smooth_l1, a.with_corner = cfg->with_corner_loss, a.car = cfg->corner_class;
  a.beta = cfg->beta, a.w_cls = cfg->loss_weight_cls, a.w_bbox = cfg->loss_weight_bbox, a.w_corner = cfg->corner_loss_weight;
  for (int k = 0; k < 7; k++) a.cw[k] = cfg->code_weights[k];
  return a;
}

}  // namespace

extern "C" int sstb200_roi_assign_sample(sstb200_ctx* c, const sstb200_roi_sample_cfg* cfg, const float* proposals, int prop_width,
                                         const int64_t* prop_labels, const float* keys, const int32_t* prop_offsets, const float* gt_boxes,
                                         int gt_width, const int64_t* gt_labels, const int32_t* gt_offsets, int batch, int64_t* out_inds,
                                         float* out_iou, int64_t* out_gt, int64_t* out_labels, int32_t* counts) {
  CHECK_ARG(c, c && cfg && prop_offsets && gt_offsets && batch >= 1 && counts && out_inds && out_iou && out_gt && out_labels);
  CHECK_ARG(c, (prop_width == 7 || prop_width == 9) && (gt_width == 7 || gt_width == 9 || gt_width == 10));
  int rc = check_offsets(c, "roi_assign_sample", gt_offsets, batch, RS_MAX_GT);
  if (rc) return rc;
  CHECK_ARG(c, prop_offsets[0] == 0);
  for (int b = 0; b < batch; b++) {
    const int n = prop_offsets[b + 1] - prop_offsets[b];
    if (n < 1) return sstb_fail(c, SSTB_ERR_ARG, "roi_assign_sample: sample %d has no proposal (the caller adds the fake box)", b);
    if (n > RS_MAX_PROPOSALS)
      return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "roi_assign_sample: sample %d has %d proposals, at most %d", b, n, RS_MAX_PROPOSALS);
  }
  const int P = prop_offsets[batch], G = gt_offsets[batch];
  CHECK_ARG(c, proposals && prop_labels && keys && (G == 0 || (gt_boxes && gt_labels)));
  const int K = cfg->per_class ? cfg->num_classes : 1;
  if (K < 1 || K > RS_MAX_CLASSES) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "roi_assign_sample: %d assigners, 1 to %d supported", K, RS_MAX_CLASSES);
  if (cfg->num_pieces < 1 || cfg->num_pieces > RS_MAX_PIECES)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "roi_assign_sample: %d IoU pieces, 1 to %d supported", cfg->num_pieces, RS_MAX_PIECES);
  CHECK_ARG(c, cfg->num >= 1 && cfg->num_pos >= 0 && cfg->num_pos <= cfg->num);
  RsArgs a;
  a.props = proposals, a.plab = prop_labels, a.keys = keys, a.gt = gt_boxes, a.glab = gt_labels;
  a.pw = prop_width, a.gw = gt_width, a.per_class = cfg->per_class != 0, a.num_classes = K;
  for (int k = 0; k < K; k++) a.pos_thr[k] = cfg->pos_iou_thr[k], a.neg_thr[k] = cfg->neg_iou_thr[k], a.min_pos[k] = cfg->min_pos_iou[k];
  a.num = cfg->num, a.num_pos = cfg->num_pos, a.num_pieces = cfg->num_pieces;
  for (int q = 0; q < cfg->num_pieces; q++) a.piece_frac[q] = cfg->piece_fractions[q], a.piece_thr[q] = cfg->piece_thrs[q];
  a.out_idx = out_inds, a.out_iou = out_iou, a.out_gt = out_gt, a.out_label = out_labels, a.counts = counts;
  int32_t* offs = nullptr;
  arena_reset(c);
  rc = arena_carve(c, [&](Carve& cv) {
    offs = cv.take<int32_t>(2 * ((size_t)batch + 1));
    a.mo = cv.take<float>(P);
    a.gi = cv.take<int>(P);
    a.sel = cv.take<int>(P);
  });
  if (rc) return rc;
  std::vector<int32_t> host(2 * ((size_t)batch + 1));
  for (int b = 0; b <= batch; b++) host[b] = prop_offsets[b], host[batch + 1 + b] = gt_offsets[b];
  CUDA_TRY(c, cudaMemcpyAsync(offs, host.data(), host.size() * 4, cudaMemcpyHostToDevice, c->stream));
  a.poff = offs, a.goff = offs + batch + 1;
  rs_assign_sample_kernel<<<batch, RS_THREADS, 0, c->stream>>>(a);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_roi_head_targets(sstb200_ctx* c, const float* rois, int roi_width, const float* iou, const int64_t* gt_rows,
                                        const int64_t* labels, int64_t num_rows, const float* gt_boxes, int gt_width, int num_classes,
                                        const double* cls_pos_thr, const double* cls_neg_thr, float* soft_labels, int64_t* reg_mask,
                                        float* bbox_targets, float* pos_gt_bboxes) {
  CHECK_ARG(c, c && num_rows >= 0 && cls_pos_thr && cls_neg_thr);
  CHECK_ARG(c, (roi_width == 7 || roi_width == 9) && (gt_width == 7 || gt_width == 9 || gt_width == 10));
  if (num_classes < 1 || num_classes > RS_MAX_CLASSES)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "roi_head_targets: %d classes, 1 to %d supported", num_classes, RS_MAX_CLASSES);
  if (num_rows == 0) return SSTB_OK;
  CHECK_ARG(c, rois && iou && gt_rows && labels && soft_labels && reg_mask && bbox_targets && pos_gt_bboxes);
  TgArgs a;
  a.rois = rois, a.iou = iou, a.gt_row = gt_rows, a.label = labels, a.gt = gt_boxes, a.rw = roi_width, a.gw = gt_width;
  a.num_classes = num_classes, a.R = num_rows;
  for (int k = 0; k < num_classes; k++) {
    a.pos_thr[k] = (float)cls_pos_thr[k], a.neg_thr[k] = (float)cls_neg_thr[k];
    a.span[k] = (float)(cls_pos_thr[k] - cls_neg_thr[k]);  // Python's pos - neg in double, then fp32 as torch takes the scalar
  }
  a.soft = soft_labels, a.reg_mask = reg_mask, a.bbox_t = bbox_targets, a.pos_gt = pos_gt_bboxes;
  rs_targets_kernel<<<(unsigned)((num_rows + 255) / 256), 256, 0, c->stream>>>(a);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_roi_head_loss_forward(sstb200_ctx* c, const sstb200_roi_loss_cfg* cfg, const float* cls_score, int64_t cls_stride,
                                             const float* bbox_pred, int64_t pred_stride, const uint8_t* nonempty, const float* soft_labels,
                                             const int64_t* reg_mask, const float* bbox_targets, const float* pos_gt_bboxes,
                                             const int64_t* labels, const float* rois, int roi_width, int64_t num_rows,
                                             const float* cls_avg_factor, const float* reg_avg_factor, float* losses, float* counts) {
  int rc = check_loss(c, cfg, cls_score, cls_stride, bbox_pred, pred_stride, nonempty, soft_labels, reg_mask, bbox_targets, pos_gt_bboxes,
                      labels, rois, roi_width, num_rows, cls_avg_factor, reg_avg_factor);
  if (rc) return rc;
  CHECK_ARG(c, losses && counts);
  const LsArgs a = loss_args(cfg, cls_score, cls_stride, bbox_pred, pred_stride, nonempty, soft_labels, reg_mask, bbox_targets,
                             pos_gt_bboxes, labels, rois, roi_width, num_rows, cls_avg_factor, reg_avg_factor);
  const int nb = loss_grid(c, num_rows);
  double* part = nullptr;
  arena_reset(c);
  rc = arena_carve(c, [&](Carve& cv) { part = cv.take<double>((size_t)RL_NPART * nb); });
  if (rc) return rc;
  rl_forward_kernel<<<nb, LOSS_THREADS, 0, c->stream>>>(a, part);
  rl_final_kernel<<<1, LOSS_THREADS, 0, c->stream>>>(a, part, nb, losses, counts);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_roi_head_loss_backward(sstb200_ctx* c, const sstb200_roi_loss_cfg* cfg, const float* cls_score, int64_t cls_stride,
                                              const float* bbox_pred, int64_t pred_stride, const uint8_t* nonempty,
                                              const float* soft_labels, const int64_t* reg_mask, const float* bbox_targets,
                                              const float* pos_gt_bboxes, const int64_t* labels, const float* rois, int roi_width,
                                              int64_t num_rows, const float* cls_avg_factor, const float* reg_avg_factor,
                                              const float* counts, const float* grad_losses, float* grad_cls, float* grad_pred) {
  int rc = check_loss(c, cfg, cls_score, cls_stride, bbox_pred, pred_stride, nonempty, soft_labels, reg_mask, bbox_targets, pos_gt_bboxes,
                      labels, rois, roi_width, num_rows, cls_avg_factor, reg_avg_factor);
  if (rc) return rc;
  CHECK_ARG(c, counts && grad_losses && grad_cls && grad_pred);
  const LsArgs a = loss_args(cfg, cls_score, cls_stride, bbox_pred, pred_stride, nonempty, soft_labels, reg_mask, bbox_targets,
                             pos_gt_bboxes, labels, rois, roi_width, num_rows, cls_avg_factor, reg_avg_factor);
  rl_backward_kernel<<<loss_grid(c, num_rows), LOSS_THREADS, 0, c->stream>>>(a, counts, grad_losses, grad_cls, grad_pred);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
