// Anchor3DHead training path (mmdet3d/models/dense_heads/anchor3d_head.py:197-379, train_mixins.py:11-346): the anchor targets of one
// level with one MaxIoUAssigner per anchor size, the sigmoid focal loss of cls_score, and the positives' L1 (sin difference on the yaw) and
// direction cross-entropy, each with its backward.  fp32, stream-ordered, no host sync.
//
// Targets, seven launches for every sample and every size-assigner of a batch.  The anchors are never materialised: anchor
// ((y W + x) S + s) R + r is (x_centers[x], y_centers[y], z[s], w[s], l[s], h[s], rotations[r]), and the [G, A] IoU matrix is never
// stored: each pass recomputes an anchor's IoUs against its sample's GTs, staged through shared memory 256 at a time.
//   init    per-GT maxima 0, per-GT argmax anchor INT_MAX, positive counters 0, the valid-GT count of every (sample, size)
//   max     per anchor: max IoU and its first argmax; per GT: the max over anchors, combined by an integer max on the fp32 bits
//           (IoU >= 0, so integer order is float order and the result does not depend on the order of the writes)
//   lowq    per anchor: the last GT whose max it attains (gt_max_assign_all) or, per GT, the first anchor attaining it (atomicMin)
//   argmax  per GT (gt_max_assign_all = False only): its argmax anchor takes the largest such GT index (atomicMax: the last GT wins)
//   assign  per anchor: MaxIoUAssigner's three rules, then the sampler-free targets of anchor_target_single_assigner
//   total   num_total_pos = sum over samples of max(positives, 1)
// The IoU is the reference's sequence of correctly rounded fp32 operations (nearest_bev, then mmdet's bbox_overlaps), written with
// __f*_rn so that no contraction into an FMA can move an IoU across a threshold.
//
// Losses: forward = block partials in double, one block sums them in a fixed order; backward = one elementwise pass recomputing each
// derivative.  Every tensor is read in place in the head's NCHW layout: element (b, y, x, a, c) is channel a C + c.
#include <stdarg.h>
#include <algorithm>
#include <climits>
#include "heads.cuh"

namespace {

#define A3_THREADS 256  // targets block
#define A3_MAX_BATCH 256
#define A3_MAX_SIZES 8
#define A3_MAX_ROTS 8
#define A3_MAX_GT 4096

// fp32 of the Python scalars np.pi, np.pi / 4 and 2 * np.pi, as a float tensor compares / divides with them
#define A3_PI 3.14159265358979323846f
#define A3_PI_4 0.785398163397448309616f
#define A3_2PI 6.28318530717958647692f

struct A3Args {
  const float* xc;   // [W]
  const float* yc;   // [H]
  const float* sz;   // [S]
  const float* wlh;  // [S, 3]
  const float* rot;  // [R]
  const float* gt;   // [N, 7] bottom-centre (x, y, z, w, l, h, yaw)
  const int64_t* gl; // [N]
  int sample_off[A3_MAX_BATCH + 1];
  float pos_thr[A3_MAX_SIZES], neg_thr[A3_MAX_SIZES], min_pos[A3_MAX_SIZES];
  int assign_all[A3_MAX_SIZES];
  int B, W, H, S, R, N, per_class, num_classes;
  float dir_offset;
  // outputs
  int64_t* labels;
  float* label_w;
  float* bbox_t;
  float* bbox_w;
  int64_t* dir_t;
  float* dir_w;
  int64_t* num_total_pos;
  // temporaries
  unsigned* gt_max;  // [S, N] fp32 bits
  int* gt_arg;       // [S, N] first anchor (within its size) attaining gt_max
  int* nvalid;       // [B, S]
  int* npos;         // [B]
  float* max_iou;    // [B, A]
  int* argmax;       // [B, A] sample-local GT index
  int* lowq;         // [B, A] sample-local GT index + 1, 0 = none
};

struct Bev {
  float x1, y1, x2, y2, area;
};

// LiDARInstance3DBoxes.nearest_bev (lidar_box3d.py:123-145): the axis-aligned BEV box, w and l swapped when
// |limit_period(yaw, 0.5, pi)| > pi / 4; then mmdet's area (x2 - x1) * (y2 - y1)
__device__ __forceinline__ Bev nearest_bev(float x, float y, float w, float l, float yaw) {
  const float lp = __fsub_rn(yaw, __fmul_rn(floorf(__fadd_rn(__fdiv_rn(yaw, A3_PI), 0.5f)), A3_PI));
  const bool swap = fabsf(lp) > A3_PI_4;
  const float hx = __fdiv_rn(swap ? l : w, 2.f), hy = __fdiv_rn(swap ? w : l, 2.f);
  Bev b;
  b.x1 = __fsub_rn(x, hx);
  b.y1 = __fsub_rn(y, hy);
  b.x2 = __fadd_rn(x, hx);
  b.y2 = __fadd_rn(y, hy);
  b.area = __fmul_rn(__fsub_rn(b.x2, b.x1), __fsub_rn(b.y2, b.y1));
  return b;
}

// mmdet 2.14 bbox_overlaps(gt, anchor), mode 'iou': clamp(rb - lt, 0), overlap / max(area_gt + area_anchor - overlap, 1e-6)
__device__ __forceinline__ float bev_iou(const Bev& g, const Bev& a) {
  const float w = fmaxf(__fsub_rn(fminf(g.x2, a.x2), fmaxf(g.x1, a.x1)), 0.f);
  const float h = fmaxf(__fsub_rn(fminf(g.y2, a.y2), fmaxf(g.y1, a.y1)), 0.f);
  const float ov = __fmul_rn(w, h);
  const float un = fmaxf(__fsub_rn(__fadd_rn(g.area, a.area), ov), 1e-6f);
  return __fdiv_rn(ov, un);
}

__device__ __forceinline__ bool gt_valid(const A3Args& a, int g, int s) { return !a.per_class || a.gl[g] == (int64_t)s; }

__device__ __forceinline__ void anchor_box(const A3Args& a, int s, int cell, int r, float* box) {
  box[0] = __ldg(a.xc + cell % a.W);
  box[1] = __ldg(a.yc + cell / a.W);
  box[2] = __ldg(a.sz + s);
  box[3] = __ldg(a.wlh + 3 * s);
  box[4] = __ldg(a.wlh + 3 * s + 1);
  box[5] = __ldg(a.wlh + 3 * s + 2);
  box[6] = __ldg(a.rot + r);
}

__global__ void a3_init_kernel(const __grid_constant__ A3Args a) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long i = i0; i < (long long)a.S * a.N; i += stride) a.gt_max[i] = 0u, a.gt_arg[i] = INT_MAX;
  for (long long i = i0; i < (long long)a.B * a.S; i += stride) a.nvalid[i] = 0;
  for (long long i = i0; i < a.B; i += stride) a.npos[i] = 0;
}

__global__ void a3_count_kernel(const __grid_constant__ A3Args a) {
  const int b = blockIdx.x;
  for (int g = a.sample_off[b] + threadIdx.x; g < a.sample_off[b + 1]; g += blockDim.x)
    for (int s = 0; s < a.S; s++)
      if (gt_valid(a, g, s)) atomicAdd(a.nvalid + b * a.S + s, 1);
}

// PASS 0 (max): max / argmax per anchor, per-GT max.  PASS 1 (lowq): the low-quality matches.
template <int PASS>
__global__ void __launch_bounds__(A3_THREADS) a3_iou_kernel(const __grid_constant__ A3Args a) {
  __shared__ Bev sg[A3_THREADS];
  __shared__ int sv[A3_THREADS];
  __shared__ unsigned smax[A3_THREADS];
  const int b = blockIdx.y / a.S, s = blockIdx.y - b * a.S;
  const int per_size = a.H * a.W * a.R;
  const int j = blockIdx.x * A3_THREADS + threadIdx.x;  // anchor within this size: cell R + r
  const bool live = j < per_size;
  const int cell = live ? j / a.R : 0, r = live ? j - cell * a.R : 0;
  float box[7];
  anchor_box(a, s, cell, r, box);
  const Bev an = nearest_bev(box[0], box[1], box[3], box[4], box[6]);
  const long long slot = (long long)b * per_size * a.S + ((long long)cell * a.S + s) * a.R + r;
  const int begin = a.sample_off[b], end = a.sample_off[b + 1];
  const float min_pos = a.min_pos[s];
  const bool all = a.assign_all[s] != 0;
  float best = -1.f;
  int arg = 0, lq = 0;
  for (int c0 = begin; c0 < end; c0 += A3_THREADS) {
    const int n = min(A3_THREADS, end - c0);
    if (threadIdx.x < n) {
      const int g = c0 + threadIdx.x;
      const float* gb = a.gt + (size_t)g * 7;
      sg[threadIdx.x] = nearest_bev(gb[0], gb[1], gb[3], gb[4], gb[6]);
      bool v = gt_valid(a, g, s);
      smax[threadIdx.x] = PASS == 0 ? 0u : a.gt_max[(size_t)s * a.N + g];
      if (PASS == 1) v = v && __uint_as_float(smax[threadIdx.x]) >= min_pos;
      sv[threadIdx.x] = v;
    }
    __syncthreads();
    for (int k = 0; k < n; k++) {
      if (!sv[k]) continue;  // uniform over the block
      const float iou = bev_iou(sg[k], an);
      if (PASS == 0) {
        if (live && iou > best) best = iou, arg = c0 + k - begin;
        const unsigned m = __reduce_max_sync(0xffffffffu, live ? __float_as_uint(iou) : 0u);
        if ((threadIdx.x & 31) == 0 && m) atomicMax(smax + k, m);
      } else if (live && __float_as_uint(iou) == smax[k]) {
        if (all) lq = c0 + k - begin + 1;
        else atomicMin(a.gt_arg + (size_t)s * a.N + c0 + k, j);
      }
    }
    __syncthreads();
    if (PASS == 0 && threadIdx.x < n && smax[threadIdx.x]) atomicMax(a.gt_max + (size_t)s * a.N + c0 + threadIdx.x, smax[threadIdx.x]);
  }
  if (!live) return;
  if (PASS == 0) {
    a.max_iou[slot] = best;
    a.argmax[slot] = arg;
  } else {
    a.lowq[slot] = lq;
  }
}

// gt_max_assign_all = False: each GT gives its own argmax anchor to itself; later GTs overwrite earlier ones
__global__ void a3_argmax_kernel(const __grid_constant__ A3Args a) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)a.S * a.N; i += stride) {
    const int s = (int)(i / a.N), g = (int)(i - (long long)s * a.N);
    const int j = a.gt_arg[i];
    if (a.assign_all[s] || j == INT_MAX) continue;
    int lo = 0, hi = a.B;  // the sample owning g: the last b with sample_off[b] <= g
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (a.sample_off[mid] <= g) lo = mid;
      else hi = mid;
    }
    const int b = lo, cell = j / a.R, r = j - cell * a.R;
    atomicMax(a.lowq + (long long)b * a.H * a.W * a.S * a.R + ((long long)cell * a.S + s) * a.R + r, g - a.sample_off[b] + 1);
  }
}

__global__ void __launch_bounds__(A3_THREADS) a3_assign_kernel(const __grid_constant__ A3Args a) {
  __shared__ int warp_pos[A3_THREADS / 32];
  const int b = blockIdx.y / a.S, s = blockIdx.y - b * a.S;
  const int per_size = a.H * a.W * a.R;
  const int j = blockIdx.x * A3_THREADS + threadIdx.x;
  bool pos = false;
  if (j < per_size) {
    const int cell = j / a.R, r = j - cell * a.R;
    const long long slot = (long long)b * per_size * a.S + ((long long)cell * a.S + s) * a.R + r;
    int gi = 0;  // assigned_gt_inds: -1 ignored, 0 negative, i + 1 positive; a sample without valid GTs is all negative
    if (a.nvalid[b * a.S + s] > 0) {
      const float m = a.max_iou[slot];
      gi = -1;
      if (m >= 0.f && m < a.neg_thr[s]) gi = 0;
      if (m >= a.pos_thr[s]) gi = a.argmax[slot] + 1;
      const int lq = a.lowq[slot];
      if (lq > 0) gi = lq;
    }
    float* bt = a.bbox_t + slot * 7;
    float* bw = a.bbox_w + slot * 7;
    if (gi > 0) {
      pos = true;
      const int g = a.sample_off[b] + gi - 1;
      float an[7];
      anchor_box(a, s, cell, r, an);
      const float* gb = a.gt + (size_t)g * 7;
      // DeltaXYZWLHRBBoxCoder.encode (delta_xyzwhlr_bbox_coder.py:22-56)
      const float za = __fadd_rn(an[2], __fdiv_rn(an[5], 2.f)), zg = __fadd_rn(gb[2], __fdiv_rn(gb[5], 2.f));
      const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(an[4], an[4]), __fmul_rn(an[3], an[3])));
      const float rt = __fsub_rn(gb[6], an[6]);
      bt[0] = __fdiv_rn(__fsub_rn(gb[0], an[0]), diag);
      bt[1] = __fdiv_rn(__fsub_rn(gb[1], an[1]), diag);
      bt[2] = __fdiv_rn(__fsub_rn(zg, za), an[5]);
      bt[3] = logf(__fdiv_rn(gb[3], an[3]));
      bt[4] = logf(__fdiv_rn(gb[4], an[4]));
      bt[5] = logf(__fdiv_rn(gb[5], an[5]));
      bt[6] = rt;
#pragma unroll
      for (int k = 0; k < 7; k++) bw[k] = 1.f;
      // get_direction_target (train_mixins.py:317-346): floor(limit_period(rt + ra - dir_offset, 0, 2 pi) / pi), clamped to [0, 1]
      const float v = __fsub_rn(__fadd_rn(rt, an[6]), a.dir_offset);
      const float lp = __fsub_rn(v, __fmul_rn(floorf(__fadd_rn(__fdiv_rn(v, A3_2PI), 0.f)), A3_2PI));
      const float d = floorf(__fdiv_rn(lp, A3_PI));
      a.dir_t[slot] = d >= 1.f ? 1 : 0;
      a.dir_w[slot] = 1.f;
      a.labels[slot] = a.gl[g];
    } else {
#pragma unroll
      for (int k = 0; k < 7; k++) bt[k] = 0.f, bw[k] = 0.f;
      a.dir_t[slot] = 0;
      a.dir_w[slot] = 0.f;
      a.labels[slot] = a.num_classes;
    }
    a.label_w[slot] = gi >= 0 ? 1.f : 0.f;
  }
  const unsigned ballot = __ballot_sync(0xffffffffu, pos);
  if ((threadIdx.x & 31) == 0) warp_pos[threadIdx.x >> 5] = __popc(ballot);
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < A3_THREADS / 32; w++) t += warp_pos[w];
    if (t) atomicAdd(a.npos + b, t);
  }
}

__global__ void a3_total_kernel(const int* npos, int B, int64_t* num_total_pos) {
  if (threadIdx.x) return;
  long long t = 0;
  for (int b = 0; b < B; b++) t += max(npos[b], 1);
  *num_total_pos = t;
}

// ---- losses -------------------------------------------------------------------------------------------------------------------------
// sigmoid focal loss, gamma 2, alpha 0.25, on heads.cuh's sig.  Not heads.cuh's sigmoid_focal: q * q is other arithmetic than
// powf(q, 2.f).
#define FOCAL_ALPHA 0.25f

__device__ __forceinline__ float focal_loss(float x, bool t) {
  const Sig g = sig(x);
  return t ? FOCAL_ALPHA * g.q * g.q * g.sp_neg : (1.f - FOCAL_ALPHA) * g.s * g.s * g.sp_pos;
}

// d/dx: t = 1: -alpha q^2 (2 s softplus(-x) + q); t = 0: (1 - alpha) s^2 (2 q softplus(x) + s)
__device__ __forceinline__ float focal_grad(float x, bool t) {
  const Sig g = sig(x);
  return t ? -FOCAL_ALPHA * g.q * g.q * (2.f * g.s * g.sp_neg + g.q) : (1.f - FOCAL_ALPHA) * g.s * g.s * (2.f * g.q * g.sp_pos + g.s);
}

struct FocalArgs {
  const float* x;  // [B, A_loc C, H, W]
  const int64_t* labels;
  const float* label_w;
  long long HW, n;
  int A_loc, C;
};

// element i of cls_score -> (its anchor's label, weight)
__device__ __forceinline__ void focal_elem(const FocalArgs& a, long long i, bool& t, float& w) {
  const long long hw = i % a.HW, bc = i / a.HW;
  const int ch = (int)(bc % ((long long)a.A_loc * a.C));
  const long long b = bc / ((long long)a.A_loc * a.C);
  const int an = ch / a.C, c = ch - an * a.C;
  const long long slot = b * a.HW * a.A_loc + hw * a.A_loc + an;
  t = __ldg(a.labels + slot) == (int64_t)c;
  w = __ldg(a.label_w + slot);
}

__global__ void __launch_bounds__(LOSS_THREADS) focal_forward_kernel(const FocalArgs a, double* part) {
  __shared__ double sh[LOSS_THREADS / 32];
  double acc = 0.0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    bool t;
    float w;
    focal_elem(a, i, t, w);
    acc += (double)(focal_loss(__ldg(a.x + i), t) * w);
  }
  acc = thread0_block_sum(acc, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(LOSS_THREADS) focal_backward_kernel(const FocalArgs a, float loss_weight, const int64_t* num_total_pos,
                                                                      const float* grad_loss, float* grad_x) {
  const float scale = (float)((double)grad_loss[0] * loss_weight / (double)*num_total_pos);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    bool t;
    float w;
    focal_elem(a, i, t, w);
    grad_x[i] = scale * w * focal_grad(__ldg(a.x + i), t);
  }
}

// sum of nparts partials (per output k: part[k * nparts + i]) in a fixed order -> out[k] = weight[k] * sum / num_total_pos
__global__ void __launch_bounds__(LOSS_THREADS) a3_final_kernel(const double* part, int nparts, int nout, float w0, float w1,
                                                                const int64_t* num_total_pos, float* out0, float* out1) {
  __shared__ double sh[LOSS_THREADS / 32];
  for (int k = 0; k < nout; k++) {
    const double acc = sum_partials(part, nparts, k, sh);
    if (threadIdx.x == 0) *(k ? out1 : out0) = (float)((double)(k ? w1 : w0) * (acc / (double)*num_total_pos));
  }
}

struct RegArgs {
  const float* bbox;  // [B, A_loc 7, H, W]
  const float* dir;   // [B, A_loc 2, H, W]
  const int64_t* labels;
  const float* bbox_t;  // [B, A, 7]
  const float* bbox_w;
  const int64_t* dir_t;
  const float* dir_w;
  float cw[7];
  long long HW, n;  // n = B A_loc HW, enumerated as (b, a, cell) with the cell fastest
  int A_loc, C;
};

__device__ __forceinline__ void reg_index(const RegArgs& a, long long i, long long& slot, long long& base) {
  const long long hw = i % a.HW, ba = i / a.HW;
  const int an = (int)(ba % a.A_loc);
  const long long b = ba / a.A_loc;
  slot = b * a.HW * a.A_loc + hw * a.A_loc + an;
  base = (b * a.A_loc + an) * a.HW + hw;  // channel an of a 1-channel-per-anchor view; scaled by 7 / 2 below
}

__device__ __forceinline__ bool is_pos(const RegArgs& a, long long slot) {
  const int64_t l = __ldg(a.labels + slot);
  return l >= 0 && l < a.C;
}

__global__ void __launch_bounds__(LOSS_THREADS) reg_forward_kernel(const RegArgs a, double* part, int nparts) {
  __shared__ double sh[LOSS_THREADS / 32];
  double l1 = 0.0, ce = 0.0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    long long slot, base;
    reg_index(a, i, slot, base);
    if (!is_pos(a, slot)) continue;
    const long long hw = i % a.HW, ba = i / a.HW;
    const float* p = a.bbox + ba * 7 * a.HW + hw;
    const float* t = a.bbox_t + slot * 7;
    const float* w = a.bbox_w + slot * 7;
#pragma unroll
    for (int k = 0; k < 6; k++) l1 += (double)(fabsf(p[k * a.HW] - t[k]) * (w[k] * a.cw[k]));
    // add_sin_difference: sin(p) cos(t) against cos(p) sin(t), each product rounded as torch rounds it (no FMA contraction)
    const float p6 = p[6 * a.HW], t6 = t[6];
    l1 += (double)(fabsf(__fsub_rn(__fmul_rn(sinf(p6), cosf(t6)), __fmul_rn(cosf(p6), sinf(t6)))) * (w[6] * a.cw[6]));
    const float* d = a.dir + ba * 2 * a.HW + hw;
    const float z0 = d[0], z1 = d[a.HW];
    const float lse = fmaxf(z0, z1) + log1pf(expf(-fabsf(z0 - z1)));
    ce += (double)((lse - (a.dir_t[slot] ? z1 : z0)) * a.dir_w[slot]);
  }
  l1 = thread0_block_sum(l1, sh);
  ce = thread0_block_sum(ce, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = l1, part[nparts + blockIdx.x] = ce;
}

// every (b, anchor, cell) owns its 7 + 2 channels: the gradients are written in full, zero off the positives
__global__ void __launch_bounds__(LOSS_THREADS) reg_backward_kernel(const RegArgs a, float w_bbox, float w_dir,
                                                                    const int64_t* num_total_pos, const float* grad_loss, float* grad_bbox,
                                                                    float* grad_dir) {
  const double inv = 1.0 / (double)*num_total_pos;
  const float sb = (float)((double)grad_loss[0] * w_bbox * inv), sd = (float)((double)grad_loss[1] * w_dir * inv);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += stride) {
    long long slot, base;
    reg_index(a, i, slot, base);
    const long long hw = i % a.HW, ba = i / a.HW;
    float* gb = grad_bbox + ba * 7 * a.HW + hw;
    float* gd = grad_dir + ba * 2 * a.HW + hw;
    if (!is_pos(a, slot)) {
#pragma unroll
      for (int k = 0; k < 7; k++) gb[k * a.HW] = 0.f;
      gd[0] = 0.f;
      gd[a.HW] = 0.f;
      continue;
    }
    const float* p = a.bbox + ba * 7 * a.HW + hw;
    const float* t = a.bbox_t + slot * 7;
    const float* w = a.bbox_w + slot * 7;
#pragma unroll
    for (int k = 0; k < 6; k++) {
      const float df = p[k * a.HW] - t[k];
      gb[k * a.HW] = sb * (w[k] * a.cw[k]) * abs_grad(df);
    }
    const float p6 = p[6 * a.HW], t6 = t[6];
    float sp, cp, st, ct;
    sincosf(p6, &sp, &cp);
    sincosf(t6, &st, &ct);
    // rounded products: a predicted yaw equal to its target gives df = 0 exactly, and so a zero gradient, as in torch; a contracted
    // sp * ct - cp * st would leave the rounding residual of one product and a full-size gradient of either sign
    const float df = __fsub_rn(__fmul_rn(sp, ct), __fmul_rn(cp, st));
    // torch.abs' gradient is 0 at a NaN difference; a NaN yaw still makes its own gradient NaN through cos(p) cos(t) + sin(p) sin(t)
    gb[6 * a.HW] = sb * (w[6] * a.cw[6]) * abs_grad(df) * (cp * ct + sp * st);
    const float* d = a.dir + ba * 2 * a.HW + hw;
    const float z0 = d[0], z1 = d[a.HW];
    const float p1 = 1.f / (1.f + expf(z0 - z1)), p0 = 1.f / (1.f + expf(z1 - z0));
    const bool t1 = a.dir_t[slot] != 0;
    const float g = sd * a.dir_w[slot];
    gd[0] = g * (p0 - (t1 ? 0.f : 1.f));
    gd[a.HW] = g * (p1 - (t1 ? 1.f : 0.f));
  }
}

int focal_args(sstb200_ctx* c, const float* cls_score, int batch, int num_anchors, int num_classes, int height, int width,
               const int64_t* labels, const float* label_weights, const int64_t* num_total_pos, FocalArgs& a) {
  CHECK_ARG(c, cls_score && labels && label_weights && num_total_pos);
  CHECK_ARG(c, batch >= 1 && num_anchors >= 1 && num_classes >= 1 && height >= 1 && width >= 1);
  a.x = cls_score, a.labels = labels, a.label_w = label_weights;
  a.HW = (long long)height * width, a.A_loc = num_anchors, a.C = num_classes;
  a.n = (long long)batch * num_anchors * num_classes * a.HW;
  return SSTB_OK;
}

int reg_args(sstb200_ctx* c, const float* bbox_pred, const float* dir_cls_preds, int batch, int num_anchors, int num_classes, int height,
             int width, const int64_t* labels, const float* bbox_targets, const float* bbox_weights, const int64_t* dir_targets,
             const float* dir_weights, const float code_weight[7], const int64_t* num_total_pos, RegArgs& a) {
  CHECK_ARG(c, bbox_pred && dir_cls_preds && labels && bbox_targets && bbox_weights && dir_targets && dir_weights && code_weight &&
                   num_total_pos);
  CHECK_ARG(c, batch >= 1 && num_anchors >= 1 && num_classes >= 1 && height >= 1 && width >= 1);
  a.bbox = bbox_pred, a.dir = dir_cls_preds, a.labels = labels, a.bbox_t = bbox_targets, a.bbox_w = bbox_weights;
  a.dir_t = dir_targets, a.dir_w = dir_weights;
  for (int k = 0; k < 7; k++) a.cw[k] = code_weight[k];
  a.HW = (long long)height * width, a.A_loc = num_anchors, a.C = num_classes;
  a.n = (long long)batch * num_anchors * a.HW;
  return SSTB_OK;
}

}  // namespace

extern "C" int sstb200_anchor3d_targets(sstb200_ctx* c, const float* x_centers, int width, const float* y_centers, int height,
                                        const float* size_z, const float* size_wlh, int num_sizes, const float* rotations, int num_rots,
                                        const float* gt_boxes, const int64_t* gt_labels, const int32_t* sample_offsets, int batch,
                                        const float* pos_iou_thr, const float* neg_iou_thr, const float* min_pos_iou,
                                        const int32_t* gt_max_assign_all, int assign_per_class, int num_classes, float dir_offset,
                                        int64_t* labels, float* label_weights, float* bbox_targets, float* bbox_weights,
                                        int64_t* dir_targets, float* dir_weights, int64_t* num_total_pos) {
  CHECK_ARG(c, x_centers && y_centers && size_z && size_wlh && rotations && sample_offsets && pos_iou_thr && neg_iou_thr &&
                   min_pos_iou && gt_max_assign_all);
  CHECK_ARG(c, labels && label_weights && bbox_targets && bbox_weights && dir_targets && dir_weights && num_total_pos);
  CHECK_ARG(c, width >= 1 && height >= 1 && num_sizes >= 1 && num_rots >= 1 && batch >= 1 && num_classes >= 1);
  if (batch > A3_MAX_BATCH || num_sizes > A3_MAX_SIZES || num_rots > A3_MAX_ROTS)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "anchor3d_targets: %d samples / %d sizes / %d rotations, at most %d / %d / %d", batch,
                     num_sizes, num_rots, A3_MAX_BATCH, A3_MAX_SIZES, A3_MAX_ROTS);
  int rc = check_offsets(c, "anchor3d_targets", sample_offsets, batch, A3_MAX_GT);
  if (rc) return rc;
  const int N = sample_offsets[batch];
  CHECK_ARG(c, N == 0 || (gt_boxes && gt_labels));
  const long long per_size = (long long)height * width * num_rots;
  const long long A = per_size * num_sizes;
  if (A * batch >= (1LL << 31) / 8 || per_size >= (1LL << 31) - A3_THREADS)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "anchor3d_targets: %lld anchors x %d samples is too many", A, batch);
  A3Args a;
  a.xc = x_centers, a.yc = y_centers, a.sz = size_z, a.wlh = size_wlh, a.rot = rotations, a.gt = gt_boxes, a.gl = gt_labels;
  for (int b = 0; b <= batch; b++) a.sample_off[b] = sample_offsets[b];
  for (int s = 0; s < num_sizes; s++) {
    a.pos_thr[s] = pos_iou_thr[s], a.neg_thr[s] = neg_iou_thr[s], a.min_pos[s] = min_pos_iou[s];
    a.assign_all[s] = gt_max_assign_all[s] != 0;
  }
  a.B = batch, a.W = width, a.H = height, a.S = num_sizes, a.R = num_rots, a.N = N, a.per_class = assign_per_class != 0;
  a.num_classes = num_classes, a.dir_offset = dir_offset;
  a.labels = labels, a.label_w = label_weights, a.bbox_t = bbox_targets, a.bbox_w = bbox_weights, a.dir_t = dir_targets;
  a.dir_w = dir_weights, a.num_total_pos = num_total_pos;
  const size_t SN = std::max<size_t>(1, (size_t)num_sizes * N), BA = (size_t)batch * A;
  arena_reset(c);
  rc = arena_carve(c, [&](Carve& cv) {
    a.gt_max = cv.take<unsigned>(SN);
    a.gt_arg = cv.take<int>(SN);
    a.nvalid = cv.take<int>((size_t)batch * num_sizes);
    a.npos = cv.take<int>(batch);
    a.max_iou = cv.take<float>(BA);
    a.argmax = cv.take<int>(BA);
    a.lowq = cv.take<int>(BA);
  });
  if (rc) return rc;
  cudaStream_t st = c->stream;
  const int small = (int)std::min<long long>(c->num_sms * 4LL, std::max<long long>(1, ((long long)SN + A3_THREADS - 1) / A3_THREADS));
  a3_init_kernel<<<std::max(small, (batch * num_sizes + A3_THREADS - 1) / A3_THREADS), A3_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  a3_count_kernel<<<batch, A3_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  const dim3 grid((unsigned)((per_size + A3_THREADS - 1) / A3_THREADS), (unsigned)(batch * num_sizes));
  a3_iou_kernel<0><<<grid, A3_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  a3_iou_kernel<1><<<grid, A3_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  a3_argmax_kernel<<<small, A3_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  a3_assign_kernel<<<grid, A3_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  a3_total_kernel<<<1, 32, 0, st>>>(a.npos, batch, num_total_pos);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_anchor_focal_loss_forward(sstb200_ctx* c, const float* cls_score, int batch, int num_anchors, int num_classes,
                                                 int height, int width, const int64_t* labels, const float* label_weights,
                                                 const int64_t* num_total_pos, float loss_weight, float* loss) {
  FocalArgs a;
  int rc = focal_args(c, cls_score, batch, num_anchors, num_classes, height, width, labels, label_weights, num_total_pos, a);
  if (rc) return rc;
  CHECK_ARG(c, loss);
  const int nb = loss_grid(c, a.n);
  arena_reset(c);
  double* part;
  rc = arena_carve(c, [&](Carve& cv) { part = cv.take<double>(nb); });
  if (rc) return rc;
  focal_forward_kernel<<<nb, LOSS_THREADS, 0, c->stream>>>(a, part);
  LAUNCH_CHECK(c);
  a3_final_kernel<<<1, LOSS_THREADS, 0, c->stream>>>(part, nb, 1, loss_weight, 0.f, num_total_pos, loss, nullptr);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_anchor_focal_loss_backward(sstb200_ctx* c, const float* cls_score, int batch, int num_anchors, int num_classes,
                                                  int height, int width, const int64_t* labels, const float* label_weights,
                                                  const int64_t* num_total_pos, float loss_weight, const float* grad_loss,
                                                  float* grad_cls_score) {
  FocalArgs a;
  int rc = focal_args(c, cls_score, batch, num_anchors, num_classes, height, width, labels, label_weights, num_total_pos, a);
  if (rc) return rc;
  CHECK_ARG(c, grad_loss && grad_cls_score);
  focal_backward_kernel<<<loss_grid(c, a.n), LOSS_THREADS, 0, c->stream>>>(a, loss_weight, num_total_pos, grad_loss, grad_cls_score);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_anchor_reg_dir_loss_forward(sstb200_ctx* c, const float* bbox_pred, const float* dir_cls_preds, int batch,
                                                   int num_anchors, int num_classes, int height, int width, const int64_t* labels,
                                                   const float* bbox_targets, const float* bbox_weights, const int64_t* dir_targets,
                                                   const float* dir_weights, const float code_weight[7], const int64_t* num_total_pos,
                                                   float loss_weight_bbox, float loss_weight_dir, float* loss_bbox, float* loss_dir) {
  RegArgs a;
  int rc = reg_args(c, bbox_pred, dir_cls_preds, batch, num_anchors, num_classes, height, width, labels, bbox_targets, bbox_weights,
                    dir_targets, dir_weights, code_weight, num_total_pos, a);
  if (rc) return rc;
  CHECK_ARG(c, loss_bbox && loss_dir);
  const int nb = loss_grid(c, a.n);
  arena_reset(c);
  double* part;
  rc = arena_carve(c, [&](Carve& cv) { part = cv.take<double>(2 * nb); });
  if (rc) return rc;
  reg_forward_kernel<<<nb, LOSS_THREADS, 0, c->stream>>>(a, part, nb);
  LAUNCH_CHECK(c);
  a3_final_kernel<<<1, LOSS_THREADS, 0, c->stream>>>(part, nb, 2, loss_weight_bbox, loss_weight_dir, num_total_pos, loss_bbox, loss_dir);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_anchor_reg_dir_loss_backward(sstb200_ctx* c, const float* bbox_pred, const float* dir_cls_preds, int batch,
                                                    int num_anchors, int num_classes, int height, int width, const int64_t* labels,
                                                    const float* bbox_targets, const float* bbox_weights, const int64_t* dir_targets,
                                                    const float* dir_weights, const float code_weight[7], const int64_t* num_total_pos,
                                                    float loss_weight_bbox, float loss_weight_dir, const float* grad_losses,
                                                    float* grad_bbox_pred, float* grad_dir_cls_preds) {
  RegArgs a;
  int rc = reg_args(c, bbox_pred, dir_cls_preds, batch, num_anchors, num_classes, height, width, labels, bbox_targets, bbox_weights,
                    dir_targets, dir_weights, code_weight, num_total_pos, a);
  if (rc) return rc;
  CHECK_ARG(c, grad_losses && grad_bbox_pred && grad_dir_cls_preds);
  reg_backward_kernel<<<loss_grid(c, a.n), LOSS_THREADS, 0, c->stream>>>(a, loss_weight_bbox, loss_weight_dir, num_total_pos, grad_losses,
                                                                         grad_bbox_pred, grad_dir_cls_preds);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
