// CenterHead training path (mmdet3d/models/dense_heads/centerpoint_head.py:421-610): heatmap targets, the Gaussian focal loss on
// clip_sigmoid(logits) and the masked, code-weighted L1 of the regression heads, each with its backward.  fp32, stream-ordered, no sync.
//
// Targets, three launches for the whole batch and every task:
//   slots  one CTA per (sample, task) walks the task's classes in order and, within a class, the sample's boxes in input order (a
//          block-wide scan gives each box its slot), so a box's slot is the reference's position in its per-class torch.where
//          concatenation.  The CTA writes ind / mask / anno_box of its slots and one draw record (class, cx, cy, radius) per drawn box;
//   zero   every task's heatmap;
//   draw   one warp per record: the clipped (2r+1)^2 window, combined by an integer atomicMax on the fp32 bit pattern (all values are
//          >= 0, so integer order is float order and the result does not depend on the order of the writes).
// The box arithmetic is the reference's sequence of correctly rounded fp32 operations, written with __f*_rn so that no contraction into
// an FMA can move int(radius) or int(center) across an integer.
//
// Focal loss: forward = one pass of block partials (loss in double, positives as integers), then one block sums them in a fixed order;
// backward = one pass recomputing d loss / d logit from (logit, target).  L1: forward = one block; backward = zero the five head
// gradients, then one CTA per sample writes each occupied cell's sum over its objects in slot order (no float atomics).
#include <stdarg.h>
#include <algorithm>
#include "common.cuh"

namespace {

#define CP_MAX_TASKS 16
#define CP_MAX_BATCH 256
#define CP_THREADS 256

struct CpTask {
  float* heatmap;
  float* anno_box;
  int64_t* ind;
  uint8_t* mask;
  int label_lo, ncls;
};

struct CpArgs {
  CpTask task[CP_MAX_TASKS];
  int sample_off[CP_MAX_BATCH + 1];
  const float* boxes;
  const int64_t* labels;
  int4* records;  // [batch, num_tasks, max_objs]: (class, cx, cy, radius), radius -1 = nothing to draw
  int T, B, box_dim, W, H, max_objs, min_radius, norm_bbox;
  float pcx, pcy, vsx, vsy, osf;
  float k1m, k1p, km2o, kom1, k4a3;  // fp32 of the Python scalars 1 - o, 1 + o, -2 o, o - 1, 4 (4 o)
};

// mmdet3d/core/utils/gaussian.py:60-87 with det_size = (height, width) = (length, width), every operation a rounded fp32 one
__device__ __forceinline__ float gaussian_radius(const CpArgs& a, float h, float w) {
  const float hw = __fadd_rn(h, w);
  const float b1 = hw;
  const float c1 = __fdiv_rn(__fmul_rn(__fmul_rn(w, h), a.k1m), a.k1p);
  const float r1 = __fdiv_rn(__fadd_rn(b1, __fsqrt_rn(__fsub_rn(__fmul_rn(b1, b1), __fmul_rn(4.f, c1)))), 2.f);
  const float b2 = __fmul_rn(2.f, hw);
  const float c2 = __fmul_rn(__fmul_rn(a.k1m, w), h);
  const float r2 = __fdiv_rn(__fadd_rn(b2, __fsqrt_rn(__fsub_rn(__fmul_rn(b2, b2), __fmul_rn(16.f, c2)))), 2.f);
  const float b3 = __fmul_rn(a.km2o, hw);
  const float c3 = __fmul_rn(__fmul_rn(a.kom1, w), h);
  const float r3 = __fdiv_rn(__fadd_rn(b3, __fsqrt_rn(__fsub_rn(__fmul_rn(b3, b3), __fmul_rn(a.k4a3, c3)))), 2.f);
  float r = r1;  // Python's min(): the first of the smallest
  if (r2 < r) r = r2;
  if (r3 < r) r = r3;
  return r;
}

// one box into its slot (the slot's ind / mask / anno_box / record were zeroed by the caller)
__device__ void place_box(const CpArgs& a, const CpTask& t, int b, int task, int cls, long long i, int slot) {
  const float* bx = a.boxes + i * a.box_dim;
  const float w = __fdiv_rn(__fdiv_rn(bx[3], a.vsx), a.osf);
  const float l = __fdiv_rn(__fdiv_rn(bx[4], a.vsy), a.osf);
  if (!(w > 0.f && l > 0.f)) return;
  const float rad = gaussian_radius(a, l, w);
  const int radius = max(a.min_radius, (int)fminf(truncf(rad), 1073741824.f));
  const float cx = __fdiv_rn(__fdiv_rn(__fsub_rn(bx[0], a.pcx), a.vsx), a.osf);
  const float cy = __fdiv_rn(__fdiv_rn(__fsub_rn(bx[1], a.pcy), a.vsy), a.osf);
  const float tx = truncf(cx), ty = truncf(cy);  // center.to(torch.int32): toward zero
  if (!(tx >= 0.f && tx < (float)a.W && ty >= 0.f && ty < (float)a.H)) return;
  const int xi = (int)tx, yi = (int)ty;
  const size_t s = (size_t)b * a.max_objs + slot;
  t.ind[s] = (int64_t)yi * a.W + xi;
  t.mask[s] = 1;
  float* ab = t.anno_box + s * 10;
  ab[0] = __fsub_rn(cx, (float)xi);
  ab[1] = __fsub_rn(cy, (float)yi);
  ab[2] = bx[2];
#pragma unroll
  for (int k = 0; k < 3; k++) ab[3 + k] = a.norm_bbox ? logf(bx[3 + k]) : bx[3 + k];
  sincosf(bx[6], ab + 6, ab + 7);
  ab[8] = a.box_dim >= 9 ? bx[7] : 0.f;
  ab[9] = a.box_dim >= 9 ? bx[8] : 0.f;
  a.records[((size_t)b * a.T + task) * a.max_objs + slot] = make_int4(cls, xi, yi, radius);
}

__global__ void __launch_bounds__(CP_THREADS) cp_slots_kernel(const __grid_constant__ CpArgs a) {
  __shared__ int warp_tot[CP_THREADS / 32];
  const int b = blockIdx.x / a.T, task = blockIdx.x - b * a.T;
  const CpTask& t = a.task[task];
  const int M = a.max_objs;
  int4* rec = a.records + ((size_t)b * a.T + task) * M;
  for (int s = threadIdx.x; s < M; s += blockDim.x) {
    const size_t o = (size_t)b * M + s;
    t.ind[o] = 0;
    t.mask[o] = 0;
    rec[s] = make_int4(0, 0, 0, -1);
#pragma unroll
    for (int k = 0; k < 10; k++) t.anno_box[o * 10 + k] = 0.f;
  }
  __syncthreads();
  const int begin = a.sample_off[b], end = a.sample_off[b + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int base = 0;
  for (int c = 0; c < t.ncls && base < M; c++) {
    const int64_t want = (int64_t)t.label_lo + c;
    for (int start = begin; start < end && base < M; start += blockDim.x) {
      const int i = start + threadIdx.x;
      const bool hit = i < end && a.labels[i] == want;
      const unsigned ballot = __ballot_sync(0xffffffffu, hit);
      if (lane == 0) warp_tot[warp] = __popc(ballot);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); w++) {
        before += w < warp ? warp_tot[w] : 0;
        total += warp_tot[w];
      }
      const int slot = base + before + __popc(ballot & ((1u << lane) - 1u));
      if (hit && slot < M) place_box(a, t, b, task, c, i, slot);
      base += total;
      __syncthreads();
    }
  }
}

__global__ void cp_zero_heatmaps_kernel(const __grid_constant__ CpArgs a) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (int task = 0; task < a.T; task++) {
    const size_t n = (size_t)a.B * a.task[task].ncls * a.H * a.W;
    float* p = a.task[task].heatmap;
    if ((n & 3) == 0 && ((uintptr_t)p & 15) == 0) {
      float4* q = (float4*)p;
      for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n / 4; i += stride) q[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = 0.f;
    }
  }
}

// mmdet3d/core/utils/gaussian.py:5-57: value exp(-(dx^2 + dy^2) / (2 sigma^2)) in double with sigma = (2r + 1) / 6, rounded to fp32,
// over the window clipped as draw_heatmap_gaussian clips it
__global__ void __launch_bounds__(CP_THREADS) cp_draw_kernel(const __grid_constant__ CpArgs a, int num_records) {
  const int rid = blockIdx.x * (CP_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (rid >= num_records) return;
  const int4 r = a.records[rid];
  if (r.w < 0) return;
  const int task = (rid / a.max_objs) % a.T, b = rid / (a.max_objs * a.T);
  const int x = r.y, y = r.z, radius = r.w;
  const int left = min(x, radius), right = min(a.W - x, radius + 1);
  const int top = min(y, radius), bottom = min(a.H - y, radius + 1);
  const int ww = left + right, hh = top + bottom;
  const double sigma = (2.0 * radius + 1.0) / 6.0;  // in double: radius reaches 2^30, where 2 radius + 1 overflows an int
  const double den = 2.0 * sigma * sigma;
  int* hm = (int*)(a.task[task].heatmap + ((size_t)b * a.task[task].ncls + r.x) * a.H * a.W);
  for (int k = lane; k < ww * hh; k += 32) {
    const int dy = k / ww - top, dx = k % ww - left;
    const float v = (float)exp(-(double)(dx * dx + dy * dy) / den);
    atomicMax(hm + (size_t)(y + dy) * a.W + (x + dx), __float_as_int(v));
  }
}

// ---- Gaussian focal loss (mmdet 2.14 gaussian_focal_loss, alpha 2, gamma 4) on clip_sigmoid(x) (eps 1e-4) ----
#define FL_EPS 1e-12f
#define FL_CLIP_LO 1e-4f
#define FL_CLIP_HI 0.9999f

__device__ __forceinline__ float fl_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// torch.clamp: a NaN sigmoid stays NaN (fminf / fmaxf would turn it into a bound and hide a NaN logit)
__device__ __forceinline__ float fl_clip(float s) { return s < FL_CLIP_LO ? FL_CLIP_LO : (s > FL_CLIP_HI ? FL_CLIP_HI : s); }

__device__ __forceinline__ float fl_loss(float x, float t) {
  const float p = fl_clip(fl_sigmoid(x));
  const float q = 1.f - p, u = 1.f - t;
  const float pos = t == 1.f ? -logf(p + FL_EPS) * q * q : 0.f;
  const float neg = -logf(q + FL_EPS) * p * p * (u * u) * (u * u);
  return pos + neg;
}

// d loss / d x: d/dp of the element's loss times the clamp's pass-through (inclusive at the bounds, as torch.clamp) times s (1 - s);
// a NaN sigmoid passes the clamp, so a NaN logit gets a NaN gradient
__device__ __forceinline__ float fl_grad(float x, float t) {
  const float s = fl_sigmoid(x);
  if (s < FL_CLIP_LO || s > FL_CLIP_HI) return 0.f;
  const float p = s, q = 1.f - p, u = 1.f - t;
  float d = (p * p / (q + FL_EPS) - 2.f * p * logf(q + FL_EPS)) * ((u * u) * (u * u));
  if (t == 1.f) d += -q * q / (p + FL_EPS) + 2.f * q * logf(p + FL_EPS);
  return d * ((1.f - s) * s);
}

__device__ __forceinline__ double block_sum_double(double v, double* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sh[w];
  __syncthreads();
  return s;  // valid in thread 0
}

__device__ __forceinline__ long long block_sum_ll(long long v, long long* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  long long s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sh[w];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(CP_THREADS) fl_forward_kernel(const float* __restrict__ x, const float* __restrict__ t, long long n,
                                                                double* part_loss, long long* part_pos) {
  __shared__ double shd[CP_THREADS / 32];
  __shared__ long long shl[CP_THREADS / 32];
  double acc = 0.0;
  long long pos = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float xv = __ldg(x + i), tv = __ldg(t + i);
    acc += (double)fl_loss(xv, tv);
    pos += tv == 1.f;
  }
  acc = block_sum_double(acc, shd);
  pos = block_sum_ll(pos, shl);
  if (threadIdx.x == 0) part_loss[blockIdx.x] = acc, part_pos[blockIdx.x] = pos;
}

__global__ void __launch_bounds__(CP_THREADS) fl_final_kernel(const double* part_loss, const long long* part_pos, int nparts,
                                                              float loss_weight, float* loss, float* num_pos) {
  __shared__ double shd[CP_THREADS / 32];
  __shared__ long long shl[CP_THREADS / 32];
  double acc = 0.0;
  long long pos = 0;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) acc += part_loss[i], pos += part_pos[i];
  acc = block_sum_double(acc, shd);
  pos = block_sum_ll(pos, shl);
  if (threadIdx.x == 0) {
    const float np = (float)pos;
    *num_pos = np;
    *loss = (float)((double)loss_weight * (acc / (double)fmaxf(np, 1.f)));
  }
}

__global__ void fl_backward_kernel(const float* __restrict__ x, const float* __restrict__ t, long long n, float loss_weight,
                                   const float* __restrict__ num_pos, const float* __restrict__ grad_loss, float* __restrict__ grad_x) {
  const float scale = grad_loss[0] * loss_weight / fmaxf(num_pos[0], 1.f);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    grad_x[i] = scale * fl_grad(__ldg(x + i), __ldg(t + i));
}

// ---- regression L1: anno_box [B, M, 10] against (reg 2, height 1, dim 3, rot 2, vel 2) gathered at ind ----
struct L1Args {
  const float* head[5];
  float* grad[5];
  const float* anno_box;
  const int64_t* ind;
  const uint8_t* mask;
  float cw[10];
  int B, M;
  long long HW;
  float loss_weight;
};

__device__ __constant__ int kL1Head[10] = {0, 0, 1, 2, 2, 2, 3, 3, 4, 4};
__device__ __constant__ int kL1Chan[10] = {0, 1, 0, 0, 1, 2, 0, 1, 0, 1};
__device__ __constant__ int kL1Nch[5] = {2, 1, 3, 2, 2};

// sum(mask) + 1e-4 in fp32, as the reference's masks.float().sum() + 1e-4 (exact: a count below 2^24)
__device__ float l1_avg_factor(const L1Args& a, long long* shl) {
  long long cnt = 0;
  for (long long i = threadIdx.x; i < (long long)a.B * a.M; i += blockDim.x) cnt += a.mask[i] != 0;
  cnt = block_sum_ll(cnt, shl);
  __shared__ float avg;
  if (threadIdx.x == 0) avg = __fadd_rn((float)cnt, 1e-4f);
  __syncthreads();
  return avg;
}

__device__ __forceinline__ float l1_pred(const L1Args& a, int b, long long cell, int c) {
  if (cell < 0 || cell >= a.HW) return __int_as_float(0x7fffffff);  // an index off the map makes the loss NaN
  const int h = kL1Head[c];
  return a.head[h][((long long)b * kL1Nch[h] + kL1Chan[c]) * a.HW + cell];
}

__device__ __forceinline__ float l1_weight(const L1Args& a, float target, int c) {
  return (target == target ? 1.f : 0.f) * a.cw[c];
}

__global__ void __launch_bounds__(CP_THREADS) l1_forward_kernel(const __grid_constant__ L1Args a, float* loss) {
  __shared__ double shd[CP_THREADS / 32];
  __shared__ long long shl[CP_THREADS / 32];
  const float avg = l1_avg_factor(a, shl);
  double acc = 0.0;
  for (long long e = threadIdx.x; e < (long long)a.B * a.M * 10; e += blockDim.x) {
    const long long bm = e / 10;
    const int c = (int)(e - bm * 10), b = (int)(bm / a.M);
    // a masked-out slot adds |pred - target| * 0, as the reference's gather at every slot does: a NaN or an off-map ind there makes
    // the loss NaN
    const float tv = a.anno_box[e];
    acc += (double)(fabsf(l1_pred(a, b, a.ind[bm], c) - tv) * (a.mask[bm] ? l1_weight(a, tv, c) : 0.f));
  }
  acc = block_sum_double(acc, shd);
  if (threadIdx.x == 0) *loss = (float)((double)a.loss_weight * (acc / (double)avg));
}

__global__ void l1_zero_grads_kernel(const __grid_constant__ L1Args a) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (int h = 0; h < 5; h++) {
    const long long n = (long long)a.B * kL1Nch[h] * a.HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) a.grad[h][i] = 0.f;
  }
}

// one CTA per sample; the first masked slot of each occupied cell writes the cell's gradient, summed over the cell's masked slots in
// slot order
__global__ void __launch_bounds__(CP_THREADS) l1_backward_kernel(const __grid_constant__ L1Args a, const float* __restrict__ grad_loss) {
  extern __shared__ long long cell[];  // [M], -1 for an unmasked slot
  __shared__ long long shl[CP_THREADS / 32];
  const float avg = l1_avg_factor(a, shl);
  const float g = __fdiv_rn(__fmul_rn(grad_loss[0], a.loss_weight), avg);
  const int b = blockIdx.x, M = a.M;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const size_t s = (size_t)b * M + m;
    cell[m] = a.mask[s] ? a.ind[s] : -1;
  }
  __syncthreads();
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    const long long here = cell[m];
    if (here < 0 || here >= a.HW) continue;
    bool first = true;
    for (int k = 0; k < m && first; k++) first = cell[k] != here;
    if (!first) continue;
    for (int c = 0; c < 10; c++) {
      const float p = l1_pred(a, b, here, c);
      float acc = 0.f;
      for (int k = m; k < M; k++) {
        if (cell[k] != here) continue;
        const float tv = a.anno_box[((size_t)b * M + k) * 10 + c];
        const float d = p - tv;
        const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
        acc += g * l1_weight(a, tv, c) * sgn;
      }
      const int h = kL1Head[c];
      a.grad[h][((long long)b * kL1Nch[h] + kL1Chan[c]) * a.HW + here] = acc;
    }
  }
}

int l1_args(sstb200_ctx* c, const float* const heads[5], int batch, int height, int width, const float* anno_box, const int64_t* ind,
            const uint8_t* mask, int max_objs, const float code_weights[10], float loss_weight, L1Args& a) {
  CHECK_ARG(c, heads && anno_box && ind && mask && code_weights);
  CHECK_ARG(c, batch >= 1 && height >= 1 && width >= 1 && max_objs >= 1);
  if (max_objs > 4096) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "centerpoint_l1: max_objs %d above 4096", max_objs);
  for (int h = 0; h < 5; h++) CHECK_ARG(c, heads[h] != nullptr);
  for (int h = 0; h < 5; h++) a.head[h] = heads[h], a.grad[h] = nullptr;
  for (int k = 0; k < 10; k++) a.cw[k] = code_weights[k];
  a.anno_box = anno_box, a.ind = ind, a.mask = mask;
  a.B = batch, a.M = max_objs, a.HW = (long long)height * width, a.loss_weight = loss_weight;
  return SSTB_OK;
}

int fl_grid(sstb200_ctx* c, long long n) {
  const long long want = (n + CP_THREADS * 8 - 1) / (CP_THREADS * 8);
  return (int)std::max(1LL, std::min(want, (long long)c->num_sms * 8));
}

}  // namespace

extern "C" int sstb200_centerpoint_targets(sstb200_ctx* c, const float* boxes, const int64_t* labels, int box_dim,
                                           const int32_t* sample_offsets, int batch, const int32_t* task_label_offsets, int num_tasks,
                                           const float pc_min[2], const float voxel_size[2], int out_size_factor, int width, int height,
                                           double gaussian_overlap, int min_radius, int max_objs, int norm_bbox, float* const* heatmaps,
                                           float* const* anno_boxes, int64_t* const* inds, uint8_t* const* masks) {
  CHECK_ARG(c, sample_offsets && task_label_offsets && pc_min && voxel_size && heatmaps && anno_boxes && inds && masks);
  CHECK_ARG(c, box_dim == 7 || box_dim == 9);
  CHECK_ARG(c, batch >= 1 && num_tasks >= 1 && out_size_factor >= 1 && width >= 1 && height >= 1 && max_objs >= 1);
  CHECK_ARG(c, voxel_size[0] > 0.f && voxel_size[1] > 0.f);
  if (batch > CP_MAX_BATCH || num_tasks > CP_MAX_TASKS)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "centerpoint_targets: %d samples / %d tasks, at most %d / %d", batch, num_tasks,
                     CP_MAX_BATCH, CP_MAX_TASKS);
  CHECK_ARG(c, sample_offsets[0] == 0);
  for (int b = 0; b < batch; b++) CHECK_ARG(c, sample_offsets[b + 1] >= sample_offsets[b]);
  CHECK_ARG(c, sample_offsets[batch] == 0 || (boxes && labels));
  for (int t = 0; t < num_tasks; t++) CHECK_ARG(c, task_label_offsets[t + 1] > task_label_offsets[t]);
  if ((long long)height * width >= (1LL << 31) || (long long)batch * num_tasks * max_objs >= (1LL << 31))
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "centerpoint_targets: map or slot count reaches 2^31");
  CpArgs a;
  for (int t = 0; t < num_tasks; t++) {
    CHECK_ARG(c, heatmaps[t] && anno_boxes[t] && inds[t] && masks[t]);
    a.task[t] = CpTask{heatmaps[t], anno_boxes[t], inds[t], masks[t], task_label_offsets[t],
                       task_label_offsets[t + 1] - task_label_offsets[t]};
  }
  for (int b = 0; b <= batch; b++) a.sample_off[b] = sample_offsets[b];
  a.boxes = boxes, a.labels = labels;
  a.T = num_tasks, a.B = batch, a.box_dim = box_dim, a.W = width, a.H = height, a.max_objs = max_objs, a.min_radius = min_radius;
  a.norm_bbox = norm_bbox != 0;
  a.pcx = pc_min[0], a.pcy = pc_min[1], a.vsx = voxel_size[0], a.vsy = voxel_size[1], a.osf = (float)out_size_factor;
  const double o = gaussian_overlap;
  a.k1m = (float)(1.0 - o), a.k1p = (float)(1.0 + o), a.km2o = (float)(-2.0 * o), a.kom1 = (float)(o - 1.0), a.k4a3 = (float)(4.0 * (4.0 * o));
  const int nrec = batch * num_tasks * max_objs;
  arena_reset(c);
  int rc = arena_reserve(c, al256((size_t)nrec * sizeof(int4)));
  if (rc) return rc;
  a.records = arena_alloc<int4>(c, nrec);
  if (!a.records) return sstb_fail(c, SSTB_ERR_WORKSPACE, "centerpoint_targets: arena too small");
  cudaStream_t st = c->stream;
  cp_slots_kernel<<<batch * num_tasks, CP_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  cp_zero_heatmaps_kernel<<<c->num_sms * 4, CP_THREADS, 0, st>>>(a);
  LAUNCH_CHECK(c);
  cp_draw_kernel<<<(nrec + CP_THREADS / 32 - 1) / (CP_THREADS / 32), CP_THREADS, 0, st>>>(a, nrec);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_gaussian_focal_loss_forward(sstb200_ctx* c, const float* logits, const float* target, int64_t n, float loss_weight,
                                                   float* loss, float* num_pos) {
  CHECK_ARG(c, n >= 1 && logits && target && loss && num_pos);
  const int nb = fl_grid(c, n);
  arena_reset(c);
  int rc = arena_reserve(c, al256(nb * sizeof(double)) + al256(nb * sizeof(long long)));
  if (rc) return rc;
  double* pl = arena_alloc<double>(c, nb);
  long long* pp = arena_alloc<long long>(c, nb);
  if (!pl || !pp) return sstb_fail(c, SSTB_ERR_WORKSPACE, "gaussian_focal_loss: arena too small");
  fl_forward_kernel<<<nb, CP_THREADS, 0, c->stream>>>(logits, target, n, pl, pp);
  LAUNCH_CHECK(c);
  fl_final_kernel<<<1, CP_THREADS, 0, c->stream>>>(pl, pp, nb, loss_weight, loss, num_pos);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_gaussian_focal_loss_backward(sstb200_ctx* c, const float* logits, const float* target, int64_t n, float loss_weight,
                                                    const float* num_pos, const float* grad_loss, float* grad_logits) {
  CHECK_ARG(c, n >= 1 && logits && target && num_pos && grad_loss && grad_logits);
  fl_backward_kernel<<<fl_grid(c, n), CP_THREADS, 0, c->stream>>>(logits, target, n, loss_weight, num_pos, grad_loss, grad_logits);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_centerpoint_l1_loss_forward(sstb200_ctx* c, const float* const heads[5], int batch, int height, int width,
                                                   const float* anno_box, const int64_t* ind, const uint8_t* mask, int max_objs,
                                                   const float code_weights[10], float loss_weight, float* loss) {
  L1Args a;
  int rc = l1_args(c, heads, batch, height, width, anno_box, ind, mask, max_objs, code_weights, loss_weight, a);
  if (rc) return rc;
  CHECK_ARG(c, loss);
  l1_forward_kernel<<<1, CP_THREADS, 0, c->stream>>>(a, loss);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_centerpoint_l1_loss_backward(sstb200_ctx* c, const float* const heads[5], int batch, int height, int width,
                                                    const float* anno_box, const int64_t* ind, const uint8_t* mask, int max_objs,
                                                    const float code_weights[10], float loss_weight, const float* grad_loss,
                                                    float* const grad_heads[5]) {
  L1Args a;
  int rc = l1_args(c, heads, batch, height, width, anno_box, ind, mask, max_objs, code_weights, loss_weight, a);
  if (rc) return rc;
  CHECK_ARG(c, grad_loss && grad_heads);
  for (int h = 0; h < 5; h++) {
    CHECK_ARG(c, grad_heads[h] != nullptr);
    a.grad[h] = grad_heads[h];
  }
  l1_zero_grads_kernel<<<c->num_sms * 4, CP_THREADS, 0, c->stream>>>(a);
  LAUNCH_CHECK(c);
  l1_backward_kernel<<<batch, CP_THREADS, (size_t)max_objs * sizeof(long long), c->stream>>>(a, grad_loss);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
