// The pieces every detection head's training kernels share (anchor3d.cu, centerpoint.cu, voteseg.cu, cluster_head.cu).  The heads'
// run-to-run determinism rests on two rules written once here: a loss is summed as per-block partials in double, then one block adds
// them in a fixed order (thread0_block_sum, sum_partials); and every head forms its sigmoid and softplus from one exp(-|x|) (sig).
#pragma once
#include <algorithm>
#include <climits>
#include "common.cuh"

namespace {

#define LOSS_THREADS 256  // block size of every loss launch; the targets kernels keep their own

// blocks of a grid-strided loss pass over n elements: enough for 8 elements per thread, at most 8 per SM
int loss_grid(sstb200_ctx* c, long long n) {
  const long long want = (n + LOSS_THREADS * 8 - 1) / (LOSS_THREADS * 8);
  return (int)std::max(1LL, std::min(want, (long long)c->num_sms * 8));
}

// Per-sample offsets of `batch` samples: off[0] = 0, non-decreasing, and at most `cap` GT boxes in a sample (INT_MAX: no cap).
int check_offsets(sstb200_ctx* c, const char* fn, const int32_t* off, int batch, int cap) {
  CHECK_ARG(c, off[0] == 0);
  for (int b = 0; b < batch; b++) {
    CHECK_ARG(c, off[b + 1] >= off[b]);
    if (off[b + 1] - off[b] > cap)
      return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "%s: sample %d has %d GT boxes, at most %d", fn, b, off[b + 1] - off[b], cap);
  }
  return SSTB_OK;
}

// Sum of v over the block, valid in thread 0 only: a warp shuffle tree, then thread 0 adds the warp sums in warp order.  Every thread
// calls it; sh holds blockDim.x / 32 values and is free again on return.  (box3d.cuh's block_sum returns its sum in every thread.)
template <typename T>
__device__ __forceinline__ T thread0_block_sum(T v, T* sh) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  T s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sh[w];
  __syncthreads();
  return s;
}

// fixed-order sum of output k's nb block partials part[k * nb + i]: thread j adds i = j, j + blockDim.x, ..., then thread0_block_sum
template <typename T>
__device__ __forceinline__ T sum_partials(const T* part, int nb, int k, T* sh) {
  T acc = 0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) acc += part[(size_t)k * nb + i];
  return thread0_block_sum(acc, sh);
}

// stable form: softplus(+-x) = max(+-x, 0) + log1p(exp(-|x|)), s = sigmoid(x), q = 1 - s = sigmoid(-x) from the same exp(-|x|)
struct Sig {
  float s, q, sp_pos, sp_neg;
};

__device__ __forceinline__ Sig sig(float x) {
  const float e = expf(-fabsf(x)), inv = 1.f / (1.f + e), l1p = log1pf(e);
  Sig r;
  r.s = x >= 0.f ? inv : e * inv;
  r.q = x >= 0.f ? e * inv : inv;
  r.sp_pos = fmaxf(x, 0.f) + l1p;
  r.sp_neg = fmaxf(-x, 0.f) + l1p;
  return r;
}

// mmdet 2.14 py_sigmoid_focal_loss element: t = 1: alpha q^gamma softplus(-x); t = 0: (1 - alpha) s^gamma softplus(x)
__device__ __forceinline__ float sigmoid_focal(float x, bool t, float alpha, float gamma) {
  const Sig g = sig(x);
  return t ? alpha * powf(g.q, gamma) * g.sp_neg : (1.f - alpha) * powf(g.s, gamma) * g.sp_pos;
}

// d/dx: t = 1: -alpha q^gamma (gamma s softplus(-x) + q); t = 0: (1 - alpha) s^gamma (gamma q softplus(x) + s)
__device__ __forceinline__ float sigmoid_focal_grad(float x, bool t, float alpha, float gamma) {
  const Sig g = sig(x);
  return t ? -alpha * powf(g.q, gamma) * (gamma * g.s * g.sp_neg + g.q) : (1.f - alpha) * powf(g.s, gamma) * (gamma * g.q * g.sp_pos + g.s);
}

// torch.abs' gradient: sign(d), 0 at 0 and at NaN
__device__ __forceinline__ float abs_grad(float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f); }

}  // namespace
