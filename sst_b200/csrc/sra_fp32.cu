// Sparse Regional Attention encoder layer - fp32 SIMT path ("exact" mode, also the bring-up path).
// Replaces, per layer, flat2window -> nn.MultiheadAttention per drop level -> window2flat -> residual/LN/FFN
// (mmdet3d/models/sst/sst_basic_block_v2.py:41-126) with ragged kernels that work on the window CSR:
// no padding to max_tokens, no per-level batches, no masks.
#include <stdarg.h>
#include "common.cuh"
#include "sra.cuh"
#include "sra_attn.cuh"

// ------------------------------------------------------------------------------------------------
// generic row GEMM  out[r, n] = epi( sum_k A'[r,k] * W[n,k] + bias[n] )   (nn.Linear layout, fp32 FFMA)
//   A'[r,k] = A[r,k] (+ pos(r,k) if pos table given and n-tile < pos_ncols)
// ------------------------------------------------------------------------------------------------
#define GBM 128
#define GBN 64
#define GBK 16

struct PosTab {
  const float* tab;        // [3][maxw][L]
  const int32_t* code;     // [rows] x | y<<8 | z<<16
  int L, maxw, ndim;
};

__device__ __forceinline__ float pos_value(const PosTab& p, int code, int k) {
  int axis = k / p.L;
  if (axis >= p.ndim) return 0.f;
  int v = (code >> (8 * axis)) & 255;
  return p.tab[((size_t)axis * p.maxw + v) * p.L + (k - axis * p.L)];
}

template <int ACT /*0 none,1 relu,2 gelu*/>
__global__ void __launch_bounds__(256) gemm_rows_kernel(const float* __restrict__ A, int lda, const float* __restrict__ W,
                                                        const float* __restrict__ bias, const float* __restrict__ res, int ldr,
                                                        float* __restrict__ out, int ldo, int M, const int32_t* __restrict__ M_dev,
                                                        int N, int K, PosTab pos, int pos_ncols, int ldw,
                                                        const long long* __restrict__ res_index) {
  pdl_wait();
  pdl_launch();
  __shared__ float As[GBK][GBM + 4];
  __shared__ float Bs[GBK][GBN + 4];
  if (M_dev) M = *M_dev;
  int row0 = blockIdx.x * GBM, col0 = blockIdx.y * GBN;
  if (row0 >= M) return;
  int tid = threadIdx.x;
  int tr = tid / 16, tc = tid % 16;  // thread tile: rows tr*8..+8, cols tc*4..+4
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
  bool use_pos = pos.tab != nullptr && col0 < pos_ncols;
  for (int k0 = 0; k0 < K; k0 += GBK) {
    // A tile: 128 x 16 = 2048 elements, 8 per thread
#pragma unroll
    for (int i = 0; i < 8; i++) {
      int e = tid + i * 256;
      int r = e / GBK, k = e % GBK;
      int gr = row0 + r, gk = k0 + k;
      float v = 0.f;
      if (gr < M && gk < K) {
        v = A[(size_t)gr * lda + gk];
        if (use_pos) v += pos_value(pos, pos.code[gr], gk);
      }
      As[k][r] = v;
    }
    // W tile: 64 x 16 = 1024 elements, 4 per thread
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int e = tid + i * 256;
      int n = e / GBK, k = e % GBK;
      int gn = col0 + n, gk = k0 + k;
      Bs[k][n] = (gn < N && gk < K) ? W[(size_t)gn * ldw + gk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < GBK; k++) {
      float a[8], b[4];
      *(float4*)&a[0] = *(const float4*)&As[k][tr * 8];
      *(float4*)&a[4] = *(const float4*)&As[k][tr * 8 + 4];
      *(float4*)&b[0] = *(const float4*)&Bs[k][tc * 4];
#pragma unroll
      for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; i++) {
    int gr = row0 + tr * 8 + i;
    if (gr >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int gn = col0 + tc * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j] + (bias ? bias[gn] : 0.f);
      if (ACT == 1) v = fmaxf(v, 0.f);
      if (ACT == 2) v = gelu_erf(v);
      if (res) v += res[(size_t)(res_index ? res_index[gr] : (long long)gr) * ldr + gn];
      out[(size_t)gr * ldo + gn] = v;
    }
  }
}

void sstb_gemm_rows_ex(cudaStream_t st, const float* A, int lda, const float* W, int ldw, const float* bias, const float* res,
                       int ldr, const long long* res_index, float* out, int ldo, int M_cap, const int32_t* M_dev, int N, int K,
                       int act, const float* pos_tab, const int32_t* pos_code, int posL, int pos_maxw, int pos_ndim, int pos_ncols) {
  if (M_cap <= 0) return;
  dim3 grid((M_cap + GBM - 1) / GBM, (N + GBN - 1) / GBN);
  PosTab p{pos_tab, pos_code, posL, pos_maxw, pos_ndim};
  if (act == 0)
    launch_pdl(gemm_rows_kernel<0>, dim3(grid), dim3(256), (size_t)(0), st, A, lda, W, bias, res, ldr, out, ldo, M_cap, M_dev, N, K, p, pos_ncols, ldw, res_index);
  else if (act == 1)
    launch_pdl(gemm_rows_kernel<1>, dim3(grid), dim3(256), (size_t)(0), st, A, lda, W, bias, res, ldr, out, ldo, M_cap, M_dev, N, K, p, pos_ncols, ldw, res_index);
  else
    launch_pdl(gemm_rows_kernel<2>, dim3(grid), dim3(256), (size_t)(0), st, A, lda, W, bias, res, ldr, out, ldo, M_cap, M_dev, N, K, p, pos_ncols, ldw, res_index);
}
void sstb_gemm_rows(cudaStream_t st, const float* A, int lda, const float* W, const float* bias, const float* res, int ldr,
                    float* out, int ldo, int M_cap, const int32_t* M_dev, int N, int K, int act, const float* pos_tab,
                    const int32_t* pos_code, int posL, int pos_maxw, int pos_ndim, int pos_ncols) {
  sstb_gemm_rows_ex(st, A, lda, W, K, bias, res, ldr, nullptr, out, ldo, M_cap, M_dev, N, K, act, pos_tab, pos_code, posL, pos_maxw,
                    pos_ndim, pos_ncols);
}

int sstb_win_attn_fp32(sstb200_ctx* c, const float* qkv, int d, int nhead, int n_cap, const int32_t* n_dev,
                       const int32_t* win_offsets, const int32_t* tok_perm, const int32_t* tok_win, const float* tau,
                       int tau_n, float tau_min, float* out) {
  return sstb_win_attn<float, float>(c, qkv, d, nhead, n_cap, n_dev, win_offsets, tok_perm, tok_win, tau, tau_n, tau_min, out);
}

// ------------------------------------------------------------------------------------------------
// out = LayerNorm(a [+ b]) * gamma + beta   (row-wise, one warp per row), or eval BatchNorm affine.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) add_norm_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta,
                                                       const float* __restrict__ bn_mean, const float* __restrict__ bn_var,
                                                       float eps, float* __restrict__ out, int n, const int32_t* __restrict__ n_dev, int d,
                                                       int act) {
  pdl_wait();
  pdl_launch();
  if (n_dev) n = *n_dev;
  int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= n) return;
  int ln = lane_id();
  const float* ap = a + (size_t)row * d;
  const float* bp = b ? b + (size_t)row * d : nullptr;
  float v[8];  // d <= 256
  float s = 0.f;
  int cnt = 0;
  for (int c = ln; c < d; c += 32, cnt++) {
    float t = ap[c] + (bp ? bp[c] : 0.f);
    v[cnt] = t;
    s += t;
  }
  if (bn_mean) {  // eval-mode BatchNorm1d (use_bn layers): per-channel affine
    cnt = 0;
    for (int c = ln; c < d; c += 32, cnt++) {
      float o = (v[cnt] - bn_mean[c]) * rsqrtf(bn_var[c] + eps) * gamma[c] + beta[c];
      if (act == 1) o = fmaxf(o, 0.f);
      if (act == 2) o = gelu_erf(o);
      out[(size_t)row * d + c] = o;
    }
    return;
  }
  float mean = warp_sum(s) / (float)d;
  float q = 0.f;
  cnt = 0;
  for (int c = ln; c < d; c += 32, cnt++) {
    float t = v[cnt] - mean;
    q += t * t;
  }
  float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
  cnt = 0;
  for (int c = ln; c < d; c += 32, cnt++) {
    float o = (v[cnt] - mean) * rstd * gamma[c] + beta[c];
    if (act == 1) o = fmaxf(o, 0.f);
    if (act == 2) o = gelu_erf(o);
    out[(size_t)row * d + c] = o;
  }
}

void sstb_add_norm_act(cudaStream_t st, const float* a, const float* b, const float* gamma, const float* beta,
                       const float* bn_mean, const float* bn_var, float eps, float* out, int n_cap, const int32_t* n_dev, int d, int act) {
  if (n_cap <= 0) return;
  unsigned grid = (unsigned)(((size_t)n_cap * 32 + 255) / 256);
  launch_pdl(add_norm_kernel, dim3(grid), dim3(256), (size_t)(0), st, a, b, gamma, beta, bn_mean, bn_var, eps, out, n_cap, n_dev, d, act);
}
void sstb_add_norm(cudaStream_t st, const float* a, const float* b, const float* gamma, const float* beta,
                   const float* bn_mean, const float* bn_var, float eps, float* out, int n_cap, const int32_t* n_dev, int d) {
  sstb_add_norm_act(st, a, b, gamma, beta, bn_mean, bn_var, eps, out, n_cap, n_dev, d, 0);
}

// ------------------------------------------------------------------------------------------------
// fp32-tolerance GEMMs on the tensor core: every Linear of the layer runs through sstb_gemm_rows_x3 (split-fp16 operands:
// hi.hi + lo.hi + hi.lo in one set of fp32 accumulators, ~2^-22 relative at any operand scale, see sra.cuh) instead of the FFMA
// kernel above; the positional term of
// q|k is added to a copy of the input first.  Shapes sstb_gemm_rows_x3 does not take (d_model or dim_ff not a multiple of 64) run
// on the FFMA kernel.
// ------------------------------------------------------------------------------------------------
__global__ void add_pos_kernel(const float* __restrict__ x, int d, PosTab pos, float* __restrict__ out, int n, const int32_t* __restrict__ n_dev) {
  pdl_wait();
  pdl_launch();
  if (n_dev) n = *n_dev;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * d) return;
  const int r = (int)(i / d), k = (int)(i % d);
  out[i] = x[i] + pos_value(pos, pos.code[r], k);
}

static int linear_fp32(sstb200_ctx* c, const float* A, int lda, const float* W, const float* bias, const float* res, int ldr, float* out,
                       int ldo, int n_cap, const int32_t* n_dev, int N, int K, int act) {
  const int rc = sstb_gemm_rows_x3(c, A, lda, W, bias, res, ldr, out, ldo, n_cap, n_dev, N, K, act);
  if (rc != SSTB_ERR_UNSUPPORTED) return rc;
  sstb_gemm_rows_ex(c->stream, A, lda, W, K, bias, res, ldr, nullptr, out, ldo, n_cap, n_dev, N, K, act, nullptr, nullptr, 0, 0, 0, 0);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// one encoder layer, fp32
// ------------------------------------------------------------------------------------------------
int sstb_sra_layer_fp32(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x, float* y,
                        int n_cap, const int32_t* n_dev) {
  int d = L->d_model, ff = L->dim_ff;
  if (d > 256 || d % 32) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "d_model %d (need multiple of 32, <= 256)", d);
  float* qkv = arena_alloc<float>(c, (size_t)n_cap * 3 * d);
  float* att = arena_alloc<float>(c, (size_t)n_cap * d);
  float* t1 = arena_alloc<float>(c, (size_t)n_cap * d);
  float* x1 = arena_alloc<float>(c, (size_t)n_cap * d);
  float* hid = arena_alloc<float>(c, (size_t)n_cap * ff);
  if (!qkv || !att || !t1 || !x1 || !hid) return sstb_fail(c, SSTB_ERR_WORKSPACE, "sra layer: arena too small");
  cudaStream_t st = c->stream;
  const float* xin = x;
  if (!L->post_norm) {  // pre-norm: src2 = norm1(src)
    sstb_add_norm(st, x, nullptr, L->norm1_w, L->norm1_b, L->norm1_mean, L->norm1_var, L->norm_eps, x1, n_cap, n_dev, d);
    xin = x1;
  }
  // q,k from (x + pos); v from x
  int rc = SSTB_OK;
  if (d % 64 == 0 && ff % 64 == 0) {
    const float* xqk = xin;
    if (P->pos_table) {
      float* xpos = arena_alloc<float>(c, (size_t)n_cap * d);
      if (!xpos) return sstb_fail(c, SSTB_ERR_WORKSPACE, "sra layer: arena too small");
      PosTab pt{P->pos_table, P->pos_code, P->pos_L, P->pos_maxw, P->pos_ndim};
      const size_t tot = (size_t)n_cap * d;
      launch_pdl(add_pos_kernel, dim3((unsigned)((tot + 255) / 256)), dim3(256), (size_t)0, st, xin, d, pt, xpos, n_cap, n_dev);
      xqk = xpos;
    }
    rc = linear_fp32(c, xqk, d, L->in_proj_w, L->in_proj_b, nullptr, 0, qkv, 3 * d, n_cap, n_dev, 2 * d, d, 0);
    if (rc) return rc;
    rc = linear_fp32(c, xin, d, L->in_proj_w + (size_t)2 * d * d, L->in_proj_b + 2 * d, nullptr, 0, qkv + 2 * d, 3 * d, n_cap, n_dev, d, d, 0);
    if (rc) return rc;
  } else {
    sstb_gemm_rows(st, xin, d, L->in_proj_w, L->in_proj_b, nullptr, 0, qkv, 3 * d, n_cap, n_dev, 3 * d, d, 0, P->pos_table,
                   P->pos_code, P->pos_L, P->pos_maxw, P->pos_ndim, 2 * d);
  }
  rc = sstb_win_attn_fp32(c, qkv, d, L->nhead, n_cap, n_dev, P->win_offsets, P->tok_perm, P->tok_win, L->tau, L->tau_n,
                              L->tau_min, att);
  if (rc) return rc;
  if (L->post_norm) {
    if ((rc = linear_fp32(c, att, d, L->out_proj_w, L->out_proj_b, nullptr, 0, t1, d, n_cap, n_dev, d, d, 0))) return rc;
    sstb_add_norm(st, x, t1, L->norm1_w, L->norm1_b, L->norm1_mean, L->norm1_var, L->norm_eps, x1, n_cap, n_dev, d);
    if ((rc = linear_fp32(c, x1, d, L->lin1_w, L->lin1_b, nullptr, 0, hid, ff, n_cap, n_dev, ff, d, L->act))) return rc;
    if ((rc = linear_fp32(c, hid, ff, L->lin2_w, L->lin2_b, nullptr, 0, t1, d, n_cap, n_dev, d, ff, 0))) return rc;
    sstb_add_norm(st, x1, t1, L->norm2_w, L->norm2_b, L->norm2_mean, L->norm2_var, L->norm_eps, y, n_cap, n_dev, d);
  } else {
    // src = src + attn ; src = src + ffn(norm2(src))
    if ((rc = linear_fp32(c, att, d, L->out_proj_w, L->out_proj_b, x, d, t1, d, n_cap, n_dev, d, d, 0))) return rc;
    sstb_add_norm(st, t1, nullptr, L->norm2_w, L->norm2_b, L->norm2_mean, L->norm2_var, L->norm_eps, x1, n_cap, n_dev, d);
    if ((rc = linear_fp32(c, x1, d, L->lin1_w, L->lin1_b, nullptr, 0, hid, ff, n_cap, n_dev, ff, d, L->act))) return rc;
    if ((rc = linear_fp32(c, hid, ff, L->lin2_w, L->lin2_b, t1, d, y, d, n_cap, n_dev, d, ff, 0))) return rc;
  }
  CUDA_TRY(c, cudaGetLastError());
  return SSTB_OK;
}
