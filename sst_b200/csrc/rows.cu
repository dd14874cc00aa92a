// fp32 row GEMM and row-wise add + norm (declarations and the argument struct in rows.cuh).
#include <stdarg.h>
#include "rows.cuh"

// ------------------------------------------------------------------------------------------------
// generic row GEMM  out[r, n] = epi( sum_k A'[r,k] * W[n,k] + bias[n] )   (nn.Linear layout, fp32 FFMA)
//   A'[r,k] = A[r,k] (+ pos(r,k) if pos table given and n-tile < pos_ncols)
// ------------------------------------------------------------------------------------------------
#define GBM 128
#define GBN 64
#define GBK 16

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

void sstb_row_gemm(cudaStream_t st, const RowGemm& g) {
  if (g.M_cap <= 0) return;
  dim3 grid((g.M_cap + GBM - 1) / GBM, (g.N + GBN - 1) / GBN);
  auto kernel = g.act == 0 ? gemm_rows_kernel<0> : g.act == 1 ? gemm_rows_kernel<1> : gemm_rows_kernel<2>;
  launch_pdl(kernel, grid, dim3(256), (size_t)(0), st, g.A, g.lda, g.W, g.bias, g.res, g.ldr, g.out, g.ldo, g.M_cap, g.M_dev, g.N, g.K,
             g.pos, g.pos_ncols, g.ldw ? g.ldw : g.K, g.res_index);
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
