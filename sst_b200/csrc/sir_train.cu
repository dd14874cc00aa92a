// SIRLayer backward (training), fp32 - the autograd graph torch builds over voxel_encoder.py:696-764 in the reference, in the
// layout of the sir.cu header comment.  Per block:
//
//   dp1   = grad_point, plus grad_group[:, C0:] at the arg-max row of each group max     (layer 1 output)
//   dt1   = LN/act backward of layer 1 (one warp per row), with d gamma1 / d beta1
//   S1    = segsum(dt1)                       dW1 = [dt1^T p0 || S1^T g0]     ([p0 || g0[group]] is never built)
//   dp0   = dt1 W1a, plus (S1 W1b + grad_group[:, :C0]) at the arg-max rows of g0
//   dt0   = LN/act backward of layer 0        dW0 = dt0^T x0                   dx0 = dt0 W0
//   gating + rel-MLP backward (one warp per point): grad_in_feats, grad_f_cluster, and per-layer dz / inputs for the rel weights
//
// p0 (from t0), g0 (p0 at the arg-max rows) and x0 (the forward's rel-gate kernel) are recomputed; the state holds only t0, t1
// and the arg-max rows.  Nothing uses float atomics: reductions over rows run over fixed row partitions with an ordered final sum,
// the segmented sum S1 accumulates in fp64 (launch_segment_reduce), and each arg-max scatter writes every (row, channel) at most
// once (a row belongs to one group).  Two calls on the same inputs give the same bits.
#include <stdarg.h>
#include "index.cuh"
#include "rows.cuh"
#include "sir.cuh"

// ---- small helpers ---------------------------------------------------------------------------------
// out[c, r] = W[r, c]   (W [rows, >= cols] with row pitch ldw)
__global__ void sirb_transpose_kernel(const float* __restrict__ W, int ldw, int rows, int cols, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  int r = i / cols, c = i % cols;
  out[(size_t)c * rows + r] = W[(size_t)r * ldw + c];
}

// dP[am[g, c], c] += src[g, col0 + c]: the backward of a group max.  Rows of different groups are distinct, so every (row, c) is
// written at most once (no race, no atomic).  am == N marks an empty group.
__global__ void sirb_scatter_max_kernel(const long long* __restrict__ am, int G, int C, const float* __restrict__ src, int lds, int col0,
                                        float* __restrict__ dP, int N) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * C) return;
  int g = (int)(i / C), c = (int)(i % C);
  long long n = am[i];
  if (n >= 0 && n < N) dP[(size_t)n * C + c] += src[(size_t)g * lds + col0 + c];
}

// g0[g, c] = p0[am[g, c], c]  (0 for an empty group)
__global__ void sirb_gather_max_kernel(const long long* __restrict__ am, int G, int C, const float* __restrict__ p, int N, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * C) return;
  long long n = am[i];
  out[i] = (n >= 0 && n < N) ? p[(size_t)n * C + i % C] : 0.f;
}

// out[(i / K) * ldo + i % K] = sum_{p < nparts} part[p * pstride + i], in order p = 0, 1, ...
__global__ void sirb_reduce_parts_kernel(const float* __restrict__ part, int nparts, size_t pstride, int n, int K, int ldo, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int p = 0; p < nparts; p++) s += part[(size_t)p * pstride + i];
  out[(size_t)(i / K) * ldo + i % K] = s;
}

__device__ __forceinline__ float act_grad(float z, int act) {
  if (act == 2) return 0.5f * (1.f + erff(z * 0.70710678118654752440f)) + z * 0.39894228040143267794f * expf(-0.5f * z * z);
  return z > 0.f ? 1.f : 0.f;
}

// ---- LayerNorm + activation backward, one warp per row ---------------------------------------------------
// t [N, d] pre-LN, dy [N, d] gradient of act(LN(t)) -> dt [N, d]; part[block][2][d] = this block's sum of dz * xhat and dz
// (dz = gradient at the LN output) over its rows.  The grid is fixed, so each warp's rows and the sum order are too.
#define LNB_WARPS 8
__global__ void __launch_bounds__(256) sirb_ln_act_bwd_kernel(const float* __restrict__ t, const float* __restrict__ dy, int N, int d,
                                                              const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                              int act, float* __restrict__ dt, float* __restrict__ part) {
  pdl_wait();
  pdl_launch();
  __shared__ float sred[LNB_WARPS][2][256];
  const int ln = lane_id(), w = threadIdx.x >> 5;
  const int warps = gridDim.x * LNB_WARPS;
  float ag[8], ab[8];
#pragma unroll
  for (int j = 0; j < 8; j++) ag[j] = ab[j] = 0.f;
  for (int row = blockIdx.x * LNB_WARPS + w; row < N; row += warps) {
    const float* tp = t + (size_t)row * d;
    float v[8], s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      int c = ln + 32 * j;
      v[j] = c < d ? tp[c] : 0.f;
      s += v[j];
    }
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < 8; j++)
      if (ln + 32 * j < d) {
        float u = v[j] - mean;
        q += u * u;
      }
    const float rstd = rsqrtf(warp_sum(q) / (float)d + eps);
    float g[8], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      int c = ln + 32 * j;
      g[j] = 0.f;
      if (c < d) {
        float xh = (v[j] - mean) * rstd;
        float dz = dy[(size_t)row * d + c] * act_grad(xh * gamma[c] + beta[c], act);
        ag[j] += dz * xh;
        ab[j] += dz;
        g[j] = dz * gamma[c];
        v[j] = xh;
        s1 += g[j];
        s2 += g[j] * xh;
      }
    }
    const float m1 = warp_sum(s1) / (float)d, m2 = warp_sum(s2) / (float)d;
#pragma unroll
    for (int j = 0; j < 8; j++) {
      int c = ln + 32 * j;
      if (c < d) dt[(size_t)row * d + c] = rstd * (g[j] - m1 - v[j] * m2);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; j++) {
    sred[w][0][ln + 32 * j] = ag[j];
    sred[w][1][ln + 32 * j] = ab[j];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * d; i += blockDim.x) {
    int k = i / d, c = i % d;
    float s = 0.f;
    for (int ww = 0; ww < LNB_WARPS; ww++) s += sred[ww][k][c];
    part[(size_t)blockIdx.x * 2 * d + i] = s;
  }
}

// ---- weight gradient: part[split][m][k] = sum over the split's rows r of A[r, m] * B[r, k] ---------------------------------
// 64 x 64 output tile per block, 4 x 4 per thread, 16 rows per step; splits partition the rows in fixed ranges.  The sums run
// over up to ~10^5 rows of terms that largely cancel, so the fp32 tile sums are flushed into fp64 every DW_FLUSH steps and the
// split partials are fp64: the fp32 rounding chain of any one sum is at most 64 rows long.
#define DWT 64
#define DWR 16
#define DW_FLUSH 4  // steps of DWR rows
__global__ void __launch_bounds__(256) sirb_dw_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, int R, int M,
                                                      int K, int rows_per_split, double* __restrict__ part) {
  pdl_wait();
  pdl_launch();
  __shared__ __align__(16) float As[DWR][DWT];
  __shared__ __align__(16) float Bs[DWR][DWT];
  const int m0 = blockIdx.x * DWT, k0 = blockIdx.y * DWT;
  const int r0 = blockIdx.z * rows_per_split, r1 = min(R, r0 + rows_per_split);
  const int tid = threadIdx.x, tm = tid / 16, tk = tid % 16;
  float acc[4][4];
  double dacc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f, dacc[i][j] = 0.0;
  int step = 0;
  for (int r = r0; r < r1; r += DWR) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      int e = tid + u * 256;
      int rr = e / DWT, cc = e % DWT;
      int gr = r + rr;
      As[rr][cc] = (gr < r1 && m0 + cc < M) ? A[(size_t)gr * lda + m0 + cc] : 0.f;
      Bs[rr][cc] = (gr < r1 && k0 + cc < K) ? B[(size_t)gr * ldb + k0 + cc] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < DWR; q++) {
      float a[4], b[4];
      *(float4*)a = *(const float4*)&As[q][tm * 4];
      *(float4*)b = *(const float4*)&Bs[q][tk * 4];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
    if (++step == DW_FLUSH) {
      step = 0;
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) dacc[i][j] += (double)acc[i][j], acc[i][j] = 0.f;
    }
  }
  double* out = part + (size_t)blockIdx.z * M * K;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    int m = m0 + tm * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int k = k0 + tk * 4 + j;
      if (k < K) out[(size_t)m * K + k] = dacc[i][j] + (double)acc[i][j];
    }
  }
}

// out[(i / K) * ldo + i % K] = sum_{p < nparts} part[p * pstride + i] in fp64, in order p = 0, 1, ...
__global__ void sirb_reduce_parts_f64_kernel(const double* __restrict__ part, int nparts, size_t pstride, int n, int K, int ldo,
                                             float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int p = 0; p < nparts; p++) s += part[(size_t)p * pstride + i];
  out[(size_t)(i / K) * ldo + i % K] = (float)s;
}

// splits for an [M, K] weight gradient over R rows: enough blocks for two waves, at least 64 rows each
static int dw_splits(const sstb200_ctx* c, int R, int M, int K) {
  int tiles = ((M + DWT - 1) / DWT) * ((K + DWT - 1) / DWT);
  int s = (2 * c->num_sms + tiles - 1) / tiles;
  int smax = (R + 63) / 64;
  if (s > smax) s = smax;
  return s < 1 ? 1 : s;
}

// out [M, K] (row pitch ldo) = A[R, M]^T . B[R, K], deterministic; part = scratch of dw_splits(R, M, K) * M * K doubles
static void sir_dw(sstb200_ctx* c, const float* A, int lda, const float* B, int ldb, int R, int M, int K, double* part, float* out, int ldo) {
  int s = dw_splits(c, R, M, K);
  int rps = (((R + s - 1) / s) + DWR - 1) / DWR * DWR;
  s = (R + rps - 1) / rps;
  if (s < 1) s = 1;
  dim3 grid((M + DWT - 1) / DWT, (K + DWT - 1) / DWT, s);
  launch_pdl(sirb_dw_kernel, grid, dim3(256), (size_t)0, c->stream, A, lda, B, ldb, R, M, K, rps, part);
  int n = M * K;
  launch_pdl(sirb_reduce_parts_f64_kernel, dim3((n + 255) / 256), dim3(256), (size_t)0, c->stream, (const double*)part, s, (size_t)n, n, K, ldo, out);
}

// ---- gating + relation-MLP backward: one warp per point --------------------------------------------------
// Recomputes the rel-MLP forward (the same arithmetic as sir_rel_gate_kernel), then runs it backwards.  Writes, per point,
// each layer's input a_l [N, in_l] (a_0 = f_cluster / rel_dist_scaler) and pre-LN gradient dz_l [N, dims[l]] for the
// weight gradients, and accumulates the LN gamma / beta gradients per warp in shared memory (each lane owns its channels).
struct RelBwd {
  float* a[4];
  float* dz[4];
  int ln_off[4];  // layer l's [2][dims[l]] slice of a ln_tot-float row (gamma, then beta)
  int ln_tot;
};

#define RELB_WARPS 8
__global__ void __launch_bounds__(256, 1) sirb_rel_bwd_kernel(RelDev r, RelBwd o, const float* __restrict__ feats, const float* __restrict__ f_cluster,
                                                           const float* __restrict__ dx0, const float* __restrict__ grad_point, int Cshort, int N,
                                                           float* __restrict__ grad_in, float* __restrict__ grad_fc, float* __restrict__ ln_part) {
  pdl_wait();
  pdl_launch();
  extern __shared__ float sm[];
  float* wl[4];  // transposed weights as in the forward: layer l stored [in_l][out_l]
  float* p = sm;
  {
    int in = r.rel_in;
#pragma unroll
    for (int l = 0; l < 4; l++) {
      wl[l] = p;
      if (l < r.n_rel) {
        for (int i = threadIdx.x; i < in * r.dims[l]; i += blockDim.x) {
          int k = i / r.dims[l], c = i % r.dims[l];
          p[i] = r.w[l][(size_t)c * in + k];
        }
        p += in * r.dims[l];
        in = r.dims[l];
      }
    }
  }
  const int ln = lane_id(), wid = threadIdx.x >> 5;
  float* acc_ln = p + (size_t)wid * o.ln_tot;  // this warp's gamma / beta sums
  for (int i = ln; i < o.ln_tot; i += 32) acc_ln[i] = 0.f;
  __syncthreads();
  const int warps = gridDim.x * RELB_WARPS;
  for (int pt = blockIdx.x * RELB_WARPS + wid; pt < N; pt += warps) {
    float cur[REL_MAXC], xh[4][REL_MAXC], rstd[4];
#pragma unroll
    for (int j = 0; j < REL_MAXC; j++) cur[j] = 0.f;
    if (ln < r.rel_in) cur[0] = f_cluster[(size_t)pt * r.rel_in + ln] / r.rel_dist_scaler;
    // forward, keeping xhat and rstd of every layer
    int in = r.rel_in;
#pragma unroll
    for (int l = 0; l < 4; l++) {
      if (l < r.n_rel) {
        const int out = r.dims[l];
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++)
          if (ln + 32 * j < in) o.a[l][(size_t)pt * in + ln + 32 * j] = cur[j];
        float acc[REL_MAXC];
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++) acc[j] = 0.f;
#pragma unroll
        for (int jk = 0; jk < REL_MAXC; jk++) {
          if (32 * jk < in) {
            int kmax = min(32, in - 32 * jk);
            for (int kk = 0; kk < kmax; kk++) {
              float xk = __shfl_sync(0xffffffffu, cur[jk], kk);
              const float* wr = wl[l] + (size_t)(32 * jk + kk) * out;
#pragma unroll
              for (int j = 0; j < REL_MAXC; j++) {
                int c = ln + 32 * j;
                if (c < out) acc[j] = fmaf(wr[c], xk, acc[j]);
              }
            }
          }
        }
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++)
          if (ln + 32 * j < out) s += acc[j];
        float mean = warp_sum(s) / (float)out;
        float q = 0.f;
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++)
          if (ln + 32 * j < out) {
            float u = acc[j] - mean;
            q += u * u;
          }
        rstd[l] = rsqrtf(warp_sum(q) / (float)out + r.eps);
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++) {
          int c = ln + 32 * j;
          xh[l][j] = c < out ? (acc[j] - mean) * rstd[l] : 0.f;
          cur[j] = c < out ? act_fn(xh[l][j] * r.g[l][c] + r.b[l][c], r.act) : 0.f;
        }
        in = out;
      }
    }
    // gating: x0 = xs * rel, xs = [xyz / normalizer || rest]
    float da[REL_MAXC];
#pragma unroll
    for (int j = 0; j < REL_MAXC; j++) {
      int c = ln + 32 * j;
      da[j] = 0.f;
      if (c < r.cin) {
        float v = feats[(size_t)pt * r.cin + c];
        float nz = c < 3 ? (c == 0 ? r.inv_norm[0] : (c == 1 ? r.inv_norm[1] : r.inv_norm[2])) : 1.f;
        float g = dx0[(size_t)pt * r.cin + c];
        da[j] = g * (c < 3 ? v / nz : v);
        if (grad_in) {
          float gi = c < 3 ? g * cur[j] / nz : g * cur[j];
          if (Cshort && c >= 3) gi += grad_point[(size_t)pt * Cshort + c - 3];
          grad_in[(size_t)pt * r.cin + c] = gi;
        }
      }
    }
    // rel-MLP backward, last layer first
#pragma unroll
    for (int l = 3; l >= 0; l--) {
      if (l < r.n_rel) {
        const int out = r.dims[l], lin = l ? r.dims[l - 1] : r.rel_in;
        float g[REL_MAXC], s1 = 0.f, s2 = 0.f;
        float* ag = acc_ln + o.ln_off[l];
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++) {
          int c = ln + 32 * j;
          g[j] = 0.f;
          if (c < out) {
            float dz = da[j] * act_grad(xh[l][j] * r.g[l][c] + r.b[l][c], r.act);
            ag[c] += dz * xh[l][j];
            ag[out + c] += dz;
            g[j] = dz * r.g[l][c];
            s1 += g[j];
            s2 += g[j] * xh[l][j];
          }
        }
        const float m1 = warp_sum(s1) / (float)out, m2 = warp_sum(s2) / (float)out;
        float dt[REL_MAXC];
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++) {
          int c = ln + 32 * j;
          dt[j] = c < out ? rstd[l] * (g[j] - m1 - xh[l][j] * m2) : 0.f;
          if (c < out) o.dz[l][(size_t)pt * out + c] = dt[j];
        }
        // d input[k] = sum_c W_l[c, k] dt[c]  (lane owns k = ln + 32 jk; W in nn.Linear layout, rows read coalesced)
        float nd[REL_MAXC];
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++) nd[j] = 0.f;
        const float* W = r.w[l];
#pragma unroll
        for (int jc = 0; jc < REL_MAXC; jc++) {
          if (32 * jc < out) {
            int cmax = min(32, out - 32 * jc);
            for (int cc = 0; cc < cmax; cc++) {
              float dc = __shfl_sync(0xffffffffu, dt[jc], cc);
              const float* wr = W + (size_t)(32 * jc + cc) * lin;
#pragma unroll
              for (int j = 0; j < REL_MAXC; j++) {
                int k = ln + 32 * j;
                if (k < lin) nd[j] = fmaf(__ldg(&wr[k]), dc, nd[j]);
              }
            }
          }
        }
#pragma unroll
        for (int j = 0; j < REL_MAXC; j++) da[j] = nd[j];
      }
    }
    if (grad_fc && ln < r.rel_in) grad_fc[(size_t)pt * r.rel_in + ln] = da[0] / r.rel_dist_scaler;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < o.ln_tot; i += blockDim.x) {
    float s = 0.f;
    for (int ww = 0; ww < RELB_WARPS; ww++) s += p[(size_t)ww * o.ln_tot + i];
    ln_part[(size_t)blockIdx.x * o.ln_tot + i] = s;
  }
}

extern "C" int sstb200_sir_layer_backward(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster,
                                          const int64_t* inv_, int N, int G, const int32_t* csr_offsets, const int32_t* csr_order,
                                          const void* state, size_t state_bytes, const float* grad_point, const float* grad_group,
                                          float* grad_in_feats, float* grad_f_cluster, const sstb200_sir_layer_grads* grads) {
  CHECK_ARG(c, c && L && grads && N >= 0 && G >= 0);
  int rc = sstb_sir_train_check(c, L);
  if (rc) return rc;
  if (N == 0 || G == 0) return SSTB_OK;
  CHECK_ARG(c, in_feats && f_cluster && inv_ && state);
  CHECK_ARG(c, (csr_offsets == nullptr) == (csr_order == nullptr));
  const long long* inv = (const long long*)inv_;
  const int cin = L->in_channels, C0 = L->feat_channels[0], C1 = L->num_vfe > 1 ? L->feat_channels[1] : 0;
  const int Cg = C0 + C1, Clast = C1 ? C1 : C0;
  for (int l = 0; l < L->num_rel; l++) CHECK_ARG(c, grads->rel_w[l] && grads->rel_ln_w[l] && grads->rel_ln_b[l]);
  for (int l = 0; l < L->num_vfe; l++) CHECK_ARG(c, grads->vfe_w[l] && grads->vfe_ln_w[l] && grads->vfe_ln_b[l] && L->vfe_w[l]);
  const size_t need = sir_state_bytes(N, G, C0, C1);
  if (state_bytes < need)
    return sstb_fail(c, SSTB_ERR_WORKSPACE, "SIRLayer training state: %zu bytes given, %zu needed", state_bytes, need);
  SirState s;
  Carve sc{(char*)state, 0};
  sir_state_carve(sc, s, N, G, C0, C1);
  RelDev rd;
  size_t wsmem = 0;
  if ((rc = sstb_sir_rel_dev(c, L, &rd, &wsmem))) return rc;
  RelBwd ob;
  int ln_tot = 0, a_tot = 0, dz_tot = 0;
  for (int l = 0; l < L->num_rel; l++) {
    ob.ln_off[l] = ln_tot;
    ln_tot += 2 * L->rel_dims[l];
    a_tot += l ? L->rel_dims[l - 1] : L->rel_in;
    dz_tot += L->rel_dims[l];
  }
  ob.ln_tot = ln_tot;
  const size_t rel_smem = wsmem + (size_t)RELB_WARPS * ln_tot * 4;
  if (rel_smem > 227 * 1024) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer training: rel-MLP does not fit shared memory");

  const int ln_blocks = c->num_sms * 2, rel_blocks = c->num_sms * 2;
  // weight-gradient scratch: the largest of the [M, K] reductions
  size_t dw_part = 0;
  auto upd = [&](int R, int M, int K) {
    size_t b = (size_t)dw_splits(c, R, M, K) * M * K;
    if (b > dw_part) dw_part = b;
  };
  upd(N, C0, cin);
  if (C1) upd(N, C1, C0), upd(G, C1, C0);
  {
    int in = L->rel_in;
    for (int l = 0; l < L->num_rel; l++) upd(N, L->rel_dims[l], in), in = L->rel_dims[l];
  }
  const size_t Nf = (size_t)N;
  arena_reset(c);
  SirGroupCsr gc;
  float *W0t, *x0, *dx0, *dP0, *dt0, *lnp, *relp, *abuf, *dzbuf;
  double* part;
  float *W1at = nullptr, *W1bt = nullptr, *p0 = nullptr, *g0 = nullptr, *dP1 = nullptr, *dt1 = nullptr, *S1 = nullptr, *dg0 = nullptr;
  rc = arena_carve(c, [&](Carve& cv) {
    if (!csr_order) sstb_sir_group_csr_carve(cv, gc, N, G);
    W0t = cv.take<float>((size_t)cin * C0);
    x0 = cv.take<float>(Nf * cin);
    dx0 = cv.take<float>(Nf * cin);
    dP0 = cv.take<float>(Nf * C0);
    dt0 = cv.take<float>(Nf * C0);
    part = cv.take<double>(dw_part);
    lnp = cv.take<float>((size_t)ln_blocks * 2 * 256);
    relp = cv.take<float>((size_t)rel_blocks * ln_tot);
    abuf = cv.take<float>(Nf * a_tot);
    dzbuf = cv.take<float>(Nf * dz_tot);
    if (C1) {
      W1at = cv.take<float>((size_t)C0 * C1);
      W1bt = cv.take<float>((size_t)C0 * C1);
      p0 = cv.take<float>(Nf * C0);
      g0 = cv.take<float>((size_t)G * C0);
      dP1 = cv.take<float>(Nf * C1);
      dt1 = cv.take<float>(Nf * C1);
      S1 = cv.take<float>((size_t)G * C1);
      dg0 = cv.take<float>((size_t)G * C0);
    }
  });
  if (rc) return rc;
  cudaStream_t st = c->stream;
  const int32_t *off = csr_offsets, *order = csr_order;
  if (!order) {
    if ((rc = sstb_sir_group_csr(c, gc, inv, N, G))) return rc;
    off = (const int32_t*)gc.csr.offsets;
    order = gc.csr.order;
  }

  auto blocks = [](size_t n) { return dim3((unsigned)((n + 255) / 256)); };
  auto ln_bwd = [&](const float* t, const float* dy, int d, int l, float* dt) {
    launch_pdl(sirb_ln_act_bwd_kernel, dim3(ln_blocks), dim3(256), (size_t)0, st, t, dy, N, d, L->vfe_ln_w[l], L->vfe_ln_b[l], L->norm_eps, L->act,
               dt, lnp);
    launch_pdl(sirb_reduce_parts_kernel, blocks(d), dim3(256), (size_t)0, st, (const float*)lnp, ln_blocks, (size_t)2 * d, d, d, d, grads->vfe_ln_w[l]);
    launch_pdl(sirb_reduce_parts_kernel, blocks(d), dim3(256), (size_t)0, st, (const float*)(lnp + d), ln_blocks, (size_t)2 * d, d, d, d,
               grads->vfe_ln_b[l]);
  };

  // x0 as the forward built it
  if ((rc = sstb_sir_rel_gate(c, L, in_feats, f_cluster, N, x0))) return rc;
  launch_pdl(sirb_transpose_kernel, blocks((size_t)C0 * cin), dim3(256), (size_t)0, st, L->vfe_w[0], cin, C0, cin, W0t);

  // dP1 / dP0: the gradient at each layer's activation output (the shortcut's share goes straight to in_feats below)
  if (C1) {
    launch_pdl(sirb_transpose_kernel, blocks((size_t)C1 * C0), dim3(256), (size_t)0, st, L->vfe_w[1], 2 * C0, C1, C0, W1at);
    launch_pdl(sirb_transpose_kernel, blocks((size_t)C1 * C0), dim3(256), (size_t)0, st, L->vfe_w[1] + C0, 2 * C0, C1, C0, W1bt);
    // p0 and g0 as the forward had them
    sstb_add_norm_act(st, s.t0, nullptr, L->vfe_ln_w[0], L->vfe_ln_b[0], nullptr, nullptr, L->norm_eps, p0, N, nullptr, C0, L->act);
    launch_pdl(sirb_gather_max_kernel, blocks((size_t)G * C0), dim3(256), (size_t)0, st, (const long long*)s.am0, G, C0, (const float*)p0, N, g0);
    // layer 1
    if (grad_point) CUDA_TRY(c, cudaMemcpyAsync(dP1, grad_point, Nf * C1 * 4, cudaMemcpyDeviceToDevice, st));
    else CUDA_TRY(c, cudaMemsetAsync(dP1, 0, Nf * C1 * 4, st));
    if (grad_group)
      launch_pdl(sirb_scatter_max_kernel, blocks((size_t)G * C1), dim3(256), (size_t)0, st, (const long long*)s.am1, G, C1, grad_group, Cg, C0, dP1, N);
    ln_bwd(s.t1, dP1, C1, 1, dt1);
    launch_segment_reduce(c, dt1, C1, (const uint32_t*)off, order, G, nullptr, SSTB200_REDUCE_SUM, 0.f, S1, nullptr, N);
    sir_dw(c, dt1, C1, p0, C0, N, C1, C0, part, grads->vfe_w[1], 2 * C0);
    sir_dw(c, S1, C1, g0, C0, G, C1, C0, part, grads->vfe_w[1] + C0, 2 * C0);
    // into layer 0: dp0 = dt1 W1a, dg0 = S1 W1b + grad_group[:, :C0] at the arg-max rows
    RowGemm dg{}, dp{};
    dg.A = S1, dg.lda = C1, dg.W = W1bt, dg.res = grad_group, dg.ldr = Cg, dg.out = dg0, dg.ldo = C0, dg.M_cap = G, dg.N = C0, dg.K = C1;
    sstb_row_gemm(st, dg);
    dp.A = dt1, dp.lda = C1, dp.W = W1at, dp.out = dP0, dp.ldo = C0, dp.M_cap = N, dp.N = C0, dp.K = C1;
    sstb_row_gemm(st, dp);
    launch_pdl(sirb_scatter_max_kernel, blocks((size_t)G * C0), dim3(256), (size_t)0, st, (const long long*)s.am0, G, C0, (const float*)dg0, C0, 0, dP0, N);
  } else {
    if (grad_point) CUDA_TRY(c, cudaMemcpyAsync(dP0, grad_point, Nf * C0 * 4, cudaMemcpyDeviceToDevice, st));
    else CUDA_TRY(c, cudaMemsetAsync(dP0, 0, Nf * C0 * 4, st));
    if (grad_group)
      launch_pdl(sirb_scatter_max_kernel, blocks((size_t)G * C0), dim3(256), (size_t)0, st, (const long long*)s.am0, G, C0, grad_group, Cg, 0, dP0, N);
  }
  // layer 0
  ln_bwd(s.t0, dP0, C0, 0, dt0);
  sir_dw(c, dt0, C0, x0, cin, N, C0, cin, part, grads->vfe_w[0], cin);
  RowGemm dx{};
  dx.A = dt0, dx.lda = C0, dx.W = W0t, dx.out = dx0, dx.ldo = cin, dx.M_cap = N, dx.N = cin, dx.K = C0;
  sstb_row_gemm(st, dx);

  // gating + rel-MLP
  {
    float* pa = abuf;
    float* pz = dzbuf;
    int in = L->rel_in;
    for (int l = 0; l < 4; l++) {
      ob.a[l] = ob.dz[l] = nullptr;
      if (l < L->num_rel) {
        ob.a[l] = pa;
        ob.dz[l] = pz;
        pa += Nf * in;
        pz += Nf * L->rel_dims[l];
        in = L->rel_dims[l];
      }
    }
    const int Cshort = (L->with_shortcut && cin - 3 == Clast && grad_point) ? Clast : 0;
    static SmemAttr sa;
    CUDA_TRY(c, ensure_smem(c, sa, sirb_rel_bwd_kernel, (size_t)227 * 1024));
    launch_pdl(sirb_rel_bwd_kernel, dim3(rel_blocks), dim3(256), rel_smem, st, rd, ob, in_feats, f_cluster, (const float*)dx0, grad_point, Cshort,
               N, grad_in_feats, grad_f_cluster, relp);
    in = L->rel_in;
    for (int l = 0; l < L->num_rel; l++) {
      const int d = L->rel_dims[l];
      sir_dw(c, ob.dz[l], d, ob.a[l], in, N, d, in, part, grads->rel_w[l], in);
      launch_pdl(sirb_reduce_parts_kernel, blocks(d), dim3(256), (size_t)0, st, (const float*)(relp + ob.ln_off[l]), rel_blocks, (size_t)ln_tot, d, d, d,
                 grads->rel_ln_w[l]);
      launch_pdl(sirb_reduce_parts_kernel, blocks(d), dim3(256), (size_t)0, st, (const float*)(relp + ob.ln_off[l] + d), rel_blocks, (size_t)ln_tot, d,
                 d, d, grads->rel_ln_b[l]);
      in = d;
    }
  }
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
