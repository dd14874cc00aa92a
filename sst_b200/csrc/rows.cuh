// fp32 row building blocks shared by the SRA encoder layer (sra_fp32.cu, sra_api.cu), the SIR layer (sir.cu, sir_train.cu) and the
// VFE's wide path (vfe.cu): one row GEMM in nn.Linear layout and one row-wise add + norm + activation (csrc/rows.cu).
#pragma once
#include "common.cuh"

// per-axis positional table of an SRA plan, added to the GEMM's A operand: A'[r, k] = A[r, k] + pos(code[r], k)
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

// out[r, n] = act(A'[r, :K] . W[n, :K] + bias[n]) + res[res_index ? res_index[r] : r, n]     for r < M (M_dev ? *M_dev : M_cap)
//   A' = A, plus pos on the columns of the output tiles below pos_ncols when pos.tab is set.  act: 0 none, 1 relu, 2 gelu.
// Value-initialise it and set the fields the GEMM uses: every pointer but A, W and out may stay null.
struct RowGemm {
  const float* A; int lda;
  const float* W; int ldw;            // W[n, k] at W[n * ldw + k]; 0 = K
  const float* bias;                  // [N] or null
  const float* res; int ldr;          // or null
  const long long* res_index;         // residual row of output row r (null: r)
  float* out; int ldo;
  int M_cap; const int32_t* M_dev;    // row count: *M_dev when set, M_cap bounds it (and the grid)
  int N, K, act;
  PosTab pos; int pos_ncols;
};

// fp32 FFMA, any shape
void sstb_row_gemm(cudaStream_t st, const RowGemm& g);
// The same GEMM at fp32 tolerance on the tensor core (csrc/spconv.cu, split-fp16 operands).  Returns SSTB_ERR_UNSUPPORTED (nothing
// launched) when it does not take the GEMM - K or N not a multiple of 64, lda / ldo / ldr not a multiple of 4, relu with a
// residual, or any of ldw != K, res_index, pos - and the caller then uses sstb_row_gemm.
// Each row of A and each output channel of W is lifted by a power of two to the top of fp16's range before it is split into an
// fp16 pair (as in sstb200_spconv_forward), so the result is homogeneous in the scale of either operand: an element within 2^-16
// of its row's (channel's) largest |value| keeps 22 significant bits, a smaller one an absolute error of 2^-38 of that largest,
// at any magnitude fp32 holds.  Unscaled, the pair loses bits for every |x| below about 2^-3 - which is where nn.Linear's default
// init (|w| <= 1 / sqrt(K)) and xavier's (|w| <= sqrt(6 / (K + N))) put the weights of an encoder layer, and where small
// activation rows lie.
int sstb_row_gemm_x3(sstb200_ctx* c, const RowGemm& g);

// out = act(LayerNorm(a [+ b]) * gamma + beta), or with bn_mean / bn_var the eval BatchNorm affine; row-wise, d <= 256
void sstb_add_norm_act(cudaStream_t st, const float* a, const float* b, const float* gamma, const float* beta,
                       const float* bn_mean, const float* bn_var, float eps, float* out, int n_cap, const int32_t* n_dev, int d, int act);
