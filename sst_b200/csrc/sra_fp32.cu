// Sparse Regional Attention encoder layer - fp32 SIMT path ("exact" mode, also the bring-up path).
// Replaces, per layer, flat2window -> nn.MultiheadAttention per drop level -> window2flat -> residual/LN/FFN
// (mmdet3d/models/sst/sst_basic_block_v2.py:41-126) with ragged kernels that work on the window CSR:
// no padding to max_tokens, no per-level batches, no masks.
#include <stdarg.h>
#include "rows.cuh"
#include "sra.cuh"
#include "sra_attn.cuh"

// ------------------------------------------------------------------------------------------------
// fp32-tolerance GEMMs on the tensor core: every Linear of the layer runs through sstb_row_gemm_x3 (split-fp16 operands:
// hi.hi + lo.hi + hi.lo in one set of fp32 accumulators, ~2^-22 relative at any operand scale, see rows.cuh) instead of the FFMA
// row GEMM; the positional term of q|k is added to a copy of the input first.  Shapes sstb_row_gemm_x3 does not take (d_model or
// dim_ff not a multiple of 64) run on the FFMA row GEMM.
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

static int linear_fp32(sstb200_ctx* c, const RowGemm& g) {
  const int rc = sstb_row_gemm_x3(c, g);
  if (rc != SSTB_ERR_UNSUPPORTED) return rc;
  sstb_row_gemm(c->stream, g);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// one encoder layer, fp32
// ------------------------------------------------------------------------------------------------
int sstb_sra_layer_fp32(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x, float* y,
                        int n_cap, const int32_t* n_dev) {
  int d = L->d_model, ff = L->dim_ff;
  if (d > 256 || d % 32) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "d_model %d (need multiple of 32, <= 256)", d);
  float *qkv, *att, *t1, *x1, *hid, *xpos = nullptr;
  int rc = arena_carve(c, [&](Carve& cv) {
    qkv = cv.take<float>((size_t)n_cap * 3 * d);
    att = cv.take<float>((size_t)n_cap * d);
    t1 = cv.take<float>((size_t)n_cap * d);
    x1 = cv.take<float>((size_t)n_cap * d);
    hid = cv.take<float>((size_t)n_cap * ff);
    if (d % 64 == 0 && ff % 64 == 0 && P->pos_table) xpos = cv.take<float>((size_t)n_cap * d);  // q|k input of the x3 route
  });
  if (rc) return rc;
  cudaStream_t st = c->stream;
  const float* xin = x;
  if (!L->post_norm) {  // pre-norm: src2 = norm1(src)
    sstb_add_norm_act(st, x, nullptr, L->norm1_w, L->norm1_b, L->norm1_mean, L->norm1_var, L->norm_eps, x1, n_cap, n_dev, d, 0);
    xin = x1;
  }
  RowGemm base{};  // the rows every Linear of the layer runs over
  base.M_cap = n_cap, base.M_dev = n_dev;
  const PosTab pt{P->pos_table, P->pos_code, P->pos_L, P->pos_maxw, P->pos_ndim};
  // q,k from (x + pos); v from x
  if (d % 64 == 0 && ff % 64 == 0) {
    const float* xqk = xin;
    if (P->pos_table) {
      const size_t tot = (size_t)n_cap * d;
      launch_pdl(add_pos_kernel, dim3((unsigned)((tot + 255) / 256)), dim3(256), (size_t)0, st, xin, d, pt, xpos, n_cap, n_dev);
      xqk = xpos;
    }
    RowGemm qk = base;
    qk.A = xqk, qk.lda = d, qk.W = L->in_proj_w, qk.bias = L->in_proj_b, qk.out = qkv, qk.ldo = 3 * d, qk.N = 2 * d, qk.K = d;
    if ((rc = linear_fp32(c, qk))) return rc;
    RowGemm v = base;
    v.A = xin, v.lda = d, v.W = L->in_proj_w + (size_t)2 * d * d, v.bias = L->in_proj_b + 2 * d, v.out = qkv + 2 * d, v.ldo = 3 * d;
    v.N = d, v.K = d;
    if ((rc = linear_fp32(c, v))) return rc;
  } else {  // q|k|v in one FFMA GEMM, the positional term added to the A loads of the q|k columns
    RowGemm g = base;
    g.A = xin, g.lda = d, g.W = L->in_proj_w, g.bias = L->in_proj_b, g.out = qkv, g.ldo = 3 * d, g.N = 3 * d, g.K = d;
    g.pos = pt, g.pos_ncols = 2 * d;
    sstb_row_gemm(st, g);
  }
  rc = sstb_win_attn<float, float>(c, qkv, d, L->nhead, n_cap, n_dev, P->win_offsets, P->tok_perm, P->tok_win, L->tau, L->tau_n,
                                   L->tau_min, att);
  if (rc) return rc;
  RowGemm proj = base, lin1 = base, lin2 = base;
  proj.A = att, proj.lda = d, proj.W = L->out_proj_w, proj.bias = L->out_proj_b, proj.out = t1, proj.ldo = d, proj.N = d, proj.K = d;
  lin1.A = x1, lin1.lda = d, lin1.W = L->lin1_w, lin1.bias = L->lin1_b, lin1.out = hid, lin1.ldo = ff, lin1.N = ff, lin1.K = d;
  lin1.act = L->act;
  lin2.A = hid, lin2.lda = ff, lin2.W = L->lin2_w, lin2.bias = L->lin2_b, lin2.out = t1, lin2.ldo = d, lin2.N = d, lin2.K = ff;
  if (L->post_norm) {
    if ((rc = linear_fp32(c, proj))) return rc;
    sstb_add_norm_act(st, x, t1, L->norm1_w, L->norm1_b, L->norm1_mean, L->norm1_var, L->norm_eps, x1, n_cap, n_dev, d, 0);
    if ((rc = linear_fp32(c, lin1))) return rc;
    if ((rc = linear_fp32(c, lin2))) return rc;
    sstb_add_norm_act(st, x1, t1, L->norm2_w, L->norm2_b, L->norm2_mean, L->norm2_var, L->norm_eps, y, n_cap, n_dev, d, 0);
  } else {
    // src = src + attn ; src = src + ffn(norm2(src))
    proj.res = x, proj.ldr = d;
    lin2.res = t1, lin2.ldr = d, lin2.out = y;
    if ((rc = linear_fp32(c, proj))) return rc;
    sstb_add_norm_act(st, t1, nullptr, L->norm2_w, L->norm2_b, L->norm2_mean, L->norm2_var, L->norm_eps, x1, n_cap, n_dev, d, 0);
    if ((rc = linear_fp32(c, lin1))) return rc;
    if ((rc = linear_fp32(c, lin2))) return rc;
  }
  CUDA_TRY(c, cudaGetLastError());
  return SSTB_OK;
}
