// C-ABI entry for the SRA encoder layer; dispatches on precision.
#include <stdarg.h>
#include "rows.cuh"
#include "sra.cuh"

extern "C" int sstb200_sra_layer_forward(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x,
                                         float* y, int n, const int32_t* n_dev, int precision) {
  CHECK_ARG(c, c && L && P && n >= 0);
  if (n == 0) return SSTB_OK;
  CHECK_ARG(c, x && y && L->d_model > 0 && L->nhead > 0 && L->d_model % L->nhead == 0 && L->dim_ff > 0);
  CHECK_ARG(c, L->in_proj_w && L->in_proj_b && L->out_proj_w && L->out_proj_b && L->lin1_w && L->lin1_b && L->lin2_w && L->lin2_b);
  CHECK_ARG(c, L->norm1_w && L->norm1_b && L->norm2_w && L->norm2_b && (L->act == 1 || L->act == 2));
  CHECK_ARG(c, P->win_offsets && P->tok_perm && P->tok_win);
  CHECK_ARG(c, P->pos_table == nullptr || (P->pos_code && P->pos_L > 0 && P->pos_maxw > 0 && P->pos_ndim >= 1 && P->pos_ndim <= 3));
  arena_reset(c);
  if (precision == SSTB200_PREC_FP32) return sstb_sra_layer_fp32(c, L, P, x, y, n, n_dev);
  if (precision == SSTB200_PREC_BF16) return sstb_sra_layer_bf16(c, L, P, x, y, n, n_dev);
  return sstb_fail(c, SSTB_ERR_ARG, "unknown precision %d", precision);
}

extern "C" int sstb200_linear(sstb200_ctx* c, const float* A, const float* W, const float* bias, float* out, int M, int N,
                              int K, int act) {
  CHECK_ARG(c, c && M >= 0 && N > 0 && K > 0 && act >= 0 && act <= 2);
  if (M == 0) return SSTB_OK;
  CHECK_ARG(c, A && W && out);
  RowGemm g{};
  g.A = A, g.lda = K, g.W = W, g.bias = bias, g.out = out, g.ldo = N, g.M_cap = M, g.N = N, g.K = K, g.act = act;
  sstb_row_gemm(c->stream, g);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_sra_stack_forward(sstb200_ctx* c, const sstb200_sra_layer* layers, int num_layers, const sstb200_sra_plan* plan_shift0,
                                         const sstb200_sra_plan* plan_shift1, const float* x, float* y, float* tmp, int n,
                                         const int32_t* n_dev, int precision) {
  CHECK_ARG(c, c && layers && num_layers >= 0 && plan_shift0 && plan_shift1 && n >= 0);
  if (n == 0 || num_layers == 0) return SSTB_OK;
  CHECK_ARG(c, x && y && tmp && x != y && tmp != y && tmp != x);
  sstb200_sra_plan plans[2] = {*plan_shift0, *plan_shift1};
  if (precision == SSTB200_PREC_BF16) {
    arena_reset(c);
    int rc = sstb_sra_stack_bf16(c, layers, num_layers, plans, x, y, tmp, n, n_dev);
    if (rc != SSTB_ERR_UNSUPPORTED) return rc;
  }
  // generic path: layer by layer, ping-pong between tmp and y so that the last layer lands in y
  const float* src = x;
  for (int l = 0; l < num_layers; l++) {
    float* dst = ((num_layers - 1 - l) & 1) ? tmp : y;
    int rc = sstb200_sra_layer_forward(c, &layers[l], &plans[l & 1], src, dst, n, n_dev, precision);
    if (rc) return rc;
    src = dst;
  }
  return SSTB_OK;
}
