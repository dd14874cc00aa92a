// 16-bit tensor-core path of the SRA encoder layer (precision 'bf16' of the API; operands are IEEE fp16 - same tensor
// throughput, 8x smaller operand rounding than bf16, and the reference's own mixed-precision setting is fp16,
// configs/sst_refactor/sst_waymoD5_1x_3class_8heads_v2.py:82): wgmma GEMMs with fp32 accumulators.
//
// Per layer: the QKV projection (generic GEMM kernel of csrc/wgmma_gemm.cuh: C[128-row tile, NT] = A[128, K] . W[NT, K]^T,
// A converted on the fly from fp32 rows + positional embedding, fp16 q|k|v out), the ragged window attention, and the fused
// post-attention chain of csrc/sra_chain2.cu (out-projection + LN1 + FFN + LN2, in the encoder stack also the next layer's
// QKV), so the stack takes 2 launches per layer.  fp32 stays the type of the residual stream, softmax, LayerNorm and all
// accumulation.
//
// Range: every 16-bit operand is IEEE fp16, largest finite value 65504.  A q|k operand x + pos, a v operand x, or an
// activation x1, h, y beyond it rounds to inf and the layer's output is no longer finite; inputs stay well inside it in the
// models this path serves (normalised residual streams), and nothing here rescales them.
#include <stdarg.h>
#include <cuda_fp16.h>
#include "sra.cuh"
#include "sra_attn.cuh"
#include "wgmma.cuh"
#include "wgmma_gemm.cuh"

namespace {

// QKV projection of a layer: q,k from fp16(x + pos), v from fp16(x); EPI_F16 writes fp16 rows for the tensor-core attention
int qkv_gemm(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x, __half* qkv, int n_cap,
             const int32_t* n_dev, bool f16_out) {
  const int d = L->d_model;
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.M_cap = n_cap;
  g.M_dev = n_dev;
  g.A = x;
  g.lda = d;
  g.W = L->in_proj_w_f16;
  g.bias = L->in_proj_b;
  g.pos_tab = P->pos_table;
  g.pos_code = P->pos_code;
  g.posL = P->pos_L;
  g.pos_maxw = P->pos_maxw;
  g.pos_ndim = P->pos_ndim;
  g.pos_ntiles = 2;
  g.out_h16 = qkv;
  g.ldo = 3 * d;
  g.out_row_map = nullptr;  // q|k|v, att and the residual stream all live in flat token order; attention gathers its windows
  return f16_out ? launch_wgmma_gemm<128, 128, PRO_F32, EPI_F16>(c, g, 3) : launch_wgmma_gemm<128, 128, PRO_F32, EPI_H16>(c, g, 3);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
int sstb_sra_layer_bf16(sstb200_ctx* c, const sstb200_sra_layer* L, const sstb200_sra_plan* P, const float* x, float* y,
                        int n_cap, const int32_t* n_dev) {
  const int d = L->d_model, ff = L->dim_ff;
  if (d != 128 || ff != 256 || !L->post_norm || L->norm1_mean || L->act != 2)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED,
                     "bf16 tensor-core path is built for d_model=128, dim_ff=256, post-norm LayerNorm, gelu (got d=%d ff=%d, %s, %s; "
                     "BatchNorm runs in the fused stack only)",
                     d, ff, !L->post_norm ? "pre-norm" : L->norm1_mean ? "post-norm BatchNorm" : "post-norm LayerNorm",
                     L->act == 2 ? "gelu" : "relu");
  if (!L->in_proj_w_f16 || !L->out_proj_w_f16 || !L->lin1_w_f16 || !L->lin2_w_f16)
    return sstb_fail(c, SSTB_ERR_ARG, "the tensor-core path needs the *_w_f16 weight copies");
  if (P->pos_table && P->pos_L % 8 != 0)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "bf16 path needs the per-axis positional length (%d) to be a multiple of 8", P->pos_L);
  __half *qkv, *att;
  int rc = arena_carve(c, [&](Carve& cv) {
    qkv = cv.take<__half>((size_t)n_cap * 3 * d);
    att = cv.take<__half>((size_t)n_cap * d);
  });
  if (rc) return rc;
  // tensor-core attention path: plain scaled-dot-product, 8 heads x 16, windows <= 144 tokens
  const bool tc_attn = L->nhead == 8 && (!L->tau || L->tau_n == 1 || L->tau_n == 8) && P->max_window_tokens > 0 && P->max_window_tokens <= ATT_MAXT &&
                       P->num_windows_dev && P->win_batch;
  // 1. QKV projection, fp16 q/k/v for either attention kernel (softmax logits need the mantissa: with bf16 q,k the logit error
  // would dominate the layer's error budget).
  rc = qkv_gemm(c, L, P, x, qkv, n_cap, n_dev, tc_attn);
  if (rc) return rc;
  // 2. ragged window attention (fp32 math on bf16 q/k/v)
  if (tc_attn)
    rc = sstb_win_attn_batch(c, qkv, P->num_windows_dev, P->win_offsets, P->win_batch, n_cap, P->tok_perm, att, false, L->tau, L->tau_n, L->tau_min);
  else  // cosine attention / unbounded windows: SIMT kernel on the bf16 operands
    rc = sstb_win_attn<__half, __half>(c, qkv, d, L->nhead, n_cap, n_dev, P->win_offsets, P->tok_perm, P->tok_win,
                                                     L->tau, L->tau_n, L->tau_min, att);
  if (rc) return rc;
  // 3-5 fused: out-projection + LN1 + FFN1 + GELU + FFN2 + LN2
  return sstb_sra_chain2(c, L, att, x, y, n_cap, n_dev);
}


// ------------------------------------------------------------------------------------------------
// whole encoder stack, bf16 tensor-core path: QKV(0) -> [attention(l) -> chain(l) (+ QKV(l+1) fused)] x L
// 2 launches per layer; q/k/v, attention output and the residual stream stay in flat token order throughout.
// ------------------------------------------------------------------------------------------------
static bool layer_supported_tc(const sstb200_sra_layer* L, const sstb200_sra_plan* P) {
  // LayerNorm or eval-mode BatchNorm (use_bn), plain or cosine attention (tau per layer or per head)
  return L->d_model == 128 && L->dim_ff == 256 && L->post_norm && L->act == 2 && L->nhead == 8 && (!L->tau || L->tau_n == 1 || L->tau_n == 8) &&
         (!L->norm1_mean || (L->norm1_var && L->norm2_mean && L->norm2_var)) &&
         L->in_proj_w_f16 && L->out_proj_w_f16 && L->lin1_w_f16 && L->lin2_w_f16 && P->max_window_tokens > 0 &&
         P->max_window_tokens <= ATT_MAXT && P->num_windows_dev && P->win_batch && P->pos_table && P->pos_code && P->pos_L % 32 == 0 &&
         P->pos_ndim >= 1 && P->pos_ndim <= 3 && P->pos_ndim * P->pos_maxw <= 32 && P->pos_ndim * P->pos_L <= 128;
}

int sstb_sra_stack_bf16(sstb200_ctx* c, const sstb200_sra_layer* layers, int num_layers, const sstb200_sra_plan* plans, const float* x,
                        float* y, float* scratch, int n_cap, const int32_t* n_dev) {
  (void)scratch;
  for (int l = 0; l < num_layers; l++)
    if (!layer_supported_tc(&layers[l], &plans[l & 1])) return SSTB_ERR_UNSUPPORTED;  // caller falls back to per-layer calls
  const int d = 128;
  if (num_layers > SSTB_MAX_STACK) return SSTB_ERR_UNSUPPORTED;
  bool any_bn = false;
  for (int l = 0; l < num_layers; l++) any_bn |= layers[l].norm1_mean != nullptr;
  __half *qkv, *att;
  float* bn_fold = nullptr;
  int rc = arena_carve(c, [&](Carve& cv) {
    qkv = cv.take<__half>((size_t)n_cap * 3 * d);
    att = cv.take<__half>((size_t)n_cap * d);
    if (any_bn) bn_fold = cv.take<float>((size_t)num_layers * 4 * 128);
  });
  if (rc) return rc;
  if (any_bn && (rc = sstb_sra_bn_fold(c, layers, num_layers, bn_fold))) return rc;
  rc = qkv_gemm(c, &layers[0], &plans[0], x, qkv, n_cap, n_dev, true);
  if (rc) return rc;
  const float* xin = x;
  for (int l = 0; l < num_layers; l++) {
    const sstb200_sra_plan* P = &plans[l & 1];
    rc = sstb_win_attn_batch(c, qkv, P->num_windows_dev, P->win_offsets, P->win_batch, n_cap, P->tok_perm, att, false, layers[l].tau,
                             layers[l].tau_n, layers[l].tau_min);
    if (rc) return rc;
    const bool has_next = l + 1 < num_layers;
    // the chain reads the residual rows of a tile before it writes the same rows of y: in-place (xin == y) is safe
    rc = sstb_sra_chain2(c, &layers[l], att, xin, y, n_cap, n_dev, has_next ? &layers[l + 1] : nullptr,
                         has_next ? &plans[(l + 1) & 1] : nullptr, has_next ? qkv : nullptr,
                         layers[l].norm1_mean ? bn_fold + (size_t)l * 4 * 128 : nullptr);
    if (rc) return rc;
    xin = y;
  }
  return SSTB_OK;
}
