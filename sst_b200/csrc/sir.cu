// SIRLayer forward (S1-S3): FSD's segmented point-group MLP + max-pool
// (mmdet3d/models/voxel_encoders/voxel_encoder.py:617-764, build_mlp ops/sst/sst_ops.py:334-361).
//
//   rel   = MLP_rel(f_cluster / rel_dist_scaler)                 3 -> 16 -> 32 -> Cin   (Linear_nobias + LN + act)
//   x0    = [xyz / xyz_normalizer || feats] * rel                [N, Cin]
//   p0    = act(LN(W0 x0))        g0 = segmax(p0)                [N, C0], [G, C0]
//   p1    = act(LN(W1a p0 + (W1b g0)[group]))   g1 = segmax(p1)  ([p0 || g0[group]] never materialised)
//   out   = p1 (+ shortcut when shapes match), group feats [g0 || g1]
//
// The reference runs this as ~25 ATen/torch_scatter launches per block with [N,256] concat tensors and float
// atomics.  Here: one warp-per-point kernel for the relation MLP + gating, FFMA row GEMMs with fused LN/act,
// and a sorted segmented max (CSR order, in-tile reduce, order-preserving atomicMax only at tile edges).
//
// Training (sstb200_sir_layer_forward_train) runs this same fp32 forward; it writes the pre-LN values to the caller's state and
// takes each group max with its arg-max row (launch_segment_reduce) - the backward is in sir_train.cu.
#include <stdarg.h>
#include "index.cuh"
#include "rows.cuh"
#include "sir.cuh"

// ---- relation MLP + gating: one warp per point -----------------------------------------------------
__global__ void __launch_bounds__(256) sir_rel_gate_kernel(RelDev r, const float* __restrict__ feats /*[N,cin]*/,
                                                           const float* __restrict__ f_cluster /*[N,3]*/, int N,
                                                           float* __restrict__ x0 /*[N,cin]*/) {
  pdl_wait();
  pdl_launch();
  extern __shared__ float sw[];  // transposed weights: layer l stored [in_l][out_l]
  float* wl[4];
  {
    float* p = sw;
    int in = r.rel_in;
    for (int l = 0; l < r.n_rel; l++) {
      wl[l] = p;
      for (int i = threadIdx.x; i < in * r.dims[l]; i += blockDim.x) {
        int k = i / r.dims[l], c = i % r.dims[l];
        p[i] = r.w[l][(size_t)c * in + k];
      }
      p += in * r.dims[l];
      in = r.dims[l];
    }
  }
  __syncthreads();
  int ln = lane_id();
  int warps = (gridDim.x * blockDim.x) >> 5;
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < N; p += warps) {
    // input: f_cluster / scaler (3 values, lanes 0..2)
    float cur[REL_MAXC];
#pragma unroll
    for (int j = 0; j < REL_MAXC; j++) cur[j] = 0.f;
    if (ln < r.rel_in) cur[0] = f_cluster[(size_t)p * r.rel_in + ln] / r.rel_dist_scaler;
    int in = r.rel_in;
    for (int l = 0; l < r.n_rel; l++) {
      int out = r.dims[l];
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
      // LayerNorm over `out` channels + activation
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < REL_MAXC; j++)
        if (ln + 32 * j < out) s += acc[j];
      float mean = warp_sum(s) / (float)out;
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < REL_MAXC; j++)
        if (ln + 32 * j < out) {
          float t = acc[j] - mean;
          q += t * t;
        }
      float rstd = rsqrtf(warp_sum(q) / (float)out + r.eps);
#pragma unroll
      for (int j = 0; j < REL_MAXC; j++) {
        int c = ln + 32 * j;
        cur[j] = c < out ? act_fn((acc[j] - mean) * rstd * r.g[l][c] + r.b[l][c], r.act) : 0.f;
      }
      in = out;
    }
    // gate: x0 = [xyz / normalizer || rest] * rel
#pragma unroll
    for (int j = 0; j < REL_MAXC; j++) {
      int c = ln + 32 * j;
      if (c < r.cin) {
        float v = feats[(size_t)p * r.cin + c];
        if (c < 3) v = v / (c == 0 ? r.inv_norm[0] : (c == 1 ? r.inv_norm[1] : r.inv_norm[2]));
        x0[(size_t)p * r.cin + c] = v * cur[j];
      }
    }
  }
}

// ---- sorted segmented max: rows visited in CSR order, one thread per channel -----------------------------
__global__ void fill_u32_kernel(uint32_t* p, size_t n, uint32_t v) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
#define SEG_ROWS 64
__global__ void __launch_bounds__(128) segmax_sorted_kernel(const float* __restrict__ src, int C, const int32_t* __restrict__ order,
                                                            const long long* __restrict__ seg_of_row, int N,
                                                            uint32_t* __restrict__ out_ord /*[G, C] order-preserving uint*/) {
  pdl_wait();
  pdl_launch();
  __shared__ int s_row[SEG_ROWS];
  __shared__ int s_seg[SEG_ROWS];
  int k0 = blockIdx.x * SEG_ROWS;
  int nrow = min(SEG_ROWS, N - k0);
  for (int i = threadIdx.x; i < nrow; i += blockDim.x) {
    int row = order[k0 + i];
    s_row[i] = row;
    s_seg[i] = (int)seg_of_row[row];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float m = -INFINITY;
    int seg = s_seg[0];
    for (int i = 0; i < nrow; i++) {
      int sg = s_seg[i];
      if (sg != seg) {
        atomicMax(&out_ord[(size_t)seg * C + c], f2ord(m));
        seg = sg;
        m = -INFINITY;
      }
      m = fmaxf(m, src[(size_t)s_row[i] * C + c]);
    }
    atomicMax(&out_ord[(size_t)seg * C + c], f2ord(m));
  }
}
__global__ void segmax_finalize_kernel(const uint32_t* __restrict__ ord, int G, int C, float* __restrict__ out, int ldo, int col0) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * C) return;
  int g = (int)(i / C), c = (int)(i % C);
  uint32_t u = ord[i];
  out[(size_t)g * ldo + col0 + c] = (u == 0u) ? 0.f : ord2f(u);  // empty segment -> 0 like torch_scatter
}

void sstb_sir_segmax_finalize(cudaStream_t st, const uint32_t* ord, int G, int C, float* out, int ldo, int col0) {
  size_t gn = (size_t)G * C;
  launch_pdl(segmax_finalize_kernel, dim3((unsigned)((gn + 255) / 256)), dim3(256), (size_t)(0), st, ord, G, C, out, ldo, col0);
}

// with_shortcut (voxel_encoder.py:753-759): point_feats += features[:, 3:] when the shapes agree
__global__ void shortcut_kernel(float* __restrict__ out, const float* __restrict__ in_feats, int N, int C, int cin) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)N * C) return;
  int p = (int)(i / C), ch = (int)(i % C);
  out[i] += in_feats[(size_t)p * cin + 3 + ch];
}

// Group CSR: points grouped by `inv`; shared by every block of a SIR backbone.  csr.offsets / csr.order set before the carve are
// the caller's own buffers.
void sstb_sir_group_csr_carve(Carve& cv, SirGroupCsr& g, int N, int G) {
  g.count = cv.take<int32_t>((size_t)G + 2);
  csr_carve(cv, g.csr, N, G);
}

int sstb_sir_group_csr(sstb200_ctx* c, SirGroupCsr& g, const long long* inv, int N, int G) {
  cudaStream_t st = c->stream;
  int32_t* count = g.count;
  CUDA_TRY(c, cudaMemsetAsync(count, 0, ((size_t)G + 2) * 4, st));
  const bool small = G <= CSR_SMALL_MAX;
  if (small)
    launch_pdl(count_small_kernel<long long>, dim3((N + CSR_SMALL_ITEMS - 1) / CSR_SMALL_ITEMS), dim3(1024), (size_t)G * 4, st, inv, N, G, count, count + G + 1);
  else
    launch_pdl(count_index_kernel, dim3((N + 255) / 256), dim3(256), (size_t)(0), st, inv, N, G, count, count + G + 1);
  int rc = csr_build<long long>(c, g.csr, inv, N, count, G, nullptr, nullptr, small ? G : 0);
  if (rc) return rc;
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_group_csr(sstb200_ctx* c, const int64_t* inv, int N, int G, int32_t* offsets, int32_t* order) {
  CHECK_ARG(c, c && N >= 0 && G >= 0);
  if (N == 0 || G == 0) return SSTB_OK;
  CHECK_ARG(c, inv && offsets && order);
  arena_reset(c);
  SirGroupCsr g;
  g.csr.offsets = (uint32_t*)offsets;
  g.csr.order = order;
  int rc = arena_carve(c, [&](Carve& cv) { sstb_sir_group_csr_carve(cv, g, N, G); });
  if (rc) return rc;
  return sstb_sir_group_csr(c, g, (const long long*)inv, N, G);
}

int sstb_sir_rel_dev(sstb200_ctx* c, const sstb200_sir_layer* L, RelDev* rd, size_t* smem_out) {
  if (L->num_rel <= 0) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer without rel-MLP is not built");
  rd->cin = L->in_channels;
  rd->n_rel = L->num_rel;
  rd->rel_in = L->rel_in;
  rd->act = L->act;
  rd->eps = L->norm_eps;
  rd->rel_dist_scaler = L->rel_dist_scaler;
  size_t smem = 0;
  int in = L->rel_in;
  for (int l = 0; l < 4; l++) {
    rd->dims[l] = l < L->num_rel ? L->rel_dims[l] : 0;
    rd->w[l] = L->rel_w[l];
    rd->g[l] = L->rel_ln_w[l];
    rd->b[l] = L->rel_ln_b[l];
    if (l < L->num_rel) {
      CHECK_ARG(c, rd->w[l] && rd->g[l] && rd->b[l]);
      smem += (size_t)in * rd->dims[l] * 4;
      in = rd->dims[l];
    }
  }
  for (int i = 0; i < 3; i++) rd->inv_norm[i] = L->xyz_normalizer[i];
  if (smem > 200 * 1024) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "rel-MLP weights do not fit shared memory");
  *smem_out = smem;
  return SSTB_OK;
}

int sstb_sir_rel_gate(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster, int N, float* x0) {
  RelDev rd;
  size_t smem = 0;
  int rc = sstb_sir_rel_dev(c, L, &rd, &smem);
  if (rc) return rc;
  static SmemAttr sa;
  CUDA_TRY(c, ensure_smem(c, sa, sir_rel_gate_kernel, (size_t)200 * 1024));
  launch_pdl(sir_rel_gate_kernel, dim3(c->num_sms * 4), dim3(256), (size_t)(smem), c->stream, rd, in_feats, f_cluster, N, x0);
  return SSTB_OK;
}

// [G, C] dense -> columns col0.. of out [G, ldo]
__global__ void copy_cols_kernel(const float* __restrict__ src, int G, int C, float* __restrict__ out, int ldo, int col0) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)G * C) return;
  out[(i / C) * ldo + col0 + i % C] = src[i];
}

// Group max of src [N, C] into columns col0.. of out_group.  Eval: sorted max kernels (no arg-max).  Training (am != NULL): the
// segmented reduce with its arg-max (lowest point index attaining the max) through the dense [G, C] scratch gtmp.
static void sir_group_max(sstb200_ctx* c, const float* src, int C, const int32_t* off, const int32_t* order, const long long* inv, int N, int G,
                          uint32_t* gord, float* gtmp, long long* am, float* out_group, int Cg, int col0) {
  cudaStream_t st = c->stream;
  size_t gn = (size_t)G * C;
  if (am) {
    launch_segment_reduce(c, src, C, (const uint32_t*)off, order, G, nullptr, SSTB200_REDUCE_MAX, 0.f, gtmp, am, N);
    launch_pdl(copy_cols_kernel, dim3((unsigned)((gn + 255) / 256)), dim3(256), (size_t)(0), st, (const float*)gtmp, G, C, out_group, Cg, col0);
    return;
  }
  launch_pdl(fill_u32_kernel, dim3((unsigned)((gn + 255) / 256)), dim3(256), (size_t)(0), st, gord, gn, 0u);
  launch_pdl(segmax_sorted_kernel, dim3((N + SEG_ROWS - 1) / SEG_ROWS), dim3(128), (size_t)(0), st, src, C, order, inv, N, gord);
  launch_pdl(segmax_finalize_kernel, dim3((unsigned)((gn + 255) / 256)), dim3(256), (size_t)(0), st, (const uint32_t*)gord, G, C, out_group, Cg, col0);
}

// scratch of the fp32 forward; t (the pre-LayerNorm values) only in eval, training keeps them in the state
struct SirFp32Ws {
  float *x0, *t, *p0;
};
static void sir_fp32_carve(Carve& cv, SirFp32Ws& w, int N, int cin, int Cmax, bool train) {
  w.x0 = cv.take<float>((size_t)N * cin);
  w.t = train ? nullptr : cv.take<float>((size_t)N * Cmax);
  w.p0 = cv.take<float>((size_t)N * Cmax);
}

// The fp32 forward.  s == NULL: eval.  s != NULL: training - t0 / t1 land in the state, the group maxima record their arg-max
// rows there (off = the group CSR offsets), everything else is the same launch sequence.
static int sir_forward_fp32(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster, const long long* inv,
                            int N, int G, const int32_t* off, const int32_t* order, uint32_t* gord, float* gterm, const SirFp32Ws& w,
                            float* out_point, float* out_group, const SirState* s) {
  cudaStream_t st = c->stream;
  const int cin = L->in_channels, C0 = L->feat_channels[0], C1 = L->num_vfe > 1 ? L->feat_channels[1] : 0;
  float *x0 = w.x0, *t = w.t, *p0 = w.p0;
  float* t0 = s ? s->t0 : t;
  float* t1 = s ? s->t1 : t;

  // 1. relation MLP + gating
  int rc = sstb_sir_rel_gate(c, L, in_feats, f_cluster, N, x0);
  if (rc) return rc;
  // 2. layer 0: p0 = act(LN(W0 x0)); g0 = segmax(p0)
  CHECK_ARG(c, L->vfe_w[0] && L->vfe_ln_w[0] && L->vfe_ln_b[0]);
  RowGemm g0{};
  g0.A = x0, g0.lda = cin, g0.W = L->vfe_w[0], g0.out = t0, g0.ldo = C0, g0.M_cap = N, g0.N = C0, g0.K = cin;
  sstb_row_gemm(st, g0);
  float* p0out = (C1 == 0) ? out_point : p0;
  sstb_add_norm_act(st, t0, nullptr, L->vfe_ln_w[0], L->vfe_ln_b[0], nullptr, nullptr, L->norm_eps, p0out, N, nullptr, C0, L->act);
  const int Cg = C0 + C1;
  sir_group_max(c, p0out, C0, off, order, inv, N, G, gord, gterm, s ? s->am0 : nullptr, out_group, Cg, 0);
  if (C1) {
    CHECK_ARG(c, L->vfe_w[1] && L->vfe_ln_w[1] && L->vfe_ln_b[1]);
    // 3. layer 1 on [p0 || g0[group]]:  W1a p0 + (W1b g0)[group]
    RowGemm gw{}, pw{};
    gw.A = out_group, gw.lda = Cg, gw.W = L->vfe_w[1] + C0, gw.ldw = 2 * C0, gw.out = gterm, gw.ldo = C1, gw.M_cap = G, gw.N = C1, gw.K = C0;
    sstb_row_gemm(st, gw);
    pw.A = p0, pw.lda = C0, pw.W = L->vfe_w[1], pw.ldw = 2 * C0, pw.res = gterm, pw.ldr = C1, pw.res_index = inv, pw.out = t1, pw.ldo = C1;
    pw.M_cap = N, pw.N = C1, pw.K = C0;
    sstb_row_gemm(st, pw);
    sstb_add_norm_act(st, t1, nullptr, L->vfe_ln_w[1], L->vfe_ln_b[1], nullptr, nullptr, L->norm_eps, out_point, N, nullptr, C1, L->act);
    sir_group_max(c, out_point, C1, off, order, inv, N, G, gord, gterm, s ? s->am1 : nullptr, out_group, Cg, C0);
  }
  {
    int Cl = C1 ? C1 : C0;
    if (L->with_shortcut && cin - 3 == Cl)
      launch_pdl(shortcut_kernel, dim3((unsigned)(((size_t)N * Cl + 255) / 256)), dim3(256), (size_t)(0), st, out_point, in_feats, N, Cl, cin);
  }
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

int sstb_sir_train_check(sstb200_ctx* c, const sstb200_sir_layer* L) {
  CHECK_ARG(c, L->num_vfe >= 1 && L->num_vfe <= 2 && L->num_rel >= 0 && L->num_rel <= 4 && (L->act == 1 || L->act == 2));
  if (!L->mode_max) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer training: only mode='max' is built");
  if (L->num_rel == 0) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer training: a layer without rel-MLP is not built");
  const int cin = L->in_channels, C0 = L->feat_channels[0], C1 = L->num_vfe > 1 ? L->feat_channels[1] : 0;
  if (cin < 3 || cin > 32 * REL_MAXC || C0 <= 0 || C0 > 256 || C1 > 256 || C0 % 32 || C1 % 32)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer training: dims (cin=%d, C0=%d, C1=%d) not supported", cin, C0, C1);
  if (L->rel_in < 1 || L->rel_in > 32) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer training: rel_mlp_in_channel %d (1..32)", L->rel_in);
  for (int l = 0; l < L->num_rel; l++)
    if (L->rel_dims[l] < 1 || L->rel_dims[l] > 32 * REL_MAXC)
      return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer training: rel-MLP width %d", L->rel_dims[l]);
  if (L->rel_dims[L->num_rel - 1] != cin) return sstb_fail(c, SSTB_ERR_ARG, "last rel-MLP layer must produce in_channels");
  return SSTB_OK;
}

extern "C" size_t sstb200_sir_layer_train_state_bytes(const sstb200_sir_layer* L, int N, int G) {
  if (!L || N < 0 || G < 0 || L->num_vfe < 1 || L->num_vfe > 2) return 0;
  return sir_state_bytes(N, G, L->feat_channels[0], L->num_vfe > 1 ? L->feat_channels[1] : 0);
}

extern "C" int sstb200_sir_layer_forward_train(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster,
                                               const int64_t* inv, int N, int G, const int32_t* csr_offsets, const int32_t* csr_order,
                                               float* out_point, float* out_group, void* state, size_t state_bytes) {
  CHECK_ARG(c, c && L && N >= 0 && G >= 0);
  int rc = sstb_sir_train_check(c, L);
  if (rc) return rc;
  if (N == 0 || G == 0) return SSTB_OK;
  CHECK_ARG(c, in_feats && f_cluster && inv && out_point && out_group && state);
  CHECK_ARG(c, (csr_offsets == nullptr) == (csr_order == nullptr));
  const int cin = L->in_channels, C0 = L->feat_channels[0], C1 = L->num_vfe > 1 ? L->feat_channels[1] : 0;
  const int Cmax = C0 > C1 ? C0 : C1;
  const size_t need = sir_state_bytes(N, G, C0, C1);
  if (state_bytes < need)
    return sstb_fail(c, SSTB_ERR_WORKSPACE, "SIRLayer training state: %zu bytes given, %zu needed", state_bytes, need);
  SirState s;
  Carve sc{(char*)state, 0};
  sir_state_carve(sc, s, N, G, C0, C1);
  arena_reset(c);
  SirGroupCsr gc;
  uint32_t* gord;
  float* gterm;
  SirFp32Ws w;
  rc = arena_carve(c, [&](Carve& cv) {
    if (!csr_order) sstb_sir_group_csr_carve(cv, gc, N, G);
    gord = cv.take<uint32_t>((size_t)G * Cmax);
    gterm = cv.take<float>((size_t)G * Cmax);
    sir_fp32_carve(cv, w, N, cin, Cmax, true);
  });
  if (rc) return rc;
  const int32_t *off = csr_offsets, *order = csr_order;
  if (!order) {
    if ((rc = sstb_sir_group_csr(c, gc, (const long long*)inv, N, G))) return rc;
    off = (const int32_t*)gc.csr.offsets;
    order = gc.csr.order;
  }
  return sir_forward_fp32(c, L, in_feats, f_cluster, (const long long*)inv, N, G, off, order, gord, gterm, w, out_point, out_group, &s);
}

int sstb_sir_layer_bf16(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster, const long long* inv,
                        const int32_t* order, int N, int G, __nv_bfloat16* p0buf, uint32_t* gord, float* gterm, float* out_point, int ldo,
                        float* out_group, int in_ld, int gap_at, int gap);

extern "C" int sstb200_sir_layer_forward_ex(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, int in_ld, int in_gap_at,
                                            int in_gap, const float* f_cluster, const int64_t* inv, int N, int G,
                                            const int32_t* csr_offsets, const int32_t* csr_order, int precision, float* out_point,
                                            int out_point_ld, float* out_group) {
  CHECK_ARG(c, c && L && N >= 0 && G >= 0);
  if (N == 0 || G == 0) return SSTB_OK;
  CHECK_ARG(c, in_feats && f_cluster && inv && out_point && out_group);
  CHECK_ARG(c, (csr_offsets == nullptr) == (csr_order == nullptr));
  CHECK_ARG(c, precision == SSTB200_PREC_FP32 || precision == SSTB200_PREC_BF16);
  CHECK_ARG(c, L->num_vfe >= 1 && L->num_vfe <= 2 && L->num_rel >= 0 && L->num_rel <= 4 && (L->act == 1 || L->act == 2));
  if (!L->mode_max) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer: only mode='max' is built");
  const int cin = L->in_channels, C0 = L->feat_channels[0], C1 = L->num_vfe > 1 ? L->feat_channels[1] : 0;
  const int Clast = C1 ? C1 : C0;
  if (out_point_ld <= 0) out_point_ld = Clast;
  CHECK_ARG(c, out_point_ld >= Clast);
  if (cin > 32 * REL_MAXC || C0 > 256 || C1 > 256 || C0 % 32 || C1 % 32)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIR dims (cin=%d, C0=%d, C1=%d) not supported", cin, C0, C1);
  if (L->num_rel > 0 && L->rel_dims[L->num_rel - 1] != cin) return sstb_fail(c, SSTB_ERR_ARG, "last rel-MLP layer must produce in_channels");
  for (int l = 0; l < L->num_rel; l++)
    if (L->rel_dims[l] > 32 * REL_MAXC) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "rel-MLP width %d", L->rel_dims[l]);
  const int Cmax = C0 > C1 ? C0 : C1;
  const bool bf16 = precision == SSTB200_PREC_BF16;
  if (in_ld <= 0) in_ld = cin, in_gap_at = cin, in_gap = 0;
  CHECK_ARG(c, in_gap >= 0 && in_gap_at >= 0 && in_gap_at <= cin && in_ld >= cin + in_gap);
  if (!bf16 && (out_point_ld != Clast || in_ld != cin || in_gap != 0))
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer fp32 path works on dense point features (ld == C, no gap)");
  // kernel B of the bf16 path reads the pooled layer-0 features back from out_group as float4
  if (bf16) CHECK_ARG(c, ((uintptr_t)out_group & 15) == 0);
  arena_reset(c);
  SirGroupCsr gc;
  uint32_t* gord;
  float* gterm;
  __nv_bfloat16* p0buf = nullptr;
  SirFp32Ws w;
  int rc = arena_carve(c, [&](Carve& cv) {
    if (!csr_order) sstb_sir_group_csr_carve(cv, gc, N, G);
    gord = cv.take<uint32_t>((size_t)G * Cmax);
    gterm = cv.take<float>((size_t)G * Cmax);
    if (bf16) p0buf = cv.take<__nv_bfloat16>(((size_t)N + 128) * 128);
    else sir_fp32_carve(cv, w, N, cin, Cmax, false);
  });
  if (rc) return rc;
  cudaStream_t st = c->stream;
  const int32_t* order = csr_order;
  if (!order) {
    if ((rc = sstb_sir_group_csr(c, gc, (const long long*)inv, N, G))) return rc;
    order = gc.csr.order;
  }
  if (bf16) {
    rc = sstb_sir_layer_bf16(c, L, in_feats, f_cluster, (const long long*)inv, order, N, G, p0buf, gord, gterm, out_point, out_point_ld, out_group, in_ld, in_gap_at,
                             in_gap);
    if (rc) return rc;
    if (L->with_shortcut && cin - 3 == Clast) {
      if (out_point_ld != Clast || in_ld != cin) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "shortcut with strided point features");
      launch_pdl(shortcut_kernel, dim3((unsigned)(((size_t)N * Clast + 255) / 256)), dim3(256), (size_t)(0), st, out_point, in_feats, N, Clast, cin);
    }
    LAUNCH_CHECK(c);
    return SSTB_OK;
  }
  return sir_forward_fp32(c, L, in_feats, f_cluster, (const long long*)inv, N, G, nullptr, order, gord, gterm, w, out_point, out_group, nullptr);
}

extern "C" int sstb200_sir_layer_forward(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster,
                                         const int64_t* inv, int N, int G, float* out_point, float* out_group) {
  return sstb200_sir_layer_forward_ex(c, L, in_feats, 0, 0, 0, f_cluster, inv, N, G, nullptr, nullptr, SSTB200_PREC_FP32, out_point, 0, out_group);
}
