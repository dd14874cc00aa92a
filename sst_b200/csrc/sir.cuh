// SIRLayer pieces shared by the forward (sir.cu) and the training backward (sir_train.cu).
#pragma once
#include "index.cuh"

// relation-MLP parameters as the warp-per-point kernels read them
struct RelDev {
  int cin, n_rel, dims[4], rel_in, act;
  float eps, inv_norm[3], rel_dist_scaler;
  const float *w[4], *g[4], *b[4];
};

#define REL_MAXC 8  // channels per lane (Cin <= 256)

__device__ __forceinline__ float act_fn(float x, int act) { return act == 2 ? gelu_erf(x) : fmaxf(x, 0.f); }

// What sstb200_sir_layer_forward_train keeps for the backward, carved out of the caller's state buffer: the pre-LayerNorm
// values of both VFE layers and the row that attains each group max (lowest point index on ties).  x0, the rel-MLP and p0 are
// recomputed by the backward.
struct SirState {
  float* t0;       // [N, C0]
  float* t1;       // [N, C1] (C1 > 0)
  long long* am0;  // [G, C0]
  long long* am1;  // [G, C1] (C1 > 0)
};
static inline void sir_state_carve(Carve& cv, SirState& s, int N, int G, int C0, int C1) {
  s.t0 = cv.take<float>((size_t)N * C0);
  s.t1 = C1 ? cv.take<float>((size_t)N * C1) : nullptr;
  s.am0 = cv.take<long long>((size_t)G * C0);
  s.am1 = C1 ? cv.take<long long>((size_t)G * C1) : nullptr;
}
static inline size_t sir_state_bytes(int N, int G, int C0, int C1) {
  return carve_bytes([&](Carve& cv) {
    SirState s;
    sir_state_carve(cv, s, N, G, C0, C1);
  });
}

// fills `rd` from the layer and checks the rel-MLP (SSTB_OK or an error code with the message set); *smem = its weight bytes
int sstb_sir_rel_dev(sstb200_ctx* c, const sstb200_sir_layer* L, RelDev* rd, size_t* smem);
// x0 = [xyz / xyz_normalizer || rest] * rel_mlp(f_cluster / rel_dist_scaler)   [N, cin]
int sstb_sir_rel_gate(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster, int N, float* x0);
// group CSR (offsets [G+1] int32 in csr.offsets, order [N] int32 in csr.order) of the points grouped by `inv`, as sstb200_group_csr
// builds it: carve, then build
struct SirGroupCsr {
  int32_t* count;  // [G + 2]: per-group counts, then an error flag
  Csr csr;
};
void sstb_sir_group_csr_carve(Carve& cv, SirGroupCsr& g, int N, int G);
int sstb_sir_group_csr(sstb200_ctx* c, SirGroupCsr& g, const long long* inv, int N, int G);
// the range the fp32 training path covers (SSTB_ERR_UNSUPPORTED / SSTB_ERR_ARG with a message otherwise)
int sstb_sir_train_check(sstb200_ctx* c, const sstb200_sir_layer* L);
// out[g, col0 + c] = the group max that ord[g, c] holds in order-preserving form (0, an empty group, gives 0)
void sstb_sir_segmax_finalize(cudaStream_t st, const uint32_t* ord, int G, int C, float* out, int ldo, int col0);
