// SIRLayer on the tensor cores (precision = BF16): two persistent wgmma kernels per layer, tiles of 128 points taken in
// group (CSR) order so that the segmented max-pool is an in-tile scan with a handful of atomics per tile.
//   models/voxel_encoders/voxel_encoder.py:696-764 (SIRLayer.forward), ops/sst/sst_ops.py:334-361 (build_mlp)
//
//   kernel A (per tile):  rel-MLP layers 1,2 in registers (thread per point)            3 -> R1 -> R2, LN + act each
//                         rel-MLP layer 3 as wgmma [128,R2] x [cin,R2]^T               LN + act in the epilogue,
//                         x0 = [xyz/normalizer || feats] * rel  -> bf16 A operand       (gating fused into that epilogue)
//                         layer 0 as wgmma [128,KP] x [128,KP]^T                         LN + act -> p0 (bf16, CSR order) + segmax g0
//   kernel B (per tile):  layer 1 as wgmma [128,256] x [128,256]^T on [p0 || g0[group]] LN + act -> out (fp32, original point
//                         (the concat exists only inside the operand tile)               order) + segmax g1
// Operands are bf16 (fp32 accumulate); LayerNorm, activations, gating, pooling and every output stay fp32.  Each GEMM is split over
// the four warpgroups (row half x column half); the fragments meet the thread-per-row epilogues in a shared-memory accumulator tile.
// The [N, 2*C0] concat of the reference is never formed; weights are converted to bf16 operands once per CTA.
#include <stdarg.h>
#include "index.cuh"
#include "sir.cuh"
#include "wgmma.cuh"

namespace {

constexpr int ST = 128;   // points per tile
constexpr int SC = 128;   // C0 == C1 == 128 on this path

struct SirDev {
  int cin, rel_in, act;
  float eps, rel_dist_scaler, nz[3];
  const float *rw[3], *rg[3], *rb[3];  // rel-MLP: weights [out,in], LayerNorm weight / bias
  const float *w0, *g0, *b0;           // vfe layer 0: [SC, cin]
  const float *w1, *g1, *b1;           // vfe layer 1: [SC, 2*SC]
};

// GELU on the hardware tanh unit (MUFU.TANH): 0.5 x (1 + tanh(sqrt(2/pi) (x + 0.044715 x^3))), ~7 instructions.  Deviation from
// the exact erf form <= ~5e-4 absolute - an order of magnitude below this path's bf16-operand error (profiles: the erf
// forms cost 15-50 instructions per element and made these epilogues instruction-cache and issue bound).
__device__ __forceinline__ float gelu_as(float x) {
  float u = 0.7978845608028654f * fmaf(0.044715f * x, x * x, x);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(u));
  return 0.5f * x * (1.0f + t);
}
template <int ACT>
__device__ __forceinline__ float act_f(float x) { return ACT == 2 ? gelu_as(x) : fmaxf(x, 0.f); }

// fp32 weight block W[r, col0 + k] (r < nrows, k < ncols) -> bf16 wgmma operand (wgmma.cuh) of NR rows x KPAD columns
__device__ __forceinline__ void stage_weight(uint8_t* dst, int NR, int KPAD, const float* __restrict__ W, int ld, int col0, int nrows,
                                             int ncols) {
  const int pieces = NR * (KPAD / 8);
  for (int idx = threadIdx.x; idx < pieces; idx += blockDim.x) {
    const int r = idx / (KPAD / 8), j = idx % (KPAD / 8);
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
      int k = j * 8 + i;
      f[i] = (r < nrows && k < ncols) ? __ldg(W + (size_t)r * ld + col0 + k) : 0.f;
    }
    *reinterpret_cast<int4*>(dst + sw128_off(NR, r, j)) = pack8_h16<FMT_BF16>(f);
  }
}

// Segmented max of a warp's 32 rows x 32 columns held in registers (thread = row, v[i] = column col0 + i), rows sorted by
// group: per column one redux.sync on the order-preserving integer image of the float, then lane i issues the atomicMax of
// column i.  Warps whose rows all belong to one group (the common case: groups span several tiles) take one pass; otherwise
// one pass per distinct group present.  `seg` < 0 marks rows past the end.
__device__ __forceinline__ void warp_segmax_ord(const float* v, int seg, int col0, uint32_t* __restrict__ gord) {
  const int lane = threadIdx.x & 31;
  unsigned todo = __ballot_sync(0xffffffffu, seg >= 0);
  while (todo) {
    const int s = __shfl_sync(0xffffffffu, seg, __ffs(todo) - 1);
    const bool mine_seg = seg == s;
    todo &= ~__ballot_sync(0xffffffffu, mine_seg);
    uint32_t mine = 0;
#pragma unroll
    for (int i = 0; i < 32; i++) {
      uint32_t m = __reduce_max_sync(0xffffffffu, mine_seg ? f2ord(v[i]) : 0u);
      if (lane == i) mine = m;
    }
    atomicMax(&gord[(size_t)s * SC + col0 + lane], mine);
  }
}

template <int N>
__device__ __forceinline__ void ln_regs(float* v, float& mean, float& rstd, float eps) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N; i++) s += v[i];
  mean = s / (float)N;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < N; i++) {
    float t = v[i] - mean;
    q = fmaf(t, t, q);
  }
  rstd = rsqrtf(q / (float)N + eps);
}

// ------------------------------------------------------------------------------------------------------------------------
// kernel A.  512 threads = 16 warps: warp w owns tile rows 32*(w%4).. and column quarter w/4 in every epilogue,
// so 4 warps per scheduler hide the latency of the dependent LayerNorm / activation chains.
// ------------------------------------------------------------------------------------------------------------------------
constexpr int NT = 512;

// C[128, N] = A . B^T over KSTEPS K-steps of 16, warpgroup w: rows 64 (w & 1).., columns N/2 (w >> 1)..; result -> acc [128][N]
template <int N, int KSTEPS>
__device__ __forceinline__ void sir_gemm(uint32_t a, uint32_t a_cp, uint32_t b, uint32_t b_cp, float* acc, bool sync_operands) {
  const int w = threadIdx.x >> 7;
  float d[N / 4];
  wg_tile_mma<N / 2, true, KSTEPS>(d, a + (w & 1) * 64 * 128, a_cp, b + (w >> 1) * (N / 2) * 128, b_cp, false);
  wgmma_wait<0>();
  if (sync_operands) __syncthreads();   // acc aliases an operand: every warpgroup must be done reading it
  wg_store_acc<N / 2>(d, acc, N, (w & 1) * 64, (w >> 1) * (N / 2));
  __syncthreads();
}

template <int KP, int R1, int R2, int ACT>
__global__ void __launch_bounds__(NT, 1) sir_a_kernel(SirDev d, const float* __restrict__ in_feats, const float* __restrict__ f_cluster,
                                                      const long long* __restrict__ inv, const int32_t* __restrict__ order, int N,
                                                      __nv_bfloat16* __restrict__ p0buf, uint32_t* __restrict__ gord, int pitch_in, int in_ld, int gap_at,
                                                      int gap) {
  pdl_wait();
  pdl_launch();
  static_assert((KP == 128 || KP == 192) && R1 == 16 && R2 == 32, "shape");
  constexpr int NQC = KP / 4;  // columns per epilogue quarter (rel-MLP layer 3); layer 0 uses SC / 4 = 32
  extern __shared__ uint8_t sira_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)sira_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* sB0 = base;                          // W0  : KP/64 chunks x SC rows x 128 B
  uint8_t* sA0 = sB0 + (size_t)SC * KP * 2;     // x0  : KP/64 chunks x ST rows x 128 B
  uint8_t* sB3 = sA0 + (size_t)ST * KP * 2;     // Wr3 : 1 chunk x KP rows x 128 B (restaged every tile: the accumulators overwrite it)
  uint8_t* sA3 = sB3 + (size_t)KP * 128;        // r2  : 1 chunk x ST rows x 128 B
  float* sIn = reinterpret_cast<float*>(sA3 + (size_t)ST * 128);  // in_feats tile [ST][pitch_in], pitch odd (thread-per-row reads)
  // accumulator tiles, from sB3 on: rel layer 3 one column quarter at a time [ST][64] (inside Wr3 + r2), layer 0 [ST][SC] (Wr3 + r2 +
  // in_feats, all dead by then)
  float* sAcc = reinterpret_cast<float*>(sB3);
  __shared__ __align__(16) float sW1[R1 * 4], sW2[R2 * R1];
  __shared__ float sG1[R1], sBt1[R1], sG2[R2], sBt2[R2], sG3[KP], sBt3[KP], sG0[SC], sBt0[SC];
  __shared__ float redA[4][ST], redB[4][ST];
  __shared__ int sRowB[2][ST], sSegB[2][ST];  // double-buffered: the next tile's point / group ids are fetched during this tile
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntiles = (N + ST - 1) / ST;
  if ((int)blockIdx.x >= ntiles) return;
  const int cin = d.cin;
  for (int i = tid; i < R1 * 4; i += NT) sW1[i] = (i % 4) < d.rel_in ? d.rw[0][(i / 4) * d.rel_in + (i % 4)] : 0.f;
  for (int i = tid; i < R2 * R1; i += NT) sW2[i] = d.rw[1][i];
  for (int i = tid; i < R1; i += NT) sG1[i] = d.rg[0][i], sBt1[i] = d.rb[0][i];
  for (int i = tid; i < R2; i += NT) sG2[i] = d.rg[1][i], sBt2[i] = d.rb[1][i];
  for (int i = tid; i < KP; i += NT) sG3[i] = i < cin ? d.rg[2][i] : 0.f, sBt3[i] = i < cin ? d.rb[2][i] : 0.f;
  for (int i = tid; i < SC; i += NT) sG0[i] = d.g0[i], sBt0[i] = d.b0[i];
  stage_weight(sB0, SC, KP, d.w0, cin, 0, SC, cin);
  const int quarter = warp >> 2;
  const int lrow = (warp & 3) * 32 + lane;
  int cur = 0;
  if (tid < ST) {
    int k = blockIdx.x * ST + tid;
    int row = k < N ? order[k] : -1;
    sRowB[0][tid] = row;
    sSegB[0][tid] = row >= 0 ? (int)inv[row] : -1;
  }
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int k0 = tile * ST;
    const int nrow = min(ST, N - k0);
    const int* sRow = sRowB[cur];
    const int* sSeg = sSegB[cur];
    __syncthreads();  // previous tile fully consumed (sIn / operands / accumulators) and this tile's ids visible
    stage_weight(sB3, KP, 64, d.rw[2], R2, 0, cin, R2);
    int nx_row = -1, nx_seg = -1;
    if (tid < ST) {
      int k = (tile + (int)gridDim.x) * ST + tid;
      if (k < N) nx_row = order[k];
    }
    // in_feats rows -> smem: one warp per row, lanes stride the columns (4-byte cp.async: rows of cin floats are only
    // 4-byte aligned in general)
    for (int r = warp; r < nrow; r += NT / 32) {
      const float* src = in_feats + (size_t)sRow[r] * in_ld;  // columns >= gap_at sit `gap` floats further (16-B aligned feature block)
      const uint32_t dst = smem_u32(sIn + r * pitch_in);
      for (int c = lane; c < cin; c += 32)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(dst + 4u * c), "l"(src + c + (c >= gap_at ? gap : 0)) : "memory");
    }
    {
      // rel-MLP layers 1, 2: four adjacent lanes per point; each owns R2/4 = 8 outputs of layer 2 (layer 1 is recomputed by
      // all four), LayerNorm statistics by two xor-shuffles; result bf16 -> A operand of the layer-3 GEMM
      const int r = tid >> 2, part = tid & 3;
      float h2[8];
      const int row = sRow[r];
      const bool alive = row >= 0;  // dead rows run the same code on zeros: the shuffles below need every lane of the warp
      {
        float x[4] = {0.f, 0.f, 0.f, 0.f};
        if (alive) {
          const float* fc = f_cluster + (size_t)row * d.rel_in;
          for (int i = 0; i < d.rel_in; i++) x[i] = fc[i] / d.rel_dist_scaler;
        }
        float h1[R1];
#pragma unroll
        for (int o = 0; o < R1; o++) {
          const float4 w = *reinterpret_cast<const float4*>(&sW1[o * 4]);
          h1[o] = fmaf(w.w, x[3], fmaf(w.z, x[2], fmaf(w.y, x[1], w.x * x[0])));
        }
        float mean, rstd;
        ln_regs<R1>(h1, mean, rstd, d.eps);
#pragma unroll
        for (int o = 0; o < R1; o++) h1[o] = act_f<ACT>((h1[o] - mean) * rstd * sG1[o] + sBt1[o]);
        float s = 0.f;
#pragma unroll
        for (int o = 0; o < 8; o++) {
          const float4* wr = reinterpret_cast<const float4*>(&sW2[(part * 8 + o) * R1]);
          float a = 0.f;
#pragma unroll
          for (int k4 = 0; k4 < R1 / 4; k4++) {
            const float4 w = wr[k4];
            a = fmaf(w.x, h1[4 * k4], fmaf(w.y, h1[4 * k4 + 1], fmaf(w.z, h1[4 * k4 + 2], fmaf(w.w, h1[4 * k4 + 3], a))));
          }
          h2[o] = a;
          s += a;
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        mean = s / (float)R2;
        float q = 0.f;
#pragma unroll
        for (int o = 0; o < 8; o++) {
          float t = h2[o] - mean;
          q = fmaf(t, t, q);
        }
        q += __shfl_xor_sync(0xffffffffu, q, 1);
        q += __shfl_xor_sync(0xffffffffu, q, 2);
        rstd = rsqrtf(q / (float)R2 + d.eps);
#pragma unroll
        for (int o = 0; o < 8; o++) h2[o] = alive ? act_f<ACT>((h2[o] - mean) * rstd * sG2[part * 8 + o] + sBt2[part * 8 + o]) : 0.f;
      }
      *reinterpret_cast<int4*>(sA3 + sw128_off(ST, r, part)) = pack8_h16<FMT_BF16>(h2);
      // K columns R2..63 are zero (the previous tile's accumulators overwrote them)
      *reinterpret_cast<int4*>(sA3 + sw128_off(ST, r, part + 4)) = make_int4(0, 0, 0, 0);
    }
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    fence_async_smem();
    __syncthreads();
    // rel layer 3: [ST, R2] x [KP rows, R2]^T, warpgroup w: rows 64 (w & 1).., columns KP/2 (w >> 1)..; the fragments reach the
    // thread-per-row epilogue one column quarter at a time through a [ST][64] tile
    float v[NQC];
    {
      const int w = tid >> 7;
      float dq[KP / 4];
      wg_tile_mma<KP / 2, true, R2 / 16>(dq, smem_u32(sA3) + (w & 1) * 64 * 128, ST * 128, smem_u32(sB3) + (w >> 1) * (KP / 2) * 128, KP * 128,
                                         false);
      wgmma_wait<0>();
      __syncthreads();   // the accumulator tile aliases both operands
#pragma unroll
      for (int q = 0; q < 4; q++) {
        if ((w >> 1) == (q >> 1)) {
          const int c0 = (q & 1) * NQC;
          wg_frag_pairs<KP / 2>(dq, [&](int r, int c, float v0, float v1) {
            if (c >= c0 && c < c0 + NQC) *reinterpret_cast<float2*>(sAcc + acc_idx(64, (w & 1) * 64 + r, c - c0)) = make_float2(v0, v1);
          });
        }
        __syncthreads();
        if (quarter == q) acc_ld<NQC>(sAcc, 64, lrow, 0, v);
        __syncthreads();
      }
    }
    if (nx_row >= 0) nx_seg = (int)inv[nx_row];
    {
      // epilogue rel3: LayerNorm over cin, act, gate with [xyz / normalizer || feats] -> x0 (bf16 A operand of layer 0)
      const int qb = quarter * NQC;
      const int nvalid = min(max(cin - qb, 0), NQC);  // warp-uniform: valid channels of this quarter
      // columns >= cin are exactly 0 (zero weight rows), so the plain sum gives the mean; the variance sums the valid columns only
      // (subtracting the pad columns' (KP - cin) mean^2 afterwards cancels when the channels share a large common part)
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NQC; i++) s += v[i];
      redA[quarter][lrow] = s;
      __syncthreads();
      const float mean = (redA[0][lrow] + redA[1][lrow] + redA[2][lrow] + redA[3][lrow]) / (float)cin;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < NQC; i++) {
        float t = i < nvalid ? v[i] - mean : 0.f;
        q = fmaf(t, t, q);
      }
      redB[quarter][lrow] = q;
      __syncthreads();
      const float rstd = rsqrtf((redB[0][lrow] + redB[1][lrow] + redB[2][lrow] + redB[3][lrow]) / (float)cin + d.eps);
      const float* frow = sIn + lrow * pitch_in;  // rows past the end hold stale data: their x0 / p0 rows are never used
#pragma unroll
      for (int j = 0; j < NQC / 8; j++) {
        int4 pk = make_int4(0, 0, 0, 0);
        if (j * 8 < nvalid) {  // warp-uniform
          float y[8];
          const bool full = j * 8 + 8 <= nvalid;  // warp-uniform
#pragma unroll
          for (int i = 0; i < 8; i++) {
            const int gc = qb + j * 8 + i;
            float o = 0.f;
            if (full || j * 8 + i < nvalid) {
              float f = frow[gc];
              if (j == 0 && i < 3 && quarter == 0) f = f / d.nz[i];
              o = act_f<ACT>((v[j * 8 + i] - mean) * rstd * sG3[gc] + sBt3[gc]) * f;
            }
            y[i] = o;
          }
          pk = pack8_h16<FMT_BF16>(y);
        }
        *reinterpret_cast<int4*>(sA0 + sw128_off(ST, lrow, qb / 8 + j)) = pk;
      }
    }
    fence_async_smem();
    __syncthreads();   // x0 complete; every thread is done reading the rel-3 accumulators
    // layer 0: [ST, KP] x [SC, KP]^T
    sir_gemm<SC, KP / 16>(smem_u32(sA0), ST * 128, smem_u32(sB0), SC * 128, sAcc, false);
    {
      // epilogue 0: LayerNorm over SC, act -> p0 (bf16 rows in CSR order for kernel B; fp32 tile for the pooled max)
      constexpr int H = SC / 4;
      float v[H];
      acc_ld<H>(sAcc, SC, lrow, quarter * H, v);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < H; i++) s += v[i];
      redA[quarter][lrow] = s;
      __syncthreads();
      const float mean = (redA[0][lrow] + redA[1][lrow] + redA[2][lrow] + redA[3][lrow]) / (float)SC;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < H; i++) {
        float t = v[i] - mean;
        q = fmaf(t, t, q);
      }
      redB[quarter][lrow] = q;
      __syncthreads();
      const float rstd = rsqrtf((redB[0][lrow] + redB[1][lrow] + redB[2][lrow] + redB[3][lrow]) / (float)SC + d.eps);
#pragma unroll
      for (int i = 0; i < H; i++) v[i] = act_f<ACT>((v[i] - mean) * rstd * sG0[quarter * H + i] + sBt0[quarter * H + i]);
      warp_segmax_ord(v, sSeg[lrow], quarter * H, gord);
      if (lrow < nrow) {
        int4* dst = reinterpret_cast<int4*>(p0buf + (size_t)(k0 + lrow) * SC + quarter * H);
#pragma unroll
        for (int j = 0; j < H / 8; j++) dst[j] = pack8_h16<FMT_BF16>(v + j * 8);
      }
    }
    if (tid < ST) {
      sRowB[cur ^ 1][tid] = nx_row;
      sSegB[cur ^ 1][tid] = nx_seg;
    }
    cur ^= 1;
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// kernel B (same thread layout)
// ------------------------------------------------------------------------------------------------------------------------
template <int ACT>
__global__ void __launch_bounds__(NT, 1) sir_b_kernel(SirDev d, const __nv_bfloat16* __restrict__ p0buf, const float* __restrict__ g0 /*[G, ldg]*/,
                                                      int ldg, const long long* __restrict__ inv, const int32_t* __restrict__ order, int N,
                                                      float* __restrict__ out_point, int ldo, bool vec_out, uint32_t* __restrict__ gord) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint8_t sirb_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)sirb_raw + 1023) & ~(uintptr_t)1023);
  constexpr int K1 = 2 * SC;                 // the reference's [p0 || g0[group]] input, formed only inside the operand tile
  uint8_t* sB = base;                        // W1  : 4 chunks x SC rows x 128 B
  uint8_t* sA = sB + (size_t)SC * K1 * 2;    // [p0 || g0[group]] : 4 chunks x ST rows x 128 B
  float* sAcc = reinterpret_cast<float*>(sA);  // accumulator tile [ST][SC] fp32, aliases the A operand
  __shared__ float sG[SC], sBt[SC];
  __shared__ float redA[4][ST], redB[4][ST];
  __shared__ int sRowB[2][ST], sSegB[2][ST];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ntiles = (N + ST - 1) / ST;
  if ((int)blockIdx.x >= ntiles) return;
  for (int i = tid; i < SC; i += NT) sG[i] = d.g1[i], sBt[i] = d.b1[i];
  stage_weight(sB, SC, K1, d.w1, K1, 0, SC, K1);
  const int quarter = warp >> 2;
  const int lrow = (warp & 3) * 32 + lane;
  constexpr int H = SC / 4;
  int cur = 0;
  if (tid < ST) {
    int k = blockIdx.x * ST + tid;
    int row = k < N ? order[k] : -1;
    sRowB[0][tid] = row;
    sSegB[0][tid] = row >= 0 ? (int)inv[row] : -1;
  }
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int k0 = tile * ST;
    const int nrow = min(ST, N - k0);
    const int* sRow = sRowB[cur];
    const int* sSeg = sSegB[cur];
    __syncthreads();  // previous tile consumed, this tile's ids visible
    int nx_row = -1, nx_seg = -1;
    if (tid < ST) {
      int k = (tile + (int)gridDim.x) * ST + tid;
      if (k < N) nx_row = order[k];
    }
    for (int idx = tid; idx < ST * (SC / 8); idx += NT) {
      int r = idx / (SC / 8), j = idx % (SC / 8);
      cp_async_piece_or_zero(sA + sw128_off(ST, r, j), p0buf + (size_t)(k0 + r) * SC + j * 8, r < nrow);
    }
    // second half of the K extent: the group's pooled layer-0 features (fp32 -> bf16), 4 pieces in flight per thread
    {
      float4 a[4], bq[4];
#pragma unroll
      for (int u = 0; u < 4; u++) {
        int idx = tid + u * NT;
        int r = idx / (SC / 8), j = idx % (SC / 8);
        a[u] = bq[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < nrow) {
          const float4* gp = reinterpret_cast<const float4*>(g0 + (size_t)sSeg[r] * ldg + j * 8);
          a[u] = __ldg(gp);
          bq[u] = __ldg(gp + 1);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; u++) {
        int idx = tid + u * NT;
        int r = idx / (SC / 8), j = idx % (SC / 8) + SC / 8;
        *reinterpret_cast<int4*>(sA + sw128_off(ST, r, j)) = pack8_h16<FMT_BF16>(a[u], bq[u]);
      }
    }
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    fence_async_smem();
    __syncthreads();
    sir_gemm<SC, K1 / 16>(smem_u32(sA), ST * 128, smem_u32(sB), SC * 128, sAcc, true);
    if (nx_row >= 0) nx_seg = (int)inv[nx_row];
    float v[H];
    acc_ld<H>(sAcc, SC, lrow, quarter * H, v);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < H; i++) s += v[i];
    redA[quarter][lrow] = s;
    __syncthreads();
    const float mean = (redA[0][lrow] + redA[1][lrow] + redA[2][lrow] + redA[3][lrow]) / (float)SC;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < H; i++) {
      float t = v[i] - mean;
      q = fmaf(t, t, q);
    }
    redB[quarter][lrow] = q;
    __syncthreads();
    const float rstd = rsqrtf((redB[0][lrow] + redB[1][lrow] + redB[2][lrow] + redB[3][lrow]) / (float)SC + d.eps);
#pragma unroll
    for (int i = 0; i < H; i++) v[i] = act_f<ACT>((v[i] - mean) * rstd * sG[quarter * H + i] + sBt[quarter * H + i]);
    warp_segmax_ord(v, sSeg[lrow], quarter * H, gord);
    if (lrow < nrow) {  // fp32 row segment (128 B) to the caller's buffer, original point order
      float* orow = out_point + (size_t)sRow[lrow] * ldo + quarter * H;
      if (vec_out) {
#pragma unroll
        for (int j = 0; j < H / 4; j++) reinterpret_cast<float4*>(orow)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
      } else {
#pragma unroll
        for (int i = 0; i < H; i++) orow[i] = v[i];
      }
    }
    if (tid < ST) {
      sRowB[cur ^ 1][tid] = nx_row;
      sSegB[cur ^ 1][tid] = nx_seg;
    }
    cur ^= 1;
  }
}

}  // namespace

// Host entry (called from sir.cu).  Returns SSTB_ERR_UNSUPPORTED for shapes outside the tensor path.
int sstb_sir_layer_bf16(sstb200_ctx* c, const sstb200_sir_layer* L, const float* in_feats, const float* f_cluster, const long long* inv,
                        const int32_t* order, int N, int G, __nv_bfloat16* p0buf, uint32_t* gord, float* gterm, float* out_point, int ldo,
                        float* out_group, int in_ld, int gap_at, int gap) {
  const int cin = L->in_channels;
  if (L->num_vfe != 2 || L->feat_channels[0] != SC || L->feat_channels[1] != SC || L->num_rel != 3 || L->rel_dims[0] != 16 ||
      L->rel_dims[1] != 32 || L->rel_dims[2] != cin || L->rel_in < 1 || L->rel_in > 4 || cin < 3 || cin > 192)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED,
                     "SIRLayer bf16 path needs feat_channels [128,128], rel-MLP [16,32,cin], cin <= 192 (got cin=%d, C=[%d,%d], rel=%d)", cin,
                     L->feat_channels[0], L->feat_channels[1], L->num_rel);
  SirDev d;
  d.cin = cin;
  d.rel_in = L->rel_in;
  d.act = L->act;
  d.eps = L->norm_eps;
  d.rel_dist_scaler = L->rel_dist_scaler;
  for (int i = 0; i < 3; i++) {
    d.nz[i] = L->xyz_normalizer[i];
    d.rw[i] = L->rel_w[i];
    d.rg[i] = L->rel_ln_w[i];
    d.rb[i] = L->rel_ln_b[i];
    CHECK_ARG(c, d.rw[i] && d.rg[i] && d.rb[i]);
  }
  d.w0 = L->vfe_w[0], d.g0 = L->vfe_ln_w[0], d.b0 = L->vfe_ln_b[0];
  d.w1 = L->vfe_w[1], d.g1 = L->vfe_ln_w[1], d.b1 = L->vfe_ln_b[1];
  CHECK_ARG(c, d.w0 && d.g0 && d.b0 && d.w1 && d.g1 && d.b1);
  cudaStream_t st = c->stream;
  const int KP = cin <= 128 ? 128 : 192;
  const int pitch_in = cin | 1;
  // in_feats region at least large enough for the layer-0 accumulator tile [ST][SC] fp32 that starts at Wr3
  size_t in_bytes = (size_t)ST * pitch_in * 4;
  const size_t acc0 = (size_t)ST * SC * 4 - (size_t)KP * 128 - (size_t)ST * 128;
  if (in_bytes < acc0) in_bytes = acc0;
  const size_t smemA = 1024 + (size_t)SC * KP * 2 + (size_t)KP * 128 + (size_t)ST * KP * 2 + (size_t)ST * 128 + in_bytes;
  const size_t smemB = 1024 + (size_t)SC * 2 * SC * 2 + (size_t)ST * 2 * SC * 2;
  if (smemA + 12 * 1024 > 227 * 1024)  // + ~11 KB of static shared memory
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "SIRLayer bf16: tile of cin=%d does not fit shared memory", cin);
  const int ntiles = (N + ST - 1) / ST;
  const int grid = ntiles < c->num_sms ? ntiles : c->num_sms;
  const size_t gn = (size_t)G * SC;
  const int Cg = 2 * SC;
  // kernel B stores point rows as float4 only when every row segment is 16-byte aligned: a view such as buf[:, 1:129] of a buffer
  // with 132 columns has ldo % 4 == 0 but a base 4 bytes off
  const bool vec_out = ldo % 4 == 0 && (reinterpret_cast<uintptr_t>(out_point) & 15) == 0;
  CUDA_TRY(c, cudaMemsetAsync(gord, 0, gn * 4, st));
#define SIR_A(KPV, ACTV)                                                                                                          \
  do {                                                                                                                            \
    static SmemAttr sa;                                                                                                           \
    CUDA_TRY(c, ensure_smem(c, sa, sir_a_kernel<KPV, 16, 32, ACTV>, smemA));                                                      \
    launch_pdl(sir_a_kernel<KPV, 16, 32, ACTV>, dim3(grid), dim3(NT), smemA, st, d, in_feats, f_cluster, inv, order, N, p0buf, gord, pitch_in, in_ld, gap_at, gap); \
  } while (0)
#define SIR_A2(KPV)            \
  do {                         \
    if (L->act == 2) SIR_A(KPV, 2); \
    else SIR_A(KPV, 1);        \
  } while (0)
  if (KP == 128) SIR_A2(128);
  else SIR_A2(192);
#undef SIR_A2
#undef SIR_A
  sstb_sir_segmax_finalize(st, gord, G, SC, out_group, Cg, 0);
  CUDA_TRY(c, cudaMemsetAsync(gord, 0, gn * 4, st));
#define SIR_B(ACTV)                                                                                                     \
  do {                                                                                                                  \
    static SmemAttr sa;                                                                                                 \
    CUDA_TRY(c, ensure_smem(c, sa, sir_b_kernel<ACTV>, smemB));                                                         \
    launch_pdl(sir_b_kernel<ACTV>, dim3(grid), dim3(NT), smemB, st, d, (const __nv_bfloat16*)p0buf, (const float*)out_group, Cg, inv, order, N, out_point, ldo, vec_out, gord); \
  } while (0)
  if (L->act == 2) SIR_B(2);
  else SIR_B(1);
#undef SIR_B
  sstb_sir_segmax_finalize(st, gord, G, SC, out_group, Cg, SC);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
