// Ragged window attention (SIMT, fp32 math), templated on the q/k/v and output element types.
// One thread per (token slot, head): online softmax over the keys of the token's window.  qkv [n, 3d] in flat
// token order; the window CSR gives the key set, so no padding, no mask, no per-level batches.
//   cosine mode (models/sst/cosine_msa.py:123-185): q,k L2-normalised, logits / clamp(tau, tau_min).
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"

template <typename T, int N>
__device__ __forceinline__ void load_vec(const T* p, float* o);
template <>
__device__ __forceinline__ void load_vec<float, 8>(const float* p, float* o) {
  float4 a = *(const float4*)p, b = *(const float4*)(p + 4);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}
template <>
__device__ __forceinline__ void load_vec<__nv_bfloat16, 8>(const __nv_bfloat16* p, float* o) {
  int4 v = *(const int4*)p;
  const __nv_bfloat162* h = (const __nv_bfloat162*)&v;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float2 f = __bfloat1622float2(h[i]);
    o[2 * i] = f.x;
    o[2 * i + 1] = f.y;
  }
}
template <>
__device__ __forceinline__ void load_vec<__half, 8>(const __half* p, float* o) {
  int4 v = *(const int4*)p;
  const __half2* h = (const __half2*)&v;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    float2 f = __half22float2(h[i]);
    o[2 * i] = f.x;
    o[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void store_vec8(__half* p, const float* v) {
  __half2 h[4];
#pragma unroll
  for (int i = 0; i < 4; i++) h[i] = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
  *(int4*)p = *(const int4*)h;
}
__device__ __forceinline__ void store_vec8(float* p, const float* v) {
  *(float4*)p = make_float4(v[0], v[1], v[2], v[3]);
  *(float4*)(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void store_vec8(__nv_bfloat16* p, const float* v) {
  __nv_bfloat162 h[4];
#pragma unroll
  for (int i = 0; i < 4; i++) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  *(int4*)p = *(const int4*)h;
}

template <typename TI, typename TO, int DH>
__global__ void __launch_bounds__(256) win_attn_kernel(const TI* __restrict__ qkv, int d, int nhead, int n,
                                                       const int32_t* __restrict__ n_dev,
                                                       const int32_t* __restrict__ win_offsets,
                                                       const int32_t* __restrict__ tok_perm,
                                                       const int32_t* __restrict__ tok_win, float scale,
                                                       const float* __restrict__ tau, int tau_n, float tau_min,
                                                       TO* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  if (n_dev) n = *n_dev;
  long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int slot = (int)(g / nhead), h = (int)(g % nhead);
  if (slot >= n) return;
  int tok = tok_perm[slot];
  int w = tok_win[tok];
  int kb = win_offsets[w], ke = win_offsets[w + 1];
  const TI* qp = qkv + (size_t)tok * 3 * d + h * DH;
  float q[DH];
#pragma unroll
  for (int i = 0; i < DH; i += 8) load_vec<TI, 8>(qp + i, q + i);
  bool cosine = tau != nullptr;
  float s_mul = scale;
  if (cosine) {
    float nq = 0.f;
#pragma unroll
    for (int i = 0; i < DH; i++) nq = fmaf(q[i], q[i], nq);
    float t = fmaxf(tau_n > 1 ? tau[h] : tau[0], tau_min);
    s_mul = 1.0f / (fmaxf(sqrtf(nq), 1e-12f) * t);  // F.normalize eps = 1e-12
  }
  float m = -INFINITY, l = 0.f, acc[DH];
#pragma unroll
  for (int i = 0; i < DH; i++) acc[i] = 0.f;
  for (int j = kb; j < ke; j++) {
    int kt = tok_perm[j];
    const TI* kp = qkv + (size_t)kt * 3 * d + d + h * DH;
    const TI* vp = kp + d;
    float kk[DH], vv[DH];
#pragma unroll
    for (int i = 0; i < DH; i += 8) {
      load_vec<TI, 8>(kp + i, kk + i);
      load_vec<TI, 8>(vp + i, vv + i);
    }
    float s = 0.f, nk = 0.f;
#pragma unroll
    for (int i = 0; i < DH; i++) {
      s = fmaf(q[i], kk[i], s);
      if (cosine) nk = fmaf(kk[i], kk[i], nk);
    }
    s *= s_mul;
    if (cosine) s /= fmaxf(sqrtf(nk), 1e-12f);
    float mn = fmaxf(m, s);
    float corr = __expf(m - mn);  // m = -inf on the first key -> 0
    float p = __expf(s - mn);
    l = l * corr + p;
#pragma unroll
    for (int i = 0; i < DH; i++) acc[i] = fmaf(acc[i], corr, p * vv[i]);
    m = mn;
  }
  float inv = 1.0f / l;
#pragma unroll
  for (int i = 0; i < DH; i++) acc[i] *= inv;
  TO* op = out + (size_t)tok * d + h * DH;
#pragma unroll
  for (int i = 0; i < DH; i += 8) store_vec8(op + i, acc + i);
}

template <typename TI, typename TO>
int sstb_win_attn(sstb200_ctx* c, const TI* qkv, int d, int nhead, int n_cap, const int32_t* n_dev, const int32_t* win_offsets,
                  const int32_t* tok_perm, const int32_t* tok_win, const float* tau, int tau_n, float tau_min, TO* out) {
  int dh = d / nhead;
  long long items = (long long)n_cap * nhead;
  unsigned grid = (unsigned)((items + 255) / 256);
  float scale = 1.0f / sqrtf((float)dh);
  if (grid == 0) return SSTB_OK;
#define LAUNCH_ATT(DH)                                                                                                  \
  launch_pdl(win_attn_kernel<TI, TO, DH>, dim3(grid), dim3(256), (size_t)(0), c->stream, qkv, d, nhead, n_cap, n_dev, win_offsets, tok_perm, tok_win, \
                                                           scale, tau, tau_n, tau_min, out)
  if (dh == 16) LAUNCH_ATT(16);
  else if (dh == 8) LAUNCH_ATT(8);
  else if (dh == 32) LAUNCH_ATT(32);
  else if (dh == 64) LAUNCH_ATT(64);
  else return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "head dim %d not supported (8/16/32/64)", dh);
#undef LAUNCH_ATT
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// Tensor-core ragged window attention helpers (mma.sync.m16n8k16, fp32 accumulate) shared by the kernels below.
// ------------------------------------------------------------------------------------------------

__device__ __forceinline__ void mma_bf16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_f16_16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}


// ------------------------------------------------------------------------------------------------

__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t ex2_h2(float a, float b) {
  uint32_t h, r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));
  asm("ex2.approx.f16x2 %0, %1;" : "=r"(r) : "r"(h));
  return r;
}

// ------------------------------------------------------------------------------------------------
// v5: batched ragged attention on mma.sync tiles, single-pass softmax.
// One CTA stages a *batch* of consecutive whole windows (<= 144 tokens each, built by win_batch_kernel): the K and V columns
// of its NHL heads, gathered row by row through the window permutation with cp.async (q|k|v and the output live in flat token
// order, SURVEY 8a B6: flat2window / window2flat never materialise).  Its 8 warps sweep the batch's 16-query tiles; a tile is
// processed for all NHL heads in turn.  Per (tile, head) the window is walked in chunks of <= 64 keys (one chunk for most
// windows, up to three for the 65..144-token ones): S = Q K^T of the chunk stays in REGISTERS (KT key tiles of 8, fully
// unrolled, no inner branches; K fragments by ldmatrix.x4), row maxima by shuffles, P = 2^(scale' S - max) computed two at a
// time on the half2 MUFU path - which is exactly the fp16 A fragment of P V - V^T fragments by ldmatrix.trans, and the row
// sums come out of the tensor core as well (a constant "ones" B fragment).  A further chunk rescales the running accumulators
// by 2^(old max - new max).  ~0.15 instructions per score; the two-pass form this replaces needed ~0.7.
// ------------------------------------------------------------------------------------------------
#define ATT_KCHUNK 64

// m0 / m1: running row maxima in log2 units; o / ol: running numerators / denominators.  kaddr / vaddr: this lane's ldmatrix
// row addresses for the chunk's first key (shared-memory byte addresses); n = keys of the window inside this chunk
// (8 * KT - 16 < n <= 8 * KT, so only the last two key tiles can be partial).
template <int KT, int LD, bool COS>
__device__ __forceinline__ void attn_chunk(const uint32_t* qa, uint32_t kaddr, uint32_t vaddr, int n, int t4, bool ones_lane, float sl2_0,
                                           float sl2_1, const float* invk, bool first, float& m0, float& m1, float (*o)[4], float* ol) {
  float s[KT][4];
#pragma unroll
  for (int jj = 0; jj < KT / 2; jj++) {
    uint32_t kf[4];
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(kf[0]), "=r"(kf[1]), "=r"(kf[2]), "=r"(kf[3])
                 : "r"(kaddr + (uint32_t)(jj * 16 * LD * 2)));
    s[2 * jj][0] = s[2 * jj][1] = s[2 * jj][2] = s[2 * jj][3] = 0.f;
    s[2 * jj + 1][0] = s[2 * jj + 1][1] = s[2 * jj + 1][2] = s[2 * jj + 1][3] = 0.f;
    mma_f16_16816(s[2 * jj], qa, kf[0], kf[1]);
    mma_f16_16816(s[2 * jj + 1], qa, kf[2], kf[3]);
  }
  if (COS) {   // cosine attention: the key's 1 / |k| per column (the query's 1 / |q| and 1 / tau ride in the row scales)
#pragma unroll
    for (int j = 0; j < KT; j++) {
      const float i0 = invk[j * 8 + 2 * t4], i1 = invk[j * 8 + 2 * t4 + 1];
      s[j][0] *= i0, s[j][1] *= i1, s[j][2] *= i0, s[j][3] *= i1;
    }
  }
  // columns past the window hold other windows' keys or zero fill: -inf (only the last two tiles can be affected)
#pragma unroll
  for (int j = KT - 2; j < KT; j++) {
    const int c0 = j * 8 + 2 * t4;
    if (c0 >= n) s[j][0] = s[j][2] = -INFINITY;
    if (c0 + 1 >= n) s[j][1] = s[j][3] = -INFINITY;
  }
  float c0m = fmaxf(s[0][0], s[0][1]), c1m = fmaxf(s[0][2], s[0][3]);
#pragma unroll
  for (int j = 1; j < KT; j++) {
    c0m = fmaxf(c0m, fmaxf(s[j][0], s[j][1]));
    c1m = fmaxf(c1m, fmaxf(s[j][2], s[j][3]));
  }
  c0m = fmaxf(c0m, __shfl_xor_sync(0xffffffffu, c0m, 1));
  c0m = fmaxf(c0m, __shfl_xor_sync(0xffffffffu, c0m, 2));
  c1m = fmaxf(c1m, __shfl_xor_sync(0xffffffffu, c1m, 1));
  c1m = fmaxf(c1m, __shfl_xor_sync(0xffffffffu, c1m, 2));
  const float n0 = fmaxf(m0, c0m * sl2_0), n1 = fmaxf(m1, c1m * sl2_1);   // (row scales are positive)
  if (!first) {   // rescale what the earlier chunks accumulated (warp-uniform)
    const float f0 = fast_ex2(m0 - n0), f1 = fast_ex2(m1 - n1);
    o[0][0] *= f0, o[0][1] *= f0, o[1][0] *= f0, o[1][1] *= f0, ol[0] *= f0, ol[1] *= f0;
    o[0][2] *= f1, o[0][3] *= f1, o[1][2] *= f1, o[1][3] *= f1, ol[2] *= f1, ol[3] *= f1;
  }
  m0 = n0;
  m1 = n1;
  const uint32_t ones = ones_lane ? 0x3C003C00u : 0u;   // B fragment whose column 0 is 1: the row sums of P
#pragma unroll
  for (int kc = 0; kc < KT / 2; kc++) {
    uint32_t pa[4];
    pa[0] = ex2_h2(fmaf(s[2 * kc][0], sl2_0, -n0), fmaf(s[2 * kc][1], sl2_0, -n0));
    pa[1] = ex2_h2(fmaf(s[2 * kc][2], sl2_1, -n1), fmaf(s[2 * kc][3], sl2_1, -n1));
    pa[2] = ex2_h2(fmaf(s[2 * kc + 1][0], sl2_0, -n0), fmaf(s[2 * kc + 1][1], sl2_0, -n0));
    pa[3] = ex2_h2(fmaf(s[2 * kc + 1][2], sl2_1, -n1), fmaf(s[2 * kc + 1][3], sl2_1, -n1));
    uint32_t vb[4];
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(vb[0]), "=r"(vb[1]), "=r"(vb[2]), "=r"(vb[3])
                 : "r"(vaddr + (uint32_t)(kc * 16 * LD * 2)));
    mma_f16_16816(o[0], pa, vb[0], vb[1]);
    mma_f16_16816(o[1], pa, vb[2], vb[3]);
    mma_f16_16816(ol, pa, ones, ones);
  }
}

// NHL = heads handled by one CTA: a batch is split over 8/NHL CTAs (each stages only its heads' Q/K/V columns), which shortens
// the critical path of batches that hold one big window and raises the number of resident warps per SM.
// A CTA's life is a chain of dependent global loads (batch record -> window permutation -> q|k|v rows), so the kernel is built
// to keep that chain short and off the producer's critical path: (1) one int4 record per batch from win_batch_kernel instead of
// win_batch -> win_offsets, (2) everything that depends only on the window plan (record, token list, q-tile table) happens
// BEFORE griddepcontrol.wait, i.e. while the tail of the kernel that produces q|k|v is still running (the plan was written by
// kernels that completed before that producer started: every kernel of the library waits before it triggers its dependents),
// (3) Q is staged with K and V by cp.async, so the compute phase never waits on global memory.
// COS: cosine attention (models/sst/cosine_msa.py:123-185): logits = (q / |q|) . (k / |k|) / clamp(tau_head, tau_min) instead of
// q . k / sqrt(dh).  q and k stay as staged; 1 / |q|, 1 / |k| per (row, head) are computed once per batch in fp32 and applied to the
// fp32 scores (no second rounding of the operands).
template <int NHL, bool OUT_BF16, bool COS>
static __global__ void __launch_bounds__(256, 3) win_attn_batch_kernel(const __half* __restrict__ qkv,
                                                                       const int32_t* __restrict__ counters,
                                                                       const int32_t* __restrict__ win_offsets,
                                                                       const int4* __restrict__ batch_rec, int rec_cap,
                                                                       const int32_t* __restrict__ tok_perm, float scale,
                                                                       const float* __restrict__ tau, int tau_n, float tau_min,
                                                                       __half* __restrict__ out) {
  pdl_launch();
  constexpr int D = 128, DH = 16, LD = NHL * 16 + 8, HSPLIT = 8 / NHL, PPR = NHL * 2;  // PPR: 16-byte pieces per row per matrix
  constexpr int NROW = ATT_BT + 16;
  extern __shared__ __align__(16) uint8_t att_smem[];
  __half* sK = reinterpret_cast<__half*>(att_smem);
  __half* sV = sK + NROW * LD;
  __half* sQ = sV + NROW * LD;
  __shared__ int sTok[NROW];           // token row of local slot r, -1 beyond the batch
  __shared__ short sTileRow[ATT_BT];   // first local row of q-tile k
  __shared__ short sTileKb[ATT_BT];    // local key range of its window
  __shared__ short sTileKe[ATT_BT];
  __shared__ int sNumTiles;
  __shared__ float sInvQ[COS ? NHL * NROW : 1], sInvK[COS ? NHL * NROW : 1];   // [head][row]: 1 / max(|q|, 1e-12), 1 / max(|k|, 1e-12)
  // record of window batch b (see ATT_CHUNK in common.cuh) = {first window, end window, first slot, end slot}
  int4 rc = batch_rec[min((int)blockIdx.x / HSPLIT, rec_cap - 1)];
  const int nbatch = counters[17];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g4 = lane >> 2, t4 = lane & 3;
  const uint32_t k0 = (uint32_t)__cvta_generic_to_shared(sK), v0 = (uint32_t)__cvta_generic_to_shared(sV),
                 q0 = (uint32_t)__cvta_generic_to_shared(sQ);
  // this lane's ldmatrix row offsets (bytes) inside a 16-row block: K fragments (non-transposed) / V^T fragments (.trans); the
  // Q (A operand) fragment uses the V pattern without .trans
  const uint32_t klane = (uint32_t)((((lane & 7) + ((lane >> 4) & 1) * 8) * LD + ((lane >> 3) & 1) * 8) * 2);
  const uint32_t vlane = (uint32_t)((((lane & 7) + ((lane >> 3) & 1) * 8) * LD + (lane >> 4) * 8) * 2);
  const float sl2 = scale * 1.4426950408889634f;   // exp(x) = 2^(x log2 e)
  for (int unit = blockIdx.x; unit < nbatch * HSPLIT; unit += gridDim.x) {
    const int b = unit / HSPLIT, hs = unit % HSPLIT;
    if (unit != (int)blockIdx.x) rc = batch_rec[b];
    const int wb = rc.x, we = rc.y, s0 = rc.z, s1 = rc.w;
    if (wb == we) continue;  // a big window covers this chunk entirely (uniform per CTA)
    const int nrow = min(s1 - s0, ATT_BT);
    const int nfill = min(((nrow + 15) & ~15) + 16, NROW);  // key chunks may run up to 15 rows past the batch: keep them finite (0)
    __syncthreads();  // previous batch fully consumed
    // staging role: lane = (row of an 8-row group, 16-byte piece p of the NHL heads' columns); a warp covers 8 rows x {K, V, Q} per
    // step, the CTA 64 rows -> <= 5 steps, all of whose token loads are in flight together
    constexpr int SROWS = 256 / PPR, SSTEPS = (NROW + SROWS - 1) / SROWS;
    const int s_r = threadIdx.x / PPR, s_p = threadIdx.x % PPR;
    int stok[SSTEPS];
#pragma unroll
    for (int j = 0; j < SSTEPS; j++) {
      const int r = s_r + j * SROWS;
      stok[j] = r < nrow ? tok_perm[s0 + r] : -1;
    }
    // q-tile table (warp 0): windows of the batch -> tiles
    if (warp == 0) {
      int cnt = 0;
      for (int w0 = wb; w0 < we; w0 += 32) {
        int w = w0 + lane;
        int kb = 0, n = 0;
        if (w < we) {
          kb = win_offsets[w] - s0;
          n = win_offsets[w + 1] - s0 - kb;
          if (kb + n > ATT_BT) n = max(ATT_BT - kb, 0);
        }
        int nt = (n + 15) >> 4;
        int x = nt;
#pragma unroll
        for (int o2 = 1; o2 < 32; o2 <<= 1) {
          int y = __shfl_up_sync(0xffffffffu, x, o2);
          if (lane >= o2) x += y;
        }
        int base = cnt + x - nt;
        for (int k = 0; k < nt; k++) {
          if (base + k < ATT_BT) {
            sTileRow[base + k] = (short)(kb + 16 * k);
            sTileKb[base + k] = (short)kb;
            sTileKe[base + k] = (short)(kb + n);
          }
        }
        cnt += __shfl_sync(0xffffffffu, x, 31);
      }
      if (lane == 0) sNumTiles = min(cnt, ATT_BT);
    }
    pdl_wait();   // q|k|v of this layer are complete and visible from here on (returns at once after the first unit)
    // K | V | Q rows (gathered through the window permutation): 16-byte pieces with cp.async, zero fill beyond the batch
#pragma unroll
    for (int j = 0; j < SSTEPS; j++) {
      const int r = s_r + j * SROWS;
      if (r < nfill) {
        const int tok = stok[j];
        if (s_p == 0) sTok[r] = tok;
        const uint32_t doff = (uint32_t)(r * LD * 2 + s_p * 16);
        if (tok >= 0) {
          const __half* src = qkv + (size_t)tok * (3 * D) + (hs * NHL) * DH + s_p * 8;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(q0 + doff), "l"(src) : "memory");
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(k0 + doff), "l"(src + D) : "memory");
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(v0 + doff), "l"(src + 2 * D) : "memory");
        } else {
          asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};\n" ::"r"(q0 + doff), "r"(0) : "memory");
          asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};\n" ::"r"(k0 + doff), "r"(0) : "memory");
          asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};\n" ::"r"(v0 + doff), "r"(0) : "memory");
        }
      }
    }
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncthreads();
    if (COS) {   // F.normalize(q), F.normalize(k) per head (eps 1e-12) as fp32 factors
      for (int idx = threadIdx.x; idx < nfill * NHL * 2; idx += 256) {
        const int r = idx / (NHL * 2), rem = idx - r * (NHL * 2), hl = rem >> 1, isk = rem & 1;
        const uint4* p = reinterpret_cast<const uint4*>((isk ? sK : sQ) + r * LD + hl * DH);
        const uint4 a = p[0], b4 = p[1];
        const uint32_t w[8] = {a.x, a.y, a.z, a.w, b4.x, b4.y, b4.z, b4.w};
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < 8; i++) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
          ss = fmaf(f.x, f.x, fmaf(f.y, f.y, ss));
        }
        (isk ? sInvK : sInvQ)[hl * NROW + r] = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
      }
      __syncthreads();
    }
#pragma unroll 1
    for (int item = warp; item < sNumTiles * NHL; item += 8) {   // (q-tile, head) items, round-robin over the warps
      const int tk = item / NHL, hl = item - tk * NHL;
      const int row = sTileRow[tk], kb = sTileKb[tk], ke = sTileKe[tk];
      const int n = ke - kb;
      const int r0 = row + g4, r1 = r0 + 8;
      const int tok0 = r0 < ke ? sTok[r0] : -1, tok1 = r1 < ke ? sTok[r1] : -1;
      const uint32_t kwin = k0 + (uint32_t)((kb * LD + hl * DH) * 2) + klane, vwin = v0 + (uint32_t)((kb * LD + hl * DH) * 2) + vlane;
      uint32_t qa[4];
      asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                   : "=r"(qa[0]), "=r"(qa[1]), "=r"(qa[2]), "=r"(qa[3])
                   : "r"(q0 + (uint32_t)((row * LD + hl * DH) * 2) + vlane));
      float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      float ol[4] = {0.f, 0.f, 0.f, 0.f};
      float m0 = -INFINITY, m1 = -INFINITY;
      float s0r = sl2, s1r = sl2;   // log2(e) x logit scale of this lane's two query rows
      if (COS) {
        const int h = hs * NHL + hl;
        const float it = 1.4426950408889634f / fmaxf(tau_n > 1 ? tau[h] : tau[0], tau_min);
        s0r = it * sInvQ[hl * NROW + min(r0, NROW - 1)];
        s1r = it * sInvQ[hl * NROW + min(r1, NROW - 1)];
      }
      const float* ikw = COS ? sInvK + hl * NROW + kb : nullptr;
#pragma unroll 1
      for (int off = 0; off < n; off += ATT_KCHUNK) {
        const int rem = n - off;   // warp-uniform
        const uint32_t ka = kwin + (uint32_t)(off * LD * 2), va = vwin + (uint32_t)(off * LD * 2);
        const float* ik = COS ? ikw + off : nullptr;
        if (rem > 48) attn_chunk<8, LD, COS>(qa, ka, va, rem, t4, g4 == 0, s0r, s1r, ik, off == 0, m0, m1, o, ol);
        else if (rem > 32) attn_chunk<6, LD, COS>(qa, ka, va, rem, t4, g4 == 0, s0r, s1r, ik, off == 0, m0, m1, o, ol);
        else if (rem > 16) attn_chunk<4, LD, COS>(qa, ka, va, rem, t4, g4 == 0, s0r, s1r, ik, off == 0, m0, m1, o, ol);
        else attn_chunk<2, LD, COS>(qa, ka, va, rem, t4, g4 == 0, s0r, s1r, ik, off == 0, m0, m1, o, ol);
      }
      const float l0 = __shfl_sync(0xffffffffu, ol[0], lane & ~3), l1 = __shfl_sync(0xffffffffu, ol[2], lane & ~3);
      if (tok0 >= 0) {
        uint32_t* op0 = reinterpret_cast<uint32_t*>(out + (size_t)tok0 * D + (hs * NHL + hl) * DH);
        const float i0 = __fdividef(1.0f, l0);
        op0[t4] = (OUT_BF16 ? pack_bf16 : pack_f16)(o[0][0] * i0, o[0][1] * i0);
        op0[t4 + 4] = (OUT_BF16 ? pack_bf16 : pack_f16)(o[1][0] * i0, o[1][1] * i0);
      }
      if (tok1 >= 0) {
        uint32_t* op1 = reinterpret_cast<uint32_t*>(out + (size_t)tok1 * D + (hs * NHL + hl) * DH);
        const float i1 = __fdividef(1.0f, l1);
        op1[t4] = (OUT_BF16 ? pack_bf16 : pack_f16)(o[0][2] * i1, o[0][3] * i1);
        op1[t4 + 4] = (OUT_BF16 ? pack_bf16 : pack_f16)(o[1][2] * i1, o[1][3] * i1);
      }
    }
  }
}

// win_batch: the per-batch records of win_batch_kernel ({first window, end window, first slot, end slot}), n_cap = the token
// capacity the window plan was built for (bounds the record array).  out: [n, 128] attention output in flat token order, IEEE fp16
// (inference) or bf16 (out_bf16: training path).  tau != nullptr: cosine attention with tau_n (1 or 8) temperatures.
static inline int sstb_win_attn_batch(sstb200_ctx* c, const __half* qkv, const int32_t* counters, const int32_t* win_offsets,
                                      const int32_t* win_batch, int n_cap, const int32_t* tok_perm, void* out_v, bool out_bf16 = false,
                                      const float* tau = nullptr, int tau_n = 0, float tau_min = 0.f) {
  constexpr int NHL = 2;   // heads per CTA -> 4 CTAs per window batch
  constexpr int CTAS_PER_SM = 9;   // grid of the persistent unit loop
  const int rec_cap = att_rec_cap(n_cap);
  __half* out = reinterpret_cast<__half*>(out_v);
  const int4* recs = reinterpret_cast<const int4*>(win_batch);
  size_t smem = (size_t)3 * (ATT_BT + 16) * (NHL * 16 + 8) * sizeof(__half);
  static SmemAttr sa, sb, sc, sd;
  auto* kern = out_bf16 ? (tau ? win_attn_batch_kernel<NHL, true, true> : win_attn_batch_kernel<NHL, true, false>)
                        : (tau ? win_attn_batch_kernel<NHL, false, true> : win_attn_batch_kernel<NHL, false, false>);
  SmemAttr& attr = out_bf16 ? (tau ? sd : sb) : (tau ? sc : sa);
  CUDA_TRY(c, ensure_smem(c, attr, kern, smem));
  const int grid = c->num_sms * CTAS_PER_SM;
  CUDA_TRY(c, launch_pdl(kern, dim3(grid), dim3(256), smem, c->stream, qkv, counters, win_offsets, recs, rec_cap, tok_perm, 0.25f, tau, tau_n,
                         tau_min, out));
  return SSTB_OK;
}
