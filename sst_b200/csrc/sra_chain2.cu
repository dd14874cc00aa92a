// Fused post-attention chain of one SRA encoder layer (d_model = 128, dim_ff = 256, post-norm LayerNorm or eval BatchNorm, GELU):
//
//     x1 = Norm1(x + att . Wo^T + bo)               GEMM1  [128 x 128] x [128 x 128]
//     h  = GELU(x1 . W1^T + b1)                     GEMM2  [128 x 128] x [128 x 256]   two N = 128 chunks
//     y  = Norm2(x1 + h . W2^T + b2)                GEMM3  [128 x 256] x [256 x 128]   two K = 128 chunks
//     q|k|v (next layer) = (y + pos | y) . Wqkv^T   GEMM4  [128 x 128] x [128 x 384]   three N = 128 chunks (optional tail)
//
// replaces mmdet3d/models/sst/sst_basic_block_v2.py:104-126 (+ the in-projection of the following layer's
// nn.MultiheadAttention, :70) for one 128-token tile per iteration of a persistent CTA.
//
// Two warpgroups, each owning 64 rows of the tile, issue wgmma.mma_async (fp16 operands, fp32 accumulators in registers) in
// ping-pong: both consume one sequence of weight chunks in the same order, and warpgroup 1 issues its MMA on a chunk only after
// warpgroup 0's MMA on it has retired, so one warpgroup's epilogue (bias, residual, LayerNorm, GELU, positional add, stores) runs
// while the other's MMA occupies the tensor core.  Weights arrive by cp.async.bulk.tensor (TMA) as 32 KB chunks ([128 rows x
// 128 K]) into a ring of three 128B-swizzled slots with per-slot mbarriers: "full" (TMA bytes landed) and "warpgroup 0 done".
// Warpgroup 1 is the last reader of every slot; one of its threads refills the slot with the chunk three ahead (also across
// tiles), which by itself bounds how far warpgroup 0 runs ahead.  Each warpgroup streams its own 64-row half of the attention
// tile by TMA, issued one tile ahead, and loads its residual rows and positional codes while its GEMM1 is in flight.  The
// scheduling unit stays the 128-row tile: both warpgroups walk every tile of the CTA and wait on and release every chunk, also
// when their half has no valid rows.  Inside a warpgroup, epilogue writes that feed the next wgmma are ordered by
// fence.proxy.async and a named barrier; the tile loop has no CTA-wide barrier.
// Epilogues run on the accumulator fragments: a row's 128 columns sit in one lane quad, so LayerNorm statistics take two
// xor-shuffles; x1 stays in registers from GEMM1 to GEMM3; x1, h, y and y + pos reach the next GEMM as 16-bit operands written
// into the swizzled K-major layout by stmatrix, 16 columns of a warp's 16 rows per instruction.  Only x (residual), y and q|k|v
// touch global memory; each warp writes its 16 rows of a q|k|v chunk into shared memory the same way and copies them out as whole
// 256-byte row segments.  All rows are in flat token order.
//
// Shared memory, per warpgroup (64 rows, K-major, 128B swizzle, 8 KB per 64-wide K block): X 16 KB (x1, then y) | T 16 KB (att) |
// H 32 KB (hidden, four K blocks; y + pos aliased onto its first 16 KB once GEMM3 has retired, q|k|v staged in its upper 16 KB);
// then the ring, 3 x 32 KB.
#include <stdarg.h>
#include <cuda_fp16.h>
#include "sra.cuh"
#include "tma.cuh"

namespace {

constexpr int TM = 128, HM = 64, D = 128;
constexpr int SLOT = 32768;   // one weight chunk: 128 rows x 128 K fp16 = two 64-wide swizzle blocks of 16 KB
constexpr int NSLOT = 3;
constexpr int WG_BYTES = 2 * SLOT;   // one warpgroup's operands
constexpr int OFF_X = 0, OFF_T = SLOT / 2, OFF_H = SLOT, OFF_RING = 2 * WG_BYTES;
constexpr int SMEM_BYTES = OFF_RING + NSLOT * SLOT + 1024;
static_assert(SMEM_BYTES <= 232448, "sra_chain2 shared memory exceeds the sm_90 per-block limit");
constexpr int NTHR = 256;
constexpr uint32_t OPB = TM * 128;   // byte pitch of one 64-wide K block of a weight chunk (128 rows)
constexpr uint32_t OPH = HM * 128;   // byte pitch of one 64-wide K block of a warpgroup's 64-row operand

struct Chain2Maps {
  CUtensorMap att, wo, w1, w2, wqkv;
};

struct Chain2Args {
  const float* x;
  float* y;
  __half* qkv;                   // [tokens, 384] next layer's q|k|v (tail only)
  // norm: LayerNorm (g1/be1/g2/be2 = weight, bias) or eval-mode BatchNorm (affine: g* = folded scale, be* = folded shift)
  const float *bo, *b1, *b2, *g1, *be1, *g2, *be2, *bqkv;
  float eps;
  int affine;
  int M_cap;
  const int32_t* M_dev;
  // next layer's per-axis positional table, added to y for the q|k chunks.  Columns [32 grp, 32 grp + 32) lie inside one axis
  // (posL % 32 == 0): pos_grp[grp] is that axis's first table row shifted back by the axis's first column, or null past the last
  // axis; byte grp of pos_shift is 8 x the axis, the position of the row's code for it in pos_code.
  const float* pos_grp[4];
  const int32_t* pos_code;
  int posL;
  int pos_shift;
};

// chunk j of a tile: 0 Wo | 1, 2 W1 rows 0-127, 128-255 | 3, 4 W2 K 0-127, 128-255 | 5, 6, 7 Wqkv rows 0-127, 128-255, 256-383
__device__ __forceinline__ void issue_chunk(const Chain2Maps& m, int j, uint32_t dst, uint32_t bar) {
  const CUtensorMap* map = &m.wqkv;
  int k0 = 0, n0 = 0;
  if (j == 0) map = &m.wo;
  else if (j <= 2) map = &m.w1, n0 = (j - 1) * 128;
  else if (j <= 4) map = &m.w2, k0 = (j - 3) * 128;
  else n0 = (j - 5) * 128;
  mbar_expect_tx(bar, SLOT);
  tma_load_2d(dst, map, k0, n0, bar);
  tma_load_2d(dst + SLOT / 2, map, k0 + 64, n0, bar);
}

// Columns 16 p .. 16 p + 15 of fragment t (pairs 2p and 2p + 1 of rows ra and rb) as 16-bit operand pieces, by one stmatrix.x4
// at the lane's stsm_base `ob` of a 64-row operand (format in wgmma.cuh).
__device__ __forceinline__ void st_op16(uint32_t ob, int p, const float (&t)[64]) {
  stsm_x4(ob, p, OPH, pack_f16(t[8 * p], t[8 * p + 1]), pack_f16(t[8 * p + 2], t[8 * p + 3]), pack_f16(t[8 * p + 4], t[8 * p + 5]),
          pack_f16(t[8 * p + 6], t[8 * p + 7]));
}

// columns 8 j + cq, cq + 1 of a row whose pointer `p` already includes the lane's cq: one base address, j an immediate offset
__device__ __forceinline__ float2 ldg2(const float* p, int j) { return __ldg(reinterpret_cast<const float2*>(p + 8 * j)); }

// t = fragment of [64 rows x 128] (rows ra: t[4j], t[4j+1]; rb: t[4j+2], t[4j+3]; columns 8j + 2 (lane & 3)): per-row normalisation.
// LayerNorm statistics take two passes over the register-resident rows, the mean and then the sum of centred squares, so a large
// common offset in a row does not cancel the variance away as E[t^2] - mean^2 would.
__device__ __forceinline__ void row_norm(float (&t)[64], const float* __restrict__ gam, const float* __restrict__ bet, float eps, bool affine) {
  const int cq = 2 * (threadIdx.x & 3);
  gam += cq, bet += cq;
  if (affine) {   // eval BatchNorm folded to one scale and shift per channel
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const float2 g2 = ldg2(gam, j), b2 = ldg2(bet, j);
      t[4 * j] = fmaf(t[4 * j], g2.x, b2.x);
      t[4 * j + 1] = fmaf(t[4 * j + 1], g2.y, b2.y);
      t[4 * j + 2] = fmaf(t[4 * j + 2], g2.x, b2.x);
      t[4 * j + 3] = fmaf(t[4 * j + 3], g2.y, b2.y);
    }
    return;
  }
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int j = 0; j < 16; j++) {
    s0 += t[4 * j] + t[4 * j + 1];
    s1 += t[4 * j + 2] + t[4 * j + 3];
  }
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  const float mean0 = s0 * (1.f / D), mean1 = s1 * (1.f / D);
  float q0 = 0.f, q1 = 0.f;
#pragma unroll
  for (int j = 0; j < 16; j++) {
    t[4 * j] -= mean0, t[4 * j + 1] -= mean0, t[4 * j + 2] -= mean1, t[4 * j + 3] -= mean1;
    q0 = fmaf(t[4 * j], t[4 * j], fmaf(t[4 * j + 1], t[4 * j + 1], q0));
    q1 = fmaf(t[4 * j + 2], t[4 * j + 2], fmaf(t[4 * j + 3], t[4 * j + 3], q1));
  }
#pragma unroll
  for (int o = 1; o < 4; o <<= 1) {
    q0 += __shfl_xor_sync(0xffffffffu, q0, o);
    q1 += __shfl_xor_sync(0xffffffffu, q1, o);
  }
  const float rstd0 = rsqrtf(q0 * (1.f / D) + eps), rstd1 = rsqrtf(q1 * (1.f / D) + eps);
#pragma unroll
  for (int j = 0; j < 16; j++) {
    const float2 g2 = ldg2(gam, j), b2 = ldg2(bet, j);
    t[4 * j] = fmaf(t[4 * j] * rstd0, g2.x, b2.x);
    t[4 * j + 1] = fmaf(t[4 * j + 1] * rstd0, g2.y, b2.y);
    t[4 * j + 2] = fmaf(t[4 * j + 2] * rstd1, g2.x, b2.x);
    t[4 * j + 3] = fmaf(t[4 * j + 3] * rstd1, g2.y, b2.y);
  }
}

// Positional table row of one row (positional code `code`) for the 32 columns [32 grp, 32 grp + 32), offset by the lane's cq:
// column 8 j + cq adds ldg2(pos_row(...), j).  Only for groups with g.pos_grp[grp] set.
__device__ __forceinline__ const float* pos_row(const Chain2Args& g, int code, int grp, int cq) {
  const int cv = (code >> ((g.pos_shift >> (8 * grp)) & 255)) & 255;
  return g.pos_grp[grp] + (cv * g.posL + cq);
}

template <bool TAIL>
__global__ void __launch_bounds__(NTHR, 1) sra_chain2_kernel(const __grid_constant__ Chain2Maps m, const Chain2Args g) {
  extern __shared__ uint8_t chain_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)chain_raw + 1023) & ~(uintptr_t)1023);
  const int tid = threadIdx.x, wg = tid >> 7, lane = tid & 31;
  const uint32_t sX = smem_u32(base + wg * WG_BYTES + OFF_X), sT = smem_u32(base + wg * WG_BYTES + OFF_T);
  const uint32_t sH = smem_u32(base + wg * WG_BYTES + OFF_H), sR = smem_u32(base + OFF_RING);
  __shared__ __align__(8) uint64_t bar_full[NSLOT], bar_wg0[NSLOT], bar_att[2];
  constexpr int NCH = TAIL ? 8 : 5;
  static_assert(NCH >= NSLOT, "the chunks loaded before the dependency wait all belong to the CTA's first tile");

  // Before the wait on the preceding kernel: barrier set-up and the first NSLOT weight chunks, all of the CTA's first tile, so the
  // weight fetch overlaps the tail of the attention kernel.  This is safe because the 16-bit weights are written only by the cast
  // when a layer's weights are (re)made, which completes before the first kernel of a forward pass starts, and no kernel of the
  // pass writes them.  Everything the preceding kernels produce (attention output, residual rows, row count, folded BatchNorm)
  // is read after the wait.  The grid has at most one CTA per tile of the capacity, so every CTA has a first tile unless the
  // device-side row count is smaller.
  if (tid == 0) {
    for (int s = 0; s < NSLOT; s++) {
      mbar_init(smem_u32(&bar_full[s]), 1);
      mbar_init(smem_u32(&bar_wg0[s]), 1);
    }
    mbar_init(smem_u32(&bar_att[0]), 1);
    mbar_init(smem_u32(&bar_att[1]), 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    for (int n = 0; n < NSLOT; n++) issue_chunk(m, n, sR + n * SLOT, smem_u32(&bar_full[n]));
  }
  pdl_wait();
  pdl_launch();

  const int M = g.M_dev ? *g.M_dev : g.M_cap;
  const int ntiles = (M + TM - 1) / TM;
  if ((int)blockIdx.x >= ntiles) {   // uniform per CTA: no tile, but the weight loads above must land before the CTA exits
    if (tid == 0)
      for (int s = 0; s < NSLOT; s++) mbar_wait(smem_u32(&bar_full[s]), 0);
    return;
  }
  // chunk `n` (counted over the CTA's whole tile sequence) belongs to a tile this CTA will process
  auto chunk_live = [&](int n) { return (int)blockIdx.x + (n / NCH) * (int)gridDim.x < ntiles; };
  const bool leader = (tid & 127) == 0;   // one elected thread per warpgroup
  // this warpgroup's half of the attention tile `tile`; a half that lies wholly past the tensor's rows only completes the phase
  auto issue_att = [&](int tile) {
    const uint32_t bar = smem_u32(&bar_att[wg]);
    const int r0 = tile * TM + wg * HM;
    if (r0 < g.M_cap) {
      mbar_expect_tx(bar, SLOT / 2);
      tma_load_2d(sT, &m.att, 0, r0, bar);
      tma_load_2d(sT + OPH, &m.att, 64, r0, bar);
    } else {
      mbar_arrive(bar);
    }
  };
  __syncthreads();
  if (leader) issue_att(blockIdx.x);

  int gc = 0;   // weight chunks consumed
  // slot of chunk gc + i once it has landed; warpgroup 1 also waits until warpgroup 0's MMA on it has retired
  auto acquire = [&](int i) -> uint32_t {
    const int n = gc + i, s = n % NSLOT;
    const uint32_t par = (uint32_t)((n / NSLOT) & 1);
    mbar_wait(smem_u32(&bar_full[s]), par);
    if (wg == 1) mbar_wait(smem_u32(&bar_wg0[s]), par);
    return sR + s * SLOT;
  };
  // after wgmma_wait<0>: once every warp of the warpgroup has passed the barrier, its MMAs have retired, so its own operand
  // buffers may be overwritten and the next `cnt` chunks released.  Warpgroup 0 signals it is done with them; warpgroup 1,
  // their last reader, refills each slot with the chunk three ahead.
  auto release = [&](int cnt) {
    named_bar_sync(1 + wg, 128);
    if (wg == 0) {
      if (leader)
        for (int i = 0; i < cnt; i++) mbar_arrive(smem_u32(&bar_wg0[(gc + i) % NSLOT]));
    } else {
      if (leader)
        for (int i = 0; i < cnt; i++)
          if (chunk_live(gc + i + NSLOT)) {
            const int s = (gc + i) % NSLOT;
            issue_chunk(m, (gc + i + NSLOT) % NCH, sR + s * SLOT, smem_u32(&bar_full[s]));
          }
    }
    gc += cnt;
  };
  auto wg_sync = [&]() {   // this warpgroup's generic-proxy shared-memory writes -> its next wgmma
    fence_async_smem();
    named_bar_sync(1 + wg, 128);
  };

  const int rl = 16 * ((tid >> 5) & 3) + (lane >> 2);   // fragment rows rl, rl + 8 of this warpgroup's half
  const int cq = 2 * (lane & 3);
  const uint32_t oX = stsm_base(sX), oH = oX + (OFF_H - OFF_X);   // this lane's stmatrix row addresses in X and H
  uint32_t att_par = 0;
  float acc[64], x1[64];
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int rowA = tile * TM + wg * HM + rl, rowB = rowA + 8;
    const bool okA = rowA < M, okB = rowB < M;

    // ---- GEMM1 + bias + residual + Norm1 -> x1 (registers, and fp16 into X) -----------------------------------------------------
    {
      const uint32_t w = acquire(0);
      mbar_wait(smem_u32(&bar_att[wg]), att_par);
      att_par ^= 1u;
      wg_tile_mma<128, false, 8>(acc, sT, OPH, w, OPB, false);
    }
    // residual rows and positional codes load while the MMA runs
    const float* xA = g.x + (size_t)rowA * D + cq;   // row rb is 8 rows further
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const float2 ra = okA ? *reinterpret_cast<const float2*>(xA + 8 * j) : make_float2(0.f, 0.f);
      const float2 rb = okB ? *reinterpret_cast<const float2*>(xA + 8 * D + 8 * j) : make_float2(0.f, 0.f);
      x1[4 * j] = ra.x, x1[4 * j + 1] = ra.y, x1[4 * j + 2] = rb.x, x1[4 * j + 3] = rb.y;
    }
    int codeA = 0, codeB = 0;
    if (TAIL) {
      codeA = okA ? g.pos_code[rowA] : 0;
      codeB = okB ? g.pos_code[rowB] : 0;
    }
    wgmma_wait<0>();
    release(1);
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const float2 b = ldg2(g.bo + cq, j);
      x1[4 * j] = acc[4 * j] + b.x + x1[4 * j];
      x1[4 * j + 1] = acc[4 * j + 1] + b.y + x1[4 * j + 1];
      x1[4 * j + 2] = acc[4 * j + 2] + b.x + x1[4 * j + 2];
      x1[4 * j + 3] = acc[4 * j + 3] + b.y + x1[4 * j + 3];
    }
    row_norm(x1, g.g1, g.be1, g.eps, g.affine);
#pragma unroll
    for (int p = 0; p < 8; p++) st_op16(oX, p, x1);
    wg_sync();   // also: every warp of this warpgroup has retired GEMM1, so T is free for the next tile's attention half
    if (leader && tile + (int)gridDim.x < ntiles) issue_att(tile + gridDim.x);

    // ---- GEMM2 + bias + GELU -> h (fp16 into H) -----------------------------------------------------------------------------------
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
      wg_tile_mma<128, false, 8>(acc, sX, OPH, acquire(0), OPB, false);
      wgmma_wait<0>();
      release(1);
#pragma unroll
      for (int p = 0; p < 8; p++) {
        uint32_t v[4];
#pragma unroll
        for (int i = 0; i < 2; i++) {
          const int j = 2 * p + i;
          const float2 b = ldg2(g.b1 + 128 * h + cq, j);
          v[2 * i] = pack_f16(gelu_ex2(acc[4 * j] + b.x), gelu_ex2(acc[4 * j + 1] + b.y));
          v[2 * i + 1] = pack_f16(gelu_ex2(acc[4 * j + 2] + b.x), gelu_ex2(acc[4 * j + 3] + b.y));
        }
        stsm_x4(oH + h * 2 * OPH, p, OPH, v[0], v[1], v[2], v[3]);
      }
    }
    wg_sync();

    // ---- GEMM3 (both K chunks back to back) + bias + x1 + Norm2 -> y (fp32 rows; fp16 y into X and y + pos into H for the tail) --
    // the accumulators start at x1 + b2, so the MMA adds the residual and the bias and x1 is dead once it is issued
#pragma unroll
    for (int j = 0; j < 16; j++) {
      const float2 b = ldg2(g.b2 + cq, j);
      acc[4 * j] = x1[4 * j] + b.x;
      acc[4 * j + 1] = x1[4 * j + 1] + b.y;
      acc[4 * j + 2] = x1[4 * j + 2] + b.x;
      acc[4 * j + 3] = x1[4 * j + 3] + b.y;
    }
    {
      const uint32_t w0 = acquire(0), w1 = acquire(1);
      wg_tile_mma<128, false, 8>(acc, sH, OPH, w0, OPB, true);
      wg_tile_mma<128, false, 8>(acc, sH + 2 * OPH, OPH, w1, OPB, true);
      wgmma_wait<0>();
      release(2);
    }
    row_norm(acc, g.g2, g.be2, g.eps, g.affine);
    {
      float* yA = g.y + (size_t)rowA * D + cq;   // row rb is 8 rows further
#pragma unroll
      for (int j = 0; j < 16; j++) {
        if (okA) *reinterpret_cast<float2*>(yA + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
        if (okB) *reinterpret_cast<float2*>(yA + 8 * D + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    if constexpr (TAIL) {   // y -> X, y + pos -> H, then GEMM4
#pragma unroll
      for (int p = 0; p < 8; p++) st_op16(oX, p, acc);
#pragma unroll
      for (int grp = 0; grp < 4; grp++) {
        const bool has = g.pos_grp[grp] != nullptr;   // uniform
        const float* posA = pos_row(g, codeA, grp, cq);
        const float* posB = pos_row(g, codeB, grp, cq);
#pragma unroll
        for (int p = 2 * grp; p < 2 * grp + 2; p++) {
          uint32_t v[4];
#pragma unroll
          for (int i = 0; i < 2; i++) {
            const int j = 2 * p + i;
            const float2 pa = has ? ldg2(posA, j) : make_float2(0.f, 0.f);
            const float2 pb = has ? ldg2(posB, j) : make_float2(0.f, 0.f);
            v[2 * i] = pack_f16(acc[4 * j] + pa.x, acc[4 * j + 1] + pa.y);
            v[2 * i + 1] = pack_f16(acc[4 * j + 2] + pb.x, acc[4 * j + 3] + pb.y);
          }
          stsm_x4(oH, p, OPH, v[0], v[1], v[2], v[3]);
        }
      }
      wg_sync();

      // ---- GEMM4: next layer's q|k (from y + pos) and v (from y) + bias -> fp16 rows ----------------------------------------------
      // Each warp stages its 16 rows of a chunk in H's upper 16 KB (free: y + pos fills the lower half) and copies them out itself:
      // per step, lanes 0-15 and 16-31 each store one row's 256 contiguous bytes.  Lane piece (lane & 15) of rows rq + 2 i.
      const int rw = 16 * ((tid >> 5) & 3) + (lane >> 4), rq = tile * TM + wg * HM + rw;
      __half* gq = g.qkv + (size_t)rq * 3 * D + 8 * (lane & 15);
      const uint32_t sq = sH + 2 * OPH + ((lane >> 3) & 1) * OPH + rw * 128 + (((lane & 7) ^ (lane >> 4)) << 4);
#pragma unroll 1
      for (int q = 0; q < 3; q++) {
        wg_tile_mma<128, false, 8>(acc, q < 2 ? sH : sX, OPH, acquire(0), OPB, false);
        wgmma_wait<0>();
        release(1);
#pragma unroll
        for (int p = 0; p < 8; p++) {
          uint32_t v[4];
#pragma unroll
          for (int i = 0; i < 2; i++) {
            const int j = 2 * p + i;
            const float2 b = ldg2(g.bqkv + 128 * q + cq, j);
            v[2 * i] = pack_f16(acc[4 * j] + b.x, acc[4 * j + 1] + b.y);
            v[2 * i + 1] = pack_f16(acc[4 * j + 2] + b.x, acc[4 * j + 3] + b.y);
          }
          stsm_x4(oH + 2 * OPH, p, OPH, v[0], v[1], v[2], v[3]);
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 8; i++) {   // row rq + 2 i sits at row & 7 = (2 i + (lane >> 4)) & 7 of its swizzle atom
          uint4 v;
          asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];\n"
                       : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                       : "r"((sq ^ ((uint32_t)(2 * i & 7) << 4)) + 256 * i)
                       : "memory");
          if (rq + 2 * i < M) *reinterpret_cast<uint4*>(gq + (size_t)2 * i * 3 * D + 128 * q) = v;
        }
      }
    }
  }
}

// eval-mode BatchNorm of layer_cfg use_bn folded to y = x s + t per channel: out[l][4][128] = {s1, t1, s2, t2}
struct BnFoldArgs {
  const float* p[8][8];   // per layer: norm1 w, b, mean, var, norm2 w, b, mean, var
  float eps[8];
};
__global__ void __launch_bounds__(128) bn_fold_kernel(BnFoldArgs a, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  const int l = blockIdx.x, c = threadIdx.x;
#pragma unroll
  for (int n = 0; n < 2; n++) {
    const float* const* q = a.p[l] + 4 * n;
    if (!q[2]) continue;   // LayerNorm layer
    const float sc = q[0][c] * rsqrtf(q[3][c] + a.eps[l]);
    out[((size_t)l * 4 + 2 * n) * 128 + c] = sc;
    out[((size_t)l * 4 + 2 * n + 1) * 128 + c] = q[1][c] - q[2][c] * sc;
  }
}

}  // namespace

int sstb_sra_bn_fold(sstb200_ctx* c, const sstb200_sra_layer* layers, int num_layers, float* out) {
  for (int l0 = 0; l0 < num_layers; l0 += 8) {
    BnFoldArgs a;
    memset(&a, 0, sizeof(a));
    const int nl = num_layers - l0 < 8 ? num_layers - l0 : 8;
    for (int l = 0; l < nl; l++) {
      const sstb200_sra_layer* L = &layers[l0 + l];
      const float* src[8] = {L->norm1_w, L->norm1_b, L->norm1_mean, L->norm1_var, L->norm2_w, L->norm2_b, L->norm2_mean, L->norm2_var};
      for (int i = 0; i < 8; i++) a.p[l][i] = src[i];
      a.eps[l] = L->norm_eps;
    }
    CUDA_TRY(c, launch_pdl(bn_fold_kernel, dim3(nl), dim3(128), (size_t)0, c->stream, a, out + (size_t)l0 * 4 * 128));
  }
  return SSTB_OK;
}

int sstb_sra_chain2(sstb200_ctx* c, const sstb200_sra_layer* L, const __half* att, const float* x, float* y, int n_cap, const int32_t* n_dev,
                    const sstb200_sra_layer* next, const sstb200_sra_plan* next_plan, void* next_qkv, const float* bn_fold) {
  Chain2Maps maps;
  Chain2Args g;
  memset(&g, 0, sizeof(g));
  memset(&maps, 0, sizeof(maps));
  const bool tail = next && next_plan && next_qkv;
  if (tail && (!next_plan->pos_table || !next_plan->pos_code || next_plan->pos_L <= 0 || next_plan->pos_L % 32 != 0 || next_plan->pos_ndim < 1 ||
               next_plan->pos_ndim > 3))
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "fused QKV tail needs the next plan's positional table with a per-axis length that is a multiple of 32");
  int rc = 0;
  rc |= tmap_2d_sw128(&maps.att, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, att, 128, (uint64_t)n_cap, 256, 64, HM);   // per-warpgroup halves
  rc |= tmap_2d_sw128(&maps.wo, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L->out_proj_w_f16, 128, 128, 256, 64, 128);
  rc |= tmap_2d_sw128(&maps.w1, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L->lin1_w_f16, 128, 256, 256, 64, 128);
  rc |= tmap_2d_sw128(&maps.w2, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, L->lin2_w_f16, 256, 128, 512, 64, 128);
  if (tail) {
    rc |= tmap_2d_sw128(&maps.wqkv, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, next->in_proj_w_f16, 128, 384, 256, 64, 128);
    g.qkv = reinterpret_cast<__half*>(next_qkv);
    g.bqkv = next->in_proj_b;
    g.pos_code = next_plan->pos_code;
    g.posL = next_plan->pos_L;
    for (int grp = 0; grp < 4; grp++) {   // table [ndim][maxw][posL]: row (axis, cv) at (axis maxw + cv) posL, its columns from axis posL on
      const int axis = 32 * grp / g.posL;
      if (axis >= next_plan->pos_ndim) continue;
      g.pos_grp[grp] = next_plan->pos_table + (size_t)axis * (next_plan->pos_maxw - 1) * g.posL;
      g.pos_shift |= (8 * axis) << (8 * grp);
    }
  }
  if (rc) return sstb_fail(c, SSTB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d): operands must be 16-byte aligned", rc);
  g.x = x;
  g.y = y;
  g.bo = L->out_proj_b;
  g.b1 = L->lin1_b;
  g.b2 = L->lin2_b;
  const bool bn = L->norm1_mean != nullptr;
  if (bn && !bn_fold) return sstb_fail(c, SSTB_ERR_ARG, "BatchNorm layer without folded scale / shift (sstb_sra_bn_fold)");
  g.g1 = bn ? bn_fold : L->norm1_w;
  g.be1 = bn ? bn_fold + 128 : L->norm1_b;
  g.g2 = bn ? bn_fold + 256 : L->norm2_w;
  g.be2 = bn ? bn_fold + 384 : L->norm2_b;
  g.affine = bn;
  g.eps = L->norm_eps;
  g.M_cap = n_cap;
  g.M_dev = n_dev;
  static SmemAttr sa[2];
  void (*kern)(const Chain2Maps, const Chain2Args) = tail ? sra_chain2_kernel<true> : sra_chain2_kernel<false>;
  CUDA_TRY(c, ensure_smem(c, sa[tail ? 1 : 0], kern, (size_t)SMEM_BYTES));
  const int tiles_cap = (n_cap + TM - 1) / TM;
  const int grid = c->num_sms < tiles_cap ? c->num_sms : tiles_cap;
  CUDA_TRY(c, launch_pdl(kern, dim3(grid), dim3(NTHR), (size_t)SMEM_BYTES, c->stream, maps, g));
  return SSTB_OK;
}
