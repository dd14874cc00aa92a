// Sparse 3-D convolution (SURVEY 8f next-1): SubMConv3d / SparseConv3d / SparseInverseConv3d of the reference's sparse U-Nets
// (mmdet3d/models/middle_encoders/sparse_unet.py:15-505, mmdet3d/ops/sparse_block.py:81-289), which the reference delegates to spconv
// (vendored v1: mmdet3d/ops/spconv/include/spconv/geometry.h:25-301 builds the index pairs, spconv_ops.h:95-260 runs one gather ->
// GEMM -> scatter-add per kernel offset).
//
// Form: OUTPUT-STATIONARY.  The rulebook is a neighbour table nbr[o][k] = input row that feeds output row o through kernel
// offset k (or -1), built from the bitmap-rank index of the active coordinates (no hash table, no sort, no atomics on features); a
// convolution is then ONE implicit-GEMM launch: an output tile gathers its <= KV input rows per offset, accumulates all offsets
// in registers and applies the folded BatchNorm (+ residual) (+ ReLU) epilogue before its single store.  The reference's
// form writes every output row KV times with atomics-free but serialised scatter-adds and keeps BN / ReLU / residual as separate
// passes over [N, C].
#include <stdarg.h>
#include <cuda_fp16.h>
#include "index.cuh"
#include "wgmma.cuh"
#include "rows.cuh"

namespace {

struct SpGeom {
  int B;
  int in_shape[3];   // z, y, x
  int out_shape[3];
  int ks[3], st[3], pd[3];
  int KV;
};

__device__ __forceinline__ int sp_rank(const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ word_prefix, long long key) {
  const size_t w = (size_t)(key >> 5);
  const uint32_t bit = 1u << (key & 31);
  const uint32_t word = bitmap[w];
  if (!(word & bit)) return -1;
  return (int)(word_prefix[w] + __popc(word & (bit - 1u)));
}

// perm[rank(row i)] = i  (rows are unique: a permutation)
__global__ void sp_perm_kernel(const long long* __restrict__ keys, int n, const int32_t* __restrict__ n_dev,
                               const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ word_prefix, int32_t* __restrict__ perm) {
  pdl_wait();
  pdl_launch();
  if (n_dev) n = min(n, *n_dev);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long key = keys[i];
  if (key < 0) return;
  const int r = sp_rank(bitmap, word_prefix, key);
  if (r >= 0) perm[r] = i;
}

// candidate outputs of a strided convolution: o = (i + pad - delta) / stride where divisible and inside the output grid
__global__ void sp_mark_out_kernel(const int32_t* __restrict__ coors, int n, SpGeom g, uint32_t* __restrict__ out_bitmap,
                                   int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n * g.KV) return;
  const int i = (int)(t / g.KV), k = (int)(t % g.KV);
  const int4 c = *reinterpret_cast<const int4*>(coors + (size_t)i * 4);  // b, z, y, x
  if (c.x < 0 || c.x >= g.B || c.y < 0 || c.y >= g.in_shape[0] || c.z < 0 || c.z >= g.in_shape[1] || c.w < 0 || c.w >= g.in_shape[2]) {
    if (k == 0) flags[1] = 1;
    return;
  }
  const int dz = k / (g.ks[1] * g.ks[2]), dy = (k / g.ks[2]) % g.ks[1], dx = k % g.ks[2];
  const int tz = c.y + g.pd[0] - dz, ty = c.z + g.pd[1] - dy, tx = c.w + g.pd[2] - dx;
  if (tz < 0 || ty < 0 || tx < 0) return;
  if (tz % g.st[0] || ty % g.st[1] || tx % g.st[2]) return;
  const int oz = tz / g.st[0], oy = ty / g.st[1], ox = tx / g.st[2];
  if (oz >= g.out_shape[0] || oy >= g.out_shape[1] || ox >= g.out_shape[2]) return;
  const long long key = (((long long)c.x * g.out_shape[0] + oz) * g.out_shape[1] + oy) * g.out_shape[2] + ox;
  bitmap_set(out_bitmap, key);
}

// nbr[o][k] = row of the input coordinate  o * stride - pad + delta_k  (or -1)
__global__ void sp_nbr_kernel(const int32_t* __restrict__ out_coors, int n_out, SpGeom g, const uint32_t* __restrict__ in_bitmap,
                              const uint32_t* __restrict__ in_prefix, const int32_t* __restrict__ in_perm, int32_t* __restrict__ nbr) {
  pdl_wait();
  pdl_launch();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n_out * g.KV) return;
  const int o = (int)(t / g.KV), k = (int)(t % g.KV);
  const int4 c = *reinterpret_cast<const int4*>(out_coors + (size_t)o * 4);
  int res = -1;
  if (c.x >= 0 && c.x < g.B && c.y >= 0 && c.z >= 0 && c.w >= 0) {
    const int dz = k / (g.ks[1] * g.ks[2]), dy = (k / g.ks[2]) % g.ks[1], dx = k % g.ks[2];
    const int iz = c.y * g.st[0] - g.pd[0] + dz, iy = c.z * g.st[1] - g.pd[1] + dy, ix = c.w * g.st[2] - g.pd[2] + dx;
    if (iz >= 0 && iz < g.in_shape[0] && iy >= 0 && iy < g.in_shape[1] && ix >= 0 && ix < g.in_shape[2]) {
      const long long key = (((long long)c.x * g.in_shape[0] + iz) * g.in_shape[1] + iy) * g.in_shape[2] + ix;
      const int r = sp_rank(in_bitmap, in_prefix, key);
      if (r >= 0) res = in_perm[r];
    }
  }
  nbr[t] = res;
}

// nbr_inv[i][k] = output row reached from input row i through offset k (the transposed table: SparseInverseConv3d), or -1
__global__ void sp_nbr_inv_kernel(const int32_t* __restrict__ in_coors, int n_in, SpGeom g, const uint32_t* __restrict__ out_bitmap,
                                  const uint32_t* __restrict__ out_prefix, const int32_t* __restrict__ out_perm,
                                  int32_t* __restrict__ nbr_inv) {
  pdl_wait();
  pdl_launch();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n_in * g.KV) return;
  const int i = (int)(t / g.KV), k = (int)(t % g.KV);
  const int4 c = *reinterpret_cast<const int4*>(in_coors + (size_t)i * 4);
  int res = -1;
  if (c.x >= 0 && c.x < g.B && c.y >= 0 && c.z >= 0 && c.w >= 0) {
    const int dz = k / (g.ks[1] * g.ks[2]), dy = (k / g.ks[2]) % g.ks[1], dx = k % g.ks[2];
    const int tz = c.y + g.pd[0] - dz, ty = c.z + g.pd[1] - dy, tx = c.w + g.pd[2] - dx;
    if (tz >= 0 && ty >= 0 && tx >= 0 && tz % g.st[0] == 0 && ty % g.st[1] == 0 && tx % g.st[2] == 0) {
      const int oz = tz / g.st[0], oy = ty / g.st[1], ox = tx / g.st[2];
      if (oz < g.out_shape[0] && oy < g.out_shape[1] && ox < g.out_shape[2]) {
        const long long key = (((long long)c.x * g.out_shape[0] + oz) * g.out_shape[1] + oy) * g.out_shape[2] + ox;
        const int r = sp_rank(out_bitmap, out_prefix, key);
        if (r >= 0) res = out_perm[r];
      }
    }
  }
  nbr_inv[t] = res;
}

static int sp_geom(sstb200_ctx* c, SpGeom& g, int B, const int32_t* in_shape, const int32_t* out_shape, const int32_t* ks,
                   const int32_t* st, const int32_t* pd) {
  CHECK_ARG(c, B >= 1 && in_shape && out_shape && ks && st && pd);
  g.B = B;
  g.KV = 1;
  for (int d = 0; d < 3; d++) {
    CHECK_ARG(c, in_shape[d] >= 1 && out_shape[d] >= 1 && ks[d] >= 1 && ks[d] <= 7 && st[d] >= 1 && pd[d] >= 0);
    g.in_shape[d] = in_shape[d];
    g.out_shape[d] = out_shape[d];
    g.ks[d] = ks[d];
    g.st[d] = st[d];
    g.pd[d] = pd[d];
    g.KV *= ks[d];
  }
  return SSTB_OK;
}

static int sp_extents(sstb200_ctx* c, Extents& e, long long* T, int B, const int* shape) {
  long long lo[4] = {0, 0, 0, 0}, hi[4] = {B - 1, shape[0] - 1, shape[1] - 1, shape[2] - 1};
  return make_extents(c, e, 4, lo, hi, T);
}

// ------------------------------------------------------------------------------------------------------------------------------
// fp32 implicit GEMM (the 1e-3 / "exact" path): 64 x 64 output tile per CTA, 4 x 4 micro-tile per thread, K = KV * Cin walked
// offset by offset in chunks of 16 channels; offsets no row of the tile uses are skipped.
// ------------------------------------------------------------------------------------------------------------------------------
#define SPF_BM 64
#define SPF_BN 64
#define SPF_BK 16
__global__ void __launch_bounds__(256) spconv_gemm_f32_kernel(const float* __restrict__ feats, int Cin, const int32_t* __restrict__ nbr,
                                                             int n_out, int KV, const float* __restrict__ W, int Cout,
                                                             const float* __restrict__ scale, const float* __restrict__ shift,
                                                             const float* __restrict__ residual, int relu, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  __shared__ __align__(16) float sA[SPF_BK][SPF_BM + 4];
  __shared__ __align__(16) float sB[SPF_BK][SPF_BN];
  __shared__ int sRow[SPF_BM];
  const int tid = threadIdx.x;
  const int row0 = blockIdx.x * SPF_BM, n0 = blockIdx.y * SPF_BN;
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
  for (int k = 0; k < KV; k++) {
    int mine = -1;
    if (tid < SPF_BM) {
      const int o = row0 + tid;
      mine = o < n_out ? nbr[(size_t)o * KV + k] : -1;
      sRow[tid] = mine;
    }
    if (!__syncthreads_or(mine >= 0)) continue;   // (barrier: sRow visible; previous chunk's reads of sA / sB are complete)
    for (int c0 = 0; c0 < Cin; c0 += SPF_BK) {
      {  // A: 64 rows x 16 channels, one float4 per thread, stored transposed
        const int r = tid >> 2, q = tid & 3;
        const int src = sRow[r];
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (src >= 0 && c0 + q * 4 < Cin) v = *reinterpret_cast<const float4*>(feats + (size_t)src * Cin + c0 + q * 4);
        sA[q * 4 + 0][r] = v.x;
        sA[q * 4 + 1][r] = v.y;
        sA[q * 4 + 2][r] = v.z;
        sA[q * 4 + 3][r] = v.w;
      }
      {  // B: 16 channels x 64 outputs
        const int kk = tid >> 4, q = tid & 15;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c0 + kk < Cin && n0 + q * 4 < Cout) v = __ldg(reinterpret_cast<const float4*>(W + ((size_t)k * Cin + c0 + kk) * Cout + n0 + q * 4));
        *reinterpret_cast<float4*>(&sB[kk][q * 4]) = v;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < SPF_BK; kk++) {
        const float4 a = *reinterpret_cast<const float4*>(&sA[kk][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&sB[kk][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  const int col = n0 + tx * 4;
  if (col >= Cout) return;
  float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
  if (scale) sc = __ldg(reinterpret_cast<const float4*>(scale + col));
  if (shift) sh = __ldg(reinterpret_cast<const float4*>(shift + col));
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int o = row0 + ty * 4 + i;
    if (o >= n_out) continue;
    float4 y;
    y.x = fmaf(acc[i][0], sc.x, sh.x);
    y.y = fmaf(acc[i][1], sc.y, sh.y);
    y.z = fmaf(acc[i][2], sc.z, sh.z);
    y.w = fmaf(acc[i][3], sc.w, sh.w);
    if (residual) {
      const float4 r4 = *reinterpret_cast<const float4*>(residual + (size_t)o * Cout + col);
      y.x += r4.x, y.y += r4.y, y.z += r4.z, y.w += r4.w;
    }
    if (relu) y.x = fmaxf(y.x, 0.f), y.y = fmaxf(y.y, 0.f), y.z = fmaxf(y.z, 0.f), y.w = fmaxf(y.w, 0.f);
    *reinterpret_cast<float4*>(out + (size_t)o * Cout + col) = y;
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// weight gradient:  dW[k] += sum over output rows o with nbr[o][k] >= 0 of  X[nbr[o][k]]^T . dY[o]      (fp32, FFMA)
// CTA = (chunk of SPW_ROWS output rows, kernel offset k, 64 x 64 tile of dW[k]).  The rows of the chunk that actually have a neighbour
// at offset k (17 % on a LiDAR sweep) are compacted into shared memory first, so the reduction only walks real pairs; the partial
// tile is added to dW with fp32 atomics (summation order across chunks is not fixed, like the reference's atomics-based backward).
// ------------------------------------------------------------------------------------------------------------------------------
#define SPW_ROWS 1024
__global__ void __launch_bounds__(256) spconv_dw_kernel(const float* __restrict__ X, int Cin, const int32_t* __restrict__ nbr, int n_out, int KV,
                                                       const float* __restrict__ dY, int Cout, float* __restrict__ dW) {
  pdl_wait();
  pdl_launch();
  __shared__ int sIn[SPW_ROWS], sOut[SPW_ROWS];
  __shared__ int sCount;
  __shared__ __align__(16) float sA[16][64];
  __shared__ __align__(16) float sB[16][64];
  const int tid = threadIdx.x;
  const int k = blockIdx.y;
  const int ncot = (Cout + 63) / 64;
  const int ci0 = ((int)blockIdx.z / ncot) * 64, co0 = ((int)blockIdx.z % ncot) * 64;
  const int r0 = blockIdx.x * SPW_ROWS;
  if (tid == 0) sCount = 0;
  __syncthreads();
  for (int j = tid; j < SPW_ROWS; j += 256) {
    const int o = r0 + j;
    if (o < n_out) {
      const int v = nbr[(size_t)o * KV + k];
      if (v >= 0) {
        const int pos = atomicAdd(&sCount, 1);
        sIn[pos] = v;
        sOut[pos] = o;
      }
    }
  }
  __syncthreads();
  const int cnt = sCount;
  if (cnt == 0) return;
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
  for (int q0 = 0; q0 < cnt; q0 += 16) {
    {
      const int r = tid >> 4, c4 = (tid & 15) * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q0 + r < cnt) {
        if (ci0 + c4 < Cin) a = *reinterpret_cast<const float4*>(X + (size_t)sIn[q0 + r] * Cin + ci0 + c4);
        if (co0 + c4 < Cout) b = *reinterpret_cast<const float4*>(dY + (size_t)sOut[q0 + r] * Cout + co0 + c4);
      }
      *reinterpret_cast<float4*>(&sA[r][c4]) = a;
      *reinterpret_cast<float4*>(&sB[r][c4]) = b;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 16; r++) {
      const float4 a = *reinterpret_cast<const float4*>(&sA[r][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&sB[r][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int ci = ci0 + ty * 4 + i;
    if (ci >= Cin) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int co = co0 + tx * 4 + j;
      if (co < Cout) atomicAdd(&dW[((size_t)k * Cin + ci) * Cout + co], acc[i][j]);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------------------
// tensor-core implicit GEMM (precision 'bf16' = 16-bit operands, fp32 accumulation): 128-row output tile x NT output channels per
// CTA, accumulators [128, NT] fp32 in registers across ALL kernel offsets (warpgroup g owns rows [64 g, 64 g + 64)), operands IEEE
// fp16 in the wgmma operand format (wgmma.cuh, staged as in wgmma_gemm.cuh).  K is walked in stages of (kernel offset,
// 64 input channels): the 256 threads gather the 128 neighbour rows (fp32 -> fp16 on the fly, absent neighbours = zero rows that are
// neither loaded nor converted) and the [NT, 64] weight slab into one of NS operand buffers, each warpgroup issues 4 wgmma (K = 16
// each) as one commit group; the global loads run TWO stages ahead in two register sets (the deep levels of a U-Net are a few CTAs
// walking 100-200 stages each: pure load latency), and a buffer is rewritten only after every warpgroup's group that read it has
// completed (wgmma.wait_group before the stage barrier).  Offsets no row of the tile uses are skipped.  Epilogue straight from the
// accumulator fragments: y = acc * scale + shift (+ residual) (ReLU), fp32 rows.
//
// Operand range.  fp16 has 5 exponent bits: unscaled, anything below 2^-14 loses bits and anything below 2^-24 is zero - which is
// where the gradients of a mean-reduced loss live (dX runs this kernel with A = grad_out).  So both operands are brought to the
// top of the fp16 range by exact powers of two before they are rounded, and the powers are taken out of the fp32 accumulators:
//   * A: sp_row_exp_kernel gives every input row the exponent that puts its largest |element| in [2^13, 2^14); an OUTPUT row uses
//     the smallest exponent among the rows it gathers (every offset of an output row meets in one accumulator row, so the exponent
//     must be one per output row; nothing forces it to be one per tensor), applied while converting, removed per accumulator row.
//   * W: one exponent per output channel, applied where the 16-bit copy is made (split_h16), removed per accumulator column.
// The result is homogeneous in the scale of either operand: x * 2^s gives out * 2^s to the last bit while fp32 can hold it.
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int SPU_TM = 128;
constexpr int SPU_A_BYTES = SPU_TM * 128;
#define SPU_MAX_KV 27

// fp32 pair -> fp16x2 with saturation to +-65504 in ONE instruction (F2FP.SATFINITE.F16.F32.PACK_AB); a = low half
__device__ __forceinline__ uint32_t sp_pack_f16(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

constexpr int SPU_EXP_TOP = 14;    // a scaled row's largest |element| lies in [2^13, 2^14): below fp16's 65504 with room for rounding
constexpr int SPU_EXP_LIM = 100;   // |exponent| bound: 2^+-100 and every product with an fp16-range value are exact fp32

// the power of two that lifts a largest |element| of bits m into [2^(SPU_EXP_TOP - 1), 2^SPU_EXP_TOP): amax = f * 2^(field - 126),
// f in [0.5, 1); an all-zero (or subnormal) row takes the largest exponent and never decides a minimum
__device__ __forceinline__ int sp_exp_of(uint32_t m) { return max(-SPU_EXP_LIM, min(SPU_EXP_LIM, SPU_EXP_TOP - ((int)(m >> 23) - 126))); }

// rexp[i] = sp_exp_of(row i's largest |element|); one warp per row
__global__ void __launch_bounds__(256) sp_row_exp_kernel(const float* __restrict__ feats, int lda, int C, int n, const int32_t* __restrict__ n_dev,
                                                        int32_t* __restrict__ rexp) {
  pdl_wait();
  pdl_launch();
  if (n_dev) n = min(n, *n_dev);
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n) return;
  const float4* p = reinterpret_cast<const float4*>(feats + (size_t)row * lda);
  uint32_t m = 0u;   // |x| as bits: ordered like the magnitudes
  for (int q = lane; q < (C >> 2); q += 32) {
    const float4 v = p[q];
    m = max(max(m, __float_as_uint(v.x) & 0x7fffffffu), max(__float_as_uint(v.y) & 0x7fffffffu, __float_as_uint(v.z) & 0x7fffffffu));
    m = max(m, __float_as_uint(v.w) & 0x7fffffffu);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) rexp[row] = sp_exp_of(m);
}

__device__ __forceinline__ float sp_exp2i(int e) { return __int_as_float((e + 127) << 23); }   // 2^e, |e| <= SPU_EXP_LIM

struct SpArgs {
  const float* feats;      // [*, lda] fp32 rows (gathered through nbr, or row o itself when nbr == nullptr)
  const int32_t* rexp;     // per-row power-of-two exponents of feats (sp_row_exp_kernel), or nullptr: operands converted as they are
  int self_exp;            // SPLIT, nbr == nullptr only: each CTA takes its rows' exponents from the rows themselves (rexp unused)
  const float* wun;        // [Cout] 2^-e of the exponent the 16-bit weight copy carries per output channel, or nullptr (1)
  int lda, Cin;
  const int32_t* nbr;      // [n_out, KV] or nullptr (KV must be 1: a plain row GEMM)
  int n_out;
  const int32_t* n_dev;    // optional device-side row count (<= n_out)
  int KV;
  const __half* Whi;       // [KV][Cout][Cin] fp16
  const __half* Wlo;       // SPLIT: the fp16 residue  W - float(Whi)
  int Cout;
  const float *scale, *shift, *residual;
  int ldr, act;            // act: 0 none, 1 ReLU, 2 GELU (erf form)
  float* out;
  int ldo;
};

template <int BU, bool SPLIT>
struct SpStageRegs {
  float4 a0[4], a1[4];            // 4 pieces of 8 gathered channels each
  int4 b[BU];                     // weight pieces
  int4 blo[SPLIT ? BU : 1];       // SPLIT: residue pieces
  uint32_t valid;                 // bit u: piece u has a source row (absent neighbours are neither loaded nor converted)
};

// SPLIT = the fp32-tolerance mode on the tensor core: every fp32 operand is carried as two fp16 numbers (hi = rn(x), lo = rn(x - hi)),
// and a stage issues the three products hi.hi + lo.hi + hi.lo into the same fp32 accumulators (the dropped lo.lo term is 2^-22
// relative).  Same staging, same epilogue; 3x the MMAs, 2x the operand bytes.  hi + lo carries 22 significant bits of an element
// while lo is a normal fp16 number, i.e. for scaled |x| >= 2^-3: elements within 2^-16 of their row group's largest.  Smaller
// ones keep an absolute error of 2^-25 scaled = 2^-38 of that largest element, which is below the fp32 rounding of the sum they
// are added to.
template <int NT, int NS, bool SPLIT>
__global__ void __launch_bounds__(256, (NT == 64 && !SPLIT) ? 2 : 1) spconv_wgmma_kernel(SpArgs g) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint8_t sp_smem_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)sp_smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int B_BYTES = NT * 128;
  constexpr int ST_BYTES = (SPLIT ? 2 : 1) * (SPU_A_BYTES + B_BYTES);   // [A_hi][A_lo][B_hi][B_lo] or [A][B]
  constexpr int OFF_ALO = SPU_A_BYTES, OFF_B = (SPLIT ? 2 : 1) * SPU_A_BYTES, OFF_BLO = OFF_B + B_BYTES;
  constexpr int BU = NT / 32;  // 16-byte weight pieces per thread and stage
  static_assert(NS >= 2, "the stage barrier retires the group of the stage NS - 1 back");
  __shared__ uint32_t used_mask;
  __shared__ int sNbr[SPU_TM][SPU_MAX_KV];   // odd row pitch: conflict-free column reads
  __shared__ int sExp[SPU_TM];               // exponent of output row r's gathered operand rows

  const int tid = threadIdx.x, lane = tid & 31;
  const int row0 = blockIdx.x * SPU_TM, n0 = blockIdx.y * NT;
  const int n_out = g.n_dev ? min(g.n_out, *g.n_dev) : g.n_out;
  if (row0 >= n_out) return;   // uniform per CTA
  const int KV = g.KV, Cin = g.Cin, Cout = g.Cout;
  const int wg = tid >> 7;
  if (tid == 0) used_mask = 0u;
  __syncthreads();
  {
    uint32_t m = 0u;
    for (int idx = tid; idx < SPU_TM * KV; idx += 256) {
      const int r = idx / KV, k = idx - r * KV;
      const int o = row0 + r;
      const int v = o < n_out ? (g.nbr ? g.nbr[(size_t)o * KV + k] : o) : -1;
      sNbr[r][k] = v;
      if (v >= 0) m |= 1u << k;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m |= __shfl_xor_sync(0xffffffffu, m, o);
    if (lane == 0 && m) atomicOr(&used_mask, m);
  }
  __syncthreads();
  if (!(SPLIT && g.self_exp) && tid < SPU_TM) {   // (GEMM mode: below, behind the first two stages' loads)
    int e = g.rexp ? SPU_EXP_LIM : 0;
    if (g.rexp)
      for (int k = 0; k < KV; k++) {
        const int v = sNbr[tid][k];
        if (v >= 0) e = min(e, __ldg(g.rexp + v));
      }
    sExp[tid] = e;
  }
  __syncthreads();
  const int nch = Cin >> 6;
  const int nst = __popc(used_mask) * nch;

  // stage iterator of the loader (stages are visited in order: used offsets ascending, 64-channel chunks inside)
  uint32_t ld_mask = used_mask;
  int ld_c = 0, loaded = 0;
  const int my_r = tid >> 3, my_jj = tid & 7;   // piece u of this thread: row my_r + 32 u, 16-byte column my_jj
  auto load_next = [&](SpStageRegs<BU, SPLIT>& R) {
    if (loaded >= nst) return;
    const int k = __ffs(ld_mask) - 1, c = ld_c;
    R.valid = 0u;
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int src = sNbr[my_r + 32 * u][k];
      if (src >= 0) {
        R.valid |= 1u << u;
        const float* ap = g.feats + (size_t)src * g.lda + c * 64 + my_jj * 8;
        R.a0[u] = *reinterpret_cast<const float4*>(ap);
        R.a1[u] = *reinterpret_cast<const float4*>(ap + 4);
      }
    }
    const size_t woff = ((size_t)k * Cout + n0 + my_r) * Cin + c * 64 + my_jj * 8;
#pragma unroll
    for (int u = 0; u < BU; u++) {
      R.b[u] = __ldg(reinterpret_cast<const int4*>(g.Whi + woff + (size_t)32 * u * Cin));
      if (SPLIT) R.blo[u] = __ldg(reinterpret_cast<const int4*>(g.Wlo + woff + (size_t)32 * u * Cin));
    }
    loaded++;
    if (++ld_c == nch) {
      ld_c = 0;
      ld_mask &= ld_mask - 1u;
    }
  };
  float acc[NT / 2];
#pragma unroll
  for (int i = 0; i < NT / 2; i++) acc[i] = 0.f;
  // buffer s % NS was last read by stage s - NS, whose groups the barrier of stage s - 1 has retired (see below)
  auto run_stage = [&](int s, SpStageRegs<BU, SPLIT>& R) {
    const int b = s % NS;
    uint8_t* sA = base + (size_t)b * ST_BYTES;
    uint8_t* sB = sA + OFF_B;
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int r = my_r + 32 * u;
      // piece my_jj of row r in the operand format of wgmma.cuh, spelled out: through sw128_off this kernel needs more registers
      // and spills
      const int off = r * 128 + ((my_jj ^ (r & 7)) << 4);
      int4 v = make_int4(0, 0, 0, 0), vl = make_int4(0, 0, 0, 0);
      if ((R.valid >> u) & 1u) {
        const float as = sp_exp2i(sExp[r]);
        const float f[8] = {R.a0[u].x * as, R.a0[u].y * as, R.a0[u].z * as, R.a0[u].w * as,
                            R.a1[u].x * as, R.a1[u].y * as, R.a1[u].z * as, R.a1[u].w * as};
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
          hi[e] = sp_pack_f16(f[2 * e], f[2 * e + 1]);
          if (SPLIT) {
            const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi[e]));
            lo[e] = sp_pack_f16(f[2 * e] - h.x, f[2 * e + 1] - h.y);
          }
        }
        v = make_int4((int)hi[0], (int)hi[1], (int)hi[2], (int)hi[3]);
        if (SPLIT) vl = make_int4((int)lo[0], (int)lo[1], (int)lo[2], (int)lo[3]);
      }
      *reinterpret_cast<int4*>(sA + off) = v;
      if (SPLIT) *reinterpret_cast<int4*>(sA + OFF_ALO + off) = vl;
    }
#pragma unroll
    for (int u = 0; u < BU; u++) {
      const int r = my_r + 32 * u;
      const int off = r * 128 + ((my_jj ^ (r & 7)) << 4);
      *reinterpret_cast<int4*>(sB + off) = R.b[u];
      if (SPLIT) *reinterpret_cast<int4*>(sA + OFF_BLO + off) = R.blo[u];
    }
    load_next(R);         // the register set is free again: fetch the stage two ahead while this one is multiplied
    fence_async_smem();   // generic-proxy smem writes -> visible to the tensor core (async proxy)
    wgmma_wait<NS - 2>(); // this warpgroup's groups up to stage s - NS + 1 are complete once every thread passes the barrier
    __syncthreads();
    {
      const uint32_t a0 = smem_u32(sA) + wg * 64 * 128, b0 = smem_u32(sB);
      wgmma_fence();
#pragma unroll
      for (int q = 0; q < 4; q++) wgmma_ss<NT, false>(acc, wg_desc_sw128(a0 + q * 32), wg_desc_sw128(b0 + q * 32), 1);
      if (SPLIT) {
        const uint32_t al = a0 + OFF_ALO, bl = smem_u32(sA) + OFF_BLO;
#pragma unroll
        for (int q = 0; q < 4; q++) wgmma_ss<NT, false>(acc, wg_desc_sw128(al + q * 32), wg_desc_sw128(b0 + q * 32), 1);   // lo . hi
#pragma unroll
        for (int q = 0; q < 4; q++) wgmma_ss<NT, false>(acc, wg_desc_sw128(a0 + q * 32), wg_desc_sw128(bl + q * 32), 1);   // hi . lo
      }
      wgmma_commit();
    }
  };

  SpStageRegs<BU, SPLIT> R0, R1;
  R0.valid = R1.valid = 0u;
  load_next(R0);
  load_next(R1);
  if (SPLIT && g.self_exp) {   // GEMM mode (sstb_row_gemm_x3), while the first two stages load: eight threads per row, 128
    // contiguous bytes per row and load
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int r = (tid >> 3) + 32 * u, o = row0 + r;
      uint32_t m = 0u;
      if (o < n_out) {
        const float4* p = reinterpret_cast<const float4*>(g.feats + (size_t)o * g.lda);
#pragma unroll 4
        for (int q = tid & 7; q < (Cin >> 2); q += 8) {   // Cin is a multiple of 64: 2 or more loads per thread, several in flight
          const float4 v = p[q];
          m = max(max(m, __float_as_uint(v.x) & 0x7fffffffu), max(__float_as_uint(v.y) & 0x7fffffffu, __float_as_uint(v.z) & 0x7fffffffu));
          m = max(m, __float_as_uint(v.w) & 0x7fffffffu);
        }
      }
#pragma unroll
      for (int x = 4; x > 0; x >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, x));
      if ((tid & 7) == 0) sExp[r] = sp_exp_of(m);
    }
    __syncthreads();
  }
  for (int s = 0; s < nst; s += 2) {
    run_stage(s, R0);
    if (s + 1 < nst) run_stage(s + 1, R1);
  }
  wgmma_wait<0>();   // every MMA of the tile is done

  // ---- epilogue, from the accumulator fragments -------------------------------------------------------------------------------
  wg_frag_pairs<NT>(acc, [&](int r, int cc, float v0, float v1) {
    const int o = row0 + wg * 64 + r;
    if (o >= n_out) return;
    const int col = n0 + cc;
    // the operands' powers of two leave the accumulator first (exact), one factor at a time so that neither can leave fp32's range alone
    const float ua = sp_exp2i(-sExp[wg * 64 + r]);
    v0 *= ua, v1 *= ua;
    if (g.wun) {
      const float2 uw = __ldg(reinterpret_cast<const float2*>(g.wun + col));
      v0 *= uw.x, v1 *= uw.y;
    }
    float2 sc = make_float2(1.f, 1.f), sh = make_float2(0.f, 0.f);
    if (g.scale) sc = __ldg(reinterpret_cast<const float2*>(g.scale + col));
    if (g.shift) sh = __ldg(reinterpret_cast<const float2*>(g.shift + col));
    float2 y = make_float2(fmaf(v0, sc.x, sh.x), fmaf(v1, sc.y, sh.y));
    if (g.act == 2) y.x = gelu_erf(y.x), y.y = gelu_erf(y.y);   // Linear -> GELU (-> + residual)
    if (g.residual) {
      const float2 r2 = *reinterpret_cast<const float2*>(g.residual + (size_t)o * g.ldr + col);
      y.x += r2.x, y.y += r2.y;
    }
    if (g.act == 1) y.x = fmaxf(y.x, 0.f), y.y = fmaxf(y.y, 0.f);  // conv + BN + res -> ReLU
    *reinterpret_cast<float2*>(g.out + (size_t)o * g.ldo + col) = y;
  });
}

template <int NT, int NS, bool SPLIT>
static int launch_spconv_wgmma(sstb200_ctx* c, const SpArgs& g) {
  auto kern = spconv_wgmma_kernel<NT, NS, SPLIT>;
  static SmemAttr sa;
  const size_t smem = (size_t)NS * (SPLIT ? 2 : 1) * (SPU_A_BYTES + NT * 128) + 1024;
  CUDA_TRY(c, ensure_smem(c, sa, kern, smem));
  dim3 grid((g.n_out + SPU_TM - 1) / SPU_TM, g.Cout / NT);
  launch_pdl(kern, grid, dim3(256), smem, c->stream, g);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

static int dispatch_spconv_wgmma(sstb200_ctx* c, const SpArgs& g, bool split) {
  // 128 output channels per CTA at most: a warpgroup's [64, NT] fp32 accumulators take NT / 2 registers per thread, beside the
  // two register sets of staged operands
  if (split) {
    if (g.Cout % 128 == 0) return launch_spconv_wgmma<128, 2, true>(c, g);
    return launch_spconv_wgmma<64, 3, true>(c, g);
  }
  if (g.Cout % 128 == 0) return launch_spconv_wgmma<128, 3, false>(c, g);
  return launch_spconv_wgmma<64, 3, false>(c, g);
}

// W [N, K] fp32 -> (hi, lo) fp16, one block per output channel: the channel is lifted by the power of two sp_exp_of gives its
// largest |w| before it is split (exact), and wun[n] = the inverse power, which the epilogue applies
__global__ void __launch_bounds__(256) split_f16_rows_kernel(const float* __restrict__ w, int K, __half* __restrict__ hi,
                                                            __half* __restrict__ lo, float* __restrict__ wun) {
  pdl_wait();
  pdl_launch();
  __shared__ uint32_t amax;
  const int n = blockIdx.x;
  const float* p = w + (size_t)n * K;
  if (threadIdx.x == 0) amax = 0u;
  __syncthreads();
  uint32_t m = 0u;   // |w| as bits, as in sp_row_exp_kernel
  for (int k = threadIdx.x; k < K; k += 256) m = max(m, __float_as_uint(p[k]) & 0x7fffffffu);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&amax, m);
  __syncthreads();
  const int e = sp_exp_of(amax);
  const float s = sp_exp2i(e);
  for (int k = threadIdx.x; k < K; k += 256) {
    const float x = p[k] * s;
    const __half h = __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f));
    hi[(size_t)n * K + k] = h;
    lo[(size_t)n * K + k] = __float2half_rn(x - __half2float(h));
  }
  if (threadIdx.x == 0) wun[n] = sp_exp2i(-e);
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------------------------------------
extern "C" int sstb200_spconv_out_coors(sstb200_ctx* c, const int32_t* in_coors, int n_in, int batch_size, const int32_t in_shape[3],
                                        const int32_t out_shape[3], const int32_t ksize[3], const int32_t stride[3],
                                        const int32_t padding[3], int32_t* out_coors, int out_cap, int32_t* num_out_dev,
                                        int32_t* num_out_host) {
  CHECK_ARG(c, c && n_in >= 0 && num_out_dev);
  SpGeom g;
  int rc = sp_geom(c, g, batch_size, in_shape, out_shape, ksize, stride, padding);
  if (rc) return rc;
  if (n_in == 0) {
    CUDA_TRY(c, cudaMemsetAsync(num_out_dev, 0, 4, c->stream));
    if (num_out_host) *num_out_host = 0;
    return SSTB_OK;
  }
  CHECK_ARG(c, in_coors && out_coors);
  // every input reaches at most prod(ceil(k / s)) outputs
  long long per_in = 1, cells = batch_size;
  for (int d = 0; d < 3; d++) {
    per_in *= (g.ks[d] + g.st[d] - 1) / g.st[d];
    cells *= g.out_shape[d];
  }
  long long bound = (long long)n_in * per_in;
  if (bound > cells) bound = cells;
  if ((long long)out_cap < bound)
    return sstb_fail(c, SSTB_ERR_ARG, "spconv_out_coors: out_cap %d < worst case %lld rows", out_cap, bound);
  Extents e;
  long long T;
  rc = sp_extents(c, e, &T, batch_size, g.out_shape);
  if (rc) return rc;
  arena_reset(c);
  KeyIndex k;
  rc = arena_carve(c, [&](Carve& cv) { key_index_carve(cv, k, 1, T); });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k))) return rc;
  const long long work = (long long)n_in * g.KV;
  launch_pdl(sp_mark_out_kernel, dim3((unsigned)((work + 255) / 256)), dim3(256), (size_t)0, c->stream, in_coors, n_in, g, k.bitmap, k.flags);
  key_index_scan(c, k);
  launch_emit_rows<int32_t>(c, k, e, 0, out_coors, num_out_dev);
  LAUNCH_CHECK(c);
  if (num_out_host) {
    rc = read_back_i32(c, num_out_dev, num_out_host);
    if (rc) return rc;
    int32_t bad = 0;
    rc = read_back_i32(c, k.flags + 1, &bad);
    if (rc) return rc;
    if (bad) return sstb_fail(c, SSTB_ERR_ARG, "spconv_out_coors: an input coordinate lies outside batch_size / in_shape");
  }
  return SSTB_OK;
}

extern "C" int sstb200_spconv_table(sstb200_ctx* c, const int32_t* in_coors, int n_in, const int32_t* out_coors, int n_out,
                                    int batch_size, const int32_t in_shape[3], const int32_t out_shape[3], const int32_t ksize[3],
                                    const int32_t stride[3], const int32_t padding[3], int32_t* nbr, int32_t* nbr_inv,
                                    int32_t* status_host) {
  CHECK_ARG(c, c && n_in >= 0 && n_out >= 0);
  SpGeom g;
  int rc = sp_geom(c, g, batch_size, in_shape, out_shape, ksize, stride, padding);
  if (rc) return rc;
  if (status_host) *status_host = 0;
  if (n_in == 0 || n_out == 0) {
    if (nbr && n_out) CUDA_TRY(c, cudaMemsetAsync(nbr, 0xFF, (size_t)n_out * g.KV * 4, c->stream));
    if (nbr_inv && n_in) CUDA_TRY(c, cudaMemsetAsync(nbr_inv, 0xFF, (size_t)n_in * g.KV * 4, c->stream));
    return SSTB_OK;
  }
  CHECK_ARG(c, in_coors && out_coors && (nbr || nbr_inv));
  Extents ei, eo;
  long long Ti, To;
  rc = sp_extents(c, ei, &Ti, batch_size, g.in_shape);
  if (rc) return rc;
  rc = sp_extents(c, eo, &To, batch_size, g.out_shape);
  if (rc) return rc;
  arena_reset(c);
  KeyIndex ki, ko;
  int32_t *perm_i = nullptr, *perm_o = nullptr;
  rc = arena_carve(c, [&](Carve& cv) {
    if (nbr) {
      key_index_carve(cv, ki, n_in, Ti);
      perm_i = cv.take<int32_t>(n_in);
    }
    if (nbr_inv) {
      key_index_carve(cv, ko, n_out, To);
      perm_o = cv.take<int32_t>(n_out);
    }
  });
  if (rc) return rc;
  if (nbr) {
    if ((rc = key_index_zero(c, ki))) return rc;
    launch_mark_rows<int32_t>(c, in_coors, n_in, ei, false, ki, nullptr);
    key_index_scan(c, ki);
    launch_pdl(sp_perm_kernel, dim3((n_in + 255) / 256), dim3(256), (size_t)0, c->stream, (const long long*)ki.keys, n_in, (const int32_t*)nullptr,
               (const uint32_t*)ki.bitmap, (const uint32_t*)ki.word_prefix, perm_i);
    const long long work = (long long)n_out * g.KV;
    launch_pdl(sp_nbr_kernel, dim3((unsigned)((work + 255) / 256)), dim3(256), (size_t)0, c->stream, out_coors, n_out, g, (const uint32_t*)ki.bitmap,
               (const uint32_t*)ki.word_prefix, (const int32_t*)perm_i, nbr);
  }
  if (nbr_inv) {
    if ((rc = key_index_zero(c, ko))) return rc;
    launch_mark_rows<int32_t>(c, out_coors, n_out, eo, false, ko, nullptr);
    key_index_scan(c, ko);
    launch_pdl(sp_perm_kernel, dim3((n_out + 255) / 256), dim3(256), (size_t)0, c->stream, (const long long*)ko.keys, n_out, (const int32_t*)nullptr,
               (const uint32_t*)ko.bitmap, (const uint32_t*)ko.word_prefix, perm_o);
    const long long work = (long long)n_in * g.KV;
    launch_pdl(sp_nbr_inv_kernel, dim3((unsigned)((work + 255) / 256)), dim3(256), (size_t)0, c->stream, in_coors, n_in, g, (const uint32_t*)ko.bitmap,
               (const uint32_t*)ko.word_prefix, (const int32_t*)perm_o, nbr_inv);
  }
  LAUNCH_CHECK(c);
  if (status_host) {
    int32_t bad = 0;
    if (nbr) {
      rc = read_back_i32(c, ki.flags, &bad);
      if (rc) return rc;
      *status_host |= bad ? 1 : 0;
    }
    if (nbr_inv) {
      rc = read_back_i32(c, ko.flags, &bad);
      if (rc) return rc;
      *status_host |= bad ? 2 : 0;
    }
    if (*status_host)
      return sstb_fail(c, SSTB_ERR_ARG, "spconv_table: coordinates outside batch_size / spatial shape (status %d)", *status_host);
  }
  return SSTB_OK;
}

extern "C" int sstb200_spconv_forward(sstb200_ctx* c, const float* feats, int n_in, int c_in, const int32_t* nbr, int n_out, int kernel_volume,
                                      const float* weight, const void* weight_h16, const float* weight_h16_unscale, int c_out,
                                      const float* scale, const float* shift, const float* residual, int relu, int precision, float* out) {
  CHECK_ARG(c, c && n_in >= 0 && n_out >= 0 && c_in >= 1 && c_out >= 1 && kernel_volume >= 1);
  if (n_out == 0) return SSTB_OK;
  CHECK_ARG(c, feats && nbr && out);
  CHECK_ARG(c, ((uintptr_t)feats & 15) == 0 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)residual & 15) == 0);
  if (precision == SSTB200_PREC_FP32) {
    CHECK_ARG(c, weight != nullptr);
    if ((c_in & 3) || (c_out & 3))
      return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "spconv_forward: channel counts must be multiples of 4 (got %d -> %d)", c_in, c_out);
    dim3 grid((n_out + SPF_BM - 1) / SPF_BM, (c_out + SPF_BN - 1) / SPF_BN);
    launch_pdl(spconv_gemm_f32_kernel, grid, dim3(256), (size_t)0, c->stream, feats, c_in, nbr, n_out, kernel_volume, weight, c_out, scale, shift,
               residual, relu, out);
    LAUNCH_CHECK(c);
    return SSTB_OK;
  }
  CHECK_ARG(c, precision == SSTB200_PREC_BF16 || precision == SSTB200_PREC_FP32_TC);
  CHECK_ARG(c, weight_h16 != nullptr && ((uintptr_t)weight_h16 & 15) == 0);
  if ((c_in & 63) || (c_out & 63) || kernel_volume > SPU_MAX_KV)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED,
                     "spconv_forward: the tensor-core path needs c_in, c_out multiples of 64 and kernel volume <= %d (got %d -> %d, %d); "
                     "use precision fp32", SPU_MAX_KV, c_in, c_out, kernel_volume);
  // per-row exponents of feats: one small launch (reads feats once; the convolution gathers it kernel_volume times)
  arena_reset(c);
  int32_t* rexp;
  int rc = arena_carve(c, [&](Carve& cv) { rexp = cv.take<int32_t>((size_t)n_in + 1); });
  if (rc) return rc;
  if (n_in) launch_pdl(sp_row_exp_kernel, dim3((n_in + 7) / 8), dim3(256), (size_t)0, c->stream, feats, c_in, c_in, n_in, (const int32_t*)nullptr, rexp);
  SpArgs g;
  g.feats = feats, g.rexp = rexp, g.self_exp = 0, g.wun = weight_h16_unscale;
  g.lda = c_in, g.Cin = c_in, g.nbr = nbr, g.n_out = n_out, g.n_dev = nullptr, g.KV = kernel_volume;
  g.Whi = (const __half*)weight_h16;
  g.Wlo = g.Whi + (size_t)kernel_volume * c_out * c_in;   // FP32_TC: the residue copy follows the hi copy
  g.Cout = c_out, g.scale = scale, g.shift = shift, g.residual = residual, g.ldr = c_out, g.act = relu ? 1 : 0, g.out = out, g.ldo = c_out;
  return dispatch_spconv_wgmma(c, g, precision == SSTB200_PREC_FP32_TC);
}

// fp32-tolerance row GEMM on the tensor core (rows.cuh; the fp32 mode of the SRA encoder, csrc/sra_fp32.cu, runs on it):
//   out[r, :N] = act(A[r, :K] . W[N, K]^T + bias) + res[r]      with every operand split into two fp16 numbers (see SPLIT above),
// each row of A and each output channel of W first lifted to the top of fp16's range by its own power of two, as in
// sstb200_spconv_forward: the result is homogeneous in the scale of either operand
int sstb_row_gemm_x3(sstb200_ctx* c, const RowGemm& r) {
  if (r.M_cap <= 0) return SSTB_OK;
  const int N = r.N, K = r.K;
  if ((K & 63) || (N & 63) || (r.lda & 3) || (r.ldo & 3) || (r.ldr & 3) || (r.act == 1 && r.res)) return SSTB_ERR_UNSUPPORTED;
  if ((r.ldw && r.ldw != K) || r.res_index || r.pos.tab) return SSTB_ERR_UNSUPPORTED;   // forms only the FFMA row GEMM takes
  // the split weights are carved after what the caller's phase already holds, without a reset
  __half *hi, *lo;
  float* wun;
  int rc = arena_carve(c, [&](Carve& cv) {
    hi = cv.take<__half>((size_t)N * K);
    lo = cv.take<__half>((size_t)N * K);
    wun = cv.take<float>(N);
  });
  if (rc) return rc;
  launch_pdl(split_f16_rows_kernel, dim3((unsigned)N), dim3(256), (size_t)0, c->stream, r.W, K, hi, lo, wun);
  SpArgs g;
  g.rexp = nullptr, g.self_exp = 1, g.wun = wun;
  g.feats = r.A, g.lda = r.lda, g.Cin = K, g.nbr = nullptr, g.n_out = r.M_cap, g.n_dev = r.M_dev, g.KV = 1, g.Whi = hi, g.Wlo = lo, g.Cout = N;
  g.scale = nullptr, g.shift = r.bias, g.residual = r.res, g.ldr = r.ldr, g.act = r.act, g.out = r.out, g.ldo = r.ldo;
  return dispatch_spconv_wgmma(c, g, true);
}

extern "C" int sstb200_spconv_backward_weight(sstb200_ctx* c, const float* feats, int c_in, const int32_t* nbr, int n_out, int kernel_volume,
                                              const float* grad_out, int c_out, float* grad_weight) {
  CHECK_ARG(c, c && n_out >= 0 && c_in >= 1 && c_out >= 1 && kernel_volume >= 1 && grad_weight);
  CUDA_TRY(c, cudaMemsetAsync(grad_weight, 0, (size_t)kernel_volume * c_in * c_out * 4, c->stream));
  if (n_out == 0) return SSTB_OK;
  CHECK_ARG(c, feats && nbr && grad_out);
  CHECK_ARG(c, ((uintptr_t)feats & 15) == 0 && ((uintptr_t)grad_out & 15) == 0);
  if ((c_in & 3) || (c_out & 3))
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "spconv_backward_weight: channel counts must be multiples of 4 (got %d -> %d)", c_in, c_out);
  const int tiles = ((c_in + 63) / 64) * ((c_out + 63) / 64);
  if (kernel_volume > 65535 || tiles > 65535) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "spconv_backward_weight: grid too large");
  dim3 grid((n_out + SPW_ROWS - 1) / SPW_ROWS, kernel_volume, tiles);
  launch_pdl(spconv_dw_kernel, grid, dim3(256), (size_t)0, c->stream, feats, c_in, nbr, n_out, kernel_volume, grad_out, c_out, grad_weight);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
