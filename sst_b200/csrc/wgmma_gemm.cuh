// Generic wgmma GEMM tile kernel shared by the SRA forward (csrc/sra_bf16.cu) and the training path (csrc/sra_train.cu):
//     C[128-row tile, NT] = A[128, K] . W[NT, K]^T      (whole K staged once, K <= 384; fp32 accumulators)
// A-operand prologues: plain 16-bit rows, or fp32 rows (+ positional embedding from the per-axis table) converted on the fly.
// Epilogues (thread per row out of the shared-memory accumulator tile, then coalesced through an XOR-swizzled staging tile):
//     EPI_H16 / EPI_F16  + bias, store 16-bit (operand format / always fp16)
//     EPI_H16_GELU       + bias, GELU, store 16-bit (optionally also the pre-activation, for the backward pass)
//     EPI_RES_LN         + bias + fp32 residual, LayerNorm, store fp32 (+ 16-bit copy, + the pre-LayerNorm sum)
//     EPI_ADD_F32        + fp32 residual, store fp32                       (dX = dY . W + skip gradient)
//     EPI_GELUGRAD       * gelu'(z), store 16-bit                          (dz = (dh . W2) * gelu'(z))
// FMT selects the 16-bit operand / output format: 0 = IEEE fp16 (inference), 1 = bf16 (training: gradients need the fp32
// exponent range, and forward + backward then share one set of saved activations).
#pragma once
#include <stdarg.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace {

enum { PRO_H16 = 0, PRO_F32 = 1 };
enum { EPI_H16 = 0, EPI_H16_GELU = 1, EPI_RES_LN = 2, EPI_F16 = 3, EPI_ADD_F32 = 4, EPI_GELUGRAD = 5 };

struct GemmArgs {
  const void* A;        // [M, lda] bf16 or fp32; tile rows are consecutive rows of A
  int lda;
  const void* W;        // [N_total, K] 16-bit (FMT)
  const float* bias;    // [N_total]
  int M_cap;
  const int32_t* M_dev;
  // prologue
  const float* pos_tab;
  const int32_t* pos_code;
  int posL, pos_maxw, pos_ndim, pos_ntiles;  // add pos for n-tile < pos_ntiles
  int ny;                                    // number of n tiles
  // epilogue
  const int32_t* out_row_map;  // nullable: output / residual row of tile row i is out_row_map[i] (scatter), else i
  void* out_h16;        // [M, ldo] 16-bit
  void* out_pre16;      // optional [M, ldo]: pre-activation (EPI_H16_GELU)
  const void* aux16;    // [M, ldo] z (EPI_GELUGRAD)
  float* out_pre;       // optional [M, NT] fp32: acc + bias + residual before LayerNorm (EPI_RES_LN)
  int ldo;
  const float* res;     // [M, NT] fp32 residual (EPI_RES_LN)
  const float *gamma, *beta;
  float eps;
  float* out_f32;       // [M, NT]
};

constexpr int TILE_M = 128;

// Persistent over (row tile, n tile) items.  Per item: stage W and A (16-byte chunks, 8 loads in flight per thread) in
// the wgmma operand format (wgmma.cuh) -> each of the two warpgroups runs the wgmma chain of its 64 rows -> the register fragments
// go to a shared-memory accumulator tile -> epilogue.  The epilogue goes through shared memory (the operand buffers are free
// once the MMAs have completed) so that every global access is a coalesced row segment: thread-per-row accumulator reads
// meet warp-per-row global traffic in an XOR-swizzled staging tile.
template <int K, int NT, int PRO, int EPI, int FMT>
__global__ void __launch_bounds__(256) wgmma_gemm_kernel(GemmArgs g) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = base;                           // K/64 chunks x 128 rows x 128 B
  uint8_t* sW = sA + (size_t)TILE_M * K * 2;    // K/64 chunks x NT rows x 128 B
  uint8_t* sE = base;                           // epilogue staging (aliases the operands)
  constexpr int STAGE = (EPI == EPI_RES_LN || EPI == EPI_ADD_F32) ? TILE_M * NT * 4 : TILE_M * NT * 2;
  float* sAcc = reinterpret_cast<float*>(base + STAGE);   // [128][NT] fp32 accumulators (aliases the operands, not the staging)
  __shared__ float red[2][TILE_M][EPI == EPI_RES_LN ? 3 : 2];   // per half-row: sum, sum of squares (, centred squares)
  __shared__ int sRow[TILE_M];

  const int tid = threadIdx.x, warp = tid >> 5;
  const int M = g.M_dev ? *g.M_dev : g.M_cap;
  const int n_items = ((M + TILE_M - 1) / TILE_M) * g.ny;
  if ((int)blockIdx.x >= n_items) return;  // uniform per CTA

  constexpr int CH = K / 8;  // 16-byte chunks per operand row
  constexpr int NTH = 256, UNR = 8;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int ytile = item % g.ny;
    const int row0 = (item / g.ny) * TILE_M;
    const int n0 = ytile * NT;
    if (tid < TILE_M) {
      int gr = row0 + tid;
      sRow[tid] = gr < M ? (g.out_row_map ? g.out_row_map[gr] : gr) : -1;
    }
    // ---- stage W tile (rows n0..n0+NT of W[., K]) ----------------------------------------------------------------
    {
      const __half* wsrc = reinterpret_cast<const __half*>(g.W) + (size_t)n0 * K;
      for (int i0 = tid; i0 < NT * CH; i0 += NTH * UNR) {
        int4 v[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
          int idx = i0 + u * NTH;
          if (idx < NT * CH) v[u] = __ldg(reinterpret_cast<const int4*>(wsrc) + idx);
        }
#pragma unroll
        for (int u = 0; u < UNR; u++) {
          int idx = i0 + u * NTH;
          if (idx < NT * CH) {
            int r = idx / CH, j = idx % CH;
            *reinterpret_cast<int4*>(sW + sw128_off(NT, r, j)) = v[u];
          }
        }
      }
    }
    // ---- stage A tile -------------------------------------------------------------------------------------------------
    const bool add_pos = (PRO == PRO_F32) && g.pos_tab != nullptr && ytile < g.pos_ntiles;
    if (PRO == PRO_H16) {
      for (int i0 = tid; i0 < TILE_M * CH; i0 += NTH * UNR) {
        int4 v[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
          int idx = i0 + u * NTH;
          int r = idx / CH, j = idx % CH;
          v[u] = make_int4(0, 0, 0, 0);
          if (idx < TILE_M * CH && row0 + r < M)
            v[u] = *reinterpret_cast<const int4*>((const __half*)g.A + (size_t)(row0 + r) * g.lda + j * 8);
        }
#pragma unroll
        for (int u = 0; u < UNR; u++) {
          int idx = i0 + u * NTH;
          if (idx < TILE_M * CH) {
            int r = idx / CH, j = idx % CH;
            *reinterpret_cast<int4*>(sA + sw128_off(TILE_M, r, j)) = v[u];
          }
        }
      }
    } else {
      constexpr int UF = 4;
      for (int i0 = tid; i0 < TILE_M * CH; i0 += NTH * UF) {
        float4 f0[UF], f1[UF];
        int code[UF];
#pragma unroll
        for (int u = 0; u < UF; u++) {
          int idx = i0 + u * NTH;
          int r = idx / CH, j = idx % CH;
          f0[u] = f1[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          code[u] = 0;
          if (idx < TILE_M * CH && row0 + r < M) {
            const float* ap = (const float*)g.A + (size_t)(row0 + r) * g.lda + j * 8;
            f0[u] = *reinterpret_cast<const float4*>(ap);
            f1[u] = *reinterpret_cast<const float4*>(ap + 4);
            if (add_pos) code[u] = g.pos_code[row0 + r];
          }
        }
#pragma unroll
        for (int u = 0; u < UF; u++) {
          int idx = i0 + u * NTH;
          if (idx < TILE_M * CH) {
            int r = idx / CH, j = idx % CH;
            float f[8] = {f0[u].x, f0[u].y, f0[u].z, f0[u].w, f1[u].x, f1[u].y, f1[u].z, f1[u].w};
            if (add_pos && row0 + r < M) {
              const int k0 = j * 8;
              const int axis = k0 / g.posL;  // posL % 8 == 0 (checked on the host): the chunk lies inside one axis
              if (axis < g.pos_ndim) {
                const int cv = (code[u] >> (8 * axis)) & 255;
                const float4* tp = reinterpret_cast<const float4*>(g.pos_tab + ((size_t)axis * g.pos_maxw + cv) * g.posL + (k0 - axis * g.posL));
                float4 p0 = __ldg(tp), p1 = __ldg(tp + 1);
                f[0] += p0.x; f[1] += p0.y; f[2] += p0.z; f[3] += p0.w;
                f[4] += p1.x; f[5] += p1.y; f[6] += p1.z; f[7] += p1.w;
              }
            }
            *reinterpret_cast<int4*>(sA + sw128_off(TILE_M, r, j)) = pack8_h16<FMT>(f);
          }
        }
      }
    }
    // generic-proxy smem writes -> visible to the tensor core (async proxy)
    fence_async_smem();
    __syncthreads();

    // ---- MMA: warpgroup g computes rows [64 g, 64 g + 64) x NT ------------------------------------------------------------
    {
      const int wg = tid >> 7;
      float acc[NT / 2];
      wg_tile_mma<NT, FMT == FMT_BF16, K / 16>(acc, smem_u32(sA) + wg * 64 * 128, TILE_M * 128, smem_u32(sW), NT * 128, false);
      wgmma_wait<0>();
      __syncthreads();   // both warpgroups are done reading the operands the accumulator tile aliases
      wg_store_acc<NT>(acc, sAcc, NT, wg * 64, 0);
      __syncthreads();
    }

    // ---- epilogue ----------------------------------------------------------------------------------------------------------
    const int half = warp >> 2;                      // warps 0-3: columns [0,NT/2), warps 4-7: [NT/2,NT)
    const int lrow = (warp & 3) * 32 + (tid & 31);   // row inside the tile
    constexpr int CB = NT / 2;
    const int cbeg = half * CB;
    if (EPI == EPI_H16 || EPI == EPI_H16_GELU || EPI == EPI_F16 || EPI == EPI_GELUGRAD) {
      // thread-per-row: bias (+GELU) / gelu' factor, pack, into the 16-bit staging tile [128][NT] (16-byte chunks XOR-swizzled by row)
      constexpr int ECH = NT / 8;
      const bool want_pre = EPI == EPI_H16_GELU && g.out_pre16 != nullptr;
      __half* out16 = reinterpret_cast<__half*>(g.out_h16);
      for (int pass = 0; pass < (want_pre ? 2 : 1); pass++) {   // pass 1 (training only): the pre-activation z
#pragma unroll 1
        for (int c0 = cbeg; c0 < cbeg + CB; c0 += 32) {
          float v[32];
          acc_ld<32>(sAcc, NT, lrow, c0, v);
          uint32_t pk[16];
          const int grow = sRow[lrow];
          if (EPI == EPI_GELUGRAD) {
            const uint4* zp = reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(g.aux16) + (size_t)max(grow, 0) * g.ldo + n0 + c0);
#pragma unroll
            for (int q = 0; q < 4; q++) {
              uint4 z4 = grow >= 0 ? zp[q] : make_uint4(0, 0, 0, 0);
              const uint32_t zz[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
              for (int e = 0; e < 4; e++) {
                const float2 zf = unpack_h16<FMT>(zz[e]);
                pk[4 * q + e] = pack_h16<FMT>(v[8 * q + 2 * e] * gelu_grad(zf.x), v[8 * q + 2 * e + 1] * gelu_grad(zf.y));
              }
            }
          } else {
            const float4* bp = reinterpret_cast<const float4*>(g.bias + n0 + c0);
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              const float4 b4 = g.bias ? __ldg(bp + (i >> 2)) : make_float4(0.f, 0.f, 0.f, 0.f);
              float a0 = v[i] + b4.x, a1 = v[i + 1] + b4.y, a2 = v[i + 2] + b4.z, a3 = v[i + 3] + b4.w;
              if (EPI == EPI_H16_GELU && pass == 0) {
                a0 = gelu_fast(a0);
                a1 = gelu_fast(a1);
                a2 = gelu_fast(a2);
                a3 = gelu_fast(a3);
              }
              pk[i >> 1] = (EPI == EPI_F16) ? pack_f16(a0, a1) : pack_h16<FMT>(a0, a1);
              pk[(i >> 1) + 1] = (EPI == EPI_F16) ? pack_f16(a2, a3) : pack_h16<FMT>(a2, a3);
            }
          }
#pragma unroll
          for (int q = 0; q < 4; q++) {
            int ch = (c0 >> 3) + q;
            *reinterpret_cast<int4*>(sE + (size_t)lrow * NT * 2 + ((ch ^ (lrow & (ECH - 1))) << 4)) =
                make_int4((int)pk[4 * q], (int)pk[4 * q + 1], (int)pk[4 * q + 2], (int)pk[4 * q + 3]);
          }
        }
        __syncthreads();
        __half* dst = pass == 0 ? out16 : reinterpret_cast<__half*>(g.out_pre16);
        for (int idx = tid; idx < TILE_M * ECH; idx += NTH) {
          int r = idx / ECH, ch = idx % ECH;
          int gr = sRow[r];
          if (gr >= 0)
            *reinterpret_cast<int4*>(dst + (size_t)gr * g.ldo + n0 + ch * 8) =
                *reinterpret_cast<const int4*>(sE + (size_t)r * NT * 2 + ((ch ^ (r & (ECH - 1))) << 4));
        }
        if (want_pre) __syncthreads();
      }
    } else {  // EPI_RES_LN / EPI_ADD_F32 : NT == row width, fp32 staging tile [128][NT] (16-byte chunks XOR-swizzled by row)
      constexpr int ECH = NT / 4;  // float4 chunks per row
      static_assert(ECH == 32, "LayerNorm epilogue is written for 128-wide rows");
      // 1. residual tile, coalesced
      for (int i0 = tid; i0 < TILE_M * ECH; i0 += NTH * UNR) {
        float4 v[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
          int idx = i0 + u * NTH;
          int r = idx / ECH, ch = idx % ECH;
          int gr = sRow[r];
          v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (gr >= 0) v[u] = *reinterpret_cast<const float4*>(g.res + (size_t)gr * NT + ch * 4);
        }
#pragma unroll
        for (int u = 0; u < UNR; u++) {
          int idx = i0 + u * NTH;
          int r = idx / ECH, ch = idx % ECH;
          *reinterpret_cast<float4*>(sE + (size_t)r * NT * 4 + ((ch ^ (r & 31)) << 4)) = v[u];
        }
      }
      __syncthreads();
      // 2. thread-per-row: t = acc + bias + residual (kept in the staging tile), row statistics
      float sum = 0.f, sq = 0.f;
#pragma unroll 1
      for (int c0 = cbeg; c0 < cbeg + CB; c0 += 32) {
        float v[32];
        acc_ld<32>(sAcc, NT, lrow, c0, v);
#pragma unroll
        for (int q = 0; q < 8; q++) {
          int ch = (c0 >> 2) + q;
          float4* sp = reinterpret_cast<float4*>(sE + (size_t)lrow * NT * 4 + ((ch ^ (lrow & 31)) << 4));
          float4 r4 = *sp;
          float4 t, b4 = EPI == EPI_ADD_F32 ? make_float4(0.f, 0.f, 0.f, 0.f) : __ldg(reinterpret_cast<const float4*>(g.bias + c0) + q);
          t.x = v[4 * q] + b4.x + r4.x;
          t.y = v[4 * q + 1] + b4.y + r4.y;
          t.z = v[4 * q + 2] + b4.z + r4.z;
          t.w = v[4 * q + 3] + b4.w + r4.w;
          *sp = t;
          sum += (t.x + t.y) + (t.z + t.w);
          sq += (t.x * t.x + t.y * t.y) + (t.z * t.z + t.w * t.w);
        }
      }
      red[half][lrow][0] = sum;
      red[half][lrow][1] = sq;
      __syncthreads();
      if (EPI == EPI_RES_LN && g.out_pre) {   // training: keep the pre-LayerNorm sum for the backward pass
        for (int idx = tid; idx < TILE_M * ECH; idx += NTH) {
          int r = idx / ECH, ch = idx % ECH;
          int gr = sRow[r];
          if (gr >= 0)
            *reinterpret_cast<float4*>(g.out_pre + (size_t)gr * NT + ch * 4) =
                *reinterpret_cast<const float4*>(sE + (size_t)r * NT * 4 + ((ch ^ (r & 31)) << 4));
        }
      }
      sum = red[0][lrow][0] + red[1][lrow][0];
      sq = red[0][lrow][1] + red[1][lrow][1];
      const float mean = sum * (1.0f / NT);
      // E[t^2] - mean^2 loses at most one bit while mean^2 <= E[t^2] / 2; past that (a large common offset in the row) it
      // cancels, and the row's variance comes from its centred values in a second pass over the staged tile.  Both threads of
      // a row see the same sums, so they agree on the branch.
      const bool centred = EPI == EPI_RES_LN && mean * mean > 0.5f * (sq * (1.0f / NT));
      float csq = 0.f;
#pragma unroll 1
      for (int c0 = cbeg; c0 < cbeg + CB && centred; c0 += 4) {
        const int ch = c0 >> 2;
        const float4 t = *reinterpret_cast<const float4*>(sE + (size_t)lrow * NT * 4 + ((ch ^ (lrow & 31)) << 4));
        const float dx = t.x - mean, dy = t.y - mean, dz = t.z - mean, dw = t.w - mean;
        csq += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
      if (EPI == EPI_RES_LN) {   // also orders the pre-LayerNorm stores above before the normalisation overwrites the tile
        red[half][lrow][2] = csq;
        __syncthreads();
      }
      const float var = centred ? (red[0][lrow][2] + red[1][lrow][2]) * (1.0f / NT) : fmaxf(sq * (1.0f / NT) - mean * mean, 0.f);
      const float rstd = rsqrtf(var + g.eps);
#pragma unroll 1
      for (int c0 = cbeg; c0 < cbeg + CB && EPI == EPI_RES_LN; c0 += 4) {
        int ch = c0 >> 2;
        float4* sp = reinterpret_cast<float4*>(sE + (size_t)lrow * NT * 4 + ((ch ^ (lrow & 31)) << 4));
        float4 t = *sp;
        const float4 g4 = __ldg(reinterpret_cast<const float4*>(g.gamma + c0)), b4 = __ldg(reinterpret_cast<const float4*>(g.beta + c0));
        t.x = (t.x - mean) * rstd * g4.x + b4.x;
        t.y = (t.y - mean) * rstd * g4.y + b4.y;
        t.z = (t.z - mean) * rstd * g4.z + b4.z;
        t.w = (t.w - mean) * rstd * g4.w + b4.w;
        *sp = t;
      }
      __syncthreads();
      // 3. coalesced stores: fp32 rows (+ bf16 copy for the next GEMM's A operand)
      for (int idx = tid; idx < TILE_M * ECH; idx += NTH) {
        int r = idx / ECH, ch = idx % ECH;
        int gr = sRow[r];
        if (gr >= 0)
          *reinterpret_cast<float4*>(g.out_f32 + (size_t)gr * NT + ch * 4) =
              *reinterpret_cast<const float4*>(sE + (size_t)r * NT * 4 + ((ch ^ (r & 31)) << 4));
      }
      if (g.out_h16) {
        for (int idx = tid; idx < TILE_M * (NT / 8); idx += NTH) {
          int r = idx / (NT / 8), c8 = idx % (NT / 8);
          int gr = sRow[r];
          if (gr >= 0) {
            float4 a = *reinterpret_cast<const float4*>(sE + (size_t)r * NT * 4 + (((2 * c8) ^ (r & 31)) << 4));
            float4 b = *reinterpret_cast<const float4*>(sE + (size_t)r * NT * 4 + (((2 * c8 + 1) ^ (r & 31)) << 4));
            *reinterpret_cast<int4*>(reinterpret_cast<__half*>(g.out_h16) + (size_t)gr * g.ldo + c8 * 8) = pack8_h16<FMT>(a, b);
          }
        }
      }
    }
    // accumulator tile fully read and the staging tile stored before the next item overwrites them
    __syncthreads();
  }  // item loop
}

template <int K, int NT, int PRO, int EPI, int FMT = FMT_F16>
int launch_wgmma_gemm(sstb200_ctx* c, const GemmArgs& g, int n_tiles_y) {
  size_t ops = (size_t)TILE_M * K * 2 + (size_t)NT * K * 2;
  size_t stage = (EPI == EPI_RES_LN || EPI == EPI_ADD_F32) ? (size_t)TILE_M * NT * 4 : (size_t)TILE_M * NT * 2;
  stage += (size_t)TILE_M * NT * 4;   // + the accumulator tile
  size_t smem = (ops > stage ? ops : stage) + 1024;
  auto kern = wgmma_gemm_kernel<K, NT, PRO, EPI, FMT>;
  static SmemAttr sa;
  CUDA_TRY(c, ensure_smem(c, sa, kern, smem));
  GemmArgs ga = g;
  ga.ny = n_tiles_y;
  int items_cap = ((g.M_cap + TILE_M - 1) / TILE_M) * n_tiles_y;
  int per_sm = (int)((220 * 1024) / (smem + 6144));
  if (per_sm < 1) per_sm = 1;
  int grid = c->num_sms * per_sm;
  if (grid > items_cap) grid = items_cap;
  launch_pdl(kern, dim3(grid), dim3(256), (size_t)(smem), c->stream, ga);
  CUDA_TRY(c, cudaGetLastError());
  return SSTB_OK;
}

}  // namespace
