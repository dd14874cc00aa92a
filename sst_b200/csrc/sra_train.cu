// Training path of the SRA encoder stack (BASELINE config 4): forward that keeps what the backward pass needs, and the
// backward pass itself.  Reference: the autograd graph torch builds over EncoderLayer.forward
// (mmdet3d/models/sst/sst_basic_block_v2.py:100-126 with WindowAttention :41-75 -> nn.MultiheadAttention) for every layer of
// SSTv2.forward (backbones/sst_v2.py:129-133); the reference re-materialises activations per block with torch.utils.checkpoint
// (:132-133), here they are simply kept (131 MB per layer and frame in bf16 / fp32 - nothing on a 180 GB part).
//
// Precision policy (the reference trains under mmcv fp16 autocast with loss_scale 32, configs/sst_refactor/...v2.py:82): GEMM
// operands and saved activations are bf16 (gradients need the fp32 exponent range, so no loss scaling), accumulation, softmax,
// LayerNorm, residual stream, weight gradients and the optimizer state are fp32.
//
// Per layer, forward:   qkv = [x+pos | x] Wqkv^T        wgmma GEMM (csrc/wgmma_gemm.cuh) , q|k|v fp16 for the attention kernel
//                       att = windowed softmax(q k^T) v  csrc/sra_attn.cuh (bf16 output; plain or cosine logits)
//                       x1 = LN1(x + att Wo^T + bo)      wgmma GEMM + LN epilogue, keeps t1   = pre-LN sum
//                       h  = GELU(z), z = x1 W1^T + b1   wgmma GEMM, keeps z  
//                       y  = LN2(x1 + h W2^T + b2)       wgmma GEMM + LN epilogue, keeps t2  
// backward:  LN2' -> dW2, dz = (dt2 W2) * gelu'(z) -> dW1, dx1 = dt2 + dz W1 -> LN1' -> dWo, datt = dt1 Wo -> attention' ->
//            dWqkv, dx = dt1 + dqkv Wqkv.  dX-type GEMMs run on wgmma (transposed bf16 weight copies), dW-type GEMMs (reduction
//            over the ~30 k tokens) on mma.sync tiles (per-split partial blocks + a deterministic reduce), attention' as a two-pass SIMT kernel per window batch.
#include <stdarg.h>
#include <cuda_fp16.h>
#include "sra.cuh"
#include "sra_attn.cuh"
#include "wgmma.cuh"
#include "wgmma_gemm.cuh"

namespace {

constexpr int DM = 128, DFF = 256;

struct TrainLayerWs {   // one layer's saved tensors
  float* y;
  __half* qkv;
  __nv_bfloat16* att;
  float *t1, *x1;
  __nv_bfloat16 *x1b, *z, *h;
  float* t2;
};
struct TrainWs {
  std::vector<TrainLayerWs> layer;
  // shared backward temporaries (after all layers)
  float* dt;
  __nv_bfloat16 *dtb, *dzb, *dattb, *dqkv;
  float *dx1, *dxa, *dxb, *stats;
};

static void train_ws_carve(Carve& cv, TrainWs& w, int n, int L) {
  const size_t N = (size_t)n;
  w.layer.resize(L);
  for (TrainLayerWs& l : w.layer) {
    l.y = cv.take<float>(N * DM);
    l.qkv = cv.take<__half>(N * 3 * DM);
    l.att = cv.take<__nv_bfloat16>(N * DM);
    l.t1 = cv.take<float>(N * DM);
    l.x1 = cv.take<float>(N * DM);
    l.x1b = cv.take<__nv_bfloat16>(N * DM);
    l.z = cv.take<__nv_bfloat16>(N * DFF);
    l.h = cv.take<__nv_bfloat16>(N * DFF);
    l.t2 = cv.take<float>(N * DM);
  }
  w.dt = cv.take<float>(N * DM);
  w.dtb = cv.take<__nv_bfloat16>(N * DM);
  w.dzb = cv.take<__nv_bfloat16>(N * DFF);
  w.dattb = cv.take<__nv_bfloat16>(N * DM);
  w.dqkv = cv.take<__nv_bfloat16>(N * 3 * DM);
  w.dx1 = cv.take<float>(N * DM);
  w.dxa = cv.take<float>(N * DM);
  w.dxb = cv.take<float>(N * DM);
  w.stats = cv.take<float>(N * 8 * 3);
}

static TrainWs train_ws(void* workspace, int n, int L) {
  TrainWs w;
  Carve cv{(char*)workspace, 0};
  train_ws_carve(cv, w, n, L);
  return w;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward over 128-wide rows: dt = rstd * (dy g - mean(dy g) - xhat mean(dy g xhat)), xhat from the saved pre-LN
// sum t, with the variance taken as the forward epilogue takes it: E[t^2] - mean^2 while mean^2 <= E[t^2] / 2 (then the
// subtraction loses at most one bit), else from the centred values in a second pass, so that a large common offset in t does
// not cancel it.  One warp per row (4 columns per lane);
// per-column sums of dy xhat (-> d gamma), dy (-> d beta) and dt (-> d of the bias that was added before the LayerNorm) are
// kept in registers across the warp's rows, summed over the block's warps in a fixed order and written to part[block][3][128];
// ln_reduce_kernel adds the blocks' partials in a fixed order, so two calls give the same bits.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ t, const float* __restrict__ gamma,
                                                     float eps, int n, float* __restrict__ dt, __nv_bfloat16* __restrict__ dtb,
                                                     float* __restrict__ part) {
  pdl_wait();
  pdl_launch();
  __shared__ float red[3][8][DM];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float4 g4 = reinterpret_cast<const float4*>(gamma)[lane];
  float4 sg = make_float4(0.f, 0.f, 0.f, 0.f), sb = sg, st = sg;
  for (int r = blockIdx.x * 8 + warp; r < n; r += gridDim.x * 8) {
    const float4 tv = reinterpret_cast<const float4*>(t + (size_t)r * DM)[lane];
    const float4 dv = reinterpret_cast<const float4*>(dy + (size_t)r * DM)[lane];
    float s = (tv.x + tv.y) + (tv.z + tv.w), q = (tv.x * tv.x + tv.y * tv.y) + (tv.z * tv.z + tv.w * tv.w);
    s = warp_sum(s);
    q = warp_sum(q);
    const float mean = s * (1.0f / DM);
    float var;
    if (mean * mean > 0.5f * (q * (1.0f / DM))) {   // E[t^2] - mean^2 would cancel: second pass over the centred values (warp-uniform)
      const float4 d = make_float4(tv.x - mean, tv.y - mean, tv.z - mean, tv.w - mean);
      var = warp_sum((d.x * d.x + d.y * d.y) + (d.z * d.z + d.w * d.w)) * (1.0f / DM);
    } else {
      var = fmaxf(q * (1.0f / DM) - mean * mean, 0.f);
    }
    const float rstd = rsqrtf(var + eps);
    const float4 xh = make_float4((tv.x - mean) * rstd, (tv.y - mean) * rstd, (tv.z - mean) * rstd, (tv.w - mean) * rstd);
    const float4 dg = make_float4(dv.x * g4.x, dv.y * g4.y, dv.z * g4.z, dv.w * g4.w);
    float c1 = (dg.x + dg.y) + (dg.z + dg.w), c2 = (dg.x * xh.x + dg.y * xh.y) + (dg.z * xh.z + dg.w * xh.w);
    c1 = warp_sum(c1) * (1.0f / DM);
    c2 = warp_sum(c2) * (1.0f / DM);
    const float4 o = make_float4(rstd * (dg.x - c1 - xh.x * c2), rstd * (dg.y - c1 - xh.y * c2), rstd * (dg.z - c1 - xh.z * c2),
                                 rstd * (dg.w - c1 - xh.w * c2));
    reinterpret_cast<float4*>(dt + (size_t)r * DM)[lane] = o;
    __nv_bfloat162 p0 = __floats2bfloat162_rn(o.x, o.y), p1 = __floats2bfloat162_rn(o.z, o.w);
    reinterpret_cast<uint2*>(dtb + (size_t)r * DM)[lane] = make_uint2(*reinterpret_cast<uint32_t*>(&p0), *reinterpret_cast<uint32_t*>(&p1));
    sg.x += dv.x * xh.x, sg.y += dv.y * xh.y, sg.z += dv.z * xh.z, sg.w += dv.w * xh.w;
    sb.x += dv.x, sb.y += dv.y, sb.z += dv.z, sb.w += dv.w;
    st.x += o.x, st.y += o.y, st.z += o.z, st.w += o.w;
  }
  reinterpret_cast<float4*>(red[0][warp])[lane] = sg;
  reinterpret_cast<float4*>(red[1][warp])[lane] = sb;
  reinterpret_cast<float4*>(red[2][warp])[lane] = st;
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * DM; i += 256) {
    const int which = i / DM, col = i % DM;
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) v += red[which][w][col];
    part[(size_t)blockIdx.x * 3 * DM + i] = v;
  }
}

// d gamma / d beta / d bias [col] += sum over the ln_bwd_kernel blocks' partials, in a fixed order.  Block = (sum, 32-column
// group), 12 blocks; warp w adds the partials of blocks w, w + 8, ... for its lane's column, then warp 0 adds the 8 warp sums
// in warp order.
__global__ void __launch_bounds__(256) ln_reduce_kernel(const float* __restrict__ part, int nblk, float* __restrict__ dgamma,
                                                        float* __restrict__ dbeta, float* __restrict__ dbias) {
  pdl_wait();
  pdl_launch();
  __shared__ float red[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + lane, which = blockIdx.x / (DM / 32);   // i indexes [3][128]
  float* dst = which == 0 ? dgamma : (which == 1 ? dbeta : dbias);
  if (!dst) return;   // uniform per block
  float s = 0.f;
#pragma unroll 4
  for (int b = warp; b < nblk; b += 8) s += part[(size_t)b * 3 * DM + i];
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; w++) t += red[w][lane];
    dst[i % DM] += t;
  }
}

static int launch_ln_bwd(sstb200_ctx* c, const float* dy, const float* t, const float* gamma, float eps, int n, float* dt, __nv_bfloat16* dtb,
                         float* dgamma, float* dbeta, float* dbias) {
  const int grid = c->num_sms * 2;
  // per-block partials in the arena; the reduce is enqueued before any later arena_reset can hand the memory out again
  arena_reset(c);
  float* part;
  int rc = arena_carve(c, [&](Carve& cv) { part = cv.take<float>((size_t)grid * 3 * DM); });
  if (rc) return rc;
  CUDA_TRY(c, launch_pdl(ln_bwd_kernel, dim3(grid), dim3(256), (size_t)0, c->stream, dy, t, gamma, eps, n, dt, dtb, part));
  CUDA_TRY(c, launch_pdl(ln_reduce_kernel, dim3(3 * DM / 32), dim3(256), (size_t)0, c->stream, (const float*)part, grid, dgamma, dbeta, dbias));
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// dW[bn*128 + 0..127, bk*128 + 0..127] += dY[:, bn*128 + ..]^T . X[:, bk*128 + ..]   (reduction over the rows)
// Work item = (output block, row split).  A CTA walks its rows in slabs of 64 (cp.async double buffer); 8 warps, warp w owns
// output rows 16w..16w+15 of the block (64 fp32 accumulators per thread); fragments come from the row-major slabs with
// ldmatrix.trans (both operands are "transposed" for mma.sync: the reduction index is the row).  X is either a bf16 matrix or
// the fp32 residual stream (+ positional table) converted while staging.  Each item writes its split's partial block (and the
// bias partials); dw_reduce_kernel adds them to dW in split order, so two calls give the same bits.
// ------------------------------------------------------------------------------------------------
struct DwArgs {
  const __nv_bfloat16* dY;
  int ldy;
  const __nv_bfloat16* X;   // bf16 operand [n, ldx], or nullptr -> Xf
  const float* Xf;          // fp32 operand [n, ldx] (+ pos)
  int ldx;
  const float* pos_tab;
  const int32_t* pos_code;
  int posL, pos_maxw, pos_ndim;
  float* dW;                // [N_out, K_in] fp32, += (by dw_reduce_kernel)
  float* part;              // [splits][nb * kb][128 x 128] fp32 partial blocks
  float* part_b;            // [splits][nb][128] column sums of dY (bias gradient), written by the bk == 0 blocks; or nullptr
  float* db;                // [N_out] fp32, += ; or nullptr
  int K_in;
  int nb, kb, splits, n;
};

constexpr int DW_ROWS = 64, DW_PITCH = 136;   // halfs per staged row (128 + 8 pad: conflict-free ldmatrix)

__global__ void __launch_bounds__(256) dw_gemm_kernel(DwArgs g) {
  pdl_wait();
  pdl_launch();
  extern __shared__ __align__(16) uint8_t dw_smem[];
  __nv_bfloat16* sY = reinterpret_cast<__nv_bfloat16*>(dw_smem);                  // [2][64][136]
  __nv_bfloat16* sX = sY + 2 * DW_ROWS * DW_PITCH;                                // [2][64][136]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int item = blockIdx.x;
  const int blk = item / g.splits, sp = item % g.splits;
  const int bn = blk / g.kb, bk = blk % g.kb;
  const int rows_per = ((g.n + g.splits - 1) / g.splits + DW_ROWS - 1) / DW_ROWS * DW_ROWS;
  const int r_begin = sp * rows_per, r_end = min(g.n, r_begin + rows_per);
  float acc[16][4];
#pragma unroll
  for (int i = 0; i < 16; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
  const bool want_b = g.part_b != nullptr && bk == 0;
  float bsum = 0.f;
  if (r_begin < r_end) {
    auto stage = [&](int buf, int r0) {
      // dY slab: 64 rows x 128 cols bf16 = 16 pieces of 16 B per row
      for (int i = tid; i < DW_ROWS * 16; i += 256) {
        const int r = i >> 4, pc = i & 15;
        const uint32_t dst = smem_u32(sY + (buf * DW_ROWS + r) * DW_PITCH + pc * 8);
        if (r0 + r < r_end) {
          const __nv_bfloat16* src = g.dY + (size_t)(r0 + r) * g.ldy + bn * 128 + pc * 8;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
        } else {
          asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};\n" ::"r"(dst), "r"(0) : "memory");
        }
      }
      if (g.X) {
        for (int i = tid; i < DW_ROWS * 16; i += 256) {
          const int r = i >> 4, pc = i & 15;
          const uint32_t dst = smem_u32(sX + (buf * DW_ROWS + r) * DW_PITCH + pc * 8);
          if (r0 + r < r_end) {
            const __nv_bfloat16* src = g.X + (size_t)(r0 + r) * g.ldx + bk * 128 + pc * 8;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
          } else {
            asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};\n" ::"r"(dst), "r"(0) : "memory");
          }
        }
      } else {   // fp32 rows (+ positional embedding) -> bf16 while staging
        for (int i = tid; i < DW_ROWS * 16; i += 256) {
          const int r = i >> 4, pc = i & 15;
          float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (r0 + r < r_end) {
            const float* src = g.Xf + (size_t)(r0 + r) * g.ldx + bk * 128 + pc * 8;
            const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
            f[0] = a.x, f[1] = a.y, f[2] = a.z, f[3] = a.w, f[4] = b.x, f[5] = b.y, f[6] = b.z, f[7] = b.w;
            if (g.pos_tab) {
              const int k0 = bk * 128 + pc * 8, axis = k0 / g.posL;
              if (axis < g.pos_ndim) {
                const int cv = (g.pos_code[r0 + r] >> (8 * axis)) & 255;
                const float4* tp = reinterpret_cast<const float4*>(g.pos_tab + ((size_t)axis * g.pos_maxw + cv) * g.posL + (k0 - axis * g.posL));
                const float4 p0 = __ldg(tp), p1 = __ldg(tp + 1);
                f[0] += p0.x, f[1] += p0.y, f[2] += p0.z, f[3] += p0.w, f[4] += p1.x, f[5] += p1.y, f[6] += p1.z, f[7] += p1.w;
              }
            }
          }
          *reinterpret_cast<int4*>(sX + (buf * DW_ROWS + r) * DW_PITCH + pc * 8) = pack8_h16<FMT_BF16>(f);
        }
      }
      asm volatile("cp.async.commit_group;\n" ::: "memory");
    };
    stage(0, r_begin);
    int buf = 0;
    // ldmatrix.trans row addresses of this lane inside a 16-row k-step: matrices (k 0-7, c 0-7), (k 0-7, c 8-15), (k 8-15, c 0-7), (k 8-15, c 8-15)
    const int lr = (lane & 7) + ((lane >> 4) & 1) * 8, lc = ((lane >> 3) & 1) * 8;       // A operand: dY^T
    const int br = (lane & 7) + ((lane >> 3) & 1) * 8, bc = (lane >> 4) * 8;              // B operand: X (as V^T in the attention kernel)
    for (int r0 = r_begin; r0 < r_end; r0 += DW_ROWS) {
      if (r0 + DW_ROWS < r_end) stage(buf ^ 1, r0 + DW_ROWS);
      if (r0 + DW_ROWS < r_end) asm volatile("cp.async.wait_group 1;\n" ::: "memory");
      else asm volatile("cp.async.wait_group 0;\n" ::: "memory");
      __syncthreads();
      const __nv_bfloat16* y0 = sY + buf * DW_ROWS * DW_PITCH;
      const __nv_bfloat16* x0 = sX + buf * DW_ROWS * DW_PITCH;
      if (want_b) {   // bias gradient: column tid & 127 over half of the slab's rows
#pragma unroll 8
        for (int r = (tid >> 7) * 32; r < (tid >> 7) * 32 + 32; r++) bsum += __bfloat162float(y0[r * DW_PITCH + (tid & 127)]);
      }
#pragma unroll
      for (int ks = 0; ks < DW_ROWS / 16; ks++) {
        uint32_t a[4];
        {
          const uint32_t addr = smem_u32(y0 + (ks * 16 + lr) * DW_PITCH + warp * 16 + lc);
          uint32_t m0, m1, m2, m3;
          asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(m0), "=r"(m1), "=r"(m2), "=r"(m3) : "r"(addr));
          // matrices arrive as (k0-7,m0-7), (k0-7,m8-15), (k8-15,m0-7), (k8-15,m8-15); the A fragment wants a0=(m0-7,k0-7), a1=(m8-15,k0-7), a2=(m0-7,k8-15), a3=(m8-15,k8-15)
          a[0] = m0, a[1] = m1, a[2] = m2, a[3] = m3;
        }
#pragma unroll
        for (int nt = 0; nt < 8; nt++) {
          const uint32_t addr = smem_u32(x0 + (ks * 16 + br) * DW_PITCH + nt * 16 + bc);
          uint32_t b0, b1, b2, b3;
          asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(b0), "=r"(b1), "=r"(b2), "=r"(b3) : "r"(addr));
          mma_bf16_16816(acc[2 * nt], a, b0, b1);
          mma_bf16_16816(acc[2 * nt + 1], a, b2, b3);
        }
      }
      __syncthreads();
      buf ^= 1;
    }
  }
  // accumulator (row g4 / g4+8 of the warp's 16 rows, columns 8 nt + 2 t4 ..) -> this split's partial block
  const int g4 = lane >> 2, t4 = lane & 3;
  float* base = g.part + ((size_t)sp * (g.nb * g.kb) + blk) * (128 * 128) + (size_t)(warp * 16) * 128;
#pragma unroll
  for (int nt = 0; nt < 16; nt++) {
    const int col = nt * 8 + 2 * t4;
    *reinterpret_cast<float2*>(base + (size_t)g4 * 128 + col) = make_float2(acc[nt][0], acc[nt][1]);
    *reinterpret_cast<float2*>(base + (size_t)(g4 + 8) * 128 + col) = make_float2(acc[nt][2], acc[nt][3]);
  }
  if (want_b) {
    __shared__ float sb2[256];
    sb2[tid] = bsum;
    __syncthreads();
    if (tid < 128) g.part_b[((size_t)sp * g.nb + bn) * 128 + tid] = sb2[tid] + sb2[tid + 128];
  }
}

// dW[block] += sum over the row splits of the partial blocks (deterministic order); same for the bias partials
__global__ void __launch_bounds__(256) dw_reduce_kernel(const float* __restrict__ part, const float* __restrict__ part_b, int splits, int nb, int kb,
                                                        int K_in, float* __restrict__ dW, float* __restrict__ db) {
  pdl_wait();
  pdl_launch();
  const int blocks = nb * kb;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < blocks * 128 * 32; i += gridDim.x * blockDim.x) {
    const int blk = i / (128 * 32), e = i % (128 * 32), r = e / 32, c4 = e % 32;
    const float4* src = reinterpret_cast<const float4*>(part + (size_t)blk * (128 * 128) + (size_t)r * 128) + c4;
    const size_t stride = (size_t)blocks * (128 * 128) / 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    int sp = 0;
    for (; sp + 4 <= splits; sp += 4) {
      const float4 v0 = src[(size_t)sp * stride], v1 = src[(size_t)(sp + 1) * stride], v2 = src[(size_t)(sp + 2) * stride], v3 = src[(size_t)(sp + 3) * stride];
      s.x += (v0.x + v1.x) + (v2.x + v3.x), s.y += (v0.y + v1.y) + (v2.y + v3.y);
      s.z += (v0.z + v1.z) + (v2.z + v3.z), s.w += (v0.w + v1.w) + (v2.w + v3.w);
    }
    for (; sp < splits; sp++) {
      const float4 v = src[(size_t)sp * stride];
      s.x += v.x, s.y += v.y, s.z += v.z, s.w += v.w;
    }
    float4* dst = reinterpret_cast<float4*>(dW + (size_t)((blk / kb) * 128 + r) * K_in + (blk % kb) * 128) + c4;
    float4 d = *dst;
    d.x += s.x, d.y += s.y, d.z += s.z, d.w += s.w;
    *dst = d;
  }
  if (db && part_b) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nb * 128; i += gridDim.x * blockDim.x) {
      float sum = 0.f;
      for (int sp = 0; sp < splits; sp++) sum += part_b[(size_t)sp * nb * 128 + i];
      db[i] += sum;
    }
  }
}

static int launch_dw(sstb200_ctx* c, const __nv_bfloat16* dY, int ldy, int n_out, const __nv_bfloat16* X, const float* Xf, int ldx, int k_in,
                     const sstb200_sra_plan* pos, float* dW, int n, float* db = nullptr) {
  DwArgs g;
  memset(&g, 0, sizeof(g));
  g.dY = dY, g.ldy = ldy, g.X = X, g.Xf = Xf, g.ldx = ldx, g.dW = dW, g.K_in = k_in, g.n = n;
  if (pos) {
    g.pos_tab = pos->pos_table, g.pos_code = pos->pos_code, g.posL = pos->pos_L, g.pos_maxw = pos->pos_maxw, g.pos_ndim = pos->pos_ndim;
  }
  g.nb = n_out / 128, g.kb = k_in / 128;
  const int blocks = g.nb * g.kb;
  g.splits = (2 * c->num_sms + blocks - 1) / blocks;   // two CTAs per SM (88 KB of shared memory each)
  const int max_splits = (n + DW_ROWS - 1) / DW_ROWS;
  if (g.splits > max_splits) g.splits = max_splits < 1 ? 1 : max_splits;
  arena_reset(c);
  int rc = arena_carve(c, [&](Carve& cv) {
    g.part = cv.take<float>((size_t)g.splits * blocks * 128 * 128);
    g.part_b = db ? cv.take<float>((size_t)g.splits * g.nb * 128) : nullptr;
  });
  if (rc) return rc;
  g.db = db;
  const size_t smem = (size_t)4 * DW_ROWS * DW_PITCH * 2;
  static SmemAttr sa;
  CUDA_TRY(c, ensure_smem(c, sa, dw_gemm_kernel, smem));
  CUDA_TRY(c, launch_pdl(dw_gemm_kernel, dim3(blocks * g.splits), dim3(256), smem, c->stream, g));
  CUDA_TRY(c, launch_pdl(dw_reduce_kernel, dim3(blocks * 16), dim3(256), (size_t)0, c->stream, (const float*)g.part, (const float*)g.part_b, g.splits,
                         g.nb, g.kb, k_in, dW, db));
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// Window attention backward (softmax(scale q k^T) v per window and head).  One CTA per (window batch, head pair) like the
// forward kernel; q, k, v (fp16, gathered through the window permutation) and dO (bf16) of the batch's rows are staged in
// shared memory.  Pass A, one thread per (query, head): row maximum / sum, D = dO . O, then dq = scale * sum_j ds_ij k_j with
// ds_ij = p_ij (dO_i . v_j - D_i).  Pass B, one thread per (key, head): dk_j = scale * sum_i ds_ij q_i, dv_j = sum_i p_ij dO_i
// using the row statistics pass A left in shared memory.  No atomics, fp32 math; dq | dk | dv leave as bf16 rows in flat
// token order.
// COS: cosine attention (models/sst/cosine_msa.py:123-185), logits s_ij = c qh_i . kh_j with qh = q iq, kh = k ik,
// iq = 1 / max(|q|, 1e-12), ik likewise, c = 1 / max(tau_h, tau_min).  iq / ik per (row, head) are recomputed from the staged
// fp16 q | k into shared memory, as the forward kernel does.  With g_ij = p_ij (dO_i . v_j - D_i): dqh_i = c sum_j g_ij kh_j and
// dq_i = iq (dqh_i - qh_i (qh_i . dqh_i)), the gradient of F.normalize (q = 0 is the only way the clamp engages for an fp16
// row, and there qh = 0, so the same formula gives dqh / 1e-12); dk symmetrically in pass B.  Pass A also sums g_ij (qh_i . kh_j)
// per head (d loss / d c); each CTA writes its per-head sums to tau_part[blockIdx.x][8] (fixed thread -> row mapping, fixed
// reduction tree), and tau_grad_kernel turns them into d tau.
// ------------------------------------------------------------------------------------------------
constexpr int AB_LD = 40;   // halfs per staged row and tensor (2 heads x 16 + 8 pad)

__device__ __forceinline__ void load16_f16(const __half* p, float* o) {
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    o[2 * i] = f.x;
    o[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void load16_bf16(const __nv_bfloat16* p, float* o) {
  const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    o[2 * i] = f.x;
    o[2 * i + 1] = f.y;
  }
}
__device__ __forceinline__ void store16_bf16(__nv_bfloat16* p, const float* v) {
  uint32_t w[8];
#pragma unroll
  for (int i = 0; i < 8; i++) w[i] = pack_bf16(v[2 * i], v[2 * i + 1]);
  reinterpret_cast<uint4*>(p)[0] = make_uint4(w[0], w[1], w[2], w[3]);
  reinterpret_cast<uint4*>(p)[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

constexpr int AB_NHL = 2, AB_NROW = ATT_BT;   // heads per CTA, staged rows

static size_t attn_bwd_smem(bool cos) {
  size_t b = (size_t)4 * AB_NROW * AB_LD * 2 + (size_t)AB_NROW * AB_NHL * 3 * 4;
  if (cos) b += (size_t)2 * AB_NHL * AB_NROW * 4 + (size_t)8 * AB_NHL * 4 + 8 * 4;   // sInvQ, sInvK, sTRed, sTAcc
  return b;
}

// Parameters after dqkv are read by the COS instantiation only (they come last so that the plain kernel's code is unchanged).
template <bool COS>
__global__ void __launch_bounds__(256) win_attn_bwd_kernel(const __half* __restrict__ qkv, const __nv_bfloat16* __restrict__ att,
                                                           const __nv_bfloat16* __restrict__ datt, const int32_t* __restrict__ counters,
                                                           const int32_t* __restrict__ win_offsets, const int32_t* __restrict__ win_batch,
                                                           const int32_t* __restrict__ tok_perm, float scale, __nv_bfloat16* __restrict__ dqkv,
                                                           const float* __restrict__ tau, int tau_n, float tau_min, float* __restrict__ tau_part) {
  pdl_wait();
  pdl_launch();
  constexpr int D = 128, DH = 16, NHL = AB_NHL, HSPLIT = 4, NROW = AB_NROW;
  extern __shared__ __align__(16) uint8_t ab_smem[];
  __half* sQ = reinterpret_cast<__half*>(ab_smem);
  __half* sK = sQ + NROW * AB_LD;
  __half* sV = sK + NROW * AB_LD;
  __nv_bfloat16* sG = reinterpret_cast<__nv_bfloat16*>(sV + NROW * AB_LD);   // dO
  float* sStat = reinterpret_cast<float*>(sG + NROW * AB_LD);                 // [NROW][NHL][3]: max, 1/sum, D
  // COS only (dynamic shared memory, so that the plain kernel's static layout is unchanged)
  float* sInvQ = sStat + NROW * NHL * 3;   // [NHL][NROW] 1 / max(|q|, 1e-12)
  float* sInvK = sInvQ + NHL * NROW;       // [NHL][NROW] 1 / max(|k|, 1e-12)
  float* sTRed = sInvK + NHL * NROW;       // [8 warps][NHL] per-warp temperature sums of the current unit
  float* sTAcc = sTRed + 8 * NHL;          // [8 heads] this CTA's temperature sums over all its units
  __shared__ int sTok[NROW];
  __shared__ short sKb[NROW], sKe[NROW];   // window key range of every local row
  if (COS && threadIdx.x < 8) sTAcc[threadIdx.x] = 0.f;
  const int nbatch = counters[17];
  for (int unit = blockIdx.x; unit < nbatch * HSPLIT; unit += gridDim.x) {
    const int b = unit / HSPLIT, hs = unit % HSPLIT;
    const int wb = win_batch[4 * b], we = win_batch[4 * b + 1];   // batch record {first window, end window, first slot, end slot}
    if (wb == we) continue;
    const int s0 = win_offsets[wb], s1 = win_offsets[we];
    const int nrow = min(s1 - s0, NROW);
    __syncthreads();
    for (int r = threadIdx.x; r < nrow; r += blockDim.x) sTok[r] = tok_perm[s0 + r];
    for (int w = wb + threadIdx.x; w < we; w += blockDim.x) {
      const int kb = win_offsets[w] - s0, ke = min(win_offsets[w + 1] - s0, NROW);
      for (int r = kb; r < ke; r++) {
        sKb[r] = (short)kb;
        sKe[r] = (short)ke;
      }
    }
    __syncthreads();
    // stage q | k | v | dO for the two heads: 4 pieces of 16 B per row and tensor
    for (int i = threadIdx.x; i < nrow * 16; i += blockDim.x) {
      const int r = i >> 4, c = i & 15, tensor = c >> 2, pc = c & 3;
      const int tok = sTok[r];
      if (tensor < 3) {
        const __half* src = qkv + (size_t)tok * (3 * D) + tensor * D + hs * NHL * DH + pc * 8;
        const uint32_t dst = smem_u32((tensor == 0 ? sQ : (tensor == 1 ? sK : sV)) + r * AB_LD + pc * 8);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
      } else {
        const __nv_bfloat16* src = datt + (size_t)tok * D + hs * NHL * DH + pc * 8;
        const uint32_t dst = smem_u32(sG + r * AB_LD + pc * 8);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(dst), "l"(src) : "memory");
      }
    }
    asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncthreads();
    if (COS) {   // F.normalize(q), F.normalize(k) per head (eps 1e-12) as fp32 factors
      for (int idx = threadIdx.x; idx < nrow * NHL * 2; idx += blockDim.x) {
        const int r = idx >> 2, hl = (idx >> 1) & 1, isk = idx & 1;
        float f[16];
        load16_f16((isk ? sK : sQ) + r * AB_LD + hl * DH, f);
        float ss = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) ss = fmaf(f[d], f[d], ss);
        (isk ? sInvK : sInvQ)[hl * NROW + r] = 1.0f / fmaxf(sqrtf(ss), 1e-12f);
      }
      __syncthreads();
    }
    // ---- pass A: per (query row, head)
    float tsum = 0.f;   // COS: sum of g_ij (qh_i . kh_j) over this thread's rows; its head is hl = threadIdx.x & 1
    for (int it = threadIdx.x; it < nrow * NHL; it += blockDim.x) {
      const int r = it >> 1, hl = it & 1;
      const int kb = sKb[r], ke = sKe[r];
      float q[16], g[16];
      load16_f16(sQ + r * AB_LD + hl * DH, q);
      load16_bf16(sG + r * AB_LD + hl * DH, g);
      float Dv = 0.f;
      if (!COS) {
        float o[16];
        load16_bf16(att + (size_t)sTok[r] * D + (hs * NHL + hl) * DH, o);
#pragma unroll
        for (int d = 0; d < 16; d++) Dv = fmaf(g[d], o[d], Dv);
      }
      // COS: logit = (q . k ik) sc with sc = c iq (the query's factors), so s below is q . kh after the key's factor.  D = dO . O
      // is formed from the recomputed fp32 probabilities (sum_j p_ij dO_i . v_j) rather than from the bf16 output: then
      // sum_j g_ij = 0 holds to fp32 rounding, which d tau - a sum of g_ij (qh_i . kh_j) over every window - depends on.
      float sc = scale, iq = 1.f, cinv = 1.f;
      if (COS) {
        cinv = 1.0f / fmaxf(tau_n > 1 ? tau[hs * NHL + hl] : tau[0], tau_min);
        iq = sInvQ[hl * NROW + r];
        sc = cinv * iq;
      }
      float m = -INFINITY;
      for (int j = kb; j < ke; j++) {
        float k[16];
        load16_f16(sK + j * AB_LD + hl * DH, k);
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) s = fmaf(q[d], k[d], s);
        if (COS) s *= sInvK[hl * NROW + j];
        m = fmaxf(m, s * sc);
      }
      float l = 0.f;
      for (int j = kb; j < ke; j++) {
        float k[16];
        load16_f16(sK + j * AB_LD + hl * DH, k);
        float s = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) s = fmaf(q[d], k[d], s);
        if (COS) {
          float v[16];
          load16_f16(sV + j * AB_LD + hl * DH, v);
          float dp = 0.f;
#pragma unroll
          for (int d = 0; d < 16; d++) dp = fmaf(g[d], v[d], dp);
          s *= sInvK[hl * NROW + j];
          const float e = __expf(s * sc - m);
          l += e;
          Dv = fmaf(e, dp, Dv);
        } else {
          l += __expf(s * sc - m);
        }
      }
      const float il = 1.0f / l;
      if (COS) Dv *= il;
      float dq[16];
#pragma unroll
      for (int d = 0; d < 16; d++) dq[d] = 0.f;
      for (int j = kb; j < ke; j++) {
        float k[16], v[16];
        load16_f16(sK + j * AB_LD + hl * DH, k);
        load16_f16(sV + j * AB_LD + hl * DH, v);
        float s = 0.f, dp = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) {
          s = fmaf(q[d], k[d], s);
          dp = fmaf(g[d], v[d], dp);
        }
        float ds;
        if (COS) {
          const float ik = sInvK[hl * NROW + j];
          s *= ik;
          const float p = __expf(s * sc - m) * il;
          const float gij = p * (dp - Dv);
          tsum = fmaf(gij, s * iq, tsum);   // g_ij (qh_i . kh_j)
          ds = gij * cinv * ik;             // dqh_i = c sum_j g_ij kh_j = sum_j (g_ij c ik_j) k_j
        } else {
          const float p = __expf(s * scale - m) * il;
          ds = p * (dp - Dv) * scale;
        }
#pragma unroll
        for (int d = 0; d < 16; d++) dq[d] = fmaf(ds, k[d], dq[d]);
      }
      if (COS) {   // dq = iq (dqh - qh (qh . dqh))
        float qd = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) qd = fmaf(q[d], dq[d], qd);
        const float t = qd * iq * iq;
#pragma unroll
        for (int d = 0; d < 16; d++) dq[d] = iq * fmaf(-q[d], t, dq[d]);
      }
      sStat[(r * NHL + hl) * 3 + 0] = m;
      sStat[(r * NHL + hl) * 3 + 1] = il;
      sStat[(r * NHL + hl) * 3 + 2] = Dv;
      store16_bf16(dqkv + (size_t)sTok[r] * (3 * D) + (hs * NHL + hl) * DH, dq);
    }
    if (COS) {   // per-warp sums of the two heads (lanes of equal parity share a head)
#pragma unroll
      for (int o2 = 2; o2 < 32; o2 <<= 1) tsum += __shfl_xor_sync(0xffffffffu, tsum, o2);
      if ((threadIdx.x & 31) < NHL) sTRed[(threadIdx.x >> 5) * NHL + (threadIdx.x & 31)] = tsum;
    }
    __syncthreads();
    if (COS && threadIdx.x < NHL) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; w++) t += sTRed[w * NHL + threadIdx.x];
      sTAcc[hs * NHL + threadIdx.x] += t;
    }
    // ---- pass B: per (key row, head)
    for (int it = threadIdx.x; it < nrow * NHL; it += blockDim.x) {
      const int r = it >> 1, hl = it & 1;
      const int kb = sKb[r], ke = sKe[r];
      float k[16], v[16], dk[16], dv[16];
      load16_f16(sK + r * AB_LD + hl * DH, k);
      load16_f16(sV + r * AB_LD + hl * DH, v);
      float ik = 1.f, cinv = 1.f;
      if (COS) {
        cinv = 1.0f / fmaxf(tau_n > 1 ? tau[hs * NHL + hl] : tau[0], tau_min);
        ik = sInvK[hl * NROW + r];
      }
#pragma unroll
      for (int d = 0; d < 16; d++) dk[d] = dv[d] = 0.f;
      for (int i = kb; i < ke; i++) {
        float q[16], g[16];
        load16_f16(sQ + i * AB_LD + hl * DH, q);
        load16_bf16(sG + i * AB_LD + hl * DH, g);
        float s = 0.f, dp = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) {
          s = fmaf(q[d], k[d], s);
          dp = fmaf(g[d], v[d], dp);
        }
        const float* st = sStat + (i * NHL + hl) * 3;
        float p, ds;
        if (COS) {   // the logit exactly as pass A formed it: (q . k ik) (c iq)
          const float iq = sInvQ[hl * NROW + i];
          p = __expf((s * ik) * (cinv * iq) - st[0]) * st[1];
          ds = p * (dp - st[2]) * (cinv * iq);   // dkh_j = c sum_i g_ij qh_i = sum_i (g_ij c iq_i) q_i
        } else {
          p = __expf(s * scale - st[0]) * st[1];
          ds = p * (dp - st[2]) * scale;
        }
#pragma unroll
        for (int d = 0; d < 16; d++) {
          dk[d] = fmaf(ds, q[d], dk[d]);
          dv[d] = fmaf(p, g[d], dv[d]);
        }
      }
      if (COS) {   // dk = ik (dkh - kh (kh . dkh))
        float kd = 0.f;
#pragma unroll
        for (int d = 0; d < 16; d++) kd = fmaf(k[d], dk[d], kd);
        const float t = kd * ik * ik;
#pragma unroll
        for (int d = 0; d < 16; d++) dk[d] = ik * fmaf(-k[d], t, dk[d]);
      }
      __nv_bfloat16* dst = dqkv + (size_t)sTok[r] * (3 * D) + (hs * NHL + hl) * DH;
      store16_bf16(dst + D, dk);
      store16_bf16(dst + 2 * D, dv);
    }
  }
  if (COS) {
    __syncthreads();
    if (threadIdx.x < 8) tau_part[blockIdx.x * 8 + threadIdx.x] = sTAcc[threadIdx.x];
  }
}

// d tau[h] += -c_h^2 sum over the CTAs' partials (sum over all 8 heads when one tau is shared), c_h = 1 / max(tau_h, tau_min);
// 0 where tau_h < tau_min (torch's clamp(min=) passes the gradient at equality).  Fixed summation order: reproducible.
__global__ void tau_grad_kernel(const float* __restrict__ part, int nparts, const float* __restrict__ tau, int tau_n, float tau_min,
                                float* __restrict__ dtau) {
  pdl_wait();
  pdl_launch();
  const int h = threadIdx.x;
  if (h >= tau_n) return;
  const int h0 = tau_n > 1 ? h : 0, h1 = tau_n > 1 ? h + 1 : 8;
  float s = 0.f;
  for (int hh = h0; hh < h1; hh++) {
    float sh = 0.f;
    for (int b = 0; b < nparts; b++) sh += part[(size_t)b * 8 + hh];
    s += sh;
  }
  const float t = tau[h];
  if (t >= tau_min) {
    const float cinv = 1.0f / t;
    dtau[h] = __fadd_rn(dtau[h], -cinv * cinv * s);   // not contracted into an FMA: the call adds exactly its own d tau
  }
}

static int launch_attn_bwd(sstb200_ctx* c, const __half* qkv, const __nv_bfloat16* att, const __nv_bfloat16* datt, const sstb200_sra_plan* P,
                           const sstb200_sra_layer* L, float* dtau, __nv_bfloat16* dqkv) {
  const int grid = c->num_sms * 2;
  if (!L->tau) {
    const size_t smem = attn_bwd_smem(false);
    static SmemAttr sa;
    CUDA_TRY(c, ensure_smem(c, sa, win_attn_bwd_kernel<false>, smem));
    CUDA_TRY(c, launch_pdl(win_attn_bwd_kernel<false>, dim3(grid), dim3(256), smem, c->stream, qkv, att, datt, P->num_windows_dev, P->win_offsets,
                           P->win_batch, P->tok_perm, 0.25f, dqkv, (const float*)nullptr, 0, 0.f, (float*)nullptr));
    return SSTB_OK;
  }
  // per-CTA temperature partials in the arena; the reduce is enqueued before any later arena_reset can hand the memory out again
  arena_reset(c);
  float* part;
  int rc = arena_carve(c, [&](Carve& cv) { part = cv.take<float>((size_t)grid * 8); });
  if (rc) return rc;
  const size_t smem = attn_bwd_smem(true);
  static SmemAttr sb;
  CUDA_TRY(c, ensure_smem(c, sb, win_attn_bwd_kernel<true>, smem));
  CUDA_TRY(c, launch_pdl(win_attn_bwd_kernel<true>, dim3(grid), dim3(256), smem, c->stream, qkv, att, datt, P->num_windows_dev, P->win_offsets,
                         P->win_batch, P->tok_perm, 0.25f, dqkv, L->tau, (int)L->tau_n, L->tau_min, part));
  CUDA_TRY(c, launch_pdl(tau_grad_kernel, dim3(1), dim3(32), (size_t)0, c->stream, (const float*)part, grid, L->tau, (int)L->tau_n, L->tau_min, dtau));
  return SSTB_OK;
}

// fused AdamW over a flat fp32 parameter buffer (torch.optim.AdamW semantics: decoupled weight decay, bias-corrected moments)
__global__ void __launch_bounds__(256) adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                    long long n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2,
                                                    float gscale) {
  pdl_wait();
  pdl_launch();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * gscale;
    float pi = p[i] * (1.0f - lr * wd);
    const float mi = b1 * m[i] + (1.0f - b1) * gi;
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    pi -= lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
    p[i] = pi;
  }
}

static bool layer_ok(const sstb200_sra_layer* L, const sstb200_sra_plan* P) {
  return L->d_model == DM && L->dim_ff == DFF && L->post_norm && !L->norm1_mean && L->act == 2 &&
         (!L->tau || ((L->tau_n == 1 || L->tau_n == 8) && L->tau_min > 0.f)) && L->nhead == 8 && L->in_proj_w_f16 && L->out_proj_w_f16 &&
         L->lin1_w_f16 && L->lin2_w_f16 && P->max_window_tokens > 0 && P->max_window_tokens <= ATT_MAXT && P->num_windows_dev && P->win_batch &&
         (!P->pos_table || P->pos_L % 8 == 0);
}

}  // namespace

extern "C" size_t sstb200_sra_train_workspace_bytes(int n, int num_layers) {
  TrainWs w;
  return carve_bytes([&](Carve& cv) { train_ws_carve(cv, w, n < 1 ? 1 : n, num_layers); });
}

// the 16-bit weight copies in `layers[].*_w_f16` are bf16 for this entry point (see the precision policy above)
extern "C" int sstb200_sra_stack_forward_train(sstb200_ctx* c, const sstb200_sra_layer* layers, int num_layers,
                                               const sstb200_sra_plan* plan_shift0, const sstb200_sra_plan* plan_shift1, const float* x,
                                               float* y_out, void* workspace, int n) {
  CHECK_ARG(c, c && layers && num_layers >= 1 && plan_shift0 && plan_shift1 && x && y_out && workspace && n >= 0);
  if (n == 0) return SSTB_OK;
  const sstb200_sra_plan plans[2] = {*plan_shift0, *plan_shift1};
  for (int l = 0; l < num_layers; l++)
    if (!layer_ok(&layers[l], &plans[l & 1]))
      return sstb_fail(c, SSTB_ERR_UNSUPPORTED,
                       "training path is built for d_model=128, dim_ff=256, 8 heads, post-norm LayerNorm, gelu, plain or cosine attention "
                       "(1 or 8 temperatures, tau_min > 0), windows <= 144 tokens");
  const TrainWs w = train_ws(workspace, n, num_layers);
  const float* xin = x;
  for (int l = 0; l < num_layers; l++) {
    const sstb200_sra_layer* L = &layers[l];
    const sstb200_sra_plan* P = &plans[l & 1];
    const TrainLayerWs& lw = w.layer[l];
    float* y = l + 1 == num_layers ? y_out : lw.y;
    GemmArgs g;
    int rc;
    // 1. q|k|v (fp16 for the attention kernel) from bf16([x+pos | x])
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = xin, g.lda = DM, g.W = L->in_proj_w_f16, g.bias = L->in_proj_b;
    g.pos_tab = P->pos_table, g.pos_code = P->pos_code, g.posL = P->pos_L, g.pos_maxw = P->pos_maxw, g.pos_ndim = P->pos_ndim, g.pos_ntiles = 2;
    g.out_h16 = lw.qkv, g.ldo = 3 * DM;
    if ((rc = launch_wgmma_gemm<128, 128, PRO_F32, EPI_F16, FMT_BF16>(c, g, 3))) return rc;
    // 2. attention (bf16 output)
    if ((rc = sstb_win_attn_batch(c, lw.qkv, P->num_windows_dev, P->win_offsets, P->win_batch, n, P->tok_perm,
                                  lw.att, /*out_bf16=*/true, L->tau, L->tau_n, L->tau_min)))
      return rc;
    // 3. x1 = LN1(x + att Wo^T + bo), keep t1
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = lw.att, g.lda = DM, g.W = L->out_proj_w_f16, g.bias = L->out_proj_b, g.res = xin, g.gamma = L->norm1_w, g.beta = L->norm1_b;
    g.eps = L->norm_eps, g.out_f32 = lw.x1, g.out_h16 = lw.x1b, g.ldo = DM, g.out_pre = lw.t1;
    if ((rc = launch_wgmma_gemm<128, 128, PRO_H16, EPI_RES_LN, FMT_BF16>(c, g, 1))) return rc;
    // 4. h = GELU(z), z = x1 W1^T + b1
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = lw.x1b, g.lda = DM, g.W = L->lin1_w_f16, g.bias = L->lin1_b, g.out_h16 = lw.h, g.out_pre16 = lw.z, g.ldo = DFF;
    if ((rc = launch_wgmma_gemm<128, 128, PRO_H16, EPI_H16_GELU, FMT_BF16>(c, g, 2))) return rc;
    // 5. y = LN2(x1 + h W2^T + b2), keep t2
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = lw.h, g.lda = DFF, g.W = L->lin2_w_f16, g.bias = L->lin2_b, g.res = lw.x1, g.gamma = L->norm2_w;
    g.beta = L->norm2_b, g.eps = L->norm_eps, g.out_f32 = y, g.out_pre = lw.t2;
    if ((rc = launch_wgmma_gemm<256, 128, PRO_H16, EPI_RES_LN, FMT_BF16>(c, g, 1))) return rc;
    xin = y;
  }
  return SSTB_OK;
}

/* wt: bf16 TRANSPOSED weight copies ([in, out] row-major) for the dX GEMMs; grads: fp32 accumulators (+=) */
extern "C" int sstb200_sra_stack_backward(sstb200_ctx* c, const sstb200_sra_layer* layers, const sstb200_sra_layer_wt* wt,
                                          const sstb200_sra_layer_grads* grads, int num_layers, const sstb200_sra_plan* plan_shift0,
                                          const sstb200_sra_plan* plan_shift1, const float* x, void* workspace, const float* dy, float* dx,
                                          int n) {
  CHECK_ARG(c, c && layers && wt && grads && num_layers >= 1 && plan_shift0 && plan_shift1 && x && workspace && dy && dx && n >= 0);
  for (int l = 0; l < num_layers; l++) CHECK_ARG(c, !layers[l].tau || grads[l].tau);   // cosine layers need their d tau accumulator
  if (n == 0) return SSTB_OK;
  const sstb200_sra_plan plans[2] = {*plan_shift0, *plan_shift1};
  const TrainWs w = train_ws(workspace, n, num_layers);
  float* dt = w.dt;
  __nv_bfloat16 *dtb = w.dtb, *dzb = w.dzb, *dattb = w.dattb, *dqkv = w.dqkv;
  float* dx1 = w.dx1;
  float* dxbuf[2] = {w.dxa, w.dxb};
  const float* dcur = dy;
  for (int l = num_layers - 1; l >= 0; l--) {
    const sstb200_sra_layer* L = &layers[l];
    const sstb200_sra_plan* P = &plans[l & 1];
    const sstb200_sra_layer_wt* T = &wt[l];
    const sstb200_sra_layer_grads* G = &grads[l];
    const TrainLayerWs& lw = w.layer[l];
    const float* xin = l == 0 ? x : w.layer[l - 1].y;
    float* dxo = l == 0 ? dx : dxbuf[l & 1];
    GemmArgs g;
    int rc;
    // LN2': dt2 (fp32 + bf16), d gamma2, d beta2, d b2
    if ((rc = launch_ln_bwd(c, dcur, lw.t2, L->norm2_w, L->norm_eps, n, dt, dtb, G->norm2_w, G->norm2_b,
                            G->lin2_b)))
      return rc;
    // dW2 += dt2^T h
    if ((rc = launch_dw(c, dtb, DM, DM, lw.h, nullptr, DFF, DFF, nullptr, G->lin2_w, n))) return rc;
    // dz = (dt2 W2) * gelu'(z)
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = dtb, g.lda = DM, g.W = T->lin2_wt, g.out_h16 = dzb, g.aux16 = lw.z, g.ldo = DFF;
    if ((rc = launch_wgmma_gemm<128, 128, PRO_H16, EPI_GELUGRAD, FMT_BF16>(c, g, 2))) return rc;
    // dW1 += dz^T x1, d b1 += colsum(dz)
    if ((rc = launch_dw(c, dzb, DFF, DFF, lw.x1b, nullptr, DM, DM, nullptr, G->lin1_w, n, G->lin1_b))) return rc;
    // dx1 = dt2 + dz W1
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = dzb, g.lda = DFF, g.W = T->lin1_wt, g.res = dt, g.out_f32 = dx1;
    if ((rc = launch_wgmma_gemm<256, 128, PRO_H16, EPI_ADD_F32, FMT_BF16>(c, g, 1))) return rc;
    // LN1': dt1, d gamma1, d beta1, d bo
    if ((rc = launch_ln_bwd(c, dx1, lw.t1, L->norm1_w, L->norm_eps, n, dt, dtb, G->norm1_w, G->norm1_b,
                            G->out_proj_b)))
      return rc;
    // dWo += dt1^T att ;  datt = dt1 Wo
    if ((rc = launch_dw(c, dtb, DM, DM, lw.att, nullptr, DM, DM, nullptr, G->out_proj_w, n))) return rc;
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = dtb, g.lda = DM, g.W = T->out_proj_wt, g.bias = nullptr, g.out_h16 = dattb, g.ldo = DM;
    if ((rc = launch_wgmma_gemm<128, 128, PRO_H16, EPI_H16, FMT_BF16>(c, g, 1))) return rc;
    // attention'
    if ((rc = launch_attn_bwd(c, lw.qkv, lw.att, dattb, P, L, G->tau,
                              dqkv)))
      return rc;
    // dWq|k += [dq|dk]^T (x + pos) ;  dWv += dv^T x ;  d bqkv += colsum(dqkv)
    if ((rc = launch_dw(c, dqkv, 3 * DM, 2 * DM, nullptr, xin, DM, DM, P->pos_table ? P : nullptr, G->in_proj_w, n, G->in_proj_b))) return rc;
    if ((rc = launch_dw(c, dqkv + 2 * DM, 3 * DM, DM, nullptr, xin, DM, DM, nullptr, G->in_proj_w + (size_t)2 * DM * DM, n, G->in_proj_b + 2 * DM)))
      return rc;
    // dx = dt1 + dqkv Wqkv
    memset(&g, 0, sizeof(g));
    g.M_cap = n, g.A = dqkv, g.lda = 3 * DM, g.W = T->in_proj_wt, g.res = dt, g.out_f32 = dxo;
    if ((rc = launch_wgmma_gemm<384, 128, PRO_H16, EPI_ADD_F32, FMT_BF16>(c, g, 1))) return rc;
    dcur = dxo;
  }
  return SSTB_OK;
}

extern "C" int sstb200_adamw_step(sstb200_ctx* c, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long long n, float lr,
                                  float beta1, float beta2, float eps, float weight_decay, int step, float grad_scale) {
  CHECK_ARG(c, c && params && grads && exp_avg && exp_avg_sq && n >= 0 && step >= 1);
  if (n == 0) return SSTB_OK;
  const float bc1 = 1.0f - powf(beta1, (float)step), bc2 = 1.0f - powf(beta2, (float)step);
  CUDA_TRY(c, launch_pdl(adamw_kernel, dim3(c->num_sms * 4), dim3(256), (size_t)0, c->stream, params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2,
                         eps, weight_decay, bc1, bc2, grad_scale));
  return SSTB_OK;
}
