// Deformable convolution (mmcv 1.3.8-1.4.0 deform_conv2d, the 'DCN' = DeformConv2dPack of CenterHead's DCNSeparateHead), fp32.
//
// Forward: one implicit GEMM per (pixel tile, conv group, output tile).  The input is transposed to NHWC once, so that a bilinear corner's
// channels are one contiguous load.  Each 16-deep slice of the reduction (tap-major: r = k * Cg + c) is sampled straight into shared
// memory - coordinates, the four corner loads and the blend - and multiplied by the group's weight slice with fp32 FFMA: no
// [Cin * K, Ho * Wo] column buffer goes to HBM.
//
// Backward (one call, no float atomics, bit-identical from run to run; the forward saves nothing, the backward re-samples):
//   grad_weight  split-K over fixed pixel chunks: every chunk writes its partial [Cout, Cg, K] block, one pass sums them in chunk order;
//   grad_offset  one warp per (output pixel, deformable group): lanes over channels, grad_col = W^T grad_y formed on the fly, the
//                channel sum is a fixed shuffle tree;
//   grad_x       the sample -> input-pixel relation inverted: every (sample, corner) with a non-zero weight emits (input pixel, sample id),
//                a radix sort makes each input pixel's contributions one contiguous run in sample order (a CSR), and one warp per
//                input pixel sums its run in that order.
#include <stdarg.h>
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"

namespace {

struct DcnGeom {
  int N, C, H, W, O, kh, kw, sh, sw, ph, pw, dh, dw, G, D;  // the 15 entries of the ABI's geom[]
  int Ho, Wo, K, Cg, Og, Cd;
  long long HoWo, NP;  // output pixels per image, in the call
};

#define DCN_THREADS 256
#define DCN_CC 16        // reduction depth of one staged slice
#define DCN_DW_SP 64     // pixels per staged step of the grad_weight kernel
#define DCN_DW_CHUNK 2048  // pixels per grad_weight split

// one sample point: the four corners' NHWC element offsets (-1 = outside the image) and bilinear weights, plus the position's fractions
struct Samp {
  long long idx[4];
  float w[4];
  float lh, lw;
  bool valid;
};

// p = (integer base) + offset as one fp32 addition; S = 0 unless -1 < p_h < H and -1 < p_w < W; corners floor(p) and floor(p) + 1
__device__ __forceinline__ Samp dcn_sample(const DcnGeom& g, const float* __restrict__ off, int n, long long pix, int k, int d) {
  Samp s;
  const int ho = (int)(pix / g.Wo), wo = (int)(pix - (long long)ho * g.Wo);
  const int ki = k / g.kw, kj = k - ki * g.kw;
  const float* o = off + ((size_t)(n * g.D + d) * 2 * g.K + 2 * k) * g.HoWo + pix;
  const float ph = (float)(ho * g.sh - g.ph + ki * g.dh) + __ldg(o);
  const float pw = (float)(wo * g.sw - g.pw + kj * g.dw) + __ldg(o + g.HoWo);
  s.valid = ph > -1.f && pw > -1.f && ph < (float)g.H && pw < (float)g.W;
  const float fh = floorf(ph), fw = floorf(pw);
  s.lh = s.valid ? ph - fh : 0.f;
  s.lw = s.valid ? pw - fw : 0.f;
  const int h0 = s.valid ? (int)fh : -2, w0 = s.valid ? (int)fw : -2;
  const float hh = 1.f - s.lh, hw = 1.f - s.lw;
  s.w[0] = hh * hw, s.w[1] = hh * s.lw, s.w[2] = s.lh * hw, s.w[3] = s.lh * s.lw;
#pragma unroll
  for (int q = 0; q < 4; q++) {
    const int h = h0 + (q >> 1), w = w0 + (q & 1);
    const bool in = s.valid && h >= 0 && w >= 0 && h < g.H && w < g.W;
    s.idx[q] = in ? (((long long)n * g.H + h) * g.W + w) * g.C : -1;
  }
  return s;
}

__device__ __forceinline__ float corner(const float* __restrict__ xT, long long idx, int c) { return idx >= 0 ? __ldg(xT + idx + c) : 0.f; }

__device__ __forceinline__ float dcn_value(const Samp& s, const float* __restrict__ xT, int c) {
  if (!s.valid) return 0.f;
  return s.w[0] * corner(xT, s.idx[0], c) + s.w[1] * corner(xT, s.idx[1], c) + s.w[2] * corner(xT, s.idx[2], c) +
         s.w[3] * corner(xT, s.idx[3], c);
}

// [N, C, HW] -> [N, HW, C] through 32 x 33 shared tiles
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const float* __restrict__ in, int C, long long HW, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  __shared__ float t[32][33];
  const int n = blockIdx.z;
  const long long p0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const float* src = in + (size_t)n * C * HW;
  float* dst = out + (size_t)n * C * HW;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i;
    const long long p = p0 + threadIdx.x;
    if (c < C && p < HW) t[i][threadIdx.x] = src[(size_t)c * HW + p];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const long long p = p0 + i;
    const int c = c0 + threadIdx.x;
    if (c < C && p < HW) dst[(size_t)p * C + c] = t[threadIdx.x][i];
  }
}

// forward: block = BM = 4096 / BN output pixels x BN outputs of one group; thread = 4 pixels x 4 outputs
template <int BN>
__global__ void __launch_bounds__(DCN_THREADS) dcn_fwd_kernel(DcnGeom g, const float* __restrict__ xT, const float* __restrict__ off,
                                                              const float* __restrict__ wt, int otiles, float* __restrict__ y) {
  pdl_wait();
  pdl_launch();
  constexpr int BM = 4096 / BN, TP = BM / 4;
  __shared__ __align__(16) float S[DCN_CC][BM];
  __shared__ __align__(16) float Wsm[DCN_CC][BN];
  const int tid = threadIdx.x, tp = tid % TP, to = tid / TP;
  const long long P0 = (long long)blockIdx.x * BM;
  const int gi = blockIdx.y / otiles, o0 = gi * g.Og + (blockIdx.y % otiles) * BN;
  const int on = min(BN, (gi + 1) * g.Og - o0);
  const int R = g.Cg * g.K;
  float acc[4][4] = {};
  for (int r0 = 0; r0 < R; r0 += DCN_CC) {
    for (int e = tid; e < DCN_CC * BM; e += DCN_THREADS) {
      const int cc = e % DCN_CC, px = e / DCN_CC, r = r0 + cc;
      const long long P = P0 + px;
      float v = 0.f;
      if (r < R && P < g.NP) {
        const int k = r / g.Cg, c = gi * g.Cg + (r - k * g.Cg);
        const int n = (int)(P / g.HoWo);
        const Samp s = dcn_sample(g, off, n, P - (long long)n * g.HoWo, k, c / g.Cd);
        v = dcn_value(s, xT, c);
      }
      S[cc][px] = v;
    }
    for (int e = tid; e < DCN_CC * BN; e += DCN_THREADS) {
      const int oo = e % BN, cc = e / BN, r = r0 + cc;
      float v = 0.f;
      if (r < R && oo < on) {
        const int k = r / g.Cg, cl = r - k * g.Cg;
        v = __ldg(wt + ((size_t)(o0 + oo) * g.Cg + cl) * g.K + k);
      }
      Wsm[cc][oo] = v;
    }
    __syncthreads();
#pragma unroll
    for (int cc = 0; cc < DCN_CC; cc++) {
      const float4 a = *reinterpret_cast<const float4*>(&S[cc][tp * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Wsm[cc][to * 4]);
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
    const long long P = P0 + tp * 4 + i;
    if (P >= g.NP) break;
    const int n = (int)(P / g.HoWo);
    const long long pix = P - (long long)n * g.HoWo;
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (to * 4 + j < on) y[((size_t)n * g.O + o0 + to * 4 + j) * g.HoWo + pix] = acc[i][j];
  }
}

// grad_weight, split-K: block = (pixel chunk, 16-deep reduction slice of one group, BN outputs); thread = 4 r x 4 o on every
// (256 / BN)-th pixel, the pixel lanes summed in lane order at the end.  part[split][o][cl][k].
template <int BN>
__global__ void __launch_bounds__(DCN_THREADS) dcn_dw_kernel(DcnGeom g, const float* __restrict__ xT, const float* __restrict__ off,
                                                             const float* __restrict__ gyT, int rchunks, float* __restrict__ part) {
  pdl_wait();
  pdl_launch();
  constexpr int PL = DCN_THREADS / BN, QO = BN / 4;
  __shared__ __align__(16) float S[DCN_DW_SP][DCN_CC];
  __shared__ __align__(16) float Gs[DCN_DW_SP][BN];
  __shared__ float red[PL][BN * 16 + 1];
  const int tid = threadIdx.x, q = tid % BN, pl = tid / BN, rq = q / QO, oq = q % QO;
  const int gi = blockIdx.y / rchunks, r0 = (blockIdx.y % rchunks) * DCN_CC;
  const int o0 = gi * g.Og + blockIdx.z * BN, on = min(BN, (gi + 1) * g.Og - o0);
  const int R = g.Cg * g.K;
  const long long Pbeg = (long long)blockIdx.x * DCN_DW_CHUNK, Pend = min(Pbeg + DCN_DW_CHUNK, g.NP);
  float acc[4][4] = {};
  for (long long P0 = Pbeg; P0 < Pend; P0 += DCN_DW_SP) {
    for (int e = tid; e < DCN_DW_SP * DCN_CC; e += DCN_THREADS) {
      const int cc = e % DCN_CC, px = e / DCN_CC, r = r0 + cc;
      const long long P = P0 + px;
      float v = 0.f;
      if (r < R && P < Pend) {
        const int k = r / g.Cg, c = gi * g.Cg + (r - k * g.Cg);
        const int n = (int)(P / g.HoWo);
        const Samp s = dcn_sample(g, off, n, P - (long long)n * g.HoWo, k, c / g.Cd);
        v = dcn_value(s, xT, c);
      }
      S[px][cc] = v;
    }
    for (int e = tid; e < DCN_DW_SP * BN; e += DCN_THREADS) {
      const int oo = e % BN, px = e / BN;
      const long long P = P0 + px;
      Gs[px][oo] = (oo < on && P < Pend) ? __ldg(gyT + (size_t)P * g.O + o0 + oo) : 0.f;
    }
    __syncthreads();
    for (int px = pl; px < DCN_DW_SP; px += PL) {
      const float4 a = *reinterpret_cast<const float4*>(&S[px][rq * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Gs[px][oq * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) red[pl][q * 16 + i * 4 + j] = acc[i][j];
  __syncthreads();
  float* dst = part + (size_t)blockIdx.x * g.O * R;
  for (int e = tid; e < BN * 16; e += DCN_THREADS) {
    const int qq = e / 16, i = (e / 4) % 4, j = e % 4;
    const int r = r0 + (qq / QO) * 4 + i, oo = (qq % QO) * 4 + j;
    if (r >= R || oo >= on) continue;
    float sum = 0.f;
    for (int l = 0; l < PL; l++) sum += red[l][e];
    const int k = r / g.Cg, cl = r - k * g.Cg;
    dst[((size_t)(o0 + oo) * g.Cg + cl) * g.K + k] = sum;
  }
}

__global__ void dcn_dw_reduce_kernel(const float* __restrict__ part, int splits, long long n, float* __restrict__ gw) {
  pdl_wait();
  pdl_launch();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int b = 0; b < splits; b++) s += part[(size_t)b * n + i];
  gw[i] = s;
}

// grad_col[c, k, P] = sum over the outputs o of c's group of W[o, cl, k] grad_y[P, o]
__device__ __forceinline__ float dcn_grad_col(const DcnGeom& g, const float* __restrict__ wt, const float* __restrict__ gyT, long long P,
                                              int c, int k) {
  const int gi = c / g.Cg, cl = c - gi * g.Cg;
  const float* w = wt + ((size_t)gi * g.Og * g.Cg + cl) * g.K + k;
  const float* gy = gyT + (size_t)P * g.O + gi * g.Og;
  float s = 0.f;
  for (int o = 0; o < g.Og; o++) s = fmaf(__ldg(w + (size_t)o * g.Cg * g.K), __ldg(gy + o), s);
  return s;
}

// grad_offset: one warp per (output pixel P, deformable group d); dS/dp with the corners held at floor(p)
__global__ void __launch_bounds__(DCN_THREADS) dcn_doff_kernel(DcnGeom g, const float* __restrict__ xT, const float* __restrict__ off,
                                                               const float* __restrict__ wt, const float* __restrict__ gyT,
                                                               float* __restrict__ goff) {
  pdl_wait();
  pdl_launch();
  const long long wid = ((long long)blockIdx.x * DCN_THREADS + threadIdx.x) >> 5;
  if (wid >= g.NP * g.D) return;
  const int lane = lane_id();
  const long long P = wid / g.D;
  const int d = (int)(wid - P * g.D);
  const int n = (int)(P / g.HoWo);
  const long long pix = P - (long long)n * g.HoWo;
  for (int k = 0; k < g.K; k++) {
    const Samp s = dcn_sample(g, off, n, pix, k, d);
    float gh = 0.f, gw = 0.f;
    if (s.valid) {
      const float hh = 1.f - s.lh, hw = 1.f - s.lw;
      for (int cl = lane; cl < g.Cd; cl += 32) {
        const int c = d * g.Cd + cl;
        const float gc = dcn_grad_col(g, wt, gyT, P, c, k);
        const float v1 = corner(xT, s.idx[0], c), v2 = corner(xT, s.idx[1], c), v3 = corner(xT, s.idx[2], c), v4 = corner(xT, s.idx[3], c);
        gh = fmaf(gc, hw * (v3 - v1) + s.lw * (v4 - v2), gh);
        gw = fmaf(gc, hh * (v2 - v1) + s.lh * (v4 - v3), gw);
      }
    }
    gh = warp_sum(gh);
    gw = warp_sum(gw);
    if (lane == 0) {
      float* o = goff + ((size_t)(n * g.D + d) * 2 * g.K + 2 * k) * g.HoWo + pix;
      o[0] = gh;
      o[g.HoWo] = gw;
    }
  }
}

// grad_x, part 1: every (sample, corner) with a non-zero weight inside the image emits key = its input pixel ((n, d, h, w) flattened) and
// value = 4 * sample + corner, sample = ((n * D + d) * K + k) * HoWo + pix; the rest get the key `none`, sorted past every pixel
__global__ void dcn_keys_kernel(DcnGeom g, const float* __restrict__ off, long long samples, uint32_t none, uint32_t* __restrict__ keys,
                                uint32_t* __restrict__ vals) {
  pdl_wait();
  pdl_launch();
  const long long sid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (sid >= samples) return;
  const long long pix = sid % g.HoWo, t = sid / g.HoWo;
  const int k = (int)(t % g.K), nd = (int)(t / g.K), n = nd / g.D, d = nd - n * g.D;
  const Samp s = dcn_sample(g, off, n, pix, k, d);
#pragma unroll
  for (int q = 0; q < 4; q++) {
    uint32_t key = none;
    if (s.idx[q] >= 0 && s.w[q] != 0.f) key = (uint32_t)((long long)nd * g.H * g.W + s.idx[q] / g.C - (long long)n * g.H * g.W);
    keys[4 * sid + q] = key;
    vals[4 * sid + q] = (uint32_t)(4 * sid + q);
  }
}

// grad_x, part 2: one warp per input pixel (n, d, h, w); lanes over d's channels; the pixel's run of the sorted keys summed in order
__global__ void __launch_bounds__(DCN_THREADS) dcn_dx_kernel(DcnGeom g, const float* __restrict__ off, const float* __restrict__ wt,
                                                             const float* __restrict__ gyT, const uint32_t* __restrict__ skeys,
                                                             const uint32_t* __restrict__ svals, long long M, float* __restrict__ gx) {
  pdl_wait();
  pdl_launch();
  const long long wid = ((long long)blockIdx.x * DCN_THREADS + threadIdx.x) >> 5;
  const long long HW = (long long)g.H * g.W;
  if (wid >= (long long)g.N * g.D * HW) return;
  const int lane = lane_id();
  const int nd = (int)(wid / HW), n = nd / g.D, d = nd - n * g.D;
  const long long hw = wid - (long long)nd * HW;
  long long lo = 0, hi = M;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (skeys[mid] < (uint32_t)wid) lo = mid + 1;
    else hi = mid;
  }
  long long end = lo;
  while (end < M && skeys[end] == (uint32_t)wid) end++;
  for (int cl = lane; cl < g.Cd; cl += 32) {
    const int c = d * g.Cd + cl;
    float acc = 0.f;
    for (long long j = lo; j < end; j++) {
      const uint32_t v = svals[j];
      const long long sid = v >> 2;
      const long long pix = sid % g.HoWo;
      const int k = (int)((sid / g.HoWo) % g.K);
      const Samp s = dcn_sample(g, off, n, pix, k, d);
      const uint32_t q = v & 3;
      const float w = q == 0 ? s.w[0] : q == 1 ? s.w[1] : q == 2 ? s.w[2] : s.w[3];
      acc = fmaf(w, dcn_grad_col(g, wt, gyT, (long long)n * g.HoWo + pix, c, k), acc);
    }
    gx[((size_t)n * g.C + c) * HW + hw] = acc;
  }
}

int dcn_geom(sstb200_ctx* c, const int32_t* a, DcnGeom& g) {
  CHECK_ARG(c, c && a);
  g.N = a[0], g.C = a[1], g.H = a[2], g.W = a[3], g.O = a[4], g.kh = a[5], g.kw = a[6], g.sh = a[7], g.sw = a[8];
  g.ph = a[9], g.pw = a[10], g.dh = a[11], g.dw = a[12], g.G = a[13], g.D = a[14];
  if (g.N < 1 || g.C < 1 || g.H < 1 || g.W < 1 || g.O < 1 || g.kh < 1 || g.kw < 1 || g.sh < 1 || g.sw < 1 || g.ph < 0 || g.pw < 0 ||
      g.dh < 1 || g.dw < 1 || g.G < 1 || g.D < 1)
    return sstb_fail(c, SSTB_ERR_ARG, "dcn: non-positive size in geom (negative padding or a size < 1)");
  if (g.C % g.G || g.O % g.G || g.C % g.D)
    return sstb_fail(c, SSTB_ERR_ARG, "dcn: Cin %d and Cout %d must divide by groups %d, Cin by deform_groups %d", g.C, g.O, g.G, g.D);
  g.Ho = (g.H + 2 * g.ph - (g.dh * (g.kh - 1) + 1)) / g.sh + 1;
  g.Wo = (g.W + 2 * g.pw - (g.dw * (g.kw - 1) + 1)) / g.sw + 1;
  if (g.H + 2 * g.ph < g.dh * (g.kh - 1) + 1 || g.W + 2 * g.pw < g.dw * (g.kw - 1) + 1)
    return sstb_fail(c, SSTB_ERR_ARG, "dcn: the dilated kernel is larger than the padded input");
  g.K = g.kh * g.kw, g.Cg = g.C / g.G, g.Og = g.O / g.G, g.Cd = g.C / g.D;
  g.HoWo = (long long)g.Ho * g.Wo;
  g.NP = (long long)g.N * g.HoWo;
  const long long samples = g.NP * g.D * g.K;
  if (4 * samples >= 0xffffffffll || (long long)g.N * g.D * g.H * g.W >= 0xffffffffll || g.NP * g.D > 0x7fffffffll * 8 ||
      (long long)g.G * ((g.Cg * g.K + DCN_CC - 1) / DCN_CC) > 65535 || (long long)g.G * ((g.Og + 15) / 16) > 65535 || g.N > 65535)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "dcn: %lld samples / %d images exceed the 32-bit sample index or the grid", samples, g.N);
  return SSTB_OK;
}

// the backward sorts M = 4 N dg K Ho Wo (key, value) pairs, and cub's radix sort takes an int item count
int dcn_bwd_geom(sstb200_ctx* c, const int32_t* a, DcnGeom& g) {
  const int rc = dcn_geom(c, a, g);
  if (rc) return rc;
  const long long M = 4 * g.NP * g.D * g.K;
  if (M > 0x7fffffffll)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "dcn_backward: %lld sample corners exceed the radix sort's 2^31 - 1 items", M);
  return SSTB_OK;
}

int dcn_bn(int Og) { return Og <= 16 ? 16 : Og <= 32 ? 32 : 64; }

cudaError_t launch_nhwc(cudaStream_t st, const float* in, int N, int C, long long HW, float* out) {
  return launch_pdl(nchw_to_nhwc_kernel, dim3((unsigned)((HW + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)N), dim3(32, 8), (size_t)0, st,
                    in, C, HW, out);
}

int bits_for(long long n) {  // bits to hold 0 .. n - 1
  int b = 0;
  while (b < 32 && (1ll << b) < n) b++;
  return b;
}

// the backward's caller-owned workspace: dcn_bwd_ws sizes it, dcn_bwd_carve lays it out
struct DcnBwdWs {
  long long M;  // 4 * samples
  int splits, end_bit;
  size_t cub_bytes;
  float *xT, *gyT, *part;
  uint32_t *keys, *vals, *skeys, *svals;
  uint8_t* cub;
};

DcnBwdWs dcn_bwd_ws(const DcnGeom& g) {
  DcnBwdWs l;
  l.M = 4 * g.NP * g.D * g.K;
  l.splits = (int)((g.NP + DCN_DW_CHUNK - 1) / DCN_DW_CHUNK);
  l.end_bit = max(1, bits_for((long long)g.N * g.D * g.H * g.W + 1));
  l.cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, l.cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int)l.M, 0, l.end_bit, (cudaStream_t)0);
  return l;
}

void dcn_bwd_carve(Carve& cv, DcnBwdWs& l, const DcnGeom& g) {
  l.xT = cv.take<float>((size_t)g.N * g.H * g.W * g.C);
  l.gyT = cv.take<float>((size_t)g.NP * g.O);
  l.keys = cv.take<uint32_t>(l.M);
  l.vals = cv.take<uint32_t>(l.M);
  l.skeys = cv.take<uint32_t>(l.M);
  l.svals = cv.take<uint32_t>(l.M);
  l.cub = cv.take<uint8_t>(l.cub_bytes + 16);
  l.part = cv.take<float>((size_t)l.splits * g.O * g.Cg * g.K);
}

size_t dcn_bwd_bytes(DcnBwdWs l, const DcnGeom& g) {
  return carve_bytes([&](Carve& cv) { dcn_bwd_carve(cv, l, g); });
}

}  // namespace

extern "C" int sstb200_dcn_forward(sstb200_ctx* c, const int32_t geom[15], const float* x, const float* offset, const float* weight, float* y) {
  DcnGeom g;
  int rc = dcn_geom(c, geom, g);
  if (rc) return rc;
  CHECK_ARG(c, x && offset && weight && y);
  arena_reset(c);
  float* xT;
  rc = arena_carve(c, [&](Carve& cv) { xT = cv.take<float>((size_t)g.N * g.H * g.W * g.C); });
  if (rc) return rc;
  cudaStream_t st = c->stream;
  CUDA_TRY(c, launch_nhwc(st, x, g.N, g.C, (long long)g.H * g.W, xT));
  const int BN = dcn_bn(g.Og), otiles = (g.Og + BN - 1) / BN;
  const long long blocks = (g.NP + 4096 / BN - 1) / (4096 / BN);
  const dim3 grid((unsigned)blocks, (unsigned)(g.G * otiles));
  if (BN == 16) CUDA_TRY(c, launch_pdl(dcn_fwd_kernel<16>, grid, dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset, weight, otiles, y));
  else if (BN == 32) CUDA_TRY(c, launch_pdl(dcn_fwd_kernel<32>, grid, dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset, weight, otiles, y));
  else CUDA_TRY(c, launch_pdl(dcn_fwd_kernel<64>, grid, dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset, weight, otiles, y));
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_dcn_backward_workspace_bytes(sstb200_ctx* c, const int32_t geom[15], int64_t* bytes) {
  DcnGeom g;
  int rc = dcn_bwd_geom(c, geom, g);
  if (rc) return rc;
  CHECK_ARG(c, bytes);
  *bytes = (int64_t)dcn_bwd_bytes(dcn_bwd_ws(g), g);
  return SSTB_OK;
}

extern "C" int sstb200_dcn_backward(sstb200_ctx* c, const int32_t geom[15], const float* x, const float* offset, const float* weight,
                                    const float* grad_y, void* workspace, int64_t workspace_bytes, float* grad_x, float* grad_offset,
                                    float* grad_weight) {
  DcnGeom g;
  int rc = dcn_bwd_geom(c, geom, g);
  if (rc) return rc;
  CHECK_ARG(c, x && offset && weight && grad_y && workspace);
  DcnBwdWs l = dcn_bwd_ws(g);
  const size_t need = dcn_bwd_bytes(l, g);
  if (workspace_bytes < (int64_t)need)
    return sstb_fail(c, SSTB_ERR_WORKSPACE, "dcn_backward: workspace of %lld bytes, %zu needed", (long long)workspace_bytes, need);
  Carve wc{(char*)workspace, 0};
  dcn_bwd_carve(wc, l, g);
  float *xT = l.xT, *gyT = l.gyT;
  cudaStream_t st = c->stream;
  CUDA_TRY(c, launch_nhwc(st, x, g.N, g.C, (long long)g.H * g.W, xT));
  CUDA_TRY(c, launch_nhwc(st, grad_y, g.N, g.O, g.HoWo, gyT));
  if (grad_weight) {
    const int BN = dcn_bn(g.Og), otiles = (g.Og + BN - 1) / BN, rchunks = (g.Cg * g.K + DCN_CC - 1) / DCN_CC;
    float* part = l.part;
    const dim3 grid((unsigned)l.splits, (unsigned)(g.G * rchunks), (unsigned)otiles);
    if (BN == 16) CUDA_TRY(c, launch_pdl(dcn_dw_kernel<16>, grid, dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset, (const float*)gyT, rchunks, part));
    else if (BN == 32) CUDA_TRY(c, launch_pdl(dcn_dw_kernel<32>, grid, dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset, (const float*)gyT, rchunks, part));
    else CUDA_TRY(c, launch_pdl(dcn_dw_kernel<64>, grid, dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset, (const float*)gyT, rchunks, part));
    const long long nw = (long long)g.O * g.Cg * g.K;
    CUDA_TRY(c, launch_pdl(dcn_dw_reduce_kernel, dim3((unsigned)((nw + 255) / 256)), dim3(256), (size_t)0, st, (const float*)part, l.splits, nw,
                           grad_weight));
  }
  if (grad_offset) {
    const long long warps = g.NP * g.D;
    CUDA_TRY(c, launch_pdl(dcn_doff_kernel, dim3((unsigned)((warps + 7) / 8)), dim3(DCN_THREADS), (size_t)0, st, g, (const float*)xT, offset,
                           weight, (const float*)gyT, grad_offset));
  }
  if (grad_x) {
    uint32_t *keys = l.keys, *vals = l.vals, *skeys = l.skeys, *svals = l.svals;
    const long long pixels = (long long)g.N * g.D * g.H * g.W, samples = l.M / 4;
    CUDA_TRY(c, launch_pdl(dcn_keys_kernel, dim3((unsigned)((samples + 255) / 256)), dim3(256), (size_t)0, st, g, offset, samples,
                           (uint32_t)pixels, keys, vals));
    size_t cub_bytes = l.cub_bytes;
    cudaError_t ce = cub::DeviceRadixSort::SortPairs(l.cub, cub_bytes, (const uint32_t*)keys, skeys, (const uint32_t*)vals, svals,
                                                     (int)l.M, 0, l.end_bit, st);
    if (ce != cudaSuccess) return sstb_fail(c, SSTB_ERR_CUDA, "cub radix sort: %s", cudaGetErrorString(ce));
    CUDA_TRY(c, launch_pdl(dcn_dx_kernel, dim3((unsigned)((pixels + 7) / 8)), dim3(DCN_THREADS), (size_t)0, st, g, offset, weight,
                           (const float*)gyT, (const uint32_t*)skeys, (const uint32_t*)svals, l.M, grad_x));
  }
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
