// SSTv2.recover_bev (mmdet3d/models/backbones/sst_v2.py:161-196): sparse voxel rows [M, C] -> dense canvas [B, C, ny, nx].
// The reference zero-fills one canvas per sample and index_puts the transposed rows; here ONE pass writes every output byte
// exactly once (HBM-write bound: B*C*ny*nx*4 bytes): a cell -> row map (4 bytes per cell) is filled first, then each block
// transposes the rows of 128 consecutive x cells, 32 channels at a time, through shared memory so that the canvas is written
// as 512-byte warp stores (float4 per lane, streaming); all-empty blocks only stream zeros.  The float4 path needs every canvas
// row to start 16-byte aligned: nx % 4 == 0 and a 16-byte-aligned canvas, which the host checks (a contiguous view of a larger
// buffer may start at any 4-byte offset); otherwise the same tiles leave through scalar stores.
#include <stdarg.h>
#include "common.cuh"

__global__ void bev_map_kernel(const long long* __restrict__ coors, int M, int B, int ny, int nx, int32_t* __restrict__ cell_map,
                               int32_t* __restrict__ err) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  long long b = coors[(size_t)i * 4], y = coors[(size_t)i * 4 + 2], x = coors[(size_t)i * 4 + 3];
  if (b < 0 || b >= B || y < 0 || y >= ny || x < 0 || x >= nx) {
    *err = 1;
    return;
  }
  cell_map[((size_t)b * ny + y) * nx + x] = i;  // a duplicated cell keeps one of its rows (the reference: the last writer)
}

#define BEV_X 128   // x cells per block
#define BEV_CC 32    // channels per pass
#define BEV_PITCH 132  // floats; == 4 (mod 32): 16-byte row reads by 32 lanes are conflict-free
__global__ void __launch_bounds__(256) bev_fill_kernel(const float* __restrict__ feat, int C, const int32_t* __restrict__ cell_map, int ny,
                                                       int nx, int vec4, float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  __shared__ __align__(16) float tile[BEV_CC][BEV_PITCH];  // [channel][cell]
  __shared__ int sRow[BEV_X];
  __shared__ int any;
  const int x0 = blockIdx.x * BEV_X, y = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) any = 0;
  __syncthreads();
  if (threadIdx.x < BEV_X) {
    int x = x0 + threadIdx.x;
    int r = x < nx ? cell_map[((size_t)b * ny + y) * nx + x] : -1;
    sRow[threadIdx.x] = r;
    if (r >= 0) any = 1;
  }
  __syncthreads();
  const bool some = any != 0;
  const int cell = threadIdx.x & (BEV_X - 1), chalf = threadIdx.x >> 7;  // phase A: thread = (cell, half of the channel pass)
  const int myrow = sRow[cell];
  const int x = x0 + lane * 4;
  const bool vec = vec4 && x + 3 < nx;
  for (int c0 = 0; c0 < C; c0 += BEV_CC) {
    if (some) {
      __syncthreads();  // previous pass read out
      const float* src = myrow >= 0 ? feat + (size_t)myrow * C + c0 + chalf * (BEV_CC / 2) : nullptr;
#pragma unroll
      for (int k = 0; k < BEV_CC / 2; k++) {
        int ch = chalf * (BEV_CC / 2) + k;
        tile[ch][cell] = (src && c0 + ch < C) ? __ldg(src + k) : 0.f;
      }
      __syncthreads();
    }
    for (int c = warp; c < BEV_CC && c0 + c < C; c += 8) {
      float4 v = some ? *reinterpret_cast<const float4*>(&tile[c][lane * 4]) : make_float4(0.f, 0.f, 0.f, 0.f);
      float* o = out + (((size_t)b * C + c0 + c) * ny + y) * nx + x;
      if (vec) {
        __stcs(reinterpret_cast<float4*>(o), v);
      } else {
        if (x < nx) __stcs(o, v.x);
        if (x + 1 < nx) __stcs(o + 1, v.y);
        if (x + 2 < nx) __stcs(o + 2, v.z);
        if (x + 3 < nx) __stcs(o + 3, v.w);
      }
    }
  }
}

// float4 rows: every (b, c, y) row of a [B, C, ny, nx] canvas starts 16-byte aligned
static inline int bev_vec4(const float* canvas, int nx) { return (nx & 3) == 0 && ((uintptr_t)canvas & 15) == 0; }

extern "C" int sstb200_recover_bev(sstb200_ctx* c, const float* voxel_feat, const int64_t* coors, int M, int C, int B, int ny, int nx,
                                   float* canvas) {
  CHECK_ARG(c, c && M >= 0 && C >= 1 && C <= 1024 && B >= 1 && ny >= 1 && nx >= 1 && canvas);
  CHECK_ARG(c, M == 0 || (voxel_feat && coors));
  CHECK_ARG(c, ny <= 65535 && B <= 65535);
  const size_t cells = (size_t)B * ny * nx;
  arena_reset(c);
  int32_t* cell_map;
  int rc = arena_carve(c, [&](Carve& cv) { cell_map = cv.take<int32_t>(cells + 64); });
  if (rc) return rc;
  int32_t* err = cell_map + cells;
  CUDA_TRY(c, cudaMemsetAsync(cell_map, 0xFF, cells * 4, c->stream));
  CUDA_TRY(c, cudaMemsetAsync(err, 0, 4, c->stream));
  if (M > 0)
    launch_pdl(bev_map_kernel, dim3((M + 255) / 256), dim3(256), (size_t)0, c->stream, (const long long*)coors, M, B, ny, nx, cell_map, err);
  launch_pdl(bev_fill_kernel, dim3((nx + BEV_X - 1) / BEV_X, ny, B), dim3(256), (size_t)0, c->stream, voxel_feat, C, (const int32_t*)cell_map, ny, nx,
             bev_vec4(canvas, nx), canvas);
  LAUNCH_CHECK(c);
  CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, err, 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (c->pinned_i32[0]) return sstb_fail(c, SSTB_ERR_ARG, "recover_bev: a voxel coordinate lies outside [0,B) x [0,ny) x [0,nx)");
  return SSTB_OK;
}

// ---- backward: grad_feat[m, :] = grad_canvas[b_m, :, y_m, x_m] for every row (the gradient torch's index_put gives) ------------
// The mirror of bev_fill_kernel: a block whose 128 cells hold a voxel reads 32-channel x 128-cell slabs of the gradient as
// 512-byte warp loads, transposes them through shared memory and stores each voxel's channels as one contiguous run of its row.
// Blocks without a voxel read nothing, so the traffic is the occupied (b, y, 128-x) segments plus the M x C rows.
__global__ void __launch_bounds__(256) bev_gather_kernel(const float* __restrict__ grad, int C, const int32_t* __restrict__ cell_map, int ny,
                                                         int nx, int vec4, float* __restrict__ grad_feat) {
  pdl_wait();
  pdl_launch();
  __shared__ __align__(16) float tile[BEV_CC][BEV_PITCH];  // [channel][cell]
  __shared__ int sRow[BEV_X];
  __shared__ int any;
  const int x0 = blockIdx.x * BEV_X, y = blockIdx.y, b = blockIdx.z;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) any = 0;
  __syncthreads();
  if (threadIdx.x < BEV_X) {
    int x = x0 + threadIdx.x;
    int r = x < nx ? cell_map[((size_t)b * ny + y) * nx + x] : -1;
    sRow[threadIdx.x] = r;
    if (r >= 0) any = 1;
  }
  __syncthreads();
  if (!any) return;
  const int cell = threadIdx.x & (BEV_X - 1), chalf = threadIdx.x >> 7;  // phase B: thread = (cell, half of the channel pass)
  const int myrow = sRow[cell];
  const int x = x0 + lane * 4;
  const size_t cstride = (size_t)ny * nx;
  const bool vec = vec4 && x + 3 < nx;
  for (int c0 = 0; c0 < C; c0 += BEV_CC) {
    __syncthreads();  // previous pass read out
    for (int c = warp; c < BEV_CC; c += 8) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c0 + c < C) {
        const float* g = grad + ((size_t)b * C + c0 + c) * cstride + (size_t)y * nx + x;
        if (vec) {
          v = __ldcs(reinterpret_cast<const float4*>(g));
        } else {
          if (x < nx) v.x = __ldcs(g);
          if (x + 1 < nx) v.y = __ldcs(g + 1);
          if (x + 2 < nx) v.z = __ldcs(g + 2);
          if (x + 3 < nx) v.w = __ldcs(g + 3);
        }
      }
      *reinterpret_cast<float4*>(&tile[c][lane * 4]) = v;
    }
    __syncthreads();
    if (myrow >= 0) {
      float* dst = grad_feat + (size_t)myrow * C + c0 + chalf * (BEV_CC / 2);
#pragma unroll
      for (int k = 0; k < BEV_CC / 2; k++) {
        int ch = chalf * (BEV_CC / 2) + k;
        if (c0 + ch < C) dst[k] = tile[ch][cell];
      }
    }
  }
}

// A cell holds one row in the map; every other row at that cell copies the kept row's gradient (one warp per row).  A row whose
// coordinate lies outside the canvas (which the forward rejects) gets zeros instead of an out-of-bounds read.
__global__ void __launch_bounds__(256) bev_dup_kernel(const long long* __restrict__ coors, int M, int C, int B, int ny, int nx,
                                                      const int32_t* __restrict__ cell_map, float* __restrict__ grad_feat) {
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= M) return;
  const long long b = coors[(size_t)i * 4], y = coors[(size_t)i * 4 + 2], x = coors[(size_t)i * 4 + 3];
  float* dst = grad_feat + (size_t)i * C;
  if (b < 0 || b >= B || y < 0 || y >= ny || x < 0 || x >= nx) {
    for (int c = lane; c < C; c += 32) dst[c] = 0.f;
    return;
  }
  const int w = cell_map[((size_t)b * ny + y) * nx + x];
  if (w == i) return;
  const float* src = grad_feat + (size_t)w * C;
  for (int c = lane; c < C; c += 32) dst[c] = src[c];
}

extern "C" int sstb200_recover_bev_backward(sstb200_ctx* c, const float* grad_canvas, const int64_t* coors, int M, int C, int B, int ny,
                                            int nx, float* grad_feat) {
  CHECK_ARG(c, c && M >= 0 && C >= 1 && C <= 1024 && B >= 1 && ny >= 1 && nx >= 1);
  if (M == 0) return SSTB_OK;
  CHECK_ARG(c, grad_canvas && coors && grad_feat);
  CHECK_ARG(c, ny <= 65535 && B <= 65535);
  const size_t cells = (size_t)B * ny * nx;
  arena_reset(c);
  int32_t* cell_map;
  int rc = arena_carve(c, [&](Carve& cv) { cell_map = cv.take<int32_t>(cells + 64); });
  if (rc) return rc;
  int32_t* err = cell_map + cells;  // bev_map_kernel's flag; out-of-canvas rows are zero-filled by bev_dup_kernel instead
  CUDA_TRY(c, cudaMemsetAsync(cell_map, 0xFF, cells * 4, c->stream));
  launch_pdl(bev_map_kernel, dim3((M + 255) / 256), dim3(256), (size_t)0, c->stream, (const long long*)coors, M, B, ny, nx, cell_map, err);
  launch_pdl(bev_gather_kernel, dim3((nx + BEV_X - 1) / BEV_X, ny, B), dim3(256), (size_t)0, c->stream, grad_canvas, C, (const int32_t*)cell_map,
             ny, nx, bev_vec4(grad_canvas, nx), grad_feat);
  launch_pdl(bev_dup_kernel, dim3((unsigned)(((size_t)M * 32 + 255) / 256)), dim3(256), (size_t)0, c->stream, (const long long*)coors, M, C, B,
             ny, nx, (const int32_t*)cell_map, grad_feat);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
