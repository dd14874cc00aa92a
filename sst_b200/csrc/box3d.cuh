// The hashed BEV point grid that finds a box's points without testing every point, on top of in_box.cuh's point-in-box test.
// Shared by roi_pool.cu (dynamic_point_pool) and roiaware.cu (points_in_boxes, RoIAwarePool3d).
//
// Grid: points are binned into 1 m BEV cells; a cell (batch, x, y) lives in bucket hash(batch, x, y) of a power-of-two table (CSR
// from csr_build, points re-laid out bucket by bucket as float4 + cell key).  for_each_hit walks the cells under the axis-aligned
// footprint of a box and tests the points whose cell key matches (a hash collision never admits a point twice).
#pragma once
#include "index.cuh"
#include "in_box.cuh"

namespace {

#define RP_THREADS 128
#define RP_CELL_INV 1.0f    // 1 / BEV cell edge (1 m: FSD RoIs are 1-6 m long, so a RoI covers a few dozen cells)
#define RP_CELL_CLAMP 32767 // cell coordinates are clamped to +-32767 (monotone, so the covering is still exact)

// RoI r: the original box and the enlarged one (same centre and yaw, dims + extra_wlh, bottom lowered by extra_h / 2)
struct RoiPair {
  Box o, e;
  int batch;
};

__device__ __forceinline__ RoiPair load_roi(const float* __restrict__ rois, const int32_t* __restrict__ rois_batch, int r, float3 ex) {
  const float* p = rois + (size_t)r * 7;
  const float cx = p[0], cy = p[1], zb = p[2], w = p[3], l = p[4], h = p[5], rz = p[6];
  RoiPair q;
  q.o = make_box(cx, cy, zb, w, l, h, rz);
  q.e = make_box(cx, cy, zb - 0.5f * ex.z, w + ex.x, l + ex.y, h + ex.z, rz);
  q.batch = rois_batch ? rois_batch[r] : 0;
  return q;
}

__device__ __forceinline__ int cell_of(float v) {
  const float f = floorf(v * RP_CELL_INV);
  if (!(f >= -(float)RP_CELL_CLAMP)) return -RP_CELL_CLAMP;  // also NaN
  return f > (float)RP_CELL_CLAMP ? RP_CELL_CLAMP : (int)f;
}
__device__ __forceinline__ uint32_t cell_key(int cx, int cy) { return ((uint32_t)(cx + 32768) << 16) | (uint32_t)(cy + 32768); }
__device__ __forceinline__ uint32_t bucket_of(int cx, int cy, int b, uint32_t mask) {
  return ((uint32_t)cx * 73856093u ^ (uint32_t)cy * 19349663u ^ (uint32_t)b * 83492791u) & mask;
}

// ---- points -> buckets -------------------------------------------------------------------------------------------------------
__global__ void rp_bin_kernel(const float* __restrict__ pts, const int32_t* __restrict__ pts_batch, int n, uint32_t mask,
                              int32_t* __restrict__ bucket, uint32_t* __restrict__ key, int32_t* __restrict__ count,
                              int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = pts_batch ? pts_batch[i] : 0;
  if (b < 0) {  // never pairs
    bucket[i] = -1;
    flags[0] = 1;
    return;
  }
  const int cx = cell_of(pts[(size_t)i * 3]), cy = cell_of(pts[(size_t)i * 3 + 1]);
  const uint32_t h = bucket_of(cx, cy, b, mask);
  bucket[i] = (int32_t)h;
  key[i] = cell_key(cx, cy);
  atomicAdd(&count[h], 1);
}

// bucket-ordered copies: (x, y, z, point index) and (cell key, batch)
__global__ void rp_gather_kernel(const float* __restrict__ pts, const int32_t* __restrict__ pts_batch, const int32_t* __restrict__ order,
                                 const uint32_t* __restrict__ key, const uint32_t* __restrict__ total, float4* __restrict__ spts,
                                 int2* __restrict__ skey) {
  pdl_wait();
  pdl_launch();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (int)*total) return;
  const int i = order[q];
  spts[q] = make_float4(pts[(size_t)i * 3], pts[(size_t)i * 3 + 1], pts[(size_t)i * 3 + 2], __int_as_float(i));
  skey[q] = make_int2((int)key[i], pts_batch ? pts_batch[i] : 0);
}

struct Grid {
  const uint32_t* offsets;  // [mask + 2]
  const float4* spts;
  const int2* skey;
  uint32_t mask;
  float3 ex;
};

// Calls f(point index, x, y, z) once for every point inside RoI q's enlarged box (any thread of the block, any order).
template <typename F>
__device__ __forceinline__ void for_each_hit(const RoiPair& q, const Grid& g, const uint32_t* __restrict__ total, F&& f) {
  if (q.batch < 0) return;
  const Box& e = q.e;
  // axis-aligned footprint of the enlarged box: |sx| <= |cos| l/2 + |sin| w/2, |sy| <= |sin| l/2 + |cos| w/2, padded for rounding
  const float pad = 0.01f + 1e-6f * (fabsf(e.cx) + fabsf(e.cy));
  const float rx = fabsf(e.ca) * e.hl + fabsf(e.sa) * e.hw + pad, ry = fabsf(e.sa) * e.hl + fabsf(e.ca) * e.hw + pad;
  const int x0 = cell_of(e.cx - rx), x1 = cell_of(e.cx + rx), y0 = cell_of(e.cy - ry), y1 = cell_of(e.cy + ry);
  if (x1 < x0 || y1 < y0) return;  // negative dims: an empty box
  const long long ny = y1 - y0 + 1, nc = (long long)(x1 - x0 + 1) * ny;
  auto test = [&](const float4 p) {
    float lx, ly;
    to_local(e, p.x, p.y, lx, ly);
    if (in_box(e, p.z, lx, ly)) f(__float_as_int(p.w), p.x, p.y, p.z);
  };
  if (nc > (long long)g.mask + 1) {  // a footprint larger than the table: every binned point once
    const int n = (int)*total;
    for (int s = threadIdx.x; s < n; s += blockDim.x)
      if (g.skey[s].y == q.batch) test(g.spts[s]);
    return;
  }
  const int warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (long long c = warp; c < nc; c += nwarps) {
    const int cx = x0 + (int)(c / ny), cy = y0 + (int)(c % ny);
    const uint32_t h = bucket_of(cx, cy, q.batch, g.mask);
    const int want = (int)cell_key(cx, cy);
    for (uint32_t s = g.offsets[h] + lane_id(); s < g.offsets[h + 1]; s += 32) {
      const int2 k = g.skey[s];
      if (k.x == want && k.y == q.batch) test(g.spts[s]);
    }
  }
}

__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane_id() == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t t = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += sh[w];
  return t;
}

// ---- host side: table size, workspace and the build of the grid over num_pts points -------------------------------------------
static uint32_t grid_table_size(int num_pts) {
  uint32_t T = 1024;
  while (T < 2u * (uint32_t)num_pts && T < (1u << 24)) T <<= 1;
  return T;
}
struct GridWs {
  int32_t* count;
  int32_t* bucket;
  uint32_t* key;
  float4* spts;
  int2* skey;
  Csr csr;
};
static void grid_carve(Carve& cv, GridWs& w, int num_pts, uint32_t T) {
  const size_t N = (size_t)num_pts;
  w.count = cv.take<int32_t>((size_t)T + 2);
  w.bucket = cv.take<int32_t>(N + 1);
  w.key = cv.take<uint32_t>(N + 1);
  w.spts = cv.take<float4>(N + 1);
  w.skey = cv.take<int2>(N + 1);
  csr_carve(cv, w.csr, N, T);
}
// Bins the points (flags[0] = 1 when a batch id is negative; flags must be zeroed already) and fills g.  *binned: device count of
// the points with a batch id >= 0 (the length of g.spts / g.skey).
static int grid_build(sstb200_ctx* c, GridWs& w, const float* pts, const int32_t* pts_batch, int N, uint32_t T, float3 ex, int32_t* flags,
                      Grid& g, const uint32_t** binned) {
  CUDA_TRY(c, cudaMemsetAsync(w.count, 0, ((size_t)T + 2) * 4, c->stream));
  if (N > 0)
    launch_pdl(rp_bin_kernel, dim3((N + 255) / 256), dim3(256), (size_t)0, c->stream, pts, pts_batch, N, T - 1, w.bucket, w.key, w.count, flags);
  int rc = csr_build<int32_t>(c, w.csr, w.bucket, N, w.count, T, nullptr);
  if (rc) return rc;
  if (N > 0)
    launch_pdl(rp_gather_kernel, dim3((N + 255) / 256), dim3(256), (size_t)0, c->stream, pts, pts_batch, (const int32_t*)w.csr.order,
               (const uint32_t*)w.key, (const uint32_t*)(w.csr.offsets + T), w.spts, w.skey);
  g.offsets = w.csr.offsets;
  g.spts = w.spts;
  g.skey = w.skey;
  g.mask = T - 1;
  g.ex = ex;
  *binned = w.csr.offsets + T;  // points with a batch id >= 0
  return SSTB_OK;
}

}  // namespace
