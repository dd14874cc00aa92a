// Point-in-box test of mmdet3d's roiaware_pool3d package and the hashed BEV point grid that finds a box's points without testing
// every point.  Shared by roi_pool.cu (dynamic_point_pool) and roiaware.cu (points_in_boxes, RoIAwarePool3d).
//
// In-box test: the arithmetic of check_pt_in_box3d (mmdet3d/ops/roiaware_pool3d/src/points_in_boxes_cuda.cu:24-49), evaluated as the
// same float expressions: centre z = bottom + h/2 in double, |z - cz| > h/2 rejects, angle rz + pi/2 formed in double, cos / sin in
// float, local x / y as (sx cos - sy sin, sx sin + sy cos) rounded as the reference kernel rounds them, strict |local| < l/2, w/2.
//
// Grid: points are binned into 1 m BEV cells; a cell (batch, x, y) lives in bucket hash(batch, x, y) of a power-of-two table (CSR
// from csr_build, points re-laid out bucket by bucket as float4 + cell key).  for_each_hit walks the cells under the axis-aligned
// footprint of a box and tests the points whose cell key matches (a hash collision never admits a point twice).
#pragma once
#include "index.cuh"

namespace {

#define RP_THREADS 128
#define RP_CELL_INV 1.0f    // 1 / BEV cell edge (1 m: FSD RoIs are 1-6 m long, so a RoI covers a few dozen cells)
#define RP_CELL_CLAMP 32767 // cell coordinates are clamped to +-32767 (monotone, so the covering is still exact)

struct Box {
  float cx, cy, ca, sa;  // centre, cos / sin of rz + pi/2
  float cz, hl, hw, hh;  // centre z, half l / w / h
};

__device__ __forceinline__ Box make_box(float cx, float cy, float zb, float w, float l, float h, float rz) {
  Box b;
  b.cx = cx;
  b.cy = cy;
  b.cz = (float)((double)zb + (double)h / 2.0);
  const float ang = (float)((double)rz + M_PI / 2.0);
  b.ca = cosf(ang);
  b.sa = sinf(ang);
  b.hl = 0.5f * l;
  b.hw = 0.5f * w;
  b.hh = 0.5f * h;
  return b;
}

// The reference's `sx * cos + sy * (-sin)` / `sx * sin + sy * cos` compiles (nvcc, sm_90a, default contraction) to the product with cos
// fused and the one with sin rounded first; left to itself the compiler contracts this file's copy the other way for local y, so the
// rounding is spelled out.
__device__ __forceinline__ void to_local(const Box& b, float x, float y, float& lx, float& ly) {
  const float sx = x - b.cx, sy = y - b.cy;
  lx = __fmaf_rn(sx, b.ca, __fmul_rn(sy, -b.sa));
  ly = __fmaf_rn(sy, b.ca, __fmul_rn(sx, b.sa));
}

__device__ __forceinline__ bool in_box(const Box& b, float z, float lx, float ly) {
  return !(fabsf(z - b.cz) > b.hh) && lx > -b.hl && lx < b.hl && ly > -b.hw && ly < b.hw;
}

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

// ---- host side: table size, arena bytes and the build of the grid over num_pts points ------------------------------------------
static uint32_t grid_table_size(int num_pts) {
  uint32_t T = 1024;
  while (T < 2u * (uint32_t)num_pts && T < (1u << 24)) T <<= 1;
  return T;
}
static size_t grid_bytes(int num_pts, uint32_t T) {
  const size_t N = (size_t)num_pts;
  return al256(((size_t)T + 2) * 4) + csr_bytes(N, T) + al256(N * 4) * 2 + al256(N * 16) + al256(N * 8);
}
// Bins the points (flags[0] = 1 when a batch id is negative; flags must be zeroed already) and fills g.  *binned: device count of
// the points with a batch id >= 0 (the length of g.spts / g.skey).
static int grid_build(sstb200_ctx* c, const float* pts, const int32_t* pts_batch, int N, uint32_t T, float3 ex, int32_t* flags, Grid& g,
                      const uint32_t** binned) {
  int32_t* count = arena_alloc<int32_t>(c, (size_t)T + 2);
  int32_t* bucket = arena_alloc<int32_t>(c, (size_t)N + 1);
  uint32_t* key = arena_alloc<uint32_t>(c, (size_t)N + 1);
  float4* spts = arena_alloc<float4>(c, (size_t)N + 1);
  int2* skey = arena_alloc<int2>(c, (size_t)N + 1);
  if (!count || !bucket || !key || !spts || !skey) return sstb_fail(c, SSTB_ERR_WORKSPACE, "point grid: arena too small");
  CUDA_TRY(c, cudaMemsetAsync(count, 0, ((size_t)T + 2) * 4, c->stream));
  if (N > 0)
    launch_pdl(rp_bin_kernel, dim3((N + 255) / 256), dim3(256), (size_t)0, c->stream, pts, pts_batch, N, T - 1, bucket, key, count, flags);
  Csr csr;
  int rc = csr_build<int32_t>(c, csr, bucket, N, count, T, nullptr);
  if (rc) return rc;
  if (N > 0)
    launch_pdl(rp_gather_kernel, dim3((N + 255) / 256), dim3(256), (size_t)0, c->stream, pts, pts_batch, (const int32_t*)csr.order,
               (const uint32_t*)key, (const uint32_t*)(csr.offsets + T), spts, skey);
  g.offsets = csr.offsets;
  g.spts = spts;
  g.skey = skey;
  g.mask = T - 1;
  g.ex = ex;
  *binned = csr.offsets + T;  // points with a batch id >= 0
  return SSTB_OK;
}

}  // namespace
