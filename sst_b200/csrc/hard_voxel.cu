// Hard voxelisation (SURVEY 8f next-4): voxel_layer.hard_voxelize, mmdet3d/ops/voxel/src/voxelization_cpu.cpp:43-142 and
// voxelization_cuda.cu:68-330 (the reference GPU version is an O(P^2) scan plus a <<<1,1>>> serial kernel).
//
// Semantics reproduced exactly: voxels are numbered in order of FIRST APPEARANCE in the point list, at most max_voxels of them;
// every voxel keeps its first max_points points in input order; points of later voxels / beyond max_points are dropped.
//
//   1. coordinates with the ROUND grid of hard_voxelize (voxelization_cpu.cpp:127-130; dynamic voxelisation uses ceil) -> key
//   2. bitmap-rank index (index.cuh): vid[i] = rank of the point's cell among the occupied cells, count[vid]
//   3. first[vid] = min point index (atomicMin); a second bitmap over point indices marks the first points; its popcount
//      prefix gives the voxel number in first-appearance order
//   4. stable grouping of the points by vid: radix sort is stable, so cub::DeviceRadixSort::SortPairs(vid, point index) over the
//      ceil(log2 M) key bits returns every voxel's points in input order; slot = position - offsets[vid]
//   5. one pass copies the kept points into voxels[number][slot][:]
#include <stdarg.h>
#include <cub/device/device_radix_sort.cuh>
#include "index.cuh"

__global__ void hv_coors_kernel(const float* __restrict__ points, int P, int F, float vx, float vy, float vz, float x0, float y0, float z0,
                                int gx, int gy, int gz, int32_t* __restrict__ coors) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float* p = points + (size_t)i * F;
  int cx = (int)floorf(__fdiv_rn(p[0] - x0, vx));
  int cy = (int)floorf(__fdiv_rn(p[1] - y0, vy));
  int cz = (int)floorf(__fdiv_rn(p[2] - z0, vz));
  cx = cx < 0 ? 0 : (cx >= gx ? gx - 1 : cx);
  cy = cy < 0 ? 0 : (cy >= gy ? gy - 1 : cy);
  cz = cz < 0 ? 0 : (cz >= gz ? gz - 1 : cz);
  coors[(size_t)i * 3 + 0] = cz;
  coors[(size_t)i * 3 + 1] = cy;
  coors[(size_t)i * 3 + 2] = cx;
}

__global__ void hv_first_kernel(const int32_t* __restrict__ vid, int P, int32_t* __restrict__ first, uint32_t* __restrict__ idx_iota) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  idx_iota[i] = (uint32_t)i;
  int v = vid[i];
  if (v >= 0) atomicMin(&first[v], i);
}

__global__ void hv_firstbits_kernel(const int32_t* __restrict__ first, const uint32_t* __restrict__ nvox, uint32_t* __restrict__ fbits) {
  pdl_wait();
  pdl_launch();
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (int)*nvox) return;
  int f = first[v];
  atomicOr(&fbits[f >> 5], 1u << (f & 31));
}

__global__ void hv_number_kernel(const int32_t* __restrict__ first, const uint32_t* __restrict__ nvox, const uint32_t* __restrict__ fbits,
                                 const uint32_t* __restrict__ fprefix, const int32_t* __restrict__ count, const int32_t* __restrict__ pcoors,
                                 int max_points, int max_voxels, int32_t* __restrict__ vnum, int32_t* __restrict__ coors_out,
                                 int32_t* __restrict__ npts_out, int32_t* __restrict__ voxel_num_dev) {
  pdl_wait();
  pdl_launch();
  int v = blockIdx.x * blockDim.x + threadIdx.x;
  const int M = (int)*nvox;
  if (v == 0) *voxel_num_dev = M < max_voxels ? M : max_voxels;
  if (v >= M) return;
  int f = first[v];
  int n = (int)fprefix[f >> 5] + __popc(fbits[f >> 5] & ((1u << (f & 31)) - 1u));
  vnum[v] = n;
  if (n < max_voxels) {
    coors_out[(size_t)n * 3 + 0] = pcoors[(size_t)f * 3 + 0];
    coors_out[(size_t)n * 3 + 1] = pcoors[(size_t)f * 3 + 1];
    coors_out[(size_t)n * 3 + 2] = pcoors[(size_t)f * 3 + 2];
    npts_out[n] = count[v] < max_points ? count[v] : max_points;
  }
}

__global__ void hv_gather_kernel(const float* __restrict__ points, int P, int F, const uint32_t* __restrict__ vid_sorted,
                                 const uint32_t* __restrict__ idx_sorted, const uint32_t* __restrict__ offsets, const int32_t* __restrict__ vnum,
                                 int max_points, int max_voxels, float* __restrict__ voxels) {
  pdl_wait();
  pdl_launch();
  // one warp per sorted position, lanes stride the features (rows are short: 3..8 floats, so several positions per warp)
  const int per_warp = F <= 4 ? 8 : (F <= 8 ? 4 : (F <= 16 ? 2 : 1));
  const int lanes = 32 / per_warp;
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long p = warp * per_warp + lane / lanes;
  if (p >= P) return;
  const uint32_t v = vid_sorted[p];
  const int vn = vnum[v];
  const int slot = (int)(p - offsets[v]);
  if (vn >= max_voxels || slot >= max_points) return;
  const float* src = points + (size_t)idx_sorted[p] * F;
  float* dst = voxels + ((size_t)vn * max_points + slot) * F;
  for (int k = lane % lanes; k < F; k += lanes) dst[k] = src[k];
}

extern "C" int sstb200_hard_voxelize(sstb200_ctx* c, const float* points, int P, int F, const float vs[3], const float r[6], int max_points,
                                     int max_voxels, float* voxels, int32_t* coors, int32_t* num_points_per_voxel, int32_t* voxel_num_dev,
                                     int32_t* voxel_num_host) {
  CHECK_ARG(c, c && P >= 0 && F >= 3 && vs && r && max_points >= 1 && max_voxels >= 1 && voxel_num_dev);
  if (P == 0) {
    CUDA_TRY(c, cudaMemsetAsync(voxel_num_dev, 0, 4, c->stream));
    if (voxel_num_host) *voxel_num_host = 0;
    return SSTB_OK;
  }
  CHECK_ARG(c, points && voxels && coors && num_points_per_voxel);
  int g[3];
  for (int i = 0; i < 3; i++) g[i] = (int)roundf((r[3 + i] - r[i]) / vs[i]);  // voxelization_cpu.cpp:127-130, float arithmetic
  CHECK_ARG(c, g[0] >= 1 && g[1] >= 1 && g[2] >= 1);
  Extents e;
  long long T;
  long long lo[3] = {0, 0, 0}, hi[3] = {g[2] - 1, g[1] - 1, g[0] - 1};
  int rc = make_extents(c, e, 3, lo, hi, &T);
  if (rc) return rc;
  cudaStream_t st = c->stream;
  int end_bit = 1;
  while ((1ll << end_bit) < (long long)P + 1 && end_bit < 32) end_bit++;
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  P, 0, end_bit, st);
  const size_t pwords = ((size_t)P + 31) / 32;
  arena_reset(c);
  KeyIndex k;
  int32_t *pcoors, *vid, *count, *first, *vnum;
  uint32_t *iota, *vid_s, *idx_s, *offsets, *fbits, *fprefix;
  ScanTemps fst, ost;
  size_t zero_bytes;
  void* cub_tmp;
  rc = arena_carve(c, [&](Carve& cv) {
    key_index_carve(cv, k, P, T);
    pcoors = cv.take<int32_t>((size_t)P * 3);
    vid = cv.take<int32_t>(P);
    count = cv.take<int32_t>((size_t)P + 2);
    first = cv.take<int32_t>(P);
    vnum = cv.take<int32_t>(P);
    iota = cv.take<uint32_t>(P);
    vid_s = cv.take<uint32_t>(P);
    idx_s = cv.take<uint32_t>(P);
    offsets = cv.take<uint32_t>((size_t)P + 2);
    // first-point bitmap + its scan state + the offsets scan's state: one zero fill
    const size_t z = cv.mark();
    fbits = cv.take<uint32_t>(pwords);
    scan_carve(cv, fst, pwords);
    scan_carve(cv, ost, P);
    zero_bytes = cv.off - z;
    fprefix = cv.take<uint32_t>(pwords + 2);
    cub_tmp = cv.take<uint8_t>(cub_bytes + 16);
  });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k))) return rc;
  CUDA_TRY(c, cudaMemsetAsync(fbits, 0, zero_bytes, st));
  CUDA_TRY(c, cudaMemsetAsync(count, 0, ((size_t)P + 2) * 4, st));
  CUDA_TRY(c, cudaMemsetAsync(first, 0x7F, (size_t)P * 4, st));
  const int nb = (P + 255) / 256;
  launch_pdl(hv_coors_kernel, dim3(nb), dim3(256), (size_t)0, st, points, P, F, vs[0], vs[1], vs[2], r[0], r[1], r[2], g[0], g[1], g[2], pcoors);
  launch_mark_rows<int32_t>(c, pcoors, P, e, true, k, nullptr);
  key_index_scan(c, k);
  launch_pdl(map_count_kernel<int32_t>, dim3(nb), dim3(256), (size_t)0, st, (const long long*)k.keys, P, (const uint32_t*)k.bitmap,
             (const uint32_t*)k.word_prefix, 0, (const int32_t*)k.flags, vid, count, (const int32_t*)nullptr);
  launch_pdl(hv_first_kernel, dim3(nb), dim3(256), (size_t)0, st, (const int32_t*)vid, P, first, iota);
  launch_pdl(hv_firstbits_kernel, dim3(nb), dim3(256), (size_t)0, st, (const int32_t*)first, (const uint32_t*)k.total, fbits);
  uint32_t* ftotal = fst.ticket + 1;
  launch_exclusive_scan(st, LoadPopc{fbits}, pwords, nullptr, fst, fprefix, ftotal, true);
  launch_pdl(hv_number_kernel, dim3(nb), dim3(256), (size_t)0, st, (const int32_t*)first, (const uint32_t*)k.total, (const uint32_t*)fbits,
             (const uint32_t*)fprefix, (const int32_t*)count, (const int32_t*)pcoors, max_points, max_voxels, vnum, coors, num_points_per_voxel,
             voxel_num_dev);
  uint32_t* ototal = ost.ticket + 1;
  launch_exclusive_scan(st, LoadU32{(const uint32_t*)count}, (size_t)P, (const int32_t*)k.total, ost, offsets, ototal, true);
  cudaError_t ce = cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, (const uint32_t*)vid, vid_s, (const uint32_t*)iota, idx_s, P, 0, end_bit, st);
  if (ce != cudaSuccess) return sstb_fail(c, SSTB_ERR_CUDA, "cub radix sort: %s", cudaGetErrorString(ce));
  {
    const int per_warp = F <= 4 ? 8 : (F <= 8 ? 4 : (F <= 16 ? 2 : 1));
    const long long warps = ((long long)P + per_warp - 1) / per_warp;
    const long long blocks = (warps * 32 + 255) / 256;
    launch_pdl(hv_gather_kernel, dim3((unsigned)blocks), dim3(256), (size_t)0, st, points, P, F, (const uint32_t*)vid_s, (const uint32_t*)idx_s,
               (const uint32_t*)offsets, (const int32_t*)vnum, max_points, max_voxels, voxels);
  }
  LAUNCH_CHECK(c);
  if (voxel_num_host) return read_back_i32(c, voxel_num_dev, voxel_num_host);
  return SSTB_OK;
}
