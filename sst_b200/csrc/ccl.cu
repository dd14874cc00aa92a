// FSD instance grouping (SURVEY 8f next-3): connected components of the voted centres under "xy distance < dist"
// (mmdet3d/models/detectors/single_stage_fsd.py:37-81 find_connected_componets{,_gpu,_single_batch}: a dense n x n distance matrix
// handed to scipy.sparse.csgraph.connected_components on the CPU, or TorchEx's connected_components on the GPU).
//
// Form: no n x n matrix.  Centres are binned into a uniform xy grid of cell >= dist through the bitmap-rank index (cells ->
// CSR of their points), every centre tests only the centres of its 3 x 3 cell neighbourhood, edges are merged in a lock-free
// union-find whose roots are always the SMALLEST index of their tree (hook the larger root under the smaller with atomicMin), and the
// labels are the rank of (batch, root) - exactly scipy's numbering (components numbered by their first node, samples in order).
// Adjacency is evaluated with the reference's fp32 arithmetic: sqrt(dx*dx + dy*dy) < dist, round-to-nearest at every step.
//
// The cell is dist * 1.01, and the binning must keep any two centres whose fp32 distance is below dist at most one cell apart.
// An fp32 distance below dist bounds the exact one by dist (1 + 2^-22), so the exact coordinate difference is under 0.991 cells
// and the binning may err by at most the remaining 0.009 cell.  In fp32, (v - x0) * inv_cell errs by about 2^-23 of the cell
// index, which exceeds that slack once an axis has more than ~2.5e5 cells (dist 6e-4 over 160 m puts two centres 5.95e-4 apart
// in cells 257258 and 257260).  So the binning runs in double: floor(((double)v - x0) / cell) with x0 and cell held in double
// errs by ~2^-52 of the cell index, under 1e-9 cell at the 1e6 cells per axis the call accepts.
#include <stdarg.h>
#include "index.cuh"

namespace {

struct CclGrid {
  double x0, y0, cell;
  int nx, ny, B;
};

__device__ __forceinline__ int ccl_cell(float v, double v0, double cell, int n) {
  const double f = floor(((double)v - v0) / cell);
  return !(f >= 0.0) ? 0 : (f >= (double)n ? n - 1 : (int)f);   // also sends NaN to cell 0, +-inf to the border cells
}

__global__ void ccl_rows_kernel(const float* __restrict__ centers, int stride, const int32_t* __restrict__ batch_idx, int n, CclGrid g,
                                int32_t* __restrict__ rows, int32_t* __restrict__ parent) {
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rows[3 * i + 0] = batch_idx ? batch_idx[i] : 0;
  rows[3 * i + 1] = ccl_cell(centers[(size_t)i * stride + 0], g.x0, g.cell, g.nx);
  rows[3 * i + 2] = ccl_cell(centers[(size_t)i * stride + 1], g.y0, g.cell, g.ny);
  parent[i] = i;
}

__device__ __forceinline__ int ccl_find(volatile int32_t* parent, int i) {
  int p = parent[i];
  while (p != i) {
    i = p;
    p = parent[i];
  }
  return i;
}

// every centre against the centres of its 3 x 3 cells; only pairs (i, j > i) are merged (each edge once)
__global__ void ccl_union_kernel(const float* __restrict__ centers, int stride, const int32_t* __restrict__ rows, int n, CclGrid g, float dist,
                                 const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ word_prefix,
                                 const uint32_t* __restrict__ offsets, const int32_t* __restrict__ order, int32_t* parent) {
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = rows[3 * i], cx = rows[3 * i + 1], cy = rows[3 * i + 2];
  if (b < 0 || b >= g.B) return;
  const float xi = centers[(size_t)i * stride], yi = centers[(size_t)i * stride + 1];
  for (int ax = max(cx - 1, 0); ax <= min(cx + 1, g.nx - 1); ax++) {
    for (int ay = max(cy - 1, 0); ay <= min(cy + 1, g.ny - 1); ay++) {
      const long long key = ((long long)b * g.nx + ax) * g.ny + ay;
      const size_t w = (size_t)(key >> 5);
      const uint32_t bit = 1u << (key & 31), word = bitmap[w];
      if (!(word & bit)) continue;
      const uint32_t cell = word_prefix[w] + __popc(word & (bit - 1u));
      for (uint32_t q = offsets[cell]; q < offsets[cell + 1]; q++) {
        const int j = order[q];
        if (j <= i) continue;
        const float dx = __fsub_rn(xi, centers[(size_t)j * stride]), dy = __fsub_rn(yi, centers[(size_t)j * stride + 1]);
        const float d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
        if (!(d < dist)) continue;
        // union(i, j): hook the larger root under the smaller one
        int ra = ccl_find(parent, i), rb = ccl_find(parent, j);
        while (ra != rb) {
          const int hi = max(ra, rb), lo = min(ra, rb);
          const int old = atomicMin(&parent[hi], lo);
          if (old == hi) break;          // hi was a root and now points at lo
          ra = ccl_find(parent, old);    // somebody re-parented hi meanwhile: merge its new ancestor with lo
          rb = ccl_find(parent, lo);
        }
      }
    }
  }
}

// root[i] = find(i); mark (batch, root) in the ranking bitmap
__global__ void ccl_root_kernel(const int32_t* __restrict__ rows, int n, int B, int32_t* parent, int32_t* __restrict__ root, uint32_t* __restrict__ root_bitmap) {
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = ccl_find(parent, i);
  root[i] = r;
  const int b = rows[3 * i];
  if (r == i && b >= 0 && b < B) bitmap_set(root_bitmap, (long long)b * n + i);
}

__global__ void ccl_label_kernel(const int32_t* __restrict__ rows, const int32_t* __restrict__ root, int n, int B, const uint32_t* __restrict__ root_bitmap,
                                 const uint32_t* __restrict__ root_prefix, int32_t* __restrict__ labels) {
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = rows[3 * i];
  if (b < 0 || b >= B) {
    labels[i] = -1;
    return;
  }
  const long long key = (long long)b * n + root[i];
  const size_t w = (size_t)(key >> 5);
  labels[i] = (int)(root_prefix[w] + __popc(root_bitmap[w] & ((1u << (key & 31)) - 1u)));
}

}  // namespace

extern "C" int sstb200_connected_components(sstb200_ctx* c, const float* centers, int stride, const int32_t* batch_idx, int n, int batch_size,
                                            float dist, const float xy_min[2], const float xy_max[2], int32_t* labels,
                                            int32_t* num_components_dev, int32_t* num_components_host) {
  CHECK_ARG(c, c && n >= 0 && num_components_dev && batch_size >= 1 && stride >= 2 && dist > 0.f && xy_min && xy_max);
  if (n == 0) {
    CUDA_TRY(c, cudaMemsetAsync(num_components_dev, 0, 4, c->stream));
    if (num_components_host) *num_components_host = 0;
    return SSTB_OK;
  }
  CHECK_ARG(c, centers && labels && xy_max[0] >= xy_min[0] && xy_max[1] >= xy_min[1]);
  CclGrid g;
  const double cell = (double)dist * 1.01;   // > dist by far more than the rounding of the fp64 binning (see the top of the file)
  g.x0 = xy_min[0];
  g.y0 = xy_min[1];
  g.cell = cell;
  // the kernel's own expression at xy_max: an in-range centre never bins past cell n - 1
  const double ex = ((double)xy_max[0] - g.x0) / cell, ey = ((double)xy_max[1] - g.y0) / cell;
  if (ex > 1e6 || ey > 1e6) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "connected_components: xy range / dist too large (%g x %g cells)", ex, ey);
  g.nx = (int)ex + 1;
  g.ny = (int)ey + 1;
  g.B = batch_size;
  Extents e, er;
  long long T, Tr;
  long long lo[3] = {0, 0, 0}, hi[3] = {batch_size - 1, g.nx - 1, g.ny - 1};
  int rc = make_extents(c, e, 3, lo, hi, &T);
  if (rc) return rc;
  long long lor[1] = {0}, hir[1] = {(long long)batch_size * n - 1};
  rc = make_extents(c, er, 1, lor, hir, &Tr);
  if (rc) return rc;
  arena_reset(c);
  KeyIndex k, kr;
  int32_t *rows, *parent, *root, *cellmap, *count;
  Csr r;
  rc = arena_carve(c, [&](Carve& cv) {
    key_index_carve(cv, k, n, T);
    key_index_carve(cv, kr, 1, Tr);
    rows = cv.take<int32_t>((size_t)n * 3);
    parent = cv.take<int32_t>(n);
    root = cv.take<int32_t>(n);
    cellmap = cv.take<int32_t>(n);
    count = cv.take<int32_t>((size_t)n + 2);
    csr_carve(cv, r, n, n);
  });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k)) || (rc = key_index_zero(c, kr))) return rc;
  CUDA_TRY(c, cudaMemsetAsync(count, 0, ((size_t)n + 2) * 4, c->stream));
  const int nb = (n + 255) / 256;
  launch_pdl(ccl_rows_kernel, dim3(nb), dim3(256), (size_t)0, c->stream, centers, stride, batch_idx, n, g, rows, parent);
  launch_mark_rows<int32_t>(c, rows, n, e, false, k, nullptr);
  key_index_scan(c, k);
  launch_pdl(map_count_kernel<int32_t>, dim3(nb), dim3(256), (size_t)0, c->stream, (const long long*)k.keys, n, (const uint32_t*)k.bitmap,
             (const uint32_t*)k.word_prefix, 0, (const int32_t*)k.flags, cellmap, count, (const int32_t*)nullptr);
  rc = csr_build<int32_t>(c, r, cellmap, n, count, n, (const int32_t*)k.total);
  if (rc) return rc;
  launch_pdl(ccl_union_kernel, dim3(nb), dim3(256), (size_t)0, c->stream, centers, stride, (const int32_t*)rows, n, g, dist, (const uint32_t*)k.bitmap,
             (const uint32_t*)k.word_prefix, (const uint32_t*)r.offsets, (const int32_t*)r.order, parent);
  launch_pdl(ccl_root_kernel, dim3(nb), dim3(256), (size_t)0, c->stream, (const int32_t*)rows, n, batch_size, parent, root, kr.bitmap);
  key_index_scan(c, kr);
  launch_pdl(ccl_label_kernel, dim3(nb), dim3(256), (size_t)0, c->stream, (const int32_t*)rows, (const int32_t*)root, n, batch_size,
             (const uint32_t*)kr.bitmap, (const uint32_t*)kr.word_prefix, labels);
  CUDA_TRY(c, cudaMemcpyAsync(num_components_dev, kr.total, 4, cudaMemcpyDeviceToDevice, c->stream));
  LAUNCH_CHECK(c);
  if (num_components_host) {
    rc = read_back_i32(c, num_components_dev, num_components_host);
    if (rc) return rc;
    int32_t bad = 0;
    rc = read_back_i32(c, k.flags, &bad);
    if (rc) return rc;
    if (bad) return sstb_fail(c, SSTB_ERR_ARG, "connected_components: a batch index lies outside [0, batch_size)");
  }
  return SSTB_OK;
}
