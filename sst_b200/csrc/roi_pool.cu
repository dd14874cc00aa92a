// FSD second stage: pool the points of every RoI (SURVEY 8f next-3).  dynamic_point_pool / dynamic_point_pool_mixed
// (mmdet3d/ops/dynamic_point_pool_op.py:9-113), whose kernel lives in the unvendored TorchEx `dynamic_point_pool_ext`; consumed by
// DynamicPointROIExtractor (mmdet3d/models/roi_heads/roi_extractors/dynamic_point_roi_extractor.py:32-136).
//
// Form: points are binned into 1 m BEV cells; a cell (batch, x, y) lives in bucket hash(batch, x, y) of a power-of-two table (CSR
// from csr_build, points re-laid out bucket by bucket as float4 + cell key).  One block per RoI walks the cells under the axis-aligned
// footprint of its enlarged box and tests the points whose cell key matches (a hash collision never admits a point twice).  Passes:
// count (hits per RoI) -> scan of min(hits, max_inbox_point) -> capacity cut per call or per sample, fake rows -> scan -> write.
// The write pass keeps each RoI's `take` smallest point indices: when hits > take a radix select over the point index (8 bits per
// pass, the RoI's candidates re-tested each pass) finds the take-th smallest, the hits up to it are gathered in shared memory and
// bitonic-sorted.  Integer atomics only; the result does not depend on scheduling.
//
// In-box test and point grid: box3d.cuh.
#include <stdarg.h>
#include "box3d.cuh"

namespace {

#define RP_MAX_INBOX 8192   // one RoI's kept points are sorted in shared memory

// ---- pass 1: hits per RoI; kept = min(hits, max_inbox_point) ------------------------------------------------------------------------
__global__ void __launch_bounds__(RP_THREADS) rp_count_kernel(const float* __restrict__ rois, const int32_t* __restrict__ rois_batch,
                                                              Grid g, const uint32_t* __restrict__ total, int max_inbox, int per_sample,
                                                              uint32_t* __restrict__ kept, int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  __shared__ uint32_t sh[RP_THREADS / 32];
  const int r = blockIdx.x;
  const RoiPair q = load_roi(rois, rois_batch, r, g.ex);
  uint32_t hits = 0;
  for_each_hit(q, g, total, [&](int, float, float, float) { hits++; });
  hits = block_sum(hits, sh);
  if (threadIdx.x == 0) {
    kept[r] = min(hits, (uint32_t)max_inbox);
    if (q.batch < 0) flags[1] = 1;
    if (per_sample && r > 0 && rois_batch[r - 1] > q.batch) flags[2] = 1;
  }
}

// ---- capacity: rows[r] = kept pairs of RoI r that fit the call's (or its sample's) max_all_pts, + 1 for a sample's fake row ----------
__global__ void rp_rows_kernel(const int32_t* __restrict__ rois_batch, int R, int per_sample, int max_all, const uint32_t* __restrict__ kept,
                               const uint32_t* __restrict__ off, uint32_t* __restrict__ take, uint32_t* __restrict__ rows,
                               int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  int s0 = 0, s1 = R;  // the RoIs of r's sample (batch ids ascending)
  if (per_sample) {
    const int b = rois_batch[r];
    int lo = 0, hi = r;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (rois_batch[m] < b) lo = m + 1;
      else hi = m;
    }
    s0 = lo;
    lo = r + 1, hi = R;
    while (lo < hi) {
      const int m = (lo + hi) >> 1;
      if (rois_batch[m] <= b) lo = m + 1;
      else hi = m;
    }
    s1 = lo;
  }
  const long long before = (long long)off[r] - off[s0], room = (long long)max_all - before;
  const uint32_t t = room <= 0 ? 0u : (uint32_t)min((long long)kept[r], room);
  const bool fake = r == s0 && off[s1] == off[s0];
  take[r] = t;
  rows[r] = t + (fake ? 1u : 0u);
  if (fake) atomicAdd(&flags[3], 1);
}

// ---- pass 2: write each RoI's `take` smallest hit indices, ascending, with their features ---------------------------------------------
__global__ void __launch_bounds__(RP_THREADS) rp_write_kernel(const float* __restrict__ rois, const int32_t* __restrict__ rois_batch,
                                                              Grid g, const uint32_t* __restrict__ total, int n_pts,
                                                              const uint32_t* __restrict__ take, const uint32_t* __restrict__ rows,
                                                              const uint32_t* __restrict__ pos, const float* __restrict__ pts,
                                                              int64_t* __restrict__ out_idx,
                                                              int64_t* __restrict__ out_roi, float* __restrict__ out_feats) {
  pdl_wait();
  pdl_launch();
  extern __shared__ int32_t buf[];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sh[RP_THREADS / 32];
  __shared__ uint32_t s_prefix, s_rank, s_fill;
  const int r = blockIdx.x;
  const uint32_t k = take[r];
  uint32_t base = pos[r];
  if (rows[r] > k) {  // the sample's fake row: no pair at all
    if (threadIdx.x == 0) {
      out_idx[base] = -1;
      out_roi[base] = -1;
    }
    if (threadIdx.x < 13) out_feats[(size_t)base * 13 + threadIdx.x] = 0.f;
    base++;
  }
  if (k == 0) return;
  const RoiPair q = load_roi(rois, rois_batch, r, g.ex);
  // threshold = the k-th smallest hit index (all hits when k equals their number)
  uint32_t hits = 0;
  for_each_hit(q, g, total, [&](int, float, float, float) { hits++; });
  hits = block_sum(hits, sh);
  uint32_t thr = 0xffffffffu;
  if (hits > k) {
    const int bits = n_pts > 1 ? 32 - __clz(n_pts - 1) : 1;
    if (threadIdx.x == 0) {
      s_prefix = 0;
      s_rank = k;
    }
    for (int shift = ((bits + 7) / 8 - 1) * 8; shift >= 0; shift -= 8) {
      for (int d = threadIdx.x; d < 256; d += blockDim.x) hist[d] = 0;
      __syncthreads();
      const uint32_t hi_mask = shift + 8 >= 32 ? 0u : (0xffffffffu << (shift + 8)), prefix = s_prefix;
      for_each_hit(q, g, total, [&](int i, float, float, float) {
        if (((uint32_t)i & hi_mask) == prefix) atomicAdd(&hist[((uint32_t)i >> shift) & 255u], 1u);
      });
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t rank = s_rank, d = 0;
        while (hist[d] < rank) rank -= hist[d++];
        s_rank = rank;
        s_prefix = prefix | (d << shift);
      }
      __syncthreads();
    }
    thr = s_prefix;
  }
  if (threadIdx.x == 0) s_fill = 0;
  __syncthreads();
  for_each_hit(q, g, total, [&](int i, float, float, float) {
    if ((uint32_t)i <= thr) buf[atomicAdd(&s_fill, 1u)] = i;
  });
  __syncthreads();
  // bitonic sort of the k gathered indices (padded to a power of two)
  uint32_t m = 1;
  while (m < k) m <<= 1;
  for (uint32_t j = k + threadIdx.x; j < m; j += blockDim.x) buf[j] = 0x7fffffff;
  __syncthreads();
  for (uint32_t size = 2; size <= m; size <<= 1) {
    for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
      for (uint32_t t = threadIdx.x; t < m / 2; t += blockDim.x) {
        const uint32_t lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const int a = buf[lo], b = buf[hi];
        if ((a > b) == ((lo & size) == 0)) {
          buf[lo] = b;
          buf[hi] = a;
        }
      }
      __syncthreads();
    }
  }
  for (uint32_t j = threadIdx.x; j < k; j += blockDim.x) {
    const int i = buf[j];
    const size_t row = (size_t)base + j;
    const float x = pts[(size_t)i * 3], y = pts[(size_t)i * 3 + 1], z = pts[(size_t)i * 3 + 2];
    float lx, ly;
    to_local(q.o, x, y, lx, ly);
    const float lz = z - q.o.cz;
    float* f = out_feats + row * 13;
    f[0] = x;
    f[1] = y;
    f[2] = z;
    f[3] = lx;
    f[4] = ly;
    f[5] = lz;
    f[6] = q.o.hl + lx;
    f[7] = q.o.hw + ly;
    f[8] = q.o.hh + lz;
    f[9] = q.o.hl - lx;
    f[10] = q.o.hw - ly;
    f[11] = q.o.hh - lz;
    f[12] = in_box(q.o, z, lx, ly) ? 0.f : 1.f;
    out_idx[row] = i;
    out_roi[row] = r;
  }
}

}  // namespace

extern "C" int sstb200_dynamic_point_pool(sstb200_ctx* c, const float* rois, const int32_t* rois_batch, int num_rois, const float* pts,
                                          const int32_t* pts_batch, int num_pts, const float extra_wlh[3], int max_inbox_point,
                                          int max_all_pts, int per_sample, int64_t* out_pts_idx, int64_t* out_roi_idx, float* out_feats,
                                          int32_t* num_out_dev, int32_t* num_pairs_host) {
  CHECK_ARG(c, c && num_rois >= 0 && num_pts >= 0 && extra_wlh && num_out_dev && out_pts_idx && out_roi_idx && out_feats);
  CHECK_ARG(c, (rois_batch == nullptr) == (pts_batch == nullptr) && (!per_sample || rois_batch));
  CHECK_ARG(c, (num_rois == 0 || rois) && (num_pts == 0 || pts));
  if (max_inbox_point < 1) return sstb_fail(c, SSTB_ERR_ARG, "dynamic_point_pool: max_inbox_point must be >= 1 (got %d)", max_inbox_point);
  if (max_inbox_point > RP_MAX_INBOX)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "dynamic_point_pool: max_inbox_point %d > %d not built", max_inbox_point, RP_MAX_INBOX);
  if (max_all_pts < 1) return sstb_fail(c, SSTB_ERR_ARG, "dynamic_point_pool: max_all_pts must be >= 1 (got %d)", max_all_pts);
  const int R = num_rois, N = num_pts;
  const uint32_t T = grid_table_size(N);
  arena_reset(c);
  const size_t Rc = (size_t)R + 1;
  uint32_t *kept, *off, *take, *rows, *pos;
  // flags [0] negative point batch, [1] negative RoI batch, [2] RoI batch ids not ascending (per-sample mode), [3] fake rows; then the
  // temporaries of the two scans
  int32_t* flags;
  ScanTemps s1, s2;
  size_t zero_bytes;
  GridWs gw;
  int rc = arena_carve(c, [&](Carve& cv) {
    kept = cv.take<uint32_t>(Rc);
    off = cv.take<uint32_t>(Rc);
    take = cv.take<uint32_t>(Rc);
    rows = cv.take<uint32_t>(Rc);
    pos = cv.take<uint32_t>(Rc);
    const size_t z = cv.mark();
    flags = cv.take<int32_t>(64);
    scan_carve(cv, s1, Rc);
    scan_carve(cv, s2, Rc);
    zero_bytes = cv.off - z;
    grid_carve(cv, gw, N, T);
  });
  if (rc) return rc;
  CUDA_TRY(c, cudaMemsetAsync(flags, 0, zero_bytes, c->stream));
  Grid g;
  const uint32_t* binned = nullptr;
  rc = grid_build(c, gw, pts, pts_batch, N, T, make_float3(extra_wlh[0], extra_wlh[1], extra_wlh[2]), flags, g, &binned);
  if (rc) return rc;
  if (R > 0)
    launch_pdl(rp_count_kernel, dim3(R), dim3(RP_THREADS), (size_t)0, c->stream, rois, rois_batch, g, binned, max_inbox_point, per_sample,
               kept, flags);
  launch_exclusive_scan(c->stream, LoadU32{kept}, (size_t)R, nullptr, s1, off, s1.ticket + 1, true);
  if (R > 0)
    launch_pdl(rp_rows_kernel, dim3((R + 255) / 256), dim3(256), (size_t)0, c->stream, rois_batch, R, per_sample, max_all_pts,
               (const uint32_t*)kept, (const uint32_t*)off, take, rows, flags);
  launch_exclusive_scan(c->stream, LoadU32{rows}, (size_t)R, nullptr, s2, pos, s2.ticket + 1, true);
  if (R > 0) {
    uint32_t m = 1;
    while (m < (uint32_t)max_inbox_point) m <<= 1;
    launch_pdl(rp_write_kernel, dim3(R), dim3(RP_THREADS), (size_t)m * 4, c->stream, rois, rois_batch, g, binned, N, (const uint32_t*)take,
               (const uint32_t*)rows, (const uint32_t*)pos, pts, out_pts_idx, out_roi_idx, out_feats);
  }
  CUDA_TRY(c, cudaMemcpyAsync(num_out_dev, s2.ticket + 1, 4, cudaMemcpyDeviceToDevice, c->stream));
  LAUNCH_CHECK(c);
  if (num_pairs_host) {
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, s2.ticket + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32 + 1, s1.ticket + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32 + 2, flags, 16, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    const int32_t* h = c->pinned_i32;
    if (h[2] || h[3]) return sstb_fail(c, SSTB_ERR_ARG, "dynamic_point_pool: a %s batch id is negative", h[2] ? "point" : "RoI");
    if (h[4]) return sstb_fail(c, SSTB_ERR_ARG, "dynamic_point_pool: per-sample capacity needs the RoIs grouped by ascending batch id");
    num_pairs_host[0] = h[0];         // rows written
    num_pairs_host[1] = h[1];         // pairs found, at most max_inbox_point per RoI
    num_pairs_host[2] = h[0] - h[5];  // pairs written (rows less fake rows)
  }
  return SSTB_OK;
}
