// Rotated bird's-eye-view overlap, IoU and NMS (mmdet3d/ops/iou3d: iou3d_utils.py, src/iou3d.cpp, src/iou3d_kernel.cu), the test-time
// box selection of every SST / FSD head (box3d_multiclass_nms, nms_gpu, nms_normal_gpu) and the BEV overlap of the 3-D assigners.
//
// Geometry.  Boxes are [x1, y1, x2, y2, r] fp32.  Box corners (x1,y1), (x2,y1), (x2,y2), (x1,y2) are turned about the box centre by
// (dx cos r + dy sin r, -dx sin r + dy cos r), the reference's convention, so world offset = R(-r) * local offset.  The overlap of a and b
// is computed in a's frame: origin at a's centre, axes along a's sides, where a is the axis-aligned rectangle |x| <= hxa, |y| <= hya and
// b has centre R(ra) * (cb - ca) and is turned by ra - rb.  b's four corners are clipped against a's four sides by a streaming
// Sutherland-Hodgman pipeline (each stage keeps its first and previous vertex in registers; no vertex array) and the shoelace area of
// what comes out is the overlap.  The centre offset is formed from the differences of the raw coordinates, so boxes 75 m from the
// origin lose nothing to their absolute position.  Boxes whose circumscribed circles are apart give exactly 0 without clipping; a
// zero-area box gives 0 (never NaN).  iou = overlap / max(sa + sb - overlap, 1e-8) with s = (x2 - x1)(y2 - y1); the axis-aligned IoU
// of nms_normal_gpu ignores r.
//
// NMS over a list sorted by (segment, score descending), segment s = boxes [off[s], off[s+1]):
//   nms_mask_kernel  one CTA per upper-triangular 64 x 64 block (row block <= column block) of every segment; bit j of row i's word
//                    j / 64 is set iff j > i and IoU(i, j) > thresh[s].  Lower-triangular words are neither written nor read.
//   nms_scan_kernel  one CTA per segment: the greedy scan, 64 rows at a time - one lane resolves the diagonal word serially (visiting
//                    only surviving rows), then all threads OR the kept rows' words into the removed-bitmap in shared memory.
//   nms_pack_kernel  one CTA per segment: the kept positions, segment after segment, into keep_out; the total into num_keep_dev.
// The mask, the per-segment lists and the counts live in the caller's workspace (sstb200_nms_bev_workspace_bytes); no atomics at all.
#include <stdarg.h>
#include "bev_overlap.cuh"

namespace {

#define NMS_BLK 64            // boxes per mask word
#define NMS_MAX_SEG 65536     // boxes per segment: the scan's removed-bitmap (NMS_MAX_SEG / 64 words) lives in shared memory
#define NMS_MASK_THREADS 256  // 4 threads per row of a 64 x 64 block, 16 columns each
#define NMS_SCAN_THREADS 256
#define PAIR_ROWS 32          // dense overlap / IoU tile: 32 rows of a x 64 columns of b
#define PAIR_COLS 64

__device__ __forceinline__ float bev_iou(const BevBox& a, const BevBox& b) {
  const float ov = bev_overlap(a, b);
  return ov / fmaxf(a.area + b.area - ov, 1e-8f);
}

// axis-aligned IoU of nms_normal_gpu (r ignored)
__device__ __forceinline__ float normal_iou(const BevBox& a, const BevBox& b) {
  const float w = fmaxf(fminf(a.x2, b.x2) - fmaxf(a.x1, b.x1), 0.f), h = fmaxf(fminf(a.y2, b.y2) - fmaxf(a.y1, b.y1), 0.f);
  const float in = w * h;
  return in / fmaxf(a.area + b.area - in, 1e-8f);
}

template <bool ROT>
__device__ __forceinline__ float nms_iou(const BevBox& a, const BevBox& b) {
  return ROT ? bev_iou(a, b) : normal_iou(a, b);
}

// ---- dense [M, N] overlap / IoU -------------------------------------------------------------------------------------------------
template <bool IOU>
__global__ void __launch_bounds__(256, 2) bev_pair_kernel(const float* __restrict__ boxes_a, int M, const float* __restrict__ boxes_b, int N,
                                                       float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  __shared__ BevBox sa[PAIR_ROWS];
  __shared__ BevBox sb[PAIR_COLS];
  const int r0 = blockIdx.y * PAIR_ROWS, c0 = blockIdx.x * PAIR_COLS;
  const int t = threadIdx.x;
  if (t < PAIR_COLS && c0 + t < N) sb[t] = make_bev(boxes_b + (size_t)(c0 + t) * 5);
  else if (t >= PAIR_COLS && t < PAIR_COLS + PAIR_ROWS && r0 + t - PAIR_COLS < M) sa[t - PAIR_COLS] = make_bev(boxes_a + (size_t)(r0 + t - PAIR_COLS) * 5);
  __syncthreads();
  const int col = t % PAIR_COLS, j = c0 + col;
  if (j >= N) return;
  const BevBox b = sb[col];
  for (int row = t / PAIR_COLS; row < PAIR_ROWS && r0 + row < M; row += 256 / PAIR_COLS) {
    const BevBox& a = sa[row];
    out[(size_t)(r0 + row) * N + j] = IOU ? bev_iou(a, b) : bev_overlap(a, b);
  }
}

// ---- segmented NMS ---------------------------------------------------------------------------------------------------------------
// Per-segment table, uploaded once per call: box start, box count, first mask word, first mask CTA, threshold (as bits).
struct SegRow {
  long long start, n, mask_base, block_start;
  float thresh;
  int pad;
};

__device__ __forceinline__ int find_segment(const SegRow* __restrict__ seg, int S, long long blk) {
  int lo = 0, hi = S - 1;  // last segment whose block_start <= blk
  while (lo < hi) {
    const int m = (lo + hi + 1) >> 1;
    if (seg[m].block_start <= blk) lo = m;
    else hi = m - 1;
  }
  return lo;
}

template <bool ROT>
__global__ void __launch_bounds__(NMS_MASK_THREADS) nms_mask_kernel(const float* __restrict__ boxes, const SegRow* __restrict__ seg, int S,
                                                                    unsigned long long* __restrict__ mask) {
  pdl_wait();
  pdl_launch();
  __shared__ BevBox cols[NMS_BLK];
  const long long blk = blockIdx.x;
  const SegRow g = seg[find_segment(seg, S, blk)];
  const int n = (int)g.n, nb = (n + NMS_BLK - 1) / NMS_BLK;
  // upper triangle, row-major; counted from the end, the rows have 1, 2, ... blocks
  const long long u = (long long)nb * (nb + 1) / 2 - 1 - (blk - g.block_start);
  int k = (int)((sqrt(8.0 * (double)u + 1.0) - 1.0) * 0.5);
  while ((long long)(k + 1) * (k + 2) / 2 <= u) k++;
  while ((long long)k * (k + 1) / 2 > u) k--;
  const int rb = nb - 1 - k, cb = rb + (int)(u - (long long)k * (k + 1) / 2);
  const float* base = boxes + (size_t)g.start * 5;
  const int t = threadIdx.x;
  if (t < NMS_BLK && cb * NMS_BLK + t < n) cols[t] = make_bev(base + (size_t)(cb * NMS_BLK + t) * 5);
  __syncthreads();
  const int row = t >> 2, part = t & 3, i = rb * NMS_BLK + row;
  unsigned long long bits = 0;
  if (i < n) {
    const BevBox a = make_bev(base + (size_t)i * 5);
    const int c_lo = part * 16, c_hi = min(c_lo + 16, n - cb * NMS_BLK);
    for (int c = max(c_lo, rb == cb ? row + 1 : 0); c < c_hi; c++)
      if (nms_iou<ROT>(a, cols[c]) > g.thresh) bits |= 1ull << c;
  }
  bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
  bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
  if (part == 0 && i < n) mask[g.mask_base + (long long)i * nb + cb] = bits;
}

__global__ void __launch_bounds__(NMS_SCAN_THREADS) nms_scan_kernel(const SegRow* __restrict__ seg, const unsigned long long* __restrict__ mask,
                                                                    int32_t* __restrict__ keep_local, int32_t* __restrict__ counts) {
  pdl_wait();
  pdl_launch();
  __shared__ unsigned long long removed[NMS_MAX_SEG / NMS_BLK];
  __shared__ unsigned long long diag[NMS_BLK];
  __shared__ unsigned long long s_keep;
  const SegRow g = seg[blockIdx.x];
  const int n = (int)g.n, nb = (n + NMS_BLK - 1) / NMS_BLK, t = threadIdx.x;
  const unsigned long long* m = mask + g.mask_base;
  int32_t* out = keep_local + g.start;
  for (int j = t; j < nb; j += NMS_SCAN_THREADS) removed[j] = 0;
  int cnt = 0;
  for (int k = 0; k < nb; k++) {
    __syncthreads();  // removed[k] is final
    const int r0 = k * NMS_BLK, rn = min(NMS_BLK, n - r0);
    if (t < 32) {  // warp 0 stages the diagonal words, lane 0 resolves them
      diag[t] = t < rn ? m[(long long)(r0 + t) * nb + k] : 0ull;
      diag[t + 32] = t + 32 < rn ? m[(long long)(r0 + t + 32) * nb + k] : 0ull;
      __syncwarp();
    }
    if (t == 0) {
      // rows past the segment count as removed; visit only the surviving rows, lowest first
      unsigned long long gone = removed[k] | (rn < NMS_BLK ? ~0ull << rn : 0ull), keep = 0;
      for (unsigned long long avail = ~gone; avail;) {
        const int b = __ffsll((long long)avail) - 1;
        keep |= 1ull << b;
        gone |= diag[b];
        avail = ~gone & (b == 63 ? 0ull : ~0ull << (b + 1));
      }
      s_keep = keep;
    }
    __syncthreads();
    const unsigned long long keep = s_keep;
    if (t < NMS_BLK && ((keep >> t) & 1ull)) out[cnt + __popcll(keep & ((1ull << t) - 1ull))] = r0 + t;
    for (int j = k + 1 + t; j < nb; j += NMS_SCAN_THREADS) {
      unsigned long long acc = removed[j];
      for (unsigned long long kb = keep; kb; kb &= kb - 1) acc |= m[(long long)(r0 + __ffsll((long long)kb) - 1) * nb + j];
      removed[j] = acc;
    }
    cnt += __popcll(keep);
  }
  if (t == 0) counts[blockIdx.x] = cnt;
}

__global__ void nms_pack_kernel(const SegRow* __restrict__ seg, int S, const int32_t* __restrict__ keep_local,
                                const int32_t* __restrict__ counts, int64_t* __restrict__ keep_out, int32_t* __restrict__ num_keep) {
  pdl_wait();
  pdl_launch();
  __shared__ int s_at;
  const int s = blockIdx.x;
  if (threadIdx.x == 0) {
    int at = 0;
    for (int q = 0; q < s; q++) at += counts[q];
    s_at = at;
    if (s == S - 1) *num_keep = at + counts[s];
  }
  __syncthreads();
  const SegRow g = seg[s];
  const int c = counts[s], at = s_at;
  for (int q = threadIdx.x; q < c; q += blockDim.x) keep_out[at + q] = g.start + keep_local[g.start + q];
}

// the caller-owned workspace: mask words | segment table | per-segment kept lists (int32 [num]) | counts
struct NmsWs {
  unsigned long long* mask;
  SegRow* table;
  int32_t *lists, *counts;
};

void nms_carve(Carve& cv, NmsWs& w, int num, const int32_t* off, int S) {
  size_t words = 0;
  for (int s = 0; s < S; s++) {
    const size_t n = (size_t)(off[s + 1] - off[s]);
    words += n * ((n + NMS_BLK - 1) / NMS_BLK);
  }
  w.mask = cv.take<unsigned long long>(words);
  w.table = cv.take<SegRow>(S);
  w.lists = cv.take<int32_t>(num);
  w.counts = cv.take<int32_t>(S);
}

size_t nms_bytes(int num, const int32_t* off, int S) {
  return carve_bytes([&](Carve& cv) {
    NmsWs w;
    nms_carve(cv, w, num, off, S);
  });
}

int check_segments(sstb200_ctx* c, int num, const int32_t* off, int S) {
  if (num < 0 || S < 0) return sstb_fail(c, SSTB_ERR_ARG, "nms_bev: negative size (num %d, num_segs %d)", num, S);
  if (S > 0 && !off) return sstb_fail(c, SSTB_ERR_ARG, "nms_bev: seg_offsets is NULL");
  if (S == 0) return num == 0 ? SSTB_OK : sstb_fail(c, SSTB_ERR_ARG, "nms_bev: %d boxes but no segment", num);
  if (off[0] != 0 || off[S] != num) return sstb_fail(c, SSTB_ERR_ARG, "nms_bev: seg_offsets must run from 0 to num (%d .. %d, num %d)", off[0], off[S], num);
  for (int s = 0; s < S; s++) {
    if (off[s + 1] < off[s]) return sstb_fail(c, SSTB_ERR_ARG, "nms_bev: seg_offsets decrease at segment %d", s);
    if (off[s + 1] - off[s] > NMS_MAX_SEG)
      return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "nms_bev: segment %d holds %d boxes; at most %d per segment are supported", s,
                       off[s + 1] - off[s], NMS_MAX_SEG);
  }
  return SSTB_OK;
}

int bev_pairs(sstb200_ctx* c, const float* a, int M, const float* b, int N, float* out, bool iou) {
  CHECK_ARG(c, c && M >= 0 && N >= 0 && (M == 0 || a) && (N == 0 || b) && ((long long)M * N == 0 || out));
  if (M == 0 || N == 0) return SSTB_OK;
  const dim3 grid((N + PAIR_COLS - 1) / PAIR_COLS, (M + PAIR_ROWS - 1) / PAIR_ROWS);
  if (grid.y > 65535) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "boxes_%s_bev: %d boxes_a exceed %d", iou ? "iou" : "overlap", M, 65535 * PAIR_ROWS);
  if (iou) CUDA_TRY(c, launch_pdl(bev_pair_kernel<true>, grid, dim3(256), (size_t)0, c->stream, a, M, b, N, out));
  else CUDA_TRY(c, launch_pdl(bev_pair_kernel<false>, grid, dim3(256), (size_t)0, c->stream, a, M, b, N, out));
  return SSTB_OK;
}

}  // namespace

extern "C" int sstb200_boxes_overlap_bev(sstb200_ctx* c, const float* boxes_a, int num_a, const float* boxes_b, int num_b, float* overlap) {
  return bev_pairs(c, boxes_a, num_a, boxes_b, num_b, overlap, false);
}

extern "C" int sstb200_boxes_iou_bev(sstb200_ctx* c, const float* boxes_a, int num_a, const float* boxes_b, int num_b, float* iou) {
  return bev_pairs(c, boxes_a, num_a, boxes_b, num_b, iou, true);
}

extern "C" int sstb200_nms_bev_workspace_bytes(sstb200_ctx* c, int num, const int32_t* seg_offsets, int num_segs, int64_t* bytes) {
  CHECK_ARG(c, c && bytes);
  const int rc = check_segments(c, num, seg_offsets, num_segs);
  if (rc) return rc;
  *bytes = (int64_t)nms_bytes(num, seg_offsets, num_segs);
  return SSTB_OK;
}

extern "C" int sstb200_nms_bev(sstb200_ctx* c, const float* boxes, int num, const int32_t* seg_offsets, int num_segs, const float* thresh,
                               int rotated, void* workspace, int64_t workspace_bytes, int64_t* keep_out, int32_t* num_keep_dev,
                               int32_t* num_keep_host) {
  CHECK_ARG(c, c && num_keep_dev);
  int rc = check_segments(c, num, seg_offsets, num_segs);
  if (rc) return rc;
  CHECK_ARG(c, (num == 0 || (boxes && keep_out)) && (num_segs == 0 || thresh));
  const size_t need = nms_bytes(num, seg_offsets, num_segs);
  if (!workspace) return sstb_fail(c, SSTB_ERR_ARG, "nms_bev: workspace is NULL (%zu bytes needed)", need);
  if (workspace_bytes < (int64_t)need)
    return sstb_fail(c, SSTB_ERR_WORKSPACE, "nms_bev: workspace of %lld bytes, %zu needed", (long long)workspace_bytes, need);
  NmsWs w;
  Carve wc{(char*)workspace, 0};
  nms_carve(wc, w, num, seg_offsets, num_segs);
  if (num_segs == 0) {
    CUDA_TRY(c, cudaMemsetAsync(num_keep_dev, 0, 4, c->stream));
  } else {
    std::vector<SegRow> tab(num_segs);
    long long words = 0, blocks = 0;
    for (int s = 0; s < num_segs; s++) {
      const long long n = seg_offsets[s + 1] - seg_offsets[s], nb = (n + NMS_BLK - 1) / NMS_BLK;
      tab[s] = SegRow{seg_offsets[s], n, words, blocks, thresh[s], 0};
      words += n * nb;
      blocks += nb * (nb + 1) / 2;
    }
    if (blocks > 0x7fffffffLL) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "nms_bev: %lld mask blocks exceed one grid", blocks);
    SegRow* dtab = w.table;
    int32_t *lists = w.lists, *counts = w.counts;
    unsigned long long* mask = w.mask;
    // from pageable memory: staged before the call returns, so `tab` may go out of scope
    CUDA_TRY(c, cudaMemcpyAsync(dtab, tab.data(), (size_t)num_segs * sizeof(SegRow), cudaMemcpyHostToDevice, c->stream));
    if (blocks > 0) {
      if (rotated) CUDA_TRY(c, launch_pdl(nms_mask_kernel<true>, dim3((unsigned)blocks), dim3(NMS_MASK_THREADS), (size_t)0, c->stream, boxes,
                                          (const SegRow*)dtab, num_segs, mask));
      else CUDA_TRY(c, launch_pdl(nms_mask_kernel<false>, dim3((unsigned)blocks), dim3(NMS_MASK_THREADS), (size_t)0, c->stream, boxes,
                                  (const SegRow*)dtab, num_segs, mask));
    }
    CUDA_TRY(c, launch_pdl(nms_scan_kernel, dim3(num_segs), dim3(NMS_SCAN_THREADS), (size_t)0, c->stream, (const SegRow*)dtab,
                           (const unsigned long long*)mask, lists, counts));
    CUDA_TRY(c, launch_pdl(nms_pack_kernel, dim3(num_segs), dim3(128), (size_t)0, c->stream, (const SegRow*)dtab, num_segs,
                           (const int32_t*)lists, (const int32_t*)counts, keep_out, num_keep_dev));
  }
  LAUNCH_CHECK(c);
  if (num_keep_host) {
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, num_keep_dev, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    *num_keep_host = c->pinned_i32[0];
  }
  return SSTB_OK;
}
