// mmdet3d/ops/roiaware_pool3d: points_in_boxes_gpu / points_in_boxes_batch (src/points_in_boxes_cuda.cu) and RoIAwarePool3d forward /
// backward (src/roiaware_pool3d_kernel.cu), as used by VoteSegHead.get_targets, SingleStageFSD(V2) (add_gt_fg_points), the LiDAR /
// Depth box structures and Single3DRoIAwareExtractor (PartA2's RoI layer).
//
// points_in_boxes: a block stages chunks of its sample's boxes in shared memory (each box turned into a Box once per block) and tests
// its points against them.  `first` keeps the lowest box index per point; `all` collects the tile's membership bits in shared memory
// (one warp ballot per point and 32 boxes) and then streams its contiguous [rows x T] int32 output range with 16-byte stores.
//
// RoIAwarePool3d: the (RoI, point) pairs come from the point grid of box3d.cuh (count pass, scan, one sync for the pair count).  The
// emit pass writes one 64-bit key (roi | voxel | point) per pair, cub's radix sort orders them, and a run-length pass over (roi, voxel)
// keeps each voxel's first m - 1 points: the occupied-voxel table and the kept-point CSR, which are all the backward needs besides
// the [occupied, C] argmax.  One pass then writes the dense pooled output.  The backward sorts the kept entries by point (stable, so
// each point's slots stay in (roi, voxel) order) and every (point, channel) sums its terms in that order: no float atomics.
#include <stdarg.h>
#include <cub/device/device_radix_sort.cuh>
#include "box3d.cuh"

namespace {

#define PIB_THREADS 256
#define PIB_CHUNK 256          // boxes staged in shared memory per step
#define PIB_MAX_ROWS 64        // points per block in `all` mode
#define PIB_BITS_SMEM (96 * 1024)

__device__ __forceinline__ Box load_box(const float* __restrict__ q) { return make_box(q[0], q[1], q[2], q[3], q[4], q[5], q[6]); }

// ---- points_in_boxes, first mode: out[b, i] = lowest k with point i inside box k of sample b, else -1 -------------------------------
__global__ void __launch_bounds__(PIB_THREADS) pib_first_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, int M, int T,
                                                                int blocks_per_sample, int32_t* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  __shared__ Box sb[PIB_CHUNK];
  const int b = blockIdx.x / blocks_per_sample;
  const int i = (blockIdx.x % blocks_per_sample) * PIB_THREADS + threadIdx.x;
  const bool live = i < M;
  float x = 0.f, y = 0.f, z = 0.f;
  if (live) {
    const float* p = pts + ((size_t)b * M + i) * 3;
    x = p[0], y = p[1], z = p[2];
  }
  const float* bx = boxes + (size_t)b * T * 7;
  int hit = -1;
  for (int k0 = 0; k0 < T; k0 += PIB_CHUNK) {
    const int n = min(PIB_CHUNK, T - k0);
    if (threadIdx.x < n) sb[threadIdx.x] = load_box(bx + (size_t)(k0 + threadIdx.x) * 7);
    __syncthreads();
    if (live && hit < 0)
      for (int k = 0; k < n; k++) {
        float lx, ly;
        to_local(sb[k], x, y, lx, ly);
        if (in_box(sb[k], z, lx, ly)) {
          hit = k0 + k;
          break;
        }
      }
    if (__syncthreads_and(!live || hit >= 0)) break;  // also orders this chunk's reads before the next chunk's stores
  }
  if (live) out[(size_t)b * M + i] = hit;
}

// ---- points_in_boxes, all mode: out[b, i, k] = 1 if point i is inside box k of sample b, else 0 ------------------------------------
__global__ void __launch_bounds__(PIB_THREADS) pib_all_kernel(const float* __restrict__ pts, const float* __restrict__ boxes, int M, int T,
                                                              int rows_per_block, int blocks_per_sample, int32_t* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint32_t bits[];  // [rows_per_block][W]: bit k & 31 of word k >> 5 = point in box k
  __shared__ Box sb[PIB_CHUNK];
  __shared__ float4 sp[PIB_MAX_ROWS];
  const int W = (T + 31) >> 5;
  const int b = blockIdx.x / blocks_per_sample;
  const int row0 = (blockIdx.x % blocks_per_sample) * rows_per_block;
  const int rows = min(rows_per_block, M - row0);
  if (threadIdx.x < rows) {
    const float* p = pts + ((size_t)b * M + row0 + threadIdx.x) * 3;
    sp[threadIdx.x] = make_float4(p[0], p[1], p[2], 0.f);
  }
  const float* bx = boxes + (size_t)b * T * 7;
  const int warp = threadIdx.x >> 5, lane = lane_id();
  for (int k0 = 0; k0 < T; k0 += PIB_CHUNK) {
    const int n = min(PIB_CHUNK, T - k0);
    __syncthreads();  // the previous chunk's boxes are consumed
    if (threadIdx.x < n) sb[threadIdx.x] = load_box(bx + (size_t)(k0 + threadIdx.x) * 7);
    __syncthreads();
    if (warp * 32 < n) {  // warp-uniform: this warp owns boxes k0 + 32 warp + lane
      const int kk = warp * 32 + lane;
      const bool valid = kk < n;
      const Box bb = sb[valid ? kk : 0];
      for (int r = 0; r < rows; r++) {
        const float4 p = sp[r];
        float lx, ly;
        to_local(bb, p.x, p.y, lx, ly);
        const unsigned word = __ballot_sync(0xffffffffu, valid && in_box(bb, p.z, lx, ly));
        if (lane == 0) bits[r * W + (k0 >> 5) + warp] = word;
      }
    }
  }
  __syncthreads();
  // the tile's output is the contiguous range [base, base + rows * T): scalar head up to 16-byte alignment, int4 body, scalar tail.
  // The head comes from the address, not from base: the caller's `out` need only be 4-byte aligned, and an `out` 4, 8 or 12 bytes past
  // a 16-byte boundary would otherwise put every int4 store off its alignment.
  const size_t base = ((size_t)b * M + row0) * (size_t)T;
  const long long E = (long long)rows * T;
  const long long head = min((long long)((4 - ((reinterpret_cast<uintptr_t>(out + base) >> 2) & 3)) & 3), E);
  auto bit = [&](int r, int col) -> int { return (int)((bits[r * W + (col >> 5)] >> (col & 31)) & 1u); };
  for (long long e = threadIdx.x; e < head; e += blockDim.x) out[base + e] = bit((int)(e / T), (int)(e % T));
  const long long nvec = (E - head) >> 2;
  int4* o4 = reinterpret_cast<int4*>(out + base + head);
  for (long long v = threadIdx.x; v < nvec; v += blockDim.x) {
    const long long e = head + 4 * v;
    int r = (int)(e / T), col = (int)(e - (long long)r * T);
    int q[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      q[u] = bit(r, col);
      if (++col == T) col = 0, r++;
    }
    o4[v] = make_int4(q[0], q[1], q[2], q[3]);
  }
  for (long long e = head + 4 * nvec + threadIdx.x; e < E; e += blockDim.x) out[base + e] = bit((int)(e / T), (int)(e % T));
}

// ---- RoIAwarePool3d ------------------------------------------------------------------------------------------------------------
struct VoxGrid {
  int ox, oy, oz;
  int vbits, pbits;  // key = roi << (vbits + pbits) | voxel << pbits | point
};

// roiaware_pool3d_kernel.cu:79-89 as the same fp32 expressions: res = dim / out, idx = int((local + dim / 2) / res) (local z from the
// bottom), then min(max(idx, 0), out - 1) on an UNSIGNED idx, so a negative index lands in the last cell as it does there
__device__ __forceinline__ uint32_t voxel_of(const float* __restrict__ roi, const VoxGrid& v, float lx, float ly, float z) {
  const float w = roi[3], l = roi[4], h = roi[5];
  const float x_res = l / v.ox, y_res = w / v.oy, z_res = h / v.oz;
  unsigned xi = (unsigned)(int)((lx + l / 2) / x_res);
  unsigned yi = (unsigned)(int)((ly + w / 2) / y_res);
  unsigned zi = (unsigned)(int)((z - roi[2]) / z_res);
  xi = min(xi, (unsigned)(v.ox - 1));
  yi = min(yi, (unsigned)(v.oy - 1));
  zi = min(zi, (unsigned)(v.oz - 1));
  return (xi * (unsigned)v.oy + yi) * (unsigned)v.oz + zi;
}

// pass 1: pairs per RoI (a negative RoI batch id sets flags[1] and pairs with nothing)
__global__ void __launch_bounds__(RP_THREADS) ra_count_kernel(const float* __restrict__ rois, const int32_t* __restrict__ rois_batch, Grid g,
                                                              const uint32_t* __restrict__ total, uint32_t* __restrict__ hits,
                                                              int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  __shared__ uint32_t sh[RP_THREADS / 32];
  const int r = blockIdx.x;
  const RoiPair q = load_roi(rois, rois_batch, r, g.ex);
  uint32_t n = 0;
  for_each_hit(q, g, total, [&](int, float, float, float) { n++; });
  n = block_sum(n, sh);
  if (threadIdx.x == 0) {
    hits[r] = n;
    if (q.batch < 0) flags[1] = 1;
  }
}

// pass 2: one key per pair at off[r] + (any order inside the RoI: the sort orders them)
__global__ void __launch_bounds__(RP_THREADS) ra_emit_kernel(const float* __restrict__ rois, const int32_t* __restrict__ rois_batch, Grid g,
                                                             const uint32_t* __restrict__ total, const uint32_t* __restrict__ off, VoxGrid v,
                                                             unsigned long long* __restrict__ keys) {
  pdl_wait();
  pdl_launch();
  __shared__ uint32_t s_fill;
  const int r = blockIdx.x;
  if (threadIdx.x == 0) s_fill = 0;
  __syncthreads();
  const RoiPair q = load_roi(rois, rois_batch, r, g.ex);
  const float* roi = rois + (size_t)r * 7;
  const unsigned long long rk = (unsigned long long)r << (v.vbits + v.pbits);
  unsigned long long* dst = keys + off[r];
  for_each_hit(q, g, total, [&](int i, float x, float y, float z) {
    float lx, ly;
    to_local(q.o, x, y, lx, ly);
    dst[atomicAdd(&s_fill, 1u)] = rk | ((unsigned long long)voxel_of(roi, v, lx, ly, z) << v.pbits) | (unsigned long long)i;
  });
}

// run-length pass over the sorted keys, part 1: head[j] = 1 where a new (roi, voxel) starts
__global__ void ra_head_kernel(const unsigned long long* __restrict__ k, long long P, int pbits, uint32_t* __restrict__ head) {
  pdl_wait();
  pdl_launch();
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  head[j] = (j == 0 || (k[j] >> pbits) != (k[j - 1] >> pbits)) ? 1u : 0u;
}

// part 2: for group g (gid = exclusive scan of head, gid[P] = groups): its first sorted position, its dense slot roi * nvox + voxel
// and its kept count min(run, m - 1)
__global__ void ra_group_kernel(const unsigned long long* __restrict__ k, long long P, const uint32_t* __restrict__ head,
                                const uint32_t* __restrict__ gid, int vbits, int pbits, long long nvox, uint32_t* __restrict__ gstart,
                                int64_t* __restrict__ slot) {
  pdl_wait();
  pdl_launch();
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j == 0) gstart[gid[P]] = (uint32_t)P;
  if (j >= P || !head[j]) return;
  const uint32_t g = gid[j];
  const unsigned long long key = k[j];
  gstart[g] = (uint32_t)j;
  slot[g] = (int64_t)(key >> (vbits + pbits)) * nvox + (int64_t)((key >> pbits) & ((1ull << vbits) - 1));
}

__global__ void ra_kept_count_kernel(const uint32_t* __restrict__ gstart, const uint32_t* __restrict__ num_groups, long long P, int keep,
                                     uint32_t* __restrict__ kcnt) {
  pdl_wait();
  pdl_launch();
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)*num_groups || g >= P) return;
  kcnt[g] = min(gstart[g + 1] - gstart[g], (uint32_t)keep);
}

// part 3: the kept-point CSR (point indices ascending within a voxel: the sort put them so)
__global__ void ra_fill_kernel(const unsigned long long* __restrict__ k, long long P, int pbits, const uint32_t* __restrict__ gid,
                               const uint32_t* __restrict__ gstart, const int32_t* __restrict__ voff, int keep, int32_t* __restrict__ kept) {
  pdl_wait();
  pdl_launch();
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const uint32_t g = gid[j + 1] - 1;  // heads in [0, j] less one
  const uint32_t rank = (uint32_t)j - gstart[g];
  if (rank < (uint32_t)keep) kept[voff[g] + rank] = (int32_t)(k[j] & ((1ull << pbits) - 1));
}

// The dense output [R * nvox, C]: one warp per 32 consecutive slots, lanes over channels.  Occupied slots pool their kept points in
// ascending point order (roiaware_pool3d_kernel.cu:140-237): max from -inf with a strict `>` (argmax = first point reaching it; an
// empty or all-NaN / -inf voxel writes 0 and argmax -1), avg as a sequential fp32 sum / count.  Every other slot writes 0.
template <bool MAX>
__global__ void __launch_bounds__(256) ra_pool_kernel(const float* __restrict__ feats, int C, long long S, const int64_t* __restrict__ slot,
                                                      const int32_t* __restrict__ voff, const int32_t* __restrict__ kept,
                                                      const int32_t* __restrict__ counts, float* __restrict__ pooled,
                                                      int32_t* __restrict__ argmax) {
  pdl_wait();
  pdl_launch();
  const long long s0 = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32;
  if (s0 >= S) return;
  const int lane = lane_id();
  const int V = counts[0];
  int lo = 0, hi = V;  // first occupied group with slot >= s0
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (slot[mid] < s0) lo = mid + 1;
    else hi = mid;
  }
  int g = lo;
  const long long s1 = min(s0 + 32, S);
  for (long long s = s0; s < s1; s++) {
    float* o = pooled + s * C;
    if (g < V && slot[g] == s) {
      const int b = voff[g], e = voff[g + 1];
      for (int c = lane; c < C; c += 32) {
        if (MAX) {
          float best = -INFINITY;
          int arg = -1;
          for (int t = b; t < e; t++) {
            const int p = kept[t];
            const float x = feats[(size_t)p * C + c];
            if (x > best) {
              best = x;
              arg = p;
            }
          }
          o[c] = arg < 0 ? 0.f : best;
          argmax[(size_t)g * C + c] = arg;
        } else {
          float sum = 0.f;
          for (int t = b; t < e; t++) sum = __fadd_rn(sum, feats[(size_t)kept[t] * C + c]);
          o[c] = e > b ? __fdiv_rn(sum, (float)(e - b)) : 0.f;
        }
      }
      g++;
    } else {
      for (int c = lane; c < C; c += 32) o[c] = 0.f;
    }
  }
}

// backward, part 1: (point, group) of every kept entry, padded to P entries with point = N (sorted past every real point)
__global__ void ra_inverse_kernel(const int32_t* __restrict__ voff, const int32_t* __restrict__ kept, const int32_t* __restrict__ counts,
                                  long long P, int N, uint32_t* __restrict__ pkey, uint32_t* __restrict__ pgroup) {
  pdl_wait();
  pdl_launch();
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P) return;
  const int V = counts[0], K = counts[1];
  if (k >= K) {
    pkey[k] = (uint32_t)N;
    pgroup[k] = 0;
    return;
  }
  int lo = 0, hi = V - 1;  // last group whose range starts at or before k (every group of a call with K > 0 keeps >= 1 point)
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (voff[mid] <= k) lo = mid;
    else hi = mid - 1;
  }
  pkey[k] = (uint32_t)kept[k];
  pgroup[k] = (uint32_t)lo;
}

// backward, part 2: grad_in[i, c] = sum over the groups holding point i, in (roi, voxel) order, of max: grad_out if argmax is i;
// avg: grad_out * (1 / max(count, 1)) (roiaware_pool3d_kernel.cu:288-352 without the atomics)
template <bool MAX>
__global__ void __launch_bounds__(256) ra_grad_kernel(const uint32_t* __restrict__ pkey, const uint32_t* __restrict__ pgroup, long long P,
                                                      int N, int C, const int64_t* __restrict__ slot, const int32_t* __restrict__ voff,
                                                      const int32_t* __restrict__ argmax, const float* __restrict__ grad_out,
                                                      float* __restrict__ grad_in) {
  pdl_wait();
  pdl_launch();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * C) return;
  const int i = (int)(t / C), c = (int)(t - (long long)i * C);
  long long lo = 0, hi = P;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (pkey[mid] < (uint32_t)i) lo = mid + 1;
    else hi = mid;
  }
  float sum = 0.f;
  for (long long j = lo; j < P && pkey[j] == (uint32_t)i; j++) {
    const uint32_t g = pgroup[j];
    const float go = grad_out[(size_t)slot[g] * C + c];
    if (MAX) {
      if (argmax[(size_t)g * C + c] == i) sum = __fadd_rn(sum, go);
    } else {
      const float cur = __fdiv_rn(1.f, fmaxf((float)(voff[g + 1] - voff[g]), 1.f));
      sum = __fadd_rn(sum, __fmul_rn(go, cur));
    }
  }
  grad_in[t] = sum;
}

static int bits_for(long long n) {  // bits to hold 0 .. n - 1
  int b = 0;
  while (b < 63 && (1ll << b) < n) b++;
  return b;
}

// what sstb200_roiaware_pool3d_plan leaves in the arena for sstb200_roiaware_pool3d_forward
struct RoiAwarePlan {
  const float* rois;
  const int32_t* rois_batch;
  int R, N;
  VoxGrid v;
  int keep;  // m - 1
  Grid g;
  const uint32_t* binned;
  const uint32_t* off;  // [R + 1] pair offsets per RoI
  long long P;
};

}  // namespace

extern "C" int sstb200_points_in_boxes(sstb200_ctx* c, const float* pts, const float* boxes, int batch, int num_pts, int num_boxes, int mode,
                                       int32_t* out) {
  CHECK_ARG(c, c && batch >= 0 && num_pts >= 0 && num_boxes >= 0);
  if (mode != SSTB200_PIB_FIRST && mode != SSTB200_PIB_ALL) return sstb_fail(c, SSTB_ERR_ARG, "points_in_boxes: mode %d is neither first nor all", mode);
  const int B = batch, M = num_pts, T = num_boxes;
  if ((long long)B * M == 0 || (mode == SSTB200_PIB_ALL && T == 0)) return SSTB_OK;
  CHECK_ARG(c, pts && out && (T == 0 || boxes));
  if (mode == SSTB200_PIB_FIRST) {
    const int nb = (M + PIB_THREADS - 1) / PIB_THREADS;
    if ((long long)nb * B > 0x7fffffffll) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "points_in_boxes: %d x %d points", B, M);
    launch_pdl(pib_first_kernel, dim3((unsigned)(nb * B)), dim3(PIB_THREADS), (size_t)0, c->stream, pts, boxes, M, T, nb, out);
  } else {
    const size_t row_bytes = (size_t)((T + 31) / 32) * 4;
    const int rows = (int)min((size_t)PIB_MAX_ROWS, PIB_BITS_SMEM / row_bytes);
    if (rows < 1) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "points_in_boxes: %d boxes per sample exceed the all-mode tile", T);
    const int nb = (M + rows - 1) / rows;
    if ((long long)nb * B > 0x7fffffffll) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "points_in_boxes: %d x %d points", B, M);
    const size_t smem = (size_t)rows * row_bytes;
    static SmemAttr sa;
    CUDA_TRY(c, ensure_smem(c, sa, pib_all_kernel, (size_t)PIB_BITS_SMEM));
    launch_pdl(pib_all_kernel, dim3((unsigned)(nb * B)), dim3(PIB_THREADS), smem, c->stream, pts, boxes, M, T, rows, nb, out);
  }
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_roiaware_pool3d_plan(sstb200_ctx* c, const float* rois, const int32_t* rois_batch, int num_rois, const float* pts,
                                            const int32_t* pts_batch, int num_pts, const int32_t out_size[3], int max_pts_per_voxel,
                                            int64_t* num_pairs_host) {
  CHECK_ARG(c, c && num_rois >= 0 && num_pts >= 0 && out_size && num_pairs_host);
  CHECK_ARG(c, (rois_batch == nullptr) == (pts_batch == nullptr));
  CHECK_ARG(c, (num_rois == 0 || rois) && (num_pts == 0 || pts));
  c->handoff.reset();
  for (int d = 0; d < 3; d++)
    if (out_size[d] < 1 || out_size[d] > 255)
      return sstb_fail(c, SSTB_ERR_ARG, "roiaware_pool3d: out_size[%d] = %d outside [1, 255]", d, out_size[d]);
  if (max_pts_per_voxel < 1) return sstb_fail(c, SSTB_ERR_ARG, "roiaware_pool3d: max_pts_per_voxel must be >= 1 (got %d)", max_pts_per_voxel);
  const int R = num_rois, N = num_pts;
  const long long nvox = (long long)out_size[0] * out_size[1] * out_size[2];
  auto plan = std::make_shared<RoiAwarePlan>();
  plan->rois = rois;
  plan->rois_batch = rois_batch;
  plan->R = R;
  plan->N = N;
  plan->v.ox = out_size[0], plan->v.oy = out_size[1], plan->v.oz = out_size[2];
  plan->v.vbits = bits_for(nvox);
  plan->v.pbits = bits_for(N);
  plan->keep = max_pts_per_voxel - 1;
  if (bits_for(R) + plan->v.vbits + plan->v.pbits > 64)
    return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "roiaware_pool3d: %d RoIs x %lld voxels x %d points exceed a 64-bit pair key", R, nvox, N);
  const uint32_t T = grid_table_size(N);
  arena_reset(c);
  const size_t Rc = (size_t)R + 1;
  uint32_t *hits, *off;
  int32_t* flags;  // [0] negative point batch, [1] negative RoI batch; then the scan's temporaries
  ScanTemps s;
  size_t zero_bytes;
  GridWs gw;
  int rc = arena_carve(c, [&](Carve& cv) {
    hits = cv.take<uint32_t>(Rc);
    off = cv.take<uint32_t>(Rc);
    const size_t z = cv.mark();
    flags = cv.take<int32_t>(64);
    scan_carve(cv, s, Rc);
    zero_bytes = cv.off - z;
    grid_carve(cv, gw, N, T);
  });
  if (rc) return rc;
  CUDA_TRY(c, cudaMemsetAsync(flags, 0, zero_bytes, c->stream));
  rc = grid_build(c, gw, pts, pts_batch, N, T, make_float3(0.f, 0.f, 0.f), flags, plan->g, &plan->binned);
  if (rc) return rc;
  if (R > 0)
    launch_pdl(ra_count_kernel, dim3(R), dim3(RP_THREADS), (size_t)0, c->stream, rois, rois_batch, plan->g, plan->binned, hits, flags);
  // a 64-bit pair total: the 32-bit scan cannot overflow silently, since hits[r] <= N and a total past 2^31 is refused below
  launch_exclusive_scan(c->stream, LoadU32{hits}, (size_t)R, nullptr, s, off, s.ticket + 1, true);
  LAUNCH_CHECK(c);
  CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, flags, 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32 + 2, s.ticket + 1, 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  const int32_t* h = c->pinned_i32;
  if (h[0] || h[1]) return sstb_fail(c, SSTB_ERR_ARG, "roiaware_pool3d: a %s batch id is negative", h[0] ? "point" : "RoI");
  const long long P = (long long)(uint32_t)h[2];
  if (P > 0x7fffffffll) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "roiaware_pool3d: %lld RoI-point pairs exceed 2^31 - 1", P);
  plan->off = off;
  plan->P = P;
  *num_pairs_host = P;
  c->handoff = plan;
  c->handoff_epoch = c->arena_epoch;
  return SSTB_OK;
}

extern "C" int sstb200_roiaware_pool3d_forward(sstb200_ctx* c, const float* pts_feature, int channels, int mode, float* pooled,
                                               int64_t* voxel_slot, int32_t* voxel_offsets, int32_t* point_idx, int32_t* argmax,
                                               int32_t* counts_dev) {
  CHECK_ARG(c, c && channels >= 0);
  if (!c->handoff || c->handoff_epoch != c->arena_epoch)
    return sstb_fail(c, SSTB_ERR_ARG, "roiaware_pool3d_forward: no sstb200_roiaware_pool3d_plan directly before it on this context");
  const RoiAwarePlan p = *std::static_pointer_cast<RoiAwarePlan>(c->handoff);
  c->handoff.reset();
  if (mode != SSTB200_POOL3D_MAX && mode != SSTB200_POOL3D_AVG)
    return sstb_fail(c, SSTB_ERR_ARG, "roiaware_pool3d_forward: mode %d is neither max (0) nor avg (1)", mode);
  CHECK_ARG(c, voxel_slot && voxel_offsets && point_idx && counts_dev && (mode != SSTB200_POOL3D_MAX || argmax));
  CHECK_ARG(c, p.N == 0 || channels == 0 || pts_feature);
  CHECK_ARG(c, (long long)p.R * channels == 0 || pooled);
  const long long P = p.P, nvox = (long long)p.v.ox * p.v.oy * p.v.oz, S = (long long)p.R * nvox;
  const int C = channels;
  cudaStream_t st = c->stream;
  const int end_bit = max(1, bits_for(p.R) + p.v.vbits + p.v.pbits);
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)P, 0, end_bit,
                                 st);
  const size_t Pc = (size_t)P + 1;
  unsigned long long *keys, *skeys;
  uint32_t *head, *gid, *gstart, *kcnt;
  ScanTemps s1, s2;
  size_t zero_bytes;
  void* cub_tmp;
  // carved after the plan's pieces, which this call still reads
  int rc = arena_carve(c, [&](Carve& cv) {
    keys = cv.take<unsigned long long>(Pc);
    skeys = cv.take<unsigned long long>(Pc);
    head = cv.take<uint32_t>(Pc + 1);
    gid = cv.take<uint32_t>(Pc + 1);
    gstart = cv.take<uint32_t>(Pc + 1);
    kcnt = cv.take<uint32_t>(Pc + 1);
    const size_t z = cv.mark();
    scan_carve(cv, s1, Pc);
    scan_carve(cv, s2, Pc);
    zero_bytes = cv.off - z;
    cub_tmp = cv.take<uint8_t>(cub_bytes + 16);
  });
  if (rc) return rc;
  CUDA_TRY(c, cudaMemsetAsync(s1.ticket, 0, zero_bytes, st));
  const int nb = (int)((P + 255) / 256);
  if (P > 0) {
    launch_pdl(ra_emit_kernel, dim3(p.R), dim3(RP_THREADS), (size_t)0, st, p.rois, p.rois_batch, p.g, p.binned, p.off, p.v, keys);
    cudaError_t ce = cub::DeviceRadixSort::SortKeys(cub_tmp, cub_bytes, (const unsigned long long*)keys, skeys, (int)P, 0, end_bit, st);
    if (ce != cudaSuccess) return sstb_fail(c, SSTB_ERR_CUDA, "cub radix sort: %s", cudaGetErrorString(ce));
    launch_pdl(ra_head_kernel, dim3(nb), dim3(256), (size_t)0, st, (const unsigned long long*)skeys, P, p.v.pbits, head);
  }
  // groups (occupied voxels) V = gid[P]; kept points K = voxel_offsets[V]
  launch_exclusive_scan(st, LoadU32{head}, (size_t)P, nullptr, s1, gid, s1.ticket + 1, true);
  launch_pdl(ra_group_kernel, dim3(nb > 0 ? nb : 1), dim3(256), (size_t)0, st, (const unsigned long long*)skeys, P, (const uint32_t*)head,
             (const uint32_t*)gid, p.v.vbits, p.v.pbits, nvox, gstart, voxel_slot);
  if (P > 0)
    launch_pdl(ra_kept_count_kernel, dim3(nb), dim3(256), (size_t)0, st, (const uint32_t*)gstart, (const uint32_t*)(s1.ticket + 1), P,
               p.keep, kcnt);
  launch_exclusive_scan(st, LoadU32{kcnt}, (size_t)P, (const int32_t*)(s1.ticket + 1), s2, (uint32_t*)voxel_offsets, s2.ticket + 1, true);
  if (P > 0)
    launch_pdl(ra_fill_kernel, dim3(nb), dim3(256), (size_t)0, st, (const unsigned long long*)skeys, P, p.v.pbits, (const uint32_t*)gid,
               (const uint32_t*)gstart, (const int32_t*)voxel_offsets, p.keep, point_idx);
  CUDA_TRY(c, cudaMemcpyAsync(counts_dev, s1.ticket + 1, 4, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(c, cudaMemcpyAsync(counts_dev + 1, s2.ticket + 1, 4, cudaMemcpyDeviceToDevice, st));
  if (S > 0 && C > 0) {
    const long long blocks = ((S + 31) / 32 * 32 + 255) / 256;
    if (mode == SSTB200_POOL3D_MAX)
      launch_pdl(ra_pool_kernel<true>, dim3((unsigned)blocks), dim3(256), (size_t)0, st, pts_feature, C, S, (const int64_t*)voxel_slot,
                 (const int32_t*)voxel_offsets, (const int32_t*)point_idx, (const int32_t*)counts_dev, pooled, argmax);
    else
      launch_pdl(ra_pool_kernel<false>, dim3((unsigned)blocks), dim3(256), (size_t)0, st, pts_feature, C, S, (const int64_t*)voxel_slot,
                 (const int32_t*)voxel_offsets, (const int32_t*)point_idx, (const int32_t*)counts_dev, pooled, argmax);
  }
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

extern "C" int sstb200_roiaware_pool3d_backward(sstb200_ctx* c, int num_pts, int channels, int mode, int64_t num_pairs,
                                                const int64_t* voxel_slot, const int32_t* voxel_offsets, const int32_t* point_idx,
                                                const int32_t* argmax, const int32_t* counts_dev, const float* grad_out, float* grad_in) {
  CHECK_ARG(c, c && num_pts >= 0 && channels >= 0 && num_pairs >= 0 && num_pairs <= 0x7fffffffll);
  if (mode != SSTB200_POOL3D_MAX && mode != SSTB200_POOL3D_AVG)
    return sstb_fail(c, SSTB_ERR_ARG, "roiaware_pool3d_backward: mode %d is neither max (0) nor avg (1)", mode);
  const int N = num_pts, C = channels;
  const long long P = num_pairs;
  if ((long long)N * C == 0) return SSTB_OK;
  CHECK_ARG(c, grad_in && voxel_slot && voxel_offsets && point_idx && counts_dev && (mode != SSTB200_POOL3D_MAX || argmax));
  CHECK_ARG(c, P == 0 || grad_out);
  cudaStream_t st = c->stream;
  const int end_bit = max(1, bits_for((long long)N + 1));
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (int)P, 0, end_bit, st);
  arena_reset(c);
  const size_t Pc = (size_t)P + 1;
  uint32_t *pkey, *pgrp, *skey, *sgrp;
  void* cub_tmp;
  int rc = arena_carve(c, [&](Carve& cv) {
    pkey = cv.take<uint32_t>(Pc);
    pgrp = cv.take<uint32_t>(Pc);
    skey = cv.take<uint32_t>(Pc);
    sgrp = cv.take<uint32_t>(Pc);
    cub_tmp = cv.take<uint8_t>(cub_bytes + 16);
  });
  if (rc) return rc;
  if (P > 0) {
    launch_pdl(ra_inverse_kernel, dim3((unsigned)((P + 255) / 256)), dim3(256), (size_t)0, st, voxel_offsets, point_idx, counts_dev, P, N,
               pkey, pgrp);
    cudaError_t ce = cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, (const uint32_t*)pkey, skey, (const uint32_t*)pgrp, sgrp, (int)P, 0,
                                                     end_bit, st);
    if (ce != cudaSuccess) return sstb_fail(c, SSTB_ERR_CUDA, "cub radix sort: %s", cudaGetErrorString(ce));
  }
  const unsigned blocks = (unsigned)(((long long)N * C + 255) / 256);
  if (mode == SSTB200_POOL3D_MAX)
    launch_pdl(ra_grad_kernel<true>, dim3(blocks), dim3(256), (size_t)0, st, (const uint32_t*)skey, (const uint32_t*)sgrp, P, N, C, voxel_slot,
               voxel_offsets, argmax, grad_out, grad_in);
  else
    launch_pdl(ra_grad_kernel<false>, dim3(blocks), dim3(256), (size_t)0, st, (const uint32_t*)skey, (const uint32_t*)sgrp, P, N, C, voxel_slot,
               voxel_offsets, argmax, grad_out, grad_in);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
