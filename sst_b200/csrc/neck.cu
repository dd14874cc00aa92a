// Voxel2PointScatterNeck.forward (mmdet3d/models/necks/voxel2point_neck.py:28-62; SURVEY 8f next-2): voxel features back to
// the points (FSD's step between the SST/sparse backbone and the point-wise heads).
//   pts_feats = voxel_feats[voxel2point_inds];  pts_mask = ~(pts_feats == padding).all(1)      (dropped voxels are padded rows)
//   results   = [pts_feats[mask] || points[mask,:3] - ((coors[mask,[3,2,1]] + 0.5) * voxel_size + pc_min) (/ (voxel_size/2))]
// The reference materialises the [N,C] gather, the mask, three filtered copies and a concat; here: one warp-per-point mask
// pass, a look-back scan over the keep flags (order-preserving compaction) and one warp-per-point write pass.
#include <stdarg.h>
#include "common.cuh"
#include "index.cuh"

__global__ void __launch_bounds__(256) v2p_mask_kernel(const float* __restrict__ voxel_feats, int C, const long long* __restrict__ inds, int N,
                                                       int M, float padding, uint32_t* __restrict__ keep, uint8_t* __restrict__ mask_out,
                                                       int32_t* __restrict__ err) {
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= N) return;
  const long long v = inds[i];
  if (v < 0 || v >= M) {
    if (lane == 0) {
      *err = 1;
      keep[i] = 0;
      mask_out[i] = 0;
    }
    return;
  }
  const float* row = voxel_feats + (size_t)v * C;
  bool all_pad = true;
  for (int c = lane; c < C; c += 32) all_pad &= (row[c] == padding);
  all_pad = __all_sync(0xffffffffu, all_pad);
  if (lane == 0) {
    keep[i] = all_pad ? 0u : 1u;
    mask_out[i] = all_pad ? 0 : 1;
  }
}

__global__ void __launch_bounds__(256) v2p_write_kernel(const float* __restrict__ points, int Cp, const long long* __restrict__ coors,
                                                        const float* __restrict__ voxel_feats, int C, const long long* __restrict__ inds, int N,
                                                        const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pos, float vx, float vy,
                                                        float vz, float x0, float y0, float z0, int with_xyz, int normalize,
                                                        float* __restrict__ out) {
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= N || !keep[i]) return;
  const int Co = C + (with_xyz ? 3 : 0);
  const float* row = voxel_feats + (size_t)inds[i] * C;
  float* o = out + (size_t)pos[i] * Co;
  for (int c = lane; c < C; c += 32) o[c] = row[c];
  if (with_xyz && lane < 3) {
    // x y z order: coors are (b, z, y, x); two roundings for (c + 0.5) * vs + min like the torch expression
    const float vs = lane == 0 ? vx : (lane == 1 ? vy : vz);
    const float mn = lane == 0 ? x0 : (lane == 1 ? y0 : z0);
    const float cc = (float)coors[(size_t)i * 4 + (3 - lane)];
    const float center = __fadd_rn(__fmul_rn(__fadd_rn(cc, 0.5f), vs), mn);
    float l = points[(size_t)i * Cp + lane] - center;
    if (normalize) l = __fdiv_rn(l, __fdiv_rn(vs, 2.0f));
    o[C + lane] = l;
  }
}

extern "C" int sstb200_voxel2point(sstb200_ctx* c, const float* points, int Cp, const int64_t* pts_coors, const float* voxel_feats, int M,
                                   int C, const int64_t* voxel2point_inds, int N, float padding, const float voxel_size[3],
                                   const float pc_min[3], int with_xyz, int normalize_local_xyz, float* out, uint8_t* mask_out,
                                   int32_t* num_out_dev, int32_t* num_out_host) {
  CHECK_ARG(c, c && N >= 0 && M >= 0 && C >= 1 && Cp >= 3 && num_out_dev);
  if (N == 0) {
    CUDA_TRY(c, cudaMemsetAsync(num_out_dev, 0, 4, c->stream));
    if (num_out_host) *num_out_host = 0;
    return SSTB_OK;
  }
  CHECK_ARG(c, points && pts_coors && voxel_feats && voxel2point_inds && out && mask_out && voxel_size && pc_min);
  arena_reset(c);
  uint32_t *keep, *pos;
  ScanTemps st;
  size_t st_bytes;
  int rc = arena_carve(c, [&](Carve& cv) {
    keep = cv.take<uint32_t>((size_t)N + 2);
    pos = cv.take<uint32_t>((size_t)N + 2);
    const size_t z = cv.mark();
    scan_carve(cv, st, N);
    st_bytes = cv.off - z;
  });
  if (rc) return rc;
  CUDA_TRY(c, cudaMemsetAsync(st.ticket, 0, st_bytes, c->stream));
  int32_t* err = (int32_t*)(st.ticket + 2);
  const unsigned blocks = (unsigned)(((size_t)N * 32 + 255) / 256);
  launch_pdl(v2p_mask_kernel, dim3(blocks), dim3(256), (size_t)0, c->stream, voxel_feats, C, (const long long*)voxel2point_inds, N, M, padding, keep,
             mask_out, err);
  launch_exclusive_scan(c->stream, LoadU32{keep}, (size_t)N, nullptr, st, pos, st.ticket + 1, true);
  launch_pdl(v2p_write_kernel, dim3(blocks), dim3(256), (size_t)0, c->stream, points, Cp, (const long long*)pts_coors, voxel_feats, C,
             (const long long*)voxel2point_inds, N, (const uint32_t*)keep, (const uint32_t*)pos, voxel_size[0], voxel_size[1], voxel_size[2], pc_min[0],
             pc_min[1], pc_min[2], with_xyz, normalize_local_xyz, out);
  LAUNCH_CHECK(c);
  CUDA_TRY(c, cudaMemcpyAsync(num_out_dev, st.ticket + 1, 4, cudaMemcpyDeviceToDevice, c->stream));
  CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, st.ticket + 1, 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32 + 1, err, 4, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (c->pinned_i32[1]) return sstb_fail(c, SSTB_ERR_ARG, "voxel2point: voxel2point_inds out of range [0, %d)", M);
  if (num_out_host) *num_out_host = c->pinned_i32[0];
  return SSTB_OK;
}

// ---- backward: grad_voxel[v] = sum of grad_out[pos(p), 0:C] over the kept points p with inds[p] == v ------------------------------
// The kept points' voxel ids are compacted to their output rows (the forward's scan over the mask), grouped into a CSR and summed
// by the shared segmented reduce, reading grad_out with its row pitch C(+3).  Its fp64 accumulation makes the sum independent of
// the CSR order, so the result is deterministic without float atomics; voxels no kept point references get 0.
struct LoadMaskU8 {
  const uint8_t* p;
  __device__ __forceinline__ uint32_t operator()(size_t i) const { return p[i] ? 1u : 0u; }
  __device__ __forceinline__ void load8(size_t base, size_t n, uint32_t* v) const {
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = (base + i < n && p[base + i]) ? 1u : 0u;
  }
};

__global__ void __launch_bounds__(256) v2p_compact_kernel(const uint8_t* __restrict__ mask, const uint32_t* __restrict__ pos,
                                                          const long long* __restrict__ inds, int N, int K, int M,
                                                          long long* __restrict__ row_voxel) {
  pdl_wait();
  pdl_launch();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N || !mask[i]) return;
  const uint32_t r = pos[i];
  if (r >= (uint32_t)K) return;  // a mask with more kept points than grad_out has rows: never write past K
  const long long v = inds[i];
  row_voxel[r] = (v >= 0 && v < M) ? v : -1;  // -1: not counted, not grouped (csr_fill skips it)
}

extern "C" int sstb200_voxel2point_backward(sstb200_ctx* c, const float* grad_out, const uint8_t* mask, const int64_t* voxel2point_inds,
                                            int N, int K, int M, int C, int with_xyz, float* grad_voxel) {
  CHECK_ARG(c, c && N >= 0 && K >= 0 && K <= N && M >= 0 && C >= 1);
  if (M == 0) return SSTB_OK;
  CHECK_ARG(c, grad_voxel);
  if (K == 0) {
    CUDA_TRY(c, cudaMemsetAsync(grad_voxel, 0, (size_t)M * C * 4, c->stream));
    return SSTB_OK;
  }
  CHECK_ARG(c, grad_out && mask && voxel2point_inds);
  const int ld = C + (with_xyz ? 3 : 0);
  arena_reset(c);
  uint32_t* pos;
  ScanTemps st;
  size_t st_bytes;
  long long* row_voxel;
  int32_t* count;
  Csr r;
  int rc = arena_carve(c, [&](Carve& cv) {
    pos = cv.take<uint32_t>((size_t)N + 2);
    const size_t z = cv.mark();
    scan_carve(cv, st, N);
    st_bytes = cv.off - z;
    row_voxel = cv.take<long long>(K);
    count = cv.take<int32_t>((size_t)M + 1);
    csr_carve(cv, r, K, M);
  });
  if (rc) return rc;
  int32_t* err = (int32_t*)(st.ticket + 2);  // count_index_kernel's flag for -1 rows; nothing reads it
  CUDA_TRY(c, cudaMemsetAsync(st.ticket, 0, st_bytes, c->stream));
  CUDA_TRY(c, cudaMemsetAsync(row_voxel, 0xFF, (size_t)K * 8, c->stream));
  CUDA_TRY(c, cudaMemsetAsync(count, 0, (size_t)M * 4, c->stream));
  launch_exclusive_scan(c->stream, LoadMaskU8{mask}, (size_t)N, nullptr, st, pos, st.ticket + 1, true);
  launch_pdl(v2p_compact_kernel, dim3((N + 255) / 256), dim3(256), (size_t)0, c->stream, mask, (const uint32_t*)pos,
             (const long long*)voxel2point_inds, N, K, M, row_voxel);
  launch_pdl(count_index_kernel, dim3((K + 255) / 256), dim3(256), (size_t)0, c->stream, (const long long*)row_voxel, K, M, count, err);
  rc = csr_build(c, r, (const long long*)row_voxel, K, count, (size_t)M, nullptr);
  if (rc) return rc;
  launch_segment_reduce(c, grad_out, C, r.offsets, r.order, M, nullptr, SSTB200_REDUCE_SUM, 0.f, grad_voxel, nullptr, K, ld);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}
