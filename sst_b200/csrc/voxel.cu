// Voxel-id ranking, DynamicScatter (fwd/bwd), unique rows, segmented reduce, in-group ranks.
//
// Design note (voxel index): instead of the reference's row sort
// (at::unique_dim, scatter_points_cuda.cu:202-205) every "unique rows, sorted" on this path is a
// *bitmap rank*: rows are linearised into a bounded grid, the grid's occupancy bitmap is built with one
// atomicOr per row, a popcount prefix-scan over the bitmap words gives every occupied cell its rank in
// lexicographic order, and rank(row) is one popc.  For the Waymo pillar grid the bitmap is 27 KB/frame and
// lives in L2; no sort, no float atomics, deterministic.  Points are then grouped per voxel by a counting
// sort (CSR) and reduced by one warp (or sub-warp) per voxel with coalesced loads.
#include <stdarg.h>
#include "common.cuh"

#include "index.cuh"

// ------------------------------------------------------------------------------------------------
// V1 dynamic_voxelize
// ------------------------------------------------------------------------------------------------
__global__ void dynamic_voxelize_kernel(const float* __restrict__ points, int P, int F, float vx, float vy, float vz,
                                        float x0, float y0, float z0, int gx, int gy, int gz, int32_t* __restrict__ coors) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const float* p = points + (size_t)i * F;
  // IEEE division + floor, exactly like voxelization_cuda.cu:38,46,54 (no fast-math anywhere in this build)
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

// FSDv2 virtual-voxel coordinates (single_stage_fsd_v2.py:108-123): coors = [batch, floor_div(p - lo, vs) in z,y,x order], NO clamp
// (the detector clips the predicted centres beforehand).  torch.div(rounding_mode='floor') on floats is c10::div_floor_floating
// (fmod-based, with a half-way correction), restated here so that the coordinates are bit-identical to the reference's.
__device__ __forceinline__ float div_floor_f32(float a, float b) {
  if (b == 0.f) return __fdiv_rn(a, b);
  const float mod = fmodf(a, b);
  float div = __fdiv_rn(a - mod, b);
  if (mod != 0.f && (b < 0.f) != (mod < 0.f)) div -= 1.0f;
  if (div != 0.f) {
    float fl = floorf(div);
    if (div - fl > 0.5f) fl += 1.0f;
    return fl;
  }
  return copysignf(0.f, __fdiv_rn(a, b));
}
__global__ void voxelize_batch_idx_kernel(const float* __restrict__ points, int n, int ldp, const long long* __restrict__ batch_idx,
                                          float vx, float vy, float vz, float x0, float y0, float z0, long long* __restrict__ coors) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = points + (size_t)i * ldp;
  longlong2 a, b;
  a.x = batch_idx[i];
  a.y = (long long)div_floor_f32(p[2] - z0, vz);
  b.x = (long long)div_floor_f32(p[1] - y0, vy);
  b.y = (long long)div_floor_f32(p[0] - x0, vx);
  reinterpret_cast<longlong2*>(coors)[2 * (size_t)i] = a;
  reinterpret_cast<longlong2*>(coors)[2 * (size_t)i + 1] = b;
}
extern "C" int sstb200_voxelize_with_batch_idx(sstb200_ctx* c, const float* points, int n, int ldp, const int64_t* batch_idx,
                                               const float voxel_size[3], const float range_lo[3], int64_t* coors) {
  CHECK_ARG(c, c && n >= 0 && ldp >= 3 && voxel_size && range_lo);
  if (n == 0) return SSTB_OK;
  CHECK_ARG(c, points && batch_idx && coors && ((uintptr_t)coors & 15) == 0);
  launch_pdl(voxelize_batch_idx_kernel, dim3((n + 255) / 256), dim3(256), (size_t)0, c->stream, points, n, ldp, (const long long*)batch_idx,
             voxel_size[0], voxel_size[1], voxel_size[2], range_lo[0], range_lo[1], range_lo[2], (long long*)coors);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

void sstb_grid_size(const float vs[3], const float r[6], int g[3]) {
  // ceil((max-min)/vs) in float32, voxelization_cuda.cu:355-357
  for (int i = 0; i < 3; i++) g[i] = (int)ceilf((r[3 + i] - r[i]) / vs[i]);
}

extern "C" int sstb200_dynamic_voxelize(sstb200_ctx* c, const float* points, int P, int F, const float vs[3],
                                        const float r[6], int32_t* coors) {
  CHECK_ARG(c, c && P >= 0 && F >= 3 && vs && r && (P == 0 || (points && coors)));
  if (P == 0) return SSTB_OK;
  int g[3];
  sstb_grid_size(vs, r, g);
  launch_pdl(dynamic_voxelize_kernel, dim3((P + 255) / 256), dim3(256), (size_t)(0), c->stream, points, P, F, vs[0], vs[1], vs[2], r[0], r[1], r[2],
                                                                   g[0], g[1], g[2], coors);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}


// ------------------------------------------------------------------------------------------------
// V1 batched / sync-free
// ------------------------------------------------------------------------------------------------
__global__ void voxelize_frames_kernel(const float* __restrict__ points, int cap, int F, const int32_t* __restrict__ offs, int B,
                                       float vx, float vy, float vz, float x0, float y0, float z0, int gx, int gy, int gz,
                                       int32_t* __restrict__ coors4) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cap) return;
  int4 o = make_int4(-1, -1, -1, -1);
  if (i < offs[B]) {
    int b = 0;
    while (b + 1 < B && i >= offs[b + 1]) b++;
    const float* p = points + (size_t)i * F;
    int cx = (int)floorf(__fdiv_rn(p[0] - x0, vx));
    int cy = (int)floorf(__fdiv_rn(p[1] - y0, vy));
    int cz = (int)floorf(__fdiv_rn(p[2] - z0, vz));
    cx = cx < 0 ? 0 : (cx >= gx ? gx - 1 : cx);
    cy = cy < 0 ? 0 : (cy >= gy ? gy - 1 : cy);
    cz = cz < 0 ? 0 : (cz >= gz ? gz - 1 : cz);
    o = make_int4(b, cz, cy, cx);
  }
  *(int4*)&coors4[(size_t)i * 4] = o;
}

extern "C" int sstb200_voxelize_frames(sstb200_ctx* c, const float* points, int cap, int F, const int32_t* offs, int B,
                                       const float vs[3], const float r[6], int32_t* coors4) {
  CHECK_ARG(c, c && cap >= 0 && F >= 3 && B >= 1 && offs && vs && r);
  if (cap == 0) return SSTB_OK;
  CHECK_ARG(c, points && coors4);
  int g[3];
  sstb_grid_size(vs, r, g);
  launch_pdl(voxelize_frames_kernel, dim3((cap + 255) / 256), dim3(256), (size_t)(0), c->stream, points, cap, F, offs, B, vs[0], vs[1], vs[2], r[0], r[1], r[2],
                                                                    g[0], g[1], g[2], coors4);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// V2 dynamic_point_to_voxel_forward
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_dynamic_point_to_voxel_forward(sstb200_ctx* c, const float* feats, const int32_t* coors, int P,
                                                      int C, int reduce_type, const int32_t lo3[3], const int32_t hi3[3],
                                                      float* reduced, int32_t* out_coors, int32_t* coors_map,
                                                      int32_t* reduce_count, int32_t* num_dev, int32_t* num_host) {
  CHECK_ARG(c, c && P >= 0 && C >= 1 && reduce_type >= 0 && reduce_type <= 2 && num_dev);
  if (P == 0) {
    CUDA_TRY(c, cudaMemsetAsync(num_dev, 0, 4, c->stream));
    if (num_host) *num_host = 0;
    return SSTB_OK;
  }
  CHECK_ARG(c, feats && coors && lo3 && hi3 && reduced && out_coors && coors_map && reduce_count);
  Extents e;
  long long T;
  long long lo[3], hi[3];
  for (int d = 0; d < 3; d++) {
    lo[d] = lo3[d] < 0 ? 0 : lo3[d];  // negatives are invalid rows, never part of the grid
    hi[d] = hi3[d] < lo[d] ? lo[d] : hi3[d];
  }
  int rc = make_extents(c, e, 3, lo, hi, &T);
  if (rc) return rc;
  arena_reset(c);
  KeyIndex k;
  Csr r;
  rc = arena_carve(c, [&](Carve& cv) {
    key_index_carve(cv, k, P, T);
    csr_carve(cv, r, P, P);
  });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k))) return rc;
  CUDA_TRY(c, cudaMemsetAsync(reduce_count, 0, (size_t)P * 4, c->stream));
  int nb = (P + 255) / 256;
  launch_mark_rows<int32_t>(c, coors, P, e, true, k, nullptr);
  key_index_scan(c, k);
  launch_emit_rows<int32_t>(c, k, e, 1, out_coors, num_dev);
  launch_pdl(map_count_kernel<int32_t>, dim3(nb), dim3(256), (size_t)(0), c->stream, k.keys, P, k.bitmap, k.word_prefix, 1, k.flags, coors_map, reduce_count, nullptr);
  LAUNCH_CHECK(c);
  rc = csr_build<int32_t>(c, r, coors_map, P, reduce_count, P, num_dev);
  if (rc) return rc;
  launch_segment_reduce(c, feats, C, r.offsets, r.order, P, num_dev, reduce_type,
                        reduce_type == SSTB200_REDUCE_MAX ? -INFINITY : 0.f, reduced, nullptr, P);
  LAUNCH_CHECK(c);
  if (num_host) {
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, num_dev, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32 + 1, k.flags + 1, 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    *num_host = c->pinned_i32[0];
    if (c->pinned_i32[1]) return sstb_fail(c, SSTB_ERR_ARG, "dynamic_point_to_voxel_forward: a non-negative row lies outside coor_lo/hi");
  }
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// V3 backward
// ------------------------------------------------------------------------------------------------
__global__ void dp2v_bwd_add_kernel(float* __restrict__ g, const float* __restrict__ gr, const int32_t* __restrict__ map,
                                    const int32_t* __restrict__ cnt, int P, int C, int mean) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)P * C) return;
  int p = (int)(i / C), ch = (int)(i % C);
  int v = map[p];
  float o = 0.f;
  if (v >= 0) {
    o = gr[(size_t)v * C + ch];
    if (mean) o = o / (float)cnt[v];
  }
  g[i] = o;
}
// max: gradient goes to the LOWEST point index attaining the max (scatter_points_cuda.cu:150-152)
__global__ void dp2v_bwd_argmin_kernel(const float* __restrict__ feats, const float* __restrict__ red,
                                       const int32_t* __restrict__ map, int P, int C, int32_t* __restrict__ from) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)P * C) return;
  int p = (int)(i / C), ch = (int)(i % C);
  int v = map[p];
  if (v < 0) return;
  if (feats[i] == red[(size_t)v * C + ch]) atomicMin(&from[(size_t)v * C + ch], p);
}
__global__ void dp2v_bwd_scatter_kernel(float* __restrict__ g, const float* __restrict__ gr,
                                        const int32_t* __restrict__ from, int M, int C, int P) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * C) return;
  int ch = (int)(i % C);
  int p = from[i];
  if (p < P) g[(size_t)p * C + ch] = gr[i];
}
__global__ void fill_i32_kernel(int32_t* p, size_t n, int32_t v) {
  pdl_wait();
  pdl_launch();
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

extern "C" int sstb200_dynamic_point_to_voxel_backward(sstb200_ctx* c, float* grad_feats, const float* grad_reduced,
                                                       const float* feats, const float* reduced,
                                                       const int32_t* coors_map, const int32_t* reduce_count, int P,
                                                       int M, int C, int reduce_type) {
  CHECK_ARG(c, c && P >= 0 && M >= 0 && C >= 1 && reduce_type >= 0 && reduce_type <= 2);
  if (P == 0) return SSTB_OK;
  CHECK_ARG(c, grad_feats);
  size_t n = (size_t)P * C;
  if (M == 0) {
    CUDA_TRY(c, cudaMemsetAsync(grad_feats, 0, n * 4, c->stream));
    return SSTB_OK;
  }
  CHECK_ARG(c, grad_reduced && feats && reduced && coors_map && reduce_count);
  unsigned nb = (unsigned)((n + 255) / 256);
  if (reduce_type != SSTB200_REDUCE_MAX) {
    launch_pdl(dp2v_bwd_add_kernel, dim3(nb), dim3(256), (size_t)(0), c->stream, grad_feats, grad_reduced, coors_map, reduce_count, P, C,
                                                   reduce_type == SSTB200_REDUCE_MEAN);
  } else {
    arena_reset(c);
    int32_t* from;
    int rc = arena_carve(c, [&](Carve& cv) { from = cv.take<int32_t>((size_t)M * C); });
    if (rc) return rc;
    size_t m = (size_t)M * C;
    unsigned mb = (unsigned)((m + 255) / 256);
    launch_pdl(fill_i32_kernel, dim3(mb), dim3(256), (size_t)(0), c->stream, from, m, P);
    CUDA_TRY(c, cudaMemsetAsync(grad_feats, 0, n * 4, c->stream));
    launch_pdl(dp2v_bwd_argmin_kernel, dim3(nb), dim3(256), (size_t)(0), c->stream, feats, reduced, coors_map, P, C, from);
    launch_pdl(dp2v_bwd_scatter_kernel, dim3(mb), dim3(256), (size_t)(0), c->stream, grad_feats, grad_reduced, from, M, C, P);
  }
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// V5a unique rows (int64)
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_unique_rows_i64(sstb200_ctx* c, const int64_t* coors, int P, int ndim, const int64_t* lo,
                                       const int64_t* hi, int64_t* new_coors, int64_t* inverse, int32_t* counts,
                                       int32_t* num_dev, int32_t* num_host) {
  CHECK_ARG(c, c && P >= 0 && ndim >= 1 && ndim <= 4 && num_dev);
  if (P == 0) {
    CUDA_TRY(c, cudaMemsetAsync(num_dev, 0, 4, c->stream));
    if (num_host) *num_host = 0;
    return SSTB_OK;
  }
  CHECK_ARG(c, coors && lo && hi && new_coors && inverse);
  Extents e;
  long long T;
  int rc = make_extents(c, e, ndim, (const long long*)lo, (const long long*)hi, &T);
  if (rc) return rc;
  arena_reset(c);
  KeyIndex k;
  rc = arena_carve(c, [&](Carve& cv) { key_index_carve(cv, k, P, T); });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k))) return rc;
  if (counts) CUDA_TRY(c, cudaMemsetAsync(counts, 0, (size_t)P * 4, c->stream));
  int nb = (P + 255) / 256;
  launch_mark_rows<long long>(c, (const long long*)coors, P, e, false, k, nullptr);
  key_index_scan(c, k);
  launch_emit_rows<long long>(c, k, e, 0, (long long*)new_coors, num_dev);
  launch_pdl(map_count_kernel<long long>, dim3(nb), dim3(256), (size_t)(0), c->stream, k.keys, P, k.bitmap, k.word_prefix, 0, k.flags,
                                                         (long long*)inverse, counts, nullptr);
  LAUNCH_CHECK(c);
  if (num_host) return read_back_i32(c, num_dev, num_host);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// V5b segment reduce by a given index
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_segment_reduce(sstb200_ctx* c, const float* src, const int64_t* index, int P, int C, int nseg,
                                      int reduce_type, float* out, int64_t* argmax) {
  CHECK_ARG(c, c && P >= 0 && C >= 1 && nseg >= 0 && reduce_type >= 0 && reduce_type <= 2);
  if (nseg == 0) return SSTB_OK;
  CHECK_ARG(c, out && (P == 0 || (src && index)));
  arena_reset(c);
  int32_t* count;
  Csr r;
  int rc = arena_carve(c, [&](Carve& cv) {
    count = cv.take<int32_t>((size_t)nseg + 2);
    csr_carve(cv, r, P, nseg);
  });
  if (rc) return rc;
  CUDA_TRY(c, cudaMemsetAsync(count, 0, ((size_t)nseg + 2) * 4, c->stream));
  if (P > 0) launch_pdl(count_index_kernel, dim3((P + 255) / 256), dim3(256), (size_t)(0), c->stream, (const long long*)index, P, nseg, count, count + nseg + 1);
  rc = csr_build<long long>(c, r, (const long long*)index, P, count, nseg, nullptr);
  if (rc) return rc;
  launch_segment_reduce(c, src, C, r.offsets, r.order, nseg, nullptr, reduce_type, 0.f, out, (long long*)argmax, P);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// B2 ingroup indices (stable rank inside the group)
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_ingroup_indices(sstb200_ctx* c, const int64_t* group, int N, int64_t max_id, int64_t* out) {
  CHECK_ARG(c, c && N >= 0 && max_id >= 0);
  if (N == 0) return SSTB_OK;
  CHECK_ARG(c, group && out);
  Extents e;
  long long T;
  long long lo = 0, hi = max_id;
  int rc = make_extents(c, e, 1, &lo, &hi, &T);
  if (rc) return rc;
  arena_reset(c);
  KeyIndex k;
  int32_t *cid, *count;
  Csr r;
  rc = arena_carve(c, [&](Carve& cv) {
    key_index_carve(cv, k, N, T);
    cid = cv.take<int32_t>(N);
    count = cv.take<int32_t>((size_t)N + 2);
    csr_carve(cv, r, N, N);
  });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k))) return rc;
  const int32_t* ng = (const int32_t*)k.total;  // #distinct groups, written by the bitmap scan
  CUDA_TRY(c, cudaMemsetAsync(count, 0, ((size_t)N + 2) * 4, c->stream));
  int nb = (N + 255) / 256;
  launch_mark_rows<long long>(c, (const long long*)group, N, e, false, k, nullptr);
  key_index_scan(c, k);
  launch_pdl(map_count_kernel<int32_t>, dim3(nb), dim3(256), (size_t)(0), c->stream, k.keys, N, k.bitmap, k.word_prefix, 0, k.flags, cid, count, nullptr);
  rc = csr_build<int32_t>(c, r, cid, N, count, N, ng);
  if (rc) return rc;
  launch_pdl(stable_rank_kernel, dim3(c->num_sms * 4), dim3(256), (size_t)(0), c->stream, r.offsets, r.order, ng, nullptr, (long long*)out, nullptr, nullptr);
  LAUNCH_CHECK(c);
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_version(void) { return 100; }

extern "C" sstb200_ctx* sstb200_create(int device) {
  if (cudaSetDevice(device) != cudaSuccess) return nullptr;
  sstb200_ctx* c = new sstb200_ctx();
  c->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->num_sms = prop.multiProcessorCount;
  if (cudaMallocHost((void**)&c->pinned_i32, 256) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_coords, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming) != cudaSuccess) {
    delete c;
    return nullptr;
  }
  return c;
}
extern "C" void sstb200_destroy(sstb200_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (c->arena) cudaFree(c->arena);
  for (void* p : c->retired) cudaFree(p);
  if (c->pinned_i32) cudaFreeHost(c->pinned_i32);
  if (c->ev_coords) cudaEventDestroy(c->ev_coords);
  if (c->ev_done) cudaEventDestroy(c->ev_done);
  delete c;
}
extern "C" int sstb200_set_stream(sstb200_ctx* c, void* s) {
  if (!c) return SSTB_ERR_ARG;
  c->stream = (cudaStream_t)s;
  return SSTB_OK;
}
extern "C" const char* sstb200_last_error(sstb200_ctx* c) { return c ? c->err.c_str() : "null context"; }
extern "C" int sstb200_num_sms(sstb200_ctx* c) { return c ? c->num_sms : 0; }

// ------------------------------------------------------------------------------------------------
// fork / join of a side branch (a second context = second stream + second arena).  The two window plans of a frame need only the
// voxel coordinates, which the VFE entry point produces in its first third: fork there, run the plans next to the VFE layers,
// join before the encoder stack.  Works on plain streams and inside a stream capture (the side stream joins the capture).
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_branch_fork(sstb200_ctx* c, sstb200_ctx* side) {
  CHECK_ARG(c, c && side && side != c && side->device == c->device && side->stream != c->stream);
  CUDA_TRY(c, cudaStreamWaitEvent(side->stream, c->ev_coords, 0));
  return SSTB_OK;
}
extern "C" int sstb200_branch_join(sstb200_ctx* c, sstb200_ctx* side) {
  CHECK_ARG(c, c && side && side != c && side->device == c->device);
  CUDA_TRY(c, cudaEventRecord(side->ev_done, side->stream));
  CUDA_TRY(c, cudaStreamWaitEvent(c->stream, side->ev_done, 0));
  return SSTB_OK;
}

// ------------------------------------------------------------------------------------------------
// CUDA graph helpers
// ------------------------------------------------------------------------------------------------
extern "C" int sstb200_graph_begin(sstb200_ctx* c) {
  CHECK_ARG(c, c);
  CUDA_TRY(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
  return SSTB_OK;
}
extern "C" int sstb200_graph_end(sstb200_ctx* c, void** exec_out, int32_t* nk, int32_t* no) {
  CHECK_ARG(c, c && exec_out);
  cudaGraph_t g = nullptr;
  CUDA_TRY(c, cudaStreamEndCapture(c->stream, &g));
  size_t n = 0;
  CUDA_TRY(c, cudaGraphGetNodes(g, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  if (n) CUDA_TRY(c, cudaGraphGetNodes(g, nodes.data(), &n));
  int kn = 0, on = 0;
  for (size_t i = 0; i < n; i++) {
    cudaGraphNodeType t;
    CUDA_TRY(c, cudaGraphNodeGetType(nodes[i], &t));
    if (t == cudaGraphNodeTypeKernel) kn++;
    else on++;
  }
  if (nk) *nk = kn;
  if (no) *no = on;
  cudaGraphExec_t ex = nullptr;
  CUDA_TRY(c, cudaGraphInstantiate(&ex, g, 0));
  CUDA_TRY(c, cudaGraphDestroy(g));
  *exec_out = (void*)ex;
  return SSTB_OK;
}
extern "C" int sstb200_graph_launch(sstb200_ctx* c, void* ex) {
  CHECK_ARG(c, c && ex);
  CUDA_TRY(c, cudaGraphLaunch((cudaGraphExec_t)ex, c->stream));
  return SSTB_OK;
}
extern "C" int sstb200_graph_destroy(sstb200_ctx* c, void* ex) {
  CHECK_ARG(c, c);
  if (ex) CUDA_TRY(c, cudaGraphExecDestroy((cudaGraphExec_t)ex));
  return SSTB_OK;
}
