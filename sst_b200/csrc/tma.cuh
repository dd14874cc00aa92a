// TMA (cp.async.bulk.tensor) + mbarrier helpers: host-side tensor-map encoding and the device-side PTX wrappers.
//   SASS evidence: cp.async.bulk.tensor loads -> UTMALDG, stores -> UTMASTG, expect_tx -> SYNCS.ARRIVE.TRANS64.
// Every tile that crosses the HBM/L2 <-> shared-memory boundary of the tensor-core kernels is one of these bulk copies,
// landing in (or leaving from) the 128-byte-swizzled layout the wgmma descriptors read, so no thread spends
// instructions on address arithmetic for operand staging.
#pragma once
#include <cuda.h>
#include "wgmma.cuh"

namespace {

// 2-D row-major tensor [rows, inner] of `elem_bytes` elements, row pitch `pitch_bytes`; box = [box_rows, box_inner] with
// box_inner * elem_bytes == 128 (one SWIZZLE_128B span).  Out-of-bounds rows are zero-filled on load, clipped on store.
static inline int tmap_2d_sw128(CUtensorMap* m, CUtensorMapDataType dt, int elem_bytes, const void* base, uint64_t inner,
                                uint64_t rows, uint64_t pitch_bytes, uint32_t box_inner, uint32_t box_rows) {
  cuuint64_t gdim[2] = {inner, rows};
  cuuint64_t gstr[1] = {pitch_bytes};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  if ((uint64_t)box_inner * elem_bytes != 128 || ((uintptr_t)base & 15) || (pitch_bytes & 15)) return -1;
  // resolved through the runtime (no link-time dependency on libcuda: the library must load on a box without a driver)
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || !fn) return -2;
    encode = (EncodeFn)fn;
  }
  CUresult r = encode(m, dt, 2, const_cast<void*>(base), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(int)r - 1000;
}

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// global -> shared tile load; completion is signalled on `mbar` as transaction bytes
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const CUtensorMap* m, int c_inner, int c_row, uint32_t mbar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n" ::"r"(smem_dst),
               "l"(reinterpret_cast<uint64_t>(m)), "r"(mbar), "r"(c_inner), "r"(c_row)
               : "memory");
}
// shared -> global tile store (bulk async group of the issuing thread)
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, int c_inner, int c_row, uint32_t smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(smem_src), "r"(c_inner), "r"(c_row)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory");
}

__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t mbar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(mbar) : "memory");
}
// named barrier over a subset of the CTA's warps (id 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory"); }

}  // namespace
