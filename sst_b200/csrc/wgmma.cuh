// Hopper tensor-core helpers (inline PTX) shared by the tensor-core kernels: the shared-memory operand format and its staging,
// wgmma descriptors and instructions, the accumulator-fragment layout, a shared-memory accumulator tile for thread-per-row
// epilogues, and mbarrier waits.
//   A 128-row tile is computed by two warpgroups (rows 0-63 and 64-127), each issuing wgmma.mma_async m64nNk16 with both
//   operands read from shared memory.  Accumulators live in registers (fp32).
//
// Operand format: K-major, 128-byte swizzled (SWIZZLE_128B), 16-bit elements.  Every kernel writes its operands in this one format
// (threads through sw128_off, TMA loads through CU_TENSOR_MAP_SWIZZLE_128B) and wg_desc_sw128 reads it.  An operand of `rows`
// rows is one block of rows x 128 B per 64-wide K chunk, 1024-B aligned.  A row of a block holds its 64 elements as eight 16-byte
// pieces; piece jj (K = 8 jj .. 8 jj + 7 of the chunk) of row r is stored at position jj ^ (r & 7) of the row, so in each 8-row
// atom of 1024 B the rows' copies of one piece fall on different banks.  A wrong swizzle gives wrong products, not a fault.
#pragma once
#include "common.cuh"

namespace {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Byte offset of 16-byte piece j (K = 8 j .. 8 j + 7) of row r in an operand of `rows` rows (operand format above)
__device__ __forceinline__ size_t sw128_off(int rows, int r, int j) {
  return (size_t)(j >> 3) * rows * 128 + r * 128 + (((j & 7) ^ (r & 7)) << 4);
}

// Accumulator fragment (m64nN layout, wg_frag_pairs below) -> 16-bit operand of a warpgroup's 64 rows, by stmatrix: one .x4 stores
// 16 columns of the warp's 16 rows, its four 8 x 8 matrices being rows 0-7 and 8-15 of columns 0-7, then of columns 8-15 (each
// lane's register holds the pair its fragment holds).  Lane l names row l & 7 of matrix l >> 3.  stsm_base gives that row's address
// for columns 0-15 of the operand at `buf` (128-B aligned); columns 16 p .. 16 p + 15 are pieces 2p & 7 and its neighbour of K
// block p >> 2, so only the swizzled piece bits (4-6) change, by an XOR with 2p & 7, and the block adds its pitch.
__device__ __forceinline__ uint32_t stsm_base(uint32_t buf) {
  const int l = threadIdx.x & 31;
  const int r = 16 * ((threadIdx.x >> 5) & 3) + (l & 15);
  return buf + r * 128 + ((((l >> 4) & 1) ^ (l & 7)) << 4);
}
__device__ __forceinline__ void stsm_x4(uint32_t base, int p, uint32_t block_pitch, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};\n" ::"r"((base ^ ((uint32_t)(2 * p & 7) << 4)) + (uint32_t)(p >> 2) * block_pitch),
               "r"(r0), "r"(r1), "r"(r2), "r"(r3)
               : "memory");
}

// One 16-byte piece of an operand: cp.async from `src` when `valid` (completed by the caller's cp.async.wait_all), zeros otherwise
__device__ __forceinline__ void cp_async_piece_or_zero(uint8_t* dst, const void* src, bool valid) {
  if (valid)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_u32(dst)), "l"(src) : "memory");
  else
    *reinterpret_cast<int4*>(dst) = make_int4(0, 0, 0, 0);
}

// wgmma shared-memory matrix descriptor of an operand in the format above.  Advancing the start address by 32 B steps K by 16.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);   // start address >> 4
  d |= (uint64_t)1 << 16;                   // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;         // stride byte offset: 8-row group pitch = 1024 B
  d |= (uint64_t)1 << 62;                   // layout type SWIZZLE_128B
  return d;
}

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, fp32 accumulators in registers; BF16 selects bf16 operands, else IEEE fp16
template <int N, bool BF16>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, int scale_d);
template <> __device__ __forceinline__ void wgmma_ss<32, false>(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<32, true>(float (&d)[16], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<64, false>(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<64, true>(float (&d)[32], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<96, false>(float (&d)[48], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<96, true>(float (&d)[48], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<128, false>(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<128, true>(float (&d)[64], uint64_t da, uint64_t db, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(PENDING) : "memory"); }

// One warpgroup: rows of A starting at `a` (already offset to the warpgroup's 64 rows), rows of B starting at `b`; KSTEPS
// steps of K = 16; a_cp / b_cp = byte pitch of one 64-wide K chunk of each operand.  Issues and commits one wgmma group;
// the caller waits with wgmma_wait.  accumulate = false starts from zero.
// Each step's descriptor is the first one plus its byte offset >> 4: shared addresses lie below 2^18, so the 14-bit start field
// of every operand address never carries into the next field, and the descriptors equal wg_desc_sw128 of each address.
template <int N, bool BF16, int KSTEPS>
__device__ __forceinline__ void wg_tile_mma(float (&d)[N / 2], uint32_t a, uint32_t a_cp, uint32_t b, uint32_t b_cp, bool accumulate) {
  const uint64_t da = wg_desc_sw128(a), db = wg_desc_sw128(b);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KSTEPS; k++) {
    const uint32_t off = (uint32_t)(k >> 2), s = (uint32_t)(k & 3) * 32u;
    wgmma_ss<N, BF16>(d, da + ((off * a_cp + s) >> 4), db + ((off * b_cp + s) >> 4), (accumulate || k) ? 1 : 0);
  }
  wgmma_commit();
}

// Accumulator fragment of m64nN: f(row, col, v[col], v[col + 1]) for every register pair of this thread; row in [0, 64)
// relative to the warpgroup's first row, col even.
template <int N, class F>
__device__ __forceinline__ void wg_frag_pairs(const float (&d)[N / 2], F f) {
  const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const int r = 16 * w + (l >> 2), c = 2 * (l & 3);
#pragma unroll
  for (int j = 0; j < N / 8; j++) {
    f(r, 8 * j + c, d[4 * j], d[4 * j + 1]);
    f(r + 8, 8 * j + c, d[4 * j + 2], d[4 * j + 3]);
  }
}

// Shared-memory accumulator tile [rows][ld] fp32 (ld a multiple of 32): 16-byte chunks XOR-swizzled by row, so that both the
// fragment stores and thread-per-row float4 reads spread over the banks.
__device__ __forceinline__ int acc_idx(int ld, int r, int c) { return r * ld + ((((c >> 2) ^ (r & 7)) << 2) | (c & 3)); }
template <int N>
__device__ __forceinline__ void wg_store_acc(const float (&d)[N / 2], float* acc, int ld, int row0, int col0) {
  wg_frag_pairs<N>(d, [&](int r, int c, float v0, float v1) {
    *reinterpret_cast<float2*>(acc + acc_idx(ld, row0 + r, col0 + c)) = make_float2(v0, v1);
  });
}
// thread-per-row read of n (multiple of 4) consecutive columns starting at c0 (multiple of 4)
template <int n>
__device__ __forceinline__ void acc_ld(const float* acc, int ld, int r, int c0, float* v) {
#pragma unroll
  for (int i = 0; i < n; i += 4) {
    const float4 q = *reinterpret_cast<const float4*>(acc + acc_idx(ld, r, c0 + i));
    v[i] = q.x, v[i + 1] = q.y, v[i + 2] = q.z, v[i + 3] = q.w;
  }
}

__device__ __forceinline__ void mbar_init(uint32_t saddr, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(saddr), "r"(count) : "memory");
}
// try_wait suspends the thread in hardware for a bounded time per attempt; the attempt counter turns a lost arrival
// (a protocol bug) into a trap - i.e. a CUDA error the caller sees - instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t saddr, uint32_t parity) {
  uint32_t done = 0, tries = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t}\n"
        : "=r"(done)
        : "r"(saddr), "r"(parity)
        : "memory");
    if (done) break;
    if (++tries > (1u << 24)) __trap();
  }
}

// generic-proxy shared-memory writes -> visible to the tensor core (async proxy)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
}  // namespace
