// Shared device/host helpers for libsstb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/sstb200.h"

#define SSTB_OK 0
#define SSTB_ERR_CUDA -1
#define SSTB_ERR_ARG -2
#define SSTB_ERR_UNSUPPORTED -3
#define SSTB_ERR_WORKSPACE -4

struct sstb200_ctx {
  int device = 0;
  cudaStream_t stream = 0;
  int num_sms = 132;
  // bump arena for temporaries; grows (with a sync) when a call needs more.
  char* arena = nullptr;
  size_t arena_cap = 0;
  size_t arena_off = 0;
  std::vector<void*> retired;  // old arenas kept alive until destroy (stream-ordered safety)
  unsigned long long arena_epoch = 0;  // bumped by arena_reset: what a call left in the arena survives while this is unchanged
  std::shared_ptr<void> handoff;       // host record of such arena contents, for the call that consumes them
  unsigned long long handoff_epoch = 0;
  std::string err;
  int32_t* pinned_i32 = nullptr;  // small pinned scratch for D2H counters
  cudaEvent_t ev_coords = nullptr;  // recorded by the VFE entry points once voxel_coors / num_dev are produced (fork point of a side branch)
  cudaEvent_t ev_done = nullptr;    // recorded by sstb200_branch_join on the side context's stream
};

inline int sstb_fail(sstb200_ctx* c, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (c) c->err = buf;
  return code;
}

#define CUDA_TRY(ctx, expr)                                                                     \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess)                                                                      \
      return sstb_fail(ctx, SSTB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,        \
                       cudaGetErrorString(_e));                                                 \
  } while (0)

#define CHECK_ARG(ctx, cond)                                                                    \
  do {                                                                                          \
    if (!(cond)) return sstb_fail(ctx, SSTB_ERR_ARG, "%s:%d bad argument: %s", __FILE__, __LINE__, #cond); \
  } while (0)

#define LAUNCH_CHECK(ctx) CUDA_TRY(ctx, cudaGetLastError())

static inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

// ---- workspace carving ----------------------------------------------------------------------------------------------------------
// A workspace layout is written once, as a carve function f(Carve&) that takes its pieces in order.  Over base == nullptr the
// cursor only measures (every take returns nullptr); over a real base it hands out the same pieces.  Each piece starts on a
// 256-byte boundary.  A carve function only carves - no launches, no memsets, no arithmetic on the pointers it gets back - and
// takes the same branches in both passes.
struct Carve {
  char* base = nullptr;
  size_t off = 0;
  template <typename T>
  T* take(size_t n) {
    off = al256(off);
    T* p = base ? (T*)(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
  size_t mark() const { return al256(off); }  // where the next piece starts: cv.off - cv.mark() spans the pieces taken since
};

// bytes of a caller-owned workspace laid out by f from offset 0
template <typename F>
static inline size_t carve_bytes(F&& f) {
  Carve m;
  f(m);
  return al256(m.off);
}

// ---- arena ---------------------------------------------------------------
// bump arena for the temporaries of one call: arena_reset starts a phase, arena_carve lays out its pieces from c->arena_off
inline void arena_reset(sstb200_ctx* c) {
  c->arena_off = 0;
  c->arena_epoch++;
}

// Measures f from c->arena_off, grows the arena (with a sync) when it is too small, then carves f out of it and advances
// c->arena_off.  Growth happens only here, before any piece of the phase is handed out, so a warm-up call sizes the arena once
// for the CUDA graph captured after it.  A grown arena retires the old one: pieces an earlier carve of the same phase handed
// out stay valid until destroy.
template <typename F>
static inline int arena_carve(sstb200_ctx* c, F&& f) {
  Carve m{nullptr, c->arena_off};
  f(m);
  if (m.off > c->arena_cap) {
    size_t cap = c->arena_cap ? c->arena_cap : (size_t)1 << 24;
    while (cap < m.off) cap *= 2;
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, cap);
    if (e != cudaSuccess) return sstb_fail(c, SSTB_ERR_WORKSPACE, "arena cudaMalloc(%zu) failed: %s", cap, cudaGetErrorString(e));
    if (c->arena) c->retired.push_back(c->arena);
    c->arena = (char*)p;
    c->arena_cap = cap;
  }
  Carve r{c->arena, c->arena_off};
  f(r);
  if (r.off != m.off) return sstb_fail(c, SSTB_ERR_WORKSPACE, "arena carve: the measuring and carving passes disagree");
  c->arena_off = r.off;
  return SSTB_OK;
}

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-DEVICE property of a kernel: remember the largest value applied per device
// (one static SmemAttr per call site / kernel instantiation), so a process that drives several GPUs sets it on each of them.
struct SmemAttr {
  size_t set[64] = {0};
};
template <typename K>
static inline cudaError_t ensure_smem(const sstb200_ctx* c, SmemAttr& a, K kern, size_t bytes) {
  const int d = c->device & 63;
  if (bytes <= a.set[d]) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) a.set[d] = bytes;
  return e;
}

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------
// Every kernel of the library starts with pdl_wait() (griddepcontrol.wait: block until the producer grid has completed
// and its writes are visible) followed by pdl_launch() (griddepcontrol.launch_dependents: allow the next kernel of the
// stream / graph to be scheduled while this one still runs).  Launches carry the programmatic-stream-serialization
// attribute, so inside the per-frame CUDA graph consecutive kernels are linked by programmatic edges and the launch
// latency of kernel N+1 overlaps the execution of kernel N.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// All kernels of the library ask for the same shared-memory carveout (max shared): consecutive kernels with different
// carveouts force the SMs to drain and re-partition L1/shared between launches, which costs more than any L1 hit here.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  static void* seen[32];  // per kernel signature & TU; the attribute is sticky per function -> set once, before any capture
  static int nseen = 0;
  bool found = false;
  for (int i = 0; i < nseen; i++) found |= (seen[i] == (void*)kern);
  if (!found) {
    cudaFuncSetAttribute((const void*)kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (nseen < 32) seen[nseen++] = (void*)kern;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// ---- window batches of the batched attention kernels ---------------------------------------------------------------------
// Batch b = the windows whose first slot lies in [b * ATT_CHUNK, (b + 1) * ATT_CHUNK) (win_batch_kernel, window.cu); with
// windows of at most ATT_MAXT tokens it holds at most ATT_CHUNK - 1 + ATT_MAXT rows, which the kernels stage in ATT_BT rows.
#define ATT_MAXT 144
#define ATT_CHUNK 112
#define ATT_BT 256
static_assert(ATT_CHUNK - 1 + ATT_MAXT <= ATT_BT, "a window batch must fit the staged rows");
// Record-array bound for a plan over n tokens.  At most n / ATT_CHUNK + 1 records are written, but the caller's win_batch buffer
// is documented (include/sstb200.h) and allocated (ops.py, engine.py) for n / 32 + 2, so that stays the bound.
static inline int att_rec_cap(int n) { return n / 32 + 2; }

// ---- device helpers ------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// order-preserving float <-> uint mapping (for atomicMax on floats of any sign)
__device__ __forceinline__ unsigned f2ord(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// exact-form GELU (x * Phi(x)) with erf from Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7): ~12 instructions instead of
// erff's ~30, same accuracy class as fp32 erff for an output that is rounded to bf16 anyway.
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));  // MUFU.RCP (__frcp_rn is a ~25-instruction subroutine)
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = 1.0f - p * t * __expf(-z * z);   // erf(|x|/sqrt2)
  return 0.5f * x * (1.0f + copysignf(e, x));
}

// exact-form GELU with one MUFU op and 9 ALU instructions, for epilogues where GELU dominates the instruction stream.
// x Phi(x) = max(x, 0) - |x| Q(|x|), Q(a) = Phi(-a) the normal tail, and log2 Q(a) is smooth on [0, 6]: a degree-6 polynomial
// (weighted minimax) holds it to 1.3e-7 of the GELU, max abs error 2.4e-7 over [-12, 12] (half an fp32 ulp of x where x ~ 4),
// at most 0.2 fp16 ulp of the result.  Past |x| = 6 the tail term stays below 1.2e-8 (rounds to 0 in fp16) and is clamped there.
// tests/test_gpu_sra_chain_epilogue.py mirrors this exact fp32 sequence.
__device__ __forceinline__ float gelu_ex2(float x) {
  const float a = fminf(fabsf(x), 6.0f);
  float p = fmaf(3.50552036e-05f, a, -7.84027274e-04f);
  p = fmaf(p, a, 8.12153984e-03f);
  p = fmaf(p, a, -5.34629487e-02f);
  p = fmaf(p, a, -4.58742619e-01f);
  p = fmaf(p, a, -1.15120757e+00f);
  p = fmaf(p, a, -9.99992907e-01f);   // log2 Q(a)
  float q;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(q) : "f"(p));   // MUFU.EX2
  return fmaf(-fabsf(x), q, fmaxf(x, 0.0f));
}

// d/dz [z Phi(z)] = Phi(z) + z phi(z)
__device__ __forceinline__ float gelu_grad(float z) {
  const float cdf = 0.5f * (1.0f + erff(z * 0.70710678118654752440f));
  return cdf + z * 0.3989422804014327f * __expf(-0.5f * z * z);
}

// ---- 16-bit pairs --------------------------------------------------------------------------------------------------------------
// Two fp32 values rounded to nearest into one 32-bit word, a in the low half.  FMT selects the 16-bit format of the pack_h16 /
// unpack_h16 forms: IEEE fp16 or bf16.
enum { FMT_F16 = 0, FMT_BF16 = 1 };
__device__ __forceinline__ uint32_t pack_f16(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <int FMT>
__device__ __forceinline__ uint32_t pack_h16(float a, float b) {
  return FMT == FMT_BF16 ? pack_bf16(a, b) : pack_f16(a, b);
}
template <int FMT>
__device__ __forceinline__ float2 unpack_h16(uint32_t u) {
  if (FMT == FMT_BF16) return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u));
  return __half22float2(*reinterpret_cast<__half2*>(&u));
}
// 8 consecutive fp32 values -> one 16-byte piece of 16-bit values
template <int FMT>
__device__ __forceinline__ int4 pack8_h16(const float* f) {
  return make_int4((int)pack_h16<FMT>(f[0], f[1]), (int)pack_h16<FMT>(f[2], f[3]), (int)pack_h16<FMT>(f[4], f[5]), (int)pack_h16<FMT>(f[6], f[7]));
}
template <int FMT>
__device__ __forceinline__ int4 pack8_h16(float4 a, float4 b) {
  return make_int4((int)pack_h16<FMT>(a.x, a.y), (int)pack_h16<FMT>(a.z, a.w), (int)pack_h16<FMT>(b.x, b.y), (int)pack_h16<FMT>(b.z, b.w));
}

// ---- generic exclusive scan over uint32 values ----------------------------------------------
// ONE launch, any length: single-pass chained scan with decoupled look-back.  Tiles of 256 threads x 8 items are
// claimed through an atomic ticket (so a tile only ever waits for tiles that are already running), publish
// (status, value) as one 64-bit word and look back 32 predecessors at a time.  `Load` maps element index -> uint32.
// ScanTemps must be zero before the launch (its owner memsets what scan_carve took; one scan per carve).
#define SCAN_ITEMS 8
#define SCAN_THREADS 256
#define SCAN_TILE (SCAN_ITEMS * SCAN_THREADS)

struct LoadU32 {
  const uint32_t* p;
  __device__ __forceinline__ uint32_t operator()(size_t i) const { return p[i]; }
  __device__ __forceinline__ void load8(size_t base, size_t n, uint32_t* v) const {
    if (base + 8 <= n && (((uintptr_t)p) & 15) == 0) {
      uint4 a = *reinterpret_cast<const uint4*>(p + base), b = *reinterpret_cast<const uint4*>(p + base + 4);
      v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; i++) v[i] = (base + i < n) ? p[base + i] : 0u;
    }
  }
};
struct LoadPopc {
  const uint32_t* p;
  __device__ __forceinline__ uint32_t operator()(size_t i) const { return __popc(p[i]); }
  __device__ __forceinline__ void load8(size_t base, size_t n, uint32_t* v) const {
    LoadU32{p}.load8(base, n, v);
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = __popc(v[i]);
  }
};

__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t* total, uint32_t* sh /*[9]*/) {
  // inclusive warp scan
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane_id() >= o) x += y;
  }
  int w = threadIdx.x >> 5;
  if (lane_id() == 31) sh[w] = x;
  __syncthreads();
  if (w == 0) {
    uint32_t s = (lane_id() < 8) ? sh[lane_id()] : 0;
    uint32_t t = s;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane_id() >= o) t += y;
    }
    if (lane_id() < 8) sh[lane_id()] = t - s;  // exclusive warp offsets
    if (lane_id() == 7) sh[8] = t;
  }
  __syncthreads();
  uint32_t res = x - v + sh[w];
  *total = sh[8];
  __syncthreads();
  return res;
}

struct ScanTemps {
  uint32_t* ticket;            // [64] words: [0] tile ticket; [1..] free for the owner (totals, flags, counters)
  unsigned long long* state;   // [tiles] (status << 32 | value); status 0 = empty, 1 = tile aggregate, 2 = inclusive prefix
};
static inline size_t scan_num_blocks(size_t n_cap) { return (n_cap + 1 + SCAN_TILE - 1) / SCAN_TILE; }
static inline void scan_carve(Carve& cv, ScanTemps& t, size_t n_cap) {
  t.ticket = cv.take<uint32_t>(64);
  t.state = cv.take<unsigned long long>(scan_num_blocks(n_cap) + 1);
}

// n may be read from device memory (n_dev != nullptr) so that data-dependent sizes never sync.
template <typename Load>
__global__ void __launch_bounds__(SCAN_THREADS) scan_lookback_kernel(Load load, size_t n_host, const int32_t* n_dev, uint32_t* out,
                                                                     uint32_t* total_out, bool write_total_at_n, ScanTemps t) {
  pdl_wait();
  pdl_launch();
  __shared__ uint32_t sh[9];
  __shared__ uint32_t tile_s, prefix_s;
  const size_t n = n_dev ? (size_t)max(*n_dev, 0) : n_host;
  if (threadIdx.x == 0) tile_s = atomicAdd(t.ticket, 1u);
  __syncthreads();
  const uint32_t tile = tile_s;
  if ((size_t)tile * SCAN_TILE > n) return;  // index n (the total's slot) lives in tile n / SCAN_TILE
  const size_t base = (size_t)tile * SCAN_TILE + (size_t)threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS], s = 0;
  load.load8(base, n, v);
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) s += v[i];
  uint32_t tot;
  uint32_t ex = block_exclusive_scan_256(s, &tot, sh);
  volatile unsigned long long* state = t.state;
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    uint32_t run = 0;
    if (tile > 0) {
      if (lane == 0) state[tile] = (1ull << 32) | tot;
      long long top = (long long)tile - 1;
      while (true) {
        long long idx = top - lane;
        unsigned long long sv = idx >= 0 ? state[idx] : (2ull << 32);
        while (__any_sync(0xffffffffu, (sv >> 32) == 0)) sv = idx >= 0 ? state[idx] : (2ull << 32);
        unsigned incl = __ballot_sync(0xffffffffu, (sv >> 32) == 2);
        int first = incl ? __ffs(incl) - 1 : 31;
        uint32_t c = lane <= first ? (uint32_t)sv : 0u;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        run += c;
        if (incl) break;
        top -= 32;
      }
    }
    if (lane == 0) {
      state[tile] = (2ull << 32) | (unsigned long long)(run + tot);
      prefix_s = run;
    }
  }
  __syncthreads();
  ex += prefix_s;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    size_t k = base + i;
    if (k < n) out[k] = ex;
    else if (k == n) {
      if (write_total_at_n) out[k] = ex;
      *total_out = ex;
    }
    ex += v[i];
  }
}

// out has n(+1 if write_total_at_n) entries; total_out receives the grand total.  `t` must be freshly zeroed.
template <typename Load>
static inline void launch_exclusive_scan(cudaStream_t st, Load load, size_t n_cap, const int32_t* n_dev,
                                         ScanTemps t, uint32_t* out, uint32_t* total_out, bool write_total_at_n) {
  unsigned nblk = (unsigned)scan_num_blocks(n_cap);
  launch_pdl(scan_lookback_kernel<Load>, dim3(nblk), dim3(SCAN_THREADS), (size_t)0, st, load, n_cap, n_dev, out, total_out, write_total_at_n, t);
}
