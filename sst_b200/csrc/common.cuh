// Shared device/host helpers for libsstb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
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

// ---- arena ---------------------------------------------------------------
inline void arena_reset(sstb200_ctx* c) {
  c->arena_off = 0;
  c->arena_epoch++;
}

// Reserve: make sure `bytes` are available from offset 0 (called once at the top of an op
// with an upper bound, so that no growth happens mid-op).
inline int arena_reserve(sstb200_ctx* c, size_t bytes) {
  bytes += 4096;
  if (bytes <= c->arena_cap) return SSTB_OK;
  size_t cap = c->arena_cap ? c->arena_cap : (size_t)1 << 24;
  while (cap < bytes) cap *= 2;
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, cap);
  if (e != cudaSuccess) return sstb_fail(c, SSTB_ERR_WORKSPACE, "arena cudaMalloc(%zu) failed: %s", cap, cudaGetErrorString(e));
  if (c->arena) c->retired.push_back(c->arena);
  c->arena = (char*)p;
  c->arena_cap = cap;
  return SSTB_OK;
}

template <typename T>
inline T* arena_alloc(sstb200_ctx* c, size_t n) {
  size_t off = (c->arena_off + 255) & ~(size_t)255;
  size_t bytes = n * sizeof(T);
  if (off + bytes > c->arena_cap) return nullptr;
  c->arena_off = off + bytes;
  return (T*)(c->arena + off);
}

static inline size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

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

// ---- generic exclusive scan over uint32 values ----------------------------------------------
// ONE launch, any length: single-pass chained scan with decoupled look-back.  Tiles of 256 threads x 8 items are
// claimed through an atomic ticket (so a tile only ever waits for tiles that are already running), publish
// (status, value) as one 64-bit word and look back 32 predecessors at a time.  `Load` maps element index -> uint32.
// ScanTemps must be zero before the launch (scan_temps_alloc memsets it; one scan per allocation).
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
static inline size_t scan_temps_bytes(size_t n_cap) { return al256(64 * 4 + (scan_num_blocks(n_cap) + 1) * 8); }

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
