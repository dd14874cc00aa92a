// Window partition + bucketing plan (B1, B2, B3-levels, B4) for one shift, zero host syncs.
//
// Reference (mmdet3d/ops/sst/sst_ops.py:266-331, :27-64 and
// models/middle_encoders/sst_input_layer_v2.py:128-150) runs ~40 small ATen ops with unique/sort and
// several .item() syncs per shift.  Here: one pass computes the window id + in-window coords per voxel and
// marks a bitmap over window slots; a popcount scan compacts non-empty windows in id order (==
// make_continuous_inds); a counting sort groups tokens per window; one warp per window ranks its tokens
// into stable order (== get_inner_win_inds_slow); one block assigns batching levels and the per-level
// window rank.  Output is both the reference's index tensors and a CSR (win_offsets, tok_perm) that the
// fused attention kernels consume directly.
#include <stdarg.h>
#include "index.cuh"

struct WinGeom {
  int wx, wy, wz;     // window shape
  int sx, sy, sz;     // shift applied to coords
  int nx, ny, nz;     // window slots per axis
  int batch;
};

static void make_geom(const sstb200_window_cfg* cfg, int do_shift, WinGeom& g) {
  // sst_ops.py:269-290
  g.wx = cfg->window_shape[0];
  g.wy = cfg->window_shape[1];
  g.wz = cfg->window_shape[2];
  g.nx = (cfg->sparse_shape[0] + g.wx - 1) / g.wx + 1;
  g.ny = (cfg->sparse_shape[1] + g.wy - 1) / g.wy + 1;
  g.nz = (cfg->sparse_shape[2] + g.wz - 1) / g.wz + 1;
  if (do_shift) {
    g.sx = g.wx / 2;
    g.sy = g.wy / 2;
    g.sz = g.wz / 2;
  } else {
    g.sx = g.wx;
    g.sy = g.wy;
    g.sz = g.wz;
  }
  if (cfg->sparse_shape[2] == g.wz) g.sz = 0;
  g.batch = cfg->batch_size;
}

template <typename TC, bool SM>
__global__ void __launch_bounds__(SM ? 1024 : 256) win_mark_kernel(const TC* __restrict__ coors, int n, const int32_t* __restrict__ n_dev, WinGeom g,
                                long long* __restrict__ keys, uint32_t* __restrict__ bitmap, int32_t* __restrict__ flags,
                                long long* __restrict__ batch_win_inds, long long* __restrict__ coors_in_win,
                                int32_t* __restrict__ pos_code, uint32_t nwords) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint32_t mark_sbm[];  // SM: block-private bitmap (see mark_rows_kernel)
  if (n_dev) n = *n_dev;
  if (SM) {
    for (uint32_t w = threadIdx.x; w < nwords; w += blockDim.x) mark_sbm[w] = 0u;
    __syncthreads();
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    long long b = (long long)coors[(size_t)i * 4 + 0];
    long long x = (long long)coors[(size_t)i * 4 + 3] + g.sx;
    long long y = (long long)coors[(size_t)i * 4 + 2] + g.sy;
    long long z = (long long)coors[(size_t)i * 4 + 1] + g.sz;
    long long wxi = x / g.wx, wyi = y / g.wy, wzi = z / g.wz;
    long long key = b * ((long long)g.nx * g.ny * g.nz) + wxi * (g.ny * g.nz) + wyi * g.nz + wzi;
    int cx = (int)(x - wxi * g.wx), cy = (int)(y - wyi * g.wy), cz = (int)(z - wzi * g.wz);
    if (batch_win_inds) batch_win_inds[i] = key;
    if (coors_in_win) {
      coors_in_win[(size_t)i * 3 + 0] = cz;
      coors_in_win[(size_t)i * 3 + 1] = cy;
      coors_in_win[(size_t)i * 3 + 2] = cx;
    }
    if (pos_code) pos_code[i] = cx | (cy << 8) | (cz << 16);
    bool bad = b < 0 || b >= g.batch || wxi < 0 || wxi >= g.nx || wyi < 0 || wyi >= g.ny || wzi < 0 || wzi >= g.nz;
    if (bad) {
      keys[i] = -1;
      flags[0] = 1;
      continue;
    }
    keys[i] = key;
    if (SM) atomicOr(&mark_sbm[key >> 5], 1u << (key & 31));
    else bitmap_set(bitmap, key);
  }
  if (SM) bitmap_merge(mark_sbm, bitmap, nwords);
}

struct LevelCfg {
  int n;
  int id[8], lo[8], hi[8], maxtok[8];
};

// Single block: level slot per window (from its token count, or carried per token from the drop phase),
// rank of the window inside its level (== make_continuous_inds on the level's subset), per-level totals.
__global__ void __launch_bounds__(1024) win_level_kernel(const uint32_t* __restrict__ offsets, const int32_t* __restrict__ order,
                                                         const int32_t* __restrict__ nwin_dev, LevelCfg lv,
                                                         const long long* __restrict__ token_level,
                                                         int32_t* __restrict__ win_level, int32_t* __restrict__ win_rank,
                                                         int32_t* __restrict__ counters /*[1+8+8]*/, int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  __shared__ int sh[8][1024 + 1];
  int R = *nwin_dev;
  int per = (R + blockDim.x - 1) / blockDim.x;
  int b = threadIdx.x * per, e = min(R, b + per);
  int cnt[8], tok[8];
#pragma unroll
  for (int l = 0; l < 8; l++) cnt[l] = tok[l] = 0;
  for (int w = b; w < e; w++) {
    int c = (int)(offsets[w + 1] - offsets[w]);
    int slot = -1;
    if (token_level) {
      long long id = token_level[order[offsets[w]]];
      for (int l = 0; l < lv.n; l++)
        if (lv.id[l] == id) slot = l;
    } else {
      for (int l = 0; l < lv.n; l++)
        if (c >= lv.lo[l] && c < lv.hi[l]) slot = l;  // later entries win, like the reference's loop
    }
    if (slot < 0) {
      flags[1] = 1;  // window count not covered by any drop_range (the reference asserts on this)
      slot = 0;
    }
    win_level[w] = slot;
#pragma unroll
    for (int l = 0; l < 8; l++)
      if (l == slot) {
        cnt[l]++;
        tok[l] += c;
      }
  }
#pragma unroll
  for (int l = 0; l < 8; l++) sh[l][threadIdx.x] = cnt[l];
  __syncthreads();
  // exclusive scan over threads, one warp per level (8 warps busy) - serial over 1024/32 chunks
  int w = threadIdx.x >> 5, ln = threadIdx.x & 31;
  if (w < 8) {
    int carry = 0;
    for (int c0 = 0; c0 < (int)blockDim.x; c0 += 32) {
      int v = sh[w][c0 + ln];
      int x = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, x, o);
        if (ln >= o) x += y;
      }
      sh[w][c0 + ln] = carry + x - v;
      carry += __shfl_sync(0xffffffffu, x, 31);
    }
    if (ln == 0) sh[w][blockDim.x] = carry;
  }
  __syncthreads();
  int run[8];
#pragma unroll
  for (int l = 0; l < 8; l++) run[l] = sh[l][threadIdx.x];
  for (int wv = b; wv < e; wv++) {
    int slot = win_level[wv];
#pragma unroll
    for (int l = 0; l < 8; l++)
      if (l == slot) win_rank[wv] = run[l]++;
  }
  // per-level token totals
#pragma unroll
  for (int l = 0; l < 8; l++) {
    int t = tok[l];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (ln == 0 && t) atomicAdd(&counters[9 + l], t);
  }
  if (threadIdx.x < 8) counters[1 + threadIdx.x] = sh[threadIdx.x][blockDim.x];
  if (threadIdx.x == 0) counters[0] = R;
}

__global__ void tok_finish_kernel(int n, const int32_t* __restrict__ n_dev, const int32_t* __restrict__ tok_win,
                                  const int32_t* __restrict__ tok_inner, const int32_t* __restrict__ win_level,
                                  const int32_t* __restrict__ win_rank, LevelCfg lv, long long* __restrict__ drop_level,
                                  long long* __restrict__ flat2win, const uint32_t* __restrict__ offsets,
                                  int32_t* __restrict__ tok_slot) {
  pdl_wait();
  pdl_launch();
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = *n_dev;
  if (i >= n) return;
  int w = tok_win[i];
  if (w < 0) {
    if (drop_level) drop_level[i] = -1;
    if (flat2win) flat2win[i] = -1;
    if (tok_slot) tok_slot[i] = -1;
    return;
  }
  if (tok_slot) tok_slot[i] = (int32_t)offsets[w] + tok_inner[i];
  int slot = win_level[w];
  if (drop_level) drop_level[i] = lv.id[slot];
  if (flat2win) flat2win[i] = (long long)win_rank[w] * lv.maxtok[slot] + tok_inner[i];
}

// Window batches for the batched attention kernels: batch b = the windows whose first slot lies in [b*ATT_CHUNK, (b+1)*ATT_CHUNK).
// One int4 record per batch {first window, end window, first slot, end slot} (two lower bounds over offsets[0..R) per thread), so
// that a consumer CTA learns everything about its batch from ONE load; counters[17] = number of batches.
__global__ void win_batch_kernel(const uint32_t* __restrict__ offsets, const int32_t* __restrict__ nwin_dev,
                                 int4* __restrict__ batch_rec, int rec_cap, int32_t* __restrict__ counters, const int32_t* __restrict__ flags) {
  pdl_wait();
  pdl_launch();
  const int R = *nwin_dev;
  const int ntok = (int)offsets[R];
  const int nb = (ntok + ATT_CHUNK - 1) / ATT_CHUNK;
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < nb && b < rec_cap; b += gridDim.x * blockDim.x) {
    int w[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const uint32_t t0 = (uint32_t)(b + e) * (uint32_t)ATT_CHUNK;
      int lo = 0, hi = R;
      while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (offsets[mid] < t0) lo = mid + 1;
        else hi = mid;
      }
      w[e] = lo;
    }
    batch_rec[b] = make_int4(w[0], w[1], (int)offsets[w[0]], (int)offsets[w[1]]);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    counters[17] = nb;
    counters[0] = R;
    counters[18] = flags[0] | (flags[1] << 1);   // status word for sync-free callers (bit0: token outside the window grid)
  }
}

__global__ void zero_counters_kernel(int32_t* c) {
  pdl_wait();
  pdl_launch();
  if (threadIdx.x < 20) c[threadIdx.x] = 0;
}

template <typename TC>
static int window_plan_impl(sstb200_ctx* c, const TC* coors, int n, const int32_t* n_dev, const sstb200_window_cfg* cfg,
                            int do_shift, const int64_t* token_level, const sstb200_window_shift* o, int32_t* err_host) {
  CHECK_ARG(c, c && cfg && o && n >= 0);
  CHECK_ARG(c, cfg->num_levels >= 1 && cfg->num_levels <= 8 && cfg->batch_size >= 1);
  CHECK_ARG(c, o->tok_win && o->tok_inner && o->win_offsets && o->tok_perm && o->win_level && o->win_rank && o->counters);
  CHECK_ARG(c, ((uintptr_t)o->win_batch & 15) == 0);   // int4 records
  WinGeom g;
  make_geom(cfg, do_shift, g);
  CHECK_ARG(c, g.wx > 0 && g.wy > 0 && g.wz > 0 && g.wx < 256 && g.wy < 256 && g.wz < 256);
  LevelCfg lv;
  lv.n = cfg->num_levels;
  for (int l = 0; l < 8; l++) {
    lv.id[l] = l < lv.n ? cfg->level_id[l] : -1;
    lv.lo[l] = l < lv.n ? cfg->level_lo[l] : 0;
    lv.hi[l] = l < lv.n ? cfg->level_hi[l] : 0;
    lv.maxtok[l] = l < lv.n ? cfg->level_max_tokens[l] : 0;
  }
  launch_pdl(zero_counters_kernel, dim3(1), dim3(32), (size_t)(0), c->stream, o->counters);
  if (n == 0) {
    LAUNCH_CHECK(c);
    return SSTB_OK;
  }
  CHECK_ARG(c, coors);
  long long T = (long long)g.batch * g.nx * g.ny * g.nz;
  if (T > ((long long)1 << 34)) return sstb_fail(c, SSTB_ERR_UNSUPPORTED, "window slot space too large");
  arena_reset(c);
  size_t nwcap = (size_t)n;  // #windows <= #tokens
  KeyIndex k;
  int32_t* count;
  Csr r;
  r.offsets = (uint32_t*)o->win_offsets;  // int32 [n+1] caller buffer (only R+1 entries are meaningful): the scan writes it in place
  int rc = arena_carve(c, [&](Carve& cv) {
    key_index_carve(cv, k, n, T);
    count = cv.take<int32_t>(nwcap + 2);
    csr_carve(cv, r, n, nwcap);
  });
  if (rc) return rc;
  if ((rc = key_index_zero(c, k))) return rc;
  CUDA_TRY(c, cudaMemsetAsync(count, 0, (nwcap + 2) * 4, c->stream));
  int nb = (n + 255) / 256;
  if (k.nwords <= 12 * 1024) {  // <= 48 KB: block-private bitmap
    int mg = (n + 1023) / 1024;
    if (mg > c->num_sms) mg = c->num_sms;
    launch_pdl(win_mark_kernel<TC, true>, dim3(mg), dim3(1024), k.nwords * 4, c->stream, coors, n, n_dev, g, k.keys, k.bitmap, k.flags,
               (long long*)o->batch_win_inds, (long long*)o->coors_in_win, o->pos_code, (uint32_t)k.nwords);
  } else {
    launch_pdl(win_mark_kernel<TC, false>, dim3(nb), dim3(256), (size_t)(0), c->stream, coors, n, n_dev, g, k.keys, k.bitmap, k.flags,
               (long long*)o->batch_win_inds, (long long*)o->coors_in_win, o->pos_code, 0u);
  }
  key_index_scan(c, k);
  launch_pdl(map_count_kernel<int32_t>, dim3(nb), dim3(256), (size_t)(0), c->stream, k.keys, n, k.bitmap, k.word_prefix, 0, k.flags, o->tok_win, count, n_dev);
  const int32_t* nwin = (const int32_t*)k.total;  // #distinct windows, written by the bitmap scan
  rc = csr_build<int32_t>(c, r, o->tok_win, n, count, nwcap, nwin, n_dev);
  if (rc) return rc;
  // the reference-layout outputs (drop level, flat2win index, per-level window rank) are only produced on request; the
  // fused kernels need the CSR, the stable in-window rank and the slot of every token - all written by stable_rank_kernel
  const bool want_levels = o->drop_level || o->flat2win_inds || token_level || err_host;
  launch_pdl(stable_rank_kernel, dim3(c->num_sms * 4), dim3(256), (size_t)(0), c->stream, r.offsets, r.order, nwin, o->tok_perm, nullptr, o->tok_inner,
             want_levels ? nullptr : o->tok_slot);
  if (want_levels) {
    launch_pdl(win_level_kernel, dim3(1), dim3(1024), (size_t)(0), c->stream, r.offsets, o->tok_perm, nwin, lv, (const long long*)token_level,
               o->win_level, o->win_rank, o->counters, k.flags);
    launch_pdl(tok_finish_kernel, dim3(nb), dim3(256), (size_t)(0), c->stream, n, n_dev, o->tok_win, o->tok_inner, o->win_level, o->win_rank, lv,
               (long long*)o->drop_level, (long long*)o->flat2win_inds, r.offsets, o->tok_slot);
  }
  if (o->win_batch) {
    launch_pdl(win_batch_kernel, dim3((n / ATT_CHUNK + 256) / 256), dim3(256), (size_t)0, c->stream, (const uint32_t*)r.offsets, (const int32_t*)nwin,
               reinterpret_cast<int4*>(o->win_batch), att_rec_cap(n), o->counters, (const int32_t*)k.flags);
  }
  LAUNCH_CHECK(c);
  if (err_host) {
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32, k.flags, 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(c->pinned_i32 + 2, o->counters, 17 * 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    err_host[0] = c->pinned_i32[0] | (c->pinned_i32[1] << 1);
    for (int i = 0; i < 17; i++) err_host[1 + i] = c->pinned_i32[2 + i];
  }
  return SSTB_OK;
}

extern "C" int sstb200_window_plan(sstb200_ctx* c, const int64_t* coors, int n, const int32_t* n_dev,
                                   const sstb200_window_cfg* cfg, int do_shift, const int64_t* token_level,
                                   const sstb200_window_shift* out, int32_t* status_host) {
  return window_plan_impl<long long>(c, (const long long*)coors, n, n_dev, cfg, do_shift, token_level, out, status_host);
}

extern "C" int sstb200_window_plan_i32(sstb200_ctx* c, const int32_t* coors, int n, const int32_t* n_dev,
                                       const sstb200_window_cfg* cfg, int do_shift, const sstb200_window_shift* out) {
  return window_plan_impl<int32_t>(c, coors, n, n_dev, cfg, do_shift, nullptr, out, nullptr);
}
