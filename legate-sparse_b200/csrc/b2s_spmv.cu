// b2s_spmv.cu — CSR SpMV for sm_90a.
//
// Replaces CSRSpMVRowSplit (reference src/sparse/array/csr/spmv.cu:30-163 = one cusparseSpMV
// call; CPU semantics spmv.cc:36-43: y[i] = sum_j vals[j] * x[crd[j]]).
//
// Two kernels:
//   * spmv_tile_kernel  — nnz-balanced streaming kernel driven by a cached plan.
//       Phase A: the CTA streams one contiguous tile of TILE_NNZ (col, val) pairs with
//                128-bit loads (L1 no_allocate, L2 evict_first), gathers x (from a shared-
//                memory window staged by one TMA bulk copy when the tile's [min col,max col]
//                image is small — banded / stencil matrices — otherwise from L2 with an
//                evict_last policy), and parks the products in shared memory.
//       Phase B: rows of the tile are reduced from shared memory by 1..32 lanes per row
//                (chosen per tile from its row count) in a fixed order → deterministic.
//       Rows that straddle tiles: the tile where the row starts owns y[r]; later tiles
//       write their piece to head[t]; a tiny fix-up kernel adds the heads in tile order.
//       No floating-point atomics anywhere.
//   * spmv_rowvec_kernel — plan-free LANES-per-row kernel (small / one-shot matrices).
#include "b2s_common.cuh"
#include "b2s_board.cuh"

namespace b2s {

constexpr int kTileThreads = 256;
constexpr int kWinCap      = 1024;  // x-window capacity in elements (== kPipeWinCap)
constexpr int kNearSpan    = 12288; // elements of x a tile may span and still live in L1 (96 KB of fp64)

struct PlanHeader {  // host-side plan object
  b2s_itype it;
  int64_t nrows, ncols, nnz;
  int64_t tile_nnz, ntiles;
  int64_t window_tiles;  // tiles whose x window fits kWinCap
  int64_t head_tiles;    // tiles that start inside a row
  // device pointers into the caller's workspace
  int64_t* tile_row;   // [ntiles+1]
  int64_t* tile_win;   // [2*ntiles]  (aligned base col, count) ; count==0 → no window
  void*    head;       // [ntiles] * 16 bytes
  void*    dotp;       // [ntiles] * 16 bytes (per-tile partials of the fused dot)
  int64_t  empty_rows; // number of rows without non-zeros
  int64_t  max_row;    // longest row (nnz) — selects the long-row pass of the products consumer
  int64_t  near_tiles; // tiles whose [min col, max col] image is <= kNearSpan elements: their x gathers
                       // re-hit L1 (products consumer then allocates the gathers in L1)
  int64_t  max_tile_rows; // most rows any tile touches (incl. empty ones): the async-gather kernel marks row
                          // starts with 16-bit tile-local row numbers
  int64_t* counters;   // [8]
};

}  // namespace b2s

struct b2s_spmv_plan : b2s::PlanHeader {};

namespace b2s {

static int64_t default_tile_nnz() {  // read at every plan creation (tools/spmv_sweep varies it)
  const char* e = getenv("B2S_SPMV_TILE_NNZ");
  int64_t t = e ? atoll(e) : 2048;
  if (t != 1024 && t != 2048 && t != 4096) t = 2048;
  return t;
}

// ------------------------------------------------------------------ plan kernels
__global__ void plan_tile_rows_kernel(int64_t nrows, int64_t ntiles, int64_t tile_nnz,
                                      const int64_t* __restrict__ indptr,
                                      int64_t* __restrict__ tile_row) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t > ntiles) return;
  if (t == 0) { tile_row[0] = 0; return; }
  if (t == ntiles) { tile_row[t] = nrows; return; }
  // last r in [0,nrows] with indptr[r] <= S  (upper_bound - 1)
  int64_t S = t * tile_nnz;
  int64_t lo = 0, hi = nrows + 1;  // search first index with indptr[idx] > S
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (indptr[mid] <= S) lo = mid + 1; else hi = mid;
  }
  tile_row[t] = lo - 1;
}

template <typename I>
__global__ void plan_tile_window_kernel(int64_t nnz, int64_t ntiles, int64_t tile_nnz,
                                        const int64_t* __restrict__ indptr,
                                        const I* __restrict__ cols,
                                        const int64_t* __restrict__ tile_row,
                                        int64_t* __restrict__ tile_win,
                                        int64_t* __restrict__ counters) {
  int64_t t = blockIdx.x;
  if (t >= ntiles) return;
  int64_t S = t * tile_nnz, E = min(S + tile_nnz, nnz);
  int64_t mn = INT64_MAX, mx = INT64_MIN;
  for (int64_t p = S + threadIdx.x; p < E; p += blockDim.x) {
    int64_t c = (int64_t)cols[p];
    mn = min(mn, c); mx = max(mx, c);
  }
  for (int o = 16; o > 0; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  __shared__ int64_t smn[32], smx[32];
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { smn[w] = mn; smx[w] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int nw = blockDim.x >> 5;
    for (int i = 1; i < nw; ++i) { mn = min(mn, smn[i]); mx = max(mx, smx[i]); }
    int64_t base = mn & ~(int64_t)3;
    int64_t cnt  = mx - base + 1;
    bool fits = (mn >= 0) && (cnt <= kWinCap);
    tile_win[2 * t]     = fits ? base : 0;
    tile_win[2 * t + 1] = fits ? cnt : 0;
    if (fits) atomicAdd((unsigned long long*)&counters[0], 1ull);
    if (mn >= 0 && mx - mn < kNearSpan) atomicAdd((unsigned long long*)&counters[4], 1ull);
    int64_t r0 = tile_row[t];
    if (indptr[r0] < S) atomicAdd((unsigned long long*)&counters[1], 1ull);
    atomicMax((unsigned long long*)&counters[5], (unsigned long long)(tile_row[t + 1] - r0 + 1));
  }
}

__global__ void plan_count_empty_kernel(int64_t nrows, const int64_t* __restrict__ indptr,
                                        int64_t* __restrict__ counters) {
  int64_t cnt = 0, mx = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t len = indptr[r + 1] - indptr[r];
    cnt += (len == 0);
    mx = max(mx, len);
  }
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (cnt) atomicAdd((unsigned long long*)&counters[2], (unsigned long long)cnt);
    if (mx) atomicMax((unsigned long long*)&counters[3], (unsigned long long)mx);
  }
}

// ------------------------------------------------------------------ helpers
template <typename T>
__device__ __forceinline__ void load_vec4(const T* p, T out[4], uint64_t pol) {
  constexpr int N16 = (int)(sizeof(T) * 4 / 16);
  uint4 raw[N16];
#pragma unroll
  for (int i = 0; i < N16; ++i) raw[i] = ld_stream_16(reinterpret_cast<const uint4*>(p) + i, pol);
  memcpy(out, raw, sizeof(T) * 4);
}

// reduce `v` over groups of LANES consecutive lanes (LANES power of two, runtime, warp-uniform)
template <typename V>
__device__ __forceinline__ V group_reduce(V v, int lanes) {
  for (int o = lanes >> 1; o > 0; o >>= 1) v = vadd(v, vshfl_xor(v, o));
  return v;
}

// ------------------------------------------------------------------ the tile kernel
template <typename V, typename I, int IPT, bool VEC, bool WINDOW, bool DOT>
__global__ void __launch_bounds__(kTileThreads)
spmv_tile_kernel(int64_t nrows, int64_t ncols, int64_t nnz,
                 const int64_t* __restrict__ indptr, const I* __restrict__ cols,
                 const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y,
                 const int64_t* __restrict__ tile_row, const int64_t* __restrict__ tile_win,
                 V* __restrict__ head, V* __restrict__ dot_partials, const V* __restrict__ w) {
  constexpr int T = kTileThreads * IPT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  V* prod = reinterpret_cast<V*>(smem_raw);
  V* xwin = reinterpret_cast<V*>(smem_raw + sizeof(V) * T);                 // WINDOW only
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + sizeof(V) * (T + kWinCap));  // WINDOW only

  const int tid = threadIdx.x;
  const int64_t t = blockIdx.x;
  const int64_t S = t * (int64_t)T;
  const int64_t E = min(S + (int64_t)T, nnz);
  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep   = policy_evict_last();

  // ---- x window: one elected thread issues a TMA bulk copy (UBLKCP) ----
  int64_t wbase = 0, wcnt = 0;
  bool win_pending = false;  // a TMA bulk copy is in flight → wait on the mbarrier before gathering
  if (WINDOW) {
    wbase = tile_win[2 * t];
    wcnt  = tile_win[2 * t + 1];
    if (wcnt > 0) {
      constexpr int PER16 = (16 / (int)sizeof(V)) > 0 ? (16 / (int)sizeof(V)) : 1;
      int64_t want  = ((wcnt + PER16 - 1) / PER16) * PER16;
      int64_t avail = ncols - wbase;
      int64_t total = want < avail ? want : avail;          // elements we may touch
      uint32_t bulk_bytes = (uint32_t)((total * (int64_t)sizeof(V)) / 16 * 16);
      int64_t bulk_elems  = bulk_bytes / sizeof(V);
      if (tid == 0) {
        mbar_init(bar, 1);
        fence_mbar_init();
        if (bulk_bytes > 0) {
          mbar_arrive_expect_tx(bar, bulk_bytes);
          tma_bulk_g2s(xwin, x + wbase, bulk_bytes, bar, pol_keep);
        }
      }
      // leftover (< 16 bytes) elements: plain loads
      for (int64_t i = bulk_elems + tid; i < total; i += kTileThreads) xwin[i] = x[wbase + i];
      __syncthreads();  // barrier init + leftover visible
      win_pending = bulk_bytes > 0;
    }
  }

  // ---- phase A: stream (col,val), gather x, park products ----
  const bool use_win = WINDOW && (wcnt > 0);
  if (VEC && (E - S == T)) {
    I c[IPT];
    V v[IPT];
#pragma unroll
    for (int g = 0; g < IPT / 4; ++g) {
      int64_t p = S + ((int64_t)g * kTileThreads + tid) * 4;
      load_vec4<I>(cols + p, &c[g * 4], pol_stream);
      load_vec4<V>(vals + p, &v[g * 4], pol_stream);
    }
    if (WINDOW && win_pending) mbar_wait(bar, 0);  // the stream loads above are already in flight
    V xv[IPT];
#pragma unroll
    for (int k = 0; k < IPT; ++k) {
      if (use_win) xv[k] = xwin[(int64_t)c[k] - wbase];
      else         xv[k] = ld_gather<V>(x + (int64_t)c[k], pol_keep);
    }
#pragma unroll
    for (int g = 0; g < IPT / 4; ++g) {
      int q = (g * kTileThreads + tid) * 4;
#pragma unroll
      for (int k = 0; k < 4; ++k) prod[q + k] = vmul(v[g * 4 + k], xv[g * 4 + k]);
    }
  } else {
    if (WINDOW && win_pending) mbar_wait(bar, 0);
#pragma unroll
    for (int k = 0; k < IPT; ++k) {
      int64_t p = S + (int64_t)k * kTileThreads + tid;
      if (p < E) {
        int64_t c = (int64_t)ld_stream<I>(cols + p, pol_stream);
        V a = ld_stream<V>(vals + p, pol_stream);
        V xx = use_win ? xwin[c - wbase] : ld_gather<V>(x + c, pol_keep);
        prod[p - S] = vmul(a, xx);
      }
    }
  }
  __syncthreads();

  // ---- phase B: per-row reduction out of shared memory ----
  const int64_t r_begin = tile_row[t];
  const int64_t r_last  = tile_row[t + 1];  // == nrows for the last tile
  const int64_t nr = r_last - r_begin + 1;  // candidate rows (last one may be the sentinel)
  // lanes per row: fill the CTA in one pass when possible
  int lanes = 1;
  while (lanes < 32 && (int64_t)(lanes * 2) * nr <= kTileThreads) lanes <<= 1;
  const int groups = kTileThreads / lanes;
  const int gl = tid & (lanes - 1);
  V dot_acc = zero_of<V>();
  for (int64_t base = 0; base < nr; base += groups) {
    int64_t r = r_begin + base + tid / lanes;
    bool valid = (base + tid / lanes < nr) && (r < nrows);
    int64_t lo_g = 0, hi_g = 0;
    if (valid) { lo_g = indptr[r]; hi_g = indptr[r + 1]; }
    int64_t lo = max(lo_g, S), hi = min(hi_g, E);
    V sum = zero_of<V>();
    for (int64_t p = lo + gl; p < hi; p += lanes) sum = vadd(sum, prod[p - S]);
    sum = group_reduce(sum, lanes);
    if (valid && gl == 0) {
      bool wrote = false;
      if (lo_g < S) { head[t] = sum; wrote = true; }                     // continues an earlier row
      else if (r < r_last || lo_g < E) { y[r] = sum; wrote = true; }     // this tile owns y[r]
      if (DOT && wrote) dot_acc = vfma(w[r], sum, dot_acc);
    }
  }
  if (DOT) {
    // deterministic block reduction of dot_acc → dot_partials[t]
    __shared__ V wsum[kTileThreads / 32];
    V s = dot_acc;
    for (int o = 16; o > 0; o >>= 1) s = vadd(s, vshfl_xor(s, o));
    if ((tid & 31) == 0) wsum[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
      V tot = wsum[0];
      for (int i = 1; i < kTileThreads / 32; ++i) tot = vadd(tot, wsum[i]);
      dot_partials[t] = tot;
    }
  }
}

// y[r] += head[t] for rows that straddle tiles, in tile order (deterministic).
template <typename V, bool DOT>
__global__ void spmv_fixup_kernel(int64_t ntiles, int64_t tile_nnz,
                                  const int64_t* __restrict__ indptr,
                                  const int64_t* __restrict__ tile_row,
                                  const V* __restrict__ head, V* __restrict__ y,
                                  const PeerOut<V> peers) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < 1 || t >= ntiles) return;
  int64_t r = tile_row[t];
  int64_t start = indptr[r];
  int64_t S = t * tile_nnz;
  if (start >= S) return;                  // tile t starts exactly at a row boundary: no head
  if (start < S - tile_nnz) return;        // tile t-1 is not the owner → an earlier thread handles r
  V acc = y[r];
  for (int64_t u = t; u < ntiles && tile_row[u] == r; ++u) acc = vadd(acc, head[u]);
  store_bcast(y, peers, r, acc);
}

// final deterministic reduction of per-tile partials → out[0]
template <typename V>
__global__ void reduce_partials_kernel(int64_t n, const V* __restrict__ partials, V* __restrict__ out,
                                       const BoardArgs<V> bx) {
  __shared__ V sh[32];
  __shared__ V xvals[kBoardRanks];
  V s = zero_of<V>();
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s = vadd(s, partials[i]);
  for (int o = 16; o > 0; o >>= 1) s = vadd(s, vshfl_xor(s, o));
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    V tot = sh[0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) tot = vadd(tot, sh[i]);   // same order in every lane
    // several ranks: the sum over the ranks is taken right here (board exchange, b2s_board.cuh)
    if (bx.nranks > 1) tot = board_exchange_warp<V>(tot, bx, xvals);
    if (threadIdx.x == 0) out[0] = tot;
  }
}

// ------------------------------------------------------------------ plan-free row-vector kernel
template <typename V, typename I, int LANES>
__global__ void __launch_bounds__(256)
spmv_rowvec_kernel(int64_t nrows, const int64_t* __restrict__ indptr, const I* __restrict__ cols,
                   const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y) {
  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep   = policy_evict_last();
  const int gl = threadIdx.x & (LANES - 1);
  const int64_t groups_per_block = blockDim.x / LANES;
  const int64_t total_groups = (int64_t)gridDim.x * groups_per_block;
  // loop bound is uniform across the warp so the shuffles are safe
  const int64_t first = (int64_t)blockIdx.x * groups_per_block;
  for (int64_t rb = first; rb < nrows; rb += total_groups) {
    int64_t r = rb + threadIdx.x / LANES;
    V sum = zero_of<V>();
    if (r < nrows) {
      int64_t lo = indptr[r], hi = indptr[r + 1];
      for (int64_t p = lo + gl; p < hi; p += LANES) {
        int64_t c = (int64_t)ld_stream<I>(cols + p, pol_stream);
        V a = ld_stream<V>(vals + p, pol_stream);
        sum = vfma(a, ld_gather<V>(x + c, pol_keep), sum);
      }
    }
#pragma unroll
    for (int o = LANES >> 1; o > 0; o >>= 1) sum = vadd(sum, vshfl_xor(sum, o));
    if (r < nrows && gl == 0) y[r] = sum;
  }
}

}  // namespace b2s
#include "b2s_spmv_pipe.cuh"
#include "b2s_spmv_agather.cuh"
namespace b2s {

// ------------------------------------------------------------------ host launchers
static int num_sms() {
  int dev = 0, v = kNumSMs;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
  return v > 0 ? v : kNumSMs;
}

constexpr int kMaxDevices = 64;
static int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}

static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}

template <typename V, typename I, int TILE, int STAGES, bool WINDOW, bool DOT, bool BCAST, int NG, bool LONGROWS = false>
static int launch_pipe_inst(const PlanHeader* P, const int64_t* indptr, const I* cols, const V* vals,
                            const V* x, V* y, V* dot_partials, const V* w, int64_t* npartials,
                            const PeerOut<V>& peers, int accumulate, cudaStream_t st) {
  using L = PipeLayout<V, I, TILE>;
  const size_t smem = L::stage_bytes(WINDOW) * STAGES + 16 * STAGES;
  auto kern = spmv_pipe_kernel<V, I, TILE, STAGES, WINDOW, DOT, BCAST, NG, LONGROWS>;
  // function attributes are per device: cache the largest resident-CTA count (registers / shared
  // memory with the maximum carve-out) per (instantiation, device)
  static std::atomic<int> max_blocks_per_sm[kMaxDevices];
  const int dev = current_device();
  int nb_max = max_blocks_per_sm[dev].load(std::memory_order_acquire);
  if (nb_max <= 0) {
    B2S_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B2S_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    B2S_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_max, kern, kPipeThreads, smem));
    if (nb_max < 1) { set_error("spmv_pipe_kernel does not fit on an SM (smem %zu)", smem); return B2S_ERR_CUDA; }
    B2S_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutDefault));
    max_blocks_per_sm[dev].store(nb_max, std::memory_order_release);
  }
  // Resident CTAs / ring depth / shared-memory carve-out (a per-LAUNCH attribute) of the products
  // consumer (1024-nnz tiles):
  //   3-stage ring, 3 CTAs/SM (130 KB of shared memory, carve-out 57 %, L1 = 124 KB): C2, the Laplacian
  //   2-stage ring, 3 CTAs/SM (carve-out 50 %)                                      : long-row (power-law)
  // Swept on an H100 SXM (700 W) with tools/launch_sweep.py, ms per SpMV: C2 (column-blocked)
  // 3 CTAs 4.86, 2 CTAs 4.90, 3 CTAs at 80 % 4.91, 4 CTAs at 80 % 4.94; the Laplacian 3 CTAs 0.516,
  // 4 CTAs at 80 % 0.531; the power-law matrix (long-row pass) 3 CTAs 1.707, 3 CTAs at 80 % 1.742.
  // The shallow ring leaves the long-row instances the larger L1 (= more requests in flight).
  // B2S_SPMV_CARVEOUT (percent) / B2S_SPMV_CTAS override for sweeps.
  const int l1_alloc = env_int("B2S_SPMV_L1_ALLOC", P->near_tiles * 2 >= P->ntiles ? 1 : 0) != 0;
  int carve = -1, cap = 0;
  if (!WINDOW) {
    if (LONGROWS) { cap = 3; carve = 50; }
    else          { cap = 3; carve = TILE == 1024 ? 57 : 80; }
  }
  carve = env_int("B2S_SPMV_CARVEOUT", carve);
  cap = env_int("B2S_SPMV_CTAS", cap);
  int nb = nb_max;
  if (cap >= 1 && cap < nb) nb = cap;
  int64_t grid = (int64_t)nb * num_sms();
  if (grid > P->ntiles) grid = P->ntiles;
  *npartials = grid;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kPipeThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  if (carve >= 0) {
    attr[0].id = cudaLaunchAttributePreferredSharedMemoryCarveout;
    attr[0].val.sharedMemCarveout = (unsigned)carve;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  B2S_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, P->nrows, P->ncols, P->nnz, P->ntiles, indptr, cols, vals, x, y,
                                  (const int64_t*)P->tile_row, (const int64_t*)P->tile_win,
                                  reinterpret_cast<V*>(P->head), dot_partials, w, peers,
                                  (accumulate ? 1 : 0) | (l1_alloc ? 2 : 0)));
  B2S_CHECK_LAUNCH();
  return B2S_OK;
}

// async-gather kernel (b2s_spmv_agather.cuh): plain y = A x / y += A x on 1024-nnz tiles, 4- and 8-byte values
template <typename V, typename I>
static int launch_agather_inst(const PlanHeader* P, const int64_t* indptr, const I* cols, const V* vals,
                               const V* x, V* y, int64_t* npartials, int accumulate, cudaStream_t st) {
  using L = AgLayout<V>;
  const size_t smem = L::total;
  auto kern = spmv_agather_kernel<V, I>;
  static std::atomic<int> max_blocks_per_sm[kMaxDevices];
  const int dev = current_device();
  int nb_max = max_blocks_per_sm[dev].load(std::memory_order_acquire);
  if (nb_max <= 0) {
    B2S_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B2S_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    B2S_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_max, kern, kPipeThreads, smem));
    if (nb_max < 1) { set_error("spmv_agather_kernel does not fit on an SM (smem %zu)", smem); return B2S_ERR_CUDA; }
    max_blocks_per_sm[dev].store(nb_max, std::memory_order_release);
  }
  int nb = nb_max;
  const int cap = env_int("B2S_SPMV_CTAS", 0);
  if (cap >= 1 && cap < nb) nb = cap;
  int64_t grid = (int64_t)nb * num_sms();
  if (grid > P->ntiles) grid = P->ntiles;
  *npartials = grid;
  kern<<<(unsigned)grid, kPipeThreads, smem, st>>>(P->nrows, P->ncols, P->nnz, P->ntiles, indptr, cols, vals, x, y,
                                                  (const int64_t*)P->tile_row, reinterpret_cast<V*>(P->head),
                                                  accumulate ? 1 : 0);
  B2S_CHECK_LAUNCH();
  return B2S_OK;
}

template <typename V, typename I, int TILE, bool DOT>
static int launch_pipe_tile(const PlanHeader* P, const int64_t* indptr, const I* cols, const V* vals,
                            const V* x, V* y, V* dot_partials, const V* w, int64_t* npartials,
                            const PeerOut<V>& peers, int accumulate, cudaStream_t st) {
  bool window = (P->window_tiles * 2 >= P->ntiles) && ((uintptr_t)x % 16 == 0) &&
                getenv("B2S_SPMV_NO_WINDOW") == nullptr;
  // window matrices (banded / stencil): row-walk consumer, 2-stage ring; others: products consumer
  // with two ping-pong consumer groups (1024-nnz tiles: 4-stage ring, 2048-nnz tiles: 2 stages).
  // Peer stores are compiled in only for the broadcast launches.
  const bool bcast = peers.n != 0;
#define B2S_PIPE(S, W, B, G) launch_pipe_inst<V, I, TILE, S, W, DOT, B, G>(P, indptr, cols, vals, x, y, dot_partials, w, npartials, peers, accumulate, st)
  if (window) return bcast ? B2S_PIPE(2, true, true, 1) : B2S_PIPE(2, true, false, 1);
  // skewed row lengths (power-law): a row much longer than the tile average would be summed by one
  // small lane group — give those rows a warp each in a second pass (plain SpMV instances only)
  bool longrows = P->max_row > 64 && P->max_row * P->nrows > 8 * P->nnz;
  longrows = env_int("B2S_SPMV_LONGROWS", longrows ? 1 : 0) != 0;
  if constexpr (!DOT && TILE == 1024 && sizeof(V) <= 8) {
    // the async-gather kernel (segmented sum, next tile's gathers in flight during the reduction) on
    // request only (B2S_SPMV_AGATHER=1, every gathered, non-window matrix): on an H100 the long-row
    // pass of the products consumer is faster on the power-law matrix (1.707 vs 1.762 ms).
    if (!bcast && P->max_tile_rows <= 65535 && P->nrows > 0 && (uintptr_t)x % 16 == 0 &&
        env_int("B2S_SPMV_AGATHER", 0) == 1) {
      return launch_agather_inst<V, I>(P, indptr, cols, vals, x, y, npartials, accumulate, st);
    }
  }
  if constexpr (!DOT && TILE == 1024) {
    if (longrows && !bcast)
      return launch_pipe_inst<V, I, TILE, 2, false, false, false, 2, true>(P, indptr, cols, vals, x, y, dot_partials, w,
                                                                          npartials, peers, accumulate, st);
  }
  if constexpr (TILE == 1024) return bcast ? B2S_PIPE(3, false, true, 2) : B2S_PIPE(3, false, false, 2);
  else                        return bcast ? B2S_PIPE(2, false, true, 2) : B2S_PIPE(2, false, false, 2);
#undef B2S_PIPE
}

// pipe kernel needs 16-byte aligned streams (TMA bulk copies) and a 1024/2048 tile
static bool pipe_ok(const PlanHeader* P, const void* indptr, const void* cols, const void* vals) {
  return (P->tile_nnz == 1024 || P->tile_nnz == 2048) && ((uintptr_t)cols % 16 == 0) &&
         ((uintptr_t)vals % 16 == 0) && ((uintptr_t)indptr % 16 == 0);
}

template <typename V, typename I, int IPT, bool VEC, bool WINDOW, bool DOT>
static int launch_tile_inst(const PlanHeader* P, const int64_t* indptr, const I* cols, const V* vals,
                            const V* x, V* y, V* dot_partials, const V* w, cudaStream_t st) {
  constexpr int T = kTileThreads * IPT;
  size_t smem = sizeof(V) * T + (WINDOW ? sizeof(V) * kWinCap + 16 : 0);
  auto kern = spmv_tile_kernel<V, I, IPT, VEC, WINDOW, DOT>;
  static std::atomic<int> attr_set[kMaxDevices];  // per (instantiation, device): attributes are per device
  const int dev = current_device();
  if (!attr_set[dev].load(std::memory_order_acquire)) {
    B2S_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set[dev].store(1, std::memory_order_release);
  }
  kern<<<(unsigned)P->ntiles, kTileThreads, smem, st>>>(P->nrows, P->ncols, P->nnz, indptr, cols, vals,
                                                        x, y, P->tile_row, P->tile_win,
                                                        reinterpret_cast<V*>(P->head), dot_partials, w);
  B2S_CHECK_LAUNCH();
  return B2S_OK;
}

template <typename V, typename I, int IPT, bool DOT>
static int launch_tile_ipt(const PlanHeader* P, const int64_t* indptr, const I* cols, const V* vals,
                           const V* x, V* y, V* dot_partials, const V* w, cudaStream_t st) {
  bool vec = ((uintptr_t)cols % 16 == 0) && ((uintptr_t)vals % 16 == 0);
  bool window = (P->window_tiles * 2 >= P->ntiles) && ((uintptr_t)x % 16 == 0) &&
                getenv("B2S_SPMV_NO_WINDOW") == nullptr;
  if (vec) {
    if (window) return launch_tile_inst<V, I, IPT, true, true, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st);
    return launch_tile_inst<V, I, IPT, true, false, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st);
  }
  if (window) return launch_tile_inst<V, I, IPT, false, true, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st);
  return launch_tile_inst<V, I, IPT, false, false, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st);
}

template <typename V, typename I, bool DOT>
static int run_tile(const PlanHeader* P, const int64_t* indptr, const I* cols, const V* vals,
                    const V* x, V* y, V* dot_out, V* dot_partials, const V* w, int mode,
                    const PeerOut<V>& peers, int accumulate, const BoardRaw* board, cudaStream_t st) {
  int rc;
  int64_t npartials = P->ntiles;
  if (mode == 1) {
    if (P->tile_nnz == 1024) rc = launch_pipe_tile<V, I, 1024, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, &npartials, peers, accumulate, st);
    else                     rc = launch_pipe_tile<V, I, 2048, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, &npartials, peers, accumulate, st);
  } else
  switch (P->tile_nnz) {
    case 1024: rc = launch_tile_ipt<V, I, 4, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st); break;
    case 2048: rc = launch_tile_ipt<V, I, 8, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st); break;
    case 4096: rc = launch_tile_ipt<V, I, 16, DOT>(P, indptr, cols, vals, x, y, dot_partials, w, st); break;
    default: set_error("plan has unsupported tile_nnz %lld", (long long)P->tile_nnz); return B2S_ERR_ARG;
  }
  if (rc) return rc;
  if (P->head_tiles > 0) {
    int thr = 256;
    spmv_fixup_kernel<V, DOT><<<(unsigned)ceil_div(P->ntiles, thr), thr, 0, st>>>(
        P->ntiles, P->tile_nnz, indptr, P->tile_row, reinterpret_cast<const V*>(P->head), y,
        mode == 1 ? peers : PeerOut<V>{});
    B2S_CHECK_LAUNCH();
  }
  if (DOT) {
    BoardArgs<V> bx{};
    if (board) {
      int rcb = make_board_args<V>(board->boards, board->rank, board->nranks, board->channel, board->seq_counters,
                                   board->cur_out, board->prev_out, board->err, &bx);
      if (rcb) return rcb;
    }
    reduce_partials_kernel<V><<<1, 1024, 0, st>>>(npartials, dot_partials, dot_out, bx);
    B2S_CHECK_LAUNCH();
  }
  return B2S_OK;
}

template <typename V, typename I>
static int run_rowvec(int64_t nrows, int64_t nnz, const int64_t* indptr, const I* cols, const V* vals,
                      const V* x, V* y, cudaStream_t st) {
  double mean = nrows > 0 ? (double)nnz / (double)nrows : 0.0;
  int lanes = 2;
  while (lanes < 32 && lanes * 2 <= mean) lanes <<= 1;  // ~mean/2 .. mean lanes per row
  const int threads = 256;
  int64_t groups_per_block = threads / lanes;
  int64_t blocks = ceil_div(nrows, groups_per_block);
  int64_t cap = (int64_t)kNumSMs * 8 * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
#define B2S_RV(L) spmv_rowvec_kernel<V, I, L><<<(unsigned)blocks, threads, 0, st>>>(nrows, indptr, cols, vals, x, y)
  switch (lanes) {
    case 2: B2S_RV(2); break;
    case 4: B2S_RV(4); break;
    case 8: B2S_RV(8); break;
    case 16: B2S_RV(16); break;
    default: B2S_RV(32); break;
  }
#undef B2S_RV
  B2S_CHECK_LAUNCH();
  return B2S_OK;
}

template <typename V>
__global__ void fill_zero_kernel(int64_t n, V* y) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = zero_of<V>();
}

template <typename V, typename I>
static int spmv_typed(int64_t nrows, int64_t ncols, int64_t nnz, const int64_t* indptr, const I* cols,
                      const V* vals, const V* x, V* y, const PlanHeader* P, int variant, V* dot_out,
                      V* dot_partials, const V* w, const PeerOut<V>& peers, int accumulate,
                      const BoardRaw* board, cudaStream_t st) {
  const bool want_dot = dot_out != nullptr;
  if (nrows == 0) {
    if (want_dot) { fill_zero_kernel<V><<<1, 32, 0, st>>>(1, dot_out); B2S_CHECK_LAUNCH(); }
    return B2S_OK;
  }
  if (nnz == 0) {
    if (!accumulate) {
      fill_zero_kernel<V><<<(unsigned)ceil_div(nrows, 256), 256, 0, st>>>(nrows, y);
      B2S_CHECK_LAUNCH();
    }
    if (want_dot) { fill_zero_kernel<V><<<1, 32, 0, st>>>(1, dot_out); B2S_CHECK_LAUNCH(); }
    return B2S_OK;
  }
  bool use_tile = (P != nullptr) && (variant != B2S_SPMV_ROWVEC);
  if ((variant == B2S_SPMV_TILE || variant == B2S_SPMV_PIPE) && P == nullptr) {
    set_error("B2S_SPMV_TILE / B2S_SPMV_PIPE require a plan");
    return B2S_ERR_ARG;
  }
  if (want_dot && !use_tile) {
    set_error("b2s_spmv_csr_dot requires a plan");
    return B2S_ERR_ARG;
  }
  if (use_tile) {
    if (P->nrows != nrows || P->nnz != nnz || P->ncols != ncols || P->it != it_code<I>::value) {
      set_error("plan does not match matrix (nrows/ncols/nnz/itype)");
      return B2S_ERR_ARG;
    }
    const bool tma_ok = pipe_ok(P, indptr, cols, vals);
    if (variant == B2S_SPMV_PIPE && !tma_ok) {
      set_error("B2S_SPMV_PIPE needs 16-byte aligned indptr/indices/data and a 1024/2048-nnz plan");
      return B2S_ERR_ARG;
    }
    int mode = 0;
    if (tma_ok && variant != B2S_SPMV_TILE) mode = 1;
    if (peers.n != 0 && mode != 1) {
      set_error("peer broadcast needs the pipe kernel (16-byte aligned arrays, 1024/2048-nnz plan)");
      return B2S_ERR_UNSUPPORTED;
    }
    if (accumulate && mode != 1) {
      set_error("y += A x needs the pipe kernel (16-byte aligned arrays, 1024/2048-nnz plan)");
      return B2S_ERR_UNSUPPORTED;
    }
    if (want_dot) return run_tile<V, I, true>(P, indptr, cols, vals, x, y, dot_out, dot_partials, w, mode, peers, accumulate, board, st);
    return run_tile<V, I, false>(P, indptr, cols, vals, x, y, nullptr, nullptr, nullptr, mode, peers, accumulate, nullptr, st);
  }
  if (peers.n != 0 || accumulate) {
    set_error("peer broadcast / accumulate need a plan");
    return B2S_ERR_UNSUPPORTED;
  }
  return run_rowvec<V, I>(nrows, nnz, indptr, cols, vals, x, y, st);
}

}  // namespace b2s

// =================================================================== C ABI
using namespace b2s;

extern "C" int64_t b2s_spmv_plan_workspace_bytes(int64_t nrows, int64_t nnz) {
  (void)nrows;
  if (nnz < 0) return -1;
  int64_t ntiles = ceil_div(nnz > 0 ? nnz : 1, 1024);  // smallest tile → upper bound
  // tile_row (ntiles+1) + tile_win (2*ntiles) int64, head 16 B/tile, counters, padding
  return (ntiles + 1) * 8 + ntiles * 16 + ntiles * 16 + ntiles * 16 + 64 + 1024;
}

namespace b2s {
// force_tile: 0 = automatic (env B2S_SPMV_TILE_NNZ, else 2048 with a 1024 re-plan when not window-friendly)
int plan_create_impl(b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                     const int64_t* indptr, const void* indices, void* workspace,
                     int64_t workspace_bytes, b2s_stream_t stream, int64_t force_tile,
                     b2s_spmv_plan** out_plan) {
  B2S_REQUIRE(out_plan != nullptr, "out_plan is null");
  *out_plan = nullptr;
  B2S_REQUIRE(nrows >= 0 && ncols >= 0 && nnz >= 0, "negative size");
  B2S_REQUIRE(it == B2S_I32 || it == B2S_I64, "bad itype");
  B2S_REQUIRE(nnz == 0 || (indptr && indices), "null matrix arrays");
  B2S_REQUIRE(workspace != nullptr, "null workspace");
  if (workspace_bytes < b2s_spmv_plan_workspace_bytes(nrows, nnz)) {
    set_error("plan workspace too small: %lld < %lld", (long long)workspace_bytes,
              (long long)b2s_spmv_plan_workspace_bytes(nrows, nnz));
    return B2S_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  auto* P = new b2s_spmv_plan();
  P->it = it; P->nrows = nrows; P->ncols = ncols; P->nnz = nnz;
  // Tile size: an explicit B2S_SPMV_TILE_NNZ wins; otherwise plan with 2048-nnz tiles first and,
  // when the matrix is not window-friendly (x gathers must go to L2), re-plan with 1024-nnz tiles
  // (the configuration each consumer flavour measured fastest with).
  const bool forced = getenv("B2S_SPMV_TILE_NNZ") != nullptr || force_tile > 0;
  int64_t candidates[2] = {getenv("B2S_SPMV_TILE_NNZ") ? default_tile_nnz() : (force_tile > 0 ? force_tile : 2048), 1024};
  for (int attempt = 0; attempt < 2; ++attempt) {
    P->tile_nnz = candidates[attempt];
    P->ntiles = ceil_div(nnz, P->tile_nnz);
    P->window_tiles = 0; P->head_tiles = 0;
    // carve workspace (256-byte aligned base assumed from the caller's allocator; align anyway)
    uintptr_t base = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
    int64_t nt = P->ntiles;
    P->counters = reinterpret_cast<int64_t*>(base);               base += 64;
    P->tile_row = reinterpret_cast<int64_t*>(base);               base += (nt + 1) * 8;
    base = (base + 15) & ~(uintptr_t)15;
    P->tile_win = reinterpret_cast<int64_t*>(base);               base += nt * 16;
    P->head = reinterpret_cast<void*>(base);                      base += nt * 16;
    P->dotp = reinterpret_cast<void*>(base);                      base += nt * 16;
    P->empty_rows = 0; P->max_row = 0; P->near_tiles = 0; P->max_tile_rows = 0;
    if (nt == 0) break;
    cudaError_t e = cudaMemsetAsync(P->counters, 0, 64, st);
    if (e != cudaSuccess) { delete P; set_error("memset failed: %s", cudaGetErrorString(e)); return B2S_ERR_CUDA; }
    plan_tile_rows_kernel<<<(unsigned)ceil_div(nt + 1, 256), 256, 0, st>>>(nrows, nt, P->tile_nnz, indptr,
                                                                          P->tile_row);
    g_launch_count.fetch_add(1);
    if (it == B2S_I32)
      plan_tile_window_kernel<int32_t><<<(unsigned)nt, 128, 0, st>>>(nnz, nt, P->tile_nnz, indptr,
          (const int32_t*)indices, P->tile_row, P->tile_win, P->counters);
    else
      plan_tile_window_kernel<int64_t><<<(unsigned)nt, 128, 0, st>>>(nnz, nt, P->tile_nnz, indptr,
          (const int64_t*)indices, P->tile_row, P->tile_win, P->counters);
    g_launch_count.fetch_add(1);
    {
      int64_t blocks = ceil_div(nrows, 256);
      if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
      if (blocks < 1) blocks = 1;
      plan_count_empty_kernel<<<(unsigned)blocks, 256, 0, st>>>(nrows, indptr, P->counters);
      g_launch_count.fetch_add(1);
    }
    int64_t h[6] = {0, 0, 0, 0, 0, 0};
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(h, P->counters, 48, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { delete P; set_error("plan build failed: %s", cudaGetErrorString(e)); return B2S_ERR_CUDA; }
    P->window_tiles = h[0];
    P->head_tiles = h[1];
    P->empty_rows = h[2];
    P->max_row = h[3];
    P->near_tiles = h[4];
    P->max_tile_rows = h[5];
    if (forced || P->window_tiles * 2 >= P->ntiles) break;   // keep this tiling
  }
  *out_plan = P;
  return B2S_OK;
}
}  // namespace b2s

extern "C" int b2s_spmv_plan_create(b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                                    const int64_t* indptr, const void* indices, void* workspace,
                                    int64_t workspace_bytes, b2s_stream_t stream,
                                    b2s_spmv_plan** out_plan) {
  return plan_create_impl(it, nrows, ncols, nnz, indptr, indices, workspace, workspace_bytes, stream, 0,
                          out_plan);
}

extern "C" void b2s_spmv_plan_destroy(b2s_spmv_plan* plan) { delete plan; }

extern "C" int b2s_spmv_plan_info(const b2s_spmv_plan* plan, int64_t* ntiles, int64_t* tile_nnz,
                                  int64_t* window_tiles) {
  B2S_REQUIRE(plan != nullptr, "plan is null");
  if (ntiles) *ntiles = plan->ntiles;
  if (tile_nnz) *tile_nnz = plan->tile_nnz;
  if (window_tiles) *window_tiles = plan->window_tiles;
  return B2S_OK;
}

namespace b2s {
int spmv_entry(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
               const int64_t* indptr, const void* indices, const void* data, const void* x,
               void* y, const b2s_spmv_plan* plan, int variant, void* dot_out, void* partials,
               const void* w, void* const* y_peers, int npeers, int accumulate, b2s_stream_t stream,
               const BoardRaw* board) {
  B2S_REQUIRE(npeers >= -1 && npeers <= kMaxPeers, "npeers must be in [-1,7]");
  B2S_REQUIRE(npeers == 0 || y_peers != nullptr, "y_peers is null");
  B2S_REQUIRE(nrows >= 0 && ncols >= 0 && nnz >= 0, "negative size");
  B2S_REQUIRE(nrows == 0 || y != nullptr, "y is null");
  B2S_REQUIRE(nrows == 0 || indptr != nullptr, "indptr is null");
  B2S_REQUIRE(nnz == 0 || (indices && data && x), "null matrix/vector arrays");
  B2S_REQUIRE(variant >= B2S_SPMV_AUTO && variant <= B2S_SPMV_PIPE, "bad variant");
  cudaStream_t st = (cudaStream_t)stream;
  B2S_DISPATCH_VT(vt, V, {
    PeerOut<V> peers{};
    peers.n = npeers;
    for (int g = 0; g < (npeers < 0 ? 1 : npeers); ++g) peers.p[g] = (V*)y_peers[g];
    B2S_DISPATCH_IT(it, I,
      return spmv_typed<V, I>(nrows, ncols, nnz, indptr, (const I*)indices, (const V*)data,
                              (const V*)x, (V*)y, plan, variant, (V*)dot_out, (V*)partials, (const V*)w,
                              peers, accumulate, board, st));
  });
  return B2S_ERR_ARG;
}
void* plan_dot_partials(const b2s_spmv_plan* plan) { return plan->dotp; }
}  // namespace b2s

extern "C" int b2s_spmv_csr(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                            const int64_t* indptr, const void* indices, const void* data,
                            const void* x, void* y, const b2s_spmv_plan* plan, int variant,
                            b2s_stream_t stream) {
  return spmv_entry(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y, plan, variant, nullptr,
                    nullptr, nullptr, nullptr, 0, 0, stream);
}

extern "C" int b2s_spmv_csr_bcast(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                                  const int64_t* indptr, const void* indices, const void* data,
                                  const void* x, void* y, void* const* y_peers, int npeers,
                                  const b2s_spmv_plan* plan, b2s_stream_t stream) {
  B2S_REQUIRE(plan != nullptr, "broadcast SpMV needs a plan");
  return spmv_entry(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y, plan, B2S_SPMV_AUTO, nullptr,
                    nullptr, nullptr, y_peers, npeers, 0, stream);
}

// b2s_spmv_csr_dot whose w.y is summed over the ranks inside the final reduction kernel (board
// exchange, see b2s_allreduce_board): dot_out[0] = sum over ranks of this rank's sum_r w[r] y[r].
extern "C" int b2s_spmv_csr_dot_allreduce(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                                          const int64_t* indptr, const void* indices, const void* data,
                                          const void* x, void* y, const void* w, const b2s_spmv_plan* plan,
                                          void* dot_out, void* const* boards, int rank, int nranks, int channel,
                                          void* seq_counters, void* err, b2s_stream_t stream) {
  B2S_REQUIRE(dot_out != nullptr, "dot_out null");
  B2S_REQUIRE(nrows == 0 || w != nullptr, "w null");
  B2S_REQUIRE(plan != nullptr, "fused dot needs a plan");
  B2S_REQUIRE(boards != nullptr && nranks >= 2, "b2s_spmv_csr_dot_allreduce needs boards of >= 2 ranks");
  BoardRaw br{boards, rank, nranks, channel, seq_counters, nullptr, nullptr, err};
  return spmv_entry(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y, plan, B2S_SPMV_AUTO,
                    dot_out, plan->dotp, w, nullptr, 0, 0, stream, &br);
}

extern "C" int b2s_spmv_csr_dot(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
                                const int64_t* indptr, const void* indices, const void* data,
                                const void* x, void* y, const void* w, const b2s_spmv_plan* plan,
                                void* dot_out, b2s_stream_t stream) {
  B2S_REQUIRE(dot_out != nullptr, "dot_out null");
  B2S_REQUIRE(nrows == 0 || w != nullptr, "w null");
  B2S_REQUIRE(plan != nullptr, "fused dot needs a plan");
  return spmv_entry(vt, it, nrows, ncols, nnz, indptr, indices, data, x, y, plan, B2S_SPMV_AUTO,
                    dot_out, plan->dotp, w, nullptr, 0, 0, stream);
}

#ifdef B2S_PIPE_TIMING
// debug builds only: read and clear the phase cycle counters of the pipe kernel
extern "C" int b2s_debug_pipe_phases(unsigned long long* out16) {
  cudaDeviceSynchronize();
  if (cudaMemcpyFromSymbol(out16, b2s::g_pipe_phase, sizeof(unsigned long long) * 16) != cudaSuccess) return 1;
  unsigned long long z[16] = {0};
  cudaMemcpyToSymbol(b2s::g_pipe_phase, z, sizeof z);
  return 0;
}
#endif
