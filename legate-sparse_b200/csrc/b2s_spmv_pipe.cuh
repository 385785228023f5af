// b2s_spmv_pipe.cuh — persistent, warp-specialised, TMA-fed CSR SpMV (the default kernel).
//
// Included by b2s_spmv.cu.  Same tiling / ownership rules as spmv_tile_kernel (nnz-balanced
// tiles from the plan; the tile where a row starts owns y[r]; later pieces go to head[t] and
// are added by spmv_fixup_kernel in tile order), different execution structure:
//
//   * persistent CTAs (grid = resident CTAs per SM x number of SMs), tiles handed out round-robin;
//   * one PRODUCER warp: an elected lane fills a STAGES-deep shared-memory ring with TMA bulk
//     copies (cp.async.bulk … mbarrier::complete_tx, SASS UBLKCP) of the tile's contiguous
//     slices: col indices, values, the indptr entries of the tile's rows and — when the plan
//     says the tile's [min col, max col] image is small (banded / stencil matrices; the
//     reference's image(crd→x, MIN_MAX), csr.py:591) — the x window itself.  The streams never
//     touch the LSU/L1TEX path or the register file, so that path is left to the x gathers;
//   * 8 CONSUMER warps, two flavours (chosen per matrix, see spmv_pipe_kernel):
//       row-walk  (window matrices): a group of 1..32 lanes owns one row of the staged tile, walks
//                 its (col,val) pairs in shared memory, reads x from the staged window, accumulates
//                 in registers, shuffle-reduces in a fixed order and writes y.  No CTA-wide barrier.
//       products  (x gathered from L2): the consumers form NG independent groups of 256/NG threads
//                 that take the CTA's tiles in turn (tile i: group i mod 2, ring stage i mod 3), so that
//                 one group's gather phase overlaps the other's reduction phase.  Every thread issues
//                 all of its gathers at once for 16-byte chunks of the staged (col,val) slices
//                 (conflict-free LDS/STS), parks the products in place, and after the group's named
//                 barrier the rows are reduced out of shared memory by 1..32 lanes per row.
//     No floating-point atomics anywhere: results are bit-reproducible.
#pragma once

namespace b2s {

#ifdef B2S_PIPE_TIMING
// phase cycle counters of consumer group 0 / thread 0 of CTA 0 (debug builds with -DB2S_PIPE_TIMING only)
__device__ unsigned long long g_pipe_phase[16];
#define B2S_T(k) do { if (blockIdx.x == 0 && tid == 0) { const long long _n = clock64(); g_pipe_phase[k] += (unsigned long long)(_n - _tprev); _tprev = _n; } } while (0)
#else
#define B2S_T(k) do { } while (0)
#endif

#ifndef B2S_LONGROW_FACTOR
#define B2S_LONGROW_FACTOR 32
#endif
constexpr int kLongRowFactor = B2S_LONGROW_FACTOR;   // rows longer than this x (lanes per row) get a warp of their own
constexpr int kPipeConsumers = 256;
constexpr int kPipeThreads   = kPipeConsumers + 32;
constexpr int kPipeWinCap    = 1024;  // x-window capacity per stage (elements)

struct PipeMeta {  // written by the producer before it arms the full barrier
  int64_t r_begin, r_last;   // rows touched by the tile (r_last may be the sentinel nrows)
  int64_t ra;                // first indptr entry staged in shared memory
  int64_t wbase;             // first x element staged (0 if none)
  int32_t rows_staged;       // 1: indptr entries [ra, …] are in shared memory
  int32_t win_staged;        // 1: x window is in shared memory
  int32_t full_tile;         // 1: (col,val) slices are in shared memory
  int32_t pad;
};

template <typename V, typename I, int TILE>
struct PipeLayout {
  static constexpr int T = TILE;
  static constexpr int RCAP = T / 4 + 4;            // indptr entries per stage
  static constexpr size_t vals_off = 0;
  static constexpr size_t cols_off = vals_off + sizeof(V) * T;
  static constexpr size_t rptr_off = (cols_off + sizeof(I) * T + 15) / 16 * 16;
  static constexpr size_t meta_off = rptr_off + 8 * RCAP;
  static constexpr size_t xwin_off = (meta_off + sizeof(PipeMeta) + 15) / 16 * 16;
  __host__ __device__ static constexpr size_t stage_bytes(bool window) {
    return (xwin_off + (window ? sizeof(V) * (kPipeWinCap + 4) : 0) + 127) / 128 * 128;
  }
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void consumer_bar_sync() {   // all consumer warps (not the producer)
  asm volatile("bar.sync 1, %0;" ::"n"(kPipeConsumers) : "memory");
}
template <int GT>
__device__ __forceinline__ void group_bar_sync(int grp) {   // one consumer group of GT threads
  asm volatile("bar.sync %0, %1;" ::"r"(2 + grp), "n"(GT) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  // generic-proxy accesses to a stage (product stores, reads) before the async proxy (TMA) refills it
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// lanes per row of a tile with nr candidate rows handled by gt threads
__device__ __forceinline__ int lanes_for(int64_t nr, int gt) {
  int lanes = 1;
  while (lanes < 32 && (int64_t)(lanes * 2) * nr <= gt) lanes <<= 1;
  return lanes;
}
template <typename V, int C> struct alignas(16) VChunk { V v[C]; };
template <typename I, int C> struct alignas((sizeof(I) * C) < 16 ? (sizeof(I) * C) : 16) IChunk { I c[C]; };

// WINDOW also selects the consumer: window matrices (banded / stencil) use the row-walk consumer,
// all others the products consumer (each measured fastest there; the cross combinations were never
// faster and are not instantiated).  BCAST compiles the peer stores in; the plain instances carry
// no trace of them (as a runtime branch the peer ranges slowed the banded kernel).
// NG = consumer groups of the products consumer (1 or 2; tile i of the CTA uses ring stage i % STAGES and
// is consumed by group i % NG, whose GT threads are the arrivals its "empty" barrier expects).
// LONGROWS (products consumer, skewed row lengths — power-law matrices): rows of the tile longer than
// 32 x (lanes per row) are not summed by their small lane group (one lane walking a 1000-entry row
// stalls its whole group at the next barrier) but
// deferred to a second pass where each gets a full warp.
template <typename V, typename I, int TILE, int STAGES, bool WINDOW, bool DOT, bool BCAST, int NG, bool LONGROWS = false>
__global__ void __launch_bounds__(kPipeThreads, (WINDOW || sizeof(V) > 8) ? 0 : (LONGROWS ? 3 : 4))   // products: 4 (long rows: 3) CTAs/SM must fit the register file
spmv_pipe_kernel(int64_t nrows, int64_t ncols, int64_t nnz, int64_t ntiles,
                 const int64_t* __restrict__ indptr, const I* __restrict__ cols,
                 const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y,
                 const int64_t* __restrict__ tile_row, const int64_t* __restrict__ tile_win,
                 V* __restrict__ head, V* __restrict__ dot_partials, const V* __restrict__ w,
                 const PeerOut<V> peers, const int flags) {
  const int accumulate = flags & 1;        // y += A x (later column blocks)
  const bool l1_alloc  = (flags & 2) != 0; // products consumer: gathers allocate in L1 (matrices whose
                                           // tiles re-touch a small x range, e.g. wide-band stencils)
  using L = PipeLayout<V, I, TILE>;
  constexpr int T = L::T;
  constexpr bool ROWWALK = WINDOW;
  constexpr int GT = kPipeConsumers / NG;          // threads per consumer group
  static_assert(STAGES >= NG && (NG == 1 || !WINDOW), "bad consumer grouping");
  constexpr size_t STAGE = L::stage_bytes(WINDOW);
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full_bar  = reinterpret_cast<uint64_t*>(smem + STAGE * STAGES);
  uint64_t* empty_bar = full_bar + STAGES;
  __shared__ V wsum[kPipeConsumers / 32];  // DOT only
  constexpr int LRCAP = LONGROWS ? TILE / kLongRowFactor + 2 : 1;
  __shared__ int lr_count[NG][3];
  __shared__ int lr_list[NG][3][LRCAP];     // deferred rows (index inside the tile), per group; 3 slots in rotation

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], ROWWALK ? kPipeConsumers : GT); }
    fence_mbar_init();
    for (int g = 0; g < NG; ++g) { lr_count[g][0] = 0; lr_count[g][1] = 0; lr_count[g][2] = 0; }
  }
  __syncthreads();

  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep   = policy_evict_last();

  if (tid >= kPipeConsumers) {
    // ============================== PRODUCER (one elected lane) ==============================
    if (tid == kPipeConsumers) {
      int64_t i = 0;
      for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++i) {
        const int s = (int)(i % STAGES);
        const uint32_t ph = (uint32_t)((i / STAGES) & 1);
        mbar_wait(&empty_bar[s], ph ^ 1u);
        fence_proxy_async_smem();
        unsigned char* st = smem + STAGE * s;
        PipeMeta* meta = reinterpret_cast<PipeMeta*>(st + L::meta_off);
        const int64_t S = t * (int64_t)T;
        const int64_t E = min(S + (int64_t)T, nnz);
        const int64_t r_begin = tile_row[t], r_last = tile_row[t + 1];
        uint32_t tx = 0;
        // rows: indptr[ra .. e] with ra even (16-byte aligned source)
        const int64_t e  = min(r_last, nrows - 1) + 1;   // last indptr entry needed
        const int64_t ra = r_begin & ~(int64_t)1;
        int64_t n_ent = e - ra + 1;
        n_ent += (n_ent & 1);
        const bool rows_ok = (n_ent <= L::RCAP) && (ra + n_ent <= nrows + 1);
        const bool full = (E - S) == T;
        int64_t wbase = 0, wcnt = 0;
        bool win_ok = false;
        uint32_t win_bytes = 0;
        if (WINDOW) {
          wbase = tile_win[2 * t];
          wcnt  = tile_win[2 * t + 1];
          if (wcnt > 0 && wcnt <= kPipeWinCap) {
            constexpr int PER16 = (16 / (int)sizeof(V)) > 0 ? (16 / (int)sizeof(V)) : 1;
            int64_t want = (wcnt + PER16 - 1) / PER16 * PER16;
            if (wbase + want <= ncols) { win_ok = true; win_bytes = (uint32_t)(want * sizeof(V)); }
          }
        }
        meta->r_begin = r_begin; meta->r_last = r_last; meta->ra = ra; meta->wbase = wbase;
        meta->rows_staged = rows_ok; meta->win_staged = win_ok; meta->full_tile = full;
        if (full) tx += (uint32_t)(T * (sizeof(I) + sizeof(V)));
        if (rows_ok) tx += (uint32_t)(n_ent * 8);
        tx += win_bytes;
        if (tx > 0) {
          mbar_arrive_expect_tx(&full_bar[s], tx);
          if (full) {
            tma_bulk_g2s(st + L::vals_off, vals + S, (uint32_t)(T * sizeof(V)), &full_bar[s], pol_stream);
            tma_bulk_g2s(st + L::cols_off, cols + S, (uint32_t)(T * sizeof(I)), &full_bar[s], pol_stream);
          }
          if (rows_ok) tma_bulk_g2s(st + L::rptr_off, indptr + ra, (uint32_t)(n_ent * 8), &full_bar[s], pol_stream);
          if (win_ok) tma_bulk_g2s(st + L::xwin_off, x + wbase, win_bytes, &full_bar[s], pol_keep);
        } else {
          mbar_arrive(&full_bar[s]);
        }
      }
    }
    return;
  }

  // ================================== CONSUMERS ==================================
  if constexpr (!ROWWALK) {
    // "products" consumer (matrices whose x gathers go to L2).  Group `grp` owns the CTA's tiles
    // i = grp, grp+NG, ... (ring stage i % STAGES).  Per tile: every thread issues ALL its gathers
    // at once (nnz-balanced, maximal memory-level parallelism) for NCH chunks of 16 bytes of values,
    // parks the products in place, and after the group's named barrier the tile's rows are reduced
    // by 1..32 lanes per row out of shared memory.
    constexpr int C   = (16 / (int)sizeof(V)) > 0 ? (16 / (int)sizeof(V)) : 1;   // values per 16-byte chunk
    constexpr int NCH = T / (GT * C);                                           // chunks per thread
    static_assert(NCH * GT * C == T, "tile size must be a multiple of the group's chunk footprint");
    using VC = VChunk<V, C>;
    using IC = IChunk<I, C>;
    const int grp = tid / GT, gtid = tid % GT;
    V dot_acc = zero_of<V>();
    // y += A_b x (later column blocks): the old y of this thread's first row is fetched ONE TILE
    // AHEAD (the rows of the next tile are known from the plan), so that its DRAM latency never
    // sits in front of a store
    // two-step software pipeline: the row range of the tile AFTER next is fetched from the plan while
    // the current tile runs, so the address of next tile's y is ready when its load is issued (the
    // dependent tile_row -> y chain used to cost ~500 exposed cycles per tile in block >= 1 launches)
    const int64_t tstride = (int64_t)NG * gridDim.x;
    auto rows_of = [&](int64_t tn, int64_t* rb, int64_t* rl) {
      if (accumulate && tn < ntiles) { *rb = tile_row[tn]; *rl = tile_row[tn + 1]; }
      else { *rb = 0; *rl = -1; }
    };
    auto fetch_y = [&](int64_t rb, int64_t rl) -> V {
      const int64_t nrn = rl - rb + 1;
      if (!accumulate || nrn <= 0) return zero_of<V>();
      const int ln = lanes_for(nrn, GT);
      const int64_t slot = gtid / ln;
      if ((gtid & (ln - 1)) == 0 && slot < nrn && rb + slot < nrows) return y[rb + slot];
      return zero_of<V>();
    };
    const int64_t tfirst = (int64_t)blockIdx.x + (int64_t)grp * gridDim.x;
    int64_t rb1, rl1, rb2, rl2;            // row ranges of the next tile and of the one after it
    rows_of(tfirst, &rb1, &rl1);
    V ynext = fetch_y(rb1, rl1);
    rows_of(tfirst + tstride, &rb1, &rl1);
#ifdef B2S_PIPE_TIMING
    long long _tprev = clock64();
#endif
    for (int64_t i = grp; ; i += NG) {
      const int64_t t = (int64_t)blockIdx.x + i * (int64_t)gridDim.x;
      if (t >= ntiles) break;
      const V ypre = ynext;
      rows_of(t + 2 * tstride, &rb2, &rl2);    // plan entries of the tile after next (consumed next iteration)
      ynext = fetch_y(rb1, rl1);                // old y of the next tile's rows (address known since last iteration)
      const int s = (int)(i % STAGES);
      const uint32_t ph = (uint32_t)((i / STAGES) & 1);
      B2S_T(0);
      mbar_wait(&full_bar[s], ph);
      B2S_T(1);
      unsigned char* st = smem + STAGE * s;
      V* svals = reinterpret_cast<V*>(st + L::vals_off);
      const I* scols = reinterpret_cast<const I*>(st + L::cols_off);
      const int64_t* srptr = reinterpret_cast<const int64_t*>(st + L::rptr_off);
      const PipeMeta meta = *reinterpret_cast<const PipeMeta*>(st + L::meta_off);
      const int64_t S = t * (int64_t)T;
      const int64_t E = min(S + (int64_t)T, nnz);
      const int64_t r_begin = meta.r_begin, r_last = meta.r_last;
      const int64_t nr = r_last - r_begin + 1;
      const int lanes = lanes_for(nr, GT);
      const int groups = GT / lanes;
      const int gl = gtid & (lanes - 1);
      const int slot = (int)((i / NG) % 3);
      if constexpr (LONGROWS) {
        // rows longer than 32 x lanes go on the tile's long-row list NOW (the row pointers are
        // already staged): the group barrier after the products then covers the list as well
        if (lanes < 32 && gl == 0) {
          for (int64_t base = 0; base < nr; base += groups) {
            const int64_t r = r_begin + base + gtid / lanes;
            if (base + gtid / lanes < nr && r < nrows) {
              int64_t lo_g, hi_g;
              if (meta.rows_staged) { lo_g = srptr[r - meta.ra]; hi_g = srptr[r - meta.ra + 1]; }
              else                  { lo_g = indptr[r];          hi_g = indptr[r + 1]; }
              if (min(hi_g, E) - max(lo_g, S) > kLongRowFactor * lanes)
                lr_list[grp][slot][atomicAdd(&lr_count[grp][slot], 1)] = (int)(base + gtid / lanes);
            }
          }
        }
      }
      B2S_T(2);
      if (meta.full_tile) {
        // Gathers are issued in batches of BCH chunks = 4 gathers per thread (fastest of 2 / 4 / 8 on
        // the column-blocked C2 matrix), with L1::no_allocate: random gathers almost never hit L1,
        // so a line per outstanding request buys nothing.  Matrices whose tiles keep re-touching a
        // small range of x (the 4096^2 Laplacian: 8 K elements per tile) want the opposite, so the
        // plan's "near tiles" statistic selects the allocating load for them (flag bit 1).
        constexpr int BCH = (4 / C) > 0 ? ((4 / C) < NCH ? (4 / C) : NCH) : 1;
        static_assert(NCH % BCH == 0, "chunks per thread must be a multiple of the gather batch");
#pragma unroll
        for (int k = 0; k < NCH; k += BCH) {
          IC pc[BCH];
          VC pv[BCH];
          V xv[BCH][C];
#pragma unroll
          for (int u = 0; u < BCH; ++u) {
            const int e = ((k + u) * GT + gtid) * C;
            pc[u] = *reinterpret_cast<const IC*>(scols + e);   // LDS.64 / LDS.128, conflict-free
            pv[u] = *reinterpret_cast<const VC*>(svals + e);   // LDS.128, conflict-free
          }
          if (l1_alloc) {
#pragma unroll
            for (int u = 0; u < BCH; ++u)
#pragma unroll
              for (int j = 0; j < C; ++j) xv[u][j] = ld_gather<V>(x + (int64_t)pc[u].c[j], pol_keep);
          } else {
#pragma unroll
            for (int u = 0; u < BCH; ++u)
#pragma unroll
              for (int j = 0; j < C; ++j) xv[u][j] = ld_gather_na<V>(x + (int64_t)pc[u].c[j], pol_keep);
          }
#pragma unroll
          for (int u = 0; u < BCH; ++u) {
#pragma unroll
            for (int j = 0; j < C; ++j) pv[u].v[j] = vmul(pv[u].v[j], xv[u][j]);
            *reinterpret_cast<VC*>(svals + ((k + u) * GT + gtid) * C) = pv[u];   // STS.128, conflict-free
          }
          asm volatile("" ::: "memory");   // keep the batches apart (the compiler would merge them)
        }
      } else {
        for (int64_t p = S + gtid; p < E; p += GT) {
          int64_t c = (int64_t)ld_stream<I>(cols + p, pol_stream);
          V a = ld_stream<V>(vals + p, pol_stream);
          svals[p - S] = vmul(a, ld_gather_na<V>(x + c, pol_keep));
        }
      }
      B2S_T(3);
      if constexpr (NG == 1) consumer_bar_sync(); else group_bar_sync<GT>(grp);
      B2S_T(4);
      // slot of the group's PREVIOUS tile = slot of its tile after next: every warp has left the
      // previous tile (it is past this barrier), and nobody appends for the tile after next before
      // the NEXT barrier, which this thread reaches only after this store
      if (LONGROWS && gtid == 0) lr_count[grp][(slot + 2) % 3] = 0;
      auto finish_row = [&](int64_t r, int64_t lo_g, V sum, V yold) {
        bool wrote = false;
        if (lo_g < S) { head[t] = sum; wrote = true; }
        else if (r < r_last || lo_g < E) {
          if (accumulate) sum = vadd(sum, yold);   // y += A_b x : later column blocks
          if constexpr (BCAST) store_bcast(y, peers, r, sum);
          else if (l1_alloc) y[r] = sum;                        // the next kernel (CG) re-reads y: let it stay in L2
          else st_stream<V>(y + r, sum, pol_stream);            // gather-bound class: y must not displace x in L2
          wrote = true;
        }
        if (DOT && wrote) dot_acc = vfma(w[r], sum, dot_acc);
      };
      for (int64_t base = 0; base < nr; base += groups) {
        const int64_t r = r_begin + base + gtid / lanes;
        const bool valid = (base + gtid / lanes < nr) && (r < nrows);
        int64_t lo_g = 0, hi_g = 0;
        if (valid) {
          if (meta.rows_staged) { lo_g = srptr[r - meta.ra]; hi_g = srptr[r - meta.ra + 1]; }
          else                  { lo_g = indptr[r];          hi_g = indptr[r + 1]; }
        }
        const int lo = (int)(max(lo_g, S) - S);
        int hi = (int)(min(hi_g, E) - S);
        bool defer = false;
        if (LONGROWS && lanes < 32 && hi - lo > kLongRowFactor * lanes) {   // uniform over the lane group; on the list already
          defer = true;
          hi = lo;   // nothing to add here; every lane still takes part in the shuffles below
        }
        V s0 = zero_of<V>(), s1 = zero_of<V>();
        int p = lo + gl;
        for (; p + 3 * lanes < hi; p += 4 * lanes) {   // 4 loads in flight, 2 accumulators
          const V a0 = svals[p], a1 = svals[p + lanes], a2 = svals[p + 2 * lanes], a3 = svals[p + 3 * lanes];
          s0 = vadd(s0, vadd(a0, a2));
          s1 = vadd(s1, vadd(a1, a3));
        }
        for (; p < hi; p += lanes) s0 = vadd(s0, svals[p]);
        const V sum = group_reduce(vadd(s0, s1), lanes);
        if (valid && gl == 0 && !defer) finish_row(r, lo_g, sum, (accumulate && base != 0) ? y[r] : ypre);
      }
      B2S_T(5);
      if constexpr (LONGROWS) {
        const int nlong = lr_count[grp][slot];   // complete since the barrier above
        const int wid = gtid >> 5, lane = gtid & 31;
        for (int e = wid; e < nlong; e += GT / 32) {
          const int64_t r = r_begin + lr_list[grp][slot][e];
          int64_t lo_g, hi_g;
          if (meta.rows_staged) { lo_g = srptr[r - meta.ra]; hi_g = srptr[r - meta.ra + 1]; }
          else                  { lo_g = indptr[r];          hi_g = indptr[r + 1]; }
          const int lo = (int)(max(lo_g, S) - S), hi = (int)(min(hi_g, E) - S);
          V s0 = zero_of<V>(), s1 = zero_of<V>();
          int p = lo + lane;
          for (; p + 96 < hi; p += 128) {
            const V a0 = svals[p], a1 = svals[p + 32], a2 = svals[p + 64], a3 = svals[p + 96];
            s0 = vadd(s0, vadd(a0, a2));
            s1 = vadd(s1, vadd(a1, a3));
          }
          for (; p < hi; p += 32) s0 = vadd(s0, svals[p]);
          const V sum = group_reduce(vadd(s0, s1), 32);
          if (lane == 0) finish_row(r, lo_g, sum, accumulate ? y[r] : zero_of<V>());
        }
      }
      B2S_T(6);
      rb1 = rb2; rl1 = rl2;   // rotate at the END of the tile: the plan loads issued at its top have landed
      // the product stores above are generic-proxy writes to memory the TMA refills later: the
      // cross-proxy fence is issued ONCE, by the producer, after it has acquired this arrival
      // (fence.proxy.async = MEMBAR.ALL.CTA + FENCE.VIEW.ASYNC: measurable when all 256 consumer
      // threads executed it per tile)
      mbar_arrive(&empty_bar[s]);
    }
    if (DOT) {
      V sacc = dot_acc;
      for (int o = 16; o > 0; o >>= 1) sacc = vadd(sacc, vshfl_xor(sacc, o));
      if ((tid & 31) == 0) wsum[tid >> 5] = sacc;
      consumer_bar_sync();
      if (tid == 0) {
        V tot = wsum[0];
        for (int k = 1; k < kPipeConsumers / 32; ++k) tot = vadd(tot, wsum[k]);
        dot_partials[blockIdx.x] = tot;
      }
    }
    return;
  }
  // Row-walk straight out of the staged tile: a group of `lanes` threads owns one row of the
  // tile, walks its (col,val) pairs in shared memory, gathers x and accumulates in registers.
  // No product round-trip through shared memory and NO CTA-wide barrier per tile: a thread
  // that is done with its row(s) releases the stage and moves on to the next tile, so gathers
  // of different tiles overlap naturally.
  int64_t i = 0;
  V dot_acc = zero_of<V>();
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++i) {
    const int s = (int)(i % STAGES);
    const uint32_t ph = (uint32_t)((i / STAGES) & 1);
    mbar_wait(&full_bar[s], ph);
    unsigned char* st = smem + STAGE * s;
    const V* svals = reinterpret_cast<const V*>(st + L::vals_off);
    const I* scols = reinterpret_cast<const I*>(st + L::cols_off);
    const int64_t* srptr = reinterpret_cast<const int64_t*>(st + L::rptr_off);
    const V* sxwin = reinterpret_cast<const V*>(st + L::xwin_off);
    const PipeMeta meta = *reinterpret_cast<const PipeMeta*>(st + L::meta_off);
    const int64_t S = t * (int64_t)T;
    const int64_t E = min(S + (int64_t)T, nnz);
    const bool use_win = WINDOW && meta.win_staged;
    const bool staged = meta.full_tile;

    const int64_t r_begin = meta.r_begin, r_last = meta.r_last;
    const int64_t nr = r_last - r_begin + 1;
    int lanes = 1;
    while (lanes < 32 && (int64_t)(lanes * 2) * nr <= kPipeConsumers) lanes <<= 1;
    const int groups = kPipeConsumers / lanes;
    const int gl = tid & (lanes - 1);
    for (int64_t base = 0; base < nr; base += groups) {
      const int64_t r = r_begin + base + tid / lanes;
      const bool valid = (base + tid / lanes < nr) && (r < nrows);
      int64_t lo_g = 0, hi_g = 0;
      if (valid) {
        if (meta.rows_staged) { lo_g = srptr[r - meta.ra]; hi_g = srptr[r - meta.ra + 1]; }
        else                  { lo_g = indptr[r];          hi_g = indptr[r + 1]; }
      }
      const int64_t lo = max(lo_g, S), hi = min(hi_g, E);
      V sum = zero_of<V>();
      int64_t p = lo + gl;
      if (staged) {
        // 4 independent gathers in flight per thread
        for (; p + 3 * lanes < hi; p += 4 * lanes) {
          const int q0 = (int)(p - S), q1 = q0 + lanes, q2 = q1 + lanes, q3 = q2 + lanes;
          const int64_t c0 = (int64_t)scols[q0], c1 = (int64_t)scols[q1], c2 = (int64_t)scols[q2],
                        c3 = (int64_t)scols[q3];
          V x0, x1, x2, x3;
          if (use_win) {
            x0 = sxwin[c0 - meta.wbase]; x1 = sxwin[c1 - meta.wbase];
            x2 = sxwin[c2 - meta.wbase]; x3 = sxwin[c3 - meta.wbase];
          } else {
            x0 = ld_gather<V>(x + c0, pol_keep); x1 = ld_gather<V>(x + c1, pol_keep);
            x2 = ld_gather<V>(x + c2, pol_keep); x3 = ld_gather<V>(x + c3, pol_keep);
          }
          sum = vfma(svals[q0], x0, sum);
          sum = vfma(svals[q1], x1, sum);
          sum = vfma(svals[q2], x2, sum);
          sum = vfma(svals[q3], x3, sum);
        }
        for (; p < hi; p += lanes) {
          const int q = (int)(p - S);
          const int64_t c = (int64_t)scols[q];
          const V xx = use_win ? sxwin[c - meta.wbase] : ld_gather<V>(x + c, pol_keep);
          sum = vfma(svals[q], xx, sum);
        }
      } else {
        // partial (last) tile: straight from global memory
        for (; p < hi; p += lanes) {
          const int64_t c = (int64_t)ld_stream<I>(cols + p, pol_stream);
          const V a = ld_stream<V>(vals + p, pol_stream);
          const V xx = use_win ? sxwin[c - meta.wbase] : ld_gather<V>(x + c, pol_keep);
          sum = vfma(a, xx, sum);
        }
      }
      sum = group_reduce(sum, lanes);
      if (valid && gl == 0) {
        bool wrote = false;
        if (lo_g < S) { head[t] = sum; wrote = true; }                  // continues an earlier row
        else if (r < r_last || lo_g < E) {                              // this tile owns y[r]
          if (accumulate) sum = vadd(sum, y[r]);
          if constexpr (BCAST) store_bcast(y, peers, r, sum); else y[r] = sum;
            wrote = true;
        }
        if (DOT && wrote) dot_acc = vfma(w[r], sum, dot_acc);
      }
    }
    mbar_arrive(&empty_bar[s]);  // this thread is done with the stage
  }
  if (DOT) {
    // one deterministic partial per CTA (fixed thread→row mapping, fixed reduction tree)
    V sacc = dot_acc;
    for (int o = 16; o > 0; o >>= 1) sacc = vadd(sacc, vshfl_xor(sacc, o));
    if ((tid & 31) == 0) wsum[tid >> 5] = sacc;
    consumer_bar_sync();
    if (tid == 0) {
      V tot = wsum[0];
      for (int k = 1; k < kPipeConsumers / 32; ++k) tot = vadd(tot, wsum[k]);
      dot_partials[blockIdx.x] = tot;
    }
  }
}

}  // namespace b2s
