// b2s_spmv_agather.cuh — "async-gather" CSR SpMV for matrices with skewed row lengths (power-law,
// BASELINE config 5; reference kernel: cusparseSpMV in src/sparse/array/csr/spmv.cu:117-152).
//
// Included by b2s_spmv.cu.  Same tiling / ownership contract as spmv_pipe_kernel (1024-nnz tiles
// from the plan; the tile where a row starts owns y[r]; later pieces go to head[t] and are added by
// spmv_fixup_kernel in tile order; no floating-point atomics, bit-reproducible), different consumer:
//
//   * the x gathers are cp.async (LDGSTS) copies from global memory STRAIGHT INTO SHARED MEMORY
//     (the same request path as a register load, but no destination register is held while the
//     request is in flight).  They are the L1-BYPASSING 16-byte form
//     (cp.async.cg, SASS LDGSTS.E.BYPASS.128: the aligned 16 bytes that hold x[col]; the reduction picks
//     its half): the 4/8-byte form exists only as .ca, which pins an L1 line per request in flight — with
//     the L1 that is left beside ~200 KB of shared memory that caps the gather rate whatever the
//     occupancy.  A thread gathers exactly the 4 elements it
//     reduces later, so completion is a per-thread cp.async.wait_group — no barrier.  The gathers of
//     tile i+1 are issued BEFORE tile i is reduced: the whole reduction of a tile overlaps the L2 /
//     DRAM latency of the next one.  (The products consumer of spmv_pipe_kernel spends most of its
//     time on this matrix class in reduction passes with no gather outstanding.)
//   * the reduction is a SEGMENTED SUM in nnz order: a thread owns 4 consecutive products
//     (val * x read back from shared memory), rows are delimited by per-element row-start marks, rows
//     that end inside a thread are stored at once, open pieces are combined by a warp-level segmented
//     scan (ballot + 5 shuffle steps) and one exchange between the 8 warps through shared memory
//     (release / acquire on a per-warp sequence number — only a thread whose row runs past its warp
//     waits; no CTA barrier in the loop).  Work per tile is the same whatever the row-length
//     distribution: no lane walks a long row alone, no separate long-row pass.
//   * the column ids and values of a tile are read by the thread that uses them (16 / 32 coalesced bytes,
//     ld.global.nc.L1::no_allocate, L2 evict_first) one tile AHEAD into registers: staging them in
//     shared memory as spmv_pipe_kernel does left too little of it for the 16 bytes per element the
//     gathers need (3 CTAs x 1-2 tiles of TMA in flight could not cover the DRAM latency).  Shared memory holds only the gathered x (2 tiles), the
//     row-start marks (4 tiles) and the row pointers (4 tiles): 53 KB, 4 CTAs per SM.
//   * a ROW-POINTER WARP does everything that needs indptr: lane 0 fetches the tile's slice of
//     indptr with a TMA bulk copy (4 tiles ahead); then all 32 lanes turn it into row-start marks
//     (16-bit tile-local row numbers), store the zeros of owned empty rows and publish "marks ready"
//     on an mbarrier, up to 3 tiles ahead of the reduction.  The other warps never read a row pointer.
#pragma once

namespace b2s {

constexpr int kAgTile = 1024;             // nnz per tile (= the plan's tile size for this class)
constexpr int kAgPer  = kAgTile / kPipeConsumers;   // elements per thread = 4

struct AgRMeta {   // per row-pointer slot, written by lane 0 of the row-pointer warp before it arms the slot's barrier
  int64_t r_begin, r_last;
  int64_t ra;            // first indptr entry staged
  int32_t rows_staged;   // 1: indptr entries [ra, ...] are in shared memory
  int32_t pad;
};
struct AgVMeta {   // per marks slot, written with the row-start marks
  int64_t r_begin;
  int32_t starts_inside; // the tile begins inside a row (its leading piece -> head[t])
  int32_t pad;
};

template <typename V>
struct AgLayout {
  static constexpr int T = kAgTile;
  static constexpr int RCAP = 3 * T / 8 + 4;         // indptr entries per slot (388; tiles that touch more rows read indptr from global memory)
  static constexpr int NR = 4;                       // row-pointer slots (private to the row-pointer warp)
  static constexpr int NM = 4;                       // marks slots: the row-pointer warp may run 3 tiles ahead
  static constexpr size_t xslot_bytes = 16 * T;      // gathered x: 16 bytes per element (the aligned chunk of x), 2 slots
  static constexpr size_t vmeta_off   = 2 * T;       // marks slot: uint16 per element + AgVMeta
  static constexpr size_t mslot_bytes = (vmeta_off + sizeof(AgVMeta) + 127) / 128 * 128;
  static constexpr size_t rmeta_off   = 8 * RCAP;
  static constexpr size_t rslot_bytes = (rmeta_off + sizeof(AgRMeta) + 127) / 128 * 128;
  static constexpr size_t total = xslot_bytes * 2 + mslot_bytes * NM + rslot_bytes * NR + 8 * (NR + 2 * NM);
};

template <int BYTES>
__device__ __forceinline__ void cp_async_gather(uint32_t dst, const void* src, uint64_t pol) {   // allocates an L1 line
  asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], %2, %3;" ::"r"(dst), "l"(src), "n"(BYTES), "l"(pol));
}
__device__ __forceinline__ void cp_async_gather16_bypass(uint32_t dst, const void* src, uint64_t pol) {   // L1 bypass
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "l"(pol));
}

// 16-byte slot of element k (0..3) of thread g inside the gathered-x array (touched by this thread only):
// the slot order rotates every 2 threads so that the 16-byte LDGSTS writes and the 8-byte read-backs of
// a warp spread over the banks (4 wavefronts per LDS.64 instead of 16 for the linear order)
__device__ __forceinline__ int ag_own_slot(int g, int k) { return 4 * g + ((k + (g >> 1)) & 3); }

// the thread's 4 consecutive column ids / values of a tile starting at nnz position S (E = end of the
// matrix' data inside the tile): vector loads for whole tiles, guarded scalar loads for the last, partial
// one (padding: column -1, value 0)
template <typename I>
__device__ __forceinline__ void ag_load_cols(const I* __restrict__ cols, int64_t S, int64_t E, int g, uint64_t pol, I c[4]) {
  const int64_t p = S + 4 * g;
  if (E - S == kAgTile) {
    if constexpr (sizeof(I) == 4) {
      const uint4 u = ld_stream_16(cols + p, pol);
      memcpy(c, &u, 16);
    } else {
      const uint4 u0 = ld_stream_16(cols + p, pol), u1 = ld_stream_16(cols + p + 2, pol);
      memcpy(c, &u0, 16);
      memcpy(c + 2, &u1, 16);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) c[k] = p + k < E ? ld_stream<I>(cols + p + k, pol) : (I)-1;
  }
}
template <typename V>
__device__ __forceinline__ void ag_load_vals(const V* __restrict__ vals, int64_t S, int64_t E, int g, uint64_t pol, V a[4]) {
  const int64_t p = S + 4 * g;
  if (E - S == kAgTile) {
    if constexpr (sizeof(V) == 4) {
      const uint4 u = ld_stream_16(vals + p, pol);
      memcpy(a, &u, 16);
    } else {
      static_assert(sizeof(V) == 8, "async-gather kernel: 4- and 8-byte values only");
      const uint4 u0 = ld_stream_16(vals + p, pol), u1 = ld_stream_16(vals + p + 2, pol);
      memcpy(a, &u0, 16);
      memcpy(a + 2, &u1, 16);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = p + k < E ? ld_stream<V>(vals + p + k, pol) : zero_of<V>();
  }
}

template <typename V, typename I>
__global__ void __launch_bounds__(kPipeThreads, sizeof(I) == 4 ? 4 : 3)
spmv_agather_kernel(int64_t nrows, int64_t ncols, int64_t nnz, int64_t ntiles,
                    const int64_t* __restrict__ indptr, const I* __restrict__ cols,
                    const V* __restrict__ vals, const V* __restrict__ x, V* __restrict__ y,
                    const int64_t* __restrict__ tile_row, V* __restrict__ head, const int accumulate) {
  using L = AgLayout<V>;
  constexpr int T = L::T;
  constexpr int GT = kPipeConsumers;
  constexpr int NW = GT / 32;
  constexpr int NR = L::NR, NM = L::NM;
  constexpr size_t XSLOT = L::xslot_bytes, MSLOT = L::mslot_bytes, RSLOT = L::rslot_bytes;
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* xring = smem;
  unsigned char* mring = xring + XSLOT * 2;
  unsigned char* rring = mring + MSLOT * NM;
  uint64_t* fullR  = reinterpret_cast<uint64_t*>(rring + RSLOT * NR);   // row pointers of a slot have landed
  uint64_t* marksB = fullR + NR;                                        // marks of a slot are written
  uint64_t* emptyM = marksB + NM;                                       // marks of a slot are consumed (and cleared)
  // Per-warp summaries of a tile, exchanged WITHOUT a CTA barrier: a warp publishes {sum of its leading open
  // piece, "a row starts inside my 128 elements"} and then the tile's sequence number (release); only a thread
  // whose row runs past the end of its warp waits (acquire) for the summaries of the following warps.  kSeq
  // buffers in rotation: the marks ring keeps the warps of a CTA within NM tiles of each other.
  constexpr int kSeq = 8;
  static_assert(kSeq > NM && (kSeq & (kSeq - 1)) == 0, "summary buffers must outnumber the marks slots");
  __shared__ V   wsum[kSeq][NW];
  __shared__ int wany[kSeq][NW];
  __shared__ int wseq[kSeq][NW];

  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < NR; ++s) mbar_init(&fullR[s], 1);
    for (int s = 0; s < NM; ++s) { mbar_init(&marksB[s], 32); mbar_init(&emptyM[s], GT); }
    fence_mbar_init();
  }
  if (tid < kSeq * NW) (&wseq[0][0])[tid] = 0;
  if (tid < GT) {   // row-start marks start out clear; afterwards every consumer clears what it has read
    for (int s = 0; s < NM; ++s) reinterpret_cast<uint2*>(mring + MSLOT * s)[tid] = make_uint2(0, 0);
  }
  __syncthreads();

  const uint64_t pol_stream = policy_evict_first();
  const uint64_t pol_keep   = policy_evict_last();
  const int my_tiles = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);   // >= 1 (grid <= ntiles)

  if (tid >= GT) {
    // =================================== ROW-POINTER WARP ===================================
    const int lane = tid - GT;
    // lane 0: indptr slice of the CTA's j-th tile -> row-pointer slot j % NR (the slot's previous tile, j - NR,
    // has had its marks written by this same warp: program order + __syncwarp, no barrier needed)
    // (the plan entries of the NEXT tile are fetched one call ahead: their latency stays off this warp's loop)
    int64_t rb_next = 0, rl_next = 0;
    if (lane == 0) { rb_next = tile_row[blockIdx.x]; rl_next = tile_row[(int64_t)blockIdx.x + 1]; }
    auto r_tma = [&](int j) {
      const int rs = j % NR;
      const int64_t t = (int64_t)blockIdx.x + (int64_t)j * gridDim.x;
      const int64_t r_begin = rb_next, r_last = rl_next;
      if (j + 1 < my_tiles) { rb_next = tile_row[t + gridDim.x]; rl_next = tile_row[t + gridDim.x + 1]; }
      fence_proxy_async_smem();   // this warp's generic-proxy reads of the slot before the async-proxy refill
      unsigned char* sl = rring + RSLOT * rs;
      AgRMeta* meta = reinterpret_cast<AgRMeta*>(sl + L::rmeta_off);
      const int64_t e  = min(r_last, nrows - 1) + 1;   // last indptr entry needed
      const int64_t ra = r_begin & ~(int64_t)1;        // 16-byte aligned source
      int64_t n_ent = e - ra + 1;
      n_ent += (n_ent & 1);
      const bool rows_ok = (n_ent <= L::RCAP) && (ra + n_ent <= nrows + 1);
      meta->r_begin = r_begin; meta->r_last = r_last; meta->ra = ra; meta->rows_staged = rows_ok;
      if (rows_ok) {
        mbar_arrive_expect_tx(&fullR[rs], (uint32_t)(n_ent * 8));
        tma_bulk_g2s(sl, indptr + ra, (uint32_t)(n_ent * 8), &fullR[rs], pol_stream);
      } else {
        mbar_arrive(&fullR[rs]);
      }
    };
    if (lane == 0)
      for (int j = 0; j < NR - 1 && j < my_tiles; ++j) r_tma(j);
    __syncwarp();
    int ms = 0; uint32_t mp = 0;      // marks slot / parity of tile j
    for (int j = 0; j < my_tiles; ++j) {
      const int rs = j % NR;
      const uint32_t rp = (uint32_t)((j / NR) & 1);
      const int64_t t = (int64_t)blockIdx.x + (int64_t)j * gridDim.x;
      const int64_t S = t * (int64_t)T;
      const int64_t E = min(S + (int64_t)T, nnz);
      if (lane == 0 && j + NR - 1 < my_tiles) r_tma(j + NR - 1);   // refills the slot of tile j-1
      // Row-start marks of tile j: element (indptr[r] - S) <- 1 + (r - r_begin) for every non-empty row the tile
      // owns; owned EMPTY rows are stored here (no element to carry a mark).
      mbar_wait(&emptyM[ms], mp ^ 1u);    // tile j-NM is reduced: its marks slot is clear and free
      mbar_wait(&fullR[rs], rp);
      {
        const unsigned char* rsl = rring + RSLOT * rs;
        const AgRMeta* meta = reinterpret_cast<const AgRMeta*>(rsl + L::rmeta_off);
        const int64_t* srptr = reinterpret_cast<const int64_t*>(rsl);
        unsigned char* msl = mring + MSLOT * ms;
        uint16_t* mk = reinterpret_cast<uint16_t*>(msl);
        AgVMeta* vmeta = reinterpret_cast<AgVMeta*>(msl + L::vmeta_off);
        const int64_t r_begin = meta->r_begin, r_last = meta->r_last, ra = meta->ra;
        const bool staged = meta->rows_staged != 0;
        const int64_t nr = r_last - r_begin + 1;
        for (int64_t base = lane; base < nr; base += 32) {
          const int64_t r = r_begin + base;
          if (r >= nrows) break;
          int64_t lo_g, hi_g;
          if (staged) { lo_g = srptr[r - ra]; hi_g = srptr[r - ra + 1]; }
          else        { lo_g = indptr[r];     hi_g = indptr[r + 1]; }
          if (base == 0) { vmeta->r_begin = r_begin; vmeta->starts_inside = lo_g < S ? 1 : 0; }
          if (lo_g < S) continue;                                   // base == 0 only: the row began in an earlier tile
          if (r < r_last || lo_g < E) {                             // this tile owns y[r]
            if (hi_g > lo_g) mk[lo_g - S] = (uint16_t)(base + 1);
            else if (!accumulate) st_stream<V>(y + r, zero_of<V>(), pol_stream);
          }
        }
      }
      mbar_arrive(&marksB[ms]);     // release: marks + slot meta are visible to whoever acquires this phase
      __syncwarp();                 // every lane is done with the row pointers before lane 0 refills their slot
      if (++ms == NM) { ms = 0; mp ^= 1u; }
    }
    return;
  }

  // ======================================= CONSUMERS =======================================
  const int g = tid, w = tid >> 5, lane = tid & 31;
  constexpr int PER16 = 16 / (int)sizeof(V);          // x elements per 16-byte chunk (2 or 4)

  using U = typename std::make_unsigned<I>::type;
  const U ncols_whole = (U)(ncols & ~(int64_t)(PER16 - 1));   // columns below this lie in a whole 16-byte chunk of x
  // byte offset of the thread's k-th 16-byte slot inside an x slot (ag_own_slot), fixed for the kernel's lifetime
  uint32_t xoff[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) xoff[k] = 16u * (uint32_t)ag_own_slot(g, k);
  const uint32_t xring_s = smem_u32(xring);

  // Issue the thread's 4 x gathers of a tile (column ids c[], -1 = padding) into x slot `xs`.  Element k lands
  // as the aligned 16-byte chunk of x that holds it; the return value packs, 2 bits per element, which
  // sizeof(V)-sized piece of the chunk it is.
  auto issue = [&](int xs, const I c[4]) -> int {
    const uint32_t sx = xring_s + (uint32_t)XSLOT * (uint32_t)xs;
    int sub = 0;
    if ((U)c[0] < ncols_whole && (U)c[1] < ncols_whole && (U)c[2] < ncols_whole && (U)c[3] < ncols_whole) {
      // the common case: four L1-bypassing 16-byte copies, issued back to back.  (Careful with this block: in an
      // experimental variant of the kernel ptxas 12.9 encoded such copies as LDGSTS [R+UR0], desc[UR1] with
      // UR0/UR1 never written -> "illegal instruction" at run time; the Makefile greps the SASS for that form.)
      const char* s0 = reinterpret_cast<const char*>(x) + (size_t)((U)c[0] & ~(U)(PER16 - 1)) * sizeof(V);
      const char* s1 = reinterpret_cast<const char*>(x) + (size_t)((U)c[1] & ~(U)(PER16 - 1)) * sizeof(V);
      const char* s2 = reinterpret_cast<const char*>(x) + (size_t)((U)c[2] & ~(U)(PER16 - 1)) * sizeof(V);
      const char* s3 = reinterpret_cast<const char*>(x) + (size_t)((U)c[3] & ~(U)(PER16 - 1)) * sizeof(V);
      asm volatile(
          "cp.async.cg.shared.global.L2::cache_hint [%0], [%4], 16, %8;\n"
          "cp.async.cg.shared.global.L2::cache_hint [%1], [%5], 16, %8;\n"
          "cp.async.cg.shared.global.L2::cache_hint [%2], [%6], 16, %8;\n"
          "cp.async.cg.shared.global.L2::cache_hint [%3], [%7], 16, %8;\n"
          "cp.async.commit_group;" ::"r"(sx + xoff[0]), "r"(sx + xoff[1]), "r"(sx + xoff[2]), "r"(sx + xoff[3]),
          "l"(s0), "l"(s1), "l"(s2), "l"(s3), "l"(pol_keep)
          : "memory");
      sub = (int)(c[0] & (PER16 - 1)) | ((int)(c[1] & (PER16 - 1)) << 2) | ((int)(c[2] & (PER16 - 1)) << 4) |
            ((int)(c[3] & (PER16 - 1)) << 6);
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        unsigned char* slot = xring + XSLOT * xs + xoff[k];
        if (c[k] < 0) {                                            // padding of the partial tile
          *reinterpret_cast<V*>(slot) = zero_of<V>();
        } else if ((U)c[k] < ncols_whole) {                        // the whole chunk lies inside x
          cp_async_gather16_bypass(smem_u32(slot), x + ((int64_t)c[k] & ~(int64_t)(PER16 - 1)), pol_keep);
          sub |= (int)(c[k] & (PER16 - 1)) << (2 * k);
        } else {                                                   // last, short chunk of x: the element alone
          cp_async_gather<(int)sizeof(V)>(smem_u32(slot), x + (int64_t)c[k], pol_keep);
        }
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    return sub;
  };

  auto tile_span = [&](int j, int64_t* S, int64_t* E) {
    *S = ((int64_t)blockIdx.x + (int64_t)j * gridDim.x) * (int64_t)T;
    *E = min(*S + (int64_t)T, nnz);
  };

  // software pipeline (per thread): gathers 1 tile ahead (shared memory), values 1 tile ahead (registers),
  // column ids 2 tiles ahead (registers)
  int64_t S, E;
  I c_next[4];
  V a_next[4];
  tile_span(0, &S, &E);
  ag_load_cols<I>(cols, S, E, g, pol_stream, c_next);
  ag_load_vals<V>(vals, S, E, g, pol_stream, a_next);
  int sub_next = issue(0, c_next);
  if (my_tiles > 1) { tile_span(1, &S, &E); ag_load_cols<I>(cols, S, E, g, pol_stream, c_next); }
  int ms = 0; uint32_t mp = 0;   // marks slot / parity of the tile being reduced
  for (int i = 0; i < my_tiles; ++i) {
    const int64_t t = (int64_t)blockIdx.x + (int64_t)i * gridDim.x;
    const int sub = sub_next;
    if (i + 1 < my_tiles) {        // gathers of the NEXT tile fly during this tile's reduction
      sub_next = issue((i + 1) & 1, c_next);
      if (i + 2 < my_tiles) { tile_span(i + 2, &S, &E); ag_load_cols<I>(cols, S, E, g, pol_stream, c_next); }
    } else {
      asm volatile("cp.async.commit_group;" ::: "memory");   // empty group: the wait below is always "all but one"
    }
    V a[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) a[k] = a_next[k];
    if (i + 1 < my_tiles) { tile_span(i + 1, &S, &E); ag_load_vals<V>(vals, S, E, g, pol_stream, a_next); }

    unsigned char* msl = mring + MSLOT * ms;
    mbar_wait(&marksB[ms], mp);                            // marks + slot meta of tile i are written
    asm volatile("cp.async.wait_group 1;" ::: "memory");   // this thread's gathers of tile i have landed
    const AgVMeta* vmeta = reinterpret_cast<const AgVMeta*>(msl + L::vmeta_off);
    const int64_t r_begin = vmeta->r_begin;
    const bool head_cur = vmeta->starts_inside != 0;
    V xv[4];
    const unsigned char* sxq = xring + XSLOT * (i & 1);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      xv[k] = *reinterpret_cast<const V*>(sxq + xoff[k] + sizeof(V) * ((sub >> (2 * k)) & 3));
    uint2* mk = reinterpret_cast<uint2*>(msl) + g;
    const uint2 mraw = *mk;
    *mk = make_uint2(0, 0);                 // clear what this thread consumed (re-marked NM tiles later)
    mbar_arrive(&emptyM[ms]);               // the marks slot is free
    if (++ms == NM) { ms = 0; mp ^= 1u; }
    const int id[4] = {(int)(mraw.x & 0xffffu), (int)(mraw.x >> 16), (int)(mraw.y & 0xffffu), (int)(mraw.y >> 16)};

    V* const yrow = y + (r_begin - 1);      // y of the tile's row number rid (1-based): yrow[rid]
    auto store_row = [&](int rid, V sum) {
      V* dst = yrow + rid;
      if (accumulate) sum = vadd(sum, *dst);
      st_stream<V>(dst, sum, pol_stream);
    };
    // serial segmented sum over the thread's 4 products
    V acc = zero_of<V>(), lead = zero_of<V>();
    bool has = false;
    int cur = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (id[k] != 0) {
        if (has) store_row(cur, acc);     // a row that starts and ends inside this thread
        else lead = acc;
        has = true; cur = id[k]; acc = zero_of<V>();
      }
      acc = vfma(a[k], xv[k], acc);
    }
    if (!has) lead = acc;                 // no row starts here: all 4 products continue the piece to the left
    // reverse segmented scan over the warp: G = sum of the leading pieces of lanes >= this one up to and
    // including the first lane where a row starts.  The row-start flags travel as one ballot.
    const unsigned above = __ballot_sync(0xffffffffu, has) >> lane;   // bit d: a row starts in lane + d
    V G = lead;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const V Go = vshfl_down(G, d);
      if (lane + d < 32 && (above & ((1u << d) - 1u)) == 0u) G = vadd(G, Go);
    }
    V Gn = vshfl_down(G, 1);
    if (lane == 31) Gn = zero_of<V>();
    const bool anyn = (above >> 1) != 0u;   // a row starts in a later lane of this warp
    if (lane == 0) {
      wsum[i & (kSeq - 1)][w] = G; wany[i & (kSeq - 1)][w] = above != 0u ? 1 : 0;
      asm volatile("st.release.cta.shared.b32 [%0], %1;" ::"r"(smem_u32(&wseq[i & (kSeq - 1)][w])), "r"(i + 1) : "memory");
    }
    // the open tail of this thread's last row: closed inside the warp -> store now
    V tail = zero_of<V>();
    if (has) {
      tail = vadd(acc, Gn);
      if (anyn) store_row(cur, tail);
    }
    // summary of warp v for tile i (waits until that warp has published it)
    auto summary_of = [&](int v, V* sum) -> bool {
      const uint32_t a = smem_u32(&wseq[i & (kSeq - 1)][v]);
      int sq;
      do { asm volatile("ld.acquire.cta.shared.b32 %0, [%1];" : "=r"(sq) : "r"(a) : "memory"); } while (sq != i + 1);
      *sum = wsum[i & (kSeq - 1)][v];
      return wany[i & (kSeq - 1)][v] != 0;
    };
    if (has && !anyn) {
      // the row runs on into the following warps (or past the tile: then this is the owner's piece and
      // spmv_fixup_kernel adds the heads of the later tiles)
      for (int v = w + 1; v < NW; ++v) {
        V sv;
        const bool stop = summary_of(v, &sv);
        tail = vadd(tail, sv);
        if (stop) break;
      }
      store_row(cur, tail);
    }
    if (g == 0 && head_cur) {
      V h = G;                     // warp 0's own leading piece (this is lane 0 of warp 0)
      if (above == 0u) {
        for (int v = 1; v < NW; ++v) {
          V sv;
          const bool stop = summary_of(v, &sv);
          h = vadd(h, sv);
          if (stop) break;
        }
      }
      head[t] = h;
    }
  }
}

}  // namespace b2s
