// b2s_vec.cu — dense vector kernels of the CG / GMRES loop (HBM-bound, 128-bit accesses,
// device-resident scalars, deterministic two-level reductions finished by the last CTA).
//
// Reference semantics:
//   AXPBY  src/sparse/linalg/axpby.cu:25-47, axpby.cc:34-44 (val = a[0]/b[0], optional negate)
//   dots / norms are cupynumeric calls in legate_sparse/linalg.py:482,510,520,529.
#include "b2s_common.cuh"
#include "b2s_board.cuh"

namespace b2s {

constexpr int kVecThreads   = 256;
constexpr int kMaxRedBlocks = kNumSMs * 8;

template <typename V> struct alignas(16) Pack {
  static constexpr int N = (16 / sizeof(V)) > 0 ? (16 / sizeof(V)) : 1;
  V v[N];
};

static inline int64_t vec_grid(int64_t n_packs) {
  int64_t b = ceil_div(n_packs, (int64_t)kVecThreads * 4);
  if (b > kMaxRedBlocks) b = kMaxRedBlocks;
  if (b < 1) b = 1;
  return b;
}

// ---------------------------------------------------------------- axpby
template <typename V, bool VEC>
__global__ void __launch_bounds__(kVecThreads)
axpby_kernel(int64_t n, V* __restrict__ y, const V* __restrict__ x, const V* __restrict__ a,
             const V* __restrict__ b, int isalpha, int negate) {
  V val = vdiv(a[0], b[0]);
  if (negate) val = vneg(val);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    using P = Pack<V>;
    const int64_t np = n / P::N;
    const P* xp = reinterpret_cast<const P*>(x);
    P* yp = reinterpret_cast<P*>(y);
    for (int64_t i = i0; i < np; i += stride) {
      P xv = xp[i], yv = yp[i];
#pragma unroll
      for (int k = 0; k < P::N; ++k)
        yv.v[k] = isalpha ? vfma(val, xv.v[k], yv.v[k]) : vfma(val, yv.v[k], xv.v[k]);
      yp[i] = yv;
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride)
      y[i] = isalpha ? vfma(val, x[i], y[i]) : vfma(val, y[i], x[i]);
  } else {
    for (int64_t i = i0; i < n; i += stride)
      y[i] = isalpha ? vfma(val, x[i], y[i]) : vfma(val, y[i], x[i]);
  }
}

// ---------------------------------------------------------------- reductions
// Block-level deterministic sum, then the last CTA to finish adds the per-CTA partials in
// index order.  `counter` wraps back to 0 (atomicInc) so the workspace is reusable.
template <typename A, typename Fin, typename O>
__device__ __forceinline__ void finish_reduce(A local, A* partials, unsigned* counter, O* out, Fin fin) {
  __shared__ A wsum[kVecThreads / 32];
  __shared__ bool is_last;
  A s = local;
  for (int o = 16; o > 0; o >>= 1) s = vadd(s, vshfl_xor(s, o));
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    A tot = wsum[0];
    for (int i = 1; i < kVecThreads / 32; ++i) tot = vadd(tot, wsum[i]);
    partials[blockIdx.x] = tot;
    __threadfence();
    unsigned prev = atomicInc(counter, gridDim.x - 1);
    is_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    // one warp sums the partials in a fixed order
    if (threadIdx.x < 32) {
      A acc = zero_of<A>();
      for (unsigned i = threadIdx.x; i < gridDim.x; i += 32) acc = vadd(acc, ld_cg(&partials[i]));
      for (int o = 16; o > 0; o >>= 1) acc = vadd(acc, vshfl_xor(acc, o));
      if (threadIdx.x == 0) out[0] = fin(acc);
    }
  }
}

// the same with the cross-rank exchange folded into the last CTA's epilogue (bx.nranks > 1)
template <typename A>
__device__ __forceinline__ void finish_reduce_exchange(A local, A* partials, unsigned* counter, A* out, const BoardArgs<A>& bx) {
  __shared__ A wsum[kVecThreads / 32];
  __shared__ A xvals[kBoardRanks];
  __shared__ bool is_last;
  A s = local;
  for (int o = 16; o > 0; o >>= 1) s = vadd(s, vshfl_xor(s, o));
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    A tot = wsum[0];
    for (int i = 1; i < kVecThreads / 32; ++i) tot = vadd(tot, wsum[i]);
    partials[blockIdx.x] = tot;
    __threadfence();
    unsigned prev = atomicInc(counter, gridDim.x - 1);
    is_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last && threadIdx.x < 32) {
    __threadfence();
    A acc = zero_of<A>();
    for (unsigned i = threadIdx.x; i < gridDim.x; i += 32) acc = vadd(acc, ld_cg(&partials[i]));
    for (int o = 16; o > 0; o >>= 1) acc = vadd(acc, vshfl_xor(acc, o));   // every lane holds the local sum
    if (bx.nranks > 1) acc = board_exchange_warp<A>(acc, bx, xvals);
    if (threadIdx.x == 0) out[0] = acc;
  }
}

template <typename V, bool VEC, bool CONJ>
__global__ void __launch_bounds__(kVecThreads)
dot_kernel(int64_t n, const V* __restrict__ x, const V* __restrict__ y, V* partials,
           unsigned* counter, V* out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  V acc = zero_of<V>();
  if (VEC) {
    using P = Pack<V>;
    const int64_t np = n / P::N;
    const P* xp = reinterpret_cast<const P*>(x);
    const P* yp = reinterpret_cast<const P*>(y);
    for (int64_t i = i0; i < np; i += stride) {
      P xv = xp[i], yv = yp[i];
#pragma unroll
      for (int k = 0; k < P::N; ++k) acc = vfma(CONJ ? vconj(xv.v[k]) : xv.v[k], yv.v[k], acc);
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride) acc = vfma(CONJ ? vconj(x[i]) : x[i], y[i], acc);
  } else {
    for (int64_t i = i0; i < n; i += stride) acc = vfma(CONJ ? vconj(x[i]) : x[i], y[i], acc);
  }
  finish_reduce(acc, partials, counter, out, [] __device__(V v) { return v; });
}

template <typename V, bool VEC>
__global__ void __launch_bounds__(kVecThreads)
nrm2_kernel(int64_t n, const V* __restrict__ x, typename vt_traits<V>::real* partials,
            unsigned* counter, typename vt_traits<V>::real* out) {
  using R = typename vt_traits<V>::real;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  R acc = 0;
  if (VEC) {
    using P = Pack<V>;
    const int64_t np = n / P::N;
    const P* xp = reinterpret_cast<const P*>(x);
    for (int64_t i = i0; i < np; i += stride) {
      P xv = xp[i];
#pragma unroll
      for (int k = 0; k < P::N; ++k) acc += vabs2(xv.v[k]);
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride) acc += vabs2(x[i]);
  } else {
    for (int64_t i = i0; i < n; i += stride) acc += vabs2(x[i]);
  }
  finish_reduce(acc, partials, counter, out, [] __device__(R v) { return (R)sqrt((double)v); });
}

// x += alpha p ; r -= alpha q ; rr = sum r*r   (alpha = rho/pq)
template <typename V, bool VEC>
__global__ void __launch_bounds__(kVecThreads)
cg_update_kernel(int64_t n, V* __restrict__ x, V* __restrict__ r, const V* __restrict__ p,
                 const V* __restrict__ q, const V* __restrict__ rho, const V* __restrict__ pq,
                 V* partials, unsigned* counter, V* rr_out, const BoardArgs<V> bx) {
  const V alpha = vdiv(rho[0], pq[0]);
  const V nalpha = vneg(alpha);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  V acc = zero_of<V>();
  if (VEC) {
    using P = Pack<V>;
    const int64_t np = n / P::N;
    P* xp = reinterpret_cast<P*>(x);
    P* rp = reinterpret_cast<P*>(r);
    const P* pp = reinterpret_cast<const P*>(p);
    const P* qp = reinterpret_cast<const P*>(q);
    for (int64_t i = i0; i < np; i += stride) {
      P xv = xp[i], rv = rp[i], pv = pp[i], qv = qp[i];
#pragma unroll
      for (int k = 0; k < P::N; ++k) {
        xv.v[k] = vfma(alpha, pv.v[k], xv.v[k]);
        rv.v[k] = vfma(nalpha, qv.v[k], rv.v[k]);
        acc = vfma(rv.v[k], rv.v[k], acc);
      }
      xp[i] = xv;
      rp[i] = rv;
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride) {
      x[i] = vfma(alpha, p[i], x[i]);
      V rv = vfma(nalpha, q[i], r[i]);
      r[i] = rv;
      acc = vfma(rv, rv, acc);
    }
  } else {
    for (int64_t i = i0; i < n; i += stride) {
      x[i] = vfma(alpha, p[i], x[i]);
      V rv = vfma(nalpha, q[i], r[i]);
      r[i] = rv;
      acc = vfma(rv, rv, acc);
    }
  }
  finish_reduce_exchange<V>(acc, partials, counter, rr_out, bx);
}

// p = r + (rho/rho1) p ; rho1 == 0 → p = r
template <typename V, bool VEC>
__global__ void __launch_bounds__(kVecThreads)
cg_pupdate_kernel(int64_t n, V* __restrict__ p, const V* __restrict__ r, const V* __restrict__ rho,
                  const V* __restrict__ rho1, const PeerOut<V> peers) {
  const V d = rho1[0];
  const bool first = vis_zero(d);
  const V beta = first ? zero_of<V>() : vdiv(rho[0], d);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    using P = Pack<V>;
    const int64_t np = n / P::N;
    P* pp = reinterpret_cast<P*>(p);
    const P* rp = reinterpret_cast<const P*>(r);
    for (int64_t i = i0; i < np; i += stride) {
      P rv = rp[i];
      if (!first) {
        P pv = pp[i];
#pragma unroll
        for (int k = 0; k < P::N; ++k) rv.v[k] = vfma(beta, pv.v[k], rv.v[k]);
      }
      pp[i] = rv;
      if (peers.n < 0) {
#pragma unroll
        for (int k = 0; k < P::N; ++k) multimem_st(peers.p[0] + i * P::N + k, rv.v[k]);   // NVLS multicast
      } else {
#pragma unroll
        for (int g = 0; g < kMaxPeers; ++g)
          if (g < peers.n && (peers.hi[g] == 0 || ((i + 1) * P::N > peers.lo[g] && i * P::N < peers.hi[g])))
            reinterpret_cast<P*>(peers.p[g])[i] = rv;   // 16-byte P2P stores (whole pack if it overlaps)
      }
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride)
      store_bcast(p, peers, i, first ? r[i] : vfma(beta, p[i], r[i]));
  } else {
    for (int64_t i = i0; i < n; i += stride) store_bcast(p, peers, i, first ? r[i] : vfma(beta, p[i], r[i]));
  }
}

static inline bool aligned16(const void* p) { return ((uintptr_t)p % 16) == 0; }

struct RedWs {
  void* partials;
  unsigned* counter;
};
static inline RedWs carve(void* ws) {
  uintptr_t b = ((uintptr_t)ws + 63) & ~(uintptr_t)63;
  RedWs r;
  r.counter = reinterpret_cast<unsigned*>(b);
  r.partials = reinterpret_cast<void*>(b + 64);
  return r;
}

}  // namespace b2s

using namespace b2s;

extern "C" int64_t b2s_reduce_workspace_bytes(void) { return 64 + 64 + (int64_t)kMaxRedBlocks * 16 + 64; }

extern "C" int b2s_axpby(b2s_dtype vt, int64_t n, void* y, const void* x, const void* a, const void* b,
                         int isalpha, int negate, b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0, "negative n");
  if (n == 0) return B2S_OK;
  B2S_REQUIRE(y && x && a && b, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  B2S_DISPATCH_VT(vt, V, {
    bool vec = aligned16(x) && aligned16(y);
    int64_t grid = vec_grid(ceil_div(n, (int64_t)Pack<V>::N));
    if (vec) axpby_kernel<V, true><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (V*)y, (const V*)x, (const V*)a, (const V*)b, isalpha, negate);
    else     axpby_kernel<V, false><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (V*)y, (const V*)x, (const V*)a, (const V*)b, isalpha, negate);
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}

extern "C" int b2s_dot(b2s_dtype vt, int64_t n, const void* x, const void* y, int conj, void* out,
                       void* partials, b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0, "negative n");
  B2S_REQUIRE(out && partials, "null out/partials");
  B2S_REQUIRE(n == 0 || (x && y), "null vectors");
  cudaStream_t st = (cudaStream_t)stream;
  RedWs w = carve(partials);
  B2S_DISPATCH_VT(vt, V, {
    bool vec = aligned16(x) && aligned16(y);
    int64_t grid = vec_grid(ceil_div(n, (int64_t)Pack<V>::N));
    if (vec) {
      if (conj) dot_kernel<V, true, true><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (const V*)x, (const V*)y, (V*)w.partials, w.counter, (V*)out);
      else      dot_kernel<V, true, false><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (const V*)x, (const V*)y, (V*)w.partials, w.counter, (V*)out);
    } else {
      if (conj) dot_kernel<V, false, true><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (const V*)x, (const V*)y, (V*)w.partials, w.counter, (V*)out);
      else      dot_kernel<V, false, false><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (const V*)x, (const V*)y, (V*)w.partials, w.counter, (V*)out);
    }
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}

extern "C" int b2s_nrm2(b2s_dtype vt, int64_t n, const void* x, void* out, void* partials,
                        b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0, "negative n");
  B2S_REQUIRE(out && partials, "null out/partials");
  B2S_REQUIRE(n == 0 || x, "null vector");
  cudaStream_t st = (cudaStream_t)stream;
  RedWs w = carve(partials);
  B2S_DISPATCH_VT(vt, V, {
    using R = typename vt_traits<V>::real;
    bool vec = aligned16(x);
    int64_t grid = vec_grid(ceil_div(n, (int64_t)Pack<V>::N));
    if (vec) nrm2_kernel<V, true><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (const V*)x, (R*)w.partials, w.counter, (R*)out);
    else     nrm2_kernel<V, false><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (const V*)x, (R*)w.partials, w.counter, (R*)out);
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}

static int cg_update_impl(b2s_dtype vt, int64_t n, void* x, void* r, const void* p, const void* q,
                          const void* rho, const void* pq, void* rr_out, void* partials, void* const* boards,
                          int rank, int nranks, int channel, void* seq_counters, void* cur_out, void* prev_out,
                          void* err, b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0, "negative n");
  B2S_REQUIRE(rr_out && partials && rho && pq, "null scalar/workspace");
  B2S_REQUIRE(n == 0 || (x && r && p && q), "null vectors");
  cudaStream_t st = (cudaStream_t)stream;
  RedWs w = carve(partials);
  B2S_DISPATCH_VT(vt, V, {
    BoardArgs<V> bx;
    int rc = make_board_args<V>(boards, rank, nranks, channel, seq_counters, cur_out, prev_out, err, &bx);
    if (rc) return rc;
    bool vec = aligned16(x) && aligned16(r) && aligned16(p) && aligned16(q);
    int64_t grid = vec_grid(ceil_div(n > 0 ? n : 1, (int64_t)Pack<V>::N));
    if (vec) cg_update_kernel<V, true><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (V*)x, (V*)r, (const V*)p, (const V*)q, (const V*)rho, (const V*)pq, (V*)w.partials, w.counter, (V*)rr_out, bx);
    else     cg_update_kernel<V, false><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (V*)x, (V*)r, (const V*)p, (const V*)q, (const V*)rho, (const V*)pq, (V*)w.partials, w.counter, (V*)rr_out, bx);
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}

extern "C" int b2s_cg_update(b2s_dtype vt, int64_t n, void* x, void* r, const void* p, const void* q,
                             const void* rho, const void* pq, void* rr_out, void* partials,
                             b2s_stream_t stream) {
  return cg_update_impl(vt, n, x, r, p, q, rho, pq, rr_out, partials, nullptr, 0, 0, 0, nullptr, nullptr, nullptr,
                        nullptr, stream);
}

// cg_update whose r.r is summed over the ranks inside the kernel's final reduction (board exchange,
// see b2s_allreduce_board): rr_out[0] = sum over ranks; optionally prev_out[0] = cur_out[0],
// cur_out[0] = sum (CG: rho1 <- rho, rho <- r.r).
extern "C" int b2s_cg_update_allreduce(b2s_dtype vt, int64_t n, void* x, void* r, const void* p, const void* q,
                                       const void* rho, const void* pq, void* rr_out, void* partials,
                                       void* const* boards, int rank, int nranks, int channel,
                                       void* seq_counters, void* cur_out, void* prev_out, void* err,
                                       b2s_stream_t stream) {
  B2S_REQUIRE(boards != nullptr && nranks >= 2, "b2s_cg_update_allreduce needs boards of >= 2 ranks");
  B2S_REQUIRE((prev_out == nullptr) || (cur_out != nullptr), "prev_out needs cur_out");
  return cg_update_impl(vt, n, x, r, p, q, rho, pq, rr_out, partials, boards, rank, nranks, channel, seq_counters,
                        cur_out, prev_out, err, stream);
}

static int cg_pupdate_impl(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                           const void* rho1, void* const* p_peers, int npeers, const int64_t* lo,
                           const int64_t* hi, b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0, "negative n");
  B2S_REQUIRE(npeers >= -1 && npeers <= kMaxPeers, "npeers must be in [-1,7]");
  if (n == 0) return B2S_OK;
  B2S_REQUIRE(p && r && rho && rho1, "null pointer");
  B2S_REQUIRE(npeers == 0 || p_peers, "p_peers is null");
  cudaStream_t st = (cudaStream_t)stream;
  B2S_DISPATCH_VT(vt, V, {
    PeerOut<V> peers{};
    peers.n = npeers;
    bool vec = aligned16(p) && aligned16(r);
    for (int g = 0; g < (npeers < 0 ? 1 : npeers); ++g) {
      peers.p[g] = (V*)p_peers[g];
      vec = vec && aligned16(p_peers[g]);
      if (lo && hi && npeers > 0) { peers.lo[g] = lo[g]; peers.hi[g] = hi[g] > lo[g] ? hi[g] : -1; }
    }
    int64_t grid = vec_grid(ceil_div(n, (int64_t)Pack<V>::N));
    if (vec) cg_pupdate_kernel<V, true><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (V*)p, (const V*)r, (const V*)rho, (const V*)rho1, peers);
    else     cg_pupdate_kernel<V, false><<<(unsigned)grid, kVecThreads, 0, st>>>(n, (V*)p, (const V*)r, (const V*)rho, (const V*)rho1, peers);
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}

extern "C" int b2s_cg_pupdate(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                              const void* rho1, b2s_stream_t stream) {
  return cg_pupdate_impl(vt, n, p, r, rho, rho1, nullptr, 0, nullptr, nullptr, stream);
}

extern "C" int b2s_cg_pupdate_bcast(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                                    const void* rho1, void* const* p_peers, int npeers,
                                    b2s_stream_t stream) {
  return cg_pupdate_impl(vt, n, p, r, rho, rho1, p_peers, npeers, nullptr, nullptr, stream);
}

extern "C" int b2s_cg_pupdate_halo(b2s_dtype vt, int64_t n, void* p, const void* r, const void* rho,
                                   const void* rho1, void* const* p_peers, int npeers,
                                   const int64_t* lo, const int64_t* hi, b2s_stream_t stream) {
  B2S_REQUIRE(npeers >= 0, "halo ranges need unicast peers");
  B2S_REQUIRE(npeers == 0 || (lo && hi), "null range arrays");
  return cg_pupdate_impl(vt, n, p, r, rho, rho1, p_peers, npeers, lo, hi, stream);
}

// =================================================================== cross-GPU scalar exchange
// All-reduce(sum) of ONE device scalar per rank without NCCL: every rank owns a small "board" in
// symmetric (peer-mapped) memory; a one-warp kernel stores its partial + a sequence number into its
// slot of EVERY rank's board (NVLink P2P stores, st.release.sys), spins until the G slots of its own
// board carry the current sequence number (ld.acquire.sys) and adds them up IN RANK ORDER — the
// result is bit-identical on every rank and from run to run.  Slots are double-buffered by the
// parity of the sequence number: a rank can be at most one exchange ahead of a peer on a channel.
// This is the CG iteration's replacement for two 1-element NCCL all-reduces and a barrier
// (reference linalg.py:519-526 gets the same values from Legate future reductions).
namespace b2s {

// inout[0]: this rank's partial on entry, the global sum on exit (stand-alone form; cg_update and
// the SpMV's fused dot fold the same exchange into their final reduction).
template <typename V>
__global__ void __launch_bounds__(32)
allreduce_board_kernel(V* __restrict__ inout, const BoardArgs<V> bx) {
  __shared__ V vals[kBoardRanks];
  const V tot = board_exchange_warp<V>(inout[0], bx, vals);
  if (threadIdx.x == 0) inout[0] = tot;
}

}  // namespace b2s

extern "C" int64_t b2s_board_bytes(void) {
  return (int64_t)sizeof(b2s::BoardSlot) * b2s::kBoardChannels * 2 * b2s::kBoardRanks;
}

// boards[g] = device address of rank g's board (own board included), all zero-initialised and
// mapped into this process (symmetric memory).  seq_counters: >= 4 local device uint64, zeroed once;
// err: optional local device int set when a peer never answers.  Every rank must call with the same
// channel sequence.  inout is a 1-element device array of dtype vt.
extern "C" int b2s_allreduce_board(b2s_dtype vt, void* inout, void* const* boards, int rank, int nranks,
                                   int channel, void* seq_counters, void* cur_out, void* prev_out, void* err,
                                   b2s_stream_t stream) {
  B2S_REQUIRE(nranks >= 1 && nranks <= kBoardRanks && rank >= 0 && rank < nranks, "bad rank / nranks");
  B2S_REQUIRE(channel >= 0 && channel < kBoardChannels, "bad channel");
  B2S_REQUIRE(inout && boards && seq_counters, "null pointer");
  B2S_REQUIRE((prev_out == nullptr) || (cur_out != nullptr), "prev_out needs cur_out");
  cudaStream_t st = (cudaStream_t)stream;
  B2S_DISPATCH_VT(vt, V, {
    BoardArgs<V> bx;
    // nranks == 1 still goes through the board (a rank exchanging with itself): same code path everywhere
    BoardArgs<V> tmp{};
    for (int g = 0; g < nranks; ++g) {
      B2S_REQUIRE(boards[g] != nullptr, "null board pointer");
      tmp.boards.b[g] = reinterpret_cast<BoardSlot*>(boards[g]);
    }
    tmp.rank = rank; tmp.nranks = nranks; tmp.channel = channel;
    tmp.seq_counters = reinterpret_cast<unsigned long long*>(seq_counters);
    tmp.cur_out = (V*)cur_out; tmp.prev_out = (V*)prev_out; tmp.err = (int*)err;
    bx = tmp;
    allreduce_board_kernel<V><<<1, 32, 0, st>>>((V*)inout, bx);
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}
