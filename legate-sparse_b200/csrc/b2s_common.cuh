// b2s_common.cuh — shared device/host helpers for libb200sparse (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <atomic>
#include <type_traits>

#include "../../include/b200sparse.h"

namespace b2s {

// ---------------------------------------------------------------- errors
void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launch_count;

#define B2S_CUDA_TRY(expr)                                                           \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::b2s::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),       \
                       __FILE__, __LINE__);                                          \
      return B2S_ERR_CUDA;                                                           \
    }                                                                                \
  } while (0)

#define B2S_CHECK_LAUNCH()                                                           \
  do {                                                                               \
    ::b2s::g_launch_count.fetch_add(1, std::memory_order_relaxed);                   \
    cudaError_t _e = cudaGetLastError();                                             \
    if (_e != cudaSuccess) {                                                         \
      ::b2s::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e),   \
                       __FILE__, __LINE__);                                          \
      return B2S_ERR_CUDA;                                                           \
    }                                                                                \
  } while (0)

#define B2S_REQUIRE(cond, msg)                                                       \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::b2s::set_error("invalid argument: %s (%s)", msg, #cond);                     \
      return B2S_ERR_ARG;                                                            \
    }                                                                                \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// ---------------------------------------------------------------- value types
struct c64  { float re, im; };
struct c128 { double re, im; };

template <typename T> struct vt_traits;
template <> struct vt_traits<float>  { using real = float;  static constexpr bool cplx = false; };
template <> struct vt_traits<double> { using real = double; static constexpr bool cplx = false; };
template <> struct vt_traits<c64>    { using real = float;  static constexpr bool cplx = true; };
template <> struct vt_traits<c128>   { using real = double; static constexpr bool cplx = true; };

__host__ __device__ __forceinline__ float  vzero(float*)  { return 0.f; }
__host__ __device__ __forceinline__ double vzero(double*) { return 0.0; }
__host__ __device__ __forceinline__ c64    vzero(c64*)    { return c64{0.f, 0.f}; }
__host__ __device__ __forceinline__ c128   vzero(c128*)   { return c128{0.0, 0.0}; }
template <typename T> __host__ __device__ __forceinline__ T zero_of() { return vzero((T*)nullptr); }

__device__ __forceinline__ float  vadd(float a, float b)   { return a + b; }
__device__ __forceinline__ double vadd(double a, double b) { return a + b; }
__device__ __forceinline__ c64    vadd(c64 a, c64 b)       { return c64{a.re + b.re, a.im + b.im}; }
__device__ __forceinline__ c128   vadd(c128 a, c128 b)     { return c128{a.re + b.re, a.im + b.im}; }

__device__ __forceinline__ float  vmul(float a, float b)   { return a * b; }
__device__ __forceinline__ double vmul(double a, double b) { return a * b; }
__device__ __forceinline__ c64 vmul(c64 a, c64 b) {
  return c64{a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}
__device__ __forceinline__ c128 vmul(c128 a, c128 b) {
  return c128{a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}
// acc + a*b
__device__ __forceinline__ float  vfma(float a, float b, float acc)    { return fmaf(a, b, acc); }
__device__ __forceinline__ double vfma(double a, double b, double acc) { return fma(a, b, acc); }
__device__ __forceinline__ c64 vfma(c64 a, c64 b, c64 acc) {
  return c64{fmaf(-a.im, b.im, fmaf(a.re, b.re, acc.re)), fmaf(a.im, b.re, fmaf(a.re, b.im, acc.im))};
}
__device__ __forceinline__ c128 vfma(c128 a, c128 b, c128 acc) {
  return c128{fma(-a.im, b.im, fma(a.re, b.re, acc.re)), fma(a.im, b.re, fma(a.re, b.im, acc.im))};
}
__device__ __forceinline__ float  vconj(float a)  { return a; }
__device__ __forceinline__ double vconj(double a) { return a; }
__device__ __forceinline__ c64    vconj(c64 a)    { return c64{a.re, -a.im}; }
__device__ __forceinline__ c128   vconj(c128 a)   { return c128{a.re, -a.im}; }
__device__ __forceinline__ float  vneg(float a)   { return -a; }
__device__ __forceinline__ double vneg(double a)  { return -a; }
__device__ __forceinline__ c64    vneg(c64 a)     { return c64{-a.re, -a.im}; }
__device__ __forceinline__ c128   vneg(c128 a)    { return c128{-a.re, -a.im}; }
__device__ __forceinline__ float  vdiv(float a, float b)   { return a / b; }
__device__ __forceinline__ double vdiv(double a, double b) { return a / b; }
template <typename C, typename R>
__device__ __forceinline__ C cdiv_impl(C a, C b) {
  // Smith's algorithm (what C99/numpy complex division does, avoids overflow)
  if (fabs((double)b.re) >= fabs((double)b.im)) {
    R ratio = b.im / b.re, den = b.re + b.im * ratio;
    return C{(a.re + a.im * ratio) / den, (a.im - a.re * ratio) / den};
  } else {
    R ratio = b.re / b.im, den = b.re * ratio + b.im;
    return C{(a.re * ratio + a.im) / den, (a.im * ratio - a.re) / den};
  }
}
__device__ __forceinline__ c64  vdiv(c64 a, c64 b)   { return cdiv_impl<c64, float>(a, b); }
__device__ __forceinline__ c128 vdiv(c128 a, c128 b) { return cdiv_impl<c128, double>(a, b); }
__device__ __forceinline__ bool vis_zero(float a)  { return a == 0.f; }
__device__ __forceinline__ bool vis_zero(double a) { return a == 0.0; }
__device__ __forceinline__ bool vis_zero(c64 a)    { return a.re == 0.f && a.im == 0.f; }
__device__ __forceinline__ bool vis_zero(c128 a)   { return a.re == 0.0 && a.im == 0.0; }
// |a|^2 as real
__device__ __forceinline__ float  vabs2(float a)  { return a * a; }
__device__ __forceinline__ double vabs2(double a) { return a * a; }
__device__ __forceinline__ float  vabs2(c64 a)    { return a.re * a.re + a.im * a.im; }
__device__ __forceinline__ double vabs2(c128 a)   { return a.re * a.re + a.im * a.im; }

// warp shuffles for all value types
__device__ __forceinline__ float  vshfl_xor(float v, int m)  { return __shfl_xor_sync(0xffffffffu, v, m); }
__device__ __forceinline__ double vshfl_xor(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
__device__ __forceinline__ c64 vshfl_xor(c64 v, int m) {
  return c64{__shfl_xor_sync(0xffffffffu, v.re, m), __shfl_xor_sync(0xffffffffu, v.im, m)};
}
__device__ __forceinline__ c128 vshfl_xor(c128 v, int m) {
  return c128{__shfl_xor_sync(0xffffffffu, v.re, m), __shfl_xor_sync(0xffffffffu, v.im, m)};
}
__device__ __forceinline__ float  vshfl_up(float v, int d)  { return __shfl_up_sync(0xffffffffu, v, d); }
__device__ __forceinline__ double vshfl_up(double v, int d) { return __shfl_up_sync(0xffffffffu, v, d); }
__device__ __forceinline__ c64 vshfl_up(c64 v, int d) {
  return c64{__shfl_up_sync(0xffffffffu, v.re, d), __shfl_up_sync(0xffffffffu, v.im, d)};
}
__device__ __forceinline__ c128 vshfl_up(c128 v, int d) {
  return c128{__shfl_up_sync(0xffffffffu, v.re, d), __shfl_up_sync(0xffffffffu, v.im, d)};
}
__device__ __forceinline__ float  vshfl_idx(float v, int l)  { return __shfl_sync(0xffffffffu, v, l); }
__device__ __forceinline__ double vshfl_idx(double v, int l) { return __shfl_sync(0xffffffffu, v, l); }
__device__ __forceinline__ c64 vshfl_idx(c64 v, int l) {
  return c64{__shfl_sync(0xffffffffu, v.re, l), __shfl_sync(0xffffffffu, v.im, l)};
}
__device__ __forceinline__ c128 vshfl_idx(c128 v, int l) {
  return c128{__shfl_sync(0xffffffffu, v.re, l), __shfl_sync(0xffffffffu, v.im, l)};
}
__device__ __forceinline__ float  vshfl_down(float v, int d)  { return __shfl_down_sync(0xffffffffu, v, d); }
__device__ __forceinline__ double vshfl_down(double v, int d) { return __shfl_down_sync(0xffffffffu, v, d); }
__device__ __forceinline__ c64 vshfl_down(c64 v, int d) {
  return c64{__shfl_down_sync(0xffffffffu, v.re, d), __shfl_down_sync(0xffffffffu, v.im, d)};
}
__device__ __forceinline__ c128 vshfl_down(c128 v, int d) {
  return c128{__shfl_down_sync(0xffffffffu, v.re, d), __shfl_down_sync(0xffffffffu, v.im, d)};
}

// ---------------------------------------------------------------- cache-hinted loads
// Matrix streams (vals / col indices) are read exactly once: do not allocate in L1 and
// mark evict_first in L2 so they do not displace the x vector, which is the only reused
// operand of SpMV (x gathers use the default / evict_last policy).
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// 16-byte streaming load
__device__ __forceinline__ uint4 ld_stream_16(const void* ptr, uint64_t pol) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(ptr), "l"(pol));
  return r;
}
__device__ __forceinline__ uint2 ld_stream_8(const void* ptr, uint64_t pol) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;"
               : "=r"(r.x), "=r"(r.y)
               : "l"(ptr), "l"(pol));
  return r;
}
__device__ __forceinline__ uint32_t ld_stream_4(const void* ptr, uint64_t pol) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;"
               : "=r"(r)
               : "l"(ptr), "l"(pol));
  return r;
}

template <typename T> __device__ __forceinline__ T ld_stream(const T* p, uint64_t pol);
template <> __device__ __forceinline__ float ld_stream<float>(const float* p, uint64_t pol) {
  return __uint_as_float(ld_stream_4(p, pol));
}
template <> __device__ __forceinline__ int32_t ld_stream<int32_t>(const int32_t* p, uint64_t pol) {
  return (int32_t)ld_stream_4(p, pol);
}
template <> __device__ __forceinline__ double ld_stream<double>(const double* p, uint64_t pol) {
  uint2 r = ld_stream_8(p, pol);
  return __hiloint2double((int)r.y, (int)r.x);
}
template <> __device__ __forceinline__ int64_t ld_stream<int64_t>(const int64_t* p, uint64_t pol) {
  uint2 r = ld_stream_8(p, pol);
  return (int64_t)(((uint64_t)r.y << 32) | r.x);
}
template <> __device__ __forceinline__ c64 ld_stream<c64>(const c64* p, uint64_t pol) {
  uint2 r = ld_stream_8(p, pol);
  return c64{__uint_as_float(r.x), __uint_as_float(r.y)};
}
template <> __device__ __forceinline__ c128 ld_stream<c128>(const c128* p, uint64_t pol) {
  uint4 r = ld_stream_16(p, pol);
  return c128{__hiloint2double((int)r.y, (int)r.x), __hiloint2double((int)r.w, (int)r.z)};
}

// x gather: read-only path, keep in L2 (evict_last policy)
template <typename T> __device__ __forceinline__ T ld_gather(const T* p, uint64_t pol);
template <> __device__ __forceinline__ float ld_gather<float>(const float* p, uint64_t pol) {
  float r;
  asm volatile("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(pol));
  return r;
}
template <> __device__ __forceinline__ double ld_gather<double>(const double* p, uint64_t pol) {
  double r;
  asm volatile("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(r) : "l"(p), "l"(pol));
  return r;
}
template <> __device__ __forceinline__ c64 ld_gather<c64>(const c64* p, uint64_t pol) {
  c64 r;
  asm volatile("ld.global.nc.L2::cache_hint.v2.f32 {%0,%1}, [%2], %3;"
               : "=f"(r.re), "=f"(r.im) : "l"(p), "l"(pol));
  return r;
}
template <> __device__ __forceinline__ c128 ld_gather<c128>(const c128* p, uint64_t pol) {
  c128 r;
  asm volatile("ld.global.nc.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
               : "=d"(r.re), "=d"(r.im) : "l"(p), "l"(pol));
  return r;
}

// the same without allocating an L1 line: the random gathers of the products consumer almost never
// hit L1, and an L1 line per outstanding request only shrinks what the miss path can keep in flight
template <typename T> __device__ __forceinline__ T ld_gather_na(const T* p, uint64_t pol);
template <> __device__ __forceinline__ float ld_gather_na<float>(const float* p, uint64_t pol) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(r) : "l"(p), "l"(pol));
  return r;
}
template <> __device__ __forceinline__ double ld_gather_na<double>(const double* p, uint64_t pol) {
  double r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(r) : "l"(p), "l"(pol));
  return r;
}
template <> __device__ __forceinline__ c64 ld_gather_na<c64>(const c64* p, uint64_t pol) {
  c64 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f32 {%0,%1}, [%2], %3;"
               : "=f"(r.re), "=f"(r.im) : "l"(p), "l"(pol));
  return r;
}
template <> __device__ __forceinline__ c128 ld_gather_na<c128>(const c128* p, uint64_t pol) {
  c128 r;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.f64 {%0,%1}, [%2], %3;"
               : "=d"(r.re), "=d"(r.im) : "l"(p), "l"(pol));
  return r;
}

// result stores of the streaming kernels: written once, not re-read by this launch — evict_first in
// L2 so that y (as large as x) does not compete with the x vector for L2 capacity
template <typename T> __device__ __forceinline__ void st_stream(T* p, T v, uint64_t pol);
template <> __device__ __forceinline__ void st_stream<float>(float* p, float v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
template <> __device__ __forceinline__ void st_stream<double>(double* p, double v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(pol) : "memory");
}
template <> __device__ __forceinline__ void st_stream<c64>(c64* p, c64 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1,%2}, %3;" ::"l"(p), "f"(v.re), "f"(v.im), "l"(pol) : "memory");
}
template <> __device__ __forceinline__ void st_stream<c128>(c128* p, c128 v, uint64_t pol) {
  asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1,%2}, %3;" ::"l"(p), "d"(v.re), "d"(v.im), "l"(pol) : "memory");
}

// L2-coherent load of a value written by another CTA (bypasses L1)
template <typename A>
__device__ __forceinline__ A ld_cg(const A* p) {
  A out;
  if constexpr (sizeof(A) == 4) {
    unsigned r = __ldcg(reinterpret_cast<const unsigned*>(p));
    memcpy(&out, &r, 4);
  } else if constexpr (sizeof(A) == 8) {
    uint2 r = __ldcg(reinterpret_cast<const uint2*>(p));
    memcpy(&out, &r, 8);
  } else {
    static_assert(sizeof(A) == 16, "unsupported size");
    uint4 r = __ldcg(reinterpret_cast<const uint4*>(p));
    memcpy(&out, &r, 16);
  }
  return out;
}

// ---------------------------------------------------------------- mbarrier + TMA bulk copy (1-D)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}
// TMA bulk (non-tensor) global→shared copy: SASS UBLKCP. 16-byte aligned src/dst, bytes%16==0.
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                             uint64_t* bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
      : "memory");
}

// ---------------------------------------------------------------- peer broadcast (NVLink P2P stores)
// Extra destinations of a result vector: the same row block inside the buffers of the OTHER
// ranks (pointers already offset to this rank's first row; peer memory mapped through CUDA
// IPC / symmetric memory).  A kernel that writes y[r] also stores the value to every peer, so
// the "all-gather" of the row blocks rides on the kernel's own stores over NVLink / NVSwitch.
constexpr int kMaxPeers = 7;
template <typename V>
struct PeerOut {
  V* p[kMaxPeers];
  int n;    // number of unicast peers, or -1: p[0] is an NVSwitch MULTICAST address (NVLS) that
            // maps the same offset of EVERY rank's buffer — one store, the switch replicates it
  // optional per-peer element range [lo, hi) of the local block that the peer actually needs
  // (halo exchange: the [min col, max col] image of the peer's rows, like the reference's
  // image(crd→x, MIN_MAX)); hi == 0 means "everything"
  int64_t lo[kMaxPeers], hi[kMaxPeers];
};
template <typename V>
__device__ __forceinline__ bool peer_wants(const PeerOut<V>& peers, int g, int64_t i) {
  return peers.hi[g] == 0 || (i >= peers.lo[g] && i < peers.hi[g]);
}
// multimem.st: the only legal way to store through a multicast address (PTX ISA, "multimem")
__device__ __forceinline__ void multimem_st(float* a, float v) {
  asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(a), "f"(v) : "memory");
}
__device__ __forceinline__ void multimem_st(double* a, double v) {
  asm volatile("multimem.st.relaxed.sys.global.f64 [%0], %1;" ::"l"(a), "d"(v) : "memory");
}
__device__ __forceinline__ void multimem_st(c64* a, c64 v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(a), "f"(v.re), "f"(v.im) : "memory");
}
__device__ __forceinline__ void multimem_st(c128* a, c128 v) {
  multimem_st(&a->re, v.re);
  multimem_st(&a->im, v.im);
}
template <typename V>
__device__ __forceinline__ void store_bcast(V* __restrict__ y, const PeerOut<V>& peers, int64_t r, V v) {
  y[r] = v;
  if (peers.n < 0) {
    multimem_st(peers.p[0] + r, v);
  } else {
#pragma unroll
    for (int g = 0; g < kMaxPeers; ++g)
      if (g < peers.n && peer_wants(peers, g, r)) peers.p[g][r] = v;
  }
}

// ---------------------------------------------------------------- misc
__host__ __device__ __forceinline__ int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------- cross-TU internals (not in the C ABI)
// b2s_spgemm.cu: in-place inclusive scan of v[0..n), first[0] = 0; blocksum = ceil(n/1024)+1 int64 scratch
int scan_inclusive_i64(int64_t n, int64_t* v, int64_t* first, int64_t* blocksum, cudaStream_t st);
// b2s_spmv.cu: the one SpMV entry (accumulate != 0: y += A x, pipe kernel only)
// raw (type-erased) arguments of a cross-rank board exchange folded into a reduction (b2s_board.cuh)
struct BoardRaw {
  void* const* boards;
  int rank, nranks, channel;
  void* seq_counters;
  void* cur_out;
  void* prev_out;
  void* err;
};
int spmv_entry(b2s_dtype vt, b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz,
               const int64_t* indptr, const void* indices, const void* data, const void* x, void* y,
               const b2s_spmv_plan* plan, int variant, void* dot_out, void* partials, const void* w,
               void* const* y_peers, int npeers, int accumulate, b2s_stream_t stream,
               const BoardRaw* board = nullptr);
int plan_create_impl(b2s_itype it, int64_t nrows, int64_t ncols, int64_t nnz, const int64_t* indptr,
                     const void* indices, void* workspace, int64_t workspace_bytes, b2s_stream_t stream,
                     int64_t force_tile, b2s_spmv_plan** out_plan);
void* plan_dot_partials(const b2s_spmv_plan* plan);

template <typename I> struct it_code;
template <> struct it_code<int32_t> { static constexpr b2s_itype value = B2S_I32; };
template <> struct it_code<int64_t> { static constexpr b2s_itype value = B2S_I64; };

inline size_t dtype_size(b2s_dtype vt) {
  switch (vt) {
    case B2S_F32: return 4;
    case B2S_F64: return 8;
    case B2S_C64: return 8;
    case B2S_C128: return 16;
  }
  return 0;
}

// type dispatch helpers (host)
#define B2S_DISPATCH_VT(vt, T, ...)                                    \
  switch (vt) {                                                        \
    case B2S_F32:  { using T = float;       __VA_ARGS__; break; }      \
    case B2S_F64:  { using T = double;      __VA_ARGS__; break; }      \
    case B2S_C64:  { using T = ::b2s::c64;  __VA_ARGS__; break; }      \
    case B2S_C128: { using T = ::b2s::c128; __VA_ARGS__; break; }      \
    default: ::b2s::set_error("bad b2s_dtype %d", (int)(vt)); return B2S_ERR_ARG; \
  }
#define B2S_DISPATCH_IT(it, I, ...)                                    \
  switch (it) {                                                        \
    case B2S_I32: { using I = int32_t; __VA_ARGS__; break; }           \
    case B2S_I64: { using I = int64_t; __VA_ARGS__; break; }           \
    default: ::b2s::set_error("bad b2s_itype %d", (int)(it)); return B2S_ERR_ARG; \
  }

}  // namespace b2s
