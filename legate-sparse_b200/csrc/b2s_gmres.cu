// b2s_gmres.cu — the tall-skinny kernels of restarted GMRES with classical Gram-Schmidt.
//
// Reference: legate_sparse/linalg.py:607-640 (Arnoldi step)
//     h = V[:, :j+1].conj().T @ u ;  u = u - V[:, :j+1] @ h ;  h_{j+1,j} = ||u|| ;  v = u / h_{j+1,j}
// and :655-657 (x += V @ y).  Upstream these are cupynumeric GEMVs on an (n, restart) array; here the
// Krylov basis is stored basis-vector-major (row c = v_c, leading dimension ldv >= n) so that every
// access is a unit-stride 128-bit stream, and each step is two passes over the basis:
//   cgs_project : h[c] = sum_i conj(V[c][i]) * u[i]            (KC columns per launch, u read once per launch)
//   cgs_update  : u[i] -= sum_c h[c] * V[c][i] ; nrm = ||u||_2 (all columns in one launch, norm fused)
// HBM-bound: (k+1)*n + (k+2)*n values per step for k basis vectors; deterministic reductions (fixed
// order, no floating-point atomics).
#include "b2s_common.cuh"

namespace b2s {

constexpr int kGmThreads   = 256;
constexpr int kGmMaxBlocks = kNumSMs * 8;   // like the other reductions
constexpr int kGmMaxK      = 1024;          // basis vectors per update launch (h staged in shared memory)

template <typename V> struct alignas(16) GPack {
  static constexpr int N = (16 / sizeof(V)) > 0 ? (16 / sizeof(V)) : 1;
  V v[N];
};

__device__ __forceinline__ float  vscale(float a, float s)   { return a * s; }
__device__ __forceinline__ double vscale(double a, double s) { return a * s; }
__device__ __forceinline__ c64    vscale(c64 a, float s)     { return c64{a.re * s, a.im * s}; }
__device__ __forceinline__ c128   vscale(c128 a, double s)   { return c128{a.re * s, a.im * s}; }

template <typename V> struct proj_cols { static constexpr int value = vt_traits<V>::cplx ? 8 : 16; };

static inline int64_t gm_grid(int64_t n_items) {
  int64_t b = ceil_div(n_items, (int64_t)kGmThreads * 2);
  if (b > kGmMaxBlocks) b = kGmMaxBlocks;
  if (b < 1) b = 1;
  return b;
}

// h[c] = sum_i conj(V[c*ldv+i]) u[i] for c < k <= KC.  partials: [gridDim.x][KC].
template <typename V, int KC, bool VEC>
__global__ void __launch_bounds__(kGmThreads)
cgs_project_kernel(int64_t n, int k, const V* __restrict__ basis, int64_t ldv, const V* __restrict__ u,
                   V* __restrict__ partials, unsigned* __restrict__ counter, V* __restrict__ h) {
  V acc[KC];
#pragma unroll
  for (int c = 0; c < KC; ++c) acc[c] = zero_of<V>();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    using P = GPack<V>;
    const int64_t np = n / P::N;
    const P* up = reinterpret_cast<const P*>(u);
    for (int64_t i = i0; i < np; i += stride) {
      const P uv = up[i];
      P vv[KC];
#pragma unroll
      for (int c = 0; c < KC; ++c)
        if (c < k) vv[c] = reinterpret_cast<const P*>(basis + (int64_t)c * ldv)[i];
#pragma unroll
      for (int c = 0; c < KC; ++c)
        if (c < k) {
#pragma unroll
          for (int e = 0; e < P::N; ++e) acc[c] = vfma(vconj(vv[c].v[e]), uv.v[e], acc[c]);
        }
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride) {
      const V uv = u[i];
#pragma unroll
      for (int c = 0; c < KC; ++c)
        if (c < k) acc[c] = vfma(vconj(basis[(int64_t)c * ldv + i]), uv, acc[c]);
    }
  } else {
    for (int64_t i = i0; i < n; i += stride) {
      const V uv = u[i];
#pragma unroll
      for (int c = 0; c < KC; ++c)
        if (c < k) acc[c] = vfma(vconj(basis[(int64_t)c * ldv + i]), uv, acc[c]);
    }
  }
  // CTA reduction in a fixed order: warp shuffles, then warp 0..: one thread per column over the warps
  __shared__ V wsum[kGmThreads / 32][KC];
  __shared__ bool is_last;
#pragma unroll
  for (int c = 0; c < KC; ++c) {
    V s = acc[c];
    for (int o = 16; o > 0; o >>= 1) s = vadd(s, vshfl_xor(s, o));
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5][c] = s;
  }
  __syncthreads();
  if (threadIdx.x < KC) {
    V tot = wsum[0][threadIdx.x];
    for (int w = 1; w < kGmThreads / 32; ++w) tot = vadd(tot, wsum[w][threadIdx.x]);
    partials[(int64_t)blockIdx.x * KC + threadIdx.x] = tot;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned prev = atomicInc(counter, gridDim.x - 1);   // wraps to 0: workspace reusable
    is_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    // warp w sums column w, w+8, ... over the CTAs: lane-strided then shuffle tree (fixed order)
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int c = w; c < k; c += kGmThreads / 32) {
      V a = zero_of<V>();
      for (unsigned b = lane; b < gridDim.x; b += 32) a = vadd(a, ld_cg(&partials[(int64_t)b * KC + c]));
      for (int o = 16; o > 0; o >>= 1) a = vadd(a, vshfl_xor(a, o));
      if (lane == 0) h[c] = a;
    }
  }
}

// u[i] += sign * sum_c h[c] V[c*ldv+i]  (sign = -1: Gram-Schmidt update, +1: x += V y);
// NORM: nrm_out = ||u_new||_2.
template <typename V, bool VEC, bool NORM>
__global__ void __launch_bounds__(kGmThreads)
cgs_update_kernel(int64_t n, int k, const V* __restrict__ basis, int64_t ldv, const V* __restrict__ h,
                  int negate, V* __restrict__ u, typename vt_traits<V>::real* partials, unsigned* counter,
                  typename vt_traits<V>::real* nrm_out) {
  using R = typename vt_traits<V>::real;
  extern __shared__ __align__(16) unsigned char gm_smem[];
  V* hs = reinterpret_cast<V*>(gm_smem);
  for (int c = threadIdx.x; c < k; c += blockDim.x) hs[c] = negate ? vneg(h[c]) : h[c];
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  R nacc = 0;
  if (VEC) {
    using P = GPack<V>;
    const int64_t np = n / P::N;
    P* up = reinterpret_cast<P*>(u);
    for (int64_t i = i0; i < np; i += stride) {
      P uv = up[i];
      int c = 0;
      for (; c + 4 <= k; c += 4) {   // 4 independent 128-bit streams in flight
        const P a0 = reinterpret_cast<const P*>(basis + (int64_t)(c + 0) * ldv)[i];
        const P a1 = reinterpret_cast<const P*>(basis + (int64_t)(c + 1) * ldv)[i];
        const P a2 = reinterpret_cast<const P*>(basis + (int64_t)(c + 2) * ldv)[i];
        const P a3 = reinterpret_cast<const P*>(basis + (int64_t)(c + 3) * ldv)[i];
#pragma unroll
        for (int e = 0; e < P::N; ++e) {
          uv.v[e] = vfma(hs[c + 0], a0.v[e], uv.v[e]);
          uv.v[e] = vfma(hs[c + 1], a1.v[e], uv.v[e]);
          uv.v[e] = vfma(hs[c + 2], a2.v[e], uv.v[e]);
          uv.v[e] = vfma(hs[c + 3], a3.v[e], uv.v[e]);
        }
      }
      for (; c < k; ++c) {
        const P a = reinterpret_cast<const P*>(basis + (int64_t)c * ldv)[i];
#pragma unroll
        for (int e = 0; e < P::N; ++e) uv.v[e] = vfma(hs[c], a.v[e], uv.v[e]);
      }
      up[i] = uv;
      if (NORM) {
#pragma unroll
        for (int e = 0; e < P::N; ++e) nacc += vabs2(uv.v[e]);
      }
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride) {
      V uv = u[i];
      for (int c = 0; c < k; ++c) uv = vfma(hs[c], basis[(int64_t)c * ldv + i], uv);
      u[i] = uv;
      if (NORM) nacc += vabs2(uv);
    }
  } else {
    for (int64_t i = i0; i < n; i += stride) {
      V uv = u[i];
      for (int c = 0; c < k; ++c) uv = vfma(hs[c], basis[(int64_t)c * ldv + i], uv);
      u[i] = uv;
      if (NORM) nacc += vabs2(uv);
    }
  }
  if (NORM) {
    __shared__ R wsum[kGmThreads / 32];
    __shared__ bool is_last;
    R s = nacc;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      R tot = wsum[0];
      for (int w = 1; w < kGmThreads / 32; ++w) tot += wsum[w];
      partials[blockIdx.x] = tot;
      __threadfence();
      unsigned prev = atomicInc(counter, gridDim.x - 1);
      is_last = (prev == gridDim.x - 1);
    }
    __syncthreads();
    if (is_last && threadIdx.x < 32) {
      __threadfence();
      R a = 0;
      for (unsigned b = threadIdx.x; b < gridDim.x; b += 32) a += ld_cg(&partials[b]);
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (threadIdx.x == 0) nrm_out[0] = (R)sqrt((double)a);
    }
  }
}

// out[i] = x[i] / s[0]   (s: device real scalar — the new basis vector v = u / ||u||)
template <typename V, bool VEC>
__global__ void __launch_bounds__(kGmThreads)
vscale_inv_kernel(int64_t n, const V* __restrict__ x, const typename vt_traits<V>::real* __restrict__ s,
                  V* __restrict__ out) {
  using R = typename vt_traits<V>::real;
  const R inv = (R)1 / s[0];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    using P = GPack<V>;
    const int64_t np = n / P::N;
    const P* xp = reinterpret_cast<const P*>(x);
    P* op = reinterpret_cast<P*>(out);
    for (int64_t i = i0; i < np; i += stride) {
      P xv = xp[i];
#pragma unroll
      for (int e = 0; e < P::N; ++e) xv.v[e] = vscale(xv.v[e], inv);
      op[i] = xv;
    }
    for (int64_t i = np * P::N + i0; i < n; i += stride) out[i] = vscale(x[i], inv);
  } else {
    for (int64_t i = i0; i < n; i += stride) out[i] = vscale(x[i], inv);
  }
}

static inline bool al16(const void* p) { return ((uintptr_t)p % 16) == 0; }

struct GmWs {
  unsigned* counter;
  void* partials;
};
static inline GmWs gm_carve(void* ws) {
  uintptr_t b = ((uintptr_t)ws + 63) & ~(uintptr_t)63;
  return GmWs{reinterpret_cast<unsigned*>(b), reinterpret_cast<void*>(b + 64)};
}

}  // namespace b2s

using namespace b2s;

// counter (64 B) + per-CTA partials of up to 16 columns of the widest type
extern "C" int64_t b2s_cgs_workspace_bytes(void) { return 64 + 64 + (int64_t)kGmMaxBlocks * 16 * 16 + 64; }

extern "C" int b2s_cgs_project(b2s_dtype vt, int64_t n, int k, const void* basis, int64_t ldv,
                               const void* u, void* h, void* workspace, b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0 && k >= 0, "negative size");
  B2S_REQUIRE(k == 0 || (h && workspace), "null h/workspace");
  B2S_REQUIRE(k == 0 || ldv >= n, "ldv < n");
  if (k == 0) return B2S_OK;
  B2S_REQUIRE(n == 0 || (basis && u), "null vectors");
  cudaStream_t st = (cudaStream_t)stream;
  GmWs w = gm_carve(workspace);
  B2S_DISPATCH_VT(vt, V, {
    constexpr int KC = proj_cols<V>::value;
    const bool vec = al16(basis) && al16(u) && ((ldv * (int64_t)sizeof(V)) % 16 == 0);
    const int64_t grid = gm_grid(ceil_div(n > 0 ? n : 1, (int64_t)GPack<V>::N));
    for (int c0 = 0; c0 < k; c0 += KC) {
      const int kk = (k - c0) < KC ? (k - c0) : KC;
      const V* b0 = (const V*)basis + (int64_t)c0 * ldv;
      if (vec) cgs_project_kernel<V, KC, true><<<(unsigned)grid, kGmThreads, 0, st>>>(n, kk, b0, ldv, (const V*)u, (V*)w.partials, w.counter, (V*)h + c0);
      else     cgs_project_kernel<V, KC, false><<<(unsigned)grid, kGmThreads, 0, st>>>(n, kk, b0, ldv, (const V*)u, (V*)w.partials, w.counter, (V*)h + c0);
      B2S_CHECK_LAUNCH();
    }
  });
  return B2S_OK;
}

extern "C" int b2s_cgs_update(b2s_dtype vt, int64_t n, int k, const void* basis, int64_t ldv,
                              const void* h, int negate, void* u, void* nrm_out, void* workspace,
                              b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0 && k >= 0, "negative size");
  B2S_REQUIRE(k <= kGmMaxK, "more than 1024 basis vectors per call");
  B2S_REQUIRE(k == 0 || ldv >= n, "ldv < n");
  B2S_REQUIRE(nrm_out == nullptr || workspace != nullptr, "norm needs the workspace");
  B2S_REQUIRE(n == 0 || u, "u is null");
  B2S_REQUIRE(k == 0 || n == 0 || (basis && h), "null basis/h");
  cudaStream_t st = (cudaStream_t)stream;
  GmWs w = gm_carve(workspace);
  B2S_DISPATCH_VT(vt, V, {
    using R = typename vt_traits<V>::real;
    const bool vec = al16(u) && (k == 0 || (al16(basis) && ((ldv * (int64_t)sizeof(V)) % 16 == 0)));
    const int64_t grid = gm_grid(ceil_div(n > 0 ? n : 1, (int64_t)GPack<V>::N));
    const size_t smem = sizeof(V) * (size_t)(k > 0 ? k : 1);
    if (nrm_out) {
      if (vec) cgs_update_kernel<V, true, true><<<(unsigned)grid, kGmThreads, smem, st>>>(n, k, (const V*)basis, ldv, (const V*)h, negate, (V*)u, (R*)w.partials, w.counter, (R*)nrm_out);
      else     cgs_update_kernel<V, false, true><<<(unsigned)grid, kGmThreads, smem, st>>>(n, k, (const V*)basis, ldv, (const V*)h, negate, (V*)u, (R*)w.partials, w.counter, (R*)nrm_out);
    } else {
      if (vec) cgs_update_kernel<V, true, false><<<(unsigned)grid, kGmThreads, smem, st>>>(n, k, (const V*)basis, ldv, (const V*)h, negate, (V*)u, nullptr, nullptr, nullptr);
      else     cgs_update_kernel<V, false, false><<<(unsigned)grid, kGmThreads, smem, st>>>(n, k, (const V*)basis, ldv, (const V*)h, negate, (V*)u, nullptr, nullptr, nullptr);
    }
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}

extern "C" int b2s_vscale_inv(b2s_dtype vt, int64_t n, const void* x, const void* s, void* out,
                              b2s_stream_t stream) {
  B2S_REQUIRE(n >= 0, "negative n");
  if (n == 0) return B2S_OK;
  B2S_REQUIRE(x && s && out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  B2S_DISPATCH_VT(vt, V, {
    using R = typename vt_traits<V>::real;
    const bool vec = al16(x) && al16(out);
    const int64_t grid = gm_grid(ceil_div(n, (int64_t)GPack<V>::N));
    if (vec) vscale_inv_kernel<V, true><<<(unsigned)grid, kGmThreads, 0, st>>>(n, (const V*)x, (const R*)s, (V*)out);
    else     vscale_inv_kernel<V, false><<<(unsigned)grid, kGmThreads, 0, st>>>(n, (const V*)x, (const R*)s, (V*)out);
    B2S_CHECK_LAUNCH();
  });
  return B2S_OK;
}
