// SIMT (CUDA-core, fp32) kernels of the MeshNet hot path: Chebyshev basis SpMM, generic GEMMs with
// the fused conv epilogue, BatchNorm statistics / apply / backward, basis backward.  These cover
// every shape (V=17 joint graph, Fin=5, Fout=3 ...) and are the parity baseline and fallback for
// the tensor-core path in cheb_umma.cu.  All of it is HBM- or FFMA-bound fp32 work; no tensor cores.
#include <cuda_runtime.h>

#include <algorithm>

#include "p2m_internal.h"

namespace p2m {

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// =====================================================================================
// Chebyshev basis  T = [T0 | T1 | T2],  T0 = x, T1 = L~ x, T2 = 2 L~ T1 - x
// (cheby_graph_conv.py:16-29).  One thread per (row, VEC features); neighbour rows are gathered
// through L2 — each is a contiguous F*4-byte segment, so a warp reads whole 128-byte lines.
// =====================================================================================
template <int VEC>
struct VecT;
template <>
struct VecT<4> {
  using type = float4;
};
template <>
struct VecT<1> {
  using type = float;
};

__device__ __forceinline__ float4 fma4(float a, float4 x, float4 acc) {
  acc.x = fmaf(a, x.x, acc.x);
  acc.y = fmaf(a, x.y, acc.y);
  acc.z = fmaf(a, x.z, acc.z);
  acc.w = fmaf(a, x.w, acc.w);
  return acc;
}
__device__ __forceinline__ float fma4(float a, float x, float acc) { return fmaf(a, x, acc); }
__device__ __forceinline__ float4 zero_of(float4) { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float zero_of(float) { return 0.f; }
// 2*s - x0
__device__ __forceinline__ float4 two_s_minus(float4 s, float4 x0) {
  return make_float4(2.f * s.x - x0.x, 2.f * s.y - x0.y, 2.f * s.z - x0.z, 2.f * s.w - x0.w);
}
__device__ __forceinline__ float two_s_minus(float s, float x0) { return 2.f * s - x0; }

template <int VEC>
__global__ void __launch_bounds__(256) k_cheb_t01(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                  const float* __restrict__ val, int V, const float* __restrict__ x,
                                                  int in_unpool, long long rows, int F, float* __restrict__ T) {
  using vec = typename VecT<VEC>::type;
  const int fg = F / VEC;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * fg) return;
  long long r = idx / fg;
  int f = (int)(idx - r * fg);
  int v = (int)(r % V);
  const vec* xv = reinterpret_cast<const vec*>(x);
  long long pr = in_unpool ? (r >> 1) : r;
  vec t0 = xv[pr * fg + f];
  vec acc = zero_of(t0);
  int p0 = rowptr[v], p1 = rowptr[v + 1];
  for (int p = p0; p < p1; ++p) {
    long long rn = r + reloff[p];
    if (in_unpool) rn >>= 1;
    acc = fma4(val[p], xv[rn * fg + f], acc);
  }
  vec* Tv = reinterpret_cast<vec*>(T);
  Tv[r * 3 * fg + f] = t0;
  Tv[r * 3 * fg + fg + f] = acc;
}

template <int VEC>
__global__ void __launch_bounds__(256) k_cheb_t2(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                 const float* __restrict__ val, int V, long long rows, int F,
                                                 float* __restrict__ T) {
  using vec = typename VecT<VEC>::type;
  const int fg = F / VEC;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * fg) return;
  long long r = idx / fg;
  int f = (int)(idx - r * fg);
  int v = (int)(r % V);
  vec* Tv = reinterpret_cast<vec*>(T);
  vec t0 = Tv[r * 3 * fg + f];
  vec acc = zero_of(t0);
  int p0 = rowptr[v], p1 = rowptr[v + 1];
  for (int p = p0; p < p1; ++p) {
    long long rn = r + reloff[p];
    acc = fma4(val[p], Tv[rn * 3 * fg + fg + f], acc);
  }
  Tv[r * 3 * fg + 2 * fg + f] = two_s_minus(acc, t0);
}

int launch_cheb_basis(const DevLevel& g, const float* x, int in_unpool, int rows, int F, float* T, cudaStream_t s) {
  if (rows % g.V != 0) {
    set_error("cheb_basis: rows not a multiple of the level size");
    return P2M_ERR_INVALID;
  }
  const bool v4 = (F % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(T) & 15) == 0);
  long long n = (long long)rows * (v4 ? F / 4 : F);
  int grid = cdiv(n, 256);
  if (v4) {
    k_cheb_t01<4><<<grid, 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, x, in_unpool, rows, F, T);
    P2M_LAUNCH_OK();
    k_cheb_t2<4><<<grid, 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, F, T);
    P2M_LAUNCH_OK();
  } else {
    k_cheb_t01<1><<<grid, 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, x, in_unpool, rows, F, T);
    P2M_LAUNCH_OK();
    k_cheb_t2<1><<<grid, 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, F, T);
    P2M_LAUNCH_OK();
  }
  return P2M_OK;
}

// =====================================================================================
// Basis backward:  U = dT1 + 2 L~ dT2 ;  dXl = dT0 - dT2 + L~ U (+ resample^T(g_res)),  optional pair-sum
// =====================================================================================
template <int VEC>
__global__ void __launch_bounds__(256) k_basis_bwd_u(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                     const float* __restrict__ val, int V, long long rows, int F,
                                                     const float* __restrict__ dT, float* __restrict__ U) {
  using vec = typename VecT<VEC>::type;
  const int fg = F / VEC;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * fg) return;
  long long r = idx / fg;
  int f = (int)(idx - r * fg);
  int v = (int)(r % V);
  const vec* Dv = reinterpret_cast<const vec*>(dT);
  vec acc = zero_of(Dv[0]);
  int p0 = rowptr[v], p1 = rowptr[v + 1];
  for (int p = p0; p < p1; ++p) {
    long long rn = r + reloff[p];
    acc = fma4(2.f * val[p], Dv[rn * 3 * fg + 2 * fg + f], acc);
  }
  vec d1 = Dv[r * 3 * fg + fg + f];
  reinterpret_cast<vec*>(U)[r * fg + f] = fma4(1.f, d1, acc);
}

// final combine: dXl = dT0 - dT2 + L~ U (+ resample^T(g_res)); VEC features per thread; pair-sum for the
// virtual unpool (the physical row p receives logical rows 2p and 2p+1)
template <int VEC>
__global__ void __launch_bounds__(256) k_basis_bwd_dx(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                      const float* __restrict__ val, int V, long long rows_out, int F,
                                                      const float* __restrict__ dT, const float* __restrict__ U,
                                                      const float* __restrict__ g_res, int res_Fout,
                                                      const int* __restrict__ t_ptr, const int* __restrict__ t_idx,
                                                      const float* __restrict__ t_w, int pairsum,
                                                      float* __restrict__ dx) {
  using vec = typename VecT<VEC>::type;
  const int fg = F / VEC;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows_out * fg) return;
  long long ro = idx / fg;
  int f = (int)(idx - ro * fg);
  float total[VEC];
#pragma unroll
  for (int e = 0; e < VEC; ++e) total[e] = 0.f;
  const int reps = pairsum ? 2 : 1;
  const vec* Uv = reinterpret_cast<const vec*>(U);
  const vec* Dv = reinterpret_cast<const vec*>(dT);
  for (int q = 0; q < reps; ++q) {
    long long r = pairsum ? (2 * ro + q) : ro;
    int v = (int)(r % V);
    vec acc = zero_of(Uv[0]);
    int p0 = rowptr[v], p1 = rowptr[v + 1];
    for (int p = p0; p < p1; ++p) acc = fma4(val[p], Uv[(r + reloff[p]) * fg + f], acc);
    vec d0 = Dv[r * 3 * fg + f], d2 = Dv[r * 3 * fg + 2 * fg + f];
    float a[VEC], b0[VEC], b2[VEC];
    *reinterpret_cast<vec*>(a) = acc;
    *reinterpret_cast<vec*>(b0) = d0;
    *reinterpret_cast<vec*>(b2) = d2;
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
      float t = a[e] + (b0[e] - b2[e]);
      if (g_res != nullptr) {
        const int fe = f * VEC + e;
        for (int p = t_ptr[fe]; p < t_ptr[fe + 1]; ++p) t = fmaf(t_w[p], g_res[r * res_Fout + t_idx[p]], t);
      }
      total[e] += t;
    }
  }
  *reinterpret_cast<vec*>(dx + (ro * fg + f) * VEC) = *reinterpret_cast<vec*>(total);
}

int launch_cheb_basis_bwd(const DevLevel& g, const float* dT, int rows, int F, float* U, const float* g_res,
                          int res_Fout, const InterpTable* it, int out_pairsum, float* dx, cudaStream_t s) {
  const bool v4 = (F % 4 == 0) && ((reinterpret_cast<uintptr_t>(dx) & 15) == 0);
  long long n = (long long)rows * (v4 ? F / 4 : F);
  if (v4) {
    k_basis_bwd_u<4><<<cdiv(n, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, F, dT, U);
  } else {
    k_basis_bwd_u<1><<<cdiv(n, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, F, dT, U);
  }
  P2M_LAUNCH_OK();
  long long rows_out = out_pairsum ? rows / 2 : rows;
  if (v4)
    k_basis_bwd_dx<4><<<cdiv(rows_out * F / 4, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows_out, F, dT, U,
                                                                 g_res, res_Fout, it ? it->t_ptr : nullptr,
                                                                 it ? it->t_idx : nullptr, it ? it->t_w : nullptr,
                                                                 out_pairsum, dx);
  else
    k_basis_bwd_dx<1><<<cdiv(rows_out * F, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows_out, F, dT, U, g_res,
                                                             res_Fout, it ? it->t_ptr : nullptr,
                                                             it ? it->t_idx : nullptr, it ? it->t_w : nullptr,
                                                             out_pairsum, dx);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// Finishing pass of the tensor-core backward-data path (p2m_api.cu): pair-sum for the virtual unpool and the
// transposed channel resampling of the residual gradient.
template <int VEC>
__global__ void __launch_bounds__(256) k_dx_finish(const float* __restrict__ dxl, long long rows_out, int F,
                                                   const float* __restrict__ g_res, int res_Fout,
                                                   const int* __restrict__ t_ptr, const int* __restrict__ t_idx,
                                                   const float* __restrict__ t_w, int pairsum, float* __restrict__ out) {
  using vec = typename VecT<VEC>::type;
  const int fg = F / VEC;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows_out * fg) return;
  const long long ro = idx / fg;
  const int f = (int)(idx - ro * fg);
  float total[VEC];
#pragma unroll
  for (int e = 0; e < VEC; ++e) total[e] = 0.f;
  const int reps = pairsum ? 2 : 1;
  for (int q = 0; q < reps; ++q) {
    const long long r = pairsum ? (2 * ro + q) : ro;
    float a[VEC];
    *reinterpret_cast<vec*>(a) = reinterpret_cast<const vec*>(dxl)[r * fg + f];
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
      float t = a[e];
      if (g_res != nullptr) {
        const int fe = f * VEC + e;
        for (int p = t_ptr[fe]; p < t_ptr[fe + 1]; ++p) t = fmaf(t_w[p], g_res[r * res_Fout + t_idx[p]], t);
      }
      total[e] += t;
    }
  }
  *reinterpret_cast<vec*>(out + (ro * fg + f) * VEC) = *reinterpret_cast<vec*>(total);
}
int launch_dx_finish(const float* dxl, int rows, int F, const float* g_res, int res_Fout, const InterpTable* it,
                     int out_pairsum, float* out, cudaStream_t s) {
  const long long rows_out = out_pairsum ? rows / 2 : rows;
  const bool v4 = (F % 4 == 0) && (((reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(dxl)) & 15) == 0);
  if (v4)
    k_dx_finish<4><<<cdiv(rows_out * F / 4, 256), 256, 0, s>>>(dxl, rows_out, F, g_res, res_Fout, it ? it->t_ptr : nullptr,
                                                              it ? it->t_idx : nullptr, it ? it->t_w : nullptr,
                                                              out_pairsum, out);
  else
    k_dx_finish<1><<<cdiv(rows_out * F, 256), 256, 0, s>>>(dxl, rows_out, F, g_res, res_Fout, it ? it->t_ptr : nullptr,
                                                          it ? it->t_idx : nullptr, it ? it->t_w : nullptr, out_pairsum,
                                                          out);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// =====================================================================================
// Generic fp32 GEMM  C = A * op(B)  with the conv epilogue
// =====================================================================================
template <int BM, int BN, int BK, bool B_KN>
__global__ void __launch_bounds__(256) k_gemm(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb,
                                              float* __restrict__ C, int ldc, int M, int N, int K, EpiDev ep) {
  constexpr int TM = 8;
  constexpr int TN = BN / 16;  // 16 thread columns; TN = 8 (BN=128) or 4 (BN=64)
  static_assert(BM == 128 && (BN == 128 || BN == 64), "tile config");
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    for (int e = tid; e < BM * BK; e += 256) {
      int row = e / BK, k = e % BK;
      long long m = m0 + row;
      As[k][row] = (m < M && k0 + k < K) ? A[m * lda + k0 + k] : 0.f;
    }
    if (B_KN) {
      for (int e = tid; e < BN * BK; e += 256) {
        int k = e / BN, n = e % BN;
        Bs[k][n] = (n0 + n < N && k0 + k < K) ? B[(long long)(k0 + k) * ldb + n0 + n] : 0.f;
      }
    } else {
      for (int e = tid; e < BN * BK; e += 256) {
        int n = e / BK, k = e % BK;
        Bs[k][n] = (n0 + n < N && k0 + k < K) ? B[(long long)(n0 + n) * ldb + k0 + k] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
      for (int h = 0; h < TN / 4; ++h) {
        float4 bv = *reinterpret_cast<const float4*>(&Bs[k][h * 64 + tx * 4]);
        b[h * 4 + 0] = bv.x; b[h * 4 + 1] = bv.y; b[h * 4 + 2] = bv.z; b[h * 4 + 3] = bv.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    long long m = m0 + ty * 8 + i;
    if (m >= M) continue;
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int n = n0 + h * 64 + tx * 4 + j;
        if (n < N) C[m * ldc + n] = apply_epilogue(acc[i][h * 4 + j], m, n, ep);
      }
    }
  }
}

int launch_gemm(const float* A, int lda, const float* B, int ldb, int b_is_kn, float* C, int ldc, int M, int N, int K,
                const Epilogue& e, cudaStream_t s) {
  if (M <= 0 || N <= 0 || K <= 0) {
    set_error("gemm: empty problem");
    return P2M_ERR_INVALID;
  }
  EpiDev ep = to_dev(e);
  if (N > 64) {
    dim3 grid(cdiv(M, 128), cdiv(N, 128));
    if (b_is_kn)
      k_gemm<128, 128, 16, true><<<grid, 256, 0, s>>>(A, lda, B, ldb, C, ldc, M, N, K, ep);
    else
      k_gemm<128, 128, 16, false><<<grid, 256, 0, s>>>(A, lda, B, ldb, C, ldc, M, N, K, ep);
  } else {
    dim3 grid(cdiv(M, 128), cdiv(N, 64));
    if (b_is_kn)
      k_gemm<128, 64, 16, true><<<grid, 256, 0, s>>>(A, lda, B, ldb, C, ldc, M, N, K, ep);
    else
      k_gemm<128, 64, 16, false><<<grid, 256, 0, s>>>(A, lda, B, ldb, C, ldc, M, N, K, ep);
  }
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// C[N1,N2] += A[M,N1]^T B[M,N2]; each CTA owns a 128x128 output tile and a chunk of M rows (8x8 register
// tile per thread); partial sums are merged with fp32 atomics (C zeroed by the caller).
constexpr int TN_CHUNK = 4096;
__global__ void __launch_bounds__(256) k_gemm_tn_atomic(const float* __restrict__ A, int lda,
                                                        const float* __restrict__ B, int ldb, float* __restrict__ C,
                                                        int ldc, int M, int N1, int N2, int a_vec, int b_vec) {
  __shared__ __align__(16) float As[16][128 + 4];
  __shared__ __align__(16) float Bs[16][128 + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int a0 = blockIdx.y * 128, b0 = blockIdx.z * 128;
  const long long mbeg = (long long)blockIdx.x * TN_CHUNK;
  const long long mend = min((long long)M, mbeg + TN_CHUNK);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (long long m0 = mbeg; m0 < mend; m0 += 16) {
    for (int e = tid; e < 16 * 32; e += 256) {  // 16 rows x 32 float4
      const int k = e >> 5, n4 = (e & 31) * 4;
      const long long m = m0 + k;
      float4 av = make_float4(0.f, 0.f, 0.f, 0.f), bv = av;
      if (m < mend) {
        if (a_vec && a0 + n4 + 3 < N1) av = *reinterpret_cast<const float4*>(A + m * lda + a0 + n4);
        else
          for (int c = 0; c < 4; ++c)
            if (a0 + n4 + c < N1) (&av.x)[c] = A[m * lda + a0 + n4 + c];
        if (b_vec && b0 + n4 + 3 < N2) bv = *reinterpret_cast<const float4*>(B + m * ldb + b0 + n4);
        else
          for (int c = 0; c < 4; ++c)
            if (b0 + n4 + c < N2) (&bv.x)[c] = B[m * ldb + b0 + n4 + c];
      }
      *reinterpret_cast<float4*>(&As[k][n4]) = av;
      *reinterpret_cast<float4*>(&Bs[k][n4]) = bv;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 a0v = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      const float4 a1v = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      const float4 b0v = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float4 b1v = *reinterpret_cast<const float4*>(&Bs[k][64 + tx * 4]);
      const float a[8] = {a0v.x, a0v.y, a0v.z, a0v.w, a1v.x, a1v.y, a1v.z, a1v.w};
      const float b[8] = {b0v.x, b0v.y, b0v.z, b0v.w, b1v.x, b1v.y, b1v.z, b1v.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int r = a0 + ty * 8 + i;
      const int c = b0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (r < N1 && c < N2) atomicAdd(&C[(long long)r * ldc + c], acc[i][j]);
    }
}

int launch_gemm_tn_atomic(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N1, int N2,
                          cudaStream_t s) {
  dim3 grid(cdiv(M, TN_CHUNK), cdiv(N1, 128), cdiv(N2, 128));
  const int a_vec = (lda % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const int b_vec = (ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);
  k_gemm_tn_atomic<<<grid, 256, 0, s>>>(A, lda, B, ldb, C, ldc, M, N1, N2, a_vec, b_vec);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// =====================================================================================
// Thin-output Chebyshev conv (Fout <= 4, the 64 -> 3 head of the network), weights first:
//   Y = X (W0 - W2) + L~ ( X W1 + 2 L~ (X W2) ) + b
// algebraically identical to [T0|T1|T2] W^T (T2 = 2 L~ L~ X - X) but the SpMMs act on 3-wide rows
// instead of Fin-wide ones, and the basis is never materialised: HBM traffic = read X once.
// =====================================================================================
// transformed weights wt[f][j], j = 4*k' + n (n < fout <= 4):  k'=0: W0-W2, 1: W1, 2: W2

__global__ void k_thin_prep(const float* __restrict__ W, int fin, int fout, float* __restrict__ out) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= fin * 12) return;
  int f = idx / 12, j = idx % 12, kk = j / 4, n = j % 4;
  float v = 0.f;
  if (n < fout) {
    const float* wr = W + (size_t)n * fin * 3 + (size_t)f * 3;  // reference layout: column = f*3 + k
    v = (kk == 0) ? (wr[0] - wr[2]) : wr[kk];
  }
  out[idx] = v;
}

// Z[r][12] = X[r][:] * Wt ; one thread per row, rows staged through shared memory (coalesced loads).
template <int FIN>
__global__ void __launch_bounds__(128) k_thin_gemm(const float* __restrict__ x, int in_unpool, long long rows,
                                                   const float* __restrict__ wt, float* __restrict__ Z) {
  __shared__ float xs[128][FIN + 1];
  __shared__ float ws[FIN * 12];
  const int tid = threadIdx.x;
  for (int i = tid; i < FIN * 12; i += 128) ws[i] = wt[i];
  const long long r0 = (long long)blockIdx.x * 128;
  for (int e = tid; e < 128 * (FIN / 4); e += 128) {
    const int row = e / (FIN / 4), c4 = e % (FIN / 4);
    const long long r = r0 + row;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < rows) v = reinterpret_cast<const float4*>(x + (in_unpool ? (r >> 1) : r) * FIN)[c4];
    xs[row][c4 * 4 + 0] = v.x;
    xs[row][c4 * 4 + 1] = v.y;
    xs[row][c4 * 4 + 2] = v.z;
    xs[row][c4 * 4 + 3] = v.w;
  }
  __syncthreads();
  float acc[12];
#pragma unroll
  for (int j = 0; j < 12; ++j) acc[j] = 0.f;
#pragma unroll 4
  for (int f = 0; f < FIN; ++f) {
    const float xv = xs[tid][f];
#pragma unroll
    for (int j = 0; j < 12; ++j) acc[j] = fmaf(xv, ws[f * 12 + j], acc[j]);
  }
  const long long r = r0 + tid;
  if (r < rows) {
    float4* zr = reinterpret_cast<float4*>(Z + r * 12);
    zr[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    zr[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    zr[2] = make_float4(acc[8], acc[9], acc[10], acc[11]);
  }
}

// U = Z1 + 2 L~ Z2   (written over the Z1 slot is not possible: neighbours still need Z2; separate buffer)
__global__ void __launch_bounds__(256) k_thin_u(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                const float* __restrict__ val, int V, long long rows,
                                                const float* __restrict__ Z, float* __restrict__ U) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  int v = (int)(r % V);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = rowptr[v]; p < rowptr[v + 1]; ++p) {
    const float4 z2 = reinterpret_cast<const float4*>(Z + (r + reloff[p]) * 12)[2];
    const float w = 2.f * val[p];
    acc.x = fmaf(w, z2.x, acc.x); acc.y = fmaf(w, z2.y, acc.y); acc.z = fmaf(w, z2.z, acc.z); acc.w = fmaf(w, z2.w, acc.w);
  }
  const float4 z1 = reinterpret_cast<const float4*>(Z + r * 12)[1];
  reinterpret_cast<float4*>(U)[r] = make_float4(acc.x + z1.x, acc.y + z1.y, acc.z + z1.z, acc.w + z1.w);
}

__global__ void __launch_bounds__(256) k_thin_out(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                  const float* __restrict__ val, int V, long long rows, int fout,
                                                  const float* __restrict__ Z, const float* __restrict__ U, EpiDev ep,
                                                  float* __restrict__ y) {
  long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  int v = (int)(r % V);
  float4 acc = reinterpret_cast<const float4*>(Z + r * 12)[0];
  for (int p = rowptr[v]; p < rowptr[v + 1]; ++p) {
    const float4 u = reinterpret_cast<const float4*>(U)[r + reloff[p]];
    const float w = val[p];
    acc.x = fmaf(w, u.x, acc.x); acc.y = fmaf(w, u.y, acc.y); acc.z = fmaf(w, u.z, acc.z); acc.w = fmaf(w, u.w, acc.w);
  }
  const float o[4] = {acc.x, acc.y, acc.z, acc.w};
  long long ro = r;
  if (ep.out_map != nullptr) {  // fused perm_reverse gather: keep only the real vertices, in mesh order
    const int slot = ep.out_map[v];
    if (slot < 0) return;
    ro = (r / V) * ep.out_rows + slot;
  }
  for (int n = 0; n < fout; ++n) y[ro * fout + n] = apply_epilogue(o[n], r, n, ep);
}

int launch_thin_prep(const float* W, int fin, int fout, float* wt, cudaStream_t s) {
  k_thin_prep<<<cdiv(fin * 12, 128), 128, 0, s>>>(W, fin, fout, wt);
  P2M_LAUNCH_OK();
  return P2M_OK;
}
int launch_thin_tail(const DevLevel& g, int rows, int fout, const float* Z, float* U, const Epilogue& e, float* y,
                     cudaStream_t s) {
  k_thin_u<<<cdiv(rows, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, Z, U);
  P2M_LAUNCH_OK();
  k_thin_out<<<cdiv(rows, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, fout, Z, U, to_dev(e), y);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

bool thin_conv_supported(int fin, int fout) { return fout <= 4 && (fin == 64 || fin == 32); }
size_t thin_conv_scratch_floats(long long rows, int fin) { return (size_t)rows * 16 + (size_t)fin * 12; }

int launch_thin_conv(const DevLevel& g, const float* x, int in_unpool, int rows, int fin, int fout, const float* W,
                     const Epilogue& e, float* scratch, float* y, cudaStream_t s) {
  float* Z = scratch;                       // [rows][12]
  float* U = Z + (size_t)rows * 12;         // [rows][4]
  float* wt = U + (size_t)rows * 4;         // [fin][12]
  k_thin_prep<<<cdiv(fin * 12, 128), 128, 0, s>>>(W, fin, fout, wt);
  P2M_LAUNCH_OK();
  const int grid = cdiv(rows, 128);
  if (fin == 64)
    k_thin_gemm<64><<<grid, 128, 0, s>>>(x, in_unpool, rows, wt, Z);
  else
    k_thin_gemm<32><<<grid, 128, 0, s>>>(x, in_unpool, rows, wt, Z);
  P2M_LAUNCH_OK();
  k_thin_u<<<cdiv(rows, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, Z, U);
  P2M_LAUNCH_OK();
  k_thin_out<<<cdiv(rows, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, fout, Z, U, to_dev(e), y);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// =====================================================================================
// Backward of the thin head (Fout <= 4), weights first as well.  With G = [dz | L~ dz | 2 L~ (L~ dz) - dz] (three
// 4-wide row blocks; L~ is symmetric):
//     dX[row, f]      = sum_{k,n} G_k[row, n] * W[n, f*3 + k]
//     dW[n, f*3 + k]  = sum_rows  G_k[row, n] * X[row, f]
// i.e. the sparse products act on the 3-wide gradient instead of the Fin-wide basis, X is read once, and neither
// the [rows, 3 Fin] basis nor dT = dz W is ever materialised (the generic path writes and re-reads both).
// =====================================================================================
__global__ void __launch_bounds__(256) k_thin_bwd_g1(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                     const float* __restrict__ val, int V, long long rows, int fout,
                                                     const float* __restrict__ dz, float* __restrict__ G) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int v = (int)(r % V);
  float g0[4] = {0.f, 0.f, 0.f, 0.f}, g1[4] = {0.f, 0.f, 0.f, 0.f};
  for (int n = 0; n < fout; ++n) g0[n] = dz[r * fout + n];
  for (int p = rowptr[v]; p < rowptr[v + 1]; ++p) {
    const float* d = dz + (r + reloff[p]) * fout;
    const float w = val[p];
    for (int n = 0; n < fout; ++n) g1[n] = fmaf(w, d[n], g1[n]);
  }
  float4* g = reinterpret_cast<float4*>(G + r * 12);
  g[0] = make_float4(g0[0], g0[1], g0[2], g0[3]);
  g[1] = make_float4(g1[0], g1[1], g1[2], g1[3]);
}
__global__ void __launch_bounds__(256) k_thin_bwd_g2(const int* __restrict__ rowptr, const int* __restrict__ reloff,
                                                     const float* __restrict__ val, int V, long long rows,
                                                     float* __restrict__ G) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int v = (int)(r % V);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = rowptr[v]; p < rowptr[v + 1]; ++p) {
    const float4 g1 = reinterpret_cast<const float4*>(G + (r + reloff[p]) * 12)[1];
    const float w = 2.f * val[p];
    acc.x = fmaf(w, g1.x, acc.x); acc.y = fmaf(w, g1.y, acc.y); acc.z = fmaf(w, g1.z, acc.z); acc.w = fmaf(w, g1.w, acc.w);
  }
  float4* g = reinterpret_cast<float4*>(G + r * 12);
  const float4 g0 = g[0];
  g[2] = make_float4(acc.x - g0.x, acc.y - g0.y, acc.z - g0.z, acc.w - g0.w);
}
// wt[f][4k + n] = W[n][f*3 + k]  (zero for n >= fout)
__global__ void k_thin_bwd_prep(const float* __restrict__ W, int fin, int fout, float* __restrict__ wt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= fin * 12) return;
  const int f = i / 12, j = i % 12, k = j >> 2, n = j & 3;
  wt[i] = (n < fout) ? W[(size_t)n * fin * 3 + f * 3 + k] : 0.f;
}
// Persistent CTAs (256 threads) over 128-row tiles; thread = (row slot 0..15, feature quad 0..FIN/4-1... ) with
// FIN = 64: 16 quads.  The thread keeps its 4 x 12 weights and its 4 x 12 dW accumulators in registers; G rows
// come from shared memory (broadcast), X and dX are accessed 256 bytes per row and half-warp (coalesced).
template <int FIN>
__global__ void __launch_bounds__(256) k_thin_bwd_main(const float* __restrict__ x, long long rows, int fout,
                                                       const float* __restrict__ G, const float* __restrict__ wt,
                                                       float* __restrict__ dx, float* __restrict__ dw) {
  static_assert(FIN == 64, "one feature quad per lane of a half-warp");
  __shared__ __align__(16) float gs[128][12];
  __shared__ float red[12][FIN];
  const int tid = threadIdx.x;
  const int q = tid & 15, slot = tid >> 4;
  float w[4][12], acc[4][12];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int j = 0; j < 12; ++j) {
      w[e][j] = wt[(4 * q + e) * 12 + j];
      acc[e][j] = 0.f;
    }
  for (int i = tid; i < 12 * FIN; i += 256) (&red[0][0])[i] = 0.f;
  const long long n_tiles = (rows + 127) / 128;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const long long r0 = t * 128;
    __syncthreads();  // the previous tile's readers of gs are done
    for (int i = tid; i < 128 * 3; i += 256) {
      const long long r = r0 + i / 3;
      reinterpret_cast<float4*>(&gs[0][0])[i] =
          (r < rows) ? reinterpret_cast<const float4*>(G + r * 12)[i % 3] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
#pragma unroll 2
    for (int rr = slot; rr < 128; rr += 16) {
      const long long r = r0 + rr;
      if (r >= rows) break;
      const float4 g0 = *reinterpret_cast<const float4*>(&gs[rr][0]);
      const float4 g1 = *reinterpret_cast<const float4*>(&gs[rr][4]);
      const float4 g2 = *reinterpret_cast<const float4*>(&gs[rr][8]);
      const float g[12] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w, g2.x, g2.y, g2.z, g2.w};
      const float4 xv = *reinterpret_cast<const float4*>(x + r * FIN + 4 * q);
      const float xe[4] = {xv.x, xv.y, xv.z, xv.w};
      float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int j = 0; j < 12; ++j) {
          o[e] = fmaf(g[j], w[e][j], o[e]);
          acc[e][j] = fmaf(g[j], xe[e], acc[e][j]);
        }
      if (dx != nullptr) *reinterpret_cast<float4*>(dx + r * FIN + 4 * q) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int j = 0; j < 12; ++j) atomicAdd(&red[j][4 * q + e], acc[e][j]);
  __syncthreads();
  for (int i = tid; i < 12 * FIN; i += 256) {
    const int j = i / FIN, f = i % FIN, k = j >> 2, n = j & 3;
    if (n < fout) atomicAdd(dw + (size_t)n * FIN * 3 + f * 3 + k, red[j][f]);
  }
}
bool thin_conv_bwd_supported(int fin, int fout) { return fout <= 4 && fin == 64; }
size_t thin_conv_bwd_scratch_floats(long long rows, int fin) { return (size_t)rows * 12 + (size_t)fin * 12; }
int launch_thin_conv_bwd(const DevLevel& g, const float* x, int rows, int fin, int fout, const float* W, const float* dz,
                         float* scratch, float* dx, float* dw, int sm_count, cudaStream_t s) {
  if (!thin_conv_bwd_supported(fin, fout)) {
    set_error("thin_conv_bwd: unsupported shape");
    return P2M_ERR_INVALID;
  }
  float* G = scratch;                       // [rows][12]
  float* wt = G + (size_t)rows * 12;        // [fin][12]
  k_thin_bwd_prep<<<cdiv(fin * 12, 128), 128, 0, s>>>(W, fin, fout, wt);
  P2M_LAUNCH_OK();
  k_thin_bwd_g1<<<cdiv(rows, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, fout, dz, G);
  P2M_LAUNCH_OK();
  k_thin_bwd_g2<<<cdiv(rows, 256), 256, 0, s>>>(g.rowptr, g.reloff, g.val, g.V, rows, G);
  P2M_LAUNCH_OK();
  P2M_CUDA_OK(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)fout * 3 * fin, s));
  const int grid = (int)std::min<long long>(((long long)rows + 127) / 128, (long long)sm_count * 4);
  k_thin_bwd_main<64><<<grid, 256, 0, s>>>(x, rows, fout, G, wt, dx, dw);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// =====================================================================================
// power-of-two scale that brings a tensor into fp16's comfortable range (tensor-core backward GEMMs)
// =====================================================================================
__global__ void __launch_bounds__(256) k_absmax(const float* __restrict__ x, long long n, unsigned int* __restrict__ out) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(x[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(out, __float_as_uint(m));  // non-negative floats order as uints
}
// the scale replaces max|x| in io, or goes to out (io zeroed for the next accumulation)
__global__ void k_scale_from_absmax(unsigned int* io, float* out, int headroom_log2) {
  const float m = __uint_as_float(*io);
  float s = 1.f;
  if (m > 0.f && isfinite(m)) {
    int e;
    frexpf(m, &e);                            // m = f * 2^e, f in [0.5, 1)
    s = ldexpf(1.f, 10 - e - headroom_log2);  // m * s in [2^(9-h), 2^(10-h))
  }
  if (out == nullptr) {
    *reinterpret_cast<float*>(io) = s;
  } else {
    *out = s;
    *io = 0u;
  }
}
// SMs of the current device: the grid-stride kernels below size their grids by it
static int current_sm_count(int* sms) {
  int dev = 0;
  P2M_CUDA_OK(cudaGetDevice(&dev));
  P2M_CUDA_OK(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return P2M_OK;
}
int launch_absmax_scale(const float* x, long long n, float* scale_out, cudaStream_t s, int headroom_log2) {
  P2M_CUDA_OK(cudaMemsetAsync(scale_out, 0, sizeof(float), s));
  int sms = 0;
  P2M_TRY(current_sm_count(&sms));
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sms * 8);
  k_absmax<<<grid, 256, 0, s>>>(x, n, reinterpret_cast<unsigned int*>(scale_out));
  P2M_LAUNCH_OK();
  k_scale_from_absmax<<<1, 1, 0, s>>>(reinterpret_cast<unsigned int*>(scale_out), nullptr, headroom_log2);
  P2M_LAUNCH_OK();
  return P2M_OK;
}
int launch_absmax_finish(unsigned int* amax, float* scale_out, cudaStream_t s, int headroom_log2) {
  k_scale_from_absmax<<<1, 1, 0, s>>>(amax, scale_out, headroom_log2);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

__global__ void __launch_bounds__(256) k_scale_by(const float* __restrict__ x, long long n, const float* __restrict__ sp,
                                                  int invert, float mul, float* __restrict__ y) {
  const float f = (invert ? 1.f / *sp : *sp) * mul;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = x[i] * f;
}
int launch_scale_by(const float* x, long long n, const float* scale, int invert, float mul, float* y, cudaStream_t s) {
  if (n <= 0) return P2M_OK;
  int sms = 0;
  P2M_TRY(current_sm_count(&sms));
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)sms * 8);
  k_scale_by<<<grid, 256, 0, s>>>(x, n, scale, invert, mul, y);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

__global__ void k_rescaled_epilogue(const float* __restrict__ bias, const float* __restrict__ scale,
                                    const float* __restrict__ shift, const float* __restrict__ w_scale, float w_packed,
                                    int n, float* __restrict__ out_scale, float* __restrict__ out_shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float sc = scale ? scale[i] : 1.f;
  out_scale[i] = sc * (w_packed / *w_scale);
  out_shift[i] = fmaf(bias ? bias[i] : 0.f, sc, shift ? shift[i] : 0.f);
}
int launch_rescaled_epilogue(const Epilogue& ep, const float* w_scale, float w_packed, int n, float* out_scale,
                             float* out_shift, cudaStream_t s) {
  k_rescaled_epilogue<<<(n + 127) / 128, 128, 0, s>>>(ep.bias, ep.scale, ep.shift, w_scale, w_packed, n, out_scale,
                                                      out_shift);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// =====================================================================================
// small helpers
// =====================================================================================
__global__ void k_permute_w(const float* __restrict__ W, float* __restrict__ Wp, int fout, int fin, int inverse) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= fout * fin * 3) return;
  int n = idx / (fin * 3), c = idx % (fin * 3);
  int f = c / 3, k = c % 3;  // reference column c = f*3 + k  (cheby_graph_conv.py:32-34)
  int cp = k * fin + f;      // ours: k-major blocks
  if (!inverse)
    Wp[n * fin * 3 + cp] = W[idx];
  else
    Wp[idx] = W[n * fin * 3 + cp];
}
int launch_permute_w(const float* W, float* Wp, int fout, int fin, cudaStream_t s) {
  k_permute_w<<<cdiv(fout * fin * 3, 256), 256, 0, s>>>(W, Wp, fout, fin, 0);
  P2M_LAUNCH_OK();
  return P2M_OK;
}
int launch_unpermute_w(const float* Wp, float* W, int fout, int fin, cudaStream_t s) {
  k_permute_w<<<cdiv(fout * fin * 3, 256), 256, 0, s>>>(Wp, W, fout, fin, 1);
  P2M_LAUNCH_OK();
  return P2M_OK;
}
__global__ void __launch_bounds__(256) k_copy_rows(float* __restrict__ y, long long mesh_stride, int F,
                                                   const int* __restrict__ dst, const int* __restrict__ src, int n,
                                                   long long total) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // (b, i, f)
  if (idx >= total) return;
  const int f = (int)(idx % F);
  const long long t = idx / F;
  const int i = (int)(t % n);
  const long long b = t / n;
  y[b * mesh_stride + (long long)dst[i] * F + f] = y[b * mesh_stride + (long long)src[i] * F + f];
}
int launch_copy_rows(float* y, int batch, int V, int F, const int* dst, const int* src, int n, cudaStream_t s) {
  if (n <= 0) return P2M_OK;
  const long long total = (long long)batch * n * F;
  k_copy_rows<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(y, (long long)V * F, F, dst, src, n, total);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int launch_fill_zero(void* p, size_t bytes, cudaStream_t s) {
  P2M_CUDA_OK(cudaMemsetAsync(p, 0, bytes, s));
  return P2M_OK;
}

// =====================================================================================
// BatchNorm1d over rows
// =====================================================================================
// scale / shift of a BatchNorm with running statistics: ((z + bias) - rm) * scale + beta.  bias == nullptr (a z that
// already carries its bias: the frozen-statistics training path) folds none; save_mean / save_invstd (optional) take
// rm and 1 / sqrt(rv + eps), what the BatchNorm backward reads
__global__ void k_bn_fold_eval(const float* gamma, const float* beta, const float* rm, const float* rv,
                               const float* bias, float eps, float* scale, float* shift, float* save_mean,
                               float* save_invstd, int F) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= F) return;
  float sc = gamma[c] / sqrtf(rv[c] + eps);
  scale[c] = sc;
  float b = bias ? bias[c] : 0.f;
  shift[c] = beta[c] + (b - rm[c]) * sc;   // ((z + b) - rm) * sc + beta
  if (save_mean) save_mean[c] = rm[c];
  if (save_invstd) save_invstd[c] = 1.f / sqrtf(rv[c] + eps);
}
int launch_bn_fold_eval(const float* gamma, const float* beta, const float* rm, const float* rv, const float* bias,
                        double eps, float* scale, float* shift, int F, cudaStream_t s, float* save_mean,
                        float* save_invstd) {
  k_bn_fold_eval<<<cdiv(F, 128), 128, 0, s>>>(gamma, beta, rm, rv, bias, (float)eps, scale, shift, save_mean,
                                              save_invstd, F);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// per-channel sum / sum of squares of the SHIFTED data z - K, K = z[0][f] (k_bn_finalize reads the same K).  The
// plain sums cancel catastrophically in var = E[z^2] - mean^2 once |mean| >> std (a constant in front of the BN);
// around a sample of the channel they stay of the order of the variance.  Block = 256 threads = (F-lanes x
// row-lanes); fp32 partials over <= STAT_ROWS/rl rows, fp64 across blocks.  Every thread runs the same number of
// channel rounds (the barriers inside), also when F > 256 is not a multiple of 256.
constexpr int STAT_ROWS = 512;
__global__ void __launch_bounds__(256) k_col_stats(const float* __restrict__ z, long long rows, int F,
                                                   double* __restrict__ sums) {
  extern __shared__ float sm[];  // [2][256]
  const int lanes = min(F, 256);
  const int rl = 256 / lanes;
  const int fl = threadIdx.x % lanes, rr = threadIdx.x / lanes;
  const long long rbeg = (long long)blockIdx.x * STAT_ROWS;
  const long long rend = min(rows, rbeg + STAT_ROWS);
  for (int f0 = 0; f0 < F; f0 += lanes) {
    const int f = f0 + fl;
    const bool live = f < F;
    float s = 0.f, q = 0.f;
    if (rr < rl && live) {
      const float k = z[f];
      for (long long r = rbeg + rr; r < rend; r += rl) {
        const float v = z[r * F + f] - k;
        s += v;
        q = fmaf(v, v, q);
      }
    }
    sm[threadIdx.x] = s;
    sm[256 + threadIdx.x] = q;
    __syncthreads();
    if (rr == 0 && live) {
      for (int j = 1; j < rl; ++j) {
        s += sm[j * lanes + fl];
        q += sm[256 + j * lanes + fl];
      }
      atomicAdd(&sums[f], (double)s);
      atomicAdd(&sums[F + f], (double)q);
    }
    __syncthreads();
  }
}
int launch_col_stats(const float* z, int rows, int F, double* sums, cudaStream_t s) {
  P2M_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * F, s));
  k_col_stats<<<cdiv(rows, STAT_ROWS), 256, 2 * 256 * sizeof(float), s>>>(z, rows, F, sums);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// sums = k_col_stats' (S, Q) of z - K around K = z[0][c]:  mean = K + S/n,  var = Q/n - (S/n)^2.
// update: running statistics (and num_batches_tracked) take the batch's, with factor `momentum`, or with cumulative
// 1 / num_batches_tracked read here after k_nbt_add1 incremented it.  Otherwise rm / rv / nbt are not touched.
__global__ void k_bn_finalize(const double* __restrict__ sums, const float* __restrict__ z, long long rows, int F,
                              const float* gamma, const float* beta, float* rm, float* rv, long long* nbt,
                              double eps, float momentum, int cumulative, int update, float* save_mean,
                              float* save_invstd, float* scale, float* shift) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (update && !cumulative && c == 0 && nbt) *nbt += 1;
  if (c >= F) return;
  double n = (double)rows;
  double d = sums[c] / n;
  double mean = (double)z[c] + d;
  double var = sums[F + c] / n - d * d;
  if (var < 0) var = 0;
  float invstd = (float)(1.0 / sqrt(var + eps));
  if (update) {
    const float mom = cumulative ? (float)(1.0 / (double)*nbt) : momentum, keep = 1.f - mom;
    const float var_u = (float)(rows > 1 ? var * n / (n - 1.0) : var);  // unbiased
    if (rm) rm[c] = fmaf(mom, (float)mean, __fmul_rn(keep, rm[c]));
    if (rv) rv[c] = fmaf(keep, rv[c], __fmul_rn(mom, var_u));
  }
  if (save_mean) save_mean[c] = (float)mean;
  if (save_invstd) save_invstd[c] = invstd;
  float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = beta[c] - (float)mean * sc;
}
__global__ void k_nbt_add1(long long* nbt) { *nbt += 1; }
int launch_bn_finalize(const double* sums, const float* z, int rows, int F, const float* gamma, const float* beta,
                       float* rm, float* rv, int64_t* nbt, const p2m_bn_opts_t& o, float* save_mean,
                       float* save_invstd, float* scale, float* shift, cudaStream_t s) {
  const int update = o.stats == P2M_BN_BATCH_UPDATE;
  if (update && o.cumulative) {  // a separate launch: every block of the finalize reads the incremented count
    k_nbt_add1<<<1, 1, 0, s>>>((long long*)nbt);
    P2M_LAUNCH_OK();
  }
  k_bn_finalize<<<cdiv(F, 128), 128, 0, s>>>(sums, z, rows, F, gamma, beta, rm, rv, (long long*)nbt, o.eps,
                                             (float)o.momentum, o.cumulative, update, save_mean, save_invstd, scale,
                                             shift);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int check_bn_opts(const p2m_bn_opts_t& o, const void* rm, const void* rv, const void* nbt, const char* where) {
  const bool stats_ok = o.stats == P2M_BN_BATCH_UPDATE || o.stats == P2M_BN_BATCH || o.stats == P2M_BN_RUNNING;
  if (!stats_ok || !(o.eps >= 0.0) || !(o.cumulative || (o.momentum >= 0.0 && o.momentum <= 1.0))) {
    set_error(std::string(where) + ": bad BatchNorm options (stats, eps or momentum)");
    return P2M_ERR_INVALID;
  }
  if (o.stats != P2M_BN_BATCH && (!rm || !rv)) {
    set_error(std::string(where) + ": BatchNorm without running statistics needs stats = P2M_BN_BATCH");
    return P2M_ERR_INVALID;
  }
  if (o.stats == P2M_BN_BATCH_UPDATE && o.cumulative && !nbt) {
    set_error(std::string(where) + ": a cumulative running average needs num_batches_tracked");
    return P2M_ERR_INVALID;
  }
  return P2M_OK;
}

int launch_bn_stats(const float* z, int rows, int F, const float* gamma, const float* beta, float* rm, float* rv,
                    int64_t* nbt, const p2m_bn_opts_t& o, double* sums, float* mean, float* invstd, float* scale,
                    float* shift, cudaStream_t s) {
  if (o.stats == P2M_BN_RUNNING)
    return launch_bn_fold_eval(gamma, beta, rm, rv, nullptr, o.eps, scale, shift, F, s, mean, invstd);
  P2M_TRY(launch_col_stats(z, rows, F, sums, s));
  return launch_bn_finalize(sums, z, rows, F, gamma, beta, rm, rv, nbt, o, mean, invstd, scale, shift, s);
}

__global__ void __launch_bounds__(256) k_affine_act(const float* __restrict__ z, long long rows, int F,
                                                    const float* __restrict__ scale, const float* __restrict__ shift,
                                                    int relu, const float* __restrict__ res, int res_F, int res_unpool,
                                                    const int* __restrict__ i0, const int* __restrict__ i1,
                                                    const float* __restrict__ lam, float* __restrict__ a) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * F) return;
  long long r = idx / F;
  int n = (int)(idx - r * F);
  float v = z[idx];
  if (scale) v = fmaf(v, scale[n], shift[n]);
  if (relu) v = fmaxf(v, 0.f);
  if (res) {
    const float* rr = res + (res_unpool ? (r >> 1) : r) * res_F;
    float l = lam[n];
    v += (1.f - l) * rr[i0[n]] + l * rr[i1[n]];
  }
  a[idx] = v;
}
// four channels per thread (F % 4 == 0, 16-byte aligned tensors); identity residual (res_F == F) as one 16-byte load
__global__ void __launch_bounds__(256) k_affine_act4(const float4* __restrict__ z, long long n4, int F4,
                                                     const float4* __restrict__ scale, const float4* __restrict__ shift,
                                                     int relu, const float* __restrict__ res, int res_F, int res_unpool,
                                                     const int* __restrict__ i0, const int* __restrict__ i1,
                                                     const float* __restrict__ lam, float4* __restrict__ a) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n4) return;
  const long long r = idx / F4;
  const int c = (int)(idx - r * F4);
  float4 v = z[idx];
  if (scale) {
    const float4 sc = __ldg(scale + c), sh = __ldg(shift + c);
    v.x = fmaf(v.x, sc.x, sh.x); v.y = fmaf(v.y, sc.y, sh.y); v.z = fmaf(v.z, sc.z, sh.z); v.w = fmaf(v.w, sc.w, sh.w);
  }
  if (relu) {
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
  }
  if (res) {
    const float* rr = res + (res_unpool ? (r >> 1) : r) * res_F;
    if (res_F == 4 * F4) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(rr) + c);
      v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    } else {
      float* ve = &v.x;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = 4 * c + e;
        const float l = lam[n];
        ve[e] += (1.f - l) * rr[i0[n]] + l * rr[i1[n]];
      }
    }
  }
  a[idx] = v;
}
int launch_affine_act(const float* z, int rows, int F, const float* scale, const float* shift, int relu,
                      const float* res, int res_F, int res_unpool, const InterpTable* it, float* a, cudaStream_t s) {
  const bool al = ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(scale) |
                    reinterpret_cast<uintptr_t>(shift) | reinterpret_cast<uintptr_t>(res)) & 15) == 0;
  if (F % 4 == 0 && al && (res == nullptr || res_F % 4 == 0)) {
    const long long n4 = (long long)rows * (F / 4);
    k_affine_act4<<<cdiv(n4, 256), 256, 0, s>>>(reinterpret_cast<const float4*>(z), n4, F / 4,
                                                reinterpret_cast<const float4*>(scale),
                                                reinterpret_cast<const float4*>(shift), relu, res, res_F, res_unpool,
                                                it ? it->i0 : nullptr, it ? it->i1 : nullptr, it ? it->lam : nullptr,
                                                reinterpret_cast<float4*>(a));
    P2M_LAUNCH_OK();
    return P2M_OK;
  }
  k_affine_act<<<cdiv((long long)rows * F, 256), 256, 0, s>>>(z, rows, F, scale, shift, relu, res, res_F, res_unpool,
                                                             it ? it->i0 : nullptr, it ? it->i1 : nullptr,
                                                             it ? it->lam : nullptr, a);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// BN + ReLU backward.  Pass 1: s1 = sum g', s2 = sum g' * zhat  with g' = g_a * [bn(z) > 0].
__global__ void __launch_bounds__(256) k_bn_bwd_reduce(const float* __restrict__ z, const float* __restrict__ g_a,
                                                       long long rows, int F, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, const float* __restrict__ mean,
                                                       const float* __restrict__ invstd, int relu,
                                                       double* __restrict__ sums) {
  extern __shared__ float sm[];
  const int lanes = min(F, 256);
  const int rl = 256 / lanes;
  const int fl = threadIdx.x % lanes, rr = threadIdx.x / lanes;
  const long long rbeg = (long long)blockIdx.x * STAT_ROWS;
  const long long rend = min(rows, rbeg + STAT_ROWS);
  for (int f = fl; f < F; f += lanes) {
    float s = 0.f, q = 0.f;
    if (rr < rl) {
      float mu = mean[f], is = invstd[f], sc = scale[f], sh = shift[f];
      for (long long r = rbeg + rr; r < rend; r += rl) {
        float zv = z[r * F + f];
        float zh = (zv - mu) * is;
        float g = g_a[r * F + f];
        if (relu && !(fmaf(zv, sc, sh) > 0.f)) g = 0.f;  // exactly the forward's activation test
        s += g;
        q = fmaf(g, zh, q);
      }
    }
    sm[threadIdx.x] = s;
    sm[256 + threadIdx.x] = q;
    __syncthreads();
    if (rr == 0) {
      for (int j = 1; j < rl; ++j) {
        s += sm[j * lanes + fl];
        q += sm[256 + j * lanes + fl];
      }
      atomicAdd(&sums[f], (double)s);
      atomicAdd(&sums[F + f], (double)q);
    }
    __syncthreads();
  }
}
__global__ void __launch_bounds__(256) k_bn_bwd_apply(const float* __restrict__ z, const float* __restrict__ g_a,
                                                      long long rows, int F, const float* __restrict__ gamma,
                                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                                      const float* __restrict__ mean,
                                                      const float* __restrict__ invstd, int relu, int frozen,
                                                      const double* __restrict__ sums, float* __restrict__ dgamma,
                                                      float* __restrict__ dbeta, float* __restrict__ dbias,
                                                      float* __restrict__ g_z) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < F) {
    dbeta[idx] = (float)sums[idx];
    dgamma[idx] = (float)sums[F + idx];
    if (dbias) dbias[idx] = (float)(sums[idx] * (double)(gamma[idx] * invstd[idx]));
  }
  if (idx >= rows * F) return;
  int f = (int)(idx % F);
  float zv = z[idx];
  float zh = (zv - mean[f]) * invstd[f];
  float g = g_a[idx];
  if (relu && !(fmaf(zv, scale[f], shift[f]) > 0.f)) g = 0.f;
  if (frozen) {
    g_z[idx] = gamma[f] * invstd[f] * g;
    return;
  }
  float m1 = (float)(sums[f] / (double)rows);
  float m2 = (float)(sums[F + f] / (double)rows);
  g_z[idx] = gamma[f] * invstd[f] * (g - m1 - zh * m2);
}
// BN + ReLU backward, pass 2, as a per-channel affine map:  g_z = a g' + b z + c  with
//   a = gamma invstd,  b = -a invstd m2,  c = -a m1 + a invstd m2 mean,   m1 = s1 / rows, m2 = s2 / rows
// (g_z = gamma invstd (g' - m1 - zhat m2), zhat = (z - mean) invstd), g' = g_a masked by the forward's own
// activation test fma(z, scale, shift) > 0.  k_bn_bwd_coef builds coef[5][F] = a | b | c | scale | shift once per
// layer; the streaming kernel then needs five 16-byte coefficient loads per four channels and no fp64.
// frozen (running statistics, constants of the forward): g_z = a g', b = c = 0, and the bias in front of the BatchNorm
// gets sum_rows g_z = a s1 (dbias, optional).
__global__ void k_bn_bwd_coef(const double* __restrict__ sums, long long rows, int F, const float* __restrict__ gamma,
                              const float* __restrict__ scale, const float* __restrict__ shift,
                              const float* __restrict__ mean, const float* __restrict__ invstd, int frozen,
                              float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ dbias,
                              float* __restrict__ coef) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  dbeta[f] = (float)sums[f];
  dgamma[f] = (float)sums[F + f];
  const float m1 = (float)(sums[f] / (double)rows), m2 = (float)(sums[F + f] / (double)rows);
  const float a = gamma[f] * invstd[f];
  coef[f] = a;
  if (frozen) {
    coef[F + f] = 0.f;
    coef[2 * F + f] = 0.f;
    coef[3 * F + f] = scale[f];
    coef[4 * F + f] = shift[f];
    if (dbias) dbias[f] = (float)(sums[f] * (double)a);
    return;
  }
  coef[F + f] = -a * invstd[f] * m2;
  coef[2 * F + f] = -a * m1 + a * invstd[f] * m2 * mean[f];
  coef[3 * F + f] = scale[f];
  coef[4 * F + f] = shift[f];
}
// four channels per thread; optionally folds max|g_z| into *amax (bits of a non-negative float, atomicMax): the
// power-of-two scale of the tensor-core backward GEMMs then needs no pass of its own
__global__ void __launch_bounds__(256) k_bn_bwd_apply4(const float4* __restrict__ z, const float4* __restrict__ g_a,
                                                       long long n4, int F4, int relu, const float4* __restrict__ coef,
                                                       float4* __restrict__ g_z, unsigned int* __restrict__ amax) {
  // grid-stride: a few CTAs per SM, ONE atomicMax per CTA (per-warp atomics on a single address serialise in L2 and
  // cost more than the whole streaming pass)
  float m = 0.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < n4;
       idx += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(idx % F4);
    const float4 zv = z[idx];
    float4 g = g_a[idx];
    const float4 ca = __ldg(coef + c), cb = __ldg(coef + F4 + c), cc = __ldg(coef + 2 * F4 + c);
    if (relu) {
      const float4 sc = __ldg(coef + 3 * F4 + c), sh = __ldg(coef + 4 * F4 + c);
      if (!(fmaf(zv.x, sc.x, sh.x) > 0.f)) g.x = 0.f;  // exactly the forward's activation test
      if (!(fmaf(zv.y, sc.y, sh.y) > 0.f)) g.y = 0.f;
      if (!(fmaf(zv.z, sc.z, sh.z) > 0.f)) g.z = 0.f;
      if (!(fmaf(zv.w, sc.w, sh.w) > 0.f)) g.w = 0.f;
    }
    float4 o;
    o.x = fmaf(ca.x, g.x, fmaf(cb.x, zv.x, cc.x));
    o.y = fmaf(ca.y, g.y, fmaf(cb.y, zv.y, cc.y));
    o.z = fmaf(ca.z, g.z, fmaf(cb.z, zv.z, cc.z));
    o.w = fmaf(ca.w, g.w, fmaf(cb.w, zv.w, cc.w));
    m = fmaxf(m, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
    g_z[idx] = o;
  }
  if (amax != nullptr) {
    __shared__ float red[8];
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
      if (m > 0.f) atomicMax(amax, __float_as_uint(m));
    }
  }
}
int launch_bn_relu_bwd(const float* z, const float* g_a, int rows, int F, const float* gamma, const float* scale,
                       const float* shift, const float* mean, const float* invstd, int relu, double* sums,
                       float* dgamma, float* dbeta, float* g_z, cudaStream_t s, float* gz_scale_out, int frozen,
                       float* dbias) {
  P2M_CUDA_OK(cudaMemsetAsync(sums, 0, sizeof(double) * 2 * F, s));
  k_bn_bwd_reduce<<<cdiv(rows, STAT_ROWS), 256, 2 * 256 * sizeof(float), s>>>(z, g_a, rows, F, scale, shift, mean,
                                                                               invstd, relu, sums);
  P2M_LAUNCH_OK();
  const bool al = ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(g_a) | reinterpret_cast<uintptr_t>(g_z)) & 15) == 0;
  if (F % 4 == 0 && al) {
    if (gz_scale_out) P2M_CUDA_OK(cudaMemsetAsync(gz_scale_out, 0, sizeof(float), s));
    const long long n4 = (long long)rows * (F / 4);
    float* coef = reinterpret_cast<float*>(sums + 2 * F);  // [5][F] floats behind the two fp64 sums
    k_bn_bwd_coef<<<cdiv(F, 128), 128, 0, s>>>(sums, rows, F, gamma, scale, shift, mean, invstd, frozen, dgamma, dbeta,
                                                dbias, coef);
    P2M_LAUNCH_OK();
    int sms = 0;
    P2M_TRY(current_sm_count(&sms));
    const int grid = (int)std::min<long long>((n4 + 255) / 256, (long long)sms * 16);
    k_bn_bwd_apply4<<<grid, 256, 0, s>>>(reinterpret_cast<const float4*>(z),
                                                  reinterpret_cast<const float4*>(g_a), n4, F / 4, relu,
                                                  reinterpret_cast<const float4*>(coef), reinterpret_cast<float4*>(g_z),
                                                  reinterpret_cast<unsigned int*>(gz_scale_out));
    P2M_LAUNCH_OK();
    if (gz_scale_out) {
      k_scale_from_absmax<<<1, 1, 0, s>>>(reinterpret_cast<unsigned int*>(gz_scale_out), nullptr, 0);
      P2M_LAUNCH_OK();
    }
    return P2M_OK;
  }
  k_bn_bwd_apply<<<cdiv((long long)rows * F, 256), 256, 0, s>>>(z, g_a, rows, F, gamma, scale, shift, mean, invstd, relu,
                                                               frozen, sums, dgamma, dbeta, dbias, g_z);
  P2M_LAUNCH_OK();
  if (gz_scale_out) return launch_absmax_scale(g_z, (long long)rows * F, gz_scale_out, s);
  return P2M_OK;
}

__global__ void __launch_bounds__(256) k_col_sum(const float* __restrict__ g, long long rows, int F,
                                                 double* __restrict__ sums) {
  extern __shared__ float sm[];
  const int lanes = min(F, 256);
  const int rl = 256 / lanes;
  const int fl = threadIdx.x % lanes, rr = threadIdx.x / lanes;
  const long long rbeg = (long long)blockIdx.x * STAT_ROWS;
  const long long rend = min(rows, rbeg + STAT_ROWS);
  for (int f = fl; f < F; f += lanes) {
    float s = 0.f;
    if (rr < rl)
      for (long long r = rbeg + rr; r < rend; r += rl) s += g[r * F + f];
    sm[threadIdx.x] = s;
    __syncthreads();
    if (rr == 0) {
      for (int j = 1; j < rl; ++j) s += sm[j * lanes + fl];
      atomicAdd(&sums[f], (double)s);
    }
    __syncthreads();
  }
}
__global__ void k_d2f(const double* in, float* out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i];
}
int launch_col_sum(const float* g, int rows, int F, double* scratch, float* out, cudaStream_t s) {
  P2M_CUDA_OK(cudaMemsetAsync(scratch, 0, sizeof(double) * F, s));
  k_col_sum<<<cdiv(rows, STAT_ROWS), 256, 256 * sizeof(float), s>>>(g, rows, F, scratch);
  P2M_LAUNCH_OK();
  k_d2f<<<cdiv(F, 128), 128, 0, s>>>(scratch, out, F);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // namespace p2m
