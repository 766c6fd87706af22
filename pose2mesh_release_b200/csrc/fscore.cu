// Row f9 of SURVEY.md §8: the FreiHAND benchmark's scores on the GPU (the dataset's eval.py / utils/eval_util.py):
//  * k_nearest_sweep + k_nearest_finish: bidirectional nearest-point distances between two point sets per sample,
//    their per-threshold counts and F-scores (calculate_fscore);
//  * k_align_w_scale: align_w_scale (centre, Frobenius-normalise, orthogonal Procrustes without reflection
//    correction, rescale), one CTA per sample;
//  * k_pck_hist: per-threshold counts of e <= t over (sample, point) pairs (EvalUtil.get_measures' PCK).
// Points are float32 or float64; all arithmetic is fp64 on their values, and every distance is
// sqrt((dx^2 + dy^2) + dz^2) with each step rounded to nearest (no contraction), so distances equal the float64 brute
// force bit for bit.  Minima of exact values and integer counts do not depend on order: results are bitwise
// deterministic and independent of batch position, batch size and how a sample is split over CTAs.
#include <cuda_runtime.h>

#include <cmath>
#include <string>

#include "p2m_internal.h"
#include "procrustes3.cuh"

namespace p2m {
namespace {

constexpr int MAX_BATCH = 1 << 24;
constexpr int MAX_POINTS = 1 << 20;
constexpr int MAX_PCK_POINTS = 1 << 24;
constexpr int MAX_GRID = 1 << 16;
constexpr int MAX_THR = 128;       // thresholds per call (passed by value)
constexpr int MAX_F_THR = 16;      // thresholds of an F-score call

// ---------------------------------------------------------------- nearest distances
// CTA tile: TR = 16 x RR rows of P (in registers, fixed for the CTA) against column tiles of TC = 16 x CC points of Q
// staged in shared memory (structure of arrays: conflict-free broadcast reads).  Thread (ty, tx) = (tid / 16,
// tid % 16) owns rows ty + 16 r and columns tx + 16 c.  Row minima stay in registers over all the CTA's column tiles;
// each tile's column minima are reduced over the 16 row groups in shared memory and merged into global memory with
// atomicMin on the bit pattern (non-negative doubles order like their uint64 bits).  Indices past n / m are clamped to
// the last point: a duplicate point changes no minimum, so the inner loop needs no bounds test.
constexpr int NT = 256;
constexpr int RR = 8, CC = 4;
constexpr int TR = 16 * RR, TC = 16 * CC;
constexpr unsigned long long POS_INF_BITS = 0x7ff0000000000000ull;

__device__ __forceinline__ double sq_dist(double x0, double x1, double x2, double y0, double y1, double y2) {
  const double d0 = __dsub_rn(x0, y0), d1 = __dsub_rn(x1, y1), d2 = __dsub_rn(x2, y2);
  return __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
}

__device__ __forceinline__ unsigned long long bits(double x) { return (unsigned long long)__double_as_longlong(x); }

__global__ void __launch_bounds__(NT) k_fill_inf(unsigned long long* __restrict__ a, long long na,
                                                 unsigned long long* __restrict__ b, long long nb) {
  for (long long i = (long long)blockIdx.x * NT + threadIdx.x; i < na + nb; i += (long long)gridDim.x * NT) {
    if (i < na) a[i] = POS_INF_BITS;
    else b[i - na] = POS_INF_BITS;
  }
}

// Work item w = ((b * row_tiles) + rt) * splits + sp: sample b, row tile rt, column tiles [sp * tps, (sp + 1) * tps).
// min_p[b, i] / min_q[b, j] (uint64 bits, +inf on entry) receive the squared distances' minima.
template <typename T>
__global__ void __launch_bounds__(NT) k_nearest_sweep(const T* __restrict__ P, const T* __restrict__ Q, int batch,
                                                      int n, int m, int row_tiles, int splits, int tps,
                                                      unsigned long long* __restrict__ min_p,
                                                      unsigned long long* __restrict__ min_q) {
  __shared__ double sq[3][TC];
  __shared__ double part[16][TC];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int col_tiles = (m + TC - 1) / TC;
  const long long work = (long long)batch * row_tiles * splits;
  for (long long w = blockIdx.x; w < work; w += gridDim.x) {
    const int sp = (int)(w % splits);
    const int rt = (int)((w / splits) % row_tiles);
    const long long b = w / ((long long)splits * row_tiles);
    const T* p = P + b * n * 3;
    const T* q = Q + b * m * 3;
    double x[RR][3], rmin[RR];
#pragma unroll
    for (int r = 0; r < RR; ++r) {
      const int i = min(rt * TR + ty + 16 * r, n - 1);
#pragma unroll
      for (int c = 0; c < 3; ++c) x[r][c] = (double)p[3LL * i + c];
      rmin[r] = __longlong_as_double((long long)POS_INF_BITS);
    }
    const int ct_end = min((sp + 1) * tps, col_tiles);
    for (int ct = sp * tps; ct < ct_end; ++ct) {
      __syncthreads();  // the previous tile's sq / part are consumed
      if (threadIdx.x < TC) {
        const int j = min(ct * TC + (int)threadIdx.x, m - 1);
#pragma unroll
        for (int c = 0; c < 3; ++c) sq[c][threadIdx.x] = (double)q[3LL * j + c];
      }
      __syncthreads();
      double y[CC][3], cmin[CC];
#pragma unroll
      for (int c = 0; c < CC; ++c) {
#pragma unroll
        for (int k = 0; k < 3; ++k) y[c][k] = sq[k][tx + 16 * c];
        cmin[c] = __longlong_as_double((long long)POS_INF_BITS);
      }
#pragma unroll
      for (int r = 0; r < RR; ++r)
#pragma unroll
        for (int c = 0; c < CC; ++c) {
          const double s = sq_dist(x[r][0], x[r][1], x[r][2], y[c][0], y[c][1], y[c][2]);
          rmin[r] = fmin(rmin[r], s);
          cmin[c] = fmin(cmin[c], s);
        }
#pragma unroll
      for (int c = 0; c < CC; ++c) part[ty][tx + 16 * c] = cmin[c];
      __syncthreads();
      if (threadIdx.x < TC) {
        const int j = ct * TC + (int)threadIdx.x;
        double v = part[0][threadIdx.x];
#pragma unroll
        for (int k = 1; k < 16; ++k) v = fmin(v, part[k][threadIdx.x]);
        if (j < m) atomicMin(min_q + b * m + j, bits(v));
      }
    }
    // row minima: reduce over the 16 threads of the half-warp that share ty, then one atomic per row
#pragma unroll
    for (int r = 0; r < RR; ++r) {
      double v = rmin[r];
      for (int o = 8; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
      const int i = rt * TR + ty + 16 * r;
      if (tx == 0 && i < n) atomicMin(min_p + b * n + i, bits(v));
    }
  }
}

// Thresholds by value: t[0 .. n) sorted ascending, finite, >= 0 (checked on the host).
struct Thresholds {
  double t[MAX_THR];
  int n;
};

// The bin of e among the sorted thresholds: the first j with e < t[j] (strict) or e <= t[j]; n when there is none
// (e past the last threshold, or NaN).  Counts of the thresholds are then prefix sums of the bins.
template <bool STRICT>
__device__ __forceinline__ int threshold_bin(double e, const Thresholds& th) {
  int lo = 0, hi = th.n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const bool in = STRICT ? (e < th.t[mid]) : (e <= th.t[mid]);
    if (in) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

template <typename T>
__device__ bool sample_finite(const T* a, long long n_val) {
  bool ok = true;
  for (long long i = threadIdx.x; i < n_val; i += NT) ok = ok && isfinite((double)a[i]);
  return ok;
}

// One CTA per sample: distances d = sqrt(min squared distance) (NaN throughout for a sample holding a non-finite
// coordinate), counts[b, dir, j] = #(d < t_j) per direction (dir 0: points of P, 1: points of Q), frac = counts / n,
// fscore[b, j] = ((2 a) b) / (a + b), 0 when a + b = 0, NaN (with frac) for a non-finite sample.
// dist_p / dist_q may alias min_p / min_q (each thread reads its bits before writing its double).
template <typename T>
__global__ void __launch_bounds__(NT) k_nearest_finish(const T* __restrict__ P, const T* __restrict__ Q, int batch,
                                                       int n, int m, const unsigned long long* min_p,
                                                       const unsigned long long* min_q, Thresholds th,
                                                       double* dist_p, double* dist_q, long long* __restrict__ counts,
                                                       double* __restrict__ frac, double* __restrict__ fscore) {
  __shared__ int hist[2][MAX_F_THR + 1];
  for (int b = blockIdx.x; b < batch; b += gridDim.x) {
    for (int k = threadIdx.x; k < 2 * (MAX_F_THR + 1); k += NT) (&hist[0][0])[k] = 0;
    const bool finite = __syncthreads_and(sample_finite(P + (long long)b * n * 3, 3LL * n) &&
                                          sample_finite(Q + (long long)b * m * 3, 3LL * m));
    for (int dir = 0; dir < 2; ++dir) {
      const int cnt = dir ? m : n;
      const unsigned long long* mn = (dir ? min_q : min_p) + (long long)b * cnt;
      double* out = dir ? dist_q : dist_p;
      for (int i = threadIdx.x; i < cnt; i += NT) {
        const double d = finite ? __dsqrt_rn(__longlong_as_double((long long)mn[i])) : nan("");
        if (out) out[(long long)b * cnt + i] = d;
        const int bin = threshold_bin<true>(d, th);
        if (bin < th.n) atomicAdd(&hist[dir][bin], 1);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      long long c[2] = {0, 0};
      for (int j = 0; j < th.n; ++j) {
        c[0] += hist[0][j];
        c[1] += hist[1][j];
        const double a = (double)c[0] / (double)n, bb = (double)c[1] / (double)m;
        const long long o = (long long)b * th.n + j;
        if (counts) {
          counts[((long long)b * 2 + 0) * th.n + j] = c[0];
          counts[((long long)b * 2 + 1) * th.n + j] = c[1];
        }
        if (frac) {
          frac[((long long)b * 2 + 0) * th.n + j] = finite ? a : nan("");
          frac[((long long)b * 2 + 1) * th.n + j] = finite ? bb : nan("");
        }
        if (fscore) fscore[o] = !finite ? nan("") : (a + bb > 0.0 ? ((2.0 * a) * bb) / (a + bb) : 0.0);
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- align_w_scale
// One CTA per sample, gt G and prediction Q [n, 3]:
//   t1 = mean(G), A = G - t1;  t2 = mean(Q), P = Q - t2;  s1 = |A|_F + 1e-8, s2 = |P|_F + 1e-8
//   U W V^T = svd(A^T P / (s1 s2));  R = U V^T, s = sum(W)  (scipy's orthogonal_procrustes(A / s1, P / s2); no
//   reflection correction: det R = -1 is kept)
//   aligned = ((P / s2) R^T) s s1 + t1;  err = |aligned - G|
// With u3 = u1 x u2 (right-handed), the SVD's third pair is (sign(w3u3) u3, |w3u3|).  A sample with a non-finite
// coordinate gets NaN in every output.
constexpr int AT = 256;
constexpr int AW = AT / 32;

template <typename TO>
__global__ void __launch_bounds__(AT) k_align_w_scale(const float* __restrict__ G, const float* __restrict__ Q,
                                                      int batch, int n, TO* __restrict__ aligned,
                                                      double* __restrict__ err) {
  __shared__ double red[11][AW];
  __shared__ double T[13];  // {s s1 / s2 * R row-major (9), t1 (3), finite}
  for (int b = blockIdx.x; b < batch; b += gridDim.x) {
    const float* g = G + (long long)b * n * 3;
    const float* q = Q + (long long)b * n * 3;
    double mu[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += AT)
      for (int c = 0; c < 3; ++c) {
        mu[c] += (double)g[3 * i + c];
        mu[3 + c] += (double)q[3 * i + c];
      }
    block_sum<6>(mu, red);
    for (int c = 0; c < 6; ++c) mu[c] /= n;
    double h[11] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // A^T P (9), |A|^2, |P|^2
    for (int i = threadIdx.x; i < n; i += AT) {
      double da[3], dp[3];
      for (int c = 0; c < 3; ++c) {
        da[c] = (double)g[3 * i + c] - mu[c];
        dp[c] = (double)q[3 * i + c] - mu[3 + c];
      }
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) h[3 * r + c] += da[r] * dp[c];
      h[9] += dot3(da, da);
      h[10] += dot3(dp, dp);
    }
    block_sum<11>(h, red);
    if (threadIdx.x == 0) {
      bool finite = true;
      for (int k = 0; k < 11; ++k) finite = finite && isfinite(h[k]);
      for (int k = 0; k < 6; ++k) finite = finite && isfinite(mu[k]);
      if (finite) {
        const double s1 = sqrt(h[9]) + 1e-8, s2 = sqrt(h[10]) + 1e-8;
        double M[9];
        for (int k = 0; k < 9; ++k) M[k] = h[k] / s1 / s2;
        Svd3 sd;
        svd3_jacobi(M, sd);
        const double sg = sd.w3u3 < 0.0 ? -1.0 : 1.0;
        const double s = (sd.s1 + sd.s2) + fabs(sd.w3u3);
        const double f = s * s1 / s2;
        for (int i = 0; i < 3; ++i)
          for (int k = 0; k < 3; ++k)
            T[3 * i + k] = f * (sd.u[0][i] * sd.v[0][k] + sd.u[1][i] * sd.v[1][k] + sg * sd.u[2][i] * sd.v[2][k]);
      }
      for (int c = 0; c < 3; ++c) T[9 + c] = mu[c];
      T[12] = finite ? 1.0 : 0.0;
    }
    __syncthreads();
    const bool finite = T[12] != 0.0;
    for (int i = threadIdx.x; i < n; i += AT) {
      double p[3];
      for (int c = 0; c < 3; ++c) p[c] = (double)q[3 * i + c] - mu[3 + c];
      double d2 = 0.0;
      for (int r = 0; r < 3; ++r) {
        const double y = finite ? dot3(T + 3 * r, p) + T[9 + r] : nan("");
        if (aligned) aligned[(3LL * b * n) + 3 * i + r] = (TO)y;
        const double d = y - (double)g[3 * i + r];
        d2 += d * d;
      }
      if (err) err[(long long)b * n + i] = sqrt(d2);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- PCK
// hist[j] += #{e : the first threshold with e <= t_j is j}; the count of e <= t_j is hist[0] + ... + hist[j].
// e comes from err [n_val] when given, else e = |P_i - G_i| (fp64, numpy's order) for n_val points, optionally
// stored to err_out.  Per-CTA shared histogram, then one 64-bit atomic per non-empty bin.
constexpr int PT = 256;

__global__ void __launch_bounds__(PT) k_pck_hist(const double* __restrict__ err, const float* __restrict__ P,
                                                 const float* __restrict__ G, long long n_val, Thresholds th,
                                                 double* __restrict__ err_out,
                                                 unsigned long long* __restrict__ hist) {
  __shared__ int h[MAX_THR];
  for (int k = threadIdx.x; k < MAX_THR; k += PT) h[k] = 0;
  __syncthreads();
  for (long long i = (long long)blockIdx.x * PT + threadIdx.x; i < n_val; i += (long long)gridDim.x * PT) {
    double e;
    if (err) {
      e = err[i];
    } else {
      e = __dsqrt_rn(sq_dist(P[3 * i], P[3 * i + 1], P[3 * i + 2], G[3 * i], G[3 * i + 1], G[3 * i + 2]));
      if (err_out) err_out[i] = e;
    }
    const int bin = threshold_bin<false>(e, th);
    if (bin < th.n) atomicAdd(&h[bin], 1);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < th.n; k += PT)
    if (h[k]) atomicAdd(hist + k, (unsigned long long)h[k]);
}

// ---------------------------------------------------------------- host helpers
// Host thresholds: 1 .. max_n values, finite, >= 0, non-decreasing.
int load_thresholds(const char* where, const double* t, int n, int max_n, Thresholds* th) {
  if (!t || n <= 0 || n > max_n) {
    set_error(std::string(where) + ": need 1 .. " + std::to_string(max_n) + " thresholds; got " + std::to_string(n));
    return P2M_ERR_INVALID;
  }
  for (int j = 0; j < n; ++j) {
    if (!std::isfinite(t[j]) || t[j] < 0.0 || (j > 0 && t[j] < t[j - 1])) {
      set_error(std::string(where) + ": thresholds must be finite, >= 0 and sorted ascending (threshold " +
                std::to_string(j) + " = " + std::to_string(t[j]) + ")");
      return P2M_ERR_INVALID;
    }
    th->t[j] = t[j];
  }
  for (int j = n; j < MAX_THR; ++j) th->t[j] = 0.0;
  th->n = n;
  return P2M_OK;
}

template <typename T>
int nearest_launch(const T* P, const T* Q, int batch, int n, int m, const Thresholds& th, unsigned long long* min_p,
                   unsigned long long* min_q, double* dist_p, double* dist_q, long long* counts, double* frac,
                   double* fscore, int dev, cudaStream_t s) {
  k_fill_inf<<<grid_for((long long)batch * (n + m), NT, MAX_GRID), NT, 0, s>>>(min_p, (long long)batch * n, min_q,
                                                                               (long long)batch * m);
  P2M_LAUNCH_OK();
  // Split a sample's column tiles over CTAs until the grid holds about four CTAs per SM (B = 1 at SMPL size still
  // fills the GPU); the minima do not depend on the split.
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int row_tiles = (n + TR - 1) / TR, col_tiles = (m + TC - 1) / TC;
  const long long base = (long long)batch * row_tiles;
  int splits = (int)std::min<long long>(col_tiles, std::max<long long>(1, (4LL * sms + base - 1) / base));
  const int tps = (col_tiles + splits - 1) / splits;
  splits = (col_tiles + tps - 1) / tps;
  k_nearest_sweep<T><<<grid_for(base * splits, 1, 1LL << 30), NT, 0, s>>>(P, Q, batch, n, m, row_tiles, splits, tps,
                                                                          min_p, min_q);
  P2M_LAUNCH_OK();
  k_nearest_finish<T><<<grid_for(batch, 1, MAX_GRID), NT, 0, s>>>(P, Q, batch, n, m, min_p, min_q, th, dist_p, dist_q,
                                                                  counts, frac, fscore);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // namespace
}  // namespace p2m

using namespace p2m;

extern "C" {

int p2m_nearest_distances(int dtype, const void* P, const void* Q, int batch, int n, int m, const double* thresholds,
                          int n_thr, double* dist_p, double* dist_q, int64_t* counts, double* frac, double* fscore,
                          p2m_stream_t stream) {
  if ((dtype != P2M_DTYPE_F32 && dtype != P2M_DTYPE_F64) || !P || !Q || batch <= 0 || batch > MAX_BATCH || n <= 0 ||
      n > MAX_POINTS || m <= 0 || m > MAX_POINTS || !(dist_p || dist_q || counts || frac || fscore)) {
    set_error("nearest_distances: bad argument (dtype code, null point array, batch outside [1, 2^24], n or m outside "
              "[1, 2^20], or no output)");
    return P2M_ERR_INVALID;
  }
  if (n_thr < 0 || n_thr > MAX_F_THR || (n_thr == 0) != (thresholds == nullptr) ||
      (n_thr == 0 && (counts || frac || fscore))) {
    set_error("nearest_distances: counts, frac and fscore need 1 .. 16 thresholds");
    return P2M_ERR_INVALID;
  }
  Thresholds th{};
  if (n_thr > 0) P2M_TRY(load_thresholds("nearest_distances", thresholds, n_thr, MAX_F_THR, &th));
  int dev;
  P2M_TRY(arrays_device("nearest_distances", {P, Q, dist_p, dist_q, counts, frac, fscore}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // the distance outputs double as the minima's bit store; a missing one gets stream-ordered scratch
  StreamBuffer<unsigned long long> sp(s), sq(s);
  unsigned long long* min_p = reinterpret_cast<unsigned long long*>(dist_p);
  unsigned long long* min_q = reinterpret_cast<unsigned long long*>(dist_q);
  if (!min_p) {
    P2M_TRY(sp.alloc((size_t)batch * n));
    min_p = sp.ptr;
  }
  if (!min_q) {
    P2M_TRY(sq.alloc((size_t)batch * m));
    min_q = sq.ptr;
  }
  long long* cnt = reinterpret_cast<long long*>(counts);
  if (dtype == P2M_DTYPE_F32)
    return nearest_launch<float>(static_cast<const float*>(P), static_cast<const float*>(Q), batch, n, m, th, min_p,
                                 min_q, dist_p, dist_q, cnt, frac, fscore, dev, s);
  return nearest_launch<double>(static_cast<const double*>(P), static_cast<const double*>(Q), batch, n, m, th, min_p,
                                min_q, dist_p, dist_q, cnt, frac, fscore, dev, s);
}

int p2m_align_w_scale(const float* gt, const float* pred, int batch, int n_point, int aligned_dtype, void* aligned,
                      double* err, p2m_stream_t stream) {
  if (!gt || !pred || batch <= 0 || batch > MAX_BATCH || n_point <= 0 || n_point > MAX_PCK_POINTS ||
      !(aligned || err) || (aligned && aligned_dtype != P2M_DTYPE_F32 && aligned_dtype != P2M_DTYPE_F64)) {
    set_error("align_w_scale: bad argument (null point array, batch or n_point outside [1, 2^24], no output, or bad "
              "aligned dtype)");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("align_w_scale", {gt, pred, aligned, err}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const unsigned grid = grid_for(batch, 1, 4096);
  if (aligned && aligned_dtype == P2M_DTYPE_F64)
    k_align_w_scale<double><<<grid, AT, 0, s>>>(gt, pred, batch, n_point, static_cast<double*>(aligned), err);
  else
    k_align_w_scale<float><<<grid, AT, 0, s>>>(gt, pred, batch, n_point, static_cast<float*>(aligned), err);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_pck_accumulate(const double* err, const float* pred, const float* gt, int64_t n_val, const double* thresholds,
                       int n_thr, double* err_out, int64_t* hist, p2m_stream_t stream) {
  if (n_val <= 0 || n_val > (int64_t)MAX_BATCH * MAX_PCK_POINTS / 64 || !hist || (err == nullptr) == (pred == nullptr) ||
      (pred == nullptr) != (gt == nullptr) || (err && err_out)) {
    set_error("pck_accumulate: give either err or both point arrays (err_out only with points), a histogram, and "
              "1 <= n_val <= 2^42");
    return P2M_ERR_INVALID;
  }
  Thresholds th{};
  P2M_TRY(load_thresholds("pck_accumulate", thresholds, n_thr, MAX_THR, &th));
  int dev;
  P2M_TRY(arrays_device("pck_accumulate", {err, pred, gt, err_out, hist}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  k_pck_hist<<<grid_for(n_val, PT, 1024), PT, 0, s>>>(err, pred, gt, n_val, th, err_out,
                                                      reinterpret_cast<unsigned long long*>(hist));
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
