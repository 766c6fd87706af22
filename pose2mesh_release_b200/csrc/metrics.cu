// Row f5 of SURVEY.md §8: the evaluation metrics of the reference's test loop on the GPU.
//  * similarity Procrustes  coord_utils.rigid_transform_3D / rigid_align   (lib/coord_utils.py:127-149), batched
//  * root-aligned point errors  compute_joint_err / compute_both_err  (data/Human36M/dataset.py:454-477,
//    data/PW3D/dataset.py:263-286, data/SURREAL/dataset.py:205-226) and the per-sample errors of the datasets'
//    evaluate methods
// One CTA per sample (grid-stride over samples); every reduction runs in a fixed order without atomics, so a sample's
// result is independent of its batch position, of the batch size and of the run.
#include <cuda_runtime.h>

#include <cmath>
#include <string>

#include "p2m_internal.h"
#include "procrustes3.cuh"

namespace p2m {
namespace {

constexpr int MT = 256;          // threads per CTA
constexpr int NW = MT / 32;      // warps per CTA
constexpr int MAX_GRID = 4096;   // CTAs of the grid-stride loop over samples
constexpr int MAX_BATCH = 1 << 24;
constexpr int MAX_POINTS = 1 << 24;

// rigid_transform_3D (coord_utils.py:127-143) from the centred statistics of one sample, fp64, one thread.
//   h[3 r + c] = sum_i (A_i - muA)_r (B_i - muB)_c / n,  varP = sum_axes var(A) (population, as np.var)
// SVD H = U diag(s) Vh by one-sided Jacobi on the columns of H (W = H V converges to U diag(s)), singular values
// sorted descending.  U is completed to a right-handed orthonormal basis u3 = u1 x u2, which makes the third singular
// value signed (s3 = <w3, u3>); then  R = V diag(1, 1, det V) U^T  and  s3 *= det V  are exactly the reference's
// R = Vh^T U^T with its `det R < 0` correction (negate s[-1] and Vh[2]), whichever sign LAPACK gave u3.
// out = {c, R row-major, t}; a sample with varP = 0 (all points of A equal, or n = 1) or non-finite statistics gets
// NaN throughout (the reference's 1/varP * sum(s) is 1/0 * 0 there).
__device__ void procrustes_3x3(const double* h, double varP, const double* mu_a, const double* mu_b, double* out) {
  bool finite = isfinite(varP);
  for (int k = 0; k < 9; ++k) finite = finite && isfinite(h[k]);
  for (int k = 0; k < 3; ++k) finite = finite && isfinite(mu_a[k]) && isfinite(mu_b[k]);
  if (!finite || !(varP > 0.0)) {
    for (int k = 0; k < 13; ++k) out[k] = nan("");
    return;
  }
  Svd3 sd;
  svd3_jacobi(h, sd);
  const double(&u)[3][3] = sd.u;
  const double(&v)[3][3] = sd.v;
  const double s1 = sd.s1, s2 = sd.s2;
  const double det_v = v[0][0] * (v[1][1] * v[2][2] - v[1][2] * v[2][1]) -
                       v[1][0] * (v[0][1] * v[2][2] - v[0][2] * v[2][1]) +
                       v[2][0] * (v[0][1] * v[1][2] - v[0][2] * v[1][1]);
  const double dv = det_v < 0.0 ? -1.0 : 1.0;
  const double s3 = sd.w3u3 * dv;
  const double c = (1.0 / varP) * ((s1 + s2) + s3);
  double R[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) R[i][j] = v[0][i] * u[0][j] + v[1][i] * u[1][j] + dv * v[2][i] * u[2][j];
  out[0] = c;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) out[1 + 3 * i + j] = R[i][j];
    out[10 + i] = -(((c * R[i][0]) * mu_a[0] + (c * R[i][1]) * mu_a[1]) + (c * R[i][2]) * mu_a[2]) + mu_b[i];
  }
}

// Batched rigid_align on A[b, idx], B[b, idx] (idx = subset[0..k) or 0..k-1): pass 1 the centroids, pass 2 the centred
// cross-covariance and varP, one thread the SVD and transform, pass 3 the aligned points c R a + t and their distances
// to B.  sums[b] = sum of the sample's distances.
__global__ void __launch_bounds__(MT) k_rigid_align(const float* __restrict__ A, const float* __restrict__ B, int batch,
                                                    int n_point, const int* __restrict__ subset, int k,
                                                    double* __restrict__ transform, float* __restrict__ aligned,
                                                    float* __restrict__ err, double* __restrict__ sums) {
  __shared__ double red[10][NW];
  __shared__ double T[13];
  for (int b = blockIdx.x; b < batch; b += gridDim.x) {
    const float* a = A + (long long)b * n_point * 3;
    const float* g = B + (long long)b * n_point * 3;
    double m[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < k; i += MT) {
      const long long p = subset ? subset[i] : i;
      for (int c = 0; c < 3; ++c) {
        m[c] += (double)a[3 * p + c];
        m[3 + c] += (double)g[3 * p + c];
      }
    }
    block_sum<6>(m, red);
    for (int c = 0; c < 6; ++c) m[c] /= k;
    double h[10] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < k; i += MT) {
      const long long p = subset ? subset[i] : i;
      double da[3], db[3];
      for (int c = 0; c < 3; ++c) {
        da[c] = (double)a[3 * p + c] - m[c];
        db[c] = (double)g[3 * p + c] - m[3 + c];
      }
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) h[3 * r + c] += da[r] * db[c];
      h[9] += dot3(da, da);
    }
    block_sum<10>(h, red);
    if (threadIdx.x == 0) {
      for (int q = 0; q < 10; ++q) h[q] /= k;
      procrustes_3x3(h, h[9], m, m + 3, T);
      if (transform)
        for (int q = 0; q < 13; ++q) transform[(long long)b * 13 + q] = T[q];
    }
    __syncthreads();
    if (aligned || err || sums) {
      double cR[9], t[3];
      for (int q = 0; q < 9; ++q) cR[q] = T[0] * T[1 + q];
      for (int q = 0; q < 3; ++q) t[q] = T[10 + q];
      double es[1] = {0.0};
      for (int i = threadIdx.x; i < k; i += MT) {
        const long long p = subset ? subset[i] : i;
        const double x[3] = {(double)a[3 * p], (double)a[3 * p + 1], (double)a[3 * p + 2]};
        double d2 = 0.0;
        for (int r = 0; r < 3; ++r) {
          const double y = dot3(cR + 3 * r, x) + t[r];
          if (aligned) aligned[((long long)b * k + i) * 3 + r] = (float)y;
          const double d = y - (double)g[3 * p + r];
          d2 += d * d;
        }
        const double e = sqrt(d2);
        if (err) err[(long long)b * k + i] = (float)e;
        es[0] += e;
      }
      block_sum<1>(es, red);
      if (sums && threadIdx.x == 0) sums[b] = es[0];
    }
  }
}

// err[b, i] = |(P[b, idx] - pr[b]) - (G[b, idx] - gr[b])| (roots optional).  FP64 = false: float32 in numpy's order
// (roots subtracted first, (d0^2 + d1^2) + d2^2, sqrt), each step rounded to nearest with no contraction, i.e. the
// bits the reference's float32 numpy gives; FP64 = true: the same in fp64, rounded once on store.
// sums[b] = the fp64 sum of the sample's errors.
template <bool FP64>
__global__ void __launch_bounds__(MT) k_point_errors(const float* __restrict__ P, const float* __restrict__ G,
                                                     const float* __restrict__ pr, const float* __restrict__ gr,
                                                     int batch, int n_point, const int* __restrict__ subset, int k,
                                                     float* __restrict__ err, double* __restrict__ sums) {
  __shared__ double red[1][NW];
  for (int b = blockIdx.x; b < batch; b += gridDim.x) {
    const float* p0 = P + (long long)b * n_point * 3;
    const float* g0 = G + (long long)b * n_point * 3;
    double es[1] = {0.0};
    for (int i = threadIdx.x; i < k; i += MT) {
      const long long p = subset ? subset[i] : i;
      double e;
      if (FP64) {
        double d2 = 0.0;
        for (int c = 0; c < 3; ++c) {
          double x = p0[3 * p + c], y = g0[3 * p + c];
          if (pr) {
            x -= (double)pr[3 * b + c];
            y -= (double)gr[3 * b + c];
          }
          d2 += (x - y) * (x - y);
        }
        e = sqrt(d2);
      } else {
        float d[3];
        for (int c = 0; c < 3; ++c) {
          float x = p0[3 * p + c], y = g0[3 * p + c];
          if (pr) {
            x = __fsub_rn(x, pr[3 * b + c]);
            y = __fsub_rn(y, gr[3 * b + c]);
          }
          d[c] = __fsub_rn(x, y);
        }
        const float s = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]));
        e = (double)__fsqrt_rn(s);
      }
      if (err) err[(long long)b * k + i] = (float)e;
      es[0] += e;
    }
    block_sum<1>(es, red);
    if (sums && threadIdx.x == 0) sums[b] = es[0];
  }
}

// sums[batch] = sum of sums[0 .. batch) in a fixed order (one CTA)
__global__ void __launch_bounds__(MT) k_batch_total(double* __restrict__ sums, int batch) {
  __shared__ double red[1][NW];
  double s[1] = {0.0};
  for (int b = threadIdx.x; b < batch; b += MT) s[0] += sums[b];
  block_sum<1>(s, red);
  if (threadIdx.x == 0) sums[batch] = s[0];
}

// Shared argument checks; the subset indices come from the caller and are checked here, on the host.
int check_args(const char* where, const float* a, const float* b, int batch, int n_point, const int32_t* subset,
               int n_subset, bool any_output) {
  if (!a || !b || batch <= 0 || batch > MAX_BATCH || n_point <= 0 || n_point > MAX_POINTS || n_subset < 0 ||
      (n_subset > 0) != (subset != nullptr) || !any_output) {
    set_error(std::string(where) + ": bad argument (null input, no output, batch or n_point out of [1, 2^24], or "
                                   "subset / n_subset inconsistent)");
    return P2M_ERR_INVALID;
  }
  for (int i = 0; i < n_subset; ++i)
    if (subset[i] < 0 || subset[i] >= n_point) {
      set_error(std::string(where) + ": subset[" + std::to_string(i) + "] = " + std::to_string(subset[i]) +
                " is outside [0, " + std::to_string(n_point) + ")");
      return P2M_ERR_INVALID;
    }
  return P2M_OK;
}

}  // namespace
}  // namespace p2m

using namespace p2m;

extern "C" {

int p2m_rigid_align(const float* A, const float* B, int batch, int n_point, const int32_t* subset, int n_subset,
                    double* transform, float* aligned, float* err, double* sums, p2m_stream_t stream) {
  P2M_TRY(check_args("rigid_align", A, B, batch, n_point, subset, n_subset, transform || aligned || err || sums));
  int dev;
  P2M_TRY(arrays_device("rigid_align", {A, B, transform, aligned, err, sums}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamBuffer<int> sub(s);
  P2M_TRY(sub.alloc(n_subset, subset));
  const int k = n_subset > 0 ? n_subset : n_point;
  k_rigid_align<<<grid_for(batch, 1, MAX_GRID), MT, 0, s>>>(A, B, batch, n_point, sub.ptr, k, transform, aligned, err,
                                                            sums);
  P2M_LAUNCH_OK();
  if (sums) {
    k_batch_total<<<1, MT, 0, s>>>(sums, batch);
    P2M_LAUNCH_OK();
  }
  return P2M_OK;
}

int p2m_point_errors(const float* pred, const float* gt, const float* pred_root, const float* gt_root, int batch,
                     int n_point, const int32_t* subset, int n_subset, int fp64, float* err, double* sums,
                     p2m_stream_t stream) {
  P2M_TRY(check_args("point_errors", pred, gt, batch, n_point, subset, n_subset, err || sums));
  if ((pred_root == nullptr) != (gt_root == nullptr)) {
    set_error("point_errors: give both root arrays or neither");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("point_errors", {pred, gt, pred_root, gt_root, err, sums}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamBuffer<int> sub(s);
  P2M_TRY(sub.alloc(n_subset, subset));
  const int k = n_subset > 0 ? n_subset : n_point;
  const unsigned grid = grid_for(batch, 1, MAX_GRID);
  if (fp64)
    k_point_errors<true><<<grid, MT, 0, s>>>(pred, gt, pred_root, gt_root, batch, n_point, sub.ptr, k, err, sums);
  else
    k_point_errors<false><<<grid, MT, 0, s>>>(pred, gt, pred_root, gt_root, batch, n_point, sub.ptr, k, err, sums);
  P2M_LAUNCH_OK();
  if (sums) {
    k_batch_total<<<1, MT, 0, s>>>(sums, batch);
    P2M_LAUNCH_OK();
  }
  return P2M_OK;
}

}  // extern "C"
