// Device pieces shared by the Procrustes kernels (csrc/metrics.cu: Pose2Mesh's rigid_align; csrc/fscore.cu: the
// FreiHAND script's align_w_scale): the fixed-order fp64 CTA reduction and the 3x3 SVD by one-sided Jacobi.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

namespace p2m {

// v[k] <- the CTA-wide sum of v[k], the same bits in every thread: xor-shuffle tree inside each warp, then the warp
// partials in warp order (NW warps per CTA).  Ends with a barrier, so `red` can be reused by the next call.
template <int N, int NW>
__device__ __forceinline__ void block_sum(double (&v)[N], double (*red)[NW]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double a = v[k];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) red[k][warp] = a;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < N; ++k) {
    double a = 0.0;
    for (int w = 0; w < NW; ++w) a += red[k][w];
    v[k] = a;
  }
  __syncthreads();
}

__device__ __forceinline__ double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// SVD of a finite 3x3 matrix h (row-major) = sum_j s_j u_j v_j^T by one-sided Jacobi on the columns of h
// (W = h V converges to U diag(s)), singular values sorted descending.  u[j] / v[j] are the j-th left / right singular
// vectors; u[2] = u[0] x u[1] completes a right-handed basis, so the third singular value comes out signed:
// w3u3 = <w_3, u_3> = +-s_3.  A zero or rank-1 h gets some orthonormal completion of u.
struct Svd3 {
  double u[3][3], v[3][3];
  double s1, s2, w3u3;
};

__device__ __forceinline__ void svd3_jacobi(const double* h, Svd3& out) {
  double W[3][3], V[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      W[r][c] = h[3 * r + c];
      V[r][c] = (r == c) ? 1.0 : 0.0;
    }
  const int P[3] = {0, 0, 1}, Q[3] = {1, 2, 2};
  for (int sweep = 0; sweep < 40; ++sweep) {
    bool rotated = false;
    for (int pq = 0; pq < 3; ++pq) {
      const int p = P[pq], q = Q[pq];
      double alpha = 0.0, beta = 0.0, gamma = 0.0;
      for (int r = 0; r < 3; ++r) {
        alpha += W[r][p] * W[r][p];
        beta += W[r][q] * W[r][q];
        gamma += W[r][p] * W[r][q];
      }
      if (!(fabs(gamma) > 1e-15 * sqrt(alpha * beta))) continue;
      const double zeta = (beta - alpha) / (2.0 * gamma);
      const double t = copysign(1.0, zeta) / (fabs(zeta) + hypot(1.0, zeta));
      const double cs = 1.0 / sqrt(1.0 + t * t), sn = cs * t;
      for (int r = 0; r < 3; ++r) {
        const double wp = W[r][p], wq = W[r][q];
        W[r][p] = cs * wp - sn * wq;
        W[r][q] = sn * wp + cs * wq;
        const double vp = V[r][p], vq = V[r][q];
        V[r][p] = cs * vp - sn * vq;
        V[r][q] = sn * vp + cs * vq;
      }
      rotated = true;
    }
    if (!rotated) break;
  }
  double sv[3];
  int ord[3] = {0, 1, 2};
  for (int j = 0; j < 3; ++j) sv[j] = sqrt(W[0][j] * W[0][j] + W[1][j] * W[1][j] + W[2][j] * W[2][j]);
  for (int i = 0; i < 2; ++i)  // stable sort, descending
    for (int j = 0; j < 2 - i; ++j)
      if (sv[ord[j]] < sv[ord[j + 1]]) {
        const int x = ord[j];
        ord[j] = ord[j + 1];
        ord[j + 1] = x;
      }
  double w[3][3];  // w[j] / out.v[j]: column j of the sorted W / V
  for (int j = 0; j < 3; ++j)
    for (int r = 0; r < 3; ++r) {
      w[j][r] = W[r][ord[j]];
      out.v[j][r] = V[r][ord[j]];
    }
  const double s1 = sv[ord[0]], s2 = sv[ord[1]];
  double (&u)[3][3] = out.u;
  if (s1 > 0.0) {
    for (int r = 0; r < 3; ++r) u[0][r] = w[0][r] / s1;
  } else {  // h = 0: any basis
    u[0][0] = 1.0, u[0][1] = 0.0, u[0][2] = 0.0;
  }
  // u2: w2 orthogonalised against u1; when w2 vanishes (rank-1 h) any unit vector orthogonal to u1
  {
    double x[3];
    const double d = dot3(w[1], u[0]);
    for (int r = 0; r < 3; ++r) x[r] = w[1][r] - d * u[0][r];
    double nx = sqrt(dot3(x, x));
    if (!(nx > 1e-12 * s1)) {
      int a = 0;  // the axis least aligned with u1
      for (int r = 1; r < 3; ++r)
        if (fabs(u[0][r]) < fabs(u[0][a])) a = r;
      const double e = u[0][a];
      for (int r = 0; r < 3; ++r) x[r] = ((r == a) ? 1.0 : 0.0) - e * u[0][r];
      nx = sqrt(dot3(x, x));
    }
    for (int r = 0; r < 3; ++r) u[1][r] = x[r] / nx;
  }
  u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
  u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
  u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  out.s1 = s1;
  out.s2 = s2;
  out.w3u3 = dot3(w[2], u[2]);
}

}  // namespace p2m
