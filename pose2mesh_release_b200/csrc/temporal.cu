// Row f8 of SURVEY.md §8: the temporal metrics of the 3DPW video block on the GPU, for ragged batches of sequences
// concatenated along frames (offsets[n_seq + 1] in frames):
//  * smooth_utils.smooth_pose / OneEuroFilter  (lib/smooth_utils.py:5-72): k_one_euro, one thread per
//    (sequence, channel) running the filter over the frames in order;
//  * coord_utils.compute_error_accel  (lib/coord_utils.py:194-222): k_accel_error, one warp per window (sequence, i);
//  * the per-video np.mean of those values: k_segment_mean, one CTA per sequence, fp64.
// Float32 and float64.  Every arithmetic step of the first two uses a round-to-nearest intrinsic (no FMA contraction)
// in numpy's dtype and operation order, so their outputs are the reference's bits; oracle/temporal_oracle.py restates
// them operation by operation.  No atomics: a sequence's results do not depend on its batch position.
#include <cuda_runtime.h>

#include <cmath>
#include <string>
#include <vector>

#include "p2m_internal.h"

namespace p2m {
namespace {

constexpr int EULER_THREADS = 128;
constexpr int PREFETCH = 4;        // frames loaded ahead of the recurrence (independent of it)
constexpr int ACCEL_WARPS = 8;     // windows per CTA
constexpr int MEAN_THREADS = 256;
constexpr int MEAN_WARPS = MEAN_THREADS / 32;
constexpr int MAX_GRID = 1 << 16;  // CTAs of the grid-stride loops
constexpr int MAX_JOINTS = 32;

__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float sqr_root(float a) { return __fsqrt_rn(a); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dvd(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double sqr_root(double a) { return __dsqrt_rn(a); }

// The filter's constants, rounded to T on the host as numpy rounds a Python float against a T array (NEP 50).
template <typename T>
struct EuroParams {
  T two_pi;          // 2 * math.pi
  T two_pi_dcutoff;  // 2 * math.pi * d_cutoff, multiplied in double first (smoothing_factor evaluates left to right)
  T min_cutoff, beta;
};

// smooth_pose on x[offsets[s] .. offsets[s + 1]) x n_ch, thread = (s, channel).  Per frame idx >= 1, in T:
//   t = T(idx), t_e = t - t_prev
//   a_d = r_d / (r_d + 1), r_d = T(2 pi d_cutoff) t_e;   dx = (x - x_prev) / t_e;   dx_hat = a_d dx + (1 - a_d) dx_prev
//   cutoff = T(min_cutoff) + T(beta) |dx_hat|;   r = (T(2 pi) cutoff) t_e;   a = r / (r + 1)
//   x_hat = a x + (1 - a) x_prev
// starting from x_prev = x[0], dx_prev = 0, t_prev = 0; frame 0 is copied.
template <typename T>
__global__ void __launch_bounds__(EULER_THREADS) k_one_euro(const T* __restrict__ x, T* __restrict__ y, long long n_ch,
                                                            const long long* __restrict__ offsets, int n_seq,
                                                            EuroParams<T> p) {
  const long long total = (long long)n_seq * n_ch;
  for (long long id = (long long)blockIdx.x * EULER_THREADS + threadIdx.x; id < total;
       id += (long long)gridDim.x * EULER_THREADS) {
    const int s = (int)(id / n_ch);
    const long long ch = id - (long long)s * n_ch;
    const long long f0 = offsets[s], n = offsets[s + 1] - f0;
    if (n <= 0) continue;
    const T* xs = x + f0 * n_ch + ch;
    T* ys = y + f0 * n_ch + ch;
    T x_prev = xs[0], dx_prev = T(0), t_prev = T(0);
    ys[0] = x_prev;
    T buf[PREFETCH];
#pragma unroll
    for (int k = 0; k < PREFETCH; ++k) buf[k] = (1 + k < n) ? xs[(1 + k) * n_ch] : T(0);
    for (long long f = 1; f < n; f += PREFETCH) {
#pragma unroll
      for (int k = 0; k < PREFETCH; ++k) {
        const long long idx = f + k;
        if (idx < n) {
          const T xv = buf[k];
          if (idx + PREFETCH < n) buf[k] = xs[(idx + PREFETCH) * n_ch];
          const T t = T(idx);
          const T te = sub(t, t_prev);
          const T r_d = mul(p.two_pi_dcutoff, te);
          const T a_d = dvd(r_d, add(r_d, T(1)));
          const T dx = dvd(sub(xv, x_prev), te);
          const T dx_hat = add(mul(a_d, dx), mul(sub(T(1), a_d), dx_prev));
          const T cutoff = add(p.min_cutoff, mul(p.beta, fabs(dx_hat)));
          const T r = mul(mul(p.two_pi, cutoff), te);
          const T a = dvd(r, add(r, T(1)));
          const T x_hat = add(mul(a, xv), mul(sub(T(1), a), x_prev));
          ys[idx * n_ch] = x_hat;
          x_prev = x_hat;
          dx_prev = dx_hat;
          t_prev = t;
        }
      }
    }
  }
}

// numpy's np.add.reduce of v[0 .. n) (n <= 32, the row of a C-contiguous array): the identity 0 plus the pairwise sum
// of all n values, which for n < 8 is sequential and otherwise runs eight accumulators over blocks of eight, adds
// them as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) and then the remaining n % 8 values in order.
template <typename T>
__device__ T numpy_row_sum(const T* v, int n) {
  T res;
  if (n < 8) {
    res = T(0);
    for (int i = 0; i < n; ++i) res = add(res, v[i]);
  } else {
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = v[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = add(r[j], v[i + j]);
    res = add(add(add(r[0], r[1]), add(r[2], r[3])), add(add(r[4], r[5]), add(r[6], r[7])));
    for (; i < n; ++i) res = add(res, v[i]);
  }
  return add(T(0), res);
}

// compute_error_accel on every window w = (s, i), i in [0, n_s - 2): lane = joint.
//   accel = (X[i] - 2 X[i+1]) + X[i+2] for gt and pred;  d = accel_pred - accel_gt;  e_j = sqrt((d0^2 + d1^2) + d2^2)
//   per_window[w] = np.mean(e, axis=1) in T;  valid[w] = vis[i] & vis[i+1] & vis[i+2] (1 without vis)
// offs = {frame offsets [n_seq + 1], window offsets [n_seq + 1]}.
template <typename T>
// (min 1 CTA per SM: without the hint ptxas holds the fp64 instantiation to 40 registers and spills 8 bytes)
__global__ void __launch_bounds__(ACCEL_WARPS * 32, 1) k_accel_error(const T* __restrict__ gt, const T* __restrict__ pred,
                                                                  int n_joint, const long long* __restrict__ offs,
                                                                  int n_seq, long long n_win,
                                                                  const unsigned char* __restrict__ vis,
                                                                  T* __restrict__ per_window,
                                                                  unsigned char* __restrict__ valid) {
  __shared__ T norms[ACCEL_WARPS][MAX_JOINTS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long* frame_off = offs;
  const long long* win_off = offs + n_seq + 1;
  for (long long w = (long long)blockIdx.x * ACCEL_WARPS + warp; w < n_win; w += (long long)gridDim.x * ACCEL_WARPS) {
    int lo = 0, hi = n_seq - 1;  // the sequence s with win_off[s] <= w < win_off[s + 1]
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (win_off[mid] <= w) lo = mid;
      else hi = mid - 1;
    }
    const long long f = frame_off[lo] + (w - win_off[lo]);  // global frame of window position i
    if (lane < n_joint) {
      const long long stride = (long long)n_joint * 3;
      const T* g = gt + f * stride + lane * 3;
      const T* q = pred + f * stride + lane * 3;
      T d[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const T ag = add(sub(g[c], mul(T(2), g[stride + c])), g[2 * stride + c]);
        const T ap = add(sub(q[c], mul(T(2), q[stride + c])), q[2 * stride + c]);
        d[c] = sub(ap, ag);
      }
      norms[warp][lane] = sqr_root(add(add(mul(d[0], d[0]), mul(d[1], d[1])), mul(d[2], d[2])));
    }
    __syncwarp();
    const T mean = dvd(numpy_row_sum(norms[warp], n_joint), T(n_joint));  // every lane: broadcast reads, no divergence
    if (lane == 0) {
      per_window[w] = mean;
      valid[w] = vis ? (unsigned char)(vis[f] && vis[f + 1] && vis[f + 2]) : (unsigned char)1;
    }
    __syncwarp();
  }
}

// out[s] = the fp64 mean of values[rows offsets[s] .. offsets[s + 1]) x width, rows with valid[row] == 0 skipped; NaN
// when no element remains.  Thread k sums the elements k, k + 256, ... of the segment's valid rows (in row order),
// then a fixed xor-shuffle tree and the warp partials in warp order: the same bits wherever the segment sits.
template <typename T>
__global__ void __launch_bounds__(MEAN_THREADS) k_segment_mean(const T* __restrict__ values, long long width,
                                                               const long long* __restrict__ offsets, int n_seg,
                                                               const unsigned char* __restrict__ valid,
                                                               double* __restrict__ out) {
  __shared__ double red[2][MEAN_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int s = blockIdx.x; s < n_seg; s += gridDim.x) {
    const long long r0 = offsets[s], n_el = (offsets[s + 1] - r0) * width;
    double sum = 0.0, cnt = 0.0;
    for (long long e = threadIdx.x; e < n_el; e += MEAN_THREADS) {
      const long long row = r0 + e / width;
      if (valid && !valid[row]) continue;
      sum += (double)values[r0 * width + e];
      cnt += 1.0;
    }
    for (int o = 16; o > 0; o >>= 1) {
      sum += __shfl_xor_sync(0xffffffffu, sum, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if (lane == 0) {
      red[0][warp] = sum;
      red[1][warp] = cnt;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double s_all = 0.0, c_all = 0.0;
      for (int k = 0; k < MEAN_WARPS; ++k) {
        s_all += red[0][k];
        c_all += red[1][k];
      }
      out[s] = c_all > 0.0 ? s_all / c_all : nan("");
    }
    __syncthreads();
  }
}

// Host offsets: offsets[0] == 0, non-decreasing, offsets[n_seq] == n_rows.
int check_offsets(const char* where, const int64_t* offsets, int n_seq, int64_t n_rows) {
  if (!offsets || n_seq <= 0 || n_rows <= 0) {
    set_error(std::string(where) + ": need offsets, n_seq > 0 and at least one frame");
    return P2M_ERR_INVALID;
  }
  if (offsets[0] != 0 || offsets[n_seq] != n_rows) {
    set_error(std::string(where) + ": offsets must run from 0 to the number of frames (" + std::to_string(n_rows) +
              "); got " + std::to_string(offsets[0]) + " .. " + std::to_string(offsets[n_seq]));
    return P2M_ERR_INVALID;
  }
  for (int s = 0; s < n_seq; ++s)
    if (offsets[s + 1] < offsets[s]) {
      set_error(std::string(where) + ": offsets decrease at sequence " + std::to_string(s));
      return P2M_ERR_INVALID;
    }
  return P2M_OK;
}

bool known_dtype(int dtype) { return dtype == P2M_DTYPE_F32 || dtype == P2M_DTYPE_F64; }

template <typename T>
EuroParams<T> euro_params(double min_cutoff, double beta, double d_cutoff) {
  const double two_pi = 2.0 * M_PI;  // == Python's 2 * math.pi
  return EuroParams<T>{(T)two_pi, (T)(two_pi * d_cutoff), (T)min_cutoff, (T)beta};
}

template <typename T>
int segment_mean_launch(const T* values, long long width, const long long* offsets, int n_seg,
                        const unsigned char* valid, double* out, cudaStream_t s) {
  k_segment_mean<T><<<grid_for(n_seg, 1, MAX_GRID), MEAN_THREADS, 0, s>>>(values, width, offsets, n_seg, valid, out);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // namespace
}  // namespace p2m

using namespace p2m;

extern "C" {

int p2m_one_euro_smooth(int dtype, const void* x, void* y, int64_t n_channel, const int64_t* offsets, int n_seq,
                        int64_t n_frames, double min_cutoff, double beta, double d_cutoff, p2m_stream_t stream) {
  if (!known_dtype(dtype) || !x || !y || n_channel <= 0) {
    set_error("one_euro_smooth: bad dtype code, null array or n_channel <= 0");
    return P2M_ERR_INVALID;
  }
  P2M_TRY(check_offsets("one_euro_smooth", offsets, n_seq, n_frames));
  int dev;
  P2M_TRY(arrays_device("one_euro_smooth", {x, y}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamBuffer<long long> off(s);
  P2M_TRY(off.alloc((size_t)n_seq + 1, offsets));
  const unsigned grid = grid_for((long long)n_seq * n_channel, EULER_THREADS, MAX_GRID);
  if (dtype == P2M_DTYPE_F32)
    k_one_euro<float><<<grid, EULER_THREADS, 0, s>>>(static_cast<const float*>(x), static_cast<float*>(y), n_channel,
                                                     off.ptr, n_seq, euro_params<float>(min_cutoff, beta, d_cutoff));
  else
    k_one_euro<double><<<grid, EULER_THREADS, 0, s>>>(static_cast<const double*>(x), static_cast<double*>(y),
                                                      n_channel, off.ptr, n_seq,
                                                      euro_params<double>(min_cutoff, beta, d_cutoff));
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_accel_error(int dtype, const void* gt, const void* pred, int n_joint, const int64_t* offsets, int n_seq,
                    int64_t n_frames, const uint8_t* vis, void* per_window, uint8_t* valid, double* seq_mean,
                    p2m_stream_t stream) {
  if (!known_dtype(dtype) || n_joint <= 0 || n_joint > MAX_JOINTS) {
    set_error("accel_error: bad dtype code or n_joint outside [1, 32]; got n_joint = " + std::to_string(n_joint));
    return P2M_ERR_INVALID;
  }
  P2M_TRY(check_offsets("accel_error", offsets, n_seq, n_frames));
  std::vector<int64_t> host((size_t)2 * (n_seq + 1));  // frame offsets, then window offsets
  host[n_seq + 1] = 0;
  for (int i = 0; i <= n_seq; ++i) host[i] = offsets[i];
  for (int i = 0; i < n_seq; ++i) {
    const int64_t n = offsets[i + 1] - offsets[i];
    host[n_seq + 2 + i] = host[n_seq + 1 + i] + (n > 2 ? n - 2 : 0);
  }
  const long long n_win = host[2 * n_seq + 1];
  if (!seq_mean || (n_win > 0 && (!gt || !pred || !per_window || !valid))) {
    set_error("accel_error: null data array");
    return P2M_ERR_INVALID;
  }
  int dev;
  if (n_win > 0) P2M_TRY(arrays_device("accel_error", {gt, pred, vis, per_window, valid, seq_mean}, &dev));
  else P2M_TRY(arrays_device("accel_error", {seq_mean}, &dev));  // no window: only seq_mean is written
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamBuffer<long long> off(s);
  P2M_TRY(off.alloc(host.size(), host.data()));
  const long long* win_off = off.ptr + n_seq + 1;
  const unsigned grid = grid_for(n_win, ACCEL_WARPS, MAX_GRID);
  if (dtype == P2M_DTYPE_F32) {
    if (n_win > 0) {
      k_accel_error<float><<<grid, ACCEL_WARPS * 32, 0, s>>>(
          static_cast<const float*>(gt), static_cast<const float*>(pred), n_joint, off.ptr, n_seq, n_win, vis,
          static_cast<float*>(per_window), valid);
      P2M_LAUNCH_OK();
    }
    P2M_TRY(segment_mean_launch<float>(static_cast<const float*>(per_window), 1, win_off, n_seq, valid, seq_mean, s));
  } else {
    if (n_win > 0) {
      k_accel_error<double><<<grid, ACCEL_WARPS * 32, 0, s>>>(
          static_cast<const double*>(gt), static_cast<const double*>(pred), n_joint, off.ptr, n_seq, n_win, vis,
          static_cast<double*>(per_window), valid);
      P2M_LAUNCH_OK();
    }
    P2M_TRY(segment_mean_launch<double>(static_cast<const double*>(per_window), 1, win_off, n_seq, valid, seq_mean, s));
  }
  return P2M_OK;
}

int p2m_segment_mean(int dtype, const void* values, int64_t width, const int64_t* offsets, int n_seg, int64_t n_rows,
                     const uint8_t* valid, double* out, p2m_stream_t stream) {
  if (!known_dtype(dtype) || !values || !out || width <= 0) {
    set_error("segment_mean: bad dtype code, null array or width <= 0");
    return P2M_ERR_INVALID;
  }
  P2M_TRY(check_offsets("segment_mean", offsets, n_seg, n_rows));
  int dev;
  P2M_TRY(arrays_device("segment_mean", {values, valid, out}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  StreamBuffer<long long> off(s);
  P2M_TRY(off.alloc((size_t)n_seg + 1, offsets));
  if (dtype == P2M_DTYPE_F32)
    return segment_mean_launch<float>(static_cast<const float*>(values), width, off.ptr, n_seg, valid, out, s);
  return segment_mean_launch<double>(static_cast<const double*>(values), width, off.ptr, n_seg, valid, out, s);
}

}  // extern "C"
