// Row f7 of SURVEY.md §8: the demo's weak-perspective camera fit on the GPU (demo/run.py:149-197 optimize_cam_param,
// lib/models/project_net.py OptimzeCamLayer), for a batch of people in ONE launch.
//
// One warp per person (grid-stride over people), lane = joint.  Each warp
//   1. builds the crop target: bbox1 = process_bbox(get_bbox(joints), aspect_ratio=1.0, scale=1.25) and
//      target = j2d_processing(joints, (crop, crop), bbox1, 0, 0, None) (lib/coord_utils.py:21-66,
//      lib/aug_utils.py:51-64,140-185), in numpy's dtypes and order: the box in float32 (get_bbox in the input's
//      dtype), the three float32 point pairs solved in float64 as cv2.getAffineTransform does (its 6 x 6 LU with
//      partial pivoting), the transformed points (t0 x + t1 y) + t2 in float64, truncated towards zero for integer
//      inputs, rounded to float32;
//   2. runs the reference's Adam loop on (s, tx, ty) in registers: out = ((p_xy + t) s) (crop/2) + crop/2, L1 loss
//      (mean over J x 2) against the first J target rows, its gradient with sign(0) = 0, and torch's single-tensor
//      Adam update (bias corrections in float64);
//   3. writes cam, bbox1, target, the loss of the final camera and, with image sizes, convert_crop_cam_to_orig_img
//      (demo/run.py:24-43) in float32.
// Every float32 step uses a round-to-nearest intrinsic (no FMA contraction) and the three gradient sums and the loss
// use one fixed xor-shuffle tree, so a person's result is bitwise deterministic, independent of its batch position,
// and reproduced bit for bit by oracle/camera_oracle.py::fit_f32_kernel_order.  No host synchronisation and no
// allocation: a fit can be captured in a CUDA graph.
#include <cuda_runtime.h>

#include <cfloat>
#include <climits>
#include <cmath>
#include <string>

#include "p2m_internal.h"

namespace p2m {
namespace {

constexpr int WARPS = 4;         // people per CTA
constexpr int MAX_GRID = 4096;   // CTAs of the grid-stride loop over people
constexpr int MAX_PHASES = 16;   // learning-rate phases

struct LrSchedule {
  int n;
  int start[MAX_PHASES];   // first step (0-based) of each phase, ascending, start[0] == 0
  double lr[MAX_PHASES];
};

// Sum over the 32 lanes by an xor butterfly; a + b == b + a, so every lane ends with the same bits.
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// torch.sgn: -1, 0 or +1, NaN for NaN
__device__ __forceinline__ float sgn(float d) { return d > 0.f ? 1.f : (d < 0.f ? -1.f : d); }

// get_bbox (coord_utils.py:21-39) in the input's arithmetic: float64 for integer and float64 inputs (numpy promotes
// the int64 sums / 2. to float64), float32 for float32 inputs.  -> [xmin, ymin, w, h] as float32
template <typename T>
__device__ __forceinline__ void get_bbox(T xmin, T xmax, T ymin, T ymax, float* box);
template <>
__device__ __forceinline__ void get_bbox<double>(double xmin, double xmax, double ymin, double ymax, float* box) {
  const double xc = __ddiv_rn(__dadd_rn(xmin, xmax), 2.0), w = __dsub_rn(xmax, xmin);
  const double yc = __ddiv_rn(__dadd_rn(ymin, ymax), 2.0), h = __dsub_rn(ymax, ymin);
  const double x0 = __dsub_rn(xc, __dmul_rn(0.5, w)), x1 = __dadd_rn(xc, __dmul_rn(0.5, w));
  const double y0 = __dsub_rn(yc, __dmul_rn(0.5, h)), y1 = __dadd_rn(yc, __dmul_rn(0.5, h));
  box[0] = __double2float_rn(x0);
  box[1] = __double2float_rn(y0);
  box[2] = __double2float_rn(__dsub_rn(x1, x0));
  box[3] = __double2float_rn(__dsub_rn(y1, y0));
}
template <>
__device__ __forceinline__ void get_bbox<float>(float xmin, float xmax, float ymin, float ymax, float* box) {
  const float xc = __fdiv_rn(__fadd_rn(xmin, xmax), 2.f), w = __fsub_rn(xmax, xmin);
  const float yc = __fdiv_rn(__fadd_rn(ymin, ymax), 2.f), h = __fsub_rn(ymax, ymin);
  const float x0 = __fsub_rn(xc, __fmul_rn(0.5f, w)), x1 = __fadd_rn(xc, __fmul_rn(0.5f, w));
  const float y0 = __fsub_rn(yc, __fmul_rn(0.5f, h)), y1 = __fadd_rn(yc, __fmul_rn(0.5f, h));
  box[0] = x0;
  box[1] = y0;
  box[2] = __fsub_rn(x1, x0);
  box[3] = __fsub_rn(y1, y0);
}

// process_bbox (coord_utils.py:42-66) in float32 on the float32 box, aspect ratio 1.0: false when the reference
// returns None (w * h <= 0 or a negative side after the w - 1 sanitising).
__device__ __forceinline__ bool process_bbox(float* b, float scale) {
  const float aspect = 1.f;
  const float x1 = b[0], y1 = b[1], x2 = __fadd_rn(b[0], __fsub_rn(b[2], 1.f)), y2 = __fadd_rn(b[1], __fsub_rn(b[3], 1.f));
  if (!(__fmul_rn(b[2], b[3]) > 0.f && x2 >= x1 && y2 >= y1)) return false;
  float w = __fsub_rn(x2, x1), h = __fsub_rn(y2, y1);
  const float cx = __fadd_rn(x1, __fdiv_rn(w, 2.f)), cy = __fadd_rn(y1, __fdiv_rn(h, 2.f));
  if (w > __fmul_rn(aspect, h)) h = __fdiv_rn(w, aspect);
  else if (w < __fmul_rn(aspect, h)) w = __fmul_rn(h, aspect);
  b[2] = __fmul_rn(w, scale);
  b[3] = __fmul_rn(h, scale);
  b[0] = __fsub_rn(cx, __fdiv_rn(b[2], 2.f));
  b[1] = __fsub_rn(cy, __fdiv_rn(b[3], 2.f));
  return true;
}

// get_3rd_point (aug_utils.py:182-185): p[2] = p[1] + (-(p[0] - p[1]).y, (p[0] - p[1]).x), float32
__device__ __forceinline__ void third_point(float (&p)[3][2]) {
  const float dx = __fsub_rn(p[0][0], p[1][0]), dy = __fsub_rn(p[0][1], p[1][1]);
  p[2][0] = __fadd_rn(p[1][0], -dy);
  p[2][1] = __fadd_rn(p[1][1], dx);
}

// Phase q of the schedule with static indices only (a dynamic index would copy the parameter to local memory)
__device__ __forceinline__ void lr_phase(const LrSchedule& s, int q, double* lr, int* next_start) {
#pragma unroll
  for (int i = 0; i < MAX_PHASES; ++i)
    if (i == q) *lr = s.lr[i];
  *next_start = INT_MAX;
#pragma unroll
  for (int i = 1; i < MAX_PHASES; ++i)
    if (i == q + 1 && i < s.n) *next_start = s.start[i];
}

// get_center_scale + get_affine_transform(rot = 0, output (crop, crop)) (coord_utils.py:7-18, aug_utils.py:140-185):
// the float32 point pairs, then cv2.getAffineTransform's float64 solve — OpenCV's LUImpl on the 6 x 6 system (partial
// pivoting on the first largest |pivot|, eliminations a += alpha b, back substitution by division).  Every loop is
// unrolled with static indices, so the system lives in registers.  false when a pivot is below 100 DBL_EPSILON
// (OpenCV's singular case).
__device__ __forceinline__ bool affine_from_box(const float* b, int crop, double* t) {
  const float ccx = __fadd_rn(b[0], __fmul_rn(b[2], 0.5f)), ccy = __fadd_rn(b[1], __fmul_rn(b[3], 0.5f));
  const float sw = b[2];
  float src[3][2], dst[3][2];
  src[0][0] = ccx;
  src[0][1] = ccy;
  src[1][0] = __double2float_rn(__dadd_rn((double)ccx, 0.0));                          // centre + (0, -src_w / 2)
  src[1][1] = __double2float_rn(__dadd_rn((double)ccy, (double)__fmul_rn(sw, -0.5f)));  // in float64, stored float32
  const double half = (double)crop * 0.5;
  dst[0][0] = (float)half;
  dst[0][1] = (float)half;
  dst[1][0] = __double2float_rn(__dadd_rn(half, 0.0));
  dst[1][1] = __double2float_rn(__dadd_rn(half, (double)__double2float_rn((double)crop * -0.5)));
  third_point(src);
  third_point(dst);
  double A[6][6], x[6];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int c = 0; c < 6; ++c) A[2 * i][c] = A[2 * i + 1][c] = 0.0;
    A[2 * i][0] = A[2 * i + 1][3] = (double)src[i][0];
    A[2 * i][1] = A[2 * i + 1][4] = (double)src[i][1];
    A[2 * i][2] = A[2 * i + 1][5] = 1.0;
    x[2 * i] = (double)dst[i][0];
    x[2 * i + 1] = (double)dst[i][1];
  }
  bool ok = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    int k = i;
    double best = fabs(A[i][i]);
#pragma unroll
    for (int j = i + 1; j < 6; ++j)
      if (fabs(A[j][i]) > best) {
        k = j;
        best = fabs(A[j][i]);
      }
    if (best < DBL_EPSILON * 100) ok = false;
#pragma unroll
    for (int j = i + 1; j < 6; ++j)
      if (j == k) {
#pragma unroll
        for (int c = i; c < 6; ++c) {
          const double s = A[i][c];
          A[i][c] = A[j][c];
          A[j][c] = s;
        }
        const double s = x[i];
        x[i] = x[j];
        x[j] = s;
      }
    const double d = __ddiv_rn(-1.0, A[i][i]);
#pragma unroll
    for (int j = i + 1; j < 6; ++j) {
      const double alpha = __dmul_rn(A[j][i], d);
#pragma unroll
      for (int c = i + 1; c < 6; ++c) A[j][c] = __dadd_rn(A[j][c], __dmul_rn(alpha, A[i][c]));
      x[j] = __dadd_rn(x[j], __dmul_rn(alpha, x[i]));
    }
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double s = x[i];
#pragma unroll
    for (int c = i + 1; c < 6; ++c) s = __dsub_rn(s, __dmul_rn(A[i][c], x[c]));
    x[i] = __ddiv_rn(s, A[i][i]);
  }
#pragma unroll
  for (int q = 0; q < 6; ++q) t[q] = x[q];
  return ok;
}

// convert_crop_cam_to_orig_img (demo/run.py:24-43) for one person, float32 in numpy's order; NaN when !ok
__device__ __forceinline__ void crop_cam_to_orig(const float* cam, const float* box, float W, float H, bool ok,
                                                 float* out) {
  const float qnan = __int_as_float(0x7fc00000);
  const float cx = __fadd_rn(box[0], __fdiv_rn(box[2], 2.f)), cy = __fadd_rn(box[1], __fdiv_rn(box[3], 2.f));
  const float hw = __fdiv_rn(W, 2.f), hh = __fdiv_rn(H, 2.f), h = box[3];
  const float sx = __fmul_rn(cam[0], __fdiv_rn(1.f, __fdiv_rn(W, h)));
  const float sy = __fmul_rn(cam[0], __fdiv_rn(1.f, __fdiv_rn(H, h)));
  const float tx = __fadd_rn(__fdiv_rn(__fdiv_rn(__fsub_rn(cx, hw), hw), sx), cam[1]);
  const float ty = __fadd_rn(__fdiv_rn(__fdiv_rn(__fsub_rn(cy, hh), hh), sy), cam[2]);
  out[0] = ok ? sx : qnan;
  out[1] = ok ? sy : qnan;
  out[2] = ok ? tx : qnan;
  out[3] = ok ? ty : qnan;
}

__global__ void __launch_bounds__(WARPS * 32) k_fit_camera(const double* __restrict__ px, int in_cols, int kind,
                                                           int n_in, const float* __restrict__ p3d, int n_joint,
                                                           const float* __restrict__ init, int batch, int crop,
                                                           int n_iter, LrSchedule sched, const float* __restrict__ img_wh,
                                                           float* __restrict__ cam_out, float* __restrict__ bbox_out,
                                                           float* __restrict__ target_out, float* __restrict__ loss_out,
                                                           float* __restrict__ orig_out) {
  const int lane = threadIdx.x & 31;
  const float qnan = __int_as_float(0x7fc00000);
  for (long long b = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5); b < batch; b += (long long)gridDim.x * WARPS) {
    // ---- 1. crop target
    const bool in_on = lane < n_in;
    const double* row = px + (b * n_in + (in_on ? lane : 0)) * in_cols;
    const double x = in_on ? row[0] : 0.0, y = in_on ? row[1] : 0.0;
    bool ok = !__any_sync(0xffffffffu, in_on && (isnan(x) || isnan(y)));
    float box[4];
    if (kind == P2M_CAM_INPUT_F32) {
      const float xf = (float)x, yf = (float)y;
      get_bbox<float>((float)warp_min(in_on ? xf : INFINITY), (float)warp_max(in_on ? xf : -INFINITY),
                      (float)warp_min(in_on ? yf : INFINITY), (float)warp_max(in_on ? yf : -INFINITY), box);
    } else {
      get_bbox<double>(warp_min(in_on ? x : INFINITY), warp_max(in_on ? x : -INFINITY), warp_min(in_on ? y : INFINITY),
                       warp_max(in_on ? y : -INFINITY), box);
    }
    double t[6];
    ok = ok && process_bbox(box, 1.25f);
    ok = ok && affine_from_box(box, crop, t);
    double X = __dadd_rn(__dadd_rn(__dmul_rn(t[0], x), __dmul_rn(t[1], y)), t[2]);
    double Y = __dadd_rn(__dadd_rn(__dmul_rn(t[3], x), __dmul_rn(t[4], y)), t[5]);
    if (kind == P2M_CAM_INPUT_INT) {  // written back into the integer array (aug_utils.py:58-59)
      X = trunc(X);
      Y = trunc(Y);
    }
    const float tgx = ok ? __double2float_rn(X) : qnan, tgy = ok ? __double2float_rn(Y) : qnan;
    if (in_on) {
      target_out[(b * n_in + lane) * 2 + 0] = tgx;
      target_out[(b * n_in + lane) * 2 + 1] = tgy;
    }
    if (lane == 0)
      for (int q = 0; q < 4; ++q) bbox_out[b * 4 + q] = ok ? box[q] : qnan;

    // ---- 2. the Adam fit of (s, tx, ty)
    const bool on = lane < n_joint;
    const float pjx = on ? p3d[(b * n_joint + lane) * 3 + 0] : 0.f;
    const float pjy = on ? p3d[(b * n_joint + lane) * 3 + 1] : 0.f;
    const float res = (float)((double)crop / 2.0);
    const float inv_n = __fdiv_rn(1.f, (float)(2 * n_joint));
    const float w1 = (float)(1.0 - 0.9), b2 = (float)0.999, w2 = (float)(1.0 - 0.999), eps = (float)1e-8;
    float p[3], m[3] = {0.f, 0.f, 0.f}, v[3] = {0.f, 0.f, 0.f};
    for (int q = 0; q < 3; ++q) p[q] = ok ? init[b * 3 + q] : qnan;
    double b1t = 1.0, b2t = 1.0;
    int phase = 0, next_start;
    double lr;
    lr_phase(sched, 0, &lr, &next_start);
    for (int it = 0; it < n_iter; ++it) {
      if (it == next_start) lr_phase(sched, ++phase, &lr, &next_start);
      const float qx = __fadd_rn(pjx, p[1]), qy = __fadd_rn(pjy, p[2]);
      const float ox = __fadd_rn(__fmul_rn(__fmul_rn(qx, p[0]), res), res);
      const float oy = __fadd_rn(__fmul_rn(__fmul_rn(qy, p[0]), res), res);
      const float gax = __fmul_rn(__fmul_rn(sgn(__fsub_rn(ox, tgx)), inv_n), res);
      const float gay = __fmul_rn(__fmul_rn(sgn(__fsub_rn(oy, tgy)), inv_n), res);
      float g[3];
      g[0] = warp_sum(on ? __fadd_rn(__fmul_rn(gax, qx), __fmul_rn(gay, qy)) : 0.f);
      g[1] = warp_sum(on ? __fmul_rn(gax, p[0]) : 0.f);
      g[2] = warp_sum(on ? __fmul_rn(gay, p[0]) : 0.f);
      b1t = __dmul_rn(b1t, 0.9);
      b2t = __dmul_rn(b2t, 0.999);
      const double step_size = __ddiv_rn(lr, __dsub_rn(1.0, b1t));
      const float bc2_sqrt = __double2float_rn(__dsqrt_rn(__dsub_rn(1.0, b2t)));
      const float neg_step = -__double2float_rn(step_size);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        m[q] = __fadd_rn(m[q], __fmul_rn(w1, __fsub_rn(g[q], m[q])));                 // exp_avg.lerp_(g, 1 - b1)
        v[q] = __fadd_rn(__fmul_rn(v[q], b2), __fmul_rn(__fmul_rn(w2, g[q]), g[q]));  // .mul_(b2).addcmul_(g, g, 1 - b2)
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v[q]), bc2_sqrt), eps);
        p[q] = __fadd_rn(p[q], __fdiv_rn(__fmul_rn(neg_step, m[q]), denom));          // addcdiv_(m, denom, -step_size)
      }
    }

    // ---- 3. epilogue: loss of the final camera, cam, orig_cam
    const float qx = __fadd_rn(pjx, p[1]), qy = __fadd_rn(pjy, p[2]);
    const float dx = __fsub_rn(__fadd_rn(__fmul_rn(__fmul_rn(qx, p[0]), res), res), tgx);
    const float dy = __fsub_rn(__fadd_rn(__fmul_rn(__fmul_rn(qy, p[0]), res), res), tgy);
    const float l1 = warp_sum(on ? __fadd_rn(fabsf(dx), fabsf(dy)) : 0.f);
    if (lane == 0) {
      loss_out[b] = __fdiv_rn(l1, (float)(2 * n_joint));
      for (int q = 0; q < 3; ++q) cam_out[b * 3 + q] = p[q];
      if (orig_out) crop_cam_to_orig(p, box, img_wh[b * 2 + 0], img_wh[b * 2 + 1], ok, orig_out + b * 4);
    }
  }
}

// convert_crop_cam_to_orig_img alone: one thread per person
__global__ void __launch_bounds__(128) k_crop_cam_to_orig(const float* __restrict__ cam, const float* __restrict__ bbox,
                                                          const float* __restrict__ img_wh, int batch,
                                                          float* __restrict__ out) {
  for (long long b = (long long)blockIdx.x * 128 + threadIdx.x; b < batch; b += (long long)gridDim.x * 128)
    crop_cam_to_orig(cam + b * 3, bbox + b * 4, img_wh[b * 2 + 0], img_wh[b * 2 + 1], true, out + b * 4);
}

}  // namespace
}  // namespace p2m

using namespace p2m;

extern "C" {

int p2m_fit_camera(const double* joints_px, int in_cols, int in_kind, int n_in_joint, const float* pred_joints3d,
                   int n_joint, const float* init_cam, int batch, int crop, int n_iter, const int32_t* lr_steps,
                   const double* lr_values, int n_lr, const float* img_wh, float* cam, float* bbox, float* target,
                   float* loss, float* orig_cam, p2m_stream_t stream) {
  if (!joints_px || !pred_joints3d || !init_cam || !cam || !bbox || !target || !loss || (!img_wh != !orig_cam)) {
    set_error("fit_camera: null input or output (img_wh and orig_cam go together)");
    return P2M_ERR_INVALID;
  }
  if (batch <= 0 || n_joint <= 0 || n_joint > 32 || n_in_joint > 32 || n_joint > n_in_joint || in_cols < 2 ||
      crop <= 0 || crop > (1 << 24) || n_iter < 0 ||
      (in_kind != P2M_CAM_INPUT_F64 && in_kind != P2M_CAM_INPUT_INT && in_kind != P2M_CAM_INPUT_F32)) {
    set_error("fit_camera: bad argument (need 0 < J <= Jin <= 32, batch > 0, 0 < crop <= 2^24, n_iter >= 0, "
              "in_cols >= 2, a known input kind); got J = " + std::to_string(n_joint) + ", Jin = " +
              std::to_string(n_in_joint) + ", batch = " + std::to_string(batch) + ", crop = " + std::to_string(crop));
    return P2M_ERR_INVALID;
  }
  if (!lr_steps || !lr_values || n_lr <= 0 || n_lr > MAX_PHASES || lr_steps[0] != 0) {
    set_error("fit_camera: the learning-rate schedule needs 1 to " + std::to_string(MAX_PHASES) +
              " phases, the first starting at step 0");
    return P2M_ERR_INVALID;
  }
  LrSchedule sched{};
  sched.n = n_lr;
  for (int i = 0; i < n_lr; ++i) {
    if ((i > 0 && lr_steps[i] <= lr_steps[i - 1]) || !std::isfinite(lr_values[i])) {
      set_error("fit_camera: learning-rate phases must start at increasing steps and have finite rates");
      return P2M_ERR_INVALID;
    }
    sched.start[i] = lr_steps[i];
    sched.lr[i] = lr_values[i];
  }
  int dev;
  P2M_TRY(arrays_device("fit_camera", {joints_px, pred_joints3d, init_cam, img_wh, cam, bbox, target, loss, orig_cam},
                        &dev));
  DeviceGuard guard(dev);
  k_fit_camera<<<grid_for(batch, WARPS, MAX_GRID), WARPS * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      joints_px, in_cols, in_kind, n_in_joint, pred_joints3d, n_joint, init_cam, batch, crop, n_iter, sched, img_wh,
      cam, bbox, target, loss, orig_cam);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_crop_cam_to_orig(const float* cam, const float* bbox, const float* img_wh, int batch, float* orig_cam,
                         p2m_stream_t stream) {
  if (!cam || !bbox || !img_wh || !orig_cam || batch <= 0) {
    set_error("crop_cam_to_orig: null array or batch <= 0");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("crop_cam_to_orig", {cam, bbox, img_wh, orig_cam}, &dev));
  DeviceGuard guard(dev);
  k_crop_cam_to_orig<<<grid_for(batch, 128, MAX_GRID), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      cam, bbox, img_wh, batch, orig_cam);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
