// The target side of the datasets' __getitem__ for a whole batch on the GPU (SURVEY.md §8 row f11):
//  * p2m_camera_frame_coords  every dataset's get_smpl_coord / get_mano_coord (Human36M, AMASS, FreiHAND, MuCo, COCO,
//                             SURREAL, 3DPW): a few flags on one implementation, five launches:
//      1. k_frame_prep    one warp per sample: the root axis-angle rotated by the camera R (fp64 Rodrigues, R M, fp64
//                         log map, rounded to float32 where the reference stores it into its float32 pose), the betas
//                         clamp (any |beta| > 3 -> zeros) and the per-sample "all-zero betas -> model betas" rule of a
//                         one-sample SMPL_Layer call, and the translation the layer takes
//      2-4. the body model's forward (k_batch_flags, k_pose, k_lbs) with P2M_BETAS_AS_GIVEN
//      5. k_frame_finish  per (sample, 256-vertex chunk): Human36M's translation compensation or AMASS's + t, the
//                         m -> mm scaling, MuCo's face-keypoint vertices appended to the joints
//  * p2m_sample_targets       the targets and meta of Human36M, COCO, MuCo and AMASS __getitem__ (pose2mesh_net and
//                             posenet) from the camera-frame mesh, one launch (k_sample_targets, one CTA per sample,
//                             branching on the dataset): both sparse joint regressors in one pass (fp64), COCO pelvis /
//                             neck, the dataset's projection, rooting, its fitting test and validity masks, and the lift
//                             target's rotation and flip; p2m_h36m_targets is its unaugmented Human36M case.  3DPW
//                             is its fifth case.
//  * p2m_layer_joint_targets  SURREAL's and FreiHAND's targets, which take the layer's own joints instead of a
//                             regressor's: one launch (k_layer_joint_targets, one CTA per sample), float32 rooting at
//                             joint 0, SURREAL's projection and its lift target's rotation and flip.
// No atomics and fixed orders: a sample's result is bitwise independent of its batch position and of the batch size;
// nothing is read back to the host, so every call can be captured in a CUDA graph.
#include <cuda_runtime.h>

#include <cmath>
#include <string>
#include <vector>

#include "p2m_internal.h"

namespace p2m {
namespace {

constexpr int PREP_WARPS = 4;        // samples per k_frame_prep CTA
constexpr int FIN_T = 256;           // threads (vertices) per k_frame_finish CTA
constexpr int H36_T = 256;           // threads per k_sample_targets CTA
constexpr int LJ_T = 256;            // threads per k_layer_joint_targets CTA
constexpr int SMPL_J = 24, MANO_J = 21;
constexpr int MAX_EXTRA = 8;         // appended vertex joints (MuCo: 5 face keypoints)
constexpr int MAX_BATCH = 1 << 24;
constexpr int NJ = 17;               // joints of each regressor
constexpr int NR = 2 * NJ;           // regressor rows: H36M 0..16, COCO 17..33
constexpr int COCO_J = NJ + 2;       // + pelvis, neck (Human36M.add_pelvis_and_neck)
constexpr int N_COCO_KPS = 17;       // COCO's annotation keypoints
constexpr int COCO_LSH = 5, COCO_RSH = 6, COCO_LHIP = 11, COCO_RHIP = 12, COCO_PELVIS = 17;

constexpr int ALL_FLAGS = P2M_FRAME_ROTATE_ROOT | P2M_FRAME_CLAMP_BETAS | P2M_FRAME_ZERO_BETAS_MODEL | P2M_FRAME_LAYER_TRANS_T |
                          P2M_FRAME_LAYER_TRANS | P2M_FRAME_H36M_COMPENSATE | P2M_FRAME_ADD_T | P2M_FRAME_TO_MM;

struct Extra {
  int n;
  int v[MAX_EXTRA];
};

// The root's rotation in fp64: M = R axangle2mat(r / |r|, |r|) (transforms3d), then its axis-angle vector.  The log map
// takes theta = atan2(|w|, c) with w the skew part and c = (tr M - 1) / 2: below 2 pi / 3 the axis is w / |w| (well
// conditioned down to angle 0, where theta / |w| -> 1), above it the axis comes from the symmetric part
// M + M^T - 2 c I = 2 (1 - c) a a^T (well conditioned up to pi), signed by w.  An exactly zero root is the identity.
__device__ void rotate_root(const float r[3], const float* Rc, float out[3]) {
  const double x = r[0], y = r[1], z = r[2];
  const double ang = sqrt(x * x + y * y + z * z);
  double A[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  if (ang > 0.0) {
    const double ax = x / ang, ay = y / ang, az = z / ang;
    const double c = cos(ang), s = sin(ang), C = 1.0 - c;
    A[0] = ax * ax * C + c, A[1] = ax * ay * C - az * s, A[2] = ax * az * C + ay * s;
    A[3] = ax * ay * C + az * s, A[4] = ay * ay * C + c, A[5] = ay * az * C - ax * s;
    A[6] = ax * az * C - ay * s, A[7] = ay * az * C + ax * s, A[8] = az * az * C + c;
  }
  double M[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      M[3 * i + j] = (double)Rc[3 * i] * A[j] + (double)Rc[3 * i + 1] * A[3 + j] + (double)Rc[3 * i + 2] * A[6 + j];
  const double w0 = 0.5 * (M[7] - M[5]), w1 = 0.5 * (M[2] - M[6]), w2 = 0.5 * (M[3] - M[1]);
  const double sn = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
  const double cs = fmin(1.0, fmax(-1.0, 0.5 * (M[0] + M[4] + M[8] - 1.0)));
  const double th = atan2(sn, cs);
  double o0, o1, o2;
  if (cs > -0.5) {
    const double k = sn > 0.0 ? th / sn : 1.0;
    o0 = w0 * k, o1 = w1 * k, o2 = w2 * k;
  } else {
    // B = (M + M^T) / 2 - c I = (1 - c) a a^T; the largest diagonal entry gives the best-conditioned axis component
    const double d0 = M[0] - cs, d1 = M[4] - cs, d2 = M[8] - cs;
    const double b01 = 0.5 * (M[1] + M[3]), b02 = 0.5 * (M[2] + M[6]), b12 = 0.5 * (M[5] + M[7]);
    double a0, a1, a2;
    if (d0 >= d1 && d0 >= d2) {
      a0 = sqrt(fmax(d0, 0.0)), a1 = b01 / a0, a2 = b02 / a0;
    } else if (d1 >= d2) {
      a1 = sqrt(fmax(d1, 0.0)), a0 = b01 / a1, a2 = b12 / a1;
    } else {
      a2 = sqrt(fmax(d2, 0.0)), a0 = b02 / a2, a1 = b12 / a2;
    }
    const double n = sqrt(a0 * a0 + a1 * a1 + a2 * a2);
    const double sg = (a0 * w0 + a1 * w1 + a2 * w2) < 0.0 ? -1.0 : 1.0;
    const double k = sg * th / n;
    o0 = a0 * k, o1 = a1 * k, o2 = a2 * k;
  }
  out[0] = (float)o0, out[1] = (float)o1, out[2] = (float)o2;
}

// One warp per sample: pose' [B, 3J], betas' [B, S] (resolved per sample), layer trans [B, 3] (when the preset has one).
__global__ void __launch_bounds__(PREP_WARPS * 32) k_frame_prep(int flags, int batch, int J, int S,
                                                                const float* __restrict__ mbetas,
                                                                const float* __restrict__ pose,
                                                                const float* __restrict__ betas,
                                                                const float* __restrict__ trans,
                                                                const float* __restrict__ R, const float* __restrict__ t,
                                                                float* __restrict__ pose_o, float* __restrict__ betas_o,
                                                                float* __restrict__ trans_o) {
  const int lane = threadIdx.x & 31;
  const long long b = (long long)blockIdx.x * PREP_WARPS + threadIdx.x / 32;
  if (b >= batch) return;
  const float* p = pose + b * 3 * J;
  float* po = pose_o + b * 3 * J;
  for (int i = lane + ((flags & P2M_FRAME_ROTATE_ROOT) ? 3 : 0); i < 3 * J; i += 32) po[i] = p[i];
  if ((flags & P2M_FRAME_ROTATE_ROOT) && lane == 0) {
    const float r[3] = {p[0], p[1], p[2]};
    float o[3];
    rotate_root(r, R + b * 9, o);
    po[0] = o[0], po[1] = o[1], po[2] = o[2];
  }
  // smpl_shape[(smpl_shape.abs() > 3).any(dim=1)] = 0, then SMPL_Layer's norm == 0 test on this one sample
  int big = 0, nonzero = 0;
  for (int s = lane; s < S; s += 32) {
    const float x = betas[b * S + s];
    big |= fabsf(x) > 3.f;
    nonzero |= !(x == 0.f);
  }
  big = __any_sync(0xffffffffu, big) && (flags & P2M_FRAME_CLAMP_BETAS);
  nonzero = __any_sync(0xffffffffu, nonzero) && !big;
  if (!(flags & P2M_FRAME_ZERO_BETAS_MODEL)) nonzero = !big;  // ManoLayer uses explicit betas as given
  for (int s = lane; s < S; s += 32) betas_o[b * S + s] = nonzero ? betas[b * S + s] : mbetas[s];
  if (lane < 3 && trans_o) {
    if (flags & P2M_FRAME_LAYER_TRANS_T) trans_o[b * 3 + lane] = t[b * 3 + lane];
    if (flags & P2M_FRAME_LAYER_TRANS) trans_o[b * 3 + lane] = trans[b * 3 + lane];
  }
}

// The steps after the layer, in the reference's float32 order.  grid (vertex chunks, samples); the chunk-0 CTA also
// writes the sample's joints: the layer's, then the extra vertex joints (MuCo's face keypoints, taken from the layer's
// mesh and scaled like it).
__global__ void __launch_bounds__(FIN_T) k_frame_finish(int flags, int V, int n_out, Extra ex,
                                                        const float* __restrict__ trans, const float* __restrict__ R,
                                                        const float* __restrict__ t,
                                                        const float* __restrict__ verts_in,
                                                        const float* __restrict__ joints_in,
                                                        float* __restrict__ verts, float* __restrict__ joints) {
  const long long b = blockIdx.y;
  const float* jin = joints_in + b * n_out * 3;
  const float* vin = verts_in + b * V * 3;
  float off[3] = {0.f, 0.f, 0.f};
  if (flags & P2M_FRAME_H36M_COMPENSATE) {
    // smpl_trans = R trans + t / 1000;  smpl_trans = smpl_trans - J_0 + R J_0  (Human36M/dataset.py:288-291)
    const float* Rb = R + b * 9;
    const float* tr = trans + b * 3;
    for (int r = 0; r < 3; ++r) {
      const float rt = __fadd_rn(__fadd_rn(__fmul_rn(Rb[3 * r], tr[0]), __fmul_rn(Rb[3 * r + 1], tr[1])),
                                 __fmul_rn(Rb[3 * r + 2], tr[2]));
      const float rj = __fadd_rn(__fadd_rn(__fmul_rn(Rb[3 * r], jin[0]), __fmul_rn(Rb[3 * r + 1], jin[1])),
                                 __fmul_rn(Rb[3 * r + 2], jin[2]));
      off[r] = __fadd_rn(__fsub_rn(__fadd_rn(rt, __fdiv_rn(t[b * 3 + r], 1000.f)), jin[r]), rj);
    }
  } else if (flags & P2M_FRAME_ADD_T) {
    for (int r = 0; r < 3; ++r) off[r] = t[b * 3 + r];
  }
  const float scale = (flags & P2M_FRAME_TO_MM) ? 1000.f : 1.f;
  const int v = blockIdx.x * FIN_T + threadIdx.x;
  if (v < V)
    for (int q = 0; q < 3; ++q) verts[(b * V + v) * 3 + q] = __fmul_rn(__fadd_rn(vin[3 * v + q], off[q]), scale);
  if (blockIdx.x == 0) {
    const int n_all = n_out + ex.n;
    for (int e = threadIdx.x; e < 3 * n_all; e += FIN_T) {
      const int o = e / 3, q = e % 3;
      const float x = o < n_out ? jin[e] : vin[3 * ex.v[o - n_out] + q];
      joints[b * n_all * 3 + e] = __fmul_rn(__fadd_rn(x, off[q]), scale);
    }
  }
}

// One CTA per sample: the target side of the four datasets' __getitem__ (Human36M/dataset.py:301-333,344-405,
// COCO/dataset.py:182-287, MuCo/dataset.py:232-330, AMASS/dataset.py:229-309).  Regression in fp64 over the
// regressors' non-zero entries in ascending vertex order.  Human36M: rows 0..16 (H36M) on the mesh rooted at the
// annotation's pelvis, the H36M joints are the annotation's; the other datasets: every row on the camera-frame mesh, the
// H36M joints are the regressed rows 0..16 (get_joints_from_mesh).  Rows 17..33 (COCO) on the camera-frame mesh.  The
// mesh target is (mesh - H36M joint 0) / 1000 rounded once.
struct SampleArgs {
  int V, coco, batch, dataset;
  double thr;
  const int* reg_ptr;      // [NR + 1]
  const int* reg_idx;      // vertex of each non-zero
  const double* reg_val;
  const float* mesh_cam;   // [B, V, 3] mm
  const float* joint_cam;  // [B, 17, 3] mm (Human36M)
  const float* f;          // [B, 2] (Human36M, MuCo, AMASS)
  const float* c;          // [B, 2]
  const float* s;          // [B, n_s] (COCO)
  int n_s;
  const float* t;          // [B, 2] (COCO)
  const float* kps;        // [B, 17, 2] (COCO's annotation keypoints)
  const float* kps_valid;  // [B, 17]
  const float* rot;        // [B] degrees, or null (the lift target's augmentation)
  const int* flip;         // [B], or null
  float* mesh;             // [B, V, 3] m
  float* lift;             // [B, J, 3]
  float* reg;              // [B, 17, 3]
  float* mesh_valid;       // [B, V]
  float* lift_valid;       // [B, J]
  float* reg_valid;        // [B, 17]
  float* joint_valid;      // [B, J] posenet's mask, or null
  float* joint_img;        // [B, J, 2]
  float* fit_err;          // [B]
};

// MuCo's get_fitting_error (MuCo/dataset.py:246-262) receives the Human3.6M-ordered joints where it expects MuCo's 21:
// it roots them at row 14 (MuCo's pelvis index) and transform_joint_to_other_db moves source row MUCO_SRC[k] into
// Human3.6M slot MUCO_DST[k] by MuCo's names; the other three slots are invalid and dropped.
__constant__ int MUCO_DST[14] = {0, 1, 2, 3, 4, 5, 6, 10, 11, 12, 13, 14, 15, 16};
__constant__ int MUCO_SRC[14] = {14, 8, 9, 10, 11, 12, 13, 16, 5, 6, 7, 2, 3, 4};
constexpr int MUCO_ROOT = 14;
constexpr int COCO_FIT_RES = 64;  // COCO.get_fitting_error's 64 x 64 crop

// the input set's joint j (absolute, mm) of the sample in shared memory
__device__ __forceinline__ double input_joint(const double (*sreg)[3], const double (*sjc)[3], int coco, int j, int q) {
  if (!coco) return sjc[j][q];
  if (j < NJ) return sreg[NJ + j][q];
  const int a = j == COCO_PELVIS ? COCO_LHIP : COCO_LSH, b = j == COCO_PELVIS ? COCO_RHIP : COCO_RSH;
  return (sreg[NJ + a][q] + sreg[NJ + b][q]) * 0.5;
}
// the dataset's projection of a camera-frame point p (mm) to image pixels, axis q
__device__ __forceinline__ double project(const SampleArgs& a, long long b, const double p[3], int q) {
  if (a.dataset == P2M_DATASET_COCO)  // (xy / 1000) s + t (COCO/dataset.py:200-210)
    return p[q] / 1000.0 * (double)a.s[b * a.n_s + (a.n_s == 2 ? q : 0)] + (double)a.t[b * 2 + q];
  if (a.dataset == P2M_DATASET_AMASS)  // cam2pixel(joint / 1000, f, c) (AMASS/dataset.py:229-241)
    return (p[q] / 1000.0) / (p[2] / 1000.0) * (double)a.f[b * 2 + q] + (double)a.c[b * 2 + q];
  return p[q] / p[2] * (double)a.f[b * 2 + q] + (double)a.c[b * 2 + q];  // cam2pixel (lib/coord_utils.py:104-109)
}

// j3d_processing's rotation (lib/aug_utils.py:67-83): x, y rotated by -rot degrees in fp64 (rot 0: untouched)
__device__ __forceinline__ void j3d_rotate(float rot, double l[3]) {
  if (rot == 0.f) return;
  double sn, cs;
  sincospi(__ddiv_rn(-(double)rot, 180.0), &sn, &cs);  // (sin, cos)(-pi rot / 180)
  const double x = l[0], y = l[1];
  l[0] = __dadd_rn(__dmul_rn(cs, x), __dmul_rn(-sn, y));
  l[1] = __dadd_rn(__dmul_rn(sn, x), __dmul_rn(cs, y));
}

__global__ void __launch_bounds__(H36_T) k_sample_targets(SampleArgs a) {
  __shared__ double sreg[NR][3], sjc[NJ][3], sroot[3], sfit[NJ][3];
  __shared__ float svalid;
  const long long b = blockIdx.x;
  const int tid = threadIdx.x, V = a.V;
  const bool h36m = a.dataset == P2M_DATASET_HUMAN36M;
  const float* mc = a.mesh_cam + b * V * 3;
  if (h36m) {
    const float* jc = a.joint_cam + b * NJ * 3;
    if (tid < 3) sroot[tid] = (double)jc[tid];
    if (tid < 3 * NJ) sjc[tid / 3][tid % 3] = (double)jc[tid];
  }
  __syncthreads();
  if (tid < 3 * NR) {
    const int r = tid / 3, q = tid % 3;
    const double sub = (h36m && r < NJ) ? sroot[q] : 0.0;
    double acc = 0.0;
    for (int e = a.reg_ptr[r]; e < a.reg_ptr[r + 1]; ++e)
      acc = fma(a.reg_val[e], (double)mc[3 * a.reg_idx[e] + q] - sub, acc);
    sreg[r][q] = acc;
  }
  __syncthreads();
  if (!h36m) {  // the regressed H36M joints are the sample's; rooting at their row 0
    if (tid < 3 * NJ) sjc[tid / 3][tid % 3] = sreg[tid / 3][tid % 3];
    if (tid < 3) sroot[tid] = sreg[0][tid];
    __syncthreads();
  }
  if (a.dataset == P2M_DATASET_MUCO && tid < 3 * NJ) {  // the regressor on the rooted mesh (get_fitting_error)
    const int r = tid / 3, q = tid % 3;
    double acc = 0.0;
    for (int e = a.reg_ptr[r]; e < a.reg_ptr[r + 1]; ++e)
      acc = fma(a.reg_val[e], (double)mc[3 * a.reg_idx[e] + q] - sroot[q], acc);
    sfit[r][q] = acc;
  }
  __syncthreads();
  const int J = a.coco ? COCO_J : NJ;
  if (h36m && tid == 0) {
    // get_fitting_error: translation-aligned mean joint distance between the annotation and the regressed H36M joints
    double mj[3] = {0, 0, 0}, ms[3] = {0, 0, 0};
    for (int j = 0; j < NJ; ++j)
      for (int q = 0; q < 3; ++q) mj[q] += sjc[j][q] - sroot[q], ms[q] += sreg[j][q];
    double err = 0.0;
    for (int j = 0; j < NJ; ++j) {
      double d2 = 0.0;
      for (int q = 0; q < 3; ++q) {
        const double d = (sjc[j][q] - sroot[q]) - (sreg[j][q] - ms[q] / NJ + mj[q] / NJ);
        d2 += d * d;
      }
      err += sqrt(d2);
    }
    err /= NJ;
    svalid = err > a.thr ? 0.f : 1.f;  // a NaN error keeps the sample, as `error > fitting_thr` does
    a.fit_err[b] = (float)err;
  } else if (a.dataset == P2M_DATASET_MUCO && tid == 0) {
    // the quirk above, kept: the scrambled, float32 copy of the rooted joints against the regressor on the rooted mesh
    const auto hj = [&](int k, int q) {  // transform_joint_to_other_db's float32 array
      return (double)(float)((sjc[MUCO_SRC[k]][q] - sroot[q]) - (sjc[MUCO_ROOT][q] - sroot[q]));
    };
    double mj[3] = {0, 0, 0}, ms[3] = {0, 0, 0};
    for (int k = 0; k < 14; ++k)
      for (int q = 0; q < 3; ++q) mj[q] += hj(k, q), ms[q] += sfit[MUCO_DST[k]][q];
    double err = 0.0;
    for (int k = 0; k < 14; ++k) {
      double d2 = 0.0;
      for (int q = 0; q < 3; ++q) {
        const double d = hj(k, q) - (sfit[MUCO_DST[k]][q] - ms[q] / 14 + mj[q] / 14);
        d2 += d * d;
      }
      err += sqrt(d2);
    }
    err /= 14;
    svalid = err > a.thr ? 0.f : 1.f;
    a.fit_err[b] = (float)err;
  } else if (a.dataset == P2M_DATASET_COCO && tid < 32) {
    // COCO.get_fitting_error (COCO/dataset.py:196-214): the box process_bbox(get_bbox(input-set joint_img), aspect 1),
    // the regressed COCO rows 0-16 and the annotation keypoints through its 64 x 64 rot-0 crop, float32 distances,
    // the mean over the annotation-visible joints (none visible: NaN, which keeps the sample)
    const int lane = tid;
    double p[3];
    float ix = 0.f, iy = 0.f;
    if (lane < J) {
      for (int q = 0; q < 3; ++q) p[q] = input_joint(sreg, sjc, a.coco, lane, q);
      ix = (float)project(a, b, p, 0), iy = (float)project(a, b, p, 1);
    }
    const PoseCrop m = pose_crop(ix, iy, lane < J, COCO_FIT_RES, COCO_FIT_RES);
    float d = 0.f;
    const bool vis = lane < N_COCO_KPS && a.kps_valid[b * N_COCO_KPS + lane] > 0.f;
    if (vis) {
      for (int q = 0; q < 3; ++q) p[q] = sreg[NJ + lane][q];
      const float2 r = crop_point(m, (float)project(a, b, p, 0), (float)project(a, b, p, 1), COCO_FIT_RES,
                                  COCO_FIT_RES, 0);
      const float2 k = crop_point(m, a.kps[(b * N_COCO_KPS + lane) * 2], a.kps[(b * N_COCO_KPS + lane) * 2 + 1],
                                  COCO_FIT_RES, COCO_FIT_RES, 0);
      const float dx = __fsub_rn(k.x, r.x), dy = __fsub_rn(k.y, r.y);
      d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
    }
    double sum = vis ? (double)d : 0.0;
    int n = __popc(__ballot_sync(0xffffffffu, vis));
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) {
      const double err = sum / n;  // 0 / 0 = NaN with no visible joint
      svalid = err > a.thr ? 0.f : 1.f;
      a.fit_err[b] = (float)err;
    }
  } else if ((a.dataset == P2M_DATASET_AMASS || a.dataset == P2M_DATASET_PW3D) && tid == 0) {
    svalid = 1.f;  // no fitting test
    a.fit_err[b] = 0.f;
  }
  __syncthreads();
  const float valid = svalid;
  // masks zeroed by the test: Human36M the mesh and (coco set) the lift; COCO and MuCo the mesh, lift and reg
  const float reg_v = (a.dataset == P2M_DATASET_COCO || a.dataset == P2M_DATASET_MUCO) ? valid : 1.f;
  const float lift_v = (h36m && !a.coco) ? 1.f : valid;
  // posenet's joint_valid: Human36M's coco set and COCO take the test, MuCo and AMASS are always valid
  const float joint_v = (h36m ? a.coco : a.dataset == P2M_DATASET_COCO) ? valid : 1.f;
  if (tid < 3 * NJ) {
    const int j = tid / 3, q = tid % 3;
    a.reg[b * NJ * 3 + tid] = (float)(sjc[j][q] - sroot[q]);
    if (q == 0) a.reg_valid[b * NJ + j] = reg_v;
  }
  if (tid < J) {
    const int j = tid;
    double p[3], l[3];
    // the lift target of joint s: j, or its flip partner (j3d_processing swaps the pairs)
    const int flip = a.flip ? a.flip[b] : 0;
    const int s = flip ? flip_partner(a.coco ? P2M_JOINTS_COCO : P2M_JOINTS_HUMAN36, j) : j;
    for (int q = 0; q < 3; ++q) {
      p[q] = input_joint(sreg, sjc, a.coco, j, q);
      if (a.coco) {
        // the regressed COCO joints with pelvis and neck, rooted at the pelvis (fp64)
        l[q] = input_joint(sreg, sjc, 1, s, q) - input_joint(sreg, sjc, 1, COCO_PELVIS, q);
      } else {
        // Human36M's joint_cam is float32 in the annotation: rooted in float32; the regressed joints in fp64
        const double d = sjc[s][q] - sroot[q];
        l[q] = h36m ? (double)(float)d : d;
      }
    }
    // j3d_processing: the rotation, then x negated under a flip; the mesh and reg_pose3d targets are never augmented
    // (data/Human36M/dataset.py:373, the same in every dataset)
    j3d_rotate(a.rot ? a.rot[b] : 0.f, l);
    if (flip) l[0] = -l[0];
    for (int q = 0; q < 3; ++q) a.lift[(b * J + j) * 3 + q] = (float)l[q];
    a.joint_img[(b * J + j) * 2] = (float)project(a, b, p, 0);
    a.joint_img[(b * J + j) * 2 + 1] = (float)project(a, b, p, 1);
    a.lift_valid[b * J + j] = lift_v;
    if (a.joint_valid) a.joint_valid[b * J + j] = joint_v;
  }
  for (int e = tid; e < 3 * V; e += H36_T) {
    a.mesh[b * V * 3 + e] = (float)(((double)mc[e] - sroot[e % 3]) / 1000.0);
    if (e < V) a.mesh_valid[b * V + e] = valid;
  }
}

// One CTA per sample: SURREAL's and FreiHAND's targets (SURREAL/dataset.py:143-203, FreiHAND/dataset.py:139-192).
// The reference roots its float32 arrays at the layer's joint 0 in float32 and divides the mesh by 1000 in float32;
// SURREAL's lift target goes through j3d_processing, and its reg_pose3d is that same reassigned array (:178,195).
struct LayerArgs {
  int dataset, V, J;
  const float* mesh_cam;   // [B, V, 3] mm
  const float* joint_cam;  // [B, J, 3] mm, the layer's joints
  const float* f;          // [B, 2] (SURREAL)
  const float* c;
  const float* rot;        // [B] degrees, or null (SURREAL)
  const int* flip;         // [B], or null (SURREAL)
  float* mesh;             // [B, V, 3] m
  float* lift;             // [B, J, 3]
  float* reg;              // [B, J, 3]
  float* mesh_valid;       // [B, V]
  float* lift_valid;       // [B, J]
  float* reg_valid;        // [B, J]
  float* joint_valid;      // [B, J], or null
  float* joint_img;        // [B, J, 2] (SURREAL)
  float* fit_err;          // [B]
};

__global__ void __launch_bounds__(LJ_T) k_layer_joint_targets(LayerArgs a) {
  const long long b = blockIdx.x;
  const int tid = threadIdx.x, V = a.V, J = a.J;
  const float* jc = a.joint_cam + b * J * 3;
  const float root[3] = {jc[0], jc[1], jc[2]};
  if (tid < J) {
    const int j = tid;
    const bool surreal = a.dataset == P2M_DATASET_SURREAL;
    const int flip = (surreal && a.flip) ? a.flip[b] : 0;
    const int s = flip ? flip_partner(P2M_JOINTS_SMPL, j) : j;
    double l[3];
    for (int q = 0; q < 3; ++q) l[q] = (double)__fsub_rn(jc[3 * s + q], root[q]);
    if (surreal) {
      j3d_rotate(a.rot ? a.rot[b] : 0.f, l);
      if (flip) l[0] = -l[0];
      // cam2pixel of the absolute joints, taken before the rooting (SURREAL/dataset.py:151-153)
      const double z = jc[3 * j + 2];
      for (int q = 0; q < 2; ++q)
        a.joint_img[(b * J + j) * 2 + q] = (float)((double)jc[3 * j + q] / z * (double)a.f[b * 2 + q] +
                                                   (double)a.c[b * 2 + q]);
    }
    for (int q = 0; q < 3; ++q) {
      a.lift[(b * J + j) * 3 + q] = (float)l[q];
      a.reg[(b * J + j) * 3 + q] = (float)l[q];
    }
    a.lift_valid[b * J + j] = 1.f;
    a.reg_valid[b * J + j] = 1.f;
    if (a.joint_valid) a.joint_valid[b * J + j] = 1.f;
  }
  if (tid == 0) a.fit_err[b] = 0.f;
  // bandwidth work: the mesh streamed once with strided threads
  const float* mc = a.mesh_cam + b * V * 3;
  for (int e = tid; e < 3 * V; e += LJ_T) {
    a.mesh[b * V * 3 + e] = __fdiv_rn(__fsub_rn(mc[e], root[e % 3]), 1000.f);
    if (e < V) a.mesh_valid[b * V + e] = 1.f;
  }
}

struct FrameLayout {
  size_t pose, betas, trans, verts, joints, body, total;
};
FrameLayout frame_layout(const BodyModelInfo& m, int batch, size_t body_bytes) {
  FrameLayout l;
  l.pose = 0;
  l.betas = l.pose + align_up(sizeof(float) * (size_t)batch * 3 * m.J);
  l.trans = l.betas + align_up(sizeof(float) * (size_t)batch * m.S);
  l.verts = l.trans + align_up(sizeof(float) * (size_t)batch * 3);
  l.joints = l.verts + align_up(sizeof(float) * (size_t)batch * m.V * 3);
  l.body = l.joints + align_up(sizeof(float) * (size_t)batch * m.n_out * 3);
  l.total = l.body + body_bytes;
  return l;
}

}  // namespace
}  // namespace p2m

using namespace p2m;

struct p2m_h36m_regressors {
  int device = 0, V = 0;
  int* ptr = nullptr;
  int* idx = nullptr;
  double* val = nullptr;
};

extern "C" {

size_t p2m_camera_frame_workspace_bytes(const p2m_body_model_t* m, int batch) {
  if (!m || batch <= 0 || batch > MAX_BATCH) return 0;
  return frame_layout(body_model_info(m), batch, p2m_body_model_workspace_bytes(m, batch)).total;
}

int p2m_camera_frame_coords(const p2m_body_model_t* m, int flags, const float* pose, const float* betas,
                            const float* trans, const float* R, const float* t, const int32_t* extra_vertices,
                            int n_extra, float* verts, float* joints, int batch, void* workspace,
                            size_t workspace_bytes, p2m_stream_t stream) {
  if (!m || (flags & ~ALL_FLAGS) || batch <= 0 || batch > MAX_BATCH || !pose || !betas || !verts || !joints) {
    set_error("camera_frame_coords: bad argument (null model / pose / betas / output, unknown flags or batch out of "
              "[1, 2^24])");
    return P2M_ERR_INVALID;
  }
  const bool need_R = flags & (P2M_FRAME_ROTATE_ROOT | P2M_FRAME_H36M_COMPENSATE);
  const bool need_t = flags & (P2M_FRAME_LAYER_TRANS_T | P2M_FRAME_H36M_COMPENSATE | P2M_FRAME_ADD_T);
  const bool need_trans = flags & (P2M_FRAME_LAYER_TRANS | P2M_FRAME_H36M_COMPENSATE);
  const bool layer_trans = flags & (P2M_FRAME_LAYER_TRANS | P2M_FRAME_LAYER_TRANS_T);
  if ((need_R && !R) || (need_t && !t) || (need_trans && !trans) ||
      ((flags & P2M_FRAME_LAYER_TRANS) && (flags & P2M_FRAME_LAYER_TRANS_T)) ||
      ((flags & P2M_FRAME_ADD_T) && (flags & P2M_FRAME_H36M_COMPENSATE))) {
    set_error("camera_frame_coords: the flags need R / t / trans that are missing, or combine two translations");
    return P2M_ERR_INVALID;
  }
  const BodyModelInfo info = body_model_info(m);
  if (n_extra < 0 || n_extra > MAX_EXTRA || (n_extra > 0 && !extra_vertices)) {
    set_error("camera_frame_coords: n_extra must be in [0, 8] with extra_vertices given");
    return P2M_ERR_INVALID;
  }
  Extra ex{n_extra, {}};
  for (int i = 0; i < n_extra; ++i) {
    if (extra_vertices[i] < 0 || extra_vertices[i] >= info.V) {
      set_error("camera_frame_coords: extra vertex " + std::to_string(extra_vertices[i]) + " is not in [0, " +
                std::to_string(info.V) + ")");
      return P2M_ERR_INVALID;
    }
    ex.v[i] = extra_vertices[i];
  }
  const size_t body_bytes = p2m_body_model_workspace_bytes(m, batch);
  const FrameLayout l = frame_layout(info, batch, body_bytes);
  if (!workspace || workspace_bytes < l.total) {
    set_error("camera_frame_coords: workspace needs " + std::to_string(l.total) + " bytes");
    return P2M_ERR_WORKSPACE;
  }
  int dev = -1;
  P2M_TRY(arrays_device("camera_frame_coords", {pose, betas, trans, R, t, verts, joints, workspace}, &dev));
  if (dev != info.device) {
    set_error("camera_frame_coords: the data arrays are on device " + std::to_string(dev) + ", the body model on " +
              std::to_string(info.device));
    return P2M_ERR_INVALID;
  }
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  float* pose_o = reinterpret_cast<float*>(ws + l.pose);
  float* betas_o = reinterpret_cast<float*>(ws + l.betas);
  float* trans_o = layer_trans ? reinterpret_cast<float*>(ws + l.trans) : nullptr;
  float* verts_l = reinterpret_cast<float*>(ws + l.verts);
  float* joints_l = reinterpret_cast<float*>(ws + l.joints);
  k_frame_prep<<<(unsigned)((batch + PREP_WARPS - 1) / PREP_WARPS), PREP_WARPS * 32, 0, s>>>(
      flags, batch, info.J, info.S, info.model_betas, pose, betas, trans, R, t, pose_o, betas_o, trans_o);
  P2M_LAUNCH_OK();
  P2M_TRY(p2m_body_model_forward(m, pose_o, betas_o, P2M_BETAS_AS_GIVEN, trans_o, -1, verts_l, joints_l, batch,
                                 ws + l.body, body_bytes, stream));
  const dim3 grid((unsigned)((info.V + FIN_T - 1) / FIN_T), (unsigned)batch);
  k_frame_finish<<<grid, FIN_T, 0, s>>>(flags, info.V, info.n_out, ex, trans, R, t, verts_l, joints_l, verts, joints);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_h36m_regressors_create(const double* reg_h36m, const double* reg_coco, int n_vertex, int device,
                               p2m_h36m_regressors_t** out) {
  if (!out) {
    set_error("h36m_regressors_create: null output pointer");
    return P2M_ERR_INVALID;
  }
  *out = nullptr;
  if (!reg_h36m || !reg_coco || n_vertex < 1 || n_vertex > (1 << 22)) {
    set_error("h36m_regressors_create: null regressor or n_vertex out of [1, 2^22]");
    return P2M_ERR_INVALID;
  }
  std::vector<int> ptr(1, 0), idx;
  std::vector<double> val;
  for (int r = 0; r < NR; ++r) {
    const double* row = (r < NJ ? reg_h36m : reg_coco) + (size_t)(r % NJ) * n_vertex;
    for (int v = 0; v < n_vertex; ++v) {
      if (!std::isfinite(row[v])) {
        set_error("h36m_regressors_create: a regressor holds a non-finite value");
        return P2M_ERR_INVALID;
      }
      if (row[v] != 0.0) idx.push_back(v), val.push_back(row[v]);
    }
    ptr.push_back((int)idx.size());
  }
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev) {
    cudaGetLastError();
    set_error("h36m_regressors_create: device " + std::to_string(device) + " is not available");
    return P2M_ERR_NOGPU;
  }
  if (idx.empty()) idx.push_back(0), val.push_back(0.0);  // keep the pointers valid for all-zero regressors
  DeviceGuard guard(device);
  auto* h = new p2m_h36m_regressors();
  h->device = device, h->V = n_vertex;
  const auto fail = [&](cudaError_t e) {
    set_error(std::string("h36m_regressors_create: ") + cudaGetErrorString(e));
    p2m_h36m_regressors_destroy(h);
    return P2M_ERR_CUDA;
  };
  cudaError_t e;
  if ((e = cudaMalloc(&h->ptr, sizeof(int) * ptr.size())) != cudaSuccess) return fail(e);
  if ((e = cudaMalloc(&h->idx, sizeof(int) * idx.size())) != cudaSuccess) return fail(e);
  if ((e = cudaMalloc(&h->val, sizeof(double) * val.size())) != cudaSuccess) return fail(e);
  if ((e = cudaMemcpy(h->ptr, ptr.data(), sizeof(int) * ptr.size(), cudaMemcpyHostToDevice)) != cudaSuccess ||
      (e = cudaMemcpy(h->idx, idx.data(), sizeof(int) * idx.size(), cudaMemcpyHostToDevice)) != cudaSuccess ||
      (e = cudaMemcpy(h->val, val.data(), sizeof(double) * val.size(), cudaMemcpyHostToDevice)) != cudaSuccess)
    return fail(e);
  *out = h;
  return P2M_OK;
}

void p2m_h36m_regressors_destroy(p2m_h36m_regressors_t* h) {
  if (!h) return;
  {
    DeviceGuard guard(h->device);
    cudaFree(h->ptr);
    cudaFree(h->idx);
    cudaFree(h->val);
  }
  delete h;
}

int p2m_h36m_targets(const p2m_h36m_regressors_t* h, int input_joint_set, float fitting_thr, const float* mesh_cam,
                     const float* joint_cam, const float* f, const float* c, int batch, float* mesh, float* lift_pose3d,
                     float* reg_pose3d, float* mesh_valid, float* lift_pose3d_valid, float* reg_pose3d_valid,
                     float* joint_img, float* fitting_error, p2m_stream_t stream) {
  if (!joint_cam || !f || !c) {
    set_error("h36m_targets: joint_cam, f and c are required");
    return P2M_ERR_INVALID;
  }
  return p2m_sample_targets(h, P2M_DATASET_HUMAN36M, input_joint_set, fitting_thr, mesh_cam, joint_cam, f, c, nullptr,
                            0, nullptr, nullptr, nullptr, nullptr, nullptr, batch, mesh, lift_pose3d, reg_pose3d,
                            mesh_valid, lift_pose3d_valid, reg_pose3d_valid, nullptr, joint_img, fitting_error,
                            stream);
}

int p2m_sample_targets(const p2m_h36m_regressors_t* h, int dataset, int input_joint_set, float fitting_thr,
                       const float* mesh_cam, const float* joint_cam, const float* f, const float* c, const float* s,
                       int n_s, const float* t, const float* keypoints, const float* keypoints_valid, const float* rot,
                       const int32_t* flip, int batch, float* mesh, float* lift_pose3d, float* reg_pose3d,
                       float* mesh_valid, float* lift_pose3d_valid, float* reg_pose3d_valid, float* joint_valid,
                       float* joint_img, float* fitting_error, p2m_stream_t stream) {
  if (!h || (input_joint_set != P2M_JOINTS_HUMAN36 && input_joint_set != P2M_JOINTS_COCO) || batch <= 0 ||
      batch > MAX_BATCH || !mesh_cam || !mesh || !lift_pose3d || !reg_pose3d || !mesh_valid || !lift_pose3d_valid ||
      !reg_pose3d_valid || !joint_img || !fitting_error) {
    set_error("sample_targets: bad argument (null handle / array, unknown joint set or batch out of [1, 2^24])");
    return P2M_ERR_INVALID;
  }
  const bool need_fc = dataset == P2M_DATASET_HUMAN36M || dataset == P2M_DATASET_MUCO || dataset == P2M_DATASET_AMASS ||
                       dataset == P2M_DATASET_PW3D;
  if (dataset < P2M_DATASET_HUMAN36M || dataset > P2M_DATASET_PW3D ||
      (dataset == P2M_DATASET_HUMAN36M && !joint_cam) || (need_fc && (!f || !c)) ||
      (dataset == P2M_DATASET_COCO && (!s || (n_s != 1 && n_s != 2) || !t || !keypoints || !keypoints_valid))) {
    set_error("sample_targets: unknown dataset, or its inputs are missing (Human36M: joint_cam, f, c; COCO: s with "
              "n_s 1 or 2, t, keypoints, keypoints_valid; MuCo, AMASS, 3DPW: f, c)");
    return P2M_ERR_INVALID;
  }
  if (dataset == P2M_DATASET_PW3D && (input_joint_set != P2M_JOINTS_COCO || rot || flip)) {
    set_error("sample_targets: 3DPW takes the P2M_JOINTS_COCO set and no augmentation (rot and flip NULL)");
    return P2M_ERR_INVALID;
  }
  int dev = -1;
  P2M_TRY(arrays_device("sample_targets", {mesh_cam, joint_cam, f, c, s, t, keypoints, keypoints_valid, rot, flip,
                                           mesh, lift_pose3d, reg_pose3d, mesh_valid, lift_pose3d_valid,
                                           reg_pose3d_valid, joint_valid, joint_img, fitting_error}, &dev));
  if (dev != h->device) {
    set_error("sample_targets: the data arrays are on device " + std::to_string(dev) + ", the regressors on " +
              std::to_string(h->device));
    return P2M_ERR_INVALID;
  }
  DeviceGuard guard(dev);
  SampleArgs a{h->V, input_joint_set == P2M_JOINTS_COCO, batch, dataset, (double)fitting_thr, h->ptr, h->idx, h->val,
               mesh_cam, joint_cam, f, c, s, n_s, t, keypoints, keypoints_valid, rot, flip, mesh, lift_pose3d,
               reg_pose3d, mesh_valid, lift_pose3d_valid, reg_pose3d_valid, joint_valid, joint_img, fitting_error};
  k_sample_targets<<<(unsigned)batch, H36_T, 0, static_cast<cudaStream_t>(stream)>>>(a);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_layer_joint_targets(int dataset, const float* mesh_cam, const float* joint_cam, int n_vertex, int n_joint,
                            const float* f, const float* c, const float* rot, const int32_t* flip, int batch,
                            float* mesh, float* lift_pose3d, float* reg_pose3d, float* mesh_valid,
                            float* lift_pose3d_valid, float* reg_pose3d_valid, float* joint_valid, float* joint_img,
                            float* fitting_error, p2m_stream_t stream) {
  if (batch <= 0 || batch > MAX_BATCH || n_vertex < 1 || n_vertex > (1 << 22) || !mesh_cam || !joint_cam || !mesh ||
      !lift_pose3d || !reg_pose3d || !mesh_valid || !lift_pose3d_valid || !reg_pose3d_valid || !fitting_error) {
    set_error("layer_joint_targets: bad argument (null array, batch out of [1, 2^24] or n_vertex out of [1, 2^22])");
    return P2M_ERR_INVALID;
  }
  if (dataset == P2M_DATASET_SURREAL) {
    if (n_joint != SMPL_J || !f || !c || !joint_img) {
      set_error("layer_joint_targets: SURREAL takes SMPL's 24 joints, f, c and joint_img");
      return P2M_ERR_INVALID;
    }
  } else if (dataset == P2M_DATASET_FREIHAND) {
    if (n_joint != MANO_J || f || c || rot || flip || joint_img) {
      set_error("layer_joint_targets: FreiHAND takes MANO's 21 joints and no f, c, rot, flip or joint_img");
      return P2M_ERR_INVALID;
    }
  } else {
    set_error("layer_joint_targets: dataset must be P2M_DATASET_SURREAL or P2M_DATASET_FREIHAND");
    return P2M_ERR_INVALID;
  }
  int dev = -1;
  P2M_TRY(arrays_device("layer_joint_targets", {mesh_cam, joint_cam, f, c, rot, flip, mesh, lift_pose3d, reg_pose3d,
                                                mesh_valid, lift_pose3d_valid, reg_pose3d_valid, joint_valid,
                                                joint_img, fitting_error}, &dev));
  DeviceGuard guard(dev);
  LayerArgs a{dataset, n_vertex, n_joint, mesh_cam, joint_cam, f, c, rot, flip, mesh, lift_pose3d, reg_pose3d,
              mesh_valid, lift_pose3d_valid, reg_pose3d_valid, joint_valid, joint_img, fitting_error};
  k_layer_joint_targets<<<(unsigned)batch, LJ_T, 0, static_cast<cudaStream_t>(stream)>>>(a);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
