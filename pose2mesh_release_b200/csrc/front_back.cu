// Rows f2 and f3 of SURVEY.md §8: what runs in front of and behind the model (stateless entry points, DESIGN.md §4.3).
#include <cuda_runtime.h>

#include "p2m_internal.h"

using namespace p2m;
// =====================================================================================
// Row f2 of SURVEY.md §8: the steps either side of the model in the reference's callers.
//  * joint regression  joints = J_regressor @ vertices   (lib/core/base.py:131,204; demo/run.py:171)
//  * the demo's input normalisation, demo/run.py:150-158: tight box of the 2-D joints (coord_utils.py:21-39) ->
//    aspect-preserving box of the network input (process_bbox, :42-66) -> affine map into the input_w x input_h
//    patch (aug_utils.py:51-64,140-179 with rot = 0: a uniform scaling that maps the box centre to the patch
//    centre) -> divide by the patch size -> per-pose zero mean / unit std per coordinate.
// =====================================================================================
namespace {
__global__ void __launch_bounds__(256) k_regress_joints(const float* __restrict__ Jr, const float* __restrict__ verts,
                                                        int n_vertex, int chans, float* __restrict__ joints) {
  // one CTA per (joint, mesh); chans <= 4
  const int j = blockIdx.x, n_joint = gridDim.x;
  const long long b = blockIdx.y;
  const float* jr = Jr + (size_t)j * n_vertex;
  const float* vb = verts + b * (long long)n_vertex * chans;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int v = threadIdx.x; v < n_vertex; v += 256) {
    const float w = __ldg(jr + v);
    for (int c = 0; c < chans; ++c) acc[c] = fmaf(w, vb[(long long)v * chans + c], acc[c]);
  }
  __shared__ float red[4][8];
  for (int c = 0; c < 4; ++c) {
    float a = acc[c];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if ((threadIdx.x & 31) == 0) red[c][threadIdx.x >> 5] = a;
  }
  __syncthreads();
  if (threadIdx.x < chans) {
    float a = 0.f;
    for (int w = 0; w < 8; ++w) a += red[threadIdx.x][w];
    joints[(b * n_joint + j) * chans + threadIdx.x] = a;
  }
}

// d_verts = Jr^T d_joints: one thread per (vertex, mesh), joints in fixed order
__global__ void __launch_bounds__(256) k_regress_joints_bwd(const float* __restrict__ Jr, const float* __restrict__ d_joints,
                                                            int n_joint, int n_vertex, int chans,
                                                            float* __restrict__ d_verts) {
  const int v = blockIdx.x * 256 + threadIdx.x;
  const long long b = blockIdx.y;
  if (v >= n_vertex) return;
  const float* g = d_joints + b * n_joint * chans;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < n_joint; ++j) {
    const float w = __ldg(Jr + (size_t)j * n_vertex + v);
    for (int c = 0; c < chans; ++c) acc[c] = fmaf(w, g[j * chans + c], acc[c]);
  }
  for (int c = 0; c < chans; ++c) d_verts[(b * n_vertex + v) * chans + c] = acc[c];
}

// one warp per pose, lane = joint (n_joint <= 32)
__global__ void __launch_bounds__(128) k_normalize_pose2d(const float* __restrict__ px, int batch, int n_joint, int in_h,
                                                          int in_w, int truncate, float* __restrict__ out) {
  const int pose = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (pose >= batch) return;
  const bool on = lane < n_joint;
  const float x = on ? px[((long long)pose * n_joint + lane) * 2 + 0] : 0.f;
  const float y = on ? px[((long long)pose * n_joint + lane) * 2 + 1] : 0.f;
  const PoseCrop c = pose_crop(x, y, on, in_h, in_w);
  const float2 t = crop_point(c, x, y, in_h, in_w, truncate);
  normalize_crop(t.x, t.y, on, n_joint, in_h, in_w, out + (long long)pose * n_joint * 2);
}
}  // namespace

extern "C" {

int p2m_regress_joints(const float* joint_regressor, const float* vertices, float* joints, int batch, int n_joint,
                       int n_vertex, int chans, p2m_stream_t stream) {
  if (!joint_regressor || !vertices || !joints || batch <= 0 || n_joint <= 0 || n_vertex <= 0 || chans <= 0 || chans > 4 ||
      batch > 65535) {
    set_error("regress_joints: bad argument");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("regress_joints", {joint_regressor, vertices, joints}, &dev));
  DeviceGuard guard(dev);
  k_regress_joints<<<dim3(n_joint, batch), 256, 0, static_cast<cudaStream_t>(stream)>>>(joint_regressor, vertices,
                                                                                       n_vertex, chans, joints);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_regress_joints_backward(const float* joint_regressor, const float* d_joints, float* d_vertices, int batch,
                                int n_joint, int n_vertex, int chans, p2m_stream_t stream) {
  if (!joint_regressor || !d_joints || !d_vertices || batch <= 0 || n_joint <= 0 || n_vertex <= 0 || chans <= 0 ||
      chans > 4 || batch > 65535) {
    set_error("regress_joints_backward: bad argument");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("regress_joints_backward", {joint_regressor, d_joints, d_vertices}, &dev));
  DeviceGuard guard(dev);
  k_regress_joints_bwd<<<dim3((n_vertex + 255) / 256, batch), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      joint_regressor, d_joints, n_joint, n_vertex, chans, d_vertices);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_normalize_pose2d(const float* joints_px, float* pose2d, int batch, int n_joint, int input_h, int input_w,
                         int truncate_like_int_input, p2m_stream_t stream) {
  if (!joints_px || !pose2d || batch <= 0 || n_joint <= 0 || n_joint > 32 || input_h <= 0 || input_w <= 0) {
    set_error("normalize_pose2d: bad argument (at most 32 joints)");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("normalize_pose2d", {joints_px, pose2d}, &dev));
  DeviceGuard guard(dev);
  k_normalize_pose2d<<<(batch + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream)>>>(joints_px, batch, n_joint, input_h,
                                                                                   input_w, truncate_like_int_input, pose2d);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"

// =====================================================================================
// Row f3 of SURVEY.md §8: the mesh losses of lib/core/loss.py on the GPU, forward and backward in one pass.
//   NormalVectorLoss (:62-87)  mean over (B, 3 Nf) of |<normalize(edge_i(out)), normal(gt)>|
//   EdgeLengthLoss   (:90-114) mean over (B, 3 Nf) of | |edge_i(out)| - |edge_i(gt)| |
//   CoordLoss        (:10-23)  mean |pred * valid - target * valid|
// The reference rebuilds a LongTensor of the faces on the device in EVERY call (:68, :97) and materialises ~20
// [B, Nf, 3] temporaries; here one thread handles one (mesh, face): 18 loads, the two loss terms, and — when
// gradients are wanted — 9 atomic adds into d(coord_out).  F.normalize semantics: v / max(|v|, 1e-12).
// =====================================================================================
namespace {
struct V3 {
  float x, y, z;
};
__device__ __forceinline__ V3 sub3(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 scale3(V3 a, float s) { return V3{a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ V3 normalize3(V3 a, float* len) {
  const float n = sqrtf(dot3(a, a));
  *len = n;
  return scale3(a, 1.f / fmaxf(n, 1e-12f));
}
__device__ __forceinline__ V3 ld3(const float* p) { return V3{p[0], p[1], p[2]}; }
__device__ __forceinline__ void atomic_add3(float* p, V3 g) {
  atomicAdd(p + 0, g.x);
  atomicAdd(p + 1, g.y);
  atomicAdd(p + 2, g.z);
}

// sums[0] += sum of the 3 normal terms, sums[1] += sum of the 3 edge terms (fp64); grad (optional, zeroed by the
// caller) += g_normal * d(normal sum)/d(out) + g_edge * d(edge sum)/d(out) with g_* already divided by 3 B Nf.
// out and grad are [B, n_rows, 3] and vertex i is their row rows[i] (rows == nullptr: row i, n_rows == n_vertex);
// gt is [B, n_vertex, 3].
__global__ void __launch_bounds__(256) k_mesh_losses(const float* __restrict__ out, const float* __restrict__ gt,
                                                     const int* __restrict__ faces, const int* __restrict__ rows,
                                                     int n_rows, int n_face, int n_vertex, int batch,
                                                     const float* __restrict__ g_scale, double* __restrict__ sums,
                                                     float* __restrict__ grad) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float ln = 0.f, le = 0.f;
  if (idx < (long long)batch * n_face) {
    const int f = (int)(idx % n_face);
    const long long b = idx / n_face;
    const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
    const int w0 = rows ? rows[i0] : i0, w1 = rows ? rows[i1] : i1, w2 = rows ? rows[i2] : i2;
    const float* ob = out + b * (long long)n_rows * 3;
    const float* gb = gt + b * (long long)n_vertex * 3;
    const V3 o0 = ld3(ob + 3 * w0), o1 = ld3(ob + 3 * w1), o2 = ld3(ob + 3 * w2);
    const V3 t0 = ld3(gb + 3 * i0), t1 = ld3(gb + 3 * i1), t2 = ld3(gb + 3 * i2);
    // ---- normal-vector term
    float l1, l2, l3, lg;
    const V3 e1 = sub3(o1, o0), e2 = sub3(o2, o0), e3 = sub3(o2, o1);
    const V3 u1 = normalize3(e1, &l1), u2 = normalize3(e2, &l2), u3 = normalize3(e3, &l3);
    const V3 a = normalize3(sub3(t1, t0), &lg), c = normalize3(sub3(t2, t0), &lg);
    const V3 n = normalize3(V3{a.y * c.z - a.z * c.y, a.z * c.x - a.x * c.z, a.x * c.y - a.y * c.x}, &lg);
    const float c1 = dot3(u1, n), c2 = dot3(u2, n), c3 = dot3(u3, n);
    ln = fabsf(c1) + fabsf(c2) + fabsf(c3);
    // ---- edge-length term (reference edge order: (0,1), (0,2), (1,2))
    const float d1 = l1, d2 = l2, d3 = l3;  // |o0-o1|, |o0-o2|, |o1-o2|
    float q1, q2, q3;
    normalize3(sub3(t0, t1), &q1);
    normalize3(sub3(t0, t2), &q2);
    normalize3(sub3(t1, t2), &q3);
    const float r1 = d1 - q1, r2 = d2 - q2, r3 = d3 - q3;
    le = fabsf(r1) + fabsf(r2) + fabsf(r3);
    if (grad != nullptr) {
      const float gn = g_scale[0], ge = g_scale[1];
      float* gr = grad + b * (long long)n_rows * 3;
      // d|<u, n>| / de = sign(<u,n>) (n - u <u,n>) / |e|   (|e| > eps); sign(0) = 0 like torch.abs
      auto dcos = [&](V3 u, float cs, float len) {
        const float sg = (cs > 0.f) - (cs < 0.f);
        const float inv = (len > 1e-12f) ? sg / len : 0.f;
        return scale3(sub3(n, scale3(u, cs)), inv * gn);
      };
      // d| |e| - q | / de = sign(|e| - q) e / |e|
      auto dlen = [&](V3 u, float r, float len) {
        const float sg = (r > 0.f) - (r < 0.f);
        return scale3(u, (len > 0.f) ? sg * ge : 0.f);
      };
      V3 g1 = dcos(u1, c1, l1), g2 = dcos(u2, c2, l2), g3 = dcos(u3, c3, l3);       // w.r.t. e1, e2, e3
      const V3 h1 = dlen(u1, r1, l1), h2 = dlen(u2, r2, l2), h3 = dlen(u3, r3, l3);  // same edges (sign-symmetric)
      g1 = V3{g1.x + h1.x, g1.y + h1.y, g1.z + h1.z};
      g2 = V3{g2.x + h2.x, g2.y + h2.y, g2.z + h2.z};
      g3 = V3{g3.x + h3.x, g3.y + h3.y, g3.z + h3.z};
      // e1 = o1 - o0, e2 = o2 - o0, e3 = o2 - o1
      atomic_add3(gr + 3 * w0, V3{-g1.x - g2.x, -g1.y - g2.y, -g1.z - g2.z});
      atomic_add3(gr + 3 * w1, V3{g1.x - g3.x, g1.y - g3.y, g1.z - g3.z});
      atomic_add3(gr + 3 * w2, V3{g2.x + g3.x, g2.y + g3.y, g2.z + g3.z});
    }
  }
  __shared__ float red[2][8];
  for (int o = 16; o > 0; o >>= 1) {
    ln += __shfl_xor_sync(0xffffffffu, ln, o);
    le += __shfl_xor_sync(0xffffffffu, le, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = ln;
    red[1][threadIdx.x >> 5] = le;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];
    atomicAdd(sums + threadIdx.x, s);
  }
}

// CoordLoss: sums[0] += sum |p v - t v|; grad (optional) = g * sign(p v - t v) * v
__global__ void __launch_bounds__(256) k_coord_loss(const float* __restrict__ pred, const float* __restrict__ target,
                                                    const float* __restrict__ valid, long long n,
                                                    const float* __restrict__ g_scale, double* __restrict__ sums,
                                                    float* __restrict__ grad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float l = 0.f;
  if (i < n) {
    const float v = valid ? valid[i] : 1.f;
    const float d = pred[i] * v - target[i] * v;
    l = fabsf(d);
    if (grad != nullptr) grad[i] = g_scale[0] * (float)((d > 0.f) - (d < 0.f)) * v;
  }
  __shared__ float red[8];
  for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += red[w];
    atomicAdd(sums, s);
  }
}

int launch_mesh_losses(const float* out, const float* gt, const int32_t* faces, const int32_t* rows, int n_rows,
                       int batch, int n_vertex, int n_face, const float* g_scale, double* sums, float* grad,
                       cudaStream_t s) {
  const long long n = (long long)batch * n_face;
  k_mesh_losses<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(out, gt, faces, rows, n_rows, n_face, n_vertex, batch,
                                                            g_scale, sums, grad);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// ---- the Trainer's objective (p2m_pose2mesh_loss).  scratch = double partials[B][4] (vertex, joint and lift L1 sums
// of mesh b, then 0), followed by one LossTail.
constexpr int MAXJ = P2M_POSE2MESH_MAX_REG_JOINT;
struct LossTail {
  double face_sums[2];   // p2m_mesh_losses' normal and edge sums
  float face_scale[2];   // the face kernel's grad_scale in the backward
  unsigned ticket;       // CTAs of k_pose2mesh_loss that have written their partials; reset by the last one
  unsigned pad;
};
static_assert(sizeof(LossTail) == 32, "scratch holds 32 (batch + 1) bytes");
__host__ __device__ inline LossTail* loss_tail(void* scratch, int batch) {
  return reinterpret_cast<LossTail*>(static_cast<char*>(scratch) + 32 * (size_t)batch);
}
__device__ __forceinline__ float sgnf(float x) { return (float)((x > 0.f) - (x < 0.f)); }  // sign(0) = 0 like torch
template <typename T>
__device__ __forceinline__ T warp_sum(T a) {
  for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  return a;
}

// One CTA per mesh: reads each real vertex's padded row once for the masked vertex L1 and the joint regression,
// then the joint and lift L1 of that mesh; the last CTA to finish sums the partials in mesh order and forms the terms.
__global__ void __launch_bounds__(256) k_pose2mesh_loss(const p2m_pose2mesh_loss_args_t a) {
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nv = a.n_vertex, nj = a.n_reg_joint, nl = a.n_lift_joint;
  const float* xb = a.cam_mesh + (size_t)b * a.n_padded * 3;
  const float* gb = a.gt_mesh + (size_t)b * nv * 3;
  const float* mb = a.mesh_valid + (size_t)b * nv;
  float acc[MAXJ][3];
#pragma unroll
  for (int j = 0; j < MAXJ; ++j) acc[j][0] = acc[j][1] = acc[j][2] = 0.f;
  float l1 = 0.f;
  for (int v = tid; v < nv; v += 256) {
    const int r = a.perm_reverse[v];
    const float x0 = xb[3 * r], x1 = xb[3 * r + 1], x2 = xb[3 * r + 2], m = mb[v];
    l1 += fabsf(x0 * m - gb[3 * v] * m) + fabsf(x1 * m - gb[3 * v + 1] * m) + fabsf(x2 * m - gb[3 * v + 2] * m);
#pragma unroll
    for (int j = 0; j < MAXJ; ++j) {
      if (j < nj) {
        const float w = __ldg(a.joint_regressor + (size_t)j * nv + v);
        acc[j][0] = fmaf(w, x0, acc[j][0]);
        acc[j][1] = fmaf(w, x1, acc[j][1]);
        acc[j][2] = fmaf(w, x2, acc[j][2]);
      }
    }
  }
  __shared__ float red[MAXJ * 3 + 1][8];
  __shared__ float pose[MAXJ * 3];
  __shared__ double part[3];
  __shared__ bool last;
#pragma unroll
  for (int j = 0; j < MAXJ; ++j) {
    if (j < nj) {
      for (int c = 0; c < 3; ++c) {
        const float s = warp_sum(acc[j][c]);
        if (lane == 0) red[3 * j + c][warp] = s;
      }
    }
  }
  l1 = warp_sum(l1);
  if (lane == 0) red[MAXJ * 3][warp] = l1;
  __syncthreads();
  if (tid < nj * 3) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[tid][w];
    pose[tid] = 1000.f * s;
    a.pred_pose[(size_t)b * nj * 3 + tid] = 1000.f * s;
  }
  __syncthreads();
  if (warp < 2) {  // warp 0: the regressed joints against gt_reg3dpose; warp 1: the lifted pose against gt_lift3dpose
    const int n = warp == 0 ? nj : nl;
    const float* p = warp == 0 ? pose : a.lift_pose + (size_t)b * nl * 3;
    const float* t = (warp == 0 ? a.gt_reg3dpose : a.gt_lift3dpose) + (size_t)b * n * 3;
    const float* mv = (warp == 0 ? a.reg3dpose_valid : a.lift3dpose_valid) + (size_t)b * n;
    float s = 0.f;
    for (int i = lane; i < 3 * n; i += 32) {
      const float m = mv[i / 3];
      s += fabsf(p[i] * m - t[i] * m);
    }
    s = warp_sum(s);
    if (lane == 0) part[1 + warp] = s;
    if (tid == 0) {
      double v = 0.0;
      for (int w = 0; w < 8; ++w) v += red[MAXJ * 3][w];
      part[0] = v;
    }
  }
  __syncthreads();
  LossTail* tail = loss_tail(a.scratch, a.batch);
  if (tid == 0) {
    double* p = static_cast<double*>(a.scratch) + 4 * (size_t)b;
    p[0] = part[0];
    p[1] = part[1];
    p[2] = part[2];
    p[3] = 0.0;
    __threadfence();
    last = atomicAdd(&tail->ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (warp < 3) {
    double s = 0.0;
    for (int i = lane; i < a.batch; i += 32) s += __ldcg(static_cast<const double*>(a.scratch) + 4 * (size_t)i + warp);
    s = warp_sum(s);
    if (lane == 0) part[warp] = s;
  }
  __syncthreads();
  if (tid == 0) {
    const double B = a.batch, nfs = 3.0 * B * a.n_face;
    double t[5];
    t[0] = part[0] / (3.0 * B * nv);
    t[1] = a.weights[0] * (tail->face_sums[0] / nfs);
    t[2] = a.edge[0] != 0.f ? a.weights[1] * (tail->face_sums[1] / nfs) : 0.0;
    t[3] = a.weights[2] * (part[1] / (3.0 * B * nj));
    t[4] = a.weights[2] * (part[2] / (3.0 * B * nl));
    for (int i = 0; i < 5; ++i) a.terms[i] = (float)t[i];
    a.loss[0] = (float)(t[0] + t[1] + t[2] + t[3] + t[4]);
    tail->ticket = 0;
  }
}

// Backward launch 1: zero d_cam_mesh; the face kernel's sums and gradient scales.
__global__ void __launch_bounds__(256) k_pose2mesh_loss_bwd_prep(const p2m_pose2mesh_loss_args_t a) {
  const long long n = (long long)a.batch * a.n_padded * 3;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    a.d_cam_mesh[i] = 0.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    LossTail* t = loss_tail(a.scratch, a.batch);
    const double g = a.grad_loss[0], nfs = 3.0 * a.batch * a.n_face;
    t->face_sums[0] = t->face_sums[1] = 0.0;
    t->face_scale[0] = (float)(g * a.weights[0] / nfs);
    t->face_scale[1] = a.edge[0] != 0.f ? (float)(g * a.weights[1] / nfs) : 0.f;
  }
}

// Backward launch 3: one thread per (vertex, mesh) adds the vertex L1 and the joint terms into its padded row
// (each row has one owner: no atomics); the first column of CTAs writes d_lift_pose.
__global__ void __launch_bounds__(256) k_pose2mesh_loss_bwd(const p2m_pose2mesh_loss_args_t a) {
  const int b = blockIdx.y, tid = threadIdx.x;
  const int nv = a.n_vertex, nj = a.n_reg_joint, nl = a.n_lift_joint;
  const double g = a.grad_loss[0];
  __shared__ float g4[MAXJ * 3];  // d loss / d (J x), times 1000
  if (tid < nj * 3) {
    const float s4 = (float)(g * a.weights[2] / (3.0 * a.batch * nj));
    const float m = a.reg3dpose_valid[(size_t)b * nj + tid / 3];
    const size_t i = (size_t)b * nj * 3 + tid;
    g4[tid] = 1000.f * (s4 * sgnf(a.pred_pose[i] * m - a.gt_reg3dpose[i] * m) * m);
  }
  __syncthreads();
  const int v = blockIdx.x * 256 + tid;
  if (v < nv) {
    const float s1 = (float)(g / (3.0 * a.batch * nv));
    const size_t row = ((size_t)b * a.n_padded + a.perm_reverse[v]) * 3;
    const float* x = a.cam_mesh + row;
    const float* t = a.gt_mesh + ((size_t)b * nv + v) * 3;
    const float m = a.mesh_valid[(size_t)b * nv + v];
    float d[3];
    for (int c = 0; c < 3; ++c) d[c] = s1 * sgnf(x[c] * m - t[c] * m) * m;
    for (int j = 0; j < nj; ++j) {
      const float w = __ldg(a.joint_regressor + (size_t)j * nv + v);
      for (int c = 0; c < 3; ++c) d[c] = fmaf(w, g4[3 * j + c], d[c]);
    }
    for (int c = 0; c < 3; ++c) a.d_cam_mesh[row + c] += d[c];
  }
  if (blockIdx.x == 0) {
    const float s5 = (float)(g * a.weights[2] / (3.0 * a.batch * nl));
    for (int i = tid; i < 3 * nl; i += 256) {
      const size_t k = (size_t)b * nl * 3 + i;
      const float m = a.lift3dpose_valid[(size_t)b * nl + i / 3];
      a.d_lift_pose[k] = s5 * sgnf(a.lift_pose[k] * m - a.gt_lift3dpose[k] * m) * m;
    }
  }
}

int pose2mesh_loss_device(const char* where, const p2m_pose2mesh_loss_args_t* a, bool backward, int* dev) {
  const bool ok = a && a->batch > 0 && a->batch <= 65535 && a->n_vertex > 0 && a->n_padded >= a->n_vertex &&
                  a->n_face > 0 && a->n_reg_joint > 0 && a->n_reg_joint <= MAXJ && a->n_lift_joint > 0 &&
                  a->cam_mesh && a->lift_pose && a->gt_mesh && a->gt_reg3dpose && a->gt_lift3dpose && a->mesh_valid &&
                  a->reg3dpose_valid && a->lift3dpose_valid && a->faces && a->joint_regressor && a->perm_reverse &&
                  a->weights && a->edge && a->pred_pose && a->scratch &&
                  (backward ? (a->grad_loss && a->d_cam_mesh && a->d_lift_pose) : (a->loss && a->terms));
  if (!ok) {
    set_error(std::string(where) + ": bad argument (batch <= 65535, n_reg_joint <= " + std::to_string(MAXJ) +
              ", n_vertex <= n_padded, every array of the call given)");
    return P2M_ERR_INVALID;
  }
  return arrays_device(where, {a->cam_mesh, a->lift_pose, a->gt_mesh, a->gt_reg3dpose, a->gt_lift3dpose, a->mesh_valid,
                               a->reg3dpose_valid, a->lift3dpose_valid, a->faces, a->joint_regressor, a->perm_reverse,
                               a->weights, a->edge, a->pred_pose, a->scratch, a->loss, a->terms, a->grad_loss,
                               a->d_cam_mesh, a->d_lift_pose},
                       dev);
}
}  // namespace

extern "C" {

int p2m_mesh_losses(const float* coord_out, const float* coord_gt, const int32_t* faces, int batch, int n_vertex,
                    int n_face, const float* grad_scale, double* sums, float* grad_out, p2m_stream_t stream) {
  if (!coord_out || !coord_gt || !faces || !sums || batch <= 0 || n_vertex <= 0 || n_face <= 0 ||
      (grad_out != nullptr && grad_scale == nullptr)) {
    set_error("mesh_losses: bad argument");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("mesh_losses", {coord_out, coord_gt, faces, grad_scale, sums, grad_out}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  P2M_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), s));
  if (grad_out) P2M_CUDA_OK(cudaMemsetAsync(grad_out, 0, sizeof(float) * 3 * (size_t)batch * n_vertex, s));
  return launch_mesh_losses(coord_out, coord_gt, faces, nullptr, n_vertex, batch, n_vertex, n_face, grad_scale, sums,
                            grad_out, s);
}

int p2m_pose2mesh_loss(const p2m_pose2mesh_loss_args_t* a, p2m_stream_t stream) {
  int dev;
  P2M_TRY(pose2mesh_loss_device("pose2mesh_loss", a, false, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  LossTail* tail = loss_tail(a->scratch, a->batch);
  P2M_CUDA_OK(cudaMemsetAsync(tail, 0, sizeof(LossTail), s));
  P2M_TRY(launch_mesh_losses(a->cam_mesh, a->gt_mesh, a->faces, a->perm_reverse, a->n_padded, a->batch, a->n_vertex,
                             a->n_face, nullptr, tail->face_sums, nullptr, s));
  k_pose2mesh_loss<<<a->batch, 256, 0, s>>>(*a);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_pose2mesh_loss_backward(const p2m_pose2mesh_loss_args_t* a, p2m_stream_t stream) {
  int dev;
  P2M_TRY(pose2mesh_loss_device("pose2mesh_loss_backward", a, true, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  LossTail* tail = loss_tail(a->scratch, a->batch);
  const long long n = (long long)a->batch * a->n_padded * 3;
  k_pose2mesh_loss_bwd_prep<<<(unsigned)std::min<long long>((n + 255) / 256, 4096), 256, 0, s>>>(*a);
  P2M_LAUNCH_OK();
  P2M_TRY(launch_mesh_losses(a->cam_mesh, a->gt_mesh, a->faces, a->perm_reverse, a->n_padded, a->batch, a->n_vertex,
                             a->n_face, tail->face_scale, tail->face_sums, a->d_cam_mesh, s));
  k_pose2mesh_loss_bwd<<<dim3((a->n_vertex + 255) / 256, a->batch), 256, 0, s>>>(*a);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_coord_loss(const float* pred, const float* target, const float* valid, int64_t n, const float* grad_scale,
                   double* sum, float* grad_out, p2m_stream_t stream) {
  if (!pred || !target || !sum || n <= 0 || (grad_out != nullptr && grad_scale == nullptr)) {
    set_error("coord_loss: bad argument");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("coord_loss", {pred, target, valid, grad_scale, sum, grad_out}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  P2M_CUDA_OK(cudaMemsetAsync(sum, 0, sizeof(double), s));
  k_coord_loss<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(pred, target, valid, n, grad_scale, sum, grad_out);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
