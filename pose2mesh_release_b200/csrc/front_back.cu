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
__global__ void __launch_bounds__(256) k_mesh_losses(const float* __restrict__ out, const float* __restrict__ gt,
                                                     const int* __restrict__ faces, int n_face, int n_vertex, int batch,
                                                     const float* __restrict__ g_scale, double* __restrict__ sums,
                                                     float* __restrict__ grad) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float ln = 0.f, le = 0.f;
  if (idx < (long long)batch * n_face) {
    const int f = (int)(idx % n_face);
    const long long b = idx / n_face;
    const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
    const float* ob = out + b * (long long)n_vertex * 3;
    const float* gb = gt + b * (long long)n_vertex * 3;
    const V3 o0 = ld3(ob + 3 * i0), o1 = ld3(ob + 3 * i1), o2 = ld3(ob + 3 * i2);
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
      float* gr = grad + b * (long long)n_vertex * 3;
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
      atomic_add3(gr + 3 * i0, V3{-g1.x - g2.x, -g1.y - g2.y, -g1.z - g2.z});
      atomic_add3(gr + 3 * i1, V3{g1.x - g3.x, g1.y - g3.y, g1.z - g3.z});
      atomic_add3(gr + 3 * i2, V3{g2.x + g3.x, g2.y + g3.y, g2.z + g3.z});
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
  const long long n = (long long)batch * n_face;
  k_mesh_losses<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(coord_out, coord_gt, faces, n_face, n_vertex, batch, grad_scale,
                                                            sums, grad_out);
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
