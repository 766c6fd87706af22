// Row f10 of SURVEY.md §8: the demo's mesh overlay (demo/renderer.py Renderer.render, demo/run.py:46-67) for many
// people over many images in one call.
//
// Per person p on image image_index[p], with orig_cam (sx, sy, tx, ty) and the reference's Rx(180°) flip folded in,
// a vertex (x, y, z) lands at pixel column u = W/2 (1 + sx (x + tx)), row v = H/2 (1 + sy (y + ty)), depth z (float32,
// in this order, no FMA contraction).  u, v are snapped to 1/256 px (U = rint(256 u), int64); pixel (i, r) samples
// (256 i + 128, 256 r + 128).  Coverage uses exact int64 edge functions with the top-left fill rule, so a pixel centre
// on an edge shared by two front faces belongs to exactly one of them; the screen-space signed area
// (u1-u0)(v2-v0) - (u2-u0)(v1-v0) must be < 0 (GL's counter-clockwise front faces seen through the top-down
// read-back); zero-area faces are dropped.  Depth is the edge-function-weighted mean of the vertex z in fp64, rounded
// once to float32; fragments with z outside [-1, 1] are clipped (the projection's P[2,2] = -1).
//
// Every fragment folds a 64-bit key into its pixel with atomicMin, so the result does not depend on launch order:
//   bits 63..48  0xFFFF - person   the later person wins wherever two people overlap (each has its own camera)
//   bits 47..16  order-preserving bits of float32 z (-0 stored as +0): nearer wins (GL_LESS)
//   bits 15..0   face              the lower face wins a depth tie (primitive order)
// The empty key is all ones.  The resolve pass shades the winning face flat: n = normalize((v1-v0) x (v2-v0)) in mesh
// coordinates, c_k = clamp(color_k (0.3 + (2.4/pi) max(0, -n_z)), 0, 1) (ambient 0.3 plus three 0.8 directional lights
// shining along the camera axis, Lambert only), stored as floor(255 c + 0.5); uncovered pixels copy the input image.
//
// Kernels: a memset of the key buffer; k_raster, one thread per (person, face) — a triangle whose clipped box holds
// more than LARGE_BOX pixels is shared by its whole warp; k_resolve, one thread per pixel.  No host synchronisation and
// no allocation: a call can be captured in a CUDA graph.
#include <cuda_runtime.h>

#include <cmath>
#include <string>

#include "p2m_internal.h"

namespace p2m {
namespace {

constexpr int RASTER_THREADS = 256;
constexpr int RESOLVE_THREADS = 256;
constexpr long long MAX_GRID = 1 << 16;
constexpr long long LARGE_BOX = 128;      // pixels of a triangle's clipped box above which its warp shares it
constexpr float GUARD_PX = 1048576.f;     // 2^20: |u|, |v| beyond this skip the triangle (int64 products < 2^58)
constexpr unsigned long long EMPTY = ~0ull;

struct Tri {
  long long u[3], v[3];  // snapped vertex positions, 1/256 px
  float z[3];
  unsigned long long tag;  // (0xFFFF - person) << 48 | face
  int img, i0, i1, r0, r1;  // image and clipped pixel box (inclusive)
};

// Project, snap, cull and clip face f of person p; false when the triangle yields no fragment to test.
__device__ __forceinline__ bool setup(const float* __restrict__ verts, int V, const int* __restrict__ faces,
                                      const float* __restrict__ cams, const int* __restrict__ image_index, int N,
                                      int H, int W, long long p, int f, Tri& t) {
  const float* cam = cams + p * 4;
  const float sx = cam[0], sy = cam[1], tx = cam[2], ty = cam[3];
  if (!(isfinite(sx) && isfinite(sy) && isfinite(tx) && isfinite(ty))) return false;
  const int img = image_index ? image_index[p] : 0;
  if (img < 0 || img >= N) return false;
  const float hw = __fmul_rn((float)W, 0.5f), hh = __fmul_rn((float)H, 0.5f);
  for (int k = 0; k < 3; ++k) {
    const int idx = faces[(long long)f * 3 + k];
    if (idx < 0 || idx >= V) return false;
    const float* x = verts + (p * V + idx) * 3;
    const float X = x[0], Y = x[1], Z = x[2];
    if (!(isfinite(X) && isfinite(Y) && isfinite(Z))) return false;
    const float u = __fmul_rn(hw, __fadd_rn(1.f, __fmul_rn(sx, __fadd_rn(X, tx))));
    const float v = __fmul_rn(hh, __fadd_rn(1.f, __fmul_rn(sy, __fadd_rn(Y, ty))));
    if (!(fabsf(u) <= GUARD_PX && fabsf(v) <= GUARD_PX)) return false;
    t.u[k] = __float2ll_rn(__fmul_rn(u, 256.f));
    t.v[k] = __float2ll_rn(__fmul_rn(v, 256.f));
    t.z[k] = Z;
  }
  const long long area = (t.u[1] - t.u[0]) * (t.v[2] - t.v[0]) - (t.u[2] - t.u[0]) * (t.v[1] - t.v[0]);
  if (area >= 0) return false;  // back-facing or degenerate
  const long long umin = min(t.u[0], min(t.u[1], t.u[2])), umax = max(t.u[0], max(t.u[1], t.u[2]));
  const long long vmin = min(t.v[0], min(t.v[1], t.v[2])), vmax = max(t.v[0], max(t.v[1], t.v[2]));
  // pixel centres 256 i + 128 inside [min, max]: arithmetic shifts floor
  const long long i0 = max((umin + 127) >> 8, 0ll), i1 = min((umax - 128) >> 8, (long long)W - 1);
  const long long r0 = max((vmin + 127) >> 8, 0ll), r1 = min((vmax - 128) >> 8, (long long)H - 1);
  if (i0 > i1 || r0 > r1) return false;
  t.i0 = (int)i0;
  t.i1 = (int)i1;
  t.r0 = (int)r0;
  t.r1 = (int)r1;
  t.img = img;
  t.tag = ((unsigned long long)(0xFFFF - p) << 48) | (unsigned long long)f;
  return true;
}

// Edge function of the edge opposite vertex e at pixel (i, r): w_e = base + i su + r sv, >= 0 inside; bias 1 for an
// edge that is not top-left (a pixel centre exactly on it is outside).
struct Edges {
  long long base[3], su[3], sv[3], bias[3];
  double den;  // w_0 + w_1 + w_2 = minus the signed area, exact
};

__device__ __forceinline__ void edges(const Tri& t, Edges& e) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = k == 2 ? 0 : k + 1, b = k == 0 ? 2 : (k == 1 ? 0 : 1);  // edges a1->a2, a2->a0, a0->a1
    const long long gu = t.v[b] - t.v[a], gv = t.u[a] - t.u[b];
    e.base[k] = gu * (128 - t.u[a]) + gv * (128 - t.v[a]);
    e.su[k] = gu * 256;
    e.sv[k] = gv * 256;
    e.bias[k] = (gu > 0 || (gu == 0 && gv > 0)) ? 0 : 1;
  }
  const long long area = (t.u[1] - t.u[0]) * (t.v[2] - t.v[0]) - (t.u[2] - t.u[0]) * (t.v[1] - t.v[0]);
  e.den = __ll2double_rn(-area);
}

__device__ __forceinline__ unsigned int z_order_bits(float z) {
  unsigned int b = __float_as_uint(z);
  if (b == 0x80000000u) b = 0u;  // -0 -> +0
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ void fragment(const Tri& t, const Edges& e, int i, int r, int H, int W,
                                         unsigned long long* __restrict__ keys) {
  long long w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = e.base[k] + (long long)i * e.su[k] + (long long)r * e.sv[k];
  if (w[0] < e.bias[0] || w[1] < e.bias[1] || w[2] < e.bias[2]) return;
  const double num = __dadd_rn(__dadd_rn(__dmul_rn(__ll2double_rn(w[0]), (double)t.z[0]),
                                         __dmul_rn(__ll2double_rn(w[1]), (double)t.z[1])),
                               __dmul_rn(__ll2double_rn(w[2]), (double)t.z[2]));
  const float z = __double2float_rn(__ddiv_rn(num, e.den));
  if (z < -1.f || z > 1.f) return;
  const unsigned long long key = t.tag | ((unsigned long long)z_order_bits(z) << 16);
  atomicMin(keys + ((long long)t.img * H + r) * W + i, key);
}

template <typename T>
__device__ __forceinline__ T shfl(T x, int src) {
  return __shfl_sync(0xffffffffu, x, src);
}

__global__ void __launch_bounds__(RASTER_THREADS) k_raster(const float* __restrict__ verts, int V,
                                                             const int* __restrict__ faces, int F,
                                                             const float* __restrict__ cams,
                                                             const int* __restrict__ image_index, long long P, int N,
                                                             int H, int W, unsigned long long* __restrict__ keys) {
  const int lane = threadIdx.x & 31;
  const long long total = P * F, stride = (long long)gridDim.x * RASTER_THREADS;
  // the loop runs per warp, so every lane of a warp takes part in the shared large-triangle loop
  for (long long base = (long long)blockIdx.x * RASTER_THREADS + (threadIdx.x & ~31); base < total; base += stride) {
    const long long id = base + lane;
    Tri t;
    bool ok = false;
    if (id < total) ok = setup(verts, V, faces, cams, image_index, N, H, W, id / F, (int)(id % F), t);
    const long long box = ok ? (long long)(t.i1 - t.i0 + 1) * (t.r1 - t.r0 + 1) : 0;
    if (ok && box <= LARGE_BOX) {
      Edges e;
      edges(t, e);
      for (int r = t.r0; r <= t.r1; ++r)
        for (int i = t.i0; i <= t.i1; ++i) fragment(t, e, i, r, H, W, keys);
    }
    unsigned large = __ballot_sync(0xffffffffu, box > LARGE_BOX);
    while (large) {
      const int src = __ffs(large) - 1;
      large &= large - 1;
      Tri s;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        s.u[k] = shfl(t.u[k], src);
        s.v[k] = shfl(t.v[k], src);
        s.z[k] = shfl(t.z[k], src);
      }
      s.tag = shfl(t.tag, src);
      s.img = shfl(t.img, src);
      s.i0 = shfl(t.i0, src);
      s.i1 = shfl(t.i1, src);
      s.r0 = shfl(t.r0, src);
      s.r1 = shfl(t.r1, src);
      Edges e;
      edges(s, e);
      const int bw = s.i1 - s.i0 + 1, n = bw * (s.r1 - s.r0 + 1);  // <= 2^28
      for (int q = lane; q < n; q += 32) fragment(s, e, s.i0 + q % bw, s.r0 + q / bw, H, W, keys);
    }
  }
}

__global__ void __launch_bounds__(RESOLVE_THREADS) k_resolve(const unsigned long long* __restrict__ keys,
                                                               long long n_pix, const float* __restrict__ verts, int V,
                                                               const int* __restrict__ faces,
                                                               const float* __restrict__ colors,
                                                               const unsigned char* images_in,
                                                               unsigned char* images_out, int* __restrict__ face_map,
                                                               int* __restrict__ person_map,
                                                               float* __restrict__ depth_map) {
  const float light = (float)(2.4 / M_PI);
  for (long long q = (long long)blockIdx.x * RESOLVE_THREADS + threadIdx.x; q < n_pix;
       q += (long long)gridDim.x * RESOLVE_THREADS) {
    const unsigned long long key = keys[q];
    if (key == EMPTY) {
      const unsigned char c0 = images_in[q * 3 + 0], c1 = images_in[q * 3 + 1], c2 = images_in[q * 3 + 2];
      images_out[q * 3 + 0] = c0;
      images_out[q * 3 + 1] = c1;
      images_out[q * 3 + 2] = c2;
      if (face_map) face_map[q] = -1;
      if (person_map) person_map[q] = -1;
      if (depth_map) depth_map[q] = __int_as_float(0x7fc00000);
      continue;
    }
    const long long p = 0xFFFF - (long long)(key >> 48);
    const int f = (int)(key & 0xFFFFull);
    const unsigned int zk = (unsigned int)(key >> 16);
    const float z = __uint_as_float((zk & 0x80000000u) ? (zk & 0x7FFFFFFFu) : ~zk);
    const float* a = verts + (p * V + faces[f * 3 + 0]) * 3;
    const float* b = verts + (p * V + faces[f * 3 + 1]) * 3;
    const float* c = verts + (p * V + faces[f * 3 + 2]) * 3;
    const float d1x = __fsub_rn(b[0], a[0]), d1y = __fsub_rn(b[1], a[1]), d1z = __fsub_rn(b[2], a[2]);
    const float d2x = __fsub_rn(c[0], a[0]), d2y = __fsub_rn(c[1], a[1]), d2z = __fsub_rn(c[2], a[2]);
    const float nx = __fsub_rn(__fmul_rn(d1y, d2z), __fmul_rn(d1z, d2y));
    const float ny = __fsub_rn(__fmul_rn(d1z, d2x), __fmul_rn(d1x, d2z));
    const float nz = __fsub_rn(__fmul_rn(d1x, d2y), __fmul_rn(d1y, d2x));
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
    const float lambert = fmaxf(0.f, -__fdiv_rn(nz, len));  // a NaN (zero-length normal) counts as 0
    const float intensity = __fadd_rn(0.3f, __fmul_rn(light, lambert));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float ck = fminf(fmaxf(__fmul_rn(colors[p * 3 + k], intensity), 0.f), 1.f);
      images_out[q * 3 + k] = (unsigned char)floorf(__fadd_rn(__fmul_rn(ck, 255.f), 0.5f));
    }
    if (face_map) face_map[q] = f;
    if (person_map) person_map[q] = (int)p;
    if (depth_map) depth_map[q] = z;
  }
}

}  // namespace
}  // namespace p2m

using namespace p2m;

extern "C" {

size_t p2m_render_workspace_bytes(int n_image, int height, int width) {
  if (n_image <= 0 || height <= 0 || width <= 0) return 0;
  return (size_t)n_image * (size_t)height * (size_t)width * sizeof(unsigned long long);
}

int p2m_render_meshes(const float* verts, int n_person, int n_vertex, const int32_t* faces, int n_face,
                      const float* cams, const float* colors, const int32_t* image_index, const uint8_t* images_in,
                      int n_image, int height, int width, uint8_t* images_out, int32_t* face_map, int32_t* person_map,
                      float* depth_map, void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  if (n_person < 0 || n_person > 65535 || n_face < 0 || n_face > 65535 || n_vertex < 0 || n_image <= 0 ||
      height <= 0 || height > 16384 || width <= 0 || width > 16384) {
    set_error("render_meshes: need 0 <= n_person <= 65535, 0 <= n_face <= 65535, n_vertex >= 0, n_image > 0 and "
              "0 < height, width <= 16384; got n_person = " + std::to_string(n_person) + ", n_face = " +
              std::to_string(n_face) + ", n_vertex = " + std::to_string(n_vertex) + ", n_image = " +
              std::to_string(n_image) + ", " + std::to_string(height) + " x " + std::to_string(width));
    return P2M_ERR_INVALID;
  }
  const bool draw = n_person > 0 && n_face > 0;
  if (!images_in || !images_out || !workspace || (draw && (!verts || !faces || !cams || !colors))) {
    set_error("render_meshes: null image, workspace or mesh array");
    return P2M_ERR_INVALID;
  }
  const size_t need = p2m_render_workspace_bytes(n_image, height, width);
  if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 8 != 0) {
    set_error("render_meshes: workspace of " + std::to_string(workspace_bytes) + " bytes (8-byte aligned) is too "
              "small; need " + std::to_string(need));
    return P2M_ERR_WORKSPACE;
  }
  int dev;
  P2M_TRY(arrays_device("render_meshes", {verts, faces, cams, colors, image_index, images_in, images_out, face_map,
                                          person_map, depth_map, workspace}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  unsigned long long* keys = static_cast<unsigned long long*>(workspace);
  const long long n_pix = (long long)n_image * height * width;
  P2M_CUDA_OK(cudaMemsetAsync(keys, 0xFF, need, s));
  if (draw) {
    k_raster<<<grid_for((long long)n_person * n_face, RASTER_THREADS, MAX_GRID), RASTER_THREADS, 0, s>>>(
        verts, n_vertex, faces, n_face, cams, image_index, n_person, n_image, height, width, keys);
    P2M_LAUNCH_OK();
  }
  k_resolve<<<grid_for(n_pix, RESOLVE_THREADS, MAX_GRID), RESOLVE_THREADS, 0, s>>>(
      keys, n_pix, verts, n_vertex, faces, colors, images_in, images_out, face_map, person_map, depth_map);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
