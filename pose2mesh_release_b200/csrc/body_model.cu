// Row f6 of SURVEY.md §8: the body-model forward of the two configurations Pose2Mesh builds its target meshes with,
// for a whole batch on the GPU.
//  * SMPL  smplpytorch/smplpytorch/pytorch/smpl_layer.py:65-158  (SMPL_Layer.forward)
//  * MANO  manopth/manopth/manolayer.py  (ManoLayer.forward with use_pca=False and axis-angle root / joints, as
//          lib/_mano.py:37 builds it)
// fp32 on the CUDA cores, the reference's arithmetic.  Three launches per forward:
//  1. k_batch_flags  the batch-wide tests of the reference (betas all zero, trans all zero): one partial flag word per
//                    CTA (up to 128 CTAs), OR-ed by every k_pose warp
//  2. k_pose         one warp per sample: Rodrigues, pose map, shaped joints, kinematic chain, relative transforms A_j,
//                    the sample's blend coefficients and its kinematic output joints
//  3. k_lbs          a 128-vertex tile of 16 samples per CTA: v_posed = v_template + [shapedirs | posedirs] c, then
//                    linear blend skinning over the vertex's non-zero weights
// No atomics and fixed summation orders: a sample's result is bitwise independent of its batch position and of the
// batch size; nothing is read back to the host, so a forward can be captured in a CUDA graph.
// The backward (p2m_body_model_backward: the VJP with respect to pose, betas and trans) keeps the same properties in
// five launches: k_batch_flags, k_pose, k_lbs_bwd, k_dcoef, k_pose_bwd (see the backward section below).
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "p2m_internal.h"

namespace p2m {
namespace {

constexpr int MAX_J = 64;
constexpr int MAX_S = 512;
constexpr int MAX_K = MAX_S + 9 * (MAX_J - 1);
constexpr int MAX_OUT = 1024;
constexpr int MAX_BATCH = 1 << 24;
constexpr int FLAG_T = 256;            // threads per k_batch_flags CTA
constexpr int MAX_FLAG_BLOCKS = 128;   // k_batch_flags CTAs (= partial flag words)

constexpr int LBS_T = 256;             // threads per k_lbs CTA
constexpr int NV = 128;                // vertices per tile (one per thread, two sample octets)
constexpr int GS = 16;                 // samples per group: each staged basis chunk serves 16 samples
constexpr int KC = 16;                 // basis rows per staged chunk
constexpr int TILE_COLS = 3 * NV;      // basis columns per tile
constexpr int CHUNK_FLOATS = KC * TILE_COLS;

inline size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// Device-side view of the handle, passed by value to the kernels.
struct ModelDev {
  int V, J, S, K, Kp, ld, n_out;
  float scale;
  const float* basis;     // [Kp, ld]  K-major: row k < S is shapedirs[:, :, k], row S + p is posedirs[:, :, p]
  const float* vtemp;     // [ld]
  const float* jtemp;     // [J, 3]     J_regressor v_template
  const float* jshape;    // [J, 3, S]  J_regressor shapedirs
  const float* mbetas;    // [S]
  const float* pmean;     // [3 (J - 1)] or null
  const int* parents;     // [J]
  const int* jmap;        // [n_out]
  const int* w_ptr;       // [V + 1]  CSR of the non-zero skinning weights
  const int* w_idx;
  const float* w_val;
  const int* vj_out;      // [n_vj] output joints that are vertices: joints[vj_out[i]] = verts[vj_vert[i]]
  const int* vj_vert;
  int n_vj;
};

struct Work {
  int* flags;     // [n_flag_blocks]  per CTA of k_batch_flags: bit 0 betas non-zero, bit 1 trans non-zero
  int n_flag_blocks;
  float* A;       // [B, J, 12]  the top three rows of A_j = G_j - pack(G_j [J_j; 0])
  float* coef;    // [B, Kp]  [betas | pose_map | 0]
  float* offs;    // [B, 3]   + trans, - centre or 0
};

// batch_rodrigues (rodrigues_layer.py): angle = |theta + 1e-8|, axis = theta / angle, half-angle quaternion, quat2mat
// with its renormalisation.  A zero rotation gives exactly the identity.
__device__ __forceinline__ void rodrigues(const float* th, float* R) {
  const float a0 = th[0] + 1e-8f, a1 = th[1] + 1e-8f, a2 = th[2] + 1e-8f;
  const float angle = sqrtf(a0 * a0 + a1 * a1 + a2 * a2);
  const float half = angle * 0.5f;
  const float c = cosf(half), s = sinf(half);
  float w = c, x = s * (th[0] / angle), y = s * (th[1] / angle), z = s * (th[2] / angle);
  const float n = sqrtf(w * w + x * x + y * y + z * z);
  w = w / n, x = x / n, y = y / n, z = z / n;
  const float w2 = w * w, x2 = x * x, y2 = y * y, z2 = z * z;
  const float wx = w * x, wy = w * y, wz = w * z, xy = x * y, xz = x * z, yz = y * z;
  R[0] = w2 + x2 - y2 - z2, R[1] = 2.f * xy - 2.f * wz, R[2] = 2.f * wy + 2.f * xz;
  R[3] = 2.f * wz + 2.f * xy, R[4] = w2 - x2 + y2 - z2, R[5] = 2.f * yz - 2.f * wx;
  R[6] = 2.f * xz - 2.f * wy, R[7] = 2.f * wx + 2.f * yz, R[8] = w2 - x2 - y2 + z2;
}

// One vertex of one sample: T = sum_j w_vj A_j over the vertex's non-zero weights (ascending j), then T [x; 1].
// k_pose (vertex centre) and k_lbs share it, so the two agree bit for bit.
__device__ __forceinline__ void skin_point(const ModelDev& m, const float* A, int v, const float x[3], float out[3]) {
  float T[12];
#pragma unroll
  for (int q = 0; q < 12; ++q) T[q] = 0.f;
  for (int e = m.w_ptr[v]; e < m.w_ptr[v + 1]; ++e) {
    const float w = m.w_val[e];
    const float* a = A + 12 * m.w_idx[e];
#pragma unroll
    for (int q = 0; q < 12; ++q) T[q] = fmaf(w, a[q], T[q]);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = fmaf(T[4 * c + 2], x[2], fmaf(T[4 * c + 1], x[1], T[4 * c] * x[0])) + T[4 * c + 3];
}

// The reference's bool(torch.norm(x) == 0) tests, decided on the device: CTA c writes flags[c] = (any betas value
// != 0 in its grid-stride share) | (the same for trans) << 1, NaN counting as non-zero.  k_pose ORs the words.
__global__ void __launch_bounds__(FLAG_T) k_batch_flags(const float* __restrict__ betas, long long n_betas,
                                                        const float* __restrict__ trans, long long n_trans,
                                                        int* __restrict__ flags) {
  const long long stride = (long long)gridDim.x * FLAG_T, i0 = (long long)blockIdx.x * FLAG_T + threadIdx.x;
  int fb = 0, ft = 0;
  for (long long i = i0; i < n_betas; i += stride) fb |= !(betas[i] == 0.f);
  for (long long i = i0; i < n_trans; i += stride) ft |= !(trans[i] == 0.f);
  fb = __syncthreads_or(fb);
  ft = __syncthreads_or(ft);
  if (threadIdx.x == 0) flags[blockIdx.x] = fb | (ft << 1);
}

// One warp per sample.
__global__ void __launch_bounds__(32) k_pose(ModelDev m, const float* __restrict__ pose,
                                             const float* __restrict__ betas, int betas_rule,
                                             const float* __restrict__ trans, int center_idx,
                                             float* __restrict__ joints, Work w) {
  __shared__ float th[3 * MAX_J], R[MAX_J][9], jp[MAX_J][3], G[MAX_J][12], As[MAX_J * 12], beta[MAX_S], cf[MAX_K + 16];
  __shared__ float off[3];
  const int b = blockIdx.x, lane = threadIdx.x, J = m.J, S = m.S;
  int flag = 0;
  for (int i = lane; i < w.n_flag_blocks; i += 32) flag |= w.flags[i];
  flag = __reduce_or_sync(0xffffffffu, flag);
  const bool given = betas != nullptr && (betas_rule == P2M_BETAS_AS_GIVEN || (flag & 1));
  for (int s = lane; s < S; s += 32) beta[s] = given ? betas[(long long)b * S + s] : m.mbetas[s];
  for (int i = lane; i < 3 * J; i += 32) {
    float x = pose[(long long)b * 3 * J + i];
    if (m.pmean && i >= 3) x = m.pmean[i - 3] + x;  // ManoLayer: th_hands_mean + th_full_hand_pose
    th[i] = x;
  }
  __syncwarp();
  for (int j = lane; j < J; j += 32) rodrigues(th + 3 * j, R[j]);
  // shaped joints J_j = J_regressor (v_template + shapedirs beta), with both products taken at creation
  for (int e = lane; e < 3 * J; e += 32) {
    float acc = m.jtemp[e];
    for (int s = 0; s < S; ++s) acc = fmaf(m.jshape[(long long)e * S + s], beta[s], acc);
    jp[e / 3][e % 3] = acc;
  }
  __syncwarp();
  // blend coefficients [beta | R_j - I for j >= 1 | 0 padding]
  for (int k = lane; k < m.Kp; k += 32) {
    float c = 0.f;
    if (k < S) {
      c = beta[k];
    } else if (k < m.K) {
      const int p = k - S, q = p % 9;
      c = R[1 + p / 9][q] - ((q == 0 || q == 4 || q == 8) ? 1.f : 0.f);
    }
    cf[k] = c;
    w.coef[(long long)b * m.Kp + k] = c;
  }
  // kinematic chain in parent order: G_0 = [R_0 | J_0], G_j = G_parent [R_j | J_j - J_parent]
  const int r = lane >> 2, c = lane & 3;
  if (lane < 12) G[0][lane] = c < 3 ? R[0][3 * r + c] : jp[0][r];
  __syncwarp();
  for (int j = 1; j < J; ++j) {
    const int p = m.parents[j];
    if (lane < 12) {
      const float* g = G[p] + 4 * r;
      float l0, l1, l2;
      if (c < 3) {
        l0 = R[j][c], l1 = R[j][3 + c], l2 = R[j][6 + c];
      } else {
        l0 = jp[j][0] - jp[p][0], l1 = jp[j][1] - jp[p][1], l2 = jp[j][2] - jp[p][2];
      }
      float v = fmaf(g[2], l2, fmaf(g[1], l1, g[0] * l0));
      if (c == 3) v = v + g[3];
      G[j][lane] = v;
    }
    __syncwarp();
  }
  for (int e = lane; e < 12 * J; e += 32) {
    const int j = e / 12, q = e % 12, rr = q >> 2;
    float a = G[j][q];
    if ((q & 3) == 3) {
      const float* g = G[j] + 4 * rr;
      a = a - fmaf(g[2], jp[j][2], fmaf(g[1], jp[j][1], g[0] * jp[j][0]));
    }
    As[e] = a;
    w.A[(long long)b * J * 12 + e] = a;
  }
  __syncwarp();
  // the per-sample offset: + trans when the batch's trans is not all zero, else - the centre joint (if any)
  if (lane == 0) {
    float o[3] = {0.f, 0.f, 0.f};
    if (trans != nullptr && (flag & 2)) {
      for (int q = 0; q < 3; ++q) o[q] = trans[(long long)b * 3 + q];
    } else if (center_idx >= 0) {
      const int e = m.jmap[center_idx];
      if (e >= 0) {
        for (int q = 0; q < 3; ++q) o[q] = -G[e][4 * q + 3];
      } else {  // a vertex joint: the same v_posed chain and skinning as k_lbs
        const int v = -1 - e;
        float x[3], y[3];
        for (int q = 0; q < 3; ++q) {
          float acc = m.vtemp[3 * v + q];
          for (int k = 0; k < m.Kp; ++k) acc = fmaf(m.basis[(long long)k * m.ld + 3 * v + q], cf[k], acc);
          x[q] = acc;
        }
        skin_point(m, As, v, x, y);
        for (int q = 0; q < 3; ++q) o[q] = -y[q];
      }
    }
    for (int q = 0; q < 3; ++q) {
      off[q] = o[q];
      w.offs[(long long)b * 3 + q] = o[q];
    }
  }
  __syncwarp();
  for (int e = lane; e < 3 * m.n_out; e += 32) {
    const int o = e / 3, q = e % 3, jj = m.jmap[o];
    if (jj >= 0) joints[(long long)b * 3 * m.n_out + e] = (G[jj][4 * q + 3] + off[q]) * m.scale;
  }
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;\n" ::); }

// grid (sample groups, vertex tiles).  Thread t: vertex t % 128 of the tile, samples 8 (t / 128) .. + 7 of the group.
// The basis tile [Kp, 384] streams through shared memory in 16-row chunks (cp.async, double-buffered); each chunk
// serves all 16 samples of the group.  The group's coefficient rows (transposed, [Kp][16]), A matrices and offsets
// sit in shared memory for the whole CTA.
__global__ void __launch_bounds__(LBS_T) k_lbs(ModelDev m, int batch, Work w, float* __restrict__ verts,
                                               float* __restrict__ joints) {
  extern __shared__ float4 smem4[];
  float* sB = reinterpret_cast<float*>(smem4);     // [2][KC][384]
  float* sC = sB + 2 * CHUNK_FLOATS;               // [Kp][16]
  float* sA = sC + m.Kp * GS;                      // [16][J * 12]
  float* sO = sA + GS * m.J * 12;                  // [16][3]
  const int tid = threadIdx.x;
  const int g0 = blockIdx.x * GS, tile = blockIdx.y;
  const int n_chunk = m.Kp / KC;
  const float* btile = m.basis + (long long)tile * TILE_COLS;

  auto load_chunk = [&](int ch, int stage) {
    float* dst = sB + stage * CHUNK_FLOATS;
    const float* src = btile + (long long)ch * KC * m.ld;
    for (int i = tid; i < CHUNK_FLOATS / 4; i += LBS_T) {
      const int row = i / (TILE_COLS / 4), q = i % (TILE_COLS / 4);
      cp_async16(dst + row * TILE_COLS + 4 * q, src + (long long)row * m.ld + 4 * q);
    }
  };
  load_chunk(0, 0);
  cp_async_commit();

  for (int i = tid; i < m.Kp * GS; i += LBS_T) {
    const int s = i % GS, k = i / GS;
    sC[i] = g0 + s < batch ? w.coef[(long long)(g0 + s) * m.Kp + k] : 0.f;
  }
  const int a_len = m.J * 12;
  for (int i = tid; i < GS * a_len; i += LBS_T) {
    const int s = i / a_len;
    sA[i] = g0 + s < batch ? w.A[(long long)g0 * a_len + i] : 0.f;
  }
  for (int i = tid; i < GS * 3; i += LBS_T) sO[i] = g0 + i / 3 < batch ? w.offs[(long long)g0 * 3 + i] : 0.f;

  const int vl = tid % NV, oct = tid / NV;
  const int v = tile * NV + vl;
  float acc[8][3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t = m.vtemp[3 * v + c];  // the padded columns hold zeros
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i][c] = t;
  }
  const float4* sC4 = reinterpret_cast<const float4*>(sC) + 2 * oct;
  for (int ch = 0; ch < n_chunk; ++ch) {
    if (ch + 1 < n_chunk) load_chunk(ch + 1, (ch + 1) & 1);
    cp_async_commit();
    cp_async_wait1();
    __syncthreads();
    const float* bs = sB + (ch & 1) * CHUNK_FLOATS + 3 * vl;
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      const float b0 = bs[kk * TILE_COLS], b1 = bs[kk * TILE_COLS + 1], b2 = bs[kk * TILE_COLS + 2];
      const float4 ca = sC4[(ch * KC + kk) * (GS / 4)], cb = sC4[(ch * KC + kk) * (GS / 4) + 1];
      const float cs[8] = {ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i][0] = fmaf(b0, cs[i], acc[i][0]);
        acc[i][1] = fmaf(b1, cs[i], acc[i][1]);
        acc[i][2] = fmaf(b2, cs[i], acc[i][2]);
      }
    }
    __syncthreads();
  }
  if (v >= m.V) return;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int sl = 8 * oct + i, s = g0 + sl;
    if (s >= batch) break;
    float y[3];
    skin_point(m, sA + sl * a_len, v, acc[i], y);
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = (y[c] + sO[3 * sl + c]) * m.scale;
    float* dst = verts + ((long long)s * m.V + v) * 3;
    dst[0] = o[0], dst[1] = o[1], dst[2] = o[2];
    for (int q = 0; q < m.n_vj; ++q)
      if (m.vj_vert[q] == v) {
        float* jd = joints + ((long long)s * m.n_out + m.vj_out[q]) * 3;
        jd[0] = o[0], jd[1] = o[1], jd[2] = o[2];
      }
  }
}

constexpr size_t lbs_smem_bytes(int Kp, int J) {
  return sizeof(float) * ((size_t)2 * CHUNK_FLOATS + (size_t)Kp * GS + (size_t)GS * J * 12 + GS * 3);
}
// What the largest model the handle accepts needs (168 KB).  The attribute belongs to the kernel on its device, not to
// a handle, so every launch sets this one value: handles of different sizes (SMPL, MANO) can then be used in any
// order and from any thread.  A launch still reserves only its own model's lbs_smem_bytes.
constexpr size_t LBS_SMEM_MAX = lbs_smem_bytes((MAX_K + KC - 1) / KC * KC, MAX_J);
static_assert(LBS_SMEM_MAX <= 227 * 1024, "k_lbs shared memory exceeds the sm_90 limit");

// ------------------------------------------------------------------------------------------------ backward
// The vector-Jacobian product of the forward above, with respect to pose, betas and trans (p2m_body_model_backward).
// It recomputes what it needs with k_batch_flags and k_pose (into the backward's own workspace), then:
//  k_lbs_bwd   the k_lbs tiles again: v_posed x, g = scale (grad_verts + grad of the vertex's output joints),
//              dx = T[:3,:3]^T g into the workspace, and per (sample, tile) partials of dA_j = sum_v w_vj g [x; 1]^T and
//              of sum_v g, each summed over the tile's vertices in ascending order by one thread
//  k_dcoef     dcoef = dx basis^T per 768-column split of the basis (a fixed split: per-(sample, split) partials)
//  k_pose_bwd  one warp per sample: sums the partials in order, recomputes R, J, G, adds the centre term, walks the
//              chain in reverse and applies the pose-blend, Rodrigues and J_regressor shapedirs backwards
constexpr int DC_T = 256;               // threads per k_dcoef CTA: a 64-sample x 64-coefficient tile, 4 x 4 per thread
constexpr int DC_BM = 64, DC_BN = 64, DC_BK = 16;
constexpr int DC_COLS = 2 * TILE_COLS;  // basis columns per split
constexpr int W_LD = NV + 1;            // row stride of k_lbs_bwd's dense weight tile (bank-conflict padding)

struct BwdWork {
  const float* dx;  // [B, ld]   T^T g per vertex column (zero in the padding)
  const float* pA;  // [B, n_tiles, 12 J + 3]  per-tile partials of dA_j and of sum g
  const float* pC;  // [B, n_split, Kp]        per-split partials of dcoef
  int n_split;
};

// The derivative of rodrigues() as autograd takes it through batch_rodrigues: quat2mat, the renormalisation, the
// half-angle quaternion, axis = theta / angle with angle = |theta + 1e-8|.  dR [9] -> dth [3].
__device__ __forceinline__ void rodrigues_vjp(const float* th, const float* g, float* dth) {
  const float a0 = th[0] + 1e-8f, a1 = th[1] + 1e-8f, a2 = th[2] + 1e-8f;
  const float angle = sqrtf(a0 * a0 + a1 * a1 + a2 * a2);
  const float half = angle * 0.5f;
  const float c = cosf(half), s = sinf(half);
  const float n0 = th[0] / angle, n1 = th[1] / angle, n2 = th[2] / angle;
  const float q0 = c, q1 = s * n0, q2 = s * n1, q3 = s * n2;
  const float qn = sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
  const float w = q0 / qn, x = q1 / qn, y = q2 / qn, z = q3 / qn;
  const float dw = 2.f * (w * (g[0] + g[4] + g[8]) + x * (g[7] - g[5]) + y * (g[2] - g[6]) + z * (g[3] - g[1]));
  const float dx = 2.f * (x * (g[0] - g[4] - g[8]) + y * (g[1] + g[3]) + z * (g[2] + g[6]) + w * (g[7] - g[5]));
  const float dy = 2.f * (y * (g[4] - g[0] - g[8]) + x * (g[1] + g[3]) + z * (g[5] + g[7]) + w * (g[2] - g[6]));
  const float dz = 2.f * (z * (g[8] - g[0] - g[4]) + x * (g[2] + g[6]) + y * (g[5] + g[7]) + w * (g[3] - g[1]));
  const float dot = w * dw + x * dx + y * dy + z * dz;  // through q / |q|
  const float e0 = (dw - w * dot) / qn, e1 = (dx - x * dot) / qn, e2 = (dy - y * dot) / qn, e3 = (dz - z * dot) / qn;
  const float dn0 = s * e1, dn1 = s * e2, dn2 = s * e3;
  const float ds = e1 * n0 + e2 * n1 + e3 * n2;
  float dangle = 0.5f * (c * ds - s * e0);
  dangle = dangle - (dn0 * th[0] + dn1 * th[1] + dn2 * th[2]) / (angle * angle);  // through theta / angle
  const float r = dangle / angle;                                                   // through |theta + 1e-8|
  dth[0] = dn0 / angle + r * a0, dth[1] = dn1 / angle + r * a1, dth[2] = dn2 / angle + r * a2;
}

// grid (sample groups, vertex tiles), the k_lbs tiling.  The basis loop is k_lbs's; then each thread stages (g, x) of
// its vertex for its 8 samples, and the CTA's threads take (sample, joint) tasks: 12 entries of dA_j over the tile's
// 128 vertices in ascending order (joint J: the 3 entries of sum g).
__global__ void __launch_bounds__(LBS_T) k_lbs_bwd(ModelDev m, int batch, Work w, const float* __restrict__ grad_verts,
                                                   const float* __restrict__ grad_joints, float* __restrict__ dx,
                                                   float* __restrict__ pA) {
  extern __shared__ float4 smem4[];
  float* sB = reinterpret_cast<float*>(smem4);     // [2][KC][384], then [16][128][6] (g, x)
  float* sC = sB + 2 * CHUNK_FLOATS;               // [Kp][16]
  float* sA = sC + m.Kp * GS;                      // [16][J * 12]
  float* sW = sA + GS * m.J * 12;                  // [J][W_LD]  dense skinning weights of the tile
  const int tid = threadIdx.x;
  const int g0 = blockIdx.x * GS, tile = blockIdx.y;
  const int n_chunk = m.Kp / KC;
  const float* btile = m.basis + (long long)tile * TILE_COLS;

  auto load_chunk = [&](int ch, int stage) {
    float* dst = sB + stage * CHUNK_FLOATS;
    const float* src = btile + (long long)ch * KC * m.ld;
    for (int i = tid; i < CHUNK_FLOATS / 4; i += LBS_T) {
      const int row = i / (TILE_COLS / 4), q = i % (TILE_COLS / 4);
      cp_async16(dst + row * TILE_COLS + 4 * q, src + (long long)row * m.ld + 4 * q);
    }
  };
  load_chunk(0, 0);
  cp_async_commit();

  for (int i = tid; i < m.Kp * GS; i += LBS_T) {
    const int s = i % GS, k = i / GS;
    sC[i] = g0 + s < batch ? w.coef[(long long)(g0 + s) * m.Kp + k] : 0.f;
  }
  const int a_len = m.J * 12;
  for (int i = tid; i < GS * a_len; i += LBS_T) {
    const int s = i / a_len;
    sA[i] = g0 + s < batch ? w.A[(long long)g0 * a_len + i] : 0.f;
  }
  const int vl = tid % NV, oct = tid / NV;
  const int v = tile * NV + vl;
  for (int j = oct; j < m.J; j += LBS_T / NV) {
    float wt = 0.f;
    if (v < m.V)
      for (int e = m.w_ptr[v]; e < m.w_ptr[v + 1]; ++e)
        if (m.w_idx[e] == j) wt = m.w_val[e];
    sW[j * W_LD + vl] = wt;
  }

  float acc[8][3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float t = m.vtemp[3 * v + c];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i][c] = t;
  }
  const float4* sC4 = reinterpret_cast<const float4*>(sC) + 2 * oct;
  for (int ch = 0; ch < n_chunk; ++ch) {
    if (ch + 1 < n_chunk) load_chunk(ch + 1, (ch + 1) & 1);
    cp_async_commit();
    cp_async_wait1();
    __syncthreads();
    const float* bs = sB + (ch & 1) * CHUNK_FLOATS + 3 * vl;
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      const float b0 = bs[kk * TILE_COLS], b1 = bs[kk * TILE_COLS + 1], b2 = bs[kk * TILE_COLS + 2];
      const float4 ca = sC4[(ch * KC + kk) * (GS / 4)], cb = sC4[(ch * KC + kk) * (GS / 4) + 1];
      const float cs[8] = {ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i][0] = fmaf(b0, cs[i], acc[i][0]);
        acc[i][1] = fmaf(b1, cs[i], acc[i][1]);
        acc[i][2] = fmaf(b2, cs[i], acc[i][2]);
      }
    }
    __syncthreads();
  }
  // the basis chunks are consumed: sB now holds (g, x) per (sample, vertex)
  float* sGX = sB;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int sl = 8 * oct + i, s = g0 + sl;
    float g[3] = {0.f, 0.f, 0.f};
    if (v < m.V && s < batch) {
      if (grad_verts)
        for (int c = 0; c < 3; ++c) g[c] = grad_verts[((long long)s * m.V + v) * 3 + c];
      if (grad_joints)
        for (int q = 0; q < m.n_vj; ++q)
          if (m.vj_vert[q] == v)
            for (int c = 0; c < 3; ++c) g[c] = g[c] + grad_joints[((long long)s * m.n_out + m.vj_out[q]) * 3 + c];
      for (int c = 0; c < 3; ++c) g[c] = g[c] * m.scale;
    }
    if (s < batch) {
      // dx = T[:3,:3]^T g with T = sum_j w_vj A_j (ascending j), as the forward skins
      float T[9];
      for (int q = 0; q < 9; ++q) T[q] = 0.f;
      if (v < m.V)
        for (int e = m.w_ptr[v]; e < m.w_ptr[v + 1]; ++e) {
          const float wt = m.w_val[e];
          const float* a = sA + sl * a_len + 12 * m.w_idx[e];
          for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) T[3 * r + c] = fmaf(wt, a[4 * r + c], T[3 * r + c]);
        }
      float* d = dx + (long long)s * m.ld + (long long)tile * TILE_COLS + 3 * vl;
      for (int c = 0; c < 3; ++c) d[c] = fmaf(T[6 + c], g[2], fmaf(T[3 + c], g[1], T[c] * g[0]));
    }
    float* st = sGX + (sl * NV + vl) * 6;
    st[0] = g[0], st[1] = g[1], st[2] = g[2], st[3] = acc[i][0], st[4] = acc[i][1], st[5] = acc[i][2];
  }
  __syncthreads();
  const int PA = 12 * m.J + 3;
  for (int t = tid; t < GS * (m.J + 1); t += LBS_T) {
    const int sl = t / (m.J + 1), j = t % (m.J + 1), s = g0 + sl;
    if (s >= batch) continue;
    const float* gx = sGX + sl * NV * 6;
    float* out = pA + ((long long)s * gridDim.y + tile) * PA;
    if (j == m.J) {  // sum g
      float r0 = 0.f, r1 = 0.f, r2 = 0.f;
      for (int u = 0; u < NV; ++u) r0 = r0 + gx[6 * u], r1 = r1 + gx[6 * u + 1], r2 = r2 + gx[6 * u + 2];
      out[12 * m.J] = r0, out[12 * m.J + 1] = r1, out[12 * m.J + 2] = r2;
      continue;
    }
    float dA[12];
#pragma unroll
    for (int q = 0; q < 12; ++q) dA[q] = 0.f;
    const float* wj = sW + j * W_LD;
    for (int u = 0; u < NV; ++u) {
      const float wt = wj[u];
      if (wt == 0.f) continue;
      const float* p = gx + 6 * u;
      const float xh[4] = {p[3], p[4], p[5], 1.f};
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const float wg = wt * p[r];
#pragma unroll
        for (int c = 0; c < 4; ++c) dA[4 * r + c] = fmaf(wg, xh[c], dA[4 * r + c]);
      }
    }
#pragma unroll
    for (int q = 0; q < 12; ++q) out[12 * j + q] = dA[q];
  }
}

// grid (sample blocks of 64, coefficient blocks of 64, column splits).  part[b, split, k] = sum over the split's columns
// (ascending) of dx[b, col] basis[k, col]; every (b, k) is one thread's sequential sum, so it does not depend on the
// sample's place in the batch.
__global__ void __launch_bounds__(DC_T) k_dcoef(ModelDev m, int batch, const float* __restrict__ dx, int n_split,
                                                float* __restrict__ part) {
  __shared__ __align__(16) float sX[DC_BK][DC_BM];
  __shared__ __align__(16) float sW[DC_BK][DC_BN];
  const int tid = threadIdx.x, b0 = blockIdx.x * DC_BM, k0 = blockIdx.y * DC_BN, sp = blockIdx.z;
  const int tx = tid % 16, ty = tid / 16;
  const int lr = tid >> 2, lc = (tid & 3) * 4;
  const int c_beg = sp * DC_COLS, c_end = min(c_beg + DC_COLS, m.ld);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int k = 0; k < 4; ++k) acc[i][k] = 0.f;
  for (int c0 = c_beg; c0 < c_end; c0 += DC_BK) {
    float4 xv = make_float4(0.f, 0.f, 0.f, 0.f), bv = xv;
    if (b0 + lr < batch) xv = *reinterpret_cast<const float4*>(dx + (long long)(b0 + lr) * m.ld + c0 + lc);
    if (k0 + lr < m.Kp) bv = *reinterpret_cast<const float4*>(m.basis + (long long)(k0 + lr) * m.ld + c0 + lc);
    __syncthreads();
    sX[lc][lr] = xv.x, sX[lc + 1][lr] = xv.y, sX[lc + 2][lr] = xv.z, sX[lc + 3][lr] = xv.w;
    sW[lc][lr] = bv.x, sW[lc + 1][lr] = bv.y, sW[lc + 2][lr] = bv.z, sW[lc + 3][lr] = bv.w;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < DC_BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&sX[kk][4 * ty]);
      const float4 bb = *reinterpret_cast<const float4*>(&sW[kk][4 * tx]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bw[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[i][k] = fmaf(av[i], bw[k], acc[i][k]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int b = b0 + 4 * ty + i;
    if (b >= batch) break;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int kc = k0 + 4 * tx + k;
      if (kc < m.Kp) part[((long long)b * n_split + sp) * m.Kp + kc] = acc[i][k];
    }
  }
}

// One warp per sample: everything after the per-vertex work, in fixed orders.
__global__ void __launch_bounds__(32) k_pose_bwd(ModelDev m, const float* __restrict__ pose,
                                                 const float* __restrict__ betas, int betas_rule,
                                                 const float* __restrict__ trans, int center_idx, Work w, BwdWork bw,
                                                 const float* __restrict__ grad_joints, float* __restrict__ grad_pose,
                                                 float* __restrict__ grad_betas, float* __restrict__ grad_trans) {
  __shared__ float th[3 * MAX_J], R[MAX_J][9], jp[MAX_J][3], G[MAX_J][12], beta[MAX_S];
  __shared__ float dA[MAX_J][12], dG[MAX_J][12], dR[MAX_J][9], dJ[MAX_J][3], gt[MAX_J][3], dcf[MAX_K + 16];
  __shared__ float goff[3], dxc[3];
  const int b = blockIdx.x, lane = threadIdx.x, J = m.J, S = m.S;
  int flag = 0;
  for (int i = lane; i < w.n_flag_blocks; i += 32) flag |= w.flags[i];
  flag = __reduce_or_sync(0xffffffffu, flag);
  const bool given = betas != nullptr && (betas_rule == P2M_BETAS_AS_GIVEN || (flag & 1));
  const bool trans_used = trans != nullptr && (flag & 2);
  for (int s = lane; s < S; s += 32) beta[s] = given ? betas[(long long)b * S + s] : m.mbetas[s];
  for (int i = lane; i < 3 * J; i += 32) {
    float x = pose[(long long)b * 3 * J + i];
    if (m.pmean && i >= 3) x = m.pmean[i - 3] + x;
    th[i] = x;
  }
  __syncwarp();
  for (int j = lane; j < J; j += 32) rodrigues(th + 3 * j, R[j]);
  for (int e = lane; e < 3 * J; e += 32) {
    float acc = m.jtemp[e];
    for (int s = 0; s < S; ++s) acc = fmaf(m.jshape[(long long)e * S + s], beta[s], acc);
    jp[e / 3][e % 3] = acc;
  }
  // the partials, each summed in tile / split order
  const int PA = 12 * J + 3, n_tiles = m.ld / TILE_COLS;
  for (int k = lane; k < m.Kp; k += 32) {
    float acc = 0.f;
    for (int sp = 0; sp < bw.n_split; ++sp) acc = acc + bw.pC[((long long)b * bw.n_split + sp) * m.Kp + k];
    dcf[k] = acc;
  }
  for (int e = lane; e < PA; e += 32) {
    float acc = 0.f;
    for (int t = 0; t < n_tiles; ++t) acc = acc + bw.pA[((long long)b * n_tiles + t) * PA + e];
    if (e < 12 * J)
      dA[e / 12][e % 12] = acc;
    else
      goff[e - 12 * J] = acc;  // sum over vertices of g, so far
  }
  __syncwarp();
  const int r = lane >> 2, c = lane & 3;
  if (lane < 12) G[0][lane] = c < 3 ? R[0][3 * r + c] : jp[0][r];
  __syncwarp();
  for (int j = 1; j < J; ++j) {
    const int p = m.parents[j];
    if (lane < 12) {
      const float* g = G[p] + 4 * r;
      float l0, l1, l2;
      if (c < 3) {
        l0 = R[j][c], l1 = R[j][3 + c], l2 = R[j][6 + c];
      } else {
        l0 = jp[j][0] - jp[p][0], l1 = jp[j][1] - jp[p][1], l2 = jp[j][2] - jp[p][2];
      }
      float v = fmaf(g[2], l2, fmaf(g[1], l1, g[0] * l0));
      if (c == 3) v = v + g[3];
      G[j][lane] = v;
    }
    __syncwarp();
  }
  // the gradient of the per-sample offset: every output moves with it
  if (lane < 3) {
    float acc = goff[lane];
    if (grad_joints)
      for (int o = 0; o < m.n_out; ++o)
        if (m.jmap[o] >= 0) acc = acc + grad_joints[((long long)b * m.n_out + o) * 3 + lane] * m.scale;
    goff[lane] = acc;
    if (grad_trans) grad_trans[(long long)b * 3 + lane] = trans_used ? acc : 0.f;
  }
  __syncwarp();
  const int ce = (!trans_used && center_idx >= 0) ? m.jmap[center_idx] : J;  // J: no centring
  for (int e = lane; e < 3 * J; e += 32) {
    const int j = e / 3, q = e % 3;
    float acc = 0.f;
    if (grad_joints)
      for (int o = 0; o < m.n_out; ++o)
        if (m.jmap[o] == j) acc = acc + grad_joints[((long long)b * m.n_out + o) * 3 + q] * m.scale;
    if (ce == j) acc = acc - goff[q];
    gt[j][q] = acc;
  }
  if (ce < 0) {  // centred on a vertex: - goff enters that vertex's skinning and v_posed
    const int v = -1 - ce;
    const float* A = w.A + (long long)b * J * 12;
    const float* cf = w.coef + (long long)b * m.Kp;
    if (lane == 0) {
      float x[3], T[9];
      for (int q = 0; q < 3; ++q) {
        float acc = m.vtemp[3 * v + q];
        for (int k = 0; k < m.Kp; ++k) acc = fmaf(m.basis[(long long)k * m.ld + 3 * v + q], cf[k], acc);
        x[q] = acc;
      }
      for (int q = 0; q < 9; ++q) T[q] = 0.f;
      for (int e = m.w_ptr[v]; e < m.w_ptr[v + 1]; ++e) {
        const float wt = m.w_val[e];
        const int j = m.w_idx[e];
        for (int rr = 0; rr < 3; ++rr)
          for (int cc = 0; cc < 3; ++cc) T[3 * rr + cc] = fmaf(wt, A[12 * j + 4 * rr + cc], T[3 * rr + cc]);
        for (int rr = 0; rr < 3; ++rr) {
          const float wg = wt * -goff[rr];
          for (int cc = 0; cc < 3; ++cc) dA[j][4 * rr + cc] = fmaf(wg, x[cc], dA[j][4 * rr + cc]);
          dA[j][4 * rr + 3] = dA[j][4 * rr + 3] + wg;
        }
      }
      for (int q = 0; q < 3; ++q) dxc[q] = -(T[q] * goff[0] + T[3 + q] * goff[1] + T[6 + q] * goff[2]);
    }
    __syncwarp();
    for (int k = lane; k < m.Kp; k += 32) {
      const float* bk = m.basis + (long long)k * m.ld + 3 * v;
      dcf[k] = dcf[k] + (bk[0] * dxc[0] + bk[1] * dxc[1] + bk[2] * dxc[2]);
    }
  }
  __syncwarp();
  // A_j = [G_j[:, :3] | G_j[:, 3] - G_j[:, :3] J_j]  ->  dG_j, dJ_j; the output joints add to dG_j[:, 3]
  for (int e = lane; e < 12 * J; e += 32) {
    const int j = e / 12, q = e % 12, rr = q >> 2, cc = q & 3;
    dG[j][q] = cc < 3 ? dA[j][q] - dA[j][4 * rr + 3] * jp[j][cc] : dA[j][q] + gt[j][rr];
  }
  for (int e = lane; e < 3 * J; e += 32) {
    const int j = e / 3, q = e % 3;
    dJ[j][q] = -(G[j][q] * dA[j][3] + G[j][4 + q] * dA[j][7] + G[j][8 + q] * dA[j][11]);
  }
  __syncwarp();
  // the chain in reverse: G_j = G_p [R_j | J_j - J_p]
  for (int j = J - 1; j >= 1; --j) {
    const int p = m.parents[j];
    if (lane < 12) {
      const float* d = dG[j] + 4 * r;
      float v = d[3];
      if (c < 3) v = d[0] * R[j][3 * c] + d[1] * R[j][3 * c + 1] + d[2] * R[j][3 * c + 2] + d[3] * (jp[j][c] - jp[p][c]);
      dG[p][lane] = dG[p][lane] + v;
    } else if (lane < 21) {
      const int k = (lane - 12) / 3, cc = (lane - 12) % 3;
      dR[j][3 * k + cc] = G[p][k] * dG[j][cc] + G[p][4 + k] * dG[j][4 + cc] + G[p][8 + k] * dG[j][8 + cc] +
                          dcf[S + 9 * (j - 1) + 3 * k + cc];
    } else if (lane < 24) {
      const int k = lane - 21;
      const float t = G[p][k] * dG[j][3] + G[p][4 + k] * dG[j][7] + G[p][8 + k] * dG[j][11];
      dJ[j][k] = dJ[j][k] + t;
      dJ[p][k] = dJ[p][k] - t;
    }
    __syncwarp();
  }
  if (lane < 9) dR[0][lane] = dG[0][4 * (lane / 3) + lane % 3];
  if (lane < 3) dJ[0][lane] = dJ[0][lane] + dG[0][4 * lane + 3];
  __syncwarp();
  for (int j = lane; j < J; j += 32) {
    float d[3];
    rodrigues_vjp(th + 3 * j, dR[j], d);
    for (int q = 0; q < 3; ++q) grad_pose[(long long)b * 3 * J + 3 * j + q] = d[q];
  }
  if (grad_betas)
    for (int s = lane; s < S; s += 32) {
      float acc = dcf[s];
      for (int e = 0; e < 3 * J; ++e) acc = fmaf(m.jshape[(long long)e * S + s], dJ[e / 3][e % 3], acc);
      grad_betas[(long long)b * S + s] = given ? acc : 0.f;
    }
}

constexpr size_t lbs_bwd_smem_bytes(int Kp, int J) {
  return sizeof(float) * ((size_t)2 * CHUNK_FLOATS + (size_t)Kp * GS + (size_t)GS * J * 12 + (size_t)J * W_LD);
}
constexpr size_t LBS_BWD_SMEM_MAX = lbs_bwd_smem_bytes((MAX_K + KC - 1) / KC * KC, MAX_J);
static_assert(LBS_BWD_SMEM_MAX <= 227 * 1024, "k_lbs_bwd shared memory exceeds the sm_90 limit");
static_assert(2 * CHUNK_FLOATS >= GS * NV * 6, "k_lbs_bwd stages (g, x) in the basis buffers");

bool all_finite(const float* p, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (!std::isfinite(p[i])) return false;
  return true;
}

}  // namespace
}  // namespace p2m

using namespace p2m;

struct p2m_body_model {
  int device = 0;
  int V = 0, J = 0, S = 0, K = 0, Kp = 0, ld = 0, n_out = 0, n_tiles = 0, n_vj = 0;
  float scale = 1.f;
  size_t lbs_smem = 0;
  std::vector<void*> owned;
  ModelDev dev{};
};

namespace p2m {
BodyModelInfo body_model_info(const p2m_body_model_t* m) {
  return BodyModelInfo{m->device, m->V, m->J, m->S, m->n_out, m->dev.mbetas};
}
}  // namespace p2m

namespace {

template <typename T>
int upload(p2m_body_model* m, const std::vector<T>& h, const T** out) {
  *out = nullptr;
  if (h.empty()) return P2M_OK;
  void* d = nullptr;
  P2M_CUDA_OK(cudaMalloc(&d, sizeof(T) * h.size()));
  m->owned.push_back(d);
  P2M_CUDA_OK(cudaMemcpy(d, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice));
  *out = static_cast<const T*>(d);
  return P2M_OK;
}

void free_model(p2m_body_model* m) {
  if (!m) return;
  {
    DeviceGuard guard(m->device);
    for (void* p : m->owned) cudaFree(p);
  }
  delete m;
}

int create_impl(const p2m_body_model_desc_t* d, p2m_body_model* m) {
  const int V = d->n_vertex, J = d->n_joint, S = d->n_betas, n_out = d->n_out_joints;
  const int P = 9 * (J - 1), K = S + P, Kp = (K + KC - 1) / KC * KC;
  const int n_tiles = (V + NV - 1) / NV, ld = n_tiles * TILE_COLS;
  m->device = d->device, m->V = V, m->J = J, m->S = S, m->K = K, m->Kp = Kp, m->ld = ld, m->n_out = n_out;
  m->n_tiles = n_tiles, m->scale = d->scale;
  // fp64 products with the joint regressor: J_template = J_regressor v_template, J_shapedirs = J_regressor shapedirs
  std::vector<double> jt((size_t)J * 3, 0.0), js((size_t)J * 3 * S, 0.0);
  for (int j = 0; j < J; ++j)
    for (int v = 0; v < V; ++v) {
      const double r = d->J_regressor[(size_t)j * V + v];
      if (r == 0.0) continue;
      for (int c = 0; c < 3; ++c) {
        jt[j * 3 + c] += r * d->v_template[(size_t)v * 3 + c];
        for (int s = 0; s < S; ++s) js[((size_t)j * 3 + c) * S + s] += r * d->shapedirs[((size_t)v * 3 + c) * S + s];
      }
    }
  std::vector<float> jtf(jt.begin(), jt.end()), jsf(js.begin(), js.end());
  std::vector<float> basis((size_t)Kp * ld, 0.f), vt((size_t)ld, 0.f);
  for (int v = 0; v < V; ++v)
    for (int c = 0; c < 3; ++c) {
      const size_t col = (size_t)v * 3 + c;
      vt[col] = d->v_template[col];
      for (int s = 0; s < S; ++s) basis[(size_t)s * ld + col] = d->shapedirs[col * S + s];
      for (int p = 0; p < P; ++p) basis[(size_t)(S + p) * ld + col] = d->posedirs[col * P + p];
    }
  std::vector<int> wp(V + 1, 0), wi;
  std::vector<float> wv;
  for (int v = 0; v < V; ++v) {
    for (int j = 0; j < J; ++j) {
      const float x = d->weights[(size_t)v * J + j];
      if (x != 0.f) wi.push_back(j), wv.push_back(x);
    }
    wp[v + 1] = (int)wi.size();
  }
  std::vector<int> vj_out, vj_vert;
  for (int o = 0; o < n_out; ++o)
    if (d->joint_map[o] < 0) vj_out.push_back(o), vj_vert.push_back(-1 - d->joint_map[o]);
  std::vector<float> mb(d->model_betas, d->model_betas + S), pm;
  if (d->pose_mean) pm.assign(d->pose_mean, d->pose_mean + 3 * (J - 1));
  std::vector<int> par(d->parents, d->parents + J), jm(d->joint_map, d->joint_map + n_out);

  DeviceGuard guard(d->device);
  ModelDev& g = m->dev;
  g.V = V, g.J = J, g.S = S, g.K = K, g.Kp = Kp, g.ld = ld, g.n_out = n_out, g.scale = d->scale;
  g.n_vj = (int)vj_out.size();
  P2M_TRY(upload(m, basis, &g.basis));
  P2M_TRY(upload(m, vt, &g.vtemp));
  P2M_TRY(upload(m, jtf, &g.jtemp));
  P2M_TRY(upload(m, jsf, &g.jshape));
  P2M_TRY(upload(m, mb, &g.mbetas));
  P2M_TRY(upload(m, pm, &g.pmean));
  P2M_TRY(upload(m, par, &g.parents));
  P2M_TRY(upload(m, jm, &g.jmap));
  P2M_TRY(upload(m, wp, &g.w_ptr));
  if (wi.empty()) wi.push_back(0), wv.push_back(0.f);  // keep the pointers valid for a model without weights
  P2M_TRY(upload(m, wi, &g.w_idx));
  P2M_TRY(upload(m, wv, &g.w_val));
  P2M_TRY(upload(m, vj_out, &g.vj_out));
  P2M_TRY(upload(m, vj_vert, &g.vj_vert));
  m->n_vj = g.n_vj;
  m->lbs_smem = lbs_smem_bytes(Kp, J);
  return P2M_OK;
}

struct WorkLayout {
  size_t flags, A, coef, offs, total;
};
WorkLayout work_layout(const p2m_body_model* m, int batch) {
  WorkLayout l;
  l.flags = 0;
  l.A = align256(sizeof(int) * MAX_FLAG_BLOCKS);
  l.coef = l.A + align256(sizeof(float) * (size_t)batch * m->J * 12);
  l.offs = l.coef + align256(sizeof(float) * (size_t)batch * m->Kp);
  l.total = l.offs + align256(sizeof(float) * (size_t)batch * 3);
  return l;
}

// The backward's workspace: the forward's, then k_pose's kinematic joints (unused), dx, and the two partial arrays.
struct BwdLayout {
  WorkLayout fwd;
  size_t joints, dx, pA, pC, total;
  int n_split;
};
BwdLayout bwd_layout(const p2m_body_model* m, int batch) {
  BwdLayout l;
  l.fwd = work_layout(m, batch);
  l.n_split = (m->ld + DC_COLS - 1) / DC_COLS;
  l.joints = l.fwd.total;
  l.dx = l.joints + align256(sizeof(float) * (size_t)batch * m->n_out * 3);
  l.pA = l.dx + align256(sizeof(float) * (size_t)batch * m->ld);
  l.pC = l.pA + align256(sizeof(float) * (size_t)batch * m->n_tiles * (12 * m->J + 3));
  l.total = l.pC + align256(sizeof(float) * (size_t)batch * l.n_split * m->Kp);
  return l;
}

}  // namespace

extern "C" {

int p2m_body_model_create(const p2m_body_model_desc_t* d, p2m_body_model_t** out) {
  if (!out) {
    set_error("body_model_create: null output pointer");
    return P2M_ERR_INVALID;
  }
  *out = nullptr;
  if (!d || !d->v_template || !d->shapedirs || !d->posedirs || !d->J_regressor || !d->weights || !d->parents ||
      !d->model_betas || !d->joint_map) {
    set_error("body_model_create: null descriptor or buffer (only pose_mean may be NULL)");
    return P2M_ERR_INVALID;
  }
  const int V = d->n_vertex, J = d->n_joint, S = d->n_betas, n_out = d->n_out_joints;
  if (V < 1 || V > (1 << 22) || J < 1 || J > MAX_J || S < 1 || S > MAX_S || n_out < 1 || n_out > MAX_OUT) {
    set_error("body_model_create: sizes out of range (n_vertex in [1, 2^22], n_joint in [1, 64], n_betas in "
              "[1, 512], n_out_joints in [1, 1024])");
    return P2M_ERR_INVALID;
  }
  if (d->parents[0] != -1) {
    set_error("body_model_create: parents[0] must be -1 (the root)");
    return P2M_ERR_INVALID;
  }
  for (int i = 1; i < J; ++i)
    if (d->parents[i] < 0 || d->parents[i] >= i) {
      set_error("body_model_create: parents[" + std::to_string(i) + "] = " + std::to_string(d->parents[i]) +
                " is not in [0, " + std::to_string(i) + "): joints must come in topological (parent-first) order");
      return P2M_ERR_INVALID;
    }
  for (int o = 0; o < n_out; ++o) {
    const int e = d->joint_map[o];
    if (e >= J || (e < 0 && -1 - e >= V)) {
      set_error("body_model_create: joint_map[" + std::to_string(o) + "] = " + std::to_string(e) +
                " names neither a joint in [0, " + std::to_string(J) + ") nor a vertex -1 - v with v in [0, " +
                std::to_string(V) + ")");
      return P2M_ERR_INVALID;
    }
  }
  const size_t P = 9 * (size_t)(J - 1);
  struct {
    const char* name;
    const float* p;
    size_t n;
  } bufs[] = {{"v_template", d->v_template, (size_t)V * 3},
              {"shapedirs", d->shapedirs, (size_t)V * 3 * S},
              {"posedirs", d->posedirs, (size_t)V * 3 * P},
              {"J_regressor", d->J_regressor, (size_t)J * V},
              {"weights", d->weights, (size_t)V * J},
              {"model_betas", d->model_betas, (size_t)S},
              {"pose_mean", d->pose_mean, d->pose_mean ? 3 * (size_t)(J - 1) : 0},
              {"scale", &d->scale, 1}};
  for (const auto& b : bufs)
    if (!all_finite(b.p, b.n)) {
      set_error(std::string("body_model_create: ") + b.name + " holds a non-finite value");
      return P2M_ERR_INVALID;
    }
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || d->device < 0 || d->device >= n_dev) {
    cudaGetLastError();
    set_error("body_model_create: device " + std::to_string(d->device) + " is not available");
    return P2M_ERR_NOGPU;
  }
  auto* m = new p2m_body_model();
  const int st = create_impl(d, m);
  if (st != P2M_OK) {
    free_model(m);
    return st;
  }
  *out = m;
  return P2M_OK;
}

void p2m_body_model_destroy(p2m_body_model_t* m) { free_model(m); }

size_t p2m_body_model_workspace_bytes(const p2m_body_model_t* m, int batch) {
  if (!m || batch <= 0 || batch > MAX_BATCH) return 0;
  return work_layout(m, batch).total;
}

int p2m_body_model_forward(const p2m_body_model_t* m, const float* pose, const float* betas, int betas_rule,
                           const float* trans, int center_idx, float* verts, float* joints, int batch,
                           void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  if (!m || !pose || !verts || !joints || batch <= 0 || batch > MAX_BATCH ||
      (betas_rule != P2M_BETAS_ZERO_MEANS_MODEL && betas_rule != P2M_BETAS_AS_GIVEN) || center_idx >= m->n_out) {
    set_error("body_model_forward: bad argument (null model / pose / output, batch out of [1, 2^24], unknown "
              "betas_rule or center_idx >= n_out_joints)");
    return P2M_ERR_INVALID;
  }
  const WorkLayout l = work_layout(m, batch);
  if (!workspace || workspace_bytes < l.total) {
    set_error("body_model_forward: workspace needs " + std::to_string(l.total) + " bytes");
    return P2M_ERR_WORKSPACE;
  }
  DeviceGuard guard(m->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  const long long n_betas = (betas && betas_rule == P2M_BETAS_ZERO_MEANS_MODEL) ? (long long)batch * m->S : 0;
  const long long n_trans = trans ? (long long)batch * 3 : 0;
  // one CTA per 16 K values to test, at most MAX_FLAG_BLOCKS
  const long long n_test = n_betas > n_trans ? n_betas : n_trans;
  const int n_flag_blocks = (int)std::min<long long>(MAX_FLAG_BLOCKS, std::max<long long>(1, n_test / (16 * 1024)));
  Work w{reinterpret_cast<int*>(ws + l.flags), n_flag_blocks, reinterpret_cast<float*>(ws + l.A),
         reinterpret_cast<float*>(ws + l.coef), reinterpret_cast<float*>(ws + l.offs)};
  k_batch_flags<<<n_flag_blocks, FLAG_T, 0, s>>>(betas, n_betas, trans, n_trans, w.flags);
  P2M_LAUNCH_OK();
  k_pose<<<batch, 32, 0, s>>>(m->dev, pose, betas, betas_rule, trans, center_idx < 0 ? -1 : center_idx, joints, w);
  P2M_LAUNCH_OK();
  const dim3 grid((unsigned)((batch + GS - 1) / GS), (unsigned)m->n_tiles);
  P2M_CUDA_OK(cudaFuncSetAttribute(k_lbs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LBS_SMEM_MAX));
  k_lbs<<<grid, LBS_T, m->lbs_smem, s>>>(m->dev, batch, w, verts, joints);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

size_t p2m_body_model_backward_workspace_bytes(const p2m_body_model_t* m, int batch) {
  if (!m || batch <= 0 || batch > MAX_BATCH) return 0;
  return bwd_layout(m, batch).total;
}

int p2m_body_model_backward(const p2m_body_model_t* m, const float* pose, const float* betas, int betas_rule,
                            const float* trans, int center_idx, const float* grad_verts, const float* grad_joints,
                            float* grad_pose, float* grad_betas, float* grad_trans, int batch, void* workspace,
                            size_t workspace_bytes, p2m_stream_t stream) {
  if (!m || !pose || !grad_pose || batch <= 0 || batch > MAX_BATCH ||
      (betas_rule != P2M_BETAS_ZERO_MEANS_MODEL && betas_rule != P2M_BETAS_AS_GIVEN) || center_idx >= m->n_out) {
    set_error("body_model_backward: bad argument (null model / pose / grad_pose, batch out of [1, 2^24], unknown "
              "betas_rule or center_idx >= n_out_joints)");
    return P2M_ERR_INVALID;
  }
  const BwdLayout l = bwd_layout(m, batch);
  if (!workspace || workspace_bytes < l.total) {
    set_error("body_model_backward: workspace needs " + std::to_string(l.total) + " bytes");
    return P2M_ERR_WORKSPACE;
  }
  DeviceGuard guard(m->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  const long long n_betas = (betas && betas_rule == P2M_BETAS_ZERO_MEANS_MODEL) ? (long long)batch * m->S : 0;
  const long long n_trans = trans ? (long long)batch * 3 : 0;
  const long long n_test = n_betas > n_trans ? n_betas : n_trans;
  const int n_flag_blocks = (int)std::min<long long>(MAX_FLAG_BLOCKS, std::max<long long>(1, n_test / (16 * 1024)));
  Work w{reinterpret_cast<int*>(ws + l.fwd.flags), n_flag_blocks, reinterpret_cast<float*>(ws + l.fwd.A),
         reinterpret_cast<float*>(ws + l.fwd.coef), reinterpret_cast<float*>(ws + l.fwd.offs)};
  float* dx = reinterpret_cast<float*>(ws + l.dx);
  float* pA = reinterpret_cast<float*>(ws + l.pA);
  float* pC = reinterpret_cast<float*>(ws + l.pC);
  const int center = center_idx < 0 ? -1 : center_idx;
  k_batch_flags<<<n_flag_blocks, FLAG_T, 0, s>>>(betas, n_betas, trans, n_trans, w.flags);
  P2M_LAUNCH_OK();
  k_pose<<<batch, 32, 0, s>>>(m->dev, pose, betas, betas_rule, trans, center,
                              reinterpret_cast<float*>(ws + l.joints), w);
  P2M_LAUNCH_OK();
  const dim3 grid((unsigned)((batch + GS - 1) / GS), (unsigned)m->n_tiles);
  P2M_CUDA_OK(cudaFuncSetAttribute(k_lbs_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LBS_BWD_SMEM_MAX));
  k_lbs_bwd<<<grid, LBS_T, lbs_bwd_smem_bytes(m->Kp, m->J), s>>>(m->dev, batch, w, grad_verts, grad_joints, dx, pA);
  P2M_LAUNCH_OK();
  const dim3 dgrid((unsigned)((batch + DC_BM - 1) / DC_BM), (unsigned)((m->Kp + DC_BN - 1) / DC_BN),
                   (unsigned)l.n_split);
  k_dcoef<<<dgrid, DC_T, 0, s>>>(m->dev, batch, dx, l.n_split, pC);
  P2M_LAUNCH_OK();
  k_pose_bwd<<<batch, 32, 0, s>>>(m->dev, pose, betas, betas_rule, trans, center, w, BwdWork{dx, pA, pC, l.n_split},
                                  grad_joints, grad_pose, grad_betas, grad_trans);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
