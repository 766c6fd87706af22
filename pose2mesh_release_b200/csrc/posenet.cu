// Row f1 of SURVEY.md §8: PoseNet, the 2-D -> 3-D lifter in front of MeshNet (lib/models/posenet.py:25-87), and
// pose_combine = cat(pose2d, pose3d / 1000), MeshNet's input (lib/models/pose2mesh_net.py:16-22).
//   y = x W1^T + b1;  per stage  y += drop(relu(bn2(drop(relu(bn1(y))) Wa^T + ba))) Wb^T + bb;  pose3d = y W2^T + b2
// Eval (p2m_posenet_forward): running-stat BatchNorm, no dropout, BatchNorm / ReLU / residual fused into the GEMM
// epilogues; the 4 H x H weight matrices (64 MB each at H = 4096) dominate the traffic and are read once per call.
// Training (lib/core/base.py:116,246-265): the forward with batch statistics and dropout, and the backward;
// include/p2m_b200.h states the math, the dropout rule and the layout of `saved`.  New here, beside the assembly of the
// library's kernels: the counter-based dropout fused into the BN-apply + ReLU pass, and its backward.
#include <cuda_runtime.h>

#include <algorithm>
#include <string>
#include <vector>

#include "p2m_internal.h"

using namespace p2m;

namespace {

// How one dropout layer treats its elements: mode 0 keeps everything unscaled (p == 0), 1 draws, 2 zeroes (p == 1)
struct Dropout {
  const long long* seed;  // device [2]
  unsigned int layer, threshold;
  float keep_scale;
  int mode;
};
// multipliers of the four elements 4 q .. 4 q + 3
__device__ __forceinline__ void dropout_mul4(const Dropout& d, unsigned long long q, float m[4]) {
  if (d.mode != 1) {
    m[0] = m[1] = m[2] = m[3] = d.mode == 0 ? 1.f : 0.f;
    return;
  }
  const unsigned long long s0 = (unsigned long long)d.seed[0];
  const uint4 w = philox4x32_10(make_uint4((unsigned int)q, (unsigned int)(q >> 32), d.layer, (unsigned int)d.seed[1]),
                                make_uint2((unsigned int)s0, (unsigned int)(s0 >> 32)));
  m[0] = w.x < d.threshold ? d.keep_scale : 0.f;
  m[1] = w.y < d.threshold ? d.keep_scale : 0.f;
  m[2] = w.z < d.threshold ? d.keep_scale : 0.f;
  m[3] = w.w < d.threshold ? d.keep_scale : 0.f;
}

// a = drop(relu(z * scale + shift)): four consecutive elements (one Philox counter) per thread; amax (optional, zero on
// entry): max(a) as uint bits, for launch_absmax_finish
__global__ void __launch_bounds__(256) k_pn_bn_relu_drop(const float* __restrict__ z, long long n, int F,
                                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                                         const Dropout d, float* __restrict__ a,
                                                         unsigned int* __restrict__ amax) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float mx = 0.f;
  if (4 * q < n) {
    float m[4];
    dropout_mul4(d, (unsigned long long)q, m);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const long long i = 4 * q + e;
      if (i < n) {
        const int f = (int)(i % F);
        a[i] = fmaxf(fmaf(z[i], scale[f], shift[f]), 0.f) * m[e];
        mx = fmaxf(mx, a[i]);
      }
    }
  }
  if (amax != nullptr) {
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0 && mx > 0.f) atomicMax(amax, __float_as_uint(mx));
  }
}
// g *= the same multipliers (in place): the gradient through drop()
__global__ void __launch_bounds__(256) k_pn_drop_bwd(float* __restrict__ g, long long n, const Dropout d) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (4 * q >= n) return;
  float m[4];
  dropout_mul4(d, (unsigned long long)q, m);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const long long i = 4 * q + e;
    if (i < n) g[i] *= m[e];
  }
}
__global__ void __launch_bounds__(256) k_pn_add(float* __restrict__ y, const float* __restrict__ x, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] += x[i];
}
// out [C, R] = in [R, C]^T
__global__ void __launch_bounds__(256) k_pn_transpose(const float* __restrict__ in, int R, int C, float* __restrict__ out) {
  __shared__ float t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8)
    if (r0 + j < R && c0 + tx < C) t[j][tx] = in[(long long)(r0 + j) * C + c0 + tx];
  __syncthreads();
  for (int j = ty; j < 32; j += 8)
    if (c0 + j < C && r0 + tx < R) out[(long long)(c0 + j) * R + r0 + tx] = t[tx][j];
}
__global__ void __launch_bounds__(256) k_bn_relu_rows(const float* __restrict__ x, long long n, int F,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      const float* __restrict__ rm, const float* __restrict__ rv,
                                                      float eps, float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = (int)(i % F);
  const float sc = gamma[f] / sqrtf(rv[f] + eps);
  y[i] = fmaxf(fmaf(x[i] - rm[f], sc, beta[f]), 0.f);
}
// dst [rows, n_col] = src[:, :n_col] (row stride ld) + bias
__global__ void __launch_bounds__(256) k_take_cols(const float* __restrict__ src, int ld, const float* __restrict__ bias,
                                                   int n_col, long long n, float* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long r = i / n_col;
  const int c = (int)(i - r * n_col);
  dst[i] = src[r * ld + c] + bias[c];
}
// out [B J, 5] = cat(pose2d [B J, 2], pose3d [B J, 3] / 1000)
__global__ void __launch_bounds__(256) k_pose_combine(const float* __restrict__ pose2d, const float* __restrict__ pose3d,
                                                      long long n_joint_rows, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // (b, j)
  if (i >= n_joint_rows) return;
  out[i * 5 + 0] = pose2d[i * 2 + 0];
  out[i * 5 + 1] = pose2d[i * 2 + 1];
  out[i * 5 + 2] = pose3d[i * 3 + 0] / 1000.f;
  out[i * 5 + 3] = pose3d[i * 3 + 1] / 1000.f;
  out[i * 5 + 4] = pose3d[i * 3 + 2] / 1000.f;
}

inline unsigned blocks(long long n) { return (unsigned)((n + 255) / 256); }

Dropout make_dropout(float p, const int64_t* seed, int layer) {
  Dropout d;
  d.seed = reinterpret_cast<const long long*>(seed);
  d.layer = (unsigned int)layer;
  d.mode = p <= 0.f ? 0 : (p >= 1.f ? 2 : 1);
  d.threshold = d.mode == 1 ? (unsigned int)std::min((1.0 - (double)p) * 4294967296.0, 4294967295.0) : 0u;
  d.keep_scale = d.mode == 1 ? 1.f / (1.f - p) : 1.f;
  return d;
}

int round_up(int x, int m) { return (x + m - 1) / m * m; }

// The eval forward's workspace, sized (null base) and carved by one map.  With tc the H x H GEMMs run on the tensor
// cores (wgmma, fp16x3: launch_umma_gemm); the thin first / last layers (K = 2J, N = 3J) stay on the fp32 SIMT GEMM.
struct EvalWork {
  float *y, *a, *h, *sc;
  int* status;
  bool tc;
  void *apack = nullptr, *wpack = nullptr;  // operand images of the tensor-core GEMMs
  size_t bytes;
  EvalWork(void* ws, int B, int H) : tc(umma_gemm_supported(B, H, H)) {
    Bump b(ws);
    y = b.take<float>((size_t)B * H);
    a = b.take<float>((size_t)B * H);
    h = b.take<float>((size_t)B * H);
    sc = b.take<float>(2 * (size_t)H);
    status = b.take<int>(1);
    if (tc) {
      apack = b.take<unsigned char>(umma_gemm_apack_bytes(B, H));
      wpack = b.take<unsigned char>(umma_gemm_wpack_bytes(H, H));
    }
    bytes = b.off;
  }
};

// Training: the shapes and the path of the H x H GEMMs, then the maps of `saved` and of the workspace (sizing as above)
struct Plan {
  int B, J, H, S;
  bool tc;      // H x H GEMMs on the tensor cores in all three directions
  int Bp;       // the dW GEMM's K = B padded with zero rows to the K-block
  size_t bh;    // floats of one [B, H] array
  Plan(int batch, int num_joint, int hidden, int num_stage)
      : B(batch), J(num_joint), H(hidden), S(num_stage), tc(umma_gemm_supported(batch, hidden, hidden)),
        Bp(round_up(batch, 32)), bh((size_t)batch * hidden) {}
  int wide() const { return std::max(H, 3 * J); }
};
// `saved` as include/p2m_b200.h lays it out: y_0 .. y_S, z2 of each stage, the statistics of its bn1 and bn2
struct Saved {
  std::vector<float*> y, z2, stats;
  size_t bytes;
  Saved(void* base, const Plan& p) {
    Bump b(base);
    for (int s = 0; s <= p.S; ++s) y.push_back(b.take<float>(p.bh));
    for (int s = 0; s < p.S; ++s) z2.push_back(b.take<float>(p.bh));
    for (int i = 0; i < 8 * p.S; ++i) stats.push_back(b.take<float>(p.H));
    bytes = b.off;
  }
  // v: 0 mean, 1 invstd, 2 scale, 3 shift of BatchNorm `bn` (0, 1) of stage s
  float* stat(int s, int bn, int v) const { return stats[(s * 2 + bn) * 4 + v]; }
};
struct Work {
  float *g, *a, *t, *gT, *h64;
  double* sums;  // launch_bn_relu_bwd's scratch: 2 F doubles + 5 F floats
  float* g_scale;  // the tensor-core GEMMs' range normalisation of the gradient g and of the activation a
  float* a_scale;
  int* status;
  unsigned int* a_max;  // bn_relu_drop's max(a): zeroed with status at the start of a call, and by every use
  void *apack = nullptr, *wpack = nullptr;
  size_t bytes;
  Work(void* ws, const Plan& p) {
    Bump b(ws);
    g = b.take<float>(p.bh);
    a = b.take<float>(p.bh);
    t = b.take<float>(p.bh);
    gT = b.take<float>((size_t)p.wide() * p.B);
    h64 = b.take<float>((size_t)p.B * 64);
    sums = reinterpret_cast<double*>(b.take<char>((size_t)p.wide() * (2 * 8 + 5 * 4)));
    g_scale = b.take<float>(1);
    a_scale = b.take<float>(1);
    status = b.take<int>(2);
    a_max = reinterpret_cast<unsigned int*>(status + 1);
    if (p.tc) {
      apack = b.take<unsigned char>(std::max(umma_gemm_apack_bytes(p.B, p.H), umma_gemm_apack_bytes(p.H, p.Bp)));
      wpack = b.take<unsigned char>(std::max(umma_gemm_wpack_bytes(p.H, p.H), umma_gemm_wpack_bytes(p.H, p.Bp)));
    }
    bytes = b.off;
  }
};

// every pointer but the running statistics, which check_bn checks against each BatchNorm's options
bool params_ok(const p2m_posenet_params_t* P) {
  if (!P || P->num_joint <= 0 || P->hidden <= 0 || P->num_stage < 0 || !P->w1_w || !P->w1_b || !P->w2_w || !P->w2_b ||
      (P->num_stage > 0 && !P->stages))
    return false;
  for (int st = 0; st < P->num_stage; ++st) {
    const p2m_posenet_stage_t& S = P->stages[st];
    if (!S.w1_w || !S.w1_b || !S.w2_w || !S.w2_b || !S.bn1_w || !S.bn1_b || !S.bn2_w || !S.bn2_b) return false;
  }
  return true;
}

// The options of a call, resolved: one record per BatchNorm (stage s: bn1 at 2 s, bn2 at 2 s + 1) and one dropout p per
// stage, the caller's or the defaults
struct Modes {
  std::vector<p2m_bn_opts_t> bn;
  std::vector<float> p;
  bool batch_stats;  // some BatchNorm uses batch statistics (the defaults of a training call: always, also at 0 stages)
  Modes(int num_stage, const p2m_bn_opts_t* opts, int default_stats, const float* p_stage, float p_all)
      : bn(2 * (size_t)std::max(num_stage, 0), bn_opts_default(default_stats)),
        p((size_t)std::max(num_stage, 0), p_all), batch_stats(!opts && default_stats != P2M_BN_RUNNING) {
    for (size_t i = 0; opts && i < bn.size(); ++i) bn[i] = opts[i];
    for (size_t i = 0; p_stage && i < p.size(); ++i) p[i] = p_stage[i];
    for (const p2m_bn_opts_t& o : bn) batch_stats = batch_stats || o.stats != P2M_BN_RUNNING;
  }
  const p2m_bn_opts_t& of(int st, int which) const { return bn[2 * st + which]; }
};

// each BatchNorm's options against its buffers (extra: the num_batches_tracked pointers, may be null)
int check_bn(const char* where, const p2m_posenet_params_t* P, const p2m_posenet_train_t* extra, const Modes& md) {
  for (int st = 0; st < P->num_stage; ++st) {
    const p2m_posenet_stage_t& S = P->stages[st];
    const p2m_posenet_train_stage_t* X = extra ? &extra->stages[st] : nullptr;
    P2M_TRY(check_bn_opts(md.of(st, 0), S.bn1_rm, S.bn1_rv, X ? X->bn1_nbt : nullptr, where));
    P2M_TRY(check_bn_opts(md.of(st, 1), S.bn2_rm, S.bn2_rv, X ? X->bn2_nbt : nullptr, where));
  }
  return P2M_OK;
}

// forward: the options are checked against the buffers too (the backward reads the saved statistics, not them)
int check_call(const char* where, const p2m_posenet_params_t* P, const p2m_posenet_train_t* extra, bool forward, int B,
               const Modes& md, bool pointers_ok, size_t saved_bytes, size_t workspace_bytes) {
  bool p_ok = true;
  for (float p : md.p) p_ok = p_ok && p >= 0.f && p <= 1.f;
  if (!pointers_ok || !params_ok(P) || B <= 0 || !p_ok) {
    set_error(std::string(where) + ": bad argument");
    return P2M_ERR_INVALID;
  }
  if (forward) P2M_TRY(check_bn(where, P, extra, md));
  if (B < 2 && md.batch_stats) {
    set_error(std::string(where) + ": train-mode BatchNorm needs more than one value per channel (batch of 1)");
    return P2M_ERR_INVALID;
  }
  const Plan plan(B, P->num_joint, P->hidden, P->num_stage);
  if (saved_bytes < Saved(nullptr, plan).bytes || workspace_bytes < Work(nullptr, plan).bytes) {
    set_error(std::string(where) + ": saved or workspace buffer too small");
    return P2M_ERR_WORKSPACE;
  }
  return P2M_OK;
}

// The three H x H GEMMs, on the tensor cores or on the fp32 CUDA-core GEMM by the plan.
struct Gemms {
  const Plan& p;
  const Work& w;
  int sm_count;
  cudaStream_t s;
  // Y [B, H] = epilogue(X [B, H] W^T), X = the activation a whose range normalisation bn_relu_drop left in w.a_scale
  int forward(const float* X, const float* W, const Epilogue& e, float* Y) const {
    const int H = p.H;
    if (p.tc)
      return launch_umma_gemm({X, H, 1}, {W, H, 1}, p.B, H, H, e, Y, w.apack, w.wpack, w.status, sm_count, s, 0, 0,
                              w.a_scale);
    return launch_gemm(X, H, W, H, 0, Y, H, p.B, H, H, e, s);
  }
  // the gradient operand of the two backward GEMMs: its range normalisation (w.g_scale) for the tensor cores unless
  // the BN backward found it, transposed once (w.gT) for the CUDA-core dW
  int prepare(const float* g, bool have_scale) const {
    if (!p.tc) return transpose(g, p.B, p.H);
    if (!have_scale) P2M_TRY(launch_absmax_scale(g, (long long)p.bh, w.g_scale, s));
    return P2M_OK;
  }
  // dX [B, H] = g [B, H] W [H, H]
  int dx(const float* g, const float* W, float* dX) const {
    const int H = p.H;
    if (p.tc)
      return launch_umma_gemm({g, H, 1}, {W, 1, H}, p.B, H, H, Epilogue(), dX, w.apack, w.wpack, w.status, sm_count, s,
                              0, 0, w.g_scale);
    return launch_gemm(g, H, W, H, 1, dX, H, p.B, H, H, Epilogue(), s);
  }
  // dW [H, H] = g^T [H, B] a [B, H]: both operands range-normalised (a by bn_relu_drop)
  int dw(const float* g, const float* a, float* dW) const {
    const int H = p.H;
    if (p.tc)
      return launch_umma_gemm({g, 1, H}, {a, 1, H}, H, H, p.Bp, Epilogue(), dW, w.apack, w.wpack, w.status, sm_count,
                              s, 0, p.B, w.g_scale, w.a_scale);
    return launch_gemm(w.gT, p.B, a, H, 1, dW, H, H, H, p.B, Epilogue(), s);
  }
  int transpose(const float* in, int R, int C) const {
    k_pn_transpose<<<dim3((C + 31) / 32, (R + 31) / 32), 256, 0, s>>>(in, R, C, w.gT);
    P2M_LAUNCH_OK();
    return P2M_OK;
  }
};

// a = drop(relu(z * scale + shift)), and on the tensor-core path its range normalisation in w.a_scale
int bn_relu_drop(const float* z, const Plan& p, const Work& w, const float* scale, const float* shift, const Dropout& d,
                 float* a, cudaStream_t s) {
  unsigned int* amax = p.tc ? w.a_max : nullptr;
  k_pn_bn_relu_drop<<<blocks(((long long)p.bh + 3) / 4), 256, 0, s>>>(z, (long long)p.bh, p.H, scale, shift, d, a,
                                                                      amax);
  P2M_LAUNCH_OK();
  return amax ? launch_absmax_finish(amax, w.a_scale, s) : P2M_OK;
}

// Both forwards' output layer pose3d = y W2^T + b2, then pose_combine (unless null).  With tc and 3J <= 64 the K = H
// reduction runs on the tensor cores too, N padded to 64 zero-weight columns (h64), then 3J columns copied out + bias.
int output_layer(const p2m_posenet_params_t* P, const float* pose2d, const float* y, int B, bool tc, float* h64,
                 void* apack, void* wpack, int* status, int sm_count, float* pose3d, float* pose_combine, cudaStream_t s) {
  const int H = P->hidden, J = P->num_joint;
  if (tc && 3 * J <= 64) {
    P2M_TRY(launch_umma_gemm({y, H, 1}, {P->w2_w, H, 1}, B, 64, H, Epilogue(), h64, apack, wpack, status, sm_count, s,
                             3 * J));
    const long long n = (long long)B * 3 * J;
    k_take_cols<<<blocks(n), 256, 0, s>>>(h64, 64, P->w2_b, 3 * J, n, pose3d);
    P2M_LAUNCH_OK();
  } else {
    Epilogue e2;
    e2.bias = P->w2_b;
    P2M_TRY(launch_gemm(y, H, P->w2_w, H, 0, pose3d, 3 * J, B, 3 * J, H, e2, s));
  }
  if (pose_combine != nullptr) {
    const long long n = (long long)B * J;
    k_pose_combine<<<blocks(n), 256, 0, s>>>(pose2d, pose3d, n, pose_combine);
    P2M_LAUNCH_OK();
  }
  return P2M_OK;
}

}  // namespace

extern "C" {

size_t p2m_posenet_workspace_bytes(int batch, int hidden) {
  if (batch <= 0 || hidden <= 0) return 0;
  return EvalWork(nullptr, batch, hidden).bytes;
}

int p2m_posenet_forward(const p2m_posenet_params_t* P, const float* pose2d, float* pose3d, float* pose_combine, int B,
                        void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  return p2m_posenet_forward_opts(P, nullptr, pose2d, pose3d, pose_combine, B, workspace, workspace_bytes, stream);
}
int p2m_posenet_forward_opts(const p2m_posenet_params_t* P, const p2m_bn_opts_t* bn, const float* pose2d,
                             float* pose3d, float* pose_combine, int B, void* workspace, size_t workspace_bytes,
                             p2m_stream_t stream) {
  if (!params_ok(P) || !pose2d || !pose3d || B <= 0 || !workspace) {
    set_error("posenet_forward: bad argument");
    return P2M_ERR_INVALID;
  }
  const Modes md(P->num_stage, bn, P2M_BN_RUNNING, nullptr, 0.f);
  P2M_TRY(check_bn("posenet_forward", P, nullptr, md));
  if (md.batch_stats) {
    set_error("posenet_forward: the eval forward needs running statistics in every BatchNorm (P2M_BN_RUNNING)");
    return P2M_ERR_INVALID;
  }
  if (workspace_bytes < p2m_posenet_workspace_bytes(B, P->hidden)) {
    set_error("posenet_forward: workspace too small");
    return P2M_ERR_WORKSPACE;
  }
  int dev;
  P2M_TRY(arrays_device("posenet_forward", {pose2d, pose3d, pose_combine, workspace}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int H = P->hidden, J = P->num_joint;
  EvalWork w(workspace, B, H);
  int sm_count = 132;
  if (w.tc) {
    P2M_CUDA_OK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev));
    P2M_CUDA_OK(cudaMemsetAsync(w.status, 0, sizeof(int), s));
  }
  auto big_gemm = [&](const float* X, const float* Wm, const Epilogue& e, float* Y) -> int {
    if (w.tc) return launch_umma_gemm({X, H, 1}, {Wm, H, 1}, B, H, H, e, Y, w.apack, w.wpack, w.status, sm_count, s);
    return launch_gemm(X, H, Wm, H, 0, Y, H, B, H, H, e, s);
  };
  Epilogue e1;
  e1.bias = P->w1_b;
  P2M_TRY(launch_gemm(pose2d, 2 * J, P->w1_w, 2 * J, 0, w.y, H, B, H, 2 * J, e1, s));
  for (int st = 0; st < P->num_stage; ++st) {
    const p2m_posenet_stage_t& S = P->stages[st];
    // a = relu(bn1(y))
    const long long n = (long long)B * H;
    k_bn_relu_rows<<<blocks(n), 256, 0, s>>>(w.y, n, H, S.bn1_w, S.bn1_b, S.bn1_rm, S.bn1_rv, (float)md.of(st, 0).eps,
                                             w.a);
    P2M_LAUNCH_OK();
    // h = relu(bn2(a Wa^T + ba)): BatchNorm folded into the GEMM epilogue
    P2M_TRY(launch_bn_fold_eval(S.bn2_w, S.bn2_b, S.bn2_rm, S.bn2_rv, S.w1_b, md.of(st, 1).eps, w.sc, w.sc + H, H, s));
    Epilogue ea;
    ea.scale = w.sc;
    ea.shift = w.sc + H;
    ea.relu = 1;
    P2M_TRY(big_gemm(w.a, S.w1_w, ea, w.h));
    // y' = y + h Wb^T + bb  (written to `a`, then the buffers swap roles)
    Epilogue eb;
    eb.bias = S.w2_b;
    eb.res = w.y;
    eb.res_F = H;
    P2M_TRY(big_gemm(w.h, S.w2_w, eb, w.a));
    std::swap(w.y, w.a);
  }
  return output_layer(P, pose2d, w.y, B, w.tc, w.h, w.apack, w.wpack, w.status, sm_count, pose3d, pose_combine, s);
}

size_t p2m_posenet_train_workspace_bytes(int batch, int num_joint, int hidden, int num_stage) {
  if (batch <= 0 || num_joint <= 0 || hidden <= 0 || num_stage < 0) return 0;
  return Work(nullptr, Plan(batch, num_joint, hidden, num_stage)).bytes;
}
size_t p2m_posenet_train_saved_bytes(int batch, int num_joint, int hidden, int num_stage) {
  if (batch <= 0 || num_joint <= 0 || hidden <= 0 || num_stage < 0) return 0;
  return Saved(nullptr, Plan(batch, num_joint, hidden, num_stage)).bytes;
}

}  // extern "C"

namespace {
int train_forward(const p2m_posenet_params_t* P, const p2m_posenet_train_t* extra, const Modes& md, const float* pose2d,
                  int B, const int64_t* seed, float* pose3d, float* pose_combine, void* saved, size_t saved_bytes,
                  void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  const bool extra_ok = !P || P->num_stage == 0 || (extra && extra->stages);
  P2M_TRY(check_call("posenet_train_forward", P, extra_ok ? extra : nullptr, true, B, md,
                     pose2d && seed && pose3d && saved && workspace && extra_ok, saved_bytes, workspace_bytes));
  int dev;
  P2M_TRY(arrays_device("posenet_train_forward", {pose2d, seed, pose3d, pose_combine, saved, workspace}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const Plan plan(B, P->num_joint, P->hidden, P->num_stage);
  const Saved sv(saved, plan);
  const Work w(workspace, plan);
  const int H = plan.H, J = plan.J;
  Gemms gemm{plan, w, 132, s};
  if (plan.tc) {
    P2M_CUDA_OK(cudaDeviceGetAttribute(&gemm.sm_count, cudaDevAttrMultiProcessorCount, dev));
    P2M_CUDA_OK(cudaMemsetAsync(w.status, 0, 2 * sizeof(int), s));  // status and a_max
  }
  Epilogue e1;
  e1.bias = P->w1_b;
  P2M_TRY(launch_gemm(pose2d, 2 * J, P->w1_w, 2 * J, 0, sv.y[0], H, B, H, 2 * J, e1, s));
  for (int st = 0; st < plan.S; ++st) {
    const p2m_posenet_stage_t& S = P->stages[st];
    const p2m_posenet_train_stage_t& X = extra->stages[st];
    const float* y = sv.y[st];
    // a = drop(relu(bn1(y)))
    P2M_TRY(launch_bn_stats(y, B, H, S.bn1_w, S.bn1_b, const_cast<float*>(S.bn1_rm), const_cast<float*>(S.bn1_rv),
                            X.bn1_nbt, md.of(st, 0), w.sums, sv.stat(st, 0, 0), sv.stat(st, 0, 1), sv.stat(st, 0, 2),
                            sv.stat(st, 0, 3), s));
    P2M_TRY(bn_relu_drop(y, plan, w, sv.stat(st, 0, 2), sv.stat(st, 0, 3), make_dropout(md.p[st], seed, 2 * st), w.a,
                         s));
    // z2 = a Wa^T + ba;  a = drop(relu(bn2(z2)))
    Epilogue ea;
    ea.bias = S.w1_b;
    P2M_TRY(gemm.forward(w.a, S.w1_w, ea, sv.z2[st]));
    P2M_TRY(launch_bn_stats(sv.z2[st], B, H, S.bn2_w, S.bn2_b, const_cast<float*>(S.bn2_rm),
                            const_cast<float*>(S.bn2_rv), X.bn2_nbt, md.of(st, 1), w.sums, sv.stat(st, 1, 0),
                            sv.stat(st, 1, 1), sv.stat(st, 1, 2), sv.stat(st, 1, 3), s));
    P2M_TRY(bn_relu_drop(sv.z2[st], plan, w, sv.stat(st, 1, 2), sv.stat(st, 1, 3),
                         make_dropout(md.p[st], seed, 2 * st + 1), w.a, s));
    // y' = y + a Wb^T + bb
    Epilogue eb;
    eb.bias = S.w2_b;
    eb.res = y;
    eb.res_F = H;
    P2M_TRY(gemm.forward(w.a, S.w2_w, eb, sv.y[st + 1]));
  }
  return output_layer(P, pose2d, sv.y[plan.S], B, plan.tc, w.h64, w.apack, w.wpack, w.status, gemm.sm_count, pose3d,
                      pose_combine, s);
}

// p2m_debug_posenet_backward_capture: n floats of src into dst, if the caller asked for that tensor
int capture_copy(float* dst, const float* src, size_t n, cudaStream_t s) {
  if (dst == nullptr) return P2M_OK;
  P2M_CUDA_OK(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return P2M_OK;
}
float* capture_slot(float* const* v, int st) { return v ? v[st] : nullptr; }

// cap (may be null): the debug capture of the backward's intermediates; null issues no copies
int backward(const p2m_posenet_params_t* P, const Modes& md, const float* pose2d, int B, const int64_t* seed,
             const void* saved, size_t saved_bytes, const float* d_pose3d, const p2m_posenet_grads_t* G,
             float* d_pose2d, void* workspace, size_t workspace_bytes, p2m_stream_t stream,
             const p2m_posenet_capture_t* cap) {
  bool ok = pose2d && seed && saved && d_pose3d && workspace && G && G->w1_w && G->w1_b && G->w2_w && G->w2_b && P &&
            (P->num_stage <= 0 || G->stages);
  for (int st = 0; ok && st < P->num_stage; ++st) {
    const p2m_posenet_stage_grads_t& g = G->stages[st];
    ok = g.w1_w && g.w1_b && g.w2_w && g.w2_b && g.bn1_w && g.bn1_b && g.bn2_w && g.bn2_b;
  }
  P2M_TRY(check_call("posenet_backward", P, nullptr, false, B, md, ok, saved_bytes, workspace_bytes));
  int dev;
  P2M_TRY(arrays_device("posenet_backward", {pose2d, seed, saved, d_pose3d, d_pose2d, workspace}, &dev));
  DeviceGuard guard(dev);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const Plan plan(B, P->num_joint, P->hidden, P->num_stage);
  const Saved sv(const_cast<void*>(saved), plan);
  const Work w(workspace, plan);
  const int H = plan.H, J = plan.J;
  const long long n = (long long)plan.bh;
  Gemms gemm{plan, w, 132, s};
  if (plan.tc) {
    P2M_CUDA_OK(cudaDeviceGetAttribute(&gemm.sm_count, cudaDevAttrMultiProcessorCount, dev));
    P2M_CUDA_OK(cudaMemsetAsync(w.status, 0, 2 * sizeof(int), s));  // status and a_max
  }
  // output layer (thin: fp32): db2, dW2 = d_pose3d^T y_S, g = d_pose3d W2
  P2M_TRY(launch_col_sum(d_pose3d, B, 3 * J, w.sums, G->w2_b, s));
  P2M_TRY(gemm.transpose(d_pose3d, B, 3 * J));
  P2M_TRY(launch_gemm(w.gT, B, sv.y[plan.S], H, 1, G->w2_w, H, 3 * J, H, B, Epilogue(), s));
  P2M_TRY(launch_gemm(d_pose3d, 3 * J, P->w2_w, H, 1, w.g, H, B, H, 3 * J, Epilogue(), s));
  for (int st = plan.S - 1; st >= 0; --st) {
    const p2m_posenet_stage_t& S = P->stages[st];
    const p2m_posenet_stage_grads_t& D = G->stages[st];
    const Dropout d1 = make_dropout(md.p[st], seed, 2 * st), d2 = make_dropout(md.p[st], seed, 2 * st + 1);
    const int frozen1 = md.of(st, 0).stats == P2M_BN_RUNNING, frozen2 = md.of(st, 1).stats == P2M_BN_RUNNING;
    // the four range normalisations of the stage's tensor-core GEMMs: a2, g_y, a1, g_z2
    float* cap_scale = cap && plan.tc ? capture_slot(cap->scale, st) : nullptr;
    auto cap_scale_copy = [&](int i, const float* sc) { return capture_copy(cap_scale ? cap_scale + i : nullptr, sc, 1, s); };
    if (cap) P2M_TRY(capture_copy(capture_slot(cap->g_y, st), w.g, n, s));
    // second Linear: y' = y + a2 Wb^T + bb with a2 = drop(relu(bn2(z2))) recomputed; g = dL/dy'
    P2M_TRY(launch_col_sum(w.g, B, H, w.sums, D.w2_b, s));
    P2M_TRY(bn_relu_drop(sv.z2[st], plan, w, sv.stat(st, 1, 2), sv.stat(st, 1, 3), d2, w.a, s));
    if (cap) {
      P2M_TRY(capture_copy(capture_slot(cap->a2, st), w.a, n, s));
      P2M_TRY(cap_scale_copy(0, w.a_scale));
    }
    P2M_TRY(gemm.prepare(w.g, false));
    if (cap) P2M_TRY(cap_scale_copy(1, w.g_scale));
    P2M_TRY(gemm.dw(w.g, w.a, D.w2_w));
    P2M_TRY(gemm.dx(w.g, S.w2_w, w.t));
    if (cap) P2M_TRY(capture_copy(capture_slot(cap->g_a2, st), w.t, n, s));
    // through drop, ReLU and bn2: t = dL/dz2 (its fp16-range scale found in the same pass on the tensor-core path)
    k_pn_drop_bwd<<<blocks((n + 3) / 4), 256, 0, s>>>(w.t, n, d2);
    P2M_LAUNCH_OK();
    P2M_TRY(launch_bn_relu_bwd(sv.z2[st], w.t, B, H, S.bn2_w, sv.stat(st, 1, 2), sv.stat(st, 1, 3), sv.stat(st, 1, 0),
                               sv.stat(st, 1, 1), 1, w.sums, D.bn2_w, D.bn2_b, w.t, s, plan.tc ? w.g_scale : nullptr,
                               frozen2));
    if (cap) {
      P2M_TRY(capture_copy(capture_slot(cap->g_z2, st), w.t, n, s));
      P2M_TRY(cap_scale_copy(3, w.g_scale));
    }
    // first Linear: z2 = a1 Wa^T + ba with a1 = drop(relu(bn1(y))) recomputed
    P2M_TRY(launch_col_sum(w.t, B, H, w.sums, D.w1_b, s));
    P2M_TRY(bn_relu_drop(sv.y[st], plan, w, sv.stat(st, 0, 2), sv.stat(st, 0, 3), d1, w.a, s));
    if (cap) {
      P2M_TRY(capture_copy(capture_slot(cap->a1, st), w.a, n, s));
      P2M_TRY(cap_scale_copy(2, w.a_scale));
    }
    P2M_TRY(gemm.prepare(w.t, true));
    P2M_TRY(gemm.dw(w.t, w.a, D.w1_w));
    P2M_TRY(gemm.dx(w.t, S.w1_w, w.a));
    if (cap) P2M_TRY(capture_copy(capture_slot(cap->g_a1, st), w.a, n, s));
    // through drop, ReLU and bn1, plus the residual branch: g += dL/dy
    k_pn_drop_bwd<<<blocks((n + 3) / 4), 256, 0, s>>>(w.a, n, d1);
    P2M_LAUNCH_OK();
    P2M_TRY(launch_bn_relu_bwd(sv.y[st], w.a, B, H, S.bn1_w, sv.stat(st, 0, 2), sv.stat(st, 0, 3), sv.stat(st, 0, 0),
                               sv.stat(st, 0, 1), 1, w.sums, D.bn1_w, D.bn1_b, w.a, s, nullptr, frozen1));
    if (cap) P2M_TRY(capture_copy(capture_slot(cap->g_bn1, st), w.a, n, s));
    k_pn_add<<<blocks(n), 256, 0, s>>>(w.g, w.a, n);
    P2M_LAUNCH_OK();
  }
  if (cap) P2M_TRY(capture_copy(cap->g_y0, w.g, n, s));
  // input layer (thin: fp32): db1, dW1 = g^T pose2d, d_pose2d = g W1
  P2M_TRY(launch_col_sum(w.g, B, H, w.sums, G->w1_b, s));
  P2M_TRY(gemm.transpose(w.g, B, H));
  P2M_TRY(launch_gemm(w.gT, B, pose2d, 2 * J, 1, G->w1_w, 2 * J, H, 2 * J, B, Epilogue(), s));
  if (d_pose2d != nullptr)
    P2M_TRY(launch_gemm(w.g, H, P->w1_w, 2 * J, 1, d_pose2d, 2 * J, B, 2 * J, H, Epilogue(), s));
  return P2M_OK;
}
}  // namespace

extern "C" {

int p2m_posenet_train_forward(const p2m_posenet_params_t* P, const p2m_posenet_train_t* extra, const float* pose2d, int B,
                              float p_dropout, const int64_t* seed, float* pose3d, float* pose_combine, void* saved,
                              size_t saved_bytes, void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  const Modes md(P ? P->num_stage : 0, nullptr, P2M_BN_BATCH_UPDATE, nullptr, p_dropout);
  return train_forward(P, extra, md, pose2d, B, seed, pose3d, pose_combine, saved, saved_bytes, workspace,
                       workspace_bytes, stream);
}
int p2m_posenet_train_forward_opts(const p2m_posenet_params_t* P, const p2m_posenet_train_t* extra,
                                   const p2m_bn_opts_t* bn, const float* p_dropout, const float* pose2d, int B,
                                   const int64_t* seed, float* pose3d, float* pose_combine, void* saved,
                                   size_t saved_bytes, void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  const Modes md(P ? P->num_stage : 0, bn, P2M_BN_BATCH_UPDATE, p_dropout, 0.f);
  return train_forward(P, extra, md, pose2d, B, seed, pose3d, pose_combine, saved, saved_bytes, workspace,
                       workspace_bytes, stream);
}
int p2m_posenet_backward(const p2m_posenet_params_t* P, const float* pose2d, int B, float p_dropout, const int64_t* seed,
                         const void* saved, size_t saved_bytes, const float* d_pose3d, const p2m_posenet_grads_t* G,
                         float* d_pose2d, void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  const Modes md(P ? P->num_stage : 0, nullptr, P2M_BN_BATCH_UPDATE, nullptr, p_dropout);
  return backward(P, md, pose2d, B, seed, saved, saved_bytes, d_pose3d, G, d_pose2d, workspace, workspace_bytes, stream,
                  nullptr);
}
int p2m_posenet_backward_opts(const p2m_posenet_params_t* P, const p2m_bn_opts_t* bn, const float* p_dropout,
                              const float* pose2d, int B, const int64_t* seed, const void* saved, size_t saved_bytes,
                              const float* d_pose3d, const p2m_posenet_grads_t* G, float* d_pose2d, void* workspace,
                              size_t workspace_bytes, p2m_stream_t stream) {
  const Modes md(P ? P->num_stage : 0, bn, P2M_BN_BATCH_UPDATE, p_dropout, 0.f);
  return backward(P, md, pose2d, B, seed, saved, saved_bytes, d_pose3d, G, d_pose2d, workspace, workspace_bytes, stream,
                  nullptr);
}

int p2m_debug_posenet_backward_capture(const p2m_posenet_params_t* P, const p2m_bn_opts_t* bn, const float* p_dropout,
                                       const float* pose2d, int B, const int64_t* seed, const void* saved,
                                       size_t saved_bytes, const float* d_pose3d, const p2m_posenet_grads_t* G,
                                       float* d_pose2d, void* workspace, size_t workspace_bytes,
                                       const p2m_posenet_capture_t* capture, p2m_stream_t stream) {
  const Modes md(P ? P->num_stage : 0, bn, P2M_BN_BATCH_UPDATE, p_dropout, 0.f);
  return backward(P, md, pose2d, B, seed, saved, saved_bytes, d_pose3d, G, d_pose2d, workspace, workspace_bytes, stream,
                  capture);
}

}  // extern "C"
