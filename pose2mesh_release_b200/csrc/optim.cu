// The RMSprop step (torch.optim.RMSprop) over a list of parameter tensors in one launch per 448 tensors: each element
// of p, g and the optimizer state is read once and written once, in fp32, in torch's _multi_tensor_rmsprop operation
// order.  The segment table travels as a __grid_constant__ kernel parameter, so a captured graph keeps its own copy.
#include <cuda_runtime.h>

#include <cmath>
#include <string>
#include <vector>

#include "p2m_internal.h"

namespace p2m {
namespace {

constexpr int RMS_THREADS = 256;
constexpr int RMS_VEC_PER_THREAD = 4;                                        // float4 per thread and array
constexpr long long RMS_CHUNK = (long long)RMS_THREADS * RMS_VEC_PER_THREAD * 4;  // elements per CTA: 4096
constexpr int RMS_MAX_SEG = 448;   // segments per launch: the table below is 29.3 KB of the 32 764 B of parameters
constexpr int RMS_MAX_GROUP = 16;  // hyperparameter groups per launch

struct RmsSeg {
  float* p;
  const float* g;
  float* s;
  float* buf;   // momentum_buffer (group momentum > 0)
  float* ga;    // grad_avg (centred group)
  float* step;  // the state's step counter (nullable): +1 by the segment's first CTA
  long long n;
  int group;
  int first_block;  // the segment's CTAs are [first_block, next segment's first_block)
};
struct RmsGroup {
  const float* lr_ptr;  // device lr, read at run time (nullable: lr below)
  float lr, alpha, one_minus_alpha, eps, wd, momentum;
  int centered, use_momentum;  // use_momentum: momentum > 0 in double, as torch decides it
};
struct RmsTable {
  int n_seg;
  RmsGroup grp[RMS_MAX_GROUP];
  RmsSeg seg[RMS_MAX_SEG];
};
static_assert(sizeof(RmsTable) <= 32764, "the segment table must fit the kernel parameter space");

struct RmsHp {
  float neg_lr, alpha, oma, eps, wd, momentum;
  bool centered, use_momentum, use_wd;
};

// torch's lerp (ATen/native/Lerp.h): self + w (end - self) for |w| < 0.5, else end - (end - self)(1 - w)
__device__ __forceinline__ float lerp_torch(float self, float end, float w) {
  return fabsf(w) < 0.5f ? __fmaf_rn(w, __fsub_rn(end, self), self)
                         : __fsub_rn(end, __fmul_rn(__fsub_rn(end, self), __fsub_rn(1.f, w)));
}

// One element.  Each line is one of torch's foreach ops on fp32 (a + alpha * op(b, c) contracts to one fma):
//   _foreach_add(g, p, alpha=wd) ; _foreach_mul_(s, alpha) ; _foreach_addcmul_(s, g, g, 1 - alpha) ;
//   centred: _foreach_lerp_(ga, g, 1 - alpha), _foreach_addcmul(s, ga, ga, -1) ; _foreach_sqrt ; _foreach_add_(eps) ;
//   momentum: _foreach_mul_(buf, mu), _foreach_addcdiv_(buf, g, avg), _foreach_add_(p, buf, alpha=-lr) ;
//   else: _foreach_addcdiv_(p, g, avg, value=-lr)
__device__ __forceinline__ void rms_element(float& p, float g, float& s, float& buf, float& ga, const RmsHp& h) {
  if (h.use_wd) g = __fmaf_rn(h.wd, p, g);
  s = __fmul_rn(s, h.alpha);
  s = __fmaf_rn(h.oma, __fmul_rn(g, g), s);
  float v = s;
  if (h.centered) {
    ga = lerp_torch(ga, g, h.oma);
    v = __fmaf_rn(-1.f, __fmul_rn(ga, ga), s);
  }
  const float avg = __fadd_rn(__fsqrt_rn(v), h.eps);
  const float q = __fdiv_rn(g, avg);
  if (h.use_momentum) {
    buf = __fmul_rn(buf, h.momentum);
    buf = __fadd_rn(buf, q);
    p = __fmaf_rn(h.neg_lr, buf, p);
  } else {
    p = __fmaf_rn(h.neg_lr, q, p);
  }
}

__device__ __forceinline__ void rms_scalar(const RmsSeg& sg, long long i, const RmsHp& h) {
  float p = sg.p[i], s = sg.s[i];
  float buf = h.use_momentum ? sg.buf[i] : 0.f, ga = h.centered ? sg.ga[i] : 0.f;
  rms_element(p, sg.g[i], s, buf, ga, h);
  sg.p[i] = p;
  sg.s[i] = s;
  if (h.use_momentum) sg.buf[i] = buf;
  if (h.centered) sg.ga[i] = ga;
}

__device__ __forceinline__ unsigned addr16(const void* p) { return (unsigned)(reinterpret_cast<uintptr_t>(p) & 15u); }

// Vector path: the elements before the first 16-byte boundary (head, < 4) and after the last whole float4 (tail) go
// through rms_scalar in the segment's first and last CTA; used when every array of the segment has the same address
// modulo 16.  Otherwise every element goes through rms_scalar (coalesced 4-byte accesses).
__global__ void __launch_bounds__(RMS_THREADS) k_rmsprop_step(const __grid_constant__ RmsTable t) {
  const int b = blockIdx.x;
  int lo = 0, hi = t.n_seg - 1;  // the last segment whose first_block <= b
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.seg[mid].first_block <= b) lo = mid;
    else hi = mid - 1;
  }
  const RmsSeg& sg = t.seg[lo];
  const RmsGroup& gr = t.grp[sg.group];
  const long long chunk = b - sg.first_block;
  RmsHp h;
  h.neg_lr = -(gr.lr_ptr ? *gr.lr_ptr : gr.lr);
  h.alpha = gr.alpha;
  h.oma = gr.one_minus_alpha;
  h.eps = gr.eps;
  h.wd = gr.wd;
  h.momentum = gr.momentum;
  h.centered = gr.centered != 0;
  h.use_momentum = gr.use_momentum != 0;
  h.use_wd = gr.wd != 0.f;
  if (chunk == 0 && threadIdx.x == 0 && sg.step) *sg.step = *sg.step + 1.f;

  const unsigned a = addr16(sg.p);
  const bool vec = addr16(sg.g) == a && addr16(sg.s) == a && (!h.use_momentum || addr16(sg.buf) == a) &&
                   (!h.centered || addr16(sg.ga) == a);
  const long long n = sg.n;
  if (!vec) {
    const long long end = min(n, (chunk + 1) * RMS_CHUNK);
    for (long long i = chunk * RMS_CHUNK + threadIdx.x; i < end; i += RMS_THREADS) rms_scalar(sg, i, h);
    return;
  }
  const long long head = min(n, (long long)((16u - a) & 15u) / 4);
  const long long nv = (n - head) / 4;
  const long long n_chunks = max(1LL, (nv + RMS_CHUNK / 4 - 1) / (RMS_CHUNK / 4));
  if (chunk == 0 && threadIdx.x < head) rms_scalar(sg, threadIdx.x, h);
  if (chunk == n_chunks - 1) {
    const long long i = head + 4 * nv + threadIdx.x;
    if (i < n) rms_scalar(sg, i, h);
  }
  float4* p4 = reinterpret_cast<float4*>(sg.p + head);
  const float4* g4 = reinterpret_cast<const float4*>(sg.g + head);
  float4* s4 = reinterpret_cast<float4*>(sg.s + head);
  float4* b4 = h.use_momentum ? reinterpret_cast<float4*>(sg.buf + head) : nullptr;
  float4* a4 = h.centered ? reinterpret_cast<float4*>(sg.ga + head) : nullptr;
  const long long v0 = chunk * (RMS_CHUNK / 4) + threadIdx.x;
  float4 P[RMS_VEC_PER_THREAD], G[RMS_VEC_PER_THREAD], S[RMS_VEC_PER_THREAD], B[RMS_VEC_PER_THREAD],
      A[RMS_VEC_PER_THREAD];
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int j = 0; j < RMS_VEC_PER_THREAD; ++j) {  // every load first: 3 to 5 x 4 float4 in flight per thread
    const long long v = v0 + (long long)j * RMS_THREADS;
    const bool on = v < nv;
    P[j] = on ? p4[v] : z;
    G[j] = on ? __ldg(g4 + v) : z;
    S[j] = on ? s4[v] : z;
    B[j] = on && b4 ? b4[v] : z;
    A[j] = on && a4 ? a4[v] : z;
  }
#pragma unroll
  for (int j = 0; j < RMS_VEC_PER_THREAD; ++j) {
    const long long v = v0 + (long long)j * RMS_THREADS;
    if (v >= nv) continue;
    rms_element(P[j].x, G[j].x, S[j].x, B[j].x, A[j].x, h);
    rms_element(P[j].y, G[j].y, S[j].y, B[j].y, A[j].y, h);
    rms_element(P[j].z, G[j].z, S[j].z, B[j].z, A[j].z, h);
    rms_element(P[j].w, G[j].w, S[j].w, B[j].w, A[j].w, h);
    p4[v] = P[j];
    s4[v] = S[j];
    if (b4) b4[v] = B[j];
    if (a4) a4[v] = A[j];
  }
}

// CTAs the segment takes: one per RMS_CHUNK elements of its vector body (or of the segment on the scalar path), at
// least one (a segment of head and tail only, or an empty one that still advances its step)
long long rms_blocks(const p2m_rmsprop_segment_t& s, const p2m_rmsprop_group_t& g) {
  auto a16 = [](const void* p) { return (unsigned)(reinterpret_cast<uintptr_t>(p) & 15u); };
  const unsigned a = a16(s.param);
  const bool vec = a16(s.grad) == a && a16(s.square_avg) == a && (g.momentum <= 0 || a16(s.momentum_buffer) == a) &&
                   (!g.centered || a16(s.grad_avg) == a);
  long long work = s.numel;
  if (vec) {
    const long long head = std::min<long long>(s.numel, ((16u - a) & 15u) / 4);
    work = (s.numel - head) / 4 * 4;
  }
  return std::max(1LL, (work + RMS_CHUNK - 1) / RMS_CHUNK);
}

bool finite_nonneg(double v) { return std::isfinite(v) && v >= 0; }

}  // namespace
}  // namespace p2m

using namespace p2m;

extern "C" {

int p2m_rmsprop_step(const p2m_rmsprop_segment_t* segments, int n_segments, const p2m_rmsprop_group_t* groups,
                     int n_groups, p2m_stream_t stream) {
  if (n_segments < 0 || (n_segments > 0 && (!segments || !groups || n_groups <= 0))) {
    set_error("rmsprop_step: null table, n_segments < 0 or no groups");
    return P2M_ERR_INVALID;
  }
  if (n_segments == 0) return P2M_OK;
  for (int k = 0; k < n_groups; ++k) {
    const p2m_rmsprop_group_t& g = groups[k];
    if ((!g.lr_device && !std::isfinite(g.lr)) || !finite_nonneg(g.alpha) || !finite_nonneg(g.eps) ||
        !finite_nonneg(g.weight_decay) || !finite_nonneg(g.momentum) || (g.centered != 0 && g.centered != 1)) {
      set_error("rmsprop_step: group " + std::to_string(k) +
                ": lr must be finite, alpha, eps, weight_decay and momentum finite and >= 0, centered 0 or 1");
      return P2M_ERR_INVALID;
    }
  }
  std::vector<const void*> arrays;
  arrays.reserve((size_t)n_segments * 6 + n_groups);
  for (int k = 0; k < n_groups; ++k) arrays.push_back(groups[k].lr_device);
  for (int i = 0; i < n_segments; ++i) {
    const p2m_rmsprop_segment_t& s = segments[i];
    if (s.group < 0 || s.group >= n_groups || s.numel < 0) {
      set_error("rmsprop_step: segment " + std::to_string(i) + ": group index out of range or numel < 0");
      return P2M_ERR_INVALID;
    }
    const p2m_rmsprop_group_t& g = groups[s.group];
    const void* need[] = {s.param, s.grad, s.square_avg, g.momentum > 0 ? s.momentum_buffer : s.param,
                          g.centered ? s.grad_avg : s.param};
    bool ok = true;
    for (const void* p : need) ok = ok && p && (reinterpret_cast<uintptr_t>(p) & 3u) == 0;
    if (!ok) {
      set_error("rmsprop_step: segment " + std::to_string(i) +
                ": param, grad, square_avg (and momentum_buffer / grad_avg where the group uses them) must be "
                "non-null, 4-byte aligned float arrays");
      return P2M_ERR_INVALID;
    }
    arrays.insert(arrays.end(), {s.param, s.grad, s.square_avg, g.momentum > 0 ? s.momentum_buffer : nullptr,
                                 g.centered ? s.grad_avg : nullptr, s.step});
  }
  int dev;
  P2M_TRY(arrays_device("rmsprop_step", arrays.data(), arrays.size(), &dev));
  DeviceGuard guard(dev);
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  // Segments in order, as many per launch as the table holds (RMS_MAX_SEG, and RMS_MAX_GROUP distinct groups)
  RmsTable t;
  std::vector<int> local(n_groups);
  int i = 0;
  while (i < n_segments) {
    t.n_seg = 0;
    int n_grp = 0;
    std::fill(local.begin(), local.end(), -1);
    long long blocks = 0;
    for (; i < n_segments && t.n_seg < RMS_MAX_SEG; ++i) {
      const p2m_rmsprop_segment_t& s = segments[i];
      const p2m_rmsprop_group_t& g = groups[s.group];
      if (local[s.group] < 0) {
        if (n_grp == RMS_MAX_GROUP) break;
        RmsGroup& d = t.grp[n_grp];
        d.lr_ptr = static_cast<const float*>(g.lr_device);
        d.lr = (float)g.lr;
        d.alpha = (float)g.alpha;
        d.one_minus_alpha = (float)(1.0 - g.alpha);  // torch: value = 1 - alpha in Python (double), then fp32
        d.eps = (float)g.eps;
        d.wd = (float)g.weight_decay;
        d.momentum = (float)g.momentum;
        d.centered = g.centered;
        d.use_momentum = g.momentum > 0;
        local[s.group] = n_grp++;
      }
      const long long nb = rms_blocks(s, g);
      if (blocks + nb > 0x7fffffffLL) {
        if (t.n_seg == 0) {
          set_error("rmsprop_step: segment " + std::to_string(i) + " needs more than 2^31 - 1 CTAs");
          return P2M_ERR_INVALID;
        }
        break;
      }
      RmsSeg& d = t.seg[t.n_seg++];
      d.p = s.param;
      d.g = s.grad;
      d.s = s.square_avg;
      d.buf = g.momentum > 0 ? s.momentum_buffer : nullptr;
      d.ga = g.centered ? s.grad_avg : nullptr;
      d.step = s.step;
      d.n = s.numel;
      d.group = local[s.group];
      d.first_block = (int)blocks;
      blocks += nb;
    }
    k_rmsprop_step<<<(unsigned)blocks, RMS_THREADS, 0, st>>>(t);
    P2M_LAUNCH_OK();
  }
  return P2M_OK;
}

}  // extern "C"
