// Row f12 of SURVEY.md §8: the network inputs of a training sample on the device, the train branch of the datasets'
// replace_joint_img (data/Human36M/dataset.py:436-445) and the crop / normalisation around it (:359-392):
//  * synthesize_pose (lib/noise_utils.py:17-285; num_overlap = 0, so no swap sources) on the COCO joints;
//  * generate_syn_error (data/Human36M/dataset.py:143-155) on the Human3.6M joints;
// and row f13, the sample's augmentation: augm_params (lib/aug_utils.py:98-117) and the rotation / flip of the crop.
// The random stream is include/p2m_b200.h's counter-based rule; DESIGN.md §4.3 (dataset inputs) argues the device's
// shortcuts (first survivor instead of a uniform survivor, the miss pick as a two-pass mixture) are exact in
// distribution.  Every loop is bounded by the reference's draw count.  Candidate geometry is fp64 with explicitly
// rounded operations, so that oracle/inputs_oracle.py restates it to rounding of the math library's sin / cos / log.
#include <cuda_runtime.h>

#include "p2m_internal.h"

using namespace p2m;

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int N_KPS = 17, N_DRAW = 500;
constexpr int SYNTH_THREADS = 9 * 32;  // one warp per joint of phase 1: joints 0, 1, 3, .., 15
// stream purposes: stream id = 16 joint + purpose
enum : unsigned { JITTER = 0, GOOD = 1, INV = 2, MISS_GT = 3, MISS_INV = 4, MISS_PICK = 5, CHOICE = 6, GAUSS = 7,
                  KEEP = 8 };
// cfg.kps_sigmas * 10 (lib/noise_utils.py:9-11), the COCO benchmark's OKS constants
__constant__ double KPS_SIGMAS_X10[N_KPS] = {.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87,
                                             .87, .89, .89};
// np.log(0.10), np.log(0.50), np.log(0.85)
constexpr double LN_010 = -2.3025850929940455, LN_050 = -0.6931471805599453, LN_085 = -0.16251892949777494;

struct ErrTable {  // by value in the kernel parameters
  p2m_h36m_error_t e[N_KPS];
};

struct Stream {
  uint2 key;       // seed[0]
  unsigned s1, b;  // low 32 bits of seed[1]; the sample index
};
__device__ __forceinline__ Stream make_stream(const long long* seed, unsigned b) {
  const unsigned long long s0 = (unsigned long long)seed[0];
  return Stream{make_uint2((unsigned)s0, (unsigned)(s0 >> 32)), (unsigned)seed[1], b};
}
__device__ __forceinline__ double u53(unsigned hi, unsigned lo) {
  return ((double)(hi >> 5) * 67108864.0 + (double)(lo >> 6)) * (1.0 / 9007199254740992.0);
}
// the two uniforms on [0, 1) of counter (d, sid, b, seed[1])
__device__ __forceinline__ double2 uniforms(const Stream& s, unsigned d, unsigned sid) {
  const uint4 w = philox4x32_10(make_uint4(d, sid, s.b, s.s1), s.key);
  return make_double2(u53(w.x, w.y), u53(w.z, w.w));
}
// floor(u n) clamped to n - 1 (u n can round up to n)
__device__ __forceinline__ int pick_index(double u, int n) {
  const int k = (int)floor(__dmul_rn(u, (double)n));
  return k < n - 1 ? k : n - 1;
}

// draw d of stream sid: angle ~ U(0, 2 pi), r ~ U(rlo, rhi) around (sx, sy), numpy's low + (high - low) u
__device__ __forceinline__ void draw_point(const Stream& s, unsigned d, unsigned sid, double sx, double sy, double rlo,
                                           double rhi, double& x, double& y, double& r) {
  const double2 u = uniforms(s, d, sid);
  r = __dadd_rn(rlo, __dmul_rn(__dsub_rn(rhi, rlo), u.y));
  double sn, cs;
  sincospi(2.0 * u.x, &sn, &cs);  // (sin, cos)(2 pi u): no argument reduction, so no local-memory slow path
  x = __dadd_rn(sx, __dmul_rn(r, cs));
  y = __dadd_rn(sy, __dmul_rn(r, sn));
}
__device__ __forceinline__ double dist(double ox, double oy, double x, double y) {
  const double dx = __dsub_rn(ox, x), dy = __dsub_rn(oy, y);
  return sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// The first of draws 0 .. n - 1 farther than r from the other source (or thr if thr >= 0), 32 draws per step.
__device__ bool first_survivor(const Stream& s, unsigned sid, int n, double sx, double sy, double rlo, double rhi,
                               double ox, double oy, bool has_other, double thr, double& X, double& Y) {
  const int lane = threadIdx.x & 31;
  for (int base = 0; base < n; base += 32) {
    const int d = base + lane;
    double x = 0.0, y = 0.0, r = 0.0;
    bool ok = false;
    if (d < n) {
      draw_point(s, d, sid, sx, sy, rlo, rhi, x, y, r);
      ok = !has_other || dist(ox, oy, x, y) > (thr >= 0.0 ? thr : r);
    }
    const unsigned m = __ballot_sync(FULL, ok);
    if (m) {
      const int at = __ffs(m) - 1;
      X = __shfl_sync(FULL, x, at);
      Y = __shfl_sync(FULL, y, at);
      return true;
    }
  }
  return false;
}
// Survivors among the 4 N miss draws of a source: farther than ks50 from the other source.
__device__ int count_survivors(const Stream& s, unsigned sid, double sx, double sy, double rlo, double rhi, double ox,
                               double oy, double thr) {
  const int lane = threadIdx.x & 31;
  int count = 0;
  for (int base = 0; base < 4 * N_DRAW; base += 32) {
    const int d = base + lane;
    bool ok = false;
    if (d < 4 * N_DRAW) {
      double x, y, r;
      draw_point(s, d, sid, sx, sy, rlo, rhi, x, y, r);
      ok = dist(ox, oy, x, y) > thr;
    }
    count += __popc(__ballot_sync(FULL, ok));
  }
  return count;
}
// The k-th survivor (0-based) of the same draws, regenerated.
__device__ void kth_survivor(const Stream& s, unsigned sid, int k, double sx, double sy, double rlo, double rhi,
                             double ox, double oy, bool has_other, double thr, double& X, double& Y) {
  const int lane = threadIdx.x & 31;
  for (int base = 0; base < 4 * N_DRAW; base += 32) {
    const int d = base + lane;
    double x = 0.0, y = 0.0, r;
    bool ok = false;
    if (d < 4 * N_DRAW) {
      draw_point(s, d, sid, sx, sy, rlo, rhi, x, y, r);
      ok = !has_other || dist(ox, oy, x, y) > thr;
    }
    const unsigned m = __ballot_sync(FULL, ok);
    const int c = __popc(m);
    if (k < c) {
      const int at = __fns(m, 0, k + 1);
      X = __shfl_sync(FULL, x, at);
      Y = __shfl_sync(FULL, y, at);
      return;
    }
    k -= c;
  }
}

// noise_utils' probability tiers of joint j
__device__ __forceinline__ void tier_probs(int j, int num_valid, double& jitter, double& miss, double& inv) {
  if (j == 0 || (j >= 13 && j <= 16)) jitter = num_valid <= 10 ? 0.15 : 0.10;
  else if (j >= 1 && j <= 10) jitter = num_valid <= 10 ? 0.20 : 0.15;
  else jitter = num_valid <= 10 ? 0.25 : 0.20;
  if (j <= 4) miss = num_valid <= 5 ? 0.15 : (num_valid <= 10 ? 0.10 : 0.02);
  else if (j == 5 || j == 6 || j == 15 || j == 16) miss = num_valid <= 5 ? 0.20 : (num_valid <= 10 ? 0.13 : 0.05);
  else miss = num_valid <= 5 ? 0.25 : (num_valid <= 10 ? 0.15 : 0.10);
  inv = j <= 4 ? 0.01 : (j <= 10 ? 0.03 : 0.06);
}

// One joint of synthesize_pose, one warp.  gt = the joint's own coordinate; inv = the pair's coordinate (its
// synthesized row in phase 2), present when the pair's ORIGINAL visibility is > 0.  -> (x, y, 1) or (0, 0, 0).
__device__ float3 synth_joint(const Stream& s, int j, double gx, double gy, bool has_inv, double ix, double iy,
                              int num_valid, double area) {
  const unsigned sid = 16u * j;
  const double sig = KPS_SIGMAS_X10[j] / 10.0, t = sig * 2.0, var = __dmul_rn(t, t);
  const double a2v = __dmul_rn(-2.0 * area, var);
  const double k10 = sqrt(__dmul_rn(a2v, LN_010)), k50 = sqrt(__dmul_rn(a2v, LN_050)),
               k85 = sqrt(__dmul_rn(a2v, LN_085));
  double jp, mp, ip;
  tier_probs(j, num_valid, jp, mp, ip);

  double jx = 0, jy = 0, mx = 0, my = 0, vx = 0, vy = 0, ox = 0, oy = 0;
  // jitter: r ~ U(ks85, ks50) around gt, farther than r from inv
  const bool jit_ok = first_survivor(s, sid + JITTER, N_DRAW, gx, gy, k85, k50, ix, iy, has_inv, -1.0, jx, jy);
  // miss: 4 N draws per source, r ~ U(ks50, ks10), farther than ks50 from the other source; gt with probability
  // S0 / (S0 + S1 / 4), then a uniform survivor of the chosen source
  int s0 = 4 * N_DRAW, s1 = 0;
  if (has_inv) {
    s0 = count_survivors(s, sid + MISS_GT, gx, gy, k50, k10, ix, iy, k50);
    s1 = count_survivors(s, sid + MISS_INV, ix, iy, k50, k10, gx, gy, k50);
  }
  const int tot = s0 + s1 / 4;
  const bool miss_ok = tot > 0;  // S0 = 0 and S1 < 4: absent (the reference raises there)
  if (miss_ok) {
    const double2 u = uniforms(s, 0, sid + MISS_PICK);
    const int k = pick_index(u.x, tot);
    if (k < s0) kth_survivor(s, sid + MISS_GT, k, gx, gy, k50, k10, ix, iy, has_inv, k50, mx, my);
    else kth_survivor(s, sid + MISS_INV, pick_index(u.y, s1), ix, iy, k50, k10, gx, gy, true, k50, mx, my);
  }
  // inv: r ~ U(0, ks50) around inv, farther than r from gt
  const bool inv_ok = has_inv && first_survivor(s, sid + INV, N_DRAW, ix, iy, 0.0, k50, gx, gy, true, -1.0, vx, vy);
  // good: N / 4 draws, r ~ U(0, ks85) around gt, farther than r from inv
  double gp = 1.0 - (((jp + mp) + ip) + 0.0);
  const bool good_ok = first_survivor(s, sid + GOOD, N_DRAW / 4, gx, gy, 0.0, k85, ix, iy, has_inv, -1.0, ox, oy);

  if (!jit_ok) jp = 0.0;
  if (!miss_ok) mp = 0.0;
  if (!inv_ok) ip = 0.0;
  if (!good_ok) gp = 0.0;
  const double norm = (((jp + mp) + ip) + 0.0) + gp;
  if (norm == 0.0) return make_float3(0.f, 0.f, 0.f);
  const double tc = __dmul_rn(uniforms(s, 0, sid + CHOICE).x, norm);
  const double c1 = jp, c2 = c1 + mp, c3 = c2 + ip;
  double X, Y;
  if (jit_ok && tc < c1) X = jx, Y = jy;
  else if (miss_ok && tc < c2) X = mx, Y = my;
  else if (inv_ok && tc < c3) X = vx, Y = vy;
  else if (good_ok) X = ox, Y = oy;  // the last present candidate takes a tc at the top of the range
  else if (inv_ok) X = vx, Y = vy;
  else if (miss_ok) X = mx, Y = my;
  else X = jx, Y = jy;
  return make_float3((float)X, (float)Y, 1.f);
}

// synthesize_pose of one sample by the CTA (SYNTH_THREADS threads): x, y, v in shared memory hold the input rows and
// receive the output rows.  Phase 1: joints 0, 1, 3, .., 15 (their pair sources are original rows); phase 2: joints
// 2, 4, .., 16 (their pair source is the phase-1 row of joint j - 1).
__device__ void synthesize_sample(const Stream& s, float* x, float* y, float* v, double area) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __shared__ float vis0[N_KPS];
  if (threadIdx.x < N_KPS) vis0[threadIdx.x] = v[threadIdx.x];
  __syncthreads();
  const int num_valid = __popc(__ballot_sync(FULL, lane < N_KPS && vis0[lane] > 0.f));
  for (int phase = 0; phase < 2; ++phase) {
    const int j = phase == 0 ? (warp == 0 ? 0 : 2 * warp - 1) : 2 * warp + 2;
    float3 r = make_float3(0.f, 0.f, 0.f);
    const bool active = phase == 0 || warp < 8;
    if (active) {
      const int p = j == 0 ? -1 : (j & 1 ? j + 1 : j - 1);
      const bool has_inv = p >= 0 && vis0[p] > 0.f;
      r = synth_joint(s, j, x[j], y[j], has_inv, has_inv ? x[p] : 0.0, has_inv ? y[p] : 0.0, num_valid, area);
    }
    __syncthreads();  // every phase-1 read of a phase-2 joint's row is done
    if (active && lane == 0) {
      x[j] = r.x;
      y[j] = r.y;
      v[j] = r.z;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(SYNTH_THREADS) k_synthesize_pose(const float* __restrict__ joints,
                                                                   const float* __restrict__ area,
                                                                   const long long* __restrict__ seed,
                                                                   float* __restrict__ out) {
  __shared__ float x[N_KPS], y[N_KPS], v[N_KPS];
  const long long b = blockIdx.x;
  const float* in = joints + b * N_KPS * 3;
  if (threadIdx.x < N_KPS) {
    x[threadIdx.x] = in[threadIdx.x * 3 + 0];
    y[threadIdx.x] = in[threadIdx.x * 3 + 1];
    v[threadIdx.x] = in[threadIdx.x * 3 + 2];
  }
  synthesize_sample(make_stream(seed, (unsigned)b), x, y, v, (double)area[b]);
  if (threadIdx.x < N_KPS) {
    float* o = out + b * N_KPS * 3;
    o[threadIdx.x * 3 + 0] = x[threadIdx.x];
    o[threadIdx.x * 3 + 1] = y[threadIdx.x];
    o[threadIdx.x * 3 + 2] = v[threadIdx.x];
  }
}

// generate_syn_error of joint i: x ~ N(mean0, std0), y ~ N(mean1, std1) by Box-Muller in fp64, stored as float32,
// kept iff float32 weight > u
__device__ __forceinline__ float2 syn_error(const Stream& s, const p2m_h36m_error_t& e, int i) {
  const double2 g = uniforms(s, 0, 16u * i + GAUSS);
  const double rad = sqrt(-2.0 * log(1.0 - g.x));
  double sn, cs;
  sincospi(2.0 * g.y, &sn, &cs);
  const float nx = (float)__dadd_rn(e.mean[0], __dmul_rn(e.std[0], __dmul_rn(rad, cs)));
  const float ny = (float)__dadd_rn(e.mean[1], __dmul_rn(e.std[1], __dmul_rn(rad, sn)));
  const bool keep = (double)(float)e.weight > uniforms(s, 0, 16u * i + KEEP).x;
  return keep ? make_float2(nx, ny) : make_float2(0.f, 0.f);
}

__global__ void __launch_bounds__(128) k_h36m_syn_error(const ErrTable table, const long long* __restrict__ seed,
                                                        int batch, float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)batch * N_KPS) return;
  const int b = (int)(t / N_KPS), i = (int)(t % N_KPS);
  const float2 n = syn_error(make_stream(seed, (unsigned)b), table.e[i], i);
  out[t * 2 + 0] = n.x;
  out[t * 2 + 1] = n.y;
}

// augm_params (lib/aug_utils.py:98-117), one thread per sample: flip with probability 1/2 when enabled; rot =
// clip(N(0, 1) rf, -2 rf, 2 rf), then 0 with probability 1/2.  Stream AUG_SID + 0 draw 0 gives the (flip, keep)
// uniforms, AUG_SID + 1 draw 0 the Box-Muller pair.
constexpr unsigned AUG_SID = 0x80000000u;
__global__ void __launch_bounds__(256) k_augm_params(int batch, int do_flip, double rf,
                                                     const long long* __restrict__ seed, int* __restrict__ flip,
                                                     float* __restrict__ rot) {
  const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const Stream s = make_stream(seed, (unsigned)b);
  const double2 u = uniforms(s, 0, AUG_SID);
  const double2 g = uniforms(s, 0, AUG_SID + 1);
  double sn, cs;
  sincospi(2.0 * g.y, &sn, &cs);
  const double z = __dmul_rn(sqrt(-2.0 * log(1.0 - g.x)), cs);
  const double r = fmin(2.0 * rf, fmax(-2.0 * rf, __dmul_rn(z, rf)));
  flip[b] = do_flip && u.x <= 0.5 ? 1 : 0;
  rot[b] = u.y <= 0.5 ? 0.f : (float)r;
}

// get_affine_transform(centre, (w, h), rot, (in_w, in_h)) for rot != 0 (lib/aug_utils.py:125-185): get_dir in fp64,
// the src / dst point pairs stored as float32 with get_3rd_point in float32, the 3-point system solved in fp64 (relative
// to the first pair, by Cramer's rule).  A point maps to q0 + A (p - s0).
struct RotCrop {
  double s0x, s0y, q0x, q0y, a00, a01, a10, a11;
};
__device__ __forceinline__ RotCrop rot_crop(const PoseCrop& c, float rot, int in_h, int in_w) {
  double sn, cs;
  sincospi(__ddiv_rn((double)rot, 180.0), &sn, &cs);  // (sin, cos)(pi rot / 180), no local-memory slow path
  const double hw = (double)(c.w * -0.5f);
  const float s0x = c.ccx, s0y = c.ccy;
  const float s1x = (float)__dadd_rn((double)s0x, __dsub_rn(0.0 * cs, __dmul_rn(hw, sn)));
  const float s1y = (float)__dadd_rn((double)s0y, __dadd_rn(0.0 * sn, __dmul_rn(hw, cs)));
  const float s2x = __fadd_rn(s1x, -__fsub_rn(s0y, s1y)), s2y = __fadd_rn(s1y, __fsub_rn(s0x, s1x));
  const float q0x = (float)(in_w * 0.5), q0y = (float)(in_h * 0.5);
  const float q1x = q0x, q1y = (float)(in_h * 0.5) + (float)(in_w * -0.5);
  const float q2x = __fadd_rn(q1x, -__fsub_rn(q0y, q1y)), q2y = __fadd_rn(q1y, __fsub_rn(q0x, q1x));
  const double e1x = (double)s1x - s0x, e1y = (double)s1y - s0y, e2x = (double)s2x - s0x, e2y = (double)s2y - s0y;
  const double f1x = (double)q1x - q0x, f1y = (double)q1y - q0y, f2x = (double)q2x - q0x, f2y = (double)q2y - q0y;
  const double det = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e2x, e1y));
  RotCrop m;
  m.s0x = s0x, m.s0y = s0y, m.q0x = q0x, m.q0y = q0y;
  m.a00 = __ddiv_rn(__dsub_rn(__dmul_rn(f1x, e2y), __dmul_rn(f2x, e1y)), det);
  m.a01 = __ddiv_rn(__dsub_rn(__dmul_rn(f2x, e1x), __dmul_rn(f1x, e2x)), det);
  m.a10 = __ddiv_rn(__dsub_rn(__dmul_rn(f1y, e2y), __dmul_rn(f2y, e1y)), det);
  m.a11 = __ddiv_rn(__dsub_rn(__dmul_rn(f2y, e1x), __dmul_rn(f1y, e2x)), det);
  return m;
}
__device__ __forceinline__ double2 rot_point(const RotCrop& m, float x, float y) {
  const double dx = (double)x - m.s0x, dy = (double)y - m.s0y;
  return make_double2(__dadd_rn(m.q0x, __dadd_rn(__dmul_rn(m.a00, dx), __dmul_rn(m.a01, dy))),
                      __dadd_rn(m.q0y, __dadd_rn(__dmul_rn(m.a10, dx), __dmul_rn(m.a11, dy))));
}
// flip_2d_joint on warp 0's row (lane = joint): x -> in_w - x - 1 in float32, then the flip pairs swapped
__device__ __forceinline__ float2 flip_row(float2 c, int joint_set, int in_w) {
  const int p = flip_partner(joint_set, threadIdx.x & 31);
  c.x = __fsub_rn(__fsub_rn((float)in_w, c.x), 1.f);
  return make_float2(__shfl_sync(FULL, c.x, p), __shfl_sync(FULL, c.y, p));
}

struct Augment {
  const float* rot;   // [B] degrees, or null
  const int* flip;    // [B], or null
  int joint_set;      // the flip pairs
  int flip_before;    // MuCo: flip inside j2d_processing (fp64, before the noise); else after the noise (float32)
};

// One sample per CTA; warp 0 does the crop and the normalisation, the COCO noise takes SYNTH_THREADS threads.
template <int NOISE>
__global__ void __launch_bounds__(NOISE == P2M_NOISE_COCO ? SYNTH_THREADS : 32)
    k_training_pose2d(const float* __restrict__ px, int n_joint, const float* __restrict__ box, int n_box,
                      int area_box, const ErrTable table, const long long* __restrict__ seed, int in_h, int in_w,
                      const Augment aug, float* __restrict__ out) {
  __shared__ float x[32], y[32], v[N_KPS];  // crop pixels of every joint; rows 0-16 go through synthesize_sample
  __shared__ double area;
  __shared__ int sflip;  // the COCO noise's flip after it, kept in shared memory rather than live across its calls
  const long long b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool on = lane < n_joint;
  if (warp == 0) {
    const int flip = aug.flip ? aug.flip[b] : 0;
    const float px_x = on ? px[(b * n_joint + lane) * 2 + 0] : 0.f, px_y = on ? px[(b * n_joint + lane) * 2 + 1] : 0.f;
    PoseCrop m;
    if (box) {
      const bool bon = lane < n_box;
      m = pose_crop(bon ? box[(b * n_box + lane) * 2 + 0] : 0.f, bon ? box[(b * n_box + lane) * 2 + 1] : 0.f, bon,
                    in_h, in_w);
    } else {
      m = pose_crop(px_x, px_y, on, in_h, in_w);
    }
    const float rot = aug.rot ? aug.rot[b] : 0.f;
    double2 t = rot == 0.f ? crop_point_d(m, px_x, px_y, in_h, in_w) : rot_point(rot_crop(m, rot, in_h, in_w), px_x, px_y);
    if (flip && aug.flip_before) t.x = __dsub_rn(__dsub_rn((double)in_w, t.x), 1.0);
    float2 c = make_float2((float)t.x, (float)t.y);
    if (flip && aug.flip_before) c = make_float2(__shfl_sync(FULL, c.x, flip_partner(aug.joint_set, lane)),
                                                 __shfl_sync(FULL, c.y, flip_partner(aug.joint_set, lane)));
    if (NOISE == P2M_NOISE_H36M && lane < N_KPS) {  // (noise / 256) * (input_w, input_h) in float32, then added
      const float2 e = syn_error(make_stream(seed, (unsigned)b), table.e[lane], lane);
      c.x = __fadd_rn(c.x, __fmul_rn(e.x / 256.f, (float)in_w));
      c.y = __fadd_rn(c.y, __fmul_rn(e.y / 256.f, (float)in_h));
    }
    if (NOISE != P2M_NOISE_COCO && flip && !aug.flip_before) c = flip_row(c, aug.joint_set, in_w);
    x[lane] = c.x;
    y[lane] = c.y;
    if (NOISE == P2M_NOISE_COCO) {
      if (lane < N_KPS) v[lane] = 1.f;  // the datasets' joint_img column 2 is 1 (get_coco_from_mesh)
      if (lane == 0) {
        sflip = flip && !aug.flip_before;
        const double w = area_box == P2M_AREA_CROP ? (double)m.w : m.tight_w;
        const double h = area_box == P2M_AREA_CROP ? (double)m.h : m.tight_h;
        area = __dmul_rn(__dmul_rn(m.sc, w), __dmul_rn(m.sc, h));
      }
    }
  }
  if (NOISE == P2M_NOISE_COCO) {
    __syncthreads();
    synthesize_sample(make_stream(seed, (unsigned)b), x, y, v, area);
  }
  if (warp == 0) {
    __syncwarp();
    float2 c = make_float2(x[lane], y[lane]);
    if (NOISE == P2M_NOISE_COCO && sflip) c = flip_row(c, aug.joint_set, in_w);
    normalize_crop(c.x, c.y, on, n_joint, in_h, in_w, out + b * n_joint * 2);
  }
}

int check_table(const char* where, const p2m_h36m_error_t* t, ErrTable* out) {
  if (!t) {
    set_error(std::string(where) + ": the Human3.6M noise needs its 17-entry error table");
    return P2M_ERR_INVALID;
  }
  for (int i = 0; i < N_KPS; ++i) {
    const p2m_h36m_error_t& e = t[i];
    bool ok = isfinite(e.weight) && e.weight >= 0.0 && e.weight <= 1.0;
    for (int c = 0; c < 2; ++c) ok = ok && isfinite(e.mean[c]) && isfinite(e.std[c]) && e.std[c] >= 0.0;
    if (!ok) {
      set_error(std::string(where) + ": error table entry " + std::to_string(i) +
                " must be finite with std >= 0 and 0 <= weight <= 1");
      return P2M_ERR_INVALID;
    }
    out->e[i] = e;
  }
  return P2M_OK;
}

}  // namespace

extern "C" {

int p2m_synthesize_pose(const float* joints, const float* area, const int64_t* seed, int batch, float* out,
                        p2m_stream_t stream) {
  if (!joints || !area || !seed || !out || batch <= 0) {
    set_error("synthesize_pose: bad argument (joints, area, seed and out required, batch > 0)");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("synthesize_pose", {joints, area, seed, out}, &dev));
  DeviceGuard guard(dev);
  k_synthesize_pose<<<batch, SYNTH_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      joints, area, reinterpret_cast<const long long*>(seed), out);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_h36m_syn_error(const p2m_h36m_error_t* error_table, const int64_t* seed, int batch, float* noise,
                       p2m_stream_t stream) {
  if (!seed || !noise || batch <= 0) {
    set_error("h36m_syn_error: bad argument (seed and noise required, batch > 0)");
    return P2M_ERR_INVALID;
  }
  ErrTable table;
  P2M_TRY(check_table("h36m_syn_error", error_table, &table));
  int dev;
  P2M_TRY(arrays_device("h36m_syn_error", {seed, noise}, &dev));
  DeviceGuard guard(dev);
  const long long n = (long long)batch * N_KPS;
  k_h36m_syn_error<<<(unsigned)((n + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      table, reinterpret_cast<const long long*>(seed), batch, noise);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_augm_params(int batch, int flip, double rotate_factor, const int64_t* seed, int32_t* flip_out, float* rot_out,
                    p2m_stream_t stream) {
  if (!seed || !flip_out || !rot_out || batch <= 0 || (flip != 0 && flip != 1) || !isfinite(rotate_factor) ||
      rotate_factor < 0.0) {
    set_error("augm_params: bad argument (seed, flip_out and rot_out required, batch > 0, flip 0 or 1, finite "
              "rotate_factor >= 0)");
    return P2M_ERR_INVALID;
  }
  int dev;
  P2M_TRY(arrays_device("augm_params", {seed, flip_out, rot_out}, &dev));
  DeviceGuard guard(dev);
  k_augm_params<<<(unsigned)((batch + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      batch, flip, rotate_factor, reinterpret_cast<const long long*>(seed), flip_out, rot_out);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

int p2m_training_pose2d(const float* joints_px, int batch, int n_joint, const float* box_joints, int n_box_joint,
                        int noise, int area_box, const p2m_h36m_error_t* error_table, const int64_t* seed, int input_h,
                        int input_w, float* pose2d, p2m_stream_t stream) {
  return p2m_training_pose2d_augmented(joints_px, batch, n_joint, box_joints, n_box_joint, noise, area_box,
                                       error_table, seed, input_h, input_w, nullptr, nullptr, P2M_JOINTS_COCO, 0,
                                       pose2d, stream);
}

int p2m_training_pose2d_augmented(const float* joints_px, int batch, int n_joint, const float* box_joints,
                                  int n_box_joint, int noise, int area_box, const p2m_h36m_error_t* error_table,
                                  const int64_t* seed, int input_h, int input_w, const float* rot,
                                  const int32_t* flip, int flip_joint_set, int flip_before_noise, float* pose2d,
                                  p2m_stream_t stream) {
  if (!joints_px || !pose2d || batch <= 0 || n_joint <= 0 || n_joint > 32 || input_h <= 0 || input_w <= 0 ||
      (box_joints && (n_box_joint <= 0 || n_box_joint > 32)) ||
      (area_box != P2M_AREA_TIGHT && area_box != P2M_AREA_CROP)) {
    set_error("training_pose2d: bad argument (batch > 0, 1 .. 32 joints and box joints, positive input size)");
    return P2M_ERR_INVALID;
  }
  if (flip_joint_set != P2M_JOINTS_HUMAN36 && flip_joint_set != P2M_JOINTS_COCO && flip_joint_set != P2M_JOINTS_SMPL &&
      flip_joint_set != P2M_JOINTS_MANO) {
    set_error("training_pose2d: the flip's joint set must be P2M_JOINTS_HUMAN36, P2M_JOINTS_COCO, P2M_JOINTS_SMPL or "
              "P2M_JOINTS_MANO");
    return P2M_ERR_INVALID;
  }
  // SURREAL's and FreiHAND's inputs are the joints themselves: no detector noise exists for these sets
  if (flip_joint_set == P2M_JOINTS_SMPL || flip_joint_set == P2M_JOINTS_MANO) {
    const bool smpl = flip_joint_set == P2M_JOINTS_SMPL;
    if (noise != P2M_NOISE_NONE || n_joint != (smpl ? 24 : 21) || (!smpl && flip)) {
      set_error("training_pose2d: P2M_JOINTS_SMPL takes 24 joints, P2M_JOINTS_MANO 21 joints and no flip, both without "
                "noise");
      return P2M_ERR_INVALID;
    }
  }
  if (flip && noise != P2M_NOISE_NONE && (noise == P2M_NOISE_H36M) != (flip_joint_set == P2M_JOINTS_HUMAN36)) {
    set_error("training_pose2d: the flip's joint set must be the noise's (Human3.6M noise: P2M_JOINTS_HUMAN36, COCO "
              "noise: P2M_JOINTS_COCO)");
    return P2M_ERR_INVALID;
  }
  if (flip && (flip_joint_set == P2M_JOINTS_HUMAN36 ? n_joint != N_KPS
                                                    : flip_joint_set == P2M_JOINTS_COCO && n_joint < N_KPS)) {
    set_error("training_pose2d: a flip needs exactly 17 Human3.6M joints or at least the 17 COCO joints");
    return P2M_ERR_INVALID;
  }
  if (noise != P2M_NOISE_NONE && noise != P2M_NOISE_COCO && noise != P2M_NOISE_H36M) {
    set_error("training_pose2d: noise must be P2M_NOISE_NONE, P2M_NOISE_COCO or P2M_NOISE_H36M");
    return P2M_ERR_INVALID;
  }
  if (noise != P2M_NOISE_NONE && !seed) {
    set_error("training_pose2d: the noise needs a seed");
    return P2M_ERR_INVALID;
  }
  if ((noise == P2M_NOISE_COCO && n_joint < N_KPS) || (noise == P2M_NOISE_H36M && n_joint != N_KPS)) {
    set_error("training_pose2d: the COCO noise needs at least 17 joints, the Human3.6M noise exactly 17");
    return P2M_ERR_INVALID;
  }
  ErrTable table = {};
  if (noise == P2M_NOISE_H36M) P2M_TRY(check_table("training_pose2d", error_table, &table));
  int dev;
  P2M_TRY(arrays_device("training_pose2d", {joints_px, box_joints, seed, rot, flip, pose2d}, &dev));
  DeviceGuard guard(dev);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long* sd = reinterpret_cast<const long long*>(seed);
  const int nb = box_joints ? n_box_joint : 0;
  const Augment aug{rot, flip, flip_joint_set, flip_before_noise ? 1 : 0};
  if (noise == P2M_NOISE_COCO)
    k_training_pose2d<P2M_NOISE_COCO><<<batch, SYNTH_THREADS, 0, s>>>(joints_px, n_joint, box_joints, nb, area_box,
                                                                      table, sd, input_h, input_w, aug, pose2d);
  else if (noise == P2M_NOISE_H36M)
    k_training_pose2d<P2M_NOISE_H36M><<<batch, 32, 0, s>>>(joints_px, n_joint, box_joints, nb, area_box, table, sd,
                                                            input_h, input_w, aug, pose2d);
  else
    k_training_pose2d<P2M_NOISE_NONE><<<batch, 32, 0, s>>>(joints_px, n_joint, box_joints, nb, area_box, table, sd,
                                                            input_h, input_w, aug, pose2d);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

}  // extern "C"
