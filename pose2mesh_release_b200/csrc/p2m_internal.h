// Internal (C++) interface between the C-ABI files (p2m_api.cu, posenet.cu, front_back.cu, ...) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <initializer_list>
#include <string>
#include <vector>

#include "../../include/p2m_b200.h"

namespace p2m {

// ---------------------------------------------------------------- error plumbing (thread-local)
void set_error(const std::string& msg);
void count_launch(int n = 1);
// p2m_debug_conv_log: one entry per launch of the tensor-core conv, dW or dense-GEMM kernel (process-wide)
enum TcKind { TC_CONV = 0, TC_DW = 1, TC_GEMM = 2 };
void log_tc_launch(int kind, int nc, int ns, int xs, int mode, int f16, dim3 grid, int n_tiles);

#define P2M_CUDA_OK(expr)                                                                     \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      p2m::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " (" +        \
                     __FILE__ + ":" + std::to_string(__LINE__) + ")");                        \
      return P2M_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

#define P2M_LAUNCH_OK()                                                                       \
  do {                                                                                        \
    p2m::count_launch();                                                                      \
    cudaError_t _e = cudaGetLastError();                                                      \
    if (_e != cudaSuccess) {                                                                  \
      p2m::set_error(std::string("kernel launch failed: ") + cudaGetErrorString(_e) + " (" +  \
                     __FILE__ + ":" + std::to_string(__LINE__) + ")");                        \
      return P2M_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

#define P2M_TRY(expr)            \
  do {                           \
    int _s = (expr);             \
    if (_s != P2M_OK) return _s; \
  } while (0)

// Every entry point that touches the device makes its device (the handle's, or for a stateless entry point the one
// arrays_device finds) current for its own duration only: the
// caller's current device is restored on every exit path (single-process multi-GPU callers, nn.DataParallel
// threads, handles garbage-collected at arbitrary times).
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) switched = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() {
    if (switched && prev >= 0) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// The device a stateless entry point (one without a handle) runs on.  `arrays` are the call's data arrays: inputs,
// outputs, optional arrays and workspace, not host-side tables.  Null entries are skipped; every other entry must be
// device or managed memory, all of one device, which is stored to *dev.  Otherwise P2M_ERR_INVALID, naming `where`.
int arrays_device(const char* where, std::initializer_list<const void*> arrays, int* dev);
int arrays_device(const char* where, const void* const* arrays, size_t n, int* dev);  // a run-time count of arrays

// n elements of T allocated on stream s (cudaMallocAsync), optionally filled from host memory, and freed on the same
// stream at scope exit, i.e. after the kernels enqueued in between.  n == 0 allocates nothing and leaves ptr null.
template <typename T>
struct StreamBuffer {
  T* ptr = nullptr;
  cudaStream_t s;
  explicit StreamBuffer(cudaStream_t st) : s(st) {}
  int alloc(size_t n, const void* host = nullptr) {
    if (n == 0) return P2M_OK;
    P2M_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&ptr), sizeof(T) * n, s));
    if (host) P2M_CUDA_OK(cudaMemcpyAsync(ptr, host, sizeof(T) * n, cudaMemcpyHostToDevice, s));
    return P2M_OK;
  }
  ~StreamBuffer() {
    if (ptr) cudaFreeAsync(ptr, s);
  }
  StreamBuffer(const StreamBuffer&) = delete;
  StreamBuffer& operator=(const StreamBuffer&) = delete;
};

// Carving a caller-provided workspace into 256-byte aligned arrays.
constexpr size_t ALIGN = 256;
inline size_t align_up(size_t x) { return (x + ALIGN - 1) / ALIGN * ALIGN; }
struct Bump {
  char* base;
  size_t off = 0;
  explicit Bump(void* p) : base(static_cast<char*>(p)) {}
  template <class T>
  T* take(size_t n) {
    T* p = reinterpret_cast<T*>(base + off);
    off += align_up(n * sizeof(T));
    return p;
  }
};

// CTAs of a grid-stride launch: ceil(work / per_cta), clamped to [1, max_ctas].
inline unsigned grid_for(long long work, int per_cta, long long max_ctas) {
  const long long g = (work + per_cta - 1) / per_cta;
  return (unsigned)(g < 1 ? 1 : (g < max_ctas ? g : max_ctas));
}

// What other translation units read of a body-model handle (body_model.cu): its device, sizes and the device copy of
// its model betas [S].
struct BodyModelInfo {
  int device, V, J, S, n_out;
  const float* model_betas;
};
BodyModelInfo body_model_info(const p2m_body_model_t* m);

// ---------------------------------------------------------------- device-resident hierarchy level
// L~ of one level in CSR with RELATIVE column offsets: the neighbour of flat activation row
// r = b*V + v is row r + reloff[p], so kernels never need (b, v) separately (block-diagonal I_B (x) L~).
// Tile blobs (the tile's own rows, their 1-hop halo, the CSR of the own rows over staged-row slots, the own rows
// in length-sorted order) of one level, for tiles of a fixed row count.
struct TileBlobs {
  const unsigned char* meta = nullptr;  // [n_pattern][stride]
  const int* bytes = nullptr;           // [n_pattern]
  int stride = 0;
  int n_pattern = 0;                    // tiles per mesh
  int max_h1 = 0;                       // largest own + 1-hop row count
};
// A family of 128-row tile patterns of one level whose rows are given by index lists instead of being the consecutive
// rows [128 p, 128 p + 128), and the same rows cut into 64-row tiles (m64: the 64-row x 128-column conv configuration).
struct TileSet : TileBlobs {
  TileBlobs m64;
};

struct DevLevel {
  int V = 0;
  int nnz = 0;
  int max_row_nnz = 0;
  int* rowptr = nullptr;   // [V+1]
  int* reloff = nullptr;   // [nnz] col - row
  float* val = nullptr;    // [nnz]
  // tensor-core path (cheb_umma.cu): tile blobs of the 128-row tiles [128 p, 128 p + 128) (k_cheb_t1, the dW kernel,
  // the 128-row conv configuration; n_pattern == 0: the level has no tensor-core metadata) and of the 64-row tiles
  // [64 p, 64 p + 64) (the 64-row x 128-column conv configuration)
  TileBlobs meta128, meta64;
  // L~ == L~^T exactly (the backward passes use L~ where the math needs L~^T), and h = ceil(log2(2 r^2 + 1)) for r the
  // largest absolute row sum of L~: max|T2| <= (2 r^2 + 1) max|x|, the headroom the single-layer fp16 split leaves
  bool symmetric = true;
  int headroom_log2 = 0;
  // Padding-vertex elision: the fake vertices of the binary-tree reorder (lib/coarsening.py:214-258) are isolated in
  // L~ and share one diagonal value iso_diag, so on them the conv is a dense map with the combined weights
  // W0 + c W1 + (2c^2 - 1) W2.  real_tiles covers the connected rows (conv path), iso_tiles the isolated ones (plain
  // GEMM).  n_iso == 0: not applicable on this level.
  int n_iso = 0;
  float iso_diag = 0.f;
  TileSet real_tiles, iso_tiles;
  // Eval-mode duplicate elimination among the isolated rows (p2m_api.cu: build_padding_classes).  The two children
  // of a fake vertex are fake too and, with BatchNorm folded, carry identical values in every layer of their level
  // (same parent row through the unpool, same dense map): only one REPRESENTATIVE per class is computed
  // (rep_tiles, plain GEMM like iso_tiles) and the network's output rows of the others are filled from it at the
  // end (copy_dst[i] <- copy_src[i], finest level only).  n_rep == 0: not applicable on this level.
  TileSet rep_tiles;
  int n_rep = 0;
  int n_copy = 0;
  int* copy_dst = nullptr;
  int* copy_src = nullptr;
};

// 2-tap channel resampling table (F.interpolate(mode='linear', align_corners=False) along channels,
// meshnet.py:109,114) and its transpose for the backward pass.
struct InterpTable {
  int fin = 0, fout = 0;
  int* i0 = nullptr;      // [fout]
  int* i1 = nullptr;      // [fout]
  float* lam = nullptr;   // [fout]  out[j] = (1-lam)*x[i0] + lam*x[i1]
  int* t_ptr = nullptr;   // [fin+1]   transpose CSR: dx[i] = sum_p t_w[p] * dout[t_idx[p]]
  int* t_idx = nullptr;
  float* t_w = nullptr;
};

// ---------------------------------------------------------------- SIMT kernels (kernels_simt.cu)
// Chebyshev basis T = [T0 | T1 | T2] (each F wide, row stride 3F) of x.  x is [rows_phys, F]; when
// in_unpool, logical row r reads physical row r>>1 (nearest x2 unpool, meshnet.py:71-78).
int launch_cheb_basis(const DevLevel& g, const float* x, int in_unpool, int rows, int F, float* T, cudaStream_t s);

struct Epilogue {
  const float* bias = nullptr;    // [N] added first
  const float* scale = nullptr;   // [N] then v = v*scale + shift
  const float* shift = nullptr;
  int relu = 0;
  const float* res = nullptr;     // residual source [rows(/2), res_F], channel-resampled to N, added last
  int res_F = 0;
  int res_unpool = 0;
  const int* res_i0 = nullptr;
  const int* res_i1 = nullptr;
  const float* res_lam = nullptr;
  // optional fused output gather (the callers' pred[:, perm_reverse[:n_real]], lib/core/base.py:130): row v of a
  // mesh is stored at slot out_map[v] of a [B, out_rows, N] tensor, or dropped when out_map[v] < 0
  const int* out_map = nullptr;
  int out_rows = 0;
  int level_V = 0;
};
#ifdef __CUDACC__
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): PoseNet's dropout masks
// (posenet.cu) and the training inputs' synthetic errors (inputs.cu)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned int hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned int hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// The crop of one pose into the (in_h, in_w) network input, one warp per pose with lane = joint (k_normalize_pose2d,
// inputs.cu): tight box of the joints (coord_utils.py:21-39) -> aspect-preserving box (process_bbox, :42-66) -> the
// rot-0 affine map (aug_utils.py:51-64,140-179: a uniform scaling that maps the box centre to the patch centre).
struct PoseCrop {
  float ccx, ccy;          // centre of the aspect-preserving box
  double sc;               // crop pixels per image pixel
  double tight_w, tight_h; // the tight box's xmax - xmin, ymax - ymin as replace_joint_img takes them
  float w, h;              // the aspect-preserving box
};
__device__ __forceinline__ PoseCrop pose_crop(float x, float y, bool on, int in_h, int in_w) {
  float xmin = on ? x : INFINITY, xmax = on ? x : -INFINITY, ymin = on ? y : INFINITY, ymax = on ? y : -INFINITY;
  for (int o = 16; o > 0; o >>= 1) {
    xmin = fminf(xmin, __shfl_xor_sync(0xffffffffu, xmin, o));
    xmax = fmaxf(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
    ymin = fminf(ymin, __shfl_xor_sync(0xffffffffu, ymin, o));
    ymax = fmaxf(ymax, __shfl_xor_sync(0xffffffffu, ymax, o));
  }
  // get_bbox (float32 arithmetic like numpy on the float32 box)
  float bx, by, bw, bh;
  {
    const double xc = ((double)xmin + (double)xmax) / 2.0, w = (double)xmax - (double)xmin;
    const double yc = ((double)ymin + (double)ymax) / 2.0, h = (double)ymax - (double)ymin;
    bx = (float)(xc - 0.5 * w); by = (float)(yc - 0.5 * h); bw = (float)w; bh = (float)h;
  }
  PoseCrop c;
  c.tight_w = (double)(bx + bw) - (double)bx;
  c.tight_h = (double)(by + bh) - (double)by;
  // process_bbox: sanitise (x2 = x + (w - 1)), grow to the aspect ratio width / height, scale 1.0
  float w = (bx + (bw - 1.f)) - bx, h = (by + (bh - 1.f)) - by;
  const float cx = bx + w / 2.f, cy = by + h / 2.f;
  const float aspect = (float)in_w / (float)in_h;
  if (w > aspect * h) h = w / aspect;
  else if (w < aspect * h) w = h * aspect;
  const float x0 = cx - w / 2.f, y0 = cy - h / 2.f;
  // get_center_scale + get_affine_transform(rot = 0): three float32 point pairs, solved in double
  c.ccx = x0 + w * 0.5f;
  c.ccy = y0 + h * 0.5f;
  const float s1y = c.ccy + w * -0.5f;                                   // src[1] = centre + (0, -src_w / 2)
  const double dst_w = (double)in_w, dst_h = (double)in_h;
  const float d1y = (float)(dst_h * 0.5) + (float)(dst_w * -0.5);        // dst[1] = (dst_w / 2, dst_h / 2 - dst_w / 2)
  c.sc = ((double)d1y - dst_h * 0.5) / ((double)s1y - (double)c.ccy);
  c.w = w;
  c.h = h;
  return c;
}
// A point through the crop's map, in crop pixels, before rounding
__device__ __forceinline__ double2 crop_point_d(const PoseCrop& c, float x, float y, int in_h, int in_w) {
  return make_double2(((double)x - (double)c.ccx) * c.sc + (double)in_w * 0.5,
                      ((double)y - (double)c.ccy) * c.sc + (double)in_h * 0.5);
}
// The same rounded to float32.  truncate: the reference writes the transformed point back into an INTEGER array
// (demo/h36m_joint_input.npy is int64): truncation towards zero before astype('float32').
__device__ __forceinline__ float2 crop_point(const PoseCrop& c, float x, float y, int in_h, int in_w, int truncate) {
  double2 t = crop_point_d(c, x, y, in_h, in_w);
  if (truncate) {
    t.x = trunc(t.x);
    t.y = trunc(t.y);
  }
  return make_float2((float)t.x, (float)t.y);
}
// The joint a horizontal flip swaps joint j with: the datasets' flip_pairs (lib/aug_utils.py flip_2d_joint /
// flip_3d_joint), the same in Human36M, COCO, MuCo and AMASS.  COCO ((1,2),(3,4),..,(15,16)) with pelvis 17 and neck 18
// fixed; Human3.6M ((1,4),(2,5),(3,6),(14,11),(15,12),(16,13)); SURREAL's SMPL ((1,2),(4,5),(7,8),(10,11),(13,14),
// (16,17),(18,19),(20,21),(22,23)); MANO has none.
__device__ __forceinline__ int flip_partner(int joint_set, int j) {
  if (joint_set == P2M_JOINTS_COCO) return (j >= 1 && j <= 16) ? ((j & 1) ? j + 1 : j - 1) : j;
  if (joint_set == P2M_JOINTS_MANO || j <= 0 || j >= 24) return j;
  if (joint_set == P2M_JOINTS_SMPL) {
    if (j >= 18) return (j & 1) ? j - 1 : j + 1;
    return j % 3 == 1 ? j + 1 : (j % 3 == 2 ? j - 1 : j);
  }
  if ((j >= 1 && j <= 3) || (j >= 11 && j <= 13)) return j + 3;
  if ((j >= 4 && j <= 6) || (j >= 14 && j <= 16)) return j - 3;
  return j;
}
// Crop pixels -> / the input size -> per-pose mean / std (population) per coordinate, stored to out [n_joint, 2]
__device__ __forceinline__ void normalize_crop(float cx, float cy, bool on, int n_joint, int in_h, int in_w,
                                               float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  float u = cx / (float)in_w, v = cy / (float)in_h;
  float su = on ? u : 0.f, sv = on ? v : 0.f;
  for (int o = 16; o > 0; o >>= 1) {
    su += __shfl_xor_sync(0xffffffffu, su, o);
    sv += __shfl_xor_sync(0xffffffffu, sv, o);
  }
  const float mu = su / n_joint, mv = sv / n_joint;
  float qu = on ? (u - mu) * (u - mu) : 0.f, qv = on ? (v - mv) * (v - mv) : 0.f;
  for (int o = 16; o > 0; o >>= 1) {
    qu += __shfl_xor_sync(0xffffffffu, qu, o);
    qv += __shfl_xor_sync(0xffffffffu, qv, o);
  }
  if (on) {
    out[lane * 2 + 0] = (u - mu) / sqrtf(qu / n_joint);
    out[lane * 2 + 1] = (v - mv) / sqrtf(qv / n_joint);
  }
}

// Device-side view of Epilogue + the per-element epilogue shared by the SIMT GEMM and the tensor-core conv.
struct EpiDev {
  const float* bias;
  const float* scale;
  const float* shift;
  int relu;
  const float* res;
  int res_F;
  int res_unpool;
  const int* i0;
  const int* i1;
  const float* lam;
  const int* out_map;
  int out_rows;
  int level_V;
};
inline EpiDev to_dev(const Epilogue& e) {
  return EpiDev{e.bias, e.scale, e.shift, e.relu, e.res, e.res_F, e.res_unpool, e.res_i0, e.res_i1, e.res_lam,
                e.out_map, e.out_rows, e.level_V};
}
__device__ __forceinline__ float apply_epilogue(float v, long long r, int n, const EpiDev& ep) {
  if (ep.bias) v += ep.bias[n];
  if (ep.scale) v = fmaf(v, ep.scale[n], ep.shift[n]);
  if (ep.relu) v = fmaxf(v, 0.f);
  if (ep.res) {
    long long pr = ep.res_unpool ? (r >> 1) : r;
    const float* rr = ep.res + pr * ep.res_F;
    if (ep.lam == nullptr) {  // no resampling table: plain residual (res_F == N)
      v += rr[n];
    } else {
      float l = ep.lam[n];
      v += (1.f - l) * rr[ep.i0[n]] + l * rr[ep.i1[n]];
    }
  }
  return v;
}
#endif

// C[M,N] = A[M,K] * op(B) (+ epilogue); b_is_kn: B stored [K,N] row-major, else [N,K] row-major.
int launch_gemm(const float* A, int lda, const float* B, int ldb, int b_is_kn, float* C, int ldc, int M, int N, int K,
                const Epilogue& ep, cudaStream_t s);
// C[N1,N2] (+)= A[M,N1]^T * B[M,N2]  (C must be zeroed by the caller; split over M with atomics)
int launch_gemm_tn_atomic(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N1, int N2,
                          cudaStream_t s);

// Thin-output conv (Fout <= 4), weights first; scratch >= thin_conv_scratch_floats(rows, fin) floats.
bool thin_conv_supported(int fin, int fout);
size_t thin_conv_scratch_floats(long long rows, int fin);
int launch_thin_conv(const DevLevel& g, const float* x, int in_unpool, int rows, int fin, int fout, const float* W,
                     const Epilogue& e, float* scratch, float* y, cudaStream_t s);
// Backward of the thin conv (fin == 64, fout <= 4, no unpool): dx [rows, fin] (may be null), dw [fout, 3 fin] in the
// reference layout (zeroed here); scratch >= thin_conv_bwd_scratch_floats(rows, fin) floats.
bool thin_conv_bwd_supported(int fin, int fout);
size_t thin_conv_bwd_scratch_floats(long long rows, int fin);
int launch_thin_conv_bwd(const DevLevel& g, const float* x, int rows, int fin, int fout, const float* W, const float* dz,
                         float* scratch, float* dx, float* dw, int sm_count, cudaStream_t s);
// The same head in two pieces, for the fused eval path: the 128 -> 64 conv's epilogue produces Z = Y W' itself
// (head_wt / head_z of UmmaConvArgs), the tail applies the two sparse products on the 4-wide rows.
int launch_thin_prep(const float* W, int fin, int fout, float* wt, cudaStream_t s);
int launch_thin_tail(const DevLevel& g, int rows, int fout, const float* Z, float* U, const Epilogue& e, float* y,
                     cudaStream_t s);

int launch_permute_w(const float* W, float* Wp, int fout, int fin, cudaStream_t s);      // [n,f*3+k] -> [n,k*fin+f]
int launch_unpermute_w(const float* Wp, float* W, int fout, int fin, cudaStream_t s);    // inverse
int launch_fill_zero(void* p, size_t bytes, cudaStream_t s);
// y[b, dst[i], :] = y[b, src[i], :]  for i < n, b < batch  (y [batch, V, F])
int launch_copy_rows(float* y, int batch, int V, int F, const int* dst, const int* src, int n, cudaStream_t s);

// BatchNorm1d over rows (cheby_graph_conv.py:38-39; meshnet.py:55).  Each BatchNorm's p2m_bn_opts_t decides its
// statistics here, in the launchers, and nowhere else; bn_opts_default is torch's nn.BatchNorm1d in train mode.
inline p2m_bn_opts_t bn_opts_default(int stats) {
  p2m_bn_opts_t o;
  o.stats = stats;
  o.cumulative = 0;
  o.momentum = 0.1;
  o.eps = 1e-5;
  return o;
}
// P2M_ERR_INVALID (with the error set) unless `o` is a valid record for a BatchNorm with these buffers
int check_bn_opts(const p2m_bn_opts_t& o, const void* rm, const void* rv, const void* nbt, const char* where);
// scale / shift from running statistics: ((z + bias) - rm) * scale + beta (bias may be null); save_mean / save_invstd
// (optional) take rm and 1 / sqrt(rv + eps)
int launch_bn_fold_eval(const float* gamma, const float* beta, const float* rm, const float* rv, const float* bias,
                        double eps, float* scale, float* shift, int F, cudaStream_t s, float* save_mean = nullptr,
                        float* save_invstd = nullptr);
// sums of z - z[0] per channel (shifted: no cancellation for |mean| >> std); launch_bn_finalize reads the same z[0]
int launch_col_stats(const float* z, int rows, int F, double* sums /*[2F] zeroed here*/, cudaStream_t s);
// batch statistics -> save_mean / save_invstd / scale / shift; with o.stats == P2M_BN_BATCH_UPDATE also the running
// statistics and num_batches_tracked (o.momentum, or 1 / num_batches_tracked with o.cumulative), never synchronising
int launch_bn_finalize(const double* sums, const float* z, int rows, int F, const float* gamma, const float* beta,
                       float* rm, float* rv, int64_t* nbt, const p2m_bn_opts_t& o, float* save_mean,
                       float* save_invstd, float* scale, float* shift, cudaStream_t s);
// The forward statistics of one BatchNorm of z [rows, F] by its options: mean / invstd (what the backward reads) and
// the scale / shift of a = z * scale + shift, from the running statistics (P2M_BN_RUNNING) or from the batch
// (launch_col_stats + launch_bn_finalize)
int launch_bn_stats(const float* z, int rows, int F, const float* gamma, const float* beta, float* rm, float* rv,
                    int64_t* nbt, const p2m_bn_opts_t& o, double* sums /*[2F]*/, float* mean, float* invstd,
                    float* scale, float* shift, cudaStream_t s);
// a = relu?(z*scale+shift) (+ resampled residual)
int launch_affine_act(const float* z, int rows, int F, const float* scale, const float* shift, int relu,
                      const float* res, int res_F, int res_unpool, const InterpTable* it, float* a, cudaStream_t s);
// BN+ReLU backward: g_a (grad wrt a = relu(bn(z)) [+ residual]) -> g_z (in place allowed); dgamma, dbeta
// written.  The ReLU mask is recomputed from z (block-end activations already include the residual).
int launch_bn_relu_bwd(const float* z, const float* g_a, int rows, int F, const float* gamma, const float* scale,
                       const float* shift, const float* mean, const float* invstd, int relu,
                       double* sums /*scratch: 2F doubles + 5F floats, 16-byte aligned*/, float* dgamma, float* dbeta,
                       float* g_z, cudaStream_t s,
                       float* gz_scale_out = nullptr /* optional device scalar: launch_absmax_scale(g_z) fused in */,
                       int frozen = 0 /* running statistics: g_z = gamma invstd g', no batch-mean terms */,
                       float* dbias = nullptr /* frozen: sum_rows g_z, the gradient of the bias in front */);
int launch_col_sum(const float* g, int rows, int F, double* scratch /*[F]*/, float* out, cudaStream_t s);

// dX of the Chebyshev basis: given dT [rows,3F] (blocks dT0|dT1|dT2):
//   dXl = dT0 - dT2 + L~ (dT1 + 2 L~ dT2)   (L~ symmetric)   [+ resample^T(g_res)]
// written to dx; when out_pairsum, dx has rows/2 rows and dx[p] = dXl[2p] + dXl[2p+1].
int launch_cheb_basis_bwd(const DevLevel& g, const float* dT, int rows, int F, float* U /*[rows,F] scratch*/,
                          const float* g_res, int res_Fout, const InterpTable* it, int out_pairsum, float* dx,
                          cudaStream_t s);

// ---------------------------------------------------------------- tensor-core path (cheb_umma.cu)
struct UmmaConvArgs {
  const DevLevel* g;
  const float* x;           // [rows(/2), Fin]
  int in_unpool;
  int batch;                // rows = batch * g->V
  int fin, fout;
  const void* wpack;        // packed fp16 hi/lo weights from launch_umma_pack_weights (WPACK_ALL)
  Epilogue ep;
  float* y;                 // [rows, fout]
  // plain-GEMM mode (isolated rows, backward dT = dz * W_k): no SpMM, x is [rows, fin] and the K-blocks are a plain
  // image (launch_umma_pack_weights, WPACK_COMBINED or one order); y is written at y[r*ldy + y_col0 + n]
  const float* t1 = nullptr;        // T1 = L~ x [rows, fin] (launch_cheb_t1): required unless plain
  int plain = 0;
  const float* a_scale = nullptr;   // device scalar from launch_absmax_scale (or null)
  long long ldy = 0;                // 0: fout
  int y_col0 = 0;
  // optional fused thin head (fout == 64 only): instead of storing y, the epilogue writes Z[row][12] = y_row * head_wt
  // (head_wt = k_thin_prep's [64][12] table); y is then not written at all
  const float* head_wt = nullptr;
  float* head_z = nullptr;
  // optional: run on this tile family instead of the level's consecutive tiles
  const TileSet* tiles = nullptr;
  long long* trace = nullptr;       // debug (P2M_UMMA_TRACE builds only): [8][512] event log of CTA 0
  // single-pass fp16 (P2M_PREC_FP16_TC, P2M_PREC_FP16_MIXED_TC): wpack is a hi-only image (launch_umma_pack_weights
  // with f16), one k16 MMA per 16 features; T1-given convs and plain GEMMs, a_scale applied before the rounding
  int f16 = 0;
};
// Host: build the per-tile halo metadata of one level (uploads; device pointers appended to `owned`).  A level whose
// tiles stage more than 512 rows or more than 65535 local-CSR entries gets none (meta128 stays empty: it runs on SIMT).
int build_umma_level_meta(const int* rowptr, const int* colidx, const float* val, int V, DevLevel* out,
                          std::vector<void*>* owned);
// Tiles of 128 (and, TileSet::m64, 64) consecutive entries of `rows` (ascending vertex ids of one level) as a TileSet.
int build_tileset(const std::vector<int>& rows, const int* rowptr, const int* colidx, const float* val, int V,
                  TileSet* ts, std::vector<void*>* owned);
bool umma_conv_supported(const DevLevel& g, int fin, int fout);
// what launch_umma_conv / launch_umma_dw would select on the level's consecutive tiles (p2m_debug_conv_path)
int umma_conv_x_stages(const DevLevel& g, int fin, int fout, bool plain);
struct UmmaConvTiling {
  int cols, ns, xs;  // output columns per CTA (64, 128 or 256), A/B ring slots, X / T1 stages (0: does not fit)
};
UmmaConvTiling umma_conv_tiling(const DevLevel& g, int fin, int fout, bool plain, bool f16 = false);
// p2m_debug_tile_families: per family (consecutive, real_tiles, iso_tiles, rep_tiles) and tile size (128, 64 rows)
// n_pattern, max_h1, blob stride, then (columns per CTA, ring slots, X stages) of what launch_n picks for a conv
// fin -> fout on it: T1-given and plain at fp16x3, T1-given and plain at fp16 ({0, 0, 0}: does not fit, or not the
// tile size fout runs on)
int umma_tile_families(const DevLevel& g, int fin, int fout, int32_t out[4][2][15]);
int umma_dw_x_stages(const DevLevel& g, bool f16 = false);
bool umma_tma_rows(const DevLevel& g);
// Weight images of a conv: fp16 [hi | lo] K-blocks of 32 k (x 2^6) from W [fout, fin*3] in the reference layout (column
// f*3 + k), rows = output channels o and K = input features f; `transposed`: rows f and K = o, the backward-data conv's
// W'[f][o*3 + k] = W[o][f*3 + k] (L~ symmetric: the forward conv run on dz gives dX).  `order` selects the image:
//   WPACK_ALL       blocks u = chunk*3 + k of all three orders, umma_wpack_bytes(K, rows) bytes (the conv);
//   WPACK_COMBINED  the isolated rows' combined weights W0 + c W1 + (2c^2 - 1) W2 (padding-vertex elision), and
//   0, 1, 2         W_k alone (the backward's dT = dz W_k): plain images of umma_plain_pack_bytes(rows, K) bytes.
// f16: the single-pass fp16 image (P2M_PREC_FP16_TC, P2M_PREC_FP16_MIXED_TC) of the same blocks, transposed or not, the round-to-nearest fp16 of W x 2^6 only (half
// the bytes; the sizes below are those of the fp16x3 image and bound both).
constexpr int WPACK_ALL = -1, WPACK_COMBINED = -2;
size_t umma_wpack_bytes(int fin, int fout);
size_t umma_plain_pack_bytes(int N, int K);
int launch_umma_pack_weights(const float* W, int fin, int fout, bool transposed, int order, float c, void* wpack,
                             cudaStream_t s, bool f16 = false);
// scale_out[0] = 2^e with max|x| * 2^e in [2^(9-h), 2^(10-h)), h = headroom_log2  (1 if x is all zero or not
// finite); scratch-free, two tiny launches
int launch_absmax_scale(const float* x, long long n, float* scale_out, cudaStream_t s, int headroom_log2 = 0);
// its second half, for a kernel that finds max|x| as it writes x: that kernel atomicMax-es the magnitudes into a
// zeroed amax[0] as uint bits (non-negative floats order as uints); this writes the scale to scale_out[0] and zeroes
// amax[0] again, so one zeroing serves a sequence of them
int launch_absmax_finish(unsigned int* amax, float* scale_out, cudaStream_t s, int headroom_log2 = 0);
// y[i] = x[i] * (invert ? 1 / scale[0] : scale[0]) * mul  (in place allowed; scale a device scalar)
int launch_scale_by(const float* x, long long n, const float* scale, int invert, float mul, float* y, cudaStream_t s);
// The epilogue of a conv whose weights were packed as W * w_scale[0] instead of W * w_packed (the fixed 2^6): per column
// out_scale = scale * w_packed / w_scale[0] and out_shift = bias * scale + shift (absent vectors: 0 / 1 / 0), i.e. the
// same affine map with the bias folded into the shift
int launch_rescaled_epilogue(const Epilogue& ep, const float* w_scale, float w_packed, int n, float* out_scale,
                             float* out_shift, cudaStream_t s);
// dW[o, f*3+k] += sum_rows dz[row,o] * T_k(x)[row,f] on tensor cores (dw_ref [fout, 3 fin] zeroed by the caller), from
// the Chebyshev basis of one side (`gathered` [rows(/2), gathered_width], t1 = L~ gathered for EVERY row, from
// launch_cheb_t1) and plain tiles of the other (`plain` [rows(/2), plain_width]).  swap = 0: gathered = x, plain = dz;
// swap = 1 (L~ symmetric: sum_rows dz (x) T_k(x) = sum_rows T_k(dz) (x) x): gathered = dz, plain = x.  a_scale (device
// scalar) scales dz into fp16's range and is divided out.  f16: the single-pass kernel (k_cheb_dw_f16_umma,
// P2M_PREC_FP16_MIXED_TC), both operands rounded once to fp16, one MMA per 16 rows; it fits wherever the fp16x3 one does.
bool umma_dw_supported(const DevLevel& g, int gathered_width, int plain_width, bool f16 = false);
int launch_umma_dw(const DevLevel& g, int batch, const float* gathered, int in_unpool, int gathered_width,
                   const float* t1, const float* plain, int g_unpool, int plain_width, int swap, const float* a_scale,
                   float* dw_ref, int* status, int sm_count, cudaStream_t s, bool f16 = false);
// T1 = L~ x for all rows of a level (tile-staged gather), t1 [batch*V, fin] fp32
int launch_cheb_t1(const DevLevel& g, const float* x, int in_unpool, int batch, int fin, float* t1, cudaStream_t s,
                   const TileSet* tiles = nullptr);
int launch_umma_conv(const UmmaConvArgs& a, int* status_flag, const float* zero_row, int sm_count, cudaStream_t s);
// Dense GEMM on the tensor cores (wgmma, fp16x3): Y [M, N] = epilogue(X [M, K] W [N, K]^T), K % 32 == 0, N % 64 == 0, X
// range-normalised before the fp16 split; apack / wpack are
// scratch of umma_gemm_apack_bytes(M, K) / umma_gemm_wpack_bytes(N, K); ep vectors and an identity residual
// (ep.res, res_F == N) are indexed by output column.  An operand's element (row r, k) is p[r ld_row + k ld_k]: a
// row-major matrix is {p, ld, 1}, its transpose {p, 1, ld}.
struct GemmOperand {
  const float* p;
  long long ld_row, ld_k;
};
bool umma_gemm_supported(int M, int N, int K);
size_t umma_gemm_apack_bytes(int M, int K);
size_t umma_gemm_wpack_bytes(int N, int K);
int launch_umma_gemm(GemmOperand X, GemmOperand W, int M, int N, int K, const Epilogue& ep, float* Y, void* apack,
                     void* wpack, int* status, int sm_count, cudaStream_t s, int n_real = 0 /* rows of W if < N */,
                     int k_real = 0 /* k >= k_real is zero padding, if < K */,
                     const float* x_scale = nullptr /* X's range normalisation (launch_absmax_scale); found if null */,
                     const float* w_scale = nullptr /* W is an activation: its range normalisation, not W_SCALE */);
// out[ro, :] = sum over the logical rows r of physical row ro (r = ro, or 2 ro and 2 ro + 1 under the virtual unpool)
// of  dxl[r, :] + resample^T(g_res[r, :])   (g_res may be null)
int launch_dx_finish(const float* dxl, int rows, int F, const float* g_res, int res_Fout, const InterpTable* it,
                     int out_pairsum, float* out, cudaStream_t s);

}  // namespace p2m
