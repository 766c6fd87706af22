// C-ABI layer (include/p2m_b200.h) of the model handle: the handle, workspace planning, the eval and training forward
// and the backward schedules of Pose2Mesh.forward (lib/models/meshnet.py:80-117 of the reference) and the single-layer
// conv entry points, expressed as sequences of the kernels in kernels_simt.cu / cheb_umma.cu on the caller's stream.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "p2m_internal.h"

namespace p2m {

static thread_local std::string g_error;
static thread_local int64_t g_launches = 0;
void set_error(const std::string& msg) { g_error = msg; }
void count_launch(int n) { g_launches += n; }

// p2m_debug_conv_log: process-wide (the autograd engine runs backwards on its own thread), bounded; a slot is claimed
// by one atomic increment, so logging costs the launch paths no lock
constexpr int CONV_LOG_CAP = 1 << 15;
constexpr int CONV_LOG_FIELDS = 9;
static int32_t g_conv_log[CONV_LOG_CAP][CONV_LOG_FIELDS];
static std::atomic<int64_t> g_conv_log_n{0};
void log_tc_launch(int kind, int nc, int ns, int xs, int mode, int f16, dim3 grid, int n_tiles) {
  const int64_t i = g_conv_log_n.fetch_add(1, std::memory_order_relaxed);
  if (i >= CONV_LOG_CAP) return;  // counted, not stored
  const int32_t e[CONV_LOG_FIELDS] = {kind, nc, ns, xs, mode, f16, (int32_t)grid.x, (int32_t)grid.y, n_tiles};
  std::memcpy(g_conv_log[i], e, sizeof(e));
}

int arrays_device(const char* where, std::initializer_list<const void*> arrays, int* dev) {
  return arrays_device(where, arrays.begin(), arrays.size(), dev);
}

int arrays_device(const char* where, const void* const* arrays, size_t n, int* dev) {
  int found = -1;
  for (size_t i = 0; i < n; ++i) {
    const void* p = arrays[i];
    if (!p) continue;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess ||
        (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged)) {
      cudaGetLastError();
      set_error(std::string(where) + ": the data arrays must be device memory");
      return P2M_ERR_INVALID;
    }
    if (found >= 0 && attr.device != found) {
      set_error(std::string(where) + ": the data arrays are on different devices");
      return P2M_ERR_INVALID;
    }
    found = attr.device;
  }
  if (found < 0) {
    set_error(std::string(where) + ": no data array given");
    return P2M_ERR_INVALID;
  }
  *dev = found;
  return P2M_OK;
}

struct Layer {
  int level, V, fin, fout;
  int bn, relu;
  int block_end;
};

struct Block {
  int first_layer, n_layers;
  int level;
  int has_residual;   // 1 <= b <= nb-2   (meshnet.py:108-115)
  int out_unpool;     // 1 <= b <  nb-2   (meshnet.py:111)
  int in_unpool;      // input of this block is the (virtually) unpooled output of the previous block
  int cin, cout;
  InterpTable interp;  // valid when has_residual
};

// p2m_debug_set_capture: the caller's device buffers (one per layer, or none) the schedules copy their tensors into
struct Capture {
  std::vector<float*> z, a, y, g_a, g_z, dx;
  float* fc_out = nullptr;
  float* fc_dx = nullptr;
};

}  // namespace p2m

using namespace p2m;

struct p2m_model {
  int device = 0;
  int sm_count = 132;            // SMs the persistent tensor-core grids are sized for (p2m_debug_set_sm_count)
  int sm_count_device = 132;     // ... the device's own count
  int precision = P2M_PREC_FP32_SIMT;
  std::vector<DevLevel> levels;
  std::vector<Layer> layers;
  std::vector<Block> blocks;
  int n_joint = 0, cin = 0, cout = 0;
  int fc_in = 0, fc_out = 0;
  int* kernel_status = nullptr;       // device alias of status_host (what the kernels write)
  volatile int* status_host = nullptr;  // mapped pinned host word: set by a tensor-core kernel whose mbarrier wait timed out
  long long* trace = nullptr;          // debug (P2M_UMMA_TRACE builds): CTA-0 event log of the tensor-core conv kernel
  int trace_seen = 0;                  // matching conv launches since the trace buffer was set (P2M_TRACE_NTH)
  int* out_map = nullptr;        // optional fused output gather (vertex -> slot, -1 = dropped)
  int out_rows = 0;
  float* zero_row = nullptr;     // 128 B of zeros (halo source for the empty slots of ragged tiles)
  int elide_padding = 1;         // tensor-core conv: isolated padding vertices through a plain GEMM with combined weights;
                                 // 1 = on levels where they are >= 40 % of the rows (measured break-even), 2 = wherever
                                 // the tile families exist, 0 = off (p2m_debug_set_elide_padding)
  int dedup_padding = 1;         // eval: among the isolated rows only one representative per class of identical rows is
                                 // computed (DevLevel::rep_tiles); needs elide_padding == 1 (p2m_debug_set_dedup_padding)
  int fuse_head = 1;             // eval: the 128 -> 64 conv's epilogue feeds the 64 -> 3 head directly (no 64-wide tensor)
  int profiling = 0;             // record a CUDA event pair around every conv layer of the eval forward
  std::unique_ptr<Capture> capture;  // debug: copies of the schedules' tensors (p2m_debug_set_capture); null = none
  std::vector<cudaEvent_t> ev_beg, ev_end;
  std::vector<void*> owned;  // device allocations to free
};

namespace {

// A tensor-core kernel whose bounded mbarrier wait expired wrote the wait's id into the mapped host status word
// (cheb_umma.cu: mbar_timeout).  Checked without any synchronisation at every entry point (and after the stream
// synchronisation of the *_host entry point): the call fails instead of handing out the results of a kernel
// that fell through its barriers.  The word is cleared once reported.
int check_kernel_status(p2m_model* m, const char* where) {
  if (m->status_host == nullptr) return P2M_OK;
  const int code = *m->status_host;
  if (code == 0) return P2M_OK;
  *m->status_host = 0;
  set_error(std::string(where) + ": a tensor-core kernel of an earlier call on this handle timed out on mbarrier wait #" +
            std::to_string(code) + " (results of that call are invalid)");
  return P2M_ERR_CUDA;
}

template <class T>
int upload(p2m_model* m, const std::vector<T>& h, T** out) {
  T* d = nullptr;
  size_t bytes = std::max<size_t>(h.size(), 1) * sizeof(T);
  P2M_CUDA_OK(cudaMalloc(&d, bytes));
  m->owned.push_back(d);
  if (!h.empty()) P2M_CUDA_OK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = d;
  return P2M_OK;
}

// F.interpolate(x, size=fout, mode='linear', align_corners=False) along the channel axis
// (meshnet.py:109,114; ATen upsample_linear1d: src = scale*(j+0.5)-0.5 clamped at 0, scale = fin/fout).
int build_interp(p2m_model* m, int fin, int fout, InterpTable* t) {
  t->fin = fin;
  t->fout = fout;
  std::vector<int> i0(fout), i1(fout);
  std::vector<float> lam(fout);
  const float scale = (float)fin / (float)fout;
  for (int j = 0; j < fout; ++j) {
    float src = scale * ((float)j + 0.5f) - 0.5f;
    if (src < 0.f) src = 0.f;
    int a = (int)src;
    if (a > fin - 1) a = fin - 1;
    int b = a + ((a < fin - 1) ? 1 : 0);
    i0[j] = a;
    i1[j] = b;
    lam[j] = src - (float)a;
  }
  std::vector<int> tp(fin + 1, 0), ti;
  std::vector<float> tw;
  for (int i = 0; i < fin; ++i) {
    for (int j = 0; j < fout; ++j) {
      float w = 0.f;
      if (i0[j] == i) w += 1.f - lam[j];
      if (i1[j] == i) w += lam[j];
      if (w != 0.f) {
        ti.push_back(j);
        tw.push_back(w);
      }
    }
    tp[i + 1] = (int)ti.size();
  }
  P2M_TRY(upload(m, i0, &t->i0));
  P2M_TRY(upload(m, i1, &t->i1));
  P2M_TRY(upload(m, lam, &t->lam));
  P2M_TRY(upload(m, tp, &t->t_ptr));
  P2M_TRY(upload(m, ti, &t->t_idx));
  P2M_TRY(upload(m, tw, &t->t_w));
  return P2M_OK;
}

struct Sizes {
  size_t max_act = 0;    // floats: max over layers of rows*fout (and fc in/out, and x)
  size_t max_T = 0;      // floats: max rows*3*fin
  size_t max_U = 0;      // floats: max rows*fin
  size_t max_w = 0;      // floats: max fout*3*fin
  size_t max_wpack = 0;  // bytes: packed fp16 hi/lo weight image of the tensor-core path
  size_t max_thin = 1;   // floats: scratch of the thin head's backward
  int max_f = 0;
};

Sizes model_sizes(const p2m_model* m, int B) {
  Sizes s;
  for (const Layer& L : m->layers) {
    size_t rows = (size_t)B * L.V;
    s.max_act = std::max(s.max_act, rows * L.fout);
    s.max_act = std::max(s.max_act, rows * L.fin);
    s.max_T = std::max(s.max_T, rows * 3 * L.fin);
    s.max_U = std::max(s.max_U, rows * L.fin);
    s.max_w = std::max(s.max_w, (size_t)L.fout * 3 * L.fin);
    if (umma_conv_supported(m->levels[L.level], L.fin, L.fout))
      s.max_wpack = std::max(s.max_wpack, umma_wpack_bytes(L.fin, L.fout));
    s.max_f = std::max(s.max_f, std::max(L.fin, L.fout));
    if (thin_conv_bwd_supported(L.fin, L.fout)) s.max_thin = std::max(s.max_thin, thin_conv_bwd_scratch_floats(rows, L.fin));
  }
  s.max_act = std::max(s.max_act, (size_t)B * m->fc_out);
  s.max_act = std::max(s.max_act, (size_t)B * m->fc_in);
  return s;
}

// Workspace of the network schedules: this prefix, then EvalWs's or TrainWs's part; a map sizes it (null base) and carves it
struct WsCommon {
  Sizes s;
  Bump b;
  float* T;
  float* wp_scratch;
  unsigned char* wpack;   // tensor-core packed weights (one layer at a time)
  float* scale_scratch;   // [2*max_f] eval folded scale/shift
  double* sums;           // [2*max_f]
  unsigned char* fc_apack = nullptr;  // operand images of the fc GEMM on the tensor cores (launch_umma_gemm)
  unsigned char* fc_wpack = nullptr;
  WsCommon(const p2m_model* m, int B, void* base) : s(model_sizes(m, B)), b(base) {
    T = b.take<float>(s.max_T);
    wp_scratch = b.take<float>(s.max_w);
    wpack = b.take<unsigned char>(std::max(s.max_wpack, (size_t)16));
    scale_scratch = b.take<float>(2 * (size_t)s.max_f);
    sums = b.take<double>(2 * (size_t)s.max_f);
    if (umma_gemm_supported(B, m->fc_out, m->fc_in)) {
      fc_apack = b.take<unsigned char>(umma_gemm_apack_bytes(B, m->fc_in));
      fc_wpack = b.take<unsigned char>(umma_gemm_wpack_bytes(m->fc_out, m->fc_in));
    }
  }
  size_t bytes() const { return b.off; }
};
// eval: three rotating activation buffers
struct EvalWs : WsCommon {
  float* rot[3];
  EvalWs(const p2m_model* m, int B, void* base) : WsCommon(m, B, base) {
    for (int i = 0; i < 3; ++i) rot[i] = b.take<float>(s.max_act);
  }
};
// training: what the forward saves for the backward
struct TrainWs : WsCommon {
  std::vector<float*> z, a, mean, invstd, scale, shift, wp;  // per layer; z .. shift null on the last layer (no BatchNorm)
  float* fc_out;
  TrainWs(const p2m_model* m, int B, void* base) : WsCommon(m, B, base) {
    const size_t nl = m->layers.size();
    for (std::vector<float*>* v : {&z, &a, &mean, &invstd, &scale, &shift, &wp}) v->assign(nl, nullptr);
    for (size_t i = 0; i < nl; ++i) {
      const Layer& L = m->layers[i];
      size_t n = (size_t)B * L.V * L.fout;
      wp[i] = b.take<float>((size_t)L.fout * 3 * L.fin);
      if (L.bn) {
        z[i] = b.take<float>(n);
        a[i] = b.take<float>(n);
        mean[i] = b.take<float>(L.fout);
        invstd[i] = b.take<float>(L.fout);
        scale[i] = b.take<float>(L.fout);
        shift[i] = b.take<float>(L.fout);
      }
    }
    fc_out = b.take<float>((size_t)B * m->fc_out);
  }
};

// Device copies of the host entry points' x and y (room for every vertex), behind their forward's workspace
struct HostIo {
  float *x, *y;
  size_t bytes;
  HostIo(const p2m_model* m, int B, void* base) {
    Bump b(base);
    x = b.take<float>((size_t)B * m->n_joint * m->cin);
    y = b.take<float>((size_t)B * m->levels[0].V * m->cout);
    bytes = b.off;
  }
};

// Bytes of the weight-image scratch a backward packs into: the network's (BwdMap::wpack, >= the backward-data image of
// any supported layer) or the single-layer workspace's (the forward image of the layer itself)
size_t wpack_capacity(bool network, int fin, int fout) {
  return network ? umma_wpack_bytes(256, 256) : umma_wpack_bytes(((fin + 31) / 32) * 32, fout);
}

struct BwdMap {
  float* G[4];
  float* U;
  float* dwp;
  double* sums;
  unsigned char* wpack;   // packed fp16 K-blocks of the backward-data conv (or of one W_k^T for the dT GEMM fallback)
  unsigned char* wpack_iso;  // combined transposed weights of the isolated rows (padding-vertex elision)
  float* thin;               // scratch of the thin head's backward
  float* a_scale;         // power-of-two gradient scale (device scalar)
  size_t bytes;
};
BwdMap map_scratch(const p2m_model* m, int B, void* base) {
  BwdMap w;
  Sizes s = model_sizes(m, B);
  Bump b(base);
  for (int i = 0; i < 4; ++i) w.G[i] = b.take<float>(s.max_act);
  w.U = b.take<float>(s.max_U);
  w.dwp = b.take<float>(std::max(s.max_w, (size_t)1));
  w.sums = b.take<double>(2 * (size_t)s.max_f + 2 * (size_t)m->fc_out);
  w.wpack = b.take<unsigned char>(wpack_capacity(true, 0, 0));
  w.wpack_iso = b.take<unsigned char>(umma_plain_pack_bytes(256, 256));
  w.thin = b.take<float>(s.max_thin);
  w.a_scale = b.take<float>(4);
  w.bytes = b.off;
  return w;
}

// ---- which kernels run a Chebyshev conv
// The precisions whose convs run on the tensor cores: fp16x3, the single-pass fp16 (eval forward only) and the
// single-pass mixed precision (training as well)
inline bool tc_precision(int precision) {
  return precision == P2M_PREC_FP16X3_TC || precision == P2M_PREC_FP16_TC || precision == P2M_PREC_FP16_MIXED_TC;
}
// The precisions whose tensor-core Chebyshev passes issue one MMA per 16 features (fp16 operands rounded once)
inline bool single_pass(int precision) { return precision == P2M_PREC_FP16_TC || precision == P2M_PREC_FP16_MIXED_TC; }
// P2M_PREC_FP16_TC is an inference precision: the entry points that train or differentiate refuse it before any device
// work (so a refused training forward leaves the running statistics as they were)
int refuse_fp16(const p2m_model* m, const char* where) {
  if (m->precision != P2M_PREC_FP16_TC) return P2M_OK;
  set_error(std::string(where) + ": precision fp16 (P2M_PREC_FP16_TC) is an inference precision; the training schedule "
            "and the backward need fp16x3 or fp32");
  return P2M_ERR_INVALID;
}

// Padding-vertex elision of a conv with `width` output columns over `rows` rows under p2m_debug_set_elide_padding's
// `mode`: connected rows through the conv on index-list tiles, isolated rows (DevLevel::n_iso) through a plain GEMM with
// the combined weights.  Mode 1 (default) takes the levels where they are >= 40 % of the rows (measured break-even),
// mode 2 every level that has the tile families, mode 0 none.
bool elided(int mode, const DevLevel& g, long long rows, int width) {
  return mode > 0 && g.n_iso > 0 && rows >= 2LL * width && (mode >= 2 || 5LL * g.n_iso >= 2LL * g.V);
}

// The path of every pass of one conv.  Neither tc_dx nor tc_dt (nor thin): dX on SIMT (dT GEMM + basis backward).
struct ConvRoute {
  bool tc = false;           // forward: T1 pass + tensor-core conv (else SIMT: thin conv or basis + GEMM) ...
  bool elide = false;        // ... with the padding-vertex elision
  bool thin = false;         // backward: dW and dX by the thin head's weights-first backward
  bool tc_dw = false;        // dW by k_cheb_dw_umma on the basis of x (else SIMT), unless dw_dz_basis
  bool dw_dz_basis = false;  // dW by k_cheb_dw_umma on the basis of dz (only with tc_dx, which reuses its L~dz)
  bool tc_dx = false;        // dX by the tensor-core conv on dz ...
  bool dx_elide = false;     // ... with the padding-vertex elision
  bool tc_dt = false;        // dX by three plain GEMMs dT = dz W_k (only without tc_dx)
};
// The one place a conv's path is chosen: fin -> fout on `level` for `batch` meshes at the handle's precision.
// network: a layer of the network schedules, which elide padding vertices, run dX as a conv on dz and take the thin
// head's backward where thin_ok (input neither unpooled nor a residual source, not the first layer); otherwise the
// single-layer entry points (and p2m_debug_conv_path), which do none of these.  need_dx: the caller wants dX.
ConvRoute conv_route(const p2m_model* m, int level, int fin, int fout, int batch, bool network, bool thin_ok = false,
                     bool need_dx = true) {
  const DevLevel& g = m->levels[level];
  const long long rows = (long long)batch * g.V;
  const bool tc = tc_precision(m->precision);
  const size_t cap = wpack_capacity(network, fin, fout);
  ConvRoute r;
  r.tc = tc && umma_conv_supported(g, fin, fout);
  r.elide = network && r.tc && elided(m->elide_padding, g, rows, fout);
  r.thin = network && thin_ok && thin_conv_bwd_supported(fin, fout);
  r.tc_dw = tc && !r.thin && umma_dw_supported(g, fin, fout);
  const bool dx_tc = tc && !r.thin && need_dx && umma_conv_supported(g, fout, fin);
  // (T1 = L~dz fills fout of the 3 fin columns of the T buffer)
  r.tc_dx = network && dx_tc && umma_wpack_bytes(fout, fin) <= cap && fout <= 3LL * fin;
  r.dw_dz_basis = r.tc_dx && umma_dw_supported(g, fout, fin);
  r.dx_elide = r.tc_dx && elided(m->elide_padding, g, rows, fin);
  r.tc_dt = dx_tc && !r.tc_dx && umma_plain_pack_bytes(fin, fout) <= cap;
  return r;
}

// UmmaConvArgs of a conv a.fin -> a.fout as the kernel runs it (the weight image is set by whoever packs it)
UmmaConvArgs umma_args(const DevLevel& g, int batch, const float* x, int in_unpool, int fin, int fout, const Epilogue& ep,
                       float* y, const float* a_scale) {
  UmmaConvArgs a;
  a.g = &g;
  a.x = x;
  a.in_unpool = in_unpool;
  a.batch = batch;
  a.fin = fin;
  a.fout = fout;
  a.wpack = nullptr;
  a.ep = ep;
  a.y = y;
  a.a_scale = a_scale;
  return a;
}

// A conv on the tensor cores: weight pack into wpack, T1 pass into T (unless t1_given: T already holds L~x for every
// row), the conv; with `elide` the conv covers the connected rows and a plain GEMM with the combined weights (packed into
// w_iso) the isolated ones: all of them (iso_mode 0), the class representatives only (1, DevLevel::rep_tiles) or none
// (2: nothing the caller reads depends on them).  W is the layer's [fout, fin*3] weight; `transposed`: the
// backward-data conv on dz, a.fin = the layer's fout, a.fout = its fin.
int run_tc_conv(p2m_model* m, UmmaConvArgs a, const float* W, bool transposed, bool elide, int iso_mode, bool t1_given,
                float* T, unsigned char* wpack, unsigned char* w_iso, cudaStream_t s) {
  const DevLevel& g = *a.g;
  const int fin = transposed ? a.fout : a.fin, fout = transposed ? a.fin : a.fout;
  if (m->trace != nullptr && !transposed) {  // trace builds only: P2M_TRACE_V / P2M_TRACE_UNPOOL pick the layer logged
    const char* tv = getenv("P2M_TRACE_V");
    const char* tu = getenv("P2M_TRACE_UNPOOL");
    const char* tf = getenv("P2M_TRACE_FOUT");
    a.trace = m->trace;
    if ((tv && atoi(tv) != g.V) || (tu && atoi(tu) != a.in_unpool) || (tf && atoi(tf) != a.fout)) a.trace = nullptr;
    // P2M_TRACE_NTH = k: only the k-th (from 0) matching conv launch since p2m_debug_set_trace is logged
    const char* tn = getenv("P2M_TRACE_NTH");
    if (a.trace != nullptr && tn && m->trace_seen++ != atoi(tn)) a.trace = nullptr;
  }
  // single-pass fp16: every conv at fp16_mixed; at fp16 the forward convs only (refuse_fp16 keeps the backward away)
  a.f16 = single_pass(m->precision) ? 1 : 0;
  P2M_TRY(launch_umma_pack_weights(W, fin, fout, transposed, WPACK_ALL, 0.f, wpack, s, a.f16 != 0));
  if (!t1_given) P2M_TRY(launch_cheb_t1(g, a.x, a.in_unpool, a.batch, a.fin, T, s, elide ? &g.real_tiles : nullptr));
  a.t1 = T;
  a.wpack = wpack;
  if (elide) a.tiles = &g.real_tiles;
  P2M_TRY(launch_umma_conv(a, m->kernel_status, m->zero_row, m->sm_count, s));
  if (!elide || iso_mode == 2) return P2M_OK;
  P2M_TRY(launch_umma_pack_weights(W, fin, fout, transposed, WPACK_COMBINED, g.iso_diag, w_iso, s, a.f16 != 0));
  a.t1 = nullptr;
  a.plain = 1;
  a.trace = nullptr;  // the trace buffer holds the connected rows' launch; the isolated rows' GEMM would overwrite it
  a.tiles = (iso_mode == 1 && g.n_rep > 0) ? &g.rep_tiles : &g.iso_tiles;
  a.wpack = w_iso;
  return launch_umma_conv(a, m->kernel_status, m->zero_row, m->sm_count, s);
}

// dT = dz * Wp  ([rows, Fout] x [Fout, 3 Fin]) into T on the tensor cores: three plain GEMMs (one per Chebyshev order,
// N = Fin, K = Fout, B_k[f][o] = W[o][f*3 + k]) with dz scaled into fp16's range by a_scale; single pass (hi-only
// images) at the single-pass precisions
int run_tc_dt(p2m_model* m, const DevLevel& g, int batch, const float* dz, int fin, int fout, const float* W,
              const Epilogue& ep, const float* a_scale, unsigned char* wpack, float* T, cudaStream_t s) {
  const bool f16 = single_pass(m->precision);
  for (int k = 0; k < 3; ++k) {
    P2M_TRY(launch_umma_pack_weights(W, fin, fout, true, k, 0.f, wpack, s, f16));
    UmmaConvArgs a = umma_args(g, batch, dz, 0, fout, fin, ep, T, a_scale);
    a.wpack = wpack;
    a.f16 = f16 ? 1 : 0;
    a.plain = 1;
    a.ldy = 3LL * fin;
    a.y_col0 = k * fin;
    P2M_TRY(launch_umma_conv(a, m->kernel_status, m->zero_row, m->sm_count, s));
  }
  return P2M_OK;
}

// ---- one conv layer, linear part + epilogue: y = epilogue( [T0|T1|T2](x) * Wp^T ) on the path r chose
// keep_wp: also leave the k-major copy of the weights in wp (what the SIMT GEMM reads) for the backward's SIMT dT GEMM
int conv_linear(p2m_model* m, const ConvRoute& r, const Layer& L, int B, const float* x, int in_unpool,
                const float* w_ref, float* T, float* wp, unsigned char* wpack, const Epilogue& ep, float* y,
                cudaStream_t s, bool keep_wp, int iso_mode = 0, const float* head_wt = nullptr,
                float* head_z = nullptr) {
  const int rows = B * L.V;
  const DevLevel& g = m->levels[L.level];
  if (keep_wp || !r.tc) P2M_TRY(launch_permute_w(w_ref, wp, L.fout, L.fin, s));
  if (r.tc) {
    UmmaConvArgs a = umma_args(g, B, x, in_unpool, L.fin, L.fout, ep, y, nullptr);
    a.head_wt = head_wt;
    a.head_z = head_z;
    // the isolated rows' combined weights go into T behind the T1 part (T is 3 Fin wide)
    return run_tc_conv(m, a, w_ref, false, r.elide, iso_mode, false, T, wpack,
                       reinterpret_cast<unsigned char*>(T + (size_t)rows * L.fin), s);
  }
  if (head_z != nullptr) {
    set_error("conv_linear: fused head requested off the tensor-core path");
    return P2M_ERR_INVALID;
  }
  if (thin_conv_supported(L.fin, L.fout) && ep.res == nullptr &&
      thin_conv_scratch_floats(rows, L.fin) <= (size_t)rows * 3 * L.fin) {
    return launch_thin_conv(g, x, in_unpool, rows, L.fin, L.fout, w_ref, ep, T, y, s);  // T doubles as scratch
  }
  P2M_TRY(launch_cheb_basis(g, x, in_unpool, rows, L.fin, T, s));
  P2M_TRY(launch_gemm(T, 3 * L.fin, wp, 3 * L.fin, 0, y, L.fout, rows, L.fout, 3 * L.fin, ep, s));
  return P2M_OK;
}

// BatchNorm of a conv's output z in the training schedule: statistics by the layer's options (launch_bn_stats: batch
// or running; saved statistics, scale / shift), then a = relu?(z * scale + shift) (+ the resampled residual res)
int bn_train_tail(const float* z, int rows, int F, const float* gamma, const float* beta, float* rm, float* rv,
                  int64_t* nbt, const p2m_bn_opts_t& o, double* sums, float* mean, float* invstd, float* scale,
                  float* shift, int relu, const float* res, int res_F, int res_unpool, const InterpTable* it, float* a,
                  cudaStream_t s) {
  P2M_TRY(launch_bn_stats(z, rows, F, gamma, beta, rm, rv, nbt, o, sums, mean, invstd, scale, shift, s));
  return launch_affine_act(z, rows, F, scale, shift, relu, res, res_F, res_unpool, it, a, s);
}

// dW [fout, 3 fin] of a conv on the CUDA cores: the basis of x into T, dWp = dz^T T into the k-major dwp, unpermuted
int simt_dw(const DevLevel& g, const float* x, int in_unpool, int rows, int fin, int fout, const float* dz, float* T,
            float* dwp, float* dw, cudaStream_t s) {
  P2M_TRY(launch_cheb_basis(g, x, in_unpool, rows, fin, T, s));
  P2M_TRY(launch_fill_zero(dwp, sizeof(float) * fout * 3 * fin, s));
  P2M_TRY(launch_gemm_tn_atomic(dz, fout, T, 3 * fin, dwp, 3 * fin, rows, fout, 3 * fin, s));
  return launch_unpermute_w(dwp, dw, fout, fin, s);
}

// dW [fout, 3 fin] of a conv on the tensor cores: T1 of one side into T, then launch_umma_dw on that basis and plain
// tiles of the other side; basis_of_dz: T1 = L~dz (swap = 1), else T1 = L~x.  a_scale scales dz into fp16's range.
// At the single-pass precisions the kernel is k_cheb_dw_f16_umma.
int tc_dw(p2m_model* m, const DevLevel& g, int batch, const float* x, int in_unpool, int fin, const float* dz, int fout,
          bool basis_of_dz, const float* a_scale, float* T, float* dw, cudaStream_t s) {
  P2M_TRY(basis_of_dz ? launch_cheb_t1(g, dz, 0, batch, fout, T, s, nullptr)
                      : launch_cheb_t1(g, x, in_unpool, batch, fin, T, s, nullptr));
  P2M_TRY(launch_fill_zero(dw, sizeof(float) * fout * 3 * fin, s));
  const bool f16 = single_pass(m->precision);
  return basis_of_dz ? launch_umma_dw(g, batch, dz, 0, fout, T, x, in_unpool, fin, 1, a_scale, dw, m->kernel_status,
                                      m->sm_count, s, f16)
                     : launch_umma_dw(g, batch, x, in_unpool, fin, T, dz, 0, fout, 0, a_scale, dw, m->kernel_status,
                                      m->sm_count, s, f16);
}

// fc: joints -> coarsest mesh level (meshnet.py:104-106), as a dense GEMM on the tensor cores (wgmma, fp16x3: also at
// the single-pass fp16 precision, which only changes the Chebyshev convs) or SIMT
int run_fc(const p2m_model* m, const p2m_params_t* P, const WsCommon& w, int B, const float* x, float* out, cudaStream_t s) {
  Epilogue ep;
  ep.bias = P->fc_b;
  if (tc_precision(m->precision) && w.fc_apack != nullptr)
    return launch_umma_gemm({x, m->fc_in, 1}, {P->fc_w, m->fc_in, 1}, B, m->fc_out, m->fc_in, ep, out, w.fc_apack,
                            w.fc_wpack, m->kernel_status, m->sm_count, s);
  return launch_gemm(x, m->fc_in, P->fc_w, m->fc_in, 0, out, m->fc_out, B, m->fc_out, m->fc_in, ep, s);
}

// Fused head (eval): when the next layer is the network's thin head (64 -> 3, same block, no residual) and layer li runs
// on the tensor cores, its epilogue writes Z = act(y) W' (12 floats per row) instead of y, and the head shrinks to its
// two 4-wide sparse products: the 64-wide activation never reaches HBM.
bool fuses_head(const p2m_model* m, const Block& blk, int li, int B, const ConvRoute& r) {
  const Layer& L = m->layers[li];
  if (!m->fuse_head || !r.tc || li + 2 != (int)m->layers.size() || li + 1 >= blk.first_layer + blk.n_layers ||
      blk.has_residual || L.fout != 64 || B * L.V < 64)
    return false;
  const Layer& H = m->layers[li + 1];
  return thin_conv_supported(H.fin, H.fout) && H.fin == L.fout && H.V == L.V;
}

// The route of layer li's backward in p2m_meshnet_backward: the thin head's weights-first backward needs an input that
// is neither unpooled nor a residual source, and not the network input.
ConvRoute backward_route(const p2m_model* m, int li, int B, bool need_dx) {
  const Layer& L = m->layers[li];
  int b = 0;
  while (m->blocks[b].first_layer + m->blocks[b].n_layers <= li) ++b;
  const Block& blk = m->blocks[b];
  const bool first = (li == blk.first_layer);
  const bool in_unpool = first && blk.in_unpool;
  const bool res_here = first && blk.has_residual;
  return conv_route(m, L.level, L.fin, L.fout, B, true, !in_unpool && !res_here && li > 0, need_dx);
}

// p2m_debug_set_capture: n floats of src into the capture slot v[li] / dst, if the caller set one
int capture_copy(float* dst, const float* src, size_t n, cudaStream_t s) {
  if (dst == nullptr) return P2M_OK;
  P2M_CUDA_OK(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return P2M_OK;
}
int capture_copy(const std::vector<float*>& v, int li, const float* src, size_t n, cudaStream_t s) {
  return capture_copy(v.empty() ? nullptr : v[li], src, n, s);
}

// The default elision policy (elide_padding == 1) on a level, whatever the batch and width.
inline bool policy_elided(const DevLevel& g) { return elided(1, g, g.V, 0); }

// Classes of identical isolated rows (eval mode, DevLevel::rep_tiles).  Levels are ordered fine -> coarse, the joint
// graph last; the parent of row r of mesh level k is row r >> 1 of level k + 1 (nearest x2 unpool, meshnet.py:71-78).
// An isolated row is a REPRESENTATIVE if its parent is a connected row (nothing to share), or if it is the left
// child of a parent whose value is computed (any row of a level that is not elided, a representative otherwise);
// every other isolated row equals a representative: its left sibling, or the left child of its parent's
// representative.  Requires what the reference's binary-tree reorder guarantees (lib/coarsening.py:214-258: fake
// nodes are added bottom-up, so both children of a fake node are fake); if a level violates it the classes are
// simply not built (n_rep stays 0) and every isolated row is computed.
int build_padding_classes(p2m_model* m, const p2m_model_desc_t* d) {
  const int n_mesh = d->n_levels - 1;  // the last level is the joint graph
  std::vector<std::vector<char>> iso(n_mesh);
  for (int k = 0; k < n_mesh; ++k) {
    const int V = d->level_size[k];
    const int32_t* rp = d->rowptr[k];
    iso[k].assign(V, 0);
    for (int v = 0; v < V; ++v) iso[k][v] = (rp[v + 1] - rp[v] == 1 && d->colidx[k][rp[v]] == v) ? 1 : 0;
  }
  std::vector<std::vector<int>> rep_of(n_mesh);  // per elided level: representative of each isolated row (itself if rep)
  for (int k = n_mesh - 1; k >= 0; --k) {
    DevLevel& g = m->levels[k];
    if (!policy_elided(g)) continue;
    const int V = g.V;
    const bool has_parent = (k + 1 < n_mesh) && (d->level_size[k + 1] * 2 == V);
    const bool parent_elided = has_parent && policy_elided(m->levels[k + 1]);
    std::vector<int>& ro = rep_of[k];
    ro.assign(V, -1);
    std::vector<int> reps, cdst, csrc;
    bool ok = true;
    for (int r = 0; r < V && ok; ++r) {
      if (!iso[k][r]) continue;
      const int p = r >> 1;
      if (!has_parent || !iso[k + 1][p]) {
        ro[r] = r;
      } else {
        if (!iso[k][r ^ 1]) ok = false;  // both children of a fake vertex must be fake
        const bool parent_computed = !parent_elided || rep_of[k + 1][p] == p;
        if (parent_computed) ro[r] = r & ~1;
        else ro[r] = 2 * rep_of[k + 1][p];
        if (ro[r] < 0 || ro[r] >= V || !iso[k][ro[r]]) ok = false;
      }
      if (ro[r] == r) reps.push_back(r);
      else {
        cdst.push_back(r);
        csrc.push_back(ro[r]);
      }
    }
    for (size_t i = 0; i < csrc.size() && ok; ++i)
      if (ro[csrc[i]] != csrc[i]) ok = false;  // a representative represents itself
    if (!ok || cdst.empty()) {
      ro.assign(V, -1);  // treat the level as fully computed
      for (int r = 0; r < V; ++r)
        if (iso[k][r]) ro[r] = r;
      continue;
    }
    P2M_TRY(build_tileset(reps, d->rowptr[k], d->colidx[k], d->values[k], V, &g.rep_tiles, &m->owned));
    P2M_TRY(upload(m, cdst, &g.copy_dst));
    P2M_TRY(upload(m, csrc, &g.copy_src));
    g.n_rep = (int)reps.size();
    g.n_copy = (int)cdst.size();
  }
  // a level's classes assume that its elided parent level is deduplicated too: keep them only in a chain from the
  // finest level down (n_rep == 0 on a level switches its children back to "parent fully computed" == still valid,
  // because a fully computed parent only adds valid rows)
  return P2M_OK;
}

// bn: the forward's resolved per-layer options, whose buffers are checked too (null: the backward, which reads none)
int check_params(const p2m_model* m, const p2m_params_t* p, const std::vector<p2m_bn_opts_t>* bn) {
  if (!p || !p->fc_w || !p->fc_b || !p->cl_w || !p->cl_b || !p->bn_w || !p->bn_b) {
    set_error("params: null table");
    return P2M_ERR_INVALID;
  }
  for (size_t i = 0; i < m->layers.size(); ++i) {
    if (!p->cl_w[i] || !p->cl_b[i]) {
      set_error("params: null conv weight/bias for layer " + std::to_string(i));
      return P2M_ERR_INVALID;
    }
    if (m->layers[i].bn) {
      if (!p->bn_w[i] || !p->bn_b[i]) {
        set_error("params: null BatchNorm tensor for layer " + std::to_string(i));
        return P2M_ERR_INVALID;
      }
      if (bn) {
        const std::string where = "params: BatchNorm of layer " + std::to_string(i);
        P2M_TRY(check_bn_opts((*bn)[i], p->bn_rm ? p->bn_rm[i] : nullptr, p->bn_rv ? p->bn_rv[i] : nullptr,
                              p->bn_nbt ? p->bn_nbt[i] : nullptr, where.c_str()));
      }
    }
  }
  return P2M_OK;
}

// One option record per layer: the caller's, or the defaults (batch statistics with update in training, running
// statistics in eval).  The last layer has no BatchNorm; its entry is ignored.
std::vector<p2m_bn_opts_t> resolve_bn_opts(const p2m_model* m, int training, const p2m_bn_opts_t* bn) {
  std::vector<p2m_bn_opts_t> out(m->layers.size(), bn_opts_default(training ? P2M_BN_BATCH_UPDATE : P2M_BN_RUNNING));
  for (size_t i = 0; bn && i < out.size(); ++i)
    if (m->layers[i].bn) out[i] = bn[i];
  return out;
}
// The eval schedule (folded BatchNorm, no saved activations) serves a forward without backward whose BatchNorms all
// use running statistics
bool eval_schedule(const p2m_model* m, int training, const std::vector<p2m_bn_opts_t>& bn) {
  if (training) return false;
  for (size_t i = 0; i < m->layers.size(); ++i)
    if (m->layers[i].bn && bn[i].stats != P2M_BN_RUNNING) return false;
  return true;
}

}  // namespace

// =====================================================================================
extern "C" {

const char* p2m_last_error(void) { return g_error.c_str(); }
const char* p2m_version(void) { return "pose2mesh_release_b200 0.1 (sm_90a)"; }
int64_t p2m_launch_count(void) { return g_launches; }
void p2m_launch_count_reset(void) { g_launches = 0; }

int64_t p2m_debug_conv_log(int32_t* out, int max_entries) {
  const int64_t n = g_conv_log_n.load(std::memory_order_relaxed);
  if (out != nullptr && max_entries > 0) {
    const int64_t k = std::min<int64_t>(std::min<int64_t>(n, CONV_LOG_CAP), max_entries);
    std::memcpy(out, g_conv_log, (size_t)k * sizeof(g_conv_log[0]));
  }
  return n;
}
void p2m_debug_conv_log_reset(void) { g_conv_log_n.store(0, std::memory_order_relaxed); }

int p2m_model_create(const p2m_model_desc_t* d, p2m_model_t** out) {
  if (!d || !out || d->n_levels < 1 || (d->n_blocks != 0 && (d->n_blocks < 3 || d->n_levels < 2))) {
    set_error("model_create: bad descriptor");
    return P2M_ERR_INVALID;
  }
  // n_blocks == 0: graph-only handle (levels without a channel plan) for the single-layer entry points
  if (d->n_blocks != 0 && d->n_levels != d->n_blocks - 1) {
    set_error("model_create: need n_levels == n_blocks - 1 (one level per block; the last block re-uses the finest)");
    return P2M_ERR_INVALID;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || d->device >= ndev) {
    set_error("model_create: no usable CUDA device (this library has no CPU path)");
    cudaGetLastError();
    return P2M_ERR_NOGPU;
  }
  cudaDeviceProp prop;
  P2M_CUDA_OK(cudaGetDeviceProperties(&prop, d->device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error(std::string("model_create: device is sm_") + std::to_string(prop.major * 10 + prop.minor) +
              ", this library is built for sm_90a only");
    return P2M_ERR_NOGPU;
  }
  DeviceGuard guard(d->device);
  p2m_model* m = new p2m_model();
  m->device = d->device;
  m->sm_count = m->sm_count_device = prop.multiProcessorCount;
  // ---- levels: CSR with relative offsets
  for (int l = 0; l < d->n_levels; ++l) {
    DevLevel g;
    g.V = d->level_size[l];
    const int32_t* rp = d->rowptr[l];
    g.nnz = rp[g.V];
    std::vector<int> rowptr(rp, rp + g.V + 1), rel(g.nnz);
    std::vector<float> val(d->values[l], d->values[l] + g.nnz);
    for (int v = 0; v < g.V; ++v) {
      g.max_row_nnz = std::max(g.max_row_nnz, rp[v + 1] - rp[v]);
      for (int p = rp[v]; p < rp[v + 1]; ++p) {
        int c = d->colidx[l][p];
        if (c < 0 || c >= g.V) {
          set_error("model_create: column index out of range");
          p2m_model_destroy(m);
          return P2M_ERR_INVALID;
        }
        rel[p] = c - v;
      }
    }
    {
      // exact symmetry of the fp32 values: the entries sorted by (row, col) against the transposed ones
      std::vector<std::tuple<int, int, float>> e, et;
      e.reserve(g.nnz);
      et.reserve(g.nnz);
      double r_max = 0.0;
      for (int v = 0; v < g.V; ++v) {
        double r = 0.0;
        for (int p = rp[v]; p < rp[v + 1]; ++p) {
          const float x = d->values[l][p];
          e.emplace_back(v, d->colidx[l][p], x);
          et.emplace_back(d->colidx[l][p], v, x);
          r += std::fabs((double)x);
        }
        r_max = std::max(r_max, r);
      }
      std::sort(e.begin(), e.end());
      std::sort(et.begin(), et.end());
      g.symmetric = (e == et);
      g.headroom_log2 = (int)std::ceil(std::log2(2.0 * r_max * r_max + 1.0));
    }
    if (d->n_blocks != 0 && !g.symmetric) {
      set_error("model_create: the Laplacian of level " + std::to_string(l) +
                " is not symmetric (the network's backward uses L~ in place of L~^T)");
      p2m_model_destroy(m);
      return P2M_ERR_INVALID;
    }
    int st;
    if ((st = upload(m, rowptr, &g.rowptr)) || (st = upload(m, rel, &g.reloff)) || (st = upload(m, val, &g.val)) ||
        (st = build_umma_level_meta(rp, d->colidx[l], d->values[l], g.V, &g, &m->owned))) {
      p2m_model_destroy(m);
      return st;
    }
    m->levels.push_back(g);
  }
  if (d->n_blocks != 0) {
    int st = build_padding_classes(m, d);
    if (st) {
      p2m_model_destroy(m);
      return st;
    }
  }
  {
    std::vector<float> zrow(64, 0.f);
    int st = upload(m, zrow, &m->zero_row);
    void* hp = nullptr;
    if (!st && (cudaHostAlloc(&hp, 64, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
                cudaHostGetDevicePointer(reinterpret_cast<void**>(&m->kernel_status), hp, 0) != cudaSuccess)) {
      set_error("model_create: cannot allocate the mapped status word");
      if (hp) cudaFreeHost(hp);
      st = P2M_ERR_CUDA;
    }
    if (st) {
      p2m_model_destroy(m);
      return st;
    }
    m->status_host = static_cast<volatile int*>(hp);
    *m->status_host = 0;
  }
  // ---- plan (meshnet.py:21-33, 86-94)
  const int nb = d->n_blocks;
  int off = 0, li = 0;
  for (int b = 0; b < nb; ++b) {
    const int32_t* ch = d->block_chans + off;
    const int len = d->block_len[b];
    if (len < 2) {
      set_error("model_create: block with < 2 channel entries");
      p2m_model_destroy(m);
      return P2M_ERR_INVALID;
    }
    Block blk{};
    blk.first_layer = li;
    blk.n_layers = len - 1;
    blk.level = (b == nb - 1) ? 0 : d->n_levels - 1 - b;
    blk.has_residual = (b >= 1 && b <= nb - 2);
    blk.out_unpool = (b >= 1 && b < nb - 2);
    blk.in_unpool = (b >= 2 && b <= nb - 2);
    blk.cin = ch[0];
    blk.cout = ch[len - 1];
    for (int j = 0; j < len - 1; ++j) {
      const bool last = (b == nb - 1) && (j == len - 2);
      m->layers.push_back(Layer{blk.level, m->levels[blk.level].V, ch[j], ch[j + 1], !last, !last, j == len - 2});
      ++li;
    }
    if (blk.has_residual) {
      int st = build_interp(m, blk.cin, blk.cout, &blk.interp);
      if (st) {
        p2m_model_destroy(m);
        return st;
      }
    }
    m->blocks.push_back(blk);
    off += len;
  }
  // consistency: unpool doubles the level size; block b+1 input channels == block b output channels
  for (int b = 1; b < nb; ++b) {
    const Block& p = m->blocks[b - 1];
    const Block& c = m->blocks[b];
    bool ok = (c.cin == p.cout);
    if (b >= 2) {
      int vp = m->levels[p.level].V, vc = m->levels[c.level].V;
      ok = ok && (p.out_unpool ? (vc == 2 * vp) : (vc == vp));
    }
    if (!ok) {
      set_error("model_create: inconsistent hierarchy / channel plan at block " + std::to_string(b));
      p2m_model_destroy(m);
      return P2M_ERR_INVALID;
    }
  }
  if (nb == 0) {
    *out = m;
    return P2M_OK;
  }
  m->n_joint = m->levels.back().V;
  m->cin = m->blocks[0].cin;
  m->cout = m->blocks[nb - 1].cout;
  m->fc_in = m->n_joint * m->blocks[0].cout;
  m->fc_out = m->levels[m->blocks[1].level].V * m->blocks[1].cin;
  *out = m;
  return P2M_OK;
}

void p2m_model_destroy(p2m_model_t* m) {
  if (!m) return;
  DeviceGuard guard(m->device);
  for (void* p : m->owned) cudaFree(p);
  if (m->status_host) cudaFreeHost(const_cast<int*>(m->status_host));
  for (cudaEvent_t e : m->ev_beg) cudaEventDestroy(e);
  for (cudaEvent_t e : m->ev_end) cudaEventDestroy(e);
  delete m;
}

int p2m_model_num_layers(const p2m_model_t* m) { return m ? (int)m->layers.size() : 0; }

int p2m_model_layer_info(const p2m_model_t* m, int layer, int32_t out[6]) {
  if (!m || layer < 0 || layer >= (int)m->layers.size()) {
    set_error("layer_info: bad layer");
    return P2M_ERR_INVALID;
  }
  const Layer& L = m->layers[layer];
  out[0] = L.level; out[1] = L.V; out[2] = L.fin; out[3] = L.fout; out[4] = L.bn; out[5] = L.relu;
  return P2M_OK;
}

int p2m_debug_kernel_status(p2m_model_t* m, int32_t* out) {
  if (!m || !out) {
    set_error("debug_kernel_status: bad argument");
    return P2M_ERR_INVALID;
  }
  DeviceGuard guard(m->device);
  P2M_CUDA_OK(cudaDeviceSynchronize());
  *out = m->status_host ? *m->status_host : 0;
  return P2M_OK;
}

// Debug: route the tensor-core conv kernel's CTA-0 event log into `dev_buf` (device, 8*512 int64) or disable (NULL).
// Only in libraries built with -DP2M_UMMA_TRACE (P2M_TRACE=1 python -m pose2mesh_release_b200.build --force).
int p2m_debug_set_trace(p2m_model_t* m, void* dev_buf) {
  if (!m) return P2M_ERR_INVALID;
#ifdef P2M_UMMA_TRACE
  m->trace = static_cast<long long*>(dev_buf);
  m->trace_seen = 0;
  return P2M_OK;
#else
  if (dev_buf == nullptr) return P2M_OK;
  set_error("debug_set_trace: this library was built without P2M_UMMA_TRACE");
  return P2M_ERR_INVALID;
#endif
}

int p2m_debug_set_sm_count(p2m_model_t* m, int n) {
  if (!m || n < 0 || n > m->sm_count_device) {
    set_error("debug_set_sm_count: need 0 <= n <= the device's SM count");
    return P2M_ERR_INVALID;
  }
  m->sm_count = n == 0 ? m->sm_count_device : n;
  return P2M_OK;
}

int p2m_debug_set_elide_padding(p2m_model_t* m, int enable) {
  if (!m) return P2M_ERR_INVALID;
  m->elide_padding = enable < 0 ? 0 : (enable > 2 ? 2 : enable);
  return P2M_OK;
}
int p2m_debug_set_dedup_padding(p2m_model_t* m, int enable) {
  if (!m) return P2M_ERR_INVALID;
  m->dedup_padding = enable ? 1 : 0;
  return P2M_OK;
}
int p2m_debug_conv_path(const p2m_model_t* m, int level, int fin, int fout, int32_t out[9]) {
  if (!m || !out || level < 0 || level >= (int)m->levels.size() || fin <= 0 || fout <= 0) {
    set_error("debug_conv_path: bad argument");
    return P2M_ERR_INVALID;
  }
  const DevLevel& g = m->levels[level];
  const ConvRoute r = conv_route(m, level, fin, fout, 1, false);  // what p2m_cheb_conv_fwd / _bwd run
  out[0] = r.tc;
  out[1] = r.tc ? umma_conv_x_stages(g, fin, fout, false) : 0;
  out[2] = r.tc_dw;
  out[3] = r.tc_dw ? umma_dw_x_stages(g) : 0;
  out[4] = r.tc_dt;
  out[5] = r.tc_dt ? umma_conv_x_stages(g, fout, fin, true) : 0;
  out[6] = (g.meta128.n_pattern > 0 && umma_tma_rows(g)) ? 1 : 0;
  out[7] = g.meta128.max_h1;
  out[8] = g.n_iso;
  return P2M_OK;
}

int p2m_debug_conv_tiling(const p2m_model_t* m, int level, int fin, int fout, int32_t out[3]) {
  if (!m || !out || level < 0 || level >= (int)m->levels.size() || fin <= 0 || fout <= 0) {
    set_error("debug_conv_tiling: bad argument");
    return P2M_ERR_INVALID;
  }
  const DevLevel& g = m->levels[level];
  const UmmaConvTiling t = conv_route(m, level, fin, fout, 1, false).tc
                               ? umma_conv_tiling(g, fin, fout, false, single_pass(m->precision))
                               : UmmaConvTiling{0, 0, 0};
  out[0] = t.cols;
  out[1] = t.ns;
  out[2] = t.xs;
  return P2M_OK;
}

int p2m_debug_tile_families(const p2m_model_t* m, int level, int fin, int fout, int32_t out[120]) {
  if (!m || !out || level < 0 || level >= (int)m->levels.size() ||
      umma_tile_families(m->levels[level], fin, fout, reinterpret_cast<int32_t(*)[2][15]>(out)) != P2M_OK) {
    set_error("debug_tile_families: bad argument");
    return P2M_ERR_INVALID;
  }
  return P2M_OK;
}

int p2m_debug_layer_route(const p2m_model_t* m, int layer, int batch, int need_dx, int32_t out[9]) {
  if (!m || !out || layer < 0 || layer >= (int)m->layers.size() || batch <= 0) {
    set_error("debug_layer_route: bad argument");
    return P2M_ERR_INVALID;
  }
  const Layer& L = m->layers[layer];
  int b = 0;
  while (m->blocks[b].first_layer + m->blocks[b].n_layers <= layer) ++b;
  const ConvRoute f = conv_route(m, L.level, L.fin, L.fout, batch, true);  // what forward_eval / forward_train run
  const ConvRoute r = backward_route(m, layer, batch, layer > 0 || need_dx);
  out[0] = f.tc;
  out[1] = f.elide;
  out[2] = r.thin;
  out[3] = r.tc_dw;
  out[4] = r.dw_dz_basis;
  out[5] = r.tc_dx;
  out[6] = r.dx_elide;
  out[7] = r.tc_dt;
  out[8] = fuses_head(m, m->blocks[b], layer, batch, f);
  return P2M_OK;
}

int p2m_debug_set_capture(p2m_model_t* m, const p2m_capture_t* c) {
  if (!m) {
    set_error("debug_set_capture: bad argument");
    return P2M_ERR_INVALID;
  }
  if (!c) {
    m->capture.reset();
    return P2M_OK;
  }
  const size_t nl = m->layers.size();
  auto take = [nl](float* const* p) { return p ? std::vector<float*>(p, p + nl) : std::vector<float*>(); };
  std::unique_ptr<Capture> cap(new Capture());
  cap->z = take(c->z);
  cap->a = take(c->a);
  cap->y = take(c->y);
  cap->g_a = take(c->g_a);
  cap->g_z = take(c->g_z);
  cap->dx = take(c->dx);
  cap->fc_out = c->fc_out;
  cap->fc_dx = c->fc_dx;
  m->capture = std::move(cap);
  return P2M_OK;
}

int p2m_debug_set_fuse_head(p2m_model_t* m, int enable) {
  if (!m) return P2M_ERR_INVALID;
  m->fuse_head = enable ? 1 : 0;
  return P2M_OK;
}

int p2m_model_set_profiling(p2m_model_t* m, int enable) {
  if (!m) {
    set_error("set_profiling: bad argument");
    return P2M_ERR_INVALID;
  }
  DeviceGuard guard(m->device);
  if (enable && m->ev_beg.empty()) {
    m->ev_beg.resize(m->layers.size());
    m->ev_end.resize(m->layers.size());
    for (size_t i = 0; i < m->layers.size(); ++i) {
      P2M_CUDA_OK(cudaEventCreate(&m->ev_beg[i]));
      P2M_CUDA_OK(cudaEventCreate(&m->ev_end[i]));
    }
  }
  m->profiling = enable ? 1 : 0;
  return P2M_OK;
}

int p2m_model_layer_times_ms(p2m_model_t* m, float* out, int n) {
  if (!m || !out || n < (int)m->layers.size() || m->ev_beg.empty()) {
    set_error("layer_times_ms: profiling was not enabled or buffer too small");
    return P2M_ERR_INVALID;
  }
  DeviceGuard guard(m->device);
  for (size_t i = 0; i < m->layers.size(); ++i) {
    P2M_CUDA_OK(cudaEventSynchronize(m->ev_end[i]));
    P2M_CUDA_OK(cudaEventElapsedTime(&out[i], m->ev_beg[i], m->ev_end[i]));
  }
  return P2M_OK;
}

int p2m_model_set_precision(p2m_model_t* m, int precision) {
  if (!m || (precision != P2M_PREC_FP32_SIMT && precision != P2M_PREC_FP16X3_TC && precision != P2M_PREC_FP16_TC &&
             precision != P2M_PREC_FP16_MIXED_TC)) {
    set_error("set_precision: bad argument");
    return P2M_ERR_INVALID;
  }
  m->precision = precision;
  return P2M_OK;
}

size_t p2m_meshnet_workspace_bytes_opts(const p2m_model_t* m, int batch, int training, const p2m_bn_opts_t* bn) {
  if (!m || batch <= 0 || m->layers.empty()) return 0;
  return eval_schedule(m, training, resolve_bn_opts(m, training, bn)) ? EvalWs(m, batch, nullptr).bytes()
                                                                      : TrainWs(m, batch, nullptr).bytes();
}
size_t p2m_meshnet_workspace_bytes(const p2m_model_t* m, int batch, int training) {
  return p2m_meshnet_workspace_bytes_opts(m, batch, training, nullptr);
}
size_t p2m_meshnet_backward_scratch_bytes(const p2m_model_t* m, int batch) {
  if (!m || batch <= 0 || m->layers.empty()) return 0;
  return map_scratch(m, batch, nullptr).bytes;
}
size_t p2m_meshnet_host_io_bytes(const p2m_model_t* m, int batch) {
  if (!m || batch <= 0 || m->layers.empty()) return 0;
  return HostIo(m, batch, nullptr).bytes;
}

// -------------------------------------------------------------------------------------
// The eval forward: folded BatchNorm, rotating buffers, fused head, padding-row dedup, fused output gather (`gathered`)
static int forward_eval(p2m_model_t* m, const p2m_params_t* P, const std::vector<p2m_bn_opts_t>& bn, const float* x,
                        float* y, int B, void* workspace, cudaStream_t s, int gathered) {
  const EvalWs w(m, B, workspace);
  const int nl = (int)m->layers.size();
  // isolated (padding) rows: only class representatives (DevLevel::rep_tiles), or — when the caller takes the gathered
  // real vertices — none at all: no connected row ever reads an isolated one
  const int iso_mode = (!m->dedup_padding || m->elide_padding < 1) ? 0 : (gathered ? 2 : 1);
  const float* cur = x;
  int cur_unpool = 0;
  int cur_buf = -1;  // rotating buffer id holding `cur`
  auto free_rot = [](int a, int b) { return a != 0 && b != 0 ? 0 : (a != 1 && b != 1 ? 1 : 2); };  // not a, not b
  float* head_z = nullptr;  // Z of the thin head, produced by the previous layer's epilogue (fuses_head)
  for (int b = 0; b < (int)m->blocks.size(); ++b) {
    const Block& blk = m->blocks[b];
    const float* block_in = cur;
    const int block_in_unpool = cur_unpool;
    const int block_in_buf = cur_buf;
    for (int j = 0; j < blk.n_layers; ++j) {
      const int li = blk.first_layer + j;
      const Layer& L = m->layers[li];
      const int rows = B * L.V;
      const bool last = (li == nl - 1);
      const bool with_res = L.block_end && blk.has_residual;
      const ConvRoute r = conv_route(m, L.level, L.fin, L.fout, B, true);
      Epilogue ep;
      float* scale = w.scale_scratch;
      float* shift = w.scale_scratch + L.fout;
      if (L.bn) {
        P2M_TRY(launch_bn_fold_eval(P->bn_w[li], P->bn_b[li], P->bn_rm[li], P->bn_rv[li], P->cl_b[li], bn[li].eps,
                                    scale, shift, L.fout, s));
        ep.scale = scale;
        ep.shift = shift;
      } else {
        ep.bias = P->cl_b[li];
      }
      ep.relu = L.relu;
      if (with_res) {
        ep.res = block_in;
        ep.res_F = blk.cin;
        ep.res_unpool = block_in_unpool;
        ep.res_i0 = blk.interp.i0;
        ep.res_i1 = blk.interp.i1;
        ep.res_lam = blk.interp.lam;
      }
      float* out;
      int out_buf = -1;
      if (last) {
        out = y;
        if (gathered) {
          if (!thin_conv_supported(L.fin, L.fout) || with_res) {
            set_error("meshnet_forward_vertices: the head layer is not on the fused-gather path");
            return P2M_ERR_INVALID;
          }
          ep.out_map = m->out_map;
          ep.out_rows = m->out_rows;
          ep.level_V = L.V;
        }
      } else {
        out_buf = free_rot(cur_buf, block_in_buf);
        out = w.rot[out_buf];
      }
      if (m->profiling) P2M_CUDA_OK(cudaEventRecord(m->ev_beg[li], s));
      if (head_z != nullptr) {  // this IS the head, its Z is already there
        P2M_TRY(launch_thin_tail(m->levels[L.level], rows, L.fout, head_z, head_z + (size_t)rows * 12, ep, out, s));
        head_z = nullptr;
      } else if (fuses_head(m, blk, li, B, r)) {
        float* Z = out;  // [rows][12] | U [rows][4] | W' [64][12] inside this layer's (unused) output buffer
        float* wt = Z + (size_t)rows * 16;
        P2M_TRY(launch_thin_prep(P->cl_w[li + 1], L.fout, m->layers[li + 1].fout, wt, s));
        P2M_TRY(conv_linear(m, r, L, B, cur, cur_unpool, P->cl_w[li], w.T, w.wp_scratch, w.wpack, ep, out, s, false,
                            iso_mode, wt, Z));
        head_z = Z;
      } else {
        P2M_TRY(conv_linear(m, r, L, B, cur, cur_unpool, P->cl_w[li], w.T, w.wp_scratch, w.wpack, ep, out, s, false,
                            iso_mode));
      }
      if (m->profiling) P2M_CUDA_OK(cudaEventRecord(m->ev_end[li], s));
      if (m->capture && head_z == nullptr && !gathered)
        P2M_TRY(capture_copy(m->capture->y, li, out, (size_t)rows * L.fout, s));
      cur = out;
      cur_buf = out_buf;
      cur_unpool = 0;
    }
    if (b == 0) {
      cur_buf = free_rot(cur_buf, -1);
      P2M_TRY(run_fc(m, P, w, B, cur, w.rot[cur_buf], s));
      if (m->capture) P2M_TRY(capture_copy(m->capture->fc_out, w.rot[cur_buf], (size_t)B * m->fc_out, s));
      cur = w.rot[cur_buf];
      cur_unpool = 0;
    } else if (blk.out_unpool) {
      cur_unpool = 1;  // nearest x2 unpool is virtual: the next block reads row r>>1
    }
  }
  if (iso_mode == 1 && m->levels[0].n_copy > 0) {
    // fill the output rows of the isolated vertices that were represented by another row of their class
    const DevLevel& g0 = m->levels[0];
    P2M_TRY(launch_copy_rows(y, B, g0.V, m->cout, g0.copy_dst, g0.copy_src, g0.n_copy, s));
  }
  return P2M_OK;
}

// The training forward: each BatchNorm with batch or running statistics by its options; saves what
// p2m_meshnet_backward reads (TrainWs).
static int forward_train(p2m_model_t* m, const p2m_params_t* P, const std::vector<p2m_bn_opts_t>& bn, const float* x,
                         float* y, int B, void* workspace, cudaStream_t s) {
  const TrainWs w(m, B, workspace);
  const float* cur = x;
  int cur_unpool = 0;
  for (int b = 0; b < (int)m->blocks.size(); ++b) {
    const Block& blk = m->blocks[b];
    const float* block_in = cur;
    const int block_in_unpool = cur_unpool;
    for (int j = 0; j < blk.n_layers; ++j) {
      const int li = blk.first_layer + j;
      const Layer& L = m->layers[li];
      const bool with_res = L.block_end && blk.has_residual;
      const ConvRoute r = conv_route(m, L.level, L.fin, L.fout, B, true);
      Epilogue ep;
      ep.bias = P->cl_b[li];
      float* z = L.bn ? w.z[li] : y;  // the last layer, the only one without BatchNorm, writes y
      P2M_TRY(conv_linear(m, r, L, B, cur, cur_unpool, P->cl_w[li], w.T, w.wp[li], w.wpack, ep, z, s, true));
      if (L.bn)
        P2M_TRY(bn_train_tail(z, B * L.V, L.fout, P->bn_w[li], P->bn_b[li], P->bn_rm ? P->bn_rm[li] : nullptr,
                              P->bn_rv ? P->bn_rv[li] : nullptr, P->bn_nbt ? P->bn_nbt[li] : nullptr, bn[li], w.sums, w.mean[li], w.invstd[li], w.scale[li],
                              w.shift[li], L.relu, with_res ? block_in : nullptr, blk.cin, block_in_unpool,
                              with_res ? &blk.interp : nullptr, w.a[li], s));
      if (m->capture && L.bn) {
        P2M_TRY(capture_copy(m->capture->z, li, z, (size_t)B * L.V * L.fout, s));
        P2M_TRY(capture_copy(m->capture->a, li, w.a[li], (size_t)B * L.V * L.fout, s));
      }
      cur = L.bn ? w.a[li] : z;
      cur_unpool = 0;
    }
    if (b == 0) {
      P2M_TRY(run_fc(m, P, w, B, cur, w.fc_out, s));
      if (m->capture) P2M_TRY(capture_copy(m->capture->fc_out, w.fc_out, (size_t)B * m->fc_out, s));
      cur = w.fc_out;
      cur_unpool = 0;
    } else if (blk.out_unpool) {
      cur_unpool = 1;
    }
  }
  return P2M_OK;
}

// Checks the arguments before anything is enqueued, then runs the eval or the training schedule
static int meshnet_forward(p2m_model_t* m, const p2m_params_t* P, const p2m_bn_opts_t* bn_opts, const float* x,
                           float* y, int B, int training, void* workspace, size_t workspace_bytes, p2m_stream_t stream,
                           int gathered) {
  if (!m || !x || !y || B <= 0 || !workspace || m->layers.empty()) {
    set_error("meshnet_forward: bad argument");
    return P2M_ERR_INVALID;
  }
  const std::vector<p2m_bn_opts_t> bn = resolve_bn_opts(m, training, bn_opts);
  const bool eval = eval_schedule(m, training, bn);
  if (gathered && !eval) {
    set_error("meshnet_forward_vertices: every BatchNorm must use running statistics");
    return P2M_ERR_INVALID;
  }
  if (!eval) P2M_TRY(refuse_fp16(m, "meshnet_forward (training schedule)"));
  P2M_TRY(check_params(m, P, &bn));
  P2M_TRY(check_kernel_status(m, "meshnet_forward"));
  DeviceGuard guard(m->device);
  const size_t need = p2m_meshnet_workspace_bytes_opts(m, B, training, bn_opts);
  if (need > workspace_bytes) {
    set_error("meshnet_forward: workspace too small (" + std::to_string(workspace_bytes) + " < " +
              std::to_string(need) + ")");
    return P2M_ERR_WORKSPACE;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return eval ? forward_eval(m, P, bn, x, y, B, workspace, s, gathered) : forward_train(m, P, bn, x, y, B, workspace, s);
}

int p2m_meshnet_forward_opts(p2m_model_t* m, const p2m_params_t* P, const p2m_bn_opts_t* bn, const float* x, float* y,
                             int B, int training, void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  return meshnet_forward(m, P, bn, x, y, B, training, workspace, workspace_bytes, stream, 0);
}
int p2m_meshnet_forward(p2m_model_t* m, const p2m_params_t* P, const float* x, float* y, int B, int training,
                        void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  return meshnet_forward(m, P, nullptr, x, y, B, training, workspace, workspace_bytes, stream, 0);
}

int p2m_model_set_output_gather(p2m_model_t* m, const int32_t* vertex_of_slot, int n_slots) {
  if (!m || m->layers.empty() || !vertex_of_slot || n_slots <= 0 || n_slots > m->levels[0].V) {
    set_error("set_output_gather: bad argument");
    return P2M_ERR_INVALID;
  }
  const int V0 = m->levels[0].V;
  std::vector<int> map(V0, -1);
  for (int j = 0; j < n_slots; ++j) {
    const int v = vertex_of_slot[j];
    if (v < 0 || v >= V0 || map[v] >= 0) {
      set_error("set_output_gather: index out of range or repeated");
      return P2M_ERR_INVALID;
    }
    map[v] = j;
  }
  DeviceGuard guard(m->device);
  if (m->out_map == nullptr) {  // one [V0] map per handle, overwritten in place by later calls
    P2M_TRY(upload(m, map, &m->out_map));
  } else {
    // earlier forwards may still be reading the old map on their streams
    P2M_CUDA_OK(cudaDeviceSynchronize());
    P2M_CUDA_OK(cudaMemcpy(m->out_map, map.data(), sizeof(int) * V0, cudaMemcpyHostToDevice));
  }
  m->out_rows = n_slots;
  return P2M_OK;
}

int p2m_meshnet_forward_vertices(p2m_model_t* m, const p2m_params_t* P, const float* x, float* y_vertices, int B,
                                 void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  if (!m || !m->out_map) {
    set_error("meshnet_forward_vertices: call p2m_model_set_output_gather first");
    return P2M_ERR_INVALID;
  }
  return meshnet_forward(m, P, nullptr, x, y_vertices, B, 0, workspace, workspace_bytes, stream, 1);
}

static int forward_host_impl(p2m_model_t* m, const p2m_params_t* P, const float* x_host, float* y_host, int B,
                             void* workspace, size_t workspace_bytes, p2m_stream_t stream, int gathered) {
  if (!m || !x_host || !y_host || B <= 0 || !workspace || m->layers.empty() || (gathered && !m->out_map)) {
    set_error(gathered && m && !m->out_map ? "meshnet_forward_vertices_host: call p2m_model_set_output_gather first"
                                           : "meshnet_forward_host: bad argument");
    return P2M_ERR_INVALID;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t out_rows = gathered ? (size_t)m->out_rows : (size_t)m->levels[0].V;
  const size_t xb = (size_t)B * m->n_joint * m->cin * 4, yb = (size_t)B * out_rows * m->cout * 4;
  const size_t need = p2m_meshnet_workspace_bytes(m, B, 0);
  const HostIo io(m, B, static_cast<char*>(workspace) + need);
  if (workspace_bytes < need + io.bytes) {
    set_error("meshnet_forward_host: workspace too small");
    return P2M_ERR_WORKSPACE;
  }
  DeviceGuard guard(m->device);
  P2M_CUDA_OK(cudaMemcpyAsync(io.x, x_host, xb, cudaMemcpyHostToDevice, s));
  P2M_TRY(meshnet_forward(m, P, nullptr, io.x, io.y, B, 0, workspace, need, stream, gathered));
  P2M_CUDA_OK(cudaMemcpyAsync(y_host, io.y, yb, cudaMemcpyDeviceToHost, s));
  P2M_CUDA_OK(cudaStreamSynchronize(s));
  return check_kernel_status(m, "meshnet_forward_host");
}

int p2m_meshnet_forward_host(p2m_model_t* m, const p2m_params_t* P, const float* x_host, float* y_host, int B,
                             void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  return forward_host_impl(m, P, x_host, y_host, B, workspace, workspace_bytes, stream, 0);
}

int p2m_meshnet_forward_vertices_host(p2m_model_t* m, const p2m_params_t* P, const float* x_host, float* y_vertices_host,
                                      int B, void* workspace, size_t workspace_bytes, p2m_stream_t stream) {
  return forward_host_impl(m, P, x_host, y_vertices_host, B, workspace, workspace_bytes, stream, 1);
}

// -------------------------------------------------------------------------------------
int p2m_meshnet_backward(p2m_model_t* m, const p2m_params_t* P, const p2m_params_t* G, const float* x, const float* dy,
                         float* dx, int B, void* workspace, size_t workspace_bytes, void* scratch, size_t scratch_bytes,
                         p2m_stream_t stream) {
  return p2m_meshnet_backward_opts(m, P, G, nullptr, x, dy, dx, B, workspace, workspace_bytes, scratch, scratch_bytes,
                                   stream);
}
int p2m_meshnet_backward_opts(p2m_model_t* m, const p2m_params_t* P, const p2m_params_t* G, const p2m_bn_opts_t* bn_opts,
                              const float* x, const float* dy, float* dx, int B, void* workspace,
                              size_t workspace_bytes, void* scratch, size_t scratch_bytes, p2m_stream_t stream) {
  if (!m || !x || !dy || B <= 0 || !workspace || !scratch || m->layers.empty()) {
    set_error("meshnet_backward: bad argument");
    return P2M_ERR_INVALID;
  }
  P2M_TRY(refuse_fp16(m, "meshnet_backward"));
  P2M_TRY(check_params(m, P, nullptr));
  P2M_TRY(check_params(m, G, nullptr));
  const std::vector<p2m_bn_opts_t> bn = resolve_bn_opts(m, 1, bn_opts);
  P2M_TRY(check_kernel_status(m, "meshnet_backward"));
  DeviceGuard guard(m->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const TrainWs w(m, B, workspace);
  BwdMap sc = map_scratch(m, B, scratch);
  if (w.bytes() > workspace_bytes || sc.bytes > scratch_bytes) {
    set_error("meshnet_backward: workspace/scratch too small");
    return P2M_ERR_WORKSPACE;
  }
  const int nb = (int)m->blocks.size();
  const float* g_cur = dy;
  int g_cur_buf = -2;  // -2: external (dy)
  int keep_buf = -1;   // buffer holding g_out of the block being processed (residual path)
  const float* keep_ptr = nullptr;
  auto free_buf = [&](int a, int b2, int c) {
    for (int i = 0; i < 4; ++i)
      if (i != a && i != b2 && i != c) return i;
    return -1;
  };
  for (int b = nb - 1; b >= 0; --b) {
    const Block& blk = m->blocks[b];
    // input of this block (physical tensor + unpool flag)
    const float* block_in;
    if (b == 0)
      block_in = x;
    else if (b == 1)
      block_in = w.fc_out;
    else
      block_in = w.a[m->blocks[b - 1].first_layer + m->blocks[b - 1].n_layers - 1];
    for (int j = blk.n_layers - 1; j >= 0; --j) {
      const int li = blk.first_layer + j;
      const Layer& L = m->layers[li];
      const DevLevel& g = m->levels[L.level];
      const int rows = B * L.V;
      const float* inp = (j == 0) ? block_in : w.a[li - 1];
      const int in_unpool = (j == 0) ? blk.in_unpool : 0;
      const float* g_z = g_cur;
      int gz_buf = g_cur_buf;
      if (L.block_end && blk.has_residual) {
        keep_buf = g_cur_buf;
        keep_ptr = g_cur;
      }
      const bool need_dx = !(li == 0 && dx == nullptr);
      const bool res_here = (j == 0) && blk.has_residual;
      const ConvRoute r = backward_route(m, li, B, need_dx);
      if (m->capture) P2M_TRY(capture_copy(m->capture->g_a, li, g_cur, (size_t)rows * L.fout, s));
      const bool want_scale = r.tc_dw || r.tc_dx || r.tc_dt;
      bool have_scale = false;
      if (L.bn) {
        int tgt = (g_cur_buf >= 0 && g_cur_buf != keep_buf) ? g_cur_buf : free_buf(g_cur_buf, keep_buf, -1);
        // frozen (running statistics): no batch-mean terms, and the conv bias gets sum_rows g_z
        const bool frozen = bn[li].stats == P2M_BN_RUNNING;
        P2M_TRY(launch_bn_relu_bwd(w.z[li], g_cur, rows, L.fout, P->bn_w[li], w.scale[li], w.shift[li], w.mean[li],
                                   w.invstd[li], L.relu, sc.sums, G->bn_w[li], G->bn_b[li], sc.G[tgt], s,
                                   want_scale ? sc.a_scale : nullptr, frozen, frozen ? G->cl_b[li] : nullptr));
        have_scale = want_scale;
        g_z = sc.G[tgt];
        gz_buf = tgt;
        // with batch statistics the bias of a conv in front of a BatchNorm has a mathematically zero gradient (the
        // batch mean removes it): db = sum_rows dz = 0 exactly, where the reference accumulates fp32 rounding noise
        if (!frozen) P2M_TRY(launch_fill_zero(G->cl_b[li], sizeof(float) * L.fout, s));
      } else {
        P2M_TRY(launch_col_sum(g_z, rows, L.fout, sc.sums, G->cl_b[li], s));
      }
      if (want_scale && !have_scale) P2M_TRY(launch_absmax_scale(g_z, (long long)rows * L.fout, sc.a_scale, s));
      if (m->capture) P2M_TRY(capture_copy(m->capture->g_z, li, g_z, (size_t)rows * L.fout, s));
      float* out = nullptr;
      int out_buf = -1;
      if (need_dx) {
        if (li == 0) {
          out = dx;
        } else {
          out_buf = free_buf(gz_buf, keep_buf, -1);
          out = sc.G[out_buf];
        }
      }
      if (r.thin) {
        // weights-first backward of the thin head: dW and dX from the 3-wide basis of dz, X read once
        P2M_TRY(launch_thin_conv_bwd(g, inp, rows, L.fin, L.fout, P->cl_w[li], g_z, sc.thin, out, G->cl_w[li],
                                     m->sm_count, s));
      } else {
        // dW.  tensor-core path: T2 of one side is formed on chip by the forward's producers from T1 = L~(that side)
        // and contracted with the (power-of-two scaled) plain tiles of the other side by MN-major wgmma; otherwise
        // SIMT: materialise T, dWp = g_z^T T.
        // With dw_dz_basis: sum_rows dz (x) T_k(X) = sum_rows T_k(dz) (x) X  (L~ symmetric), the basis of the GRADIENT,
        // whose first sparse product the backward-data pass below needs anyway, contracted with plain tiles of the layer
        // input.  Otherwise the basis of the layer input (w.T is overwritten by the dX pass's own T1 pass below).
        if (r.dw_dz_basis || r.tc_dw)
          P2M_TRY(tc_dw(m, g, B, inp, in_unpool, L.fin, g_z, L.fout, r.dw_dz_basis, sc.a_scale, w.T, G->cl_w[li], s));
        else
          P2M_TRY(simt_dw(g, inp, in_unpool, rows, L.fin, L.fout, g_z, w.T, sc.dwp, G->cl_w[li], s));
      }
      // dX
      if (need_dx && r.tc_dx) {
        // Backward-data IS a forward conv: dXl = [dz | L~dz | (2L~^2 - I)dz] W'^T with W'[f][o*3+k] = W[o][f*3+k]
        // (L~ symmetric) — the T1 pass and the tensor-core conv kernel of the forward, run on dz (scaled into fp16's
        // range by a power of two), with the padding-vertex elision of the forward.  An identity residual gradient
        // is added in the epilogue; the pair-sum of the virtual unpool and a resampled residual need a finishing pass.
        const bool identity_res = res_here && blk.cin == blk.cout;
        const bool finish = in_unpool || (res_here && !identity_res);
        float* dst = finish ? sc.U : out;
        Epilogue ep;
        if (identity_res) {
          ep.res = keep_ptr;
          ep.res_F = blk.cout;
          ep.res_i0 = blk.interp.i0;
          ep.res_i1 = blk.interp.i1;
          ep.res_lam = blk.interp.lam;
        }
        // (the dW from the basis of dz above already left L~dz of every row in w.T)
        P2M_TRY(run_tc_conv(m, umma_args(g, B, g_z, 0, L.fout, L.fin, ep, dst, sc.a_scale), P->cl_w[li], true,
                            r.dx_elide, 0, r.dw_dz_basis, w.T, sc.wpack, sc.wpack_iso, s));
        if (finish)
          P2M_TRY(launch_dx_finish(dst, rows, L.fin, (res_here && !identity_res) ? keep_ptr : nullptr, blk.cout,
                                   (res_here && !identity_res) ? &blk.interp : nullptr, in_unpool, out, s));
      } else if (need_dx && !r.thin) {
        // dT = g_z * Wp  ([rows, Fout] x [Fout, 3 Fin]) on the tensor cores or SIMT
        if (r.tc_dt)
          P2M_TRY(run_tc_dt(m, g, B, g_z, L.fin, L.fout, P->cl_w[li], Epilogue(), sc.a_scale, sc.wpack, w.T, s));
        else
          P2M_TRY(launch_gemm(g_z, L.fout, w.wp[li], 3 * L.fin, 1, w.T, 3 * L.fin, rows, 3 * L.fin, L.fout, Epilogue(),
                              s));
        P2M_TRY(launch_cheb_basis_bwd(g, w.T, rows, L.fin, sc.U, res_here ? keep_ptr : nullptr, blk.cout,
                                      res_here ? &blk.interp : nullptr, in_unpool, out, s));
      }
      if (need_dx) {
        if (m->capture)  // (an unpooled input has half the layer's rows)
          P2M_TRY(capture_copy(m->capture->dx, li, out, (size_t)(in_unpool ? rows / 2 : rows) * L.fin, s));
        g_cur = out;
        g_cur_buf = out_buf;
      }
      if (j == 0) {
        keep_buf = -1;
        keep_ptr = nullptr;
      }
    }
    if (b == 1) {  // fc backward (meshnet.py:104-106)
      const float* a0 = w.a[m->blocks[0].first_layer + m->blocks[0].n_layers - 1];  // [B, fc_in]
      P2M_TRY(launch_col_sum(g_cur, B, m->fc_out, sc.sums, G->fc_b, s));
      P2M_TRY(launch_fill_zero(G->fc_w, sizeof(float) * (size_t)m->fc_out * m->fc_in, s));
      P2M_TRY(launch_gemm_tn_atomic(g_cur, m->fc_out, a0, m->fc_in, G->fc_w, m->fc_in, B, m->fc_out, m->fc_in, s));
      int out_buf = free_buf(g_cur_buf, -1, -1);
      Epilogue none;
      P2M_TRY(launch_gemm(g_cur, m->fc_out, P->fc_w, m->fc_in, 1, sc.G[out_buf], m->fc_in, B, m->fc_in, m->fc_out, none, s));
      g_cur = sc.G[out_buf];
      g_cur_buf = out_buf;
      if (m->capture) P2M_TRY(capture_copy(m->capture->fc_dx, g_cur, (size_t)B * m->fc_in, s));
    }
  }
  return P2M_OK;
}

// -------------------------------------------------------------------------------------
}  // extern "C"

namespace {
// The single-layer entry points take arbitrary user tensors, so on the tensor cores both fp16x3 operands are brought
// into fp16's range first: the basis by a power of two from max|x| that leaves 2^h of headroom for T1 and T2
// (DevLevel::headroom_log2; the kernel's a_scale, undone in its epilogue), the weights by a power of two from max|W|
// that replaces their fixed 2^6 packing scale (undone by a rescaled epilogue).  Both are exact: the result is the one
// an unscaled split would give wherever that split neither overflows nor loses its lo part to fp16's subnormals.
struct RangeScales {
  float* a_scale;  // device scalars
  float* w_scale;
  float* x_scale;
  float* vec;      // [2 max(fin, fout)]: rescaled epilogue scale | shift
};
// w_out = W * w_scale / 2^6: what launch_umma_pack_weights (x 2^6) then turns into W * w_scale
int prescale_weights(const float* W, long long n, const RangeScales& r, float* w_out, cudaStream_t s) {
  P2M_TRY(launch_absmax_scale(W, n, r.w_scale, s));
  return launch_scale_by(W, n, r.w_scale, 0, 1.f / 64.f, w_out, s);
}

// Workspace of the single-layer entry points (one map for forward and backward)
struct LayerWs {
  float* T;              // [rows, 3 fin]: basis, T1 (+ the isolated rows' image) or dT
  float* wp;             // k-major weights of the SIMT GEMMs
  float* w2;             // range-normalised weights (tensor cores); backward: first the SIMT dW in k-major order
  float* U;              // backward: [rows, fin] range-normalised input, then scratch of the basis backward
  float* z;              // forward: [rows, fout] pre-BatchNorm output
  double* sums;          // [2 max(fin, fout)]
  float* sc;             // [2 fout]: BatchNorm scale | shift (forward), a_scale (backward)
  unsigned char* wpack;  // weight images of the tensor-core conv / dT GEMMs
  RangeScales rs;
  size_t bytes;
};
LayerWs map_layer_workspace(void* base, size_t rows, int fin, int fout) {
  LayerWs w;
  Bump b(base);
  w.T = b.take<float>(rows * 3 * fin);
  w.wp = b.take<float>((size_t)fout * 3 * fin);
  w.w2 = b.take<float>((size_t)fout * 3 * fin);
  w.U = b.take<float>(rows * fin);
  w.z = b.take<float>(rows * fout);
  w.sums = b.take<double>(2 * (size_t)std::max(fin, fout));
  w.sc = b.take<float>(2 * (size_t)fout);
  w.wpack = b.take<unsigned char>(wpack_capacity(false, fin, fout) + 16);
  float* sc = b.take<float>(4);
  w.rs = RangeScales{sc, sc + 1, sc + 2, b.take<float>(2 * (size_t)std::max(fin, fout))};
  w.bytes = b.off;
  return w;
}
}  // namespace

extern "C" {

size_t p2m_cheb_conv_workspace_bytes(const p2m_model_t* m, int level, int batch, int fin, int fout) {
  if (!m || level < 0 || level >= (int)m->levels.size()) return 0;
  return map_layer_workspace(nullptr, (size_t)batch * m->levels[level].V, fin, fout).bytes + ALIGN;
}

int p2m_cheb_conv_fwd(p2m_model_t* m, const p2m_conv_fwd_args_t* a, void* workspace, size_t workspace_bytes,
                      p2m_stream_t stream) {
  if (!m || !a || !a->x || !a->weight || !a->bias || !a->y || a->level < 0 || a->level >= (int)m->levels.size()) {
    set_error("cheb_conv_fwd: bad argument");
    return P2M_ERR_INVALID;
  }
  if (a->bn_mode == 2) P2M_TRY(refuse_fp16(m, "cheb_conv_fwd (batch-statistics BatchNorm)"));
  if (workspace_bytes < p2m_cheb_conv_workspace_bytes(m, a->level, a->batch, a->fin, a->fout)) {
    set_error("cheb_conv_fwd: workspace too small");
    return P2M_ERR_WORKSPACE;
  }
  P2M_TRY(check_kernel_status(m, "cheb_conv_fwd"));
  DeviceGuard guard(m->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const DevLevel& g = m->levels[a->level];
  const Layer L{a->level, g.V, a->fin, a->fout};
  const size_t rows = (size_t)a->batch * L.V;
  const LayerWs w = map_layer_workspace(workspace, rows, L.fin, L.fout);
  const ConvRoute r = conv_route(m, a->level, L.fin, L.fout, a->batch, false);
  // on the tensor cores: range-normalised operands (RangeScales).  That kernel moves x and output rows in 16-byte
  // pieces, so a caller's x or y off 16-byte alignment (e.g. a tensor view at an odd offset) takes the CUDA-core conv.
  auto conv = [&](const Epilogue& e, float* out) -> int {
    if (!r.tc || ((reinterpret_cast<uintptr_t>(a->x) | reinterpret_cast<uintptr_t>(out)) & 15)) {
      ConvRoute simt = r;
      simt.tc = false;
      return conv_linear(m, simt, L, a->batch, a->x, 0, a->weight, w.T, w.wp, w.wpack, e, out, s, false);
    }
    P2M_TRY(prescale_weights(a->weight, (long long)L.fout * 3 * L.fin, w.rs, w.w2, s));
    P2M_TRY(launch_absmax_scale(a->x, (long long)rows * L.fin, w.rs.a_scale, s, g.headroom_log2));
    Epilogue er;
    er.scale = w.rs.vec;
    er.shift = w.rs.vec + L.fout;
    er.relu = e.relu;
    P2M_TRY(launch_rescaled_epilogue(e, w.rs.w_scale, 64.f, L.fout, w.rs.vec, w.rs.vec + L.fout, s));
    return run_tc_conv(m, umma_args(g, a->batch, a->x, 0, L.fin, L.fout, er, out, w.rs.a_scale), w.w2, false, false, 0,
                       false, w.T, w.wpack, nullptr, s);
  };
  Epilogue ep;
  if (a->bn_mode == 0) {
    ep.bias = a->bias;
    ep.relu = a->relu;
    return conv(ep, a->y);
  }
  if (!a->bn_weight || !a->bn_bias) {
    set_error("cheb_conv_fwd: BatchNorm parameters missing");
    return P2M_ERR_INVALID;
  }
  if (a->bn_mode == 1) {
    if (!a->bn_running_mean || !a->bn_running_var) {
      set_error("cheb_conv_fwd: running stats missing");
      return P2M_ERR_INVALID;
    }
    P2M_TRY(launch_bn_fold_eval(a->bn_weight, a->bn_bias, a->bn_running_mean, a->bn_running_var, a->bias, 1e-5, w.sc,
                                w.sc + L.fout, L.fout, s));
    ep.scale = w.sc;
    ep.shift = w.sc + L.fout;
    ep.relu = a->relu;
    return conv(ep, a->y);
  }
  ep.bias = a->bias;
  P2M_TRY(conv(ep, w.z));
  return bn_train_tail(w.z, (int)rows, L.fout, a->bn_weight, a->bn_bias, a->bn_running_mean, a->bn_running_var,
                       a->bn_num_batches_tracked, bn_opts_default(P2M_BN_BATCH_UPDATE), w.sums, a->save_mean, a->save_invstd, w.sc, w.sc + L.fout, a->relu,
                       nullptr, 0, 0, nullptr, a->y, s);
}

int p2m_cheb_conv_bwd(p2m_model_t* m, const p2m_conv_bwd_args_t* a, void* workspace, size_t workspace_bytes,
                      p2m_stream_t stream) {
  if (!m || !a || !a->x || !a->weight || !a->dz || !a->dweight || !a->dbias || a->level < 0 ||
      a->level >= (int)m->levels.size()) {
    set_error("cheb_conv_bwd: bad argument");
    return P2M_ERR_INVALID;
  }
  P2M_TRY(refuse_fp16(m, "cheb_conv_bwd"));
  if (workspace_bytes < p2m_cheb_conv_workspace_bytes(m, a->level, a->batch, a->fin, a->fout)) {
    set_error("cheb_conv_bwd: workspace too small");
    return P2M_ERR_WORKSPACE;
  }
  P2M_TRY(check_kernel_status(m, "cheb_conv_bwd"));
  DeviceGuard guard(m->device);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const DevLevel& g = m->levels[a->level];
  const int fin = a->fin, fout = a->fout;
  const size_t rows = (size_t)a->batch * g.V;
  const LayerWs w = map_layer_workspace(workspace, rows, fin, fout);
  const RangeScales& rs = w.rs;
  float* a_scale = w.sc;  // device scalar for the tensor-core paths (the forward's scale/shift slot is free here)
  const ConvRoute r = conv_route(m, a->level, fin, fout, a->batch, false, false, a->dx != nullptr);
  if (!g.symmetric) {
    set_error("cheb_conv_bwd: the Laplacian is not symmetric; the backward kernels apply L~ where the gradient needs "
              "L~^T");
    return P2M_ERR_INVALID;
  }
  P2M_TRY(launch_col_sum(a->dz, (int)rows, fout, w.sums, a->dbias, s));
  if (r.tc_dw) {
    P2M_TRY(launch_absmax_scale(a->dz, (long long)rows * fout, a_scale, s));
    // the layer input into fp16's range as well (with the basis headroom), in U (free until the dX pass); dW then
    // comes out multiplied by that power of two.  L~U goes into the first rows x fin floats of T, which nothing reads
    // before the dX pass overwrites it.
    P2M_TRY(launch_absmax_scale(a->x, (long long)rows * fin, rs.x_scale, s, g.headroom_log2));
    P2M_TRY(launch_scale_by(a->x, (long long)rows * fin, rs.x_scale, 0, 1.f, w.U, s));
    P2M_TRY(tc_dw(m, g, a->batch, w.U, 0, fin, a->dz, fout, false, a_scale, w.T, a->dweight, s));
    P2M_TRY(launch_scale_by(a->dweight, (long long)fout * 3 * fin, rs.x_scale, 1, 1.f, a->dweight, s));
  } else {
    P2M_TRY(simt_dw(g, a->x, 0, (int)rows, fin, fout, a->dz, w.T, w.w2, a->dweight, s));
  }
  if (a->dx) {
    Epilogue none;
    if (r.tc_dt) {
      if (!r.tc_dw) P2M_TRY(launch_absmax_scale(a->dz, (long long)rows * fout, a_scale, s));
      // weights range-normalised into w2 (the SIMT weight gradient above is done with it); the plain GEMMs' epilogue
      // undoes the scale
      P2M_TRY(prescale_weights(a->weight, (long long)fout * 3 * fin, rs, w.w2, s));
      none.scale = rs.vec;
      none.shift = rs.vec + fin;
      P2M_TRY(launch_rescaled_epilogue(Epilogue(), rs.w_scale, 64.f, fin, rs.vec, rs.vec + fin, s));
      P2M_TRY(run_tc_dt(m, g, a->batch, a->dz, fin, fout, w.w2, none, a_scale, w.wpack, w.T, s));
    } else {
      P2M_TRY(launch_permute_w(a->weight, w.wp, fout, fin, s));
      P2M_TRY(launch_gemm(a->dz, fout, w.wp, 3 * fin, 1, w.T, 3 * fin, (int)rows, 3 * fin, fout, none, s));
    }
    P2M_TRY(launch_cheb_basis_bwd(g, w.T, (int)rows, fin, w.U, nullptr, 0, nullptr, 0, a->dx, s));
  }
  return P2M_OK;
}

}  // extern "C"
