/*
 * p2m_b200.h — C ABI of libp2m_b200.so: the H100-native (sm_90a) MeshNet hot path of
 * hongsukchoi/Pose2Mesh_RELEASE.
 *
 * The reference has no FFI / operator registry: its boundary is the Python nn.Module contract
 *   models.meshnet.get_model(...) / Pose2Mesh.forward(x)              lib/models/meshnet.py:80-123
 *   models.backbones.cheby_graph_conv.graph_conv_cheby(x,cl,bn,L,..)  lib/models/backbones/cheby_graph_conv.py:5
 * (SURVEY.md §8b).  This header is the C boundary a binding (ctypes here, see INTEGRATION.md) sits
 * on: plain pointers and sizes, no torch types.  All `const float*` / `float*` data arguments are
 * DEVICE pointers owned by the caller unless a function name ends in `_host`.  Every function
 * returns 0 on success or a non-zero p2m_status; p2m_last_error() gives the message (thread-local).
 * Nothing here throws or aborts, and the library keeps no global mutable state (per-handle device
 * buffers and thread-local error / launch-count bookkeeping only), so one handle per device can be
 * driven from concurrent threads (nn.DataParallel, lib/core/base.py:108).  Entry points that touch
 * the device make the handle's device (without a handle: the data arrays' device) current for their
 * own duration and restore the caller's.
 */
#ifndef P2M_B200_H_
#define P2M_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct p2m_model p2m_model_t;
typedef void* p2m_stream_t; /* cudaStream_t */

enum p2m_status {
  P2M_OK = 0,
  P2M_ERR_INVALID = 1,   /* bad argument / unsupported shape */
  P2M_ERR_CUDA = 2,      /* a CUDA runtime call or kernel launch failed */
  P2M_ERR_WORKSPACE = 3, /* workspace too small */
  P2M_ERR_NOGPU = 4      /* no usable sm_90 device */
};

enum p2m_precision {
  P2M_PREC_FP32_SIMT = 0, /* fp32 FFMA on CUDA cores (all shapes; the parity baseline)          */
  P2M_PREC_FP16X3_TC = 1, /* wgmma f16 -> f32, error-compensated 3-term fp16 split (~2^-21) */
  P2M_PREC_FP16_TC = 2,   /* inference only: single-pass wgmma, fp16 operands, fp32 accumulate   */
  P2M_PREC_FP16_MIXED_TC = 3 /* mixed-precision training: single-pass wgmma in forward and backward */
};
/* P2M_PREC_FP16_TC: the Chebyshev convs of the eval forward round both operands to the nearest fp16 (activations
 * unscaled, weights x 2^6) and accumulate in fp32: one MMA per 16 features instead of three, a per-product relative
 * error of at most 2^-10 + 2^-22 (fp16x3: ~2^-21).  Everything else runs as at fp16x3: the T1 pass, the epilogues, the
 * fc dense GEMM (fp16x3) and the thin head.  Entry points at this precision: p2m_meshnet_forward(_opts) in the eval
 * schedule, p2m_meshnet_forward_vertices, p2m_meshnet_forward_host (and _vertices_host) and p2m_cheb_conv_fwd (bn_mode
 * 0 or 1).  The training schedule (training = 1, or BatchNorm options that select it), p2m_meshnet_backward(_opts),
 * p2m_cheb_conv_bwd and p2m_cheb_conv_fwd with bn_mode 2 return P2M_ERR_INVALID before any device work.            */
/* P2M_PREC_FP16_MIXED_TC: fp16 operands, fp32 accumulation, fp32 master weights and fp32 BatchNorm, for training.  The
 * eval forward runs exactly the kernels of P2M_PREC_FP16_TC (bitwise equal outputs).  In the training forward and the
 * backward every Chebyshev-conv pass that runs on the tensor cores at fp16x3 runs single-pass instead: the forward
 * convs (with the padding elision's index-list tiles and isolated-row GEMM), backward-data (the conv on dz, its
 * isolated-row GEMM, or the three dT GEMMs; dz scaled into fp16's range by a power of two found on the device) and the
 * weight gradient (k_cheb_dw_f16_umma).  Each pass runs where it runs at fp16x3 (the same routes).  The fc keeps its
 * fp16x3 dense GEMM, the thin layers their CUDA-core kernels and PoseNet its fp16x3 GEMMs.  Every entry point accepts it. */

/* ---- the fixed mesh hierarchy + channel plan ---------------------------------------------------
 * Replaces what Pose2Mesh.__init__ derives from graph_L (meshnet.py:17-37,61-62): `n_levels`
 * Laplacians ordered fine -> coarse with the joint graph LAST and the second-coarsest mesh level
 * already removed (meshnet.py:35).  CSR arrays are HOST pointers (copied to the device here);
 * values are the float32 cast of the reference's float64 CSR (graph_utils.py:98-109).
 * `block_chans` is the concatenation of the per-block channel chains (meshnet.py:21-33), e.g. for
 * the SMPL plan {5,32,64,64, 64,128,256, ...}; `block_len[i]` is the length of chain i.           */
typedef struct {
  int32_t n_levels;
  const int32_t* level_size;        /* [n_levels] vertices per level                                  */
  const int32_t* const* rowptr;     /* [n_levels][V+1]                                                */
  const int32_t* const* colidx;     /* [n_levels][nnz]                                                */
  const float* const* values;       /* [n_levels][nnz]                                                */
  int32_t n_blocks;
  const int32_t* block_len;         /* [n_blocks]                                                     */
  const int32_t* block_chans;       /* [sum(block_len)]                                               */
  int32_t device;                   /* CUDA device ordinal                                            */
} p2m_model_desc_t;

/* Parameter / gradient tables: device pointers with the reference's state_dict layout
 * (SURVEY.md §8b): cl_w[i] is [Fout, 3*Fin] with column = fin*3 + k; bn_* entries are NULL for the
 * last conv (meshnet.py:52-53).  For gradients the same struct is used with d(.) pointers; bn_rm,
 * bn_rv, bn_nbt are ignored there.                                                                 */
typedef struct {
  float* fc_w;                 /* [V1*C1, J*C0]            */
  float* fc_b;                 /* [V1*C1]                  */
  float* const* cl_w;          /* [n_layers]               */
  float* const* cl_b;          /* [n_layers]               */
  float* const* bn_w;          /* [n_layers] gamma         */
  float* const* bn_b;          /* [n_layers] beta          */
  float* const* bn_rm;         /* [n_layers] running_mean  */
  float* const* bn_rv;         /* [n_layers] running_var   */
  int64_t* const* bn_nbt;      /* [n_layers] num_batches_tracked (may be NULL) */
} p2m_params_t;

int p2m_model_create(const p2m_model_desc_t* desc, p2m_model_t** out);
void p2m_model_destroy(p2m_model_t* m);
int p2m_model_num_layers(const p2m_model_t* m);
/* layer geometry: out[0]=level index, [1]=V, [2]=Fin, [3]=Fout, [4]=has_bn, [5]=relu */
int p2m_model_layer_info(const p2m_model_t* m, int layer, int32_t out[6]);
/* precision: a P2M_PREC_* value: fp32, fp16x3 (the default), fp16 (inference only) or fp16_mixed (training too) */
int p2m_model_set_precision(p2m_model_t* m, int precision);
/* Profiling: when enabled, the eval forward records a CUDA event pair (on the caller's stream) around
 * every conv layer; p2m_model_layer_times_ms returns the last forward's per-layer device times.      */
int p2m_model_set_profiling(p2m_model_t* m, int enable);
int p2m_model_layer_times_ms(p2m_model_t* m, float* out_ms, int n);
/* Every mbarrier wait of the tensor-core kernels is time-bounded (2 s).  A kernel whose wait expired records the
 * wait's id in a per-handle status word the host can read without a copy; the NEXT entry point called on
 * the handle (and p2m_meshnet_forward_host itself, after its stream synchronisation) then fails with
 * P2M_ERR_CUDA and clears the word — results of a timed-out kernel are never returned silently.
 * p2m_debug_kernel_status device-synchronises and returns the word without clearing it (0 = clean).  */
int p2m_debug_kernel_status(p2m_model_t* m, int32_t* out);
/* Debug (libraries built with -DP2M_UMMA_TRACE only; P2M_ERR_INVALID otherwise): CTA 0 of this handle's
 * tensor-core conv kernels logs (event << 48 | SM clock) into dev_buf [8][512] int64; NULL = off.        */
int p2m_debug_set_trace(p2m_model_t* m, void* dev_buf);
/* Debug / ablation: 1 (default) = in eval mode the 128->64 conv's epilogue produces the 64->3 head's projections
 * itself (the 64-wide activation is never written); 0 = the two layers run separately.                         */
int p2m_debug_set_fuse_head(p2m_model_t* m, int enable);
/* Padding-vertex elision: the isolated padding vertices of each level (the fake nodes of the reference's binary-tree
 * reorder, lib/coarsening.py:214-258) go through a plain GEMM with the combined weights W0 + c W1 + (2c^2-1) W2, the
 * connected rows through the conv on index-list tiles.  Same results up to fp32 association.  1 (default) = on levels
 * where at least 40 % of the rows are isolated, 2 = wherever the tile families exist, 0 = off.                       */
int p2m_debug_set_elide_padding(p2m_model_t* m, int enable);
/* Eval mode, on the elided levels: both children of a fake vertex are fake and carry identical values, so only one
 * representative per class of identical isolated rows is computed and the output rows of the others are filled from
 * it at the end; p2m_meshnet_forward_vertices (which returns connected rows only) computes no isolated row at all.
 * 1 (default) = on, 0 = every isolated row is computed.  Training always computes every row (BatchNorm statistics). */
int p2m_debug_set_dedup_padding(p2m_model_t* m, int enable);
/* Debug: which kernels the single-layer entry points (p2m_cheb_conv_fwd / _bwd) select for one layer of `level` at
 * the handle's current precision.  out[0] = forward conv on tensor cores, out[1] its X staging depth (1 or 2; 0 off
 * the tensor cores), out[2] / out[3] = the same for the weight gradient, out[4] / out[5] = the backward-data GEMM
 * (dT = dz W_k), out[6] = own rows arrive by TMA (V % 128 == 0), out[7] = the level's largest staged-row count (own
 * rows + 1-hop halo) per 128-row tile (0 when the level has no tensor-core metadata), out[8] = isolated rows that
 * padding elision would route to the dense path (0: elision not applicable).                                    */
int p2m_debug_conv_path(const p2m_model_t* m, int level, int fin, int fout, int32_t out[9]);
/* Debug: how the tensor-core forward conv of that layer (T1 given, the level's consecutive tiles) is laid out.  out[0] =
 * output columns per CTA: 64 (128 x 64 tiles), 128 (64 x 128; a 256-wide layer as two column slices) or 256 (64 x 256,
 * both MMA warpgroups on one tile: Fin = Fout = 256), out[1] = A/B ring slots, out[2] = T1 stages; all 0 off the
 * tensor cores.                                                                                                    */
int p2m_debug_conv_tiling(const p2m_model_t* m, int level, int fin, int fout, int32_t out[3]);
/* Debug: the level's tile families and what a tensor-core conv fin -> fout would launch on each (host only, no device
 * work).  out[f][k][15] for family f = consecutive tiles, padding elision's connected-row tiles (real_tiles), its
 * isolated-row tiles (iso_tiles), its eval-mode class representatives (rep_tiles), and tile size k = 128 rows, 64
 * rows: [0] tiles (0: the family does not exist), [1] largest staged-row count (own rows + 1-hop halo), [2] metadata
 * blob stride in bytes; then (output columns per CTA, A/B ring slots, X / T1 stages) for the T1-given conv at fp16x3
 * [3..5], the plain GEMM at fp16x3 [6..8], the T1-given conv at fp16 [9..11], the plain GEMM at fp16 [12..14], all 0
 * where it does not fit shared memory or on the tile size a conv to fout does not run on (fout 64: 128-row tiles,
 * 128 and 256: 64-row tiles).  fin a multiple of 32 in [32, 256], fout 64, 128 or 256.                            */
int p2m_debug_tile_families(const p2m_model_t* m, int level, int fin, int fout, int32_t out[120]);
/* Debug: size this handle's persistent tensor-core grids (conv, dW, the fc's dense GEMM) for n SMs instead of the
 * device's count, as on a part with fewer SMs: a CTA walks ceil(n_tiles / grid.x) tiles.  No route reads the count, so
 * the same kernels run; only which CTA (and warpgroup) takes each tile changes.  0 <= n <= the device's count;
 * 0 restores it.                                                                                                    */
int p2m_debug_set_sm_count(p2m_model_t* m, int n);
/* Debug: the paths the network schedules (p2m_meshnet_forward / _backward) take for layer `layer` at batch `batch`,
 * from the same route decision the schedules make.  need_dx only matters for layer 0 (the network input's gradient).
 * out[0] = forward conv on tensor cores, out[1] = its padding-vertex elision, out[2] = backward by the thin head's
 * weights-first kernel, out[3] = dW on tensor cores from the basis of x, out[4] = ... from the basis of dz,
 * out[5] = dX as a tensor-core conv on dz, out[6] = its padding-vertex elision, out[7] = dX by the three tensor-core
 * dT GEMMs, out[8] = in eval mode this layer's epilogue computes the next (64 -> 3 head) layer's projections.      */
int p2m_debug_layer_route(const p2m_model_t* m, int layer, int batch, int need_dx, int32_t out[9]);

/* Debug capture of the network schedules' intermediate tensors.  Every pointer is device memory and nullable (a null
 * array, or a null entry of one, is not written); the arrays hold one entry per layer (p2m_model_num_layers).  While
 * a capture is set, the schedules copy into it on their stream (cudaMemcpyAsync), so the values are those of the
 * latest call once the stream reaches that point.  Row-major [B * V_layer, F] like every activation.
 *   training forward:  z[l] = conv output in front of the BatchNorm, a[l] = the layer's output (BatchNorm, ReLU,
 *                      residual; layers without BatchNorm: nothing), fc_out = the fc's output [B, fc_out];
 *   eval forward:      y[l] = the layer's output as written (not written for a layer whose output the fused head
 *                      replaced by its projections), fc_out;
 *   backward:          g_a[l] = gradient entering the layer's output, g_z[l] = gradient of the conv output (after
 *                      the BatchNorm backward), dx[l] = gradient of the layer's input (after the unpool pair-sum and the
 *                      residual; layer 0: only when the caller asks for dx), fc_dx = gradient of the fc's input.
 * p2m_debug_set_capture copies the struct and the arrays; NULL clears the capture.  Without one the schedules issue
 * exactly the launches they issue without this facility.                                                         */
typedef struct {
  float* const* z;
  float* const* a;
  float* const* y;
  float* fc_out;
  float* const* g_a;
  float* const* g_z;
  float* const* dx;
  float* fc_dx;
} p2m_capture_t;
int p2m_debug_set_capture(p2m_model_t* m, const p2m_capture_t* capture);

/* ---- per-BatchNorm options -------------------------------------------------------------------------
 * One record per BatchNorm, the state torch's _BatchNorm.forward reads (torch/nn/modules/batchnorm.py):
 *   stats  P2M_BN_BATCH_UPDATE: batch statistics, running statistics updated and num_batches_tracked += 1 (bn.training
 *            with track_running_stats);
 *          P2M_BN_BATCH: batch statistics, nothing updated (bn.training without track_running_stats, or an eval-mode
 *            BatchNorm whose running buffers are None); the running-statistic pointers may be NULL;
 *          P2M_BN_RUNNING: running statistics (eval-mode BatchNorm, also inside a train-mode model: frozen statistics).
 *   cumulative  momentum None: the update factor is 1 / num_batches_tracked after its increment, read on the device
 *            (the call never synchronises); needs num_batches_tracked.
 *   momentum  the update factor otherwise (used as a float);  eps  added to the variance (the biased one of the batch,
 *            or the running one).
 * Batch statistics normalise with the biased variance and update the running variance with the unbiased one (n = the
 * rows the BatchNorm sees: B * V for MeshNet, B for PoseNet).  A NULL option array means today's defaults: momentum 0.1,
 * eps 1e-5, and P2M_BN_BATCH_UPDATE in training / P2M_BN_RUNNING in eval; those give bitwise the results of the entry
 * points without options, which are calls with NULL.                                                      */
#define P2M_BN_BATCH_UPDATE 0
#define P2M_BN_BATCH 1
#define P2M_BN_RUNNING 2
typedef struct {
  int32_t stats;       /* P2M_BN_BATCH_UPDATE | P2M_BN_BATCH | P2M_BN_RUNNING */
  int32_t cumulative;  /* 1: momentum None (cumulative moving average) */
  double momentum;
  double eps;
} p2m_bn_opts_t;

/* Bytes of device workspace p2m_meshnet_forward needs for batch B.  In training mode the workspace
 * also carries what p2m_meshnet_backward reads, so it must stay alive and untouched in between.   */
size_t p2m_meshnet_workspace_bytes(const p2m_model_t* m, int batch, int training);
size_t p2m_meshnet_backward_scratch_bytes(const p2m_model_t* m, int batch);

/* Pose2Mesh.forward (meshnet.py:80-117): x [B, J, Cin] -> y [B, V0, Cout].
 * training=0: BatchNorm uses running stats (folded into the conv epilogue).
 * training=1: batch statistics, running stats updated (momentum 0.1, eps 1e-5), activations kept. */
int p2m_meshnet_forward(p2m_model_t* m, const p2m_params_t* params, const float* x, float* y, int batch,
                        int training, void* workspace, size_t workspace_bytes, p2m_stream_t stream);

/* Fused output gather (SURVEY.md §8a row a9): the callers' `pred[:, perm_reverse[:n_real], :]`
 * (lib/core/base.py:130,201; demo/run.py:170) folded into the head layer's store.  `vertex_of_slot` (HOST,
 * int32[n_slots]) is perm_reverse[:n_real]; p2m_meshnet_forward_vertices then writes y_vertices [B, n_slots, Cout]
 * (eval mode) instead of the padded [B, V0, Cout].                                                    */
int p2m_model_set_output_gather(p2m_model_t* m, const int32_t* vertex_of_slot, int n_slots);
int p2m_meshnet_forward_vertices(p2m_model_t* m, const p2m_params_t* params, const float* x, float* y_vertices,
                                 int batch, void* workspace, size_t workspace_bytes, p2m_stream_t stream);

/* Backward of the training forward above.  dy [B,V0,Cout]; dx [B,J,Cin] (may be NULL).  Gradients
 * are WRITTEN (not accumulated) into `grads`.                                                     */
int p2m_meshnet_backward(p2m_model_t* m, const p2m_params_t* params, const p2m_params_t* grads, const float* x,
                         const float* dy, float* dx, int batch, void* workspace, size_t workspace_bytes,
                         void* scratch, size_t scratch_bytes, p2m_stream_t stream);

/* The same three with one p2m_bn_opts_t per layer (`bn` [n_layers], host memory; the last layer's entry, which has no
 * BatchNorm, is ignored; NULL: the defaults above).  The eval schedule (BatchNorm folded into the conv epilogues,
 * padding elision and dedup, fused head) runs when training == 0 and every BatchNorm uses P2M_BN_RUNNING, with each
 * layer's eps.  Otherwise the training schedule runs with per-layer statistics (with training == 0, e.g. an eval-mode
 * BatchNorm without running buffers, it is not followed by a backward).  A layer with P2M_BN_RUNNING in the training schedule is a frozen BatchNorm: its
 * backward has no batch-mean terms and the conv bias in front of it gets sum_rows g_z, where a batch-statistics layer
 * writes exactly 0.  The workspace size depends on the options; the backward takes the options of the forward that
 * wrote the workspace.                                                                                    */
size_t p2m_meshnet_workspace_bytes_opts(const p2m_model_t* m, int batch, int training, const p2m_bn_opts_t* bn);
int p2m_meshnet_forward_opts(p2m_model_t* m, const p2m_params_t* params, const p2m_bn_opts_t* bn, const float* x,
                             float* y, int batch, int training, void* workspace, size_t workspace_bytes,
                             p2m_stream_t stream);
int p2m_meshnet_backward_opts(p2m_model_t* m, const p2m_params_t* params, const p2m_params_t* grads,
                              const p2m_bn_opts_t* bn, const float* x, const float* dy, float* dx, int batch,
                              void* workspace, size_t workspace_bytes, void* scratch, size_t scratch_bytes,
                              p2m_stream_t stream);

/* End-to-end inference with HOST buffers (pageable or pinned): H2D of x, forward (eval), D2H of y,
 * stream-synchronised on return.  `workspace` must additionally hold x and y
 * (p2m_meshnet_workspace_bytes(...) + p2m_meshnet_host_io_bytes(...)).                             */
size_t p2m_meshnet_host_io_bytes(const p2m_model_t* m, int batch);
int p2m_meshnet_forward_host(p2m_model_t* m, const p2m_params_t* params, const float* x_host, float* y_host,
                             int batch, void* workspace, size_t workspace_bytes, p2m_stream_t stream);
/* Same with the fused output gather (p2m_model_set_output_gather): y_vertices_host is [B, n_slots, Cout], i.e. what
 * the reference's callers keep of a mesh (lib/core/base.py:130,201; demo/run.py:170) — 6890 of the 12288 rows.   */
int p2m_meshnet_forward_vertices_host(p2m_model_t* m, const p2m_params_t* params, const float* x_host,
                                      float* y_vertices_host, int batch, void* workspace, size_t workspace_bytes,
                                      p2m_stream_t stream);

/* ---- single Chebyshev graph convolution ----------------------------------------------------------
 * graph_conv_cheby (cheby_graph_conv.py:5-42) on hierarchy level `level`:
 *   y = act( bn( [T0|T1|T2] W^T + b ) ),  T0=x, T1=L~x, T2=2L~T1-x,   x [B,V,Fin] -> y [B,V,Fout]
 * bn_mode 0: none; 1: eval affine from running stats; 2: batch statistics (running stats updated,
 *            save_mean/save_invstd [Fout] written if non-NULL).                                    */
typedef struct {
  int32_t level, batch, fin, fout;
  const float* x;
  const float* weight;      /* [Fout, 3*Fin], column = fin*3 + k */
  const float* bias;        /* [Fout]                            */
  int32_t bn_mode;
  const float* bn_weight;
  const float* bn_bias;
  float* bn_running_mean;
  float* bn_running_var;
  int64_t* bn_num_batches_tracked;
  float* save_mean;
  float* save_invstd;
  int32_t relu;
  float* y;
} p2m_conv_fwd_args_t;

size_t p2m_cheb_conv_workspace_bytes(const p2m_model_t* m, int level, int batch, int fin, int fout);
int p2m_cheb_conv_fwd(p2m_model_t* m, const p2m_conv_fwd_args_t* a, void* workspace, size_t workspace_bytes,
                      p2m_stream_t stream);

/* Backward of the linear part  z = [T0|T1|T2] W^T + b  (BatchNorm / ReLU backward are the caller's):
 * dz [B,V,Fout] -> dx [B,V,Fin] (may be NULL), dweight [Fout,3Fin], dbias [Fout].                  */
typedef struct {
  int32_t level, batch, fin, fout;
  const float* x;
  const float* weight;
  const float* dz;
  float* dx;
  float* dweight;
  float* dbias;
} p2m_conv_bwd_args_t;
int p2m_cheb_conv_bwd(p2m_model_t* m, const p2m_conv_bwd_args_t* a, void* workspace, size_t workspace_bytes,
                      p2m_stream_t stream);

/* ==== stateless entry points: from here to the body model, no function takes a handle ==================
 * A call's data arrays (the device pointers of its signature: inputs, outputs, optional arrays and workspace) must be
 * device memory of one device; NULL optional arrays are skipped.  Host-side tables (subsets, offsets, thresholds,
 * learning-rate schedules, the PoseNet parameter struct) stay in host memory and are not data arrays.  The call runs on
 * the data arrays' device, enqueued on `stream`, and restores the caller's current device.  A host pointer or arrays
 * on two devices give P2M_ERR_INVALID before any device work.                                              */

/* ---- the step in front of MeshNet (SURVEY.md §8 row f1) --------------------------------------------
 * FlatPose2Mesh.forward (lib/models/pose2mesh_net.py:16-22) in eval mode: PoseNet, the 2-D -> 3-D pose lifter
 * (lib/models/posenet.py:41-87: Linear(2J,H), `num_stage` residual stages of BN-ReLU-Linear(H,H)-BN-ReLU-Linear(H,H),
 * Linear(H,3J); running-stat BatchNorm, dropout off), and pose_combine = cat(pose2d, pose3d / 1000) [B, J, 5],
 * MeshNet's input.  All pointers are device pointers with the reference's state_dict shapes.               */
typedef struct {
  const float* w1_w; const float* w1_b;                                     /* [H, H], [H]   */
  const float* w2_w; const float* w2_b;
  const float* bn1_w; const float* bn1_b; const float* bn1_rm; const float* bn1_rv;   /* [H] each */
  const float* bn2_w; const float* bn2_b; const float* bn2_rm; const float* bn2_rv;
} p2m_posenet_stage_t;
typedef struct {
  int32_t num_joint, hidden, num_stage;
  const float* w1_w; const float* w1_b;        /* [H, 2J], [H]  */
  const float* w2_w; const float* w2_b;        /* [3J, H], [3J] */
  const p2m_posenet_stage_t* stages;           /* [num_stage] (host array of device pointers) */
} p2m_posenet_params_t;
size_t p2m_posenet_workspace_bytes(int batch, int hidden);
/* pose2d [B, 2J] -> pose3d [B, 3J]; pose_combine (optional) [B, J, 5]. */
int p2m_posenet_forward(const p2m_posenet_params_t* params, const float* pose2d, float* pose3d, float* pose_combine,
                        int batch, void* workspace, size_t workspace_bytes, p2m_stream_t stream);

/* ---- PoseNet in training mode: forward with batch statistics and dropout, and its backward ------------
 * The reference's train-mode op sequence (lib/models/posenet.py:25-38,77-87), fp32 storage:
 *   y = x W1^T + b1;  per stage  y += Wb drop(relu(bn2(Wa drop(relu(bn1(y))) + ba))) + bb;  pose3d = y W2^T + b2.
 * BatchNorm: biased batch variance in the normalisation, unbiased in the running update, momentum 0.1, eps 1e-5;
 * running_mean / running_var (the const pointers of p2m_posenet_stage_t) are updated in place and
 * num_batches_tracked += 1 on the device.  The H x H layers run on the tensor cores (fp16x3, as in eval) when
 * H % 64 == 0, in the forward, dX and dW GEMMs alike, and on the fp32 CUDA-core GEMM otherwise.  Every gradient operand
 * of a tensor-core GEMM is scaled into fp16's range by a power of two found on the device and the scale is divided out
 * of the result, so gradients of any magnitude keep fp32's relative accuracy; the activation operand of dW is packed
 * times 2^6 like the weights and must stay below 2^10 in magnitude (a train-mode BatchNorm output is at most
 * (sqrt(B - 1) |gamma| + |beta|) / (1 - p)).
 *
 * Dropout rule.  The mask is never stored: both calls derive it from `seed` (two int64 in DEVICE memory, read by the
 * kernels, so the calls never synchronise and a captured graph can be replayed with fresh seeds).  Element i (flat
 * index into [B, H]) of dropout layer d = 2 stage + {0 after bn1, 1 after bn2} is KEPT iff word (i & 3) of
 *   Philox4x32-10(key = (low 32 bits of seed[0], high 32 bits of seed[0]),
 *                 counter = (low 32 bits of i >> 2, high 32 bits of i >> 2, d, low 32 bits of seed[1]))
 * is < min(floor((1 - p) 2^32), 2^32 - 1), (1 - p) evaluated in double from the float p; a kept value is multiplied by the float
 * 1 / (1 - p).  p == 0: no dropout (no random numbers are drawn); p == 1: everything is zeroed.
 *
 * `saved` (p2m_posenet_train_saved_bytes; written by the forward, read by the backward) holds, each array starting
 * at a multiple of 256 bytes: y_0 .. y_S [B, H] each (S = num_stage; y_s is the input of stage s, y_S of the output
 * layer), then z2_0 .. z2_{S-1} [B, H] (the pre-bn2 output of each stage's first Linear), then per stage and per
 * BatchNorm (bn1, bn2) the vectors mean | invstd | scale | shift [H] each.  The dropped activations are recomputed in
 * the backward.  One workspace size serves both calls.  Gradients are written, not accumulated.  batch >= 2
 * (a batch of one has no batch statistics: P2M_ERR_INVALID).                                              */
typedef struct {
  int64_t* bn1_nbt; int64_t* bn2_nbt;          /* num_batches_tracked of the stage's BatchNorms (device, may be NULL) */
} p2m_posenet_train_stage_t;
typedef struct {
  const p2m_posenet_train_stage_t* stages;     /* [num_stage] (host array of device pointers) */
} p2m_posenet_train_t;
typedef struct {
  float* w1_w; float* w1_b; float* w2_w; float* w2_b;
  float* bn1_w; float* bn1_b; float* bn2_w; float* bn2_b;
} p2m_posenet_stage_grads_t;
typedef struct {
  float* w1_w; float* w1_b; float* w2_w; float* w2_b;     /* shapes of the parameters */
  const p2m_posenet_stage_grads_t* stages;                /* [num_stage] (host array of device pointers) */
} p2m_posenet_grads_t;
size_t p2m_posenet_train_workspace_bytes(int batch, int num_joint, int hidden, int num_stage);
size_t p2m_posenet_train_saved_bytes(int batch, int num_joint, int hidden, int num_stage);
/* pose2d [B, 2J] -> pose3d [B, 3J]; pose_combine (optional) [B, J, 5] as in p2m_posenet_forward. */
int p2m_posenet_train_forward(const p2m_posenet_params_t* params, const p2m_posenet_train_t* extra, const float* pose2d,
                              int batch, float p_dropout, const int64_t* seed, float* pose3d, float* pose_combine,
                              void* saved, size_t saved_bytes, void* workspace, size_t workspace_bytes,
                              p2m_stream_t stream);
/* d_pose3d [B, 3J] -> grads (every pointer required) and, optionally, d_pose2d [B, 2J]; params, pose2d, p_dropout,
 * seed and saved as in the forward that wrote `saved`. */
int p2m_posenet_backward(const p2m_posenet_params_t* params, const float* pose2d, int batch, float p_dropout,
                         const int64_t* seed, const void* saved, size_t saved_bytes, const float* d_pose3d,
                         const p2m_posenet_grads_t* grads, float* d_pose2d, void* workspace, size_t workspace_bytes,
                         p2m_stream_t stream);

/* The PoseNet entry points with options: `bn` [2 num_stage] (host; stage s's bn1 at 2 s, bn2 at 2 s + 1; NULL: the
 * defaults, P2M_BN_RUNNING for the eval forward, P2M_BN_BATCH_UPDATE for the training calls), `p_dropout` [num_stage]
 * (host; the p of stage s's Dropout, 0 when it is in eval mode; NULL: no dropout).  The dropout rule above holds with
 * each stage's own p, so p_dropout[s] == the scalar p of the calls without options gives their masks bitwise.  The eval
 * forward needs P2M_BN_RUNNING everywhere and reads each eps.  In the training calls a P2M_BN_RUNNING BatchNorm is
 * frozen: scale / shift from its running statistics, backward without the batch-mean terms; batch >= 2 is required
 * only when some BatchNorm uses batch statistics.  The running-statistic pointers of a P2M_BN_BATCH BatchNorm may be
 * NULL.  The workspace and saved sizes do not depend on the options.  The backward takes the options and p_dropout of
 * the forward that wrote `saved`. */
int p2m_posenet_forward_opts(const p2m_posenet_params_t* params, const p2m_bn_opts_t* bn, const float* pose2d,
                             float* pose3d, float* pose_combine, int batch, void* workspace, size_t workspace_bytes,
                             p2m_stream_t stream);
int p2m_posenet_train_forward_opts(const p2m_posenet_params_t* params, const p2m_posenet_train_t* extra,
                                   const p2m_bn_opts_t* bn, const float* p_dropout, const float* pose2d, int batch,
                                   const int64_t* seed, float* pose3d, float* pose_combine, void* saved,
                                   size_t saved_bytes, void* workspace, size_t workspace_bytes, p2m_stream_t stream);
int p2m_posenet_backward_opts(const p2m_posenet_params_t* params, const p2m_bn_opts_t* bn, const float* p_dropout,
                              const float* pose2d, int batch, const int64_t* seed, const void* saved,
                              size_t saved_bytes, const float* d_pose3d, const p2m_posenet_grads_t* grads,
                              float* d_pose2d, void* workspace, size_t workspace_bytes, p2m_stream_t stream);

/* Debug capture of the PoseNet backward's intermediates, which live only in the workspace (the forward's are in
 * `saved`).  Every pointer is device memory and nullable; the per-stage fields are host arrays [num_stage] of device
 * pointers (a null array, or a null entry, is not written).  [B, H] row-major unless stated.  For stage s:
 *   g_y[s]    dL/dy_{s+1}, the gradient entering the stage's backward;
 *   a2[s]     the recomputed drop(relu(bn2(z2_s)));
 *   g_a2[s]   g_y[s] Wb, the gradient of a2 (before the dropout backward);
 *   g_z2[s]   dL/dz2_s after the dropout, ReLU and bn2 backward;
 *   a1[s], g_a1[s]  the same as a2, g_a2 for drop(relu(bn1(y_s))) and g_z2[s] Wa;
 *   g_bn1[s]  the gradient of y_s through bn1 alone (g_y[s - 1] = g_y[s] + g_bn1[s]);
 *   scale[s]  float[4]: the power-of-two range normalisations of the stage's tensor-core GEMM operands a2, g_y[s], a1,
 *             g_z2[s] (not written on the fp32 path);
 *   g_y0      dL/dy_0, the gradient entering the input layer's backward.
 * p2m_debug_posenet_backward_capture is p2m_posenet_backward_opts plus the copies (cudaMemcpyAsync on `stream`); the
 * results are bitwise those of p2m_posenet_backward_opts.                                                    */
typedef struct {
  float* const* g_y;
  float* const* a2;
  float* const* g_a2;
  float* const* g_z2;
  float* const* a1;
  float* const* g_a1;
  float* const* g_bn1;
  float* const* scale;
  float* g_y0;
} p2m_posenet_capture_t;
int p2m_debug_posenet_backward_capture(const p2m_posenet_params_t* params, const p2m_bn_opts_t* bn,
                                       const float* p_dropout, const float* pose2d, int batch, const int64_t* seed,
                                       const void* saved, size_t saved_bytes, const float* d_pose3d,
                                       const p2m_posenet_grads_t* grads, float* d_pose2d, void* workspace,
                                       size_t workspace_bytes, const p2m_posenet_capture_t* capture,
                                       p2m_stream_t stream);

/* ---- the steps either side of the model in the reference's callers (SURVEY.md §8 row f2) ----------
 * Joint regression (lib/core/base.py:131,204; demo/run.py:171): joints [B, n_joint, C] = joint_regressor
 * [n_joint, n_vertex] @ vertices [B, n_vertex, C] (C <= 4), on the gathered vertices of
 * p2m_meshnet_forward_vertices.                                                                        */
int p2m_regress_joints(const float* joint_regressor, const float* vertices, float* joints, int batch, int n_joint,
                       int n_vertex, int chans, p2m_stream_t stream);
/* Its backward: d_vertices [B, n_vertex, C] = joint_regressor^T @ d_joints [B, n_joint, C] (written, not accumulated;
 * one thread per (mesh, vertex) walks the joints in order: no atomics, bitwise reproducible). */
int p2m_regress_joints_backward(const float* joint_regressor, const float* d_joints, float* d_vertices, int batch,
                                int n_joint, int n_vertex, int chans, p2m_stream_t stream);
/* The demo's input normalisation (demo/run.py:150-158): joints_px [B, J, 2] in image pixels -> pose2d [B, J, 2],
 * zero mean / unit std per pose and coordinate in the aspect-preserving box of the (input_h, input_w) network input
 * (cfg.MODEL.input_shape = (384, 288)).  truncate_like_int_input = 1 reproduces the reference on INTEGER joint
 * arrays (demo/h36m_joint_input.npy is int64: the transformed coordinates are truncated when written back). */
int p2m_normalize_pose2d(const float* joints_px, float* pose2d, int batch, int n_joint, int input_h, int input_w,
                         int truncate_like_int_input, p2m_stream_t stream);

/* ---- the mesh losses (SURVEY.md §8 row f3; lib/core/loss.py:10-23,62-114) ---------------------------
 * One pass over (mesh, face): sums[0] = sum of the NormalVectorLoss terms, sums[1] = sum of the EdgeLengthLoss terms
 * over (B, 3 n_face) (fp64, device; the losses are sums / (3 B n_face)).  If grad_out [B, n_vertex, 3] is given it
 * receives  grad_scale[0] * d sums[0] / d coord_out + grad_scale[1] * d sums[1] / d coord_out  (grad_scale: device
 * float[2], i.e. upstream gradient / (3 B n_face)).  faces: device int32 [n_face, 3].                    */
int p2m_mesh_losses(const float* coord_out, const float* coord_gt, const int32_t* faces, int batch, int n_vertex,
                    int n_face, const float* grad_scale, double* sums, float* grad_out, p2m_stream_t stream);
/* CoordLoss: *sum = sum |pred * valid - target * valid| over n elements (valid may be NULL = ones, else same shape);
 * grad_out (optional, n floats) = grad_scale[0] * sign(.) * valid.                                        */
int p2m_coord_loss(const float* pred, const float* target, const float* valid, int64_t n, const float* grad_scale,
                   double* sum, float* grad_out, p2m_stream_t stream);

/* ---- the Trainer's objective (lib/core/base.py:129-143) ---------------------------------------------------
 * With x = cam_mesh[:, perm_reverse[:n_vertex]] (the real rows of the padded output) and pred_pose = J (1000 x):
 *   loss1 = mean |x m - gt_mesh m|                               m = mesh_valid [B, n_vertex] (per vertex)
 *   loss2 = w_normal NormalVectorLoss(x, gt_mesh)
 *   loss3 = w_edge EdgeLengthLoss(x, gt_mesh) if *edge != 0, else 0
 *   loss4 = w_joint mean |pred_pose m - gt_reg3dpose m|         m = reg3dpose_valid [B, n_reg_joint]
 *   loss5 = w_joint mean |lift_pose m - gt_lift3dpose m|        m = lift3dpose_valid [B, n_lift_joint]
 *   loss  = loss1 + loss2 + loss3 + loss4 + loss5
 * Every pointer is device memory of one device.  weights (normal, edge, joint) and the edge flag are read on the
 * device, so a captured graph picks up a flag written between replays; the backward must see the values of the
 * forward it differentiates.  scratch holds at least 32 (batch + 1) bytes; its contents on entry do not matter.
 * Reductions: loss1, loss4 and loss5 are per-mesh partials summed in fixed order (bitwise reproducible); loss2 and
 * loss3 are p2m_mesh_losses' sums (fp64 atomics across CTAs), and its gradient is accumulated with fp32 atomics.
 * batch <= 65535, n_reg_joint <= P2M_POSE2MESH_MAX_REG_JOINT, perm_reverse holds distinct rows in [0, n_padded). */
#define P2M_POSE2MESH_MAX_REG_JOINT 24
typedef struct {
  int32_t batch, n_padded, n_vertex, n_face, n_reg_joint, n_lift_joint;
  const float* cam_mesh;          /* [B, n_padded, 3]      the model's output            */
  const float* lift_pose;         /* [B, n_lift_joint, 3]  PoseNet's output, mm          */
  const float* gt_mesh;           /* [B, n_vertex, 3]                                    */
  const float* gt_reg3dpose;      /* [B, n_reg_joint, 3]                                 */
  const float* gt_lift3dpose;     /* [B, n_lift_joint, 3]                                */
  const float* mesh_valid;        /* [B, n_vertex]                                       */
  const float* reg3dpose_valid;   /* [B, n_reg_joint]                                    */
  const float* lift3dpose_valid;  /* [B, n_lift_joint]                                   */
  const int32_t* faces;           /* [n_face, 3] into 0 .. n_vertex - 1                  */
  const float* joint_regressor;   /* [n_reg_joint, n_vertex]                             */
  const int32_t* perm_reverse;    /* [n_vertex]: padded row of vertex v                  */
  const float* weights;           /* [3]: normal, edge, joint weight                     */
  const float* edge;              /* [1]: nonzero adds the edge term                     */
  float* pred_pose;               /* [B, n_reg_joint, 3]: written by the forward, read by the backward */
  void* scratch;
  float* loss;                    /* [1]  forward output                                 */
  float* terms;                   /* [5]  forward output: loss1 .. loss5                 */
  const float* grad_loss;         /* [1]  backward input: d objective / d loss           */
  float* d_cam_mesh;              /* [B, n_padded, 3] backward output, padding rows 0    */
  float* d_lift_pose;             /* [B, n_lift_joint, 3] backward output                */
} p2m_pose2mesh_loss_args_t;
/* Forward: loss, terms and pred_pose (one vertex / joint launch and the face kernel of p2m_mesh_losses). */
int p2m_pose2mesh_loss(const p2m_pose2mesh_loss_args_t* a, p2m_stream_t stream);
/* Backward: d_cam_mesh (zeroed, then the face kernel reading and accumulating through perm_reverse, then one thread per
 * (mesh, vertex) adding the vertex and joint terms) and d_lift_pose; reads pred_pose of the forward. */
int p2m_pose2mesh_loss_backward(const p2m_pose2mesh_loss_args_t* a, p2m_stream_t stream);

/* ---- evaluation metrics (SURVEY.md §8 row f5; lib/coord_utils.py:127-149, the datasets' compute_*_err) ----------
 * Both take a batch of point sets pred/A, gt/B [batch, n_point, 3] and an optional subset of point indices (HOST
 * int32 [n_subset], checked here: every index in [0, n_point); NULL with n_subset = 0 = all points; k = the number of
 * points used).  Outputs are nullable, but at least one must be given.  sums (double [batch + 1]) receives the
 * per-sample sums of the errors and, last, their total (fp64, fixed summation order: a sample's values do not depend
 * on its batch position).  batch and n_point are at most 2^24.
 *
 * Similarity Procrustes of A[b, subset] onto B[b, subset] (rigid_transform_3D / rigid_align): fp64 centroids,
 * centred cross-covariance and 3x3 SVD; R = Vh^T U^T with the reference's det < 0 correction, c = sum(s) / varP,
 * t = muB - c R muA.  transform [batch, 13] = {c, R row-major, t} (double); aligned [batch, k, 3] = c R a + t;
 * err [batch, k] = |c R a + t - b|.  A sample whose A points are all equal (varP = 0) or that holds a non-finite
 * value gets NaN in every output; the other samples are unaffected.                                             */
int p2m_rigid_align(const float* A, const float* B, int batch, int n_point, const int32_t* subset, int n_subset,
                    double* transform, float* aligned, float* err, double* sums, p2m_stream_t stream);
/* Root-aligned point errors: err [batch, k] = |(pred[b, i] - pred_root[b]) - (gt[b, i] - gt_root[b])|, roots
 * [batch, 3] (both or neither; NULL = no root subtraction).  fp64 = 0: float32 arithmetic in numpy's order, the bits
 * of the reference's float32 compute_*_err; fp64 = 1: fp64 arithmetic, rounded once to float32 on store.          */
int p2m_point_errors(const float* pred, const float* gt, const float* pred_root, const float* gt_root, int batch,
                     int n_point, const int32_t* subset, int n_subset, int fp64, float* err, double* sums,
                     p2m_stream_t stream);

/* ---- demo camera fit (SURVEY.md §8 row f7; demo/run.py:149-197 optimize_cam_param, lib/models/project_net.py) --
 * One launch fits the weak-perspective camera (s, tx, ty) of every person, one warp per person:
 *   bbox [batch, 4]     process_bbox(get_bbox(joints), aspect_ratio=1.0, scale=1.25), float32
 *   target [batch, n_in_joint, 2]   j2d_processing(joints, (crop, crop), bbox, 0, 0, None)[:, :2]
 *   cam [batch, 3]      n_iter steps of Adam (betas (0.9, 0.999), eps 1e-8) on the L1 loss between
 *                       ((pred_joints3d[..., :2] + cam[1:]) cam[0]) crop/2 + crop/2 and target[:, :n_joint],
 *                       starting from init_cam [batch, 3]; step i runs at lr_values[p] for the last phase p with
 *                       lr_steps[p] <= i (lr_steps[0] == 0, increasing; at most 16 phases)
 *   loss [batch]        the L1 loss of the final camera
 *   orig_cam [batch, 4] convert_crop_cam_to_orig_img(cam, bbox, img_wh[b, 0], img_wh[b, 1]) (demo/run.py:24-43); only
 *                       when img_wh [batch, 2] (float32 pixel sizes) is given
 * joints_px is float64 [batch, n_in_joint, in_cols] (columns past the first two are ignored) holding the caller's
 * values exactly; in_kind says which dtype they came from, because the reference's arithmetic depends on it:
 * integer inputs truncate the transformed points towards zero, float32 inputs take their box in float32.  A person
 * whose box the reference rejects (process_bbox returns None) or whose joints hold a NaN gets NaN outputs; the
 * others are unaffected.  Requires 0 < n_joint <= n_in_joint <= 32, batch > 0, 0 < crop <= 2^24.  No host
 * synchronisation and no allocation (capturable in a CUDA graph).                                              */
enum p2m_cam_input {
  P2M_CAM_INPUT_F64 = 0,
  P2M_CAM_INPUT_INT = 1,
  P2M_CAM_INPUT_F32 = 2
};
int p2m_fit_camera(const double* joints_px, int in_cols, int in_kind, int n_in_joint, const float* pred_joints3d,
                   int n_joint, const float* init_cam, int batch, int crop, int n_iter, const int32_t* lr_steps,
                   const double* lr_values, int n_lr, const float* img_wh, float* cam, float* bbox, float* target,
                   float* loss, float* orig_cam, p2m_stream_t stream);
/* convert_crop_cam_to_orig_img alone: orig_cam [batch, 4] from cam [batch, 3], bbox [batch, 4], img_wh [batch, 2]. */
int p2m_crop_cam_to_orig(const float* cam, const float* bbox, const float* img_wh, int batch, float* orig_cam,
                         p2m_stream_t stream);

/* ---- temporal metrics (SURVEY.md §8 row f8; lib/smooth_utils.py:5-72, lib/coord_utils.py:194-222) ----------------
 * Ragged batches of sequences concatenated along frames: offsets (HOST int64 [n_seq + 1], checked here: offsets[0] = 0,
 * non-decreasing, offsets[n_seq] = n_frames >= 1; empty sequences allowed) are copied to the device with a
 * stream-ordered allocation.  dtype is P2M_DTYPE_F32 or P2M_DTYPE_F64 for every data array of a call.  No other host
 * allocation or synchronisation.  A sequence's results do not depend on its batch position.
 *
 * One-Euro filter (smooth_pose, OneEuroFilter): y[f, c] for x [n_frames, n_channel], per sequence along its frames,
 * in numpy's dtype and operation order (bitwise the reference's result; t = frame index, dx0 = 0).  One launch.     */
enum p2m_dtype {
  P2M_DTYPE_F32 = 0,
  P2M_DTYPE_F64 = 1
};
int p2m_one_euro_smooth(int dtype, const void* x, void* y, int64_t n_channel, const int64_t* offsets, int n_seq,
                        int64_t n_frames, double min_cutoff, double beta, double d_cutoff, p2m_stream_t stream);
/* Acceleration error (compute_error_accel) of gt, pred [n_frames, n_joint, 3], n_joint <= 32: for every window
 * (s, i), i < n_s - 2, in the order of the sequences, per_window = the joint mean of |accel_pred - accel_gt| with
 * accel = (X[i] - 2 X[i+1]) + X[i+2] (the reference's bits), valid (uint8) = vis[i] & vis[i+1] & vis[i+2] (vis: device
 * uint8 [n_frames] or NULL = all visible), and seq_mean (double [n_seq]) = the fp64 mean of the sequence's valid
 * windows, NaN when it has none.  Two launches (one when no sequence has 3 frames).                                */
int p2m_accel_error(int dtype, const void* gt, const void* pred, int n_joint, const int64_t* offsets, int n_seq,
                    int64_t n_frames, const uint8_t* vis, void* per_window, uint8_t* valid, double* seq_mean,
                    p2m_stream_t stream);
/* out[s] = the fp64 mean of values [n_rows, width] over rows offsets[s] .. offsets[s + 1) whose valid (device uint8
 * [n_rows], or NULL = all) is non-zero, in a fixed order without atomics; NaN for a segment with no such row.       */
int p2m_segment_mean(int dtype, const void* values, int64_t width, const int64_t* offsets, int n_seg, int64_t n_rows,
                     const uint8_t* valid, double* out, p2m_stream_t stream);

/* ---- FreiHAND scores (SURVEY.md §8 row f9; the FreiHAND dataset's eval.py / utils/eval_util.py) ----------------
 * All arithmetic is fp64 on the inputs' values; a distance is sqrt((dx^2 + dy^2) + dz^2), each step rounded to
 * nearest.  Thresholds are HOST double arrays, checked here (finite, >= 0, sorted ascending) and passed to the kernels
 * by value.  No host synchronisation.  Results are bitwise deterministic and do not depend on a sample's batch
 * position.
 *
 * Nearest distances between P [batch, n, 3] and Q [batch, m, 3] (dtype P2M_DTYPE_F32 or _F64 for both; n, m <= 2^20):
 * dist_p [batch, n] = min_j |P_i - Q_j|, dist_q [batch, m] = min_i |Q_j - P_i| (f64, equal to the brute force bit for
 * bit), from one sweep of the n x m pairs.  With 1 .. 16 thresholds t: counts [batch, 2, n_thr] (int64) = #(dist_p <
 * t), #(dist_q < t); frac [batch, 2, n_thr] = counts / n, / m; fscore [batch, n_thr] = ((2 a) b) / (a + b), 0 when
 * a + b = 0.  A sample holding a non-finite coordinate gets NaN distances, zero counts and NaN frac / fscore.  Every
 * output is nullable (at least one given); a missing distance output gets stream-ordered scratch.  Three launches. */
int p2m_nearest_distances(int dtype, const void* P, const void* Q, int batch, int n, int m, const double* thresholds,
                          int n_thr, double* dist_p, double* dist_q, int64_t* counts, double* frac, double* fscore,
                          p2m_stream_t stream);
/* align_w_scale(gt, pred) per sample of [batch, n_point, 3] float32: both centred and scaled by their Frobenius norm
 * (+ 1e-8), R = U V^T and s = sum(W) for U W V^T = svd(A^T P) (no reflection correction), aligned = (P R^T) s s1 + t1
 * (nullable, [batch, n_point, 3] in aligned_dtype), err [batch, n_point] f64 = |aligned - gt| (nullable).  A sample
 * holding a non-finite coordinate gets NaN.  One launch.                                                           */
int p2m_align_w_scale(const float* gt, const float* pred, int batch, int n_point, int aligned_dtype, void* aligned,
                      double* err, p2m_stream_t stream);
/* PCK histogram: hist[j] (device int64 [n_thr], accumulated, not cleared) += the number of errors e whose first
 * threshold with e <= t_j is j (NaN and e > t_last count nowhere); the count of e <= t_j is hist[0] + ... + hist[j].
 * The errors are err [n_val] (f64), or e = |pred_i - gt_i| for n_val float32 points (then optionally stored to
 * err_out [n_val] f64).  1 .. 128 thresholds.  One launch; integer atomics, so the histogram is order-free.         */
int p2m_pck_accumulate(const double* err, const float* pred, const float* gt, int64_t n_val, const double* thresholds,
                       int n_thr, double* err_out, int64_t* hist, p2m_stream_t stream);

/* ---- demo mesh overlay (SURVEY.md §8 row f10; demo/renderer.py:28-35,66-114 Renderer.render, demo/run.py:46-67) ---
 * Draws person p's mesh verts [n_person, n_vertex, 3] (faces [n_face, 3] int32) over image image_index[p] (int32
 * [n_person], NULL = all on image 0) of images_in [n_image, height, width, 3] (uint8) into images_out (same shape; may
 * equal images_in), people in order, the later person winning where two overlap.  cams [n_person, 4] is orig_cam
 * (sx, sy, tx, ty) of convert_crop_cam_to_orig_img; with the reference's Rx(180°) flip and weak-perspective matrix a
 * vertex (x, y, z) lands at column u = W/2 (1 + sx (x + tx)), row v = H/2 (1 + sy (y + ty)), depth z; fragments with z
 * outside [-1, 1] are clipped, nearer z wins and a depth tie goes to the lower face.  Coverage, depth, back-face culling,
 * clipping and compositing order follow the reference; coverage is exact (positions snapped to 1/256 px, int64 edge
 * functions, top-left fill rule).  The shading is this library's own, not pyrender's: flat Lambert of ambient 0.3 plus
 * 2.4 along the camera axis, c_k = clamp(colors[p, k] (0.3 + (2.4/pi) max(0, -n_z)), 0, 1) for the face normal n in
 * mesh coordinates, stored as floor(255 c + 0.5) into channel k.  Skipped: a triangle with a non-finite vertex or
 * camera value, a face index outside [0, n_vertex) or a vertex beyond +-2^20 px; a person whose image_index is outside
 * [0, n_image).  Optional outputs [n_image, height, width] (NULL = not written): face_map and person_map (int32, -1
 * where uncovered), depth_map (float32, NaN).  Limits: n_person, n_face <= 65535; height, width <= 16384.
 * workspace >= p2m_render_workspace_bytes (8-byte aligned).  A memset and two launches, no host synchronisation,
 * bitwise deterministic.                                                                                           */
size_t p2m_render_workspace_bytes(int n_image, int height, int width);
int p2m_render_meshes(const float* verts, int n_person, int n_vertex, const int32_t* faces, int n_face,
                      const float* cams, const float* colors, const int32_t* image_index, const uint8_t* images_in,
                      int n_image, int height, int width, uint8_t* images_out, int32_t* face_map, int32_t* person_map,
                      float* depth_map, void* workspace, size_t workspace_bytes, p2m_stream_t stream);

/* ---- body model: batched SMPL / MANO forward (SURVEY.md §8 row f6; smplpytorch SMPL_Layer.forward,
 * manopth ManoLayer.forward) --------------------------------------------------------------------------------------
 * The descriptor holds HOST arrays in the reference's buffer layouts (all float32, row-major):
 *   v_template [V, 3], shapedirs [V, 3, S], posedirs [V, 3, 9 (J - 1)], J_regressor [J, V], weights [V, J],
 *   parents [J] (parents[0] = -1, parents[i] < i), model_betas [S] (used when the betas are absent or, under
 *   P2M_BETAS_ZERO_MEANS_MODEL, when the whole batch's betas are zero), pose_mean [3 (J - 1)] added to the non-root
 *   axis-angle values (MANO's hands_mean; NULL = none), joint_map [n_out_joints] (entry e >= 0: kinematic joint e;
 *   e < 0: vertex -1 - e), scale (1 for SMPL metres, 1000 for MANO millimetres), device.
 * Create rejects non-topological parents, out-of-range map entries and non-finite buffers with P2M_ERR_INVALID.
 * J <= 64, S <= 512.  fp32 on the CUDA cores, three launches per forward, no host synchronisation. */
typedef struct p2m_body_model p2m_body_model_t;
typedef struct {
  int32_t n_vertex, n_joint, n_betas, n_out_joints;
  const float* v_template;
  const float* shapedirs;
  const float* posedirs;
  const float* J_regressor;
  const float* weights;
  const int32_t* parents;
  const float* model_betas;
  const float* pose_mean;
  const int32_t* joint_map;
  float scale;
  int32_t device;
} p2m_body_model_desc_t;
enum {
  P2M_BETAS_ZERO_MEANS_MODEL = 0, /* SMPL_Layer: an all-zero (norm 0) betas batch is replaced by model_betas */
  P2M_BETAS_AS_GIVEN = 1          /* ManoLayer: given betas are used as they are                               */
};
int p2m_body_model_create(const p2m_body_model_desc_t* desc, p2m_body_model_t** out);
void p2m_body_model_destroy(p2m_body_model_t* m);
size_t p2m_body_model_workspace_bytes(const p2m_body_model_t* m, int batch);
/* pose [batch, 3 J] axis-angle, betas [batch, S] or NULL (= model_betas), trans [batch, 3] or NULL, all device
 * float32 on the model's device.  trans is added when the batch's trans holds any non-zero (or NaN) value;
 * otherwise, with center_idx >= 0, everything is re-centred on output joint center_idx.  Then * scale.
 * verts [batch, V, 3], joints [batch, n_out_joints, 3] (device float32).  Enqueued on `stream`; decides the
 * batch-wide betas / trans tests on the device (sync-free, CUDA-graph capturable).  A sample's result is bitwise
 * independent of its batch position and of the batch size. */
int p2m_body_model_forward(const p2m_body_model_t* m, const float* pose, const float* betas, int betas_rule,
                           const float* trans, int center_idx, float* verts, float* joints, int batch,
                           void* workspace, size_t workspace_bytes, p2m_stream_t stream);
/* The vector-Jacobian product of p2m_body_model_forward with respect to pose, betas and trans: the gradient the
 * reference layer's autograd gives for the same call (same inputs, same betas_rule / center_idx).  grad_verts
 * [batch, V, 3] and grad_joints [batch, n_out_joints, 3] are the cotangents (either NULL = zero).  Writes grad_pose
 * [batch, 3 J] (the gradient of the axis-angle input; pose_mean is a constant), and, when not NULL, grad_betas
 * [batch, S] (zeros when the forward does not use the given betas: NULL betas, or an all-zero batch under
 * P2M_BETAS_ZERO_MEANS_MODEL) and grad_trans [batch, 3] (zeros when trans is not added).  With centring, the centre's
 * gradient flows back through the centre joint (or vertex).  Recomputes what it needs; no state from the forward.
 * fp32 on the CUDA cores, five launches, no atomics, no host synchronisation (CUDA-graph capturable); a sample's
 * gradient is bitwise independent of its batch position and of the batch size.  Workspace >=
 * p2m_body_model_backward_workspace_bytes (256-byte aligned). */
size_t p2m_body_model_backward_workspace_bytes(const p2m_body_model_t* m, int batch);
int p2m_body_model_backward(const p2m_body_model_t* m, const float* pose, const float* betas, int betas_rule,
                            const float* trans, int center_idx, const float* grad_verts, const float* grad_joints,
                            float* grad_pose, float* grad_betas, float* grad_trans, int batch, void* workspace,
                            size_t workspace_bytes, p2m_stream_t stream);

/* ---- dataset targets: camera-frame meshes and Human3.6M sample targets (SURVEY.md §8 row f11; the datasets'
 * get_smpl_coord / get_mano_coord and Human36M.__getitem__) -------------------------------------------------------
 * One batched call does what each dataset's get_*_coord does for one sample, as a combination of flags:
 *   ROTATE_ROOT       the root axis-angle becomes log(R exp(root)) (fp64, rounded to float32 as the reference stores
 *                     it); an exactly zero root counts as the identity (the reference raises there)
 *   CLAMP_BETAS       a sample with any |beta| > 3 gets zero betas
 *   ZERO_BETAS_MODEL  a sample whose betas are all zero (after the clamp) uses model_betas: SMPL_Layer's rule applied to
 *                     each sample on its own, as the datasets' one-sample calls do (set it for SMPL, not for MANO)
 *   LAYER_TRANS_T / LAYER_TRANS   the layer's trans is t / trans
 *   H36M_COMPENSATE   + R trans + t / 1000 - J_0 + R J_0 (J_0 the layer's root joint) after the layer
 *   ADD_T             + t after the layer
 *   TO_MM             then * 1000
 * pose [batch, 3 J], betas [batch, S], trans / t [batch, 3], R [batch, 3, 3] row-major (NULL where the flags do not
 * read them), all device float32 on the model's device.  verts [batch, V, 3]; joints [batch, n_out_joints + n_extra, 3]
 * where the extra joints are the vertices extra_vertices (HOST int32 [n_extra], n_extra <= 8; MuCo's face keypoints),
 * transformed like the mesh.  The model runs with P2M_BETAS_AS_GIVEN and no centring.  Five launches (prep, the body
 * model's three, finish), no host synchronisation (CUDA-graph capturable); a sample's result is bitwise independent of
 * its batch position and of the batch size.  Workspace >= p2m_camera_frame_workspace_bytes (256-byte aligned). */
enum {
  P2M_FRAME_ROTATE_ROOT = 1,
  P2M_FRAME_CLAMP_BETAS = 2,
  P2M_FRAME_ZERO_BETAS_MODEL = 4,
  P2M_FRAME_LAYER_TRANS_T = 8,
  P2M_FRAME_LAYER_TRANS = 16,
  P2M_FRAME_H36M_COMPENSATE = 32,
  P2M_FRAME_ADD_T = 64,
  P2M_FRAME_TO_MM = 128
};
size_t p2m_camera_frame_workspace_bytes(const p2m_body_model_t* m, int batch);
int p2m_camera_frame_coords(const p2m_body_model_t* m, int flags, const float* pose, const float* betas,
                            const float* trans, const float* R, const float* t, const int32_t* extra_vertices,
                            int n_extra, float* verts, float* joints, int batch, void* workspace,
                            size_t workspace_bytes, p2m_stream_t stream);
/* Human3.6M's two joint regressors (J_regressor_h36m_correct.npy and J_regressor_coco.npy, HOST float64 [17,
 * n_vertex] each), kept on `device` as their non-zero entries.  Create rejects non-finite values. */
typedef struct p2m_h36m_regressors p2m_h36m_regressors_t;
int p2m_h36m_regressors_create(const double* reg_h36m, const double* reg_coco, int n_vertex, int device,
                               p2m_h36m_regressors_t** out);
void p2m_h36m_regressors_destroy(p2m_h36m_regressors_t* h);
/* The targets and meta of Human36M.__getitem__ (pose2mesh_net; posenet's joint_valid is lift_pose3d_valid) with
 * augmentation off, from the camera-frame mesh mesh_cam [batch, n_vertex, 3] (mm, the H36M_COMPENSATE | TO_MM
 * output), the annotation's joint_cam [batch, 17, 3] (mm), focal f and principal point c [batch, 2].  J = 17
 * (P2M_JOINTS_HUMAN36) or 19 (P2M_JOINTS_COCO: the COCO joints with pelvis and neck).  Outputs, device float32:
 *   mesh [batch, n_vertex, 3]   (mesh_cam - joint_cam[0]) / 1000 (metres)
 *   lift_pose3d [batch, J, 3]   COCO: the regressed joints rooted at the pelvis; human36: joint_cam - joint_cam[0]
 *   reg_pose3d [batch, 17, 3]   joint_cam - joint_cam[0]
 *   joint_img [batch, J, 2]     cam2pixel of the regressed COCO joints / of joint_cam (pixels)
 *   fitting_error [batch]       get_fitting_error (mm)
 *   mesh_valid [batch, n_vertex], lift_pose3d_valid [batch, J], reg_pose3d_valid [batch, 17]: 0 where
 *   fitting_error > fitting_thr (the lift mask for COCO only), else 1.
 * Regression, projection and the error in fp64, each output rounded once.  One launch, no host synchronisation. */
enum {
  P2M_JOINTS_HUMAN36 = 0,
  P2M_JOINTS_COCO = 1,
  P2M_JOINTS_SMPL = 2,  /* SMPL's 24 joints (SURREAL): p2m_training_pose2d_augmented's crop and flip only */
  P2M_JOINTS_MANO = 3   /* MANO's 21 joints (FreiHAND): p2m_training_pose2d_augmented's crop only, no flip */
};
int p2m_h36m_targets(const p2m_h36m_regressors_t* h, int input_joint_set, float fitting_thr, const float* mesh_cam,
                     const float* joint_cam, const float* f, const float* c, int batch, float* mesh, float* lift_pose3d,
                     float* reg_pose3d, float* mesh_valid, float* lift_pose3d_valid, float* reg_pose3d_valid,
                     float* joint_img, float* fitting_error, p2m_stream_t stream);
/* The target side of one dataset's __getitem__ for a batch (pose2mesh_net and posenet), generalising
 * p2m_h36m_targets, which is its Human36M case without augmentation.  dataset:
 *   P2M_DATASET_HUMAN36M  joint_cam, f, c as p2m_h36m_targets; fitting test 25 mm (the caller's fitting_thr) against
 *                         the annotation; masks zeroed: mesh, lift (coco set only); joint_valid = lift_pose3d_valid
 *   P2M_DATASET_COCO      joint_img = (xy / 1000) s + t with s [batch, n_s] (n_s 1 or 2) and t [batch, 2]; fitting
 *                         test (3 px) in the 64 x 64 crop of process_bbox(get_bbox(the input set's joint_img), aspect
 *                         1): keypoints [batch, 17, 2] and the projected regressed COCO rows 0-16, float32 distances,
 *                         mean over keypoints_valid [batch, 17] > 0 (none: NaN, the sample stays valid); masks zeroed:
 *                         mesh, lift, reg; joint_valid follows the test
 *   P2M_DATASET_MUCO      joint_img = cam2pixel(joint, f, c); fitting test (45 mm) with the reference's quirk: the
 *                         Human3.6M-ordered joints rooted at row 14 and permuted by MuCo's names against the regressor
 *                         (DESIGN.md §4.3, sample targets); masks zeroed: mesh, lift, reg; joint_valid all ones
 *   P2M_DATASET_AMASS     joint_img = cam2pixel(joint / 1000, f, c); no fitting test (fitting_error 0, every mask 1)
 *   P2M_DATASET_PW3D      P2M_JOINTS_COCO only; joint_img = cam2pixel(joint, f, c); no fitting test (fitting_error 0,
 *                         every mask 1) and no augmentation (rot and flip must be NULL)
 * For every dataset but Human36M the Human3.6M joints are the regressed ones: the mesh is rooted at their row 0 and
 * reg_pose3d is them rooted at row 0.  mesh_cam is the camera-frame mesh (mm) of the dataset's p2m_camera_frame_coords
 * preset.  rot [batch] degrees and flip [batch] int32 (p2m_augm_params; either NULL for none) augment lift_pose3d as
 * j3d_processing does: x, y rotated by -rot degrees in fp64 and rounded once, then under a flip the joint set's flip
 * pairs swapped (those of p2m_training_pose2d_augmented) and x negated; the other outputs are never augmented.
 * joint_valid [batch, J] may be NULL.  With rot and flip NULL (or all zero), bitwise p2m_h36m_targets for Human36M.
 * One launch, no host synchronisation. */
enum {
  P2M_DATASET_HUMAN36M = 0,
  P2M_DATASET_COCO = 1,
  P2M_DATASET_MUCO = 2,
  P2M_DATASET_AMASS = 3,
  P2M_DATASET_PW3D = 4,
  P2M_DATASET_SURREAL = 5,  /* p2m_layer_joint_targets only */
  P2M_DATASET_FREIHAND = 6  /* p2m_layer_joint_targets only */
};
int p2m_sample_targets(const p2m_h36m_regressors_t* h, int dataset, int input_joint_set, float fitting_thr,
                       const float* mesh_cam, const float* joint_cam, const float* f, const float* c, const float* s,
                       int n_s, const float* t, const float* keypoints, const float* keypoints_valid, const float* rot,
                       const int32_t* flip, int batch, float* mesh, float* lift_pose3d, float* reg_pose3d,
                       float* mesh_valid, float* lift_pose3d_valid, float* reg_pose3d_valid, float* joint_valid,
                       float* joint_img, float* fitting_error, p2m_stream_t stream);
/* The targets and meta of the datasets that take the body model's own joints as both the lift and the regression
 * target, with no joint regressor: mesh_cam [batch, n_vertex, 3] and joint_cam [batch, n_joint, 3] (the layer's
 * joints) are p2m_camera_frame_coords' outputs for the dataset's preset (mm).  Root: joint 0.  dataset:
 *   P2M_DATASET_SURREAL   n_joint 24 (SMPL).  joint_img [batch, 24, 2] = cam2pixel(joint_cam, f, c) of the absolute
 *                         joints in fp64, rounded once (f, c [batch, 2]).  lift_pose3d = j3d_processing(joint_cam -
 *                         root): the float32 rooting, x, y rotated by -rot degrees in fp64 and rounded once, then under
 *                         a flip SMPL's flip pairs swapped and x negated (rot [batch] degrees, flip [batch] int32, either
 *                         NULL for none).  reg_pose3d is the same augmented array, as in the reference.
 *   P2M_DATASET_FREIHAND  n_joint 21 (MANO).  lift_pose3d = reg_pose3d = joint_cam - root in float32.  f, c, rot,
 *                         flip and joint_img must be NULL: no projection, no augmentation.
 * Both: mesh [batch, n_vertex, 3] = (mesh_cam - root) / 1000 in float32 (metres); every mask (mesh_valid [batch,
 * n_vertex], lift_pose3d_valid, reg_pose3d_valid, joint_valid [batch, n_joint], the last nullable) is 1 and
 * fitting_error [batch] is 0.  One launch, no host synchronisation. */
int p2m_layer_joint_targets(int dataset, const float* mesh_cam, const float* joint_cam, int n_vertex, int n_joint,
                            const float* f, const float* c, const float* rot, const int32_t* flip, int batch,
                            float* mesh, float* lift_pose3d, float* reg_pose3d, float* mesh_valid,
                            float* lift_pose3d_valid, float* reg_pose3d_valid, float* joint_valid, float* joint_img,
                            float* fitting_error, p2m_stream_t stream);

/* ---- dataset inputs: synthetic detector errors and the training crop (SURVEY.md §8 row f12; lib/noise_utils.py,
 * the datasets' generate_syn_error and replace_joint_img) --------------------------------------------------------
 * Random-number rule.  `seed` is two int64 in DEVICE memory, read by the kernels (no host synchronisation; a captured
 * graph replays with whatever the seed tensor holds).  Every draw is one Philox4x32-10 call with
 *   key = (low 32 bits of seed[0], high 32 bits of seed[0]),
 *   counter = (draw index d, stream id 16 j + purpose, sample index b, low 32 bits of seed[1])
 * for joint j and purpose 0 jitter, 1 good, 2 inv, 3 miss around gt, 4 miss around inv, 5 miss pick, 6 choice,
 * 7 Gaussian pair, 8 keep.  Its words (w0, w1, w2, w3) give two float64 uniforms on [0, 1),
 * u = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 and the same of (w2, w3); U(a, b) = a + (b - a) u as numpy computes it;
 * normals are Box-Muller in fp64, sqrt(-2 ln(1 - u0)) (cos, sin)(2 pi u1).  Stream ids 2^31 + purpose are the
 * augmentation's domain (p2m_augm_params: 0 the flip and keep uniforms, 1 the Gaussian pair), disjoint from the
 * detector noise's 16 j + purpose, so one seed can drive both without correlating them.  A sample's output depends
 * only on its own inputs, its index b and the seed, not on the batch size or on other samples.  DESIGN.md §4.3
 * (dataset inputs) gives the draws each step takes and why the result has the reference's distribution.
 *
 * synthesize_pose (num_overlap = 0) on joints [batch, 17, 3] (x, y, visibility; COCO order) with area [batch] (the
 * crop-space box area the OKS radii scale with) -> out [batch, 17, 3] float32 rows (x, y, 1), or (0, 0, 0) where
 * every candidate is absent.  One launch, one CTA of 288 threads per sample.  Deliberate difference: where the
 * reference's miss candidate list is empty but its inv-source part was drawn (1 to 3 inv-source survivors, none around
 * the joint) it raises; here the miss candidate is absent. */
typedef struct {
  double mean[2];
  double std[2];
  double weight;
} p2m_h36m_error_t;
int p2m_synthesize_pose(const float* joints, const float* area, const int64_t* seed, int batch, float* out,
                        p2m_stream_t stream);
/* generate_syn_error: noise [batch, 17, 2] float32 from error_table (HOST, 17 entries in the Human3.6M joint order,
 * copied into the kernel parameters; finite, std >= 0, 0 <= weight <= 1, else P2M_ERR_INVALID): per joint x ~ N(mean[0],
 * std[0]), y ~ N(mean[1], std[1]) stored as float32, kept iff float32 weight > u, else (0, 0).  One launch. */
int p2m_h36m_syn_error(const p2m_h36m_error_t* error_table, const int64_t* seed, int batch, float* noise,
                       p2m_stream_t stream);
/* A training sample's network input: joints_px [batch, n_joint, 2] image pixels -> pose2d [batch, n_joint, 2].  The
 * crop box is get_bbox -> process_bbox of box_joints [batch, n_box_joint, 2] (NULL: of joints_px) and every joint goes
 * through its rot-0 map into the (input_h, input_w) crop, as p2m_normalize_pose2d computes it; then the noise, then
 * / input size and zero mean / unit std per pose and coordinate.  noise:
 *   P2M_NOISE_NONE  nothing (seed may be NULL); with box_joints the test split's detections mapped through the box of
 *                   the ground-truth joints, without it bitwise p2m_normalize_pose2d
 *   P2M_NOISE_COCO  rows 0-16 (n_joint >= 17) through p2m_synthesize_pose's rule with every joint visible and area =
 *                   the tight box (P2M_AREA_TIGHT) or the processed box (P2M_AREA_CROP, MuCo) mapped into the crop
 *   P2M_NOISE_H36M  n_joint == 17: + (p2m_h36m_syn_error's noise / 256) (input_w, input_h), float32
 * n_joint, n_box_joint <= 32.  One launch, no workspace, no host synchronisation. */
enum {
  P2M_NOISE_NONE = 0,
  P2M_NOISE_COCO = 1,
  P2M_NOISE_H36M = 2
};
enum {
  P2M_AREA_TIGHT = 0,
  P2M_AREA_CROP = 1
};
int p2m_training_pose2d(const float* joints_px, int batch, int n_joint, const float* box_joints, int n_box_joint,
                        int noise, int area_box, const p2m_h36m_error_t* error_table, const int64_t* seed, int input_h,
                        int input_w, float* pose2d, p2m_stream_t stream);
/* A training sample's augmentation parameters (augm_params, lib/aug_utils.py:98-117) for a batch: flip_out [batch]
 * int32 is 1 with probability 1/2 when flip is 1 (else 0); rot_out [batch] float32 degrees is
 * clip(N(0, 1) rotate_factor, +-2 rotate_factor), then 0 with probability 1/2.  Draws from the augmentation's stream
 * domain under the rule above; sample b's draw depends only on (seed, b).  rotate_factor finite and >= 0.  One
 * launch, no host synchronisation. */
int p2m_augm_params(int batch, int flip, double rotate_factor, const int64_t* seed, int32_t* flip_out, float* rot_out,
                    p2m_stream_t stream);
/* p2m_training_pose2d with the sample's augmentation (rot [batch] degrees, flip [batch] int32: device arrays from
 * p2m_augm_params, either NULL for none).  rot != 0 goes into the crop's affine map as get_affine_transform builds it
 * (get_dir in fp64, float32 point pairs, the system solved in fp64); the crop-space area of the COCO noise is
 * unchanged (a rotation keeps the box's corner distances).  A flip is x -> input_w - x - 1 followed by swapping the
 * flip pairs of flip_joint_set (P2M_JOINTS_COCO: n_joint >= 17, P2M_JOINTS_HUMAN36: n_joint == 17): after the noise
 * in float32 (flip_before_noise 0: Human36M, COCO, AMASS), or in fp64 on the crop map's output before the noise
 * (flip_before_noise 1: MuCo's j2d_processing).  With rot and flip NULL, bitwise p2m_training_pose2d, which is this
 * call's no-augmentation case; rot = 0 and flip = 0 give the same bits.  flip_joint_set P2M_JOINTS_SMPL (n_joint ==
 * 24, SURREAL) and P2M_JOINTS_MANO (n_joint == 21, FreiHAND) take no noise; MANO has no flip pairs, so flip must be
 * NULL.  SURREAL's j2d_processing flips in the joints' own dtype: float32 detections flip after the float32 crop
 * (flip_before_noise 0), float64 ground-truth joints flip in fp64 before it is rounded (flip_before_noise 1).  One
 * launch. */
int p2m_training_pose2d_augmented(const float* joints_px, int batch, int n_joint, const float* box_joints,
                                  int n_box_joint, int noise, int area_box, const p2m_h36m_error_t* error_table,
                                  const int64_t* seed, int input_h, int input_w, const float* rot,
                                  const int32_t* flip, int flip_joint_set, int flip_before_noise, float* pose2d,
                                  p2m_stream_t stream);

/* ---- optimizer: the RMSprop step (torch.optim.RMSprop, lib/funcs_utils.py:87-91) ---------------------------------
 * One step of every segment, a segment being one parameter tensor of numel float32 elements: param, grad and
 * square_avg, momentum_buffer when its group has momentum > 0, grad_avg when it is centred (the others may be NULL),
 * and step (a float32 scalar, nullable) incremented by 1.  Per element, in fp32 and in torch's _multi_tensor_rmsprop
 * operation order (each foreach op rounded once, a + alpha * op(b, c) as one fma):
 *   g = g + wd p (wd != 0);  s = s alpha;  s = s + (1 - alpha) g^2;
 *   centred: ga = lerp(ga, g, 1 - alpha), avg = sqrt(s - ga^2) + eps;  else avg = sqrt(s) + eps;
 *   momentum: buf = buf mu + g / avg, p = p - lr buf;  else p = p - lr (g / avg).
 * A group's lr is read from lr_device (a device float32 scalar, read when the kernel runs: a captured step follows a
 * schedule that writes it) or, when that is NULL, is the host lr.  Each element is read and written once: 16-byte
 * accesses where every array of a segment has the same address modulo 16, 4-byte ones for the rest.  Up to 448
 * segments of up to 16 groups per launch, more take more launches.  The segment table is passed as a kernel parameter
 * (capture-safe), no host synchronisation, no atomics: bitwise deterministic.  Every data array is checked to be
 * device memory of one device.                                                                                    */
typedef struct {
  float* param;
  const float* grad;
  float* square_avg;
  float* momentum_buffer;
  float* grad_avg;
  float* step;
  int64_t numel;
  int32_t group; /* index into the groups array */
} p2m_rmsprop_segment_t;
typedef struct {
  double lr;              /* used when lr_device is NULL; finite */
  const void* lr_device;  /* device float32 scalar, or NULL */
  double alpha, eps, weight_decay, momentum; /* finite, >= 0 */
  int32_t centered;       /* 0 or 1 */
} p2m_rmsprop_group_t;
int p2m_rmsprop_step(const p2m_rmsprop_segment_t* segments, int n_segments, const p2m_rmsprop_group_t* groups,
                     int n_groups, p2m_stream_t stream);

/* ---- host-side graph baking helper (CPU; no device work) -------------------------------------------
 * One level of the reference's greedy heavy-edge matching (lib/coarsening.py:153-211, HEM_one_level),
 * entries sorted by (row, col); returns the number of clusters (or -1).  Driven by
 * pose2mesh_release_b200/graph.py, which replaces build_coarse_graphs (lib/graph_utils.py:75-95).   */
int32_t p2m_graph_match_level(int64_t nnz, const int32_t* rows, const int32_t* cols, const double* vals,
                              const int64_t* visit_order, const double* weights, int32_t* cluster_out);

/* ---- misc ----------------------------------------------------------------------------------------*/
const char* p2m_last_error(void);
const char* p2m_version(void);
/* Number of kernels this library launched on behalf of the calling thread since the last reset.    */
int64_t p2m_launch_count(void);
void p2m_launch_count_reset(void);
/* Debug: the process-wide log of tensor-core launches since the last reset, one entry of 9 int32 per launch:
 * kind (0 = Chebyshev conv, 1 = dW, 2 = dense GEMM), output columns per CTA, ring slots, X / T1 stages, MODE (1 = T1
 * given, 0 = plain GEMM), single-pass fp16 (0 / 1), grid.x, grid.y, tiles.  Copies the first min(count, 32768,
 * max_entries) entries into out (NULL: none) and returns the count, which keeps counting past the 32768 it stores. */
int64_t p2m_debug_conv_log(int32_t* out, int max_entries);
void p2m_debug_conv_log_reset(void);

#ifdef __cplusplus
}
#endif
#endif /* P2M_B200_H_ */
