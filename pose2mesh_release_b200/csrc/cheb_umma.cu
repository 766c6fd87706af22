// Hopper (sm_90a) tensor-core kernels of the MeshNet hot path: fp16x3 wgmma with register accumulators.
//
// A Chebyshev graph-conv layer  Y = epilogue( [T0 | T1 | T2](X) * W^T ),  T1 = L~ X, T2 = 2 L~ T1 - X  is two launches:
//
// k_cheb_t1        — T1 = L~ X for every row, written once to HBM (fp32): a 4-deep cp.async ring per 128-row tile,
//                    gathers out of shared memory.
// k_cheb_conv_umma — persistent CTAs; a tile is 128 (or 64) consecutive vertices of one mesh (a compact patch: the
// / _wide            reference's binary-tree vertex order makes rows [128p,128p+128) the descendants of one coarse
//                    node), and a CTA computes 64 (or 128) output columns of its tiles: 128 x 64 for the 64-wide
//                    layers (k_cheb_conv_umma), 64 x 128 for the T1-given and plain convs of the 128- and 256-wide
//                    layers (k_cheb_conv_wide), whose A operand is then built once per 128 output columns.  The two
//                    kernels share one body.
//   * 16 producer warps build the A operand on chip, 32 features at a time: they run the second sparse product from
//     shared memory with a tile-local CSR (the T1 rows of the tile and its 1-hop halo, staged one chunk ahead), read
//     their own X rows straight from global memory, split every fp32 value into an fp16 (hi, lo) pair and write it
//     into the 128B-swizzled K-major operand layout.  T2 is never materialised in HBM.
//   * 2 loader warps stage what the producers gather from: the tile's own T1 rows as one 2-D TMA box where the tile
//     is a run of consecutive rows, every other row (halo, index-list tiles) by 16-byte cp.async with completion
//     through cp.async.mbarrier.arrive.noinc; thread 0 also prefetches the next tile's metadata blob.  1 thread
//     streams the pre-packed fp16 (hi|lo) weight blocks of the CTA's column slice (cp.async.bulk, mbarrier
//     complete_tx).
//   * 1 warpgroup issues wgmma.mma_async (f16 -> f32) into register accumulators: m64n64k16 on both 64-row halves of
//     the tile, or m64n128k16 over the whole weight block in the 64 x 128 configuration (k_cheb_conv_wide, 640
//     threads): per 16 features three MMAs — hi*Whi + lo*Whi + hi*Wlo — an error-compensated product with ~2^-21
//     relative error, which is what keeps the 1e-4 fp32 parity bar (plain TF32/FP16 does not, SURVEY.md §7
//     "hard parts" 1).  After the tile's last K-block the same warpgroup applies the fused epilogue — bias / folded
//     BatchNorm, ReLU, channel-resampled residual (or, for the network's last block, the 64 -> 3 head's projection) —
//     through a per-warp staging buffer, while the producers already fill the ring for the next tile.  N = 64: the
//     accumulator is transposed through swizzled staging so that global accesses are coalesced.  N = 128: two such
//     warpgroups alternate tiles (one runs its epilogue while the other issues the next tile's MMAs; 8 producer warps
//     then build the A operand); the epilogue runs in the fragment layout, in place in linear 512-byte staging rows
//     that the copy engine fills with the identity residual and drains to HBM by cp.async.bulk stores.
// The unpool between levels is virtual: with in_unpool the rows are read from row r>>1 of the coarser
// tensor.  Weights are pre-scaled by 2^6 so that their lo parts stay normal fp16 numbers (undone exactly in the
// epilogue).  The same kernel in `plain` mode is the backward dT GEMM and, with pre-packed A blocks, the dense GEMM;
// k_cheb_dw_umma (below) is the dW reduction with MN-major operands.  Every mbarrier wait is time-bounded (a protocol
// bug sets a status word instead of hanging the GPU) and tools/umma_trace.py dumps a per-role event timeline of CTA 0.
#include <cuda.h>  // CUtensorMap types only: the encoder is fetched through cudaGetDriverEntryPoint
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

#include "p2m_internal.h"

namespace p2m {

namespace {

constexpr int TILE_M = 128;
constexpr int FC = 32;                         // features per chunk (= 128 B of fp32 per row)
constexpr int A_BLOCK_BYTES = TILE_M * 128;    // one K-block of A: 128 rows x (32 hi | 32 lo) fp16
constexpr float W_SCALE = 64.f;
constexpr float W_INV_SCALE = 1.f / 64.f;

// ------------------------------------------------------------------ per-tile metadata blob
// A tile of tm (128 or 64) rows: its own rows (slots 0..tm-1) and their 1-hop halo are staged; the local CSR covers the
// own rows only.
struct TileHeader {  // 64 bytes
  int n_rows;     // valid vertices in this tile (<= tm)
  int h1;         // staged rows: tm tile slots + 1-hop halo
  int nnz;
  int off_halo;   // int32 [h1]    vertex id of staged row i (-1: empty slot)
  int off_rp;     // uint16 [tm+1] local CSR: row i < tm lists the neighbours of vertex halo[i]
  int off_ent;    // uint2 [nnz]   {byte offset of the neighbour's staged row (slot*128), value bits}
  int off_ord2;   // uint16 [tm]   tile rows sorted by decreasing length (warps see equal trip counts)
  int bytes;
  int pad[8];
};
static_assert(sizeof(TileHeader) == 64, "header size");

inline int up16(int x) { return (x + 15) & ~15; }

// Epilogue staging of the 64 x 128 (N = 128) configuration: each MMA warp's 16 x 128 fp32 block as 16 linear rows of
// 512 bytes (what one cp.async.bulk moves) at a stride of 544 bytes.  136 floats is 8 banks mod 32, so the four rows a
// half-warp's 64-bit fragment access touches (8 consecutive words each) cover the 32 banks exactly once.
constexpr int STG_ROW_BYTES = 544;
// per-warp epilogue staging: a 32 x 32 fp32 sub-slab (N = 64), or 16 rows of STG_ROW_BYTES (N = 128)
__host__ __device__ constexpr int stg_warp_bytes(int N) { return N == 128 ? 16 * STG_ROW_BYTES : 32 * 32 * 4; }

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(20000u)  // suspend-time hint (ns): sleep in hardware instead of spinning,
      : "memory");                          // so waiting warps do not take issue slots from the loader warps
  return ok != 0;
}
// Bounded wait: a protocol bug must not hang the GPU box.  On timeout (2 s of %globaltimer: three orders of magnitude
// beyond any legitimate wait, preempted / time-sliced contexts included) the CTA-wide abort flag is raised so that
// every later wait of this CTA falls through, and the wait's id is written to the model's status word — a word of
// MAPPED HOST memory, so the host sees it without a copy: every API entry point checks it and fails with
// P2M_ERR_CUDA (p2m_api.cu: check_kernel_status), i.e. a timed-out kernel never hands results to the caller silently.
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
constexpr unsigned long long MBAR_TIMEOUT_NS = 2000000000ull;
__device__ __noinline__ void mbar_timeout(volatile int* abort_flag, int* status, int code) {
  *abort_flag = 1;
  *reinterpret_cast<volatile int*>(status) = code;
  __threadfence_system();
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, volatile int* abort_flag, int* status,
                                          int code) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0 = 0;
  for (unsigned spin = 0;; ++spin) {
#pragma unroll 1
    for (int it = 0; it < 64; ++it) {
      if (mbar_try_wait(bar, parity)) return;
    }
    if (*abort_flag) return;
    if ((spin & 63u) == 63u) {  // the timer is only consulted every 4096 failed polls (~80 ms of hardware-suspended waits)
      const unsigned long long t = global_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > MBAR_TIMEOUT_NS) break;
    }
  }
  mbar_timeout(abort_flag, status, code);
}
// Same, but with a nanosleep back-off between polls: for the roles whose waits span most of a tile
// (epilogue, loaders) so that their polling does not steal issue slots from the producers.
template <unsigned SLEEP_NS = 200>
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity, volatile int* abort_flag, int* status,
                                                  int code) {
  if (mbar_try_wait(bar, parity)) return;
  unsigned long long t0 = 0;
  for (unsigned spin = 0;; ++spin) {
#pragma unroll 1
    for (int it = 0; it < 16; ++it) {
      if (mbar_try_wait(bar, parity)) return;
      __nanosleep(SLEEP_NS);
    }
    if (*abort_flag) return;
    if ((spin & 255u) == 255u) {
      const unsigned long long t = global_ns();
      if (t0 == 0) t0 = t;
      else if (t - t0 > MBAR_TIMEOUT_NS) break;
    }
  }
  mbar_timeout(abort_flag, status, code);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_async_proxy() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// shared -> global bulk copy, completed through the issuing thread's bulk async-groups (no mbarrier)
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the thread's bulk stores have finished READING their shared-memory source (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... and have completed
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// src_bytes = 16: plain copy; 0: the 16 destination bytes are zero-filled and the source is not read
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// One 2-D tiled TMA load (box = 32 floats x box rows of the tensor map) into dense 128-byte rows.
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* ptr) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
}
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
  // the mbarrier gets this thread's arrival once all of its earlier cp.async copies have landed
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
template <int NT>
__device__ __forceinline__ void producer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory"); }
// explicit shared-window accesses (32-bit addresses): keeps the hot loops on LDS/STS instead of generic LD/ST
__device__ __forceinline__ float4 lds_f4(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ uint2 lds_u2(uint32_t a) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) {
  unsigned short v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts_f4(uint32_t a, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts_f2(uint32_t a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void sts_u2(uint32_t a, const uint2& v) {
  asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ void fma4(float4& acc, float w, const float4& x) {
  acc.x = fmaf(w, x.x, acc.x);
  acc.y = fmaf(w, x.y, acc.y);
  acc.z = fmaf(w, x.z, acc.z);
  acc.w = fmaf(w, x.w, acc.w);
}
// One CSR row with four entries in flight: the four (slot, value) pairs are fetched first, then the four
// 16-byte row pieces, then the FMAs on two accumulators — the row's dependent chain is ~2 shared-memory round
// trips per four entries instead of two per entry (rows have <= 14 entries).  (Fetching each entry once per row and
// passing it round the row's 8 lanes with width-8 shuffles was measured in round 2: 15 % SLOWER — shuffles run on
// the same MIO/shared-memory pipe that bounds these kernels.)
// T2 = 2 (L~ T1) - X, one FMA per element (2 g is exact, so this rounds like the subtraction of the doubled value)
__device__ __forceinline__ float4 cheb_t2(const float4& g, const float4& x) {
  return make_float4(fmaf(2.f, g.x, -x.x), fmaf(2.f, g.y, -x.y), fmaf(2.f, g.z, -x.z), fmaf(2.f, g.w, -x.w));
}
__device__ __forceinline__ float4 gather_row4(uint32_t ent, uint32_t e, uint32_t e1, uint32_t rows_q) {
  float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
  for (; e + 3 < e1; e += 4) {
    const uint2 a0 = lds_u2(ent + e * 8), a1 = lds_u2(ent + e * 8 + 8), a2 = lds_u2(ent + e * 8 + 16),
                a3 = lds_u2(ent + e * 8 + 24);
    const float4 x0 = lds_f4(rows_q + a0.x), x1 = lds_f4(rows_q + a1.x), x2 = lds_f4(rows_q + a2.x),
                 x3 = lds_f4(rows_q + a3.x);
    fma4(acc0, __uint_as_float(a0.y), x0);
    fma4(acc1, __uint_as_float(a1.y), x1);
    fma4(acc0, __uint_as_float(a2.y), x2);
    fma4(acc1, __uint_as_float(a3.y), x3);
  }
  if (e + 1 < e1) {
    const uint2 a0 = lds_u2(ent + e * 8), a1 = lds_u2(ent + e * 8 + 8);
    const float4 x0 = lds_f4(rows_q + a0.x), x1 = lds_f4(rows_q + a1.x);
    fma4(acc0, __uint_as_float(a0.y), x0);
    fma4(acc1, __uint_as_float(a1.y), x1);
    e += 2;
  }
  if (e < e1) {
    const uint2 a0 = lds_u2(ent + e * 8);
    fma4(acc0, __uint_as_float(a0.y), lds_f4(rows_q + a0.x));
  }
  return make_float4(acc0.x + acc1.x, acc0.y + acc1.y, acc0.z + acc1.z, acc0.w + acc1.w);
}

// wgmma (Hopper warpgroup MMA): D[regs] += A[smem] * B[smem]^T (scale-d = 1: always accumulate), f16 -> f32, M = 64 rows
// per warpgroup.
// Accumulator fragment of thread t: d[4j + 2r + c] = D[16 (t/32) + (t%32)/4 + 8r][8j + 2 (t%4) + c].
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// both operands K-major in shared memory (the immediates after p: scale-a, scale-b, transpose-a, transpose-b)
__device__ __forceinline__ void wgmma_m64n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}
// the same with N = 128 (64 accumulator registers): d[h][j] is element j + 32 h of the fragment, i.e. d[h] holds the
// 64-column half h exactly as an m64n64 on that half would
__device__ __forceinline__ void wgmma_m64n128(float (&d)[2][32], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0][0]), "+f"(d[0][1]), "+f"(d[0][2]), "+f"(d[0][3]), "+f"(d[0][4]), "+f"(d[0][5]), "+f"(d[0][6]),
        "+f"(d[0][7]), "+f"(d[0][8]), "+f"(d[0][9]), "+f"(d[0][10]), "+f"(d[0][11]), "+f"(d[0][12]), "+f"(d[0][13]),
        "+f"(d[0][14]), "+f"(d[0][15]), "+f"(d[0][16]), "+f"(d[0][17]), "+f"(d[0][18]), "+f"(d[0][19]), "+f"(d[0][20]),
        "+f"(d[0][21]), "+f"(d[0][22]), "+f"(d[0][23]), "+f"(d[0][24]), "+f"(d[0][25]), "+f"(d[0][26]), "+f"(d[0][27]),
        "+f"(d[0][28]), "+f"(d[0][29]), "+f"(d[0][30]), "+f"(d[0][31]), "+f"(d[1][0]), "+f"(d[1][1]), "+f"(d[1][2]),
        "+f"(d[1][3]), "+f"(d[1][4]), "+f"(d[1][5]), "+f"(d[1][6]), "+f"(d[1][7]), "+f"(d[1][8]), "+f"(d[1][9]),
        "+f"(d[1][10]), "+f"(d[1][11]), "+f"(d[1][12]), "+f"(d[1][13]), "+f"(d[1][14]), "+f"(d[1][15]), "+f"(d[1][16]),
        "+f"(d[1][17]), "+f"(d[1][18]), "+f"(d[1][19]), "+f"(d[1][20]), "+f"(d[1][21]), "+f"(d[1][22]), "+f"(d[1][23]),
        "+f"(d[1][24]), "+f"(d[1][25]), "+f"(d[1][26]), "+f"(d[1][27]), "+f"(d[1][28]), "+f"(d[1][29]), "+f"(d[1][30]),
        "+f"(d[1][31])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}
// M = 64, N = 32 (16 accumulator registers), both operands MN-major (transposed: 1, 1) in shared memory
__device__ __forceinline__ void wgmma_m64n32(float (&d)[16], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(desc_a), "l"(desc_b)
      : "memory");
}

// K-major, 128B-swizzled operand block (rows of 128 bytes, 8-row atoms of 1024 bytes).
// wgmma matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset [49,52) = 0 (blocks are
// 1024-byte aligned), layout type [62,64) with SWIZZLE_128B = 1.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;            // LBO (unused for swizzled K-major) = 16 B
  d |= (uint64_t)(1024 >> 4) << 32;  // SBO = 1024 B between 8-row groups
  d |= (uint64_t)1 << 62;            // SWIZZLE_128B
  return d;
}

// byte offset of 16-byte chunk `chunk` (0..7) of row `row` inside a 128B-swizzled block
__host__ __device__ __forceinline__ uint32_t sw128_off(int row, int chunk) {
  return (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
}

// K-major, 64B-swizzled operand block of the single-pass fp16 precision (rows of 64 bytes = 32 fp16, 8-row atoms of
// 512 bytes): the hardware XORs address bits [4,6) with bits [7,9), i.e. the 16-byte chunk with (row >> 1) & 3.
// Descriptor: as above with SBO = 512 B and layout type SWIZZLE_64B = 2 (blocks are 512-byte aligned).
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;           // LBO (unused for swizzled K-major) = 16 B
  d |= (uint64_t)(512 >> 4) << 32;  // SBO = 512 B between 8-row groups
  d |= (uint64_t)2 << 62;           // SWIZZLE_64B
  return d;
}
// byte offset of 16-byte chunk `chunk` (0..3) of row `row` inside a 64B-swizzled block
__host__ __device__ __forceinline__ uint32_t sw64_off(int row, int chunk) {
  return (uint32_t)row * 64u + (uint32_t)((chunk ^ ((row >> 1) & 3)) << 4);
}
// bytes per operand row of a K-block (32 features): fp16 (hi | lo) for fp16x3, hi only for the single pass
__host__ __device__ constexpr int op_row_bytes(bool f16) { return f16 ? 64 : 128; }

struct Half4 {
  __half2 a, b;
};
// fp16 round-to-nearest of four values (the single-pass precision's operand)
__device__ __forceinline__ uint2 half4(const float4& v) {
  __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  return make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
}
__device__ __forceinline__ void split4(const float4& v, uint2& hi, uint2& lo) {
  __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
  __half2 l0 = __floats2half2_rn(v.x - f0.x, v.y - f0.y), l1 = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
  hi.x = *reinterpret_cast<uint32_t*>(&h0);
  hi.y = *reinterpret_cast<uint32_t*>(&h1);
  lo.x = *reinterpret_cast<uint32_t*>(&l0);
  lo.y = *reinterpret_cast<uint32_t*>(&l1);
}

struct KParams {
  const float* x;
  int in_unpool;
  int V, P, fin;
  int n_tiles;
  const unsigned char* meta;
  const int* meta_bytes;
  int meta_stride, max_h1;
  const unsigned char* wpack;
  const float* zero_row;  // 128 bytes of zeros: source of the empty halo slots of ragged tiles
  EpiDev ep;
  int res_identity;       // residual resampling is the identity (Fin_block == Fout): vector path
  const float* t1;        // MODE 1: T1 = L~ x, [rows, fin] at LOGICAL rows (k_cheb_t1): the conv kernel stages the
                          // T1 rows of the tile and its 1-hop halo and only runs the second sparse product on chip
  const float* a_scale;   // optional device scalar: x is multiplied by it before the fp16 split (power of two,
                          // chosen from max|x|: gradients are far below fp16's range) and divided out afterwards
  const float* b_scale;   // dense GEMM, optional: the device scalar the B operand was packed with in place of W_SCALE
  long long ldy;          // row stride of y in floats, and first output column
  int y_col0;
  float* y;
  int* status;
  long long* trace;  // optional [8][512] event log of CTA 0 (debug): (event << 48) | clock
  int own_table;         // 1: the tile's rows are the index list at the head of its metadata blob (TileSet), not
                         //    the consecutive rows [TM pat, TM pat + TM) (TM = tile rows of the configuration)
  const float* head_wt;  // optional fused thin head (N == 64): epilogue writes head_z[row][12] = y_row * head_wt[64][12]
  float* head_z;
  // Dense GEMM mode (launch_umma_gemm: PoseNet's Linear layers): the A operand is PRE-PACKED like a weight image
  // (k_pack on the activation matrix: one 16 KB block per (128-row tile, 32-feature chunk)), so both operands of
  // every K-block arrive by cp.async.bulk and no producer warp runs; blockIdx.y selects an N-wide slice of the output
  // columns (its weight image, epilogue vectors and output / residual columns).
  const unsigned char* apack;
  long long wslice_bytes;  // offset of this CTA's N-slice (blockIdx.y) in the weight image
  long long wblock_stride; // bytes between consecutive K-blocks of the weight image
  int tma;           // 1: the tile's own rows of x (and t1) arrive by one 2-D TMA load each (consecutive tiles on
                     //    levels whose size is a multiple of 128); with in_unpool the x box is the TM / 2 source rows
  CUtensorMap tm_x, tm_t1;
};

// Event timeline of CTA 0 (tools/umma_trace.py): compiled in only with -DP2M_UMMA_TRACE (build.py: P2M_TRACE=1);
// production kernels carry no clock reads.
#ifdef P2M_UMMA_TRACE
__device__ __forceinline__ void trace_ev(const KParams& p, int role, int& n, int ev) {
  if (p.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && n < 512) {
    p.trace[role * 512 + n] = ((long long)ev << 48) | (clock64() & 0xFFFFFFFFFFFFll);
    ++n;
  }
}
#else
__device__ __forceinline__ void trace_ev(const KParams&, int, int&, int) {}
#endif

// Warp roles of the 128 x 64 configuration (N = 64, k_cheb_conv_umma: 24 warps = 6 warpgroups, one persistent CTA
// per SM):
//   0..15  producers: SpMM out of shared memory + fp16 (hi,lo) split + swizzled A-block stores
//   16,17  loaders: stage the T1 (and, where the producers do not read it directly, X) rows of the next chunk; thread 0 also fetches
//          the next tile's metadata (cp.async.bulk), thread 32 issues the TMA boxes
//   18     weight-block loader (one thread, cp.async.bulk)
//   19     idle
//   20..23 MMA + epilogue warpgroup: wgmma into register accumulators -> fused epilogue -> HBM
constexpr int W_PROD = 16;
constexpr int W_XLOAD = 16, N_XLOAD = 2, W_BLOAD = 18, W_EPI0 = 20;
constexpr int NUM_THREADS2 = 24 * 32;
constexpr int REGS_LAUNCH = 80, REGS_UTIL = 40, REGS_EPI = 120;  // setmaxnreg targets per warpgroup (see the kernel)
// setmaxnreg.inc draws on the pool the CTA's own setmaxnreg.dec filled: requests beyond it would spin forever
static_assert(128 * (REGS_EPI - REGS_LAUNCH) <= 128 * (REGS_LAUNCH - REGS_UTIL), "register pool balance");
static_assert(W_XLOAD % 4 == 0 && W_EPI0 % 4 == 0 && W_EPI0 - W_XLOAD == 4, "setmaxnreg works on aligned warpgroups");
// The 64 x 128 configuration (N = 128, k_cheb_conv_wide: 20 warps = 5 warpgroups) has two MMA + epilogue warpgroups
// that alternate tiles, so that one runs its epilogue while the other issues the next tile's MMAs, and half the
// producers (two tile rows per thread).  640 threads launch with 96 registers (65536 / 640, rounded down to a multiple
// of 8), enough for one m64n128k16 per K step, whose 64 accumulator registers ptxas refuses below 90:
//   0..7   producers          8..11  MMA + epilogue warpgroup 1 (the CTA's odd tiles)
//   12..15 loaders (12, 13), weight-block loader (14), idle (15)
//   16..19 MMA + epilogue warpgroup 0 (the even tiles)
constexpr int W_PROD_W = 8, W_EPI1_W = 8, W_XLOAD_W = 12, W_BLOAD_W = 14, W_EPI0_W = 16;
constexpr int NUM_THREADS_W = 20 * 32;
constexpr int REGS_LAUNCH_W = 96, REGS_UTIL_W = 40, REGS_PROD_W = 88, REGS_EPI_W = 128;
static_assert(2 * 128 * (REGS_EPI_W - REGS_LAUNCH_W) <=
                  128 * (REGS_LAUNCH_W - REGS_UTIL_W) + 2 * 128 * (REGS_LAUNCH_W - REGS_PROD_W),
              "register pool balance of the 64 x 128 layout");
static_assert(REGS_LAUNCH_W * NUM_THREADS_W <= 65536 && (REGS_LAUNCH_W + 8) * NUM_THREADS_W > 65536,
              "__launch_bounds__(NUM_THREADS_W, 1) gives REGS_LAUNCH_W registers per thread");
static_assert(W_EPI1_W == W_PROD_W && W_EPI1_W % 4 == 0 && W_XLOAD_W == W_EPI1_W + 4 && W_EPI0_W == W_XLOAD_W + 4 &&
                  (W_EPI0_W + 4) * 32 == NUM_THREADS_W,
              "setmaxnreg works on aligned warpgroups");
// the role map and register targets of configuration N
template <int N>
struct ConvRoles {
  static constexpr int threads = NUM_THREADS2, prod = W_PROD, xload = W_XLOAD, bload = W_BLOAD, epi0 = W_EPI0,
                       epi1 = -1;
  static constexpr int regs_launch = REGS_LAUNCH, regs_util = REGS_UTIL, regs_prod = REGS_LAUNCH, regs_epi = REGS_EPI;
};
template <>
struct ConvRoles<128> {
  static constexpr int threads = NUM_THREADS_W, prod = W_PROD_W, xload = W_XLOAD_W, bload = W_BLOAD_W,
                       epi0 = W_EPI0_W, epi1 = W_EPI1_W;
  static constexpr int regs_launch = REGS_LAUNCH_W, regs_util = REGS_UTIL_W, regs_prod = REGS_PROD_W,
                       regs_epi = REGS_EPI_W;
};

// Two tile shapes, both a 64-register fp32 accumulator per thread of the one MMA warpgroup:
//   N = 64:  a CTA computes 128 tile rows x the 64 output columns [64 blockIdx.y, 64 blockIdx.y + 64); used for the
//            64-wide layers (and the fused thin head) and the dense GEMM.
//   N = 128: a CTA computes 64 tile rows x the 128 output columns [128 blockIdx.y, 128 blockIdx.y + 128); used for every
//            conv with Fout % 128 == 0, so that a tile row's A operand is built once per 128 output columns instead of
//            once per 64.  The tiles are the 64-row metadata families (DevLevel::meta64, TileSet::m64).
// MODE 1: T1 given (k_cheb_t1): the producers run the second sparse product out of the staged T1 rows.
// MODE 0: plain GEMM, no sparse product (the isolated rows of padding elision, the backward dT GEMMs, the dense GEMM).
template <int N>
__host__ __device__ constexpr int tile_rows() { return N == 128 ? 64 : TILE_M; }

// ------------------------------------------------------------------ dynamic shared-memory layouts
// conv_smem, dw_smem and t1_smem describe each kernel's dynamic shared memory once: the kernel carves its buffers at
// these byte offsets from its 1024-byte aligned base, the host takes the launch size and every fit test from `bytes`
// (the conv and dW sizes include 1024 + 32 bytes of slack that the kernels do not use).  Stage sizes are in floats.

// cheb_conv_body<N, NC, NS, XS, MODE, F16> (NC output columns per CTA: 64, 128 or 256) on tiles of at most max_h1
// staged rows, metadata blobs meta_stride bytes apart
struct ConvSmem {
  size_t xs, xs_stage, t1s, t1_stage, meta, bars, flags, ep, stage, own, tail, bytes;
};
__host__ __device__ __forceinline__ ConvSmem conv_smem(int NC, int NS, int XS, int MODE, int max_h1, int meta_stride,
                                                       bool f16 = false) {
  const int N = NC == 64 ? 64 : 128;  // accumulator columns of an MMA warpgroup
  const int tm = N == 128 ? 64 : TILE_M;
  size_t at = 0, sum = 0;  // next offset; total size of the buffers
  auto take = [&](size_t bytes) { sum += bytes; at += bytes; return at - bytes; };
  ConvSmem L;
  // the ring at offset 0, [NS] slots: A block (tm rows) + B block (NC rows) of 128 B (fp16x3) or 64 B (fp16) rows
  take((size_t)NS * (tm + NC) * op_row_bytes(f16));
  // [XS][tm][32] fp32 own X rows: read in MODE 0 only (MODE 1 reads X from global memory); none at MODE 1, tm = 64
  L.xs_stage = (MODE == 1 && tm == 64) ? 0 : (size_t)tm * FC;
  L.xs = take(XS * L.xs_stage * 4);
  L.t1_stage = MODE == 1 ? (size_t)max_h1 * FC : 0;  // [XS][max_h1][32] fp32: T1 rows of the tile and its 1-hop halo
  L.t1s = take(XS * L.t1_stage * 4);
  L.meta = take(2 * (size_t)meta_stride);    // [2] tile metadata blobs (the dense GEMM: none)
  L.bars = take(8 * (2 * NS + 2 * XS + 6));  // the kernel's barrier map
  L.flags = take(16);                        // word 1: the CTA's abort flag
  L.ep = take(2 * 4 * NC);                   // epilogue vectors ep_mul, ep_add [NC]
  at = (at + 127) & ~(size_t)127;
  L.stage = take(4 * stg_warp_bytes(N));  // [4 warps] epilogue staging, 128-byte aligned
  L.own = take(4 * 32 * 4);               // [NWG][4 warps][ER] epilogue rows' vertex ids (NWG * ER = 32)
  L.tail = take(N == 64 ? 64 * 12 * 4 : 4 * 8);  // N = 64: fused-head weights [64][12]; N = 128: 4 residual mbarriers
  L.bytes = sum + 128 + 1024 + 32;               // (128: the staging buffer's alignment)
  return L;
}

// The body of both conv kernels: k_cheb_conv_umma (N = 64) and k_cheb_conv_wide (N = 128) differ in their role map
// and register targets (ConvRoles<N>) and in their launch size.  NC = output columns per CTA: N, or 2 N (64 x 256,
// k_cheb_conv_wide only), where both MMA warpgroups work on every tile, warpgroup g on the CTA's columns
// [g N, g N + N), and read the one A block the producers built for them.
// F16: the single-pass fp16 precisions (P2M_PREC_FP16_TC, P2M_PREC_FP16_MIXED_TC): a K-block holds only the fp16
// round-to-nearest of each operand (64-byte rows, 64B-swizzled) and every 16 features take one k16 MMA instead of three.
// Same chunks, slots and barrier protocol; T1-given and plain convs (a_scale applied before the rounding), no dense-GEMM
// mode.
template <int N, int NC, int NS, int XS, int MODE, bool F16>
__device__ __forceinline__ void cheb_conv_body(const KParams& p) {
  static_assert(N == 64 || N == 128, "one warpgroup holds the CTA's 128 x 64 or 64 x 128 accumulator in registers");
  static_assert(NC == N || (N == 128 && NC == 2 * N && MODE == 1),
                "64 x 256: both MMA warpgroups of the 64 x 128 layout, T1-given convs only (conv_cols)");
  static_assert(NS == 3 || NS == 6, "the producers fill a chunk's three slots back to back");
  using R = ConvRoles<N>;
  constexpr int TM = tile_rows<N>();  // tile rows
  constexpr int NPW = R::prod;        // producer warps
  constexpr int NRG = NPW * 4;        // producer row groups (8 threads each)
  constexpr int RPT = TM / NRG;       // tile rows per producer thread (2: row groups rg and NRG + rg of the row order)
  constexpr int NWG = N == 128 ? 2 : 1;  // MMA + epilogue warpgroups (they alternate tiles, or split NC columns)
  constexpr bool COLS = NC != N;         // 64 x 256: the warpgroups split the columns of every tile
  static_assert(RPT == 2, "both configurations give a producer thread two tile rows");
  constexpr int H = TM / 64;          // M = 64 halves of the tile (one accumulator each)
  constexpr int ER = 16 * H;          // epilogue rows per warp of the MMA warpgroup
  constexpr bool KT1 = (MODE == 1);
  constexpr bool plain = !KT1;
  constexpr int RB = op_row_bytes(F16);  // bytes per operand row of a K-block
  constexpr int A_BYTES = TM * RB;       // one K-block of A: TM rows x (32 hi | 32 lo) fp16, or 32 fp16 (F16)
  constexpr int B_BLOCK_BYTES = NC * RB;
  constexpr int SLOT_BYTES = A_BYTES + B_BLOCK_BYTES;
  static_assert(NWG * ER == 32 && SLOT_BYTES == (TM + NC) * RB, "conv_smem describes this configuration");
  static_assert(SLOT_BYTES % 1024 == 0 && A_BYTES % 1024 == 0, "swizzled blocks stay aligned to their atoms");

  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const ConvSmem L = conv_smem(NC, NS, XS, MODE, p.max_h1, p.meta_stride, F16);
  unsigned char* ring = smem_raw;  // 128B-swizzled blocks need 1024-byte alignment (checked below)
  float* Xs = reinterpret_cast<float*>(smem_raw + L.xs);
  float* T1s = reinterpret_cast<float*>(smem_raw + L.t1s);
  unsigned char* meta_s = smem_raw + L.meta;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + L.bars);
  // barrier map
  uint64_t* b_ab_full = bars;                // [NS]
  uint64_t* b_ab_empty = b_ab_full + NS;     // [NS]
  uint64_t* b_x_full = b_ab_empty + NS;      // [XS]
  uint64_t* b_x_empty = b_x_full + XS;       // [XS]
  uint64_t* b_m_full = b_x_empty + XS;       // [2]
  uint64_t* b_m_empty = b_m_full + 2;        // [2]
  // N = 128: the output stores of the epilogue before have read the staging buffer, which passes from one MMA
  // warpgroup's epilogue to the other's (one arrival per warp); the tile before has finished its main loop (one arrival
  // per warp; not used at NC = 2 N)
  uint64_t* b_stg_free = b_m_empty + 2;      // [1]
  uint64_t* b_turn = b_stg_free + 1;         // [1]
  uint32_t* flags = reinterpret_cast<uint32_t*>(smem_raw + L.flags);
  volatile int* abort_flag = reinterpret_cast<volatile int*>(flags + 1);
  float* ep_mul = reinterpret_cast<float*>(smem_raw + L.ep);  // [NC] acc * mul + add  (weight scale, bias, folded BN)
  float* ep_add = ep_mul + NC;
  // epilogue staging: N = 64: [4 warps][32 rows][EC floats], 16-byte chunks XOR-swizzled by the row, one 32-column
  // sub-slab at a time; N = 128: [4 warps][16 rows][STG_ROW_BYTES], a warp's whole 16 x 128 block in linear rows
  constexpr int EC = 32;
  constexpr int STG_WARP_BYTES = stg_warp_bytes(N);
  unsigned char* epi_stage = smem_raw + L.stage;
  // (N = 128: the two MMA warpgroups share the staging buffer, one tile after the other)
  int* own_s = reinterpret_cast<int*>(smem_raw + L.own);  // [NWG][4 warps][ER] vertex id of each epilogue row
  float* head_w_s = reinterpret_cast<float*>(smem_raw + L.tail);  // [64][12] (N == 64 with a fused head)
  uint64_t* b_res = reinterpret_cast<uint64_t*>(head_w_s);  // [4] (N = 128: no head) per staging block: its tile's
                                                            // identity-residual rows have landed in it

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int n_chunk = p.fin / FC;
  const int n_use = 3 * n_chunk;

  if (tid == 0) {
    for (int s = 0; s < NS; ++s) {
      // one elected arrive per producer warp + the weight loader (dense GEMM mode: the loader alone)
      mbar_init(smem_u32(b_ab_full + s), p.apack != nullptr ? 1 : NPW + 1);
      mbar_init(smem_u32(b_ab_empty + s), COLS ? 8 : 4);  // one arrival per warp of each MMA warpgroup reading it
    }
    for (int s = 0; s < XS; ++s) {
      mbar_init(smem_u32(b_x_full + s), N_XLOAD * 32 + 1);  // every loader thread (cp.async.mbarrier.arrive.noinc)
                                                            // + one expect_tx (TMA) / plain arrival of loader thread 32
      mbar_init(smem_u32(b_x_empty + s), 1);
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(b_m_full + s), 1);
      mbar_init(smem_u32(b_m_empty + s), 1);
    }
    if (N == 128) {
      for (int w = 0; w < 4; ++w) mbar_init(smem_u32(b_res + w), 1);  // the warp's expect_tx arrival + its copies' bytes
      mbar_init(smem_u32(b_stg_free), 4);
      mbar_init(smem_u32(b_turn), 4);
    }
    *abort_flag = (smem_u32(ring) & 1023u) ? 1 : 0;
    if (*abort_flag) mbar_timeout(abort_flag, p.status, 100);
    fence_barrier_init();
  }
  const float a_scale = p.a_scale ? *p.a_scale : 1.f;
  const float b_inv = p.b_scale ? 1.f / *p.b_scale : W_INV_SCALE;
  const int ccol0 = (int)blockIdx.y * NC;  // first output column of this CTA's column slice
  for (int n = threadIdx.x; n < NC; n += R::threads) {
    const float sc = (p.ep.scale ? p.ep.scale[ccol0 + n] : 1.f) / a_scale;
    const float sh = p.ep.scale ? p.ep.shift[ccol0 + n] : 0.f;
    const float bi = p.ep.bias ? p.ep.bias[ccol0 + n] : 0.f;
    ep_mul[n] = b_inv * sc;
    ep_add[n] = fmaf(bi, p.ep.scale ? p.ep.scale[ccol0 + n] : 1.f, sh);
  }
  if (N == 64 && p.head_z != nullptr)
    for (int i = threadIdx.x; i < 64 * 12; i += R::threads) head_w_s[i] = p.head_wt[i];
  __syncthreads();

  // Register split by warpgroup.  N = 64 (launched with 80 per thread: 768 x 80 = 60 K of the SM's 64 K): the
  // utility warpgroup (loaders, weight loader) drops to 40 per thread and the MMA + epilogue warpgroup takes exactly
  // what that frees (120 per thread): the 64 accumulator registers plus the epilogue's addresses and residual state
  // (at 104 ptxas spilled twice as much).  The producers stay at 80.  N = 128 (launched with 96: 640 x 96 = 60 K): the
  // utility warpgroup drops to 40 and the two producer warpgroups to 88, which pays for the two MMA + epilogue
  // warpgroups at 128.
  // (each budget is set at the top of its own region: after a join ptxas has to assume the smallest one)
  const int mma_g = warp >= R::epi0 ? 0 : (NWG == 2 && warp >= R::epi1 && warp < R::epi1 + 4) ? 1 : -1;
  if (warp >= R::xload && warp < R::epi0) {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R::regs_util));
  if (warp >= R::xload && warp < R::xload + N_XLOAD) {
    // ------------------------------------------------------------ loaders (two warps): tile metadata, own rows, halo rows
    // Per stage (tile, 32-feature chunk) they bring in what the producers read: the tile's metadata blob (thread 0,
    // cp.async.bulk, one tile ahead), the own rows of X / T1 (one 2-D TMA box each where the tile is a run of
    // consecutive rows — thread 32), and every other staged row with 16-byte cp.async copies (8 lanes per 128-byte row,
    // all 64 threads): the T1 rows of the 1-hop halo, or all rows where the tile is an index list.
    // A stage needs ~60 warp-level copies; issued by the 16 producer warps (round 2 until this change) every warp paid
    // the whole preamble for its one to four rows — a fifth of the producers' instruction stream per chunk.
    if (p.apack == nullptr) {
      const int lt = tid - R::xload * 32;  // 0..63
      const int lq = lt & 7, lrg = lt >> 3;
      const int my_tiles = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
      if (lt == 32 && p.tma) {
        if (plain) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&p.tm_x)) : "memory");
        if (KT1) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&p.tm_t1)) : "memory");
      }
      auto fetch_meta = [&](int itf) {  // thread 0: blob of this CTA's tile number itf into buffer itf & 1
        const int pat = (blockIdx.x + itf * gridDim.x) % p.P;
        const int m = itf & 1;
        mbar_wait_relaxed(smem_u32(b_m_empty + m), ((itf >> 1) & 1) ^ 1, abort_flag, p.status, 1);
        const int mbytes = p.meta_bytes[pat];
        mbar_arrive_expect_tx(smem_u32(b_m_full + m), mbytes);
        bulk_g2s(smem_u32(meta_s + (size_t)m * p.meta_stride), p.meta + (size_t)pat * p.meta_stride, mbytes,
                 smem_u32(b_m_full + m));
      };
      if (lt == 0 && my_tiles > 0) fetch_meta(0);
      const uint32_t fin_bytes = (uint32_t)p.fin * 4u;
      const int sh = p.in_unpool ? 1 : 0;
      int g2 = 0;
      int ltn = 0;
      for (int it2 = 0; it2 < my_tiles; ++it2) {
        const int tile2 = blockIdx.x + it2 * gridDim.x;
        const long long mesh_row0 = (long long)(tile2 / p.P) * p.V;
        const int m2 = it2 & 1;
        mbar_wait_relaxed(smem_u32(b_m_full + m2), (it2 >> 1) & 1, abort_flag, p.status, 8);
        const unsigned char* mb2 = meta_s + (size_t)m2 * p.meta_stride;
        const TileHeader* hdr2 = reinterpret_cast<const TileHeader*>(mb2);
        const int* halo = reinterpret_cast<const int*>(mb2 + hdr2->off_halo);
        const int h1 = hdr2->h1;
        for (int c2 = 0; c2 < n_chunk; ++c2, ++g2) {
          const int xs2 = g2 % XS;
          mbar_wait_relaxed(smem_u32(b_x_empty + xs2), ((g2 / XS) & 1) ^ 1, abort_flag, p.status, 11);
          if (lt == 0) trace_ev(p, 4, ltn, 1);
          const uint32_t xbar = smem_u32(b_x_full + xs2);
          // a row's byte offset inside its mesh fits 32 bits: one 32 x 32 -> 64-bit multiply-add per row; empty slots
          // (-1) are zero-filled by the copy itself (src-size 0)
          auto stage_rows = [&](uint32_t dbase, const char* sbase, int first, int n_rows, int shift) {
            for (int i0 = first + lrg; i0 < n_rows; i0 += 32) {
              int v[4];
#pragma unroll
              for (int u = 0; u < 4; ++u) v[u] = (i0 + 8 * u < n_rows) ? halo[i0 + 8 * u] : -2;
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                if (v[u] != -2) {
                  const uint32_t srow = (uint32_t)max(v[u], 0) >> shift;
                  cp_async16_zfill(dbase + (i0 + 8 * u) * 128, sbase + (uint64_t)srow * (uint64_t)fin_bytes,
                                   v[u] >= 0 ? 16u : 0u);
                }
              }
            }
          };
          const char* t1_mesh =
              reinterpret_cast<const char*>(KT1 ? p.t1 + mesh_row0 * p.fin + c2 * FC + lq * 4 : nullptr);
          const char* x_mesh = reinterpret_cast<const char*>(p.x + (mesh_row0 >> sh) * p.fin + c2 * FC + lq * 4);
          const uint32_t t1_dst = smem_u32(T1s + xs2 * L.t1_stage) + lq * 16;
          const uint32_t x_dst = smem_u32(Xs + xs2 * L.xs_stage) + lq * 16;
          if (p.tma) {
            if (lt == 32) {
              const int own0 = tile2 * TM;  // V is a multiple of 128: tiles never straddle meshes
              mbar_arrive_expect_tx(xbar, KT1 ? TM * 128 : (p.in_unpool ? TM / 2 : TM) * 128);
              if (plain)
                tma_load_2d(smem_u32(Xs + xs2 * L.xs_stage), &p.tm_x, c2 * FC, p.in_unpool ? own0 >> 1 : own0, xbar);
              if (KT1) tma_load_2d(smem_u32(T1s + xs2 * L.t1_stage), &p.tm_t1, c2 * FC, own0, xbar);
            }
            if (KT1) stage_rows(t1_dst, t1_mesh, TM, h1, 0);  // only the halo rows are left
          } else {
            if (KT1) stage_rows(t1_dst, t1_mesh, 0, h1, 0);
            if (plain) stage_rows(x_dst, x_mesh, 0, TM, sh);
            if (lt == 32) mbar_arrive(xbar);
          }
          cp_async_arrive_noinc(xbar);  // this thread's arrival once its copies have landed
          if (lt == 0) trace_ev(p, 4, ltn, 2);
          // next tile's metadata: its buffer was last read for tile it2 - 1, which the producers have left by the time
          // the second chunk of this tile could be staged (single-chunk layers: by the time its only chunk could)
          if (lt == 0 && c2 == (n_chunk > 1 ? 1 : 0) && it2 + 1 < my_tiles) fetch_meta(it2 + 1);
        }
      }
    }
  } else if (warp == R::bload) {
    // ------------------------------------------------------------ weight-block loader (one thread)
    if (lane == 0) {
      uint32_t ucnt = 0;
      int tn = 0;
      const int uses = plain ? n_chunk : n_use;
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        for (int u = 0; u < uses; ++u, ++ucnt) {
          const int s = ucnt % NS;
          const uint32_t par = (ucnt / NS) & 1;
          mbar_wait_relaxed(smem_u32(b_ab_empty + s), par ^ 1, abort_flag, p.status, 4);
          trace_ev(p, 1, tn, 10 + u);
          const unsigned char* wsl = p.wpack + (size_t)blockIdx.y * (size_t)p.wslice_bytes;
          if (p.apack != nullptr) {  // dense GEMM mode: the tile's pre-packed A block of chunk u rides along
            mbar_arrive_expect_tx(smem_u32(b_ab_full + s), B_BLOCK_BYTES + A_BYTES);
            bulk_g2s(smem_u32(ring + s * SLOT_BYTES), p.apack + ((size_t)tile * uses + u) * A_BYTES, A_BYTES,
                     smem_u32(b_ab_full + s));
          } else {
            mbar_arrive_expect_tx(smem_u32(b_ab_full + s), B_BLOCK_BYTES);
          }
          bulk_g2s(smem_u32(ring + s * SLOT_BYTES + A_BYTES), wsl + (size_t)u * (size_t)p.wblock_stride, B_BLOCK_BYTES,
                   smem_u32(b_ab_full + s));
        }
      }
    }
  }
  } else if (mma_g >= 0) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R::regs_epi));
    // ------------------------------------------------------------ MMA + epilogue warpgroup(s)
    // wgmma into register accumulators acc[2][32].  N = 64: two 64 x 64 ones (m64n64), the two M = 64 row halves of the
    // 128-row tile.  N = 128: one m64n128 fragment over the 64-row tile, whose element j + 32 h is acc[h][j], i.e. acc[h]
    // is the tile's 64-column half h.  Warp wq of the warpgroup holds rows 16 wq .. 16 wq + 15 of each row half (its ER
    // "epilogue rows": local row lr <-> tile row 64 (lr / 16) + 16 wq + lr % 16).
    // A thread's fragment covers two columns of every 8-column group, so storing it directly would scatter.  N = 64: the
    // rows are transposed through a small per-warp staging buffer so that a warp-wide 16-byte access covers whole
    // 128-byte row pieces, and the fused epilogue (affine, ReLU, residual) runs in that layout, where the residual reads
    // coalesce.  N = 128: the epilogue writes its results in place into the warp's linear staging rows, which then
    // leave whole by bulk copy.
    // N = 128: warpgroup g takes the CTA's tiles it = g, g + 2, ...  Both walk the one A/B ring (tile it's K-blocks are
    // uses it * uses ..), so main loops run in tile order: a warpgroup starts one when the other has finished the tile
    // before (b_turn; the ring's parity waits then never run more than one phase ahead), and runs its epilogue while the
    // other issues the next tile's MMAs.  The staging buffer passes from one epilogue to the next (b_stg_free).
    // NC = 2 N: both warpgroups take every tile, warpgroup g its columns [g N, g N + N) (the B block's rows g N ..),
    // each slot is freed by the eight warps that read it, and the epilogues take the staging buffer in turn (warpgroup 0,
    // then 1) while the producers fill the ring for the next tile.
    const int g = mma_g;
    const int ecol0 = ccol0 + (COLS ? g * N : 0);  // first output column of this warpgroup's accumulator
    const float* ep_mul_g = ep_mul + (COLS ? g * N : 0);
    const float* ep_add_g = ep_add + (COLS ? g * N : 0);
    const int wq = warp - (g == 0 ? R::epi0 : R::epi1);
    const int tr = 3 + 2 * g;  // trace role of the warpgroup's warp 0
    constexpr int CPR = EC / 4;             // 16-byte chunks per staged row
    constexpr int RPI = 32 / CPR;           // rows covered by one warp-wide 16-byte access
    const uint32_t stg = smem_u32(epi_stage) + (uint32_t)wq * STG_WARP_BYTES;
    const int prow = lane / CPR, pc = lane % CPR;
    constexpr int NP = ER / RPI;            // phase-2 rows (pieces) per thread and sub-slab
    int colk[2];  // column (inside a sub-slab) of the 16-byte chunk this thread handles for rows of swizzle class k
#pragma unroll
    for (int k = 0; k < 2; ++k) colk[k] = (int)(((uint32_t)pc ^ (uint32_t)((k * RPI + prow) & 7)) << 2);
    const int trow = (lane >> 4) * 64 + wq * 16 + (lane & 15);  // tile row of local row `lane` (lane < ER)
    const int uses = plain ? n_chunk : n_use;
    int etn = 0;
    for (int it = COLS ? 0 : g; (int)blockIdx.x + it * (int)gridDim.x < p.n_tiles; it += COLS ? 1 : NWG) {
      const int e = COLS ? 2 * it + g : it;  // this epilogue's turn at the staging buffer
      const int tile = blockIdx.x + it * gridDim.x;
      const int b = tile / p.P, pat = tile - b * p.P;
      const long long mesh0 = (long long)b * p.V;
      int* own_w = own_s + (g * 4 + wq) * ER;
      {
        int v;
        if (lane >= ER) {
          v = -1;
        } else if (p.own_table) {
          v = __ldg(reinterpret_cast<const int*>(p.meta + (size_t)pat * p.meta_stride + 64) + trow);
        } else {
          v = pat * TM + trow;
          if (v >= p.V) v = -1;
        }
        __syncwarp();  // the previous tile's readers of own_w are done
        if (lane < ER) own_w[lane] = v;  // (own_w is only read at rows < ER)
        __syncwarp();
      }
      int own_v[NP];
#pragma unroll
      for (int i = 0; i < NP; ++i) own_v[i] = own_w[i * RPI + prow];
      if (p.ep.res != nullptr) {
        // pull this tile's residual rows into L2 while its main loop is still running (only the CTA's own columns
        // where they are read by column: dense GEMM, and the identity residual of N = 128)
        const bool own_cols = p.apack != nullptr || (N == 128 && p.res_identity);
        const int lpr = ((own_cols ? N : p.ep.res_F) * 4 + 127) >> 7;
        for (int j = lane; j < ER * lpr; j += 32) {
          const int rr = j / lpr, ln = j - rr * lpr;
          const int vtx = own_w[rr];
          if (vtx >= 0) {
            const long long r = mesh0 + vtx;
            prefetch_l2(p.ep.res + (p.ep.res_unpool ? (r >> 1) : r) * p.ep.res_F + (own_cols ? ecol0 : 0) + ln * 32);
          }
        }
      }
      float acc[2][32];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;
      if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 1);
      if (NWG == 2 && !COLS && it > 0) {
        mbar_wait(smem_u32(b_turn), (uint32_t)(it - 1) & 1u, abort_flag, p.status, 13);
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 3);
      }
      uint32_t ucnt = (uint32_t)it * (uint32_t)uses;
      for (int u = 0; u < uses; ++u, ++ucnt) {
        const uint32_t s = ucnt % NS;
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 4);
        mbar_wait(smem_u32(b_ab_full + s), (ucnt / NS) & 1, abort_flag, p.status, 6);
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 5);
        const uint32_t a0 = smem_u32(ring + s * SLOT_BYTES);
        wg_fence();
        // A block columns: [hi 0..31 | lo 32..63], B block columns: [Whi 0..31 | Wlo 32..63] (fp16); a 16-element K
        // step is 32 bytes = +2 in the descriptor's start-address field.  F16: columns 0..31 only, two k16 steps.
        if constexpr (F16 && N == 128) {
          const uint64_t da = make_desc_sw64(a0);
          const uint64_t db = make_desc_sw64(a0 + A_BYTES + (COLS ? (uint32_t)g * (N * RB) : 0u));
          wgmma_m64n128(acc, da + 0, db + 0);
          wgmma_m64n128(acc, da + 2, db + 2);
        } else if constexpr (F16) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint64_t da = make_desc_sw64(a0 + (uint32_t)h * (64 * RB));
            const uint64_t db = make_desc_sw64(a0 + A_BYTES);
            wgmma_m64n64(acc[h], da + 0, db + 0);
            wgmma_m64n64(acc[h], da + 2, db + 2);
          }
        } else if constexpr (N == 128) {
          // the whole 128-row B block is one N = 128 operand (its rows 64..127 are the next eight 1024-byte atoms), so
          // each A sub-block is read once per K step; every output element sees the same six k16 MMAs in the same
          // order as with two m64n64 column halves
          const uint64_t da = make_desc_sw128(a0);
          const uint64_t db = make_desc_sw128(a0 + A_BYTES + (COLS ? (uint32_t)g * (N * 128) : 0u));
          wgmma_m64n128(acc, da + 0, db + 0);  // hi * Whi
          wgmma_m64n128(acc, da + 2, db + 2);
          wgmma_m64n128(acc, da + 4, db + 0);  // lo * Whi
          wgmma_m64n128(acc, da + 6, db + 2);
          wgmma_m64n128(acc, da + 0, db + 4);  // hi * Wlo
          wgmma_m64n128(acc, da + 2, db + 6);
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            // rows 64..127 of the A block (the tile's second M = 64 half) start 8 KB further on
            const uint64_t da = make_desc_sw128(a0 + (uint32_t)h * (64 * 128));
            const uint64_t db = make_desc_sw128(a0 + A_BYTES);
            wgmma_m64n64(acc[h], da + 0, db + 0);  // hi * Whi
            wgmma_m64n64(acc[h], da + 2, db + 2);
            wgmma_m64n64(acc[h], da + 4, db + 0);  // lo * Whi
            wgmma_m64n64(acc[h], da + 6, db + 2);
            wgmma_m64n64(acc[h], da + 0, db + 4);  // hi * Wlo
            wgmma_m64n64(acc[h], da + 2, db + 6);
          }
        }
        wg_commit();
        wg_wait0();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(b_ab_empty + s));  // this warp is done reading the slot
      }
      if (NWG == 2 && !COLS && lane == 0) mbar_arrive(smem_u32(b_turn));  // the next tile's main loop may start
      if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 2);
      // N = 64, phase 1 of sub-slab cb (32 columns): the fragment into the staging rows (16-byte chunks XOR-swizzled by
      // row)
      auto stage_slab = [&](int cb) {
#pragma unroll
        for (int h = 0; h < H; ++h)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const int lr = 16 * h + (lane >> 2) + 8 * r;
              const int cc = 8 * jj + 2 * (lane & 3);
              const int j = 4 * (cb / 8 + jj) + 2 * r;
              sts_f2(stg + lr * (EC * 4) + ((((uint32_t)(cc >> 2)) ^ (uint32_t)(lr & 7)) << 4) + (cc & 3) * 4,
                     acc[h][j], acc[h][j + 1]);
            }
        __syncwarp();
      };
      if (N == 64 && p.head_z != nullptr) {
        // fused thin head: thread = local row; y_n = act(acc_n * mul_n + add_n) never leaves the chip, only the
        // 12 projections Z = y W' (W' = [W0 - W2 | W1 | W2] of the 64 -> 3 layer, 4-padded) are written
        float z[12];
#pragma unroll
        for (int j = 0; j < 12; ++j) z[j] = 0.f;
#pragma unroll
        for (int cb = 0; cb < N; cb += 32) {
          stage_slab(cb);
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            const float4 a = lds_f4(stg + lane * (EC * 4) + (((uint32_t)c ^ (uint32_t)(lane & 7)) << 4));
            const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int n = cb + 4 * c + e;
              float t = fmaf(av[e], ep_mul[n], ep_add[n]);
              if (p.ep.relu) t = fmaxf(t, 0.f);
              const float4 w0 = *reinterpret_cast<const float4*>(head_w_s + n * 12);
              const float4 w1 = *reinterpret_cast<const float4*>(head_w_s + n * 12 + 4);
              const float4 w2 = *reinterpret_cast<const float4*>(head_w_s + n * 12 + 8);
              z[0] = fmaf(t, w0.x, z[0]); z[1] = fmaf(t, w0.y, z[1]); z[2] = fmaf(t, w0.z, z[2]); z[3] = fmaf(t, w0.w, z[3]);
              z[4] = fmaf(t, w1.x, z[4]); z[5] = fmaf(t, w1.y, z[5]); z[6] = fmaf(t, w1.z, z[6]); z[7] = fmaf(t, w1.w, z[7]);
              z[8] = fmaf(t, w2.x, z[8]); z[9] = fmaf(t, w2.y, z[9]); z[10] = fmaf(t, w2.z, z[10]); z[11] = fmaf(t, w2.w, z[11]);
            }
          }
          __syncwarp();
        }
        if (own_w[lane] >= 0) {
          float4* zr = reinterpret_cast<float4*>(p.head_z + (mesh0 + own_w[lane]) * 12);
          zr[0] = make_float4(z[0], z[1], z[2], z[3]);
          zr[1] = make_float4(z[4], z[5], z[6], z[7]);
          zr[2] = make_float4(z[8], z[9], z[10], z[11]);
        }
      } else if (N == 128) {
        // The staging block is this tile's once the tile before (the other warpgroup's) has handed it over: its output
        // stores have read it.  An identity residual then lands in it by bulk copy (one 512-byte row per valid row,
        // straight into the row's slot, from L2: prefetched at tile start).  In the accumulator's own layout, in place:
        // o = act(acc * mul + add), plus that residual, goes to the element's slot of its linear staging row.
        // (b_res[wq] is armed and waited for by one epilogue at a time, in turn order: its phase is the turn's parity)
        if (e > 0) mbar_wait(smem_u32(b_stg_free), (uint32_t)(e - 1) & 1u, abort_flag, p.status, 14);
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 20);
        const bool res_id = p.ep.res != nullptr && p.res_identity;
        if (res_id) {
          const uint32_t rbar = smem_u32(b_res + wq);
          const int n_valid = __popc(__ballot_sync(0xFFFFFFFFu, lane < ER && own_w[lane] >= 0));
          if (lane == 0) mbar_arrive_expect_tx(rbar, (uint32_t)n_valid * (N * 4));
          __syncwarp();
          if (lane < ER && own_w[lane] >= 0) {
            const long long r = mesh0 + own_w[lane];
            bulk_g2s(stg + lane * STG_ROW_BYTES, p.ep.res + (p.ep.res_unpool ? (r >> 1) : r) * p.ep.res_F + ecol0, N * 4,
                     rbar);
          }
          mbar_wait(rbar, (uint32_t)e & 1u, abort_flag, p.status, 12);
        }
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 21);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int jg = 0; jg < 8; ++jg) {
            const int n = 64 * h + 8 * jg + 2 * (lane & 3);  // column pair of acc[h][4 jg + 2 r + {0, 1}]
            const float2 mu = *reinterpret_cast<const float2*>(ep_mul_g + n);
            const float2 ad = *reinterpret_cast<const float2*>(ep_add_g + n);
#pragma unroll
            for (int r = 0; r < 2; ++r) {
              const int j = 4 * jg + 2 * r;
              const uint32_t a = stg + ((lane >> 2) + 8 * r) * STG_ROW_BYTES + n * 4;
              float o0 = fmaf(acc[h][j], mu.x, ad.x), o1 = fmaf(acc[h][j + 1], mu.y, ad.y);
              if (p.ep.relu) {
                o0 = fmaxf(o0, 0.f);
                o1 = fmaxf(o1, 0.f);
              }
              if (res_id) {
                const float2 rv = lds_f2(a);
                o0 += rv.x;
                o1 += rv.y;
              }
              sts_f2(a, o0, o1);
            }
          }
        if (p.ep.res != nullptr && !p.res_identity) {
          // channel-resampled residual (its rows are wider than a staging row: no prefetch): one row-major pass over
          // the staged rows, 4 columns per lane
          __syncwarp();
          const int gn = ecol0 + 4 * lane;  // column of the layer's output
          for (int rr = 0; rr < ER; ++rr) {
            const int vtx = own_w[rr];
            if (vtx >= 0) {
              const long long r = mesh0 + vtx;
              const float* res_row = p.ep.res + (p.ep.res_unpool ? (r >> 1) : r) * p.ep.res_F;
              const uint32_t a = stg + rr * STG_ROW_BYTES + lane * 16;
              const float4 v = lds_f4(a);
              float o[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float l = __ldg(p.ep.lam + gn + e);
                o[e] += (1.f - l) * __ldg(res_row + __ldg(p.ep.i0 + gn + e)) + l * __ldg(res_row + __ldg(p.ep.i1 + gn + e));
              }
              sts_f4(a, make_float4(o[0], o[1], o[2], o[3]));
            }
          }
        }
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 22);
        // Out by bulk copy, one 512-byte row per valid row; the warpgroup waits only until the copies have read the
        // staging block, then hands it to the next tile's epilogue
        fence_async_proxy();  // this thread's staging writes -> the async proxy the copies read through
        __syncwarp();
        if (lane < ER) {
          if (own_w[lane] >= 0)
            bulk_s2g(p.y + (mesh0 + own_w[lane]) * p.ldy + p.y_col0 + ecol0, stg + lane * STG_ROW_BYTES, N * 4);
          bulk_commit();
        }
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 23);
        if (lane < ER) bulk_wait_read0();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(b_stg_free));
        if (wq == 0 && lane == 0) trace_ev(p, tr, etn, 24);
      } else {
#pragma unroll
        for (int cb = 0; cb < N; cb += 32) {
          stage_slab(cb);
          // phase 2: lane = (row inside an RPI-row group, 16-byte chunk); the thread's output columns of this
          // sub-slab and their affine coefficients are fetched once per sub-slab
          float4 mu_k[2], ad_k[2];
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            mu_k[k] = *reinterpret_cast<const float4*>(ep_mul + cb + colk[k]);
            ad_k[k] = *reinterpret_cast<const float4*>(ep_add + cb + colk[k]);
          }
#pragma unroll
          for (int i = 0; i < NP; ++i) {
            const int rr = i * RPI + prow;
            const int n = cb + colk[i & 1];
            const int gn = ecol0 + n;  // column of the layer's output
            const float4 a = lds_f4(stg + rr * (EC * 4) + (pc << 4));
            const int vtx = own_v[i];
            if (vtx >= 0) {
              const float4 mu = mu_k[i & 1], ad = ad_k[i & 1];
              float o[4] = {fmaf(a.x, mu.x, ad.x), fmaf(a.y, mu.y, ad.y), fmaf(a.z, mu.z, ad.z), fmaf(a.w, mu.w, ad.w)};
              if (p.ep.relu) {
#pragma unroll
                for (int e = 0; e < 4; ++e) o[e] = fmaxf(o[e], 0.f);
              }
              const long long r = mesh0 + vtx;
              if (p.ep.res != nullptr) {
                const float* res_row = p.ep.res + (p.ep.res_unpool ? (r >> 1) : r) * p.ep.res_F;
                if (p.res_identity) {
                  const float4 rv = __ldg(reinterpret_cast<const float4*>(res_row + gn));
                  o[0] += rv.x; o[1] += rv.y; o[2] += rv.z; o[3] += rv.w;
                } else {
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float l = __ldg(p.ep.lam + gn + e);
                    o[e] += (1.f - l) * __ldg(res_row + __ldg(p.ep.i0 + gn + e)) + l * __ldg(res_row + __ldg(p.ep.i1 + gn + e));
                  }
                }
              }
              *reinterpret_cast<float4*>(p.y + r * p.ldy + p.y_col0 + gn) = make_float4(o[0], o[1], o[2], o[3]);
            }
          }
          __syncwarp();
        }
      }
    }
    if (N == 128 && lane < ER) bulk_wait0();  // the last tile's output stores read shared memory until they complete
  } else {
    if (R::regs_prod < R::regs_launch) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R::regs_prod));
    if (p.apack == nullptr) {
    // ------------------------------------------------------------ producers (16 warps; N = 128: 8)
    const int q = tid & 7;     // float4 lane inside the 32-feature chunk
    const int rg = tid >> 3;   // row group 0..NRG-1
    const uint32_t t1s_a = smem_u32(T1s);
    const uint32_t ring_a = smem_u32(ring);
    const int my_tiles = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int n_stage = my_tiles * n_chunk;  // flat sequence of (tile, chunk) stages of this CTA

    // this thread's tile rows (row groups rg and NRG + rg of the tile's row order) and their CSR extents
    uint32_t row[RPT], re[RPT], ent_a = 0;
    int ptn = 0;
    // A/B ring cursor (slot, phase parity) kept incrementally, and the store offsets of this thread's rows inside an
    // A block (first / second 8-byte store of each row: odd row groups store lo first, see emit()) — per-tile
    // constants: the hot loop carries no modulo, division or swizzle arithmetic
    uint32_t slot = 0, spar = 0;
    uint32_t so_f[RPT], so_s[RPT];
#pragma unroll
    for (int ps = 0; ps < RPT; ++ps) row[ps] = re[ps] = so_f[ps] = so_s[ps] = 0;
    const bool odd = (rg & 1) != 0;
    auto next_slot = [&]() {
      if (++slot == (uint32_t)NS) {
        slot = 0;
        spar ^= 1u;
      }
    };

    const int xsh = (p.tma && p.in_unpool) ? 1 : 0;  // TMA-staged unpooled input: staged row = tile row >> 1
    // T1 given: the thread's own X rows come straight from global memory.  Their only reader is the producer thread
    // that emits them, so staging them would cost a shared-memory write plus a read back (8 % of the kernel's
    // shared-memory traffic, and more than half of the loaders' copies on index-list tiles) for nothing.
    const float* xp[RPT];  // this thread's own X rows (nullptr: empty slot), at its 16-byte column
#pragma unroll
    for (int ps = 0; ps < RPT; ++ps) xp[ps] = nullptr;
    int it = 0, c = -1;
    for (int g = 0; g < n_stage; ++g) {
      if (++c == n_chunk) {
        c = 0;
        ++it;
      }
      const int m = it & 1;
      const int xs = g % XS;
      float4 xd[RPT];
#pragma unroll
      for (int ps = 0; ps < RPT; ++ps) {
        xd[ps] = make_float4(0.f, 0.f, 0.f, 0.f);
        // in flight while the stage wait and the gather run (first chunk: below, after the tile setup)
        if (KT1 && c != 0 && xp[ps]) xd[ps] = __ldg(reinterpret_cast<const float4*>(xp[ps] + c * FC));
      }
      if (tid == 0) trace_ev(p, 0, ptn, 1);
      mbar_wait(smem_u32(b_x_full + xs), (g / XS) & 1, abort_flag, p.status, 9);
      if (tid == 0) trace_ev(p, 0, ptn, 2);

      if (c == 0) {  // per-tile bookkeeping: which rows this thread owns and where their CSR rows start/end
        mbar_wait(smem_u32(b_m_full + m), (it >> 1) & 1, abort_flag, p.status, 8);  // (long complete: the loaders read it)
        const unsigned char* mb = meta_s + (size_t)m * p.meta_stride;
        const TileHeader* hdr = reinterpret_cast<const TileHeader*>(mb);
        const uint32_t mb_a = smem_u32(mb);
        const uint32_t rp_a = mb_a + hdr->off_rp, ord2_a = mb_a + hdr->off_ord2;
        ent_a = mb_a + hdr->off_ent;
#pragma unroll
        for (int ps = 0; ps < RPT; ++ps) {
          // plain GEMM: the thread's rows are the consecutive slots rg and NRG + rg
          row[ps] = plain ? (uint32_t)(NRG * ps + rg) : lds_u16(ord2_a + 2 * (NRG * ps + rg));
          re[ps] = plain ? 0u : (lds_u16(rp_a + 2 * row[ps]) | (lds_u16(rp_a + 2 * row[ps] + 2) << 16));
          const uint32_t i = row[ps];
          if (F16) {  // one 8-byte piece per row (a row lies in the 64-byte bank half of its parity)
            so_f[ps] = so_s[ps] = sw64_off(i, q >> 1) + (q & 1) * 8;
          } else {
            const uint32_t a_hi = sw128_off(i, q >> 1) + (q & 1) * 8, a_lo = sw128_off(i, 4 + (q >> 1)) + (q & 1) * 8;
            so_f[ps] = odd ? a_lo : a_hi;
            so_s[ps] = odd ? a_hi : a_lo;
          }
        }
        if (KT1) {
          const int* halo = reinterpret_cast<const int*>(mb + hdr->off_halo);  // slots 0..TM-1 = the tile's own rows
          const int sh = p.in_unpool ? 1 : 0;
          const long long mesh_row0 = (long long)((blockIdx.x + (unsigned)it * gridDim.x) / (unsigned)p.P) * p.V;
          const float* xm = p.x + (mesh_row0 >> sh) * p.fin + q * 4;
#pragma unroll
          for (int ps = 0; ps < RPT; ++ps) {
            const int v = halo[row[ps]];
            xp[ps] = (v >= 0) ? xm + (size_t)((uint32_t)v >> sh) * (uint32_t)p.fin : nullptr;
            if (xp[ps]) xd[ps] = __ldg(reinterpret_cast<const float4*>(xp[ps]));
          }
        }
      }
      const uint32_t xs_q = smem_u32(Xs + xs * L.xs_stage) + q * 16;
      const uint32_t t1s_q = t1s_a + (uint32_t)(xs * L.t1_stage * 4) + q * 16;
      if (plain) {
        // plain GEMM: the staged rows ARE the A operand (scaled into fp16 range if a_scale is given)
        const uint32_t s = slot;
        mbar_wait(smem_u32(b_ab_empty + s), spar ^ 1u, abort_flag, p.status, 10);
        const uint32_t ablk = ring_a + s * SLOT_BYTES;
#pragma unroll
        for (int ps = 0; ps < RPT; ++ps) {
          const uint32_t i = ps * NRG + rg;
          float4 v = lds_f4(xs_q + (i >> xsh) * 128);
          v.x *= a_scale; v.y *= a_scale; v.z *= a_scale; v.w *= a_scale;
          if (F16) {  // rows rg and rg + 1 of a half-warp have opposite parity: different 64-byte bank halves
            sts_u2(ablk + so_f[ps], half4(v));
            continue;
          }
          uint2 hi, lo;
          split4(v, hi, lo);
          // the four consecutive rows of a warp share (row & 4), i.e. the 64-byte half their hi parts go to: odd row
          // groups store lo first (selects, see emit()), so that both rows of a half-warp cover different bank halves
          sts_u2(ablk + so_f[ps], odd ? lo : hi);
          sts_u2(ablk + so_s[ps], odd ? hi : lo);
        }
        fence_async_proxy();
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(smem_u32(b_ab_full + s));
        next_slot();
        producer_barrier<NPW * 32>();
        if (tid == 0) mbar_arrive(smem_u32(b_x_empty + xs));  // stage free: the loaders may refill it
        if (tid == 0 && c == n_chunk - 1) mbar_arrive(smem_u32(b_m_empty + m));
        continue;
      }
      // Split to fp16 (hi, lo) and write the three K-blocks (X, T1, T2 = 2 L~ T1 - X) of the tile rows this thread
      // finishes: the gather first (measured faster than emitting X and T1 before it: the gather then overlaps the
      // previous chunk's tail instead of this chunk's own stores), then the three blocks back to back under ONE
      // generic->async proxy fence (it drains the thread's outstanding shared stores and is expensive).  Odd row groups
      // store lo first: a warp then covers both 64-byte halves of its rows per store.
      const uint32_t slot0 = slot;
      auto emit = [&](const float4 (&vv)[RPT]) {
        const uint32_t ablk = ring_a + slot * SLOT_BYTES;
#pragma unroll
        for (int ps = 0; ps < RPT; ++ps) {
          uint2 hi, lo;
          float4 v = vv[ps];
          if (p.a_scale != nullptr) {  // backward-data pass: gradients are scaled into fp16's range (power of two)
            v.x *= a_scale; v.y *= a_scale; v.z *= a_scale; v.w *= a_scale;
          }
          if (F16) {  // (two rows of one parity in a half-warp take two wavefronts: see balance_store_halves)
            sts_u2(ablk + so_f[ps], half4(v));
            continue;
          }
          split4(v, hi, lo);
          // 64-bit shared stores are served per HALF-warp (two rows here).  Odd row groups store lo first — by
          // selects, not branches: a predicated store would leave each half-warp's wavefront half empty — and the
          // row order pairs rows so that the two 64-byte pieces of a half-warp fall into different bank halves
          sts_u2(ablk + so_f[ps], odd ? lo : hi);
          sts_u2(ablk + so_s[ps], odd ? hi : lo);
        }
        next_slot();
      };
      float4 t1v[RPT], t2[RPT];
#pragma unroll
      for (int ps = 0; ps < RPT; ++ps) t2[ps] = gather_row4(ent_a, re[ps] & 0xFFFFu, re[ps] >> 16, t1s_q);
#pragma unroll
      for (int ps = 0; ps < RPT; ++ps) t1v[ps] = lds_f4(t1s_q + row[ps] * 128);
      if (tid == 0) trace_ev(p, 0, ptn, 6);
      {
        // one wait for the chunk's three slots: the MMA issuer commits them in order, so the last one being free
        // implies the other two (each mbarrier wait is a ~200-cycle round trip on the critical path of the chunk)
        uint32_t s2 = slot + 2, p2 = spar;
        if (s2 >= (uint32_t)NS) {
          s2 -= (uint32_t)NS;
          p2 ^= 1u;
        }
        mbar_wait(smem_u32(b_ab_empty + s2), p2 ^ 1u, abort_flag, p.status, 10);
      }
      emit(xd);
      emit(t1v);
#pragma unroll
      for (int ps = 0; ps < RPT; ++ps) t2[ps] = cheb_t2(t2[ps], xd[ps]);
      emit(t2);
      fence_async_proxy();
      __syncwarp();
      if ((tid & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 3; ++k) mbar_arrive(smem_u32(b_ab_full + (slot0 + k) % NS));  // one arrival per warp
      }
      if (tid == 0) trace_ev(p, 0, ptn, 7);
      producer_barrier<NPW * 32>();  // everybody is done with Xs[xs] and T1s
      if (tid == 0) trace_ev(p, 0, ptn, 8);
      if (tid == 0) mbar_arrive(smem_u32(b_x_empty + xs));  // stage free: the loaders may refill it
      if (tid == 0 && c == n_chunk - 1) mbar_arrive(smem_u32(b_m_empty + m));
    }
    }
  }
}

template <int N, int NS, int XS, int MODE>
__global__ void __launch_bounds__(NUM_THREADS2, 1) k_cheb_conv_umma(const __grid_constant__ KParams p) {
  static_assert(N == 64, "the 64 x 128 configuration is k_cheb_conv_wide");
  cheb_conv_body<N, N, NS, XS, MODE, false>(p);
}
// NC = 128 (64 x 128) or 256 (64 x 256) output columns per CTA
template <int NC, int NS, int XS, int MODE>
__global__ void __launch_bounds__(NUM_THREADS_W, 1) k_cheb_conv_wide(const __grid_constant__ KParams p) {
  cheb_conv_body<128, NC, NS, XS, MODE, false>(p);
}
// The same two configurations at the single-pass fp16 precisions (fp16, fp16_mixed): one body, F16 = true
template <int N, int NS, int XS, int MODE>
__global__ void __launch_bounds__(NUM_THREADS2, 1) k_cheb_conv_f16_umma(const __grid_constant__ KParams p) {
  static_assert(N == 64, "the 64 x 128 configuration is k_cheb_conv_f16_wide");
  cheb_conv_body<N, N, NS, XS, MODE, true>(p);
}
template <int NC, int NS, int XS, int MODE>
__global__ void __launch_bounds__(NUM_THREADS_W, 1) k_cheb_conv_f16_wide(const __grid_constant__ KParams p) {
  cheb_conv_body<128, NC, NS, XS, MODE, true>(p);
}

// =====================================================================================
// dW on tensor cores:  dW[o, (f,k)] = sum_rows dz[row, o] * T_k[row, f]
//
// The reduction runs over the ROWS, so both operands are "MN-major" for the tensor core (the K index of the
// MMA is the mesh row).  The 128B-swizzled row-major blocks the forward kernel already builds — 128 rows x
// [hi 32 | lo 32] fp16 of T_k for one 32-feature chunk — are exactly a canonical MN-major SWIZZLE_128B tile
// (K = 128 rows of 128 bytes, MN = 64 elements), so the producers are shared with the forward and T2 is
// formed on chip from the given T1 instead of being materialised (the SIMT path writes and re-reads 3x the activations).
// A = the plain-side tile (dz, or the layer input in swapped mode), split (hi, lo) and stored the same way
// ([128 rows] x 64 channels per block).  Per T block: 8 K-steps x three wgmma.m64n32k16 (g_hi T_hi + g_lo T_hi +
// g_hi T_lo, the lo half of T addressed 64 bytes into the swizzle row) with M = 64 channels, N = 32 features,
// accumulated in registers across ALL tiles of the CTA: one feature chunk (T0, T1, T2: 3 x 16 registers) and 64
// channels per launch; one atomicAdd pass per CTA at the end.
// =====================================================================================
// Two operand roles (L~ symmetric:  sum_rows dz (x) T_k(X) = sum_rows T_k(dz) (x) X), selected by `swap`:
//   swap = 0: `x` is the layer INPUT [rows(/2), fin] whose basis the producers build, `g` the gradient dz [rows,
//             fout_total] (plain tile, scaled by a_scale); dw[o][f*3+k] with o from the plain side.
//   swap = 1: `x` is the GRADIENT dz [rows, fin := layer Fout] (gathered, scaled by a_scale), `g` the layer input
//             [rows(/2), fout_total := layer Fin] (plain tile, unscaled, read at row >> 1 under the virtual unpool);
//             the accumulator rows are then input features and the columns output channels: dw[o][f*3+k] with o from
//             the gathered side.
// Either way `t1` = L~ x for every row of the level (launch_cheb_t1): the producers stage the T1 rows of the tile and its
// 1-hop halo and form T2 on chip.
struct DwParams {
  const float* x;        // gathered side
  int in_unpool;
  int V, P, fin;
  int n_tiles;
  const unsigned char* meta;
  const int* meta_bytes;
  int meta_stride, max_h1;
  const float* g;        // plain side [rows(/2), fout_total]
  int fout_total, m_off, m_cols;
  int chunk0;            // feature chunk of this launch (its T0, T1, T2 are the MMA warpgroup's three accumulators)
  const float* a_scale;  // device scalar (power of two) applied to the gradient tensor before the fp16 split
  float* dw;             // reference layout [Fout, 3 Fin], column = f*3 + k, accumulated atomically
  int* status;
  const float* t1;
  int g_unpool;
  int swap;
  int tma;                 // consecutive tiles, V % 128 == 0, no unpool: the own rows of x and t1 arrive by one 2-D TMA box each
  CUtensorMap tm_x, tm_t1;
};

__device__ __forceinline__ uint64_t make_desc_sw128_mn(uint32_t saddr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;  // LBO: distance between 64-element MN groups
  d |= (uint64_t)(1024 >> 4) << 32;                  // SBO: distance between 8-row K groups
  d |= (uint64_t)1 << 62;                            // SWIZZLE_128B
  return d;
}

// The single-pass fp16 weight gradient (k_cheb_dw_f16_umma, P2M_PREC_FP16_MIXED_TC) keeps the chunks, ring, barriers
// and producers, and stores only the fp16 round-to-nearest of each operand: a T block is 128 rows x 32 fp16 = 64-byte
// rows, the canonical MN-major SWIZZLE_64B tile (8-row K groups of 512 bytes, N = 32 = one swizzle atom), and the
// plain-side tile is the hi block of its 64 channels alone (128-byte rows, MN-major SWIZZLE_128B as above).  Each
// 16-row K step issues one wgmma.m64n32k16 (g T) where fp16x3 issues three.
__device__ __forceinline__ uint64_t make_desc_sw64_mn(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)(8192 >> 4) << 16;  // LBO: distance between 32-element MN groups (N = 32: only one is read)
  d |= (uint64_t)(512 >> 4) << 32;   // SBO: distance between 8-row K groups
  d |= (uint64_t)2 << 62;            // SWIZZLE_64B
  return d;
}

constexpr int DW_NS = 3;
constexpr int DW_G_BYTES = 4 * A_BLOCK_BYTES;  // dz tile: (hi, lo) x two 64-channel groups
// bytes of one ring slot (a T block) and of the plain-side tile; f16: the single-pass layout
__host__ __device__ constexpr int dw_t_bytes(bool f16) { return f16 ? TILE_M * 64 : A_BLOCK_BYTES; }
__host__ __device__ constexpr int dw_g_bytes(bool f16) { return f16 ? A_BLOCK_BYTES : DW_G_BYTES; }

// k_cheb_dw_umma<XS> (k_cheb_dw_f16_umma<XS>: f16) on the level's 128-row tiles (at most max_h1 staged rows, blobs
// meta_stride bytes apart)
struct DwSmem {
  size_t gblk, xs, t1s, t1_stage, meta, bars, flags, bytes;
};
__host__ __device__ __forceinline__ DwSmem dw_smem(int XS, int max_h1, int meta_stride, bool f16 = false) {
  size_t at = 0;
  auto take = [&](size_t bytes) { at += bytes; return at - bytes; };
  DwSmem L;
  take(DW_NS * (size_t)dw_t_bytes(f16));      // the ring at offset 0: [DW_NS] T blocks
  L.gblk = take(dw_g_bytes(f16));             // dz tile blocks: hi g0, hi g1, lo g0, lo g1 (f16: hi g0)
  L.xs = take(XS * (size_t)TILE_M * FC * 4);  // [XS][128][32] fp32: the tile's own rows of x
  L.t1_stage = (size_t)max_h1 * FC;           // [XS][max_h1][32] fp32: T1 rows of the tile and its 1-hop halo
  L.t1s = take(XS * L.t1_stage * 4);
  L.meta = take(2 * (size_t)meta_stride);        // [2] tile metadata blobs
  L.bars = take(8 * (2 * DW_NS + 2 * XS + 6));  // the kernel's barrier map
  L.flags = take(16);                            // word 1: the CTA's abort flag
  L.bytes = at + 1024 + 32;
  return L;
}

// The body of both dW kernels: k_cheb_dw_umma (fp16x3) and k_cheb_dw_f16_umma (F16: the single-pass layout above)
template <int XS, bool F16>
__device__ __forceinline__ void cheb_dw_body(const DwParams& p) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const DwSmem L = dw_smem(XS, p.max_h1, p.meta_stride, F16);
  constexpr int T_BYTES = dw_t_bytes(F16);
  unsigned char* ring = smem_raw;                      // [DW_NS] T blocks
  unsigned char* gblk = smem_raw + L.gblk;
  float* Xs = reinterpret_cast<float*>(smem_raw + L.xs);
  constexpr size_t xs_stage_floats = (size_t)TILE_M * FC;
  float* T1s = reinterpret_cast<float*>(smem_raw + L.t1s);
  const size_t t1_stage_floats = L.t1_stage;
  unsigned char* meta_s = smem_raw + L.meta;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + L.bars);
  uint64_t* b_t_full = bars;                 // [DW_NS]
  uint64_t* b_t_empty = b_t_full + DW_NS;    // [DW_NS]
  uint64_t* b_x_full = b_t_empty + DW_NS;    // [XS]
  uint64_t* b_x_empty = b_x_full + XS;       // [XS]
  uint64_t* b_m_full = b_x_empty + XS;       // [2]
  uint64_t* b_m_empty = b_m_full + 2;        // [2]
  uint64_t* b_g_full = b_m_empty + 2;        // [1]
  uint64_t* b_g_empty = b_g_full + 1;        // [1]
  uint32_t* flags = reinterpret_cast<uint32_t*>(smem_raw + L.flags);
  volatile int* abort_flag = reinterpret_cast<volatile int*>(flags + 1);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int n_chunk = 1;  // one feature chunk per launch: the MMA warpgroup holds its three accumulators
  const int my_tiles = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (tid == 0) {
    for (int s = 0; s < DW_NS; ++s) {
      mbar_init(smem_u32(b_t_full + s), W_PROD);
      mbar_init(smem_u32(b_t_empty + s), 4);  // one arrival per warp of the MMA warpgroup
    }
    for (int s = 0; s < XS; ++s) {
      mbar_init(smem_u32(b_x_full + s), N_XLOAD * 32 + 1);  // the loader threads' cp.async arrivals + one expect_tx / plain arrival
      mbar_init(smem_u32(b_x_empty + s), 1);
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(smem_u32(b_m_full + s), 1);
      mbar_init(smem_u32(b_m_empty + s), 1);
    }
    mbar_init(smem_u32(b_g_full), W_PROD);
    mbar_init(smem_u32(b_g_empty), 4);
    *abort_flag = (smem_u32(ring) & 1023u) ? 1 : 0;
    if (*abort_flag) mbar_timeout(abort_flag, p.status, 100);
    fence_barrier_init();
  }
  const float a_scale = p.a_scale ? *p.a_scale : 1.f;
  __syncthreads();

  if (warp >= W_XLOAD && warp < W_XLOAD + N_XLOAD) {
    // ------------------------------------------------------------ row loaders + tile metadata (as in the forward)
    const int lt = tid - W_XLOAD * 32;
    const int q = lt & 7, rg = lt >> 3;
    auto fetch_meta = [&](int it2) {
      const int pat = (blockIdx.x + it2 * gridDim.x) % p.P;
      const int m2 = it2 & 1;
      mbar_wait_relaxed(smem_u32(b_m_empty + m2), ((it2 >> 1) & 1) ^ 1, abort_flag, p.status, 21);
      const int mbytes = p.meta_bytes[pat];
      mbar_arrive_expect_tx(smem_u32(b_m_full + m2), mbytes);
      bulk_g2s(smem_u32(meta_s + (size_t)m2 * p.meta_stride), p.meta + (size_t)pat * p.meta_stride, mbytes,
               smem_u32(b_m_full + m2));
    };
    if (lt == 0 && my_tiles > 0) fetch_meta(0);
    uint32_t g = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int tile = blockIdx.x + it * gridDim.x;
      const int b = tile / p.P;
      const int m = it & 1;
      mbar_wait_relaxed(smem_u32(b_m_full + m), (it >> 1) & 1, abort_flag, p.status, 22);
      const unsigned char* mb = meta_s + (size_t)m * p.meta_stride;
      const TileHeader* hdr = reinterpret_cast<const TileHeader*>(mb);
      const int h1 = hdr->h1;
      const int* halo = reinterpret_cast<const int*>(mb + hdr->off_halo);
      const long long mesh_row0 = (long long)b * p.V;
      if (it + 1 < my_tiles) {
        // the producers read the NEXT tile's plain-side rows straight from global memory at the start of that tile:
        // pull them into L2 now (consecutive tiles only; index-list tiles would need the next blob first)
        const int tile2 = blockIdx.x + (it + 1) * gridDim.x;
        const long long r2 = (long long)(tile2 / p.P) * p.V + (long long)(tile2 % p.P) * TILE_M;
        const int lpr = (p.m_cols * 4 + 127) >> 7;  // 128-byte lines per row of this launch's channel slice
        for (int j = lt; j < TILE_M * lpr; j += N_XLOAD * 32) {
          const long long rr = r2 + j / lpr;
          if (rr < (long long)(tile2 / p.P + 1) * p.V)
            prefetch_l2(p.g + (p.g_unpool ? (rr >> 1) : rr) * p.fout_total + p.m_off + (j % lpr) * 32);
        }
      }
      for (int c = 0; c < n_chunk; ++c, ++g) {
        const int xs = g % XS;
        mbar_wait_relaxed(smem_u32(b_x_empty + xs), ((g / XS) & 1) ^ 1, abort_flag, p.status, 23);
        const uint32_t dst0 = smem_u32(Xs + xs * xs_stage_floats) + q * 16;
        const float* src0 = p.x + (p.chunk0 + c) * FC + q * 4;
        const uint32_t xbar = smem_u32(b_x_full + xs);
        if (lt == 0) {
          if (p.tma) {  // own rows of x and t1: one TMA box each, landing asynchronously
            const int own0 = tile * TILE_M;  // V is a multiple of 128: tiles never straddle meshes
            mbar_arrive_expect_tx(xbar, 2 * TILE_M * 128);
            tma_load_2d(smem_u32(Xs + xs * xs_stage_floats), &p.tm_x, (p.chunk0 + c) * FC, own0, xbar);
            tma_load_2d(smem_u32(T1s + xs * t1_stage_floats), &p.tm_t1, (p.chunk0 + c) * FC, own0, xbar);
          } else {
            mbar_arrive(xbar);
          }
        }
        if (!p.tma)  // the tile's own rows of x ...
        for (int i = rg; i < TILE_M; i += 8) {
          const int v = halo[i];
          if (v >= 0) {
            long long r = mesh_row0 + v;
            if (p.in_unpool) r >>= 1;
            cp_async16(dst0 + i * 128, src0 + r * p.fin);
          } else {
            sts_f4(dst0 + i * 128, make_float4(0.f, 0.f, 0.f, 0.f));
          }
        }
        {  // ... plus the T1 rows of the tile and its 1-hop halo
          const uint32_t dst1 = smem_u32(T1s + xs * t1_stage_floats) + q * 16;
          const float* src1 = p.t1 + (p.chunk0 + c) * FC + q * 4;
          for (int i = (p.tma ? TILE_M : 0) + rg; i < h1; i += 8) {  // (TMA: only the halo rows are left)
            const int v = halo[i];
            if (v >= 0)
              cp_async16(dst1 + i * 128, src1 + (mesh_row0 + v) * p.fin);
            else
              sts_f4(dst1 + i * 128, make_float4(0.f, 0.f, 0.f, 0.f));
          }
        }
        cp_async_arrive_noinc(xbar);
        if (c == 0 && lt == 0 && it + 1 < my_tiles) fetch_meta(it + 1);
      }
    }
  } else if (warp >= W_EPI0) {
    // ------------------------------------------------------------ MMA warpgroup: wgmma across all tiles, then atomicAdd
    // Accumulator u = k of the launch's one feature chunk: D[channel][feature] (M = 64 plain-side channels, N = 32
    // features), the hi and lo halves of the T block folded into the same columns: g_hi T_hi + g_lo T_hi + g_hi T_lo
    // per 16-row K step (the lo half is addressed by starting the MN-major descriptor 64 bytes into the swizzle row).
    const int wq = warp - W_EPI0;
    float acc[3][16];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[k][j] = 0.f;
    uint32_t ucnt = 0;
    const uint32_t g_hi = smem_u32(gblk), g_lo = g_hi + 2 * A_BLOCK_BYTES;
    const uint64_t dh = make_desc_sw128_mn(g_hi, A_BLOCK_BYTES), dl = make_desc_sw128_mn(g_lo, A_BLOCK_BYTES);
    for (int it = 0; it < my_tiles; ++it) {
      mbar_wait(smem_u32(b_g_full), it & 1, abort_flag, p.status, 24);
#pragma unroll
      for (int k = 0; k < 3; ++k, ++ucnt) {
        const int s = ucnt % DW_NS;
        mbar_wait(smem_u32(b_t_full + s), (ucnt / DW_NS) & 1, abort_flag, p.status, 25);
        if constexpr (F16) {
          const uint64_t dt = make_desc_sw64_mn(smem_u32(ring + s * T_BYTES));
          wg_fence();
#pragma unroll
          for (int ks = 0; ks < 8; ++ks)  // 16 mesh rows: 2048 bytes of g (+128), 1024 bytes of T (+64)
            wgmma_m64n32(acc[k], dh + ks * 128, dt + ks * 64);
        } else {
          const uint64_t dt = make_desc_sw128_mn(smem_u32(ring + s * A_BLOCK_BYTES), A_BLOCK_BYTES);
          wg_fence();
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) {  // 16 mesh rows per K step = 2048 bytes = +128 in the address field
            wgmma_m64n32(acc[k], dh + ks * 128, dt + ks * 128);      // g_hi T_hi
            wgmma_m64n32(acc[k], dl + ks * 128, dt + ks * 128);      // g_lo T_hi
            wgmma_m64n32(acc[k], dh + ks * 128, dt + ks * 128 + 4);  // g_hi T_lo (+64 B)
          }
        }
        wg_commit();
        wg_wait0();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(b_t_empty + s));
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(b_g_empty));  // the dz blocks may be overwritten
    }
    const float inv = 1.f / a_scale;
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const int o_local = 16 * wq + (lane >> 2) + 8 * ((i >> 1) & 1);  // plain-side channel inside the slice
        const int f = p.chunk0 * FC + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);  // channel of the gathered side
        if (o_local < p.m_cols && my_tiles > 0) {
          const float v = acc[k][i] * inv;
          if (p.swap)  // accumulator row = input feature (plain side), column = output channel
            atomicAdd(p.dw + (size_t)f * 3 * p.fout_total + (size_t)(p.m_off + o_local) * 3 + k, v);
          else
            atomicAdd(p.dw + (size_t)(p.m_off + o_local) * 3 * p.fin + f * 3 + k, v);
        }
      }
  } else if (warp < W_PROD) {
    // ------------------------------------------------------------ producers
    const int q = tid & 7, rg = tid >> 3;
    const uint32_t t1s_a = smem_u32(T1s), ring_a = smem_u32(ring), g_a = smem_u32(gblk);
    uint32_t ucnt = 0, gcnt = 0;
    uint32_t row0 = 0, row1 = 0, r0e = 0, r1e = 0, ent_a = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int tile = blockIdx.x + it * gridDim.x;
      const int b = tile / p.P, pat = tile - b * p.P;
      const int m = it & 1;
      // The plain-side tile goes global -> registers -> fp16 blocks.  Its loads are issued FIRST, so that their
      // latency overlaps the waits below (metadata, and above all g_empty: the previous tile's MMAs still read the
      // single-buffered plain blocks) instead of following them.
      constexpr int NJ = F16 ? 2 : 4;  // 32-channel pieces per row (F16: the 64 channels of the launch's slice only)
      float4 pv[2][NJ];
      {
        const int n_rows = min(TILE_M, p.V - pat * TILE_M);
        const long long r_base = (long long)b * p.V + (long long)pat * TILE_M;
#pragma unroll
        for (int ps = 0; ps < 2; ++ps) {
          const int i = ps * 64 + rg;
#pragma unroll
          for (int jj = 0; jj < NJ; ++jj) {
            const int col = q * 4 + 32 * (jj ^ (rg & 1));
            pv[ps][jj] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < n_rows && col < p.m_cols) {
              const long long rr = p.g_unpool ? ((r_base + i) >> 1) : (r_base + i);
              pv[ps][jj] = __ldg(reinterpret_cast<const float4*>(p.g + rr * p.fout_total + p.m_off + col));
            }
          }
        }
      }
      mbar_wait(smem_u32(b_m_full + m), (it >> 1) & 1, abort_flag, p.status, 27);
      {
        const unsigned char* mb = meta_s + (size_t)m * p.meta_stride;
        const TileHeader* hdr = reinterpret_cast<const TileHeader*>(mb);
        const uint32_t mb_a = smem_u32(mb);
        const uint32_t rp_a = mb_a + hdr->off_rp, ord2_a = mb_a + hdr->off_ord2;
        ent_a = mb_a + hdr->off_ent;
        row0 =lds_u16(ord2_a + 2 * rg);
        row1 = lds_u16(ord2_a + 2 * (64 + rg));
        r0e = lds_u16(rp_a + 2 * row0) | (lds_u16(rp_a + 2 * row0 + 2) << 16);
        r1e = lds_u16(rp_a + 2 * row1) | (lds_u16(rp_a + 2 * row1 + 2) << 16);
      }
      // plain-side tile (dz, or the layer input in swapped mode) -> (hi, lo) fp16 blocks, MN-major [row][channel]
      mbar_wait(smem_u32(b_g_empty), (it & 1) ^ 1, abort_flag, p.status, 28);
      {
#pragma unroll
        for (int ps = 0; ps < 2; ++ps) {
          const int i = ps * 64 + rg;
#pragma unroll
          for (int jj = 0; jj < NJ; ++jj) {
            // odd row groups take the 32-channel pieces in the order 1,0,3,2: the two rows of a half-warp then store
            // into different 64-byte bank halves (their swizzle bits agree: consecutive rows)
            const int col = q * 4 + 32 * (jj ^ (rg & 1));  // channel inside this launch's slice (< m_cols <= 64)
            float4 v = pv[ps][jj];
            if (!p.swap) {  // input role: this side is the gradient
              v.x *= a_scale; v.y *= a_scale; v.z *= a_scale; v.w *= a_scale;
            }
            if constexpr (F16) {  // the hi block alone
              sts_u2(g_a + sw128_off(i, col >> 3) + ((col >> 2) & 1) * 8, half4(v));
              continue;
            }
            uint2 hi, lo;
            split4(v, hi, lo);
            const uint32_t off = (uint32_t)(col >> 6) * A_BLOCK_BYTES + sw128_off(i, (col & 63) >> 3) + ((col >> 2) & 1) * 8;
            sts_u2(g_a + off, hi);  // (rows i = ps*64 + rg: 8 lanes x 8 B = 64 B per row and store, hi and lo blocks apart)
            sts_u2(g_a + 2 * A_BLOCK_BYTES + off, lo);
          }
        }
        fence_async_proxy();
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(smem_u32(b_g_full));
      }
      for (int c = 0; c < n_chunk; ++c, ++gcnt) {
        const int xs = gcnt % XS;
        mbar_wait(smem_u32(b_x_full + xs), (gcnt / XS) & 1, abort_flag, p.status, 29);
        const uint32_t xs_q = smem_u32(Xs + xs * xs_stage_floats) + q * 16;
        const uint32_t t1s_q = t1s_a + (uint32_t)(xs * t1_stage_floats * 4) + q * 16;
        float4 tv[3][2];
        {
          const float4 g0 = gather_row4(ent_a, r0e & 0xFFFFu, r0e >> 16, t1s_q);
          const float4 g1 = gather_row4(ent_a, r1e & 0xFFFFu, r1e >> 16, t1s_q);
          tv[0][0] = lds_f4(xs_q + row0 * 128);
          tv[0][1] = lds_f4(xs_q + row1 * 128);
          tv[1][0] = lds_f4(t1s_q + row0 * 128);
          tv[1][1] = lds_f4(t1s_q + row1 * 128);
          const float4 a = tv[0][0], c2 = tv[0][1];
          tv[2][0] = cheb_t2(g0, a);
          tv[2][1] = cheb_t2(g1, c2);
          if (p.swap) {  // the gathered side is the gradient: into fp16's range before the split
#pragma unroll
            for (int k = 0; k < 3; ++k)
#pragma unroll
              for (int ps = 0; ps < 2; ++ps) {
                tv[k][ps].x *= a_scale; tv[k][ps].y *= a_scale; tv[k][ps].z *= a_scale; tv[k][ps].w *= a_scale;
              }
          }
        }
        const uint32_t u0 = ucnt;
#pragma unroll
        for (int k = 0; k < 3; ++k, ++ucnt) {
          const int s = ucnt % DW_NS;
          mbar_wait(smem_u32(b_t_empty + s), ((ucnt / DW_NS) & 1) ^ 1, abort_flag, p.status, 30);
          const uint32_t blk = ring_a + s * T_BYTES + (q & 1) * 8;
#pragma unroll
          for (int ps = 0; ps < 2; ++ps) {
            const uint32_t i = ps ? row1 : row0;
            if constexpr (F16) {  // one 8-byte piece per row, as in the conv's F16 producers
              sts_u2(blk + sw64_off(i, q >> 1), half4(tv[k][ps]));
              continue;
            }
            uint2 hi, lo;
            split4(tv[k][ps], hi, lo);
            const uint32_t a_hi = blk + sw128_off(i, q >> 1), a_lo = blk + sw128_off(i, 4 + (q >> 1));
            const bool odd = (rg & 1) != 0;  // see emit() of the conv kernel
            sts_u2(odd ? a_lo : a_hi, odd ? lo : hi);
            sts_u2(odd ? a_hi : a_lo, odd ? hi : lo);
          }
        }
        fence_async_proxy();
        __syncwarp();
        if ((tid & 31) == 0) {
#pragma unroll
          for (int k = 0; k < 3; ++k) mbar_arrive(smem_u32(b_t_full + (u0 + k) % DW_NS));
        }
        producer_barrier<W_PROD * 32>();
        if (tid == 0) {
          mbar_arrive(smem_u32(b_x_empty + xs));
          if (c == n_chunk - 1) mbar_arrive(smem_u32(b_m_empty + m));
        }
      }
    }
  }
}

template <int XS>
__global__ void __launch_bounds__(NUM_THREADS2, 1) k_cheb_dw_umma(const __grid_constant__ DwParams p) {
  cheb_dw_body<XS, false>(p);
}
// the single-pass fp16 weight gradient (P2M_PREC_FP16_MIXED_TC): one wgmma per K step
template <int XS>
__global__ void __launch_bounds__(NUM_THREADS2, 1) k_cheb_dw_f16_umma(const __grid_constant__ DwParams p) {
  cheb_dw_body<XS, true>(p);
}

// =====================================================================================
// k_cheb_t1 — T1 = L~ X for every row, written once to HBM (fp32, logical rows).  With it the conv and dW kernels
// only need the tile's own X rows and the T1 rows of its 1-hop halo; no tile recomputes T1 on its halo rows.
// Simple kernel: one CTA (512 threads, two per SM) per 128-row tile; the 1-hop halo of X is staged chunk by chunk
// through a 4-deep cp.async ring (one barrier per chunk), the gather runs out of shared memory.
// =====================================================================================
struct T1Params {
  const float* x;
  int in_unpool;
  int V, P, fin;
  const unsigned char* meta;
  const int* meta_bytes;
  int meta_stride, max_h1;
  float* t1;
};

// k_cheb_t1<T1_STAGES>: the tile's metadata blob at offset 0, then [T1_STAGES][max_h1][32] fp32 X rows of the tile and
// its 1-hop halo, and 16 bytes of slack
struct T1Smem {
  size_t xs, stage, bytes;
};
__host__ __device__ __forceinline__ T1Smem t1_smem(int T1_STAGES, int max_h1, int meta_stride) {
  const size_t stage = (size_t)max_h1 * FC;
  return {(size_t)meta_stride, stage, meta_stride + T1_STAGES * stage * 4 + 16};
}

// T1_STAGES = cp.async ring depth (chunks in flight per CTA): 4 when two CTAs of that size fit an SM, else 3 or 2
template <int T1_STAGES>
__global__ void __launch_bounds__(512, 2) k_cheb_t1(const T1Params p) {
  extern __shared__ __align__(16) unsigned char smem_t1[];
  const T1Smem L = t1_smem(T1_STAGES, p.max_h1, p.meta_stride);
  unsigned char* meta_s = smem_t1;
  float* Xs = reinterpret_cast<float*>(smem_t1 + L.xs);
  const size_t stage_floats = L.stage;
  const int tid = threadIdx.x, q = tid & 7, rg = tid >> 3;
  const int tile = blockIdx.x;
  const int b = tile / p.P, pat = tile - b * p.P;
  const long long mesh_row0 = (long long)b * p.V;
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.meta + (size_t)pat * p.meta_stride);
    uint4* dst = reinterpret_cast<uint4*>(meta_s);
    const int n16 = p.meta_bytes[pat] >> 4;
    for (int i = tid; i < n16; i += 512) dst[i] = src[i];
  }
  __syncthreads();
  const TileHeader* hdr = reinterpret_cast<const TileHeader*>(meta_s);
  const int h1 = hdr->h1;
  const int* halo = reinterpret_cast<const int*>(meta_s + hdr->off_halo);
  const uint32_t mb_a = smem_u32(meta_s);
  const uint32_t rp_a = mb_a + hdr->off_rp, ent_a = mb_a + hdr->off_ent, ord2_a = mb_a + hdr->off_ord2;
  const int n_chunk = p.fin / FC;
  // source rows of the staged slots this thread copies (same for every chunk): slots rg, rg + 64, ...
  long long srow[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int i = rg + 64 * u;
    const int v = (i < h1) ? halo[i] : -2;
    long long r = mesh_row0 + v;
    if (p.in_unpool) r >>= 1;
    srow[u] = (v >= 0) ? r * p.fin : (long long)v;  // -1: empty slot (zero-filled), -2: beyond the halo
  }
  auto stage = [&](int c) {
    if (c < n_chunk) {
      const uint32_t dst0 = smem_u32(Xs + (c % T1_STAGES) * stage_floats) + q * 16;
      const float* src0 = p.x + c * FC + q * 4;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = rg + 64 * u;
        if (srow[u] >= 0)
          cp_async16(dst0 + i * 128, src0 + srow[u]);
        else if (srow[u] == -1)
          sts_f4(dst0 + i * 128, make_float4(0.f, 0.f, 0.f, 0.f));
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");  // (possibly empty: keeps the group count uniform)
  };
  // rows this thread produces, taken in length-sorted order: the four rows of a warp then have similar lengths
  int vtx[2];
  uint32_t re[2];
#pragma unroll
  for (int ps = 0; ps < 2; ++ps) {
    const int i = lds_u16(ord2_a + 2 * (ps * 64 + rg));
    vtx[ps] = halo[i];
    re[ps] = lds_u16(rp_a + 2 * i) | (lds_u16(rp_a + 2 * i + 2) << 16);
  }
#pragma unroll
  for (int c = 0; c < T1_STAGES - 1; ++c) stage(c);
  for (int c = 0; c < n_chunk; ++c) {
    asm volatile("cp.async.wait_group %0;" ::"n"(T1_STAGES - 2) : "memory");  // chunk c has landed (this thread's part)
    __syncthreads();  // ... and everybody's; also: everybody is done with chunk c - 1, whose stage is refilled next
    stage(c + T1_STAGES - 1);
    const uint32_t xs_q = smem_u32(Xs + (c % T1_STAGES) * stage_floats) + q * 16;
#pragma unroll
    for (int ps = 0; ps < 2; ++ps) {
      if (vtx[ps] >= 0) {
        const float4 acc = gather_row4(ent_a, re[ps] & 0xFFFFu, re[ps] >> 16, xs_q);
        *reinterpret_cast<float4*>(p.t1 + (mesh_row0 + vtx[ps]) * p.fin + c * FC + q * 4) = acc;
      }
    }
  }
}

// What k_pack turns into an operand image: K-blocks of `rows` rows x 32 k as fp16 [hi 32 | lo 32] per 128-byte row, in
// the exact shared-memory image (128B-swizzled), so a kernel fetches a block with a single cp.async.bulk.  Block
// b = (t * n_chunk + chunk) * orders + order holds rows n = t * rows + [0, rows) and k = 32 chunk + [0, 32):
// p[n ld_row + k ld_k + order] * scale, zero for n >= n_real or k >= k_real (never read there); `combined`: the isolated
// rows' combined weights (p[a] + c p[a + 1] + (2c^2 - 1) p[a + 2]) * scale at a = n ld_row + k ld_k.  With dscale the
// scale is scale * *dscale.  hi_only: the single-pass fp16 image, 64-byte rows of the 32 fp16 values (no lo part),
// 64B-swizzled.
struct PackSrc {
  const float* p;
  long long ld_row, ld_k;
  int rows, n_chunk, orders, n_real;
  float scale;  // W_SCALE for weights, 1 for range-normalised activations (dscale)
  int combined;
  float c;
  int k_real = INT_MAX;
  const float* dscale = nullptr;  // device scalar: a power of two found from the operand's largest magnitude
  int hi_only = 0;
};
__global__ void __launch_bounds__(256) k_pack(const PackSrc s, long long total, unsigned char* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one 16-byte chunk each
  if (idx >= total) return;
  const int cl2 = s.hi_only ? 2 : 3;  // log2 of the 16-byte chunks per row
  const int j = (int)(idx & ((1 << cl2) - 1));
  const int row = (int)((idx >> cl2) % s.rows);
  const long long blk = (idx >> cl2) / s.rows;
  const int per_tile = s.n_chunk * s.orders;
  const long long n = blk / per_tile * s.rows + row;
  const int u = (int)(blk % per_tile);
  const int k0 = (u / s.orders) * FC + (j & 3) * 8;
  const float* src = s.p + n * s.ld_row + (long long)k0 * s.ld_k + u % s.orders;
  const float c = s.c, c2 = 2.f * c * c - 1.f;
  const float scale = s.dscale ? s.scale * *s.dscale : s.scale;
  __align__(16) __half h[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float* wr = src + e * s.ld_k;
    float w = 0.f;
    if (n < s.n_real && k0 + e < s.k_real) w = s.combined ? (wr[0] + c * wr[1] + c2 * wr[2]) * scale : wr[0] * scale;
    const __half hi = __float2half_rn(w);
    h[e] = (j < 4) ? hi : __float2half_rn(w - __half2float(hi));
  }
  const size_t at = s.hi_only ? blk * s.rows * 64 + sw64_off(row, j) : blk * s.rows * 128 + sw128_off(row, j);
  *reinterpret_cast<uint4*>(out + at) = *reinterpret_cast<const uint4*>(h);
}
int launch_pack(const PackSrc& src, long long n_blocks, void* out, cudaStream_t s) {
  const long long total = n_blocks * src.rows * (src.hi_only ? 4 : 8);
  k_pack<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(src, total, static_cast<unsigned char*>(out));
  P2M_LAUNCH_OK();
  return P2M_OK;
}

constexpr size_t SMEM_LIMIT = 227 * 1024;
constexpr int CONV_N = 64;  // output columns per CTA of the 128-row conv configuration (one column slice)
constexpr int WIDE_N = 128; // ... and of the 64-row configuration (convs with Fout % 128 == 0)
constexpr int PAIR_N = 256; // ... and of its 64 x 256 mode (both MMA warpgroups on one tile: Fout == 256)
inline int conv_n(int fout) { return fout % WIDE_N == 0 ? WIDE_N : CONV_N; }
// the tile metadata a launch with N output columns per CTA runs on: the level's consecutive tiles or the tile family the
// caller selected, 128-row blobs for N = 64 and 64-row blobs for N = 128
const TileBlobs& conv_tiles(int N, const DevLevel& g, const TileSet* tiles) {
  if (tiles != nullptr) return N == WIDE_N ? tiles->m64 : *tiles;
  return N == WIDE_N ? g.meta64 : g.meta128;
}
// A/B ring depth and X staging depth of a conv launch with NC output columns per CTA: the deepest that fit, the ring
// first (NC = 128: 6 slots = two chunks, the producers run a chunk ahead of the MMAs, or 3 = one chunk; NC = 64 and
// NC = 256, whose six 40 KB slots never fit: 3), then 2 X stages (prefetch the next chunk's rows during the current
// chunk) or 1.  {0, 0}: does not fit.
struct ConvCfg {
  int ns, xs;
};
ConvCfg conv_cfg(int NC, const TileBlobs& t, bool t1_given, bool f16) {
  for (int ns = NC == WIDE_N ? 6 : 3; ns >= 3; ns -= 3)
    for (int xs = 2; xs >= 1; --xs)
      if (conv_smem(NC, ns, xs, t1_given, t.max_h1, t.stride, f16).bytes <= SMEM_LIMIT) return {ns, xs};
  return {0, 0};
}
// A tile family the conv can run on with N accumulator columns per MMA warpgroup (64: its 128-row tiles, 128: its
// 64-row tiles): the T1-given conv and the plain GEMM both fit one ring of 3 and one X stage at fp16x3, whose slots
// are twice the single-pass fp16 ones, and k_cheb_t1 stages its rows (at most 256)
bool conv_family_fits(const TileBlobs& t, int N) {
  return t.n_pattern > 0 && t.max_h1 <= 256 && conv_smem(N, 3, 1, 1, t.max_h1, t.stride).bytes <= SMEM_LIMIT &&
         conv_smem(N, 3, 1, 0, t.max_h1, t.stride).bytes <= SMEM_LIMIT;
}
// Output columns per CTA of a conv Fin -> Fout on tiles t.  The 64 x 256 mode builds each A block once for all 256
// columns, but its two warpgroups finish a tile together, so each tile's epilogue runs behind its main loop instead of
// under the other warpgroup's: that pays where the main loop is long, the T1-given 256 -> 256 conv (24 K-blocks per
// tile: 13-21 % faster layers), and not at 12 (128 -> 256: 8 % slower; H100 SXM, README).  It is taken there when its
// ring of three slots fits; every other conv with Fout % 128 == 0 runs as 128-column slices.
int conv_cols(int fin, int fout, const TileBlobs& t, bool t1_given, bool f16) {
  const bool pair = fout == PAIR_N && fin == PAIR_N && t1_given && conv_cfg(PAIR_N, t, true, f16).ns > 0;
  return pair ? PAIR_N : conv_n(fout);
}

// cuTensorMapEncodeTiled through the runtime's driver entry point lookup (no link-time dependency on libcuda)
typedef CUresult (*TmapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
TmapEncodeFn tmap_encoder() {
  static TmapEncodeFn fn = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    return reinterpret_cast<TmapEncodeFn>(f);
  }();
  return fn;
}
// [rows, fin] fp32 row-major matrix, box = 32 features x box_rows rows, dense (unswizzled) 128-byte rows in shared memory
bool make_row_tmap(CUtensorMap* tm, const float* base, long long rows, int fin, int box_rows) {
  TmapEncodeFn enc = tmap_encoder();
  if (enc == nullptr || (reinterpret_cast<uintptr_t>(base) & 15u) != 0) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)fin, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)fin * 4};
  const cuuint32_t box[2] = {(cuuint32_t)FC, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// The conv kernel with NC output columns per CTA: k_cheb_conv_umma (64) or k_cheb_conv_wide (128, 256); F16: their
// single-pass fp16 instantiations
template <int NC, int NS, int XS, int MODE, bool F16 = false>
constexpr auto conv_kernel() {
  if constexpr (F16 && NC != CONV_N) return k_cheb_conv_f16_wide<NC, NS, XS, MODE>;
  else if constexpr (F16) return k_cheb_conv_f16_umma<NC, NS, XS, MODE>;
  else if constexpr (NC != CONV_N) return k_cheb_conv_wide<NC, NS, XS, MODE>;
  else return k_cheb_conv_umma<NC, NS, XS, MODE>;
}
// A conv kernel's setmaxnreg split is balanced for a launch allocation of ConvRoles<N>::regs_launch registers per
// thread (80 for k_cheb_conv_umma, 96 for k_cheb_conv_wide): a build that ends up with another count would leave the
// epilogue's setmaxnreg.inc spinning on an empty pool.
template <int NC, int NS, int XS, int MODE, bool F16 = false>
int check_launch_regs() {
  constexpr int N = NC == CONV_N ? CONV_N : WIDE_N;
  static int state = 0;  // per instantiation; racing first calls all compute the same value
  if (state == 0) {
    cudaFuncAttributes fa;
    P2M_CUDA_OK(cudaFuncGetAttributes(&fa, conv_kernel<NC, NS, XS, MODE, F16>()));
    state = (fa.numRegs == ConvRoles<N>::regs_launch) ? 1 : -1;
  }
  if (state < 0) {
    set_error(N == WIDE_N
                  ? "k_cheb_conv_wide was compiled with a register count other than the one its setmaxnreg split assumes"
                  : "k_cheb_conv_umma was compiled with a register count other than the one its setmaxnreg split assumes");
    return P2M_ERR_CUDA;
  }
  return P2M_OK;
}

// MODE 0 (plain GEMM, a.plain) or MODE 1 (T1 given); NC output columns per CTA; F16 the single-pass fp16 precision
// (a.f16)
template <int NC, int NS, int XS, int MODE, bool F16>
int launch_cfg(const UmmaConvArgs& a, int* status, const float* zero_row, int sm_count, cudaStream_t s) {
  constexpr int N = NC == CONV_N ? CONV_N : WIDE_N;
  constexpr int TM = tile_rows<N>();
  const DevLevel& g = *a.g;
  const TileBlobs& t = conv_tiles(N, g, a.tiles);
  const size_t smem = conv_smem(NC, NS, XS, MODE, t.max_h1, t.stride, F16).bytes;
  auto kern = conv_kernel<NC, NS, XS, MODE, F16>();
  P2M_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  P2M_TRY((check_launch_regs<NC, NS, XS, MODE, F16>()));
  KParams p;
  p.x = a.x;
  p.in_unpool = a.in_unpool;
  p.V = g.V;
  p.P = t.n_pattern;
  p.fin = a.fin;
  p.meta = t.meta;
  p.meta_bytes = t.bytes;
  p.meta_stride = t.stride;
  p.max_h1 = t.max_h1;
  p.own_table = a.tiles != nullptr ? 1 : 0;
  p.n_tiles = a.batch * p.P;
  p.wpack = static_cast<const unsigned char*>(a.wpack);
  p.apack = nullptr;
  // the weight image holds K-blocks of fout rows x 128 (F16: 64) bytes; column slice y starts y * NC rows into each
  p.wslice_bytes = (long long)NC * op_row_bytes(F16);
  p.wblock_stride = (long long)a.fout * op_row_bytes(F16);
  p.zero_row = zero_row;
  p.ep = to_dev(a.ep);
  p.res_identity = (a.ep.res != nullptr && a.ep.res_F == a.fout) ? 1 : 0;
  p.y = a.y;
  p.t1 = a.t1;
  p.a_scale = a.a_scale;
  p.b_scale = nullptr;
  p.ldy = a.ldy > 0 ? a.ldy : a.fout;
  p.y_col0 = a.y_col0;
  p.status = status;
  p.trace = a.trace;
  p.head_wt = a.fout == 64 ? a.head_wt : nullptr;
  p.head_z = a.fout == 64 ? a.head_z : nullptr;
  if (N == WIDE_N) {
    // the epilogue moves whole 512-byte output rows (and identity-residual rows) by cp.async.bulk, which needs 16-byte
    // aligned addresses (a warpgroup's first column, a multiple of 128, keeps that)
    const bool y_ok = (reinterpret_cast<uintptr_t>(p.y) & 15u) == 0 && (p.ldy * 4) % 16 == 0 && (p.y_col0 * 4) % 16 == 0;
    const bool res_ok = !p.res_identity || ((reinterpret_cast<uintptr_t>(p.ep.res) & 15u) == 0 && (p.ep.res_F * 4) % 16 == 0);
    if (!y_ok || !res_ok) {
      set_error("umma_conv: the 128-column epilogue needs 16-byte aligned output and identity-residual rows");
      return P2M_ERR_INVALID;
    }
  }
  p.tma = 0;
  std::memset(&p.tm_x, 0, sizeof(p.tm_x));
  std::memset(&p.tm_t1, 0, sizeof(p.tm_t1));
  if (a.tiles == nullptr && g.V % TILE_M == 0) {
    const long long rows = (long long)a.batch * g.V;
    bool ok = make_row_tmap(&p.tm_x, a.x, a.in_unpool ? rows / 2 : rows, a.fin, a.in_unpool ? TM / 2 : TM);
    if (ok && a.t1 != nullptr) ok = make_row_tmap(&p.tm_t1, a.t1, rows, a.fin, TM);
    p.tma = ok ? 1 : 0;
  }
  const int n_slices = a.fout / NC;
  const dim3 grid(std::min(p.n_tiles, std::max(1, sm_count / n_slices)), n_slices);
  kern<<<grid, ConvRoles<N>::threads, smem, s>>>(p);
  log_tc_launch(TC_CONV, NC, NS, XS, MODE, F16, grid, p.n_tiles);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// The instantiations launch_n can select.  Every family a conv runs on fits one ring of 3 fp16x3 slots with one stage
// (umma_conv_supported, build_umma_level_meta), and six fp16 slots take no more (6 (64 + 128) 64 B = 3 (64 + 128) 128 B;
// the barrier map's 48 B more fit the 64 B that conv_smem's fixed terms leave below any multiple of 128): at fp16 the
// 64 x 128 ring is always 6.  The single-pass fp16 plain GEMM runs only on the isolated rows' tiles (their own rows,
// one CSR entry each: blobs of at most 2176 B), where the deepest ring and both X stages fit.  The 64 x 256 mode is
// T1-given only (conv_cols).
template <int NC, int NS, int XS, int MODE, bool F16>
constexpr bool launchable() {
  if (MODE == 0 && (NC == PAIR_N || (F16 && (XS != 2 || NS != (NC == WIDE_N ? 6 : 3))))) return false;
  return !(F16 && NC == WIDE_N && NS != 6);
}
template <int NC, int NS, int XS, bool F16>
int launch_mode(const UmmaConvArgs& a, int* status, const float* zero_row, int sm_count, cudaStream_t s) {
  if (a.plain) {
    if constexpr (launchable<NC, NS, XS, 0, F16>()) return launch_cfg<NC, NS, XS, 0, F16>(a, status, zero_row, sm_count, s);
  } else {
    if constexpr (launchable<NC, NS, XS, 1, F16>()) return launch_cfg<NC, NS, XS, 1, F16>(a, status, zero_row, sm_count, s);
  }
  set_error("umma_conv: no kernel instantiation for this tile family's shared-memory configuration");
  return P2M_ERR_INVALID;
}

template <bool F16>
int launch_n(const UmmaConvArgs& a, int* status, const float* zero_row, int sm_count, cudaStream_t s) {
  const int N = conv_n(a.fout);
  const TileBlobs& t = conv_tiles(N, *a.g, a.tiles);
  const int NC = conv_cols(a.fin, a.fout, t, !a.plain, F16);
  const ConvCfg c = conv_cfg(NC, t, !a.plain, F16);
  if (c.ns == 0) {
    set_error("umma_conv: tile family does not fit shared memory");
    return P2M_ERR_INVALID;
  }
  if (NC == PAIR_N)
    return c.xs == 2 ? launch_mode<PAIR_N, 3, 2, F16>(a, status, zero_row, sm_count, s)
                     : launch_mode<PAIR_N, 3, 1, F16>(a, status, zero_row, sm_count, s);
  if (N == CONV_N)
    return c.xs == 2 ? launch_mode<CONV_N, 3, 2, F16>(a, status, zero_row, sm_count, s)
                     : launch_mode<CONV_N, 3, 1, F16>(a, status, zero_row, sm_count, s);
  if (c.ns == 6)
    return c.xs == 2 ? launch_mode<WIDE_N, 6, 2, F16>(a, status, zero_row, sm_count, s)
                     : launch_mode<WIDE_N, 6, 1, F16>(a, status, zero_row, sm_count, s);
  return c.xs == 2 ? launch_mode<WIDE_N, 3, 2, F16>(a, status, zero_row, sm_count, s)
                   : launch_mode<WIDE_N, 3, 1, F16>(a, status, zero_row, sm_count, s);
}

}  // namespace

// =====================================================================================
// host side
// =====================================================================================
namespace {
// The producers store a tile row's fp16 hi part into one 64-byte half of its 128-byte A-block row and the lo part
// into the other; which half is which follows the row's swizzle bit (row & 4).  A warp stores four rows per
// instruction (row groups 4w .. 4w+3 of the order below, odd groups lo first) and 64-bit shared stores are served per
// half-warp, i.e. per PAIR of rows (positions 0,1 and 2,3 of an aligned group of four): a pair is free of bank
// replays iff its two 64-byte pieces fall into different halves — with the odd group storing the other part first,
// iff both rows of the pair have the SAME half class.  Re-deal a length-sorted order accordingly: [c0 c0 c1 c1] per
// group, taken in sorted order (a group's rows still have similar lengths).  Pure re-ordering of which thread
// produces which row: results are unchanged.
// (The single-pass fp16 precision stores one 64-byte row per tile row, in the bank half of its parity: there a pair
// of equal parity costs one replay.  Dealing by parity as well cost the fp16x3 schedules about 0.6 % on an H100, so
// this order, which both precisions share, stays the fp16x3 one.)
void balance_store_halves(std::vector<unsigned short>* ord) {
  std::vector<unsigned short> q0, q1;
  for (unsigned short r : *ord) ((r & 4) ? q1 : q0).push_back(r);
  if (q0.size() != q1.size() || (q0.size() & 1)) return;
  size_t o = 0;
  for (size_t g = 0; g + 1 < q0.size(); g += 2) {
    (*ord)[o++] = q0[g];
    (*ord)[o++] = q0[g + 1];
    (*ord)[o++] = q1[g];
    (*ord)[o++] = q1[g + 1];
  }
}

// Blob of one tile whose tm (128 or 64) own rows are given by an index list (-1 = empty slot): own rows, their
// 1-hop halo, the CSR of the own rows with staged-row slots as columns, the own rows in length-sorted order.
bool make_indexed_blob(const std::vector<int>& own, int tm, const int* rowptr, const int* colidx, const float* val,
                       std::vector<int>* slot_of, std::vector<unsigned char>* blob, int* h1_out) {
  std::vector<int> halo(own);
  int n_rows = 0;
  for (int i = 0; i < tm; ++i)
    if (own[i] >= 0) {
      (*slot_of)[own[i]] = i;
      ++n_rows;
    }
  for (int i = 0; i < tm; ++i) {
    if (own[i] < 0) continue;
    for (int e = rowptr[own[i]]; e < rowptr[own[i] + 1]; ++e) {
      const int v = colidx[e];
      if ((*slot_of)[v] < 0) {
        (*slot_of)[v] = (int)halo.size();
        halo.push_back(v);
      }
    }
  }
  const int h1 = (int)halo.size();
  std::vector<unsigned short> rp(tm + 1, 0);
  std::vector<unsigned int> ent;
  for (int i = 0; i < tm; ++i) {
    if (own[i] >= 0)
      for (int e = rowptr[own[i]]; e < rowptr[own[i] + 1]; ++e) {
        unsigned int bits;
        std::memcpy(&bits, &val[e], 4);
        ent.push_back((unsigned int)(*slot_of)[colidx[e]] * 128u);
        ent.push_back(bits);
      }
    rp[i + 1] = (unsigned short)(ent.size() / 2);
  }
  for (int v : halo)
    if (v >= 0) (*slot_of)[v] = -1;
  const int nnz = (int)(ent.size() / 2);
  // at most 512 staged rows (no kernel stages more than 256) and 16-bit local-CSR offsets
  if (h1 > 512 || nnz > 65535) return false;
  std::vector<unsigned short> ord2(tm);
  for (int i = 0; i < tm; ++i) ord2[i] = (unsigned short)i;
  std::stable_sort(ord2.begin(), ord2.end(), [&](unsigned short a, unsigned short b2) {
    return (int)rp[a + 1] - (int)rp[a] > (int)rp[b2 + 1] - (int)rp[b2];
  });
  // 64-row tiles: 32 row groups, a thread's second row sits 32 positions on (128 rows: 64), so the half-warp pairs are
  // the same aligned positions (0,1), (2,3) of each group of four for both tile sizes
  balance_store_halves(&ord2);
  TileHeader t{};
  t.n_rows = n_rows;
  t.h1 = h1;
  t.nnz = nnz;
  int o1 = 64;
  t.off_halo = o1; o1 += up16(h1 * 4);
  t.off_rp = o1;   o1 += up16((tm + 1) * 2);
  t.off_ent = o1;  o1 += up16(nnz * 8);
  t.off_ord2 = o1; o1 += up16(tm * 2);
  t.bytes = o1;
  blob->assign(o1, 0);
  std::memcpy(blob->data(), &t, sizeof(t));
  std::memcpy(blob->data() + t.off_halo, halo.data(), (size_t)h1 * 4);
  std::memcpy(blob->data() + t.off_rp, rp.data(), (tm + 1) * 2);
  if (nnz) std::memcpy(blob->data() + t.off_ent, ent.data(), (size_t)nnz * 8);
  std::memcpy(blob->data() + t.off_ord2, ord2.data(), tm * 2);
  *h1_out = h1;
  return true;
}

// Tiles of tm consecutive entries of `rows` (ascending vertex ids), uploaded as one set of blobs.
int build_blobs(const std::vector<int>& rows, int tm, const int* rowptr, const int* colidx, const float* val, int V,
                TileBlobs* ts, std::vector<void*>* owned) {
  const int P = ((int)rows.size() + tm - 1) / tm;
  std::vector<std::vector<unsigned char>> blobs(P);
  std::vector<int> slot_of(V, -1);
  int stride = 0, max_h1 = 0;
  for (int pt = 0; pt < P; ++pt) {
    std::vector<int> own(tm, -1);
    for (int i = 0; i < tm && pt * tm + i < (int)rows.size(); ++i) own[i] = rows[pt * tm + i];
    int h1 = 0;
    if (!make_indexed_blob(own, tm, rowptr, colidx, val, &slot_of, &blobs[pt], &h1)) return P2M_ERR_INVALID;
    stride = std::max(stride, (int)blobs[pt].size());
    max_h1 = std::max(max_h1, h1);
  }
  stride = (stride + 127) & ~127;
  std::vector<unsigned char> all((size_t)P * stride, 0);
  std::vector<int> bytes(P);
  for (int pt = 0; pt < P; ++pt) {
    std::memcpy(all.data() + (size_t)pt * stride, blobs[pt].data(), blobs[pt].size());
    bytes[pt] = (int)blobs[pt].size();
  }
  unsigned char* d_meta = nullptr;
  int* d_bytes = nullptr;
  P2M_CUDA_OK(cudaMalloc(&d_meta, all.size()));
  owned->push_back(d_meta);
  P2M_CUDA_OK(cudaMalloc(&d_bytes, sizeof(int) * P));
  owned->push_back(d_bytes);
  P2M_CUDA_OK(cudaMemcpy(d_meta, all.data(), all.size(), cudaMemcpyHostToDevice));
  P2M_CUDA_OK(cudaMemcpy(d_bytes, bytes.data(), sizeof(int) * P, cudaMemcpyHostToDevice));
  ts->meta = d_meta;
  ts->bytes = d_bytes;
  ts->stride = stride;
  ts->n_pattern = P;
  ts->max_h1 = max_h1;
  return P2M_OK;
}
}  // namespace

int build_tileset(const std::vector<int>& rows, const int* rowptr, const int* colidx, const float* val, int V,
                  TileSet* ts, std::vector<void*>* owned) {
  P2M_TRY(build_blobs(rows, TILE_M, rowptr, colidx, val, V, ts, owned));
  return build_blobs(rows, 64, rowptr, colidx, val, V, &ts->m64, owned);
}

int build_umma_level_meta(const int* rowptr, const int* colidx, const float* val, int V, DevLevel* out,
                          std::vector<void*>* owned) {
  // 128-row and 64-row tiles of the consecutive rows (a 64-row tile's halo is within its 128-row tile's)
  std::vector<int> all_rows(V);
  for (int v = 0; v < V; ++v) all_rows[v] = v;
  int st = build_blobs(all_rows, TILE_M, rowptr, colidx, val, V, &out->meta128, owned);
  if (st == P2M_OK) st = build_blobs(all_rows, 64, rowptr, colidx, val, V, &out->meta64, owned);
  if (st == P2M_ERR_INVALID) return P2M_OK;  // beyond the blob limits: no tensor-core metadata, the level runs on SIMT
  if (st != P2M_OK) return st;
  {
    // padding-vertex elision: rows whose only entry is the diagonal, all with the same value
    std::vector<int> real_rows, iso_rows;
    float c = 0.f;
    bool uniform = true;
    for (int v = 0; v < V; ++v) {
      const bool iso = (rowptr[v + 1] - rowptr[v] == 1) && colidx[rowptr[v]] == v;
      if (iso) {
        if (iso_rows.empty()) c = val[rowptr[v]];
        if (val[rowptr[v]] != c) uniform = false;
        iso_rows.push_back(v);
      } else {
        real_rows.push_back(v);
      }
    }
    out->n_iso = 0;
    // the families are kept only where every conv a layer of any width can launch on them fits, as on the consecutive
    // tiles (umma_conv_supported): connected rows packed 128 to a tile have larger halos and blobs than the
    // consecutive tiles, which hold the isolated rows too.  Otherwise the level runs on the consecutive tiles.
    auto fits = [](const TileSet& t) { return conv_family_fits(t, CONV_N) && conv_family_fits(t.m64, WIDE_N); };
    if (uniform && (int)iso_rows.size() >= TILE_M && (int)real_rows.size() >= TILE_M) {
      TileSet rt, it;
      if (build_tileset(real_rows, rowptr, colidx, val, V, &rt, owned) == P2M_OK &&
          build_tileset(iso_rows, rowptr, colidx, val, V, &it, owned) == P2M_OK && fits(rt) && fits(it)) {
        out->real_tiles = rt;
        out->iso_tiles = it;
        out->n_iso = (int)iso_rows.size();
        out->iso_diag = c;
      }
    }
  }
  return P2M_OK;
}


bool umma_dw_supported(const DevLevel& g, int gathered_width, int plain_width, bool f16) {
  if (g.meta128.n_pattern <= 0 || g.meta128.max_h1 > 256) return false;
  if (gathered_width % FC != 0 || gathered_width < FC || gathered_width > 256) return false;
  if (plain_width != 64 && plain_width != 128 && plain_width != 256) return false;
  return dw_smem(1, g.meta128.max_h1, g.meta128.stride, f16).bytes <= SMEM_LIMIT;
}
int umma_dw_x_stages(const DevLevel& g, bool f16) {
  return dw_smem(2, g.meta128.max_h1, g.meta128.stride, f16).bytes <= SMEM_LIMIT ? 2 : 1;
}

int launch_umma_dw(const DevLevel& g, int batch, const float* gathered, int in_unpool, int gathered_width,
                   const float* t1, const float* plain, int g_unpool, int plain_width, int swap, const float* a_scale,
                   float* dw_ref, int* status, int sm_count, cudaStream_t s, bool f16) {
  if (!umma_dw_supported(g, gathered_width, plain_width, f16) || t1 == nullptr) {
    set_error("umma_dw: unsupported shape");
    return P2M_ERR_INVALID;
  }
  const TileBlobs& t = g.meta128;
  DwParams p;
  p.x = gathered;
  p.in_unpool = in_unpool;
  p.V = g.V;
  p.P = t.n_pattern;
  p.fin = gathered_width;
  p.n_tiles = batch * t.n_pattern;
  p.meta = t.meta;
  p.meta_bytes = t.bytes;
  p.meta_stride = t.stride;
  p.max_h1 = t.max_h1;
  p.g = plain;
  p.fout_total = plain_width;
  p.a_scale = a_scale;
  p.dw = dw_ref;
  p.status = status;
  p.t1 = t1;
  p.g_unpool = g_unpool;
  p.swap = swap;
  p.tma = 0;
  std::memset(&p.tm_x, 0, sizeof(p.tm_x));
  std::memset(&p.tm_t1, 0, sizeof(p.tm_t1));
  if (g.V % TILE_M == 0 && !in_unpool) {
    const long long rows = (long long)batch * g.V;
    p.tma = (make_row_tmap(&p.tm_x, gathered, rows, gathered_width, TILE_M) &&
             make_row_tmap(&p.tm_t1, t1, rows, gathered_width, TILE_M)) ? 1 : 0;
  }
  const int xs = umma_dw_x_stages(g, f16);
  const size_t smem = dw_smem(xs, t.max_h1, t.stride, f16).bytes;
  auto kern = f16 ? (xs == 2 ? k_cheb_dw_f16_umma<2> : k_cheb_dw_f16_umma<1>)
                  : (xs == 2 ? k_cheb_dw_umma<2> : k_cheb_dw_umma<1>);
  P2M_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = std::min(p.n_tiles, sm_count);
  for (int m_off = 0; m_off < plain_width; m_off += 64) {
    p.m_off = m_off;
    p.m_cols = std::min(64, plain_width - m_off);  // M = 64 plain-side channels per launch
    for (int c0 = 0; c0 < gathered_width / FC; ++c0) {  // one feature chunk per launch (the kernel's n_chunk)
      p.chunk0 = c0;
      kern<<<grid, NUM_THREADS2, smem, s>>>(p);
      log_tc_launch(TC_DW, p.m_cols, DW_NS, xs, 1, f16 ? 1 : 0, dim3(grid), p.n_tiles);
      P2M_LAUNCH_OK();
    }
  }
  return P2M_OK;
}

int launch_cheb_t1(const DevLevel& g, const float* x, int in_unpool, int batch, int fin, float* t1, cudaStream_t s,
                   const TileSet* tiles) {
  const TileBlobs& t = tiles ? *tiles : g.meta128;
  if (t.n_pattern <= 0 || fin % FC != 0) {
    set_error("cheb_t1: unsupported shape");
    return P2M_ERR_INVALID;
  }
  if (t.max_h1 > 256) {  // 4 staged slots per row group
    set_error("cheb_t1: halo too large");
    return P2M_ERR_INVALID;
  }
  const size_t half_sm = (228 * 1024) / 2 - 1024;  // two CTAs per SM (1 KB per CTA is reserved by the system)
  int stages = 4;
  while (stages > 2 && t1_smem(stages, t.max_h1, t.stride).bytes > half_sm) --stages;
  const size_t smem = t1_smem(stages, t.max_h1, t.stride).bytes;
  auto kern = stages == 4 ? k_cheb_t1<4> : (stages == 3 ? k_cheb_t1<3> : k_cheb_t1<2>);
  P2M_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  T1Params p;
  p.x = x;
  p.in_unpool = in_unpool;
  p.V = g.V;
  p.P = t.n_pattern;
  p.fin = fin;
  p.meta = t.meta;
  p.meta_bytes = t.bytes;
  p.meta_stride = t.stride;
  p.max_h1 = t.max_h1;
  p.t1 = t1;
  kern<<<batch * t.n_pattern, 512, smem, s>>>(p);
  P2M_LAUNCH_OK();
  return P2M_OK;
}

// What launch_n runs on the level's consecutive tiles: the T1-given conv and the plain GEMM, both with one ring of 3
// and one X stage at least, on the 64-row tiles for Fout % 128 == 0 and on the 128-row tiles otherwise.
bool umma_conv_supported(const DevLevel& g, int fin, int fout) {
  if (g.meta128.n_pattern <= 0) return false;
  if (fin % FC != 0 || fin < FC || fin > 256) return false;
  if (g.meta128.max_h1 > 256) return false;  // k_cheb_t1 keeps <= 4 staged rows per row group
  if (fout != 64 && fout != 128 && fout != 256) return false;
  const int N = conv_n(fout);
  return conv_family_fits(conv_tiles(N, g, nullptr), N);
}

int umma_tile_families(const DevLevel& g, int fin, int fout, int32_t out[4][2][15]) {
  if (fin % FC != 0 || fin < FC || fin > 256 || (fout != 64 && fout != 128 && fout != 256)) return P2M_ERR_INVALID;
  const TileBlobs* fams[4][2] = {{&g.meta128, &g.meta64},
                                 {&g.real_tiles, &g.real_tiles.m64},
                                 {&g.iso_tiles, &g.iso_tiles.m64},
                                 {&g.rep_tiles, &g.rep_tiles.m64}};
  const int N = conv_n(fout);
  for (int f = 0; f < 4; ++f)
    for (int k = 0; k < 2; ++k) {
      const TileBlobs& t = *fams[f][k];
      int32_t* o = out[f][k];
      std::fill(o, o + 15, 0);
      o[0] = t.n_pattern;
      o[1] = t.max_h1;
      o[2] = t.stride;
      if (t.n_pattern <= 0 || (k == 0) != (N == CONV_N)) continue;  // only the tile size a conv to fout runs on
      for (int c = 0; c < 4; ++c) {  // T1-given fp16x3, plain fp16x3, T1-given fp16, plain fp16
        const bool t1_given = (c & 1) == 0, f16 = c >= 2;
        const int NC = conv_cols(fin, fout, t, t1_given, f16);
        const ConvCfg cfg = conv_cfg(NC, t, t1_given, f16);
        o[3 + 3 * c] = cfg.ns > 0 ? NC : 0;
        o[4 + 3 * c] = cfg.ns;
        o[5 + 3 * c] = cfg.xs;
      }
    }
  return P2M_OK;
}

// What launch_n picks for a conv Fin -> Fout on the level's consecutive tiles (T1 given, or plain): its X staging
// depth, and its output columns per CTA, ring slots and X stages
int umma_conv_x_stages(const DevLevel& g, int fin, int fout, bool plain) {
  return umma_conv_tiling(g, fin, fout, plain).xs;
}
UmmaConvTiling umma_conv_tiling(const DevLevel& g, int fin, int fout, bool plain, bool f16) {
  const int N = conv_n(fout);
  const TileBlobs& t = conv_tiles(N, g, nullptr);
  const int NC = conv_cols(fin, fout, t, !plain, f16);
  const ConvCfg c = conv_cfg(NC, t, !plain, f16);
  return {NC, c.ns, c.xs};
}
bool umma_tma_rows(const DevLevel& g) { return g.V % TILE_M == 0 && tmap_encoder() != nullptr; }

size_t umma_plain_pack_bytes(int N, int K) { return (size_t)(K / FC) * N * 128; }

// ---------------------------------------------------------------- dense GEMM on the conv kernel's plain mode
// the X image, then the device scalar of X's range normalisation (128 bytes keep the image's successors aligned)
static size_t gemm_x_image_bytes(int M, int K) { return (size_t)((M + TILE_M - 1) / TILE_M) * (K / FC) * A_BLOCK_BYTES; }
size_t umma_gemm_apack_bytes(int M, int K) { return gemm_x_image_bytes(M, K) + 128; }
size_t umma_gemm_wpack_bytes(int N, int K) { return (size_t)(K / FC) * N * 128; }
bool umma_gemm_supported(int M, int N, int K) { return M > 0 && K >= FC && K % FC == 0 && N >= 64 && N % 64 == 0; }

namespace {
template <int N>
int launch_gemm_cfg(KParams p, int n_slices, int sm_count, cudaStream_t s) {
  constexpr int NS = 3;
  const size_t smem = conv_smem(N, NS, 1, 0, 0, 0).bytes;  // no tile metadata
  auto kern = conv_kernel<N, NS, 1, 0>();
  P2M_TRY((check_launch_regs<N, NS, 1, 0>()));
  P2M_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  p.wslice_bytes = (long long)umma_gemm_wpack_bytes(N, p.fin);
  p.wblock_stride = (long long)N * 128;
  const dim3 grid(std::min(p.n_tiles, sm_count), n_slices);
  kern<<<grid, ConvRoles<N>::threads, smem, s>>>(p);
  log_tc_launch(TC_GEMM, N, NS, 1, 0, 0, grid, p.n_tiles);
  P2M_LAUNCH_OK();
  return P2M_OK;
}
}  // namespace

// Y [M, N] = epilogue( X [M, K] * W [N, K]^T )  on the tensor cores (wgmma, fp16x3): X and W are packed into operand images first
// (apack / wpack: caller-provided scratch of umma_gemm_{a,w}pack_bytes), then every K-block of both operands is
// streamed by cp.async.bulk into the conv kernel's A/B ring — no producer warps, one CTA per (128-row tile, output
// column slice).  The epilogue vectors and an identity residual (ep.res with res_F == N) are indexed by output column.
// Either operand is read by row and k stride, so a transposed view costs nothing: the backward's dX = g W is
// X = g, W = {W, 1, ld} and dW = g^T a is X = {g, 1, ld}, W = {a, 1, ld}.  k >= k_real is zero padding.
// Operand range: X always enters the fp16 split scaled into [2^9, 2^10) by a power of two (x_scale, a device scalar
// from launch_absmax_scale; found here over the span X's view covers when not given), so the result does not depend
// on the scale of the activations or gradients.  W enters times the fixed W_SCALE (weights), or, when it is an
// activation too (dW's a), times the device scalar w_scale.  The epilogue divides both out.
int launch_umma_gemm(GemmOperand X, GemmOperand W, int M, int N, int K, const Epilogue& ep, float* Y, void* apack,
                     void* wpack, int* status, int sm_count, cudaStream_t s, int n_real, int k_real,
                     const float* x_scale, const float* w_scale) {
  if (n_real <= 0 || n_real > N) n_real = N;  // W has n_real rows; output columns >= n_real are zero-weight padding
  if (k_real <= 0 || k_real > K) k_real = K;
  if (!umma_gemm_supported(M, N, K) || (ep.res != nullptr && ep.res_F != N)) {
    set_error("umma_gemm: unsupported shape");
    return P2M_ERR_INVALID;
  }
  const int tiles = (M + TILE_M - 1) / TILE_M;
  const int ns = CONV_N;  // one warpgroup's register accumulator: 64 output columns per CTA
  if (x_scale == nullptr) {
    float* sc = reinterpret_cast<float*>(static_cast<unsigned char*>(apack) + gemm_x_image_bytes(M, K));
    P2M_TRY(launch_absmax_scale(X.p, (M - 1) * X.ld_row + (k_real - 1) * X.ld_k + 1, sc, s));
    x_scale = sc;
  }
  // A: one 16 KB block per (128-row tile, 32-column chunk), rows >= M zero (what the producers would have built);
  // W: the images of all output-column slices, slice j = rows [j ns, (j + 1) ns) of W, rows >= n_real zero
  P2M_TRY(launch_pack(PackSrc{X.p, X.ld_row, X.ld_k, TILE_M, K / FC, 1, M, 1.f, 0, 0.f, k_real, x_scale},
                      (long long)tiles * (K / FC), apack, s));
  P2M_TRY(launch_pack(PackSrc{W.p, W.ld_row, W.ld_k, ns, K / FC, 1, n_real, w_scale ? 1.f : W_SCALE, 0, 0.f, k_real,
                              w_scale},
                      (long long)(N / ns) * (K / FC), wpack, s));
  KParams p;
  std::memset(&p, 0, sizeof(p));
  p.V = M;                // one "mesh" of M rows: the epilogue masks rows >= V of the last tile
  p.P = tiles;
  p.fin = K;
  p.n_tiles = tiles;
  p.wpack = static_cast<const unsigned char*>(wpack);
  p.apack = static_cast<const unsigned char*>(apack);
  p.a_scale = x_scale;
  p.b_scale = w_scale;
  p.ep = to_dev(ep);
  p.res_identity = (ep.res != nullptr) ? 1 : 0;
  p.ldy = N;
  p.y = Y;
  p.status = status;
  return launch_gemm_cfg<CONV_N>(p, N / ns, sm_count, s);
}

size_t umma_wpack_bytes(int fin, int fout) { return (size_t)(fin / FC) * 3 * fout * 128; }

int launch_umma_pack_weights(const float* W, int fin, int fout, bool transposed, int order, float c, void* wpack,
                             cudaStream_t s, bool f16) {
  const int rows = transposed ? fin : fout, K = transposed ? fout : fin;
  PackSrc src{W, transposed ? 3 : 3LL * fin, transposed ? 3LL * fin : 3, rows, K / FC, 1, rows, W_SCALE, 0, c};
  src.hi_only = f16 ? 1 : 0;
  if (order == WPACK_ALL) src.orders = 3;
  else if (order == WPACK_COMBINED) src.combined = 1;
  else src.p = W + order;
  return launch_pack(src, (long long)(K / FC) * src.orders, wpack, s);
}

int launch_umma_conv(const UmmaConvArgs& a, int* status, const float* zero_row, int sm_count, cudaStream_t s) {
  if (!umma_conv_supported(*a.g, a.fin, a.fout)) {
    set_error("umma_conv: unsupported shape");
    return P2M_ERR_INVALID;
  }
  if (a.head_z != nullptr && (a.fout != 64 || a.head_wt == nullptr || a.ep.res != nullptr)) {
    set_error("umma_conv: the fused head needs fout == 64 and no residual");
    return P2M_ERR_INVALID;
  }
  if (a.t1 == nullptr && !a.plain) {
    set_error("umma_conv: the conv needs T1 = L~x (launch_cheb_t1) unless it is a plain GEMM");
    return P2M_ERR_INVALID;
  }
  if (a.tiles != nullptr && (a.tiles->max_h1 > 256 || a.tiles->n_pattern <= 0 ||
                             (a.fout % WIDE_N == 0 && a.tiles->m64.n_pattern <= 0))) {
    set_error("umma_conv: index-list tiles need at most 256 staged rows");
    return P2M_ERR_INVALID;
  }
  return a.f16 ? launch_n<true>(a, status, zero_row, sm_count, s) : launch_n<false>(a, status, zero_row, sm_count, s);
}

}  // namespace p2m
