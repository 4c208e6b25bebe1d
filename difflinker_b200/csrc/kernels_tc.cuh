// Tensor-core edge kernel (sm_90a wgmma): the second Linear of every edge / coord MLP (85-91 % of the path's FLOPs,
// SURVEY.md section 8(d)), fused with its producer (first Linear + SiLU) and its consumer (bias + SiLU + edge weight +
// segment sum), so no per-edge tensor ever reaches HBM or L2.
//
// Numerics: fp32 operands are split into fp16 hi + lo (x = hi + lo, |lo| <= 2^-11 |x|) and the product is
// accumulated as  W_hi s_hi + W_hi s_lo + W_lo s_hi  in fp32 register accumulators ("3xFP16", ~2^-22 relative
// per product) -- fp32-grade, which is what the 1e-4 end-to-end tolerance needs; plain bf16/tf32 operands
// do not meet it.  Range: W is pre-scaled per matrix, and every edge's activation row per tile, by exact powers
// of two chosen from a-priori bounds so that |operand| < 2^14 (fp16 tops out at 65504 and diverging samples do
// exceed it); the combined descale is folded into the epilogue's first FMA, so scaling costs no accuracy.
//
// Layouts (no swizzle, K-major, canonical "interleave" form of the wgmma shared-memory descriptor):
//   operand tile in smem = [kc 0..15][row][8 halves]   (kc = 16-byte chunk along K=128)
//   core matrix = 8 rows x 16 B contiguous (SBO = 128 B between 8-row groups, LBO = slab pitch between kc)
// GCL  (swapped operands): D[c, e] = sum_k W2[c,k] s[e,k]; warpgroup g owns channels 64g..64g+63. The producers place
//        edge e at operand row 8 * ((e % 32) / 2) + 2 * (e / 32) + e % 2, so the accumulator fragment of a thread
//        holds 32 CONSECUTIVE edges (quad lane q: edges 32q..32q+31) of two channels: the segment sum over j is an
//        in-register walk plus a fixed-order carry across the four lanes of a quad (deterministic, no atomics).
// COORD (natural operands): D[e, c], warpgroup g owns edges 64g..64g+63; a thread reduces its channels with w5 in
//        registers (coord_mlp.4), the quad combines them with two shuffles, then a 3-wide segment sum through shared
//        memory.
#pragma once
#include <cuda_fp16.h>

#include <cmath>
#include <cstdio>
#include <type_traits>
#include <vector>

#include "../../include/difflinker_b200.h"
#include "kernels_simt.cuh"

namespace dl {
namespace tc {

constexpr bool AVAILABLE = true;
constexpr int TN = 128;                    // edges per tile (wgmma N for the GCL, 2 x wgmma M for the coord variant)
constexpr int MAXR = 32;                   // rows per tile
constexpr int KC = 16;                     // 16-byte chunks per K=128 row of fp16
constexpr int W_LBO = H * 16;              // 2048 B: W slab pitch
constexpr int B_LBO = TN * 16 + 16;        // 2064 B: activation slab pitch (+16 B: conflict-free producer stores)
constexpr int SBO = 128;
constexpr int W_BYTES = KC * W_LBO;        // 32 KB per fp16 copy
constexpr int B_BYTES = KC * B_LBO;        // 33,024 B per fp16 copy
constexpr float F16_TARGET = 16384.0f;     // operands are scaled by exact powers of two to stay below 2^14

constexpr int N_STAGE = 2;                 // activation operand stages in shared memory
constexpr int N_ACC = 4;                   // per-tile table ring depth

// warp roles of k_edge_tc: 20 warps = 5 warpgroups. The two MMA warpgroups hold a 64 x 128 fp32 accumulator each (64
// registers a thread), so registers are re-balanced with setmaxnreg: launch 96/thread, the control group gives 32 back,
// the MMA groups take 16 more (256 x 112 + 128 x 64 + 256 x 96 = all 61,440 the launch holds; no role spills).
constexpr int W_EPI = 0;                   // warps 0-7   (WG 0,1): wgmma issue + epilogue, WG g = channel (GCL) / edge (COORD) half
constexpr int N_EPI_WARPS = 8;
constexpr int W_LOAD = 8;                  // warp  8     (WG 2)  : W2 bulk copy
constexpr int W_TBL = 9;                   // warps 9-11  (WG 2)  : per-edge table builders (run ahead of everyone)
constexpr int N_TBL_WARPS = 3;
constexpr int W_PROD = 12;                 // warps 12-19 (WG 3,4): producers (first Linear + SiLU -> fp16 operand tile)
constexpr int N_PROD_WARPS = 8;
constexpr int EDGE_TC_THREADS = 32 * (W_PROD + N_PROD_WARPS);   // 640
constexpr int REGS_EPI = 112, REGS_CTRL = 64;
// GCL: named barriers that pass the wgmma issue turn between the two MMA warpgroups (id 2 is the COORD epilogue's)
constexpr int BAR_TURN0 = 3, BAR_TURN1 = 4;

// shared memory map (bytes from a 1024-aligned base)
constexpr int OFF_WHI = 0;
constexpr int OFF_WLO = OFF_WHI + W_BYTES;
constexpr int OFF_ST = OFF_WLO + W_BYTES;                // N_STAGE x [hi | lo]
constexpr int STAGE_BYTES = 2 * B_BYTES;
constexpr int OFF_TBL = OFF_ST + N_STAGE * STAGE_BYTES;  // N_ACC x per-tile tables
constexpr int TBL_HDR = 0;                               // int [16]: Et, nrt, ncc, flags(first|last<<1), gb_lo, gb_hi, end
constexpr int TBL_ROWOFF = 64;                           // int  [TN]  AB offset (floats) of the edge's row node
constexpr int TBL_COLOFF = TBL_ROWOFF + TN * 4;          // int  [TN]  AB offset of the column node's B half
constexpr int TBL_D = TBL_COLOFF + TN * 4;               // f32  [TN]  |x_i-x_j|^2 of this block
constexpr int TBL_D0 = TBL_D + TN * 4;                   // f32  [TN]  |x0_i-x0_j|^2 of the call's input
constexpr int TBL_SC = TBL_D0 + TN * 4;                  // f32  [TN]  power-of-two scale of the edge's fp16 operand row
constexpr int TBL_EM = TBL_SC + TN * 4;                  // f32x2[TN]  (edge weight, accumulator descale)
constexpr int TBL_CD = TBL_EM + TN * 8;                  // f32  [TN][3] normalised difference (COORD)
constexpr int TBL_ROWNODE = TBL_CD + TN * 12;            // int  [MAXR] node index of each tile row
constexpr int TBL_ROWSTART = TBL_ROWNODE + MAXR * 4;     // int  [MAXR+1] first tile column of each row (neighbour-list tiles)
constexpr int TBL_BYTES = TBL_ROWSTART + (MAXR + 4) * 4;
constexpr int OFF_B2W5 = OFF_TBL + N_ACC * TBL_BYTES;    // float2 [128] (b2, w5)
constexpr int OFF_TX = OFF_B2W5 + H * 8;                 // f32 [TN][3] per-edge translation (COORD epilogue)
constexpr int OFF_BAR = OFF_TX + TN * 12;                // mbarriers
constexpr int BAR_W = 0, BAR_FULL = 8, BAR_EMPTY = BAR_FULL + 8 * N_STAGE, BAR_TBL = BAR_EMPTY + 8 * N_STAGE,
              BAR_TEMPTY = BAR_TBL + 8 * N_ACC, BAR_END = BAR_TEMPTY + 8 * N_ACC;
constexpr int SMEM_BYTES = OFF_BAR + BAR_END + 1024;     // + alignment slack
static_assert(SMEM_BYTES <= 232448, "k_edge_tc exceeds the 227 KB of shared memory a CTA can opt into");
static_assert(TBL_BYTES % 16 == 0, "table slots must keep 16-byte alignment");

// ---------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded spin: a protocol bug must surface as a launch error, never as a hung GPU.
// How a waiting thread waits (set once per process from DL_WAIT_MODE, experiment switch):
//   0  bare try_wait loop
//   1  try_wait with a suspend-time hint: the hardware parks the thread until the phase completes or the time limit passes
//   2  try_wait, then nanosleep(32) between polls
__device__ __constant__ int c_wait_mode = 1;
constexpr uint32_t WAIT_HINT_NS = 20000;
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const int mode = c_wait_mode;
  if (mode == 1) {
    for (uint32_t spin = 0; spin < (1u << 20); ++spin) {
      asm volatile(
          "{\n\t.reg .pred p;\n\t"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
          "selp.u32 %0, 1, 0, p;\n\t}"
          : "=r"(done)
          : "r"(bar), "r"(parity), "r"(WAIT_HINT_NS)
          : "memory");
      if (done) return;
    }
    __trap();
  }
  for (uint32_t spin = 0; spin < (1u << 28); ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return;
    if (mode == 2) __nanosleep(32);
  }
  __trap();
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void named_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Same, for roles that run far ahead of (or lag behind) the critical path: back off between polls so the spin does
// not steal issue slots from the producer / epilogue warps sharing the scheduler.
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < (1u << 24); ++spin) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return;
    __nanosleep(64);
  }
  __trap();
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// 1-D bulk copy global -> shared through the TMA engine, completion on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// wgmma shared-memory matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset 0, layout
// type [62,64) = 0 (interleave, no swizzle). K-major operand: LBO = pitch between 16-byte K chunks, SBO = pitch between
// 8-row groups; MN-major operand: LBO = pitch between 8-deep K groups, SBO = pitch between 8-wide M/N groups.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (64 x 128 fp32, registers of the issuing warpgroup) (+)= A (64 x 16, K-major smem) * B (128 x 16 smem; TRANS_B = 1:
// MN-major). Fragment of thread t (warp w = t / 32 of the group, lane l): rows 16 w + l / 4 (+ 8 for d[4j + 2..3]),
// columns 8 j + 2 (l % 4) + {0, 1}.
template <int TRANS_B>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, %67;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TRANS_B));
}
// One 3xFP16 product over K = 16 * nks: d (+)= A_lo B_hi + A_hi B_lo + A_hi B_hi (all operands K-major unless TRANS_B).
template <int TRANS_B = 0>
__device__ __forceinline__ void mma_3xf16(float (&d)[64], uint32_t a_hi, uint32_t a_lo, uint32_t a_lbo, uint32_t b_hi,
                                          uint32_t b_lo, uint32_t b_lbo, uint32_t b_ks_stride, int nks, bool accumulate) {
#pragma unroll
  for (int ks = 0; ks < nks; ++ks) {
    const uint64_t ah = wg_desc(a_hi + ks * 2 * a_lbo, a_lbo, SBO), al = wg_desc(a_lo + ks * 2 * a_lbo, a_lbo, SBO);
    const uint64_t bh = wg_desc(b_hi + ks * b_ks_stride, b_lbo, SBO), bl = wg_desc(b_lo + ks * b_ks_stride, b_lbo, SBO);
    wgmma_m64n128k16<TRANS_B>(d, al, bh, (accumulate || ks > 0) ? 1u : 0u);
    wgmma_m64n128k16<TRANS_B>(d, ah, bl, 1u);
    wgmma_m64n128k16<TRANS_B>(d, ah, bh, 1u);
  }
}
// The whole 3xFP16 GEMM of one warpgroup: fence, issue, commit, wait.
template <int TRANS_B = 0>
__device__ __forceinline__ void gemm_3xf16(float (&d)[64], uint32_t a_hi, uint32_t a_lo, uint32_t a_lbo, uint32_t b_hi,
                                           uint32_t b_lo, uint32_t b_lbo, uint32_t b_ks_stride, int nks, bool accumulate) {
  fence_acc(d);
  wg_fence();
  mma_3xf16<TRANS_B>(d, a_hi, a_lo, a_lbo, b_hi, b_lo, b_lbo, b_ks_stride, nks, accumulate);
  wg_commit();
  wg_wait_all();
  fence_acc(d);
}

// fp32 pair -> fp16x2 hi and lo words
__device__ __forceinline__ void split2v(float2 v, uint32_t& hi, uint32_t& lo) {
  __half2 h = __float22half2_rn(v);
  float2 back = __half22float2(h);
  __half2 l = __float22half2_rn(fadd2(v, make_float2(-back.x, -back.y)));
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
// fp32 -> fp16 hi/lo pair of two values
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  __half2 h = __floats2half2_rn(a, b);
  float2 back = __half22float2(h);
  __half2 l = __floats2half2_rn(a - back.x, b - back.y);
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
// GCL operand row of tile edge e (see the file comment): thread quad lane q then holds edges 32q .. 32q+31 in order
__device__ __forceinline__ int gcl_row_of_edge(int e) { return 8 * ((e & 31) >> 1) + 2 * (e >> 5) + (e & 1); }
// ---------------------------------------------------------------------------------------------------------
// Tile iteration (table warps only): a CTA walks its work items (static round-robin) -> row groups ->
// 128-column chunks. A tile is whole rows x all live columns (or one row x a 128-column chunk when nc > 128), so
// the segment sum over j never crosses CTAs.
// ---------------------------------------------------------------------------------------------------------
struct Tile {
  int b, nc, slot0, nrt, c0, ncc;
  bool first_chunk, last_chunk;
  const int* rows;
  // neighbour-list (SPARSE) tiles only; per-lane values: lane l describes tile row l
  int Et;        // edges in the tile (uniform)
  int start;     // first tile column of row l (exclusive prefix of the row degrees)
  int node;      // node index of row l
};

// Warp-synchronous (all 32 lanes of a table warp call it together): the CTA's contiguous slice of the work-item
// list is read 32 items at a time with one coalesced load and served from registers by shuffles, so walking the
// list costs no dependent global round trip per tile (items carry their molecule's live column count).
template <bool COORD>
struct TileIter {
  const int4* list;
  const int* rowlist;
  int N, wi_end, wi, rt, c0, cache_base, lane;
  int4 cache;
  __device__ TileIter(const Plan& p, int N_) : N(N_), rt(0), c0(0), cache_base(-(1 << 30)), lane(threadIdx.x & 31) {
    // blocked distribution: CTA c owns the contiguous work items [lo, hi) -- consecutive tiles then mostly belong to
    // the same molecule, so the table warps' and producers' L2 lines are reused while they are hot.
    list = COORD ? p.xitems : p.items;
    rowlist = COORD ? p.xrowidx : p.rowidx;
    const int total = COORD ? *p.n_xitems : *p.n_items;
    const int per = total / (int)gridDim.x, extra = total % (int)gridDim.x, c = (int)blockIdx.x;
    wi = c * per + min(c, extra);
    wi_end = wi + per + (c < extra ? 1 : 0);
    cache = make_int4(0, 0, 0, 0);
  }
  __device__ bool next(Tile& t) {
    while (wi < wi_end) {
      if (wi - cache_base >= 32) {                        // refill (warp-uniform)
        cache_base = wi;
        cache = list[min(wi + lane, wi_end - 1)];
      }
      const int src = wi - cache_base;
      const int b = __shfl_sync(0xffffffffu, cache.x, src), r_begin = __shfl_sync(0xffffffffu, cache.y, src);
      const int r_count = __shfl_sync(0xffffffffu, cache.z, src), nc = __shfl_sync(0xffffffffu, cache.w, src);
      int per = nc >= TN ? 1 : TN / max(nc, 1);
      if (per > MAXR) per = MAXR;
      if (rt >= r_count || nc <= 0) { wi += 1; rt = 0; c0 = 0; continue; }
      t.b = b; t.nc = nc; t.slot0 = r_begin + rt; t.nrt = min(per, r_count - rt);
      t.c0 = c0; t.ncc = min(TN, nc - c0);
      t.first_chunk = c0 == 0; t.last_chunk = c0 + TN >= nc;
      t.rows = rowlist + (size_t)b * N;
      c0 += TN;
      if (c0 >= nc) { c0 = 0; rt += per; }
      return true;
    }
    return false;
  }
};

// Cut-off graphs: the CTA walks the tile records k_nbr packed for this call (round-robin over CTAs: records cost one
// tile, or ceil(degree / 128) chunk tiles for a row with more than 128 neighbours -- its sum is carried in the epilogue's
// registers, so the chunks stay on one CTA). Warp-synchronous; lane l holds int l of the 128-byte record and the
// next record is prefetched while the current one is served.
struct RecIter {
  const int* recs;
  int n, k, G, lane, cur, nxt, chunk;
  __device__ RecIter(const int* recs_, const int* n_recs) : recs(recs_), lane(threadIdx.x & 31), cur(0), chunk(0) {
    n = *n_recs; G = (int)gridDim.x; k = (int)blockIdx.x;
    nxt = k < n ? recs[(size_t)k * CUT_REC + lane] : 0;
  }
  __device__ bool next(Tile& t) {
    if (chunk == 0) {
      if (k >= n) return false;
      cur = nxt;
      const int kn = k + G;
      nxt = kn < n ? recs[(size_t)kn * CUT_REC + lane] : 0;
    }
    const int w1 = __shfl_sync(0xffffffffu, cur, 1), v2 = __shfl_sync(0xffffffffu, cur, 2);
    const int info = __shfl_sync(0xffffffffu, cur, (4 + lane) & 31);
    t.b = __shfl_sync(0xffffffffu, cur, 0);
    t.nc = 0; t.slot0 = 0; t.rows = nullptr;
    if (((w1 >> 8) & 1) == 0) {
      t.nrt = w1 & 0xff; t.Et = v2; t.ncc = v2; t.c0 = 0; t.first_chunk = true; t.last_chunk = true;
      t.node = info & 0xffff; t.start = info >> 16;
      k += G;
    } else {
      const int deg = v2, c0 = chunk * TN;
      t.nrt = 1; t.Et = min(TN, deg - c0); t.ncc = t.Et; t.c0 = c0;
      t.first_chunk = chunk == 0; t.last_chunk = c0 + TN >= deg;
      t.node = __shfl_sync(0xffffffffu, cur, 4) & 0xffff;
      t.start = lane == 0 ? 0 : t.Et;
      ++chunk;
      if (t.last_chunk) { chunk = 0; k += G; }
    }
    return true;
  }
};

template <bool COORD, bool SPARSE>
__device__ __forceinline__ typename std::conditional<SPARSE, RecIter, TileIter<COORD>>::type make_iter(const EdgeArgs& a, int N) {
  if constexpr (SPARSE) return RecIter(a.recs, a.n_recs);
  else return TileIter<COORD>(a.plan, N);
}

// ---------------------------------------------------------------------------------------------------------
// The kernel: persistent, 1 CTA / SM, 20 warps in four roles connected by mbarrier rings.
//
//   table warps (3)  : walk the CTA's tile list; per edge (i,j): node offsets, d_ij, d0_ij, edge weight, operand
//                      scale, normalised difference -> table ring slot a = t % 4          [tbl[a]]
//   producers (8)    : A_i + B_j + d w_d + d0 w_0 -> SiLU -> fp16 hi/lo operand tile, stage s = t % 2
//                      (register prefetch of the next item's A/B rows)                      [full[s]]
//   MMA warpgroups (2): 24 x wgmma (3xFP16, K=128) into registers, then the epilogue from those registers:
//                      bias + SiLU + edge weight + segment sum                              [empty[s], tempty[a]]
//   loader (1)       : W2 hi|lo, one bulk copy per launch                                    [w]
//
// Every role works on a different tile at any moment, so L2 latency (producers) and the tensor pipe + epilogue overlap.
// GCL: the two MMA warpgroups take turns at the tensor pipe (ping-pong, named barriers BAR_TURN0/1): WG 0 issues tile t,
// WG 1 issues tile t as soon as WG 0 has committed, WG 0 runs its epilogue of t while WG 1's wgmma run, then issues t + 1
// as soon as WG 1 has committed, and so on. The accumulator lives in the registers of the group that runs the epilogue,
// so this alternation is what keeps the tensor pipe busy during epilogues. COORD keeps both groups in lockstep: its
// epilogue combines the two edge halves through shared memory.
// SPARSE = true: cut-off (pocket) graphs -- tiles are packed from the per-row neighbour lists k_nbr built for this
// forward call, so only edges the reference creates are processed (egnn.py:554-596); FC graphs use SPARSE = false.
// OPT (OPT_TANH | OPT_MEAN, common.cuh): OPT_TANH bounds the COORD update, trans = (cd * tanh(phi)) * coords_range * EM;
// OPT_MEAN divides each row's sum by its edge count in the reference's edge list: N on FC graphs; on cut-off graphs the
// row's neighbour-list length, which is its degree, or 1 for an isolated row (its one padding edge) -- taken from the
// tile's row starts, or from the header (hdr[6]) for the chunk tiles of a row with more than 128 neighbours.
// ---------------------------------------------------------------------------------------------------------
// OPT_SIN: the table's d / d0 are the radials in the reference's rounding order, and the producers replace d w_d + d0 w_0
// by sum_k e_k w_k over the 24 sinusoidal features: lane k < 12 of an edge's 16-lane half evaluates sincos of one
// (radial, frequency) pair, the features reach the other lanes by shuffles, and w_k comes through L1.
template <bool COORD, bool SPARSE = false, int OPT = 0>
__global__ void __launch_bounds__(EDGE_TC_THREADS, 1) k_edge_tc(Geom gm, EdgeArgs a, const __half* __restrict__ w2tc) {
  constexpr bool MEAN = (OPT & OPT_MEAN) != 0, TANH = (OPT & OPT_TANH) != 0, EMB = (OPT & OPT_SIN) != 0;
  static_assert(COORD || !TANH, "tanh only bounds the coordinate update");
  extern __shared__ uint8_t smem_raw[];
  // keep the pointer derived from the __shared__ array (no integer round trip) so accesses compile to LDS/STS
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(sm);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = gm.N;

  const uint32_t bars = sbase + OFF_BAR;
  float2* b2w5 = reinterpret_cast<float2*>(sm + OFF_B2W5);

  if (tid == 0) {
    mbar_init(bars + BAR_W, 1);
    for (int i = 0; i < N_STAGE; ++i) { mbar_init(bars + BAR_FULL + 8 * i, N_PROD_WARPS); mbar_init(bars + BAR_EMPTY + 8 * i, N_EPI_WARPS); }
    for (int i = 0; i < N_ACC; ++i) {
      mbar_init(bars + BAR_TBL + 8 * i, 1);
      mbar_init(bars + BAR_TEMPTY + 8 * i, N_EPI_WARPS);
    }
    fence_barrier_init();
  }
  if (tid < H) b2w5[tid] = make_float2(a.b2[tid], COORD ? a.w5[tid] : 0.f);
  __syncthreads();

  // Register re-balancing happens at the top of each role branch (warpgroup-aligned: every warp of a group runs the
  // same setmaxnreg; ptxas allocates each branch against the budget set by the instruction that dominates it).
  if (warp >= W_LOAD && warp < W_PROD) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS_CTRL));
  if (warp >= W_TBL && warp < W_TBL + N_TBL_WARPS) {
    // =================================== table warps ===================================================================
    // Tile-parallel: table warp k builds the tables of tiles t = k, k+3, ... on its own (4 edges per lane), so the
    // three warps overlap their dependent L2 round trips (index -> coordinates / maxima / mask) across tiles.
    const int tw = warp - W_TBL;
    typename std::conditional<SPARSE, RecIter, TileIter<COORD>>::type iter = make_iter<COORD, SPARSE>(a, N);
    Tile cur;
    for (int t = 0;; ++t) {
      const int acc = t & (N_ACC - 1);
      const bool more = iter.next(cur);
      if (t % N_TBL_WARPS != tw) { if (!more) break; continue; }
      if (t >= N_ACC) mbar_wait_relaxed(bars + BAR_TEMPTY + 8 * acc, ((t - N_ACC) / N_ACC) & 1);   // slot's previous tile fully consumed
      uint8_t* tb = sm + OFF_TBL + acc * TBL_BYTES;
      int* hdr = reinterpret_cast<int*>(tb + TBL_HDR);
      if (more) {
        const int Et = SPARSE ? cur.Et : cur.nrt * cur.ncc;
        const size_t gb = (size_t)cur.b * N;
        int heavy_deg = 0;                                 // OPT_MEAN: degree of a row served in chunk tiles (its record)
        if constexpr (MEAN && SPARSE) {
          const int w1 = __shfl_sync(0xffffffffu, iter.cur, 1), v2 = __shfl_sync(0xffffffffu, iter.cur, 2);
          heavy_deg = ((w1 >> 8) & 1) ? v2 : 0;
        }
        if (lane == 0) {
          hdr[0] = Et; hdr[1] = cur.nrt; hdr[2] = cur.ncc;
          hdr[3] = (cur.first_chunk ? 1 : 0) | (cur.last_chunk ? 2 : 0);
          hdr[4] = cur.b;
          if (MEAN && SPARSE) hdr[6] = heavy_deg;
        }
        if (SPARSE) {
          if (lane < cur.nrt) {
            reinterpret_cast<int*>(tb + TBL_ROWNODE)[lane] = cur.node;
            reinterpret_cast<int*>(tb + TBL_ROWSTART)[lane] = cur.start;
          }
          if (lane == 0) reinterpret_cast<int*>(tb + TBL_ROWSTART)[cur.nrt] = Et;
        } else {
          if (lane < cur.nrt) {
            reinterpret_cast<int*>(tb + TBL_ROWNODE)[lane] = cur.rows[cur.slot0 + lane];
            reinterpret_cast<int*>(tb + TBL_ROWSTART)[lane] = lane * cur.ncc;
          }
          if (lane == 0) reinterpret_cast<int*>(tb + TBL_ROWSTART)[cur.nrt] = Et;
        }
        bool any_rescale = false;
#pragma unroll
        for (int e = lane; e < TN; e += 32) {
          const int ev = min(e, Et - 1);                   // slots past Et mirror the last edge: producers may prefetch them
          int i, j;
          float ew_list = 1.f;
          if (SPARSE) {
            int rr = 0;                                    // tile row of this edge: rows start at ascending columns
            for (int r = 1; r < cur.nrt; ++r) rr += ev >= __shfl_sync(0xffffffffu, cur.start, r) ? 1 : 0;
            i = __shfl_sync(0xffffffffu, cur.node, rr);
            const int first_col = __shfl_sync(0xffffffffu, cur.start, rr);
            const int raw = a.nbr[(gb + i) * N + cur.c0 + (ev - first_col)];
            j = raw & 0x7fffffff;
            ew_list = raw < 0 ? 0.f : 1.f;                 // padding edge of an isolated row
          } else {
            const int rr = ev / cur.ncc, jj = ev - rr * cur.ncc;
            i = cur.rows[cur.slot0 + rr];
            j = a.plan.colidx[gb + cur.c0 + jj];
          }
          const float4 xi = a.x4[gb + i], xj = a.x4[gb + j], yi = a.x04[gb + i], yj = a.x04[gb + j];   // 16-byte gathers
          const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
          const float ex = yi.x - yj.x, ey = yi.y - yj.y, ez = yi.z - yj.z;
          float d, d0;
          if constexpr (EMB) {                                               // sinusoid arguments: torch's rounding order
            d = radial_rn(dx, dy, dz); d0 = radial_rn(ex, ey, ez);
          } else {
            d = dx * dx + dy * dy + dz * dz;                                 // egnn.py:297-298
            d0 = ex * ex + ey * ey + ez * ez;                                // egnn.py:220
          }
          int ci = 0, cj = 0;
          if (!SPARSE && gm.graph_type != 0) { ci = a.cls[gb + i]; cj = a.cls[gb + j]; }
          reinterpret_cast<int*>(tb + TBL_ROWOFF)[e] = (int)((gb + i) * 2 * H);
          reinterpret_cast<int*>(tb + TBL_COLOFF)[e] = (int)((gb + j) * 2 * H + H);
          reinterpret_cast<float*>(tb + TBL_D)[e] = d;
          reinterpret_cast<float*>(tb + TBL_D0)[e] = d0;
          // |silu(pre)| <= |pre| <= max|A_i| + max|B_j| + d max|wd| + d0 max|w0|: exact power-of-two scale that keeps the
          // fp16 hi/lo operands of this edge below 2^14 (activations of diverging samples exceed fp16's 65504).
          // (with OPT_SIN: + sum_k max|w_k|, since |sin|, |cos| <= 1)
          const float bound = EMB ? a.ABmax[(gb + i) * 2] + a.ABmax[(gb + j) * 2 + 1] + a.wdmax
                                  : a.ABmax[(gb + i) * 2] + a.ABmax[(gb + j) * 2 + 1] + d * a.wdmax + d0 * a.w0max;
          float sc = 1.0f;
          if (!(bound <= F16_TARGET)) {
            const int ex2 = ((__float_as_int(bound) >> 23) & 0xff) - 127;
            sc = __int_as_float(max(127 + 13 - ex2, 1) << 23);
          }
          reinterpret_cast<float*>(tb + TBL_SC)[e] = sc;
          any_rescale |= (sc != 1.0f);
          // GCL epilogue works in the log2 domain: u = -log2(e) * (D*descale + b2) is one FMA, sigmoid = 1/(1+2^u), and
          // the -ln(2) that turns u*sigmoid back into silu rides on the edge weight (one rounding of a constant).
          const float ew = SPARSE ? ew_list
                                  : edge_weight(gm.graph_type, a.edge_mask ? a.edge_mask + gb * N : nullptr, N, i, j, ci, cj, d0);
          reinterpret_cast<float2*>(tb + TBL_EM)[e] =
              COORD ? make_float2(ew, a.w2_descale / sc)
                    : make_float2(ew * -0.6931471805599453f, (a.w2_descale / sc) * -1.4426950408889634f);
          if (COORD) {
            const float inv = 1.0f / (sqrtf(d + 1e-8f) + gm.norm_constant);  // egnn.py:299-300
            float* cds = reinterpret_cast<float*>(tb + TBL_CD);
            cds[e * 3 + 0] = dx * inv; cds[e * 3 + 1] = dy * inv; cds[e * 3 + 2] = dz * inv;
          }
        }
        any_rescale = __any_sync(0xffffffffu, any_rescale);
        if (lane == 0) hdr[5] = any_rescale ? 1 : 0;       // tile-level flag: producers skip the scale multiply
      } else if (lane == 0) {
        hdr[0] = 0;                                      // end marker travels through the whole pipeline
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + BAR_TBL + 8 * acc);
      if (!more) break;
    }
  } else if (warp == W_LOAD) {
    if (lane == 0) {                                     // W2 hi|lo tiles: one 64 KB bulk copy, resident for the launch
      mbar_expect_tx(bars + BAR_W, 2 * W_BYTES);
      bulk_g2s(sbase + OFF_WHI, w2tc, 2 * W_BYTES, bars + BAR_W);
    }
  }
  } else if (warp >= W_PROD) {
    // =================================== producers =====================================================================
    const int pw = warp - W_PROD;
    const int kc = lane & 15, esub = lane >> 4;            // this thread always owns k = kc*8 .. kc*8+7
    float2 wdr[4], w0r[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      wdr[q] = make_float2(__ldg(a.wd + kc * 8 + 2 * q), __ldg(a.wd + kc * 8 + 2 * q + 1));
      w0r[q] = make_float2(__ldg(a.w0 + kc * 8 + 2 * q), __ldg(a.w0 + kc * 8 + 2 * q + 1));
    }
    for (int t = 0;; ++t) {
      const int acc = t & (N_ACC - 1), s = t & (N_STAGE - 1);
      mbar_wait(bars + BAR_TBL + 8 * acc, (t / N_ACC) & 1);
      const uint8_t* tb = sm + OFF_TBL + acc * TBL_BYTES;
      const int Et = reinterpret_cast<const int*>(tb + TBL_HDR)[0];
      if (t >= N_STAGE) mbar_wait(bars + BAR_EMPTY + 8 * s, ((t - N_STAGE) / N_STAGE) & 1);   // MMA(t-2) has read this stage
      if (Et > 0) {
        const int* rowoff = reinterpret_cast<const int*>(tb + TBL_ROWOFF);
        const int* coloff = reinterpret_cast<const int*>(tb + TBL_COLOFF);
        const float* dv = reinterpret_cast<const float*>(tb + TBL_D);
        const float* d0v = reinterpret_cast<const float*>(tb + TBL_D0);
        const float* scv = reinterpret_cast<const float*>(tb + TBL_SC);
        uint8_t* bhi = sm + OFF_ST + s * STAGE_BYTES + kc * B_LBO;
        uint8_t* blo = bhi + B_BYTES;
        const bool rescale = reinterpret_cast<const int*>(tb + TBL_HDR)[5] != 0;
        constexpr int ITEMS = TN / (2 * N_PROD_WARPS);       // 8 edges per thread per tile
        // Two B_j chunks are kept in flight in registers (these loads are L2 round trips). Table slots past Et mirror
        // the last edge: no clamping here. A thread takes ITEMS consecutive edges of the tile: they share the row
        // (almost always), so the A_i chunk is loaded once and only the B_j chunks stream.
        float4 pa0, pa1, pb[2][2];
        const int e_base = ITEMS * (2 * pw + esub);
        int ro_cur = rowoff[e_base];
        {
          const float* ap = a.AB + ro_cur + kc * 8;
          pa0 = __ldg(reinterpret_cast<const float4*>(ap)); pa1 = __ldg(reinterpret_cast<const float4*>(ap + 4));
        }
#pragma unroll
        for (int pf = 0; pf < 2; ++pf) {
          const float* bp = a.AB + coloff[e_base + pf] + kc * 8;
          pb[pf][0] = __ldg(reinterpret_cast<const float4*>(bp)); pb[pf][1] = __ldg(reinterpret_cast<const float4*>(bp + 4));
        }
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) {
          const int e = e_base + it;
          const int slot = it & 1;
          const float4 b0 = pb[slot][0], b1 = pb[slot][1];
          if (it + 2 < ITEMS) {
            const float* bp = a.AB + coloff[e + 2] + kc * 8;
            pb[slot][0] = __ldg(reinterpret_cast<const float4*>(bp)); pb[slot][1] = __ldg(reinterpret_cast<const float4*>(bp + 4));
          }
          const int ro = rowoff[e];
          if (ro != ro_cur) {                              // row boundary inside this thread's run (rare): reload A_i
            ro_cur = ro;
            const float* ap = a.AB + ro + kc * 8;
            pa0 = __ldg(reinterpret_cast<const float4*>(ap)); pa1 = __ldg(reinterpret_cast<const float4*>(ap + 4));
          }
          const float4 a0 = pa0, a1 = pa1;
          float2 pre_emb[4];
          if constexpr (EMB) {                             // all lanes (shuffles): slots past Et mirror the last edge
            const int kf = kc < 12 ? kc : kc - 12;          // lanes 12-15 repeat lanes 0-3; their values are not read
            float sn, cs;
            sincosf(sin_arg(kf < N_SIN_FREQ ? dv[e] : d0v[e], kf % N_SIN_FREQ), &sn, &cs);
            pre_emb[0] = fadd2(make_float2(a0.x, a0.y), make_float2(b0.x, b0.y));
            pre_emb[1] = fadd2(make_float2(a0.z, a0.w), make_float2(b0.z, b0.w));
            pre_emb[2] = fadd2(make_float2(a1.x, a1.y), make_float2(b1.x, b1.y));
            pre_emb[3] = fadd2(make_float2(a1.z, a1.w), make_float2(b1.z, b1.w));
#pragma unroll 2                                   // unrolled further, the weight loads are hoisted and spill
            for (int k = 0; k < N_SIN_FEAT; ++k) {         // feature k: [sin d f, cos d f, sin d0 f, cos d0 f][k % 6]
              const int src = (k / 12) * N_SIN_FREQ + k % N_SIN_FREQ;
              const float ev = __shfl_sync(0xffffffffu, (k % 12) < N_SIN_FREQ ? sn : cs, src, 16);
              const float4 w0 = __ldg(reinterpret_cast<const float4*>(a.we + k * H + kc * 8));
              const float4 w1 = __ldg(reinterpret_cast<const float4*>(a.we + k * H + kc * 8 + 4));
              const float2 ee = make_float2(ev, ev);
              pre_emb[0] = ffma2(ee, make_float2(w0.x, w0.y), pre_emb[0]);
              pre_emb[1] = ffma2(ee, make_float2(w0.z, w0.w), pre_emb[1]);
              pre_emb[2] = ffma2(ee, make_float2(w1.x, w1.y), pre_emb[2]);
              pre_emb[3] = ffma2(ee, make_float2(w1.z, w1.w), pre_emb[3]);
            }
          }
          if (e < Et) {
            float2 sv[4];
            if constexpr (EMB) {
#pragma unroll
              for (int q = 0; q < 4; ++q) sv[q] = usig2(pre_emb[q]);
            } else {
              const float d = dv[e], d0 = d0v[e];
              const float2 dd = make_float2(d, d), dd0 = make_float2(d0, d0);
              const float2 av[4] = {make_float2(a0.x, a0.y), make_float2(a0.z, a0.w), make_float2(a1.x, a1.y), make_float2(a1.z, a1.w)};
              const float2 bv[4] = {make_float2(b0.x, b0.y), make_float2(b0.z, b0.w), make_float2(b1.x, b1.y), make_float2(b1.z, b1.w)};
  #pragma unroll
              for (int q = 0; q < 4; ++q)                     // egnn.py:49-50
                sv[q] = usig2(ffma2(dd0, w0r[q], ffma2(dd, wdr[q], fadd2(av[q], bv[q]))));   // log2 domain (see pack_w2)
            }
            if (rescale) {                                 // rare: diverging samples only (tile-uniform)
              const float sc = scv[e];
#pragma unroll
              for (int q = 0; q < 4; ++q) sv[q] = fmul2(sv[q], make_float2(sc, sc));
            }
            uint4 hi, lo;
            split2v(sv[0], hi.x, lo.x); split2v(sv[1], hi.y, lo.y);
            split2v(sv[2], hi.z, lo.z); split2v(sv[3], hi.w, lo.w);
            const int row = COORD ? e : gcl_row_of_edge(e);
            *reinterpret_cast<uint4*>(bhi + row * 16) = hi;
            *reinterpret_cast<uint4*>(blo + row * 16) = lo;
          }
        }
        fence_proxy_async();      // generic-proxy smem writes -> visible to the tensor core (async proxy)
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + BAR_FULL + 8 * s);
      if (Et <= 0) break;
    }
  } else {
    // =================================== MMA + epilogue warpgroups ========================================================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS_EPI));
    const int g = warp >> 2;                               // warpgroup: channel half (GCL) / edge half (COORD)
    const int wq = warp & 3, q = lane & 3;
    const int r0 = 64 * g + 16 * wq + (lane >> 2);         // accumulator rows r0 and r0 + 8
    float* txs = reinterpret_cast<float*>(sm + OFF_TX);
    float2 run = make_float2(0.f, 0.f);                    // GCL: row sum carried across column chunks
    float run3 = 0.f;                                      // COORD: (row, dim) sum carried across column chunks
    float d[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) d[i] = 0.f;
    mbar_wait(bars + BAR_W, 0);
    for (int t = 0;; ++t) {
      const int acc = t & (N_ACC - 1), s = t & (N_STAGE - 1);
      // GCL ping-pong: WG 0 issues tile t once WG 1 has issued tile t - 1 (also before the end marker, so every arrive on a
      // turn barrier is matched by a sync), and WG 1 issues tile t once WG 0 has.
      if (!COORD && g == 0 && t > 0) named_sync(BAR_TURN0, 32 * N_EPI_WARPS);
      mbar_wait(bars + BAR_TBL + 8 * acc, (t / N_ACC) & 1);
      const uint8_t* tb = sm + OFF_TBL + acc * TBL_BYTES;
      const int* hdr = reinterpret_cast<const int*>(tb + TBL_HDR);
      const int Et = hdr[0];
      if (Et <= 0) break;
      const uint32_t bhi = sbase + OFF_ST + s * STAGE_BYTES, blo = bhi + B_BYTES;
      if (!COORD) {
        if (g == 1) named_sync(BAR_TURN1, 32 * N_EPI_WARPS);
        mbar_wait(bars + BAR_FULL + 8 * s, (t / N_STAGE) & 1);
        fence_acc(d);
        wg_fence();
        mma_3xf16(d, sbase + OFF_WHI + g * 1024, sbase + OFF_WLO + g * 1024, W_LBO, bhi, blo, B_LBO, 2 * B_LBO, 8, false);
        wg_commit();
        // Hand the turn over once committed, not completed: the other group's wgmma queue behind these and the tensor
        // pipe never drains, while this group's epilogue below overlaps them.
        named_arrive(g == 0 ? BAR_TURN1 : BAR_TURN0, 32 * N_EPI_WARPS);
        wg_wait_all();
        fence_acc(d);
      } else {
        mbar_wait(bars + BAR_FULL + 8 * s, (t / N_STAGE) & 1);
        gemm_3xf16(d, bhi + g * 1024, blo + g * 1024, B_LBO, sbase + OFF_WHI, sbase + OFF_WLO, W_LBO, 2 * W_LBO, 8, false);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + BAR_EMPTY + 8 * s);   // operand stage reusable: this warpgroup's wgmma are complete

      const int nrt = hdr[1];
      const bool first_chunk = hdr[3] & 1, last_chunk = hdr[3] & 2;
      const size_t gb = (size_t)hdr[4] * N;
      const float2* emds = reinterpret_cast<const float2*>(tb + TBL_EM);
      const int* rownode = reinterpret_cast<const int*>(tb + TBL_ROWNODE);
      const int* rowstart = reinterpret_cast<const int*>(tb + TBL_ROWSTART);
      if (!COORD) {
        // Thread = channels (r0, r0 + 8) x edges E0 .. E0 + 31. Rows are contiguous edge ranges. Bit tt of bmask marks a
        // row start at edge E0 + tt inside the run; the tile end Et counts as one, so edges past it land in a sum nobody
        // reads. The per-edge path is arithmetic plus one running sum: at a boundary the sum closes the run's first row
        // (hsum, finished below with the carry from earlier lanes) or a row that lies wholly inside the run (written at
        // once); the partial sum of a row that leaves the run is passed to the next quad lane.
        const float2 bias = make_float2(b2w5[r0].x * -1.4426950408889634f, b2w5[r0 + 8].x * -1.4426950408889634f);
        const float inv_norm = 1.0f / gm.normalization_factor;
        // agg_i = row sum / normalization_factor, or with OPT_MEAN / the row's edge count (egnn.py:312-319). Both multiply by a
        // reciprocal, as the division by normalization_factor always has (within 2 ulp of the reference's division): an IEEE
        // division in this unrolled loop costs 13 % of the launch.
        const float inv_n = 1.0f / (float)N;
        auto put = [&](int r, float2 v) {
          float* dst = a.agg + (gb + rownode[r]) * H;
          if constexpr (MEAN) {
            const float inv = SPARSE ? rcp_approx((float)(hdr[6] > 0 ? hdr[6] : rowstart[r + 1] - rowstart[r])) : inv_n;
            dst[r0] = v.x * inv; dst[r0 + 8] = v.y * inv;
          } else {
            dst[r0] = v.x * inv_norm; dst[r0 + 8] = v.y * inv_norm;
          }
        };
        const int E0 = 32 * q;
        const bool has = E0 < Et;
        int cur = 0;
        if (has) { while (rowstart[cur + 1] <= E0) ++cur; }
        const int hrow = cur;
        uint32_t bmask = 0;
        int nr = cur + 1;
        if (has) { for (; nr <= nrt && rowstart[nr] < E0 + 32; ++nr) bmask |= 1u << (rowstart[nr] - E0); }
        const bool open_end = has && nr <= nrt && rowstart[nr] > E0 + 32;   // the last row continues in the next lane's run
        const bool cut = Et < E0 + 32;                     // the tile ends inside the run
        const uint32_t wmask = __reduce_or_sync(0xffffffffu, bmask);
        float2 hsum = make_float2(0.f, 0.f), sum = make_float2(0.f, 0.f);
        bool in_head = true;
#pragma unroll
        for (int tt = 0; tt < 32; ++tt) {
          if (wmask & (1u << tt)) {                        // warp-uniform: some lane's run has a row start at tt
            const bool here = (bmask >> tt) & 1u;          // this lane leaves row `cur`
            if (here && !in_head) put(cur, sum);
            hsum = here && in_head ? sum : hsum;
            sum = here ? make_float2(0.f, 0.f) : sum;
            in_head = in_head && !here;
            cur += here ? 1 : 0;
          }
          const float2 ed = emds[E0 + tt];
          const float2 u = ffma2(make_float2(d[(tt >> 1) * 4 + (tt & 1)], d[(tt >> 1) * 4 + 2 + (tt & 1)]),
                                 make_float2(ed.y, ed.y), bias);
          const float2 v = fmul2(usig2(u), make_float2(ed.x, ed.x));
          sum = fadd2(sum, v);
        }
        if (in_head) hsum = sum;
        const float2 lsum = sum;                           // the row open at the run's end (unless `cut`)
        // carry across the quad in lane order (fixed order: deterministic)
        const bool cont_in = has && rowstart[hrow] < E0;   // this run's first row started in an earlier lane
        float2 cin = (q == 0 && nrt == 1 && !first_chunk) ? run : make_float2(0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float2 cout = in_head ? fadd2(cin, hsum) : lsum;
          const float px = __shfl_up_sync(0xffffffffu, cout.x, 1, 4), py = __shfl_up_sync(0xffffffffu, cout.y, 1, 4);
          if (q == k + 1 && cont_in) cin = make_float2(px, py);
        }
        const float2 htot = fadd2(cin, hsum);
        if (nrt == 1) {                                    // one row: its tile total ends in the lane holding edge Et - 1
          const int src = (lane & ~3) | ((Et - 1) >> 5);
          run = make_float2(__shfl_sync(0xffffffffu, htot.x, src), __shfl_sync(0xffffffffu, htot.y, src));
        }
        if (has && last_chunk) {
          if (!in_head || !open_end) put(hrow, htot);     // the first row ends in this run (egnn.py:312-313)
          if (!in_head && !open_end && !cut) put(cur, lsum);   // so does the last one, unless the tile end closed it above
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bars + BAR_TEMPTY + 8 * acc);
      } else {
        // Thread = edges (r0, r0 + 8) x channels 8j + 2q + {0, 1}: phi_e = sum_c silu(D descale + b2) w5 (coord_mlp.2 + .4)
        const float2 eda = emds[min(r0, Et - 1)], edb = emds[min(r0 + 8, Et - 1)];
        float2 pa = make_float2(0.f, 0.f), pb = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float2 w0 = b2w5[8 * j + 2 * q], w1 = b2w5[8 * j + 2 * q + 1];
          const float2 va = ffma2(make_float2(d[4 * j], d[4 * j + 1]), make_float2(eda.y, eda.y), make_float2(w0.x, w1.x));
          const float2 vb = ffma2(make_float2(d[4 * j + 2], d[4 * j + 3]), make_float2(edb.y, edb.y), make_float2(w0.x, w1.x));
          pa = ffma2(silu2(va), make_float2(w0.y, w1.y), pa);
          pb = ffma2(silu2(vb), make_float2(w0.y, w1.y), pb);
        }
        float phia = pa.x + pa.y, phib = pb.x + pb.y;
        phia += __shfl_xor_sync(0xffffffffu, phia, 1); phib += __shfl_xor_sync(0xffffffffu, phib, 1);
        phia += __shfl_xor_sync(0xffffffffu, phia, 2); phib += __shfl_xor_sync(0xffffffffu, phib, 2);
        const float* cds = reinterpret_cast<const float*>(tb + TBL_CD);
        if constexpr (TANH) {                              // egnn.py:104-109, evaluated left to right
          const float range = a.coords_range;
          if (q == 0 && r0 < Et) {
            const float th = tanhf(phia);
#pragma unroll
            for (int k = 0; k < 3; ++k) txs[r0 * 3 + k] = cds[r0 * 3 + k] * th * range * eda.x;
          }
          if (q == 0 && r0 + 8 < Et) {
            const int e = r0 + 8;
            const float th = tanhf(phib);
#pragma unroll
            for (int k = 0; k < 3; ++k) txs[e * 3 + k] = cds[e * 3 + k] * th * range * edb.x;
          }
        } else {
          if (q == 0 && r0 < Et) {                         // egnn.py:107-109
            const float w = phia * eda.x;
            txs[r0 * 3 + 0] = cds[r0 * 3 + 0] * w; txs[r0 * 3 + 1] = cds[r0 * 3 + 1] * w; txs[r0 * 3 + 2] = cds[r0 * 3 + 2] * w;
          }
          if (q == 0 && r0 + 8 < Et) {
            const int e = r0 + 8;
            const float w = phib * edb.x;
            txs[e * 3 + 0] = cds[e * 3 + 0] * w; txs[e * 3 + 1] = cds[e * 3 + 1] * w; txs[e * 3 + 2] = cds[e * 3 + 2] * w;
          }
        }
        named_sync(2, 32 * N_EPI_WARPS);                   // both warpgroups: txs complete
        if (tid < nrt * 3) {
          const int rr = tid / 3, dim = tid - rr * 3;
          float sacc = (nrt == 1 && !first_chunk) ? run3 : 0.f;
          const int col0 = rowstart[rr];
          const int ncc = rowstart[rr + 1] - col0;
          for (int jj = 0; jj < ncc; ++jj) sacc += txs[(col0 + jj) * 3 + dim];
          if (nrt == 1) run3 = sacc;
          if (last_chunk) {
            const int i = rownode[rr];
            const float lm = a.linker_mask ? a.linker_mask[gb + i] : 1.f;
            const float xv = a.x[(gb + i) * 3 + dim];
            float div = gm.normalization_factor;
            if constexpr (MEAN) div = SPARSE ? (float)(hdr[6] > 0 ? hdr[6] : ncc) : (float)N;
            const float xn = (xv + (sacc / div) * lm) * a.nm[gb + i];                 // egnn.py:110-124
            a.x_out[(gb + i) * 3 + dim] = xn;
            reinterpret_cast<float*>(a.x4_out + gb + i)[dim] = xn;
          }
        }
        named_sync(2, 32 * N_EPI_WARPS);                   // txs and the table slot may be reused
        if (lane == 0) mbar_arrive(bars + BAR_TEMPTY + 8 * acc);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------------------
template <typename K>
inline bool opt_in_smem(K kern) {
  return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) == cudaSuccess;
}
constexpr int OPT_ALL = OPT_TANH | OPT_MEAN | OPT_SIN;
// The instantiations of one (COORD, SPARSE) pair, walked at compile time: every OPT, OPT_TANH only for the coordinate update.
template <bool COORD, bool SPARSE, int OPT = 0>
inline bool opt_in_all() {
  if constexpr (OPT > OPT_ALL) {
    return true;
  } else {
    if constexpr (COORD || !(OPT & OPT_TANH))
      if (!opt_in_smem(k_edge_tc<COORD, SPARSE, OPT>)) return false;
    return opt_in_all<COORD, SPARSE, OPT + 1>();
  }
}
inline dl_status configure() {
  const bool ok = opt_in_all<true, false>() && opt_in_all<true, true>() && opt_in_all<false, false>() && opt_in_all<false, true>();
  return ok ? DL_OK : DL_ERR_CUDA;
}

// Log2-domain first layer (tensor-core path): the node kernel's projection weights, b1, wd and w0 are pre-multiplied by
// -log2(e) (dl_finalize_weights), so the producers form u = -log2(e) * pre directly and s' = u / (1 + 2^u) =
// -log2(e) * silu(pre) costs no scaling multiply; the -ln(2) that undoes it is folded into this operand
// (W2' = -ln2 * W2, computed in double before the fp16 hi/lo split).
constexpr double NEG_LN2 = -0.6931471805599453094;
constexpr double NEG_LOG2E = -1.4426950408889634074;

// edge_mlp.2 / coord_mlp.2 weight (out=128, in=128, row-major) -> [hi|lo][kc][out][8] fp16, scaled by the power of
// two that puts max|W| in [2^13, 2^14). Returns the offset (in halves) inside `blob`; *descale = 1/scale.
inline size_t pack_w2(const std::vector<float>& W_in, std::vector<__half>& blob, float* descale) {
  std::vector<float> W(W_in.size());
  for (size_t i = 0; i < W.size(); ++i) W[i] = (float)((double)W_in[i] * NEG_LN2);
  while (blob.size() % 64) blob.push_back(__float2half(0.f));           // keep 128-byte alignment for the bulk copy
  const size_t off = blob.size();
  blob.resize(off + 2 * (size_t)KC * H * 8);
  float mx = 0.f;
  for (float v : W) mx = std::max(mx, std::fabs(v));
  int ex = 0;
  if (mx > 0.f && std::isfinite(mx)) { std::frexp(mx, &ex); ex -= 1; }   // mx in [2^ex, 2^(ex+1))
  const int sh = std::min(std::max(13 - ex, -40), 40);
  const float scale = std::ldexp(1.0f, sh);
  *descale = std::ldexp(1.0f, -sh);
  for (int kc = 0; kc < KC; ++kc)
    for (int c = 0; c < H; ++c)
      for (int u = 0; u < 8; ++u) {
        const float v = W[(size_t)c * H + kc * 8 + u] * scale;
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        blob[off + ((size_t)kc * H + c) * 8 + u] = hi;
        blob[off + (size_t)KC * H * 8 + ((size_t)kc * H + c) * 8 + u] = lo;
      }
  return off;
}

template <bool COORD, bool SPARSE, int OPT = 0>
inline void launch_opt(int opt, const Geom& gm, const EdgeArgs& ea, const __half* w, int num_sms, cudaStream_t st) {
  if constexpr (OPT <= OPT_ALL) {
    if constexpr (COORD || !(OPT & OPT_TANH))
      if (opt == OPT) { k_edge_tc<COORD, SPARSE, OPT><<<num_sms, EDGE_TC_THREADS, SMEM_BYTES, st>>>(gm, ea, w); return; }
    launch_opt<COORD, SPARSE, OPT + 1>(opt, gm, ea, w, num_sms, st);
  }
}

// opt: the OPT bits of this launch (OPT_TANH only for the coordinate update). Cut-off graphs always come with the
// neighbour-list records (ea.recs), so OPT_MEAN's FC divisor N is right whenever SPARSE is false.
inline dl_status launch_edge_tc(const Geom& gm, const EdgeArgs& ea, bool coord, int opt, const void* w2_tc, int num_sms,
                                cudaStream_t st) {
  if (!coord && (opt & OPT_TANH)) return DL_ERR_INVALID;
  if (ea.recs == nullptr && gm.graph_type != 0 && (opt & OPT_MEAN)) return DL_ERR_INVALID;
  const __half* w = reinterpret_cast<const __half*>(w2_tc);
  if (ea.recs != nullptr) {
    if (coord) launch_opt<true, true>(opt, gm, ea, w, num_sms, st);
    else launch_opt<false, true>(opt, gm, ea, w, num_sms, st);
  } else if (coord) launch_opt<true, false>(opt, gm, ea, w, num_sms, st);
  else launch_opt<false, false>(opt, gm, ea, w, num_sms, st);
  return DL_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Self test: one 128 x 256 x 128 3xFP16 wgmma chain against a CPU fp64 result. Exercises descriptors, the
// canonical layouts and the accumulator fragment layout in isolation.
// ---------------------------------------------------------------------------------------------------------
constexpr int PN = 256;                          // probe: B operand rows (two wgmma N = 128 halves)
constexpr int P_LBO = PN * 16 + 16;
constexpr int P_OFF_BHI = 2 * W_BYTES, P_OFF_BLO = P_OFF_BHI + KC * P_LBO;
constexpr int P_SMEM_BYTES = P_OFF_BLO + KC * P_LBO + 1024;
// B_MN = true: the B operand is laid out MN-major (canonical no-swizzle form ((8,n),(8,k)):((1,SBO),(8,LBO)) in halves: 8
// consecutive N-rows of one k are contiguous 16 bytes; the transpose-B immediate of wgmma set).
template <bool B_MN>
__global__ void __launch_bounds__(256, 1) k_wgmma_probe(const __half* __restrict__ A /*[2][kc][128][8]*/,
                                                        const __half* __restrict__ Bm /*[2][kc][256][8]*/,
                                                        float* __restrict__ D /*[128][256]*/) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const uint32_t sbase = smem_u32(sm);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // A -> W slots (pitch W_LBO), B -> activation slots (pitch P_LBO) with ordinary stores
  for (int idx = tid; idx < 2 * KC * H; idx += 256) {
    const int copy = idx / (KC * H), rem = idx % (KC * H), kcx = rem / H, row = rem % H;
    *reinterpret_cast<uint4*>(sm + (copy ? OFF_WLO : OFF_WHI) + kcx * W_LBO + row * 16) =
        *reinterpret_cast<const uint4*>(A + (size_t)idx * 8);
  }
  constexpr int MN_LBO = (PN / 8) * 128;             // MN-major: pitch between 8-deep K groups; SBO = 128 B between 8-wide N groups
  for (int idx = tid; idx < 2 * KC * PN; idx += 256) {
    const int copy = idx / (KC * PN), rem = idx % (KC * PN), kcx = rem / PN, row = rem % PN;
    if (!B_MN) {
      *reinterpret_cast<uint4*>(sm + (copy ? P_OFF_BLO : P_OFF_BHI) + kcx * P_LBO + row * 16) =
          *reinterpret_cast<const uint4*>(Bm + (size_t)idx * 8);
    } else {
      for (int u = 0; u < 8; ++u)                      // element (n = row, k = kcx*8 + u)
        *reinterpret_cast<__half*>(sm + (copy ? P_OFF_BLO : P_OFF_BHI) + kcx * MN_LBO + (row >> 3) * 128 + u * 16 + (row & 7) * 2) =
            Bm[(size_t)idx * 8 + u];
    }
  }
  fence_proxy_async();
  __syncthreads();
  const int g = warp >> 2;
  const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2), q = lane & 3;
  float d[64];
  for (int nh = 0; nh < 2; ++nh) {
    const uint32_t bhi = sbase + P_OFF_BHI + nh * (B_MN ? 16 * 128 : 128 * 16), blo = bhi + (P_OFF_BLO - P_OFF_BHI);
    if (B_MN)
      gemm_3xf16<1>(d, sbase + OFF_WHI + g * 1024, sbase + OFF_WLO + g * 1024, W_LBO, bhi, blo, MN_LBO, 2 * MN_LBO, 8, false);
    else
      gemm_3xf16<0>(d, sbase + OFF_WHI + g * 1024, sbase + OFF_WLO + g * 1024, W_LBO, bhi, blo, P_LBO, 2 * P_LBO, 8, false);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = nh * 128 + 8 * j + 2 * q;
      D[(size_t)r0 * PN + col] = d[4 * j]; D[(size_t)r0 * PN + col + 1] = d[4 * j + 1];
      D[(size_t)(r0 + 8) * PN + col] = d[4 * j + 2]; D[(size_t)(r0 + 8) * PN + col + 1] = d[4 * j + 3];
    }
  }
}

inline dl_status selftest(int /*num_sms*/, float* max_abs_err, float* max_rel_err, bool b_mn_major = false) {
  std::vector<float> A((size_t)H * H), Bv((size_t)PN * H);
  uint32_t s = 12345u;
  auto rnd = [&]() { s = s * 1664525u + 1013904223u; return ((s >> 8) & 0xFFFF) / 65536.0f - 0.5f; };
  for (auto& v : A) v = rnd() * 0.2f;
  for (auto& v : Bv) v = rnd() * 3.0f;
  auto pack = [&](const std::vector<float>& M, int rows) {
    std::vector<__half> out(2 * (size_t)KC * rows * 8);
    for (int kc = 0; kc < KC; ++kc)
      for (int r = 0; r < rows; ++r)
        for (int u = 0; u < 8; ++u) {
          const float v = M[(size_t)r * H + kc * 8 + u];
          const __half hi = __float2half_rn(v);
          out[((size_t)kc * rows + r) * 8 + u] = hi;
          out[(size_t)KC * rows * 8 + ((size_t)kc * rows + r) * 8 + u] = __float2half_rn(v - __half2float(hi));
        }
    return out;
  };
  std::vector<__half> Ap = pack(A, H), Bp = pack(Bv, PN);
  __half *dA = nullptr, *dB = nullptr;
  float* dD = nullptr;
  if (cudaMalloc(&dA, Ap.size() * 2) != cudaSuccess || cudaMalloc(&dB, Bp.size() * 2) != cudaSuccess ||
      cudaMalloc(&dD, (size_t)H * PN * 4) != cudaSuccess)
    return DL_ERR_CUDA;
  cudaMemcpy(dA, Ap.data(), Ap.size() * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(dB, Bp.data(), Bp.size() * 2, cudaMemcpyHostToDevice);
  cudaMemset(dD, 0, (size_t)H * PN * 4);
  if (b_mn_major) {
    cudaFuncSetAttribute(k_wgmma_probe<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM_BYTES);
    k_wgmma_probe<true><<<1, 256, P_SMEM_BYTES>>>(dA, dB, dD);
  } else {
    cudaFuncSetAttribute(k_wgmma_probe<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, P_SMEM_BYTES);
    k_wgmma_probe<false><<<1, 256, P_SMEM_BYTES>>>(dA, dB, dD);
  }
  cudaError_t err = cudaDeviceSynchronize();
  std::vector<float> D((size_t)H * PN);
  cudaMemcpy(D.data(), dD, D.size() * 4, cudaMemcpyDeviceToHost);
  cudaFree(dA); cudaFree(dB); cudaFree(dD);
  if (err != cudaSuccess) {
    fprintf(stderr, "[dl selftest] k_wgmma_probe failed: %s\n", cudaGetErrorString(err));
    return DL_ERR_CUDA;
  }
  double ma = 0, mr = 0, mref = 0;
  for (int m = 0; m < H; ++m)
    for (int n = 0; n < PN; ++n) {
      double ref = 0;
      for (int k = 0; k < H; ++k) ref += (double)A[(size_t)m * H + k] * (double)Bv[(size_t)n * H + k];
      ma = std::max(ma, std::fabs(ref - (double)D[(size_t)m * PN + n]));
      mref = std::max(mref, std::fabs(ref));
    }
  mr = ma / std::max(mref, 1e-30);
  if (max_abs_err) *max_abs_err = (float)ma;
  if (max_rel_err) *max_rel_err = (float)mr;
  fprintf(stderr, "[dl selftest] 3xFP16 wgmma 128x256x128 (B %s-major): max abs err %.3e (rel to max |ref| %.3e)\n",
          b_mn_major ? "MN" : "K", ma, mr);
  return DL_OK;
}

}  // namespace tc
}  // namespace dl
