// SizeGNN at hidden_nf = 256: the width of the reference README's size-model recipe (train_size_gnn.py --hidden_nf 256
// --n_layers 5). Same arithmetic as the 128-wide SizeGNN path of kernels_simt.cuh (fp32 SIMT, ReLU, radial < 6 in torch's
// rounding order, fixed-order segment sums without atomics), in kernels of their own so that the denoiser's k_prep /
// k_node / k_edge_simt stay exactly as they are:
//   k_szw_prep -> [k_szw_edge -> k_szw_node] x n_layers -> k_szw_out
// The 128-wide edge kernel keeps all of W2 (64 KB) and a 128-edge tile of first-layer activations in shared memory. At 256
// W2 alone is 256 KB, past the 227 KB a CTA can have, so k_szw_edge splits the work (DESIGN.md section 6, "SizeGNN at hidden_nf 256"):
//   - the 256 output channels are two halves of 128, one after the other on the same tile;
//   - each half streams K = 256 in four slabs of 64: the slab's 64 x 128 block of W2, the slab's B columns of the tile's
//     live columns, and the first layer recomputed on that slab (one add and one FMA per element, next to the 128 FMAs
//     of the GEMM per element), so no (256 x 128-edge) activation tile is ever held.
// The work plan, tile shape (128 edges = whole rows, <= 8 rows, or one row in 128-column chunks) and the order of every
// segment sum are the 128-wide kernel's.
#pragma once
#include "kernels_simt.cuh"

namespace dl {
namespace szw {

constexpr int W = 256;             // hidden_nf
constexpr int HALF = W / 2;        // output channels per pass of the edge kernel
constexpr int TM = 32;             // nodes per CTA of the node-level kernels (warp w: nodes 4w..4w+3)
constexpr int LDW = W + 4;         // node-kernel smem row stride (floats), keeps float4 alignment
constexpr int KS = 64;             // K slab of the edge kernel
constexpr int LDBS = KS + 1;       // Bs slab row stride (bank-conflict-free column walks)
constexpr int NODE_SMEM = 3 * TM * LDW * (int)sizeof(float);
constexpr int EDGE_SMEM =
    (int)sizeof(float) * (KS * ET /*S1 slab*/ + KS * HALF /*W2 slab*/ + ET * LDBS /*Bs slab*/ + MAXR * W /*As*/ +
                          2 * W /*b2, wd*/ + 2 * ET /*ems, ds*/);
static_assert(KS * ET + KS * HALF >= ET * HALF, "the output tile reuses the S1 and W2 slabs");

__device__ __forceinline__ void zero8(float (&acc)[4][8]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[r][c] = 0.f;
}

// acc[r][0..3] += xs[r][0:K] . Wt[0:K][lane*4 .. +3], acc[r][4..7] += ... Wt[0:K][128 + lane*4 .. +3]; Wt is k-major [K][256]
template <int K>
__device__ __forceinline__ void warp_gemm(const float* __restrict__ xs, const float* __restrict__ Wt, int lane,
                                          float (&acc)[4][8]) {
#pragma unroll 2
  for (int k = 0; k < K; k += 4) {
    float4 w[4][2], x[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      w[q][0] = __ldg(reinterpret_cast<const float4*>(Wt + (size_t)(k + q) * W + lane * 4));
      w[q][1] = __ldg(reinterpret_cast<const float4*>(Wt + (size_t)(k + q) * W + HALF + lane * 4));
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) x[r] = *reinterpret_cast<const float4*>(xs + r * LDW + k);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float xv[4] = {x[r].x, x[r].y, x[r].z, x[r].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          acc[r][4 * hh + 0] = fmaf(xv[q], w[q][hh].x, acc[r][4 * hh + 0]);
          acc[r][4 * hh + 1] = fmaf(xv[q], w[q][hh].y, acc[r][4 * hh + 1]);
          acc[r][4 * hh + 2] = fmaf(xv[q], w[q][hh].z, acc[r][4 * hh + 2]);
          acc[r][4 * hh + 3] = fmaf(xv[q], w[q][hh].w, acc[r][4 * hh + 3]);
        }
      }
    }
  }
}

// the lane's two float4 channel groups of a 256-wide row: [lane*4, +4) and [128 + lane*4, +4)
__device__ __forceinline__ void store_row(float* row, int lane, const float (&o)[8]) {
  *reinterpret_cast<float4*>(row + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
  *reinterpret_cast<float4*>(row + HALF + lane * 4) = make_float4(o[4], o[5], o[6], o[7]);
}
__device__ __forceinline__ void load_row(const float* row, int lane, float (&o)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(row + lane * 4);
  const float4 b = *reinterpret_cast<const float4*>(row + HALF + lane * 4);
  o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}

// AB[g] = [h W1a^T + b1 | h W1b^T] (B*N, 512): the first Linear of the next edge MLP split per node (as project_ab).
__device__ __forceinline__ void project(const float* hs_warp, const ProjW& pw, float* __restrict__ AB, int g0, int n_total,
                                        int warp, int lane) {
  float acc[4][8];
  zero8(acc);
  warp_gemm<W>(hs_warp, pw.W1a_t, lane, acc);
  float bb[8];
  load_row(pw.b1, lane, bb);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int g = g0 + warp * 4 + r;
    float o[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) o[c] = acc[r][c] + bb[c];
    if (g < n_total) store_row(AB + (size_t)g * 2 * W, lane, o);
  }
  zero8(acc);
  warp_gemm<W>(hs_warp, pw.W1b_t, lane, acc);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int g = g0 + warp * 4 + r;
    if (g < n_total) store_row(AB + (size_t)g * 2 * W + W, lane, acc[r]);
  }
}

// SizeGNN.forward prologue (linker_size.py:85-87): x0 = positions * fragment_mask, h = embedding_in(one_hot * fragment_mask)
// (every row, masked ones included: they hold the bias), nm = fragment_mask, then the first GCL's projections.
struct PrepArgsW {
  const float* xh;          // (B*N, 3+F)
  const int8_t* node_mask;  // (B*N) fragment mask
  const float* We_t;        // [F][256]
  const float* be;          // [256]
  ProjW proj;
  float* nm;                // out (B*N)
  float* x0;                // out (B*N,3)
  float* h;                 // out (B*N,256)
  float* AB;                // out (B*N,512)
};

__global__ void __launch_bounds__(256) k_szw_prep(Geom gm, PrepArgsW a) {
  __shared__ __align__(16) float hs[TM * LDW];
  __shared__ float hin[TM][MAX_DIN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_total = gm.B * gm.N;
  const int g0 = blockIdx.x * TM;
  const int xd = 3 + gm.F;
  for (int idx = tid; idx < TM * MAX_DIN; idx += 256) {
    const int r = idx / MAX_DIN, d = idx % MAX_DIN, g = g0 + r;
    hin[r][d] = (g < n_total && d < gm.F) ? a.xh[(size_t)g * xd + 3 + d] * (float)a.node_mask[g] : 0.f;
  }
  if (tid < TM) {
    const int g = g0 + tid;
    if (g < n_total) {
      const float m = (float)a.node_mask[g];
      a.nm[g] = m;
      for (int d = 0; d < 3; ++d) a.x0[(size_t)g * 3 + d] = a.xh[(size_t)g * xd + d] * m;
    }
  }
  __syncthreads();
  float acc[4][8];
  zero8(acc);
  for (int d = 0; d < gm.F; ++d) {
    float w[8];
    load_row(a.We_t + (size_t)d * W, lane, w);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float xv = hin[warp * 4 + r][d];
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = fmaf(xv, w[c], acc[r][c]);
    }
  }
  float bb[8];
  load_row(a.be, lane, bb);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    float o[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) o[c] = acc[r][c] + bb[c];
    store_row(hs + (warp * 4 + r) * LDW, lane, o);
    const int g = g0 + warp * 4 + r;
    if (g < n_total) store_row(a.h + (size_t)g * W, lane, o);
  }
  __syncwarp();
  project(hs + warp * 4 * LDW, a.proj, a.AB, g0, n_total, warp, lane);
}

// GCL.node_model + node_mask (egnn.py:62-80): h = (h + W4 relu(W3 [h, agg] + b3) + b4) * nm, eval-mode batch norm folded
// into W3/b3 and W4/b4 on the host; then the next GCL's projections (proj1 / AB1; AB1 == nullptr after the last layer).
__global__ void __launch_bounds__(256) k_szw_node(int n_total, NodeArgs a) {
  extern __shared__ __align__(16) float sm_szw_node[];
  float* hs = sm_szw_node;                 // [32][LDW]
  float* as = hs + TM * LDW;               // [32][LDW]
  float* hid = as + TM * LDW;              // [32][LDW]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g0 = blockIdx.x * TM;
#pragma unroll
  for (int r = 0; r < 4; ++r) {              // each warp loads and later reads only its own 4 rows
    const int row = warp * 4 + r, g = g0 + row;
    float hv[8] = {0, 0, 0, 0, 0, 0, 0, 0}, av[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (g < n_total) { load_row(a.h + (size_t)g * W, lane, hv); load_row(a.agg + (size_t)g * W, lane, av); }
    store_row(hs + row * LDW, lane, hv);
    store_row(as + row * LDW, lane, av);
  }
  __syncwarp();
  float acc[4][8];
  zero8(acc);
  warp_gemm<W>(hs + warp * 4 * LDW, a.W3_t, lane, acc);
  warp_gemm<W>(as + warp * 4 * LDW, a.W3_t + (size_t)W * W, lane, acc);
  {
    float bb[8];
    load_row(a.b3, lane, bb);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float o[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) o[c] = fmaxf(acc[r][c] + bb[c], 0.f);
      store_row(hid + (warp * 4 + r) * LDW, lane, o);
    }
  }
  __syncwarp();
  zero8(acc);
  warp_gemm<W>(hid + warp * 4 * LDW, a.W4_t, lane, acc);
  {
    float bb[8];
    load_row(a.b4, lane, bb);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int row = warp * 4 + r, g = g0 + row;
      const float m = g < n_total ? a.nm[g] : 0.f;
      float hv[8], o[8];
      load_row(hs + row * LDW, lane, hv);
#pragma unroll
      for (int c = 0; c < 8; ++c) o[c] = (hv[c] + (acc[r][c] + bb[c])) * m;
      __syncwarp();
      store_row(hs + row * LDW, lane, o);
      if (g < n_total) store_row(a.h + (size_t)g * W, lane, o);
    }
  }
  __syncwarp();
  if (a.AB1 != nullptr) project(hs + warp * 4 * LDW, a.proj1, a.AB1, g0, n_total, warp, lane);
}

// GCL edge model + aggregation (egnn.py:45-66 with ReLU, linker_size.py:53-83):
//   agg_i = sum_j relu(W2 relu(A_i + B_j + d_ij wd) + b2) * [edge_mask_ij != 0 and d_ij < 6]
// with A, B from AB (b1 folded into A) and d_ij the squared distance in torch's rounding order (radial_rn).
// Reads a.AB (B*N,512), a.x0, a.edge_mask, a.W2_t ([256][256] k-major), a.b2, a.wd, a.plan; writes a.agg (B*N,256) for
// every live row. One work item of the plan at a time, per CTA (persistent grid).
__global__ void __launch_bounds__(256, 2) k_szw_edge(Geom gm, EdgeArgs a) {
  extern __shared__ __align__(16) float sm_szw_edge[];
  float* S1 = sm_szw_edge;                 // [KS][ET]   first-layer activations of the slab
  float* W2s = S1 + KS * ET;               // [KS][HALF] the slab's block of W2 for the current half
  float* Outs = S1;                        // [ET][HALF] messages of the half (overlays S1 and W2s after the GEMM)
  float* Bs = W2s + KS * HALF;             // [ET][LDBS] the slab's B columns of the tile's live columns
  float* As = Bs + ET * LDBS;              // [MAXR][W]  A of the tile's rows
  float* b2s = As + MAXR * W;
  float* wds = b2s + W;
  float* ems = wds + W;                    // [ET] edge weight 0/1
  float* ds = ems + ET;                    // [ET] squared distance

  const int tid = threadIdx.x;
  const int N = gm.N;
  for (int k = tid; k < W; k += 256) { b2s[k] = a.b2[k]; wds[k] = a.wd[k]; }

  const int n_work = *a.plan.n_items;
  for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
    const int4 it = a.plan.items[wi];
    const int b = it.x, r_begin = it.y, r_count = it.z;
    const int nc = a.plan.nc[b];
    const int* rows = a.plan.rowidx + (size_t)b * N;
    const int* cols = a.plan.colidx + (size_t)b * N;
    const size_t gb = (size_t)b * N;
    const int8_t* em_mol = a.edge_mask ? a.edge_mask + gb * N : nullptr;
    int per = nc >= ET ? 1 : ET / nc;
    if (per > MAXR) per = MAXR;

    for (int rt = 0; rt < r_count; rt += per) {           // row groups (the plan's items hold exactly one)
      const int nrt = min(per, r_count - rt);
      __syncthreads();                                     // previous group's As no longer read
      for (int idx = tid; idx < nrt * (W / 4); idx += 256) {
        const int r = idx / (W / 4), k4 = idx - r * (W / 4);
        reinterpret_cast<float4*>(As + r * W)[k4] =
            reinterpret_cast<const float4*>(a.AB + (gb + rows[r_begin + rt + r]) * 2 * W)[k4];
      }
      float run = 0.f;                                     // one-row tiles: running sum of channel tid across chunks
      for (int c0 = 0; c0 < nc; c0 += ET) {
        const int ncc = min(ET, nc - c0);
        const int Et = nrt * ncc;
        __syncthreads();                                   // previous chunk's segment sum done
        if (tid < ET) {
          const int e = tid;
          float w = 0.f, d = 0.f;
          if (e < Et) {
            const int rr = e / ncc, jj = e - rr * ncc;
            const int i = rows[r_begin + rt + rr], j = cols[c0 + jj];
            const float* xi = a.x0 + (gb + i) * 3; const float* xj = a.x0 + (gb + j) * 3;
            d = radial_rn(xi[0] - xj[0], xi[1] - xj[1], xi[2] - xj[2]);
            w = edge_weight(4, em_mol, N, i, j, 0, 0, d);
          }
          ems[e] = w; ds[e] = d;
        }
        for (int oh = 0; oh < 2; ++oh) {                   // output channels [oh*128, oh*128 + 128)
          const int ty = tid >> 4, tx = tid & 15;
          float acc[8][8];
#pragma unroll
          for (int p = 0; p < 8; ++p)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[p][q] = 0.f;
          for (int ks = 0; ks < W; ks += KS) {
            __syncthreads();                               // previous slab's GEMM / previous half's segment sum done
            for (int idx = tid; idx < ncc * KS; idx += 256) {
              const int jj = idx / KS, k = idx - jj * KS;
              Bs[jj * LDBS + k] = a.AB[(gb + cols[c0 + jj]) * 2 * W + W + ks + k];
            }
            for (int idx = tid; idx < KS * HALF / 4; idx += 256) {
              const int k = idx / (HALF / 4), c4 = idx - k * (HALF / 4);
              reinterpret_cast<float4*>(W2s + k * HALF)[c4] =
                  __ldg(reinterpret_cast<const float4*>(a.W2_t + (size_t)(ks + k) * W + oh * HALF) + c4);
            }
            __syncthreads();
            {                                              // first layer + ReLU on the slab -> S1[k][e]
              const int e = tid & (ET - 1), kh = tid >> 7;
              const bool valid = e < Et;
              const int rr = valid ? e / ncc : 0, jj = valid ? e - rr * ncc : 0;
              const float d = ds[e];
              const float* Ar = As + rr * W + ks;
              const float* Br = Bs + jj * LDBS;
              const float* wk = wds + ks;
#pragma unroll 8
              for (int kk = 0; kk < KS / 2; ++kk) {
                const int k = kh * (KS / 2) + kk;
                const float pre = Ar[k] + Br[k] + d * wk[k];
                S1[k * ET + e] = valid ? fmaxf(pre, 0.f) : 0.f;
              }
            }
            __syncthreads();
#pragma unroll 4
            for (int k = 0; k < KS; ++k) {                 // 128 edges x 128 channels x 64, 8x8 register tile
              const float4 a0 = *reinterpret_cast<const float4*>(S1 + k * ET + ty * 4);
              const float4 a1 = *reinterpret_cast<const float4*>(S1 + k * ET + 64 + ty * 4);
              const float4 b0 = *reinterpret_cast<const float4*>(W2s + k * HALF + tx * 4);
              const float4 b1 = *reinterpret_cast<const float4*>(W2s + k * HALF + 64 + tx * 4);
              const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
              const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
              for (int p = 0; p < 8; ++p)
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[p][q] = fmaf(av[p], bv[q], acc[p][q]);
            }
          }
          __syncthreads();                                 // S1 and W2s no longer read -> Outs[e][c]
#pragma unroll
          for (int p = 0; p < 8; ++p) {
            const int e = p < 4 ? ty * 4 + p : 64 + ty * 4 + (p - 4);
            const float w = ems[e];
#pragma unroll
            for (int qh = 0; qh < 2; ++qh) {
              const int c = qh * 64 + tx * 4;
              const float* bb = b2s + oh * HALF + c;
              *reinterpret_cast<float4*>(Outs + e * HALF + c) =
                  make_float4(fmaxf(acc[p][qh * 4 + 0] + bb[0], 0.f) * w, fmaxf(acc[p][qh * 4 + 1] + bb[1], 0.f) * w,
                              fmaxf(acc[p][qh * 4 + 2] + bb[2], 0.f) * w, fmaxf(acc[p][qh * 4 + 3] + bb[3], 0.f) * w);
            }
          }
          __syncthreads();
          // segment sum over j in column order, thread = (row parity, channel); normalization_factor = 1
          const int c = tid & (HALF - 1);
          if (nc <= ET) {
            for (int rr = tid >> 7; rr < nrt; rr += 2) {
              float s = 0.f;
              for (int jj = 0; jj < ncc; ++jj) s += Outs[(rr * ncc + jj) * HALF + c];
              a.agg[(gb + rows[r_begin + rt + rr]) * W + oh * HALF + c] = s;
            }
          } else if ((tid >> 7) == oh) {
            for (int jj = 0; jj < ncc; ++jj) run += Outs[jj * HALF + c];
            if (c0 + ET >= nc) a.agg[(gb + rows[r_begin + rt]) * W + oh * HALF + c] = run;
          }
        }
      }
    }
  }
}

// SizeGNN head (linker_size.py:88-91 + linker_size_lightning.py:110): out[b] = mean over ALL N padded rows of
// embedding_out(h[b, n]), as k_sz_out: one CTA per molecule, warp per node (strided), per-warp sums combined in warp order.
__global__ void __launch_bounds__(256) k_szw_out(int N, int out_nf, const float* __restrict__ h, const float* __restrict__ Wo,
                                                const float* __restrict__ bo, float* __restrict__ out) {
  __shared__ float part[8][SZ_MAX_OUT];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int o = lane; o < out_nf; o += 32) part[warp][o] = 0.f;
  __syncwarp();
  for (int n = warp; n < N; n += 8) {
    float hv[8];
    load_row(h + ((size_t)b * N + n) * W, lane, hv);
    for (int o = 0; o < out_nf; ++o) {
      float w[8];
      load_row(Wo + (size_t)o * W, lane, w);
      float s = 0.f;
#pragma unroll
      for (int c = 0; c < 8; ++c) s = fmaf(hv[c], w[c], s);
#pragma unroll
      for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
      if (lane == 0) part[warp][o] += s + bo[o];
    }
  }
  __syncthreads();
  if (tid < out_nf) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += part[w][tid];
    out[(size_t)b * out_nf + tid] = s / (float)N;
  }
}

}  // namespace szw
}  // namespace dl
