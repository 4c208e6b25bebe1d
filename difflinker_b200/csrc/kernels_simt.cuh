// fp32 SIMT kernels of the DiffLinker hot path: work plan, node-level layers, reference edge kernel,
// output/z-update.  The tensor-core edge kernel (kernels_tc.cuh) replaces k_edge_simt on the product path;
// k_edge_simt stays as the on-device cross-check (dl_selftest_tc, DL_EDGE_SIMT).
#pragma once
#include <curand_kernel.h>

#include "common.cuh"

namespace dl {

// ------------------------------------------------------------------------------------------------
// Work plan
// ------------------------------------------------------------------------------------------------
// One CTA per molecule. Finds rows/columns of the (N x N) edge-weight matrix that carry any non-zero
// weight; everything else is skipped exactly (0 * finite == 0, DESIGN.md "masked work").
// FC graphs: weights are the caller's int8 edge_mask (datasets.py:365-369) or all ones when NULL.
// Pocket graphs: the weight is a per-step distance predicate, so every valid node is live.
__global__ void k_plan_mol(int N, int graph_type, const int8_t* __restrict__ edge_mask,
                           const int8_t* __restrict__ node_mask, const float* __restrict__ linker_mask,
                           int* __restrict__ rowidx, int* __restrict__ colidx, int* __restrict__ xrowidx,
                           int* __restrict__ nr, int* __restrict__ nc, int* __restrict__ nxr) {
  extern __shared__ int sm_plan[];
  int* rowlive = sm_plan;        // [N]
  int* collive = sm_plan + N;    // [N]
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  for (int i = tid; i < N; i += blockDim.x) { rowlive[i] = 0; collive[i] = 0; }
  __syncthreads();
  if ((graph_type == 0 || graph_type == 4) && edge_mask != nullptr) {
    const int8_t* em = edge_mask + (size_t)b * N * N;
    for (int i = warp; i < N; i += nwarp) {
      int any = 0;
      for (int j = lane; j < N; j += 32) {
        int v = em[(size_t)i * N + j];
        if (v != 0) { any = 1; collive[j] = 1; }
      }
      any = __any_sync(0xffffffffu, any);
      if (lane == 0 && any) rowlive[i] = 1;
    }
  } else if (graph_type == 0 || graph_type == 4) {
    for (int i = tid; i < N; i += blockDim.x) { rowlive[i] = 1; collive[i] = 1; }
  } else {
    for (int i = tid; i < N; i += blockDim.x) {
      int v = node_mask[(size_t)b * N + i] != 0;
      rowlive[i] = v; collive[i] = v;
    }
  }
  __syncthreads();
  if (tid == 0) {
    int a = 0, c = 0, x = 0;
    for (int i = 0; i < N; ++i) {
      if (rowlive[i]) {
        rowidx[(size_t)b * N + a++] = i;
        if (linker_mask == nullptr || linker_mask[(size_t)b * N + i] != 0.0f) xrowidx[(size_t)b * N + x++] = i;
      }
      if (collive[i]) colidx[(size_t)b * N + c++] = i;
    }
    nr[b] = a; nc[b] = c; nxr[b] = x;
  }
}

// Single thread: flatten per-molecule row groups into the GCL work list. A work item is `rows_per_tile`
// complete rows (so the segment sum over j never crosses CTAs and stays order-deterministic).
__global__ void k_plan_items(int B, int tile_edges, int max_rows, int col_pad, int max_rows_gcl, const int* __restrict__ nr,
                             const int* __restrict__ nc, const int* __restrict__ nxr, int4* __restrict__ items,
                             int* __restrict__ n_items, int* __restrict__ xmols, int* __restrict__ n_xmols,
                             int4* __restrict__ xitems, int* __restrict__ n_xitems, int n_cta = 0,
                             int* __restrict__ cta_begin = nullptr, int* __restrict__ xcta_begin = nullptr) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int cnt = 0, xc = 0, xi = 0;
  for (int b = 0; b < B; ++b) {
    int r = nr[b], c = nc[b];
    if (r > 0 && c > 0) {
      const int cp = (c + col_pad - 1) / col_pad * col_pad;   // rows padded to a multiple of col_pad columns
      int per = cp >= tile_edges ? 1 : tile_edges / cp;
      if (per > max_rows_gcl) per = max_rows_gcl;
      for (int r0 = 0; r0 < r; r0 += per) items[cnt++] = make_int4(b, r0, min(per, r - r0), c);
    }
    if (nxr[b] > 0 && c > 0) {
      xmols[xc++] = b;
      int per;
      if (col_pad > 1) {                                     // same rows-per-tile rule as the GCL tiles
        const int cp = (c + col_pad - 1) / col_pad * col_pad;
        per = cp >= tile_edges ? 1 : tile_edges / cp;
        if (per > max_rows_gcl) per = max_rows_gcl;
      } else {
        per = c >= tile_edges ? 1 : tile_edges / c;
        if (per > max_rows) per = max_rows;
      }
      for (int r0 = 0; r0 < nxr[b]; r0 += per) xitems[xi++] = make_int4(b, r0, min(per, nxr[b] - r0), c);
    }
  }
  *n_items = cnt;
  *n_xmols = xc;
  *n_xitems = xi;
  // optional: contiguous slices of the tile lists per CTA, balanced by cost (padded edges + a per-tile constant) instead of
  // by tile count -- single-row tiles at the end of a molecule cost a third of a full tile
  if (n_cta > 0 && cta_begin != nullptr) {
    for (int pass = 0; pass < 2; ++pass) {
      const int4* list = pass == 0 ? items : xitems;
      const int total = pass == 0 ? cnt : xi;
      int* out = pass == 0 ? cta_begin : xcta_begin;
      if (out == nullptr) continue;
      long long sum = 0;
      for (int k = 0; k < total; ++k) sum += (long long)list[k].z * ((list[k].w + col_pad - 1) / col_pad * col_pad) + 32;
      long long run = 0;
      int c = 0;
      out[0] = 0;
      for (int k = 0; k < total; ++k) {
        // CTA c ends before item k once its share is reached
        while (c + 1 < n_cta && run * n_cta >= (long long)(c + 1) * sum) out[++c] = k;
        run += (long long)list[k].z * ((list[k].w + col_pad - 1) / col_pad * col_pad) + 32;
      }
      while (c < n_cta) out[++c] = total;
    }
  }
}

// Activation of the fp32 SIMT kernels: SiLU for the denoiser (egnn.py:325), ReLU for SizeGNN (linker_size.py:60).
constexpr int ACT_SILU = 0, ACT_RELU = 1;
template <int ACT>
__device__ __forceinline__ float act_f(float x) { return ACT == ACT_RELU ? fmaxf(x, 0.f) : silu_f(x); }

// ------------------------------------------------------------------------------------------------
// Node-level SIMT tile GEMM: 32 nodes x 128 channels per CTA (256 threads).
// warp w owns nodes 4w..4w+3, lane owns channels 4*lane..4*lane+3.
// ------------------------------------------------------------------------------------------------
constexpr int NODE_TM = 32;
constexpr int LDX = 132;  // smem row stride (floats), keeps float4 alignment

template <int K>
__device__ __forceinline__ void warp_gemm_4x4(const float* __restrict__ xs, const float* __restrict__ Wt, int lane,
                                              float (&acc)[4][4]) {
#pragma unroll 2
  for (int k = 0; k < K; k += 4) {
    float4 w[4], x[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) w[q] = __ldg(reinterpret_cast<const float4*>(Wt + (size_t)(k + q) * H + lane * 4));
#pragma unroll
    for (int r = 0; r < 4; ++r) x[r] = *reinterpret_cast<const float4*>(xs + r * LDX + k);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const float xv[4] = {x[r].x, x[r].y, x[r].z, x[r].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        acc[r][0] = fmaf(xv[q], w[q].x, acc[r][0]);
        acc[r][1] = fmaf(xv[q], w[q].y, acc[r][1]);
        acc[r][2] = fmaf(xv[q], w[q].z, acc[r][2]);
        acc[r][3] = fmaf(xv[q], w[q].w, acc[r][3]);
      }
    }
  }
}

__device__ __forceinline__ void zero_acc(float (&acc)[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
}

// A = hs W1a^T + b1 -> AB[:, 0:128];  B = hs W1b^T -> AB[:, 128:256]   (first Linear of an edge MLP,
// split per SURVEY.md section 8(a) "verified restatement": egnn.py:45-50 / 103 with the concat distributed).
__device__ __forceinline__ float warp_absmax4(const float (&v)[4]) {
  float m = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  return m;
}

// ABmax[g] = (max_k |A[g][k]|, max_k |B[g][k]|): bounds the first-layer pre-activation of every edge, which the
// tensor-core path uses to pick an exact power-of-two scale that keeps its fp16 operands in range.
__device__ __forceinline__ void project_ab(const float* hs_warp, const ProjW& pw, float* __restrict__ AB,
                                           float* __restrict__ ABmax, int g0, int n_total, int warp, int lane) {
  float acc[4][4];
  zero_acc(acc);
  warp_gemm_4x4<H>(hs_warp, pw.W1a_t, lane, acc);
  const float4 bb = __ldg(reinterpret_cast<const float4*>(pw.b1 + lane * 4));
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int g = g0 + warp * 4 + r;
    const float o[4] = {acc[r][0] + bb.x, acc[r][1] + bb.y, acc[r][2] + bb.z, acc[r][3] + bb.w};
    const float mx = warp_absmax4(o);
    if (g < n_total) {
      *reinterpret_cast<float4*>(AB + (size_t)g * 2 * H + lane * 4) = make_float4(o[0], o[1], o[2], o[3]);
      if (lane == 0) ABmax[(size_t)g * 2] = mx;
    }
  }
  zero_acc(acc);
  warp_gemm_4x4<H>(hs_warp, pw.W1b_t, lane, acc);
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int g = g0 + warp * 4 + r;
    const float mx = warp_absmax4(acc[r]);
    if (g < n_total) {
      *reinterpret_cast<float4*>(AB + (size_t)g * 2 * H + H + lane * 4) =
          make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
      if (lane == 0) ABmax[(size_t)g * 2 + 1] = mx;
    }
  }
}

// Dynamics.forward prologue (egnn.py:387-407) + EGNN.embedding (egnn.py:224) + first projection.
//   nm = node_mask; x0 = xh[:, :3]*nm; h_in = [xh[:, 3:]*nm, t, context]; h = We h_in + be
// In sampler mode (step_ctr != nullptr) `xh` is the engine's z buffer and t comes from coef[step].
struct PrepArgs {
  const float* xh;          // (B*N, 3+F)
  const int8_t* node_mask;  // (B*N)
  const float* linker_mask; // (B*N) or null
  const float* t;           // (t_numel) or null in sampler mode
  int t_numel;
  const float* context;     // (B*N, C) or null
  const float* We_t;        // [D][128]
  const float* be;          // [128]
  ProjW proj;
  float* nm;                // out (B*N)
  float* x0;                // out (B*N,3)
  float* x;                 // out (B*N,3)
  float4* x04;              // out (B*N) padded copies (x0 | x) for 16-byte gathers in the tensor-core table warps; may be null
  float4* x4;
  int* cls;                 // out (B*N) node class for pocket graphs: 0 invalid, 1 ligand, 2 pocket
  float* h;                 // out (B*N,128)
  float* AB;                // out (B*N,256)
  float* ABmax;             // out (B*N,2)
  const float* coef;        // device dl_step_coef table (8 floats per row) or null
  const int* step_prep;     // device counter read here
  int* step_fin;            // device counter written here
};

__global__ void __launch_bounds__(256) k_prep(Geom gm, PrepArgs a) {
  __shared__ __align__(16) float hs[NODE_TM * LDX];
  __shared__ float hin[NODE_TM][MAX_DIN];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_total = gm.B * gm.N;
  const int g0 = blockIdx.x * NODE_TM;
  const int xd = 3 + gm.F;
  int step = 0;
  chain_wait();
  chain_release();
  if (a.step_prep != nullptr) {
    step = *a.step_prep;
    if (blockIdx.x == 0 && tid == 0) *a.step_fin = step;
  }
  for (int idx = tid; idx < NODE_TM * MAX_DIN; idx += 256) {
    int r = idx / MAX_DIN, d = idx % MAX_DIN;
    int g = g0 + r;
    float v = 0.f;
    if (g < n_total && d < gm.D) {
      float m = (float)a.node_mask[g];
      if (d < gm.F) {
        v = a.xh[(size_t)g * xd + 3 + d] * m;
      } else if (d == gm.F && gm.D > gm.F + gm.C) {  // time column (condition_time)
        if (a.coef != nullptr) v = a.coef[(size_t)step * 8 + 0];
        else v = a.t[a.t_numel == 1 ? 0 : g / gm.N];
      } else {
        int cidx = d - (gm.D - gm.C);
        v = a.context[(size_t)g * gm.C + cidx];
      }
    }
    hin[r][d] = v;
  }
  if (tid < NODE_TM) {
    int g = g0 + tid;
    if (g < n_total) {
      float m = (float)a.node_mask[g];
      a.nm[g] = m;
      for (int d = 0; d < 3; ++d) {
        float v = a.xh[(size_t)g * xd + d] * m;
        a.x0[(size_t)g * 3 + d] = v;
        a.x[(size_t)g * 3 + d] = v;
        if (a.x4 != nullptr) {
          reinterpret_cast<float*>(a.x04 + g)[d] = v;
          reinterpret_cast<float*>(a.x4 + g)[d] = v;
        }
      }
      if (gm.graph_type >= 1 && gm.graph_type <= 3) {
        // egnn.py:566-570: ligand = (linker | fragment_only) & valid ; pocket = pocket_only & valid
        int valid = m != 0.f;
        int pk = a.context[(size_t)g * gm.C + gm.C - 1] != 0.f;
        int fr = a.context[(size_t)g * gm.C + gm.C - 2] != 0.f;
        int lk = a.linker_mask != nullptr ? (a.linker_mask[g] != 0.f) : 0;
        int c = 0;
        if (valid) {
          if (gm.graph_type == 1) c = 1;  // '4A': a single class, one cut-off
          else c = (lk || fr) ? 1 : (pk ? 2 : 3);
        }
        a.cls[g] = c;
      }
    }
  }
  __syncthreads();
  // embedding: K = D (tiny) -> straight dot products
  {
    float acc[4][4];
    zero_acc(acc);
    for (int d = 0; d < gm.D; ++d) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(a.We_t + (size_t)d * H + lane * 4));
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        float xv = hin[warp * 4 + r][d];
        acc[r][0] = fmaf(xv, w.x, acc[r][0]);
        acc[r][1] = fmaf(xv, w.y, acc[r][1]);
        acc[r][2] = fmaf(xv, w.z, acc[r][2]);
        acc[r][3] = fmaf(xv, w.w, acc[r][3]);
      }
    }
    const float4 bb = __ldg(reinterpret_cast<const float4*>(a.be + lane * 4));
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float4 o = make_float4(acc[r][0] + bb.x, acc[r][1] + bb.y, acc[r][2] + bb.z, acc[r][3] + bb.w);
      *reinterpret_cast<float4*>(hs + (warp * 4 + r) * LDX + lane * 4) = o;
      int g = g0 + warp * 4 + r;
      if (g < n_total) *reinterpret_cast<float4*>(a.h + (size_t)g * H + lane * 4) = o;
    }
  }
  __syncwarp();
  // tensor-core path: the projection of the first edge MLP runs on the tensor cores right after (k_node_tc, proj_only)
  if (a.AB != nullptr) project_ab(hs + warp * 4 * LDX, a.proj, a.AB, a.ABmax, g0, n_total, warp, lane);
}

// GCL.node_model + node_mask (egnn.py:62-80), then the first-layer projections of whatever edge MLP
// consumes the new h next (the following GCL, and/or the block's coord_mlp + the next block's gcl_0).
struct NodeArgs {
  float* h;             // (B*N,128) in/out (rows are CTA-private)
  const float* agg;     // (B*N,128)  sum_j m_ij*EM_ij / normalization_factor
  const float* nm;      // (B*N)
  const float* W3_t; const float* b3; const float* W4_t; const float* b4;
  ProjW proj1; float* AB1; float* ABmax1;
  ProjW proj2; float* AB2; float* ABmax2;  // AB2 == nullptr -> skip
};

template <int ACT = ACT_SILU>
__global__ void __launch_bounds__(256) k_node(int n_total, NodeArgs a) {
  extern __shared__ __align__(16) float sm_node[];
  float* hs = sm_node;                    // [32][LDX]
  float* as = sm_node + NODE_TM * LDX;    // [32][LDX]
  float* hid = as + NODE_TM * LDX;        // [32][LDX]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g0 = blockIdx.x * NODE_TM;
  // each warp loads its own 4 rows (all later reads of those rows are by the same warp)
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    int row = warp * 4 + r, g = g0 + row;
    float4 hv = make_float4(0, 0, 0, 0), av = hv;
    if (g < n_total) {
      hv = *reinterpret_cast<const float4*>(a.h + (size_t)g * H + lane * 4);
      av = *reinterpret_cast<const float4*>(a.agg + (size_t)g * H + lane * 4);
    }
    *reinterpret_cast<float4*>(hs + row * LDX + lane * 4) = hv;
    *reinterpret_cast<float4*>(as + row * LDX + lane * 4) = av;
  }
  __syncwarp();
  float acc[4][4];
  zero_acc(acc);
  warp_gemm_4x4<H>(hs + warp * 4 * LDX, a.W3_t, lane, acc);
  warp_gemm_4x4<H>(as + warp * 4 * LDX, a.W3_t + (size_t)H * H, lane, acc);
  {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(a.b3 + lane * 4));
#pragma unroll
    for (int r = 0; r < 4; ++r)
      *reinterpret_cast<float4*>(hid + (warp * 4 + r) * LDX + lane * 4) =
          make_float4(act_f<ACT>(acc[r][0] + bb.x), act_f<ACT>(acc[r][1] + bb.y), act_f<ACT>(acc[r][2] + bb.z),
                      act_f<ACT>(acc[r][3] + bb.w));
  }
  __syncwarp();
  zero_acc(acc);
  warp_gemm_4x4<H>(hid + warp * 4 * LDX, a.W4_t, lane, acc);
  {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(a.b4 + lane * 4));
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      int row = warp * 4 + r, g = g0 + row;
      float m = g < n_total ? a.nm[g] : 0.f;
      float4 hv = *reinterpret_cast<const float4*>(hs + row * LDX + lane * 4);
      float4 o = make_float4((hv.x + (acc[r][0] + bb.x)) * m, (hv.y + (acc[r][1] + bb.y)) * m,
                             (hv.z + (acc[r][2] + bb.z)) * m, (hv.w + (acc[r][3] + bb.w)) * m);
      __syncwarp();
      *reinterpret_cast<float4*>(hs + row * LDX + lane * 4) = o;
      if (g < n_total) *reinterpret_cast<float4*>(a.h + (size_t)g * H + lane * 4) = o;
    }
  }
  __syncwarp();
  if (a.AB1 != nullptr) project_ab(hs + warp * 4 * LDX, a.proj1, a.AB1, a.ABmax1, g0, n_total, warp, lane);
  if (a.AB2 != nullptr) project_ab(hs + warp * 4 * LDX, a.proj2, a.AB2, a.ABmax2, g0, n_total, warp, lane);
}

// ------------------------------------------------------------------------------------------------
// Edge weights
// ------------------------------------------------------------------------------------------------
// FC graphs: the caller's int8 edge_mask value (0/-1/-2, datasets.py:365-369) or 1 when absent.
// Pocket graphs (egnn.py:554-596): a 0/1 predicate on the *input* coordinates of this forward call.
__device__ __forceinline__ float edge_weight(int graph_type, const int8_t* __restrict__ em_mol, int N, int i, int j,
                                             int ci, int cj, float d0) {
  if (graph_type == 0) return em_mol != nullptr ? (float)em_mol[(size_t)i * N + j] : 1.0f;
  if (graph_type == 4)  // SizeGNN: (edge_mask.bool() & (radial < 6)).long() -- on the SQUARED distance (linker_size_lightning.py:107-108)
    return ((em_mol == nullptr || em_mol[(size_t)i * N + j] != 0) && d0 < 6.0f) ? 1.f : 0.f;
  if (i == j || ci == 0 || cj == 0) return 0.f;
  float dist = sqrtf(d0);
  if (graph_type == 1) return dist <= 4.0f ? 1.f : 0.f;
  if (ci == 3 || cj == 3) return 0.f;               // valid atom that is neither ligand nor pocket
  if (ci == 1 && cj == 1) return 1.f;               // ligand-ligand: fully connected
  if (ci == 2 && cj == 2) return dist <= 4.0f ? 1.f : 0.f;
  float cut = graph_type == 2 ? 4.0f : 10.0f;       // FC-4A : FC-10A-4A
  return dist <= cut ? 1.f : 0.f;
}

// Cut-off graphs on the tensor-core path: per-row neighbour lists of this forward call (the graph is a function of the
// call's input coordinates, egnn.py:554-596) and the 128-edge tiles packed from them, so that edges the reference
// never creates cost nothing and tiles are full.
// One CTA per molecule; coordinates / classes / live columns are staged in shared memory.
//   1. one warp per row slot compacts the row's neighbours in ascending column order (ballot + popc: deterministic)
//        nbr[(b*N + i)*N + k] = k-th neighbour of node i  (bit 31 set: padding edge of weight 0 -- a live row without
//                               any neighbour still owns one tile column, so its aggregate is written as exactly 0)
//   2. rows with <= 128 neighbours are bin-packed into tiles, first-fit over the rows in decreasing degree (ties by
//      row slot: the packing, hence the summation order of every row, is a pure function of the graph);
//      a row with more neighbours becomes one record that the edge kernel expands into 128-column chunk tiles
//   3. tile records (32 ints) are appended to the launch-wide list (one atomicAdd per molecule; the order of the
//      molecules' ranges does not influence any result):
//        [0] molecule  [1] rows | heavy << 8  [2] edges (heavy: the row's degree)  [3] 0
//        [4 + r] node | first tile column << 16   for row r of the tile (<= CUT_MAXR rows)
// Done twice: for all live rows (GCL tiles) and for the coordinate-update rows (linker rows; COORD tiles).
constexpr int CUT_TN = 128;       // = tc::TN
constexpr int CUT_MAXR = 28;      // rows per packed tile (record = 4 + 28 ints = 128 bytes)
constexpr int CUT_REC = 32;

__device__ __forceinline__ void cut_pack_rows(int b, int N, int nrows, const int* __restrict__ rowlist /*global, slot order*/,
                                              const int* degn, int* srt, int* row_bin, int* row_pos, int* row_start,
                                              int* bin_rem, int* bin_cnt, int* misc, int* __restrict__ recs,
                                              int* __restrict__ n_recs) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // rank of every light row among the light rows: degree descending, slot ascending
  if (tid == 0) { misc[0] = 0; misc[1] = 0; }
  __syncthreads();
  for (int s = tid; s < nrows; s += blockDim.x) {
    const int node = rowlist[s], d = degn[node];
    if (d <= CUT_TN) {
      int rank = 0;
      for (int s2 = 0; s2 < nrows; ++s2) {
        const int d2 = degn[rowlist[s2]];
        rank += (d2 <= CUT_TN && (d2 > d || (d2 == d && s2 < s))) ? 1 : 0;
      }
      srt[rank] = node;
      atomicAdd(&misc[0], 1);                              // number of light rows
    } else {
      row_pos[node] = atomicAdd(&misc[1], 1);              // heavy rows: any distinct record slot will do
    }
  }
  __syncthreads();
  const int n_light = misc[0], n_heavy = misc[1];
  if (warp == 0) {
    int nb = 0, first_open = 0;
    const int d_min = n_light > 0 ? degn[srt[n_light - 1]] : 0;
    for (int idx = 0; idx < n_light; ++idx) {
      const int node = srt[idx], d = degn[node];
      int found = -1;
      for (int base = first_open; base < nb && found < 0; base += 32) {
        const int bb = base + lane;
        const bool ok = bb < nb && bin_rem[bb] >= d && bin_cnt[bb] < CUT_MAXR;
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        if (m) found = base + __ffs(m) - 1;
      }
      if (lane == 0) {
        if (found < 0) { bin_rem[nb] = CUT_TN; bin_cnt[nb] = 0; }
      }
      if (found < 0) { found = nb; ++nb; }
      __syncwarp();
      if (lane == 0) {
        row_bin[node] = found; row_pos[node] = bin_cnt[found]; row_start[node] = CUT_TN - bin_rem[found];
        bin_rem[found] -= d; bin_cnt[found] += 1;
      }
      __syncwarp();
      while (first_open < nb && (bin_rem[first_open] < d_min || bin_cnt[first_open] >= CUT_MAXR)) ++first_open;
    }
    if (lane == 0) {
      misc[2] = nb;
      misc[3] = atomicAdd(n_recs, nb + n_heavy);           // this molecule's range in the launch-wide list
    }
  }
  __syncthreads();
  const int nb = misc[2];
  int* out = recs + (size_t)misc[3] * CUT_REC;
  for (int bb = tid; bb < nb; bb += blockDim.x) {
    int* r = out + (size_t)bb * CUT_REC;
    r[0] = b; r[1] = bin_cnt[bb]; r[2] = CUT_TN - bin_rem[bb]; r[3] = 0;
  }
  for (int s = tid; s < nrows; s += blockDim.x) {
    const int node = rowlist[s], d = degn[node];
    if (d <= CUT_TN) {
      out[(size_t)row_bin[node] * CUT_REC + 4 + row_pos[node]] = node | (row_start[node] << 16);
    } else {
      int* r = out + (size_t)(nb + row_pos[node]) * CUT_REC;
      r[0] = b; r[1] = 1 | (1 << 8); r[2] = d; r[3] = 0; r[4] = node;
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(512) k_nbr(int N, int graph_type, const float4* __restrict__ x04,
                                             const int* __restrict__ cls, const int* __restrict__ rowidx,
                                             const int* __restrict__ colidx, const int* __restrict__ xrowidx,
                                             const int* __restrict__ nr, const int* __restrict__ nc,
                                             const int* __restrict__ nxr, int* __restrict__ nbr,
                                             int* __restrict__ recs, int* __restrict__ xrecs,
                                             int* __restrict__ n_recs /*[2]: GCL, COORD*/) {
  extern __shared__ uint8_t sm_nbr[];
  float4* xs = reinterpret_cast<float4*>(sm_nbr);             // [N]
  int* cl = reinterpret_cast<int*>(xs + N);                   // [N]
  int* col = cl + N;                                          // [N]
  int* degn = col + N;                                        // [N] degree by node
  int* srt = degn + N;                                        // [N] light rows, degree descending
  int* row_bin = srt + N; int* row_pos = row_bin + N; int* row_start = row_pos + N;
  int* bin_rem = row_start + N; int* bin_cnt = bin_rem + N;   // [N] each
  __shared__ int misc[4];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
  const size_t gb = (size_t)b * N;
  const int nrows = nr[b], ncols = nc[b];
  for (int i = tid; i < N; i += blockDim.x) {
    xs[i] = x04[gb + i]; cl[i] = cls[gb + i];
    col[i] = i < ncols ? colidx[gb + i] : 0;
    degn[i] = 0;
  }
  __syncthreads();
  for (int slot = warp; slot < nrows; slot += nwarp) {
    const int i = rowidx[gb + slot];
    const float4 xi = xs[i];
    const int ci = cl[i];
    int* out = nbr + (gb + i) * N;
    int count = 0;
    for (int c0 = 0; c0 < ncols; c0 += 32) {
      const int c = c0 + lane;
      bool keep = false;
      int j = 0;
      if (c < ncols) {
        j = col[c];
        const float4 xj = xs[j];
        const float ex = xi.x - xj.x, ey = xi.y - xj.y, ez = xi.z - xj.z;
        const float d0 = ex * ex + ey * ey + ez * ez;
        keep = edge_weight(graph_type, nullptr, N, i, j, ci, cl[j], d0) != 0.f;
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) out[count + __popc(m & ((1u << lane) - 1u))] = j;
      count += __popc(m);
    }
    if (lane == 0) {
      if (count == 0) { out[0] = i | (int)0x80000000; count = 1; }
      degn[i] = count;
    }
  }
  __syncthreads();
  cut_pack_rows(b, N, nrows, rowidx + gb, degn, srt, row_bin, row_pos, row_start, bin_rem, bin_cnt, misc, recs, n_recs);
  cut_pack_rows(b, N, nxr[b], xrowidx + gb, degn, srt, row_bin, row_pos, row_start, bin_rem, bin_cnt, misc, xrecs, n_recs + 1);
}
constexpr int CUT_SMEM_PER_NODE = 16 + 9 * 4;

// ------------------------------------------------------------------------------------------------
// Reference fp32 SIMT edge kernel: second Linear of the edge / coord MLP as a 128x128x128 tile GEMM.
//   GCL   (egnn.py:45-66):   agg_i = sum_j silu(W2 silu(A_i+B_j+d_ij wd+d0_ij w0)+b2) * EM_ij / nf
//   COORD (egnn.py:101-117): x_i  += (sum_j cd_ij * (w5 . silu(W2 silu(...)+b2)) * EM_ij / nf) * linker_mask_i
// Tile = up to 128 edges = whole rows x all live columns (or one row x 128-column chunks when nc > 128).
// ------------------------------------------------------------------------------------------------
constexpr int ET = 128;          // edges per tile
constexpr int MAXR = 8;          // max rows per tile
constexpr int LDB = H + 1;       // Bs row stride (bank-conflict-free column walks)

struct EdgeArgs {
  const float* AB;          // (B*N,256)
  const float* ABmax;       // (B*N,2) row maxima of |A|, |B|
  float w2_descale, wdmax, w0max;
  const float* x;           // (B*N,3) current coordinates
  const float* x0;          // (B*N,3) input coordinates (d0)
  const float4* x4;         // (B*N) padded copies of x / x0 (tensor-core path)
  const float4* x04;
  float4* x4_out;
  const int8_t* edge_mask;  // (B*N*N) or null
  const int* cls;           // (B*N) pocket classes (graph_type != 0)
  const float* nm;          // (B*N)
  const float* linker_mask; // (B*N) or null
  const float* W2_t; const float* b2; const float* wd; const float* w0; const float* w5;
  Plan plan;
  float* agg;               // GCL out (B*N,128)
  float* x_out;             // COORD out (B*N,3)
  const int* nbr;           // cut-off graphs, tensor-core path: per-row neighbour lists (k_nbr) or null
  const int* recs;          // ... and this launch's packed tile records (GCL or COORD list), CUT_REC ints each
  const int* n_recs;        // [1]
  float coords_range;       // OPT_TANH: bound of the coordinate update
  const float* we;          // OPT_SIN: [24][128] embedding columns of the first layer (log2 domain on the tensor-core path)
};

constexpr size_t EDGE_SIMT_SMEM =
    sizeof(float) * ((size_t)H * H /*W2s*/ + (size_t)H * ET /*S1*/ + (size_t)ET * LDB /*Bs*/ + (size_t)MAXR * H /*As*/ +
                     4 * H /*b2,wd,w0,w5*/ + ET /*ems*/ + ET * 3 /*cds*/ + ET /*phis*/);

// OPT (OPT_TANH | OPT_MEAN): with OPT_MEAN a row's divisor is N on FC graphs and its number of live edges (cut-off edges
// have weight 1, every other pair 0) on cut-off graphs, counted alongside the sum.
template <bool COORD, int ACT = ACT_SILU, int OPT = 0>
__global__ void __launch_bounds__(256, 1) k_edge_simt(Geom gm, EdgeArgs a) {
  constexpr bool MEAN = (OPT & OPT_MEAN) != 0, TANH = (OPT & OPT_TANH) != 0, EMB = (OPT & OPT_SIN) != 0;
  extern __shared__ __align__(16) float sm_edge[];
  float* W2s = sm_edge;
  float* S1 = W2s + H * H;
  float* Bs = S1 + H * ET;
  float* As = Bs + ET * LDB;
  float* b2s = As + MAXR * H;
  float* wds = b2s + H;
  float* w0s = wds + H;
  float* w5s = w0s + H;
  float* ems = w5s + H;
  float* cds = ems + ET;
  float* phis = cds + ET * 3;
  __shared__ float xacc[COORD ? 1 : 1];  // placeholder to keep static smem trivial
  (void)xacc;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = gm.N;
  for (int idx = tid; idx < H * H / 4; idx += 256)
    reinterpret_cast<float4*>(W2s)[idx] = __ldg(reinterpret_cast<const float4*>(a.W2_t) + idx);
  if (tid < H) {
    b2s[tid] = a.b2[tid]; wds[tid] = a.wd[tid]; w0s[tid] = a.w0[tid];
    w5s[tid] = COORD ? a.w5[tid] : 0.f;
  }
  __syncthreads();

  // aggregation divisor of a row with `cnt` live edges (egnn.py:312-319)
  auto divisor = [&](float cnt) { return !MEAN ? gm.normalization_factor : gm.graph_type == 0 ? (float)N : fmaxf(cnt, 1.f); };
  const int n_work = COORD ? *a.plan.n_xmols : *a.plan.n_items;
  for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
    int b, r_begin, r_count;
    if (COORD) { b = a.plan.xmols[wi]; r_begin = 0; r_count = a.plan.nxr[b]; }
    else { int4 it = a.plan.items[wi]; b = it.x; r_begin = it.y; r_count = it.z; }
    const int nc = a.plan.nc[b];
    const int* rows = (COORD ? a.plan.xrowidx : a.plan.rowidx) + (size_t)b * N;
    const int* cols = a.plan.colidx + (size_t)b * N;
    const size_t gb = (size_t)b * N;
    const int8_t* em_mol = a.edge_mask ? a.edge_mask + gb * N : nullptr;
    int per = nc >= ET ? 1 : ET / nc;
    if (per > MAXR) per = MAXR;

    for (int rt = 0; rt < r_count; rt += per) {          // row groups (GCL items hold exactly one)
      const int nrt = min(per, r_count - rt);
      for (int r = warp; r < nrt; r += 8) {               // A rows
        int i = rows[r_begin + rt + r];
        *reinterpret_cast<float4*>(As + r * H + lane * 4) =
            *reinterpret_cast<const float4*>(a.AB + (gb + i) * 2 * H + lane * 4);
      }
      float run = 0.f;                                    // GCL: running row sum across column chunks
      float xrun = 0.f;                                   // COORD: thread (r,dim) running sum
      float runc = 0.f;                                   // OPT_MEAN: running live-edge count of the same row
      for (int c0 = 0; c0 < nc; c0 += ET) {
        const int ncc = min(ET, nc - c0);
        const int Et = nrt * ncc;
        __syncthreads();                                  // previous tile fully consumed
        for (int idx = tid; idx < ncc * H; idx += 256) {  // B rows of the live columns
          int jj = idx >> 7, k = idx & (H - 1);
          Bs[jj * LDB + k] = a.AB[(gb + cols[c0 + jj]) * 2 * H + H + k];
        }
        __syncthreads();
        {                                                 // first layer + SiLU -> S1[k][e]
          const int e = tid & (ET - 1), kh = tid >> 7;
          const bool valid = e < Et;
          int rr = 0, jj = 0;
          float d = 0.f, d0 = 0.f;
          float emb[EMB ? N_SIN_FEAT : 1];                // OPT_SIN: [sin d f_k, cos d f_k, sin d0 f_k, cos d0 f_k]
          if (valid) {
            rr = e / ncc; jj = e - rr * ncc;
            const int i = rows[r_begin + rt + rr], j = cols[c0 + jj];
            const float* xi = a.x + (gb + i) * 3; const float* xj = a.x + (gb + j) * 3;
            const float* yi = a.x0 + (gb + i) * 3; const float* yj = a.x0 + (gb + j) * 3;
            float dx = xi[0] - xj[0], dy = xi[1] - xj[1], dz = xi[2] - xj[2];
            d = dx * dx + dy * dy + dz * dz;
            float ex = yi[0] - yj[0], ey = yi[1] - yj[1], ez = yi[2] - yj[2];
            d0 = ex * ex + ey * ey + ez * ez;
            // the reference's rounding order, not the contracted FMA form, where it decides something: the sinusoid
            // arguments, and SizeGNN's edge set (radial < 6)
            if constexpr (EMB || ACT == ACT_RELU) { d = radial_rn(dx, dy, dz); d0 = radial_rn(ex, ey, ez); }
            if constexpr (EMB) {
#pragma unroll
              for (int k = 0; k < N_SIN_FREQ; ++k) {
                sincosf(sin_arg(d, k), &emb[k], &emb[N_SIN_FREQ + k]);
                sincosf(sin_arg(d0, k), &emb[2 * N_SIN_FREQ + k], &emb[3 * N_SIN_FREQ + k]);
              }
            }
            if (kh == 0) {
              int ci = 0, cj = 0;
              if (gm.graph_type >= 1 && gm.graph_type <= 3) { ci = a.cls[gb + i]; cj = a.cls[gb + j]; }
              ems[e] = edge_weight(gm.graph_type, em_mol, N, i, j, ci, cj, d0);
              if (COORD) {
                float inv = 1.0f / (sqrtf(d + 1e-8f) + gm.norm_constant);   // egnn.py:299-300
                cds[e * 3 + 0] = dx * inv; cds[e * 3 + 1] = dy * inv; cds[e * 3 + 2] = dz * inv;
              }
            }
          } else if (kh == 0) {
            ems[e] = 0.f;
            if (COORD) { cds[e * 3 + 0] = 0.f; cds[e * 3 + 1] = 0.f; cds[e * 3 + 2] = 0.f; }
          }
          const float* Ar = As + rr * H;
          const float* Br = Bs + jj * LDB;
#pragma unroll 8
          for (int kk = 0; kk < H / 2; ++kk) {
            int k = kh * (H / 2) + kk;
            float pre;
            if constexpr (EMB) {
              pre = Ar[k] + Br[k];
#pragma unroll
              for (int f = 0; f < N_SIN_FEAT; ++f) pre += (valid ? emb[f] : 0.f) * __ldg(a.we + f * H + k);
            } else {
              pre = Ar[k] + Br[k] + d * wds[k] + d0 * w0s[k];
            }
            S1[k * ET + e] = valid ? act_f<ACT>(pre) : 0.f;
          }
        }
        __syncthreads();
        // 128x128x128 GEMM, 8x8 register tile
        const int ty = tid >> 4, tx = tid & 15;
        float acc[8][8];
#pragma unroll
        for (int p = 0; p < 8; ++p)
#pragma unroll
          for (int q = 0; q < 8; ++q) acc[p][q] = 0.f;
#pragma unroll 4
        for (int k = 0; k < H; ++k) {
          float4 a0 = *reinterpret_cast<const float4*>(S1 + k * ET + ty * 4);
          float4 a1 = *reinterpret_cast<const float4*>(S1 + k * ET + 64 + ty * 4);
          float4 b0 = *reinterpret_cast<const float4*>(W2s + k * H + tx * 4);
          float4 b1 = *reinterpret_cast<const float4*>(W2s + k * H + 64 + tx * 4);
          const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
          const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
          for (int p = 0; p < 8; ++p)
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[p][q] = fmaf(av[p], bv[q], acc[p][q]);
        }
        __syncthreads();                                  // S1 no longer read -> reuse as Outs[e][c]
        float* Outs = S1;
#pragma unroll
        for (int p = 0; p < 8; ++p) {
          int e = (p < 4 ? ty * 4 + p : 64 + ty * 4 + (p - 4));
          float w = COORD ? 1.f : ems[e];
#pragma unroll
          for (int qh = 0; qh < 2; ++qh) {
            int c = qh * 64 + tx * 4;
            float4 o;
            o.x = act_f<ACT>(acc[p][qh * 4 + 0] + b2s[c + 0]) * w;
            o.y = act_f<ACT>(acc[p][qh * 4 + 1] + b2s[c + 1]) * w;
            o.z = act_f<ACT>(acc[p][qh * 4 + 2] + b2s[c + 2]) * w;
            o.w = act_f<ACT>(acc[p][qh * 4 + 3] + b2s[c + 3]) * w;
            *reinterpret_cast<float4*>(Outs + e * H + c) = o;
          }
        }
        __syncthreads();
        if (!COORD) {
          // deterministic segment sum over j, thread = (row parity, channel)
          const int c = tid & (H - 1);
          if (nc <= ET) {
            for (int rr = tid >> 7; rr < nrt; rr += 2) {
              float s = 0.f, cnt = 0.f;
              for (int jj = 0; jj < ncc; ++jj) {
                s += Outs[(rr * ncc + jj) * H + c];
                if (MEAN) cnt += ems[rr * ncc + jj] != 0.f ? 1.f : 0.f;
              }
              a.agg[(gb + rows[r_begin + rt + rr]) * H + c] = s / divisor(cnt);
            }
          } else if (tid < H) {
            for (int jj = 0; jj < ncc; ++jj) {
              run += Outs[jj * H + c];
              if (MEAN) runc += ems[jj] != 0.f ? 1.f : 0.f;
            }
            if (c0 + ET >= nc) a.agg[(gb + rows[r_begin + rt]) * H + c] = run / divisor(runc);
          }
        } else {
          for (int e = warp; e < Et; e += 8) {            // phi_e = w5 . m_e  (coord_mlp.4, egnn.py:90-97)
            float s = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) s = fmaf(Outs[e * H + lane + 32 * q], w5s[lane + 32 * q], s);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) phis[e] = TANH ? tanhf(s) * a.coords_range * ems[e] : s * ems[e];   // egnn.py:104-109
          }
          __syncthreads();
          if (tid < nrt * 3) {
            int rr = tid / 3, dim = tid - rr * 3;
            float s = 0.f;
            for (int jj = 0; jj < ncc; ++jj) {
              s += cds[(rr * ncc + jj) * 3 + dim] * phis[rr * ncc + jj];
              if (MEAN) runc += ems[rr * ncc + jj] != 0.f ? 1.f : 0.f;
            }
            xrun += s;
            if (c0 + ET >= nc) {
              int i = rows[r_begin + rt + rr];
              float lm = a.linker_mask ? a.linker_mask[gb + i] : 1.f;
              float xv = a.x[(gb + i) * 3 + dim];
              a.x_out[(gb + i) * 3 + dim] = (xv + (xrun / divisor(runc)) * lm) * a.nm[gb + i];
            }
          }
        }
      }
    }
  }
}

// Rows the coordinate update does not touch keep x (x is already masked: (x + 0)*nm == x).
// Runs before k_edge<COORD> writes the updated rows into the same buffer.
__global__ void k_copy_x(int n3, const float* __restrict__ src, float* __restrict__ dst, const float4* __restrict__ src4,
                         float4* __restrict__ dst4) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n3) dst[i] = src[i];
  if (src4 != nullptr && i * 3 < n3) dst4[i] = src4[i];
}

// ------------------------------------------------------------------------------------------------
// Output stage: EGNN.embedding_out (egnn.py:235-237), vel (egnn.py:420), slicing (430-435), NaN flags (441),
// and -- in sampler mode -- the reverse-diffusion update of z fused in (edm.py:196-206 / 225-233).
// 16 threads per node (one per output column), 16 nodes per CTA.
// ------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------
// Device-side noise in the reference's stream order. The reference draws, per noise sample, torch.randn(B,N,3) then
// torch.randn(B,N,F) (edm.py:328-340, utils.py:189-192). On a CUDA device torch serves each call with Philox4x32-10:
//   grid = min(SMs * (maxThreadsPerSM / 256), ceil(numel / 256)) blocks of 256 threads, thread idx = subsequence idx,
//   element e is component (e mod 4S) / S of the (e / 4S)-th curand_normal4 of thread e mod S (S = 256 * grid), and the
//   call advances the generator's offset by ((numel - 1) / (4S) + 1) * 4
// (ATen/native/cuda/DistributionTemplates.h: calc_execution_policy, distribution_elementwise_grid_stride_kernel,
// normal_and_transform). Reproducing that mapping with the same cuRAND device functions gives the SAME numbers the
// reference would draw on this GPU for the same seed and offset -- without the (T+2) x 2 randn launches, the
// (T+2,B,N,3+F) slab and its interleaving copy.
//
// Per-molecule stream (kernels instantiated with PER_MOL = true): molecule b draws what the batch stream gives a batch of
// that one molecule from generator state (seeds[b], 0). Such a batch has numel <= S for both calls (up to 256 * 8 * SMs
// elements), so element e of a call is component .x of the curand_normal4 of subsequence e, the x call of draw r sits at
// offset 8r and the h call at 8r + 4:
//   element d of atom n of molecule b in draw r = curand_normal4(curand_init(seeds[b], e, 8r + (d >= 3 ? 4 : 0))).x,
//   e = 3n + d (d < 3) or F n + (d - 3)
// Nothing in it depends on B, on N, on the molecule's row or on the device, so a molecule samples the same whatever its
// batch. The per-molecule kernels read the seeds through the union below and N from the field that otherwise pads the
// struct: the batch-stream instantiations see the parameter layout they always saw.
// ------------------------------------------------------------------------------------------------
enum { NOISE_TENSOR = 0, NOISE_BATCH = 1, NOISE_PER_MOLECULE = 2 };
struct NoiseRng {
  union {
    unsigned long long seed;         // batch stream: torch CUDA generator state when EDM.sample_chain was entered
    const unsigned long long* seeds; // per-molecule stream: B seeds in device memory (the engine's copy)
  };
  unsigned long long offset;
  unsigned long long per_draw;       // offset consumed by one draw (x call + h call)
  unsigned long long cx;             // ... by the x call alone
  int Sx, Sh;                        // 256 * grid of the x / h call
  int F;
  int on;                            // NOISE_TENSOR: read the caller's noise tensor instead; else NOISE_BATCH / _PER_MOLECULE
  int g0;                            // first node row of this engine's slice inside the full batch (strong scaling: the slice
                                     // consumes exactly the rows of the full-batch draw, so results do not depend on the split)
  int N;                             // per-molecule stream: atoms per molecule (node g is atom g % N of molecule g / N)
};
static_assert(sizeof(NoiseRng) == 56, "NoiseRng: the batch-stream kernels' parameter layout");
__device__ __forceinline__ float philox_normal_elem(unsigned long long seed, unsigned long long offset, int S, long long e) {
  const long long per_round = 4LL * S;
  const long long rr = e / per_round;
  const int rem = (int)(e - rr * per_round);
  const int ii = rem / S, idx = rem - ii * S;
  curandStatePhilox4_32_10_t st;
  curand_init(seed, (unsigned long long)idx, offset + 4ULL * (unsigned long long)rr, &st);
  const float4 v = curand_normal4(&st);
  return ii == 0 ? v.x : ii == 1 ? v.y : ii == 2 ? v.z : v.w;
}
// element d of node g (of n_total) of noise draw r
template <bool PER_MOL = false>
__device__ __forceinline__ float noise_draw(const NoiseRng& q, int r, int g, int d) {
  if constexpr (PER_MOL) {
    const int b = g / q.N, n = g - b * q.N;
    const unsigned long long e = d < 3 ? 3ULL * n + d : (unsigned long long)q.F * n + (d - 3);
    curandStatePhilox4_32_10_t st;
    curand_init(q.seeds[b], e, 8ULL * (unsigned long long)r + (d < 3 ? 0ULL : 4ULL), &st);
    return curand_normal4(&st).x;
  }
  const unsigned long long base = q.offset + (unsigned long long)r * q.per_draw;
  const long long gg = (long long)g + q.g0;
  if (d < 3) return philox_normal_elem(q.seed, base, q.Sx, gg * 3 + d);
  return philox_normal_elem(q.seed, base + q.cx, q.Sh, gg * q.F + (d - 3));
}

// Per-molecule start steps (dl_set_start_steps): the engine's rows are the caller's, ordered by start step t0 descending,
// and loop step r computes the prefix of rows that have started. Row i is caller row src[i]; it started lag[i] = t0max - t0
// steps after the loop did, so its own draw k is loop draw k + lag[i] and its NaN tag counts from its own start. The caller's
// noise tensor, chain frames and NaN flags keep the caller's n_full = B * N node rows.
struct RowStarts {
  const int* lag;
  const int* src;
  int n_full;
};

struct FinishArgs {
  const float* h;        // (B*N,128) final hidden state
  const float* x;        // (B*N,3) final coordinates
  const float* x0;       // (B*N,3)
  const float* nm;
  const float* Wo;       // [D][128] embedding_out.weight (first F rows used)
  const float* bo;       // [D]
  float* out;            // Dynamics.forward output (B*N,3+F) or null
  int* nan_flags;        // (B) or null
  // sampler mode
  float* z;              // (B*N,3+F) in/out, null when not sampling
  const float* fragment_mask; const float* linker_mask;
  const float* noise;    // (T+2,B*N,3+F), or null with rng.on
  NoiseRng rng;
  const float* coef;     // device table, 8 floats per row
  const int* step_fin; int* step_prep;
  int T;
  float norm0, norm1, bias1;
  float* chain;          // (keep,B*N,3+F)
  const int* tag_step;   // non-sampler mode inside the inpainting loop: step counter used to tag NaN flags (or null)
  RowStarts rows;        // per-molecule start steps (dl_set_start_steps), or lag = null
  // ODE solvers (dl_set_solver, k_finish<., true>): the solver table of the loop's rows, 8 floats per row in coef's row
  // order, and the DPM-Solver++(2M) history -- every node's data prediction of its previous step -- or null (DDIM)
  const float* ode;
  float* hist;
  // fixed atoms (dl_set_fixed_atoms, k_finish<., ., true>): the linker rows to keep (B*N int8 in the workspace's row
  // order), the normalised input xh they keep, and the (alpha_s, sigma_s) of the loop's rows, 2 floats per row in coef's
  // row order
  const int8_t* fixed;
  const float* xh0;
  const float* fix;
  // linker types (dl_set_linker_types, k_finish<., ., ., true>): one mask of allowed type channels per molecule (bit c:
  // channel 3 + c), in the caller's row order (rows.src maps a workspace row to it), and the (alpha_t, sigma_t) of the
  // loop's rows, 2 floats per row in coef's row order
  const uint32_t* types;
  const float* tsc;
};

// A kept row's z_s = alpha_s xh + sigma_s eps, every product and the sum rounded on their own as k_init_z_rows rounds them.
__device__ __forceinline__ float fixed_state(const float* sc, float xh, float eps) {
  return __fadd_rn(__fmul_rn(sc[0], xh), __fmul_rn(sc[1], eps));
}

// TYPES: on a free linker row (linker_mask != 0, not kept), a type channel its molecule's mask excludes predicts the
// one-hot's normalised "off" value, off = (0 - bias1) / norm1: the ODE update sets xhat = off, the ancestral update reads
// eps = (z_t - alpha_t off) / sigma_t, which is the same, and the final decode takes the argmax over the allowed channels.
template <bool PER_MOL = false, bool ODE = false, bool FIX = false, bool TYPES = false>
__global__ void __launch_bounds__(256) k_finish(Geom gm, FinishArgs a) {
  const int tid = threadIdx.x;
  const int d = tid & 15, r = tid >> 4;
  const int n_total = gm.B * gm.N;
  const int g = blockIdx.x * 16 + r;
  const int xd = 3 + gm.F;
  const bool act = g < n_total && d < xd;
  // embedding_out operands staged in shared memory: the 16 nodes' h rows (coalesced loads) and Wo transposed to [k][j], so
  // the 16 lanes of a node read 16 consecutive floats per k (the direct form -- every lane streaming its own 512-byte
  // Wo row -- was bound by L1 wavefronts: 23 us for 14 MFLOP)
  __shared__ __align__(16) float hs[16][H + 4];
  __shared__ float ws[H][16];
  for (int idx = tid; idx < 16 * H; idx += 256) {           // weights: not produced by the chain, staged before the wait
    const int j = idx / H, k = idx - j * H;
    ws[k][j] = j < gm.F ? __ldg(a.Wo + (size_t)j * H + k) : 0.f;
  }
  chain_wait();
  chain_release();
  int step = 0;
  if (a.z != nullptr) {
    step = *a.step_fin;
    if (blockIdx.x == 0 && tid == 0) *a.step_prep = step + 1;
  } else if (a.tag_step != nullptr) {
    step = *a.tag_step;
  }
  // this row's draw offset, and node g's row in the caller's noise, chain and flags
  int lag = 0;
  size_t gc = g, nc = n_total;
  if (a.rows.lag != nullptr && g < n_total) {
    const int b = g / gm.N;
    lag = a.rows.lag[b];
    gc = (size_t)a.rows.src[b] * gm.N + (g - b * gm.N);
    nc = a.rows.n_full;
  }
  const uint32_t allowed = TYPES && g < n_total ? a.types[gc / gm.N] : ~0u;   // the molecule's mask, in the caller's order
  for (int idx = tid; idx < 16 * (H / 4); idx += 256) {
    const int rr = idx / (H / 4), k4 = idx - rr * (H / 4);
    const int gg = blockIdx.x * 16 + rr;
    const float4 v = gg < n_total ? *reinterpret_cast<const float4*>(a.h + (size_t)gg * H + k4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(&hs[rr][k4 * 4]) = v;
  }
  __syncthreads();
  float e = 0.f;
  if (act) {
    float m = a.nm[g];
    if (d < 3) {
      e = (a.x[(size_t)g * 3 + d] - a.x0[(size_t)g * 3 + d]) * m;
    } else {
      const int j = d - 3;
      float s = 0.f;                                          // same summation order as before: k ascending
#pragma unroll 8
      for (int k = 0; k < H; k += 4) {
        const float4 hv = *reinterpret_cast<const float4*>(&hs[r][k]);
        s = fmaf(hv.x, ws[k][j], s); s = fmaf(hv.y, ws[k + 1][j], s); s = fmaf(hv.z, ws[k + 2][j], s); s = fmaf(hv.w, ws[k + 3][j], s);
      }
      e = (s + a.bo[j]) * m;
    }
    if (e != e && a.nan_flags != nullptr) {
      // bit0: NaN in vel, bit1: NaN in h (utils.py:274-282); bits 8.. = 1 + index of the first failing
      // reverse step. Later steps do not add bits: the reference raises at the first failing step.
      const int bits = d < 3 ? 1 : 2;
      const int tag = ((a.z != nullptr || a.tag_step != nullptr) ? step + 1 - lag : 0) << 8;
      int* p = a.nan_flags + gc / gm.N;
      const int old = atomicCAS(p, 0, bits | tag);
      if (old != 0 && (old & ~0xff) == tag) atomicOr(p, bits);
    }
    if (a.out != nullptr) a.out[(size_t)g * xd + d] = e;
  }
  if (a.z == nullptr) return;

  const float* cf = a.coef + (size_t)step * 8;
  const float ca = cf[1], cb = cf[2], cc = cf[3];
  const int frame = __float_as_int(cf[4]);
  float znew = 0.f;
  float lm = 0.f, fm = 0.f;
  bool excl = false;   // TYPES: channel d is an excluded type of a free linker row
  if constexpr (ODE) {
    // deterministic update from the solver row sv = (sigma_t, 1/alpha_t, sigma_s/sigma_t, c1, c2a, c2b, h, 0): the data
    // prediction xhat = (z_t - sigma_t eps) / alpha_t, then z_s = (sigma_s/sigma_t) z_t + c1 xhat at a row's first step
    // (DDIM always), + c2a xhat + c2b xhat' after it; the final row returns xhat. No draw is read.
    // FIX: a kept row then takes alpha_s xh + sigma_s eps_0 with its own draw 0 instead, so its history does not enter
    if (act) {
      lm = a.linker_mask[g]; fm = a.fragment_mask[g];
      const size_t gi = (size_t)g * xd + d;
      const float zt = a.z[gi];
      const float eps = e * lm;
      const float* sv = a.ode + (size_t)step * 8;
      float xhat = sv[1] * (zt - sv[0] * eps);
      const bool kept = FIX && a.fixed[g] != 0;
      excl = TYPES && d >= 3 && lm != 0.f && !kept && ((allowed >> (d - 3)) & 1u) == 0;
      if (excl) xhat = __fdiv_rn(__fsub_rn(0.f, a.bias1), a.norm1);   // TYPES: the projected xhat, which the 2M history keeps
      if (step < a.T) {
        float zs;
        if (a.hist != nullptr && step > lag) zs = sv[2] * zt + (sv[4] * xhat + sv[5] * a.hist[gi]);
        else zs = sv[2] * zt + sv[3] * xhat;
        if (kept) {
          const float eps0 = a.rng.on ? noise_draw<PER_MOL>(a.rng, 0, g, d) : a.noise[gc * xd + d];
          zs = fixed_state(a.fix + (size_t)step * 2, a.xh0[gi], eps0);
        }
        if (a.hist != nullptr) a.hist[gi] = xhat;
        znew = zt * fm + zs * lm;
        a.z[gi] = znew;
        if (frame >= 0) {
          float o = d < 3 ? znew * a.norm0 : znew * a.norm1 + a.bias1;
          a.chain[((size_t)frame * nc + gc) * xd + d] = o;
        }
      } else {
        znew = zt * fm + (kept ? a.xh0[gi] : xhat) * lm;
      }
    }
  } else if (act) {
    lm = a.linker_mask[g]; fm = a.fragment_mask[g];
    const float zt = a.z[(size_t)g * xd + d];
    float eps = e * lm;                                                       // edm.py:196 / 225
    const float nz = (a.rng.on ? noise_draw<PER_MOL>(a.rng, step + 1 - lag, g, d)
                               : a.noise[((size_t)(step + 1 - lag) * nc + gc) * xd + d]) * lm;  // utils.py:189-192
    // FIX: a kept row takes alpha_s xh + sigma_s nz_s from the draw the update reads, and the input at the final step
    const bool kept = FIX && a.fixed[g] != 0;
    excl = TYPES && d >= 3 && lm != 0.f && !kept && ((allowed >> (d - 3)) & 1u) == 0;
    if (excl) {   // TYPES: the eps of xhat = off, with the (alpha_t, sigma_t) of this row
      const float* ts = a.tsc + (size_t)step * 2;
      const float off = __fdiv_rn(__fsub_rn(0.f, a.bias1), a.norm1);
      eps = __fdiv_rn(__fsub_rn(zt, __fmul_rn(ts[0], off)), ts[1]);
    }
    if (step < a.T) {
      float mu = zt / ca - cb * eps;                                          // edm.py:199
      float zs = mu + cc * nz;                                                // edm.py:205, 342-345
      if (kept) zs = fixed_state(a.fix + (size_t)step * 2, a.xh0[(size_t)g * xd + d], nz);
      znew = zt * fm + zs * lm;                                               // edm.py:206
      a.z[(size_t)g * xd + d] = znew;
      if (frame >= 0) {
        float o = d < 3 ? znew * a.norm0 : znew * a.norm1 + a.bias1;          // edm.py:352-361
        a.chain[((size_t)frame * nc + gc) * xd + d] = o;
      }
    } else {
      float mux = ca * (zt - cb * eps);                                       // edm.py:241 (ca = 1/alpha_0)
      float xo = mux + cc * nz;                                               // edm.py:228
      if (kept) xo = a.xh0[(size_t)g * xd + d];
      znew = zt * fm + xo * lm;                                               // edm.py:229
    }
  }
  if (step >= a.T) {
    // edm.py:231-233: unnormalise, h = one_hot(argmax(h)) * node_mask. argmax over the 16-lane group.
    float hv = (act && d >= 3 && !excl) ? znew * a.norm1 + a.bias1 : -INFINITY;   // TYPES: the allowed channels only
    int best = d;
    float bv = hv;
    const unsigned gmask = 0xffffffffu;
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(gmask, bv, o, 16);
      int oi = __shfl_xor_sync(gmask, best, o, 16);
      if (ov > bv || (ov == bv && oi < best)) { bv = ov; best = oi; }
    }
    if (act) {
      float o = d < 3 ? znew * a.norm0 : ((d == best ? 1.f : 0.f) * a.nm[g]);
      a.chain[gc * xd + d] = o;                                               // chain[0], edm.py:174
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Per-molecule stage of inpainting models (one CTA per molecule; deterministic tree reductions):
//   mode 0: Dynamics.forward with centering=True -- vel -= mean_valid(vel) * node_mask  (egnn.py:444-445, utils.py:56-63)
//   mode 1: one reverse step of InpaintingEDM.sample_chain (edm.py:549-612): centred eps, p(z_s|z_t) on all atoms,
//           q(z_s|z_t,x) on the fragment atoms, recombination, centre-of-mass projection, chain frame;
//           the last row does sample_p_xh_given_z0 / sample_q_xh_given_z0_and_x (edm.py:689-721).
// The draws are masked and COM-projected (utils.py:158-168): draw 0 = init, 1+2r / 2+2r = step r (all atoms / fragment
// atoms), 2T+1 / 2T+2 = final draws. They arrive as prepared slabs, or with rng.on are regenerated in the CTA
// (com_free_means / com_free_value below).
// ------------------------------------------------------------------------------------------------
struct InpaintArgs {
  int mode;
  float* eps;               // (B*N,3+F) raw dynamics output (k_finish); mode 0: centred in place
  const float* nm;          // (B*N)
  float* z;                 // (B*N,3+F)
  const float* xh0;         // (B*N,3+F) normalised input (fragments are re-noised from it)
  const float* fragment_mask; const float* linker_mask;
  const float* noise;       // (2T+3,B*N,3+F) prepared draws, or null with rng.on
  NoiseRng rng;
  const float* coef;
  int* step_prep; const int* step_fin;
  int T;
  float norm0, norm1, bias1;
  float* chain;
  // RePaint resampling (k_inpaint<PER_MOL, true>): R passes per reverse step. The step counters then count passes, and
  // coef is the engine's table of T*R + 1 rows, row k*R + u being step k's row (frame -1 but on its last pass u = R-1).
  int R;
  const float* jump;        // (T, 2) (alpha_t|s, sigma_t|s) of step k, for the re-noise after every pass but the last
  int* step_tag;            // written here: the step of the next pass, which k_finish tags NaN flags with
};

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  // fixed-shape tree: warp shuffles then 8 partials summed in order by every thread
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w];
  return s;
}

// ------------------------------------------------------------------------------------------------
// The inpainting sampler's draws from the device-side stream. Draw r of a molecule is what
// InpaintingEDM.draw_noise_inpaint makes of the raw draw r = noise_draw(q, r, ...):
//   coordinates  xm - (sum_n xm / sum_n m) * m,  xm = raw * m   (sample_center_gravity_zero_gaussian_with_mask)
//   features     raw * m
// with m the fragment mask for draws 2, 4, ..., 2T (q(z_s|z_t,x) of the reverse steps) and the node mask otherwise.
// com_free_means reduces a molecule's three coordinate sums and its mask count in a fixed order (strided per-thread
// partials, then block_sum_256), so a molecule's draw depends neither on the batch split nor on the launch; every thread
// of the 256-thread CTA must call it. com_free_value then regenerates any element. Nothing is stored: the CTA draws the
// 3 coordinate normals of every atom once for the sums and again for the values. A per-molecule copy does not fit in
// shared memory at N = 4000 (pocket graphs), and a workspace copy would trade that second Philox evaluation of 3 of the
// 3+F columns for a global write and read of the whole draw. An empty mask gives 0/0 means, as in the tensor path.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool com_free_on_fragments(int r, int T) { return r >= 2 && r <= 2 * T && (r & 1) == 0; }
// The same with R resampling passes per step (dl_set_resamplings): step k's draws are 1 + k(3R-1) + 3u + {0, 1, 2} for
// pass u -- p(z_s|z_t), q(z_s|z_t,x) and, on every pass but the last, the re-noise draw -- so the fragment draws are those
// at offset 1 mod 3 within a step's 3R - 1. R = 1 is the function above.
__device__ __forceinline__ bool com_free_on_fragments(int r, int T, int R) {
  return r >= 1 && r <= T * (3 * R - 1) && (r - 1) % (3 * R - 1) % 3 == 1;
}

template <bool PER_MOL, typename M>
__device__ float3 com_free_means(const NoiseRng& q, int r, int b, int N, const M* __restrict__ mask, float* red) {
  // one (atom, coordinate) pair per thread and pass: ceil(3N / 256) Philox evaluations in a row, not 3 ceil(N / 256)
  float cnt = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
  for (int idx = threadIdx.x; idx < 3 * N; idx += 256) {
    const int n = idx / 3, d = idx - 3 * n, g = b * N + n;
    const float m = (float)mask[g];
    const float v = __fmul_rn(noise_draw<PER_MOL>(q, r, g, d), m);
    if (d == 0) { cnt += m; sx += v; } else if (d == 1) sy += v; else sz += v;
  }
  cnt = block_sum_256(cnt, red);
  sx = block_sum_256(sx, red); sy = block_sum_256(sy, red); sz = block_sum_256(sz, red);
  return make_float3(sx / cnt, sy / cnt, sz / cnt);
}

// element d of node g of draw r, mask value m, means from com_free_means (rounded step by step as the torch ops are)
template <bool PER_MOL>
__device__ __forceinline__ float com_free_value(const NoiseRng& q, int r, int g, int d, float m, float3 mean) {
  const float xm = __fmul_rn(noise_draw<PER_MOL>(q, r, g, d), m);
  if (d >= 3) return xm;
  return __fsub_rn(xm, __fmul_rn(d == 0 ? mean.x : d == 1 ? mean.y : mean.z, m));
}

// RES (RePaint, dl_set_resamplings): `step` counts passes, a.T = T*R of them before the final one. Pass u < R-1 of step k
// ends with the re-noise z <- alpha_t|s * z + sigma_t|s * eps on every atom (eps: draw rC, COM-free on the node mask),
// rounded op by op as the torch expression is, after the projection and instead of advancing to step k+1.
template <bool PER_MOL = false, bool RES = false>
__global__ void __launch_bounds__(256) k_inpaint(Geom gm, InpaintArgs a) {
  __shared__ float red[8];
  __shared__ float means[4];
  __shared__ float renoise[5];      // RES: the re-noise draw's means, alpha_t|s and sigma_t|s (shared: no registers held)
  const int b = blockIdx.x, tid = threadIdx.x, N = gm.N, xd = 3 + gm.F;
  const size_t g0 = (size_t)b * N;
  int step = 0;
  if (a.mode == 1) step = *a.step_fin;
  // number of valid atoms and mean velocity
  float cnt = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
  for (int n = tid; n < N; n += 256) {
    const float m = a.nm[g0 + n];
    cnt += m;
    sx += a.eps[(g0 + n) * xd + 0]; sy += a.eps[(g0 + n) * xd + 1]; sz += a.eps[(g0 + n) * xd + 2];
  }
  cnt = block_sum_256(cnt, red);
  sx = block_sum_256(sx, red); sy = block_sum_256(sy, red); sz = block_sum_256(sz, red);
  const float mvx = sx / cnt, mvy = sy / cnt, mvz = sz / cnt;        // utils.py:60-61
  if (a.mode == 0) {
    for (int n = tid; n < N; n += 256) {
      const float m = a.nm[g0 + n];
      a.eps[(g0 + n) * xd + 0] -= mvx * m; a.eps[(g0 + n) * xd + 1] -= mvy * m; a.eps[(g0 + n) * xd + 2] -= mvz * m;
    }
    return;
  }
  const float* cf = a.coef + (size_t)step * 8;
  const float ca = cf[1], cb = cf[2], cc = cf[3], qa = cf[5], qb = cf[6];
  const int frame = __float_as_int(cf[4]);
  const size_t slab = (size_t)gm.B * N * xd;
  // draw rA: p(z_s|z_t) on all atoms; draw rB: q(z_s|z_t,x) on the fragment atoms, or the final q draw on all atoms
  int rA = 1 + 2 * step, rC = -1;   // rC: the re-noise draw, or -1
  if constexpr (RES) {
    const int k = step / a.R, u = step - k * a.R;
    rA = 1 + k * (3 * a.R - 1) + 3 * u;
    if (step < a.T && u < a.R - 1) {
      rC = rA + 2;
      if (tid == 0) { renoise[3] = a.jump[2 * k]; renoise[4] = a.jump[2 * k + 1]; }   // read after the barriers below
    }
  }
  const int rB = rA + 1;
  const float* nA = a.rng.on ? nullptr : a.noise + (size_t)rA * slab;
  const float* nB = a.rng.on ? nullptr : a.noise + (size_t)rB * slab;
  const float* nC = a.rng.on || rC < 0 ? nullptr : a.noise + (size_t)rC * slab;
  float3 meanA{}, meanB{};
  if (a.rng.on) {
    meanA = com_free_means<PER_MOL>(a.rng, rA, b, N, a.nm, red);
    meanB = (RES ? step < a.T : com_free_on_fragments(rB, a.T)) ? com_free_means<PER_MOL>(a.rng, rB, b, N, a.fragment_mask, red)
                                                                : com_free_means<PER_MOL>(a.rng, rB, b, N, a.nm, red);
    if (RES && rC >= 0) {                                                  // uniform over the CTA
      const float3 mc = com_free_means<PER_MOL>(a.rng, rC, b, N, a.nm, red);
      if (tid == 0) { renoise[0] = mc.x; renoise[1] = mc.y; renoise[2] = mc.z; }
    }
  }
  if (step < a.T) {
    // pass 1: new latent before the centre-of-mass projection
    float cx = 0.f, cy = 0.f, cz = 0.f;
    for (int idx = tid; idx < N * xd; idx += 256) {
      const int n = idx / xd, d = idx - n * xd;
      const float m = a.nm[g0 + n], lm = a.linker_mask[g0 + n], fm = a.fragment_mask[g0 + n];
      const size_t gi = (g0 + n) * xd + d;
      float e = a.eps[gi];
      if (d < 3) e -= (d == 0 ? mvx : d == 1 ? mvy : mvz) * m;
      const float zt = a.z[gi];
      const float na = a.rng.on ? com_free_value<PER_MOL>(a.rng, rA, (int)(g0 + n), d, m, meanA) : nA[gi];
      const float nb = a.rng.on ? com_free_value<PER_MOL>(a.rng, rB, (int)(g0 + n), d, fm, meanB) : nB[gi];
      const float zl = (zt / ca - cb * e) + cc * na;                             // edm.py:634-642
      const float zf = (qa * zt + qb * (a.xh0[gi] * fm)) + cc * nb;               // edm.py:655-668
      const float zn = zl * lm + zf * fm;                                        // edm.py:589
      a.z[gi] = zn;
      if (d == 0) cx += zn; else if (d == 1) cy += zn; else if (d == 2) cz += zn;
    }
    cx = block_sum_256(cx, red); cy = block_sum_256(cy, red); cz = block_sum_256(cz, red);
    if (tid == 0) { means[0] = cx / cnt; means[1] = cy / cnt; means[2] = cz / cnt; }
    __syncthreads();
    for (int idx = tid; idx < N * xd; idx += 256) {
      const int n = idx / xd, d = idx - n * xd;
      const size_t gi = (g0 + n) * xd + d;
      float zn = a.z[gi];
      if (d < 3) { zn -= means[d] * a.nm[g0 + n]; a.z[gi] = zn; }                // edm.py:592, utils.py:56-63
      if (frame >= 0) a.chain[(size_t)frame * slab + gi] = d < 3 ? zn * a.norm0 : zn * a.norm1 + a.bias1;
      if (RES && rC >= 0) {
        const float m = a.nm[g0 + n];
        const float ec = a.rng.on ? com_free_value<PER_MOL>(a.rng, rC, (int)(g0 + n), d, m,
                                                            make_float3(renoise[0], renoise[1], renoise[2]))
                                  : nC[gi];
        a.z[gi] = __fadd_rn(__fmul_rn(renoise[3], zn), __fmul_rn(renoise[4], ec));
      }
    }
  } else {
    // final step: thread per atom, both variants and their argmax (edm.py:689-721)
    for (int n = tid; n < N; n += 256) {
      const float m = a.nm[g0 + n], lm = a.linker_mask[g0 + n], fm = a.fragment_mask[g0 + n];
      int bl = 0, bf = 0;
      float vl = -INFINITY, vf = -INFINITY;
      for (int d = 0; d < xd; ++d) {
        const size_t gi = (g0 + n) * xd + d;
        float e = a.eps[gi];
        if (d < 3) e -= (d == 0 ? mvx : d == 1 ? mvy : mvz) * m;
        const float zt = a.z[gi];
        const float na = a.rng.on ? com_free_value<PER_MOL>(a.rng, rA, (int)(g0 + n), d, m, meanA) : nA[gi];
        const float nb = a.rng.on ? com_free_value<PER_MOL>(a.rng, rB, (int)(g0 + n), d, m, meanB) : nB[gi];
        const float xl = ca * (zt - cb * e) + cc * na;                           // edm.py:701-702 (ca = 1/alpha_0, cb = sigma_0)
        const float xf = ca * zt - qa * nb;                                      // edm.py:716 (qa = sigma_0/alpha_0)
        if (d < 3) {
          a.chain[gi] = (xl * a.norm0) * lm + (xf * a.norm0) * fm;
        } else {
          const float hl = xl * a.norm1 + a.bias1, hf = xf * a.norm1 + a.bias1;
          if (hl > vl) { vl = hl; bl = d; }
          if (hf > vf) { vf = hf; bf = d; }
        }
      }
      for (int d = 3; d < xd; ++d)
        a.chain[(g0 + n) * xd + d] = ((d == bl ? 1.f : 0.f) * m) * lm + ((d == bf ? 1.f : 0.f) * m) * fm;
    }
  }
  if (tid == 0 && b == 0) {
    *a.step_prep = step + 1;
    if constexpr (RES) *a.step_tag = (step + 1) / a.R;
  }
}

// z0 = xh*fragment_mask + (noise[0]*linker_mask)*linker_mask   (edm.py:136-137)
template <bool PER_MOL = false>
__global__ void k_init_z(int n_total, int xd, const float* __restrict__ xh, const float* __restrict__ fm,
                         const float* __restrict__ lm, const float* __restrict__ noise, NoiseRng rng, float* __restrict__ z) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_total * xd) return;
  int g = idx / xd;
  float l = lm[g];
  const float nz = rng.on ? noise_draw<PER_MOL>(rng, 0, g, idx - g * xd) : noise[idx];
  z[idx] = xh[idx] * fm[g] + (nz * l) * l;
}

// Partial diffusion: z_t0 ~ q(z_t0 | x) on the linker, the input on the fragments, as EDM.forward noises (edm.py:69-74):
//   eps = noise[0]*linker_mask;  z_t0 = alpha_t0*xh + sigma_t0*eps;  z = xh*fragment_mask + z_t0*linker_mask
// Every product and sum is rounded on its own, as torch's elementwise ops round them (no contraction into FMAs).
template <bool PER_MOL = false>
__global__ void k_init_z_partial(int n_total, int xd, const float* __restrict__ xh, const float* __restrict__ fm,
                                 const float* __restrict__ lm, const float* __restrict__ noise, NoiseRng rng, float alpha,
                                 float sigma, float* __restrict__ z) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_total * xd) return;
  int g = idx / xd;
  const float l = lm[g], v = xh[idx];
  const float nz = rng.on ? noise_draw<PER_MOL>(rng, 0, g, idx - g * xd) : noise[idx];
  const float zt = __fadd_rn(__fmul_rn(alpha, v), __fmul_rn(sigma, __fmul_rn(nz, l)));
  z[idx] = __fadd_rn(__fmul_rn(v, fm[g]), __fmul_rn(zt, l));
}

// k_init_z_partial with per-molecule start steps (dl_set_start_steps): row b of the engine's order starts from its own
// alpha[b] and sigma[b], and reads draw 0 of a noise tensor at its caller row rows.src[b].
template <bool PER_MOL = false>
__global__ void k_init_z_rows(int n_total, int N, int xd, const float* __restrict__ xh, const float* __restrict__ fm,
                              const float* __restrict__ lm, const float* __restrict__ noise, NoiseRng rng,
                              const float* __restrict__ alpha, const float* __restrict__ sigma, RowStarts rows,
                              float* __restrict__ z) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_total * xd) return;
  const int g = idx / xd, b = g / N, d = idx - g * xd;
  const float l = lm[g], v = xh[idx];
  const float nz = rng.on ? noise_draw<PER_MOL>(rng, 0, g, d) : noise[((size_t)rows.src[b] * N + (g - b * N)) * xd + d];
  const float zt = __fadd_rn(__fmul_rn(alpha[b], v), __fmul_rn(sigma[b], __fmul_rn(nz, l)));
  z[idx] = __fadd_rn(__fmul_rn(v, fm[g]), __fmul_rn(zt, l));
}

// Fixed atoms (dl_set_fixed_atoms): after the start above, the kept linker rows start from q(z_t | x) of the input with the
// formula of k_init_z_rows -- the scalars alpha, sigma of the call's start, or alpha_rows[b], sigma_rows[b] of each row's
// own start step when given -- and the row's draw 0. Every other row keeps what the start wrote.
template <bool PER_MOL = false>
__global__ void k_init_z_fixed(int n_total, int N, int xd, const float* __restrict__ xh, const float* __restrict__ fm,
                               const float* __restrict__ lm, const int8_t* __restrict__ fixed,
                               const float* __restrict__ noise, NoiseRng rng, float alpha, float sigma,
                               const float* __restrict__ alpha_rows, const float* __restrict__ sigma_rows, RowStarts rows,
                               float* __restrict__ z) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_total * xd) return;
  const int g = idx / xd, b = g / N, d = idx - g * xd;
  if (fixed[g] == 0) return;
  const size_t gc = rows.src != nullptr ? (size_t)rows.src[b] * N + (g - b * N) : (size_t)g;
  const float al = alpha_rows != nullptr ? alpha_rows[b] : alpha, sg = sigma_rows != nullptr ? sigma_rows[b] : sigma;
  const float l = lm[g], v = xh[idx];
  const float nz = rng.on ? noise_draw<PER_MOL>(rng, 0, g, d) : noise[gc * xd + d];
  const float zt = __fadd_rn(__fmul_rn(al, v), __fmul_rn(sg, __fmul_rn(nz, l)));
  z[idx] = __fadd_rn(__fmul_rn(v, fm[g]), __fmul_rn(zt, l));
}

// dl_set_fixed_atoms' vetting of a call's flags: bad[0] = 1 + a node row whose flag is set but which
// is not a live linker row (node_mask, linker_mask != 0, fragment_mask == 0), bad[1] = 1 + a flagged row whose type channels are not a
// one-hot as normalised: exactly one channel equal to (1 - bias1) / norm1 and every other to (0 - bias1) / norm1.
__global__ void k_fixed_check(int n_total, int xd, const int8_t* __restrict__ fixed, const int8_t* __restrict__ node_mask,
                              const float* __restrict__ fm, const float* __restrict__ lm, const float* __restrict__ xh,
                              float norm1, float bias1, int* bad) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_total || fixed[g] == 0) return;
  if (node_mask[g] == 0 || lm[g] == 0.f || fm[g] != 0.f) atomicCAS(bad, 0, g + 1);
  const float one = __fdiv_rn(__fsub_rn(1.f, bias1), norm1), zero = __fdiv_rn(__fsub_rn(0.f, bias1), norm1);
  int ones = 0, others = 0;
  for (int d = 3; d < xd; ++d) {
    const float v = xh[(size_t)g * xd + d];
    ones += v == one;
    others += v != one && v != zero;
  }
  if (ones != 1 || others != 0) atomicCAS(bad + 1, 0, g + 1);
}

// dl_set_linker_types with dl_set_fixed_atoms: *bad = 1 + a flagged row whose type -- the channel equal to the normalised
// one, (1 - bias1) / norm1 -- its molecule's mask excludes. k_fixed_check vets the one-hot itself.
__global__ void k_kept_types_check(int n_total, int N, int xd, const int8_t* __restrict__ fixed, const float* __restrict__ xh,
                                   const uint32_t* __restrict__ masks, float norm1, float bias1, int* bad) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_total || fixed[g] == 0) return;
  const float one = __fdiv_rn(__fsub_rn(1.f, bias1), norm1);
  const uint32_t m = masks[g / N];
  for (int d = 3; d < xd; ++d)
    if (xh[(size_t)g * xd + d] == one && ((m >> (d - 3)) & 1u) == 0) atomicCAS(bad, 0, g + 1);
}

// Debug / test helper: the (n_draws, n_total, 3+F) tensor the device-side stream stands for.
__global__ void k_noise_fill(int n_draws, int n_total, int xd, NoiseRng rng, float* __restrict__ out) {
  const long long total = (long long)n_draws * n_total * xd;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int d = (int)(i % xd);
    const long long gi = i / xd;
    out[i] = noise_draw(rng, (int)(gi / n_total), (int)(gi % n_total), d);
  }
}

// Draws [0, gridDim.y) of the inpainting sampler's stream, masked and COM-projected, one CTA per (molecule, draw):
// out is (gridDim.y, B = gridDim.x, N, xd). All 2T+3 for dl_noise_fill_inpaint; draw 0 -- the initial z (edm.py:565) --
// straight into the workspace when the sampler draws on the device. RES: the 1 + T(3R-1) + 2 draws of R resampling passes.
template <bool PER_MOL = false, bool RES = false>
__global__ void __launch_bounds__(256) k_com_free_draws(int N, int xd, int T, NoiseRng rng, const int8_t* __restrict__ node_mask,
                                                        const float* __restrict__ fragment_mask, float* __restrict__ out,
                                                        int R = 1) {
  __shared__ float red[8];
  const int b = blockIdx.x, r = blockIdx.y;
  const bool frag = RES ? com_free_on_fragments(r, T, R) : com_free_on_fragments(r, T);
  const float3 mean = frag ? com_free_means<PER_MOL>(rng, r, b, N, fragment_mask, red)
                           : com_free_means<PER_MOL>(rng, r, b, N, node_mask, red);
  float* o = out + ((size_t)blockIdx.y * gridDim.x + b) * N * xd;
  for (int idx = threadIdx.x; idx < N * xd; idx += 256) {
    const int n = idx / xd, d = idx - n * xd, g = b * N + n;
    o[idx] = com_free_value<PER_MOL>(rng, r, g, d, frag ? fragment_mask[g] : (float)node_mask[g], mean);
  }
}

// SizeGNN head (linker_size.py:88-91 + linker_size_lightning.py:110): out[b] = mean over ALL N padded rows of
// embedding_out(h[b, n]) -- masked rows hold h = 0 and contribute the bias, exactly as in the reference.
// One CTA per molecule, warp per node (strided), lanes over channels; per-warp partial sums are combined in warp order.
constexpr int SZ_MAX_OUT = 64;
__global__ void __launch_bounds__(256) k_sz_out(int N, int out_nf, const float* __restrict__ h, const float* __restrict__ Wo,
                                               const float* __restrict__ bo, float* __restrict__ out) {
  __shared__ float part[8][SZ_MAX_OUT];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int o = lane; o < out_nf; o += 32) part[warp][o] = 0.f;
  __syncwarp();
  for (int n = warp; n < N; n += 8) {
    const float4 hv = *reinterpret_cast<const float4*>(h + ((size_t)b * N + n) * H + lane * 4);
    for (int o = 0; o < out_nf; ++o) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(Wo + (size_t)o * H + lane * 4));
      float s = hv.x * w.x + hv.y * w.y + hv.z * w.z + hv.w * w.w;
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


}  // namespace dl
