// Per-molecule NaN recovery (dl_sample_chain_retry): the seed of a molecule's next attempt, and the row gather /
// scatter between the caller's full batch and the sub-batch of the molecules that are sampled again.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <utility>

#include "bonds.cuh"

namespace dl {

// dl_retry_seed: attempt 0 (or below) is the molecule's own seed; attempt a >= 1 is output a of a splitmix64 generator
// started from the seed. For one attempt the map seed -> retry seed is a bijection, so distinct seeds never share a stream.
__host__ __device__ inline unsigned long long retry_seed(unsigned long long seed, int attempt) {
  if (attempt <= 0) return seed;
  unsigned long long z = seed + (unsigned long long)attempt * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// dl_size_uniform: the uniform in [0, 1) that draws a molecule's linker size from `seed` -- the top 53 bits of the
// splitmix64 finaliser of seed ^ SIZE_DRAW_TAG, times 2^-53. The tag keeps it apart from the Philox streams and from
// retry_seed, which feed no finaliser with it.
constexpr unsigned long long SIZE_DRAW_TAG = 0x6C696E6B65722D6Eull;   // "linker-n" in ASCII
__host__ __device__ inline double size_uniform(unsigned long long seed) {
  unsigned long long z = seed ^ SIZE_DRAW_TAG;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (double)(z >> 11) * 0x1.0p-53;
}

// The index dl_size_draw draws from the C logits l (stated at dl_size_draw in the header): in fp64 and in index order,
// m = max l, e_i = exp(l_i - m), S = sum e_i, c_i = e_0 + ... + e_i; the first i with u * S < c_i, else the last i with
// e_i > 0. Warp-collective (all 32 lanes, converged); every lane returns the index. The sums run in index order on every
// lane -- each lane adds the 32 values of a chunk one after another through shuffles -- so they are the sequential sums.
__device__ inline int size_draw_index(const float* l, int C, double u) {
  const int lane = threadIdx.x & 31;
  double m = -INFINITY;
  for (int i = lane; i < C; i += 32) m = fmax(m, (double)l[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  double S = 0.0;
  int last = 0;
  for (int i0 = 0; i0 < C; i0 += 32) {
    const double e = i0 + lane < C ? exp((double)l[i0 + lane] - m) : 0.0;
    for (int k = 0; k < 32 && i0 + k < C; ++k) S += __shfl_sync(0xffffffffu, e, k);
    const unsigned pos = __ballot_sync(0xffffffffu, e > 0.0);
    if (pos) last = i0 + 31 - __clz(pos);
  }
  const double t = u * S;
  double c = 0.0;
  for (int i0 = 0; i0 < C; i0 += 32) {
    const double e = i0 + lane < C ? exp((double)l[i0 + lane] - m) : 0.0;
    double mine = 0.0;
    for (int k = 0; k < 32 && i0 + k < C; ++k) {
      c += __shfl_sync(0xffffffffu, e, k);
      if (k == lane) mine = c;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, i0 + lane < C && t < mine);
    if (hit) return i0 + __ffs(hit) - 1;
  }
  return last;
}

// The size tables of a redraw (dl_size_redraw of the header), as the kernels read them.
struct SizeDrawArgs {
  int C, logits_stride;
  const float* logits;                   // (B, logits_stride): molecule b's C logits from column 0
  const int32_t* sizes;                  // (C)
};

// dl_size_draw: one warp per molecule b writes sizes[index drawn with size_uniform(retry_seed(seeds[b], attempt))].
__global__ void __launch_bounds__(256) k_size_draw(SizeDrawArgs a, int B, const unsigned long long* seeds, int attempt,
                                                   int32_t* out) {
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;                                 // whole warps leave together
  const int i = size_draw_index(a.logits + (size_t)b * a.logits_stride, a.C, size_uniform(retry_seed(seeds[b], attempt)));
  if ((threadIdx.x & 31) == 0) out[b] = a.sizes[i];
}

// One recovery round: the Bs failed molecules rows[i] (ascending batch rows) of the B-molecule batch. The src_* pointers
// are the caller's full-batch inputs, the dst_* ones the sub-batch workspace, row i holding molecule rows[i].
struct RowGatherArgs {
  const int* rows;
  int N, xd, C, attempt;
  const float *xh, *fragment_mask, *linker_mask, *context;
  const int8_t *node_mask, *edge_mask;   // edge_mask: FC graphs' (B,N,N) int8 blocks, or null (all ones / cut-off graphs)
  const unsigned long long* seeds;       // the caller's base seeds, or null: no seeds to gather
  float *s_xh, *s_fragment_mask, *s_linker_mask, *s_context;
  int8_t *s_node_mask, *s_edge_mask;
  unsigned long long* s_seeds;           // retry_seed(seeds[rows[i]], attempt)
};

// What a resizing round reads and writes besides RowGatherArgs / RowScatterArgs. Kernel parameters of their own, passed to
// the resizing instantiations only, so the code of the fixed-size ones stays as it was.
struct RowResizeArgs {
  SizeDrawArgs draw;
  const int32_t* n_frag;                 // (B) fragment rows of every molecule (pocket rows included)
  const float* linker_x;                 // (B, 3) the xh coordinates of molecule b's linker rows in its template
  int32_t* s_sizes;                      // (Bs) out: the size drawn for sub-batch row i
};
struct RowSizeArgs {
  const int32_t* s_sizes;                // (Bs) the sub-batch's sizes
  int32_t* sizes;                        // (B) the caller's sizes: written where a row is taken
};

// What the gather of a call with fixed atoms (dl_set_fixed_atoms) reads and writes besides RowGatherArgs: the caller's
// (B, N) flags and the sub-batch's. A kernel parameter of its own, as RowResizeArgs is.
struct RowFixedArgs {
  const int8_t* fixed;
  int8_t* s_fixed;
};

// One CTA per failed molecule: copies its rows of every input, and derives its seed for this attempt.
__device__ __forceinline__ void gather_rows(const RowGatherArgs& a) {
  const int i = blockIdx.x;
  const size_t b = a.rows[i], N = a.N;
  for (size_t k = threadIdx.x; k < N * a.xd; k += blockDim.x) a.s_xh[i * N * a.xd + k] = a.xh[b * N * a.xd + k];
  for (size_t k = threadIdx.x; k < N; k += blockDim.x) {
    a.s_node_mask[i * N + k] = a.node_mask[b * N + k];
    a.s_fragment_mask[i * N + k] = a.fragment_mask[b * N + k];
    a.s_linker_mask[i * N + k] = a.linker_mask[b * N + k];
  }
  if (a.context)
    for (size_t k = threadIdx.x; k < N * a.C; k += blockDim.x) a.s_context[i * N * a.C + k] = a.context[b * N * a.C + k];
  if (a.edge_mask)
    for (size_t k = threadIdx.x; k < N * N; k += blockDim.x) a.s_edge_mask[i * N * N + k] = a.edge_mask[b * N * N + k];
  if (threadIdx.x == 0 && a.seeds) a.s_seeds[i] = retry_seed(a.seeds[b], a.attempt);
}
template <bool RESIZE>
__global__ void __launch_bounds__(256) k_gather_rows(RowGatherArgs a) {
  static_assert(!RESIZE, "the resizing gather takes RowResizeArgs");
  gather_rows(a);
}
// ... and the molecule's fixed-atom flags.
template <bool RESIZE>
__global__ void __launch_bounds__(256) k_gather_rows(RowGatherArgs a, RowFixedArgs f) {
  static_assert(!RESIZE, "a size redraw takes no fixed atoms");
  gather_rows(a);
  const size_t b = a.rows[blockIdx.x], N = a.N;
  for (size_t k = threadIdx.x; k < N; k += blockDim.x) f.s_fixed[blockIdx.x * N + k] = f.fixed[b * N + k];
}

// The resizing gather: warp 0 draws the molecule's size s' with this attempt's seed, then the CTA writes the template of
// that size -- rows [0, n_frag) copied from the caller's input, rows [n_frag, n_frag + s') linker rows (node_mask 1,
// linker_mask 1, fragment_mask 0, x = linker_x[b], h 0, context 0), every later row zero, and on FC graphs the edge-mask
// block of batching._add_masks over the n_frag + s' live rows (-1 off the diagonal, -2 on it). The host guarantees
// n_frag + s' <= N.
template <bool RESIZE>
__global__ void __launch_bounds__(256) k_gather_rows(RowGatherArgs a, RowResizeArgs r) {
  static_assert(RESIZE, "only the resizing gather takes RowResizeArgs");
  __shared__ int s_live;
  const int i = blockIdx.x;
  const size_t b = a.rows[i], N = a.N;
  const unsigned long long seed = retry_seed(a.seeds[b], a.attempt);
  if (threadIdx.x < 32) {
    const int k = size_draw_index(r.draw.logits + b * r.draw.logits_stride, r.draw.C, size_uniform(seed));
    if (threadIdx.x == 0) {
      const int size = r.draw.sizes[k];
      s_live = r.n_frag[b] + size;
      r.s_sizes[i] = size;
      a.s_seeds[i] = seed;
    }
  }
  __syncthreads();
  const size_t nf = r.n_frag[b], live = s_live;
  for (size_t k = threadIdx.x; k < N * a.xd; k += blockDim.x) {
    const size_t n = k / a.xd, c = k - n * a.xd;
    a.s_xh[i * N * a.xd + k] = n < nf ? a.xh[b * N * a.xd + k] : (n < live && c < 3 ? r.linker_x[b * 3 + c] : 0.f);
  }
  for (size_t k = threadIdx.x; k < N; k += blockDim.x) {
    a.s_node_mask[i * N + k] = k < nf ? a.node_mask[b * N + k] : (int8_t)(k < live);
    a.s_fragment_mask[i * N + k] = k < nf ? a.fragment_mask[b * N + k] : 0.f;
    a.s_linker_mask[i * N + k] = k < nf ? a.linker_mask[b * N + k] : (k < live ? 1.f : 0.f);
  }
  if (a.context)
    for (size_t k = threadIdx.x; k < N * a.C; k += blockDim.x)
      a.s_context[i * N * a.C + k] = k / a.C < nf ? a.context[b * N * a.C + k] : 0.f;
  if (a.edge_mask)
    for (size_t k = threadIdx.x; k < N * N; k += blockDim.x) {
      const size_t p = k / N, q = k - p * N;
      a.s_edge_mask[i * N * N + k] = p < live && q < live ? (p == q ? (int8_t)-2 : (int8_t)-1) : (int8_t)0;
    }
}

struct RowScatterArgs {
  const int* rows;
  int B, Bs, N, xd, attempt;
  const float* s_chain;                  // (keep_frames, Bs, N, xd)
  const int32_t* s_flags;
  const unsigned long long* s_seeds;
  float* chain;                          // (keep_frames, B, N, xd)
  int32_t* flags;
  unsigned long long* seeds_used;
  int32_t* attempts;
  // CHECKED rounds only: take[i] (k_molecule_check) says whether sub-batch row i replaces the caller's row; s_passed /
  // passed are the sub-batch's and the caller's check verdicts
  const int32_t *take, *s_passed;
  int32_t* passed;
};

// grid (Bs, keep_frames): CTA (i, f) writes frame f of sub-batch row i over row rows[i] of the caller's chain; the f = 0
// CTAs also write the molecule's flags, the seed that produced the row and the attempt. CHECKED: only rows with take[i]
// set, and their check verdicts with them.
// SIZED (resizing rounds, with RowSizeArgs): the f = 0 CTAs also write the row's size.
template <bool CHECKED, bool SIZED>
__device__ __forceinline__ void scatter_rows(const RowScatterArgs& a, const RowSizeArgs& z) {
  const int i = blockIdx.x, f = blockIdx.y;
  if (CHECKED && !a.take[i]) return;
  const size_t b = a.rows[i], row = (size_t)a.N * a.xd;
  const float* src = a.s_chain + ((size_t)f * a.Bs + i) * row;
  float* dst = a.chain + ((size_t)f * a.B + b) * row;
  for (size_t k = threadIdx.x; k < row; k += blockDim.x) dst[k] = src[k];
  if (f == 0 && threadIdx.x == 0) {
    a.flags[b] = a.s_flags[i];
    a.seeds_used[b] = a.s_seeds[i];
    a.attempts[b] = a.attempt;
    if (CHECKED) a.passed[b] = a.s_passed[i];
    if (SIZED) z.sizes[b] = z.s_sizes[i];
  }
}

template <bool CHECKED>
__global__ void __launch_bounds__(256) k_scatter_rows(RowScatterArgs a) {
  scatter_rows<CHECKED, false>(a, RowSizeArgs{});
}

template <bool CHECKED>
__global__ void __launch_bounds__(256) k_scatter_rows(RowScatterArgs a, RowSizeArgs z) {
  scatter_rows<CHECKED, true>(a, z);
}

// ---- molecule checks: is the final molecule in one piece, and is every atom within its valence? -----------------------
// The atoms of molecule b are its rows n with node_mask != 0, minus the pocket atoms (context column C - 1 set) when
// drop_pocket, with types argmax(h[:n_types]).
// CHECK_CONNECTED: atoms i and j bond iff bond_pair (get_bond_order > 0); the bit is set iff that graph has exactly one
// component (a single atom is connected, no atom is not): len(Chem.GetMolFrags(mol)) == 1 for the molecule build_molecule
// makes of them (lightning.py:364-377, metrics.py:20-27).
// CHECK_VALENCE: an atom's valence is the sum of bond_order_pair (get_bond_order) over the other checked atoms; the bit is
// set iff every atom's valence is <= max_valence[its type] (no atom: set).
// Both measure a pair as torch.cdist does over the n checked atoms, the later atom first (bonds.cuh): n counts the atoms
// after drop_pocket, and the linker hash of CHECK_NOVEL measures over the linker atoms alone.
// CHECK_CLASH (always with drop_pocket): the linker atoms are the checked atoms with linker_mask != 0, the pocket atoms the
// rows with node_mask != 0 and context column C - 1 != 0; the bit is set iff no linker atom clashes (clash_pair) with any
// pocket atom (no linker or no pocket atom: set). The predicates are stated in full at dl_molecule_checks in the header.
// CHECK_UNIQUE: the kernel writes each molecule's graph hash (stated at DL_CHECK_UNIQUE in the header) and leaves the bit
// clear; k_unique_verdict sets it, since it compares molecules with each other.
// CHECK_NOVEL: the bit is set iff the linker hash L -- the graph hash of the checked atoms with linker_mask != 0 -- is not
// in the caller's sorted set of known linker hashes (stated at DL_CHECK_NOVEL in the header).
// CHECK_RINGS: the bit is set iff the molecule's ring-size mask -- the smallest ring of every bond with a linker end, over
// the graph of all its checked atoms -- lies inside the caller's allowed mask (stated at DL_CHECK_RINGS in the header).
// CHECK_ANCHORS: the bit is set iff the linker bonds to each anchor by exactly one bond and to no other fragment atom
// (stated at DL_CHECK_ANCHORS in the header). It runs in k_anchor_check, a launch of its own after k_molecule_check.
constexpr int CHECK_CONNECTED = 1, CHECK_VALENCE = 2, CHECK_CLASH = 4, CHECK_UNIQUE = 8;   // DL_CHECK_* of the header
constexpr int CHECK_NOVEL = 16, CHECK_RINGS = 32, CHECK_ANCHORS = 64;
constexpr int CONN_MAX_N = 8192;                                     // rows per molecule: 20 bytes of shared memory each
constexpr int CONN_SMEM_MAX = CONN_MAX_N * (int)(sizeof(float4) + sizeof(int));
// With CHECK_UNIQUE a molecule also takes 8 bytes per row (the atoms' rows and the CSR offsets) and 4 bytes per stored
// directed bond: up to HASH_EDGES_PER_ROW per row, within the opt-in shared memory of a block on sm_90 (227 KB, less the
// kernel's static shared memory).
constexpr int HASH_SMEM_MAX = 226 * 1024;
constexpr int HASH_EDGES_PER_ROW = 16;
constexpr unsigned long long GRAPH_HASH_TAG = 0x67726170682D776Cull;   // "graph-wl" in ASCII
constexpr unsigned long long GRAPH_HASH_ORDER = 0x9E3779B97F4A7C15ull;

// mix() of the graph hash: the splitmix64 finaliser of size_uniform.
__host__ __device__ inline unsigned long long hash_mix(unsigned long long z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// What CHECK_UNIQUE writes besides CheckArgs, a kernel parameter of the instantiations with the bit only.
struct HashArgs {
  unsigned long long* hash;              // (B) out: every molecule's graph hash
  int edge_cap;                          // directed bonds the shared-memory CSR holds (set by launch_molecule_check_as)
};

struct CheckArgs {
  const float* xh;                       // (B, N, row_stride): x at columns 0..2, h from column 3 -- chain[0]
  int N, row_stride, n_types, C, drop_pocket;
  const float *thr1, *thr2, *thr3;       // (n_types, n_types) bond thresholds in pm, [min type][max type]; thr2, thr3 and
  const int32_t* max_valence;            // max_valence (n_types) are read by CHECK_VALENCE only
  const int8_t* node_mask;               // (B, N)
  const float* context;                  // (B, N, C); read only when drop_pocket
  int32_t* passed;                       // (B) out: OR of the CHECK_* bits the molecule satisfies, among those checked
  int32_t* valence;                      // (B, N) or null: the valence of every checked row (CHECK_VALENCE; other rows are
                                         // not written)
  // recovery rounds (rows != null): the molecules are sub-batch rows; take[i] = whether row i replaces the caller's row
  // rows[i] -- always, unless the caller's row is finite (flags == 0) and the resampled one diverged
  const int* rows;
  const int32_t *flags, *s_flags;
  int32_t* take;
};

// What CHECK_CLASH reads and writes besides CheckArgs. It is a kernel parameter of its own, passed to the instantiations
// with the clash bit only: CheckArgs is 128 bytes, and any field appended to it changes the code ptxas generates for the
// other instantiations.
struct ClashArgs {
  const float* linker_mask;              // (B, N): the checked atoms with linker_mask != 0 are the linker atoms
  const float* clash;                    // (n_types, n_types) clash distances in pm, [min type][max type]
  int32_t* clashes;                      // (B, N) or null: every linker atom's count of pocket atoms it clashes with (other
                                         // rows are not written)
};

// What CHECK_NOVEL reads besides CheckArgs, a kernel parameter of the instantiations with the bit only.
struct NovelArgs {
  const float* linker_mask;              // (B, N): the checked atoms with linker_mask != 0 are the linker atoms
  const unsigned long long* known;       // (n_known) ascending, unsigned order: the known linker hashes
  long long n_known;
  unsigned long long* linker_hash;       // out or null: molecule b's L at row b, or in a recovery round (CheckArgs::rows)
                                         // at the caller's row rows[b], where the row is taken
};

// What CHECK_RINGS reads and writes besides CheckArgs: NovelArgs, whose linker_mask it shares, and its own fields. The
// instantiations with the bit take it in place of NovelArgs, and molecule_check reads the fields below through its NovelArgs
// reference, so that the other instantiations keep their code (their shared variables' names follow its signature).
struct RingArgs : NovelArgs {
  unsigned long long allowed;            // bit k set: a smallest ring of k atoms passes (bit 63: of 63 or more)
  unsigned long long* ring_sizes;        // out or null: molecule b's mask at row b, or in a recovery round (CheckArgs::rows)
                                         // at the caller's row rows[b], where the row is taken
};
// The ring stage's breadth-first searches keep three bitsets over the rows per warp: visited, frontier and next frontier.
constexpr int RING_BITSETS = 3 * 8;

// Whether v is among s[0, n), ascending in unsigned order (duplicates allowed): a binary search for the first entry >= v,
// with 64-bit indices and unsigned compares.
__host__ __device__ inline bool sorted_contains(const unsigned long long* s, long long n, unsigned long long v) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (s[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && s[lo] == v;
}

// An atom's type, the rule of every check and of clash guidance: torch.argmax over the row's n_types type channels (from
// column 3), i.e. the first maximum, NaN winning. k_clash_guide calls it. load_atom and molecule_check's two staging loops
// spell the same loop out: routed through this function, all 65 k_molecule_check and k_anchor_check instantiations
// compile to different SASS, so they keep their own copies, which must stay the same as this one.
__device__ __forceinline__ int first_type(const float* row, int n_types) {
  int best = 0;
  for (int k = 1; k < n_types; ++k) {
    const float v = row[3 + k], cur = row[3 + best];
    if (v > cur || (isnan(v) && !isnan(cur))) best = k;
  }
  return best;
}

// Row r of the molecule at g0 as the staging below makes its atom: x, y, z and the type (first_type's rule) as int bits.
// The graph hash reads the atoms whose bonds do not fit its shared-memory CSR this way.
__device__ __forceinline__ float4 load_atom(const CheckArgs& a, size_t g0, int r) {
  const float* row = a.xh + (g0 + r) * a.row_stride;
  int best = 0;
  for (int k = 1; k < a.n_types; ++k) {
    const float v = row[3 + k], cur = row[3 + best];
    if (v > cur || (isnan(v) && !isnan(cur))) best = k;
  }
  return make_float4(row[0], row[1], row[2], __int_as_float(best));
}

// The staged atoms i != j (coordinates and type bits) of a molecule of n checked atoms, as a pair of bonds.cuh: the later
// atom max(i, j) first, the orientation torch.cdist's matrix is read in (dists[i, j], i > j).
__device__ __forceinline__ bool staged_bonded(const CheckArgs& a, int i, float4 pi, int j, float4 pj, int n) {
  const float4 p = i > j ? pi : pj, q = i > j ? pj : pi;
  float dist;
  return bond_pair(make_float3(p.x, p.y, p.z), make_float3(q.x, q.y, q.z), __float_as_int(p.w), __float_as_int(q.w),
                   a.n_types, a.thr1, n, &dist) >= 0;
}

__device__ __forceinline__ int staged_order(const CheckArgs& a, int i, float4 pi, int j, float4 pj, int n) {
  const float4 p = i > j ? pi : pj, q = i > j ? pj : pi;
  return bond_order_pair(make_float3(p.x, p.y, p.z), make_float3(q.x, q.y, q.z), __float_as_int(p.w), __float_as_int(q.w),
                         a.n_types, a.thr1, a.thr2, a.thr3, n);
}

// The graph hash of the n staged atoms s_at[0, n) (rows s_row), stated at DL_CHECK_UNIQUE in the header: R = min(n, 64)
// rounds of colour refinement c' (i) = mix(c(i) + sum over bonded j of mix(c(j) + o_ij * GRAPH_HASH_ORDER)), then
// H = mix(n + sum_i c(i)). Block-collective; returns H on every thread.
// The bonds are found once: a warp per atom counts them (all pairs, bond_pair), the counts are scanned into CSR offsets in
// s_off, and a warp per atom writes its neighbours j | order << 16 in ascending j into s_edge. Atoms whose list would end
// beyond edge_cap (a prefix of the atoms is stored, since the offsets ascend) rescan every atom in every round, reading the
// rows from global memory (load_atom). The colours then live over s_at, two arrays of N, and the rounds add integers only:
// the hash does not depend on the order the lanes add in.
__device__ __forceinline__ unsigned long long graph_hash(const CheckArgs& a, const HashArgs& hk, size_t g0, int n,
                                                        float4* s_at, int* s_off, const int* s_row, unsigned* s_edge) {
  __shared__ int s_wsum[8], s_e;
  __shared__ unsigned long long s_hsum[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = warp; i < n; i += 8) {                 // degrees
    const float4 pi = s_at[i];
    int d = 0;
    for (int j = lane; j < n; j += 32) {
      const float4 pj = s_at[j];
      d += j != i && staged_bonded(a, i, pi, j, pj, n);
    }
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) s_off[i] = d;
  }
  if (tid == 0) s_e = 0;
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += 256) {               // exclusive scan of the degrees, 256 atoms at a time
    const int i = i0 + tid;
    const int v = i < n ? s_off[i] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_wsum[warp] = x;
    __syncthreads();
    int before = s_e, total = 0;
    for (int w = 0; w < 8; ++w) { before += w < warp ? s_wsum[w] : 0; total += s_wsum[w]; }
    if (i < n) s_off[i] = before + x - v;
    __syncthreads();
    if (tid == 0) s_e += total;
    __syncthreads();
  }
  const int E = s_e;
  auto end_of = [&](int i) { return i + 1 < n ? s_off[i + 1] : E; };
  for (int i = warp; i < n; i += 8) {                 // the stored lists
    const int start = s_off[i];
    if (end_of(i) > hk.edge_cap) continue;
    const float4 pi = s_at[i];
    int at = start;
    for (int j0 = 0; j0 < n; j0 += 32) {
      const int j = j0 + lane;
      int o = 0;
      if (j < n && j != i) {
        const float4 pj = s_at[j];
        o = staged_order(a, i, pi, j, pj, n);
      }
      const unsigned m = __ballot_sync(0xffffffffu, o > 0);
      if (o > 0) s_edge[at + __popc(m & ((1u << lane) - 1u))] = (unsigned)j | ((unsigned)o << 16);
      at += __popc(m);
    }
  }
  __syncthreads();
  unsigned long long* c = reinterpret_cast<unsigned long long*>(s_at);   // [N]: this round's colours
  unsigned long long* c2 = c + a.N;                                        // [N]: the next round's
  for (int i0 = 0; i0 < n; i0 += 256) {               // c_0, over the atoms of this chunk and the ones before it only
    const int i = i0 + tid;
    const int t = i < n ? __float_as_int(s_at[i].w) : 0;
    __syncthreads();
    if (i < n) c[i] = hash_mix(GRAPH_HASH_TAG ^ (unsigned long long)(t + 1));
  }
  __syncthreads();
  const int R = min(n, 64);
  for (int k = 0; k < R; ++k) {
    for (int i = warp; i < n; i += 8) {
      unsigned long long s = 0;
      const int start = s_off[i], end = end_of(i);
      if (end <= hk.edge_cap) {
        for (int e = start + lane; e < end; e += 32) {
          const unsigned v = s_edge[e];
          s += hash_mix(c[v & 0xffffu] + (unsigned long long)(v >> 16) * GRAPH_HASH_ORDER);
        }
      } else {
        const float4 pi = load_atom(a, g0, s_row[i]);
        for (int j = lane; j < n; j += 32) {
          if (j == i) continue;
          const float4 pj = load_atom(a, g0, s_row[j]);
          const int o = staged_order(a, i, pi, j, pj, n);
          if (o > 0) s += hash_mix(c[j] + (unsigned long long)o * GRAPH_HASH_ORDER);
        }
      }
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) c2[i] = hash_mix(c[i] + s);
    }
    __syncthreads();
    unsigned long long* t = c; c = c2; c2 = t;
  }
  unsigned long long s = 0;
  for (int i = tid; i < n; i += 256) s += c[i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) s_hsum[warp] = s;
  __syncthreads();
  s = (unsigned long long)n;
  for (int w = 0; w < 8; ++w) s += s_hsum[w];
  return hash_mix(s);
}

// The ring-size mask of the n staged atoms s_at[0, n), s_link[i] != 0 for a linker atom (stated at DL_CHECK_RINGS in the
// header). Block-collective; returns the mask on every thread.
// The bonds are found once into a CSR of neighbour indices (s_off, s_edge), as graph_hash finds them: atoms whose list
// would end beyond edge_cap find their neighbours by testing every staged atom instead. Then a warp per atom u takes each
// bond (u, v > u) with a linker end and searches breadth-first from u, level by level, for v in the graph without that
// bond: bottom-up, each lane asks whether an atom not yet reached has a neighbour on the frontier, and a ballot writes 32
// atoms' answers as one word of the next frontier. v reached at level d closes a smallest ring of d + 1 atoms. Bits are only
// ever ORed into a warp's own register and then over the warps, so the mask does not depend on the order the warps run in.
__device__ __forceinline__ unsigned long long ring_mask(const CheckArgs& a, int edge_cap, int n, const float4* s_at,
                                                        int* s_off, const int* s_link, unsigned* s_bits, int* s_edge) {
  __shared__ int s_wsum[8], s_e;
  __shared__ unsigned long long s_rmask[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = warp; i < n; i += 8) {                 // degrees
    const float4 pi = s_at[i];
    int d = 0;
    for (int j = lane; j < n; j += 32) d += j != i && staged_bonded(a, i, pi, j, s_at[j], n);
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) s_off[i] = d;
  }
  if (tid == 0) s_e = 0;
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += 256) {               // exclusive scan of the degrees, 256 atoms at a time
    const int i = i0 + tid;
    const int v = i < n ? s_off[i] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_wsum[warp] = x;
    __syncthreads();
    int before = s_e, total = 0;
    for (int w = 0; w < 8; ++w) { before += w < warp ? s_wsum[w] : 0; total += s_wsum[w]; }
    if (i < n) s_off[i] = before + x - v;
    __syncthreads();
    if (tid == 0) s_e += total;
    __syncthreads();
  }
  const int E = s_e;
  auto end_of = [&](int i) { return i + 1 < n ? s_off[i + 1] : E; };
  for (int i = warp; i < n; i += 8) {                 // the stored lists, ascending
    if (end_of(i) > edge_cap) continue;
    const float4 pi = s_at[i];
    int at = s_off[i];
    for (int j0 = 0; j0 < n; j0 += 32) {
      const int j = j0 + lane;
      const bool bonded = j < n && j != i && staged_bonded(a, i, pi, j, s_at[j], n);
      const unsigned m = __ballot_sync(0xffffffffu, bonded);
      if (bonded) s_edge[at + __popc(m & ((1u << lane) - 1u))] = j;
      at += __popc(m);
    }
  }
  __syncthreads();
  const int W = (n + 31) >> 5, WN = (a.N + 31) >> 5;
  unsigned* vis = s_bits + warp * 3 * WN;
  unsigned long long mask = 0;
  for (int u = warp; u < n; u += 8) {
    const bool stored_u = end_of(u) <= edge_cap;
    const float4 pu = s_at[u];
    // the neighbours v > u of u, 32 candidates at a time: from its list, or by testing every later atom
    for (int k0 = stored_u ? s_off[u] : u + 1, k_end = stored_u ? end_of(u) : n; k0 < k_end; k0 += 32) {
      const int k = k0 + lane;
      int v = -1;
      if (k < k_end) {
        if (stored_u) v = s_edge[k] > u ? s_edge[k] : -1;
        else v = staged_bonded(a, u, pu, k, s_at[k], n) ? k : -1;
      }
      unsigned todo = __ballot_sync(0xffffffffu, v >= 0 && (s_link[u] != 0 || s_link[v] != 0));
      while (todo) {                                  // one bond (u, v) at a time, the whole warp on it
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int vv = __shfl_sync(0xffffffffu, v, src);
        unsigned *fr = vis + WN, *nx = fr + WN;
        for (int w = lane; w < W; w += 32) {
          const unsigned m = w == (u >> 5) ? 1u << (u & 31) : 0u;
          vis[w] = m;
          fr[w] = m;
        }
        __syncwarp();
        int ring = 0;
        for (int d = 1;; ++d) {                       // level d: the atoms at distance d from u
          unsigned any = 0;
          bool found = false;
          for (int w = 0; w < W; ++w) {
            const int j = (w << 5) + lane;
            bool hit = false;
            if (j < n && !((vis[w] >> lane) & 1u)) {
              auto on_frontier = [&](int q) { return (j != vv || q != u) && ((fr[q >> 5] >> (q & 31)) & 1u); };
              if (end_of(j) <= edge_cap) {
                for (int e = s_off[j], e_end = end_of(j); e < e_end && !hit; ++e) hit = on_frontier(s_edge[e]);
              } else {
                const float4 pj = s_at[j];
                for (int q = 0; q < n && !hit; ++q) hit = q != j && on_frontier(q) && staged_bonded(a, j, pj, q, s_at[q], n);
              }
            }
            const unsigned m = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) nx[w] = m;
            any |= m;
            found |= w == (vv >> 5) && ((m >> (vv & 31)) & 1u);
          }
          if (found) { ring = d + 1; break; }
          if (!any) break;
          __syncwarp();
          for (int w = lane; w < W; w += 32) vis[w] |= nx[w];
          unsigned* t = fr; fr = nx; nx = t;
          __syncwarp();
        }
        __syncwarp();                                 // the next bond's search resets the bitsets
        if (ring) mask |= 1ull << min(ring, 63);
      }
    }
  }
  if (lane == 0) s_rmask[warp] = mask;
  __syncthreads();
  mask = 0;
  for (int w = 0; w < 8; ++w) mask |= s_rmask[w];
  return mask;
}

// One CTA per molecule. The checked atoms are compacted, in row order, into shared memory (coordinates and type; padded
// and pocket rows are never read beyond their masks).
// Valence: a warp per atom sums the integer bond orders of its pairs with every other atom, so the sums do not depend on
// the order the lanes add in.
// Components are found by min-label hooking: every bonded pair whose trees differ hooks the larger root under the smaller
// (atomicMin), trees are flattened, and this repeats until a pass over all pairs hooks nothing. Labels only ever decrease
// and each root is its tree's smallest atom, so the final labels -- every atom's component minimum -- and the flag do not
// depend on the order the threads hook in.
// Clash: the pocket atoms are compacted into the same buffer from its back, s_at[N - 1 - k] (the checked atoms and the
// pocket atoms are disjoint rows, so the two never meet), and s_lab[i] holds atom i's row with bit 31 set for a linker
// atom until the clash pass is done. A warp per linker atom counts, in integers, the pocket atoms it clashes with; the
// count and the verdict do not depend on the order the lanes add in.
// Hash (CHECK_UNIQUE): s_row[i] keeps atom i's row, and after the other checks graph_hash takes over the buffer: s_lab
// holds the CSR offsets, the bonds follow s_row, and the colours overwrite s_at.
// Linker hash (CHECK_NOVEL): last, the linker atoms are staged again from global memory, in row order, over whatever the
// checks above left in the buffer, and graph_hash runs on them alone.
// Rings (CHECK_RINGS): last, every checked atom is staged again from global memory, in row order, with its linker flag in
// s_row; ring_mask builds its CSR over s_lab and the bitsets and bonds after s_row.
// The body of the k_molecule_check kernels below; cl is read with CHECK_CLASH only, hk with CHECK_UNIQUE, CHECK_NOVEL or
// CHECK_RINGS (its edge_cap) only, nv with CHECK_NOVEL or CHECK_RINGS only.
template <int CHECKS>
__device__ __forceinline__ void molecule_check(const CheckArgs& a, const ClashArgs& cl, const HashArgs& hk,
                                               const NovelArgs& nv) {
  extern __shared__ float4 s_at[];                    // [n]: x, y, z, type (int bits)
  int* s_lab = reinterpret_cast<int*>(s_at + a.N);    // [n]: the atoms' rows (valence), then parent pointers (components)
  int* s_row = s_lab + a.N;                           // [n] (CHECK_UNIQUE): the atoms' rows
  __shared__ int s_warp[8], s_n, s_changed;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x;
  const size_t g0 = (size_t)b * a.N;
  int n_pocket = 0;
  if constexpr ((CHECKS & CHECK_CLASH) != 0) {
    __shared__ int s_pwarp[8], s_np;
    if (tid == 0) s_n = s_np = 0;
    __syncthreads();
    for (int r0 = 0; r0 < a.N; r0 += 256) {
      const int r = r0 + tid;
      const bool live = r < a.N && a.node_mask[g0 + r] != 0;
      const bool ok = live && a.context[(g0 + r) * a.C + a.C - 1] == 0.f, pocket = live && !ok;
      const bool linker = ok && cl.linker_mask[g0 + r] != 0.f;
      const unsigned m = __ballot_sync(0xffffffffu, ok), mp = __ballot_sync(0xffffffffu, pocket);
      if (lane == 0) { s_warp[warp] = __popc(m); s_pwarp[warp] = __popc(mp); }
      __syncthreads();
      const unsigned below = (1u << lane) - 1u;
      int off = s_n + __popc(m & below), poff = s_np + __popc(mp & below), total = 0, ptotal = 0;
      for (int w = 0; w < 8; ++w) {
        off += w < warp ? s_warp[w] : 0; total += s_warp[w];
        poff += w < warp ? s_pwarp[w] : 0; ptotal += s_pwarp[w];
      }
      if (ok || pocket) {
        const float* row = a.xh + (g0 + r) * a.row_stride;
        int best = 0;                                 // torch.argmax: the first maximum; NaN wins
        for (int k = 1; k < a.n_types; ++k) {
          const float v = row[3 + k], cur = row[3 + best];
          if (v > cur || (isnan(v) && !isnan(cur))) best = k;
        }
        const float4 at = make_float4(row[0], row[1], row[2], __int_as_float(best));
        if (ok) {
          s_at[off] = at;
          s_lab[off] = r | (linker ? (int)0x80000000u : 0);
          if (CHECKS & CHECK_UNIQUE) s_row[off] = r;
        } else {
          s_at[a.N - 1 - poff] = at;
        }
      }
      __syncthreads();
      if (tid == 0) { s_n += total; s_np += ptotal; }
      __syncthreads();
    }
    n_pocket = s_np;
  } else {
    if (tid == 0) s_n = 0;
    __syncthreads();
    for (int r0 = 0; r0 < a.N; r0 += 256) {
      const int r = r0 + tid;
      bool ok = r < a.N && a.node_mask[g0 + r] != 0;
      if (ok && a.drop_pocket) ok = a.context[(g0 + r) * a.C + a.C - 1] == 0.f;
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) s_warp[warp] = __popc(m);
      __syncthreads();
      int off = s_n + __popc(m & ((1u << lane) - 1u)), total = 0;
      for (int w = 0; w < 8; ++w) { off += w < warp ? s_warp[w] : 0; total += s_warp[w]; }
      if (ok) {
        const float* row = a.xh + (g0 + r) * a.row_stride;
        int best = 0;                                 // torch.argmax: the first maximum; NaN wins
        for (int k = 1; k < a.n_types; ++k) {
          const float v = row[3 + k], cur = row[3 + best];
          if (v > cur || (isnan(v) && !isnan(cur))) best = k;
        }
        s_at[off] = make_float4(row[0], row[1], row[2], __int_as_float(best));
        s_lab[off] = (CHECKS & CHECK_VALENCE) ? r : off;
        if (CHECKS & CHECK_UNIQUE) s_row[off] = r;
      }
      __syncthreads();
      if (tid == 0) s_n += total;
      __syncthreads();
    }
  }
  const int n = s_n;
  int verdict = 0;
  if constexpr ((CHECKS & CHECK_CLASH) != 0) {
    int hit = 0;
    for (int i = warp; i < n; i += 8) {               // warp per linker atom i, lanes over the pocket atoms
      const int tag = s_lab[i];
      if (tag >= 0) continue;                         // not a linker atom: bit 31 clear
      const float4 pi = s_at[i];
      int c = 0;
      for (int j = lane; j < n_pocket; j += 32) {
        const float4 pj = s_at[a.N - 1 - j];
        c += clash_pair(make_float3(pi.x, pi.y, pi.z), make_float3(pj.x, pj.y, pj.z), __float_as_int(pi.w),
                        __float_as_int(pj.w), a.n_types, cl.clash);
      }
      for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
      if (lane == 0) {
        hit |= c > 0;
        if (cl.clashes) cl.clashes[g0 + (tag & 0x7fffffff)] = c;
      }
    }
    if (!__syncthreads_or(hit)) verdict |= CHECK_CLASH;
    if (CHECKS & (CHECK_CONNECTED | CHECK_VALENCE)) {   // what the other checks expect: rows (valence) or labels
      for (int i = tid; i < n; i += 256) s_lab[i] = (CHECKS & CHECK_VALENCE) ? (s_lab[i] & 0x7fffffff) : i;
      __syncthreads();
    }
  }
  if (CHECKS & CHECK_VALENCE) {
    int over = 0;
    for (int i = warp; i < n; i += 8) {               // warp per atom i, lanes over its partners j != i
      const float4 pi = s_at[i];
      int v = 0;
      for (int j = lane; j < n; j += 32) {
        const float4 pj = s_at[j];
        if (j != i) v += staged_order(a, i, pi, j, pj, n);
      }
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) {
        over |= v > a.max_valence[__float_as_int(pi.w)];
        if (a.valence) a.valence[g0 + s_lab[i]] = v;
      }
    }
    if (!__syncthreads_or(over)) verdict |= CHECK_VALENCE;
    if (CHECKS & CHECK_CONNECTED) {
      for (int i = tid; i < n; i += 256) s_lab[i] = i;
      __syncthreads();
    }
  }
  if (CHECKS & CHECK_CONNECTED) {
    volatile int* lab = s_lab;
    for (;;) {
      if (tid == 0) s_changed = 0;
      __syncthreads();
      for (int i = warp; i < n; i += 8) {             // warp per row i, lanes over the pairs (i, j < i)
        const float4 pi = s_at[i];
        for (int j = lane; j < i; j += 32) {
          const float4 pj = s_at[j];
          if (!staged_bonded(a, i, pi, j, pj, n)) continue;
          int ri = i, rj = j;
          while (lab[ri] != ri) ri = lab[ri];
          while (lab[rj] != rj) rj = lab[rj];
          if (ri != rj) {
            atomicMin(&s_lab[max(ri, rj)], min(ri, rj));
            s_changed = 1;
          }
        }
      }
      __syncthreads();
      const int changed = s_changed;
      for (int i = tid; i < n; i += 256) {            // flatten: every atom points at its root
        int r = i;
        while (lab[r] != r) r = lab[r];
        lab[i] = r;
      }
      __syncthreads();
      if (!changed) break;
    }
    int roots = 0;
    for (int i0 = 0; i0 < n; i0 += 256) roots += __syncthreads_count(i0 + tid < n && lab[i0 + tid] == i0 + tid);
    if (roots == 1) verdict |= CHECK_CONNECTED;
  }
  if constexpr ((CHECKS & CHECK_UNIQUE) != 0) {
    __syncthreads();                                  // s_lab is read above until here
    const unsigned long long h = graph_hash(a, hk, g0, n, s_at, s_lab, s_row, reinterpret_cast<unsigned*>(s_row + a.N));
    if (tid == 0) hk.hash[b] = h;
  }
  if constexpr ((CHECKS & CHECK_NOVEL) != 0) {
    __syncthreads();                                  // the buffer is read above until here
    if (tid == 0) s_n = 0;
    __syncthreads();
    for (int r0 = 0; r0 < a.N; r0 += 256) {           // the linker atoms: checked atoms with linker_mask != 0
      const int r = r0 + tid;
      bool ok = r < a.N && a.node_mask[g0 + r] != 0 && nv.linker_mask[g0 + r] != 0.f;
      if (ok && a.drop_pocket) ok = a.context[(g0 + r) * a.C + a.C - 1] == 0.f;
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) s_warp[warp] = __popc(m);
      __syncthreads();
      int off = s_n + __popc(m & ((1u << lane) - 1u)), total = 0;
      for (int w = 0; w < 8; ++w) { off += w < warp ? s_warp[w] : 0; total += s_warp[w]; }
      if (ok) {
        s_at[off] = load_atom(a, g0, r);
        s_row[off] = r;
      }
      __syncthreads();
      if (tid == 0) s_n += total;
      __syncthreads();
    }
    const int n_linker = s_n;
    const unsigned long long l = graph_hash(a, hk, g0, n_linker, s_at, s_lab, s_row,
                                            reinterpret_cast<unsigned*>(s_row + a.N));
    if (tid == 0) {
      if (!sorted_contains(nv.known, nv.n_known, l)) verdict |= CHECK_NOVEL;
      if (nv.linker_hash) {                           // the take rule of the end of this function
        if (!a.rows) nv.linker_hash[b] = l;
        else if (!(a.flags[a.rows[b]] == 0 && a.s_flags[b] != 0)) nv.linker_hash[a.rows[b]] = l;
      }
    }
  }
  if constexpr ((CHECKS & CHECK_RINGS) != 0) {
    const RingArgs& rg = static_cast<const RingArgs&>(nv);   // the kernel's parameter is a RingArgs
    __syncthreads();                                  // the buffer is read above until here
    if (tid == 0) s_n = 0;
    __syncthreads();
    for (int r0 = 0; r0 < a.N; r0 += 256) {           // every checked atom again, with its linker flag in s_row
      const int r = r0 + tid;
      bool ok = r < a.N && a.node_mask[g0 + r] != 0;
      if (ok && a.drop_pocket) ok = a.context[(g0 + r) * a.C + a.C - 1] == 0.f;
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      if (lane == 0) s_warp[warp] = __popc(m);
      __syncthreads();
      int off = s_n + __popc(m & ((1u << lane) - 1u)), total = 0;
      for (int w = 0; w < 8; ++w) { off += w < warp ? s_warp[w] : 0; total += s_warp[w]; }
      if (ok) {
        s_at[off] = load_atom(a, g0, r);
        s_row[off] = rg.linker_mask[g0 + r] != 0.f;
      }
      __syncthreads();
      if (tid == 0) s_n += total;
      __syncthreads();
    }
    unsigned* s_bits = reinterpret_cast<unsigned*>(s_row + a.N);
    const unsigned long long mask = ring_mask(a, hk.edge_cap, s_n, s_at, s_lab, s_row, s_bits,
                                              reinterpret_cast<int*>(s_bits + RING_BITSETS * ((a.N + 31) >> 5)));
    if (tid == 0) {
      if ((mask & ~rg.allowed) == 0) verdict |= CHECK_RINGS;
      if (rg.ring_sizes) {                            // the take rule of the end of this function
        if (!a.rows) rg.ring_sizes[b] = mask;
        else if (!(a.flags[a.rows[b]] == 0 && a.s_flags[b] != 0)) rg.ring_sizes[a.rows[b]] = mask;
      }
    }
  }
  if (tid == 0) {
    if (!(CHECKS & CHECK_UNIQUE) || a.passed) a.passed[b] = verdict;   // dl_molecule_hash has no verdicts
    if (a.rows) a.take[b] = !(a.flags[a.rows[b]] == 0 && a.s_flags[b] != 0);
  }
}

// The instantiations without the clash and hash bits, with the clash bit, with the hash bit, with the linker hash bit, and
// with the ring bit.
template <int CHECKS>
__global__ void __launch_bounds__(256) k_molecule_check(CheckArgs a) {
  static_assert((CHECKS & (CHECK_CLASH | CHECK_UNIQUE | CHECK_NOVEL)) == 0,
                "the clash check takes ClashArgs, the hash HashArgs, the linker hash NovelArgs");
  molecule_check<CHECKS>(a, ClashArgs{}, HashArgs{}, NovelArgs{});
}

// (With __launch_bounds__(256) alone ptxas fits <6> into 32 registers and spills; a minimum of one CTA per SM lets it take
// the 38-39 it needs.)
template <int CHECKS>
__global__ void __launch_bounds__(256, 1) k_molecule_check(CheckArgs a, ClashArgs k) {
  static_assert((CHECKS & CHECK_CLASH) != 0 && (CHECKS & (CHECK_UNIQUE | CHECK_NOVEL)) == 0,
                "only the clash check takes ClashArgs alone");
  molecule_check<CHECKS>(a, k, HashArgs{}, NovelArgs{});
}

template <int CHECKS>
__global__ void __launch_bounds__(256, 1) k_molecule_check(CheckArgs a, ClashArgs k, HashArgs h) {
  static_assert((CHECKS & CHECK_UNIQUE) != 0 && (CHECKS & CHECK_NOVEL) == 0, "only the hash takes HashArgs alone");
  molecule_check<CHECKS>(a, k, h, NovelArgs{});
}

template <int CHECKS>
__global__ void __launch_bounds__(256, 1) k_molecule_check(CheckArgs a, ClashArgs k, HashArgs h, NovelArgs v) {
  static_assert((CHECKS & CHECK_NOVEL) != 0, "only the linker hash takes NovelArgs");
  molecule_check<CHECKS>(a, k, h, v);
}

template <int CHECKS>
__global__ void __launch_bounds__(256, 1) k_molecule_check(CheckArgs a, ClashArgs k, HashArgs h, RingArgs g) {
  static_assert((CHECKS & CHECK_RINGS) != 0, "only the ring check takes RingArgs");
  molecule_check<CHECKS>(a, k, h, g);
}

template <int CHECKS>
cudaError_t launch_molecule_check_as(const CheckArgs& a, const ClashArgs& k, const HashArgs& h, const NovelArgs& v,
                                     unsigned long long ring_allowed, unsigned long long* ring_sizes, int B,
                                     cudaStream_t st) {
  const size_t smem = (size_t)a.N * (sizeof(float4) + sizeof(int));
  if constexpr ((CHECKS & CHECK_RINGS) != 0) {
    // the hash's 24 bytes per row, the ring search's bitsets, then the bonds: HASH_EDGES_PER_ROW per row or what
    // HASH_SMEM_MAX leaves (2560 at N = 8192). The hash stages, if any, store their bonds in the same room.
    const size_t base = smem + (size_t)a.N * sizeof(int) + (size_t)RING_BITSETS * ((a.N + 31) / 32) * sizeof(unsigned);
    const size_t cap = std::min((size_t)a.N * HASH_EDGES_PER_ROW, (HASH_SMEM_MAX - base) / sizeof(unsigned));
    const size_t total = base + cap * sizeof(unsigned);
    HashArgs hh = h;
    hh.edge_cap = (int)cap;
    void (*kernel)(CheckArgs, ClashArgs, HashArgs, RingArgs) = k_molecule_check<CHECKS>;
    if (total > 48 * 1024) {
      const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HASH_SMEM_MAX);
      if (err != cudaSuccess) return err;
    }
    kernel<<<B, 256, total, st>>>(a, k, hh, RingArgs{v, ring_allowed, ring_sizes});
  } else if constexpr ((CHECKS & (CHECK_UNIQUE | CHECK_NOVEL)) != 0) {
    // 8 more bytes per row, then the bonds: HASH_EDGES_PER_ROW per row or what HASH_SMEM_MAX leaves (512 at N = 8192;
    // graph_hash rescans the atoms whose bonds do not fit)
    const size_t base = smem + (size_t)a.N * 2 * sizeof(int);
    const size_t cap = std::min((size_t)a.N * HASH_EDGES_PER_ROW, (HASH_SMEM_MAX - base) / sizeof(unsigned));
    const size_t total = base + cap * sizeof(unsigned);
    HashArgs hh = h;
    hh.edge_cap = (int)cap;
    if constexpr ((CHECKS & CHECK_NOVEL) != 0) {
      void (*kernel)(CheckArgs, ClashArgs, HashArgs, NovelArgs) = k_molecule_check<CHECKS>;
      if (total > 48 * 1024) {
        const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HASH_SMEM_MAX);
        if (err != cudaSuccess) return err;
      }
      kernel<<<B, 256, total, st>>>(a, k, hh, v);
    } else {
      void (*kernel)(CheckArgs, ClashArgs, HashArgs) = k_molecule_check<CHECKS>;
      if (total > 48 * 1024) {
        const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, HASH_SMEM_MAX);
        if (err != cudaSuccess) return err;
      }
      kernel<<<B, 256, total, st>>>(a, k, hh);
    }
  } else if constexpr ((CHECKS & CHECK_CLASH) != 0) {
    void (*kernel)(CheckArgs, ClashArgs) = k_molecule_check<CHECKS>;
    if (smem > 48 * 1024) {
      const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CONN_SMEM_MAX);
      if (err != cudaSuccess) return err;
    }
    kernel<<<B, 256, smem, st>>>(a, k);
  } else {
    void (*kernel)(CheckArgs) = k_molecule_check<CHECKS>;
    if (smem > 48 * 1024) {
      const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CONN_SMEM_MAX);
      if (err != cudaSuccess) return err;
    }
    kernel<<<B, 256, smem, st>>>(a);
  }
  return cudaGetLastError();
}

// launch_molecule_check_as<C> for the one C in {1, ..., sizeof...(C)} that equals checks.
template <int... C>
cudaError_t launch_molecule_check_of(int checks, const CheckArgs& a, const ClashArgs& k, const HashArgs& h,
                                     const NovelArgs& v, unsigned long long ring_allowed, unsigned long long* ring_sizes,
                                     int B, cudaStream_t st, std::integer_sequence<int, C...>) {
  cudaError_t err = cudaErrorInvalidValue;
  (void)((checks == C + 1 &&
          ((err = launch_molecule_check_as<C + 1>(a, k, h, v, ring_allowed, ring_sizes, B, st)), true)) || ...);
  return err;
}

// Launches k_molecule_check<checks> over B molecules; checks is a non-empty OR of CHECK_*, N <= CONN_MAX_N.
// The shared-memory limit is raised to its one maximum the first time a molecule needs more than the default, so
// concurrent callers never lower it under each other.
// CHECK_UNIQUE writes the hashes to h.hash; CHECK_NOVEL reads v; CHECK_RINGS reads v.linker_mask and ring_allowed and
// writes the masks to ring_sizes (or null).
inline cudaError_t launch_molecule_check(int checks, const CheckArgs& a, const ClashArgs& k, const HashArgs& h, int B,
                                         cudaStream_t st, const NovelArgs& v = NovelArgs{},
                                         unsigned long long ring_allowed = 0, unsigned long long* ring_sizes = nullptr) {
  return launch_molecule_check_of(checks, a, k, h, v, ring_allowed, ring_sizes, B, st,
                                  std::make_integer_sequence<int, 2 * CHECK_RINGS - 1>{});
}

// What CHECK_ANCHORS reads and writes besides CheckArgs, whose xh, N, row_stride, n_types, thr1, node_mask, context, C,
// drop_pocket and passed it reads, and in a recovery round rows, flags, s_flags and take.
struct AnchorArgs {
  const float* linker_mask;              // (B, N): the checked atoms with linker_mask != 0 are the linker atoms
  const int8_t* anchors;                 // (B, N): the anchor flags of molecule b at row b, or in a recovery round at the
                                         // caller's row rows[b] (the fragment rows keep their positions in the sub-batch)
  int32_t* attachments;                  // (B, N) or null: a_i on every fragment atom, 0 on every other row; at row b, or in
                                         // a recovery round at the caller's row rows[b], where the row is taken
  int or_into;                           // 1: ORs the bit into passed[b], which k_molecule_check wrote; 0: writes passed[b]
                                         // (and take[b] in a round), with no k_molecule_check launch before it
};
// Shared memory per row: the staged atom, its role (row, linker and anchor bits) and the linker atoms' list.
constexpr int ANCHOR_SMEM_PER_ROW = (int)(sizeof(float4) + 2 * sizeof(int));
constexpr int ANCHOR_LINKER = 1 << 30, ANCHOR_FLAG = 1 << 29, ANCHOR_ROW = (1 << 29) - 1;

// One CTA per molecule. The checked atoms are compacted, in row order, into shared memory as k_molecule_check compacts them
// (so the pair orientation and n of staged_bonded are the other bits'), with their role beside them; the linker atoms' staged
// indices are listed in the same pass. A warp per fragment atom i then counts, lanes over the linker atoms, the bonds a_i
// between i and the linker, and the counts are reduced by shuffles: no atomics, and neither a_i nor the verdict depends on
// the order the lanes or warps run in. (As for k_molecule_check, a minimum of one CTA per SM lets ptxas take the registers
// it needs without spilling.)
__global__ void __launch_bounds__(256, 1) k_anchor_check(CheckArgs a, AnchorArgs g) {
  extern __shared__ float4 s_at[];                    // [n]: x, y, z, type (int bits)
  int* s_role = reinterpret_cast<int*>(s_at + a.N);   // [n]: row | ANCHOR_LINKER | ANCHOR_FLAG
  int* s_lnk = s_role + a.N;                          // [n_linker]: the staged indices of the linker atoms, ascending
  __shared__ int s_warp[8], s_lwarp[8], s_n, s_nl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x;
  const size_t g0 = (size_t)b * a.N;
  const bool take = !a.rows || !(a.flags[a.rows[b]] == 0 && a.s_flags[b] != 0);   // k_molecule_check's take rule
  const size_t caller0 = (size_t)(a.rows ? a.rows[b] : b) * a.N;
  int32_t* att = g.attachments && take ? g.attachments + caller0 : nullptr;
  if (tid == 0) s_n = s_nl = 0;
  __syncthreads();
  for (int r0 = 0; r0 < a.N; r0 += 256) {
    const int r = r0 + tid;
    bool ok = r < a.N && a.node_mask[g0 + r] != 0;
    if (ok && a.drop_pocket) ok = a.context[(g0 + r) * a.C + a.C - 1] == 0.f;
    const bool linker = ok && g.linker_mask[g0 + r] != 0.f;
    const unsigned m = __ballot_sync(0xffffffffu, ok), ml = __ballot_sync(0xffffffffu, linker);
    if (lane == 0) { s_warp[warp] = __popc(m); s_lwarp[warp] = __popc(ml); }
    __syncthreads();
    const unsigned below = (1u << lane) - 1u;
    int off = s_n + __popc(m & below), loff = s_nl + __popc(ml & below), total = 0, ltotal = 0;
    for (int w = 0; w < 8; ++w) {
      off += w < warp ? s_warp[w] : 0; total += s_warp[w];
      loff += w < warp ? s_lwarp[w] : 0; ltotal += s_lwarp[w];
    }
    if (ok) {
      s_at[off] = load_atom(a, g0, r);
      s_role[off] = r | (linker ? ANCHOR_LINKER : 0) | (!linker && g.anchors[caller0 + r] != 0 ? ANCHOR_FLAG : 0);
      if (linker) s_lnk[loff] = off;
    }
    if (att && r < a.N && (!ok || linker)) att[r] = 0;   // the fragment atoms' rows are written below
    __syncthreads();
    if (tid == 0) { s_n += total; s_nl += ltotal; }
    __syncthreads();
  }
  const int n = s_n, n_linker = s_nl;
  int bad = 0, anchored = 0;
  for (int i = warp; i < n; i += 8) {                 // warp per fragment atom i, lanes over the linker atoms
    const int role = s_role[i];
    if (role & ANCHOR_LINKER) continue;
    anchored |= role & ANCHOR_FLAG;
    const float4 pi = s_at[i];
    int c = 0;
    for (int k = lane; k < n_linker; k += 32) {
      const int j = s_lnk[k];
      c += staged_bonded(a, i, pi, j, s_at[j], n);
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) {
      bad |= c != ((role & ANCHOR_FLAG) ? 1 : 0);
      if (att) att[role & ANCHOR_ROW] = c;
    }
  }
  const bool any_anchor = __syncthreads_or(anchored) != 0;
  const bool ok = !any_anchor || !__syncthreads_or(bad);   // a molecule with no anchor passes
  if (tid == 0) {
    if (g.or_into) {
      if (ok) a.passed[b] |= CHECK_ANCHORS;
    } else {
      a.passed[b] = ok ? CHECK_ANCHORS : 0;
      if (a.rows) a.take[b] = take;
    }
  }
}

// Launches k_anchor_check over B molecules, N <= CONN_MAX_N. The shared-memory limit is raised to its one maximum the first
// time a molecule needs more than the default, as launch_molecule_check raises it.
inline cudaError_t launch_anchor_check(const CheckArgs& a, const AnchorArgs& g, int B, cudaStream_t st) {
  const size_t smem = (size_t)a.N * ANCHOR_SMEM_PER_ROW;
  if (smem > 48 * 1024) {
    const cudaError_t err = cudaFuncSetAttribute(k_anchor_check, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 CONN_MAX_N * ANCHOR_SMEM_PER_ROW);
    if (err != cudaSuccess) return err;
  }
  k_anchor_check<<<B, 256, smem, st>>>(a, g);
  return cudaGetLastError();
}

// Clash guidance (dl_set_clash_guidance, dl_clash_guide; stated at dl_set_clash_guidance in the header): every linker atom
// i of a molecule moves by scale * sum_k max(0, r_ik - d_ik) (p_i - p_k) / d_ik over its pocket atoms k, r_ik the clash
// table's entry for the pair in Angstrom. The rows are those of CHECK_CLASH: linker atoms have node_mask, linker_mask and
// context column C - 1 == 0; pocket atoms node_mask and column C - 1 != 0.
struct GuideArgs {
  float* xh;                             // (B, N, row_stride) in/out: x at columns 0..2 (the linker rows' are rewritten),
                                         // the types' channels from column 3
  int N, row_stride, n_types, C;
  float scale;
  const float* clash;                    // (n_types, n_types) clash distances in pm, [min type][max type]
  const int8_t* node_mask;               // (B, N)
  const float* linker_mask;              // (B, N)
  const float* context;                  // (B, N, C)
  // in the reverse loop (step != null): loop row *step is guided iff T - steps <= *step < T, and the frame of its
  // dl_step_coef row (coef, 8 floats per row) receives the moved coordinates times norm0
  const int* step;
  int T, steps;
  const float* coef;
  float* chain;                          // (keep, B*N, row_stride)
  float norm0;
  const int8_t* fixed;                   // k_clash_guide<true>: (B, N) fixed-atom flags (dl_set_fixed_atoms), rows it never moves
};
// Shared memory per row: the staged pocket atom and the linker atoms' list.
constexpr int GUIDE_SMEM_PER_ROW = (int)(sizeof(float4) + sizeof(int));

// One CTA per molecule. The pocket atoms are compacted, in row order, into shared memory (coordinates and type) and the
// linker rows listed beside them in the same pass. A warp per linker atom then sums its push, lanes over the pocket atoms
// in a fixed assignment, and reduces the three sums with xor shuffles: no atomics, and the result depends neither on the
// order the warps run in nor on the molecule's batch-mates. The pair's distance is the clash check's (pair_dist_pm, in pm),
// so an atom moves iff the check counts a clash for it; (r - d) / d is taken in pm, where it is the same ratio. A pair at
// d = 0 or with a NaN distance contributes nothing, and an atom with no contributing pair is not written. FIXED: the linker
// rows flagged in a.fixed are not listed, so they neither move nor push (they are no pocket atoms either).
template <bool FIXED = false>
__global__ void __launch_bounds__(256) k_clash_guide(GuideArgs a) {
  extern __shared__ float4 s_pk[];                    // [n_pocket]: x, y, z, type (int bits)
  int* s_lnk = reinterpret_cast<int*>(s_pk + a.N);    // [n_linker]: the linker atoms' rows, ascending
  __shared__ int s_warp[8], s_lwarp[8], s_np, s_nl;
  int frame = -1;
  if (a.step != nullptr) {
    const int step = *a.step;                         // the same for every CTA: the whole grid returns or none does
    if (step >= a.T || step < a.T - a.steps) return;
    frame = __float_as_int(a.coef[(size_t)step * 8 + 4]);
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t g0 = (size_t)blockIdx.x * a.N;
  if (tid == 0) s_np = s_nl = 0;
  __syncthreads();
  for (int r0 = 0; r0 < a.N; r0 += 256) {
    const int r = r0 + tid;
    const bool live = r < a.N && a.node_mask[g0 + r] != 0;
    const bool pocket = live && a.context[(g0 + r) * a.C + a.C - 1] != 0.f;
    const bool linker = live && !pocket && a.linker_mask[g0 + r] != 0.f && (!FIXED || a.fixed[g0 + r] == 0);
    const unsigned mp = __ballot_sync(0xffffffffu, pocket), ml = __ballot_sync(0xffffffffu, linker);
    if (lane == 0) { s_warp[warp] = __popc(mp); s_lwarp[warp] = __popc(ml); }
    __syncthreads();
    const unsigned below = (1u << lane) - 1u;
    int poff = s_np + __popc(mp & below), loff = s_nl + __popc(ml & below), ptotal = 0, ltotal = 0;
    for (int w = 0; w < 8; ++w) {
      poff += w < warp ? s_warp[w] : 0; ptotal += s_warp[w];
      loff += w < warp ? s_lwarp[w] : 0; ltotal += s_lwarp[w];
    }
    if (pocket) {
      const float* row = a.xh + (g0 + r) * a.row_stride;
      s_pk[poff] = make_float4(row[0], row[1], row[2], __int_as_float(first_type(row, a.n_types)));
    }
    if (linker) s_lnk[loff] = r;
    __syncthreads();
    if (tid == 0) { s_np += ptotal; s_nl += ltotal; }
    __syncthreads();
  }
  const int n_pocket = s_np, n_linker = s_nl;
  for (int i = warp; i < n_linker; i += 8) {          // warp per linker atom, lanes over the pocket atoms
    const int r = s_lnk[i];
    float* row = a.xh + (g0 + r) * a.row_stride;
    const float3 pi = make_float3(row[0], row[1], row[2]);
    const int ti = first_type(row, a.n_types);
    float fx = 0.f, fy = 0.f, fz = 0.f;
    int hits = 0;
    for (int k = lane; k < n_pocket; k += 32) {
      const float4 pk = s_pk[k];
      const float3 pj = make_float3(pk.x, pk.y, pk.z);
      const int tj = __float_as_int(pk.w);
      const float d = pair_dist_pm(pi, pj);
      const float t = a.clash[min(ti, tj) * a.n_types + max(ti, tj)];
      if (t >= 0.f && d < t && d > 0.f) {             // false for a NaN distance
        const float w = (t - d) / d;
        fx = fmaf(w, pi.x - pj.x, fx); fy = fmaf(w, pi.y - pj.y, fy); fz = fmaf(w, pi.z - pj.z, fz);
        ++hits;
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      fx += __shfl_xor_sync(0xffffffffu, fx, o);
      fy += __shfl_xor_sync(0xffffffffu, fy, o);
      fz += __shfl_xor_sync(0xffffffffu, fz, o);
      hits += __shfl_xor_sync(0xffffffffu, hits, o);
    }
    if (hits == 0 || lane >= 3) continue;
    const float p = lane == 0 ? pi.x : lane == 1 ? pi.y : pi.z;
    const float f = lane == 0 ? fx : lane == 1 ? fy : fz;
    const float v = fmaf(a.scale, f, p);
    row[lane] = v;
    if (frame >= 0) a.chain[((size_t)frame * gridDim.x * a.N + g0 + r) * a.row_stride + lane] = v * a.norm0;
  }
}

// Launches k_clash_guide over B molecules, N <= CONN_MAX_N. Every caller first raises the kernel's shared-memory limit to
// its one maximum (clash_guide_opt_in), whatever N: the 48 KB default counts the static shared memory too. A reverse loop
// raises it before it captures its step (the attribute is not a stream operation).
inline cudaError_t clash_guide_opt_in() {
  const cudaError_t err = cudaFuncSetAttribute(k_clash_guide<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               CONN_MAX_N * GUIDE_SMEM_PER_ROW);
  if (err != cudaSuccess) return err;
  return cudaFuncSetAttribute(k_clash_guide<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, CONN_MAX_N * GUIDE_SMEM_PER_ROW);
}
// a.fixed != null launches the instantiation that leaves the flagged rows in place
inline cudaError_t launch_clash_guide(const GuideArgs& a, int B, cudaStream_t st) {
  const size_t smem = (size_t)a.N * GUIDE_SMEM_PER_ROW;
  if (a.fixed != nullptr) k_clash_guide<true><<<B, 256, smem, st>>>(a);
  else k_clash_guide<false><<<B, 256, smem, st>>>(a);
  return cudaGetLastError();
}

// dl_sample_chain_retry's vetting of a caller's hash set: bad[0] = 1 if some s[i] > s[i + 1] in unsigned order.
__global__ void __launch_bounds__(256) k_sorted_check(const unsigned long long* s, long long n, int32_t* bad) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i + 1 < n; i += (long long)gridDim.x * 256)
    if (s[i] > s[i + 1]) *bad = 1;
}

// The uniqueness verdict over a batch of B molecules whose graph hashes are hash[b] (stated at DL_CHECK_UNIQUE in the
// header). Candidates: every row (rows == null: the first loop), or the Bs rows rows[i] (ascending) of a recovery round,
// whose hash is then s_hash[i] where take[i] is set and hash[rows[i]] where it is not. Keepers: the rows that are not
// candidates and pass every bit of `require`. Eligible: a candidate with flags == 0 and every other bit of `require`.
struct UniqueArgs {
  int B, Bs, require;
  unsigned long long* hash;              // (B); a round writes s_hash[i] to hash[rows[i]] where take[i] is set
  const int32_t* flags;                  // (B)
  int32_t* passed;                       // (B): DL_CHECK_UNIQUE set or cleared on the candidates
  const int* rows;
  const int32_t* take;
  const unsigned long long* s_hash;      // (Bs)
};

// The hashes of a caller's seen set, which count as keepers: a kernel parameter of the verdict with a set only.
struct SeenArgs {
  const unsigned long long* seen;        // (n_seen) ascending, unsigned order
  long long n_seen;
};

// A thread per candidate: the bit iff its hash equals no keeper's and no eligible earlier candidate's (SEEN: and is not in
// the seen set). Each thread writes only its own row's bit and hash; the bits and hashes other threads read are not among
// them (a keeper is never written, and a candidate's other bits and its hash are read from where they do not change), so
// the verdict does not depend on the order the threads run in.
template <bool SEEN>
__device__ __forceinline__ void unique_verdict(const UniqueArgs& u, const SeenArgs& s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int nc = u.rows ? u.Bs : u.B;
  if (i >= nc) return;
  const int other = u.require & ~CHECK_UNIQUE;
  auto row = [&](int k) { return u.rows ? u.rows[k] : k; };
  auto hash_of = [&](int k) { return u.rows && u.take[k] ? u.s_hash[k] : u.hash[row(k)]; };
  const int b = row(i);
  const unsigned long long h = hash_of(i);
  bool dup = SEEN && sorted_contains(s.seen, s.n_seen, h);
  if (u.rows)
    for (int k = 0, p = 0; k < u.B && !dup; ++k) {   // keepers: the rows between the candidates
      if (p < u.Bs && u.rows[p] == k) { ++p; continue; }
      dup = u.flags[k] == 0 && (u.passed[k] & u.require) == u.require && u.hash[k] == h;
    }
  for (int k = 0; k < i && !dup; ++k) {
    const int bk = row(k);
    dup = u.flags[bk] == 0 && (u.passed[bk] & other) == other && hash_of(k) == h;
  }
  u.passed[b] = dup ? (u.passed[b] & ~CHECK_UNIQUE) : (u.passed[b] | CHECK_UNIQUE);
  if (u.rows && u.take[i]) u.hash[b] = u.s_hash[i];
}

__global__ void __launch_bounds__(256) k_unique_verdict(UniqueArgs u) { unique_verdict<false>(u, SeenArgs{}); }

__global__ void __launch_bounds__(256) k_unique_verdict(UniqueArgs u, SeenArgs s) { unique_verdict<true>(u, s); }

}  // namespace dl
