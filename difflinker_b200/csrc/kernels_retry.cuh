// Per-molecule NaN recovery (dl_sample_chain_seeded_retry): the seed of a molecule's next attempt, and the row gather /
// scatter between the caller's full batch and the sub-batch of the molecules that are sampled again.
#pragma once
#include <stdint.h>

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

// One recovery round: the Bs failed molecules rows[i] (ascending batch rows) of the B-molecule batch. The src_* pointers
// are the caller's full-batch inputs, the dst_* ones the sub-batch workspace, row i holding molecule rows[i].
struct RowGatherArgs {
  const int* rows;
  int N, xd, C, attempt;
  const float *xh, *fragment_mask, *linker_mask, *context;
  const int8_t *node_mask, *edge_mask;   // edge_mask: FC graphs' (B,N,N) int8 blocks, or null (all ones / cut-off graphs)
  const unsigned long long* seeds;       // the caller's base seeds
  float *s_xh, *s_fragment_mask, *s_linker_mask, *s_context;
  int8_t *s_node_mask, *s_edge_mask;
  unsigned long long* s_seeds;           // retry_seed(seeds[rows[i]], attempt)
};

// One CTA per failed molecule: copies its rows of every input, and derives its seed for this attempt.
__global__ void __launch_bounds__(256) k_gather_rows(RowGatherArgs a) {
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
  if (threadIdx.x == 0) a.s_seeds[i] = retry_seed(a.seeds[b], a.attempt);
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
};

// grid (Bs, keep_frames): CTA (i, f) writes frame f of sub-batch row i over row rows[i] of the caller's chain; the f = 0
// CTAs also write the molecule's flags, the seed that produced the row and the attempt.
__global__ void __launch_bounds__(256) k_scatter_rows(RowScatterArgs a) {
  const int i = blockIdx.x, f = blockIdx.y;
  const size_t b = a.rows[i], row = (size_t)a.N * a.xd;
  const float* src = a.s_chain + ((size_t)f * a.Bs + i) * row;
  float* dst = a.chain + ((size_t)f * a.B + b) * row;
  for (size_t k = threadIdx.x; k < row; k += blockDim.x) dst[k] = src[k];
  if (f == 0 && threadIdx.x == 0) {
    a.flags[b] = a.s_flags[i];
    a.seeds_used[b] = a.s_seeds[i];
    a.attempts[b] = a.attempt;
  }
}

}  // namespace dl
