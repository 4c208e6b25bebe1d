// Output stage of the samplers' callers (SURVEY.md section 8(f) rank 2): the step right after sample_chain.
//   dl_restore_frame : generate.py:163-171 -- x += mean(positions * com_mask) * node_mask, on the device, in place
//   dl_format_xyz    : visualizer.save_xyz_file (visualizer.py:14-31) for a whole batch in one call instead of a
//                      Python loop with one .item() per atom; produces the exact text ("%d\n\n", "%s %.9f %.9f %.9f\n")
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

#include "../../include/difflinker_b200.h"
#include "bonds.cuh"

namespace {

// One CTA per molecule; fixed-shape reduction (lane-strided partials, shuffle tree, 8 warp partials in order).
__global__ void __launch_bounds__(256) k_restore_frame(int N, int N_pos, int xd, float* __restrict__ xh,
                                                       const float* __restrict__ positions,
                                                       const float* __restrict__ com_mask,
                                                       const int8_t* __restrict__ node_mask) {
  __shared__ float red[4][8];
  __shared__ float mean[3];
  const int b = blockIdx.x, tid = threadIdx.x;
  const size_t g0 = (size_t)b * N;
  const size_t p0 = (size_t)b * N_pos;   // positions / com_mask keep the INPUT batch's padding (generate.py:165-171)
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int n = tid; n < N_pos; n += 256) {
    const float m = com_mask[p0 + n];
    s[0] += positions[(p0 + n) * 3 + 0] * m;
    s[1] += positions[(p0 + n) * 3 + 1] * m;
    s[2] += positions[(p0 + n) * 3 + 2] * m;
    s[3] += m;
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s[q] += __shfl_xor_sync(0xffffffffu, s[q], o);
    if ((tid & 31) == 0) red[q][tid >> 5] = s[q];
  }
  __syncthreads();
  if (tid < 3) {
    float a = 0.f, c = 0.f;
    for (int w = 0; w < 8; ++w) { a += red[tid][w]; c += red[3][w]; }
    mean[tid] = a / c;
  }
  __syncthreads();
  for (int idx = tid; idx < N * 3; idx += 256) {
    const int n = idx / 3, d = idx - n * 3;
    xh[(g0 + n) * xd + d] += mean[d] * (float)node_mask[g0 + n];
  }
}

// "%.9f" % float(v) as CPython prints it (correctly rounded; 'nan' / 'inf' / '-inf' without glibc's "-nan")
inline int fmt9(char* p, size_t cap, float v) {
  if (std::isnan(v)) return snprintf(p, cap, "nan");
  if (std::isinf(v)) return snprintf(p, cap, v > 0 ? "inf" : "-inf");
  return snprintf(p, cap, "%.9f", (double)v);
}

}  // namespace

extern "C" dl_status dl_restore_frame2(int32_t B, int32_t N, int32_t N_pos, int32_t row_stride, float* xh,
                                       const float* positions, const float* com_mask, const int8_t* node_mask,
                                       void* stream) {
  if (B <= 0 || N <= 0 || N_pos <= 0 || row_stride < 3 || !xh || !positions || !com_mask || !node_mask) return DL_ERR_INVALID;
  k_restore_frame<<<B, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(N, N_pos, row_stride, xh, positions, com_mask, node_mask);
  return cudaGetLastError() == cudaSuccess ? DL_OK : DL_ERR_CUDA;
}

extern "C" dl_status dl_restore_frame(int32_t B, int32_t N, int32_t row_stride, float* xh, const float* positions,
                                      const float* com_mask, const int8_t* node_mask, void* stream) {
  return dl_restore_frame2(B, N, N, row_stride, xh, positions, com_mask, node_mask, stream);
}

extern "C" int64_t dl_format_xyz(int32_t B, int32_t N, int32_t F, const float* positions, int32_t pos_row_stride,
                                 const float* one_hot, int32_t oh_row_stride, const int8_t* node_mask,
                                 const char* const* symbols, int32_t n_symbols, char* out, int64_t out_cap,
                                 int64_t* offsets) {
  if (B < 0 || N <= 0 || F <= 0 || !positions || !one_hot || !node_mask || !symbols || !offsets || pos_row_stride < 3 ||
      oh_row_stride < F || n_symbols < F)
    return DL_ERR_INVALID;
  // Sizing pass and writing pass share the code: text beyond out_cap is counted but not stored.
  int64_t pos = 0;
  char line[256];
  auto emit = [&](const char* s, int len) {
    if (out && pos + len <= out_cap) memcpy(out + pos, s, (size_t)len);
    pos += len;
  };
  for (int b = 0; b < B; ++b) {
    offsets[b] = pos;
    const int8_t* nm = node_mask + (size_t)b * N;
    int n_atoms = 0;
    for (int i = 0; i < N; ++i) n_atoms += nm[i];                               // mask.sum() (visualizer.py:19)
    emit(line, snprintf(line, sizeof(line), "%d\n\n", n_atoms));
    for (int i = 0; i < N; ++i) {
      if (!nm[i]) continue;                                                     // torch.where(mask) (visualizer.py:20)
      const float* oh = one_hot + ((size_t)b * N + i) * oh_row_stride;
      int best = 0;                                                             // torch.argmax: first maximum; NaN wins
      for (int k = 1; k < F; ++k) {
        const float v = oh[k], cur = oh[best];
        if ((v > cur || (std::isnan(v) && !std::isnan(cur)))) best = k;
      }
      const float* x = positions + ((size_t)b * N + i) * pos_row_stride;
      int len = snprintf(line, sizeof(line), "%s ", symbols[best]);
      for (int d = 0; d < 3; ++d) {
        len += fmt9(line + len, sizeof(line) - len, x[d]);
        line[len++] = d < 2 ? ' ' : '\n';
      }
      emit(line, len);
    }
  }
  offsets[B] = pos;
  return pos;
}

// ------------------------------------------------------------------------------------------------------------------
// Bond inference: molecule_builder.build_xae_molecule / get_bond_order (src/molecule_builder.py:44-102) for a whole
// padded batch. E[b][i][j] (i > j, both atoms valid) = bond order 0..3 decided by the pair's distance in pm against the
// tabulated single / double / triple bond lengths (+ margins) of the type pair ordered by type index
// (`sorted([atom_types[i], atom_types[j]])`); the upper triangle and masked rows are 0 ("the graph is DIRECTED").
// The distance is torch.cdist's over the molecule's n rows with node_mask != 0 (bonds.cuh): each block counts them.
// thr1/thr2/thr3: (T x T) fp32 thresholds indexed [min type][max type]; a negative entry = pair absent from that table.
// ------------------------------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256) k_bond_orders(int N, int T, const float* __restrict__ x, int x_stride,
                                                     const int32_t* __restrict__ types, const int8_t* __restrict__ node_mask,
                                                     const float* __restrict__ thr1, const float* __restrict__ thr2,
                                                     const float* __restrict__ thr3, int8_t* __restrict__ E) {
  const int b = blockIdx.y;
  const size_t g0 = (size_t)b * N;
  int n = 0;
  for (int r0 = 0; r0 < N; r0 += 256) n += __syncthreads_count(r0 + (int)threadIdx.x < N && node_mask[g0 + r0 + threadIdx.x]);
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < N * N; idx += gridDim.x * blockDim.x) {
    const int i = idx / N, j = idx - i * N;
    int8_t order = 0;
    if (j < i && node_mask[g0 + i] && node_mask[g0 + j]) {
      const float* xi = x + (g0 + i) * x_stride;
      const float* xj = x + (g0 + j) * x_stride;
      order = (int8_t)dl::bond_order_pair(make_float3(xi[0], xi[1], xi[2]), make_float3(xj[0], xj[1], xj[2]), types[g0 + i],
                                          types[g0 + j], T, thr1, thr2, thr3, n);
    }
    E[g0 * N + idx] = order;
  }
}
}  // namespace

extern "C" dl_status dl_bond_orders(int32_t B, int32_t N, int32_t n_types, const float* x, int32_t x_row_stride,
                                    const int32_t* atom_types, const int8_t* node_mask, const float* thr1,
                                    const float* thr2, const float* thr3, int8_t* E, void* stream) {
  if (B <= 0 || N <= 0 || n_types <= 0 || x_row_stride < 3 || !x || !atom_types || !node_mask || !thr1 || !thr2 || !thr3 || !E)
    return DL_ERR_INVALID;
  const dim3 grid((unsigned)std::min(64, (N * N + 255) / 256), (unsigned)B);
  k_bond_orders<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(N, n_types, x, x_row_stride, atom_types, node_mask,
                                                                           thr1, thr2, thr3, E);
  return cudaGetLastError() == cudaSuccess ? DL_OK : DL_ERR_CUDA;
}
