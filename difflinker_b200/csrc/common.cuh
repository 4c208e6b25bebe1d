// Shared device helpers and parameter blocks for the DiffLinker hot-path kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dl {

constexpr int H = 128;         // hidden_nf (configs/*.yml `nf: 128`), compile-time specialisation
constexpr int MAX_DIN = 32;    // F + C + 1 upper bound
constexpr int MAX_XHD = 16;    // 3 + F upper bound (threads per node in k_finish)

// EGNN options of the edge kernels (template bits, dl_egnn_options): each set of options is its own instantiation, so the
// default model's kernels carry no branch for them.
constexpr int OPT_TANH = 1;    // coordinate update trans = coord_diff * tanh(phi) * coords_range (egnn.py:104-105)
constexpr int OPT_MEAN = 2;    // aggregation_method='mean': divide by the row's edge count in the reference's edge list
                               // (egnn.py:315-319): N for FC graphs, the cut-off degree (0 -> 1) otherwise
constexpr int OPT_SIN = 4;     // sin_embedding: the two distance columns of every edge MLP's first layer become the 24
                               // features [sin, cos](sqrt(r + 1e-8) f_k) of both radials (SinusoidsEmbeddingNew, egnn.py:281-292)
constexpr int N_SIN_FREQ = 6;  // f_k = 2 pi 4^k / 15 (max_res 15, min_res 15/2000, div_factor 4)
constexpr int N_SIN_FEAT = 4 * N_SIN_FREQ;
// The fp32 values torch computes for 2 * math.pi * 4 ** torch.arange(6) / 15: exact power-of-4 multiples of f_0.
__device__ __forceinline__ float sin_freq(int k) { return __int_as_float(__float_as_int(0x1.aceeap-2f) + (k << 24)); }
// sqrt(r + 1e-8) * f_k in the reference's rounding order (no contraction); r itself must be (dx^2 + dy^2) + dz^2, each rounded
__device__ __forceinline__ float sin_arg(float r, int k) { return __fmul_rn(__fsqrt_rn(__fadd_rn(r, 1e-8f)), sin_freq(k)); }
__device__ __forceinline__ float radial_rn(float dx, float dy, float dz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// ---- programmatic dependent launch (PDL) ------------------------------------------------------------------------------
// The kernels of one forward form a strict chain on one stream. Launched with the programmatic-stream-serialization
// attribute (launch_chain below), a kernel's CTAs may become resident while the previous kernel is still draining: they run
// their prologue (barrier init, weight staging -- nothing the chain writes) and then block in chain_wait()
// until the previous grid has COMPLETED and its memory operations are visible. Every kernel of the chain calls chain_wait()
// before it touches anything another kernel of the chain produces or still reads, and only then chain_release()
// (griddepcontrol.launch_dependents), so at most two consecutive kernels overlap and completion is transitive along the
// chain. Without the launch attribute both instructions are no-ops.
__device__ __forceinline__ void chain_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void chain_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool& chain_overlap_enabled() { static bool on = true; return on; }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = chain_overlap_enabled() ? 1 : 0;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(static_cast<Args&&>(args))...);
}

// silu(x) = x * sigmoid(x) (nn.SiLU, reference src/lightning.py:23-27) = x / (1 + 2^(-x log2 e)).
// Raw ex2.approx / rcp.approx (2 MUFU + 3 FP32 ops; ~2 ulp each, far inside the 1e-4 end-to-end tolerance,
// DESIGN.md "numerics"); the libdevice wrappers (__expf, __fdividef) add range-fixup instructions that this
// path does not need: x -> -inf gives 2^(+inf) = inf, rcp(inf) = 0, x*0 = -0; x -> +inf gives x * 1.
__device__ __forceinline__ float silu_f(float x) {
  float t, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + t));
  return x * r;
}

// u / (1 + 2^u) for u = -log2(e)*x: equals -log2(e) * silu(x); callers fold the -ln(2) into a downstream constant.
__device__ __forceinline__ float usig_f(float u) {
  float t, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(u));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + t));
  return u * r;
}

// ---- fp32x2 arithmetic on register pairs: sm_90 has no packed fp32 instructions, so each is two round-to-nearest ops ------
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// Two sigmoids for three MUFU ops: 1/a and 1/b from ONE reciprocal of the product, (1/(ab))*b and (1/(ab))*a.
// The exponent is clamped at 63 so the product stays finite (a, b <= 1 + 2^63); that only alters silu for
// x < -43.7, where |silu(x)| < 5e-18.
__device__ __forceinline__ float2 sigmoid_pair_log2(float2 u) {
  const float2 den = fadd2(make_float2(ex2_approx(fminf(u.x, 63.0f)), ex2_approx(fminf(u.y, 63.0f))), make_float2(1.0f, 1.0f));
  const float r = rcp_approx(den.x * den.y);
  return fmul2(make_float2(r, r), make_float2(den.y, den.x));
}
// Four sigmoids for FIVE MUFU ops (4 ex2 + 1 rcp): with a,b,c,d the four denominators 1 + 2^u,
//   m = (a,b)*(c,d) = (ac, bd),  r = 1/(ac*bd),  (r*bd, r*ac) = (1/(ac), 1/(bd)),  times (c,d) -> (1/a, 1/b), times (a,b) -> (1/c, 1/d).
// The products work on register pairs that already exist (no shuffling of halves). The exponent is
// clamped at 31 so the product of four denominators stays below 2^125; that only alters u*sigmoid for u > 31
// (pre-activation < -21.5), where it changes the result by less than |u| * 4.7e-10 -- below fp32 resolution of the O(1)
// activations it is added to.
__device__ __forceinline__ void usig4(float2 u01, float2 u23, float2& s01, float2& s23) {
  const float2 one = make_float2(1.0f, 1.0f);
  const float2 ab = fadd2(make_float2(ex2_approx(fminf(u01.x, 31.0f)), ex2_approx(fminf(u01.y, 31.0f))), one);
  const float2 cd = fadd2(make_float2(ex2_approx(fminf(u23.x, 31.0f)), ex2_approx(fminf(u23.y, 31.0f))), one);
  const float2 m = fmul2(ab, cd);
  const float r = rcp_approx(m.x * m.y);
  const float2 rm = fmul2(make_float2(r, r), make_float2(m.y, m.x));
  s01 = fmul2(u01, fmul2(rm, cd));
  s23 = fmul2(u23, fmul2(rm, ab));
}
// (u0, u1) -> (u0/(1+2^u0), u1/(1+2^u1)): two sigmoids in the log2 domain
__device__ __forceinline__ float2 usig2(float2 u) { return fmul2(u, sigmoid_pair_log2(u)); }
// (x0, x1) -> (silu(x0), silu(x1))
__device__ __forceinline__ float2 silu2(float2 x) {
  return fmul2(x, sigmoid_pair_log2(fmul2(x, make_float2(-1.4426950408889634f, -1.4426950408889634f))));
}

// Packed weights of an edge MLP: a GCL's edge_mlp (src/egnn.py:19-30) or an EquivariantUpdate's coord_mlp (src/egnn.py:90-97),
// whose first Linear reads [h_i, h_j, d, d0] (SizeGNN: [h_i, h_j, d], w0 = 0). *_t = k-major ("transposed") [K][128].
struct EdgeMlpW {
  const float* W1a_t;  // [128][128]  .0.weight[:, 0:H]^T     (h_row part)
  const float* W1b_t;  // [128][128]  .0.weight[:, H:2H]^T    (h_col part)
  const float* b1;     // [128]
  const float* wd;     // [128]       .0.weight[:, 2H]        (block distance column)
  const float* w0;     // [128]       .0.weight[:, 2H+1]      (input distance column)
  const float* W2_t;   // [128][128]  .2.weight^T
  const float* b2;     // [128]
  const void* W2_tc;   // fp16 hi/lo wgmma-canonical tiles of .2.weight (tensor-core path)
  float w2_descale;    // 1 / (power-of-two scale applied to W2_tc)
  float wdmax, w0max;  // max|wd|, max|w0|: per-edge bound on the first-layer activations
  const void* W1_tc;   // .0.weight[:, 0:2H] as two packed 128x128 fp16 hi/lo blocks (node kernel projections)
  float w1_descale;
  // tensor-core path, log2-domain first layer (kernels_tc.cuh pack_w2): b1, wd, w0 times -log2(e); W1_tc is packed from the
  // scaled matrix, W2_tc carries the compensating -ln2.
  const float* b1_u;
  const float* wd_u;
  const float* w0_u;
  // sin_embedding: .0.weight[:, 2H:2H+24]^T ([24][128]: features [sin d f_k, cos d f_k, sin d0 f_k, cos d0 f_k]) and its
  // log2-domain copy; wdmax then holds sum_k max_c |w_k[c]| (|sin|, |cos| <= 1) and w0max 0
  const float* we;
  const float* we_u;
};

// Packed weights of one GCL: its edge MLP plus node_mlp.
struct GclW : EdgeMlpW {
  const float* W3_t;   // [256][128]  node_mlp.0.weight^T  (rows 0..127: h part, 128..255: agg part)
  const float* b3;     // [128]
  const float* W4_t;   // [128][128]  node_mlp.2.weight^T
  const float* b4;     // [128]
  const void* W3_tc;   // node_mlp.0.weight as two packed blocks
  const void* W4_tc;   // node_mlp.2.weight as one packed block
  float w3_descale, w4_descale;
};

// Packed weights of one EquivariantUpdate: its coord MLP plus the output row.
struct EqW : EdgeMlpW {
  const float* w5;     // [128] coord_mlp.4.weight (no bias)
};

// First-layer projection of an edge MLP applied per node: A = h W1a^T + b1, B = h W1b^T.
struct ProjW {
  const float* W1a_t;
  const float* W1b_t;
  const float* b1;
};

// Per-(B,N) work plan, built once per mask set by k_plan_* (masks are constant over the T steps).
struct Plan {
  const int* rowidx;   // [B][N] live rows (any non-zero edge weight), ascending
  const int* colidx;   // [B][N] live columns
  const int* xrowidx;  // [B][N] live rows that also have linker_mask != 0 (coordinate update rows)
  const int* nr;       // [B]
  const int* nc;       // [B]
  const int* nxr;      // [B]
  const int4* items;   // GCL work items (b, first row slot, row count, live column count nc)
  const int* n_items;  // [1]
  const int* xmols;    // molecules with nxr > 0 (coordinate-update work items of the SIMT kernel)
  const int* n_xmols;  // [1]
  const int4* xitems;  // coordinate-update work items of the tensor-core kernel: (b, first xrow slot, row count, nc)
  const int* n_xitems; // [1]
};

struct Geom {
  int B, N;
  int F;       // in_node_nf
  int C;       // context_node_nf
  int D;       // F + C + condition_time
  int graph_type;
  float norm_constant;
  float normalization_factor;
};

}  // namespace dl
