// The bond predicate and the bond order of molecule_builder.get_bond_order (src/molecule_builder.py:77-102), shared by
// dl_bond_orders (output_stage.cu) and the connectivity, valence and hash checks of the recovery rounds
// (kernels_retry.cuh), so all of them decide "bonded" and "the order of a pair" with the same arithmetic: the arithmetic of
// torch.cdist(pos, pos) on the CPU over the molecule's n checked atoms, which is what build_xae_molecule reads.
//   n <= 25  the direct form, 100 sqrt(fma(dz, dz, fma(dy, dy, dx * dx))), d = x_i - x_j;
//   n >  25  torch's _euclidean_dist: c = ((((-2 x_i0) x_j0 + (-2 x_i1) x_j1) + (-2 x_i2) x_j2) + |x_i|^2) + |x_j|^2, the
//            products after the first fused, |x|^2 = (x0^2 + x1^2) + x2^2 with every step rounded; then a NaN-keeping
//            clamp at 0, a correctly rounded sqrt and x 100.
// The matmul form is not symmetric: atom i is the later atom of the pair in the molecule's compacted atom order, as the
// reference reads dists[i, j] with i > j. The pocket-clash check is this project's own predicate and keeps the direct form
// at every n (clash_pair).
#pragma once

namespace dl {

// torch.cdist switches to its matmul formulation above this many rows.
constexpr int CDIST_MM_ROWS = 25;

// The distance of atoms at xi, xj in pm ("we change the metric") in the direct form: 100 |xi - xj| in fp32, the squares
// summed as fma(dz, dz, fma(dy, dy, dx * dx)).
__device__ __forceinline__ float pair_dist_pm(float3 xi, float3 xj) {
  const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
  return 100.0f * __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx))));
}

// (x0^2 + x1^2) + x2^2, every step rounded: x.pow(2).sum(-1) of torch.
__device__ __forceinline__ float sq_norm_rn(float3 x) {
  return __fadd_rn(__fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y)), __fmul_rn(x.z, x.z));
}

// The distance in pm of the pair (i, j) of a molecule of n checked atoms, xi the LATER atom (i > j), as torch.cdist
// measures it for n rows (the forms at the top of this file). fmaxf(NaN, 0) is 0, which would bond NaN atoms; the clamp
// below keeps NaN, as torch's clamp_min does.
__device__ __forceinline__ float bond_dist_pm(float3 xi, float3 xj, int n) {
  if (n <= CDIST_MM_ROWS) return pair_dist_pm(xi, xj);
  float c = __fmul_rn(-2.0f * xi.x, xj.x);
  c = __fmaf_rn(-2.0f * xi.y, xj.y, c);
  c = __fmaf_rn(-2.0f * xi.z, xj.z, c);
  c = __fadd_rn(__fadd_rn(c, sq_norm_rn(xi)), sq_norm_rn(xj));
  c = c < 0.0f ? 0.0f : c;
  return 100.0f * __fsqrt_rn(c);
}

// get_bond_order(...) > 0 for atoms at xi (the later atom), xj of types ti, tj in a molecule of n checked atoms: the
// pair's distance in pm (bond_dist_pm) is below the single-bond threshold thr1 of the type pair ordered by type index,
// [min type][max type] of the (T x T) table, and that threshold exists (>= 0). Returns the pair's table index min * T + max
// when the atoms bond, else -1; *dist_pm receives the distance in pm for the double / triple tests.
__device__ __forceinline__ int bond_pair(float3 xi, float3 xj, int ti, int tj, int T, const float* __restrict__ thr1,
                                         int n, float* dist_pm) {
  const float dist = bond_dist_pm(xi, xj, n);
  *dist_pm = dist;
  const int a = min(ti, tj), c = max(ti, tj);
  if (a < 0 || c >= T) return -1;
  const float t1 = thr1[a * T + c];
  return (t1 >= 0.f && dist < t1) ? a * T + c : -1;
}

// get_bond_order(...) itself: 0 when the atoms do not bond (bond_pair), else 1, 2 or 3 -- double when the distance is also
// below the pair's thr2 entry and that entry exists, triple when it is below thr3 as well. xi is the later atom.
__device__ __forceinline__ int bond_order_pair(float3 xi, float3 xj, int ti, int tj, int T, const float* __restrict__ thr1,
                                               const float* __restrict__ thr2, const float* __restrict__ thr3, int n) {
  float dist;
  const int k = bond_pair(xi, xj, ti, tj, T, thr1, n, &dist);
  if (k < 0) return 0;
  const float t2 = thr2[k];
  if (!(t2 >= 0.f && dist < t2)) return 1;
  const float t3 = thr3[k];
  return (t3 >= 0.f && dist < t3) ? 3 : 2;
}

// The pocket-clash predicate of DL_CHECK_CLASH (stated at dl_molecule_checks in the header): atoms at xi, xj of types ti,
// tj clash iff their distance in pm in the direct form (pair_dist_pm, at any atom count) is below clash[min type][max
// type] of the (T x T) table and that entry is >= 0 (a negative entry: the pair never clashes). A NaN distance compares
// false: no clash.
__device__ __forceinline__ bool clash_pair(float3 xi, float3 xj, int ti, int tj, int T, const float* __restrict__ clash) {
  const float dist = pair_dist_pm(xi, xj);
  const int a = min(ti, tj), c = max(ti, tj);
  if (a < 0 || c >= T) return false;
  const float t = clash[a * T + c];
  return t >= 0.f && dist < t;
}

}  // namespace dl
