// The bond predicate and the bond order of molecule_builder.get_bond_order (src/molecule_builder.py:77-102), shared by
// dl_bond_orders (output_stage.cu) and the connectivity and valence checks of the recovery rounds (kernels_retry.cuh), so
// all of them decide "bonded" and "the order of a pair" with the same arithmetic. The pocket-clash check measures its
// pairs with that arithmetic too.
#pragma once

namespace dl {

// The distance of atoms at xi, xj in pm ("we change the metric"): 100 |xi - xj| in fp32.
__device__ __forceinline__ float pair_dist_pm(float3 xi, float3 xj) {
  const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
  return 100.0f * sqrtf(dx * dx + dy * dy + dz * dz);
}

// get_bond_order(...) > 0 for atoms at xi, xj of types ti, tj: the pair's distance in pm (pair_dist_pm) is
// below the single-bond threshold thr1 of the type pair ordered by type index, [min type][max type] of the (T x T) table,
// and that threshold exists (>= 0). Returns the pair's table index min * T + max when the atoms bond, else -1;
// *dist_pm receives the distance in pm for the double / triple tests.
__device__ __forceinline__ int bond_pair(float3 xi, float3 xj, int ti, int tj, int T, const float* __restrict__ thr1,
                                         float* dist_pm) {
  const float dist = pair_dist_pm(xi, xj);
  *dist_pm = dist;
  const int a = min(ti, tj), c = max(ti, tj);
  if (a < 0 || c >= T) return -1;
  const float t1 = thr1[a * T + c];
  return (t1 >= 0.f && dist < t1) ? a * T + c : -1;
}

// get_bond_order(...) itself: 0 when the atoms do not bond (bond_pair), else 1, 2 or 3 -- double when the distance is also
// below the pair's thr2 entry and that entry exists, triple when it is below thr3 as well.
__device__ __forceinline__ int bond_order_pair(float3 xi, float3 xj, int ti, int tj, int T, const float* __restrict__ thr1,
                                               const float* __restrict__ thr2, const float* __restrict__ thr3) {
  float dist;
  const int k = bond_pair(xi, xj, ti, tj, T, thr1, &dist);
  if (k < 0) return 0;
  const float t2 = thr2[k];
  if (!(t2 >= 0.f && dist < t2)) return 1;
  const float t3 = thr3[k];
  return (t3 >= 0.f && dist < t3) ? 3 : 2;
}

// The pocket-clash predicate of DL_CHECK_CLASH (stated at dl_molecule_checks in the header): atoms at xi, xj of types ti,
// tj clash iff their distance in pm (pair_dist_pm) is below clash[min type][max type] of the (T x T) table and that entry
// is >= 0 (a negative entry: the pair never clashes). A NaN distance compares false: no clash.
__device__ __forceinline__ bool clash_pair(float3 xi, float3 xj, int ti, int tj, int T, const float* __restrict__ clash) {
  const float dist = pair_dist_pm(xi, xj);
  const int a = min(ti, tj), c = max(ti, tj);
  if (a < 0 || c >= T) return false;
  const float t = clash[a * T + c];
  return t >= 0.f && dist < t;
}

}  // namespace dl
