"""The fp32 arithmetic the bond predicate measures a pair in, restated in numpy with an exact fused multiply-add.

The reference decides bonds on the CPU (molecule_builder.build_molecules calls .cpu()) from torch.cdist(pos, pos) over the
molecule's n atoms, read as dists[i, j] with i > j, and torch.cdist changes formulation with n:

  n <= 25  the direct form, sqrt(fma(dz, dz, fma(dy, dy, dx * dx))) with d = x_i - x_j;
  n >  25  _euclidean_dist: [-2 x_i, |x_i|^2, 1] . [x_j, 1, |x_j|^2] through the BLAS, clamped at 0 and square-rooted,
           where |x|^2 = (x0^2 + x1^2) + x2^2 (x.pow(2).sum(-1)). Stated order: acc = (-2 x_i0) x_j0, then
           fma(-2 x_i1, x_j1, acc), fma(-2 x_i2, x_j2, acc), + |x_i|^2, + |x_j|^2, then a correctly rounded sqrt.
           With torch 2.11 and MKL 2024.2 (AVX-512) the sgemm entries equal this order bitwise; the square root does
           not always: torch's CPU sqrt goes through MKL's vector math (vsSqrt), which rounds a fraction of a percent of
           its results one ulp away from the correctly rounded root. That residual is the ambiguity the tests measure.

The matmul form is not symmetric: the later atom of the pair (i > j) is the row. Both forms end in 100 * (the fp32 distance)
("we change the metric"). fma32 rounds a * b + c once: a * b is exact in float64, TwoSum gives the float64 sum and its
exact error, and rounding that sum to odd before the cast to fp32 makes the double rounding exact (53 >= 2 * 24 + 2)."""
import numpy as np

CDIST_MM_ROWS = 25          # torch.cdist uses _euclidean_dist when either operand has more rows than this


def fma32(a, b, c):
    """fp32 a * b + c rounded once to nearest even, elementwise (numpy broadcasting)."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b                                        # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                    # TwoSum: s + e == p + c exactly
    bits = np.asarray(s).view(np.int64)
    odd = np.isfinite(s) & (e != 0) & ((bits & 1) == 0)
    s = np.where(odd, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return np.asarray(s).astype(np.float32)


def direct_dist_pm(xi, xj):
    """100 |xi - xj| in pm, the direct form: d = xi - xj, sqrt(fma(dz, dz, fma(dy, dy, dx * dx))) (elementwise over the
    leading axes; the last axis holds x, y, z). The clash check measures every pair this way."""
    d = np.asarray(xi, np.float32) - np.asarray(xj, np.float32)
    s = d[..., 0] * d[..., 0]
    s = fma32(d[..., 1], d[..., 1], s)
    s = fma32(d[..., 2], d[..., 2], s)
    with np.errstate(invalid='ignore'):
        return np.float32(100) * np.sqrt(s)


def sq_norm(x):
    """(x0^2 + x1^2) + x2^2, each step rounded: x.pow(2).sum(-1) of torch, radial_rn on the device."""
    x = np.asarray(x, np.float32)
    return (x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2]


def matmul_entry(xi, xj):
    """The _euclidean_dist entry c of row xi (the later atom) and column xj in the stated order, before the clamp."""
    xi, xj = np.asarray(xi, np.float32), np.asarray(xj, np.float32)
    m2 = np.float32(-2)
    acc = (m2 * xi[..., 0]) * xj[..., 0]
    acc = fma32(m2 * xi[..., 1], xj[..., 1], acc)
    acc = fma32(m2 * xi[..., 2], xj[..., 2], acc)
    return (acc + sq_norm(xi)) + sq_norm(xj)


def matmul_dist_pm(xi, xj):
    """100 * sqrt(clamp_min(c, 0)) in pm, c = matmul_entry(xi, xj); the clamp keeps NaN, as torch's does."""
    acc = matmul_entry(xi, xj)
    with np.errstate(invalid='ignore'):
        acc = np.where(acc < 0, np.float32(0), acc)
        return np.float32(100) * np.sqrt(acc)


def pair_dist_pm(x, n=None):
    """(m, m) fp32 distances in pm of the atoms x (m, 3), in their order, as the bond predicate measures them in a molecule
    of n checked atoms (default m): entry [i, j] and [j, i] both hold the pair measured with the later atom max(i, j) as the
    row, in the direct form for n <= 25 and the matmul form above. The diagonal is the form's own value for (i, i)."""
    x = np.asarray(x, np.float32).reshape(-1, 3)
    n = x.shape[0] if n is None else n
    if n <= CDIST_MM_ROWS:
        return direct_dist_pm(x[:, None, :], x[None, :, :])
    d = matmul_dist_pm(x[:, None, :], x[None, :, :])               # row i, column j: correct for i > j
    lower = np.tril(np.ones(d.shape, dtype=bool), -1)
    return np.where(lower, d, d.T)


def torch_dist_pm(x):
    """(m, m) 100 * torch.cdist(x, x) in fp32 on the CPU, symmetrised from the lower triangle (i > j, the reference's
    reading)."""
    import torch
    x = np.asarray(x, np.float32).reshape(-1, 3)
    t = torch.from_numpy(x.copy())[None]
    d = (torch.cdist(t, t, p=2)[0] * 100).numpy()
    lower = np.tril(np.ones(d.shape, dtype=bool), -1)
    return np.where(lower, d, d.T)


def threshold_lookup(types, thr):
    """The (m, m) thresholds of each table in thr = (thr1, thr2, thr3), read [min type][max type]."""
    types = np.asarray(types)
    lo, hi = np.minimum(types[:, None], types[None, :]), np.maximum(types[:, None], types[None, :])
    return [np.asarray(t, np.float32)[lo, hi] for t in thr]


def orders_of(d, types, thr):
    """(m, m) int64 symmetric bond orders of get_bond_order for the pair distances d in pm, zero diagonal."""
    t1, t2, t3 = threshold_lookup(types, thr)
    with np.errstate(invalid='ignore'):
        b1 = (t1 >= 0) & (d < t1)
        b2 = b1 & (t2 >= 0) & (d < t2)
        b3 = b2 & (t3 >= 0) & (d < t3)
    o = b1.astype(np.int64) + b2 + b3
    np.fill_diagonal(o, 0)
    return o


def bond_orders(x, types, thr, n=None):
    """(m, m) symmetric bond orders of the atoms x with types, decided on pair_dist_pm(x, n)."""
    return orders_of(pair_dist_pm(x, n), types, thr)


# ---- designed molecules: pairs whose bond decision differs between the two forms -------------------------------------

def _unit(rng, m):
    u = rng.standard_normal((m, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


def straddling_pair(rng, t, offset, direct_below, tries=64):
    """Atoms (xj, xi) in fp32, xi the later one, whose distance in pm falls below threshold t in the direct form and at or
    above it in the matmul form (direct_below), or the other way round; found by exact search over fp32 candidates within
    a few ulps of t around a point 5 A from `offset` (A, on every axis). Raises when none is found."""
    for _ in range(tries):
        m = 4096
        xj = (np.float32(offset) + rng.uniform(-5, 5, (m, 3))).astype(np.float32)
        d = t / 100.0 * (1 + rng.integers(-12, 13, (m, 1)) * 2.0 ** -23)
        xi = (xj + _unit(rng, m) * d).astype(np.float32)
        dd, dm = direct_dist_pm(xi, xj), matmul_dist_pm(xi, xj)
        ok = (dd < t) & (dm >= t) if direct_below else (dm < t) & (dd >= t)
        k = np.flatnonzero(ok)
        if k.size:
            return xj[k[0]], xi[k[0]]
    raise RuntimeError(f"no pair straddles {t} pm at offset {offset}")


def chain_spacing(tc, ty, thr):
    """A distance in A at which an atom of type ty bonds singly and firmly to its carbon chain neighbour (type tc): halfway
    between the pair's double and single thresholds, or 10 pm inside the single one."""
    a, c = min(tc, ty), max(tc, ty)
    t1, t2 = float(thr[0][a][c]), float(thr[1][a][c])
    return ((t1 + t2) / 2 if t2 >= 0 else t1 - 10) / 100.0


def chain_around(xj, xi, tj, ti, n_before, n_after, thr):
    """A straight chain of carbon atoms through the pair: n_before atoms leading up to xj (earlier in the molecule's order),
    then xj, xi, and n_after atoms beyond xi, along the pair's direction, so that the pair is the chain's only link between
    its halves. Returns (x (n, 3) fp32, types (n,), j, i)."""
    u = (xi.astype(np.float64) - xj) / np.linalg.norm(xi.astype(np.float64) - xj)
    before = [xj - u * (chain_spacing(0, tj, thr) + 1.45 * k) for k in range(n_before)][::-1]
    after = [xi + u * (chain_spacing(0, ti, thr) + 1.45 * k) for k in range(n_after)]
    x = np.array(before + [xj, xi] + after, np.float32)
    types = np.zeros(len(x), np.int64)
    types[n_before], types[n_before + 1] = tj, ti
    return x, types, n_before, n_before + 1


def threshold_cases(thr):
    """(table k, min type a, max type c, threshold in pm) for every threshold of the (T, T) tables thr = (thr1, thr2, thr3)."""
    T = np.asarray(thr[0]).shape[0]
    return [(k, a, c, float(thr[k][a][c])) for k in range(3) for a in range(T) for c in range(a, T) if thr[k][a][c] >= 0]


# ---- the designed batches (tests/test_bond_rounding.py, tests/golden/bonds_thresholds.npz) -----------------------------
# thr = (thr1, thr2, thr3) as numpy (T, T) tables. Every generator is seeded, so the tests and the fixture writer build the
# same molecules.

DESIGN_OFFSETS = (0.0, 20.0, 40.0, 80.0)


def designed(thr, seed, n_lo=26, n_hi=60, offsets=DESIGN_OFFSETS):
    """One molecule per (threshold, direction, offset): (x, types, j, i, case), the pair (j, i) straddling the threshold
    between the two forms and linking the two halves of a carbon chain of n in [n_lo, n_hi] atoms."""
    rng = np.random.default_rng(seed)
    out = []
    for k, a, c, t in threshold_cases(thr):
        for below in (True, False):
            for off in offsets:
                xj, xi = straddling_pair(rng, t, off, below)
                n = int(rng.integers(n_lo, n_hi + 1))
                nb = int(rng.integers(1, n - 2))
                tj, ti = (a, c) if rng.random() < 0.5 else (c, a)
                x, ty, j, i = chain_around(xj, xi, tj, ti, nb, n - 2 - nb, thr)
                out.append((x, ty, j, i, (k + 1, a, c, t, 'direct<' if below else 'matmul<', off)))
    return out


def twins(thr, seed=3):
    """Molecules of 25 and 26 atoms around the same straddling pair (the 26th atom extends the chain), one per single
    threshold of carbon and per direction: (x25, x26, types25, types26, j, i)."""
    rng = np.random.default_rng(seed)
    out = []
    for k, a, c, t in threshold_cases(thr):
        if k != 0 or a != 0:
            continue
        for below in (True, False):
            xj, xi = straddling_pair(rng, t, 20.0, below)
            x, ty, j, i = chain_around(xj, xi, a, c, 12, 12, thr)
            out.append((x[:25], x, ty[:25], ty, j, i))
    return out


def pocket_designs(thr, seed=9):
    """Ligands of 20 atoms followed by 10 pocket rows 30 A away, one per single threshold of carbon and per direction:
    (x (30, 3), types (30,), j, i). Without the pocket the pair is measured in the direct form, with it in the matmul form;
    the pocket bonds to nothing."""
    rng = np.random.default_rng(seed)
    out = []
    for k, a, c, t in threshold_cases(thr):
        if k != 0 or a != 0:
            continue
        for below in (True, False):
            xj, xi = straddling_pair(rng, t, 40.0, below)
            x, ty, j, i = chain_around(xj, xi, a, c, 9, 9, thr)
            pocket = (xj + 30 + 4 * np.arange(10)[:, None] * np.ones(3)).astype(np.float32)
            out.append((np.concatenate([x, pocket]), np.concatenate([ty, np.zeros(10, np.int64)]), j, i))
    return out


def linker_designs(thr, seed=13):
    """Molecules of 30 atoms whose linker is the straddling pair and two atoms either side, for the carbon thresholds of
    double and triple bonds and the C-C, C-O, C-N single ones: (x, types, linker mask (30,)). The linker hash measures the
    pair over 6 atoms (direct form), the molecule's hash over 30 (matmul form)."""
    rng = np.random.default_rng(seed)
    out = []
    for k, a, c, t in threshold_cases(thr):
        if a != 0 or k == 0 and c not in (0, 1, 2):
            continue
        for below in (True, False):
            xj, xi = straddling_pair(rng, t, 20.0, below)
            x, ty, j, i = chain_around(xj, xi, a, c, 14, 14, thr)
            lm = np.zeros(len(x), np.float32)
            lm[j - 2:i + 3] = 1
            out.append((x, ty, lm))
    return out


def golden_molecules(thr, seed):
    """The molecules of tests/golden/bonds_thresholds.npz for one table, as (group, x, types): designed pairs in molecules
    of 26-28 atoms, the 25/26 twins, the pocket designs with and without their pocket, and the linker designs whole and
    their linker alone."""
    out = [("designed", x, ty) for x, ty, _, _, _ in designed(thr, seed, 26, 28)]
    for x25, x26, t25, t26, _, _ in twins(thr):
        out += [("twin25", x25, t25), ("twin26", x26, t26)]
    for x, ty, _, _ in pocket_designs(thr):
        out += [("pocket_all", x, ty), ("pocket_dropped", x[:20], ty[:20])]
    for x, ty, lm in linker_designs(thr):
        rows = np.flatnonzero(lm)
        out += [("linker_whole", x, ty), ("linker_alone", x[rows], ty[rows])]
    return out
