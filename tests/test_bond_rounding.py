"""The bond predicate against torch.cdist's own rounding, at the atom counts where torch changes formulation.

The reference decides bonds on the CPU from torch.cdist over a molecule's n atoms: the direct form for n <= 25 and the
matmul form (_euclidean_dist) above, read with the later atom of a pair as the row. oracle/bond_rounding.py restates both
with an exact fused multiply-add; the kernels (bonds.cuh) follow the same arithmetic, so the GPU tests compare them with
that emulation on every pair and with the live torch.cdist everywhere but the ambiguous pairs -- those where the
emulation and torch decide differently, which torch's one-ulp square root on the CPU leaves. Ambiguous pairs are counted,
reported and bounded.

The designed batches put one pair of each molecule where the two forms decide differently, for every single, double and
triple threshold of the ZINC and GEOM tables, in both directions, at frame offsets of 0, 20, 40 and 80 A; the pair is the
only link between two carbon chains, so it decides connectivity, its atoms' valences and the graph hash."""
import numpy as np
import pytest
import torch

from difflinker_b200 import molecule_builder as mb
from oracle import bond_rounding as br
import graph_hash_oracle as gho

OFFSETS = br.DESIGN_OFFSETS


def tables(is_geom):
    return [t.numpy() for t in mb.threshold_tables(is_geom)]


def n_types(is_geom):
    return 9 if is_geom else 8


def random_chain(rng, n, offset, T):
    """A chain-like molecule of n atoms (bonded steps of 1.05-1.65 A) around `offset` A, mostly carbon."""
    step = rng.standard_normal((n, 3))
    step *= (1.05 + 0.6 * rng.random((n, 1))) / np.linalg.norm(step, axis=1, keepdims=True)
    x = np.cumsum(step, 0)
    x = (x - x.mean(0) + offset).astype(np.float32)
    types = rng.integers(0, T, n)
    types[rng.random(n) < 0.5] = 0
    return x, types


def designed(is_geom, seed=7, n_lo=26, n_hi=60):
    """br.designed for one table: (x, types, j, i, case) per threshold, direction and offset."""
    return br.designed(tables(is_geom), seed + int(is_geom), n_lo, n_hi, OFFSETS)


def pack(mols, T, N=None):
    """(xh (B, N, 3 + T) with one-hot types, node_mask (B, N) int8) of [(x, types), ...], padded at the end."""
    N = N or max(len(m[0]) for m in mols)
    xh = torch.zeros(len(mols), N, 3 + T)
    nm = torch.zeros(len(mols), N, dtype=torch.int8)
    for b, (x, ty) in enumerate(mols):
        n = len(x)
        xh[b, :n, :3] = torch.from_numpy(np.asarray(x, np.float32))
        xh[b, :n, 3:] = torch.nn.functional.one_hot(torch.as_tensor(ty), T).float()
        nm[b, :n] = 1
    return xh, nm


def decisions(x, types, thr, n=None):
    """(emulated orders, torch.cdist orders, ambiguous mask) of one molecule's atoms, all (m, m) symmetric."""
    mine = br.bond_orders(x, types, thr, n)
    theirs = br.orders_of(br.torch_dist_pm(x), types, thr) if n is None or n == len(x) else None
    return mine, theirs, (None if theirs is None else mine != theirs)


def ulps(a, b):
    a, b = np.asarray(a, np.float32).view(np.int32).astype(np.int64), np.asarray(b, np.float32).view(np.int32)
    return np.abs(a - b)


# ---- CPU ----------------------------------------------------------------------------------------------------------------

def test_fma32_rounds_once():
    """Cases where rounding a float64 sum to fp32 rounds twice, and random ones, against exact rationals."""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    a = rng.standard_normal(2000).astype(np.float32)
    b = rng.standard_normal(2000).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.integers(-4, 5, 2000) * 2.0 ** -24)).astype(np.float32)
    a = np.append(a, np.float32(1 + 2 ** -12)); b = np.append(b, np.float32(1 + 2 ** -12))
    c = np.append(c, np.float32(2 ** -48))
    got = br.fma32(a, b, c)
    for k in range(len(a)):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        errs = [abs(Fraction(float(v)) - exact) for v in cands]
        best = min(errs)
        ties = [v for v, e in zip(cands, errs) if e == best]
        want = ties[0] if len(ties) == 1 else [v for v in ties if int(np.float32(v).view(np.int32)) % 2 == 0][0]
        assert got[k] == want, (k, a[k], b[k], c[k], got[k], want)


@pytest.mark.parametrize("offset", OFFSETS)
def test_emulation_is_torch_cdist_bitwise_up_to_25_atoms(offset):
    rng = np.random.default_rng(int(offset) + 11)
    pairs = 0
    for n in list(range(2, 26)) * 8:
        x, _ = random_chain(rng, n, offset, 8)
        lo = np.tril(np.ones((n, n), bool), -1)
        mine, theirs = br.pair_dist_pm(x)[lo], br.torch_dist_pm(x)[lo]
        assert np.array_equal(mine.view(np.int32), theirs.view(np.int32)), (n, offset)
        pairs += lo.sum()
    assert pairs > 10000


def test_emulation_is_torch_cdist_within_one_ulp_above_25_atoms():
    """Above 25 atoms torch's sgemm entries equal the stated order bitwise, and torch's CPU square root rounds a fraction
    of its results one ulp away from the correctly rounded root: the distances in A differ by at most one ulp, on a small,
    reported share of pairs. A torch or MKL build that changes either fails here."""
    rng = np.random.default_rng(5)
    diff = total = 0
    for offset in OFFSETS:
        for n in (26, 30, 45, 60):
            for _ in range(6):
                x, _ = random_chain(rng, n, offset, 8)
                lo = np.tril(np.ones((n, n), bool), -1)
                c = torch_entries(x)
                assert np.array_equal(c[lo].view(np.int32), br.matmul_entry(x[:, None], x[None, :])[lo].view(np.int32))
                t = torch.from_numpy(x)[None]
                u = ulps(np.sqrt(np.maximum(c, 0))[lo], torch.cdist(t, t)[0].numpy()[lo])
                assert u.max() <= 1, (offset, n, int(u.max()))
                diff += int((u != 0).sum())
                total += int(lo.sum())
    print(f"torch.cdist vs the correctly rounded root above 25 atoms: {diff} of {total} pairs one ulp apart")
    assert 0 < diff <= 0.02 * total


def torch_entries(x):
    """torch's _euclidean_dist matrix for the rows x, before the clamp and square root."""
    t = torch.from_numpy(np.asarray(x, np.float32))
    nrm = t.pow(2).sum(-1, keepdim=True)
    a = torch.cat([t.mul(-2), nrm, torch.ones_like(nrm)], -1)
    b = torch.cat([t, torch.ones_like(nrm), nrm], -1)
    return a.matmul(b.mT).numpy()


@pytest.mark.parametrize("is_geom", [False, True])
def test_designed_pairs_straddle_their_thresholds(is_geom):
    """Every designed pair decides differently in the two forms; at its molecule's n the emulation decides as torch.cdist
    does, except on ambiguous pairs; the pair is the only link between the chain's halves."""
    thr = tables(is_geom)
    mols = designed(is_geom)
    assert len(mols) == len(br.threshold_cases(thr)) * 2 * len(OFFSETS)
    amb = 0
    for x, ty, j, i, case in mols:
        n = len(x)
        assert n > br.CDIST_MM_ROWS
        direct = br.orders_of(br.direct_dist_pm(x[:, None], x[None, :]), ty, thr)
        mine, theirs, a = decisions(x, ty, thr)
        assert direct[i, j] != mine[i, j], case
        off = np.ones_like(mine, bool)
        off[i, j] = off[j, i] = False
        assert np.array_equal(direct[off], mine[off]), case                 # only the pair flips
        chain = np.abs(np.subtract.outer(np.arange(n), np.arange(n))) == 1
        assert np.array_equal(mine[off] > 0, chain[off]), case              # a chain, linked through the pair
        amb += int(a[i, j])
        assert not (a & off).any(), case
    print(f"{'geom' if is_geom else 'zinc'}: {amb} of {len(mols)} designed pairs ambiguous")
    assert amb <= 0.01 * len(mols)


def twins(is_geom):
    return br.twins(tables(is_geom))


@pytest.mark.parametrize("is_geom", [False, True])
def test_twin_molecules_of_25_and_26_atoms_decide_the_pair_differently(is_geom):
    thr = tables(is_geom)
    for x25, x26, t25, t26, j, i in twins(is_geom):
        o25, c25, a25 = decisions(x25, t25, thr)
        o26, c26, a26 = decisions(x26, t26, thr)
        assert np.array_equal(o25, c25)                                     # n <= 25: never ambiguous
        assert o25[i, j] != o26[i, j]
        assert a26[i, j] or c25[i, j] != c26[i, j]                          # what the reference itself does


def pocket_designs(is_geom):
    """br.pocket_designs packed: (xh, node_mask, pocket_only with the last 10 rows set, [(j, i)])."""
    mols = br.pocket_designs(tables(is_geom))
    xh, nm = pack([(x, ty) for x, ty, _, _ in mols], n_types(is_geom))
    po = torch.zeros(nm.shape)
    po[:, 20:30] = 1
    return xh, nm, po, [(j, i) for _, _, j, i in mols]


@pytest.mark.parametrize("is_geom", [False, True])
def test_pocket_designs_cross_25_when_the_pocket_is_dropped(is_geom):
    thr = tables(is_geom)
    xh, nm, po, pairs = pocket_designs(is_geom)
    for b, (j, i) in enumerate(pairs):
        x, ty = xh[b, :30, :3].numpy(), xh[b, :30, 3:].argmax(1).numpy()
        assert br.bond_orders(x[:20], ty[:20], thr)[i, j] != br.bond_orders(x, ty, thr)[i, j]
        assert br.bond_orders(x, ty, thr)[20:, :].sum() == 0                # the pocket bonds to nothing


def linker_designs(is_geom):
    """br.linker_designs packed: (xh, node_mask, linker_mask)."""
    mols = br.linker_designs(tables(is_geom))
    xh, nm = pack([(x, ty) for x, ty, _ in mols], n_types(is_geom))
    return xh, nm, torch.from_numpy(np.stack([lm for _, _, lm in mols]))


def oracle_hash(x, ty, thr, n=None):
    return gho.as_int64(gho.graph_hash(ty, br.bond_orders(x, ty, thr, n)))


@pytest.mark.parametrize("is_geom", [False, True])
def test_linker_designs_hash_one_pair_differently_in_l_and_h(is_geom):
    thr = tables(is_geom)
    xh, nm, lm = linker_designs(is_geom)
    for b in range(xh.shape[0]):
        x, ty = xh[b, :, :3].numpy(), xh[b, :, 3:].argmax(1).numpy()
        rows = np.flatnonzero(lm[b].numpy())
        whole = br.bond_orders(x, ty, thr)
        alone = br.bond_orders(x[rows], ty[rows], thr)
        assert not np.array_equal(whole[np.ix_(rows, rows)], alone), b


def nan_designs(is_geom):
    """The designed molecules with one chain atom (not of the pair) set to NaN."""
    out = []
    for x, ty, j, i, case in designed(is_geom, seed=21)[::4]:
        x = x.copy()
        x[0 if j > 0 else len(x) - 1] = np.nan
        out.append((x, ty, j, i, case))
    return out


# ---- GPU ----------------------------------------------------------------------------------------------------------------

def dev():
    return torch.device("cuda", 0)


def device_orders(xh, nm, is_geom):
    T = n_types(is_geom)
    return mb.bond_orders(xh[:, :, 3:3 + T].to(dev()), xh[:, :, :3].to(dev()), nm.to(dev()), is_geom).cpu().numpy()


def compare_orders(E, mols, thr, label):
    """E (B, N, N) lower-triangular against the emulation on every pair and torch.cdist except on ambiguous pairs; returns
    the ambiguous count. The failure lists the molecules and pairs."""
    bad, amb = [], 0
    for b, (x, ty) in enumerate(mols):
        n = len(x)
        mine, theirs, a = decisions(x, ty, thr)
        lo = np.tril(np.ones((n, n), bool), -1)
        got = E[b, :n, :n]
        for i, j in zip(*np.nonzero(lo & (got != mine))):
            d = br.pair_dist_pm(x)[i, j]
            bad.append(f"mol {b} (n={n}) pair ({i},{j}) types ({ty[i]},{ty[j]}): E={got[i, j]} emulation={mine[i, j]} "
                       f"cdist={theirs[i, j]} d={d!r} pm")
        amb += int((a & lo).sum())
    assert not bad, f"{label}: {len(bad)} pairs differ from the emulation:\n" + "\n".join(bad[:60])
    return amb


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_bond_orders_of_designed_pairs_follow_torch_cdist(is_geom):
    thr = tables(is_geom)
    mols = designed(is_geom) + twins_flat(is_geom) + nan_designs(is_geom)
    xh, nm = pack([(m[0], m[1]) for m in mols], n_types(is_geom))
    amb = compare_orders(device_orders(xh, nm, is_geom), [(m[0], m[1]) for m in mols], thr, "designed")
    print(f"{'geom' if is_geom else 'zinc'}: {amb} ambiguous pairs in {len(mols)} designed molecules")
    assert amb <= 0.01 * len(mols)


def twins_flat(is_geom):
    out = []
    for x25, x26, t25, t26, j, i in twins(is_geom):
        out += [(x25, t25, j, i, None), (x26, t26, j, i, None)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("offset", OFFSETS)
def test_bond_orders_of_random_chains_follow_torch_cdist(offset):
    rng = np.random.default_rng(int(offset) + 101)
    for is_geom in (False, True):
        thr = tables(is_geom)
        mols = [random_chain(rng, int(rng.integers(20, 61)), offset, n_types(is_geom)) for _ in range(1024)]
        xh, nm = pack(mols, n_types(is_geom), N=60)
        amb = compare_orders(device_orders(xh, nm, is_geom), mols, thr, f"random chains at {offset} A")
        print(f"offset {offset} A, {'geom' if is_geom else 'zinc'}: {amb} ambiguous pairs in {len(mols)} molecules")


def check_verdicts(xh, nm, is_geom, po=None, linker=None):
    """connected, valences and graph_hashes (and linker_hashes) of the device against the emulation on every molecule.
    torch.cdist enters through the ambiguity count: a molecule is ambiguous when live torch.cdist decides one of its pairs
    differently from the emulation, and the count is returned for the caller to bound. (Where nothing is ambiguous the
    cdist verdicts are the emulation's, so they are not compared again.)"""
    thr = tables(is_geom)
    d = dev()
    pod = None if po is None else po.to(d)
    conn = mb.connected(xh.to(d), nm.to(d), is_geom, pod).cpu().numpy()
    val = mb.valences(xh.to(d), nm.to(d), is_geom, pod).cpu().numpy()
    H = mb.graph_hashes(xh.to(d), nm.to(d), is_geom, pod).cpu().numpy()
    L = None if linker is None else mb.linker_hashes(xh.to(d), nm.to(d), linker.to(d), is_geom, pod).cpu().numpy()
    bad, amb = [], 0
    for b in range(xh.shape[0]):
        keep = nm[b].numpy() != 0
        if po is not None:
            keep &= po[b].numpy() == 0
        rows = np.flatnonzero(keep)
        x, ty = xh[b, rows, :3].numpy(), xh[b, rows, 3:].argmax(1).numpy()
        mine, theirs, a = decisions(x, ty, thr)
        amb += bool(a.any())
        for label, o in (("emulation", mine),):
            c = gho_connected(o)
            v = np.zeros(xh.shape[1], np.int64)
            v[rows] = o.sum(1)
            h = gho.as_int64(gho.graph_hash(ty, o))
            if bool(conn[b]) != c or not np.array_equal(val[b], v) or int(H[b]) != h:
                bad.append(f"mol {b} (n={len(rows)}) vs {label}: connected {bool(conn[b])}/{c}, valences "
                           f"{np.flatnonzero(val[b] != v).tolist()} differ, hash {'ok' if int(H[b]) == h else 'differs'}")
        if L is not None:
            lr = np.flatnonzero(keep & (linker[b].numpy() != 0))
            xl, tl = xh[b, lr, :3].numpy(), xh[b, lr, 3:].argmax(1).numpy()
            if int(L[b]) != oracle_hash(xl, tl, thr):
                bad.append(f"mol {b}: linker hash differs from the emulation over its {len(lr)} linker atoms")
    assert not bad, f"{len(bad)} verdicts differ:\n" + "\n".join(bad[:60])
    return amb


def gho_connected(o):
    n = o.shape[0]
    if n == 0:
        return False
    seen, todo = {0}, [0]
    while todo:
        k = todo.pop()
        for m in np.flatnonzero(o[k]):
            if int(m) not in seen:
                seen.add(int(m))
                todo.append(int(m))
    return len(seen) == n


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_checks_of_designed_molecules_follow_torch_cdist(is_geom):
    mols = designed(is_geom) + twins_flat(is_geom)
    xh, nm = pack([(m[0], m[1]) for m in mols], n_types(is_geom))
    amb = check_verdicts(xh, nm, is_geom)
    print(f"{'geom' if is_geom else 'zinc'}: {amb} of {len(mols)} designed molecules hold an ambiguous pair")
    assert amb <= 0.01 * len(mols) + 1


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_checks_measure_over_the_atoms_left_after_the_pocket(is_geom):
    thr = tables(is_geom)
    xh, nm, po, pairs = pocket_designs(is_geom)
    check_verdicts(xh, nm, is_geom, po=po)
    E = device_orders(xh, nm, is_geom)
    mols = [(xh[b, :30, :3].numpy(), xh[b, :30, 3:].argmax(1).numpy()) for b in range(xh.shape[0])]
    compare_orders(E, mols, thr, "pocket designs, all rows")
    for b, (j, i) in enumerate(pairs):
        conn = mb.connected(xh[b:b + 1].to(dev()), nm[b:b + 1].to(dev()), is_geom, po[b:b + 1].to(dev())).item()
        assert conn == bool(br.bond_orders(mols[b][0][:20], mols[b][1][:20], thr)[i, j]), b
        assert (E[b, i, j] > 0) != conn, b                                 # bond_orders decides the pair the other way


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_linker_hash_measures_over_the_linker_atoms(is_geom):
    xh, nm, lm = linker_designs(is_geom)
    check_verdicts(xh, nm, is_geom, linker=lm)


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_pocket_clashes_keep_the_direct_form_above_25_atoms(is_geom):
    """The clash check is the project's own predicate: a linker atom and a pocket atom straddling the clash distance
    between the forms clash as the direct form says, in molecules of 60 rows with 30 pocket atoms and 30 checked atoms, so
    that a check measuring over the checked atoms, the pocket atoms or all rows would each use the matmul form."""
    rng = np.random.default_rng(17)
    T = n_types(is_geom)
    table = mb.clash_table(is_geom).numpy()
    thr = tables(is_geom)
    mols, want = [], []
    for below in (True, False):
        for off in OFFSETS:
            t = float(table[0, 0])
            xj, xi = br.straddling_pair(rng, t, off, below)
            x, ty, j, i = br.chain_around(xj, xi, 0, 0, 29, 29, thr)
            mols.append((x, ty))
            want.append((j, i, below))
    xh, nm = pack(mols, T)
    lm = torch.zeros(nm.shape)
    po = torch.zeros(nm.shape)
    for b, (j, i, below) in enumerate(want):
        assert j + 1 > br.CDIST_MM_ROWS and len(mols[b][0]) - j - 1 > br.CDIST_MM_ROWS
        po[b, :j + 1] = 1                                                  # the chain up to the pair is pocket
        lm[b, i] = 1                                                       # the pair's later atom is the linker atom
    counts = mb.pocket_clashes(xh.to(dev()), nm.to(dev()), lm.to(dev()), po.to(dev()), is_geom).cpu().numpy()
    for b, (j, i, below) in enumerate(want):
        x = mols[b][0]
        d = br.direct_dist_pm(x[i][None], x[:j + 1])
        assert counts[b, i] == int((d < table[0, 0]).sum()), b
        assert (d[-1] < table[0, 0]) == below, b


@pytest.mark.gpu
def test_sample_chain_verdicts_on_a_geom_batch_over_25_atoms():
    """One sample_chain(require_connected=True, require_valid=True) with two recovery rounds on a GEOM batch of 28-36 atoms
    per molecule: the rounds check resampled rows through their row map, and the flags the call reports equal the
    oracle's on the returned chain[0], decided on the emulation; molecules where live torch.cdist decides a pair
    differently are counted and bounded."""
    from difflinker_b200 import synthetic
    from difflinker_b200.batching import collate
    from difflinker_b200.ddpm import sampler_inputs
    import dl_helpers as helpers
    B = 16
    spec = synthetic.WorkloadSpec("bonds_geom", B=B, N=36, n_min=28, l_min=3, l_max=6, F=9, L=2, T=10, seed=4)
    ddpm, _ = helpers.build_ddpm(spec, 0)
    ddpm.edm.T = 10
    ddpm = ddpm.to(dev())
    assert ddpm.edm.is_geom
    data = {k: (v.to(dev()) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data)
    chain = ddpm.edm.sample_chain(**kw, keep_frames=2, seeds=list(range(40, 40 + B)), nan_retries=2, require_valid=True,
                                  require_connected=True)
    edm = ddpm.edm
    assert int(edm.last_attempts.max()) > 0                               # some rows went through the recovery rounds
    chain0 = chain[0].cpu()
    nm = kw['node_mask'].reshape(B, -1).cpu() != 0
    thr = tables(True)
    max_val = mb.max_valence_table(True).numpy()
    amb = 0
    for b in range(B):
        rows = np.flatnonzero(nm[b].numpy())
        assert len(rows) > br.CDIST_MM_ROWS
        x, ty = chain0[b, rows, :3].numpy(), chain0[b, rows, 3:12].argmax(1).numpy()
        mine, theirs, a = decisions(x, ty, thr)
        amb += bool(a.any())
        assert bool(edm.last_connected[b]) == gho_connected(mine), b
        assert bool(edm.last_valid[b]) == bool((mine.sum(1) <= max_val[ty]).all()), b
    print(f"sample_chain on GEOM: attempts {edm.last_attempts.tolist()}, valid {int(edm.last_valid.sum())}, connected "
          f"{int(edm.last_connected.sum())} of {B}; {amb} molecules hold an ambiguous pair")
    assert amb <= 1
