"""The linker-size classifier's kernels (dl_sizegnn_forward: k_prep -> [k_edge_simt<GCL, ReLU> -> k_node<ReLU>] x L ->
k_sz_out) against the oracle in float64, at the shapes they run at, molecule by molecule.

Since linker sizes are drawn on the device from each molecule's seed, these logits decide discrete outcomes: the draw is a
step function of them, and one edge more or less moves them far. So the batches here are built so that every layout occurs
by design, and every molecule has one layout, so that a failing molecule names it:

- FC batches (ZINC and GEOM types) padded to N = 300, with 0 .. 257 fragment atoms (8 .. 1 rows per 128-edge tile, rows of
  exactly 128 columns, 2- and 3-chunk rows with a one-column last chunk) and linker rows between the fragment rows, so the
  live columns are not contiguous. Even molecules lie in a 1.2 A ball (every pair an edge, large sums); odd ones are groups
  of 1, 2 and 3 atoms 10 A apart (sparse graphs, isolated atoms with only their self loop; no fragment: the bias).
- Node-kernel tails: B * N = 1 and 31 modulo the 32-node tile.
- The pocket path, size_logits(with_pocket=True, adjust_shape=True): every pocket atom moves to the origin and joins every
  other at radial 0, so each pocket row sums a clique of n_pocket messages: B = 64, N = 300 (3 chunks per row), B = 2,
  N = 4000 (a whole protein) and B = 1, N = 6144 (the largest N the work plan takes). Some fragment atoms sit within
  sqrt(6) A of the origin and join the clique.
- Models: ZINC (8 -> 10, 3 layers) with and without batch norm, GEOM (9 -> 33, batch norm), 1 and 4 layers, 64 classes,
  32 input features, and batch norm with running variances down to 1e-3 (large folded gains).
- radial < 6 in torch's rounding order: pairs whose squared distance falls on different sides of 6 in torch's order
  ((dx^2 + dy^2) + dz^2, each term rounded) and in the contracted FMA form, one pair per molecule.

The criterion (the rule of fp64_rows): max_c |got - ref64| <= max(C_DRIFT * drift_b, TAU * S_b) for every molecule b, with
drift_b = max_c |ref32 - ref64| the oracle's own fp32 error on the molecule and S_b = max_c |ref64[b]|, and at least half of
a case's molecules within TAU * S_b outright. The seeded draw on the GPU's logits must then equal the oracle's draw on ref64
rounded to fp32 for every (molecule, seed) pair whose u does not lie in the band around a normalised cumulative boundary
P_i = c_i / S that an error of eps_b (the molecule's bound, plus the rounding of ref64 to fp32) per logit can move: logit
errors within eps of each other scale every softmax weight by a factor within [1, e^w] of a common one, w = 2 eps, which
moves P_i by at most (e^w - 1) P_i (1 - P_i). At most 1 % of at least 10^4 pairs per case may be excluded.
"""
import functools
import itertools
from fractions import Fraction

import numpy as np
import pytest
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
from difflinker_b200.linker_size import (GEOM_TRAIN_LINKER_ID2SIZE, GEOM_TRAIN_LINKER_SIZE2ID, SizeClassifier,
                                         collate_with_fragment_edges, draw_sizes)
from fp64_rows import C_DRIFT, TAU, _full_fp32_matmul, dev
from oracle import difflinker_oracle as orc

N_FC = 300
FRAGS = (0, 1, 2, 8, 16, 17, 32, 33, 64, 65, 127, 128, 129, 255, 256, 257)
NODE_TM = 32
PLAN_MAX_N = 6144
MIN_PAIRS = 10_000                       # (molecule, seed) pairs per case for the draw comparison
WORST = {}                               # case -> (worst err / bound, worst err / S_b, molecules within TAU, excluded draws)


# ------------------------------------------------------------------------------------------------------------ batches
def size_collate(items):
    """collate_with_fragment_edges without its (B*N*N) `edges` list (600 MB at N = 6144), which the kernels never read."""
    out = collate(items)
    frag = out['fragment_mask'].squeeze(-1).to(torch.int8)
    B, N = frag.shape
    em = frag[:, None, :] * frag[:, :, None] * ~torch.eye(N, dtype=torch.int8).unsqueeze(0)
    out['edge_mask'] = em.view(B * N * N, 1)
    return out


def _one_hot(g, n, F, last_free=True):
    types = torch.randint(0, F if last_free else F - 1, (n,), generator=g)
    return torch.nn.functional.one_hot(types, F).float()


def _grid(k, spacing):
    """k points of a cubic grid `spacing` A apart, nearest to the origin first."""
    m = int(np.ceil(k ** (1 / 3))) + 1
    ax = (torch.arange(m, dtype=torch.float64) - m // 2) * spacing
    pts = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), dim=-1).reshape(-1, 3)
    return pts[torch.argsort(pts.norm(dim=1), stable=True)][:k]


def _ball(g, n, radius):
    v = torch.randn((n, 3), generator=g, dtype=torch.float64)
    v = v / v.norm(dim=1, keepdim=True).clamp(min=1e-12)
    return v * radius * torch.rand((n, 1), generator=g, dtype=torch.float64) ** (1 / 3)


def fc_molecule(g, n_frag, ball, F):
    """n_frag fragment atoms with a linker row after every third one (so the live columns are not contiguous), filled up
    with linker rows to N_FC when n_frag = max(FRAGS). ball: a 0.6 A radius ball; otherwise groups of 1, 2, 3 atoms
    (cycling) within 0.3 A of grid points 10 A apart. Returns the item and its fragment rows' degree histogram."""
    n_link = N_FC - n_frag if n_frag == max(FRAGS) else min(n_frag // 3 + 2, N_FC - n_frag)
    role = []
    f = 0
    while f < n_frag or len(role) < n_frag + n_link:
        if f < n_frag and (len(role) % 4 != 3 or role.count('l') >= n_link):
            role.append('f'); f += 1
        else:
            role.append('l')
    n = len(role)
    deg = {}
    if ball:
        frag_pos = _ball(g, n_frag, 0.6)
        if n_frag:
            deg[n_frag] = n_frag
    else:
        sizes, k = [], 0
        while sum(sizes) < n_frag:
            sizes.append(min(1 + k % 3, n_frag - sum(sizes))); k += 1
        centres = _grid(len(sizes), 10.0)
        frag_pos = torch.cat([c + _ball(g, s, 0.3) for s, c in zip(sizes, centres)]) if sizes else torch.zeros((0, 3))
        for s in sizes:
            deg[s] = deg.get(s, 0) + s
    pos = 20.0 * torch.randn((n, 3), generator=g, dtype=torch.float64)     # linker rows: anywhere, masked
    fm = torch.tensor([1.0 if r == 'f' else 0.0 for r in role])
    pos[fm != 0] = frag_pos
    item = {'positions': pos.float(), 'one_hot': _one_hot(g, n, F), 'fragment_mask': fm, 'linker_mask': 1.0 - fm}
    return item, deg


def pocket_molecule(g, n_pocket, F, n_near=5, n_far=15, n_link=8):
    """Fragment-only atoms (n_near within 1.5 A of the origin, n_far on a 7 A grid beyond 5 A), a pocket of n_pocket atoms
    and n_link linker atoms, in the datasets' row order. The one-hot has F columns, the last one zero on fragment-only rows
    and used by some pocket atoms: adjust_shape drops it."""
    far = _grid(n_far + 1, 7.0)[1:]
    frag = torch.cat([_ball(g, n_near, 1.5), far])
    pocket = 8.0 * torch.randn((n_pocket, 3), generator=g, dtype=torch.float64)       # moved to the origin by with_pocket
    link = 3.0 * torch.randn((n_link, 3), generator=g, dtype=torch.float64)
    nf = n_near + n_far
    n = nf + n_pocket + n_link
    oh = torch.cat([_one_hot(g, nf, F, last_free=False), _one_hot(g, n_pocket, F), _one_hot(g, n_link, F)])
    fo = torch.zeros(n); fo[:nf] = 1
    pk = torch.zeros(n); pk[nf:nf + n_pocket] = 1
    return {'positions': torch.cat([frag, pocket, link]).float(), 'one_hot': oh, 'fragment_mask': fo + pk,
            'linker_mask': 1.0 - fo - pk, 'fragment_only_mask': fo, 'pocket_mask': pk}


# Squared distances that fall on different sides of 6 in torch's order and in the contracted forms ptxas emits for
# ex*ex + ey*ey + ez*ez (k_edge_simt<false, ACT_RELU> before radial_rn: FMUL then two chained FFMA; every order of the three
# terms is kept, so the pairs do not depend on which one the compiler multiplies first).
def _round32(v):
    """Round the rational v to the nearest fp32 (ties to even); v is in fp32's normal range or 0."""
    if v == 0:
        return Fraction(0)
    s = -1 if v < 0 else 1
    a = abs(v)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    ulp = Fraction(2) ** (e - 23)
    q = a / ulp
    n = q.numerator // q.denominator
    r = q - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return s * n * ulp


def torch_radial(d):
    x, y, z = (Fraction(float(c)) for c in d)
    return _round32(_round32(_round32(x * x) + _round32(y * y)) + _round32(z * z))


def fma_radials(d):
    out = []
    for a, b, c in itertools.permutations([Fraction(float(v)) for v in d]):
        out.append(_round32(c * c + _round32(b * b + _round32(a * a))))
    return out


@functools.lru_cache(maxsize=None)
def rounding_pairs(per_side=6, seed=91):
    """(below, above): fp32 difference vectors with torch's radial < 6 but every FMA form >= 6, and the reverse."""
    rng = np.random.default_rng(seed)
    below, above = [], []
    while len(below) < per_side or len(above) < per_side:
        v = rng.standard_normal(3)
        d = (v / np.linalg.norm(v) * np.sqrt(6.0)).astype(np.float32)
        if np.min(np.abs(d)) < 0.1:
            continue
        t, fm = torch_radial(d), fma_radials(d)
        if t < 6 and all(r >= 6 for r in fm) and len(below) < per_side:
            below.append(tuple(float(c) for c in d))
        elif t >= 6 and all(r < 6 for r in fm) and len(above) < per_side:
            above.append(tuple(float(c) for c in d))
    return below, above


def rounding_molecule(g, d, F):
    """An isolated fragment pair (one atom at the origin, the other at d), two fragment atoms 20 A away and two linker rows."""
    pos = torch.tensor([[0.0, 0.0, 0.0], list(d), [20.0, 0, 0], [0, 20.0, 0], [1.0, 1, 1], [2.0, 0, 1]], dtype=torch.float32)
    fm = torch.tensor([1.0, 1, 1, 1, 0, 0])
    return {'positions': pos, 'one_hot': _one_hot(g, 6, F), 'fragment_mask': fm, 'linker_mask': 1.0 - fm}


@functools.lru_cache(maxsize=None)
def batch(name):
    """(data, designed degree histograms per molecule or None)."""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if name.startswith("fc"):                                              # fc8, fc9, fc32: one-hot width
        F = int(name[2:])
        mols = [fc_molecule(g, n, k % 2 == 0, F) for k, n in enumerate(FRAGS)]
        return size_collate([m for m, _ in mols]), [d for _, d in mols]
    if name.startswith("tail"):                                            # tail1 / tail31: B * N mod NODE_TM
        B, N = {"tail1": (3, 11), "tail31": (5, 19)}[name]
        items = []
        for b in range(B):
            n = N if b == 0 else N - 1 - b
            fm = (torch.arange(n) % 3 != 2).float()
            items.append({'positions': _ball(g, n, 0.6 + b).float(), 'one_hot': _one_hot(g, n, 8), 'fragment_mask': fm,
                          'linker_mask': 1.0 - fm})
        return size_collate(items), None
    if name.startswith("pocket"):
        B, N = {"pocket_cfg4": (64, 300), "pocket_protein": (2, 4000), "pocket_6144": (1, PLAN_MAX_N)}[name]
        items = [pocket_molecule(g, N - 28 - 3 * (b % 5), 10) for b in range(B)]     # 20 fragment, 8 linker atoms
        return size_collate(items), None
    if name == "rounding":
        below, above = rounding_pairs()
        return size_collate([rounding_molecule(g, d, 8) for d in below + above]), None
    raise KeyError(name)


# -------------------------------------------------------------------------------------------------------------- models
MODELS = {   # name: (in_node_nf, out_node_nf, n_layers, normalization)
    "zinc": (8, 10, 3, None), "zinc_bn": (8, 10, 3, "batch_norm"), "geom_bn": (9, 33, 3, "batch_norm"),
    "zinc_L1": (8, 10, 1, None), "zinc_L4": (8, 10, 4, "batch_norm"), "out64": (8, 64, 3, None),
    "in32": (32, 10, 2, "batch_norm"), "bn_small_var": (8, 10, 3, "batch_norm"),
}


@functools.lru_cache(maxsize=None)
def model(name):
    F, C, L, norm = MODELS[name]
    if C == len(GEOM_TRAIN_LINKER_ID2SIZE):
        tables = dict(linker_id2size=GEOM_TRAIN_LINKER_ID2SIZE, linker_size2id=GEOM_TRAIN_LINKER_SIZE2ID)
    else:
        table = list(range(1, C + 1))
        tables = dict(linker_id2size=table, linker_size2id={s: i for i, s in enumerate(table)})
    torch.manual_seed(100 + len(name))
    m = SizeClassifier(in_node_nf=F, out_node_nf=C, n_layers=L, normalization=norm, **tables)
    synthetic.init_size_gnn_like_trained(m, 7)
    if name == "bn_small_var":
        g = torch.Generator().manual_seed(8)
        with torch.no_grad():
            for k, b in m.named_buffers():
                if k.endswith("running_var"):
                    b.copy_(10.0 ** (-3.0 * torch.rand(b.shape, generator=g)))          # 1e-3 .. 1
    return m.eval()


B_OF = {"fc8": 16, "fc9": 16, "fc32": 16, "tail1": 3, "tail31": 5, "pocket_cfg4": 64, "pocket_protein": 2,
        "pocket_6144": 1, "rounding": 12}
CASES = {    # case: (batch, model, pocket)
    "fc_zinc": ("fc8", "zinc", False), "fc_zinc_bn": ("fc8", "zinc_bn", False), "fc_geom_bn": ("fc9", "geom_bn", False),
    "fc_L1": ("fc8", "zinc_L1", False), "fc_L4": ("fc8", "zinc_L4", False), "fc_out64": ("fc8", "out64", False),
    "fc_in32": ("fc32", "in32", False), "fc_bn_small_var": ("fc8", "bn_small_var", False),
    "tail1": ("tail1", "zinc", False), "tail31": ("tail31", "zinc_bn", False),
    "pocket_cfg4": ("pocket_cfg4", "geom_bn", True), "pocket_protein": ("pocket_protein", "geom_bn", True),
    "pocket_6144": ("pocket_6144", "geom_bn", True), "rounding": ("rounding", "zinc", False),
}


def oracle_logits(m, data, pocket, dtype, device):
    kw = dict(with_pocket=pocket, adjust_shape=pocket)
    dd = {k: v.to(device) for k, v in data.items() if torch.is_tensor(v)}
    with torch.no_grad(), _full_fp32_matmul():
        out = orc.size_classifier_forward(m.state_dict(), dd, m.in_node_nf, m.gnn.n_layers, m.gnn.normalization,
                                          dtype=dtype, **kw)
    return out.double().cpu()


_REFS = {}


def references(case):
    if case not in _REFS:
        bname, mname, pocket = CASES[case]
        data, m = batch(bname)[0], model(mname)
        _REFS[case] = (oracle_logits(m, data, pocket, torch.float64, dev()), oracle_logits(m, data, pocket, torch.float32, dev()))
    return _REFS[case]


def gpu_logits(m, data, pocket):
    d = dev()
    dd = {k: v.to(d) for k, v in data.items() if torch.is_tensor(v)}
    return m.to(d).size_logits(dd, with_pocket=pocket, adjust_shape=pocket).double().cpu()


# ----------------------------------------------------------------------------------------------------------- criterion
def check_molecules(case, got, ref64, ref32, half_within_tau=True):
    """max_c |got - ref64| <= max(C_DRIFT * drift_b, TAU * S_b) per molecule, and (half_within_tau) half of them within
    TAU * S_b; returns the per-molecule bounds."""
    err = (got - ref64).abs().amax(1)
    drift = (ref32 - ref64).abs().amax(1)
    scale = ref64.abs().amax(1)
    bound = torch.maximum(C_DRIFT * drift, TAU * scale)
    ratio = torch.where(err == 0, 0.0, err / bound)
    within = int((err <= TAU * scale).sum())
    WORST[case] = [ratio.max().item(), (err / scale.clamp(min=1e-300)).max().item(), f"{within}/{got.shape[0]}", None,
                   scale.max().item()]
    bad = [f"molecule {b}: err {err[b]:.3e}, drift {drift[b]:.3e}, S_b {scale[b]:.3e}" for b in torch.nonzero(ratio > 1).flatten().tolist()]
    assert not bad, f"{case}:\n" + "\n".join(bad[:10])
    assert torch.isfinite(ref32).all()
    assert not half_within_tau or 2 * within >= got.shape[0], f"{case}: only {within} of {got.shape[0]} molecules within {TAU} * S_b"
    return bound


def draw_bounds(logits32, width, u):
    """Per row: whether u lies within (e^width - 1) P_i (1 - P_i) + 1e-12 of a normalised cumulative boundary P_i = c_i / S of
    the header's draw (the first i with u * S < c_i). A second logit row whose difference from this one spans at most
    `width` (max_c - min_c) scales every softmax weight by a factor within [1, e^width] of a common one; that moves the odds
    P_i / (1 - P_i) by a factor within e^(+-width), hence P_i by at most (e^width - 1) P_i (1 - P_i), so the two rows' draws
    can differ only for such u (1e-12: the fp64 evaluation of either draw). Computed in log space: the band is tight where
    the softmax is peaked, whatever the logits' scale."""
    l = logits32.astype(np.float64)
    log_c = np.logaddexp.accumulate(l, axis=1)                              # log of the prefix sums
    log_s = log_c[:, -1:]
    log_tail = np.full_like(l, -np.inf)
    log_tail[:, :-1] = np.logaddexp.accumulate(l[:, ::-1], axis=1)[:, ::-1][:, 1:]   # log of the sums after i
    with np.errstate(over='ignore', divide='ignore'):
        log_gain = np.where(width > 30, width, np.log(np.expm1(width)))[:, None]
    P = np.exp(log_c - log_s)
    band = np.exp(np.minimum(log_gain + (log_c - log_s) + (log_tail - log_s), 0.0))
    return (np.abs(u[:, None] - P) <= band + 1e-12).any(1)


def draw_width(bound, ref64):
    """2 (eps_b + rounding of ref64 to fp32): the spread of got - fp32(ref64) over the classes that the bound allows."""
    return (2 * (bound + (ref64 - ref64.float().double()).abs().amax(1))).numpy()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst per-molecule ratios (err / bound, err / S_b, molecules within TAU * S_b, excluded draws, max S_b):")
        for k, (w, r, f, x, sm) in WORST.items():
            print(f"  {k:20s} {w:9.3e} {r:9.3e} {f:>7s}  {str(x):>11s}  {sm:9.3e}")                   # x: None if not reached


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_size_collate_is_collate_with_fragment_edges_without_edges():
    data, _ = batch("fc8")
    items = [fc_molecule(torch.Generator().manual_seed(3), n, n % 2 == 0, 8)[0] for n in (0, 5, 17)]
    a, b = size_collate(items), collate_with_fragment_edges(items)
    assert 'edges' not in a and set(a) == set(b) - {'edges'}
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_fc_batches_have_the_designed_layouts():
    """Live columns per molecule (the work plan's nc: the fragment rows), rows per 128-edge tile and chunks per row, non-
    contiguous live columns, and the designed degree histogram of the oracle's edge set."""
    for name in ("fc8", "fc9", "fc32"):
        data, degs = batch(name)
        B, N = data['positions'].shape[:2]
        assert (B, N) == (len(FRAGS), N_FC)
        em = data['edge_mask'].view(B, N, N) != 0
        nc = em.any(1).sum(1).tolist()
        assert nc == list(FRAGS)
        per = [min(8, 128 // c) if c < 128 else 1 for c in nc if c]
        chunks = [-(-c // 128) for c in nc if c]
        assert set(per) == {8, 7, 4, 3, 2, 1} and {1, 2, 3} <= set(chunks)
        assert 129 in nc and 257 in nc and 128 in nc                     # one-column last chunks, an exact 128-column row
        cols = em.any(1)
        for b, n in enumerate(FRAGS):
            idx = torch.nonzero(cols[b]).flatten()
            if n > 3:
                assert int(idx[-1] - idx[0]) + 1 > n, b                   # linker rows between the fragment rows
        x = data['positions'].reshape(B * N, 3) * data['fragment_mask'].reshape(B * N, 1)
        row = torch.cat([r for r, _ in orc.size_live_edges(x, data['edge_mask'].reshape(-1), B, N)])
        deg = torch.bincount(row, minlength=B * N).reshape(B, N)
        fm = data['fragment_mask'].reshape(B, N) != 0
        for b in range(B):
            got = {}
            for v in deg[b][fm[b]].tolist():
                got[v] = got.get(v, 0) + 1
            assert got == degs[b], (name, b, got, degs[b])
            assert not deg[b][~fm[b]].any()
        isolated = sum(int(d.get(1, 0)) for d in degs)
        assert isolated > 50


def test_tail_and_pocket_batches_have_the_designed_shapes():
    for name, tail in (("tail1", 1), ("tail31", 31)):
        data, _ = batch(name)
        B, N = data['positions'].shape[:2]
        assert (B * N) % NODE_TM == tail
    for name, (B, N) in (("pocket_cfg4", (64, 300)), ("pocket_protein", (2, 4000)), ("pocket_6144", (1, PLAN_MAX_N))):
        data, _ = batch(name)
        assert tuple(data['positions'].shape[:2]) == (B, N)
        fo = data['fragment_only_mask'].squeeze(-1)
        pk = data['pocket_mask'].squeeze(-1)
        assert (data['one_hot'][..., -1] * fo == 0).all() and (data['one_hot'][..., -1] * pk).sum() > 0
        # with_pocket: the pocket rows sit at the origin, each an edge of every other pocket atom and the near fragments
        n_pk = pk.sum(1)
        em = data['edge_mask'].view(B, N, N) != 0
        live_cols = em.any(1).sum(1)
        assert torch.equal(live_cols, (fo + pk).sum(1).long())
        assert int(n_pk.max()) > 128 * (2 if N == 300 else 30)


def test_rounding_pairs_straddle_6_in_the_two_orders():
    below, above = rounding_pairs()
    assert len(below) == len(above) == 6
    for d in below:
        assert torch_radial(d) < 6 and all(r >= 6 for r in fma_radials(d))
    for d in above:
        assert torch_radial(d) >= 6 and all(r < 6 for r in fma_radials(d))
    # torch itself, on the CPU, rounds as torch_radial says, and so does the oracle's edge predicate
    x = torch.tensor(below + above, dtype=torch.float32)
    assert ((x.pow(2).sum(1) < 6).tolist()) == [True] * 6 + [False] * 6
    data, _ = batch("rounding")
    B, N = data['positions'].shape[:2]
    x = data['positions'].reshape(B * N, 3) * data['fragment_mask'].reshape(B * N, 1)
    edges = torch.cat([torch.stack(e) for e in orc.size_live_edges(x, data['edge_mask'].reshape(-1), B, N)], 1)
    pairs = {(int(i) % N, int(j) % N, int(i) // N) for i, j in edges.t().tolist() if i % N != j % N}
    assert pairs == {(a, b, m) for m in range(6) for a, b in ((0, 1), (1, 0))}


def test_one_rounding_edge_moves_the_logits_far_past_the_bound():
    """Each pair's edge, had it been taken on the other side of 6, changes its molecule's fp64 logits by more than 100 times
    the TAU * S_b floor: a kernel that rounds the radial differently fails the GPU test."""
    data, _ = batch("rounding")
    m = model("zinc")
    want = oracle_logits(m, data, False, torch.float64, "cpu")
    moved = dict(data, positions=data['positions'].clone())
    B = want.shape[0]
    for b in range(B):                                   # below: push out to radial 6.05; above: pull in to 5.95
        s = (6.05 if b < B // 2 else 5.95) / 6.0
        moved['positions'][b, 1] *= s ** 0.5
    other = oracle_logits(m, moved, False, torch.float64, "cpu")
    diff = (other - want).abs().amax(1)
    assert (diff > 100 * TAU * want.abs().amax(1)).all(), diff


def test_oracle_fp64_agrees_with_its_fp32_self_and_keeps_the_edge_set():
    for bname, mname in (("fc8", "zinc_bn"), ("rounding", "zinc")):
        data, m = batch(bname)[0], model(mname)
        r64 = oracle_logits(m, data, False, torch.float64, "cpu")
        r32 = oracle_logits(m, data, False, torch.float32, "cpu")
        assert r64.dtype == torch.float64
        assert ((r32 - r64).abs().amax(1) <= 1e-4 * r64.abs().amax(1).clamp(min=1)).all()
    data, m = batch("fc8")[0], model("zinc")
    r64 = oracle_logits(m, data, False, torch.float64, "cpu")
    assert torch.equal(r64[FRAGS.index(0)], m.gnn.embedding_out.bias.detach().double())   # no fragment: the bias


def test_the_draw_band_holds_every_disagreement_and_is_tight_on_peaked_rows():
    """draw_bounds against brute force: rows perturbed by errors within +-eps per logit draw differently only inside the band
    of width 2 eps; and on peaked rows of large logits the band excludes almost nothing, while a flat (e^w - 1) * S band
    would exclude every u."""
    from test_seeded_linker_sizes import oracle_index
    rng = np.random.default_rng(17)
    n, inside, differ = 0, 0, 0
    for scale, C, eps in ((1.0, 10, 1e-3), (5.0, 33, 1e-2), (300.0, 10, 0.5), (1e4, 64, 2.0)):
        l = (scale * rng.standard_normal((200, C))).astype(np.float32)
        e = rng.uniform(-eps, eps, l.shape)
        l2 = (l.astype(np.float64) + e).astype(np.float32)
        w = 2 * (eps + np.abs(l2.astype(np.float64) - (l.astype(np.float64) + e)).max(1))
        for k in range(10):
            u = rng.random(l.shape[0])
            near = draw_bounds(l, w, u)
            for r in range(l.shape[0]):
                a, b = oracle_index(l[r], u[r])[0], oracle_index(l2[r], u[r])[0]
                differ += a != b
                assert a == b or near[r], (scale, C, eps, r)
            inside += int(near.sum())
            n += l.shape[0]
    assert differ > 0 and inside <= 0.05 * n, (differ, inside, n)
    peaked = np.array([[0.0, 47.0, 1e4 - 47, 1e4]], dtype=np.float32).repeat(1000, 0)
    u = rng.random(1000)
    assert not draw_bounds(peaked, np.full(1000, 1.0), u).any()


def test_creation_refuses_65_classes_and_33_input_features():
    from difflinker_b200 import _native
    for F, C in ((8, 65), (33, 10)):
        m = SizeClassifier(in_node_nf=F, out_node_nf=C, n_layers=1)
        with pytest.raises(_native.NativeError, match="unsupported shape"):
            m.gnn.engine(0)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_logits_match_fp64_per_molecule_and_draw_the_oracle_size(case):
    bname, mname, pocket = CASES[case]
    data, m = batch(bname)[0], model(mname)
    ref64, ref32 = references(case)
    got = gpu_logits(m, data, pocket)
    # The whole-protein shapes hold one and two molecules whose pocket rows sum 4000 - 6000 messages: there the oracle's own
    # fp32 error is about 3e-5 of S_b, and so is the kernel's; they are held to the drift bound alone.
    bound = check_molecules(case, got, ref64, ref32, half_within_tau=B_OF[bname] > 2)
    # the seeded draw on the GPU's logits against the oracle's on ref64 rounded to fp32
    from test_seeded_linker_sizes import M64, oracle_sizes, oracle_uniform
    B = got.shape[0]
    K = -(-MIN_PAIRS // B)
    seeds = [int(s) for s in np.random.default_rng(len(case)).integers(0, 1 << 62, B * K, dtype=np.int64)]
    rows = torch.arange(B).repeat_interleave(K)
    table = list(m.linker_id2size)
    drawn = draw_sizes(got.float()[rows].to(dev()), table, seeds).cpu().tolist()
    ref = ref64.float()[rows].numpy()
    want = oracle_sizes(ref, table, seeds)
    u = np.array([oracle_uniform(s & M64) for s in seeds])
    near = draw_bounds(ref, draw_width(bound, ref64)[rows.numpy()], u)
    bad = [(int(rows[k]), seeds[k]) for k in range(B * K) if drawn[k] != want[k] and not near[k]]
    WORST[case][3] = f"{int(near.sum())}/{B * K}"
    assert not bad, f"{case}: draws differ outside the exclusion band: {bad[:5]}"
    assert near.sum() <= 0.01 * B * K, f"{case}: {int(near.sum())} of {B * K} draws excluded"


@pytest.mark.gpu
def test_n_above_the_plan_limit_is_refused_by_name():
    from difflinker_b200 import _native
    m = model("zinc").to(dev())
    B, N = 1, PLAN_MAX_N + 1
    d = dev()
    with pytest.raises(_native.NativeError, match=f"N = {N} exceeds the work plan's limit of {PLAN_MAX_N}"):
        m.gnn.logits(torch.zeros((B, N, 8), device=d), torch.zeros((B, N, 3), device=d), torch.ones((B, N), device=d),
                     None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fc", "pocket_4A"])
def test_sample_chain_draws_the_oracle_size_from_the_input_batch(case):
    """DDPM.sample_chain(linker_sizes=<trained-like SizeClassifier>): last_sizes is the oracle's draw from the fp64 logits of
    the input batch, with_pocket and adjust_shape on the pocket model (ddpm.size_distribution's wiring)."""
    from test_seeded_linker_sizes import M64, SEEDS, model_and_data, oracle_sizes, oracle_uniform
    ddpm, data = model_and_data(case, "simt")
    pocket = case.startswith("pocket")
    F = data['one_hot'].shape[-1]
    table = [0, 1, 2, 3, 4, 6]
    torch.manual_seed(12)
    nn = SizeClassifier(in_node_nf=F - 1 if pocket else F, out_node_nf=len(table), linker_id2size=table,
                        linker_size2id={s: i for i, s in enumerate(table)})
    synthetic.init_size_gnn_like_trained(nn, 12)
    nn = nn.eval().to(dev())
    with torch.no_grad():                                      # centre the logits over the batch, so the draw is the molecule's
        nn.gnn.embedding_out.bias.sub_(oracle_logits(nn, data, pocket, torch.float64, dev()).mean(0).float().to(dev()))
    if pocket:                                                             # adjust_shape drops a column that is zero here
        fo = data['fragment_only_mask'].squeeze(-1)
        assert (data['one_hot'][..., -1] * fo == 0).all()
    ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, keep_frames=2)
    got = ddpm.edm.last_sizes.tolist()
    ref64 = oracle_logits(nn, data, pocket, torch.float64, dev())
    ref32 = oracle_logits(nn, data, pocket, torch.float32, dev())
    eps = torch.maximum(C_DRIFT * (ref32 - ref64).abs().amax(1), TAU * ref64.abs().amax(1))
    want = oracle_sizes(ref64.float().numpy(), table, SEEDS)
    u = np.array([oracle_uniform(s & M64) for s in SEEDS])
    near = draw_bounds(ref64.float().numpy(), draw_width(eps, ref64), u)
    assert all(g == w or n for g, w, n in zip(got, want, near)), (got, want, near)
    assert not near.any() and len(set(want)) > 1, (want, near)
