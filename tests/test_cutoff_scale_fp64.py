"""The pocket denoiser against an fp64 oracle at whole-protein sizes, row by row.

test_edge_tiles_fp64.py holds every tile layout of the edge kernels to fp64 on batches of N <= 1000, where no row has more
than 257 neighbours. What only matters at scale is checked here: k_nbr staging up to 4000 rows in shared memory and
compacting rows of up to 3969 neighbours, cut_pack_rows packing thousands of rows, heavy records whose row sum is carried
across up to 32 column chunks (GCL and COORD tiles), record fields at row indices above 2048, the 'mean' divisor counted
over thousands of edges, and the SIMT kernel's cut-off tiles over 48 column chunks at N = 6144.

Batches (seeded, checked on the CPU: designed degrees, no pair within DELTA of a cut-off, the same edge set in fp32 and
fp64):

- "protein": the layout of the N = 4000 sampler cases, B = 2, N = 4000, molecules of (30 fragment, 3960 pocket, 10 linker)
  and (25, 2900, 12) atoms. Pocket atoms on a jittered cubic lattice at protein heavy-atom density (0.05 A^-3) around a
  compact ligand, about 40 A from the origin so fp32 coordinates carry real rounding: pocket rows have about 13 neighbours
  under 4 A, ligand rows about 200 under FC-10A-4A.
- "dense": 1.2 A-wide clusters whose surfaces are at least 4.2 A apart, so every degree is exact. Around each ligand (in a
  0.8 A ball) one cluster overlaps the ligand and 20 sit on a sphere of radius 8.5 A, all within 9.9 A of every ligand
  atom. FC-10A-4A: ligand (and linker) rows of degree 3969 = 31 * 128 + 1 in molecule 0 and 3840 = 30 * 128 in molecule 1,
  pocket rows of 215 .. 257, 30 and 53 isolated pocket rows (light tiles of 28 degree-0 rows; 53 also tells 28-row from
  24-row tiles apart). FC-4A: ligand rows of 257 and 256 (the sphere is beyond 4 A), the rest as above.
- "cluster4A": one cluster of 1500 atoms (degree 1499, 12 chunks), clusters of 129, 128 and 1, padded to N = 4000, linker
  atoms in the big cluster and in the singleton.
- "simt6144" / "simt4001": one protein-like molecule at N = 6144 (the work plan's limit) and at N = 4001, the first size
  the tensor-core path refuses; SIMT only.

Criterion: fp64_rows.check_rows (one layer, one GCL unless stated: a wrong row names itself), with at least half the live
rows of every case within TAU * S_b. No case is exempt: rows of thousands of messages carry an oracle fp32 error of the
order of TAU * S_b, but they are a small share of each batch's rows, and even in "cluster4A", where 1500 of 1758 rows have
1499 messages, over 99 % of the rows meet the plain bound (DESIGN.md). A range witness (test_range_rescale_fp64.py) shows
that every case keeps the tensor-core operand scales at 1. The tile-record counts of dl_cut_graph_stats are compared with
a plain restatement of cut_pack_rows, exactly.
"""
import collections
import ctypes as C
import functools
import itertools
import math
import time

import pytest
import torch

from difflinker_b200 import _native
from difflinker_b200.batching import collate
from fp64_rows import build_model, check_rows, dev, make_case, node_tile, oracle_forward, pocket_item, run_dyn
from oracle import difflinker_oracle as orc
from test_range_rescale_fp64 import QUIET, witness

F_PK = 9
DELTA = 1e-3                    # no pair within this distance (A) of 4 A or 10 A
CUT_TN, CUT_MAXR = 128, 28      # kernels_simt.cuh: columns per tile, rows per packed light tile
IMPLS = ["simt", "auto"]
OPTIONS = list(itertools.product((False, True), repeat=3))      # (tanh, mean, sin_embedding)
DEFAULT, TMS = (False, False, False), (True, True, True)
CENTRE = (24.0, -23.0, 22.0)    # about 40 A from the origin

WORST = {}          # test label -> (worst err / bound, C needed beside TAU, worst err / S_b, fraction within TAU)
MEMORY = {}         # reference key -> peak device memory of its oracle runs (bytes)


def opt_id(o):
    return "-".join(n for n, on in zip(("tanh", "mean", "sin"), o) if on) or "default"


# ------------------------------------------------------------------------------------------------------------ batches
def _ball(g, m, centre, radius):
    """m points in a ball of the given radius: every pair is closer than 2 * radius."""
    v = torch.randn((m, 3), generator=g, dtype=torch.float64)
    v = v / v.norm(dim=1, keepdim=True)
    r = radius * 0.999 * torch.rand((m, 1), generator=g, dtype=torch.float64) ** (1 / 3)
    return centre + v * r


def _lattice(spacing, extent):
    ax = torch.arange(-extent, extent + 1, dtype=torch.float64) * spacing
    grid = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), dim=-1).reshape(-1, 3)
    return grid[torch.argsort(grid.norm(dim=1), stable=True)]


def near_cutoff(pos, pocket):
    """Pairs of the fp32-rounded positions within DELTA of a cut-off that applies to them: 4 A for any pair, 10 A for a
    ligand-pocket pair. `pocket`: bool per atom."""
    p = pos.float().double()
    d = torch.cdist(p, p)
    cross = pocket[:, None] != pocket[None, :]
    return ((d - 4).abs() <= DELTA) | (cross & ((d - 10).abs() <= DELTA))


def _clear_band(g, pos, role):
    """Moves atoms by up to 0.01 A (seeded) until no pair lies within DELTA of a cut-off that applies to it."""
    pos = pos.clone()
    pocket = torch.tensor([r == 'p' for r in role])
    for _ in range(100):
        bad = near_cutoff(pos, pocket)
        if not bad.any():
            return pos
        idx = torch.unique(torch.nonzero(torch.triu(bad, 1))[:, 1])
        pos[idx] += 0.01 * (2 * torch.rand((idx.numel(), 3), generator=g, dtype=torch.float64) - 1)
    raise AssertionError("atoms still within DELTA of a cut-off")


def _protein_molecule(g, n_frag, n_pocket, n_link):
    """A compact ligand (jittered 1.5 A lattice) in a cavity of a pocket on a jittered 2.71 A lattice (0.05 A^-3)."""
    n_lig = n_frag + n_link
    lig = _lattice(1.5, 3)[:n_lig] + 0.15 * torch.randn((n_lig, 3), generator=g, dtype=torch.float64)
    grid = _lattice(0.05 ** (-1 / 3), 16)
    grid = grid[torch.cdist(grid, lig).amin(1) > 3.0][:n_pocket]
    pk = grid + 0.25 * torch.randn(grid.shape, generator=g, dtype=torch.float64)
    role = ['f'] * n_frag + ['l'] * n_link + ['p'] * n_pocket
    perm = torch.randperm(len(role), generator=g)
    pos = (torch.cat([lig, pk]) + torch.tensor(CENTRE, dtype=torch.float64))[perm]
    role = [role[k] for k in perm.tolist()]
    return _clear_band(g, pos, role), role


def _sphere_points(k, radius):
    """k points on a sphere (Fibonacci lattice)."""
    i = torch.arange(k, dtype=torch.float64) + 0.5
    phi = torch.acos(1 - 2 * i / k)
    theta = math.pi * (1 + 5 ** 0.5) * i
    return radius * torch.stack([torch.cos(theta) * torch.sin(phi), torch.sin(theta) * torch.sin(phi), torch.cos(phi)], 1)


SHELL, SHELL_R, CLUSTER_R, LIGAND_R = 20, 8.5, 0.6, 0.8


def _dense_molecule(g, n_frag, n_link, n_close, n_shell, n_isolated):
    """Ligand in a LIGAND_R ball, a pocket cluster of n_close atoms overlapping it, n_shell pocket atoms in SHELL clusters on
    a sphere of radius SHELL_R around it, and n_isolated pocket atoms in a row 20 A away and 5.3 A apart. Returns positions,
    roles and the degree histograms {graph type: Counter}."""
    c = torch.tensor(CENTRE, dtype=torch.float64)
    n_lig = n_frag + n_link
    sizes = [n_shell // SHELL + (1 if k < n_shell % SHELL else 0) for k in range(SHELL)]
    parts = [_ball(g, n_lig, c, LIGAND_R), _ball(g, n_close, c, CLUSTER_R)]
    parts += [_ball(g, m, c + p, CLUSTER_R) for m, p in zip(sizes, _sphere_points(SHELL, SHELL_R))]
    parts.append(c + torch.tensor([[20.0 + 5.3 * k, 0.0, 0.0] for k in range(n_isolated)], dtype=torch.float64).reshape(-1, 3))
    role = ['f'] * n_frag + ['l'] * n_link + ['p'] * (n_close + n_shell + n_isolated)
    n_pk = n_close + n_shell
    deg = {}
    for gt in ('FC-10A-4A', 'FC-4A'):
        far = gt == 'FC-10A-4A'                                    # the shell is within the cross cut-off
        deg[gt] = collections.Counter()
        deg[gt][n_lig - 1 + (n_pk if far else n_close)] += n_lig
        deg[gt][n_close - 1 + n_lig] += n_close
        deg[gt][0] += n_isolated
        for m in sizes:
            deg[gt][m - 1 + (n_lig if far else 0)] += m
    perm = torch.randperm(len(role), generator=g)
    return torch.cat(parts)[perm], [role[k] for k in perm.tolist()], deg


# (fragment, linker, close cluster, shell, isolated): FC-10A-4A ligand rows of 3969 and 3840, FC-4A ligand rows of 257, 256
DENSE = [(30, 10, 218, 3712, 30), (25, 12, 220, 3584, 53)]
CLUSTERS_4A = [(1500, 3), (129, 0), (128, 0), (1, 1)]       # (atoms, linker atoms)


def _cluster_molecule(g):
    c = torch.tensor(CENTRE, dtype=torch.float64)
    parts, role, deg = [], [], collections.Counter()
    for k, (m, n_link) in enumerate(CLUSTERS_4A):
        parts.append(_ball(g, m, c + torch.tensor([25.0 * k, 0.0, 0.0], dtype=torch.float64), 1.2))
        role += ['l'] * n_link + ['f' if s % 3 == 0 else 'p' for s in range(m - n_link)]
        deg[m - 1] += m
    return torch.cat(parts), role, {'4A': deg}


def _pad(batch, N):
    """A collated batch padded with empty rows to N (pocket batches: edge_mask is the molecule index of every node)."""
    out = {}
    for k, v in batch.items():
        if k == 'edge_mask':
            B = batch['positions'].shape[0]
            out[k] = torch.arange(B, dtype=torch.int64).repeat_interleave(N).to(v.dtype)
        elif torch.is_tensor(v) and v.dim() >= 2:
            pad = list(v.shape)
            pad[1] = N - v.shape[1]
            out[k] = torch.cat([v, v.new_zeros(pad)], dim=1)
        else:
            out[k] = v
    return out


@functools.lru_cache(maxsize=None)
def batch_of(name):
    """(collated batch, per molecule {graph type: designed degree histogram} or None)."""
    g = torch.Generator().manual_seed({"protein": 201, "dense": 202, "cluster4A": 203, "simt6144": 204, "simt4001": 205}[name])
    if name == "protein":
        mols = [_protein_molecule(g, 30, 3960, 10), _protein_molecule(g, 25, 2900, 12)]
        return collate([pocket_item(g, p, r, F_PK) for p, r in mols]), None
    if name == "dense":
        mols = [_dense_molecule(g, *m) for m in DENSE]
        return _pad(collate([pocket_item(g, p, r, F_PK) for p, r, _ in mols]), 4000), [d for _, _, d in mols]
    if name == "cluster4A":
        p, r, d = _cluster_molecule(g)
        return _pad(collate([pocket_item(g, p, r, F_PK)]), 4000), [d]
    n = 6144 if name == "simt6144" else 4001
    p, r = _protein_molecule(g, 30, n - 40, 10)
    return collate([pocket_item(g, p, r, F_PK)]), None


GRAPHS = {"protein": ("4A", "FC-4A", "FC-10A-4A"), "dense": ("FC-4A", "FC-10A-4A"), "cluster4A": ("4A",),
          "simt6144": ("4A", "FC-10A-4A"), "simt4001": ("FC-10A-4A",)}
BATCH_GRAPHS = [(b, gt) for b, gts in GRAPHS.items() for gt in gts]


@functools.lru_cache(maxsize=None)
def case_of(name, graph_type):
    return make_case(batch_of(name)[0], F_PK, graph_type, 211)


def edge_list(case, dtype=torch.float64, device="cpu"):
    """The oracle's cut-off edge list (egnn.py:554-596) of a case in a dtype on a device, as CPU (B*N,) indices."""
    B, N = case['z'].shape[:2]
    with torch.device(device):
        nm = case['atom_mask'].reshape(B * N, 1).to(device, dtype)
        x = case['z'].reshape(B * N, -1)[:, :3].to(device, dtype) * nm
        ctx = case['context'].reshape(B * N, -1).to(device, dtype)
        r, c = orc.pocket_edge_index(x, nm, case['edge_mask'].reshape(-1).to(device),
                                     case['linker_mask'].reshape(B * N, 1).to(device, dtype), ctx[:, -2], ctx[:, -1],
                                     case['graph_type'])
    return r.cpu(), c.cpu()


@functools.lru_cache(maxsize=None)
def degrees_of(name, graph_type):
    """(B, N) degrees in the oracle's fp64 edge list."""
    case = case_of(name, graph_type)
    B, N = case['z'].shape[:2]
    row, _ = edge_list(case)
    return torch.bincount(row, minlength=B * N).reshape(B, N)


# ---------------------------------------------------------------------------------------------- cut_pack_rows restated
def pack_rows(degrees, maxr=CUT_MAXR):
    """cut_pack_rows (kernels_simt.cuh) for one molecule: `degrees` of its rows in slot order, a degree-0 row counted as one
    padding column. Rows of <= 128 columns go first-fit, by decreasing degree with slot order breaking ties, into 128-column
    bins of at most `maxr` rows; each heavier row is a record of its own. Returns (bins as lists of slots, heavy slots)."""
    d = [max(int(x), 1) for x in degrees]
    light = sorted((s for s in range(len(d)) if d[s] <= CUT_TN), key=lambda s: (-d[s], s))
    bins, rem = [], []
    for s in light:
        for k in range(len(bins)):
            if rem[k] >= d[s] and len(bins[k]) < maxr:
                bins[k].append(s)
                rem[k] -= d[s]
                break
        else:
            bins.append([s])
            rem.append(CUT_TN - d[s])
    return bins, [s for s in range(len(d)) if d[s] > CUT_TN]


def pack_stats(degrees, maxr=CUT_MAXR):
    """(records, tiles, edges including padding columns) of one molecule's rows."""
    d = [max(int(x), 1) for x in degrees]
    bins, heavy = pack_rows(d, maxr)
    return (len(bins) + len(heavy), len(bins) + sum(-(-d[s] // CUT_TN) for s in heavy),
            sum(d[s] for b in bins for s in b) + sum(d[s] for s in heavy))


def expected_graph_stats(case, deg, maxr=CUT_MAXR):
    """dl_cut_graph_stats of a forward on this case: GCL records, GCL tiles, GCL edges, COORD records, over the batch.
    GCL rows are the live rows, COORD rows the live linker rows, each in ascending index (the work plan's slot order)."""
    B, N = case['z'].shape[:2]
    live = case['atom_mask'].reshape(B, N) != 0
    lk = (case['linker_mask'].reshape(B, N) != 0) & live
    out = [0, 0, 0, 0]
    for b in range(B):
        rec, tiles, edges = pack_stats(deg[b][live[b]].tolist(), maxr)
        out[0] += rec; out[1] += tiles; out[2] += edges
        out[3] += pack_stats(deg[b][lk[b]].tolist(), maxr)[0]
    return out


def graph_stats(dyn):
    stats = (C.c_int64 * 4)()
    _native.check(_native.load_library().dl_cut_graph_stats(dyn.engine(0), stats), "dl_cut_graph_stats")
    return list(stats)


# -------------------------------------------------------------------------------------------------- models and oracle
_REFS = {}


def references(key, dyn, cfg, case):
    """(ref64, ref32) of a case and model, once per key. ref64 comes with the range witness, which must show every tensor-core
    operand scale at 1 (bounds <= 2^12, a factor 4 below the rescale threshold) for the node tile of this B * N."""
    if key not in _REFS:
        sd = dyn.state_dict()
        torch.cuda.reset_peak_memory_stats()
        w, ref64 = witness(sd, cfg, case)
        ref32 = oracle_forward(sd, cfg, case, torch.float32, dev())
        MEMORY[key] = torch.cuda.max_memory_allocated()
        B, N = case['z'].shape[:2]
        res = w.outcome(node_tile(B * N, torch.cuda.get_device_properties(0).multi_processor_count))
        over = {k: v for k, v in res.items() if k in ('s1', 's2', 's3', 's1_proj', 'gcl_max', 'coord_max') and v > QUIET}
        assert not over, f"{key}: operand bounds past 2^12 would rescale: {over}"
        _REFS[key] = (ref64, ref32)
    return _REFS[key]


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if WORST:
        print("\nworst per-row ratios (err / bound, C needed beside TAU, err / S_b, fraction of rows within TAU * S_b):")
        for k, (w, c, r, f) in WORST.items():
            print(f"  {k:52s} {w:9.3e} {c:9.3e} {r:9.3e} {f:6.3f}")
    if MEMORY:
        print(f"oracle peak device memory: {max(MEMORY.values()) / 2 ** 30:.2f} GiB; file wall time {time.time() - t0:.0f} s")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_batches_have_the_designed_shapes():
    for name, (B, N) in {"protein": (2, 4000), "dense": (2, 4000), "cluster4A": (1, 4000), "simt6144": (1, 6144),
                         "simt4001": (1, 4001)}.items():
        batch, _ = batch_of(name)
        assert tuple(batch['positions'].shape[:2]) == (B, N), name
    batch, _ = batch_of("protein")
    count = lambda k: batch[k].reshape(2, -1).sum(1).tolist()
    live = batch['atom_mask'].reshape(2, -1).sum(1).tolist()
    assert live == [4000, 2937] and count('linker_mask') == [10, 12] and count('pocket_mask') == [3960, 2900]
    batch, _ = batch_of("dense")
    assert batch['atom_mask'].reshape(2, -1).sum(1).tolist() == [4000, 3894]
    assert bool((batch['atom_mask'].reshape(2, -1)[:, 2048:] != 0).any(1).all())


@pytest.mark.parametrize("name,graph_type", [p for p in BATCH_GRAPHS if p[0] in ("dense", "cluster4A")])
def test_designed_batches_have_the_designed_degrees(name, graph_type):
    """Every degree of the clustered batches is exact: the heavy rows of 3969 / 3840 / 1499 / 257 neighbours, the pocket rows
    of a few hundred and the isolated rows exist as designed."""
    deg = degrees_of(name, graph_type)
    case = case_of(name, graph_type)
    B, N = case['z'].shape[:2]
    live = case['atom_mask'].reshape(B, N) != 0
    designed = batch_of(name)[1]
    for b in range(B):
        got = collections.Counter(deg[b][live[b]].tolist())
        assert got == designed[b][graph_type], (b, sorted(got.items()), sorted(designed[b][graph_type].items()))
    lk = (case['linker_mask'].reshape(B, N) != 0) & live
    if name == "dense" and graph_type == "FC-10A-4A":
        assert sorted(set(deg[0][lk[0]].tolist())) == [3969] and sorted(set(deg[1][lk[1]].tolist())) == [3840]
    if name == "cluster4A":
        assert sorted(deg[lk].tolist()) == [0, 1499, 1499, 1499]


@pytest.mark.parametrize("name,graph_type", [p for p in BATCH_GRAPHS if p[0] not in ("dense", "cluster4A")])
def test_protein_batches_have_protein_like_degrees(name, graph_type):
    """About 13 neighbours per pocket row under 4 A, about 200 per ligand row under FC-10A-4A; no isolated row."""
    deg = degrees_of(name, graph_type)
    batch = batch_of(name)[0]
    B, N = deg.shape
    live = batch['atom_mask'].reshape(B, N) != 0
    pk = (batch['pocket_mask'].reshape(B, N) != 0) & live
    lig = live & ~pk
    assert 10 <= deg[pk].double().mean().item() <= 18
    assert deg[live].min().item() >= 1
    if graph_type == "FC-10A-4A":
        for b in range(B):
            n_lig = int(lig[b].sum())
            assert 150 <= (deg[b][lig[b]].double().mean().item() - (n_lig - 1)) <= 260
    assert deg.sum().item() <= 2_500_000


@pytest.mark.parametrize("name,graph_type", BATCH_GRAPHS)
def test_no_pair_near_a_cutoff(name, graph_type):
    """No pair of a molecule lies within DELTA of 4 A, and no ligand-pocket pair within DELTA of 10 A, measured in fp64 on
    the fp32 positions the kernels get; every case stays within 2.5 M directed edges."""
    case = case_of(name, graph_type)
    batch = batch_of(name)[0]
    B, N = case['z'].shape[:2]
    live = case['atom_mask'].reshape(B, N) != 0
    pocket = batch['pocket_mask'].reshape(B, N) != 0
    for b in range(B):
        assert not near_cutoff(case['z'][b][live[b]][:, :3], pocket[b][live[b]]).any(), (name, b)
    assert degrees_of(name, graph_type).sum().item() <= 2_500_000


@pytest.mark.parametrize("name,graph_type", BATCH_GRAPHS)
def test_fp32_and_fp64_oracles_build_the_same_graph(name, graph_type):
    """The fp32 oracle's edge set is the fp64 one, so check_rows' drift term compares runs over the same graph (on the CPU
    here; the GPU test repeats it where the fp32 oracle runs)."""
    case = case_of(name, graph_type)
    r64, c64 = edge_list(case)
    r32, c32 = edge_list(case, torch.float32)
    assert torch.equal(r64, r32) and torch.equal(c64, c32)


def test_pack_rows_restatement():
    """The restatement on small hand-worked inputs: first-fit decreasing with slot-order ties, the row cap, padding columns
    of degree-0 rows and heavy records."""
    bins, heavy = pack_rows([128, 0, 127, 64, 64, 64, 1])
    assert bins == [[0], [2, 1], [3, 4], [5, 6]] and heavy == []
    assert pack_stats([128, 0, 127, 64, 64, 64, 1]) == (4, 4, 449)
    bins, heavy = pack_rows([0] * 30)
    assert [len(b) for b in bins] == [28, 2] and bins[0] == list(range(28))
    assert pack_stats([0] * 53) == (2, 2, 53)
    assert pack_stats([4] * 60) == (3, 3, 240)                 # 28 rows of 4 columns fill 112 of 128
    assert pack_stats([129, 3969, 3840, 256, 5, 0]) == (5, 2 + 32 + 30 + 2 + 1, 129 + 3969 + 3840 + 256 + 5 + 1)
    bins, heavy = pack_rows([30, 100, 30, 98, 30])
    assert bins == [[1], [3, 0], [2, 4]] and heavy == []


def test_dense_packing_sees_the_row_cap():
    """The dense batch's 53 isolated rows take two 28-row tiles, three at 24 rows: the exact count sees the cap."""
    case = case_of("dense", "FC-10A-4A")
    deg = degrees_of("dense", "FC-10A-4A")
    assert expected_graph_stats(case, deg, 24)[0] == expected_graph_stats(case, deg)[0] + 1


# ---------------------------------------------------------------------------------------------------------------- GPU
def _rows_params():
    out = []
    for name, gt in BATCH_GRAPHS:
        if name.startswith("simt"):
            continue
        for o in (OPTIONS if (name, gt) == ("dense", "FC-10A-4A") else (DEFAULT, TMS)):
            out.append((name, gt, o))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name,graph_type,opts", _rows_params(), ids=lambda v: opt_id(v) if isinstance(v, tuple) else v)
def test_rows_match_fp64(name, graph_type, opts, impl):
    """Every row against fp64; on the tensor-core path also the exact tile-record counts of cut_pack_rows."""
    case = case_of(name, graph_type)
    dyn, cfg = build_model(graph_type, F_PK, opts, impl, 221)
    ref64, ref32 = references((name, graph_type, opts, 1), dyn, cfg, case)
    check_rows(f"{name} {graph_type} {opt_id(opts)} {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST, min_tau_frac=0.5)
    if impl == "auto":
        assert graph_stats(dyn) == expected_graph_stats(case, degrees_of(name, graph_type))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_two_blocks_of_two_gcls_match_fp64(impl):
    """L = 2 blocks of S = 2 GCLs on the protein batch: all three node-launch kinds at 8000 nodes."""
    case = case_of("protein", "FC-10A-4A")
    dyn, cfg = build_model("FC-10A-4A", F_PK, DEFAULT, impl, 222, n_layers=2, inv_sublayers=2)
    ref64, ref32 = references(("protein", "FC-10A-4A", DEFAULT, 2), dyn, cfg, case)
    check_rows(f"protein FC-10A-4A L2 S2 {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST, min_tau_frac=0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("name,graph_type,opts", [("simt6144", "4A", DEFAULT), ("simt6144", "FC-10A-4A", DEFAULT),
                                                  ("simt6144", "FC-10A-4A", TMS), ("simt4001", "FC-10A-4A", DEFAULT)],
                         ids=lambda v: opt_id(v) if isinstance(v, tuple) else v)
def test_simt_limits_match_fp64(name, graph_type, opts):
    """The SIMT path at N = 6144 (48 column chunks per row) and at N = 4001."""
    case = case_of(name, graph_type)
    dyn, cfg = build_model(graph_type, F_PK, opts, "simt", 223)
    ref64, ref32 = references((name, graph_type, opts, 1), dyn, cfg, case)
    check_rows(f"{name} {graph_type} {opt_id(opts)} simt", run_dyn(dyn, case), ref64, ref32, case, WORST, min_tau_frac=0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("name,graph_type", BATCH_GRAPHS)
def test_fp32_oracle_builds_the_fp64_graph_on_the_gpu(name, graph_type):
    case = case_of(name, graph_type)
    r64, c64 = edge_list(case)
    r32, c32 = edge_list(case, torch.float32, dev())
    assert torch.equal(r64, r32) and torch.equal(c64, c32)


def _with_n(case, N):
    """A case cut or padded to N rows per molecule (rows past the live ones only)."""
    B, N0 = case['z'].shape[:2]
    out = dict(case)
    for k in ('z', 'atom_mask', 'linker_mask', 'context'):
        v = case[k]
        if N <= N0:
            out[k] = v[:, :N]
        else:
            pad = list(v.shape)
            pad[1] = N - N0
            out[k] = torch.cat([v, v.new_zeros(pad)], dim=1)
    out['edge_mask'] = torch.arange(B, dtype=torch.int64).repeat_interleave(N).to(case['edge_mask'].dtype)
    return out


def _molecule(case, b):
    out = {k: (v[b:b + 1] if k in ('z', 'atom_mask', 'linker_mask', 'context', 't') else v) for k, v in case.items()}
    N = case['z'].shape[1]
    out['edge_mask'] = torch.zeros(N, dtype=case['edge_mask'].dtype)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["auto", "wgmma"])
def test_tensor_core_path_refuses_n4001(impl):
    """N = 4001 is refused by name, and the same module then runs an N = 4000 forward correctly."""
    case = case_of("protein", "FC-10A-4A")
    dyn, cfg = build_model("FC-10A-4A", F_PK, DEFAULT, impl, 221)
    with pytest.raises(_native.NativeError, match="N = 4001 exceeds the neighbour-list kernel's shared-memory staging"):
        run_dyn(dyn, case_of("simt4001", "FC-10A-4A"))
    ref64, ref32 = references(("protein", "FC-10A-4A", DEFAULT, 1), dyn, cfg, case)
    check_rows(f"protein FC-10A-4A after refusal {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST, min_tau_frac=0.5)


@pytest.mark.gpu
def test_simt_path_refuses_n6145():
    """N = 6145 is refused by the work plan, and the same module then runs an N = 6144 forward correctly."""
    case = case_of("simt6144", "FC-10A-4A")
    dyn, cfg = build_model("FC-10A-4A", F_PK, DEFAULT, "simt", 223)
    with pytest.raises(_native.NativeError, match="N = 6145 exceeds the work plan's limit of 6144 rows per molecule"):
        run_dyn(dyn, _with_n(case, 6145))
    ref64, ref32 = references(("simt6144", "FC-10A-4A", DEFAULT, 1), dyn, cfg, case)
    check_rows("simt6144 FC-10A-4A after refusal simt", run_dyn(dyn, case), ref64, ref32, case, WORST, min_tau_frac=0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", ["protein", "dense"])
def test_molecules_are_independent_bit_for_bit(name, impl):
    """Each molecule's rows are the same bits in the batch, alone at its own N and alone padded to N = 4000; a second run
    of the batch repeats the first (k_nbr's atomicAdd orders the molecules' record ranges, not the results)."""
    case = case_of(name, "FC-10A-4A")
    dyn, _ = build_model("FC-10A-4A", F_PK, TMS, impl, 224)
    full = run_dyn(dyn, case)
    assert torch.equal(full, run_dyn(dyn, case)), "a second run differs"
    B, N = case['z'].shape[:2]
    for b in range(B):
        one = _molecule(case, b)
        n = int((case['atom_mask'].reshape(B, N)[b] != 0).nonzero().max()) + 1
        alone = run_dyn(dyn, _with_n(one, n))
        assert torch.equal(alone[0], full[b, :n]), f"molecule {b} alone at N = {n}"
        padded = run_dyn(dyn, _with_n(one, 4000))
        assert torch.equal(padded[0], full[b]), f"molecule {b} alone at N = 4000"
