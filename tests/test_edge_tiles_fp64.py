"""Edge-tile layouts and EGNN option instantiations against an fp64 oracle, row by row.

Most of what can go wrong in the edge kernels without crashing is tile bookkeeping: which rows share a tile, where a row
starts, how a row's sum is carried across 32-edge runs and 128-column chunks, and what divisor 'mean' uses. The batches
here are built so that every layout is hit on purpose rather than by chance:

- FC graphs: molecules of 1 .. 257 live atoms padded to N = 257, and a batch padded to exactly N = 128 (nc = N), with
  linker counts 0, 1, 2, n - 1, n. That gives tiles of 1 .. 32 whole rows, rows of 128 and 256 columns, and rows with a
  one-column last chunk, for the GCL tiles and for the coordinate-update (COORD) tiles over the linker rows.
- Cut-off graphs: clusters 25 A apart whose members lie within a 1.4 A ball, so every degree is exact and no distance is
  near a cut-off. '4A' has rows of degree 0, 1, 3, 127, 128, 129, 256 and 257, enough light rows to fill several 28-row
  tiles, and linker atoms in a singleton, a pair and the heavy clusters. 'FC-4A' and 'FC-10A-4A' have heavy ligand and
  pocket rows and isolated pocket atoms.
- Every combination of tanh, mean and sin_embedding, on both edge paths (SIMT and tensor-core).
- Pairs at exactly the cut-offs (squared distances 16 / 17 and 100 / 101 with integer coordinates, exact in fp32 and fp64),
  and SizeGNN's strict `radial < 6` (squared distances 5 / 6).
- Node-kernel tiles of 8, a middle size and 128 nodes with a one-node last tile, and 8 exactly.

The reference is the in-repo oracle run in float64 (on the GPU: it is not code under test, and at these shapes the CPU
takes minutes). Each live row i of molecule b is checked on its own, separately on the coordinate columns and the feature
columns: err_i = max|got - ref64| must satisfy err_i <= max(C_DRIFT * drift_i, TAU * S_b), where drift_i = max|ref32 - ref64|
is the same oracle's own float32 error on that row (how well conditioned the row is) and S_b the largest |ref64| over the
molecule's live rows (fp64_rows.check_rows). One layer with one GCL keeps a wrong aggregate in row i from reaching any
other row, so a failure names the row, and through the molecule's size and linker count, the tile shape. Padded rows, and
the coordinate rows outside the linker mask, must be exactly 0.

Every input here keeps the tensor-core kernels' operand scale factors at 1. The fp16 range-rescale paths (the node
kernel's per-tile scales and the edge kernel's per-edge scale and descale) are driven on purpose, and checked with the same
per-row rule, in test_range_rescale_fp64.py. Batch-mate effects of tile-level scaling are out of scope for both files.
"""
import collections
import ctypes as C
import functools
import itertools

import pytest
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
from fp64_rows import (build_model, check_rows, dev, make_case, node_tail_shape, node_tile, oracle_forward, pocket_item,
                       run_dyn)
from oracle import difflinker_oracle as orc

IMPLS = ["simt", "auto"]
OPTIONS = list(itertools.product((False, True), repeat=3))      # (tanh, mean, sin_embedding)
F_FC, F_PK = 8, 9
FC_SIZES = (1, 2, 3, 4, 5, 16, 17, 31, 32, 33, 42, 43, 63, 64, 65, 127, 128, 129, 255, 256, 257)
FC_SIZES_128 = (128, 127, 65, 64, 33, 2, 1)

WORST = {}          # test label -> (worst err / bound, C needed beside TAU, worst err / S_b, fraction within TAU)


def opt_id(o):
    return "-".join(n for n, on in zip(("tanh", "mean", "sin"), o) if on) or "default"


# ------------------------------------------------------------------------------------------------------------ batches
def _fc_batch(sizes, seed):
    g = torch.Generator().manual_seed(seed)
    items = []
    for k, n in enumerate(sizes):
        lk = min((0, 1, 2, n - 1, n)[k % 5], n)
        lm = torch.zeros(n)
        lm[n - lk:] = 1.0
        types = torch.randint(0, F_FC, (n,), generator=g)
        items.append({'positions': 1.5 * torch.randn((n, 3), generator=g),
                      'one_hot': torch.nn.functional.one_hot(types, F_FC).float(),
                      'fragment_mask': 1.0 - lm, 'linker_mask': lm})
    return collate(items)


@functools.lru_cache(maxsize=None)
def fc_case(name):
    sizes, seed = {"ragged257": (FC_SIZES, 31), "full128": (FC_SIZES_128, 32)}[name]
    return make_case(_fc_batch(sizes, seed), F_FC, 'FC', seed)


def _centres(k):
    """k cluster centres 25 A apart on a cubic grid, nearest to the origin first."""
    ax = torch.arange(-3, 4, dtype=torch.float64) * 25.0
    grid = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), dim=-1).reshape(-1, 3)
    return grid[torch.argsort(grid.norm(dim=1), stable=True)][:k]


def _ball(g, m, centre, radius=1.4):
    """m points in a ball of the given radius: every pair is closer than 2 * radius."""
    v = torch.randn((m, 3), generator=g, dtype=torch.float64)
    v = v / v.norm(dim=1, keepdim=True)
    r = radius * 0.999 * torch.rand((m, 1), generator=g, dtype=torch.float64) ** (1 / 3)
    return centre + v * r


# '4A' clusters per molecule: (atoms, linker atoms among them). A cluster of m atoms gives m rows of degree m - 1.
CLUSTERS_4A = (
    [(258, 1), (130, 1), (1, 1), (257, 1), (129, 1), (128, 0), (4, 0)] + [(1, 0)] * 10,
    [(1, 1), (2, 1), (4, 0)] + [(1, 0)] * 39 + [(2, 0)] * 29,
)


def _cluster_molecule(g, clusters):
    centres = _centres(len(clusters))
    pos, role, deg = [], [], collections.Counter()
    for (m, n_link), c in zip(clusters, centres):
        pos.append(_ball(g, m, c))
        role += ['l'] * n_link + ['f' if (len(role) + k) % 3 == 0 else 'p' for k in range(m - n_link)]
        deg[m - 1] += m
    return torch.cat(pos), role, deg


def _ligand_pocket_molecule(g, n_pocket, n_isolated, pocket_offset, far_ligand):
    """10 ligand atoms (6 fragment-only, 4 linker) in a 1.4 A ball at the origin, a pocket cluster of n_pocket atoms in a
    1.4 A ball `pocket_offset` A away (within the cross cut-off of every ligand atom), optionally a fragment-only atom
    25 A away (joined to the ligand by the FC ligand-ligand rule only) and n_isolated pocket atoms outside every cut-off."""
    centres = _centres(2 + n_isolated + 2)[2:]                     # grid points >= 25 A from the origin
    parts = [_ball(g, 10, torch.zeros(3, dtype=torch.float64)),
             _ball(g, n_pocket, torch.tensor([pocket_offset, 0.0, 0.0], dtype=torch.float64))]
    role = ['f'] * 6 + ['l'] * 4 + ['p'] * n_pocket
    n_lig = 10
    deg = collections.Counter()
    if far_ligand:
        parts.append(centres[-1:])
        role += ['f']
        n_lig = 11
        deg[n_lig - 1] += 1                                        # the far atom: the other ligand atoms only
    parts.append(centres[:n_isolated])
    role += ['p'] * n_isolated
    deg[(n_lig - 1) + n_pocket] += 10
    deg[(n_pocket - 1) + 10] += n_pocket
    deg[0] += n_isolated
    return torch.cat(parts), role, deg


@functools.lru_cache(maxsize=None)
def cutoff_case(graph_type):
    g = torch.Generator().manual_seed(41)
    if graph_type == '4A':
        mols = [_cluster_molecule(g, cl) for cl in CLUSTERS_4A]
    else:
        off = 0.0 if graph_type == 'FC-4A' else 6.0                # FC-10A-4A: cross distances 3.2 .. 8.8 A
        mols = [_ligand_pocket_molecule(g, 150, 8, off, False), _ligand_pocket_molecule(g, 100, 3, off, True)]
    batch = collate([pocket_item(g, pos, role, F_PK) for pos, role, _ in mols])
    return make_case(batch, F_PK, graph_type, 43, degrees=[deg for _, _, deg in mols])


# Exact cut-off boundaries: integer coordinates, so every squared distance is an exact integer in fp32 and fp64.
BOUNDARY_ATOMS = [           # (position, role)
    ((0, 0, 0), 'f'),        # 0  l1
    ((0, 0, 1), 'l'),        # 1  l2 (linker)
    ((10, 0, 0), 'p'),       # 2  |l1|^2 = 100, |l2|^2 = 101
    ((-10, 0, -1), 'p'),     # 3  |l1|^2 = 101, |l2|^2 = 104
    ((4, 0, 0), 'p'),        # 4  |l1|^2 = 16,  |l2|^2 = 17
    ((0, -4, -1), 'p'),      # 5  |l1|^2 = 17,  |l2|^2 = 20
    ((0, 30, 0), 'p'),       # 6  pocket pair at 16
    ((4, 30, 0), 'p'),       # 7
    ((0, -30, 0), 'p'),      # 8  pocket pair at 17
    ((4, -30, 1), 'p'),      # 9
]
BOUNDARY_EDGES = {           # undirected, per graph type
    '4A': {(0, 1), (0, 4), (6, 7)},
    'FC-4A': {(0, 1), (0, 4), (6, 7)},
    'FC-10A-4A': {(0, 1), (0, 2), (0, 4), (1, 4), (0, 5), (1, 5), (6, 7)},
}


@functools.lru_cache(maxsize=None)
def boundary_case(graph_type):
    g = torch.Generator().manual_seed(51)
    pos = torch.tensor([p for p, _ in BOUNDARY_ATOMS], dtype=torch.float64)
    role = [r for _, r in BOUNDARY_ATOMS]
    # a second, padded molecule: the same atoms without the far pocket pairs, shifted by an integer vector
    batch = collate([pocket_item(g, pos, role, F_PK), pocket_item(g, pos[:6] + torch.tensor([3.0, -2.0, 5.0], dtype=torch.float64),
                                                              role[:6], F_PK)])
    return make_case(batch, F_PK, graph_type, 53)


def oracle_edges(case):
    """The oracle's cut-off edge list (egnn.py:554-596) of a case, as (B*N,) row / column indices, computed on the CPU."""
    B, N = case['z'].shape[:2]
    nm = case['atom_mask'].reshape(B * N, 1).double()
    x = case['z'].reshape(B * N, -1)[:, :3].double() * nm
    ctx = case['context'].reshape(B * N, -1)
    return orc.pocket_edge_index(x, nm, case['edge_mask'].reshape(-1), case['linker_mask'].reshape(B * N, 1), ctx[:, -2],
                                 ctx[:, -1], case['graph_type'])


# -------------------------------------------------------------------------------------------------- models and oracle
_REFS = {}


def references(key, dyn, cfg, case):
    """(ref64, ref32) of a case and model, computed once per key: the weights do not depend on the edge implementation."""
    if key not in _REFS:
        sd = dyn.state_dict()
        _REFS[key] = (oracle_forward(sd, cfg, case, torch.float64, dev()), oracle_forward(sd, cfg, case, torch.float32, dev()))
    return _REFS[key]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst per-row ratios (err / bound, C needed beside TAU, err / S_b, fraction of rows within TAU * S_b):")
        for k, (w, c, r, f) in WORST.items():
            print(f"  {k:48s} {w:9.3e} {c:9.3e} {r:9.3e} {f:6.3f}")


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_fc_batches_have_the_designed_rows():
    for name, sizes in (("ragged257", FC_SIZES), ("full128", FC_SIZES_128)):
        c = fc_case(name)
        B, N = c['z'].shape[:2]
        assert N == max(sizes) and B == len(sizes)
        live = (c['atom_mask'].reshape(B, N) != 0).sum(1).tolist()
        links = (c['linker_mask'].reshape(B, N) != 0).sum(1).tolist()
        assert live == list(sizes)
        assert links == [min((0, 1, 2, n - 1, n)[k % 5], n) for k, n in enumerate(sizes)]


@pytest.mark.parametrize("graph_type", ["4A", "FC-4A", "FC-10A-4A"])
def test_cutoff_batches_have_the_designed_degrees(graph_type):
    """The generator's clusters give exactly the designed degree histogram in the oracle's edge list, so the tile shapes
    the GPU tests are written for (28-row light tiles, heavy rows of 129 / 256 / 257 neighbours, isolated rows) exist."""
    c = cutoff_case(graph_type)
    B, N = c['z'].shape[:2]
    assert N <= 1000
    row, _ = oracle_edges(c)
    deg = torch.bincount(row, minlength=B * N).reshape(B, N)
    live = c['atom_mask'].reshape(B, N) != 0
    for b in range(B):
        got = collections.Counter(deg[b][live[b]].tolist())
        assert got == c['degrees'][b], (b, sorted(got.items()), sorted(c['degrees'][b].items()))
    light = sum((deg[live] <= 4).tolist())
    if graph_type == '4A':
        assert light == 4 + 11 + 4 + 40 + 60
        lk = c['linker_mask'].reshape(B, N) != 0
        assert sorted(deg[lk].tolist()) == [0, 0, 1, 128, 129, 256, 257]
    else:
        assert light == 8 + 3


@pytest.mark.parametrize("graph_type", ["4A", "FC-4A", "FC-10A-4A"])
def test_boundary_edges_are_the_designed_ones(graph_type):
    """Pairs at exactly 4 A and 10 A are edges (<=), pairs at sqrt(17) and sqrt(101) A are not."""
    c = boundary_case(graph_type)
    B, N = c['z'].shape[:2]
    row, col = oracle_edges(c)
    want = BOUNDARY_EDGES[graph_type]
    for b, n in ((0, 10), (1, 6)):
        got = {(int(i) - b * N, int(j) - b * N) for i, j in zip(row.tolist(), col.tolist()) if b * N <= i < (b + 1) * N}
        mine = {(i, j) for i, j in want if i < n and j < n}
        assert got == mine | {(j, i) for i, j in mine}, (b, sorted(got))


def _size_gnn_batch():
    """Fragment atoms at squared distance 5 (an edge) and 6 (not an edge, radial < 6 is strict), linker atoms, padding."""
    g = torch.Generator().manual_seed(61)
    mols = [[((0, 0, 0), 1), ((2, 1, 0), 1), ((10, 0, 0), 1), ((12, 1, 1), 1), ((0, 10, 0), 0), ((1, 10, 2), 0)],
            [((0, 0, 0), 1), ((1, 2, 0), 1), ((0, 0, 2), 0)]]
    items = []
    for atoms in mols:
        n = len(atoms)
        fm = torch.tensor([float(f) for _, f in atoms])
        types = torch.randint(0, F_FC, (n,), generator=g)
        items.append({'positions': torch.tensor([p for p, _ in atoms], dtype=torch.float32),
                      'one_hot': torch.nn.functional.one_hot(types, F_FC).float(), 'fragment_mask': fm,
                      'linker_mask': 1.0 - fm})
    from difflinker_b200 import linker_size
    return linker_size.collate_with_fragment_edges(items)


def _size_model():
    from difflinker_b200 import linker_size
    torch.manual_seed(62)
    model = linker_size.SizeClassifier(in_node_nf=F_FC, hidden_nf=128, out_node_nf=10, n_layers=3, normalization=None)
    synthetic.init_size_gnn_like_trained(model, 62)
    return model.eval()


def test_size_gnn_boundary_edges_are_the_designed_ones():
    """SizeGNN's edges (linker_size_lightning.py:107-108): live fragment pairs with squared distance < 6, self loops included.
    The pair at 5 is one and the pair at 6 is not; moving the second pair to 5 changes the logits far beyond the GPU test's tolerance."""
    data = _size_gnn_batch()
    B, N = data['positions'].shape[:2]
    fm = data['fragment_mask'].reshape(B * N, 1).float()
    x = data['positions'].reshape(B * N, 3).float() * fm
    row, col = orc.fc_edge_index(N, B)
    radial, _ = orc.pair_geometry(x, row, col)
    keep = (data['edge_mask'].reshape(-1, 1).bool() & (radial < 6)).view(-1)
    got = {(int(i), int(j)) for i, j in zip(row[keep].tolist(), col[keep].tolist())}
    loops = {(i, i) for i in (0, 1, 2, 3, N, N + 1)}         # the edge mask's -2 diagonal keeps fragment self loops
    assert got == {(0, 1), (1, 0), (N, N + 1), (N + 1, N)} | loops
    model = _size_model()
    with torch.no_grad():
        want = orc.size_classifier_forward(model.state_dict(), data, F_FC, 3)
        moved = dict(data, positions=data['positions'].clone())
        moved['positions'][0, 3] = torch.tensor([12.0, 1.0, 0.0])
        other = orc.size_classifier_forward(model.state_dict(), moved, F_FC, 3)
    assert (other - want).abs().max().item() > 100 * 1e-5 * want.abs().max().item()


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("opts", OPTIONS, ids=opt_id)
@pytest.mark.parametrize("batch", ["ragged257", "full128"])
def test_fc_tiles_match_fp64_per_row(batch, opts, impl):
    """Every FC tile layout of both edge paths and every option instantiation; with 'mean' the divisor is the padded N."""
    case = fc_case(batch)
    dyn, cfg = build_model('FC', F_FC, opts, impl, 71)
    ref64, ref32 = references(("fc", batch, opts), dyn, cfg, case)
    check_rows(f"fc {batch} {opt_id(opts)} {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("opts", OPTIONS, ids=opt_id)
@pytest.mark.parametrize("graph_type", ["4A", "FC-4A", "FC-10A-4A"])
def test_cutoff_tiles_match_fp64_per_row(graph_type, opts, impl):
    """Packed light tiles up to 28 rows, chunked heavy rows (degree 129 / 256 / 257, also as COORD rows) and isolated rows;
    with 'mean' the divisor is the row's degree (1 for an isolated row)."""
    case = cutoff_case(graph_type)
    dyn, cfg = build_model(graph_type, F_PK, opts, impl, 72)
    ref64, ref32 = references(("cut", graph_type, opts), dyn, cfg, case)
    check_rows(f"cut {graph_type} {opt_id(opts)} {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST)
    if impl == "auto":
        from difflinker_b200 import _native
        stats = (C.c_int64 * 4)()
        _native.check(_native.load_library().dl_cut_graph_stats(dyn.engine(0), stats), "dl_cut_graph_stats")
        B, N = case['z'].shape[:2]
        row, _ = oracle_edges(case)
        live = (case['atom_mask'].reshape(-1) != 0)
        isolated = int(((torch.bincount(row, minlength=B * N) == 0) & live).sum())
        assert stats[2] == row.numel() + isolated
        assert stats[1] > stats[0], "no row with more than 128 neighbours"


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("opts", [(False, False, False), (True, True, True)], ids=opt_id)
@pytest.mark.parametrize("graph_type", ["4A", "FC-4A", "FC-10A-4A"])
def test_boundary_edges_match_fp64_per_row(graph_type, opts, impl):
    """Pairs at exactly the cut-off are edges in the kernels too: one missing or extra edge moves its row far past the bound."""
    case = boundary_case(graph_type)
    dyn, cfg = build_model(graph_type, F_PK, opts, impl, 73)
    ref64, ref32 = references(("edge", graph_type, opts), dyn, cfg, case)
    check_rows(f"boundary {graph_type} {opt_id(opts)} {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST)
    if impl == "auto":
        from difflinker_b200 import _native
        stats = (C.c_int64 * 4)()
        _native.check(_native.load_library().dl_cut_graph_stats(dyn.engine(0), stats), "dl_cut_graph_stats")
        B, N = case['z'].shape[:2]
        row, _ = oracle_edges(case)
        live = (case['atom_mask'].reshape(-1) != 0)
        isolated = int(((torch.bincount(row, minlength=B * N) == 0) & live).sum())
        assert stats[2] == row.numel() + isolated


@pytest.mark.gpu
def test_size_gnn_boundary_edges_match_the_oracle():
    """SizeGNN on the GPU drops the fragment pair at squared distance 6 and keeps the one at 5 (fp32 oracle, 1e-5)."""
    data = _size_gnn_batch()
    model = _size_model()
    with torch.no_grad():
        want = orc.size_classifier_forward(model.state_dict(), data, F_FC, 3)
    d = dev()
    got, _ = model.forward({k: (v.to(d) if torch.is_tensor(v) else v) for k, v in data.items()}, return_loss=False)
    got = got.cpu()
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()


def test_node_tail_shapes_give_the_requested_tiles():
    for sms in (132, 114, 78):
        for kind in ("tile8_tail1", "tile8_exact", "tile64_tail1", "tile128_tail1"):
            B, N = node_tail_shape(kind, sms)
            tile = int(kind.split("_")[0][4:])
            assert node_tile(B * N, sms) == tile
            assert (B * N) % tile == (0 if kind.endswith("exact") else 1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["tile8_tail1", "tile8_exact", "tile64_tail1", "tile128_tail1"])
def test_node_tile_tails_match_fp64_per_row(kind):
    """Two blocks of two GCLs, so the projection-only launch, the two-projection launch at the block boundary and the
    one-projection launch all run, at node counts that leave a one-node last tile (or none)."""
    B, N = node_tail_shape(kind, torch.cuda.get_device_properties(0).multi_processor_count)
    spec = synthetic.WorkloadSpec(f"tail_{kind}", B=B, N=N, n_min=max(3, N // 2), l_min=1, l_max=8, F=F_FC, L=2, T=10,
                                  seed=81)
    case = make_case(collate(synthetic.make_items(spec)), F_FC, 'FC', 82)
    dyn, cfg = build_model('FC', F_FC, (False, False, False), "auto", 74, n_layers=2, inv_sublayers=2)
    ref64, ref32 = references(("node", kind), dyn, cfg, case)
    check_rows(f"node {kind} B={B} N={N}", run_dyn(dyn, case), ref64, ref32, case, WORST)
