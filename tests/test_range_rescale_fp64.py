"""The tensor-core kernels' fp16 range-rescale paths against an fp64 oracle, row by row.

The tensor-core path splits every fp32 operand into fp16 hi + lo, which only works while the operand stays below
F16_TARGET = 2^14. Beyond that the kernels scale the operand by an exact power of two and fold the descale into an
epilogue FMA:

- k_node_tc (kernels_node_tc.cuh), one scale per node tile: s1 from max |[h, agg]| (the operands of G1 are rewritten
  scaled), s2 from the largest pre-SiLU value (epilogue 1's second pass), s3 from max |h'| (epilogue 2 rewrites XA, and the
  projections descale by p_descale / s3). It writes ABmax, the node-tile maximum of |A| and of |B| of each consumer.
- k_edge_tc (kernels_tc.cuh), one scale per edge from the bound ABmax[i] + ABmax[j] + d max|wd| + d0 max|w0| (with
  sin_embedding: + sum_k max|w_k|), all in the log2 domain (x log2 e). The edge's descale w2_descale / sc rides in the
  per-edge table, and a tile-level flag tells the producers to multiply by sc; one row's sum can add edges of different
  scales.

Each case below multiplies weight slices (or the input coordinates) by exact powers of two, so the fp64 oracle runs exactly
the model the kernels run, and it drives one branch on purpose. A range witness (`witness`) recomputes, from the oracle's
own fp64 run, every bound in the kernels' terms: per node tile, per consumer and per edge. Each case asserts its designed
outcome with a factor-4 margin on both sides of 2^14 (a branch that must fire has a bound >= 2^16, one that must not has
a bound <= 2^12), on the CPU for 132, 114 and 78 SMs and on the GPU for the device's own SM count, so a case cannot pass by
not rescaling. The 'simt' edge path is fp32 without scaling and runs every case as the control that it is well posed.

Criterion: fp64_rows.check_rows, as in test_edge_tiles_fp64.py, plus: ref32 is finite, and at least half the live rows of
every case meet the plain TAU * S_b bound, so the drift term cannot carry a case. S_b is per molecule while node-tile
scales are shared, so every batch whose molecules are driven unequally has N a multiple of the node tile.

Models: L = 2 blocks of S = 2 GCLs, so the projection-only node launch (after the embedding), the one-projection launch
and the two-projection launch (a block's last GCL: its coordinate MLP and the next block's first GCL) all run.
"""
import functools
import itertools
import math
import re

import pytest
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
from fp64_rows import (build_model, check_rows, dev, make_case, node_tail_shape, node_tile, oracle_forward, pocket_item,
                       run_dyn)
from oracle import difflinker_oracle as orc

H = 128
LOG2E = 1.4426950408889634
FIRE, QUIET = 2.0 ** 16, 2.0 ** 12      # 2^14 with a factor-4 margin either way
SM_COUNTS = (132, 114, 78)
F_FC, F_PK = 8, 9
IMPLS = ["simt", "auto"]
OPTIONS = list(itertools.product((False, True), repeat=3))      # (tanh, mean, sin_embedding)
DEFAULT, TMS = (False, False, False), (True, True, True)
SIN = (False, False, True)

WORST = {}          # test label -> (worst err / bound, C needed beside TAU, worst err / S_b, fraction within TAU)


def opt_id(o):
    return "-".join(n for n, on in zip(("tanh", "mean", "sin"), o) if on) or "default"


# ------------------------------------------------------------------------------------------------------------ batches
FC_SIZES = (32, 27, 20, 9)          # live atoms per molecule, N = 32: a multiple of every node tile these batches get
FC_LINKERS = (5, 1, 4, 9)
SPREAD = (1.0, 64.0, 256.0, 1.0)    # coordinate gains per molecule: two compact, two spread over hundreds of A


def _fc_batch(seed, gains):
    g = torch.Generator().manual_seed(seed)
    items = []
    for n, lk, s in zip(FC_SIZES, FC_LINKERS, gains):
        lm = torch.zeros(n)
        lm[n - lk:] = 1.0
        types = torch.randint(0, F_FC, (n,), generator=g)
        items.append({'positions': s * 1.5 * torch.randn((n, 3), generator=g),
                      'one_hot': torch.nn.functional.one_hot(types, F_FC).float(),
                      'fragment_mask': 1.0 - lm, 'linker_mask': lm})
    return collate(items)


def _pocket_molecule(g, n_pocket, n_isolated):
    """A 10-atom ligand (6 fragment-only, 4 linker) around the origin, n_pocket pocket atoms 3 .. 12 A from it, and
    n_isolated pocket atoms 40 A away from everything (rows of degree 0)."""
    lig = 1.2 * torch.randn((10, 3), generator=g, dtype=torch.float64)
    v = torch.randn((n_pocket, 3), generator=g, dtype=torch.float64)
    pk = v / v.norm(dim=1, keepdim=True) * (4.0 + 6.0 * torch.rand((n_pocket, 1), generator=g, dtype=torch.float64))
    iso = 40.0 * torch.tensor([[1.0 + k, 0.0, 0.0] for k in range(n_isolated)], dtype=torch.float64)
    return torch.cat([lig, pk, iso]), ['f'] * 6 + ['l'] * 4 + ['p'] * (n_pocket + n_isolated)


@functools.lru_cache(maxsize=None)
def batch_case(name):
    if name == "fc":
        return make_case(_fc_batch(91, (1.0,) * 4), F_FC, 'FC', 92)
    if name == "fc_spread":
        return make_case(_fc_batch(91, SPREAD), F_FC, 'FC', 92)
    if name == "pocket":
        g = torch.Generator().manual_seed(93)
        mols = [_pocket_molecule(g, 30, 2), _pocket_molecule(g, 21, 1)]
        batch = collate([pocket_item(g, pos, role, F_PK) for pos, role in mols])
        return make_case(batch, F_PK, 'FC-10A-4A', 94)
    kind, sms = name.split("@")                  # "tile128@132": 128-node tiles on that many SMs
    B, N = node_tail_shape(kind, int(sms))
    spec = synthetic.WorkloadSpec(f"rescale_{kind}", B=B, N=N, n_min=max(3, N // 2), l_min=1, l_max=8, F=F_FC, L=2, T=10,
                                  seed=95)
    return make_case(collate(synthetic.make_items(spec)), F_FC, 'FC', 96)


# ---------------------------------------------------------------------------------------------------------- the levers
GCL = r"dynamics\.e_block_\d+\.gcl_\d+\."
EQ = r"dynamics\.e_block_\d+\.gcl_equiv\."
HCOLS, WD, W0, EMB24 = slice(0, 2 * H), slice(2 * H, 2 * H + 1), slice(2 * H + 1, 2 * H + 2), slice(2 * H, 2 * H + 24)


def _edge_gain(mlp, cols, k):
    """First-layer columns (and with HCOLS the bias) x 2^k, the second layer's weight x 2^-k: the operands of the second
    GEMM grow by ~2^k, the MLP's output stays in range (silu is ~linear or ~0 far from 0)."""
    pre = GCL + "edge_mlp." if mlp == "edge" else EQ + "coord_mlp."
    out = [(pre + r"0\.weight", cols, k), (pre + r"2\.weight", None, -k)]
    if cols == HCOLS:
        out.append((pre + r"0\.bias", None, k))
    return out


# name -> (batch, options, levers(opts) -> [(parameter regex, column slice or None, exponent)], expected(opts) -> dict).
# Expected outcomes: 's1' / 's2' / 's3' (any node launch), 's1_proj' (the projection-only launch): 'fire' or 'quiet';
# 'gcl' / 'coord' (edge launches): 'all' (every edge rescales), 'fire' (some edge), 'quiet' (none), 'mixed' (some row
# sums edges that rescale and edges that do not).
NODE_QUIET = dict(s1='quiet', s2='quiet', s3='quiet')
SPREAD_COMP = [(GCL + r"edge_mlp\.2\.weight", None, -20), (EQ + r"coord_mlp\.2\.weight", None, -20)]
CASES = {
    # A / B bound: edge (and coordinate) MLP h-columns and bias; every edge rescales, the node kernel never does
    "ab": ("fc", OPTIONS, lambda o: _edge_gain("edge", HCOLS, 17),
           lambda o: dict(NODE_QUIET, gcl='all', coord='quiet')),
    "ab_coord": ("fc", OPTIONS, lambda o: _edge_gain("edge", HCOLS, 17) + _edge_gain("coord", HCOLS, 17),
                 lambda o: dict(NODE_QUIET, gcl='all', coord='all')),
    # distance term: without the embedding column 2H is wd and only far pairs rescale (mixed scales in one row's sum);
    # with it, column 2H is the sin(d f_0) column and enters every edge's bound
    "dist": ("fc", OPTIONS, lambda o: _edge_gain("edge", WD, 20 if o[2] else 14),
             lambda o: dict(NODE_QUIET, gcl='all' if o[2] else 'mixed')),
    # molecules spread over hundreds of A: d max|wd| alone passes 2^16 on far pairs (the second layers x 2^-20 keep the
    # messages in range); with the embedding the bound has no d term, and no edge rescales
    "spread": ("fc_spread", OPTIONS, lambda o: [] if o[2] else SPREAD_COMP,
               lambda o: dict(NODE_QUIET, gcl='quiet', coord='quiet') if o[2] else dict(NODE_QUIET, gcl='mixed')),
    # d0 term (column 2H + 1; with the embedding, the sin(d f_1) column)
    "d0": ("fc", (DEFAULT, TMS), lambda o: _edge_gain("edge", W0, 20 if o[2] else 14),
           lambda o: dict(NODE_QUIET, gcl='all' if o[2] else 'fire')),
    # the 24 embedding columns, on the spread batch: every edge
    "emb_cols": ("fc_spread", (SIN, TMS), lambda o: _edge_gain("edge", EMB24, 16), lambda o: dict(NODE_QUIET, gcl='all')),
    # agg only: messages x 2^18, node_mlp.0's agg columns x 2^-18: s1 through agg
    "agg": ("fc", (DEFAULT, TMS), lambda o: [(GCL + r"edge_mlp\.2\.weight", None, 18),
                                           (GCL + r"edge_mlp\.2\.bias", None, 18),
                                           (GCL + r"node_mlp\.0\.weight", slice(H, 2 * H), -18)],
            lambda o: dict(s1='fire', s2='quiet', s3='quiet', s1_proj='quiet', gcl='quiet', coord='quiet')),
    # pre-SiLU only: node_mlp.0 x 2^17, node_mlp.2.weight x 2^-17: s2
    "pre": ("fc", (DEFAULT, TMS), lambda o: [(GCL + r"node_mlp\.0\.weight", None, 17),
                                           (GCL + r"node_mlp\.0\.bias", None, 17),
                                           (GCL + r"node_mlp\.2\.weight", None, -17)],
            lambda o: dict(s1='quiet', s2='fire', s3='quiet', gcl='quiet', coord='quiet')),
    # h': node_mlp.2.bias x 2^20: s3, the projections of the next launch and the edge scales they feed
    "hprime": ("fc", (DEFAULT, TMS), lambda o: [(GCL + r"node_mlp\.2\.bias", None, 20)],
               lambda o: dict(s3='fire', s1_proj='quiet', gcl='fire', coord='fire')),
    # embedding layer x 2^17: s1 in the projection-only launch (where s3 = s1)
    "embed": ("fc", (DEFAULT, TMS), lambda o: [(r"dynamics\.embedding\.weight", None, 17)],
              lambda o: dict(s1_proj='fire', gcl='all')),
}
# everything at once: operands up to ~2^41 (scales ~2^-28), every value finite in fp32
ALL_LEVERS = lambda o: (_edge_gain("edge", HCOLS, 24) + _edge_gain("coord", HCOLS, 24)
                        + [(GCL + r"node_mlp\.0\.weight", None, 27), (GCL + r"node_mlp\.0\.bias", None, 27),
                           (GCL + r"node_mlp\.2\.weight", None, -27), (GCL + r"edge_mlp\.2\.bias", None, 8),
                           (GCL + r"edge_mlp\.2\.weight", None, 8), (GCL + r"node_mlp\.0\.weight", slice(H, 2 * H), -8),
                           (GCL + r"node_mlp\.2\.bias", None, 6), (r"dynamics\.embedding\.weight", None, 16)])
ALL_EXPECT = lambda o: dict(s1='fire', s2='fire', s3='fire', s1_proj='fire', gcl='all', coord='all')
CASES["all"] = ("fc", (DEFAULT, TMS), ALL_LEVERS, ALL_EXPECT)
# the same cases on a cut-off graph (sparse tiles), default and tanh + mean + sin; there the distance case is the wd gain
POCKET_CASES = ("ab", "ab_coord", "dist", "d0", "agg", "pre", "hprime", "embed", "all")
CASES.update({f"pocket_{c}": ("pocket", (DEFAULT, TMS)) + CASES[c][2:] for c in POCKET_CASES})
# 128-node tiles (B * N > 120 SMs, N <= 64), every molecule driven alike: s2 in the node kernel and every edge scale. A node
# tile here spans two or three molecules, and the scale follows the tile's largest value; under the "all" gains (operands
# ~2^41) that costs a smaller batch-mate's rows precision (measured on an H100: a coordinate row at 2.3e-5 * S_b, 47 times the
# oracle's own fp32 error), which is the per-tile scaling policy and not checked here.
CASES["tile128_pre_ab"] = ("tile128_tail1", (DEFAULT,),
                           lambda o: CASES["pre"][2](o) + CASES["ab_coord"][2](o),
                           lambda o: dict(s1='quiet', s2='fire', s3='quiet', gcl='all', coord='all'))

GPU_PARAMS = [(c, o) for c, (_, opts, _, _) in CASES.items() for o in opts]


def apply_levers(dyn, levers):
    params = dict(dyn.named_parameters())
    with torch.no_grad():
        for pattern, cols, k in levers:
            hit = [n for n in params if re.fullmatch(pattern, n)]
            assert hit, pattern
            for n in hit:
                p = params[n]
                (p if cols is None else p[:, cols]).mul_(2.0 ** k)


def case_model(case_name, opts, impl):
    batch, _, levers, _ = CASES[case_name]
    graph = 'FC' if batch != 'pocket' else 'FC-10A-4A'
    dyn, cfg = build_model(graph, F_FC if graph == 'FC' else F_PK, opts, impl, 101, n_layers=2, inv_sublayers=2)
    apply_levers(dyn, levers(opts))
    return dyn, cfg


def case_batch(case_name, num_sms):
    batch = CASES[case_name][0]
    return batch_case(f"{batch}@{num_sms}" if batch.startswith("tile") else batch)


# ------------------------------------------------------------------------------------------------------- range witness
class Witness:
    """Per-node and per-edge quantities of one fp64 oracle forward, in the kernels' terms; `outcome(tile)` reduces them for
    a node tile size."""

    def __init__(self, case, sin):
        B, N = case['z'].shape[:2]
        self.nm = (case['atom_mask'].reshape(B * N) != 0)
        self.lk = (case['linker_mask'].reshape(B * N) != 0) & self.nm
        self.sin = sin
        self.node = []          # node launches: dict(hagg, pre, hp, proj) per node (B*N,)
        self.edges = []         # edge launches: dict(coord, launch, proj, row, col, wterm)
        self.h = self.pending = self.rowcol = None

    def lin(self, orig, sd, prefix, v):
        out = orig(sd, prefix, v)
        amax = lambda t: t.abs().amax(1).cpu()
        if prefix.endswith(".embedding"):                               # projection-only launch: s3 = s1 = max |h|
            self.h = out
            self.node.append(dict(hagg=amax(out), pre=None, hp=amax(out), proj=[]))
        elif prefix.endswith(".node_mlp.0"):
            self.pending = (v, out)
        elif prefix.endswith(".node_mlp.2"):
            n_in, pre = self.pending
            self.h = (n_in[:, :H] + out) * self.nm.to(out)[:, None]
            self.node.append(dict(hagg=amax(n_in), pre=amax(pre), hp=amax(self.h), proj=[]))
        elif prefix.endswith(".edge_mlp.0") or prefix.endswith(".coord_mlp.0"):
            W, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
            launch = self.node[-1]
            launch['proj'].append((amax(self.h @ W[:, :H].T + b), amax(self.h @ W[:, H:2 * H].T)))
            row, col = self.rowcol
            wmax = W[:, 2 * H:].abs().amax(0).cpu() * LOG2E
            if self.sin:
                wterm = torch.full((row.numel(),), wmax.sum().item(), dtype=torch.float64, device='cpu')
            else:
                wterm = (v[:, 2 * H] * wmax[0] + v[:, 2 * H + 1] * wmax[1]).cpu()
            self.edges.append(dict(coord=prefix.endswith(".coord_mlp.0"), launch=len(self.node) - 1,
                                   proj=len(launch['proj']) - 1, row=row.cpu(), col=col.cpu(), wterm=wterm))
        return out

    def outcome(self, tile):
        def tile_max(v):
            n = v.numel()
            t = torch.cat([v, v.new_zeros((-n) % tile)]).reshape(-1, tile).amax(1)
            return t.repeat_interleave(tile)[:n]
        res = dict(s1_proj=self.node[0]['hagg'].max().item(),
                   s1=max(x['hagg'].max().item() for x in self.node),
                   s2=max(x['pre'].max().item() for x in self.node[1:]),
                   s3=max(x['hp'].max().item() for x in self.node))
        mixed = {False: False, True: False}
        for coord in (False, True):
            lo, hi = math.inf, 0.0
            for e in self.edges:
                if e['coord'] != coord:
                    continue
                amax_a, amax_b = self.node[e['launch']]['proj'][e['proj']]
                row, col = e['row'], e['col']
                keep = self.nm[row] & self.nm[col] & (self.lk[row] if coord else True)
                bound = LOG2E * (tile_max(amax_a)[row] + tile_max(amax_b)[col]) + e['wterm']
                bound, row, col = bound[keep], row[keep], col[keep]
                lo, hi = min(lo, bound.min().item()), max(hi, bound.max().item())
                off = row != col
                n = self.nm.numel()
                rmax = torch.zeros(n, dtype=torch.float64).scatter_reduce_(0, row[off], bound[off], 'amax')
                rmin = torch.full((n,), math.inf, dtype=torch.float64).scatter_reduce_(0, row[off], bound[off], 'amin')
                mixed[coord] |= bool(((rmax >= FIRE) & (rmin <= QUIET)).any())
            key = 'coord' if coord else 'gcl'
            res[key + '_min'], res[key + '_max'], res[key + '_mixed'] = lo, hi, mixed[coord]
        return res


def witness(sd, cfg, case):
    """Runs the oracle in fp64 on the CPU while recording the witness (the pattern of egnn_options_oracle._with_egnn)."""
    w = Witness(case, cfg.sin_embedding)
    orig_lin, orig_geom = orc._lin, orc.pair_geometry

    def geom(x, row, col, *args):
        w.rowcol = (row, col)
        return orig_geom(x, row, col, *args)

    orc._lin = functools.partial(w.lin, orig_lin)
    orc.pair_geometry = geom
    try:
        out = oracle_forward(sd, cfg, case, torch.float64, torch.device("cpu") if not torch.cuda.is_available() else dev())
    finally:
        orc._lin, orc.pair_geometry = orig_lin, orig_geom
    return w, out


def check_outcome(label, res, expected):
    bad = []
    for key, want in expected.items():
        if key in ('gcl', 'coord'):
            lo, hi, mixed = res[key + '_min'], res[key + '_max'], res[key + '_mixed']
            ok = {'all': lo >= FIRE, 'fire': hi >= FIRE, 'quiet': hi <= QUIET, 'mixed': mixed}[want]
            got = f"min {lo:.3g}, max {hi:.3g}, mixed row {mixed}"
        else:
            ok = res[key] >= FIRE if want == 'fire' else res[key] <= QUIET
            got = f"{res[key]:.3g}"
        if not ok:
            bad.append(f"{key} must be '{want}': {got}")
    assert not bad, f"{label}: " + "; ".join(bad)


def check_tiles(case_name, case, tile):
    """A node tile never spans two molecules in a batch whose molecules are driven unequally."""
    if CASES[case_name][0] == "fc_spread":
        assert case['z'].shape[1] % tile == 0, (case_name, tile)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst per-row ratios (err / bound, C needed beside TAU, err / S_b, fraction of rows within TAU * S_b):")
        for k, (w, c, r, f) in WORST.items():
            print(f"  {k:48s} {w:9.3e} {c:9.3e} {r:9.3e} {f:6.3f}")


# ---------------------------------------------------------------------------------------------------------------- CPU
_CPU_WITNESS = {}


def _cpu_witness(case_name, opts, sms):
    key = (case_name, opts, sms if CASES[case_name][0].startswith("tile") else None)
    if key not in _CPU_WITNESS:
        dyn, cfg = case_model(case_name, opts, "simt")
        case = case_batch(case_name, sms)
        w, out = witness(dyn.state_dict(), cfg, case)
        assert torch.isfinite(out).all()
        _CPU_WITNESS[key] = w
    return _CPU_WITNESS[key]


@pytest.mark.parametrize("case_name,opts", [p for p in GPU_PARAMS if not CASES[p[0]][0].startswith("tile")],
                         ids=lambda v: v if isinstance(v, str) else opt_id(v))
def test_cases_drive_their_branches(case_name, opts):
    """Every case fires the branches it is built for, and only those, for 132, 114 and 78 SMs."""
    for sms in SM_COUNTS:
        case = case_batch(case_name, sms)
        B, N = case['z'].shape[:2]
        tile = node_tile(B * N, sms)
        check_tiles(case_name, case, tile)
        check_outcome(f"{case_name} {opt_id(opts)} {sms} SMs", _cpu_witness(case_name, opts, sms).outcome(tile),
                      CASES[case_name][3](opts))


def test_tile128_case_drives_its_branches():
    for sms in SM_COUNTS:
        case = case_batch("tile128_pre_ab", sms)
        B, N = case['z'].shape[:2]
        assert node_tile(B * N, sms) == 128 and N <= 64
        check_outcome(f"tile128_pre_ab {sms} SMs", _cpu_witness("tile128_pre_ab", DEFAULT, sms).outcome(128),
                      CASES["tile128_pre_ab"][3](DEFAULT))


def test_pocket_batch_has_no_pair_near_a_cutoff():
    """No squared distance within 1e-3 of 16 or 100, so fp32 and fp64 agree on every edge; some ligand-pocket pairs are
    edges, some are not, and the isolated pocket atoms have no edge at all."""
    case = batch_case("pocket")
    B, N = case['z'].shape[:2]
    x = case['z'][..., :3].double()
    live = case['atom_mask'].reshape(B, N) != 0
    for b in range(B):
        d2 = torch.cdist(x[b][live[b]], x[b][live[b]]) ** 2
        assert ((d2 - 16).abs() > 1e-3).all() and ((d2 - 100).abs() > 1e-3).all()
        assert (d2 < 100).sum() < d2.numel()


# ---------------------------------------------------------------------------------------------------------------- GPU
_REFS = {}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case_name,opts", GPU_PARAMS, ids=lambda v: v if isinstance(v, str) else opt_id(v))
def test_rescale_matches_fp64_per_row(case_name, opts, impl):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    case = case_batch(case_name, sms)
    dyn, cfg = case_model(case_name, opts, impl)
    key = (case_name, opts)
    if key not in _REFS:
        B, N = case['z'].shape[:2]
        tile = node_tile(B * N, sms)
        check_tiles(case_name, case, tile)
        w, ref64 = witness(dyn.state_dict(), cfg, case)
        check_outcome(f"{case_name} {opt_id(opts)} {sms} SMs", w.outcome(tile), CASES[case_name][3](opts))
        _REFS.clear()                                     # one case at a time: the 128-node-tile references are large
        _REFS[key] = (ref64, oracle_forward(dyn.state_dict(), cfg, case, torch.float32, dev()))
    ref64, ref32 = _REFS[key]
    check_rows(f"{case_name} {opt_id(opts)} {impl}", run_dyn(dyn, case), ref64, ref32, case, WORST, min_tau_frac=0.5)
