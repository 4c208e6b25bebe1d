"""Shared by the per-row fp64 tests (test_edge_tiles_fp64.py, test_range_rescale_fp64.py): batches in the form
Dynamics.forward takes, models with their option-aware oracle config, the oracle run in any dtype on any device, the
node kernel's tile size and the per-row criterion.

The criterion: each live row i of molecule b is checked on its own, separately on the coordinate columns and the feature
columns: err_i = max|got - ref64| must satisfy err_i <= max(C_DRIFT * drift_i, TAU * S_b), where drift_i = max|ref32 - ref64|
is the oracle's own float32 error on that row (how well conditioned the row is) and S_b the largest |ref64| over the
molecule's live rows. Padded rows, and the coordinate rows outside the linker mask, must be exactly 0.
"""
import contextlib

import torch

from difflinker_b200 import Dynamics, DynamicsWithPockets, synthetic
import egnn_options_oracle as eo

# Measured on an H100 80GB HBM3 (400 W): where a row's error exceeds TAU * S_b it is at most 15.5 times the oracle's own fp32
# error on that row (FC, 128 columns, tanh + mean + sin_embedding; 11.1 on the cut-off boundary batch, <= 9 elsewhere). Those
# rows are coordinate rows far from the origin, where both fp32 runs round x + agg alike, and rows with the ill-conditioned
# sinusoidal embedding.
TAU = 1e-5          # floor of the per-row bound, relative to the molecule's scale
C_DRIFT = 30.0      # multiple of the oracle's own fp32-vs-fp64 error on the row


# ------------------------------------------------------------------------------------------------------------ batches
def latent(batch, F, seed):
    """z: the batch's positions, one_hot / 4 on context rows and N(0, 1) features on linker rows, garbage on padded rows."""
    g = torch.Generator().manual_seed(seed)
    B, N = batch['positions'].shape[:2]
    live = batch['atom_mask'].reshape(B, N, 1) != 0
    lk = batch['linker_mask'].reshape(B, N, 1) != 0
    h = torch.where(lk, torch.randn((B, N, F), generator=g), batch['one_hot'].float() / 4)
    z = torch.cat([batch['positions'].float(), h], dim=2)
    z = torch.where(live, z, 3.0 * torch.randn(z.shape, generator=g))
    t = torch.rand((B, 1), generator=g)
    return z, t


def make_case(batch, F, graph_type, seed, **extra):
    """The arguments of one Dynamics.forward on a collated batch, with its graph type and feature count."""
    z, t = latent(batch, F, seed)
    if graph_type == 'FC':
        ctx = batch['fragment_mask'].float()
    else:
        fo = batch['fragment_only_mask'].float()
        ctx = torch.cat([fo, batch['fragment_mask'].float() - fo], dim=-1)
    return dict(t=t, z=z, atom_mask=batch['atom_mask'], linker_mask=batch['linker_mask'].float(),
                edge_mask=batch['edge_mask'], context=ctx, graph_type=graph_type, F=F, **extra)


def pocket_item(g, pos, role, n_types):
    """One molecule of a pocket batch; role per atom: 'f' fragment-only, 'p' pocket, 'l' linker."""
    n = pos.shape[0]
    mask = lambda c: torch.tensor([1.0 if r == c else 0.0 for r in role])
    fo, pk, lm = mask('f'), mask('p'), mask('l')
    types = torch.randint(0, n_types, (n,), generator=g)
    return {'positions': pos.float(), 'one_hot': torch.nn.functional.one_hot(types, n_types).float(),
            'fragment_mask': fo + pk, 'linker_mask': lm, 'fragment_only_mask': fo, 'pocket_mask': pk}


# -------------------------------------------------------------------------------------------------- models and oracle
def build_model(graph_type, F, opts, impl, seed, n_layers=1, inv_sublayers=1):
    """A Dynamics of the given depth (dl_helpers.build_dynamics fixes inv_sublayers from the spec) and its oracle config."""
    tanh, mean, sin = opts
    ctx_nf = 1 if graph_type == 'FC' else 2
    kw = dict(n_layers=n_layers, inv_sublayers=inv_sublayers, norm_constant=1e-6, normalization_factor=100,
              graph_type=graph_type)
    torch.manual_seed(seed)
    cls = Dynamics if graph_type == 'FC' else DynamicsWithPockets
    dyn = cls(in_node_nf=F, n_dims=3, context_node_nf=ctx_nf, hidden_nf=128, edge_impl=impl, **kw,
              **eo.options_kw(tanh, mean, sin))
    synthetic.init_reference_like_weights(dyn)
    cfg = eo.OptionsConfig(in_node_nf=F, context_node_nf=ctx_nf, aggregation_method='mean' if mean else 'sum',
                           tanh=tanh, sin_embedding=sin, **kw)
    return dyn, cfg


@contextlib.contextmanager
def _full_fp32_matmul():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def oracle_forward(sd, cfg, case, dtype, device):
    """The option-aware oracle's Dynamics.forward in `dtype` on `device` (factory calls inside it follow the device)."""
    def cast(v):
        return v.to(device=device, dtype=dtype) if v.is_floating_point() else v.to(device)
    with torch.no_grad(), torch.device(device), _full_fp32_matmul():
        out = eo.dynamics_forward({k: cast(v) for k, v in sd.items()}, cfg, cast(case['t']), cast(case['z']),
                                  cast(case['atom_mask']), cast(case['linker_mask']), cast(case['edge_mask']),
                                  cast(case['context']))
    return out.double().cpu()


def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda", 0)


def run_dyn(dyn, case):
    d = dev()
    with torch.no_grad():
        return dyn(case['t'].to(d), case['z'].to(d), case['atom_mask'].to(d), case['linker_mask'].to(d),
                   case['edge_mask'].to(d), case['context'].to(d)).double().cpu()


def node_tile(n, num_sms):
    """The node kernel's tile size for n = B * N nodes (kernels_node_tc.cuh pick_tile_nodes)."""
    per = -(-n // max(num_sms, 1))
    return min(128, max(8, (per + 7) & ~7))


def node_tail_shape(kind, num_sms):
    """(B, N) with B * N nodes giving the requested node-kernel tiling: the tile size and the last tile's node count."""
    tile, tail = {"tile8_tail1": (8, 1), "tile8_exact": (8, 0), "tile64_tail1": (64, 1), "tile128_tail1": (128, 1)}[kind]
    lo = 1 if tile == 8 else (tile - 8) * num_sms + 1
    for n in range(max(lo, 16), 64 * 1024):
        if node_tile(n, num_sms) != tile or n % tile != tail:
            continue
        for N in range(64, 11, -1):
            if n % N == 0 and n // N >= 2:
                return n // N, N
    raise AssertionError(f"no (B, N) for {kind} on {num_sms} SMs")


# ------------------------------------------------------------------------------------------------- per-row criterion
def check_rows(label, got, ref64, ref32, case, report, min_tau_frac=None):
    """err_i <= max(C_DRIFT * drift_i, TAU * S_b) for every live row, on the coordinate and on the feature columns;
    padded rows and coordinate rows outside the linker mask exactly 0. report[label] gets (worst err / bound, C needed
    beside TAU, worst err / S_b, fraction of live rows within TAU * S_b on both parts). With min_tau_frac, ref32 must be
    finite and at least that fraction of the live rows must meet the plain TAU * S_b bound, so the drift term cannot carry
    a whole case."""
    B, N = got.shape[:2]
    live = case['atom_mask'].reshape(B, N) != 0
    lk = (case['linker_mask'].reshape(B, N) != 0) & live
    assert torch.equal(got[~live], torch.zeros_like(got[~live])), f"{label}: a padded row is not exactly 0"
    still = got[..., :3][live & ~lk]
    assert torch.equal(still, torch.zeros_like(still)), f"{label}: a coordinate row outside the linker mask is not exactly 0"
    sizes, links = live.sum(1), lk.sum(1)
    worst, need_c, rel = 0.0, 0.0, 0.0
    within = live.clone()
    fails = []
    for part, cols in (("vel", slice(0, 3)), ("h", slice(3, None))):
        err = (got[..., cols] - ref64[..., cols]).abs().amax(-1)
        drift = (ref32[..., cols] - ref64[..., cols]).abs().amax(-1)
        scale = torch.where(live, ref64[..., cols].abs().amax(-1), 0.0).amax(1, keepdim=True).expand(B, N)
        bound = torch.maximum(C_DRIFT * drift, TAU * scale)
        ratio = torch.where(err == 0, 0.0, err / bound)
        ratio = torch.where(live, ratio, 0.0)
        worst = max(worst, ratio.max().item())
        over_tau = live & (err > TAU * scale)
        within &= ~over_tau
        if over_tau.any():
            need_c = max(need_c, (err[over_tau] / drift[over_tau]).max().item())
        rel = max(rel, torch.where(live & (scale > 0), err / scale, 0.0).max().item())
        for b, i in torch.nonzero(ratio > 1).tolist()[:5]:
            fails.append(f"{part} row {i} of molecule {b} ({int(sizes[b])} live, {int(links[b])} linker): err "
                         f"{err[b, i].item():.3e}, drift {drift[b, i].item():.3e}, S_b {scale[b, i].item():.3e}")
    frac = within.sum().item() / max(live.sum().item(), 1)
    report[label] = (worst, need_c, rel, frac)
    assert not fails, f"{label}:\n" + "\n".join(fails)
    if min_tau_frac is not None:
        assert torch.isfinite(ref32).all(), f"{label}: the fp32 oracle is not finite"
        assert frac >= min_tau_frac, f"{label}: only {frac:.3f} of the live rows within {TAU} * S_b"
