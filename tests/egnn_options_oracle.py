"""TEST INFRASTRUCTURE ONLY -- the CPU oracle (oracle/difflinker_oracle.py) extended to the EGNN options of the reference
trainer: `tanh` (egnn.py:104-105), `sin_embedding` (SinusoidsEmbeddingNew, egnn.py:281-292) and
`aggregation_method='mean'` (egnn.py:315-319).

The options are fields of `OptionsConfig` (an OracleConfig), read by this module's layer functions. 'mean' needs nothing new: the
oracle's segment_reduce already divides by the per-row edge count of the edge list it is given. The entry points below
(dynamics_forward, edm_sample_chain, inpainting_sample_chain) run the oracle's own loops with this module's egnn_forward; with
every option off it computes exactly what oracle.egnn_forward does. tools/make_golden_opts.py checks it against the live
reference and writes tests/golden/*opts*.npz.
"""
import dataclasses
import math

import torch
import torch.nn.functional as F

from difflinker_b200 import synthetic
from oracle import difflinker_oracle as orc

# name -> spec; the specs are small so the reference runs them on a CPU in seconds
OPTION_SPECS = {
    "small_fc": synthetic.WorkloadSpec("small_fc", B=3, N=12, n_min=7, l_min=2, l_max=4, F=8, L=2, T=20, seed=11),
    "opts_cfg1": synthetic.WorkloadSpec("opts_cfg1", B=4, N=30, n_min=21, l_min=3, l_max=7, F=8, L=4, T=50, seed=1),
    "small_pocket_FC-10A-4A": synthetic.WorkloadSpec("small_pocket_FC-10A-4A", B=2, N=70, n_min=70, l_min=5, l_max=5,
                                                     F=9, L=2, T=20, seed=13, pocket=50, graph_type="FC-10A-4A"),
    # padded molecules (n_min < N) on a 4A graph
    "opts_pocket_4A": synthetic.WorkloadSpec("opts_pocket_4A", B=3, N=40, n_min=30, l_min=3, l_max=4, F=9, L=2, T=20,
                                             seed=21, pocket=20, graph_type="4A"),
}


@dataclasses.dataclass
class OptionsConfig(orc.OracleConfig):
    tanh: bool = False
    coords_range: float = 15.0     # EGNN passes its own coords_range=15 to every block (egnn.py:183-209)
    sin_embedding: bool = False


def options_kw(tanh, mean, sin=False):
    return dict(tanh=bool(tanh), aggregation_method='mean' if mean else 'sum', sin_embedding=bool(sin))


def oracle_cfg(hp):
    return OptionsConfig(in_node_nf=hp['in_node_nf'], context_node_nf=hp['context_node_nf'], n_layers=hp['n_layers'],
                         inv_sublayers=hp['inv_sublayers'], norm_constant=hp['norm_constant'],
                         normalization_factor=hp['normalization_factor'], graph_type=hp['graph_type'],
                         aggregation_method=hp['aggregation_method'], tanh=bool(hp['tanh']),
                         sin_embedding=bool(hp['sin_embedding']))


def sin_embedding(radial):
    """SinusoidsEmbeddingNew.forward (egnn.py:288-292) with its default max_res=15, min_res=15/2000, div_factor=4."""
    n = int(math.log(15. / (15. / 2000.), 4)) + 1
    freqs = 2 * math.pi * 4 ** torch.arange(n) / 15.
    emb = torch.sqrt(radial + 1e-8) * freqs[None, :]
    return torch.cat((emb.sin(), emb.cos()), dim=-1)


def coord_update(sd, prefix, h, x, row, col, unit_diff, edge_attr, linker_mask, node_mask, edge_mask, cfg):
    """EquivariantUpdate.coord_model (egnn.py:101-125), tanh branch included."""
    e_in = torch.cat([h.index_select(0, row), h.index_select(0, col), edge_attr], dim=1)
    phi = F.silu(orc._lin(sd, prefix + ".coord_mlp.0", e_in))
    phi = F.silu(orc._lin(sd, prefix + ".coord_mlp.2", phi))
    phi = F.linear(phi, sd[prefix + ".coord_mlp.4.weight"])
    if getattr(cfg, "tanh", False):
        trans = unit_diff * torch.tanh(phi) * cfg.coords_range
    else:
        trans = unit_diff * phi
    if edge_mask is not None:
        trans = trans * edge_mask
    agg = orc.segment_reduce(trans, row, x.shape[0], cfg.normalization_factor, cfg.aggregation_method)
    if linker_mask is not None:
        agg = agg * linker_mask
    x = x + agg
    if node_mask is not None:
        x = x * node_mask
    return x


def egnn_forward(sd, h, x, row, col, node_mask, linker_mask, edge_mask, cfg, prefix="dynamics"):
    """EGNN.forward (egnn.py:218-238) with EquivariantBlock.forward (egnn.py:157-178), reading the OptionsConfig fields."""
    emb = sin_embedding if getattr(cfg, "sin_embedding", False) else (lambda r: r)
    d0, _ = orc.pair_geometry(x, row, col)
    d0 = emb(d0)                                                          # egnn.py:220-222
    h = orc._lin(sd, prefix + ".embedding", h)
    for l in range(cfg.n_layers):
        blk = f"{prefix}.e_block_{l}"
        d_blk, unit = orc.pair_geometry(x, row, col, cfg.norm_constant)
        edge_attr = torch.cat([emb(d_blk), d0], dim=1)                    # egnn.py:159-162
        for s in range(cfg.inv_sublayers):
            h = orc.gcl_forward(sd, f"{blk}.gcl_{s}", h, row, col, edge_attr, node_mask, edge_mask, cfg)
        x = coord_update(sd, f"{blk}.gcl_equiv", h, x, row, col, unit, edge_attr, linker_mask, node_mask, edge_mask, cfg)
        if node_mask is not None:
            h = h * node_mask
    h = orc._lin(sd, prefix + ".embedding_out", h)
    if node_mask is not None:
        h = h * node_mask
    return h, x


def _with_egnn(fn):
    """An oracle entry point that runs with this module's egnn_forward for the duration of the call."""
    def run(*args, **kwargs):
        orig = orc.egnn_forward
        orc.egnn_forward = egnn_forward
        try:
            return fn(*args, **kwargs)
        finally:
            orc.egnn_forward = orig
    run.__doc__ = fn.__doc__
    return run


dynamics_forward = _with_egnn(orc.dynamics_forward)
edm_sample_chain = _with_egnn(orc.edm_sample_chain)
inpainting_sample_chain = _with_egnn(orc.inpainting_sample_chain)


def isolate_one_pocket_atom(z, batch, b=1):
    """Moves the first pocket atom of molecule b 60 A away, so it has no neighbour in any cut-off graph. Its row's sum is
    exactly 0, so this guards the divisor against 0 (which would give NaN), not its value; the padded-N and chunked-row
    cases check the counts."""
    z = z.clone()
    i = int(torch.nonzero(batch['pocket_mask'][b].reshape(-1))[0])
    z[b, i, 0] += 60.0
    return z, i


def spec_with_options(spec_name, tanh, mean, sin=False):
    return dataclasses.replace(OPTION_SPECS[spec_name], hparams=options_kw(tanh, mean, sin))


# fixture -> (spec, tanh, mean, sin_embedding, batch, seed); the Dynamics.forward cases
DYN_FIXTURES = {
    "dyn_opts_tanh_small_fc": ("small_fc", True, False, False, 3, 3),
    "dyn_opts_mean_small_fc": ("small_fc", False, True, False, 3, 3),
    "dyn_opts_sin_small_fc": ("small_fc", False, False, True, 3, 3),
    "dyn_opts_all_cfg1": ("opts_cfg1", True, True, True, 4, 4),
    "dyn_opts_all_pocket_FC-10A-4A": ("small_pocket_FC-10A-4A", True, True, True, 2, 5),
    "dyn_opts_mean_pocket_4A": ("opts_pocket_4A", False, True, False, 3, 6),   # padded molecules, one isolated pocket row
}
# fixture -> (spec, tanh, mean, sin_embedding, batch, seed, keep_frames, inpainting)
CHAIN_FIXTURES = {
    "chain_opts_all_cfg1": ("opts_cfg1", True, True, True, 4, 7, 5, False),
    "inpaint_chain_opts_tanh_mean_cfg1": ("opts_cfg1", True, True, False, 4, 8, 3, True),
}
