"""TEST INFRASTRUCTURE ONLY -- golden vectors for the EGNN options `tanh` and `aggregation_method='mean'`, from the LIVE,
UNMODIFIED reference (build container only, like oracle/make_golden.py), written as NEW files tests/golden/*opts*.npz.

The generator lives outside oracle/, whose files pin the existing fixtures and stay as they are.
For every fixture the reference's own Dynamics / DDPM is built with the options, the option-aware oracle
(tests/egnn_options_oracle.py) is asserted to reproduce it (max |delta| printed), and for the chains the reference's own
fp32-vs-fp64 drift per molecule is recorded (`drift64`, as oracle/make_golden_r2.py drift does).
Run:  python tools/make_golden_opts.py [fixture ...]
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from difflinker_b200 import synthetic  # noqa: E402
from difflinker_b200.egnn import Dynamics as NativeDynamics, DynamicsWithPockets as NativePockets  # noqa: E402
from oracle import difflinker_oracle as orc, make_golden as mg, make_golden_r2 as mg2  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
import egnn_options_oracle as eo  # noqa: E402


def golden_dynamics_opts(ns, name, spec_name, tanh, mean, sin, nb, seed):
    spec = eo.spec_with_options(spec_name, tanh, mean, sin)
    hp = synthetic.model_hparams(spec)
    kw = dict(in_node_nf=hp['in_node_nf'], n_dims=3, context_node_nf=hp['context_node_nf'], hidden_nf=128,
              n_layers=hp['n_layers'], norm_constant=hp['norm_constant'], inv_sublayers=hp['inv_sublayers'],
              normalization_factor=hp['normalization_factor'], graph_type=hp['graph_type'], tanh=hp['tanh'],
              aggregation_method=hp['aggregation_method'], sin_embedding=hp['sin_embedding'])
    torch.manual_seed(seed)
    dyn = (ns.egnn.DynamicsWithPockets if spec.pocket else ns.egnn.Dynamics)(**kw)
    synthetic.init_reference_like_weights(dyn)
    dyn.eval()
    batch = mg.check_batching(ns, spec, nb)
    g = torch.Generator().manual_seed(seed + 7)
    com = batch['fragment_only_mask'] if spec.pocket else batch['fragment_mask']
    x = ns.utils.remove_partial_mean_with_mask(batch['positions'], batch['atom_mask'], com)
    z = torch.cat([x, batch['one_hot'] / 4], dim=2)
    z = z * batch['fragment_mask'] + torch.randn(z.shape, generator=g) * batch['linker_mask']
    z = z + 3.0 * torch.randn(z.shape, generator=g) * (1 - batch['atom_mask'].float())
    isolated = -1
    if spec.graph_type == '4A':
        z, isolated = eo.isolate_one_pocket_atom(z, batch)
    t = torch.rand((z.shape[0], 1), generator=g)
    ctx = mg.context_of(batch, spec)
    with torch.no_grad():
        out = dyn(t, z, batch['atom_mask'], batch['linker_mask'], batch['edge_mask'], ctx)
        sd = dyn.state_dict()
        o2 = eo.dynamics_forward(sd, eo.oracle_cfg(hp), t, z, batch['atom_mask'], batch['linker_mask'],
                                 batch['edge_mask'], ctx)
    err = (out - o2).abs().max().item()
    print(f"  {name}: oracle vs reference max|d| = {err:.2e}")
    assert err < 2e-6, f"{name}: oracle vs reference {err}"
    torch.manual_seed(seed)
    mine = (NativePockets if spec.pocket else NativeDynamics)(**kw)
    synthetic.init_reference_like_weights(mine)
    assert mg.state_sha(mine.state_dict()) == mg.state_sha(sd), "native parameter construction order diverged"
    meta = dict(kind="dynamics", spec=spec_name, batch=nb, seed=seed, pocket=bool(spec.pocket), sha=mg.state_sha(sd),
                oracle_max_abs_err=err, graph_type=hp['graph_type'], tanh=tanh, mean=mean, sin_embedding=sin,
                isolated_row=isolated)
    mg.save(name, meta, t=t, xh=z, node_mask=batch['atom_mask'], linker_mask=batch['linker_mask'],
            edge_mask=batch['edge_mask'], context=ctx, out=out)


def main():
    torch.set_num_threads(8)
    ns = load_reference()
    only = set(sys.argv[1:])
    for name, (spec_name, tanh, mean, sin, nb, seed) in eo.DYN_FIXTURES.items():
        if not only or name in only:
            golden_dynamics_opts(ns, name, spec_name, tanh, mean, sin, nb, seed)
    # the chain generators of oracle/make_golden.py, run with the option-aware oracle config and oracle loops
    saved = mg.oracle_cfg, mg.orc
    mg.oracle_cfg, mg.orc = eo.oracle_cfg, _OptionsOracle()
    try:
        for name, (spec_name, tanh, mean, sin, nb, seed, keep, inpaint) in eo.CHAIN_FIXTURES.items():
            if only and name not in only:
                continue
            spec = eo.spec_with_options(spec_name, tanh, mean, sin)
            if inpaint:
                mg.golden_inpaint_chain(ns, name, spec, nb, seed, keep)
            else:
                mg.golden_chain(ns, name, spec, nb, seed, keep)
                mg2.add_fp64_drift(ns, name, spec, nb, seed, keep)
    finally:
        mg.oracle_cfg, mg.orc = saved


class _OptionsOracle:
    """The oracle module as make_golden's chain generators see it, with the option-aware sampler loops."""
    edm_sample_chain = staticmethod(eo.edm_sample_chain)
    inpainting_sample_chain = staticmethod(eo.inpainting_sample_chain)

    def __getattr__(self, name):
        return getattr(orc, name)


if __name__ == "__main__":
    main()
