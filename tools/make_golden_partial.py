"""TEST INFRASTRUCTURE ONLY -- golden vectors for partial diffusion (EDM.sample_chain from step t0), from the LIVE,
UNMODIFIED reference (build container only, like oracle/make_golden.py), written as NEW files tests/golden/partial_*.npz.

The reference has no partial-diffusion entry point, so the chain is composed of the reference's own methods, called in
this order on a reference DDPM with seeded weights (verified by sha256) and the batch's own linker kept in the template:
`normalize`, `sample_combined_position_feature_noise`, `gamma` / `alpha` / `sigma` at t0 / T, the two noising lines of
EDM.forward (edm.py:73-74, restated below), then `sample_p_zs_given_zt_only_linker` for s = t0-1 .. 0 and
`sample_p_xh_given_z0_only_linker`, with the frames written as EDM.sample_chain writes them (edm.py:143-174).
The oracle (tests/partial_diffusion_oracle.py) is asserted to reproduce that composition with max |delta| = 0.0, and the
same composition in float64 gives each molecule's fp32-vs-fp64 drift (`drift64`, as oracle/make_golden_r2.py records it).
Run:  python tools/make_golden_partial.py [fixture ...]
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from difflinker_b200 import synthetic  # noqa: E402
from oracle import difflinker_oracle as orc, make_golden as mg  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402
import partial_diffusion_oracle as po  # noqa: E402

# one trajectory per entry, written as fixture f"{base}_k{keep}" for every keep_frames in keeps:
# base -> (spec, batch, weight seed, t0, keeps). t0 = 500 runs 4 molecules: three passes of 500 reference steps at B = 16 take
# the better part of an hour of CPU.
FIXTURES = {f"partial_cfg2_zinc_t{t0}": ("cfg2_zinc", 16, 0, t0, (1, 10)) for t0 in (1, 50, 250)}
FIXTURES["partial_cfg2_zinc_t500"] = ("cfg2_zinc", 4, 0, 500, (1, 10))
FIXTURES["partial_cfg4_pockets_t100"] = ("cfg4_pockets", 3, 0, 100, (1,))


def reference_inputs(ns, ddpm, data):
    """DDPM.sample_chain's inputs (lightning.py:405-452) with sample_fn=None, the template's linker rows holding the batch's
    own linker: the reference's template, its context columns and its centre-of-mass removal."""
    tpl = ns.datasets.create_templates_for_linker_generation(data, data['linker_mask'].sum(1).view(-1).int())
    n = tpl['linker_mask'].shape[1]
    keep = tpl['linker_mask'].bool()
    assert torch.equal(data['linker_mask'][:, :n], tpl['linker_mask']) and not data['linker_mask'][:, n:].any()
    x = torch.where(keep, data['positions'][:, :n], tpl['positions'])
    h = torch.where(keep, data['one_hot'][:, :n], tpl['one_hot'])
    fragment_mask, linker_mask, node_mask = tpl['fragment_mask'], tpl['linker_mask'], tpl['atom_mask']
    if '.' in ddpm.train_data_prefix:
        fo = tpl['fragment_only_mask']
        parts = [fo, fragment_mask - fo]
        com = fo                                                   # MOADDataset val_dataset, lightning.py:441-442
    else:
        parts = [fragment_mask]
        com = fragment_mask
    if ddpm.anchors_context:
        parts = [tpl['anchors']] + parts
    context = torch.cat(parts, dim=-1)
    x = ns.utils.remove_partial_mean_with_mask(x, node_mask, com)
    return dict(x=x, h=h, node_mask=node_mask, edge_mask=tpl['edge_mask'], fragment_mask=fragment_mask,
                linker_mask=linker_mask, context=context)


def reference_partial_chain(ns, edm, kw, t0, keeps, draw):
    """The reference's methods composed into a partial chain, one per keep_frames in `keeps` (the same trajectory, its
    frames written as EDM.sample_chain writes them for that keep_frames); `draw` supplies sample_gaussian_with_mask's
    numbers."""
    orig = ns.utils.sample_gaussian_with_mask
    ns.utils.sample_gaussian_with_mask = lambda size, device, node_mask: draw(size).to(node_mask.dtype) * node_mask
    try:
        x, h, node_mask, fragment_mask, linker_mask = kw['x'], kw['h'], kw['node_mask'], kw['fragment_mask'], kw['linker_mask']
        edge_mask, context = kw['edge_mask'], kw['context']
        B, N = x.size(0), x.size(1)
        x, h = edm.normalize(x, h)
        xh = torch.cat([x, h], dim=2)
        eps_t = edm.sample_combined_position_feature_noise(n_samples=B, n_nodes=N, mask=linker_mask)
        t = torch.full((B, 1), fill_value=float(t0)) / edm.T      # edm.py:50-52 (t_int is a float tensor)
        gamma_t = edm.inflate_batch_array(edm.gamma(t), x)
        alpha_t, sigma_t = edm.alpha(gamma_t, x), edm.sigma(gamma_t, x)
        if xh.dtype == torch.float64:
            alpha_t, sigma_t = alpha_t.double(), sigma_t.double()
        z = alpha_t * xh + sigma_t * eps_t                          # edm.py:73
        z = xh * fragment_mask + z * linker_mask                    # edm.py:74
        chains = {k: torch.zeros((k,) + z.size(), dtype=z.dtype) for k in keeps}
        for s in reversed(range(0, t0)):                            # edm.py:146-163
            s_array = torch.full((B, 1), fill_value=s)
            t_array = s_array + 1
            s_array = s_array / edm.T
            t_array = t_array / edm.T
            z = edm.sample_p_zs_given_zt_only_linker(s=s_array, t=t_array, z_t=z, node_mask=node_mask,
                                                     fragment_mask=fragment_mask, linker_mask=linker_mask,
                                                     edge_mask=edge_mask, context=context)
            for k, chain in chains.items():
                chain[(s * k) // edm.T] = edm.unnormalize_z(z)
        x, h = edm.sample_p_xh_given_z0_only_linker(z_0=z, node_mask=node_mask, fragment_mask=fragment_mask,
                                                    linker_mask=linker_mask, edge_mask=edge_mask, context=context)
        for chain in chains.values():
            chain[0] = torch.cat([x, h], dim=2)                     # edm.py:166-174
        return chains
    finally:
        ns.utils.sample_gaussian_with_mask = orig


def golden_partial(ns, base, spec_name, nb, seed, t0, keeps):
    spec = synthetic.SPECS[spec_name]
    hp = synthetic.model_hparams(spec)
    torch.manual_seed(seed)
    ddpm = ns.lightning.DDPM(**hp, data_path=None, batch_size=nb, lr=1e-4, torch_device='cpu', test_epochs=1,
                             n_stability_samples=1)
    synthetic.init_reference_like_weights(ddpm)
    ddpm.eval()
    items = synthetic.make_items(spec, batch=nb)
    if spec.pocket:                                                 # generate_with_pocket.py:249-250
        ddpm.val_dataset = ns.datasets.MOADDataset(data=items)
    data = ns.datasets.collate(items)
    T = ddpm.edm.T
    kw = reference_inputs(ns, ddpm, data)
    noise_seed = seed + 3000 + t0
    keep = max(keeps)
    with torch.no_grad():
        chains = reference_partial_chain(ns, ddpm.edm, kw, t0, keeps, mg.seeded_noise(noise_seed))
        sd_dyn = {k[len("edm.dynamics."):]: v for k, v in ddpm.state_dict().items() if k.startswith("edm.dynamics.")}
        gam = orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])
        assert torch.equal(gam, ddpm.edm.gamma.gamma.detach()), "oracle gamma table differs"
        oc = po.linker_partial_chain(sd_dyn, mg.oracle_cfg(hp), gam, T, t0, kw['x'], kw['h'], kw['node_mask'],
                                     kw['fragment_mask'], kw['linker_mask'], kw['edge_mask'], kw['context'],
                                     keep_frames=keep, norm_values=tuple(hp['normalize_factors']),
                                     noise_fn=mg.seeded_noise(noise_seed))
    err = (oc - chains[keep]).abs().max().item()
    assert err == 0.0, f"{base}: oracle vs reference composition {err}"
    # the same composition in float64: how well-conditioned each molecule's trajectory is
    ddpm64 = ddpm.double()
    kw64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
    draw = mg.seeded_noise(noise_seed)
    with torch.no_grad():
        chain64 = reference_partial_chain(ns, ddpm64.edm, kw64, t0, (1,), lambda size: draw(size).double())[1]
    nm = kw['node_mask'].float()
    final = chains[keep][0]
    drift = ((chain64[0][..., :3].float() - final[..., :3]) * nm).abs().flatten(1).max(1).values
    types_equal = bool(torch.equal(chain64[0][..., 3:].float(), final[..., 3:]))
    alpha, sigma = po.start_scalars(gam, t0, T, nb, hp['diffusion_steps'])
    for k in keeps:
        meta = dict(kind="partial_chain", spec=spec_name, batch=nb, seed=seed, noise_seed=noise_seed, t0=t0,
                    keep_frames=k, T=T, table_timesteps=hp['diffusion_steps'], sha=mg.state_sha(sd_dyn),
                    oracle_max_abs_err=err, moad_val_dataset=bool(spec.pocket), fp64_types_equal=types_equal,
                    alpha_t0=float(alpha[0]), sigma_t0=float(sigma[0]))
        mg.save(f"{base}_k{k}", meta, chain=chains[k], drift64=drift, **kw)
    print(f"  {base}: drift64 " + " ".join(f"{v:.1e}" for v in drift.tolist()) + f" (types equal: {types_equal})",
          flush=True)


def main():
    torch.set_num_threads(int(os.environ.get("GOLDEN_THREADS", "8")))
    ns = load_reference()
    only = set(sys.argv[1:])
    for base, args in FIXTURES.items():
        if not only or base in only:
            golden_partial(ns, base, *args)


if __name__ == "__main__":
    main()
