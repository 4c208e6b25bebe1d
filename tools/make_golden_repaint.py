"""TEST INFRASTRUCTURE ONLY -- golden vectors for RePaint resampling (InpaintingEDM.sample_chain with r passes per step),
from the LIVE, UNMODIFIED reference (build container only, like oracle/make_golden.py), written as NEW files
tests/golden/repaint_*.npz.

The reference has no resampling entry point, so the chain is composed of the reference's own methods, called on a
reference DDPM(inpainting=True) with seeded weights (verified by sha256): `normalize`, `sample_combined_position_feature_noise`,
then for s = T-1 .. 0 and pass u = 0 .. r-1 `sample_p_zs_given_zt`, `sample_q_zs_given_zt_and_x`, the recombination and
`utils.remove_mean_with_mask` of InpaintingEDM.sample_chain (edm.py:574-594), and for u < r-1 `gamma`,
`sigma_and_alpha_t_given_s`, `sample_combined_position_feature_noise` and the re-noise line (restated below); then
`sample_p_xh_given_z0` and `sample_q_xh_given_z0_and_x`, with the frames written as sample_chain writes them. The draws
are patched in as oracle/make_golden.py patches them for the inpainting chain. The oracle (tests/repaint_oracle.py) is
asserted to reproduce that composition with max |delta| = 0.0, and the same composition in float64 gives each molecule's
fp32-vs-fp64 drift (`drift64`). Each fixture also holds `jump`, the (T, 2) (alpha_t|s, sigma_t|s) of the reference's
sigma_and_alpha_t_given_s at the batch size, in dl_step_coef row order.
Run:  python tools/make_golden_repaint.py [fixture ...]
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
import dl_helpers as helpers  # noqa: E402
import repaint_oracle as ro  # noqa: E402

# name -> (spec, batch, weight seed, r, keep_frames). cfg1 stops at r = 3: with its synthetic weights the reference's own fp32
# chain reaches NaN at r = 4 for every noise seed tried (4000 .. 4011), and coordinates in the thousands at r = 3.
# There is no pocket fixture: the reference's InpaintingEDM cannot sample a pocket model, whose DynamicsWithPockets asserts on
# the linker_mask=None that InpaintingEDM passes (egnn.py:488); tests/test_inpaint_resampling.py covers pocket graphs on the
# GPU against fp64 and against the engine's own noise paths instead.
FIXTURES = {f"repaint_cfg1_r{r}_k{k}": ("cfg1_plumbing", 4, 0, r, k) for r in (2, 3) for k in (1, 5)}


def reference_inputs(ns, ddpm, data, spec):
    """DDPM.sample_chain's inputs with inpainting=True (lightning.py:405-452): the batch itself as the template, its context
    columns, and its centre of mass over every atom removed."""
    node_mask = data['atom_mask']
    x = ns.utils.remove_partial_mean_with_mask(data['positions'], node_mask, node_mask)
    return dict(x=x, h=data['one_hot'], node_mask=node_mask, edge_mask=data['edge_mask'],
                fragment_mask=data['fragment_mask'], linker_mask=data['linker_mask'],
                context=mg.context_of(data, spec))


def reference_repaint_chain(ns, edm, kw, r, keep_frames, draw):
    """The reference's methods composed into an r-pass inpainting chain; `draw` supplies the standard-normal numbers of
    sample_gaussian_with_mask and sample_center_gravity_zero_gaussian_with_mask."""
    utils = ns.utils
    o1, o2 = utils.sample_gaussian_with_mask, utils.sample_center_gravity_zero_gaussian_with_mask
    utils.sample_gaussian_with_mask = lambda size, device, node_mask: draw(size) * node_mask
    utils.sample_center_gravity_zero_gaussian_with_mask = \
        lambda size, device, node_mask: utils.remove_mean_with_mask(draw(size) * node_mask, node_mask)
    try:
        x, h, node_mask, fragment_mask, linker_mask = kw['x'], kw['h'], kw['node_mask'], kw['fragment_mask'], kw['linker_mask']
        edge_mask, context = kw['edge_mask'], kw['context']
        B, N = x.size(0), x.size(1)
        x, h = edm.normalize(x, h)
        xh = torch.cat([x, h], dim=2)
        z = edm.sample_combined_position_feature_noise(B, N, node_mask)          # edm.py:559
        chain = torch.zeros((keep_frames,) + z.size(), dtype=z.dtype)
        for s in reversed(range(0, edm.T)):                                       # edm.py:568-598
            s_array = torch.full((B, 1), fill_value=s)
            t_array = s_array + 1
            s_array = s_array / edm.T
            t_array = t_array / edm.T
            for u in range(r):
                z_lin = edm.sample_p_zs_given_zt(s=s_array, t=t_array, z_t=z, node_mask=node_mask, edge_mask=edge_mask,
                                                 context=context)
                z_frag = edm.sample_q_zs_given_zt_and_x(s=s_array, t=t_array, z_t=z, x=xh * fragment_mask,
                                                        node_mask=fragment_mask)
                z = z_lin * linker_mask + z_frag * fragment_mask
                z_x = utils.remove_mean_with_mask(z[:, :, :edm.n_dims], node_mask)
                z = torch.cat([z_x, z[:, :, edm.n_dims:]], dim=2)
                if u < r - 1:
                    gamma_s, gamma_t = edm.gamma(s_array), edm.gamma(t_array)
                    _, sigma_ts, alpha_ts = edm.sigma_and_alpha_t_given_s(gamma_t, gamma_s, z)
                    if z.dtype == torch.float64:
                        sigma_ts, alpha_ts = sigma_ts.double(), alpha_ts.double()
                    eps = edm.sample_combined_position_feature_noise(B, N, node_mask)
                    z = alpha_ts * z + sigma_ts * eps                             # the re-noise (RePaint)
            chain[(s * keep_frames) // edm.T] = edm.unnormalize_z(z)
        x_l, h_l = edm.sample_p_xh_given_z0(z_0=z, node_mask=node_mask, edge_mask=edge_mask, context=context)
        x_f, h_f = edm.sample_q_xh_given_z0_and_x(z_0=z, node_mask=node_mask)
        chain[0] = torch.cat([x_l, h_l], dim=2) * linker_mask + torch.cat([x_f, h_f], dim=2) * fragment_mask
        return chain
    finally:
        utils.sample_gaussian_with_mask, utils.sample_center_gravity_zero_gaussian_with_mask = o1, o2


def golden_repaint(ns, name, spec_name, nb, seed, r, keep):
    spec = helpers.spec_by_name(spec_name)
    hp = synthetic.model_hparams(spec)
    hp['inpainting'] = True
    torch.manual_seed(seed)
    ddpm = ns.lightning.DDPM(**hp, data_path=None, batch_size=nb, lr=1e-4, torch_device='cpu', test_epochs=1,
                             n_stability_samples=1)
    synthetic.init_reference_like_weights(ddpm)
    ddpm.eval()
    T = ddpm.edm.T
    data = ns.datasets.collate(synthetic.make_items(spec, batch=nb))
    kw = reference_inputs(ns, ddpm, data, spec)
    noise_seed = seed + 4000 + r
    with torch.no_grad():
        chain = reference_repaint_chain(ns, ddpm.edm, kw, r, keep, mg.seeded_noise(noise_seed))
        sd_dyn = {k[len("edm.dynamics."):]: v for k, v in ddpm.state_dict().items() if k.startswith("edm.dynamics.")}
        gam = orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])
        assert torch.equal(gam, ddpm.edm.gamma.gamma.detach()), "oracle gamma table differs"
        ocfg = mg.oracle_cfg(hp)
        ocfg.centering = True
        oc = ro.repaint_chain(sd_dyn, ocfg, gam, T, r, kw['x'], kw['h'], kw['node_mask'], kw['fragment_mask'],
                              kw['linker_mask'], kw['edge_mask'], kw['context'], keep_frames=keep,
                              norm_values=tuple(hp['normalize_factors']), noise_fn=mg.seeded_noise(noise_seed))
    err = (oc - chain).abs().max().item()
    assert err == 0.0, f"{name}: oracle vs reference composition {err}"
    # the reference's jump coefficients at this batch size, rows in dl_step_coef order
    jump = torch.zeros((T, 2))
    for row in range(T):
        s = T - 1 - row
        s_arr = torch.full((nb, 1), fill_value=s)
        t_arr = (s_arr + 1) / T
        _, sig, al = ddpm.edm.sigma_and_alpha_t_given_s(ddpm.edm.gamma(t_arr), ddpm.edm.gamma(s_arr / T),
                                                          torch.zeros(nb, 1, 1))
        jump[row, 0], jump[row, 1] = al.reshape(-1)[0], sig.reshape(-1)[0]
    # the same composition in float64: how well-conditioned each molecule's trajectory is
    ddpm64 = ddpm.double()
    kw64 = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
    draw = mg.seeded_noise(noise_seed)
    with torch.no_grad():
        chain64 = reference_repaint_chain(ns, ddpm64.edm, kw64, r, 1, lambda size: draw(size).double())
    nm = kw['node_mask'].float()
    drift = ((chain64[0][..., :3].float() - chain[0][..., :3]) * nm).abs().flatten(1).max(1).values
    types_equal = bool(torch.equal(chain64[0][..., 3:].float(), chain[0][..., 3:]))
    meta = dict(kind="repaint_chain", spec=spec_name, batch=nb, seed=seed, noise_seed=noise_seed, resamplings=r,
                keep_frames=keep, T=T, sha=mg.state_sha(sd_dyn), oracle_max_abs_err=err, fp64_types_equal=types_equal)
    mg.save(name, meta, chain=chain, drift64=drift, jump=jump, **kw)
    print(f"  {name}: drift64 " + " ".join(f"{v:.1e}" for v in drift.tolist()) + f" (types equal: {types_equal})",
          flush=True)


def main():
    torch.set_num_threads(int(os.environ.get("GOLDEN_THREADS", "8")))
    ns = load_reference()
    only = set(sys.argv[1:])
    for name, args in FIXTURES.items():
        if not only or name in only:
            golden_repaint(ns, name, *args)


if __name__ == "__main__":
    main()
