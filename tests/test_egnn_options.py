"""EGNN options of the reference trainer: `tanh` (bounded coordinate update, egnn.py:104-105), `sin_embedding`
(sinusoidal distance features, egnn.py:281-292) and `aggregation_method='mean'` (egnn.py:315-319). CPU tests pin the
option-aware oracle against fixtures of the live reference (tools/make_golden_opts.py) and the host plumbing; GPU tests run both edge paths against those fixtures."""
import ctypes as C
import hashlib

import pytest
import torch

from difflinker_b200 import DDPM, Dynamics, EDM, synthetic
from difflinker_b200.batching import collate, create_templates_for_linker_generation
import dl_helpers as helpers
import egnn_options_oracle as eo
from oracle import difflinker_oracle as orc

REL_TOL = 1e-4
IMPLS = ["simt", "auto"]
ALL = eo.options_kw(True, True, True)


def build_dynamics(spec_name, tanh, mean, sin, seed, edge_impl='auto'):
    return helpers.build_dynamics(eo.spec_with_options(spec_name, tanh, mean, sin), seed, edge_impl=edge_impl,
                                  **eo.options_kw(tanh, mean, sin))


def build_ddpm(spec_name, tanh, mean, sin, seed, edge_impl='auto', **over):
    spec = eo.spec_with_options(spec_name, tanh, mean, sin)
    return helpers.build_ddpm(spec, seed, edge_impl=edge_impl, **over)


def rel_err(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.double().abs().max().item(), 1e-30)


def dyn_fixture(name, edge_impl='auto'):
    meta, a = helpers.load_golden(name)
    spec_name, tanh, mean, sin, _, seed = eo.DYN_FIXTURES[name]
    dyn, hp = build_dynamics(spec_name, tanh, mean, sin, seed, edge_impl)
    assert helpers.state_sha(dyn.state_dict()) == meta["sha"], "parameters differ from the reference's under the same seed"
    return meta, a, dyn, hp


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", list(eo.DYN_FIXTURES))
def test_oracle_dynamics_matches_option_fixtures(name):
    meta, a, dyn, hp = dyn_fixture(name)
    with torch.no_grad():
        out = eo.dynamics_forward(dyn.state_dict(), eo.oracle_cfg(hp), a["t"], a["xh"], a["node_mask"], a["linker_mask"],
                                   a["edge_mask"], a["context"])
    assert (out - a["out"]).abs().max().item() < 2e-6


def test_mean_fixtures_cover_padding_and_an_isolated_row():
    meta, a = helpers.load_golden("dyn_opts_mean_pocket_4A")
    nm = a["node_mask"].reshape(a["xh"].shape[0], -1)
    assert (nm.sum(1) < nm.shape[1]).any(), "no padded molecule"
    x = a["xh"][1, :, :3]
    i = meta["isolated_row"]
    others = torch.cat([x[:i], x[i + 1:]])[nm[1].bool()[torch.arange(nm.shape[1]) != i]]
    assert nm[1, i] == 1 and (others - x[i]).norm(dim=1).min() > 4.0


@pytest.mark.parametrize("name", list(eo.CHAIN_FIXTURES))
def test_oracle_chains_match_option_fixtures(name):
    meta, a = helpers.load_golden(name)
    spec_name, tanh, mean, sin, nb, seed, keep, inpaint = eo.CHAIN_FIXTURES[name]
    ddpm, hp = build_ddpm(spec_name, tanh, mean, sin, seed, inpainting=inpaint)
    assert helpers.state_sha(ddpm.edm.dynamics.state_dict()) == meta["sha"]
    sd = {k[len("edm.dynamics."):]: v for k, v in ddpm.state_dict().items() if k.startswith("edm.dynamics.")}
    spec = eo.OPTION_SPECS[spec_name]
    gam = orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])
    data = orc.collate_molecules(synthetic.make_items(spec, batch=nb))
    cfg = eo.oracle_cfg(hp)
    with torch.no_grad():
        if inpaint:
            cfg.centering = True
            x = orc.remove_partial_mean(data['positions'], data['atom_mask'], data['atom_mask'])
            got = eo.inpainting_sample_chain(sd, cfg, gam, meta["T"], x, data['one_hot'], data['atom_mask'],
                                              data['fragment_mask'], data['linker_mask'], data['edge_mask'],
                                              data['fragment_mask'], keep_frames=keep, noise_fn=helpers.seeded_noise(meta["noise_seed"]))
        else:
            tpl = orc.linker_templates(data, data['linker_mask'].sum(1).view(-1).int())
            x = orc.remove_partial_mean(tpl['positions'], tpl['atom_mask'], tpl['fragment_mask'])
            got = eo.edm_sample_chain(sd, cfg, gam, meta["T"], x, tpl['one_hot'], tpl['atom_mask'], tpl['fragment_mask'],
                                       tpl['linker_mask'], tpl['edge_mask'], tpl['fragment_mask'], keep_frames=keep,
                                       noise_fn=helpers.seeded_noise(meta["noise_seed"]))
    assert (got - a["chain"]).abs().max().item() < 5e-5


def test_options_construct_with_the_reference_parameter_layout():
    """tanh and mean change no parameter: state_dict keys, shapes and construction order (hence the seeded weights) are the
    default model's. sin_embedding widens every edge_mlp.0 / coord_mlp.0 to 2H + 24 inputs and nothing else. The fixtures'
    sha256 check that the seeded weights equal the reference's in every case."""
    kw = dict(n_dims=3, in_node_nf=8, context_node_nf=1, hidden_nf=128, n_layers=3)
    torch.manual_seed(0)
    ref = Dynamics(**kw)
    torch.manual_seed(0)
    opt = Dynamics(**kw, tanh=True, aggregation_method='mean')
    assert opt.tanh and opt.aggregation_method == 'mean'
    assert [(k, v.shape) for k, v in ref.state_dict().items()] == [(k, v.shape) for k, v in opt.state_dict().items()]
    assert helpers.state_sha(ref.state_dict()) == helpers.state_sha(opt.state_dict())
    emb = Dynamics(**kw, **ALL)
    wide = {k for k, v in emb.state_dict().items() if v.shape != ref.state_dict()[k].shape}
    assert list(emb.state_dict()) == list(ref.state_dict())
    assert wide == {k for k in ref.state_dict() if k.endswith(("edge_mlp.0.weight", "coord_mlp.0.weight"))}
    assert all(emb.state_dict()[k].shape == (128, 280) for k in wide)
    n = sum(v.numel() for v in ref.state_dict().values())
    assert sum(v.numel() for v in emb.state_dict().values()) == n + len(wide) * 128 * 22
    o = emb.egnn_options()
    assert (o.tanh, o.coords_range, o.sin_embedding, o.aggregation) == (1, 15.0, 1, 1)
    assert ref.egnn_options().is_default() and not opt.egnn_options().is_default()


def test_sin_embedding_frequencies_are_the_references():
    """The kernels use f_k = 0x1.aceeap-2 * 4^k (common.cuh sin_freq); the reference computes
    2 * math.pi * 4 ** torch.arange(6) / 15 in fp32 (egnn.py:284)."""
    import math
    f = 2 * math.pi * 4 ** torch.arange(6) / 15.
    assert f.dtype == torch.float32
    assert f.tolist() == [float.fromhex("0x1.aceeap-2") * 4 ** k for k in range(6)]


def test_remaining_unsupported_options_still_refuse():
    for kw in (dict(attention=True), dict(model='gnn_dynamics'), dict(aggregation_method='max')):
        with pytest.raises(NotImplementedError):
            Dynamics(n_dims=3, in_node_nf=8, context_node_nf=1, hidden_nf=128, **kw)
    with pytest.raises(NotImplementedError):
        EDM(dynamics=None, in_node_nf=8, n_dims=3, noise_schedule='learned')


def test_load_from_checkpoint_carries_the_options(tmp_path):
    spec = eo.spec_with_options("small_fc", True, True, True)
    src, hp = helpers.build_ddpm(spec, 3)
    path = str(tmp_path / "opts.ckpt")
    torch.save({"hyper_parameters": hp, "state_dict": src.state_dict()}, path)
    m = DDPM.load_from_checkpoint(path, strict=True)
    dyn = m.edm.dynamics
    assert dyn.tanh is True and dyn.aggregation_method == 'mean' and dyn.sin_embedding is True
    assert m.state_dict()["edm.dynamics.dynamics.e_block_0.gcl_equiv.coord_mlp.0.weight"].shape == (128, 280)
    assert helpers.state_sha(m.state_dict()) == helpers.state_sha(src.state_dict())


def _job_inputs(ddpm, nb=3):
    from difflinker_b200.ddpm import sampler_inputs
    data = collate(synthetic.make_items(eo.OPTION_SPECS["small_fc"], batch=nb))
    return sampler_inputs(ddpm, data)


def test_job_files_default_models_keep_version_one_options_write_version_two(tmp_path):
    from difflinker_b200 import _native, export_job
    plain, _ = build_ddpm("small_fc", False, False, False, 3)
    opts, _ = build_ddpm("small_fc", True, True, False, 3)
    kw = _job_inputs(plain)
    p1, p2 = str(tmp_path / "a.bin"), str(tmp_path / "b.bin")
    export_job.write_job(p1, plain.edm, **kw, keep_frames=2, seed=1)
    export_job.write_job(p2, opts.edm, **kw, keep_frames=2, seed=1)
    b1, b2 = open(p1, "rb").read(), open(p2, "rb").read()
    # the bytes the exporter wrote for this default model before the options existed
    assert hashlib.sha256(b1).hexdigest() == "1b8a2f862895a9b852fc350cdb8b71d3a17dbeb164b832bee80f25a60cd0d7cd"
    assert b1[:8] == b"DLJOB1\0\0" and b2[:8] == b"DLJOB2\0\0"
    # version 2 is version 1 with the 16-byte dl_egnn_options after the 52-byte dl_config
    assert b2[8:60] == b1[8:60] and b2[76:] == b1[60:]
    o = _native.DLEgnnOptions.from_buffer_copy(b2[60:76])
    assert (o.tanh, o.coords_range, o.sin_embedding, o.aggregation) == (1, 15.0, 0, 1)


# ---------------------------------------------------------------------------------------------------------------- GPU
def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def run_dyn(dyn, t, z, nm, lm, em, ctx, device):
    mv = lambda v: None if v is None else v.to(device)
    return dyn(mv(t), mv(z), mv(nm), mv(lm), mv(em), mv(ctx)).cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", list(eo.DYN_FIXTURES))
def test_dynamics_forward_matches_option_fixtures(name, impl):
    meta, a, dyn, hp = dyn_fixture(name, impl)
    out = run_dyn(dyn, a["t"], a["xh"], a["node_mask"], a["linker_mask"], a["edge_mask"], a["context"], dev())
    assert rel_err(out[..., :3], a["out"][..., :3]) <= REL_TOL
    assert rel_err(out[..., 3:], a["out"][..., 3:]) <= REL_TOL
    assert torch.equal(out * (1 - a["node_mask"].float()), torch.zeros_like(out))


def _chain_tolerance_check(chain, want, mask, drift64=None):
    """Coordinates within 1e-4 relative; for a fixture that records the reference's own fp32-vs-fp64 drift per molecule, within
    max(1e-4 * scale, 30 * drift64) per molecule (DESIGN.md section 2)."""
    err = ((chain[..., :3] - want[..., :3]) * mask).abs().flatten(1).max(1).values
    scale = (want[..., :3] * mask).abs().max().item()
    tol = torch.full_like(err, REL_TOL * scale)
    if drift64 is not None:
        tol = torch.maximum(tol, 30.0 * drift64.float())
    assert (err <= tol).all(), (err.tolist(), tol.tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_sample_chain_matches_option_fixture(impl):
    meta, a = helpers.load_golden("chain_opts_all_cfg1")
    spec_name, tanh, mean, sin, nb, seed, keep, _ = eo.CHAIN_FIXTURES["chain_opts_all_cfg1"]
    ddpm, hp = build_ddpm(spec_name, tanh, mean, sin, seed, edge_impl=impl)
    spec = eo.OPTION_SPECS[spec_name]
    d = dev()
    data = collate(synthetic.make_items(spec, batch=nb))
    tpl = create_templates_for_linker_generation(data, data['linker_mask'].sum(1).view(-1).int())
    B, N = tpl['positions'].shape[:2]
    noise = helpers.noise_tensor(meta["noise_seed"], meta["T"], B, N, spec.F)
    from difflinker_b200 import utils
    x = utils.remove_partial_mean_with_mask(tpl['positions'], tpl['atom_mask'], tpl['fragment_mask'])
    mv = lambda v: v.to(d)
    chain = ddpm.edm.sample_chain(x=mv(x), h=mv(tpl['one_hot']), node_mask=mv(tpl['atom_mask']),
                                  fragment_mask=mv(tpl['fragment_mask']), linker_mask=mv(tpl['linker_mask']),
                                  edge_mask=mv(tpl['edge_mask']), context=mv(tpl['fragment_mask']),
                                  keep_frames=keep, noise=mv(noise)).cpu()
    want = a["chain"]
    assert chain.shape == want.shape
    assert torch.equal(chain[0][..., 3:], want[0][..., 3:]), "atom types differ"
    _chain_tolerance_check(chain[0], want[0], tpl['linker_mask'], a["drift64"])
    for f in range(1, keep):
        assert rel_err(chain[f], want[f]) <= REL_TOL, f


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_inpainting_sample_chain_matches_option_fixture(impl):
    meta, a = helpers.load_golden("inpaint_chain_opts_tanh_mean_cfg1")
    spec_name, tanh, mean, sin, nb, seed, keep, _ = eo.CHAIN_FIXTURES["inpaint_chain_opts_tanh_mean_cfg1"]
    ddpm, hp = build_ddpm(spec_name, tanh, mean, sin, seed, edge_impl=impl, inpainting=True)
    spec = eo.OPTION_SPECS[spec_name]
    d = dev()
    data = collate(synthetic.make_items(spec, batch=nb))
    B, N = data['positions'].shape[:2]
    noise = helpers.inpaint_noise_tensor(meta["noise_seed"], meta["T"], B, N, spec.F, data['atom_mask'], data['fragment_mask'])
    from difflinker_b200 import utils
    x = utils.remove_partial_mean_with_mask(data['positions'], data['atom_mask'], data['atom_mask'])
    mv = lambda v: v.to(d)
    chain = ddpm.edm.sample_chain(x=mv(x), h=mv(data['one_hot']), node_mask=mv(data['atom_mask']),
                                  fragment_mask=mv(data['fragment_mask']), linker_mask=mv(data['linker_mask']),
                                  edge_mask=mv(data['edge_mask']), context=mv(data['fragment_mask']),
                                  keep_frames=keep, noise=mv(noise)).cpu()
    want = a["chain"]
    assert torch.equal(chain[0][..., 3:], want[0][..., 3:]), "atom types differ"
    for f in range(keep):
        assert rel_err(chain[f], want[f]) <= REL_TOL, f


@pytest.mark.gpu
@pytest.mark.parametrize("tanh,mean,sin", [(True, False, False), (False, True, False), (False, False, True),
                                          (True, True, True)])
def test_simt_and_wgmma_agree_with_options_vs_oracle(tanh, mean, sin):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    batch = collate(synthetic.make_items(spec, batch=16))
    z, t = helpers.random_latent(batch, 5)
    outs = {}
    for impl in ("simt", "wgmma"):
        dyn, hp = helpers.build_dynamics(spec, 0, edge_impl=impl, **eo.options_kw(tanh, mean, sin))
        outs[impl] = run_dyn(dyn, t, z, batch['atom_mask'], batch['linker_mask'], batch['edge_mask'], batch['fragment_mask'], dev())
    hp.update(eo.options_kw(tanh, mean, sin))
    with torch.no_grad():
        want = eo.dynamics_forward(dyn.state_dict(), eo.oracle_cfg(hp), t, z, batch['atom_mask'], batch['linker_mask'],
                                    batch['edge_mask'], batch['fragment_mask'])
    assert rel_err(outs["wgmma"], outs["simt"]) <= 2e-5
    for o in outs.values():
        assert rel_err(o[..., :3], want[..., :3]) <= REL_TOL
        assert rel_err(o[..., 3:], want[..., 3:]) <= REL_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("graph_type", ["4A", "FC-10A-4A"])
def test_mean_counts_on_cutoff_graphs_with_isolated_and_chunked_rows(graph_type, impl):
    """'mean' divides by each row's degree in the cut-off graph: padded molecules, and under FC-10A-4A ligand rows with more
    than 128 neighbours (the tensor-core path's chunk tiles, whose degree travels in the tile header). The isolated pocket
    rows only guard against a zero divisor: their sums are exactly 0 whatever they are divided by."""
    base = synthetic.SPECS["cfg4_pockets"]
    spec = synthetic.WorkloadSpec(base.name, B=3, N=base.N, n_min=280, l_min=base.l_min, l_max=base.l_max, F=base.F, L=2,
                                  T=10, seed=7, pocket=base.pocket, graph_type=graph_type)
    dyn, hp = helpers.build_dynamics(spec, 1, edge_impl=impl, **ALL)
    batch = collate(synthetic.make_items(spec, batch=3))
    assert (batch['atom_mask'].sum(1) < spec.N).any()
    z, t = helpers.random_latent(batch, 17, pad_garbage=False)
    pk = torch.nonzero(batch['pocket_mask'][1, :, 0] > 0).view(-1)[:5]
    for k, idx in enumerate(pk.tolist()):
        z[1, idx, :3] = torch.tensor([200.0 + 50.0 * k, -150.0, 90.0])
    ctx = helpers.context_of(batch, spec)
    hp.update(ALL)
    with torch.no_grad():
        want = eo.dynamics_forward(dyn.state_dict(), eo.oracle_cfg(hp), t, z, batch['atom_mask'], batch['linker_mask'],
                                    batch['edge_mask'], ctx)
    got = run_dyn(dyn, t, z, batch['atom_mask'], batch['linker_mask'], batch['edge_mask'], ctx, dev())
    assert rel_err(got[..., :3], want[..., :3]) <= REL_TOL
    assert rel_err(got[..., 3:], want[..., 3:]) <= REL_TOL
    if graph_type == "FC-10A-4A" and impl == "auto":
        from difflinker_b200 import _native
        stats = (C.c_int64 * 4)()
        _native.check(_native.load_library().dl_cut_graph_stats(dyn.engine(0), stats), "dl_cut_graph_stats")
        assert stats[1] > stats[0], "no row with more than 128 neighbours"


@pytest.mark.gpu
def test_e3_equivariance_with_options():
    spec = helpers.EXTRA_SPECS["small_fc"]
    dyn, hp = helpers.build_dynamics(spec, 6, **ALL)
    batch = collate(synthetic.make_items(spec))
    z, t = helpers.random_latent(batch, 8, pad_garbage=False)
    g = torch.Generator().manual_seed(1)
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    z2 = z.clone()
    z2[..., :3] = (z[..., :3] @ q.T + torch.tensor([1.5, -2.0, 0.7])) * batch['atom_mask'].float()
    a = run_dyn(dyn, t, z, batch['atom_mask'], batch['linker_mask'], batch['edge_mask'], batch['fragment_mask'], dev())
    b = run_dyn(dyn, t, z2, batch['atom_mask'], batch['linker_mask'], batch['edge_mask'], batch['fragment_mask'], dev())
    assert (b[..., :3] - a[..., :3] @ q.T).abs().max().item() <= 2e-4 * max(a[..., :3].abs().max().item(), 1e-3)
    assert rel_err(b[..., 3:], a[..., 3:]) <= 2e-4


def _ragged_ddpm(inpainting=False):
    spec = eo.spec_with_options("opts_cfg1", True, True, True)
    spec = synthetic.WorkloadSpec("opts_ragged", B=7, N=40, n_min=24, l_min=3, l_max=12, F=8, L=3, T=12, seed=2,
                                  hparams=spec.hparams)
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=inpainting)
    d = dev()
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=7)).items()}
    return ddpm, data, d


@pytest.mark.gpu
@pytest.mark.parametrize("inpainting", [False, True])
@pytest.mark.parametrize("world", [2, 3])
def test_batch_slices_with_options_reproduce_the_single_gpu_chain(world, inpainting):
    from difflinker_b200.ddpm import sampler_inputs
    from difflinker_b200.distributed import shard_range, slice_sampler_inputs
    ddpm, data, d = _ragged_ddpm(inpainting)
    torch.manual_seed(5)
    full, _ = ddpm.sample_chain(data, keep_frames=2)
    kw = sampler_inputs(ddpm, data)
    parts = []
    for r in range(world):
        lo, hi = shard_range(7, r, world)
        torch.manual_seed(5)
        parts.append(ddpm.edm.sample_chain(**slice_sampler_inputs(kw, lo, hi), keep_frames=2, batch_slice=(lo, 7)))
    assert torch.equal(torch.cat(parts, dim=1), full)


@pytest.mark.gpu
@pytest.mark.parametrize("inpainting", [False, True])
def test_plain_c_caller_samples_a_version_two_job(tmp_path, inpainting):
    import subprocess
    from difflinker_b200 import export_job
    from difflinker_b200.ddpm import sampler_inputs
    ddpm, data, d = _ragged_ddpm(inpainting)
    kw = sampler_inputs(ddpm, data)
    seed = 20240607
    torch.manual_seed(seed)
    gen = torch.cuda.default_generators[d.index or 0]
    off0 = gen.get_offset()
    want = ddpm.edm.sample_chain(**kw, keep_frames=3).cpu()
    job, out = str(tmp_path / "job.bin"), str(tmp_path / "out.bin")
    meta = export_job.write_job(job, ddpm.edm, **kw, keep_frames=3, seed=seed, offset=off0, device_index=d.index or 0)
    assert open(job, "rb").read(8) == b"DLJOB2\0\0"
    exe = helpers.build_c_example(tmp_path)
    res = subprocess.run([exe, job, out], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, (res.stdout, res.stderr)
    status, consumed, chain, flags = export_job.read_result(out, meta["B"], meta["N"], meta["keep_frames"], meta["xd"])
    assert status == 0 and not flags.any()
    assert consumed == gen.get_offset() - off0
    assert torch.equal(chain, want)
