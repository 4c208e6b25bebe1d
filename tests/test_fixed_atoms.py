"""Fixed atoms for the linker sampler: `EDM.sample_chain(..., fixed_atoms=M)`, EDM.fixed_atom_scalars, the DDPM and
sample_many pass-throughs and dl_set_fixed_atoms.

fixed_atoms_oracle restates the loop with replacement in fp64. CPU tests pin the scalar table to start_scalars, check the
binding, the refusals that need no device and the oracle's own properties. GPU tests check that no mask is today's call
bit for bit, every device step against the oracle's step applied to the GPU's own earlier frames (the known-eps
construction of test_sampler_steps_fp64.py), real-weight chains against the fp64 oracle, and the composition with seeds,
start steps, the recovery rounds, clash guidance, solvers, device splits, batch slices, sample_many and DDPM."""
import ctypes as C
import dataclasses
import os

import pytest
import torch

from difflinker_b200 import _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import EDM
import dl_helpers as helpers
import egnn_options_oracle as eo
import fixed_atoms_oracle as fao
import ode_solver_oracle as oso
import test_clash_guidance as tcg
from test_sampler_steps_fp64 import NORM, U, Checker, dev, f64, fc_batch, known_eps_model, oracle_eps, unnorm_frame
from oracle import difflinker_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def half_mask(kw):
    """(B, N) flags on the first half (rounded down) of every molecule's linker rows."""
    lm = kw['linker_mask'].reshape(kw['x'].shape[:2]) != 0
    rank = lm.long().cumsum(1)
    return (lm & (rank <= lm.sum(1, keepdim=True) // 2)).to(torch.int8)


def xh_of(kw, d):
    return torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)


# ---- CPU: the table, the binding, the refusals, the oracle ----------------------------------------------------------

@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("T", [10, 50])
def test_scalar_table_is_start_scalars_row_by_row_and_cached(T, B):
    edm = EDM(None, 8, 3, timesteps=500, noise_schedule='polynomial_2', noise_precision=1e-5)
    edm.T = T
    tab = edm.fixed_atom_scalars(B)
    assert len(tab) == 2 * (T + 1)
    for r in range(T):
        assert (tab[2 * r], tab[2 * r + 1]) == edm.start_scalars(T - 1 - r, B), r
    assert (tab[2 * T], tab[2 * T + 1]) == edm.start_scalars(T, B)
    assert edm.fixed_atom_scalars(B) is tab


def test_binding_and_header():
    lib = _native.load_library()
    assert lib.dl_set_fixed_atoms(None, 1, 1, None, 1, None, None) == -1     # DL_ERR_INVALID before any pointer is read
    assert b"dl_set_fixed_atoms" in lib.dl_last_error()
    with open(os.path.join(ROOT, "include", "difflinker_b200.h")) as f:
        h = f.read()
    assert ("dl_status dl_set_fixed_atoms(dl_engine* e, int32_t B, int32_t N, const int8_t* fixed, int32_t T, "
            "const float* scalars,\n                             void* stream);") in h
    assert _native.SYMBOLS["dl_set_fixed_atoms"][1] == [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                                         C.c_void_p, C.c_void_p]


def cpu_model(inpainting=False):
    spec = synthetic.WorkloadSpec("fixed_refuse", B=3, N=12, n_min=9, l_min=3, l_max=4, F=8, L=1, T=20, seed=3)
    ddpm, _ = helpers.build_ddpm(spec, 0, inpainting=inpainting)
    data = collate(synthetic.make_items(spec))
    return ddpm, data, sampler_inputs(ddpm, data, keep_linker=True)


def test_refusals_without_a_device():
    ddpm, data, kw = cpu_model()
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    good = half_mask(kw)
    with pytest.raises(ValueError, match="tensor for B"):
        edm.sample_chain(**kw, fixed_atoms=good[:, :-1])
    with pytest.raises(ValueError, match="tensor for B"):
        edm.sample_chain(**kw, fixed_atoms=good.tolist())
    frag = (kw['fragment_mask'].reshape(B, N) != 0).to(torch.int8)
    with pytest.raises(ValueError, match="not a linker row"):
        edm.sample_chain(**kw, fixed_atoms=frag)
    pad = (kw['node_mask'].reshape(B, N) == 0)
    if pad.any():
        with pytest.raises(ValueError, match="not a linker row"):
            edm.sample_chain(**kw, fixed_atoms=pad.to(torch.int8))
    h = kw['h'].clone()
    h[good != 0] = 0.5
    with pytest.raises(ValueError, match="one-hot"):
        edm.sample_chain(**dict(kw, h=h), fixed_atoms=good)
    with pytest.raises(ValueError, match="sample_fn"):
        ddpm.sample_chain(data, sample_fn=lambda d: d['linker_mask'].sum(1).view(-1).int(), fixed_atoms=good)
    with pytest.raises(ValueError, match="linker_sizes"):
        ddpm.sample_chain(data, linker_sizes=3, fixed_atoms=good)
    inp, idata, ikw = cpu_model(inpainting=True)
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.edm.sample_chain(**ikw, fixed_atoms=good)


def test_oracle_keeps_every_linker_row_when_all_are_fixed():
    """With every linker row fixed, chain[0] is the input and the state after step s is alpha_s xh + sigma_s nz_s."""
    spec = synthetic.WorkloadSpec("fixed_oracle", B=2, N=10, n_min=8, l_min=2, l_max=3, F=8, L=1, T=12, seed=4)
    dyn, hp = helpers.build_dynamics(spec, 4)
    cfg = helpers.oracle_cfg(hp)
    sd = {k: v.detach().double() for k, v in dyn.state_dict().items()}
    batch = collate(synthetic.make_items(spec))
    nm, fm, lm = (batch[k].double() for k in ('atom_mask', 'fragment_mask', 'linker_mask'))
    em, ctx = batch['edge_mask'].double(), batch['fragment_mask'].double()
    xh = torch.cat([batch['positions'], batch['one_hot'] / 4], 2).double()
    B, N = xh.shape[:2]
    T = spec.T
    edm = EDM(None, 8, 3, timesteps=T, noise_schedule=hp['diffusion_noise_schedule'],
              noise_precision=hp['diffusion_noise_precision'])
    tab = fao.table(edm, B)
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], T, hp['diffusion_noise_precision'])
    draws = helpers.noise_tensor(8, T, B, N, 8).double()
    fwd = lambda t, z: orc.dynamics_forward(sd, cfg, t, z, nm, lm, em, ctx)
    out, zs = fao.sample_ancestral(fwd, xh, draws, fm, lm, lm, gamma, tab, T, B)
    assert torch.equal(out * lm, xh * lm)
    for i, z in enumerate(zs):
        s = T - 1 - i
        want = tab[T - 1 - s, 0] * xh + tab[T - 1 - s, 1] * draws[T - s] * lm
        assert torch.equal(z * lm, want * lm), s
    # a solver's kept rows follow the probability-flow path of the input, alpha_s xh + sigma_s eps_0
    table = oso.table64(gamma, T, 'dpmpp_2m')
    out, zs = fao.sample_ode(fwd, xh, draws[0], fm, lm, lm, table, 'dpmpp_2m', tab, T)
    assert torch.equal(out * lm, xh * lm)
    assert torch.equal(zs[-1] * lm, (tab[T - 1, 0] * xh + tab[T - 1, 1] * draws[0] * lm) * lm)
    # no fixed row: the plain loops
    plain = fao.sample_ancestral(fwd, xh, draws, fm, lm, torch.zeros_like(lm), gamma, tab, T, B)[0]
    z = xh * fm + draws[0] * lm * lm
    for s in range(T - 1, -1, -1):
        z = orc.linker_step(z, fwd(oso.time_feature(s, T), z), orc.step_scalars(gamma, s, T, B, T), draws[T - s], fm, lm)
    sc = orc.step_scalars(gamma, -1, T, B, T)
    assert torch.equal(plain, orc.linker_final(z, fwd(torch.zeros((1, 1), dtype=torch.float64), z), sc, draws[T + 1], fm, lm))


# ---- GPU: no mask is today's call -------------------------------------------------------------------------------------

def small_fc(impl="simt", T=20, B=6, seed=5):
    spec = synthetic.WorkloadSpec("fixed_fc", B=B, N=18, n_min=10, l_min=3, l_max=6, F=8, L=2, T=100, seed=seed)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    d = dev()
    ddpm = ddpm.to(d)
    ddpm.edm.T = T
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    return ddpm, sampler_inputs(ddpm, data, keep_linker=True), data


def pocket(impl="simt", rows=8, known_eps=False):
    ddpm, _ = tcg.build("4A", impl, rows=rows, known_eps=known_eps)
    d = dev()
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(tcg.pocket_items(rows, 2.5)).items()}
    return ddpm, sampler_inputs(ddpm, data, keep_linker=True)


def rows(kw, lo, hi):
    """Molecules [lo, hi) of sampler inputs; the FC edge mask is flattened over (B, N, N)."""
    B = kw['x'].shape[0]
    cut = lambda n, v: (v.reshape(B, -1, *v.shape[1:])[lo:hi].reshape(-1, *v.shape[1:]) if n == 'edge_mask' else v[lo:hi])
    return {n: (None if v is None else cut(n, v)) for n, v in kw.items()}


def launches(edm):
    return int(_native.load_library().dl_launch_count(edm.dynamics.engine(0)))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("graph", ["FC", "4A"])
def test_no_mask_and_an_all_zero_mask_are_todays_call(graph, impl):
    ddpm, kw = (small_fc(impl)[:2] if graph == "FC" else pocket(impl))
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    zero = torch.zeros((B, N, 1), dtype=torch.float32, device=kw['x'].device)
    seeds = list(range(40, 40 + B))
    plain = edm.sample_chain(**kw, keep_frames=4, seeds=seeds)           # the engine exists before counting
    counts = [launches(edm)]
    for m in (None, zero, None):                                         # the same chain
        assert torch.equal(edm.sample_chain(**kw, keep_frames=4, seeds=seeds, fixed_atoms=m), plain)
        counts.append(launches(edm))
    edm.sample_chain(**kw, keep_frames=4, seeds=seeds)
    counts.append(launches(edm))
    steps = [b - a for a, b in zip(counts, counts[1:])]
    assert steps[1:] == [steps[-1]] * 3, steps                           # the same launches as the plain call
    plain = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, nan_retries=1, require_connected=True)
    flags, used = edm.last_connected.clone(), edm.last_seeds.clone()
    for m in (None, zero):                                               # the recovery rounds: flags and seeds too
        got = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, nan_retries=1, require_connected=True, fixed_atoms=m)
        assert torch.equal(got, plain)
        assert torch.equal(edm.last_connected, flags) and torch.equal(edm.last_seeds, used)
    torch.manual_seed(3)                                                 # the batch stream
    a = edm.sample_chain(**kw, keep_frames=2)
    off = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(3)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, fixed_atoms=zero[..., 0]), a)
    assert torch.cuda.default_generators[0].get_offset() == off


# ---- GPU: steps against fp64 with a known eps --------------------------------------------------------------------------

def check_fixed_chain(label, chain, kw, fixed, draws, bias, gamma, tab, T, kind=None, solver=None):
    """Every frame (keep_frames = T) against one oracle step from the GPU's previous frame, on free and kept rows: the free
    rows under check_linker_chain's / check_solver_chain's bound, the kept rows within 2u of their two terms; chain[0]'s kept
    rows equal the input bit for bit."""
    d = chain.device
    chain = f64(chain, d)
    B, N, D = chain.shape[1:]
    nm, fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    fx = f64(fixed, d).reshape(B, N, 1)
    live, kept = nm[..., 0] != 0, fx[..., 0] != 0
    draws = f64(draws, d)
    xh = xh_of(kw, d)
    eps = torch.zeros_like(xh)
    eps[..., 3:] = f64(torch.tensor(bias), d) * nm
    tab = f64(tab, d)
    ck = Checker(label)
    z = fao.start(xh, fm, lm, draws[0], fx, tab, T)
    hist = e_hist = None
    for s in range(T - 1, 0, -1):
        r = T - 1 - s
        if kind is None:
            sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
            a, b, c = (orc._sc(sc, k, z) for k in ("a", "b", "c"))
            n = draws[T - s] * lm
            ref = fao.replace(orc.linker_step(z, eps, sc, draws[T - s], fm, lm), xh, tab[r], n, fx)
            e_free = 4 * U * (z.abs() / a.abs() + (b * eps * lm).abs() + (c * n).abs()) * lm
        else:
            # the step from the GPU's previous frame; the 2M history is the data prediction of the frame before it
            n = draws[0] * lm
            row = f64(solver[r], d)
            second = kind == 'dpmpp_2m' and hist is not None
            zs, xhat = oso.step(z, eps, row, fm, lm, hist if second else None)
            ref = fao.replace(zs, xh, tab[r], n, fx)
            e_x = 8 * U * row[1].abs() * (z.abs() + (row[0] * eps).abs())
            c = row[4] if second else row[3]
            e_free = (8 * U * ((row[2] * z).abs() + (c * xhat).abs() + ((row[5] * hist).abs() if second else 0))
                      + c.abs() * e_x + (row[5].abs() * e_hist if second else 0)) * lm
            hist, e_hist = xhat, e_x
        e_kept = 2 * U * ((tab[r, 0] * xh).abs() + (tab[r, 1] * n).abs())
        got = unnorm_frame(chain[s])
        ck.close(f"kept s={s}", got, ref, e_kept, kept)
        ck.close(f"free s={s}", got, ref, e_free + 1e-300, live & ~kept)
        z = got
    got0 = chain[0]
    assert torch.equal(got0[kept][..., :3], (xh * NORM[0])[kept][..., :3]), f"{label}: a kept row's final x moved"
    assert torch.equal(got0[kept][..., 3:], f64(kw['h'], d)[kept]), f"{label}: a kept row's final type changed"
    ck.record()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [None, "ddim", "dpmpp_2m"])
@pytest.mark.parametrize("source", ["tensor", "seeds"])
def test_every_step_vs_fp64_with_a_known_eps(source, kind):
    F, T = 8, 20
    edm, hp, bias = known_eps_model(F, 50, "auto")
    edm.T = T
    kw = fc_batch([(16, 5), (12, 3), (9, 4), (0, 0), (14, 6)], F, seed=17)
    d = dev()
    kw = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    fixed = half_mask(kw)
    if source == "tensor":
        draws = helpers.noise_tensor(23, T, B, N, F).to(d)
        chain = edm.sample_chain(**kw, keep_frames=T, noise=draws, fixed_atoms=fixed, solver=kind or 'ancestral')
    else:
        seeds = [23 + 7919 * b for b in range(B)]
        parts = []
        for s in seeds:
            torch.cuda.manual_seed(s)
            parts.append(edm.draw_noise(T + 2, 1, N, d))
        draws = torch.cat(parts, dim=1)
        chain = edm.sample_chain(**kw, keep_frames=T, seeds=seeds, fixed_atoms=fixed, solver=kind or 'ancestral')
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], 50, hp['diffusion_noise_precision'])
    solver = None if kind is None else torch.tensor(list(edm.solver_coefficients(kind))).reshape(T + 1, 8)
    check_fixed_chain(f"{kind or 'ancestral'} {source}", chain, kw, fixed, draws, bias, gamma, fao.table(edm, B), T,
                      kind, solver)


# ---- GPU: real weights against the fp64 oracle -------------------------------------------------------------------------
REL_TOL = 1e-4


def rel_err(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.double().abs().max().item(), 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [50, 500])
@pytest.mark.parametrize("case", ["cfg2_zinc", "small_pocket_4A"])
def test_real_weight_chain_vs_fp64_oracle(case, T):
    """cfg2_zinc's model (ZINC shapes: N = 40, F = 8, six layers) on 16 of its molecules, and a 4 A pocket model."""
    spec = helpers.spec_by_name(case)
    if spec.B > 16:
        spec = dataclasses.replace(spec, B=16)
    ddpm, hp = helpers.build_ddpm(spec, 0, diffusion_steps=500)
    d = dev()
    ddpm = ddpm.to(d)
    edm = ddpm.edm
    edm.T = T
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data, keep_linker=True)
    B, N = kw['x'].shape[:2]
    keep = min(T, 50)
    fixed = half_mask(kw)
    noise = helpers.noise_tensor(61, T, B, N, spec.F).to(d)
    chain = edm.sample_chain(**kw, keep_frames=keep, noise=noise, fixed_atoms=fixed)
    cfg = eo.oracle_cfg(hp)
    sd = {k: v.detach() for k, v in edm.dynamics.state_dict().items()}
    fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("fragment_mask", "linker_mask"))
    fx = f64(fixed, d).reshape(B, N, 1)
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], 500, hp['diffusion_noise_precision'])
    fwd = lambda t, z: oracle_eps(sd, cfg, t, z, kw, False, torch.float64, d)
    out, zs = fao.sample_ancestral(fwd, xh_of(kw, d), f64(noise, d), fm, lm, fx, gamma, f64(fao.table(edm, B), d), T, B)
    want0 = orc.final_frame(out, f64(kw['node_mask'], d).reshape(B, N, 1), 3, NORM)
    assert torch.equal(chain[0][..., 3:].double(), want0[..., 3:]), "atom types differ"
    assert rel_err(chain[0][..., :3] * lm, want0[..., :3] * lm) <= REL_TOL
    kept = fx[..., 0] != 0
    assert torch.equal(chain[0][kept].double(), want0[kept])
    unnorm = lambda z: torch.cat([z[..., :3] * NORM[0], z[..., 3:] * NORM[1]], dim=-1)
    frame_of = {(s * keep) // T: s for s in range(T - 1, 0, -1) if (s * keep) // T > 0}
    worst = 0.0
    for f, s in frame_of.items():
        err = rel_err(chain[f], unnorm(zs[T - 1 - s]))
        worst = max(worst, err)
        assert err <= REL_TOL, (f, s, err)
    print(f"{case} T={T}: worst frame rel err {worst:.3g}")


# ---- GPU: composition ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ancestral", "dpmpp_2m"])
def test_rows_equal_their_single_molecule_calls(kind):
    """SIMT edge path: every row of a seeded call, of a per-molecule and of an int start-step call, and of a sample_many
    launch equals the molecule sampled alone with its seed, start step and mask row; a row without kept atoms is the
    plain call's."""
    ddpm, kw, _ = small_fc("simt")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    fixed = half_mask(kw)
    fixed[1] = 0
    seeds = [11 * b + 3 for b in range(B)]
    t0 = [20, 7, 13, 20, 1, 9]
    one = lambda b, **k: edm.sample_chain(**rows(kw, b, b + 1), keep_frames=3, seeds=[seeds[b]], solver=kind,
                                          fixed_atoms=fixed[b:b + 1], **k)[:, 0]
    full = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, solver=kind, fixed_atoms=fixed)
    mixed = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, start_step=t0, solver=kind, fixed_atoms=fixed)
    at12 = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, start_step=12, solver=kind, fixed_atoms=fixed)
    halves = [dict(rows(kw, lo, hi), fixed_atoms=fixed[lo:hi]) for lo, hi in ((0, 2), (2, B))]
    many = edm.sample_many(halves, keep_frames=3, seeds=[seeds[:2], seeds[2:]], start_step=[t0[:2], t0[2:]], solver=kind)
    for b in range(B):
        assert torch.equal(full[:, b], one(b)), b
        alone = one(b, start_step=t0[b])
        assert torch.equal(mixed[:, b], alone), b
        assert torch.equal(many[0 if b < 2 else 1][:, b if b < 2 else b - 2], alone), b
        assert torch.equal(at12[:, b], one(b, start_step=12)), b
    kept = fixed.bool()
    assert torch.equal(full[0][kept], torch.cat([kw['x'], kw['h']], -1)[kept])
    assert not torch.equal(full[0], edm.sample_chain(**kw, keep_frames=3, seeds=seeds, solver=kind)[0])


@pytest.mark.gpu
def test_recovery_rounds_keep_the_fixed_atoms():
    ddpm, kw, _ = small_fc("simt", B=12)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    fixed = half_mask(kw)
    seeds = list(range(500, 500 + B))
    plain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, fixed_atoms=fixed)
    got = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, nan_retries=3, require_connected=True, require_valid=True,
                           fixed_atoms=fixed)
    attempts, used = edm.last_attempts.clone(), edm.last_seeds.clone()
    assert (attempts > 0).any(), "no row was resampled"
    kept = fixed.bool()
    assert torch.equal(got[0][kept], torch.cat([kw['x'], kw['h']], -1)[kept])
    for b in range(B):
        if attempts[b] == 0:
            assert torch.equal(got[:, b], plain[:, b]), b
        else:
            alone = edm.sample_chain(**rows(kw, b, b + 1), keep_frames=2, seeds=[int(used[b])], fixed_atoms=fixed[b:b + 1])
            assert torch.equal(got[:, b], alone[:, 0]), b


@pytest.mark.gpu
def test_clash_guidance_moves_only_free_linker_atoms():
    """The kept rows' frames are those of the unguided call bit for bit (they do not depend on the free rows), the free
    linker rows move, and a split over devices=[0, 0] is the one-slice chain."""
    ddpm, kw = pocket("simt", rows=8)
    edm = ddpm.edm
    T = edm.T
    B = kw['x'].shape[0]
    fixed = half_mask(kw)
    assert fixed.any()
    seeds = list(range(700, 700 + B))
    plain = edm.sample_chain(**kw, keep_frames=T, seeds=seeds, fixed_atoms=fixed)
    guided = edm.sample_chain(**kw, keep_frames=T, seeds=seeds, fixed_atoms=fixed, clash_guidance=(0.8, T))
    kept = fixed.bool()
    free = (kw['linker_mask'].reshape(kept.shape) != 0) & ~kept
    assert torch.equal(guided[:, kept], plain[:, kept])
    assert not torch.equal(guided[:, free], plain[:, free])
    edm.devices = [0, 0]
    try:
        split = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, fixed_atoms=fixed, clash_guidance=(0.8, T))
    finally:
        edm.devices = None
    assert torch.equal(split, edm.sample_chain(**kw, keep_frames=2, seeds=seeds, fixed_atoms=fixed,
                                               clash_guidance=(0.8, T)))


@pytest.mark.gpu
def test_batch_slices_and_the_batch_stream():
    """batch_slice=(b0, B): the slice's rows of the batch stream and its mask rows give the full call's rows."""
    ddpm, kw, _ = small_fc("simt")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    fixed = half_mask(kw)
    torch.manual_seed(21)
    full = edm.sample_chain(**kw, keep_frames=2, fixed_atoms=fixed)
    torch.manual_seed(21)
    part = edm.sample_chain(**rows(kw, 2, 5), keep_frames=2, fixed_atoms=fixed[2:5], batch_slice=(2, B))
    assert torch.equal(part, full[:, 2:5])


@pytest.mark.gpu
def test_ddpm_sample_chain_and_sample_many_keep_the_batch_linker_atoms():
    ddpm, kw, data = small_fc("simt")
    B = kw['x'].shape[0]
    fixed = half_mask(kw)
    seeds = list(range(80, 80 + B))
    chain, nm = ddpm.sample_chain(data, keep_frames=2, seeds=seeds, fixed_atoms=fixed)
    assert torch.equal(chain, ddpm.edm.sample_chain(**kw, keep_frames=2, seeds=seeds, fixed_atoms=fixed))
    seeds2 = list(range(90, 90 + B))
    many = ddpm.sample_many([data, data], keep_frames=2, seeds=[seeds, seeds2], fixed_atoms=[fixed, None])
    assert torch.equal(many[0][0], chain)
    assert torch.equal(many[1][0], ddpm.sample_chain(data, keep_frames=2, seeds=seeds2)[0])


@pytest.mark.gpu
def test_setter_refusals_on_an_engine():
    ddpm, kw, _ = small_fc("auto")
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    B, N = kw['x'].shape[:2]
    T = edm.T
    fixed = half_mask(kw).contiguous()
    tab = edm.fixed_atom_scalars(B)
    assert lib.dl_set_fixed_atoms(eng, 0, N, fixed.data_ptr(), T, tab, None) == -1
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), 0, tab, None) == -1
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), T, None, None) == -1
    bad = list(tab)
    bad[5] = float('inf')
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), T, (C.c_float * len(bad))(*bad), None) == -1
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), T, tab, None) == 0
    seeds = list(range(B))
    edm.T = T - 1                                                        # refused at the call, which clears it
    try:
        with pytest.raises(_native.NativeError, match="dl_set_fixed_atoms"):
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    finally:
        edm.T = T
    plain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds)             # cleared: today's call
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), T, tab, None) == 0
    assert not torch.equal(edm.sample_chain(**kw, keep_frames=1, seeds=seeds), plain)
    # the device vetting of the call: a flag on a fragment row, a kept row that is not a one-hot
    frag = (kw['fragment_mask'].reshape(B, N) != 0).to(torch.int8).contiguous()
    assert lib.dl_set_fixed_atoms(eng, B, N, frag.data_ptr(), T, tab, None) == 0
    with pytest.raises(_native.NativeError, match="not a live linker row"):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    h = kw['h'].clone()
    h[fixed.bool()] = 0.25
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), T, tab, None) == 0
    with pytest.raises(_native.NativeError, match="one-hot"):
        edm.sample_chain(**dict(kw, h=h), keep_frames=1, seeds=seeds)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=1, seeds=seeds), plain)
