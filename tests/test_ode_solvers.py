"""ODE solvers for the linker sampler: `EDM.sample_chain(..., solver='ddim' | 'dpmpp_2m')`, `edm.solver`,
EDM.solver_coefficients and dl_set_solver.

ode_solver_oracle restates the update in fp64. CPU tests pin the solver table to the fp64 closed form rounded once, check
the refusals and the binding, and measure the order of convergence of the oracle's solvers. GPU tests check every step of
the device loop against the oracle's step applied to the GPU's own earlier frames (the known-eps construction of
test_sampler_steps_fp64.py), whole real-weight chains against the fp64 oracle, that 'ancestral' is today's call bit for
bit, and the composition with seeds, start steps, sample_many, the recovery rounds, clash guidance and device splits."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, molecule_builder as mb, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import EDM
import clash_guidance_oracle as cgo
import dl_helpers as helpers
import egnn_options_oracle as eo
import ode_solver_oracle as oso
import test_clash_guidance as tcg
from test_sampler_steps_fp64 import (NORM, U, Checker, dev, f64, fc_batch, known_eps_model, oracle_eps, pocket_batch,
                                     sample, stored_steps, unnorm_frame)
from oracle import difflinker_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["ddim", "dpmpp_2m"]


def bare_edm(schedule, timesteps, T):
    edm = EDM(None, 8, 3, timesteps=timesteps, noise_schedule=schedule, noise_precision=1e-5)
    edm.T = T
    return edm


# ---- CPU: the table, the refusals, the binding --------------------------------------------------------------------

@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("T", [10, 20, 50, 500])
@pytest.mark.parametrize("schedule", ["polynomial_2", "cosine"])
def test_solver_table_is_the_fp64_closed_form_rounded_once(schedule, T, kind):
    edm = bare_edm(schedule, 500, T)
    got = torch.tensor(list(edm.solver_coefficients(kind)), dtype=torch.float32).reshape(T + 1, 8)
    want = oso.table64(orc.gamma_table(schedule, 500, 1e-5), T, kind, 500)
    assert torch.equal(got, want.float())
    assert (want[:T, 6] > 0).all()
    assert torch.equal(got[0, 4], got[0, 3]) and got[0, 5] == 0           # row 0 is first order for both kinds
    if kind == 'ddim':
        assert torch.equal(got[:, 4], got[:, 3]) and (got[:, 5] == 0).all()
    assert edm.solver_coefficients(kind) is edm.solver_coefficients(kind)   # cached
    # the gamma entries are step_coefficients' own: its time feature and sigma_t agree with the table's row
    coef = edm.step_coefficients(T, 1)
    for r in (0, T // 2, T - 1):
        s = T - 1 - r
        assert coef[r].t == float(torch.tensor((s + 1) / T, dtype=torch.float32))


def test_solver_refusals():
    spec = synthetic.WorkloadSpec("ode_refuse", B=2, N=10, n_min=8, l_min=2, l_max=3, F=8, L=1, T=20, seed=3)
    ddpm, _ = helpers.build_ddpm(spec, 0)
    kw = sampler_inputs(ddpm, collate(synthetic.make_items(spec)))
    for bad in ('rk4', 'DDIM', ('ddim',), 2):
        with pytest.raises(ValueError, match="solver"):
            ddpm.edm.sample_chain(**kw, solver=bad)
    with pytest.raises(ValueError, match="solver"):
        ddpm.sample_chain(collate(synthetic.make_items(spec)), solver='euler')
    ddpm.edm.solver = 'heun'
    with pytest.raises(ValueError, match="solver"):
        ddpm.edm.sample_chain(**kw)
    ddpm.edm.solver = 'ancestral'
    ddpm.edm.T = 21                                                     # above the schedule's 20 timesteps
    with pytest.raises(ValueError, match="timesteps"):
        ddpm.edm.sample_chain(**kw, solver='dpmpp_2m')
    with pytest.raises(ValueError):
        ddpm.edm.solver_coefficients('ancestral')
    inp, _ = helpers.build_ddpm(spec, 0, inpainting=True)
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.edm.sample_chain(**kw, solver='ddim')
    inp.edm.solver = 'dpmpp_2m'
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.edm.sample_chain(**kw)


def test_binding_and_header():
    lib = _native.load_library()
    assert lib.dl_set_solver(None, _native.SOLVERS['ddim'], 10, None) == -1    # DL_ERR_INVALID before any pointer is read
    assert b"dl_set_solver" in lib.dl_last_error()
    with open(os.path.join(ROOT, "include", "difflinker_b200.h")) as f:
        h = f.read()
    assert "DL_SOLVER_ANCESTRAL = 0, DL_SOLVER_DDIM = 1, DL_SOLVER_DPMPP_2M = 2" in h
    assert _native.SOLVERS == {"ancestral": 0, "ddim": 1, "dpmpp_2m": 2}
    assert "dl_status dl_set_solver(dl_engine* e, int32_t kind, int32_t T, const float* table);" in h


# Order of convergence on the fp64 oracle: an FC model with the synthetic weights, one fixed start, the final continuous
# (x, h) on the linker rows at K = 25, 50 and 100 steps against K = 500. The loop starts from a fixed z at t = 0.6
# (start_step = 0.6 K, q(z_t0 | x) of one draw): from z_T, the first step of the schedule's uniform t grid covers a lambda
# interval that shrinks only like log K (alpha_T = 3e-3), and an untrained network's data prediction is of order 1/alpha_T
# there, so that step's error swamps the rest at any K a test can afford. Measured here: error ratios per doubling
# (25 -> 50, 50 -> 100) of 2.10 and 2.25 for 'ddim', 4.84 and 4.80 for 'dpmpp_2m' (polynomial_2, timesteps 1000).
CONV_RATIO = {'ddim': (1.7, 2.6), 'dpmpp_2m': (3.5, math.inf)}


@pytest.mark.parametrize("kind", KINDS)
def test_order_of_convergence_on_the_fp64_oracle(kind):
    spec = synthetic.WorkloadSpec("conv", B=2, N=10, n_min=8, l_min=3, l_max=4, F=8, L=2, T=1000, seed=31)
    dyn, hp = helpers.build_dynamics(spec, 31)
    cfg = helpers.oracle_cfg(hp)
    sd = {k: v.detach().double() for k, v in dyn.state_dict().items()}
    batch = collate(synthetic.make_items(spec))
    nm, fm, lm = (batch[k].double() for k in ('atom_mask', 'fragment_mask', 'linker_mask'))
    em, ctx = batch['edge_mask'].double(), batch['fragment_mask'].double()
    xh = torch.cat([batch['positions'], batch['one_hot'] / 4], 2).double()
    gamma = orc.gamma_table('polynomial_2', 1000, 1e-5)
    g = float(orc.gamma_lookup(gamma, torch.tensor([[0.6]]), 1000)[0, 0])
    n0 = torch.randn(xh.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    z0 = xh * fm + (math.sqrt(1 / (1 + math.exp(g))) * xh + math.sqrt(1 / (1 + math.exp(-g))) * n0) * lm
    fwd = lambda t, z: orc.dynamics_forward(sd, cfg, t, z, nm, lm, em, ctx)
    run = lambda K: oso.sample(fwd, z0, oso.table64(gamma, K, kind), kind, K, fm, lm, t0=K * 3 // 5)[0]
    ref = run(500)
    errs = [((run(K) - ref) * lm).abs().max().item() for K in (25, 50, 100)]
    ratios = [errs[0] / errs[1], errs[1] / errs[2]]
    print(f"{kind}: errors {errs}, ratios {ratios}")
    lo, hi = CONV_RATIO[kind]
    assert all(lo <= r <= hi for r in ratios), ratios


# ---- GPU: steps against fp64 with a known eps ----------------------------------------------------------------------

def solver_table32(edm, kind):
    return torch.tensor(list(edm.solver_coefficients(kind)), dtype=torch.float32).reshape(edm.T + 1, 8)


def check_solver_chain(label, chain, kw, z_start, e_start, bias, table, kind, T, keep, t0=None):
    """Every stored frame against oso.step applied in fp64 to the GPU's own earlier state, with the fp32 table the GPU used.
    The bound per element: the incoming error times the step's gains, plus 8u times every term of the step (the data
    prediction's two roundings and the update's products and sums). z_start is the fp64 start (z_T or z_t0) and e_start its
    bound. The final row is checked as the composite z_1 -> z_0 -> x, and atom types where the fp64 gap is decided."""
    d = chain.device
    chain = f64(chain, d)
    B, N, D = chain.shape[1:]
    nm, fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    live, lk, fr = nm[..., 0] != 0, lm[..., 0] != 0, fm[..., 0] != 0
    eps = torch.zeros((B, N, D), dtype=torch.float64, device=d)
    eps[..., 3:] = f64(torch.tensor(bias), d) * nm
    tab = f64(table, d)
    frame_of = {s: f for f, s in stored_steps(T, keep).items()}
    ck = Checker(label)
    assert torch.equal(chain[:, ~live], torch.zeros_like(chain[:, ~live])), f"{label}: a padded row is not 0"
    t0 = T if t0 is None else t0
    z, e, hist, e_hist = z_start, e_start, None, None
    for s in range(t0 - 1, -1, -1):
        row = tab[T - 1 - s]
        st, ia, r, c1, c2a, c2b = (row[i] for i in range(6))
        second = kind == 'dpmpp_2m' and hist is not None
        ref, xhat = oso.step(z, eps, row, fm, lm, hist if second else None)
        e_x = ia.abs() * e + 8 * U * ia.abs() * (z.abs() + (st * eps).abs())
        c = c2a if second else c1
        rnd = 8 * U * ((r * z).abs() + (c * xhat).abs() + ((c2b * hist).abs() if second else 0))
        e = ((r.abs() * e + c.abs() * e_x + (c2b.abs() * e_hist if second else 0) + rnd) * lm + e * fm)
        z, hist, e_hist = ref, xhat, e_x
        if s in frame_of:
            got = unnorm_frame(chain[frame_of[s]])
            assert torch.equal(got[fr & ~lk], z_start[fr & ~lk]), f"{label}: a fragment row of frame {frame_of[s]} moved"
            ck.close(f"step s={s}", got, z, e, live)
            # continue from the GPU's own state; its history is the data prediction of the frame before
            z, e = got, torch.zeros_like(e)
    row = tab[T]
    out = oso.final(z, eps, row, fm, lm)
    e_f = (row[1].abs() * e + 8 * U * row[1].abs() * (z.abs() + (row[0] * eps).abs())) * lm
    got = chain[0]
    assert torch.equal(got[..., :3][fr & ~lk], z_start[..., :3][fr & ~lk]), f"{label}: a final fragment row moved"
    ck.close("final x", got[..., :3], out[..., :3] * NORM[0], e_f[..., :3] * NORM[0] + 1e-300, live)
    ck.types("final h", got[..., 3:], out[..., 3:], e_f[..., 3:], live, nm[..., 0])
    ck.record()


# label -> (F, molecule sizes (atoms, linker atoms), T, table T, keep_frames, draws); as test_sampler_steps_fp64's cases
SOLVER_FC = {
    "F8_T20_tensor": (8, [(16, 5), (12, 3), (9, 4), (0, 0), (16, 16)], 20, 50, 20, "tensor"),
    "F9_T50_stream": (9, [(24, 6), (15, 4), (1, 1)], 50, 200, 50, "stream"),
    "F13_T10_seeds": (13, [(19, 5), (10, 0), (14, 6)], 10, 10, 10, "seeds"),
    "F8_T20_keep4_seeds": (8, [(11, 3), (6, 2), (9, 4)], 20, 50, 4, "seeds"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", list(SOLVER_FC))
def test_solver_steps_vs_fp64(case, impl, kind):
    F, sizes, T, table_T, keep, source = SOLVER_FC[case]
    edm, hp, bias = known_eps_model(F, table_T, impl)
    edm.T = T
    edm.solver = kind                                                   # the attribute path, as reference call sites use it
    kw = fc_batch(sizes, F, seed=len(sizes) * 100 + F)
    chain, draws = sample(edm, kw, T, keep, source, 23, False)
    d = chain.device
    B, N = chain.shape[1:3]
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("fragment_mask", "linker_mask"))
    z_T = xh * fm + (f64(draws[0], d) * lm) * lm
    check_solver_chain(f"{kind} {case} {impl}", chain, kw, z_T, torch.zeros_like(z_T), bias, solver_table32(edm, kind),
                       kind, T, keep)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("graph", ["4A", "FC-10A-4A"])
def test_pocket_solver_steps_vs_fp64(graph, kind):
    F, T = 9, 20
    edm, hp, bias = known_eps_model(F, 100, "auto", graph_type=graph)
    edm.T = T
    kw = pocket_batch([(6, 40, 5), (5, 28, 7)], F, seed=7)
    d = dev()
    kwd = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    draws = helpers.noise_tensor(31, T, B, N, F).to(d)
    chain = edm.sample_chain(**kwd, keep_frames=T, noise=draws, solver=kind)
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("fragment_mask", "linker_mask"))
    z_T = xh * fm + (f64(draws[0], d) * lm) * lm
    check_solver_chain(f"{kind} pocket {graph}", chain, kw, z_T, torch.zeros_like(z_T), bias, solver_table32(edm, kind),
                       kind, T, T)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_scalar_start_step_starts_first_order(kind):
    """From start_step t0 the loop's first step is first order: the check's oracle uses c1 there, and a second-order
    update from a stale history would be far outside the bound. z_t0 = xh fm + (alpha xh + sigma n) lm in fp32 on the
    device carries 3u of its terms."""
    F, T, t0 = 8, 30, 12
    edm, hp, bias = known_eps_model(F, 50, "auto")
    edm.T = T
    kw = fc_batch([(16, 5), (12, 3), (9, 4)], F, seed=41)
    d = dev()
    kwd = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    draws = helpers.noise_tensor(43, t0, B, N, F).to(d)
    edm.sample_chain(**kwd, keep_frames=T, noise=helpers.noise_tensor(44, T, B, N, F).to(d), solver='dpmpp_2m')
    chain = edm.sample_chain(**kwd, keep_frames=T, noise=draws, start_step=t0, solver=kind)
    al, sg = edm.start_scalars(t0, B)
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("fragment_mask", "linker_mask"))
    n0 = f64(draws[0], d) * lm
    z0 = xh * fm + (al * xh + sg * n0) * lm
    e0 = 3 * U * ((al * xh).abs() + (sg * n0).abs()) * lm
    check_solver_chain(f"{kind} start_step {t0}", chain, kw, z0, e0, bias, solver_table32(edm, kind), kind, T, T, t0=t0)


# ---- GPU: real weights against the fp64 oracle ---------------------------------------------------------------------
# Whole chains from the same z_T (draw 0 of an injected noise tensor) against the oracle's solver loop in fp64 on the
# option-aware oracle forward, under the tolerance of test_gpu_parity's chain checks: 1e-4 of the largest magnitude on
# every frame and on the final linker coordinates, atom types identical.
REL_TOL = 1e-4
REAL = {"cfg1_plumbing": "cfg1_plumbing", "pocket_4A": "small_pocket_4A", "pocket_FC-10A-4A": "small_pocket_FC-10A-4A"}


def rel_err(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.double().abs().max().item(), 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [20, 50])
@pytest.mark.parametrize("case", list(REAL))
def test_real_weight_chain_vs_fp64_oracle(case, K, kind):
    spec = helpers.spec_by_name(REAL[case])
    ddpm, hp = helpers.build_ddpm(spec, 0, diffusion_steps=500)
    d = dev()
    ddpm = ddpm.to(d)
    edm = ddpm.edm
    edm.T = K
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    noise = helpers.noise_tensor(61, K, B, N, spec.F).to(d)
    chain = edm.sample_chain(**kw, keep_frames=K, noise=noise, solver=kind)
    cfg = eo.oracle_cfg(hp)
    sd = {k: v.detach() for k, v in edm.dynamics.state_dict().items()}
    fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("fragment_mask", "linker_mask"))
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    z_T = xh * fm + (f64(noise[0], d) * lm) * lm
    fwd = lambda t, z: oracle_eps(sd, cfg, t, z, kw, False, torch.float64, d)
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], 500, hp['diffusion_noise_precision'])
    out, zs = oso.sample(fwd, z_T, oso.table64(gamma, K, kind, 500), kind, K, fm, lm)
    want0 = orc.final_frame(out, f64(kw['node_mask'], d).reshape(B, N, 1), 3, NORM)
    assert torch.equal(chain[0][..., 3:].double(), want0[..., 3:]), "atom types differ"
    assert rel_err(chain[0][..., :3] * lm, want0[..., :3] * lm) <= REL_TOL
    unnorm = lambda z: torch.cat([z[..., :3] * NORM[0], z[..., 3:] * NORM[1]], dim=-1)
    worst = 0.0
    for f in range(1, K):
        err = rel_err(chain[f], unnorm(zs[K - 1 - f]))
        worst = max(worst, err)
        assert err <= REL_TOL, (f, err)
    print(f"{case} K={K} {kind}: worst frame rel err {worst:.3g}")


# ---- GPU: identities and composition ---------------------------------------------------------------------------------

def small_fc(impl="simt", T=20, B=6):
    spec = synthetic.WorkloadSpec("ode_fc", B=B, N=18, n_min=10, l_min=2, l_max=6, F=8, L=2, T=100, seed=5)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    d = dev()
    ddpm = ddpm.to(d)
    ddpm.edm.T = T
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    return ddpm, sampler_inputs(ddpm, data), spec


def rows(kw, lo, hi):
    """Molecules [lo, hi) of sampler inputs; the FC edge mask is flattened over (B, N, N)."""
    B = kw['x'].shape[0]
    cut = lambda n, v: (v.reshape(B, -1, *v.shape[1:])[lo:hi].reshape(-1, *v.shape[1:]) if n == 'edge_mask' else v[lo:hi])
    return {n: (None if v is None else cut(n, v)) for n, v in kw.items()}


@pytest.mark.gpu
def test_ancestral_is_todays_call_and_seeds_replay_bit_for_bit():
    ddpm, kw, _ = small_fc("auto")
    edm = ddpm.edm
    lib = _native.load_library()
    seeds = list(range(300, 306))
    count = lambda: int(lib.dl_launch_count(edm.dynamics.engine(0)))
    edm.sample_chain(**kw, keep_frames=4, seeds=seeds)                  # the engine exists before counting
    n0 = count()
    plain = edm.sample_chain(**kw, keep_frames=4, seeds=seeds)
    n1 = count()
    named = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, solver='ancestral')
    n2 = count()
    ode = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, solver='dpmpp_2m')
    assert n2 - n1 == n1 - n0 and count() - n2 == n1 - n0              # the solver adds no launch
    assert torch.equal(plain, named)
    assert not torch.equal(ode[0, ..., :3], plain[0, ..., :3])
    assert torch.equal(edm.sample_chain(**kw, keep_frames=4, seeds=seeds, solver='dpmpp_2m'), ode)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=4, seeds=seeds), plain)   # the engine is back to ancestral
    # the batch stream: the generator advances by the ancestral loop's draws
    torch.manual_seed(5)
    a = edm.sample_chain(**kw, keep_frames=2)
    off_a = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(5)
    b = edm.sample_chain(**kw, keep_frames=2, solver='ddim')
    assert torch.cuda.default_generators[0].get_offset() == off_a
    torch.manual_seed(5)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, solver='ddim'), b)
    assert not torch.equal(a, b)
    # noise_mode='per_molecule' samples the same streams as seeds
    edm.noise_mode = 'per_molecule'
    torch.manual_seed(9)
    pm = edm.sample_chain(**kw, keep_frames=2, solver='dpmpp_2m')
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, seeds=edm.last_seeds, solver='dpmpp_2m'), pm)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_rows_equal_their_single_molecule_calls(kind):
    """The per-molecule rule under the solver, on the SIMT edge path: every row of a seeded call, of a sample_many launch and
    of a per-molecule start-step call equals the molecule sampled alone with its seed (and start step)."""
    ddpm, kw, _ = small_fc("simt")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = [11 * b + 3 for b in range(B)]
    t0 = [20, 7, 13, 20, 1, 9]
    one = lambda b, **k: edm.sample_chain(**rows(kw, b, b + 1), keep_frames=2, seeds=[seeds[b]], solver=kind, **k)
    full = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, solver=kind)
    mixed = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, start_step=t0, solver=kind)
    halves = [rows(kw, lo, hi) for lo, hi in ((0, 2), (2, B))]
    many = edm.sample_many(halves, keep_frames=2, seeds=[seeds[:2], seeds[2:]], start_step=[t0[:2], t0[2:]], solver=kind)
    for b in range(B):
        assert torch.equal(full[:, b], one(b)[:, 0]), b
        alone = one(b, start_step=t0[b])[:, 0]
        assert torch.equal(mixed[:, b], alone), b
        assert torch.equal(many[0 if b < 2 else 1][:, b if b < 2 else b - 2], alone), b


@pytest.mark.gpu
def test_recovery_rounds_resample_with_the_solver():
    """nan_retries with require_connected: the resampled rows are the solver's chains of their round's seeds, the rows
    round 0 kept are the plain solver call's."""
    ddpm, kw, _ = small_fc("simt", B=12)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(500, 500 + B))
    plain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, solver='dpmpp_2m')
    got = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=3, require_connected=True, solver='dpmpp_2m')
    attempts, used = edm.last_attempts.clone(), edm.last_seeds.clone()
    assert (attempts > 0).any(), "no row was resampled"
    for b in range(B):
        if attempts[b] == 0:
            assert torch.equal(got[:, b], plain[:, b]), b
        else:
            alone = edm.sample_chain(**rows(kw, b, b + 1), keep_frames=1, seeds=[int(used[b])], solver='dpmpp_2m')
            assert torch.equal(got[:, b], alone[:, 0]), b


@pytest.mark.gpu
def test_clash_guidance_pushes_the_solver_step_and_splits_equal_one_slice():
    """Known eps (eps_x = 0): on the coordinates the 2M step is z_s = r z_t + c2a ia z_t + c2b ia' z_{t'} from the GPU's own
    frames (keep_frames = T; the history is the data prediction of the state k_finish read, before guidance moved it,
    which the frame holds after). At a guided step the frame must be the clash oracle's push of that step, within
    test_clash_guidance's bound; then devices=[0, 0] must give the one-slice chain bit for bit."""
    ddpm, kw = tcg.build("4A", "simt", known_eps=True)
    edm = ddpm.edm
    T = tcg.T_LOOP
    B, N = kw['x'].shape[:2]
    K, scale = 6, 0.8
    noise = helpers.noise_tensor(5, T, B, N, 9).to(kw['x'].device)
    guided = edm.sample_chain(**kw, keep_frames=T, noise=noise, clash_guidance=(scale, K), solver='dpmpp_2m').cpu()
    tab = solver_table32(edm, 'dpmpp_2m').double()
    table = mb.clash_table(edm.is_geom)
    nm, lm, fm = (kw[k].reshape(B, N).cpu() for k in ('node_mask', 'linker_mask', 'fragment_mask'))
    po = kw['context'][..., -1].reshape(B, N).cpu()
    pushed = 0
    for s in range(1, min(K, T - 2)):
        row = tab[T - 1 - s]
        prev = tab[T - 2 - s]
        zt, zp = guided[s + 1, ..., :3].double(), guided[s + 2, ..., :3].double()
        zs = zt * fm[..., None] + (row[2] * zt + (row[4] * row[1] * zt + row[5] * prev[1] * zp)) * lm[..., None]
        types = cgo.first_argmax(guided[s, ..., 3:3 + table.shape[0]].numpy())
        want, moved, bound, slack = cgo.push(zs.numpy(), types, nm.numpy(), lm.numpy(), po.numpy(), table.numpy(), scale)
        linker, _ = cgo.rows(nm.numpy(), lm.numpy(), po.numpy())
        step_bound = 8 * cgo.U * (np.abs(row[2].item() * zt.numpy()) + np.abs(row[4].item() * row[1].item() * zt.numpy())
                                  + np.abs(row[5].item() * prev[1].item() * zp.numpy())).max(-1)
        tol = 2 * (step_bound * (1 + scale * 50) + bound) + 1e-30
        got = guided[s, ..., :3].double().numpy()
        judged = linker & (slack > 1e-3)
        err = np.abs(got - want).max(-1)
        assert (err[judged] <= tol[judged]).all(), (s, (err[judged] / tol[judged]).max())
        pushed += int((judged & moved).sum())
    assert pushed > 5, pushed
    seeds = list(range(700, 700 + B))
    one = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, clash_guidance=(scale, K), solver='dpmpp_2m')
    edm.devices = [0, 0]
    try:
        split = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, clash_guidance=(scale, K), solver='dpmpp_2m')
    finally:
        edm.devices = None
    assert torch.equal(split, one)


@pytest.mark.gpu
def test_setter_refusals_on_an_engine():
    ddpm, kw, _ = small_fc("auto")
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    T = edm.T
    good = edm.solver_coefficients('dpmpp_2m')
    assert lib.dl_set_solver(eng, 3, T, good) == -1
    assert lib.dl_set_solver(eng, 2, T, None) == -1
    assert lib.dl_set_solver(eng, 2, 0, good) == -1
    bad = list(good)
    bad[8 * 3 + 1] = float('nan')
    assert lib.dl_set_solver(eng, 2, T, (C.c_float * len(bad))(*bad)) == -1
    bad = list(good)
    bad[8 * 4 + 6] = 0.0
    assert lib.dl_set_solver(eng, 2, T, (C.c_float * len(bad))(*bad)) == -1
    # accepted, then refused at a call of another T and by the inpainting sampler's engine
    assert lib.dl_set_solver(eng, 2, T, good) == 0
    try:
        edm.T = T - 1
        with pytest.raises(_native.NativeError, match="dl_set_solver"):
            edm.sample_chain(**kw, keep_frames=1, seeds=list(range(kw['x'].shape[0])))
    finally:
        lib.dl_set_solver(eng, 0, 0, None)
        edm.T = T


@pytest.mark.gpu
def test_linker_size_redraws_with_the_solver():
    """ddpm.sample_chain(linker_sizes=...) with the recovery rounds under 'dpmpp_2m' (SIMT path): rows round 0 kept are the
    plain solver call's, and a recovered row, sizes included, is its molecule sampled alone with the seed recorded for it."""
    import test_seeded_linker_sizes as tsl
    ddpm, data = tsl.model_and_data("fc", "simt")
    edm = ddpm.edm
    nn = tsl.size_model(tsl.dev(), [0, 1, 2], bias=[-1.0, 0.5, 0.2])
    seeds = tsl.SEEDS
    base, _ = ddpm.sample_chain(data, linker_sizes=nn, seeds=seeds, keep_frames=2, solver='dpmpp_2m')
    chain, nm = ddpm.sample_chain(data, linker_sizes=nn, seeds=seeds, keep_frames=2, nan_retries=3,
                                  require_connected=True, solver='dpmpp_2m')
    attempts, used, sizes = edm.last_attempts.clone(), edm.last_seeds.clone(), edm.last_sizes.clone()
    assert (attempts > 0).any() and (attempts == 0).any(), attempts.tolist()
    for b in range(len(seeds)):
        if attempts[b] == 0:
            assert torch.equal(chain[:, b], base[:, b]), b
            continue
        alone, nm_b = ddpm.sample_chain(tsl.rows_of(data, [b]), linker_sizes=nn, seeds=[int(used[b])], keep_frames=2,
                                        solver='dpmpp_2m')
        assert int(edm.last_sizes[0]) == int(sizes[b]), b
        n = nm_b.shape[1]
        assert torch.equal(chain[:, b, :n], alone[:, 0]), b
