"""Partial diffusion: EDM.sample_chain(start_step=t0) varies the linker a batch holds -- q(z_t0 | x) on the linker, then the
plain reverse loop from step t0 down to 0.

CPU: argument checks, the oracle (tests/partial_diffusion_oracle.py) against the reference's goldens (partial_*.npz,
tools/make_golden_partial.py), DDPM's template with the batch's own linker, the launch-planning key and the C-ABI.
GPU, on both edge paths: the goldens, every stored state against fp64 with the exact-dynamics construction of
test_sampler_steps_fp64.py, the three noise sources, the recovery rounds and sample_many."""
import math
import os
import shutil
import subprocess

import pytest
import torch

from difflinker_b200 import _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.distributed import plan_launches
from difflinker_b200.edm import retry_seed, seeds_tensor
from difflinker_b200.utils import FoundNaNException
import dl_helpers as helpers
import partial_diffusion_oracle as po
import test_sampler_steps_fp64 as steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = [f"partial_cfg2_zinc_t{t0}_k{k}" for t0 in (1, 50, 250, 500) for k in (1, 10)] + ["partial_cfg4_pockets_t100_k1"]
INPUTS = ("x", "h", "node_mask", "fragment_mask", "linker_mask", "edge_mask", "context")


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def golden_model(meta, impl='auto'):
    spec = synthetic.SPECS[meta["spec"]]
    ddpm, hp = helpers.build_ddpm(spec, meta["seed"], edge_impl=impl, diffusion_steps=meta["table_timesteps"])
    assert helpers.state_sha(ddpm.edm.dynamics.state_dict()) == meta["sha"], "seeded weights differ from the fixture's"
    ddpm.edm.T = meta["T"]
    return ddpm, hp, spec


def cfg1_model(**over):
    ddpm, hp = helpers.build_ddpm(synthetic.SPECS["cfg1_plumbing"], 0, **over)
    data = collate(synthetic.make_items(synthetic.SPECS["cfg1_plumbing"]))
    return ddpm, data


# ---- CPU ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bad", [1.5, True, "3", -1, 21, 10 ** 12])
def test_start_step_must_be_an_int_in_0_to_T(bad):
    ddpm, data = cfg1_model()
    ddpm.edm.T = 20
    kw = sampler_inputs(ddpm, data)
    with pytest.raises(ValueError, match="start_step"):
        ddpm.edm.sample_chain(**kw, start_step=bad)
    with pytest.raises(ValueError, match="start_step"):
        ddpm.edm.sample_many([kw], seeds=[[0] * kw['x'].shape[0]], start_step=bad)


def test_sample_fn_and_inpainting_refuse_a_start_step():
    ddpm, data = cfg1_model()
    with pytest.raises(ValueError, match="sample_fn"):
        ddpm.sample_chain(data, sample_fn=lambda d: d['linker_mask'].sum(1).view(-1).int(), start_step=3)
    with pytest.raises(ValueError, match="sample_fn"):
        ddpm.sample_many([data], sample_fn=lambda d: d['linker_mask'].sum(1).view(-1).int(), start_step=3)
    inp, data = cfg1_model(inpainting=True)
    kw = sampler_inputs(inp, data)
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.edm.sample_chain(**kw, start_step=3)
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.sample_chain(data, start_step=0)


def test_ddpm_template_keeps_the_batch_linker_and_refuses_one_elsewhere():
    """sampler_inputs with the batch's own linker equals the inputs the reference composition sampled (stored in the
    fixtures), and a batch whose linker rows do not follow the fragment rows is refused."""
    for name in ("partial_cfg2_zinc_t1_k1", "partial_cfg4_pockets_t100_k1"):
        meta, a = helpers.load_golden(name)
        ddpm, hp, spec = golden_model(meta)
        if meta["moad_val_dataset"]:
            ddpm.val_dataset = type("MOADDataset", (list,), {})()
        data = collate(synthetic.make_items(spec, batch=meta["batch"]))
        kw = sampler_inputs(ddpm, data, keep_linker=True)
        for k in INPUTS:
            assert torch.equal(kw[k], a[k]), (name, k)
        assert not torch.equal(sampler_inputs(ddpm, data)["x"], kw["x"])   # the plain template has no linker
    ddpm, data = cfg1_model()
    moved = dict(data)
    moved['linker_mask'] = data['linker_mask'].roll(1, dims=1)
    with pytest.raises(ValueError, match="linker rows"):
        ddpm.sample_chain(moved, start_step=3)


@pytest.mark.parametrize("name", ["partial_cfg2_zinc_t1_k1", "partial_cfg2_zinc_t1_k10", "partial_cfg2_zinc_t50_k1",
                                  "partial_cfg2_zinc_t50_k10"])
def test_oracle_matches_the_reference_composition(name):
    """The oracle replays the reference's composition exactly (the longer fixtures were pinned when they were generated)."""
    meta, a = helpers.load_golden(name)
    ddpm, hp, spec = golden_model(meta)
    gam = steps.gamma_of(hp)
    with torch.no_grad():
        chain = po.linker_partial_chain(ddpm.edm.dynamics.state_dict(), helpers.oracle_cfg(hp), gam, meta["T"], meta["t0"],
                                        *(a[k] for k in INPUTS), keep_frames=meta["keep_frames"],
                                        norm_values=tuple(hp['normalize_factors']),
                                        noise_fn=helpers.seeded_noise(meta["noise_seed"]))
    assert (chain - a["chain"]).abs().max().item() == 0.0
    alpha, sigma = ddpm.edm.start_scalars(meta["t0"], meta["batch"])
    assert (alpha, sigma) == (meta["alpha_t0"], meta["sigma_t0"])
    written = po.written_frames(meta["t0"], meta["T"], meta["keep_frames"])
    for f in range(meta["keep_frames"]):
        assert (f in written) or not a["chain"][f].any(), f


def test_start_scalars_are_edm_forwards_and_key_the_launch_plan():
    ddpm, _ = cfg1_model()
    edm = ddpm.edm
    gam = edm.gamma.gamma.detach()
    for t0 in (0, 1, 7, edm.T):
        for B in (1, 31, 32, 64):
            a, s = po.start_scalars(gam, t0, edm.T, B, edm.gamma.timesteps)
            assert edm.start_scalars(t0, B) == (float(a[0]), float(s[0]))
    sizes, nodes = [3, 3, 40, 3, 40], [30, 31, 30, 32, 30]
    coefs, starts, keys = edm._launch_keys(sizes, nodes, 2, 5)
    assert starts[3] == (5,) + edm.start_scalars(5, 3) and starts[40] == (5,) + edm.start_scalars(5, 40)
    for k, b in enumerate(sizes):
        assert keys[k][1] == starts[b]
    for ks, _ in plan_launches(sizes, nodes, 256, keys):
        assert len({keys[k] for k in ks}) == 1
        assert len({(bytes(coefs[sizes[k]]), starts[sizes[k]]) for k in ks}) == 1
    _, starts_none, keys_none = edm._launch_keys(sizes, nodes, 2, None)
    assert set(starts_none.values()) == {None} and [k[1] for k in keys_none] == [None] * len(sizes)


def test_library_exports_the_setter_and_the_header_compiles_as_c99(tmp_path):
    lib = _native.load_library()
    assert hasattr(lib, "dl_set_start_step") and "dl_set_start_step" in _native.SYMBOLS
    assert lib.dl_set_start_step(None, 5, 1.0, 0.0) == -1               # DL_ERR_INVALID: no engine
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "start.c"
    src.write_text('#include "difflinker_b200.h"\n'
                   "int main(void) {\n"
                   "  dl_status s = dl_set_start_step((dl_engine*)0, 5, 1.0f, 0.0f);\n"
                   "  return s == DL_ERR_INVALID ? 0 : 1;\n"
                   "}\n")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib_dir = os.path.dirname(_native.LIB_PATH)
    exe = str(tmp_path / "start")
    res = subprocess.run([gcc, "-std=c99", "-Wall", str(src), "-I" + os.path.join(ROOT, "include"),
                          "-L" + lib_dir, "-ldifflinker_b200", "-L" + os.path.join(cuda, "lib64"), "-lcudart",
                          "-Wl,-rpath," + lib_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    assert subprocess.run([exe]).returncode == 0


# ---- GPU: the goldens ---------------------------------------------------------------------------------------------------

def per_molecule_ok(got, want, rows, drift, scale):
    """The repository's per-molecule rule: max(1e-4 * scale, 30 * drift64) per molecule, at least half inside 1e-4 * scale."""
    err = ((got - want) * rows).abs().flatten(1).max(1).values
    tol = torch.maximum(torch.full_like(err, 1e-4 * scale), 30.0 * drift.float())
    assert (err <= tol).all(), (err.tolist(), tol.tolist())
    assert (err <= 1e-4 * scale).sum() >= (err.numel() + 1) // 2, (err.tolist(), 1e-4 * scale)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("name", GOLDENS)
def test_chain_matches_the_reference_golden(name, impl):
    meta, a = helpers.load_golden(name)
    ddpm, hp, spec = golden_model(meta, impl)
    d = dev()
    ddpm = ddpm.to(d)
    t0, keep, T = meta["t0"], meta["keep_frames"], meta["T"]
    B, N = a["x"].shape[:2]
    noise = helpers.noise_tensor(meta["noise_seed"], t0, B, N, spec.F)  # t0 + 2 draws
    kw = {k: a[k].to(d) for k in INPUTS}
    chain = ddpm.edm.sample_chain(**kw, keep_frames=keep, noise=noise.to(d), start_step=t0).cpu()
    want = a["chain"]
    assert chain.shape == want.shape
    nm, fm, lm = (a[k].float() for k in ("node_mask", "fragment_mask", "linker_mask"))
    assert torch.equal(chain[0][..., 3:], want[0][..., 3:]), "atom types differ"
    fr = (fm[..., 0] != 0) & (lm[..., 0] == 0)
    assert torch.equal(chain[0][..., :3][fr], a["x"][fr]), "a fragment row differs from the input"
    assert not chain[:, nm[..., 0] == 0].any(), "a padded row is not 0"
    written = po.written_frames(t0, T, keep)
    for f in range(keep):
        if f not in written:
            assert not chain[f].any(), f"frame {f} has no writer and is not 0"
            continue
        x_got, x_want = chain[f][..., :3], want[f][..., :3]
        per_molecule_ok(x_got, x_want, lm, a["drift64"], want[f][..., :3].abs().max().item())
        if f > 0:
            assert torch.equal(chain[f][fr], want[f][fr])


# ---- GPU: step by step against fp64 ------------------------------------------------------------------------------------

# label -> (F, molecule sizes (atoms, linker atoms), T, table T, t0, draws); B * N = 33, 95 and 48 nodes (1, 15, 0 mod 16)
CASES = {
    "t0_0": (8, [(11, 3), (6, 2), (9, 9)], 50, 50, 0, "tensor"),
    "t0_1": (13, [(19, 5), (1, 1), (0, 0), (10, 0), (14, 6)], 50, 50, 1, "seeds"),
    "t0_half": (1, [(12, 4), (1, 1), (0, 0), (7, 0)], 50, 50, 25, "stream"),
    "t0_T_nsteps": (8, [(11, 3), (6, 2), (9, 4)], 20, 50, 20, "tensor"),
    "t0_T_seeds": (13, [(19, 5), (1, 1), (0, 0), (10, 0), (14, 6)], 30, 30, 30, "seeds"),
    "t0_half_stream": (8, [(11, 3), (6, 2), (9, 9)], 40, 40, 20, "stream"),
}


def sample_partial(edm, kw, t0, keep, source, seed):
    """(chain, draws): the chain from step t0 and the t0 + 2 draws it must have used (see steps.sample)."""
    d = dev()
    kw = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    F = edm.in_node_nf
    if source == "tensor":
        draws = helpers.noise_tensor(seed, t0, B, N, F).to(d)
        return edm.sample_chain(**kw, keep_frames=keep, noise=draws, start_step=t0), draws
    if source == "seeds":
        seeds = [seed + 7919 * b for b in range(B)]
        parts = []
        for s in seeds:
            torch.cuda.manual_seed(s)
            parts.append(edm.draw_noise(t0 + 2, 1, N, d))
        return edm.sample_chain(**kw, keep_frames=keep, seeds=seeds, start_step=t0), torch.cat(parts, dim=1)
    gen = torch.cuda.default_generators[d.index or 0]
    torch.manual_seed(seed)
    draws = edm.draw_noise(t0 + 2, B, N, d)
    end = gen.get_offset()
    torch.manual_seed(seed)
    chain = edm.sample_chain(**kw, keep_frames=keep, start_step=t0)
    assert gen.get_offset() == end, "the batch stream must advance by t0 + 2 draws"
    return chain, draws


def check_partial_chain(label, chain, kw, draws, bias, gamma, T, t0, start):
    """steps.check_linker_chain from q(z_t0 | x): z_{t0-1} against the fp64 step of the fp64 start, every later stored state
    against the fp64 step of the GPU's previous one, the final step likewise; frames at or above t0 exactly 0."""
    d = chain.device
    chain = steps.f64(chain, d)
    keep, B, N, D = chain.shape
    U = steps.U
    nm, fm, lm = (steps.f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    live, lk, fr = nm[..., 0] != 0, lm[..., 0] != 0, fm[..., 0] != 0
    draws = steps.f64(draws, d)
    xh = torch.cat([steps.f64(kw['x'], d) / steps.NORM[0], steps.f64(kw['h'], d) / steps.NORM[1]], dim=2)
    eps = torch.zeros_like(xh)
    eps[..., 3:] = steps.f64(torch.tensor(bias), d) * nm
    al = torch.full((B, 1), start[1], dtype=torch.float64, device=d)
    sg = torch.full((B, 1), start[2], dtype=torch.float64, device=d)
    eps_t = draws[0] * lm
    z = po.partial_start(xh, eps_t, al, sg, fm, lm)
    # fp32 start: alpha*xh, sigma*eps and their sum each rounded once (the masks are 0 or 1)
    e = 4 * U * ((al[:, :, None] * xh).abs() + (sg[:, :, None] * eps_t).abs()) * lm
    sc = steps.scalars(gamma, T, B)
    frame_of = {s: f for f, s in steps.stored_steps(T, keep).items() if s < t0}
    for f in range(1, keep):
        if f not in frame_of.values():
            assert not chain[f].any(), f"{label}: frame {f} has no writer below t0 and is not 0"
    ck = steps.Checker(label)
    assert torch.equal(chain[:, ~live], torch.zeros_like(chain[:, ~live])), f"{label}: a padded row is not 0"
    for s in range(t0 - 1, -1, -1):
        a, b, c = (helpers.orc._sc(sc[s], k, z) for k in ("a", "b", "c"))
        n = draws[t0 - s]
        ref = helpers.orc.linker_step(z, eps, sc[s], n, fm, lm)
        e = (e / a.abs() + 4 * U * ((z.abs() + e) / a.abs() + (b * eps * lm).abs() + (c * n * lm).abs())) * lm + e * fm
        z = ref
        if s in frame_of:
            got = steps.unnorm_frame(chain[frame_of[s]])
            assert torch.equal(got[fr & ~lk], xh[fr & ~lk]), f"{label}: a fragment row of frame {frame_of[s]} is not the input"
            ck.close(f"step s={s}", got, z, e, live)
            z, e = got, torch.zeros_like(e)
    inv_a0, sig0, snr0 = (helpers.orc._sc(sc[-1], k, z) for k in ("inv_alpha0", "sigma0", "snr0"))
    n = draws[t0 + 1]
    out = helpers.orc.linker_final(z, eps, sc[-1], n, fm, lm)
    e = (inv_a0 * e + 4 * U * (inv_a0 * (z.abs() + e) + inv_a0 * (sig0 * eps * lm).abs() + (snr0 * n * lm).abs())) * lm
    got = chain[0]
    assert torch.equal(got[..., :3][fr & ~lk], xh[..., :3][fr & ~lk]), f"{label}: a final fragment row is not the input"
    ck.close("final x", got[..., :3], out[..., :3] * steps.NORM[0], e[..., :3] * steps.NORM[0], live)
    ck.types("final h", got[..., 3:], out[..., 3:], e[..., 3:], live, nm[..., 0])
    ck.record()


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", list(CASES))
def test_partial_steps_vs_fp64(case, impl):
    F, sizes, T, table_T, t0, source = CASES[case]
    edm, hp, bias = steps.known_eps_model(F, table_T, impl)
    edm.T = T
    kw = steps.fc_batch(sizes, F, seed=len(sizes) * 100 + F)
    B = kw['x'].shape[0]
    start = edm._start(t0, B)
    chain, draws = sample_partial(edm, kw, t0, T, source, 23)
    check_partial_chain(f"partial {case} {impl} {source}", chain, kw, draws, bias, steps.gamma_of(hp), T, t0, start)


# ---- GPU: noise streams, recovery, sample_many --------------------------------------------------------------------------

def zinc_model(impl, T=12, rows=7, gain=1.0):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    if gain != 1.0:
        with torch.no_grad():
            for name, p in ddpm.named_parameters():
                if name.endswith("coord_mlp.4.weight"):
                    p.mul_(gain)
    ddpm.edm.T = T
    d = dev()
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=rows)).items()}
    return ddpm, data, sampler_inputs(ddpm, data, keep_linker=True)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_batch_stream_equals_its_tensor_and_advances_t0_plus_2_draws(impl):
    ddpm, data, kw = zinc_model(impl)
    d = dev()
    gen = torch.cuda.default_generators[d.index or 0]
    for t0 in (0, 5, 12):
        torch.manual_seed(99)
        off0 = gen.get_offset()
        chain_dev, _ = ddpm.sample_chain(data, keep_frames=3, start_step=t0)
        end_dev = gen.get_offset()
        torch.manual_seed(99)
        ddpm.edm.noise_mode = 'reference_tensor'
        chain_ten, _ = ddpm.sample_chain(data, keep_frames=3, start_step=t0)
        ddpm.edm.noise_mode = 'reference_stream'
        assert gen.get_offset() == end_dev, t0
        assert torch.equal(chain_dev, chain_ten), t0
        torch.manual_seed(99)
        ddpm.edm.draw_noise(t0 + 2, *kw['x'].shape[:2], d)                 # t0 + 2 randn pairs
        assert gen.get_offset() == end_dev and end_dev > off0, t0
    torch.manual_seed(99)
    plain, _ = ddpm.sample_chain(data, keep_frames=3)                       # no start step: the plain sampler, unchanged
    torch.manual_seed(99)
    again, _ = ddpm.sample_chain(data, keep_frames=3, start_step=None)
    assert torch.equal(plain, again)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_per_molecule_chain_is_the_same_in_any_batch_row_and_split(impl):
    ddpm, data, kw = zinc_model(impl)
    edm = ddpm.edm
    seeds = [3, 1 << 62, -9, 77, 5, 12, 2024]
    t0 = 7
    full = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, start_step=t0)
    b = 4
    alone = edm.sample_chain(**steps_take(kw, [b]), keep_frames=4, seeds=[seeds[b]], start_step=t0)
    moved = edm.sample_chain(**steps_take(kw, [2, b, 0]), keep_frames=4, seeds=[seeds[2], seeds[b], seeds[0]], start_step=t0)
    assert torch.equal(full[:, b], alone[:, 0]) and torch.equal(full[:, b], moved[:, 1])
    edm.devices = [0, 0]
    try:
        split = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, start_step=t0)
    finally:
        edm.devices = None
    assert torch.equal(split, full)
    assert not torch.equal(full, edm.sample_chain(**kw, keep_frames=4, seeds=seeds, start_step=t0 - 1))


def steps_take(kw, idx):
    """Rows `idx` of FC sampler inputs (the edge mask holds B equal blocks)."""
    B = kw['x'].shape[0]
    ix = torch.tensor(idx, device=kw['x'].device)
    out = {}
    for k, v in kw.items():
        out[k] = None if v is None else (v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:]) if k == 'edge_mask'
                                         else v[ix])
    return out


def first_draw(edm, kw, seeds, keep_frames, t0):
    """(chain, flags) of dl_sample_chain_seeded from step t0 on the whole batch, kept even where a row diverges."""
    lib = _native.load_library()
    B, N = kw['x'].shape[:2]
    t = edm._sampler_tensors(**kw)
    sd = seeds_tensor(seeds, B).to(kw['x'].device)
    chain = torch.empty((keep_frames, B, N, 3 + edm.in_node_nf), device=kw['x'].device)
    flags = torch.zeros(B, dtype=torch.int32, device=kw['x'].device)
    eng = edm.dynamics.engine(0)
    _native.check(lib.dl_set_start_step(eng, *edm._start(t0, B)), "dl_set_start_step")
    try:
        st = lib.dl_sample_chain_seeded(eng, *edm._head(B, N, keep_frames, t), sd.data_ptr(),
                                        edm.step_coefficients(keep_frames, B), edm._norm(), chain.data_ptr(), flags.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    finally:
        lib.dl_set_start_step(eng, -1, 0.0, 0.0)
    assert st >= 0, lib.dl_last_error()
    return chain, flags.cpu()


# coord_mlp gain 5 at T = 10: some molecules diverge for some seeds (test_nan_recovery.py measured 17 % of the (molecule,
# seed) pairs from noise). From t0 = T the start keeps alpha_T * xh, a small term; 24 seeds make a batch with both kinds.
# Below 32 molecules torch's CPU kernels give the batch and a molecule alone the same step coefficients and start scalars.
GAIN_SEEDS = list(range(101, 125))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("connected", [False, True])
def test_recovery_rounds_resample_from_the_same_start(impl, connected):
    ddpm, data, kw = zinc_model(impl, T=10, rows=len(GAIN_SEEDS), gain=5.0)
    edm = ddpm.edm
    B, t0 = len(GAIN_SEEDS), 10
    first, flags0 = first_draw(edm, kw, GAIN_SEEDS, 3, t0)
    bad = flags0.nonzero().flatten().tolist()
    assert 1 <= len(bad) < B, bad
    extra = dict(require_connected=True) if connected else {}
    edm.is_geom = False
    try:
        chain = edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4, start_step=t0, **extra)
    except FoundNaNException as exc:                                    # a row may diverge in all four rounds
        chain = exc.chain
    attempts = edm.last_attempts.tolist()
    untouched = [b for b in range(B) if attempts[b] == 0]
    assert set(bad).isdisjoint(untouched)
    assert torch.equal(chain[:, untouched], first[:, untouched])
    used = edm.last_seeds
    recovered = [b for b in range(B) if attempts[b] > 0 and torch.isfinite(chain[:, b]).all()]
    assert recovered
    for b in recovered:
        assert int(used[b]) == retry_seed(GAIN_SEEDS[b], attempts[b])
        alone = edm.sample_chain(**steps_take(kw, [b]), keep_frames=3, seeds=[int(used[b])], start_step=t0)
        if impl == "simt":
            assert torch.equal(chain[:, b], alone[:, 0]), b
        else:
            assert (chain[:, b] - alone[:, 0]).abs().max() <= 1e-4 * alone[:, 0].abs().max().clamp(min=1.0), b


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_sample_many_equals_per_request_sample_chain(impl):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    ddpm.edm.T = 12
    d = dev()
    ddpm = ddpm.to(d)
    datas = [{k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=b)).items()}
             for b in (3, 1, 5, 2)]
    seeds = [[11 * k + b for b in range(x['linker_mask'].shape[0])] for k, x in enumerate(datas)]
    for t0 in (0, 6, 12):
        many = ddpm.sample_many(datas, keep_frames=3, seeds=seeds, start_step=t0)
        for k, data in enumerate(datas):
            want, nm = ddpm.sample_chain(data, keep_frames=3, seeds=seeds[k], start_step=t0)
            assert torch.equal(many[k][0], want) and torch.equal(many[k][1], nm), (t0, k)
