"""RePaint resampling: InpaintingEDM.sample_chain(resamplings=r) runs every reverse step as r passes, each pass but the last
followed by the re-noise z <- alpha_t|s z + sigma_t|s eps (dl_set_resamplings).

CPU: the oracle (tests/repaint_oracle.py) against the reference's goldens (repaint_*.npz, tools/make_golden_repaint.py), the
jump coefficients against the reference's sigma_and_alpha_t_given_s, the draw count and order, the refusals and the C-ABI.
GPU, on both edge paths: the goldens, every stored state against fp64 with the known-eps construction of
test_sampler_steps_fp64.py, r = 1 against the plain call, the batch stream against its tensor, per-molecule streams alone,
in a batch and split, the recovery rounds and sample_many."""
import ctypes as C
import os
import shutil
import subprocess

import pytest
import torch

from difflinker_b200 import _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import retry_seed
from difflinker_b200.utils import FoundNaNException
import dl_helpers as helpers
import repaint_oracle as ro
import test_sampler_steps_fp64 as steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = [f"repaint_cfg1_r{r}_k{k}" for r in (2, 3) for k in (1, 5)]
INPUTS = ("x", "h", "node_mask", "fragment_mask", "linker_mask", "edge_mask", "context")
IMPLS = ["simt", "auto"]


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def golden_model(meta, impl='auto'):
    spec = helpers.spec_by_name(meta["spec"])
    ddpm, hp = helpers.build_ddpm(spec, meta["seed"], edge_impl=impl, inpainting=True)
    assert helpers.state_sha(ddpm.edm.dynamics.state_dict()) == meta["sha"], "seeded weights differ from the fixture's"
    assert ddpm.edm.T == meta["T"]
    return ddpm, hp, spec


def repaint_draws(seed, T, r, B, N, F, node_mask, fragment_mask):
    """The prepared (1 + T(3r-1) + 2, B, N, 3+F) draws of an r-pass chain from seeded_noise(seed), in call order."""
    draw = helpers.seeded_noise(seed)
    masks = ro.draw_masks(T, r, node_mask.float(), fragment_mask.float())
    return torch.stack([helpers.orc.com_free_noise(draw, B, N, 3, F, m) for m in masks])


def cfg1_model(T=None, impl='auto'):
    spec = synthetic.SPECS["cfg1_plumbing"]
    ddpm, hp = helpers.build_ddpm(spec, 0, edge_impl=impl, inpainting=True)
    if T is not None:
        ddpm.edm.T = T
    return ddpm, collate(synthetic.make_items(spec))


# ---- CPU ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", GOLDENS)
def test_oracle_matches_the_reference_composition(name):
    meta, a = helpers.load_golden(name)
    ddpm, hp, spec = golden_model(meta)
    gam = helpers.orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])
    ocfg = helpers.oracle_cfg(hp)
    ocfg.centering = True
    with torch.no_grad():
        chain = ro.repaint_chain(ddpm.edm.dynamics.state_dict(), ocfg, gam, meta["T"], meta["resamplings"],
                                 *(a[k] for k in INPUTS), keep_frames=meta["keep_frames"],
                                 norm_values=tuple(hp['normalize_factors']), noise_fn=helpers.seeded_noise(meta["noise_seed"]))
    assert chain.shape == a["chain"].shape
    assert (chain - a["chain"]).abs().max().item() == 0.0


@pytest.mark.parametrize("name", ["repaint_cfg1_r2_k1", "repaint_cfg1_r3_k1"])
def test_jump_coefficients_are_the_references(name):
    """edm.jump_coefficients(B) holds, bit for bit, the (alpha_t|s, sigma_t|s) the reference's sigma_and_alpha_t_given_s
    gives at that batch size, in dl_step_coef row order; the oracle's jump_scalars agree."""
    meta, a = helpers.load_golden(name)
    ddpm, hp, _ = golden_model(meta)
    B, T = meta["batch"], meta["T"]
    got = torch.tensor(list(ddpm.edm.jump_coefficients(B)), dtype=torch.float32).reshape(T, 2)
    assert torch.equal(got, a["jump"])
    gam = helpers.orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])
    for row in (0, T // 2, T - 1):
        al, sg = ro.jump_scalars(gam, T - 1 - row, T, B, hp['diffusion_steps'])
        assert float(al[0]) == float(got[row, 0]) and float(sg[0]) == float(got[row, 1])


@pytest.mark.parametrize("r", [1, 2, 5])
def test_draw_count_and_order(r):
    """draw_noise_inpaint(resamplings=r) makes 1 + T(3r-1) + 2 draws: z_T, per step and pass the p and q draws and, but on the
    last pass, the re-noise draw on every atom, then the two final draws; r = 1 is the plain call."""
    ddpm, data = cfg1_model(T=3)
    edm = ddpm.edm
    B, N = data['positions'].shape[:2]
    nm, fm = data['atom_mask'].float(), data['fragment_mask'].float()
    assert edm._n_draws(r) == 1 + 3 * (3 * r - 1) + 2
    got = edm.draw_noise_inpaint(B, N, 'cpu', nm, fm, generator=torch.Generator().manual_seed(3), resamplings=r)
    g = torch.Generator().manual_seed(3)
    want = torch.stack([helpers.orc.com_free_noise(lambda shape: torch.randn(shape, generator=g), B, N, 3, 8, m)
                        for m in ro.draw_masks(3, r, nm, fm)])
    assert got.shape[0] == edm._n_draws(r) and torch.equal(got, want)
    if r == 1:
        assert torch.equal(got, edm.draw_noise_inpaint(B, N, 'cpu', nm, fm, generator=torch.Generator().manual_seed(3)))


@pytest.mark.parametrize("bad", [0, -2, 1.5, True, "2", 1 << 40])
def test_resamplings_must_be_an_int_of_at_least_1(bad):
    ddpm, data = cfg1_model(T=4)
    kw = sampler_inputs(ddpm, data)
    with pytest.raises(ValueError, match="resamplings"):
        ddpm.edm.sample_chain(**kw, keep_frames=1, resamplings=bad)
    ddpm.edm.resamplings = bad
    with pytest.raises(ValueError, match="resamplings"):
        ddpm.edm.sample_chain(**kw, keep_frames=1)


def test_linker_sampler_refuses_resampling_and_inpainting_keeps_its_refusals():
    spec = synthetic.SPECS["cfg1_plumbing"]
    ddpm, _ = helpers.build_ddpm(spec, 0)
    data = collate(synthetic.make_items(spec))
    kw = sampler_inputs(ddpm, data)
    with pytest.raises(ValueError, match="resamplings"):
        ddpm.edm.sample_chain(**kw, keep_frames=1, resamplings=2)
    with pytest.raises(ValueError, match="resamplings"):
        ddpm.sample_chain(data, keep_frames=1, resamplings=3)
    with pytest.raises(ValueError, match="resamplings"):
        ddpm.edm.sample_many([kw], keep_frames=1, seeds=[list(range(4))], resamplings=2)
    ip, ipdata = cfg1_model(T=4)
    ikw = sampler_inputs(ip, ipdata)
    with pytest.raises(ValueError, match="start_step"):
        ip.edm.sample_chain(**ikw, keep_frames=1, resamplings=2, start_step=2)
    with pytest.raises(ValueError, match="require_clash_free"):
        ip.edm.sample_chain(**ikw, keep_frames=1, resamplings=2, require_clash_free=True, seeds=[1, 2, 3, 4])
    with pytest.raises(ValueError, match="linker_sizes"):
        ip.sample_chain(ipdata, keep_frames=1, resamplings=2, linker_sizes=5, seeds=[1, 2, 3, 4])


def test_noise_tensor_must_hold_the_resampled_draws():
    """noise= holds 1 + T(3r-1) + 2 slabs: a tensor of the plain loop's 2T+3 is refused with r = 2."""
    ddpm, data = cfg1_model(T=4)
    kw = sampler_inputs(ddpm, data)
    B, N = data['positions'].shape[:2]
    plain = torch.zeros((2 * 4 + 3, B, N, 11))
    with pytest.raises(AssertionError):
        ddpm.edm.sample_chain(**kw, keep_frames=1, noise=plain, resamplings=2)


def test_library_exports_the_setter_and_the_header_compiles_as_c99(tmp_path):
    lib = _native.load_library()
    assert hasattr(lib, "dl_set_resamplings") and "dl_set_resamplings" in _native.SYMBOLS
    assert lib.dl_set_resamplings(None, 2, 5, None) == -1               # DL_ERR_INVALID: no engine
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "repaint.c"
    src.write_text('#include "difflinker_b200.h"\n'
                   "int main(void) {\n"
                   "  const float jump[4] = {1.0f, 0.0f, 1.0f, 0.0f};\n"
                   "  dl_status s = dl_set_resamplings((dl_engine*)0, 2, 2, jump);\n"
                   "  return s == DL_ERR_INVALID ? 0 : 1;\n"
                   "}\n")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib_dir = os.path.dirname(_native.LIB_PATH)
    exe = str(tmp_path / "repaint")
    res = subprocess.run([gcc, "-std=c99", "-Wall", str(src), "-I" + os.path.join(ROOT, "include"),
                          "-L" + lib_dir, "-ldifflinker_b200", "-L" + os.path.join(cuda, "lib64"), "-lcudart",
                          "-Wl,-rpath," + lib_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    assert subprocess.run([exe]).returncode == 0


# ---- GPU: the engine's refusals -----------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_engine_refuses_what_resampling_does_not_take():
    lib = _native.load_library()
    ddpm, data = cfg1_model(T=4)
    d = dev()
    ddpm = ddpm.to(d)
    edm = ddpm.edm
    eng = edm.dynamics.engine(d.index or 0)
    jump = edm.jump_coefficients(4)
    assert lib.dl_set_resamplings(eng, 0, 4, jump) == -1
    assert lib.dl_set_resamplings(eng, 2, 4, None) == -1
    assert lib.dl_set_resamplings(eng, 1, 0, None) == 0
    kw = sampler_inputs(ddpm, {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in data.items()})
    t = edm._sampler_tensors(**kw)
    B, N = kw['x'].shape[:2]
    chain = torch.empty((1, B, N, 11), device=d)
    flags = torch.zeros(B, dtype=torch.int32, device=d)
    seeds = torch.arange(B, dtype=torch.int64, device=d)

    def seeded(sampler, T):
        head = (sampler, B, N, T, 1) + edm._head(B, N, 1, t)[5:]
        return lib.dl_sample_chain_seeded(eng, *head, seeds.data_ptr(), edm.step_coefficients(1, B), edm._norm(),
                                          chain.data_ptr(), flags.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _native.check(lib.dl_set_resamplings(eng, 2, 4, jump), "dl_set_resamplings")
    try:
        assert seeded(_native.SAMPLER_INPAINT, 3) == -1                 # T differs from the one set
        assert b"T = 4" in lib.dl_last_error()
        assert seeded(_native.SAMPLER_LINKER, 4) == -1                  # the linker sampler (the engine refuses the model too)
        assert seeded(_native.SAMPLER_INPAINT, 4) == 0
    finally:
        lib.dl_set_resamplings(eng, 1, 0, None)
    torch.cuda.synchronize()


# ---- GPU: the goldens ---------------------------------------------------------------------------------------------------

def rel_err(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.double().abs().max().item(), 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("name", GOLDENS)
def test_chain_matches_the_reference_golden(name, impl):
    """The rule of test_gpu_parity's inpaint_chain_cfg1 test: identical atom types, every frame within 1e-4 relative."""
    meta, a = helpers.load_golden(name)
    ddpm, hp, spec = golden_model(meta, impl)
    d = dev()
    ddpm = ddpm.to(d)
    r, keep, T = meta["resamplings"], meta["keep_frames"], meta["T"]
    B, N = a["x"].shape[:2]
    noise = repaint_draws(meta["noise_seed"], T, r, B, N, spec.F, a["node_mask"], a["fragment_mask"])
    kw = {k: a[k].to(d) for k in INPUTS}
    chain = ddpm.edm.sample_chain(**kw, keep_frames=keep, noise=noise.to(d), resamplings=r).cpu()
    want = a["chain"]
    assert chain.shape == want.shape
    assert torch.equal(chain[0][..., 3:], want[0][..., 3:]), "atom types differ"
    errs = [rel_err(chain[f], want[f]) for f in range(keep)]
    print(f"\n[{name} {impl}] relative frame errors {[f'{e:.2g}' for e in errs]}, drift64 {a['drift64'].tolist()}")
    assert max(errs) <= 1e-4, errs


# ---- GPU: every stored state against fp64 ------------------------------------------------------------------------------

def check_repaint_chain(label, chain, kw, draws, bias, gamma, T, r):
    """steps.check_inpaint_chain with r passes per step: each pass's inpainting step and, for u < r-1, the re-noise
    z <- alpha_t|s z + sigma_t|s eps (products and sum rounded once each: error |alpha| e + 2U(|alpha z| + |sigma eps|) +
    U |result|) replayed in fp64 from the GPU's previous stored state (keep_frames = T: every step but s = 0 has a frame of
    its own), then the final step as there."""
    d = chain.device
    U = steps.U
    chain = steps.f64(chain, d)
    B, N, D = chain.shape[1:]
    nm, fm, lm = (steps.f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    live = nm[..., 0] != 0
    draws = steps.f64(draws, d)
    xh = torch.cat([steps.f64(kw['x'], d) / steps.NORM[0], steps.f64(kw['h'], d) / steps.NORM[1]], dim=2)
    eps = torch.zeros_like(xh)
    eps[..., 3:] = steps.f64(torch.tensor(bias), d) * nm
    sc = steps.scalars(gamma, T, B)
    frame_of = {s: f for f, s in steps.stored_steps(T, T).items()}
    ck = steps.Checker(label)
    z, e = draws[0], torch.zeros_like(xh)
    for s in range(T - 1, -1, -1):
        k = T - 1 - s
        a, b, c, qa, qb = (helpers.orc._sc(sc[s], key, z) for key in ("a", "b", "c", "qa", "qb"))
        al, sg = (helpers.orc._bcast(v).to(z) for v in ro.jump_scalars(gamma, s, T, B, gamma.numel() - 1))
        for u in range(r):
            base = 1 + k * (3 * r - 1) + 3 * u
            n_p, n_q = draws[base], draws[base + 1]
            za = z.abs() + e
            zn = (z / a - b * eps + c * n_p) * lm + (qa * z + qb * (xh * fm) + c * n_q) * fm
            pre = ((e / a.abs() + 4 * U * (za / a.abs() + (b * eps).abs() + (c * n_p).abs())) * lm
                   + (qa.abs() * e + 4 * U * (qa.abs() * za + (qb * xh * fm).abs() + (c * n_q).abs())) * fm)
            ref = helpers.orc.inpaint_step(z, eps, sc[s], n_p, n_q, xh, nm, fm, lm)
            e = pre.clone()
            e[..., :3] = (pre[..., :3] + steps.projection_bound(zn, pre, nm, D) + U * ref[..., :3].abs()) * nm
            z = ref
            if u < r - 1:
                n_r = draws[base + 2]
                z = ro.renoise(z, n_r, al, sg)
                e = (al.abs() * e + 2 * U * ((al * ref).abs() + (sg * n_r).abs()) + U * z.abs()) * nm
        if s in frame_of:
            got = steps.unnorm_frame(chain[frame_of[s]])
            ck.close(f"step s={s}", got, z, e, live)
            z, e = got, torch.zeros_like(e)
    inv_a0, sig0, snr0, qa0 = (helpers.orc._sc(sc[-1], key, z) for key in ("inv_alpha0", "sigma0", "snr0", "qa0"))
    n_p, n_q = draws[1 + T * (3 * r - 1)], draws[2 + T * (3 * r - 1)]
    out_l, out_f = helpers.orc.inpaint_final(z, eps, sc[-1], n_p, n_q)
    za = z.abs() + e
    e_l = inv_a0 * e + 4 * U * (inv_a0 * za + inv_a0 * (sig0 * eps).abs() + (snr0 * n_p).abs())
    e_f = inv_a0 * e + 4 * U * (inv_a0 * za + (qa0 * n_q).abs())
    got = chain[0]
    ck.close("final x", got[..., :3], (out_l[..., :3] * lm + out_f[..., :3] * fm) * steps.NORM[0],
             (e_l[..., :3] * lm + e_f[..., :3] * fm) * steps.NORM[0], live)
    lk, fr = (lm[..., 0] != 0) & live, (fm[..., 0] != 0) & live
    ck.types("final h (p variant, linker rows)", got[..., 3:] * lm, out_l[..., 3:], e_l[..., 3:], lk, (nm * lm)[..., 0])
    ck.types("final h (q variant, fragment rows)", got[..., 3:] * fm, out_f[..., 3:], e_f[..., 3:], fr, (nm * fm)[..., 0])
    ck.record()


# label -> (graph type, F, molecule sizes, T, r): FC molecules (atoms, linker atoms) or pocket molecules (fragment, pocket,
# linker atoms), as test_sampler_steps_fp64's INPAINT cases
FP64_CASES = {
    "FC_N30_T6_r2": ("FC", 8, [(30, 6), (22, 4), (25, 9), (7, 1)], 6, 2),
    "FC_N257_T3_r4_F13": ("FC", 13, [(257, 12), (200, 7), (40, 3)], 3, 4),
    "4A_N300_T2_r3": ("4A", 9, [(30, 260, 10), (25, 200, 12)], 2, 3),
}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", list(FP64_CASES))
def test_resampled_steps_vs_fp64(case, impl):
    graph_type, F, sizes, T, r = FP64_CASES[case]
    edm, hp, bias = steps.known_eps_model(F, T, impl, graph_type=graph_type, inpainting=True)
    kw = steps.fc_batch(sizes, F, seed=31) if graph_type == "FC" else steps.pocket_inputs(sizes, 2, 6)
    d = dev()
    kw = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    draws = repaint_draws(41, T, r, B, N, F, kw['node_mask'].reshape(B, N, 1).cpu(),
                          kw['fragment_mask'].reshape(B, N, 1).cpu()).to(d)
    chain = edm.sample_chain(**kw, keep_frames=T, noise=draws, resamplings=r)
    check_repaint_chain(f"repaint {case} {impl}", chain, kw, draws, bias, steps.gamma_of(hp), T, r)


# ---- GPU: r = 1, noise streams, recovery, sample_many ------------------------------------------------------------------

def zinc_model(impl, T=8, rows=7, gain=1.0, spec_name="cfg2_zinc_ragged"):
    spec = helpers.spec_by_name(spec_name)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, inpainting=True)
    if gain != 1.0:
        with torch.no_grad():
            for name, p in ddpm.named_parameters():
                if name.endswith("coord_mlp.4.weight"):
                    p.mul_(gain)
    ddpm.edm.T = T
    d = dev()
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=rows)).items()}
    return ddpm, data, sampler_inputs(ddpm, data)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_one_pass_is_the_plain_sampler_with_the_same_launches(impl):
    ddpm, data, kw = zinc_model(impl)
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    for extra in (dict(seeds=list(range(7))), {}):
        torch.manual_seed(4)
        n0 = lib.dl_launch_count(eng)
        plain = edm.sample_chain(**kw, keep_frames=3, **extra)
        n1 = lib.dl_launch_count(eng)
        torch.manual_seed(4)
        one = edm.sample_chain(**kw, keep_frames=3, resamplings=1, **extra)
        n2 = lib.dl_launch_count(eng)
        assert torch.equal(plain, one) and n2 - n1 == n1 - n0
        torch.manual_seed(4)
        two = edm.sample_chain(**kw, keep_frames=3, resamplings=2, **extra)
        n3 = lib.dl_launch_count(eng)
        assert not torch.equal(two, plain)
        assert lib.dl_last_molecule_steps(eng) == 7 * (2 * edm.T + 1)
        edm.sample_chain(**kw, keep_frames=3, resamplings=3, **extra)
        n4 = lib.dl_launch_count(eng)
        # every pass launches what a plain step launches: T more step graphs per extra pass, the same setup
        per_pass, rem = divmod((n3 - n2) - (n1 - n0), edm.T)
        assert rem == 0 and per_pass > 0 and n4 - n3 == (n3 - n2) + per_pass * edm.T


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("spec_name", ["cfg2_zinc_ragged", "small_pocket_4A"])
def test_batch_stream_equals_torch_draws_in_the_stated_order(impl, spec_name):
    """The device-side batch stream against draw_noise_inpaint(resamplings=r) of the same generator state
    (noise_mode='reference_tensor'): identical atom types, frames within the existing inpainting-stream test's 1e-5 (1e-4 on
    pocket graphs), the same generator advance, 1 + T(3r-1) + 2 draws."""
    ddpm, data, kw = zinc_model(impl, T=6, rows=5 if spec_name.startswith("cfg2") else None, spec_name=spec_name)
    d = dev()
    gen = torch.cuda.default_generators[d.index or 0]
    tol = 1e-5 if spec_name.startswith("cfg2") else 1e-4
    for r in (2, 3):
        torch.manual_seed(77)
        off0 = gen.get_offset()
        chain_dev, _ = ddpm.sample_chain(data, keep_frames=3, resamplings=r)
        end_dev = gen.get_offset()
        torch.manual_seed(77)
        ddpm.edm.noise_mode = 'reference_tensor'
        try:
            chain_ten, _ = ddpm.sample_chain(data, keep_frames=3, resamplings=r)
        finally:
            ddpm.edm.noise_mode = 'reference_stream'
        assert gen.get_offset() == end_dev > off0
        assert torch.equal(chain_dev[0][..., 3:], chain_ten[0][..., 3:]), "atom types differ"
        errs = [rel_err(chain_dev[f], chain_ten[f]) for f in range(3)]
        assert max(errs) <= tol, (r, errs)
        B, N = kw['x'].shape[:2]
        per_draw = (end_dev - off0) // (1 + 6 * (3 * r - 1) + 2)
        assert per_draw * (1 + 6 * (3 * r - 1) + 2) == end_dev - off0
        torch.manual_seed(77)
        torch.randn((B, N, 3), device=d)
        torch.randn((B, N, 8 if spec_name.startswith("cfg2") else 9), device=d)
        assert gen.get_offset() - off0 == per_draw


@pytest.mark.gpu
def test_device_fill_writes_the_resampled_draws():
    """dl_noise_fill_inpaint with r passes set writes draw_noise_inpaint(resamplings=r)'s tensor: features bit for bit,
    coordinates within the existing fill test's 2e-6."""
    lib = _native.load_library()
    ddpm, data, kw = zinc_model("auto", T=3, rows=4)
    edm = ddpm.edm
    d = dev()
    B, N = kw['x'].shape[:2]
    nm, fm = kw['node_mask'].reshape(B, N, 1), kw['fragment_mask'].reshape(B, N, 1)
    eng = edm.dynamics.engine(0)
    r = 3
    torch.manual_seed(12)
    gen = torch.cuda.default_generators[d.index or 0]
    seed, offset = gen.initial_seed(), gen.get_offset()
    got = torch.empty((edm._n_draws(r), B, N, 11), device=d)
    used = C.c_uint64(0)
    _native.check(lib.dl_set_resamplings(eng, r, 3, edm.jump_coefficients(B)), "dl_set_resamplings")
    try:
        _native.check(lib.dl_noise_fill_inpaint(eng, 3, B, N, nm.reshape(B, N).to(torch.int8).contiguous().data_ptr(),
                                                fm.reshape(B, N).float().contiguous().data_ptr(), seed, offset,
                                                got.data_ptr(), C.byref(used), torch.cuda.current_stream().cuda_stream),
                      "dl_noise_fill_inpaint")
        torch.cuda.synchronize()
    finally:
        lib.dl_set_resamplings(eng, 1, 0, None)
    want = edm.draw_noise_inpaint(B, N, d, nm.float(), fm.float(), resamplings=r)
    assert gen.get_offset() == offset + used.value
    assert torch.equal(got[..., 3:], want[..., 3:])
    ok = ~torch.isnan(want[..., :3])
    assert torch.equal(ok, ~torch.isnan(got[..., :3]))
    assert (got[..., :3][ok] - want[..., :3][ok]).abs().max().item() <= 2e-6


def take(kw, idx):
    """Rows `idx` of sampler inputs (an FC edge mask holds B equal blocks)."""
    B = kw['x'].shape[0]
    ix = torch.tensor(idx, device=kw['x'].device)
    return {k: None if v is None else (v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:]) if k == 'edge_mask'
                                       else v[ix]) for k, v in kw.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("spec_name", ["cfg2_zinc_ragged", "small_pocket_4A"])
def test_per_molecule_rows_are_the_molecule_alone_and_split(impl, spec_name):
    """With seeds, row b is molecule b sampled alone (bit for bit on the SIMT path, within 1e-4 relative on the tensor-core
    path) and devices=[0, 0] gives the single-device chain bit for bit on the SIMT path."""
    pocket = spec_name.startswith("small")
    ddpm, data, kw = zinc_model(impl, T=6, rows=None if pocket else 5, spec_name=spec_name)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = [3, 1 << 62, -9, 77, 5][:B]
    full = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, resamplings=3)
    for b in range(B):
        alone = edm.sample_chain(**take(kw, [b]), keep_frames=3, seeds=[seeds[b]], resamplings=3)
        if impl == "simt":
            assert torch.equal(full[:, b], alone[:, 0]), b
        else:
            assert rel_err(full[:, b], alone[:, 0]) <= 1e-4, b
    edm.devices = [0, 0]
    try:
        split = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, resamplings=3)
    finally:
        edm.devices = None
    if impl == "simt":
        assert torch.equal(split, full)
    else:
        assert rel_err(split, full) <= 1e-4


# coord_mlp gain 5: some molecules diverge for some seeds, as in test_partial_diffusion's recovery test
GAIN_SEEDS = list(range(101, 125))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_recovery_rounds_resample_with_the_same_passes(impl):
    """nan_retries with require_connected: rows the rounds did not touch are those of the plain seeded call, and every
    resampled row replays alone from its recorded seed with the same r."""
    ddpm, data, kw = zinc_model(impl, T=6, rows=len(GAIN_SEEDS), gain=5.0)
    edm = ddpm.edm
    B, r = len(GAIN_SEEDS), 2
    try:
        first = edm.sample_chain(**kw, keep_frames=2, seeds=GAIN_SEEDS, resamplings=r)
    except FoundNaNException:
        first = None
    edm.is_geom = False
    try:
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=GAIN_SEEDS, nan_retries=3, require_connected=True,
                                 resamplings=r)
    except FoundNaNException as exc:
        chain = exc.chain
    attempts, used = edm.last_attempts.tolist(), edm.last_seeds.clone()     # the replays below overwrite them
    untouched = [b for b in range(B) if attempts[b] == 0]
    resampled = [b for b in range(B) if attempts[b] > 0 and torch.isfinite(chain[:, b]).all()]
    assert resampled, attempts
    for b in untouched:
        alone = edm.sample_chain(**take(kw, [b]), keep_frames=2, seeds=[GAIN_SEEDS[b]], resamplings=r)
        if impl == "simt":
            assert torch.equal(chain[:, b], alone[:, 0]), b
        if first is not None and impl == "simt":
            assert torch.equal(chain[:, b], first[:, b]), b
    for b in resampled:
        assert int(used[b]) == retry_seed(GAIN_SEEDS[b], attempts[b])
        try:
            alone = edm.sample_chain(**take(kw, [b]), keep_frames=2, seeds=[int(used[b])], resamplings=r)
        except FoundNaNException:
            pytest.fail(f"row {b} was kept finite but its seed diverges alone")
        if impl == "simt":
            assert torch.equal(chain[:, b], alone[:, 0]), b
        else:
            assert rel_err(chain[:, b], alone[:, 0]) <= 1e-4, b


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_sample_many_equals_per_request_sample_chain(impl):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, inpainting=True)
    ddpm.edm.T = 6
    d = dev()
    ddpm = ddpm.to(d)
    datas = [{k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=b)).items()}
             for b in (3, 1, 5, 2)]
    seeds = [[11 * k + b for b in range(x['atom_mask'].shape[0])] for k, x in enumerate(datas)]
    many = ddpm.sample_many(datas, keep_frames=3, seeds=seeds, resamplings=3)
    for k, data in enumerate(datas):
        want, nm = ddpm.sample_chain(data, keep_frames=3, seeds=seeds[k], resamplings=3)
        if impl == "simt":
            assert torch.equal(many[k][0], want), k
        else:
            assert rel_err(many[k][0], want) <= 1e-4, k
        assert torch.equal(many[k][1], nm), k
    ddpm.edm.resamplings = 3                                            # the attribute stands in for the argument
    try:
        again = ddpm.sample_many(datas, keep_frames=3, seeds=seeds)
    finally:
        ddpm.edm.resamplings = 1
    assert all(torch.equal(a[0], b[0]) for a, b in zip(again, many))
