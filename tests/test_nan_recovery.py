"""NaN recovery: `sample_chain(..., nan_retries=)`, dl_sample_chain_retry, dl_retry_seed and `c_sampler --retries`.

With per-molecule seeds a molecule's chain does not depend on its batch, so resampling only the molecules that diverged,
with seeds derived from their own, is itself an exact sample: the rows that did not fail stay bit for bit what they were,
and a recovered row is the molecule sampled alone with the seed recorded for it. CPU tests pin the retry seeds and the
argument checks; the GPU tests use a molecule that fails on every attempt (a NaN coordinate) and weights whose divergence
depends on the noise."""
import os
import shutil
import subprocess

import pytest
import torch

from difflinker_b200 import _native, export_job, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import draw_seeds, retry_seed, seeds_tensor
from difflinker_b200.utils import FoundNaNException
import dl_helpers as helpers

U64 = 1 << 64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def splitmix64(seed, attempt):
    """The formula include/difflinker_b200.h documents for dl_retry_seed."""
    if attempt <= 0:
        return seed
    z = (seed + attempt * 0x9E3779B97F4A7C15) % U64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) % U64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) % U64
    return z ^ (z >> 31)


# ---- CPU --------------------------------------------------------------------------------------------------------------

PINNED = [(0, 0, 0), (0, 1, 0xE220A8397B1DCDAF),                     # splitmix64's first output from state 0
          (1, 1, 10451216379200822465), (1, 2, 13757245211066428519),
          (U64 - 1, 0, U64 - 1), (U64 - 1, 1, 16490336266968443936), (U64 - 1, 7, 17388166129998380965),
          (20240607, 3, 18316511635328169175), (1 << 63, 1, 5196802822362493915)]


def test_retry_seeds_are_pinned():
    lib = _native.load_library()
    for seed, attempt, want in PINNED:
        assert lib.dl_retry_seed(seed, attempt) == want == splitmix64(seed, attempt), (seed, attempt)
    assert lib.dl_retry_seed(12345, -3) == 12345                       # no attempt below the first draw


def test_retry_seeds_do_not_collide():
    lib = _native.load_library()
    seeds = list(range(256)) + [U64 - 1 - i for i in range(64)] + [(1 << 63) + i for i in range(64)] + [20240607, 1 << 32]
    values = [lib.dl_retry_seed(s, a) for s in seeds for a in range(6)]
    assert len(set(values)) == len(values)


def test_python_wrapper_agrees_with_the_library():
    lib = _native.load_library()
    g = torch.Generator().manual_seed(3)
    seeds = [0, -1, -(1 << 63), (1 << 63) - 1, 1 << 63, U64 - 1] + torch.randint(-(1 << 63), (1 << 63) - 1, (20,), generator=g).tolist()
    for s in seeds:
        for a in (0, 1, 2, 5, 31):
            r = retry_seed(s, a)
            assert r == int(seeds_tensor([lib.dl_retry_seed(s % U64, a)], 1)[0])    # the int64 form last_seeds holds
            assert r % U64 == splitmix64(s % U64, a)
    assert retry_seed(-1, 0) == -1 and retry_seed(U64 - 1, 0) == -1
    with pytest.raises(ValueError):
        retry_seed(U64, 1)
    with pytest.raises(ValueError):
        retry_seed(1, 1 << 31)


def _cpu_model(inpainting=False):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    over = {"inpainting": True} if inpainting else {}
    ddpm, _ = helpers.build_ddpm(spec, 0, **over)
    ddpm.edm.T = 4
    return ddpm, sampler_inputs(ddpm, collate(synthetic.make_items(spec, batch=3)))


@pytest.mark.parametrize("inpainting", [False, True])
def test_recovery_refuses_what_cannot_resample_one_molecule(inpainting):
    ddpm, kw = _cpu_model(inpainting)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    assert edm.nan_retries == 0 and edm.last_attempts is None
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="nan_retries"):
            edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3], nan_retries=bad)
    with pytest.raises(ValueError, match="per-molecule streams"):            # the batch stream
        edm.sample_chain(**kw, keep_frames=2, nan_retries=2)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, nan_retries=2, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, nan_retries=2, seeds=[1, 2, 3], noise=torch.zeros(1))
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, nan_retries=2, seeds=[1, 2, 3], batch_slice=(0, B))
    with pytest.raises(ValueError, match="nan_retries needs CUDA inputs"):  # host inputs
        edm.sample_chain(**kw, keep_frames=2, nan_retries=2, seeds=[1, 2, 3])
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="replaced"):
        edm.sample_chain(**kw, keep_frames=2, nan_retries=2, seeds=[1, 2, 3])
    delattr(edm, name)
    edm.nan_retries = 2                                                 # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.noise_mode = 'per_molecule'
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, batch_slice=(0, B))
    with pytest.raises(ValueError, match="nan_retries needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.nan_retries = -2
    with pytest.raises(ValueError, match=">= 0"):
        edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3])
    assert edm.last_attempts is None


def test_header_compiles_as_c99_with_the_one_recovery_entry(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "retry_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2]; int32_t attempts[2], flags[2];\n"
        "  dl_status st = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                       NULL, NULL, NULL, NULL, flags, 3, used, attempts, NULL, NULL, NULL, NULL, NULL);\n"
        '  printf("%d|%llu|%llu|%.1f|%s\\n", (int)st, (unsigned long long)dl_retry_seed(0, 1),\n'
        "         (unsigned long long)dl_retry_seed(UINT64_MAX, 0), (double)dl_last_retry_ms(NULL), dl_last_error());\n"
        "  return 0;\n}\n")
    exe = tmp_path / "retry_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    status, first, same, ms, err = res.stdout.strip().split("|", 4)
    assert int(status) == -1 and "null engine" in err
    assert int(first) == 0xE220A8397B1DCDAF and int(same) == U64 - 1 and float(ms) == -1.0


def test_c_caller_takes_retries_only_for_seeded_jobs(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    _native.load_library()
    ddpm, kw = _cpu_model()
    job, out = str(tmp_path / "job.bin"), str(tmp_path / "out.bin")
    export_job.write_job(job, ddpm.edm, **kw, keep_frames=2, seed=1)
    exe = helpers.build_c_example(tmp_path)
    res = subprocess.run([exe, "--retries", "2", job, out], capture_output=True, text=True, timeout=120)
    assert res.returncode == 2 and "seeded" in res.stderr
    for bad in ("-1", "x", ""):
        res = subprocess.run([exe, "--retries", bad, job, out], capture_output=True, text=True, timeout=120)
        assert res.returncode == 2 and "--retries" in res.stderr
    assert not os.path.exists(out)


# ---- GPU --------------------------------------------------------------------------------------------------------------

# Extra scale of coord_mlp.4 (on top of the fixtures' 100) at which, at T = 10, the cfg2_zinc_ragged molecules diverge for
# some seeds and not for others: measured on an H100 over 12 seed sets of 8 molecules, 17 % of the (molecule, seed) pairs
# diverge on either edge path, with either sampler (none at 3, 85 % at 8).
COORD_GAIN = 5.0
GAIN_SEEDS = [1, 2, 3, 4, 5, 6, 7, 8]        # rows 4 and 7 diverge at the first draw
SEEDS = [11, -3, 1 << 63, 20240607, 5]


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def take(kw, idx):
    """Rows `idx` of the sampler inputs; the FC edge mask holds B equal blocks, the pocket one per-node batch ids."""
    B = kw['x'].shape[0]
    ix = torch.tensor(idx, device=kw['x'].device)
    out = {}
    for k, v in kw.items():
        if v is None:
            out[k] = None
        elif k == 'edge_mask':
            out[k] = v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:])
        else:
            out[k] = v[ix]
    return out


def build(case, impl, rows, gain=1.0):
    d = dev()
    over = {}
    if case == "fc":
        spec = synthetic.SPECS["cfg2_zinc_ragged"]
    elif case == "fc_inpainting":
        spec, over = synthetic.SPECS["cfg2_zinc_ragged"], {"inpainting": True}
    else:
        spec = helpers.EXTRA_SPECS[f"small_{case}"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    if gain != 1.0:
        with torch.no_grad():
            for name, p in ddpm.named_parameters():
                if name.endswith("coord_mlp.4.weight"):
                    p.mul_(gain)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=rows)).items()}
    return ddpm, sampler_inputs(ddpm, data)


def first_draw(edm, kw, seeds, keep_frames):
    """(chain, flags) of dl_sample_chain_seeded on the whole batch: what nan_retries=0 samples, kept even where it fails."""
    lib = _native.load_library()
    B, N = kw['x'].shape[:2]
    t = edm._sampler_tensors(**kw)
    sd = seeds_tensor(seeds, B).to(kw['x'].device)
    chain = torch.empty((keep_frames, B, N, 3 + edm.in_node_nf), device=kw['x'].device)
    flags = torch.zeros(B, dtype=torch.int32, device=kw['x'].device)
    st = lib.dl_sample_chain_seeded(edm.dynamics.engine(0), *edm._head(B, N, keep_frames, t), sd.data_ptr(),
                                    edm.step_coefficients(keep_frames, B), edm._norm(), chain.data_ptr(), flags.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert st >= 0, lib.dl_last_error()
    return chain, flags.cpu()


def failed(exc):
    return sorted(exc.x_h_nan_idx | exc.only_x_nan_idx | exc.only_h_nan_idx)


def close(got, want):
    """The suite's fp32 tolerance: 1e-4 of the values' scale (at least 1)."""
    return bool((got - want).abs().max() <= 1e-4 * want.abs().max().clamp(min=1.0))


ALWAYS_CASES = [("fc", "simt", 5), ("fc", "auto", 5), ("fc_inpainting", "simt", 5), ("fc_inpainting", "auto", 5),
                ("pocket_FC-10A-4A", "auto", 4), ("pocket_FC-10A-4A", "simt", 4), ("pocket_4A", "auto", 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl,rows", ALWAYS_CASES)
def test_a_molecule_that_always_fails_is_the_only_one_reported(case, impl, rows):
    ddpm, kw = build(case, impl, rows)
    edm = ddpm.edm
    bad = 2
    kw['x'] = kw['x'].clone()
    kw['x'][bad, 0, 0] = float('nan')                                    # a fragment coordinate: every attempt fails
    seeds = SEEDS[:rows]
    want, flags0 = first_draw(edm, kw, seeds, 3)
    assert flags0.nonzero().flatten().tolist() == [bad]
    for devices in (None, [0, 0, 0]):
        edm.devices = devices
        with pytest.raises(FoundNaNException) as info:
            edm.sample_chain(**kw, keep_frames=3, seeds=seeds, nan_retries=3)
        exc = info.value
        assert failed(exc) == [bad], devices
        attempts = [0] * rows
        attempts[bad] = 3
        assert edm.last_attempts.dtype == torch.int32 and edm.last_attempts.tolist() == attempts
        used = seeds_tensor(seeds, rows)
        used[bad] = retry_seed(seeds[bad], 3)
        assert torch.equal(edm.last_seeds, used)
        others = [b for b in range(rows) if b != bad]
        assert torch.equal(exc.chain[:, others], want[:, others]), devices
    edm.devices = None
    with pytest.raises(FoundNaNException) as info:                      # without recovery: as before, no chain attached
        edm.sample_chain(**kw, keep_frames=3, seeds=seeds)
    assert failed(info.value) == [bad] and not hasattr(info.value, "chain") and edm.last_attempts is None


def gain_model(impl):
    ddpm, kw = build("fc", impl, len(GAIN_SEEDS), gain=COORD_GAIN)
    return ddpm, kw


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_only_the_diverged_molecules_are_resampled(impl):
    ddpm, kw = gain_model(impl)
    edm = ddpm.edm
    B = len(GAIN_SEEDS)
    first, flags0 = first_draw(edm, kw, GAIN_SEEDS, 3)
    bad = flags0.nonzero().flatten().tolist()
    assert 1 <= len(bad) < B, bad                                       # the gain still splits the batch
    chain = edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4)
    assert torch.isfinite(chain).all()
    attempts = edm.last_attempts.tolist()
    healthy = [b for b in range(B) if b not in bad]
    assert [attempts[b] for b in healthy] == [0] * len(healthy) and all(attempts[b] >= 1 for b in bad)
    assert torch.equal(chain[:, healthy], first[:, healthy])
    used = edm.last_seeds
    for b in range(B):
        assert int(used[b]) == retry_seed(GAIN_SEEDS[b], attempts[b])
    for b in bad:
        alone = edm.sample_chain(**take(kw, [b]), keep_frames=3, seeds=[int(used[b])])
        for f in range(3):                                              # every frame of the row was replaced
            assert not torch.equal(chain[f, b], first[f, b]), (b, f)
            if impl == "simt":
                assert torch.equal(chain[f, b], alone[f, 0]), (b, f)
            else:
                assert close(chain[f, b], alone[f, 0]), (b, f)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_splits_recover_what_the_unsplit_call_recovers(impl):
    ddpm, kw = gain_model(impl)
    edm = ddpm.edm
    want = edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4)
    seeds, attempts = edm.last_seeds, edm.last_attempts
    assert attempts.any()
    for devices in ([0, 0], [0, 0, 0]):
        edm.devices = devices
        got = edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4)
        assert torch.equal(edm.last_attempts, attempts) and torch.equal(edm.last_seeds, seeds), devices
        if impl == "simt":
            assert torch.equal(got, want), devices
        else:
            assert close(got, want), devices
    edm.devices = None


@pytest.mark.gpu
def test_per_molecule_mode_draws_its_seeds_once():
    ddpm, kw = gain_model("auto")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    d = kw['x'].device
    gen = torch.cuda.default_generators[0]
    torch.manual_seed(9)
    base = draw_seeds(B, d).cpu()
    off_after = gen.get_offset()
    edm.noise_mode = 'per_molecule'
    edm.nan_retries = 4                                                 # what an unmodified generate.py sets after accelerate()
    torch.manual_seed(9)
    chain = edm.sample_chain(**kw, keep_frames=3)
    assert gen.get_offset() == off_after                                # one torch.randint call, whatever the rounds
    assert torch.isfinite(chain).all()
    attempts = edm.last_attempts.tolist()
    for b in range(B):
        assert int(edm.last_seeds[b]) == retry_seed(int(base[b]), attempts[b])
    torch.manual_seed(9)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=3), chain)


@pytest.mark.gpu
def test_ddpm_passes_the_retries_through():
    ddpm, kw = gain_model("auto")
    d = kw['x'].device
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=len(GAIN_SEEDS))).items()}
    chain, _ = ddpm.sample_chain(data, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4)
    attempts = ddpm.edm.last_attempts
    want = ddpm.edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4)
    assert torch.equal(chain, want) and torch.equal(ddpm.edm.last_attempts, attempts) and attempts.any()


@pytest.mark.gpu
def test_c_caller_recovers_what_python_recovers(tmp_path):
    ddpm, kw = gain_model("auto")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    want = edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4).cpu()
    job, out = str(tmp_path / "job.bin"), str(tmp_path / "out.bin")
    meta = export_job.write_seeded_job(job, edm, **kw, keep_frames=3, seeds=GAIN_SEEDS, device_index=0)
    exe = helpers.build_c_example(tmp_path)
    res = subprocess.run([exe, "--retries", "4", job, out], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, (res.stdout, res.stderr)
    status, consumed, chain, flags, used, attempts = export_job.read_retry_result(out, B, meta["N"], 3, meta["xd"])
    assert status == 0 and consumed == 0 and not flags.any()
    assert torch.equal(chain, want)
    assert torch.equal(used, edm.last_seeds) and torch.equal(attempts, edm.last_attempts) and attempts.any()
