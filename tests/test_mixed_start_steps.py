"""Per-molecule start steps: EDM.sample_chain(start_step=[t0_0, t0_1, ...]) varies each molecule's linker from its own step
in one launch (dl_set_start_steps). Row b must equal row b of the single-step call start_step=t0_b on the same batch, with
the same seeds or noise rows: bit for bit on the SIMT edge path, within the per-molecule rule on the tensor-core path.

CPU: argument refusals, the oracle composed row by row against the reference's goldens, sample_many's launch keys with
per-request steps, and the C-ABI.
GPU, on both edge paths: a batch composed of the partial_cfg2_zinc goldens, equivalence with the single-step calls on FC
and pocket batches, the molecule-steps count, the recovery rounds and sample_many."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from difflinker_b200 import _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.distributed import plan_launches
from difflinker_b200.edm import StartSteps, retry_seed
from difflinker_b200.utils import FoundNaNException
import dl_helpers as helpers
import partial_diffusion_oracle as po
import test_sampler_steps_fp64 as steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INPUTS = ("x", "h", "node_mask", "fragment_mask", "linker_mask", "edge_mask", "context")


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def cfg1_model(**over):
    ddpm, hp = helpers.build_ddpm(synthetic.SPECS["cfg1_plumbing"], 0, **over)
    data = collate(synthetic.make_items(synthetic.SPECS["cfg1_plumbing"]))
    return ddpm, data


def golden_model(meta, impl='auto'):
    spec = synthetic.SPECS[meta["spec"]]
    ddpm, hp = helpers.build_ddpm(spec, meta["seed"], edge_impl=impl, diffusion_steps=meta["table_timesteps"])
    assert helpers.state_sha(ddpm.edm.dynamics.state_dict()) == meta["sha"], "seeded weights differ from the fixture's"
    ddpm.edm.T = meta["T"]
    return ddpm, hp, spec


# ---- CPU ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("bad", [[1, 2], [1, 2, 3, 4, 5], [0, 1, 2, 21], [0, -1, 2, 3], [0, 1.5, 2, 3], [True, 1, 2, 3],
                                 torch.tensor([0.0, 1.0, 2.0, 3.0]), torch.tensor([True, False, True, False])])
def test_a_step_sequence_must_hold_one_int_in_0_to_T_per_molecule(bad):
    ddpm, data = cfg1_model()
    ddpm.edm.T = 20
    kw = sampler_inputs(ddpm, data)
    assert kw['x'].shape[0] == 4
    with pytest.raises(ValueError, match="start_step"):
        ddpm.edm.sample_chain(**kw, start_step=bad)
    with pytest.raises(ValueError, match="start_step"):
        ddpm.edm.sample_many([kw], seeds=[[0] * 4], start_step=[bad])


def test_a_step_sequence_takes_ints_and_integer_tensors():
    ddpm, _ = cfg1_model()
    edm = ddpm.edm
    for steps_ in ([3, 0, 3, 50], (3, 0, 3, 50), torch.tensor([3, 0, 3, 50]), torch.tensor([3, 0, 3, 50], dtype=torch.int32)):
        st = edm._start(steps_, 4)
        assert isinstance(st, StartSteps) and st.t0 == [3, 0, 3, 50]
        for t0, a, s in zip(*st):
            assert (a, s) == edm.start_scalars(t0, 4)
    assert edm._start(7, 4) == (7,) + edm.start_scalars(7, 4)        # an int is the scalar form, unchanged


def test_inpainting_sample_fn_and_linker_sizes_refuse_a_step_sequence():
    ddpm, data = cfg1_model()
    with pytest.raises(ValueError, match="sample_fn"):
        ddpm.sample_chain(data, sample_fn=lambda d: d['linker_mask'].sum(1).view(-1).int(), start_step=[1, 2, 3, 4])
    with pytest.raises(ValueError, match="linker_sizes"):
        ddpm.sample_chain(data, seeds=[1, 2, 3, 4], linker_sizes=5, start_step=[1, 2, 3, 4])
    inp, data = cfg1_model(inpainting=True)
    kw = sampler_inputs(inp, data)
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.edm.sample_chain(**kw, start_step=[1, 2, 3, 4])


def mixed_oracle(parts, T, keep):
    """The chain of a batch composed of `parts` [(state_dict, cfg, gamma, t0, inputs, noise_fn, norm, rows)]: the oracle run
    once per part at that part's t0 on its whole batch, then rows `rows` of it, in order."""
    chains = []
    for sd, cfg, gam, t0, inputs, noise_fn, norm, rows in parts:
        with torch.no_grad():
            c = po.linker_partial_chain(sd, cfg, gam, T, t0, *inputs, keep_frames=keep, norm_values=norm, noise_fn=noise_fn)
        chains.append(c[:, rows])
    return torch.cat(chains, dim=1)


def test_the_composed_oracle_matches_the_composed_goldens():
    """Rows of the t1 and t50 goldens, each from its own fixture's oracle run, compose a mixed batch whose chain is the
    goldens' rows: frames with no writer below a row's own t0 are zero for that row alone."""
    keep = 10
    parts, want, t0s = [], [], []
    for t0, rows in ((50, [0, 3, 5]), (1, [1, 2, 7, 11])):
        meta, a = helpers.load_golden(f"partial_cfg2_zinc_t{t0}_k{keep}")
        ddpm, hp, _ = golden_model(meta)
        parts.append((ddpm.edm.dynamics.state_dict(), helpers.oracle_cfg(hp), steps.gamma_of(hp), t0,
                      [a[k] for k in INPUTS], helpers.seeded_noise(meta["noise_seed"]), tuple(hp['normalize_factors']), rows))
        want.append(a["chain"][:, rows])
        t0s += [t0] * len(rows)
    chain = mixed_oracle(parts, 500, keep)
    want = torch.cat(want, dim=1)
    assert (chain - want).abs().max().item() == 0.0
    for b, t0 in enumerate(t0s):
        written = po.written_frames(t0, 500, keep)
        for f in range(keep):
            assert (f in written) or not chain[f, b].any(), (b, f)


def test_per_request_steps_key_launches_by_the_coefficient_table_alone():
    ddpm, _ = cfg1_model()
    edm = ddpm.edm
    sizes, nodes = [3, 3, 40, 3, 40], [30, 31, 30, 32, 30]
    steps_ = [5, [1, 2, 3], 7, 0, list(range(40))]
    coefs, starts, keys = edm._launch_keys(sizes, nodes, 2, steps_)
    for k, (b, s) in enumerate(zip(sizes, steps_)):
        assert keys[k] == (bytes(coefs[b]), None, None)
        t0 = s if isinstance(s, list) else [s] * b
        assert starts[k] == StartSteps(t0, *map(list, zip(*(edm.start_scalars(t, b) for t in t0))))
    launches = plan_launches(sizes, nodes, 256, keys)
    assert sorted(k for ks, _ in launches for k in ks) == list(range(5))
    assert any(len({steps_[k] if isinstance(steps_[k], int) else -1 for k in ks}) > 1 for ks, _ in launches)
    # the scalar form plans exactly as before
    _, starts5, keys5 = edm._launch_keys(sizes, nodes, 2, 5)
    assert starts5[3] == (5,) + edm.start_scalars(5, 3) and [k[1] for k in keys5] == [starts5[b] for b in sizes]
    with pytest.raises(ValueError, match="start_step"):
        edm.sample_many([{}] * 2, seeds=[[0]] * 2, start_step=[1])


def test_library_exports_the_setter_and_the_header_compiles_as_c99(tmp_path):
    lib = _native.load_library()
    for name in ("dl_set_start_steps", "dl_last_molecule_steps"):
        assert hasattr(lib, name) and name in _native.SYMBOLS
    assert lib.dl_set_start_steps(None, 0, None, None, None) == -1      # DL_ERR_INVALID: no engine
    assert lib.dl_last_molecule_steps(None) == 0
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "starts.c"
    src.write_text('#include "difflinker_b200.h"\n'
                   "int main(void) {\n"
                   "  const int32_t t0[2] = {3, 1};\n"
                   "  const float alpha[2] = {0.5f, 0.9f}, sigma[2] = {0.8f, 0.4f};\n"
                   "  dl_status s = dl_set_start_steps((dl_engine*)0, 2, t0, alpha, sigma);\n"
                   "  int64_t n = dl_last_molecule_steps((dl_engine*)0);\n"
                   "  return s == DL_ERR_INVALID && n == 0 ? 0 : 1;\n"
                   "}\n")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib_dir = os.path.dirname(_native.LIB_PATH)
    exe = str(tmp_path / "starts")
    res = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", str(src), "-I" + os.path.join(ROOT, "include"),
                          "-L" + lib_dir, "-ldifflinker_b200", "-L" + os.path.join(cuda, "lib64"), "-lcudart",
                          "-Wl,-rpath," + lib_dir, "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-o", exe],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-3000:]
    assert subprocess.run([exe]).returncode == 0


# ---- GPU: helpers -------------------------------------------------------------------------------------------------------

def run_rows(edm, kw, keep, start, noise=None, seeds=None):
    """(chain, flags) of one engine call over the batch kw with `start` (a StartSteps with the caller's own scalars, or a
    scalar start), the draws of `noise` or `seeds`; the flags are kept even where a row diverges."""
    lib = _native.load_library()
    B = kw['x'].shape[0]
    d = kw['x'].device
    dev_i = edm.dynamics._device_index(kw['x'])
    engines = edm.dynamics.engines([(dev_i, 0)])
    dev_seeds = None if seeds is None else torch.tensor(seeds, dtype=torch.int64, device=d)
    calls, finish = edm._enqueue_batch(lib, edm._sampler_tensors(**kw), keep, edm.step_coefficients(keep, B),
                                       [(dev_i, 0, 0, B)], engines, [d], d, noise=noise, dev_seeds=dev_seeds, start=start)
    calls[0][1]()
    out = finish()
    return out['chain'], out['flags'].cpu(), engines[0]


def per_molecule_ok(got, want, rows, drift, scale):
    """The repository's per-molecule rule: max(1e-4 * scale, 30 * drift64) per molecule, at least half inside 1e-4 * scale."""
    err = ((got - want) * rows).abs().flatten(1).max(1).values
    tol = torch.maximum(torch.full_like(err, 1e-4 * scale), 30.0 * drift.float())
    assert (err <= tol).all(), (err.tolist(), tol.tolist())
    assert (err <= 1e-4 * scale).sum() >= (err.numel() + 1) // 2, (err.tolist(), 1e-4 * scale)


def take(kw, idx):
    """Rows `idx` of FC or pocket sampler inputs (an FC edge mask holds B blocks of N*N)."""
    B = kw['x'].shape[0]
    ix = torch.tensor(idx, device=kw['x'].device)
    out = {}
    for k, v in kw.items():
        out[k] = None if v is None else (v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:]) if k == 'edge_mask'
                                         else v[ix])
    return out


# ---- GPU: the goldens ---------------------------------------------------------------------------------------------------

# rows of each fixture in the composed batch: 25 molecules, below the 32 at which torch's CPU kernels start to round the
# step coefficients and start scalars differently from the fixtures' batches of 16 and 4
GOLDEN_ROWS = {1: [0, 4, 9, 15, 2, 7], 50: [1, 3, 8, 12, 14, 6, 10], 250: [0, 5, 11, 13, 2, 9, 15, 4], 500: [0, 1, 2, 3]}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("keep", [1, 10])
def test_a_batch_composed_of_the_goldens_meets_each_fixtures_checks(keep, impl):
    fixtures = {t0: helpers.load_golden(f"partial_cfg2_zinc_t{t0}_k{keep}") for t0 in GOLDEN_ROWS}
    assert len({meta["sha"] for meta, _ in fixtures.values()}) == 1, "the fixtures must share one model"
    meta0 = fixtures[1][0]
    ddpm, hp, spec = golden_model(meta0, impl)
    d = dev()
    ddpm = ddpm.to(d)
    T = meta0["T"]
    # interleave the fixtures' rows so that the engine's order differs from the caller's
    order = [(t0, j) for i in range(8) for t0 in (250, 1, 500, 50) if i < len(GOLDEN_ROWS[t0]) for j in [GOLDEN_ROWS[t0][i]]]
    t0max = max(GOLDEN_ROWS)
    B, N = len(order), fixtures[1][1]["x"].shape[1]
    noise = torch.zeros((t0max + 2, B, N, 3 + spec.F))
    full = {t0: helpers.noise_tensor(m["noise_seed"], t0, m["batch"], N, spec.F) for t0, (m, _) in fixtures.items()}
    for b, (t0, j) in enumerate(order):
        noise[:t0 + 2, b] = full[t0][:, j]
    kw = {k: torch.stack([fixtures[t0][1][k][j] for t0, j in order]).to(d) for k in INPUTS if k != 'edge_mask'}
    kw['edge_mask'] = torch.cat([fixtures[t0][1]['edge_mask'].reshape(fixtures[t0][0]["batch"], -1)[j] for t0, j in order]
                                ).reshape(-1, 1).to(d)
    start = StartSteps([t0 for t0, _ in order], [fixtures[t0][0]["alpha_t0"] for t0, _ in order],
                       [fixtures[t0][0]["sigma_t0"] for t0, _ in order])
    chain, flags, _ = run_rows(ddpm.edm, kw, keep, start, noise=noise.to(d))
    chain = chain.cpu()
    assert not flags.any()
    for b, (t0, j) in enumerate(order):
        meta, a = fixtures[t0]
        got, want = chain[:, b], a["chain"][:, j]
        nm, fm, lm = (a[k][j].float() for k in ("node_mask", "fragment_mask", "linker_mask"))
        assert torch.equal(got[0][..., 3:], want[0][..., 3:]), (b, t0, "atom types differ")
        fr = (fm[..., 0] != 0) & (lm[..., 0] == 0)
        assert torch.equal(got[0][..., :3][fr], a["x"][j][fr]), (b, t0, "a fragment row differs from the input")
        assert not got[:, nm[..., 0] == 0].any(), (b, t0, "a padded row is not 0")
        written = po.written_frames(t0, T, keep)
        for f in range(keep):
            if f not in written:
                assert not got[f].any(), (b, t0, f"frame {f} has no writer and is not 0")
                continue
            per_molecule_ok(got[f][None, ..., :3], want[f][None, ..., :3], lm[None], a["drift64"][j:j + 1],
                            a["chain"][f][..., :3].abs().max().item())
            if f > 0:
                assert torch.equal(got[f][fr], want[f][fr])


# ---- GPU: equivalence with the single-step calls ------------------------------------------------------------------------

def model(kind, impl, T=12, rows=7, gain=1.0):
    """(ddpm, data, sampler inputs) of a cfg2_zinc_ragged FC batch at T, or of the partial_cfg4_pockets 4A batch (its T = 1000
    model, on which its three molecules run from t0 = 100 without diverging) repeated to `rows` molecules."""
    if kind == "pocket":
        meta, a = helpers.load_golden("partial_cfg4_pockets_t100_k1")
        ddpm, _, _ = golden_model(meta, impl)
        d = dev()
        idx = [b % meta["batch"] for b in range(rows)]
        kw = {k: a[k][idx].to(d) for k in INPUTS if k != 'edge_mask'}
        kw['edge_mask'] = a['edge_mask'].reshape(meta["batch"], -1)[idx].reshape(-1).to(d)
        return ddpm.to(d), None, kw
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


def assert_row(got, want, impl, what):
    if impl == "simt":
        assert torch.equal(got, want), what
    else:
        assert (got - want).abs().max() <= 1e-4 * want.abs().max().clamp(min=1.0), what


MIXED = [12, 0, 5, 1, 12, 5, 3]        # 0, 1, T and duplicates, not in order
MIXED_POCKET = [100, 0, 40, 1, 100, 40, 7]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("kind", ["fc", "pocket"])
@pytest.mark.parametrize("keep", [1, 4])
@pytest.mark.parametrize("source", ["seeds", "tensor"])
def test_each_row_equals_its_single_step_call(source, keep, kind, impl):
    mixed = MIXED if kind == "fc" else MIXED_POCKET
    ddpm, data, kw = model(kind, impl, rows=len(mixed))
    edm = ddpm.edm
    lib = _native.load_library()
    B, N = kw['x'].shape[:2]
    seeds = [3, 1 << 62, -9, 77, 5, 12, 2024]
    noise = torch.randn((max(mixed) + 2, B, N, 3 + edm.in_node_nf), generator=torch.Generator().manual_seed(5)).to(kw['x'])
    draws = dict(seeds=seeds) if source == "seeds" else dict(noise=noise)
    chain = edm.sample_chain(**kw, keep_frames=keep, start_step=mixed, **draws)
    assert lib.dl_last_molecule_steps(edm.dynamics.engine(0)) == sum(t + 1 for t in mixed)
    for t0 in sorted(set(mixed)):
        d1 = dict(seeds=seeds) if source == "seeds" else dict(noise=noise[:t0 + 2])
        single = edm.sample_chain(**kw, keep_frames=keep, start_step=t0, **d1)
        assert lib.dl_last_molecule_steps(edm.dynamics.engine(0)) == B * (t0 + 1)
        for b in (b for b in range(B) if mixed[b] == t0):
            assert_row(chain[:, b], single[:, b], impl, (t0, b))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("kind", ["fc", "pocket"])
def test_an_all_equal_sequence_is_the_scalar_call_bit_for_bit(kind, impl):
    ddpm, data, kw = model(kind, impl)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(40, 40 + B))
    for t0 in (0, 7, 12):
        scalar = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, start_step=t0)
        rows = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, start_step=torch.full((B,), t0))
        assert torch.equal(scalar, rows), t0


@pytest.mark.gpu
def test_the_batch_stream_refuses_a_step_sequence():
    ddpm, data, kw = model("fc", "simt")
    with pytest.raises(ValueError, match="per-molecule"):
        ddpm.edm.sample_chain(**kw, keep_frames=2, start_step=MIXED)
    eng = ddpm.edm.dynamics.engine(0)
    lib = _native.load_library()
    n = len(MIXED)
    t0 = (ctypes.c_int32 * n)(*MIXED)
    al, sg = (ctypes.c_float * n)(*[0.5] * n), (ctypes.c_float * n)(*[0.5] * n)
    assert lib.dl_set_start_steps(eng, n, t0, al, (ctypes.c_float * n)(*[float('nan')] * n)) == -1
    assert lib.dl_set_start_steps(eng, n, (ctypes.c_int32 * n)(*[-1] * n), al, sg) == -1
    assert lib.dl_set_start_steps(eng, n, t0, al, sg) == 0
    try:
        with pytest.raises(_native.NativeError, match="molecules"):   # a call of another B
            ddpm.edm.sample_chain(**take(kw, [0, 1]), keep_frames=2, seeds=[1, 2])
    finally:
        lib.dl_set_start_steps(eng, 0, None, None, None)


# ---- GPU: recovery rounds and sample_many -------------------------------------------------------------------------------

GAIN_SEEDS = list(range(101, 125))


@pytest.mark.gpu
@pytest.mark.parametrize("connected", [False, True])
def test_recovered_rows_equal_their_single_step_call_with_the_seed_used(connected):
    ddpm, data, kw = model("fc", "simt", T=10, rows=len(GAIN_SEEDS), gain=5.0)
    edm = ddpm.edm
    B = len(GAIN_SEEDS)
    t0s = [(10, 10, 6, 3, 10, 8)[b % 6] for b in range(B)]
    extra = dict(require_connected=True) if connected else {}
    edm.is_geom = False
    try:
        chain = edm.sample_chain(**kw, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4, start_step=t0s, **extra)
    except FoundNaNException as exc:
        chain = exc.chain
    attempts, used = edm.last_attempts.tolist(), edm.last_seeds
    assert any(a > 0 for a in attempts), "the gain must make some rows diverge"
    for b in range(B):
        if not torch.isfinite(chain[:, b]).all():
            continue
        assert int(used[b]) == retry_seed(GAIN_SEEDS[b], attempts[b])
        alone = edm.sample_chain(**take(kw, [b]), keep_frames=3, seeds=[int(used[b])], start_step=t0s[b])
        assert torch.equal(chain[:, b], alone[:, 0]), b


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_sample_many_with_per_request_steps_equals_the_per_request_calls(impl):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    ddpm.edm.T = 12
    d = dev()
    ddpm = ddpm.to(d)
    datas = [{k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=b)).items()}
             for b in (3, 1, 5, 2)]
    seeds = [[11 * k + b for b in range(x['linker_mask'].shape[0])] for k, x in enumerate(datas)]
    steps_ = [12, 0, [6, 1, 12, 6, 0], 3]
    many = ddpm.sample_many(datas, keep_frames=3, seeds=seeds, start_step=steps_)
    assert len(ddpm.edm.last_loop_ms_many) < len(datas), "a sweep of steps must share launches"
    for k, data in enumerate(datas):
        want, nm = ddpm.sample_chain(data, keep_frames=3, seeds=seeds[k], start_step=steps_[k])
        assert torch.equal(many[k][1], nm), k
        if impl == "simt":
            assert torch.equal(many[k][0], want), k
        else:
            assert (many[k][0] - want).abs().max() <= 1e-4 * want.abs().max().clamp(min=1.0), k
