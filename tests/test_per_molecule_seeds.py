"""Per-molecule seeds: `sample_chain(..., seeds=)`, noise_mode='per_molecule', dl_sample_chain_seeded and seeded C jobs.

Molecule b of a seeded call draws what the reference draws for it sampled alone after torch.cuda.manual_seed(seeds[b]),
so its chain must not depend on its batch: not on its batch-mates, their order, the batch size, the padding or a split.
CPU tests cover the argument checks, the seed reduction and the seeded job layout; the GPU tests pin the stream to torch's
own through the reference_stream path and check every invariance on both edge paths."""
import struct
import subprocess

import pytest
import torch

from difflinker_b200 import _native, export_job, synthetic
from difflinker_b200 import distributed
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import draw_seeds, seeds_tensor
import dl_helpers as helpers
import egnn_options_oracle as eo

U64 = 1 << 64


# ---- CPU --------------------------------------------------------------------------------------------------------------

def test_seeds_are_reduced_as_torch_reduces_a_manual_seed():
    values = [0, 1, 7, -1, -2, -(1 << 63), (1 << 63) - 1, 1 << 63, U64 - 1, U64 - 2]
    t = seeds_tensor(values, len(values))
    assert t.dtype == torch.int64 and t.device.type == 'cpu'
    for v, s in zip(values, t.tolist()):
        want = torch.Generator().manual_seed(v).initial_seed()        # the binding torch.cuda.manual_seed goes through
        assert s % U64 == want == v % U64
        assert torch.Generator().manual_seed(s).initial_seed() == want  # the recorded value replays the same stream
    assert torch.equal(seeds_tensor(torch.tensor([3, -1]), 2), torch.tensor([3, -1]))
    assert torch.equal(seeds_tensor(torch.tensor([3, 4], dtype=torch.int32), 2), torch.tensor([3, 4]))
    assert seeds_tensor([U64 - 1], 1).item() == seeds_tensor([-1], 1).item() == -1
    for bad in ([U64], [-(1 << 63) - 1], [1.5], [True]):
        with pytest.raises(ValueError):
            seeds_tensor(bad, 1)
    with pytest.raises(ValueError, match="holds 2 values for a batch of 3"):
        seeds_tensor([1, 2], 3)
    with pytest.raises(ValueError):
        seeds_tensor(torch.tensor([1.0, 2.0]), 2)
    with pytest.raises(ValueError):
        seeds_tensor(torch.tensor([[1, 2]]), 2)


def _cpu_model(inpainting=False):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    over = {"inpainting": True} if inpainting else {}
    ddpm, _ = helpers.build_ddpm(spec, 0, **over)
    ddpm.edm.T = 4
    return ddpm, sampler_inputs(ddpm, collate(synthetic.make_items(spec, batch=3)))


@pytest.mark.parametrize("inpainting", [False, True])
def test_seeded_calls_refuse_what_cannot_take_the_per_molecule_stream(inpainting):
    ddpm, kw = _cpu_model(inpainting)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    with pytest.raises(ValueError, match="CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3])
    with pytest.raises(ValueError, match="both supply the draws"):
        edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3], noise=torch.zeros(1))
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3], batch_slice=(0, B))
    with pytest.raises(ValueError, match="holds 2 values"):
        edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2])
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="replaced"):
        edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3])
    delattr(edm, name)
    edm.noise_mode = 'per_molecule'
    with pytest.raises(ValueError, match="per_molecule.*CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2)
    assert edm.last_seeds is None
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, batch_slice=(0, B))


def test_default_noise_mode_is_unchanged():
    ddpm, _ = _cpu_model()
    assert ddpm.edm.noise_mode == 'reference_stream' and ddpm.edm.last_seeds is None


def _weights_bytes(edm):
    sd = edm.dynamics.dynamics.state_dict()
    return 4 + sum(4 + len(f"dynamics.{k}".encode()) + 8 + 4 * v.numel() for k, v in sd.items())


@pytest.mark.parametrize("options", [False, True])
def test_seeded_job_layout(tmp_path, options):
    """A seeded job is the (seed, offset) job of the same model with its own magic, an options flag (and the options) after
    the dl_config, and the B seeds as uint64 in place of the 16-byte generator state; the older versions stay as they were."""
    ddpm, _ = eo_ddpm(options)
    kw = sampler_inputs(ddpm, collate(synthetic.make_items(eo.OPTION_SPECS["small_fc"], batch=3)))
    old, new = str(tmp_path / "old.bin"), str(tmp_path / "new.bin")
    export_job.write_job(old, ddpm.edm, **kw, keep_frames=2, seed=1)
    seeds = [5, -1, U64 - 2]
    meta = export_job.write_seeded_job(new, ddpm.edm, **kw, keep_frames=2, seeds=seeds)
    b_old, b_new = open(old, "rb").read(), open(new, "rb").read()
    assert meta["B"] == 3
    head_old = 60 + (16 if options else 0)
    assert b_old[:8] == (b"DLJOB2\0\0" if options else b"DLJOB1\0\0") and b_new[:8] == b"DLJOB3\0\0"
    assert b_new[8:60] == b_old[8:60]
    assert struct.unpack_from("<i", b_new, 60)[0] == int(options)
    head_new = 64 + (16 if options else 0)
    assert b_new[64:head_new] == b_old[60:head_old]                   # the options, when present
    mid = _weights_bytes(ddpm.edm) + 24                               # weights, then B, N, T, keep_frames, xd, C
    assert b_new[head_new:head_new + mid] == b_old[head_old:head_old + mid]
    assert struct.unpack_from("<2Q", b_old, head_old + mid) == (1, 0)
    assert list(struct.unpack_from("<3Q", b_new, head_new + mid)) == [s % U64 for s in seeds]
    assert b_new[head_new + mid + 24:] == b_old[head_old + mid + 16:]


def eo_ddpm(options, **over):
    spec = eo.spec_with_options("small_fc", True, True, False) if options else eo.OPTION_SPECS["small_fc"]
    return helpers.build_ddpm(spec, 3, **over)


# ---- GPU --------------------------------------------------------------------------------------------------------------

CASES = ["default", "tanh_mean_sin", "pocket_FC-10A-4A", "inpainting"]
PADDING_CASES = ["default", "pocket_FC-10A-4A", "inpainting"]      # mean aggregation divides by the padded N on FC graphs
SEEDS = [11, -3, 1 << 63, 20240607, 5]


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def build(case, impl):
    """(edm on cuda:0 with T = 10, the sampler inputs of a ragged batch of 5 -- 4 for the pocket case, whose fifth molecule
    diverges on the reference stream)."""
    d = dev()
    if case == "default":
        spec, over, rows = synthetic.SPECS["cfg2_zinc_ragged"], {}, 5
    elif case == "tanh_mean_sin":
        spec, over, rows = eo.spec_with_options("opts_cfg1", True, True, True), {}, 5
    elif case == "pocket_FC-10A-4A":
        spec, over, rows = helpers.EXTRA_SPECS["small_pocket_FC-10A-4A"], {}, 4
    elif case == "inpainting":
        spec, over, rows = synthetic.SPECS["cfg2_zinc_ragged"], {"inpainting": True}, 5
    else:
        raise KeyError(case)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=5)).items()}
    kw = take(sampler_inputs(ddpm, data), list(range(rows)))
    return ddpm, kw


def take(kw, idx):
    """Rows `idx` (in that order, repeats allowed) of the sampler inputs; the edge mask holds B equal blocks."""
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


def pad(kw, extra):
    """The same molecules padded with `extra` dead atoms each."""
    B, N = kw['x'].shape[:2]
    out = {}
    for k, v in kw.items():
        if v is None:
            out[k] = None
        elif k == 'edge_mask':
            if v.shape[0] == B * N * N:                                  # FC: (B N N, 1)
                m = v.reshape(B, N, N, -1)
                out[k] = torch.nn.functional.pad(m, (0, 0, 0, extra, 0, extra)).reshape(-1, v.shape[-1])
            else:                                                       # pocket graphs: the per-node batch ids
                out[k] = torch.arange(B, device=v.device).repeat_interleave(N + extra).reshape(-1, *v.shape[1:]).to(v.dtype)
        else:
            out[k] = torch.nn.functional.pad(v, (0, 0, 0, extra))
    return out


def seeded(edm, kw, seeds, keep_frames=3):
    return edm.sample_chain(**kw, keep_frames=keep_frames, seeds=seeds)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", CASES)
def test_each_row_is_the_molecule_sampled_alone_on_the_reference_stream(case, impl):
    """Row b of a seeded batch equals, bit for bit, the chain of a batch holding only molecule b (same N), sampled on the
    reference stream after torch.cuda.manual_seed(seeds[b]) -- torch's own randn, which the suite pins to the reference."""
    ddpm, kw = build(case, impl)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = SEEDS[:B]
    gen = torch.cuda.default_generators[0]
    torch.manual_seed(1)
    off = gen.get_offset()
    chain = seeded(edm, kw, seeds)
    assert gen.get_offset() == off                                      # explicit seeds leave the generator alone
    assert torch.equal(edm.last_seeds, seeds_tensor(seeds, B))
    assert torch.isfinite(chain).all()
    for b in range(B):
        torch.cuda.manual_seed(seeds[b])
        alone = edm.sample_chain(**take(kw, [b]), keep_frames=3)
        assert edm.last_seeds is None
        assert torch.equal(chain[:, b:b + 1], alone), (case, impl, b)
    assert not torch.equal(chain[:, 0], chain[:, 1])


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", CASES)
def test_rows_do_not_depend_on_the_batch(case, impl):
    ddpm, kw = build(case, impl)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = SEEDS[:B]
    want = seeded(edm, kw, seeds)
    rev = list(range(B))[::-1]
    assert torch.equal(seeded(edm, take(kw, rev), [seeds[i] for i in rev]), want[:, rev])
    more = list(range(B)) + [1, 0, 2]                                   # the batch plus molecules under other seeds
    got = seeded(edm, take(kw, more), seeds + [101, 102, 103])
    assert torch.equal(got[:, :B], want)
    for b in (0, B - 1):
        assert torch.equal(seeded(edm, take(kw, [b]), [seeds[b]]), want[:, b:b + 1])
    twin = seeded(edm, take(kw, [2, 2, 2]), [seeds[2], seeds[2], 77])
    assert torch.equal(twin[:, 0], twin[:, 1]) and torch.equal(twin[:, 0], want[:, 2])
    assert not torch.equal(twin[:, 2], twin[:, 0])


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", PADDING_CASES)
def test_padding_changes_no_live_row(case, impl):
    ddpm, kw = build(case, impl)
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    seeds = SEEDS[:B]
    want = seeded(edm, kw, seeds)
    got = seeded(edm, pad(kw, 9), seeds)
    assert got.shape[2] == N + 9
    assert torch.equal(got[:, :, :N], want)
    assert not got[:, :, N:].any()


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", CASES)
def test_splits_reproduce_the_unsplit_seeded_chain(case, impl, monkeypatch):
    ddpm, kw = build(case, impl)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = SEEDS[:B]
    want = seeded(edm, kw, seeds)
    edm.devices = [0, 0, 0]
    gen = torch.cuda.default_generators[0]
    off = gen.get_offset()
    assert torch.equal(seeded(edm, kw, seeds), want)
    assert gen.get_offset() == off and torch.equal(edm.last_seeds, seeds_tensor(seeds, B))
    edm.devices = None
    # sample_chain_sharded on emulated ranks: each samples its rows with its rows of the seeds
    model = type("M", (), {})()
    model.edm = edm
    world = 3
    monkeypatch.setattr(distributed.dist, "is_available", lambda: True)
    monkeypatch.setattr(distributed.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(distributed.dist, "get_world_size", lambda: world)
    import difflinker_b200.ddpm as ddpm_mod
    monkeypatch.setattr(ddpm_mod, "sampler_inputs", lambda m, data, fn=None: kw)    # the batch is already prepared
    parts = []
    for r in range(world):
        monkeypatch.setattr(distributed.dist, "get_rank", lambda r=r: r)
        chain, _ = distributed.sample_chain_sharded(model, None, keep_frames=3, gather=False, seeds=seeds)
        parts.append(chain)
    assert torch.equal(torch.cat(parts, dim=1), want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["default", "inpainting"])
def test_per_molecule_mode_derives_seeds_from_the_generator(case):
    ddpm, kw = build(case, "auto")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    d = kw['x'].device
    gen = torch.cuda.default_generators[0]
    torch.manual_seed(9)
    expected = draw_seeds(B, d).cpu()
    off_after = gen.get_offset()
    edm.noise_mode = 'per_molecule'
    torch.manual_seed(9)
    first = edm.sample_chain(**kw, keep_frames=3)
    seeds1 = edm.last_seeds
    assert gen.get_offset() == off_after                                # the one documented call, nothing else
    assert seeds1.dtype == torch.int64 and seeds1.device.type == 'cpu' and torch.equal(seeds1, expected)
    torch.manual_seed(9)
    again = edm.sample_chain(**kw, keep_frames=3)
    assert torch.equal(again, first) and torch.equal(edm.last_seeds, seeds1)
    assert not torch.equal(edm.sample_chain(**kw, keep_frames=3), first)   # the generator moved on: fresh seeds
    for b in (0, B - 1):
        alone = edm.sample_chain(**take(kw, [b]), keep_frames=3, seeds=[int(seeds1[b])])
        assert torch.equal(alone, first[:, b:b + 1])
    edm.noise_mode = 'reference_stream'                                 # explicit seeds select the stream in any mode
    assert torch.equal(edm.sample_chain(**kw, keep_frames=3, seeds=seeds1), first)


@pytest.mark.gpu
def test_ddpm_passes_the_seeds_through():
    ddpm, _ = helpers.build_ddpm(synthetic.SPECS["cfg2_zinc_ragged"], 0)
    ddpm.edm.T = 10
    d = dev()
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=5)).items()}
    chain, nm = ddpm.sample_chain(data, keep_frames=3, seeds=SEEDS)
    want = ddpm.edm.sample_chain(**sampler_inputs(ddpm, data), keep_frames=3, seeds=SEEDS)
    assert torch.equal(chain, want) and torch.equal(ddpm.edm.last_seeds, seeds_tensor(SEEDS, 5))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["default", "tanh_mean_sin", "inpainting"])
def test_c_caller_samples_a_seeded_job(case, tmp_path):
    ddpm, kw = build(case, "auto")
    B = kw['x'].shape[0]
    seeds = SEEDS[:B]
    want = seeded(ddpm.edm, kw, seeds).cpu()
    job, out = str(tmp_path / "job.bin"), str(tmp_path / "out.bin")
    meta = export_job.write_seeded_job(job, ddpm.edm, **kw, keep_frames=3, seeds=seeds, device_index=0)
    exe = helpers.build_c_example(tmp_path)
    res = subprocess.run([exe, job, out], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, (res.stdout, res.stderr)
    status, consumed, chain, flags = export_job.read_result(out, meta["B"], meta["N"], meta["keep_frames"], meta["xd"])
    assert status == 0 and consumed == 0 and not flags.any()
    assert torch.equal(chain, want)


@pytest.mark.gpu
def test_null_seeds_pointer_is_invalid():
    ddpm, kw = build("default", "auto")
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    seeded(edm, kw, SEEDS[:B])                                         # engine built, weights uploaded
    lib = _native.load_library()
    t = edm._sampler_tensors(**kw)
    chain = torch.empty((3, B, N, 3 + edm.in_node_nf), device=kw['x'].device)
    flags = torch.zeros(B, dtype=torch.int32, device=kw['x'].device)
    st = lib.dl_sample_chain_seeded(edm.dynamics.engine(0), *edm._head(B, N, 3, t), None, edm.step_coefficients(3, B),
                                    edm._norm(), chain.data_ptr(), flags.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == -1 and b"null" in lib.dl_last_error()
    assert lib.dl_sample_chain_seeded(None, *edm._head(B, N, 3, t), None, edm.step_coefficients(3, B), edm._norm(),
                                      chain.data_ptr(), flags.data_ptr(), None) == -1
