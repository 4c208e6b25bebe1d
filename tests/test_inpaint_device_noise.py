"""InpaintingEDM with device-side noise: the 2T+3 masked, centre-of-mass-free draws of `draw_noise_inpaint` regenerated inside
the per-molecule kernel from the torch generator's (seed, offset) (dl_sample_chain_rng with DL_SAMPLER_INPAINT,
dl_noise_fill_inpaint), batch slices of an inpainting model, and the plain C caller on an inpainting job."""
import ctypes as C

import pytest
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
import dl_helpers as helpers


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def rel_err(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.double().abs().max().item(), 1e-30)


def to_dev(data, d):
    return {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in data.items()}


def ragged_masks(B, N, seed):
    """(B,N,1) float node and fragment masks: ragged molecule sizes, fragment atoms a random subset of each molecule's
    atoms, and molecule 1 without fragment atoms (its q draws are 0/0 in the reference's projection)."""
    g = torch.Generator().manual_seed(seed)
    sizes = torch.randint(N // 2, N + 1, (B,), generator=g)
    sizes[0] = N
    node = (torch.arange(N)[None, :] < sizes[:, None]).float()
    frag = node * (torch.rand((B, N), generator=g) < 0.6).float()
    frag[1] = 0.0
    return node[..., None], frag[..., None]


@pytest.mark.gpu
@pytest.mark.parametrize("spec_name,B,N,T", [("cfg1_plumbing", 4, 30, 3), ("cfg2_zinc", 256, 40, 2), ("cfg3_geom", 512, 300, 2)])
def test_device_inpaint_draws_equal_the_prepared_tensor(spec_name, B, N, T):
    """dl_noise_fill_inpaint writes the (2T+3,B,N,3+F) tensor that draw_noise_inpaint draws from the same generator state: the
    feature columns and every masked row bit for bit, the projected coordinates within 2e-6 (each molecule's sums are
    taken in a fixed order of the kernel's own), zero centre of mass on every slab, the same generator advance. The
    (512,300) case needs more than one randn grid per call; the generator does not start at offset 0."""
    from difflinker_b200 import _native
    lib = _native.load_library()
    d = dev()
    spec = synthetic.SPECS[spec_name]
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    edm = ddpm.edm
    edm.T = T
    eng = edm.dynamics.engine(d.index or 0)
    nm, fm = (m.to(d) for m in ragged_masks(B, N, 7 + B))
    torch.manual_seed(4321 + B)
    for _ in range(3):
        torch.randn((7, 13), device=d)
    gen = torch.cuda.default_generators[d.index or 0]
    seed, offset = gen.initial_seed(), gen.get_offset()
    assert offset > 0
    got = torch.empty((2 * T + 3, B, N, 3 + spec.F), device=d)
    used = C.c_uint64(0)
    nm8 = nm.reshape(B, N).to(torch.int8).contiguous()
    fm32 = fm.reshape(B, N).contiguous()
    with torch.cuda.device(d):
        _native.check(lib.dl_noise_fill_inpaint(eng, T, B, N, nm8.data_ptr(), fm32.data_ptr(), seed, offset, got.data_ptr(),
                                                C.byref(used), torch.cuda.current_stream(d).cuda_stream),
                      "dl_noise_fill_inpaint")
    want = edm.draw_noise_inpaint(B, N, d, nm, fm)
    assert gen.get_offset() == offset + used.value
    assert torch.equal(got[..., 3:], want[..., 3:])
    masks = torch.stack([nm] + [nm, fm] * T + [nm, nm])                   # (2T+3,B,N,1), the order of draw_noise_inpaint
    off = (masks == 0).expand_as(got)
    torch.testing.assert_close(got[off], want[off], rtol=0, atol=0, equal_nan=True)
    gx, wx = got[..., :3], want[..., :3]
    assert torch.equal(torch.isnan(gx), torch.isnan(wx))
    assert torch.isnan(wx[2, 1]).all() and not torch.isnan(wx[1]).any()     # the fragment-free molecule: 0/0, as in torch
    ok = ~torch.isnan(wx)
    err = (gx[ok] - wx[ok]).abs().max().item()
    print(f"\n[{spec_name} B={B} N={N}] max |coordinate difference| = {err:.3g}")
    assert err <= 2e-6
    m = masks.double()
    com = (gx.double() * m).sum(2) / m.sum(2)                               # (2T+3,B,3)
    com = com[~torch.isnan(com)]
    assert com.abs().max().item() <= 1e-6


CHAIN_CASES = [("cfg1_plumbing", None, None, 1e-5), ("cfg2_zinc_ragged", 256, 20, 1e-5),
               ("small_pocket_FC-10A-4A", None, None, 1e-4)]


@pytest.mark.gpu
@pytest.mark.parametrize("spec_name,batch,T,tol", CHAIN_CASES)
def test_inpainting_chain_with_device_noise_matches_the_prepared_tensor_chain(spec_name, batch, T, tol):
    """DDPM(inpainting=True).sample_chain draws inside the kernels by default on CUDA; from the same seed it matches the chain
    sampled from draw_noise_inpaint's tensor (noise_mode='reference_tensor') -- identical atom types, every frame within
    `tol` -- and leaves the generator at the same offset. The frames of the reverse steps are centre-of-mass free."""
    spec = helpers.spec_by_name(spec_name)
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    if T is not None:
        ddpm.edm.T = T
    d = dev()
    ddpm = ddpm.to(d)
    data = to_dev(collate(synthetic.make_items(spec, batch=batch)), d)
    gen = torch.cuda.default_generators[d.index or 0]
    keep = 4
    torch.manual_seed(31)
    chain_dev, nm = ddpm.sample_chain(data, keep_frames=keep)
    end_dev = gen.get_offset()
    torch.manual_seed(31)
    ddpm.edm.noise_mode = 'reference_tensor'
    chain_ten, _ = ddpm.sample_chain(data, keep_frames=keep)
    assert gen.get_offset() == end_dev
    assert torch.equal(chain_dev[0][..., 3:], chain_ten[0][..., 3:]), "atom types differ"
    errs = [rel_err(chain_dev[f], chain_ten[f]) for f in range(keep)]
    print(f"\n[{spec_name}] max relative frame difference per frame: {[f'{e:.3g}' for e in errs]}")
    assert max(errs) <= tol, errs
    # frame 0 mixes the linker and fragment variants of the final step (edm.py:716-725) and is not projected
    m = nm.double()
    for chain in (chain_dev, chain_ten):
        com = (chain[1:, ..., :3].double() * m).sum(2) / m.sum(1)
        assert com.abs().max().item() <= 1e-5


@pytest.mark.gpu
def test_replaced_draw_noise_inpaint_takes_the_tensor_path(monkeypatch):
    """An instance attribute, a subclass or a class-level patch of draw_noise_inpaint supplies the draws, as before."""
    from difflinker_b200 import InpaintingEDM
    spec = synthetic.SPECS["cfg1_plumbing"]
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    ddpm.edm.T = 4
    d = dev()
    ddpm = ddpm.to(d)
    data = to_dev(collate(synthetic.make_items(spec)), d)
    original = InpaintingEDM.draw_noise_inpaint
    calls = []

    def counted(self, *a, **k):
        calls.append(1)
        return original(self, *a, **k)
    ddpm.edm.draw_noise_inpaint = counted.__get__(ddpm.edm)
    ddpm.sample_chain(data, keep_frames=1)
    assert len(calls) == 1
    del ddpm.edm.draw_noise_inpaint
    monkeypatch.setattr(InpaintingEDM, "draw_noise_inpaint", counted)
    ddpm.sample_chain(data, keep_frames=1)
    assert len(calls) == 2
    monkeypatch.undo()
    ddpm.sample_chain(data, keep_frames=1)
    assert len(calls) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_inpainting_batch_slices_reproduce_the_single_gpu_chain(world):
    """Strong scaling of an inpainting model, emulated on one GPU: the slices sampled with batch_slice=(lo, B) from the same
    generator state concatenate to the unsplit device-stream chain bit for bit (each molecule's projection sums only its own
    rows of the full-batch draws)."""
    from difflinker_b200.ddpm import sampler_inputs
    from difflinker_b200.distributed import shard_range, slice_sampler_inputs
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    ddpm.edm.T = 12
    d = dev()
    ddpm = ddpm.to(d)
    data = to_dev(collate(synthetic.make_items(spec, batch=7)), d)
    torch.manual_seed(5)
    full, _ = ddpm.sample_chain(data, keep_frames=2)
    end = torch.cuda.default_generators[d.index or 0].get_offset()
    kw = sampler_inputs(ddpm, data)
    parts = []
    for r in range(world):
        lo, hi = shard_range(7, r, world)
        torch.manual_seed(5)
        parts.append(ddpm.edm.sample_chain(**slice_sampler_inputs(kw, lo, hi), keep_frames=2, batch_slice=(lo, 7)))
        assert torch.cuda.default_generators[d.index or 0].get_offset() == end
    assert torch.equal(torch.cat(parts, dim=1), full)


@pytest.mark.gpu
def test_sharded_sampling_of_an_inpainting_model_at_world_size_one():
    """distributed.sample_chain_sharded passes batch_slice to InpaintingEDM.sample_chain like to EDM.sample_chain."""
    from difflinker_b200.distributed import sample_chain_sharded
    spec = synthetic.SPECS["cfg1_plumbing"]
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    ddpm.edm.T = 10
    d = dev()
    ddpm = ddpm.to(d)
    data = to_dev(collate(synthetic.make_items(spec)), d)
    torch.manual_seed(8)
    want, want_nm = ddpm.sample_chain(data, keep_frames=2)
    torch.manual_seed(8)
    got, nm = sample_chain_sharded(ddpm, data, keep_frames=2)
    assert torch.equal(got, want) and torch.equal(nm, want_nm)


@pytest.mark.gpu
def test_plain_c_caller_samples_the_inpainting_chain_the_python_entry_produces(tmp_path):
    """examples/c_sampler.c on a job exported from an InpaintingEDM (config centering = 1, qa/qb in the coefficient table)
    samples through dl_sample_chain_rng(DL_SAMPLER_INPAINT): the chain InpaintingEDM.sample_chain gives in Python for a
    generator in that state, bit for bit, and the same generator advance."""
    import subprocess
    from difflinker_b200 import export_job
    from difflinker_b200.ddpm import sampler_inputs
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    ddpm.edm.T = 25
    d = dev()
    ddpm = ddpm.to(d)
    data = to_dev(collate(synthetic.make_items(spec, batch=6)), d)
    kw = sampler_inputs(ddpm, data)
    seed = 20240607
    torch.manual_seed(seed)
    torch.randn((5, 5), device=d)
    gen = torch.cuda.default_generators[d.index or 0]
    off0 = gen.get_offset()
    want = ddpm.edm.sample_chain(**kw, keep_frames=3).cpu()
    job, out = str(tmp_path / "job.bin"), str(tmp_path / "out.bin")
    meta = export_job.write_job(job, ddpm.edm, **kw, keep_frames=3, seed=seed, offset=off0, device_index=d.index or 0)
    exe = helpers.build_c_example(tmp_path)
    res = subprocess.run([exe, job, out], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, (res.stdout, res.stderr)
    status, consumed, chain, flags = export_job.read_result(out, meta["B"], meta["N"], meta["keep_frames"], meta["xd"])
    assert status == 0 and not flags.any()
    assert consumed == gen.get_offset() - off0
    assert torch.equal(chain, want)


def test_inpainting_batch_slice_needs_the_device_stream():
    """batch_slice selects rows of the device-side draws; with CPU tensors (host-buffer path) it is refused before any work."""
    spec = synthetic.SPECS["cfg1_plumbing"]
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=True)
    from difflinker_b200.ddpm import sampler_inputs
    kw = sampler_inputs(ddpm, collate(synthetic.make_items(spec)))
    with pytest.raises(ValueError, match="batch_slice"):
        ddpm.edm.sample_chain(**kw, keep_frames=1, batch_slice=(0, 8))
