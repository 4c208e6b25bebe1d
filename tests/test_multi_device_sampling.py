"""One sampling batch split over several local GPUs from one process (`EDM.devices`, `accelerate(ddpm, devices=...)`).

CPU tests cover the argument validation and the slice planning. GPU tests need one H100: a device listed several times gets
an engine per listing, so `devices=[0, 0]` exercises the whole split -- slicing, per-device threads, batch-global NaN
indices, gathering -- and must reproduce the single-device chain bit for bit (on the tensor-core path: while no sample
diverges, see test_split_chain_equals_the_single_device_chain). The tests with two GPUs or more skip on a machine with one."""
import threading
import time

import numpy as np
import pytest
import torch

import difflinker_b200
from difflinker_b200 import EDM, FoundNaNException, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.distributed import device_slices, place_rows, resolve_devices, shard_range
import dl_helpers as helpers
import egnn_options_oracle as eo


# ---- CPU: argument validation and slice planning ---------------------------------------------------------------------

def test_resolve_devices_validates_indices():
    assert resolve_devices(None, 2) is None
    assert resolve_devices('all', 3) == [0, 1, 2]
    assert resolve_devices([1, 0, 1], 2) == [1, 0, 1]
    assert resolve_devices((np.int64(1),), 2) == [1]
    with pytest.raises(ValueError, match="empty"):
        resolve_devices([], 2)
    with pytest.raises(ValueError, match="unknown CUDA device 2"):
        resolve_devices([0, 2], 2)
    with pytest.raises(ValueError, match="unknown CUDA device -1"):
        resolve_devices([-1], 2)
    with pytest.raises(ValueError, match="no CUDA device"):
        resolve_devices('all', 0)
    with pytest.raises(ValueError):
        resolve_devices('cuda:0', 2)
    with pytest.raises(TypeError):
        resolve_devices([True], 2)
    with pytest.raises(TypeError):
        resolve_devices([0.0], 2)


def test_devices_setting_on_the_sampler_and_the_public_entry_points(monkeypatch):
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 2)
    spec = synthetic.SPECS["cfg1_plumbing"]
    ddpm, hp = helpers.build_ddpm(spec, 0)
    assert ddpm.edm.devices is None                                  # default: the data's device
    ddpm.edm.devices = 'all'
    assert ddpm.edm.devices == [0, 1]
    with pytest.raises(ValueError):
        ddpm.edm.devices = [2]
    assert ddpm.edm.devices == [0, 1]                                # a refused value leaves the setting as it was
    edm = difflinker_b200.DDPM(**hp, devices=[1, 1]).edm
    assert isinstance(edm, EDM) and edm.devices == [1, 1]
    assert 'devices' not in difflinker_b200.DDPM(**hp, devices=[1]).hparams
    inpaint = difflinker_b200.DDPM(**dict(hp, inpainting=True), devices=[0]).edm
    assert type(inpaint).__name__ == 'InpaintingEDM' and inpaint.devices == [0]
    # accelerate: the setting travels with the swapped-in sampler; a bad list leaves the module untouched
    before = ddpm.edm
    with pytest.raises(ValueError):
        difflinker_b200.accelerate(ddpm, devices=[])
    assert ddpm.edm is before
    assert difflinker_b200.accelerate(ddpm, devices=[0, 1]).edm.devices == [0, 1]
    assert difflinker_b200.accelerate(ddpm).edm.devices is None


def test_device_slices_are_contiguous_balanced_and_drop_empty_ones():
    assert device_slices(7, [0, 0, 0]) == [(0, 0, 0, 3), (0, 1, 3, 5), (0, 2, 5, 7)]
    assert device_slices(64, [0, 1, 2, 3, 4, 5, 6, 7]) == [(d, 0, 8 * d, 8 * d + 8) for d in range(8)]
    assert device_slices(5, [1, 0, 1]) == [(1, 0, 0, 2), (0, 0, 2, 4), (1, 1, 4, 5)]
    assert device_slices(2, [0, 1, 2, 3]) == [(0, 0, 0, 1), (1, 0, 1, 2)]         # B < number of devices
    assert device_slices(0, [0, 1]) == []
    for B in range(1, 40):
        for devices in ([0], [0, 1], [0, 0, 0], [3, 1, 2, 0, 4]):
            s = device_slices(B, devices)
            assert [lo for *_, lo, _ in s] == [0] + [hi for *_, hi in s[:-1]] and s[-1][3] == B
            sizes = [hi - lo for *_, lo, hi in s]
            assert max(sizes) - min(sizes) <= 1 and min(sizes) >= 1
            assert all((lo, hi) == shard_range(B, i, len(devices)) for i, (*_, lo, hi) in enumerate(s))


def test_per_slice_nan_flags_map_to_batch_global_indices():
    slices = device_slices(7, [0, 0, 0])                              # rows [0,3), [3,5), [5,7)
    parts = [torch.tensor([0, 0, 0], dtype=torch.int32),
             torch.tensor([0, 3 | (4 << 8)], dtype=torch.int32),      # molecule 4: coordinates and features, step 3
             torch.tensor([1 | (9 << 8), 2 | (6 << 8)], dtype=torch.int32)]
    flags = place_rows(torch.zeros(7, dtype=torch.int32), parts, slices)
    assert flags.tolist() == [0, 0, 0, 0, 3 | (4 << 8), 1 | (9 << 8), 2 | (6 << 8)]
    e = FoundNaNException(flags=flags.tolist())
    assert e.x_h_nan_idx == {4} and e.only_x_nan_idx == {5} and e.only_h_nan_idx == {6} and e.first_step == 3
    chain = place_rows(torch.zeros(2, 7, 1, 1), [torch.full((2, hi - lo, 1, 1), float(i)) for i, (*_, lo, hi) in
                                                 enumerate(slices)], slices, dim=1)
    assert chain[:, :, 0, 0].tolist() == [[0, 0, 0, 1, 1, 2, 2]] * 2


def test_per_device_threads_are_all_joined_before_an_error_propagates():
    """Each device's calls run in order on a thread of their own; when one fails, the others still finish and every thread
    has ended before the error reaches the caller."""
    from difflinker_b200.edm import _run_per_device
    done, before = [], set(threading.enumerate())

    def fail():
        raise RuntimeError("engine on device 0 failed")

    def slow(tag):
        time.sleep(0.2)
        done.append(tag)
    with pytest.raises(RuntimeError, match="device 0 failed"):
        _run_per_device({0: [fail, lambda: done.append("never")], 1: [lambda: slow("a"), lambda: slow("b")]})
    assert done == ["a", "b"] and set(threading.enumerate()) == before
    _run_per_device({0: [lambda: done.append(0)], 3: [lambda: done.append(3)]})
    assert sorted(done[2:]) == [0, 3] and set(threading.enumerate()) == before


# ---- GPU --------------------------------------------------------------------------------------------------------------

def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def to_dev(data, d):
    return {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in data.items()}


def build(case, impl="auto"):
    """(ddpm on cuda:0, data on cuda:0) of one test case; T is shortened through the edm.T override (generate.py:103-104)."""
    d = dev()
    if case == "cfg1_fc":
        spec, over, batch = synthetic.SPECS["cfg1_plumbing"], {}, None
    elif case == "ragged_B7":
        spec, over, batch = synthetic.SPECS["cfg2_zinc_ragged"], {}, 7
    elif case == "pocket_FC-10A-4A":
        spec, over, batch = helpers.EXTRA_SPECS["small_pocket_FC-10A-4A"], {}, 5
    elif case == "inpainting":
        spec, over, batch = synthetic.SPECS["cfg2_zinc_ragged"], {"inpainting": True}, 7
    elif case == "tanh_mean":
        spec, over, batch = eo.spec_with_options("opts_cfg1", True, True, False), {}, None
    else:
        raise KeyError(case)
    ddpm, hp = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    return ddpm, to_dev(collate(synthetic.make_items(spec, batch=batch)), d)


def two_calls(ddpm, data, devices, seed=5, keep_frames=3):
    """Two consecutive ddpm.sample_chain calls from torch.manual_seed(seed) with `devices`: the chains, the node mask of the
    first, and the generator offset after each call."""
    gen = torch.cuda.default_generators[0]
    ddpm.edm.devices = devices
    torch.manual_seed(seed)
    first, nm = ddpm.sample_chain(data, keep_frames=keep_frames)
    off1 = gen.get_offset()
    second, _ = ddpm.sample_chain(data, keep_frames=keep_frames)
    return first, second, nm, off1, gen.get_offset()


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case,devices", [("cfg1_fc", [0, 0]), ("ragged_B7", [0, 0, 0]), ("pocket_FC-10A-4A", [0, 0]),
                                          ("inpainting", [0, 0, 0]), ("tanh_mean", [0, 0]), ("cfg1_fc", [0, 0, 0, 0, 0, 0])])
def test_split_chain_equals_the_single_device_chain(case, devices, impl):
    """The split chain is the single-device chain bit for bit, on the caller's device, for even and uneven splits and for
    more devices than molecules (cfg1 has 4 molecules: two listings get nothing); the generator ends where one device leaves
    it after each call, so a second call continues the stream identically.
    One exception, on the tensor-core path: in the pocket case's second draw molecule 4 diverges (|x| ~ 4e3), which makes
    the kernels rescale the fp16 operands of the tiles holding its rows by a power of two chosen per tile. Tile extents
    depend on the batch, so after the split that molecule rounds differently (the SIMT path, fp32 throughout, stays exact):
    the chains then agree to 1e-6 relative."""
    ddpm, data = build(case, impl)
    want1, want2, want_nm, want_off1, want_off2 = two_calls(ddpm, data, None)
    got1, got2, nm, off1, off2 = two_calls(ddpm, data, devices)
    B = want1.shape[1]
    assert got1.device == want1.device and got1.shape == want1.shape
    assert torch.equal(got1, want1) and torch.equal(nm, want_nm)
    if (case, impl) == ("pocket_FC-10A-4A", "auto"):
        assert (got2 - want2).abs().max().item() <= 1e-6 * want2.abs().max().item()
    else:
        assert torch.equal(got2, want2)
    assert not torch.equal(got2, got1)
    assert (off1, off2) == (want_off1, want_off2) and off1 > 0
    slices = ddpm.edm.last_slice_loop_ms
    assert [(lo, hi) for _, lo, hi, _ in slices] == [(lo, hi) for *_, lo, hi in device_slices(B, devices)]
    assert len(slices) == min(B, len(devices)) and ddpm.edm.last_loop_ms == max(ms for *_, ms in slices) > 0


@pytest.mark.gpu
def test_split_leaves_the_single_device_path_as_it_was():
    """Single-device calls after split ones sample exactly what they sampled before. Each listing of a device has an engine
    of its own (replica 0 is the single-device engine); a single-device call keeps only its own engine, as a module used on
    one device always did."""
    ddpm, data = build("ragged_B7")
    want, _, _, _, _ = two_calls(ddpm, data, None)
    two_calls(ddpm, data, [0, 0, 0])
    dyn = ddpm.edm.dynamics
    assert sorted(dyn._engines) == [(0, 0), (0, 1), (0, 2)]
    engines = [h.value for h in dyn.engines([(0, 0), (0, 1), (0, 2)])]
    assert len(set(engines)) == 3
    got, _, _, _, _ = two_calls(ddpm, data, None)
    assert torch.equal(got, want) and ddpm.edm.last_slice_loop_ms is None
    assert list(dyn._engines) == [(0, 0)] and dyn.engine(0).value == engines[0]
    two_calls(ddpm, data, [0, 0])                                     # split again: the released replica is re-created
    assert sorted(dyn._engines) == [(0, 0), (0, 1)]


@pytest.mark.gpu
def test_changed_weights_reach_every_engine():
    """The weights are read from the module again only when a parameter changed -- and then every device's engine gets them."""
    ddpm, data = build("cfg1_fc")
    two_calls(ddpm, data, [0, 0])
    with torch.no_grad():
        for p in ddpm.edm.dynamics.parameters():
            p.mul_(1.01)
    want, _, _, _, _ = two_calls(ddpm, data, None)
    got, _, _, _, _ = two_calls(ddpm, data, [0, 0])
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_nan_in_the_second_slice_raises_with_batch_global_indices():
    """A molecule whose input coordinates hold a NaN (the construction of test_gpu_parity.py's NaN test, on the sampler's
    input) poisons only itself; placed in the second of two slices, the exception's three index sets and first step are the
    single-device ones, and the generator is advanced as on one device."""
    ddpm, data = build("cfg1_fc")
    kw = sampler_inputs(ddpm, data)
    k = 3                                                             # slices [0, 2) and [2, 4)
    atom = int(torch.nonzero(kw['fragment_mask'][k, :, 0])[0])
    kw['x'][k, atom, 0] = float('nan')
    gen = torch.cuda.default_generators[0]
    raised = []
    for devices in (None, [0, 0]):
        ddpm.edm.devices = devices
        torch.manual_seed(3)
        with pytest.raises(FoundNaNException) as ei:
            ddpm.edm.sample_chain(**kw, keep_frames=2)
        e = ei.value
        raised.append((e.x_h_nan_idx, e.only_x_nan_idx, e.only_h_nan_idx, e.first_step, gen.get_offset()))
    assert raised[1] == raised[0]
    assert k in raised[0][0] | raised[0][1] | raised[0][2]
    # and every engine samples again afterwards
    kw['x'][k, atom, 0] = 0.0
    assert torch.isfinite(ddpm.edm.sample_chain(**kw, keep_frames=2)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ragged_B7", "inpainting"])
def test_injected_noise_tensor_is_split_by_rows(case):
    """noise= keeps its meaning: each slice samples its rows of the injected tensor."""
    ddpm, data = build(case)
    kw = sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    edm = ddpm.edm
    if case == "inpainting":
        noise = helpers.inpaint_noise_tensor(7, edm.T, B, N, edm.in_node_nf, kw['node_mask'].cpu(), kw['fragment_mask'].cpu())
    else:
        noise = helpers.noise_tensor(7, edm.T, B, N, edm.in_node_nf)
    noise = noise.to(kw['x'].device)
    edm.devices = None
    want = edm.sample_chain(**kw, keep_frames=3, noise=noise)
    edm.devices = [0, 0, 0]
    got = edm.sample_chain(**kw, keep_frames=3, noise=noise)
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_replaced_draw_noise_and_reference_tensor_mode_draw_the_whole_batch_once():
    """An overridden draw_noise, or noise_mode='reference_tensor', draws the full batch once on the caller's device; the
    slices sample its rows."""
    ddpm, data = build("ragged_B7")
    calls = []

    def draw(n_draws, n_samples, n_nodes, device, generator=None):
        calls.append(n_samples)
        return EDM.draw_noise(ddpm.edm, n_draws, n_samples, n_nodes, device, generator)
    ddpm.edm.draw_noise = draw
    want, want2, _, off1, off2 = two_calls(ddpm, data, None)
    got, got2, _, g1, g2 = two_calls(ddpm, data, [0, 0, 0])
    assert calls == [7] * 4 and torch.equal(got, want) and torch.equal(got2, want2) and (g1, g2) == (off1, off2)
    del ddpm.edm.draw_noise
    ddpm.edm.noise_mode = 'reference_tensor'
    got3, _, _, _, _ = two_calls(ddpm, data, [0, 0, 0])
    assert torch.equal(got3, want)                                    # the tensor the device-side stream stands for


@pytest.mark.gpu
def test_accelerate_with_devices_samples_the_same_chain():
    ddpm, data = build("ragged_B7")
    want, _, _, _, _ = two_calls(ddpm, data, None)
    ddpm = difflinker_b200.accelerate(ddpm, devices=[0, 0])
    torch.manual_seed(5)
    got, _ = ddpm.sample_chain(data, keep_frames=3)
    assert torch.equal(got, want)


def _need_gpus(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip(f"needs {n} visible GPUs")


@pytest.mark.gpu
@pytest.mark.parametrize("devices", [[0, 1], 'all', [1, 0, 1]])
def test_several_gpus_reproduce_the_single_gpu_chain(devices):
    _need_gpus(2)
    ddpm, data = build("ragged_B7")
    want1, want2, _, off1, off2 = two_calls(ddpm, data, None)
    got1, got2, _, g1, g2 = two_calls(ddpm, data, devices)
    assert got1.device == torch.device("cuda", 0)
    assert torch.equal(got1, want1) and torch.equal(got2, want2) and (g1, g2) == (off1, off2)
    used = {d for d, *_ in ddpm.edm.last_slice_loop_ms}
    assert used == set(ddpm.edm.devices[:7])
