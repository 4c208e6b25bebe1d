"""Many requests in shared launches: `EDM.sample_many`, `DDPM.sample_many` and the launch plan in distributed.py.

With per-molecule seeds a molecule's chain does not depend on its batch, so requests can share a reverse loop and each still
get exactly what its own sample_chain call returns. CPU tests cover the plan, the dealing of launches to devices, the argument
checks and the packing of requests into a launch and back; the GPU tests compare sample_many with the sequence of sample_chain
calls on both edge paths."""
import pytest
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.distributed import deal_launches, pack_requests, plan_launches, unpack_rows
from difflinker_b200.edm import seeds_tensor
from difflinker_b200.utils import FoundNaNException
import dl_helpers as helpers
import egnn_options_oracle as eo


# ---- CPU: the plan --------------------------------------------------------------------------------------------------------

def _check_plan(plan, sizes, nodes, max_molecules):
    seen = sorted(k for ks, _ in plan for k in ks)
    assert seen == list(range(len(sizes)))                              # every request once, none split
    for ks, n in plan:
        assert n == max(nodes[k] for k in ks)
        total = sum(sizes[k] for k in ks)
        assert total <= max_molecules or len(ks) == 1, (ks, total)


def test_the_plan_covers_every_request_once_within_the_limit():
    g = torch.Generator().manual_seed(5)
    for trial in range(50):
        K = int(torch.randint(1, 40, (1,), generator=g))
        sizes = torch.randint(1, 80, (K,), generator=g).tolist()
        nodes = torch.randint(20, 60, (K,), generator=g).tolist()
        m = int(torch.randint(1, 160, (1,), generator=g))
        plan = plan_launches(sizes, nodes, m)
        _check_plan(plan, sizes, nodes, m)
        assert plan == plan_launches(list(sizes), list(nodes), m)     # deterministic
    sizes, nodes = [10] * 64, [30 + k % 16 for k in range(64)]
    plan = plan_launches(sizes, nodes, 256)
    assert [sum(sizes[k] for k in ks) for ks, _ in plan] == [250, 250, 140]
    assert [n for _, n in plan] == sorted(n for _, n in plan)           # grouped by N: little padding


def test_a_request_larger_than_the_limit_gets_a_launch_of_its_own():
    plan = plan_launches([2, 300, 3, 1], [40, 30, 35, 50], 256)
    assert ([1], 30) in plan and sum(len(ks) for ks, _ in plan) == 4
    assert plan_launches([5, 5], [10, 10], 1) == [([0], 10), ([1], 10)]
    assert plan_launches([1, 2, 3], [10, 11, 12], 6) == [([0, 1, 2], 12)]


def test_keys_keep_requests_apart():
    sizes, nodes = [4, 4, 4, 4, 4], [30, 31, 30, 31, 32]
    plan = plan_launches(sizes, nodes, 256, keys=nodes)                  # the mean-FC rule: equal N only
    assert sorted(plan) == [([0, 2], 30), ([1, 3], 31), ([4], 32)]
    for ks, n in plan:
        assert {nodes[k] for k in ks} == {n}
    plan = plan_launches(sizes, nodes, 256, keys=['a', 'b', 'a', 'a', 'b'])
    assert plan == [([0, 2, 3], 31), ([1, 4], 32)]                     # groups in the order of their first request
    with pytest.raises(ValueError):
        plan_launches([1], [1], 0)
    with pytest.raises(ValueError):
        plan_launches([1, 2], [1], 4)


def test_launches_are_balanced_by_cost():
    assert deal_launches([10, 9, 8, 1, 1, 1], 2) == [0, 1, 1, 0, 0, 0]   # loads 13 and 17
    assert deal_launches([5, 5, 5], 3) == [0, 1, 2]
    assert deal_launches([7], 4) == [0]
    g = torch.Generator().manual_seed(2)
    for _ in range(30):
        costs = torch.randint(1, 1000, (int(torch.randint(1, 30, (1,), generator=g)),), generator=g).tolist()
        slots = int(torch.randint(1, 5, (1,), generator=g))
        out = deal_launches(costs, slots)
        load = [sum(c for c, s in zip(costs, out) if s == i) for i in range(slots)]
        assert max(load) - min(load) <= max(costs)                     # the greedy longest-first bound


# ---- CPU: refusals and packing ---------------------------------------------------------------------------------------------

def _cpu_model(inpainting=False):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    over = {"inpainting": True} if inpainting else {}
    ddpm, _ = helpers.build_ddpm(spec, 0, **over)
    ddpm.edm.T = 4
    return ddpm, sampler_inputs(ddpm, collate(synthetic.make_items(spec, batch=3)))


@pytest.mark.parametrize("inpainting", [False, True])
def test_sample_many_refuses_what_it_cannot_pack(inpainting):
    ddpm, kw = _cpu_model(inpainting)
    edm = ddpm.edm
    reqs = [kw, kw]
    seeds = [[1, 2, 3], [4, 5, 6]]
    with pytest.raises(ValueError, match="at least one request"):
        edm.sample_many([], seeds=[])
    with pytest.raises(ValueError, match="per-molecule streams"):        # the batch stream
        edm.sample_many(reqs)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_many([kw, dict(kw, noise=torch.zeros(1))], seeds=seeds)
    with pytest.raises(ValueError, match="exactly the inputs"):
        edm.sample_many([{k: v for k, v in kw.items() if k != 'context'}], seeds=seeds[:1])
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="replaced"):
        edm.sample_many(reqs, seeds=seeds)
    delattr(edm, name)
    with pytest.raises(ValueError, match="2 lists for 1 requests"):
        edm.sample_many([kw], seeds=seeds)
    with pytest.raises(ValueError, match="request 1: seeds holds 2 values"):
        edm.sample_many(reqs, seeds=[[1, 2, 3], [4, 5]])
    with pytest.raises(ValueError, match="different devices"):
        edm.sample_many([kw, {k: (None if v is None else v.to('meta')) for k, v in kw.items()}], seeds=seeds)
    with pytest.raises(ValueError, match="atom features"):
        edm.sample_many([kw, dict(kw, h=kw['h'][..., :-1])], seeds=seeds)
    with pytest.raises(ValueError, match="context"):
        edm.sample_many([kw, dict(kw, context=torch.cat([kw['context'], kw['context']], dim=-1))], seeds=seeds)
    with pytest.raises(ValueError, match="CUDA inputs"):                 # host inputs
        edm.sample_many(reqs, seeds=seeds)
    edm.noise_mode = 'per_molecule'
    with pytest.raises(ValueError, match="CUDA inputs"):
        edm.sample_many(reqs)
    assert edm.last_seeds_many is None


def _requests(kw, rows, extras):
    """Requests made of rows of the sampler inputs `kw`: request k holds rows[k], padded with extras[k] dead atoms."""
    B = kw['x'].shape[0]
    out = []
    for idx, extra in zip(rows, extras):
        r = {}
        for name, v in kw.items():
            if v is None:
                r[name] = None
            elif name == 'edge_mask':
                N = kw['x'].shape[1]
                if v.shape[0] == B * N * N:                                 # FC: (B N N, 1)
                    m = v.reshape(B, N, N, -1)[idx]
                    r[name] = torch.nn.functional.pad(m, (0, 0, 0, extra, 0, extra)).reshape(-1, v.shape[-1])
                else:                                                       # cut-off graphs: per-node batch ids
                    r[name] = torch.arange(len(idx), device=v.device).repeat_interleave(N + extra).to(v.dtype)
            else:
                r[name] = torch.cat([v[idx], v.new_zeros((len(idx), extra) + tuple(v.shape[2:]))], dim=1)
        out.append(r)
    return out


PACK_CASES = {"fc": (synthetic.SPECS["cfg2_zinc_ragged"], {}), "inpainting": (synthetic.SPECS["cfg2_zinc_ragged"], {"inpainting": True}),
              "pocket_4A": (helpers.EXTRA_SPECS["small_pocket_4A"], {})}


@pytest.mark.parametrize("case", sorted(PACK_CASES))
def test_packing_round_trip_returns_each_request_unchanged(case):
    """A stub for the single-launch path returns its inputs as the chain: unpacking it gives back every request's tensors,
    and the packed launch holds each request's rows, masks and edge-mask blocks, with zeros in the padding."""
    spec, over = PACK_CASES[case]
    ddpm, _ = helpers.build_ddpm(spec, 0, **over)
    kw = sampler_inputs(ddpm, collate(synthetic.make_items(spec, batch=4)))
    fc = ddpm.edm.dynamics.graph_type == 'FC'
    reqs = _requests(kw, [[0], [1, 2, 3], [3, 0]], [5, 0, 2])
    sizes = [r['x'].shape[0] for r in reqs]
    nodes = [r['x'].shape[1] for r in reqs]
    plan = plan_launches(sizes, nodes, 4)
    assert len(plan) == 2
    got = [None] * len(reqs)
    for ks, n in plan:
        packed = pack_requests([reqs[k] for k in ks], n, fc)
        B = sum(sizes[k] for k in ks)
        assert packed['x'].shape[:2] == (B, n)
        if fc:
            em = packed['edge_mask'].reshape(B, n, n)
        else:
            assert torch.equal(packed['edge_mask'], torch.arange(B).repeat_interleave(n).to(packed['edge_mask'].dtype))
        lo = 0
        for k in ks:
            b, nk = sizes[k], nodes[k]
            if fc:
                assert torch.equal(em[lo:lo + b, :nk, :nk], reqs[k]['edge_mask'].reshape(b, nk, nk))
                assert not em[lo:lo + b, nk:].any() and not em[lo:lo + b, :, nk:].any()
            for name in ('x', 'h', 'node_mask', 'fragment_mask', 'linker_mask', 'context'):
                assert torch.equal(packed[name][lo:lo + b, :nk], reqs[k][name]), (name, k)
                assert not packed[name][lo:lo + b, nk:].any(), (name, k)
            lo += b
        # the stub: three frames of the packed inputs side by side
        cols = torch.cat([packed[name].float() for name in ('x', 'h', 'node_mask', 'fragment_mask', 'linker_mask', 'context')], -1)
        chain = cols.unsqueeze(0).expand(3, *cols.shape).contiguous()
        for k, part in zip(ks, unpack_rows(chain, [sizes[k] for k in ks], [nodes[k] for k in ks], dim=1)):
            got[k] = part
    for k, r in enumerate(reqs):
        want = torch.cat([r[name].float() for name in ('x', 'h', 'node_mask', 'fragment_mask', 'linker_mask', 'context')], -1)
        assert got[k].is_contiguous() and torch.equal(got[k], want.unsqueeze(0).expand(3, *want.shape))


# ---- GPU ------------------------------------------------------------------------------------------------------------------

CASES = ["default", "inpainting", "pocket_4A", "pocket_FC-10A-4A", "tanh", "mean", "sin"]
IMPLS = ["simt", "auto"]


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


def build(case, impl):
    """(ddpm on cuda:0 with T = 10, the sampler inputs of a batch, the rows requests may use). The pocket_FC-10A-4A batch
    keeps its first four molecules, as in test_per_molecule_seeds.py."""
    d = dev()
    rows, over = 5, {}
    if case == "default":
        spec = synthetic.SPECS["cfg2_zinc_ragged"]
    elif case == "inpainting":
        spec, over = synthetic.SPECS["cfg2_zinc_ragged"], {"inpainting": True}
    elif case.startswith("pocket"):
        spec = helpers.EXTRA_SPECS[f"small_{case}"]
        rows = 4
    else:
        spec = eo.spec_with_options("opts_cfg1", case == "tanh", case == "mean", case == "sin")
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=rows)).items()}
    return ddpm, sampler_inputs(ddpm, data), rows


def five_requests(kw, rows):
    """Five requests of different (B_k, N_k): B_k = 1, 3, 6, 2 and 1, padded with 0, 4, 2, 7 and 0 dead atoms."""
    sizes, extras = [1, 3, 6, 2, 1], [0, 4, 2, 7, 0]
    idx, i = [], 0
    for b in sizes:
        idx.append([(i + j) % rows for j in range(b)])
        i += b
    return _requests(kw, idx, extras)


SEEDS = [[11], [-3, 1 << 63, 20240607], [5, 6, 7, 8, 9, 10], [101, 102], [-77]]


def sequential(edm, reqs, seeds, **kw):
    return [edm.sample_chain(**r, keep_frames=3, seeds=s, **kw) for r, s in zip(reqs, seeds)]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", CASES)
def test_each_result_is_its_own_sample_chain_call(case, impl):
    ddpm, kw, rows = build(case, impl)
    edm = ddpm.edm
    reqs = five_requests(kw, rows)
    want = sequential(edm, reqs, SEEDS)
    got = edm.sample_many(reqs, keep_frames=3, seeds=SEEDS, max_molecules=4)          # the request of 6 goes alone
    assert len(got) == len(reqs)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.device == w.device and g.is_contiguous(), k
        assert torch.equal(g, w), (case, impl, k)
        assert torch.equal(edm.last_seeds_many[k], seeds_tensor(SEEDS[k], len(SEEDS[k])))
    assert edm.last_attempts_many == [None] * 5 and edm.last_connected_many == [None] * 5
    launches = edm.last_loop_ms_many
    assert sorted(k for _, ks, _ in launches for k in ks) == list(range(5))
    assert [2] in [ks for _, ks, _ in launches] and all(ms > 0 and d == 0 for d, _, ms in launches)
    if case == "mean":                                                  # the reference's mean divides by the padded N
        for _, ks, _ in launches:
            assert len({reqs[k]['x'].shape[1] for k in ks}) == 1, ks


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", CASES)
def test_per_molecule_mode_matches_the_sequence_of_calls(case, impl):
    ddpm, kw, rows = build(case, impl)
    edm = ddpm.edm
    edm.noise_mode = 'per_molecule'
    reqs = five_requests(kw, rows)
    gen = torch.cuda.default_generators[0]
    torch.manual_seed(9)
    want, want_seeds = [], []
    for r in reqs:
        want.append(edm.sample_chain(**r, keep_frames=3))
        want_seeds.append(edm.last_seeds)
    off = gen.get_offset()
    torch.manual_seed(9)
    got = edm.sample_many(reqs, keep_frames=3)
    assert gen.get_offset() == off
    for k in range(len(reqs)):
        assert torch.equal(got[k], want[k]) and torch.equal(edm.last_seeds_many[k], want_seeds[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", CASES)
def test_launch_sizes_and_request_order_change_nothing(case, impl):
    ddpm, kw, rows = build(case, impl)
    edm = ddpm.edm
    reqs = five_requests(kw, rows)
    want = sequential(edm, reqs, SEEDS)
    counts = []
    for m in (1, 2, 256):
        got = edm.sample_many(reqs, keep_frames=3, seeds=SEEDS, max_molecules=m)
        counts.append(len(edm.last_loop_ms_many))
        assert all(torch.equal(g, w) for g, w in zip(got, want)), m
    assert counts[0] == 5 and counts[0] >= counts[1] >= counts[2]
    if case != "mean":
        assert counts[2] == 1                                           # all in one launch
    perm = [3, 0, 4, 2, 1]
    got = edm.sample_many([reqs[k] for k in perm], keep_frames=3, seeds=[SEEDS[k] for k in perm])
    assert all(torch.equal(g, want[k]) for g, k in zip(got, perm))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_a_mean_fc_model_with_mixed_n_still_matches(impl):
    ddpm, kw, rows = build("mean", impl)
    edm = ddpm.edm
    reqs = _requests(kw, [[0, 1], [2], [3, 4], [1], [0]], [0, 3, 0, 3, 6])
    seeds = [[1, 2], [3], [4, 5], [6], [7]]
    want = sequential(edm, reqs, seeds)
    got = edm.sample_many(reqs, keep_frames=3, seeds=seeds)
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    assert sorted(ks for _, ks, _ in edm.last_loop_ms_many) == [[0, 2], [1, 3], [4]]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
@pytest.mark.parametrize("case", ["default", "inpainting", "pocket_4A"])
def test_launches_dealt_to_devices_reproduce_the_single_device_results(case, impl):
    ddpm, kw, rows = build(case, impl)
    edm = ddpm.edm
    reqs = five_requests(kw, rows)
    want = edm.sample_many(reqs, keep_frames=3, seeds=SEEDS, max_molecules=4)
    edm.devices = [0, 0, 0]
    try:
        got = edm.sample_many(reqs, keep_frames=3, seeds=SEEDS, max_molecules=4)
    finally:
        edm.devices = None
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    assert len(edm.last_loop_ms_many) >= 3


# NaN recovery: the weights of test_nan_recovery.py, on which some draws diverge at T = 10
COORD_GAIN = 5.0
GAIN_SEEDS = [[1, 2, 3], [4], [5, 6, 7, 8]]


def gain_model(impl):
    d = dev()
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(COORD_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=8)).items()}
    kw = sampler_inputs(ddpm, data)
    return ddpm, _requests(kw, [[0, 1, 2], [3], [4, 5, 6, 7]], [0, 2, 5])


def close(got, want):
    """The suite's fp32 tolerance: 1e-4 of the values' scale (at least 1)."""
    return bool((got - want).abs().max() <= 1e-4 * want.abs().max().clamp(min=1.0))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_recovery_rounds_match_the_per_request_calls(impl):
    ddpm, reqs = gain_model(impl)
    edm = ddpm.edm
    want, attempts, used = [], [], []
    for r, s in zip(reqs, GAIN_SEEDS):
        want.append(edm.sample_chain(**r, keep_frames=3, seeds=s, nan_retries=4))
        attempts.append(edm.last_attempts)
        used.append(edm.last_seeds)
    assert any(a.any() for a in attempts)                               # some rows were resampled
    got = edm.sample_many(reqs, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=4)
    for k in range(len(reqs)):
        assert torch.equal(edm.last_attempts_many[k], attempts[k]) and torch.equal(edm.last_seeds_many[k], used[k]), k
        healthy = (attempts[k] == 0).nonzero().flatten().tolist()
        assert torch.equal(got[k][:, healthy], want[k][:, healthy]), k
        assert torch.equal(got[k], want[k]) if impl == "simt" else close(got[k], want[k]), k


@pytest.mark.gpu
def test_rows_that_always_fail_name_their_request():
    ddpm, reqs = gain_model("simt")
    edm = ddpm.edm
    reqs[2] = dict(reqs[2], x=reqs[2]['x'].clone())
    reqs[2]['x'][1, 0, 0] = float('nan')                                # a fragment coordinate: every attempt fails
    with pytest.raises(FoundNaNException) as info:
        edm.sample_chain(**reqs[2], keep_frames=3, seeds=GAIN_SEEDS[2], nan_retries=2)
    alone, alone_attempts = info.value, edm.last_attempts
    with pytest.raises(FoundNaNException) as info:
        edm.sample_many(reqs, keep_frames=3, seeds=GAIN_SEEDS, nan_retries=2)
    exc = info.value
    failed = lambda e: sorted(e.x_h_nan_idx | e.only_x_nan_idx | e.only_h_nan_idx)
    assert exc.request == 2 and failed(exc) == failed(alone) == [1]
    assert len(exc.results) == 3 and exc.chain is exc.results[2]
    # the failing row holds its last round's draw, NaNs included
    assert torch.allclose(exc.results[2], alone.chain, rtol=0, atol=0, equal_nan=True)
    assert torch.equal(edm.last_attempts_many[2], alone_attempts) and alone_attempts[1] == 2
    for k in (0, 1):
        assert torch.equal(exc.results[k], edm.sample_chain(**reqs[k], keep_frames=3, seeds=GAIN_SEEDS[k], nan_retries=2))


@pytest.mark.gpu
@pytest.mark.parametrize("impl", IMPLS)
def test_connectivity_rounds_match_the_per_request_calls(impl):
    import test_connected_resampling as tc
    ddpm, kw = tc.build("fc", impl)
    edm = ddpm.edm
    reqs = _requests(kw, [[0, 1, 2], [3, 4], [5, 6, 7]], [0, 0, 0])
    seeds = [tc.SEEDS[0:3], tc.SEEDS[3:5], tc.SEEDS[5:8]]
    want, conn, attempts = [], [], []
    for r, s in zip(reqs, seeds):
        want.append(edm.sample_chain(**r, keep_frames=2, seeds=s, nan_retries=tc.ROUNDS, require_connected=True))
        conn.append(edm.last_connected)
        attempts.append(edm.last_attempts)
    got = edm.sample_many(reqs, keep_frames=2, seeds=seeds, nan_retries=tc.ROUNDS, require_connected=True)
    for k in range(len(reqs)):
        assert torch.equal(edm.last_connected_many[k], conn[k]) and torch.equal(edm.last_attempts_many[k], attempts[k]), k
        assert torch.equal(got[k], want[k]) if impl == "simt" else close(got[k], want[k]), k
    assert any(a.any() for a in attempts)                               # some rows were resampled to connect them


@pytest.mark.gpu
def test_ddpm_sample_many_calls_sample_fn_as_the_sequential_calls_do():
    d = dev()
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    ddpm.edm.noise_mode = 'per_molecule'
    datas = []
    for b, off in ((3, 0), (1, 1), (4, 2)):
        datas.append({k: (v.to(d) if torch.is_tensor(v) else v)
                      for k, v in collate(synthetic.make_items(spec, batch=b, seed_offset=off)).items()})

    def sample_fn(data):                                                # draws from the CUDA generator, as a size model does
        n = data['fragment_mask'].shape[0]
        return torch.randint(2, 6, (n,), device=d)
    gen = torch.cuda.default_generators[0]
    torch.manual_seed(4)
    want = [ddpm.sample_chain(data, sample_fn=sample_fn, keep_frames=2) for data in datas]
    off = gen.get_offset()
    torch.manual_seed(4)
    got = ddpm.sample_many(datas, sample_fn=sample_fn, keep_frames=2)
    assert gen.get_offset() == off
    for (c, nm), (wc, wnm) in zip(got, want):
        assert torch.equal(nm, wnm) and torch.equal(c, wc)
