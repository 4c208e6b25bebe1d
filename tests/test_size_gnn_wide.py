"""The linker-size classifier at hidden_nf = 256, the width of the reference README's size-model recipe
(`train_size_gnn.py --hidden_nf 256 --n_layers 5 --normalization batch_norm`): dl_sizegnn_forward's 256-wide kernels
(k_szw_prep -> [k_szw_edge -> k_szw_node] x L -> k_szw_out), up to SizeClassifier and the sampler's size draws.

CPU: the oracle against the reference fixtures (tools/make_golden_size_wide.py), the reference's parameter layout and
seeded construction, Lightning checkpoints, and the refusal of every other width.
GPU: the logits against the fixtures; against the fp64 oracle molecule by molecule with the batches, the error bound and
the draw-exclusion rule of test_size_gnn_fp64 (its builders are imported through the module, so none of its tests is
collected twice); the sampler end to end, first draw and recovery-round redraws.
"""
import contextlib
import ctypes as C
import functools

import numpy as np
import pytest
import torch

import dl_helpers as helpers
import test_size_gnn_fp64 as base
from difflinker_b200 import _native, synthetic
from difflinker_b200.linker_size import (GEOM_TRAIN_LINKER_ID2SIZE, GEOM_TRAIN_LINKER_SIZE2ID, SizeClassifier,
                                         draw_sizes)
from fp64_rows import C_DRIFT, TAU, dev
from oracle import difflinker_oracle as orc

WIDTH = 256
FIXTURES = ["size_gnn_zinc_h256", "size_gnn_pocket_geom_h256", "size_gnn_geom_h256"]


def build_wide_classifier(meta):
    """helpers.build_size_classifier at the fixture's width: same seed and construction order as the reference."""
    spec = helpers.spec_by_name(meta["spec"])
    kw = helpers.size_forward_kw(meta)
    tables = dict(linker_size2id=GEOM_TRAIN_LINKER_SIZE2ID, linker_id2size=GEOM_TRAIN_LINKER_ID2SIZE) \
        if meta["out_nf"] == len(GEOM_TRAIN_LINKER_ID2SIZE) else {}
    torch.manual_seed(meta["seed"])
    model = SizeClassifier(in_node_nf=kw["in_node_nf"], hidden_nf=meta["hidden_nf"], out_node_nf=meta["out_nf"],
                           n_layers=kw["n_layers"], normalization=meta["normalization"], **tables)
    synthetic.init_size_gnn_like_trained(model, meta["seed"])
    model.eval()
    from difflinker_b200.linker_size import collate_with_fragment_edges
    data = collate_with_fragment_edges(synthetic.size_gnn_items(spec, meta["batch"]))
    return model, data


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_the_wide_reference_fixtures(name):
    meta, a = helpers.load_golden(name)
    assert meta["hidden_nf"] == WIDTH
    model, data = build_wide_classifier(meta)
    assert helpers.state_sha(model.state_dict()) == meta["sha"]
    with torch.no_grad():
        out = orc.size_classifier_forward(model.state_dict(), data, **helpers.size_forward_kw(meta))
    assert out.shape == a["logits"].shape
    assert (out - a["logits"]).abs().max().item() <= 2e-6 * max(1.0, a["logits"].abs().max().item())


def test_the_fixtures_cover_the_recipe_a_pocket_model_and_no_normalization():
    metas = [helpers.load_golden(n)[0] for n in FIXTURES]
    assert any(m["n_layers"] == 5 and m["normalization"] == "batch_norm" and m["out_nf"] == 10 for m in metas)
    assert any(m["with_pocket"] and m["adjust_shape"] for m in metas)
    assert any(m["normalization"] is None for m in metas)


def test_parameter_layout_is_the_reference_s_and_the_seeded_sha_matches_it():
    """Keys and shapes of SizeClassifier(hidden_nf=256, n_layers=5, batch_norm), and the reference's sha from the seed."""
    torch.manual_seed(0)
    m = SizeClassifier(in_node_nf=8, hidden_nf=WIDTH, out_node_nf=10, n_layers=5, normalization='batch_norm')
    sd = m.state_dict()
    want = {"gnn.embedding_in.weight": (WIDTH, 8), "gnn.embedding_in.bias": (WIDTH,),
            "gnn.embedding_out.weight": (10, WIDTH), "gnn.embedding_out.bias": (10,)}
    for p in ["gnn.gcl1"] + [f"gnn.gcl_layers.{l}" for l in range(4)]:
        want.update({f"{p}.edge_mlp.0.weight": (WIDTH, 2 * WIDTH + 1), f"{p}.edge_mlp.0.bias": (WIDTH,),
                     f"{p}.edge_mlp.2.weight": (WIDTH, WIDTH), f"{p}.edge_mlp.2.bias": (WIDTH,),
                     f"{p}.node_mlp.0.weight": (WIDTH, 2 * WIDTH), f"{p}.node_mlp.0.bias": (WIDTH,),
                     f"{p}.node_mlp.3.weight": (WIDTH, WIDTH), f"{p}.node_mlp.3.bias": (WIDTH,)})
        for bn in ("node_mlp.1", "node_mlp.4"):
            want.update({f"{p}.{bn}.{k}": (WIDTH,) for k in ("weight", "bias", "running_mean", "running_var")})
            want[f"{p}.{bn}.num_batches_tracked"] = ()
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    assert [k for k in sd if k.startswith("gnn.gcl1.")][0] == "gnn.gcl1.edge_mlp.0.weight"
    meta, _ = helpers.load_golden("size_gnn_zinc_h256")
    model, _ = build_wide_classifier(meta)
    assert helpers.state_sha(model.state_dict()) == meta["sha"]


def test_load_from_checkpoint_builds_the_256_wide_model(tmp_path):
    sc = SizeClassifier(in_node_nf=8, hidden_nf=WIDTH, out_node_nf=10, n_layers=5, normalization='batch_norm')
    synthetic.init_size_gnn_like_trained(sc, 1)
    path = str(tmp_path / "zinc_size_gnn.ckpt")
    hp = dict(sc.hparams, task='classification')
    torch.save({"epoch": 1, "hyper_parameters": hp, "state_dict": sc.state_dict()}, path)
    sc2 = SizeClassifier.load_from_checkpoint(path, map_location="cpu")
    assert sc2.gnn.hidden_nf == WIDTH and sc2.gnn.n_layers == 5 and sc2.gnn.normalization == 'batch_norm'
    assert list(sc2.state_dict()) == list(sc.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(sc.state_dict().values(), sc2.state_dict().values()))


@pytest.mark.parametrize("width", [64, 192])
def test_other_widths_are_refused_in_python_and_by_dl_sizegnn_create(width):
    with pytest.raises(NotImplementedError, match="128.*256"):
        SizeClassifier(in_node_nf=8, hidden_nf=width, out_node_nf=10, n_layers=3)
    lib = _native.load_library()
    cfg = _native.DLSizeGNNConfig(in_node_nf=8, hidden_nf=width, out_node_nf=10, n_layers=3, device=0)
    handle = C.c_void_p()
    with pytest.raises(_native.NativeError, match=f"hidden_nf must be 128 or 256 \\(got {width}\\)"):
        _native.check(lib.dl_sizegnn_create(C.byref(cfg), C.byref(handle)), "dl_sizegnn_create")
    assert not handle.value


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", FIXTURES)
def test_logits_match_the_wide_reference_fixtures(name):
    meta, a = helpers.load_golden(name)
    model, data = build_wide_classifier(meta)
    d = dev()
    dd = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in data.items()}
    kw = helpers.size_forward_kw(meta)
    out = model.to(d).size_logits(dd, with_pocket=kw["with_pocket"], adjust_shape=kw["adjust_shape"]).cpu()
    assert out.shape == a["logits"].shape
    err = (out - a["logits"]).abs().max().item() / a["logits"].abs().max().item()
    assert err <= 1e-5, err


MODELS = {   # name: (in_node_nf, out_node_nf, n_layers, normalization), all 256 wide
    "zinc_recipe": (8, 10, 5, "batch_norm"), "zinc": (8, 10, 3, None), "geom_bn": (9, 33, 3, "batch_norm"),
    "zinc_L1": (8, 10, 1, None), "out64": (8, 64, 3, None), "in32": (32, 10, 2, "batch_norm"),
    "bn_small_var": (8, 10, 3, "batch_norm"),
}
CASES = {    # case: (test_size_gnn_fp64 batch, model, pocket)
    "fc_zinc_recipe": ("fc8", "zinc_recipe", False), "fc_zinc": ("fc8", "zinc", False),
    "fc_geom_bn": ("fc9", "geom_bn", False), "fc_L1": ("fc8", "zinc_L1", False), "fc_out64": ("fc8", "out64", False),
    "fc_in32": ("fc32", "in32", False), "fc_bn_small_var": ("fc8", "bn_small_var", False),
    "tail1": ("tail1", "zinc", False), "tail31": ("tail31", "zinc_recipe", False),
    "pocket_cfg4": ("pocket_cfg4", "geom_bn", True), "pocket_protein": ("pocket_protein", "geom_bn", True),
    "pocket_6144": ("pocket_6144", "geom_bn", True), "rounding": ("rounding", "zinc", False),
}


@functools.lru_cache(maxsize=None)
def model(name):
    F, Cc, L, norm = MODELS[name]
    if Cc == len(GEOM_TRAIN_LINKER_ID2SIZE):
        tables = dict(linker_id2size=GEOM_TRAIN_LINKER_ID2SIZE, linker_size2id=GEOM_TRAIN_LINKER_SIZE2ID)
    else:
        table = list(range(1, Cc + 1))
        tables = dict(linker_id2size=table, linker_size2id={s: i for i, s in enumerate(table)})
    torch.manual_seed(200 + len(name))
    m = SizeClassifier(in_node_nf=F, hidden_nf=WIDTH, out_node_nf=Cc, n_layers=L, normalization=norm, **tables)
    synthetic.init_size_gnn_like_trained(m, 9)
    if name == "bn_small_var":
        g = torch.Generator().manual_seed(8)
        with torch.no_grad():
            for k, b in m.named_buffers():
                if k.endswith("running_var"):
                    b.copy_(10.0 ** (-3.0 * torch.rand(b.shape, generator=g)))          # 1e-3 .. 1
    return m.eval()


@contextlib.contextmanager
def half_edge_blocks():
    """The oracle's edge blocks at half their default size: at 256 wide, fp64 blocks of 2^20 pocket-clique edges would
    hold several 2^20 x 513 activations at once at N = 6144."""
    full = orc.size_live_edges
    orc.size_live_edges = functools.partial(full, max_pairs=1 << 19)
    try:
        yield
    finally:
        orc.size_live_edges = full


def oracle_logits(m, data, pocket, dtype, device):
    with half_edge_blocks():
        return base.oracle_logits(m, data, pocket, dtype, device)


def test_half_edge_blocks_keep_the_oracle_s_edge_list():
    data, _ = base.batch("fc8")
    B, N = data['positions'].shape[:2]
    x = data['positions'].reshape(B * N, 3) * data['fragment_mask'].reshape(B * N, 1)
    em = data['edge_mask'].reshape(-1)
    whole = [torch.cat(t) for t in zip(*orc.size_live_edges(x, em, B, N))]
    with half_edge_blocks():
        halves = [torch.cat(t) for t in zip(*orc.size_live_edges(x, em, B, N))]
    assert all(torch.equal(a, b) for a, b in zip(whole, halves))
    assert orc.size_live_edges.__name__ == "size_live_edges"


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    rows = {k: v for k, v in base.WORST.items() if k in CASES}
    if rows:
        print("\n256 wide: worst per-molecule ratios (err / bound, err / S_b, molecules within TAU * S_b, excluded draws, "
              "max S_b):")
        for k, (w, r, f, x, sm) in rows.items():
            print(f"  {k:20s} {w:9.3e} {r:9.3e} {f:>7s}  {str(x):>11s}  {sm:9.3e}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_logits_match_fp64_per_molecule_and_draw_the_oracle_size(case):
    from test_seeded_linker_sizes import M64, oracle_sizes, oracle_uniform
    bname, mname, pocket = CASES[case]
    data, m = base.batch(bname)[0], model(mname)
    ref64 = oracle_logits(m, data, pocket, torch.float64, dev())
    ref32 = oracle_logits(m, data, pocket, torch.float32, dev())
    got = base.gpu_logits(m, data, pocket)
    # as in test_size_gnn_fp64: the one- and two-molecule whole-protein shapes are held to the drift bound alone
    bound = base.check_molecules(case, got, ref64, ref32, half_within_tau=base.B_OF[bname] > 2)
    B = got.shape[0]
    K = -(-base.MIN_PAIRS // B)
    seeds = [int(s) for s in np.random.default_rng(len(case) + 1000).integers(0, 1 << 62, B * K, dtype=np.int64)]
    rows = torch.arange(B).repeat_interleave(K)
    table = list(m.linker_id2size)
    drawn = draw_sizes(got.float()[rows].to(dev()), table, seeds).cpu().tolist()
    ref = ref64.float()[rows].numpy()
    want = oracle_sizes(ref, table, seeds)
    u = np.array([oracle_uniform(s & M64) for s in seeds])
    near = base.draw_bounds(ref, base.draw_width(bound, ref64)[rows.numpy()], u)
    bad = [(int(rows[k]), seeds[k]) for k in range(B * K) if drawn[k] != want[k] and not near[k]]
    base.WORST[case][3] = f"{int(near.sum())}/{B * K}"
    assert B * K >= 10_000
    assert not bad, f"{case}: draws differ outside the exclusion band: {bad[:5]}"
    assert near.sum() <= 0.01 * B * K, f"{case}: {int(near.sum())} of {B * K} draws excluded"


@pytest.mark.gpu
def test_n_above_the_plan_limit_is_refused_by_name_at_256():
    m = model("zinc").to(dev())
    N = base.PLAN_MAX_N + 1
    d = dev()
    with pytest.raises(_native.NativeError, match=f"N = {N} exceeds the work plan's limit of {base.PLAN_MAX_N}"):
        m.gnn.logits(torch.zeros((1, N, 8), device=d), torch.zeros((1, N, 3), device=d), torch.ones((1, N), device=d), None)


def wide_size_model(F, table, n_layers, seed):
    torch.manual_seed(seed)
    nn = SizeClassifier(in_node_nf=F, hidden_nf=WIDTH, out_node_nf=len(table), n_layers=n_layers,
                        normalization='batch_norm', linker_id2size=list(table),
                        linker_size2id={s: i for i, s in enumerate(table)})
    synthetic.init_size_gnn_like_trained(nn, seed)
    return nn.eval().to(dev())


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fc", "pocket_4A"])
def test_sample_chain_draws_the_oracle_size_and_samples_its_template(case):
    """DDPM.sample_chain(linker_sizes=<256-wide SizeClassifier>, seeds=...): last_sizes is draw_sizes of the oracle's logits
    of the input batch (with_pocket / adjust_shape on the pocket model), and the chain is the seeded path on the template of
    those sizes. ZINC: the README recipe (5 layers, batch norm); pocket: 3 layers, batch norm."""
    from difflinker_b200 import ddpm as ddpm_mod
    from test_seeded_linker_sizes import M64, SEEDS, model_and_data, oracle_sizes, oracle_uniform
    ddpm, data = model_and_data(case, "simt")
    pocket = case.startswith("pocket")
    F = data['one_hot'].shape[-1]
    table = [0, 1, 2, 3, 4, 6]
    nn = wide_size_model(F - 1 if pocket else F, table, 3 if pocket else 5, 21)
    with torch.no_grad():                                      # centre the logits over the batch, so the draw is the molecule's
        nn.gnn.embedding_out.bias.sub_(oracle_logits(nn, data, pocket, torch.float64, dev()).mean(0).float().to(dev()))
    chain, nm = ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, keep_frames=2)
    got = ddpm.edm.last_sizes.tolist()
    ref64 = oracle_logits(nn, data, pocket, torch.float64, dev())
    ref32 = oracle_logits(nn, data, pocket, torch.float32, dev())
    eps = torch.maximum(C_DRIFT * (ref32 - ref64).abs().amax(1), TAU * ref64.abs().amax(1))
    want = oracle_sizes(ref64.float().numpy(), table, SEEDS)
    u = np.array([oracle_uniform(s & M64) for s in SEEDS])
    near = base.draw_bounds(ref64.float().numpy(), base.draw_width(eps, ref64), u)
    assert not near.any() and len(set(want)) > 1, (want, near)
    assert got == want
    # the GPU's own logits draw the same sizes through draw_sizes
    own = nn.size_logits(data, with_pocket=pocket, adjust_shape=pocket)
    assert draw_sizes(own, table, SEEDS).tolist() == want
    # the chain is the existing seeded path on the template of those sizes, padded to the capacity linker_sizes uses
    B = len(SEEDS)
    n_cap = int(data['fragment_mask'].reshape(B, -1).sum(1).max()) + max(table)
    kw, _ = ddpm_mod._template_inputs(ddpm, data, torch.tensor(want, device=dev()), n_nodes=n_cap)
    assert torch.equal(kw['node_mask'], nm)
    assert torch.equal(chain, ddpm.edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS))


@pytest.mark.gpu
def test_recovery_rounds_redraw_sizes_from_the_retry_seed_of_the_same_logits():
    """nan_retries + require_connected with a 256-wide size model: every row's size is dl_size_draw of its molecule's logits
    with dl_retry_seed(seed, attempt), the rows that were resampled included."""
    from difflinker_b200.edm import retry_seed
    from test_seeded_linker_sizes import ROUNDS, SEEDS, model_and_data
    ddpm, data = model_and_data("fc", "simt")
    edm = ddpm.edm
    table = [0, 1, 2]
    nn = wide_size_model(data['one_hot'].shape[-1], table, 5, 22)
    with torch.no_grad():                                      # logits = [-1, 0.5, 0.2] for every molecule, at any width
        nn.gnn.embedding_out.weight.zero_()
        nn.gnn.embedding_out.bias.copy_(torch.tensor([-1.0, 0.5, 0.2]))
    chain, nm = ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, keep_frames=2, nan_retries=ROUNDS,
                                  require_connected=True)
    assert torch.isfinite(chain).all()
    logits = nn.size_logits(data)
    attempts, used, sizes = edm.last_attempts.tolist(), edm.last_seeds, edm.last_sizes.tolist()
    assert any(a > 0 for a in attempts), attempts                       # some row was resampled and its size redrawn
    for b, s in enumerate(SEEDS):
        assert int(used[b]) == retry_seed(s, attempts[b])
        assert sizes[b] == int(draw_sizes(logits[b:b + 1], table, [s], attempt=attempts[b])[0]), b
