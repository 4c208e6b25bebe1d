"""Linker sizes drawn from each molecule's seed: dl_size_uniform, dl_size_draw and dl_sample_chain_retry, up to
`ddpm.sample_chain(data, linker_sizes=...)`.

The oracle restates the draw of the header in numpy: u from a splitmix64 finaliser of seed ^ TAG, then the fp64 inverse CDF
of the softmax, summed in index order. CPU tests pin the restatement to the exported dl_size_uniform, check the refusals and
compile a C99 caller; GPU tests check the kernel against the oracle, the distribution, the first draw against the existing
seeded path on the same template, replay, and the recovery rounds that redraw sizes."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, synthetic
from difflinker_b200 import ddpm as ddpm_mod
from difflinker_b200.batching import collate, create_templates_for_linker_generation
from difflinker_b200.distributed import sample_chain_sharded
from difflinker_b200.edm import LinkerSizes, retry_seed, seeds_tensor
from difflinker_b200.linker_size import SizeClassifier, collate_with_fragment_edges, draw_sizes, size_uniform
import dl_helpers as helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1
TAG = 0x6C696E6B65722D6E


# ---- the oracle ---------------------------------------------------------------------------------------------------------

def oracle_uniform(seed):
    z = (seed & M64) ^ TAG
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    z ^= z >> 31
    return float(np.float64(z >> 11) * np.float64(2.0 ** -53))


def oracle_index(logits, u):
    """(drawn index, whether u * S lies within 1e-12 S of a cumulative boundary) of the header's rule."""
    l = np.asarray(logits, dtype=np.float32).astype(np.float64)
    e = np.exp(l - l.max())
    c = np.cumsum(e)                     # sequential, in index order
    S = c[-1]
    t = u * S
    hit = np.nonzero(t < c)[0]
    i = int(hit[0]) if hit.size else int(np.nonzero(e > 0)[0][-1])
    return i, bool(np.any(np.abs(c - t) <= 1e-12 * S))


def oracle_sizes(logits, table, seeds, attempt=0):
    out = []
    for row, s in zip(np.asarray(logits), seeds):
        u = oracle_uniform(retry_seed(int(s), attempt) & M64)
        out.append(table[oracle_index(row, u)[0]])
    return out


# ---- CPU ----------------------------------------------------------------------------------------------------------------

def test_the_uniform_is_the_restated_splitmix64_finaliser():
    rng = np.random.default_rng(5)
    seeds = [0, 1, 2, M64, 1 << 63, TAG, TAG ^ 1] + [int(v) for v in rng.integers(0, 1 << 63, 200, dtype=np.int64)]
    for s in seeds:
        u = size_uniform(s)
        assert u == oracle_uniform(s), s
        assert 0.0 <= u < 1.0
    assert size_uniform(-1) == size_uniform(M64)             # reduced modulo 2^64, as the seeds are
    assert size_uniform(TAG) == 0.0                          # the finaliser maps 0 to 0: the tag is what it is xored with


def test_a_uniform_range_draws_lo_plus_floor_u_c():
    for lo, hi in ((0, 0), (3, 12), (5, 7), (0, 40)):
        C = hi - lo + 1
        for s in range(300):
            u = oracle_uniform(s)
            assert lo + oracle_index(np.zeros(C), u)[0] == lo + int(np.floor(u * C)), (lo, hi, s)


def _cpu_ddpm(inpainting=False):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, **({"inpainting": True} if inpainting else {}))
    ddpm.edm.T = 4
    return ddpm, collate(synthetic.make_items(spec, batch=3))


def test_every_refusal_names_the_conflicting_argument():
    ddpm, data = _cpu_ddpm()
    seeds = [1, 2, 3]
    with pytest.raises(ValueError, match="sample_fn"):
        ddpm.sample_chain(data, linker_sizes=3, seeds=seeds, sample_fn=lambda d: torch.full((3,), 3))
    with pytest.raises(ValueError, match="start_step"):
        ddpm.sample_chain(data, linker_sizes=3, seeds=seeds, start_step=2)
    with pytest.raises(ValueError, match="CUDA inputs"):
        ddpm.sample_chain(data, linker_sizes=3, seeds=seeds)
    with pytest.raises(ValueError, match="sample_fn"):
        ddpm.sample_many([data], linker_sizes=3, sample_fn=lambda d: torch.full((3,), 3))
    for bad in ("3", (3,), (5, 2), (-1, 2), True, 2.0):
        with pytest.raises(ValueError, match="linker_sizes"):
            ddpm_mod.size_distribution(ddpm, data, bad)
    with pytest.raises(ValueError, match="linker_sizes"):
        sample_chain_sharded(ddpm, data, seeds=seeds, linker_sizes=3)
    ddpm_i, data_i = _cpu_ddpm(inpainting=True)
    with pytest.raises(ValueError, match="inpainting"):
        ddpm_i.sample_chain(data_i, linker_sizes=3, seeds=seeds)
    # EDM level: a LinkerSizes for the template of the sampler inputs
    edm = ddpm.edm
    kw = ddpm_mod.sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    ls = LinkerSizes(torch.zeros(B, 1), [0], torch.zeros(B, dtype=torch.long), torch.zeros(B, 3))
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, linker_sizes=ls, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, linker_sizes=ls, seeds=seeds, batch_slice=(0, B))
    with pytest.raises(ValueError, match="per-molecule streams"):               # the batch stream
        edm.sample_chain(**kw, linker_sizes=ls)
    with pytest.raises(ValueError, match="linker_sizes needs seeds"):
        edm.noise_mode = 'per_molecule'
        edm.sample_chain(**kw, linker_sizes=ls)
    edm.noise_mode = 'reference_stream'
    with pytest.raises(ValueError, match="linker_sizes does not take start_step"):
        edm.sample_chain(**kw, linker_sizes=ls, seeds=seeds, start_step=1)
    with pytest.raises(ValueError, match="linker_sizes needs CUDA inputs"):
        edm.sample_chain(**kw, linker_sizes=ls, seeds=seeds)
    edm.draw_noise = lambda *a, **k: None
    with pytest.raises(ValueError, match="replaced"):
        edm.sample_chain(**kw, linker_sizes=ls, seeds=seeds)
    del edm.draw_noise
    with pytest.raises(ValueError, match="linker_sizes does not take InpaintingEDM"):
        kw_i = ddpm_mod.sampler_inputs(ddpm_i, data_i)
        ddpm_i.edm.sample_chain(**kw_i, linker_sizes=ls, seeds=seeds)
    with pytest.raises(ValueError, match="n_nodes"):
        create_templates_for_linker_generation(data, [3, 3, 3], n_nodes=2)


def test_header_declares_the_draw_and_a_c99_retry_caller_compiles(tmp_path):
    with open(os.path.join(ROOT, "include", "difflinker_b200.h")) as f:
        header = f.read()
    assert "typedef struct dl_size_redraw" in header
    for name in ("dl_size_uniform", "dl_size_draw", "dl_sample_chain_retry"):
        assert f"{name}(" in header and name in _native.SYMBOLS, name
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "sizes_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  int32_t sizes[1] = {3}, used[2];\n"
        "  dl_size_redraw rz = {1, 1, NULL, sizes, NULL, NULL};\n"
        "  dl_status a = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 20, 10, 1, NULL, NULL, NULL, NULL,\n"
        "      NULL, NULL, NULL, NULL, NULL, NULL, NULL, 1, NULL, NULL, NULL, NULL, &rz, used, NULL);\n"
        '  printf("%d|%s\\n", (int)a, dl_last_error());\n'
        "  dl_status b = dl_size_draw(0, 1, NULL, 1, NULL, NULL, 0, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)b, dl_last_error());\n'
        '  printf("%.17g\\n", dl_size_uniform(12345u));\n'
        "  return 0;\n}\n")
    exe = tmp_path / "sizes_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, b, u = res.stdout.strip().split("\n")
    assert a.startswith("-1|") and "null engine" in a
    assert b.startswith("-1|") and "dl_size_draw" in b
    assert float(u) == oracle_uniform(12345)


# ---- GPU: the draw ------------------------------------------------------------------------------------------------------

def dev():
    assert torch.cuda.is_available(), "needs an H100"
    return torch.device("cuda", 0)


@pytest.mark.gpu
def test_the_kernel_draws_the_oracle_index():
    d = dev()
    g = torch.Generator().manual_seed(3)
    near, total = 0, 0
    for B, C, kind in ((4096, 1, "one"), (4096, 10, "randn"), (1000, 40, "randn"), (2048, 33, "large"), (512, 7, "equal"),
                       (3000, 2, "large"), (777, 40, "spiky")):
        if kind == "equal":
            logits = torch.full((B, C), 2.5)
        elif kind == "large":
            logits = 80.0 * torch.randn((B, C), generator=g)
        elif kind == "spiky":
            logits = torch.randn((B, C), generator=g)
            logits[:, 5] = 60.0
            logits[::3, 9] = 60.0                                         # two equal peaks
        else:
            logits = torch.randn((B, C), generator=g)
        seeds = torch.randint(-(1 << 62), 1 << 62, (B,), generator=g)
        for attempt in (0, 3):
            got = draw_sizes(logits.to(d), list(range(C)), seeds, attempt=attempt).cpu().tolist()
            for b in range(B):
                u = oracle_uniform(retry_seed(int(seeds[b]), attempt) & M64)
                want, at_edge = oracle_index(logits[b].numpy(), u)
                near += at_edge
                assert got[b] == want or at_edge, (kind, B, C, attempt, b)
            total += B
    print(f"rows within 1e-12 S of a boundary: {near} of {total}")
    assert near <= total // 10000


@pytest.mark.gpu
def test_the_draws_follow_the_softmax():
    from scipy.stats import chisquare
    d = dev()
    logits = torch.tensor([0.3, -1.0, 2.0, 0.0, 1.1, -0.5, 0.7, -2.0])
    n = 100_000
    got = draw_sizes(logits.expand(n, -1).contiguous().to(d), list(range(8)), list(range(n))).cpu()
    counts = torch.bincount(got.long(), minlength=8).double().numpy()
    p = torch.softmax(logits.double(), 0).numpy()
    stat, pval = chisquare(counts, p * n)
    print(f"chi2 {stat:.2f}, p {pval:.3g}")
    assert pval > 1e-6


# ---- GPU: the sampler ---------------------------------------------------------------------------------------------------

from test_connected_resampling import COORD_GAIN, NF, SEEDS, model_spec, small_fragment_items  # noqa: E402

ROUNDS = 4


def size_model(d, table, bias=None):
    """A SizeClassifier over `table` on the ZINC types; `bias` zeroes embedding_out's weight and sets its bias, so the
    logits are the bias whatever the input."""
    torch.manual_seed(4)
    nn = SizeClassifier(in_node_nf=8, out_node_nf=len(table), linker_id2size=list(table),
                        linker_size2id={s: i for i, s in enumerate(table)})
    if bias is not None:
        with torch.no_grad():
            nn.gnn.embedding_out.weight.zero_()
            nn.gnn.embedding_out.bias.copy_(torch.tensor(bias))
    return nn.eval().to(d)


def model_and_data(case, impl, rows=len(SEEDS)):
    d = dev()
    spec, over = model_spec(case, rows)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(COORD_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    items = small_fragment_items(case, rows)
    data = collate_with_fragment_edges(items) if case.startswith("pocket") else collate(items)
    return ddpm, {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in data.items()}


def rows_of(data, idx):
    """Molecules `idx` of a collated batch, keeping its padding."""
    B = data['positions'].shape[0]
    ix = torch.tensor(idx, device=data['positions'].device)
    out = {}
    for k, v in data.items():
        if k == 'edges':                                                 # collate_with_fragment_edges' edge list
            continue
        if not torch.is_tensor(v):
            out[k] = [v[i] for i in idx]
        elif k == 'edge_mask':
            out[k] = v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:])
        else:
            out[k] = v[ix]
    return out


def pocket_args(case):
    return case.startswith("pocket")


FIRST_CASES = [("fc", "simt"), ("fc", "auto"), ("pocket_4A", "simt"), ("pocket_4A", "auto"), ("pocket_FC-10A-4A", "simt"),
               ("pocket_FC-10A-4A", "auto")]


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", FIRST_CASES)
def test_the_first_draw_is_the_seeded_path_on_its_template(case, impl, monkeypatch):
    if case == "pocket_FC-10A-4A":
        from test_connected_resampling import NOISE_PRECISION
        monkeypatch.setitem(NOISE_PRECISION, case, 0.4)
    ddpm, data = model_and_data(case, impl)
    table = [0, 1, 2, 3, 4, 6]
    nn = size_model(dev(), table)
    B = len(SEEDS)
    chain, nm = ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, keep_frames=2)
    sizes = ddpm.edm.last_sizes
    pocket = pocket_args(case)
    logits = nn.size_logits(data, with_pocket=pocket, adjust_shape=pocket).cpu()
    want = oracle_sizes(logits.numpy(), table, SEEDS)
    assert sizes.dtype == torch.int32 and sizes.tolist() == want
    assert len(set(want)) > 1, want
    n_frag = data['fragment_mask'].reshape(B, -1).sum(1).long()
    n_cap = int(n_frag.max()) + max(table)
    assert chain.shape[2] == n_cap and nm.shape[1] == n_cap
    # the existing seeded path on create_templates_for_linker_generation of those sizes, padded to N_cap
    kw, _ = ddpm_mod._template_inputs(ddpm, data, torch.tensor(want, device=dev()), n_nodes=n_cap)
    assert torch.equal(kw['node_mask'], nm)
    ref = ddpm.edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    assert torch.equal(chain, ref)
    # the template itself: create_templates at those sizes (to its own padding), with the rows after it dead
    t = create_templates_for_linker_generation(data, torch.tensor(want, device=dev()))
    n = t['atom_mask'].shape[1]
    assert torch.equal(nm[:, :n], t['atom_mask']) and not nm[:, n:].any()


def draw_counts(ddpm, data, nn, seeds, rounds, table):
    """Connected rows after `rounds` rounds that keep the first size (sample_fn with the seeded draw)."""
    pocket = '.' in ddpm.train_data_prefix
    fn = lambda dd: draw_sizes(nn.size_logits(dd, with_pocket=pocket, adjust_shape=pocket), table, seeds)
    ddpm.sample_chain(data, sample_fn=fn, seeds=seeds, keep_frames=2, nan_retries=rounds, require_connected=True)
    return int(ddpm.edm.last_connected.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", [("fc", "simt"), ("fc", "auto"), ("pocket_4A", "simt")])
def test_rounds_redraw_the_sizes_of_the_rows_they_resample(case, impl):
    ddpm, data = model_and_data(case, impl)
    edm = ddpm.edm
    table = [0, 1, 2]
    nn = size_model(dev(), table, bias=[-1.0, 0.5, 0.2])
    B = len(SEEDS)
    pocket = pocket_args(case)
    logits = nn.size_logits(data, with_pocket=pocket, adjust_shape=pocket).cpu().numpy()
    n_frag = data['fragment_mask'].reshape(B, -1).sum(1).long().cpu()
    runs = []
    for r in range(ROUNDS + 1):
        chain, nm = ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, keep_frames=2, nan_retries=r,
                                      require_connected=True)
        runs.append((chain, nm, edm.last_sizes.clone(), edm.last_connected.clone(), edm.last_attempts.clone(),
                     edm.last_seeds.clone()))
    chain, nm, sizes, conn, attempts, used = runs[-1]
    base, _, sizes0, conn0, _, _ = runs[0]
    assert torch.isfinite(chain).all()
    # every row's size is the draw of the seed that produced it, and the node mask that of those sizes
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
    assert sizes.tolist() == oracle_sizes(logits, table, [int(s) for s in used])
    for c_r, nm_r, s_r, *_ in runs:
        live = torch.arange(nm_r.shape[1])[None, :] < (n_frag + s_r.long())[:, None]
        assert torch.equal(nm_r.reshape(B, -1).cpu(), live.to(nm_r.dtype))
    # rows that were never resampled are the first draw's, sizes included
    healthy = conn0.nonzero().flatten().tolist()
    assert 0 < len(healthy) < B, healthy
    assert torch.equal(chain[:, healthy], base[:, healthy]) and torch.equal(sizes[healthy], sizes0[healthy])
    assert all(int(attempts[b]) == 0 for b in healthy)
    # fewer rounds reproduce the prefix: a row is the longer run's from the round that connected it on
    first = [int(attempts[b]) if conn[b] else None for b in range(B)]
    counts = []
    for r, (c_r, _, s_r, conn_r, att_r, _) in enumerate(runs):
        counts.append(int(conn_r.sum()))
        for b in range(B):
            if first[b] is not None and first[b] <= r:
                assert bool(conn_r[b]) and int(att_r[b]) == first[b], (r, b)
                assert torch.equal(c_r[:, b], chain[:, b]) and int(s_r[b]) == int(sizes[b]), (r, b)
    assert counts == sorted(counts), counts
    # a recovered row is its molecule sampled alone, its input padded as in the batch, with the seed recorded for it
    recovered = [b for b in range(B) if int(attempts[b]) > 0]
    for b in recovered:
        alone, nm_b = ddpm.sample_chain(rows_of(data, [b]), linker_sizes=nn, seeds=[int(used[b])], keep_frames=2)
        assert int(edm.last_sizes[0]) == int(sizes[b]), b
        n = nm_b.shape[1]
        assert torch.equal(nm_b[0], nm[b, :n]) and not nm[b, n:].any()
        got = chain[:, b, :n]
        assert torch.equal(got, alone[:, 0]) if impl == "simt" else \
            bool((got - alone[:, 0]).abs().max() <= 1e-4 * alone.abs().max().clamp(min=1.0)), b
    fixed = draw_counts(ddpm, data, nn, SEEDS, ROUNDS, table)
    print(f"{case}/{impl}: connected after rounds 0..{ROUNDS} with redraws: {counts} of {B}; sizes {sizes.tolist()} "
          f"(first draw {sizes0.tolist()}); recovered rows {recovered}; the fixed-size rounds connect {fixed} of {B}")


@pytest.mark.gpu
def test_sample_many_and_a_device_split_equal_the_single_calls():
    ddpm, data = model_and_data("fc", "simt", rows=8)
    edm = ddpm.edm
    nn = size_model(dev(), [0, 1, 2], bias=[-1.0, 0.5, 0.2])
    parts = [[0, 1, 2], [3, 4, 5, 6, 7]]
    datas = [collate([small_fragment_items("fc", 8)[i] for i in p]) for p in parts]
    datas = [{k: (v.to(dev()) if torch.is_tensor(v) else v) for k, v in dd.items()} for dd in datas]
    seeds = [[SEEDS[i] for i in p] for p in parts]
    opts = dict(keep_frames=2, nan_retries=ROUNDS, require_connected=True)
    singles = []
    for dd, s in zip(datas, seeds):
        chain, nm = ddpm.sample_chain(dd, linker_sizes=nn, seeds=s, **opts)
        singles.append((chain, nm, edm.last_sizes, edm.last_seeds))
    many = ddpm.sample_many(datas, linker_sizes=nn, seeds=seeds, **opts)
    for k, ((chain, nm), (c1, nm1, s1, u1)) in enumerate(zip(many, singles)):
        assert torch.equal(chain, c1) and torch.equal(nm, nm1), k
        assert torch.equal(edm.last_sizes_many[k], s1) and torch.equal(edm.last_seeds_many[k], u1), k
    whole, nm = ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, **opts)
    sizes, used = edm.last_sizes, edm.last_seeds
    edm.devices = [0, 0]
    try:
        split, nm_s = ddpm.sample_chain(data, linker_sizes=nn, seeds=SEEDS, **opts)
    finally:
        edm.devices = None
    assert torch.equal(split, whole) and torch.equal(nm_s, nm)
    assert torch.equal(edm.last_sizes, sizes) and torch.equal(edm.last_seeds, used)
    assert int(edm.last_attempts.max()) > 0                             # some row was redrawn


@pytest.mark.gpu
def test_ranges_and_ints_and_the_seeded_sample_sizes():
    ddpm, data = model_and_data("fc", "simt")
    B = len(SEEDS)
    ddpm.sample_chain(data, linker_sizes=(1, 3), seeds=SEEDS, keep_frames=2)
    assert ddpm.edm.last_sizes.tolist() == [1 + int(np.floor(oracle_uniform(s & M64) * 3)) for s in SEEDS]
    ddpm.sample_chain(data, linker_sizes=2, seeds=SEEDS, keep_frames=2)
    assert ddpm.edm.last_sizes.tolist() == [2] * B
    nn = size_model(dev(), [0, 1, 2, 5])
    got = nn.sample_sizes(data, seeds=SEEDS)
    want = oracle_sizes(nn.size_logits(data).cpu().numpy(), [0, 1, 2, 5], SEEDS)
    assert got.dtype == torch.int8 and got.tolist() == want
    ddpm.edm.noise_mode = 'per_molecule'                               # seeds from draw_seeds, recorded in last_seeds
    torch.manual_seed(9)
    ddpm.sample_chain(data, linker_sizes=nn, keep_frames=2)
    assert ddpm.edm.last_sizes.tolist() == oracle_sizes(nn.size_logits(data).cpu().numpy(), [0, 1, 2, 5],
                                                        seeds_tensor(ddpm.edm.last_seeds, B).tolist())
