"""Uniqueness in the recovery rounds: `sample_chain(..., require_unique=True)`, dl_sample_chain_retry with DL_CHECK_UNIQUE,
and the graph hash alone, dl_molecule_hash / molecule_builder.graph_hashes.

The hash (Weisfeiler-Lehman colour refinement over the checked atoms, their types and get_bond_order orders) and the
verdict are stated at DL_CHECK_UNIQUE in the header; graph_hash_oracle restates both on the host. CPU tests check the
oracle's invariances and limits, the verdict rule, the refusals, the binding and the header; the GPU tests check the
kernel bit for bit against the oracle and the sampler end to end."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, molecule_builder as mb, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import retry_seed
import dl_helpers as helpers
import graph_hash_oracle as gho
import test_connected_resampling as tcr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
C, O, N_, F, S, CL, BR, I, P = range(9)


def orders_of(n, bonds):
    o = np.zeros((n, n), np.int64)
    for i, j, k in bonds:
        o[i, j] = o[j, i] = k
    return o


def relabel(types, orders, perm):
    """The same graph with atom perm[i] renamed i."""
    types = np.asarray(types)[perm]
    return types, orders[np.ix_(perm, perm)]


# ---- CPU: the oracle ----------------------------------------------------------------------------------------------------

# small molecules as (types, bonds): each of the others differs from "propanol" in one element, one order or one bond
PROPANOL = ([C, C, C, O], [(0, 1, 1), (1, 2, 1), (2, 3, 1)])
NEIGHBOURS = {
    "propylamine": ([C, C, C, N_], [(0, 1, 1), (1, 2, 1), (2, 3, 1)]),
    "propanal": ([C, C, C, O], [(0, 1, 1), (1, 2, 1), (2, 3, 2)]),
    "propene-ol": ([C, C, C, O], [(0, 1, 2), (1, 2, 1), (2, 3, 1)]),
    "isopropanol": ([C, C, C, O], [(0, 1, 1), (1, 2, 1), (1, 3, 1)]),
    "cyclopropanol": ([C, C, C, O], [(0, 1, 1), (1, 2, 1), (2, 3, 1), (0, 2, 1)]),
    "propane + water": ([C, C, C, O], [(0, 1, 1), (1, 2, 1)]),
    "methoxyethane": ([C, C, O, C], [(0, 1, 1), (1, 2, 1), (2, 3, 1)]),
    "fluoropropane": ([C, C, C, F], [(0, 1, 1), (1, 2, 1), (2, 3, 1)]),
}


def test_oracle_hash_is_invariant_under_relabelling():
    types, bonds = PROPANOL
    o = orders_of(4, bonds)
    h = gho.graph_hash(types, o)
    rng = np.random.default_rng(0)
    for _ in range(10):
        perm = rng.permutation(4)
        assert gho.graph_hash(*relabel(types, o, perm)) == h
    # a larger ring with a branch, relabelled
    types = [C] * 6 + [O, N_]
    o = orders_of(8, [(k, (k + 1) % 6, 1 + (k % 2)) for k in range(6)] + [(0, 6, 1), (3, 7, 1)])
    h = gho.graph_hash(types, o)
    for _ in range(10):
        assert gho.graph_hash(*relabel(types, o, rng.permutation(8))) == h
    assert gho.graph_hash([], np.zeros((0, 0))) == gho.mix(0) == 0


def test_oracle_hash_tells_apart_molecules_one_edit_away():
    hashes = {"propanol": gho.graph_hash(PROPANOL[0], orders_of(4, PROPANOL[1]))}
    for name, (types, bonds) in NEIGHBOURS.items():
        hashes[name] = gho.graph_hash(types, orders_of(len(types), bonds))
    assert len(set(hashes.values())) == len(hashes), hashes


def test_oracle_hash_cannot_tell_1wl_equivalent_graphs_apart():
    """Decalin (two fused six-rings) and bicyclopentyl (two five-rings joined by a bond): ten carbons, eleven single bonds,
    two atoms of degree 3 and eight of degree 2 with the same colour-refinement histories. The hash documents this limit."""
    decalin = orders_of(10, [(k, (k + 1) % 6, 1) for k in range(6)] +
                        [(0, 6, 1), (6, 7, 1), (7, 8, 1), (8, 9, 1), (9, 5, 1)])
    bicyclopentyl = orders_of(10, [(k, (k + 1) % 5, 1) for k in range(5)] +
                              [(5 + k, 5 + (k + 1) % 5, 1) for k in range(5)] + [(0, 5, 1)])
    assert decalin.sum() == bicyclopentyl.sum() == 22
    assert gho.graph_hash([C] * 10, decalin) == gho.graph_hash([C] * 10, bicyclopentyl)


def coords_molecule():
    """A small molecule with coordinates: a bent C-C-C-O chain with a C=O branch and a C#N, every pair more than 1 pm away
    from its thresholds (ZINC tables)."""
    x = np.array([[0.0, 0.0, 0.0], [1.5, 0.0, 0.0], [2.2, 1.3, 0.0], [3.6, 1.3, 0.0], [1.9, -1.1, 0.2],
                  [-0.8, -1.0, -0.6], [-1.3, -1.8, -1.1]], np.float32)
    types = np.array([C, C, C, O, O, C, N_])
    return x, types


def rotation(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def test_oracle_hash_is_invariant_under_padding_and_rigid_motion():
    x, types = coords_molecule()
    thr = [t.numpy() for t in mb.threshold_tables(False)]
    o, near = gho.bond_order_matrix(x, types, thr)
    assert near > 1.0 and o.sum() > 0
    assert set(o.flatten().tolist()) == {0, 1, 2, 3}                     # single, double and triple bonds
    h = gho.graph_hash(types, o)
    F8 = 8
    for seed in range(4):
        xr = (x @ rotation(seed).T + np.random.default_rng(seed).normal(size=3) * 10).astype(np.float32)
        perm = np.random.default_rng(seed + 10).permutation(7)
        N = 12
        xh = torch.zeros(1, N, 3 + F8)
        rows = np.random.default_rng(seed + 20).choice(N, 7, replace=False)
        nm = torch.zeros(1, N, dtype=torch.int8)
        xh[0, :, :3] = 50.0                                              # padding rows, somewhere
        for k, r in enumerate(rows):
            xh[0, r, :3] = torch.from_numpy(xr[perm[k]])
            xh[0, r, 3:] = 0.0
            xh[0, r, 3 + int(types[perm[k]])] = 1.0
            nm[0, r] = 1
        got, near_b = gho.batch_hashes(xh, nm, False)
        assert near_b[0] > 1.0 and got[0] == h, seed


def test_verdict_oracle_rule():
    U, CN = gho.UNIQUE, 1
    req = U | CN
    # first loop: every row a candidate, the lower index wins among eligible ones
    assert gho.verdict([5, 5, 6], [0, 0, 0], [CN, CN, CN], req) == [CN | U, CN, CN | U]
    # an ineligible earlier duplicate (disconnected, or diverged) does not block a later row
    assert gho.verdict([5, 5], [0, 0], [0, CN], req) == [U, CN | U]
    assert gho.verdict([5, 5], [1, 0], [CN, CN], req) == [CN | U, CN | U]
    # a round: row 0 is a keeper and never loses the bit; candidate 2 repeats it, candidate 3 repeats candidate 1
    passed = [CN | U, CN, CN, CN]
    out = gho.verdict([7, 8, 7, 8], [0, 0, 0, 0], passed, req, candidates=[1, 2, 3])
    assert out == [CN | U, CN | U, CN, CN]
    # a row outside the candidates that does not pass every bit is no keeper
    out = gho.verdict([7, 7], [0, 0], [CN, CN], req, candidates=[1])
    assert out == [CN, CN | U]


# ---- CPU: refusals, binding, header -------------------------------------------------------------------------------------

@pytest.mark.parametrize("inpainting", [False, True])
def test_require_unique_refuses_what_cannot_recover_one_call(inpainting):
    ddpm, kw = tcr._cpu_model(inpainting)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(1, B + 1))
    assert edm.require_unique is False and edm.last_unique is None and edm.last_graph_hashes is None
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_unique"):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_unique=bad)
    with pytest.raises(ValueError, match="require_unique needs per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2, require_unique=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_unique=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="require_unique does not take batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_unique=True, seeds=seeds, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_unique needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_unique=True, seeds=seeds)
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="require_unique.*replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_unique=True, seeds=seeds)
    delattr(edm, name)
    edm.require_unique = True                                            # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.is_geom = None
    with pytest.raises(ValueError, match="require_unique needs the bond tables"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    assert edm.last_unique is None and edm.last_graph_hashes is None


def test_require_unique_refuses_a_split_and_sample_many(monkeypatch):
    """A split into several slices is refused before any engine is built (the slices recover independently), and
    sample_many refuses the attribute (a launch packs several requests). Host inputs reach both checks: the split check
    reads only the slices, and sample_many refuses before it looks at the device."""
    ddpm, kw = tcr._cpu_model()
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(1, B + 1))
    # stand in for CUDA inputs and two visible devices up to the point where the slices are known
    from difflinker_b200 import edm as edm_mod
    monkeypatch.setattr(type(edm), "_require_check", lambda self, name, value, *a: bool(
        getattr(self, name) if value is None else value))
    monkeypatch.setattr(type(edm), "_per_molecule_seeds", lambda self, *a: torch.zeros(B, dtype=torch.int64))
    monkeypatch.setattr(type(edm.dynamics), "_check_graph_type", lambda self: None)
    monkeypatch.setattr(edm_mod, "device_slices", lambda n, devices: [(0, 0, 0, 1), (0, 1, 1, n)])
    monkeypatch.setattr(edm, "_devices", [0, 0])                        # what devices = [0, 0] sets on a GPU machine
    with pytest.raises(ValueError, match="require_unique.*2 slices"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_unique=True)
    monkeypatch.undo()
    edm.require_unique = True
    with pytest.raises(ValueError, match="sample_many does not take require_unique"):
        edm.sample_many([kw], keep_frames=2, seeds=[seeds])
    with pytest.raises(TypeError):
        edm.sample_many([kw], keep_frames=2, seeds=[seeds], require_unique=True)


def test_ddpm_passes_require_unique_to_the_edm():
    ddpm, _ = tcr._cpu_model()
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append(k.get('require_unique', 'unset'))
    from difflinker_b200 import ddpm as ddpm_mod
    ddpm.sample_chain(data, keep_frames=2, require_unique=True)
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, require_unique=False)
    assert seen == [True, 'unset', False]


def test_native_binds_the_hash_and_refuses_bad_arguments():
    lib = _native.load_library()
    assert "dl_molecule_hash" in _native.SYMBOLS and _native.CHECK_UNIQUE == 8
    assert lib.dl_molecule_hash.argtypes[2]._type_ is _native.DLMoleculeChecks
    ck = _native.DLMoleculeChecks(_native.CHECK_UNIQUE, 8, 1, 1, 1, None, None)
    # dl_molecule_check keeps refusing the bit, and says where the hashes are
    assert lib.dl_molecule_check(1, 4, ck, 1, 11, 1, None, 0, 0, 1, None, None) == -1
    err = lib.dl_last_error()
    assert b"require" in err and b"dl_molecule_hash" in err
    # the retry entry accepts the bit (it fails on the null engine first) and still refuses unknown bits
    for require in (8, 8 | 1):
        c = _native.DLMoleculeChecks(require, 8, 1, 1, 1, None, None)
        assert lib.dl_sample_chain_retry(None, 0, 2, 4, 10, 1, *[None] * 10, 1, 3, 1, 1, c, 1, None, None, None) == -1
        assert b"null engine" in lib.dl_last_error()
    # refusals before any pointer is read
    no_thr = _native.DLMoleculeChecks(0, 8, 1, None, 1, None, None)
    for args, why in (((1, 4, None, 1, 11, 1, None, 0, 0, 1, None), b"null checks"),
                      ((0, 4, ck, 1, 11, 1, None, 0, 0, 1, None), b"B and N"),
                      ((1, 8193, ck, 1, 11, 1, None, 0, 0, 1, None), b"8192"),
                      ((1, 4, ck, 1, 10, 1, None, 0, 0, 1, None), b"n_types"),
                      ((1, 4, no_thr, 1, 11, 1, None, 0, 0, 1, None), b"thr1, thr2 and thr3"),
                      ((1, 4, ck, None, 11, 1, None, 0, 0, 1, None), b"invalid argument"),
                      ((1, 4, ck, 1, 11, 1, None, 0, 0, None, None), b"invalid argument"),
                      ((1, 4, ck, 1, 11, 1, None, 0, 1, 1, None), b"invalid argument")):
        assert lib.dl_molecule_hash(*args) == -1, why
        assert why in lib.dl_last_error() and b"dl_molecule_hash" in lib.dl_last_error(), why


def test_header_compiles_as_c99_with_the_unique_bit_and_the_hash(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "unique_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2], hash[2]; int32_t attempts[2], flags[2], passed[2];\n"
        "  float thr[64] = {0}, xh[22] = {0}; int8_t nm[2] = {0};\n"
        "  dl_molecule_checks ck = {DL_CHECK_UNIQUE | DL_CHECK_CONNECTED, 8, thr, thr, thr, NULL, NULL};\n"
        "  dl_status a = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                      NULL, NULL, NULL, NULL, flags, 3, used, attempts, &ck, passed, NULL, NULL,\n"
        "                                      NULL);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  dl_status b = dl_molecule_hash(2, 8193, &ck, xh, 11, nm, NULL, 0, 0, hash, NULL);\n"
        '  printf("%d|%s|", (int)b, dl_last_error());\n'
        "  ck.require = DL_CHECK_UNIQUE;\n"
        "  dl_status c = dl_molecule_check(2, 4, &ck, xh, 11, nm, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)c, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "unique_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, err_a, b, err_b, c, err_c = res.stdout.strip().split("|", 5)
    assert int(a) == -1 and "null engine" in err_a
    assert int(b) == -1 and "dl_molecule_hash" in err_b and "8192" in err_b
    assert int(c) == -1 and "require" in err_c and "dl_molecule_hash" in err_c


# ---- GPU: the hash, molecule by molecule --------------------------------------------------------------------------------

def device_hashes(xh, nm, is_geom, po=None):
    d = tcr.dev()
    return mb.graph_hashes(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d)).cpu()


def assert_hashes_match(xh, nm, is_geom, po=None):
    """The kernel against the oracle on every molecule, which measures its pairs as the kernel does; returns the oracle's
    hashes."""
    got = device_hashes(xh, nm, is_geom, po)
    want, _ = gho.batch_hashes(xh, nm, is_geom, po)
    assert [int(h) for h in got] == [gho.as_int64(w) for w in want]
    return want


def one_hot_rows(x, types, N, F=9, far=50.0):
    xh = torch.zeros(N, 3 + F)
    xh[:, :3] = far
    xh[:, 3] = 1.0
    n = len(types)
    xh[:n, :3] = torch.as_tensor(np.asarray(x, np.float32))
    xh[:n, 3:] = torch.nn.functional.one_hot(torch.as_tensor(np.asarray(types), dtype=torch.long), F).float()
    nm = torch.zeros(N, dtype=torch.int8)
    nm[:n] = 1
    return xh, nm


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_kernel_matches_the_oracle_on_random_batches(is_geom):
    T = 9 if is_geom else 8
    g = torch.Generator().manual_seed(5)
    B, N = 96, 48
    n = torch.randint(0, N + 1, (B,), generator=g)
    nm = (torch.arange(N)[None, :] < n[:, None]).to(torch.int8)
    scale = 1.0 + 5.0 * torch.rand(B, 1, 1, generator=g)
    xh = torch.cat([torch.rand(B, N, 3, generator=g) * scale,
                    torch.nn.functional.one_hot(torch.randint(0, T, (B, N), generator=g), T).float()], 2)
    want = assert_hashes_match(xh, nm, is_geom)
    assert len(set(want)) > B // 2


@pytest.mark.gpu
def test_kernel_matches_the_oracle_on_purpose_built_molecules():
    x, types = coords_molecule()
    mols = [one_hot_rows(x, types, 16)]
    for seed in range(3):                                                # moved, turned and relabelled: the same hash
        perm = np.random.default_rng(seed).permutation(7)
        xr = (x @ rotation(seed).T + 3.0 * seed).astype(np.float32)
        mols.append(one_hot_rows(xr[perm], types[perm], 16))
    for k in range(7):                                                   # one element changed: a different hash
        t2 = types.copy()
        t2[k] = S if t2[k] != S else C
        mols.append(one_hot_rows(x, t2, 16))
    mols.append(one_hot_rows(np.zeros((0, 3)), [], 16))                  # no atom
    mols.append(one_hot_rows(x[:1], types[:1], 16))                      # one atom
    xh, nm = [torch.stack(t) for t in zip(*mols)]
    want = assert_hashes_match(xh, nm, False)
    assert len(set(want[:4])) == 1 and len(set(want[3:11])) == 8 and want[11] == 0


@pytest.mark.gpu
def test_kernel_drops_the_pocket_on_cut_off_batches_and_keeps_it_for_inpainting():
    """With pocket_only, pocket rows are not atoms (cut-off graphs); without it every atom counts (inpainting). A pocket
    that moves changes the second hash and not the first."""
    x, types = coords_molecule()
    g = torch.Generator().manual_seed(2)
    N, P_ = 40, 20
    mols, pos = [], []
    for k in range(3):
        v = torch.randn(P_, 3, generator=g)
        pocket = (6.0 + k) * v / v.norm(dim=1, keepdim=True)
        xa = np.concatenate([x, pocket.numpy()])
        ta = np.concatenate([types, torch.randint(0, 3, (P_,), generator=g).numpy()])
        mols.append(one_hot_rows(xa, ta, N))
        po = torch.zeros(N)
        po[7:7 + P_] = 1.0
        pos.append(po)
    xh, nm = [torch.stack(t) for t in zip(*mols)]
    po = torch.stack(pos)
    cut = assert_hashes_match(xh, nm, True, po)
    whole = assert_hashes_match(xh, nm, True)
    assert len(set(cut)) == 1 and len(set(whole)) == 3


@pytest.mark.gpu
def test_kernel_matches_the_oracle_on_rows_with_nan():
    x, types = coords_molecule()
    a, nm_a = one_hot_rows(x, types, 12)
    b = a.clone()
    b[2, 0] = float('nan')                                               # a NaN coordinate: that atom bonds to nothing
    c = a.clone()
    c[4, 3 + 2] = float('nan')                                           # a NaN feature: argmax takes it
    d = a.clone()
    d[:, :] = float('nan')
    xh = torch.stack([a, b, c, d])
    nm = torch.stack([nm_a] * 4)
    want = assert_hashes_match(xh, nm, False)
    assert len(set(want)) == 4


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4000, 8192])
def test_kernel_holds_up_to_the_checks_row_limit(N):
    """Molecule 0: a pocket of N - 60 rows around a 60-atom ligand, dropped as pocket rows (few atoms, many rows).
    Molecule 1: every row an atom -- chains of carbons 1.5 A apart, 2 bonds per atom, more than the shared-memory CSR holds
    at N = 8192, so some atoms rescan all pairs in every round. Molecule 2 is molecule 1 with its rows reversed."""
    g = torch.Generator().manual_seed(4)
    F9 = 9
    xh = torch.zeros(3, N, 3 + F9)
    nm = torch.ones(3, N, dtype=torch.int8)
    po = torch.zeros(3, N)
    types = torch.randint(0, 3, (N,), generator=g)
    v = torch.randn(N, 3, generator=g)
    xh[0, :, :3] = (20.0 + 30.0 * torch.rand(N, 1, generator=g)) * v / v.norm(dim=1, keepdim=True)
    lig = torch.randperm(N, generator=g)[:60]
    xh[0, lig, :3] = torch.tensor([[1.45 * (k % 6), 1.45 * (k // 6), 0.0] for k in range(60)])   # 5 pm from every threshold
    po[0] = 1.0
    po[0, lig] = 0.0
    xh[:, :, 3:] = torch.nn.functional.one_hot(types, F9).float()
    L = 64                                                               # chains of 64 carbons, 10 A apart
    k = torch.arange(N)
    xh[1, :, 0] = 1.5 * (k % L).float()
    xh[1, :, 1] = 10.0 * (k // L % 32).float()
    xh[1, :, 2] = 10.0 * (k // (L * 32)).float()
    xh[1, :, 3:] = torch.nn.functional.one_hot(torch.zeros(N, dtype=torch.long), F9).float()
    xh[2] = xh[1].flip(0)
    got = device_hashes(xh, nm, True, po)
    want0, near0 = gho.batch_hashes(xh[:1], nm[:1], True, po[:1])
    assert near0[0] > 0.01 and int(got[0]) == gho.as_int64(want0[0])
    # molecules 1 and 2: disjoint chains of carbons, bonded to their neighbours in the chain only (1.5 A; the chains 10 A
    # apart), so the oracle takes the bonds by construction instead of N^2 distances
    o = np.zeros((N, N), np.int8)
    for i in range(N - 1):
        if (i + 1) % L:
            o[i, i + 1] = o[i + 1, i] = 1
    want1 = gho.graph_hash([C] * N, o)
    assert int(got[1]) == int(got[2]) == gho.as_int64(want1) and int(got[1]) != int(got[0])


# ---- GPU: the sampler, end to end ---------------------------------------------------------------------------------------

SEEDS = list(range(201, 217))
ROUNDS = 4
DUP_CASES = [(g, impl) for g in ("fc", "pocket_4A") for impl in ("simt", "auto")]


def copies_items(case, rows):
    """One input copied `rows` times: the connectivity tests' carbon fragment and one linker atom (pocket cases add their
    12 pocket atoms). A single linker atom has few graphs to land on -- next to the fragment or away from it, with one of
    a few types -- so the seeds repeat each other's molecules."""
    one = tcr.small_fragment_items(case, 2)[1]                          # b % 3 == 1: one linker atom
    return [dict(one, uuid=b, name=f'dup_{b}') for b in range(rows)]


def build_copies(case, impl, rows=len(SEEDS)):
    d = tcr.dev()
    spec, over = tcr.model_spec(case, rows)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(tcr.COORD_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(copies_items(case, rows)).items()}
    return ddpm, sampler_inputs(ddpm, data), data


def pocket_only(ddpm, kw):
    return kw['context'][..., -1] if ddpm.edm.dynamics.graph_type != 'FC' else None


def check_hashes(ddpm, kw, chain0, got):
    """last_graph_hashes against graph_hashes and the oracle."""
    is_geom, po = ddpm.edm.is_geom, pocket_only(ddpm, kw)
    assert torch.equal(got, mb.graph_hashes(chain0, kw['node_mask'], is_geom, po).cpu())
    want, _ = gho.batch_hashes(chain0, kw['node_mask'], is_geom, po)
    assert [int(h) for h in got] == [gho.as_int64(w) for w in want]


def unsigned(hashes):
    return [int(h) % (1 << 64) for h in hashes]


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", DUP_CASES)
def test_report_only_keeps_the_chain_and_gives_the_oracle_verdict(case, impl):
    ddpm, kw, _ = build_copies(case, impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    assert edm.last_unique is None and edm.last_graph_hashes is None
    for extra in ({}, {'require_connected': True}):
        r0 = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=0, require_unique=True, **extra)
        assert torch.equal(r0, base)
        u, h = edm.last_unique, edm.last_graph_hashes
        assert u.dtype == torch.bool and u.shape == (B,) and h.dtype == torch.int64 and h.shape == (B,)
        check_hashes(ddpm, kw, base[0], h)
        passed = [_native.CHECK_CONNECTED if extra and edm.last_connected[b] else 0 for b in range(B)]
        require = gho.UNIQUE | (_native.CHECK_CONNECTED if extra else 0)
        want = gho.verdict(unsigned(h), [0] * B, passed, require)
        assert u.tolist() == [bool(w & gho.UNIQUE) for w in want], extra
    assert len(set(h.tolist())) < B                                      # the copies repeat each other


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", DUP_CASES)
@pytest.mark.parametrize("extra", [{}, {'require_connected': True}, {'require_valid': True}])
def test_rounds_resample_only_the_repeated_molecules(case, impl, extra):
    ddpm, kw, _ = build_copies(case, impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_unique=True, **extra)
    first = edm.last_unique.clone()
    for k in extra:                                                      # rows passing every check after the first loop
        first &= getattr(edm, {'require_connected': 'last_connected', 'require_valid': 'last_valid'}[k])
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=ROUNDS, require_unique=True, **extra)
    u, h, attempts, used = edm.last_unique, edm.last_graph_hashes, edm.last_attempts, edm.last_seeds
    assert torch.isfinite(chain).all()
    check_hashes(ddpm, kw, chain[0], h)
    # no two rows that pass every required check share a hash (rows failing another check may: they block no one)
    passing = u.clone()
    for k in extra:
        passing &= getattr(edm, {'require_connected': 'last_connected', 'require_valid': 'last_valid'}[k])
    kept = passing.nonzero().flatten().tolist()
    assert len({int(h[b]) for b in kept}) == len(kept)
    good = first.nonzero().flatten().tolist()
    if 'require_valid' in extra:                                         # the lattice's 1.2 A bonds are triple C-C bonds:
        assert not good and not kept                                     # no row is valid, every row is resampled
        assert (attempts == ROUNDS).all(), attempts
        return
    assert 0 < len(good) < B, good
    assert torch.equal(chain[:, good], base[:, good]) and all(int(attempts[b]) == 0 for b in good)
    assert all(bool(u[b]) for b in good)
    assert int(u.sum()) >= len(good)
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
        if int(attempts[b]) > 0:                                         # a resampled row is its molecule sampled alone
            alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert tcr.same(chain[:, b], alone[:, 0], impl), b
    print(f"{case}/{impl}/{sorted(extra)}: unique and passing {len(good)} of {B} after the loop, "
          f"{int(u.sum())} unique after {ROUNDS} rounds; attempts {attempts.tolist()}")


@pytest.mark.gpu
def test_redrawn_sizes_and_the_returned_node_mask_agree():
    ddpm, kw, data = build_copies("fc", "simt")
    edm = ddpm.edm
    B = len(SEEDS)
    chain, nm = ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS, nan_retries=ROUNDS, require_unique=True,
                                  linker_sizes=(1, 3))
    sizes, h, u = edm.last_sizes, edm.last_graph_hashes, edm.last_unique
    assert sizes.shape == (B,) and set(sizes.tolist()) <= {1, 2, 3}
    n_frag = int(data['fragment_mask'][0].sum())
    assert (nm.reshape(B, -1).ne(0).sum(1).cpu() == n_frag + sizes).all()
    assert torch.equal(h, mb.graph_hashes(chain[0], nm, edm.is_geom).cpu())
    kept = u.nonzero().flatten().tolist()
    assert len({int(h[b]) for b in kept}) == len(kept) and len(kept) > B // 2


@pytest.mark.gpu
def test_require_unique_false_launches_what_the_call_launched_before():
    ddpm, kw, _ = build_copies("fc", "simt")
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    counts = []
    for flag in ('unset', False, True):
        extra = {} if flag == 'unset' else {'require_unique': flag}
        n0 = int(lib.dl_launch_count(eng))
        edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=0, require_connected=True, **extra)
        counts.append(int(lib.dl_launch_count(eng)) - n0)
    assert counts[0] == counts[1] and counts[2] == counts[0] + 1        # the bit adds the verdict launch only
