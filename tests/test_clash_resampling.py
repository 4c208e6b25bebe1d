"""Pocket clashes in the recovery rounds: `sample_chain(..., require_clash_free=True)`, dl_sample_chain_retry with
DL_CHECK_CLASH, and dl_clash_check.

A linker atom of chain[0] clashes with a pocket atom when 100 |x_i - x_j| in pm is below clash[min type][max type] and that
entry is >= 0; a molecule passes when none of its linker atoms clashes with any pocket atom. This is the project's own
predicate (the reference has none), stated at dl_molecule_checks in the header. The oracle below restates it in numpy fp32.
CPU tests check the oracle, the default table, the refusals, the binding and the header; the GPU tests check the kernel
atom by atom on purpose-built and random batches, and the sampler end to end on pocket graphs."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, molecule_builder as mb, output, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import retry_seed, seeds_tensor
from oracle import bond_rounding as br
import dl_helpers as helpers
import test_connected_resampling as tcr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dist_pm(xi, xj):
    """100 |xi - xj| in fp32 in the direct form the clash check measures every pair in, at any atom count
    (sqrt(fma(dz, dz, fma(dy, dy, dx * dx))), oracle/bond_rounding.py)."""
    return br.direct_dist_pm(xi, xj)


def oracle_clashes(x, types, node_mask, linker_mask, pocket_only, table):
    """The oracle for one molecule: (N,) int64 counts of the pocket atoms each linker atom clashes with (0 elsewhere)."""
    x = np.asarray(x, np.float32)
    types = np.asarray(types)
    live = np.asarray(node_mask) != 0
    pocket = live & (np.asarray(pocket_only) != 0)
    linker = live & (np.asarray(linker_mask) != 0) & (np.asarray(pocket_only) == 0)
    table = np.asarray(table, np.float32)
    li, pi = np.nonzero(linker)[0], np.nonzero(pocket)[0]
    counts = np.zeros(x.shape[0], np.int64)
    if len(li) and len(pi):
        d = dist_pm(x[li][:, None, :], x[pi][None, :, :])
        t = table[np.minimum(types[li][:, None], types[pi][None, :]), np.maximum(types[li][:, None], types[pi][None, :])]
        hit = (t >= 0) & (d < t)                                          # a NaN distance compares false
        counts[li] = hit.sum(1)
    return counts


def oracle_batch(xh, nm, lm, po, is_geom, table=None):
    """((B,N) counts, (B,) clash-free) of a chain[0]-style batch."""
    T = 9 if is_geom else 8
    table = mb.clash_table(is_geom) if table is None else table
    xh = xh.cpu()
    types = torch.argmax(xh[:, :, 3:3 + T], dim=2).numpy()
    counts, ok = [], []
    for b in range(xh.shape[0]):
        c = oracle_clashes(xh[b, :, :3].numpy(), types[b], nm[b].cpu().numpy(), lm[b].cpu().numpy(),
                              po[b].cpu().numpy(), table.numpy())
        counts.append(torch.from_numpy(c))
        ok.append(not c.any())
    return torch.stack(counts), torch.tensor(ok)


# ---- CPU --------------------------------------------------------------------------------------------------------------

def threshold_pair(thr, inside):
    """A distance in A along one axis whose fp32 distance in pm is just below `thr` (inside) or exactly at / above it."""
    d = np.float32(thr / 100.0)
    step = np.float32(np.inf if not inside else -np.inf)
    while (dist_pm([0, 0, 0], [d, 0, 0]) < thr) != inside:
        d = np.nextafter(d, step)
    return float(d)


def test_clash_table_is_the_scaled_sum_of_bondi_radii():
    for is_geom, idx2atom in ((False, output.IDX2ATOM), (True, output.GEOM_IDX2ATOM)):
        t = mb.clash_table(is_geom)
        T = len(idx2atom)
        assert t.dtype == torch.float32 and t.shape == (T, T) and torch.equal(t, t.T)
        for a in range(T):
            for b in range(T):
                want = np.float32(100.0 * 0.75 * (mb.VDW_RADII[idx2atom[a]] + mb.VDW_RADII[idx2atom[b]]))
                assert t[a, b].item() == want, (a, b)
        half = mb.clash_table(is_geom, scale=0.5)
        assert torch.allclose(half, t * (0.5 / 0.75))
    t = mb.clash_table(True)
    C, O, N_ = 0, 1, 2
    assert t[C, C].item() == np.float32(255.0) and t[N_, O].item() == np.float32(230.25)
    assert set(mb.VDW_RADII) == set(output.GEOM_IDX2ATOM.values())


def test_oracle_on_pairs_either_side_of_every_threshold():
    for is_geom in (False, True):
        table = mb.clash_table(is_geom)
        T = table.shape[0]
        for a in range(T):
            for b in range(a, T):
                thr = table[a, b].item()
                for inside in (True, False):
                    d = threshold_pair(thr, inside)
                    x = np.array([[0, 0, 0], [d, 0, 0]], np.float32)
                    # the linker atom may be either type of the pair: the table is read [min][max]
                    for types in ((a, b), (b, a)):
                        c = oracle_clashes(x, np.array(types), [1, 1], [1, 0], [0, 1], table)
                        assert c.tolist() == [int(inside), 0], (is_geom, a, b, inside)
    table = mb.clash_table(False).clone()
    table[0, 0] = -1.0                                                   # a negative entry: the pair never clashes
    c = oracle_clashes(np.zeros((2, 3), np.float32), np.array([0, 0]), [1, 1], [1, 0], [0, 1], table)
    assert c.tolist() == [0, 0]


def _pocket_cpu_model():
    spec = synthetic.SPECS["cfg4_pockets"]
    ddpm, _ = helpers.build_ddpm(spec, 0)
    ddpm.edm.T = 4
    items = synthetic.make_items(spec, batch=3)
    return ddpm, sampler_inputs(ddpm, collate(items))


@pytest.mark.parametrize("kind", ["fc", "inpainting", "pocket"])
def test_clash_check_refuses_what_it_cannot_check(kind):
    """The refusals of require_valid (test_valence_refuses_what_connectivity_refuses), and FC graphs and InpaintingEDM."""
    ddpm, kw = _pocket_cpu_model() if kind == "pocket" else tcr._cpu_model(kind == "inpainting")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(1, B + 1))
    assert edm.require_clash_free is False and edm.last_clash_free is None and edm.last_clash_free_many is None
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_clash_free"):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_clash_free=bad)
    if kind != "pocket":
        why = "InpaintingEDM" if kind == "inpainting" else "FC graphs"
        with pytest.raises(ValueError, match=why):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_clash_free=True)
        edm.require_clash_free = True                                    # the attribute stands in for a missing argument
        with pytest.raises(ValueError, match=why):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
        assert edm.last_clash_free is None
        return
    with pytest.raises(ValueError, match="require_clash_free needs per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2, require_clash_free=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_clash_free=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="require_clash_free does not take batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_clash_free=True, seeds=seeds, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_clash_free needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_clash_free=True, seeds=seeds)
    setattr(edm, 'draw_noise', lambda *a, **k: None)
    with pytest.raises(ValueError, match="require_clash_free.*replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_clash_free=True, seeds=seeds)
    delattr(edm, 'draw_noise')
    edm.require_clash_free = True
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.is_geom = None
    with pytest.raises(ValueError, match="require_clash_free needs the bond tables"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    assert edm.last_clash_free is None


def test_models_pass_require_clash_free_to_the_edm():
    ddpm, _ = tcr._cpu_model()
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append(k.get('require_clash_free', 'unset'))
    ddpm.edm.sample_many = lambda reqs, **k: seen.append(k.get('require_clash_free', 'unset')) or [None] * len(reqs)
    from difflinker_b200 import ddpm as ddpm_mod, distributed
    ddpm.sample_chain(data, keep_frames=2, require_clash_free=True)
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, require_clash_free=False)
    ddpm.sample_many([data], keep_frames=2, seeds=[[1, 2, 3]], require_clash_free=True)
    ddpm_mod.sample_many(ddpm, [data], keep_frames=2, seeds=[[1, 2, 3]])
    distributed.sample_chain_sharded(ddpm, data, keep_frames=2, seeds=[1, 2, 3], require_clash_free=True)
    assert seen == [True, 'unset', False, True, 'unset', True]


def test_native_binds_the_clash_check_and_the_retry_entry():
    lib = _native.load_library()
    assert "dl_sample_chain_retry" in _native.SYMBOLS and "dl_clash_check" in _native.SYMBOLS
    assert _native.CHECK_CLASH == 4
    ck = _native.DLMoleculeChecks(_native.CHECK_CLASH, 8, 1, 1, 1, 1)   # the clash check alone runs through dl_clash_check
    assert lib.dl_molecule_check(1, 4, ck, 1, 11, 1, None, 0, 0, 1, None, None) == -1
    err = lib.dl_last_error()
    assert b"require" in err and b"dl_clash_check" in err
    assert lib.dl_sample_chain_retry(None, 0, 2, 4, 10, 1, *[None] * 10, 1, 3, 1, 1, ck, 1, None, None, None) == -1
    assert b"null engine" in lib.dl_last_error()
    # refusals before any pointer is read
    for args, why in (((0, 4, 8, 1, 1, 11, 1, 1, 1, 1, 1, None, None), b"B and N"),
                      ((1, 8193, 8, 1, 1, 11, 1, 1, 1, 1, 1, None, None), b"8192"),
                      ((1, 4, 9, 1, 1, 11, 1, 1, 1, 1, 1, None, None), b"n_types"),
                      ((1, 4, 8, None, 1, 11, 1, 1, 1, 1, 1, None, None), b"clash table"),
                      ((1, 4, 8, 1, 1, 11, 1, 1, None, 1, 1, None, None), b"invalid argument")):
        assert lib.dl_clash_check(*args) == -1, why
        assert why in lib.dl_last_error() and b"dl_clash_check" in lib.dl_last_error()


def test_header_compiles_as_c99_with_the_clash_table_in_the_checks(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "clash_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2]; int32_t attempts[2], flags[2], passed[2];\n"
        "  float clash[64] = {0}, xh[22] = {0}, lm[2] = {0}, ctx[2] = {0}; int8_t nm[2] = {0};\n"
        "  dl_molecule_checks ck = {DL_CHECK_CONNECTED | DL_CHECK_CLASH, 8, clash, NULL, NULL, NULL, clash};\n"
        "  dl_molecule_checks clash_only = {DL_CHECK_CLASH, 8, NULL, NULL, NULL, NULL, clash};\n"
        "  dl_status a = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                      NULL, NULL, NULL, NULL, flags, 3, used, attempts, &ck, passed, NULL, NULL,\n"
        "                                      NULL);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  dl_status b = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                      NULL, NULL, NULL, NULL, flags, 3, used, attempts, &clash_only, passed, NULL,\n"
        "                                      NULL, NULL);\n"
        '  printf("%d|%s|", (int)b, dl_last_error());\n'
        "  dl_status c = dl_clash_check(2, 8193, 8, clash, xh, 11, nm, lm, ctx, 1, passed, NULL, NULL);\n"
        '  printf("%d|%s|", (int)c, dl_last_error());\n'
        "  dl_status d = dl_clash_check(2, 1, 8, NULL, xh, 11, nm, lm, ctx, 1, passed, NULL, NULL);\n"
        '  printf("%d|%s|", (int)d, dl_last_error());\n'
        "  ck.require = DL_CHECK_CLASH;\n"
        "  dl_status e = dl_molecule_check(2, 4, &ck, xh, 11, nm, ctx, 1, 1, passed, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)e, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "clash_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, err_a, b, err_b, c, err_c, d, err_d, e, err_e = res.stdout.strip().split("|", 9)
    assert int(a) == -1 and "null engine" in err_a
    assert int(b) == -1 and "null engine" in err_b
    assert int(c) == -1 and "dl_clash_check" in err_c and "8192" in err_c
    assert int(d) == -1 and "dl_clash_check" in err_d and "clash table" in err_d
    assert int(e) == -1 and "require" in err_e and "dl_clash_check" in err_e


# ---- GPU: the kernel, atom by atom --------------------------------------------------------------------------------------

C, O, N_, F, S, CL, BR, I, P = range(9)
FAR = 50.0                                                               # A: padding and spare atoms, out of every reach


def run_clash(xh, nm, lm, po, is_geom, table=None):
    """dl_clash_check on the device: ((B,) clash-free, (B,N) counts) on the host."""
    d = tcr.dev()
    args = (xh.to(d), nm.to(d), lm.to(d), po.to(d), is_geom)
    ok = mb.clash_free(*args, clash=table).cpu()
    counts = mb.pocket_clashes(*args, clash=table).cpu()
    return ok, counts


def assert_matches_oracle(xh, nm, lm, po, is_geom, table=None):
    ok, counts = run_clash(xh, nm, lm, po, is_geom, table)
    want_counts, want_ok = oracle_batch(xh, nm, lm, po, is_geom, table)
    assert torch.equal(counts.long(), want_counts)
    assert torch.equal(ok, want_ok)
    return ok, counts


def molecule(rows, N, F=9):
    """One (N, 3+F) molecule and its (N,) masks from rows (pos, type, kind) with kind in 'linker', 'frag', 'pocket',
    'pad'; the rest padded far away."""
    xh = torch.zeros(N, 3 + F)
    xh[:, :3] = FAR
    xh[:, 3] = 1.0
    nm, lm, po = torch.zeros(N, dtype=torch.int8), torch.zeros(N), torch.zeros(N)
    for r, (pos, t, kind) in enumerate(rows):
        xh[r, :3] = torch.as_tensor(pos, dtype=torch.float32)
        xh[r, 3:] = 0.0
        xh[r, 3 + t] = 1.0
        nm[r] = kind != 'pad'
        lm[r] = kind == 'linker'
        po[r] = kind == 'pocket'
    return xh, nm, lm, po


def stack(mols):
    return [torch.stack(t) for t in zip(*mols)]


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_kernel_matches_the_oracle_either_side_of_every_threshold(is_geom):
    """One molecule per type pair and side: a linker atom at the origin and a pocket atom just inside or just outside the
    pair's threshold on the x axis (one non-zero component, so the fp32 distance is exact on either side)."""
    table = mb.clash_table(is_geom)
    T = table.shape[0]
    mols, want = [], []
    for a in range(T):
        for b in range(T):
            for inside in (True, False):
                d = threshold_pair(table[a, b].item(), inside)
                mols.append(molecule([((0, 0, 0), a, 'linker'), ((d, 0, 0), b, 'pocket')], 4))
                want.append(not inside)
    xh, nm, lm, po = stack(mols)
    ok, counts = assert_matches_oracle(xh, nm, lm, po, is_geom)
    assert ok.tolist() == want
    assert counts[:, 0].tolist() == [int(not w) for w in want] and not counts[:, 1:].any()
    # a negative entry exempts the pair; the other pairs keep their verdicts
    own = table.clone()
    own[C, O] = own[O, C] = -1.0
    ok2, _ = assert_matches_oracle(xh, nm, lm, po, is_geom, own)
    for k in range(len(mols)):
        a, b = divmod(k // 2, T)
        assert bool(ok2[k]) == (want[k] or {a, b} == {C, O}), (a, b)


@pytest.mark.gpu
def test_kernel_ignores_what_is_not_a_linker_pocket_pair():
    close = 1.0                                                          # A: closer than every threshold
    cases = [
        ("linker clashes", [((0, 0, 0), C, 'linker'), ((close, 0, 0), C, 'pocket')], False, [1, 0]),
        ("fragment-pocket contact", [((0, 0, 0), C, 'frag'), ((close, 0, 0), C, 'pocket')], True, [0, 0]),
        ("pocket-pocket contact", [((0, 0, 0), C, 'pocket'), ((close, 0, 0), C, 'pocket'), ((9, 0, 0), C, 'linker')],
         True, [0, 0, 0]),
        ("linker-fragment contact", [((0, 0, 0), C, 'linker'), ((close, 0, 0), C, 'frag')], True, [0, 0]),
        ("padded pocket row", [((0, 0, 0), C, 'linker'), ((close, 0, 0), C, 'pad')], True, [0, 0]),
        ("no linker atom", [((0, 0, 0), C, 'frag'), ((5, 0, 0), C, 'pocket')], True, [0, 0]),
        ("no pocket atom", [((0, 0, 0), C, 'linker'), ((close, 0, 0), C, 'linker')], True, [0, 0]),
        ("no atom", [((0, 0, 0), C, 'pad')], True, [0]),
        ("two pocket atoms", [((0, 0, 0), N_, 'linker'), ((close, 0, 0), O, 'pocket'), ((0, close, 0), S, 'pocket'),
                              ((0, 0, 4.0), C, 'pocket')], False, [2, 0, 0, 0]),
        ("NaN linker row", [((float('nan'), 0, 0), C, 'linker'), ((0, 0, 0), C, 'pocket')], True, [0, 0]),
    ]
    mols = [molecule(rows, 6) for _, rows, _, _ in cases]
    xh, nm, lm, po = stack(mols)
    # a linker row flagged in the pocket column is a pocket atom, not a linker atom
    x2, n2, l2, p2 = molecule([((0, 0, 0), C, 'linker'), ((close, 0, 0), C, 'pocket')], 6)
    p2[0] = 1.0
    xh, nm, lm, po = [torch.cat([t, u[None]]) for t, u in zip((xh, nm, lm, po), (x2, n2, l2, p2))]
    ok, counts = assert_matches_oracle(xh, nm, lm, po, True)
    for b, (name, rows, want, want_counts) in enumerate(cases):
        assert bool(ok[b]) == want, name
        assert counts[b, :len(want_counts)].tolist() == want_counts and not counts[b, len(want_counts):].any(), name
    assert bool(ok[-1]) and not counts[-1].any()


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4000, 8192])
def test_a_linker_in_a_whole_protein_pocket(N):
    """A pocket of N - 40 rows spread over every 256-row chunk of the compaction (80 KB or more of shared memory), a ligand
    of 40 rows among them, 20 of them linker atoms; molecule 1 moves two pocket atoms onto linker atoms."""
    g = torch.Generator().manual_seed(3)
    xh = torch.zeros(2, N, 12)
    types = torch.randint(0, 9, (2, N), generator=g)
    xh[:, :, 3:] = torch.nn.functional.one_hot(types, 9).float()
    nm = torch.ones(2, N, dtype=torch.int8)
    po = torch.ones(2, N)
    lm = torch.zeros(2, N)
    lig = torch.randperm(N, generator=g)[:40]
    link = lig[:20]
    v = torch.randn(N, 3, generator=g)
    shell = (8.0 + 30.0 * torch.rand(N, 1, generator=g)) * v / v.norm(dim=1, keepdim=True)   # pocket: 8 A and beyond
    ligand = 2.0 * torch.rand(40, 3, generator=g) - 1.0                                       # ligand: within 1.8 A
    for b in range(2):
        xh[b, :, :3] = shell
        xh[b, lig, :3] = ligand
        po[b, lig] = 0.0
        lm[b, link] = 1.0
    nm[:, lig[-1]] = 0                                                   # a padded ligand row
    pocket_rows = torch.tensor([r for r in range(N) if r not in set(lig.tolist())][:2])
    xh[1, pocket_rows, :3] = xh[1, link[:2], :3] + torch.tensor([0.5, 0.0, 0.0])
    ok, counts = assert_matches_oracle(xh, nm, lm, po, True)
    assert ok.tolist() == [True, False] and int(counts[1].sum()) >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_kernel_matches_the_oracle_on_random_batches(is_geom):
    """Random ligands in random pockets, every molecule compared: the oracle measures in the kernel's direct form."""
    T = 9 if is_geom else 8
    g = torch.Generator().manual_seed(11)
    B, N = 128, 60
    n = torch.randint(1, N + 1, (B,), generator=g)
    nm = (torch.arange(N)[None, :] < n[:, None]).to(torch.int8)
    po = (torch.rand(B, N, generator=g) < 0.6).float()
    lm = ((torch.rand(B, N, generator=g) < 0.5) & (po == 0)).float()
    scale = 1.0 + 6.0 * torch.rand(B, 1, 1, generator=g)
    xh = torch.cat([torch.rand(B, N, 3, generator=g) * scale,
                    torch.nn.functional.one_hot(torch.randint(0, T, (B, N), generator=g), T).float()], 2)
    ok, counts = run_clash(xh, nm, lm, po, is_geom)
    want_counts, want_ok = oracle_batch(xh, nm, lm, po, is_geom)
    assert torch.equal(counts.long(), want_counts) and torch.equal(ok, want_ok)
    assert 0 < int(want_ok.sum()) < B, int(want_ok.sum())              # both outcomes are exercised


# ---- GPU: the sampler, end to end ---------------------------------------------------------------------------------------

SEEDS = list(range(31, 47))
ROUNDS = 4
CASES = [(g, impl) for g in ("4A", "FC-10A-4A") for impl in ("simt", "auto")]
# The lattice, noise precision and coordinate gain of the connectivity tests, whose linker atoms end next to the fragment
# for some seeds and away from it for others. Here pocket atoms sit on a shell POCKET_R from the fragment's centre, so a
# linker atom that ends out on that shell's side comes within a clash distance of one of them and one near the fragment
# does not.
FRAG = tcr.FRAG
NF = tcr.NF
POCKET = 24
POCKET_R = 4.0


def pocket_items(rows):
    g = torch.Generator().manual_seed(79)
    items = []
    for b in range(rows):
        link = torch.tensor([[0.0, 0.0, 1.8], [0.0, 0.0, 3.0]])[:1 + b % 2]
        v = torch.randn(POCKET, 3, generator=g)
        pos = torch.cat([FRAG, POCKET_R * v / v.norm(dim=1, keepdim=True), link])
        n = pos.shape[0]
        types = torch.zeros(n, dtype=torch.long)
        types[NF:NF + POCKET] = torch.randint(0, 3, (POCKET,), generator=g)
        frag_only = torch.zeros(n); frag_only[:NF] = 1.0
        pocket_mask = torch.zeros(n); pocket_mask[NF:NF + POCKET] = 1.0
        linker_mask = torch.zeros(n); linker_mask[NF + POCKET:] = 1.0
        anchors = torch.zeros(n); anchors[[0, NF - 1]] = 1.0
        items.append({'uuid': b, 'name': f'clash_{b}', 'positions': pos,
                      'one_hot': torch.nn.functional.one_hot(types, 9).float(), 'anchors': anchors,
                      'fragment_mask': frag_only + pocket_mask, 'linker_mask': linker_mask, 'num_atoms': n,
                      'fragment_only_mask': frag_only, 'pocket_mask': pocket_mask})
    return items


def build(graph, impl, rows=len(SEEDS)):
    d = tcr.dev()
    spec = synthetic.WorkloadSpec("clash_pocket", B=rows, N=NF + POCKET + 2, n_min=NF + POCKET + 1, l_min=1, l_max=2, F=9,
                                  L=2, T=10, seed=0, pocket=POCKET, graph_type=graph)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, diffusion_noise_precision=tcr.NOISE_PRECISION["pocket_4A"])
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(tcr.COORD_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(pocket_items(rows)).items()}
    return ddpm, sampler_inputs(ddpm, data), data


def oracle_rows(ddpm, kw, chain0):
    """(B,) clash-free of a returned chain[0], by the host oracle and by molecule_builder.clash_free (which must agree)."""
    B, N = chain0.shape[:2]
    nm, lm, po = kw['node_mask'].reshape(B, N), kw['linker_mask'].reshape(B, N), kw['context'][..., -1].reshape(B, N)
    _, want = oracle_batch(chain0, nm, lm, po, ddpm.edm.is_geom)
    got = mb.clash_free(chain0, nm, lm, po, ddpm.edm.is_geom).cpu()
    assert torch.equal(got, want)
    return want


def launches(ddpm):
    return int(_native.load_library().dl_launch_count(ddpm.edm.dynamics.engine(0)))


@pytest.mark.gpu
@pytest.mark.parametrize("graph,impl", CASES)
def test_rounds_resample_only_the_molecules_that_clash(graph, impl):
    ddpm, kw, _ = build(graph, impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    assert edm.last_clash_free is None
    # nan_retries = 0: the check only reports, and the chain is the one sampled without it
    r0 = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_clash_free=True)
    ok0 = edm.last_clash_free
    assert torch.equal(r0, base) and ok0.dtype == torch.bool and ok0.shape == (B,)
    assert torch.equal(ok0, oracle_rows(ddpm, kw, base[0]))
    assert edm.last_attempts.tolist() == [0] * B and torch.equal(edm.last_seeds, seeds_tensor(SEEDS, B))
    runs = []
    for r in range(ROUNDS + 1):
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=r, require_clash_free=True)
        runs.append((chain, edm.last_clash_free, edm.last_attempts, edm.last_seeds))
        assert torch.equal(edm.last_clash_free, oracle_rows(ddpm, kw, chain[0])), r
    chain, good, attempts, used = runs[-1]
    assert torch.isfinite(chain).all()
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
    healthy = ok0.nonzero().flatten().tolist()
    assert 0 < len(healthy) < B, healthy                                 # some rows clash at round 0, some do not
    assert torch.equal(chain[:, healthy], base[:, healthy]) and all(int(attempts[b]) == 0 for b in healthy)
    first = [int(attempts[b]) if good[b] else None for b in range(B)]
    recovered = [b for b in range(B) if first[b] is not None and first[b] > 0]
    assert recovered, first
    counts = []
    for r, (c_r, good_r, att_r, _) in enumerate(runs):
        counts.append(int(good_r.sum()))
        for b in range(B):
            want_att = first[b] if first[b] is not None and first[b] <= r else (r if not ok0[b] else 0)
            assert int(att_r[b]) == want_att, (r, b)
            if first[b] is not None and first[b] <= r:
                assert bool(good_r[b]) and torch.equal(c_r[:, b], chain[:, b]), (r, b)
    assert counts == sorted(counts) and counts[-1] > counts[0], counts
    for b in range(B):                                                   # a resampled row is its molecule sampled alone
        if int(attempts[b]) > 0:
            alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert tcr.same(chain[:, b], alone[:, 0], impl), b
    print(f"{graph}/{impl}: clash-free {int(ok0.sum())} of {B} at round 0; after rounds 0..{ROUNDS}: {counts}; "
          f"recovered rows {recovered} (rounds {[first[b] for b in recovered]})")


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_every_combination_of_checks_reports_what_each_check_reports_alone(impl):
    """Each of the seven instantiations, through the sampler's report-only call: the bits equal the standalone checks on
    the returned chain[0], and the clash check adds no launch to the connectivity check."""
    ddpm, kw, _ = build("4A", impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    N = base.shape[2]
    nm, lm, po = kw['node_mask'].reshape(B, N), kw['linker_mask'].reshape(B, N), kw['context'][..., -1].reshape(B, N)
    want = {'require_connected': mb.connected(base[0], nm, True, po).cpu(),
            'require_valid': mb.valence_ok(base[0], nm, True, po).cpu(),
            'require_clash_free': mb.clash_free(base[0], nm, lm, po, True).cpu()}
    got_attr = {'require_connected': 'last_connected', 'require_valid': 'last_valid', 'require_clash_free': 'last_clash_free'}
    for mask in range(1, 8):
        flags = {k: True for i, k in enumerate(want) if mask >> i & 1}
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, **flags)
        assert torch.equal(chain, base), flags
        for k, attr in got_attr.items():
            v = getattr(edm, attr)
            assert (v is None) == (k not in flags) and (v is None or torch.equal(v, want[k])), (flags, k)
    n0 = launches(ddpm)
    edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_connected=True)
    conn = launches(ddpm) - n0
    n0 = launches(ddpm)
    edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_connected=True, require_clash_free=True)
    assert launches(ddpm) - n0 == conn


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_a_split_and_sample_many_resample_what_the_plain_call_resamples(impl):
    ddpm, kw, data = build("4A", impl)
    edm = ddpm.edm
    opts = dict(keep_frames=2, nan_retries=ROUNDS, require_clash_free=True, require_connected=True)
    want = edm.sample_chain(**kw, seeds=SEEDS, **opts)
    ok, attempts, used = edm.last_clash_free, edm.last_attempts, edm.last_seeds
    edm.devices = [0, 0]
    try:
        got = edm.sample_chain(**kw, seeds=SEEDS, **opts)
    finally:
        edm.devices = None
    assert torch.equal(edm.last_clash_free, ok) and torch.equal(edm.last_attempts, attempts)
    assert torch.equal(edm.last_seeds, used) and tcr.same(got, want, impl)
    cuts = [(0, 10), (10, len(SEEDS))]
    reqs = [tcr.take(kw, list(range(lo, hi))) for lo, hi in cuts]
    outs = edm.sample_many(reqs, seeds=[SEEDS[lo:hi] for lo, hi in cuts], **opts)
    for k, (lo, hi) in enumerate(cuts):
        alone = edm.sample_chain(**reqs[k], seeds=SEEDS[lo:hi], **opts)
        assert tcr.same(outs[k], alone, impl), k
        assert torch.equal(edm.last_clash_free_many[k], edm.last_clash_free)
        assert torch.equal(edm.last_attempts_many[k], edm.last_attempts)
        assert torch.equal(edm.last_clash_free, ok[lo:hi]) and torch.equal(edm.last_attempts, attempts[lo:hi])
    # the attribute and DDPM opt in as for the other checks
    edm.nan_retries, edm.require_clash_free, edm.require_connected = ROUNDS, True, True
    chain, _ = ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS)
    assert tcr.same(chain, want, impl) and torch.equal(edm.last_clash_free, ok)
    ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS, require_clash_free=False, require_connected=False, nan_retries=0)
    assert edm.last_clash_free is None
