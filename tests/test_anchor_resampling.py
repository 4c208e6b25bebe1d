"""Anchors in the recovery rounds: `sample_chain(..., require_anchors=True, anchors=...)`, and dl_sample_chain_retry,
dl_set_anchors and dl_anchor_check with DL_CHECK_ANCHORS.

The bit holds when the linker bonds to each anchor by exactly one bond and to no other fragment atom (stated at
DL_CHECK_ANCHORS in the header); anchor_oracle restates it in Python over the bonds of build_xae_molecule's arithmetic. CPU
tests pin the oracle to purpose-built molecules, and check the refusals, the binding and the header; the GPU tests check
the kernel against the oracle, on those molecules and on sampled batches, and the sampler end to end."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, distributed, molecule_builder as mb
from difflinker_b200.edm import retry_seed
from difflinker_b200.utils import FoundNaNException
from oracle import bond_rounding as br
import anchor_oracle as ao
import dl_helpers as helpers
import ring_oracle as ro
import test_connected_resampling as tcr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANCHORS = 64
FAR = 60.0                                  # A: padding rows, out of every bond's reach
D = 1.5                                     # A: a C-C single bond; 2 D and more is no bond


def line(xs, y=0.0):
    return [[x, y, 0.0] for x in xs]


def molecules():
    """(name, positions (n,3), linker flags, anchor flags, pocket flags, bonds, expected verdict, expected a (n,)); every
    atom is carbon. The pocket flag drops a row as the pocket's."""
    mols = []

    def add(name, pos, linker, anchor, bonds, want, att, pocket=None):
        n = len(pos)
        mols.append((name, np.asarray(pos, np.float32), np.asarray(linker, bool), np.asarray(anchor, bool),
                     np.zeros(n, bool) if pocket is None else np.asarray(pocket, bool), bonds, want,
                     np.asarray(att, np.int64)))
    # fragment 0-1, linker 4-5, fragment 2-3 on one line: 0 - 1 - 4 - 5 - 2 - 3
    chain = line([0, D, 4 * D, 5 * D, 2 * D, 3 * D])
    chain_bonds = {(0, 1), (1, 4), (4, 5), (2, 5), (2, 3)}
    lk = [0, 0, 0, 0, 1, 1]
    add("two fragments joined at their anchors", chain, lk, [0, 1, 1, 0, 0, 0], chain_bonds, True, [0, 1, 1, 0, 0, 0])
    add("the linker bonded to an anchor's neighbour", chain, lk, [1, 0, 1, 0, 0, 0], chain_bonds, False,
        [0, 1, 1, 0, 0, 0])
    add("an anchor with two linker bonds", [[0, 0, 0], [-D, 0, 0], [0, D, 0], [0, -D, 0]], [0, 0, 1, 1], [1, 0, 0, 0],
        {(0, 1), (0, 2), (0, 3)}, False, [2, 0, 0, 0])
    free = line([0, D, 7 * D, 8 * D, 2 * D, 3 * D])
    add("one anchor left free", free, lk, [0, 1, 1, 0, 0, 0], {(0, 1), (1, 4), (4, 5), (2, 3)}, False,
        [0, 1, 0, 0, 0, 0])
    # one linker atom L between two anchors 2.6 A apart
    both = [[-D, 0, 0], [0, 0, 0], [2.6, 0, 0], [2.6 + D, 0, 0], [1.3, 0.75, 0]]
    add("a linker atom bonded to both anchors", both, [0, 0, 0, 0, 1], [0, 1, 1, 0, 0], {(0, 1), (1, 4), (2, 4), (2, 3)},
        True, [0, 1, 1, 0, 0])
    # the same anchors and L, and a bond between the two fragments (atoms 0 and 3)
    ff = [[0.55, -1.4, 0], [0, 0, 0], [2.6, 0, 0], [2.05, -1.4, 0], [1.3, 0.75, 0]]
    add("a fragment-fragment bond does not count", ff, [0, 0, 0, 0, 1], [0, 1, 1, 0, 0],
        {(0, 1), (0, 3), (1, 4), (2, 4), (2, 3)}, True, [0, 1, 1, 0, 0])
    # the joined chain, and a pocket atom within bond distance of anchor 1 and linker atom 4
    add("pocket atoms near an anchor do not count", chain + [[1.5 * D, 1.3, 0]], lk + [0], [0, 1, 1, 0, 0, 0, 0],
        chain_bonds, True, [0, 1, 1, 0, 0, 0, 0], pocket=[0, 0, 0, 0, 0, 0, 1])
    add("no anchors", chain, lk, [0] * 6, chain_bonds, True, [0, 1, 1, 0, 0, 0])
    # anchor flags on a linker row are ignored
    add("a flag on a linker row is ignored", chain, lk, [0, 1, 1, 0, 1, 0], chain_bonds, True, [0, 1, 1, 0, 0, 0])
    nan = np.array(chain, np.float32)
    nan[4] = np.nan                         # the linker atom next to anchor 1 is bonded to nothing
    add("a NaN linker atom", nan, lk, [0, 1, 1, 0, 0, 0], {(0, 1), (2, 5), (2, 3)}, False, [0, 0, 1, 0, 0, 0])
    return mols


def pack(mols, N, F=8):
    """A padded (B,N,3+F) carbon batch of the molecules, with node, linker, anchor and pocket masks."""
    B = len(mols)
    xh = torch.zeros(B, N, 3 + F)
    xh[:, :, :3] = FAR
    xh[:, :, 3] = 1.0
    nm, lm = torch.zeros(B, N, dtype=torch.int8), torch.zeros(B, N)
    an, po = torch.zeros(B, N, dtype=torch.int8), torch.zeros(B, N)
    for b, (_, pos, linker, anchor, pocket, *_) in enumerate(mols):
        n = pos.shape[0]
        xh[b, :n, :3] = torch.from_numpy(pos)
        nm[b, :n] = 1
        lm[b, :n] = torch.from_numpy(linker.astype(np.float32))
        an[b, :n] = torch.from_numpy(anchor.astype(np.int8))
        po[b, :n] = torch.from_numpy(pocket.astype(np.float32))
    return xh, nm, lm, an, po


def straddling_molecules():
    """26-atom chains (oracle.bond_rounding.twins) whose only linker-fragment pair (j, i) straddles a single-bond threshold
    of carbon: bonded in one of the two distance forms and not in the other. Rows [0, j] are fragment, j the anchor; rows
    [i, 26) are linker. Over 26 atoms the pair is measured in the matmul form: (xh (1, 32, 11) padded with far carbon rows,
    node mask, linker, anchor, bonded over 26 atoms, bonded in the direct form)."""
    thr = [t.numpy() for t in mb.threshold_tables(False)]
    out = []
    for _, x26, _, t26, j, i in br.twins(thr):
        n = len(x26)
        xh = torch.zeros(1, 32, 11)
        xh[0, :, :3] = FAR
        xh[0, :, 3] = 1.0
        xh[0, :n, :3] = torch.from_numpy(x26)
        xh[0, :n, 3:] = torch.nn.functional.one_hot(torch.from_numpy(t26), 8).float()
        nm = torch.zeros(1, 32, dtype=torch.int8)
        nm[0, :n] = 1
        linker = torch.zeros(1, 32)
        linker[0, i:n] = 1.0
        anchor = torch.zeros(1, 32, dtype=torch.int8)
        anchor[0, j] = 1
        t = thr[0][min(t26[i], t26[j])][max(t26[i], t26[j])]
        b26 = bool(br.bond_orders(x26, t26, thr)[i, j] > 0)
        b_direct = bool(br.direct_dist_pm(x26[i][None], x26[j][None])[0] < t)
        out.append((xh, nm, linker, anchor, b26, b_direct))
    return out


# ---- CPU --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", [m[0] for m in molecules()])
def test_oracle_on_purpose_built_molecules(name):
    """The oracle's bond graph is the intended one, then its verdict and attachments are the intended ones."""
    mol, = [m for m in molecules() if m[0] == name]
    _, pos, linker, anchor, pocket, bonds, want, att = mol
    rows = np.nonzero(~pocket)[0]
    adj = ro.bonds(pos[rows], np.zeros(len(rows), int), False)
    got = {(int(rows[i]), int(rows[j])) for i, j in zip(*np.nonzero(np.triu(adj)))}
    assert got == bonds, name
    xh, nm, lm, an, po = pack([mol], N=12)
    ok, a = ao.batch(xh, nm, lm, an, False, po)
    assert ok == [want] and a[0, :len(pos)].tolist() == att.tolist(), name
    if pocket.any():                        # counted as a fragment atom, the pocket atom would attach to the linker
        assert ao.batch(xh, nm, lm, an, False, None)[0] == [False]


def test_a_pair_the_two_distance_forms_decide_differently_is_measured_over_all_checked_atoms():
    mols = straddling_molecules()
    assert len(mols) >= 2 and all(b26 != bd for *_, b26, bd in mols) and {b26 for *_, b26, _ in mols} == {True, False}
    for xh, nm, linker, anchor, b26, _ in mols:
        ok, a = ao.batch(xh, nm, linker, anchor, False)
        j = int(anchor[0].nonzero()[0])
        assert ok == [b26] and int(a[0, j]) == int(b26) and int(a[0].sum()) == int(b26)


@pytest.mark.parametrize("inpainting", [False, True])
def test_require_anchors_refuses_what_cannot_recover_and_names_what_is_wrong(inpainting):
    ddpm, kw = tcr._cpu_model(inpainting)
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    seeds = list(range(1, B + 1))
    assert edm.require_anchors is False and edm.last_anchors_ok is None and edm.last_anchors_ok_many is None
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_anchors"):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_anchors=bad)
    with pytest.raises(ValueError, match="require_anchors needs per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2, require_anchors=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_anchors=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="require_anchors does not take batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_anchors=True, seeds=seeds, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_anchors needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_anchors=True, seeds=seeds)
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="require_anchors.*replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_anchors=True, seeds=seeds)
    delattr(edm, name)
    with pytest.raises(ValueError, match="sample_many needs CUDA inputs"):
        edm.sample_many([kw], keep_frames=2, seeds=[seeds], require_anchors=True)
    edm.require_anchors = True                                           # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    assert edm.last_anchors_ok is None


def test_the_anchor_flags_are_vetted_before_sampling():
    """_anchors, the vetting sample_chain and sample_many run before they sample: what it refuses, and what it returns."""
    ddpm, kw = tcr._cpu_model()
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    lm, nm = kw['linker_mask'].reshape(B, N), kw['node_mask'].reshape(B, N)
    frag = (nm != 0) & (lm == 0)
    good = torch.zeros(B, N)
    for b in range(B):
        good[b, int(frag[b].nonzero()[0])] = 1.0
    vet = lambda a, check=ANCHORS: edm._anchors(check, a, kw['x'], kw['node_mask'], kw['linker_mask'], kw['context'])
    assert vet(None, 0) is None and vet("not read", 0) is None          # without the bit nothing is read
    with pytest.raises(ValueError, match="require_anchors needs the anchor flags: pass anchors="):
        vet(None)
    for shape in ((B, N + 1), (B - 1, N), (B, N, 2)):
        with pytest.raises(ValueError, match=r"\(B, N\) or \(B, N, 1\)"):
            vet(torch.zeros(shape))
    on_linker = good.clone()
    b = 1
    on_linker[b, int(lm[b].nonzero()[0])] = 1.0
    with pytest.raises(ValueError, match=f"molecule {b} has an anchor flag on a linker row"):
        vet(on_linker)
    none = good.clone()
    none[2] = 0.0
    with pytest.raises(ValueError, match="molecule 2 has no anchor atom.*--anchors"):
        vet(none)
    got = vet(good[:, :, None])
    assert got.dtype == torch.int8 and got.shape == (B, N) and torch.equal(got, (good != 0).to(torch.int8))


def test_a_flag_on_a_pocket_row_is_refused():
    ddpm, kw = tcr._cpu_model()
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    ctx = torch.zeros(B, N, 2)
    ctx[0, 0, -1] = 1.0                      # row 0 of molecule 0 is a pocket row
    an = torch.zeros(B, N)
    an[:, 0] = 1.0
    edm.dynamics.graph_type = '4A'
    try:
        with pytest.raises(ValueError, match="molecule 0 has an anchor flag on a pocket row"):
            edm._anchors(ANCHORS, an, kw['x'], kw['node_mask'], kw['linker_mask'], ctx)
    finally:
        edm.dynamics.graph_type = 'FC'


def test_ddpm_and_the_sharded_sampler_pass_the_template_anchors():
    ddpm, _ = tcr._cpu_model()
    from difflinker_b200 import ddpm as ddpm_mod, synthetic
    from difflinker_b200.batching import collate
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append((k.get('require_anchors', 'unset'), k.get('anchors')))
    ddpm.edm.sample_many = lambda reqs, **k: seen.append((k.get('require_anchors', 'unset'),
                                                          [r.get('anchors') for r in reqs])) or [None] * len(reqs)
    ddpm.sample_chain(data, keep_frames=2, require_anchors=True)
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, require_anchors=False)
    ddpm.sample_many([data], keep_frames=2, seeds=[[1, 2, 3]], require_anchors=True)
    distributed.sample_chain_sharded(ddpm, data, keep_frames=2, seeds=[1, 2, 3], require_anchors=True)
    ddpm.edm.require_anchors = True                                      # the attribute alone also passes them
    ddpm.sample_chain(data, keep_frames=2)
    assert [s[0] for s in seen] == [True, 'unset', False, True, True, 'unset']
    assert seen[1][1] is None and seen[2][1] is None
    B, n_old = data['anchors'].shape[:2]
    n_frag = data['fragment_mask'].reshape(B, -1).sum(1).long()
    for got in (seen[0][1], seen[3][1][0], seen[4][1], seen[5][1]):
        n = got.shape[1]
        for b in range(B):
            f = int(n_frag[b])
            assert torch.equal(got[b, :f], data['anchors'].reshape(B, n_old)[b, :f]) and not got[b, f:].any()


def test_template_anchors_follow_the_fragment_rows_at_any_padding():
    from difflinker_b200 import ddpm as ddpm_mod, synthetic
    from difflinker_b200.batching import collate, create_templates_for_linker_generation
    ddpm, _ = tcr._cpu_model()
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=4))
    B = data['anchors'].shape[0]
    sizes = torch.tensor([3, 5, 2, 6])
    for n in (None, 40):
        t = create_templates_for_linker_generation(data, sizes, n)
        n_rows = t['anchors'].shape[1]
        assert torch.equal(ddpm_mod.template_anchors(ddpm, data, n_rows), t['anchors'].reshape(B, n_rows))


def test_binding_and_a_c99_caller_get_the_new_entries_and_refusals(tmp_path):
    lib = _native.load_library()
    assert _native.CHECK_ANCHORS == ANCHORS
    for name in ("dl_anchor_check", "dl_set_anchors"):
        assert name in _native.SYMBOLS and getattr(lib, name).argtypes == _native.SYMBOLS[name][1]
    assert lib.dl_set_anchors(None, 2, 4, 1, None) == -1 and b"null engine" in lib.dl_last_error()
    for args, why in (((0, 4, 8, 1, 1, 11, 1, 1, 1, None, 0, 0, 1, None, None), b"B and N"),
                      ((1, 8193, 8, 1, 1, 11, 1, 1, 1, None, 0, 0, 1, None, None), b"8192"),
                      ((1, 4, 9, 1, 1, 11, 1, 1, 1, None, 0, 0, 1, None, None), b"n_types"),
                      ((1, 4, 8, None, 1, 11, 1, 1, 1, None, 0, 0, 1, None, None), b"invalid argument"),
                      ((1, 4, 8, 1, 1, 11, 1, 1, None, None, 0, 0, 1, None, None), b"invalid argument"),
                      ((1, 4, 8, 1, 1, 11, 1, 1, 1, None, 0, 1, 1, None, None), b"invalid argument")):
        assert lib.dl_anchor_check(*args) == -1, why
        assert why in lib.dl_last_error() and b"dl_anchor_check" in lib.dl_last_error()
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "anchor_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2]; int32_t attempts[2], flags[2], passed[2], att[8];\n"
        "  float thr[64] = {0}, xh[22] = {0}; int8_t nm[8] = {0}, an[8] = {0};\n"
        "  dl_molecule_checks ck = {DL_CHECK_CONNECTED | DL_CHECK_ANCHORS, 8, thr, thr, thr, NULL, NULL};\n"
        "  dl_status a = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                      NULL, NULL, NULL, NULL, flags, 3, used, attempts, &ck, passed, NULL, NULL,\n"
        "                                      NULL);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  dl_status b = dl_anchor_check(2, 4, 8, thr, xh, 11, nm, thr, NULL, NULL, 0, 0, passed, att, NULL);\n"
        '  printf("%d|%s|", (int)b, dl_last_error());\n'
        "  ck.require = DL_CHECK_ANCHORS;\n"
        "  dl_status c = dl_molecule_check(2, 4, &ck, xh, 11, nm, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s|", (int)c, dl_last_error());\n'
        "  ck.require = DL_CHECK_NOVEL | DL_CHECK_ANCHORS;\n"
        "  dl_status d = dl_novel_check(2, 4, &ck, NULL, xh, 11, nm, thr, NULL, 0, 0, passed, used, NULL, NULL);\n"
        '  printf("%d|%s|", (int)d, dl_last_error());\n'
        "  dl_status e = dl_set_anchors(NULL, 2, 4, an, NULL);\n"
        '  printf("%d|%s|", (int)e, dl_last_error());\n'
        "  ck.require = DL_CHECK_CONNECTED | 128;\n"
        "  dl_status f = dl_molecule_check(2, 4, &ck, xh, 11, nm, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)f, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "anchor_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe),
                    _native.LIB_PATH, f"-Wl,-rpath,{os.path.dirname(_native.LIB_PATH)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, err_a, b, err_b, c, err_c, d, err_d, e, err_e, f, err_f = res.stdout.strip().split("|", 11)
    assert int(a) == -1 and "null engine" in err_a
    assert int(b) == -1 and "dl_anchor_check" in err_b and "invalid argument" in err_b
    assert int(c) == -1 and "require" in err_c and "dl_anchor_check" in err_c
    assert int(d) == -1 and "dl_novel_check" in err_d and "dl_anchor_check" in err_d
    assert int(e) == -1 and "null engine" in err_e
    assert int(f) == -1 and "require" in err_f


# ---- GPU: the kernel, molecule by molecule ------------------------------------------------------------------------------

def kernel_check(xh, nm, lm, an, po, is_geom):
    """(passed bools, attachments (B, N) int64) of dl_anchor_check on the device."""
    d = tcr.dev()
    pocket = None if po is None else po.to(d)
    ok = mb.anchors_ok(xh.to(d), nm.to(d), lm.to(d), an.to(d), is_geom, pocket)
    att = mb.attachments(xh.to(d), nm.to(d), lm.to(d), is_geom, pocket)
    assert att.dtype == torch.int32 and ok.dtype == torch.bool
    return ok.cpu().tolist(), att.cpu().long().numpy()


def assert_matches_oracle(xh, nm, lm, an, po, is_geom):
    want_ok, want_att = ao.batch(xh, nm, lm, an, is_geom, po)
    got_ok, got_att = kernel_check(xh, nm, lm, an, po, is_geom)
    assert got_ok == want_ok
    assert np.array_equal(got_att, want_att)
    return want_ok, want_att


@pytest.mark.gpu
def test_kernel_matches_the_oracle_on_purpose_built_molecules():
    mols = molecules()
    xh, nm, lm, an, po = pack(mols, N=12)
    ok, att = assert_matches_oracle(xh, nm, lm, an, po, False)
    assert ok == [m[6] for m in mols]
    for b, m in enumerate(mols):
        assert att[b, :len(m[1])].tolist() == m[7].tolist(), m[0]
    # counted as atoms, the pocket atom attaches to the linker and fails the molecule
    i = [m[0] for m in mols].index("pocket atoms near an anchor do not count")
    assert kernel_check(xh[i:i + 1], nm[i:i + 1], lm[i:i + 1], an[i:i + 1], None, False)[0] == [False]


@pytest.mark.gpu
def test_kernel_measures_a_straddling_pair_over_all_checked_atoms():
    mols = straddling_molecules()
    xh, nm, lm, an = (torch.cat([m[k] for m in mols]) for k in range(4))
    ok, _ = assert_matches_oracle(xh, nm, lm, an, None, False)
    assert ok == [m[4] for m in mols]


@pytest.mark.gpu
def test_the_check_holds_up_to_the_checks_row_limit():
    """N = 8192: the joined chain in rows spread over the batch, a clump of 200 mutually bonded atoms (fragment and
    linker), the rest padding."""
    N = 8192
    xh = torch.zeros(1, N, 11)
    xh[:, :, :3] = FAR
    xh[:, :, 3] = 1.0
    nm, lm, an = torch.zeros(1, N, dtype=torch.int8), torch.zeros(1, N), torch.zeros(1, N, dtype=torch.int8)
    (_, pos, linker, anchor, *_), = [m for m in molecules() if m[0] == "two fragments joined at their anchors"]
    rows = torch.tensor([7, 900, 3000, 5000, 6001, 8190])
    xh[0, rows, :3] = torch.from_numpy(pos)
    nm[0, rows] = 1
    lm[0, rows] = torch.from_numpy(linker.astype(np.float32))
    an[0, rows] = torch.from_numpy(anchor.astype(np.int8))
    g = torch.Generator().manual_seed(5)
    clump = torch.arange(1000, 1200)
    xh[0, clump, :3] = 30.0 + 0.7 * torch.rand(200, 3, generator=g)
    nm[0, clump] = 1
    lm[0, clump[150:]] = 1.0
    an[0, clump[:3]] = 1
    ok, att = assert_matches_oracle(xh, nm, lm, an, None, False)
    assert ok == [False] and att[0, rows[1]] == 1 and att[0, clump[:150]].sum() > 150
    lm[0, clump] = 0.0                      # the clump is all fragment: the chain alone attaches
    an[0, clump] = 0
    ok, _ = assert_matches_oracle(xh, nm, lm, an, None, False)
    assert ok == [True]


def sampled(case, impl, rows=16):
    ddpm, kw = tcr.build(case, impl, rows=rows)
    edm = ddpm.edm
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=list(range(1, rows + 1)))
    po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
    return ddpm, kw, chain[0], po


def some_anchors(kw, chain0, is_geom, po):
    """(B, N) anchor flags that let some rows pass and fail others: on even rows, the fragment atoms the sampled linker
    bonds to; on odd rows, and on rows whose linker bonds to no fragment atom, the first fragment atom."""
    B, N = kw['x'].shape[:2]
    _, att = ao.batch(chain0, kw['node_mask'], kw['linker_mask'], torch.zeros(B, N), is_geom, po)
    frag = (kw['node_mask'].reshape(B, N).cpu() != 0) & (kw['linker_mask'].reshape(B, N).cpu() == 0)
    if po is not None:
        frag &= po.reshape(B, N).cpu() == 0
    an = torch.zeros(B, N, dtype=torch.int8)
    for b in range(B):
        hit = np.flatnonzero(att[b] > 0)
        if b % 2 == 0 and hit.size:
            an[b, torch.from_numpy(hit)] = 1
        else:
            an[b, int(frag[b].nonzero()[0])] = 1
    return an.to(kw['x'].device)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fc", "pocket_4A", "fc_inpainting"])
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_kernel_matches_the_oracle_on_sampled_batches(case, impl):
    ddpm, kw, chain0, po = sampled(case, impl)
    an = some_anchors(kw, chain0, ddpm.edm.is_geom, po)
    ok, att = assert_matches_oracle(chain0, kw['node_mask'], kw['linker_mask'], an, po, ddpm.edm.is_geom)
    print(f"{case}/{impl}: {sum(ok)} of {len(ok)} rows pass; attachments per row {att.sum(1).tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_kernel_matches_the_oracle_on_zinc_and_geom_batches(is_geom, impl):
    """Sampled FC batches of the benchmark's ZINC (cfg2_zinc) and GEOM (cfg3_geom) shapes, with the batch's own anchors."""
    from difflinker_b200 import synthetic
    from difflinker_b200.ddpm import sampler_inputs, template_anchors
    from difflinker_b200.batching import collate
    spec = synthetic.SPECS["cfg3_geom" if is_geom else "cfg2_zinc"]
    d = tcr.dev()
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=32)).items()}
    kw = sampler_inputs(ddpm, data)
    try:                                    # the synthetic GEOM model diverges on some rows; NaN pairs are not bonded
        chain = ddpm.edm.sample_chain(**kw, keep_frames=1, seeds=list(range(1, 33)), nan_retries=1)
    except FoundNaNException as e:
        chain = e.chain
    an = template_anchors(ddpm, data, kw['x'].shape[1])
    ok, att = assert_matches_oracle(chain[0], kw['node_mask'], kw['linker_mask'], an, None, ddpm.edm.is_geom)
    print(f"{spec.name}/{impl}: {sum(ok)} of {len(ok)} rows pass; {int((att > 0).sum())} attached fragment atoms")


@pytest.mark.gpu
def test_kernel_matches_the_oracle_on_a_pocket_batch():
    """B = 64, N = 300: the cfg4_pockets batch, ligands among 270 pocket rows, which the check drops."""
    from difflinker_b200 import synthetic
    from difflinker_b200.batching import collate
    spec = synthetic.SPECS["cfg4_pockets"]
    data = collate(synthetic.make_items(spec, batch=64))
    B, N = data['positions'].shape[:2]
    assert (B, N) == (64, 300)
    F = data['one_hot'].shape[-1]
    xh = torch.cat([data['positions'], data['one_hot']], dim=2)
    # the synthetic ligands sit far apart; pull every linker atom onto a bond from a random fragment atom
    g = torch.Generator().manual_seed(11)
    frag = data['fragment_only_mask'].reshape(B, N) != 0
    lm = data['linker_mask'].reshape(B, N)
    for b in range(B):
        f = frag[b].nonzero().flatten()
        for r in (lm[b] != 0).nonzero().flatten().tolist()[:3]:
            u = torch.randn(3, generator=g)
            xh[b, r, :3] = xh[b, f[int(torch.randint(len(f), (1,), generator=g))], :3] + 1.45 * u / u.norm()
    po = data['pocket_mask'].reshape(B, N)
    nm = data['atom_mask'].reshape(B, N)
    an = data['anchors'].reshape(B, N) * frag
    ok, att = assert_matches_oracle(xh, nm, lm, an, po, F == 9)
    print(f"cfg4_pockets: {sum(ok)} of {B} rows pass; {int((att > 0).sum())} attached fragment atoms")


# ---- GPU: the sampler, end to end ---------------------------------------------------------------------------------------

SEEDS = list(range(1, 17))


def oracle_ok(ddpm, kw, chain0, an):
    po = kw['context'][..., -1] if ddpm.edm.dynamics.graph_type != 'FC' else None
    return ao.batch(chain0, kw['node_mask'], kw['linker_mask'], an, ddpm.edm.is_geom, po)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", tcr.CASES)
def test_rounds_resample_only_the_molecules_that_miss_their_anchors(case, impl):
    ddpm, kw = tcr.build(case, impl, rows=len(SEEDS))
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
    an = some_anchors(kw, base[0], edm.is_geom, po)
    r0 = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_anchors=True, anchors=an)
    ok0 = edm.last_anchors_ok
    assert torch.equal(r0, base) and ok0.dtype == torch.bool and ok0.shape == (B,)
    want0 = oracle_ok(ddpm, kw, base[0], an)
    assert ok0.tolist() == want0 and any(want0) and not all(want0)
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=4, require_anchors=True, anchors=an[:, :, None])
    ok, attempts, used = edm.last_anchors_ok, edm.last_attempts, edm.last_seeds
    assert ok.tolist() == oracle_ok(ddpm, kw, chain[0], an)
    pocket = None if po is None else po.to(chain.device)
    assert ok.tolist() == mb.anchors_ok(chain[0], kw['node_mask'], kw['linker_mask'], an, edm.is_geom, pocket).cpu().tolist()
    healthy = [b for b in range(B) if want0[b]]
    assert torch.equal(chain[:, healthy], base[:, healthy]) and all(int(attempts[b]) == 0 for b in healthy)
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
        if int(attempts[b]) > 0:                                         # a resampled row replays alone from its seed
            alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert tcr.same(chain[:, b], alone[:, 0], impl), b
    print(f"{case}/{impl}: {sum(want0)} of {B} rows pass at attempt 0, {int(ok.sum())} after the rounds")


@pytest.mark.gpu
def test_size_redraws_read_each_rows_own_anchor_flags():
    """linker_sizes redraws: the rounds regather the fragment rows in place, so the caller's flags still name them."""
    from difflinker_b200 import ddpm as ddpm_mod
    from difflinker_b200.batching import collate
    d = tcr.dev()
    ddpm, _ = tcr.build("fc", "simt", rows=len(SEEDS))
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(tcr.small_fragment_items("fc", 16)).items()}
    B = len(SEEDS)
    chain, nm = ddpm_mod.sample_chain(ddpm, data, keep_frames=2, seeds=SEEDS, linker_sizes=(1, 2), nan_retries=3,
                                      require_anchors=True)
    edm = ddpm.edm
    n = chain.shape[2]
    lm = (torch.arange(n, device=d)[None, :] >= data['fragment_mask'].reshape(B, -1).sum(1, keepdim=True)) & (nm[..., 0] != 0)
    an = ddpm_mod.template_anchors(ddpm, data, n)
    want = ao.batch(chain[0], nm, lm.float(), an, edm.is_geom)[0]
    ok, attempts, used = edm.last_anchors_ok, edm.last_attempts, edm.last_seeds
    assert ok.tolist() == want
    for b in range(B):
        if int(attempts[b]) > 0:
            alone, _ = ddpm_mod.sample_chain(ddpm, {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in data.items()},
                                             keep_frames=2, seeds=[int(used[b])], linker_sizes=(1, 2))
            k = alone.shape[2]
            assert torch.equal(chain[:, b, :k], alone[:, 0]), b
    print(f"linker_sizes: {int(ok.sum())} of {B} rows pass after the rounds, {int((attempts > 0).sum())} resampled")


@pytest.mark.gpu
@pytest.mark.parametrize("other", ["require_connected", "require_valid", "require_clash_free", "require_unique",
                                   "require_novel", "require_ring_sizes"])
def test_the_bit_combines_with_each_other_check(other):
    case = "pocket_4A" if other == "require_clash_free" else "fc"
    ddpm, kw = tcr.build(case, "simt", rows=len(SEEDS))
    edm = ddpm.edm
    edm.allowed_ring_sizes = [5, 6]
    edm.known_linkers = torch.tensor([], dtype=torch.int64)
    attr = {"require_connected": "last_connected", "require_valid": "last_valid", "require_clash_free": "last_clash_free",
            "require_unique": "last_unique", "require_novel": "last_novel",
            "require_ring_sizes": "last_ring_sizes_ok"}[other]
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, **{other: True})
    other_alone = getattr(edm, attr)
    po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
    an = some_anchors(kw, base[0], edm.is_geom, po)
    alone_bits = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_anchors=True, anchors=an)
    anchors_alone = edm.last_anchors_ok
    both = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_anchors=True, anchors=an, **{other: True})
    assert torch.equal(both, base) and torch.equal(both, alone_bits)
    assert torch.equal(edm.last_anchors_ok, anchors_alone)
    if other != "require_unique":           # the uniqueness verdict counts the other required bits, so it may change
        assert torch.equal(getattr(edm, attr), other_alone)
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=3, require_anchors=True, anchors=an,
                             **{other: True})
    assert edm.last_anchors_ok.tolist() == oracle_ok(ddpm, kw, chain[0], an)


@pytest.mark.gpu
def test_a_row_that_misses_its_anchors_does_not_block_a_later_duplicate():
    """Rows 0 and 1 are one molecule sampled with one seed; row 0's anchors fail it, row 1's pass it. The uniqueness
    verdict, which runs after the anchor check, counts only eligible earlier rows, so row 1 is unique."""
    ddpm, kw = tcr.build("fc", "simt", rows=len(SEEDS))
    edm = ddpm.edm
    pair = tcr.take(kw, [2, 2])             # a molecule with two linker atoms
    N = pair['x'].shape[1]
    frag = (pair['node_mask'].reshape(2, N)[0] != 0) & (pair['linker_mask'].reshape(2, N)[0] == 0)
    for seed in range(1, 65):               # a seed whose linker attaches by single bonds
        base = edm.sample_chain(**pair, keep_frames=2, seeds=[seed, seed])
        _, att = ao.batch(base[0, :1], pair['node_mask'][:1], pair['linker_mask'][:1], torch.zeros(1, N), edm.is_geom)
        if att.max() == 1:
            break
    assert att.max() == 1 and torch.equal(base[:, 0], base[:, 1])
    good = torch.from_numpy(att[0] == 1).to(torch.int8)
    bad = torch.zeros(N, dtype=torch.int8)
    bad[int((frag.cpu() & torch.from_numpy(att[0] == 0)).nonzero()[0])] = 1   # a fragment atom the linker does not bond to
    an = torch.stack([bad, good]).to(pair['x'].device)
    edm.sample_chain(**pair, keep_frames=2, seeds=[seed, seed], nan_retries=0, require_anchors=True, require_unique=True,
                     anchors=an)
    assert edm.last_anchors_ok.tolist() == [False, True]
    assert edm.last_unique.tolist() == [True, True]
    edm.sample_chain(**pair, keep_frames=2, seeds=[seed, seed], nan_retries=0, require_unique=True)
    assert edm.last_unique.tolist() == [True, False]                     # without the bit, row 1 repeats row 0


@pytest.mark.gpu
def test_a_split_and_sample_many_return_what_the_plain_call_returns():
    ddpm, kw = tcr.build("fc", "simt", rows=len(SEEDS))
    edm = ddpm.edm
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    an = some_anchors(kw, base[0], edm.is_geom, None)
    want = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=3, require_anchors=True, anchors=an)
    ok, used = edm.last_anchors_ok, edm.last_seeds
    edm.devices = [0, 0]
    got = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=3, require_anchors=True, anchors=an)
    assert torch.equal(got, want) and torch.equal(edm.last_anchors_ok, ok) and torch.equal(edm.last_seeds, used)
    edm.devices = None
    idx = [list(range(8)), list(range(8, 16))]
    halves = [dict(tcr.take(kw, ix), anchors=an[ix]) for ix in idx]
    seeds = [SEEDS[:8], SEEDS[8:]]
    res = edm.sample_many(halves, keep_frames=2, seeds=seeds, nan_retries=3, require_anchors=True)
    ok_many = edm.last_anchors_ok_many
    for k in range(2):
        plain = {n: v for n, v in halves[k].items() if n != 'anchors'}
        alone = edm.sample_chain(**plain, keep_frames=2, seeds=seeds[k], nan_retries=3, require_anchors=True,
                                 anchors=halves[k]['anchors'])
        assert torch.equal(res[k], alone) and torch.equal(ok_many[k], edm.last_anchors_ok)


@pytest.mark.gpu
def test_ddpm_picks_up_the_batchs_anchors():
    from difflinker_b200 import ddpm as ddpm_mod
    from difflinker_b200.batching import collate
    d = tcr.dev()
    ddpm, kw = tcr.build("fc", "simt", rows=len(SEEDS))
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(tcr.small_fragment_items("fc", 16)).items()}
    has_linker = [b for b in range(len(SEEDS)) if b % 3]                  # a molecule without a linker has no bond to judge
    data = {k: (v[has_linker] if torch.is_tensor(v) else v) for k, v in data.items()}
    seeds = [SEEDS[b] for b in has_linker]
    chain, nm = ddpm.sample_chain(data, keep_frames=2, seeds=seeds, nan_retries=2, require_anchors=True)
    an = ddpm_mod.template_anchors(ddpm, data, chain.shape[2])
    kw = ddpm_mod.sampler_inputs(ddpm, data)
    want = ao.batch(chain[0], kw['node_mask'], kw['linker_mask'], an, ddpm.edm.is_geom)[0]
    assert ddpm.edm.last_anchors_ok.tolist() == want


@pytest.mark.gpu
def test_the_engine_reads_the_flags_once_and_refuses_a_call_without_them():
    ddpm, kw = tcr.build("fc", "simt", rows=4)
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3, 4])
    an = some_anchors(kw, base[0], edm.is_geom, None)
    edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3, 4], require_anchors=True, anchors=an)
    # the flags were cleared by that call: a retry call that requires the bit without setting them is refused
    t = edm._sampler_tensors(**kw)          # alive while the calls below read it
    head = edm._head(4, kw['x'].shape[1], 2, t)
    assert lib.dl_set_anchors(eng, 0, 4, an.data_ptr(), None) == -1 and b"B and N" in lib.dl_last_error()
    assert lib.dl_set_anchors(eng, 4, 4, None, None) == -1 and b"null anchors" in lib.dl_last_error()
    from difflinker_b200.edm import _sample_slice
    out = torch.empty((2,) + tuple(base.shape[1:]), device=base.device)
    flags = torch.zeros(4, dtype=torch.int32, device=base.device)
    used = torch.empty(4, dtype=torch.int64, device=base.device)
    attempts = torch.empty(4, dtype=torch.int32, device=base.device)
    passed = torch.empty(4, dtype=torch.int32, device=base.device)
    seeds = torch.tensor([1, 2, 3, 4], dtype=torch.int64, device=base.device)
    tables = [t.to(base.device) for t in edm._check_tables(ANCHORS)]
    stream = torch.cuda.current_stream().cuda_stream
    tail = (edm.step_coefficients(2, 4), edm._norm(), out.data_ptr(), flags.data_ptr())
    with pytest.raises(Exception, match="dl_set_anchors"):
        _sample_slice(lib, eng, head, tail, stream, seeds=seeds,
                      retry=(0, used, attempts, ANCHORS, (tables, None), passed, None, None, None, None, None))
    bad = torch.zeros(4, kw['x'].shape[1] + 1, dtype=torch.int8, device=base.device)
    assert lib.dl_set_anchors(eng, 4, kw['x'].shape[1] + 1, bad.data_ptr(), stream) == 0
    with pytest.raises(Exception, match="another B or N"):
        _sample_slice(lib, eng, head, tail, stream, seeds=seeds,
                      retry=(0, used, attempts, ANCHORS, (tables, None), passed, None, None, None, None, None))
    # a call that does not require the bit clears them too
    assert lib.dl_set_anchors(eng, 4, kw['x'].shape[1], an.data_ptr(), stream) == 0
    edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3, 4], require_connected=True)
    with pytest.raises(Exception, match="dl_set_anchors"):
        _sample_slice(lib, eng, head, tail, stream, seeds=seeds,
                      retry=(0, used, attempts, ANCHORS, (tables, None), passed, None, None, None, None, None))
    torch.cuda.synchronize()
