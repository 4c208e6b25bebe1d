"""Valence in the recovery rounds: `sample_chain(..., require_valid=True)`, dl_sample_chain_retry and
dl_molecule_check.

An atom's valence is the sum of get_bond_order over its pairs with the other checked atoms of chain[0] -- without the
pocket on cut-off graphs -- and a molecule passes when no atom exceeds max_valence of its type. The oracle is the CPU
restatement of build_xae_molecule (oracle/difflinker_oracle.py), symmetrised and summed per atom. CPU tests pin that oracle
to the reference's bond fixtures and check the tables, the argument refusals, the header and the binding; the GPU tests
check the kernel atom by atom on purpose-built batches, and the sampler end to end."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import DDPM, _native, molecule_builder as mb, output, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import accelerate, sampler_inputs
from difflinker_b200.edm import retry_seed, seeds_tensor
from difflinker_b200.utils import FoundNaNException
from oracle import difflinker_oracle as orc
import dl_helpers as helpers
import test_connected_resampling as tcr
from test_connected_resampling import C_C, THR_CC, line, pack

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOTH = _native.CHECK_CONNECTED | _native.CHECK_VALENCE


def valence_of(E):
    """Per-atom valence of a lower-triangular bond-order matrix: its row plus its column sums."""
    E = torch.as_tensor(E).to(torch.int64)
    return E.sum(0) + E.sum(1)


def oracle_valence(x, types, keep, is_geom):
    """The oracle: build_xae_molecule's bond orders over the rows `keep`, summed per atom; 0 on the other rows."""
    idx = torch.nonzero(keep).flatten()
    out = torch.zeros(x.shape[0], dtype=torch.int64)
    if idx.numel():
        idx2atom = output.GEOM_IDX2ATOM if is_geom else output.IDX2ATOM
        _, _, E = orc.xae_molecule(x[idx].float(), types[idx], idx2atom, mb.SINGLE, mb.DOUBLE, mb.TRIPLE, mb.MARGINS_EDM)
        out[idx] = valence_of(E)
    return out


def oracle_ok(valence, types, keep, is_geom):
    table = mb.max_valence_table(is_geom).long()
    return bool((valence[keep] <= table[types[keep]]).all())


def oracle_chain(chain0, node_mask, is_geom, n_types, pocket_only=None):
    """((B,N) valences, (B,) valence-ok, (B,) connected) of a chain[0] (B,N,3+F) by the host oracle."""
    chain0 = chain0.cpu()
    B, N = chain0.shape[:2]
    keep = node_mask.reshape(B, N).cpu() != 0
    if pocket_only is not None:
        keep = keep & (pocket_only.reshape(B, N).cpu() == 0)
    types = torch.argmax(chain0[:, :, 3:3 + n_types], dim=2)
    val = torch.stack([oracle_valence(chain0[b, :, :3], types[b], keep[b], is_geom) for b in range(B)])
    ok = torch.tensor([oracle_ok(val[b], types[b], keep[b], is_geom) for b in range(B)])
    conn = torch.tensor([tcr.oracle_connected(chain0[b, :, :3], types[b], keep[b], is_geom) if keep[b].any() else False
                         for b in range(B)])
    return val, ok, conn


# ---- CPU --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["bonds_zinc", "bonds_geom"])
def test_oracle_valence_reproduces_the_reference_bond_sums(name):
    meta, a = helpers.load_golden(name)
    over = 0
    for b in range(a["positions"].shape[0]):
        n = int(a["node_mask"][b].sum())
        keep = a["node_mask"][b] != 0
        want = valence_of(a["E"][b, :n, :n])                             # the reference's own bond orders
        got = oracle_valence(a["positions"][b], a["types"][b], keep, meta["is_geom"])
        assert torch.equal(got[:n], want) and not got[n:].any(), b
        over += not oracle_ok(got, a["types"][b].long(), keep, meta["is_geom"])
    print(f"{name}: {over} of {a['positions'].shape[0]} molecules hold an atom beyond its valence")


def test_max_valence_table_has_one_entry_per_atom_type():
    for is_geom, idx2atom in ((False, output.IDX2ATOM), (True, output.GEOM_IDX2ATOM)):
        t = mb.max_valence_table(is_geom)
        assert t.dtype == torch.int32 and t.shape == (len(idx2atom),) == (mb.threshold_tables(is_geom)[0].shape[0],)
        assert t.tolist() == [mb.MAX_VALENCE[idx2atom[k]] for k in range(len(idx2atom))]
    assert mb.max_valence_table(True).tolist() == [4, 2, 3, 1, 6, 1, 1, 5, 7]
    assert set(mb.MAX_VALENCE) == set(output.GEOM_IDX2ATOM.values())


@pytest.mark.parametrize("inpainting", [False, True])
def test_valence_refuses_what_connectivity_refuses(inpainting):
    """Case for case the refusals of test_connectivity_refuses_what_cannot_resample_one_molecule."""
    ddpm, kw = tcr._cpu_model(inpainting)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    assert edm.require_valid is False and edm.last_valid is None
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_valid"):
            edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3], require_valid=bad)
    with pytest.raises(ValueError, match="require_valid needs per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2, require_valid=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_valid=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="require_valid does not take batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_valid=True, seeds=[1, 2, 3], batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_valid needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_valid=True, seeds=[1, 2, 3])
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="require_valid.*replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_valid=True, seeds=[1, 2, 3])
    delattr(edm, name)
    edm.require_valid = True                                             # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.noise_mode = 'per_molecule'
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_valid needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.is_geom = None
    with pytest.raises(ValueError, match="require_valid needs the bond tables"):
        edm.sample_chain(**kw, keep_frames=2)
    assert edm.last_valid is None and edm.last_connected is None


def test_models_pass_the_keyword_and_the_tables_to_the_edm():
    """DDPM and accelerate()d modules give the EDM its is_geom, from which it takes the four tables; every sampling entry
    hands `require_valid` down to EDM.sample_chain / sample_many."""
    for name, T in (("cfg2_zinc", 8), ("cfg3_geom", 9)):
        ddpm = accelerate(DDPM(**synthetic.model_hparams(synthetic.SPECS[name])))
        tables = ddpm.edm._check_tables(BOTH)
        assert [tuple(t.shape) for t in tables] == [(T, T)] * 3 + [(T,)] and tables[3].dtype == torch.int32
        assert len(ddpm.edm._check_tables(_native.CHECK_CONNECTED)) == 1
    ddpm, _ = tcr._cpu_model()
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append(k.get('require_valid', 'unset'))
    ddpm.edm.sample_many = lambda reqs, **k: seen.append(k.get('require_valid', 'unset')) or [None] * len(reqs)
    from difflinker_b200 import ddpm as ddpm_mod, distributed
    ddpm.sample_chain(data, keep_frames=2, require_valid=True)
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, require_valid=False)
    ddpm.sample_many([data], keep_frames=2, seeds=[[1, 2, 3]], require_valid=True)
    ddpm_mod.sample_many(ddpm, [data], keep_frames=2, seeds=[[1, 2, 3]])
    distributed.sample_chain_sharded(ddpm, data, keep_frames=2, seeds=[1, 2, 3], require_valid=True)
    assert seen == [True, 'unset', False, True, 'unset', True]


def test_native_binds_the_check_entry_and_the_one_retry_entry():
    lib = _native.load_library()
    assert "dl_sample_chain_retry" in _native.SYMBOLS and "dl_molecule_check" in _native.SYMBOLS
    argtypes = lib.dl_sample_chain_retry.argtypes
    assert argtypes[20]._type_ is _native.DLMoleculeChecks and argtypes[22]._type_ is _native.DLSizeRedraw
    # connectivity alone, NaN recovery alone, checks, size redraws and the clash table all run through dl_sample_chain_retry
    for gone in ("dl_sample_chain_seeded_retry_connected", "dl_molecule_connected", "dl_sample_chain_seeded_retry",
                 "dl_sample_chain_seeded_retry_checked", "dl_sample_chain_seeded_retry_sized", "dl_set_clash_table"):
        assert gone not in _native.SYMBOLS and not hasattr(lib, gone)
    assert lib.dl_molecule_check.argtypes[2]._type_ is _native.DLMoleculeChecks
    assert (_native.CHECK_CONNECTED, _native.CHECK_VALENCE) == (1, 2)
    assert _native.DLMoleculeChecks.of(3, [torch.zeros(8, 8)]).n_types == 8
    for require in (0, 4, 7):                                            # outside the known bits, before any pointer is read
        ck = _native.DLMoleculeChecks(require, 8, 1, 1, 1, 1)
        assert lib.dl_molecule_check(1, 4, ck, 1, 11, 1, None, 0, 0, 1, None, None) == -1
        assert b"require" in lib.dl_last_error()


def test_header_compiles_as_c99_with_the_checks_of_the_retry_entry(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "checked_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2]; int32_t attempts[2], flags[2], passed[2];\n"
        "  dl_molecule_checks ck = {DL_CHECK_CONNECTED | DL_CHECK_VALENCE, 8, NULL, NULL, NULL, NULL, NULL};\n"
        "  dl_status a = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                      NULL, NULL, NULL, NULL, flags, 3, used, attempts, &ck, passed, NULL, NULL,\n"
        "                                      NULL);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  dl_status b = dl_molecule_check(2, 4, &ck, NULL, 11, NULL, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s|", (int)b, dl_last_error());\n'
        "  ck.require = 8;\n"
        "  dl_status c = dl_molecule_check(2, 4, &ck, NULL, 11, NULL, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)c, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "checked_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, err_a, b, err_b, c, err_c = res.stdout.strip().split("|", 5)
    assert int(a) == -1 and "null engine" in err_a
    assert int(b) == -1 and "dl_molecule_check" in err_b and "thr1" in err_b
    assert int(c) == -1 and "require" in err_c


# ---- GPU: the kernel, atom by atom --------------------------------------------------------------------------------------

C, O, N_, F, S, CL, BR, I = range(8)


def star(k, d=C_C):
    """A centre at the origin and k neighbours at distance d on the axes (pairwise d * sqrt(2) apart or more)."""
    axes = torch.tensor([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [0, -1.0, 0], [0, 0, 1.0], [0, 0, -1.0]])
    return torch.cat([torch.zeros(1, 3), d * axes[:k]])


def purpose_built():
    """(name, positions, types, pocket flags, valid rows, valence-ok) molecules, in the tuple layout of tcr.pack."""
    mols = []

    def add(name, pos, want, types=None, pocket=None, valid=None):
        n = pos.shape[0]
        mols.append((name, pos, torch.zeros(n, dtype=torch.long) if types is None else torch.tensor(types),
                     torch.zeros(n) if pocket is None else torch.tensor(pocket),
                     torch.ones(n, dtype=torch.bool) if valid is None else torch.tensor(valid), want))
    add("carbon, 4 single bonds", star(4), True)
    add("carbon, 5 single bonds", star(5), False)
    double, triple = torch.tensor([[1.35, 0.0, 0.0]]), torch.tensor([[1.2, 0.0, 0.0]])
    add("C=C and two singles", torch.cat([torch.zeros(1, 3), double, star(4)[3:]]), True)
    add("C#C and two singles", torch.cat([torch.zeros(1, 3), triple, star(4)[3:]]), False)
    add("fluorine, one neighbour", star(1, 1.3), True, types=[F, C])
    add("fluorine, two neighbours", star(2, 1.3), False, types=[F, C, C])
    add("pair at the single threshold", torch.cat([line(1), line(1, start=THR_CC)]), True)
    add("at the double threshold: single", torch.cat([line(1), line(1, start=1.39)]), True)
    add("at the triple threshold: double", torch.cat([line(1), line(1, start=1.22)]), True)
    add("Cl-I: no bond length", star(1, 1.0), True, types=[CL, I])
    add("oxygen, three neighbours", star(3, 1.4), False, types=[O, C, C, C])
    add("no atom", star(2), True, valid=[False, False, False])
    add("one atom", line(1), True)
    add("one atom among padding", star(5), True, valid=[False, False, True, False, False, False])
    # the fifth neighbour is a pocket atom: not a partner
    add("fifth neighbour in the pocket", star(5), True, pocket=[0.0, 0, 0, 0, 0, 1.0])
    add("fifth neighbour padded", star(5), True, valid=[True, True, True, True, True, False])
    add("chlorine bridging two carbons", star(2, 1.7), False, types=[CL, C, C])
    return mols


def run_check(xh, nm, is_geom, po=None, require=BOTH, max_valence=None):
    """dl_molecule_check on the device: ((B,) bits, (B,N) valences) on the host."""
    d = tcr.dev()
    passed, val = mb._molecule_check(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d), max_valence, require,
                                     bool(require & _native.CHECK_VALENCE))
    return passed.cpu(), None if val is None else val.cpu()


def assert_matches_oracle(xh, nm, is_geom, po=None):
    """Both verdict bits and every valence equal the oracle's, the connected bit also molecule_builder.connected's, and each
    check alone gives its own bit."""
    d = tcr.dev()
    T = 9 if is_geom else 8
    passed, val = run_check(xh, nm, is_geom, po)
    want_val, want_ok, want_conn = oracle_chain(xh, nm, is_geom, T, po)
    assert torch.equal(val.long(), want_val)
    assert torch.equal((passed & 2) != 0, want_ok), ((passed & 2) != 0, want_ok)
    assert torch.equal((passed & 1) != 0, want_conn)
    conn = mb.connected(xh.to(d), nm.to(d), is_geom, pocket_only=None if po is None else po.to(d)).cpu()
    assert torch.equal((passed & 1) != 0, conn)
    only_v, val_v = run_check(xh, nm, is_geom, po, require=_native.CHECK_VALENCE)
    only_c, _ = run_check(xh, nm, is_geom, po, require=_native.CHECK_CONNECTED)
    assert torch.equal(only_v, passed & 2) and torch.equal(only_c, passed & 1) and torch.equal(val_v, val)
    assert torch.equal(mb.valence_ok(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d)).cpu(), want_ok)
    assert torch.equal(mb.valences(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d)).cpu(), val)
    return passed, val


@pytest.mark.gpu
def test_check_matches_the_oracle_on_purpose_built_molecules():
    for v in (THR_CC, 1.39, 1.22):                                       # the pairs really sit on the thresholds in fp32
        assert float(np.float32(100) * np.sqrt(np.float32(v) ** 2)) == round(100 * v)
    mols = purpose_built()
    xh, nm, po = pack(mols, N=8)
    passed, val = assert_matches_oracle(xh, nm, False, po)
    for b, (name, *_, want) in enumerate(mols):
        assert bool(passed[b] & 2) == want, name
    by = {m[0]: b for b, m in enumerate(mols)}
    assert val[by["carbon, 5 single bonds"], 0] == 5 and val[by["C#C and two singles"], :2].tolist() == [5, 3]
    assert val[by["at the double threshold: single"], :2].tolist() == [1, 1]
    assert val[by["at the triple threshold: double"], :2].tolist() == [2, 2]
    assert not val[by["pair at the single threshold"]].any() and not val[by["Cl-I: no bond length"]].any()
    # counted, the pocket atom is the fifth bond
    b = by["fifth neighbour in the pocket"]
    p2, v2 = run_check(xh[b:b + 1], nm[b:b + 1], False)
    assert not p2[0] & 2 and v2[0, 0] == 5
    # a caller's own table: five-valent carbon allowed, two-valent oxygen still not
    own = mb.max_valence_table(False).clone(); own[C] = 5
    p3, _ = run_check(xh, nm, False, po, max_valence=own)
    assert p3[by["carbon, 5 single bonds"]] & 2 and not p3[by["oxygen, three neighbours"]] & 2
    with pytest.raises(ValueError, match="one entry per atom type"):
        run_check(xh, nm, False, po, max_valence=[4, 2])


@pytest.mark.gpu
def test_nan_data_is_compared_like_the_oracle_compares_it():
    """A NaN coordinate bonds to nothing; a NaN among the type features wins the argmax, as torch.argmax has it."""
    pos = star(4)
    xh, nm, po = pack([("nan x", pos, torch.zeros(5, dtype=torch.long), torch.zeros(5), torch.ones(5, dtype=torch.bool), True),
                       ("nan h", pos, torch.zeros(5, dtype=torch.long), torch.zeros(5), torch.ones(5, dtype=torch.bool), False),
                       ("nan h row", pos, torch.zeros(5, dtype=torch.long), torch.zeros(5), torch.ones(5, dtype=torch.bool), True)],
                      N=6)
    xh[0, 1, 0] = float('nan')
    xh[1, 0, 3 + N_] = float('nan')                                      # the centre reads as nitrogen: 4 bonds > 3
    xh[2, 0, 3:] = float('nan')                                          # every feature NaN: the first one wins, carbon
    passed, val = assert_matches_oracle(xh, nm, False, po)
    assert val[0, :5].tolist() == [3, 0, 1, 1, 1] and val[1, 0] == 4 and val[2, 0] == 4
    assert [(int(p) & 2) != 0 for p in passed] == [True, False, True]


def zigzag(n):
    return torch.stack([1.25 * torch.arange(n, dtype=torch.float32), 0.8 * (torch.arange(n) % 2).float(), torch.zeros(n)], 1)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [255, 256, 257])
def test_molecules_that_fill_the_compaction_chunks(N):
    """Every row an atom, around the 256-row chunk of the compaction: a chain (valence 2 inside), and the same chain with
    four more neighbours around its last atom."""
    xh = torch.zeros(2, N, 11)
    xh[:, :, 3] = 1.0
    nm = torch.ones(2, N, dtype=torch.int8)
    xh[0, :, :3] = zigzag(N)
    xh[1, :N - 4, :3] = zigzag(N - 4)
    away = 1.0 if (N - 5) % 2 else -1.0                                  # the side of y the chain does not come from
    xh[1, N - 4:, :3] = xh[1, N - 5, :3] + C_C * torch.tensor([[0.0, 0, 1.0], [0, 0, -1.0], [1.0, 0, 0], [0, away, 0]])
    passed, val = assert_matches_oracle(xh, nm, False)
    assert passed.tolist() == [3, 1] and val[0].tolist() == [1] + [2] * (N - 2) + [1] and val[1, N - 5] == 5


@pytest.mark.gpu
def test_a_ligand_of_more_than_128_atoms_spread_over_a_4000_row_pocket_batch():
    """N = 4000 takes 80 KB of shared memory; the 150 ligand rows lie in every 256-row chunk. Each ligand atom has a pocket
    atom and a padded row 1.5 A above and below it, which would be its third and fourth bonds -- and, in molecule 1, one
    ligand atom has three more ligand neighbours, five bonds in all."""
    N, n_lig = 4000, 150
    rows = torch.arange(n_lig) * 26 + 3
    xh = torch.zeros(2, N, 11)
    xh[:, :, 3] = 1.0
    xh[:, :, :3] = torch.tensor([0.0, 500.0, 0.0])
    nm = torch.zeros(2, N, dtype=torch.int8)
    po = torch.zeros(2, N)
    lig = zigzag(n_lig)
    for b in range(2):
        xh[b, rows, :3] = lig
        nm[b, rows] = 1
        xh[b, rows + 1, :3] = lig + torch.tensor([0.0, 0.0, 1.5])        # pocket atoms
        nm[b, rows + 1] = 1
        po[b, rows + 1] = 1.0
        xh[b, rows + 2, :3] = lig - torch.tensor([0.0, 0.0, 1.5])        # padded rows
    extra = torch.tensor([3990, 3991, 3995])                             # three more ligand rows around ligand atom 75
    xh[1, extra, :3] = lig[75] + torch.tensor([[0.0, 0.0, 1.45], [0.0, 0.0, -1.45], [0.0, 1.45 * (-1.0) ** 76, 0.0]])
    nm[1, extra] = 1
    passed, val = assert_matches_oracle(xh, nm, False, po)
    assert passed.tolist() == [3, 1] and val[1, rows[75]] == 5 and int(val[0].max()) == 2
    assert not val[:, rows + 1].any() and not val[:, rows + 2].any()
    # counted as atoms, the pocket atoms are a third bond of every ligand atom: still within carbon's four
    p2, v2 = run_check(xh[:1], nm[:1], False)
    assert p2[0] & 2 and int(v2[0].max()) == 3


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_valence_is_the_row_plus_column_sum_of_bond_orders(is_geom):
    d = tcr.dev()
    T = 9 if is_geom else 8
    g = torch.Generator().manual_seed(5)
    B, N = 96, 40
    n = torch.randint(1, N + 1, (B,), generator=g)
    nm = (torch.arange(N)[None, :] < n[:, None]).to(torch.int8)
    scale = (0.5 + 2.5 * torch.rand(B, 1, 1, generator=g)) * n[:, None, None].float().pow(1 / 3)
    types = torch.randint(0, T, (B, N), generator=g)
    xh = torch.cat([torch.rand(B, N, 3, generator=g) * scale, torch.nn.functional.one_hot(types, T).float()], 2)
    passed, val = run_check(xh, nm, is_geom)
    E = mb.bond_orders(xh[:, :, 3:].to(d), xh.to(d), nm.to(d), is_geom).cpu().long()
    want = E.sum(1) + E.sum(2)
    assert torch.equal(val.long(), want)
    assert int((E == 2).sum()) > 0 and int((E == 3).sum()) > 0           # every order takes part
    table = mb.max_valence_table(is_geom).long()
    ok = ((want <= table[types]) | (nm == 0)).all(1)
    assert torch.equal((passed & 2) != 0, ok) and 0 < int(ok.sum()) < B, int(ok.sum())
    assert torch.equal((passed & 1) != 0, mb.connected(xh.to(d), nm.to(d), is_geom).cpu())


# ---- GPU: the sampler, end to end ---------------------------------------------------------------------------------------

SEEDS = list(range(11, 27))
ROUNDS = 4
CASES = tcr.CASES
# A 3 x 2 x 2 carbon lattice with 1.5 A single bonds: the four middle atoms hold four bonds already, the corners three. A
# linker atom that ends within bonding distance of a middle atom gives it a fifth bond; one that ends next to a corner, or
# away from the fragment, does not. The models and their noise precision are those of the connectivity tests.
FRAG = torch.stack(torch.meshgrid(torch.arange(3.0), torch.arange(2.0), torch.arange(2.0), indexing='ij'), -1).reshape(-1, 3)
FRAG = 1.5 * (FRAG - FRAG.mean(0))
NF = FRAG.shape[0]


def fragment_items(case, rows):
    """FRAG and none, one or two linker atoms per molecule; pocket cases add 12 pocket atoms on a 6 A shell."""
    g = torch.Generator().manual_seed(78)
    pocket = 12 if case.startswith("pocket") else 0
    Fw = 9 if pocket else 8
    items = []
    for b in range(rows):
        link = torch.tensor([[0.0, 0.0, 2.2], [0.0, 0.0, 3.4]])[:b % 3]
        parts = [FRAG]
        if pocket:
            v = torch.randn(pocket, 3, generator=g)
            parts.append(6.0 * v / v.norm(dim=1, keepdim=True))
        parts.append(link)
        pos = torch.cat(parts)
        n = pos.shape[0]
        types = torch.zeros(n, dtype=torch.long)
        if pocket:
            types[NF:NF + pocket] = torch.randint(0, 3, (pocket,), generator=g)
        frag_only = torch.zeros(n); frag_only[:NF] = 1.0
        pocket_mask = torch.zeros(n); pocket_mask[NF:NF + pocket] = 1.0
        linker_mask = torch.zeros(n); linker_mask[NF + pocket:] = 1.0
        anchors = torch.zeros(n); anchors[[0, NF - 1]] = 1.0
        item = {'uuid': b, 'name': f'valence_{b}', 'positions': pos, 'one_hot': torch.nn.functional.one_hot(types, Fw).float(),
                'anchors': anchors, 'fragment_mask': frag_only + pocket_mask, 'linker_mask': linker_mask, 'num_atoms': n}
        if pocket:
            item['fragment_only_mask'] = frag_only
            item['pocket_mask'] = pocket_mask
        items.append(item)
    return items


def build(case, impl, rows=len(SEEDS)):
    d = tcr.dev()
    spec, over = tcr.model_spec(case, rows)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(tcr.COORD_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(fragment_items(case, rows)).items()}
    return ddpm, sampler_inputs(ddpm, data), data


def oracle_rows(ddpm, kw, chain0):
    """((B,) valence-ok, (B,) connected) of a returned chain[0] by the host oracle."""
    pocket_only = kw['context'][..., -1] if ddpm.edm.dynamics.graph_type != 'FC' else None
    _, ok, conn = oracle_chain(chain0, kw['node_mask'], ddpm.edm.is_geom, 9 if ddpm.edm.is_geom else 8, pocket_only)
    return ok, conn


def launches(ddpm):
    eng = ddpm.edm.dynamics.engine(0)
    return int(_native.load_library().dl_launch_count(eng))


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", CASES)
def test_rounds_resample_only_the_molecules_that_fail_a_required_check(case, impl):
    ddpm, kw, _ = build(case, impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    n0 = launches(ddpm)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS), base)
    per_call = launches(ddpm) - n0
    assert edm.last_valid is None and edm.last_connected is None
    # nan_retries = 0: the checks only report, and the chain is the one sampled without them -- one more launch
    n0 = launches(ddpm)
    r0 = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_valid=True, require_connected=True)
    assert launches(ddpm) - n0 == per_call + 1
    ok0, conn0 = edm.last_valid, edm.last_connected
    assert torch.equal(r0, base) and ok0.dtype == torch.bool and ok0.shape == (B,)
    want_ok, want_conn = oracle_rows(ddpm, kw, base[0])
    assert torch.equal(ok0, want_ok) and torch.equal(conn0, want_conn)
    assert edm.last_attempts.tolist() == [0] * B and torch.equal(edm.last_seeds, seeds_tensor(SEEDS, B))
    good0 = ok0 & conn0
    runs = []
    for r in range(ROUNDS + 1):
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=r, require_valid=True, require_connected=True)
        runs.append((chain, edm.last_valid & edm.last_connected, edm.last_attempts, edm.last_seeds))
        ok_r, conn_r = oracle_rows(ddpm, kw, chain[0])                   # the flags of the rows each round wrote back
        assert torch.equal(edm.last_valid, ok_r) and torch.equal(edm.last_connected, conn_r), r
    chain, good, attempts, used = runs[-1]
    assert torch.isfinite(chain).all()
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
    healthy = good0.nonzero().flatten().tolist()
    # The linker sampler leaves the lattice where it is, so the batch mixes rows that pass with rows that do not. The
    # inpainting sampler re-noises the fragment too, by more than the 0.1 A a 1.5 A bond has to either threshold: there no
    # row need pass, and what is checked is that the rounds keep their invariants on rows that all fail.
    mixes = case != "fc_inpainting"
    assert len(healthy) < B and (len(healthy) > 0 or not mixes), healthy
    assert torch.equal(chain[:, healthy], base[:, healthy]) and all(int(attempts[b]) == 0 for b in healthy)
    first = [int(attempts[b]) if good[b] else None for b in range(B)]
    recovered = [b for b in range(B) if first[b] is not None and first[b] > 0]
    assert recovered or not mixes, first                                 # some rows pass in a round
    counts = []
    for r, (c_r, good_r, att_r, _) in enumerate(runs):
        counts.append(int(good_r.sum()))
        for b in range(B):
            # a run with fewer rounds is the prefix: a row is kept from the round that passed it, else resampled each round
            want_att = first[b] if first[b] is not None and first[b] <= r else (r if not good0[b] else 0)
            assert int(att_r[b]) == want_att, (r, b)
            if first[b] is not None and first[b] <= r:
                assert bool(good_r[b]) and torch.equal(c_r[:, b], chain[:, b]), (r, b)
    assert counts == sorted(counts) and (counts[-1] > counts[0] or not mixes), counts   # more passing rows, never fewer
    for b in range(B):                                                   # a resampled row is its molecule sampled alone
        if int(attempts[b]) > 0:
            alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert tcr.same(chain[:, b], alone[:, 0], impl), b
    print(f"{case}/{impl}: valence-ok {int(ok0.sum())}, connected {int(conn0.sum())} of {B} at round 0; passing both after "
          f"rounds 0..{ROUNDS}: {counts}; recovered rows {recovered} (rounds {[first[b] for b in recovered]})")


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_each_flag_alone_and_both_resample_their_own_rows(impl):
    ddpm, kw, _ = build("fc", impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_valid=True, require_connected=True)
    ok0, conn0 = edm.last_valid, edm.last_connected
    assert len({(bool(o), bool(c)) for o, c in zip(ok0, conn0)}) >= 3, (ok0, conn0)   # rows failing either check alone
    n0 = launches(ddpm)
    edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_connected=True)
    with_conn = launches(ddpm) - n0
    for flags, fails0 in (({'require_valid': True}, ~ok0), ({'require_connected': True}, ~conn0),
                          ({'require_valid': True, 'require_connected': True}, ~(ok0 & conn0))):
        got = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=1, **flags)
        assert (edm.last_attempts != 0).tolist() == fails0.tolist(), flags
        kept = (~fails0).nonzero().flatten().tolist()
        assert torch.equal(got[:, kept], base[:, kept])
        assert (edm.last_valid is None) == ('require_valid' not in flags)
        assert (edm.last_connected is None) == ('require_connected' not in flags)
        ok, conn = oracle_rows(ddpm, kw, got[0])
        assert edm.last_valid is None or torch.equal(edm.last_valid, ok)
        assert edm.last_connected is None or torch.equal(edm.last_connected, conn)
    # the default and the connectivity-only call launch what they launched before valence existed: one check kernel more
    n0 = launches(ddpm)
    edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    plain = launches(ddpm) - n0
    n0 = launches(ddpm)
    edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_valid=True)
    assert with_conn == plain + 1 and launches(ddpm) - n0 == plain + 1


@pytest.mark.gpu
def test_a_finite_row_is_not_replaced_by_a_resample_that_diverged_with_the_valence_check_on():
    """The molecules of test_a_finite_row_is_not_replaced_by_a_resample_that_diverged: random point clouds, never connected,
    some diverging at round 0 and some only in round 1."""
    d = tcr.dev()
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl="simt")
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(tcr.DIVERGE_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    edm = ddpm.edm
    seeds = tcr.DIVERGE_SEEDS
    B = len(seeds)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=B)).items()}
    kw = sampler_inputs(ddpm, data)

    def run(rounds):
        try:
            chain, bad = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, nan_retries=rounds, require_valid=True,
                                          require_connected=True), []
        except FoundNaNException as e:
            chain, bad = e.chain, sorted(e.x_h_nan_idx | e.only_x_nan_idx | e.only_h_nan_idx)
        return chain, bad, edm.last_attempts.clone(), (edm.last_valid & edm.last_connected).clone()
    base, bad0, _, good0 = run(0)
    got, bad1, attempts, _ = run(1)
    assert not good0.any() and 0 < len(bad0) < B, bad0
    kept = []
    for b in range(B):
        try:
            edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[retry_seed(seeds[b], 1)])
            diverges = False
        except FoundNaNException:
            diverges = True
        if b not in bad0 and diverges:
            kept.append(b)
            assert int(attempts[b]) == 0 and b not in bad1 and torch.equal(got[:, b], base[:, b]), b
        else:
            assert int(attempts[b]) == 1 and (b in bad1) == diverges, b
    assert kept, bad0


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_a_split_and_sample_many_resample_what_the_plain_call_resamples(impl):
    ddpm, kw, data = build("fc", impl)
    edm = ddpm.edm
    opts = dict(keep_frames=2, nan_retries=ROUNDS, require_valid=True, require_connected=True)
    want = edm.sample_chain(**kw, seeds=SEEDS, **opts)
    ok, conn, attempts, used = edm.last_valid, edm.last_connected, edm.last_attempts, edm.last_seeds
    edm.devices = [0, 0]
    try:
        got = edm.sample_chain(**kw, seeds=SEEDS, **opts)
    finally:
        edm.devices = None
    assert torch.equal(edm.last_valid, ok) and torch.equal(edm.last_connected, conn)
    assert torch.equal(edm.last_attempts, attempts) and torch.equal(edm.last_seeds, used) and tcr.same(got, want, impl)
    # two requests, rows 0..9 and 10..15, in one launch
    cuts = [(0, 10), (10, len(SEEDS))]
    reqs = [tcr.take(kw, list(range(lo, hi))) for lo, hi in cuts]
    outs = edm.sample_many(reqs, seeds=[SEEDS[lo:hi] for lo, hi in cuts], **opts)
    for k, (lo, hi) in enumerate(cuts):
        alone = edm.sample_chain(**reqs[k], seeds=SEEDS[lo:hi], **opts)
        assert tcr.same(outs[k], alone, impl), k
        assert torch.equal(edm.last_valid_many[k], edm.last_valid) and torch.equal(edm.last_connected_many[k], edm.last_connected)
        assert torch.equal(edm.last_attempts_many[k], edm.last_attempts)
        assert torch.equal(edm.last_valid, ok[lo:hi]) and torch.equal(edm.last_attempts, attempts[lo:hi])
    # the attribute and DDPM opt in as for require_connected
    edm.nan_retries, edm.require_valid, edm.require_connected = ROUNDS, True, True
    chain, _ = ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS)
    assert tcr.same(chain, want, impl) and torch.equal(edm.last_valid, ok)
    ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS, require_valid=False, require_connected=False, nan_retries=0)
    assert edm.last_valid is None and edm.last_connected is None
