"""Novelty in the recovery rounds -- `sample_chain(..., require_novel=True)`, dl_sample_chain_retry_sets with
DL_CHECK_NOVEL and a known set -- and uniqueness across calls, `sample_chain(..., require_unique=True, exclude_hashes=...)`.

The linker hash L is the graph hash of DL_CHECK_UNIQUE on the linker rows alone (stated at DL_CHECK_NOVEL in the header),
so graph_hash_oracle restates it. CPU tests check the oracle's L, the unsigned sort, the refusals, the binding and the header;
the GPU tests check the kernel's bits against the oracle with planted sets, and the sampler end to end."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, distributed, molecule_builder as mb
from difflinker_b200 import edm as edm_mod
from difflinker_b200.edm import retry_seed
import graph_hash_oracle as gho
import test_connected_resampling as tcr
import test_unique_resampling as tur

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NOVEL, UNIQUE = 16, 8
C, O, N_ = 0, 1, 2


def oracle_linker_hashes(xh, nm, lm, is_geom, po=None):
    """((B,) L as Python ints, (B,) smallest |distance - threshold|) by the host oracle: graph_hash over the linker rows."""
    B, N = xh.shape[:2]
    keep = (nm.detach().cpu().reshape(B, N) != 0) & (lm.detach().cpu().reshape(B, N) != 0)
    return gho.batch_hashes(xh, keep.to(torch.int8), is_geom, po)


def unsigned(t):
    return [int(v) % (1 << 64) for v in t.tolist()]


# ---- CPU -------------------------------------------------------------------------------------------------------------

def ring_with_tail():
    """A carbon six-ring (1.45 A bonds) with an O tail at 1.36 A: the linker, and a fragment carbon bonded to the ring. Every
    pair lies at least 5 pm from its thresholds (ZINC and GEOM tables)."""
    ang = np.arange(6) * np.pi / 3
    ring = np.stack([1.45 * np.cos(ang), 1.45 * np.sin(ang), np.zeros(6)], 1)
    tail = ring[0] * (1 + 1.36 / 1.45)
    frag = ring[3] * (1 + 1.50 / 1.45)
    x = np.concatenate([ring, tail[None], frag[None]]).astype(np.float32)
    types = np.array([C] * 6 + [O, C])
    linker = np.array([1] * 7 + [0], np.float32)
    return x, types, linker


def test_oracle_linker_hash_is_the_graph_hash_of_the_linker_rows():
    x, types, linker = ring_with_tail()
    thr = [t.numpy() for t in mb.threshold_tables(False)]
    o, near = gho.bond_order_matrix(x[:7], types[:7], thr)
    assert near > 1.0 and o.sum() == 2 * 7                               # six ring bonds and the tail
    want = gho.graph_hash(types[:7], o)
    N = 14
    for seed in range(4):                                                # any row order, pose and padding
        rng = np.random.default_rng(seed)
        rows = rng.choice(N, 8, replace=False)
        xr = (x @ tur.rotation(seed).T + rng.normal(size=3) * 5).astype(np.float32)
        xh = torch.zeros(1, N, 3 + 8)
        xh[0, :, :3] = 40.0
        nm, lm = torch.zeros(1, N, dtype=torch.int8), torch.zeros(1, N)
        for k, r in enumerate(rows):
            xh[0, r, :3] = torch.from_numpy(xr[k])
            xh[0, r, 3 + int(types[k])] = 1.0
            nm[0, r], lm[0, r] = 1, float(linker[k])
        got, near_b = oracle_linker_hashes(xh, nm, lm, False)
        assert near_b[0] > 1.0 and got[0] == want, seed
        whole, _ = gho.batch_hashes(xh, nm, False)
        assert whole[0] != want                                          # the fragment atom is not part of L
        none, _ = oracle_linker_hashes(xh, nm, torch.zeros_like(lm), False)
        assert none[0] == gho.mix(0) == 0


def test_sort_unsigned_orders_high_hashes_last_and_keeps_duplicates():
    vals = [5, -1, 0, -(1 << 63), (1 << 63) - 1, 5, -2, 7, -1]          # int64 bits; negatives are hashes >= 2^63
    got = mb.sort_unsigned(torch.tensor(vals, dtype=torch.int64))
    assert got.dtype == torch.int64
    assert unsigned(got) == sorted(v % (1 << 64) for v in vals)
    assert mb.sort_unsigned(torch.zeros(0, dtype=torch.int64)).numel() == 0


def test_require_novel_refuses_what_cannot_recover_and_names_what_is_missing():
    ddpm, kw = tcr._cpu_model()
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(1, B + 1))
    assert edm.require_novel is False and edm.known_linkers is None
    assert edm.last_novel is None and edm.last_linker_hashes is None and edm.last_novel_many is None
    with pytest.raises(ValueError, match="require_novel needs the known linker hashes.*known_linkers"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True)
    edm.known_linkers = torch.tensor([3, -4], dtype=torch.int64)
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_novel"):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=bad)
    with pytest.raises(ValueError, match="require_novel needs per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2, require_novel=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_novel=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="require_novel does not take batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_novel=True, seeds=seeds, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_novel needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_novel=True, seeds=seeds)
    edm.draw_noise = lambda *a, **k: None
    with pytest.raises(ValueError, match="require_novel.*replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_novel=True, seeds=seeds)
    del edm.draw_noise
    with pytest.raises(ValueError, match="sample_many needs CUDA inputs"):   # sample_many takes it, on CUDA inputs
        edm.sample_many([kw], keep_frames=2, seeds=[seeds], require_novel=True)
    with pytest.raises(ValueError, match="exclude_hashes.*require_unique"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, exclude_hashes=torch.tensor([1]))
    edm.require_novel = True                                             # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.is_geom = None
    with pytest.raises(ValueError, match="require_novel needs the bond tables"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    assert edm.last_novel is None and edm.last_linker_hashes is None
    # sample_many and a split keep refusing require_unique as before
    edm.require_novel, edm.require_unique = False, True
    with pytest.raises(ValueError, match="sample_many does not take require_unique"):
        edm.sample_many([kw], keep_frames=2, seeds=[seeds])


def test_hash_sets_are_refused_unless_they_are_int64_vectors():
    ddpm, _ = tcr._cpu_model()
    edm = ddpm.edm
    edm.known_linkers = torch.tensor([1.0, 2.0])
    with pytest.raises(ValueError, match="known_linkers is a 1-D int64 tensor"):
        edm._hash_sets(_native.CHECK_NOVEL, None, torch.device('cpu'))
    with pytest.raises(ValueError, match="exclude_hashes is a 1-D int64 tensor"):
        edm._hash_sets(_native.CHECK_UNIQUE, [1, 2], torch.device('cpu'))
    edm.known_linkers = torch.tensor([7, -1, 3, 7], dtype=torch.int64)  # any order; sorted per call
    known, seen = edm._hash_sets(_native.CHECK_NOVEL | _native.CHECK_UNIQUE, torch.tensor([-5, 2]), torch.device('cpu'))
    assert unsigned(known) == sorted(unsigned(edm.known_linkers)) and unsigned(seen) == sorted(unsigned(torch.tensor([-5, 2])))
    assert edm._hash_sets(_native.CHECK_UNIQUE, None, torch.device('cpu')) is None


def test_ddpm_and_the_sharded_sampler_pass_the_new_options():
    ddpm, _ = tcr._cpu_model()
    from difflinker_b200 import ddpm as ddpm_mod, synthetic
    from difflinker_b200.batching import collate
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append((k.get('require_novel', 'unset'), k.get('exclude_hashes', 'unset')))
    ex = torch.tensor([4], dtype=torch.int64)
    ddpm.sample_chain(data, keep_frames=2, require_novel=True, exclude_hashes=ex)
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, require_novel=False)
    distributed.sample_chain_sharded(ddpm, data, keep_frames=2, require_novel=True)
    assert seen[0][0] is True and seen[0][1] is ex
    assert seen[1:] == [('unset', 'unset'), (False, 'unset'), (True, 'unset')]
    many = []
    ddpm.edm.sample_many = lambda reqs, **k: many.append(k.get('require_novel', 'unset')) or [None] * len(reqs)
    ddpm.sample_many([data], keep_frames=2, require_novel=True)
    assert many == [True]


def test_binding_matches_the_header_and_a_c99_caller_gets_the_refusals(tmp_path):
    lib = _native.load_library()
    assert _native.CHECK_NOVEL == NOVEL and "dl_sample_chain_retry_sets" in _native.SYMBOLS
    args = lib.dl_sample_chain_retry_sets.argtypes
    assert args[20]._type_ is _native.DLMoleculeChecks and args[21]._type_ is _native.DLHashSets
    assert args[24]._type_ is _native.DLSizeRedraw
    assert lib.dl_novel_check.argtypes[2]._type_ is _native.DLMoleculeChecks
    assert lib.dl_novel_check.argtypes[3]._type_ is _native.DLHashSets
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "novel_abi.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2], known[3] = {1, 2, 3}; int32_t attempts[2], flags[2], passed[2];\n"
        "  float thr[64] = {0}, xh[22] = {0}; int8_t nm[2] = {0};\n"
        "  dl_molecule_checks ck = {DL_CHECK_NOVEL | DL_CHECK_UNIQUE, 8, thr, thr, thr, NULL, NULL};\n"
        "  dl_hash_sets sets = {known, 3, known, 2};\n"
        '  printf("%d %d %d %d %d|", (int)offsetof(dl_hash_sets, known), (int)offsetof(dl_hash_sets, n_known),\n'
        "         (int)offsetof(dl_hash_sets, seen), (int)offsetof(dl_hash_sets, n_seen), (int)sizeof(dl_hash_sets));\n"
        "  dl_status a = dl_sample_chain_retry_sets(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL,\n"
        "                                           NULL, NULL, NULL, NULL, NULL, flags, 3, used, attempts, &ck, &sets,\n"
        "                                           passed, NULL, NULL, NULL, NULL);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  ck.require = DL_CHECK_CONNECTED;\n"
        "  dl_status n = dl_novel_check(2, 4, &ck, &sets, xh, 11, nm, thr, NULL, 0, 0, passed, used, NULL, NULL);\n"
        '  printf("%d|%s|", (int)n, dl_last_error());\n'
        "  ck.require = DL_CHECK_NOVEL;\n"
        "  dl_status c = dl_molecule_check(2, 4, &ck, xh, 11, nm, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)c, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "novel_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe),
                    _native.LIB_PATH, f"-Wl,-rpath,{os.path.dirname(_native.LIB_PATH)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    offs, a, err_a, n, err_n, c, err_c = res.stdout.strip().split("|", 6)
    assert int(n) == -1 and "dl_novel_check" in err_n and "DL_CHECK_NOVEL" in err_n
    want = [getattr(_native.DLHashSets, f).offset for f in ("known", "n_known", "seen", "n_seen")]
    assert [int(v) for v in offs.split()] == want + [ctypes.sizeof(_native.DLHashSets)]
    assert int(a) == -1 and "null engine" in err_a
    assert int(c) == -1 and "require" in err_c and "linker_mask" in err_c and "dl_molecule_hash" in err_c


# ---- GPU: the kernel's bits, with planted sets ------------------------------------------------------------------------

CV = 1 | 2
# every kind of instantiation: the linker hash alone, with the molecule hash, with the bond checks, with the clash check
REQUIRES = [NOVEL, NOVEL | UNIQUE, NOVEL | CV, NOVEL | 4 | 1, NOVEL | UNIQUE | 4 | CV]


def novel_check(xh, nm, lm, known, is_geom, require, po=None):
    """dl_novel_check (the check launch of the sampler's rounds) on a chain[0]-style batch: ((B,) int32 bits, (B,) int64 L,
    (B,) int64 H or None), on the CPU. `known` is a sorted int64 set or None; `po` marks pocket rows (drop_pocket)."""
    d = tcr.dev()
    B, N = xh.shape[:2]
    xs = xh.float().to(d).contiguous()
    nm_ = (nm.reshape(B, N) != 0).to(torch.int8).to(d).contiguous()
    lm_ = lm.reshape(B, N).float().to(d).contiguous()
    po_ = None if po is None else po.reshape(B, N, 1).float().to(d).contiguous()
    tables = [t.to(d) for t in mb.check_tables(is_geom, require)]
    clash = mb.clash_table(is_geom).to(d) if require & 4 else None
    ck = _native.DLMoleculeChecks.of(require, tables, clash)
    kn = None if known is None else known.to(d).contiguous()
    sets = _native.DLHashSets.of(kn, None)
    passed = torch.empty(B, dtype=torch.int32, device=d)
    L = torch.empty(B, dtype=torch.int64, device=d)
    H = torch.empty(B, dtype=torch.int64, device=d) if require & UNIQUE else None
    lib = _native.load_library()
    with torch.cuda.device(d):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_novel_check(B, N, ck, sets, xs.data_ptr(), xs.shape[2], nm_.data_ptr(), lm_.data_ptr(),
                                         None if po_ is None else po_.data_ptr(), 1, int(po_ is not None), passed.data_ptr(),
                                         L.data_ptr(), None if H is None else H.data_ptr(), st), "dl_novel_check")
    torch.cuda.synchronize(d)
    return passed.cpu(), L.cpu(), None if H is None else H.cpu()


def assert_check_matches(xh, nm, lm, po, is_geom, want_L, sets, requires=REQUIRES):
    """For every instantiation in `requires` and every set: L equals the oracle's want_L bit for bit, the NOVEL bit is 'L
    not in the set', and the other bits and H equal the checks run alone."""
    d = tcr.dev()
    B, N = xh.shape[:2]
    alone = {1: mb.connected(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d)).cpu(),
             2: mb.valence_ok(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d)).cpu()}
    if po is not None:
        alone[4] = mb.clash_free(xh.to(d), nm.to(d), lm.to(d), po.to(d), is_geom).cpu()
    H_alone = mb.graph_hashes(xh.to(d), nm.to(d), is_geom, None if po is None else po.to(d)).cpu()
    want = [gho.as_int64(w) for w in want_L]
    for require in requires:
        if require & 4 and po is None:
            continue
        for name, known in sets.items():
            passed, L, H = novel_check(xh, nm, lm, known, is_geom, require, po)
            assert L.tolist() == want, (require, name)
            members = set(unsigned(known)) if known is not None else set()
            assert [bool(v & NOVEL) for v in passed.tolist()] == [w % (1 << 64) not in members for w in want], \
                (require, name)
            assert not any(v & UNIQUE for v in passed.tolist())
            for bit, ok in alone.items():
                if require & bit:
                    assert [bool(v & bit) for v in passed.tolist()] == ok.tolist(), (require, name, bit)
            if require & UNIQUE:
                assert torch.equal(H, H_alone), (require, name)


def planted_sets(distinct, skip):
    """Sets of size 0, 1 and 2^20 over the distinct hashes `distinct` (ints mod 2^64): the big one plants every one but
    `skip`, with the smallest and largest planted values its first and last entries and values on both sides of 2^63."""
    planted = [v for v in distinct if v != skip]
    assert any(v >= 1 << 63 for v in planted) and any(v < 1 << 63 for v in planted), [hex(v) for v in planted]
    assert min(planted) < skip < max(planted)
    big = mb.sort_unsigned(planted_set(planted, 1 << 20, 0))
    assert unsigned(big[:1])[0] == min(planted) and unsigned(big[-1:])[0] == max(planted)
    return {'none': None, 'empty': torch.zeros(0, dtype=torch.int64),
            'one': torch.tensor([gho.as_int64(planted[0])]), 'big': big}


@pytest.mark.gpu
def test_the_check_launch_matches_the_oracle_on_purpose_built_batches():
    """Rings, permuted isomorphs, size-0 and size-1 linkers (of elements whose single-atom hash lies either side of 2^63),
    pocket rows that carry linker_mask, and NaN rows, through dl_novel_check, the kernels the rounds launch: L, the NOVEL bit
    and every other bit against the oracle and the checks alone, for each kind of instantiation."""
    x, types, linker = ring_with_tail()
    N, F = 24, 9
    mols = []

    def add(xm, tm, lm, pocket=0, nan=None):
        xh = torch.zeros(N, 3 + F)
        xh[:, :3] = 60.0
        xh[:, 3] = 1.0
        n = len(tm)
        xh[:n, :3] = torch.as_tensor(np.asarray(xm, np.float32))
        xh[:n, 3:] = torch.nn.functional.one_hot(torch.as_tensor(np.asarray(tm), dtype=torch.long), F).float()
        nm, lmask, po = torch.zeros(N, dtype=torch.int8), torch.zeros(N), torch.zeros(N)
        nm[:n], lmask[:n] = 1, torch.as_tensor(np.asarray(lm, np.float32))
        if pocket:
            g = torch.Generator().manual_seed(len(mols))
            v = torch.randn(pocket, 3, generator=g)
            xh[n:n + pocket, :3] = torch.as_tensor(x[0]) + 1.45 * v / v.norm(dim=1, keepdim=True)   # bonded to the ring
            nm[n:n + pocket], po[n:n + pocket] = 1, 1.0
            lmask[n:n + pocket] = 1.0                                   # linker_mask set: only drop_pocket keeps them out
        if nan is not None:
            xh[nan] = float('nan')
        mols.append((xh, nm, lmask, po))
    add(x, types, linker)                                                # 0: the ring with its tail
    for seed in range(3):                                                # 1-3: moved, turned, relabelled
        perm = np.random.default_rng(seed).permutation(8)
        add((x @ tur.rotation(seed).T + seed).astype(np.float32)[perm], types[perm], linker[perm])
    add(x, types, np.zeros(8))                                           # 4: size-0 linker, L = 0
    add(x, types, np.eye(8)[6])                                          # 5: size-1 linker, the O alone
    t3 = types.copy()
    t3[6] = 3
    add(x, t3, np.eye(8)[6])                                             # 6: size-1 linker of type 3 (hash >= 2^63)
    add(x, types, linker, pocket=6)                                      # 7: the same linker with pocket rows
    add(x, types, linker, nan=2)                                         # 8: a NaN row: that atom bonds to nothing
    add(x[:7], types[:7], linker[:7])                                    # 9: the linker alone, no fragment
    xh, nm, lm, po = [torch.stack(t) for t in zip(*mols)]
    want, near = oracle_linker_hashes(xh, nm, lm, True, po)
    assert all(m > 0.01 for m in near)
    assert len(set(want[:4])) == 1 and want[4] == 0 and want[7] == want[0] == want[9]
    assert want[6] >= 1 << 63 and want[5] < 1 << 63 and want[8] != want[0]
    distinct = sorted(set(want))
    sets = planted_sets(distinct, sorted(set(want) - {min(want), max(want)})[0])
    assert_check_matches(xh, nm, lm, po, True, want, sets)
    # without drop_pocket the pocket rows of molecule 7 are linker atoms: its L changes, the others' do not
    want_all, _ = oracle_linker_hashes(xh, nm, lm, True)
    assert want_all[7] != want[7] and want_all[:7] == want[:7]
    assert_check_matches(xh, nm, lm, None, True, want_all, {'big': sets['big']}, [NOVEL, NOVEL | UNIQUE, NOVEL | CV])


@pytest.mark.gpu
@pytest.mark.parametrize("N", [4000, 8192])
def test_the_check_launch_holds_up_to_the_checks_row_limit(N):
    """Every row an atom: chains of 64 carbons 1.5 A apart; the linker is 16 whole chains and a 3-carbon piece, spread over
    the batch (at N = 8192 more bonds than the shared-memory CSR holds, so atoms rescan from global memory). Molecule 1 is
    molecule 0 with its rows reversed; molecule 2 also marks some pocket rows as linker rows, which drop_pocket keeps out."""
    Lc = 64
    k = torch.arange(N)
    xh = torch.zeros(3, N, 3 + 9)
    xh[0, :, 0] = 1.5 * (k % Lc).float()
    xh[0, :, 1] = 10.0 * (k // Lc % 32).float()
    xh[0, :, 2] = 10.0 * (k // (Lc * 32)).float()
    xh[0, :, 3] = 1.0
    lm = torch.zeros(3, N)
    chains = list(range(0, 2 * 16, 2))
    for c in chains:
        lm[0, c * Lc:(c + 1) * Lc] = 1.0
    lm[0, 41 * Lc:41 * Lc + 3] = 1.0
    xh[1], lm[1] = xh[0].flip(0), lm[0].flip(0)
    xh[2], lm[2] = xh[0], lm[0]
    po = torch.zeros(3, N)
    po[2, 50 * Lc:52 * Lc] = 1.0                                          # pocket rows ...
    lm[2, 50 * Lc:52 * Lc] = 1.0                                          # ... with linker_mask set
    nm = torch.ones(3, N, dtype=torch.int8)
    n = int(lm[0].sum())
    o = np.zeros((n, n), np.int8)
    rows = lm[0].nonzero().flatten().tolist()
    for a in range(n - 1):
        if rows[a + 1] == rows[a] + 1 and rows[a + 1] % Lc:
            o[a, a + 1] = o[a + 1, a] = 1
    L0 = gho.graph_hash([C] * n, o)
    piece = gho.graph_hash([C] * 3, np.array([[0, 1, 0], [1, 0, 1], [0, 1, 0]]))
    sets = {'empty': torch.zeros(0, dtype=torch.int64), 'planted': mb.sort_unsigned(planted_set([L0, piece], 1 << 20, 1)),
            'other': mb.sort_unsigned(planted_set([piece, piece ^ 1], 1 << 10, 2))}
    for require in (NOVEL, NOVEL | UNIQUE):
        for name, known in sets.items():
            passed, L, H = novel_check(xh, nm, lm, known, True, require, po)
            assert L.tolist() == [gho.as_int64(L0)] * 3, (N, require, name)
            assert [bool(v & NOVEL) for v in passed.tolist()] == [name != 'planted'] * 3, (N, require, name)
            if H is not None:
                assert H[0] == H[1] and H[0] != H[2]                     # molecule 2 drops its pocket rows from H too


def planted_set(planted, size, seed):
    """A (size,) int64 set holding the hashes `planted` (ints mod 2^64), its smallest and largest value among them, filled
    with random values strictly between the two, shuffled."""
    lo, hi = min(planted), max(planted)
    rng = np.random.default_rng(seed)
    fill = size - len(planted)
    if hi - lo > 1 and fill > 0:
        r = rng.integers(0, 1 << 63, size=fill, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=fill, dtype=np.uint64)
        vals = (r % np.uint64(hi - lo - 1)) + np.uint64(lo + 1)
    else:
        vals = np.full(max(fill, 0), lo, np.uint64)
    allv = np.concatenate([np.array(planted, np.uint64), vals]).view(np.int64)
    return torch.from_numpy(allv[rng.permutation(len(allv))].copy())


def linker_hashes_of(ddpm, kw, chain0):
    po = tur.pocket_only(ddpm, kw)
    return mb.linker_hashes(chain0, kw['node_mask'], kw['linker_mask'], ddpm.edm.is_geom, po).cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", [("fc", "simt"), ("pocket_4A", "auto")])
def test_novel_bits_against_the_oracle_with_planted_sets(case, impl):
    """Report-only calls (no rounds): the chain is the plain call's, last_linker_hashes the oracle's L, and the NOVEL bit is
    'L not in the set' for sets of size 0, 1 and 2^20 with planted members at both ends, above and below 2^63."""
    ddpm, kw, _ = tcr_build(case, impl, rows=32)
    edm = ddpm.edm
    B = 32
    seeds = list(range(501, 501 + B))
    base = edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    L = linker_hashes_of(ddpm, kw, base[0])
    want, _ = oracle_linker_hashes(base[0], kw['node_mask'], kw['linker_mask'], edm.is_geom, tur.pocket_only(ddpm, kw))
    assert [int(h) for h in L] == [gho.as_int64(w) for w in want]
    distinct = sorted(set(unsigned(L)))
    print(f"{case}/{impl}: {len(distinct)} distinct linker hashes, {sum(v >= 1 << 63 for v in distinct)} of them >= 2^63")
    assert len(distinct) >= 3
    sets = {'empty': torch.zeros(0, dtype=torch.int64), 'one': torch.tensor([gho.as_int64(distinct[1])])}
    planted = distinct[::2]
    sets['big'] = planted_set(planted, 1 << 20, 0)
    sets['ends'] = planted_set([distinct[0], distinct[-1]], 1 << 12, 1)
    for name, known in sets.items():
        edm.known_linkers = known
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True)
        assert torch.equal(chain, base), name
        assert torch.equal(edm.last_linker_hashes, L), name
        members = set(unsigned(known))
        assert edm.last_novel.tolist() == [v not in members for v in unsigned(L)], name
    # every combination with the other checks reports what each reports alone
    others = {'require_connected': 'last_connected', 'require_valid': 'last_valid', 'require_unique': 'last_unique'}
    if case.startswith("pocket"):
        others['require_clash_free'] = 'last_clash_free'
    alone = {}
    for k, attr in others.items():
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, **{k: True})
        alone[k] = getattr(edm, attr).clone()
    edm.known_linkers = sets['big']
    edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True)
    novel = edm.last_novel.clone()
    names = list(others)
    for mask in range(1, 1 << len(names)):
        flags = {k: True for i, k in enumerate(names) if mask >> i & 1}
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True, **flags)
        assert torch.equal(chain, base) and torch.equal(edm.last_novel, novel), flags
        for k in flags:
            if k != 'require_unique':
                assert torch.equal(getattr(edm, others[k]), alone[k]), (flags, k)
        if 'require_unique' in flags:                                    # eligibility includes the NOVEL bit
            passed = [sum(bit for k, bit in (('require_connected', 1), ('require_valid', 2), ('require_clash_free', 4))
                          if k in flags and bool(alone[k][b])) | (NOVEL if novel[b] else 0) for b in range(B)]
            require = UNIQUE | NOVEL | sum(bit for k, bit in (('require_connected', 1), ('require_valid', 2),
                                                               ('require_clash_free', 4)) if k in flags)
            v = gho.verdict(unsigned(edm.last_graph_hashes), [0] * B, passed, require)
            assert edm.last_unique.tolist() == [bool(w & UNIQUE) for w in v], flags


def tcr_build(case, impl, rows=16):
    """The copies of tur.build_copies: one input, a single linker atom, so linker graphs repeat across seeds. The end-to-end
    tests keep tur's 16 rows, whose step coefficients are those of a molecule sampled alone (torch's CPU kernels round the
    table differently for some batch sizes), so a resampled row replays alone bit for bit."""
    return tur.build_copies(case, impl, rows=rows)


@pytest.mark.gpu
def test_known_linkers_is_the_sorted_distinct_linker_hashes_of_the_items():
    """ZINC-shaped items and MOAD-shaped ones (pocket_mask, pocket rows before the linker rows): the set equals the sorted,
    de-duplicated linker_hashes of the collated batch, a pocket item hashes its linker rows only, and the batch size of
    the collation changes nothing."""
    from difflinker_b200 import synthetic
    from difflinker_b200.batching import collate
    d = tcr.dev()
    items = synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=40)
    items += items[:5]                                                   # repeats: one hash each
    keys = ('positions', 'one_hot', 'fragment_mask', 'linker_mask')
    batch = collate([{k: it[k].to(d) for k in keys} for it in items])
    L = mb.linker_hashes(torch.cat([batch['positions'], batch['one_hot']], 2), batch['atom_mask'], batch['linker_mask'],
                         False)
    want = sorted(set(unsigned(L)))
    for bs in (1, 7, 256):
        got = mb.known_linkers(items, False, batch_size=bs)
        assert got.device.type == 'cuda' and unsigned(got.cpu()) == want, bs
    pocket = tcr.small_fragment_items("pocket_4A", 9)                    # 12 pocket rows, then 0-2 linker rows
    bare = []
    for it in pocket:
        keep = it['pocket_mask'] == 0
        bare.append({k: it[k][keep] for k in keys})
    got = mb.known_linkers(pocket, True, batch_size=4)
    assert unsigned(got.cpu()) == unsigned(mb.known_linkers(bare, True, batch_size=4).cpu())
    want = set()
    for it in pocket:                                                    # the oracle on each item's linker rows
        rows = it['linker_mask'] != 0
        o, _ = gho.bond_order_matrix(it['positions'][rows].numpy(), it['one_hot'][rows].argmax(1).numpy(),
                                     [t.numpy() for t in mb.threshold_tables(True)])
        want.add(gho.graph_hash(it['one_hot'][rows].argmax(1).numpy(), o))
    assert unsigned(got.cpu()) == sorted(want)


# ---- GPU: the sampler, end to end --------------------------------------------------------------------------------------

ROUNDS = 3
END_CASES = [(g, impl) for g in ("fc", "pocket_4A") for impl in ("simt", "auto")]


def plant(L, rows):
    """known_linkers holding the linker hashes of `rows`, unsorted and with a duplicate."""
    vals = [int(L[b]) for b in rows]
    return torch.tensor(vals[::-1] + vals[:1], dtype=torch.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", END_CASES)
@pytest.mark.parametrize("extra", [{}, {'require_connected': True}, {'require_valid': True}, {'require_unique': True}])
def test_rounds_resample_only_the_known_linkers(case, impl, extra):
    ddpm, kw, _ = tcr_build(case, impl)
    edm = ddpm.edm
    B = 16
    seeds = list(range(701, 701 + B))
    base = edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    L = linker_hashes_of(ddpm, kw, base[0])
    counts = {}
    for v in L.tolist():
        counts[v] = counts.get(v, 0) + 1
    common = max(counts, key=counts.get)                                 # plant the most common linker
    edm.known_linkers = plant(L, [b for b in range(B) if int(L[b]) == common][:1])
    known = set(unsigned(edm.known_linkers))
    planted_rows = [b for b in range(B) if int(L[b]) == common]
    assert 0 < len(planted_rows) < B, counts
    # attempt 0 verdicts, report-only
    edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True, **extra)
    first = edm.last_novel.clone()
    for k, attr in (('require_connected', 'last_connected'), ('require_valid', 'last_valid'),
                    ('require_unique', 'last_unique')):
        if k in extra:
            first &= getattr(edm, attr)
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, nan_retries=ROUNDS, require_novel=True, **extra)
    novel, Lr, attempts, used = edm.last_novel, edm.last_linker_hashes, edm.last_attempts, edm.last_seeds
    assert torch.isfinite(chain).all()
    assert torch.equal(Lr, linker_hashes_of(ddpm, kw, chain[0]))
    assert novel.tolist() == [v not in known for v in unsigned(Lr)]      # every row with the bit has L outside the set
    good = first.nonzero().flatten().tolist()
    assert torch.equal(chain[:, good], base[:, good]) and all(int(attempts[b]) == 0 for b in good)
    assert not any(b in good for b in planted_rows)
    assert any(int(attempts[b]) > 0 for b in planted_rows)
    if 'require_unique' in extra:
        kept = [b for b in range(B) if novel[b] and edm.last_unique[b]]
        assert len({int(edm.last_graph_hashes[b]) for b in kept}) == len(kept)
    for b in range(B):
        assert int(used[b]) == retry_seed(seeds[b], int(attempts[b]))
        if int(attempts[b]) > 0:                                         # a resampled row is its molecule sampled alone
            alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert tcr.same(chain[:, b], alone[:, 0], impl), b
    print(f"{case}/{impl}/{sorted(extra)}: planted {len(planted_rows)} rows; novel {int(novel.sum())} of {B} after "
          f"{ROUNDS} rounds; attempts {attempts.tolist()}")


@pytest.mark.gpu
def test_redrawn_sizes_are_hashed_with_the_sub_batch_linker_rows():
    ddpm, kw, data = tcr_build("fc", "simt")
    edm = ddpm.edm
    B = 16
    seeds = list(range(801, 801 + B))
    chain0, nm0 = ddpm.sample_chain(data, keep_frames=2, seeds=seeds, linker_sizes=(1, 3))
    sizes0 = edm.last_sizes.clone()
    n_frag = int(data['fragment_mask'][0].sum())

    def linker_of(nm):
        rows = torch.arange(nm.reshape(B, -1).shape[1], device=nm.device)[None, :]
        return (rows >= n_frag).float() * (nm.reshape(B, -1) != 0).float()
    L0 = mb.linker_hashes(chain0[0], nm0, linker_of(nm0), edm.is_geom).cpu()
    edm.known_linkers = plant(L0, list(range(12)))                      # most rows fail: long sub-batches
    known = set(unsigned(edm.known_linkers))
    chain, nm = ddpm.sample_chain(data, keep_frames=2, seeds=seeds, linker_sizes=(1, 3), nan_retries=ROUNDS,
                                  require_novel=True)
    sizes, Lr, novel = edm.last_sizes, edm.last_linker_hashes, edm.last_novel
    assert (nm.reshape(B, -1).ne(0).sum(1).cpu() == n_frag + sizes).all()
    assert torch.equal(Lr, mb.linker_hashes(chain[0], nm, linker_of(nm), edm.is_geom).cpu())
    assert novel.tolist() == [v not in known for v in unsigned(Lr)]
    assert int(novel.sum()) > int(sum(v not in known for v in unsigned(L0)))
    attempts = edm.last_attempts
    assert torch.isfinite(chain).all() and (attempts > 0).any()
    # Round a's sub-batch holds the rows still failing after round a - 1, those whose last attempt is >= a (no row
    # diverges), in row order. Some row was taken at a size above the attempt-0 size of the full batch's row at its
    # sub-batch index, so a check reading the full batch's linker_mask there would see fewer linker atoms and another L.
    index = lambda b: sum(1 for c in range(b) if int(attempts[c]) >= int(attempts[b]))
    assert any(int(attempts[b]) > 0 and int(sizes0[index(b)]) < int(sizes[b]) for b in range(B)), (attempts, sizes0, sizes)


@pytest.mark.gpu
def test_sample_many_and_a_split_equal_the_plain_calls():
    ddpm, kw, _ = tcr_build("fc", "simt")
    edm = ddpm.edm
    B = 16
    seeds = list(range(901, 901 + B))
    base = edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    edm.known_linkers = plant(linker_hashes_of(ddpm, kw, base[0]), [0, 3])
    opts = dict(keep_frames=2, nan_retries=ROUNDS, require_novel=True, require_connected=True)
    want = edm.sample_chain(**kw, seeds=seeds, **opts)
    novel, attempts, used = edm.last_novel, edm.last_attempts, edm.last_seeds
    edm.devices = [0, 0]
    try:
        got = edm.sample_chain(**kw, seeds=seeds, **opts)
    finally:
        edm.devices = None
    assert torch.equal(got, want) and torch.equal(edm.last_novel, novel) and torch.equal(edm.last_attempts, attempts)
    assert torch.equal(edm.last_seeds, used)
    cuts = [(0, 6), (6, B)]
    reqs = [tcr.take(kw, list(range(lo, hi))) for lo, hi in cuts]
    outs = edm.sample_many(reqs, seeds=[seeds[lo:hi] for lo, hi in cuts], **opts)
    for k, (lo, hi) in enumerate(cuts):
        alone = edm.sample_chain(**reqs[k], seeds=seeds[lo:hi], **opts)
        assert torch.equal(outs[k], alone), k
        assert torch.equal(edm.last_novel_many[k], edm.last_novel)
        assert torch.equal(edm.last_attempts_many[k], edm.last_attempts)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fc", "pocket_4A"])
def test_exclude_hashes_extends_uniqueness_across_calls(case):
    ddpm, kw, _ = tur.build_copies(case, "simt")
    edm = ddpm.edm
    B = len(tur.SEEDS)
    edm.sample_chain(**kw, keep_frames=2, seeds=tur.SEEDS, nan_retries=tur.ROUNDS, require_unique=True)
    h1 = edm.last_graph_hashes.clone()
    taken = set(unsigned(h1[edm.last_unique]))
    seeds2 = [s + 1000 for s in tur.SEEDS]
    # report-only: the verdict treats the seen hashes as keepers
    base2 = edm.sample_chain(**kw, keep_frames=2, seeds=seeds2)
    r0 = edm.sample_chain(**kw, keep_frames=2, seeds=seeds2, require_unique=True, exclude_hashes=h1)
    assert torch.equal(r0, base2)
    h0, u0 = edm.last_graph_hashes, edm.last_unique.clone()
    seen = sorted(set(unsigned(h1)))
    hs = seen + unsigned(h0)
    want = gho.verdict(hs, [0] * len(hs), [UNIQUE] * len(seen) + [0] * B, UNIQUE,
                       candidates=list(range(len(seen), len(hs))))
    assert u0.tolist() == [bool(w & UNIQUE) for w in want[len(seen):]]
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds2, nan_retries=tur.ROUNDS, require_unique=True,
                             exclude_hashes=h1)
    h2, u2, attempts = edm.last_graph_hashes, edm.last_unique, edm.last_attempts
    kept = u2.nonzero().flatten().tolist()
    assert kept and not any(unsigned(h2[[b]])[0] in set(seen) for b in kept)
    assert len({int(h2[b]) for b in kept}) == len(kept)
    good = u0.nonzero().flatten().tolist()
    assert torch.equal(chain[:, good], base2[:, good]) and all(int(attempts[b]) == 0 for b in good)
    print(f"{case}: call 1 kept {len(taken)} hashes; call 2 unique {len(good)} at attempt 0, {len(kept)} after rounds")


@pytest.mark.gpu
def test_the_engine_refuses_unsorted_sets_and_unknown_bits(monkeypatch):
    ddpm, kw, _ = tcr_build("fc", "simt")
    edm = ddpm.edm
    seeds = list(range(1, 17))
    edm.known_linkers = torch.tensor([5, 1, -3], dtype=torch.int64)
    monkeypatch.setattr(edm_mod, "sort_unsigned", lambda t: t)           # hand the engine the set as it is
    with pytest.raises(_native.NativeError, match="known is not in ascending unsigned order"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True)
    monkeypatch.setattr(edm_mod, "sort_unsigned", lambda t: torch.sort(t).values)   # a signed sort
    with pytest.raises(_native.NativeError, match="not in ascending unsigned order"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_novel=True)
    with pytest.raises(_native.NativeError, match="seen is not in ascending"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_unique=True, exclude_hashes=torch.tensor([2, -1]))
    monkeypatch.undo()
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    # a real two-molecule call's buffers, so that nothing but the refusal decides the outcome
    d = tcr.dev()
    B, N, T, F = 2, 4, edm.T, edm.in_node_nf
    Cn = edm.dynamics.context_node_nf
    xh, fm, lm = torch.zeros(B, N, 3 + F, device=d), torch.zeros(B, N, device=d), torch.ones(B, N, device=d)
    nm, ctx = torch.ones(B, N, dtype=torch.int8, device=d), torch.zeros(B, N, max(Cn, 1), device=d)
    sd, used = torch.arange(B, dtype=torch.int64, device=d), torch.empty(B, dtype=torch.int64, device=d)
    chain, flags = torch.empty(1, B, N, 3 + F, device=d), torch.zeros(B, dtype=torch.int32, device=d)
    attempts, passed = torch.empty(B, dtype=torch.int32, device=d), torch.empty(B, dtype=torch.int32, device=d)
    lh = torch.empty(B, dtype=torch.int64, device=d)
    coef, norm = edm.step_coefficients(1, B), edm._norm()
    tables = [t.to(d) for t in mb.check_tables(edm.is_geom, NOVEL)]
    host = torch.tensor([1, 2], dtype=torch.int64).pin_memory()          # sorted, in (pinned) host memory
    for require, sets, why in ((32 | 1, None, b"require"), (NOVEL, _native.DLHashSets(None, 2, None, 0), b"null sets"),
                               (NOVEL, _native.DLHashSets(None, -1, None, 0), b"n_known"),
                               (NOVEL, _native.DLHashSets(host.data_ptr(), 2, None, 0), b"device (or managed) memory")):
        ck = _native.DLMoleculeChecks.of(require, tables)
        st = lib.dl_sample_chain_retry_sets(
            eng, 0, B, N, T, 1, xh.data_ptr(), nm.data_ptr(), fm.data_ptr(), lm.data_ptr(), None,
            ctx.data_ptr() if Cn else None, sd.data_ptr(), coef, norm, chain.data_ptr(), flags.data_ptr(), 1,
            used.data_ptr(), attempts.data_ptr(), ck, sets, passed.data_ptr(), lh.data_ptr(), None, None,
            torch.cuda.current_stream(d).cuda_stream)
        assert st == -1 and why in lib.dl_last_error(), why


@pytest.mark.gpu
def test_without_the_bit_and_sets_the_call_launches_what_it_launched_before():
    ddpm, kw, _ = tcr_build("fc", "simt")
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    seeds = list(range(1, 17))
    counts = []
    for extra in ({}, {'require_novel': False}, {'exclude_hashes': None}):
        n0 = int(lib.dl_launch_count(eng))
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, nan_retries=0, require_connected=True, **extra)
        counts.append(int(lib.dl_launch_count(eng)) - n0)
    edm.known_linkers = torch.tensor([], dtype=torch.int64)
    n0 = int(lib.dl_launch_count(eng))
    edm.sample_chain(**kw, keep_frames=2, seeds=seeds, nan_retries=0, require_connected=True, require_novel=True)
    counts.append(int(lib.dl_launch_count(eng)) - n0)
    assert counts[0] == counts[1] == counts[2] == counts[3]             # the bit shares the check launch
