"""Ring sizes in the recovery rounds: `sample_chain(..., require_ring_sizes=True)` with `allowed_ring_sizes`, and
dl_sample_chain_retry, dl_set_ring_sizes, dl_last_ring_sizes and dl_ring_check with DL_CHECK_RINGS.

A molecule's ring-size mask has bit k when some bond with a linker end has a smallest ring of k atoms, on the bond graph of
all its checked atoms (stated at DL_CHECK_RINGS in the header); ring_oracle restates it with a Python BFS. CPU tests pin the
oracle to purpose-built molecules, and check the refusals, the binding and the header; the GPU tests check the kernel
against the oracle, on those molecules and on sampled batches, and the sampler end to end."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, distributed, molecule_builder as mb
from difflinker_b200.edm import retry_seed
import ring_oracle as ro
import test_connected_resampling as tcr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RINGS = 32
FAR = 60.0                                  # A: padding rows, out of every bond's reach


def polygon(k, side, centre=(0.0, 0.0, 0.0)):
    """A regular k-gon of the given side in the xy-plane."""
    r = side / (2 * np.sin(np.pi / k))
    a = 2 * np.pi * np.arange(k) / k
    return np.stack([r * np.cos(a), r * np.sin(a), np.zeros(k)], 1) + np.asarray(centre)


def kekule_benzene():
    """An equiangular hexagon of alternating 1.33 A (double) and 1.47 A (single) sides."""
    p, out = np.zeros(3), []
    for i, side in enumerate([1.33, 1.47] * 3):
        out.append(p.copy())
        a = np.pi / 3 * i
        p = p + side * np.array([np.cos(a), np.sin(a), 0.0])
    return np.array(out)


def norbornane():
    """Bicyclo[2.2.1]heptane: bridgeheads 0 and 3, two-carbon bridges 1-2 and 4-5, the one-carbon bridge 6."""
    h = np.sqrt(1.54 ** 2 - 1.125 ** 2)
    y = np.sqrt(1.54 ** 2 - 0.345 ** 2 - 0.25)
    return np.array([[-1.125, 0, 0], [-0.78, y, -0.5], [0.78, y, -0.5], [1.125, 0, 0], [0.78, -y, -0.5],
                     [-0.78, -y, -0.5], [0, 0, h]])


def spiro_octane():
    """Spiro[2.5]octane: a 1.53 A hexagon whose vertex 0 (the spiro atom) carries a perpendicular cyclopropane."""
    hexa = polygon(6, 1.53) - polygon(6, 1.53)[0]
    x = np.sqrt(1.51 ** 2 - 0.755 ** 2)
    return np.concatenate([hexa, [[x, 0, 0.755], [x, 0, -0.755]]])


def edges_of(*cycles):
    """The undirected edges of the given atom cycles."""
    out = set()
    for c in cycles:
        for i in range(len(c)):
            out.add(tuple(sorted((c[i], c[(i + 1) % len(c)]))))
    return out


def molecules():
    """(name, positions (n,3), linker flags (n,), pocket flags (n,), valid rows (n,), bonds, expected mask)."""
    mols = []

    def add(name, pos, bonds, want, linker=None, pocket=None, valid=None):
        pos = np.asarray(pos, np.float32)
        n = pos.shape[0]
        mols.append((name, pos, np.ones(n, bool) if linker is None else np.asarray(linker, bool),
                     np.zeros(n, bool) if pocket is None else np.asarray(pocket, bool),
                     np.ones(n, bool) if valid is None else np.asarray(valid, bool), bonds, want))
    add("cyclopropane", polygon(3, 1.51), edges_of(range(3)), 1 << 3)
    cube = np.array([[i, j, k] for i in (0, 1) for j in (0, 1) for k in (0, 1)], np.float32) * 1.57
    add("cubane", cube, {(a, b) for a in range(8) for b in range(a + 1, 8) if bin(a ^ b).count("1") == 1}, 1 << 4)
    add("cyclopentane", polygon(5, 1.54), edges_of(range(5)), 1 << 5)
    add("norbornane", norbornane(), edges_of(range(6)) | {(0, 6), (3, 6)}, 1 << 5)
    add("Kekule benzene", kekule_benzene(), edges_of(range(6)), 1 << 6)
    h1 = polygon(6, 1.45)
    h2 = h1 + h1[0] + h1[1]                 # h1 mirrored across its bond 0-1: its vertices 3 and 4 are h1's 1 and 0
    add("naphthalene", np.concatenate([h1, h2[[0, 1, 2, 5]]]), edges_of(range(6), [6, 7, 8, 1, 0, 9]), 1 << 6)
    add("spiro[2.5]octane", spiro_octane(), edges_of(range(6), [0, 6, 7]), (1 << 3) | (1 << 6))
    add("12-membered macrocycle", polygon(12, 1.52), edges_of(range(12)), 1 << 12)
    add("70-membered macrocycle", polygon(70, 1.52), edges_of(range(70)), 1 << 63)
    ring = polygon(6, 1.52)
    add("ring closed between linker and fragment", ring, edges_of(range(6)), 1 << 6, linker=[1, 1, 1, 0, 0, 0])
    tail = np.concatenate([ring, ring[[0]] * (1 + 1.52 / np.linalg.norm(ring[0])),
                           ring[[0]] * (1 + 3.0 / np.linalg.norm(ring[0]))])
    add("ring wholly inside a fragment", tail, edges_of(range(6)) | {(0, 6), (6, 7)}, 0, linker=[0] * 6 + [1, 1])
    chain = np.stack([1.25 * np.arange(6.0), 0.8 * (np.arange(6) % 2), np.zeros(6)], 1)
    add("acyclic linker", chain, {(i, i + 1) for i in range(5)}, 0)
    # a pocket atom closes the ring: dropped with the pocket, the linker is a chain
    add("pocket ring through a linker atom", polygon(5, 1.54), {(0, 1), (1, 2), (2, 3)}, 0,
        pocket=[0, 0, 0, 0, 1])
    add("padding inside a ring", polygon(6, 1.52), {(0, 1), (1, 2), (4, 5), (0, 5)}, 0,
        valid=[1, 1, 1, 0, 1, 1])
    nan = polygon(4, 1.52)
    nan[2] = np.nan
    add("a NaN atom in a ring", nan, {(0, 1), (0, 3)}, 0)
    return mols


def pack(mols, N, F=8):
    """A padded (B,N,3+F) batch of the molecules (carbon unless stated), with node, linker and pocket masks."""
    B = len(mols)
    xh = torch.zeros(B, N, 3 + F)
    xh[:, :, :3] = FAR
    xh[:, :, 3] = 1.0
    nm, lm, po = torch.zeros(B, N, dtype=torch.int8), torch.zeros(B, N), torch.zeros(B, N)
    for b, (_, pos, linker, pocket, valid, _, _) in enumerate(mols):
        n = pos.shape[0]
        xh[b, :n, :3] = torch.from_numpy(pos)
        nm[b, :n] = torch.from_numpy(valid.astype(np.int8))
        lm[b, :n] = torch.from_numpy(linker.astype(np.float32))
        po[b, :n] = torch.from_numpy(pocket.astype(np.float32))
    return xh, nm, lm, po


# ---- CPU --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", [m[0] for m in molecules()])
def test_oracle_on_purpose_built_molecules(name):
    """The oracle's bond graph is the intended one, then its mask is the intended one."""
    (_, pos, linker, pocket, valid, bonds, want), = [m for m in molecules() if m[0] == name]
    keep = valid & ~pocket
    rows = np.nonzero(keep)[0]
    adj = ro.bonds(pos[rows], np.zeros(len(rows), int), False)
    got = {(int(rows[i]), int(rows[j])) for i, j in zip(*np.nonzero(np.triu(adj)))}
    assert got == bonds, name
    assert ro.ring_mask(adj, linker[rows]) == want, name
    xh, nm, lm, po = pack([m for m in molecules() if m[0] == name], N=80)
    assert ro.batch_masks(xh, nm, lm, False, po) == [want]


def test_ring_size_mask_takes_ints_from_3_to_63():
    assert mb.ring_size_mask([5, 6, 63]) == (1 << 5) | (1 << 6) | (1 << 63)
    assert mb.ring_size_mask([]) == 0 and mb.ring_size_mask(range(5, 7)) == 96
    for bad in ([2], [64], [5.0], [True], ["6"]):
        with pytest.raises(ValueError, match="ring sizes"):
            mb.ring_size_mask(bad)


@pytest.mark.parametrize("inpainting", [False, True])
def test_require_ring_sizes_refuses_what_cannot_recover_and_names_what_is_missing(inpainting):
    ddpm, kw = tcr._cpu_model(inpainting)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(1, B + 1))
    assert edm.require_ring_sizes is False and edm.allowed_ring_sizes is None
    assert edm.last_ring_sizes_ok is None and edm.last_ring_sizes is None
    assert edm.last_ring_sizes_ok_many is None and edm.last_ring_sizes_many is None
    with pytest.raises(ValueError, match="require_ring_sizes needs the ring sizes to allow.*allowed_ring_sizes"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_ring_sizes=True)
    edm.allowed_ring_sizes = [2, 5]
    with pytest.raises(ValueError, match="ring sizes are ints in"):
        edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_ring_sizes=True)
    edm.allowed_ring_sizes = range(5, 7)
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_ring_sizes"):
            edm.sample_chain(**kw, keep_frames=2, seeds=seeds, require_ring_sizes=bad)
    with pytest.raises(ValueError, match="require_ring_sizes needs per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2, require_ring_sizes=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_ring_sizes=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="require_ring_sizes does not take batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_ring_sizes=True, seeds=seeds, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_ring_sizes needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_ring_sizes=True, seeds=seeds)
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="require_ring_sizes.*replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_ring_sizes=True, seeds=seeds)
    delattr(edm, name)
    with pytest.raises(ValueError, match="sample_many needs CUDA inputs"):
        edm.sample_many([kw], keep_frames=2, seeds=[seeds], require_ring_sizes=True)
    edm.require_ring_sizes = True                                        # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    assert edm.last_ring_sizes_ok is None


def test_ddpm_and_the_sharded_sampler_pass_require_ring_sizes():
    ddpm, _ = tcr._cpu_model()
    from difflinker_b200 import ddpm as ddpm_mod, synthetic
    from difflinker_b200.batching import collate
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append(k.get('require_ring_sizes', 'unset'))
    ddpm.edm.sample_many = lambda reqs, **k: seen.append(k.get('require_ring_sizes', 'unset')) or [None] * len(reqs)
    ddpm.sample_chain(data, keep_frames=2, require_ring_sizes=True)
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, require_ring_sizes=False)
    ddpm.sample_many([data], keep_frames=2, seeds=[[1, 2, 3]], require_ring_sizes=True)
    ddpm_mod.sample_many(ddpm, [data], keep_frames=2, seeds=[[1, 2, 3]])
    distributed.sample_chain_sharded(ddpm, data, keep_frames=2, seeds=[1, 2, 3], require_ring_sizes=True)
    assert seen == [True, 'unset', False, True, 'unset', True]


def test_binding_and_a_c99_caller_get_the_new_entries_and_refusals(tmp_path):
    lib = _native.load_library()
    assert _native.CHECK_RINGS == RINGS
    for name in ("dl_ring_check", "dl_set_ring_sizes", "dl_last_ring_sizes"):
        assert name in _native.SYMBOLS and getattr(lib, name).argtypes == _native.SYMBOLS[name][1]
    assert lib.dl_set_ring_sizes(None, 1 << 6) == -1 and b"null engine" in lib.dl_last_error()
    assert lib.dl_last_ring_sizes(None, 2, 1, None) == -1
    for args, why in (((0, 4, 8, 1, 1, 11, 1, 1, None, 0, 0, 64, 1, None, None), b"B and N"),
                      ((1, 8193, 8, 1, 1, 11, 1, 1, None, 0, 0, 64, 1, None, None), b"8192"),
                      ((1, 4, 9, 1, 1, 11, 1, 1, None, 0, 0, 64, 1, None, None), b"n_types"),
                      ((1, 4, 8, 1, 1, 11, 1, 1, None, 0, 0, 4, 1, None, None), b"bits 0-2"),
                      ((1, 4, 8, None, 1, 11, 1, 1, None, 0, 0, 64, 1, None, None), b"invalid argument"),
                      ((1, 4, 8, 1, 1, 11, 1, 1, None, 0, 1, 64, 1, None, None), b"invalid argument")):
        assert lib.dl_ring_check(*args) == -1, why
        assert why in lib.dl_last_error() and b"dl_ring_check" in lib.dl_last_error()
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    src = tmp_path / "ring_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  uint64_t used[2], masks[2]; int32_t attempts[2], flags[2], passed[2];\n"
        "  float thr[64] = {0}, xh[22] = {0}; int8_t nm[2] = {0};\n"
        "  dl_molecule_checks ck = {DL_CHECK_CONNECTED | DL_CHECK_RINGS, 8, thr, thr, thr, NULL, NULL};\n"
        "  dl_status a = dl_sample_chain_retry(NULL, DL_SAMPLER_LINKER, 2, 4, 10, 1, NULL, NULL, NULL, NULL, NULL, NULL,\n"
        "                                      NULL, NULL, NULL, NULL, flags, 3, used, attempts, &ck, passed, NULL, NULL,\n"
        "                                      NULL);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  dl_status b = dl_ring_check(2, 4, 8, thr, xh, 11, nm, thr, NULL, 0, 0, (uint64_t)1 << 2, passed, masks, NULL);\n"
        '  printf("%d|%s|", (int)b, dl_last_error());\n'
        "  ck.require = DL_CHECK_RINGS;\n"
        "  dl_status c = dl_molecule_check(2, 4, &ck, xh, 11, nm, NULL, 0, 0, passed, NULL, NULL);\n"
        '  printf("%d|%s|", (int)c, dl_last_error());\n'
        "  ck.require = DL_CHECK_NOVEL | DL_CHECK_RINGS;\n"
        "  dl_status d = dl_novel_check(2, 4, &ck, NULL, xh, 11, nm, thr, NULL, 0, 0, passed, used, NULL, NULL);\n"
        '  printf("%d|%s|", (int)d, dl_last_error());\n'
        "  dl_status e = dl_set_ring_sizes(NULL, 64);\n"
        '  printf("%d|%s\\n", (int)e, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "ring_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe),
                    _native.LIB_PATH, f"-Wl,-rpath,{os.path.dirname(_native.LIB_PATH)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, err_a, b, err_b, c, err_c, d, err_d, e, err_e = res.stdout.strip().split("|", 9)
    assert int(a) == -1 and "null engine" in err_a
    assert int(b) == -1 and "dl_ring_check" in err_b and "bits 0-2" in err_b
    assert int(c) == -1 and "require" in err_c and "dl_ring_check" in err_c
    assert int(d) == -1 and "dl_novel_check" in err_d and "dl_ring_check" in err_d
    assert int(e) == -1 and "null engine" in err_e


# ---- GPU: the kernel, molecule by molecule ------------------------------------------------------------------------------

def kernel_masks(xh, nm, lm, po, is_geom, allowed=0):
    """(masks as Python ints, passed bools) of dl_ring_check on the device."""
    d = tcr.dev()
    passed, masks = mb._ring_check(xh.to(d), nm.to(d), lm.to(d), is_geom, None if po is None else po.to(d), allowed)
    return [int(v) % (1 << 64) for v in masks.cpu().tolist()], ((passed.cpu() & RINGS) != 0).tolist()


def assert_matches_oracle(xh, nm, lm, po, is_geom, allowed=(1 << 5) | (1 << 6)):
    want = ro.batch_masks(xh, nm, lm, is_geom, po)
    got, ok = kernel_masks(xh, nm, lm, po, is_geom, allowed)
    assert got == want
    assert ok == [m & ~allowed == 0 for m in want]
    return want


@pytest.mark.gpu
def test_kernel_matches_the_oracle_on_purpose_built_molecules():
    mols = molecules()
    xh, nm, lm, po = pack(mols, N=80)
    want = assert_matches_oracle(xh, nm, lm, po, False)
    assert want == [m[-1] for m in mols]
    # counted as atoms, the pocket atom closes the five-ring
    i = [m[0] for m in mols].index("pocket ring through a linker atom")
    assert kernel_masks(xh[i:i + 1], nm[i:i + 1], lm[i:i + 1], None, False)[0] == [1 << 5]
    assert mb.ring_sizes_ok(xh.cuda(), nm.cuda(), lm.cuda(), False, [3, 4, 5, 6, 12, 63], po.cuda()).all()


@pytest.mark.gpu
def test_the_check_holds_up_to_the_checks_row_limit():
    """N = 8192: a 12-ring in the first rows, then a clump of 56 mutually bonded atoms whose bond lists do not fit the
    shared-memory CSR (they are found by testing every atom), the rest padding; and a 150-atom ligand ring in a 4000-row
    pocket batch."""
    N = 8192
    xh = torch.zeros(2, N, 11)
    xh[:, :, :3] = FAR
    xh[:, :, 3] = 1.0
    nm, lm = torch.zeros(2, N, dtype=torch.int8), torch.zeros(2, N)
    g = torch.Generator().manual_seed(3)
    xh[0, :12, :3] = torch.from_numpy(polygon(12, 1.52)).float()
    xh[0, 100:156, :3] = 20.0 + 0.6 * torch.rand(56, 3, generator=g)
    nm[0, :12] = nm[0, 100:156] = 1
    lm[0, :12] = 1.0
    lm[0, 140:156] = 1.0
    xh[1, 5000:5007, :3] = torch.from_numpy(polygon(7, 1.52)).float()
    nm[1, 5000:5007] = 1
    lm[1, 5003] = 1.0
    want = assert_matches_oracle(xh, nm, lm, None, False)
    assert want == [(1 << 12) | (1 << 3), 1 << 7]
    N, n_lig = 4000, 150
    xh = torch.zeros(1, N, 12)
    xh[:, :, 3] = 1.0
    nm, lm, po = torch.zeros(1, N, dtype=torch.int8), torch.zeros(1, N), torch.zeros(1, N)
    rows = torch.linspace(3, N - 2, n_lig).long()
    xh[0, :, :3] = 80.0 + 20.0 * torch.rand(N, 3, generator=g)
    nm[0, :3990] = 1
    po[0, :3990] = 1.0
    xh[0, rows, :3] = torch.from_numpy(polygon(n_lig, 1.52)).float()
    nm[0, rows], po[0, rows], lm[0, rows[:20]] = 1, 0.0, 1.0
    assert assert_matches_oracle(xh, nm, lm, po, True) == [1 << 63]


def sampled(case, impl, rows=16):
    ddpm, kw = tcr.build(case, impl, rows=rows)
    edm = ddpm.edm
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=list(range(1, rows + 1)))
    po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
    return ddpm, kw, chain[0], po


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fc", "pocket_4A", "fc_inpainting"])
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_kernel_matches_the_oracle_on_sampled_batches(case, impl):
    ddpm, kw, chain0, po = sampled(case, impl)
    want = assert_matches_oracle(chain0, kw['node_mask'], kw['linker_mask'], po, ddpm.edm.is_geom)
    print(f"{case}/{impl}: ring masks {[hex(m) for m in want]}")


# ---- GPU: the sampler, end to end ---------------------------------------------------------------------------------------

ALLOWED = [5, 6]
SEEDS = list(range(1, 17))


def oracle_ok(ddpm, kw, chain0):
    po = kw['context'][..., -1] if ddpm.edm.dynamics.graph_type != 'FC' else None
    masks = ro.batch_masks(chain0, kw['node_mask'], kw['linker_mask'], ddpm.edm.is_geom, po)
    allowed = mb.ring_size_mask(ALLOWED)
    return masks, [m & ~allowed == 0 for m in masks]


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", tcr.CASES)
def test_rounds_resample_only_the_molecules_with_unwanted_rings(case, impl):
    ddpm, kw = tcr.build(case, impl, rows=len(SEEDS))
    edm = ddpm.edm
    edm.allowed_ring_sizes = ALLOWED
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    r0 = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_ring_sizes=True)
    ok0 = edm.last_ring_sizes_ok
    assert torch.equal(r0, base) and ok0.dtype == torch.bool and ok0.shape == (B,)
    masks0, want0 = oracle_ok(ddpm, kw, base[0])
    assert ok0.tolist() == want0 and [int(m) % (1 << 64) for m in edm.last_ring_sizes.tolist()] == masks0
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=4, require_ring_sizes=True)
    ok, masks, attempts, used = edm.last_ring_sizes_ok, edm.last_ring_sizes, edm.last_attempts, edm.last_seeds
    want_masks, want_ok = oracle_ok(ddpm, kw, chain[0])
    assert ok.tolist() == want_ok and [int(m) % (1 << 64) for m in masks.tolist()] == want_masks
    healthy = [b for b in range(B) if want0[b]]
    assert torch.equal(chain[:, healthy], base[:, healthy]) and all(int(attempts[b]) == 0 for b in healthy)
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
        if int(attempts[b]) > 0:                                         # a resampled row replays alone from its seed
            alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert tcr.same(chain[:, b], alone[:, 0], impl), b
    print(f"{case}/{impl}: allowed {ALLOWED}: {sum(want0)} of {B} rows pass at attempt 0, {int(ok.sum())} after the "
          f"rounds; masks {[hex(m) for m in want_masks]}")


@pytest.mark.gpu
@pytest.mark.parametrize("other", ["require_connected", "require_valid", "require_clash_free", "require_unique",
                                   "require_novel"])
def test_the_bit_combines_with_each_other_check(other):
    case = "pocket_4A" if other == "require_clash_free" else "fc"
    ddpm, kw = tcr.build(case, "simt", rows=len(SEEDS))
    edm = ddpm.edm
    edm.allowed_ring_sizes = ALLOWED
    edm.known_linkers = torch.tensor([], dtype=torch.int64)
    attr = {"require_connected": "last_connected", "require_valid": "last_valid", "require_clash_free": "last_clash_free",
            "require_unique": "last_unique", "require_novel": "last_novel"}[other]
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, **{other: True})
    other_alone = getattr(edm, attr)
    alone_bits = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_ring_sizes=True)
    rings_alone = edm.last_ring_sizes_ok
    both = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_ring_sizes=True, **{other: True})
    assert torch.equal(both, base) and torch.equal(both, alone_bits)
    assert torch.equal(edm.last_ring_sizes_ok, rings_alone)
    if other != "require_unique":           # the uniqueness verdict counts the other required bits, so it may change
        assert torch.equal(getattr(edm, attr), other_alone)
    chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=3, require_ring_sizes=True, **{other: True})
    _, want_ok = oracle_ok(ddpm, kw, chain[0])
    assert edm.last_ring_sizes_ok.tolist() == want_ok


@pytest.mark.gpu
def test_a_split_and_sample_many_return_what_the_plain_call_returns():
    ddpm, kw = tcr.build("fc", "simt", rows=len(SEEDS))
    edm = ddpm.edm
    edm.allowed_ring_sizes = ALLOWED
    want = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=3, require_ring_sizes=True)
    ok, masks, used = edm.last_ring_sizes_ok, edm.last_ring_sizes, edm.last_seeds
    edm.devices = [0, 0]
    got = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=3, require_ring_sizes=True)
    assert torch.equal(got, want) and torch.equal(edm.last_ring_sizes_ok, ok) and torch.equal(edm.last_ring_sizes, masks)
    assert torch.equal(edm.last_seeds, used)
    edm.devices = None
    halves, seeds = [tcr.take(kw, list(range(8))), tcr.take(kw, list(range(8, 16)))], [SEEDS[:8], SEEDS[8:]]
    res = edm.sample_many(halves, keep_frames=2, seeds=seeds, nan_retries=3, require_ring_sizes=True)
    ok_many, masks_many = edm.last_ring_sizes_ok_many, edm.last_ring_sizes_many
    for k in range(2):
        alone = edm.sample_chain(**halves[k], keep_frames=2, seeds=seeds[k], nan_retries=3, require_ring_sizes=True)
        assert torch.equal(res[k], alone)
        assert torch.equal(ok_many[k], edm.last_ring_sizes_ok) and torch.equal(masks_many[k], edm.last_ring_sizes)


@pytest.mark.gpu
def test_the_engine_needs_the_allowed_sizes_and_refuses_low_bits():
    ddpm, kw = tcr.build("fc", "simt", rows=4)
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    assert lib.dl_set_ring_sizes(eng, 1 << 2) == -1 and b"bits 0-2" in lib.dl_last_error()
    assert lib.dl_last_ring_sizes(eng, 4, 1, None) == -1 and b"did not require" in lib.dl_last_error()
    edm.allowed_ring_sizes = [6]
    edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3, 4], require_ring_sizes=True)
    out = torch.empty(3, dtype=torch.int64, device=kw['x'].device)
    assert lib.dl_last_ring_sizes(eng, 3, out.data_ptr(), None) == -1 and b"B differs" in lib.dl_last_error()
    edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3, 4], require_connected=True)
    assert lib.dl_last_ring_sizes(eng, 4, out.data_ptr(), None) == -1    # that call did not require the bit
