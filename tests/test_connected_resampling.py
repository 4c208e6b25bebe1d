"""Connectivity in the recovery rounds: `sample_chain(..., require_connected=True)`, and dl_sample_chain_retry
and dl_molecule_check with DL_CHECK_CONNECTED.

A molecule is connected when the atoms of chain[0] -- without the pocket on cut-off graphs -- form one component under
get_bond_order > 0 (what `is_connected` of the reference's metrics counts for the molecule build_molecule makes). The oracle
here is the CPU restatement of build_xae_molecule (oracle/difflinker_oracle.py) followed by scipy's connected_components.
CPU tests pin that oracle to the reference's bond fixtures and check the argument refusals and the header; the GPU tests
check the kernel molecule by molecule on purpose-built batches, and the sampler end to end."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

from difflinker_b200 import DDPM, _native, molecule_builder as mb, output, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import accelerate, sampler_inputs
from difflinker_b200.edm import retry_seed, seeds_tensor
from difflinker_b200.utils import FoundNaNException
from oracle import difflinker_oracle as orc
import dl_helpers as helpers

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def components(E):
    """Number of connected components of the undirected graph whose edges are E != 0 (lower triangle suffices)."""
    E = np.asarray(E) != 0
    if E.shape[0] == 0:
        return 0
    return connected_components(csr_matrix(E), directed=False)[0]


def oracle_connected(x, types, keep, is_geom):
    """The oracle predicate: build_xae_molecule's bonds over the rows `keep`, then exactly one component."""
    idx = torch.nonzero(keep).flatten()
    idx2atom = output.GEOM_IDX2ATOM if is_geom else output.IDX2ATOM
    _, _, E = orc.xae_molecule(x[idx].float(), types[idx], idx2atom, mb.SINGLE, mb.DOUBLE, mb.TRIPLE, mb.MARGINS_EDM)
    return components(E.numpy()) == 1


def oracle_chain_connected(chain0, node_mask, is_geom, n_types, pocket_only=None):
    """oracle_connected for every row of a chain[0] (B,N,3+F) on the host."""
    chain0 = chain0.cpu()
    B, N = chain0.shape[:2]
    keep = node_mask.reshape(B, N).cpu() != 0
    if pocket_only is not None:
        keep = keep & (pocket_only.reshape(B, N).cpu() == 0)
    types = torch.argmax(chain0[:, :, 3:3 + n_types], dim=2)
    return torch.tensor([oracle_connected(chain0[b, :, :3], types[b], keep[b], is_geom) for b in range(B)])


# ---- CPU --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["bonds_zinc", "bonds_geom"])
def test_oracle_predicate_agrees_with_the_reference_bonds(name):
    meta, a = helpers.load_golden(name)
    counts = []
    for b in range(a["positions"].shape[0]):
        n = int(a["node_mask"][b].sum())
        keep = a["node_mask"][b] != 0
        want = components(a["E"][b, :n, :n].numpy()) == 1                # the reference's own bonds
        assert oracle_connected(a["positions"][b], a["types"][b], keep, meta["is_geom"]) == want, b
        counts.append(want)
    print(f"{name}: {sum(counts)} of {len(counts)} molecules connected")


def _cpu_model(inpainting=False):
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    over = {"inpainting": True} if inpainting else {}
    ddpm, _ = helpers.build_ddpm(spec, 0, **over)
    ddpm.edm.T = 4
    return ddpm, sampler_inputs(ddpm, collate(synthetic.make_items(spec, batch=3)))


@pytest.mark.parametrize("inpainting", [False, True])
def test_connectivity_refuses_what_cannot_resample_one_molecule(inpainting):
    ddpm, kw = _cpu_model(inpainting)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    assert edm.require_connected is False and edm.last_connected is None and edm.is_geom is False
    for bad in (1, "yes", 0.0):
        with pytest.raises(ValueError, match="require_connected"):
            edm.sample_chain(**kw, keep_frames=2, seeds=[1, 2, 3], require_connected=bad)
    with pytest.raises(ValueError, match="per-molecule streams"):            # the batch stream
        edm.sample_chain(**kw, keep_frames=2, require_connected=True)
    with pytest.raises(ValueError, match="noise="):
        edm.sample_chain(**kw, keep_frames=2, require_connected=True, noise=torch.zeros(1))
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, require_connected=True, seeds=[1, 2, 3], batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_connected needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2, require_connected=True, seeds=[1, 2, 3])
    name = 'draw_noise_inpaint' if inpainting else 'draw_noise'
    setattr(edm, name, lambda *a, **k: None)
    with pytest.raises(ValueError, match="replaced"):
        edm.sample_chain(**kw, keep_frames=2, require_connected=True, seeds=[1, 2, 3])
    delattr(edm, name)
    edm.require_connected = True                                         # the attribute stands in for a missing argument
    with pytest.raises(ValueError, match="per-molecule streams"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.noise_mode = 'per_molecule'
    with pytest.raises(ValueError, match="batch_slice"):
        edm.sample_chain(**kw, keep_frames=2, batch_slice=(0, B))
    with pytest.raises(ValueError, match="require_connected needs CUDA inputs"):
        edm.sample_chain(**kw, keep_frames=2)
    edm.is_geom = None                                                   # a bare EDM built without is_geom
    with pytest.raises(ValueError, match="is_geom"):
        edm.sample_chain(**kw, keep_frames=2)
    assert edm.last_connected is None


def test_models_hand_the_edm_their_bond_tables():
    for spec, want in ((synthetic.SPECS["cfg2_zinc"], False), (synthetic.SPECS["cfg3_geom"], True),
                       (synthetic.SPECS["cfg4_pockets"], True)):
        hp = synthetic.model_hparams(spec)
        ddpm = DDPM(**hp)
        assert ddpm.edm.is_geom is want and ddpm.is_geom is want, spec.name
        ddpm.is_geom = not want                                          # accelerate takes the module's own is_geom
        assert accelerate(ddpm).edm.is_geom is (not want)
    from difflinker_b200 import EDM
    assert EDM(dynamics=None, in_node_nf=8, n_dims=3, noise_schedule='polynomial_2', timesteps=10).is_geom is None
    assert EDM(dynamics=None, in_node_nf=9, n_dims=3, noise_schedule='polynomial_2', timesteps=10, is_geom=True).is_geom


def test_header_compiles_as_c99_with_a_connectivity_only_checks_struct(tmp_path):
    """dl_molecule_check with DL_CHECK_CONNECTED alone refuses N beyond the check's limit, naming itself and the limit.
    (A null engine is refused as test_valid_resampling's header test checks.)"""
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "connected_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  int32_t conn[2];\n"
        "  float thr1[64] = {0};\n"
        "  dl_molecule_checks ck = {DL_CHECK_CONNECTED, 8, thr1, NULL, NULL, NULL, NULL};\n"
        "  dl_status b = dl_molecule_check(2, 9000, &ck, NULL, 11, NULL, NULL, 0, 0, conn, NULL, NULL);\n"
        '  printf("%d|%s\\n", (int)b, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "connected_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    b, err_b = res.stdout.strip().split("|", 1)
    assert int(b) == -1 and "dl_molecule_check" in err_b and "8192" in err_b


# ---- GPU: the kernel, molecule by molecule ------------------------------------------------------------------------------

def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


C_C = 1.5                  # a C-C distance that bonds (single-bond threshold 154 + 10 pm)
THR_CC = 1.64              # exactly the C-C threshold in Angstrom: 100 * |x_i - x_j| == 164 in fp32, which does not bond


def line(n, start=0.0, step=C_C, axis=0):
    p = torch.zeros(n, 3)
    p[:, axis] = start + step * torch.arange(n, dtype=torch.float32)
    return p


def purpose_built():
    """(name, positions (n,3), types (n,), pocket flags (n,), valid rows (n,), expected) molecules for the kernel."""
    mols = []

    def add(name, pos, want, types=None, pocket=None, valid=None):
        n = pos.shape[0]
        mols.append((name, pos, torch.zeros(n, dtype=torch.long) if types is None else types,
                     torch.zeros(n) if pocket is None else pocket, torch.ones(n, dtype=torch.bool) if valid is None else valid,
                     want))
    add("chain", line(7), True)
    add("zigzag", torch.stack([1.25 * torch.arange(6.0), 0.8 * (torch.arange(6) % 2).float(), torch.zeros(6)], 1), True)
    add("two clusters", torch.cat([line(3), line(3, start=10.0)]), False)
    add("isolated atom", torch.cat([line(4), torch.tensor([[0.0, 5.0, 0.0]])]), False)
    add("pair at the threshold", torch.cat([line(1), line(1, start=THR_CC)]), False)
    add("pair below the threshold", torch.cat([line(1), line(1, start=1.6399)]), True)
    add("Cl-I: no bond length", torch.cat([line(1), line(1, start=1.0)]), False, types=torch.tensor([5, 7]))
    add("C-N chain", line(5, step=1.5), True, types=torch.tensor([0, 2, 0, 2, 0]))
    # two ligand parts that touch only through a pocket atom: not one molecule
    add("joined through the pocket", torch.cat([line(2), line(1, start=C_C * 2), line(2, start=C_C * 3)]), False,
        pocket=torch.tensor([0.0, 0.0, 1.0, 0.0, 0.0]))
    # padded rows between the two atoms would bridge them if they were read
    add("padded bridge", torch.cat([line(1), line(5, start=C_C), line(1, start=C_C * 6)]), False,
        valid=torch.tensor([True, False, False, False, False, False, True]))
    add("one atom", line(1), True)
    add("one atom among padding", line(4), True, valid=torch.tensor([False, False, True, False]))
    return mols


def pack(mols, N):
    """A padded (B,N,3+8) batch of the molecules, padded rows holding coordinates that continue the last molecule's line."""
    B = len(mols)
    xh = torch.zeros(B, N, 11)
    nm = torch.zeros(B, N, dtype=torch.int8)
    po = torch.zeros(B, N)
    for b, (_, pos, types, pocket, valid, _) in enumerate(mols):
        n = pos.shape[0]
        xh[b, :n, :3] = pos
        xh[b, :n, 3:] = torch.nn.functional.one_hot(types, 8).float()
        nm[b, :n] = valid.to(torch.int8)
        po[b, :n] = pocket
        xh[b, n:, :3] = line(N - n, start=pos[-1, 0] + C_C) if n < N else 0   # would bond to the last atom
        xh[b, n:, 3] = 1.0
    return xh, nm, po


@pytest.mark.gpu
def test_kernel_matches_the_oracle_on_purpose_built_molecules():
    d = dev()
    assert np.float32(100) * np.sqrt(np.float32(THR_CC) ** 2) == np.float32(164)   # the pair really sits on the threshold
    mols = purpose_built()
    xh, nm, po = pack(mols, N=12)
    got = mb.connected(xh.to(d), nm.to(d), False, pocket_only=po.to(d)).cpu()
    for b, (name, pos, types, pocket, valid, want) in enumerate(mols):
        keep = valid & (pocket == 0)
        assert oracle_connected(pos, types, keep, False) == want, name
        assert bool(got[b]) == want, name
    # without dropping the pocket, the pocket atom joins the two parts
    i = [m[0] for m in mols].index("joined through the pocket")
    assert bool(mb.connected(xh[i:i + 1].to(d), nm[i:i + 1].to(d), False).cpu()[0])


@pytest.mark.gpu
def test_a_ligand_of_more_than_128_atoms_in_a_pocket_batch():
    d = dev()
    N, n_lig, n_pocket = 300, 150, 140
    xh = torch.zeros(2, N, 12)
    nm = torch.zeros(2, N, dtype=torch.int8)
    po = torch.zeros(2, N)
    lig = torch.stack([1.25 * torch.arange(n_lig, dtype=torch.float32), 0.8 * (torch.arange(n_lig) % 2).float(),
                       torch.zeros(n_lig)], 1)
    pocket = line(n_pocket, step=1.2) + torch.tensor([0.0, 5.0, 0.0])  # a bonded line of pocket atoms 5 A away
    for b in range(2):
        xh[b, :n_lig, :3] = lig
        xh[b, n_lig:n_lig + n_pocket, :3] = pocket
        xh[b, :n_lig + n_pocket, 3] = 1.0
        nm[b, :n_lig + n_pocket] = 1
        po[b, n_lig:n_lig + n_pocket] = 1.0
    xh[1, 100:, :3] += torch.tensor([0.0, 0.0, 3.0]) * (torch.arange(N)[100:] < n_lig)[:, None]   # break the ligand at 100
    got = mb.connected(xh.to(d), nm.to(d), True, pocket_only=po.to(d)).cpu()
    want = oracle_chain_connected(xh, nm, True, 9, pocket_only=po)
    assert want.tolist() == [True, False] and got.tolist() == want.tolist()


@pytest.mark.gpu
def test_ligand_rows_spread_over_a_4000_row_pocket_batch():
    """N = 4000 takes 80 KB of shared memory (past the 48 KB default), and the ligand rows lie in several 256-row chunks of
    the compaction. Molecule 0's ligand is one chain; molecule 1's is cut, with pocket and padded rows bridging the cut."""
    d = dev()
    N = 4000
    rows = [3, 255, 256, 700, 1999, 2600, 3998]                          # ligand rows, across chunk boundaries
    xh = torch.zeros(2, N, 11)
    xh[:, :, 3] = 1.0
    nm = torch.zeros(2, N, dtype=torch.int8)
    po = torch.zeros(2, N)
    g = torch.Generator().manual_seed(9)
    for b in range(2):
        nm[b, :3990] = 1                                                 # rows 3990.. are padding, except ligand row 3998
        po[b, :3990] = 1.0
        xh[b, :3990, :3] = 50.0 + 20.0 * torch.rand(3990, 3, generator=g)   # pocket atoms, away from the ligand
        for k, r in enumerate(rows):
            xh[b, r, :3] = torch.tensor([C_C * k, 0.0, 0.0])
            nm[b, r] = 1
            po[b, r] = 0.0
    xh[1, rows[4:], 0] += 3.0                                            # a 4.5 A gap between rows 700 and 1999 ...
    for k, r in enumerate((10, 3995)):                                   # ... bridged by a pocket atom and a padded row
        xh[1, r, :3] = torch.tensor([C_C * 3 + 1.5 * (k + 1), 0.0, 0.0])
    nm[1, 3995] = 0
    got = mb.connected(xh.to(d), nm.to(d), False, pocket_only=po.to(d)).cpu()
    want = oracle_chain_connected(xh, nm, False, 8, pocket_only=po)
    assert want.tolist() == [True, False] and got.tolist() == want.tolist()
    # counted as atoms, the pocket atom (row 10) does not bridge either: only the padded row could
    po[1, 10] = 0.0
    want = oracle_chain_connected(xh[1:], nm[1:], False, 8, pocket_only=po[1:])
    got = mb.connected(xh[1:].to(d), nm[1:].to(d), False, pocket_only=po[1:].to(d)).cpu()
    assert got.tolist() == want.tolist() == [False]


@pytest.mark.gpu
@pytest.mark.parametrize("is_geom", [False, True])
def test_kernel_agrees_with_bond_orders_on_random_molecules(is_geom):
    """Random clouds of varying density, some in one piece and some not: the kernel equals the oracle and the components
    of dl_bond_orders' E, the same predicate."""
    d = dev()
    T = 9 if is_geom else 8
    g = torch.Generator().manual_seed(5)
    B, N = 96, 40
    n = torch.randint(1, N + 1, (B,), generator=g)
    nm = (torch.arange(N)[None, :] < n[:, None]).to(torch.int8)
    scale = (0.5 + 2.5 * torch.rand(B, 1, 1, generator=g)) * n[:, None, None].float().pow(1 / 3)
    xh = torch.cat([torch.rand(B, N, 3, generator=g) * scale,
                    torch.nn.functional.one_hot(torch.randint(0, T, (B, N), generator=g), T).float()], 2)
    got = mb.connected(xh.to(d), nm.to(d), is_geom).cpu()
    want = oracle_chain_connected(xh, nm, is_geom, T)
    E = mb.bond_orders(xh[:, :, 3:].to(d), xh.to(d), nm.to(d), is_geom).cpu()
    from_E = torch.tensor([components(E[b, :int(n[b]), :int(n[b])].numpy()) == 1 for b in range(B)])
    assert torch.equal(got, want) and torch.equal(got, from_E)
    assert 0 < int(want.sum()) < B, int(want.sum())                              # both outcomes are exercised


# ---- GPU: the sampler, end to end ---------------------------------------------------------------------------------------

SEEDS = [101, 7, -5, 1 << 62, 33, 2024, 9, 4242]
ROUNDS = 4
# Scale of coord_mlp.4 on top of the fixtures' 100: with it, the random weights move the linker atoms far from the fragment
# and no seed connects; at 0.01 they stay at the scale of the noise next to it, where some seeds connect and others not.
COORD_GAIN = 0.01
# With coordinate updates that small the network predicts almost no noise, and the reverse loop divides a linker atom's
# initial draw by about alpha_T = sqrt(precision) of the polynomial schedule: 300x at the configs' 1e-5, which throws every
# linker far from the fragment. At this precision alpha_T is about 0.6 and the linker ends within bonding distance of the
# fragment for some seeds (measured with the CPU oracle sampler on 20 linker rows: 14 of them connect for the FC linker
# sampler, 11 on the pocket graph). The inpainting sampler also re-noises the fragment, by about sqrt(precision) at the end,
# so it takes a lower one, where 4 of 20 linker rows connect and most fragments stay in one piece.
NOISE_PRECISION = {"fc": 0.4, "pocket_4A": 0.4, "fc_inpainting": 0.1}
CASES = [("fc", "simt"), ("fc", "auto"), ("fc_inpainting", "simt"), ("fc_inpainting", "auto"), ("pocket_4A", "simt"),
         ("pocket_4A", "auto")]


FRAG = torch.stack(torch.meshgrid(torch.arange(3.0), torch.arange(3.0), torch.arange(2.0), indexing='ij'), -1).reshape(-1, 3)
FRAG = 1.2 * (FRAG - FRAG.mean(0))        # a 3 x 3 x 2 carbon lattice, 1.2 A bonds: one piece, and it stays one under noise
NF = FRAG.shape[0]


def small_fragment_items(case, rows):
    """One connected carbon fragment (FRAG) and none, one or two linker atoms; pocket cases add 12 pocket atoms on a 6 A
    shell. Fixed, so the outcome depends on the seeds only. The molecules without a linker are connected at round 0 and
    stay untouched; a linker atom ends where the reverse loop carries its draws, next to the fragment for some seeds and
    away from it for others (see NOISE_PRECISION), so the rounds reconnect some rows and not others."""
    g = torch.Generator().manual_seed(77)
    pocket = 12 if case.startswith("pocket") else 0
    F = 9 if pocket else 8
    items = []
    for b in range(rows):
        lk = b % 3
        link = torch.tensor([[0.0, 0.0, 1.8], [0.0, 0.0, 3.0]])[:lk]
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
        item = {'uuid': b, 'name': f'conn_{b}', 'positions': pos, 'one_hot': torch.nn.functional.one_hot(types, F).float(),
                'anchors': anchors, 'fragment_mask': frag_only + pocket_mask, 'linker_mask': linker_mask, 'num_atoms': n}
        if pocket:
            item['fragment_only_mask'] = frag_only
            item['pocket_mask'] = pocket_mask
        items.append(item)
    return items


def model_spec(case, rows):
    """(spec, DDPM overrides) of the end-to-end models: small, T = 10, the noise precision NOISE_PRECISION."""
    over = {"diffusion_noise_precision": NOISE_PRECISION[case]}
    if case.startswith("pocket"):
        spec = synthetic.WorkloadSpec("conn_pocket", B=rows, N=NF + 14, n_min=NF + 14, l_min=1, l_max=2, F=9, L=2, T=10,
                                      seed=0, pocket=12, graph_type=case.split("_", 1)[1])
    else:
        spec = synthetic.WorkloadSpec("conn_fc", B=rows, N=NF + 2, n_min=NF + 1, l_min=1, l_max=2, F=8, L=2, T=10, seed=0)
        if case == "fc_inpainting":
            over["inpainting"] = True
    return spec, over


def build(case, impl, rows=len(SEEDS)):
    d = dev()
    spec, over = model_spec(case, rows)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, **over)
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(COORD_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(small_fragment_items(case, rows)).items()}
    return ddpm, sampler_inputs(ddpm, data)


def take(kw, idx):
    """Rows `idx` of the sampler inputs; the FC edge mask holds B equal blocks, the pocket one per-node batch ids."""
    B = kw['x'].shape[0]
    ix = torch.tensor(idx, device=kw['x'].device)
    out = {}
    for k, v in kw.items():
        if v is None:
            out[k] = None
        elif k == 'edge_mask':
            out[k] = v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:])
        else:
            out[k] = v[ix]
    return out


def close(got, want):
    """The suite's fp32 tolerance: 1e-4 of the values' scale (at least 1)."""
    return bool((got - want).abs().max() <= 1e-4 * want.abs().max().clamp(min=1.0))


def same(got, want, impl):
    return torch.equal(got, want) if impl == "simt" else close(got, want)


def oracle_rows(ddpm, kw, chain0):
    pocket_only = kw['context'][..., -1] if ddpm.edm.dynamics.graph_type != 'FC' else None
    n_types = 9 if ddpm.edm.is_geom else 8
    return oracle_chain_connected(chain0, kw['node_mask'], ddpm.edm.is_geom, n_types, pocket_only)


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", CASES)
def test_rounds_resample_only_the_disconnected_molecules(case, impl):
    ddpm, kw = build(case, impl)
    edm = ddpm.edm
    B = len(SEEDS)
    base = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS)
    assert edm.last_connected is None
    # nan_retries = 0: the check only reports, and the chain is the one sampled without it
    r0 = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_connected=True)
    conn0 = edm.last_connected
    assert torch.equal(r0, base) and conn0.dtype == torch.bool and conn0.shape == (B,)
    assert torch.equal(conn0, oracle_rows(ddpm, kw, base[0]))
    assert edm.last_attempts.tolist() == [0] * B and torch.equal(edm.last_seeds, seeds_tensor(SEEDS, B))
    runs = []
    for r in range(ROUNDS + 1):
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=r, require_connected=True)
        runs.append((chain, edm.last_connected, edm.last_attempts, edm.last_seeds))
    chain, conn, attempts, used = runs[-1]
    assert torch.isfinite(chain).all()
    assert torch.equal(conn, oracle_rows(ddpm, kw, chain[0]))           # every returned row's flag is the oracle's
    for b in range(B):
        assert int(used[b]) == retry_seed(SEEDS[b], int(attempts[b]))
    healthy = conn0.nonzero().flatten().tolist()
    assert 0 < len(healthy) < B, healthy                                 # the batch mixes both kinds of rows
    assert torch.equal(chain[:, healthy], base[:, healthy]) and all(int(attempts[b]) == 0 for b in healthy)
    # round a' of a run with fewer rounds: each row is the one the longer run had when it first connected, or the last
    # round's draw
    first = [int(attempts[b]) if conn[b] else None for b in range(B)]
    recovered = [b for b in range(B) if first[b] is not None and first[b] > 0]
    assert recovered, first                                              # some rows connect in a round ...
    assert any(first[b] is None for b in range(B)) or all(conn), first
    counts = []
    for r, (c_r, conn_r, att_r, _) in enumerate(runs):
        counts.append(int(conn_r.sum()))
        assert torch.equal(conn_r, oracle_rows(ddpm, kw, c_r[0])), r     # the flags of the rows each round wrote back
        for b in range(B):
            # ... are kept from the round that connected them on, and not resampled again
            want_att = first[b] if first[b] is not None and first[b] <= r else (r if not conn0[b] else 0)
            assert int(att_r[b]) == want_att, (r, b)
            if first[b] is not None and first[b] <= r:
                assert bool(conn_r[b]) and torch.equal(c_r[:, b], chain[:, b]), (r, b)
    assert counts == sorted(counts) and counts[-1] > counts[0], counts   # more connected rows, never fewer
    # a resampled row is its molecule sampled alone with the seed recorded for it
    for b in range(B):
        if int(attempts[b]) > 0:
            alone = edm.sample_chain(**take(kw, [b]), keep_frames=2, seeds=[int(used[b])])
            assert same(chain[:, b], alone[:, 0], impl), b
    print(f"{case}/{impl}: connected after rounds 0..{ROUNDS}: {counts} of {B}; recovered rows {recovered} "
          f"(rounds {[first[b] for b in recovered]})")


# Extra scale of coord_mlp.4 at which, at T = 10, cfg2_zinc_ragged molecules diverge for some seeds and not for others
# (between the NaN recovery tests' 5 and the 8 where most do). Their fragments are random point clouds, so no row is ever
# connected and every finite row is resampled in round 1: with these seeds three of those resamples diverge.
DIVERGE_GAIN = 7.0
DIVERGE_SEEDS = list(range(1, 33))


@pytest.mark.gpu
def test_a_finite_row_is_not_replaced_by_a_resample_that_diverged():
    d = dev()
    spec = synthetic.SPECS["cfg2_zinc_ragged"]
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl="simt")
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(DIVERGE_GAIN)
    ddpm.edm.T = 10
    ddpm = ddpm.to(d)
    edm = ddpm.edm
    B = len(DIVERGE_SEEDS)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=B)).items()}
    kw = sampler_inputs(ddpm, data)

    def run(rounds):
        try:
            chain, bad = edm.sample_chain(**kw, keep_frames=2, seeds=DIVERGE_SEEDS, nan_retries=rounds,
                                          require_connected=True), []
        except FoundNaNException as e:
            chain, bad = e.chain, sorted(e.x_h_nan_idx | e.only_x_nan_idx | e.only_h_nan_idx)
        return chain, bad, edm.last_attempts.clone(), edm.last_connected.clone()
    base, bad0, _, conn0 = run(0)
    got, bad1, attempts, conn1 = run(1)
    assert not conn0.any() and 0 < len(bad0) < B, bad0
    kept = []
    for b in range(B):
        try:                                                             # round 1's draw of molecule b, alone
            edm.sample_chain(**take(kw, [b]), keep_frames=2, seeds=[retry_seed(DIVERGE_SEEDS[b], 1)])
            diverges = False
        except FoundNaNException:
            diverges = True
        if b not in bad0 and diverges:                                   # finite and disconnected: keep it
            kept.append(b)
            assert int(attempts[b]) == 0 and b not in bad1 and torch.equal(got[:, b], base[:, b]), b
        else:                                                            # otherwise the round's draw replaces it
            assert int(attempts[b]) == 1 and (b in bad1) == diverges, b
    assert kept, bad0
    print(f"rows kept over a diverged resample: {kept}; diverged at round 0: {bad0}, after round 1: {bad1}")


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_a_split_resamples_what_the_unsplit_call_resamples(impl):
    ddpm, kw = build("fc", impl)
    edm = ddpm.edm
    want = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=ROUNDS, require_connected=True)
    conn, attempts, used = edm.last_connected, edm.last_attempts, edm.last_seeds
    edm.devices = [0, 0]
    try:
        got = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=ROUNDS, require_connected=True)
    finally:
        edm.devices = None
    assert torch.equal(edm.last_connected, conn) and torch.equal(edm.last_attempts, attempts)
    assert torch.equal(edm.last_seeds, used) and same(got, want, impl)


@pytest.mark.gpu
def test_the_attribute_and_ddpm_opt_in_like_nan_retries():
    ddpm, kw = build("fc", "auto")
    edm = ddpm.edm
    want = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=ROUNDS, require_connected=True)
    conn = edm.last_connected
    d = kw['x'].device
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(small_fragment_items("fc", len(SEEDS))).items()}
    edm.nan_retries, edm.require_connected = ROUNDS, True               # what an unmodified generate.py sets after accelerate()
    chain, _ = ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS)
    assert torch.equal(chain, want) and torch.equal(edm.last_connected, conn)
    chain, _ = ddpm.sample_chain(data, keep_frames=2, seeds=SEEDS, require_connected=False, nan_retries=0)
    assert edm.last_connected is None


@pytest.mark.gpu
def test_a_molecule_that_always_diverges_still_raises():
    ddpm, kw = build("fc", "auto", rows=4)
    edm = ddpm.edm
    kw['x'] = kw['x'].clone()
    kw['x'][2, 0, 0] = float('nan')                                      # a fragment coordinate: every attempt diverges
    with pytest.raises(FoundNaNException) as info:
        edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS[:4], nan_retries=2, require_connected=True)
    exc = info.value
    assert sorted(exc.x_h_nan_idx | exc.only_x_nan_idx | exc.only_h_nan_idx) == [2]
    assert edm.last_attempts[2] == 2 and not edm.last_connected[2]
    assert torch.isfinite(exc.chain[:, [0, 1, 3]]).all()
