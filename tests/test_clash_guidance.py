"""Clash guidance: `EDM.sample_chain(..., clash_guidance=(scale, steps))`, dl_set_clash_guidance and dl_clash_guide.

After the reverse update has produced z_s at a step s < steps, every linker atom i of a molecule moves to
p_i + scale * sum_k max(0, r_ik - d_ik) (p_i - p_k) / d_ik over the molecule's pocket atoms k, with r_ik the clash table's
entry for the pair in Angstrom (stated at dl_set_clash_guidance in the header). clash_guidance_oracle restates the push in
numpy fp64. CPU tests pin the oracle's properties and molecule_builder.clash_guide to it, and check the refusals, the
binding and the header. GPU tests check the kernel against fp64, each guided step of the sampler against the oracle's push
of the plain step, that guidance off is the plain call, the independence of rows, and the recovery rounds."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from difflinker_b200 import _native, molecule_builder as mb
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import seeds_tensor
from difflinker_b200 import synthetic
import clash_guidance_oracle as cgo
import dl_helpers as helpers
import test_clash_resampling as tcl
import test_connected_resampling as tcr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = mb.clash_table(False)                                            # the ZINC types' table: 8 x 8, in pm
NT = TABLE.shape[0]


def random_batch(B, N, seed, box, n_pocket, n_linker, F=NT + 1):
    """A (B,N) batch of fp32 rows (x, one-hot types and a spare feature column) with the pocket rows first, then the linker
    rows, then fragment rows, and the last rows padding (node_mask 0) at every molecule's end. Returns (xh, node_mask,
    linker_mask, pocket_only, types)."""
    g = torch.Generator().manual_seed(seed)
    xh = torch.zeros(B, N, 3 + F)
    xh[..., :3] = box * (torch.rand(B, N, 3, generator=g) - 0.5)
    types = torch.randint(0, NT, (B, N), generator=g)
    xh[..., 3:3 + NT] = torch.nn.functional.one_hot(types, NT).float() * 0.25
    xh[..., 3 + NT:] = torch.rand(B, N, F - NT, generator=g)
    live = N - 1 - (torch.arange(B) % 3)                                 # one to three padded rows per molecule
    nm = (torch.arange(N)[None] < live[:, None]).to(torch.int8)
    po = torch.zeros(B, N)
    po[:, :n_pocket] = 1.0
    lm = torch.zeros(B, N)
    lm[:, n_pocket:n_pocket + n_linker] = 1.0
    xh[nm == 0, :3] = 1e3 * torch.rand(int((nm == 0).sum()), 3, generator=g)   # padding: garbage that must not move
    return xh, nm, lm, po, types


def oracle_push(xh, nm, lm, po, scale, table=TABLE):
    types = cgo.first_argmax(xh[..., 3:3 + table.shape[0]].numpy())
    return cgo.push(xh[..., :3].numpy(), types, nm.numpy(), lm.numpy(), po.numpy(), table.numpy(), scale)


# ---- CPU: the oracle, the host statement, the refusals, the binding --------------------------------------------------

def test_one_contact_at_scale_one_lands_exactly_at_the_clash_distance():
    r = float(TABLE[0, 2]) / 100.0                                       # C-O
    for d0 in (0.3, 1.0, 2.0, r - 1e-6):
        x = np.array([[[0.0, 0.0, 0.0], [d0 * 0.6, -d0 * 0.8, 0.0]]])
        types = np.array([[0, 2]])
        out, moved, _, _ = cgo.push(x, types, np.ones((1, 2)), np.array([[0.0, 1.0]]), np.array([[1.0, 0.0]]),
                                    TABLE.numpy(), 1.0)
        assert moved.tolist() == [[False, True]]
        assert np.array_equal(out[0, 0], x[0, 0])
        assert abs(np.linalg.norm(out[0, 1] - out[0, 0]) - r) < 1e-12
        assert np.allclose(out[0, 1] / np.linalg.norm(out[0, 1]), x[0, 1] / d0, atol=1e-12)   # along the pair's axis
    # beyond r, nothing moves
    x = np.array([[[0.0, 0.0, 0.0], [0.0, 0.0, r + 1e-6]]])
    out, moved, _, _ = cgo.push(x, np.array([[0, 2]]), np.ones((1, 2)), np.array([[0.0, 1.0]]), np.array([[1.0, 0.0]]),
                                TABLE.numpy(), 1.0)
    assert not moved.any() and np.array_equal(out, x)


def test_exempt_coincident_and_nan_pairs_do_not_move():
    table = TABLE.clone()
    table[0, 1] = table[1, 0] = -1.0                                     # C-N exempt
    x = np.array([[[0.0, 0.0, 0.0],                                      # pocket N
                   [4.0, 4.0, 4.0],                                      # pocket C
                   [np.nan, 0.0, 0.0],                                   # pocket C, NaN
                   [0.5, 0.0, 0.0],                                      # linker C: only the exempt N is near
                   [4.0, 4.0, 4.0],                                      # linker O on the pocket C: d = 0
                   [7.0, 7.0, 7.0]]])                                    # linker C far away
    types = np.array([[1, 0, 0, 0, 2, 0]])
    po = np.array([[1.0, 1.0, 1.0, 0.0, 0.0, 0.0]])
    lm = np.array([[0.0, 0.0, 0.0, 1.0, 1.0, 1.0]])
    out, moved, _, _ = cgo.push(x, types, np.ones((1, 6)), lm, po, table.numpy(), 3.0)
    assert not moved.any()
    assert np.array_equal(out, x, equal_nan=True)
    xh = torch.cat([torch.tensor(x, dtype=torch.float64), torch.nn.functional.one_hot(torch.tensor(types), NT).double()], -1)
    got = mb.clash_guide(xh, torch.ones(1, 6), torch.tensor(lm), torch.tensor(po), False, 3.0, clash=table)
    assert torch.equal(torch.nan_to_num(got, nan=-7.0), torch.nan_to_num(xh, nan=-7.0))


def test_only_linker_coordinates_change_and_the_host_statement_is_the_oracle():
    xh, nm, lm, po, _ = random_batch(6, 40, 3, 5.0, 24, 6)
    xh64 = xh.double()
    got = mb.clash_guide(xh64, nm, lm, po, False, 0.7)
    want, moved, _, _ = oracle_push(xh64, nm, lm, po, 0.7)
    linker, _ = cgo.rows(nm.numpy(), lm.numpy(), po.numpy())
    assert moved.sum() > 10                                              # the batch has contacts to push
    assert np.abs(got[..., :3].numpy() - want).max() < 1e-12
    changed = (got != xh64).numpy()
    assert not changed[..., 3:].any()                                    # atom types and the spare column
    assert not changed[~linker].any()                                    # fragment, pocket and padding rows
    assert changed[moved][:, :3].any(-1).all()
    # a fp32 batch comes back fp32, rounded from the fp64 push
    got32 = mb.clash_guide(xh, nm, lm, po, False, 0.7)
    assert got32.dtype == torch.float32 and torch.equal(got32, got.float())


def test_the_push_is_equivariant_under_rotation_and_translation():
    xh, nm, lm, po, types = random_batch(4, 30, 5, 5.0, 18, 5)
    x = xh[..., :3].double().numpy()
    q, _ = np.linalg.qr(np.random.default_rng(7).standard_normal((3, 3)))
    shift = np.array([3.0, -11.0, 0.5])
    args = (types.numpy(), nm.numpy(), lm.numpy(), po.numpy(), TABLE.numpy(), 0.9)
    a, moved_a, _, _ = cgo.push(x, *args)
    b, moved_b, _, _ = cgo.push(x @ q.T + shift, *args)
    assert moved_a.any() and np.array_equal(moved_a, moved_b)
    live = nm.numpy() != 0
    assert np.abs((a @ q.T + shift)[live] - b[live]).max() < 1e-12


def _models():
    return {"pocket": tcl._pocket_cpu_model(), "fc": tcr._cpu_model(False), "inpainting": tcr._cpu_model(True)}


@pytest.mark.parametrize("kind", ["fc", "inpainting", "pocket"])
def test_clash_guidance_refuses_what_it_cannot_guide(kind):
    ddpm, kw = _models()[kind]
    edm = ddpm.edm
    B = kw['x'].shape[0]
    assert edm.clash_guidance is None
    if kind != "pocket":
        why = "InpaintingEDM" if kind == "inpainting" else "FC graphs"
        for g in ((1.0, 2), (0.0, 0)):                                   # refused even when it would guide nothing
            with pytest.raises(ValueError, match=why):
                edm.sample_chain(**kw, keep_frames=2, clash_guidance=g)
        edm.clash_guidance = (1.0, 2)                                    # the attribute stands in for a missing argument
        with pytest.raises(ValueError, match=why):
            edm.sample_chain(**kw, keep_frames=2)
        return
    T = edm.T
    for bad in ((True, 2), (np.bool_(True), 2), (-1.0, 2), (float("nan"), 2), (float("inf"), 2), (1e39, 2), ("1", 2),
                (None, 2), (np.float32(-1), 2), (1.0, -1), (1.0, T + 1), (1.0, 2.0), (1.0, True), (1.0, np.bool_(True)),
                1.0, (1.0,), (1.0, 2, 3)):
        with pytest.raises(ValueError, match="clash_guidance"):
            edm.sample_chain(**kw, keep_frames=2, clash_guidance=bad)
    with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
        edm.sample_chain(**kw, keep_frames=2, start_step=2, clash_guidance=(1.0, 2))
    with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
        edm.sample_chain(**kw, keep_frames=2, start_step=list(range(1, B + 1)), clash_guidance=(1.0, 2))
    with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
        edm.sample_many([kw], keep_frames=2, seeds=[list(range(B))], start_step=2, clash_guidance=(1.0, 2))
    with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
        edm.sample_many([kw], keep_frames=2, seeds=[list(range(B))], start_step=[2], clash_guidance=(1.0, 2))
    # one rule for both entry points: a setting that guides nothing is refused with start_step too
    for off in ((0.0, 2), (1.0, 0)):
        with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
            edm.sample_chain(**kw, keep_frames=2, start_step=2, clash_guidance=off)
        with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
            edm.sample_chain(**kw, keep_frames=2, start_step=list(range(1, B + 1)), clash_guidance=off)
        with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
            edm.sample_many([kw], keep_frames=2, seeds=[list(range(B))], start_step=2, clash_guidance=off)
        with pytest.raises(ValueError, match="clash_guidance does not take start_step"):
            edm.sample_many([kw], keep_frames=2, seeds=[list(range(B))], start_step=[2], clash_guidance=off)
    edm.clash_guidance = (1.0, T + 1)
    with pytest.raises(ValueError, match="clash_guidance's steps"):
        edm.sample_chain(**kw, keep_frames=2)
    # the edge values are accepted: (0, K) and (scale, 0) guide nothing, and K = T every step
    assert edm._clash_guidance((0.0, T), None) is None and edm._clash_guidance((2.5, 0), None) is None
    scale, steps, table = edm._clash_guidance((2.5, T), None)
    assert (scale, steps) == (2.5, T) and torch.equal(table, mb.clash_table(edm.is_geom))
    assert edm._clash_guidance((torch.tensor(0.1), np.int64(3)), None)[:2] == (np.float32(0.1), 3)
    for scale in (np.float32(1.5), np.float64(1.5), np.int64(1), 1, 1.5):                 # Python and numpy reals
        assert edm._clash_guidance((scale, np.int32(4)), None)[:2] == (float(scale), 4)


def test_models_pass_clash_guidance_to_the_edm():
    ddpm, _ = tcr._cpu_model()
    data = collate(synthetic.make_items(synthetic.SPECS["cfg2_zinc_ragged"], batch=3))
    seen = []
    ddpm.edm.sample_chain = lambda **k: seen.append(k.get('clash_guidance', 'unset'))
    ddpm.edm.sample_many = lambda reqs, **k: seen.append(k.get('clash_guidance', 'unset')) or [None] * len(reqs)
    from difflinker_b200 import ddpm as ddpm_mod
    ddpm.sample_chain(data, keep_frames=2, clash_guidance=(1.0, 5))
    ddpm.sample_chain(data, keep_frames=2)
    ddpm_mod.sample_chain(ddpm, data, keep_frames=2, clash_guidance=(0.5, 2))
    ddpm.sample_many([data], keep_frames=2, seeds=[[1, 2, 3]], clash_guidance=(1.0, 5))
    ddpm_mod.sample_many(ddpm, [data], keep_frames=2, seeds=[[1, 2, 3]])
    assert seen == [(1.0, 5), 'unset', (0.5, 2), (1.0, 5), 'unset']


def test_native_binds_the_guidance_entries_and_refuses_before_reading_pointers():
    lib = _native.load_library()
    assert "dl_set_clash_guidance" in _native.SYMBOLS and "dl_clash_guide" in _native.SYMBOLS
    assert lib.dl_set_clash_guidance(None, 1.0, 5, NT, None) == -1 and b"null engine" in lib.dl_last_error()
    ok = (2, 4, NT, 1, 1.0, 1, NT + 3, 1, 1, 1, 1, None)
    for k, v, why in ((0, 0, b"B and N"), (1, 8193, b"8192"), (2, NT + 1, b"n_types"), (3, None, b"clash table"),
                      (4, -1.0, b"scale"), (4, float("nan"), b"scale"), (4, float("inf"), b"scale"),
                      (5, None, b"invalid argument"), (10, 0, b"invalid argument")):
        args = list(ok)
        args[k] = v
        assert lib.dl_clash_guide(*args) == -1, why
        assert why in lib.dl_last_error() and b"dl_clash_guide" in lib.dl_last_error()


def test_header_compiles_as_c99_with_the_guidance_entries(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib = _native.LIB_PATH
    _native.load_library()
    src = tmp_path / "guide_abi.c"
    src.write_text(
        '#include <stdio.h>\n#include "difflinker_b200.h"\n'
        "int main(void) {\n"
        "  float clash[81] = {0}, xh[26] = {0}, lm[2] = {0}, ctx[2] = {0}; int8_t nm[2] = {0};\n"
        "  dl_status a = dl_set_clash_guidance(NULL, 1.0f, 50, 9, clash);\n"
        '  printf("%d|%s|", (int)a, dl_last_error());\n'
        "  dl_status b = dl_clash_guide(2, 8193, 9, clash, 1.0f, xh, 13, nm, lm, ctx, 1, NULL);\n"
        '  printf("%d|%s|", (int)b, dl_last_error());\n'
        "  dl_status c = dl_clash_guide(2, 1, 9, clash, -1.0f, xh, 13, nm, lm, ctx, 1, NULL);\n"
        '  printf("%d|%s\\n", (int)c, dl_last_error());\n'
        "  return 0;\n}\n")
    exe = tmp_path / "guide_abi"
    inc = os.path.join(ROOT, "include")
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{inc}", str(src), "-o", str(exe), lib,
                    f"-Wl,-rpath,{os.path.dirname(lib)}"], check=True, capture_output=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, (res.stdout, res.stderr)
    a, err_a, b, err_b, c, err_c = res.stdout.strip().split("|", 5)
    assert int(a) == -1 and "null engine" in err_a
    assert int(b) == -1 and "dl_clash_guide" in err_b and "8192" in err_b
    assert int(c) == -1 and "dl_clash_guide" in err_c and "scale" in err_c


# ---- GPU: dl_clash_guide against fp64 ---------------------------------------------------------------------------------

def run_guide(xh, nm, lm, po, scale, table=TABLE):
    d = tcr.dev()
    xs = xh.to(d).contiguous()
    nmd, lmd = nm.to(d).contiguous(), lm.to(d).contiguous()
    pod = po.reshape(*po.shape, 1).to(d).contiguous()
    tab = table.to(d).contiguous()
    lib = _native.load_library()
    B, N = nm.shape
    with torch.cuda.device(d):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_clash_guide(B, N, table.shape[0], tab.data_ptr(), scale, xs.data_ptr(), xs.shape[2],
                                         nmd.data_ptr(), lmd.data_ptr(), pod.data_ptr(), 1, st), "dl_clash_guide")
    return xs.cpu()


SLACK = 1e-3      # A: pairs this close to their r_ik are left out (an fp32 distance a few ulp off may decide them the other way)


def assert_guide_matches_fp64(xh, nm, lm, po, scale, table=TABLE):
    got = run_guide(xh, nm, lm, po, scale, table)
    want, moved, bound, slack = oracle_push(xh.double(), nm, lm, po, scale, table)
    linker, _ = cgo.rows(nm.numpy(), lm.numpy(), po.numpy())
    changed = ~((got == xh) | (torch.isnan(got) & torch.isnan(xh))).numpy()
    assert not changed[..., 3:].any() and not changed[~linker].any()     # bit for bit: types, non-linker rows
    judged = linker & (slack > SLACK)
    assert not changed[judged & ~moved].any()                            # an atom with no contact is not written
    err = np.abs(got[..., :3].double().numpy() - want).max(-1)
    sel = judged & moved
    assert (err[sel] <= bound[sel]).all(), (err[sel] / bound[sel]).max()
    return int(sel.sum()), int((linker & ~judged).sum()), float((err[sel] / bound[sel]).max()) if sel.any() else 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("B,N,box", [(64, 300, 9.0), (4, 4000, 24.0)])
def test_kernel_matches_fp64_on_random_batches(B, N, box):
    """The tolerance is the oracle's bound: 16 u (|p_i| + scale sum_k (r_ik + w_ik d_ik)) per coordinate, which covers the
    handful of fp32 roundings of each term, the fixed five-round shuffle sum and the final fma."""
    n_pocket = int(0.8 * N)
    xh, nm, lm, po, _ = random_batch(B, N, 11 + N, box, n_pocket, 12)
    lm[0] = 0.0                                                          # molecule 0: no linker atom
    po[1] = 0.0                                                          # molecule 1: no pocket atom
    xh[2, n_pocket + 3, 1] = float("nan")                                # a NaN linker atom
    xh[3, 5, 0] = float("nan")                                           # a NaN pocket atom
    for scale in (1.0, 0.3, 2.0):
        judged, left_out, worst = assert_guide_matches_fp64(xh, nm, lm, po, scale)
        assert judged > (50 if B > 4 else 5)
        print(f"B={B} N={N} scale={scale}: {judged} moved atoms judged, {left_out} linker atoms within {SLACK} A of a "
              f"threshold left out, worst err/bound {worst:.3f}")
    assert torch.equal(run_guide(xh, nm, lm, po, 0.0).nan_to_num(nan=7.0), xh.nan_to_num(nan=7.0))   # scale 0: no launch


@pytest.mark.gpu
@pytest.mark.parametrize("N", [2454, 2457])
def test_kernel_runs_where_dynamic_and_static_shared_memory_just_pass_48_kb(N):
    """N * 20 bytes of staging is at most 48 KB here, but with the kernel's static shared memory it is over: the launch
    must not depend on whether something raised the kernel's limit before."""
    xh, nm, lm, po, _ = random_batch(2, N, 9, 20.0, N - 40, 20)
    judged, _, _ = assert_guide_matches_fp64(xh, nm, lm, po, 1.0)
    assert judged > 0


@pytest.mark.gpu
def test_kernel_matches_fp64_at_the_row_limit_and_with_exempt_pairs():
    xh, nm, lm, po, _ = random_batch(1, 8192, 5, 40.0, 8000, 40)
    table = TABLE.clone()
    table[0, :] = table[:, 0] = -1.0                                     # every pair with a carbon exempt
    judged, _, _ = assert_guide_matches_fp64(xh, nm, lm, po, 1.0, table)
    assert judged > 5


# ---- GPU: the sampler ------------------------------------------------------------------------------------------------

POCKET = 24
T_LOOP = 10


def pocket_items(rows, radius):
    """test_clash_resampling's lattice and pocket shell with the shell at `radius` from the fragment's centre."""
    g = torch.Generator().manual_seed(79)
    items = []
    for b in range(rows):
        link = torch.tensor([[0.0, 0.0, 1.8], [0.0, 0.0, 3.0]])[:1 + b % 2]
        v = torch.randn(POCKET, 3, generator=g)
        pos = torch.cat([tcr.FRAG, radius * v / v.norm(dim=1, keepdim=True), link])
        n = pos.shape[0]
        types = torch.zeros(n, dtype=torch.long)
        types[tcr.NF:tcr.NF + POCKET] = torch.randint(0, 3, (POCKET,), generator=g)
        frag_only = torch.zeros(n); frag_only[:tcr.NF] = 1.0
        pocket_mask = torch.zeros(n); pocket_mask[tcr.NF:tcr.NF + POCKET] = 1.0
        linker_mask = torch.zeros(n); linker_mask[tcr.NF + POCKET:] = 1.0
        items.append({'uuid': b, 'name': f'guide_{b}', 'positions': pos,
                      'one_hot': torch.nn.functional.one_hot(types, 9).float(), 'anchors': torch.zeros(n),
                      'fragment_mask': frag_only + pocket_mask, 'linker_mask': linker_mask, 'num_atoms': n,
                      'fragment_only_mask': frag_only, 'pocket_mask': pocket_mask})
    return items


def build(graph, impl, rows=16, radius=2.5, known_eps=False, T=T_LOOP):
    d = tcr.dev()
    spec = synthetic.WorkloadSpec("guide_pocket", B=rows, N=tcr.NF + POCKET + 2, n_min=tcr.NF + POCKET + 1, l_min=1,
                                  l_max=2, F=9, L=2, T=T, seed=0, pocket=POCKET, graph_type=graph)
    ddpm, _ = helpers.build_ddpm(spec, 0, edge_impl=impl, diffusion_noise_precision=tcr.NOISE_PRECISION["pocket_4A"])
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if known_eps and (name.endswith("embedding_out.weight") or name.endswith("coord_mlp.4.weight")):
                p.zero_()                                                # eps_x = 0, eps_h = embedding_out.bias
            elif name.endswith("coord_mlp.4.weight"):
                p.mul_(tcr.COORD_GAIN)
    ddpm.edm.T = T
    ddpm = ddpm.to(d)
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(pocket_items(rows, radius)).items()}
    return ddpm, sampler_inputs(ddpm, data)


def launches(edm):
    return int(_native.load_library().dl_launch_count(edm.dynamics.engine(0)))


GRAPH_CASES = [(g, impl) for g in ("4A", "FC-10A-4A") for impl in ("simt", "auto")]


@pytest.mark.gpu
@pytest.mark.parametrize("graph,impl", GRAPH_CASES)
def test_each_guided_step_is_the_oracles_push_of_the_plain_step(graph, impl):
    """Known eps (test_sampler_steps_fp64.py's construction): eps_x = 0 and eps_h = b_j, so z_s = z_t / a - b eps + c n on
    the linker rows, evaluated in fp64 from the GPU's own z_t (frame s + 1, keep_frames = T). At a guided step the frame
    must be the oracle's push of that plain step, within (1 + scale sum_k r_ik / d_ik) times the step's rounding bound
    4u (|z_t / a| + |c n|) -- the push's gain on an input error -- plus the push's own bound; the steps before guidance
    starts and every atom-type channel are those of the unguided chain bit for bit."""
    ddpm, kw = build(graph, impl, known_eps=True)
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    F, K, scale = 9, 6, 0.8
    noise = helpers.noise_tensor(5, T_LOOP, B, N, F).to(kw['x'].device)
    plain = edm.sample_chain(**kw, keep_frames=T_LOOP, noise=noise).cpu()
    guided = edm.sample_chain(**kw, keep_frames=T_LOOP, noise=noise, clash_guidance=(scale, K)).cpu()
    assert torch.equal(guided[..., 3:], plain[..., 3:])                  # types: eps_h does not depend on x
    for s in range(K, T_LOOP):
        assert torch.equal(guided[s], plain[s]), s                       # before guidance starts
    coef = edm.step_coefficients(T_LOOP, B)
    table = mb.clash_table(edm.is_geom)                                  # the table sample_chain guides with
    nm = kw['node_mask'].reshape(B, N).cpu()
    lm = kw['linker_mask'].reshape(B, N).cpu()
    fm = kw['fragment_mask'].reshape(B, N).cpu()
    po = kw['context'][..., -1].reshape(B, N).cpu()
    nz = noise.cpu().double()
    pushed = 0
    for s in range(1, K):
        row = T_LOOP - 1 - s
        a, c = float(coef[row].a), float(coef[row].c)
        zt = guided[s + 1, ..., :3].double()
        n = nz[row + 1, ..., :3] * lm[..., None].double()
        zs = zt * fm[..., None].double() + (zt / a + c * n) * lm[..., None].double()
        types = cgo.first_argmax(guided[s, ..., 3:3 + table.shape[0]].numpy())
        want, moved, bound, slack = cgo.push(zs.numpy(), types, nm.numpy(), lm.numpy(), po.numpy(), table.numpy(), scale)
        linker, _ = cgo.rows(nm.numpy(), lm.numpy(), po.numpy())
        step_bound = 4 * cgo.U * (np.abs(zt.numpy() / a) + np.abs(c * n.numpy())).max(-1)
        x = zs.numpy()
        gain = np.ones((B, N))
        for b in range(B):                                               # 1 + scale sum_k r_ik / d_ik over contacts
            for i in np.nonzero(linker[b])[0]:
                for k in np.nonzero((nm[b] != 0).numpy() & (po[b] != 0).numpy())[0]:
                    d = np.linalg.norm(x[b, i] - x[b, k])
                    r = float(table[min(types[b, i], types[b, k]), max(types[b, i], types[b, k])]) / 100
                    if 0 < d < r:
                        gain[b, i] += scale * r / d
        tol = 2 * (gain * step_bound + bound) + 1e-30
        got = guided[s, ..., :3].double().numpy()
        judged = linker & (slack > 1e-3)
        err = np.abs(got - want).max(-1)
        assert (err[judged] <= tol[judged]).all(), (s, (err[judged] / tol[judged]).max())
        assert np.array_equal(got[~linker], guided[s + 1, ..., :3].numpy()[~linker])   # fragment, pocket, padding rows
        pushed += int((judged & moved).sum())
    assert pushed > 10, pushed
    print(f"{graph}/{impl}: {pushed} pushed linker atoms over steps 1..{K - 1}")


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_guidance_off_is_the_plain_call_and_on_adds_one_launch_per_step(impl):
    ddpm, kw = build("4A", impl)
    edm = ddpm.edm
    seeds = list(range(100, 116))
    edm.sample_chain(**kw, keep_frames=2, seeds=seeds)                  # the engine exists before counting
    n0 = launches(edm)
    plain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    per_call = launches(edm) - n0
    for g in ((0.0, T_LOOP), (1.0, 0), (0.0, 0)):
        n0 = launches(edm)
        off = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, clash_guidance=g)
        assert torch.equal(off, plain) and launches(edm) - n0 == per_call, g
    n0 = launches(edm)
    on = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, clash_guidance=(1.0, T_LOOP))
    assert launches(edm) - n0 == per_call + T_LOOP + 1                   # one guidance launch in every step graph
    assert not torch.equal(on[0, ..., :3], plain[0, ..., :3])
    # the attribute stands in for a missing argument, and the engine's setting does not outlive the call
    edm.clash_guidance = (1.0, T_LOOP)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, seeds=seeds), on)
    edm.clash_guidance = None
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, seeds=seeds), plain)


@pytest.mark.gpu
def test_a_call_keeps_the_table_set_for_it_while_a_later_call_sets_another():
    """Two engine calls enqueued back to back on one stream with no synchronisation between them, the second after a new
    table was set (_sample_slice sets it right before its call and clears it after): the first, still running when the
    second sets its table, guides with its own table. Each result equals the same call made alone."""
    ddpm, kw = build("4A", "simt", T=200)
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    dev = kw['x'].device
    seeds = list(range(300, 300 + B))
    alone_a = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, clash_guidance=(1.0, edm.T))
    plain = edm.sample_chain(**kw, keep_frames=2, seeds=seeds)
    assert not torch.equal(alone_a, plain)
    table = mb.clash_table(edm.is_geom)                                  # table A: the model's, as sample_chain passes it
    exempt = torch.full_like(table, -1.0)                                # table B: every pair exempt, i.e. the plain loop
    lib = _native.load_library()
    full = edm._sampler_tensors(kw['x'], kw['h'], kw['node_mask'], kw['fragment_mask'], kw['linker_mask'],
                                kw['edge_mask'], kw['context'])
    idx = edm.dynamics._device_index(kw['x'])
    engines = edm.dynamics.engines([(idx, 0)])
    coef = edm.step_coefficients(2, B)
    dev_seeds = seeds_tensor(seeds, B).to(dev)
    runs = []
    for tab in (table, exempt):
        runs.append(edm._enqueue_batch(lib, full, 2, coef, [(idx, 0, 0, B)], engines, [dev], dev, dev_seeds=dev_seeds,
                                       guide=(1.0, edm.T, tab.contiguous())))
    with torch.cuda.device(dev):
        for calls, _ in runs:                                            # both loops enqueued before either is read
            calls[0][1]()
    got_a, got_b = (finish()['chain'] for _, finish in runs)
    assert torch.equal(got_a, alone_a)
    assert torch.equal(got_b, plain)


@pytest.mark.gpu
@pytest.mark.parametrize("graph,impl", GRAPH_CASES)
def test_rows_do_not_depend_on_their_batch_its_split_or_its_packing(graph, impl):
    ddpm, kw = build(graph, impl)
    edm = ddpm.edm
    B = kw['x'].shape[0]
    seeds = list(range(200, 200 + B))
    g = (1.0, T_LOOP)
    full = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, clash_guidance=g)
    assert torch.isfinite(full).all()
    for b in (0, 5, B - 1):
        alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=3, seeds=[seeds[b]], clash_guidance=g)
        assert tcr.same(full[:, b], alone[:, 0], impl), b
    edm.devices = [0, 0]
    try:
        split = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, clash_guidance=g)
    finally:
        edm.devices = None
    assert tcr.same(split, full, impl)
    parts = [list(range(0, 5)), list(range(5, 12)), list(range(12, B))]
    reqs = [tcr.take(kw, p) for p in parts]
    many = edm.sample_many(reqs, keep_frames=3, seeds=[[seeds[i] for i in p] for p in parts], clash_guidance=g,
                           max_molecules=8)
    for p, req, got in zip(parts, reqs, many):
        want = edm.sample_chain(**req, keep_frames=3, seeds=[seeds[i] for i in p], clash_guidance=g)
        assert tcr.same(got, want, impl)
    # the batch stream, on the device and as the materialised tensor, and a noise= tensor, all guided
    chains = []
    for mode in ("reference_stream", "reference_tensor"):
        edm.noise_mode = mode
        torch.manual_seed(17)
        chains.append(edm.sample_chain(**kw, keep_frames=3, clash_guidance=g))
    edm.noise_mode = "reference_stream"
    assert torch.equal(chains[0], chains[1])
    noise = helpers.noise_tensor(3, T_LOOP, B, kw['x'].shape[1], 9).to(kw['x'].device)
    a = edm.sample_chain(**kw, keep_frames=3, noise=noise, clash_guidance=g)
    b = edm.sample_chain(**kw, keep_frames=3, noise=noise)
    assert torch.isfinite(a).all() and not torch.equal(a, b)


SEEDS = list(range(31, 47))
ROUNDS = 6


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
def test_recovery_rounds_are_guided_like_round_zero(impl):
    """The pocket shell of test_clash_resampling.py pulled in from 4 A to 2.5 A, so that linker atoms clash with it."""
    ddpm, kw = build("4A", impl, rows=len(SEEDS))
    edm = ddpm.edm
    B = len(SEEDS)
    nm, lm = kw['node_mask'].reshape(B, -1), kw['linker_mask'].reshape(B, -1)
    po = kw['context'][..., -1].reshape(B, -1)
    fails = {}
    for name, g in (("unguided", None), ("guided", (1.0, T_LOOP))):
        edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, require_clash_free=True, clash_guidance=g)
        fails[name] = B - int(edm.last_clash_free.sum())
        chain = edm.sample_chain(**kw, keep_frames=2, seeds=SEEDS, nan_retries=ROUNDS, require_clash_free=True,
                                 clash_guidance=g)
        ok, attempts, used = edm.last_clash_free, edm.last_attempts, edm.last_seeds
        assert torch.equal(ok, mb.clash_free(chain[0], nm, lm, po, edm.is_geom).cpu())
        if name == "guided":
            assert ok.all(), ok                                          # every returned row passes
            for b in range(B):                                           # a resampled row is its molecule guided alone
                if int(attempts[b]) > 0:
                    alone = edm.sample_chain(**tcr.take(kw, [b]), keep_frames=2, seeds=[int(used[b])], clash_guidance=g)
                    assert tcr.same(chain[:, b], alone[:, 0], impl), b
                else:
                    assert int(used[b]) == int(seeds_tensor(SEEDS, B)[b])
    print(f"4A/{impl}: round-0 clash failures of {B} rows: {fails}")
    assert fails == {"unguided": 13, "guided": 2}, fails                 # measured on an H100 80GB HBM3, both edge paths
