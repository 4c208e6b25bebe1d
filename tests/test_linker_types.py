"""Linker types for the linker sampler: `EDM.sample_chain(..., linker_types=M)`, the `edm.linker_types` attribute, the
DDPM symbol mapping, the sample_many key, sample_chain_sharded and dl_set_linker_types.

linker_types_oracle restates the projected loop in fp64. CPU tests check the symbol mapping, the refusals that need no
device, that a None or all-allowed set reaches no engine, and the binding. GPU tests check that None and an all-allowed
set are today's call bit for bit, every device step against the oracle's step applied to the GPU's own earlier frames
(the known-eps construction of test_sampler_steps_fp64.py), real-weight chains against the fp64 oracle, that every linker
atom of chain[0] has an allowed type under every composition, batch-mate independence, and the C setter."""
import ctypes as C
import dataclasses

import pytest
import torch

from difflinker_b200 import _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import linker_types_mask, sampler_inputs
from difflinker_b200.distributed import sample_chain_sharded
from difflinker_b200.edm import EDM
import dl_helpers as helpers
import egnn_options_oracle as eo
import fixed_atoms_oracle as fao
import linker_types_oracle as lto
from test_fixed_atoms import cpu_model, half_mask, launches, pocket, rows, small_fc, xh_of
from test_seeded_linker_sizes import size_model
from test_sampler_steps_fp64 import NORM, U, Checker, dev, f64, fc_batch, known_eps_model, oracle_eps, unnorm_frame
from oracle import difflinker_oracle as orc

F = 8
CNO = torch.tensor([True, True, True, False, False, False, False, False])      # C, O, N in IDX2ATOM order


def per_molecule_sets(B, F=F):
    """(B, F) sets that differ within the batch: C/O/N, C only, all but C, O/N/F/S, all but I, N/Cl/I."""
    base = [[0, 1, 2], [0], list(range(1, F)), [1, 2, 3, 4], list(range(F - 1)), [2, 5, 7]]
    m = torch.zeros((B, F), dtype=torch.bool)
    for b in range(B):
        m[b, base[b % len(base)]] = True
    return m


def linker_types_ok(chain0, kw, sets):
    """Every linker atom of chain[0] has a one-hot type its molecule's set allows."""
    B, N = chain0.shape[:2]
    lm = kw['linker_mask'].reshape(B, N) != 0
    nm = kw['node_mask'].reshape(B, N) != 0
    h = chain0[..., 3:]
    sets = sets.to(chain0.device).expand(B, -1)
    live = lm & nm
    onehot = (h.sum(-1) == 1) & ((h == 0) | (h == 1)).all(-1)
    allowed = torch.gather(sets, 1, h.argmax(-1))
    return bool((onehot & allowed)[live].all())


# ---- CPU: mapping, refusals, the plain path, the binding ---------------------------------------------------------------

def test_symbols_map_through_the_atom_tables():
    zinc = EDM(None, 8, 3, timesteps=20, noise_schedule='polynomial_2', noise_precision=1e-5, is_geom=False)
    assert torch.equal(linker_types_mask(zinc, ['C', 'N', 'O']), CNO)
    assert torch.equal(linker_types_mask(zinc, 'I'), torch.tensor([False] * 7 + [True]))
    assert torch.equal(linker_types_mask(zinc, ['Cl', 'Br']), torch.tensor([False] * 5 + [True, True, False]))
    with pytest.raises(ValueError, match="unknown element 'P'"):
        linker_types_mask(zinc, ['C', 'P'])
    geom = EDM(None, 9, 3, timesteps=20, noise_schedule='polynomial_2', noise_precision=1e-5, is_geom=True)
    assert torch.equal(linker_types_mask(geom, ['P', 'C']), torch.tensor([True] + [False] * 7 + [True]))
    with pytest.raises(ValueError, match="unknown element 'Si'"):
        linker_types_mask(geom, ['Si'])
    with pytest.raises(ValueError, match="is_geom"):
        linker_types_mask(EDM(None, 8, 3, timesteps=20, noise_schedule='polynomial_2', noise_precision=1e-5), ['C'])
    m = torch.ones(8, dtype=torch.bool)
    assert linker_types_mask(zinc, m) is m and linker_types_mask(zinc, None) is None


def test_refusals_without_a_device():
    ddpm, data, kw = cpu_model()
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    empty = CNO.clone().expand(B, F).clone()
    empty[1] = False
    with pytest.raises(ValueError, match="molecule 1 allows no atom type"):
        edm.sample_chain(**kw, linker_types=empty)
    with pytest.raises(ValueError, match="shape"):
        edm.sample_chain(**kw, linker_types=CNO[:7])
    with pytest.raises(ValueError, match="shape"):
        edm.sample_chain(**kw, linker_types=CNO.expand(B + 1, F))
    with pytest.raises(ValueError, match="bool tensor"):
        edm.sample_chain(**kw, linker_types=CNO.int())
    with pytest.raises(ValueError, match="bool tensor"):
        edm.sample_chain(**kw, linker_types=CNO.tolist())
    with pytest.raises(ValueError, match="unknown element"):
        ddpm.sample_chain(data, linker_types=['C', 'Xx'])
    edm.linker_types = CNO[:5]                                            # the attribute is read like the argument
    try:
        with pytest.raises(ValueError, match="shape"):
            edm.sample_chain(**kw)
    finally:
        edm.linker_types = None
    # a kept row whose type the set excludes
    fixed = half_mask(kw)
    kept_types = kw['h'].reshape(B, N, F).argmax(-1)[fixed.bool()]
    bad = torch.ones(F, dtype=torch.bool)
    bad[kept_types[0]] = False
    with pytest.raises(ValueError, match="is kept"):
        edm.sample_chain(**kw, fixed_atoms=fixed, linker_types=bad)
    inp, _, ikw = cpu_model(inpainting=True)
    with pytest.raises(ValueError, match="InpaintingEDM"):
        inp.edm.sample_chain(**ikw, linker_types=CNO)


class _Reached(Exception):
    pass


def test_none_and_all_allowed_reach_no_engine(monkeypatch):
    """The host decides the plain call: _enqueue_batch gets types=None, so no dl_set_linker_types is made."""
    ddpm, _, kw = cpu_model()
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    noise = torch.zeros((edm.T + 2, B, N, 3 + F))
    seen = []

    def enqueue(*a, **k):
        seen.append(k.get('types'))
        raise _Reached
    monkeypatch.setattr(edm, '_enqueue_batch', enqueue)
    monkeypatch.setattr(edm.dynamics, 'engines', lambda places: [None] * len(places))
    monkeypatch.setattr(edm.dynamics, '_device_index', lambda x: 0)
    for m in (None, torch.ones(F, dtype=torch.bool), torch.ones((B, F), dtype=torch.bool), CNO):
        with pytest.raises(_Reached):
            edm.sample_chain(**kw, noise=noise, linker_types=m)
    assert seen[:3] == [None, None, None]
    masks, f, scalars = seen[3]
    assert f == F and torch.equal(masks, torch.full((B,), 0b111, dtype=torch.int32))
    assert list(scalars) == list(edm.fixed_atom_scalars(B))
    per = per_molecule_sets(B)
    with pytest.raises(_Reached):
        edm.sample_chain(**kw, noise=noise, linker_types=per)
    assert seen[4][0].tolist() == [sum(1 << c for c in range(F) if per[b, c]) for b in range(B)]


def test_binding_and_header():
    lib = _native.load_library()
    assert lib.dl_set_linker_types(None, 1, 8, None, 1, None) == -1
    assert b"dl_set_linker_types" in lib.dl_last_error()
    with open(helpers.__file__.replace("tests/dl_helpers.py", "include/difflinker_b200.h")) as f:
        h = f.read()
    assert ("dl_status dl_set_linker_types(dl_engine* e, int32_t B, int32_t F, const uint32_t* masks, int32_t T, "
            "const float* scalars);") in h
    assert _native.SYMBOLS["dl_set_linker_types"][1] == [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                                          C.c_void_p]


def test_oracle_projection_is_the_data_prediction_of_off():
    """The replaced eps gives xhat = off exactly in fp64 arithmetic's rounding."""
    g = torch.Generator().manual_seed(5)
    z = torch.randn((2, 5, 11), generator=g, dtype=torch.float64)
    eps = torch.randn((2, 5, 11), generator=g, dtype=torch.float64)
    lm = torch.ones((2, 5, 1), dtype=torch.float64)
    allowed = torch.zeros((2, 8), dtype=torch.bool)
    allowed[:, 0] = True
    ex = lto.excluded(allowed, lm)
    row = torch.tensor([0.6, 0.8], dtype=torch.float64)
    off = lto.off_value(4.0)
    e2 = lto.project_eps(z, eps, row, ex, off)
    xhat = (z - row[1] * e2) / row[0]
    assert torch.allclose(xhat[ex], torch.full_like(xhat[ex], off), atol=1e-12)
    assert torch.equal(e2[~ex], eps[~ex])


# ---- GPU: None and an all-allowed set are today's call -----------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("graph", ["FC", "4A"])
def test_none_and_all_allowed_are_todays_call(graph):
    ddpm, kw = (small_fc("auto")[:2] if graph == "FC" else pocket("auto"))
    edm = ddpm.edm
    B, nf = kw['x'].shape[0], edm.in_node_nf
    every = [torch.ones(nf, dtype=torch.bool), torch.ones((B, nf), dtype=torch.bool)]
    seeds = list(range(40, 40 + B))
    plain = edm.sample_chain(**kw, keep_frames=4, seeds=seeds)
    counts = [launches(edm)]
    for m in [None] + every:
        assert torch.equal(edm.sample_chain(**kw, keep_frames=4, seeds=seeds, linker_types=m), plain)
        counts.append(launches(edm))
    steps = [b - a for a, b in zip(counts, counts[1:])]
    assert steps == [steps[0]] * 3, steps
    plain = edm.sample_chain(**kw, keep_frames=4, seeds=seeds, nan_retries=1, require_connected=True)
    flags, used = edm.last_connected.clone(), edm.last_seeds.clone()
    for m in every:
        assert torch.equal(edm.sample_chain(**kw, keep_frames=4, seeds=seeds, nan_retries=1, require_connected=True,
                                            linker_types=m), plain)
        assert torch.equal(edm.last_connected, flags) and torch.equal(edm.last_seeds, used)
    torch.manual_seed(3)
    a = edm.sample_chain(**kw, keep_frames=2)
    off = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(3)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=2, linker_types=every[0]), a)
    assert torch.cuda.default_generators[0].get_offset() == off


# ---- GPU: every step against fp64 with a known eps ----------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind", [None, "ddim", "dpmpp_2m"])
def test_every_step_vs_fp64_with_a_known_eps(kind):
    """Every frame against one oracle step from the GPU's previous frame, on excluded, allowed and kept channels."""
    T = 20
    edm, hp, bias = known_eps_model(F, 50, "auto")
    edm.T = T
    kw = fc_batch([(16, 5), (12, 3), (9, 4), (0, 0), (14, 6)], F, seed=17)
    d = dev()
    kw = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    fixed = half_mask(kw)
    fixed[0] = 0
    sets = per_molecule_sets(B)
    h = kw['h'].reshape(B, N, F).clone()                                  # kept rows of allowed types
    for b in range(B):
        for n in range(N):
            if fixed[b, n]:
                h[b, n] = 0
                h[b, n, int(sets[b].nonzero()[0])] = 1
    kw['h'] = h
    draws = helpers.noise_tensor(23, T, B, N, F).to(d)
    chain = edm.sample_chain(**kw, keep_frames=T, noise=draws, fixed_atoms=fixed, linker_types=sets,
                             solver=kind or 'ancestral')
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], 50, hp['diffusion_noise_precision'])
    tab = f64(fao.table(edm, B), d)
    solver = None if kind is None else f64(torch.tensor(list(edm.solver_coefficients(kind))).reshape(T + 1, 8), d)
    chain64 = f64(chain, d)
    nm, fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    fx = f64(fixed, d).reshape(B, N, 1)
    live, kept = nm[..., 0] != 0, fx[..., 0] != 0
    draws = f64(draws, d)
    xh = xh_of(kw, d)
    eps = torch.zeros_like(xh)
    eps[..., 3:] = f64(torch.tensor(bias), d) * nm
    ex = lto.excluded(sets, lm, fx)
    off = lto.off_value(NORM[1])
    ck = Checker(f"types {kind or 'ancestral'}")
    z = fao.start(xh, fm, lm, draws[0], fx, tab, T)
    hist = e_hist = None
    for s in range(T - 1, 0, -1):
        r = T - 1 - s
        if kind is None:
            sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
            a, b, c = (orc._sc(sc, k, z) for k in ("a", "b", "c"))
            n = draws[T - s] * lm
            row_t = fao.start_row(tab, T, s + 1)
            e2 = lto.project_eps(z, eps, row_t, ex, off)
            ref = fao.replace(orc.linker_step(z, e2, sc, draws[T - s], fm, lm), xh, tab[r], n, fx)
            e_eps = torch.where(ex, 4 * U * (z.abs() + (row_t[0] * off).abs()) / row_t[1], torch.zeros_like(z))
            e_free = (4 * U * (z.abs() / a.abs() + (b * e2 * lm).abs() + (c * n).abs()) + b.abs() * e_eps) * lm
        else:
            n = draws[0] * lm
            row = solver[r]
            second = kind == 'dpmpp_2m' and hist is not None
            zs, xhat = lto.ode_step(z, eps, row, fm, lm, ex, off, hist if second else None)
            ref = fao.replace(zs, xh, tab[r], n, fx)
            e_x = 8 * U * (row[1].abs() * (z.abs() + (row[0] * eps).abs()) + off)
            c = row[4] if second else row[3]
            e_free = (8 * U * ((row[2] * z).abs() + (c * xhat).abs() + ((row[5] * hist).abs() if second else 0))
                      + c.abs() * e_x + (row[5].abs() * e_hist if second else 0)) * lm
            hist, e_hist = xhat, e_x
        e_kept = 2 * U * ((tab[r, 0] * xh).abs() + (tab[r, 1] * n).abs())
        got = unnorm_frame(chain64[s])
        ck.close(f"kept s={s}", got, ref, e_kept, kept)
        ck.close(f"free s={s}", got, ref, e_free + 1e-300, live & ~kept)
        z = got
    ck.record()
    assert linker_types_ok(chain[0], kw, sets)
    assert torch.equal(chain64[0][kept][..., 3:], f64(kw['h'], d)[kept])


# ---- GPU: real weights against the fp64 oracle -------------------------------------------------------------------------
REL_TOL = 1e-4


def rel_err(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.double().abs().max().item(), 1e-30)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [50, 500])
@pytest.mark.parametrize("case", ["cfg2_zinc", "small_pocket_4A"])
def test_real_weight_chain_vs_fp64_oracle(case, T):
    """cfg2_zinc's model (ZINC shapes: N = 40, F = 8, six layers) on 16 of its molecules, and a 4 A pocket model, with
    per-molecule sets that differ within the batch."""
    spec = helpers.spec_by_name(case)
    if spec.B > 16:
        spec = dataclasses.replace(spec, B=16)
    ddpm, hp = helpers.build_ddpm(spec, 0, diffusion_steps=500)
    d = dev()
    ddpm = ddpm.to(d)
    edm = ddpm.edm
    edm.T = T
    data = {k: (v.to(d) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    sets = per_molecule_sets(B, spec.F)
    keep = min(T, 50)
    noise = helpers.noise_tensor(61, T, B, N, spec.F).to(d)
    chain = edm.sample_chain(**kw, keep_frames=keep, noise=noise, linker_types=sets)
    cfg = eo.oracle_cfg(hp)
    sd = {k: v.detach() for k, v in edm.dynamics.state_dict().items()}
    fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("fragment_mask", "linker_mask"))
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], 500, hp['diffusion_noise_precision'])
    fwd = lambda t, z: oracle_eps(sd, cfg, t, z, kw, False, torch.float64, d)
    out, zs = lto.sample_ancestral(fwd, xh_of(kw, d), f64(noise, d), fm, lm, sets, gamma, f64(fao.table(edm, B), d), T, B,
                                   lto.off_value(NORM[1]))
    want0 = lto.final_frame(out, f64(kw['node_mask'], d).reshape(B, N, 1), sets, lm, NORM)
    assert torch.equal(chain[0][..., 3:].double(), want0[..., 3:]), "atom types differ"
    assert rel_err(chain[0][..., :3] * lm, want0[..., :3] * lm) <= REL_TOL
    assert linker_types_ok(chain[0], kw, sets)
    unnorm = lambda z: torch.cat([z[..., :3] * NORM[0], z[..., 3:] * NORM[1]], dim=-1)
    frame_of = {(s * keep) // T: s for s in range(T - 1, 0, -1) if (s * keep) // T > 0}
    worst = 0.0
    for f, s in frame_of.items():
        err = rel_err(chain[f], unnorm(zs[T - 1 - s]))
        worst = max(worst, err)
        assert err <= REL_TOL, (f, s, err)
    print(f"{case} T={T}: worst frame rel err {worst:.3g}")


# ---- GPU: the guarantee under every composition ------------------------------------------------------------------------

@pytest.mark.gpu
def test_every_linker_atom_is_allowed_under_every_composition():
    ddpm, kw, data = small_fc("simt", B=12)
    edm = ddpm.edm
    edm.is_geom = False
    B = kw['x'].shape[0]
    sets = per_molecule_sets(B)
    for k in range(4):
        seeds = list(range(100 * k, 100 * k + B))
        ok = lambda ch: linker_types_ok(ch[0], kw, sets)
        assert ok(edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=sets))
        assert ok(edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=sets, start_step=9))
        t0 = [(7 * b + k) % 21 for b in range(B)]
        assert ok(edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=sets, start_step=t0))
        for kind in ("ddim", "dpmpp_2m"):
            assert ok(edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=sets, solver=kind))
        got = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=sets, nan_retries=3, require_connected=True,
                               require_valid=True, require_unique=True)
        assert ok(got)
        fixed = half_mask(kw)
        h = kw['h'].clone()
        h[fixed.bool()] = 0
        h[..., 0][fixed.bool()] = 1                                        # kept carbons, which every set below allows
        cset = sets.clone()
        cset[:, 0] = True
        got = edm.sample_chain(**dict(kw, h=h), keep_frames=1, seeds=seeds, linker_types=cset, fixed_atoms=fixed,
                               nan_retries=2, require_connected=True)
        assert linker_types_ok(got[0], kw, cset)
        assert torch.equal(got[0][fixed.bool()], torch.cat([kw['x'], h], -1)[fixed.bool()])
    assert (edm.last_attempts > 0).any(), "no row was resampled"
    # linker_sizes with redraws: the sets compose with each molecule's drawn (and redrawn) size
    nn = size_model(dev(), [3, 4, 5, 6])
    chain, nm = ddpm.sample_chain(data, keep_frames=1, seeds=list(range(B)), linker_sizes=nn, linker_types=sets,
                                  nan_retries=2, require_connected=True)
    live = nm.reshape(B, -1) != 0
    frag = data['fragment_mask'].reshape(B, -1).sum(1).long()
    link = live & (torch.arange(live.shape[1], device=live.device)[None] >= frag[:, None])
    assert link.any()
    assert linker_types_ok(chain[0], {'linker_mask': link.float(), 'node_mask': nm}, sets)


@pytest.mark.gpu
def test_clash_guidance_and_a_device_split():
    """Pocket model: the sets hold with clash guidance, and a devices=[0, 0] split is the one-slice chain (SIMT path)."""
    ddpm, kw = pocket("simt", rows=8)
    edm = ddpm.edm
    T = edm.T
    B = kw['x'].shape[0]
    sets = per_molecule_sets(B, edm.in_node_nf)
    seeds = list(range(700, 700 + B))
    guided = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, linker_types=sets, clash_guidance=(0.8, T))
    assert linker_types_ok(guided[0], kw, sets)
    edm.devices = [0, 0]
    try:
        split = edm.sample_chain(**kw, keep_frames=2, seeds=seeds, linker_types=sets, clash_guidance=(0.8, T))
        torch.manual_seed(9)
        split_stream = edm.sample_chain(**kw, keep_frames=2, linker_types=sets)
    finally:
        edm.devices = None
    assert torch.equal(split, guided)
    torch.manual_seed(9)
    assert torch.equal(split_stream, edm.sample_chain(**kw, keep_frames=2, linker_types=sets))
    torch.manual_seed(9)                                                   # batch_slice: the slice's rows of the stream
    full = edm.sample_chain(**kw, keep_frames=2, linker_types=sets)
    torch.manual_seed(9)
    part = edm.sample_chain(**rows(kw, 1, 3), keep_frames=2, linker_types=sets[1:3], batch_slice=(1, B))
    assert torch.equal(part, full[:, 1:3])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ancestral", "dpmpp_2m"])
def test_rows_equal_their_single_molecule_calls(kind):
    """Every row of a seeded call, of a per-molecule and an int start-step call, and of a sample_many launch that packs
    requests with different sets equals the molecule sampled alone with its seed, start step and set."""
    ddpm, kw, data = small_fc("simt")
    edm = ddpm.edm
    B = kw['x'].shape[0]
    sets = per_molecule_sets(B)
    seeds = [11 * b + 3 for b in range(B)]
    t0 = [20, 7, 13, 20, 1, 9]
    one = lambda b, **k: edm.sample_chain(**rows(kw, b, b + 1), keep_frames=3, seeds=[seeds[b]], solver=kind,
                                          linker_types=sets[b], **k)[:, 0]
    full = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, solver=kind, linker_types=sets)
    mixed = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, start_step=t0, solver=kind, linker_types=sets)
    reqs = [dict(rows(kw, lo, hi), linker_types=sets[lo:hi]) for lo, hi in ((0, 2), (2, B))]
    many = edm.sample_many(reqs, keep_frames=3, seeds=[seeds[:2], seeds[2:]], solver=kind)
    assert len(edm.last_loop_ms_many) == 1, "the requests did not share a launch"
    for b in range(B):
        alone = one(b)
        assert torch.equal(full[:, b], alone), b
        assert torch.equal(many[0 if b < 2 else 1][:, b if b < 2 else b - 2], alone), b
        assert torch.equal(mixed[:, b], one(b, start_step=t0[b])), b
    plain = edm.sample_chain(**kw, keep_frames=3, seeds=seeds, solver=kind)
    assert not torch.equal(full[0], plain[0])
    # a request without a set takes a launch of its own, so it is its own sample_chain call bit for bit
    many = edm.sample_many([reqs[0], rows(kw, 2, B)], keep_frames=3, seeds=[seeds[:2], seeds[2:]], solver=kind)
    assert len(edm.last_loop_ms_many) == 2
    assert torch.equal(many[1], plain[:, 2:]) and torch.equal(many[0], full[:, :2])
    # DDPM: symbols, one set for every batch of sample_many, the attribute
    chain, _ = ddpm.sample_chain(data, keep_frames=3, seeds=seeds, solver=kind, linker_types=['C', 'N', 'O'])
    assert torch.equal(chain, edm.sample_chain(**kw, keep_frames=3, seeds=seeds, solver=kind, linker_types=CNO))
    many = ddpm.sample_many([data, data], keep_frames=3, seeds=[seeds, seeds], solver=kind, linker_types=['C', 'N', 'O'])
    assert torch.equal(many[0][0], chain) and torch.equal(many[1][0], chain)
    edm.linker_types = CNO
    try:
        assert torch.equal(edm.sample_chain(**kw, keep_frames=3, seeds=seeds, solver=kind), chain)
        assert torch.equal(sample_chain_sharded(ddpm, data, keep_frames=3, seeds=seeds)[0],
                           edm.sample_chain(**kw, keep_frames=3, seeds=seeds))
    finally:
        edm.linker_types = None


@pytest.mark.gpu
def test_setter_is_consumed_by_one_call_and_its_refusals():
    ddpm, kw, _ = small_fc("auto")
    edm = ddpm.edm
    lib = _native.load_library()
    eng = edm.dynamics.engine(0)
    B = kw['x'].shape[0]
    T = edm.T
    tab = edm.fixed_atom_scalars(B)
    masks = (C.c_uint32 * B)(*([0b111] * B))
    assert lib.dl_set_linker_types(eng, 0, F, masks, T, tab) == -1
    assert lib.dl_set_linker_types(eng, B, F - 1, masks, T, tab) == -1
    assert lib.dl_set_linker_types(eng, B, F, masks, 0, tab) == -1
    assert lib.dl_set_linker_types(eng, B, F, masks, T, None) == -1
    for bad in (0, 1 << F):
        m = (C.c_uint32 * B)(*([0b111] * (B - 1) + [bad]))
        assert lib.dl_set_linker_types(eng, B, F, m, T, tab) == -1
        assert b"molecule %d" % (B - 1) in lib.dl_last_error()
    inf = list(tab)
    inf[3] = float('inf')
    assert lib.dl_set_linker_types(eng, B, F, masks, T, (C.c_float * len(inf))(*inf)) == -1
    seeds = list(range(B))
    plain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    want = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=CNO)
    assert lib.dl_set_linker_types(eng, B, F, masks, T, tab) == 0
    assert torch.equal(edm.sample_chain(**kw, keep_frames=1, seeds=seeds), want)    # read by the next call ...
    assert torch.equal(edm.sample_chain(**kw, keep_frames=1, seeds=seeds), plain)   # ... and cleared
    assert lib.dl_set_linker_types(eng, B, F, masks, T, tab) == 0
    edm.T = T - 1                                                        # refused at the call, which clears it
    try:
        with pytest.raises(_native.NativeError, match="dl_set_linker_types"):
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    finally:
        edm.T = T
    assert torch.equal(edm.sample_chain(**kw, keep_frames=1, seeds=seeds), plain)
    # a kept row of an excluded type, vetted with the fixed atoms
    fixed = half_mask(kw).contiguous()
    kept_types = kw['h'].reshape(B, -1, F).argmax(-1)[fixed.bool()]
    excl = (C.c_uint32 * B)(*([((1 << F) - 1) & ~(1 << int(kept_types[0]))] * B))
    N = kw['x'].shape[1]
    assert lib.dl_set_fixed_atoms(eng, B, N, fixed.data_ptr(), T, tab, None) == 0
    assert lib.dl_set_linker_types(eng, B, F, excl, T, tab) == 0
    with pytest.raises(_native.NativeError, match="excludes"):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    assert torch.equal(edm.sample_chain(**kw, keep_frames=1, seeds=seeds), plain)
