"""The sampler kernels against fp64, step by step: k_init_z and the sampler half of k_finish (linker sampler), k_inpaint and
k_com_free_draws (inpainting sampler), and k_restore_frame, the output stage right after the sampler.

Chains run with keep_frames = T, so chain[s] is the unnormalised z_s of every reverse step s = 1..T-1 and chain[0] the final
sample (the last-writer rule of EDM.step_coefficients). z_T is rebuilt in fp64 from the inputs and draw 0 -- exactly, since
the masks are 0/1 -- and each step is checked on its own: the oracle's step function (oracle.difflinker_oracle.linker_step,
inpaint_step) applied in fp64 to the GPU's own z_{s+1} must land within a rounding bound of the GPU's z_s. z_0 is not
stored, so the last step is checked as the composite z_1 -> z_0 -> final sample, with z_0's bound carried into the final one.

The dynamics output is made known exactly: embedding_out.weight and the last Linear of every coord_mlp are zeroed and
embedding_out.bias[:F] holds distinct dyadic values b_j, so eps_x = 0 and eps_h = b_j * node_mask whatever the forward
computes. That isolates the sampler arithmetic from the network. The bound per element, from the fp32 step scalars promoted
to fp64 (u = 2^-24), is 4u (|z_t / a| + |b eps| + |c n|) plus the incoming error scaled by the step (1/a, and qa on
inpainting fragment atoms). Inpainting adds the q terms and, on coordinates, the centre-of-mass projection's mean: each
thread of k_inpaint's 256-thread CTA sums up to ceil(N gcd(3+F, 256) / 256) coordinates of one column in sequence before the
shuffle and warp-partial tree, so the mean gets (that + 16) u sum|z| / count, plus the mean of the incoming errors.
Exact checks: padded rows are 0 in every frame, the linker sampler's fragment rows equal z_T bit for bit, final one-hot rows
sum to the node mask, and a designed tie gives the first feature as torch.argmax does. Atom types are compared wherever the
fp64 top-two gap exceeds twice the bound; the report gives the fraction compared.

These known-eps checks have a zero velocity and an eps that does not depend on t. So they do not see velocity centring, or the t
and the masks of the forward inside the loop. The real-weight checks at the end of the file cover those. For inpainting, the
device-stream draws expected here come from dl_noise_fill_inpaint. It shares its device functions with k_inpaint, so those
functions are checked against torch separately: test_inpaint_device_noise.py against the fp32 projection, and
test_inpainting_draws_at_n4000_vs_fp64_projection below against fp64.
"""
import ctypes as C
import dataclasses
import math

import pytest
import torch

from difflinker_b200 import _native, output, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.edm import EDM, InpaintingEDM
import dl_helpers as helpers
import egnn_options_oracle as eo
from fp64_rows import C_DRIFT, TAU, _full_fp32_matmul, pocket_item
from oracle import difflinker_oracle as orc

U = 2.0 ** -24
NORM = (1.0, 4.0, 10.0)       # normalize_factors of every config; x * 1 and h * 4 round nothing, so frames unnormalise exactly
REPORT = {}


def dev():
    assert torch.cuda.is_available()
    torch.cuda.init()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nworst err / bound per case (and the fraction of live rows whose atom type was compared):")
        for k, v in REPORT.items():
            print(f"  {k}: {v}")


# ------------------------------------------------------------------------------------------------------------- CPU
SCALAR_CASES = [("polynomial_2", 1, 1, 1, 3), ("polynomial_2", 2, 2, 2, 5), ("polynomial_2", 50, 50, 50, 4),
                ("polynomial_2", 50, 50, 4, 4), ("polynomial_2", 1000, 1000, 1000, 4), ("polynomial_2", 1000, 1000, 7, 64),
                ("polynomial_2", 50, 20, 20, 4), ("polynomial_2", 50, 20, 3, 2), ("cosine", 200, 200, 200, 16)]


@pytest.mark.parametrize("inpainting", [False, True])
@pytest.mark.parametrize("schedule,table_T,T,K,B", SCALAR_CASES)
def test_step_scalars_equal_the_step_coefficient_table(schedule, table_T, T, K, B, inpainting):
    """orc.step_scalars equals every row of EDM.step_coefficients(K, B) bit for bit -- t, a, b, c, qa, qb and the final row
    1/alpha_0, sigma_0, SNR(-0.5 g_0), sigma_0/alpha_0 -- for polynomial_2 at T = 1, 2, 50, 1000, the n_steps override (T = 20
    on a 50-step table) and cosine; the frame column follows the last-writer rule; every molecule's scalars are equal."""
    cls = InpaintingEDM if inpainting else EDM
    edm = cls(dynamics=torch.nn.Identity(), in_node_nf=8, n_dims=3, timesteps=table_T, noise_schedule=schedule,
              noise_precision=1e-5, loss_type='l2', norm_values=NORM)
    edm.T = T
    rows = edm.step_coefficients(K, B)
    gamma = orc.gamma_table(schedule, table_T, 1e-5)
    assert torch.equal(gamma, edm.gamma.gamma.detach())
    for r in range(T):
        s = T - 1 - r
        sc = orc.step_scalars(gamma, s, T, B, table_T)
        for v in sc.values():
            assert v.dtype == torch.float32 and v.shape == (B, 1) and torch.equal(v, v[:1].expand(B, 1))
        got = (rows[r].t, rows[r].a, rows[r].b, rows[r].c)
        assert got == tuple(float(sc[k][0]) for k in ("t", "a", "b", "c")), (s, got)
        if inpainting:
            assert (rows[r].qa, rows[r].qb) == (float(sc["qa"][0]), float(sc["qb"][0])), s
        else:
            assert (rows[r].qa, rows[r].qb) == (0.0, 0.0)
        f = (s * K) // T
        last = f > 0 and (s == 0 or ((s - 1) * K) // T != f)
        assert rows[r].frame == (f if last else -1), (s, rows[r].frame)
    fin = orc.step_scalars(gamma, -1, T, B, table_T)
    assert (rows[T].t, rows[T].a, rows[T].b, rows[T].c, rows[T].frame) == (
        0.0, float(fin["inv_alpha0"][0]), float(fin["sigma0"][0]), float(fin["snr0"][0]), -1)
    assert rows[T].qa == (float(fin["qa0"][0]) if inpainting else 0.0)


def replay_linker(sd, cfg, gamma, T, keep, x, h, nm, fm, lm, em, ctx, draws, forward):
    """EDM.sample_chain driven from outside through the oracle's step functions: z_T from draw 0 as k_init_z forms it, step
    s = T-1-r with draw r+1, the final step with draw T+1, frames by (s * keep) // T."""
    B = x.shape[0]
    xh = torch.cat([x / NORM[0], h.float() / NORM[1]], dim=2)
    z = xh * fm + (draws[0] * lm) * lm
    chain = torch.zeros((keep,) + z.shape)
    for s in reversed(range(T)):
        sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
        z = orc.linker_step(z, forward(sd, cfg, sc["t"], z, nm, lm, em, ctx), sc, draws[T - s], fm, lm)
        chain[(s * keep) // T] = torch.cat([z[..., :3] * NORM[0], z[..., 3:] * NORM[1]], dim=2)
    out = orc.linker_final(z, forward(sd, cfg, torch.zeros((B, 1)), z, nm, lm, em, ctx),
                           orc.step_scalars(gamma, -1, T, B, gamma.numel() - 1), draws[T + 1], fm, lm)
    chain[0] = orc.final_frame(out, nm, 3, NORM)
    return chain


def replay_inpaint(sd, cfg, gamma, T, keep, x, h, nm, fm, lm, em, ctx, draws, forward):
    """InpaintingEDM.sample_chain the same way: z_T = draw 0, step s with draws 2r+1 (p) and 2r+2 (q), final draws 2T+1, 2T+2."""
    B = x.shape[0]
    xh = torch.cat([x / NORM[0], h.float() / NORM[1]], dim=2)
    nmf = nm.float()
    z = draws[0]
    chain = torch.zeros((keep,) + z.shape)
    for s in reversed(range(T)):
        r = T - 1 - s
        sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
        z = orc.inpaint_step(z, forward(sd, cfg, sc["t"], z, nm, None, em, ctx), sc, draws[2 * r + 1], draws[2 * r + 2],
                             xh, nmf, fm, lm)
        chain[(s * keep) // T] = torch.cat([z[..., :3] * NORM[0], z[..., 3:] * NORM[1]], dim=2)
    out_l, out_f = orc.inpaint_final(z, forward(sd, cfg, torch.zeros((B, 1)), z, nm, None, em, ctx),
                                     orc.step_scalars(gamma, -1, T, B, gamma.numel() - 1), draws[2 * T + 1], draws[2 * T + 2])
    chain[0] = orc.final_frame(out_l, nm, 3, NORM) * lm + orc.final_frame(out_f, nm, 3, NORM) * fm
    return chain


@pytest.mark.parametrize("name", ["chain_cfg1", "chain_cfg1_nsteps20", "inpaint_chain_cfg1"])
def test_step_functions_replay_the_reference_golden_chain(name):
    """The step functions in fp32 with the oracle's eps, driven with the draw indexing, z_T and frame bookkeeping the GPU
    checks below use, reproduce the live reference's chain exactly (max |delta| = 0)."""
    meta, a = helpers.load_golden(name)
    spec = helpers.spec_by_name(meta["spec"])
    inpaint = name.startswith("inpaint")
    ddpm, hp = helpers.build_ddpm(spec, meta["seed"], diffusion_steps=meta.get("table_timesteps", spec.T), inpainting=inpaint)
    assert helpers.state_sha(ddpm.edm.dynamics.state_dict()) == meta["sha"]
    data = orc.collate_molecules(synthetic.make_items(spec, batch=meta["batch"]))
    gamma = orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])
    cfg = helpers.oracle_cfg(hp)
    T, keep = meta["T"], meta["keep_frames"]
    if inpaint:
        cfg.centering = True
        tpl = data
        x = orc.remove_partial_mean(tpl['positions'], tpl['atom_mask'], tpl['atom_mask'])
        B, N = x.shape[:2]
        draws = helpers.inpaint_noise_tensor(meta["noise_seed"], T, B, N, spec.F, tpl['atom_mask'], tpl['fragment_mask'])
        replay = replay_inpaint
    else:
        tpl = orc.linker_templates(data, data['linker_mask'].sum(1).view(-1).int())
        x = orc.remove_partial_mean(tpl['positions'], tpl['atom_mask'], tpl['fragment_mask'])
        B, N = x.shape[:2]
        draws = helpers.noise_tensor(meta["noise_seed"], T, B, N, spec.F)
        replay = replay_linker
    with torch.no_grad():
        chain = replay(ddpm.edm.dynamics.state_dict(), cfg, gamma, T, keep, x, tpl['one_hot'], tpl['atom_mask'],
                       tpl['fragment_mask'], tpl['linker_mask'], tpl['edge_mask'], tpl['fragment_mask'], draws,
                       orc.dynamics_forward)
    assert chain.shape == a["chain"].shape
    assert (chain - a["chain"]).abs().max().item() == 0.0


# ---------------------------------------------------------------------------------------------------- batches, models
def fc_batch(sizes, F, seed):
    """A collated FC batch: molecule b has sizes[b] = (atoms, linker atoms), fragments first; (0, 0) is a fully padded row."""
    g = torch.Generator().manual_seed(seed)
    items = []
    for b, (n, l) in enumerate(sizes):
        ar = torch.arange(n)
        items.append(dict(uuid=b, name=str(b), positions=2.5 * torch.randn((n, 3), generator=g),
                          one_hot=torch.nn.functional.one_hot(torch.randint(0, F, (n,), generator=g), F).float(),
                          anchors=torch.zeros(n), fragment_mask=(ar < n - l).float(), linker_mask=(ar >= n - l).float(),
                          num_atoms=n))
    batch = collate(items)
    return dict(x=batch['positions'], h=batch['one_hot'], node_mask=batch['atom_mask'], fragment_mask=batch['fragment_mask'],
                linker_mask=batch['linker_mask'], edge_mask=batch['edge_mask'], context=batch['fragment_mask'])


def pocket_batch(sizes, F, seed):
    """A collated pocket batch: molecule b has sizes[b] = (fragment, pocket, linker) atoms on a jittered 1.6 A lattice (so
    a 4 A graph has a few dozen neighbours per atom), fragments first, then pocket, then linker atoms."""
    g = torch.Generator().manual_seed(seed)
    items = []
    for nf, npk, nl in sizes:
        n = nf + npk + nl
        side = math.ceil(n ** (1 / 3))
        ax = torch.arange(side, dtype=torch.float32) * 1.6
        grid = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), dim=-1).reshape(-1, 3)[:n]
        pos = grid - grid.mean(0) + 0.2 * torch.randn(grid.shape, generator=g)
        items.append(pocket_item(g, pos, 'f' * nf + 'p' * npk + 'l' * nl, F))
    batch = collate(items)
    fo = batch['fragment_only_mask']
    return dict(x=batch['positions'], h=batch['one_hot'], node_mask=batch['atom_mask'], fragment_mask=batch['fragment_mask'],
                linker_mask=batch['linker_mask'], edge_mask=batch['edge_mask'],
                context=torch.cat([fo, batch['fragment_mask'] - fo], dim=-1))


def dyadic_bias(F):
    return [(-1) ** j * (j + 1) / 8 for j in range(F)]


def known_eps_model(F, table_T, impl, graph_type="FC", inpainting=False, schedule="polynomial_2", bias=None):
    """An EDM whose dynamics output is eps_x = 0, eps_h = bias_j * node_mask exactly: embedding_out.weight and every
    coord_mlp's last Linear zeroed, embedding_out.bias[:F] = bias (dyadic, distinct by default)."""
    pocket = graph_type != "FC"
    spec = synthetic.WorkloadSpec("steps", B=1, N=8, n_min=8, l_min=1, l_max=1, F=F, L=2, T=table_T, seed=9,
                                  pocket=1 if pocket else 0, graph_type=graph_type,
                                  hparams=dict(diffusion_noise_schedule=schedule))
    ddpm, hp = helpers.build_ddpm(spec, 9, edge_impl=impl, inpainting=inpainting)
    bias = dyadic_bias(F) if bias is None else bias
    with torch.no_grad():
        seen = 0
        for name, p in ddpm.edm.dynamics.named_parameters():
            if name.endswith("embedding_out.weight") or name.endswith("coord_mlp.4.weight"):
                p.zero_()
                seen += 1
            elif name.endswith("embedding_out.bias"):
                p.zero_()
                p[:F] = torch.tensor(bias)
                seen += 1
        assert seen == 2 + hp['n_layers']
    return ddpm.edm, hp, bias


def sample(edm, kw, T, keep, source, seed, inpainting):
    """(chain, draws): the chain sampled with the draws from `source` and the draws it must have used, on the device --
    'tensor' injects them (the linker sampler's raw draws, or inpaint_noise_tensor's prepared ones), 'stream' is the
    default generator's batch stream (expected: edm.draw_noise from the entry state, or dl_noise_fill_inpaint, which
    runs the device functions k_inpaint draws with), 'seeds' the per-molecule streams (expected: one-molecule draws after
    torch.cuda.manual_seed(seed_b))."""
    d = dev()
    kw = {k: (None if v is None else v.to(d)) for k, v in kw.items()}
    B, N = kw['x'].shape[:2]
    F = edm.in_node_nf
    if source == "tensor":
        if inpainting:
            draws = helpers.inpaint_noise_tensor(seed, T, B, N, F, kw['node_mask'].cpu(), kw['fragment_mask'].cpu()).to(d)
        else:
            draws = helpers.noise_tensor(seed, T, B, N, F).to(d)
        return edm.sample_chain(**kw, keep_frames=keep, noise=draws), draws
    if source == "seeds":
        assert not inpainting
        seeds = [seed + 7919 * b for b in range(B)]
        parts = []
        for s in seeds:
            torch.cuda.manual_seed(s)
            parts.append(edm.draw_noise(T + 2, 1, N, d))
        return edm.sample_chain(**kw, keep_frames=keep, seeds=seeds), torch.cat(parts, dim=1)
    torch.manual_seed(seed)
    if inpainting:
        lib = _native.load_library()
        gen = torch.cuda.default_generators[d.index or 0]
        draws = torch.empty((2 * T + 3, B, N, 3 + F), device=d)
        used = C.c_uint64(0)
        nm8 = kw['node_mask'].reshape(B, N).to(torch.int8).contiguous()
        fm32 = kw['fragment_mask'].reshape(B, N).float().contiguous()
        eng = edm.dynamics.engine(d.index or 0)
        _native.check(lib.dl_noise_fill_inpaint(eng, T, B, N, nm8.data_ptr(), fm32.data_ptr(), gen.initial_seed(),
                                                gen.get_offset(), draws.data_ptr(), C.byref(used),
                                                torch.cuda.current_stream(d).cuda_stream), "dl_noise_fill_inpaint")
    else:
        draws = edm.draw_noise(T + 2, B, N, d)
    torch.manual_seed(seed)
    return edm.sample_chain(**kw, keep_frames=keep), draws


# -------------------------------------------------------------------------------------------------------- checking
class Checker:
    """Compares GPU values with fp64 references under elementwise bounds and records the worst err / bound of a case."""

    def __init__(self, label):
        self.label, self.worst, self.decided, self.live = label, 0.0, 0, 0

    def close(self, what, got, ref, bound, rows):
        """|got - ref| <= bound on `rows` (B,N); where the bound is 0 the values must be equal."""
        err = (got - ref).abs()
        m = rows[..., None].expand_as(err)
        bad = m & ~(err <= bound)
        if bad.any():
            i = torch.nonzero(bad)[0].tolist()
            raise AssertionError(f"{self.label}, {what}: {int(bad.sum())} elements out of bound; first at {i}: got "
                                 f"{got[tuple(i)].item():.9g}, fp64 {ref[tuple(i)].item():.9g}, bound {bound[tuple(i)].item():.3g}")
        r = torch.where(m & (bound > 0), err / bound.clamp_min(1e-300), 0.0)
        self.worst = max(self.worst, r.max().item() if r.numel() else 0.0)

    def types(self, what, got_onehot, ref_h, bound_h, rows, nm):
        """One-hot rows sum to the node mask; the GPU's type equals the fp64 argmax wherever the top-two gap exceeds twice
        the bound of the row's feature values."""
        assert torch.equal(got_onehot.sum(-1), nm.expand(got_onehot.shape[:2])), f"{self.label}, {what}: one-hot rows"
        assert ((got_onehot == 0) | (got_onehot == 1)).all()
        if ref_h.shape[-1] > 1:
            top = ref_h.topk(2, dim=-1).values
            gap = top[..., 0] - top[..., 1]
        else:
            gap = torch.full(ref_h.shape[:2], math.inf, dtype=ref_h.dtype, device=ref_h.device)
        dec = rows & (gap > 2 * bound_h.amax(-1))
        want = ref_h.argmax(-1)
        got = got_onehot.argmax(-1)
        bad = dec & (got != want)
        assert not bad.any(), f"{self.label}, {what}: atom types differ at {torch.nonzero(bad)[:5].tolist()}"
        self.decided += int(dec.sum())
        self.live += int(rows.sum())

    def record(self):
        REPORT[self.label] = (f"{self.worst:.3g}", f"{self.decided / max(self.live, 1):.3f}")


def f64(v, d):
    return v.to(device=d, dtype=torch.float64)


def unnorm_frame(frame):
    """A stored frame in the normalised units of z (x * 1 and h * 4 are exact)."""
    return torch.cat([frame[..., :3] / NORM[0], frame[..., 3:] / NORM[1]], dim=-1)


def scalars(gamma, T, B):
    return {s: orc.step_scalars(gamma, s, T, B, gamma.numel() - 1) for s in range(-1, T)}


def stored_steps(T, keep):
    """frame -> the reverse step s whose z_s it holds (the last writer), frames 1..keep-1."""
    return {(s * keep) // T: s for s in range(T - 1, 0, -1) if (s * keep) // T > 0}


def check_linker_chain(label, chain, kw, draws, bias, gamma, T, keep):
    d = chain.device
    chain = f64(chain, d)
    B, N, D = chain.shape[1:]
    nm, fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    live, lk, fr = nm[..., 0] != 0, lm[..., 0] != 0, fm[..., 0] != 0
    draws = f64(draws, d)
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    eps = torch.zeros_like(xh)
    eps[..., 3:] = f64(torch.tensor(bias), d) * nm
    z_T = xh * fm + (draws[0] * lm) * lm
    sc = scalars(gamma, T, B)
    frame_of = {s: f for f, s in stored_steps(T, keep).items()}
    ck = Checker(label)
    assert torch.equal(chain[:, ~live], torch.zeros_like(chain[:, ~live])), f"{label}: a padded row is not 0"
    z, e = z_T, torch.zeros_like(z_T)
    for s in range(T - 1, -1, -1):
        a, b, c = (orc._sc(sc[s], k, z) for k in ("a", "b", "c"))
        n = draws[T - s]
        ref = orc.linker_step(z, eps, sc[s], n, fm, lm)
        e = (e / a.abs() + 4 * U * ((z.abs() + e) / a.abs() + (b * eps * lm).abs() + (c * n * lm).abs())) * lm + e * fm
        z = ref
        if s in frame_of:
            got = unnorm_frame(chain[frame_of[s]])
            assert torch.equal(got[fr & ~lk], z_T[fr & ~lk]), f"{label}: a fragment row of frame {frame_of[s]} differs from z_T"
            ck.close(f"step s={s}", got, z, e, live)
            z, e = got, torch.zeros_like(e)
    inv_a0, sig0, snr0 = (orc._sc(sc[-1], k, z) for k in ("inv_alpha0", "sigma0", "snr0"))
    n = draws[T + 1]
    out = orc.linker_final(z, eps, sc[-1], n, fm, lm)
    e = (inv_a0 * e + 4 * U * (inv_a0 * (z.abs() + e) + inv_a0 * (sig0 * eps * lm).abs() + (snr0 * n * lm).abs())) * lm
    got = chain[0]
    assert torch.equal(got[..., :3][fr & ~lk], z_T[..., :3][fr & ~lk]), f"{label}: a final fragment row differs from z_T"
    ck.close("final x", got[..., :3], out[..., :3] * NORM[0], e[..., :3] * NORM[0], live)
    ck.types("final h", got[..., 3:], out[..., 3:], e[..., 3:], live, nm[..., 0])
    ck.record()


def projection_bound(zn, pre, nm, xd):
    """Error of the GPU's centre-of-mass mean of the coordinate columns of zn, per molecule (B,1,3): the mean of the incoming
    errors `pre` plus the fp32 summation (k_inpaint: strided per-thread partials, shuffle tree, 8 warp partials)."""
    N = zn.shape[1]
    chain_len = math.ceil(N * math.gcd(xd, 256) / 256) + 16
    cnt = nm.sum(1, keepdim=True)
    return ((pre[..., :3] * nm).sum(1, keepdim=True) + chain_len * U * (zn[..., :3] * nm).abs().sum(1, keepdim=True)) / cnt


def check_inpaint_chain(label, chain, kw, draws, bias, gamma, T, keep):
    d = chain.device
    chain = f64(chain, d)
    B, N, D = chain.shape[1:]
    nm, fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    live = nm[..., 0] != 0
    draws = f64(draws, d)
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    eps = torch.zeros_like(xh)
    eps[..., 3:] = f64(torch.tensor(bias), d) * nm
    sc = scalars(gamma, T, B)
    frame_of = {s: f for f, s in stored_steps(T, keep).items()}
    ck = Checker(label)
    assert torch.equal(chain[:, ~live], torch.zeros_like(chain[:, ~live])), f"{label}: a padded row is not 0"
    z, e = draws[0], torch.zeros_like(xh)
    for s in range(T - 1, -1, -1):
        r = T - 1 - s
        a, b, c, qa, qb = (orc._sc(sc[s], k, z) for k in ("a", "b", "c", "qa", "qb"))
        n_p, n_q = draws[2 * r + 1], draws[2 * r + 2]
        za = z.abs() + e
        # before the projection: zn = (z/a - b eps + c n_p) lm + (qa z + qb xh fm + c n_q) fm
        zn = (z / a - b * eps + c * n_p) * lm + (qa * z + qb * (xh * fm) + c * n_q) * fm
        pre = ((e / a.abs() + 4 * U * (za / a.abs() + (b * eps).abs() + (c * n_p).abs())) * lm
               + (qa.abs() * e + 4 * U * (qa.abs() * za + (qb * xh * fm).abs() + (c * n_q).abs())) * fm)
        ref = orc.inpaint_step(z, eps, sc[s], n_p, n_q, xh, nm, fm, lm)
        e = pre.clone()
        e[..., :3] = (pre[..., :3] + projection_bound(zn, pre, nm, D) + U * ref[..., :3].abs()) * nm
        z = ref
        if s in frame_of:
            got = unnorm_frame(chain[frame_of[s]])
            ck.close(f"step s={s}", got, z, e, live)
            z, e = got, torch.zeros_like(e)
    inv_a0, sig0, snr0, qa0 = (orc._sc(sc[-1], k, z) for k in ("inv_alpha0", "sigma0", "snr0", "qa0"))
    n_p, n_q = draws[2 * T + 1], draws[2 * T + 2]
    out_l, out_f = orc.inpaint_final(z, eps, sc[-1], n_p, n_q)
    za = z.abs() + e
    e_l = inv_a0 * e + 4 * U * (inv_a0 * za + inv_a0 * (sig0 * eps).abs() + (snr0 * n_p).abs())
    e_f = inv_a0 * e + 4 * U * (inv_a0 * za + (qa0 * n_q).abs())
    got = chain[0]
    ck.close("final x", got[..., :3], (out_l[..., :3] * lm + out_f[..., :3] * fm) * NORM[0],
             (e_l[..., :3] * lm + e_f[..., :3] * fm) * NORM[0], live)
    lk, fr = (lm[..., 0] != 0) & live, (fm[..., 0] != 0) & live
    ck.types("final h (p variant, linker rows)", got[..., 3:] * lm, out_l[..., 3:], e_l[..., 3:], lk, (nm * lm)[..., 0])
    ck.types("final h (q variant, fragment rows)", got[..., 3:] * fm, out_f[..., 3:], e_f[..., 3:], fr, (nm * fm)[..., 0])
    ck.record()


# ------------------------------------------------------------------------------------------------------------- GPU
def gamma_of(hp):
    return orc.gamma_table(hp['diffusion_noise_schedule'], hp['diffusion_steps'], hp['diffusion_noise_precision'])


# label -> (F, molecule sizes (atoms, linker atoms), T, table T, schedule, keep_frames, draws). B * N = 48, 33 and 95 nodes
# (0, 1 and 15 mod 16, the node groups of k_finish); a 1-atom molecule, a fully padded row and an empty linker; 3 + F = 4, 11, 16.
LINKER_FC = {
    "F1_T50": (1, [(12, 4), (1, 1), (0, 0), (7, 0)], 50, 50, "polynomial_2", 50, "tensor"),
    "F8_T2": (8, [(11, 3), (6, 2), (9, 9)], 2, 2, "polynomial_2", 2, "stream"),
    "F13_T1": (13, [(19, 5), (1, 1), (0, 0), (10, 0), (14, 6)], 1, 1, "polynomial_2", 1, "seeds"),
    "nsteps20_of_50": (8, [(16, 5), (12, 3), (9, 4), (16, 16)], 20, 50, "polynomial_2", 20, "tensor"),
    "cosine_T200": (9, [(24, 6), (15, 4)], 200, 200, "cosine", 200, "stream"),
    "keep4_T50": (8, [(11, 3), (6, 2), (9, 4)], 50, 50, "polynomial_2", 4, "seeds"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["simt", "auto"])
@pytest.mark.parametrize("case", list(LINKER_FC))
def test_linker_sampler_steps_vs_fp64(case, impl):
    F, sizes, T, table_T, schedule, keep, source = LINKER_FC[case]
    edm, hp, bias = known_eps_model(F, table_T, impl, schedule=schedule)
    edm.T = T
    kw = fc_batch(sizes, F, seed=len(sizes) * 100 + F)
    chain, draws = sample(edm, kw, T, keep, source, 17, False)
    check_linker_chain(f"linker {case} {impl} {source}", chain, kw, draws, bias, gamma_of(hp), T, keep)


POCKET_LINKER = {
    # the benchmarked pocket shape (cfg4_pockets) at its T, and the cut-off graphs' largest N
    "FC-10A-4A_N300_T1000": ("FC-10A-4A", None, 1000, "stream"),
    "4A_N4000_T3": ("4A", [(30, 3960, 10), (25, 2900, 12)], 3, "seeds"),
}


def pocket_inputs(sizes, B, seed):
    if sizes is None:
        batch = collate(synthetic.make_items(synthetic.SPECS["cfg4_pockets"], batch=B))
        fo = batch['fragment_only_mask']
        return dict(x=batch['positions'], h=batch['one_hot'], node_mask=batch['atom_mask'],
                    fragment_mask=batch['fragment_mask'], linker_mask=batch['linker_mask'], edge_mask=batch['edge_mask'],
                    context=torch.cat([fo, batch['fragment_mask'] - fo], dim=-1))
    return pocket_batch(sizes, 9, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(POCKET_LINKER))
def test_pocket_linker_sampler_steps_vs_fp64(case):
    graph_type, sizes, T, source = POCKET_LINKER[case]
    edm, hp, bias = known_eps_model(9, T, "auto", graph_type=graph_type)
    kw = pocket_inputs(sizes, 4, 5)
    chain, draws = sample(edm, kw, T, T, source, 23, False)
    check_linker_chain(f"linker pocket {case} {source}", chain, kw, draws, bias, gamma_of(hp), T, T)


# label -> (graph type, F, molecule sizes, T, draws, impls): FC molecules (atoms, linker atoms) or pocket molecules (fragment,
# pocket, linker atoms); ragged batches, N around k_inpaint's 256-thread CTA and the cut-off graphs' N = 4000
INPAINT = {
    "FC_N30_T50": ("FC", 8, [(30, 6), (22, 4), (25, 9), (7, 1)], 50, "tensor", ("simt", "auto")),
    "FC_N255_T2": ("FC", 8, [(255, 10), (180, 30)], 2, "stream", ("auto",)),
    "FC_N256_T1": ("FC", 8, [(256, 8), (100, 5)], 1, "tensor", ("auto",)),
    "FC_N257_T2_F13": ("FC", 13, [(257, 12), (200, 7), (40, 3)], 2, "stream", ("simt", "auto")),
    "FC-10A-4A_N300_T2": ("FC-10A-4A", 9, None, 2, "stream", ("auto",)),
    "4A_N4000_T2": ("4A", 9, [(30, 3960, 10), (25, 2900, 12)], 2, "stream", ("auto",)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case,impl", [(c, i) for c, v in INPAINT.items() for i in v[5]])
def test_inpainting_sampler_steps_vs_fp64(case, impl):
    graph_type, F, sizes, T, source, _ = INPAINT[case]
    edm, hp, bias = known_eps_model(F, T, impl, graph_type=graph_type, inpainting=True)
    kw = fc_batch(sizes, F, seed=31) if graph_type == "FC" else pocket_inputs(sizes, 2, 6)
    chain, draws = sample(edm, kw, T, T, source, 29, True)
    check_inpaint_chain(f"inpaint {case} {impl} {source}", chain, kw, draws, bias, gamma_of(hp), T, T)


@pytest.mark.gpu
@pytest.mark.parametrize("inpainting", [False, True])
def test_exact_atom_type_tie_gives_the_first_feature(inpainting):
    """Equal biases, equal feature columns in the input and in every draw: every feature of every atom ties through the whole
    chain, and k_finish's 16-lane argmax (linker sampler) and both final variants of k_inpaint pick feature 0, as torch.argmax
    does."""
    F, T = 8, 2
    edm, hp, bias = known_eps_model(F, T, "simt", inpainting=inpainting, bias=[0.5] * F)
    kw = fc_batch([(6, 3), (5, 2), (4, 4 if not inpainting else 1)], F, seed=3)
    kw['h'] = torch.full_like(kw['h'], 0.25)
    B, N = kw['x'].shape[:2]
    d = dev()
    if inpainting:
        draws = helpers.inpaint_noise_tensor(41, T, B, N, F, kw['node_mask'], kw['fragment_mask'])
    else:
        draws = helpers.noise_tensor(41, T, B, N, F)
    draws[..., 3:] = draws[..., 3:4].clone()
    kwd = {k: v.to(d) for k, v in kw.items()}
    chain = edm.sample_chain(**kwd, keep_frames=1, noise=draws.to(d)).cpu()
    live = kw['node_mask'].reshape(B, N) != 0
    want = torch.zeros((B, N, F))
    want[..., 0] = live.float()
    assert torch.equal(chain[0][..., 3:], want)


@pytest.mark.gpu
@pytest.mark.parametrize("n_pos", [255, 256, 257, 4000])
def test_restore_frame_vs_fp64(n_pos):
    """k_restore_frame (dl_restore_frame2, generate.py:165-171): chain[0]'s coordinates plus the mean of the input batch's
    positions over an anchor com_mask, with the template's N != the input's N_pos and anchors up to row N_pos - 1."""
    d = dev()
    g = torch.Generator().manual_seed(n_pos)
    B, F = 3, 9
    N = n_pos + 5 if n_pos % 2 else n_pos - 7
    sizes = [n_pos, n_pos // 2 + 1, 9]
    pos_mask = torch.stack([(torch.arange(n_pos) < s).float() for s in sizes])
    positions = (3 * torch.randn((B, n_pos, 3), generator=g) + torch.tensor([11.0, -7.0, 3.5])) * pos_mask[..., None]
    anchors = (torch.rand((B, n_pos), generator=g) < 0.1).float() * pos_mask
    for b, s in enumerate(sizes):
        anchors[b, s - 1] = 1.0
    node_mask = torch.stack([(torch.arange(N) < min(s, N)).to(torch.int8) for s in sizes])[..., None]
    chain0 = torch.randn((B, N, 3 + F), generator=g)
    got = output.restore_frame(chain0.clone().to(d), positions.to(d), anchors[..., None].to(d), node_mask.to(d)).cpu()
    p64, m64 = positions.double(), anchors.double()[..., None]
    cnt = m64.sum(1, keepdim=True)
    mean = (p64 * m64).sum(1, keepdim=True) / cnt
    want = chain0[..., :3].double() + mean * node_mask.double()
    L = math.ceil(n_pos / 256) + 16
    bound = (L * U * (p64 * m64).abs().sum(1, keepdim=True) / cnt + U * mean.abs()) * node_mask.double() + U * want.abs()
    err = (got[..., :3].double() - want).abs()
    assert (err <= bound).all(), (err / bound).max().item()
    assert torch.equal(got[..., 3:], chain0[..., 3:])
    REPORT[f"restore_frame N_pos={n_pos}"] = f"{(err / bound).max().item():.3g}"


@pytest.mark.gpu
def test_inpainting_draws_at_n4000_vs_fp64_projection():
    """dl_noise_fill_inpaint (k_com_free_draws, the device functions k_inpaint draws with) at N = 4000 against the fp64
    projection of torch's raw draws from the same generator state: features and masked rows exact, coordinates within the
    bound of the kernel's fp32 sums (ceil(3N / 256) strided partials, then the shuffle and warp-partial tree)."""
    d = dev()
    lib = _native.load_library()
    edm, hp, _ = known_eps_model(9, 1, "auto", graph_type="4A", inpainting=True)
    B, N, T, F = 2, 4000, 1, 9
    g = torch.Generator().manual_seed(4)
    nm = torch.stack([(torch.arange(N) < s).float() for s in (N, 3100)])[..., None]
    fm = nm * (torch.rand((B, N, 1), generator=g) < 0.3).float()
    torch.manual_seed(77)
    gen = torch.cuda.default_generators[d.index or 0]
    seed, offset = gen.initial_seed(), gen.get_offset()
    raw = []
    for _ in range(2 * T + 3):
        raw.append(torch.cat([torch.randn((B, N, 3), device=d), torch.randn((B, N, F), device=d)], dim=2))
    got = torch.empty((2 * T + 3, B, N, 3 + F), device=d)
    used = C.c_uint64(0)
    nm8 = nm.reshape(B, N).to(torch.int8).to(d)
    fm32 = fm.reshape(B, N).to(d).contiguous()
    _native.check(lib.dl_noise_fill_inpaint(edm.dynamics.engine(d.index or 0), T, B, N, nm8.data_ptr(), fm32.data_ptr(), seed,
                                            offset, got.data_ptr(), C.byref(used), torch.cuda.current_stream(d).cuda_stream),
                  "dl_noise_fill_inpaint")
    assert offset + used.value == gen.get_offset()
    worst = 0.0
    L = math.ceil(3 * N / 256) + 16
    for r, m in enumerate([nm] + [nm, fm] * T + [nm, nm]):
        m = f64(m, d)
        xm = raw[r].double() * m
        cnt = m.sum(1, keepdim=True)
        want = xm[..., :3] - (xm[..., :3].sum(1, keepdim=True) / cnt) * m
        bound = (L * U * xm[..., :3].abs().sum(1, keepdim=True) / cnt) * m + 2 * U * want.abs()
        gr = got[r].double()
        assert torch.equal(gr[..., 3:], xm[..., 3:]), r
        err = (gr[..., :3] - want).abs()
        assert (err <= bound).all(), (r, (err / bound).max().item())
        worst = max(worst, (err / bound.clamp_min(1e-300)).max().item())
    REPORT["dl_noise_fill_inpaint N=4000"] = f"{worst:.3g}"


# ------------------------------------------------------------------------------------------- GPU, real weights (tier 2)
# The synthetic weights (coord_mlp gain 100): a nonzero velocity for k_inpaint to centre over N > 256 atoms, and a dynamics
# output that depends on t and on the masks, so a wrong time row or mask in the loop's forward changes eps. At a few steps s
# the oracle forward runs in fp64 and in fp32 on the GPU's own z_{s+1}, the step is applied in fp64 and in the reference's
# fp32 order, and each live row of the GPU's z_s must meet, on the coordinate and on the feature columns,
#   |got - ref64| <= max(C_DRIFT * drift_i, TAU * S_b) + (the rounding bound of the step's non-eps terms)
# with drift_i = max |ref32 - ref64| on the row and S_b the molecule's largest |b * eps64| (fp64_rows' per-row rule, applied
# to the eps term of the step). The final step is checked as the composite z_1 -> z_0 -> final sample.
# label -> (spec, molecules, inpainting, draws, graph type). The inpainting pocket case runs the 4A graph: InpaintingEDM calls
# the dynamics without a linker mask (edm.py:626-633), which FC-10A-4A's ligand class needs (egnn.py:566-570).
REAL_WEIGHTS = {
    "cfg2_zinc_B16_T500": ("cfg2_zinc", 16, False, "stream", "FC"),
    "cfg4_pockets_B3_T1000": ("cfg4_pockets", 3, False, "seeds", "FC-10A-4A"),
    "inpaint_cfg4_pockets_4A_B2_N300_T1000": ("cfg4_pockets", 2, True, "stream", "4A"),
}


def oracle_eps(sd, cfg, t, z, kw, inpainting, dtype, d):
    """The option-aware oracle's Dynamics.forward in `dtype` on the device, as the sampler calls it (edm.py:196, 626-633)."""
    cast = lambda v: None if v is None else (v.to(device=d, dtype=dtype) if v.is_floating_point() else v.to(d))
    with torch.no_grad(), torch.device(d), _full_fp32_matmul():
        return eo.dynamics_forward({k: cast(v) for k, v in sd.items()}, cfg, cast(t), cast(z), cast(kw['node_mask']),
                                   None if inpainting else cast(kw['linker_mask']), cast(kw['edge_mask']),
                                   cast(kw['context']))


def rowwise(ck, what, got, ref64, ref32, rounding, scale, live):
    """fp64_rows' per-row rule on the coordinate and the feature columns, plus the rounding bound of the non-eps terms."""
    for cols in (slice(0, 3), slice(3, None)):
        drift = (ref32[..., cols] - ref64[..., cols]).abs().amax(-1, keepdim=True)
        bound = torch.maximum(C_DRIFT * drift, TAU * scale) + rounding[..., cols]
        ck.close(what, got[..., cols], ref64[..., cols], bound, live)


@pytest.mark.gpu
@pytest.mark.parametrize("opts", ["default", "tanh_mean"])
@pytest.mark.parametrize("case", list(REAL_WEIGHTS))
def test_sampler_steps_with_real_weights_vs_fp64(case, opts):
    spec_name, B, inpainting, source, graph_type = REAL_WEIGHTS[case]
    tanh = mean = opts == "tanh_mean"
    spec = dataclasses.replace(synthetic.SPECS[spec_name], graph_type=graph_type, hparams=eo.options_kw(tanh, mean))
    ddpm, hp = helpers.build_ddpm(spec, 0, inpainting=inpainting)
    edm, T, d = ddpm.edm, spec.T, dev()
    cfg = eo.oracle_cfg(hp)
    cfg.centering = inpainting
    kw = sampler_inputs(ddpm, collate(synthetic.make_items(spec, batch=B)))
    chain, draws = sample(edm, kw, T, T, source, 53, inpainting)
    sd = {k: v.detach() for k, v in edm.dynamics.state_dict().items()}
    gamma = gamma_of(hp)
    chain64, draws64, draws32 = f64(chain, d), f64(draws, d), draws.float()
    N, D = chain.shape[2:]
    nm, fm, lm = (f64(kw[k], d).reshape(B, N, 1) for k in ("node_mask", "fragment_mask", "linker_mask"))
    live = nm[..., 0] != 0
    xh = torch.cat([f64(kw['x'], d) / NORM[0], f64(kw['h'], d) / NORM[1]], dim=2)
    z_T = draws64[0] if inpainting else xh * fm + (draws64[0] * lm) * lm
    ck = Checker(f"real weights {case} {opts} {source}")

    def z_at(s):                                                          # the GPU's z_s; z_T rebuilt exactly
        return z_T if s == T else unnorm_frame(chain64[s])

    def step(s, z, eps, dtype):
        """(z_s, zn, rounding): the step in `dtype`; before the projection (inpainting) and the non-eps rounding bound."""
        sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
        dr = draws64 if dtype == torch.float64 else draws32
        masks = [m.to(dtype) for m in (nm, fm, lm)]
        if not inpainting:
            n = dr[T - s]
            out = orc.linker_step(z, eps, sc, n, masks[1], masks[2])
            a, c = orc._sc(sc, "a", z), orc._sc(sc, "c", z)
            return out, None, 4 * U * ((z.abs() / a) + (c * n * masks[2]).abs()) * masks[2]
        r = T - 1 - s
        n_p, n_q = dr[2 * r + 1], dr[2 * r + 2]
        out = orc.inpaint_step(z, eps, sc, n_p, n_q, xh.to(dtype), masks[0], masks[1], masks[2])
        a, b, c, qa, qb = (orc._sc(sc, k, z) for k in ("a", "b", "c", "qa", "qb"))
        zn = (z / a - b * eps + c * n_p) * masks[2] + (qa * z + qb * (xh.to(dtype) * masks[1]) + c * n_q) * masks[1]
        pre = (4 * U * (z.abs() / a + (c * n_p).abs()) * masks[2]
               + 4 * U * ((qa * z).abs() + (qb * xh.to(dtype) * masks[1]).abs() + (c * n_q).abs()) * masks[1])
        rnd = pre.clone()
        rnd[..., :3] = (pre[..., :3] + projection_bound(zn, pre, masks[0], D) + U * out[..., :3].abs()) * masks[0]
        return out, zn, rnd

    def eps_pair(s, z64, z32):
        t = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)["t"] if s >= 0 else torch.zeros((B, 1))
        return (oracle_eps(sd, cfg, t, z64, kw, inpainting, torch.float64, d),
                oracle_eps(sd, cfg, t, z32, kw, inpainting, torch.float32, d).double())

    def eps_scale(s, eps64, mask):
        b = orc._sc(orc.step_scalars(gamma, s, T, B, gamma.numel() - 1), "b", eps64)
        return torch.where(live[..., None], (b * eps64 * mask).abs(), 0.0).amax(dim=(1, 2), keepdim=True)

    emask = nm if inpainting else lm
    for s in sorted({T - 1, T - 2, T // 2, 2, 1}, reverse=True):
        zt = z_at(s + 1)
        e64, e32 = eps_pair(s, zt, zt.float())
        ref64, _, rnd = step(s, zt, e64, torch.float64)
        ref32 = step(s, zt.float(), e32.float(), torch.float32)[0].double()
        rowwise(ck, f"step s={s}", z_at(s), ref64, ref32, rnd, eps_scale(s, e64, emask), live)
    # final composite: z_1 -> z_0 -> sample, both in fp64 and in fp32
    z1 = z_at(1)
    e64, e32 = eps_pair(0, z1, z1.float())
    z0_64, _, rnd0 = step(0, z1, e64, torch.float64)
    z0_32 = step(0, z1.float(), e32.float(), torch.float32)[0]
    scale0 = eps_scale(0, e64, emask)
    f64e, f32e = eps_pair(-1, z0_64, z0_32)
    fin = orc.step_scalars(gamma, -1, T, B, gamma.numel() - 1)
    inv_a0, sig0, snr0, qa0 = (orc._sc(fin, k, z0_64) for k in ("inv_alpha0", "sigma0", "snr0", "qa0"))
    if inpainting:
        l64, f64_ = orc.inpaint_final(z0_64, f64e, fin, draws64[2 * T + 1], draws64[2 * T + 2])
        l32, f32_ = (v.double() for v in orc.inpaint_final(z0_32, f32e.float(), fin, draws32[2 * T + 1], draws32[2 * T + 2]))
        out64, out32 = l64 * lm + f64_ * fm, l32 * lm + f32_ * fm
        n_round = ((snr0 * draws64[2 * T + 1]).abs() * lm + (qa0 * draws64[2 * T + 2]).abs() * fm)
    else:
        out64 = orc.linker_final(z0_64, f64e, fin, draws64[T + 1], fm, lm)
        out32 = orc.linker_final(z0_32, f32e.float(), fin, draws32[T + 1], fm.float(), lm.float()).double()
        n_round = (snr0 * draws64[T + 1] * lm).abs()
    scale = torch.maximum(inv_a0 * scale0, torch.where(live[..., None], (inv_a0 * sig0 * f64e * emask).abs(), 0.0)
                          .amax(dim=(1, 2), keepdim=True))
    rnd = inv_a0 * rnd0 + 4 * U * (inv_a0 * z0_64.abs() + n_round)
    if not inpainting:
        rnd = rnd * lm
    got = chain64[0]
    drift_x = (out32[..., :3] - out64[..., :3]).abs().amax(-1, keepdim=True)
    bound_x = torch.maximum(C_DRIFT * drift_x, TAU * scale) + rnd[..., :3]
    ck.close("final x", got[..., :3], out64[..., :3] * NORM[0], bound_x * NORM[0], live)
    drift_h = (out32[..., 3:] - out64[..., 3:]).abs().amax(-1, keepdim=True)
    bound_h = (torch.maximum(C_DRIFT * drift_h, TAU * scale) + rnd[..., 3:]).expand_as(out64[..., 3:])
    if inpainting:
        lk, fr = live & (lm[..., 0] != 0), live & (fm[..., 0] != 0)
        ck.types("final h (p variant)", got[..., 3:] * lm, l64[..., 3:], bound_h, lk, (nm * lm)[..., 0])
        ck.types("final h (q variant)", got[..., 3:] * fm, f64_[..., 3:], bound_h, fr, (nm * fm)[..., 0])
    else:
        ck.types("final h", got[..., 3:], out64[..., 3:], bound_h, live, nm[..., 0])
    ck.record()
