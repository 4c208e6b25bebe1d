"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the DiffLinker denoising hot path.

A functional (stateless) torch-CPU restatement of the reference's algorithm, in the reference's own
edge-list formulation (gather -> concat -> Linear -> scatter-add), so that it doubles as the "port"
CPU baseline of bench.py.  Every function cites the reference file:line it follows
(paths relative to the upstream repo igashov/DiffLinker @ fafbe47).

PINNING: oracle/make_golden.py checks every function here against the *live, unmodified*
reference code (imported from /root/reference in the build container) and writes the golden
vectors under tests/golden/; tests/test_oracle_golden.py re-checks the oracle against those vectors
wherever the test-suite runs.  The reference itself ships no tests / golden vectors (SURVEY.md section 4).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product (difflinker_b200/) never does.

Weights are passed as a flat dict with the reference's `Dynamics.state_dict()` key names
(`dynamics.embedding.weight`, `dynamics.e_block_0.gcl_0.edge_mlp.0.weight`, ...).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

Tensor = torch.Tensor


@dataclass
class OracleConfig:
    n_dims: int = 3
    in_node_nf: int = 8            # F: atom-type one-hot width (+charges)
    context_node_nf: int = 1       # C
    hidden_nf: int = 128           # H
    n_layers: int = 6              # L equivariant blocks
    inv_sublayers: int = 2         # S GCLs per block
    norm_constant: float = 1e-6
    normalization_factor: float = 100.0
    aggregation_method: str = "sum"
    condition_time: bool = True
    centering: bool = False
    graph_type: str = "FC"         # FC | 4A | FC-4A | FC-10A-4A

    @property
    def dyn_in_nf(self) -> int:    # egnn.py:339
        return self.in_node_nf + self.context_node_nf + int(self.condition_time)


# ------------------------------------------------------------------------------------------------
# graph + geometry
# ------------------------------------------------------------------------------------------------
def fc_edge_index(n_nodes: int, batch_size: int):
    """Fully-connected intra-molecule edge list incl. self loops, e = b*N*N + i*N + j
    (egnn.py:449-467; the python triple loop is vectorised, same ordering)."""
    i = torch.arange(n_nodes).repeat_interleave(n_nodes)
    j = torch.arange(n_nodes).repeat(n_nodes)
    off = (torch.arange(batch_size) * n_nodes).repeat_interleave(n_nodes * n_nodes)
    return i.repeat(batch_size) + off, j.repeat(batch_size) + off


def pair_geometry(x: Tensor, row: Tensor, col: Tensor, norm_constant: float = 1.0):
    """radial = |x_row - x_col|^2, and the normalised difference (egnn.py:295-301)."""
    delta = x.index_select(0, row) - x.index_select(0, col)
    radial = delta.pow(2).sum(dim=1, keepdim=True)
    return radial, delta / (torch.sqrt(radial + 1e-8) + norm_constant)


def segment_reduce(values: Tensor, seg: Tensor, n_seg: int, normalization_factor: float, method: str):
    """scatter-add of per-edge rows into their source node (egnn.py:304-320)."""
    out = values.new_zeros((n_seg, values.shape[1]))
    out.index_add_(0, seg, values)
    if method == "sum":
        out = out / normalization_factor
    elif method == "mean":
        cnt = values.new_zeros((n_seg, values.shape[1]))
        cnt.index_add_(0, seg, torch.ones_like(values))
        cnt[cnt == 0] = 1
        out = out / cnt
    return out


# ------------------------------------------------------------------------------------------------
# EGNN pieces
# ------------------------------------------------------------------------------------------------
def _lin(sd: Dict[str, Tensor], prefix: str, v: Tensor) -> Tensor:
    return F.linear(v, sd[prefix + ".weight"], sd.get(prefix + ".bias"))


def gcl_forward(sd, prefix, h, row, col, edge_attr, node_mask, edge_mask, cfg: OracleConfig):
    """One GCL: edge MLP on [h_row, h_col, edge_attr], masked, segment-summed by row, node MLP with
    residual (egnn.py:45-80; layer shapes egnn.py:19-30; attention is off in every config)."""
    e_in = torch.cat([h.index_select(0, row), h.index_select(0, col), edge_attr], dim=1)
    m = F.silu(_lin(sd, prefix + ".edge_mlp.0", e_in))
    m = F.silu(_lin(sd, prefix + ".edge_mlp.2", m))
    if edge_mask is not None:
        m = m * edge_mask
    agg = segment_reduce(m, row, h.shape[0], cfg.normalization_factor, cfg.aggregation_method)
    n_in = torch.cat([h, agg], dim=1)
    upd = _lin(sd, prefix + ".node_mlp.2", F.silu(_lin(sd, prefix + ".node_mlp.0", n_in)))
    h = h + upd
    if node_mask is not None:
        h = h * node_mask
    return h


def coord_update_forward(sd, prefix, h, x, row, col, unit_diff, edge_attr, linker_mask, node_mask, edge_mask,
                         cfg: OracleConfig):
    """Equivariant coordinate update (egnn.py:101-125; coord_mlp egnn.py:90-97; tanh branch unused)."""
    e_in = torch.cat([h.index_select(0, row), h.index_select(0, col), edge_attr], dim=1)
    phi = F.silu(_lin(sd, prefix + ".coord_mlp.0", e_in))
    phi = F.silu(_lin(sd, prefix + ".coord_mlp.2", phi))
    phi = F.linear(phi, sd[prefix + ".coord_mlp.4.weight"])
    trans = unit_diff * phi
    if edge_mask is not None:
        trans = trans * edge_mask
    agg = segment_reduce(trans, row, x.shape[0], cfg.normalization_factor, cfg.aggregation_method)
    if linker_mask is not None:
        agg = agg * linker_mask
    x = x + agg
    if node_mask is not None:
        x = x * node_mask
    return x


def egnn_forward(sd, h, x, row, col, node_mask, linker_mask, edge_mask, cfg: OracleConfig, prefix="dynamics"):
    """EGNN.forward (egnn.py:218-238) with EquivariantBlock.forward inlined (egnn.py:157-178)."""
    d0, _ = pair_geometry(x, row, col)                                    # egnn.py:220
    h = _lin(sd, prefix + ".embedding", h)                                # egnn.py:224
    for l in range(cfg.n_layers):
        blk = f"{prefix}.e_block_{l}"
        d_blk, unit = pair_geometry(x, row, col, cfg.norm_constant)       # egnn.py:159
        edge_attr = torch.cat([d_blk, d0], dim=1)                         # egnn.py:162
        for s in range(cfg.inv_sublayers):
            h = gcl_forward(sd, f"{blk}.gcl_{s}", h, row, col, edge_attr, node_mask, edge_mask, cfg)
        x = coord_update_forward(sd, f"{blk}.gcl_equiv", h, x, row, col, unit, edge_attr, linker_mask,
                                 node_mask, edge_mask, cfg)
        if node_mask is not None:
            h = h * node_mask                                             # egnn.py:176-177
    h = _lin(sd, prefix + ".embedding_out", h)                            # egnn.py:235
    if node_mask is not None:
        h = h * node_mask
    return h, x


class OracleNaN(Exception):
    """Stand-in for utils.FoundNaNException (utils.py:274-289): per-molecule index sets."""

    def __init__(self, vel: Tensor, h: Tensor):
        xs = {i for i in range(vel.shape[0]) if torch.isnan(vel[i]).any()}
        hs = {i for i in range(h.shape[0]) if torch.isnan(h[i]).any()}
        self.x_h_nan_idx = xs & hs
        self.only_x_nan_idx = xs - hs
        self.only_h_nan_idx = hs - xs
        super().__init__(f"NaN in dynamics output: x&h={self.x_h_nan_idx} x={self.only_x_nan_idx} h={self.only_h_nan_idx}")


def pocket_edge_index(x, node_mask, batch_ids, linker_mask, frag_only, pocket_only, graph_type: str):
    """Cut-off graphs of DynamicsWithPockets (egnn.py:554-596). x:(BN,3); masks:(BN,1) or (BN,)"""
    nm = node_mask.reshape(-1).bool()
    same_mol = batch_ids[:, None] == batch_ids[None, :]
    both_valid = nm[:, None] & nm[None, :]
    off_diag = ~torch.eye(x.shape[0], dtype=torch.bool)
    base = same_mol & both_valid & off_diag
    dist = torch.cdist(x, x)
    if graph_type == "4A":
        adj = base & (dist <= 4)                                          # egnn.py:555-563
    else:
        lk = linker_mask.reshape(-1).bool() & nm
        fr = frag_only.reshape(-1).bool() & nm
        pk = pocket_only.reshape(-1).bool() & nm
        lig = lk | fr
        cut = 4 if graph_type == "FC-4A" else 10                          # egnn.py:588
        lig_lig = lig[:, None] & lig[None, :]
        pk_pk = (pk[:, None] & pk[None, :]) & (dist <= 4)
        cross = ((lig[:, None] & pk[None, :]) | (pk[:, None] & lig[None, :])) & (dist <= cut)
        adj = (lig_lig | pk_pk | cross) & base
    r, c = torch.where(adj)
    return r, c


def dynamics_forward(sd, cfg: OracleConfig, t, xh, node_mask, linker_mask, edge_mask, context):
    """Dynamics.forward (egnn.py:374-447) and DynamicsWithPockets.forward (egnn.py:471-552).

    t:(B,1) or 1 element; xh:(B,N,3+F); node_mask:(B,N,1); linker_mask:(B,N,1)|None;
    edge_mask:(B*N*N,1) for FC graphs, or the (B*N,) batch-id vector for pocket graphs; context:(B,N,C).
    Returns (B,N,3+F)."""
    B, N = xh.shape[0], xh.shape[1]
    nm = node_mask.reshape(B * N, 1).to(xh.dtype)
    lm = None if linker_mask is None else linker_mask.reshape(B * N, 1)
    flat = xh.reshape(B * N, -1) * nm                                     # egnn.py:393
    x = flat[:, : cfg.n_dims].clone()
    h = flat[:, cfg.n_dims:].clone()
    if cfg.graph_type == "FC":
        row, col = fc_edge_index(N, B)
        em = edge_mask
    else:
        ctx = context.reshape(B * N, -1)
        row, col = pocket_edge_index(x, nm, edge_mask.reshape(-1), lm, ctx[:, -2], ctx[:, -1], cfg.graph_type)
        em = None                                                         # egnn.py:523
    if cfg.condition_time:
        if t.numel() == 1:
            tcol = torch.full_like(h[:, 0:1], float(t.reshape(-1)[0]))    # egnn.py:397-399
        else:
            tcol = t.reshape(B, 1).repeat(1, N).reshape(B * N, 1)         # egnn.py:402-403
        h = torch.cat([h, tcol], dim=1)
    if context is not None:
        h = torch.cat([h, context.reshape(B * N, cfg.context_node_nf)], dim=1)
    h_out, x_out = egnn_forward(sd, h, x, row, col, nm, lm, em, cfg)
    vel = (x_out - x) * nm                                                # egnn.py:420
    if context is not None:
        h_out = h_out[:, : -cfg.context_node_nf]
    if cfg.condition_time:
        h_out = h_out[:, :-1]
    vel = vel.reshape(B, N, -1)
    h_out = h_out.reshape(B, N, -1)
    if torch.isnan(vel).any() or torch.isnan(h_out).any():                # egnn.py:441-442
        raise OracleNaN(vel, h_out)
    if cfg.centering:                                                     # egnn.py:444-445, utils.py:56-63
        nmb = nm.reshape(B, N, 1)
        vel = vel - (vel.sum(dim=1, keepdim=True) / nmb.sum(1, keepdim=True)) * nmb
    return torch.cat([vel, h_out], dim=2)


# ------------------------------------------------------------------------------------------------
# noise schedule (noise.py)
# ------------------------------------------------------------------------------------------------
def gamma_table(noise_schedule: str, timesteps: int, precision: float) -> Tensor:
    """PredefinedNoiseSchedule.__init__ (noise.py:92-124) -> fp32 table of length timesteps+1."""
    if noise_schedule == "cosine":                                        # noise.py:39-56
        steps = timesteps + 2
        u = np.linspace(0, steps, steps)
        ac = np.cos(((u / steps) + 0.008) / 1.008 * np.pi * 0.5) ** 2
        ac = ac / ac[0]
        betas = np.clip(1 - ac[1:] / ac[:-1], a_min=0, a_max=0.999)
        alphas2 = np.cumprod(1.0 - betas, axis=0)
    elif "polynomial" in noise_schedule:                                  # noise.py:22-36
        power = float(noise_schedule.split("_")[1])
        steps = timesteps + 1
        u = np.linspace(0, steps, steps)
        alphas2 = (1 - np.power(u / steps, power)) ** 2
        ext = np.concatenate([np.ones(1), alphas2], axis=0)               # noise.py:7-19
        alphas2 = np.cumprod(np.clip(ext[1:] / ext[:-1], a_min=0.001, a_max=1.0), axis=0)
        alphas2 = (1 - 2 * precision) * alphas2 + precision
    else:
        raise ValueError(noise_schedule)
    g = -(np.log(alphas2) - np.log(1 - alphas2))
    return torch.from_numpy(g).float()


def gamma_lookup(table: Tensor, t: Tensor, timesteps: int) -> Tensor:
    """PredefinedNoiseSchedule.forward (noise.py:126-128). `timesteps` is the table's own length-1."""
    return table[torch.round(t * timesteps).long()]


# ------------------------------------------------------------------------------------------------
# EDM sampler (edm.py)
# ------------------------------------------------------------------------------------------------
def _sigma(g):  # edm.py:369-371
    return torch.sqrt(torch.sigmoid(g))


def _alpha(g):  # edm.py:373-375
    return torch.sqrt(torch.sigmoid(-g))


def _sigma_alpha_t_given_s(g_t, g_s):
    """edm.py:381-403."""
    sigma2 = -torch.expm1(F.softplus(g_s) - F.softplus(g_t))
    alpha = torch.exp(0.5 * (F.logsigmoid(-g_t) - F.logsigmoid(-g_s)))
    return sigma2, torch.sqrt(sigma2), alpha


def _bcast(v: Tensor) -> Tensor:  # edm.py:410-416 for a (B,N,D) target
    return v.reshape(v.shape[0], 1, 1)


NoiseFn = Callable[[tuple], Tensor]


def masked_noise(noise_fn: NoiseFn, B: int, N: int, n_dims: int, F_: int, mask: Tensor) -> Tensor:
    """edm.py:328-340 + utils.py:189-192: randn(B,N,3)*mask then randn(B,N,F)*mask, concatenated."""
    zx = noise_fn((B, N, n_dims)) * mask
    zh = noise_fn((B, N, F_)) * mask
    return torch.cat([zx, zh], dim=2)


def step_scalars(gamma: Tensor, s: int, T: int, B: int, table_timesteps: int) -> Dict[str, Tensor]:
    """The fp32 (B,1) scalars of reverse step s (edm.py:146-150, 196-205, 655-668), evaluated by the reference's ops in the
    reference's order on (B,1) tensors: t, a = alpha_t|s, b = sigma2_t|s / alpha_t|s / sigma_t, c = sigma_t|s * sigma_s /
    sigma_t and the q(z_s|z_t,x) pair qa = alpha_t|s sigma_s^2 / sigma_t^2, qb = alpha_s sigma2_t|s / sigma_t^2.
    s = -1 is the final p(x,h|z_0) step (edm.py:210-242, 700-716): inv_alpha0 = 1/alpha_0, sigma0, snr0 = SNR(-0.5 g_0) and
    qa0 = sigma_0 / alpha_0.  These are the rows of EDM.step_coefficients: row r is step s = T-1-r."""
    if s < 0:
        g0 = gamma_lookup(gamma, torch.zeros((B, 1)), table_timesteps)
        return dict(inv_alpha0=1.0 / _alpha(g0), sigma0=_sigma(g0), snr0=torch.exp(-(-0.5 * g0)),   # edm.py:216,377-379
                    qa0=_sigma(g0) / _alpha(g0))
    s_arr = torch.full((B, 1), fill_value=s)
    t_arr = (s_arr + 1) / T
    s_arr = s_arr / T
    g_s = gamma_lookup(gamma, s_arr, table_timesteps)
    g_t = gamma_lookup(gamma, t_arr, table_timesteps)
    sig2_ts, sig_ts, a_ts = _sigma_alpha_t_given_s(g_t, g_s)
    sig_s, sig_t, al_s = _sigma(g_s), _sigma(g_t), _alpha(g_s)
    return dict(t=t_arr, a=a_ts, b=sig2_ts / a_ts / sig_t, c=sig_ts * sig_s / sig_t,
                qa=a_ts * (sig_s ** 2) / (sig_t ** 2), qb=al_s * sig2_ts / (sig_t ** 2))


def _sc(scalars: Dict[str, Tensor], key: str, like: Tensor) -> Tensor:
    """A (B,1) step scalar as a (B,1,1) tensor of `like`'s dtype and device (fp32 scalars promoted exactly)."""
    return _bcast(scalars[key]).to(dtype=like.dtype, device=like.device)


def linker_step(z, eps, scalars, draw, fm, lm):
    """One reverse step of the linker sampler, sample_p_zs_given_zt_only_linker (edm.py:178-208), in z's dtype: `eps` is
    the raw dynamics output and `draw` the step's standard-normal draw, both masked here by the linker mask."""
    a, b, c = (_sc(scalars, k, z) for k in ("a", "b", "c"))
    eps = eps * lm                                                        # edm.py:196
    mu = z / a - b * eps                                                  # edm.py:199
    z_s = mu + c * (draw * lm)                                            # edm.py:202-205, utils.py:189-192
    return z * fm + z_s * lm                                              # edm.py:206


def linker_final(z, eps, scalars, draw, fm, lm):
    """sample_p_xh_given_z0_only_linker (edm.py:210-235) up to the unnormalisation: the final normalised (x,h)."""
    inv_a0, sig0, snr0 = (_sc(scalars, k, z) for k in ("inv_alpha0", "sigma0", "snr0"))
    eps = eps * lm
    mu_x = inv_a0 * (z - sig0 * eps)                                      # edm.py:237-242
    out = mu_x + snr0 * (draw * lm)                                       # edm.py:228
    return z * fm + out * lm                                              # edm.py:229


def inpaint_step(z, eps, scalars, draw_p, draw_q, xh, nm, fm, lm, n_dims=3):
    """One reverse step of InpaintingEDM.sample_chain (edm.py:575-594) in z's dtype: p(z_s|z_t) on every atom from the
    (centred) dynamics output `eps` and the prepared draw `draw_p`, q(z_s|z_t,x) on the fragment atoms from the normalised
    data `xh` and `draw_q`, recombination and the centre-of-mass projection over the node mask. The draws are masked and
    centre-of-mass free as com_free_noise makes them."""
    a, b, c, qa, qb = (_sc(scalars, k, z) for k in ("a", "b", "c", "qa", "qb"))
    mu = z / a - b * eps                                                  # edm.py:634-642
    z_lin = mu + c * draw_p                                               # edm.py:645
    mu_q = qa * z + qb * (xh * fm)                                        # edm.py:655-664
    z_frag = mu_q + c * draw_q                                            # edm.py:669
    z = z_lin * lm + z_frag * fm                                          # edm.py:589
    return torch.cat([remove_mean(z[:, :, :n_dims], nm), z[:, :, n_dims:]], dim=2)   # edm.py:592-594


def inpaint_final(z, eps, scalars, draw_p, draw_q):
    """The two final variants of InpaintingEDM (edm.py:689-716) up to the unnormalisation: sample_p_xh_given_z0 with
    `draw_p` and sample_q_xh_given_z0_and_x with `draw_q`, both normalised (x,h) on every atom."""
    inv_a0, sig0, snr0, qa0 = (_sc(scalars, k, z) for k in ("inv_alpha0", "sigma0", "snr0", "qa0"))
    out_l = inv_a0 * (z - sig0 * eps) + snr0 * draw_p                     # edm.py:689-690, 237-242
    out_f = inv_a0 * z - qa0 * draw_q                                     # edm.py:706-716
    return out_l, out_f


def final_frame(out, node_mask, n_dims=3, norm_values=(1.0, 4.0, 10.0), norm_biases=(None, 0.0, 0.0)):
    """chain[0] of a final (x,h): unnormalised coordinates and one_hot(argmax(h)) * node_mask (edm.py:231-233)."""
    xo = out[:, :, :n_dims] * norm_values[0]
    ho = out[:, :, n_dims:] * norm_values[1] + norm_biases[1]
    ho = F.one_hot(torch.argmax(ho, dim=2), ho.shape[2]) * node_mask
    return torch.cat([xo, ho], dim=2)


def edm_sample_chain(sd, cfg: OracleConfig, gamma: Tensor, T: int, x, h, node_mask, fragment_mask, linker_mask,
                     edge_mask, context, keep_frames=None, norm_values=(1.0, 4.0, 10.0),
                     norm_biases=(None, 0.0, 0.0), noise_fn: Optional[NoiseFn] = None,
                     table_timesteps: Optional[int] = None):
    """EDM.sample_chain (edm.py:126-176) with sample_p_zs_given_zt_only_linker (178-208) and
    sample_p_xh_given_z0_only_linker (210-235) as linker_step / linker_final.  `gamma` is the fp32 table; `T` is edm.T
    (may have been overridden by --n_steps, generate.py:103-104) while `table_timesteps` is the table's own length-1."""
    if noise_fn is None:
        noise_fn = lambda shape: torch.randn(shape)
    if table_timesteps is None:
        table_timesteps = gamma.numel() - 1
    B, N = x.shape[0], x.shape[1]
    nd, F_ = cfg.n_dims, cfg.in_node_nf
    x = x / norm_values[0]                                                # edm.py:347-350
    h = (h.float() - norm_biases[1]) / norm_values[1]
    xh = torch.cat([x, h], dim=2)
    z = masked_noise(noise_fn, B, N, nd, F_, linker_mask)                 # edm.py:136
    z = xh * fragment_mask + z * linker_mask
    if keep_frames is None:
        keep_frames = T
    assert keep_frames <= T
    chain = torch.zeros((keep_frames,) + z.shape)

    def unnorm(zz):                                                       # edm.py:352-361
        return torch.cat([zz[:, :, :nd] * norm_values[0], zz[:, :, nd:] * norm_values[1] + norm_biases[1]], dim=2)

    for s in reversed(range(T)):
        sc = step_scalars(gamma, s, T, B, table_timesteps)
        eps = dynamics_forward(sd, cfg, sc["t"], z, node_mask, linker_mask, edge_mask, context)
        z = linker_step(z, eps, sc, masked_noise(noise_fn, B, N, nd, F_, linker_mask), fragment_mask, linker_mask)
        chain[(s * keep_frames) // T] = unnorm(z)

    zeros = torch.zeros((B, 1))
    eps = dynamics_forward(sd, cfg, zeros, z, node_mask, linker_mask, edge_mask, context)
    out = linker_final(z, eps, step_scalars(gamma, -1, T, B, table_timesteps),
                       masked_noise(noise_fn, B, N, nd, F_, linker_mask), fragment_mask, linker_mask)
    chain[0] = final_frame(out, node_mask, nd, norm_values, norm_biases)
    return chain


def remove_mean(x, node_mask):
    """utils.remove_mean_with_mask (utils.py:56-63)."""
    return x - (x.sum(dim=1, keepdim=True) / node_mask.sum(1, keepdim=True)) * node_mask


def com_free_noise(noise_fn: NoiseFn, B: int, N: int, n_dims: int, F_: int, mask: Tensor) -> Tensor:
    """InpaintingEDM.sample_combined_position_feature_noise (edm.py:715-727): the coordinate part is masked and
    projected to zero centre of mass (utils.py:158-168), the feature part only masked."""
    zx = remove_mean(noise_fn((B, N, n_dims)) * mask, mask)
    zh = noise_fn((B, N, F_)) * mask
    return torch.cat([zx, zh], dim=2)


def inpainting_sample_chain(sd, cfg: OracleConfig, gamma: Tensor, T: int, x, h, node_mask, fragment_mask, linker_mask,
                            edge_mask, context, keep_frames=None, norm_values=(1.0, 4.0, 10.0),
                            norm_biases=(None, 0.0, 0.0), noise_fn: Optional[NoiseFn] = None,
                            table_timesteps: Optional[int] = None):
    """InpaintingEDM.sample_chain (edm.py:549-612) with sample_p_zs_given_zt (614-646), sample_q_zs_given_zt_and_x
    (648-670), sample_p_xh_given_z0 (672-698) and sample_q_xh_given_z0_and_x (700-713) inlined.
    `cfg.centering` must be True (lightning.py:99) and the dynamics are called with linker_mask=None."""
    assert cfg.centering
    if noise_fn is None:
        noise_fn = lambda shape: torch.randn(shape)
    if table_timesteps is None:
        table_timesteps = gamma.numel() - 1
    B, N = x.shape[0], x.shape[1]
    nd, F_ = cfg.n_dims, cfg.in_node_nf
    nmf = node_mask.to(x.dtype)
    x = x / norm_values[0]
    h = (h.float() - norm_biases[1]) / norm_values[1]
    xh = torch.cat([x, h], dim=2)
    z = com_free_noise(noise_fn, B, N, nd, F_, nmf)                        # edm.py:565
    if keep_frames is None:
        keep_frames = T
    chain = torch.zeros((keep_frames,) + z.shape)

    def unnorm(zz):
        return torch.cat([zz[:, :, :nd] * norm_values[0], zz[:, :, nd:] * norm_values[1] + norm_biases[1]], dim=2)

    for s in reversed(range(T)):
        sc = step_scalars(gamma, s, T, B, table_timesteps)
        eps = dynamics_forward(sd, cfg, sc["t"], z, node_mask, None, edge_mask, context)             # edm.py:626-633
        draw_p = com_free_noise(noise_fn, B, N, nd, F_, nmf)                                          # edm.py:645
        draw_q = com_free_noise(noise_fn, B, N, nd, F_, fragment_mask)                                # edm.py:669
        z = inpaint_step(z, eps, sc, draw_p, draw_q, xh, nmf, fragment_mask, linker_mask, nd)
        chain[(s * keep_frames) // T] = unnorm(z)

    zeros = torch.zeros((B, 1))
    eps = dynamics_forward(sd, cfg, zeros, z, node_mask, None, edge_mask, context)
    draw_p = com_free_noise(noise_fn, B, N, nd, F_, nmf)                                              # edm.py:689-690
    draw_q = com_free_noise(noise_fn, B, N, nd, F_, nmf)                                              # edm.py:706
    out_l, out_f = inpaint_final(z, eps, step_scalars(gamma, -1, T, B, table_timesteps), draw_p, draw_q)
    chain[0] = (final_frame(out_l, node_mask, nd, norm_values, norm_biases) * linker_mask
                + final_frame(out_f, node_mask, nd, norm_values, norm_biases) * fragment_mask)        # edm.py:603-608
    return chain


# ------------------------------------------------------------------------------------------------
# linker-size classifier (linker_size.py:45-91, linker_size_lightning.py:83-110)
# ------------------------------------------------------------------------------------------------
def _bn_eval(sd, prefix, v, eps=1e-5):
    """nn.BatchNorm1d in eval mode (running statistics)."""
    return (v - sd[prefix + ".running_mean"]) / torch.sqrt(sd[prefix + ".running_var"] + eps) * sd[prefix + ".weight"] \
        + sd[prefix + ".bias"]


def size_gcl_forward(sd, prefix, h, edge_blocks, node_mask, normalization):
    """egnn.GCL with activation=ReLU, edges_in_d=1, normalization_factor=1, 'sum' (egnn.py:10-80 as built by
    linker_size.py:53-83), over the live edges only: a masked edge contributes m * 0 = 0 to the sum exactly, so leaving it
    out changes nothing. `edge_blocks` holds (row, col, radial) blocks of live edges in the reference's edge order."""
    agg = h.new_zeros(h.shape)
    for row, col, radial in edge_blocks:
        e_in = torch.cat([h.index_select(0, row), h.index_select(0, col), radial], dim=1)
        m = F.relu(_lin(sd, prefix + ".edge_mlp.0", e_in))
        m = F.relu(_lin(sd, prefix + ".edge_mlp.2", m))
        agg.index_add_(0, row, m)
    n_in = torch.cat([h, agg], dim=1)
    if normalization is None:
        upd = _lin(sd, prefix + ".node_mlp.2", F.relu(_lin(sd, prefix + ".node_mlp.0", n_in)))
    else:
        upd = _bn_eval(sd, prefix + ".node_mlp.1", _lin(sd, prefix + ".node_mlp.0", n_in))
        upd = _bn_eval(sd, prefix + ".node_mlp.4", _lin(sd, prefix + ".node_mlp.3", F.relu(upd)))
    return (h + upd) * node_mask


def size_live_edges(x32, edge_mask, B, N, max_pairs=1 << 20):
    """The size classifier's edges (linker_size_lightning.py:107-108): e = b*N*N + i*N + j is one when edge_mask[e] != 0
    and the fp32 squared distance is < 6, with the squared distance in torch's rounding order, (dx^2 + dy^2) + dz^2 with
    every term rounded. Returns (row, col) int64 blocks of global node indices, in edge order, each block from at most
    `max_pairs` candidate pairs, so that the whole (B*N*N) edge list never exists at once."""
    em = edge_mask.reshape(B, N, N)
    xb = x32.reshape(B, N, 3)
    rows = max(1, max_pairs // N)
    out = []
    for b in range(B):
        for i0 in range(0, N, rows):
            i1 = min(N, i0 + rows)
            d = xb[b, i0:i1, None, :] - xb[b, None, :, :]                # (rows, N, 3) fp32
            sq = d * d
            radial = (sq[..., 0] + sq[..., 1]) + sq[..., 2]
            ii, jj = torch.nonzero((em[b, i0:i1] != 0) & (radial < 6), as_tuple=True)
            if ii.numel():
                out.append((ii + (b * N + i0), jj + b * N))
    return out


def size_classifier_forward(sd, data, in_node_nf, n_layers, normalization=None, with_pocket=False, adjust_shape=False,
                            prefix="gnn", dtype=torch.float32):
    """SizeClassifier.forward(return_loss=False) (linker_size_lightning.py:83-110) with SizeGNN.forward inlined
    (linker_size.py:85-91). `data` as produced by collate_with_fragment_edges (its `edges` list is not read). Returns the
    (B, classes) logits in `dtype`, computed on the device of data['positions'].

    The edge set is the reference's in any dtype: radial < 6 is evaluated on the fp32 radial in torch's rounding order.
    The state dict, positions and one-hot are then cast to `dtype` before any arithmetic, and the edge MLP runs over the
    live edges in blocks, so the peak memory stays a few GB up to N = 6144 in float64."""
    dev = data['positions'].device
    fragment_mask = (data['fragment_only_mask'] if with_pocket else data['fragment_mask']).float()
    x32 = data['positions'].float() * fragment_mask
    B, N = x32.shape[0], x32.shape[1]
    blocks = size_live_edges(x32.reshape(B * N, 3), data['edge_mask'].reshape(-1).to(dev), B, N)
    sd = {k: v.to(device=dev, dtype=dtype) if v.is_floating_point() else v.to(dev) for k, v in sd.items()}
    fragment_mask = fragment_mask.to(dtype)
    x = (data['positions'].to(dtype) * fragment_mask).reshape(B * N, 3)
    h = data['one_hot'].to(dtype) * fragment_mask
    if h.shape[-1] != in_node_nf and adjust_shape:
        h = h[..., :-1]
    fm = fragment_mask.reshape(B * N, 1)
    h = h.reshape(B * N, -1)
    edge_blocks = []
    for row, col in blocks:                                               # coord2diff: SQUARED distance, in `dtype`
        edge_blocks.append((row, col, (x.index_select(0, row) - x.index_select(0, col)).pow(2).sum(1, keepdim=True)))
    h = _lin(sd, prefix + ".embedding_in", h)
    h = size_gcl_forward(sd, prefix + ".gcl1", h, edge_blocks, fm, normalization)
    for l in range(n_layers - 1):
        h = size_gcl_forward(sd, f"{prefix}.gcl_layers.{l}", h, edge_blocks, fm, normalization)
    out = _lin(sd, prefix + ".embedding_out", h)
    return out.view(B, N, -1).mean(1)


# ------------------------------------------------------------------------------------------------
# output stage (generate.py:163-171, visualizer.py:14-31)
# ------------------------------------------------------------------------------------------------
def restore_frame(x, positions, com_mask, node_mask):
    """generate.py:165-171."""
    pos_masked = positions * com_mask
    n = com_mask.sum(1, keepdims=True)
    mean = torch.sum(pos_masked, dim=1, keepdim=True) / n
    return x + mean * node_mask


def xyz_text(one_hot, positions, node_mask, idx2atom):
    """visualizer.save_xyz_file (visualizer.py:14-31) returning the file contents instead of writing them."""
    out = []
    for b in range(one_hot.size(0)):
        mask = node_mask[b].squeeze()
        lines = ["%d\n\n" % mask.sum()]
        atoms = torch.argmax(one_hot[b], dim=1)
        for i in torch.where(mask)[0]:
            lines.append("%s %.9f %.9f %.9f\n" % (idx2atom[atoms[i].item()], positions[b, i, 0], positions[b, i, 1],
                                                positions[b, i, 2]))
        out.append("".join(lines))
    return out


# ------------------------------------------------------------------------------------------------
# bond inference (molecule_builder.py:44-102)
# ------------------------------------------------------------------------------------------------
def bond_order(sym1, sym2, distance, single, double, triple, margins):
    """get_bond_order (molecule_builder.py:77-102); tables keyed by the (sym1, sym2) pair in type-index order."""
    distance = 100 * distance
    if (sym1, sym2) not in single:
        return 0
    if distance < single[(sym1, sym2)] + margins[0]:
        if (sym1, sym2) in double and distance < double[(sym1, sym2)] + margins[1]:
            if (sym1, sym2) in triple and distance < triple[(sym1, sym2)] + margins[2]:
                return 3
            return 2
        return 1
    return 0


def xae_molecule(positions, atom_types, idx2atom, single, double, triple, margins=(10, 5, 2)):
    """build_xae_molecule (molecule_builder.py:44-74): python pair loop over the lower triangle."""
    n = positions.shape[0]
    E = torch.zeros((n, n), dtype=torch.int)
    dists = torch.cdist(positions.unsqueeze(0), positions.unsqueeze(0), p=2).squeeze(0)
    for i in range(n):
        for j in range(i):
            a, c = sorted([int(atom_types[i]), int(atom_types[j])])
            E[i, j] = bond_order(idx2atom[a], idx2atom[c], dists[i, j], single, double, triple, margins)
    return atom_types, E.bool(), E


# ------------------------------------------------------------------------------------------------
# batching contract (datasets.py) -- restated for fixtures; int8 masks incl. the -1/-2 edge mask
# ------------------------------------------------------------------------------------------------
PAD_KEYS = ("positions", "one_hot", "charges", "anchors", "fragment_mask", "linker_mask", "pocket_mask",
            "fragment_only_mask")                                         # const.py:42-44
LAST_DIM_KEYS = ("charges", "anchors", "fragment_mask", "linker_mask", "pocket_mask", "fragment_only_mask")
LIST_KEYS = ("uuid", "name", "fragments_smi", "linker_smi", "num_atoms")  # const.py:39-41


def collate_molecules(items: List[dict]) -> dict:
    """datasets.collate (datasets.py:332-375)."""
    out: Dict[str, list] = {}
    for it in items:
        for k, v in it.items():
            out.setdefault(k, []).append(v)
    for k in list(out.keys()):
        if k in LIST_KEYS:
            continue
        if k not in PAD_KEYS:
            raise KeyError(k)
        out[k] = torch.nn.utils.rnn.pad_sequence(out[k], batch_first=True, padding_value=0)
    atom = (out["fragment_mask"].bool() | out["linker_mask"].bool()).to(torch.int8)
    out["atom_mask"] = atom[:, :, None]
    B, N = atom.shape
    if "pocket_mask" in items[0]:
        out["edge_mask"] = torch.cat([torch.ones(N, dtype=torch.int8) * i for i in range(B)])
    else:
        em = atom[:, None, :] * atom[:, :, None]
        em = em * (~torch.eye(N, dtype=torch.int8)).unsqueeze(0)          # bitwise NOT: 0 -> -1, 1 -> -2
        out["edge_mask"] = em.view(B * N * N, 1)
    for k in LAST_DIM_KEYS:
        if k in out:
            out[k] = out[k][:, :, None]
    return out


def linker_templates(data: dict, linker_sizes) -> dict:
    """datasets.create_templates_for_linker_generation (datasets.py:476-512)."""
    per_mol = []
    for i, ls in enumerate(linker_sizes):
        ls = int(ls)
        nfrag = int(data["fragment_mask"][i].squeeze().sum())
        d = {}
        for k, v in data.items():
            if k == "num_atoms":
                d[k] = nfrag + ls
            elif k in LIST_KEYS:
                d[k] = v[i]
            elif k in PAD_KEYS:
                keep = v[i][:nfrag]
                fill = 1 if k == "linker_mask" else 0
                add = torch.ones(ls, keep.shape[1], dtype=keep.dtype) * fill
                tpl = torch.cat([keep, add], dim=0)
                d[k] = tpl.squeeze(-1) if k in LAST_DIM_KEYS else tpl
        per_mol.append(d)
    return collate_molecules(per_mol)


def remove_partial_mean(x, node_mask, com_mask):
    """utils.remove_partial_mean_with_mask (utils.py:66-74)."""
    mean = (x * com_mask).sum(dim=1, keepdim=True) / com_mask.sum(1, keepdim=True)
    return x - mean * node_mask
