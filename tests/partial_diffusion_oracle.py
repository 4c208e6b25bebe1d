"""Oracle of partial diffusion: EDM.sample_chain started at step t0 from q(z_t0 | x) instead of from noise at T.

Composed of the reference's own arithmetic, restated by oracle/difflinker_oracle.py: the forward noising of EDM.forward
(edm.py:50-74) and the reverse steps of the linker sampler (orc.step_scalars, linker_step, linker_final; edm.py:146-235).
It lives here rather than in oracle/, whose files pin the existing fixtures and stay as they are.
"""
from typing import Optional

import torch

from oracle import difflinker_oracle as orc


def start_scalars(gamma, t0: int, T: int, B: int, table_timesteps: int):
    """(alpha_t0, sigma_t0) as (B,1) fp32 tensors, evaluated as EDM.forward evaluates them (edm.py:50-65): t = t0 / T on a
    (B,1) fp32 tensor (t_int is a float tensor there), gamma(t), sqrt(sigmoid(-gamma)), sqrt(sigmoid(gamma))."""
    t = torch.full((B, 1), fill_value=float(t0)) / T
    g = orc.gamma_lookup(gamma, t, table_timesteps)
    return orc._alpha(g), orc._sigma(g)


def partial_start(xh, eps, alpha, sigma, fragment_mask, linker_mask):
    """q(z_t0 | x) on the linker, the data on the fragments (edm.py:73-74), in xh's dtype. `eps` is the masked draw."""
    a, s = orc._bcast(alpha).to(xh.dtype), orc._bcast(sigma).to(xh.dtype)
    z = a * xh + s * eps
    return xh * fragment_mask + z * linker_mask


def linker_partial_chain(sd, cfg: orc.OracleConfig, gamma, T: int, t0: int, x, h, node_mask, fragment_mask, linker_mask,
                         edge_mask, context, keep_frames=None, norm_values=(1.0, 4.0, 10.0), norm_biases=(None, 0.0, 0.0),
                         noise_fn: Optional[orc.NoiseFn] = None, table_timesteps: Optional[int] = None,
                         dynamics_forward=orc.dynamics_forward):
    """EDM.sample_chain from step t0: x, h hold the linker to vary on its linker_mask rows. Draws in the reference's call
    order: eps (sample_combined_position_feature_noise, as z_T is drawn), one per step s = t0-1 .. 0, the final draw.
    Returns the (keep_frames, B, N, 3+F) chain; frames no step below t0 writes stay zero."""
    if noise_fn is None:
        noise_fn = lambda shape: torch.randn(shape)
    if table_timesteps is None:
        table_timesteps = gamma.numel() - 1
    assert 0 <= t0 <= T
    B, N = x.shape[0], x.shape[1]
    nd, F_ = cfg.n_dims, cfg.in_node_nf
    x = x / norm_values[0]                                                # edm.py:347-350
    h = (h.float() - norm_biases[1]) / norm_values[1]
    xh = torch.cat([x, h], dim=2)
    eps = orc.masked_noise(noise_fn, B, N, nd, F_, linker_mask)           # edm.py:69
    alpha, sigma = start_scalars(gamma, t0, T, B, table_timesteps)        # edm.py:50-65
    z = partial_start(xh, eps, alpha, sigma, fragment_mask, linker_mask)  # edm.py:73-74
    if keep_frames is None:
        keep_frames = T
    assert keep_frames <= T
    chain = torch.zeros((keep_frames,) + z.shape)

    def unnorm(zz):                                                       # edm.py:352-361
        return torch.cat([zz[:, :, :nd] * norm_values[0], zz[:, :, nd:] * norm_values[1] + norm_biases[1]], dim=2)

    for s in reversed(range(t0)):
        sc = orc.step_scalars(gamma, s, T, B, table_timesteps)
        eps_hat = dynamics_forward(sd, cfg, sc["t"], z, node_mask, linker_mask, edge_mask, context)
        z = orc.linker_step(z, eps_hat, sc, orc.masked_noise(noise_fn, B, N, nd, F_, linker_mask), fragment_mask,
                            linker_mask)
        chain[(s * keep_frames) // T] = unnorm(z)

    zeros = torch.zeros((B, 1))
    eps_hat = dynamics_forward(sd, cfg, zeros, z, node_mask, linker_mask, edge_mask, context)
    out = orc.linker_final(z, eps_hat, orc.step_scalars(gamma, -1, T, B, table_timesteps),
                           orc.masked_noise(noise_fn, B, N, nd, F_, linker_mask), fragment_mask, linker_mask)
    chain[0] = orc.final_frame(out, node_mask, nd, norm_values, norm_biases)
    return chain


def written_frames(t0: int, T: int, keep_frames: int):
    """The frames some step s < t0 writes (frame 0 always: the final sample)."""
    return sorted({0} | {(s * keep_frames) // T for s in range(t0)})
