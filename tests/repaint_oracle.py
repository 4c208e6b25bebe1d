"""Oracle of RePaint resampling for InpaintingEDM: every reverse step of the inpainting sampler run as r passes, each pass
but the last followed by a re-noise z <- alpha_t|s z + sigma_t|s eps back to step t.

Composed of the reference's own arithmetic, restated by oracle/difflinker_oracle.py: the inpainting step and final step
(orc.step_scalars, inpaint_step, inpaint_final; edm.py:549-713) and sigma_and_alpha_t_given_s (edm.py:273-285). Only the
re-noise line is new. It lives here rather than in oracle/, whose files pin the existing fixtures and stay as they are.
"""
from typing import Optional

import torch

from oracle import difflinker_oracle as orc


def jump_scalars(gamma, s: int, T: int, B: int, table_timesteps: int):
    """(alpha_t|s, sigma_t|s) of reverse step s as (B,1) fp32 tensors: sigma_and_alpha_t_given_s(gamma(t), gamma(s)) with
    s / T and t = (s+1) / T on (B,1) tensors, as the step's other scalars are evaluated."""
    s_arr = torch.full((B, 1), fill_value=s)
    t_arr = (s_arr + 1) / T
    s_arr = s_arr / T
    _, sigma_ts, alpha_ts = orc._sigma_alpha_t_given_s(orc.gamma_lookup(gamma, t_arr, table_timesteps),
                                                       orc.gamma_lookup(gamma, s_arr, table_timesteps))
    return alpha_ts, sigma_ts


def renoise(z, eps, alpha, sigma):
    """z <- alpha_t|s * z + sigma_t|s * eps in z's dtype; `eps` is the COM-free, masked draw."""
    return orc._bcast(alpha).to(z.dtype) * z + orc._bcast(sigma).to(z.dtype) * eps


def repaint_chain(sd, cfg: orc.OracleConfig, gamma, T: int, r: int, x, h, node_mask, fragment_mask, linker_mask,
                  edge_mask, context, keep_frames=None, norm_values=(1.0, 4.0, 10.0), norm_biases=(None, 0.0, 0.0),
                  noise_fn: Optional[orc.NoiseFn] = None, table_timesteps: Optional[int] = None,
                  dynamics_forward=orc.dynamics_forward):
    """orc.inpainting_sample_chain with r passes per reverse step. Draws in call order: z_T; per step and pass u the p draw
    (node mask), the q draw (fragment mask) and, for u < r-1, the re-noise draw (node mask); the two final draws. The
    frame of step s is written after its last pass. r = 1 is orc.inpainting_sample_chain."""
    assert cfg.centering and r >= 1
    if noise_fn is None:
        noise_fn = lambda shape: torch.randn(shape)
    if table_timesteps is None:
        table_timesteps = gamma.numel() - 1
    B, N = x.shape[0], x.shape[1]
    nd, F_ = cfg.n_dims, cfg.in_node_nf
    nmf = node_mask.to(x.dtype)
    x = x / norm_values[0]
    h = (h.to(x.dtype) - norm_biases[1]) / norm_values[1]
    xh = torch.cat([x, h], dim=2)
    z = orc.com_free_noise(noise_fn, B, N, nd, F_, nmf)                                  # edm.py:565
    if keep_frames is None:
        keep_frames = T
    chain = torch.zeros((keep_frames,) + z.shape, dtype=z.dtype)

    def unnorm(zz):
        return torch.cat([zz[:, :, :nd] * norm_values[0], zz[:, :, nd:] * norm_values[1] + norm_biases[1]], dim=2)

    for s in reversed(range(T)):
        sc = orc.step_scalars(gamma, s, T, B, table_timesteps)
        for u in range(r):
            eps = dynamics_forward(sd, cfg, sc["t"], z, node_mask, None, edge_mask, context)   # edm.py:626-633
            draw_p = orc.com_free_noise(noise_fn, B, N, nd, F_, nmf)                          # edm.py:645
            draw_q = orc.com_free_noise(noise_fn, B, N, nd, F_, fragment_mask)                # edm.py:669
            z = orc.inpaint_step(z, eps, sc, draw_p, draw_q, xh, nmf, fragment_mask, linker_mask, nd)
            if u < r - 1:
                alpha, sigma = jump_scalars(gamma, s, T, B, table_timesteps)
                z = renoise(z, orc.com_free_noise(noise_fn, B, N, nd, F_, nmf), alpha, sigma)
        chain[(s * keep_frames) // T] = unnorm(z)

    zeros = torch.zeros((B, 1))
    eps = dynamics_forward(sd, cfg, zeros, z, node_mask, None, edge_mask, context)
    draw_p = orc.com_free_noise(noise_fn, B, N, nd, F_, nmf)                                  # edm.py:689-690
    draw_q = orc.com_free_noise(noise_fn, B, N, nd, F_, nmf)                                  # edm.py:706
    out_l, out_f = orc.inpaint_final(z, eps, orc.step_scalars(gamma, -1, T, B, table_timesteps), draw_p, draw_q)
    chain[0] = (orc.final_frame(out_l, node_mask, nd, norm_values, norm_biases) * linker_mask
                + orc.final_frame(out_f, node_mask, nd, norm_values, norm_biases) * fragment_mask)   # edm.py:603-608
    return chain


def draw_masks(T: int, r: int, node_mask, fragment_mask):
    """The mask of every draw of an r-pass chain, in call order: 1 + T(3r-1) + 2 entries."""
    step = [node_mask, fragment_mask, node_mask] * (r - 1) + [node_mask, fragment_mask]
    return [node_mask] + step * T + [node_mask, node_mask]
