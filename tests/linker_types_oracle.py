"""fp64 restatement of the linker sampler's loop with linker types (dl_set_linker_types, the TYPES half of k_finish).

With off = (0 - bias1) / norm1 the normalised value of a one-hot's zero and (alpha_t, sigma_t) = start_scalars(t)
(EDM.fixed_atom_scalars: row T-1-t, row T for t = T), a type channel c that molecule b's set excludes, on a linker row
that fixed_atoms does not keep, has its data prediction xhat_c = (z_t,c - sigma_t eps_c) / alpha_t set to off:
  ancestral step from t   eps_c replaced by (z_t,c - alpha_t off) / sigma_t, then the plain update
                          (oracle.difflinker_oracle.linker_step; linker_final at t = 0)
  ODE step from t         xhat_c = off in the solver's update (ode_solver_oracle.step), and in the 2M history
  final decode            the argmax over the allowed channels only
Everything here is float64; the scalar table is the fp32 one, promoted."""
import torch

import ode_solver_oracle as oso
from oracle import difflinker_oracle as orc

import fixed_atoms_oracle as fao


def off_value(norm1, bias1=0.0):
    return (0.0 - bias1) / norm1


def excluded(allowed, lm, fixed=None, n_dims=3):
    """(B, N, 3+F) bool: the channels the projection touches. `allowed` (B, F) bool, lm (B, N, 1), fixed (B, N, 1) or None."""
    B, F = allowed.shape
    N = lm.shape[1]
    ex = torch.zeros((B, N, n_dims + F), dtype=torch.bool, device=lm.device)
    ex[..., n_dims:] = ~allowed.to(lm.device)[:, None, :]
    row = lm[..., 0] != 0
    if fixed is not None:
        row &= fixed[..., 0] == 0
    return ex & row[..., None]


def project_eps(z, eps, row, ex, off):
    """eps with the excluded channels ex replaced by (z - alpha off) / sigma, row = (alpha_t, sigma_t)."""
    row = row.to(dtype=z.dtype, device=z.device)
    return torch.where(ex, (z - row[0] * off) / row[1], eps)


def sample_ancestral(forward, xh, draws, fm, lm, allowed, gamma, tab, T, B, off, fixed=None, t0=None):
    """The ancestral loop with linker types (and fixed atoms, when `fixed` is given) from step t0 (None: T): (final
    normalised (x, h), [z_s of every step])."""
    fx = torch.zeros_like(lm) if fixed is None else fixed
    ex = excluded(allowed, lm, fx)
    z = fao.start(xh, fm, lm, draws[0], fx, tab, T, t0)
    t0 = T if t0 is None else t0
    zs = []
    for s in range(t0 - 1, -1, -1):
        sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
        n = draws[t0 - s]
        eps = project_eps(z, forward(oso.time_feature(s, T), z), fao.start_row(tab, T, s + 1), ex, off)
        z = orc.linker_step(z, eps, sc, n, fm, lm)
        z = fao.replace(z, xh, tab[T - 1 - s], n * lm, fx)
        zs.append(z)
    sc = orc.step_scalars(gamma, -1, T, B, gamma.numel() - 1)
    eps = project_eps(z, forward(torch.zeros((1, 1), dtype=torch.float64), z), tab[T - 1], ex, off)
    out = orc.linker_final(z, eps, sc, draws[t0 + 1], fm, lm)
    return torch.where(fx != 0, xh, out), zs


def ode_step(z, eps, row, fm, lm, ex, off, hist=None):
    """ode_solver_oracle.step with xhat = off on the excluded channels: (z_s, the projected xhat)."""
    row = row.to(dtype=z.dtype, device=z.device)
    xhat = torch.where(ex, torch.full_like(z, off), row[1] * (z - row[0] * eps * lm))
    zs = row[2] * z + row[3] * xhat if hist is None else row[2] * z + (row[4] * xhat + row[5] * hist)
    return z * fm + zs * lm, xhat


def sample_ode(forward, xh, eps0, fm, lm, allowed, solver_table, kind, tab, T, off, t0=None):
    """The ODE solver's loop with linker types: (final normalised (x, h), [z_s of every step])."""
    fx = torch.zeros_like(lm)
    ex = excluded(allowed, lm)
    z = fao.start(xh, fm, lm, eps0, fx, tab, T, t0)
    t0 = T if t0 is None else t0
    hist, zs = None, []
    for s in range(t0 - 1, -1, -1):
        z, hist_new = ode_step(z, forward(oso.time_feature(s, T), z), solver_table[T - 1 - s], fm, lm, ex, off,
                               hist if kind == 'dpmpp_2m' else None)
        hist = hist_new
        zs.append(z)
    row = solver_table[T].to(z.dtype)
    xhat = torch.where(ex, torch.full_like(z, off), row[1] * (z - row[0] * forward(torch.zeros((1, 1), dtype=torch.float64), z) * lm))
    return z * fm + xhat * lm, zs


def final_frame(out, node_mask, allowed, lm, norm=(1.0, 4.0, 10.0), fixed=None, n_dims=3):
    """chain[0] of a final (x, h): orc.final_frame with the excluded channels of the free linker rows out of the argmax."""
    ex = excluded(allowed, lm, fixed, n_dims)
    ho = out[..., n_dims:] * norm[1]
    ho = torch.where(ex[..., n_dims:], torch.full_like(ho, -float('inf')), ho)
    onehot = torch.nn.functional.one_hot(ho.argmax(dim=2), ho.shape[2]).to(out.dtype) * node_mask
    return torch.cat([out[..., :n_dims] * norm[0], onehot], dim=2)
