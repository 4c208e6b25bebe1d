"""fp64 restatement of the linker sampler's loop with fixed atoms (dl_set_fixed_atoms, the FIX half of k_finish).

With xh the normalised input, eps_0 a row's draw 0, nz_s the draw the ancestral update of step s reads, and (alpha_s,
sigma_s) = start_scalars(s) (EDM.fixed_atom_scalars: row T-1-s, row T = the start at T), a kept linker row is
  start         alpha xh + sigma eps_0 with the scalars of the call's start
  step s < T    alpha_s xh + sigma_s nz_s (ancestral), alpha_s xh + sigma_s eps_0 (ODE solvers)
  final         xh
and every other row takes the plain update (oracle.difflinker_oracle.linker_step / ode_solver_oracle.step) from the
replaced state. Everything here is float64; the scalar table is the fp32 one, promoted."""
import torch

import ode_solver_oracle as oso
from oracle import difflinker_oracle as orc


def table(edm, n_samples):
    """EDM.fixed_atom_scalars(n_samples) as a (T + 1, 2) float64 tensor."""
    return torch.tensor(list(edm.fixed_atom_scalars(n_samples)), dtype=torch.float64).reshape(edm.T + 1, 2)


def replace(z, xh, row, eps, fixed):
    """z with the kept rows (fixed (B, N, 1), 0 or 1) set to row[0] xh + row[1] eps."""
    row = row.to(dtype=z.dtype, device=z.device)
    return torch.where(fixed != 0, row[0] * xh + row[1] * eps, z)


def start_row(tab, T, t0):
    """The scalars (alpha, sigma) = start_scalars(t0) of the table: row T at t0 = T, else the row of step t0."""
    return tab[T] if t0 == T else tab[T - 1 - t0]


def start(xh, fm, lm, eps0, fixed, tab, T, t0=None):
    """z of the loop's start: from noise (t0 None: xh on fragments, eps_0 on linker rows) or q(z_t0 | x) (partial
    diffusion), the kept rows from q(z_t | x) at the start either way."""
    eps0 = eps0 * lm
    row = start_row(tab, T, T if t0 is None else t0).to(xh.dtype)
    z = xh * fm + (eps0 if t0 is None else row[0] * xh + row[1] * eps0) * lm
    return replace(z, xh, row, eps0, fixed)


def sample_ancestral(forward, xh, draws, fm, lm, fixed, gamma, tab, T, B, t0=None):
    """The ancestral loop with fixed atoms from step t0 (None: T): (final normalised (x, h), [z_s of every step]).
    `draws` holds the call's draws (t0 + 2 of them, the row's own order), `tab` the (T + 1, 2) scalars."""
    z = start(xh, fm, lm, draws[0], fixed, tab, T, t0)
    t0 = T if t0 is None else t0
    zs = []
    for s in range(t0 - 1, -1, -1):
        sc = orc.step_scalars(gamma, s, T, B, gamma.numel() - 1)
        n = draws[t0 - s]
        z = orc.linker_step(z, forward(oso.time_feature(s, T), z), sc, n, fm, lm)
        z = replace(z, xh, tab[T - 1 - s], n * lm, fixed)
        zs.append(z)
    sc = orc.step_scalars(gamma, -1, T, B, gamma.numel() - 1)
    out = orc.linker_final(z, forward(torch.zeros((1, 1), dtype=torch.float64), z), sc, draws[t0 + 1], fm, lm)
    return torch.where(fixed != 0, xh, out), zs


def sample_ode(forward, xh, eps0, fm, lm, fixed, solver_table, kind, tab, T, t0=None):
    """The ODE solver's loop (ode_solver_oracle.sample) with fixed atoms: the kept rows take alpha_s xh + sigma_s eps_0 and
    their 2M history never enters (it is the free update's data prediction, which only the kept row would use)."""
    z = start(xh, fm, lm, eps0, fixed, tab, T, t0)
    t0 = T if t0 is None else t0
    hist, zs = None, []
    for s in range(t0 - 1, -1, -1):
        r = T - 1 - s
        z, xhat = oso.step(z, forward(oso.time_feature(s, T), z), solver_table[r], fm, lm,
                           hist if kind == 'dpmpp_2m' else None)
        z = replace(z, xh, tab[r], eps0 * lm, fixed)
        hist = xhat
        zs.append(z)
    out = oso.final(z, forward(torch.zeros((1, 1), dtype=torch.float64), z), solver_table[T], fm, lm)
    return torch.where(fixed != 0, xh, out), zs
