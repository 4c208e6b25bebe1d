"""fp64 restatement of the ODE solvers of dl_set_solver (EDM.solver_coefficients, the `ode` half of k_finish).

With gamma the schedule's fp32 entries at t = (s+1)/T and s/T (oracle.difflinker_oracle.gamma_lookup), alpha =
sqrt(sigmoid(-gamma)), sigma = sqrt(sigmoid(gamma)), lambda = -gamma/2 and h = lambda_s - lambda_t, one reverse step t -> s
of the linker sampler is, on linker rows (eps = dynamics output * linker_mask):
  xhat = (z_t - sigma_t eps) / alpha_t
  z_s  = (sigma_s / sigma_t) z_t - alpha_s expm1(-h) * D,   D = xhat (DDIM; DPM-Solver++(2M) at a row's first step)
                                                             D = (1 + 1/(2 rho)) xhat - 1/(2 rho) xhat',  rho = h'/h (2M)
and the final row returns xhat at t = 0, with no noise. Fragment rows keep z_t, padded rows stay 0.
Everything here is float64; the fp32 table is the fp64 one rounded once."""
import math

import torch

from oracle import difflinker_oracle as orc


def schedule(gamma, T, table_timesteps=None):
    """[(gamma_t, gamma_s)] of rows r = 0..T-1 (step s = T-1-r) and gamma_0, as Python floats (exact fp32 entries)."""
    if table_timesteps is None:
        table_timesteps = gamma.numel() - 1
    look = lambda v: float(orc.gamma_lookup(gamma, torch.full((1, 1), fill_value=v) / T, table_timesteps)[0, 0])
    rows = [(look(T - r), look(T - 1 - r)) for r in range(T)]
    return rows, float(orc.gamma_lookup(gamma, torch.zeros((1, 1)), table_timesteps)[0, 0])


def _alpha(g):
    return math.sqrt(1.0 / (1.0 + math.exp(g)))


def _sigma(g):
    return math.sqrt(1.0 / (1.0 + math.exp(-g)))


def table64(gamma, T, kind, table_timesteps=None):
    """The (T+1, 8) float64 table of dl_set_solver (header layout) for kind 'ddim' or 'dpmpp_2m'."""
    rows, g0 = schedule(gamma, T, table_timesteps)
    out = torch.zeros((T + 1, 8), dtype=torch.float64)
    h_prev = None
    for r, (g_t, g_s) in enumerate(rows):
        h = (g_t - g_s) / 2.0
        c1 = -_alpha(g_s) * math.expm1(-h)
        c2a, c2b = c1, 0.0
        if kind == 'dpmpp_2m' and r > 0:
            rho = h_prev / h
            c2a, c2b = c1 * (1 + 1 / (2 * rho)), -c1 / (2 * rho)
        out[r] = torch.tensor([_sigma(g_t), 1 / _alpha(g_t), _sigma(g_s) / _sigma(g_t), c1, c2a, c2b, h, 0.0],
                              dtype=torch.float64)
        h_prev = h
    out[T, 0], out[T, 1] = _sigma(g0), 1 / _alpha(g0)
    return out


def step(z, eps, row, fm, lm, hist=None):
    """One solver step with table row `row` (8 values, any float dtype, promoted to z's): (z_s, xhat). `hist` is the
    previous step's xhat for the second-order update, None for a first-order one."""
    row = row.to(dtype=z.dtype, device=z.device)
    eps = eps * lm
    xhat = row[1] * (z - row[0] * eps)
    if hist is None:
        zs = row[2] * z + row[3] * xhat
    else:
        zs = row[2] * z + (row[4] * xhat + row[5] * hist)
    return z * fm + zs * lm, xhat


def final(z, eps, row, fm, lm):
    """The final row: the normalised (x, h) = xhat on linker rows, z on fragment rows."""
    row = row.to(dtype=z.dtype, device=z.device)
    return z * fm + row[1] * (z - row[0] * eps * lm) * lm


def time_feature(s, T):
    """The time feature of step s as the engine gets it from dl_step_coef: fp32 (s+1)/T, as a (1,1) tensor."""
    return (torch.full((1, 1), fill_value=s + 1) / T).to(torch.float64)


def sample(forward, z_T, table, kind, T, fm, lm, t0=None):
    """The solver's loop from z_T (or z_t0 with start step t0): returns the normalised continuous final (x, h) before the
    unnormalisation and argmax, and [z_s] of every step. `forward(t, z)` is the dynamics output; `table` the (T+1, 8) solver
    table (fp64 or its fp32 rounding)."""
    t0 = T if t0 is None else t0
    z, hist, zs = z_T, None, []
    for s in range(t0 - 1, -1, -1):
        r = T - 1 - s
        z, xhat = step(z, forward(time_feature(s, T), z), table[r], fm, lm, hist if kind == 'dpmpp_2m' else None)
        hist = xhat
        zs.append(z)
    return final(z, forward(torch.zeros((1, 1), dtype=torch.float64), z), table[T], fm, lm), zs
