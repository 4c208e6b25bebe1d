"""Clash guidance restated in numpy fp64: the push of dl_set_clash_guidance / dl_clash_guide on (B,N) batches.

Linker atoms are the rows with node_mask, linker_mask and pocket_only == 0; pocket atoms the rows with node_mask and
pocket_only != 0. Each linker atom i moves to

    p_i + scale * sum_k max(0, r_ik - d_ik) (p_i - p_k) / d_ik,   d_ik = |p_i - p_k|,

k over the pocket atoms, r_ik = table[min type][max type] / 100 Angstrom (a negative entry exempts the pair). Every term comes
from the input state; a pair at d_ik = 0 or with a NaN distance contributes nothing."""
import numpy as np

U = 2.0 ** -24


def rows(node_mask, linker_mask, pocket_only):
    """(linker, pocket) (B,N) bool masks."""
    live = np.asarray(node_mask) != 0
    pocket = live & (np.asarray(pocket_only) != 0)
    linker = live & ~pocket & (np.asarray(linker_mask) != 0)
    return linker, pocket


def push(x, types, node_mask, linker_mask, pocket_only, table, scale):
    """(x_new (B,N,3) fp64, moved (B,N) bool, bound (B,N) fp64, slack (B,N) fp64).

    moved: linker atoms with at least one contributing pair. bound: an error bound for an fp32 evaluation of the push
    from the same fp32 inputs, 16 u (|p_i| + scale sum_k (r_ik + w_ik d_ik)) per coordinate: every term of the sum is
    rounded a handful of times (the difference, the distance's fma chain and square root, r - d, the division, the fma
    into the lane's sum) and the 32 lane sums are added in five shuffle rounds, each step relative u on a quantity
    bounded by r_ik or w_ik d_ik; the final fma rounds once on |p_i|. slack: min_k |d_ik - r_ik| over the atom's
    non-exempt pairs, the distance to the nearest threshold (an fp32 distance within a few ulp of r_ik may decide the
    pair the other way)."""
    x = np.asarray(x, dtype=np.float64)
    types = np.asarray(types)
    table = np.asarray(table, dtype=np.float64)
    linker, pocket = rows(node_mask, linker_mask, pocket_only)
    B, N = linker.shape
    out = x.copy()
    moved = np.zeros((B, N), dtype=bool)
    bound = np.zeros((B, N))
    slack = np.full((B, N), np.inf)
    for b in range(B):
        li, pk = np.nonzero(linker[b])[0], np.nonzero(pocket[b])[0]
        if len(li) == 0 or len(pk) == 0:
            continue
        diff = x[b][li][:, None, :] - x[b][pk][None, :, :]
        with np.errstate(invalid="ignore"):
            d = np.sqrt((diff * diff).sum(-1))
            ti, tk = types[b][li][:, None], types[b][pk][None, :]
            r = table[np.minimum(ti, tk), np.maximum(ti, tk)] / 100.0
            on = (r >= 0) & (d < r) & (d > 0)
            w = np.where(on, (r - d) / np.where(on, d, 1.0), 0.0)
            term = np.where(on[..., None], w[..., None] * diff, 0.0)
            gap = np.where(r >= 0, np.abs(d - r), np.inf)
        out[b, li] = x[b, li] + scale * term.sum(1)
        moved[b, li] = on.any(1)
        bound[b, li] = 16 * U * (np.abs(x[b, li]).max(-1) + scale * np.where(on, r + w * d, 0.0).sum(1))
        slack[b, li] = np.where(np.isnan(gap), np.inf, gap).min(1)
    return out, moved, bound, slack


def first_argmax(h):
    """torch.argmax over the last axis: the first maximum, NaN winning."""
    h = np.asarray(h)
    nan = np.isnan(h)
    return np.where(nan.any(-1), nan.argmax(-1), np.nan_to_num(h, nan=-np.inf).argmax(-1))
