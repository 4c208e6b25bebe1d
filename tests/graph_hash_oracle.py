"""A host restatement of the graph hash and the uniqueness verdict of DL_CHECK_UNIQUE (stated at DL_CHECK_UNIQUE in
include/difflinker_b200.h), for the tests: Python ints masked to 64 bits, and bond orders from fp32 distances as
dl_bond_orders computes them: torch.cdist's arithmetic over the molecule's atoms (oracle/bond_rounding.py)."""
import numpy as np
import torch

from difflinker_b200 import molecule_builder as mb
from oracle import bond_rounding as br

M64 = (1 << 64) - 1
TAG = 0x67726170682D776C                      # "graph-wl"
ORDER = 0x9E3779B97F4A7C15
UNIQUE = 8


def mix(z):
    """The splitmix64 finaliser of dl_size_uniform, modulo 2^64."""
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def graph_hash(types, orders):
    """H of a graph of n atoms with types[i] and the symmetric (n, n) bond orders orders[i][j] in {0, 1, 2, 3}."""
    n = len(types)
    c = [mix(TAG ^ (int(t) + 1)) for t in types]
    orders = np.asarray(orders)
    nbrs = [[] for _ in range(n)]
    for i, j in zip(*np.nonzero(orders)):
        if i != j:
            nbrs[int(i)].append((int(j), int(orders[i, j])))
    for _ in range(min(n, 64)):
        c = [mix(c[i] + sum(mix(c[j] + o * ORDER) for j, o in nbrs[i])) for i in range(n)]
    return mix(n + sum(c))


def bond_order_matrix(x, types, thr):
    """(n, n) bond orders of get_bond_order with the (T, T) threshold tables thr = (thr1, thr2, thr3) read [min][max], and
    the smallest |distance - threshold| over every existing threshold of every pair. The pairs are measured as the
    kernels measure them in a molecule of these n atoms (br.pair_dist_pm)."""
    x = np.asarray(x, np.float32)
    types = np.asarray(types)
    n = len(types)
    if n == 0:
        return np.zeros((0, 0), np.int64), np.inf
    d = br.pair_dist_pm(x)
    t1, t2, t3 = br.threshold_lookup(types, thr)
    o = br.orders_of(d, types, thr)
    near = np.inf
    off = ~np.eye(n, dtype=bool)
    for t in (t1, t2, t3):
        m = np.abs(d - t)[(t >= 0) & off & ~np.isnan(d)]
        if m.size:
            near = min(near, float(m.min()))
    return o, near


def batch_hashes(xh, node_mask, is_geom, pocket_only=None):
    """((B,) hashes as Python ints, (B,) smallest |distance - threshold|) of a chain[0]-style (B, N, 3+F) batch: the atoms
    are the rows with node_mask != 0, minus those with pocket_only != 0 when given; the types are the first argmax of the
    first T feature columns (torch.argmax: NaN wins)."""
    T = 9 if is_geom else 8
    xh = xh.detach().cpu().float()
    B, N = xh.shape[:2]
    types = torch.argmax(xh[:, :, 3:3 + T], dim=2).numpy()
    keep = node_mask.detach().cpu().reshape(B, N) != 0
    if pocket_only is not None:
        keep &= pocket_only.detach().cpu().reshape(B, N) == 0
    thr = [t.numpy() for t in mb.threshold_tables(is_geom)]
    hashes, near = [], []
    for b in range(B):
        rows = keep[b].nonzero().flatten().numpy()
        o, m = bond_order_matrix(xh[b, rows, :3].numpy(), types[b, rows], thr)
        hashes.append(graph_hash(types[b, rows], o))
        near.append(m)
    return hashes, near


def verdict(hashes, flags, passed, require, candidates=None):
    """The passed bits after the uniqueness verdict: `candidates` are the rows evaluated (None: every row, as after the first
    loop), the other rows that pass every bit of `require` are keepers, and a candidate is eligible when its flag is 0 and
    it has every other required bit. Candidate b gets UNIQUE iff its hash equals no keeper's and no eligible candidate
    b' < b has the same hash."""
    B = len(hashes)
    cand = list(range(B)) if candidates is None else sorted(candidates)
    cset = set(cand)
    other = require & ~UNIQUE
    keeper = {hashes[k] for k in range(B) if k not in cset and flags[k] == 0 and passed[k] & require == require}
    out = list(passed)
    for i, b in enumerate(cand):
        dup = hashes[b] in keeper or any(flags[c] == 0 and passed[c] & other == other and hashes[c] == hashes[b]
                                         for c in cand[:i])
        out[b] = passed[b] & ~UNIQUE if dup else passed[b] | UNIQUE
    return out


def as_int64(h):
    """The int64 with the 64 bits of hash h, as graph_hashes returns it."""
    return h - (1 << 64) if h >= 1 << 63 else h
