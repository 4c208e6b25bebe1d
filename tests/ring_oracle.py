"""A host restatement of the ring-size mask of DL_CHECK_RINGS (stated at DL_CHECK_RINGS in include/difflinker_b200.h), for
the tests: bonds from fp32 distances as dl_bond_orders decides them over a molecule's checked atoms
(oracle/bond_rounding.py), then a breadth-first search per bond with a linker end, in plain Python."""
from collections import deque

import numpy as np
import torch

from difflinker_b200 import molecule_builder as mb
from oracle import bond_rounding as br

RINGS = 32


def bonds(x, types, is_geom):
    """(n, n) bool adjacency of the atoms x (n, 3) with types: get_bond_order > 0 over these n atoms (br.bond_orders)."""
    thr = [t.numpy() for t in mb.threshold_tables(is_geom)]
    x = np.asarray(x, np.float32).reshape(-1, 3)
    if x.shape[0] == 0:
        return np.zeros((0, 0), bool)
    return br.bond_orders(x, np.asarray(types), thr) > 0


def smallest_ring(adj, u, v):
    """Atoms on a shortest cycle through the bond (u, v): 1 + the u-v distance without that bond; 0 on no cycle."""
    n = adj.shape[0]
    dist = [-1] * n
    dist[u] = 0
    q = deque([u])
    while q:
        i = q.popleft()
        for j in np.nonzero(adj[i])[0]:
            j = int(j)
            if (i, j) in ((u, v), (v, u)) or dist[j] >= 0:
                continue
            dist[j] = dist[i] + 1
            if j == v:
                return dist[j] + 1
            q.append(j)
    return 0


def ring_mask(adj, linker):
    """The mask: bit min(k, 63) for every bond with a linker end whose smallest ring has k atoms."""
    mask = 0
    n = adj.shape[0]
    for u in range(n):
        for v in range(u + 1, n):
            if adj[u, v] and (linker[u] or linker[v]):
                k = smallest_ring(adj, u, v)
                if k:
                    mask |= 1 << min(k, 63)
    return mask


def batch_masks(xh, node_mask, linker_mask, is_geom, pocket_only=None):
    """(B,) masks as Python ints of a chain[0]-style (B, N, 3+F) batch: the checked atoms are the rows with node_mask != 0,
    minus those with pocket_only != 0 when given; the types are the first argmax of the first T feature columns."""
    T = 9 if is_geom else 8
    xh = xh.detach().cpu().float()
    B, N = xh.shape[:2]
    types = torch.argmax(xh[:, :, 3:3 + T], dim=2).numpy()
    keep = node_mask.detach().cpu().reshape(B, N) != 0
    if pocket_only is not None:
        keep &= pocket_only.detach().cpu().reshape(B, N) == 0
    lm = linker_mask.detach().cpu().reshape(B, N) != 0
    out = []
    for b in range(B):
        rows = keep[b].nonzero().flatten().numpy()
        adj = bonds(xh[b, rows, :3].numpy(), types[b, rows], is_geom)
        out.append(ring_mask(adj, lm[b, rows].numpy()))
    return out


def as_int64(m):
    """The int64 with the 64 bits of mask m, as the library returns it."""
    return m - (1 << 64) if m >= 1 << 63 else m
