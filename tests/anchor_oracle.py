"""A host restatement of DL_CHECK_ANCHORS (stated at DL_CHECK_ANCHORS in include/difflinker_b200.h), for the tests: bonds
from fp32 distances as dl_bond_orders decides them over a molecule's checked atoms (oracle/bond_rounding.py, the
arithmetic build_xae_molecule's torch.cdist uses), then every fragment atom's count of linker neighbours, in plain Python."""
import numpy as np
import torch

import ring_oracle as ro

ANCHORS = 64


def attachments(adj, linker):
    """a_i of every atom of the (n, n) adjacency: its bonds to linker atoms on a fragment atom, 0 on a linker atom."""
    linker = np.asarray(linker, bool)
    a = adj[:, linker].sum(1).astype(np.int64)
    a[linker] = 0
    return a


def verdict(a, linker, anchor):
    """The bit: a_i == 1 on every anchor and 0 on every other fragment atom (anchor flags on linker atoms are ignored); a
    molecule with no anchor passes."""
    linker, anchor = np.asarray(linker, bool), np.asarray(anchor, bool)
    frag = ~linker
    if not (frag & anchor).any():
        return True
    return bool(np.all(a[frag & anchor] == 1) and np.all(a[frag & ~anchor] == 0))


def batch(xh, node_mask, linker_mask, anchors, is_geom, pocket_only=None):
    """(verdicts (B,) bools, attachments (B, N) int64) of a chain[0]-style (B, N, 3+F) batch: the checked atoms are the rows
    with node_mask != 0, minus those with pocket_only != 0 when given; the types are the first argmax of the first T
    feature columns; a_i sits at atom i's row, 0 on every row that is not a checked fragment atom."""
    T = 9 if is_geom else 8
    xh = xh.detach().cpu().float()
    B, N = xh.shape[:2]
    types = torch.argmax(xh[:, :, 3:3 + T], dim=2).numpy()
    keep = node_mask.detach().cpu().reshape(B, N) != 0
    if pocket_only is not None:
        keep &= pocket_only.detach().cpu().reshape(B, N) == 0
    lm = (linker_mask.detach().cpu().reshape(B, N) != 0).numpy()
    an = (anchors.detach().cpu().reshape(B, N) != 0).numpy()
    ok, att = [], np.zeros((B, N), np.int64)
    for b in range(B):
        rows = keep[b].nonzero().flatten().numpy()
        adj = ro.bonds(xh[b, rows, :3].numpy(), types[b, rows], is_geom)
        a = attachments(adj, lm[b, rows])
        att[b, rows] = a
        ok.append(verdict(a, lm[b, rows], an[b, rows]))
    return ok, att
