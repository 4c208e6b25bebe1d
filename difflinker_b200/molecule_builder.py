"""Bond inference: `src/molecule_builder.py::build_xae_molecule` / `get_bond_order` (lines 44-102) for whole batches on the
GPU (`dl_bond_orders`) instead of an O(n^2) Python loop with one `.item()` per atom pair.
RDKit molecule construction (`build_molecule`, molecule_builder.py:29-42) stays with the caller: RDKit is not part of
the path (SURVEY.md section 8(f) rank 4). `connected` and `valence_ok` decide on the device what the reference's
`validity_and_connectivity` asks of those molecules, the latter as "explicit valence within a table". `clash_free` is this
project's own check, with no reference counterpart: whether a linker runs into the pocket. `graph_hashes` gives the hash
behind uniqueness (compute_metrics.py's share of distinct molecules): equal for isomorphic bond graphs. `linker_hashes`
and `known_linkers` give the linker-scoped hash behind novelty (the share of linkers not in the training set).
`ring_sizes` and `ring_sizes_ok` give the smallest rings the linker closes, for a ring-size rule. `attachments` and
`anchors_ok` give where the linker bonds to the fragments (compute_metrics.py's find_exit), for the anchors of --anchors.
"""
import operator

import torch

from . import _native
from .output import GEOM_IDX2ATOM, IDX2ATOM

# Bond lengths in pm for the atom types of the one-hot encodings (src/const.py:66-146, tables BONDS_1/2/3), keyed by the
# pair ORDERED BY TYPE INDEX -- `sorted([atom_types[i], atom_types[j]])` (molecule_builder.py:66) -- which is the only
# direction the reference ever looks up; a missing key means "no typical bond length" (get_bond_order returns 0).
SINGLE = {('C', 'C'): 154, ('C', 'O'): 143, ('C', 'N'): 147, ('C', 'F'): 135, ('C', 'S'): 182, ('C', 'Cl'): 177,
          ('C', 'Br'): 194, ('C', 'I'): 214, ('C', 'P'): 184, ('O', 'O'): 148, ('O', 'N'): 140, ('O', 'F'): 142,
          ('O', 'S'): 151, ('O', 'Cl'): 164, ('O', 'Br'): 172, ('O', 'I'): 194, ('O', 'P'): 163, ('N', 'N'): 145,
          ('N', 'F'): 136, ('N', 'S'): 168, ('N', 'Cl'): 175, ('N', 'Br'): 214, ('N', 'I'): 222, ('N', 'P'): 177,
          ('F', 'F'): 142, ('F', 'S'): 158, ('F', 'Cl'): 166, ('F', 'Br'): 178, ('F', 'I'): 187, ('F', 'P'): 156,
          ('S', 'S'): 204, ('S', 'Cl'): 207, ('S', 'Br'): 225, ('S', 'I'): 234, ('S', 'P'): 210, ('Cl', 'Cl'): 199,
          ('Cl', 'Br'): 214, ('Cl', 'P'): 203, ('Br', 'Br'): 228, ('Br', 'P'): 222, ('I', 'I'): 266, ('P', 'P'): 221}
DOUBLE = {('C', 'C'): 134, ('C', 'O'): 120, ('C', 'N'): 129, ('C', 'S'): 160, ('O', 'O'): 121, ('O', 'N'): 121,
          ('O', 'P'): 150, ('N', 'N'): 125, ('S', 'P'): 186}
TRIPLE = {('C', 'C'): 120, ('C', 'O'): 113, ('C', 'N'): 116, ('N', 'N'): 110}
MARGINS_EDM = [10, 5, 2]                                                                   # src/const.py:180
# The most bond order an atom of each element may carry in valences / valence_ok: the largest entry of RDKit's default
# valence list for the element.
MAX_VALENCE = {'C': 4, 'N': 3, 'O': 2, 'F': 1, 'S': 6, 'Cl': 1, 'Br': 1, 'I': 5, 'P': 7}
# Bondi van der Waals radii in Angstrom (J. Phys. Chem. 68, 441 (1964)), for the pocket-clash check's default table.
VDW_RADII = {'C': 1.70, 'N': 1.55, 'O': 1.52, 'F': 1.47, 'P': 1.80, 'S': 1.80, 'Cl': 1.75, 'Br': 1.85, 'I': 1.98}


def threshold_tables(is_geom, margins=MARGINS_EDM):
    """(T,T) fp32 thresholds [min type][max type] = bond length + margin in pm; -1 where the pair is absent."""
    idx2atom = GEOM_IDX2ATOM if is_geom else IDX2ATOM
    T = len(idx2atom)
    out = []
    for table, margin in ((SINGLE, margins[0]), (DOUBLE, margins[1]), (TRIPLE, margins[2])):
        t = torch.full((T, T), -1.0)
        for a in range(T):
            for c in range(a, T):
                v = table.get((idx2atom[a], idx2atom[c]))
                if v is not None:
                    t[a, c] = float(v + margin)
        out.append(t)
    return out


def max_valence_table(is_geom):
    """(T,) int32: MAX_VALENCE by atom type index (IDX2ATOM, or GEOM_IDX2ATOM with is_geom)."""
    idx2atom = GEOM_IDX2ATOM if is_geom else IDX2ATOM
    return torch.tensor([MAX_VALENCE[idx2atom[t]] for t in range(len(idx2atom))], dtype=torch.int32)


def check_tables(is_geom, require, max_valence=None):
    """The CPU tables the molecule checks `require` (an OR of _native.CHECK_*) read: [thr1] for connectivity alone,
    [thr1, thr2, thr3] for CHECK_UNIQUE or CHECK_NOVEL (the bond orders of the graph hash), and [thr1, thr2, thr3,
    max_valence] once CHECK_VALENCE is required (threshold_tables; `max_valence` a (T,) integer table by atom type index, by
    default max_valence_table(is_geom))."""
    thr = threshold_tables(is_geom)
    if not require & _native.CHECK_VALENCE:
        return thr if require & (_native.CHECK_UNIQUE | _native.CHECK_NOVEL) else thr[:1]
    mv = max_valence_table(is_geom) if max_valence is None else torch.as_tensor(max_valence).to(torch.int32).contiguous()
    if mv.shape != (thr[0].shape[0],):
        raise ValueError(f"max_valence holds one entry per atom type, {thr[0].shape[0]} (got shape {tuple(mv.shape)})")
    return thr + [mv]


def clash_table(is_geom, scale=0.75):
    """(T,T) fp32 clash distances in pm for the pocket-clash check (sample_chain(require_clash_free=True), clash_free): entry
    [a][b] = fp32(100 * scale * (R_a + R_b)), evaluated in double, with R the VDW_RADII of the two atom types (IDX2ATOM, or
    GEOM_IDX2ATOM with is_geom). Symmetric; the check reads [min type][max type]. A linker atom closer than that to a pocket
    atom clashes with it. The default scale, 0.75, is a common protein-ligand contact tolerance (C-C 2.55 A, N-O 2.30 A, below
    hydrogen-bond distances); it is a default, not validated against any docking tool. A caller may set entries negative
    to exempt a pair (e.g. a covalent warhead's element)."""
    idx2atom = GEOM_IDX2ATOM if is_geom else IDX2ATOM
    T = len(idx2atom)
    r = [VDW_RADII[idx2atom[t]] for t in range(T)]
    return torch.tensor([[100.0 * scale * (r[a] + r[b]) for b in range(T)] for a in range(T)], dtype=torch.float32)


@torch.no_grad()
def bond_orders(one_hot, x, node_mask, is_geom, margins=MARGINS_EDM):
    """Batched E of build_xae_molecule: (B,N,N) int8 on the inputs' device, E[b,i,j] (i > j) = bond order, else 0.
    `x` may be (B,N,3) or chain[0]-style (B,N,3+F); atom types are argmax(one_hot) (molecule_builder.py:20).
    Distances are torch.cdist's on the CPU over each molecule's n rows with node_mask != 0, row i the later atom: the direct
    form for n <= 25, the matmul form (_euclidean_dist) above, as stated at dl_molecule_checks in the header. torch's CPU
    sqrt (MKL vsSqrt) is not always correctly rounded, so a pair within one ulp of a threshold can be decided the other way
    by the reference; oracle/bond_rounding.py restates this arithmetic exactly."""
    dev = x.device
    if dev.type != 'cuda':
        raise RuntimeError("bond_orders runs on the GPU (no CPU fallback); move the tensors to the device")
    B, N = x.shape[:2]
    xs = x.float().contiguous()
    types = torch.argmax(one_hot, dim=2).to(torch.int32).contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    t1, t2, t3 = [t.to(dev).contiguous() for t in threshold_tables(is_geom, margins)]
    E = torch.empty((B, N, N), dtype=torch.int8, device=dev)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_bond_orders(B, N, t1.shape[0], xs.data_ptr(), xs.shape[2], types.data_ptr(), nm.data_ptr(),
                                         t1.data_ptr(), t2.data_ptr(), t3.data_ptr(), E.data_ptr(), st), "dl_bond_orders")
    return E


@torch.no_grad()
def connected(xh, node_mask, is_geom, pocket_only=None):
    """(B,) bool on the device: whether each molecule is in one piece (dl_molecule_check with CHECK_CONNECTED, the check
    behind sample_chain(require_connected=True)). Its atoms are the rows with node_mask != 0, minus those with
    pocket_only != 0 when given; atoms i and j bond iff get_bond_order > 0 on a distance measured as in bond_orders, over
    these checked atoms (so dropping the pocket can change the form a pair is measured in). `xh` is
    chain[0]-style (B,N,3+F): the atom types are argmax of its first T feature columns (T = 9 with is_geom, else 8). One
    atom is connected, none is not."""
    passed, _ = _molecule_check(xh, node_mask, is_geom, pocket_only, None, _native.CHECK_CONNECTED, False)
    return (passed & _native.CHECK_CONNECTED) != 0


@torch.no_grad()
def _molecule_check(xh, node_mask, is_geom, pocket_only, max_valence, require, want_valence):
    """dl_molecule_check on a chain[0]-style batch: ((B,) int32 verdict bits, (B,N) int32 valences or None)."""
    dev = xh.device
    if dev.type != 'cuda':
        raise RuntimeError("the molecule checks run on the GPU (no CPU fallback); move the tensors to the device")
    B, N = xh.shape[:2]
    xs = xh.float().contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    po = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    tables = [t.to(dev) for t in check_tables(is_geom, require, max_valence)]
    checks = _native.DLMoleculeChecks.of(require, tables)
    passed = torch.empty(B, dtype=torch.int32, device=dev)
    valence = torch.empty((B, N), dtype=torch.int32, device=dev) if want_valence else None
    lib = _native.load_library()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_molecule_check(B, N, checks, xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                            None if po is None else po.data_ptr(), 1, int(po is not None), passed.data_ptr(),
                                            None if valence is None else valence.data_ptr(), st), "dl_molecule_check")
    return passed, valence


def valences(xh, node_mask, is_geom, pocket_only=None, max_valence=None):
    """(B,N) int32 on the device: every checked atom's valence -- the sum of get_bond_order over its pairs with the other
    checked atoms, i.e. the row-plus-column sum of bond_orders' E -- and 0 on the other rows (dl_molecule_check, the check
    behind sample_chain(require_valid=True)). `xh`, `node_mask`, `pocket_only` and the checked atoms as in connected(). Each
    pair is measured as torch.cdist measures it over the n checked atoms, the later atom as the row (bond_orders): with a
    pocket dropped, n counts the atoms left."""
    return _molecule_check(xh, node_mask, is_geom, pocket_only, max_valence, _native.CHECK_VALENCE, True)[1]


def valence_ok(xh, node_mask, is_geom, pocket_only=None, max_valence=None):
    """(B,) bool on the device: whether every checked atom of a molecule has valence <= max_valence[its type]; a molecule
    without atoms passes. `max_valence` is a (T,) integer table by atom type index, by default max_valence_table(is_geom).
    This is "explicit valence within the table" on bond_orders' own orders. The molecules build_molecule makes carry single,
    double and triple bonds only, no aromatic flags and no formal charges, so it is how they are expected to fail
    Chem.SanitizeMol; that equivalence has not been verified against RDKit."""
    passed, _ = _molecule_check(xh, node_mask, is_geom, pocket_only, max_valence, _native.CHECK_VALENCE, False)
    return (passed & _native.CHECK_VALENCE) != 0


@torch.no_grad()
def graph_hashes(xh, node_mask, is_geom, pocket_only=None):
    """(B,) int64 on the device, holding the uint64 bits of every molecule's graph hash (dl_molecule_hash, the hash behind
    sample_chain(require_unique=True)): Weisfeiler-Lehman colour refinement over the atoms, their types and bond_orders'
    orders, stated at DL_CHECK_UNIQUE in the header. The atoms and types are those of connected(). Isomorphic graphs
    always hash equal, whatever the row order, pose or padding; non-isomorphic graphs can collide (1-WL-equivalent pairs
    always do, and a 64-bit collision is possible); stereochemistry is ignored, and equal hashes have not been verified to
    mean equal RDKit canonical SMILES. Compare these to deduplicate across calls or devices. The bond orders are
    measured as torch.cdist measures them over the n hashed atoms, the later atom as the row (bond_orders): the direct form
    for n <= 25, the matmul form above."""
    dev = xh.device
    if dev.type != 'cuda':
        raise RuntimeError("the molecule checks run on the GPU (no CPU fallback); move the tensors to the device")
    B, N = xh.shape[:2]
    xs = xh.float().contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    po = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    tables = [t.to(dev) for t in check_tables(is_geom, _native.CHECK_UNIQUE)]
    checks = _native.DLMoleculeChecks.of(_native.CHECK_UNIQUE, tables)
    out = torch.empty(B, dtype=torch.int64, device=dev)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_molecule_hash(B, N, checks, xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                           None if po is None else po.data_ptr(), 1, int(po is not None), out.data_ptr(),
                                           st), "dl_molecule_hash")
    return out


def linker_hashes(xh, node_mask, linker_mask, is_geom, pocket_only=None):
    """(B,) int64 on the device: every molecule's linker hash (the L of DL_CHECK_NOVEL, the hash behind
    sample_chain(require_novel=True)) -- graph_hashes over the rows with node_mask != 0 and linker_mask != 0, i.e. the graph
    the linker atoms induce, as the reference's linker is the molecule with every fragment atom removed. A molecule without
    linker atoms hashes to 0. The pairs are measured over the linker atoms alone (n is their count, bond_orders), so a
    pair can be decided differently here than in graph_hashes of the whole molecule, as the reference decides it when it
    builds the linker on its own."""
    B, N = xh.shape[:2]
    nm = (node_mask.reshape(B, N) != 0) & (linker_mask.reshape(B, N).to(node_mask.device) != 0)
    return graph_hashes(xh, nm, is_geom, pocket_only)


def sort_unsigned(hashes):
    """A 1-D int64 tensor of uint64 bits sorted in unsigned order, on its own device: the sign bit is flipped, the values
    sorted as int64 and the bit flipped back (flipping the sign bit maps unsigned order onto signed order)."""
    sign = torch.tensor(-(1 << 63), dtype=torch.int64, device=hashes.device)
    return torch.sort(hashes.to(torch.int64) ^ sign).values ^ sign


@torch.no_grad()
def known_linkers(items, is_geom, batch_size=256, device=None):
    """(K,) int64 on the device: the sorted (unsigned order), de-duplicated linker hashes of dataset items -- the dicts
    ZincDataset / MOADDataset hold in .data, with 'positions' (n, 3) in Angstrom, 'one_hot' (n, F) and 'linker_mask' (n,)
    (plus 'fragment_mask') -- for EDM.known_linkers. Items are collated with batching.collate, `batch_size` at a time, on
    `device` (default: the current CUDA device), and hashed with linker_hashes. Saving the set is the caller's business."""
    from .batching import collate
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != 'cuda':
        raise RuntimeError("known_linkers hashes on the GPU (no CPU fallback); pass a CUDA device")
    items = list(items)
    keys = ('positions', 'one_hot', 'fragment_mask', 'linker_mask')
    out = []
    for b0 in range(0, len(items), batch_size):
        batch = collate([{k: torch.as_tensor(it[k]).to(dev) for k in keys} for it in items[b0:b0 + batch_size]])
        xh = torch.cat([batch['positions'].float(), batch['one_hot'].float()], dim=2)
        out.append(linker_hashes(xh, batch['atom_mask'], batch['linker_mask'], is_geom))
    if not out:
        return torch.zeros(0, dtype=torch.int64, device=dev)
    s = sort_unsigned(torch.cat(out))
    keep = torch.ones_like(s, dtype=torch.bool)
    keep[1:] = s[1:] != s[:-1]
    return s[keep]


@torch.no_grad()
def pocket_clashes(xh, node_mask, linker_mask, pocket_only, is_geom, clash=None):
    """(B,N) int32 on the device (dl_clash_check, the check behind sample_chain(require_clash_free=True)): for each linker
    atom -- node_mask != 0, linker_mask != 0, pocket_only == 0 -- the number of pocket atoms (node_mask != 0, pocket_only !=
    0) it clashes with, and 0 on every other row. Two atoms clash when 100 |x_i - x_j| in pm is below clash[min type][max
    type] and that entry is >= 0; `clash` is a (T,T) table, by default clash_table(is_geom). `xh` is chain[0]-style
    (B,N,3+F) and the atom types are argmax of its first T feature columns, as in connected(). A NaN coordinate clashes with
    nothing. To vet inputs, pass the fragment rows as `linker_mask`."""
    return _clash_check(xh, node_mask, linker_mask, pocket_only, is_geom, clash, True)[1]


def clash_free(xh, node_mask, linker_mask, pocket_only, is_geom, clash=None):
    """(B,) bool on the device: whether no linker atom of a molecule clashes with a pocket atom (pocket_clashes); a molecule
    without linker or pocket atoms passes."""
    passed, _ = _clash_check(xh, node_mask, linker_mask, pocket_only, is_geom, clash, False)
    return (passed & _native.CHECK_CLASH) != 0


@torch.no_grad()
def clash_guide(xh, node_mask, linker_mask, pocket_only, is_geom, scale, clash=None):
    """One clash-guidance push (sample_chain(clash_guidance=...), dl_clash_guide) stated on the host in fp64: a copy of
    `xh` (B,N,3+F) in which every linker atom i -- the rows of pocket_clashes -- has moved to
        p_i + scale * sum_k max(0, r_ik - d_ik) (p_i - p_k) / d_ik,   d_ik = |p_i - p_k|,
    k over the pocket atoms, r_ik = clash[min type][max type] / 100 Angstrom (`clash` by default clash_table(is_geom); a
    negative entry exempts the pair), an atom's type the argmax of its first T feature columns. Every term comes from the
    input state; a pair at d_ik = 0 or with a NaN distance contributes nothing, and only linker coordinates change. With
    scale = 1 a linker atom in contact with one pocket atom lands at r_ik from it. The engine evaluates the same push in
    fp32 and leaves an atom with no contributing pair unwritten."""
    B, N = xh.shape[:2]
    T = len(GEOM_IDX2ATOM if is_geom else IDX2ATOM)
    table = (clash_table(is_geom) if clash is None else torch.as_tensor(clash, dtype=torch.float32)).double().cpu()
    if table.shape != (T, T):
        raise ValueError(f"clash is a ({T}, {T}) table, one row and column per atom type (got shape {tuple(table.shape)})")
    out = xh.detach().clone()
    x = xh[..., :3].detach().double().cpu()
    types = xh[..., 3:3 + T].detach().cpu().argmax(-1)
    live = node_mask.reshape(B, N).cpu() != 0
    pocket = live & (pocket_only.reshape(B, N).cpu() != 0)
    linker = live & ~pocket & (linker_mask.reshape(B, N).cpu() != 0)
    for b in range(B):
        li, pk = linker[b].nonzero().flatten(), pocket[b].nonzero().flatten()
        if len(li) == 0 or len(pk) == 0:
            continue
        diff = x[b][li][:, None, :] - x[b][pk][None, :, :]                 # (n_linker, n_pocket, 3): p_i - p_k
        d = diff.norm(dim=-1)
        ti, tk = types[b][li][:, None], types[b][pk][None, :]
        r = table[torch.minimum(ti, tk), torch.maximum(ti, tk)] / 100.0
        on = (r >= 0) & (d < r) & (d > 0)                                    # False for a NaN distance
        w = torch.where(on, (r - d) / torch.where(on, d, torch.ones_like(d)), torch.zeros_like(d))
        push = torch.where(on[..., None], w[..., None] * diff, torch.zeros_like(diff)).sum(1)
        out[b, li, :3] = (x[b, li] + float(scale) * push).to(out.dtype).to(out.device)
    return out


@torch.no_grad()
def _clash_check(xh, node_mask, linker_mask, pocket_only, is_geom, clash, want_counts):
    """dl_clash_check on a chain[0]-style batch: ((B,) int32 verdict bits, (B,N) int32 counts or None)."""
    dev = xh.device
    if dev.type != 'cuda':
        raise RuntimeError("the molecule checks run on the GPU (no CPU fallback); move the tensors to the device")
    B, N = xh.shape[:2]
    T = len(GEOM_IDX2ATOM if is_geom else IDX2ATOM)
    table = clash_table(is_geom) if clash is None else torch.as_tensor(clash, dtype=torch.float32)
    if table.shape != (T, T):
        raise ValueError(f"clash is a ({T}, {T}) table, one row and column per atom type (got shape {tuple(table.shape)})")
    table = table.to(dev).contiguous()
    xs = xh.float().contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    lm = linker_mask.reshape(B, N).float().contiguous()
    po = pocket_only.reshape(B, N, 1).float().contiguous()
    passed = torch.empty(B, dtype=torch.int32, device=dev)
    counts = torch.empty((B, N), dtype=torch.int32, device=dev) if want_counts else None
    lib = _native.load_library()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_clash_check(B, N, T, table.data_ptr(), xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                         lm.data_ptr(), po.data_ptr(), 1, passed.data_ptr(),
                                         None if counts is None else counts.data_ptr(), st), "dl_clash_check")
    return passed, counts


def ring_size_mask(sizes):
    """The uint64 ring-size mask of an iterable of ring sizes, as a Python int: bit k for each size k, an int in [3, 63],
    where 63 stands for every ring of 63 or more atoms (stated at DL_CHECK_RINGS in the header)."""
    mask = 0
    for k in sizes:
        if isinstance(k, bool):
            raise ValueError(f"ring sizes are ints in [3, 63] (got {k!r})")
        try:
            k = operator.index(k)
        except TypeError:
            raise ValueError(f"ring sizes are ints in [3, 63] (got {k!r})") from None
        if not 3 <= k <= 63:
            raise ValueError(f"ring sizes are ints in [3, 63], 63 meaning 63 or more atoms (got {k})")
        mask |= 1 << k
    return mask


def ring_sizes(xh, node_mask, linker_mask, is_geom, pocket_only=None):
    """(B,) int64 on the device, holding the uint64 bits of every molecule's ring-size mask (dl_ring_check, the check behind
    sample_chain(require_ring_sizes=True)): bit k is set iff some bond with a linker end -- a checked atom with linker_mask
    != 0 -- has a smallest ring of k atoms (3 <= k <= 62; bit 63: 63 or more). The checked atoms and bonds are those of
    connected(), over the whole molecule; rings of fragment atoms alone are not counted. These are rings of bond_orders'
    graph, not RDKit's SSSR, as stated at DL_CHECK_RINGS in the header."""
    return _ring_check(xh, node_mask, linker_mask, is_geom, pocket_only, 0)[1]


def ring_sizes_ok(xh, node_mask, linker_mask, is_geom, allowed, pocket_only=None):
    """(B,) bool on the device: whether every smallest ring of a molecule's linker bonds (ring_sizes) has a size in
    `allowed`, an iterable of ints in [3, 63], 63 meaning 63 or more atoms. A linker on no ring passes."""
    passed, _ = _ring_check(xh, node_mask, linker_mask, is_geom, pocket_only, ring_size_mask(allowed))
    return (passed & _native.CHECK_RINGS) != 0


@torch.no_grad()
def _ring_check(xh, node_mask, linker_mask, is_geom, pocket_only, allowed):
    """dl_ring_check on a chain[0]-style batch: ((B,) int32 verdict bits, (B,) int64 masks)."""
    dev = xh.device
    if dev.type != 'cuda':
        raise RuntimeError("the molecule checks run on the GPU (no CPU fallback); move the tensors to the device")
    B, N = xh.shape[:2]
    xs = xh.float().contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    lm = linker_mask.reshape(B, N).float().contiguous()
    po = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    thr1 = threshold_tables(is_geom)[0].to(dev).contiguous()
    passed = torch.empty(B, dtype=torch.int32, device=dev)
    masks = torch.empty(B, dtype=torch.int64, device=dev)
    lib = _native.load_library()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_ring_check(B, N, thr1.shape[0], thr1.data_ptr(), xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                        lm.data_ptr(), None if po is None else po.data_ptr(), 1, int(po is not None),
                                        allowed, passed.data_ptr(), masks.data_ptr(), st), "dl_ring_check")
    return passed, masks


def attachments(xh, node_mask, linker_mask, is_geom, pocket_only=None):
    """(B, N) int32 on the device (dl_anchor_check, the check behind sample_chain(require_anchors=True)): a_i, the number
    of bonds between fragment atom i -- a checked atom with linker_mask == 0 -- and the linker atoms (linker_mask != 0),
    and 0 on every other row. The checked atoms and bonds are those of connected(), over the whole molecule, so the bond
    predicate takes the same n. These are bond_orders' bonds, not OpenBabel's, as stated at DL_CHECK_ANCHORS in the header."""
    B, N = xh.shape[:2]
    anchors = torch.zeros((B, N), dtype=torch.int8, device=xh.device)
    return _anchor_check(xh, node_mask, linker_mask, anchors, is_geom, pocket_only, True)[1]


def anchors_ok(xh, node_mask, linker_mask, anchors, is_geom, pocket_only=None):
    """(B,) bool on the device: whether the linker attaches by exactly one bond at each anchor -- a fragment atom whose
    `anchors` flag, (B, N) or (B, N, 1), is non-zero -- and by none anywhere else on the fragments (attachments). Flags on
    linker rows, pocket rows and rows that are not checked are ignored; a molecule with no anchor passes."""
    passed, _ = _anchor_check(xh, node_mask, linker_mask, anchors, is_geom, pocket_only, False)
    return (passed & _native.CHECK_ANCHORS) != 0


@torch.no_grad()
def _anchor_check(xh, node_mask, linker_mask, anchors, is_geom, pocket_only, want_attachments):
    """dl_anchor_check on a chain[0]-style batch: ((B,) int32 verdict bits, (B, N) int32 attachments or None)."""
    dev = xh.device
    if dev.type != 'cuda':
        raise RuntimeError("the molecule checks run on the GPU (no CPU fallback); move the tensors to the device")
    B, N = xh.shape[:2]
    xs = xh.float().contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    lm = linker_mask.reshape(B, N).float().contiguous()
    an = (anchors.reshape(B, N) != 0).to(device=dev, dtype=torch.int8).contiguous()
    po = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    thr1 = threshold_tables(is_geom)[0].to(dev).contiguous()
    passed = torch.empty(B, dtype=torch.int32, device=dev)
    att = torch.empty((B, N), dtype=torch.int32, device=dev) if want_attachments else None
    lib = _native.load_library()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _native.check(lib.dl_anchor_check(B, N, thr1.shape[0], thr1.data_ptr(), xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                          lm.data_ptr(), an.data_ptr(), None if po is None else po.data_ptr(), 1,
                                          int(po is not None), passed.data_ptr(), None if att is None else att.data_ptr(),
                                          st), "dl_anchor_check")
    return passed, att


def build_xae_molecule(positions, atom_types, is_geom, margins=MARGINS_EDM):
    """Reference signature (molecule_builder.py:44): one molecule, positions (n,3) already masked, atom_types (n,).
    Returns (X, A, E) with A bool, E int32, lower-triangular ("the graph should be DIRECTED")."""
    n = positions.shape[0]
    T = len(GEOM_IDX2ATOM if is_geom else IDX2ATOM)
    one_hot = torch.nn.functional.one_hot(atom_types.long(), T).unsqueeze(0)
    E = bond_orders(one_hot.to(positions.device), positions.unsqueeze(0), torch.ones((1, n), device=positions.device),
                    is_geom, margins)[0].to(torch.int)
    return atom_types, E != 0, E
