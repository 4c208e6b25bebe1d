"""Input contract of the hot path: padded batches and linker templates (src/datasets.py:332-375, 476-512;
src/const.py:6-7, 39-47).  Pure host-side torch; reproduces the reference's dtypes bit-exactly, including the
int8 edge mask whose live values are -1 (off-diagonal) and -2 (self loops) because the reference applies a
*bitwise* NOT to an int8 identity."""
import torch

TORCH_FLOAT = torch.float32
TORCH_INT = torch.int8

DATA_LIST_ATTRS = {"uuid", "name", "fragments_smi", "linker_smi", "num_atoms"}
DATA_ATTRS_TO_PAD = {"positions", "one_hot", "charges", "anchors", "fragment_mask", "linker_mask", "pocket_mask",
                     "fragment_only_mask"}
DATA_ATTRS_TO_ADD_LAST_DIM = {"charges", "anchors", "fragment_mask", "linker_mask", "pocket_mask",
                              "fragment_only_mask"}


def _stack_and_pad(batch):
    out = {}
    for item in batch:
        for key, value in item.items():
            out.setdefault(key, []).append(value)
    for key in list(out):
        if key in DATA_LIST_ATTRS:
            continue
        if key not in DATA_ATTRS_TO_PAD:
            raise Exception(f"Unknown batch key: {key}")
        out[key] = torch.nn.utils.rnn.pad_sequence(out[key], batch_first=True, padding_value=0)
    return out


def _add_masks(out, pocket):
    """atom_mask, edge_mask and the trailing singleton dims (datasets.py:353-375)."""
    atom_mask = (out["fragment_mask"].bool() | out["linker_mask"].bool()).to(TORCH_INT)
    out["atom_mask"] = atom_mask[:, :, None]
    bs, n = atom_mask.shape
    if pocket:
        # pocket models: `edge_mask` carries the molecule index of every node (int8!) instead of a mask
        out["edge_mask"] = torch.arange(bs, dtype=torch.int64, device=atom_mask.device).repeat_interleave(n).to(TORCH_INT)
    else:
        pair = atom_mask[:, None, :] * atom_mask[:, :, None]
        pair = pair * (~torch.eye(n, dtype=TORCH_INT, device=atom_mask.device)).unsqueeze(0)
        out["edge_mask"] = pair.view(bs * n * n, 1)
    for key in DATA_ATTRS_TO_ADD_LAST_DIM:
        if key in out:
            out[key] = out[key][:, :, None]
    return out


def collate(batch):
    return _add_masks(_stack_and_pad(batch), "pocket_mask" in batch[0])


def create_templates_for_linker_generation(data, linker_sizes, n_nodes=None):
    """Keep the fragment rows of every padded attribute and append `linker_size` template rows (ones for linker_mask,
    zeros elsewhere), then re-collate (datasets.py:483-512). Batched: the reference decouples the batch into one dict per
    molecule and collates again (a few thousand tiny ops per call on the GPU); the same tensors come out of a handful of
    masked selects on the padded batch -- one host sync for the new padded length. `n_nodes` pads the template to that
    many rows instead of the largest molecule's (it must not be smaller)."""
    fm = data["fragment_mask"]
    dev = fm.device
    bs, n_old = fm.shape[0], fm.shape[1]
    n_frag = fm.reshape(bs, n_old).sum(1).long()                       # fragment atoms come first (datasets.py:493-494)
    sizes = torch.as_tensor(linker_sizes, device=dev).reshape(-1).long()
    n_tot = n_frag + sizes
    n_new = int(n_tot.max())
    if n_nodes is not None:
        if n_nodes < n_new:
            raise ValueError(f"n_nodes = {n_nodes} is fewer rows than the largest template's {n_new}")
        n_new = n_nodes
    idx = torch.arange(n_new, device=dev)[None, :]
    is_frag = (idx < n_frag[:, None])[:, :, None]
    is_link = ((idx >= n_frag[:, None]) & (idx < n_tot[:, None]))[:, :, None]
    out = {}
    for key, value in data.items():
        if key == "num_atoms":
            out[key] = n_tot.tolist()
        elif key in DATA_LIST_ATTRS:
            out[key] = list(value)
        elif key in DATA_ATTRS_TO_PAD:
            v = value if value.dim() == 3 else value[:, :, None]
            if n_new <= n_old:
                v = v[:, :n_new]
            else:
                v = torch.cat([v, torch.zeros((bs, n_new - n_old, v.shape[2]), dtype=v.dtype, device=dev)], dim=1)
            v = torch.where(is_frag, v, torch.zeros((), dtype=v.dtype, device=dev))
            if key == "linker_mask":
                v = torch.where(is_link, torch.ones((), dtype=v.dtype, device=dev), v)
            out[key] = v.squeeze(-1) if key in DATA_ATTRS_TO_ADD_LAST_DIM else v
    return _add_masks(out, "pocket_mask" in data)


def _create_templates_per_molecule(data, linker_sizes):
    """The reference's own formulation (decouple -> per-molecule template -> collate); kept as the cross-check of the batched
    version above (tests/test_host_logic.py)."""
    singles = []
    for i, linker_size in enumerate(linker_sizes):
        linker_size = int(linker_size)
        n_frag = int(data["fragment_mask"][i].squeeze().sum())
        item = {}
        for key, value in data.items():
            if key == "num_atoms":
                item[key] = n_frag + linker_size
            elif key in DATA_LIST_ATTRS:
                item[key] = value[i]
            elif key in DATA_ATTRS_TO_PAD:
                head = value[i][:n_frag]
                tail = torch.full((linker_size, head.shape[1]), 1 if key == "linker_mask" else 0, dtype=head.dtype,
                                  device=head.device)
                rows = torch.cat([head, tail], dim=0)
                item[key] = rows.squeeze(-1) if key in DATA_ATTRS_TO_ADD_LAST_DIM else rows
        singles.append(item)
    return collate(singles)
