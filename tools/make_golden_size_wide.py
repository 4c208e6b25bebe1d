"""TEST INFRASTRUCTURE ONLY -- golden vectors for the 256-wide linker-size classifier (the reference README's recipe,
`train_size_gnn.py --hidden_nf 256 --n_layers 5 --normalization batch_norm`), from the LIVE, UNMODIFIED reference (build
container only, like oracle/make_golden.py), written as NEW files tests/golden/size_gnn_*_h256.npz.

The generator lives outside oracle/, whose files pin the existing fixtures and stay as they are. Like the existing size
fixtures it stores the reference's logits, the spec, the seed and the sha256 of the reference state_dict, not the weights:
the inputs come back from synthetic.size_gnn_items and the weights from the seed and synthetic.init_size_gnn_like_trained.
For every fixture the host SizeClassifier is checked to build the reference's parameters (keys, shapes, values) from the
same seed, and oracle.size_classifier_forward to reproduce the reference's logits.
Run:  python tools/make_golden_size_wide.py [fixture ...]
"""
import importlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from difflinker_b200 import linker_size as mine, synthetic  # noqa: E402
from oracle import difflinker_oracle as orc, make_golden as mg  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402

WIDTH = 256
# name: (spec, batch, normalization, seed, n_layers, table ('zinc' | 'geom'), in_node_nf (None: the spec's F), pocket)
FIXTURES = {
    "size_gnn_zinc_h256": ("cfg2_zinc_ragged", 6, "batch_norm", 31, 5, "zinc", None, False),
    "size_gnn_pocket_geom_h256": ("size_pocket_geom", 3, "batch_norm", 32, 3, "geom", 9, True),
    "size_gnn_geom_h256": ("size_geom", 5, None, 33, 2, "geom", None, False),
}


def spec_of(name):
    return synthetic.SPECS.get(name) or synthetic.SIZE_GNN_SPECS[name]


def golden_size_wide(ns, name, spec_name, nb, normalization, seed, n_layers, table, in_nf, pocket):
    lsl = importlib.import_module("src.linker_size_lightning")
    id2size, size2id = (ns.const.ZINC_TRAIN_LINKER_ID2SIZE, ns.const.ZINC_TRAIN_LINKER_SIZE2ID) if table == "zinc" else \
        (ns.const.GEOM_TRAIN_LINKER_ID2SIZE, ns.const.GEOM_TRAIN_LINKER_SIZE2ID)
    spec = spec_of(spec_name)
    in_nf = in_nf or spec.F
    out_nf = len(id2size)
    torch.manual_seed(seed)
    ref = lsl.SizeClassifier(None, None, None, in_node_nf=in_nf, hidden_nf=WIDTH, out_node_nf=out_nf, n_layers=n_layers,
                             batch_size=nb, lr=1e-3, torch_device='cpu', normalization=normalization,
                             linker_size2id=size2id, linker_id2size=id2size)
    torch.manual_seed(seed)
    host = mine.SizeClassifier(in_node_nf=in_nf, hidden_nf=WIDTH, out_node_nf=out_nf, n_layers=n_layers,
                               normalization=normalization, linker_size2id=size2id, linker_id2size=id2size)
    assert list(ref.state_dict().keys()) == list(host.state_dict().keys()), name
    for k, v in ref.state_dict().items():
        assert v.shape == host.state_dict()[k].shape and torch.equal(v, host.state_dict()[k]), (name, k)
    synthetic.init_size_gnn_like_trained(ref, seed)
    ref.eval()
    items = synthetic.size_gnn_items(spec, nb)
    data = ns.datasets.collate_with_fragment_edges(items)
    mydata = mine.collate_with_fragment_edges(items)
    assert torch.equal(data['edge_mask'], mydata['edge_mask']), name
    if pocket:
        fo = data['fragment_only_mask'][..., 0]
        assert data['one_hot'].shape[-1] == in_nf + 1 and (data['one_hot'][..., -1] * fo == 0).all()
        live = (data['edge_mask'].view(nb, spec.N, spec.N) != 0).sum(-1)
        assert int(live.max()) > 128, name
    with torch.no_grad():
        out, _ = ref.forward(data, return_loss=False, with_pocket=pocket, adjust_shape=pocket)
        ora = orc.size_classifier_forward(ref.state_dict(), data, in_nf, n_layers, normalization, with_pocket=pocket,
                                          adjust_shape=pocket)
    err = (out - ora).abs().max().item()
    print(f"  {name}: oracle vs reference max|d| = {err:.2e} (max |logit| {out.abs().max().item():.3e})")
    assert err <= 1e-6 * max(1.0, out.abs().max().item()), f"{name}: oracle vs reference {err}"
    mg.save(name, dict(kind="size_gnn", spec=spec.name, batch=nb, seed=seed, normalization=normalization, out_nf=out_nf,
                       n_layers=n_layers, in_node_nf=in_nf, hidden_nf=WIDTH, with_pocket=pocket, adjust_shape=pocket,
                       sha=mg.state_sha(ref.state_dict()), oracle_max_abs_err=err), logits=out)


def main():
    torch.set_num_threads(8)
    ns = load_reference()
    only = set(sys.argv[1:])
    for name, args in FIXTURES.items():
        if not only or name in only:
            golden_size_wide(ns, name, *args)


if __name__ == "__main__":
    main()
