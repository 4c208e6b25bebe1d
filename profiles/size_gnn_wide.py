"""The linker-size classifier at hidden_nf 128 and 256: what the 256-wide model of the README's recipe costs next to the
sampling it sizes.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * dl_sizegnn_forward alone at widths 128 and 256 (5 layers, batch norm folded), at the cfg2_zinc shape (B=256, N=40,
    fragment edges) and the pocket shape of cfg4_pockets (B=64, N=300, with_pocket: the fragment-only atoms): CUDA events
    around --launches back-to-back calls after a warm-up, per call;
  * beside them the seeded reverse loop at the same shape (edm.last_loop_ms, median of --reps calls of
    `ddpm.sample_chain(data, linker_sizes=<256-wide model>, seeds=...)`, T = --T), whose sizes that model draws.
The size models are SizeClassifiers with trained-like random weights (synthetic.init_size_gnn_like_trained). It needs a GPU.

    python profiles/size_gnn_wide.py [--T 500] [--launches 100] [--reps 3]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, synthetic
from difflinker_b200.linker_size import (GEOM_TRAIN_LINKER_ID2SIZE, GEOM_TRAIN_LINKER_SIZE2ID, ZINC_TRAIN_LINKER_ID2SIZE,
                                         ZINC_TRAIN_LINKER_SIZE2ID, SizeClassifier, collate_with_fragment_edges)
from profiles.connected_resampling import card

SHAPES = {   # name: (spec, size table, pocket)
    "cfg2_zinc": ("cfg2_zinc", (ZINC_TRAIN_LINKER_ID2SIZE, ZINC_TRAIN_LINKER_SIZE2ID), False),
    "cfg4_pockets": ("cfg4_pockets", (GEOM_TRAIN_LINKER_ID2SIZE, GEOM_TRAIN_LINKER_SIZE2ID), True),
}


def size_model(width, F, tables, dev):
    torch.manual_seed(5)
    nn = SizeClassifier(in_node_nf=F, hidden_nf=width, out_node_nf=len(tables[0]), n_layers=5,
                        normalization='batch_norm', linker_id2size=tables[0], linker_size2id=tables[1])
    synthetic.init_size_gnn_like_trained(nn, 5)
    return nn.eval().to(dev)


def forward_us(nn, data, pocket, launches):
    """Per-call device time of dl_sizegnn_forward, as SizeGNN.logits launches it."""
    fm = data['fragment_only_mask'] if pocket else data['fragment_mask']
    B, N = data['positions'].shape[:2]
    g = nn.gnn
    dev = data['positions'].device
    xh = torch.cat([data['positions'].float(), data['one_hot'].float()], dim=2).contiguous()
    fm8 = (fm.reshape(B, N) != 0).to(torch.int8).contiguous()
    em = (data['edge_mask'].reshape(B, N, N) != 0).to(torch.int8).contiguous()
    out = torch.empty((B, g.out_node_nf), device=dev)
    lib = _native.load_library()
    eng = g.engine(dev.index or 0)
    st = torch.cuda.current_stream()
    launch = lambda: _native.check(lib.dl_sizegnn_forward(eng, B, N, xh.data_ptr(), fm8.data_ptr(), em.data_ptr(),
                                                          out.data_ptr(), st.cuda_stream), "dl_sizegnn_forward")
    for _ in range(10):
        launch()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(st)
    for _ in range(launches):
        launch()
    ev1.record(st)
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches


def loop_ms(spec, T, data, nn, reps, dev):
    hp = synthetic.model_hparams(spec)
    hp['diffusion_steps'] = T
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=1.0)
    ddpm = ddpm.to(dev)
    B = data['positions'].shape[0]
    seeds = list(range(1000, 1000 + B))
    out = []
    for _ in range(reps + 1):                     # the first call builds the engine and the plan: not timed
        ddpm.sample_chain(data, keep_frames=1, linker_sizes=nn, seeds=seeds)
        torch.cuda.synchronize()
        out.append(ddpm.edm.last_loop_ms)
    return statistics.median(out[1:]), sorted(set(ddpm.edm.last_sizes.tolist()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=500)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    where = card()
    for name, (spec_name, tables, pocket) in SHAPES.items():
        spec = synthetic.SPECS[spec_name]
        data = {k: (v.to(dev) if torch.is_tensor(v) else v)
                for k, v in collate_with_fragment_edges(synthetic.make_items(spec)).items()}
        B, N = data['positions'].shape[:2]
        F = data['one_hot'].shape[-1]
        us = {w: forward_us(size_model(w, F, tables, dev), data, pocket, args.launches) for w in (128, 256)}
        ms, sizes = loop_ms(spec, args.T, data, size_model(256, F, tables, dev), args.reps, dev)
        print(f"{name} B={B} N={N}: dl_sizegnn_forward (5 layers) width 128 {us[128]:9.1f} us, width 256 {us[256]:9.1f} us "
              f"({us[256] / us[128]:.2f}x); seeded reverse loop T={args.T} {ms:9.2f} ms (forward at 256 = "
              f"{100 * us[256] / (1e3 * ms):.2f}% of it); sizes drawn {sizes} [{where}]")


if __name__ == "__main__":
    main()
