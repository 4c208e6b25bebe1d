"""Linker sizes drawn from each molecule's seed (`ddpm.sample_chain(data, linker_sizes=size_nn, seeds=...)`): what the draw
and the capacity padding cost.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * dl_size_draw alone at B = 256 and 4096 over the ZINC (10 sizes) and GEOM (33 sizes) tables: CUDA events around
    --launches back-to-back launches after a warm-up, per launch;
  * the seeded reverse loop (edm.last_loop_ms, median of --reps calls) of cfg2_zinc (B=256, T=--T) and cfg3_geom on the
    template the reference builds -- padded to max_b(n_frag + size_b) -- against the same sizes padded to the capacity
    N_cap = max n_frag + max(sizes) that linker_sizes uses, so a redrawn size always fits;
  * one recovery round of the same rows, every row resampled (require_connected with random weights connects no row), with
    size redraws (linker_sizes) against one with the first sizes kept (sample_fn): dl_last_retry_ms, the device time of
    the round from its row gather to its row scatter.
The size model is a SizeClassifier with random weights over the table; the sizes drawn are printed with the numbers.
It needs a GPU.

    python profiles/seeded_linker_sizes.py [--T 500] [--launches 200] [--reps 3]
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, synthetic
from difflinker_b200.linker_size import (GEOM_TRAIN_LINKER_ID2SIZE, ZINC_TRAIN_LINKER_ID2SIZE, SizeClassifier,
                                         collate_with_fragment_edges, draw_sizes)
from profiles.connected_resampling import card


def draw_us(B, table, launches, dev):
    g = torch.Generator().manual_seed(1)
    logits = torch.randn((B, len(table)), generator=g).to(dev)
    seeds = list(range(B))
    draw_sizes(logits, table, seeds)
    lib = _native.load_library()
    tab = torch.tensor(table, dtype=torch.int32, device=dev)
    sd = torch.arange(B, dtype=torch.int64, device=dev)
    out = torch.empty(B, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream()
    launch = lambda: _native.check(lib.dl_size_draw(B, len(table), logits.data_ptr(), len(table), tab.data_ptr(),
                                                    sd.data_ptr(), 0, out.data_ptr(), st.cuda_stream), "dl_size_draw")
    for _ in range(10):
        launch()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(st)
    for _ in range(launches):
        launch()
    ev1.record(st)
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches


def model(spec, T, dev, table):
    hp = synthetic.model_hparams(spec)
    hp['diffusion_steps'] = T
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=1.0)
    ddpm = ddpm.to(dev)
    data = {k: (v.to(dev) if torch.is_tensor(v) else v)
            for k, v in collate_with_fragment_edges(synthetic.make_items(spec)).items()}
    nn = SizeClassifier(in_node_nf=spec.F, out_node_nf=len(table), linker_id2size=table,
                        linker_size2id={s: i for i, s in enumerate(table)}).eval().to(dev)
    return ddpm, data, nn


def loop_ms(ddpm, data, reps, **kw):
    out = []
    for _ in range(reps):
        chain, _ = ddpm.sample_chain(data, keep_frames=1, **kw)
        torch.cuda.synchronize()
        out.append(ddpm.edm.last_loop_ms)
    return statistics.median(out), chain.shape[2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=500)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    where = card()
    lib = _native.load_library()
    for name, table in (("ZINC", ZINC_TRAIN_LINKER_ID2SIZE), ("GEOM", GEOM_TRAIN_LINKER_ID2SIZE)):
        for B in (256, 4096):
            print(f"dl_size_draw {name} (C={len(table)}) B={B}: {draw_us(B, table, args.launches, dev):7.2f} us/launch [{where}]")
    for spec_name, table in (("cfg2_zinc", ZINC_TRAIN_LINKER_ID2SIZE), ("cfg3_geom", GEOM_TRAIN_LINKER_ID2SIZE)):
        spec = synthetic.SPECS[spec_name]
        ddpm, data, nn = model(spec, args.T, dev, table)
        B = data['positions'].shape[0]
        seeds = list(range(1000, 1000 + B))
        sizes = draw_sizes(nn.size_logits(data), table, seeds)
        fixed = lambda d, s=sizes: s
        ms_ref, n_ref = loop_ms(ddpm, data, args.reps, sample_fn=fixed, seeds=seeds)
        ms_cap, n_cap = loop_ms(ddpm, data, args.reps, linker_sizes=nn, seeds=seeds)
        print(f"{spec_name} B={B} T={args.T}: seeded loop at the reference's template N={n_ref} {ms_ref:9.2f} ms, at "
              f"N_cap={n_cap} {ms_cap:9.2f} ms ({100 * (ms_cap / ms_ref - 1):+.1f}%); sizes drawn "
              f"{sorted(set(sizes.tolist()))} [{where}]")
        eng = ddpm.edm.dynamics.engine(0)
        rounds = {}
        for label, kw in (("redraw", dict(linker_sizes=nn)), ("fixed", dict(sample_fn=fixed))):
            ddpm.sample_chain(data, keep_frames=1, seeds=seeds, nan_retries=1, require_connected=True, **kw)
            rounds[label] = (float(lib.dl_last_retry_ms(eng)), int((ddpm.edm.last_attempts == 1).sum()))
        print(f"{spec_name}: one round of {rounds['redraw'][1]} rows with size redraws {rounds['redraw'][0]:9.2f} ms; "
              f"of {rounds['fixed'][1]} rows at the first sizes {rounds['fixed'][0]:9.2f} ms [{where}]")


if __name__ == "__main__":
    main()
