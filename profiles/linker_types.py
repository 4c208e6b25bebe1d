"""Linker types in the reverse loop: what `sample_chain(..., linker_types=M)` costs.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number, and the median
edm.last_loop_ms (CUDA events around the device loop) of --runs seeded calls, after one warm-up call of each setup, for
  * the plain call (no set);
  * a set that allows every type, which the host turns into the plain call;
  * {C, N, O}, which runs the projecting k_finish instantiation,
alternating the three setups, on the ZINC config (cfg2_zinc: B=256, N=40, L=6, T=500) and on the pocket config
(cfg4_pockets: B=64, N=300, FC-10A-4A, T=1000). It also prints the share of linker atoms of chain[0] that {C, N, O}
allows in each setup. Synthetic weights: sample quality is not measured. It needs a GPU.

    python profiles/linker_types.py [--runs 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import linker_types_mask, sampler_inputs
from profiles.clash_resampling import model
from profiles.connected_resampling import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("linker_types.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    for name in ("cfg2_zinc", "cfg4_pockets"):
        spec = synthetic.SPECS[name]
        ddpm, _ = model(spec, spec.T, dev)
        ddpm.edm.is_geom = False
        data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
        kw = sampler_inputs(ddpm, data)
        edm = ddpm.edm
        B, N = kw['x'].shape[:2]
        cno = linker_types_mask(edm, ['C', 'N', 'O'])
        setups = {"plain": None, "all allowed": torch.ones(edm.in_node_nf, dtype=torch.bool), "{C, N, O}": cno}
        print(f"workload {name}: B={B} N={N} L={spec.L} graph {spec.graph_type}, T={edm.T}, F={edm.in_node_nf}")
        seeds = list(range(1000, 1000 + B))
        lm = (kw['linker_mask'].reshape(B, N) != 0) & (kw['node_mask'].reshape(B, N) != 0)
        share = {}
        for s, m in setups.items():                                     # warm-up of every setup
            chain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=m)
            types = chain[0][..., 3:].argmax(-1)[lm]
            share[s] = cno.to(dev)[types].float().mean().item()
        loops = {s: [] for s in setups}
        for _ in range(args.runs):
            for s, m in setups.items():
                edm.sample_chain(**kw, keep_frames=1, seeds=seeds, linker_types=m)
                torch.cuda.synchronize()
                loops[s].append(edm.last_loop_ms)
        base = sorted(loops["plain"])[len(loops["plain"]) // 2]
        for s, v in loops.items():
            med = sorted(v)[len(v) // 2]
            print(f"  {s:12s}: device loop {med:10.2f} ms median ({med / base - 1:+.2%} vs plain; runs "
                  f"{', '.join(f'{x:.2f}' for x in v)}); linker atoms in C, N, O {share[s]:.1%} [{where}]")


if __name__ == "__main__":
    main()
