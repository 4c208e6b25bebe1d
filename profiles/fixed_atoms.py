"""Fixed atoms in the reverse loop: what `sample_chain(..., fixed_atoms=M)` costs.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number, and the median
edm.last_loop_ms (CUDA events around the device loop) of --runs seeded calls, after one warm-up call of each setup, for
  * the plain call (no mask);
  * an all-zero mask, which the host turns into the plain call;
  * half of each molecule's linker rows kept (the first half, rounded down),
alternating the three setups, on the ZINC config (cfg2_zinc: B=256, N=40, L=6, T=500) and on the pocket config
(cfg4_pockets: B=64, N=300, FC-10A-4A, T=1000). Synthetic weights: sample quality is not measured. It needs a GPU.

    python profiles/fixed_atoms.py [--runs 3]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from difflinker_b200 import synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from profiles.clash_resampling import model
from profiles.connected_resampling import card


def half_mask(kw):
    lm = kw['linker_mask'].reshape(kw['x'].shape[:2]) != 0
    rank = lm.long().cumsum(1)
    return (lm & (rank <= lm.sum(1, keepdim=True) // 2)).to(torch.int8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fixed_atoms.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    for name in ("cfg2_zinc", "cfg4_pockets"):
        spec = synthetic.SPECS[name]
        ddpm, _ = model(spec, spec.T, dev)
        data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
        kw = sampler_inputs(ddpm, data, keep_linker=True)              # the batch's own linker rows, which the mask keeps
        edm = ddpm.edm
        B, N = kw['x'].shape[:2]
        half = half_mask(kw)
        setups = {"plain": None, "all-zero mask": torch.zeros_like(half), "half kept": half}
        print(f"workload {name}: B={B} N={N} L={spec.L} graph {spec.graph_type}, T={edm.T}, "
              f"{int(half.sum())} of {int(kw['linker_mask'].sum())} linker rows kept in 'half kept'")
        seeds = list(range(1000, 1000 + B))
        for m in setups.values():                                       # warm-up of every setup
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds, fixed_atoms=m)
        loops = {s: [] for s in setups}
        for _ in range(args.runs):
            for s, m in setups.items():
                edm.sample_chain(**kw, keep_frames=1, seeds=seeds, fixed_atoms=m)
                torch.cuda.synchronize()
                loops[s].append(edm.last_loop_ms)
        base = sorted(loops["plain"])[len(loops["plain"]) // 2]
        for s, v in loops.items():
            med = sorted(v)[len(v) // 2]
            print(f"  {s:14s}: device loop {med:10.2f} ms median ({med / base - 1:+.2%} vs plain; runs "
                  f"{', '.join(f'{x:.2f}' for x in v)}) [{where}]")


if __name__ == "__main__":
    main()
