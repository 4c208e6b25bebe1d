"""ODE solvers in the reverse loop: what `sample_chain(..., solver='ddim' | 'dpmpp_2m')` costs per step, and the throughput
of a loop shortened to K steps against the ancestral loop at the trained T.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the device loop per step (edm.last_loop_ms / (T + 1)) of 'ancestral', 'ddim' and 'dpmpp_2m' at the same T (--T-equal),
    alternating the three over --runs runs;
  * molecules/s -- B over the host wall time of one sample_chain call that ends in a device synchronise, with the device
    loop's share beside it -- of 'ddim' and 'dpmpp_2m' at K in {20, 50, 100} and of 'ancestral' at the trained T, on the
    ZINC config (cfg2_zinc: B=256, N=40, L=6, T=500) and on the pocket config (cfg4_pockets: B=64, N=300, FC-10A-4A,
    T=1000), best of --runs alternated runs.
Synthetic weights only: whether K solver steps match the ancestral sampler's sample quality on a trained checkpoint is not
measured here. It needs a GPU.

    python profiles/ode_solvers.py [--runs 3] [--T-equal 100]
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from difflinker_b200 import synthetic
from profiles.clash_resampling import model
from profiles.connected_resampling import card

SOLVERS = ("ancestral", "ddim", "dpmpp_2m")


def timed_call(edm, kw, solver):
    """(wall ms, device loop ms) of one sampler call from the batch stream."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    edm.sample_chain(**kw, keep_frames=1, solver=solver)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), edm.last_loop_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--T-equal", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ode_solvers.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    for name in ("cfg2_zinc", "cfg4_pockets"):
        spec = synthetic.SPECS[name]
        ddpm, kw = model(spec, spec.T, dev)
        edm = ddpm.edm
        B, N = kw['x'].shape[:2]
        print(f"workload {name}: B={B} N={N} L={spec.L} graph {spec.graph_type}, trained T={spec.T}")
        edm.T = args.T_equal
        for s in SOLVERS:                                                # warm-up of every setting
            timed_call(edm, kw, s)
        per_step = {s: [] for s in SOLVERS}
        for _ in range(args.runs):
            for s in SOLVERS:
                per_step[s].append(timed_call(edm, kw, s)[1] / (edm.T + 1))
        for s in SOLVERS:
            v = sorted(per_step[s])
            print(f"  T={edm.T} {s:9s}: device loop per step {v[len(v) // 2] * 1e3:8.1f} us (median; runs "
                  f"{', '.join(f'{x * 1e3:.1f}' for x in per_step[s])}) [{where}]")
        settings = [("ancestral", spec.T)] + [(s, K) for K in (20, 50, 100) for s in ("ddim", "dpmpp_2m")]
        best = {}
        for _ in range(args.runs):
            for s, K in settings:
                edm.T = K
                if (s, K) not in best:
                    timed_call(edm, kw, s)                               # warm-up at this T
                wall, loop = timed_call(edm, kw, s)
                if (s, K) not in best or wall < best[(s, K)][0]:
                    best[(s, K)] = (wall, loop)
        base = B / (best[("ancestral", spec.T)][0] / 1e3)
        for s, K in settings:
            wall, loop = best[(s, K)]
            rate = B / (wall / 1e3)
            print(f"  {s:9s} K={K:5d}: {rate:9.1f} molecules/s ({rate / base:6.1f}x ancestral at T={spec.T}); call "
                  f"{wall:9.2f} ms, device loop {loop:9.2f} ms [{where}]")
        edm.T = spec.T


if __name__ == "__main__":
    main()
