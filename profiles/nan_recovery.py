"""NaN recovery: the device time of one recovery round of dl_sample_chain_retry against a full-batch resample.

Samples a workload (synthetic weights, seeds 0..B-1, keep_frames=1) with `nan_retries=1` while k molecules carry a NaN
fragment coordinate, so exactly those k fail the first loop and are resampled as one sub-batch of k (they fail again: the
round still runs all T+1 steps, so its time is that of a real round). Per run it prints the device time of the first loop
over the whole batch (edm.last_loop_ms -- what resampling the whole batch costs, as the reference's callers do) and of the
round (dl_last_retry_ms: row gather, the wait for the host to capture the sub-batch's step graph, the sub-batch loop, row
scatter), for k = 1, 4 and 16, and the card's name, power limit and maximum SM clock. For a handful of rows a round runs
the same ~39 kernels per step on a tiny grid, so it should be bound by graph-launch latency rather than by arithmetic.

    python profiles/nan_recovery.py [--workload cfg2_zinc] [--workload cfg4_pockets] [--T 500] [--reps 3]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from difflinker_b200.utils import FoundNaNException


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def profile(spec, T, reps, dev, counts=(1, 4, 16)):
    hp = synthetic.model_hparams(spec)
    if T is not None:
        hp['diffusion_steps'] = T
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=100.0 if spec.N <= 64 else 1.0)
    ddpm = ddpm.to(dev)
    edm = ddpm.edm
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    seeds = list(range(B))
    lib = _native.load_library()
    print(f"workload {spec.name}: B={B} N={N} L={spec.L} T={edm.T} F={spec.F} graph {spec.graph_type}, keep_frames=1")

    def run(k):
        x = kw['x'].clone()
        rows = torch.linspace(0, B - 1, k).round().long().tolist()       # spread over the batch
        x[rows, 0, 0] = float('nan')
        try:
            edm.sample_chain(**dict(kw, x=x), keep_frames=1, seeds=seeds, nan_retries=1)
            raise RuntimeError("the NaN molecules did not fail")
        except FoundNaNException as e:
            assert set(rows) <= set(e.x_h_nan_idx | e.only_x_nan_idx | e.only_h_nan_idx)
        resampled = int((edm.last_attempts > 0).sum())                 # k, unless a healthy molecule diverged as well
        return edm.last_loop_ms, float(lib.dl_last_retry_ms(edm.dynamics.engine(dev.index or 0))), resampled

    for k in counts:                                                   # warm-up: workspaces, graph capture
        run(k)
    res = {k: [] for k in counts}
    for _ in range(reps):
        for k in counts:
            full, rnd, resampled = run(k)
            res[k].append((full, rnd))
            print(f"  k={k:3d}  full-batch loop {full:9.2f} ms  recovery round of {resampled} molecules {rnd:8.2f} ms "
                  f"({1e3 * rnd / (edm.T + 1):6.1f} us per step)")
    for k, rows in res.items():
        fulls, rnds = zip(*rows)
        print(f"  k={k:3d}: round {min(rnds):.2f}-{max(rnds):.2f} ms, full-batch resample {min(fulls):.2f}-{max(fulls):.2f} ms, "
              f"round / full {min(rnds) / min(fulls):.3f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", action="append", default=None)
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nan_recovery.py needs a GPU")
    dev = torch.device("cuda", 0)
    print(f"card: {card()}")
    for name in args.workload or ["cfg2_zinc", "cfg4_pockets"]:
        profile(synthetic.SPECS[name], args.T, args.reps, dev)


if __name__ == "__main__":
    main()
