"""Partial diffusion: the device loop of `EDM.sample_chain(start_step=t0)` against the plain sampler, at the benchmarked shape.

The workload is cfg2_zinc (B=256, N=40, 8 linker atoms, L=6, synthetic weights) at T=500 and keep_frames=1, with the batch's
own linker kept in the template (DDPM.sample_chain with start_step). Runs are alternated -- the plain sampler, then every t0
in turn -- for --reps rounds after one warm-up round, on the default edge path and the device-side batch stream. Per run it
prints the device loop time (edm.last_loop_ms: CUDA events around the graph replays) and the molecules/s of the call's wall
time (host clock around a synchronised call); then per t0 the median loop time, its ratio to the plain sampler's and the
expected ratio (t0 + 1) / (T + 1); then the card's name and power limit, read in the same run.

    python profiles/partial_diffusion.py [--t0 50 125 250 500] [--reps 3]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, synthetic
from difflinker_b200.batching import collate


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--t0", type=int, nargs="+", default=[50, 125, 250, 500])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("partial_diffusion.py needs a GPU")
    dev = torch.device("cuda", 0)
    spec = synthetic.SPECS["cfg2_zinc"]
    hp = synthetic.model_hparams(spec)
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm)
    ddpm = ddpm.to(dev)
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    B, T = data['positions'].shape[0], ddpm.edm.T
    print(f"cfg2_zinc B={B} N={data['positions'].shape[1]} L={hp['n_layers']} T={T}, keep_frames=1, default edge path")
    runs = [None] + list(args.t0)
    loops = {t0: [] for t0 in runs}

    def one(t0, record):
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        ddpm.sample_chain(data, keep_frames=1, start_step=t0)
        torch.cuda.synchronize()
        wall = time.perf_counter() - w0
        if record:
            loops[t0].append(ddpm.edm.last_loop_ms)
            label = "plain" if t0 is None else f"t0={t0}"
            print(f"  {label:8s} loop {ddpm.edm.last_loop_ms:9.2f} ms  wall {wall * 1e3:9.1f} ms  {B / wall:8.1f} molecules/s")
    for t0 in runs:                                         # warm-up: workspace, graph capture, module loads
        one(t0, False)
    for _ in range(args.reps):
        for t0 in runs:
            one(t0, True)
    plain = statistics.median(loops[None])
    print(f"plain sampler: median loop {plain:.2f} ms, {B / (plain / 1e3):.1f} molecules/s (loop only)")
    for t0 in args.t0:
        m = statistics.median(loops[t0])
        print(f"t0={t0:4d}: median loop {m:9.2f} ms  {B / (m / 1e3):8.1f} molecules/s (loop only)  ratio {m / plain:.3f}  "
              f"(t0+1)/(T+1) = {(t0 + 1) / (T + 1):.3f}")
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
