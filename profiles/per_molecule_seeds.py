"""Per-molecule seeds against the batch stream: the cost of sampling with `seeds=` (dl_sample_chain_seeded).

Samples the cfg2_zinc shape (B=256, N=40, L=6, T=500, synthetic weights) with the linker sampler and with the inpainting
sampler, alternating noise_mode='reference_stream' and a seeded call (seeds 0..B-1), three runs each, and prints per run
the wall time of ddpm.sample_chain (host clock around a synchronised call) and the device time of the reverse loop
(edm.last_loop_ms), then each mode's range, and the card's name and power limit. Per element both streams do one Philox
initialisation and one curand_normal4, so the loops should take the same time.

    python profiles/per_molecule_seeds.py [--workload cfg2_zinc] [--T 500] [--reps 3]
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, synthetic
from difflinker_b200.batching import collate


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def profile(spec, T, reps, inpainting, dev):
    hp = synthetic.model_hparams(spec)
    hp['inpainting'] = inpainting
    if T is not None:
        hp['diffusion_steps'] = T
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=100.0 if spec.N <= 64 else 1.0)
    ddpm = ddpm.to(dev)
    edm = ddpm.edm
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    B, N = data['positions'].shape[:2]
    seeds = list(range(B))
    sampler = "inpainting" if inpainting else "linker"
    print(f"{sampler} sampler, workload {spec.name}: B={B} N={N} L={spec.L} T={edm.T} F={spec.F}, keep_frames=1")

    def run(mode):
        torch.manual_seed(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ddpm.sample_chain(data, keep_frames=1, seeds=seeds if mode == "seeded" else None)
        torch.cuda.synchronize()
        return 1e3 * (time.perf_counter() - t0), edm.last_loop_ms

    modes = ("reference_stream", "seeded")
    for mode in modes:                                          # warm-up: graph capture, allocator
        run(mode)
    res = {mode: [] for mode in modes}
    for _ in range(reps):
        for mode in modes:
            wall, loop = run(mode)
            res[mode].append((wall, loop))
            print(f"  {mode:17s} wall {wall:9.2f} ms  device loop {loop:9.2f} ms")
    for mode, rows in res.items():
        walls, loops = zip(*rows)
        print(f"  {mode:17s} wall {min(walls):.2f}-{max(walls):.2f} ms, loop {min(loops):.2f}-{max(loops):.2f} ms, "
              f"{B * 1e3 / min(loops):.1f} molecules/s on the best loop")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2_zinc")
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("per_molecule_seeds.py needs a GPU")
    dev = torch.device("cuda", 0)
    print(f"card: {card()}")
    spec = synthetic.SPECS[args.workload]
    for inpainting in (False, True):
        profile(spec, args.T, args.reps, inpainting, dev)


if __name__ == "__main__":
    main()
