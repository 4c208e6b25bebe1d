"""InpaintingEDM: device-side noise (the default on CUDA) against the prepared draw tensor (noise_mode='reference_tensor').

Samples an inpainting DDPM at the cfg2_zinc shape (B=256, N=40, L=6, T=500, synthetic weights) from the same seed in both
modes, alternating them, and prints per run the wall time of ddpm.sample_chain (host clock around a synchronised call),
the device time of the reverse loop (edm.last_loop_ms) and the peak torch.cuda.max_memory_allocated; then the max
relative difference of chain[0] between the modes, and the card's name and power limit.

    python profiles/inpaint_sampling.py [--workload cfg2_zinc] [--T 500] [--reps 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2_zinc")
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inpaint_sampling.py needs a GPU")
    spec = synthetic.SPECS[args.workload]
    hp = synthetic.model_hparams(spec)
    hp['inpainting'] = True
    if args.T is not None:
        hp['diffusion_steps'] = args.T
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=100.0 if spec.N <= 64 else 1.0)
    ddpm = ddpm.to(dev)
    edm = ddpm.edm
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    B, N = data['positions'].shape[:2]
    print(f"card: {card()}")
    print(f"workload {spec.name}: B={B} N={N} L={spec.L} T={edm.T} F={spec.F}, inpainting, keep_frames=1")

    def run(mode):
        edm.noise_mode = mode
        torch.manual_seed(1)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        chain, _ = ddpm.sample_chain(data, keep_frames=1)
        torch.cuda.synchronize()
        wall = 1e3 * (time.perf_counter() - t0)
        return chain, wall, edm.last_loop_ms, torch.cuda.max_memory_allocated(dev) / 2**20

    for mode in ("reference_stream", "reference_tensor"):       # warm-up: graph capture, allocator, randn kernels
        run(mode)
    res = {"reference_stream": [], "reference_tensor": []}
    chains = {}
    for _ in range(args.reps):
        for mode in res:
            chain, wall, loop, peak = run(mode)
            chains[mode] = chain
            res[mode].append((wall, loop, peak))
            print(f"{mode:17s} wall {wall:9.2f} ms  device loop {loop:9.2f} ms  peak allocated {peak:9.1f} MiB")
    for mode, rows in res.items():
        walls, loops, peaks = zip(*rows)
        print(f"{mode:17s} wall {min(walls):.2f}-{max(walls):.2f} ms, loop {min(loops):.2f}-{max(loops):.2f} ms, "
              f"peak {max(peaks):.1f} MiB")
    a, b = chains["reference_stream"][0].double(), chains["reference_tensor"][0].double()
    rel = (a[..., :3] - b[..., :3]).abs().max().item() / max(b[..., :3].abs().max().item(), 1e-30)
    same_types = torch.equal(a[..., 3:], b[..., 3:])
    print(f"chain[0]: max relative coordinate difference {rel:.3g}, atom types identical: {same_types}")


if __name__ == "__main__":
    main()
