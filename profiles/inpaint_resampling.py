"""RePaint resampling: the device loop of `InpaintingEDM.sample_chain(resamplings=r)` against the plain inpainting loop.

Two workloads, synthetic weights with the coordinate MLPs' output layers scaled by --coord-gain (0.1: at 1 the untrained
inpainting chains diverge at T = 500, and NaN coordinates would change a cut-off graph's work), keep_frames=1, default
edge path, device-side batch stream:
  - cfg2_zinc as an inpainting model (B=256, N=40, L=6) at T=500;
  - a cfg4_pockets batch (B=64, N=300 with 270 pocket atoms, FC-10A-4A graph) at T=100 (--pocket-T).
Runs are alternated -- every r in turn -- for --reps rounds after one warm-up round. Per run it prints the device loop time
(edm.last_loop_ms: CUDA events around the graph replays) and how many molecules diverged; then per r the median, its
ratio to the first r's (r0, 1 by default) and the pass ratio (T r + 1) / (T r0 + 1). Then, under torch.profiler, one
T = 20 call at r = 1 and one at r = 2 on the cfg2_zinc batch: the per-launch time of the inpainting step kernel without
(k_inpaint<., false>) and with the fused re-noise (k_inpaint<., true>), whose difference is the re-noise's cost per
pass. Last, the card's name and power limit, read in the same run.

    python profiles/inpaint_resampling.py [--r 1 2 5 10] [--reps 2] [--pocket-T 100] [--coord-gain 0.1]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.utils import FoundNaNException


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def model(spec_name, T, dev, gain):
    spec = synthetic.SPECS[spec_name]
    hp = synthetic.model_hparams(spec)
    hp['inpainting'] = True
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm)
    with torch.no_grad():
        for name, p in ddpm.named_parameters():
            if name.endswith("coord_mlp.4.weight"):
                p.mul_(gain)
    ddpm = ddpm.to(dev)
    ddpm.edm.T = T
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    return ddpm, data


def sweep(label, ddpm, data, rs, reps):
    B, N = data['positions'].shape[:2]
    T = ddpm.edm.T
    print(f"{label}: B={B} N={N} T={T}, keep_frames=1, default edge path")
    loops = {r: [] for r in rs}

    def one(r, record):
        torch.manual_seed(1)
        diverged = 0
        try:
            ddpm.sample_chain(data, keep_frames=1, resamplings=r)
        except FoundNaNException as exc:                    # the loop ran to its end: its time stands
            diverged = len(exc.x_h_nan_idx | exc.only_x_nan_idx | exc.only_h_nan_idx)
        torch.cuda.synchronize()
        if record:
            loops[r].append(ddpm.edm.last_loop_ms)
            print(f"  r={r:3d}  loop {ddpm.edm.last_loop_ms:10.2f} ms  diverged molecules {diverged}")
    for r in rs:                                            # warm-up: workspace, graph capture, module loads
        one(r, False)
    for _ in range(reps):
        for r in rs:
            one(r, True)
    base = statistics.median(loops[rs[0]])
    for r in rs:
        m = statistics.median(loops[r])
        print(f"  r={r:3d}: median loop {m:10.2f} ms  {B / (m / 1e3):8.1f} molecules/s (loop only)  ratio {m / base:6.3f}  "
              f"pass ratio (T r + 1)/(T r0 + 1) = {(T * r + 1) / (T * rs[0] + 1):6.3f}")


def renoise_cost(ddpm, data):
    """Per-launch device time of k_inpaint without and with the fused re-noise, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    ddpm.edm.T = 20

    def call(r):
        try:
            ddpm.sample_chain(data, keep_frames=1, resamplings=r)
        except FoundNaNException:
            pass
    for r in (1, 2):                                        # warm-up
        call(r)
    torch.cuda.synchronize()
    stats = {}
    for r in (1, 2):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(r)
            torch.cuda.synchronize()
        for ev in prof.key_averages():
            if "k_inpaint" in ev.key:
                stats[(r, ev.key)] = (ev.count, ev.device_time_total / max(ev.count, 1))
    if not stats:
        print("torch.profiler recorded no k_inpaint launches")
    for (r, key), (count, us) in sorted(stats.items()):
        print(f"  r={r}  {key[:60]:60s} {count:5d} launches  {us:8.2f} us each")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--r", type=int, nargs="+", default=[1, 2, 5, 10])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--pocket-T", type=int, default=100)
    ap.add_argument("--coord-gain", type=float, default=0.1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inpaint_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    ddpm, data = model("cfg2_zinc", 500, dev, args.coord_gain)
    print(f"coordinate MLP output gain {args.coord_gain}")
    sweep("cfg2_zinc inpainting", ddpm, data, args.r, args.reps)
    print("re-noise cost (cfg2_zinc, T=20):")
    renoise_cost(ddpm, data)
    del ddpm, data
    ddpm, data = model("cfg4_pockets", args.pocket_T, dev, args.coord_gain)
    sweep("cfg4_pockets inpainting", ddpm, data, args.r, args.reps)
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
