"""One sampling batch split over several local GPUs from one process (EDM.devices).

For the cfg2_zinc shape (N=40, L=6, T=500, synthetic weights) at B=64 (generate.py's batch) and B=256, on 1, 2, 4 and 8
devices (as many as are visible; with one visible GPU, also two engines on GPU 0), prints per run:
  - the wall time of ddpm.sample_chain (host clock around a call that starts and ends with every device synchronised);
  - each slice's CUDA-event loop time (edm.last_slice_loop_ms) and the host time its dl_sample_chain_rng call took to return
    (whether the enqueue blocks until the loop has run);
  - whether the chain equals the 1-device chain bit for bit, and if not, by how much it differs.
Then, in a separate profiled call per configuration (torch.profiler, CUDA activity), each device's window from its first to
its last sampler kernel on the profiler's common clock, and how much of the windows all devices share. The card's name and
power limit come first.

    python profiles/multi_device_sampling.py [--workload cfg2_zinc] [--batches 64 256] [--T 500] [--reps 3] [--no-trace]
"""
import argparse
import os
import re
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, synthetic
from difflinker_b200 import edm as edm_module
from difflinker_b200.batching import collate

SAMPLER_KERNEL = re.compile(r"\bk_[a-z]")     # the engine's kernels (k_edge_tc, k_node_tc, k_prep, ...), not torch's copies


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def sync_all():
    for i in range(torch.cuda.device_count()):
        torch.cuda.synchronize(i)


# host time each slice's dl_sample_chain_rng call takes to return, per thread (wraps the function every slice is sampled by)
_enqueue = []
_sample_slice = edm_module._sample_slice


def _timed_sample_slice(*args, **kwargs):
    t0 = time.perf_counter()
    out = _sample_slice(*args, **kwargs)
    _enqueue.append((threading.current_thread().name, 1e3 * (time.perf_counter() - t0)))
    return out


edm_module._sample_slice = _timed_sample_slice


def device_windows(prof):
    """{device: (first sampler-kernel start, last sampler-kernel end)} in ms on the profiler's clock."""
    win = {}
    for e in prof.profiler.kineto_results.events():
        if e.device_type() != torch.autograd.DeviceType.CUDA or not SAMPLER_KERNEL.search(e.name()):
            continue
        lo, hi = win.get(e.device_index(), (float('inf'), float('-inf')))
        win[e.device_index()] = (min(lo, e.start_ns() * 1e-6), max(hi, e.end_ns() * 1e-6))
    return win


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2_zinc")
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-trace", action="store_true", help="skip the profiled call that checks the windows overlap")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_device_sampling.py needs a GPU")
    visible = torch.cuda.device_count()
    spec = synthetic.SPECS[args.workload]
    hp = synthetic.model_hparams(spec)
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=100.0 if spec.N <= 64 else 1.0)
    ddpm = ddpm.to(dev)
    edm = ddpm.edm
    if args.T is not None:
        edm.T = args.T
    setups = [(f"{n} GPU" + ("s" if n > 1 else ""), list(range(n)) if n > 1 else None) for n in (1, 2, 4, 8) if n <= visible]
    if visible == 1:
        setups.append(("2 engines on GPU 0", [0, 0]))
    print(f"cards:\n{card()}")
    print(f"visible GPUs: {visible}; workload {spec.name}: N={spec.N} L={spec.L} T={edm.T} F={spec.F}, keep_frames=1")

    for B in args.batches:
        data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec, batch=B)).items()}

        def run(devices):
            edm.devices = devices
            torch.manual_seed(1)
            _enqueue.clear()
            sync_all()
            t0 = time.perf_counter()
            chain, _ = ddpm.sample_chain(data, keep_frames=1)
            sync_all()
            return chain, 1e3 * (time.perf_counter() - t0)

        reference = None
        for label, devices in setups:
            run(devices)                                        # warm-up: engines, graph capture, allocator
            walls = []
            for _ in range(args.reps):
                chain, wall = run(devices)
                walls.append(wall)
                if reference is None:
                    reference = chain
                if torch.equal(chain, reference):
                    same = "bit-identical to 1 GPU"
                else:                                       # rounding of fp16 tiles rescaled for large values (DESIGN.md 6)
                    diff = (chain - reference).abs().amax(dim=(0, 2, 3))
                    same = (f"{int((diff > 0).sum())} of {B} molecules differ from 1 GPU, max |d| / max |x| = "
                            f"{diff.max().item() / reference.abs().max().item():.2g}")
                if devices is None:
                    loops = f"loop {edm.last_loop_ms:.2f} ms"
                else:
                    loops = "loops " + ", ".join(f"cuda{d}[{lo}:{hi}] {ms:.2f}" for d, lo, hi, ms in edm.last_slice_loop_ms)
                    loops += " ms; enqueue returned after " + ", ".join(f"{ms:.1f}" for _, ms in _enqueue) + " ms"
                print(f"B={B:4d} {label:19s} wall {wall:9.2f} ms  {B / wall * 1e3:8.1f} molecules/s  {loops}  {same}")
            print(f"B={B:4d} {label:19s} wall {min(walls):.2f}-{max(walls):.2f} ms over {args.reps} runs")
            if devices is None or args.no_trace or len(set(devices)) < 2:     # windows are per device
                continue
            edm.devices = devices
            torch.manual_seed(1)
            sync_all()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                ddpm.sample_chain(data, keep_frames=1)
                sync_all()
            win = device_windows(prof)
            if not win:
                print(f"B={B:4d} {label:19s} profiler recorded no sampler kernels")
                continue
            t0 = min(lo for lo, _ in win.values())
            common = min(hi for _, hi in win.values()) - max(lo for lo, _ in win.values())
            shortest = min(hi - lo for lo, hi in win.values())
            print(f"B={B:4d} {label:19s} profiled windows (ms from the first kernel): " +
                  ", ".join(f"cuda{d} {lo - t0:.2f}-{hi - t0:.2f}" for d, (lo, hi) in sorted(win.items())) +
                  f"; all devices busy together for {max(common, 0.0):.2f} ms = {100 * max(common, 0.0) / shortest:.0f}% "
                  "of the shortest window")


if __name__ == "__main__":
    main()
