"""Per-molecule start steps: one mixed-t0 launch against one launch per t0, at the benchmarked shape.

The workload is cfg2_zinc (B=256, N=40, 8 linker atoms, L=6, synthetic weights) at T=500 and keep_frames=1, with the batch's
own linker kept in the template and per-molecule seeds. A sweep t0 in {50, 100, 250, 500} in equal shares (64 molecules each)
runs as
  mixed     one EDM.sample_chain call with start_step = one t0 per molecule;
  split     four single-t0 calls of the 64 molecules of each t0 (summed);
  scalar    one call of all 256 at t0 = 500, the cost the mixed call would have without skipping unstarted molecules;
  distinct  one call with all-distinct t0 (t0 = 500 - b for b in 0..255): a step graph per prefix length.
Runs are alternated for --reps rounds after one warm-up round, on the default edge path. Per case it prints the median
device loop time (edm.last_loop_ms: CUDA events around the loop, plan rebuilds and graph replays included), the median
wall time of the synchronised call, and their difference -- the host-side capture, graph update and gather overhead plus
Python -- and the molecule-steps the loop computed (dl_last_molecule_steps); then the card's name and power limit, read in
the same run.

    python profiles/mixed_start_steps.py [--reps 3] [--impl auto|simt]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs

SWEEP = (50, 100, 250, 500)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--impl", default="auto")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mixed_start_steps.py needs a GPU")
    dev = torch.device("cuda", 0)
    spec = synthetic.SPECS["cfg2_zinc"]
    hp = synthetic.model_hparams(spec)
    torch.manual_seed(0)
    ddpm = DDPM(**hp, edge_impl=args.impl)
    synthetic.init_reference_like_weights(ddpm)
    ddpm = ddpm.to(dev)
    edm = ddpm.edm
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data, keep_linker=True)
    B, N, T = kw['x'].shape[0], kw['x'].shape[1], edm.T
    assert B == 256 and T == 500
    seeds = list(range(1000, 1000 + B))
    share = B // len(SWEEP)
    mixed = [SWEEP[b % len(SWEEP)] for b in range(B)]
    distinct = [T - b for b in range(B)]
    lib = _native.load_library()
    print(f"cfg2_zinc B={B} N={N} L={hp['n_layers']} T={T}, keep_frames=1, edge_impl={args.impl}, per-molecule seeds; "
          f"sweep {SWEEP} in shares of {share}")

    def rows(idx):
        ix = torch.tensor(idx, device=dev)
        out = {}
        for k, v in kw.items():
            out[k] = None if v is None else (v.reshape(B, -1, *v.shape[1:])[ix].reshape(-1, *v.shape[1:])
                                             if k == 'edge_mask' else v[ix])
        return out

    def call(k, s, st):
        torch.cuda.synchronize()
        w0 = time.perf_counter()
        edm.sample_chain(**k, keep_frames=1, seeds=s, start_step=st)
        torch.cuda.synchronize()
        return edm.last_loop_ms, (time.perf_counter() - w0) * 1e3, int(lib.dl_last_molecule_steps(edm.dynamics.engine(0)))

    groups = [[b for b in range(B) if mixed[b] == t0] for t0 in SWEEP]
    cases = {
        "mixed": lambda: [call(kw, seeds, mixed)],
        "split": lambda: [call(rows(g), [seeds[b] for b in g], t0) for g, t0 in zip(groups, SWEEP)],
        "scalar": lambda: [call(kw, seeds, T)],
        "distinct": lambda: [call(kw, seeds, distinct)],
    }
    res = {name: [] for name in cases}
    for name, fn in cases.items():                 # warm-up: workspaces, module loads
        fn()
    for _ in range(args.reps):
        for name, fn in cases.items():
            runs = fn()
            res[name].append(tuple(sum(r[i] for r in runs) for i in range(3)))
    print(f"{'case':9s} {'loop ms':>10s} {'wall ms':>10s} {'wall-loop':>10s} {'mol-steps':>10s}")
    for name, rs in res.items():
        loop = statistics.median(r[0] for r in rs)
        wall = statistics.median(r[1] for r in rs)
        print(f"{name:9s} {loop:10.1f} {wall:10.1f} {wall - loop:10.1f} {rs[0][2]:10d}")
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
