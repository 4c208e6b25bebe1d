"""Many small requests: one `EDM.sample_many` against the sequence of `sample_chain` calls it replaces.

The workload is what generate.py sends: 64 fragment pairs x 10 samples, one request each, ZINC-shaped (the cfg2_zinc model,
L=6, synthetic weights, 8 linker atoms) with N varying from 30 to 45 across the requests, at T = 500, keep_frames=1 and
seeds 10k..10k+9 for request k. Alternates the sequential calls and one sample_many, three runs each, on one GPU and with
devices='all', and prints per run the wall time (host clock around synchronised calls), molecules/s, and for sample_many
each launch's device loop ms (edm.last_loop_ms_many); then the card's name and power limit, read in the same run. Timed on
the default edge path. The outputs are compared request by request first: on the SIMT edge path they must be equal bit for
bit (asserted); on the tensor-core path the count of bit-identical requests and the largest difference are printed, since
these weights drive coordinates to hundreds of Angstrom, where node tiles rescale their fp16 operands (DESIGN.md section 6).

    python profiles/sample_many.py [--requests 64] [--samples 10] [--T 500] [--reps 3]
"""
import argparse
import dataclasses
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def workload(ddpm, n_requests, n_samples, dev):
    base = synthetic.SPECS["cfg2_zinc"]
    reqs, seeds = [], []
    for k in range(n_requests):
        n = 30 + k % 16
        spec = dataclasses.replace(base, name=f"cfg2_zinc_N{n}", B=n_samples, N=n, n_min=n)
        data = {key: (v.to(dev) if torch.is_tensor(v) else v)
                for key, v in collate(synthetic.make_items(spec, batch=n_samples, seed_offset=k)).items()}
        reqs.append(sampler_inputs(ddpm, data))
        seeds.append(list(range(n_samples * k, n_samples * (k + 1))))
    return reqs, seeds


def build(hp, edge_impl, dev):
    torch.manual_seed(0)
    ddpm = DDPM(**hp, edge_impl=edge_impl)
    synthetic.init_reference_like_weights(ddpm, coord_gain=100.0)
    return ddpm.to(dev)


def compare(got, want):
    exact = sum(torch.equal(g, w) for g, w in zip(got, want))
    worst = max(((g - w).abs().max() / w.abs().max().clamp(min=1.0)).item() for g, w in zip(got, want))
    return exact, worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--samples", type=int, default=10)
    ap.add_argument("--T", type=int, default=500)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_many.py needs a GPU")
    dev = torch.device("cuda", 0)
    hp = synthetic.model_hparams(synthetic.SPECS["cfg2_zinc"])
    hp['diffusion_steps'] = args.T
    ddpm = build(hp, 'simt', dev)
    reqs, seeds = workload(ddpm, args.requests, args.samples, dev)
    n_mol = sum(len(s) for s in seeds)
    print(f"{args.requests} requests x {args.samples} molecules, N 30-45, L={hp['n_layers']} T={ddpm.edm.T}, keep_frames=1")
    edm = ddpm.edm

    def sequential():
        return [edm.sample_chain(**r, keep_frames=1, seeds=s) for r, s in zip(reqs, seeds)]

    def many():
        return edm.sample_many(reqs, keep_frames=1, seeds=seeds)
    exact, worst = compare(many(), sequential())
    print(f"SIMT edge path: {exact} of {len(reqs)} requests bit-identical, worst difference {worst:.2e} of max|x|")
    assert exact == len(reqs)
    ddpm.edm.dynamics.close()
    ddpm = build(hp, 'auto', dev)
    edm = ddpm.edm

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0

    for devices in (None, 'all'):
        edm.devices = devices
        label = "1 GPU" if devices is None else f"devices={edm.devices}"
        want, _ = timed(sequential)                                 # warm-up: every shape's workspace and graph
        got, _ = timed(many)
        exact, worst = compare(got, want)
        print(f"{label}, default edge path: {exact} of {len(want)} requests bit-identical, worst difference {worst:.2e} "
              "of max|x|")
        res = {"sequential sample_chain": [], "one sample_many": []}
        for _ in range(args.reps):
            for name, fn in (("sequential sample_chain", sequential), ("one sample_many", many)):
                _, wall = timed(fn)
                res[name].append(wall)
                line = f"  {name:24s} wall {wall * 1e3:9.1f} ms  {n_mol / wall:7.1f} molecules/s"
                if fn is many:
                    line += "  launches (device, molecules, loop ms): " + ", ".join(
                        f"({d}, {sum(len(seeds[k]) for k in ks)}, {ms:.1f})" for d, ks, ms in edm.last_loop_ms_many)
                print(line)
        for name, walls in res.items():
            print(f"  {label} {name:24s} {n_mol / max(walls):.1f}-{n_mol / min(walls):.1f} molecules/s")
    edm.devices = None
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
