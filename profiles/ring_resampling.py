"""Ring sizes in the recovery rounds: the cost of the smallest-ring search in the check launch, and of one recovery round
of `sample_chain(..., require_ring_sizes=True)`.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the check launch with and without DL_CHECK_RINGS as device times of the sampler's report-only check from
    torch.profiler over --calls calls of a T=10 model, at cfg2_zinc (B=256, N=40) and cfg4_pockets (B=64, N=300), for
    k_molecule_check<3> against <35> (connectivity and valence, and the same plus the ring sizes) and <1> against <33>;
  * dl_ring_check alone (molecule_builder.ring_sizes) on the first loop's chain[0] of the same batches, by CUDA events
    over --calls calls;
  * the time of one recovery round (dl_last_retry_ms) with require_ring_sizes=True, allowed sizes 5 and 6, nan_retries=1:
    at cfg2_zinc, T=--T, and on the connectivity tests' small-fragment FC model (tests/test_connected_resampling.py, T=10,
    B=256), whose linker atoms often close a three-membered ring with the fragment lattice, so the round has rows to
    resample.
The weights are synthetic. It needs a GPU.

    python profiles/ring_resampling.py [--calls 20] [--T 100]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import _native, molecule_builder as mb, synthetic
from difflinker_b200.ddpm import sampler_inputs
from profiles.connected_resampling import card
from profiles.unique_resampling import kernel_us, model

ALLOWED = [5, 6]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--T", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ring_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")

    for name in ("cfg2_zinc", "cfg4_pockets"):
        ddpm, data = model(synthetic.SPECS[name], 10, dev)
        edm = ddpm.edm
        edm.allowed_ring_sizes = ALLOWED
        kw = sampler_inputs(ddpm, data)
        B, N = kw['x'].shape[:2]
        seeds = list(range(B))
        print(f"workload {name}: B={B} N={N} graph {edm.dynamics.graph_type}")
        one, two = dict(require_connected=True), dict(require_connected=True, require_valid=True)
        for run in range(2):                                             # alternating
            for label, flags in (("<1>  connected", one), ("<33> connected + rings", dict(one, require_ring_sizes=True)),
                                 ("<3>  connected + valence", two),
                                 ("<35> connected + valence + rings", dict(two, require_ring_sizes=True))):
                t = kernel_us(edm, kw, seeds, flags, args.calls)
                print(f"  run {run}: {label:34s} k_molecule_check {t['k_molecule_check']:7.1f} us "
                      f"(mean over {args.calls} calls) [{where}]")
        chain0 = edm.sample_chain(**kw, keep_frames=1, seeds=seeds)[0]
        po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
        masks = mb.ring_sizes(chain0, kw['node_mask'], kw['linker_mask'], edm.is_geom, po)
        sizes = sorted({k for m in masks.tolist() for k in range(3, 64) if (m >> k) & 1})
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(args.calls):
            mb.ring_sizes(chain0, kw['node_mask'], kw['linker_mask'], edm.is_geom, po)
        ev1.record()
        ev1.synchronize()
        print(f"  molecule_builder.ring_sizes: {1e3 * ev0.elapsed_time(ev1) / args.calls:7.1f} us per call, including "
              f"its table and mask copies; {int((masks != 0).sum())} of {B} rows with a linker ring, sizes {sizes} "
              f"[{where}]")

    ddpm, data = model(synthetic.SPECS["cfg2_zinc"], args.T, dev)
    edm = ddpm.edm
    edm.allowed_ring_sizes = ALLOWED
    kw = sampler_inputs(ddpm, data)
    B = kw['x'].shape[0]
    seeds = list(range(2000, 2000 + B))
    lib = _native.load_library()
    for run in range(3):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=1, require_ring_sizes=True)
        resampled = int((edm.last_attempts > 0).sum())
        print(f"  run {run}: one recovery round, cfg2_zinc T={edm.T}, allowed {ALLOWED}: {resampled} of {B} rows "
              f"resampled, round time {float(lib.dl_last_retry_ms(edm.dynamics.engine(0))):.1f} ms, first loop "
              f"{edm.last_loop_ms:.1f} ms [{where}]")

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import test_connected_resampling as tcr
    ddpm, kw = tcr.build("fc", "simt", rows=256)
    edm = ddpm.edm
    edm.allowed_ring_sizes = ALLOWED
    seeds = list(range(1, 257))
    for run in range(3):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=1, require_ring_sizes=True)
        resampled = int((edm.last_attempts > 0).sum())
        print(f"  run {run}: one recovery round, small-fragment FC model T={edm.T}, B=256, allowed {ALLOWED}: "
              f"{resampled} rows resampled, round time {float(lib.dl_last_retry_ms(edm.dynamics.engine(0))):.2f} ms, "
              f"first loop {edm.last_loop_ms:.2f} ms, {int(edm.last_ring_sizes_ok.sum())} rows pass after it [{where}]")


if __name__ == "__main__":
    main()
