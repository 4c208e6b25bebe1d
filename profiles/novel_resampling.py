"""Novelty in the recovery rounds: the cost of the linker hash and the known-set search in the check launch, of building a
known set, and of one recovery round of `sample_chain(..., require_novel=True)`.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the check launch with and without DL_CHECK_NOVEL as device times of the sampler's report-only check from
    torch.profiler over --calls calls of a T=10 model, at cfg2_zinc (B=256, N=40) and cfg4_pockets (B=64, N=300), for known
    sets of 0, 10^4 and 10^6 random hashes (0: the bit with an empty set; the search is then skipped by the count, the hash
    is not). Two pairs: k_molecule_check<3> against <19> (connectivity and valence, and the same plus the linker hash),
    which differ in launch bounds as well -- every hashing instantiation is compiled for one CTA per SM and takes more
    registers -- and <11> against <27> (the same with the molecule hash), which share launch bounds and shared-memory
    layout, so their difference is the linker hash and the search alone;
  * the rate of molecule_builder.known_linkers over --items dataset items of the cfg2_zinc shape;
  * the time of one recovery round (dl_last_retry_ms) with require_novel=True, nan_retries=1, T=--T, on cfg2_zinc with
    the linker hashes of a quarter of the rows planted in the set.
The weights are synthetic. It needs a GPU.

    python profiles/novel_resampling.py [--calls 20] [--items 20000] [--T 100]
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import _native, molecule_builder as mb, synthetic
from difflinker_b200.ddpm import sampler_inputs
from profiles.connected_resampling import card
from profiles.unique_resampling import kernel_us, model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--items", type=int, default=20000)
    ap.add_argument("--T", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("novel_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    g = torch.Generator().manual_seed(0)
    sets = {n: torch.randint(-(1 << 63), (1 << 63) - 1, (n,), generator=g, dtype=torch.int64) for n in (0, 10 ** 4, 10 ** 6)}

    for name in ("cfg2_zinc", "cfg4_pockets"):
        ddpm, data = model(synthetic.SPECS[name], 10, dev)
        edm = ddpm.edm
        kw = sampler_inputs(ddpm, data)
        B, N = kw['x'].shape[:2]
        seeds = list(range(B))
        links = int((kw['linker_mask'].reshape(B, N) != 0).sum()) // B
        print(f"workload {name}: B={B} N={N} graph {edm.dynamics.graph_type}, {links} linker atoms per molecule on average")
        two = dict(require_connected=True, require_valid=True)
        three = dict(two, require_unique=True)
        for run in range(2):                                             # alternating
            for label, flags in (("<3>  connected + valence", two), ("<11> connected + valence + unique", three)):
                t = kernel_us(edm, kw, seeds, flags, args.calls)
                print(f"  run {run}: {label:38s} k_molecule_check {t['k_molecule_check']:7.1f} us "
                      f"(mean over {args.calls} calls) [{where}]")
                for n, known in sets.items():
                    edm.known_linkers = known
                    t = kernel_us(edm, kw, seeds, dict(flags, require_novel=True), args.calls)
                    print(f"  run {run}: {'  + novel, %7d known hashes' % n:38s} k_molecule_check "
                          f"{t['k_molecule_check']:7.1f} us (mean over {args.calls} calls) [{where}]")

    spec = synthetic.SPECS["cfg2_zinc"]
    items = synthetic.make_items(spec, batch=args.items)
    for _ in range(2):
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        ev0.record()
        known = mb.known_linkers(items, False)
        ev1.record()
        ev1.synchronize()
        wall = time.perf_counter() - t0
        print(f"known_linkers: {len(items)} items -> {known.numel()} distinct hashes in {1e3 * wall:.1f} ms wall "
              f"({len(items) / wall:.0f} items/s; {ev0.elapsed_time(ev1):.1f} ms between events) [{where}]")

    ddpm, data = model(spec, args.T, dev)
    edm = ddpm.edm
    kw = sampler_inputs(ddpm, data)
    B = kw['x'].shape[0]
    seeds = list(range(2000, 2000 + B))
    base = edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    L = mb.linker_hashes(base[0], kw['node_mask'], kw['linker_mask'], edm.is_geom)
    edm.known_linkers = torch.cat([sets[10 ** 6].to(dev), L[: B // 4]])
    lib = _native.load_library()
    for run in range(3):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=1, require_novel=True)
        resampled = int((edm.last_attempts > 0).sum())
        print(f"  run {run}: one recovery round, cfg2_zinc T={edm.T}: {resampled} of {B} rows resampled, round time "
              f"{float(lib.dl_last_retry_ms(edm.dynamics.engine(0))):.1f} ms, first loop "
              f"{edm.last_loop_ms:.1f} ms [{where}]")


if __name__ == "__main__":
    main()
