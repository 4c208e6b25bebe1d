"""Anchors in the recovery rounds: the cost of the anchor check (k_anchor_check) and of `sample_chain(...,
require_anchors=True)`.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * dl_anchor_check alone, launched directly with tables built once, on the first loop's chain[0] of a T=10 model with the
    batch's own anchors: device time per launch by CUDA events over --launches launches after 20 warm-up launches, at
    cfg2_zinc (B=256, N=40) and cfg4_pockets (B=64, N=300);
  * the first loop plus its checks, report-only (nan_retries=0), with require_connected and with require_connected plus
    require_anchors: the median host time of --calls seeded calls each, alternated, at cfg2_zinc with T=--T;
  * rounds and rows resampled with require_anchors=True and nan_retries=3 at cfg2_zinc, T=--T: how many rows each
    attempt produced, the rounds' time (dl_last_retry_ms) and how many rows pass after them.
The weights and the anchors are synthetic, so the counts say nothing about any published model's attachment rate. It
needs a GPU.

    python profiles/anchor_resampling.py [--launches 200] [--calls 3] [--T 100]
"""
import argparse
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import _native, molecule_builder as mb, synthetic
from difflinker_b200.ddpm import sampler_inputs, template_anchors
from profiles.connected_resampling import card
from profiles.unique_resampling import model


def anchor_check_us(edm, chain0, kw, anchors, pocket_only, launches):
    """Device time per launch (us) of dl_anchor_check over the batch: events around `launches` launches after 20 more."""
    lib = _native.load_library()
    B, N = chain0.shape[:2]
    dev = chain0.device
    xs = chain0.float().contiguous()
    nm = (kw['node_mask'].reshape(B, N) != 0).to(torch.int8).contiguous()
    lm = kw['linker_mask'].reshape(B, N).float().contiguous()
    an = (anchors.reshape(B, N) != 0).to(torch.int8).contiguous()
    po = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    thr1 = mb.threshold_tables(edm.is_geom)[0].to(dev).contiguous()
    passed = torch.empty(B, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream().cuda_stream

    def launch():
        _native.check(lib.dl_anchor_check(B, N, thr1.shape[0], thr1.data_ptr(), xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                          lm.data_ptr(), an.data_ptr(), None if po is None else po.data_ptr(), 1,
                                          int(po is not None), passed.data_ptr(), None, st), "dl_anchor_check")
    for _ in range(20):
        launch()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(launches):
        launch()
    ev1.record()
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches, int(((passed & _native.CHECK_ANCHORS) != 0).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--T", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("anchor_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")

    for name in ("cfg2_zinc", "cfg4_pockets"):
        ddpm, data = model(synthetic.SPECS[name], 10, dev)
        edm = ddpm.edm
        kw = sampler_inputs(ddpm, data)
        B, N = kw['x'].shape[:2]
        anchors = template_anchors(ddpm, data, N)
        po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
        if po is not None:
            anchors = anchors * (po.reshape(B, N) == 0)
        chain0 = edm.sample_chain(**kw, keep_frames=1, seeds=list(range(B)))[0]
        for run in range(2):
            us, n_ok = anchor_check_us(edm, chain0, kw, anchors, po, args.launches)
            print(f"workload {name}: B={B} N={N}: run {run}: dl_anchor_check {us:7.2f} us per launch (mean over "
                  f"{args.launches} launches); {n_ok} of {B} rows pass [{where}]")

    ddpm, data = model(synthetic.SPECS["cfg2_zinc"], args.T, dev)
    edm = ddpm.edm
    kw = sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    anchors = template_anchors(ddpm, data, N)
    seeds = list(range(2000, 2000 + B))
    plain, anchored = dict(require_connected=True), dict(require_connected=True, require_anchors=True, anchors=anchors)
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=0, **anchored)   # warm-up
    times = {"connected": [], "connected + anchors": []}
    for _ in range(args.calls):                                          # alternating
        for label, flags in (("connected", plain), ("connected + anchors", anchored)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=0, **flags)
            torch.cuda.synchronize()
            times[label].append(1e3 * (time.perf_counter() - t0))
    for label, ts in times.items():
        print(f"  cfg2_zinc T={edm.T}: first loop + checks, {label:20s}: median {statistics.median(ts):8.1f} ms over "
              f"{len(ts)} calls ({', '.join(f'{t:.1f}' for t in ts)}) [{where}]")
    lib = _native.load_library()
    for run in range(2):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=3, require_anchors=True, anchors=anchors)
        att = edm.last_attempts
        per = [int((att == a).sum()) for a in range(4)]
        print(f"  run {run}: cfg2_zinc T={edm.T}, nan_retries=3: rows per attempt {per} (attempt 0 first), rounds "
              f"{float(lib.dl_last_retry_ms(edm.dynamics.engine(0))):.1f} ms, first loop {edm.last_loop_ms:.1f} ms, "
              f"{int(edm.last_anchors_ok.sum())} of {B} rows pass after the rounds [{where}]")


if __name__ == "__main__":
    main()
