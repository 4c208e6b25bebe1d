"""Clash guidance in the reverse loop: what `sample_chain(..., clash_guidance=(scale, steps))` costs, and how often round 0
still clashes with it.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the device loop (edm.last_loop_ms) at cfg4_pockets (B=64, N=300, T=--T) for steps K in {0, 50, 200, T}, scale 1,
    alternating the settings over --runs runs, with the round-0 clash verdict of each call (require_clash_free=True
    reports it; nan_retries=0 resamples nothing), and the cut-off graph the call's last forward built (dl_cut_graph_stats:
    GCL tile records, tiles, edges and coordinate-update records of the final step, tensor-core path);
  * k_clash_guide per launch inside the loop, from torch.profiler over one call with K = --profile-steps: the guided
    launches (the last K of the call) and the ones that return at once;
  * dl_clash_guide alone (CUDA events around --launches back-to-back launches after a warm-up, per launch) at
    cfg4_pockets on the chain[0] the model samples, and at a whole-protein shape (B=16, N=4000), with scale 1e-6 so that
    the geometry, and the work, barely changes from launch to launch;
  * the round-0 clash-failure fraction on the pulled-in lattice batch of tests/test_clash_guidance.py (a 24-atom pocket
    shell at 2.5 A around a 3 x 3 x 2 fragment lattice, T=10), guided (1, T) and not, over --rows rows.
Synthetic weights only: whether guidance raises a trained pocket model's clash-free rate is not measured here.
It needs a GPU.

    python profiles/clash_guidance.py [--T 1000] [--runs 2] [--launches 200] [--rows 256] [--profile-steps 200]
"""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(1, os.path.join(ROOT, "tests"))
import torch

from difflinker_b200 import _native, molecule_builder as mb, synthetic
from profiles.clash_resampling import model, whole_protein
from profiles.connected_resampling import card


def guide_us(xh, nm, lm, po, is_geom, launches):
    """Device time per launch (us) of dl_clash_guide over a copy of the batch: events around `launches` launches after 10
    more, scale 1e-6."""
    lib = _native.load_library()
    B, N = xh.shape[:2]
    table = mb.clash_table(is_geom).to(xh.device)
    xs = xh.float().contiguous().clone()
    nm = (nm.reshape(B, N) != 0).to(torch.int8).contiguous()
    lm = lm.reshape(B, N).float().contiguous()
    po = po.reshape(B, N, 1).float().contiguous()
    st = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def launch():
        _native.check(lib.dl_clash_guide(B, N, table.shape[0], table.data_ptr(), 1e-6, xs.data_ptr(), xs.shape[2],
                                         nm.data_ptr(), lm.data_ptr(), po.data_ptr(), 1, st.cuda_stream), "dl_clash_guide")
    for _ in range(10):
        launch()
    ev0.record(st)
    for _ in range(launches):
        launch()
    ev1.record(st)
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--profile-steps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clash_guidance.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    spec = synthetic.SPECS["cfg4_pockets"]

    ddpm, kw = model(spec, args.T, dev)
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    seeds = list(range(B))
    settings = [0, 50, 200, args.T]
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_clash_free=True)   # warm-up
    print(f"workload {spec.name}: B={B} N={N} graph {spec.graph_type} T={edm.T}; scale 1")
    lib = _native.load_library()
    eng = edm.dynamics.engine(dev.index or 0)
    stats = (ctypes.c_int64 * 4)()
    for run in range(args.runs):
        for K in settings:
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_clash_free=True,
                             clash_guidance=None if K == 0 else (1.0, K))
            ms = edm.last_loop_ms
            _native.check(lib.dl_cut_graph_stats(eng, stats), "dl_cut_graph_stats")
            print(f"  run {run}: K={K:5d}  device loop {ms:9.2f} ms; round-0 clash failures "
                  f"{B - int(edm.last_clash_free.sum())} of {B}; final step's cut-off graph: {stats[0]} GCL records, "
                  f"{stats[1]} tiles, {stats[2]} edges, {stats[3]} coordinate records [{where}]")

    K = args.profile_steps
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, clash_guidance=(1.0, K))
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if 'k_clash_guide' in e.name and e.device_time > 0),
                key=lambda e: e.time_range.start)
    assert len(ev) == edm.T + 1, len(ev)
    idle, guided = [e.device_time for e in ev[:edm.T - K]], [e.device_time for e in ev[edm.T - K:edm.T]]
    print(f"  k_clash_guide in the loop (torch.profiler, one call, K={K}): guided {sum(guided) / len(guided):7.2f} us mean "
          f"over {len(guided)} launches; unguided steps {sum(idle) / max(len(idle), 1):7.2f} us mean over {len(idle)} "
          f"[{where}]")

    chain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds)
    nm, lm, po = kw['node_mask'].reshape(B, N), kw['linker_mask'].reshape(B, N), kw['context'][..., -1].reshape(B, N)
    us = guide_us(chain[0], nm, lm, po, edm.is_geom, args.launches)
    print(f"  dl_clash_guide on chain[0]: {us:7.2f} us per launch over {args.launches} launches [{where}]")
    xh, nm4, lm4, po4, lo, hi = whole_protein(dev)
    us = guide_us(xh, nm4, lm4, po4, True, args.launches)
    print(f"whole-protein shape: B={xh.shape[0]} N={xh.shape[1]}, {lo}-{hi} linker atoms per molecule")
    print(f"  dl_clash_guide: {us:7.2f} us per launch over {args.launches} launches [{where}]")

    import test_clash_guidance as tg
    rows = args.rows
    seeds = list(range(1000, 1000 + rows))
    for impl in ("simt", "auto"):
        ddpm, kw = tg.build("4A", impl, rows=rows)
        edm = ddpm.edm
        for name, g in (("unguided", None), ("guided (1, T)", (1.0, edm.T))):
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_clash_free=True, clash_guidance=g)
            fails = rows - int(edm.last_clash_free.sum())
            print(f"pulled-in lattice batch, 4A/{impl}, T={edm.T}: {name:14s} round-0 clash failures {fails} of {rows} "
                  f"({fails / rows:.3f})")


if __name__ == "__main__":
    main()
