"""Uniqueness in the recovery rounds: the cost of the graph hash and of the uniqueness verdict, and how many rows and rounds
`sample_chain(..., require_unique=True)` spends on one input sampled B times.

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the check launch with and without DL_CHECK_UNIQUE (k_molecule_check<3> against <11>: connectivity and valence, and
    the same plus the hash) and the verdict kernel (k_unique_verdict), as device times of the sampler's report-only check
    from torch.profiler over --calls calls of a T=10 model (neither depends on T), at
      cfg2_zinc (B=256, N=40), cfg4_pockets (B=64, N=300, the pocket rows dropped), and an inpainting batch at N=300 (the
      cfg4_pockets shape as whole molecules of up to 300 atoms under an inpainting model on FC graphs, which checks and
      hashes every atom);
  * dl_molecule_hash alone (CUDA events over --launches launches) on the same three batches;
  * rows resampled and rounds used with require_unique=True, nan_retries=--rounds, on one cfg2_zinc input copied B=64
    times with a linker size of 2, sampled from noise and with start_step=--t0.
The weights are synthetic, so the duplicate rates say nothing about a trained checkpoint. It needs a GPU.

    python profiles/unique_resampling.py [--calls 20] [--launches 200] [--rounds 8] [--t0 5]
"""
import argparse
import dataclasses
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, molecule_builder as mb, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from profiles.connected_resampling import card


def model(spec, T, dev, inpainting=False, items=None):
    if inpainting:                                                       # the same shape as whole molecules on FC graphs
        spec = dataclasses.replace(spec, graph_type='FC', pocket=0)
    hp = synthetic.model_hparams(spec)
    hp['diffusion_steps'] = T
    if inpainting:
        hp['inpainting'] = True
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=1.0)
    ddpm = ddpm.to(dev)
    items = synthetic.make_items(spec) if items is None else items
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(items).items()}
    return ddpm, data


def kernel_us(edm, kw, seeds, flags, calls):
    """{kernel: mean device time (us)} of the check and verdict kernels of the sampler's report-only check."""
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, **flags)         # warm-up
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds, **flags)
        torch.cuda.synchronize()
    out = {}
    for key in ('k_molecule_check', 'k_unique_verdict'):
        times = [e.device_time for e in prof.events() if key in e.name and e.device_time > 0]
        if times:                                                        # per kernel event (the profiler may list one twice)
            out[key] = sum(times) / len(times)
    return out


def hash_us(edm, chain0, node_mask, pocket_only, launches):
    """Device time per launch (us) of dl_molecule_hash over the batch, called directly with tables built once (graph_hashes
    builds them on the host per call): events around `launches` launches after 10 more."""
    lib = _native.load_library()
    B, N = chain0.shape[:2]
    dev = chain0.device
    xs = chain0.float().contiguous()
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    po = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    tables = [t.to(dev) for t in mb.check_tables(edm.is_geom, _native.CHECK_UNIQUE)]
    checks = _native.DLMoleculeChecks.of(_native.CHECK_UNIQUE, tables)
    h = torch.empty(B, dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def launch():
        _native.check(lib.dl_molecule_hash(B, N, checks, xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                           None if po is None else po.data_ptr(), 1, int(po is not None), h.data_ptr(),
                                           st.cuda_stream), "dl_molecule_hash")
    for _ in range(10):
        launch()
    ev0.record(st)
    for _ in range(launches):
        launch()
    ev1.record(st)
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches, h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--t0", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("unique_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")

    for name, spec, inpainting in (("cfg2_zinc", synthetic.SPECS["cfg2_zinc"], False),
                                   ("cfg4_pockets", synthetic.SPECS["cfg4_pockets"], False),
                                   ("inpainting, cfg4_pockets batch", synthetic.SPECS["cfg4_pockets"], True)):
        ddpm, data = model(spec, 10, dev, inpainting)
        edm = ddpm.edm
        kw = sampler_inputs(ddpm, data)
        B, N = kw['x'].shape[:2]
        seeds = list(range(B))
        po = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
        nm = kw['node_mask'].reshape(B, N)
        atoms = int(((nm != 0) & (po.reshape(B, N) == 0 if po is not None else True)).sum()) // B
        print(f"workload {name}: B={B} N={N} graph {edm.dynamics.graph_type}, {atoms} checked atoms per molecule on average")
        two = dict(require_connected=True, require_valid=True)
        for run in range(2):                                             # alternating
            for label, flags in (("connected + valence", two), ("connected + valence + unique", dict(two, require_unique=True))):
                t = kernel_us(edm, kw, seeds, flags, args.calls)
                extra = f", k_unique_verdict {t['k_unique_verdict']:6.1f} us" if 'k_unique_verdict' in t else ""
                print(f"  run {run}: {label:30s} k_molecule_check {t['k_molecule_check']:7.1f} us{extra} "
                      f"(mean over {args.calls} calls) [{where}]")
        chain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_unique=True)
        us, h = hash_us(edm, chain[0], nm, po, args.launches)
        assert torch.equal(h.cpu(), edm.last_graph_hashes)
        print(f"  dl_molecule_hash: {us:7.1f} us per launch over {args.launches} launches; {len(set(h.tolist()))} distinct "
              f"hashes among {B} rows, {int(edm.last_unique.sum())} rows keep the bit [{where}]")

    # one input copied B times, a linker of 2 atoms: from noise, and from step t0
    spec = synthetic.SPECS["cfg2_zinc"]
    B = 64
    item = synthetic.make_items(spec, batch=1)[0]
    ddpm, data = model(spec, 100, dev, items=[dict(item, uuid=b) for b in range(B)])
    edm = ddpm.edm
    seeds = list(range(1000, 1000 + B))
    for label, opts in (("from noise, linker size 2", dict(linker_sizes=2)), (f"start_step={args.t0}", dict(start_step=args.t0))):
        ddpm.sample_chain(data, keep_frames=1, seeds=seeds, nan_retries=0, require_unique=True, **opts)
        first = int(edm.last_unique.sum())
        ddpm.sample_chain(data, keep_frames=1, seeds=seeds, nan_retries=args.rounds, require_unique=True, **opts)
        att = edm.last_attempts
        rounds_used = int(att.max())
        print(f"one cfg2_zinc input x {B}, T={edm.T}, {label}: {first} of {B} rows unique after the loop; after up to "
              f"{args.rounds} rounds {int(edm.last_unique.sum())} unique, {int((att > 0).sum())} rows replaced, last round "
              f"that replaced a row {rounds_used}, retry time {float(_native.load_library().dl_last_retry_ms(edm.dynamics.engine(0))):.1f} ms "
              f"[{where}] (synthetic weights)")


if __name__ == "__main__":
    main()
