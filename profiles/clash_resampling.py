"""Pocket clashes in the recovery rounds: the cost of the device-side clash check and of a round that resamples the molecules
whose linker clashes with the pocket (`sample_chain(..., require_clash_free=True)`, dl_sample_chain_retry).

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the clash check alone (dl_clash_check; CUDA events around --launches back-to-back launches after a warm-up, per launch)
    at cfg4_pockets (B=64, N=300) on the chain[0] the model samples, and at a whole-protein shape (B=16, N=4000: a pocket
    of about 3960 atoms on shells from 4 A outwards, a ligand of 40 rows of which 10-30 are linker atoms);
  * the three-check launch (connectivity, valence, clash: k_molecule_check<7>) against the two-check launch
    (k_molecule_check<3>), each the device time of the sampler's report-only check at cfg4_pockets, from torch.profiler
    over --calls calls of a T=10 model (the check does not depend on T);
  * one recovery round with the clash check on at cfg4_pockets, T=1000: the device time of round 1 (dl_last_retry_ms)
    next to edm.last_loop_ms of the same call.
It needs a GPU.

    python profiles/clash_resampling.py [--T 1000] [--launches 200] [--calls 20]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, molecule_builder as mb, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from profiles.connected_resampling import card


def clash_us(xh, nm, lm, po, is_geom, launches):
    """Device time per launch (us) of dl_clash_check over the batch: events around `launches` launches after 10 more."""
    lib = _native.load_library()
    B, N = xh.shape[:2]
    dev = xh.device
    table = mb.clash_table(is_geom).to(dev)
    xs = xh.float().contiguous()
    nm = (nm.reshape(B, N) != 0).to(torch.int8).contiguous()
    lm = lm.reshape(B, N).float().contiguous()
    po = po.reshape(B, N, 1).float().contiguous()
    out = torch.empty(B, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def launch():
        _native.check(lib.dl_clash_check(B, N, table.shape[0], table.data_ptr(), xs.data_ptr(), xs.shape[2], nm.data_ptr(),
                                         lm.data_ptr(), po.data_ptr(), 1, out.data_ptr(), None, st.cuda_stream),
                      "dl_clash_check")
    for _ in range(10):
        launch()
    ev0.record(st)
    for _ in range(launches):
        launch()
    ev1.record(st)
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches, out


def model(spec, T, dev):
    hp = synthetic.model_hparams(spec)
    hp['diffusion_steps'] = T
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=1.0)
    ddpm = ddpm.to(dev)
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    return ddpm, sampler_inputs(ddpm, data)


def check_kernel_us(edm, kw, seeds, flags, calls):
    """Mean device time (us) of the k_molecule_check kernel of the sampler's report-only check, from torch.profiler."""
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, **flags)         # warm-up
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            edm.sample_chain(**kw, keep_frames=1, seeds=seeds, **flags)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if 'k_molecule_check' in e.name and e.device_time > 0]
    assert len(times) == calls, len(times)
    return sum(times) / len(times), sorted(times)[len(times) // 2]


def whole_protein(dev, B=16, N=4000, n_lig=40):
    """A (B, N) chain[0]-style batch: a pocket on shells from 4 A outwards around a ligand within 2 A, GEOM types."""
    g = torch.Generator().manual_seed(5)
    xh = torch.zeros(B, N, 12)
    xh[:, :, 3:] = torch.nn.functional.one_hot(torch.randint(0, 9, (B, N), generator=g), 9).float()
    v = torch.randn(B, N, 3, generator=g)
    xh[:, :, :3] = (4.0 + 36.0 * torch.rand(B, N, 1, generator=g)) * v / v.norm(dim=2, keepdim=True)
    nm = torch.ones(B, N, dtype=torch.int8)
    nm[:, N - 40:] = 0                                                   # some padding
    po = torch.ones(B, N)
    lm = torch.zeros(B, N)
    n_link = torch.randint(10, 31, (B,), generator=g)
    for b in range(B):
        rows = torch.randperm(N - 40, generator=g)[:n_lig]
        xh[b, rows, :3] = 4.0 * torch.rand(n_lig, 3, generator=g) - 2.0
        po[b, rows] = 0.0
        lm[b, rows[:n_link[b]]] = 1.0
    return xh.to(dev), nm.to(dev), lm.to(dev), po.to(dev), int(n_link.min()), int(n_link.max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=1000)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("clash_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    spec = synthetic.SPECS["cfg4_pockets"]
    lib = _native.load_library()

    # the checks alone and in one launch, on a T = 10 model's chain[0]
    ddpm, kw = model(spec, 10, dev)
    edm = ddpm.edm
    B, N = kw['x'].shape[:2]
    seeds = list(range(B))
    nm, lm, po = kw['node_mask'].reshape(B, N), kw['linker_mask'].reshape(B, N), kw['context'][..., -1].reshape(B, N)
    chain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_clash_free=True)
    ok0 = edm.last_clash_free
    us, out = clash_us(chain[0], nm, lm, po, edm.is_geom, args.launches)
    assert torch.equal((out.cpu() & _native.CHECK_CLASH) != 0, ok0)
    n_link = int(((nm != 0) & (lm != 0) & (po == 0)).sum())
    n_pocket = int(((nm != 0) & (po != 0)).sum())
    print(f"workload {spec.name}: B={B} N={N} graph {spec.graph_type}; {n_link} linker atoms, {n_pocket} pocket atoms; "
          f"{int(ok0.sum())} of {B} rows clash-free at T=10")
    print(f"  dl_clash_check: {us:7.1f} us per launch over {args.launches} launches [{where}]")
    two = dict(require_connected=True, require_valid=True)
    three = dict(require_connected=True, require_valid=True, require_clash_free=True)
    for run in range(2):                                                 # alternating
        for name, flags in (("two checks (connected, valence)", two), ("three checks (+ clash)", three)):
            mean, med = check_kernel_us(edm, kw, seeds, flags, args.calls)
            print(f"  run {run}: {name:34s} k_molecule_check {mean:7.1f} us mean, {med:7.1f} us median over {args.calls} "
                  f"calls [{where}]")

    xh, nm4, lm4, po4, lo, hi = whole_protein(dev)
    us, out = clash_us(xh, nm4, lm4, po4, True, args.launches)
    print(f"whole-protein shape: B={xh.shape[0]} N={xh.shape[1]}, {lo}-{hi} linker atoms per molecule, "
          f"{int(((nm4 != 0) & (po4 != 0)).sum()) // xh.shape[0]} pocket atoms per molecule; "
          f"{int((out != 0).sum())} of {xh.shape[0]} clash-free")
    print(f"  dl_clash_check: {us:7.1f} us per launch over {args.launches} launches [{where}]")

    # one round at T = args.T
    ddpm, kw = model(spec, args.T, dev)
    edm = ddpm.edm
    eng = edm.dynamics.engine(dev.index or 0)
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_clash_free=True)   # report only; warms the loop up
    print(f"workload {spec.name} at T={edm.T}: {int(edm.last_clash_free.sum())} of {B} rows clash-free at round 0; the "
          f"round includes the sub-batch's first graph capture")
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=1, require_clash_free=True)
    print(f"  full-batch loop {edm.last_loop_ms:9.2f} ms; round 1 ({int((edm.last_attempts == 1).sum())} rows kept from it) "
          f"{float(lib.dl_last_retry_ms(eng)):9.2f} ms; clash-free after it {int(edm.last_clash_free.sum())} of {B} [{where}]")


if __name__ == "__main__":
    main()
