"""Valence in the recovery rounds: the cost of the device-side molecule checks and of the rounds that resample the molecules
failing them (`sample_chain(..., require_valid=True, require_connected=True)`, dl_sample_chain_retry).

It prints the card's name, power limit and maximum SM clock, read in this run, beside every number:
  * the check alone (dl_molecule_check: valence, connectivity, both; CUDA events around --launches back-to-back launches
    after a warm-up, per launch) at cfg2_zinc (B=256, N=40) and at the pocket shape cfg4_pockets (B=64, N=300), on the
    chain[0] the model samples;
  * the cost of a recovery round with both checks on against the full-batch loop, three alternating runs: the device time
    of round 1 (dl_last_retry_ms: row gather, the wait for the host to capture the sub-batch's step graph, the sub-batch
    loop, its check, row scatter) next to edm.last_loop_ms of the same call.
The synthetic workloads' fragments are random point clouds, not molecules, so no row is connected: the round resamples
the whole batch and its time is the worst case. tests/test_valid_resampling.py samples a carbon lattice with one or two
linker atoms, where the rounds do repair rows (DESIGN.md section 6 lists how many). It needs a GPU.

    python profiles/valid_resampling.py [--workload cfg2_zinc] [--workload cfg4_pockets] [--T 500] [--launches 200]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs
from profiles.connected_resampling import card

CHECKS = {"valence": _native.CHECK_VALENCE, "connectivity": _native.CHECK_CONNECTED,
          "both": _native.CHECK_VALENCE | _native.CHECK_CONNECTED}


def check_us(edm, require, chain0, node_mask, pocket_only, launches):
    """Device time per launch (us) of dl_molecule_check over the batch: events around `launches` launches after 10 more."""
    lib = _native.load_library()
    B, N = chain0.shape[:2]
    tables = [t.to(chain0.device) for t in edm._check_tables(require)]
    checks = _native.DLMoleculeChecks.of(require, tables)
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    ctx = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    out = torch.empty(B, dtype=torch.int32, device=chain0.device)
    st = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def launch():
        _native.check(lib.dl_molecule_check(B, N, checks, chain0.data_ptr(), chain0.shape[2], nm.data_ptr(),
                                            None if ctx is None else ctx.data_ptr(), 1, int(ctx is not None), out.data_ptr(),
                                            None, st.cuda_stream), "dl_molecule_check")
    for _ in range(10):
        launch()
    ev0.record(st)
    for _ in range(launches):
        launch()
    ev1.record(st)
    ev1.synchronize()
    return 1e3 * ev0.elapsed_time(ev1) / launches, out


def profile(spec, T, launches, dev, where):
    hp = synthetic.model_hparams(spec)
    if T is not None:
        hp['diffusion_steps'] = T
    torch.manual_seed(0)
    ddpm = DDPM(**hp)
    synthetic.init_reference_like_weights(ddpm, coord_gain=100.0 if spec.N <= 64 else 1.0)
    ddpm = ddpm.to(dev)
    edm = ddpm.edm
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    kw = sampler_inputs(ddpm, data)
    B, N = kw['x'].shape[:2]
    seeds = list(range(B))
    lib = _native.load_library()
    eng = edm.dynamics.engine(dev.index or 0)
    pocket_only = kw['context'][..., -1] if edm.dynamics.graph_type != 'FC' else None
    print(f"workload {spec.name}: B={B} N={N} L={spec.L} T={edm.T} F={spec.F} graph {spec.graph_type}, keep_frames=1")
    both = dict(require_valid=True, require_connected=True)
    chain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, **both)   # round 0 only: a report
    ok0, conn0 = edm.last_valid, edm.last_connected
    checked = int(((kw['node_mask'].reshape(B, N) != 0) & (True if pocket_only is None else pocket_only.reshape(B, N) == 0)).sum())
    chain0 = chain[0].contiguous()
    for name, require in CHECKS.items():
        us, out = check_us(edm, require, chain0, kw['node_mask'], pocket_only, launches)
        out = out.cpu()
        assert not require & _native.CHECK_VALENCE or torch.equal((out & _native.CHECK_VALENCE) != 0, ok0)
        assert not require & _native.CHECK_CONNECTED or torch.equal((out & _native.CHECK_CONNECTED) != 0, conn0)
        print(f"  check alone, {name:12s}: {us:7.1f} us per launch over {launches} launches, {B} molecules ({checked} checked "
              f"atoms of {B * N} rows) [{where}]")
    print(f"  round 0: {int(ok0.sum())} of {B} rows within valence, {int(conn0.sum())} connected, {int((ok0 & conn0).sum())} both")
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=1, **both)   # warm-up: the round's workspace and graph
    for run in range(3):                                                 # the loop and the round alternate within each call
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=1, **both)
        print(f"  run {run}: full-batch loop {edm.last_loop_ms:9.2f} ms; round 1 ({int((edm.last_attempts == 1).sum())} rows kept "
              f"from it) {float(lib.dl_last_retry_ms(eng)):9.2f} ms; passing both after it "
              f"{int((edm.last_valid & edm.last_connected).sum())} of {B} [{where}]")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", action="append", default=None)
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("valid_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    where = card()
    print(f"card (name, power limit, max SM clock): {where}")
    for name in args.workload or ["cfg2_zinc", "cfg4_pockets"]:
        profile(synthetic.SPECS[name], args.T, args.launches, dev, where)


if __name__ == "__main__":
    main()
