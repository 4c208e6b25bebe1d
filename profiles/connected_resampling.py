"""Connectivity in the recovery rounds: the cost of the device-side check and of the rounds that resample the disconnected
molecules (`sample_chain(..., require_connected=True)`, dl_sample_chain_retry).

Per workload (synthetic weights, seeds 0..B-1, keep_frames=1) it prints:
  * the device time of the check alone (dl_molecule_check with DL_CHECK_CONNECTED, CUDA events, median of --reps calls) on
    the sampled chain[0];
  * the fraction of rows that are disconnected after the first loop (round 0);
  * the device time of each recovery round (dl_last_retry_ms of runs with 1, 2, ... rounds, differenced: row gather, the
    wait for the host to capture the sub-batch's step graph, the sub-batch loop, its check, row scatter) next to the
    full-batch loop (edm.last_loop_ms -- what resampling the whole batch costs), and the connected rows after each round;
and the card's name, power limit and maximum SM clock. The synthetic workloads' fragments are random point clouds, not
molecules, so no row can connect: every round resamples the whole batch, and the round times are the worst case, a round
of B molecules. tests/test_connected_resampling.py samples a connected fragment with one or two linker atoms, where the
rounds do reconnect rows (DESIGN.md section 6 lists how many).

    python profiles/connected_resampling.py [--workload cfg2_zinc] [--workload cfg4_pockets] [--T 500] [--rounds 3]
"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, _native, molecule_builder, synthetic
from difflinker_b200.batching import collate
from difflinker_b200.ddpm import sampler_inputs


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi printed nothing"
    except (OSError, subprocess.SubprocessError) as e:
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def check_ms(edm, chain0, node_mask, pocket_only, reps):
    """Median device time of dl_molecule_check with connectivity alone over the batch, as the engine launches it."""
    lib = _native.load_library()
    B, N = chain0.shape[:2]
    require = _native.CHECK_CONNECTED
    tables = [t.to(chain0.device) for t in edm._check_tables(require)]
    checks = _native.DLMoleculeChecks.of(require, tables)
    nm = (node_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
    ctx = None if pocket_only is None else pocket_only.reshape(B, N, 1).float().contiguous()
    out = torch.empty(B, dtype=torch.int32, device=chain0.device)
    st = torch.cuda.current_stream()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(reps + 3):
        ev0.record(st)
        _native.check(lib.dl_molecule_check(B, N, checks, chain0.data_ptr(), chain0.shape[2], nm.data_ptr(),
                                            None if ctx is None else ctx.data_ptr(), 1, int(ctx is not None), out.data_ptr(),
                                            None, st.cuda_stream), "dl_molecule_check")
        ev1.record(st)
        ev1.synchronize()
        times.append(ev0.elapsed_time(ev1))
    times = sorted(times[3:])
    return times[len(times) // 2], out


def profile(spec, T, rounds, reps, dev):
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

    chain = edm.sample_chain(**kw, keep_frames=1, seeds=seeds, require_connected=True)       # round 0 only: a report
    conn0 = edm.last_connected
    ms, out = check_ms(edm, chain[0].contiguous(), kw['node_mask'], pocket_only, reps)
    assert torch.equal(out.cpu() != 0, conn0)
    checked = int(((kw['node_mask'].reshape(B, N) != 0) & (True if pocket_only is None else pocket_only.reshape(B, N) == 0)).sum())
    print(f"  check alone: {1e3 * ms:8.1f} us for {B} molecules ({checked} checked atoms of {B * N} rows)")
    print(f"  round 0: {B - int(conn0.sum())} of {B} rows disconnected ({100.0 * (1 - conn0.float().mean()):.1f} %)")
    # warm-up: every sub-batch size of the rounds gets its workspace and step graph, so the rounds below time sampling only
    edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=rounds, require_connected=True)
    prev = 0.0
    for r in range(1, rounds + 1):
        edm.sample_chain(**kw, keep_frames=1, seeds=seeds, nan_retries=r, require_connected=True)
        total = float(lib.dl_last_retry_ms(eng))
        resampled = int((edm.last_attempts == r).sum())                 # rows the round resampled and kept
        print(f"  round {r}: {resampled:4d} rows from it, {total - prev:9.2f} ms; full-batch loop {edm.last_loop_ms:9.2f} ms; "
              f"connected after it {int(edm.last_connected.sum())} of {B}")
        prev = total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", action="append", default=None)
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("connected_resampling.py needs a GPU")
    dev = torch.device("cuda", 0)
    print(f"card: {card()}")
    for name in args.workload or ["cfg2_zinc", "cfg4_pockets"]:
        profile(synthetic.SPECS[name], args.T, args.rounds, args.reps, dev)


if __name__ == "__main__":
    main()
