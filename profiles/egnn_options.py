"""Sampling throughput of models trained with the EGNN options tanh, sin_embedding and aggregation_method='mean'.

Samples a cfg2_zinc-shaped DDPM (B=256, N=40, L=6, T=500, synthetic weights) with the default options, each option and
all three, alternating the five models rep by rep, and prints molecules/s per run (B over the wall time of a synchronised
ddpm.sample_chain), then the card's name and power limit. With --forwards K it instead runs K Dynamics.forward calls per
model; run it with DL_TIME_KERNELS=1 to get the engine's per-kernel CUDA-event times (printed when each engine closes).

    python profiles/egnn_options.py [--workload cfg2_zinc] [--T 500] [--reps 3] [--forwards K]
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from difflinker_b200 import DDPM, synthetic
from difflinker_b200.batching import collate
from inpaint_sampling import card

VARIANTS = {"default": {}, "tanh": dict(tanh=True), "mean": dict(aggregation_method='mean'),
            "sin": dict(sin_embedding=True),
            "all three": dict(tanh=True, aggregation_method='mean', sin_embedding=True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2_zinc")
    ap.add_argument("--T", type=int, default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--forwards", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("egnn_options.py needs a GPU")
    spec = synthetic.SPECS[args.workload]
    dev = torch.device("cuda", 0)
    data = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in collate(synthetic.make_items(spec)).items()}
    B, N = data['positions'].shape[:2]
    models = {}
    for name, over in VARIANTS.items():
        hp = synthetic.model_hparams(spec)
        hp.update(over)
        if args.T is not None:
            hp['diffusion_steps'] = args.T
        torch.manual_seed(0)
        ddpm = DDPM(**hp)
        synthetic.init_reference_like_weights(ddpm)
        models[name] = ddpm.to(dev)
    print(f"card: {card()}")
    print(f"workload {spec.name}: B={B} N={N} L={spec.L} T={models['default'].edm.T} F={spec.F}, keep_frames=1")

    if args.forwards:
        from difflinker_b200.ddpm import sampler_inputs
        kw = sampler_inputs(models['default'], data)
        z = torch.cat([kw['x'], kw['h']], dim=2)
        t = torch.full((B, 1), 0.5, device=dev)
        for name, ddpm in models.items():
            dyn = ddpm.edm.dynamics
            for _ in range(args.forwards):
                dyn(t, z, kw['node_mask'], kw['linker_mask'], kw['edge_mask'], kw['context'])
            torch.cuda.synchronize()
            print(f"--- {name}: {args.forwards} forwards", flush=True)
            dyn.close()                                         # prints the DL_TIME_KERNELS table of this model
        return

    def run(ddpm):
        torch.manual_seed(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ddpm.sample_chain(data, keep_frames=1)
        torch.cuda.synchronize()
        return B / (time.perf_counter() - t0)

    for ddpm in models.values():                                # warm-up: graph capture, allocator
        run(ddpm)
    rates = {name: [] for name in models}
    for _ in range(args.reps):
        for name, ddpm in models.items():
            rates[name].append(run(ddpm))
            print(f"{name:10s} {rates[name][-1]:8.2f} molecules/s", flush=True)
    for name, r in rates.items():
        print(f"{name:10s} {min(r):.2f}-{max(r):.2f} molecules/s")


if __name__ == "__main__":
    main()
