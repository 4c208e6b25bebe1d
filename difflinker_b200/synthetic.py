"""Seeded synthetic workloads shaped like BASELINE.json's configs (SURVEY.md section 8(d)): no dataset or checkpoint is
reachable offline, so molecules are random point clouds with the reference's exact batch layout
(datasets.collate dtypes, fragments first, then [pocket,] then linker atoms)."""
from dataclasses import dataclass, field
from typing import Optional

import torch

from .batching import collate


@dataclass
class WorkloadSpec:
    name: str
    B: int
    N: int
    n_min: int            # valid atoms per molecule drawn from U{n_min..N}; molecule 0 always has N
    l_min: int
    l_max: int            # linker atoms U{l_min..l_max}
    F: int = 8            # in_node_nf
    L: int = 6            # n_layers
    S: int = 2            # inv_sublayers
    T: int = 500
    seed: int = 0
    pocket: int = 0       # pocket atoms per molecule (0 = ligand-only workload)
    graph_type: str = 'FC'
    anchors_context: bool = False
    hparams: dict = field(default_factory=dict)

    @property
    def context_node_nf(self):
        base = 2 if self.pocket else 1
        return base + (1 if self.anchors_context else 0)


SPECS = {
    # configs[0]: the reference's own CPU-runnable plumbing case
    "cfg1_plumbing": WorkloadSpec("cfg1_plumbing", B=4, N=30, n_min=21, l_min=3, l_max=7, F=8, L=4, T=50, seed=1),
    # configs[1]: the headline ZINC case; roofline variant has every molecule at full size
    "cfg2_zinc": WorkloadSpec("cfg2_zinc", B=256, N=40, n_min=40, l_min=8, l_max=8, F=8, L=6, T=500, seed=2),
    "cfg2_zinc_ragged": WorkloadSpec("cfg2_zinc_ragged", B=256, N=40, n_min=24, l_min=3, l_max=12, F=8, L=6, T=500,
                                     seed=2),
    "cfg2_zinc_L8": WorkloadSpec("cfg2_zinc_L8", B=256, N=40, n_min=40, l_min=8, l_max=8, F=8, L=8, T=500, seed=2),
    "cfg3_geom": WorkloadSpec("cfg3_geom", B=256, N=60, n_min=60, l_min=10, l_max=10, F=9, L=6, T=500, seed=3),
    "cfg3_geom_ragged": WorkloadSpec("cfg3_geom_ragged", B=256, N=60, n_min=36, l_min=3, l_max=20, F=9, L=6, T=500,
                                     seed=3),
    "cfg4_pockets": WorkloadSpec("cfg4_pockets", B=64, N=300, n_min=300, l_min=8, l_max=8, F=9, L=6, T=1000, seed=4,
                                 pocket=270, graph_type='FC-10A-4A'),
}
for _n in (32, 64, 128, 256, 512):
    SPECS[f"cfg5_sweep_N{_n}"] = WorkloadSpec(f"cfg5_sweep_N{_n}", B=128, N=_n, n_min=_n, l_min=8, l_max=8, F=8, L=6,
                                              T=10, seed=5)


# Linker-size classifier batches: GEOM types without pockets, and a pocket batch on a 10-column one-hot whose pockets (140
# atoms) give every pocket row more than 128 live columns once with_pocket moves them to the origin.
SIZE_GNN_SPECS = {
    "size_geom": WorkloadSpec("size_geom", B=5, N=40, n_min=15, l_min=2, l_max=10, F=9, L=2, T=10, seed=24),
    "size_pocket_geom": WorkloadSpec("size_pocket_geom", B=3, N=160, n_min=150, l_min=4, l_max=8, F=10, L=2, T=10,
                                     seed=23, pocket=140, graph_type='4A'),
}


def size_gnn_items(spec: WorkloadSpec, batch: int):
    """make_items, and on pocket specs the fragment-only atoms of the last type moved to type 0: the last one-hot column
    is then zero on every fragment-only row, as SizeClassifier.forward(adjust_shape=True) requires before dropping it."""
    items = make_items(spec, batch=batch)
    if spec.pocket:
        for it in items:
            oh = it['one_hot']
            move = (it['fragment_only_mask'] != 0) & (oh[:, -1] != 0)
            oh[move, -1] = 0.0
            oh[move, 0] = 1.0
    return items


def model_hparams(spec: WorkloadSpec) -> dict:
    """DDPM hyper-parameters of the corresponding published config (configs/*.yml: nf 128, inv_sublayers 2,
    norm_constant 1e-6, normalization_factor 100, normalize_factors [1,4,10], polynomial_2, precision 1e-5)."""
    hp = dict(
        in_node_nf=spec.F, n_dims=3, context_node_nf=spec.context_node_nf, hidden_nf=128, activation='silu',
        tanh=False, n_layers=spec.L, attention=False, norm_constant=1e-6, inv_sublayers=spec.S, sin_embedding=False,
        normalization_factor=100, aggregation_method='sum', diffusion_steps=spec.T,
        diffusion_noise_schedule='polynomial_2', diffusion_noise_precision=1e-5, diffusion_loss_type='l2',
        normalize_factors=[1, 4, 10], include_charges=False, model='egnn_dynamics',
        train_data_prefix='MOAD_train.full' if spec.pocket else ('geom_train' if spec.F == 9 else 'zinc_train'),
        val_data_prefix='val', center_of_mass='fragments', inpainting=False, anchors_context=spec.anchors_context,
        graph_type=spec.graph_type,
        normalization='batch_norm',   # every configs/*.yml sets it; the reference ignores it for egnn_dynamics (egnn.py:355-368)
    )
    hp.update(spec.hparams)
    return hp


def _pocket_points(gen, ligand_pos, count):
    """Jittered 1.5 A cubic lattice inside a 12 A ball, >= 3 A away from every ligand atom."""
    ax = torch.arange(-12.0, 12.01, 1.5)
    grid = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), dim=-1).reshape(-1, 3)
    grid = grid + 0.3 * torch.randn(grid.shape, generator=gen)
    grid = grid[grid.norm(dim=1) <= 12.0]
    far = torch.cdist(grid, ligand_pos).min(dim=1).values >= 3.0
    grid = grid[far]
    order = torch.argsort(grid.norm(dim=1))        # closest shell first: a pocket hugging the ligand
    pts = grid[order][:count]
    assert pts.shape[0] == count, "not enough lattice points for the pocket"
    return pts


def make_items(spec: WorkloadSpec, batch: Optional[int] = None, seed_offset: int = 0):
    """Per-molecule dicts in the layout datasets return (src/datasets.py:96-125, 296-323)."""
    gen = torch.Generator().manual_seed(1000 * spec.seed + 17 + seed_offset)
    B = spec.B if batch is None else batch
    items = []
    for b in range(B):
        n_lig_max = spec.N - spec.pocket
        lk = int(torch.randint(spec.l_min, spec.l_max + 1, (1,), generator=gen))
        if b == 0 or spec.n_min >= spec.N:
            n_lig = n_lig_max
        else:
            n_lig = int(torch.randint(spec.n_min - spec.pocket, n_lig_max + 1, (1,), generator=gen))
        lk = min(lk, n_lig - 2)
        n_frag = n_lig - lk
        frag_pos = 2.5 * torch.randn((n_frag, 3), generator=gen)
        link_pos = 2.5 * torch.randn((lk, 3), generator=gen)
        if spec.pocket:
            frag_pos = frag_pos * 0.6              # compact ligand so the pocket shell fits the 12 A ball
            pocket_pos = _pocket_points(gen, torch.cat([frag_pos, link_pos]), spec.pocket)
            pos = torch.cat([frag_pos, pocket_pos, link_pos], dim=0)
        else:
            pos = torch.cat([frag_pos, link_pos], dim=0)
        n = pos.shape[0]
        types = torch.randint(0, spec.F, (n,), generator=gen)
        one_hot = torch.nn.functional.one_hot(types, spec.F).float()
        anchors = torch.zeros(n)
        anchors[torch.randperm(n_frag, generator=gen)[:2]] = 1.0
        frag_only = torch.zeros(n); frag_only[:n_frag] = 1.0
        pocket_mask = torch.zeros(n); pocket_mask[n_frag:n_frag + spec.pocket] = 1.0
        linker_mask = torch.zeros(n); linker_mask[n_frag + spec.pocket:] = 1.0
        item = {
            'uuid': b, 'name': f'{spec.name}_{b}', 'positions': pos, 'one_hot': one_hot, 'anchors': anchors,
            'fragment_mask': frag_only + pocket_mask, 'linker_mask': linker_mask, 'num_atoms': n,
        }
        if spec.pocket:
            item['fragment_only_mask'] = frag_only
            item['pocket_mask'] = pocket_mask
        items.append(item)
    return items


def make_batch(spec: WorkloadSpec, batch: Optional[int] = None, seed_offset: int = 0, collate_fn=collate):
    return collate_fn(make_items(spec, batch, seed_offset))


def init_reference_like_weights(module: torch.nn.Module, seed: int = 0, coord_gain: float = 100.0):
    """SURVEY.md section 8(c): default init is what the caller already did under its own seed; the last coord_mlp
    layer has xavier gain 1e-3 (egnn.py:90-91) which would make the coordinate path numerically invisible with
    random weights, so it is scaled up for benchmarks/fixtures."""
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith('coord_mlp.4.weight'):
                p.mul_(coord_gain)
    return module


def flops_alg(n: int, l: int, spec: WorkloadSpec, edges: float = None, linker_edges: float = None) -> float:
    """Algorithmic FLOPs of one Dynamics.forward for one molecule with n valid atoms, l linker atoms
    (SURVEY.md section 8(d)). Cut-off graphs: `edges` / `linker_edges` = the molecule's true edge count and the edges
    whose row is a linker atom replace n^2 and l*n."""
    H, D = 128, spec.F + spec.context_node_nf + 1
    e = n * n if edges is None else edges
    ex = l * n if linker_edges is None else linker_edges
    gcl = 2 * H * H * e + 10 * H * H * n + 10 * H * e
    coord = 2 * H * H * ex + 4 * H * H * n + 8 * H * ex
    return 2 * D * H * n + spec.L * (spec.S * gcl + coord) + 2 * H * spec.F * l


def cutoff_edge_counts(batch, graph_type: str):
    """Per-molecule (edges, edges on linker rows) of the cut-off graph at the batch's input coordinates
    (egnn.py:554-596); the graph is re-derived from the current coordinates every step, so this is the count the
    roofline uses for the whole chain (only the <= 12 linker atoms move)."""
    x = batch['positions'].float()
    nm = batch['atom_mask'].reshape(x.shape[0], -1) != 0
    pk = batch['pocket_mask'].reshape(x.shape[0], -1) > 0
    lig = nm & ~pk
    lm = batch['linker_mask'].reshape(x.shape[0], -1) > 0
    out = []
    for b in range(x.shape[0]):
        d = torch.cdist(x[b], x[b])
        ll = lig[b][:, None] & lig[b][None, :]
        pp = pk[b][:, None] & pk[b][None, :]
        lp = (lig[b][:, None] & pk[b][None, :]) | (pk[b][:, None] & lig[b][None, :])
        if graph_type == '4A':
            adj = (nm[b][:, None] & nm[b][None, :]) & (d <= 4)
        else:
            cut = 4.0 if graph_type == 'FC-4A' else 10.0
            adj = ll | (pp & (d <= 4)) | (lp & (d <= cut))
        adj = adj & ~torch.eye(adj.shape[0], dtype=torch.bool)
        out.append((float(adj.sum()), float(adj[lm[b]].sum())))
    return out


def bytes_alg(N: int, spec: WorkloadSpec) -> float:
    return spec.L * (2 * spec.S + 1) * N * 128 * 4 + 64 * N


def init_size_gnn_like_trained(module, seed: int):
    """Default torch init leaves the size classifier's logits almost constant; scale the weights a little and give the
    BatchNorm layers non-trivial running statistics so that every term of the forward pass matters in parity tests."""
    g = torch.Generator().manual_seed(4242 + seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if p.dim() == 2:
                p.mul_(1.5)
        for name, b in module.named_buffers():
            if name.endswith("running_mean"):
                b.copy_(0.1 * torch.randn(b.shape, generator=g))
            elif name.endswith("running_var"):
                b.copy_(0.5 + torch.rand(b.shape, generator=g))
        for name, p in module.named_parameters():
            if ".node_mlp.1." in name or ".node_mlp.4." in name:            # BatchNorm affine
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g) if name.endswith("weight")
                        else 0.1 * torch.randn(p.shape, generator=g))
