"""compute-sanitizer target: one small call of every native entry point (run: compute-sanitizer --tool memcheck python profiles/sanitize.py)."""
import os, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')  # repo root
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch
import dl_helpers as helpers
from difflinker_b200 import synthetic, linker_size, molecule_builder, output
from difflinker_b200.batching import collate

d = torch.device('cuda:0')
IMPL = os.environ.get('DL_SAN_IMPL', 'auto')      # racecheck run: 'simt' keeps the mbarrier/TMA kernels out of the tool's way
mv = lambda t: t.to(d) if torch.is_tensor(t) else t

# FC forward + short linker chain (tensor-core path), ragged masks
spec = synthetic.WorkloadSpec("san_fc", B=3, N=23, n_min=11, l_min=2, l_max=6, F=8, L=2, T=4, seed=31)
ddpm, hp = helpers.build_ddpm(spec, 0, edge_impl=IMPL)
ddpm = ddpm.to(d)
data = {k: mv(v) for k, v in collate(synthetic.make_items(spec)).items()}
chain, nm = ddpm.sample_chain(data, keep_frames=2)
print("fc chain", tuple(chain.shape), bool(torch.isfinite(chain).all()))

# inpainting chain
ddpm_i, _ = helpers.build_ddpm(spec, 0, edge_impl=IMPL, inpainting=True)
ddpm_i = ddpm_i.to(d)
chain, nm = ddpm_i.sample_chain(data, keep_frames=1)
print("inpaint chain", tuple(chain.shape), bool(torch.isfinite(chain).all()))

# N > 64: column-split epilogue, chunked rows
spec2 = synthetic.WorkloadSpec("san_big", B=2, N=150, n_min=150, l_min=8, l_max=8, F=8, L=1, T=2, seed=32)
dyn, _ = helpers.build_dynamics(spec2, 0, edge_impl=IMPL)
b2 = collate(synthetic.make_items(spec2))
z, t = helpers.random_latent(b2, 3)
out = dyn(mv(t), mv(z), mv(b2['atom_mask']), mv(b2['linker_mask']), mv(b2['edge_mask']), mv(b2['fragment_mask']))
print("N=150 forward", bool(torch.isfinite(out).all()))

# cut-off graph: neighbour lists + packed tiles
base = synthetic.SPECS["cfg4_pockets"]
spec3 = synthetic.WorkloadSpec(base.name, B=2, N=90, n_min=90, l_min=5, l_max=5, F=9, L=1, T=2, seed=33, pocket=60,
                               graph_type="FC-10A-4A")
dyn3, _ = helpers.build_dynamics(spec3, 1)
b3 = collate(synthetic.make_items(spec3))
z, t = helpers.random_latent(b3, 4, pad_garbage=False)
ctx = helpers.context_of(b3, spec3)
out = dyn3(mv(t), mv(z), mv(b3['atom_mask']), mv(b3['linker_mask']), mv(b3['edge_mask']), mv(ctx))
print("pocket forward", bool(torch.isfinite(out).all()))

# size classifier, bond orders, frame restore
model = linker_size.SizeClassifier(in_node_nf=8, out_node_nf=10, n_layers=3).eval()
sd = {k: mv(v) for k, v in linker_size.collate_with_fragment_edges(synthetic.make_items(spec)).items()}
print("sizes", model.sample_sizes(sd).tolist())
E = molecule_builder.bond_orders(sd['one_hot'], sd['positions'], sd['atom_mask'], False)
print("bonds", int((E != 0).sum()))
x = output.restore_frame(torch.cat([sd['positions'], sd['one_hot']], dim=2).contiguous(), sd['positions'], sd['fragment_mask'],
                         sd['atom_mask'])
print("restore", bool(torch.isfinite(x).all()))

# connectivity check, alone and in the recovery rounds (FC and cut-off graphs)
xh = torch.cat([sd['positions'], sd['one_hot']], dim=2).contiguous()
print("connected", molecule_builder.connected(xh, sd['atom_mask'], False).tolist())
chain, nm = ddpm.sample_chain(data, keep_frames=1, seeds=[1, 2, 3], nan_retries=2, require_connected=True)
print("connected rounds", ddpm.edm.last_connected.tolist(), ddpm.edm.last_attempts.tolist())
ddpm3, _ = helpers.build_ddpm(spec3, 0, edge_impl=IMPL)
ddpm3 = ddpm3.to(d)
ddpm3.edm.T = 2
chain, nm = ddpm3.sample_chain({k: mv(v) for k, v in b3.items()}, keep_frames=1, seeds=[1, 2], nan_retries=1,
                               require_connected=True)
print("pocket connected rounds", ddpm3.edm.last_connected.tolist(), ddpm3.edm.last_attempts.tolist())

# valence check, alone and with the connectivity check in the recovery rounds (dl_molecule_check,
# dl_sample_chain_retry)
print("valences", molecule_builder.valences(xh, sd['atom_mask'], False).sum(1).tolist(),
      molecule_builder.valence_ok(xh, sd['atom_mask'], False).tolist())
chain, nm = ddpm.sample_chain(data, keep_frames=1, seeds=[1, 2, 3], nan_retries=2, require_connected=True, require_valid=True)
print("checked rounds", ddpm.edm.last_valid.tolist(), ddpm.edm.last_connected.tolist(), ddpm.edm.last_attempts.tolist())
chain, nm = ddpm3.sample_chain({k: mv(v) for k, v in b3.items()}, keep_frames=1, seeds=[1, 2], nan_retries=1,
                               require_valid=True)
print("pocket valence rounds", ddpm3.edm.last_valid.tolist(), ddpm3.edm.last_attempts.tolist())
