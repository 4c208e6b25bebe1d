"""Replica-level data parallelism (SURVEY.md section 8(e)): molecules never interact across a batch, so sampling shards
with no data-path collective. The only exchange is one broadcast of the weights at start-up (NCCL on GPUs,
gloo in the CPU tests); optionally the final results are gathered. `resolve_devices`, `device_slices` and `place_rows` plan and
gather the split of one batch over several local GPUs that `EDM.devices` makes from a single process; `plan_launches`,
`deal_launches`, `pack_requests` and `unpack_rows` plan, assemble and take apart the shared launches of `EDM.sample_many`."""
import operator

import torch
import torch.distributed as dist


def shard_range(n_items: int, rank: int, world: int):
    """Contiguous, balanced [lo, hi) slice of `n_items` for `rank` (first n_items % world ranks get one more)."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def resolve_devices(devices, device_count=None):
    """`EDM.devices` as a list of CUDA device indices: None stays None (the caller's device), 'all' is every visible device,
    otherwise a non-empty list of visible indices (one may repeat: each listing gets an engine of its own)."""
    if devices is None:
        return None
    n = torch.cuda.device_count() if device_count is None else device_count
    if isinstance(devices, str):
        if devices != 'all':
            raise ValueError(f"devices must be a list of CUDA device indices, 'all' or None (got {devices!r})")
        if n == 0:
            raise ValueError("devices='all': no CUDA device is visible")
        return list(range(n))
    out = []
    for d in devices:
        if isinstance(d, bool):
            raise TypeError(f"CUDA device indices are integers (got {d!r})")
        d = operator.index(d)
        if not 0 <= d < n:
            raise ValueError(f"unknown CUDA device {d} ({n} visible)")
        out.append(d)
    if not out:
        raise ValueError("devices is empty: list at least one CUDA device, or pass None for the caller's device")
    return out


def device_slices(n_items: int, devices):
    """The split of one batch over `devices`: [(device, replica, lo, hi)], slot i getting shard_range(n_items, i, len(devices)).
    `replica` counts earlier listings of the same device (each listing has an engine of its own); slots whose slice would be
    empty (n_items < len(devices)) are left out."""
    out, seen = [], {}
    for i, d in enumerate(devices):
        lo, hi = shard_range(n_items, i, len(devices))
        replica = seen.get(d, 0)
        seen[d] = replica + 1
        if hi > lo:
            out.append((d, replica, lo, hi))
    return out


def place_rows(out: torch.Tensor, parts, slices, dim: int = 0):
    """Copies every slice's result into rows [lo, hi) of `out` along `dim` (stream-ordered, also across devices); returns `out`.
    Per-molecule NaN flags placed this way carry batch-global molecule indices."""
    for part, (_, _, lo, hi) in zip(parts, slices):
        out.narrow(dim, lo, hi - lo).copy_(part)
    return out


def plan_launches(sizes, nodes, max_molecules: int, keys=None):
    """How `EDM.sample_many` packs requests into launches: [(request indices, N)], every request in exactly one launch and
    never split, N the largest N_k of the launch (the others are padded to it). Requests share a launch only with requests of
    the same key (`keys`: one hashable per request, None for all the same; EDM.sample_many's holds what sets how a launch
    samples: step coefficients, start scalars, jump coefficients, clash guidance), so each group is planned on its own,
    groups in the order of their first request. Within a group the requests are sorted by (N_k, index), which keeps the padding small,
    and filled in that order into launches of at most `max_molecules` molecules; a request larger than that gets a launch
    of its own. Deterministic: the same inputs give the same plan."""
    if len(sizes) != len(nodes) or (keys is not None and len(keys) != len(sizes)):
        raise ValueError("sizes, nodes and keys need one entry per request")
    if max_molecules < 1:
        raise ValueError(f"max_molecules must be >= 1 (got {max_molecules})")
    groups = {}
    for k in range(len(sizes)):
        groups.setdefault(None if keys is None else keys[k], []).append(k)
    launches = []
    for members in groups.values():
        current, total = [], 0
        for k in sorted(members, key=lambda k: (nodes[k], k)):
            if current and total + sizes[k] > max_molecules:
                launches.append(current)
                current, total = [], 0
            current.append(k)
            total += sizes[k]
        launches.append(current)
    return [(ks, max(nodes[k] for k in ks)) for ks in launches]


def deal_launches(costs, n_slots: int):
    """The slot (index into the listed devices) of every launch: the costliest launch first, each to the slot with the least
    cost so far, the lowest slot on a tie. Each slot then runs its launches in launch order."""
    load, out = [0] * n_slots, [None] * len(costs)
    for i in sorted(range(len(costs)), key=lambda i: (-costs[i], i)):
        s = min(range(n_slots), key=lambda s: (load[s], s))
        out[i] = s
        load[s] += costs[i]
    return out


def pack_requests(requests, n_nodes: int, fc: bool):
    """One launch's inputs from several requests' keyword arguments of `EDM.sample_chain`: each request's tensors padded with
    dead atoms (zeros) to `n_nodes`, then concatenated along B in request order. On FC graphs (`fc`) the flattened edge mask
    becomes each molecule's (N, N) block padded with 0 and is returned as (B N N, 1), the datasets.collate layout; on
    cut-off graphs the per-node batch ids are rebuilt for the launch (the engine does not read them)."""
    out = {}
    for name in requests[0]:
        vals = [r[name] for r in requests]
        if all(v is None for v in vals):
            out[name] = None
        elif any(v is None for v in vals):
            raise ValueError(f"some requests give {name} and others do not")
        elif name != 'edge_mask':
            out[name] = torch.cat([torch.cat([v, v.new_zeros((v.shape[0], n_nodes - v.shape[1]) + tuple(v.shape[2:]))], dim=1)
                                   for v in vals])
        elif fc:
            blocks = []
            for v, r in zip(vals, requests):
                B, N = r['x'].shape[:2]
                blocks.append(torch.nn.functional.pad(v.reshape(B, N, N), (0, n_nodes - N, 0, n_nodes - N)))
            out[name] = torch.cat(blocks).reshape(-1, 1)
        else:
            B = sum(r['x'].shape[0] for r in requests)
            out[name] = torch.arange(B, device=vals[0].device).repeat_interleave(n_nodes).to(vals[0].dtype)
    return out


def unpack_rows(t: torch.Tensor, sizes, nodes, dim: int = 0):
    """The inverse of pack_requests for a launch's result `t`: request k's rows (along `dim`, in request order) and, when
    `nodes` is given, its first N_k atoms (the dimension after `dim`), each as a contiguous tensor."""
    out, lo = [], 0
    for k, b in enumerate(sizes):
        part = t.narrow(dim, lo, b)
        if nodes is not None:
            part = part.narrow(dim + 1, 0, nodes[k])
        out.append(part.contiguous())
        lo += b
    return out


def batch_ids_for_rank(n_batches: int, rank: int, world: int):
    """Round-robin whole batches {rank, rank+world, ...}: weak scaling, seed = seed0 + batch id."""
    return list(range(rank, n_batches, world))


def broadcast_module_weights(module: torch.nn.Module, src: int = 0, device=None):
    """One flat fp32 broadcast of every parameter/buffer (about 6 MB at L=6). Returns the number of floats."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 0
    tensors = [p.data for p in module.parameters()] + [b.data for b in module.buffers()]
    if not tensors:
        return 0
    dev = device if device is not None else tensors[0].device
    flat = torch.cat([t.reshape(-1).to(device=dev, dtype=torch.float32) for t in tensors])
    dist.broadcast(flat, src=src)
    off = 0
    with torch.no_grad():
        for t in tensors:
            n = t.numel()
            t.copy_(flat[off:off + n].reshape(t.shape).to(device=t.device, dtype=t.dtype))
            off += n
    return off


def gather_chains(chain: torch.Tensor, dst: int = 0):
    """Optional final gather of per-rank (keep,B,N,D) results on `dst` (92 KB per rank for cfg 3)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [chain]
    out = [torch.empty_like(chain) for _ in range(dist.get_world_size())] if dist.get_rank() == dst else None
    dist.gather(chain, out, dst=dst)
    return out


def slice_sampler_inputs(kw: dict, lo: int, hi: int):
    """Rows [lo, hi) of the keyword arguments `ddpm.sampler_inputs` builds for `EDM.sample_chain`. The FC edge mask is the
    flattened (B*N*N, 1) tensor of datasets.collate; the pocket variant is the per-node batch-id vector (B*N)."""
    B, N = kw['x'].shape[0], kw['x'].shape[1]
    out = {}
    for k, v in kw.items():
        if k == 'edge_mask' and v is not None:
            per = v.shape[0] // B
            out[k] = v[lo * per:hi * per]
        else:
            out[k] = None if v is None else v[lo:hi]
    return out


def sample_chain_sharded(model, data, sample_fn=None, keep_frames=None, gather=True, seeds=None, nan_retries=None,
                         require_connected=None, require_valid=None, require_clash_free=None, linker_sizes=None,
                         require_novel=None, require_ring_sizes=None, require_anchors=None, linker_types=None):
    """Strong scaling of ONE batch (SURVEY.md section 8(e)): the template batch is built once (so every rank pads to the same
    N), each rank runs the reverse loop for its contiguous slice of the molecules with the slice's rows of the full-batch
    noise, and the chains are gathered -- the result equals `model.sample_chain(data)` on one GPU bit for bit, for any
    world size, on the SIMT path and on the tensor-core path while no sample diverges far enough for the node GEMM to
    rescale a tile's fp16 operands (DESIGN.md section 6). No collective inside the loop. Returns (chain, node_mask) with
    the full batch on every rank when `gather`, else the local slice.
    `seeds`: the full batch's B per-molecule seeds (EDM.sample_chain); each rank samples its rows with its rows of them,
    so the result equals `model.sample_chain(data, seeds=seeds)` on one GPU in the same sense. `nan_retries` (with seeds):
    each rank resamples its own diverged molecules (EDM.sample_chain); a FoundNaNException names the rank's local rows.
    `require_connected` (with seeds): each rank also resamples its own disconnected molecules; `model.edm.last_connected`
    holds the rank's rows. `require_valid` likewise for the molecules with an atom beyond its valence (`last_valid`), and
    `require_clash_free` for those whose linker clashes with the pocket (`last_clash_free`), and `require_novel` for those
    whose linker hash is in `model.edm.known_linkers` (`last_novel`), and `require_ring_sizes` for those whose linker closes
    a ring of a size not in `model.edm.allowed_ring_sizes` (`last_ring_sizes_ok`), and `require_anchors` for those whose
    linker does not attach at `data['anchors']` alone (`last_anchors_ok`; each rank takes its rows of the template's
    anchors). `linker_types` (or, when None, `model.edm.linker_types`) as in ddpm.sample_chain: a (B, F) set gives each
    rank its rows. `linker_sizes` is refused
    (ValueError): sample the batch with ddpm.sample_chain(linker_sizes=...) and EDM.devices instead."""
    if linker_sizes is not None:
        raise ValueError("sample_chain_sharded does not take linker_sizes: use ddpm.sample_chain(linker_sizes=...), which "
                         "EDM.devices splits over local GPUs")
    from .ddpm import _anchor_extra, linker_types_mask, sampler_inputs
    from .edm import seeds_tensor
    kw = sampler_inputs(model, data, sample_fn)
    B = kw['x'].shape[0]
    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    lo, hi = shard_range(B, rank, world)
    local = slice_sampler_inputs(kw, lo, hi)
    extra = {} if nan_retries is None else {'nan_retries': nan_retries}
    if require_connected is not None:
        extra['require_connected'] = require_connected
    if require_valid is not None:
        extra['require_valid'] = require_valid
    if require_clash_free is not None:
        extra['require_clash_free'] = require_clash_free
    if require_novel is not None:
        extra['require_novel'] = require_novel
    if require_ring_sizes is not None:
        extra['require_ring_sizes'] = require_ring_sizes
    _anchor_extra(model, data, kw['x'].shape[1], require_anchors, extra)
    if 'anchors' in extra:
        extra['anchors'] = extra['anchors'][lo:hi]
    if linker_types is None:
        linker_types = getattr(model.edm, 'linker_types', None)
    types = linker_types_mask(model.edm, linker_types)
    if types is not None:
        extra['linker_types'] = types[lo:hi] if types.dim() == 2 else types
    if seeds is not None:
        chain = model.edm.sample_chain(**local, keep_frames=keep_frames, seeds=seeds_tensor(seeds, B)[lo:hi], **extra)
    else:
        chain = model.edm.sample_chain(**local, keep_frames=keep_frames, batch_slice=(lo, B) if world > 1 else None, **extra)
    if world == 1:
        return chain, kw['node_mask']
    if not gather:
        return chain, local['node_mask']
    # ranks may hold different numbers of molecules: pad to the largest slice, all_gather, trim
    counts = [shard_range(B, r, world)[1] - shard_range(B, r, world)[0] for r in range(world)]
    m = max(counts)
    pad = torch.zeros((chain.shape[0], m) + tuple(chain.shape[2:]), dtype=chain.dtype, device=chain.device)
    pad[:, :hi - lo] = chain
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    full = torch.cat([p[:, :c] for p, c in zip(parts, counts)], dim=1)
    return full, kw['node_mask']

