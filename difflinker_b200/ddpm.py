"""Outer drop-in boundary: `DDPM.sample_chain(data, sample_fn=None, keep_frames=None) -> (chain, node_mask)`
(reference: src/lightning.py:405-463; constructor wiring src/lightning.py:39-113), and `DDPM.sample_many(datas, ...)`,
which samples many such batches in shared launches.

Two ways in:
  * `DDPM(**hparams)` -- a plain nn.Module with the reference's hyper-parameter names and state_dict layout
    (`edm.gamma.gamma`, `edm.dynamics.dynamics....`), for environments without pytorch_lightning;
  * `accelerate(ddpm)` -- swaps the `.edm` of an existing *reference* DDPM (e.g. one returned by
    `DDPM.load_from_checkpoint`) for the native one in place, so generate.py / sample.py run unchanged.
Both take `devices=[...]` (or 'all') to split every sampling batch over several local GPUs from one process.
Training, datasets, metrics and visualisation are out of scope (SURVEY.md section 2).
"""
import operator

import torch
import torch.nn as nn

from . import utils
from .batching import create_templates_for_linker_generation
from .edm import EDM, InpaintingEDM, LinkerSizes, draw_seeds, seeds_tensor
from .egnn import Dynamics, DynamicsWithPockets
from .linker_size import SizeClassifier, draw_sizes
from .output import GEOM_IDX2ATOM, IDX2ATOM


def _is_geom(hp: dict):
    """The reference DDPM's is_geom (lightning.py:73): the GEOM / MOAD atom types, whose bond tables include P."""
    prefix = hp.get('train_data_prefix') or ''
    return ('geom' in prefix) or ('MOAD' in prefix)


def _build_edm(hp: dict, edge_impl='auto', is_geom=None):
    pocket = '.' in (hp.get('train_data_prefix') or '')
    graph_type = hp.get('graph_type')
    if graph_type is None:
        graph_type = '4A' if pocket else 'FC'                              # lightning.py:75-76
    activation = hp.get('activation', 'silu')
    if isinstance(activation, str):
        if activation != 'silu':
            raise Exception("activation fn not supported yet. Add it here.")  # lightning.py:23-27
        activation = nn.SiLU()
    dyn_cls = DynamicsWithPockets if pocket else Dynamics                  # lightning.py:81
    dynamics = dyn_cls(
        in_node_nf=hp['in_node_nf'], n_dims=hp['n_dims'], context_node_nf=hp['context_node_nf'],
        device=hp.get('torch_device', 'cpu'), hidden_nf=hp['hidden_nf'], activation=activation,
        n_layers=hp['n_layers'], attention=hp['attention'], tanh=hp['tanh'], norm_constant=hp['norm_constant'],
        inv_sublayers=hp['inv_sublayers'], sin_embedding=hp['sin_embedding'],
        normalization_factor=hp['normalization_factor'], aggregation_method=hp['aggregation_method'],
        model=hp['model'], normalization=hp.get('normalization'), centering=bool(hp.get('inpainting', False)),
        graph_type=graph_type, edge_impl=edge_impl)
    edm_cls = InpaintingEDM if hp.get('inpainting') else EDM                 # lightning.py:102
    return edm_cls(dynamics=dynamics, in_node_nf=hp['in_node_nf'], n_dims=hp['n_dims'],
               timesteps=hp['diffusion_steps'], noise_schedule=hp['diffusion_noise_schedule'],
               noise_precision=hp['diffusion_noise_precision'], loss_type=hp['diffusion_loss_type'],
               norm_values=hp['normalize_factors'], is_geom=_is_geom(hp) if is_geom is None else bool(is_geom))


def _keep_linker(data, template, what="start_step varies the batch's linker"):
    """The template's positions and one-hot with the linker rows of `data` filled in, for partial diffusion, which varies
    the linker the batch holds. create_templates_for_linker_generation puts a molecule's fragment atoms first and its
    linker after them; a batch whose linker rows lie elsewhere raises ValueError."""
    lm = template['linker_mask']
    n = lm.shape[1]
    same = (data['linker_mask'].shape[1] >= n and torch.equal(data['linker_mask'][:, :n].to(lm.dtype), lm)
            and not data['linker_mask'][:, n:].any())
    if not same:
        raise ValueError(f"{what}, so each molecule's linker rows must follow its fragment rows, where the sampling "
                         "template puts them")
    keep = lm.bool()
    return (torch.where(keep, data['positions'][:, :n], template['positions']),
            torch.where(keep, data['one_hot'][:, :n], template['one_hot']))


def sampler_inputs(model, data, sample_fn=None, keep_linker=False, what="start_step varies the batch's linker"):
    """What DDPM.sample_chain hands to EDM.sample_chain (lightning.py:405-452): the template batch, the context
    columns and the centred coordinates, as the keyword arguments of `edm.sample_chain`. `keep_linker` (partial diffusion)
    fills the template's linker rows with the batch's own linker before the coordinates are centred; `what` opens the
    ValueError of a batch whose linker rows do not follow its fragment rows.
    `model` needs .inpainting, .anchors_context, .train_data_prefix, .center_of_mass, .val_dataset."""
    if sample_fn is None:
        linker_sizes = data['linker_mask'].sum(1).view(-1).int()
    else:
        linker_sizes = sample_fn(data)
    return _template_inputs(model, data, linker_sizes, keep_linker, what=what)[0]


def _template_inputs(model, data, linker_sizes, keep_linker=False, n_nodes=None, what="start_step varies the batch's linker"):
    """(sampler_inputs of the template of `linker_sizes` padded to `n_nodes` rows, the centre of mass (B, 1, 3) that was
    subtracted from its coordinates)."""
    template = data if model.inpainting else create_templates_for_linker_generation(data, linker_sizes, n_nodes)
    x, h = template['positions'], template['one_hot']
    if keep_linker and not model.inpainting:
        x, h = _keep_linker(data, template, what)
    node_mask, edge_mask = template['atom_mask'], template['edge_mask']
    anchors, fragment_mask, linker_mask = template['anchors'], template['fragment_mask'], template['linker_mask']
    pocket = '.' in model.train_data_prefix
    if pocket:
        fragment_only = template['fragment_only_mask']
        pocket_only = fragment_mask - fragment_only
        parts = [anchors, fragment_only, pocket_only] if model.anchors_context else [fragment_only, pocket_only]
        context = torch.cat(parts, dim=-1)
    else:
        context = torch.cat([anchors, fragment_mask], dim=-1) if model.anchors_context else fragment_mask
    if model.inpainting:
        com_mask = node_mask
    elif type(getattr(model, 'val_dataset', None)).__name__ == 'MOADDataset' and model.center_of_mass == 'fragments':
        com_mask = template['fragment_only_mask']
    elif model.center_of_mass == 'fragments':
        com_mask = fragment_mask
    elif model.center_of_mass == 'anchors':
        com_mask = anchors
    else:
        raise NotImplementedError(model.center_of_mass)
    mean = utils.partial_mean(x, com_mask)                  # utils.remove_partial_mean_with_mask, with its mean kept
    x = x - mean * node_mask
    return dict(x=x, h=h, node_mask=node_mask, edge_mask=edge_mask, fragment_mask=fragment_mask,
                linker_mask=linker_mask, context=context), mean


def size_distribution(model, data, linker_sizes):
    """(logits (B, C) fp32 on the batch's device, size table) of `linker_sizes` for the batch `data`: a SizeClassifier's
    size_logits -- with_pocket and adjust_shape on pocket models, as generate_with_protein.py:182 calls it -- over its
    linker_id2size; all-zero logits over lo..hi for a pair (lo, hi), as generate.py:76-84 draws with torch.randint; or
    the one-entry table [n] for an int n."""
    B = data['positions'].shape[0]
    dev = data['positions'].device
    if isinstance(linker_sizes, SizeClassifier):
        pocket = '.' in (model.train_data_prefix or '')
        logits = linker_sizes.size_logits(data, with_pocket=pocket, adjust_shape=pocket)
        return logits.to(torch.float32), list(linker_sizes.linker_id2size)
    try:
        if isinstance(linker_sizes, bool):
            raise TypeError
        if isinstance(linker_sizes, (tuple, list)):
            if len(linker_sizes) != 2 or any(isinstance(v, bool) for v in linker_sizes):
                raise TypeError
            lo, hi = (operator.index(v) for v in linker_sizes)
        else:
            lo = hi = operator.index(linker_sizes)
    except TypeError:
        raise ValueError("linker_sizes is a SizeClassifier, a pair (lo, hi) of ints or an int "
                         f"(got {linker_sizes!r})") from None
    if not 0 <= lo <= hi:
        raise ValueError(f"linker_sizes needs 0 <= lo <= hi (got {lo}, {hi})")
    return torch.zeros((B, hi - lo + 1), dtype=torch.float32, device=dev), list(range(lo, hi + 1))


def _check_linker_sizes(model, sample_fn, start_step):
    if sample_fn is not None:
        raise ValueError("linker_sizes and sample_fn both choose the linker sizes: pass one of them")
    if start_step is not None:
        raise ValueError("linker_sizes does not take start_step: partial diffusion varies the batch's own linker")
    if model.inpainting:
        raise ValueError("linker_sizes does not take an inpainting model: it samples every atom, with no linker size")


def _sized_inputs(model, data, linker_sizes, seeds):
    """(sampler_inputs of the template at the sizes drawn from `seeds` (attempt 0) padded to its capacity N_cap =
    max n_frag + max(sizes), the (B,) CPU int64 seeds, the edm.LinkerSizes of the call)."""
    x = data['positions']
    if x.device.type != 'cuda':
        raise ValueError(f"linker_sizes needs CUDA inputs (got {x.device})")
    edm = model.edm
    B = x.shape[0]
    if seeds is None:
        if edm.noise_mode != 'per_molecule':
            raise ValueError("linker_sizes needs per-molecule streams: pass seeds= or set noise_mode='per_molecule' (the "
                             f"batch stream, noise_mode={edm.noise_mode!r}, cannot give one molecule new draws)")
        with torch.cuda.device(x.device):
            seeds = draw_seeds(B, x.device)
    cpu_seeds = seeds_tensor(seeds, B)
    logits, table = size_distribution(model, data, linker_sizes)
    sizes = draw_sizes(logits, table, cpu_seeds)
    fm = data['fragment_mask']
    n_frag = fm.reshape(B, fm.shape[1]).sum(1).long()
    n_cap = int(n_frag.max()) + max(table)
    kw, mean = _template_inputs(model, data, sizes, n_nodes=n_cap)
    linker_x = (torch.zeros_like(mean) - mean).reshape(B, 3)   # x - mean * node_mask of a linker row, whose x is 0
    return kw, cpu_seeds, LinkerSizes(logits, table, n_frag, linker_x)


def _final_node_mask(kw, linker_sizes, sizes):
    """The template's atom mask at the returned sizes: rows [0, n_frag + size) of every molecule."""
    n = kw['node_mask'].shape[1]
    live = linker_sizes.n_frag.to(kw['node_mask'].device) + sizes.to(kw['node_mask'].device)
    return (torch.arange(n, device=live.device)[None, :] < live[:, None]).to(kw['node_mask'].dtype)[:, :, None]


def template_anchors(model, data, n_nodes):
    """The (B, n_nodes) anchor flags of the sampling template of `data` padded to n_nodes rows: the batch's 'anchors' on
    its fragment rows, which the template keeps in place (create_templates_for_linker_generation), and 0 on every other
    row; an inpainting model samples the batch itself, so its flags are the batch's."""
    anchors = data['anchors']
    B, n_old = anchors.shape[:2]
    anchors = anchors.reshape(B, n_old)
    if model.inpainting:
        return anchors
    if n_nodes > n_old:
        anchors = torch.cat([anchors, anchors.new_zeros((B, n_nodes - n_old))], dim=1)
    anchors = anchors[:, :n_nodes]
    fm = data['fragment_mask']
    n_frag = fm.reshape(B, fm.shape[1]).sum(1).long()
    keep = torch.arange(n_nodes, device=anchors.device)[None, :] < n_frag.to(anchors.device)[:, None]
    return torch.where(keep, anchors, torch.zeros((), dtype=anchors.dtype, device=anchors.device))


def _anchor_extra(model, data, n_nodes, require_anchors, extra):
    """Adds `require_anchors` (when given) and, when the call requires the check, the template's anchors (template_anchors)
    to the keyword arguments `extra` of edm.sample_chain."""
    if require_anchors is not None:
        extra['require_anchors'] = require_anchors
    require = getattr(model.edm, 'require_anchors', False) if require_anchors is None else require_anchors
    if require is True and 'anchors' in data:
        extra['anchors'] = template_anchors(model, data, n_nodes)


def _with_anchors(model, data, kw, require_anchors):
    """The sample_many request `kw`, with the template's anchors added when the call requires the check."""
    extra = {}
    _anchor_extra(model, data, kw['x'].shape[1], require_anchors, extra)
    return dict(kw, anchors=extra['anchors']) if 'anchors' in extra else kw


def _check_start(sample_fn, start_step):
    if sample_fn is not None and start_step is not None:
        raise ValueError("start_step varies the batch's own linker, so its size is the batch's: pass no sample_fn")


def _check_fixed(sample_fn, linker_sizes, fixed_atoms):
    if fixed_atoms is None:
        return
    if sample_fn is not None:
        raise ValueError("fixed_atoms keeps atoms of the batch's own linker rows, so its linker sizes are the batch's: pass "
                         "no sample_fn")
    if linker_sizes is not None:
        raise ValueError("fixed_atoms does not take linker_sizes: a size redraw rebuilds the linker rows at new sizes")


def linker_types_mask(edm, linker_types):
    """EDM.sample_chain's `linker_types` of `linker_types` as the DDPM level takes it: None; a (F,) or (B, F) bool tensor,
    returned as it is; or element symbols (['C', 'N', 'O']), the (F,) bool set of their type channels in output.IDX2ATOM
    (ZINC), or output.GEOM_IDX2ATOM with edm.is_geom (GEOM / MOAD), the tables molecule_builder reads types with.
    ValueError for an unknown symbol, and for symbols when edm.is_geom is None."""
    if linker_types is None or torch.is_tensor(linker_types):
        return linker_types
    symbols = [linker_types] if isinstance(linker_types, str) else list(linker_types)
    if not all(isinstance(v, str) for v in symbols):
        raise ValueError(f"linker_types is a bool tensor or a list of element symbols (got {linker_types!r})")
    if edm.is_geom is None:
        raise ValueError("linker_types by element symbol needs the atom types: build the EDM with is_geom=True (GEOM / MOAD) "
                         "or False (ZINC), or set edm.is_geom")
    idx2atom = GEOM_IDX2ATOM if edm.is_geom else IDX2ATOM
    index = {a: i for i, a in idx2atom.items() if i < edm.in_node_nf}
    mask = torch.zeros(edm.in_node_nf, dtype=torch.bool)
    for a in symbols:
        if a not in index:
            raise ValueError(f"linker_types: unknown element {a!r}; this model's types are {sorted(index, key=index.get)}")
        mask[index[a]] = True
    return mask


def _sampler_kw(model, data, sample_fn, start_step, fixed_atoms):
    """sampler_inputs of a call, with the batch's own linker rows for start_step or fixed_atoms, and the latter as
    EDM.sample_chain's `fixed_atoms` of the template's rows (the batch's linker rows keep their place in it)."""
    if fixed_atoms is None:
        return sampler_inputs(model, data, sample_fn, keep_linker=start_step is not None)
    what = "start_step varies the batch's linker" if start_step is not None else "fixed_atoms keeps the batch's linker atoms"
    kw = sampler_inputs(model, data, sample_fn, keep_linker=True, what=what)
    B, n = kw['x'].shape[:2]
    flags = fixed_atoms.detach().reshape(B, -1) if torch.is_tensor(fixed_atoms) else fixed_atoms
    if torch.is_tensor(flags) and flags.shape[1] > n:
        if flags[:, n:].any():
            raise ValueError("fixed_atoms flags a row beyond the sampling template's, which holds the batch's linker rows")
        flags = flags[:, :n]
    return dict(kw, fixed_atoms=flags)


def sample_chain(model, data, sample_fn=None, keep_frames=None, seeds=None, nan_retries=None, require_connected=None,
                 start_step=None, require_valid=None, require_clash_free=None, linker_sizes=None, require_unique=None,
                 require_novel=None, exclude_hashes=None, resamplings=None, require_ring_sizes=None, require_anchors=None,
                 clash_guidance=None, solver=None, fixed_atoms=None, linker_types=None):
    """Body of DDPM.sample_chain (lightning.py:405-463), shared by `DDPM` below and by accelerated reference
    modules (`model` additionally needs .edm). `seeds`: one per molecule, see EDM.sample_chain. Linker sizes drawn by
    `sample_fn` still come from the batch's generator: to replay a molecule, keep its template or its linker size.
    `nan_retries`: rounds that resample only the diverged molecules (EDM.sample_chain; None uses `model.edm.nan_retries`).
    `require_connected`: the rounds also resample the disconnected molecules (None uses `model.edm.require_connected`).
    `require_valid`: ... and the molecules with an atom beyond its valence (None uses `model.edm.require_valid`).
    `require_clash_free`: ... and, on pocket graphs, the molecules whose linker clashes with the pocket (None uses
    `model.edm.require_clash_free`).
    `require_unique`: ... and the molecules whose bond graph repeats a batch-mate's (None uses `model.edm.require_unique`);
    `exclude_hashes` (with it) also counts those graph hashes as taken.
    `require_novel`: ... and the molecules whose linker hash is in `model.edm.known_linkers` (None uses
    `model.edm.require_novel`).
    `require_ring_sizes`: ... and the molecules whose linker closes a smallest ring of a size not in
    `model.edm.allowed_ring_sizes` (None uses `model.edm.require_ring_sizes`).
    `require_anchors`: ... and the molecules whose linker does not attach by exactly one bond at each anchor of
    `data['anchors']` and nowhere else (None uses `model.edm.require_anchors`); the template's flags (template_anchors,
    at the padded size with `linker_sizes`) are passed as EDM.sample_chain's `anchors`.
    `start_step` = t0 (partial diffusion, EDM.sample_chain): the template of sample_fn=None with the batch's own linker
    positions and atom types on its linker rows, sampled from step t0 -- or from one step per molecule, a 1-D sequence or
    integer tensor (EDM.sample_chain); ValueError with a sample_fn, or when the batch's linker rows do not directly follow
    its fragment rows.
    `linker_sizes` -- a SizeClassifier, a pair (lo, hi) or an int (size_distribution) -- draws molecule b's linker size from
    its own seed (dl_size_draw; `seeds`, or draw_seeds with noise_mode='per_molecule'), builds the template at those sizes
    padded to its capacity N_cap = max n_frag + max(sizes), and makes every recovery round redraw the size of each row it
    resamples from that round's seed (EDM.sample_chain). A row's size and chain are then functions of `last_seeds[b]`:
    molecule b alone, its input padded to the same number of rows (the size model mean-pools over the padding), with
    seeds=[last_seeds[b]], gives the same size and row. `model.edm.last_sizes` holds the sizes, and the returned node_mask
    is the template's at those sizes. ValueError with sample_fn, start_step, an inpainting model, host inputs, the batch
    stream without seeds, and where EDM.sample_chain refuses it.
    `resamplings` = r: r RePaint passes per reverse step of an inpainting model (InpaintingEDM.sample_chain; None uses
    `model.edm.resamplings`).
    `clash_guidance` = (scale, steps): push the linker atoms out of the pocket at the last `steps` reverse steps
    (EDM.sample_chain; None uses `model.edm.clash_guidance`).
    `solver` = 'ancestral', 'ddim' or 'dpmpp_2m': the reverse update (EDM.sample_chain; None uses `model.edm.solver`).
    `fixed_atoms` ((B, N) or (B, N, 1), non-zero on the batch's linker atoms to keep): the template of sample_fn=None with
    the batch's own linker rows, as for start_step, of which the flagged atoms are kept and the rest sampled around them
    (EDM.sample_chain); ValueError with a sample_fn or linker_sizes, and when the batch's linker rows do not directly follow
    its fragment rows.
    `linker_types`: the types the linker atoms may take (EDM.sample_chain; None uses `model.edm.linker_types`), also as
    element symbols, ['C', 'N', 'O'] (linker_types_mask)."""
    _check_start(sample_fn, start_step)
    linker_types = linker_types_mask(model.edm, linker_types)
    _check_fixed(sample_fn, linker_sizes, fixed_atoms)
    if linker_sizes is not None:
        _check_linker_sizes(model, sample_fn, start_step)
        kw, seeds, sized = _sized_inputs(model, data, linker_sizes, seeds)
    else:
        kw, sized = _sampler_kw(model, data, sample_fn, start_step, fixed_atoms), None
    extra = {} if seeds is None else {'seeds': seeds}
    if sized is not None:
        extra['linker_sizes'] = sized
    if nan_retries is not None:
        extra['nan_retries'] = nan_retries
    if require_connected is not None:
        extra['require_connected'] = require_connected
    if require_valid is not None:
        extra['require_valid'] = require_valid
    if require_clash_free is not None:
        extra['require_clash_free'] = require_clash_free
    if require_unique is not None:
        extra['require_unique'] = require_unique
    if require_novel is not None:
        extra['require_novel'] = require_novel
    if require_ring_sizes is not None:
        extra['require_ring_sizes'] = require_ring_sizes
    _anchor_extra(model, data, kw['x'].shape[1], require_anchors, extra)
    if exclude_hashes is not None:
        extra['exclude_hashes'] = exclude_hashes
    if start_step is not None:
        extra['start_step'] = start_step
    if resamplings is not None:
        extra['resamplings'] = resamplings
    if clash_guidance is not None:
        extra['clash_guidance'] = clash_guidance
    if solver is not None:
        extra['solver'] = solver
    if linker_types is not None:
        extra['linker_types'] = linker_types
    chain = model.edm.sample_chain(**kw, keep_frames=keep_frames, **extra)
    if sized is not None:
        return chain, _final_node_mask(kw, sized, model.edm.last_sizes)
    return chain, kw['node_mask']


def _with_types(request, linker_types):
    """The request with its `linker_types` key when it has a set."""
    return request if linker_types is None else dict(request, linker_types=linker_types)


def sample_many(model, datas, sample_fn=None, keep_frames=None, seeds=None, nan_retries=None, require_connected=None,
                max_molecules=256, start_step=None, require_valid=None, require_clash_free=None, linker_sizes=None,
                require_novel=None, resamplings=None, require_ring_sizes=None, require_anchors=None, clash_guidance=None,
                solver=None, fixed_atoms=None, linker_types=None):
    """The body of sample_chain for many batches `datas` at once, sampled in shared launches by EDM.sample_many: returns
    [(chain_k, node_mask_k)] in the order of `datas`, each equal to what sample_chain(model, datas[k], ...) returns (with
    seeds[k]) in the sense of EDM.sample_many. `model` as for sample_chain, so accelerated reference modules take it too.
    `sample_fn`, and with noise_mode='per_molecule' and no `seeds` draw_seeds, are called once per batch, in the order the
    sequential sample_chain calls call them: linker sizes, seeds and the generator's final state are theirs. `start_step`,
    one for every batch, as in sample_chain. `linker_sizes`, one for every batch, as in sample_chain: each batch's sizes
    are drawn from its own seeds and its template padded to its own N_cap, so packing changes neither;
    `edm.last_sizes_many` holds them. `resamplings` and `require_anchors` as in sample_chain: each request then holds its
    batch's template anchors. `clash_guidance` and `solver` as in sample_chain. `fixed_atoms`, one per batch (or None for a
    batch that keeps none), as in sample_chain: each request then holds its batch's flags. `linker_types` as in
    sample_chain, one set for every batch, or a list of one per batch (None for a batch that takes `edm.linker_types`):
    each request then holds its batch's set."""
    _check_start(sample_fn, start_step)
    per_batch = isinstance(linker_types, (list, tuple)) and not all(isinstance(v, str) for v in linker_types)
    if per_batch and len(linker_types) != len(datas):
        raise ValueError(f"linker_types holds {len(linker_types)} entries for {len(datas)} batches")
    types = ([linker_types_mask(model.edm, v) for v in linker_types] if per_batch
             else [linker_types_mask(model.edm, linker_types)] * len(datas))
    if fixed_atoms is not None:
        if len(fixed_atoms) != len(datas):
            raise ValueError(f"fixed_atoms holds {len(fixed_atoms)} entries for {len(datas)} batches")
        for f in fixed_atoms:
            _check_fixed(sample_fn, linker_sizes, f)
    edm = model.edm
    if linker_sizes is not None:
        _check_linker_sizes(model, sample_fn, start_step)
        if seeds is not None and len(seeds) != len(datas):
            raise ValueError(f"seeds holds {len(seeds)} lists for {len(datas)} batches")
        sized = [_sized_inputs(model, data, linker_sizes, None if seeds is None else seeds[k])
                 for k, data in enumerate(datas)]
        extra = {} if nan_retries is None else {'nan_retries': nan_retries}
        for name, v in (('require_connected', require_connected), ('require_valid', require_valid),
                        ('require_clash_free', require_clash_free), ('require_novel', require_novel),
                        ('require_ring_sizes', require_ring_sizes), ('clash_guidance', clash_guidance),
                        ('solver', solver)):
            if v is not None:
                extra[name] = v
        requests = [_with_types(_with_anchors(model, data, kw, require_anchors), m) for data, (kw, _, _), m
                    in zip(datas, sized, types)]
        if require_anchors is not None:
            extra['require_anchors'] = require_anchors
        chains = edm.sample_many(requests, keep_frames=keep_frames, seeds=[s for _, s, _ in sized],
                                 max_molecules=max_molecules, linker_sizes=[ls for _, _, ls in sized], **extra)
        return [(chain, _final_node_mask(kw, ls, sizes))
                for chain, (kw, _, ls), sizes in zip(chains, sized, edm.last_sizes_many)]
    derive = seeds is None and edm.noise_mode == 'per_molecule'
    requests, drawn = [], []
    for k, data in enumerate(datas):
        kw = _sampler_kw(model, data, sample_fn, start_step, None if fixed_atoms is None else fixed_atoms[k])
        requests.append(_with_types(_with_anchors(model, data, kw, require_anchors), types[k]))
        x = kw['x']
        if derive and x.is_cuda:                # a host batch is refused by EDM.sample_many
            with torch.cuda.device(x.device):
                drawn.append(draw_seeds(x.shape[0], x.device))
    if derive and len(drawn) == len(requests):
        seeds = drawn
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
    if require_anchors is not None:
        extra['require_anchors'] = require_anchors
    if start_step is not None:
        extra['start_step'] = start_step
    if resamplings is not None:
        extra['resamplings'] = resamplings
    if clash_guidance is not None:
        extra['clash_guidance'] = clash_guidance
    if solver is not None:
        extra['solver'] = solver
    chains = edm.sample_many(requests, keep_frames=keep_frames, seeds=seeds, max_molecules=max_molecules, **extra)
    return [(chain, kw['node_mask']) for chain, kw in zip(chains, requests)]


class DDPM(nn.Module):
    """Hyper-parameter-compatible stand-in for the Lightning module (sampling API only)."""
    train_dataset = None
    val_dataset = None
    test_dataset = None
    FRAMES = 100

    def __init__(
        self,
        in_node_nf, n_dims, context_node_nf, hidden_nf, activation, tanh, n_layers, attention, norm_constant,
        inv_sublayers, sin_embedding, normalization_factor, aggregation_method,
        diffusion_steps, diffusion_noise_schedule, diffusion_noise_precision, diffusion_loss_type,
        normalize_factors, include_charges, model,
        data_path=None, train_data_prefix='', val_data_prefix='', batch_size=64, lr=2e-4, torch_device='cpu',
        test_epochs=None, n_stability_samples=None,
        normalization=None, log_iterations=None, samples_dir=None, data_augmentation=False,
        center_of_mass='fragments', inpainting=False, anchors_context=True, graph_type=None, edge_impl='auto',
        devices=None,
    ):
        super().__init__()
        self.hparams = {k: v for k, v in locals().items() if k not in ('self', '__class__', 'edge_impl', 'devices')}
        self.data_path, self.train_data_prefix, self.val_data_prefix = data_path, train_data_prefix, val_data_prefix
        self.batch_size, self.lr, self.torch_device = batch_size, lr, torch_device
        self.include_charges = include_charges
        self.samples_dir = samples_dir
        self.center_of_mass = center_of_mass
        self.inpainting = inpainting
        self.loss_type = diffusion_loss_type
        self.n_dims = n_dims
        self.num_classes = in_node_nf - include_charges
        self.anchors_context = anchors_context
        self.is_geom = ('geom' in train_data_prefix) or ('MOAD' in train_data_prefix)
        self.edm = _build_edm(self.hparams, edge_impl=edge_impl)
        self.edm.devices = devices          # EDM.devices: split each sampling batch over these CUDA devices

    def sample_chain(self, data, sample_fn=None, keep_frames=None, seeds=None, nan_retries=None, require_connected=None,
                     start_step=None, require_valid=None, require_clash_free=None, linker_sizes=None, require_unique=None,
                     require_novel=None, exclude_hashes=None, resamplings=None, require_ring_sizes=None,
                     require_anchors=None, clash_guidance=None, solver=None, fixed_atoms=None, linker_types=None):
        return sample_chain(self, data, sample_fn=sample_fn, keep_frames=keep_frames, seeds=seeds, nan_retries=nan_retries,
                            require_connected=require_connected, start_step=start_step, require_valid=require_valid,
                            require_clash_free=require_clash_free, linker_sizes=linker_sizes, require_unique=require_unique,
                            require_novel=require_novel, exclude_hashes=exclude_hashes, resamplings=resamplings,
                            require_ring_sizes=require_ring_sizes, require_anchors=require_anchors,
                            clash_guidance=clash_guidance, solver=solver, fixed_atoms=fixed_atoms,
                            linker_types=linker_types)

    def sample_many(self, datas, sample_fn=None, keep_frames=None, seeds=None, nan_retries=None, require_connected=None,
                    max_molecules=256, start_step=None, require_valid=None, require_clash_free=None, linker_sizes=None,
                    require_novel=None, resamplings=None, require_ring_sizes=None, require_anchors=None,
                    clash_guidance=None, solver=None, fixed_atoms=None, linker_types=None):
        return sample_many(self, datas, sample_fn=sample_fn, keep_frames=keep_frames, seeds=seeds, nan_retries=nan_retries,
                           require_connected=require_connected, max_molecules=max_molecules, start_step=start_step,
                           require_valid=require_valid, require_clash_free=require_clash_free, linker_sizes=linker_sizes,
                           require_novel=require_novel, resamplings=resamplings, require_ring_sizes=require_ring_sizes,
                           require_anchors=require_anchors, clash_guidance=clash_guidance, solver=solver,
                           fixed_atoms=fixed_atoms, linker_types=linker_types)

    def forward(self, *a, **k):
        raise NotImplementedError("training is outside the difflinker_b200 hot path")

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path, map_location=None, strict=True, **overrides):
        """`DDPM.load_from_checkpoint(args.model, map_location=device)` (generate.py:101, sample.py:84) without
        pytorch_lightning: a Lightning checkpoint is a dict with `hyper_parameters` (what `save_hyperparameters()` stored,
        lightning.py:51) and `state_dict`. Keyword overrides replace saved hyper-parameters, as in Lightning."""
        return _load_lightning_checkpoint(cls, checkpoint_path, map_location, strict, overrides)


def _load_lightning_checkpoint(cls, checkpoint_path, map_location, strict, overrides):
    try:
        ckpt = torch.load(checkpoint_path, map_location='cpu', weights_only=False)
    except TypeError:                                        # older torch without the weights_only argument
        ckpt = torch.load(checkpoint_path, map_location='cpu')
    if 'state_dict' not in ckpt or 'hyper_parameters' not in ckpt:
        raise KeyError("not a Lightning checkpoint: expected the keys 'state_dict' and 'hyper_parameters'")
    hp = dict(ckpt['hyper_parameters'])
    hp.update(overrides)
    model = cls(**hp)
    model.load_state_dict(ckpt['state_dict'], strict=strict)
    if map_location is not None:
        model = model.to(map_location)
    return model


def accelerate(ddpm, edge_impl='auto', devices=None):
    """Replace `ddpm.edm` of a *reference* DDPM (src/lightning.py) by the native EDM, copying its weights
    (strict state_dict match) and its possibly overridden `.T` (generate.py:103-104). Returns `ddpm`.
    `devices` (a list of CUDA device indices, or 'all') makes `ddpm.sample_chain` split each batch over those devices from
    this one process (EDM.devices); None samples on the data's device."""
    hp = dict(ddpm.hparams) if hasattr(ddpm, 'hparams') and len(dict(ddpm.hparams)) else None
    if hp is None:
        raise ValueError("the module carries no hparams; construct difflinker_b200.DDPM(**hparams) instead")
    new_edm = _build_edm(hp, edge_impl=edge_impl, is_geom=getattr(ddpm, 'is_geom', None))
    new_edm.load_state_dict(ddpm.edm.state_dict(), strict=True)
    new_edm.T = ddpm.edm.T
    new_edm.devices = devices
    ddpm.edm = new_edm
    return ddpm
