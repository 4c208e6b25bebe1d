"""Drop-in `Dynamics` / `DynamicsWithPockets` (reference: src/egnn.py:323-596) backed by the native sm_90a engine.

The classes keep the reference's constructor kwargs, `forward(t, xh, node_mask, linker_mask, edge_mask, context)`
signature, exception behaviour (`FoundNaNException`) and -- so published checkpoints load with strict=True --
its `state_dict` key names (`dynamics.embedding.weight`, `dynamics.e_block_0.gcl_0.edge_mlp.0.weight`, ...).
The parameter containers below exist only to own tensors under those names (and to initialise them in the
reference's construction order, so `torch.manual_seed(s); Dynamics(...)` yields the same random weights);
all arithmetic happens in libdifflinker_b200.so.  There is no CPU fallback.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _native
from .utils import FoundNaNException, nan_exception_class


SIN_EMBEDDING_DIM = 12   # SinusoidsEmbeddingNew().dim: sin and cos of 6 frequencies (src/egnn.py:281-286)


class _GCLParams(nn.Module):
    """Parameters of one GCL (src/egnn.py:19-30): edge_mlp.{0,2}, node_mlp.{0,2}."""

    def __init__(self, hidden_nf, edges_in_d, act):
        super().__init__()
        self.edge_mlp = nn.Sequential(nn.Linear(2 * hidden_nf + edges_in_d, hidden_nf), act,
                                      nn.Linear(hidden_nf, hidden_nf), act)
        self.node_mlp = nn.Sequential(nn.Linear(2 * hidden_nf, hidden_nf), act, nn.Linear(hidden_nf, hidden_nf))


class _CoordParams(nn.Module):
    """Parameters of one EquivariantUpdate (src/egnn.py:89-97): coord_mlp.{0,2,4}; the final H->1 layer has no
    bias and is created first with xavier gain 1e-3."""

    def __init__(self, hidden_nf, edges_in_d, act):
        super().__init__()
        last = nn.Linear(hidden_nf, 1, bias=False)
        nn.init.xavier_uniform_(last.weight, gain=0.001)
        self.coord_mlp = nn.Sequential(nn.Linear(2 * hidden_nf + edges_in_d, hidden_nf), act,
                                       nn.Linear(hidden_nf, hidden_nf), act, last)


class _BlockParams(nn.Module):
    def __init__(self, hidden_nf, inv_sublayers, act, edge_feat_nf):
        super().__init__()
        for s in range(inv_sublayers):
            self.add_module(f"gcl_{s}", _GCLParams(hidden_nf, edge_feat_nf, act))
        self.add_module("gcl_equiv", _CoordParams(hidden_nf, edge_feat_nf, act))


class _EGNNParams(nn.Module):
    """Parameter tree of EGNN (src/egnn.py:195-212): with sin_embedding every first layer reads 2 x 12 sinusoidal
    features instead of the two distances (SinusoidsEmbeddingNew has no parameters)."""

    def __init__(self, in_node_nf, hidden_nf, n_layers, inv_sublayers, act, sin_embedding=False):
        super().__init__()
        edge_feat_nf = 2 * SIN_EMBEDDING_DIM if sin_embedding else 2
        self.embedding = nn.Linear(in_node_nf, hidden_nf)
        self.embedding_out = nn.Linear(hidden_nf, in_node_nf)
        for l in range(n_layers):
            self.add_module(f"e_block_{l}", _BlockParams(hidden_nf, inv_sublayers, act, edge_feat_nf))


class Dynamics(nn.Module):
    def __init__(
            self, n_dims, in_node_nf, context_node_nf, hidden_nf=64, device='cpu', activation=nn.SiLU(),
            n_layers=4, attention=False, condition_time=True, tanh=False, norm_constant=0, inv_sublayers=2,
            sin_embedding=False, normalization_factor=100, aggregation_method='sum', model='egnn_dynamics',
            normalization=None, centering=False, graph_type='FC', edge_impl='auto',
    ):
        super().__init__()
        unsupported = []
        if model != 'egnn_dynamics': unsupported.append(f"model={model!r}")
        if attention: unsupported.append("attention=True")
        if aggregation_method not in _native.AGGREGATIONS: unsupported.append(f"aggregation_method={aggregation_method!r}")
        # `normalization` is accepted and ignored exactly as the reference does for model='egnn_dynamics': it is only
        # forwarded to GNN (src/egnn.py:355-368); every configs/*.yml and train_difflinker.py's default set
        # normalization='batch_norm', so every published checkpoint carries it in its hyper-parameters.
        if not isinstance(activation, nn.SiLU): unsupported.append(f"activation={activation!r}")
        if unsupported:
            # no published config (configs/*.yml) uses these; refuse rather than silently differ
            raise NotImplementedError("difflinker_b200 hot path does not implement: " + ", ".join(unsupported))
        self.device = device
        self.n_dims = n_dims
        self.in_node_nf = in_node_nf
        self.context_node_nf = context_node_nf
        self.hidden_nf = hidden_nf
        self.n_layers = n_layers
        self.inv_sublayers = inv_sublayers
        self.condition_time = condition_time
        self.norm_constant = norm_constant
        self.normalization_factor = normalization_factor
        self.aggregation_method = aggregation_method
        self.tanh = tanh
        self.sin_embedding = sin_embedding
        self.model = model
        self.centering = centering
        self.graph_type = graph_type
        self.edge_impl = edge_impl
        self.dynamics = _EGNNParams(in_node_nf + context_node_nf + int(condition_time), hidden_nf, n_layers,
                                    inv_sublayers, activation, sin_embedding=bool(sin_embedding))
        self._engines = {}          # (device index, replica) -> (handle, (edge_impl, weights version) uploaded)
        self._host_weights = None   # (weights version, [(name, fp32 CPU tensor)]): read once, uploaded to every engine

    # ---- native engine management -------------------------------------------------------------------------
    def _weights_version(self):
        return tuple((p.data_ptr(), p._version) for p in self.dynamics.parameters())

    def _weights_on_host(self, version):
        """The parameters as fp32 host tensors under their C-ABI names, read from the module once per weights version."""
        if self._host_weights is None or self._host_weights[0] != version:
            self._host_weights = (version, [(f"dynamics.{name}".encode(), p.detach().to(device='cpu', dtype=torch.float32).contiguous())
                                            for name, p in self.dynamics.state_dict().items()])
        return self._host_weights[1]

    def _check_graph_type(self):
        assert self.graph_type == 'FC'  # src/egnn.py:383

    def dl_config(self, device_index: int):
        """The dl_config the engine on CUDA device `device_index` is created with."""
        return _native.DLConfig(
            n_dims=self.n_dims, in_node_nf=self.in_node_nf, context_node_nf=self.context_node_nf,
            hidden_nf=self.hidden_nf, n_layers=self.n_layers, inv_sublayers=self.inv_sublayers,
            condition_time=int(self.condition_time), centering=int(self.centering),
            graph_type=_native.GRAPH_TYPES[self.graph_type], device=device_index,
            edge_impl=_native.EDGE_IMPLS[self.edge_impl], norm_constant=float(self.norm_constant),
            normalization_factor=float(self.normalization_factor))

    def egnn_options(self):
        """The EGNN options the engine is created with (dl_create_ex)."""
        return _native.DLEgnnOptions(tanh=int(bool(self.tanh)), coords_range=_native.COORDS_RANGE,
                                     sin_embedding=int(bool(self.sin_embedding)),
                                     aggregation=_native.AGGREGATIONS[self.aggregation_method])

    def engine(self, device_index: int):
        """Creates the native engine on first use and re-uploads weights whenever a parameter changed. A module used on one
        device keeps one engine: engines of other devices (the device the module was on before, or the slices of a split
        batch) are destroyed."""
        self._release_all_but({(device_index, 0)})
        return self._engine_at(device_index, 0)

    def engines(self, slots):
        """The engines of `slots` [(device, replica)], for a batch split over several devices (EDM.devices): replica > 0 are
        further engines on the same device, for a device listed more than once. Every engine gets the same host copy of the
        weights; the module's engines outside `slots` are destroyed."""
        self._release_all_but(set(slots))
        out = []
        for device_index, replica in slots:
            with torch.cuda.device(device_index):            # dl_create_ex selects the device on the calling thread
                out.append(self._engine_at(device_index, replica))
        return out

    def _engine_at(self, device_index: int, replica: int):
        lib = _native.load_library()
        slot, key = (device_index, replica), (self.edge_impl, self._weights_version())
        handle, uploaded = self._engines.get(slot, (None, None))
        if handle is not None and uploaded == key:
            return handle
        if handle is None or uploaded is None or uploaded[0] != key[0]:
            self._destroy(slot)
            cfg = self.dl_config(device_index)
            handle = C.c_void_p()
            _native.check(lib.dl_create_ex(C.byref(cfg), C.byref(self.egnn_options()), C.byref(handle)), "dl_create_ex")
            self._engines[slot] = (handle, None)
        for name, w in self._weights_on_host(key[1]):
            _native.check(lib.dl_set_weight(handle, name, w.data_ptr(), w.numel()), f"dl_set_weight({name.decode()})")
        _native.check(lib.dl_finalize_weights(handle), "dl_finalize_weights")
        self._engines[slot] = (handle, key)
        return handle

    def _release_all_but(self, keep):
        for slot in [slot for slot in self._engines if slot not in keep]:
            self._destroy(slot)

    def _destroy(self, slot):
        handle, _ = self._engines.pop(slot, (None, None))
        if handle is not None:
            _native.load_library().dl_destroy(handle)

    def close(self):
        for slot in list(getattr(self, '_engines', {})):
            self._destroy(slot)
        self._host_weights = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _device_index(t: torch.Tensor) -> int:
        if not torch.cuda.is_available():
            raise RuntimeError("difflinker_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        if t.is_cuda:
            return t.device.index if t.device.index is not None else torch.cuda.current_device()
        return torch.cuda.current_device()

    # ---- reference-facing call ----------------------------------------------------------------------------
    def forward(self, t, xh, node_mask, linker_mask, edge_mask, context):
        """
        - t: (B, 1) or a single element
        - xh: (B, N, 3 + nf)
        - node_mask: (B, N, 1)
        - linker_mask: (B, N, 1) or None
        - edge_mask: (B*N*N, 1) for FC graphs; the (B*N,) molecule-index vector for pocket graphs
        - context: (B, N, C)
        Tensors may live on a CUDA device (stream-ordered, zero-copy) or on the host (copied by the engine).
        """
        self._check_graph_type()
        lib = _native.load_library()
        bs, n_nodes = xh.shape[0], xh.shape[1]
        dev = xh.device
        eng = self.engine(self._device_index(xh))

        def prep(v, dtype):
            return None if v is None else v.detach().to(device=dev, dtype=dtype).contiguous()

        xh_c = prep(xh, torch.float32)
        nm = prep(node_mask.reshape(bs, n_nodes), torch.int8)
        lm = None if linker_mask is None else prep(linker_mask.reshape(bs, n_nodes), torch.float32)
        em = None
        if self.graph_type == 'FC' and edge_mask is not None:
            em = prep(edge_mask.reshape(-1), torch.int8)
            if em.numel() != bs * n_nodes * n_nodes:
                raise ValueError(f"edge_mask has {em.numel()} entries, expected B*N*N = {bs * n_nodes * n_nodes}")
        ctx = None if context is None else prep(context.reshape(bs, n_nodes, self.context_node_nf), torch.float32)
        t_c = None if t is None else prep(t.reshape(-1), torch.float32)
        if t_c is not None and t_c.numel() not in (1, bs):
            raise ValueError("t must have 1 or B elements")
        out = torch.empty_like(xh_c)
        flags = torch.zeros(bs, dtype=torch.int32, device=dev)
        ptr = lambda v: None if v is None else v.data_ptr()
        if dev.type == 'cuda':
            with torch.cuda.device(dev):
                stream = torch.cuda.current_stream(dev).cuda_stream
                st = lib.dl_dynamics_forward(eng, bs, n_nodes, ptr(t_c), 0 if t_c is None else t_c.numel(), ptr(xh_c),
                                             ptr(nm), ptr(lm), ptr(em), ptr(ctx), ptr(out), ptr(flags), stream)
                _native.check(st, "dl_dynamics_forward")
                bad = bool(flags.any().item())  # the reference also syncs here (src/egnn.py:441)
        else:
            st = lib.dl_dynamics_forward_host(eng, bs, n_nodes, ptr(t_c), 0 if t_c is None else t_c.numel(), ptr(xh_c),
                                              ptr(nm), ptr(lm), ptr(em), ptr(ctx), ptr(out), ptr(flags))
            _native.check(st, "dl_dynamics_forward_host")
            bad = st == _native.DL_NAN_DETECTED
        if bad:
            raise nan_exception_class()(flags=flags.cpu().tolist())
        return out

    def get_edges(self, n_nodes, batch_size):
        """Kept for API compatibility (src/egnn.py:449-467); the engine never materialises an edge list."""
        i = torch.arange(n_nodes).repeat_interleave(n_nodes).repeat(batch_size)
        j = torch.arange(n_nodes).repeat(n_nodes * batch_size)
        off = (torch.arange(batch_size) * n_nodes).repeat_interleave(n_nodes * n_nodes)
        return [(i + off).to(self.device), (j + off).to(self.device)]


class DynamicsWithPockets(Dynamics):
    """Cut-off graphs ('4A', 'FC-4A', 'FC-10A-4A', src/egnn.py:470-596): the edge predicate is evaluated inside
    the edge kernel from the call's input coordinates instead of building a (B*N)^2 adjacency."""

    def _check_graph_type(self):
        assert self.graph_type in ['4A', 'FC-4A', 'FC-10A-4A']  # src/egnn.py:495
