"""Linker-size classifier: drop-in for `src/linker_size.py::SizeGNN` + `src/linker_size_lightning.py::SizeClassifier`
(inference). `SizeClassifier.forward(data, return_loss=False)` -- the call `generate.py:91` makes in its `sample_fn` --
runs as one native pass (`dl_sizegnn_forward`); parameter names and construction order are the reference's, so a
reference checkpoint's `state_dict` loads with `strict=True`. No CPU fallback.
"""
import ctypes as C
import operator

import torch
import torch.nn as nn
from torch.nn.functional import cross_entropy

from . import _native
from .batching import collate

ZINC_TRAIN_LINKER_ID2SIZE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 12]                             # src/const.py:181
ZINC_TRAIN_LINKER_SIZE2ID = {size: idx for idx, size in enumerate(ZINC_TRAIN_LINKER_ID2SIZE)}
GEOM_TRAIN_LINKER_ID2SIZE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19,   # src/const.py:200-203
                             20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 36, 38, 41]
GEOM_TRAIN_LINKER_SIZE2ID = {size: idx for idx, size in enumerate(GEOM_TRAIN_LINKER_ID2SIZE)}
SIZE_GNN_WIDTHS = (128, 256)    # hidden_nf values the native SizeGNN has kernels for


class _GCLParams(nn.Module):
    """Parameter container with the layout of egnn.GCL(edges_in_d=1, activation=ReLU) (src/egnn.py:10-43)."""

    def __init__(self, hidden_nf, normalization):
        super().__init__()
        self.edge_mlp = nn.Sequential(nn.Linear(2 * hidden_nf + 1, hidden_nf), nn.ReLU(), nn.Linear(hidden_nf, hidden_nf),
                                      nn.ReLU())
        if normalization is None:
            self.node_mlp = nn.Sequential(nn.Linear(2 * hidden_nf, hidden_nf), nn.ReLU(), nn.Linear(hidden_nf, hidden_nf))
        elif normalization == 'batch_norm':
            self.node_mlp = nn.Sequential(nn.Linear(2 * hidden_nf, hidden_nf), nn.BatchNorm1d(hidden_nf), nn.ReLU(),
                                          nn.Linear(hidden_nf, hidden_nf), nn.BatchNorm1d(hidden_nf))
        else:
            raise NotImplementedError(normalization)


def _fold_bn(linear, bn):
    """Eval-mode BatchNorm1d after a Linear is an affine map per output channel."""
    w, b = linear.weight.detach().float(), linear.bias.detach().float()
    if bn is None:
        return w, b
    g = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    return w * g[:, None], (b - bn.running_mean.detach().float()) * g + bn.bias.detach().float()


class SizeGNN(nn.Module):
    """src/linker_size.py:45-91. Holds the parameters; the arithmetic happens in the native engine."""

    def __init__(self, in_node_nf, hidden_nf, out_node_nf, n_layers, normalization, device='cpu'):
        super().__init__()
        if hidden_nf not in SIZE_GNN_WIDTHS:
            raise NotImplementedError(f"the native SizeGNN supports hidden_nf = 128 (train_size_gnn.py:19) or 256 (the "
                                      f"README's size-model recipe), not {hidden_nf}")
        self.in_node_nf, self.hidden_nf, self.out_node_nf, self.n_layers = in_node_nf, hidden_nf, out_node_nf, n_layers
        self.normalization = normalization
        self.embedding_in = nn.Linear(in_node_nf, hidden_nf)
        self.gcl1 = _GCLParams(hidden_nf, normalization)
        self.gcl_layers = nn.ModuleList([_GCLParams(hidden_nf, normalization) for _ in range(n_layers - 1)])
        self.embedding_out = nn.Linear(hidden_nf, out_node_nf)
        self._engine = None
        self._engine_key = None

    def _weights_version(self):
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))

    def engine(self, device_index):
        lib = _native.load_library()
        key = (device_index, self._weights_version(), self.training)
        if self._engine is not None and self._engine_key == key:
            return self._engine
        if self.normalization == 'batch_norm' and self.training:
            raise RuntimeError("the native SizeGNN folds BatchNorm in eval mode only: call .eval() first")
        self.close()
        cfg = _native.DLSizeGNNConfig(in_node_nf=self.in_node_nf, hidden_nf=self.hidden_nf, out_node_nf=self.out_node_nf,
                                      n_layers=self.n_layers, device=device_index)
        handle = C.c_void_p()
        _native.check(lib.dl_sizegnn_create(C.byref(cfg), C.byref(handle)), "dl_sizegnn_create")

        def put(name, tensor):
            t = tensor.detach().float().cpu().contiguous()
            _native.check(lib.dl_sizegnn_set_weight(handle, name.encode(), C.c_void_p(t.data_ptr()), t.numel()),
                          f"dl_sizegnn_set_weight({name})")

        put("embedding_in.weight", self.embedding_in.weight); put("embedding_in.bias", self.embedding_in.bias)
        put("embedding_out.weight", self.embedding_out.weight); put("embedding_out.bias", self.embedding_out.bias)
        for l, gcl in enumerate([self.gcl1] + list(self.gcl_layers)):
            put(f"layer{l}.edge_mlp.0.weight", gcl.edge_mlp[0].weight); put(f"layer{l}.edge_mlp.0.bias", gcl.edge_mlp[0].bias)
            put(f"layer{l}.edge_mlp.2.weight", gcl.edge_mlp[2].weight); put(f"layer{l}.edge_mlp.2.bias", gcl.edge_mlp[2].bias)
            if self.normalization is None:
                w3, b3 = _fold_bn(gcl.node_mlp[0], None)
                w4, b4 = _fold_bn(gcl.node_mlp[2], None)
            else:
                w3, b3 = _fold_bn(gcl.node_mlp[0], gcl.node_mlp[1])
                w4, b4 = _fold_bn(gcl.node_mlp[3], gcl.node_mlp[4])
            put(f"layer{l}.node_mlp.0.weight", w3); put(f"layer{l}.node_mlp.0.bias", b3)
            put(f"layer{l}.node_mlp.2.weight", w4); put(f"layer{l}.node_mlp.2.bias", b4)
        _native.check(lib.dl_sizegnn_finalize_weights(handle), "dl_sizegnn_finalize_weights")
        self._engine, self._engine_key = handle, key
        return handle

    def close(self):
        if self._engine is not None:
            _native.load_library().dl_sizegnn_destroy(self._engine)
            self._engine = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @torch.no_grad()
    def logits(self, one_hot, positions, fragment_mask, edge_mask):
        """(B,N,F), (B,N,3), (B,N[,1]) 0/1, (B*N*N[,1]) non-zero = live  ->  (B, out_node_nf) on the inputs' device."""
        dev = positions.device
        if dev.type != 'cuda':
            raise RuntimeError("difflinker_b200.SizeGNN runs on an H100 only (no CPU fallback); move the batch to the GPU")
        B, N = positions.shape[:2]
        xh = torch.cat([positions.float(), one_hot.float()], dim=2).contiguous()
        fm = (fragment_mask.reshape(B, N) != 0).to(torch.int8).contiguous()
        em = None if edge_mask is None else (edge_mask.reshape(B, N, N) != 0).to(torch.int8).contiguous()
        out = torch.empty((B, self.out_node_nf), device=dev, dtype=torch.float32)
        lib = _native.load_library()
        with torch.cuda.device(dev):
            eng = self.engine(dev.index if dev.index is not None else torch.cuda.current_device())
            st = torch.cuda.current_stream().cuda_stream
            _native.check(lib.dl_sizegnn_forward(eng, B, N, xh.data_ptr(), fm.data_ptr(), None if em is None else em.data_ptr(),
                                                 out.data_ptr(), st), "dl_sizegnn_forward")
        return out

    def forward(self, h, edges, distances, node_mask, edge_mask):
        raise NotImplementedError("call SizeClassifier.forward (or SizeGNN.logits): the native pass starts from positions")


def collate_with_fragment_edges(batch):
    """datasets.collate_with_fragment_edges (datasets.py:378-422) without the python triple loop: the edge list is the
    fully connected e = b*N*N + i*N + j ordering that Dynamics.get_edges also uses."""
    out = collate(batch)
    frag = out['fragment_mask'].squeeze(-1)
    em = frag[:, None, :] * frag[:, :, None]
    diag = ~torch.eye(em.size(1), dtype=torch.int8, device=frag.device).unsqueeze(0)
    em = em * diag
    B, N = frag.shape
    out['edge_mask'] = em.view(B * N * N, 1)
    i = torch.arange(N, device=frag.device).repeat_interleave(N)
    j = torch.arange(N, device=frag.device).repeat(N)
    off = (torch.arange(B, device=frag.device) * N).repeat_interleave(N * N)
    out['edges'] = [i.repeat(B) + off, j.repeat(B) + off]
    return out


class SizeClassifier(nn.Module):
    """src/linker_size_lightning.py:14-110 (inference API): same constructor kwargs, `forward(data, return_loss,
    with_pocket, adjust_shape) -> (logits, loss)`, `linker_id2size` / `linker_size2id`, state_dict keys `gnn.*`."""

    def __init__(self, data_path=None, train_data_prefix=None, val_data_prefix=None, in_node_nf=8, hidden_nf=128,
                 out_node_nf=10, n_layers=3, batch_size=64, lr=1e-3, torch_device='cpu', normalization=None,
                 loss_weights=None, min_linker_size=None, linker_size2id=ZINC_TRAIN_LINKER_SIZE2ID,
                 linker_id2size=ZINC_TRAIN_LINKER_ID2SIZE, task='classification'):
        super().__init__()
        self.hparams = {k: v for k, v in locals().items() if k not in ('self', '__class__')}
        self.min_linker_size = min_linker_size
        self.linker_size2id, self.linker_id2size = linker_size2id, linker_id2size
        self.loss_weights = None if loss_weights is None else torch.tensor(loss_weights)
        self.in_node_nf = in_node_nf
        self.gnn = SizeGNN(in_node_nf=in_node_nf, hidden_nf=hidden_nf, out_node_nf=out_node_nf, n_layers=n_layers,
                           normalization=normalization)

    def size_logits(self, data, with_pocket=False, adjust_shape=False):
        """(B, out_node_nf) fp32 logits over linker_id2size: forward(data, return_loss=False, ...)'s output. They mean-pool
        over the padded rows of `data`, so they depend on its padding."""
        return self.forward(data, return_loss=False, with_pocket=with_pocket, adjust_shape=adjust_shape)[0]

    def forward(self, data, return_loss=True, with_pocket=False, adjust_shape=False):
        h, x = data['one_hot'], data['positions']
        fragment_mask = data['fragment_only_mask'] if with_pocket else data['fragment_mask']
        if h.shape[-1] != self.in_node_nf and adjust_shape:                    # linker_size_lightning.py:96-98
            assert torch.allclose(h[..., -1] * fragment_mask[..., 0], torch.zeros_like(h[..., -1]))
            h = h[..., :-1]
        output = self.gnn.logits(h, x, fragment_mask, data['edge_mask'])
        loss = None
        if return_loss:
            true = self.get_true_labels(data['linker_mask'])
            w = None if self.loss_weights is None else self.loss_weights.to(output.device)
            loss = cross_entropy(output, true, weight=w)
        return output, loss

    def get_true_labels(self, linker_mask):                                     # linker_size_lightning.py:118-127
        sizes = linker_mask.squeeze(-1).sum(-1).long().detach().cpu().numpy()
        labels = []
        for size in sizes:
            label = self.linker_size2id.get(int(size))
            if label is None:
                label = self.linker_size2id[max(self.linker_id2size)]
            labels.append(label)
        return torch.tensor(labels, device=linker_mask.device, dtype=torch.long)

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path, map_location=None, strict=True, **overrides):
        """`SizeClassifier.load_from_checkpoint(linker_size, map_location=device)` (generate.py:88) without Lightning."""
        from .ddpm import _load_lightning_checkpoint
        return _load_lightning_checkpoint(cls, checkpoint_path, map_location, strict, overrides)

    @torch.no_grad()
    def sample_sizes(self, data, generator=None, seeds=None):
        """The `sample_fn` of generate.py:90-99: softmax -> Categorical -> linker sizes (int8, on the batch's device).
        With `seeds` (one per molecule), molecule b's size is instead draw_sizes' draw from seeds[b]: a function of its seed
        and its logits alone; `generator` is then not read."""
        out, _ = self.forward(data, return_loss=False)
        if seeds is not None:
            return draw_sizes(out, self.linker_id2size, seeds).to(torch.int8)
        idx = torch.multinomial(torch.softmax(out, dim=1), 1, generator=generator).view(-1)
        table = torch.tensor(self.linker_id2size, device=idx.device)
        return table[idx].to(torch.int8)


def size_uniform(seed):
    """dl_size_uniform: the 53-bit uniform in [0, 1) a linker size is drawn with from `seed` (an int, reduced modulo 2^64)."""
    return float(_native.load_library().dl_size_uniform(operator.index(seed) % (1 << 64)))


@torch.no_grad()
def draw_sizes(logits, sizes, seeds, attempt=0):
    """dl_size_draw: molecule b's linker size drawn from its (C,) row of the (B, C) CUDA `logits` over the size table
    `sizes` with the seed dl_retry_seed(seeds[b], attempt) -- the fp64 inverse-CDF rule stated in the header. Returns (B,)
    int32 on the logits' device."""
    from .edm import seeds_tensor
    if not torch.is_tensor(logits) or logits.dim() != 2 or logits.device.type != 'cuda':
        raise ValueError("draw_sizes takes (B, C) CUDA logits")
    B, C = logits.shape
    dev = logits.device
    table = torch.tensor([operator.index(v) for v in sizes], dtype=torch.int32, device=dev)
    if table.numel() != C:
        raise ValueError(f"the size table holds {table.numel()} sizes for {C} logits")
    lg = logits.detach().to(torch.float32).contiguous()
    sd = seeds_tensor(seeds, B).to(dev)
    out = torch.empty(B, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _native.check(_native.load_library().dl_size_draw(B, C, lg.data_ptr(), C, table.data_ptr(), sd.data_ptr(), attempt,
                                                         out.data_ptr(), torch.cuda.current_stream().cuda_stream),
                      "dl_size_draw")
    return out
