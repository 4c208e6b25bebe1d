"""Serialise one sampling job for a caller that has no Python: the engine configuration, the weights under the reference's
state_dict names, the prepared inputs of `EDM.sample_chain` (reference src/edm.py:126-176) or `InpaintingEDM.sample_chain`
(its configuration has centering = 1; its coefficient table carries qa / qb), the per-step coefficient table of the noise
schedule and a Philox (seed, offset) pair -- or, in a seeded job (`write_seeded_job`), one seed per molecule.
`examples/c_sampler.c` reads the file and samples through the C-ABI (`dl_sample_chain_rng`, or `dl_sample_chain_seeded`);
`read_result` parses what it writes back (`read_retry_result` what it writes with `--retries k`)."""
import ctypes as C
import struct

import numpy as np
import torch

from . import _native

MAGIC = b"DLJOB1\0\0"
MAGIC_OPTS = b"DLJOB2\0\0"   # a model with non-default EGNN options: the dl_egnn_options follow the dl_config
# seeded job: the dl_config, an int32 flag and (flag = 1) the dl_egnn_options, then the layout of the other versions with the
# B uint64 per-molecule seeds in place of the (seed, offset) pair
MAGIC_SEEDED = b"DLJOB3\0\0"


def write_job(path, edm, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context, keep_frames, seed, offset=0,
              device_index=0):
    """Arguments as `EDM.sample_chain` takes them (`ddpm.sampler_inputs` builds them from a collated batch)."""
    assert offset % 4 == 0
    return _write(path, edm, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context, keep_frames, device_index,
                  False, struct.pack("<2Q", seed & 0xFFFFFFFFFFFFFFFF, offset))


def write_seeded_job(path, edm, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context, keep_frames, seeds,
                     device_index=0):
    """A job the C caller samples with `dl_sample_chain_seeded`: as write_job, with one seed per molecule (B ints or an
    integer tensor, reduced as EDM.sample_chain(seeds=...) reduces them) instead of a generator state."""
    from .edm import seeds_tensor
    s = seeds_tensor(seeds, x.size(0))
    return _write(path, edm, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context, keep_frames, device_index,
                  True, s.numpy().astype("<i8").tobytes())


def _write(path, edm, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context, keep_frames, device_index, seeded, rng):
    """The job file: a seeded one, or a (seed, offset) one of the first two versions; `rng` holds the bytes naming the noise."""
    dyn = edm.dynamics
    B, N = x.size(0), x.size(1)
    T = edm.T
    xd = edm.n_dims + edm.in_node_nf
    assert 1 <= keep_frames <= T
    xn, hn = edm.normalize(x, h)
    xh = torch.cat([xn, hn], dim=2).to(torch.float32).cpu().contiguous()
    cfg = dyn.dl_config(device_index)
    opts = dyn.egnn_options()
    assert C.sizeof(cfg) == 13 * 4 and C.sizeof(_native.DLStepCoef) == 32 and C.sizeof(opts) == 16
    coef = edm.step_coefficients(keep_frames, B)
    f32 = lambda t: t.detach().to(device='cpu', dtype=torch.float32).contiguous().numpy().tobytes()
    i8 = lambda t: t.detach().to(device='cpu', dtype=torch.int8).contiguous().numpy().tobytes()
    with open(path, "wb") as f:
        if seeded:
            f.write(MAGIC_SEEDED)
            f.write(bytes(cfg))
            f.write(struct.pack("<i", int(not opts.is_default())))
            if not opts.is_default():
                f.write(bytes(opts))
        elif opts.is_default():                        # jobs of default models keep the first version, byte for byte
            f.write(MAGIC)
            f.write(bytes(cfg))
        else:
            f.write(MAGIC_OPTS)
            f.write(bytes(cfg))
            f.write(bytes(opts))
        sd = dyn.dynamics.state_dict()
        f.write(struct.pack("<i", len(sd)))
        for name, p in sd.items():
            nb = f"dynamics.{name}".encode()
            f.write(struct.pack("<i", len(nb)) + nb + struct.pack("<q", p.numel()) + f32(p))
        f.write(struct.pack("<6i", B, N, T, keep_frames, xd, dyn.context_node_nf))
        f.write(rng)
        f.write(struct.pack("<3f", float(edm.norm_values[0]), float(edm.norm_values[1]), float(edm.norm_biases[1])))
        f.write(bytes(coef)[:(T + 1) * 32])
        f.write(xh.numpy().tobytes())
        f.write(i8(node_mask.reshape(B, N)))
        f.write(f32(fragment_mask.reshape(B, N)))
        f.write(f32(linker_mask.reshape(B, N)))
        has_em = dyn.graph_type == 'FC' and edge_mask is not None
        f.write(struct.pack("<i", int(has_em)))
        if has_em:
            em = i8(edge_mask.reshape(-1))
            assert len(em) == B * N * N
            f.write(em)
        f.write(struct.pack("<i", int(context is not None)))
        if context is not None:
            f.write(f32(context.reshape(B, N, dyn.context_node_nf)))
    return {"B": B, "N": N, "T": T, "keep_frames": keep_frames, "xd": xd}


def read_result(path, B, N, keep_frames, xd):
    """(status, philox offset consumed (0 for a seeded job), chain (keep_frames,B,N,xd) float32 tensor, flags (B,) int32
    tensor)."""
    raw = open(path, "rb").read()
    status, consumed = struct.unpack_from("<iQ", raw, 0)
    n = keep_frames * B * N * xd
    chain = torch.from_numpy(np.frombuffer(raw, dtype=np.float32, count=n, offset=12).copy()).view(keep_frames, B, N, xd)
    flags = torch.from_numpy(np.frombuffer(raw, dtype=np.int32, count=B, offset=12 + 4 * n).copy())
    assert len(raw) == 12 + 4 * n + 4 * B
    return status, consumed, chain, flags


def read_retry_result(path, B, N, keep_frames, xd):
    """What `c_sampler --retries k` writes: read_result's (status, consumed, chain, flags), then the seeds that produced the
    rows as a (B,) int64 tensor with their 64 bits (the form EDM.last_seeds holds) and the (B,) int32 attempts."""
    raw = open(path, "rb").read()
    n = 12 + 4 * keep_frames * B * N * xd + 4 * B
    assert len(raw) == n + 12 * B
    status, consumed = struct.unpack_from("<iQ", raw, 0)
    chain = torch.from_numpy(np.frombuffer(raw, dtype=np.float32, count=keep_frames * B * N * xd, offset=12).copy())
    flags = torch.from_numpy(np.frombuffer(raw, dtype=np.int32, count=B, offset=n - 4 * B).copy())
    used = torch.from_numpy(np.frombuffer(raw, dtype="<i8", count=B, offset=n).copy())
    attempts = torch.from_numpy(np.frombuffer(raw, dtype=np.int32, count=B, offset=n + 8 * B).copy())
    return status, consumed, chain.view(keep_frames, B, N, xd), flags, used, attempts
