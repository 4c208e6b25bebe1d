"""Drop-in `EDM` sampler (reference: src/edm.py:14-463, sampling half) running the whole reverse-diffusion loop on
the device through `dl_sample_chain`: one CUDA-graph replay per step, no host synchronisation inside the loop.

What stays in Python (plumbing): normalisation of the inputs, the per-step scalar table -- computed with the very
torch ops the reference uses (edm.py:369-403) so the coefficients are bit-identical -- and the random draws, which
are made with the reference's `torch.randn` call order and shapes (edm.py:328-345) on the tensors' device, so a given
torch seed produces the same noise stream as the reference would on that device.
"""
import ctypes as C
import functools
import math
import numbers
import operator
import threading
from typing import NamedTuple

import numpy as np
import torch
import torch.nn.functional as F

from . import _native
from .distributed import (deal_launches, device_slices, pack_requests, place_rows, plan_launches, resolve_devices,
                          slice_sampler_inputs, unpack_rows)
from .molecule_builder import check_tables, clash_table, graph_hashes, ring_size_mask, sort_unsigned
from .noise import PredefinedNoiseSchedule
from .utils import FoundNaNException, nan_exception_class


def _generator_of(dev):
    return torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]


class LinkerSizes(NamedTuple):
    """What EDM.sample_chain redraws linker sizes from in its recovery rounds (dl_sample_chain_retry), for a
    template built at the sizes dl_size_draw gives the call's seeds at attempt 0 and padded to at least
    max(n_frag) + max(sizes) rows. ddpm.sample_chain(linker_sizes=...) builds it.
      logits    (B, C) fp32 CUDA: every molecule's size logits
      sizes     the C sizes of the table, ints >= 0
      n_frag    (B) ints: every molecule's fragment rows (pocket rows included), which come first in the template
      linker_x  (B, 3): the centred (not normalised) coordinates of every molecule's template linker rows"""
    logits: torch.Tensor
    sizes: list
    n_frag: torch.Tensor
    linker_x: torch.Tensor


class StartSteps(NamedTuple):
    """Per-molecule start steps of a call (dl_set_start_steps): row b starts at step t0[b] with the scalars alpha[b],
    sigma[b] of start_scalars(t0[b], B) at the call's own B."""
    t0: list
    alpha: list
    sigma: list

    def rows(self, lo, hi):
        return StartSteps(self.t0[lo:hi], self.alpha[lo:hi], self.sigma[lo:hi])

    @staticmethod
    def cat(parts):
        return StartSteps(*(sum((list(p[i]) for p in parts), []) for i in range(3)))

    def set_on(self, lib, eng):
        n = len(self.t0)
        _native.check(lib.dl_set_start_steps(eng, n, (C.c_int32 * n)(*self.t0), (C.c_float * n)(*self.alpha),
                                             (C.c_float * n)(*self.sigma)), "dl_set_start_steps")


def _loop_steps(start):
    """The step a call's loop starts from: t0 of a scalar start, the largest t0 of per-molecule ones, or None."""
    if start is None:
        return None
    return max(start.t0) if isinstance(start, StartSteps) else start[0]


def _sample_slice(lib, eng, head, tail, stream, noise=None, seeds=None, rng=None, retry=None, start=None, resample=None,
                  guide=None, solver=None, fixed=None, types=None):
    """One slice's reverse loop on its engine: dl_sample_chain_*(eng, *head, <draws>, *tail, stream). The draws are the
    per-molecule `seeds`, the batch stream `rng` = (seed, offset, b0, B_full) -- the call's B rows are rows [b0, b0 + B) of a
    B_full-molecule batch, set on the engine for the duration of the call -- or else the `noise` tensor. `stream` None
    samples host inputs (dl_sample_chain_host). With `seeds`, `retry` = (max_retries, seeds_used, attempts, require, checks,
    passed, redraw, sets, linker_hashes, rings, anchors) resamples the molecules that diverged (dl_sample_chain_retry_sets, which blocks until its rounds
    are done) and, with `require` != 0, those that miss a required check, whose verdict bits go to `passed`; `checks` =
    (tables, clash) on the slice's device, `tables` as molecule_builder.check_tables returns them and `clash` the (T,T) clash
    table or None. `redraw` = (logits, size table, n_frag, normalised linker_x, sizes_used), device tensors, redraws the
    resampled rows' linker sizes; None keeps them. `sets` = (known, seen), sorted int64 device tensors or None, are the
    hash sets of CHECK_NOVEL and CHECK_UNIQUE; None is two empty sets. `linker_hashes`, an int64 device tensor or None,
    receives every returned row's linker hash (CHECK_NOVEL). `rings` = (allowed mask, (B,) int64 device tensor), or None,
    sets the ring sizes CHECK_RINGS allows on the engine (dl_set_ring_sizes) and receives every returned row's ring-size
    mask (dl_last_ring_sizes). `anchors`, a (B, N) int8 device tensor or None, are the anchor flags CHECK_ANCHORS reads
    (dl_set_anchors, right before the call, which clears them).
    `start` = (t0, alpha_t0, sigma_t0) starts the loop at step t0 from q(z_t0 | x), set on the engine for the duration of
    the call (dl_set_start_step); a StartSteps starts each row at its own step (dl_set_start_steps). `resample` = (r, T,
    jump) runs r RePaint passes per step, set on the engine for the duration of the call (dl_set_resamplings). `guide` =
    (scale, steps, clash table) pushes the linker atoms out of the pocket at the last `steps` steps, set on the engine for
    the duration of the call (dl_set_clash_guidance). `solver` = (kind, T, table) replaces the ancestral update by an ODE
    solver's, set on the engine for the duration of the call (dl_set_solver). `fixed` = ((B, N) int8 flags on the slice's
    device, or on the host with host inputs, T, scalars) keeps the flagged linker rows (dl_set_fixed_atoms, right before
    the call, which clears it). `types` = ((B,) int32 CPU masks, F, T, scalars) gives the linker atoms allowed types only
    (dl_set_linker_types, right before the call, which clears it). Returns (status, what the batch stream consumed)."""
    per_row = isinstance(start, StartSteps)
    if per_row:
        start.set_on(lib, eng)
    elif start is not None:
        _native.check(lib.dl_set_start_step(eng, *start), "dl_set_start_step")
    try:
        if resample is not None:
            _native.check(lib.dl_set_resamplings(eng, *resample), "dl_set_resamplings")
        if guide is not None:
            scale, steps, table = guide
            _native.check(lib.dl_set_clash_guidance(eng, scale, steps, table.shape[0], table.data_ptr()),
                          "dl_set_clash_guidance")
        if solver is not None:
            _native.check(lib.dl_set_solver(eng, *solver), "dl_set_solver")
        if fixed is not None:
            flags, T, scalars = fixed
            _native.check(lib.dl_set_fixed_atoms(eng, head[1], head[2], flags.data_ptr(), T, scalars, stream),
                          "dl_set_fixed_atoms")
        if types is not None:
            masks, F, T, scalars = types
            _native.check(lib.dl_set_linker_types(eng, head[1], F, masks.data_ptr(), T, scalars),
                          "dl_set_linker_types")
        return _sample_slice_draws(lib, eng, head, tail, stream, noise, seeds, rng, retry)
    finally:
        if types is not None:               # a call that failed before the engine read the masks
            lib.dl_set_linker_types(eng, 0, 0, None, 0, None)
        if fixed is not None:               # a call that failed before the engine read the flags
            lib.dl_set_fixed_atoms(eng, 0, 0, None, 0, None, None)
        if solver is not None:
            lib.dl_set_solver(eng, _native.SOLVERS['ancestral'], 0, None)
        if guide is not None:
            lib.dl_set_clash_guidance(eng, 0.0, 0, 0, None)
        if resample is not None:
            lib.dl_set_resamplings(eng, 1, 0, None)
        if per_row:
            lib.dl_set_start_steps(eng, 0, None, None, None)
        elif start is not None:
            lib.dl_set_start_step(eng, -1, 0.0, 0.0)


def _sample_slice_draws(lib, eng, head, tail, stream, noise, seeds, rng, retry):
    """_sample_slice's call of the entry point that matches its draws."""
    if stream is None:
        return _native.check(lib.dl_sample_chain_host(eng, *head, noise.data_ptr(), *tail), "dl_sample_chain_host"), 0
    if retry is not None:
        max_retries, used, attempts, require, checks, passed, redraw, sets, linker_hashes, rings, anchors = retry
        ck = _native.DLMoleculeChecks.of(require, *checks) if require else None
        if rings is not None:
            _native.check(lib.dl_set_ring_sizes(eng, rings[0]), "dl_set_ring_sizes")
        if anchors is not None:
            _native.check(lib.dl_set_anchors(eng, head[1], head[2], anchors.data_ptr(), stream), "dl_set_anchors")
        hs = None if sets is None else _native.DLHashSets.of(*sets)
        rz = sizes = None
        if redraw is not None:
            logits, table, n_frag, linker_x, sizes = redraw
            rz = _native.DLSizeRedraw(table.numel(), logits.stride(0), logits.data_ptr(), table.data_ptr(), n_frag.data_ptr(),
                                      linker_x.data_ptr())
        st = _native.check(lib.dl_sample_chain_retry_sets(
            eng, *head, seeds.data_ptr(), *tail, max_retries, used.data_ptr(), attempts.data_ptr(), ck, hs,
            passed.data_ptr() if require else None, None if linker_hashes is None else linker_hashes.data_ptr(), rz,
            None if sizes is None else sizes.data_ptr(), stream),
            "dl_sample_chain_retry_sets")
        if rings is not None:
            _native.check(lib.dl_last_ring_sizes(eng, head[1], rings[1].data_ptr(), stream), "dl_last_ring_sizes")
        return st, 0
    if seeds is not None:
        return _native.check(lib.dl_sample_chain_seeded(eng, *head, seeds.data_ptr(), *tail, stream),
                             "dl_sample_chain_seeded"), 0
    if rng is None:
        return _native.check(lib.dl_sample_chain(eng, *head, noise.data_ptr(), *tail, stream), "dl_sample_chain"), 0
    seed, offset, b0, b_full = rng
    used = C.c_uint64(0)
    _native.check(lib.dl_set_noise_slice(eng, b_full, b0), "dl_set_noise_slice")
    try:
        st = lib.dl_sample_chain_rng(eng, *head, seed, offset, C.byref(used), *tail, stream)
    finally:
        lib.dl_set_noise_slice(eng, 0, 0)
    return _native.check(st, "dl_sample_chain_rng"), used.value


def seeds_tensor(seeds, n_samples):
    """Per-molecule seeds -- an integer tensor or a sequence of ints, one per molecule -- as a CPU int64 tensor. Each seed is
    reduced modulo 2^64 as torch.cuda.manual_seed reduces it (values in [-2^63, 2^64); -1 and 2^64 - 1 name the same
    stream) and kept as the int64 with the same 64 bits, which torch.cuda.manual_seed accepts back unchanged."""
    if torch.is_tensor(seeds):
        if seeds.dim() != 1 or seeds.dtype.is_floating_point or seeds.dtype.is_complex or seeds.dtype == torch.bool:
            raise ValueError(f"seeds must be a 1-D integer tensor (got {seeds.dtype} of shape {tuple(seeds.shape)})")
        seeds = seeds.tolist()
    out = []
    for s in seeds:
        if isinstance(s, bool):
            raise ValueError(f"seeds are integers (got {s!r})")
        try:
            s = operator.index(s)
        except TypeError:
            raise ValueError(f"seeds are integers (got {s!r})") from None
        if not -(1 << 63) <= s < (1 << 64):
            raise ValueError(f"seed {s} is outside [-2^63, 2^64), the range torch.cuda.manual_seed accepts")
        out.append(s - (1 << 64) if s >= (1 << 63) else s)
    if len(out) != n_samples:
        raise ValueError(f"seeds holds {len(out)} values for a batch of {n_samples} molecules")
    return torch.tensor(out, dtype=torch.int64)


def retry_seed(seed, attempt):
    """The seed of attempt `attempt` of a molecule seeded with `seed` (dl_retry_seed: attempt 0 is the seed itself, attempt
    a >= 1 is output a of a splitmix64 generator started from it), in the int64 form `last_seeds` holds. The seed is reduced
    as seeds_tensor reduces it, so replaying with the returned value samples that attempt's stream."""
    s = int(seeds_tensor([seed], 1)[0]) % (1 << 64)
    attempt = operator.index(attempt)
    if not -(1 << 31) <= attempt < (1 << 31):
        raise ValueError(f"attempt {attempt} does not fit an int32")
    r = int(_native.load_library().dl_retry_seed(s, attempt))
    return r - (1 << 64) if r >= (1 << 63) else r


def draw_seeds(n_samples, device):
    """The seeds noise_mode='per_molecule' derives when none are given: one call on `device`'s default CUDA generator,
    torch.randint(2**63 - 1, (n_samples,), dtype=torch.int64, device=device), so torch.manual_seed governs them."""
    return torch.randint(2 ** 63 - 1, (n_samples,), dtype=torch.int64, device=device)


def _run_per_device(calls_by_device):
    """Runs each device's calls, in order, on a host thread of its own (the C-ABI allows one host thread per engine, and ctypes
    releases the GIL), so every device's reverse loop is enqueued even if one device's enqueue blocks. Every thread is joined
    before the first error is re-raised."""
    errors = []

    def run(calls):
        try:
            for call in calls:
                call()
        except BaseException as e:                      # re-raised on the caller's thread below
            errors.append(e)
    threads = [threading.Thread(target=run, args=(calls,), name=f"difflinker_b200-cuda{d}")
               for d, calls in calls_by_device.items()]
    started = []
    try:
        for t in threads:
            t.start()
            started.append(t)
    finally:
        for t in started:
            t.join()
    if errors:
        raise errors[0]


class EDM(torch.nn.Module):
    def __init__(
            self,
            dynamics,
            in_node_nf: int,
            n_dims: int,
            timesteps: int = 1000,
            noise_schedule='learned',
            noise_precision=1e-4,
            loss_type='vlb',
            norm_values=(1., 1., 1.),
            norm_biases=(None, 0., 0.),
            is_geom=None,
    ):
        super().__init__()
        if noise_schedule == 'learned':
            # GammaNetwork (src/noise.py:131-169) is only valid with the vlb loss; every config trains with
            # l2 + polynomial_2 (train_difflinker.py:140-142). Out of scope for the sampling hot path.
            raise NotImplementedError("learned noise schedules are outside the difflinker_b200 hot path")
        self.gamma = PredefinedNoiseSchedule(noise_schedule, timesteps=timesteps, precision=noise_precision)
        self.dynamics = dynamics
        self.in_node_nf = in_node_nf
        self.n_dims = n_dims
        self.T = timesteps
        self.norm_values = norm_values
        self.norm_biases = norm_biases
        # 'reference_stream' (default): the reference's torch.randn call order, so seeds line up with the reference run on
        #   the same kind of device. On CUDA the numbers are regenerated INSIDE the kernels that consume them from the torch
        #   generator's (seed, offset) -- same values as the randn calls, no tensor, no launches (dl_sample_chain_rng).
        # 'reference_tensor': the same stream materialised with torch.randn (two launches per draw).
        # 'bulk': one randn call for the whole chain (a different stream).
        # 'per_molecule': every molecule draws from a stream of its own (see sample_chain's `seeds`); without `seeds` the B
        #   seeds come from one draw_seeds call on the inputs' device, so torch.manual_seed still governs the run.
        self.noise_mode = 'reference_stream'
        self.last_seeds = None                 # per-molecule stream: the (B,) CPU int64 seeds of the last call, else None
        # NaN recovery: how many times sample_chain resamples the molecules that diverged, with new seeds derived from their
        # own (dl_retry_seed); needs per-molecule streams. 0, the default, raises FoundNaNException for the batch as before.
        self.nan_retries = 0
        self.last_attempts = None              # calls with nan_retries > 0: the (B,) CPU int32 attempt of every row, else None
        # Connectivity: sample_chain also resamples, in the nan_retries rounds, the molecules whose final molecule is in more
        # than one piece (dl_sample_chain_retry); needs per-molecule streams and the bond tables of
        # `is_geom` (the ZINC or the GEOM / MOAD atom types, molecule_builder.threshold_tables), which DDPM, accelerate and
        # load_from_checkpoint set from the model's training data. False, the default, checks nothing.
        self.is_geom = is_geom
        self.require_connected = False
        self.last_connected = None             # calls with require_connected: the (B,) CPU bool connectivity of every row
        # Valence: likewise for the molecules with an atom whose bond orders sum to more than its element allows
        # (molecule_builder.max_valence_table), in the same check launch. With require_connected it is the
        # reference's validity_and_connectivity, as far as "explicit valence within the table" is RDKit's sanitization
        # (not verified, see molecule_builder.valence_ok). Same needs; False, the default, checks nothing.
        self.require_valid = False
        self.last_valid = None                 # calls with require_valid: the (B,) CPU bool valence verdict of every row
        # Pocket clashes (cut-off graphs only): likewise for the molecules with a linker atom closer to a pocket atom than
        # molecule_builder.clash_table(is_geom) allows, in the same check launch. Same needs; False, the default, checks
        # nothing.
        self.require_clash_free = False
        self.last_clash_free = None            # calls with require_clash_free: the (B,) CPU bool clash verdict of every row
        # Uniqueness: likewise for the molecules whose bond graph repeats a batch-mate's (molecule_builder.graph_hashes), in
        # the same check launch and a verdict over the call's rows. Same needs, and one slice; False, the default, checks
        # nothing.
        self.require_unique = False
        self.last_unique = None                # calls with require_unique: the (B,) CPU bool uniqueness verdict of every row
        self.last_graph_hashes = None          # calls with require_unique: the (B,) CPU int64 graph hash of every row
        # Novelty: likewise for the molecules whose linker hash (molecule_builder.linker_hashes) is in `known_linkers`, a
        # 1-D int64 tensor of uint64 hashes in any order (molecule_builder.known_linkers builds it from a dataset), in the
        # same check launch. Same needs; False, the default, checks nothing.
        self.require_novel = False
        self.known_linkers = None
        self.last_novel = None                 # calls with require_novel: the (B,) CPU bool novelty verdict of every row
        self.last_linker_hashes = None         # calls with require_novel: the (B,) CPU int64 linker hash of every row
        # Ring sizes: likewise for the molecules whose linker closes a smallest ring of a size not in `allowed_ring_sizes`,
        # an iterable of ints >= 3 (63 meaning 63 or more atoms; molecule_builder.ring_sizes), in the same check launch.
        # Which sizes to allow is the caller's policy: there is no default. Same needs; False, the default, checks nothing.
        self.require_ring_sizes = False
        self.allowed_ring_sizes = None
        self.last_ring_sizes_ok = None         # calls with require_ring_sizes: the (B,) CPU bool ring verdict of every row
        self.last_ring_sizes = None            # calls with require_ring_sizes: the (B,) CPU int64 ring-size mask of every row
        # Anchors: likewise for the molecules whose linker does not attach by exactly one bond at each anchor and nowhere
        # else on the fragments (molecule_builder.attachments), in a launch right after the check launch. The anchors are
        # per-call input (sample_chain's `anchors=`). Same needs; False, the default, checks nothing.
        self.require_anchors = False
        self.last_anchors_ok = None            # calls with require_anchors: the (B,) CPU bool anchor verdict of every row
        self.last_sizes = None                # calls with linker_sizes: the (B,) CPU int32 linker size of every returned row
        # RePaint resampling (InpaintingEDM only): the passes of every reverse step when sample_chain / sample_many get no
        # `resamplings`; 1, the default, is the plain loop
        self.resamplings = 1
        # Clash guidance (EDM on cut-off graphs only): (scale, steps) pushes the linker atoms that overlap pocket atoms back
        # towards molecule_builder.clash_table(is_geom)'s distances at the last `steps` reverse steps, when sample_chain /
        # sample_many get no `clash_guidance`; None, the default, guides nothing
        self.clash_guidance = None
        # Reverse update (EDM only): 'ancestral' (the default) samples p(z_s | z_t) as the reference does; 'ddim' and
        # 'dpmpp_2m' take deterministic steps of the probability-flow ODE (solver_coefficients), for calls that get no
        # `solver`. Meant for a shortened loop: edm.T = 20; edm.solver = 'dpmpp_2m'
        self.solver = 'ancestral'
        # Linker types (EDM only): the allowed type channels of the linker atoms, a (F,) or (B, F) bool tensor, for calls
        # that get no `linker_types` (sample_chain); None, the default, allows every type
        self.linker_types = None
        self.devices = None
        self.last_loop_ms = None               # device time of the last reverse loop (CUDA events); the slowest slice's if split
        self.last_slice_loop_ms = None         # split calls: [(device, lo, hi, loop ms)] per slice of the batch
        # sample_many: per request, what last_seeds / last_attempts / last_connected / last_valid hold after its own
        # sample_chain call; per launch, (device, the requests it held, loop ms)
        self.last_seeds_many = self.last_attempts_many = self.last_connected_many = self.last_loop_ms_many = None
        self.last_valid_many = self.last_clash_free_many = self.last_sizes_many = self.last_novel_many = None
        self.last_ring_sizes_ok_many = self.last_ring_sizes_many = None
        self.last_anchors_ok_many = None

    @property
    def devices(self):
        """None (the default): sample_chain samples each batch as one slice on the inputs' device. A list of CUDA device
        indices, or 'all' when set: it makes one contiguous, balanced slice per listed device instead, samples them
        concurrently and returns the whole chain on the inputs' device. That chain is the one a single device samples, bit
        for bit on the fp32 SIMT edge path, and on the tensor-core path while no sample diverges: the node GEMM rescales the
        fp16 operands of a tile by a power of two chosen from the tile's maximum once values approach the fp16 range, and
        since tiles span molecules and follow the batch, such molecules round differently after a split (DESIGN.md section
        6). A device may be listed more than once: each listing gets an engine of its own, and engines sharing a device run
        their loops one after the other. Calls without `devices` keep one engine, so switching between split and
        single-device calls re-creates engines."""
        return self._devices

    @devices.setter
    def devices(self, devices):
        self._devices = resolve_devices(devices)

    def forward(self, *args, **kwargs):
        raise NotImplementedError("training (src/edm.py:41-124) is outside the difflinker_b200 hot path")

    # ---- scalar helpers, same names/semantics as the reference -------------------------------------------------
    def sigma(self, gamma, target_tensor=None):
        return torch.sqrt(torch.sigmoid(gamma))

    def alpha(self, gamma, target_tensor=None):
        return torch.sqrt(torch.sigmoid(-gamma))

    @staticmethod
    def SNR(gamma):
        return torch.exp(-gamma)

    @staticmethod
    def sigma_and_alpha_t_given_s(gamma_t, gamma_s):
        sigma2_t_given_s = -torch.expm1(F.softplus(gamma_s) - F.softplus(gamma_t))
        alpha_t_given_s = torch.exp(0.5 * (F.logsigmoid(-gamma_t) - F.logsigmoid(-gamma_s)))
        return sigma2_t_given_s, torch.sqrt(sigma2_t_given_s), alpha_t_given_s

    def normalize(self, x, h):
        return x / self.norm_values[0], (h.float() - self.norm_biases[1]) / self.norm_values[1]

    def unnormalize(self, x, h):
        return x * self.norm_values[0], h * self.norm_values[1] + self.norm_biases[1]

    def _cpu_gamma(self):
        """The noise schedule as a CPU module: the coefficients are evaluated on the CPU whatever the model's device."""
        gamma = PredefinedNoiseSchedule.__new__(PredefinedNoiseSchedule)
        torch.nn.Module.__init__(gamma)
        gamma.timesteps = self.gamma.timesteps
        gamma.gamma = torch.nn.Parameter(self.gamma.gamma.detach().cpu(), requires_grad=False)
        return gamma

    def _q_coefficients(self, g_s, sigma_s, sigma_t, sigma2_ts, alpha_ts):
        """(qa, qb) of a reverse step: the linker sampler does not re-noise known atoms."""
        return 0.0, 0.0

    def _final_qa(self, g0):
        return 0.0

    def step_coefficients(self, keep_frames, n_samples=1):
        """(T+1) rows of dl_step_coef: row r is reverse step s = T-1-r (edm.py:146-163, 178-208); row T is the
        final p(x,h|z_0) step (edm.py:210-235).  Evaluated on (n_samples,1) fp32 CPU tensors exactly as the
        reference does: torch's CPU transcendental kernels round differently for different tensor sizes, so this
        is what makes the scalars bit-identical to the reference's for the same batch size. Cached for the last few batch
        sizes (sample_many needs one table per request size)."""
        T = self.T
        key = (T, keep_frames, n_samples, self.gamma.gamma._version, self.gamma.gamma.data_ptr())
        cache = self.__dict__.setdefault('_coef_cache', {})
        if key in cache:
            return cache[key]
        gamma = self._cpu_gamma()
        rows = (_native.DLStepCoef * (T + 1))()
        for r in range(T):
            s = T - 1 - r
            s_arr = torch.full((n_samples, 1), fill_value=s)
            t_arr = (s_arr + 1) / T                  # int64 / int -> fp32 true division, as edm.py:147-150
            s_arr = s_arr / T
            g_s, g_t = gamma(s_arr), gamma(t_arr)
            sigma2_ts, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(g_t, g_s)
            sigma_s, sigma_t = self.sigma(g_s), self.sigma(g_t)
            b = sigma2_ts / alpha_ts / sigma_t       # edm.py:199
            c = sigma_ts * sigma_s / sigma_t         # edm.py:202
            qa, qb = self._q_coefficients(g_s, sigma_s, sigma_t, sigma2_ts, alpha_ts)
            frame = (s * keep_frames) // T
            # only the last writer of a frame matters; frame 0 is finally overwritten by chain[0] (edm.py:174)
            last_writer = frame > 0 and (s == 0 or ((s - 1) * keep_frames) // T != frame)
            rows[r] = _native.DLStepCoef(float(t_arr[0]), float(alpha_ts[0]), float(b[0]), float(c[0]),
                                         frame if last_writer else -1, qa, qb, 0.0)
        g0 = gamma(torch.zeros(size=(n_samples, 1)))
        inv_alpha0 = 1. / self.alpha(g0)
        rows[T] = _native.DLStepCoef(0.0, float(inv_alpha0[0]), float(self.sigma(g0)[0]),
                                     float(self.SNR(-0.5 * g0)[0]), -1, self._final_qa(g0), 0.0, 0.0)
        if len(cache) >= 8:
            cache.pop(next(iter(cache)))
        cache[key] = rows
        return rows

    def jump_coefficients(self, n_samples=1):
        """The (T, 2) jump coefficients of dl_set_resamplings as a flat ctypes float array: row r, in step_coefficients' row
        order (step s = T-1-r), holds (alpha_t|s, sigma_t|s) of sigma_and_alpha_t_given_s(gamma(t), gamma(s)), t = (s+1)/T,
        evaluated on (n_samples, 1) fp32 CPU tensors as step_coefficients evaluates its rows. Cached likewise."""
        T = self.T
        key = ('jump', T, n_samples, self.gamma.gamma._version, self.gamma.gamma.data_ptr())
        cache = self.__dict__.setdefault('_coef_cache', {})
        if key in cache:
            return cache[key]
        gamma = self._cpu_gamma()
        out = (C.c_float * (2 * T))()
        for r in range(T):
            s_arr = torch.full((n_samples, 1), fill_value=T - 1 - r)
            t_arr = (s_arr + 1) / T
            _, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma(t_arr), gamma(s_arr / T))
            out[2 * r], out[2 * r + 1] = float(alpha_ts[0]), float(sigma_ts[0])
        if len(cache) >= 8:
            cache.pop(next(iter(cache)))
        cache[key] = out
        return out

    def _resamplings(self, resamplings):
        """The RePaint passes of a call: `resamplings`, or the `resamplings` attribute when None. ValueError unless an int
        >= 1 (not a bool); the linker sampler, which does not inpaint, takes 1 only."""
        r = self.resamplings if resamplings is None else resamplings
        try:
            if isinstance(r, bool):
                raise TypeError
            r = operator.index(r)
        except TypeError:
            raise ValueError(f"resamplings is a count of passes per step (got {r!r})") from None
        if r < 1:
            raise ValueError(f"resamplings must be >= 1 (got {r})")
        if r >= 1 << 31:
            raise ValueError(f"resamplings {r} does not fit an int32")
        if r > 1 and self._SAMPLER != _native.SAMPLER_INPAINT:
            raise ValueError("resamplings re-noises an inpainting step: EDM samples the linker alone and takes 1 only "
                             "(use InpaintingEDM)")
        return r

    def _resample(self, r, n_samples):
        """_sample_slice's `resample` of r passes at batch size n_samples, or None for the plain loop."""
        return None if r == 1 else (r, self.T, self.jump_coefficients(n_samples))

    def solver_coefficients(self, kind):
        """The (T+1, 8) table of dl_set_solver for the solver `kind` ('ddim' or 'dpmpp_2m') as a flat ctypes float array,
        in step_coefficients' row order. gamma_t and gamma_s are the schedule's fp32 entries at t = (s+1)/T and s/T (looked up
        as step_coefficients looks them up); alpha = sqrt(sigmoid(-gamma)), sigma = sqrt(sigmoid(gamma)), lambda = -gamma/2
        and h = lambda_s - lambda_t. Row r < T (step s = T-1-r): sigma_t, 1/alpha_t, sigma_s/sigma_t, c1 = -alpha_s
        expm1(-h), c2a = c1 (1 + 1/(2 rho)), c2b = -c1/(2 rho) with rho = h_{r-1}/h_r (DPM-Solver++(2M); c2a = c1 and c2b = 0
        for 'ddim' and in row 0), h, 0. Row T: sigma_0, 1/alpha_0 and zeros. Every entry is evaluated in fp64 and rounded to
        fp32 once; the table does not depend on the batch size. Cached like jump_coefficients. ValueError for another kind
        and for T above the schedule's timesteps, where grid points repeat and h would be 0."""
        if kind not in ('ddim', 'dpmpp_2m'):
            raise ValueError(f"solver_coefficients takes 'ddim' or 'dpmpp_2m' (got {kind!r})")
        T = self.T
        if T > self.gamma.timesteps:
            raise ValueError(f"the ODE solvers need T <= the schedule's timesteps ({self.gamma.timesteps}); T = {T} would "
                             "repeat grid points")
        key = ('solver', kind, T, self.gamma.gamma._version, self.gamma.gamma.data_ptr())
        cache = self.__dict__.setdefault('_coef_cache', {})
        if key in cache:
            return cache[key]
        gamma = self._cpu_gamma()
        one = lambda v: float(gamma(torch.full((1, 1), fill_value=v) / T)[0, 0])   # exact: an fp32 table entry
        g = [one(T - r) for r in range(T)] + [float(gamma(torch.zeros((1, 1)))[0, 0])]   # g[r] = gamma_t of row r
        alpha = lambda v: math.sqrt(1.0 / (1.0 + math.exp(v)))
        sigma = lambda v: math.sqrt(1.0 / (1.0 + math.exp(-v)))
        out = (C.c_float * (8 * (T + 1)))()
        h_prev = None
        for r in range(T):
            g_t, g_s = g[r], g[r + 1]
            h = (g_t - g_s) / 2.0
            c1 = -alpha(g_s) * math.expm1(-h)
            c2a, c2b = c1, 0.0
            if kind == 'dpmpp_2m' and r > 0:
                rho = h_prev / h
                c2a, c2b = c1 * (1.0 + 1.0 / (2.0 * rho)), -c1 / (2.0 * rho)
            out[8 * r:8 * r + 8] = [sigma(g_t), 1.0 / alpha(g_t), sigma(g_s) / sigma(g_t), c1, c2a, c2b, h, 0.0]
            h_prev = h
        out[8 * T:8 * T + 8] = [sigma(g[T]), 1.0 / alpha(g[T])] + [0.0] * 6
        if len(cache) >= 8:
            cache.pop(next(iter(cache)))
        cache[key] = out
        return out

    def _solver(self, solver):
        """_sample_slice's `solver` of a call: (kind, T, table) from `solver`, or the `solver` attribute when None; None for
        'ancestral'. ValueError for another name than 'ancestral', 'ddim' and 'dpmpp_2m', for an ODE solver on
        InpaintingEDM, and where solver_coefficients raises."""
        name = self.solver if solver is None else solver
        if not isinstance(name, str) or name not in _native.SOLVERS:
            raise ValueError(f"solver is one of {sorted(_native.SOLVERS)} (got {name!r})")
        if name == 'ancestral':
            return None
        if self._SAMPLER == _native.SAMPLER_INPAINT:
            raise ValueError(f"solver={name!r} takes the linker sampler (EDM) only: InpaintingEDM's q(z_s | z_t, x) and "
                             "centre-of-mass projection have no deterministic counterpart here")
        return _native.SOLVERS[name], self.T, self.solver_coefficients(name)

    def _clash_guidance(self, clash_guidance, start_step):
        """_sample_slice's `guide` of a call: (scale, steps, clash table) from `clash_guidance`, or the `clash_guidance`
        attribute when None; None when neither is set or when scale or steps is 0 (the plain loop). ValueError unless a
        pair of a finite real scale >= 0 (a Python or numpy real or a 0-d floating tensor, not a bool) and an integer
        0 <= steps <= T; and, for any setting given, even one that guides nothing, for InpaintingEDM, FC graphs and a
        start_step (`start_step` as the call got it: an int, a sequence or None)."""
        g = self.clash_guidance if clash_guidance is None else clash_guidance
        if g is None:
            return None
        try:
            scale, steps = g
        except (TypeError, ValueError):
            raise ValueError(f"clash_guidance is a pair (scale, steps) (got {g!r})") from None
        if isinstance(scale, (bool, np.bool_)) or not isinstance(scale, numbers.Real) and not (
                torch.is_tensor(scale) and scale.dim() == 0 and scale.dtype.is_floating_point):
            raise ValueError(f"clash_guidance's scale is a real number (got {scale!r})")
        scale = C.c_float(float(scale)).value   # the engine's fp32
        if not math.isfinite(scale) or scale < 0:
            raise ValueError(f"clash_guidance's scale must be finite and >= 0 in fp32 (got {g[0]!r})")
        try:
            if isinstance(steps, (bool, np.bool_)):
                raise TypeError
            steps = operator.index(steps)
        except TypeError:
            raise ValueError(f"clash_guidance's steps is a count of reverse steps (got {steps!r})") from None
        if not 0 <= steps <= self.T:
            raise ValueError(f"clash_guidance's steps must lie in [0, T = {self.T}] (got {steps})")
        if self._SAMPLER == _native.SAMPLER_INPAINT:
            raise ValueError("clash_guidance does not take InpaintingEDM: its loop re-noises the pocket")
        if self.dynamics.graph_type == 'FC':
            raise ValueError("clash_guidance needs a pocket: FC graphs have no pocket rows (use a pocket model on a cut-off "
                             "graph)")
        if start_step is not None:
            raise ValueError("clash_guidance does not take start_step: guidance is a tool of the sampler from noise")
        if scale == 0 or steps == 0:
            return None
        return scale, steps, clash_table(self.is_geom).contiguous()

    def draw_noise(self, n_draws, n_samples, n_nodes, device, generator=None):
        """(n_draws, B, N, 3+F) standard normal. 'reference_stream': the reference's call order -- for every
        draw randn(B,N,3) then randn(B,N,F) (edm.py:328-340, utils.py:189-192) -- so seeds line up."""
        d = self.n_dims + self.in_node_nf
        if self.noise_mode == 'bulk':
            return torch.randn((n_draws, n_samples, n_nodes, d), device=device, generator=generator)
        # two launches per draw (straight into contiguous slabs: `out=` consumes the generator exactly like a fresh randn
        # of that shape) and one interleaving copy at the end, instead of four launches per draw
        zx = torch.empty((n_draws, n_samples, n_nodes, self.n_dims), device=device, dtype=torch.float32)
        zh = torch.empty((n_draws, n_samples, n_nodes, self.in_node_nf), device=device, dtype=torch.float32)
        for r in range(n_draws):
            torch.randn((n_samples, n_nodes, self.n_dims), generator=generator, out=zx[r])
            torch.randn((n_samples, n_nodes, self.in_node_nf), generator=generator, out=zh[r])
        return torch.cat([zx, zh], dim=3)

    # ---- what the two samplers differ in: the device sampler, the number of draws and how a noise tensor is drawn ----
    _SAMPLER = _native.SAMPLER_LINKER

    def _n_draws(self, resamplings=1):
        return self.T + 2

    def _draw_tensor(self, n_samples, n_nodes, device, node_mask, fragment_mask, resamplings=1):
        return self.draw_noise(self.T + 2, n_samples, n_nodes, device)

    def _draws_replaced(self):
        """A draw_noise replaced on the instance supplies the draws instead of the device-side stream."""
        return 'draw_noise' in self.__dict__

    def _sampler_tensors(self, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context):
        """The engine's inputs on x's device, as keyword arguments of `distributed.slice_sampler_inputs`: the normalised xh
        (B,N,3+F) fp32 under 'x', the node mask int8, fragment / linker masks fp32, the flattened FC edge mask int8 (None on
        cut-off graphs) and the context fp32."""
        n_samples, n_nodes = x.size(0), x.size(1)
        dev = x.device
        xn, hn = self.normalize(x, h)
        xh = torch.cat([xn, hn], dim=2).to(torch.float32).contiguous()
        prep = lambda v, dt: None if v is None else v.detach().to(device=dev, dtype=dt).contiguous()
        em = None
        if self.dynamics.graph_type == 'FC' and edge_mask is not None:
            em = prep(edge_mask.reshape(-1), torch.int8)
            assert em.numel() == n_samples * n_nodes * n_nodes
        ctx = None if context is None else prep(
            context.reshape(n_samples, n_nodes, self.dynamics.context_node_nf), torch.float32)   # wrong width -> raises
        return dict(x=xh, node_mask=prep(node_mask.reshape(n_samples, n_nodes), torch.int8),
                    fragment_mask=prep(fragment_mask.reshape(n_samples, n_nodes), torch.float32),
                    linker_mask=prep(linker_mask.reshape(n_samples, n_nodes), torch.float32), edge_mask=em, context=ctx)

    def _noise(self, noise, x, node_mask, fragment_mask, start_step=None, resamplings=1):
        """(on_device, noise): the device-side stream unless a tensor is injected (tests), the draw function is replaced, or
        another mode is set; otherwise the whole batch's draws on x's device -- t0 + 2 of them from a start step t0, those
        of `resamplings` passes per step for the inpainting sampler."""
        n_samples, n_nodes = x.size(0), x.size(1)
        dev = x.device
        on_device = (noise is None and dev.type == 'cuda' and self.noise_mode == 'reference_stream'
                     and not self._draws_replaced())
        n_draws = self._n_draws(resamplings) if start_step is None else start_step + 2
        if not on_device:
            if noise is None:
                noise = (self._draw_tensor(n_samples, n_nodes, dev, node_mask, fragment_mask, resamplings) if start_step is None
                         else self.draw_noise(n_draws, n_samples, n_nodes, dev))
            noise = noise.to(device=dev, dtype=torch.float32).contiguous()
            assert noise.shape == (n_draws, n_samples, n_nodes, self.n_dims + self.in_node_nf), noise.shape
        return on_device, noise

    def start_scalars(self, t0, n_samples=1):
        """(alpha_t0, sigma_t0) of q(z_t0 | x) as EDM.forward evaluates them (edm.py:50-65): t = t0 / T on an (n_samples, 1)
        fp32 CPU tensor, gamma(t), then sqrt(sigmoid(-gamma)) and sqrt(sigmoid(gamma)). Like step_coefficients, the values
        are those of torch's CPU kernels at this batch size."""
        g = self._cpu_gamma()(torch.full((n_samples, 1), fill_value=float(t0)) / self.T)
        return float(self.alpha(g)[0]), float(self.sigma(g)[0])

    def fixed_atom_scalars(self, n_samples=1):
        """The (T + 1, 2) scalars of dl_set_fixed_atoms as a flat ctypes float array: row r < T, in step_coefficients' row
        order (step s = T-1-r), holds start_scalars(s, n_samples) -- the (alpha_s, sigma_s) of q(z_s | x) a kept row is
        drawn from at that step -- and row T holds start_scalars(T, n_samples), where a call from noise starts its kept
        rows. A row that starts at t0 therefore sees the same scalars at its start and in the row of step t0. Cached like
        step_coefficients."""
        T = self.T
        key = ('fixed', T, n_samples, self.gamma.gamma._version, self.gamma.gamma.data_ptr())
        cache = self.__dict__.setdefault('_coef_cache', {})
        if key in cache:
            return cache[key]
        out = (C.c_float * (2 * (T + 1)))()
        for r in range(T + 1):
            out[2 * r], out[2 * r + 1] = self.start_scalars(T - 1 - r if r < T else T, n_samples)
        if len(cache) >= 8:
            cache.pop(next(iter(cache)))
        cache[key] = out
        return out

    def _fixed_atoms(self, fixed_atoms, x, h, node_mask, fragment_mask, linker_mask, context, what="fixed_atoms"):
        """The (B, N) int8 flags on x's device of the linker rows a call keeps, or None without `fixed_atoms` or when it
        flags no row (the plain call). ValueError for InpaintingEDM, a shape other than (B, N) or (B, N, 1), a flag on a
        row that is not a live linker row (fragment, pocket or padding rows), and a flagged row whose types h are not a
        one-hot."""
        if fixed_atoms is None:
            return None
        if self._SAMPLER == _native.SAMPLER_INPAINT:
            raise ValueError("fixed_atoms takes the linker sampler (EDM) only: InpaintingEDM samples every atom and "
                             "re-noises the known ones itself")
        B, N = x.shape[:2]
        if not torch.is_tensor(fixed_atoms) or tuple(fixed_atoms.shape) not in ((B, N), (B, N, 1)):
            got = tuple(fixed_atoms.shape) if torch.is_tensor(fixed_atoms) else type(fixed_atoms).__name__
            raise ValueError(f"{what} must be a (B, N) or (B, N, 1) tensor for B = {B}, N = {N} (got {got})")
        dev = x.device
        flags = fixed_atoms.detach().reshape(B, N).to(dev) != 0
        if not flags.any():
            return None
        live_linker = ((node_mask.detach().reshape(B, N).to(dev) != 0) & (linker_mask.detach().reshape(B, N).to(dev) != 0)
                       & (fragment_mask.detach().reshape(B, N).to(dev) == 0))
        if context is not None and self.dynamics.graph_type != 'FC':
            live_linker &= context.detach()[..., -1].reshape(B, N).to(dev) == 0
        off = flags & ~live_linker
        if off.any():
            b, n = (int(v) for v in off.nonzero()[0])
            raise ValueError(f"{what}: row {n} of molecule {b} is flagged but is not a linker row; only linker atoms can be "
                             "kept (fragment and pocket atoms are kept anyway, padding rows hold no atom)")
        types = h.detach().reshape(B, N, -1).to(dev)[flags]
        if not (((types == 0) | (types == 1)).all(dim=1) & (types == 1).sum(dim=1).eq(1)).all():
            raise ValueError(f"{what}: a kept row's types h must be a one-hot, as it is decoded into chain[0]")
        return flags.to(torch.int8).contiguous()

    def _fixed(self, flags, n_samples):
        """_enqueue_batch's `fixed` of flags returned by _fixed_atoms: (flags, scalars at n_samples), or None."""
        return None if flags is None else (flags, self.fixed_atom_scalars(n_samples))

    def _linker_types(self, linker_types, n_samples, fixed=None, h=None, what="linker_types"):
        """The (B,) CPU int32 masks of the type channels a call's linker atoms may take (bit c: channel c), or None without
        `linker_types` or when it allows every type (the plain call). `linker_types` is a (F,) bool tensor, one set for the
        call, or (B, F), one per molecule; `fixed` (the flags of _fixed_atoms, or None) and the one-hot `h` are the kept rows,
        whose types must be allowed. ValueError for InpaintingEDM, another shape or dtype, and a molecule that allows no
        type."""
        if linker_types is None:
            return None
        if self._SAMPLER == _native.SAMPLER_INPAINT:
            raise ValueError("linker_types takes the linker sampler (EDM) only: InpaintingEDM generates its atoms in its own "
                             "update")
        F = self.in_node_nf
        m = linker_types.detach() if torch.is_tensor(linker_types) else None
        if m is None or m.dtype != torch.bool or tuple(m.shape) not in ((F,), (n_samples, F)):
            got = (f"{m.dtype} of shape {tuple(m.shape)}" if m is not None else type(linker_types).__name__)
            raise ValueError(f"{what} must be a bool tensor of shape (F,) or (B, F) for F = {F}, B = {n_samples} (got {got})")
        m = m.cpu().expand(n_samples, F)
        empty = (~m.any(dim=1)).nonzero()
        if len(empty):
            raise ValueError(f"{what}: molecule {int(empty[0])} allows no atom type")
        if m.all():
            return None
        if fixed is not None:
            kept = fixed.cpu() != 0
            types = h.detach().reshape(n_samples, kept.shape[1], F).cpu().argmax(dim=2)
            off = kept & ~torch.gather(m, 1, types)
            if off.any():
                b, n = (int(v) for v in off.nonzero()[0])
                raise ValueError(f"{what}: row {n} of molecule {b} is kept (fixed_atoms) but its type {int(types[b, n])} "
                                 "is one the molecule's set excludes")
        return (m.to(torch.int64) << torch.arange(F)).sum(dim=1).to(torch.int32).contiguous()

    def _types(self, masks, n_samples):
        """_enqueue_batch's `types` of masks returned by _linker_types: (masks, F, scalars at n_samples), or None."""
        return None if masks is None else (masks, self.in_node_nf, self.fixed_atom_scalars(n_samples))

    def _start(self, start_step, n_samples):
        """(t0, alpha_t0, sigma_t0) of a call of n_samples molecules that starts at step `start_step`, or None for one that
        starts from noise at T; for a 1-D sequence or integer tensor of one step per molecule, their StartSteps, every
        scalar evaluated at n_samples. Raises ValueError unless every step is an int with 0 <= t0 <= T, and for a sequence
        of another length."""
        if start_step is None:
            return None
        if torch.is_tensor(start_step) and start_step.dim() == 1 or isinstance(start_step, (list, tuple, range)):
            if torch.is_tensor(start_step):
                if start_step.dtype.is_floating_point or start_step.dtype.is_complex or start_step.dtype == torch.bool:
                    raise ValueError(f"start_step is a tensor of integer steps (got {start_step.dtype})")
                start_step = start_step.tolist()
            t0 = [self._start_step(v) for v in start_step]
            if len(t0) != n_samples:
                raise ValueError(f"start_step holds {len(t0)} steps for a batch of {n_samples} molecules")
            scalars = {t: self.start_scalars(t, n_samples) for t in sorted(set(t0))}
            return StartSteps(t0, [scalars[t][0] for t in t0], [scalars[t][1] for t in t0])
        t0 = self._start_step(start_step)
        return (t0,) + self.start_scalars(t0, n_samples)

    def _start_step(self, v):
        """v as a start step: an int in [0, T], else ValueError."""
        try:
            if isinstance(v, bool):
                raise TypeError
            t0 = operator.index(v)
        except TypeError:
            raise ValueError(f"start_step is an integer step (got {v!r})") from None
        if not 0 <= t0 <= self.T:
            raise ValueError(f"start_step must lie in [0, T = {self.T}] (got {t0})")
        return t0

    def _nan_exception(self, flags, start):
        """The FoundNaNException of (B,) NaN flags. The engine tags a flag with the row of the loop it ran; from a start step
        t0 that loop begins at row T - t0 of the table, so the tag is moved there and first_step names the table's row."""
        flags = flags.cpu().tolist()
        if isinstance(start, StartSteps):
            flags = [f + ((self.T - t0) << 8) if f >> 8 else f for f, t0 in zip(flags, start.t0)]
        elif start is not None:
            flags = [f + ((self.T - start[0]) << 8) if f >> 8 else f for f in flags]
        return nan_exception_class()(flags=flags)

    def _per_molecule_seeds(self, seeds, noise, batch_slice, x):
        """The (B,) int64 seeds on x's device when this call samples the per-molecule stream -- `seeds` are given, or
        noise_mode is 'per_molecule' and no noise tensor is -- else None. Records them in `last_seeds` (None otherwise)."""
        self.last_seeds = None
        if seeds is None and (self.noise_mode != 'per_molecule' or noise is not None):
            return None
        what = "seeds" if seeds is not None else "noise_mode='per_molecule'"
        if noise is not None:
            raise ValueError("seeds and noise= both supply the draws: pass one of them")
        if self._draws_replaced():
            raise ValueError(f"{what} selects the device-side per-molecule stream, but this model's draw function is "
                             "replaced; restore it or inject the noise")
        if batch_slice is not None:
            raise ValueError(f"{what} does not take batch_slice: the seeds already name the molecules, so pass each slice "
                             "its rows of the seeds")
        cpu = None if seeds is None else seeds_tensor(seeds, x.size(0))
        if x.device.type != 'cuda':
            raise ValueError(f"{what} needs CUDA inputs (got {x.device})")
        if cpu is None:
            with torch.cuda.device(x.device):
                dev_seeds = draw_seeds(x.size(0), x.device)
            cpu = dev_seeds.cpu()
        else:
            dev_seeds = cpu.to(x.device)
        self.last_seeds = cpu
        return dev_seeds

    def _nan_retries(self, nan_retries, seeds, noise, batch_slice, x):
        """The recovery rounds of a call: `nan_retries`, or the `nan_retries` attribute when None. More than 0 needs the
        per-molecule stream on CUDA inputs, and no noise tensor, replaced draw function or batch_slice."""
        n = self.nan_retries if nan_retries is None else nan_retries
        try:
            if isinstance(n, bool):
                raise TypeError
            n = operator.index(n)
        except TypeError:
            raise ValueError(f"nan_retries is a count of rounds (got {n!r})") from None
        if n < 0:
            raise ValueError(f"nan_retries must be >= 0 (got {n})")
        if n >= 1 << 31:
            raise ValueError(f"nan_retries {n} does not fit an int32")
        if n == 0:
            return 0
        self._refuse_without_new_draws('nan_retries', seeds, noise, batch_slice)
        if x.device.type != 'cuda':
            raise ValueError(f"nan_retries needs CUDA inputs (got {x.device})")
        return n

    def _refuse_without_new_draws(self, name, seeds, noise, batch_slice):
        """Raises ValueError when the option `name` (nan_retries, require_connected or require_valid) could not give one
        molecule new draws: it needs the per-molecule stream, and no noise tensor, replaced draw function or batch_slice."""
        if noise is not None:
            raise ValueError(f"{name} resamples molecules with new seeds; an injected noise= tensor has no new draws")
        if self._draws_replaced():
            raise ValueError(f"{name} needs the device-side per-molecule stream, but this model's draw function is replaced")
        if batch_slice is not None:
            raise ValueError(f"{name} does not take batch_slice: pass each slice its rows of the seeds instead")
        if seeds is None and self.noise_mode != 'per_molecule':
            raise ValueError(f"{name} needs per-molecule streams: pass seeds= or set noise_mode='per_molecule' (the "
                             f"batch stream, noise_mode={self.noise_mode!r}, cannot give one molecule new draws)")

    def _require_check(self, name, value, seeds, noise, batch_slice, x):
        """Whether a call runs the molecule check `name` (require_connected or require_valid): `value`, or the attribute of
        that name when None. True needs what nan_retries > 0 needs -- the per-molecule stream on CUDA inputs, no noise
        tensor, replaced draw function or batch_slice -- and the bond tables of `is_geom`."""
        c = getattr(self, name) if value is None else value
        if not isinstance(c, bool):
            raise ValueError(f"{name} is True or False (got {c!r})")
        if not c:
            return False
        self._refuse_without_new_draws(name, seeds, noise, batch_slice)
        if self.is_geom is None:
            raise ValueError(f"{name} needs the bond tables: build the EDM with is_geom=True (GEOM / MOAD atom "
                             "types) or False (ZINC), or set edm.is_geom")
        if x.device.type != 'cuda':
            raise ValueError(f"{name} needs CUDA inputs (got {x.device})")
        return True

    def _checks(self, require_connected, require_valid, seeds, noise, batch_slice, x, require_clash_free=None,
                require_unique=None, require_novel=None, require_ring_sizes=None, require_anchors=None):
        """The molecule checks of a call as the OR of _native.CHECK_*; 0 checks nothing."""
        return ((_native.CHECK_CONNECTED if self._require_check('require_connected', require_connected, seeds, noise,
                                                                batch_slice, x) else 0) |
                (_native.CHECK_VALENCE if self._require_check('require_valid', require_valid, seeds, noise, batch_slice, x)
                 else 0) |
                (_native.CHECK_CLASH if self._require_clash_free(require_clash_free, seeds, noise, batch_slice, x) else 0) |
                (_native.CHECK_UNIQUE if self._require_check('require_unique', require_unique, seeds, noise, batch_slice, x)
                 else 0) |
                (_native.CHECK_NOVEL if self._require_novel(require_novel, seeds, noise, batch_slice, x) else 0) |
                (_native.CHECK_RINGS if self._require_ring_sizes(require_ring_sizes, seeds, noise, batch_slice, x) else 0) |
                (_native.CHECK_ANCHORS if self._require_check('require_anchors', require_anchors, seeds, noise, batch_slice, x)
                 else 0))

    def _anchors(self, check, anchors, x, node_mask, linker_mask, context, what="anchors"):
        """The (B, N) int8 anchor flags on x's device of a call with the checks `check`, or None without CHECK_ANCHORS
        (`anchors` is then not read). ValueError without `anchors`, for a shape other than (B, N) or (B, N, 1), for a flag
        on a linker row or (on cut-off graphs) a pocket row, and for a molecule with no anchor on its atoms."""
        if not check & _native.CHECK_ANCHORS:
            return None
        B, N = x.shape[:2]
        if anchors is None:
            raise ValueError("require_anchors needs the anchor flags: pass anchors=, a (B, N) or (B, N, 1) tensor that is "
                             "non-zero on each molecule's anchor atoms (the batch's 'anchors', as generate.py --anchors "
                             "sets them)")
        if not torch.is_tensor(anchors) or tuple(anchors.shape) not in ((B, N), (B, N, 1)):
            got = tuple(anchors.shape) if torch.is_tensor(anchors) else type(anchors).__name__
            raise ValueError(f"{what} must be a (B, N) or (B, N, 1) tensor for B = {B}, N = {N} (got {got})")
        flags = anchors.detach().reshape(B, N).to(x.device) != 0
        on_linker = flags & (linker_mask.detach().reshape(B, N).to(x.device) != 0)
        if on_linker.any():
            b = int(on_linker.any(1).nonzero()[0])
            raise ValueError(f"{what}: molecule {b} has an anchor flag on a linker row; anchors are fragment atoms")
        if self.dynamics.graph_type != 'FC' and context is not None:
            on_pocket = flags & (context.detach()[..., -1].reshape(B, N).to(x.device) != 0)
            if on_pocket.any():
                b = int(on_pocket.any(1).nonzero()[0])
                raise ValueError(f"{what}: molecule {b} has an anchor flag on a pocket row; anchors are ligand fragment "
                                 "atoms")
        none = ~(flags & (node_mask.detach().reshape(B, N).to(x.device) != 0)).any(1)
        if none.any():
            b = int(none.nonzero()[0])
            raise ValueError(f"{what}: molecule {b} has no anchor atom, so require_anchors asks nothing of it; a batch "
                             "built without --anchors has none (set the anchors, or sample without require_anchors)")
        return flags.to(torch.int8).contiguous()

    def _require_ring_sizes(self, value, seeds, noise, batch_slice, x):
        """_require_check for require_ring_sizes, which also needs the `allowed_ring_sizes` policy."""
        if (self.require_ring_sizes if value is None else value) is True and self.allowed_ring_sizes is None:
            raise ValueError("require_ring_sizes needs the ring sizes to allow: set edm.allowed_ring_sizes (ints >= 3, 63 "
                             "meaning 63 or more atoms; e.g. range(5, 7) for five- and six-membered rings only)")
        if (self.require_ring_sizes if value is None else value) is True:
            ring_size_mask(self.allowed_ring_sizes)   # ValueError for anything but ints in [3, 63]
        return self._require_check('require_ring_sizes', value, seeds, noise, batch_slice, x)

    def _require_novel(self, value, seeds, noise, batch_slice, x):
        """_require_check for require_novel, which also needs the `known_linkers` set."""
        if (self.require_novel if value is None else value) is True and self.known_linkers is None:
            raise ValueError("require_novel needs the known linker hashes: set edm.known_linkers (e.g. "
                             "molecule_builder.known_linkers of the training set)")
        return self._require_check('require_novel', value, seeds, noise, batch_slice, x)

    def _hash_sets(self, check, exclude_hashes, dev):
        """(known, seen) of a call with the checks `check`: `known_linkers` with CHECK_NOVEL and `exclude_hashes` (with
        CHECK_UNIQUE only), each sorted in unsigned order on `dev` (molecule_builder.sort_unsigned), or None; None without
        either."""
        def sorted_set(name, t):
            if not torch.is_tensor(t) or t.dim() != 1 or t.dtype != torch.int64:
                raise ValueError(f"{name} is a 1-D int64 tensor of uint64 hash bits (got "
                                 f"{type(t).__name__ if not torch.is_tensor(t) else f'{t.dtype} of shape {tuple(t.shape)}'})")
            return sort_unsigned(t.detach().to(dev))
        if exclude_hashes is not None and not check & _native.CHECK_UNIQUE:
            raise ValueError("exclude_hashes feeds the uniqueness verdict: it needs require_unique=True")
        known = sorted_set('known_linkers', self.known_linkers) if check & _native.CHECK_NOVEL else None
        seen = None if exclude_hashes is None else sorted_set('exclude_hashes', exclude_hashes)
        return None if known is None and seen is None else (known, seen)

    def _require_clash_free(self, value, seeds, noise, batch_slice, x):
        """_require_check for require_clash_free, which also needs a pocket that stays put: a cut-off (pocket) graph and the
        linker sampler -- the inpainting sampler re-noises the pocket."""
        if (self.require_clash_free if value is None else value) is True:
            if self._SAMPLER == _native.SAMPLER_INPAINT:
                raise ValueError("require_clash_free does not take InpaintingEDM: its loop re-noises the pocket")
            if self.dynamics.graph_type == 'FC':
                raise ValueError("require_clash_free needs a pocket: FC graphs have no pocket rows (use a pocket model on a "
                                 "cut-off graph such as '4A' or 'FC-10A-4A')")
        return self._require_check('require_clash_free', value, seeds, noise, batch_slice, x)

    def _linker_sizes(self, linker_sizes, seeds, noise, batch_slice, start_step, x, linker_mask):
        """The device tensors (logits, size table, n_frag, normalised linker_x, attempt-0 sizes) of a call's `linker_sizes`
        (a LinkerSizes for the (B, N) template x), or None without one. ValueError for what cannot redraw one molecule's
        size: InpaintingEDM, start_step, no `seeds`, noise=, a replaced draw function, batch_slice, host inputs, and a
        template of fewer rows than max(n_frag) + max(sizes)."""
        if linker_sizes is None:
            return None
        if self._SAMPLER == _native.SAMPLER_INPAINT:
            raise ValueError("linker_sizes does not take InpaintingEDM: it samples every atom and has no linker size")
        if start_step is not None:
            raise ValueError("linker_sizes does not take start_step: partial diffusion varies the batch's own linker, "
                             "whose size is given")
        self._refuse_without_new_draws('linker_sizes', seeds, noise, batch_slice)
        if seeds is None:
            raise ValueError("linker_sizes needs seeds=: the template's sizes are dl_size_draw's attempt-0 draws from them")
        if x.device.type != 'cuda':
            raise ValueError(f"linker_sizes needs CUDA inputs (got {x.device})")
        if not isinstance(linker_sizes, LinkerSizes):
            raise ValueError(f"linker_sizes is an edm.LinkerSizes at this level (got {type(linker_sizes).__name__}); "
                             "ddpm.sample_chain resolves a size model, a range or an int")
        B, N = x.shape[:2]
        dev = x.device
        table = torch.tensor([operator.index(v) for v in linker_sizes.sizes], dtype=torch.int32)
        logits = linker_sizes.logits.detach().to(device=dev, dtype=torch.float32).contiguous()
        n_frag = torch.as_tensor(linker_sizes.n_frag).detach().reshape(-1).to(device='cpu', dtype=torch.int32)
        if table.numel() < 1 or (table < 0).any():
            raise ValueError("linker_sizes.sizes must hold at least one size, each >= 0")
        if tuple(logits.shape) != (B, table.numel()) or n_frag.numel() != B or linker_sizes.linker_x.numel() != 3 * B:
            raise ValueError(f"linker_sizes must hold (B, C) logits, B n_frag and (B, 3) linker_x for B = {B} molecules and "
                             f"C = {table.numel()} sizes (got {tuple(logits.shape)}, {n_frag.numel()} and "
                             f"{tuple(linker_sizes.linker_x.shape)})")
        need = int(n_frag.max()) + int(table.max())
        if N < need:
            raise ValueError(f"linker_sizes: the template has {N} rows, fewer than its capacity max(n_frag) + max(sizes) = "
                             f"{need}, which every redrawn size must fit")
        linker_x = linker_sizes.linker_x.detach().to(device=dev, dtype=torch.float32).reshape(B, 3) / self.norm_values[0]
        sizes = linker_mask.detach().reshape(B, N).to(dev).sum(1).to(torch.int32)
        return logits, table.to(dev), n_frag.to(dev), linker_x.contiguous(), sizes

    def _check_tables(self, check):
        """The CPU tables the checks `check` read with this model's atom types (molecule_builder.check_tables)."""
        return check_tables(self.is_geom, check)

    def _head(self, n_samples, n_nodes, keep_frames, t):
        ptr = lambda v: None if v is None else v.data_ptr()
        return (self._SAMPLER, n_samples, n_nodes, self.T, keep_frames, ptr(t['x']), ptr(t['node_mask']),
                ptr(t['fragment_mask']), ptr(t['linker_mask']), ptr(t['edge_mask']), ptr(t['context']))

    def _norm(self):
        return (C.c_float * 3)(float(self.norm_values[0]), float(self.norm_values[1]), float(self.norm_biases[1]))

    @torch.no_grad()
    def sample_chain(self, x, h, node_mask, fragment_mask, linker_mask, edge_mask, context, keep_frames=None,
                     noise=None, batch_slice=None, seeds=None, nan_retries=None, require_connected=None, start_step=None,
                     require_valid=None, require_clash_free=None, linker_sizes=None, require_unique=None,
                     require_novel=None, exclude_hashes=None, resamplings=None, require_ring_sizes=None,
                     require_anchors=None, anchors=None, clash_guidance=None, solver=None, fixed_atoms=None,
                     linker_types=None):
        """Same contract as the reference (edm.py:126-176): returns (keep_frames, B, N, 3+F); chain[0] holds the
        final coordinates and one-hot atom types. `noise` optionally injects the (T+2,B,N,3+F) draws (tests).
        `start_step` = t0, an int in [0, T] (partial diffusion; None, the default, samples from noise at T): the linker on
        the linker_mask rows of x, h is varied instead of sampled from noise. The loop starts from q(z_t0 | x) as EDM.forward
        draws it (edm.py:67-74) -- eps drawn as z_T is drawn today, z = xh * fragment_mask + (alpha_t0 xh + sigma_t0 eps) *
        linker_mask with the scalars of start_scalars -- and runs steps t0-1 .. 0 and the final step as the plain loop runs
        them. The draws are eps, one per step and the final draw: t0 + 2 (noise= holds t0 + 2 slabs; the batch stream
        advances by t0 + 2 draws; per-molecule streams use their draws 0 .. t0+1). Frames that no step below t0 writes are
        zero. t0 bounds how far a sample may move from its input; t0 = T is not the plain sampler (z_T keeps alpha_T xh).
        Everything below -- seeds, recovery rounds, devices, batch_slice -- applies unchanged.
        `start_step` may also be a 1-D sequence, or integer tensor, of one t0 per molecule (dl_set_start_steps): molecule b
        is then sampled as the call with start_step=t0[b] samples it on the same batch, with the same seeds or noise rows
        (scalars of start_scalars(t0[b], B)) -- bit for bit on the SIMT edge path, on the tensor-core path within the
        per-molecule rule -- and an all-equal sequence is the int call bit for bit. noise= then holds max(t0) + 2 slabs, of
        which row b reads 0 .. t0[b]+1. One launch computes only the molecules that have started: sum_b (t0[b] + 1)
        molecule-steps. It needs per-molecule streams (seeds or noise_mode='per_molecule') or noise=, works with the
        recovery rounds, every require_* and `devices`, and raises ValueError for a wrong length, an entry that is not an
        int in [0, T], the batch stream, InpaintingEDM, sample_fn and linker_sizes.
        `batch_slice=(b0, B_full)`: the inputs are rows [b0, b0+B) of a batch of B_full molecules (strong scaling,
        distributed.sample_chain_sharded); the device-side noise is then those rows of the full batch's draws.
        `seeds` (B ints, or an integer tensor; CUDA inputs): molecule b draws exactly what the reference draws for it
        sampled alone after torch.cuda.manual_seed(seeds[b]) (dl_sample_chain_seeded), whatever noise_mode is. Its chain
        then depends neither on its batch-mates, the batch size, its row, the padding nor a split over devices -- on the
        tensor-core path while no sample diverges far enough for the node GEMM to rescale a tile's fp16 operands (tiles
        span molecules, DESIGN.md section 6), and with aggregation_method='mean' on FC graphs except for the padding,
        which the reference's mean counts. The generator does not advance. noise_mode='per_molecule' samples that stream
        without `seeds` from draw_seeds. Either way `last_seeds` records the seeds; replaying one molecule with its seed
        reproduces its row, including a NaN divergence, so retry a diverged molecule with a new seed.
        `nan_retries` (None: the `nan_retries` attribute, default 0) does that on the device: after the loop, up to that many
        rounds resample only the molecules whose flags are set, as a sub-batch, with seeds dl_retry_seed(seed, round)
        (dl_sample_chain_retry). It needs the per-molecule stream -- `seeds` or noise_mode='per_molecule' -- and raises
        ValueError with the batch stream, noise=, a replaced draw function, host inputs or batch_slice. Rows that did not fail
        are untouched, bit for bit; `last_seeds[b]` is then the seed that produced row b, so molecule b sampled alone with it
        reproduces the row -- bit for bit on the SIMT edge path, and on the tensor-core path while no node tile rescales
        (DESIGN.md section 6) -- and `last_attempts[b]` the round (0 = the first draw). Rows that still fail after the last
        round raise FoundNaNException with their batch-global indices only; its `chain` attribute holds the recovered chain.
        `require_connected` (None: the `require_connected` attribute, default False) adds a second reason to resample a row:
        its final molecule -- chain[0]'s atoms, without the pocket on cut-off graphs, bonded where get_bond_order > 0 with
        the tables of `is_geom` -- is in more than one piece (dl_sample_chain_retry's checks). The check runs on the
        device after the loop and after every round; the rounds are the nan_retries rounds, so nan_retries=0 only reports.
        A resampled row replaces the old one unless the old one was finite and the new one diverged. Rows that are still
        disconnected after the last round are returned; `last_connected` (B,) CPU bool tells which rows are connected. It
        raises ValueError where nan_retries does, and without `is_geom`.
        `require_valid` (None: the `require_valid` attribute, default False) adds a third, in the same rounds and with the
        same refusals: some atom of that molecule carries more bond order -- the sum of get_bond_order over its pairs -- than
        molecule_builder.max_valence_table allows its element (both checks share one launch). `last_valid` (B,) CPU bool tells which rows pass. This is "explicit valence within the table", how
        build_molecule's molecules are expected to fail RDKit's sanitization; that has not been verified against RDKit.
        A row whose fragments alone break the rule cannot be repaired by a new linker: it is resampled every round and
        comes back flagged, so vet inputs with molecule_builder.valence_ok. Either flag alone or both.
        `require_clash_free` (None: the `require_clash_free` attribute, default False) adds a fourth, on cut-off (pocket)
        graphs, in the same rounds and launch: some linker atom of chain[0] lies closer to a pocket atom than
        molecule_builder.clash_table(is_geom) allows for the two atom types (this project's own predicate, stated at
        dl_molecule_checks in the header; fragment atoms are not checked). `last_clash_free` (B,) CPU bool tells which rows
        pass. Refusals as for require_valid, plus ValueError on FC graphs and for InpaintingEDM.
        `require_unique` (None: the `require_unique` attribute, default False) adds a fifth, in the same rounds and launch:
        the row's bond graph -- chain[0]'s checked atoms, types and get_bond_order orders -- repeats a batch-mate's, by the
        graph hash of molecule_builder.graph_hashes. After the loop every row is a candidate; in a round, the rows it
        resampled are. A candidate keeps the bit unless its hash equals that of a row outside the candidates that passes
        every required check, or of an earlier candidate that is finite and passes every other required check. Rows that
        pass are never resampled, and no two returned rows that pass every required check share a hash (a row failing
        another check blocks no one, so two such rows may keep the bit with one hash). The group is this call: uniqueness
        across calls is the caller's, with `last_graph_hashes` (B,) CPU int64 (one dl_molecule_hash of the returned
        chain[0]). `last_unique` (B,) CPU bool tells which rows pass. Equal hashes mean isomorphic graphs up to the hash's
        limits (1-WL-equivalent graphs and 64-bit collisions hash equal; stereochemistry is ignored; not verified against
        RDKit canonical SMILES). Refusals as for require_valid, plus ValueError when `devices` splits the batch into more
        than one slice: the slices recover on their engines independently, so no verdict sees the whole batch.
        `exclude_hashes` (a 1-D int64 tensor of graph hashes, e.g. an earlier call's `last_graph_hashes`; needs
        require_unique) extends that group across calls: its hashes count as keepers, so no returned row that passes every
        required check has a hash among them. It is sorted in unsigned order on the device for every call.
        `require_novel` (None: the `require_novel` attribute, default False) adds a sixth, in the same rounds and launch: the
        row's linker hash -- molecule_builder.linker_hashes of chain[0], the graph hash of its checked atoms on the
        linker_mask rows (with a size redraw, the row's returned linker rows) -- is in `known_linkers`, a 1-D int64 tensor of
        uint64 hashes in any order (molecule_builder.known_linkers of a training set), sorted in unsigned order on the
        device for every call. `last_novel` (B,) CPU bool tells which rows pass, `last_linker_hashes` (B,) CPU int64 holds
        every row's linker hash, as the check launch computed it for the bit. Novel means "by this hash, against linkers hashed the same way", with the hash's limits
        above. Refusals as for require_valid, plus ValueError without `known_linkers`.
        `require_ring_sizes` (None: the `require_ring_sizes` attribute, default False) adds a seventh, in the same rounds
        and launch: some bond of chain[0] with a linker end (a checked atom on the linker_mask rows, with a size redraw the
        row's returned linker rows) has a smallest ring whose size is not in `allowed_ring_sizes`, an iterable of ints >= 3
        where 63 stands for 63 or more atoms (molecule_builder.ring_sizes, stated at DL_CHECK_RINGS in the header). The
        bonds are decided over all the checked atoms, so rings through the fragment count; rings of fragment atoms alone do
        not. `last_ring_sizes_ok` (B,) CPU bool tells which rows pass, `last_ring_sizes` (B,) CPU int64 holds every row's
        ring-size mask (bit k: a smallest ring of k atoms), the one its bit was decided on. These are rings of bond_orders'
        graph, not RDKit's SSSR. Refusals as for require_valid, plus ValueError without `allowed_ring_sizes`.
        `require_anchors` (None: the `require_anchors` attribute, default False) adds an eighth, in the same rounds, in a
        launch right after the check launch: the linker of chain[0] does not attach by exactly one bond at each anchor and
        nowhere else on the fragments (molecule_builder.attachments, stated at DL_CHECK_ANCHORS in the header). `anchors`
        is a (B, N) or (B, N, 1) tensor, non-zero on each molecule's anchor atoms (the batch's 'anchors'; ddpm.sample_chain
        passes them); a round reads row b's own flags, since its fragment rows keep their positions. The bonds are
        bond_orders', over all the checked atoms. `last_anchors_ok` (B,) CPU bool tells which rows pass. Refusals as for
        require_valid, plus ValueError without `anchors`, for a flag on a linker or pocket row, for a molecule with no
        anchor (nothing would be asked of it) and for the wrong shape.
        `linker_sizes` (a LinkerSizes; ddpm.sample_chain builds it) makes every round redraw the linker size of the rows it
        resamples, from the round's seed (dl_sample_chain_retry's redraw), and rebuild their template rows at that size
        inside the padded template. The inputs must be the template of the sizes dl_size_draw gives `seeds` at attempt 0,
        padded to max(n_frag) + max(sizes) rows or more. `last_sizes` (B,) CPU int32 holds every returned row's size. It
        needs `seeds` and raises ValueError where nan_retries does, with start_step and for InpaintingEDM.
        `resamplings` (None: the `resamplings` attribute, default 1) is InpaintingEDM's; this class raises ValueError for
        anything but 1 (or None), and for a value that is not an int >= 1.
        `clash_guidance` = (scale, steps) (None: the `clash_guidance` attribute, default None) steers the linker away from
        the pocket while it is sampled (dl_set_clash_guidance): after each reverse step s < steps has produced z_s, every
        linker atom i moves by scale * sum_k max(0, r_ik - d_ik) (p_i - p_k) / d_ik over the pocket atoms k, r_ik the
        clash_table(is_geom) distance of the two atom types (argmax of z_s's type channels) in Angstrom, and the remaining
        steps rebuild the linker around it (molecule_builder.clash_guide states the push). It draws nothing, so draws,
        seeds and recovery rounds are as without it; the rounds are guided too. scale = 0 or steps = 0 is the plain call,
        bit for bit. A sampler tool with no claim about chemistry. ValueError for a bool, negative or non-finite scale,
        steps outside [0, T], FC graphs, start_step and InpaintingEDM.
        `solver` (None: the `solver` attribute, default 'ancestral') picks the reverse update (dl_set_solver): 'ancestral'
        is the reference's p(z_s | z_t); 'ddim' (first order) and 'dpmpp_2m' (DPM-Solver++(2M), second order from a row's
        second step on) are deterministic steps of the probability-flow ODE with the same eps-network, meant for a loop
        shortened with `T` (edm.T = 20, as the reference's --n_steps sets it). The final step returns the data prediction
        with no noise, so a sample is a function of its z_T (or its q(z_t0 | x)) alone. The draws stay those of the
        ancestral loop in count and order (only draw 0 is read), so seeds, noise=, the batch stream's offset, start_step in
        both forms (a row's own start step is its first), the recovery rounds (which start their rows afresh),
        linker_sizes, clash_guidance (which pushes z_s after the update) and `devices` work as without it. The effect on
        a trained model's samples is not measured. ValueError for another name, for InpaintingEDM and for T above the
        schedule's timesteps.
        `fixed_atoms` (a (B, N) or (B, N, 1) tensor, non-zero on the linker rows to keep; None, the default, keeps none)
        generates the rest of the linker around the kept atoms (dl_set_fixed_atoms): the kept rows are x's and h's linker
        rows, as start_step reads them, and the other linker rows are sampled -- their inputs are ignored. The kept rows
        stay noisy linker rows, replaced at every step by a draw of q(z_s | x) (replacement, as RePaint keeps known pixels,
        without its re-noising passes): they start from alpha xh + sigma eps_0 at the call's start (T, or start_step in
        either form), step s sets them to alpha_s xh + sigma_s nz_s with the draw the ancestral update reads for the row
        (alpha_s xh + sigma_s eps_0 with an ODE `solver`), with the scalars of fixed_atom_scalars, and chain[0] holds their
        input x and types. The draws are those of the call without it, so seeds, noise=, the batch stream, start_step, the
        recovery rounds (resampled rows keep their kept atoms, which every check counts as linker atoms), clash_guidance
        (which moves only the free linker atoms), `solver`, keep_frames, `devices` and batch_slice work as without it. A
        mask that flags no row is the plain call, bit for bit. ValueError for a flag off the linker rows, a kept row whose
        h is not a one-hot, the wrong shape, InpaintingEDM and linker_sizes.
        `linker_types` (a bool tensor, (F,) for one set of allowed type channels for the call or (B, F) for one per
        molecule; None, the default, uses `edm.linker_types`) gives every linker atom of chain[0] an allowed type
        (dl_set_linker_types): at every step, on every linker row that fixed_atoms does not keep, the data prediction
        xhat = (z_t - sigma_t eps) / alpha_t of an excluded channel is set to the one-hot's normalised off value (0 - bias1)
        / norm1 -- the ancestral update reads eps = (z_t - alpha_t off) / sigma_t instead, with the (alpha_t, sigma_t) of
        fixed_atom_scalars, an ODE `solver` takes xhat itself, 2M history included -- and the final one-hot is the argmax
        over the allowed channels. So the constraint holds by construction, including the rows of recovery rounds and NaN
        retries; intermediate keep_frames frames are continuous states and carry no such guarantee. The draws are those
        of the call without it, so seeds, noise=, the batch stream, start_step, the recovery rounds, linker_sizes,
        clash_guidance, `solver`, keep_frames, `devices` and batch_slice work as without it. A set that allows every type
        is the plain call, bit for bit. ValueError for a molecule that allows no type, the wrong shape or dtype,
        InpaintingEDM, and a fixed_atoms row whose type is excluded.
        The batch is sampled in slices, each on an engine of its own: one covering it on x's device or, with `devices` set
        and no batch_slice, one per listed device (distributed.device_slices). Inputs and draws are prepared once on x's
        device; each slice samples its rows of them with the full batch's step coefficients, several slices from one host
        thread per device, and their chains and NaN flags are copied back. The batch stream advances the generator once."""
        if keep_frames is None:
            keep_frames = self.T
        else:
            assert keep_frames <= self.T
        lib = _native.load_library()
        n_samples = x.size(0)
        dev = x.device
        self.last_attempts = None
        self.last_connected = self.last_valid = self.last_clash_free = self.last_sizes = None
        self.last_unique = self.last_graph_hashes = self.last_novel = self.last_linker_hashes = None
        self.last_ring_sizes_ok = self.last_ring_sizes = None
        self.last_anchors_ok = None
        start = self._start(start_step, n_samples)
        r = self._resamplings(resamplings)
        guide = self._clash_guidance(clash_guidance, start_step)
        ode = self._solver(solver)
        redraw = self._linker_sizes(linker_sizes, seeds, noise, batch_slice, start_step, x, linker_mask)
        retries = self._nan_retries(nan_retries, seeds, noise, batch_slice, x)
        check = self._checks(require_connected, require_valid, seeds, noise, batch_slice, x, require_clash_free,
                             require_unique, require_novel, require_ring_sizes, require_anchors)
        anchor_flags = self._anchors(check, anchors, x, node_mask, linker_mask, context)
        fixed = self._fixed_atoms(fixed_atoms, x, h, node_mask, fragment_mask, linker_mask, context)
        if fixed is not None and redraw is not None:
            raise ValueError("fixed_atoms does not take linker_sizes: a size redraw rebuilds the linker rows at new sizes")
        masks = self._linker_types(self.linker_types if linker_types is None else linker_types, n_samples, fixed, h)
        sets = self._hash_sets(check, exclude_hashes, dev)
        recover = retries > 0 or check != 0 # the recovery entry point: seeds used and attempts come back
        dev_seeds = self._per_molecule_seeds(seeds, noise, batch_slice, x)
        full = self._sampler_tensors(x, h, node_mask, fragment_mask, linker_mask, edge_mask, context)
        on_device, noise = ((False, None) if dev_seeds is not None
                            else self._noise(noise, x, node_mask, fragment_mask, _loop_steps(start), r))
        if isinstance(start, StartSteps) and on_device:
            raise ValueError("per-molecule start steps need per-molecule streams (seeds= or noise_mode='per_molecule') or "
                             f"noise=: the batch stream, noise_mode={self.noise_mode!r}, does not draw per molecule")
        if batch_slice is not None and not on_device:
            raise ValueError("batch_slice needs the device-side noise stream (CUDA tensors, noise_mode='reference_stream')")
        self.dynamics._check_graph_type()
        split = self.devices is not None and batch_slice is None
        slices = device_slices(n_samples, self.devices) if split else [(self.dynamics._device_index(x), 0, 0, n_samples)]
        if not slices:
            raise ValueError("sample_chain needs at least one molecule")
        if check & _native.CHECK_UNIQUE and len(slices) > 1:
            raise ValueError(f"require_unique compares the rows of one engine call, but devices={self.devices!r} splits the "
                             f"batch into {len(slices)} slices that recover independently; sample on one device, or "
                             "deduplicate the slices with last_graph_hashes / molecule_builder.graph_hashes")
        if on_device:
            gen = _generator_of(dev)
            # the device-side stream reproduces torch's randn launch geometry, which depends on the device's SM count
            geometry = lambda i: (torch.cuda.get_device_properties(i).multi_processor_count,
                                  torch.cuda.get_device_properties(i).max_threads_per_multi_processor)
            odd = sorted({s[0] for s in slices if geometry(s[0]) != geometry(gen.device.index)})
            if odd:
                raise ValueError(f"devices {odd} differ from {dev} in SM count or threads per SM, so they cannot reproduce its "
                                 "noise stream; list devices of one model, or inject the noise")
            seed, offset = gen.initial_seed() & 0xFFFFFFFFFFFFFFFF, gen.get_offset()
            b0, b_full = (0, n_samples) if batch_slice is None else map(int, batch_slice)
        engines = self.dynamics.engines([(dev_i, replica) for dev_i, replica, _, _ in slices])
        places = [torch.device('cuda', dev_i) for dev_i, *_ in slices] if split else [dev]
        calls, finish = self._enqueue_batch(lib, full, keep_frames, self.step_coefficients(keep_frames, n_samples), slices,
                                            engines, places, dev, noise=noise, dev_seeds=dev_seeds,
                                            rng=(seed, offset, b0, b_full) if on_device else None, retries=retries, check=check,
                                            start=start, redraw=redraw, sets=sets,
                                            resample=self._resample(r, n_samples), anchors=anchor_flags, guide=guide,
                                            solver=ode, fixed=self._fixed(fixed, n_samples),
                                            types=self._types(masks, n_samples))
        by_device = {}
        for dev_i, c in calls:
            by_device.setdefault(dev_i, []).append(c)
        try:
            if len(slices) == 1:            # on the caller's thread
                with torch.cuda.device(slices[0][0]):
                    calls[0][1]()
            else:
                _run_per_device(by_device)
        except BaseException:
            for dev_i in by_device:         # let the loops that were enqueued finish before their inputs are released
                try:
                    torch.cuda.synchronize(dev_i)
                except Exception:
                    pass
            raise
        out = finish()
        if on_device:
            assert len(set(out['consumed'])) == 1, out['consumed']
            gen.set_offset(offset + out['consumed'][0])
        loop_ms = []
        for (dev_i, _, lo, hi), eng in zip(slices, engines):
            with torch.cuda.device(dev_i):
                loop_ms.append((dev_i, lo, hi, float(lib.dl_last_elapsed_ms(eng))))
        self.last_loop_ms = max(ms for *_, ms in loop_ms)
        self.last_slice_loop_ms = loop_ms if split else None
        if recover:
            self.last_seeds, self.last_attempts = out['used'].cpu(), out['attempts'].cpu()
        if redraw is not None:
            self.last_sizes = (out['sizes'] if recover else redraw[4]).cpu()
        if check & _native.CHECK_CONNECTED:
            self.last_connected = (out['passed'].cpu() & _native.CHECK_CONNECTED) != 0
        if check & _native.CHECK_VALENCE:
            self.last_valid = (out['passed'].cpu() & _native.CHECK_VALENCE) != 0
        if check & _native.CHECK_CLASH:
            self.last_clash_free = (out['passed'].cpu() & _native.CHECK_CLASH) != 0
        if check & _native.CHECK_UNIQUE:
            self.last_unique = (out['passed'].cpu() & _native.CHECK_UNIQUE) != 0
            self.last_graph_hashes = self._graph_hashes(full, out['chain'][0], redraw, out['sizes']).cpu()
        if check & _native.CHECK_NOVEL:
            self.last_novel = (out['passed'].cpu() & _native.CHECK_NOVEL) != 0
            self.last_linker_hashes = out['linker_hashes'].cpu()
        if check & _native.CHECK_RINGS:
            self.last_ring_sizes_ok = (out['passed'].cpu() & _native.CHECK_RINGS) != 0
            self.last_ring_sizes = out['ring_sizes'].cpu()
        if check & _native.CHECK_ANCHORS:
            self.last_anchors_ok = (out['passed'].cpu() & _native.CHECK_ANCHORS) != 0
        if out['bad']:
            exc = self._nan_exception(out['flags'], start)
            if recover:
                exc.chain = out['chain']    # the rows that did not fail, or were recovered, are good molecules
            raise exc
        return out['chain']

    def _graph_hashes(self, full, chain0, redraw, sizes):
        """graph_hashes of a returned chain[0] over the atoms the engine checked: the node mask of the inputs `full` or,
        with a size redraw, of every row's template at its returned size (rows below n_frag as given, then `sizes` linker
        rows); without the pocket on cut-off graphs."""
        nm = full['node_mask']
        if redraw is not None:
            n_frag = redraw[2].to(torch.int64)[:, None]
            rows = torch.arange(nm.shape[1], device=nm.device)[None, :]
            nm = torch.where(rows < n_frag, nm, (rows < n_frag + sizes.to(torch.int64)[:, None]).to(nm.dtype))
        pocket_only = full['context'][..., -1] if self.dynamics.graph_type != 'FC' else None
        return graph_hashes(chain0, nm, self.is_geom, pocket_only)

    # the keyword arguments of sample_chain that make up one request of sample_many
    _REQUEST_INPUTS = ('x', 'h', 'node_mask', 'fragment_mask', 'linker_mask', 'edge_mask', 'context')

    @torch.no_grad()
    def sample_many(self, requests, keep_frames=None, seeds=None, nan_retries=None, require_connected=None,
                    max_molecules=256, start_step=None, require_valid=None, require_clash_free=None, linker_sizes=None,
                    require_novel=None, resamplings=None, require_ring_sizes=None, require_anchors=None,
                    clash_guidance=None, solver=None):
        """Samples many requests -- each a dict of sample_chain's inputs (x, h, node_mask, fragment_mask, linker_mask,
        edge_mask, context) holding its own (B_k, N_k) batch on one CUDA device -- in a few shared launches, and returns their
        (keep_frames, B_k, N_k, 3+F) chains in request order on that device. results[k] equals, bit for bit,
        sample_chain(**requests[k], keep_frames=keep_frames, seeds=seeds[k], nan_retries=..., require_connected=...,
        require_valid=..., start_step=start_step): always
        on the SIMT edge path, and on the tensor-core path while no node tile rescales its fp16 operands (DESIGN.md
        section 6). It needs per-molecule streams: `seeds`, one list of B_k seeds per request, or noise_mode='per_molecule',
        which draws them with one draw_seeds(B_k) per request in request order -- the results and the generator's final
        offset are then those of the sequence of sample_chain calls.
        Launches (distributed.plan_launches): whole requests, at most `max_molecules` molecules each unless one request is
        larger, padded to the largest N_k in the launch. Requests share a launch only when sample_chain would give them the
        same step coefficients (torch's CPU kernels round them differently for some batch sizes) -- with a `start_step`, one
        for the whole call, also the same start_scalars, which depend on the batch size the same way -- and, with
        aggregation_method='mean' on FC graphs, where the reference divides by the padded N, only with requests of the same
        N. With `devices` set, whole launches are dealt to the listed devices by their cost (distributed.deal_launches), and
        each device runs its launches in order, from a host thread of its own; a launch is never split.
        `nan_retries`, `require_connected`, `require_valid` and `require_clash_free` run their rounds inside each launch, over its rows. Rows still diverging after
        the last round raise once, after every launch: the FoundNaNException of the first such request, its index sets
        local to that request, with `request` = k and `results` = every request's chain (and `chain` = its own when rounds
        ran, as in sample_chain). `last_seeds_many`, `last_attempts_many`, `last_connected_many`, `last_valid_many` and
        `last_clash_free_many` hold per
        request what last_seeds, last_attempts, last_connected and last_valid would hold after its own call; `last_loop_ms_many` holds (device,
        requests, loop ms) per launch. The single-call attributes are left as they were.
        `require_novel` likewise, against `known_linkers`; `last_novel_many` holds every request's verdict.
        `require_ring_sizes` likewise, against `allowed_ring_sizes`; `last_ring_sizes_ok_many` and `last_ring_sizes_many`
        hold every request's verdicts and masks.
        `require_anchors` likewise; each request then also holds `anchors`, its (B_k, N_k) or (B_k, N_k, 1) anchor flags (a
        request may hold them without the check, which ignores them), and `last_anchors_ok_many` holds every request's
        verdicts.
        `fixed_atoms` likewise: a request may hold its (B_k, N_k) or (B_k, N_k, 1) flags of the linker rows to keep, as
        sample_chain's `fixed_atoms`. They travel per row, and requests then share a launch only where sample_chain would
        give them the same fixed_atom_scalars.
        `linker_types` likewise: a request may hold its (F,) or (B_k, F) bool set of allowed types, as sample_chain's
        `linker_types`; a request without one takes `edm.linker_types`. The masks travel per row, so requests with
        different sets share a launch; a request whose set allows every type runs the plain update, as its own
        sample_chain call does, and shares launches only with other such requests.
        `linker_sizes`, one LinkerSizes per request, all of one size table, redraws sizes in those rounds as in sample_chain
        (it needs `seeds`); `last_sizes_many` holds every request's sizes. Each request's sizes come from its own seeds, so
        packing does not change them.
        `start_step` may also be a list with one entry per request, each an int or one step per molecule of that request:
        results[k] then equals sample_chain with that request's steps (their scalars at its own B_k), and requests of
        different steps share launches, since the steps travel per row.
        `resamplings` as in sample_chain, for every request; requests then also share a launch only where sample_chain
        would give them the same jump coefficients (jump_coefficients, which depend on the batch size as the table does).
        `clash_guidance` as in sample_chain, for every request; it is part of every launch's key, and it draws nothing, so
        packing does not change a request's rows. `solver` as in sample_chain, for every request: its table does not
        depend on the batch size, so it adds nothing to the key.
        Raises ValueError for an empty list, the batch stream (its draws depend on B and N), noise= or a replaced draw
        function, host inputs, requests on different devices or of different feature or context widths, and seeds that do
        not match the requests. It takes no `require_unique`, and raises ValueError when the attribute is set: a launch packs
        several requests, whose rows one verdict would compare with each other."""
        if keep_frames is None:
            keep_frames = self.T
        else:
            assert keep_frames <= self.T
        requests = list(requests)
        if not requests:
            raise ValueError("sample_many needs at least one request")
        if self.require_unique is not False:
            raise ValueError("sample_many does not take require_unique: a launch packs several requests, so their rows would "
                             "be compared with each other; call sample_chain per request, or deduplicate with "
                             "molecule_builder.graph_hashes")
        per_request = isinstance(start_step, (list, tuple))
        if per_request and len(start_step) != len(requests):
            raise ValueError(f"start_step holds {len(start_step)} entries for {len(requests)} requests")
        if not per_request:
            self._start(start_step, 1)      # validates it before anything else is checked
        r_passes = self._resamplings(resamplings)
        guide = self._clash_guidance(clash_guidance, start_step)
        ode = self._solver(solver)
        for k, r in enumerate(requests):
            if 'noise' in r or 'batch_slice' in r:
                raise ValueError(f"request {k} passes noise= or batch_slice=: sample_many samples per-molecule streams, "
                                 "which need neither")
            if set(r) - {'anchors', 'fixed_atoms', 'linker_types'} != set(self._REQUEST_INPUTS):
                raise ValueError(f"request {k} must hold exactly the inputs {self._REQUEST_INPUTS}, and may hold "
                                 f"'anchors', 'fixed_atoms' and 'linker_types' (got {sorted(r)})")
        if self._draws_replaced():
            raise ValueError("sample_many needs the device-side per-molecule stream, but this model's draw function is replaced")
        if seeds is None and self.noise_mode != 'per_molecule':
            raise ValueError("sample_many needs per-molecule streams: pass seeds= or set noise_mode='per_molecule' (the batch "
                             f"stream, noise_mode={self.noise_mode!r}, draws depending on B and N, so packing would change them)")
        if seeds is not None and len(seeds) != len(requests):
            raise ValueError(f"seeds holds {len(seeds)} lists for {len(requests)} requests")
        x0 = requests[0]['x']
        ctx_nf = self.dynamics.context_node_nf
        for k, r in enumerate(requests):
            x, h, ctx = r['x'], r['h'], r['context']
            if x.device != x0.device:
                raise ValueError(f"requests 0 and {k} are on different devices ({x0.device}, {x.device})")
            if x.dim() != 3 or x.shape[0] < 1 or x.shape[2] != self.n_dims or h.shape[:2] != x.shape[:2]:
                raise ValueError(f"request {k}: x must be (B, N, {self.n_dims}) with B >= 1 and h (B, N, F) "
                                 f"(got {tuple(x.shape)} and {tuple(h.shape)})")
            if h.shape[-1] != self.in_node_nf or h.shape[-1] != requests[0]['h'].shape[-1]:
                raise ValueError(f"request {k} has {h.shape[-1]} atom features; the model and request 0 have "
                                 f"{self.in_node_nf} and {requests[0]['h'].shape[-1]}")
            if (ctx is None) != (requests[0]['context'] is None) or (ctx is not None and ctx.shape[-1] != ctx_nf):
                raise ValueError(f"request {k}'s context is {None if ctx is None else ctx.shape[-1]} wide; the model takes "
                                 f"{ctx_nf} columns and every request must give them")
        sizes = [r['x'].shape[0] for r in requests]
        nodes = [r['x'].shape[1] for r in requests]
        if per_request:                     # validates every request's steps before anything else is checked
            for k, (s, b) in enumerate(zip(start_step, sizes)):
                if s is None:
                    raise ValueError(f"start_step[{k}] is None: a start_step list holds an int or one step per molecule "
                                     "for every request")
                self._start(s, b)
        if seeds is not None:
            cpu_seeds = []
            for k, (s, b) in enumerate(zip(seeds, sizes)):
                try:
                    cpu_seeds.append(seeds_tensor(s, b))
                except ValueError as e:
                    raise ValueError(f"request {k}: {e}") from None
        dev = x0.device
        if dev.type != 'cuda':
            raise ValueError(f"sample_many needs CUDA inputs (got {dev})")
        retries = self._nan_retries(nan_retries, seeds, None, None, x0)
        check = self._checks(require_connected, require_valid, seeds, None, None, x0, require_clash_free,
                             require_novel=require_novel, require_ring_sizes=require_ring_sizes,
                             require_anchors=require_anchors)
        anchors_many = [self._anchors(check, r.get('anchors'), r['x'], r['node_mask'], r['linker_mask'], r['context'],
                                      f"request {k}'s anchors") for k, r in enumerate(requests)]
        fixed_many = [self._fixed_atoms(r.get('fixed_atoms'), r['x'], r['h'], r['node_mask'], r['fragment_mask'],
                                        r['linker_mask'], r['context'], f"request {k}'s fixed_atoms")
                      for k, r in enumerate(requests)]
        any_fixed = any(f is not None for f in fixed_many)
        if any_fixed and linker_sizes is not None:
            raise ValueError("fixed_atoms does not take linker_sizes: a size redraw rebuilds the linker rows at new sizes")
        types_many = [self._linker_types(r.get('linker_types', self.linker_types), r['x'].shape[0], fixed_many[k], r['h'],
                                         f"request {k}'s linker_types") for k, r in enumerate(requests)]
        any_types = any(m is not None for m in types_many)
        sets = self._hash_sets(check, None, dev)
        recover = retries > 0 or check != 0
        redraws = None
        if linker_sizes is not None:
            if len(linker_sizes) != len(requests):
                raise ValueError(f"linker_sizes holds {len(linker_sizes)} entries for {len(requests)} requests")
            redraws = [self._linker_sizes(ls, seeds, None, None, start_step, r['x'], r['linker_mask'])
                       for ls, r in zip(linker_sizes, requests)]
            if any(not torch.equal(rd[1], redraws[0][1]) for rd in redraws):
                raise ValueError("linker_sizes: every request must draw from the same size table")
        self.dynamics._check_graph_type()
        if seeds is None:
            with torch.cuda.device(dev):    # one draw per request, in request order, as the sample_chain calls draw them
                cpu_seeds = list(torch.cat([draw_seeds(b, dev) for b in sizes]).cpu().split(sizes))
        coefs, starts, keys = self._launch_keys(sizes, nodes, keep_frames, start_step)
        if r_passes > 1:                    # the jump coefficients depend on the batch size as the table does
            keys = [k + (bytes(self.jump_coefficients(b)),) for k, b in zip(keys, sizes)]
        if guide is not None:               # the same for every request of a call: launches are sampled as it says
            keys = [k + (guide[:2],) for k in keys]
        if any_fixed or any_types:          # the kept rows' scalars depend on the batch size as the table does
            keys = [k + (bytes(self.fixed_atom_scalars(b)),) for k, b in zip(keys, sizes)]
        if any_types:                       # a request without a set runs the plain instantiation, as its own call does
            keys = [k + (m is not None,) for k, m in zip(keys, types_many)]
        fc = self.dynamics.graph_type == 'FC'
        launches = plan_launches(sizes, nodes, max_molecules, keys)
        if fc:                              # edges of the launch's padded molecules
            costs = [sum(sizes[k] for k in ks) * n * n for ks, n in launches]
        else:                               # live atoms, a proxy for the cut-off graph's edges
            live = torch.stack([r['node_mask'].reshape(b, n).ne(0).sum() for r, b, n in zip(requests, sizes, nodes)]).tolist()
            costs = [sum(live[k] for k in ks) for ks, _ in launches]
        devices = [self.dynamics._device_index(x0)] if self.devices is None else self.devices
        slots = [(d, replica) for d, replica, _, _ in device_slices(len(devices), devices)]
        slot_of = deal_launches(costs, len(slots))
        busy = sorted(set(slot_of))
        engine_of = dict(zip(busy, self.dynamics.engines([slots[s] for s in busy])))
        lib = _native.load_library()
        finishes, by_device, loop_ms = [], {}, [None] * len(launches)

        def timed(i, call, eng, dev_i, stream):
            call()
            stream.synchronize()            # the loop's events are read before the engine's next launch records them again
            with torch.cuda.device(dev_i):
                loop_ms[i] = float(lib.dl_last_elapsed_ms(eng))
        for i, (ks, n) in enumerate(launches):
            dev_i, replica = slots[slot_of[i]]
            b = sum(sizes[k] for k in ks)
            full = self._sampler_tensors(**pack_requests([{name: requests[k][name] for name in self._REQUEST_INPUTS}
                                                          for k in ks], n, fc))
            anchors = None
            if check & _native.CHECK_ANCHORS:
                anchors = torch.cat([torch.nn.functional.pad(anchors_many[k], (0, n - nodes[k])) for k in ks])
            fixed = None
            if any(fixed_many[k] is not None for k in ks):
                fixed = self._fixed(torch.cat([torch.nn.functional.pad(
                    fixed_many[k] if fixed_many[k] is not None else torch.zeros((sizes[k], nodes[k]), dtype=torch.int8,
                                                                                device=dev), (0, n - nodes[k]))
                    for k in ks]), sizes[ks[0]])
            types = None                    # the launch key keeps requests with and without a set apart
            if types_many[ks[0]] is not None:
                types = self._types(torch.cat([types_many[k] for k in ks]), sizes[ks[0]])
            dev_seeds = torch.cat([cpu_seeds[k] for k in ks]).to(dev)
            where = torch.device('cuda', dev_i)
            eng = engine_of[slot_of[i]]
            redraw = None
            if redraws is not None:
                redraw = tuple(redraws[ks[0]][1] if j == 1 else torch.cat([redraws[k][j] for k in ks]) for j in range(5))
            start = StartSteps.cat([starts[k] for k in ks]) if per_request else starts[sizes[ks[0]]]
            [(_, call)], finish = self._enqueue_batch(lib, full, keep_frames, coefs[sizes[ks[0]]], [(dev_i, replica, 0, b)], [eng],
                                                      [where], dev, dev_seeds=dev_seeds, retries=retries, check=check,
                                                      start=start, redraw=redraw, sets=sets,
                                                      resample=self._resample(r_passes, sizes[ks[0]]), anchors=anchors,
                                                      guide=guide, solver=ode, fixed=fixed, types=types)
            finishes.append(finish)
            by_device.setdefault(dev_i, []).append(
                functools.partial(timed, i, call, eng, dev_i, torch.cuda.current_stream(where)))
        try:
            _run_per_device(by_device)
        except BaseException:
            for dev_i in by_device:         # let the loops that were enqueued finish before their inputs are released
                try:
                    torch.cuda.synchronize(dev_i)
                except Exception:
                    pass
            raise
        results, flags = [None] * len(requests), [None] * len(requests)
        seeds_many, attempts_many = list(cpu_seeds), [None] * len(requests)
        connected_many, valid_many, clash_free_many = [None] * len(requests), [None] * len(requests), [None] * len(requests)
        novel_many = [None] * len(requests)
        rings_ok_many, rings_many = [None] * len(requests), [None] * len(requests)
        anchors_ok_many = [None] * len(requests)
        sizes_many = [None] * len(requests) if redraws is None else [rd[4].cpu() for rd in redraws]
        for (ks, _), finish in zip(launches, finishes):
            out = finish()
            rows = [sizes[k] for k in ks]
            parts = {'chain': unpack_rows(out['chain'], rows, [nodes[k] for k in ks], dim=1),
                     'flags': unpack_rows(out['flags'].cpu(), rows, None)}
            if recover:
                parts['used'] = unpack_rows(out['used'].cpu(), rows, None)
                parts['attempts'] = unpack_rows(out['attempts'].cpu(), rows, None)
            if check:
                parts['passed'] = unpack_rows(out['passed'].cpu(), rows, None)
            if out['sizes'] is not None:
                parts['sizes'] = unpack_rows(out['sizes'].cpu(), rows, None)
            if check & _native.CHECK_RINGS:
                parts['ring_sizes'] = unpack_rows(out['ring_sizes'].cpu(), rows, None)
            for j, k in enumerate(ks):
                results[k], flags[k] = parts['chain'][j], parts['flags'][j]
                if recover:
                    seeds_many[k], attempts_many[k] = parts['used'][j], parts['attempts'][j]
                if 'sizes' in parts:
                    sizes_many[k] = parts['sizes'][j]
                if check & _native.CHECK_CONNECTED:
                    connected_many[k] = (parts['passed'][j] & _native.CHECK_CONNECTED) != 0
                if check & _native.CHECK_VALENCE:
                    valid_many[k] = (parts['passed'][j] & _native.CHECK_VALENCE) != 0
                if check & _native.CHECK_CLASH:
                    clash_free_many[k] = (parts['passed'][j] & _native.CHECK_CLASH) != 0
                if check & _native.CHECK_NOVEL:
                    novel_many[k] = (parts['passed'][j] & _native.CHECK_NOVEL) != 0
                if check & _native.CHECK_RINGS:
                    rings_ok_many[k] = (parts['passed'][j] & _native.CHECK_RINGS) != 0
                    rings_many[k] = parts['ring_sizes'][j]
                if check & _native.CHECK_ANCHORS:
                    anchors_ok_many[k] = (parts['passed'][j] & _native.CHECK_ANCHORS) != 0
        self.last_seeds_many, self.last_attempts_many, self.last_connected_many = seeds_many, attempts_many, connected_many
        self.last_valid_many, self.last_clash_free_many, self.last_sizes_many = valid_many, clash_free_many, sizes_many
        self.last_novel_many = novel_many
        self.last_ring_sizes_ok_many, self.last_ring_sizes_many = rings_ok_many, rings_many
        self.last_anchors_ok_many = anchors_ok_many
        self.last_loop_ms_many = [(slots[slot_of[i]][0], sorted(ks), loop_ms[i]) for i, (ks, _) in enumerate(launches)]
        for k, f in enumerate(flags):
            if f.any():
                exc = self._nan_exception(f, starts[k] if per_request else starts[sizes[k]])
                exc.request, exc.results = k, results
                if recover:
                    exc.chain = results[k]
                raise exc
        return results

    def _launch_keys(self, sizes, nodes, keep_frames, start_step):
        """({B: step coefficients}, {B: _start}, the plan_launches key of every request) of sample_many's requests of sizes
        B_k and N_k: requests share a launch only where sample_chain would give them the same coefficient table and start
        scalars and, with mean aggregation on FC graphs, the same N. With a list `start_step`, one entry per request (an int
        or one step per molecule), the starts are every request's StartSteps at its own B_k, which travel per row: the key
        is then the coefficient table (and N) alone, so requests of different steps share launches."""
        coefs = {b: self.step_coefficients(keep_frames, b) for b in sorted(set(sizes))}
        same_n = self.dynamics.graph_type == 'FC' and self.dynamics.aggregation_method == 'mean'
        if isinstance(start_step, (list, tuple)):
            starts = [self._start(s, b) for s, b in zip(start_step, sizes)]
            starts = [s if isinstance(s, StartSteps) else StartSteps(*([v] * b for v in s)) for s, b in zip(starts, sizes)]
            keys = [(bytes(coefs[b]), None, n if same_n else None) for b, n in zip(sizes, nodes)]
            return coefs, starts, keys
        starts = {b: self._start(start_step, b) for b in sorted(set(sizes))}
        keys = [(bytes(coefs[b]), starts[b], n if same_n else None) for b, n in zip(sizes, nodes)]
        return coefs, starts, keys

    def _enqueue_batch(self, lib, full, keep_frames, coef, slices, engines, places, dev, noise=None, dev_seeds=None, rng=None,
                       retries=0, check=0, start=None, redraw=None, sets=None, resample=None, anchors=None, guide=None,
                       solver=None, fixed=None, types=None):
        """The reverse loops of one batch, the single-launch path under sample_chain and sample_many: `full` (the prepared
        inputs of B molecules on `dev`, _sampler_tensors) sampled with the step coefficients `coef` in `slices` [(device,
        replica, lo, hi)], slice i on engines[i] with its inputs on places[i] -- the caller's tensors themselves when one slice
        covers the batch where it is. The draws are the per-molecule `dev_seeds`, the batch stream `rng` = (seed, offset,
        b0, B_full) or the `noise` tensor; `retries` and `check` as returned by _nan_retries and _checks; `start` as
        returned by _start; `redraw` as returned by _linker_sizes (its rounds then redraw sizes, into `sizes`); `sets` as
        returned by _hash_sets, copied to each slice's device; `resample` as returned by _resample; `anchors` as returned
        by _anchors, each slice's rows on its device; `guide` as returned by _clash_guidance; `solver` as returned by
        _solver; `fixed` as returned by _fixed, each slice's rows of the flags on its device; `types` as returned by _types,
        each slice's rows of the masks.
        Allocates and copies on the calling thread and returns ([(device, call)], finish): each call runs one slice's loop
        (from a host thread of its device, in order per device), and finish(), after every call, copies the slices' rows
        back and returns dict(chain, flags, used, attempts, passed, sizes, bad, consumed) on `dev`; `passed` holds
        every row's _native.CHECK_* verdict bits. `bad` reads the flags: one
        synchronisation, after every loop and copy."""
        n_samples, n_nodes = full['x'].shape[:2]
        d = self.n_dims + self.in_node_nf
        recover = retries > 0 or check != 0
        norm = self._norm()
        chain = torch.empty((keep_frames, n_samples, n_nodes, d), device=dev, dtype=torch.float32)
        flags = torch.zeros(n_samples, dtype=torch.int32, device=dev)
        # recovery: the seed that produced every row and its attempt
        used, attempts = ((torch.empty(n_samples, dtype=torch.int64, device=dev), torch.empty(n_samples, dtype=torch.int32, device=dev))
                          if recover else (None, None))
        # molecule checks: every row's verdict bits, and the tables they read on each slice's device
        passed = torch.empty(n_samples, dtype=torch.int32, device=dev) if check else None
        # CHECK_NOVEL: the linker hash the check decided every returned row's bit on
        novel = bool(check & _native.CHECK_NOVEL)
        linker_hashes = torch.empty(n_samples, dtype=torch.int64, device=dev) if novel else None
        # CHECK_RINGS: the allowed sizes, and the ring-size mask the check decided every returned row's bit on
        rings = bool(check & _native.CHECK_RINGS)
        allowed = ring_size_mask(self.allowed_ring_sizes) if rings else 0
        ring_sizes = torch.empty(n_samples, dtype=torch.int64, device=dev) if rings else None
        # size redraws: every row's size, the attempt-0 sizes on entry
        redraw = redraw if recover else None
        sizes = None if redraw is None else redraw[4].clone()
        tables = self._check_tables(check) if check else None
        clash = clash_table(self.is_geom) if check & _native.CHECK_CLASH else None
        whole = places == [dev]             # one slice, the whole batch where it is: it samples the caller's tensors
        results, calls, parts = [], [], []  # (status, consumed) of every slice; every slice's call; every slice's tensors

        def call(*args):
            results.append(_sample_slice(lib, *args))
        for (dev_i, _, lo, hi), eng, where in zip(slices, engines, places):
            if whole:
                part = (full, noise, dev_seeds, chain, flags, used, attempts, passed)
            else:
                to = lambda v: None if v is None else v.to(where).contiguous()
                with torch.cuda.device(where):
                    part = ({k: to(v) for k, v in slice_sampler_inputs(full, lo, hi).items()},
                            to(None if noise is None else noise[:, lo:hi]), to(None if dev_seeds is None else dev_seeds[lo:hi]),
                            torch.empty((keep_frames, hi - lo, n_nodes, d), device=where, dtype=torch.float32),
                            torch.zeros(hi - lo, dtype=torch.int32, device=where),
                            *((torch.empty(hi - lo, dtype=torch.int64, device=where),
                               torch.empty(hi - lo, dtype=torch.int32, device=where)) if recover else (None, None)),
                            torch.empty(hi - lo, dtype=torch.int32, device=where) if check else None)
            redraw_i = None
            if redraw is not None:
                logits, table, n_frag, linker_x, _ = redraw
                redraw_i = ((logits, table, n_frag, linker_x, sizes) if whole else
                            tuple(v.to(where).contiguous() for v in (logits[lo:hi], table, n_frag[lo:hi], linker_x[lo:hi],
                                                                     sizes[lo:hi])))
            checks_i = None if tables is None else ([t.to(where) for t in tables], None if clash is None else clash.to(where))
            sets_i = None if sets is None else tuple(None if s is None else s.to(where) for s in sets)
            lh_i = linker_hashes if whole or not novel else torch.empty(hi - lo, dtype=torch.int64, device=where)
            rs_i = ring_sizes if whole or not rings else torch.empty(hi - lo, dtype=torch.int64, device=where)
            an_i = anchors if whole or anchors is None else anchors[lo:hi].to(where).contiguous()
            fx_i = None if fixed is None else (fixed[0] if whole else fixed[0][lo:hi].to(where).contiguous())
            part = part + (checks_i, redraw_i, sets_i, lh_i, rs_i, an_i, fx_i)
            parts.append(part)              # alive until the flags have been read below
            t, nz, sd, chain_i, flags_i, used_i, attempts_i, passed_i, checks_i, redraw_i, sets_i, lh_i, rs_i, an_i, fx_i = part
            stream = torch.cuda.current_stream(where).cuda_stream if where.type == 'cuda' else None
            rng_i = None if rng is None else (rng[0], rng[1], rng[2] + lo, rng[3])
            calls.append((dev_i, functools.partial(
                call, eng, self._head(hi - lo, n_nodes, keep_frames, t), (coef, norm, chain_i.data_ptr(), flags_i.data_ptr()),
                stream, nz, sd, rng_i,
                (retries, used_i, attempts_i, check, checks_i, passed_i, redraw_i, sets_i, lh_i,
                 (allowed, rs_i) if rings else None, an_i) if recover else None,
                start.rows(lo, hi) if isinstance(start, StartSteps) else start, resample, guide, solver,
                None if fixed is None else (fx_i, self.T, fixed[1]),
                None if types is None else (types[0][lo:hi].contiguous(), types[1], self.T, types[2]))))

        def finish():
            if not whole:
                place_rows(chain, [p[3] for p in parts], slices, dim=1)
                place_rows(flags, [p[4] for p in parts], slices)
                if recover:
                    place_rows(used, [p[5] for p in parts], slices)
                    place_rows(attempts, [p[6] for p in parts], slices)
                if check:
                    place_rows(passed, [p[7] for p in parts], slices)
                if redraw is not None:
                    place_rows(sizes, [p[9][4] for p in parts], slices)
                if novel:
                    place_rows(linker_hashes, [p[11] for p in parts], slices)
                if rings:
                    place_rows(ring_sizes, [p[12] for p in parts], slices)
            # the host sampler reports NaNs in its status; on the device, one sync per chain instead of one per step
            # (egnn.py:441), after every slice's loop and copy
            bad = _native.DL_NAN_DETECTED in [st for st, _ in results] or bool(flags.any().item())
            return dict(chain=chain, flags=flags, used=used, attempts=attempts, passed=passed, sizes=sizes,
                        linker_hashes=linker_hashes, ring_sizes=ring_sizes, bad=bad, consumed=[c for _, c in results])
        return calls, finish


class InpaintingEDM(EDM):
    """Full-molecule variant (reference: src/edm.py:466-730, sampling half): every atom is denoised by the network
    (`linker_mask=None`, dynamics built with centering=True), fragment atoms are then re-noised from the known
    fragments with q(z_s | z_t, x), and the centre of mass is projected out every step.
    NB the reference's positional order differs from EDM.sample_chain (edge_mask comes third): call by keyword."""
    _SAMPLER = _native.SAMPLER_INPAINT

    @staticmethod
    def _com_free(x, mask):
        """utils.sample_center_gravity_zero_gaussian_with_mask (utils.py:158-168) applied to a raw draw."""
        xm = x * mask
        return xm - (xm.sum(dim=-2, keepdim=True) / mask.sum(dim=-2, keepdim=True)) * mask

    def draw_noise_inpaint(self, n_samples, n_nodes, device, node_mask, fragment_mask, generator=None, resamplings=1):
        """(2T+3, B, N, 3+F): the reference's draws in call order, already masked and COM-projected:
        init (all atoms); per step: p(z_s|z_t) on all atoms then q(z_s|z_t,x) on fragment atoms; final p and q draws.
        With r = `resamplings` passes per step, each pass draws the pair and, but on the last, the re-noise draw on all
        atoms: (1 + T(3r-1) + 2, B, N, 3+F)."""
        T, nd, nf = self.T, self.n_dims, self.in_node_nf
        step = [node_mask, fragment_mask, node_mask] * (resamplings - 1) + [node_mask, fragment_mask]
        masks = [node_mask] + step * T + [node_mask, node_mask]
        out = torch.empty((len(masks), n_samples, n_nodes, nd + nf), device=device, dtype=torch.float32)
        for r, m in enumerate(masks):
            m = m.to(device=device, dtype=torch.float32)
            out[r, :, :, :nd] = self._com_free(torch.randn((n_samples, n_nodes, nd), device=device, generator=generator), m)
            out[r, :, :, nd:] = torch.randn((n_samples, n_nodes, nf), device=device, generator=generator) * m
        return out

    def _q_coefficients(self, g_s, sigma_s, sigma_t, sigma2_ts, alpha_ts):
        """q(z_s | z_t, x), which re-noises the fragment atoms from the known fragments (edm.py:661-664)."""
        qa = float((alpha_ts * (sigma_s ** 2) / (sigma_t ** 2))[0])
        qb = float((self.alpha(g_s) * sigma2_ts / (sigma_t ** 2))[0])
        return qa, qb

    def _final_qa(self, g0):
        return float((self.sigma(g0) / self.alpha(g0))[0])                         # edm.py:716

    def _n_draws(self, resamplings=1):
        return 1 + self.T * (3 * resamplings - 1) + 2

    def _draw_tensor(self, n_samples, n_nodes, device, node_mask, fragment_mask, resamplings=1):
        if resamplings == 1:                # the plain loop: the draw function as it is called without resampling
            return self.draw_noise_inpaint(n_samples, n_nodes, device, node_mask, fragment_mask)
        return self.draw_noise_inpaint(n_samples, n_nodes, device, node_mask, fragment_mask, resamplings=resamplings)

    def _draws_replaced(self):
        """draw_noise_inpaint replaced on the instance, in a subclass or on the class supplies the draws."""
        return 'draw_noise_inpaint' in self.__dict__ or type(self).draw_noise_inpaint is not _DRAW_NOISE_INPAINT

    def _start(self, start_step, n_samples):
        """Partial diffusion noises the linker from the data with EDM.forward's q(z_t | x); this class noises the whole
        molecule without a centre of mass, which has no such start."""
        if start_step is not None:
            raise ValueError("InpaintingEDM does not take start_step: partial diffusion starts the linker sampler (EDM) only")
        return None

    def sample_chain(self, x, h, node_mask, edge_mask, fragment_mask, linker_mask, context, keep_frames=None,
                     noise=None, batch_slice=None, seeds=None, nan_retries=None, require_connected=None, start_step=None,
                     require_valid=None, require_clash_free=None, linker_sizes=None, require_unique=None,
                     require_novel=None, exclude_hashes=None, resamplings=None, require_ring_sizes=None,
                     require_anchors=None, anchors=None, clash_guidance=None, solver=None, fixed_atoms=None,
                     linker_types=None):
        """EDM.sample_chain in the reference's positional order for this class (edge_mask third). `noise` optionally
        injects the (2T+3,B,N,3+F) prepared draws of `draw_noise_inpaint` (tests). Without it, on CUDA and with noise_mode
        'reference_stream', the draws are made inside the kernels from the default generator's state
        (dl_sample_chain_rng), unless `draw_noise_inpaint` is replaced -- on the instance, in a subclass or on the class --
        in which case the replacement draws them. `batch_slice=(b0, B_full)` and `seeds` as in EDM.sample_chain: with
        seeds, molecule b's 2T+3 raw draws are those of the molecule sampled alone after torch.cuda.manual_seed(seeds[b]),
        masked and projected per molecule as always. `nan_retries`, `require_connected`, `require_valid` and `require_unique`
        as in EDM.sample_chain; the checks and the hash cover every atom of the molecule. `require_novel` and
        `exclude_hashes` as there; the linker hash covers the linker_mask rows. `require_ring_sizes` as there: the rings of
        the bonds with an end on the linker_mask rows. `require_anchors` and `anchors` as there: the linker atoms are the
        linker_mask rows, the fragment atoms every other atom. `start_step` raises ValueError unless None, and `require_clash_free`
        unless None or False: this loop re-noises the pocket; `linker_sizes` unless None: this model has no linker size.
        `resamplings` = r (None: the `resamplings` attribute, default 1) runs every reverse step as r RePaint passes
        (Lugmayr et al., 2022; DiffSBDD's inpaint(..., resamplings=r); dl_set_resamplings): pass u denoises as the plain
        step does, with time feature (s+1)/T, and every pass but the last then re-noises z <- alpha_t|s z + sigma_t|s eps
        on every atom (eps COM-free on the node mask, as sample_combined_position_feature_noise draws it; the two scalars
        are jump_coefficients'), so the generated atoms can adapt to the known ones. The frame of step s is written after
        its last pass. The draws are z_T, per step and pass the p and q draws plus the re-noise draw for u < r-1, then the
        two final draws: 1 + T(3r-1) + 2 (noise= holds that many prepared slabs, draw_noise_inpaint(resamplings=r) makes
        them; the batch stream advances by as many draws; per-molecule streams use their draws in that order). r = 1 is
        the plain sampler, bit for bit. A call costs about r times the loop. ValueError for a non-integer, a bool or
        r < 1. `clash_guidance` raises ValueError unless None: this loop re-noises the pocket. `solver` unless None or
        'ancestral': this sampler has no ODE update. `fixed_atoms` unless None: this sampler keeps known atoms its own way.
        `linker_types` unless None: this sampler generates its atoms in its own update."""
        return super().sample_chain(x=x, h=h, node_mask=node_mask, fragment_mask=fragment_mask, linker_mask=linker_mask,
                                    edge_mask=edge_mask, context=context, keep_frames=keep_frames, noise=noise,
                                    batch_slice=batch_slice, seeds=seeds, nan_retries=nan_retries,
                                    require_connected=require_connected, start_step=start_step, require_valid=require_valid,
                                    require_clash_free=require_clash_free, linker_sizes=linker_sizes,
                                    require_unique=require_unique, require_novel=require_novel,
                                    exclude_hashes=exclude_hashes, resamplings=resamplings,
                                    require_ring_sizes=require_ring_sizes, require_anchors=require_anchors,
                                    anchors=anchors, clash_guidance=clash_guidance, solver=solver, fixed_atoms=fixed_atoms,
                                    linker_types=linker_types)


# the draws the device-side stream reproduces; a replaced draw_noise_inpaint takes the tensor path
_DRAW_NOISE_INPAINT = InpaintingEDM.draw_noise_inpaint
