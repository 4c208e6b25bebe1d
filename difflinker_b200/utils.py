"""Host-side helpers of the sampling path, with the reference's names (src/utils.py)."""
import sys

import torch


class FoundNaNException(Exception):
    """Same attributes as the reference exception (src/utils.py:274-289), built from the per-molecule
    flags the device path reports (bit0: NaN in coordinates/velocity, bit1: NaN in features)."""

    def __init__(self, x=None, h=None, flags=None):
        if flags is not None:
            f = [int(v) for v in flags]
            x_idx = {i for i, v in enumerate(f) if v & 1}
            h_idx = {i for i, v in enumerate(f) if v & 2}
            steps = [v >> 8 for v in f if v >> 8]
            self.first_step = min(steps) - 1 if steps else None
        else:
            x_idx = {i for i in range(x.shape[0]) if bool(torch.isnan(x[i]).any())}
            h_idx = {i for i in range(h.shape[0]) if bool(torch.isnan(h[i]).any())}
            self.first_step = None
        self.x_h_nan_idx = x_idx & h_idx
        self.only_x_nan_idx = x_idx - h_idx
        self.only_h_nan_idx = h_idx - x_idx
        # Exception.__init__ directly (not super()): in the compat subclass below the MRO continues with the reference's
        # class, whose constructor takes (x, h) tensors
        Exception.__init__(self, f"NaN in dynamics output (x&h: {sorted(self.x_h_nan_idx)}, x: {sorted(self.only_x_nan_idx)}, "
                                 f"h: {sorted(self.only_h_nan_idx)})")


_COMPAT_CLASSES = {}


def nan_exception_class():
    """The class the device paths raise. When the reference package is loaded in this process (generate.py, sample.py
    and lightning.py import `src.utils`), it is a subclass of BOTH this module's FoundNaNException and the reference's
    `src.utils.FoundNaNException`, so the callers' existing `except FoundNaNException` retry loops (generate.py:154-159)
    and the skip logic of lightning.py:350-362 keep catching NaNs raised by the native sampler."""
    for modname in ("src.utils", "utils"):
        mod = sys.modules.get(modname)
        ref = getattr(mod, "FoundNaNException", None) if mod is not None else None
        if isinstance(ref, type) and issubclass(ref, Exception) and ref is not FoundNaNException \
                and not issubclass(ref, FoundNaNException) and getattr(ref, "__module__", "").split(".")[0] != "difflinker_b200":
            if ref not in _COMPAT_CLASSES:
                _COMPAT_CLASSES[ref] = type("FoundNaNException", (FoundNaNException, ref), {"__module__": __name__})
            return _COMPAT_CLASSES[ref]
    return FoundNaNException


def sample_gaussian_with_mask(size, device, node_mask):
    """src/utils.py:189-192."""
    return torch.randn(size, device=device) * node_mask


def remove_mean_with_mask(x, node_mask):
    """src/utils.py:56-63 (the .item() assert of the reference is dropped: it is a host sync)."""
    n = node_mask.sum(1, keepdims=True)
    return x - (torch.sum(x, dim=1, keepdim=True) / n) * node_mask


def partial_mean(x, center_of_mass_mask):
    """The (B, 1, 3) centre of mass of the `center_of_mass_mask` atoms that remove_partial_mean_with_mask subtracts."""
    n = center_of_mass_mask.sum(1, keepdims=True)
    return torch.sum(x * center_of_mass_mask, dim=1, keepdim=True) / n


def remove_partial_mean_with_mask(x, node_mask, center_of_mass_mask):
    """src/utils.py:66-74: subtract the centre of mass of the `center_of_mass_mask` atoms from all atoms."""
    return x - partial_mean(x, center_of_mass_mask) * node_mask


def assert_correctly_masked(variable, node_mask):
    """src/utils.py:99-101."""
    assert (variable * (1 - node_mask)).abs().max().item() < 1e-4, "Variables not masked properly."
