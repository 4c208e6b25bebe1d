"""ctypes binding of libdifflinker_b200.so (include/difflinker_b200.h). No CPU fallback: if the library or an
H100 is missing, calls fail loudly."""
import ctypes as C
import os

from .build import LIB_PATH, build_native, is_stale, nvcc_path

DL_OK, DL_NAN_DETECTED = 0, 1
GRAPH_TYPES = {"FC": 0, "4A": 1, "FC-4A": 2, "FC-10A-4A": 3}
EDGE_IMPLS = {"auto": 0, "simt": 1, "wgmma": 2}
SAMPLER_LINKER, SAMPLER_INPAINT = 0, 1
SOLVERS = {"ancestral": 0, "ddim": 1, "dpmpp_2m": 2}   # DL_SOLVER_*
AGGREGATIONS = {"sum": 0, "mean": 1}
CHECK_CONNECTED, CHECK_VALENCE, CHECK_CLASH, CHECK_UNIQUE, CHECK_NOVEL, CHECK_RINGS = 1, 2, 4, 8, 16, 32   # DL_CHECK_*
CHECK_ANCHORS = 64
COORDS_RANGE = 15.0   # EGNN hands its own coords_range=15 to every EquivariantBlock (src/egnn.py:183,209)


class DLConfig(C.Structure):
    _fields_ = [("n_dims", C.c_int32), ("in_node_nf", C.c_int32), ("context_node_nf", C.c_int32),
                ("hidden_nf", C.c_int32), ("n_layers", C.c_int32), ("inv_sublayers", C.c_int32),
                ("condition_time", C.c_int32), ("centering", C.c_int32), ("graph_type", C.c_int32),
                ("device", C.c_int32), ("edge_impl", C.c_int32), ("norm_constant", C.c_float),
                ("normalization_factor", C.c_float)]


class DLEgnnOptions(C.Structure):
    _fields_ = [("tanh", C.c_int32), ("coords_range", C.c_float), ("sin_embedding", C.c_int32),
                ("aggregation", C.c_int32)]

    def is_default(self):
        return bytes(self) == bytes(DLEgnnOptions(0, COORDS_RANGE, 0, AGGREGATIONS["sum"]))


class DLSizeGNNConfig(C.Structure):
    _fields_ = [("in_node_nf", C.c_int32), ("hidden_nf", C.c_int32), ("out_node_nf", C.c_int32),
                ("n_layers", C.c_int32), ("device", C.c_int32)]


class DLMoleculeChecks(C.Structure):
    _fields_ = [("require", C.c_int32), ("n_types", C.c_int32), ("thr1", C.c_void_p), ("thr2", C.c_void_p),
                ("thr3", C.c_void_p), ("max_valence", C.c_void_p), ("clash", C.c_void_p)]

    @classmethod
    def of(cls, require, tables, clash=None):
        """The struct over `tables` = [thr1], [thr1, thr2, thr3] or [thr1, thr2, thr3, max_valence] and the (T,T) `clash`
        table (None: none), device tensors the caller keeps alive."""
        ptrs = [t.data_ptr() for t in tables] + [None] * (4 - len(tables))
        return cls(require, tables[0].shape[0], *ptrs, None if clash is None else clash.data_ptr())


class DLHashSets(C.Structure):
    _fields_ = [("known", C.c_void_p), ("n_known", C.c_int64), ("seen", C.c_void_p), ("n_seen", C.c_int64)]

    @classmethod
    def of(cls, known, seen):
        """The struct over two 1-D int64 device tensors of uint64 bits in ascending unsigned order, or None (an empty set),
        which the caller keeps alive."""
        ptr = lambda t: (None, 0) if t is None else (t.data_ptr(), t.numel())
        return cls(*ptr(known), *ptr(seen))


class DLSizeRedraw(C.Structure):
    _fields_ = [("C", C.c_int32), ("logits_row_stride", C.c_int32), ("logits", C.c_void_p), ("sizes", C.c_void_p),
                ("n_frag", C.c_void_p), ("linker_x", C.c_void_p)]


class DLStepCoef(C.Structure):
    _fields_ = [("t", C.c_float), ("a", C.c_float), ("b", C.c_float), ("c", C.c_float), ("frame", C.c_int32),
                ("qa", C.c_float), ("qb", C.c_float), ("pad", C.c_float)]


# every symbol include/difflinker_b200.h declares: name -> (restype, argtypes)
_P, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
SYMBOLS = {
    "dl_version": (C.c_char_p, []),
    "dl_last_error": (C.c_char_p, []),
    "dl_create": (_I32, [C.POINTER(DLConfig), C.POINTER(_P)]),
    "dl_create_ex": (_I32, [C.POINTER(DLConfig), C.POINTER(DLEgnnOptions), C.POINTER(_P)]),
    "dl_destroy": (_I32, [_P]),
    "dl_set_weight": (_I32, [_P, C.c_char_p, _P, _I64]),
    "dl_finalize_weights": (_I32, [_P]),
    "dl_expected_param_count": (_I64, [_P]),
    "dl_dynamics_forward": (_I32, [_P, _I32, _I32, _P, _I32, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dl_dynamics_forward_host": (_I32, [_P, _I32, _I32, _P, _I32, _P, _P, _P, _P, _P, _P, _P]),
    "dl_sample_chain": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dl_sample_chain_rng": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, C.c_uint64, C.c_uint64, _P, _P, _P, _P,
                                   _P, _P]),
    "dl_sample_chain_seeded": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dl_retry_seed": (C.c_uint64, [C.c_uint64, _I32]),
    "dl_sample_chain_retry": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _P,
                                     _P, C.POINTER(DLMoleculeChecks), _P, C.POINTER(DLSizeRedraw), _P, _P]),
    "dl_sample_chain_retry_sets": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32,
                                          _P, _P, C.POINTER(DLMoleculeChecks), C.POINTER(DLHashSets), _P, _P,
                                          C.POINTER(DLSizeRedraw), _P, _P]),
    "dl_novel_check": (_I32, [_I32, _I32, C.POINTER(DLMoleculeChecks), C.POINTER(DLHashSets), _P, _I32, _P, _P, _P, _I32,
                              _I32, _P, _P, _P, _P]),
    "dl_size_draw": (_I32, [_I32, _I32, _P, _I32, _P, _P, _I32, _P, _P]),
    "dl_size_uniform": (C.c_double, [C.c_uint64]),
    "dl_molecule_check": (_I32, [_I32, _I32, C.POINTER(DLMoleculeChecks), _P, _I32, _P, _P, _I32, _I32, _P, _P, _P]),
    "dl_clash_check": (_I32, [_I32, _I32, _I32, _P, _P, _I32, _P, _P, _P, _I32, _P, _P, _P]),
    "dl_ring_check": (_I32, [_I32, _I32, _I32, _P, _P, _I32, _P, _P, _P, _I32, _I32, C.c_uint64, _P, _P, _P]),
    "dl_set_ring_sizes": (_I32, [_P, C.c_uint64]),
    "dl_last_ring_sizes": (_I32, [_P, _I32, _P, _P]),
    "dl_anchor_check": (_I32, [_I32, _I32, _I32, _P, _P, _I32, _P, _P, _P, _P, _I32, _I32, _P, _P, _P]),
    "dl_set_anchors": (_I32, [_P, _I32, _I32, _P, _P]),
    "dl_molecule_hash": (_I32, [_I32, _I32, C.POINTER(DLMoleculeChecks), _P, _I32, _P, _P, _I32, _I32, _P, _P]),
    "dl_last_retry_ms": (_F, [_P]),
    "dl_set_noise_slice": (_I32, [_P, _I32, _I32]),
    "dl_set_start_step": (_I32, [_P, _I32, _F, _F]),
    "dl_set_start_steps": (_I32, [_P, _I32, _P, _P, _P]),
    "dl_set_resamplings": (_I32, [_P, _I32, _I32, _P]),
    "dl_set_clash_guidance": (_I32, [_P, C.c_float, _I32, _I32, _P]),
    "dl_set_solver": (_I32, [_P, _I32, _I32, _P]),
    "dl_set_fixed_atoms": (_I32, [_P, _I32, _I32, _P, _I32, _P, _P]),
    "dl_set_linker_types": (_I32, [_P, _I32, _I32, _P, _I32, _P]),
    "dl_clash_guide": (_I32, [_I32, _I32, _I32, _P, C.c_float, _P, _I32, _P, _P, _P, _I32, _P]),
    "dl_noise_fill": (_I32, [_P, _I32, _I32, _I32, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "dl_noise_fill_inpaint": (_I32, [_P, _I32, _I32, _I32, _P, _P, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "dl_sample_chain_host": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dl_launch_count": (_I64, [_P]),
    "dl_last_molecule_steps": (_I64, [_P]),
    "dl_last_elapsed_ms": (_F, [_P]),
    "dl_time_edge_kernel": (_F, [_P, _I32]),
    "dl_selftest_tc": (_I32, [_P, C.POINTER(_F), C.POINTER(_F)]),
    "dl_selftest_tc_layout": (_I32, [_P, _I32, C.POINTER(_F), C.POINTER(_F)]),
    "dl_cut_graph_stats": (_I32, [_P, C.POINTER(_I64)]),
    "dl_sizegnn_create": (_I32, [C.POINTER(DLSizeGNNConfig), C.POINTER(_P)]),
    "dl_sizegnn_destroy": (_I32, [_P]),
    "dl_sizegnn_set_weight": (_I32, [_P, C.c_char_p, _P, _I64]),
    "dl_sizegnn_finalize_weights": (_I32, [_P]),
    "dl_sizegnn_forward": (_I32, [_P, _I32, _I32, _P, _P, _P, _P, _P]),
    "dl_restore_frame": (_I32, [_I32, _I32, _I32, _P, _P, _P, _P, _P]),
    "dl_restore_frame2": (_I32, [_I32, _I32, _I32, _I32, _P, _P, _P, _P, _P]),
    "dl_bond_orders": (_I32, [_I32, _I32, _I32, _P, _I32, _P, _P, _P, _P, _P, _P, _P]),
    "dl_format_xyz": (_I64, [_I32, _I32, _I32, _P, _I32, _P, _I32, _P, C.POINTER(C.c_char_p), _I32, _P, _I64, _P]),
}

_lib = None


def load_library():
    """Loads (building first when stale and nvcc is around) the native library. Raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    if is_stale():
        if nvcc_path() is not None:
            build_native()
        elif not os.path.isfile(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing and nvcc is unavailable; build it with `python -m difflinker_b200.build`. "
                "difflinker_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class NativeError(RuntimeError):
    pass


def check(status: int, what: str):
    if status < 0:
        raise NativeError(f"{what} failed with status {status}: {load_library().dl_last_error().decode()}")
    return status
