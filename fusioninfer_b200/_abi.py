"""ctypes binding of include/fi_epp.h (the C ABI of libfi_epp.so).

This is the same stub a Go EPP would write with cgo (INTEGRATION.md); Python is
used here only because the image has no Go toolchain (SURVEY.md §0 F2).  The
library is loaded from fusioninfer_b200/lib/ (built in-tree by `make` /
`__graft_entry__.build()`); a missing library is a hard error — there is no
Python or CPU fallback for the pick path.
"""
from __future__ import annotations

import ctypes as C
import os

FI_EPP_ABI_VERSION = 2
FI_EPP_MAX_PROFILES = 4
FI_EPP_MAX_SCORERS = 4
FI_EPP_MAX_FILTERS = 4
FI_EPP_MAX_LABELS = 24
FI_ROLE_FIRST_FREE = 8
FI_EPP_MAX_BLOCKS = 4095
FI_EPP_MAX_RANKED = 16
FI_NO_ENDPOINT = 0xFFFFFFFF
FI_EPP_UNIQUE_ID_BYTES = 128

FI_OK = 0
FI_ERR_INVALID = -1
FI_ERR_CUDA = -2
FI_ERR_NOMEM = -3
FI_ERR_CAPACITY = -4
FI_ERR_STATE = -5
FI_ERR_COMM = -6
FI_ERR_CONFIG = -7

FI_MATCH_UPSTREAM = 0
FI_MATCH_LPM = 1

FI_SCORER_PREFIX = 1
FI_SCORER_KV_UTIL = 2
FI_SCORER_QUEUE = 3
FI_SCORER_LORA = 4

FI_ROLE_WORKER = 1
FI_ROLE_PREFILLER = 2
FI_ROLE_DECODER = 4
FI_ENDPOINT_ALIVE = 1

FI_OP_SET = 1
FI_OP_CLEAR = 2


class fi_scorer(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("weight", C.c_int32)]


class fi_profile(C.Structure):
    _fields_ = [
        ("name", C.c_char * 32),
        ("role_mask", C.c_uint32),
        ("n_scorers", C.c_uint32),
        ("scorers", fi_scorer * FI_EPP_MAX_SCORERS),
        ("n_more_filters", C.c_uint32),
        ("more_filters", C.c_uint32 * (FI_EPP_MAX_FILTERS - 1)),
    ]


class fi_label_bit(C.Structure):
    _fields_ = [
        ("label", C.c_char * 64),
        ("value", C.c_char * 56),
        ("bit", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


class fi_epp_config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("abi_version", C.c_uint32),
        ("device", C.c_int32),
        ("block_bytes", C.c_uint32),
        ("max_blocks", C.c_uint32),
        ("lru_capacity", C.c_uint32),
        ("num_endpoints", C.c_uint32),
        ("endpoint_begin", C.c_uint32),
        ("endpoint_count", C.c_uint32),
        ("match_mode", C.c_uint32),
        ("max_batch", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("max_prompt_bytes", C.c_uint64),
        ("index_slots", C.c_uint64),
        ("n_profiles", C.c_uint32),
        ("pd_enabled", C.c_uint32),
        ("pd_decode_profile", C.c_uint32),
        ("pd_prefill_profile", C.c_uint32),
        ("pd_threshold", C.c_double),
        ("profiles", fi_profile * FI_EPP_MAX_PROFILES),
        ("n_labels", C.c_uint32),
        ("reserved1", C.c_uint32),
        ("labels", fi_label_bit * FI_EPP_MAX_LABELS),
    ]


class fi_endpoint_state(C.Structure):
    _fields_ = [
        ("endpoint", C.c_uint32),
        ("role_mask", C.c_uint32),
        ("kv_util", C.c_double),
        ("queue_depth", C.c_int32),
        ("flags", C.c_uint32),
    ]


FI_EPP_MAX_LORA = 8


class fi_endpoint_lora(C.Structure):
    _fields_ = [
        ("endpoint", C.c_uint32),
        ("max_active", C.c_uint32),
        ("n_active", C.c_uint32),
        ("n_waiting", C.c_uint32),
        ("active", C.c_uint64 * FI_EPP_MAX_LORA),
        ("waiting", C.c_uint64 * FI_EPP_MAX_LORA),
    ]


class fi_index_op(C.Structure):
    _fields_ = [("hash", C.c_uint64), ("endpoint", C.c_uint32), ("op", C.c_uint32)]


class fi_pick(C.Structure):
    _fields_ = [
        ("endpoint", C.c_uint32),
        ("match_blocks", C.c_uint16),
        ("n_blocks", C.c_uint16),
        ("score", C.c_double),
    ]


class fi_match_entry(C.Structure):
    _fields_ = [("endpoint", C.c_uint32), ("match_blocks", C.c_uint16), ("reserved", C.c_uint16)]


class fi_index_stats(C.Structure):
    _fields_ = [
        ("slots", C.c_uint64),
        ("used", C.c_uint64),
        ("tombstones", C.c_uint64),
        ("rebuilds", C.c_uint64),
        ("ops_applied", C.c_uint64),
        ("lru_entries", C.c_uint64),
    ]


class fi_epp_snapshot_info(C.Structure):
    _fields_ = [
        ("block_bytes", C.c_uint32),
        ("max_blocks", C.c_uint32),
        ("lru_capacity", C.c_uint32),
        ("num_endpoints", C.c_uint32),
        ("n_nodes", C.c_uint64),
        ("n_lru", C.c_uint64),
        ("pairs", C.c_uint64),
        ("bytes", C.c_uint64),
    ]


class fi_epp_stats(C.Structure):
    _fields_ = [
        ("kernel_launches", C.c_uint64),
        ("pick_calls", C.c_uint64),
        ("requests", C.c_uint64),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("ms_hash_blocks", C.c_double),
        ("ms_chain_probe", C.c_double),
        ("ms_match_pick", C.c_double),
        ("ms_index_apply", C.c_double),
        ("ms_other", C.c_double),
        ("n_hash_blocks", C.c_uint64),
        ("n_chain_probe", C.c_uint64),
        ("n_match_pick", C.c_uint64),
        ("n_index_apply", C.c_uint64),
        ("n_other", C.c_uint64),
        ("probed_blocks", C.c_uint64),
        ("hashed_blocks", C.c_uint64),
    ]


# numpy dtypes with the same layout (structured arrays travel through the ABI without copies)
def np_dtypes():
    import numpy as np

    pick = np.dtype(
        [("endpoint", "<u4"), ("match_blocks", "<u2"), ("n_blocks", "<u2"), ("score", "<f8")], align=True
    )
    op = np.dtype([("hash", "<u8"), ("endpoint", "<u4"), ("op", "<u4")], align=True)
    ep = np.dtype(
        [("endpoint", "<u4"), ("role_mask", "<u4"), ("kv_util", "<f8"), ("queue_depth", "<i4"), ("flags", "<u4")],
        align=True,
    )
    assert pick.itemsize == C.sizeof(fi_pick) == 16
    assert op.itemsize == C.sizeof(fi_index_op) == 16
    assert ep.itemsize == C.sizeof(fi_endpoint_state) == 24
    return pick, op, ep


def match_entry_dtype():
    """one entry of fi_epp_match_lists (fi_match_entry, 8 bytes)"""
    import numpy as np

    dt = np.dtype([("endpoint", "<u4"), ("match_blocks", "<u2"), ("reserved", "<u2")], align=True)
    assert dt.itemsize == C.sizeof(fi_match_entry) == 8
    return dt


def lora_dtype():
    import numpy as np

    dt = np.dtype([("endpoint", "<u4"), ("max_active", "<u4"), ("n_active", "<u4"), ("n_waiting", "<u4"),
                   ("active", "<u8", (FI_EPP_MAX_LORA,)), ("waiting", "<u8", (FI_EPP_MAX_LORA,))], align=True)
    assert dt.itemsize == C.sizeof(fi_endpoint_lora) == 144
    return dt


LIB_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib")
LIB_PATH = os.path.join(LIB_DIR, "libfi_epp.so")

# every symbol include/fi_epp.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("fi_epp_abi_version", C.c_uint32, []),
    ("fi_epp_status_string", C.c_char_p, [C.c_int]),
    ("fi_epp_config_default", C.c_int, [C.POINTER(fi_epp_config)]),
    ("fi_epp_config_from_yaml", C.c_int, [C.c_char_p, C.c_size_t, C.POINTER(fi_epp_config), C.c_char_p, C.c_size_t]),
    ("fi_epp_config_picker_endpoints", C.c_int, [C.c_char_p, C.c_size_t, _P, C.c_char_p, C.c_size_t]),
    ("fi_epp_create", C.c_int, [C.POINTER(fi_epp_config), C.POINTER(_P)]),
    ("fi_epp_destroy", None, [_P]),
    ("fi_epp_last_error", C.c_char_p, [_P]),
    ("fi_epp_model_seed", C.c_int, [_P, C.c_size_t, _P, C.c_size_t, C.POINTER(C.c_uint64)]),
    ("fi_epp_endpoints_update", C.c_int, [_P, _P, C.c_uint32]),
    ("fi_epp_endpoints_lora_update", C.c_int, [_P, _P, C.c_uint32]),
    ("fi_epp_index_apply", C.c_int, [_P, _P, C.c_uint64]),
    ("fi_epp_index_remove_endpoints", C.c_int, [_P, _P, C.c_uint32, _P]),
    ("fi_epp_resize_pool", C.c_int, [_P, C.c_uint32, _P]),
    ("fi_epp_snapshot_save", C.c_int, [_P, _P, C.c_uint64, C.POINTER(C.c_uint64)]),
    ("fi_epp_snapshot_load", C.c_int, [_P, _P, C.c_uint64]),
    ("fi_epp_snapshot_info", C.c_int, [_P, C.c_uint64, C.POINTER(fi_epp_snapshot_info)]),
    ("fi_epp_snapshot_capture", C.c_int, [_P, C.POINTER(_P), C.POINTER(C.c_uint64)]),
    ("fi_epp_snapshot_read", C.c_int, [_P, _P, C.c_uint64]),
    ("fi_epp_snapshot_free", None, [_P]),
    ("fi_epp_set_lru_capacities", C.c_int, [_P, _P, _P, C.c_uint32, _P]),
    ("fi_epp_index_add_chain", C.c_int, [_P, C.c_uint32, _P, C.c_uint32]),
    ("fi_epp_index_add_chains", C.c_int, [_P, _P, _P, C.c_uint32, _P, C.c_uint32]),
    ("fi_epp_index_add_chains_device", C.c_int, [_P, _P, _P, C.c_uint32, _P, C.c_uint32, _P]),
    ("fi_epp_lru_dump", C.c_int, [_P, C.c_uint32, _P, C.c_uint32, _P]),
    ("fi_epp_lru_counters", C.c_int, [_P, _P]),
    ("fi_epp_pipeline_info", C.c_int, [_P, _P]),
    ("fi_epp_set_option", C.c_int, [_P, C.c_char_p, C.c_int64]),
    ("fi_epp_index_sync", C.c_int, [_P]),
    ("fi_epp_index_contains", C.c_int, [_P, _P, C.c_uint64, _P]),
    ("fi_epp_index_stats", C.c_int, [_P, C.POINTER(fi_index_stats)]),
    ("fi_epp_hash_batch", C.c_int, [_P, _P, _P, _P, C.c_uint32, _P, _P]),
    ("fi_epp_pick_batch", C.c_int, [_P, _P, _P, _P, C.c_uint32, _P, _P]),
    ("fi_epp_pick_batch_device", C.c_int, [_P, _P, _P, _P, C.c_uint32, C.c_uint64, _P, _P, _P]),
    ("fi_epp_pick_batch_lora", C.c_int, [_P, _P, _P, _P, _P, C.c_uint32, _P, _P]),
    ("fi_epp_pick_batch_device_lora", C.c_int, [_P, _P, _P, _P, _P, C.c_uint32, C.c_uint64, _P, _P, _P]),
    ("fi_epp_pick_batch_ranked", C.c_int, [_P, _P, _P, _P, _P, C.c_uint32, C.c_uint32, _P, _P]),
    ("fi_epp_pick_batch_device_ranked", C.c_int,
     [_P, _P, _P, _P, _P, C.c_uint32, C.c_uint64, C.c_uint32, _P, _P, _P]),
    ("fi_epp_pick_batch_subset", C.c_int, [_P, _P, _P, _P, _P, _P, C.c_uint32, C.c_uint32, _P, _P]),
    ("fi_epp_pick_batch_device_subset", C.c_int,
     [_P, _P, _P, _P, _P, _P, C.c_uint32, C.c_uint64, C.c_uint32, _P, _P, _P]),
    ("fi_epp_match_counts", C.c_int, [_P, _P, _P, _P, C.c_uint32, _P, _P, _P]),
    ("fi_epp_match_counts_device", C.c_int, [_P, _P, _P, _P, C.c_uint32, C.c_uint64, _P, _P, _P, _P]),
    ("fi_epp_match_lists", C.c_int, [_P, _P, _P, _P, C.c_uint32, _P, _P, C.c_uint64, _P, _P]),
    ("fi_epp_match_lists_device", C.c_int,
     [_P, _P, _P, _P, C.c_uint32, C.c_uint64, _P, _P, C.c_uint64, _P, _P, _P]),
    ("fi_epp_pinned_alloc", _P, [C.c_size_t]),
    ("fi_epp_pinned_free", None, [_P]),
    ("fi_epp_comm_unique_id", C.c_int, [_P]),
    ("fi_epp_pick_submit", C.c_int, [_P, _P, _P, _P, C.c_uint32, C.c_uint64, _P, _P]),
    ("fi_epp_pick_wait", C.c_int, [_P, _P]),
    ("fi_epp_pick_submit_ex", C.c_int,
     [_P, _P, _P, _P, _P, _P, C.c_uint32, C.c_uint64, C.c_uint32, _P, _P, _P, C.POINTER(C.c_uint64)]),
    ("fi_epp_pick_wait_batch", C.c_int, [_P, C.c_uint64, _P]),
    ("fi_epp_index_add_submitted", C.c_int, [_P, C.c_uint64, _P, _P, C.c_uint32]),
    ("fi_epp_comm_init", C.c_int, [_P, _P, C.c_uint32, C.c_uint32]),
    ("fi_epp_comm_exchange", C.c_int, [_P]),
    ("fi_epp_set_profiling", C.c_int, [_P, C.c_int]),
    ("fi_epp_get_stats", C.c_int, [_P, C.POINTER(fi_epp_stats)]),
    ("fi_epp_reset_stats", C.c_int, [_P]),
]

_lib = None


def load() -> C.CDLL:
    """Load libfi_epp.so and bind every declared symbol.  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("FI_EPP_LIB", LIB_PATH)  # tuning: an alternative build of the same library
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `make` (or __graft_entry__.build()). "
            "fusioninfer_b200 has no CPU fallback for the pick path."
        )
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.fi_epp_abi_version() != FI_EPP_ABI_VERSION:
        raise RuntimeError("libfi_epp.so ABI version mismatch")
    _lib = lib
    return lib
