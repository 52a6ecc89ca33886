"""fusioninfer_b200 — H100-native prefix-cache-aware Endpoint Picker hot path.

One path only (BASELINE.json north_star, SURVEY.md §8): hash prompts into chained
block keys → look them up in a GPU-resident (endpoint, block-hash) index →
weighted fp64 score → argmax, behind the C ABI of include/fi_epp.h.
"""
from . import _abi  # noqa: F401
from .picker import (  # noqa: F401
    ENDPOINT_DTYPE,
    LORA_DTYPE,
    OP_DTYPE,
    PICK_DTYPE,
    EndpointPicker,
    FiEppError,
    PinnedBuffer,
    SnapshotCapture,
    config_from_yaml,
    config_picker_endpoints,
    default_config,
    make_config,
    model_seed,
    snapshot_info,
    subset_bitsets,
)

__all__ = [
    "EndpointPicker",
    "FiEppError",
    "PinnedBuffer",
    "SnapshotCapture",
    "config_from_yaml",
    "config_picker_endpoints",
    "default_config",
    "make_config",
    "model_seed",
    "snapshot_info",
    "subset_bitsets",
    "PICK_DTYPE",
    "OP_DTYPE",
    "ENDPOINT_DTYPE",
    "LORA_DTYPE",
]
