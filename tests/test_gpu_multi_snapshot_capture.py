"""GPU (-m gpu, needs >= 2 devices): fi_epp_snapshot_capture refuses a sharded pool (docs/SPEC.md S.2d) with
FI_ERR_STATE on every rank, returns no capture, and the handle keeps serving picks."""
import ctypes as C
import threading

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.dist import shard_range
from tests import helpers as H

pytestmark = pytest.mark.gpu


def test_sharded_pool_is_refused(gpu_count):
    if gpu_count < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2
    wl = H.small_workload(E=64, R=16)
    uid = EndpointPicker.comm_unique_id()
    results, errors = [None] * world, []

    def worker(rank):
        try:
            begin, count = shard_range(wl.E, rank, world)
            p = EndpointPicker(H.config_for(wl, device=rank, endpoint_begin=begin, endpoint_count=count))
            p.comm_init(uid, rank, world)
            out, n = C.c_void_p(), C.c_uint64(0)
            rc = p._lib.fi_epp_snapshot_capture(p._h, C.byref(out), C.byref(n))
            results[rank] = (rc, out.value is None)
            p.close()
        except Exception as e:  # pragma: no cover
            errors.append((rank, repr(e)))

    ths = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=600)
    assert not errors, errors
    assert results == [(abi.FI_ERR_STATE, True)] * world
