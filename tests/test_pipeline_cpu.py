"""CPU: the planning behind fi_epp_index_add_submitted (docs/SPEC.md S.9).

Its sub-batches are cut with lru_touch_bound (lru_plan.h) so that the device LRU's touch kernel can never find a
table full, which lets the call go without the overflow readback of fi_epp_index_add_chains.  Checked here through
libfi_hostcheck.so: the bound against lru_maintain_kernel's thresholds and the insert limit on every table state, a
model of the tables under random request streams, and the plans' equality with sequential Adds.  The packed layout
both Add paths stage a plan in is read back the way the LRU kernels are handed it.
"""
import ctypes as C
import os

import numpy as np
import pytest

from fusioninfer_b200 import _abi as abi

LIB = os.path.join(abi.LIB_DIR, "libfi_hostcheck.so")


@pytest.fixture(scope="module")
def hc():
    lib = C.CDLL(LIB)
    lib.fihc_lru_touch_bound.restype = C.c_uint32
    lib.fihc_lru_touch_bound.argtypes = [C.c_uint32, C.c_uint32]
    lib.fihc_lru_bound_check.restype = C.c_int
    lib.fihc_lru_bound_check.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                         C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.fihc_lru_plan_check.restype = C.c_int
    lib.fihc_lru_plan_check.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                        C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p]
    lib.fihc_lru_plan_pack_check.restype = C.c_int
    lib.fihc_lru_plan_pack_check.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                             C.c_uint64, C.c_uint32, C.c_void_p]
    return lib


def _fits(used, count, add, C_, TS):
    """lru_maintain_kernel's decision, then the touch kernel's reservations: can `add` touches all get a slot?"""
    limit, addc = TS * 85 // 100, min(add, C_)
    if (used + addc) * 10 > TS * 6:
        used = count  # rebuilt from the live entries
    return used + add <= limit


@pytest.mark.parametrize("C_,TS", [(1, 4), (3, 16), (5, 32), (7, 32), (10, 64), (10, 320), (13, 512), (16, 64)])
def test_touch_bound_is_exact_over_every_table_state(hc, C_, TS):
    """every (used <= insert limit, count <= C) state takes `bound` touches; some state cannot take one more"""
    bound = hc.fihc_lru_touch_bound(TS, C_)
    assert bound >= 2 * C_
    limit = TS * 85 // 100
    states = [(u, c) for u in range(limit + 1) for c in range(min(C_, u) + 1)]
    for add in range(1, bound + 1):
        assert all(_fits(u, c, add, C_, TS) for u, c in states), add
    assert not all(_fits(u, c, bound + 1, C_, TS) for u, c in states)


def test_touch_bound_at_serving_sizes(hc):
    """lruCapacityPerServer 31 250 and the table sizes alloc_dev_lru picks (4 C .. 32 C, powers of two)"""
    C_ = 31250
    for TS in (1 << 17, 1 << 18, 1 << 19, 1 << 20):
        limit, calm = TS * 85 // 100, TS * 6 // 10
        assert hc.fihc_lru_touch_bound(TS, C_) == min(limit - calm + C_, limit - C_) >= 2 * C_


def _stream(rng, E, R, pitch, batches, hot):
    pool = rng.integers(1, 2**63, size=(40, pitch), dtype=np.uint64)
    eps = rng.integers(0, E, size=(batches, R)).astype(np.uint32)
    eps[rng.random((batches, R)) < hot] = 1  # one endpoint takes most of the traffic
    eps[1, :] = 2                            # and another a whole batch
    chains = pool[rng.integers(0, 40, size=(batches, R))].copy()
    fresh = rng.random((batches, R)) < 0.5   # many requests end in blocks nobody has seen
    chains[fresh, pitch // 4:] = rng.integers(1, 2**63, size=(int(fresh.sum()), pitch - pitch // 4), dtype=np.uint64)
    nb = rng.integers(0, pitch + 1, size=(batches, R)).astype(np.uint32)
    return eps, np.ascontiguousarray(chains), nb


@pytest.mark.parametrize("ts_mult", [4, 32])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_tables_never_pass_the_insert_limit(hc, ts_mult, seed):
    """random request streams with endpoints that receive many times their capacity in one batch"""
    rng = np.random.default_rng(seed * 10 + ts_mult)
    E, cap, R, pitch, batches = 6, 48, 400, 40, 8
    TS = 1 << (ts_mult * cap - 1).bit_length()  # pow2_ceil(ts_mult * C), as alloc_dev_lru sizes it
    eps, chains, nb = _stream(rng, E, R, pitch, batches, hot=0.6)
    assert int(nb[eps == 1].sum()) > 20 * cap
    pct, subs = C.c_double(0), C.c_uint32(0)
    rc = hc.fihc_lru_bound_check(E, cap, TS, eps.ctypes.data, chains.ctypes.data, pitch, nb.ctypes.data, R, batches,
                                 1 << 30, 1 << 30, C.byref(pct), C.byref(subs))
    assert rc == 0
    assert pct.value <= 85.0
    assert subs.value > batches  # the hot endpoints really were cut into several sub-batches


@pytest.mark.parametrize("ts_mult", [4, 32])
@pytest.mark.parametrize("cap_touches,cap_requests", [(1 << 30, 1 << 30), (500, 1 << 30), (1 << 30, 9)])
def test_plans_with_the_bound_equal_sequential_adds(hc, ts_mult, cap_touches, cap_requests):
    """request order within each endpoint, at most `bound` touches per endpoint and sub-batch, and the same recency
    order and content as one indexer.Add after the other (fihc_lru_plan_check)"""
    rng = np.random.default_rng(ts_mult + cap_requests)
    E, cap, R, pitch, batches = 5, 40, 300, 30, 6
    TS = 1 << (ts_mult * cap - 1).bit_length()
    bound = hc.fihc_lru_touch_bound(TS, cap)
    eps, chains, nb = _stream(rng, E, R, pitch, batches, hot=0.5)
    eps[eps == 4] = 0xFFFFFFFF  # FI_NO_ENDPOINT: skipped
    subs = C.c_uint32(0)
    rc = hc.fihc_lru_plan_check(E, cap, eps.ctypes.data, chains.ctypes.data, pitch, nb.ctypes.data, R, batches, bound,
                                cap_touches, cap_requests, C.byref(subs))
    assert rc == 0
    assert subs.value >= 2


# each case cuts its sub-batches on a different limit: touches per endpoint, touches, requests
@pytest.mark.parametrize("plan_cap,cap_touches,cap_requests", [(40, 1 << 30, 1 << 30), (0xFFFFFFFF, 50, 1 << 30),
                                                               (0xFFFFFFFF, 1 << 30, 9)])
def test_packed_plan_reads_back_through_the_offsets(hc, plan_cap, cap_touches, cap_requests):
    """the staging layout of a plan (lru_plan_pack) read back sub-batch by sub-batch through lru_plan_offsets, as the
    LRU kernels are handed it: every array equals the plan's, and the sections tile the packed words"""
    rng = np.random.default_rng(7)
    E, R, pitch, batches = 5, 300, 30, 6
    eps, _, nb = _stream(rng, E, R, pitch, batches, hot=0.5)
    eps[eps == 4] = 0xFFFFFFFF  # FI_NO_ENDPOINT: skipped
    eps[3, :] = 0xFFFFFFFF      # a batch with nothing to add: an empty plan

    def check(plan_cap, cap_touches, cap_requests):
        subs = C.c_uint32(0)
        rc = hc.fihc_lru_plan_pack_check(E, eps.ctypes.data, nb.ctypes.data, R, batches, plan_cap, cap_touches,
                                         cap_requests, C.byref(subs))
        assert rc == 0
        return subs.value

    uncut = check(0xFFFFFFFF, 1 << 30, 1 << 30)  # one sub-batch per non-empty batch
    assert uncut == batches - 1
    assert check(plan_cap, cap_touches, cap_requests) > 4 * uncut


def test_new_entry_points_are_declared_and_bound():
    import re

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "fi_epp.h")) as f:
        src = f.read()
    bound = {name: args for name, _, args in abi.SYMBOLS}
    for name in ("fi_epp_pick_submit_ex", "fi_epp_pick_wait_batch", "fi_epp_index_add_submitted"):
        decl = re.search(name + r"\s*\(([^)]*)\)", src)
        assert decl, name
        assert len(decl.group(1).split(",")) == len(bound[name]), name
