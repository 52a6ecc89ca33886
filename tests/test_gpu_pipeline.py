"""GPU (-m gpu): the pipelined calls of a serving loop (docs/SPEC.md S.9) — fi_epp_pick_submit_ex,
fi_epp_pick_wait_batch and fi_epp_index_add_submitted — through the C ABI, bit-exact against the stream-ordered calls
made at the same point on a second handle fed the same calls.
"""
import ctypes as C

import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.picker import FiEppError
from tests import helpers as H
from tests.test_gpu_ranked import CASES, _cold, _device_batch, _eq, _lora, _states

pytestmark = pytest.mark.gpu


def _torch():
    import torch

    return torch


def _pair(wl, case, mode, rng, prefill=True, **kw):
    """two handles in the same state: A runs the pipelined calls, B the stream-ordered ones"""
    spec = dict(CASES[case])
    if case == "pd":  # a threshold that splits the batch between prefill and skip
        spec["pd"] = dict(spec["pd"], threshold=0.6 * wl.T * 4)
    cfg = H.config_for(wl, match_mode=mode, max_prompt_bytes=wl.R * wl.T * 4, **spec, **kw)
    a, b = EndpointPicker(cfg), EndpointPicker(cfg)
    st = _states(wl, rng)
    lo = _lora(wl.E, rng) if case == "lora" else None
    ops = list(wl.index_ops()) if prefill else []
    for g in (a, b):
        g.update_endpoints(st)
        if lo is not None:
            g.update_endpoints_lora(lo)
        for o in ops:
            g.index_apply(o)
    return a, b


def _dev(a, dtype=np.int64):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a).view(dtype)).cuda()


def _picks(t, R, Pn, k):
    return t.cpu().numpy().view(H.PICK_DTYPE).reshape((R, Pn, k) if k else (R, Pn))


def _stream_ordered(g, b, R, nbytes, k, d_ad, d_sub, d_ch, s):
    """the counterpart of fi_epp_pick_submit_ex(k, adapters, subsets) on handle g"""
    if k == 0:
        rc = abi.load().fi_epp_pick_batch_device_lora(g._h, b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), d_ad, R,
                                                       nbytes, b[3].data_ptr(), d_ch, s)
        g._check(rc, "fi_epp_pick_batch_device_lora")
    else:
        g.pick_batch_device_subset(b[0].data_ptr(), b[1].data_ptr(), b[2].data_ptr(), R, nbytes, k, b[3].data_ptr(),
                                   d_sub or 0, d_ch or 0, s, d_ad or 0)


SHAPES = [(32, 64, 600), (4096, 32, 512), (100, 1023, 16 * 1023 + 40)]  # (E, max_blocks, tokens per prompt)


@pytest.mark.parametrize("case", ["weighted", "lora", "pd"])
@pytest.mark.parametrize("mode", [abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"E{e}-mb{m}" for e, m, _ in SHAPES])
def test_submit_ex_equals_the_stream_ordered_call(case, mode, shape):
    """every mode of fi_epp_pick_submit_ex with three batches in flight and index_apply / remove_endpoints between the
    submits: each batch equals the counterpart called at the same point, and d_chains_out equals fi_epp_hash_batch"""
    torch = _torch()
    E, max_blocks, T = shape
    rng = np.random.default_rng(E + max_blocks + mode)
    wl = H.small_workload(E=E, R=96, T=T, max_blocks=max_blocks, holes=True, lru_capacity=max_blocks)
    a, b = _pair(wl, case, mode, rng)
    Pn = len(CASES[case]["profiles"])
    s = torch.cuda.current_stream().cuda_stream
    batches = []
    for i in range(3):
        tok, offs = wl.prompts(batch=i)
        batches.append((tok, _cold(offs) if i == 0 else offs))
    ad = (rng.integers(0, 14, wl.R) + 1000).astype(np.uint64) if case == "lora" else None
    d_ad = _dev(ad) if ad is not None else None
    variants = [(0, False, True), (1, False, True), (1, True, True), (4, False, True), (4, True, True),
                (16, False, True), (16, True, True)]
    if case == "lora":
        variants.append((0, False, False))  # a LoRA profile with no adapter ids
    # every input built up front and one sync: the three submits of a variant then run back to back, with nothing
    # but the calls themselves between them
    chains0 = b.hash_batch(*batches[0], wl.h0)[0]
    ops = H.ops_array([(int(chains0[r, j]), (r * 7) % E, abi.FI_OP_SET)
                       for r in range(0, wl.R, 3) for j in range(min(4, max_blocks))])
    inputs = []
    for k, with_sub, with_ad in variants:
        per = []
        for tok, offs in batches:
            sub = subset_bitsets([rng.choice(E, min(E, [1, 8, E // 2, E][r % 4]), replace=False).tolist()
                                  for r in range(wl.R)], E) if with_sub else None
            per.append((_dev(sub, np.int32) if with_sub else None,
                        _device_batch(tok, offs, wl.h0, wl.R, max(k, 1), Pn), _device_batch(tok, offs, wl.h0, wl.R, max(k, 1), Pn),
                        torch.zeros(wl.R * max_blocks, dtype=torch.int64, device="cuda"),
                        torch.zeros(wl.R * max_blocks, dtype=torch.int64, device="cuda")))
        inputs.append(per)
    torch.cuda.synchronize()
    for (k, with_sub, with_ad), per in zip(variants, inputs):
        ad_ptr = d_ad.data_ptr() if (d_ad is not None and with_ad) else None
        pending = []
        for i, ((tok, offs), (d_sub, da, db, ch_a, ch_b)) in enumerate(zip(batches, per)):
            t = a.pick_submit_ex(da[0].data_ptr(), da[1].data_ptr(), da[2].data_ptr(), wl.R, tok.nbytes, da[3].data_ptr(),
                                 k=k, d_adapters=ad_ptr or 0, d_subsets=d_sub.data_ptr() if with_sub else 0,
                                 d_chains=ch_a.data_ptr(), stream=s)
            _stream_ordered(b, db, wl.R, tok.nbytes, k, ad_ptr, d_sub.data_ptr() if with_sub else None, ch_b.data_ptr(), s)
            pending.append((t, da, db, ch_a, ch_b, d_sub, tok, offs))
            # index updates between the submits: the next batch sees them, this one does not
            if i == 0:
                a.index_apply(ops)
                b.index_apply(ops)
            elif i == 1:
                victims = [0, E // 2, E - 1]
                a.remove_endpoints(victims)
                b.remove_endpoints(victims)
        a.pick_wait_batch(pending[-1][0], s)
        torch.cuda.synchronize()
        for i, (t, da, db, ch_a, ch_b, _, tok, offs) in enumerate(pending):
            what = f"k={k} subsets={with_sub} adapters={ad_ptr is not None} batch {i}"
            _eq(_picks(da[3], wl.R, Pn, k), _picks(db[3], wl.R, Pn, k), what)
            want = b.hash_batch(tok, offs, wl.h0)[0]
            assert np.array_equal(ch_a.cpu().numpy().view(np.uint64).reshape(wl.R, max_blocks), want), what
            assert np.array_equal(ch_b.cpu().numpy().view(np.uint64).reshape(wl.R, max_blocks), want), what
        assert [p[0] for p in pending] == list(range(pending[0][0], pending[0][0] + 3))
    a.close()
    b.close()


def test_wait_batch_completes_a_batch_and_tickets_are_shared():
    torch = _torch()
    rng = np.random.default_rng(9)
    wl = H.small_workload(E=64, R=512, T=4096, max_blocks=256, holes=True, lru_capacity=256)
    a, b = _pair(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng)
    s = torch.cuda.current_stream().cuda_stream
    side = torch.cuda.Stream()
    tok0, offs0 = wl.prompts(batch=0)
    small = 32
    d0 = _device_batch(tok0, offs0, wl.h0, small, 1, 1)
    tok1, offs1 = wl.prompts(batch=1)
    d1 = _device_batch(tok1, offs1, wl.h0, wl.R, 1, 1)
    torch.cuda.synchronize()
    t0 = a.pick_submit_ex(d0[0].data_ptr(), d0[1].data_ptr(), d0[2].data_ptr(), small, int(offs0[small]), d0[3].data_ptr(),
                          stream=s)
    t1 = a.pick_submit_ex(d1[0].data_ptr(), d1[1].data_ptr(), d1[2].data_ptr(), wl.R, tok1.nbytes, d1[3].data_ptr(), stream=s)
    a.pick_wait_batch(t0, side.cuda_stream)  # batch t1 is still submitted
    side.synchronize()
    _eq(_picks(d0[3], small, 1, 0), b.pick_batch(tok0[:small], offs0[: small + 1], wl.h0), "batch t0 after wait_batch(t0)")
    a.pick_wait_batch(t1, side.cuda_stream)
    side.synchronize()
    _eq(_picks(d1[3], wl.R, 1, 0), b.pick_batch(tok1, offs1, wl.h0), "batch t1 after wait_batch(t1)")
    # one sequence for both submit calls: fi_epp_pick_submit takes a number too
    a.pick_submit(d1[0].data_ptr(), d1[1].data_ptr(), d1[2].data_ptr(), wl.R, tok1.nbytes, d1[3].data_ptr(), s)
    t3 = a.pick_submit_ex(d0[0].data_ptr(), d0[1].data_ptr(), d0[2].data_ptr(), small, int(offs0[small]), d0[3].data_ptr(),
                          stream=s)
    assert (t0, t1, t3) == (t0, t0 + 1, t0 + 3)
    # a ticket more than the ring's length old: its wait still covers it (the ten later batches write elsewhere)
    later = [torch.zeros(small * 16, dtype=torch.uint8, device="cuda") for _ in range(10)]
    a.pick_wait(s)
    d0[3].zero_()
    torch.cuda.synchronize()
    t4 = a.pick_submit_ex(d0[0].data_ptr(), d0[1].data_ptr(), d0[2].data_ptr(), small, int(offs0[small]), d0[3].data_ptr(),
                          stream=s)
    for o in later:
        a.pick_submit_ex(d0[0].data_ptr(), d0[1].data_ptr(), d0[2].data_ptr(), small, int(offs0[small]), o.data_ptr(),
                         stream=s)
    assert t4 == t3 + 1
    a.pick_wait_batch(t4, side.cuda_stream)
    side.synchronize()
    _eq(_picks(d0[3], small, 1, 0), b.pick_batch(tok0[:small], offs0[: small + 1], wl.h0), "batch t4 after ten more")
    a.pick_wait(s)
    torch.cuda.synchronize()
    a.close()
    b.close()


LOOP = [  # (lru_capacity, lru_table_slots (0: default), index_slots (0: sized from the pool), check every n steps)
    (64, 4 * 64, 0, 1),
    (64, 0, 0, 3),  # several Adds in flight between two checks
    (64, 4 * 64, 4096, 1),  # a small index: rebuilds inside the loop
]


@pytest.mark.parametrize("cap,table_slots,index_slots,check_every", LOOP)
def test_serving_loop_equals_the_stream_ordered_loop(cap, table_slots, index_slots, check_every):
    """A: submit_ex(k+1), wait_batch(k), add_submitted(k), with no device-wide sync anywhere: batch k+1 is in flight
    while batch k is read and added, and Add(k) is in flight when batch k+2 is submitted.  B: the stream-ordered pick
    and fi_epp_index_add_chains with its chains, in the same logical order.  Every step's picks are equal; the index
    over every pair and the LRU of every endpoint the Adds touched are equal at every check, which is made after the
    next submit (so it does not drain the pipeline).  Half of every batch goes to one endpoint, many times the touch
    bound (several sub-batches)."""
    torch = _torch()
    rng = np.random.default_rng(cap + table_slots + index_slots + check_every)
    E, R, steps = 16, 160, 12
    wl = H.small_workload(E=E, R=R, T=600, max_blocks=32, lru_capacity=cap)
    kw = dict(lru_capacity=cap)
    if index_slots:
        kw["index_slots"] = index_slots
    a, b = _pair(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng, prefill=False, **kw)  # the Adds fill the index
    if table_slots:
        a.set_option("lru_table_slots", table_slots)
        b.set_option("lru_table_slots", table_slots)
    stream = torch.cuda.current_stream()
    s = stream.cuda_stream
    Pn = 1
    host = [wl.prompts(batch=i) for i in range(steps + 1)]
    dev = [_device_batch(tok, offs, wl.h0, R, 1, Pn) for tok, offs in host]
    torch.cuda.synchronize()  # the inputs are in place; from here on only the caller's stream is ever synchronised

    def submit(i):
        d = dev[i]
        return a.pick_submit_ex(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), R, host[i][0].nbytes, d[3].data_ptr(),
                                stream=s)

    def route(picks):
        eps = picks[:, 0]["endpoint"].copy()
        eps[: R // 2] = 3  # the hot endpoint
        return eps, picks[:, 0]["n_blocks"].astype(np.uint32)

    touched = []  # (pairs, endpoints) added since the last check

    def check(after):
        q = H.ops_array([x for pairs, _ in touched for x in pairs])
        assert np.array_equal(a.index_contains(q), b.index_contains(q)), f"index after {after}"
        for e in sorted(set(e for _, eps in touched for e in eps)):
            assert np.array_equal(a.lru_dump(e), b.lru_dump(e)), f"LRU of endpoint {e} after {after}"
        touched.clear()

    tickets = {0: submit(0)}
    want = {0: b.pick_batch(*host[0], wl.h0, want_chains=True)}
    for k in range(steps):
        tickets[k + 1] = submit(k + 1)
        want[k + 1] = b.pick_batch(*host[k + 1], wl.h0, want_chains=True)
        if touched and k % check_every == 0:
            check(f"Add {k - 1}")  # ordered after Add(k-1) and before Add(k) on A's index stream
        a.pick_wait_batch(tickets[k], s)
        stream.synchronize()
        got = _picks(dev[k][3], R, Pn, 0)
        wp, wc = want.pop(k)
        _eq(got, wp, f"step {k}")
        eps, nb = route(got)
        a.index_add_submitted(tickets[k], eps, nb)
        b.index_add_chains(eps, wc, nb)
        touched.append(([(int(wc[r, j]), int(eps[r]), abi.FI_OP_SET) for r in range(R) for j in range(int(nb[r]))],
                        [int(x) for x in eps if x != abi.FI_NO_ENDPOINT]))
    check("the last Add")
    a.pick_wait(s)
    torch.cuda.synchronize()
    ca = a.lru_counters()
    assert ca["deferred_requests"] == 0
    assert ca["sub_batches"] > 2 * steps  # the hot endpoint's touches were cut into several sub-batches
    if index_slots:
        assert a.index_stats().rebuilds > 0
    a.index_sync()  # reports a broken device-LRU invariant, if any
    a.close()
    b.close()


def _status(fn):
    try:
        fn()
    except FiEppError as e:
        return e.status
    return abi.FI_OK


def test_errors():
    torch = _torch()
    lib = abi.load()
    rng = np.random.default_rng(1)
    wl = H.small_workload(E=40, R=32, lru_capacity=64)
    a, _ = _pair(wl, "weighted", abi.FI_MATCH_UPSTREAM, rng, lru_capacity=64)
    s = torch.cuda.current_stream().cuda_stream
    tok, offs = wl.prompts()
    d = _device_batch(tok, offs, wl.h0, wl.R, 4, 1)
    d_sub = _dev(subset_bitsets([None] * wl.R, wl.E), np.int32)
    torch.cuda.synchronize()
    p = [x.data_ptr() for x in d]
    t = C.c_uint64(0)

    def sub_ex(R=wl.R, k=0, out=p[3], subsets=None, offsets=p[1]):
        return lib.fi_epp_pick_submit_ex(a._h, p[0], offsets, p[2], None, subsets, R, tok.nbytes, k, out, None, s, C.byref(t))

    assert sub_ex(k=0, subsets=d_sub.data_ptr()) == abi.FI_ERR_INVALID  # subsets need k >= 1
    assert sub_ex(k=abi.FI_EPP_MAX_RANKED + 1) == abi.FI_ERR_INVALID
    assert sub_ex(k=2, out=None, R=0) == abi.FI_ERR_INVALID
    assert sub_ex(offsets=None) == abi.FI_ERR_INVALID
    assert sub_ex(R=wl.R + 1) == abi.FI_ERR_CAPACITY
    assert sub_ex(R=wl.R + 1, k=2) == abi.FI_ERR_CAPACITY
    assert lib.fi_epp_pick_wait_batch(a._h, 10**9, s) == abi.FI_ERR_INVALID
    eps = np.zeros(wl.R, dtype=np.uint32)
    nb = np.full(wl.R, 2, dtype=np.uint32)
    assert _status(lambda: a.index_add_submitted(10**9, eps, nb)) == abi.FI_ERR_INVALID  # never issued
    t0 = a.pick_submit_ex(p[0], p[1], p[2], wl.R, tok.nbytes, p[3], k=4, d_subsets=d_sub.data_ptr(), stream=s)
    t1 = a.pick_submit_ex(p[0], p[1], p[2], wl.R, tok.nbytes, p[3], stream=s)
    assert _status(lambda: a.index_add_submitted(t0, np.concatenate([eps, eps]), np.concatenate([nb, nb]))) == abi.FI_ERR_STATE
    bad = eps.copy()
    bad[3] = wl.E
    assert _status(lambda: a.index_add_submitted(t0, bad, nb)) == abi.FI_ERR_INVALID
    assert _status(lambda: a.index_add_submitted(t0, eps, nb + np.uint32(wl.max_blocks))) == abi.FI_ERR_INVALID
    a.index_add_submitted(t0, eps, nb)
    a.pick_submit_ex(p[0], p[1], p[2], wl.R, tok.nbytes, p[3], stream=s)
    assert _status(lambda: a.index_add_submitted(t0, eps, nb)) == abi.FI_ERR_STATE  # two submits later
    a.index_add_submitted(t1, eps, nb)
    t3 = a.pick_submit_ex(p[0], p[1], p[2], wl.R, tok.nbytes, p[3], stream=s)
    a.pick_batch(tok, offs, wl.h0)  # a stream-ordered pick
    assert _status(lambda: a.index_add_submitted(t3, eps, nb)) == abi.FI_ERR_STATE
    t4 = a.pick_submit_ex(p[0], p[1], p[2], wl.R, tok.nbytes, p[3], stream=s)
    a.hash_batch(tok, offs, wl.h0)  # a stream-ordered hash
    assert _status(lambda: a.index_add_submitted(t4, eps, nb)) == abi.FI_ERR_STATE
    a.pick_wait(s)
    torch.cuda.synchronize()
    a.close()
    # the host LRU, and no LRU at all
    for opts, kw in (({"device_lru": 0}, dict(lru_capacity=64)), ({}, dict(lru_capacity=0))):
        g = EndpointPicker(H.config_for(wl, **kw))
        for n, v in opts.items():
            g.set_option(n, v)
        tk = g.pick_submit_ex(p[0], p[1], p[2], wl.R, tok.nbytes, p[3], stream=s)
        assert _status(lambda: g.index_add_submitted(tk, eps, nb)) == abi.FI_ERR_STATE
        g.pick_wait(s)
        torch.cuda.synchronize()
        g.close()
    # a handle over part of the pool: subsets refused, the ranked submit served
    wl2 = H.small_workload(E=300, R=32, holes=True)
    g = EndpointPicker(H.config_for(wl2, endpoint_begin=100, endpoint_count=150))
    g.update_endpoints(wl2.endpoint_states())
    tok2, offs2 = wl2.prompts()
    d2 = _device_batch(tok2, offs2, wl2.h0, wl2.R, 2, 1)
    d_sub2 = _dev(subset_bitsets([None] * wl2.R, wl2.E), np.int32)
    torch.cuda.synchronize()
    assert _status(lambda: g.pick_submit_ex(d2[0].data_ptr(), d2[1].data_ptr(), d2[2].data_ptr(), wl2.R, tok2.nbytes,
                                            d2[3].data_ptr(), k=2, d_subsets=d_sub2.data_ptr(), stream=s)) == abi.FI_ERR_STATE
    tk = g.pick_submit_ex(d2[0].data_ptr(), d2[1].data_ptr(), d2[2].data_ptr(), wl2.R, tok2.nbytes, d2[3].data_ptr(), k=2,
                          stream=s)
    g.pick_wait_batch(tk, s)
    torch.cuda.synchronize()
    _eq(_picks(d2[3], wl2.R, 1, 2), g.pick_batch_ranked(tok2, offs2, wl2.h0, 2), "sub-range ranked submit")
    g.close()


def test_odd_block_size_takes_the_stream_ordered_path():
    """block_bytes % 32 != 0: the counterpart runs inside; the ticket is issued, its chains are not kept"""
    torch = _torch()
    wl = H.small_workload(E=40, R=64, block_tokens=5, lru_capacity=64)
    g = EndpointPicker(H.config_for(wl, lru_capacity=64, max_prompt_bytes=wl.R * wl.T * 4))
    g.update_endpoints(wl.endpoint_states())
    tok, offs = wl.prompts()
    d = _device_batch(tok, offs, wl.h0, wl.R, 4, 1)
    torch.cuda.synchronize()
    s = torch.cuda.current_stream().cuda_stream
    t = g.pick_submit_ex(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), wl.R, tok.nbytes, d[3].data_ptr(), k=4, stream=s)
    g.pick_wait_batch(t, s)
    torch.cuda.synchronize()
    _eq(_picks(d[3], wl.R, 1, 4), g.pick_batch_ranked(tok, offs, wl.h0, 4), "odd block size, ranked submit")
    eps = np.zeros(wl.R, dtype=np.uint32)
    assert _status(lambda: g.index_add_submitted(t, eps, np.ones(wl.R, dtype=np.uint32))) == abi.FI_ERR_STATE
    g.close()
