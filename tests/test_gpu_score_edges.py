"""GPU (-m gpu): the scoring edge cases of tests/score_edges.py through every pick entry point, bit for bit against
the CPU oracles and, for the single pick, the exact reference spec_total.

Pool sizes 3, 40, 100, 1024, 2048 and 4096 give membership rows of 1, 2, 4, 32, 64 and 128 words: every
match_pick_kernel row shape and tie_first_local word count.  The non-LoRA cases run the single pick's zero-match
shortcut (the per-batch zero best and its tie set), the LoRA case the kernel that scores every endpoint.  A few
hundred requests per case start the tie rotation at many different endpoints."""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker
from fusioninfer_b200 import _abi as abi
from fusioninfer_b200.dist import shard_range
from fusioninfer_b200.picker import FiEppError
from oracle import epp_oracle as eo
from tests import score_edges as S
from tests.helpers import describe_diff
from tests.ext_oracle import ExtOracle

pytestmark = pytest.mark.gpu


def _eq(got, want, what):
    assert got.tobytes() == want.tobytes(), what + "\n" + describe_diff(got, want)


def _device_inputs(c, k, Pn, sub=None):
    import torch

    d_tok = torch.from_numpy(c.tok.copy()).cuda()
    d_off = torch.from_numpy(c.offs.view(np.int64).copy()).cuda()
    d_h0 = torch.full((c.R,), np.uint64(c.h0).astype(np.int64), dtype=torch.int64, device="cuda")
    d_out = torch.zeros(c.R * Pn * max(k, 1) * 16, dtype=torch.uint8, device="cuda")
    d_ad = torch.from_numpy(c.adapters.view(np.int64).copy()).cuda() if c.adapters is not None else None
    d_sub = torch.from_numpy(sub.view(np.int32).copy()).cuda() if sub is not None else None
    return d_tok, d_off, d_h0, d_out, d_ad, d_sub


@pytest.mark.parametrize("kind,E", S.GPU_CASES, ids=[f"{k}-E{e}" for k, e in S.GPU_CASES])
def test_every_entry_point_on_the_edges(kind, E):
    import torch

    c = S.gpu_case(kind, E)
    cfg = c.config()
    Pn = len(c.profiles)
    g, o = EndpointPicker(cfg), ExtOracle(cfg)
    for x in (g, o):
        c.load(x)
    spec = S.Spec(c)
    ad = c.adapters

    # the single pick: zero-match shortcut (no LoRA scorer) or every endpoint scored (LoRA)
    single = g.pick_batch(c.tok, c.offs, c.h0, adapters=ad)
    _eq(single, o.pick_batch(c.tok, c.offs, c.h0, adapters=ad), "pick_batch vs the oracle")
    _eq(single, spec.picks(), "pick_batch vs spec_total")

    # ranked: k = 16 is above the eligible count of the small pools and of the edge cases' "few" profile
    for k in (1, 5, 16):
        got = g.pick_batch_ranked(c.tok, c.offs, c.h0, k, adapters=ad)
        _eq(got, o.pick_batch_ranked(c.tok, c.offs, c.h0, k, adapters=ad), f"pick_batch_ranked k={k} vs the oracle")
        _eq(np.ascontiguousarray(got[:, :, 0]), single, f"pick_batch_ranked k={k} entry 0 vs pick_batch")
    if kind == "edges" or E == 3:
        elig = int(spec.elig[1 if kind == "edges" else 0].sum())
        assert elig < 16, elig

    # subsets: random, singleton, empty, full, and with the queue extremes inside and outside
    sub = S.subset_rows(c, seed=E)
    for k in (1, 5):
        got = g.pick_batch_subset(c.tok, c.offs, c.h0, sub, k, adapters=ad)
        _eq(got, o.pick_batch_subset(c.tok, c.offs, c.h0, sub, k, adapters=ad), f"pick_batch_subset k={k} vs the oracle")
    if E <= 100:
        _eq(got, spec.ranked(5, sub), "pick_batch_subset k=5 vs the subset-aware spec")

    # the pipelined submit: k = 0 (the single pick on device buffers) and k = 5 with subsets
    s = torch.cuda.current_stream().cuda_stream
    d0 = _device_inputs(c, 0, Pn)
    d5 = _device_inputs(c, 5, Pn, sub)
    torch.cuda.synchronize()
    nbytes = int(c.offs[-1])
    t0 = g.pick_submit_ex(d0[0].data_ptr(), d0[1].data_ptr(), d0[2].data_ptr(), c.R, nbytes, d0[3].data_ptr(), k=0,
                          d_adapters=d0[4].data_ptr() if ad is not None else 0, stream=s)
    t5 = g.pick_submit_ex(d5[0].data_ptr(), d5[1].data_ptr(), d5[2].data_ptr(), c.R, nbytes, d5[3].data_ptr(), k=5,
                          d_adapters=d5[4].data_ptr() if ad is not None else 0, d_subsets=d5[5].data_ptr(), stream=s)
    g.pick_wait_batch(t5, s)
    torch.cuda.synchronize()
    assert t5 == t0 + 1
    _eq(d0[3].cpu().numpy().view(S.PICK_DTYPE).reshape(c.R, Pn), single, "pick_submit_ex k=0 vs pick_batch")
    _eq(d5[3].cpu().numpy().view(S.PICK_DTYPE).reshape(c.R, Pn, 5),
        o.pick_batch_subset(c.tok, c.offs, c.h0, sub, 5, adapters=ad), "pick_submit_ex k=5 with subsets vs the oracle")
    g.close()
    o.close()


@pytest.mark.parametrize("E", [40, 1024])
def test_zero_match_ties_are_rotated_against_matched_endpoints(E):
    """prefix weight 0 next to kv and queue scorers, most of the pool in one identical best state: matched and
    unmatched endpoints tie, the matched ones sit on both sides of the rotation start, and the rotation alone picks.
    Some picks go to an unmatched endpoint ahead of a tied matched one, and some to a matched one."""
    c = S.gpu_case("zero_tie", E)
    spec = S.Spec(c)
    want = spec.picks()
    g = EndpointPicker(c.config())
    c.load(g)
    _eq(g.pick_batch(c.tok, c.offs, c.h0), want, "pick_batch vs spec_total")
    g.close()
    n_unmatched_wins = n_matched_wins = 0
    for r in range(c.R):
        n, _, matches, start = spec.requests[r]
        e, score = int(want[r, 0]["endpoint"]), float(want[r, 0]["score"])
        # matched eligible endpoints whose own total equals the pick's: they tie with it
        tied_matched = [m for m in matches if m != e and spec.elig[0][m] and spec.total_of(0, r, m) == score]
        if not tied_matched:
            continue
        if e in matches:
            n_matched_wins += 1  # a matched endpoint comes first in rotation among the tied ones
        elif e not in matches and all((m - start) % E > (e - start) % E for m in tied_matched):
            n_unmatched_wins += 1  # an unmatched endpoint ahead of every tied matched one
    assert n_unmatched_wins > 0 and n_matched_wins > 0, (n_unmatched_wins, n_matched_wins)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), float("-inf")])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_update_endpoints_with_a_non_finite_kv_applies_nothing(bad, where):
    """fi_epp_endpoints_update with a NaN or infinite kv_util in any entry is FI_ERR_INVALID and applies none of the
    entries, the valid ones included: the picks after the call equal those before it"""
    c = S.gpu_case("edges", 100)
    g = EndpointPicker(c.config())
    c.load(g)
    before = g.pick_batch(c.tok, c.offs, c.h0)
    upd = c.states.copy()
    upd["kv_util"] = upd["kv_util"][::-1].copy()  # a change that moves picks when it is applied
    upd["queue_depth"] = upd["queue_depth"][::-1].copy()
    i = {"first": 0, "middle": c.E // 2, "last": c.E - 1}[where]
    upd["kv_util"][i] = bad
    with pytest.raises(FiEppError) as ei:
        g.update_endpoints(upd)
    assert ei.value.status == abi.FI_ERR_INVALID
    _eq(g.pick_batch(c.tok, c.offs, c.h0), before, "picks after a rejected update")
    upd["kv_util"][i] = 0.5
    g.update_endpoints(upd)
    assert g.pick_batch(c.tok, c.offs, c.h0).tobytes() != before.tobytes(), "the update would have moved picks"
    g.close()


def test_sharded_pd_edges_merge(gpu_count):
    """merge_picks_kernel: a pool sharded by endpoint range over two GPUs reduces the ranks' picks and applies the PD
    rule with the threshold exactly on (1 - hit) * len; equal to the unsharded oracle and spec_total"""
    if gpu_count < 2:
        pytest.skip("needs >= 2 GPUs")
    import threading

    c = S.gpu_case("pd_exact", 100)
    uid = EndpointPicker.comm_unique_id()
    results, errors = [None, None], []

    def worker(rank):
        try:
            begin, count = shard_range(c.E, rank, 2)
            p = EndpointPicker(c.config(device=rank, endpoint_begin=begin, endpoint_count=count))
            p.comm_init(uid, rank, 2)
            c.load(p)
            results[rank] = p.pick_batch(c.tok, c.offs, c.h0)
            p.close()
        except Exception as e:  # pragma: no cover
            errors.append((rank, repr(e)))

    ths = [threading.Thread(target=worker, args=(r,)) for r in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join(timeout=600)
    assert not errors, errors
    o = eo.Oracle(c.config())
    c.load(o)
    want = o.pick_batch(c.tok, c.offs, c.h0)
    _eq(want, S.spec_picks(c), "oracle vs spec_total")
    for rank in range(2):
        _eq(results[rank], want, f"rank {rank} vs the oracle")
