"""GPU (-m gpu): early-exit hashing.  A pick without chains_out on a single-rank handle with lru_capacity == 0 lets
hash_chain stop each request after its first block the index does not hold (hash_kernels.cu "early exit"; half-SM
tiles only, i.e. batches of more than 64 requests per SM).  Its picks must be bit-identical to the oracle's and to
the same call with chains_out given (which hashes whole chains), over every index state, prompt shape, block size,
tile shape and pick variant, and when index updates land between pipelined submits.  chains_out and
fi_epp_hash_batch still return whole chains.
"""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, subset_bitsets
from fusioninfer_b200 import _abi as abi
from oracle import epp_oracle as eo
from tests import helpers as H
from tests.test_gpu_ranked import CASES, _device_batch, _eq, _lora, _states

pytestmark = pytest.mark.gpu
UP, LPM = abi.FI_MATCH_UPSTREAM, abi.FI_MATCH_LPM
STATES = ["empty", "whole", "groups", "holes", "shuffled"]


def _big_R():
    """a batch of half-SM tiles on this device: more than 64 requests per SM"""
    import torch

    return 64 * torch.cuda.get_device_properties(0).multi_processor_count + 200


def _chain_ops(chains, nb, endpoints, lo=0, hi=None, op=abi.FI_OP_SET):
    """ops of blocks [lo, min(hi, nb[r])) of every row of chains for endpoints[r]"""
    j = np.arange(chains.shape[1])[None, :]
    mask = (j >= lo) & (j < nb[:, None].astype(np.int64)) & (j < (hi if hi is not None else chains.shape[1]))
    ops = np.zeros(int(mask.sum()), dtype=H.OP_DTYPE)
    ops["hash"] = chains[mask]
    ops["endpoint"] = np.broadcast_to(np.asarray(endpoints, dtype=np.uint32)[:, None], chains.shape)[mask]
    ops["op"] = op
    return ops


def _torch():
    import torch

    return torch


def _state_ops(wl, state, tok, offs, ref):
    """SET ops of one index state; ref hashes whole chains (fi_epp_hash_batch)"""
    if state == "empty":
        return []
    if state == "whole":  # every prompt's whole chain: no request stops
        chains, nb = ref.hash_batch(tok, offs, wl.h0)
        return [_chain_ops(chains, nb, np.arange(wl.R) % wl.E)]
    ops = list(wl.index_ops())
    if state == "shuffled":
        o = np.concatenate(ops)
        return [o[np.random.default_rng(11).permutation(len(o))]]
    return ops


def _handles(wl, state, mode, tok, offs, **kw):
    """the GPU handle copies host prompts in one piece: slices of the sliced host feed would be small batches, which
    hash whole chains"""
    cfg = H.config_for(wl, match_mode=mode, max_prompt_bytes=int(offs[-1]) + 4 * wl.R + 64, **kw)
    gpu, cpu = EndpointPicker(cfg), eo.Oracle(cfg)
    gpu.set_option("feed_slices", 1)
    st = wl.endpoint_states()
    gpu.update_endpoints(st)
    cpu.update_endpoints(st)
    for o in _state_ops(wl, state, tok, offs, gpu):
        gpu.index_apply(o)
        cpu.index_apply(o)
    return gpu, cpu


def _unaligned(tok, offs):
    """the same prompts with 1-3 junk bytes after each (inside its partial last block, so no block count changes):
    every prompt after the first starts off 8- and 16-byte alignment"""
    raw = np.ascontiguousarray(tok).view(np.uint8).reshape(-1)
    blobs = [raw[int(offs[r]):int(offs[r + 1])].tobytes() + b"\x01" * (1 + r % 3) for r in range(len(offs) - 1)]
    return H.pack_prompts(blobs)


def _check_batch(gpu, cpu, wl, tok, offs, what):
    """early exit (no chains) == oracle == the whole-chain call; chains_out == fi_epp_hash_batch"""
    got = gpu.pick_batch(tok, offs, wl.h0)
    full, chains = gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
    want = cpu.pick_batch(tok, offs, wl.h0)
    _eq(got, want, what + " (oracle)")
    _eq(got, full, what + " (chains_out)")
    ref, nb = gpu.hash_batch(tok, offs, wl.h0)
    assert np.array_equal(chains, ref), what
    assert np.array_equal(got[:, 0]["n_blocks"], nb), what
    return got, nb


# (block tokens, max_blocks, tokens per prompt): n % 8 != 0 for every block size, and prompts past the cap
SHAPES = [(8, 64, 8 * 61 + 5), (16, 64, 16 * 59 + 9), (24, 48, 24 * 45 + 7), (32, 40, 32 * 37 + 3)]


@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("mode", [UP, LPM])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{4 * s[0]}" for s in SHAPES])
def test_early_exit_equals_whole_chains(shape, mode, state):
    bt, M, T = shape
    wl = H.small_workload(E=40, R=_big_R(), T=T, max_blocks=M, block_tokens=bt, holes=state == "holes", lru_capacity=M)
    tok, offs = wl.prompts()
    gpu, cpu = _handles(wl, state, mode, tok, offs, index_slots=1 << 21)
    what = f"B={4 * bt} mode={mode} {state}"
    got, _ = _check_batch(gpu, cpu, wl, tok, offs, what)
    ut, uo = _unaligned(tok, offs)
    got_u, _ = _check_batch(gpu, cpu, wl, ut, uo, what + " unaligned")
    _eq(got_u, got, what + " unaligned vs aligned")
    if state != "empty" and mode == UP:
        assert (got[:, 0]["match_blocks"] > 0).any(), what
    gpu.close()
    cpu.close()


@pytest.mark.parametrize("state", ["empty", "whole", "groups", "shuffled"])
def test_hashed_blocks_counter(state):
    """An empty index stops every request within its first groups, a whole-chain index stops none; the hashed
    blocks always cover every request's blocks up to and including its first miss (N_probe)"""
    M = 256
    wl = H.small_workload(E=40, R=_big_R(), T=16 * M + 21, max_blocks=M, lru_capacity=M)
    tok, offs = wl.prompts()
    gpu, cpu = _handles(wl, state, UP, tok, offs, index_slots=1 << 23)
    gpu.set_profiling(True)
    gpu.reset_stats()
    got = gpu.pick_batch(tok, offs, wl.h0)
    st = gpu.stats()
    gpu.set_profiling(False)
    _eq(got, cpu.pick_batch(tok, offs, wl.h0), state)
    total = int(got[:, 0]["n_blocks"].astype(np.int64).sum())
    assert st.probed_blocks <= st.hashed_blocks <= total, (st.probed_blocks, st.hashed_blocks, total)
    if state == "whole":
        assert st.hashed_blocks == total
    if state == "empty":
        assert st.hashed_blocks < total // 2
    # the whole-chain call counts every block
    gpu.set_profiling(True)
    gpu.reset_stats()
    gpu.pick_batch(tok, offs, wl.h0, want_chains=True)
    assert gpu.stats().hashed_blocks == total
    gpu.set_profiling(False)
    gpu.close()
    cpu.close()


@pytest.mark.parametrize("R", [32, 64, 5000, 0])
def test_every_tile_shape(R):
    """whole-SM tiles of 32 and 64 requests (whole chains) and half-SM tiles of 64 (early exit; R = 0: more than 64
    requests per SM), 1 023-block prompts"""
    R = R or _big_R()
    M = 1023
    wl = H.small_workload(E=64, R=R, T=16 * M + 37, max_blocks=M, lru_capacity=M)
    tok, offs = wl.prompts()
    gpu, cpu = _handles(wl, "groups", UP, tok, offs, index_slots=1 << 22)
    _check_batch(gpu, cpu, wl, tok, offs, f"R={R}")
    gpu.close()
    cpu.close()


@pytest.mark.parametrize("case", ["pd", "lora", "weighted"])
@pytest.mark.parametrize("mode", [UP, LPM])
def test_pick_variants(case, mode):
    """PD, LoRA, ranked and subset picks with and without chains_out"""
    rng = np.random.default_rng(7 + mode)
    wl = H.small_workload(E=100, R=_big_R(), T=16 * 250 + 40, max_blocks=256, holes=True, lru_capacity=256)
    spec = dict(CASES[case])
    if case == "pd":
        spec["pd"] = dict(spec["pd"], threshold=0.6 * wl.T * 4)
    tok, offs = wl.prompts()
    cfg = H.config_for(wl, match_mode=mode, max_prompt_bytes=int(offs[-1]) + 64, index_slots=1 << 21, **spec)
    gpu = EndpointPicker(cfg)
    gpu.set_option("feed_slices", 1)
    gpu.update_endpoints(_states(wl, rng))
    if case == "lora":
        gpu.update_endpoints_lora(_lora(wl.E, rng))
    for o in wl.index_ops():
        gpu.index_apply(o)
    ad = (rng.integers(0, 14, wl.R) + 1000).astype(np.uint64) if case == "lora" else None
    sub = subset_bitsets([rng.choice(wl.E, [1, 8, 50, 100][r % 4], replace=False).tolist() for r in range(wl.R)], wl.E)
    for what, call in [
        ("single", lambda ch: gpu.pick_batch(tok, offs, wl.h0, want_chains=ch, adapters=ad)),
        ("ranked", lambda ch: gpu.pick_batch_ranked(tok, offs, wl.h0, 4, want_chains=ch, adapters=ad)),
        ("subset", lambda ch: gpu.pick_batch_subset(tok, offs, wl.h0, sub, 3, adapters=ad, want_chains=ch)),
    ]:
        early = call(False)
        full, _ = call(True)
        _eq(early, full, f"{case} mode={mode} {what}")
    gpu.close()


@pytest.mark.parametrize("update", ["set", "clear", "remove", "rebuild"])
def test_pipelined_submits_see_the_index_of_their_submit(update):
    """A submits three batches without chains (early exit), B runs the stream-ordered whole-chain picks at the same
    points; an index update between the submits changes where the next batch's chains stop"""
    torch = _torch()
    E, R, M = 32, _big_R(), 64
    wl = H.small_workload(E=E, R=R, T=16 * 61 + 9, max_blocks=M, lru_capacity=M)
    host = [wl.prompts(batch=0)] * 3
    cfg = H.config_for(wl, max_prompt_bytes=int(host[0][1][-1]) + 64, index_slots=1 << 18 if update == "rebuild" else 1 << 21)
    a, b = EndpointPicker(cfg), EndpointPicker(cfg)
    st = wl.endpoint_states()
    chains, nb = a.hash_batch(*host[0], wl.h0)
    # initial index: the first 20 blocks of every request's chain (10 where a rebuild is forced: the live keys stay
    # below 60 % of a small table)
    eps = np.arange(R) % E
    first = _chain_ops(chains, nb, eps, 0, 10 if update == "rebuild" else 20)
    for g in (a, b):
        g.update_endpoints(st)
        g.index_apply(first)
    if update == "set":  # extends every chain to its end
        ops = _chain_ops(chains, nb, eps, 20)
    elif update == "clear":  # cuts every chain at block 10
        ops = _chain_ops(chains, nb, eps, 10, 20, abi.FI_OP_CLEAR)
    elif update == "rebuild":  # keys that come and go leave tombstones until a rebuild compacts the table; the
        # chains then grow to 15 blocks
        junk = np.random.default_rng(3).integers(1, 2**63, (10, 20000), dtype=np.uint64)
        ops = []
        for k in range(10):
            fill = np.zeros(junk.shape[1], dtype=H.OP_DTYPE)
            fill["hash"] = junk[k]
            fill["op"] = abi.FI_OP_SET
            gone = fill.copy()
            gone["op"] = abi.FI_OP_CLEAR
            ops += [fill, gone]
        ops.append(_chain_ops(chains, nb, eps, 10, 15))
    s = torch.cuda.current_stream().cuda_stream
    dev = [_device_batch(tok, offs, wl.h0, R, 1, 1) for tok, offs in host]
    d_ch = torch.zeros(R * M, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    tickets, want = [], []
    rebuilds0 = a.index_stats().rebuilds
    for i in range(3):
        d = dev[i]
        tickets.append(a.pick_submit_ex(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), R, host[i][0].nbytes,
                                        d[3].data_ptr(), d_chains=d_ch.data_ptr() if i == 2 else 0, stream=s))
        want.append(b.pick_batch(*host[i], wl.h0, want_chains=True))
        if i == 0:
            for g in (a, b):
                if update == "remove":
                    g.remove_endpoints(list(range(0, E, 2)))
                elif update == "rebuild":
                    for o in ops:
                        g.index_apply(o)
                else:
                    g.index_apply(ops)
    a.pick_wait_batch(tickets[-1], s)
    torch.cuda.synchronize()
    for i in range(3):
        got = dev[i][3].cpu().numpy().view(H.PICK_DTYPE).reshape(R, 1)
        _eq(got, want[i][0], f"{update} batch {i}")
    # the batches before and after the update differ: the update did change where the chains stop
    assert not H.picks_equal(want[0][0], want[1][0]), update
    assert np.array_equal(d_ch.cpu().numpy().view(np.uint64).reshape(R, M), want[2][1]), "chains_out of a submit"
    if update == "rebuild":
        assert a.index_stats().rebuilds > rebuilds0
    a.close()
    b.close()
