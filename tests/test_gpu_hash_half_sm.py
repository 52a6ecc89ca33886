"""GPU (-m gpu): batches of more than 64 requests per SM hash with half-SM hash_chain tiles (16 warps: 2 walkers + 14
hashers, 64 requests per CTA, two CTAs per SM).  Pipelined submits of such batches, where the tiles of batch k+1 start
on the SMs that match_pick of batch k is leaving, must equal the stream-ordered call byte for byte, and the chains
must equal the oracle's."""
import numpy as np
import pytest

from fusioninfer_b200 import EndpointPicker, synth
from oracle import epp_oracle as eo
from tests import helpers as H

pytestmark = pytest.mark.gpu


def test_pipelined_half_sm_batches_equal_the_stream_ordered_call():
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    R = 64 * sms + 77  # more tiles of 64 than SMs, and a partial last tile
    wl = synth.Workload(R=R, E=64, T=512, seed=synth.SEEDS[1], max_blocks=32, lru_capacity=600)
    cfg = H.config_for(wl, max_prompt_bytes=R * wl.T * 4, profiles=[{"name": "default", "scorers": [(H.P, 100), (H.K, 10), (H.Q, 10)]}])
    gpu, cpu = EndpointPicker(cfg), eo.Oracle(cfg)
    gpu.update_endpoints(wl.endpoint_states())
    for ops in wl.index_ops():
        gpu.index_apply(ops)
    gpu.index_sync()
    n_batches = 5
    host = [wl.prompts(batch=b) for b in range(n_batches)]
    d_tok = [torch.from_numpy(t.view(np.int32)).cuda() for t, _ in host]
    d_off = [torch.from_numpy(o.view(np.int64)).cuda() for _, o in host]
    d_h0 = torch.full((R,), int(np.uint64(wl.h0).astype(np.int64)), dtype=torch.int64, device="cuda")
    nbytes = R * wl.T * 4
    piped = [torch.zeros(R * 16, dtype=torch.uint8, device="cuda") for _ in range(n_batches)]
    s = torch.cuda.current_stream().cuda_stream
    for b in range(n_batches):
        gpu.pick_submit(d_tok[b].data_ptr(), d_off[b].data_ptr(), d_h0.data_ptr(), R, nbytes, piped[b].data_ptr(), s)
    gpu.pick_wait(s)
    torch.cuda.synchronize()
    ordered = torch.zeros(R * 16, dtype=torch.uint8, device="cuda")
    matched = 0
    for b in range(n_batches):
        gpu.pick_batch_device(d_tok[b].data_ptr(), d_off[b].data_ptr(), d_h0.data_ptr(), R, nbytes, ordered.data_ptr(), 0, s)
        torch.cuda.synchronize()
        assert torch.equal(piped[b], ordered), f"batch {b}"
        matched += int((ordered.cpu().numpy().view(H.PICK_DTYPE)["match_blocks"] > 0).sum())
    assert matched > 0
    gc, gn = gpu.hash_batch(host[0][0], host[0][1], wl.h0)
    wc, wn = cpu.hash_batch(host[0][0], host[0][1], wl.h0)
    assert np.array_equal(gn, wn) and np.array_equal(gc, wc)
    gpu.close()
    cpu.close()
