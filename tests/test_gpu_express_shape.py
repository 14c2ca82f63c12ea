"""The express kernel's residency: narrow-id models run it as 2 blocks of 14 warps per SM (28 warps, 72 registers,
shared memory inside the 132 KB carve-out).  The profile's per-warp buffer covers the larger of the express grid and
the buffer-path grid, so a batch that fills every SM reports the express kernel's resident warps."""
import os

import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)


def test_express_kernel_holds_28_warps_per_sm(oracle):
    import torch
    import xllm_service_b200 as x
    from xllm_service_b200 import workload
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    texts = [s.encode() for s in workload.sentences(30 * n_sm, (1, 12), seed=11)]
    b = workload.pack_prompts(texts)
    model = os.path.join(HERE, "golden", "sp_bpe_8k")
    h = x.Ingest(tokenizer_path=model)
    try:
        n_ids, status, warp_ns = h.encode_batch_profile(b.text, b.offsets, 128)
        ids, n_ids2, status2 = h.encode_batch(b.text, b.offsets, 128)
    finally:
        h.close()
    assert (status == 0).all() and (n_ids == n_ids2).all() and (status == status2).all()
    # the buffer-path kernel holds at most 27 one-warp blocks per SM, so 28 per SM can only be the express kernel's
    assert warp_ns.size == 28 * n_sm, (warp_ns.size, n_sm)
    sp = oracle.SentencePieceOracle(model)
    for r in range(0, b.n, 61):
        assert ids[r, :n_ids[r]].tolist() == sp.encode(b.prompt(r)).tolist(), r
