"""Full-DEPTH, full-WIDTH parity of BASELINE.json configs[2..4] (VERDICT r01 item 1a): the 1e-3 cosine bar through all
24 / 28 / 30 bf16 layers of SGPT-1.3B (GPT-Neo), SGPT-5.8B (GPT-J, specb brackets, S = 300) and sgpt-bloom-7b1, each at
the batch x seq_len the config names.  The GPU encodes the whole batch; a few rows (always one full-length row and one
ragged row) are recomputed by the CPU oracle in fp32 from the SAME bf16-rounded weights.  Sequences are independent
(ragged execution, tests/test_oracle.py::test_ragged_equals_padded), so the oracle only needs those rows."""
import numpy as np
import pytest
import torch

from oracle import bloom, gpt_neo, gptj, pooling
from tests.helpers import full_size_weights, min_row_cosine, ragged_batch

pytestmark = pytest.mark.gpu

COS_TOL = 1e-3  # north_star: "within 1e-3 cosine on pooled embeddings"


def _check(enc, fwd, spec, lw, ids, mask, rows):
    out = enc.encode_tokens(ids.numpy(), mask.numpy(), method="weightedmean").cpu()
    assert torch.isfinite(out).all()
    with torch.no_grad():
        hs = fwd(spec, lw, ids[rows], mask[rows])[-1]
    want = pooling.weighted_mean(hs, mask[rows])
    cos = min_row_cosine(out[rows], want)
    print(f"[full depth] {type(spec).__name__} {spec.n_layer} layers d={spec.d_model}: min pooled-embedding cosine vs fp32 oracle "
          f"= {cos:.7f}")
    assert cos > 1 - COS_TOL, f"pooled-embedding cosine {cos:.6f} through {spec.n_layer} layers"
    again = enc.encode_tokens(ids.numpy(), mask.numpy(), method="weightedmean").cpu()
    assert torch.equal(again, out), "non-deterministic"
    return cos


def test_config3_sgpt_1_3b_full_depth_b64_s256():
    """SGPT-1.3B (GPT-Neo: 24 layers, d 2048, 16 heads of 128, local window 256 == causal at S 256), batch 64 x 256."""
    from sgpt_b200 import Encoder, preset

    spec = gpt_neo.NeoSpec(**gpt_neo.SGPT_1_3B)
    w, lw = full_size_weights("gpt_neo", spec, seed=3)
    enc = Encoder(preset("sgpt-1.3b"), w, device="cuda:0", max_tokens=64 * 256, max_batch=64)
    del w
    ids, mask = ragged_batch(64, 256, spec.vocab, seed=1236, pad_id=50256)
    mask[2:34] = 1  # half of the rows full length
    ids = torch.where(mask.bool(), ids, torch.full_like(ids, 50256))
    _check(enc, gpt_neo.forward, spec, lw, ids, mask, rows=[0, 1, 2, 40])
    enc.close()


def test_config4_sgpt_5_8b_gptj_full_depth_b32_s300_specb():
    """SGPT-5.8B (GPT-J: 28 layers, d 4096, 16 heads of 256, rotary 64, parallel residual), batch 32 x 300 with the
    asymmetric specb brackets: queries `[` ... `]` (ids 58/60), documents `{` ... `}` (ids 90/92), BDR:186-191."""
    from sgpt_b200 import Encoder, preset

    spec = gptj.GPTJSpec()
    w, lw = full_size_weights("gptj", spec, seed=4)
    enc = Encoder(preset("sgpt-5.8b"), w, device="cuda:0", max_tokens=32 * 300, max_batch=32)
    del w
    ids, mask = ragged_batch(32, 300, spec.vocab, seed=1237, pad_id=50256)
    mask[2:18] = 1
    lens = mask.sum(1)
    for b in range(32):
        if lens[b] >= 2:
            o, c = (58, 60) if b % 2 == 0 else (90, 92)  # even rows are queries, odd rows documents
            ids[b, 0], ids[b, lens[b] - 1] = o, c
    ids = torch.where(mask.bool(), ids, torch.full_like(ids, 50256))
    _check(enc, gptj.forward, spec, lw, ids, mask, rows=[2, 21])
    enc.close()


def test_config5_sgpt_bloom_7b1_full_depth_b32_s300():
    """sgpt-bloom-7b1 (BLOOM: 30 layers, d 4096, 32 heads of 128, ALiBi, embedding LayerNorm), batch 32 x 300."""
    from sgpt_b200 import Encoder, preset

    spec = bloom.BloomSpec()
    w, lw = full_size_weights("bloom", spec, seed=5)
    enc = Encoder(preset("sgpt-bloom-7b1"), w, device="cuda:0", max_tokens=32 * 300, max_batch=32)
    del w
    ids, mask = ragged_batch(32, 300, spec.vocab, seed=1238, pad_id=3)
    mask[2:18] = 1
    ids = torch.where(mask.bool(), ids, torch.full_like(ids, 3))
    _check(enc, bloom.forward, spec, lw, ids, mask, rows=[2, 25])
    enc.close()
