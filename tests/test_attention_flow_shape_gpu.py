"""GPU: the wgmma flash attention at the flow estimator's real launch shape - 64 ragged sequences (32 batch-32 Z10 utterances x 2 CFG
branches of 550, 620 or 690 mel frames), 8 heads, full attention and block-causal chunks of 50.  The grid then holds hundreds of co-resident
CTAs and many last query tiles with at most 64 valid rows (whose second warpgroup has nothing to compute), at the size the
benchmark runs.  Checked against the fp64 bound of test_kernel_edges_gpu, and each sequence computed alone must equal its rows of
the batched call bit for bit."""
import pytest
import torch

import kernel_refs as kr
from test_kernel_edges_gpu import _bf16_randn, _check_attention, _run_attention

pytestmark = pytest.mark.gpu

N_TEXT = [40 + (i * 7) % 21 for i in range(32)]               # synth.batch32_zero_shot(32)
FLOW_LENS = [150 + 10 * n for n in N_TEXT] * 2                 # 150 prompt frames + 2 x 5 x n_text; both CFG branches


@pytest.mark.parametrize("chunk", [0, 50])
def test_attention_estimator_shape(chunk):
    H = 8
    lens = FLOW_LENS
    # last query tiles of 38 (550), 108 (620) and 50 (690) rows: both warpgroups busy, or the second one idle
    assert sorted(set(lens)) == [550, 620, 690]
    g = torch.Generator().manual_seed(640 + chunk)
    R = sum(lens)
    q = _bf16_randn(R, H * 64, g=g)
    k = _bf16_randn(R, H * 64, g=g)
    v = _bf16_randn(R, H * 64, g=g)
    o = 0
    for i, L in enumerate(lens):
        if i % 2:        # a key tile read across a sequence edge is then an O(1) error in the neighbour
            v[o:o + L] = kr.bf16(v[o:o + L] * 1e4)
        o += L
    _check_attention(q, k, v, lens, lens, [0] * len(lens), H, H, chunk, "estimator", paths=[("bf16", 1)])
    full = _run_attention("bf16", 1, q, k, v, lens, lens, [0] * len(lens), H, H, chunk=chunk)
    o = 0
    for b, L in enumerate(lens):
        alone = _run_attention("bf16", 1, q[o:o + L], k[o:o + L], v[o:o + L], [L], [L], [0], H, H, chunk=chunk)
        assert torch.equal(alone, full[o:o + L]), (chunk, b, L, (alone - full[o:o + L]).abs().max().item())
        o += L
