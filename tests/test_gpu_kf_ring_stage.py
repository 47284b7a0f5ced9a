"""The stage of the fused ring of the 4/2 fp32 step is laid out per launch from the record planes it copies
and the number of steps, and the CTAs per SM follow from that size: every layout, from no varying word and
one step (the smallest stage, 4 CTAs per SM) to all 37 words and 8 steps (the largest, 3 CTAs per SM), is
bit for bit the same as separate steps, over enough tiles that every CTA refills both of its stages."""
import numpy as np
import pytest

from test_gpu_kf_ring import BANKS, _CBank, _same_bits

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K", [1, 3, 5, 6, 7, 8])
@pytest.mark.parametrize("kind", ["bench", "one_model", "all_words"])
def test_every_stage_layout_equals_separate_steps_bit_for_bit(kind, K):
    N = (1 << 19) + 77                                  # a ragged last tile, some eight tiles per CTA
    make, k = BANKS[kind]
    b = _CBank(make(N), N)
    assert bin(b.hmap.varying).count("1") == k
    rc, x, P = b.ring(b.zs[:K])
    assert rc == 0, b.lib.bke_last_error()
    xs, Ps = b.stepwise(b.zs[:K])
    _same_bits(x, xs, "x"); _same_bits(P, Ps, "P")
    assert np.isfinite(x.cpu().numpy()).all()
