"""GPU parity: K1 when every persistent CTA walks many work units.

Each CTA of the filter GEMM keeps two A buffers whose barrier phases wrap every other unit; the small sets of the other
tests give most CTAs one or two units.  Twenty images of 1000-1100 features matched exhaustively make about 950
256-row units in the row direction alone, several per CTA on any current GPU."""
import numpy as np
import pytest

import oracle
from pycolmap_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def test_many_units_per_cta_equal_oracle(ctx):
    rng = np.random.default_rng(11)
    nf = [int(n) for n in rng.integers(1000, 1101, 20)]
    descs = [syn.sift_like(rng, n) for n in nf]
    for a in range(0, 20, 2):
        b = (a + 5) % 20
        k = 300 + 10 * a
        descs[b][:k] = syn.perturb(rng, descs[a][:k])
    ctx.set_images(descs)
    pairs = syn.exhaustive_pairs(len(nf))
    res = ctx.match_pairs(pairs)
    want = oracle.fast_match_pairs(np.concatenate(descs), nf, pairs)
    assert len(res) == len(pairs)
    total = 0
    for k in range(len(pairs)):
        got = res.matches(k)
        assert np.array_equal(got, want[k]), (k, pairs[k])
        total += len(got)
    assert res.total_matches == total and total > 1000
