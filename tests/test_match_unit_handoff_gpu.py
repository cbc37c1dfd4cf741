"""GPU parity: K1's hand-off of each work unit's row decisions from the consumer warpgroups to the finishing warps.

The consumers hand (best, S1, slot) of every row of a unit to two shared-memory buffers, and the producer publishes
each unit's tile count beside its A strip.  Here every pair shares descriptors, so consecutive units of one CTA all
produce candidates; feature counts are not multiples of 256, so the last unit of an image has rows past its end; one
image is empty, so some units have no column tile at all.  Fifteen images matched exhaustively make 630 row-direction
units (1260 with both directions in one launch), several per CTA and more than the two decision buffers."""
import os

import numpy as np
import pytest

import oracle
import pycolmap_b200 as pb
from pycolmap_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _images(rng):
    base = syn.sift_like(rng, 1500)
    descs = []
    for i in range(15):
        if i == 5:
            descs.append(np.zeros((0, 128), np.uint8))
            continue
        n = int(rng.integers(700, 1400))
        n += n % 256 == 0
        d = syn.sift_like(rng, n)
        k = n // 2
        d[:k] = syn.perturb(rng, base[rng.choice(len(base), k, replace=False)])
        descs.append(d[rng.permutation(n)])
    return descs


@pytest.mark.parametrize("mode", [None, "full"])
def test_every_unit_has_candidates_equal_oracle(mode):
    rng = np.random.default_rng(23)
    descs = _images(rng)
    nf = [len(d) for d in descs]
    pairs = syn.exhaustive_pairs(len(descs))
    want = oracle.fast_match_pairs(np.concatenate(descs), nf, pairs)
    assert all(len(w) > 40 for w, (a, b) in zip(want, pairs) if nf[a] and nf[b])
    if mode is None:
        os.environ.pop("B2M_K1_DIR1", None)
    else:
        os.environ["B2M_K1_DIR1"] = mode
    try:
        c = pb.Context(device=0)
    finally:
        os.environ.pop("B2M_K1_DIR1", None)
    try:
        c.set_images(descs)
        for _ in range(2):   # the default context switches its column-direction schedule after the first call
            res = c.match_pairs(pairs)
            for k in range(len(pairs)):
                assert np.array_equal(res.matches(k), want[k]), (mode, k, tuple(pairs[k]))
            res.free()
    finally:
        c.close()
