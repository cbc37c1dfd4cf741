"""Shared checks of the SIFT tests: pairing of two feature lists (GPU against oracle, or an image against its
transpose) keypoint by keypoint, with the oracle's decision margins to excuse what rounding can flip."""
import math

import numpy as np

# UBC layout, transposed image: cell (by, bx) -> (3 - by, bx) and orientation bin u -> (8 - u) mod 8
TRANSPOSE_PERM = np.array([8 * ((3 - by) * 4 + bx) + (8 - u) % 8 for by in range(4) for bx in range(4) for u in range(8)])


def groups(kp):
    """[start, end) row runs of one keypoint (its orientations are consecutive and share x, y)."""
    if not len(kp):
        return []
    starts = [0] + [i for i in range(1, len(kp)) if kp[i, 0] != kp[i - 1, 0] or kp[i, 1] != kp[i - 1, 1]]
    return list(zip(starts, starts[1:] + [len(kp)]))


def wrap(a):
    return (a + math.pi) % (2 * math.pi) - math.pi
