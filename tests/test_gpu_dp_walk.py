"""The half-warp DP's traceback at its edges: the actions of a slot are packed 16 rows to a word, so the cases put indels
on both sides of the word boundaries, two in one word, at the first and the last step of the path and where the path
meets row 0 or column 0 off the corner, next to all-diagonal paths of one or two whole words and one row more or less,
on both sides of the 192-column limit of the shared-memory buffers.  Against the reference's
GlobalAlignment_PosWeight: the edit string (w_dp_equal_half) and the side statistics of pairs (w_side_pair)."""
import numpy as np
import pytest

import parity_cases as pc
from test_gpu_extend import _side_stats
from trust4_b200 import api

pytestmark = pytest.mark.gpu


def _problem(rng, t, p):
    """Columns that support t[j] alone against the read p (same length); more than 2 diagonal mismatches, so that the
    callers of the warp DP would run it."""
    tw = np.zeros((len(t), 4), dtype=np.int32)
    for j, c in enumerate(t):
        tw[j, c] = int(rng.integers(5, 30))
    ps = "".join("ACGT"[c] for c in p)
    assert len(p) == len(t) and pc._diag_mismatches(tw, ps) > 2, (len(t), ps)
    return tw, ps


def _shifted(rng, L, row, width=1, back=None, subs=()):
    """A read that lacks `width` bases of the target from `row` on and has `width` bases of its own before `back`
    (default: its end): the best path leaves the diagonal at row `row` and returns to it at `back`."""
    while True:
        t = [int(c) for c in rng.integers(0, 4, size=L)]
        p = list(t)
        del p[row:row + width]
        at = len(p) if back is None else back - width
        for _ in range(width):
            p.insert(at, int(rng.integers(4)))
        for x in subs:
            p[x] = (p[x] + 1) % 4
        tw = np.zeros((L, 4), dtype=np.int32)
        for j, c in enumerate(t):
            tw[j, c] = 9
        if pc._diag_mismatches(tw, "".join("ACGT"[c] for c in p)) > 2:
            return _problem(rng, t, p)


def _substituted(rng, L, at):
    t = [int(c) for c in rng.integers(0, 4, size=L)]
    p = list(t)
    for x in at:
        p[x] = (p[x] + 1) % 4
    return _problem(rng, t, p)


def walk_cases(seed=7):
    rng = np.random.default_rng(seed)
    out = []
    # an indel at each side of the boundaries of the 16-row traceback words, the path back on the diagonal 8 rows on
    for row in (14, 15, 16, 17, 30, 31, 32, 33, 47, 48, 49):
        for width in (1, 2):
            out.append(_shifted(rng, 80, row, width, back=row + 8 + width))
    # two departures inside one word, and two words apart
    for row in (18, 34):
        out.append(_shifted(rng, 90, row, 1, back=row + 4, subs=(60, 70, 80)))
    # an indel as the first and as the last step of the path; frames that meet row 0 / column 0 off the corner
    for width in (1, 2, 3, 4, 5):
        out.append(_shifted(rng, 40 + width, 0, width))
        t = [int(c) for c in rng.integers(0, 4, size=60)]
        own = [int(c) for c in rng.integers(0, 4, size=width)]
        out.append(_problem(rng, t, own + t[:-width]))
        out.append(_problem(rng, t, t[width:] + own))
    # all-diagonal paths of exactly 15, 16, 17, 31, 32, 33 rows (one or two whole words and one row more or less)
    for L in (15, 16, 17, 31, 32, 33, 48):
        out.append(_substituted(rng, L, (0, L // 2, L - 1)))
        out.append(_substituted(rng, L, (1, 2, 3, L - 2)))
    # on both sides of the 192 columns up to which edit string and traceback words stay in shared memory
    for L in (190, 191, 192, 193, 300, 511):
        out.append(_shifted(rng, L, L // 3, 2, back=L // 3 + 20))
        out.append(_shifted(rng, L, 16, 1))
        out.append(_substituted(rng, L, (0, 15, 16, L - 1)))
    return out


def test_gpu_dp_walk_edit_strings(gpu_lib, ref):
    cases = walk_cases()
    got = api.dp_hot_path_batch(cases, 1, gpu_lib)
    indels = 0
    for k, ((tw, p), (sc, ed)) in enumerate(zip(cases, got)):
        rs, re_ = ref.dp_pos_weight(tw, p)
        assert (sc, ed) == (rs, re_), (k, len(p), p, sc, rs, ed, re_)
        indels += any(e > 1 for e in re_)
    assert indels > len(cases) // 3, indels


def test_gpu_dp_walk_side_pairs(gpu_lib, ref):
    """The same problems as the two sides of half-warp pairs, in both assignments to the halves (a left side is read from
    its end), and with an odd one out."""
    cases = walk_cases(8)
    for batch in (cases, cases[1:] + cases[:1], cases[:-1][::-1]):
        got = api.dp_hot_path_batch(batch, 2, gpu_lib)
        for k, ((tw, p), st) in enumerate(zip(batch, got)):
            ed = ref.dp_pos_weight(tw, p)[1]
            assert st == _side_stats(ed, k % 2 == 0), (k, len(p), p, st, ed)
