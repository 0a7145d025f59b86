"""The half-warp DP fills one row per step and settles a row's left moves (EDIT_DELETE: a target column without a read
base) with a warp vote and a max-plus scan along the row.  The cases reach that code's edges: runs of 1-5 left moves in
one row, up to the band's edge; such runs in rows 1-6, where column 0 lies inside the band; ties between the three moves
(columns that match every base, 'N' read bases, homopolymers); pairs on one warp whose halves differ in length, or
where one half is idle; and lengths 1-13 (a matrix narrower than the band), 15-17, 191-193 and 511.  Against the
reference's GlobalAlignment_PosWeight: the edit string (w_dp_equal_half) and the side statistics of pairs (w_side_pair)."""
import numpy as np
import pytest

import parity_cases as pc
from test_gpu_extend import _side_stats
from trust4_b200 import api

pytestmark = pytest.mark.gpu

DELETE = 3


def _columns(rng, t, zero=()):
    """posWeight columns that support t[j] alone; the columns in `zero` are empty and match every base."""
    tw = np.zeros((len(t), 4), dtype=np.int32)
    for j, c in enumerate(t):
        if j not in zero:
            tw[j, c] = int(rng.integers(5, 30))
    return tw


def _read(p):
    return "".join("ACGTN"[c] for c in p)


def delete_runs(ed):
    """(row, length) of every run of EDIT_DELETE in an edit string; row = the read bases consumed before the run, i.e.
    the matrix row in which its left moves lie."""
    out, row, k = [], 0, 0
    while k < len(ed):
        if ed[k] == DELETE:
            s = k
            while k < len(ed) and ed[k] == DELETE:
                k += 1
            out.append((row, k - s))
        else:
            row += 1
            k += 1
    return out


def _left_run(ref, rng, L, row, width, zero=(), n_at=(), homopolymer=False, exact=True):
    """A target with `width` bases that the read lacks at `row`; the read makes up the length with its own bases 4 width + 8
    rows later (or at its end), so the best path takes `width` left moves in row `row` and returns to the diagonal.  Retried
    until the diagonal has more than 2 mismatches and (exact) the reference's edit string has exactly that run."""
    for _ in range(500):
        t = [int(c) for c in rng.integers(0, 4, size=L)]
        if homopolymer:
            t[row:row + width + 3] = [t[row]] * len(t[row:row + width + 3])
        p = t[:row] + t[row + width:]
        back = min(len(p), row + 4 * width + 8)
        p = p[:back] + [int(c) for c in rng.integers(0, 4, size=width)] + p[back:]
        for x in n_at:
            p[x] = 4
        tw, ps = _columns(rng, t, zero), _read(p)
        if pc._diag_mismatches(tw, ps) <= 2:
            continue
        if exact and (row, width) not in delete_runs(ref.dp_pos_weight(tw, ps)[1]):
            continue
        return tw, ps
    raise AssertionError("no case for", L, row, width)


def _unrelated(rng, L):
    """Unrelated bases; at lengths 1 and 2, which cannot have more than 2 diagonal mismatches, any bases (the banded
    DP's path is then the diagonal, the path of the reference's shortcut)."""
    while True:
        t = [int(c) for c in rng.integers(0, 4, size=L)]
        p = [int(c) for c in rng.integers(0, 4, size=L)]
        tw, ps = _columns(rng, t), _read(p)
        if L <= 2 or pc._diag_mismatches(tw, ps) > 2:
            return tw, ps


def row_cases(ref, seed=11):
    """(problem, (row, width) the reference's edit string must have a left-move run at, or None)."""
    rng = np.random.default_rng(seed)
    out = []
    # left moves deep inside the matrix, up to the band's edge (5), at both sides of a traceback word boundary
    for width in (1, 2, 3, 4, 5):
        for row in (9, 15, 16, 40):
            out.append((_left_run(ref, rng, 64, row, width), (row, width)))
    # rows 1-6, where column 0 is inside the band
    for width in (1, 2, 3, 5):
        for row in (1, 2, 3, 4, 5, 6):
            out.append((_left_run(ref, rng, 40, row, width), (row, width)))
    # ties of left, up and diagonal: columns that match every base, 'N' read bases, homopolymer runs
    for width in (2, 4):
        for row in (3, 20):
            out.append((_left_run(ref, rng, 48, row, width, zero=range(row, row + width + 2), exact=False), None))
            out.append((_left_run(ref, rng, 48, row, width, n_at=range(row, row + width + 2), exact=False), None))
            out.append((_left_run(ref, rng, 48, row, width, homopolymer=True, exact=False), None))
    tw, p = _left_run(ref, rng, 48, 10, 3, exact=False)
    tw[:] = 0
    out.append(((tw, "".join("N" if k % 3 == 0 else c for k, c in enumerate(p))), None))
    # lengths: narrower than the band, around one traceback word, around the shared-memory limit of 192, the longest read
    for L in list(range(1, 14)) + [15, 16, 17, 191, 192, 193, 511]:
        out.append((_unrelated(rng, L), None))
        if L >= 8:
            out.append((_left_run(ref, rng, L, L // 2 - 2, min(5, L // 4), exact=False), None))
    return out


def test_gpu_dp_rows_edit_strings(gpu_lib, ref):
    cases = row_cases(ref)
    probs = [c for c, _ in cases]
    refs = [ref.dp_pos_weight(tw, p) for tw, p in probs]
    for (_, want), (_, ed) in zip(cases, refs):
        assert want is None or want in delete_runs(ed), (want, delete_runs(ed))
    # chained left moves (the vote fires) in at least 40 problems, in rows 1-6 in at least 18
    chained = [[r for r, w in delete_runs(ed) if w >= 2] for _, ed in refs]
    assert sum(bool(c) for c in chained) >= 40 and sum(any(1 <= r <= 6 for r in c) for c in chained) >= 18
    got = api.dp_hot_path_batch(probs, 1, gpu_lib)
    for k, ((tw, p), g, r) in enumerate(zip(probs, got, refs)):
        assert g == r, (k, len(p), p, g, r)


def test_gpu_dp_rows_side_pairs(gpu_lib, ref):
    """The same problems as the two halves of one warp: next to an idle half (length 0), next to a half that ends long
    before or after it, and next to a half with left moves in other rows."""
    probs = [c for c, _ in row_cases(ref, 12)]
    empty = (np.zeros((0, 4), dtype=np.int32), "")
    rng = np.random.default_rng(13)
    short = [_unrelated(rng, L) for L in (1, 3, 5)]
    batches = [probs,
               [x for p in probs for x in (p, empty)],
               [x for p in probs for x in (empty, p)],
               [x for k, p in enumerate(probs) for x in (p, short[k % 3])],
               [x for k, p in enumerate(probs) for x in (short[k % 3], p)],
               probs[1:] + probs[:1],
               probs[::-1]]
    for batch in batches:
        got = api.dp_hot_path_batch(batch, 2, gpu_lib)
        for k, ((tw, p), st) in enumerate(zip(batch, got)):
            want = _side_stats(ref.dp_pos_weight(tw, p)[1], k % 2 == 0) if p else (0, 0, 0, 0)
            assert st == want, (k, len(p), p, st, want)
