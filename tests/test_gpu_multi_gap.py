"""Overlap scoring with two to five same-diagonal gaps in one overlap, each with > 2 mismatches (banded DP), with <= 2
(none) or with a frame shift (a path with indels, which fails the overlap), in every order.  Overlaps and similarity
doubles against the reference, and the number of gap DPs (counter 7): the gaps with > 2 mismatches, in hit order, up to
and including the first one whose path has an indel."""
import numpy as np
import pytest

import long_read_cases as lr
from parity_cases import _diag_mismatches

pytestmark = pytest.mark.gpu

K = 9
DP, FEW, SHIFT = "dp", "few", "shift"    # > 2 mismatches on the diagonal; <= 2 (no DP); a frame shift of 2 (indel path)
PLANS = [
    [DP, DP], [DP, DP, DP], [SHIFT, DP], [DP, SHIFT], [SHIFT, SHIFT], [DP, DP, SHIFT], [DP, SHIFT, DP], [SHIFT, DP, DP],
    [FEW, DP], [DP, FEW, DP], [FEW, SHIFT, DP], [DP, DP, DP, DP, SHIFT], [DP, DP, DP, DP, DP],
]
GAP = 34


def _build(lib, ref, seed, n_contigs=5):
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    g, r = lr._pair(lib, ref, K)
    core = list(lr._rand(rng, lr.EXT + lr.CORE + lr.EXT))
    laid = []
    for pl in PLANS:
        flank = max(30, (GAP * len(pl) + 12) // (len(pl) + 1) + 1)
        need = GAP * len(pl) + flank * (len(pl) + 1)
        assert need <= lr.CORE
        b0 = lr.EXT + int(rng.integers(0, lr.CORE - need + 1))
        spans = [(b0 + flank + j * (GAP + flank), b0 + flank + j * (GAP + flank) + GAP) for j in range(len(pl))]
        laid.append((b0, b0 + need, spans))
        for lo, hi in spans:                  # the columns next to the bordering hits may take an N: not A
            for q in (lo, hi - 1):
                if core[q] == "A":
                    core[q] = "CGT"[int(rng.integers(3))]
    core = "".join(core)
    for _ in range(n_contigs):
        a = int(rng.integers(1, 12))
        lr._input(g, r, lr._rand(rng, a) + core[lr.EXT:lr.EXT + lr.CORE] + lr._rand(rng, int(rng.integers(1, 13 - a))))
    reads = []
    for pl, (s, e, spans) in zip(PLANS, laid):
        ed = {}
        for kind, (lo, hi) in zip(pl, spans):
            b = lr.breaks(core, lo, hi, K - (2 if kind == SHIFT else 0), rng, True, True, kind == FEW)
            ed.update(b)
        rd = lr._apply(core, s, e, ed)
        for kind, (lo, hi) in zip(pl, spans):
            if kind == SHIFT:                 # two columns less early in the gap, two more late: the same diagonal on both sides
                x, y = lo - s + GAP // 3, hi - s - GAP // 3
                rd = rd[:x] + rd[x + 2:y] + lr._rand(rng, 2) + rd[y:]
        assert len(rd) == e - s
        reads.append(rd)
    return g, r, reads


@pytest.mark.parametrize("seed", [4, 5])
def test_gpu_multi_gap(gpu_lib, ref, seed):
    g, r, reads = _build(gpu_lib, ref, seed)
    n_contigs = r.size()
    seen = set()
    before = int(lr.counters(gpu_lib)[7])     # the counters run on from one call to the next
    for i, (pl, rd) in enumerate(zip(PLANS, reads)):
        n, o, sim = lr._same_overlaps(g, r, rd, tag=(i, pl))
        after = int(lr.counters(gpu_lib)[7])
        got, before = after - before, after
        want, failed = 0, []
        for idx in range(n_contigs):
            gaps = [x for x in lr._contig_gaps(r, rd, K)[(idx, 1)] if x[0] >= 2]
            assert len(gaps) == len(pl), (i, idx, gaps)
            pw = r.get_contig(idx)["pos_weight"]
            fail, kinds = False, []
            for gap, a, b in gaps:
                cols, bases = pw[b:b + gap], rd[a:a + gap]
                dp = _diag_mismatches(cols, bases) > 2
                indel = dp and any(e > 1 for e in ref.dp_pos_weight(cols, bases)[1])
                kinds.append(SHIFT if indel else DP if dp else FEW)
                if not fail:
                    want += dp
                    fail = indel
            failed.append(fail)
            seen.add(tuple(kinds))
        assert got == want, ("gap DPs", i, pl, got, want)
        if all(failed):
            assert n <= 0 or (sim == 0).all(), (i, pl, sim)
        elif not any(failed):
            assert n == n_contigs and (sim > 0).all(), (i, pl, n, sim)
    for pl in PLANS:                          # the reads are what the plans say
        assert tuple(pl) in seen, ("no overlap with the gaps", pl, sorted(seen))
