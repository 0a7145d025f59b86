"""ExtendOverlap's overhang pass in the stream kernel: the half-warp pair routine (w_side_pair) against the reference's
GlobalAlignment_PosWeight, and noisy batches whose reads take every route of the pass (deferred DPs of non-easy reads,
the sides the bridging loop needs, the on-demand fallback of the decision loop) against the reference."""
import numpy as np
import pytest

import parity_cases as pc
from trust4_b200 import api, synth


def _side_stats(ed, from_end):
    """What ExtendOverlap takes from one overhang's edit string (SeqSet.hpp:1176-1224): match / mismatch / indel counts
    and the longest prefix (seen from the anchor) of match/mismatch ops whose running match fraction exceeds 0.75."""
    m, x = ed.count(0), ed.count(1)
    good, tm = 0, 0
    for kk, e in enumerate(ed[::-1] if from_end else ed):
        if e == 0:
            tm += 1
            if tm > 0.75 * (kk + 1):
                good = kk + 1
        elif e != 1:
            break
    return (m, x, len(ed) - m - x, good)


def _overhang(rng, L):
    """One overhang as the stream kernel aligns it: > 2 diagonal mismatches (substitutions, an in-band frame shift,
    unrelated bases, N's), so the banded DP runs; at length 2, which can never have more, any bases."""
    while True:
        t = rng.integers(0, 4, size=L)
        p = list(t)
        kind = int(rng.integers(0, 4))
        if kind == 0:
            for _ in range(int(rng.integers(3, 4 + L // 8))):
                y = int(rng.integers(L))
                p[y] = (p[y] + 1 + int(rng.integers(3))) % 4
        elif kind == 1 and L > 12:
            d = int(rng.integers(1, 5))
            y = int(rng.integers(1, L - d - 4))
            del p[y:y + d]
            z = int(rng.integers(y + 1, len(p)))
            for _ in range(d):
                p.insert(z, int(rng.integers(4)))
        elif kind == 2:
            p = list(rng.integers(0, 4, size=L))
        else:
            for _ in range(int(rng.integers(1, 4))):
                p[int(rng.integers(L))] = 4
            for _ in range(int(rng.integers(3, 9))):
                p[int(rng.integers(L))] = int(rng.integers(4))
        tw = np.zeros((L, 4), dtype=np.int32)
        for j in range(L):
            tw[j, t[j]] = int(rng.integers(1, 30))
            if rng.random() < 0.3:
                tw[j, int(rng.integers(4))] += int(rng.integers(0, 12))
            if rng.random() < 0.03:
                tw[j] = 0
        ps = "".join("ACGTN"[c] for c in p)
        if L == 2 or pc._diag_mismatches(tw, ps) > 2:
            return tw, ps


def _empty_or_one(rng, L):
    tw = np.zeros((L, 4), dtype=np.int32)
    if L:
        tw[0, int(rng.integers(4))] = int(rng.integers(1, 30))
    return tw, "".join("ACGTN"[int(c)] for c in rng.integers(0, 5, size=L))


def side_pair_cases(seed, n_pairs=240):
    """Pairs (left side, right side) of unequal lengths 2..511 on both sides of the 192-column shared-memory limit,
    every third pair with one side of length 0 or 1 (the other half-warp idles or runs a one-cell DP)."""
    rng = np.random.default_rng(seed)
    lens = [2, 3, 7, 13, 64, 150, 190, 191, 192, 193, 250, 300, 400, 510, 511]
    out = []
    for i in range(n_pairs):
        a = int(rng.choice(lens)) if i % 2 else int(rng.integers(2, 512))
        if i % 3 == 0:
            b = int(rng.integers(0, 2))
            pair = [_overhang(rng, a), _empty_or_one(rng, b)]
        else:
            b = a
            while b == a:
                b = int(rng.choice(lens)) if i % 2 == 0 else int(rng.integers(2, 512))
            pair = [_overhang(rng, a), _overhang(rng, b)]
        if rng.random() < 0.5:
            pair.reverse()
        out += pair
    return out


@pytest.mark.gpu
def test_gpu_dp_hot_path_side_pair(gpu_lib, ref):
    """w_side_pair -- two overhang sides per warp, one per half-warp, as the stream kernel's ExtendOverlap pass runs
    them -- each side's statistics vs the reference's GlobalAlignment_PosWeight edit string (left sides from their end)."""
    for seed in (31, 32):
        cases = side_pair_cases(seed)
        got = api.dp_hot_path_batch(cases, 2, gpu_lib)
        for k, ((tw, p), st) in enumerate(zip(cases, got)):
            ed = ref.dp_pos_weight(tw, p)[1] if len(p) else []
            assert st == _side_stats(ed, k % 2 == 0), (seed, k, len(p), p, st, ed)
    # an odd number of problems: the last warp runs one side
    cases = side_pair_cases(33, 3)[:5]
    got = api.dp_hot_path_batch(cases, 2, gpu_lib)
    for k, ((tw, p), st) in enumerate(zip(cases, got)):
        ed = ref.dp_pos_weight(tw, p)[1] if len(p) else []
        assert st == _side_stats(ed, k % 2 == 0)


def _noisy_batch(lib, ref, seed, sub_rate, n_shards):
    """A batch of reads with sub_rate substitutions against the reference, per shard; returns the run's counters."""
    lib.check(lib.reset())
    cl = synth.make_clones(60, seed)
    w = synth.build_workload(cl, synth.sample_pairs(cl, 2500, 150, seed, sub_rate=sub_rate))
    cfg = synth.run_cfg()
    off, descs = synth.shard_workload(w, n_shards)
    sets = api.SeqSet.create_many(n_shards, 9, lib)
    ret, strands, resc = api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    c = np.zeros(api.N_COUNTERS, dtype=np.uint64)
    lib.check(lib.last_counters(c.ctypes.data))
    for j in range(n_shards):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(9)
        _, rret, rstr, rresc = r.run_descs(cfg, descs[lo:hi].copy(), w.pool, w.names)
        assert (rret == ret[lo:hi]).all(), ("ret", j, np.flatnonzero(rret != ret[lo:hi])[:5])
        assert (rstr == strands[lo:hi]).all(), ("strand", j)
        assert (rresc == resc[lo:hi]).all(), ("rescue", j)
        assert r.output() == sets[j].output(), ("contigs", j)
        assert r.index_checksum() == sets[j].index_checksum(), ("index", j)
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("seed,sub_rate", [(96, 0.04), (97, 0.04)])
def test_gpu_extend_noisy_batch(gpu_lib, ref, seed, sub_rate):
    """Noisy reads: overhang DPs ran in the parallel pass (counter 1), some reads were not easy (counter 20 below the
    reads, counter 0), and the decision loop made at least one overlap exact on demand (counter 21)."""
    c = _noisy_batch(gpu_lib, ref, seed, sub_rate, 6)
    assert c[1] > 1000 and c[20] < c[0] and c[21] > 0, c.tolist()


def test_emu_extend_noisy_batch(emu_lib, ref):
    """The same batch through the emulation's one-side-at-a-time form of the pass."""
    c = _noisy_batch(emu_lib, ref, 96, 0.04, 6)
    assert c[1] > 1000 and c[21] > 0, c.tolist()
