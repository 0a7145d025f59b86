"""The main hit sort of GetOverlapsFromRead and its chain pass on the device.

The device sorts a read's hit keys stably on their (strand | contig | diagonal) prefix only, in a shared-memory tile up
to T4_HIT_TILE keys and in global memory above it, and finds group and run heads in one neighbour-compare pass.  The
hook t4_test_group_hits runs both on keys given in the probe's emission order; every case is checked against numpy's
sort of the whole 64-bit keys.  The overlap cases build sets whose reads reach the tile's edge, the `filter == 1`
pre-pass with more than 100 and more than 1000 possible groups, runs of one-hit groups (the pre-pass's skip quirk) and
the path of k-mers with more than 10 000 postings, and compare GetOverlapsFromRead with the reference."""
import numpy as np
import pytest

from trust4_b200 import api

pytestmark = pytest.mark.gpu

TILE = 512                       # T4_HIT_TILE of the build
INVALID = np.uint64(0xFFFFFFFFFFFFFFFF)
BIAS = 1 << 20
B_MAX = (1 << 19) - 1
IDX_MAX = (1 << 22) - 1


def key(strand, idx, q, off, rep=0):
    return (int(strand == 1) << 63) | (idx << 41) | ((q - off + BIAS) << 20) | (off << 1) | rep


def emit(rng, n, strands=(1, -1), idx_lo=0, idx_hi=40, off_lo=0, off_hi=2000, rep_frac=0.0):
    """n keys in the order c_get_hits emits them for one read: pass 0 (strand +1) then pass 1, ascending q < 512, one
    position's postings distinct (contig, offset) pairs."""
    top = 2 * (n // (512 * len(strands))) + 2
    out = []
    for s in strands:
        for q in range(512):
            seen = set()
            for _ in range(int(rng.integers(1, top + 1))):
                p = (int(rng.integers(idx_lo, idx_hi + 1)), int(rng.integers(off_lo, off_hi + 1)))
                if p not in seen:
                    seen.add(p)
                    out.append(key(s, p[0], q, p[1], int(rng.random() < rep_frac)))
    assert len(out) >= n
    return np.array(out[:n], dtype=np.uint64)


def expected_heads(sorted_keys):
    v = sorted_keys[sorted_keys != INVALID]
    n = len(v)
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), n
    g = np.flatnonzero(np.r_[True, (v[1:] >> np.uint64(41)) != (v[:-1] >> np.uint64(41))])
    r = np.flatnonzero(np.r_[True, (v[1:] >> np.uint64(20)) != (v[:-1] >> np.uint64(20))])
    return g, r, n


def check(lib, s, keys):
    got, grp, run = s.group_hits(keys)
    want = np.sort(keys)
    assert (got == want).all(), ("order", len(keys), int(np.flatnonzero(got != want)[0]))
    g, r, n = expected_heads(want)
    assert (grp[:-1] == g).all() and grp[-1] == n, ("group heads", len(keys))
    assert (run[:-1] == r).all() and run[-1] == n, ("run heads", len(keys))


@pytest.fixture(scope="module")
def hook_set(gpu_lib):
    gpu_lib.check(gpu_lib.reset())
    s = api.SeqSet(9, gpu_lib)
    yield s


@pytest.mark.parametrize("n", [0, 1, 2, 1023, 1024, 1025, TILE - 1, TILE, TILE + 1, 2 * TILE + 1, 12001])
def test_sort_sizes(gpu_lib, hook_set, n):
    rng = np.random.default_rng(n)
    check(gpu_lib, hook_set, emit(rng, n, rep_frac=0.1))


@pytest.mark.parametrize("n", [700, TILE, 5000])
def test_trailing_invalid_keys(gpu_lib, hook_set, n):
    rng = np.random.default_rng(100 + n)
    keys = emit(rng, n)
    keys[rng.random(n) < 0.3] = INVALID          # the barcode filter's keys, anywhere in emission order
    check(gpu_lib, hook_set, keys)
    keys[:] = INVALID
    check(gpu_lib, hook_set, keys)


@pytest.mark.parametrize("n", [900, TILE + 1])
def test_field_edges(gpu_lib, hook_set, n):
    """contig indices up to 2^22 - 1 and diagonals at both ends (offsets 0 and 2^19 - 1 against q up to 511): a
    varying span of more than 32 bits, both strands, repeat flags."""
    rng = np.random.default_rng(200 + n)
    a = emit(rng, n // 2, idx_lo=IDX_MAX - 3, idx_hi=IDX_MAX, off_lo=B_MAX - 50, off_hi=B_MAX, rep_frac=0.5)
    b = emit(rng, n - n // 2, idx_lo=0, idx_hi=3, off_lo=0, off_hi=50, rep_frac=0.5)
    # emission order of one read: merge the two by (pass, q)
    both = np.concatenate([a, b])
    strand_first = np.where((both >> np.uint64(63)) == 1, 0, 1)
    q = (((both >> np.uint64(20)) & np.uint64((1 << 21) - 1)).astype(np.int64) - BIAS) + ((both >> np.uint64(1)) & np.uint64(B_MAX)).astype(np.int64)
    order = np.lexsort((np.arange(len(both)), q, strand_first))
    keys = both[order]
    assert (keys >> np.uint64(20)).max() - (keys >> np.uint64(20)).min() > (1 << 32)
    check(gpu_lib, hook_set, keys)


@pytest.mark.parametrize("n", [64, 1000])
def test_one_bit_span(gpu_lib, hook_set, n):
    """one strand, one contig, two diagonals that differ in the lowest bit of the diagonal field only"""
    keys = np.array([key(1, 7, q, q - 10 - d) for q in range(10, 512) for d in (0, 1) if q - 10 - d >= 0][:n], np.uint64)
    vary = np.bitwise_or.reduce(keys >> np.uint64(20)) ^ np.bitwise_and.reduce(keys >> np.uint64(20))
    assert int(vary) == 1
    check(gpu_lib, hook_set, keys)


# ---- GetOverlapsFromRead against the reference -------------------------------------------------------------------

def _rand_seq(rng, n):
    return "".join("ACGT"[x] for x in rng.integers(0, 4, n))


def _build(ref, lib, contigs):
    lib.check(lib.reset())
    g = api.SeqSet(9, lib)
    r = ref.RefSeqSet(9)
    for i, c in enumerate(contigs):
        for s in (g, r):
            s.input_novel_read("TRBV%d" % (i % 7), c, 1, -1)
    return g, r


def _compare(g, r, read):
    hr = r.get_hits(read, 0)
    hg = g.get_hits(read, 0)
    assert len(hr) == len(hg)
    for sk in (False, True):
        n1, o1, s1 = r.get_overlaps(read, 0, -1, sk)
        n2, o2, s2 = g.get_overlaps(read, 0, -1, sk)
        assert n1 == n2, ("overlap count", sk, n1, n2)
        if n1 > 0:
            assert (o1 == o2).all(), ("overlaps", sk)
            assert (s1 == s2).all(), ("similarity", sk)
    return len(hg)


def _windows(rng, read, n_contigs, w, flank=30):
    out = []
    for j in range(n_contigs):
        s = int(rng.integers(0, len(read) - w + 1))
        out.append(_rand_seq(rng, flank) + read[s:s + w] + _rand_seq(rng, flank))
    return out


@pytest.mark.parametrize("n_contigs,w,lo,hi", [(70, 40, 1200, 3500),      # H beyond the tile
                                               (160, 40, 3000, 12000),    # > 100 possible groups
                                               (1100, 24, 1, 10 ** 7)])   # > 1000 possible groups
def test_overlaps_many_groups(gpu_lib, ref, n_contigs, w, lo, hi):
    rng = np.random.default_rng(n_contigs)
    read = _rand_seq(rng, 150)
    contigs = _windows(rng, read, n_contigs, w) + [read[:120] + _rand_seq(rng, 40)]
    g, r = _build(ref, gpu_lib, contigs)
    h = _compare(g, r, read)
    assert lo <= h <= hi, h


def test_overlaps_one_hit_groups(gpu_lib, ref):
    """runs of contigs that share one k-mer with the read (groups of one hit) between longer groups: the pre-pass
    enters a group at its first or second hit, or skips it"""
    rng = np.random.default_rng(7)
    read = _rand_seq(rng, 150)
    contigs = []
    for j in range(400):
        if j % 5 == 4:
            contigs += _windows(rng, read, 1, 60)
        else:
            s = int(rng.integers(0, 141))
            contigs.append(_rand_seq(rng, 30) + read[s:s + 9] + _rand_seq(rng, 30))
    g, r = _build(ref, gpu_lib, contigs)
    _compare(g, r, read)


def test_overlaps_big_repeat(gpu_lib, ref):
    """a k-mer with more than 10 000 postings: GetOverlapsFromHits consults the SortHits-order copy"""
    rng = np.random.default_rng(11)
    read = _rand_seq(rng, 150)
    rep = read[50:59]
    contigs = [_rand_seq(rng, 20) + rep + _rand_seq(rng, 20) for _ in range(10050)]
    contigs += _windows(rng, read, 30, 50)
    g, r = _build(ref, gpu_lib, contigs)
    _compare(g, r, read)
