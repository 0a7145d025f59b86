"""Shared checks of the per-cell (--barcode) pre-processing: t4_barcode_kmer_count_stats against the reference's
barcode-wise KmerCount loop (main.cpp:1128-1153) and t4_sort_reads_barcode against std::sort with CompReadWithBarcode
(main.cpp:128-136).  Used by test_gpu_barcode_stats.py (libtrust4_b200.so) and test_emu_barcode_stats.py (the emulation)."""
import numpy as np

from trust4_b200 import api, synth
from parity_cases import _check_sorted_records, _ref_sort_bytes, reads_pool

BC21 = 1 << 21
BC_TOP = (1 << 31) - 1


def barcode_groups(bc):
    """Index arrays of the reads of every barcode, in barcode order (each in the reads' order)."""
    bc = np.asarray(bc, dtype=np.int64)
    g = np.argsort(bc, kind="stable")
    cuts = np.flatnonzero(np.diff(bc[g])) + 1
    return np.split(g, cuts) if len(g) else []


def ref_bc_stats(ref, pool, off, lens, bc, k=21):
    """The driver's barcode-wise loop (main.cpp:1129-1153) over the compiled reference: for every barcode a fresh
    KmerCount( k ) -- the same as the driver's KmerCount( 21, 23 ) after Clear(): the second argument only sets how many
    std::maps share the keys -- gets AddCount of the barcode's reads, then GetCountStatsAndTrim( read, NULL, ... ) of each
    (t4ref_kmer_count_stats on that group alone)."""
    n = len(lens)
    off = np.asarray(off, dtype=np.uint64)
    lens = np.asarray(lens, dtype=np.int32)
    out = [np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)]
    for g in barcode_groups(bc):
        mn, med, avg, _ = ref.kmer_count_stats(pool, off[g], lens[g], k)
        out[0][g], out[1][g], out[2][g] = mn, med, avg
    return out


def check_bc_stats(lib, ref, reads, bc, k=21):
    """Per read, barcodeMinCnt / barcodeMedianCnt equal and barcodeAvgCnt the same float bits as the reference's."""
    pool, off, lens = reads_pool(reads)
    bc = np.asarray(bc, dtype=np.int32)
    gmn, gmed, gavg = api.barcode_kmer_count_stats(pool, off, lens, bc, k, lib)
    rmn, rmed, ravg = ref_bc_stats(ref, pool, off, lens, bc, k)
    assert (gmn == rmn).all(), ("min", np.flatnonzero(gmn != rmn)[:5])
    assert (gmed == rmed).all(), ("median", np.flatnonzero(gmed != rmed)[:5])
    assert (gavg.view(np.uint32) == ravg.view(np.uint32)).all(), ("avg", np.flatnonzero(gavg.view(np.uint32) != ravg.view(np.uint32))[:5])
    return gmn, gmed, gavg


def cell_reads(seed, n_cells, reads_per_cell, L=150):
    """configs[3]-style cells (synth.sample_single_cell) with ragged sizes: every cell keeps a random 20..100 % of its reads.
    Returns (reads as bytes, barcode ids 0..n_cells-1), grouped by barcode."""
    rng = np.random.default_rng(seed)
    cl = synth.make_clones(max(20, n_cells // 2), seed)
    rd, bc = synth.sample_single_cell(cl, n_cells, reads_per_cell, L, seed)
    keep = rng.random(len(bc)) < rng.uniform(0.2, 1.0, size=n_cells)[bc]
    pool = np.frombuffer(b"ACGT", dtype=np.uint8)[rd.codes[keep]]
    return [r.tobytes() for r in pool], bc[keep].astype(np.int32)


def case_many_cells(seed=201, n_cells=250, reads_per_cell=240):
    return cell_reads(seed, n_cells, reads_per_cell)


def case_random_order(seed=202):
    reads, bc = cell_reads(seed, 120, 200)
    p = np.random.default_rng(seed).permutation(len(reads))
    return [reads[i] for i in p], bc[p]


def case_one_cell(seed=203):
    reads, bc = cell_reads(seed, 40, 150)
    return reads, np.full(len(reads), 5, dtype=np.int32)


def case_single_read_cells(seed=204):
    reads, bc = cell_reads(seed, 30, 100)
    reads = reads[:600]
    return reads, (np.arange(len(reads), dtype=np.int64) * 3 + 1).astype(np.int32)


def case_shared_reads(seed=205):
    """The same read strings in two cells, one of them holding extra copies: counts of one cell must not leak into the other."""
    reads, bc = cell_reads(seed, 6, 300)
    a = [r for r, b in zip(reads, bc) if b == 0]
    c = [r for r, b in zip(reads, bc) if b == 1]
    rr = a + a + a[: len(a) // 2] + c
    bb = [10] * len(a) + [11] * len(a) + [11] * (len(a) // 2) + [12] * len(c)
    return rr, np.array(bb, dtype=np.int32)


def case_wide_barcodes(seed=206):
    """Barcode ids on both sides of 2^21 and near 2^31 - 1 in one call; cells whose ids agree in the low 21 bits hold the
    same reads in different numbers, so a key that kept only 21 barcode bits, or none, would merge them."""
    reads, bc = cell_reads(seed, 8, 200)
    groups = [[r for r, b in zip(reads, bc) if b == j] for j in range(4)]
    ids = [(0, 0), (1, 1), (BC21 - 1, 2), (BC21, 0), (BC21 + 1, 1), (BC_TOP - 1, 3), (BC_TOP, 2), (BC21 * 700 + 1, 1), (2 * BC21 + 1, 3)]
    rr, bb = [], []
    for j, (b, g) in enumerate(ids):
        take = groups[g][: len(groups[g]) * (j % 3 + 1) // 3] or groups[g]
        rr += take
        bb += [b] * len(take)
    p = np.random.default_rng(seed).permutation(len(rr))
    return [rr[i] for i in p], np.array(bb, dtype=np.int64)[p].astype(np.int32)


def case_ragged(seed=207):
    """N's, reads shorter than 21, reads of exactly 512 bp, reads of N's only, homopolymers; a few cells."""
    rng = np.random.default_rng(seed)

    def rnd(L):
        return bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=L))

    src = [rnd(600) for _ in range(6)]
    reads, bc = [], []
    for i in range(3000):
        s = src[int(rng.integers(len(src)))]
        kind = int(rng.integers(0, 7))
        L = int(rng.integers(1, 513))
        st = int(rng.integers(0, 600 - L + 1))
        t = bytearray(s[st:st + L])
        if kind == 0:
            t = bytearray(b"N" * L)
        elif kind == 1:
            t = bytearray(s[:20 - int(rng.integers(0, 15))])
        elif kind == 2:
            t = bytearray(s[int(rng.integers(0, 88)):][:512])
        elif kind == 3:
            for p in rng.integers(0, len(t), size=int(rng.integers(1, 6))):
                t[int(p)] = ord("N")
        elif kind == 4:
            t = bytearray(b"ACGT"[int(rng.integers(4)):][:1] * L)
        reads.append(bytes(t))
        bc.append(int(rng.integers(0, 12)))
    assert max(len(r) for r in reads) == 512
    return reads, np.array(bc, dtype=np.int32)


STATS_CASES = {"many_cells": case_many_cells, "random_order": case_random_order, "one_cell": case_one_cell,
               "single_read_cells": case_single_read_cells, "shared_reads": case_shared_reads, "wide_barcodes": case_wide_barcodes,
               "ragged": case_ragged}


def check_stats_case(lib, ref, name):
    reads, bc = STATS_CASES[name]()
    mn, med, avg = check_bc_stats(lib, ref, reads, bc)
    if name == "shared_reads":
        # the copies in cell 11 see higher counts than the same strings in cell 10
        n10 = int((bc == 10).sum())
        assert (med[n10: 2 * n10] > med[:n10]).any()
    if name == "ragged":
        assert (mn < 0).sum() > 10 and (mn == 0).sum() > 10
    return len(reads)


def bc_key(reads, ids, mn, med, avg, bc, bmin):
    """CompReadWithBarcode (main.cpp:128-136) for barcodes >= 0 as a Python key: barcode ascending, barcodeMinCnt
    descending, then _sortRead::operator< (parity_cases.sort_key)."""
    return lambda i: (int(bc[i]), -int(bmin[i]), -int(mn[i]), -int(med[i]), -float(avg[i]), -len(reads[i]), reads[i], ids[i])


def _ref_sort_bc(ref, reads, ids, mn, med, avg, bc, bmin):
    """std::sort with CompReadWithBarcode (main.cpp:128-136) for barcodes >= 0: the records ordered by (barcode ascending,
    barcodeMinCnt descending) and, within each such group, by the reference's own std::sort under _sortRead::operator<
    (t4ref_sort_reads) -- for barcodes >= 0 the comparator is exactly that lexicographic order."""
    bc = np.asarray(bc, dtype=np.int64)
    bmin = np.asarray(bmin, dtype=np.int64)
    g = np.lexsort((-bmin, bc))
    cuts = np.flatnonzero((np.diff(bc[g]) != 0) | (np.diff(bmin[g]) != 0)) + 1
    order = []
    for grp in np.split(g, cuts):
        sub = _ref_sort_bytes(ref, [reads[i] for i in grp], [ids[i] for i in grp], np.asarray(mn)[grp], np.asarray(med)[grp],
                              np.asarray(avg)[grp])
        order.extend(grp[sub].tolist())
    return np.array(order, dtype=np.int64)


def sort_records(lib, seed, reads, bc):
    """Records with their real global and per-cell statistics, half of them coarsened so that many cells share a
    barcodeMinCnt and long runs tie on the counts; mates share an id; a tenth of the records are exact copies."""
    rng = np.random.default_rng(seed)
    pool, off, lens = reads_pool(reads)
    mn, med, avg, _ = api.kmer_count_stats(pool, off, lens, 21, lib)
    bmin, _, _ = api.barcode_kmer_count_stats(pool, off, lens, bc, 21, lib)
    n = len(reads)
    coarse = rng.random(n) < 0.5
    mn = np.where(coarse, np.minimum(mn, 2), mn).astype(np.int32)
    med = np.where(coarse, np.minimum(med, 3), med).astype(np.int32)
    avg = np.where(coarse, np.float32(2.5), avg).astype(np.float32)
    bmin = np.where(rng.random(n) < 0.5, np.minimum(bmin, 1), bmin).astype(np.int32)
    ids = [b"r%d" % (i // 2) for i in range(n)]
    reads, ids, bc = list(reads), list(ids), np.asarray(bc, dtype=np.int32).copy()
    dup = rng.integers(0, n, size=n // 10)
    reads += [reads[j] for j in dup]
    ids += [ids[j] for j in dup]
    mn, med, avg = np.r_[mn, mn[dup]], np.r_[med, med[dup]], np.r_[avg, avg[dup]]
    bc, bmin = np.r_[bc, bc[dup]], np.r_[bmin, bmin[dup]]
    p = rng.permutation(len(reads))
    return ([reads[i] for i in p], [ids[i] for i in p], mn[p].astype(np.int32), med[p].astype(np.int32), avg[p].astype(np.float32),
            bc[p].astype(np.int32), bmin[p].astype(np.int32))


def check_sort_barcode(lib, ref, seed=211):
    """t4_sort_reads_barcode against the reference's std::sort with CompReadWithBarcode and the Python key."""
    reads, bc = cell_reads(seed, 150, 120)
    wide = np.where(np.random.default_rng(seed).random(len(bc)) < 0.3, bc + BC21, bc).astype(np.int32)   # some ids above 2^21
    reads, ids, mn, med, avg, bc, bmin = sort_records(lib, seed, reads, wide)
    pool, off, lens = reads_pool(reads)
    go = api.sort_reads_barcode(pool, off, lens, ids, mn, med, avg, bc, bmin, lib)
    key = bc_key(reads, ids, mn.tolist(), med.tolist(), avg.tolist(), bc.tolist(), bmin.tolist())
    keys = [key(i) for i in range(len(reads))]
    _check_sorted_records(go, keys, _ref_sort_bc(ref, reads, ids, mn, med, avg, bc, bmin))
    want = sorted(range(len(reads)), key=keys.__getitem__)
    _check_sorted_records(go, keys, want)
    # cells with equal barcodeMinCnt, and records that tie under the comparator, really occur
    assert sum(1 for a, b in zip(want, want[1:]) if keys[a][:2] == keys[b][:2]) > len(reads) // 2
    assert sum(1 for a, b in zip(want, want[1:]) if keys[a] == keys[b]) > 10
    return len(reads)


def check_sort_barcode_large(lib, seed=213, n=(1 << 20) + 3):
    """t4_sort_reads_barcode at 2^20 + 3 records (the grid-stride loop turns more than once) against the Python key: 4000
    cells, per-cell statistics coarsened into few values, duplicated records."""
    rng = np.random.default_rng(seed)
    cl = synth.make_clones(400, seed)
    rd, bc = synth.sample_single_cell(cl, 4000, (n + 3999) // 4000, 150, seed)
    L = rd.codes.shape[1]
    pool = np.concatenate([np.frombuffer(b"ACGT", dtype=np.uint8)[rd.codes[:n]].reshape(-1), np.zeros(16, dtype=np.uint8)])
    off = np.arange(n, dtype=np.uint64) * np.uint64(L)
    lens = np.where(rng.random(n) < 0.3, rng.integers(20, L + 1, size=n), L).astype(np.int32)
    bc = bc[:n].astype(np.int32)
    ids = [b"r%d" % (i // 2) for i in range(n)]
    mn, med, avg, _ = api.kmer_count_stats(pool, off, lens, 21, lib)
    bmin, _, _ = api.barcode_kmer_count_stats(pool, off, lens, bc, 21, lib)
    coarse = rng.random(n) < 0.5
    mn = np.where(coarse, np.minimum(mn, 2), mn).astype(np.int32)
    med = np.where(coarse, np.minimum(med, 3), med).astype(np.int32)
    avg = np.where(coarse, np.float32(2.5), avg).astype(np.float32)
    bmin = np.minimum(bmin, 3).astype(np.int32)
    p = rng.permutation(n)
    off, lens, bc, mn, med, avg, bmin = off[p], lens[p], bc[p], mn[p], med[p], avg[p], bmin[p]
    ids = [ids[i] for i in p]
    go = api.sort_reads_barcode(pool, off, lens, ids, mn, med, avg, bc, bmin, lib)
    pb = pool.tobytes()
    reads = [pb[o:o + l] for o, l in zip(off.tolist(), lens.tolist())]
    key = bc_key(reads, ids, mn.tolist(), med.tolist(), avg.tolist(), bc.tolist(), bmin.tolist())
    keys = [key(i) for i in range(n)]
    want = sorted(range(n), key=keys.__getitem__)
    _check_sorted_records(go, keys, want)
    assert sum(1 for a, b in zip(want, want[1:]) if keys[a][:2] == keys[b][:2]) > n // 2
    return n


def _expect(lib, code, fn, *a):
    r = fn(*a)
    assert r == code, (r, lib.err())


def check_errors(lib, ref):
    """Bad input is refused with the documented code, and the next calls still answer as the reference does."""
    reads, bc = cell_reads(215, 10, 60)
    pool, off, lens = reads_pool(reads)
    bc = np.ascontiguousarray(bc, dtype=np.int32)
    o = [np.zeros(len(reads), t) for t in (np.int32, np.int32, np.float32)]
    args = lambda b, ln, k: (pool.ctypes.data, pool.nbytes, off.ctypes.data, ln.ctypes.data, b.ctypes.data, len(reads), k,
                             o[0].ctypes.data, o[1].ctypes.data, o[2].ctypes.data)
    neg = bc.copy()
    neg[len(neg) // 2] = -1
    _expect(lib, api.T4_E_INVAL, lib.barcode_kmer_count_stats, *args(neg, lens, 21))
    _expect(lib, api.T4_E_INVAL, lib.barcode_kmer_count_stats, *args(bc, lens, 22))
    long_pool, long_off, long_lens = reads_pool(reads[:-1] + [b"ACGT" * 129])
    lbc = np.ascontiguousarray(bc, dtype=np.int32)
    r = lib.barcode_kmer_count_stats(long_pool.ctypes.data, long_pool.nbytes, long_off.ctypes.data, long_lens.ctypes.data, lbc.ctypes.data,
                                     len(reads), 21, o[0].ctypes.data, o[1].ctypes.data, o[2].ctypes.data)
    assert r == api.T4_E_UNSUPPORTED, (r, lib.err())
    ids = [b"r%d" % i for i in range(len(reads))]
    z = np.zeros(len(reads), np.int32)
    try:
        api.sort_reads_barcode(pool, off, lens, ids, z, z, z.astype(np.float32), neg, z, lib)
        assert False, "negative barcode accepted"
    except api.T4Error as e:
        assert e.code == api.T4_E_INVAL
    check_bc_stats(lib, ref, reads, bc)
    gs = api.sort_reads_barcode(pool, off, lens, ids, z, z, z.astype(np.float32), bc, z, lib)
    assert gs.tolist() == _ref_sort_bc(ref, reads, ids, z, z, z.astype(np.float32), bc, z).tolist()


def check_device_form(lib, ref, dev):
    """t4_barcode_kmer_count_stats_device on device buffers (`dev(np array)` -> (keep-alive object, address)): the same
    numbers as the host form; a barcode above barcode_max is reported through t4_kmer_count_table_stats."""
    reads, bc = STATS_CASES["wide_barcodes"]()
    pool, off, lens = reads_pool(reads)
    bc = np.ascontiguousarray(bc, dtype=np.int32)
    n = len(reads)
    inst = int(np.maximum(lens - 20, 0).sum())
    tb = lib.kmer_count_table_bytes(inst)
    bufs = [dev(pool), dev(off), dev(lens), dev(bc), dev(np.zeros(tb, np.uint8)), dev(np.zeros(n, np.int32)), dev(np.zeros(n, np.int32)),
            dev(np.zeros(n, np.float32))]
    p = [b[1] for b in bufs]
    st = np.zeros(4, dtype=np.uint64)
    lib.check(lib.barcode_kmer_count_stats_device(p[0], p[1], p[2], p[3], n, int(bc.max()), 21, p[4], tb, p[5], p[6], p[7], None))
    lib.check(lib.kmer_count_table_stats(p[4], tb, st.ctypes.data))
    assert st[3] == 0 and st[0] == inst, st
    got = [b[2]() for b in bufs[5:]]
    rmn, rmed, ravg = ref_bc_stats(ref, pool, off, lens, bc)
    assert (got[0] == rmn).all() and (got[1] == rmed).all() and (got[2].view(np.uint32) == ravg.view(np.uint32)).all()
    lib.check(lib.barcode_kmer_count_stats_device(p[0], p[1], p[2], p[3], n, int(bc.max()) - 1, 21, p[4], tb, p[5], p[6], p[7], None))
    lib.check(lib.kmer_count_table_stats(p[4], tb, st.ctypes.data))
    assert st[3] == 2, st
