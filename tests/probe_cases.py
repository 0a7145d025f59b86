"""Checks of the k-mer lookup (SeqSet::GetHitsFromRead + KmerIndex::Search) at its edges, shared by the GPU and the
emulation test modules: barcodes that the reference's index hashes into one postings list, postings lists of exactly the
sizes where the rules and the probe kernel's emit paths switch, read lengths around the packing words and the probe
tiles, the probe's counters and its key-buffer overflow.  `lib` is an api.Lib, `ref` the refharness module."""
import re

import numpy as np

from parity_cases import _canon4, canon_hits
from trust4_b200 import api, synth

P = 1000003                      # KINDEX_HASH_MAX (KmerIndex.hpp:21): barcodes equal modulo P share one postings list
_RC = str.maketrans("ACGTN", "TGCAN")


def revcomp(s):
    return s.translate(_RC)[::-1]


def _rand(rng, n):
    return "".join("ACGT"[c] for c in rng.integers(0, 4, size=n))


def _pair(lib, ref, k, consider_barcode, hit_len=13):
    """An empty device set and an empty reference set configured alike."""
    g = api.SeqSet(k, lib)
    r = ref.RefSeqSet(k)
    g.set_hit_len_required(hit_len)
    r.set_hit_len_required(hit_len)
    if consider_barcode:
        g.set_consider_barcode_in_hash(1)
        ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
    return g, r


def _input(g, r, name, seq, strand, barcode):
    a = g.input_novel_read(name, seq, strand, barcode)
    b = r.input_novel_read(name, seq, strand, barcode)
    assert a == b, ("InputNovelRead", a, b)


def _records(reads, strands, barcodes):
    d = np.zeros(len(reads), dtype=synth.READ_DESC)
    o = 0
    for i, (s, st, bc) in enumerate(zip(reads, strands, barcodes)):
        d[i]["seq_off"], d[i]["len"], d[i]["strand_in"], d[i]["barcode"] = o, len(s), st, bc
        o += len(s)
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    return d, pool


def _same_hits(g, r, read, strand, barcode, skip=False, tag=()):
    hr = canon_hits(r.get_hits(read, strand, barcode, skip))
    hg = canon_hits(g.get_hits(read, strand, barcode, skip))
    assert hr.shape == hg.shape and (hr == hg).all(), ("get_hits",) + tuple(tag) + (hr.shape, hg.shape)
    return hr


def _same_overlaps(g, r, read, strand, barcode, tag=()):
    n1, o1, s1 = r.get_overlaps(read, strand, barcode)
    n2, o2, s2 = g.get_overlaps(read, strand, barcode)
    assert n1 == n2, ("overlap count",) + tuple(tag) + (n1, n2)
    if n1 > 0:
        assert (o1 == o2).all(), ("overlaps",) + tuple(tag)
        assert (s1.view(np.uint64) == s2.view(np.uint64)).all(), ("similarity bits",) + tuple(tag)
    return n1


def _probe(lib, sets, reads, strands, barcodes, off, skip, cap=8 << 20):
    """t4_streams_get_hits over `reads` against `sets` (record i belongs to set j iff off[j] <= i < off[j + 1])."""
    d, pool = _records(reads, strands, barcodes)
    wl = api.Workload(d, pool, [], lib)
    hits = api.Hits(max(1, len(reads)), cap, lib)
    api.streams_get_hits(sets, wl, off, hits, allow_total_skip=skip)
    st = hits.stats()
    got = [hits.fetch(i) for i in range(len(reads))]
    wl.close()
    hits.close()
    return st, got


# ---- 1. barcodes the reference hashes together ------------------------------------------------------------------------

COLLIDING = {"5~1000008": (5, 5 + P), "7~2000013": (7, 7 + 2 * P), "-1~1000002": (-1, P - 1), "999997~2000000": (999997, 2000000)}
CONTROL = {"5~6": (5, 6)}
# contigs per barcode: each list below 100 and their sum above; one barcode's list alone at 100 and more
COUNTS = {"sum>=100": (60, 55), "one>=100": (130, 30)}


def build_colliding(lib, ref, k, barcodes, counts, seed):
    """Two barcodes' contigs in one barcode-salted set: every contig carries one 80-bp core (so each core k-mer's list
    holds counts[0] + counts[1] postings in the reference when the barcodes collide) between tails of its own."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    core = _rand(rng, 80)
    g, r = _pair(lib, ref, k, True)
    contigs = {b: [] for b in barcodes}
    order = [b for b, n in zip(barcodes, counts) for _ in range(n)]
    rng.shuffle(order)                                    # the two cells' contigs enter the index interleaved
    for b in order:
        s = _rand(rng, 12) + core + _rand(rng, 20)
        _input(g, r, "IGHV1-2*01", s, 1, int(b))
        contigs[int(b)].append(s)
    assert g.size() == r.size() == sum(counts)
    assert g.index_checksum() == r.index_checksum()
    queries = [contigs[barcodes[0]][0], core, revcomp(contigs[barcodes[1]][-1]), core[:40] + _rand(rng, 60),
               _rand(rng, 30) + core[20:70] + _rand(rng, 30), _rand(rng, 100)]
    return g, r, core, contigs, queries


def check_colliding_barcodes(lib, ref, k, barcodes, counts, seed=0, n_add=24):
    """GetHitsFromRead, GetOverlapsFromRead, AddRead and Output on a barcode-salted set whose two barcodes share their
    postings lists in the reference (or not: the control).  The >= 100-postings skip rule sees the shared list's size,
    and a read without a barcode gets the hits of the barcode its -1 collides with (1000002)."""
    g, r, core, contigs, queries = build_colliding(lib, ref, k, barcodes, counts, seed)
    qbc = list(barcodes) + [-1, 3]
    nz = 0
    for qi, q in enumerate(queries):
        for b in qbc:
            for strand in (0, 1, -1):
                nz += len(_same_hits(g, r, q, strand, b, tag=(qi, b, strand))) > 0
            _same_overlaps(g, r, q, 0, b, tag=(qi, b))
    assert nz > 10
    if sum(counts) > 10000:
        hr = r.get_hits(core, 0, -1)
        assert hr[:, 4].max() > 10000          # the scenario really has a list of more than 10000 postings for barcode -1
    rng = np.random.default_rng(seed + 1)
    for t in range(n_add):
        b = qbc[t % 3]
        src = contigs[barcodes[t % 2]][int(rng.integers(len(contigs[barcodes[t % 2]])))]
        s = list(src)
        s[int(rng.integers(len(s)))] = "ACGT"[int(rng.integers(4))]
        s = "".join(s) + _rand(rng, int(rng.integers(0, 30)))
        if t % 4 == 3:
            s = revcomp(s)
        a1 = g.add_read(s, "IGHV", 0, b, 1, 0, 0.9)
        a2 = r.add_read(s, "IGHV", 0, b, 1, 0, 0.9)
        assert a1 == a2, ("AddRead", t, b, a1, a2)
    assert g.output() == r.output()
    assert g.index_checksum() == r.index_checksum()


def check_colliding_probe(lib, ref, k, barcodes, counts, seed=0):
    """t4_streams_get_hits over the sets of check_colliding_barcodes, records carrying barcodes: the probe kernel's salt
    and barcode filter against the reference's GetHitsFromRead with the same barcode; flags bit 0 (a list of more than
    10000 postings) only for records without a barcode (the reference sets repeats = 1 otherwise)."""
    g, r, core, contigs, queries = build_colliding(lib, ref, k, barcodes, counts, seed)
    reads, strands, bcs = [], [], []
    for q in queries:
        for b in list(barcodes) + [-1, 3]:
            for strand in (0, 1, -1):
                reads.append(q)
                strands.append(strand)
                bcs.append(b)
    total = flagged = 0
    for skip in (0, 1):
        st, got = _probe(lib, [g], reads, strands, bcs, [0, len(reads)], skip)
        flagged += sum(fl & 1 for _, fl in got)
        assert st["records"] == len(reads) and st["unsupported"] == 0
        for i, (hg, fl) in enumerate(got):
            hr = r.get_hits(reads[i], strands[i], bcs[i], bool(skip))
            a, b = _canon4(hr), _canon4(hg)
            assert a.shape == b.shape and (a == b).all(), ("probe", i, bcs[i], strands[i], skip, a.shape, b.shape)
            big = bool(len(hr)) and hr[:, 4].max() > 10000
            assert bool(fl & 1) == big, ("flags", i, bcs[i], fl)
            if bcs[i] != -1:
                assert not fl & 1
            total += len(a)
    assert total > 100
    if sum(counts) > 10000:
        assert flagged > 0            # without allowTotalSkip some record without a barcode takes a list of > 10000


def check_colliding_batch(lib, ref, seed=35):
    """The batch loop (t4_seqset_add_reads_batch) with has_barcode = 1 over interleaved cells whose barcodes collide in
    the reference's index (3 and 1000006; 1000002 and reads without a barcode), release_barcodes off and on: return codes,
    strands, rescue codes, Output and the index checksum against the reference's restated loop."""
    cl = synth.make_clones(6, seed)
    w = synth.build_workload(cl, synth.sample_pairs(cl, 400, 150, seed))
    d = w.descs.copy()
    reads = w.pool.reshape(-1, w.L)
    h = (reads.astype(np.int64) * np.arange(1, w.L + 1)).sum(axis=1)
    cells = np.array([3, 3 + P, P - 1, -1, 8], dtype=np.int32)
    d["barcode"] = cells[h % len(cells)]
    d["mate_idx"] = -1
    d["sim_threshold"] = 0.9
    n = len(d)
    same_prev = np.zeros(n, dtype=bool)
    same_prev[1:] = (reads[1:] == reads[:-1]).all(axis=1) & (d["barcode"][1:] == d["barcode"][:-1])
    d["flags"] = np.where(same_prev, d["flags"] | synth.RD_DUP, d["flags"] & ~np.uint32(synth.RD_DUP))
    d["eq_lo"] = np.arange(n)
    d["eq_hi"] = np.arange(n) + 1
    for release in (0, 1):
        lib.check(lib.reset())
        cfg = synth.run_cfg(has_barcode=1, release_barcodes=release)
        g, r = _pair(lib, ref, 9, True)
        _, gret, gstr, gres = g.run_descs(cfg, d, w.pool, w.names)
        _, rret, rstr, rres = r.run_descs(cfg, d, w.pool, w.names)
        assert (gret == rret).all(), ("ret", release, np.flatnonzero(gret != rret)[:5])
        assert (gstr == rstr).all() and (gres == rres).all()
        assert g.output() == r.output()
        assert g.index_checksum() == r.index_checksum()
        assert g.size() == r.size()
        assert (rret >= 0).sum() > n // 2


# ---- 3. postings lists of exactly the sizes where the rules and the probe's emit paths switch -------------------------

LIST_SIZES = (1, 4, 5, 99, 100, 101, 255, 256, 257, 10000, 10001)
SEG = 24


def _kmers(s, k):
    return [s[i:i + k] for i in range(len(s) - k + 1)]


def kmer_code(s):
    v = 0
    for c in s:
        v = v * 4 + max(0, "ACGT".find(c))       # N reads as A
    return v


def build_list_sizes(lib, ref, k=9, seed=7):
    """A set where every k-mer of segment j has exactly LIST_SIZES[j] postings: contig c is the concatenation, in j order,
    of the segments j with LIST_SIZES[j] > c (10001 contigs by InputNovelRead, barcode -1, unsalted index)."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    while True:
        segs = [_rand(rng, SEG) for _ in LIST_SIZES]
        km = [x for s in segs for x in _kmers(s, k)]
        if len(set(km)) == len(km) and all(kmer_code(x) for x in km):
            break
    g, r = _pair(lib, ref, k, False, hit_len=31)
    for c in range(max(LIST_SIZES)):
        _input(g, r, "IGHV1-2*01", "".join(s for s, n in zip(segs, LIST_SIZES) if n > c), 1, -1)
    for s, n in zip(segs, LIST_SIZES):
        for x in _kmers(s, k):
            assert len(r.index_lookup(kmer_code(x))) == n, (n, x)
    assert g.index_checksum() == r.index_checksum()
    return g, r, segs


def list_size_reads(segs, seed=8):
    """Reads that hit each segment with its first, last and a middle position, mixtures, and reads whose one probe tile
    stages more than 448 postings in fewer and in more than 32 lists of 5..256."""
    rng = np.random.default_rng(seed)
    by = dict(zip(LIST_SIZES, segs))
    reads = []
    for s in segs:
        reads += [s + _rand(rng, 40), _rand(rng, 40) + s, _rand(rng, 20) + s + _rand(rng, 20), s[3:21]]
    reads += [
        by[99] + _rand(rng, 30),                                  # 16 lists of 99: 1584 staged postings, < 32 lists
        (by[99] + by[5]) * 3,                                     # > 32 lists of 5..99, > 448 postings, fast path
        (by[5] + by[99] + by[4] + by[256]) * 2,                   # staged and one-sector lists with the serial rules
        by[255] + by[257] + by[101] + by[100],
        "".join(segs),                                            # 264 bp at k = 9: two tiles, every list size
        by[10000] + by[1] + by[10001],
        by[100][:12] + "N" + by[100][13:] + by[101],
    ]
    return reads + [revcomp(x) for x in reads]


def check_list_sizes(lib, ref, seed=7, per_call=True):
    """GetHitsFromRead at postings lists of exactly 1, 4, 5, 99, 100, 101, 255, 256, 257, 10000 and 10001 entries, through
    t4_streams_get_hits (strand -1 / 0 / +1, allowTotalSkip 0 / 1) and, per_call, the stream engine's own lookup."""
    g, r, segs = build_list_sizes(lib, ref, seed=seed)
    reads = list_size_reads(segs)
    strands = [(0, 1, -1)[i % 3] for i in range(len(reads))]
    n = 0
    for skip in (0, 1):
        for rot in range(3):
            st_ = [(0, 1, -1)[(i + rot) % 3] for i in range(len(reads))]
            st, got = _probe(lib, [g], reads, st_, [-1] * len(reads), [0, len(reads)], skip)
            assert st["records"] == len(reads)
            for i, (hg, fl) in enumerate(got):
                hr = r.get_hits(reads[i], st_[i], -1, bool(skip))
                a, b = _canon4(hr), _canon4(hg)
                assert a.shape == b.shape and (a == b).all(), ("list sizes", i, len(reads[i]), st_[i], skip, a.shape, b.shape)
                assert bool(fl & 1) == (bool(len(hr)) and hr[:, 4].max() > 10000), ("flags", i, fl)
                n += len(a)
    assert n > 100000
    if per_call:
        for i, q in enumerate(reads):
            _same_hits(g, r, q, strands[i], -1, skip=bool(i & 1), tag=("per call", i))


# ---- 4. read lengths around the packing words and the probe tiles; 5. counters; 6. key buffer overflow ----------------

EDGE_LENGTHS = (32, 33, 64, 65, 152, 153, 400, 511, 512, 513)


def build_edge_sets(lib, ref, ks=(9, 17, 31), seed=11):
    """One set per k of 24 random 500-bp contigs, each entered 1..6 times (lists of one sector and TMA-staged lists, none
    near 100)."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    out = []
    for k in ks:
        g, r = _pair(lib, ref, k, False, hit_len=31)
        contigs = [_rand(rng, 500) for _ in range(24)]
        for c in contigs:
            for _ in range(int(rng.integers(1, 7))):
                _input(g, r, "IGHV1-2*01", c, 1, -1)
        out.append((k, g, r, contigs))
    return out


def edge_reads(k, contigs, rng):
    """Reads of lengths k - 1, k and EDGE_LENGTHS cut from the contigs, clean and with N's at 31 / 32 / 63 / 64 and
    inside the last k bases."""
    reads = []
    for L in (k - 1, k) + EDGE_LENGTHS:
        for v in range(3):
            a, b = rng.integers(len(contigs), size=2)
            src = contigs[a] + contigs[b]
            o = int(rng.integers(0, len(src) - L + 1))
            s = list(src[o:o + L])
            if v == 1:
                for p in (31, 32, 63, 64):
                    if p < L:
                        s[p] = "N"
            if v == 2 and L > 0:
                s[L - 1 - int(rng.integers(min(k, L)))] = "N"
            s = "".join(s)
            reads.append(revcomp(s) if rng.random() < 0.3 else s)
    return reads


def python_lookups(read, strand, k):
    """The reference loop's lookup count when no list reaches 100 postings: per active strand pass, the first k-mer and
    every k-mer whose code (N read as A) differs from the previous one's."""
    n = 0
    for p, s in ((0, read), (1, revcomp(read))):
        if (p == 0 and strand == -1) or (p == 1 and strand == 1) or len(s) < k:
            continue
        codes = [kmer_code(s[q:q + k]) for q in range(len(s) - k + 1)]
        n += 1 + sum(codes[q] != codes[q - 1] for q in range(1, len(codes)))
    return n


def edge_batch(lib, ref, seed=11):
    """Records of every edge length over three sets (k = 9, 17, 31) in ONE launch, with empty desc_off ranges before,
    between and after them: (sets, reads, strands, desc_off, set index per record, reference set per record)."""
    es = build_edge_sets(lib, ref, seed=seed)
    rng = np.random.default_rng(seed + 1)
    sets, off, reads, owner = [], [0], [], []
    filler = es[0][1]
    for j, (k, g, r, contigs) in enumerate(es):
        sets.append(filler)                               # an empty range
        off.append(len(reads))
        rs = edge_reads(k, contigs, rng)
        reads += rs
        owner += [j] * len(rs)
        sets.append(g)
        off.append(len(reads))
    sets.append(filler)
    off.append(len(reads))
    strands = [int(rng.choice([0, 0, 1, -1])) for _ in reads]
    return es, sets, reads, strands, np.array(off, dtype=np.int64), owner


def check_read_length_edges(lib, ref, seed=11):
    """t4_streams_get_hits at read lengths k - 1, k, 32/33, 64/65 (packing words), 152/153 (one or two probe tiles at
    k = 9), 400, 511, 512 and 513 (over the device limit: 0 hits, counted as unsupported), N's at the word edges and in
    the last k bases, sets of k = 9, 17 and 31 in one launch with empty set ranges."""
    es, sets, reads, strands, off, owner = edge_batch(lib, ref, seed)
    for skip in (0, 1):
        st, got = _probe(lib, sets, reads, strands, [-1] * len(reads), off, skip)
        assert st["records"] == len(reads)
        assert st["unsupported"] == sum(len(x) > 512 for x in reads) > 0
        nz = 0
        for i, (hg, fl) in enumerate(got):
            k, g, r, _ = es[owner[i]]
            if len(reads[i]) > 512:
                assert len(hg) == 0 and fl == 0, ("over the device limit", i)
                continue
            a = _canon4(r.get_hits(reads[i], strands[i], -1, bool(skip)))
            b = _canon4(hg)
            assert a.shape == b.shape and (a == b).all(), ("length edges", i, k, len(reads[i]), strands[i], skip, a.shape, b.shape)
            nz += len(a) > 0
        assert nz > len(reads) // 2


def check_hits_counters(lib, ref, seed=11):
    """t4_hits_stats against plain counts over the records of check_read_length_edges (no list reaches 100 postings):
    [0] hits = the reference's, [1] lookups = python_lookups, [2] postings = hits (no barcodes), [3] packed bytes
    ceil(L / 4) of the records the probe reads (k <= L <= 512), [4] / [5] the header's byte formulas, [6] records over
    512 bp, [7] records."""
    es, sets, reads, strands, off, owner = edge_batch(lib, ref, seed)
    st, _ = _probe(lib, sets, reads, strands, [-1] * len(reads), off, 0)
    want_hits = want_looks = want_bytes = 0
    for i, q in enumerate(reads):
        k, g, r, _ = es[owner[i]]
        if len(q) > 512 or len(q) < k:
            continue
        want_hits += len(r.get_hits(q, strands[i], -1))
        want_looks += python_lookups(q, strands[i], k)
        want_bytes += (len(q) + 3) // 4
    assert st["hits"] == want_hits > 0
    assert st["lookups"] == want_looks
    assert st["postings"] == want_hits
    assert st["read_bytes"] == want_bytes
    assert st["algorithmic_bytes"] == want_bytes + 8 * want_looks + 8 * want_hits + 8 * want_hits
    assert st["algorithmic_bytes_16B_hits"] == want_bytes + 8 * want_looks + 8 * want_hits + 16 * want_hits
    assert st["unsupported"] == sum(len(q) > 512 for q in reads)
    assert st["records"] == len(reads)
    return want_hits


def check_key_buffer_too_small(lib, ref, seed=11):
    """A hit buffer one key too small: t4_hits_stats returns T4_E_NOMEM and t4_last_error names the keys needed; a buffer
    of exactly that many keys then gives every record's exact hits, and the small one fails the same way again."""
    es, sets, reads, strands, off, owner = edge_batch(lib, ref, seed)
    need = sum(len(es[owner[i]][2].get_hits(q, strands[i], -1)) for i, q in enumerate(reads)
               if es[owner[i]][0] <= len(q) <= 512)
    d, pool = _records(reads, strands, [-1] * len(reads))
    wl = api.Workload(d, pool, [], lib)
    for cap in (need - 1, 1000, need, need - 1):
        hits = api.Hits(len(reads), cap, lib)
        api.streams_get_hits(sets, wl, off, hits)
        if cap < need:
            try:
                hits.stats()
                raise AssertionError("no T4_E_NOMEM with %d of %d keys" % (cap, need))
            except api.T4Error as e:
                assert e.code == api.T4_E_NOMEM
                m = re.search(r"(\d+) keys needed", lib.err())
                assert m and int(m.group(1)) == need, lib.err()
        else:
            st = hits.stats()
            assert st["hits"] == need
            for i, q in enumerate(reads):
                k, g, r, _ = es[owner[i]]
                hg, _ = hits.fetch(i)
                if len(q) > 512:
                    assert len(hg) == 0
                    continue
                a, b = _canon4(r.get_hits(q, strands[i], -1)), _canon4(hg)
                assert a.shape == b.shape and (a == b).all(), ("after overflow", i)
        hits.close()
    wl.close()
