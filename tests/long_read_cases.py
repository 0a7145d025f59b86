"""Checks of the stream kernel and the AssignRead pass on reads of 201-512 bp in a short-read set (first read <= 200 bp,
so isLongSeqSet stays off), shared by the GPU and the emulation test modules.  These are the lengths at which the warp
DPs of overlap scoring and of ExtendOverlap keep their traceback in the arena instead of shared memory (>= 192
columns), the overhang masks use their upper eight words (257-511 columns), the deferred-side list crosses a ballot
word (> 16 overlaps) and the hit sort switches from the bitonic to the radix sort (> 1024 keys).

Sets and reads are built by hand: random contigs entered by InputNovelRead on both sides, reads cut from them with
placed edits.  Every case proves from the reference's own data (sorted hits, overlaps, posWeight) that it reached the
edge it is meant to test, so a generator change that loses the edge fails instead of passing vacuously.
`lib` is an api.Lib, `ref` the refharness module."""
import numpy as np

from parity_cases import _diag_mismatches, _same_sets, canon_hits, check_assign_pass
from trust4_b200 import api, synth

NAME = "IGHV1-2*01"
P = 1000003                      # KINDEX_HASH_MAX (KmerIndex.hpp:21): barcodes equal modulo P share one postings list
_RC = str.maketrans("ACGTN", "TGCAN")


def revcomp(s):
    return s.translate(_RC)[::-1]


def _rand(rng, n):
    return "".join("ACGT"[c] for c in rng.integers(0, 4, size=n))


def _sub(rng, c):
    return "ACGT".replace(c, "")[int(rng.integers(3))]


def counters(lib):
    c = np.zeros(api.N_COUNTERS, dtype=np.uint64)
    lib.check(lib.last_counters(c.ctypes.data))
    return c


def _pair(lib, ref, k, hit_len=None, consider_barcode=False):
    g = api.SeqSet(k, lib)
    r = ref.RefSeqSet(k)
    if hit_len is not None:
        g.set_hit_len_required(hit_len)
        r.set_hit_len_required(hit_len)
    if consider_barcode:
        g.set_consider_barcode_in_hash(1)
        ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
    return g, r


def _input(g, r, seq, barcode=-1, name=NAME):
    a = g.input_novel_read(name, seq, 1, barcode)
    b = r.input_novel_read(name, seq, 1, barcode)
    assert a == b, ("InputNovelRead", a, b)


def _same_overlaps(g, r, read, tag=()):
    n1, o1, s1 = r.get_overlaps(read)
    n2, o2, s2 = g.get_overlaps(read)
    assert n1 == n2, ("overlap count",) + tuple(tag) + (n1, n2)
    if n1 > 0:
        assert (o1 == o2).all(), ("overlaps",) + tuple(tag) + (o1.tolist(), o2.tolist())
        assert (s1.view(np.uint64) == s2.view(np.uint64)).all(), ("similarity bits",) + tuple(tag) + (s1.tolist(), s2.tolist())
    return n1, o1, s1


def breaks(cons, lo, hi, k, rng, hit_left, hit_right, use_n):
    """Edits of cons[lo:hi] (read aligned on the contig's diagonal) that leave no k-mer of the read on that diagonal
    starting in the region: every k-window of the read that starts in it, or reaches into it from a hit on the left,
    holds an edit.  hit_left / hit_right: a hit of the diagonal borders the region (else the read ends there).  use_n: the
    edit is an N where the contig base is not A (GetHitsFromRead reads N as A, so the k-mer misses, while IsBaseEqual
    counts N as equal: no mismatch on the diagonal), else a substitution.  Returns {contig position: base}."""
    p0 = lo - k + 1 if hit_left else lo
    p1 = hi - 1 if hit_right else hi - k
    out = {}
    cur = p0
    while cur <= p1:
        top = min(cur + k - 1, hi - 1)
        low = max(cur, lo)
        b = top                           # as sparse as the rule allows: the fewest mismatches, the highest similarity
        if use_n:
            for q in range(b, low - 1, -1):
                if cons[q] != "A":
                    b = q
                    break
        out[b] = "N" if use_n and cons[b] != "A" else _sub(rng, cons[b])
        cur = b + 1
    return out


def _apply(cons, s, e, edits):
    return "".join(edits.get(p, cons[p]) for p in range(s, e))


def _gaps_on(h, idx, strand, diag, k):
    a = np.unique(h[(h[:, 0] == idx) & (h[:, 3] == strand) & (h[:, 2] - h[:, 1] == diag)][:, 2])
    return [(int(a1 - a0 - k), int(a0 + k), int(a0 + k - diag)) for a0, a1 in zip(a[:-1], a[1:]) if a0 + k - 1 < a1]


def _diagonal_gaps(r, read, o, k):
    """Gaps a1 - (a0 + k) between consecutive hits of the overlap's diagonal (the reference's sorted hits): (gap, read
    offset, contig offset of its first column)."""
    return _gaps_on(canon_hits(r.get_hits(read, 0)), o[0], o[5], o[1] - o[3], k)


def _contig_gaps(r, read, k):
    """{(contig, strand): gaps of its most populated diagonal} from the reference's sorted hits of the read."""
    h = canon_hits(r.get_hits(read, 0))
    out = {}
    for idx, strand in set(map(tuple, h[:, [0, 3]].tolist())):
        sel = h[(h[:, 0] == idx) & (h[:, 3] == strand)]
        dg, cnt = np.unique(sel[:, 2] - sel[:, 1], return_counts=True)
        out[(idx, strand)] = _gaps_on(h, idx, strand, int(dg[np.argmax(cnt)]), k)
    return out


def _oriented(read, strand):
    return read if strand == 1 else revcomp(read)


# ---- 1. overlap scoring gaps ------------------------------------------------------------------------------------------

def gap_lengths(k, lim):
    """The single-gap lengths of one case.  An overlap on a novel contig needs hits over half its span (SeqSet.hpp:1042),
    so a read of <= 512 bp holds a gap of at most ~245 columns: at k = 9 the gap limit (288) is out of reach and the
    lengths stop at 240; at k = 7 they straddle the limit (137)."""
    return (2, 3, 190, 191, 192, 193, 240) if k == 9 else (2, 3, lim - 1, lim, lim + 1)


def _gap_reads(rng, k, lim, core):
    """(plan, read start, read end, gap spans): one same-diagonal gap of each length with <= 2 and with > 2 mismatches,
    an in-band frame shift inside gaps of >= 192, a long (arena) and a short (shared-memory) gap in one overlap, and a
    failing gap (frame shift) after a passing one.  The clean stretches around the gaps hold hits over half the span."""
    plans = []
    for gap in gap_lengths(k, lim):
        for few in (True, False):
            if gap == 2 and not few:
                continue              # two columns hold at most two mismatches
            plans.append(dict(gaps=[gap], few=few, indel=0))
    if k == 9:
        for gap in (192, 230):
            plans.append(dict(gaps=[gap], few=False, indel=1 + gap % 3))
        plans.append(dict(gaps=[192, 40], few=False, indel=0))
        plans.append(dict(gaps=[40, 193], few=True, indel=0))
        plans.append(dict(gaps=[192, 40], few=False, indel=0, indel_second=2))
    out = []
    for i, pl in enumerate(plans):
        nf = len(pl["gaps"]) + 1
        flank = max(30, (sum(pl["gaps"]) + 12 + nf - 1) // nf)
        need = sum(pl["gaps"]) + flank * nf
        assert need <= CORE
        b0 = EXT + int(rng.integers(0, CORE - need + 1))          # the hits and gaps lie inside the core
        L = min(512, max(250 + int(rng.integers(0, 40)), need + int(rng.integers(0, 60))))
        s = max(0, min(b0 - int(rng.integers(0, L - need + 1)), len(core) - L))
        pos, spans = b0 + flank, []
        for gap in pl["gaps"]:
            spans.append((pos, pos + gap))
            pos += gap + flank
        assert s <= b0 and b0 + need <= s + L <= len(core)
        out.append((pl, s, s + L, spans))
    return out


CORE, EXT = 500, 12              # contigs hold the core (InputNovelRead takes <= 512 bp); reads may run EXT bases past it


def build_gap_case(lib, ref, k, seed, n_contigs=6):
    """A set of n_contigs random contigs (500-512 bp, the most InputNovelRead takes on the device) that share one
    500-bp core, and reads cut from the core (and up to EXT bases of sequence outside every contig) with gaps."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    g, r = _pair(lib, ref, k)
    lim = ref.lib().t4ref_nomatch_gap_limit(r.h)
    assert lim == {9: 288, 7: 137}[k], lim
    core = list(_rand(rng, EXT + CORE + EXT))
    plans = _gap_reads(rng, k, lim, core)
    for _, _, _, spans in plans:          # the columns next to the bordering hits take an N: make them not A
        for lo, hi in spans:
            for q in (lo, hi - 1):
                if core[q] == "A":
                    core[q] = "CGT"[int(rng.integers(3))]
    core = "".join(core)
    contigs = []
    for _ in range(n_contigs):
        a = int(rng.integers(1, 12))
        contigs.append(_rand(rng, a) + core[EXT:EXT + CORE] + _rand(rng, int(rng.integers(1, 13 - a))))
        _input(g, r, contigs[-1])
    reads = []
    for pl, s, e, spans in plans:
        ed = {}
        for j, (lo, hi) in enumerate(spans):
            d = pl["indel"] if j == 0 else pl.get("indel_second", 0)
            b = breaks(core, lo, hi, k - d, rng, True, True, pl["few"])
            for q in range(lo, hi):
                if not pl["few"] and len(b) < 3 and q not in b:      # a short gap: > 2 mismatches need a third one
                    b[q] = _sub(rng, core[q])
            ed.update(b)
        rd = _apply(core, s, e, ed)
        for j, (lo, hi) in enumerate(spans):
            d = pl["indel"] if j == 0 else pl.get("indel_second", 0)
            if d:                         # delete d columns early in the gap and insert d late: same diagonal on both sides
                x, y = lo - s + (hi - lo) // 3, hi - s - (hi - lo) // 3
                rd = rd[:x] + rd[x + d:y] + _rand(rng, d) + rd[y:]
        assert len(rd) == e - s
        reads.append(revcomp(rd) if len(reads) % 3 == 2 else rd)
    return g, r, core, plans, reads


def check_gap_scoring(lib, ref, k, seed=1):
    """GetOverlapsFromRead on reads with same-diagonal gaps of 2, 3, 190-193, limit - 1, limit and limit + 1 columns
    (k = 9: limit 288; k = 7: 137) at <= 2 and > 2 diagonal mismatches, frame shifts inside gaps of >= 192, two long
    gaps in one overlap and a failing gap after a passing one, every read on >= 5 overlaps: overlaps and bit-equal
    similarity doubles; then AddRead of every read (return, strand), Output, the index checksum and numRead per slot."""
    g, r, core, plans, reads = build_gap_case(lib, ref, k, seed)
    n_contigs = r.size()
    lim = ref.lib().t4ref_nomatch_gap_limit(r.h)
    reached = set()
    fulldp = 0
    for i, ((pl, s, e, spans), rd) in enumerate(zip(plans, reads)):
        n, o, sim = _same_overlaps(g, r, rd, tag=(i, pl))
        fulldp += int(counters(lib)[7])
        frame_shift = bool(pl["indel"] or pl.get("indel_second"))
        if frame_shift or max(pl["gaps"]) > lim:
            assert n <= 0 or (sim == 0).all(), (i, "a gap over the limit or with an indel scores 0")
        else:
            assert n == n_contigs and (sim > 0).all(), (i, n, sim)     # every warp of the CTA scores some overlap
        cg = _contig_gaps(r, rd, k)
        for idx in range(n_contigs):
            strand = -1 if i % 3 == 2 else 1                            # build_gap_case reverses every third read
            gaps = cg[(idx, strand)]
            got = sorted(x for x, _, _ in gaps if x >= 2)
            assert got == sorted(pl["gaps"]), ("gap lengths", i, idx, got, pl["gaps"])
            ro = _oriented(rd, strand)
            pw = r.get_contig(idx)["pos_weight"]
            for gap, a, b in gaps:
                if gap < 2:
                    continue
                mis = _diag_mismatches(pw[b:b + gap], ro[a:a + gap])
                if not frame_shift:
                    assert (mis <= 2) == pl["few"], ("mismatches", i, gap, mis)
                    reached.add((gap, mis > 2))
    for gap in gap_lengths(k, lim):
        assert (gap, False) in reached, ("no gap of %d with <= 2 mismatches" % gap)
        if gap > 2:
            assert (gap, True) in reached, ("no gap of %d with > 2 mismatches" % gap)
    assert fulldp > 0                     # the banded DP of a gap ran
    added = 0
    for i, rd in enumerate(reads):
        a1 = g.add_read(rd, "IGHV", 0, -1, 1, 0, 0.9)
        a2 = r.add_read(rd, "IGHV", 0, -1, 1, 0, 0.9)
        assert a1 == a2, ("AddRead", i, a1, a2)
        added += a2[0] >= 0
    assert added > 3
    _same_sets(g, r)
    return fulldp


# ---- 2. ExtendOverlap sides -------------------------------------------------------------------------------------------

SIDES = (0, 1, 2, 31, 32, 33, 63, 64, 191, 192, 193, 256, 257, 300, 460)
WORD_EDGES = (31, 32, 63, 64, 95, 96, 255, 256, 257, 287, 288)
FLANK = 460                      # A and B; contigs hold at most 512 bp, so no side is longer than FLANK + 11
HIT = 40                         # the clean stretch holding the overlap's hits
HALF = 230                       # the third contig shape: A[-HALF:] + H + B[:HALF]


def side_pairs(n_overlaps):
    """(left, right) side lengths of the reads of one case (a read holds at most 512 bp: L + R <= 472)."""
    mx = 512 - HIT
    if n_overlaps > 8:        # many overlaps per read: sides that all need the DP, both halves of a pair on the arena
        return [(192, 192), (215, 225), (300, 33), (33, 300), (193, 230), (64, 257)]
    out = []
    for s in SIDES:
        out += [(s, 0), (0, s), (s, min(192, mx - s)), (min(256, mx - s), s)]
    out += [(192, 192), (200, 225), (230, 215), (229, 229)]
    return out


def _side_edits(rng, A, B, L, R, k, few_l, few_r, indel):
    """Edits of the left side A[FLANK - L:] and of the right side B[:R]: no hit of the diagonal in either; few = N's
    (<= 2 mismatches), else substitutions plus extra substitutions at the 32-column word edges of the side."""
    el = breaks(A, FLANK - L, FLANK, k - indel, rng, False, True, few_l) if L else {}
    er = breaks(B, 0, R, k - indel, rng, True, False, few_r) if R else {}
    if not few_l:
        for c in WORD_EDGES:
            if c < L:
                el[FLANK - L + c] = _sub(rng, A[FLANK - L + c])
    if not few_r:
        for c in WORD_EDGES:
            if c < R:
                er[R - 1 - c] = _sub(rng, B[R - 1 - c])
    left = _apply(A, FLANK - L, FLANK, el)
    right = _apply(B, 0, R, er)
    if indel and L > 8 * k:
        x, y = 3 * k, L - 3 * k
        left = left[:x] + left[x + indel:y] + _rand(rng, indel) + left[y:]
    if indel and R > 8 * k:
        x, y = 3 * k, R - 3 * k
        right = right[:x] + right[x + indel:y] + _rand(rng, indel) + right[y:]
    return left, right


def build_side_case(lib, ref, n_overlaps, seed, k=9):
    """n_overlaps contigs of three shapes around one 40-bp stretch H: A + H and H + B with a short random pad of their own,
    and A[-230 - p:] + H + B[:242 - p] (A, B: 460 bp); reads = a left side cut from A, all of H, a right side cut from B.  Returns
    the sets, the reads and their (left, right) side lengths."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    g, r = _pair(lib, ref, k)
    A, H, B = list(_rand(rng, FLANK)), _rand(rng, HIT), list(_rand(rng, FLANK))
    A[-1] = "CGT"[int(rng.integers(3))]     # next to the hits: an N there must miss
    B[0] = "CGT"[int(rng.integers(3))]
    A, B = "".join(A), "".join(B)
    for i in range(n_overlaps):
        pad = int(rng.integers(1, 12))
        if i % 3 == 2:                  # the pads come from A and B: every side of this shape is A or B
            pad = 1 + (i // 3) % 11
            _input(g, r, A[-HALF - pad:] + H + B[:HALF + 12 - pad])
        else:
            _input(g, r, _rand(rng, pad) + A + H if i % 3 == 0 else H + B + _rand(rng, pad))
    reads, sides = [], []
    if n_overlaps <= 8:
        # First, on the fresh contigs: long sides with <= 2 mismatches (settled from all 16 mask words, no DP), then the
        # same sides with all their mismatches in mask words 8-15 (columns >= 256 counted from col0 = the far end of a
        # left side, the anchor of a right one): only those words tell that these sides need the DP.
        shapes = ((460, 0), (0, 460), (300, 0), (0, 300))
        for tail in (False, True):
            for L, R in shapes:
                left, right = _side_edits(rng, A, B, L, R, k, True, True, 0)
                if tail and L:
                    left = left[:256] + _rand(rng, L - 256)
                if tail and R:
                    right = right[:256] + _rand(rng, R - 256)
                reads.append(left + H + right)
                sides.append((L, R, "upper words") if tail else (L, R))
    for i, (L, R, few_l) in enumerate((L, R, f) for L, R in side_pairs(n_overlaps) for f in (True, False)):
        few_r = not few_l if i % 4 < 2 else few_l       # every side length with <= 2 and with > 2 mismatches
        indel = 2 if (i % 5 == 4) else 0
        left, right = _side_edits(rng, A, B, L, R, k, few_l, few_r, indel)
        rd = left + H + right
        assert len(rd) <= 512
        reads.append(revcomp(rd) if i % 3 == 1 else rd)
        sides.append((L, R))
    return g, r, reads, sides


def _side_spans(r, read, n, o, k):
    """Side lengths of every overlap of the read from the reference's overlaps: min(readStart, seqStart) and
    min(len - 1 - readEnd, seqLen - 1 - seqEnd); and whether each needs the banded DP (>= 2 columns, > 2 mismatches
    on the diagonal under IsBaseEqual)."""
    out = []
    for j in range(n):
        c = r.get_contig(int(o[j, 0]))
        seqLen = len(c["consensus"])
        ro = _oriented(read, o[j, 5])
        rs, re_, ss, se = (int(x) for x in o[j, 1:5])
        L = min(rs, ss)
        R = min(len(read) - 1 - re_, seqLen - 1 - se)
        ml = _diag_mismatches(c["pos_weight"][ss - L:ss], ro[rs - L:rs])
        mr = _diag_mismatches(c["pos_weight"][se + 1:se + 1 + R], ro[re_ + 1:re_ + 1 + R])
        out.append((L, R, L >= 2 and ml > 2, R >= 2 and mr > 2, ml, mr))
    return out


def check_extend_sides(lib, ref, n_overlaps, seed=3, k=9):
    """ExtendOverlap (per-call AddRead) on reads whose overlaps have left and right overhang sides of 0-460 columns,
    <= 2 and > 2 diagonal mismatches (extra ones at the 32-column word edges), frame shifts inside long sides, both
    sides of an overlap >= 192 (both half-warps of one pair on the arena), and n_overlaps overlaps per read (> 16: the
    deferred-side list crosses a ballot word; > 50: the bestNovelOverlap pre-filter): AddRead return and strand, then
    Output, the index checksum and numRead per slot.  Counter 1 of each call must be > 0 exactly when some side needs the
    banded DP (from the reference's overlaps and posWeight); clean sides of >= 257 columns are settled from all 16 mask
    words.  Returns [(read index, (left, right), counter 21 = on-demand ExtendOverlap of that call)]."""
    g, r, reads, sides = build_side_case(lib, ref, n_overlaps, seed, k)
    reached_l, reached_r, both_long, fallbacks = set(), set(), 0, []
    dp_reads = 0
    ns = []
    upper = clean_long = 0
    for i, (rd, case) in enumerate(zip(reads, sides)):
        L, R = case[:2]
        n, o, _ = r.get_overlaps(rd)
        assert n >= 4 or n_overlaps > 8, (i, n)       # every warp of the CTA handles some overlap
        ns.append(n)
        sp = _side_spans(r, rd, n, o, k)
        if len(case) == 3:                    # the DP is needed because of mask words 8-15 alone
            for j in range(n):
                c = r.get_contig(int(o[j, 0]))
                rs, re_, ss, se = (int(x) for x in o[j, 1:5])
                Lx, Rx = sp[j][:2]
                if Lx >= 300:
                    lo_words = _diag_mismatches(c["pos_weight"][ss - Lx:ss - Lx + 256], rd[rs - Lx:rs - Lx + 256])
                    upper += lo_words <= 2 and sp[j][4] > 2
                if Rx >= 300:
                    lo_words = _diag_mismatches(c["pos_weight"][se + 1:se + 257], rd[re_ + 1:re_ + 257])
                    upper += lo_words <= 2 and sp[j][5] > 2
        need = any(a or b for _, _, a, b, _, _ in sp)
        for Lx, Rx, dl, dr, ml, mr in sp:
            reached_l.add((Lx, ml > 2))
            reached_r.add((Rx, mr > 2))
            both_long += Lx >= 192 and Rx >= 192 and dl and dr
        c0 = counters(lib)                    # the counters accumulate over launches: take this call's share
        a1 = g.add_read(rd, "IGHV", 0, -1, 1, 0, 0.9)
        c = counters(lib) - c0
        a2 = r.add_read(rd, "IGHV", 0, -1, 1, 0, 0.9)
        assert a1 == a2, ("AddRead", i, (L, R), a1, a2)
        # counter 1 = overhang sides aligned by the banded DP.  Only a side of >= 2 columns with > 2 mismatches may go
        # there (an "easy" read skips the sides of its provably failing overlaps), each at most once.
        n_need = sum(int(a) + int(b) for _, _, a, b, _, _ in sp)
        assert c[1] <= n_need, ("overhang DPs on sides the masks settle", i, (L, R), int(c[1]), n_need)
        dp_reads += c[1] > 0
        if not need:
            clean_long += max(max(x[0], x[1]) for x in sp) >= 257 if n > 0 else 0
        fallbacks.append((i, (L, R), int(c[21])))
    _same_sets(g, r)
    if n_overlaps > 8:                        # > 16 overlaps: more than 32 sides to defer; > 50: the pre-filter
        edge = 50 if n_overlaps > 50 else 16
        assert sum(x > edge for x in ns) >= len(ns) // 2, ns
    want = SIDES if n_overlaps <= 8 else ()
    for s in want:
        assert any(x == s for x, _ in reached_l), ("left side of %d columns not reached" % s)
        assert any(x == s for x, _ in reached_r), ("right side of %d columns not reached" % s)
    if n_overlaps <= 8:
        for s in (31, 32, 33, 63, 64, 191, 192, 193, 256, 257, 300, 460):
            assert (s, False) in reached_l and (s, True) in reached_l, ("left side mismatch classes", s)
            assert (s, False) in reached_r and (s, True) in reached_r, ("right side mismatch classes", s)
    assert both_long > 0 and dp_reads > 0
    assert (upper >= 4 and clean_long >= 4) or n_overlaps > 8, (upper, clean_long)     # mask words 8-15 decide
    return fallbacks


def _records(reads, gene4=b"IGHV", name_id=0, flags=0):
    d = np.zeros(len(reads), dtype=synth.READ_DESC)
    o = 0
    for i, s in enumerate(reads):
        d[i]["seq_off"], d[i]["len"] = o, len(s)
        o += len(s)
    d["barcode"] = -1
    d["min_cnt"] = 1
    d["min_kmer_count"] = 1
    d["sim_threshold"] = 0.9
    d["name_id"] = name_id
    d["mate_idx"] = -1
    d["eq_lo"] = np.arange(len(reads))
    d["eq_hi"] = np.arange(len(reads)) + 1
    d["flags"] = flags
    d["novel_strand"] = 1
    d["gene4"] = gene4
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    return d, pool


def check_extend_sides_batch(lib, ref, n_overlaps, seed=3, k=9):
    """The reads of check_extend_sides through the batch loop (t4_seqset_add_reads_batch, first read length 150), every
    other one allowed to seed a contig when it fails: return, strand and rescue codes, Output, the index checksum and
    numRead per slot."""
    g, r, reads, sides = build_side_case(lib, ref, n_overlaps, seed, k)
    d, pool = _records(reads)
    d["flags"][1::2] = synth.RD_NOVEL_ON_FAIL
    cfg = synth.run_cfg(first_read_len=150)
    _, gret, gstr, gres = g.run_descs(cfg, d, pool, [NAME.encode()])
    _, rret, rstr, rres = r.run_descs(cfg, d, pool, [NAME.encode()])
    assert (gret == rret).all(), ("ret", np.flatnonzero(gret != rret)[:5])
    assert (gstr == rstr).all() and (gres == rres).all()
    _same_sets(g, r)
    assert (rret >= 0).sum() > 3
    return int((rret >= 0).sum())


def check_contig_growth(lib, ref, seed=5, k=9, step=310):
    """Contigs extended by >= 300 bases at once, three times to the left and three times to the right, and one short
    contig extended on both sides by one read: AddRead returns, Output and the index checksum after every read."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    g, r = _pair(lib, ref, k)
    G = _rand(rng, 480)
    S = _rand(rng, 90)
    _input(g, r, G)
    _input(g, r, S)
    cur = G
    grown = 0
    for t in range(6):
        new = _rand(rng, step)
        if t % 2 == 0:
            rd = new + cur[:190]
            cur = new + cur
        else:
            rd = cur[-190:] + new
            cur = cur + new
        before = len(r.get_contig(0)["consensus"])
        a1 = g.add_read(rd if t != 3 else revcomp(rd), "IGHV", 0, -1, 1, 0, 0.9)
        a2 = r.add_read(rd if t != 3 else revcomp(rd), "IGHV", 0, -1, 1, 0, 0.9)
        assert a1 == a2, ("AddRead", t, a1, a2)
        assert g.output() == r.output(), ("Output", t)
        assert g.index_checksum() == r.index_checksum(), ("index", t)
        grown += len(r.get_contig(0)["consensus"]) - before >= 300
    assert grown == 6, grown
    rd = _rand(rng, 200) + S + _rand(rng, 200)
    before = len(r.get_contig(1)["consensus"])
    assert g.add_read(rd, "IGHV", 0, -1, 1, 0, 0.9) == r.add_read(rd, "IGHV", 0, -1, 1, 0, 0.9)
    assert len(r.get_contig(1)["consensus"]) - before == 400
    _same_sets(g, r)


# ---- 3. hit sort ------------------------------------------------------------------------------------------------------

HIT_COUNTS = (1, 2, 1023, 1024, 1025, 2048, 2049)
KEY_SETS = ("one_contig", "idx_byte", "both_strands", "barcode")


def _tune(count, target, h_max, l_max, k):
    """(h, l) with count(h, l) == target; count grows with both arguments."""
    lo, hi = 0, h_max
    while lo < hi:                          # largest h with count(h, 0) <= target
        mid = (lo + hi + 1) // 2
        if count(mid, 0) <= target:
            lo = mid
        else:
            hi = mid - 1
    for h in range(lo, max(-1, lo - 40), -1):
        a, b = 0, l_max - h
        while a < b:
            mid = (a + b) // 2
            if count(h, mid) < target:
                a = mid + 1
            else:
                b = mid
        if count(h, a) == target:
            return h, a
    raise AssertionError("no read with exactly %d hits" % target)


def build_hit_sort_case(lib, ref, kind, seed=9, k=9):
    """A set and a read generator read(h, l) for one key set: h bases of a high-multiplicity region (every k-mer has
    20-30 postings, below the 100 of the skip rule) followed by l bases of a unique one.  Returns (g, r, read, strand,
    barcode)."""
    lib.check(lib.reset())
    rng = np.random.default_rng(seed)
    if kind == "one_contig":              # one contig, one strand: a 40-bp unit repeated 10 times, then unique sequence
        g, r = _pair(lib, ref, k)
        unit, U = _rand(rng, 40), _rand(rng, 112)
        c = unit * 10 + U
        _input(g, r, c)
        Lp = 40 * 10
        return g, r, (lambda h, l: c[max(0, Lp - h):Lp + l]), 1, -1
    if kind == "idx_byte":                # 300 contigs; the shared region sits in contigs 240..299 (index crosses 255)
        g, r = _pair(lib, ref, k)
        Q = _rand(rng, 100)
        for i in range(300):
            own = _rand(rng, 400)
            _input(g, r, own + (Q if i >= 240 else "") + _rand(rng, 12))
            if i == 299:
                U = own
        return g, r, (lambda h, l: U[len(U) - l:] + Q[:h] if l else Q[:h]), 1, -1
    if kind == "both_strands":            # 25 contigs carry Q; a unique region W of another contig is read reverse-complemented
        g, r = _pair(lib, ref, k)
        Q, W = _rand(rng, 300), _rand(rng, 500)
        for i in range(25):
            _input(g, r, _rand(rng, 100) + Q + _rand(rng, 100))
        _input(g, r, W)
        return g, r, (lambda h, l: revcomp(W[:100 + l]) + Q[:h]), 0, -1     # >= 92 hits on the minus strand
    assert kind == "barcode"              # salted index: barcode 5 and 5 + P share every list (20 + 30 postings)
    g, r = _pair(lib, ref, k, consider_barcode=True)
    Q, U = _rand(rng, 300), _rand(rng, 500)
    for i in range(50):
        _input(g, r, _rand(rng, 100) + Q + _rand(rng, 100), barcode=5 if i % 5 < 2 else 5 + P)
    _input(g, r, U, barcode=5)
    return g, r, (lambda h, l: Q[:h] + U[:l]), 0, 5


def check_hit_sort(lib, ref, kind, seed=9, k=9):
    """GetHitsFromRead (sorted on the device: bitonic up to 1024 keys, radix above) on reads with exactly 1, 2, 1023,
    1024, 1025, 2048 and 2049 hits, in the order the device returns them against the reference's SortHits order, then
    GetOverlapsFromRead on the same reads."""
    g, r, read, strand, bc = build_hit_sort_case(lib, ref, kind, seed, k)

    def count(h, l):
        s = read(h, l)
        return len(r.get_hits(s, strand, bc)) if len(s) >= k else 0

    for target in HIT_COUNTS:
        if kind == "both_strands" and target < 100:
            continue
        h, l = _tune(count, target, 512 - k, 512, k)
        s = read(h, l)
        assert len(s) <= 512
        hr = canon_hits(r.get_hits(s, strand, bc))
        assert len(hr) == target, (kind, target, len(hr))
        assert hr[:, 4].max() < 100                       # no list reaches the skip rule
        hg = g.get_hits(s, strand, bc)
        assert hg.shape == hr.shape and (hg == hr).all(), ("hit order", kind, target)
        if kind == "idx_byte" and target > 1000:
            assert hr[:, 0].min() < 256 <= hr[:, 0].max()
        if kind == "both_strands" and target > 1000:
            assert set(hr[:, 3].tolist()) == {-1, 1}
        if kind == "barcode" and target > 1000:
            assert len(r.get_hits(s, strand, 5 + P)) > 0     # the other barcode's postings share the lists
        if kind == "one_contig" and target > 2:
            assert len(set(hr[:, 0].tolist())) == 1 and len(set(hr[:, 3].tolist())) == 1
        n1, o1, s1 = r.get_overlaps(s, strand, bc)
        n2, o2, s2 = g.get_overlaps(s, strand, bc)
        assert n1 == n2, ("overlaps", kind, target, n1, n2)
        if n1 > 0:
            assert (o1 == o2).all() and (s1.view(np.uint64) == s2.view(np.uint64)).all(), ("overlaps", kind, target)


# ---- 4./5. the batch loop and the AssignRead pass on a mixed-length workload --------------------------------------------

def mixed_workload(seed, nclones=8, npairs=300, k=9):
    """150-bp pairs whose overlapping mates are merged into one read of 151-285 bp (ProcessRead, main.cpp:290-315), the
    other pairs kept, plus reads of 300-512 bp: denser substitutions (2 %), a same-diagonal gap of 192-260 columns, or a
    side of 301-360 columns without hits.  Records keep the synthetic driver's fields of the first mate; the long reads
    follow.  Returns (synth.Workload, indices of the gap reads, indices of the side reads)."""
    cl = synth.make_clones(nclones, seed)
    rd = synth.sample_pairs(cl, npairs, 150, seed)
    w = synth.build_workload(cl, rd)
    rng = np.random.default_rng(seed)
    L = w.L
    pair = rd.pair[w.order]
    by_pair = {}
    for i, p in enumerate(pair):
        by_pair.setdefault(int(p), []).append(i)
    keep, seqs, merged = [], [], set()
    for i in range(len(w.descs)):
        s = w.read(i)
        p = by_pair[int(pair[i])]
        if len(p) == 2 and i == p[1] and int(p[0]) in merged:
            continue
        if len(p) == 2 and i == p[0]:
            o = w.order[p]
            t = rd.tstart[o]
            c = int(rd.clone[o[0]])
            a, b = int(t.min()), int(t.max()) + L
            if b - a < 2 * L - 15:                      # the mates overlap by >= 15 bases: one merged read
                tx = synth.decode(cl.seq[cl.off[c] + a:cl.off[c] + b])
                s = tx if rd.strand[o[0]] == 1 else revcomp(tx)
                merged.add(i)
        keep.append(i)
        seqs.append(s)
    # long reads from the clone transcripts, after the short ones
    tx = [synth.decode(cl.seq[cl.off[c]:cl.off[c + 1]]) for c in range(nclones)]
    longs, kinds = [], []
    for t in range(36):
        c = int(rng.integers(nclones))
        T = tx[c]
        kind = t % 3
        # a gap read keeps hits over half the overlap's span (SeqSet.hpp:1042): >= 394 bp for a gap of >= 192
        n = int(min(len(T), rng.integers(420 if kind == 1 else 300, 513)))
        s0 = int(rng.integers(0, len(T) - n + 1))
        ed = {}
        if kind == 0:
            for q in range(n):
                if rng.random() < 0.02:
                    ed[s0 + q] = _sub(rng, T[s0 + q])
        elif kind == 1 and n >= 394:                     # one gap of 192-260 columns between clean stretches
            gap = int(rng.integers(192, min(261, (n - 10) // 2 + 1)))
            lo = s0 + int(rng.integers(30, n - gap - 29))
            ed = breaks(T, lo, lo + gap, k, rng, True, True, False)
        elif n >= 360:                                    # a left or right side of 301-360 columns without hits
            side = int(rng.integers(301, min(361, n - 40)))
            ed = breaks(T, s0, s0 + side, k, rng, False, True, False) if t % 2 else breaks(T, s0 + n - side, s0 + n, k, rng, True, False, False)
        s = _apply(T, s0, s0 + n, ed)
        longs.append(s if rng.random() < 0.5 else revcomp(s))
        kinds.append(kind)
    d = w.descs[keep].copy()
    ld =np.zeros(len(longs), dtype=synth.READ_DESC)
    ld["name_id"] = max(0, int(d["name_id"].max()))
    ld["gene4"] = b"IGHV"
    ld["flags"] = synth.RD_NOVEL_ON_FAIL
    ld["novel_strand"] = 1
    ld["min_cnt"] = 1
    ld["min_kmer_count"] = 1
    ld["sim_threshold"] = 0.9
    d = np.concatenate([d, ld])
    n = len(d)
    allseq = seqs + longs
    off = np.zeros(n, dtype=np.uint64)
    off[1:] = np.cumsum([len(s) for s in allseq[:-1]])
    d["seq_off"] = off
    d["len"] = [len(s) for s in allseq]
    d["barcode"] = -1
    d["mate_idx"] = -1
    d["flags"] &= ~np.uint32(synth.RD_DUP)
    d["eq_lo"] = np.arange(n)
    d["eq_hi"] = np.arange(n) + 1
    pool = np.frombuffer(("".join(allseq) + "\0" * 16).encode(), dtype=np.uint8).copy()
    wl = synth.Workload(d, pool, w.names, L, np.arange(n), np.ones(n, dtype=np.int32))
    base = len(seqs)
    return wl, [base + j for j, x in enumerate(kinds) if x == 1], [base + j for j, x in enumerate(kinds) if x == 2]


def _long_edges(r, wl, gap_idx, side_idx, k):
    """The reads of gap_idx with a same-diagonal gap of >= 192 columns on some overlap of the set r, and the reads of
    side_idx with a side of >= 301 columns that needs the banded DP (> 2 mismatches on the diagonal)."""
    gaps, sides = [], []
    for i in gap_idx:
        rd = wl.read(i)
        n, o, _ = r.get_overlaps(rd)
        if any(x >= 192 for j in range(max(0, n)) for x, _, _ in _diagonal_gaps(r, rd, o[j], k)):
            gaps.append(i)
    for i in side_idx:
        rd = wl.read(i)
        n, o, _ = r.get_overlaps(rd)
        if n > 0 and any((a >= 301 and ml > 2) or (b >= 301 and mr > 2) for a, b, _, _, ml, mr in _side_spans(r, rd, n, o, k)):
            sides.append(i)
    return gaps, sides


def _edges_before_add(ref, descs, pool, names, gap_idx, side_idx):
    """_long_edges on the reference set as the batch loop leaves it just before each read: the loop over the records
    before it (no final consensus update, no rescue pass)."""
    cfg = synth.run_cfg(first_read_len=150, final_update=0, do_rescue=0)
    wl = synth.Workload(descs, pool, names, 150, None)
    gaps, sides = [], []
    for i in sorted(set(gap_idx) | set(side_idx)):
        r = ref.RefSeqSet(9)
        r.run_descs(cfg, descs[:i].copy(), pool, names)
        g_, s_ = _long_edges(r, wl, [i] if i in gap_idx else [], [i] if i in side_idx else [], 9)
        gaps += g_
        sides += s_
        r.close()
    return gaps, sides


def check_mixed_batch(lib, ref, n_streams, seed=13):
    """t4_streams_run (first read length 150) over merged mates of 151-285 bp, 150-bp reads and reads of 300-512 bp in
    n_streams contiguous streams: per stream the return, strand and rescue codes, Output and the index checksum against
    the reference's restated loop.  At least three reads meet a gap of >= 192 columns, and three a side of >= 301 that
    needs the DP, in the reference's set just before their AddRead."""
    lib.check(lib.reset())
    wl, gap_idx, side_idx = mixed_workload(seed)
    lens = wl.descs["len"]
    assert ((lens > 150) & (lens <= 285)).sum() > 50 and (lens > 300).sum() >= 30 and lens.max() <= 512
    cfg = synth.run_cfg(first_read_len=150)
    off, descs = synth.shard_workload(wl, n_streams)
    sets = api.SeqSet.create_many(len(off) - 1, 9, lib)
    ret, strands, resc = api.streams_run(sets, cfg, descs, off, wl.pool, wl.names, lib)
    ngap = nside = 0
    for j in range(len(off) - 1):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(9)
        _, rret, rstr, rres = r.run_descs(cfg, descs[lo:hi].copy(), wl.pool, wl.names)
        assert (rret == ret[lo:hi]).all(), ("ret", j, np.flatnonzero(rret != ret[lo:hi])[:5])
        assert (rstr == strands[lo:hi]).all() and (rres == resc[lo:hi]).all(), ("strand/rescue", j)
        assert r.output() == sets[j].output(), ("contigs", j)
        assert r.index_checksum() == sets[j].index_checksum(), ("index", j)
        g_, s_ = _edges_before_add(ref, descs[lo:hi].copy(), wl.pool, wl.names, [i - lo for i in gap_idx if lo <= i < hi],
                                   [i - lo for i in side_idx if lo <= i < hi])
        ngap += len(g_)
        nside += len(s_)
    assert int((ret >= 0).sum()) > len(descs) // 2
    assert ngap >= 3 and nside >= 3, (ngap, nside)


def check_mixed_assign(lib, ref, kmer, n_streams=2, seed=13):
    """The AssignRead pass (t4_streams_assign_reads) over the sets the mixed-length workload builds, as check_assign_pass:
    per read the contig, coordinates, strand, matchCnt and similarity; per extended set Output and the index checksum.
    On the reference's extended sets (k = kmer) at least three listed reads have a same-diagonal gap of >= 192 columns
    and three a side of >= 301 columns that needs the DP (the thread-per-side t4_dp_equal of the pass)."""
    wl, gap_idx, side_idx = mixed_workload(seed)
    cfg = synth.run_cfg(first_read_len=150)
    n_listed, n_assigned = check_assign_pass(lib, ref, seed, n_streams, workload=wl, kmer=kmer, cfg=cfg)
    assert n_assigned > len(wl.descs) // 2
    off, descs = synth.shard_workload(wl, n_streams)          # the streams check_assign_pass ran
    gaps, sides = [], []
    for j in range(len(off) - 1):
        lo, hi = int(off[j]), int(off[j + 1])
        d = descs[lo:hi].copy()
        r = ref.RefSeqSet(9)
        _, rret, rstr, rres = r.run_descs(cfg, d, wl.pool, wl.names)
        lst = ref.assembled_list(rret, rres)
        ext, _, _ = ref.assign_pass(r, kmer, d, wl.pool, lst, rstr)
        sub = synth.Workload(d, wl.pool, wl.names, 150, None)
        listed = set(int(x) for x in lst)
        g_, s_ = _long_edges(ext, sub, [i - lo for i in gap_idx if lo <= i < hi and i - lo in listed],
                             [i - lo for i in side_idx if lo <= i < hi and i - lo in listed], kmer)
        gaps += g_
        sides += s_
    assert len(gaps) >= 3 and len(sides) >= 3, (len(gaps), len(sides))
    return n_listed, n_assigned
