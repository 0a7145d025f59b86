"""Parity checks shared by the emulation (CPU, tests/emu) and GPU test modules.  `lib` is an api.Lib."""
import gzip
import hashlib
import json
import os

import numpy as np

from trust4_b200 import api, synth
import tracereplay as tr

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gold_trace(name):
    return tr.load_trace(os.path.join(GOLD, name + ".trace.gz"))


def gold_raw(name):
    return gzip.open(os.path.join(GOLD, name + "_raw.out.gz")).read()


def check_trace_replay(lib, name):
    """Every SeqSet call of a real trust4 run, one C-ABI call each: return values, strand outputs and the
    final Output text must equal what the reference binary produced."""
    lib.check(lib.reset())
    s, bad = tr.replay(gold_trace(name), lambda k: api.SeqSet(k, lib))
    assert not bad, bad[:1]
    assert s.output() == gold_raw(name)


def small_workload(seed, nclones=25, npairs=400, L=150):
    cl = synth.make_clones(nclones, seed)
    rd = synth.sample_pairs(cl, npairs, L, seed)
    return synth.build_workload(cl, rd)


BATCH_GOLD = os.path.join(GOLD, "batch_ref.json.gz")


def batch_inputs(lib, seed, n_shards, nclones=25, npairs=400, cfg=None, deal=False, group="", c_mode=None):
    """Workload, loop configuration and read shards of one batch case; key = its name in batch_ref.json.gz."""
    w = small_workload(seed, nclones, npairs)
    cfg = cfg if cfg is not None else synth.run_cfg()
    if c_mode is not None:
        off, descs, _ = api.shard_reads(w.descs, n_shards, c_mode, lib)
    else:
        off, descs = synth.shard_workload(w, n_shards, deal=deal, balance="cost" if group else "reads", group=group)
    key = "seed=%d shards=%d clones=%d pairs=%d deal=%d group=%s c_mode=%s cfg=%s" % (
        seed, n_shards, nclones, npairs, deal, group, c_mode, hashlib.sha256(cfg.tobytes()).hexdigest()[:16])
    return key, w, cfg, off, descs


def _sha(b):
    return hashlib.sha256(b).hexdigest()


def shard_digest(ret, strands, resc, output, index_checksum, size):
    """What one shard of a batch run produced, digested: the same for the reference and for the engine iff equal."""
    a = lambda x: _sha(np.ascontiguousarray(x, dtype=np.int64).tobytes())
    return {"ret": a(ret), "strand": a(strands), "rescue": a(resc), "contigs": _sha(output),
            "index": [int(index_checksum[0]), int(index_checksum[1])], "size": int(size)}


def ref_batch_digests(ref, w, cfg, off, descs, k=9):
    out = []
    for j in range(len(off) - 1):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(k)
        _, rret, rstr, rresc = r.run_descs(cfg, descs[lo:hi].copy(), w.pool, w.names)
        out.append(shard_digest(rret, rstr, rresc, r.output(), r.index_checksum(), r.size()))
        r.close()
    return out


def check_batch_vs_ref(lib, ref, seed, n_shards, nclones=25, npairs=400, cfg=None, deal=False, group="", c_mode=None):
    """t4_streams_run over read shards == the reference SeqSet driven by the restated loop, per shard.
    c_mode: shard with the library's t4_shard_reads (what the batch drop-in calls) instead of synth.shard_workload.
    ref = None: compare with the reference's results stored in tests/golden/batch_ref.json.gz (make_batch_ref.py)."""
    lib.check(lib.reset())
    key, w, cfg, off, descs = batch_inputs(lib, seed, n_shards, nclones, npairs, cfg, deal, group, c_mode)
    gold = json.load(gzip.open(BATCH_GOLD))[key]
    n_shards = len(off) - 1
    assert len(gold) == n_shards, ("shards", len(gold), n_shards)
    k = 9
    sets = api.SeqSet.create_many(n_shards, k, lib)
    ret, strands, resc = api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    for j in range(n_shards):
        lo, hi = int(off[j]), int(off[j + 1])
        if ref is not None:
            r = ref.RefSeqSet(k)
            _, rret, rstr, rresc = r.run_descs(cfg, descs[lo:hi].copy(), w.pool, w.names)
            assert (rret == ret[lo:hi]).all(), ("ret", j, np.flatnonzero(rret != ret[lo:hi])[:5])
            assert (rstr == strands[lo:hi]).all(), ("strand", j)
            assert (rresc == resc[lo:hi]).all(), ("rescue", j)
            assert r.output() == sets[j].output(), ("contigs", j)
            assert r.index_checksum() == sets[j].index_checksum(), ("index", j)
            assert r.size() == sets[j].size()
            assert shard_digest(rret, rstr, rresc, r.output(), r.index_checksum(), r.size()) == gold[j], ("stored reference results", j)
        got = shard_digest(ret[lo:hi], strands[lo:hi], resc[lo:hi], sets[j].output(), sets[j].index_checksum(), sets[j].size())
        for f in gold[j]:
            assert got[f] == gold[j][f], (f, j)
    return int((ret >= 0).sum())


def _canon4(h):
    if len(h) == 0:
        return h[:, :4]
    h = h[:, :4]
    return h[np.lexsort((h[:, 1], h[:, 2], h[:, 0], h[:, 3]))]


def _ragged_records(rng, sources, n, kmer=9):
    """Probe records of mixed lengths (shorter than k .. 400 bp: the probe tiles 288 positions), N's, all strand modes."""
    reads, descs = [], np.zeros(n, dtype=synth.READ_DESC)
    off = 0
    for i in range(n):
        src = sources[int(rng.integers(len(sources)))]
        L = int(rng.choice([5, kmer - 1, kmer, kmer + 1, 31, 64, 100, 144, 145, 150, 152, 153, 200, 290, 400]))
        while len(src) < L:
            src = src + sources[int(rng.integers(len(sources)))]
        a = int(rng.integers(0, len(src) - L + 1))
        s = list(src[a:a + L])
        for _ in range(int(rng.integers(0, 4))):
            s[int(rng.integers(L))] = "ACGTN"[int(rng.integers(5))]
        if rng.random() < 0.15:
            p0 = int(rng.integers(L))
            s[p0:p0 + 14] = list("A" * len(s[p0:p0 + 14]))                             # homopolymer: equal consecutive k-mers
        s = "".join(s)
        assert len(s) == L
        if rng.random() < 0.4:
            s = "".join({"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}[c] for c in reversed(s))
        reads.append(s)
        descs[i]["seq_off"] = off
        descs[i]["len"] = L
        descs[i]["barcode"] = -1
        descs[i]["strand_in"] = int(rng.choice([0, 0, 1, -1]))
        off += L
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    return reads, descs, pool


def check_probe_batch(lib, ref, seed=41, n_shards=5, sample=160):
    """t4_streams_get_hits (the grid-wide warp-per-read probe: 2-bit packed reads, directory + postings over frozen sets)
    against SeqSet::GetHitsFromRead of the reference on the same sets: hit multisets per record, for the assembled reads
    of every shard and for ragged records (lengths 5..400, N's, homopolymers, both strands, strand -1/0/+1 modes)."""
    lib.check(lib.reset())
    w = small_workload(seed, 25, 500)
    cfg = synth.run_cfg()
    off, descs = synth.shard_workload(w, n_shards)
    sets = api.SeqSet.create_many(n_shards, 9, lib)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    refs = []
    for j in range(n_shards):
        r = ref.RefSeqSet(9)
        r.run_descs(cfg, descs[int(off[j]):int(off[j + 1])].copy(), w.pool, w.names)
        assert r.index_checksum() == sets[j].index_checksum()
        refs.append(r)
    rng = np.random.default_rng(seed)
    # (1) the workload's own records
    wl = api.Workload(descs, w.pool, w.names, lib)
    hits = api.Hits(len(descs), 4 << 20, lib)
    api.streams_get_hits(sets, wl, off, hits)
    st = hits.stats()
    assert st["records"] == len(descs) and st["hits"] > 1000 and st["unsupported"] == 0
    reads = w.pool[: len(w.descs) * w.L].reshape(-1, w.L)
    total = 0
    for i in rng.choice(len(descs), size=min(sample, len(descs)), replace=False):
        j = int(np.searchsorted(off, i, side="right") - 1)
        d = descs[i]
        rd = bytes(w.pool[int(d["seq_off"]):int(d["seq_off"]) + int(d["len"])]).decode()
        hr = _canon4(refs[j].get_hits(rd, int(d["strand_in"]), int(d["barcode"])))
        hg, _ = hits.fetch(int(i))
        hg = _canon4(hg)
        assert hr.shape == hg.shape and (hr == hg).all(), ("probe", int(i), j, hr.shape, hg.shape)
        total += len(hr)
    assert total > 100
    wl.close()
    # (2) ragged records against the same frozen sets
    srcs = []
    for j in range(n_shards):
        for line in sets[j].output().split(b"\n"):
            if line and line[:1] in b"ACGT" and len(line) > 60 and b" " not in line:
                srcs.append(line.decode())
    assert len(srcs) >= n_shards
    n = 300
    rreads, rdescs, rpool = _ragged_records(rng, srcs, n)
    roff = np.linspace(0, n, n_shards + 1).astype(np.int64)
    wl = api.Workload(rdescs, rpool, [], lib)
    for skip in (0, 1):
        api.streams_get_hits(sets, wl, roff, hits, allow_total_skip=skip)
        st = hits.stats()
        assert st["records"] == n
        nz = 0
        for i in range(n):
            j = int(np.searchsorted(roff, i, side="right") - 1)
            hr = _canon4(refs[j].get_hits(rreads[i], int(rdescs[i]["strand_in"]), -1, bool(skip)))
            hg, _ = hits.fetch(i)
            hg = _canon4(hg)
            assert hr.shape == hg.shape and (hr == hg).all(), ("ragged", i, len(rreads[i]), int(rdescs[i]["strand_in"]), hr.shape, hg.shape)
            nz += len(hr) > 0
        assert nz > n // 3
    wl.close()
    hits.close()


def check_stage_parity(lib, ref, name="synth2k", every=97, max_checks=60):
    """k-mer hits (after SortHits) and scored overlaps of individual reads against a frozen snapshot:
    replay the golden trace on both sides and compare the stage outputs at sampled AddRead calls."""
    lib.check(lib.reset())
    ops = gold_trace(name)
    g = None
    r = None
    checks = 0
    for i, t in enumerate(ops):
        if t[0] == "A" and i % every == 0 and checks < max_checks:
            read, sin = t[1], int(t[3])
            hr = canon_hits(r.get_hits(read, sin))
            hg = g.get_hits(read, sin)
            assert hr.shape == hg.shape and (hr == hg).all(), ("hits", i)
            n1, o1, s1 = r.get_overlaps(read, sin)
            n2, o2, s2 = g.get_overlaps(read, sin)
            assert n1 == n2, ("overlap count", i, n1, n2)
            if n1 > 0:
                assert (o1 == o2).all(), ("overlaps", i)
                assert (s1 == s2).all(), ("similarity", i)   # IEEE doubles, bit-equal
            assert r.index_checksum() == g.index_checksum(), ("index", i)
            checks += 1
        if t[0] == "C":
            g = api.SeqSet(int(t[1]), lib)
            r = ref.RefSeqSet(int(t[1]))
        elif t[0] == "O":
            break
        else:
            tr.replay([t], lambda k: None) if False else None
            _apply(t, r)
            _apply(t, g)
    assert checks > 5


def canon_hits(h):
    """The reference's SortHits (SeqSet.hpp:1306) orders hits by (strand, seqIdx, readOffset) and leaves hits of
    one k-mer on one contig in postings (insertion) order, which nothing downstream observes
    (GetOverlapsFromHits re-sorts every group by diagonal).  Compare in the canonical order
    (strand, seqIdx, readOffset, seqOffset) the C ABI documents."""
    if len(h) == 0:
        return h
    order = np.lexsort((h[:, 1], h[:, 2], h[:, 0], h[:, 3]))
    return h[order]


def _apply(t, s):
    c = t[0]
    if c == "A":
        s.add_read(t[1], "" if t[2] == "." else t[2], int(t[3]), int(t[4]), int(t[5]), int(t[6]), float(t[7]))
    elif c == "R":
        s.repeat_add_read(t[1])
    elif c == "N":
        s.input_novel_read(t[1], t[2], int(t[3]), int(t[4]))
    elif c == "U":
        s.update_all_consensus()
    elif c == "K":
        s.change_kmer_length(int(t[1]))
    elif c == "H":
        s.set_hit_len_required(int(t[1]))


def dp_cases(seed, n=300):
    """Random GlobalAlignment_PosWeight problems: equal and unequal lengths, clean / noisy / indel inputs."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        lent = int(rng.integers(0, 70))
        kind = rng.integers(0, 5)
        t = rng.integers(0, 4, size=lent)
        p = list(t)
        if kind == 0:
            pass
        elif kind == 1:                      # substitutions
            for _ in range(int(rng.integers(1, 6))):
                if p:
                    p[int(rng.integers(len(p)))] = int(rng.integers(4))
        elif kind == 2:                      # an indel
            if len(p) > 3:
                x = int(rng.integers(1, len(p) - 1))
                if rng.random() < 0.5:
                    del p[x]
                else:
                    p.insert(x, int(rng.integers(4)))
        elif kind == 3:                      # unrelated, maybe other length
            p = list(rng.integers(0, 4, size=max(0, lent + int(rng.integers(-4, 5)))))
        else:                                # indel + substitutions, N's
            if len(p) > 6:
                x = int(rng.integers(2, len(p) - 2))
                del p[x:x + int(rng.integers(1, 3))]
                p[int(rng.integers(len(p)))] = 4
        tw = np.zeros((lent, 4), dtype=np.int32)
        for j in range(lent):
            tw[j, t[j]] = int(rng.integers(1, 30))
            if rng.random() < 0.3:
                tw[j, int(rng.integers(4))] += int(rng.integers(0, 12))
            if rng.random() < 0.03:
                tw[j] = 0
        ps = "".join("ACGTN"[c] for c in p)
        out.append((tw, ps))
    return out


def check_dp(lib, ref, seed=5):
    cases = dp_cases(seed)
    got = api.dp_pos_weight_batch(cases, lib)
    for (tw, p), (sc, ed) in zip(cases, got):
        rs, re_ = ref.dp_pos_weight(tw, p)
        assert (sc, ed) == (rs, re_), (tw.tolist(), p, sc, rs, ed, re_)


def dp_equal_cases(seed=11, n=260):
    """Equal-length GlobalAlignment_PosWeight problems as the hot path poses them (overhangs, same-diagonal gaps):
    clean, substitution bursts, frame shifts that an in-band gap pair can repair, N's, mixed-support columns,
    lengths on both sides of the shared-memory limit of the half-warp DP (192)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        L = int(rng.choice([2, 3, 7, 12, 13, 14, 30, 45, 64, 100, 150, 191, 192, 230, 300])) if i % 3 == 0 else int(rng.integers(2, 160))
        t = rng.integers(0, 4, size=L)
        p = list(t)
        kind = int(rng.integers(0, 6))
        if kind == 1:
            for _ in range(int(rng.integers(1, 4))):
                p[int(rng.integers(L))] = int(rng.integers(4))
        elif kind == 2:                      # > 2 substitutions: forces the banded DP, answer stays on the diagonal
            for _ in range(int(rng.integers(3, 9))):
                x = int(rng.integers(L))
                p[x] = (p[x] + 1 + int(rng.integers(3))) % 4
        elif kind == 3 and L > 12:           # delete d bases early, insert d later: a frame shift inside the band
            d = int(rng.integers(1, 5))
            x = int(rng.integers(1, L - d - 4))
            del p[x:x + d]
            y = int(rng.integers(x + 1, len(p)))
            for _ in range(d):
                p.insert(y, int(rng.integers(4)))
        elif kind == 4:                      # unrelated
            p = list(rng.integers(0, 4, size=L))
        elif kind == 5:                      # N's + substitutions
            for _ in range(int(rng.integers(1, 4))):
                p[int(rng.integers(L))] = 4
            for _ in range(int(rng.integers(0, 6))):
                p[int(rng.integers(L))] = int(rng.integers(4))
        assert len(p) == L
        tw = np.zeros((L, 4), dtype=np.int32)
        for j in range(L):
            tw[j, t[j]] = int(rng.integers(1, 30))
            if rng.random() < 0.3:
                tw[j, int(rng.integers(4))] += int(rng.integers(0, 12))
            if rng.random() < 0.03:
                tw[j] = 0
        out.append((tw, "".join("ACGTN"[c] for c in p)))
    return out


def _diag_mismatches(tw, p):
    """Mismatches of the all-diagonal alignment under AlignAlgo::IsBaseEqual (AlignAlgo.hpp:49-55)."""
    x = 0
    for j, c in enumerate(p):
        s = int(tw[j].sum())
        if s == 0 or c == "N":
            continue
        if not s < 3 * int(tw[j, "ACGT".index(c)]):
            x += 1
    return x


def check_dp_hot(lib, ref, seed, variant):
    """The DP routines the stream kernel really runs, against AlignAlgo::GlobalAlignment_PosWeight (AlignAlgo.hpp:57-216):
    score and edit string.  variant 0 = t4_dp_equal (has the reference's <= 2-mismatch fast path), variant 1 =
    w_dp_equal_half (always the banded DP; its caller only invokes it beyond 2 mismatches, so only those cases count)."""
    cases = dp_equal_cases(seed)
    if variant == 1:
        cases = [(tw, p) for tw, p in cases if _diag_mismatches(tw, p) > 2]
        assert len(cases) > 40
    got = api.dp_hot_path_batch(cases, variant, lib)
    for (tw, p), (sc, ed) in zip(cases, got):
        rs, re_ = ref.dp_pos_weight(tw, p)
        assert (sc, ed) == (rs, re_), (variant, len(p), p, sc, rs, ed, re_)


def check_big_repeats(lib, ref, n_copies=10050):
    """A k-mer with more than 10000 postings: the `repeats > 10000` rules of GetOverlapsFromHits, including the
    run-local `hits[k]` indexing slip (SeqSet.hpp:931-947), and the >=100-postings skip rule of GetHitsFromRead."""
    lib.check(lib.reset())
    rng = np.random.default_rng(77)
    base = "".join("ACGT"[c] for c in rng.integers(0, 4, size=120))
    other = "".join("ACGT"[c] for c in rng.integers(0, 4, size=150))
    g = api.SeqSet(9, lib)
    r = ref.RefSeqSet(9)
    # many contigs that all carry the k-mers of `base`; each gets a unique tail so they stay distinct sequences
    tails = ["".join("ACGT"[c] for c in rng.integers(0, 4, size=30)) for _ in range(64)]
    reads = [base + tails[i % 64] for i in range(n_copies)]
    for rd in reads:
        r.input_novel_read("IGHV1-2*01", rd, 1, -1)
        g.input_novel_read("IGHV1-2*01", rd, 1, -1)
    assert g.size() == r.size() == n_copies
    assert g.index_checksum() == r.index_checksum()
    for q in (base[10:110] + other[:50], other[:60] + base[:90], base[:100], other):
        for strand in (0, 1):
            hr = canon_hits(r.get_hits(q, strand))
            hg = g.get_hits(q, strand)
            assert hr.shape == hg.shape and (hr == hg).all()
            if q is not other:
                assert hr[:, 4].max() > 10000      # the scenario really has a k-mer with > 10000 postings
            n1, o1, s1 = r.get_overlaps(q, strand)
            n2, o2, s2 = g.get_overlaps(q, strand)
            assert n1 == n2, (n1, n2)
            if n1 > 0:
                assert (o1 == o2).all() and (s1 == s2).all()
        assert g.add_read(q, "IGHV", 0, -1, 1, 0, 0.9) == r.add_read(q, "IGHV", 0, -1, 1, 0, 0.9)
    assert g.index_checksum() == r.index_checksum()
    # the batch probe on the same set: lists of > 10000 postings (streamed, `repeats > 10000` flag), the >= 100 rules
    qs = [base[10:110] + other[:50], other[:60] + base[:90], base[:100], other, base + other + base[:60]]
    d = np.zeros(2 * len(qs), dtype=synth.READ_DESC)
    o = 0
    for i, q in enumerate(qs + qs):
        d[i]["seq_off"], d[i]["len"], d[i]["barcode"], d[i]["strand_in"] = o, len(q), -1, 0 if i < len(qs) else 1
        o += len(q)
    pool = np.frombuffer(("".join(qs + qs) + "\0" * 16).encode(), dtype=np.uint8).copy()
    wl = api.Workload(d, pool, [], lib)
    hits = api.Hits(len(d), 24 << 20, lib)
    for skip in (0, 1):
        api.streams_get_hits([g], wl, [0, len(d)], hits, allow_total_skip=skip)
        assert hits.stats()["records"] == len(d)       # also raises when the key buffer was too small
        for i, q in enumerate(qs + qs):
            hr = _canon4(r.get_hits(q, int(d[i]["strand_in"]), -1, bool(skip)))
            hg, fl = hits.fetch(i)
            hg = _canon4(hg)
            assert hr.shape == hg.shape and (hr == hg).all(), ("big probe", i, skip)
            if skip == 0 and q is not other:
                assert fl & 1
    wl.close()
    hits.close()


def check_barcode_mode(lib, ref, seed=31, n_barcodes=5):
    """Barcode mode inside one stream (BASELINE configs[3] flavour): barcode-salted index keys
    (KmerIndex.hpp:29-33), per-hit barcode filter and repeats = 1 (SeqSet.hpp:1394-1418), hitLenRequired 13,
    ExtendOverlap mismatch factor 2.0, no periodic consensus update (main.cpp:1549-1560, 1862).
    ReleaseFinishedBarcodeSeq is not part of this path (both sides skip it)."""
    lib.check(lib.reset())
    w = small_workload(seed, 20, 500)
    d = w.descs.copy()
    L = w.L
    reads = w.pool.reshape(-1, L)
    h = (reads.astype(np.int64) * np.arange(1, L + 1)).sum(axis=1)
    d["barcode"] = (h % n_barcodes).astype(np.int32)
    d["sim_threshold"] = 0.9
    d["mate_idx"] = -1
    cfg = synth.run_cfg(has_barcode=1)
    g = api.SeqSet(9, lib)
    r = ref.RefSeqSet(9)
    for s in (g, r):
        s.set_hit_len_required(13)
    g.set_consider_barcode_in_hash(1)
    ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
    _, gret, gstr, gres = g.run_descs(cfg, d, w.pool, w.names)
    _, rret, rstr, rres = r.run_descs(cfg, d, w.pool, w.names)
    assert (gret == rret).all() and (gstr == rstr).all() and (gres == rres).all()
    assert g.output() == r.output()
    assert g.index_checksum() == r.index_checksum()
    assert len(set(c["barcode"] for c in (g.get_contig(i) for i in range(g.size())) if c)) > 1


def _barcode_descs(seed, n_barcodes=3, nclones=6, npairs=400):
    """A barcode-sorted record list (main.cpp:1126 CompReadWithBarcode order) over a small synthetic library."""
    cl = synth.make_clones(nclones, seed)
    rd = synth.sample_pairs(cl, npairs, 150, seed)
    w = synth.build_workload(cl, rd)
    d = w.descs.copy()
    reads = w.pool.reshape(-1, w.L)
    h = (reads.astype(np.int64) * np.arange(1, w.L + 1)).sum(axis=1) % n_barcodes
    order = np.argsort(h, kind="stable")
    d = d[order]
    d["barcode"] = h[order].astype(np.int32)
    d["mate_idx"] = -1
    d["sim_threshold"] = 0.9
    n = len(d)
    same_prev = np.zeros(n, dtype=bool)
    rs = reads[order]
    same_prev[1:] = (rs[1:] == rs[:-1]).all(axis=1) & (d["barcode"][1:] == d["barcode"][:-1])
    d["flags"] = np.where(same_prev, d["flags"] | synth.RD_DUP, d["flags"] & ~np.uint32(synth.RD_DUP))
    d["eq_lo"] = np.arange(n)
    d["eq_hi"] = np.arange(n) + 1
    return w, d


def _same_sets(g, r):
    assert g.size() == r.size()
    assert g.output() == r.output()
    assert g.index_checksum() == r.index_checksum()
    for i in range(g.size()):
        gc = g.get_contig(i)
        assert (gc is None) == (r.num_read(i) < 0), i
        if gc is not None:
            assert gc["num_read"] == r.num_read(i), i


def check_barcode_release(lib, ref, seed=33):
    """SeqSet::ReleaseFinishedBarcodeSeq (SeqSet.hpp:10815; driver main.cpp:1846-1859: only reads with addRet >= 0 count
    towards "finished"), ReleaseShallowContigs (SeqSet.hpp:10928) and IsContigShallow (:2512): inside the batch loop
    (cfg.release_barcodes, contig_min_cov 0 / 2 / 20) and through the per-call entries, against the reference --
    Output text, slot count, numRead of every slot and the index multiset (purged contigs leave the index)."""
    w, d = _barcode_descs(seed)
    base_sum = None
    for min_cov in (0, 2, 20):
        lib.check(lib.reset())
        outs = []
        for release in (0, 1):
            cfg = synth.run_cfg(has_barcode=1, release_barcodes=release, contig_min_cov=min_cov)
            r = ref.RefSeqSet(9)
            r.set_hit_len_required(13)
            ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
            _, rret, rstr, rres = r.run_descs(cfg, d, w.pool, w.names)
            g = api.SeqSet(9, lib)
            g.set_hit_len_required(13)
            g.set_consider_barcode_in_hash(1)
            _, gret, gstr, gres = g.run_descs(cfg, d, w.pool, w.names)
            assert (gret == rret).all() and (gstr == rstr).all() and (gres == rres).all()
            _same_sets(g, r)
            outs.append((r.output(), r.index_checksum()[0]))
            if release == 1 and min_cov > 0:
                # --contigMinCov: the driver's last step before Output (main.cpp:1952-1955)
                r.release_shallow_contigs(min_cov)
                g.release_shallow_contigs(min_cov)
                assert g.output() == r.output()
                assert g.size() == r.size()
                outs.append((r.output(), 0))
        if min_cov == 0:
            assert outs[1][1] < outs[0][1]       # the purge really happened: postings left the index ...
            assert outs[0][0] == outs[1][0]      # ... and is invisible in Output when nothing is shallow
            assert len(outs[0][0]) > 1000
        if min_cov == 20:
            assert 0 < len(outs[1][0]) < len(outs[0][0])    # shallow contigs were dropped inside the loop, deep ones stayed
    # per-call route, like the driver: assemble one barcode, purge it (the purge walks the slots from the end and stops at
    # the first contig of another barcode or an already purged one), go on with the next
    lib.check(lib.reset())
    cfg = synth.run_cfg(has_barcode=1, final_update=0, do_rescue=0)
    r = ref.RefSeqSet(9)
    r.set_hit_len_required(13)
    ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
    g = api.SeqSet(9, lib)
    g.set_hit_len_required(13)
    g.set_consider_barcode_in_hash(1)
    for bc, cov in ((0, 0), (1, 20), (2, 2)):
        part = d[d["barcode"] == bc].copy()
        part["flags"][0] &= ~np.uint32(synth.RD_DUP)
        _, rret, _, _ = r.run_descs(cfg, part, w.pool, w.names)
        _, gret, _, _ = g.run_descs(cfg, part, w.pool, w.names)
        assert (gret == rret).all()
        if bc == 2:
            r.release_finished_barcode(1, 0)     # stops at once: the tail belongs to barcode 2
            g.release_finished_barcode(1, 0)
            _same_sets(g, r)
        r.release_finished_barcode(bc, cov)
        g.release_finished_barcode(bc, cov)
        _same_sets(g, r)
    purged = [g.contig_flags(i) for i in range(g.size())]
    assert 1 in purged and -1 in purged      # purged contigs and (barcode 1, cov 20) dropped ones
    # a purged set survives UpdateAllConsensus and ChangeKmerLength (Clean skips contigs with index == false)
    r.update_all_consensus()
    g.update_all_consensus()
    _same_sets(g, r)


def check_single_cell(lib, ref, seed=51, n_barcodes=24, reads_per_barcode=150, n_shards=5, contig_min_cov=0):
    """BASELINE configs[3] in small: 10x-style barcoded single-end reads, whole barcodes per stream (SURVEY.md 8e),
    hitLenRequired 13, barcode-salted index, finished barcodes purged -- per stream against the reference SeqSet driven
    by the restated loop (return codes, strands, rescue codes, Output with barcode slots, index multiset, numRead)."""
    lib.check(lib.reset())
    cl = synth.make_clones(60, seed)
    rd, bc = synth.sample_single_cell(cl, n_barcodes, reads_per_barcode, 150, seed)
    w = synth.build_workload(cl, rd, barcode=bc)
    cfg = synth.run_cfg(has_barcode=1, release_barcodes=1, contig_min_cov=contig_min_cov)
    off, descs = synth.shard_workload(w, n_shards, align="barcode")
    for j in range(1, n_shards):     # no barcode straddles two streams
        assert descs["barcode"][off[j] - 1] != descs["barcode"][off[j]]
    sets = api.SeqSet.create_many(n_shards, 9, lib, hit_len_required=13, consider_barcode=1)
    ret, strands, resc = api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    total = 0
    for j in range(n_shards):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(9)
        r.set_hit_len_required(13)
        ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
        _, rret, rstr, rresc = r.run_descs(cfg, descs[lo:hi].copy(), w.pool, w.names)
        assert (rret == ret[lo:hi]).all(), ("ret", j, np.flatnonzero(rret != ret[lo:hi])[:5])
        assert (rstr == strands[lo:hi]).all() and (rresc == resc[lo:hi]).all(), ("strand/rescue", j)
        _same_sets(sets[j], r)
        total += int((rret >= 0).sum())
    assert total > n_barcodes * reads_per_barcode // 2
    return total


def check_repseq(lib, ref, seed=61, n_reads=4000, n_shards=3):
    """BASELINE configs[4] in small: --repseq (trimLevel 2) amplicon TCR-seq reads, 100 bp single end: repetitiveData = true
    (skip-repeats first pass SeqSet.hpp:1520-1531, ExtendOverlap mismatch factor 2.0 :1226-1237), V-gene pseudo barcodes
    on an unsalted index (main.cpp:1224-1235), halved k-change threshold (main.cpp:1567)."""
    lib.check(lib.reset())
    cl = synth.make_clones(120, seed, chains=("TRB",))
    rd = synth.sample_amplicon(cl, n_reads, 100, seed)
    w = synth.build_workload(cl, rd, repseq=True)
    assert (w.descs["barcode"] >= 0).mean() > 0.5
    cfg = synth.run_cfg(repetitive=1, change_k_threshold=40, first_read_len=100)      # small threshold: k changes mid-run
    off, descs = synth.shard_workload(w, n_shards)
    sets = api.SeqSet.create_many(n_shards, 9, lib, hit_len_required=50)           # main.cpp:1541-1547: max(21, L/2) when L/2 < 31 -> here L/2 = 50 > 31 keeps 31; exercise the setter anyway
    for s_ in sets:
        s_.set_hit_len_required(31)
    ret, strands, resc = api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    for j in range(n_shards):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(9)
        _, rret, rstr, rresc = r.run_descs(cfg, descs[lo:hi].copy(), w.pool, w.names)
        assert (rret == ret[lo:hi]).all(), ("ret", j, np.flatnonzero(rret != ret[lo:hi])[:5])
        assert (rstr == strands[lo:hi]).all() and (rresc == resc[lo:hi]).all(), ("strand/rescue", j)
        assert r.output() == sets[j].output(), ("contigs", j)
        assert r.index_checksum() == sets[j].index_checksum(), ("index", j)
        assert r.kmer_length() == sets[j].kmer_length()
    assert int((ret >= 0).sum()) > n_reads // 2


def check_dup_runs(lib, ref, seed=71):
    """Long runs of duplicate records (amplicon data: every read of a clonotype is the same string): the device applies a
    run of RepeatAddRead calls in one pass; the periodic UpdateAllConsensus (here every 37 assembled reads) and a pending
    k change must still see exactly the reference's state."""
    lib.check(lib.reset())
    cl = synth.make_clones(7, seed, chains=("TRB",))
    rd = synth.sample_amplicon(cl, 6000, 100, seed, alpha=0.7, sub_rate=0.001)
    w = synth.build_workload(cl, rd, repseq=True)
    assert (w.descs["flags"] & synth.RD_DUP).mean() > 0.8
    for every, chk in ((37, 4096), (10000, 3), (5000, 4096)):
        lib.check(lib.reset())
        cfg = synth.run_cfg(repetitive=1, change_k_threshold=chk, update_consensus_every=every, first_read_len=100)
        g = api.SeqSet(9, lib)
        r = ref.RefSeqSet(9)
        _, gret, gstr, gres = g.run_descs(cfg, w.descs, w.pool, w.names)
        _, rret, rstr, rres = r.run_descs(cfg, w.descs, w.pool, w.names)
        assert (gret == rret).all() and (gstr == rstr).all() and (gres == rres).all(), (every, chk)
        assert g.output() == r.output(), (every, chk)
        assert g.index_checksum() == r.index_checksum() and g.kmer_length() == r.kmer_length()
        for i in range(g.size()):
            c = g.get_contig(i)
            assert (c is None) == (r.num_read(i) < 0) and (c is None or c["num_read"] == r.num_read(i))


def check_input_novel_fa(lib, ref, tmp_path):
    """SeqSet::InputNovelFa (SeqSet.hpp:2986, --debug-ns)."""
    lib.check(lib.reset())
    rng = np.random.default_rng(3)
    fa = tmp_path / "ns.fa"
    with open(fa, "w") as f:
        for i in range(7):
            s = "".join("ACGT"[c] for c in rng.integers(0, 4, size=int(rng.integers(40, 400))))
            f.write(">ns%d some comment\n" % i)
            for j in range(0, len(s), 60):
                f.write(s[j:j + 60] + "\n")
    r = ref.RefSeqSet(9)
    g = api.SeqSet(9, lib)
    r.input_novel_fa(str(fa))
    assert g.input_novel_fa(str(fa)) == 7
    assert g.output() == r.output() and len(g.output()) > 500
    assert g.index_checksum() == r.index_checksum()


def _run_resident(lib, sets, cfg, wl, off):
    hs = (api.C.c_void_p * len(sets))(*[s.h for s in sets])
    off = np.ascontiguousarray(off, dtype=np.int64)
    lib.check(lib.streams_run_resident(hs, len(sets), cfg.ctypes.data, wl.h, off.ctypes.data, None))
    n = wl.n
    ret = np.zeros(n, dtype=np.int32)
    strands = np.zeros(n, dtype=np.int8)
    resc = np.zeros(n, dtype=np.int32)
    lib.check(lib.workload_results(wl.h, ret.ctypes.data, strands.ctypes.data, resc.ctypes.data))
    return ret, strands, resc


def check_assign_pass(lib, ref, seed, n_shards, nclones=25, npairs=400, kmer=17, group="", workload=None, cfg=None, n_workers=0,
                      drop=0.0):
    """t4_streams_assign_reads (SURVEY.md 8f-2) against the reference's own pass (main.cpp:2047-2118): for every shard the
    extended set built by InputSeqSet at k, AssignRead of every assembled read in the driver's order (identical
    neighbours share a call) with novelSeqSimilarity 0.95, and RecomputePosWeight -- per read the assigned contig,
    coordinates, strand, matchCnt and the similarity double; per extended set the Output text (consensus + recomputed
    posWeight) and the index checksum."""
    lib.check(lib.reset())
    w = workload if workload is not None else small_workload(seed, nclones, npairs)
    cfg = cfg if cfg is not None else synth.run_cfg()
    off, descs = synth.shard_workload(w, n_shards, balance="cost" if group else "reads", group=group)
    n_shards = len(off) - 1
    if drop > 0:   # reads the driver's gene-order / constant-gene filters reject (main.cpp:1609-1654): never assembled, never listed
        descs = descs.copy()
        rng = np.random.default_rng(seed)
        descs["flags"] |= np.where(rng.random(len(descs)) < drop, synth.RD_FILTERED, 0).astype(descs["flags"].dtype)
    sets = api.SeqSet.create_many(n_shards, 9, lib)
    wl = api.Workload(descs, w.pool, w.names, lib)
    ret, strands, resc = _run_resident(lib, sets, cfg, wl, off)
    a = api.Assign(sets, wl, off, kmer, n_workers=n_workers)
    ga, gs = a.results()
    st = a.stats()
    n_listed = n_assigned = n_calls = 0
    for j in range(n_shards):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(9)
        d = descs[lo:hi].copy()
        _, rret, rstr, rresc = r.run_descs(cfg, d, w.pool, w.names)
        assert (rret == ret[lo:hi]).all() and (rstr == strands[lo:hi]).all() and (rresc == resc[lo:hi]).all(), ("assembly", j)
        lst = ref.assembled_list(rret, rresc)
        ext, ra, rs = ref.assign_pass(r, kmer, d, w.pool, lst, rstr)
        listed = np.zeros(hi - lo, dtype=bool)
        listed[lst] = True
        assert (ga[lo:hi][~listed, 0] == api.ASSIGN_NOT_LISTED).all(), ("not listed", j)
        g = ga[lo:hi][lst]
        assert (g[:, 0] == ra[:, 0]).all(), ("seqIdx", j, np.flatnonzero(g[:, 0] != ra[:, 0])[:5])
        ok = ra[:, 0] >= 0
        assert (g[ok] == ra[ok]).all(), ("overlap", j, np.flatnonzero((g[ok] != ra[ok]).any(axis=1))[:5])
        assert (gs[lo:hi][lst][ok] == rs[ok]).all(), ("similarity", j)
        ge = a.extended_set(j)
        assert ge.kmer_length() == kmer and ge.size() == ext.size()
        assert ge.output() == ext.output(), ("extended set", j)
        assert ge.index_checksum() == ext.index_checksum(), ("extended index", j)
        n_listed += len(lst)
        n_assigned += int(ok.sum())
        rd = [bytes(w.pool[int(x["seq_off"]):int(x["seq_off"]) + int(x["len"])]) for x in d[lst]]
        n_calls += sum(1 for i in range(len(rd)) if i == 0 or rd[i] != rd[i - 1])
    assert st["reads"] == n_listed and st["assigned"] == n_assigned and st["assign_calls"] == n_calls, (st, n_listed, n_assigned, n_calls)
    a.close()
    wl.close()
    return n_listed, n_assigned


def check_kmer_count_stats(lib, ref, seed=101, n=1500, k=21):
    """t4_kmer_count_stats (SURVEY.md 8f-3) against the reference's KmerCount: AddCount of every read, then
    GetCountStatsAndTrim without trimming -- min / median exact, avg the same float.  Reads: sampled pairs of a clone set
    (shared k-mers with high counts) plus ragged ones: lengths 5..400, N's, reads of N's only, homopolymers, duplicates."""
    rng = np.random.default_rng(seed)
    cl = synth.make_clones(30, seed)
    rd = synth.sample_pairs(cl, n // 3, 150, seed, sub_rate=0.01)
    reads = [synth.decode(c) for c in rd.codes]
    src = reads[: 50]
    while len(reads) < n:
        s = src[int(rng.integers(len(src)))]
        L = int(rng.integers(5, 401))
        t = (s * 4)[int(rng.integers(0, 100)):][:L]
        kind = int(rng.integers(0, 8))
        if kind == 0:
            t = "N" * L
        elif kind == 1:
            t = "ACGT"[int(rng.integers(4))] * L
        elif kind in (2, 3):
            t = list(t)
            for p in rng.integers(0, L, size=int(rng.integers(1, 6))):
                t[int(p)] = "N"
            t = "".join(t)
        elif kind == 4 and len(reads) > 3:
            t = reads[int(rng.integers(len(reads)))]
        reads.append(t)
    lens = np.array([len(r) for r in reads], dtype=np.int32)
    off = np.zeros(len(reads), dtype=np.uint64)
    off[1:] = np.cumsum(lens[:-1])
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    # qualities: mostly good; a third of the N-free reads get a bad tail (Phred <= 15 from some position on, some sparse,
    # some whole reads) so that the trimming rules fire: cut positions, reads cut below k (dropped), untouched reads
    quals = []
    for t in reads:
        q = ["I"] * len(t)
        if "N" not in t and len(t) > 30 and rng.random() < 0.35:
            mode = int(rng.integers(0, 4))
            st = int(rng.integers(0, len(t))) if mode != 3 else 0
            for p in range(st, len(t)):
                if mode == 1 and rng.random() < 0.5:
                    continue
                q[p] = "#$%&'()*+,-./0"[int(rng.integers(0, 14))]     # Phred 2..15
            if mode == 2:
                q[-1] = "I"
        quals.append("".join(q))
    qpool = np.frombuffer(("".join(quals) + "\0" * 16).encode(), dtype=np.uint8).copy()
    n_trim = 0
    for qp in (None, qpool):
        rmn, rmed, ravg, rnl = ref.kmer_count_stats(pool, off, lens, k, qual=qp)
        gmn, gmed, gavg, gnl = api.kmer_count_stats(pool, off, lens, k, lib, qual=qp)
        assert (gnl == rnl).all(), ("new length", qp is not None, np.flatnonzero(gnl != rnl)[:5])
        assert (gmn == rmn).all(), ("min", qp is not None, np.flatnonzero(gmn != rmn)[:5])
        assert (gmed == rmed).all(), ("median", qp is not None, np.flatnonzero(gmed != rmed)[:5])
        assert (gavg.view(np.uint32) == ravg.view(np.uint32)).all(), ("avg", qp is not None, np.flatnonzero(gavg.view(np.uint32) != ravg.view(np.uint32))[:5])
        if qp is None:
            assert (rnl == lens).all()
            assert (rmn < 0).sum() > 10 and (rmn == 0).sum() > 10 and (rmn > 1).sum() > 100 and rmed.max() > 20
        else:
            n_trim = int((rnl < lens).sum())
            assert n_trim > 50 and ((rnl == 0) & (lens >= k)).sum() > 3
    return int(len(reads))


def write_gene_fasta(path, messy=True):
    """The bundled gene pool as FASTA; `messy` adds what InputRefFa has to clean up: IMGT '.' gaps, lower case, ambiguity
    codes, a duplicated sequence under another name, the same record twice, a '/OR' pseudo-gene, multi-line records."""
    pool = synth.load_gene_pool()
    recs = []
    for ch in pool.values():
        for seg in ch.values():
            for name, seq in seg:
                recs.append((name, seq))
    out = []
    for i, (name, seq) in enumerate(recs):
        s = seq
        if messy and i % 7 == 0:
            s = s[:30] + "..." + s[30:60] + "......" + s[60:]
        if messy and i % 11 == 0 and len(s) > 80:
            s = s[:70] + s[70:75].lower() + s[75:]
        if messy and i % 13 == 0 and len(s) > 90:
            s = s[:85] + "RY" + s[87:]
        out.append((name, s))
    if messy:
        out.insert(5, ("IGHV9-99*01 extra words", recs[2][1]))                 # same sequence as another gene: names joined
        out.insert(9, (recs[3][0], recs[3][1]))                                 # the same record again: dropped
        out.insert(12, ("IGHV3/OR16-9*01", recs[20][1][:200] + "ACGTACGTTTGACCA"))  # /OR pseudo-gene: skipped
        out.insert(14, ("TRBD1*01", "GGGACAGGGGGC"))                            # D genes are kept (short: below k + a few)
    with open(path, "w") as f:
        for name, s in out:
            f.write(">%s\n" % name)
            for p in range(0, len(s), 60):
                f.write(s[p:p + 60] + "\n")
    return recs


def check_refset_scan(lib, ref, tmp_path, seed=121, n=1200, radius=None, hit_len=27, k=9):
    """t4_refset_create_from_fa + t4_refset_scan (SURVEY.md 8f-4) against the reference: InputRefFa (kept sequences, joined
    names, the k-mer index) and, per read, IsLowComplexity and HasHitInSet(read, 0) -- candidate reads from clonotypes on both
    strands, random reads, chimeras of a gene piece and random sequence, reads with N's, low-complexity reads, short reads,
    reads with indels against the gene (several diagonals inside the radius)."""
    rng = np.random.default_rng(seed)
    fa = os.path.join(str(tmp_path), "genes_%d.fa" % seed)
    recs = write_gene_fasta(fa)
    lib.check(lib.reset())
    g = api.RefSet(fa, k, lib, hit_len_required=hit_len)
    r = ref.RefGeneSet(fa, k, hit_len_required=hit_len)
    if radius is not None:
        g.set_radius(radius)
        r.set_radius(radius)
    assert g.names() == r.names() and g.size() > 100
    assert g.seqset().index_checksum() == r.index_checksum()
    cl = synth.make_clones(40, seed)
    rd = synth.sample_pairs(cl, 200, 150, seed, sub_rate=0.02)
    reads = [synth.decode(c) for c in rd.codes]
    comp = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
    genes = [s for _, s in recs if len(s) > 200]

    def rnd(L):
        return "".join("ACGT"[c] for c in rng.integers(0, 4, size=L))

    while len(reads) < n:
        kind = int(rng.integers(0, 10))
        L = int(rng.integers(20, 260))
        gs = genes[int(rng.integers(len(genes)))]
        p = int(rng.integers(0, max(1, len(gs) - 60)))
        piece = gs[p:p + L]
        if kind == 0:
            t = rnd(L)
        elif kind == 1:
            t = piece[: max(10, len(piece) // 3)] + rnd(L)
        elif kind == 2:
            t = rnd(L // 2) + piece[: 20 + int(rng.integers(0, 40))] + rnd(L // 3)
        elif kind == 3:
            t = "".join(comp[c] for c in reversed(piece))
        elif kind == 4:
            t = list(piece)
            for q in rng.integers(0, max(1, len(t)), size=int(rng.integers(1, 8))):
                t[int(q)] = "N"
            t = "".join(t)
        elif kind == 5:
            t = "ACGT"[int(rng.integers(4))] * (L // 2) + piece[: L // 3]
        elif kind == 6:     # indels: deletions / insertions of 1-6 bases move the chain across neighbouring diagonals
            t = piece
            for _ in range(int(rng.integers(1, 4))):
                q = int(rng.integers(5, max(6, len(t) - 5)))
                d = int(rng.integers(1, 7))
                t = t[:q] + (rnd(d) if rng.random() < 0.5 else "") + t[q + (d if rng.random() < 0.5 else 0):]
        elif kind == 7:
            t = piece[: int(rng.integers(5, 30))]
        elif kind == 8:     # two genes in one read
            g2 = genes[int(rng.integers(len(genes)))]
            t = piece[: L // 2] + g2[-(L // 2):]
        else:
            t = piece
        if len(t) < 1:
            t = "A"
        reads.append(t[:400])
    lens = np.array([len(x) for x in reads], dtype=np.int32)
    off = np.zeros(len(reads), dtype=np.uint64)
    off[1:] = np.cumsum(lens[:-1])
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    gs_, gl_, st = g.scan(pool, off, lens)
    rs_ = np.array([r.has_hit_in_set(x, 0) for x in reads], dtype=np.int8)
    rl_ = np.array([ref.is_low_complexity(x) for x in reads], dtype=np.uint8)
    assert (gl_ == rl_).all(), ("low complexity", np.flatnonzero(gl_ != rl_)[:5])
    assert (gs_ == rs_).all(), ("HasHitInSet", np.flatnonzero(gs_ != rs_)[:8], gs_[gs_ != rs_][:8], rs_[gs_ != rs_][:8])
    assert st["with_hit"] == int((rs_ != 0).sum()) and st["low_complexity"] == int(rl_.sum())
    assert (rs_ == 1).sum() > 50 and (rs_ == -1).sum() > 50 and (rs_ == 0).sum() > 50 and rl_.sum() > 10
    g.close()
    return int((rs_ != 0).sum())


def check_refset_overlaps(lib, ref, tmp_path, seed=131, n=500, radius=None, hit_len=31, k=9):
    """t4_refset_get_overlaps against SeqSet::GetOverlapsFromRead(read, 0, -1, 0, false) on the reference's gene set (the call
    AnnotateRead makes per read): every overlap's gene, coordinates, strand, matchCnt, indelCnt and the similarity double,
    in order.  Reads: clonotype reads (V + junction + J + C: several genes per read), gene pieces with substitutions and
    indels (gaps scored by the affine GlobalAlignment), chimeras, reverse strands, short V-end / J-start reads (the
    GetVJOverlapsFromHits rescue), random reads."""
    rng = np.random.default_rng(seed)
    fa = os.path.join(str(tmp_path), "genes_o%d.fa" % seed)
    recs = write_gene_fasta(fa)
    lib.check(lib.reset())
    g = api.RefSet(fa, k, lib, hit_len_required=hit_len)
    r = ref.RefGeneSet(fa, k, hit_len_required=hit_len)
    if radius is not None:
        g.set_radius(radius)
        r.set_radius(radius)
    cl = synth.make_clones(30, seed)
    rd = synth.sample_pairs(cl, n // 4, 150, seed, sub_rate=0.02)
    reads = [synth.decode(c) for c in rd.codes]
    comp = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
    byname = dict(recs)
    vjs_v = [(nm, s) for nm, s in recs if len(nm) > 3 and nm[3] == "V" and len(s) > 250]
    vjs_j = [(nm, s) for nm, s in recs if len(nm) > 3 and nm[3] == "J" and len(s) > 35]
    genes = [s for _, s in recs if len(s) > 200]

    def rnd(L):
        return "".join("ACGT"[c] for c in rng.integers(0, 4, size=L))

    def mutate(t, subs, indels):
        t = list(t)
        for _ in range(subs):
            q = int(rng.integers(0, len(t)))
            t[q] = "ACGT"[int(rng.integers(4))]
        t = "".join(t)
        for _ in range(indels):
            q = int(rng.integers(12, max(13, len(t) - 12)))
            d = int(rng.integers(1, 5))
            t = t[:q] + (rnd(d) if rng.random() < 0.5 else "") + t[q + (d if rng.random() < 0.5 else 0):]
        return t

    while len(reads) < n:
        kind = int(rng.integers(0, 8))
        gs = genes[int(rng.integers(len(genes)))]
        L = int(rng.integers(60, 220))
        p = int(rng.integers(0, max(1, len(gs) - 80)))
        piece = gs[p:p + L]
        if kind == 0:
            t = mutate(piece, int(rng.integers(0, 6)), 0)
        elif kind == 1:
            t = mutate(piece, int(rng.integers(0, 4)), int(rng.integers(1, 4)))
        elif kind == 2:     # V end + random junction + J start of one chain type: the short-anchor rescue (GetVJOverlapsFromHits)
            vn, v = vjs_v[int(rng.integers(len(vjs_v)))]
            cand = [x for x in vjs_j if x[0][:3] == vn[:3]] or vjs_j
            j = cand[int(rng.integers(len(cand)))][1]
            t = v[-int(rng.integers(18, 30)):] + rnd(int(rng.integers(3, 15))) + j[: int(rng.integers(18, 30))]
        elif kind == 3:
            t = "".join(comp[c] for c in reversed(mutate(piece, 2, int(rng.integers(0, 2)))))
        elif kind == 4:
            t = rnd(L)
        elif kind == 5:
            g2 = genes[int(rng.integers(len(genes)))]
            t = piece[: L // 2] + g2[-(L // 2):]
        elif kind == 6:     # a long unmatched stretch between two anchors of the same gene: gap alignment
            q = min(len(piece) - 30, 40)
            t = piece[:q] + mutate(piece[q:q + 40], 12, 0) + piece[q + 40:]
        else:
            t = piece
        reads.append(t[:400] if len(t) >= 1 else "A")
    n_ovl = n_reads = n_vj = n_indel = 0
    for i, t in enumerate(reads):
        gn, go, gsim = g.get_overlaps(t)
        rn, ro, rsim = r.get_overlaps(t, 0, -1, False)
        assert gn == rn, ("count", i, gn, rn, t)
        if rn > 0:
            assert (go == ro).all(), ("overlap", i, go[(go != ro).any(axis=1)][:2], ro[(go != ro).any(axis=1)][:2], t)
            assert (gsim == rsim).all(), ("similarity", i)
            n_ovl += rn
            n_reads += 1
            n_indel += int((ro[:, 7] > 0).any())
    assert n_reads > n // 3 and n_ovl > n and (n_indel > 5 or radius == 0), (n_reads, n_ovl, n_indel)
    g.close()
    return n_ovl


def annotate_reads(recs, n, seed):
    """Reads for the rough annotation: clonotype reads (V + junction + J + C in one read), mutated gene pieces, V/J-only ends,
    reverse strands, chimeras of two chains (one chain per read rule), random reads, reads cut into several contigs by runs
    of N's, short constant-gene matches.  recs: the (name, sequence) list write_gene_fasta returns."""
    rng = np.random.default_rng(seed)
    cl = synth.make_clones(60, seed)
    rd = synth.sample_pairs(cl, n // 3, 150, seed, sub_rate=0.02)
    reads = [synth.decode(c) for c in rd.codes]
    comp = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
    genes = [s for _, s in recs if len(s) > 200]
    cgenes = [s for nm, s in recs if len(nm) > 3 and nm[3] not in "VDJ" and len(s) > 150]
    src = list(reads)

    def rnd(L):
        return "".join("ACGT"[c] for c in rng.integers(0, 4, size=L))

    while len(reads) < n:
        kind = int(rng.integers(0, 8))
        base = src[int(rng.integers(len(src)))]
        gs = genes[int(rng.integers(len(genes)))]
        p = int(rng.integers(0, max(1, len(gs) - 80)))
        piece = gs[p:p + int(rng.integers(60, 200))]
        if kind == 0:       # a run of N's splits the read into contigs
            q = int(rng.integers(20, len(base) - 30))
            t = base[:q] + "N" * int(rng.integers(7, 15)) + base[q + 10:]
        elif kind == 1:     # sparse N's: still one contig
            t = list(base)
            for q in rng.integers(0, len(t), size=int(rng.integers(1, 6))):
                t[int(q)] = "N"
            t = "".join(t)
        elif kind == 2:
            t = "".join(comp[c] for c in reversed(base))
        elif kind == 3:     # two chains in one read
            o = src[int(rng.integers(len(src)))]
            t = base[:75] + o[75:]
        elif kind == 4:
            t = rnd(int(rng.integers(40, 200)))
        elif kind == 5:     # V or J piece followed by a short constant-gene piece deep inside the gene
            c = cgenes[int(rng.integers(len(cgenes)))]
            q = int(rng.integers(100, max(101, len(c) - 45)))
            t = piece[:90] + c[q:q + int(rng.integers(30, 45))]
        elif kind == 6:
            t = piece
        else:
            t = base[: int(rng.integers(30, 100))]
        reads.append(t[:400])
    return reads[:n]


def reads_pool(reads):
    """(pool, seq_off, lens) of a list of str / bytes reads laid end to end."""
    rb = [x if isinstance(x, bytes) else x.encode() for x in reads]
    lens = np.array([len(x) for x in rb], dtype=np.int32)
    off = np.zeros(len(rb), dtype=np.uint64)
    if len(rb) > 1:
        off[1:] = np.cumsum(lens[:-1])
    pool = np.frombuffer(b"".join(rb) + b"\0" * 16, dtype=np.uint8).copy()
    return pool, off, lens


def compare_annotations(go, gsim, reads, ann, tag=""):
    """t4_refset_annotate's output for `reads` against the reference's AnnotateRead results `ann` (one (int32[4, 8],
    similarity[4]) pair per read); returns how many gene entries per type V, D, J, C are set."""
    assert len(go) == len(reads) == len(ann), (tag, len(go), len(reads), len(ann))
    n_set = np.zeros(4, dtype=np.int64)
    for i, t in enumerate(reads):
        ro, rsim = ann[i]
        assert (go[i][:, 0] == ro[:, 0]).all(), ("gene", tag, i, go[i][:, 0], ro[:, 0], t)
        for tt in range(4):
            if ro[tt, 0] >= 0:
                assert (go[i][tt] == ro[tt]).all() and gsim[i][tt] == rsim[tt], ("overlap", tag, i, tt, go[i][tt], ro[tt], gsim[i][tt], rsim[tt], t)
                n_set[tt] += 1
            else:
                assert go[i][tt][5] == 1, (tag, i)       # strand of an unset entry
    return n_set


def check_refset_annotate(lib, ref, tmp_path, seed=141, n=600, radius=None, hit_len=31, k=9):
    """t4_refset_annotate against SeqSet::AnnotateRead(read, 0, geneOverlap, NULL, NULL) -- the rough annotation the stage-1
    driver runs on every read (main.cpp:1084-1120): per gene type V / D / J / C the chosen gene, coordinates, strand, matchCnt,
    indelCnt, similarity.  Reads: see annotate_reads."""
    fa = os.path.join(str(tmp_path), "genes_a%d.fa" % seed)
    recs = write_gene_fasta(fa)
    lib.check(lib.reset())
    g = api.RefSet(fa, k, lib, hit_len_required=hit_len)
    r = ref.RefGeneSet(fa, k, hit_len_required=hit_len)
    if radius is not None:
        g.set_radius(radius)
        r.set_radius(radius)
    reads = annotate_reads(recs, n, seed)
    go, gsim = g.annotate(*reads_pool(reads))
    n_set = compare_annotations(go, gsim, reads, [r.annotate_read(t) for t in reads])
    assert n_set[0] > n // 5 and n_set[2] > n // 20 and n_set[3] > n // 10, n_set
    g.close()
    return int(n_set.sum())


def check_sort_reads(lib, ref, seed=151, n=5000):
    """t4_sort_reads against std::sort with the driver's _sortRead::operator< (main.cpp:103-125, 1078): reads with their real
    k-mer statistics plus adversarial ties -- equal statistics with different strings, prefixes of each other, identical
    reads under different ids (mates, the '.1' copies), negative statistics, N's."""
    rng = np.random.default_rng(seed)
    cl = synth.make_clones(40, seed)
    rd = synth.sample_pairs(cl, n // 4, 150, seed, sub_rate=0.01)
    reads = [synth.decode(c) for c in rd.codes]
    ids = ["r%d" % (i // 2) for i in range(len(reads))]                 # mates share an id (main.cpp:1069)
    src = list(reads)
    while len(reads) < n:
        kind = int(rng.integers(0, 6))
        s = src[int(rng.integers(len(src)))]
        if kind == 0:
            t = s[: int(rng.integers(20, 150))]
        elif kind == 1:
            t = s
        elif kind == 2:
            t = list(s)
            t[int(rng.integers(len(t)))] = "N"
            t = "".join(t)
        elif kind == 3:
            t = "".join("ACGT"[c] for c in rng.integers(0, 4, size=int(rng.integers(10, 160))))
        elif kind == 4:
            t = s[:75]
        else:
            t = s[10:]
        reads.append(t)
        ids.append(("r%d" % int(rng.integers(0, n))) + (".1" if rng.random() < 0.2 else ""))
    lens = np.array([len(x) for x in reads], dtype=np.int32)
    off = np.zeros(len(reads), dtype=np.uint64)
    off[1:] = np.cumsum(lens[:-1])
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    mn, med, avg, _ = ref.kmer_count_stats(pool, off, lens, 21)
    # coarsen a part of the statistics so that long runs of equal (min, median, avg, len) must be decided by the strings
    coarse = rng.random(len(reads)) < 0.5
    mn = np.where(coarse, np.minimum(mn, 2), mn).astype(np.int32)
    med = np.where(coarse, np.minimum(med, 3), med).astype(np.int32)
    avg = np.where(coarse, np.float32(2.5), avg).astype(np.float32)
    ro = ref.sort_reads(reads, ids, mn, med, avg)
    go = api.sort_reads(pool, off, lens, ids, mn, med, avg, lib)
    key = lambda i: (reads[i], ids[i], int(mn[i]), int(med[i]), float(avg[i]))
    assert sorted(go.tolist()) == list(range(len(reads)))
    # records that compare equal in every field may come in either order: compare the sorted RECORDS, not the indices
    assert [key(i) for i in go] == [key(i) for i in ro], np.flatnonzero(np.array([key(i) != key(j) for i, j in zip(go, ro)]))[:5]
    return len(reads)


def check_mate_overlap(lib, ref, seed=161, n=3000):
    """t4_mate_overlap_batch against AlignAlgo::IsMateOverlap (AlignAlgo.hpp:1027-1096): return value, offset, bestMatchCnt
    for overlapping mates (with mismatches), read-through pairs, unrelated pairs, tandem repeats, both checkTandem settings
    and the two minOverlap formulas of ProcessRead (main.cpp:244-249)."""
    import ctypes as C
    rng = np.random.default_rng(seed)

    def rnd(L):
        return "".join("ACGT"[c] for c in rng.integers(0, 4, size=L))

    fr, sr = [], []
    for i in range(n):
        kind = int(rng.integers(0, 6))
        L1, L2 = int(rng.integers(30, 160)), int(rng.integers(30, 160))
        if kind == 0:       # suffix of f = prefix of s
            ov = int(rng.integers(5, min(L1, L2)))
            f = rnd(L1)
            s = f[L1 - ov:] + rnd(L2 - ov)
        elif kind == 1:     # the same with a few mismatches
            ov = int(rng.integers(10, min(L1, L2)))
            f = rnd(L1)
            t = list(f[L1 - ov:])
            for q in rng.integers(0, ov, size=int(rng.integers(1, 5))):
                t[int(q)] = "ACGT"[int(rng.integers(4))]
            s = "".join(t) + rnd(L2 - ov)
        elif kind == 2:     # read-through: s inside f
            f = rnd(L1)
            st = int(rng.integers(0, L1 // 2))
            s = f[st:st + L2]
        elif kind == 3:     # tandem repeats
            u = rnd(int(rng.integers(1, 5)))
            f = rnd(L1 // 2) + u * 20
            s = u * 20 + rnd(L2 // 2)
        elif kind == 4:
            f, s = rnd(L1), rnd(L2)
        else:               # two candidate offsets: ambiguous
            core = rnd(25)
            f = rnd(20) + core + rnd(15) + core
            s = core + rnd(L2)
        fr.append(f)
        sr.append(s)
    reads = fr + sr
    lens = np.array([len(x) for x in reads], dtype=np.int32)
    off = np.zeros(len(reads), dtype=np.uint64)
    off[1:] = np.cumsum(lens[:-1])
    pool = np.frombuffer(("".join(reads) + "\0" * 16).encode(), dtype=np.uint8).copy()
    fo, so = off[:n].copy(), off[n:].copy()
    fl, sl = lens[:n].copy(), lens[n:].copy()
    tot = fl + sl
    mo = np.where(rng.random(n) < 0.5, np.minimum(tot // 10, 31), np.minimum(tot // 20, 31)).astype(np.int32)
    ct = (rng.random(n) < 0.6).astype(np.uint8)
    gos, gof, gbm = (np.zeros(n, dtype=np.int32) for _ in range(3))
    lib.check(lib.mate_overlap_batch(pool.ctypes.data, pool.nbytes, fo.ctypes.data, fl.ctypes.data, so.ctypes.data, sl.ctypes.data, mo.ctypes.data,
                                     ct.ctypes.data, n, gos.ctypes.data, gof.ctypes.data, gbm.ctypes.data))
    l = ref.lib()
    n_pos = 0
    for i in range(n):
        o, b = C.c_int32(), C.c_int32()
        r = l.t4ref_is_mate_overlap(fr[i].encode(), len(fr[i]), sr[i].encode(), len(sr[i]), int(mo[i]), int(ct[i]), C.byref(o), C.byref(b))
        assert (r, o.value, b.value) == (int(gos[i]), int(gof[i]), int(gbm[i])), (i, r, o.value, b.value, gos[i], gof[i], gbm[i], fr[i], sr[i])
        n_pos += r >= 0
    assert n_pos > n // 5 and n_pos < n
    return n_pos


def check_sort_reads_tiny(lib, ref):
    """t4_sort_reads on 0 .. 3 records (no pass, one pass, a ragged last run)."""
    pool = np.frombuffer(b"ACGTACGTAC" + b"\0" * 16, dtype=np.uint8).copy()
    for n in (0, 1, 2, 3):
        ids = ["r%d" % (9 - i) for i in range(n)]
        order = api.sort_reads(pool, np.arange(n, dtype=np.uint64), np.full(n, 5, dtype=np.int32), ids,
                               np.ones(n, np.int32), np.ones(n, np.int32), np.ones(n, np.float32), lib)
        reads = [bytes(pool[i:i + 5]).decode() for i in range(n)]
        assert order.tolist() == ref.sort_reads(reads, ids, np.ones(n), np.ones(n), np.ones(n)).tolist()


def sort_key(reads, ids, mn, med, avg):
    """_sortRead::operator< (main.cpp:103-125) as a Python key: counts and length descending, then the read and the id as
    bytes -- Python orders bytes like strcmp on unsigned char, the shorter string first on a common prefix.  -0.0 and 0.0
    are equal keys, as they are equal floats in the comparator."""
    return lambda i: (-int(mn[i]), -int(med[i]), -float(avg[i]), -len(reads[i]), reads[i], ids[i])


def _check_sorted_records(go, keys, want):
    """go (the library's order) holds every index once and lists the same records as `want`; records equal in every field
    may come in either order, so the records are compared, not the indices."""
    n = len(keys)
    assert len(go) == n and (np.sort(go) == np.arange(n)).all(), "not a permutation"
    bad = [j for j, (a, b) in enumerate(zip(go, want)) if keys[a] != keys[b]]
    assert not bad, ("order", bad[:5], [keys[go[j]][:4] for j in bad[:2]], [keys[want[j]][:4] for j in bad[:2]])


def _ref_sort_bytes(ref, reads, ids, mn, med, avg):
    """The reference's std::sort on byte strings (bytes >= 0x80 included)."""
    import ctypes as C
    n = len(reads)
    ra = (C.c_char_p * max(1, n))(*reads)
    ia = (C.c_char_p * max(1, n))(*ids)
    order = np.zeros(max(1, n), dtype=np.int64)
    ref.lib().t4ref_sort_reads(ra, ia, np.ascontiguousarray(mn, dtype=np.int32).ctypes.data, np.ascontiguousarray(med, dtype=np.int32).ctypes.data,
                               np.ascontiguousarray(avg, dtype=np.float32).ctypes.data, n, order.ctypes.data)
    return order[:n]


def check_sort_reads_large(lib, seed=153, n=(1 << 20) + 3):
    """t4_sort_reads at a size where the sort kernel's grid-stride loop turns more than once (n above the launch cap, a ragged
    last run): synthetic read pairs with their real 21-mer statistics (t4_kmer_count_stats), lengths cut at random, half
    of the statistics coarsened so that long runs of ties are decided by the read strings and then the ids -- against the
    plain Python restatement of the comparator (sort_key)."""
    rng = np.random.default_rng(seed)
    cl = synth.make_clones(200, seed)
    rd = synth.sample_pairs(cl, (n + 1) // 2, 150, seed, sub_rate=0.01)
    L = rd.codes.shape[1]
    pool = np.concatenate([np.frombuffer(b"ACGT", dtype=np.uint8)[rd.codes[:n]].reshape(-1), np.zeros(16, dtype=np.uint8)])
    off = (np.arange(n, dtype=np.uint64) * np.uint64(L))
    lens = np.where(rng.random(n) < 0.3, rng.integers(20, L + 1, size=n), L).astype(np.int32)
    ids = [b"r%d" % (i // 2) + (b".1" if x < 0.1 else b"") for i, x in zip(range(n), rng.random(n))]
    mn, med, avg, _ = api.kmer_count_stats(pool, off, lens, 21, lib)
    coarse = rng.random(n) < 0.5
    mn = np.where(coarse, np.minimum(mn, 2), mn).astype(np.int32)
    med = np.where(coarse, np.minimum(med, 3), med).astype(np.int32)
    avg = np.where(coarse, np.float32(2.5), avg).astype(np.float32)
    go = api.sort_reads(pool, off, lens, ids, mn, med, avg, lib)
    pb = pool.tobytes()
    reads = [pb[o:o + l] for o, l in zip(off.tolist(), lens.tolist())]
    key = sort_key(reads, ids, mn.tolist(), med.tolist(), avg.tolist())
    keys = [key(i) for i in range(n)]
    want = sorted(range(n), key=keys.__getitem__)
    _check_sorted_records(go, keys, want)
    ties = sum(1 for a, b in zip(want, want[1:]) if keys[a][:4] == keys[b][:4])
    assert ties > n // 4, ties       # the strings really decide a large part of the order
    return n


def sort_edge_records(seed, n_base=1500):
    """Records for the comparator's edges: (reads, ids, min, median, avg).  Few distinct counts (long ties); reads and ids
    that differ first at a byte >= 0x80 against one < 0x80; reads longer than 512 bp that differ only late; avg values one
    float ulp apart, -0.0 next to 0.0; negative counts; groups of records equal in every field, scattered over the array so
    that equal records meet in different runs of every merge pass."""
    rng = np.random.default_rng(seed)
    avgs = [np.float32(1.0), np.nextafter(np.float32(1.0), np.float32(2)), np.nextafter(np.float32(1.0), np.float32(0)),
            np.float32(0.0), np.float32(-0.0), np.float32(2.5), np.float32(-1.5)]

    def rnd(L):
        return bytes(rng.choice(np.frombuffer(b"ACGT", dtype=np.uint8), size=L))

    recs = []

    def stats():
        return int(rng.choice([-1, 0, 1, 2])), int(rng.choice([0, 1, 3])), avgs[int(rng.integers(len(avgs)))]

    for i in range(n_base):
        kind = int(rng.integers(0, 6))
        mn, med, av = stats()
        if kind == 0:                      # a high byte against a low one at the same position, same counts and length
            r = bytearray(rnd(int(rng.integers(10, 40))))
            p = int(rng.integers(len(r)))
            r2 = bytearray(r)
            r[p] = int(rng.integers(0x80, 0x100))
            r2[p] = int(rng.integers(0x41, 0x80))
            recs.append((bytes(r), b"h%d" % i, mn, med, av))
            recs.append((bytes(r2), b"h%d" % i, mn, med, av))
        elif kind == 1:                    # same read, ids that differ at a high byte / are prefixes of each other
            r = rnd(int(rng.integers(10, 40)))
            for idb in (b"id\xe9", b"id\x7f", b"id", b"id\xff\x01", b"id\x80"):
                recs.append((r, idb, mn, med, av))
        elif kind == 2:                    # longer than 512 bp, differing only after position 512 (or a prefix)
            base = rnd(int(rng.integers(513, 1001)))
            q = int(rng.integers(512, len(base)))
            other = base[:q] + (b"A" if base[q:q + 1] != b"A" else b"C") + base[q + 1:]
            recs.append((base, b"l%d" % i, mn, med, av))
            recs.append((other, b"l%d" % i, mn, med, av))
            recs.append((base[:q], b"l%d" % i, mn, med, av))
        elif kind == 3:                    # avg one ulp apart, -0.0 next to 0.0, everything else equal
            r = rnd(int(rng.integers(10, 40)))
            for av2 in avgs:
                recs.append((r, b"u%d" % i, mn, med, av2))
        elif kind == 4:                    # a group of records equal in every field
            rec = (rnd(int(rng.integers(5, 30))), b"e%d" % (i % 7), mn, med, av)
            recs.extend([rec] * int(rng.choice([2, 3, 5, 17, 40])))
        else:
            recs.append((rnd(int(rng.integers(5, 60))), b"r%d" % int(rng.integers(0, 50)), mn, med, av))
    perm = rng.permutation(len(recs))
    recs = [recs[int(j)] for j in perm]
    reads = [x[0] for x in recs]
    ids = [x[1] for x in recs]
    mn = np.array([x[2] for x in recs], dtype=np.int32)
    med = np.array([x[3] for x in recs], dtype=np.int32)
    avg = np.array([x[4] for x in recs], dtype=np.float32)
    return reads, ids, mn, med, avg


def check_sort_reads_edges(lib, ref, seed=154, n_base=1500):
    """t4_sort_reads at the comparator's edges (sort_edge_records), against the reference's std::sort and the Python key."""
    reads, ids, mn, med, avg = sort_edge_records(seed, n_base)
    pool, off, lens = reads_pool(reads)
    go = api.sort_reads(pool, off, lens, ids, mn, med, avg, lib)
    key = sort_key(reads, ids, mn.tolist(), med.tolist(), avg.tolist())
    keys = [key(i) for i in range(len(reads))]
    _check_sorted_records(go, keys, _ref_sort_bytes(ref, reads, ids, mn, med, avg))
    _check_sorted_records(go, keys, sorted(range(len(reads)), key=keys.__getitem__))
    assert max(lens) > 512 and any(b >= 0x80 for r in reads for b in r)
    return len(reads)


def _mate_batch(lib, fr, sr, mo, ct):
    """t4_mate_overlap_batch over the pairs (fr[i], sr[i]) (str or bytes): (overlap_size, offset, best_match_cnt)."""
    n = len(fr)
    pool, off, lens = reads_pool(list(fr) + list(sr))
    fo, so = off[:n].copy(), off[n:].copy()
    fl, sl = lens[:n].copy(), lens[n:].copy()
    mo = np.ascontiguousarray(mo, dtype=np.int32)
    ct = np.ascontiguousarray(ct, dtype=np.uint8)
    gos, gof, gbm = (np.zeros(max(1, n), dtype=np.int32) for _ in range(3))
    lib.check(lib.mate_overlap_batch(pool.ctypes.data, pool.nbytes, fo.ctypes.data, fl.ctypes.data, so.ctypes.data, sl.ctypes.data,
                                     mo.ctypes.data, ct.ctypes.data, n, gos.ctypes.data, gof.ctypes.data, gbm.ctypes.data))
    return gos[:n], gof[:n], gbm[:n]


def _mate_ref_check(ref, fr, sr, mo, ct, got):
    """Every pair against AlignAlgo::IsMateOverlap of the reference; returns the return values."""
    import ctypes as C
    l = ref.lib()
    gos, gof, gbm = got
    out = np.zeros(len(fr), dtype=np.int32)
    o, b = C.c_int32(), C.c_int32()
    for i in range(len(fr)):
        f = fr[i] if isinstance(fr[i], bytes) else fr[i].encode()
        s = sr[i] if isinstance(sr[i], bytes) else sr[i].encode()
        r = l.t4ref_is_mate_overlap(f, len(f), s, len(s), int(mo[i]), int(ct[i]), C.byref(o), C.byref(b))
        assert (r, o.value, b.value) == (int(gos[i]), int(gof[i]), int(gbm[i])), (i, r, o.value, b.value, gos[i], gof[i], gbm[i], f, s, int(mo[i]), int(ct[i]))
        out[i] = r
    return out


def _mate_threshold_count(L):
    """int(L * similarityThreshold) of IsMateOverlap for an overlap of L bases (AlignAlgo.hpp:1042-1047)."""
    t = 0.95
    if L >= 100:
        t = 0.85
    elif L >= 50:
        t = 0.85 + (L - 50) / 50.0 * 0.1
    return int(L * t)


def mate_edge_pairs(seed, reps=6):
    """Pairs at the edges of IsMateOverlap: (fr, sr, minOverlap, checkTandem, tag) lists.
    - zero-length mates; minOverlap >= flen; minOverlap = 0;
    - mates up to 1000 bp whose only overlap has L = 49, 50, 51, 99, 100, 101 (the 0.95 / sloped / 0.85 threshold steps) or
      more bases, with exactly as many mismatches as the threshold allows, one fewer and one more;
    - N's and lower-case bases (compared as plain characters);
    - an overlap of exactly 2 x minOverlap that is a tandem repeat (w + w, |w| = minOverlap), and the same one base longer."""
    rng = np.random.default_rng(seed)
    comp = {"A": "C", "C": "G", "G": "T", "T": "A"}

    def rnd(L):
        return "".join("ACGT"[c] for c in rng.integers(0, 4, size=L))

    fr, sr, mo, ct, tag = [], [], [], [], []

    def add(f, s, m, c, t):
        fr.append(f); sr.append(s); mo.append(m); ct.append(c); tag.append(t)

    for c in (0, 1):
        add("", "", 0, c, "empty")
        add("", rnd(50), 5, c, "empty f")
        add(rnd(50), "", 5, c, "empty s")
        add("", "", 3, c, "empty")
    for _ in range(reps):
        for c in (0, 1):
            f = rnd(int(rng.integers(1, 60)))
            add(f, f, len(f), c, "minOverlap = flen")
            add(f, f, len(f) + int(rng.integers(1, 20)), c, "minOverlap > flen")
            g = rnd(int(rng.integers(20, 120)))
            q = int(rng.integers(1, len(g)))
            add(g, g[len(g) - q:] + rnd(int(rng.integers(0, 30))), 0, c, "minOverlap 0")
            add(g, rnd(int(rng.integers(0, 80))), 0, c, "minOverlap 0, random")
    for L in (49, 50, 51, 99, 100, 101, 150, 400, 1000):
        need = _mate_threshold_count(L)
        for extra in (-1, 0, 1):
            x = L - need + extra           # mismatches: need - 1 matches fail, need pass
            if x < 0:
                continue
            for _ in range(reps):
                flen = int(rng.integers(L, 1001))
                f = rnd(flen)
                ov = list(f[flen - L:])
                for p in rng.choice(L, size=x, replace=False):
                    ov[int(p)] = comp[ov[int(p)]]
                s = "".join(ov) + rnd(int(rng.integers(0, 1001 - L)))
                add(f, s, int(rng.integers(5, 32)), int(rng.integers(0, 2)), "threshold L=%d mismatches=%d" % (L, x))
    for _ in range(8 * reps):
        L = int(rng.integers(20, 160))
        f = list(rnd(L + int(rng.integers(0, 60))))
        j = len(f) - L
        s = f[j:] + list(rnd(int(rng.integers(0, 60))))
        for p in rng.integers(0, len(s), size=int(rng.integers(1, 6))):
            s[int(p)] = "N" if rng.random() < 0.5 else s[int(p)].lower()
        for p in rng.integers(0, len(f), size=int(rng.integers(0, 4))):
            f[int(p)] = "N" if rng.random() < 0.5 else f[int(p)].lower()
        add("".join(f), "".join(s), int(rng.integers(5, 20)), int(rng.integers(0, 2)), "N / lower case")
    for m in (3, 5, 8, 12, 20, 31):
        for _ in range(reps):
            w = rnd(m)
            for longer in (0, 1):
                core = w + w + (rnd(1) if longer else "")
                f = rnd(int(rng.integers(10, 80))) + core
                s = core + rnd(int(rng.integers(0, 80)))
                for c in (0, 1):
                    add(f, s, m, c, "tandem 2 x minOverlap" + (" + 1" if longer else ""))
    return fr, sr, mo, ct, tag


def check_mate_overlap_edges(lib, ref, seed=163, reps=6):
    """t4_mate_overlap_batch at the edges of IsMateOverlap (mate_edge_pairs) against the reference, pair by pair; the
    threshold and tandem cases must really land on both sides."""
    fr, sr, mo, ct, tag = mate_edge_pairs(seed, reps)
    ret = _mate_ref_check(ref, fr, sr, mo, ct, _mate_batch(lib, fr, sr, mo, ct))
    by = {}
    for t, r in zip(tag, ret):
        by.setdefault(t, []).append(int(r))
    for L in (49, 50, 51, 99, 100, 101):
        need = _mate_threshold_count(L)
        assert all(r == -1 for r in by["threshold L=%d mismatches=%d" % (L, L - need + 1)]), L
        assert sum(r == L for r in by["threshold L=%d mismatches=%d" % (L, L - need)]) >= len(by["threshold L=%d mismatches=%d" % (L, L - need)]) // 2, L
    assert all(r == -1 for t, rs in by.items() if t.startswith("empty") or t.startswith("minOverlap >") for r in rs)
    tandem = [r for t, rs in by.items() if t == "tandem 2 x minOverlap" for r in rs]
    assert -1 in tandem and any(r > 0 for r in tandem)
    return len(fr)


def write_bad_gene_fasta(path):
    """The bundled gene pool plus one gene of 2000 ACG repeats: a read of ACG repeats has far more seed hits on it than the
    per-read scratch of the annotation holds (T4_E_NOMEM), while every other read is answered as usual."""
    recs = write_gene_fasta(path)
    s = "ACG" * 2000
    with open(path, "a") as f:
        f.write(">IGHV9-99*01\n")
        for p in range(0, len(s), 60):
            f.write(s[p:p + 60] + "\n")
    return recs


BAD_READ = "ACG" * 100


def _expect_error(code, fn, *a):
    try:
        fn(*a)
    except api.T4Error as e:
        assert e.code == code, (e.code, code, str(e))
        return
    raise AssertionError("expected error %d" % code)


def _check_overlaps_read(g, r, t):
    gn, go, gsim = g.get_overlaps(t)
    rn, ro, rsim = r.get_overlaps(t, 0, -1, False)
    assert gn == rn, ("count", gn, rn, t)
    if rn > 0:
        assert (go == ro).all() and (gsim == rsim).all(), ("overlaps", t)
    return rn


def _check_scan(g, r, ref, reads):
    gs_, gl_, st = g.scan(*reads_pool(reads))
    rs_ = np.array([r.has_hit_in_set(x, 0) for x in reads], dtype=np.int8)
    rl_ = np.array([ref.is_low_complexity(x) for x in reads], dtype=np.uint8)
    assert (gl_ == rl_).all() and (gs_ == rs_).all(), ("scan", np.flatnonzero(gs_ != rs_)[:5], np.flatnonzero(gl_ != rl_)[:5])
    assert st["with_hit"] == int((rs_ != 0).sum())
    return int((rs_ != 0).sum())


def check_refset_error_isolation(lib, ref, tmp_path, batch, seed=146):
    """A read that fails on the device (more hits than the per-read scratch) fails its own call with T4_E_NOMEM, and only
    that call: later get_overlaps, annotate and scan calls on the same gene set -- the annotate and scan launches reuse the
    same worker shells, `batch` reads keep their count unchanged -- answer as the reference does.  A batch that contains
    the failing read fails as a whole."""
    fa = os.path.join(str(tmp_path), "genes_bad%d.fa" % seed)
    recs = write_bad_gene_fasta(fa)
    lib.check(lib.reset())
    g = api.RefSet(fa, 9, lib, hit_len_required=31)
    r = ref.RefGeneSet(fa, 9, hit_len_required=31)
    good = annotate_reads(recs, batch, seed)
    ann = [r.annotate_read(t) for t in good]
    pool, off, lens = reads_pool(good)
    with_bad = lambda j: reads_pool(good[:j] + [BAD_READ] + good[j + 1:])
    nonempty = [t for t, a in zip(good, ann) if (a[0][:, 0] >= 0).any()][:6]
    assert len(nonempty) >= 3
    for t in nonempty[:2]:
        _check_overlaps_read(g, r, t)
    _expect_error(api.T4_E_NOMEM, g.get_overlaps, BAD_READ)
    assert sum(_check_overlaps_read(g, r, t) for t in nonempty) > 0
    _expect_error(api.T4_E_NOMEM, g.annotate, *with_bad(0))
    compare_annotations(*g.annotate(pool, off, lens), good, ann, "after a failed annotate")
    _expect_error(api.T4_E_NOMEM, g.annotate, *with_bad(batch // 2))
    assert _check_scan(g, r, ref, good) > batch // 4
    compare_annotations(*g.annotate(pool, off, lens), good, ann, "after a failed annotate and a scan")
    _expect_error(api.T4_E_NOMEM, g.get_overlaps, BAD_READ)
    _expect_error(api.T4_E_NOMEM, g.annotate, *with_bad(batch - 1))
    for t in nonempty:
        _check_overlaps_read(g, r, t)
    compare_annotations(*g.annotate(pool, off, lens), good, ann, "at the end")
    g.close()


def check_refset_annotate_batches(lib, ref, tmp_path, n_workers, seed=144):
    """t4_refset_annotate at batch sizes around the worker count (one read, fewer reads than workers, one short, exactly as
    many, one more, three rounds and a few): every read against the reference; n = 0 returns 0; the largest batch twice on
    the same set gives byte-identical output (results do not depend on which worker took which read)."""
    fa = os.path.join(str(tmp_path), "genes_b%d.fa" % seed)
    recs = write_gene_fasta(fa)
    lib.check(lib.reset())
    g = api.RefSet(fa, 9, lib, hit_len_required=31)
    r = ref.RefGeneSet(fa, 9, hit_len_required=31)
    sizes = sorted(set([1, 37, n_workers - 1, n_workers, n_workers + 1, 3 * n_workers + 5]) - {0})
    reads = annotate_reads(recs, max(sizes) + 101, seed)
    ann = [r.annotate_read(t) for t in reads]
    z = np.zeros(16, dtype=np.uint8)
    zo = np.zeros(1, dtype=np.uint64)
    zl = np.zeros(1, dtype=np.int32)
    out = np.zeros((1, 4, 8), dtype=np.int32)
    sim = np.zeros((1, 4), dtype=np.float64)
    assert lib.refset_annotate(g.h, z.ctypes.data, z.nbytes, zo.ctypes.data, zl.ctypes.data, 0, out.ctypes.data, sim.ctypes.data) == 0
    for j, n in enumerate(sizes):
        s0 = (j * 17) % (len(reads) - n + 1)
        part = reads[s0:s0 + n]
        go, gsim = g.annotate(*reads_pool(part))
        compare_annotations(go, gsim, part, ann[s0:s0 + n], "n=%d" % n)
    part = reads[: max(sizes)]
    pool, off, lens = reads_pool(part)
    a1, s1 = g.annotate(pool, off, lens)
    a2, s2 = g.annotate(pool, off, lens)
    assert a1.tobytes() == a2.tobytes() and s1.tobytes() == s2.tobytes()
    n_set = compare_annotations(a1, s1, part, ann[: max(sizes)], "repeat")
    assert n_set[0] > len(part) // 5, n_set
    g.close()
    return sizes


def check_refset_interleaved(lib, ref, tmp_path, n, seed=145):
    """scan -> annotate -> scan -> get_overlaps -> annotate on one gene set: the scan and annotate launches share the worker
    shells (the annotate also writes their key buffers); every result must equal the reference's."""
    fa = os.path.join(str(tmp_path), "genes_i%d.fa" % seed)
    recs = write_gene_fasta(fa)
    lib.check(lib.reset())
    g = api.RefSet(fa, 9, lib, hit_len_required=31)
    r = ref.RefGeneSet(fa, 9, hit_len_required=31)
    ra = annotate_reads(recs, n, seed)
    rb = annotate_reads(recs, n, seed + 1000)
    assert _check_scan(g, r, ref, rb) > n // 4
    compare_annotations(*g.annotate(*reads_pool(ra)), ra, [r.annotate_read(t) for t in ra], "first annotate")
    assert _check_scan(g, r, ref, ra) > n // 4
    assert sum(_check_overlaps_read(g, r, t) for t in rb[:200]) > 100
    n_set = compare_annotations(*g.annotate(*reads_pool(rb)), rb, [r.annotate_read(t) for t in rb], "second annotate")
    assert n_set[0] > n // 5, n_set
    g.close()


def example_reads():
    """The reads of the shipped example (tests/golden/example_{1,2}.fq.gz), both mates, in file order."""
    out = []
    for m in (1, 2):
        lines = gzip.open(os.path.join(GOLD, "example_%d.fq.gz" % m)).read().decode().split("\n")
        out.extend(lines[1::4][: len(lines) // 4])
    return out


def check_refset_annotate_example(lib, ref, tmp_path):
    """The rough annotation of the shipped example's 396 reads against the reference's own hg38 gene set
    (tests/golden/hg38_bcrtcr.fa.gz): real reads and real IMGT genes, with C genes and their names."""
    fa = os.path.join(str(tmp_path), "hg38_bcrtcr.fa")
    with open(fa, "wb") as f:
        f.write(gzip.open(os.path.join(GOLD, "hg38_bcrtcr.fa.gz")).read())
    reads = example_reads()
    assert len(reads) == 396
    lib.check(lib.reset())
    g = api.RefSet(fa, 9, lib, hit_len_required=17)
    r = ref.RefGeneSet(fa, 9, hit_len_required=17)
    assert g.names() == r.names()
    n_set = compare_annotations(*g.annotate(*reads_pool(reads)), reads, [r.annotate_read(t) for t in reads], "example")
    assert n_set[0] > 100 and n_set[2] > 50, n_set
    for t in reads[::9]:
        _check_overlaps_read(g, r, t)
    g.close()
    return n_set
