"""Packed stage-1 contigs (t4_streams_pack_contigs: t4_pack_size_kernel + t4_pack_kernel, the buffer bench.py ends every
step with, the all-gather exchanges, bench/quality.py decodes and the merge oracle is defined on) against the reference,
shared by the GPU and emulation test modules.  `lib` is an api.Lib, `dev` the torch device the packed buffer lives on
("cuda"; "cpu" for the emulation, whose "device" memory is host memory).

Every case packs a list of sets, decodes the records and checks them with check_packed(): the Output text, slot, barcode
and numRead of every record against the reference SeqSet that ran the same reads, the record layout, and that the bytes
do not depend on what the buffer held before.  Each case returns counts of what it is about, so that a generator that
drifts away from its edge fails instead of passing vacuously."""
import ctypes as C
import os
import sys

import numpy as np
import torch

import parity_cases as pc
from trust4_b200 import api, dist, synth

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bench"))
import quality  # noqa: E402

U16_MAX = 65535
T4_E_INVAL = -19          # include/trust4_b200.h
T4_CONTIG_PURGED = 1


def _handles(sets):
    return (C.c_void_p * max(1, len(sets)))(*[s.h if s is not None else None for s in sets])


def _sync(dev):
    if torch.device(dev).type == "cuda":
        torch.cuda.synchronize()


def pack_call(lib, sets, buf=None, offset=0, cap=None):
    """One t4_streams_pack_contigs call into buf[offset:] (buf None: sizes only) -> (return code, bytes_needed, n_contigs)."""
    need, n = C.c_size_t(0), C.c_int64(0)
    if buf is None:
        ptr, cap = None, 0
    else:
        ptr = buf.data_ptr() + offset
        cap = buf.numel() - offset if cap is None else cap
    r = lib.streams_pack_contigs(_handles(sets), len(sets), ptr, cap, C.byref(need), C.byref(n))
    return r, int(need.value), int(n.value)


def record_bytes(ln, name_len, narrow):
    """t4_pack_record_bytes: 32-byte header + consensus + 4 u16 (narrow) or 4 i32 columns per base + name, padded to 16."""
    return (32 + (9 if narrow else 17) * ln + name_len + 15) & ~15


def ref_fields(r, slot):
    """(barcode, numRead) of the reference's seqs[slot], None when the slot holds no contig.  posWeight is not read: a
    purged contig keeps it compressed or released."""
    bc, nr = C.c_int(), C.c_int()
    if r.l.t4ref_get_contig(r.h, slot, None, 0, None, None, 0, C.byref(bc), C.byref(nr), None, None) < 0:
        return None
    return bc.value, nr.value


def _headers(a):
    """(offset, header u32[8]) of every record of a packed buffer; the records must tile it exactly."""
    out = []
    o = 0
    while o < len(a):
        assert o + 32 <= len(a), ("record header past the end", o, len(a))
        h = a[o:o + 32].copy().view(np.uint32)
        assert h[6] >= 32 and h[6] % 16 == 0, ("record bytes", o, int(h[6]))
        out.append((o, h))
        o += int(h[6])
    assert o == len(a), ("records overrun bytes_needed", o, len(a))
    return out


def check_deterministic(lib, dev, sets, want):
    """The same bytes over [0, bytes_needed) whatever the buffer held: zeros, 0xFF, and an earlier, larger pack's records
    (bench.py keeps one buffer across steps).  Nothing is written past bytes_needed."""
    need = len(want)
    for fill in (0x00, 0xFF):
        b = torch.full((need + 256,), fill, dtype=torch.uint8, device=dev)
        r, nd, _ = pack_call(lib, sets, b)
        lib.check(r)
        _sync(dev)
        got = b.cpu().numpy()
        assert nd == need
        assert (got[:need] == want).all(), ("bytes depend on the buffer's old contents", fill, np.flatnonzero(got[:need] != want)[:8])
        assert (got[need:] == fill).all(), ("bytes written past bytes_needed", fill)
    # an earlier step's records, twice over and in the other set order, fill the buffer first
    b = torch.full((2 * need + 1024,), 0x5A, dtype=torch.uint8, device=dev)
    for off in (0, need):
        lib.check(pack_call(lib, sets[::-1], b, offset=off)[0])
    lib.check(pack_call(lib, sets, b)[0])
    _sync(dev)
    got = b[:need].cpu().numpy()
    assert (got == want).all(), ("bytes depend on a stale pack", np.flatnonzero(got != want)[:8])


def check_packed(lib, dev, sets, refs, deterministic=True):
    """Pack `sets` as bench.py does (one device buffer) and check every record.  refs: {index in `sets`: reference
    SeqSet that ran the same reads} for the sets compared with the reference (the layout is checked on all of them).
    Returns counts: records, wide records (i32 columns), sets without records, holes (dead slots below a compared set's
    size), purged contigs, purged contigs with flat coverage (Output prints numRead), the records themselves."""
    nd0, n0 = pack_call(lib, sets)[1:]
    buf, n = dist.pack_contigs(lib, sets, device=dev)
    _sync(dev)
    assert buf.device.type == torch.device(dev).type
    a = buf.cpu().numpy().copy()
    assert len(a) == nd0 and n == n0
    heads = _headers(a)
    recs = dist.unpack_contigs(a)
    assert len(heads) == len(recs) == n
    st = dict(records=n, wide=0, empty_sets=0, holes=0, purged=0, flat=0, recs=recs)
    prev = (-1, -1)
    for (o, h), c in zip(heads, recs):
        j, slot, ln, nl = int(h[0]), int(h[1]), int(h[2]), int(h[3])
        assert 0 <= j < len(sets), ("set index within the call", j)
        assert (j, slot) > prev, ("records in (set, slot) order", prev, (j, slot))
        prev = (j, slot)
        pw = c["pos_weight"]
        narrow = int(pw.max(initial=0)) <= U16_MAX
        assert pw.min(initial=0) >= 0
        assert int(h[7]) == (1 if narrow else 0), ("flags: u16 columns iff every count fits", j, slot, int(h[7]), int(pw.max(initial=0)))
        assert int(h[6]) == record_bytes(ln, nl, narrow), (j, slot)
        assert len(c["consensus"]) == ln and len(c["name"]) == nl and set(c["consensus"]) <= set("ACGTN")
        end = o + 32 + (9 if narrow else 17) * ln + nl
        assert (a[end:o + int(h[6])] == 0).all(), ("tail padding", j, slot)
        st["wide"] += not narrow
    codes, coff, nq = quality.contigs_from_packed(a)
    assert nq == n
    lut = np.full(256, 4, dtype=np.uint8)
    lut[np.frombuffer(b"ACGT", dtype=np.uint8)] = np.arange(4, dtype=np.uint8)
    for i, c in enumerate(recs):
        assert (codes[coff[i]:coff[i + 1]] == lut[np.frombuffer(c["consensus"].encode(), dtype=np.uint8)]).all(), i
    have = {c["set"] for c in recs}
    st["empty_sets"] = sum(1 for j in range(len(sets)) if j not in have)
    if deterministic:
        check_deterministic(lib, dev, sets, a)
    out = dist.format_output(recs)
    for j, r in refs.items():
        want = r.output()
        if want:
            assert out.get(j) == want, ("Output text", j)
        else:
            assert j not in out, ("records of a set without live contigs", j)
        mine = [c for c in recs if c["set"] == j]
        live = {}
        for i in range(r.size()):
            f = ref_fields(r, i)
            if f is None:
                st["holes"] += 1
            else:
                live[i] = f
        assert [c["slot"] for c in mine] == sorted(live), ("slots", j)
        for c in mine:
            assert (c["barcode"], c["num_read"]) == live[c["slot"]], ("barcode / numRead", j, c["slot"], (c["barcode"], c["num_read"]), live[c["slot"]])
            if sets[j].contig_flags(c["slot"]) == T4_CONTIG_PURGED:
                st["purged"] += 1
                pw = c["pos_weight"]
                if ((pw > 0).sum(axis=1) == 1).all() and (pw.max(axis=1) == c["num_read"]).all():
                    st["flat"] += 1
    return st


def _refs_for(ref, w, cfg, off, descs, which, k=9, hit_len=None, consider_barcode=0):
    refs = {}
    for j in which:
        r = ref.RefSeqSet(k)
        if hit_len is not None:
            r.set_hit_len_required(hit_len)
        if consider_barcode:
            ref.lib().t4ref_set_consider_barcode_in_hash(r.h, 1)
        lo, hi = int(off[j]), int(off[j + 1])
        r.run_descs(cfg, descs[lo:hi].copy(), w.pool, w.names)
        refs[j] = r
    return refs


def case_bench_shapes(lib, ref, dev, seed, n_streams, nclones, npairs, deal=False, group="", sample=None):
    """configs[1] as bench.py packs it: rank-block, dealt or gene-grouped streams; `sample` sets (seeded, like
    bench.py's parity_spot_check) or all of them compared with the reference, the layout checked on all."""
    lib.check(lib.reset())
    _, w, cfg, off, descs = pc.batch_inputs(lib, seed, n_streams, nclones, npairs, deal=deal, group=group)
    S = len(off) - 1
    sets = api.SeqSet.create_many(S, 9, lib)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    which = range(S) if sample is None else np.sort(np.random.default_rng(seed).choice(S, size=sample, replace=False))
    st = check_packed(lib, dev, sets, _refs_for(ref, w, cfg, off, descs, which))
    st["sets"] = S
    return st


def case_change_kmer_length(lib, ref, dev, seed=21):
    """ChangeKmerLength in mid-stream (k 9 -> 11 -> 13: slots compacted and renumbered, full re-index)."""
    lib.check(lib.reset())
    w = pc.small_workload(seed, 60, 1500)
    cfg = synth.run_cfg(change_k_threshold=20)
    g = api.SeqSet(9, lib)
    r = ref.RefSeqSet(9)
    g.run_descs(cfg, w.descs, w.pool, w.names)
    r.run_descs(cfg, w.descs, w.pool, w.names)
    assert g.kmer_length() == r.kmer_length() > 9
    st = check_packed(lib, dev, [g], {0: r})
    st["kmer_length"] = g.kmer_length()
    return st


def case_release_shallow(lib, ref, dev, min_cov, seed=2, n_streams=3):
    """ReleaseShallowContigs(min_cov) after the batch loop (--contigMinCov, main.cpp:1952-1955): dead slots between live ones."""
    lib.check(lib.reset())
    _, w, cfg, off, descs = pc.batch_inputs(lib, seed, n_streams, 25, 400)
    sets = api.SeqSet.create_many(n_streams, 9, lib)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    refs = _refs_for(ref, w, cfg, off, descs, range(n_streams))
    for j in range(n_streams):
        sets[j].release_shallow_contigs(min_cov)
        refs[j].release_shallow_contigs(min_cov)
    return check_packed(lib, dev, sets, refs)


def case_empty_sets_between(lib, ref, dev, seed=3):
    """A handle list with sets that never received a read before, between and after full ones."""
    lib.check(lib.reset())
    _, w, cfg, off, descs = pc.batch_inputs(lib, seed, 3, 25, 400)
    full = [1, 4, 5]                    # of 8 sets: 0, 2, 3, 6, 7 stay empty
    S = 8
    off8 = np.zeros(S + 1, dtype=np.int64)
    for j in range(S):
        off8[j + 1] = off8[j] + ((off[full.index(j) + 1] - off[full.index(j)]) if j in full else 0)
    sets = api.SeqSet.create_many(S, 9, lib)
    api.streams_run(sets, cfg, descs, off8, w.pool, w.names, lib)
    st = check_packed(lib, dev, sets, _refs_for(ref, w, cfg, off8, descs, range(S)))
    st["full"] = len(full)
    return st


def case_single_cell(lib, ref, dev, contig_min_cov, seed=51, n_barcodes=24, reads_per_barcode=150, n_streams=5):
    """configs[3]: barcode-partitioned streams, barcode-salted index, finished barcodes purged (ReleaseFinishedBarcodeSeq:
    posWeight compressed, or released with numRead = the flat coverage), contigMinCov."""
    lib.check(lib.reset())
    cl = synth.make_clones(60, seed)
    rd, bc = synth.sample_single_cell(cl, n_barcodes, reads_per_barcode, 150, seed)
    w = synth.build_workload(cl, rd, barcode=bc)
    cfg = synth.run_cfg(has_barcode=1, release_barcodes=1, contig_min_cov=contig_min_cov)
    off, descs = synth.shard_workload(w, n_streams, align="barcode")
    sets = api.SeqSet.create_many(n_streams, 9, lib, hit_len_required=13, consider_barcode=1)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    refs = _refs_for(ref, w, cfg, off, descs, range(n_streams), hit_len=13, consider_barcode=1)
    st = check_packed(lib, dev, sets, refs)
    st["barcoded"] = sum(1 for c in st["recs"] if c["barcode"] >= 0)
    return st


def case_repseq(lib, ref, dev, seed=61, n_reads=4000, n_streams=3):
    """configs[4]: --repseq amplicon reads (repetitiveData), V-gene pseudo barcodes, k changes in mid-run."""
    lib.check(lib.reset())
    cl = synth.make_clones(120, seed, chains=("TRB",))
    w = synth.build_workload(cl, synth.sample_amplicon(cl, n_reads, 100, seed), repseq=True)
    cfg = synth.run_cfg(repetitive=1, change_k_threshold=40, first_read_len=100)
    off, descs = synth.shard_workload(w, n_streams)
    sets = api.SeqSet.create_many(n_streams, 9, lib)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    st = check_packed(lib, dev, sets, _refs_for(ref, w, cfg, off, descs, range(n_streams)))
    st["barcoded"] = sum(1 for c in st["recs"] if c["barcode"] >= 0)
    st["kmer_changed"] = sum(1 for s in sets if s.kmer_length() > 9)
    return st


def case_assign_extended(lib, ref, dev, seed=82, n_streams=4, nclones=30, npairs=500, kmer=17):
    """The AssignRead pass's extended sets (InputSeqSet at k + RecomputePosWeight), t4_assign_extended_set(a, j) for
    every j packed in one call, against the reference's own pass (main.cpp:2047-2118)."""
    lib.check(lib.reset())
    w = pc.small_workload(seed, nclones, npairs)
    cfg = synth.run_cfg()
    off, descs = synth.shard_workload(w, n_streams)
    sets = api.SeqSet.create_many(n_streams, 9, lib)
    wl = api.Workload(descs, w.pool, w.names, lib)
    pc._run_resident(lib, sets, cfg, wl, off)
    a = api.Assign(sets, wl, off, kmer)
    ext = [a.extended_set(j) for j in range(n_streams)]
    refs = {}
    for j in range(n_streams):
        lo, hi = int(off[j]), int(off[j + 1])
        r = ref.RefSeqSet(9)
        d = descs[lo:hi].copy()
        _, rret, rstr, rresc = r.run_descs(cfg, d, w.pool, w.names)
        refs[j] = ref.assign_pass(r, kmer, d, w.pool, ref.assembled_list(rret, rresc), rstr)[0]
    st = check_packed(lib, dev, ext, refs)
    a.close()
    wl.close()
    return st


def _run_descs(runs, offs, lens):
    """Records of runs of one sequence each: (sequence, records, first record starts a novel contig).  A run's first
    record calls AddRead (then InputNovelRead where AddRead fails and the run is novel), the others are its duplicates
    (RepeatAddRead)."""
    n = sum(r[1] for r in runs)
    d = np.zeros(n, dtype=synth.READ_DESC)
    i = 0
    for s, cnt, novel in runs:
        d["seq_off"][i:i + cnt] = offs[s]
        d["len"][i:i + cnt] = lens[s]
        d["eq_lo"][i:i + cnt] = i
        d["eq_hi"][i:i + cnt] = i + cnt
        d["flags"][i + 1:i + cnt] = synth.RD_DUP
        if novel:
            d["flags"][i] = synth.RD_NOVEL_ON_FAIL
        i += cnt
    d["barcode"] = -1
    d["mate_idx"] = -1
    d["min_kmer_count"] = 1
    d["min_cnt"] = 1
    d["sim_threshold"] = 0.9
    d["novel_strand"] = 1
    d["gene4"] = b"IGHV"
    return d


def boundary_workload(seed=7):
    """One set, three contigs of odd length (the u16 columns start at an odd byte), built by InputNovelRead and runs of
    duplicate records through the batch loop, in two batches:
      first: slot 0 (121 bp) and slot 1 (131 bp) with every count exactly 65 535, slot 2 (201 bp) with counts 1;
      second: one more copy of slot 1's read (every count 65 536), and two half reads of slot 2 overlapping in column
      100, whose base alone reaches 65 536 (the other columns stay at most 32 769).
    Returns (pool, [descs of each batch], names, [{slot: (largest count, counts over 65 535)} after each batch])."""
    rng = np.random.default_rng(seed)
    rnd = lambda n: "".join("ACGT"[x] for x in rng.integers(0, 4, size=n))
    a, b, c = rnd(121), rnd(131), rnd(201)
    x, y = c[:101], c[100:]
    nx, ny = 32768, 32767
    seqs = [a, b, c, x, y]
    offs = np.cumsum([0] + [len(s) for s in seqs])
    lens = [len(s) for s in seqs]
    pool = np.frombuffer("".join(seqs).encode() + b"\0" * 16, dtype=np.uint8).copy()
    batches = [_run_descs([(0, U16_MAX, True), (1, U16_MAX, True), (2, 1, True)], offs, lens),
               _run_descs([(1, 1, False), (3, nx, False), (4, ny, False)], offs, lens)]
    want = [{0: (U16_MAX, 0), 1: (U16_MAX, 0), 2: (1, 0)},
            {0: (U16_MAX, 0), 1: (U16_MAX + 1, 131), 2: (U16_MAX + 1, 1)}]
    return pool, batches, [b"IGHV1-2*01"], want


def case_u16_boundary(lib, ref, dev):
    """The 16-bit decision at its edge: largest counts 65 535 (narrow) and 65 536 (wide), a contig where one base of one
    column alone passes 65 535, and a contig packed narrow once that has since grown wide."""
    lib.check(lib.reset())
    pool, batches, names, want = boundary_workload()
    cfg = synth.run_cfg(do_rescue=0)
    g = api.SeqSet(9, lib)
    r = ref.RefSeqSet(9)
    wide = []
    for d, wb in zip(batches, want):
        _, gret, _, _ = g.run_descs(cfg, d, pool, names)
        _, rret, _, _ = r.run_descs(cfg, d, pool, names)
        assert (gret == rret).all() and (gret >= 0).all()
        st = check_packed(lib, dev, [g], {0: r})
        recs = st["recs"]
        assert [c["slot"] for c in recs] == [0, 1, 2]
        for c in recs:
            top, over = wb[c["slot"]]
            pw = c["pos_weight"]
            assert len(c["consensus"]) % 2 == 1
            assert int(pw.max()) == top and int((pw > U16_MAX).sum()) == over, (c["slot"], int(pw.max()), int((pw > U16_MAX).sum()))
        wide.append(st["wide"])
    assert wide == [0, 2]
    return st


def case_two_ranks_merge(lib, ref, dev, seed=2, n_streams=6, nclones=25, npairs=600):
    """What the merge step's all-gather carries: two per-rank pack calls over disjoint handle lists, each numbering its
    sets from 0, concatenated in rank order.  Rebuilt into reference sets, the merge oracle (InputSeqSet +
    ChangeKmerLength(31) + RemoveRedundantSeq) gives the same set and removed count as merging the reference's own
    shard sets."""
    lib.check(lib.reset())
    _, w, cfg, off, descs = pc.batch_inputs(lib, seed, n_streams, nclones, npairs)
    S = len(off) - 1
    sets = api.SeqSet.create_many(S, 9, lib)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    refs = _refs_for(ref, w, cfg, off, descs, range(S))
    half = S // 2
    ranks = [list(range(half)), list(range(half, S))]
    parts = []
    for js in ranks:
        buf, n = dist.pack_contigs(lib, [sets[j] for j in js], device=dev)
        _sync(dev)
        parts.append(buf)
        assert len(dist.unpack_contigs(buf)) == n
    gathered = torch.cat(parts).cpu().numpy()
    assert len(gathered) == sum(p.numel() for p in parts)
    rebuilt, direct, o = [], [], 0
    for js, p in zip(ranks, parts):
        recs = dist.unpack_contigs(gathered[o:o + p.numel()])
        o += p.numel()
        assert {c["set"] for c in recs} <= set(range(len(js)))
        for i, j in enumerate(js):
            rebuilt.append(ref.set_from_contigs([c for c in recs if c["set"] == i]))
            direct.append(refs[j])
    m1, removed1 = ref.merge_sets(rebuilt)
    m2, removed2 = ref.merge_sets(direct)
    assert m1.output() == m2.output() and removed1 == removed2
    return dict(removed=removed1, contigs=sum(1 for s in rebuilt for i in range(s.size())))


def check_abi_edges(lib, dev, seed=4):
    """t4_streams_pack_contigs at its argument edges: sizes only, an exact and a one-byte-short buffer, no sets, stale
    and null handles."""
    lib.check(lib.reset())
    _, w, cfg, off, descs = pc.batch_inputs(lib, seed, 3, 25, 400)
    sets = api.SeqSet.create_many(3, 9, lib)
    api.streams_run(sets, cfg, descs, off, w.pool, w.names, lib)
    r, need, n = pack_call(lib, sets)
    assert r == 0 and need > 0 and n > 0 and need % 16 == 0
    want = dist.pack_contigs(lib, sets, device=dev)[0].cpu().numpy()
    assert len(want) == need
    exact = torch.full((need,), 0xFF, dtype=torch.uint8, device=dev)
    assert pack_call(lib, sets, exact) == (0, need, n)
    _sync(dev)
    assert (exact.cpu().numpy() == want).all()
    short = torch.full((need + 64,), 0x5A, dtype=torch.uint8, device=dev)
    assert pack_call(lib, sets, short, cap=need - 1)[0] == T4_E_INVAL
    _sync(dev)
    assert (short.cpu().numpy() == 0x5A).all(), "a refused pack wrote to the buffer"
    assert lib.streams_pack_contigs(_handles([]), 0, None, 0, None, None) == T4_E_INVAL
    assert lib.streams_pack_contigs(_handles([]), 0, short.data_ptr(), short.numel(), None, None) == T4_E_INVAL
    assert pack_call(lib, [sets[0], None, sets[2]])[0] == T4_E_INVAL
    lib.check(lib.reset())              # the arena is reclaimed: the handles are stale
    for s in sets:
        assert pack_call(lib, [s])[0] == T4_E_INVAL
    assert pack_call(lib, sets, short)[0] == T4_E_INVAL
    _sync(dev)
    assert (short.cpu().numpy() == 0x5A).all()
    fresh = api.SeqSet.create_many(2, 9, lib)
    assert pack_call(lib, [fresh[0], sets[1]])[0] == T4_E_INVAL
    assert pack_call(lib, fresh) == (0, 0, 0)
    return n
