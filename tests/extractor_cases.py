"""Inputs of the stage-0 drop-in tests and of bench/stage0_extract.py: synthetic FASTQ read sets for `fastq-extractor`.

Candidates are windows of synthetic clonotypes (V + junction + J + C of the bundled gene pool, synth.make_clones) with a
few sequencing errors; decoys are random sequence, the share of a read set that does not come from an immune receptor.
`edge_pairs` adds the reads at the rules' edges: low complexity (homopolymers, N's at and below a tenth of the read, two
bases at most twice), pairs where only read 2 is a candidate or neither is, reads shorter than k, reads of exactly
T4_MAX_READ_LEN and one base longer (the host path of the drop-in)."""
import gzip
import os
import re
import subprocess

import numpy as np

from trust4_b200 import synth

MAX_READ = 512                 # T4_MAX_READ_LEN (include/trust4_b200.h): longer reads are answered on the host
LUT = np.frombuffer(b"ACGTN", dtype=np.uint8)


def gene_fasta(path):
    """The bundled gene pool as the -f file."""
    pool = synth.load_gene_pool()
    with open(path, "w") as f:
        for ch in pool.values():
            for seg in ch.values():
                for name, seq in seg:
                    f.write(">%s\n%s\n" % (name, seq))
    return path


def _candidates(rng, clones, n, L, sub_rate=0.005):
    """n fragments of the clonotypes: read 1 forward from the fragment start, read 2 the reverse complement of its end
    (mates swapped for half of them).  Windows past a clonotype's end are filled with random bases."""
    ncl = len(clones.off) - 1
    cl = rng.integers(0, ncl, size=n)
    lo = clones.off[cl]
    tlen = clones.off[cl + 1] - lo
    ins = np.clip(rng.normal(2 * L, L / 3.0, size=n).astype(np.int64), L, np.maximum(tlen, L))
    start = (rng.random(n) * np.maximum(tlen - ins + 1, 1)).astype(np.int64)
    ar = np.arange(L, dtype=np.int64)
    p1 = start[:, None] + ar[None, :]
    p2 = (start + ins - 1)[:, None] - ar[None, :]
    last = len(clones.seq) - 1
    r1 = clones.seq[np.clip(lo[:, None] + p1, 0, last)]
    r2 = 3 - clones.seq[np.clip(lo[:, None] + p2, 0, last)]
    r1 = np.where((p1 < tlen[:, None]), r1, rng.integers(0, 4, size=(n, L)))
    r2 = np.where((p2 >= 0) & (p2 < tlen[:, None]), r2, rng.integers(0, 4, size=(n, L)))
    for r in (r1, r2):
        m = rng.random((n, L)) < sub_rate
        r[m] = (r[m] + rng.integers(1, 4, size=int(m.sum()))) % 4
    swap = rng.random(n) < 0.5
    a = np.where(swap[:, None], r2, r1).astype(np.uint8)
    b = np.where(swap[:, None], r1, r2).astype(np.uint8)
    return a, b


def bulk_pairs(rng, clones, n, L, decoy):
    """n pairs of length L as (n, L) code arrays (A C G T N = 0..4): a share `decoy` of random pairs, the rest candidates."""
    a = rng.integers(0, 4, size=(n, L), dtype=np.uint8)
    b = rng.integers(0, 4, size=(n, L), dtype=np.uint8)
    cand = np.nonzero(rng.random(n) >= decoy)[0]
    if len(cand):
        ca, cb = _candidates(rng, clones, len(cand), L)
        a[cand], b[cand] = ca, cb
    return a, b


def _s(codes):
    return LUT[codes].tobytes().decode()


def edge_pairs(rng, clones, L):
    """(read 1, read 2) strings at the edges of IsLowComplexity, HasHitInSet and the device's read length limit.  Each
    edge read is paired with a decoy, so that the pair is kept iff the edge read is a candidate, and a few with a
    candidate mate."""
    def cand_len(l, n=1):
        return [_s(x) for x in _candidates(rng, clones, n, l)[0]]

    def cand(n):
        return cand_len(L, n)

    def rand(l):
        return _s(rng.integers(0, 4, size=l, dtype=np.uint8))

    edge = []
    edge += ["A" * L, "C" * L, "N" * L, "AC" * (L // 2) + "A" * (L % 2)]           # homopolymers, two bases
    for c in cand(6):                                                               # N's: L / 10 is low, one fewer is not
        s = list(c)
        pos = rng.choice(L, size=L // 10, replace=False)
        for p in pos:
            s[p] = "N"
        edge.append("".join(s))
        s[pos[0]] = c[pos[0]]
        edge.append("".join(s))
    for c in cand(4):                                                               # one base on half of the read
        edge.append("A" * (L // 2) + c[L // 2:])
        edge.append("A" * (L // 2 - 1) + c[L // 2 - 1:])
    two = list(rand(L).replace("C", "A").replace("G", "T"))                         # two bases at most twice
    two[3], two[7], two[11] = "C", "G", "C"
    edge.append("".join(two))
    two[11] = "G"
    edge.append("".join(two))
    for l in (1, 5, 8, 9, 10, 22, 31):                                              # shorter than k, around k, short
        edge += cand_len(l) + [rand(l)]
    for l in (MAX_READ - 1, MAX_READ, MAX_READ + 1, MAX_READ + 90):                 # the device limit and past it
        edge += cand_len(l, 3) + [rand(l)]
    pairs = [(e, rand(L)) for e in edge]
    pairs += [(rand(L), e) for e in edge[::3]]
    only2 = cand(8)                                                                 # only read 2 is a candidate
    pairs += [(rand(L), c) for c in only2]
    pairs += [("A" * L, c) for c in only2[:2]]
    pairs += [(rand(L), rand(L)) for _ in range(8)]                                 # neither
    long2 = cand_len(MAX_READ + 1, 4)                                               # long read 2, short read 1
    pairs += [(rand(L), c) for c in long2]
    return pairs


def fastq_records(ids, seqs, qual_char="I"):
    return "".join("@%s\n%s\n+\n%s\n" % (i, s, qual_char * len(s)) for i, s in zip(ids, seqs))


def write_text(path, text, gz=False):
    if gz:
        with gzip.open(path, "wt", compresslevel=1) as f:
            f.write(text)
    else:
        with open(path, "w") as f:
            f.write(text)
    return path


def write_pairs(tmp, name, r1, r2, gz=False, mate_suffix=True):
    """<tmp>/<name>_1.fq[.gz] and _2.fq[.gz]; ids p<i>/1 and p<i>/2 (the Illumina mate suffix) unless mate_suffix is False."""
    ext = ".fq.gz" if gz else ".fq"
    ids = ["p%d" % i for i in range(len(r1))]
    s1, s2 = ("/1", "/2") if mate_suffix else ("", "")
    f1 = write_text(os.path.join(tmp, name + "_1" + ext), fastq_records([i + s1 for i in ids], r1), gz)
    f2 = write_text(os.path.join(tmp, name + "_2" + ext), fastq_records([i + s2 for i in ids], r2), gz) if r2 is not None else None
    return f1, f2


def mixed_set(seed, npairs, L, decoy=0.6, edges=True, head=1000):
    """npairs pairs of length L plus the edge pairs, the edge pairs after the first `head` pairs (which set
    hitLenRequired, FastqExtractor.cpp:436-455).  Returns the two lists of read strings."""
    rng = np.random.default_rng([seed, 0x5E0])
    clones = synth.make_clones(40, seed)
    a, b = bulk_pairs(rng, clones, npairs, L, decoy)
    r1 = [_s(x) for x in a]
    r2 = [_s(x) for x in b]
    if edges:
        ep = edge_pairs(rng, clones, L)
        at = np.sort(rng.integers(min(head, npairs), npairs + 1, size=len(ep)))[::-1]
        for (x, y), p in zip(ep[::-1], at):
            r1.insert(int(p), x)
            r2.insert(int(p), y)
    return r1, r2


def write_bulk_fastq(path1, path2, seed, npairs, L, decoy, chunk=200000, gz=False):
    """A large pair set straight to disk, chunk by chunk (bench/stage0_extract.py, the GPU size test)."""
    rng = np.random.default_rng([seed, 0xB0C])
    clones = synth.make_clones(200, seed)
    q = b"I" * L
    op = (lambda p: gzip.open(p, "wb", compresslevel=1)) if gz else (lambda p: open(p, "wb"))
    with op(path1) as f1, op(path2) as f2:
        for c0 in range(0, npairs, chunk):
            n = min(chunk, npairs - c0)
            a, b = bulk_pairs(rng, clones, n, L, decoy)
            for f, x, m in ((f1, a, b"/1"), (f2, b, b"/2")):
                rows = LUT[x]
                f.write(b"".join(b"@p%d%s\n%s\n+\n%s\n" % (c0 + i, m, rows[i].tobytes(), q) for i in range(n)))



def barcode_inputs(tmp, seed=9, npairs=1500):
    """Paired reads with a 10x-style barcode file (28 bp: 16 bp barcode, read reverse-complemented, then the UMI), a UMI
    file, and a whitelist of the true barcodes; some barcodes carry one error the whitelist corrects, some are not on it.
    A few barcode records equal their read 1 or read 2 and are low complexity (FastqExtractor.cpp:215-221)."""
    rng = np.random.default_rng([seed, 0xBC])
    r1, r2 = mixed_set(seed, npairs, 150, edges=False)
    cells = ["".join("ACGT"[c] for c in rng.integers(0, 4, size=16)) for _ in range(40)]
    comp = str.maketrans("ACGT", "TGCA")
    bcs, umis = [], []
    for i in range(len(r1)):
        bc = cells[int(rng.integers(len(cells)))]
        if rng.random() < 0.05:
            p = int(rng.integers(16))
            bc = bc[:p] + "ACGT"[("ACGT".index(bc[p]) + 1) % 4] + bc[p + 1:]
        elif rng.random() < 0.03:
            bc = "".join("ACGT"[c] for c in rng.integers(0, 4, size=16))
        raw = bc.translate(comp)[::-1]                     # --barcodeRevComp turns it back
        bcs.append("GG" + raw + "".join("ACGT"[c] for c in rng.integers(0, 4, size=10)))
        umis.append("".join("ACGT"[c] for c in rng.integers(0, 4, size=12)))
    for j, i in enumerate(range(1100, 1100 + 12)):          # barcode == read, low complexity: dropped even with a candidate mate
        low = ("A" * 150) if j % 3 else ("AC" * 75)
        if j % 2:
            r1[i] = low
        else:
            r2[i] = low
        bcs[i] = low
    for i in range(1200, 1206):                             # barcode == read 1 but not low complexity: kept if a candidate
        bcs[i] = r1[i]
    fa = gene_fasta(os.path.join(tmp, "genes.fa"))
    f1, f2 = write_pairs(tmp, "reads", r1, r2)
    ids = ["p%d" % i for i in range(len(r1))]
    fb = write_text(os.path.join(tmp, "bc.fq"), fastq_records(ids, bcs))
    fu = write_text(os.path.join(tmp, "umi.fq"), fastq_records(ids, umis))
    wl = write_text(os.path.join(tmp, "whitelist.txt"), "".join(c + "\n" for c in cells))
    args = ["-f", fa, "-1", f1, "-2", f2, "--barcode", fb, "--barcodeStart", "2", "--barcodeEnd", "17", "--barcodeRevComp",
            "--UMI", fu, "--umiStart", "1", "--umiEnd", "10", "--barcodeWhitelist", wl]
    return args, r1 + r2


def short_set(n, seed):
    """n single-end reads, cheap for the emulation: mostly 24 bp decoys, every 50th a 150 bp candidate."""
    rng = np.random.default_rng([seed, 0x24])
    clones = synth.make_clones(20, seed)
    cand = [_s(x) for x in _candidates(rng, clones, n // 50 + 1, 150)[0]]
    dec = LUT[rng.integers(0, 4, size=(n, 24), dtype=np.uint8)]
    return [cand[i // 50] if i % 50 == 0 else dec[i].tobytes().decode() for i in range(n)]


# ---- running the stock binary and a drop-in side by side --------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INTEGRATION = os.path.join(ROOT, "integration")
STOCK = os.path.join(ROOT, "oracle", "_ref", "fastq-extractor")
GOLDEN = os.path.join(ROOT, "tests", "golden")
ROUTE = re.compile(r"\[trust4_b200\] stage-0 route: (\d+) reads scanned on the device, (\d+) on the host")


def extractor_binary(name):
    """integration/_build/<name>, (re)built by integration/Makefile where the reference sources are present; elsewhere the
    GPU binary the oracle build linked (oracle/stage0.mk: oracle/_ref/fastq-extractor-gpu).  Skips when neither exists."""
    import pytest
    if not os.path.exists(STOCK):
        pytest.skip("oracle/_ref/fastq-extractor not built")
    if subprocess.run(["make", "-s", "-C", INTEGRATION, "has-reference"], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL).returncode == 0:
        subprocess.run(["make", "-C", INTEGRATION, "_build/" + name], check=True, stdout=subprocess.DEVNULL)
        return os.path.join(INTEGRATION, "_build", name)
    built = os.path.join(ROOT, "oracle", "_ref", name)
    if os.path.exists(built):
        return built
    pytest.skip("reference sources not present (the drop-in compiles its FastqExtractor.cpp) and oracle/_ref/%s not built" % name)


def example_inputs(tmp):
    """The reference's shipped example: example_1.fq + example_2.fq against hg38_bcrtcr.fa (tests/golden/)."""
    names = ("hg38_bcrtcr.fa", "example_1.fq", "example_2.fq")
    for n in names:
        with gzip.open(os.path.join(GOLDEN, n + ".gz"), "rb") as f, open(os.path.join(tmp, n), "wb") as g:
            g.write(f.read())
    return ["-f", os.path.join(tmp, names[0]), "-1", os.path.join(tmp, names[1]), "-2", os.path.join(tmp, names[2])]


def route_counts(reads):
    """The route line's expected (device, host) counts for these read strings (every read of every mate file)."""
    n = sum(1 for r in reads if len(r) <= MAX_READ)
    return n, len(reads) - n


def run_and_compare(binary, args, tmp, threads, env=None, expect_fail=False, timeout=1800):
    """Runs the stock fastq-extractor and `binary` with the same flags at -t `threads`, each with its own -o prefix, and
    asserts the same exit status and the same files, byte for byte (.fq or _1.fq / _2.fq, _bc.fa, _umi.fa: whatever the
    stock run writes).  Returns the drop-in's route counts (None when it printed no route line) and its stderr."""
    outs = {}
    for tag, exe in (("stock", STOCK), ("dropin", binary)):
        d = os.path.join(tmp, "%s_t%d" % (tag, threads))
        os.makedirs(d, exist_ok=True)
        r = subprocess.run([exe, "-t", str(threads), "-o", os.path.join(d, "out")] + list(args), stdout=subprocess.DEVNULL,
                           stderr=subprocess.PIPE, timeout=timeout, env=dict(os.environ, **(env or {})), text=True)
        assert (r.returncode != 0) == expect_fail, (tag, r.returncode, r.stderr[-2000:])
        files = {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}
        outs[tag] = (r, files)
    (rs, fs), (rd, fd) = outs["stock"], outs["dropin"]
    assert rs.returncode == rd.returncode
    assert sorted(fs) == sorted(fd), (sorted(fs), sorted(fd))
    for f in fs:
        same = fs[f] == fd[f]       # compared outside the assert: pytest's diff of large byte strings takes minutes
        assert same, "%s differs from the stock binary's: %s" % (f, first_difference(fs[f], fd[f]))
    m = ROUTE.search(rd.stderr)
    return (tuple(int(x) for x in m.groups()) if m else None), rd.stderr, fs


def first_difference(a, b):
    la, lb = a.split(b"\n"), b.split(b"\n")
    for i, (x, y) in enumerate(zip(la, lb)):
        if x != y:
            return "line %d: %r vs %r" % (i + 1, x[:200], y[:200])
    return "%d vs %d lines" % (len(la), len(lb))


# (read length, paired, gzip, -t): hitLenRequired is 27 (paired, 100 bp: 20 < 27), 30 (150 / 5), 101 (512 / 5 = 102,
# capped), 23 (single-end, 100 bp), FastqExtractor.cpp:436-455
SYNTH = [(150, True, False, 1), (150, True, True, 3), (100, True, False, 2), (512, True, False, 1), (100, False, True, 1),
         (150, False, False, 4)]
SYNTH_IDS = ["%dbp-%s%s-t%d" % (L, "pe" if p else "se", "-gz" if g else "", t) for L, p, g, t in SYNTH]


# ---- the cases, for the emulation (test_extractor_cli.py) and the GPU binary (test_gpu_extractor.py) -----------------
def case_shipped_example(binary, tmp, threads):
    """example_1.fq + example_2.fq against hg38_bcrtcr.fa.  Its read ids end in /1 and /2, which the stock binary
    strips at -t 1 only: the drop-in must write what the stock binary writes at each -t."""
    args = example_inputs(tmp)
    counts, _, files = run_and_compare(binary, args, tmp, threads)
    assert counts == (2 * 198, 0)
    assert len(files["out_1.fq"]) > 0


def case_synthetic_with_edges(binary, tmp, L, paired, gz, threads):
    """Candidates and decoys plus the edge reads (edge_pairs: low complexity, N's, only read 2 a candidate, neither,
    shorter than k, exactly T4_MAX_READ_LEN and longer)."""
    r1, r2 = mixed_set(40 + L + threads, 1500, L)
    fa = gene_fasta(os.path.join(tmp, "genes.fa"))
    f1, f2 = write_pairs(tmp, "reads", r1, r2 if paired else None, gz=gz, mate_suffix=paired)
    args = ["-f", fa, "-1", f1, "-2", f2] if paired else ["-f", fa, "-u", f1]
    counts, _, files = run_and_compare(binary, args, tmp, threads)
    assert counts == route_counts(r1 + r2 if paired else r1)
    assert counts[1] > 0                                   # reads over the device limit went to the host
    kept = files["out_1.fq" if paired else "out.fq"].count(b"\n") // 4
    assert 200 < kept < len(r1) - 200, kept                 # both outcomes occur


def case_single_end(binary, tmp, threads):
    """-u: one read file, <prefix>.fq."""
    r1, _ = mixed_set(7, 2000, 150, edges=False)
    fa = gene_fasta(os.path.join(tmp, "genes.fa"))
    f1, _ = write_pairs(tmp, "reads", r1, None, mate_suffix=False)
    counts, _, files = run_and_compare(binary, ["-f", fa, "-u", f1], tmp, threads)
    assert counts == (2000, 0) and sorted(files) == ["out.fq"]


def case_barcode_umi_whitelist(binary, tmp, threads, extra):
    args, reads = barcode_inputs(tmp)
    counts, _, files = run_and_compare(binary, args + list(extra), tmp, threads)
    assert counts == route_counts(reads)
    assert sorted(files) == ["out_1.fq", "out_2.fq", "out_bc.fa", "out_umi.fa"]
    assert files["out_bc.fa"].count(b">") == files["out_1.fq"].count(b"\n") // 4 > 100


def case_read_format_range(binary, tmp, threads):
    """--readFormat with a range on read 1 (ReadFormatter cuts the output; the candidate test sees the whole read)."""
    r1, r2 = mixed_set(11, 1500, 150, edges=False)
    fa = gene_fasta(os.path.join(tmp, "genes.fa"))
    f1, f2 = write_pairs(tmp, "reads", r1, r2)
    counts, _, files = run_and_compare(binary, ["-f", fa, "-1", f1, "-2", f2, "--readFormat", "r1:10:109"], tmp, threads)
    assert counts == (2 * len(r1), 0)
    assert b"\n" + b"I" * 100 + b"\n" in files["out_1.fq"]


def case_batch_size_edges(binary, tmp, n):
    """A read count of exactly one batch (2^18 reads at -t 1), one more (a second batch of one read), and an empty read
    file (the stock binary stops with "Read file is empty." before writing anything)."""
    reads = short_set(n, 5)
    fa = gene_fasta(os.path.join(tmp, "genes.fa"))
    f1, _ = write_pairs(tmp, "reads", reads, None, mate_suffix=False)
    counts, err, files = run_and_compare(binary, ["-f", fa, "-u", f1], tmp, 1, expect_fail=(n == 0))
    if n == 0:
        assert counts is None and files == {} and "Read file is empty." in err
    else:
        assert counts == (n, 0)
        assert files["out.fq"].count(b"\n") // 4 > n // 100
        m = re.search(r"\((\d+) batches", err)
        assert int(m.group(1)) == (1 if n == 1 << 18 else 2)


def case_large(binary, tmp, npairs, threads):
    """A read set of a size a user runs: npairs pairs of 150 bp, 90 % decoys, at -t `threads`."""
    fa = gene_fasta(os.path.join(tmp, "genes.fa"))
    f1, f2 = os.path.join(tmp, "reads_1.fq"), os.path.join(tmp, "reads_2.fq")
    if not os.path.exists(f2):
        write_bulk_fastq(f1, f2, 3, npairs, 150, 0.9)
    counts, _, files = run_and_compare(binary, ["-f", fa, "-1", f1, "-2", f2], tmp, threads)
    assert counts == (2 * npairs, 0)
    assert files["out_1.fq"].count(b"\n") // 4 > npairs // 20
