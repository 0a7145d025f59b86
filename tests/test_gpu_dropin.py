"""The drop-in stage-1 binaries on the GPU, end to end: a whole FASTQ run through the unmodified reference driver with
every offloaded pass on the device, compared byte for byte (_raw.out, _final.out, _assembled_reads.fa) with the stock
binary (oracle/_ref/trust4) on the same inputs and flags at -t 1.  Only such runs show how the passes combine in one
process: the rough annotation's resident workers sharing one read cursor, the collective index primitive's directory
claims and growth, the AssignRead workers' follower writes, several passes sharing one arena and the library's streams.

Every batch case lists the `[trust4_b200] batch route: ...` lines it expects and asserts exactly those: each adapter pass
quietly leaves the work to the CPU code when one of its conditions fails, and a byte-identical output would then prove
nothing about the device.  The driver reaches the AssignRead pass only for paired-end input without --barcode and
without --skipMateExtension (main.cpp:2018).  The k-mer statistics pass does not apply with --contigMinCov (reads may be
removed after counting).  Inputs and the comparison: test_dropin_cli.py; emulation twins there and in
test_emu_barcode_stats.py."""
import os
import re
import subprocess

import pytest

from test_dropin_cli import (_degrade_qualities, dropin_binary, dropin_env, example_inputs, run_and_compare,
                             write_barcode_inputs, write_inputs)

pytestmark = pytest.mark.gpu

# the stderr line of each batch pass (integration/t4_seqset_adapter.hpp), most specific pattern first
PASSES = (("bcstats", "per-cell 21-mer statistics and barcode sort on the device"),
          ("kmerstats", "21-mer statistics on the device"),
          ("sort", "reads sorted on the device"),
          ("annotate", "rough annotation on the device"),
          ("streams", "device stream(s)"),
          ("assign", "AssignRead pass on the device"))
PRE = {"T4_KMERSTATS": "1", "T4_SORT": "1", "T4_ANNOTATE": "1"}         # the opt-in pre-processing lines of bulk input
PAIRED = ("streams", "assign")                                           # the default passes of paired-end bulk input


def route_passes(stderr):
    """The batch passes that reported on stderr, one name per line, sorted."""
    out = []
    for line in stderr.splitlines():
        if line.startswith("[trust4_b200] batch route: "):
            out.append(next(name for name, pat in PASSES if pat in line))
    return sorted(out)


def batch(tmp, args, expect, extra=(), env=None):
    """The batch drop-in at T4_STREAMS=1 against the stock binary; exactly the passes `expect` must have run."""
    e = {"T4_STREAMS": "1"}
    e.update(env or {})
    err = run_and_compare(dropin_binary("trust4_gpu_batch"), args, tmp, extra=extra, env=e)
    assert route_passes(err) == sorted(expect), err[-1500:]
    return err


def per_call(tmp, args, extra=()):
    err = run_and_compare(dropin_binary("trust4_gpu"), args, tmp, extra=extra)
    assert route_passes(err) == [], err[-1500:]


def trimmed(err):
    m = re.search(r"21-mer statistics on the device, (\d+) of (\d+) reads trimmed", err)
    return int(m.group(1))


def threshold_tails(prefix, seed):
    """Give a quarter of the reads of <prefix>_1.fq / _2.fq a tail of qualities around the trimming threshold: Phred 14
    ('/', bad: `qual - 32 <= 15`, KmerCount.hpp:252), 15 ('0', good: one above it) and 16 ('1'), with a third of the tail
    bases changed so that its k-mers are singletons and the trimming scan reaches it.  A threshold off by one moves the
    cut of most of these reads."""
    import numpy as np
    rng = np.random.default_rng(seed)
    for m in ("_1.fq", "_2.fq"):
        lines = open(prefix + m).read().split("\n")
        for i in range(3, len(lines), 4):
            if lines[i] and rng.random() < 0.25:
                n = len(lines[i])
                q = int(rng.integers(n // 2, n - 10))
                lines[i] = lines[i][:q] + "".join("/01"[int(x)] for x in rng.integers(0, 3, size=n - q))
                seq = list(lines[i - 2])
                for x in range(q, n):
                    if rng.random() < 0.33:
                        seq[x] = "ACGT"[int(rng.integers(4))]
                lines[i - 2] = "".join(seq)
        open(prefix + m, "w").write("\n".join(lines))


def single_end_inputs(tmp, npairs, nclones, seed):
    """-u input without barcodes: the first mates of write_inputs, a quarter of them with a tail at the quality threshold."""
    args = write_inputs(tmp, npairs, nclones, seed)
    threshold_tails(os.path.join(tmp, "reads"), seed)
    return args[:2] + ["-u", args[3]]


# ---- GPU twins of the emulation-only batch tests (test_dropin_cli.py) ------------------------------------------------

def test_batch_gpu_shipped_example(tmp_path):
    """BASELINE.json configs[0]: example_1.fq + example_2.fq, -f hg38_bcrtcr.fa."""
    batch(str(tmp_path), example_inputs(str(tmp_path)), PAIRED)


def test_batch_gpu_synthetic(tmp_path):
    batch(str(tmp_path), write_inputs(str(tmp_path)), PAIRED)


@pytest.mark.parametrize("on", [True, False])
def test_batch_gpu_assign_pass(tmp_path, on):
    """The AssignRead pass on the device (default) and on the CPU (T4_ASSIGN=0); _final.out depends on its assignments."""
    batch(str(tmp_path), write_inputs(str(tmp_path), 2500, 80, 31), PAIRED if on else ("streams",),
          env=None if on else {"T4_ASSIGN": "0"})


@pytest.mark.parametrize("case", ["synthetic", "example", "repseq"])
def test_batch_gpu_annotate(tmp_path, case):
    """T4_ANNOTATE=1: the rough annotation on a gene set rebuilt on the device from the -f file; --trimLevel 2 re-indexes
    it at k = 7, radius 0 (main.cpp:766-771, 1082-1083)."""
    tmp = str(tmp_path)
    if case == "synthetic":
        batch(tmp, write_inputs(tmp, 1500, 50, 33), PAIRED + ("annotate",), env={"T4_ANNOTATE": "1"})
    elif case == "example":
        batch(tmp, example_inputs(tmp), PAIRED + ("annotate",), env={"T4_ANNOTATE": "1"})
    else:
        batch(tmp, write_inputs(tmp, 800, 25, 34), ("streams", "annotate"), extra=("--trimLevel", "2", "--skipMateExtension"),
              env={"T4_ANNOTATE": "1"})


def test_batch_gpu_all_passes(tmp_path):
    """Every bulk pass on the device, on reads whose low-quality tails really get trimmed."""
    tmp = str(tmp_path)
    args = write_inputs(tmp, 1500, 50, 35)
    _degrade_qualities(os.path.join(tmp, "reads"))
    err = batch(tmp, args, PAIRED + ("kmerstats", "sort", "annotate"), env=PRE)
    assert trimmed(err) > 100, err[-1500:]


def test_batch_gpu_repseq_and_min_cov(tmp_path):
    batch(str(tmp_path), write_inputs(str(tmp_path), 800, 25, 22), ("streams",),
          extra=("--trimLevel", "2", "--skipMateExtension", "--contigMinCov", "2"))


def test_batch_gpu_barcodes_min_cov(tmp_path):
    batch(str(tmp_path), write_barcode_inputs(str(tmp_path)), ("streams",), extra=("--contigMinCov", "4"))


# ---- GPU twins of the per-call tests -----------------------------------------------------------------------------------

def test_dropin_gpu_shipped_example(tmp_path):
    per_call(str(tmp_path), example_inputs(str(tmp_path)))


def test_dropin_gpu_repseq_flags(tmp_path):
    per_call(str(tmp_path), write_inputs(str(tmp_path), 800, 25, 22), extra=("--trimLevel", "2", "--skipMateExtension"))


def test_dropin_gpu_contig_min_cov(tmp_path):
    per_call(str(tmp_path), write_inputs(str(tmp_path), 800, 25, 24), extra=("--contigMinCov", "3"))


@pytest.mark.parametrize("extra", [(), ("--contigMinCov", "4")])
def test_dropin_gpu_barcodes_per_call(tmp_path, extra):
    per_call(str(tmp_path), write_barcode_inputs(str(tmp_path)), extra=extra)


# ---- edges the emulation twins do not reach -----------------------------------------------------------------------------

def test_batch_gpu_trim_level_0(tmp_path):
    """--trimLevel 0: the device k-mer statistics run without qualities (no quality trimming), with the other passes."""
    tmp = str(tmp_path)
    args = write_inputs(tmp, 1500, 50, 36)
    _degrade_qualities(os.path.join(tmp, "reads"))
    batch(tmp, args, PAIRED + ("kmerstats", "sort", "annotate"), extra=("--trimLevel", "0"), env=PRE)


def test_batch_gpu_single_end(tmp_path):
    """-u input without barcodes, every opt-in line set: no AssignRead pass (no mates), no per-cell pass (no barcodes)."""
    tmp = str(tmp_path)
    err = batch(tmp, single_end_inputs(tmp, 2000, 50, 37), ("streams", "kmerstats", "sort", "annotate"),
                env=dict(PRE, T4_BCSTATS="1"))
    assert trimmed(err) > 100, err[-1500:]


@pytest.mark.parametrize("extra", [(), ("--contigMinCov", "4")])
def test_batch_gpu_many_cells(tmp_path, extra):
    """A barcoded run of 300 cells (two clonotypes each, plus ambient reads) with the per-cell statistics, the read sort
    and the rough annotation on the device; --contigMinCov 4 also drops the cells with fewer than 4 reads."""
    tmp = str(tmp_path)
    args = write_barcode_inputs(tmp, 6000, 600, 300, 41)
    err = batch(tmp, args, ("streams", "sort", "annotate", "bcstats"), extra=extra,
                env={"T4_BCSTATS": "1", "T4_SORT": "1", "T4_ANNOTATE": "1"})
    cells = int(re.search(r"reads in (\d+) cells", err).group(1))
    assert cells >= 250, err[-1500:]


def test_batch_gpu_large_bulk(tmp_path):
    """30 000 pairs with every line on: the rough annotation hands each of its 528 resident workers about 100 reads, the
    read sort merges many runs, the AssignRead workers take many 8-slot batches.  Read tails at the quality threshold.
    The stock binary takes about a minute on it."""
    tmp = str(tmp_path)
    args = write_inputs(tmp, 30000, 600, 43)
    threshold_tails(os.path.join(tmp, "reads"), 43)
    err = batch(tmp, args, PAIRED + ("kmerstats", "sort", "annotate"), env=dict(PRE, T4_BCSTATS="1"))
    assert trimmed(err) > 1000, err[-1500:]


# ---- read-sharded runs (S > 1) ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("streams", [3, 64])
def test_batch_gpu_sharded_runs(tmp_path, streams):
    """S > 1 with the pre-processing lines on.  The output differs from the unsharded run by definition, so only the
    invariants of test_batch_emu_sharded_runs are checked: global slot names are unique, every assembled read is
    reported once, and grouping the reads by gene (T4_SHARD_BY=gene) fragments the assembly no more than rank blocks."""
    tmp = str(tmp_path)
    args = write_inputs(tmp, 3000, 80, 25)
    binary = dropin_binary("trust4_gpu_batch")
    n_contigs = {}
    for by in ("gene", "rank"):
        pre = os.path.join(tmp, "s%d%s" % (streams, by))
        r = subprocess.run([binary, "-t", "1", "-o", pre] + args, check=True, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE,
                           timeout=900, text=True, env=dropin_env(binary, dict(PRE, T4_STREAMS=str(streams), T4_SHARD_BY=by)))
        assert route_passes(r.stderr) == sorted(PAIRED + ("kmerstats", "sort", "annotate")), r.stderr[-1500:]
        s = int(re.search(r"reads on (\d+) device stream", r.stderr).group(1))
        assert 1 < s <= streams, r.stderr[-1500:]
        names = [l.split()[0] for l in open(pre + "_raw.out") if l.startswith(">")]
        assert len(names) > 5 and len(set(names)) == len(names)
        reads = [l for l in open(pre + "_assembled_reads.fa") if l.startswith(">")]
        assert len(reads) > 3000 and len(set(reads)) == len(reads)
        n_contigs[by] = len(names)
    assert n_contigs["gene"] <= n_contigs["rank"], n_contigs
