"""CPU checks of the engine's bit-exact logic through the TEST-ONLY emulation build (tests/emu): the same
t4_engine.h compiled by g++ with one emulated thread per stream.  The product path is exercised by
test_gpu_parity.py on the GPU; this module only guards the logic while developing without a GPU."""
import pytest

import parity_cases as pc


@pytest.mark.parametrize("name", ["example", "synth2k"])
def test_emu_trace_replay(emu_lib, name):
    pc.check_trace_replay(emu_lib, name)


@pytest.mark.parametrize("seed,shards", [(1, 1), (2, 3), (3, 8)])
def test_emu_batch_vs_reference(emu_lib, ref_or_golden, seed, shards):
    assert pc.check_batch_vs_ref(emu_lib, ref_or_golden, seed, shards) > 100


def test_emu_batch_dealt_shards(emu_lib, ref_or_golden):
    assert pc.check_batch_vs_ref(emu_lib, ref_or_golden, 6, 5, nclones=30, npairs=600, deal=True) > 100


def test_emu_batch_gene_grouped_shards(emu_lib, ref_or_golden):
    assert pc.check_batch_vs_ref(emu_lib, ref_or_golden, 8, 9, nclones=40, npairs=700, group="gene") > 100


def test_emu_stage_parity(emu_lib, ref):
    pc.check_stage_parity(emu_lib, ref, "synth2k", every=131, max_checks=25)


def test_emu_dp(emu_lib, ref):
    pc.check_dp(emu_lib, ref)
    pc.check_dp_hot(emu_lib, ref, 11, 0)      # t4_dp_equal, the register DP of the hot path (host-compilable)


def test_emu_probe_batch(emu_lib, ref):
    """API plumbing of t4_streams_get_hits (the emulation answers through the engine's own GetHitsFromRead)."""
    pc.check_probe_batch(emu_lib, ref, sample=60)


def test_emu_big_repeats(emu_lib, ref):
    pc.check_big_repeats(emu_lib, ref)


def test_emu_barcode_mode(emu_lib, ref):
    pc.check_barcode_mode(emu_lib, ref)


def test_emu_barcode_release(emu_lib, ref):
    pc.check_barcode_release(emu_lib, ref)


def test_emu_single_cell_streams(emu_lib, ref):
    pc.check_single_cell(emu_lib, ref)
    pc.check_single_cell(emu_lib, ref, seed=52, n_barcodes=9, reads_per_barcode=260, n_shards=2, contig_min_cov=3)


def test_emu_repseq_streams(emu_lib, ref):
    pc.check_repseq(emu_lib, ref)


def test_emu_dup_runs(emu_lib, ref):
    pc.check_dup_runs(emu_lib, ref)


def test_emu_input_novel_fa(emu_lib, ref, tmp_path):
    pc.check_input_novel_fa(emu_lib, ref, tmp_path)


def test_emu_single_stream_at_scale(emu_lib, ref_or_golden):
    """One stream, 80 000 reads: thousands of contigs, ChangeKmerLength 9 -> 11 in mid-run (slot compaction + full
    re-index), periodic UpdateAllConsensus, reads with more than 50 candidate overlaps (the order-dependent
    bestNovelOverlap pre-filters, SeqSet.hpp:1705-1794), postings lists over the 100-entry skip rule.
    (The same check on 300 000 reads / 10 019 contigs / 58 overlaps per read also passes -- 4.5 min, not part of the suite.)"""
    from trust4_b200 import synth
    cfg = synth.run_cfg(change_k_threshold=1500)
    n = pc.check_batch_vs_ref(emu_lib, ref_or_golden, 43, 1, nclones=3000, npairs=40000, cfg=cfg)
    assert n > 70000


@pytest.mark.parametrize("seed,shards,kmer,drop", [(81, 1, 17, 0.0), (82, 4, 17, 0.15), (83, 3, 19, 0.0)])
def test_emu_assign_pass(emu_lib, ref, seed, shards, kmer, drop):
    """SURVEY.md 8f-2: InputSeqSet + AssignRead of every assembled read + RecomputePosWeight (main.cpp:2047-2118)."""
    listed, assigned = pc.check_assign_pass(emu_lib, ref, seed, shards, nclones=30, npairs=500, kmer=kmer, drop=drop)
    assert listed > 500 and assigned > 300


def test_emu_assign_pass_noisy_and_duplicates(emu_lib, ref):
    """Reads AssignRead cannot place (4 % substitutions: several ExtendOverlap attempts per read, some -1 results) and
    amplicon data where most list neighbours are identical strings and share one AssignRead call."""
    from trust4_b200 import synth
    cl = synth.make_clones(60, 92)
    w = synth.build_workload(cl, synth.sample_pairs(cl, 1200, 150, 92, sub_rate=0.04))
    listed, assigned = pc.check_assign_pass(emu_lib, ref, 92, 2, workload=w)
    assert listed - assigned > 50
    cl = synth.make_clones(9, 95, chains=("TRB",))
    w = synth.build_workload(cl, synth.sample_amplicon(cl, 5000, 100, 95, alpha=0.7, sub_rate=0.002), repseq=True)
    pc.check_assign_pass(emu_lib, ref, 95, 2, workload=w, cfg=synth.run_cfg(repetitive=1, first_read_len=100))


@pytest.mark.parametrize("k", [21, 9, 31])
def test_emu_kmer_count_stats(emu_lib, ref, k):
    """SURVEY.md 8f-3: canonical k-mer counts + per-read min / median / avg (KmerCount.hpp) -- the numbers that order the reads."""
    assert pc.check_kmer_count_stats(emu_lib, ref, seed=100 + k, k=k) >= 1500


@pytest.mark.parametrize("seed,radius,hit_len", [(121, None, 27), (122, 0, 23), (123, 10, 31)])
def test_emu_refset_scan(emu_lib, ref, tmp_path, seed, radius, hit_len):
    """SURVEY.md 8f-4: fastq-extractor's candidate predicate (InputRefFa + IsLowComplexity + HasHitInSet(read, 0))."""
    assert pc.check_refset_scan(emu_lib, ref, tmp_path, seed=seed, radius=radius, hit_len=hit_len) > 100


@pytest.mark.parametrize("seed,radius,hit_len", [(131, None, 31), (132, 0, 27), (133, 10, 21)])
def test_emu_refset_overlaps(emu_lib, ref, tmp_path, seed, radius, hit_len):
    """SURVEY.md 8f-1, first half: SeqSet::GetOverlapsFromRead on the reference gene set (emulation only, see t4_annot.h)."""
    assert pc.check_refset_overlaps(emu_lib, ref, tmp_path, seed=seed, radius=radius, hit_len=hit_len) > 500


@pytest.mark.parametrize("seed,radius,hit_len", [(141, None, 31), (142, 0, 27), (143, 10, 21)])
def test_emu_refset_annotate(emu_lib, ref, tmp_path, seed, radius, hit_len):
    """SURVEY.md 8f-1: SeqSet::AnnotateRead(read, 0, ...) on the reference gene set (emulation only, see t4_annot.h)."""
    assert pc.check_refset_annotate(emu_lib, ref, tmp_path, seed=seed, radius=radius, hit_len=hit_len) > 300


def test_emu_sort_reads(emu_lib, ref):
    """SURVEY.md 8f-3, the sort: std::sort(sortedReads) with _sortRead::operator< (emulation only, see t4_readsort.h)."""
    import numpy as np
    from trust4_b200 import api
    assert pc.check_sort_reads(emu_lib, ref) == 5000
    assert pc.check_sort_reads(emu_lib, ref, seed=152, n=777) == 777          # not a power of two: ragged last runs
    pool = np.frombuffer(b"ACGTACGTAC" + b"\0" * 16, dtype=np.uint8).copy()
    for n in (0, 1, 2, 3):
        order = api.sort_reads(pool, np.arange(n, dtype=np.uint64), np.full(n, 5, dtype=np.int32), ["r%d" % (9 - i) for i in range(n)],
                               np.ones(n, np.int32), np.ones(n, np.int32), np.ones(n, np.float32), emu_lib)
        reads = [bytes(pool[i:i + 5]).decode() for i in range(n)]
        assert order.tolist() == ref.sort_reads(reads, ["r%d" % (9 - i) for i in range(n)], np.ones(n), np.ones(n), np.ones(n)).tolist()


def test_emu_mate_overlap(emu_lib, ref):
    """SURVEY.md 8f-3, mate read-through / merge detection: AlignAlgo::IsMateOverlap per pair (emulation only)."""
    assert pc.check_mate_overlap(emu_lib, ref) > 600


@pytest.mark.parametrize("seed,radius,hit_len,k", [(134, None, 31, 11), (135, 0, 17, 7)])
def test_emu_refset_overlaps_other_k(emu_lib, ref, tmp_path, seed, radius, hit_len, k):
    """GetOverlapsFromRead on gene sets indexed at k = 11 and at k = 7 with hitLenRequired 17 (the --trimLevel 2 re-index)."""
    assert pc.check_refset_overlaps(emu_lib, ref, tmp_path, seed=seed, n=300, radius=radius, hit_len=hit_len, k=k) > 300


def test_emu_refset_annotate_example(emu_lib, ref, tmp_path):
    """AnnotateRead of the shipped example's reads on the reference's hg38 gene set."""
    pc.check_refset_annotate_example(emu_lib, ref, tmp_path)


def test_emu_refset_annotate_batches(emu_lib, ref, tmp_path):
    """Batch sizes around the emulation's worker count (2), n = 0, a repeated batch byte for byte."""
    pc.check_refset_annotate_batches(emu_lib, ref, tmp_path, n_workers=2)


def test_emu_refset_interleaved(emu_lib, ref, tmp_path):
    pc.check_refset_interleaved(emu_lib, ref, tmp_path, n=300)


def test_emu_refset_error_isolation(emu_lib, ref, tmp_path):
    """A read over the per-read hit limit fails its own call only; the gene set and its worker shells stay usable."""
    pc.check_refset_error_isolation(emu_lib, ref, tmp_path, batch=12)


def test_emu_sort_reads_edges(emu_lib, ref):
    """Bytes >= 0x80, reads over 512 bp, avg one ulp apart and -0.0 / 0.0, groups of records equal in every field."""
    assert pc.check_sort_reads_edges(emu_lib, ref, n_base=600) > 1000


def test_emu_sort_reads_python_key(emu_lib):
    """The sort against the plain Python restatement of the comparator, ragged size."""
    assert pc.check_sort_reads_large(emu_lib, n=20011) == 20011


def test_emu_mate_overlap_edges(emu_lib, ref):
    """Zero-length mates, minOverlap >= flen and 0, the threshold steps at 50 / 100 bases, N's, lower case, tandem repeats."""
    assert pc.check_mate_overlap_edges(emu_lib, ref, reps=3) > 200
