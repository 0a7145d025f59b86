"""The stage-1 preprocessing entry points on the GPU, against the oracle (oracle/_ref/libt4ref.so) or a plain Python
restatement: the rough annotation on the reference gene set (t4_refset_get_overlaps / t4_refset_annotate, t4_annot_kernel),
the read sort (t4_sort_reads, t4_readsort_kernel) and the mate overlap test (t4_mate_overlap_batch, t4_mate_overlap_kernel).
The sizes are chosen for the device: hundreds of annotation workers drawing reads from one cursor, and sort / mate-overlap
launches larger than one grid so that the grid-stride loops turn more than once."""
import pytest

import parity_cases as pc

pytestmark = pytest.mark.gpu

MIN_BLOCKS = 4   # resident CTAs per SM of the op kernels (T4_MIN_BLOCKS): the annotation and scan launch SMs x 4 workers


@pytest.fixture(scope="module")
def n_workers():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * MIN_BLOCKS


@pytest.mark.parametrize("seed,radius,hit_len,k", [(131, None, 31, 9), (132, 0, 27, 9), (133, 10, 21, 9), (134, None, 31, 11),
                                                   (135, 0, 17, 7)])
def test_gpu_refset_overlaps(gpu_lib, ref, tmp_path, seed, radius, hit_len, k):
    """SeqSet::GetOverlapsFromRead(read, 0, -1, 0, false) on the gene set: every overlap's gene, coordinates, strand,
    matchCnt, indelCnt and similarity double, in order.  k = 7 with hitLenRequired 17 is the --trimLevel 2 re-index."""
    assert pc.check_refset_overlaps(gpu_lib, ref, tmp_path, seed=seed, radius=radius, hit_len=hit_len, k=k) > 500


@pytest.mark.parametrize("seed,radius,hit_len", [(141, None, 31), (142, 0, 27), (143, 10, 21)])
def test_gpu_refset_annotate(gpu_lib, ref, tmp_path, seed, radius, hit_len):
    """SeqSet::AnnotateRead(read, 0, ...) for 4000 reads: about 8 reads per worker."""
    assert pc.check_refset_annotate(gpu_lib, ref, tmp_path, seed=seed, n=4000, radius=radius, hit_len=hit_len) > 2000


def test_gpu_refset_annotate_example(gpu_lib, ref, tmp_path):
    """The shipped example's 396 reads on the reference's hg38 gene set."""
    pc.check_refset_annotate_example(gpu_lib, ref, tmp_path)


def test_gpu_refset_annotate_batches(gpu_lib, ref, tmp_path, n_workers):
    """n = 1, 37, workers - 1, workers, workers + 1, 3 x workers + 5; n = 0; the same batch twice byte for byte."""
    assert n_workers - 1 in pc.check_refset_annotate_batches(gpu_lib, ref, tmp_path, n_workers)


def test_gpu_refset_interleaved(gpu_lib, ref, tmp_path):
    """scan -> annotate -> scan -> get_overlaps -> annotate on one set, sharing the worker shells."""
    pc.check_refset_interleaved(gpu_lib, ref, tmp_path, n=2000)


def test_gpu_refset_error_isolation(gpu_lib, ref, tmp_path, n_workers):
    """One read over the per-read hit limit fails its own call only.  Batches of more reads than workers keep the worker
    count of annotate and scan the same, so every call reuses the shells the failed one used."""
    pc.check_refset_error_isolation(gpu_lib, ref, tmp_path, batch=n_workers + 72)


def test_gpu_sort_reads(gpu_lib, ref):
    """std::sort with _sortRead::operator< (the emulation test's cases): 5000 and 777 records, 0 .. 3 records."""
    assert pc.check_sort_reads(gpu_lib, ref) == 5000
    assert pc.check_sort_reads(gpu_lib, ref, seed=152, n=777) == 777
    pc.check_sort_reads_tiny(gpu_lib, ref)


def test_gpu_sort_reads_large(gpu_lib):
    """2^20 + 3 records: more than one grid (sms x 16 CTAs of 256 threads), a ragged last run; Python comparator."""
    assert pc.check_sort_reads_large(gpu_lib) == (1 << 20) + 3


def test_gpu_sort_reads_edges(gpu_lib, ref):
    """Bytes >= 0x80, reads over 512 bp, avg one ulp apart and -0.0 / 0.0, groups of records equal in every field."""
    assert pc.check_sort_reads_edges(gpu_lib, ref) > 2000


def test_gpu_mate_overlap(gpu_lib, ref):
    """AlignAlgo::IsMateOverlap per pair: the emulation test's 3000 pairs, then 300 000 (more than one grid of 128-thread
    CTAs), every pair against the reference."""
    assert pc.check_mate_overlap(gpu_lib, ref) > 600
    assert pc.check_mate_overlap(gpu_lib, ref, seed=162, n=300000) > 60000


def test_gpu_mate_overlap_edges(gpu_lib, ref):
    """Zero-length mates, minOverlap >= flen and 0, mates up to 1000 bp at the 50 / 100 threshold steps, N's and lower case,
    tandem repeats of exactly 2 x minOverlap."""
    assert pc.check_mate_overlap_edges(gpu_lib, ref) > 400
