"""The stream kernel and the AssignRead pass on reads of 201-512 bp in a short-read set, on the GPU, against the compiled
reference: overlap-scoring gaps around the arena limit (192 columns) and the gap limit, ExtendOverlap sides of 0-472
columns on half-warp pairs, the deferred-side list past one ballot word, contig growth, the hit sort around 1024 keys, and
the batch loop and the AssignRead pass on a workload of merged mates and long reads."""
import pytest

import long_read_cases as lr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", [9, 7])
def test_gpu_gap_scoring(gpu_lib, ref, k):
    assert lr.check_gap_scoring(gpu_lib, ref, k) > 0


@pytest.mark.parametrize("n_overlaps", [8, 20, 55])
def test_gpu_extend_sides(gpu_lib, ref, n_overlaps, record_property):
    fallbacks = lr.check_extend_sides(gpu_lib, ref, n_overlaps)
    # counter 21 (ExtendOverlap made exact on demand by the decision loop) per read: (read index, (left, right), count)
    record_property("counter_21", fallbacks)
    record_property("counter_21_total", sum(c for _, _, c in fallbacks))


@pytest.mark.parametrize("n_overlaps", [8, 20])
def test_gpu_extend_sides_batch(gpu_lib, ref, n_overlaps):
    lr.check_extend_sides_batch(gpu_lib, ref, n_overlaps)


def test_gpu_contig_growth(gpu_lib, ref):
    lr.check_contig_growth(gpu_lib, ref)


@pytest.mark.parametrize("kind", lr.KEY_SETS)
def test_gpu_hit_sort(gpu_lib, ref, kind):
    lr.check_hit_sort(gpu_lib, ref, kind)


@pytest.mark.parametrize("n_streams", [1, 3])
def test_gpu_mixed_batch(gpu_lib, ref, n_streams):
    lr.check_mixed_batch(gpu_lib, ref, n_streams)


@pytest.mark.parametrize("kmer", [17, 19])
def test_gpu_mixed_assign(gpu_lib, ref, kmer):
    lr.check_mixed_assign(gpu_lib, ref, kmer)
