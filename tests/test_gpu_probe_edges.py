"""The k-mer lookup at its edges on the GPU: the stream engine's GetHitsFromRead and the warp-per-read probe kernel
(t4_probe_kernel) against the compiled reference, on barcodes the reference's index hashes together, postings lists of
exactly the sizes where the rules and the emit paths switch, read lengths around the packing words and the probe tiles,
the probe's counters and its key-buffer overflow."""
import pytest

import probe_cases as pb

pytestmark = pytest.mark.gpu

PAIRS = dict(pb.COLLIDING, **pb.CONTROL)
CASES = [(k, p, c) for k in (9, 15) for p in PAIRS for c in pb.COUNTS]


@pytest.mark.parametrize("k,pair,counts", CASES)
def test_gpu_colliding_barcodes(gpu_lib, ref, k, pair, counts):
    pb.check_colliding_barcodes(gpu_lib, ref, k, PAIRS[pair], pb.COUNTS[counts], seed=k)


def test_gpu_colliding_barcodes_big_list(gpu_lib, ref):
    """Barcode -1 and 1000002 together hold more than 10000 postings of the core k-mers: the `repeats > 10000` rules
    for a read without a barcode."""
    pb.check_colliding_barcodes(gpu_lib, ref, 9, PAIRS["-1~1000002"], (5000, 5001), seed=3, n_add=6)


def test_gpu_colliding_barcodes_batch(gpu_lib, ref):
    pb.check_colliding_batch(gpu_lib, ref)


@pytest.mark.parametrize("k,pair,counts", CASES + [(9, "-1~1000002", "big")])
def test_gpu_probe_barcoded_sets(gpu_lib, ref, k, pair, counts):
    pb.check_colliding_probe(gpu_lib, ref, k, PAIRS[pair], (5000, 5001) if counts == "big" else pb.COUNTS[counts], seed=k)


def test_gpu_probe_list_sizes(gpu_lib, ref):
    pb.check_list_sizes(gpu_lib, ref)


def test_gpu_probe_read_length_edges(gpu_lib, ref):
    pb.check_read_length_edges(gpu_lib, ref)


def test_gpu_probe_counters(gpu_lib, ref):
    assert pb.check_hits_counters(gpu_lib, ref) > 1000


def test_gpu_probe_key_buffer_too_small(gpu_lib, ref):
    pb.check_key_buffer_too_small(gpu_lib, ref)
