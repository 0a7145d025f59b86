"""Emulation twins of test_gpu_probe_edges.py (tests/emu, no GPU).  The emulation runs the stream engine's own
GetHitsFromRead, so the barcode, list-size and counter cases check the engine's lookup; t4_streams_get_hits is answered
through that same engine code, so the probe cases here check only the API around it (records, barcodes, strand modes,
flags, counters, the overflow report), not the probe kernel."""
import pytest

import probe_cases as pb

PAIRS = dict(pb.COLLIDING, **pb.CONTROL)
CASES = [(k, p, c) for k in (9, 15) for p in PAIRS for c in pb.COUNTS]


@pytest.mark.parametrize("k,pair,counts", CASES)
def test_emu_colliding_barcodes(emu_lib, ref, k, pair, counts):
    pb.check_colliding_barcodes(emu_lib, ref, k, PAIRS[pair], pb.COUNTS[counts], seed=k)


def test_emu_colliding_barcodes_big_list(emu_lib, ref):
    pb.check_colliding_barcodes(emu_lib, ref, 9, PAIRS["-1~1000002"], (5000, 5001), seed=3, n_add=6)


def test_emu_colliding_barcodes_batch(emu_lib, ref):
    pb.check_colliding_batch(emu_lib, ref)


@pytest.mark.parametrize("k,pair,counts", [(9, "5~1000008", "sum>=100"), (15, "-1~1000002", "one>=100"), (9, "-1~1000002", "big")])
def test_emu_probe_barcoded_sets(emu_lib, ref, k, pair, counts):
    """API plumbing only: records carrying barcodes reach the lookup with their barcode and strand, flags come back."""
    pb.check_colliding_probe(emu_lib, ref, k, PAIRS[pair], (5000, 5001) if counts == "big" else pb.COUNTS[counts], seed=k)


def test_emu_probe_list_sizes(emu_lib, ref):
    pb.check_list_sizes(emu_lib, ref)


def test_emu_probe_read_length_edges(emu_lib, ref):
    pb.check_read_length_edges(emu_lib, ref)


def test_emu_probe_counters(emu_lib, ref):
    assert pb.check_hits_counters(emu_lib, ref) > 1000


def test_emu_probe_key_buffer_too_small(emu_lib, ref):
    pb.check_key_buffer_too_small(emu_lib, ref)
