"""Emulation twins of test_gpu_long_reads.py (tests/emu, no GPU).  The emulation replaces the device-only routines these
cases aim at (the warp DPs of overlap scoring and ExtendOverlap, the overhang masks, the deferred-side ballot, the hit
sort) with host stand-ins, so here the cases check the engine's logic and that every case still reaches its edge in the
reference's own data."""
import pytest

import long_read_cases as lr


@pytest.mark.parametrize("k", [9, 7])
def test_emu_gap_scoring(emu_lib, ref, k):
    assert lr.check_gap_scoring(emu_lib, ref, k) > 0


@pytest.mark.parametrize("n_overlaps", [8, 20, 55])
def test_emu_extend_sides(emu_lib, ref, n_overlaps, record_property):
    fallbacks = lr.check_extend_sides(emu_lib, ref, n_overlaps)
    record_property("counter_21_total", sum(c for _, _, c in fallbacks))


@pytest.mark.parametrize("n_overlaps", [8, 20])
def test_emu_extend_sides_batch(emu_lib, ref, n_overlaps):
    lr.check_extend_sides_batch(emu_lib, ref, n_overlaps)


def test_emu_contig_growth(emu_lib, ref):
    lr.check_contig_growth(emu_lib, ref)


@pytest.mark.parametrize("kind", lr.KEY_SETS)
def test_emu_hit_sort(emu_lib, ref, kind):
    lr.check_hit_sort(emu_lib, ref, kind)


@pytest.mark.parametrize("n_streams", [1, 3])
def test_emu_mixed_batch(emu_lib, ref, n_streams):
    lr.check_mixed_batch(emu_lib, ref, n_streams)


@pytest.mark.parametrize("kmer", [17, 19])
def test_emu_mixed_assign(emu_lib, ref, kmer):
    lr.check_mixed_assign(emu_lib, ref, kmer)
