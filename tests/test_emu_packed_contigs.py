"""The packed stage-1 contig checks of test_gpu_packed_contigs.py on the TEST-ONLY emulation build (tests/emu): the same
pack bodies with one emulated thread per set, packed into host memory.  Guards the cases and the record layout while
developing without a GPU; the 128-thread stores and the grid of thousands of sets only run on the device."""
import pytest

import packed_cases as pk

DEV = "cpu"


@pytest.mark.parametrize("seed,streams,shard", [(1, 1, "block"), (11, 7, "deal"), (8, 9, "gene"), (12, 96, "deal")])
def test_emu_pack_bench_shapes(emu_lib, ref, seed, streams, shard):
    st = pk.case_bench_shapes(emu_lib, ref, DEV, seed, streams, 30, 600, deal=shard == "deal", group="gene" if shard == "gene" else "")
    assert st["records"] > 20


def test_emu_pack_many_sets_sampled(emu_lib, ref):
    """4096 sets (bench.py's stream count) on few reads: a contig or two per set."""
    st = pk.case_bench_shapes(emu_lib, ref, DEV, 13, 4096, 60, 3000, deal=True, sample=64)
    assert st["sets"] == 4096 and st["records"] > 4096


def test_emu_pack_change_kmer_length(emu_lib, ref):
    assert pk.case_change_kmer_length(emu_lib, ref, DEV)["records"] > 20


@pytest.mark.parametrize("min_cov", [2, 20])
def test_emu_pack_release_shallow(emu_lib, ref, min_cov):
    st = pk.case_release_shallow(emu_lib, ref, DEV, min_cov)
    assert st["holes"] > 0 and st["records"] > 0


def test_emu_pack_empty_sets_between(emu_lib, ref):
    st = pk.case_empty_sets_between(emu_lib, ref, DEV)
    assert st["empty_sets"] == 5 and st["records"] > 20


@pytest.mark.parametrize("min_cov", [0, 3])
def test_emu_pack_single_cell(emu_lib, ref, min_cov):
    st = pk.case_single_cell(emu_lib, ref, DEV, min_cov)
    assert st["purged"] > 0 and st["barcoded"] == st["records"]
    assert st["flat"] > 0 if min_cov == 0 else st["holes"] > 0


def test_emu_pack_repseq(emu_lib, ref):
    st = pk.case_repseq(emu_lib, ref, DEV)
    assert st["records"] > 20 and st["barcoded"] > 0 and st["kmer_changed"] > 0


def test_emu_pack_assign_extended_sets(emu_lib, ref):
    assert pk.case_assign_extended(emu_lib, ref, DEV)["records"] > 20


def test_emu_pack_u16_boundary(emu_lib, ref):
    st = pk.case_u16_boundary(emu_lib, ref, DEV)
    assert st["wide"] == 2 and st["records"] == 3


def test_emu_pack_two_ranks_merge(emu_lib, ref):
    st = pk.case_two_ranks_merge(emu_lib, ref, DEV)
    assert st["removed"] > 0


def test_emu_pack_abi_edges(emu_lib):
    assert pk.check_abi_edges(emu_lib, DEV) > 0
