"""The packed stage-1 contigs on the device (t4_pack_size_kernel + t4_pack_kernel, 128 threads per set) against the
reference: what bench.py ends every step with, what the merge step all-gathers, what bench/quality.py decodes.  Packed
into a device tensor the way bench.py packs; every case also checks the record layout and that the bytes do not depend
on the buffer's old contents (packed_cases.check_packed)."""
import pytest

import packed_cases as pk

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.mark.parametrize("seed,streams,shard", [(1, 1, "block"), (2, 7, "block"), (3, 96, "block"), (11, 7, "deal"),
                                                (12, 96, "deal"), (8, 9, "gene"), (14, 96, "gene")])
def test_gpu_pack_bench_shapes(gpu_lib, ref, seed, streams, shard):
    """configs[1] in rank-block, dealt and gene-grouped streams, every set compared with the reference."""
    st = pk.case_bench_shapes(gpu_lib, ref, DEV, seed, streams, 60, 2500, deal=shard == "deal", group="gene" if shard == "gene" else "")
    assert st["records"] > 50


def test_gpu_pack_many_sets_sampled(gpu_lib, ref):
    """4096 sets (bench.py's stream count) in one pack call on few reads; a seeded sample of 64 sets compared with the
    reference, the layout checked on all."""
    st = pk.case_bench_shapes(gpu_lib, ref, DEV, 13, 4096, 60, 3000, deal=True, sample=64)
    assert st["sets"] == 4096 and st["records"] > 4096


def test_gpu_pack_change_kmer_length(gpu_lib, ref):
    assert pk.case_change_kmer_length(gpu_lib, ref, DEV)["records"] > 20


@pytest.mark.parametrize("min_cov", [2, 20])
def test_gpu_pack_release_shallow(gpu_lib, ref, min_cov):
    st = pk.case_release_shallow(gpu_lib, ref, DEV, min_cov)
    assert st["holes"] > 0 and st["records"] > 0


def test_gpu_pack_empty_sets_between(gpu_lib, ref):
    st = pk.case_empty_sets_between(gpu_lib, ref, DEV)
    assert st["empty_sets"] == 5 and st["records"] > 20


@pytest.mark.parametrize("min_cov", [0, 3])
def test_gpu_pack_single_cell(gpu_lib, ref, min_cov):
    """configs[3]: purged contigs pack the numbers the reference's Output prints from its compressed or released posWeight."""
    st = pk.case_single_cell(gpu_lib, ref, DEV, min_cov, n_barcodes=60, reads_per_barcode=400, n_streams=7)
    assert st["purged"] > 0 and st["barcoded"] == st["records"]
    assert st["flat"] > 0 if min_cov == 0 else st["holes"] > 0


def test_gpu_pack_repseq(gpu_lib, ref):
    st = pk.case_repseq(gpu_lib, ref, DEV, n_reads=12000, n_streams=4)
    assert st["records"] > 20 and st["barcoded"] > 0 and st["kmer_changed"] > 0


def test_gpu_pack_assign_extended_sets(gpu_lib, ref):
    assert pk.case_assign_extended(gpu_lib, ref, DEV, n_streams=6, nclones=60, npairs=2500)["records"] > 50


def test_gpu_pack_u16_boundary(gpu_lib, ref):
    st = pk.case_u16_boundary(gpu_lib, ref, DEV)
    assert st["wide"] == 2 and st["records"] == 3


def test_gpu_pack_two_ranks_merge(gpu_lib, ref):
    st = pk.case_two_ranks_merge(gpu_lib, ref, DEV, n_streams=8, nclones=40, npairs=1500)
    assert st["removed"] > 0


def test_gpu_pack_abi_edges(gpu_lib):
    assert pk.check_abi_edges(gpu_lib, DEV) > 0
