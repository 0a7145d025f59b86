"""The drop-in stage-0 binary through the CPU emulation of the engine: `fastq-extractor-emu` is the reference's
FastqExtractor.cpp as integration/make_extractor_main.py patches it, with integration/t4_extractor_adapter.hpp
force-included and linked against tests/emu/libt4emu.so.  Every case runs the stock `fastq-extractor`
(oracle/_ref/) and the drop-in on the same inputs and flags and compares every file the run writes byte for byte, and
checks the drop-in's route line: how many reads the (emulated) device scanned and how many went to the host.
The same cases on an H100, plus a large read set: tests/test_gpu_extractor.py."""
import pytest

import extractor_cases as xc


@pytest.fixture(scope="module")
def emu_extractor(emu_lib):
    return xc.extractor_binary("fastq-extractor-emu")


@pytest.mark.parametrize("threads", [1, 4])
def test_shipped_example(emu_extractor, tmp_path, threads):
    xc.case_shipped_example(emu_extractor, str(tmp_path), threads)


@pytest.mark.parametrize("L,paired,gz,threads", xc.SYNTH, ids=xc.SYNTH_IDS)
def test_synthetic_with_edges(emu_extractor, tmp_path, L, paired, gz, threads):
    xc.case_synthetic_with_edges(emu_extractor, str(tmp_path), L, paired, gz, threads)


@pytest.mark.parametrize("threads", [1, 2])
def test_single_end(emu_extractor, tmp_path, threads):
    xc.case_single_end(emu_extractor, str(tmp_path), threads)


@pytest.mark.parametrize("threads,extra", [(1, ()), (4, ()), (2, ("--skipBarcodeErrorRead",))])
def test_barcode_umi_whitelist(emu_extractor, tmp_path, threads, extra):
    xc.case_barcode_umi_whitelist(emu_extractor, str(tmp_path), threads, extra)


@pytest.mark.parametrize("threads", [1, 3])
def test_read_format_range(emu_extractor, tmp_path, threads):
    xc.case_read_format_range(emu_extractor, str(tmp_path), threads)


@pytest.mark.parametrize("n", [1 << 18, (1 << 18) + 1, 0], ids=["one-batch", "one-batch-plus-1", "empty"])
def test_batch_size_edges(emu_extractor, tmp_path, n):
    xc.case_batch_size_edges(emu_extractor, str(tmp_path), n)
