"""The drop-in stage-0 binary on an H100: `fastq-extractor-gpu` (integration/_build/, or oracle/_ref/ where the reference
sources are absent) against the stock `fastq-extractor` (oracle/_ref/).  The cases of test_extractor_cli.py, whose
candidate tests run on the device here, and a read set of a million pairs at -t 1 and at all host cores.  Every file the
runs write is compared byte for byte; the route line tells how many reads the device scanned."""
import os

import pytest

import extractor_cases as xc


@pytest.fixture(scope="module")
def gpu_extractor():
    return xc.extractor_binary("fastq-extractor-gpu")


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 4])
def test_gpu_shipped_example(gpu_extractor, tmp_path, threads):
    xc.case_shipped_example(gpu_extractor, str(tmp_path), threads)


@pytest.mark.gpu
@pytest.mark.parametrize("L,paired,gz,threads", xc.SYNTH, ids=xc.SYNTH_IDS)
def test_gpu_synthetic_with_edges(gpu_extractor, tmp_path, L, paired, gz, threads):
    xc.case_synthetic_with_edges(gpu_extractor, str(tmp_path), L, paired, gz, threads)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 2])
def test_gpu_single_end(gpu_extractor, tmp_path, threads):
    xc.case_single_end(gpu_extractor, str(tmp_path), threads)


@pytest.mark.gpu
@pytest.mark.parametrize("threads,extra", [(1, ()), (4, ()), (2, ("--skipBarcodeErrorRead",))])
def test_gpu_barcode_umi_whitelist(gpu_extractor, tmp_path, threads, extra):
    xc.case_barcode_umi_whitelist(gpu_extractor, str(tmp_path), threads, extra)


@pytest.mark.gpu
@pytest.mark.parametrize("threads", [1, 3])
def test_gpu_read_format_range(gpu_extractor, tmp_path, threads):
    xc.case_read_format_range(gpu_extractor, str(tmp_path), threads)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1 << 18, (1 << 18) + 1, 0], ids=["one-batch", "one-batch-plus-1", "empty"])
def test_gpu_batch_size_edges(gpu_extractor, tmp_path, n):
    xc.case_batch_size_edges(gpu_extractor, str(tmp_path), n)


@pytest.mark.gpu
def test_gpu_million_pairs(gpu_extractor, tmp_path):
    """1 M pairs of 150 bp (four batches of 2^18 reads per mate) at -t 1 and at all host cores."""
    for threads in (1, os.cpu_count() or 1):
        xc.case_large(gpu_extractor, str(tmp_path), 1 << 20, threads)
