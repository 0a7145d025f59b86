"""The per-cell statistics and the barcode sort of --barcode runs, through the CPU emulation of the device code (g++
-DT4_EMU, the same kernel bodies run with one thread), against the compiled reference; and the batch drop-in with those
passes on the emulated device.  GPU twins: test_gpu_barcode_stats.py."""
import os
import subprocess

import numpy as np
import pytest

import barcode_cases as bcc
from test_dropin_cli import STOCK, SUFFIXES, dropin_binary, write_barcode_inputs


@pytest.mark.parametrize("case", sorted(bcc.STATS_CASES))
def test_emu_barcode_kmer_stats(emu_lib, ref, case):
    assert bcc.check_stats_case(emu_lib, ref, case) > 0


def test_emu_barcode_kmer_stats_device_form(emu_lib, ref):
    def host(a):
        b = np.ascontiguousarray(a).copy()
        return b, b.ctypes.data, lambda: b
    bcc.check_device_form(emu_lib, ref, host)


def test_emu_sort_reads_barcode(emu_lib, ref):
    assert bcc.check_sort_barcode(emu_lib, ref) > 10000


def test_emu_barcode_errors(emu_lib, ref):
    bcc.check_errors(emu_lib, ref)


@pytest.fixture(scope="module")
def emu_batch_binary(emu_lib):
    return dropin_binary("trust4_emu_batch")


def run_barcode_dropin(binary, tmp, extra):
    """The stock binary and the batch drop-in with every opt-in pre-processing pass on the device; the three output files
    must be byte-identical and the per-cell pass must have run."""
    args = write_barcode_inputs(tmp)
    subprocess.run([STOCK, "-t", "1", "-o", os.path.join(tmp, "stock")] + list(extra) + args, check=True, stdout=subprocess.DEVNULL,
                   stderr=subprocess.DEVNULL, timeout=900)
    env = dict(os.environ, T4_STREAMS="1", T4_BCSTATS="1", T4_SORT="1", T4_ANNOTATE="1")
    r = subprocess.run([binary, "-t", "1", "-o", os.path.join(tmp, "dev")] + list(extra) + args, check=True, stdout=subprocess.DEVNULL,
                       stderr=subprocess.PIPE, timeout=900, env=env, text=True)
    assert "per-cell 21-mer statistics and barcode sort on the device" in r.stderr, r.stderr[-600:]
    for suf in SUFFIXES:
        a = open(os.path.join(tmp, "stock" + suf), "rb").read()
        assert len(a) > 0 and a == open(os.path.join(tmp, "dev" + suf), "rb").read(), suf


@pytest.mark.parametrize("extra", [(), ("--contigMinCov", "4")])
def test_batch_emu_barcode_stats_on_device(emu_batch_binary, tmp_path, extra):
    run_barcode_dropin(emu_batch_binary, str(tmp_path), extra)
