"""The per-cell statistics and the barcode sort of --barcode runs on the GPU (t4_kcount_bc_kernel, t4_readsort_bc_kernel),
against the compiled reference (its KmerCount on each cell's reads, its std::sort within each (barcode, barcodeMinCnt)
group; see barcode_cases.py), and the batch drop-in with those passes on the device.  Emulation twins: test_emu_barcode_stats.py."""
import numpy as np
import pytest

import barcode_cases as bcc
from test_dropin_cli import dropin_binary
from test_emu_barcode_stats import run_barcode_dropin

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", sorted(bcc.STATS_CASES))
def test_gpu_barcode_kmer_stats(gpu_lib, ref, case):
    assert bcc.check_stats_case(gpu_lib, ref, case) > 0


def test_gpu_barcode_kmer_stats_device_form(gpu_lib, ref):
    import torch

    def dev(a):
        t = torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()
        return t, t.data_ptr(), lambda: t.cpu().numpy()
    bcc.check_device_form(gpu_lib, ref, dev)


def test_gpu_sort_reads_barcode(gpu_lib, ref):
    assert bcc.check_sort_barcode(gpu_lib, ref) > 10000


def test_gpu_sort_reads_barcode_large(gpu_lib):
    assert bcc.check_sort_barcode_large(gpu_lib) == (1 << 20) + 3


def test_gpu_barcode_errors(gpu_lib, ref):
    bcc.check_errors(gpu_lib, ref)


@pytest.mark.parametrize("extra", [(), ("--contigMinCov", "4")])
def test_batch_gpu_barcode_stats_on_device(tmp_path, extra):
    run_barcode_dropin(dropin_binary("trust4_gpu_batch"), str(tmp_path), extra)
