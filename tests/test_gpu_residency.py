"""The stream kernel's residency: its registers are bounded for T4_STREAM_BLOCKS CTAs per SM (t4_api.cu), and at the
launch t4_streams_run uses (128 threads, the hit tile in dynamic shared memory) that many CTAs really are resident.
A register more, or a T4Smem grown past the budget, costs a stream slot on every SM; this fails instead."""
import ctypes

import pytest

pytestmark = pytest.mark.gpu

STREAM_BLOCKS = 4   # T4_STREAM_BLOCKS


def test_gpu_stream_kernel_resident(gpu_lib):
    target, resident = ctypes.c_int(), ctypes.c_int()
    gpu_lib.check(gpu_lib.stream_residency(ctypes.byref(target), ctypes.byref(resident)))
    assert target.value == STREAM_BLOCKS
    assert resident.value >= STREAM_BLOCKS, (resident.value, STREAM_BLOCKS)
