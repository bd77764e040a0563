"""CPU-only checks of the C-ABI boundary: the library builds, loads, and exports every symbol
that include/gen6d_b200.h declares; the ctypes binding covers all of them; the product path
fails loudly without a GPU (no fallback)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from gen6d_b200 import _lib


@pytest.fixture(scope='module')
def built():
    from gen6d_b200.build import build
    return build()


def test_library_exports_every_declared_symbol(built):
    lib = ctypes.CDLL(built)
    names = _lib.header_symbols()
    assert len(names) >= 30
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/gen6d_b200.h but not exported'


def test_binding_covers_header(built):
    bound = set(_lib._SIGNATURES) | {'g6d_last_error', 'g6d_version', 'g6d_launch_count'}
    assert set(_lib.header_symbols()) == bound


def test_error_reporting_without_gpu(built):
    l = _lib.lib()
    assert l.g6d_version() >= 100
    d = _lib.ConvDesc()  # all zeros -> invalid
    assert l.g6d_conv_workspace_bytes(ctypes.byref(d)) == -1
    assert b'bad dims' in l.g6d_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_compute_fails_loudly_without_cuda():
    from gen6d_b200.network import name2network
    det = name2network['detector']({})
    with pytest.raises(Exception):
        det.load_ref_imgs(np.zeros((2, 128, 128, 3), np.uint8))


def test_bench_batch_choice_deals_lanes_evenly():
    """bench.py's pick_batch: the timed region of `steps` poses is always whole batches (the batch divides `steps`, so
    exactly `steps` poses are timed), dealt to the lanes as equal numbers of full batches whenever the step count
    allows it (20 steps on 2 lanes -> 2 x 10)."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location('g6d_bench', os.path.join(root, 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    if bench.E2E_BATCH > 0:
        pytest.skip('G6D_E2E_BATCH overrides the choice')
    want = {(20, 2): 10, (16, 2): 8, (24, 2): 6, (14, 2): 7, (20, 1): 10, (4, 2): 2, (2, 2): 1, (22, 2): 2, (5, 2): 5,
            (9, 2): 9, (40, 2): 10, (30, 3): 10, (13, 2): 1, (1, 2): 1}
    for (steps, lanes), b in want.items():
        assert bench.pick_batch(steps, lanes) == b, (steps, lanes)
    for steps in range(1, 64):
        for lanes in (1, 2, 3, 4):
            assert steps % bench.pick_batch(steps, lanes) == 0, (steps, lanes)      # exactly `steps` poses timed
        if steps % lanes == 0 and (steps // lanes) % b == 0:
            assert (steps // b) % lanes == 0          # every lane runs the same number of batches
