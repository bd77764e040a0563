"""g6d_det_parse_peaks on the H100: instance 0 against g6d_det_parse bit for bit, every valid row against g6d_det_parse on
a map where only that cell remains, the chosen cells against the numpy restatement, and capture into a CUDA graph."""
import numpy as np
import pytest
import torch

from det_peaks_oracle import det_peaks

pytestmark = pytest.mark.gpu
F32 = np.float32


def _maps(n, hs, ws, seed, nan=False):
    g = torch.Generator().manual_seed(seed)
    sc = torch.randn(n, hs, ws, 1, generator=g)
    if nan:
        sc[0, hs // 2, ws // 3, 0] = float('nan')                   # a NaN argmax
        sc[n - 1, ::5, ::7, 0] = float('nan')
        sc[n - 1, 0, 0, 0] = 0.0
    scl = torch.randn(n, hs, ws, 1, generator=g) * 0.5
    off = torch.rand(n, hs, ws, 2, generator=g) - 0.5
    return sc.cuda(), scl.cuda(), off.cuda()


def _bits(t):
    return t.cpu().numpy().view(np.int32) if t.dtype == torch.float32 else t.cpu().numpy()


CASES = [(3, 30, 40, False), (2, 60, 80, True), (1, 135, 240, False), (4, 1, 1, False), (2, 7, 5, True)]


@pytest.mark.parametrize('n,hs,ws,nan', CASES)
@pytest.mark.parametrize('radius', [0, 1, 3])
def test_rows_equal_det_parse(n, hs, ws, nan, radius):
    from gen6d_b200 import ops
    sc, scl, off = _maps(n, hs, ws, seed=hs * 100 + ws + radius, nan=nan)
    det, idx, valid, count = ops.det_parse_peaks(sc, scl, off, 8, radius, 0.3, 16.0)
    ref, ref_idx = ops.det_parse(sc, scl, off)
    np.testing.assert_array_equal(_bits(det[0]), _bits(ref))
    np.testing.assert_array_equal(idx[0].cpu().numpy(), ref_idx.cpu().numpy())
    valid_h, count_h, idx_h = valid.cpu().numpy(), count.cpu().numpy(), idx.cpu().numpy()
    for j in range(n):
        assert (valid_h[:count_h[j], j] == 1).all() and (valid_h[count_h[j]:, j] == 0).all()
    # every valid row decodes as det_parse decodes the same cell when it is the only finite one
    for m in range(det.shape[0]):
        for j in range(n):
            if not valid_h[m, j]:
                continue
            only = torch.full_like(sc[j:j + 1], float('-inf'))
            only.view(-1)[idx_h[m, j]] = sc[j].view(-1)[idx_h[m, j]]
            want, wi = ops.det_parse(only, scl[j:j + 1], off[j:j + 1])
            assert int(wi[0]) == idx_h[m, j]
            np.testing.assert_array_equal(_bits(det[m, j]), _bits(want[0]))


@pytest.mark.parametrize('n,hs,ws,nan', CASES)
@pytest.mark.parametrize('radius,nms_iou,box', [(1, 0.3, 16.0), (0, 0.5, 12.0), (2, 0.1, 24.0), (1, 0.3, 128.0)])
def test_chosen_cells_equal_oracle(n, hs, ws, nan, radius, nms_iou, box):
    from gen6d_b200 import ops
    sc, scl, off = _maps(n, hs, ws, seed=7 * hs + ws, nan=nan)
    det, idx, valid, count = ops.det_parse_peaks(sc, scl, off, 6, radius, nms_iou, box, min_score=-1.0)
    args = [t.cpu().numpy() for t in (sc, scl, off)]
    trace = []
    want = det_peaks(*args, max_inst=6, radius=radius, nms_iou=nms_iou, box_size=box, min_score=-1.0, trace=trace)
    # the device decodes the scale with ex2.approx, the oracle in float64: a few ulp apart.  No decision may hinge on
    # that: every IoU the greedy pass compares with nms_iou is at least 1e-4 away from it.
    trace = np.asarray(trace, F32)
    assert not (np.abs(trace - F32(nms_iou)) < 1e-4).any(), trace[np.abs(trace - F32(nms_iou)) < 1e-4]
    np.testing.assert_array_equal(idx.cpu().numpy(), want[1])
    np.testing.assert_array_equal(valid.cpu().numpy(), want[2])
    np.testing.assert_array_equal(count.cpu().numpy(), want[3])
    d = det.cpu().numpy()
    np.testing.assert_array_equal(d[..., :2], want[0][..., :2])
    np.testing.assert_array_equal(d[..., 3], want[0][..., 3])
    np.testing.assert_allclose(d[..., 2], want[0][..., 2], rtol=1e-6)


def test_capture_and_replay():
    from gen6d_b200 import ops
    sc, scl, off = _maps(5, 60, 80, seed=3)
    eager = ops.det_parse_peaks(sc, scl, off, 8, 1, 0.3, 16.0, min_score=0.5)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ops.det_parse_peaks(sc, scl, off, 8, 1, 0.3, 16.0, min_score=0.5)
    for t in out:
        t.zero_()
    g.replay()
    for a, b in zip(eager, out):
        np.testing.assert_array_equal(_bits(a), _bits(b))
    sc.mul_(-1)                                                      # new inputs in the same buffers
    g.replay()
    fresh = ops.det_parse_peaks(sc, scl, off, 8, 1, 0.3, 16.0, min_score=0.5)
    for a, b in zip(fresh, out):
        np.testing.assert_array_equal(_bits(a), _bits(b))


def test_bad_arguments_raise():
    from gen6d_b200 import _lib, ops
    sc, scl, off = _maps(1, 8, 8, seed=1)
    for kw in (dict(max_inst=0), dict(max_inst=17), dict(radius=4), dict(nms_iou=1.5)):
        a = {'max_inst': 4, 'radius': 1, 'nms_iou': 0.3, **kw}
        with pytest.raises(_lib.Gen6DLibraryError, match='g6d_det_parse_peaks'):
            ops.det_parse_peaks(sc, scl, off, a['max_inst'], a['radius'], a['nms_iou'])
