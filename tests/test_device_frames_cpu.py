"""Frames already on the GPU (gen6d_b200/frames.py, csrc/frames.cu, row f14) without a GPU: g6d_frames_gather_host (the
same code as the device gather) against cv2.cvtColor(COLOR_YUV2RGB_NV12) bit for bit and as a pitched RGB copy into the
FramePlan layout, g6d_frames_table_check's rejections, the device-frame graph names and the argument errors."""
import ctypes as C
import types

import cv2
import numpy as np
import pytest
import torch

from gen6d_b200 import _lib, ops
from gen6d_b200 import frames as fr


def _nv12(h, w, rng, pitch=None, shift=0):
    """A random NV12 image as a host decoder surface: -> (y view, uv view, the [h*3/2, w] reference image, keep-alive)
    with row pitch `pitch` and the planes starting `shift` bytes into their buffer."""
    pitch = pitch or w
    yuv = rng.randint(0, 256, (h * 3 // 2, w)).astype(np.uint8)
    buf = rng.randint(0, 256, shift + (h * 3 // 2) * pitch).astype(np.uint8)
    surf = buf[shift:].reshape(h * 3 // 2, pitch)
    surf[:, :w] = yuv
    return surf[:h, :w], surf[h:, :w], yuv, buf


def _row(fmt, p0, p1, pitch0, pitch1, h, w, off):
    return ops.DeviceFrame(p0, p1, pitch0, pitch1, h, w, fmt, off)


def _nv12_row(y, uv, off):
    return _row(_lib.G6D_FRAME_NV12, y.ctypes.data, uv.ctypes.data, y.strides[0], uv.strides[0], y.shape[0], y.shape[1], off)


def _rgb_row(img, off):
    return _row(_lib.G6D_FRAME_RGB, img.ctypes.data, None, img.strides[0], 0, img.shape[0], img.shape[1], off)


def _table(rows):
    return (ops.DeviceFrame * len(rows))(*rows)


def test_struct_layout_matches_the_header():
    assert C.sizeof(ops.DeviceFrame) == 56
    assert [getattr(ops.DeviceFrame, f).offset for f in ('plane0', 'plane1', 'pitch0', 'pitch1', 'rows', 'cols', 'format', 'offset')] == \
        [0, 8, 16, 24, 32, 36, 40, 48]


@pytest.mark.parametrize('h,w', [(2, 2), (6, 10), (480, 640), (1080, 1920)])
@pytest.mark.parametrize('pitch_pad,shift', [(0, 0), (64, 0), (3, 1), (0, 7)])
def test_nv12_gather_equals_cv2(h, w, pitch_pad, shift):
    """Random NV12, tight and wider row pitches, planes at odd byte offsets; the packed image at a nonzero offset."""
    rng = np.random.RandomState(h * 7 + w + pitch_pad + shift)
    y, uv, yuv, _keep = _nv12(h, w, rng, w + pitch_pad, shift)
    off = 256
    got = ops.frames_gather_host(_table([_nv12_row(y, uv, off)]), off + h * w * 3 + 100)
    want = cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)
    np.testing.assert_array_equal(got[off:off + h * w * 3].reshape(h, w, 3), want)
    assert not got[:off].any() and not got[off + h * w * 3:].any()        # bytes no frame covers are 0


def test_nv12_saturating_corners():
    """Every Y in {0, 15, 16, 235, 255} against every (U, V) in {0, 16, 128, 240, 255}^2: one 2x2 block per (U, V)."""
    ys, cs = [0, 15, 16, 235, 255], [0, 16, 128, 240, 255]
    pairs = [(u, v) for u in cs for v in cs]
    h, w = 2 * len(ys), 2 * len(pairs)
    y = np.repeat(np.repeat(np.asarray(ys, np.uint8)[:, None], 2, 0), w, 1)
    uv = np.zeros((h // 2, w), np.uint8)
    uv[:, 0::2] = [u for u, _ in pairs]
    uv[:, 1::2] = [v for _, v in pairs]
    yuv = np.vstack([y, uv])
    got = ops.frames_gather_host(_table([_nv12_row(yuv[:h], yuv[h:], 0)]), h * w * 3)
    want = cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)
    np.testing.assert_array_equal(got.reshape(h, w, 3), want)
    assert {0, 255} <= set(np.unique(want).tolist())                            # the corners do saturate


def test_rgb_and_nv12_mixed_into_the_plan_layout():
    """Pitched RGB views (odd sizes included) and NV12 frames at their FramePlan offsets; the padding between groups is 0
    even over a garbage-filled buffer (every byte is written)."""
    rng = np.random.RandomState(3)
    sizes = [(5, 7), (6, 10), (5, 7), (3, 1), (6, 10), (1, 9)]
    nv12 = {1, 4}
    plan = fr.FramePlan(sizes)
    rows, want, keep = [], [], []
    for i, (h, w) in enumerate(sizes):
        off = plan.table[i][0]
        if i in nv12:
            y, uv, yuv, buf = _nv12(h, w, rng, w + 5, 3)
            rows.append(_nv12_row(y, uv, off))
            want.append(cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12))
            keep.append(buf)
        else:
            big = rng.randint(0, 256, (h + 3, w + 4, 3)).astype(np.uint8)
            view = big[2:2 + h, 3:3 + w]                                         # pitch (w + 4) * 3, odd start
            rows.append(_rgb_row(view, off))
            want.append(view.copy())
            keep.append(big)
    table = _table(rows)
    ops.frames_table_check(table, plan.nbytes)
    out = np.full(plan.nbytes, 0xAB, np.uint8)
    _lib.check(_lib.lib().g6d_frames_gather_host(table, len(rows), out.ctypes.data_as(C.c_void_p), plan.nbytes),
               'g6d_frames_gather_host')
    covered = np.zeros(plan.nbytes, bool)
    for (off, h, w), img in zip(plan.table, want):
        np.testing.assert_array_equal(out[off:off + h * w * 3].reshape(h, w, 3), img)
        covered[off:off + h * w * 3] = True
    assert (~covered).any() and not out[~covered].any()


def test_table_check_rejects_malformed_tables():
    rng = np.random.RandomState(0)
    y, uv, _, _keep = _nv12(4, 6, rng)
    img = np.zeros((3, 5, 3), np.uint8)
    good = [_nv12_row(y, uv, 0), _rgb_row(img, 256)]
    ops.frames_table_check(_table(good), 512)

    def bad(rows, nbytes, match, n=None):
        t = _table(rows)
        rc = _lib.lib().g6d_frames_table_check(t, len(rows) if n is None else n, nbytes)
        assert rc == -1                                                          # G6D_EINVAL
        assert match in _lib.lib().g6d_last_error().decode(), _lib.lib().g6d_last_error()

    p = y.ctypes.data
    bad([_row(_lib.G6D_FRAME_NV12, p, uv.ctypes.data, 6, 6, 3, 6, 0)], 512, 'even')
    bad([_row(_lib.G6D_FRAME_NV12, p, uv.ctypes.data, 5, 6, 4, 5, 0)], 512, 'even')
    bad([_row(_lib.G6D_FRAME_NV12, p, uv.ctypes.data, 5, 6, 4, 6, 0)], 512, 'below its width')
    bad([_row(_lib.G6D_FRAME_NV12, p, uv.ctypes.data, 6, 4, 4, 6, 0)], 512, 'below its width')
    bad([_row(_lib.G6D_FRAME_RGB, img.ctypes.data, None, 14, 0, 3, 5, 0)], 512, 'below 3 x its width')
    bad([good[0], _rgb_row(img, 512 - 44)], 512, 'outside')
    bad([_rgb_row(img, -1)], 512, 'outside')
    bad([_row(2, p, uv.ctypes.data, 6, 6, 4, 6, 0)], 512, 'unknown format')
    bad([_row(_lib.G6D_FRAME_RGB, None, None, 15, 0, 3, 5, 0)], 512, 'null plane')
    bad([_row(_lib.G6D_FRAME_RGB, img.ctypes.data, None, 15, 0, 0, 5, 0)], 512, 'is 0 x 5')
    bad([good[0], _rgb_row(img, 40)], 512, 'overlap')
    bad(good, 512, 'need 1..1024', n=0)
    bad([_rgb_row(img, 48 * i) for i in range(_lib.G6D_FRAMES_MAX + 1)], 48 * 1025, 'need 1..1024')
    with pytest.raises(_lib.Gen6DLibraryError, match='below 3 x its width'):          # ops raises the message
        ops.frames_table_check(_table([_row(_lib.G6D_FRAME_RGB, img.ctypes.data, None, 14, 0, 3, 5, 0)]), 512)


class _Module:
    """What frames.stage / bind read of a network: its device and the upload of small inputs (kept on the host)."""

    def __init__(self, device='cpu'):
        self.device = torch.device(device)

    def _to_dev(self, a):
        return torch.from_numpy(np.ascontiguousarray(a).copy())

    def upload_frame(self, frames):
        return torch.from_numpy(np.stack(frames))

    def upload_packed(self, arrays, offsets, nbytes):
        buf = np.zeros(nbytes, np.uint8)
        for a, off in zip(arrays, offsets):
            buf[off:off + a.nbytes] = a.reshape(-1)
        return torch.from_numpy(buf)


def _pitched(h, w, pad, seed):
    big = torch.from_numpy(np.random.RandomState(seed).randint(0, 256, (h, w + pad, 3)).astype(np.uint8))
    return big[:, :w]


def _nv12_tensor(h, w, pad, seed):
    t = torch.from_numpy(np.random.RandomState(seed).randint(0, 256, (h * 3 // 2, w + pad)).astype(np.uint8))
    return fr.NV12(t[:h, :w], t[h:, :w])


def test_device_graph_names_key_on_the_size_pattern_only():
    """Device frames: the name is the pattern's, one size included, never the pointers or pitches; two calls over fresh
    allocations with other pitches have the same name and input shapes (they replay one graph); numpy names unchanged."""
    mod = _Module()
    fn = lambda *x: x
    one = [_pitched(16, 24, 0, 0), _pitched(16, 24, 8, 1), _nv12_tensor(16, 24, 4, 2)]
    again = [_nv12_tensor(16, 24, 12, 3), _pitched(16, 24, 2, 4), _pitched(16, 24, 0, 5)]
    name, body, inputs = fr.stage(mod, 'predict', fn, fr.as_frames(one, 'x', mod))
    name2, _, inputs2 = fr.stage(mod, 'predict', fn, fr.as_frames(again, 'x', mod))
    assert name == name2 == ('device', 'predict', ((16, 24),) * 3)
    assert body is not fn and len(inputs) == 1 and inputs[0].dtype == torch.uint8
    assert [tuple(t.shape) for t in inputs] == [tuple(t.shape) for t in inputs2] == [(3 * C.sizeof(ops.DeviceFrame),)]
    assert not torch.equal(inputs[0], inputs2[0])                                # the pointers and pitches are in the table
    # numpy frames of the same pattern keep their graph and name
    imgs = [np.zeros((16, 24, 3), np.uint8)] * 3
    nname, nbody, ninputs = fr.stage(mod, 'predict', fn, imgs)
    assert nname == 'predict' and nbody is fn and tuple(ninputs[0].shape) == (3, 16, 24, 3)
    # several sizes: the numpy key, and the device key with the frame order as a second input
    mixed = [_pitched(16, 24, 0, 6), _nv12_tensor(8, 10, 0, 7), _pitched(16, 24, 4, 8)]
    mname, _, minputs = fr.stage(mod, 'predict', fn, fr.as_frames(mixed, 'x', mod))
    pattern = ((16, 24), (8, 10), (16, 24))
    assert mname == ('device', ('predict', 'sizes', pattern), pattern)
    assert len(minputs) == 2 and minputs[1].tolist() == [0, 2, 1]
    numpy_name, _, _ = fr.stage(mod, 'predict', fn, [np.zeros((h, w, 3), np.uint8) for h, w in pattern])
    assert numpy_name == ('predict', 'sizes', pattern) != mname
    # a 4-D tensor is qn frames
    four = torch.zeros(2, 6, 8, 3, dtype=torch.uint8)
    assert fr.size_pattern(fr.as_frames(four, 'x', mod)) == ((6, 8), (6, 8))
    assert fr.is_device(four) and fr.is_device(one) and not fr.is_device(imgs) and not fr.is_mixed(one) and fr.is_mixed(mixed)


def test_table_rows_hold_pointers_pitches_and_offsets():
    mod = _Module()
    frames = fr.as_frames([_pitched(5, 7, 3, 0), _nv12_tensor(4, 6, 2, 1), _pitched(5, 7, 0, 2)], 'x', mod)
    plan = fr.FramePlan(fr.size_pattern(frames))
    t = fr.device_table(frames, plan)
    assert [(r.rows, r.cols, r.format, r.offset) for r in t] == \
        [(5, 7, 0, plan.table[0][0]), (4, 6, 1, plan.table[1][0]), (5, 7, 0, plan.table[2][0])]
    assert (t[0].plane0, t[0].pitch0) == (frames[0].data_ptr(), 30)
    assert (t[1].plane0, t[1].plane1, t[1].pitch0, t[1].pitch1) == (frames[1].y.data_ptr(), frames[1].uv.data_ptr(), 8, 8)
    assert t[2].pitch0 == 21


def test_malformed_device_frames_raise_value_error():
    mod = _Module()
    ok = _pitched(4, 6, 0, 0)
    cases = [
        ([ok.to(torch.int16)], 'uint8'),
        ([ok[..., :2]], r'need \[4, 6, 3\]'),
        ([ok[:, ::2]], 'strides'),                                               # non-unit column step
        ([ok.permute(1, 0, 2)], 'strides'),
        ([torch.zeros(4, 6, 3, dtype=torch.uint8).as_strided((4, 6, 3), (3, 3, 1))], 'strides'),   # pitch below the width
        ([fr.NV12(torch.zeros(3, 6, dtype=torch.uint8), torch.zeros(1, 6, dtype=torch.uint8))], 'even'),
        ([fr.NV12(torch.zeros(4, 5, dtype=torch.uint8), torch.zeros(2, 5, dtype=torch.uint8))], 'even'),
        ([fr.NV12(torch.zeros(4, 6, dtype=torch.uint8), torch.zeros(2, 4, dtype=torch.uint8))], r'UV plane is \[2, 4\]'),
        ([fr.NV12(torch.zeros(4, 12, dtype=torch.uint8)[:, ::2], torch.zeros(2, 6, dtype=torch.uint8))], 'strides'),
        ([ok, np.zeros((4, 6, 3), np.uint8)], 'all numpy arrays or all device frames'),
        ([np.zeros((4, 6, 3), np.uint8), ok], 'all numpy arrays or all device frames'),
        (torch.zeros(4, 6, 3, dtype=torch.uint8), r'\[qn, h, w, 3\]'),
    ]
    for frames, match in cases:
        with pytest.raises(ValueError, match=match):
            fr.as_frames(frames, 'x', mod)
    with pytest.raises(ValueError, match='is on cpu; device frames must be on cuda:0'):               # a CPU tensor
        fr.as_frames([ok], 'x', _Module('cuda:0'))
    with pytest.raises(ValueError, match='is on cpu; device frames must be on cuda:0'):
        fr.as_frames([_nv12_tensor(4, 6, 0, 1)], 'x', _Module('cuda:0'))


def _host_estimator():
    """An estimator with the device glue off (the host-sequenced path); its networks are never reached."""
    from gen6d_b200.estimator import Gen6DEstimator
    mod = lambda: types.SimpleNamespace(generation=0, weights_generation=0)
    return Gen6DEstimator({'device_glue': False}, modules={'detector': mod(), 'selector': mod(), 'refiner': mod()})


def test_host_sequenced_paths_reject_device_frames_before_any_launch():
    est = _host_estimator()
    frames, Ks = [_nv12_tensor(32, 32, 0, 0), _nv12_tensor(32, 32, 0, 1)], [np.eye(3)] * 2
    with pytest.raises(TypeError, match="numpy.*device_glue"):
        est.predict_batch(frames, Ks)
    with pytest.raises(TypeError, match="numpy.*device pipeline"):
        est.predict(frames[0], Ks[0])
    with pytest.raises(TypeError, match="numpy.*device pipeline"):
        est.predict_many(frames, Ks)
    trk = est.tracker(num_sequences=2, bbox_3d=np.asarray([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32))
    with pytest.raises(TypeError, match="numpy.*device_glue"):
        trk.step(frames, Ks)
