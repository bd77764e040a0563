"""Device frames at a working resolution (gen6d_b200/frames.py Resized, csrc/frames.cu, DESIGN.md row f15) without a
GPU: g6d_frames_gather_resized_host (the same code as the device kernel) against cv2.rotate(cv2.resize(..., INTER_LINEAR))
bit for bit for RGB and NV12 sources, every rotation and the size cases OpenCV treats differently; video2image's
max_side rule, the rejected upscales, g6d_frames_resized_table_check's rejections, Resized.intrinsics, the graph names
and the host-sequenced paths' rejections."""
import ctypes as C
import types

import cv2
import numpy as np
import pytest
import torch

from gen6d_b200 import _lib, ops
from gen6d_b200 import frames as fr

ROTATE = {0: None, 90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}


def _reference(rgb, rows, cols, rotate):
    """predict.py's video2image on an RGB frame: cv2.resize to (cols, rows) with INTER_LINEAR, then cv2.rotate."""
    out = cv2.resize(rgb, (cols, rows), interpolation=cv2.INTER_LINEAR)
    return out if rotate == 0 else cv2.rotate(out, ROTATE[rotate])


def _source(h, w, nv12, rng, pad=0, shift=0):
    """A random source frame in a pitched host buffer -> (ResizedFrame fields without size/rotation/offset, its RGB
    bytes as cv2 sees them, keep-alive)."""
    if nv12:
        pitch = w + pad
        buf = rng.randint(0, 256, shift + (h * 3 // 2) * pitch).astype(np.uint8)
        surf = buf[shift:].reshape(h * 3 // 2, pitch)
        y, uv = surf[:h, :w], surf[h:, :w]
        rgb = cv2.cvtColor(np.ascontiguousarray(surf[:, :w]), cv2.COLOR_YUV2RGB_NV12)
        return (y.ctypes.data, uv.ctypes.data, pitch, pitch, h, w, _lib.G6D_FRAME_NV12), rgb, buf
    big = rng.randint(0, 256, (h + 1, w + pad, 3)).astype(np.uint8)
    view = big[1:, :w]
    return (view.ctypes.data, None, view.strides[0], 0, h, w, _lib.G6D_FRAME_RGB), np.ascontiguousarray(view), big


def _row(src, rows, cols, rotate, off):
    return ops.ResizedFrame(*src, rows, cols, rotate, off)


def _table(rows):
    return (ops.ResizedFrame * len(rows))(*rows)


def test_struct_layout_matches_the_header():
    assert C.sizeof(ops.ResizedFrame) == 64
    names = ('plane0', 'plane1', 'pitch0', 'pitch1', 'src_rows', 'src_cols', 'format', 'rows', 'cols', 'rotate', 'offset')
    assert [getattr(ops.ResizedFrame, f).offset for f in names] == [0, 8, 16, 24, 32, 36, 40, 44, 48, 52, 56]
    assert C.sizeof(ops.DeviceFrame) == 56                                       # the plain gather's rows are unchanged


# (source rows, cols) -> (resized rows, cols): exact 2x (OpenCV's INTER_AREA switch), 4x, non-integer ratios in both
# axes, working rows of 3*cols bytes that are not multiples of 16, odd sizes, one row / one column, one axis halved only,
# identity
SIZES = [((1080, 1920), (540, 960)), ((2160, 3840), (540, 960)), ((1080, 1920), (539, 958)), ((720, 1280), (540, 960)),
         ((1080, 1920), (608, 1080)), ((102, 78), (33, 19)), ((38, 54), (35, 17)), ((100, 130), (1, 7)),
         ((100, 130), (9, 1)), ((100, 130), (1, 1)), ((64, 64), (32, 40)), ((6, 10), (3, 5)), ((48, 64), (48, 64)),
         ((64, 64), (63, 64))]


@pytest.mark.parametrize('nv12', [False, True], ids=['rgb', 'nv12'])
@pytest.mark.parametrize('src,dst', SIZES, ids=[f'{a[0]}x{a[1]}-{b[0]}x{b[1]}' for a, b in SIZES])
def test_host_twin_equals_cv2_resize_and_rotate(src, dst, nv12):
    rng = np.random.RandomState(src[0] * 31 + dst[1] + nv12)
    h, w = src
    source, rgb, _keep = _source(h, w, nv12, rng, pad=5 if nv12 else 3, shift=3)
    n = dst[0] * dst[1] * 3
    rows, wants = [], []
    for k, rot in enumerate(ROTATE):
        rows.append(_row(source, dst[0], dst[1], rot, 256 * k + k * -(-n // 256) * 256))
        wants.append(_reference(rgb, dst[0], dst[1], rot))
    nbytes = rows[-1].offset + n + 77
    out = np.full(nbytes, 0xAB, np.uint8)                                        # every byte is written, gaps included
    _lib.check(_lib.lib().g6d_frames_gather_resized_host(_table(rows), len(rows), out.ctypes.data_as(C.c_void_p), nbytes),
               'g6d_frames_gather_resized_host')
    covered = np.zeros(nbytes, bool)
    for r, want in zip(rows, wants):
        np.testing.assert_array_equal(out[r.offset:r.offset + n].reshape(want.shape), want, err_msg=f'rotate {r.rotate}')
        covered[r.offset:r.offset + n] = True
    assert not out[~covered].any()


def test_identity_is_a_copy_and_rgb_nv12_mix_in_one_table():
    """Plain frames as identity rows next to resized ones, at their FramePlan offsets of working sizes."""
    rng = np.random.RandomState(5)
    specs = [((40, 60), (40, 60), 0, False), ((40, 60), (20, 30), 90, True), ((33, 47), (33, 47), 0, False),
             ((40, 60), (25, 37), 270, True), ((33, 47), (11, 46), 180, False)]
    rows_rgb, keep = [], []
    for (h, w), (rh, rw), rot, nv in specs:
        s, rgb, k = _source(h, w, nv, rng, pad=2, shift=1)
        rows_rgb.append((s, rgb, rh, rw, rot))
        keep.append(k)
    shapes = [(rw, rh) if rot in (90, 270) else (rh, rw) for _, _, rh, rw, rot in rows_rgb]
    plan = fr.FramePlan(shapes)
    table = _table([_row(s, rh, rw, rot, plan.table[i][0]) for i, (s, _, rh, rw, rot) in enumerate(rows_rgb)])
    ops.frames_resized_table_check(table, plan.nbytes)
    out = ops.frames_gather_resized_host(table, plan.nbytes)
    covered = np.zeros(plan.nbytes, bool)
    for (off, h, w), (_, rgb, rh, rw, rot) in zip(plan.table, rows_rgb):
        np.testing.assert_array_equal(out[off:off + h * w * 3].reshape(h, w, 3), _reference(rgb, rh, rw, rot))
        covered[off:off + h * w * 3] = True
    np.testing.assert_array_equal(out[plan.table[0][0]:][:40 * 60 * 3].reshape(40, 60, 3), rows_rgb[0][1])
    assert (~covered).any() and not out[~covered].any()


def test_table_check_rejects_malformed_rows():
    rng = np.random.RandomState(0)
    nv, _, _k1 = _source(8, 12, True, rng)
    rgb, _, _k2 = _source(5, 7, False, rng)
    good = [_row(nv, 4, 6, 90, 0), _row(rgb, 5, 7, 0, 256)]
    ops.frames_resized_table_check(_table(good), 512)

    def bad(rows, nbytes, match, n=None):
        rc = _lib.lib().g6d_frames_resized_table_check(_table(rows), len(rows) if n is None else n, nbytes)
        assert rc == -1                                                          # G6D_EINVAL
        assert match in _lib.lib().g6d_last_error().decode(), _lib.lib().g6d_last_error()

    y, uv, p = nv[0], nv[1], rgb[0]
    NV, RGB = _lib.G6D_FRAME_NV12, _lib.G6D_FRAME_RGB
    bad([ops.ResizedFrame(y, uv, 12, 12, 8, 12, 2, 4, 6, 0, 0)], 512, 'unknown format')
    for rot in (45, -90, 360):
        bad([ops.ResizedFrame(y, uv, 12, 12, 8, 12, NV, 4, 6, rot, 0)], 512, 'rotation')
    bad([ops.ResizedFrame(y, uv, 12, 12, 7, 12, NV, 4, 6, 0, 0)], 512, 'even')
    bad([ops.ResizedFrame(y, uv, 12, 12, 8, 11, NV, 4, 6, 0, 0)], 512, 'even')
    bad([ops.ResizedFrame(None, uv, 12, 12, 8, 12, NV, 4, 6, 0, 0)], 512, 'null plane')
    bad([ops.ResizedFrame(y, None, 12, 12, 8, 12, NV, 4, 6, 0, 0)], 512, 'null plane')
    bad([ops.ResizedFrame(y, uv, 11, 12, 8, 12, NV, 4, 6, 0, 0)], 512, 'below its width')
    bad([ops.ResizedFrame(y, uv, 12, 10, 8, 12, NV, 4, 6, 0, 0)], 512, 'below its width')
    bad([ops.ResizedFrame(p, None, 20, 0, 5, 7, RGB, 5, 7, 0, 0)], 512, 'below 3 x its width')
    bad([ops.ResizedFrame(p, None, 21, 0, 5, 7, RGB, 6, 7, 0, 0)], 512, 'no upscaling')     # larger than the source
    bad([ops.ResizedFrame(p, None, 21, 0, 5, 7, RGB, 5, 8, 90, 0)], 512, 'no upscaling')
    bad([ops.ResizedFrame(p, None, 21, 0, 5, 7, RGB, 0, 7, 0, 0)], 512, 'at least 1 x 1')
    bad([ops.ResizedFrame(p, None, 21, 0, 5, 7, RGB, 5, 0, 0, 0)], 512, 'at least 1 x 1')
    bad([ops.ResizedFrame(p, None, 21, 0, 0, 7, RGB, 0, 7, 0, 0)], 512, 'source')
    bad([good[0], _row(rgb, 5, 7, 0, 512 - 100)], 512, 'outside')
    bad([_row(rgb, 5, 7, 0, -1)], 512, 'outside')
    bad([good[0], _row(rgb, 5, 7, 0, 40)], 512, 'overlap')
    bad(good, 512, 'need 1..1024', n=0)
    bad([_row(rgb, 1, 1, 0, 3 * i) for i in range(_lib.G6D_FRAMES_MAX + 1)], 3 * 1025, 'need 1..1024')
    with pytest.raises(_lib.Gen6DLibraryError, match='no upscaling'):
        ops.frames_resized_table_check(_table([ops.ResizedFrame(p, None, 21, 0, 5, 7, RGB, 6, 7, 0, 0)]), 512)
    # the host twin checks first
    out = np.zeros(512, np.uint8)
    assert _lib.lib().g6d_frames_gather_resized_host(_table([_row(rgb, 6, 7, 0, 0)]), 1, out.ctypes.data_as(C.c_void_p), 512) == -1


# ------------------------------------------------------------------------------------------ Resized
def _t(h, w):
    return torch.zeros(h, w, 3, dtype=torch.uint8)


def _nv(h, w, pad=0, seed=0):
    t = torch.from_numpy(np.random.RandomState(seed).randint(0, 256, (h * 3 // 2, w + pad)).astype(np.uint8))
    return fr.NV12(t[:h, :w], t[h:, :w])


@pytest.mark.parametrize('h,w,side', [(1080, 1920, 960), (2160, 3840, 960), (720, 1280, 960), (1920, 1080, 960),
                                      (537, 1074, 960), (1081, 1081, 960), (480, 640, 333), (1000, 999, 10)])
def test_max_side_is_video2image_rule(h, w, side):
    """ratio = max_side / max(h, w), (int(ratio*h), int(ratio*w)) in Python floats; 537 x 1074 and 1081 x 1081 at 960
    land just below integers (479.99999999999994 and 959.99999999999994, 959.9999999999999) and truncate as video2image
    truncates: not even the long side reaches max_side."""
    ratio = side / max(h, w)
    want = (int(ratio * h), int(ratio * w))
    for f in (_t(h, w), _nv(h - h % 2, w - w % 2) if h % 2 == 0 and w % 2 == 0 else _t(h, w)):
        r = fr.Resized(f, max_side=side)
        assert r.size == want and r.shape == want + (3,)
        assert fr.Resized(f, max_side=side, rotate=90).shape == (want[1], want[0], 3)
    if (h, w) == (537, 1074):
        assert want == (479, 959)
    if (h, w) == (1081, 1081):
        assert want == (959, 959)


def test_resized_arguments():
    assert fr.Resized(_t(40, 60), size=(20, 30), rotate=270).shape == (30, 20, 3)
    assert fr.Resized(_t(40, 60), size=(40, 60)).shape == (40, 60, 3)                  # identity
    for kw, match in [(dict(size=(41, 60)), 'upscales'), (dict(size=(40, 61)), 'upscales'), (dict(max_side=61), 'upscales'),
                      (dict(size=(0, 5)), r'>= \(1, 1\)'), (dict(max_side=1, size=(2, 2)), 'exactly one'), ({}, 'exactly one'),
                      (dict(size=(20, 30), rotate=45), 'rotate'), (dict(max_side=0), 'max_side'), (dict(max_side=0.5), r'>= \(1, 1\)')]:
        with pytest.raises(ValueError, match=match):
            fr.Resized(_t(40, 60), **kw)
    with pytest.raises(ValueError, match='upscales'):
        fr.Resized(_nv(40, 60), size=(42, 60))
    with pytest.raises(ValueError, match='ndarray'):
        fr.Resized(np.zeros((40, 60, 3), np.uint8), size=(20, 30))
    with pytest.raises(ValueError, match='need'):
        fr.Resized(torch.zeros(40, 60, dtype=torch.uint8), size=(20, 30))
    with pytest.raises(ValueError, match='Resized'):
        fr.Resized(fr.Resized(_t(40, 60), size=(20, 30)), size=(10, 15))


@pytest.mark.parametrize('rotate', [0, 90, 180, 270])
def test_intrinsics_follow_the_resize_and_rotation(rotate):
    """Project synthetic points with K in the source frame, map the pixel through the resize's pixel-centre convention
    and the rotation by hand; the mapped K projects the same points there."""
    h, w = 1080, 1920
    r = fr.Resized(_t(h, w), size=(539, 958), rotate=rotate)
    K = np.array([[1500.0, 0, 955.3], [0, 1490.0, 541.7], [0, 0, 1]])
    X = np.random.RandomState(0).uniform([-1, -1, 2], [1, 1, 6], (50, 3))
    x = X @ K.T
    x = x[:, :2] / x[:, 2:]
    rh, rw = r.size
    px = (x[:, 0] + 0.5) * rw / w - 0.5
    py = (x[:, 1] + 0.5) * rh / h - 0.5
    want = {0: (px, py), 90: (rh - 1 - py, px), 180: (rw - 1 - px, rh - 1 - py), 270: (py, rw - 1 - px)}[rotate]
    Kw = r.intrinsics(K)
    y = X @ Kw.T
    np.testing.assert_allclose(y[:, :2] / y[:, 2:], np.stack(want, 1), rtol=0, atol=1e-9)
    # M = K_w @ Rz: Rz the linear part of the pixel rotation, K_w upper triangular with positive focal lengths
    c, s = {0: (1, 0), 90: (0, 1), 180: (-1, 0), 270: (0, -1)}[rotate]
    Kw_ = Kw @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]).T
    assert np.allclose(np.tril(Kw_, -1), 0, atol=1e-12) and Kw_[0, 0] > 0 and Kw_[1, 1] > 0
    # and a pixel the rotation moves: the working image of an indicator frame puts it where the mapping says
    img = np.zeros((h, w, 3), np.uint8)
    img[100:110, 200:210] = 255
    out = _reference(img, rh, rw, rotate)
    cy, cx = np.argwhere(out[..., 0] > 128).mean(0)
    pt = Kw @ np.linalg.solve(K, np.array([204.5, 104.5, 1.0]))
    assert abs(pt[0] / pt[2] - cx) < 0.6 and abs(pt[1] / pt[2] - cy) < 0.6


# ------------------------------------------------------------------------------------------ plumbing
class _Module:
    """What frames.stage / bind read of a network: its device and the upload of small inputs (kept on the host)."""

    def __init__(self, device='cpu'):
        self.device = torch.device(device)

    def _to_dev(self, a):
        return torch.from_numpy(np.ascontiguousarray(a).copy())

    def upload_frame(self, frames):
        return torch.from_numpy(np.stack(frames))


def _pitched(h, w, pad, seed):
    big = torch.from_numpy(np.random.RandomState(seed).randint(0, 256, (h, w + pad, 3)).astype(np.uint8))
    return big[:, :w]


def test_graph_names_key_on_the_working_pattern():
    mod = _Module()
    fn = lambda *x: x
    one = [fr.Resized(_nv(1080, 1920, 64, 0), max_side=960), _pitched(540, 960, 3, 1), fr.Resized(_pitched(720, 1280, 0, 2), size=(540, 960))]
    again = [fr.Resized(_nv(2160, 3840, 0, 3), max_side=960), _pitched(540, 960, 0, 4), fr.Resized(_nv(1080, 1920, 8, 5), max_side=960)]
    name, body, inputs = fr.stage(mod, 'predict', fn, fr.as_frames(one, 'x', mod))
    name2, _, inputs2 = fr.stage(mod, 'predict', fn, fr.as_frames(again, 'x', mod))
    assert name == name2 == ('device-resized', 'predict', ((540, 960),) * 3)
    assert body is not fn and [tuple(t.shape) for t in inputs] == [tuple(t.shape) for t in inputs2] == [(3 * 64,)]
    t = np.frombuffer(inputs[0].numpy().tobytes(), np.uint8)
    rows = (ops.ResizedFrame * 3).from_buffer_copy(t)
    assert [(r.src_rows, r.src_cols, r.rows, r.cols, r.rotate, r.format) for r in rows] == \
        [(1080, 1920, 540, 960, 0, 1), (540, 960, 540, 960, 0, 0), (720, 1280, 540, 960, 0, 0)]
    assert (rows[0].pitch0, rows[0].pitch1, rows[1].pitch0) == (1984, 1984, 963 * 3)
    # two working sizes and a rotation: the numpy path's pattern name inside the device-resized key, the order input
    mixed = [fr.Resized(_nv(1080, 1920, 0, 6), max_side=960, rotate=90), _pitched(540, 960, 0, 7), fr.Resized(_nv(1080, 1920, 0, 8), max_side=960)]
    pattern = ((960, 540), (540, 960), (540, 960))
    mname, _, minputs = fr.stage(mod, 'predict', fn, fr.as_frames(mixed, 'x', mod))
    assert mname == ('device-resized', ('predict', 'sizes', pattern), pattern)
    assert len(minputs) == 2 and minputs[1].tolist() == [0, 1, 2]
    # without a Resized frame: today's names
    plain = [_pitched(540, 960, 0, 9), _nv(540, 960, 0, 10)]
    assert fr.stage(mod, 'predict', fn, fr.as_frames(plain, 'x', mod))[0] == ('device', 'predict', ((540, 960),) * 2)
    assert fr.stage(mod, 'predict', fn, [np.zeros((540, 960, 3), np.uint8)] * 2)[0] == 'predict'
    assert fr.is_device(one) and fr.has_resized(one) and not fr.has_resized(plain)


def test_resized_sources_are_checked_like_device_frames():
    mod = _Module()
    with pytest.raises(ValueError, match='strides'):
        fr.as_frames([fr.Resized(_t(8, 12)[:, ::2], size=(4, 6))], 'x', mod)
    with pytest.raises(ValueError, match='UV plane'):
        fr.as_frames([fr.Resized(fr.NV12(torch.zeros(8, 12, dtype=torch.uint8), torch.zeros(4, 10, dtype=torch.uint8)), size=(4, 6))],
                     'x', mod)
    with pytest.raises(ValueError, match='is on cpu; device frames must be on cuda:0'):
        fr.as_frames([fr.Resized(_t(8, 12), size=(4, 6))], 'x', _Module('cuda:0'))
    with pytest.raises(ValueError, match='all numpy arrays or all device frames'):
        fr.as_frames([fr.Resized(_t(8, 12), size=(4, 6)), np.zeros((4, 6, 3), np.uint8)], 'x', mod)


def _host_estimator():
    """An estimator with the device glue off (the host-sequenced path); its networks are never reached."""
    from gen6d_b200.estimator import Gen6DEstimator
    mod = lambda: types.SimpleNamespace(generation=0, weights_generation=0)
    return Gen6DEstimator({'device_glue': False}, modules={'detector': mod(), 'selector': mod(), 'refiner': mod()})


def test_host_sequenced_paths_reject_resized_before_any_launch():
    est = _host_estimator()
    frames, Ks = [fr.Resized(_nv(64, 64, 0, s), size=(32, 32)) for s in (0, 1)], [np.eye(3)] * 2
    with pytest.raises(TypeError, match="numpy.*device_glue"):
        est.predict_batch(frames, Ks)
    with pytest.raises(TypeError, match="numpy.*device pipeline"):
        est.predict(frames[0], Ks[0])
    with pytest.raises(TypeError, match="numpy.*device pipeline"):
        est.predict_many(frames, Ks)
    with pytest.raises(TypeError, match="numpy.*device_glue"):
        est.predict_batch(frames, Ks, pose_inits=[np.eye(3, 4)] * 2)
    trk = est.tracker(num_sequences=2, bbox_3d=np.asarray([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32))
    with pytest.raises(TypeError, match="numpy.*device_glue"):
        trk.step(frames, Ks)
