"""Drawn frames (row f16) on the CPU: the host twin of g6d_draw_boxes against live cv2 running predict.py's
draw_bbox_3d (utils/draw_utils.py), the NV12 twin against cv2.cvtColor(COLOR_RGB2YUV_I420), and argument errors."""
import ctypes as C

import cv2
import numpy as np
import pytest

from gen6d_b200 import _lib, draw as dr, ops

EDGES = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]


def project(bbox, pose, K):
    """utils/base_utils.py project_points, restated."""
    pts = np.matmul(bbox, pose[:, :3].transpose()) + pose[:, 3:].transpose()
    pts = np.matmul(pts, K.transpose())
    dpt = pts[:, 2]
    mask0 = (np.abs(dpt) < 1e-4) & (np.abs(dpt) > 0)
    if np.sum(mask0) > 0:
        dpt[mask0] = 1e-4
    return pts[:, :2] / dpt[:, None]


def cv_draw_bbox_3d(img, pts2d, color):
    """utils/draw_utils.py draw_keypoints + draw_bbox_3d, restated on live cv2."""
    out = img.copy()
    with np.errstate(invalid='ignore'):
        p = np.round(pts2d).astype(np.int32)
    for q in p:
        cv2.circle(out, (int(q[0]), int(q[1])), 2, (255, 0, 0), -1)
    for a, b in EDGES:
        out = cv2.line(out, (int(p[a][0]), int(p[a][1])), (int(p[b][0]), int(p[b][1])), color, 2)
    return out


def host_draw(img, boxes, nv12=False):
    """g6d_draw_boxes_host on one frame: boxes [(pose [3,4], pose_f32, K, bbox [8,3], colour)] -> the drawn RGB frame, or
    the (Y, UV) planes."""
    h, w = img.shape[:2]
    img = np.ascontiguousarray(img)
    n = len(boxes)
    poses = np.ascontiguousarray([np.asarray(b[0], np.float64).reshape(12) for b in boxes] or np.zeros((1, 12)))
    Ks = np.ascontiguousarray([np.asarray(b[2], np.float64).reshape(9) for b in boxes] or np.zeros((1, 9)))
    bb = np.ascontiguousarray([np.asarray(b[3], np.float32) for b in boxes] or np.zeros((1, 8, 3), np.float32))
    src = (ops.DrawSrc * 1)(ops.DrawSrc(0, w * 3, h, w))
    tb = (ops.DrawBox * max(n, 1))(*[ops.DrawBox(0, i, i, i, int(b[1]), -1, (C.c_uint8 * 4)(*b[4], 0)) for i, b in enumerate(boxes)])
    if nv12:
        y, uv = np.zeros((h, w), np.uint8), np.zeros((h // 2, w), np.uint8)
        dst = (ops.DeviceFrame * 1)(ops.DeviceFrame(y.ctypes.data, uv.ctypes.data, w, w, h, w, _lib.G6D_FRAME_NV12, 0))
    else:
        out = np.zeros_like(img)
        dst = (ops.DeviceFrame * 1)(ops.DeviceFrame(out.ctypes.data, None, w * 3, 0, h, w, _lib.G6D_FRAME_RGB, 0))
    _lib.check(_lib.lib().g6d_draw_boxes_host(img.ctypes.data, src, 1, poses.ctypes.data, len(poses), Ks.ctypes.data, len(Ks),
                                              bb.ctypes.data, len(bb), None, 0, tb, n, dst, 1), 'g6d_draw_boxes_host')
    return (y, uv) if nv12 else out


def nv12_of(img):
    """cv2.cvtColor(COLOR_RGB2YUV_I420) with U and V interleaved -> (Y [h,w], UV [h/2,w])."""
    h, w = img.shape[:2]
    f = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420).reshape(-1)
    q = h * w // 4
    u, v = f[h * w:h * w + q].reshape(h // 2, w // 2), f[h * w + q:].reshape(h // 2, w // 2)
    return f[:h * w].reshape(h, w), np.stack([u, v], -1).reshape(h // 2, w)


def random_case(rng, h, w, f32):
    bbox = (rng.randn(8, 3) * 0.5).astype(np.float32)
    R, _ = cv2.Rodrigues(rng.randn(3))
    t = np.array([rng.randn() * 0.5, rng.randn() * 0.5, rng.uniform(-0.5, 4) if rng.rand() < 0.2 else rng.uniform(1.5, 4)])
    pose = np.concatenate([R, t[:, None]], 1)
    f = rng.uniform(10, 80)
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]], np.float32)
    return (pose.astype(np.float32) if f32 else pose), K, bbox


def corner_case(P2):
    """A box whose projection with the identity pose and K is exactly the 2-D points P2 [8,2] (float64 projection)."""
    bbox = np.concatenate([np.asarray(P2, np.float32), np.ones((8, 1), np.float32)], 1)
    return np.concatenate([np.eye(3), np.zeros((3, 1))], 1), np.eye(3, dtype=np.float32), bbox


@pytest.mark.parametrize('f32', [True, False])
def test_host_twin_equals_cv2_random_boxes(f32):
    """1500 seeded boxes per precision on frames of 1..60 rows and columns (inside, across borders, behind the camera)."""
    rng = np.random.RandomState(11 + f32)
    for it in range(1500):
        h, w = rng.randint(1, 61), rng.randint(1, 61)
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        pose, K, bbox = random_case(rng, h, w, f32)
        color = tuple(int(c) for c in rng.randint(0, 256, 3))
        want = cv_draw_bbox_3d(img, project(bbox, pose, K), color)
        np.testing.assert_array_equal(host_draw(img, [(pose, f32, K, bbox, color)]), want, err_msg=f'case {it}')


def test_host_twin_equals_cv2_edge_corners():
    """Half-integer corners (round half to even), corners far outside int32 (INT_MIN after the conversion), degenerate
    boxes, NaN corners, and 1-row / 1-column / 2x2 frames."""
    rng = np.random.RandomState(5)
    for it in range(600):
        h, w = [(1, 1), (1, 30), (30, 1), (2, 2), (25, 40)][it % 5]
        P2 = rng.randint(-30, 60, (8, 2)).astype(np.float64) + rng.choice([0, 0.5, -0.5, 1.5], (8, 2))
        if it % 7 == 0:
            P2[rng.randint(8)] = [1e12, -3e12]
        if it % 11 == 0:
            P2[rng.randint(8)] = [-3e9, 5]
        if it % 13 == 0:
            P2[:] = P2[0]
        if it % 17 == 0:
            P2[rng.randint(8), rng.randint(2)] = np.nan
        pose, K, bbox = corner_case(P2)
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        want = cv_draw_bbox_3d(img, project(bbox, pose, K), (0, 0, 255))
        np.testing.assert_array_equal(host_draw(img, [(pose, False, K, bbox, (0, 0, 255))]), want, err_msg=f'case {it}')


def test_host_twin_overlapping_boxes_in_order():
    """Several boxes on one frame are drawn one after the other: the later box's dots cover the earlier box's edges."""
    rng = np.random.RandomState(9)
    for it in range(200):
        img = rng.randint(0, 256, (40, 50, 3)).astype(np.uint8)
        boxes, want = [], img
        for j in range(rng.randint(2, 6)):
            pose, K, bbox = corner_case(rng.randint(-5, 55, (8, 2)))
            color = tuple(int(c) for c in rng.randint(0, 256, 3))
            boxes.append((pose, False, K, bbox, color))
            want = cv_draw_bbox_3d(want, project(bbox, pose, K), color)
        np.testing.assert_array_equal(host_draw(img, boxes), want, err_msg=f'case {it}')


def test_host_twin_nv12_destination():
    rng = np.random.RandomState(2)
    for h, w in [(2, 2), (4, 6), (30, 40)]:
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        pose, K, bbox = random_case(rng, h, w, True)
        y, uv = host_draw(img, [(pose, True, K, bbox, (0, 0, 255))], nv12=True)
        wy, wuv = nv12_of(cv_draw_bbox_3d(img, project(bbox, pose, K), (0, 0, 255)))
        np.testing.assert_array_equal(y, wy)
        np.testing.assert_array_equal(uv, wuv)


def test_rgb_to_nv12_host_equals_cv2():
    rng = np.random.RandomState(4)
    for h, w in [(2, 2), (2, 8), (6, 4), (30, 40)]:
        for img in [rng.randint(0, 256, (h, w, 3)).astype(np.uint8), np.full((h, w, 3), 255, np.uint8), np.zeros((h, w, 3), np.uint8),
                    (rng.rand(h, w, 3) > 0.5).astype(np.uint8) * 255]:
            y, uv = np.full((h, w + 3), 7, np.uint8), np.full((h // 2, w + 5), 7, np.uint8)
            _lib.check(_lib.lib().g6d_rgb_to_nv12_host(img.ctypes.data, w * 3, h, w, y.ctypes.data, w + 3, uv.ctypes.data, w + 5),
                       'g6d_rgb_to_nv12_host')
            wy, wuv = nv12_of(img)
            np.testing.assert_array_equal(y[:, :w], wy)
            np.testing.assert_array_equal(uv[:, :w], wuv)


def test_argument_errors():
    for bad in ['both', ('raw', 'raw'), (), ('smooth',)]:
        with pytest.raises(ValueError, match='draw must be'):
            dr.parse_kinds(bad)
    assert dr.parse_kinds(('smoothed', 'raw')) == ('raw', 'smoothed') and dr.parse_kinds(None) is None
    with pytest.raises(ValueError, match='draw_color'):
        dr.parse_color((0, 0, 256))
    src = (ops.DrawSrc * 1)(ops.DrawSrc(0, 30, 4, 10))
    buf = np.zeros((5, 12, 3), np.uint8)
    ok = ops.DeviceFrame(buf.ctypes.data, None, 36, 0, 4, 10, _lib.G6D_FRAME_RGB, 0)
    box = lambda **k: ops.DrawBox(k.get('dst', 0), k.get('pose', 0), 0, 0, 1, k.get('valid', -1), (C.c_uint8 * 4)(0, 0, 255, 0))
    one = lambda b: (ops.DrawBox * len(b))(*b)
    ops.draw_check(src, one([box()]), (ops.DeviceFrame * 1)(ok), 1, 1, 1)
    cases = [((ops.DeviceFrame * 1)(ops.DeviceFrame(buf.ctypes.data, None, 36, 0, 4, 11, 0, 0)), one([box()]), 'its source'),
             ((ops.DeviceFrame * 1)(ops.DeviceFrame(buf.ctypes.data, buf.ctypes.data, 10, 10, 4, 10, 1, 0)), one([box()]), None),
             ((ops.DeviceFrame * 1)(ops.DeviceFrame(buf.ctypes.data, None, 20, 0, 4, 10, 0, 0)), one([box()]), 'pitch'),
             ((ops.DeviceFrame * 1)(ok), one([box(pose=3)]), 'indexes outside'),
             ((ops.DeviceFrame * 1)(ok), one([box()] * 17), 'at most'),
             ((ops.DeviceFrame * 1)(ok), one([box(valid=0)]), 'indexes outside')]
    for dst, boxes, msg in cases:
        if msg is None:
            ops.draw_check(src, boxes, dst, 1, 1, 1)          # an even NV12 destination is fine
            continue
        with pytest.raises(_lib.Gen6DLibraryError, match=msg):
            ops.draw_check(src, boxes, dst, 1, 1, 1)
    odd = (ops.DrawSrc * 1)(ops.DrawSrc(0, 30, 3, 10))
    with pytest.raises(_lib.Gen6DLibraryError, match='even'):
        ops.draw_check(odd, one([box()]), (ops.DeviceFrame * 1)(ops.DeviceFrame(buf.ctypes.data, buf.ctypes.data, 10, 10, 3, 10, 1, 0)),
                       1, 1, 1)
