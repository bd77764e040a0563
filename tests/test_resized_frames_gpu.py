"""Device frames at a working resolution (gen6d_b200/frames.py Resized, DESIGN.md row f15) on the H100:
g6d_frames_gather_resized against its host twin over every byte of the packed buffer, and every entry point that takes
device frames (predict_batch, predict_instances, ObjectSet.predict / predict_instances and the four trackers) against
the numpy path on the frames cv2.resize + cv2.rotate make from the same source bytes, bit for bit; a call mixing
Resized NV12, plain RGB tensors and two working sizes; graph replay over a new source resolution."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))
ROTATE = {0: None, 90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}


def _same(got, want, where=''):
    """Every returned array equal, bit for bit (NaN where NaN), through dicts, lists and tuples."""
    if isinstance(want, dict):
        assert set(got) == set(want), (where, set(got) ^ set(want))
        for k in want:
            _same(got[k], want[k], f'{where}.{k}')
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f'{where}[{i}]')
    else:
        g, w = np.asarray(got), np.asarray(want)
        assert g.dtype == w.dtype and g.shape == w.shape, (where, g.dtype, w.dtype, g.shape, w.shape)
        np.testing.assert_array_equal(g, w, err_msg=where)


def _nv12_of(img, pad=0):
    """RGB uint8 [h,w,3] -> (an NV12 surface on the device with row pitch w + pad, the cv2 conversion of its bytes)."""
    from gen6d_b200.frames import NV12
    h, w = img.shape[:2]
    i420 = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    yuv = np.vstack([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])
    surf = torch.randint(0, 256, (h * 3 // 2, w + pad), dtype=torch.uint8, device='cuda')
    surf[:, :w] = torch.from_numpy(yuv).cuda()
    return NV12(surf[:h, :w], surf[h:, :w]), cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)


def _pitched(img, pad=7, y0=1, x0=3):
    """RGB uint8 [h,w,3] -> a view of it inside a larger, garbage-filled device buffer (pitched rows, odd start)."""
    h, w = img.shape[:2]
    big = torch.randint(0, 256, (h + y0 + 2, w + x0 + pad, 3), dtype=torch.uint8, device='cuda')
    big[y0:y0 + h, x0:x0 + w] = torch.from_numpy(img).cuda()
    return big[y0:y0 + h, x0:x0 + w]


def _reference(rgb, size, rotate):
    """predict.py's video2image on RGB bytes: cv2.resize with INTER_LINEAR, then cv2.rotate."""
    out = cv2.resize(rgb, (size[1], size[0]), interpolation=cv2.INTER_LINEAR)
    return out if rotate == 0 else cv2.rotate(out, ROTATE[rotate])


def _frames(imgs, specs, pad=0):
    """specs per frame: (kind, source (H, W) or None, rotate); kind 'n' NV12, 'p' a pitched RGB view.  A frame with a
    source size is the image upscaled to it on the host, put on the device and wrapped in Resized back to the image's
    size (max_side); without one it is the image as a plain device frame.  -> (device frames, the numpy frames the numpy
    path gets: cv2's bytes of the same sources)."""
    from gen6d_b200.frames import Resized
    dev, ref = [], []
    for j, (img, (kind, src, rot)) in enumerate(zip(imgs, specs)):
        h, w = img.shape[:2]
        big = img if src is None else cv2.resize(img, (src[1], src[0]), interpolation=cv2.INTER_CUBIC)
        f, rgb = _nv12_of(big, pad + 2 * j) if kind == 'n' else (_pitched(big, pad + j + 1), big)
        if src is None:
            dev.append(f)
            ref.append(rgb)
        else:
            r = Resized(f, max_side=max(h, w), rotate=rot)
            assert r.size == (h, w)
            dev.append(r)
            ref.append(_reference(rgb, r.size, rot))
    return dev, ref


@pytest.fixture(scope='module')
def est():
    from gen6d_b200.synthetic import build_estimator
    e, db = build_estimator()
    e.cfg['device_glue'] = True
    return e, db


@pytest.fixture(scope='module')
def frames(est):
    _, db = est
    ids = db.get_img_ids()[:4]
    return [np.ascontiguousarray(db.get_image(i)) for i in ids], [db.get_K(i) for i in ids]


@pytest.fixture(scope='module')
def objs(est):
    from gen6d_b200.synthetic import synthetic_database
    e, db = est
    o = e.object_set()
    o.add('a', db)
    o.add('b', synthetic_database(seed=8))
    return o


def _rot_K(K, rot, h, w):
    """The upper-triangular K_w of an h x w image rotated by rot: Resized.intrinsics of an identity resize times Rz.T."""
    from gen6d_b200.frames import Resized
    M = Resized(torch.zeros(h, w, 3, dtype=torch.uint8), size=(h, w), rotate=rot).intrinsics(K)
    c, s = {0: (1, 0), 90: (0, 1), 180: (-1, 0), 270: (0, -1)}[rot]
    return M @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]).T


# ------------------------------------------------------------------------------------------ 1. the kernel
def test_gather_resized_kernel_equals_host_twin():
    """Random RGB and NV12 surfaces with padded pitches and odd plane starts, every rotation, identity rows among resized
    ones (the 2x switch, 4x, non-integer ratios, one row, one column), into a garbage-filled packed buffer: every byte
    against g6d_frames_gather_resized_host; then the same launch over other allocations (the sources live in the table)."""
    from gen6d_b200 import _lib, ops
    from gen6d_b200 import frames as fr
    specs = [((1080, 1920), (540, 960), 0, 'n'), ((1080, 1920), (540, 960), 90, 'p'), ((2160, 3840), (540, 960), 180, 'n'),
             ((720, 1280), (539, 958), 270, 'n'), ((37, 53), (37, 53), 0, 'p'), ((38, 54), (35, 17), 90, 'p'),
             ((100, 130), (1, 7), 180, 'n'), ((100, 130), (9, 1), 270, 'p'), ((64, 64), (64, 64), 90, 'n'), ((6, 10), (3, 5), 0, 'n')]
    shapes = [(d[1], d[0]) if rot in (90, 270) else d for _, d, rot, _ in specs]

    def build(seed):
        g = torch.Generator(device='cuda').manual_seed(seed)
        plan = fr.FramePlan(shapes)
        rows, host, keep = [], [], []
        for i, ((h, w), (rh, rw), rot, k) in enumerate(specs):
            off = plan.table[i][0]
            if k == 'n':
                p = w + 5 + seed
                buf = torch.randint(0, 256, (3 + (h * 3 // 2) * p,), dtype=torch.uint8, device='cuda', generator=g)
                surf = buf[3:].view(h * 3 // 2, p)
                keep.append(buf)
                rows.append(ops.ResizedFrame(surf[:h].data_ptr(), surf[h:].data_ptr(), p, p, h, w, _lib.G6D_FRAME_NV12, rh, rw, rot, off))
                hs = surf.cpu().numpy()
                host.append((hs, ops.ResizedFrame(hs[:h].ctypes.data, hs[h:].ctypes.data, p, p, h, w, _lib.G6D_FRAME_NV12, rh, rw, rot, off)))
            else:
                big = torch.randint(0, 256, (h + 1, w + 3 + seed, 3), dtype=torch.uint8, device='cuda', generator=g)
                v = big[1:, 1:1 + w]
                keep.append(big)
                rows.append(ops.ResizedFrame(v.data_ptr(), None, v.stride(0), 0, h, w, _lib.G6D_FRAME_RGB, rh, rw, rot, off))
                hv = v.cpu().numpy()
                host.append((hv, ops.ResizedFrame(hv.ctypes.data, None, hv.strides[0], 0, h, w, _lib.G6D_FRAME_RGB, rh, rw, rot, off)))
        return plan, rows, host, keep

    plan, rows, host, keep = build(1)
    t = (ops.ResizedFrame * len(rows))(*rows)
    ops.frames_resized_table_check(t, plan.nbytes)
    table = torch.from_numpy(np.frombuffer(bytes(t), np.uint8).copy()).cuda()
    out = torch.full((plan.nbytes,), 0xAB, dtype=torch.uint8, device='cuda')
    ops._call('g6d_frames_gather_resized', ops._p(table, torch.uint8), len(rows), plan.H, plan.W, ops._p(out, torch.uint8),
              plan.nbytes, ops._stream())
    want = ops.frames_gather_resized_host((ops.ResizedFrame * len(host))(*[r for _, r in host]), plan.nbytes)
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    np.testing.assert_array_equal(ops.frames_gather_resized(table, len(rows), plan.H, plan.W, plan.nbytes).cpu().numpy(), want)
    off, h, w = plan.table[0]                                                     # and the host twin is cv2's
    hs = host[0][0]
    np.testing.assert_array_equal(want[off:off + h * w * 3].reshape(h, w, 3),
                                  _reference(cv2.cvtColor(np.ascontiguousarray(hs[:, :1920]), cv2.COLOR_YUV2RGB_NV12), (540, 960), 0))
    _, rows2, host2, keep2 = build(2)
    table.copy_(torch.from_numpy(np.frombuffer(bytes((ops.ResizedFrame * len(rows2))(*rows2)), np.uint8).copy()).cuda())
    out.fill_(0xCD)
    ops._call('g6d_frames_gather_resized', ops._p(table, torch.uint8), len(rows2), plan.H, plan.W, ops._p(out, torch.uint8),
              plan.nbytes, ops._stream())
    want2 = ops.frames_gather_resized_host((ops.ResizedFrame * len(host2))(*[r for _, r in host2]), plan.nbytes)
    np.testing.assert_array_equal(out.cpu().numpy(), want2)


# ------------------------------------------------------------------------------------------ 2. batch entry points
def test_predict_batch_resized(est, frames):
    from gen6d_b200 import ops
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    imgs, Ks = frames
    qn = len(imgs)
    dev, ref = _frames(imgs, [('n', (960, 1280), 0), ('p', (720, 960), 0), ('n', (720, 960), 0), ('p', (960, 1280), 0)])
    _same(e.predict_batch(dev, Ks), e.predict_batch(ref, Ks), 'Resized NV12 + RGB')
    n = len(e.stages.stages)
    assert ('device-resized', 'predict', ((480, 640),) * qn) in [k[0] for k in e.stages.stages]
    # a new source resolution, pitch and allocation with the same working sizes: the same graph, only the table uploaded
    dev, ref = _frames(imgs, [('p', (600, 800), 0), ('n', (960, 1280), 0), ('p', (480, 640), 0), ('n', (1440, 1920), 0)], pad=9)
    h0 = IO_BYTES['h2d']
    got = e.predict_batch(dev, Ks)
    assert IO_BYTES['h2d'] - h0 == qn * C.sizeof(ops.ResizedFrame) + qn * 20 * 8          # the table and the cameras only
    assert len(e.stages.stages) == n
    _same(got, e.predict_batch(ref, Ks), 'new source resolution')
    # Resized NV12, plain RGB tensors and plain NV12, two working sizes (a 90-degree rotation), a 180-degree rotation
    specs = [('n', (960, 1280), 90), ('p', None, 0), ('n', (720, 960), 180), ('n', None, 0)]
    dev, ref = _frames(imgs, specs)
    mKs = [_rot_K(K, rot, 480, 640) for K, (_, _, rot) in zip(Ks, specs)]
    _same(e.predict_batch(dev, mKs), e.predict_batch(ref, mKs), 'mixed')
    pattern = ((640, 480), (480, 640), (480, 640), (480, 640))
    assert ('device-resized', ('predict', 'sizes', pattern), pattern) in [k[0] for k in e.stages.stages]


def test_predict_instances_resized(est, frames):
    e, _ = est
    imgs, Ks = frames
    dev, ref = _frames(imgs, [('n', (960, 1280), 0), ('p', None, 0), ('p', (720, 960), 0), ('n', None, 0)])
    _same(e.predict_instances(dev, Ks, max_instances=2), e.predict_instances(ref, Ks, max_instances=2), 'instances')
    specs = [('p', (720, 960), 270), ('n', (960, 1280), 0), ('n', None, 0), ('p', (960, 1280), 90)]
    dev, ref = _frames(imgs, specs)
    mKs = [_rot_K(K, rot, 480, 640) for K, (_, _, rot) in zip(Ks, specs)]
    _same(e.predict_instances(dev, mKs, max_instances=2), e.predict_instances(ref, mKs, max_instances=2), 'instances mixed')


def test_object_set_resized(objs, frames):
    imgs, Ks = frames
    dev, ref = _frames(imgs, [('n', (960, 1280), 0), ('p', (720, 960), 0), ('n', None, 0), ('p', None, 0)])
    _same(objs.predict(dev, Ks), objs.predict(ref, Ks), 'objs')
    _same(objs.predict_instances(dev, Ks, max_instances=2), objs.predict_instances(ref, Ks, max_instances=2), 'objs instances')
    specs = [('n', (960, 1280), 90), ('p', None, 0), ('n', (720, 960), 0), ('p', (960, 1280), 180)]
    dev, ref = _frames(imgs, specs)
    mKs = [_rot_K(K, rot, 480, 640) for K, (_, _, rot) in zip(Ks, specs)]
    _same(objs.predict(dev, mKs), objs.predict(ref, mKs), 'objs mixed')
    _same(objs.predict_instances(dev, mKs, max_instances=2), objs.predict_instances(ref, mKs, max_instances=2), 'objs instances mixed')


# ------------------------------------------------------------------------------------------ 3. trackers
@pytest.fixture(scope='module')
def video(est):
    _, db = est
    K = TG['track.K']
    return [db.render(p, K) for p in TG['track.gt_poses']], K


def _track_pair(make, video, specs, reset=(), steps=3):
    """The same steps on a Resized-frame tracker and a numpy tracker: a full step, refine steps, a reset(reset) mixed step
    and one more refine step, every output equal; the sources alternate between two resolutions.  -> the device tracker."""
    frames, K = video
    dt, nt = make(), make()
    Ks = [_rot_K(K, rot, 480, 640) for _, _, rot in specs]
    for t in range(steps + 2):
        if t == steps and reset:
            dt.reset(list(reset))
            nt.reset(list(reset))
        step_specs = [(k, None if src is None else (src if t % 2 == 0 else (720, 960)), rot) for k, src, rot in specs]
        dev, ref = _frames([frames[(t + s) % len(frames)] for s in range(len(specs))], step_specs, pad=t)
        _same(dt.step(dev, Ks), nt.step(ref, Ks), f'step {t} {specs}')
    return dt


def test_tracker_resized(est, video):
    e, _ = est
    dt = _track_pair(lambda: e.tracker(num_sequences=3), video, [('n', (1080, 1440), 0), ('p', None, 0), ('n', (960, 1280), 0)],
                     reset=[1])
    assert all(k[0][0] == 'device-resized' for k in dt.stages.stages)
    _track_pair(lambda: e.tracker(num_sequences=3), video, [('n', (960, 1280), 90), ('n', (960, 1280), 0), ('p', None, 0)], reset=[0])


def test_object_tracker_resized(objs, video):
    _track_pair(lambda: objs.tracker(num_sequences=2), video, [('n', (960, 1280), 0), ('p', (1080, 1440), 0)], reset=[0])
    _track_pair(lambda: objs.tracker(num_sequences=2), video, [('n', (960, 1280), 270), ('p', None, 0)], reset=[1])


def test_instance_trackers_resized(est, objs, video):
    """Re-detection every second step: ids and every output as the numpy run's."""
    e, _ = est
    for specs in ([('n', (960, 1280), 0), ('p', None, 0)], [('n', (960, 1280), 90), ('n', None, 0), ('p', (720, 960), 0)]):
        _track_pair(lambda: e.instance_tracker(num_sequences=len(specs), max_instances=2, gate=1e6, redetect_every=2),
                    video, specs, steps=4)
        _track_pair(lambda: objs.instance_tracker(num_sequences=len(specs), max_instances=2, gate=1e6, redetect_every=2),
                    video, specs, steps=3)


def test_resized_rejected_on_host_paths(est, frames):
    from gen6d_b200.frames import Resized
    e, _ = est
    imgs, Ks = frames
    dev = [Resized(torch.from_numpy(img).cuda(), size=(240, 320)) for img in imgs]
    with pytest.raises(TypeError, match='pose_inits'):
        e.predict_batch(dev, Ks, pose_inits=[np.eye(3, 4)] * len(imgs))
    with pytest.raises(TypeError, match='device pipeline'):
        e.predict(dev[0], Ks[0])
    with pytest.raises(ValueError, match='upscales'):
        Resized(torch.from_numpy(imgs[0]).cuda(), size=(481, 640))
