"""Frames already on the GPU (gen6d_b200/frames.py, DESIGN.md row f14) on the H100: g6d_frames_gather against its host
twin, and every entry point that takes device frames (predict_batch, predict_instances, ObjectSet.predict /
predict_instances and the four trackers) against the numpy path on the same RGB bytes, bit for bit, for one [qn,h,w,3]
tensor, pitched views, NV12 surfaces (against the numpy path on their cv2 conversion) and mixed sizes; graph reuse over
fresh allocations and pitches, and the upload bytes of a device-frame call."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TG = np.load(os.path.join(HERE, 'golden', 'track_golden.npz'))
CROPS = {'A': (0, 0, 480, 640), 'B': (16, 32, 448, 576), 'C': (48, 64, 384, 512)}


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
    h, w = img.shape[:2]
    i420 = cv2.cvtColor(img, cv2.COLOR_RGB2YUV_I420)
    u, v = i420[h:h + h // 4].reshape(h // 2, w // 2), i420[h + h // 4:].reshape(h // 2, w // 2)
    yuv = np.vstack([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])
    surf = torch.randint(0, 256, (h * 3 // 2, w + pad), dtype=torch.uint8, device='cuda')
    surf[:, :w] = torch.from_numpy(yuv).cuda()
    from gen6d_b200.frames import NV12
    return NV12(surf[:h, :w], surf[h:, :w]), cv2.cvtColor(yuv, cv2.COLOR_YUV2RGB_NV12)


def _pitched(img, pad=7, y0=1, x0=3):
    """RGB uint8 [h,w,3] -> a view of it inside a larger, garbage-filled device buffer (pitched rows, odd start)."""
    h, w = img.shape[:2]
    big = torch.randint(0, 256, (h + y0 + 2, w + x0 + pad, 3), dtype=torch.uint8, device='cuda')
    big[y0:y0 + h, x0:x0 + w] = torch.from_numpy(img).cuda()
    return big[y0:y0 + h, x0:x0 + w]


def _device(imgs, kinds):
    """kinds per frame: 'p' a pitched RGB view, 'n' NV12 -> (device frames, the numpy frames the numpy path gets)."""
    dev, ref = [], []
    for j, (img, k) in enumerate(zip(imgs, kinds)):
        if k == 'n':
            f, r = _nv12_of(img, pad=2 * j)
            dev.append(f)
            ref.append(r)
        else:
            dev.append(_pitched(img, pad=j + 1))
            ref.append(img)
    return dev, ref


def crop(img, K, which):
    y0, x0, h, w = CROPS[which]
    K = np.array(K, np.float64)
    K[0, 2] -= x0
    K[1, 2] -= y0
    return np.ascontiguousarray(img[y0:y0 + h, x0:x0 + w]), K


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


# ------------------------------------------------------------------------------------------ 1. the kernel
def test_gather_kernel_equals_host_twin():
    """One table of pitched RGB views (odd sizes, odd starts) and NV12 surfaces (wider pitches, planes at odd offsets,
    the saturating corners, 1080x1920) into a garbage-filled packed buffer, against g6d_frames_gather_host on the same
    bytes; then the same table rewritten to other allocations in place (the pointers live in the table)."""
    from gen6d_b200 import _lib, ops
    from gen6d_b200 import frames as fr
    sizes = [(7, 13), (2, 2), (6, 10), (480, 640), (1080, 1920), (7, 13), (1, 1), (10, 50)]
    kinds = 'pnnnnppn'
    # the saturating corners: Y in {0, 15, 16, 235, 255} (a row pair each) against every (U, V) in {0, 16, 128, 240, 255}^2
    corners_y = np.repeat(np.asarray([0, 15, 16, 235, 255], np.uint8), 2)[:, None].repeat(50, 1)
    cs = [0, 16, 128, 240, 255]
    corners_uv = np.asarray([[c for u in cs for v in cs for c in (u, v)]] * 5, np.uint8)

    def build(seed):
        g = torch.Generator(device='cuda').manual_seed(seed)
        rows, host, keep = [], [], []             # keep: the device buffers the table points into
        plan = fr.FramePlan(sizes)
        for i, ((h, w), k) in enumerate(zip(sizes, kinds)):
            off = plan.table[i][0]
            if k == 'n':
                buf = torch.randint(0, 256, (3 + (h * 3 // 2) * (w + 5),), dtype=torch.uint8, device='cuda', generator=g)
                surf = buf[3:].view(h * 3 // 2, w + 5)
                keep.append(buf)
                if (h, w) == (10, 50):
                    surf[:h, :w] = torch.from_numpy(corners_y).cuda()
                    surf[h:, :w] = torch.from_numpy(corners_uv).cuda()
                y, uv = surf[:h, :w], surf[h:, :w]
                rows.append(ops.DeviceFrame(y.data_ptr(), uv.data_ptr(), w + 5, w + 5, h, w, _lib.G6D_FRAME_NV12, off))
                hs = surf.cpu().numpy()
                host.append((hs, ops.DeviceFrame(hs[:h].ctypes.data, hs[h:].ctypes.data, w + 5, w + 5, h, w, _lib.G6D_FRAME_NV12, off)))
            else:
                big = torch.randint(0, 256, (h + 1, w + 3, 3), dtype=torch.uint8, device='cuda', generator=g)
                v = big[1:, 1:1 + w]
                keep.append(big)
                rows.append(ops.DeviceFrame(v.data_ptr(), None, v.stride(0), 0, h, w, _lib.G6D_FRAME_RGB, off))
                hv = v.cpu().numpy()
                host.append((hv, ops.DeviceFrame(hv.ctypes.data, None, hv.strides[0], 0, h, w, _lib.G6D_FRAME_RGB, off)))
        return plan, rows, host, keep

    plan, rows, host, keep = build(1)
    dev_table = (ops.DeviceFrame * len(rows))(*rows)
    ops.frames_table_check(dev_table, plan.nbytes)
    table = torch.from_numpy(np.frombuffer(bytes(dev_table), np.uint8).copy()).cuda()
    out = ops.frames_gather(table, len(rows), plan.H, plan.W, plan.nbytes)
    want = ops.frames_gather_host((ops.DeviceFrame * len(host))(*[r for _, r in host]), plan.nbytes)
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    off, h, w = plan.table[7]
    np.testing.assert_array_equal(want[off:off + h * w * 3].reshape(h, w, 3),
                                  cv2.cvtColor(np.vstack([corners_y, corners_uv]), cv2.COLOR_YUV2RGB_NV12))
    # the same launch over other allocations: only the table's contents change
    _, rows2, host2, keep2 = build(2)
    table.copy_(torch.from_numpy(np.frombuffer(bytes((ops.DeviceFrame * len(rows2))(*rows2)), np.uint8).copy()).cuda())
    out.fill_(0xAB)
    ops._call('g6d_frames_gather', ops._p(table, torch.uint8), len(rows2), plan.H, plan.W, ops._p(out, torch.uint8), plan.nbytes,
              ops._stream())
    want2 = ops.frames_gather_host((ops.DeviceFrame * len(host2))(*[r for _, r in host2]), plan.nbytes)
    np.testing.assert_array_equal(out.cpu().numpy(), want2)


# ------------------------------------------------------------------------------------------ 2. batch entry points
def test_predict_batch_device_frames(est, frames):
    from gen6d_b200 import ops
    from gen6d_b200.network.base import IO_BYTES
    e, _ = est
    imgs, Ks = frames
    want = e.predict_batch(imgs, Ks)
    _same(e.predict_batch(torch.from_numpy(np.stack(imgs)).cuda(), Ks), want, 'tensor [qn,h,w,3]')
    dev, _ = _device(imgs, 'pppp')
    h0 = IO_BYTES['h2d']
    _same(e.predict_batch(dev, Ks), want, 'pitched views')
    qn = len(imgs)
    assert IO_BYTES['h2d'] - h0 == qn * C.sizeof(ops.DeviceFrame) + qn * 20 * 8          # the table and the cameras only
    dev, ref = _device(imgs, 'npnp')
    _same(e.predict_batch(dev, Ks), e.predict_batch(ref, Ks), 'NV12 + RGB')
    # mixed sizes: pitched crops of the device frames, RGB and NV12
    pattern = 'ABCA'
    cut = [crop(img, K, z) for img, K, z in zip(imgs, Ks, pattern)]
    full = [torch.from_numpy(img).cuda() for img in imgs]
    dev, ref = [], []
    for j, (z, (c, _)) in enumerate(zip(pattern, cut)):
        if j % 2:
            f, r = _nv12_of(c, pad=4)
            dev.append(f)
            ref.append(r)
        else:
            y0, x0, h, w = CROPS[z]
            dev.append(full[j][y0:y0 + h, x0:x0 + w])
            ref.append(c)
    mKs = [k for _, k in cut]
    _same(e.predict_batch(dev, mKs), e.predict_batch(ref, mKs), 'mixed sizes')


def test_predict_instances_device_frames(est, frames):
    e, _ = est
    imgs, Ks = frames
    dev, ref = _device(imgs, 'pnpn')
    _same(e.predict_instances(dev, Ks, max_instances=2), e.predict_instances(ref, Ks, max_instances=2), 'instances')
    cut = [crop(img, K, z) for img, K, z in zip(imgs, Ks, 'ABAC')]
    dev, ref = _device([c for c, _ in cut], 'nppn')
    mKs = [k for _, k in cut]
    _same(e.predict_instances(dev, mKs, max_instances=2), e.predict_instances(ref, mKs, max_instances=2), 'instances mixed')


def test_object_set_device_frames(objs, frames):
    imgs, Ks = frames
    _same(objs.predict(torch.from_numpy(np.stack(imgs)).cuda(), Ks), objs.predict(imgs, Ks), 'objs tensor')
    dev, ref = _device(imgs, 'npnp')
    _same(objs.predict(dev, Ks), objs.predict(ref, Ks), 'objs NV12')
    _same(objs.predict_instances(dev, Ks, max_instances=2), objs.predict_instances(ref, Ks, max_instances=2), 'objs instances')
    cut = [crop(img, K, z) for img, K, z in zip(imgs, Ks, 'ABCB')]
    dev, ref = _device([c for c, _ in cut], 'pnpn')
    mKs = [k for _, k in cut]
    _same(objs.predict(dev, mKs), objs.predict(ref, mKs), 'objs mixed')
    _same(objs.predict_instances(dev, mKs, max_instances=2), objs.predict_instances(ref, mKs, max_instances=2), 'objs instances mixed')


def test_graph_reuse_over_fresh_allocations_and_overwrites(est, frames):
    """Two calls over fresh allocations with other pitches replay the first call's graph (no new stage) with the right
    results; overwriting the caller's tensor after a call and calling again follows the new contents."""
    e, _ = est
    imgs, Ks = frames
    a = [_pitched(img, pad=3) for img in imgs]
    want = e.predict_batch(imgs, Ks)
    _same(e.predict_batch(a, Ks), want, 'first')
    n = len(e.stages.stages)
    b = [_pitched(img, pad=11, y0=2, x0=5) for img in imgs]
    del a
    torch.cuda.empty_cache()
    _same(e.predict_batch(b, Ks), want, 'fresh allocations')
    assert len(e.stages.stages) == n
    t = torch.from_numpy(np.stack(imgs)).cuda()
    _same(e.predict_batch(t, Ks), want, 'tensor')
    t.copy_(torch.from_numpy(np.stack(imgs[::-1])).cuda())                    # the caller reuses its buffer
    _same(e.predict_batch(t, Ks[::-1]), e.predict_batch(imgs[::-1], Ks[::-1]), 'overwritten')
    assert len(e.stages.stages) == n


# ------------------------------------------------------------------------------------------ 3. trackers
@pytest.fixture(scope='module')
def video(est):
    _, db = est
    K = TG['track.K']
    return [db.render(p, K) for p in TG['track.gt_poses']], K


def _step_frames(video, t, pattern, kinds):
    """Step t's frames (sizes `pattern`) -> (device frames, numpy frames of the same RGB bytes, Ks)."""
    frames, K = video
    cut = [crop(frames[(t + s) % len(frames)], K, z) for s, z in enumerate(pattern)]
    dev, ref = _device([c for c, _ in cut], kinds)
    return dev, ref, [k for _, k in cut]


def _track_pair(make, video, pattern, kinds, reset=(), steps=3):
    """The same steps on a device-frame tracker and a numpy tracker: a full step, refine steps, a reset(reset) mixed
    step and one more refine step, every output equal.  -> the two trackers."""
    dt, nt = make(), make()
    for t in range(steps + 2):
        if t == steps and reset:
            dt.reset(list(reset))
            nt.reset(list(reset))
        dev, ref, Ks = _step_frames(video, t, pattern, kinds)
        _same(dt.step(dev, Ks), nt.step(ref, Ks), f'step {t} {pattern} {kinds}')
    return dt, nt


def test_tracker_device_frames(est, video):
    e, _ = est
    dt, _ = _track_pair(lambda: e.tracker(num_sequences=3), video, 'AAA', 'pnp', reset=[1])
    assert all(k[0][0] == 'device' for k in dt.stages.stages)          # k[0]: the graph name
    n = len(dt.stages.stages)
    dev, _, Ks = _step_frames(video, 9, 'AAA', 'npp')                            # other allocations and pitches
    dt.step(dev, Ks)
    assert len(dt.stages.stages) == n
    _track_pair(lambda: e.tracker(num_sequences=4), video, 'ABCA', 'pnnp', reset=[2])
    # est.track goes through step()
    frames, K = video
    dev = [_pitched(frames[t]) for t in range(3)]
    for (p, s, i), (wp, ws, wi) in zip(e.track(dev, K), e.track(frames[:3], K)):
        _same((p, s, i), (wp, ws, wi), 'track')


def test_object_tracker_device_frames(objs, video):
    _track_pair(lambda: objs.tracker(num_sequences=2), video, 'AA', 'np', reset=[0])
    _track_pair(lambda: objs.tracker(num_sequences=3), video, 'ABA', 'pnn', reset=[1])


def test_instance_trackers_device_frames(est, objs, video):
    """Re-detection every second step: ids and every output as the numpy run's."""
    e, _ = est
    for pattern, kinds in (('AA', 'pn'), ('ABC', 'npn')):
        _track_pair(lambda: e.instance_tracker(num_sequences=len(pattern), max_instances=2, gate=1e6, redetect_every=2),
                    video, pattern, kinds, steps=4)
        _track_pair(lambda: objs.instance_tracker(num_sequences=len(pattern), max_instances=2, gate=1e6, redetect_every=2),
                    video, pattern, kinds, steps=3)


def test_device_frames_rejected_on_the_wrong_device_or_path(est, frames):
    e, _ = est
    imgs, Ks = frames
    dev = torch.from_numpy(np.stack(imgs)).cuda()
    with pytest.raises(ValueError, match='uint8'):
        e.predict_batch(dev.to(torch.int16), Ks)
    with pytest.raises(ValueError, match='is on cpu'):
        e.predict_batch(list(dev.cpu()), Ks)
    with pytest.raises(ValueError, match='strides'):
        e.predict_batch(list(dev[:, :, ::2]), Ks)
    with pytest.raises(TypeError, match='pose_inits'):
        e.predict_batch(dev, Ks, pose_inits=[np.eye(3, 4)] * len(imgs))
    with pytest.raises(TypeError, match='device pipeline'):
        e.predict(dev[0], Ks[0])
