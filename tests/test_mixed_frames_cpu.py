"""Frames of different sizes (gen6d_b200/frames.py) without a GPU: the packing plan, the size pattern in the graph names,
the scatter of per-size detection rows back to frame order, and the argument errors."""
import types

import numpy as np
import pytest
import torch

from gen6d_b200 import frames as fr


def _frames(sizes, seed=0):
    rng = np.random.RandomState(seed)
    return [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in sizes]


class _Uploader:
    """The two upload methods FramePlan.upload calls, on the host (the device copy is PackedModule's)."""

    def upload_packed(self, arrays, offsets, nbytes):
        buf = np.zeros(nbytes, np.uint8)
        for a, off in zip(arrays, offsets):
            buf[off:off + a.nbytes] = a.reshape(-1)
        return torch.from_numpy(buf)

    def upload_frame(self, frames):
        return torch.from_numpy(np.stack(frames))

    def _to_dev(self, a):
        return torch.from_numpy(np.ascontiguousarray(a))


def test_plan_groups_offsets_and_table():
    pattern = [(5, 7), (3, 9), (5, 7), (2, 2), (3, 9), (5, 7)]
    plan = fr.FramePlan(pattern)
    assert plan.mixed and plan.pattern == tuple(pattern) and (plan.H, plan.W) == (5, 9)
    assert [(h, w) for h, w, _, _ in plan.groups] == [(5, 7), (3, 9), (2, 2)]          # order of first appearance
    assert [g[2].tolist() for g in plan.groups] == [[0, 2, 5], [1, 4], [3]]           # input order inside a group
    offs = [g[3] for g in plan.groups]
    assert offs == [0, 3 * 105 + (-3 * 105) % 256, 512 + 256]
    assert all(o % fr.ALIGN == 0 for o in offs)
    assert plan.nbytes == 768 + 256
    assert plan.order.tolist() == [0, 2, 5, 1, 4, 3]
    want = {0: (0, 5, 7), 2: (105, 5, 7), 5: (210, 5, 7), 1: (512, 3, 9), 4: (512 + 81, 3, 9), 3: (768, 2, 2)}
    assert plan.table == [want[i] for i in range(6)]
    assert not fr.FramePlan([(4, 4)] * 3).mixed


def test_packed_upload_holds_each_frame_at_its_table_offset():
    sizes = [(5, 7), (3, 9), (5, 7), (2, 2)]
    imgs = _frames(sizes)
    plan = fr.FramePlan(fr.size_pattern(imgs))
    packed, order = plan.upload(_Uploader(), imgs)
    packed = packed.numpy()
    assert packed.shape == (plan.nbytes,) and order.tolist() == plan.order.tolist()
    for img, (off, h, w) in zip(imgs, plan.table):
        np.testing.assert_array_equal(packed[off:off + h * w * 3].reshape(h, w, 3), img)
    # what the canvas kernel makes of it (the GPU test pins g6d_frames_canvas to this)
    canvas = np.zeros((len(imgs), plan.H, plan.W, 3), np.uint8)
    for i, (off, h, w) in enumerate(plan.table):
        canvas[i, :h, :w] = packed[off:off + h * w * 3].reshape(h, w, 3)
    for i, img in enumerate(imgs):
        np.testing.assert_array_equal(canvas[i, :img.shape[0], :img.shape[1]], img)


def test_same_packed_length_different_patterns_get_different_graph_names():
    a, b = [(16, 16), (8, 32), (16, 16)], [(8, 32), (16, 16), (16, 16)]
    pa, pb = fr.FramePlan(a), fr.FramePlan(b)
    assert pa.nbytes == pb.nbytes and pa.key('predict') != pb.key('predict')
    up = _Uploader()
    na, _, ia = fr.stage(up, 'predict', lambda *x: x, _frames(a))
    nb, _, ib = fr.stage(up, 'predict', lambda *x: x, _frames(b))
    assert [tuple(t.shape) for t in ia] == [tuple(t.shape) for t in ib]          # equal input shapes ...
    assert na != nb                                                               # ... different graphs
    one = _frames([(16, 16)] * 3)
    fn = lambda *x: x
    name, body, inputs = fr.stage(up, 'predict', fn, one)
    assert name == 'predict' and body is fn and len(inputs) == 1 and tuple(inputs[0].shape) == (3, 16, 16, 3)


@pytest.mark.parametrize('L', [1, 3, 8])
def test_scatter_rows_matches_numpy(L):
    """L = 1: frame-major rows; L = K: object-major; L = M or M*K: instance-major.  Group rows l*g + j go to l*n + idx[j]."""
    pattern = [(4, 4), (2, 6), (4, 4), (4, 4), (3, 3), (2, 6)]
    plan = fr.FramePlan(pattern)
    n = len(pattern)
    rng = np.random.RandomState(L)
    parts = [rng.randn(L * len(idx), 4).astype(np.float32) for _, _, idx, _ in plan.groups]
    want = np.full((L * n, 4), np.nan, np.float32)
    for p, (_, _, idx, _) in zip(parts, plan.groups):
        g = len(idx)
        for l in range(L):
            for j in range(g):
                want[l * n + idx[j]] = p[l * g + j]
    assert not np.isnan(want).any()
    got = fr.scatter_rows([torch.from_numpy(p) for p in parts], [torch.from_numpy(g[2]) for g in plan.groups], n)
    np.testing.assert_array_equal(got.numpy(), want)
    # per_size: detection once per group, rows back in frame order (int tensors and tuples too)
    canvas = torch.zeros(n, 4, 6, 3, dtype=torch.uint8)
    groups = [(torch.full((len(idx), h, w, 3), z, dtype=torch.uint8), torch.from_numpy(idx))
              for z, (h, w, idx, _) in enumerate(plan.groups)]
    detect = lambda u8: (u8[:, 0, 0, 0].to(torch.int32).repeat(L), torch.full((L * u8.shape[0],), u8.shape[1]))
    with fr._registered(canvas, groups):
        zid, rows = fr.per_size(detect, canvas)
    size_of = {i: z for z, (_, _, idx, _) in enumerate(plan.groups) for i in idx}
    assert zid.tolist() == [size_of[i] for _ in range(L) for i in range(n)]
    assert rows.tolist() == [pattern[i][0] for _ in range(L) for i in range(n)]
    assert fr.per_size(lambda u8: u8.shape[0], canvas) == n                      # not registered any more: detect(frames)


def test_size_buckets_per_size():
    from gen6d_b200.track import _bucket, _mixed_inputs, _size_buckets
    pattern = [(4, 4), (2, 6), (4, 4), (2, 6), (4, 4), (4, 4), (2, 6)]
    plan = fr.FramePlan(pattern)
    S = len(pattern)
    for reinit in ([1], [0, 2, 4], [0, 1], [3, 5, 6], list(range(S))):
        reinit = np.asarray(reinit)
        seq, blocks, pick = _size_buckets(reinit, plan)
        s = 0
        for (_, _, idx, _), b in zip(plan.groups, blocks):
            mine = [r for r in reinit if r in idx]
            assert b == _bucket(len(mine), len(idx))
            assert seq[s:s + b].tolist() == mine + [mine[-1]] * (b - len(mine)) if b else True
            s += b
        assert len(seq) == sum(blocks) and (seq[pick] == reinit).all()
        pending = np.zeros(S, bool)
        pending[reinit] = True
        got, b, (gseq, tgt, _, _) = _mixed_inputs(S, 2, pending, np.ones(S, bool), 3, 1, 'cpu', plan)
        assert b == len(seq) and gseq.tolist() == seq.tolist() and got.tolist() == reinit.tolist()
        t = S + np.arange(b)
        t[pick] = reinit
        assert tgt.tolist() == t.tolist() + (S + b + t).tolist()


def test_argument_errors():
    good = _frames([(4, 4), (6, 6)])
    Ks = [np.eye(3)] * 2
    assert len(fr.check_frames(good, Ks, 'x')) == 2
    with pytest.raises(ValueError, match='uint8'):
        fr.check_frames([good[0], good[1].astype(np.float32)], Ks, 'x')
    with pytest.raises(ValueError, match='uint8 \\[h, w, 3\\]'):
        fr.check_frames([good[0], good[1][..., :2]], Ks, 'x')
    with pytest.raises(ValueError, match='at least one frame'):
        fr.check_frames([], [], 'x')
    with pytest.raises(ValueError, match='one K per frame'):
        fr.check_frames(good, Ks[:1], 'x')
    fr.require_one_size(_frames([(4, 4)] * 3), 'x')
    with pytest.raises(ValueError, match='one size'):
        fr.require_one_size(good, 'x')


def _host_estimator():
    """An estimator with the device glue off (the host-sequenced path); its networks are never reached."""
    from gen6d_b200.estimator import Gen6DEstimator
    mod = lambda: types.SimpleNamespace(generation=0, weights_generation=0)
    return Gen6DEstimator({'device_glue': False}, modules={'detector': mod(), 'selector': mod(), 'refiner': mod()})


def test_host_paths_reject_mixed_sizes_before_uploading():
    est = _host_estimator()
    imgs, Ks = _frames([(32, 32), (32, 64)]), [np.eye(3)] * 2
    with pytest.raises(ValueError, match="one size.*device_glue"):
        est.predict_batch(imgs, Ks)
    trk = est.tracker(num_sequences=2, bbox_3d=np.asarray([[x, y, z] for x in (0, 1) for y in (0, 1) for z in (0, 1)], np.float32))
    with pytest.raises(ValueError, match="one size.*device_glue"):
        trk.step(imgs, Ks)
