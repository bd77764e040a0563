"""Boxes from another detector (row f19) without a GPU: g6d_det_from_boxes_host against the numpy restatement bit for
bit, the record layout, the box arguments of gen6d_b200/boxes.py, the box graph names, and the instance tracker's
re-detection schedule with boxes."""
import numpy as np
import pytest
import torch

import boxes_oracle as O
from gen6d_b200 import _lib
from gen6d_b200 import boxes as B
from gen6d_b200.instance_track import InstanceTracker, Schedule, mixed_name
from gen6d_b200.frames import FramePlan
from gen6d_b200.track import PartialStep

INV = B.inv_box_size(128)
DEV = 'cuda:0'


@pytest.fixture(scope='module', autouse=True)
def built():
    from gen6d_b200.build import build
    build()


def _same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert g.tobytes() == w.tobytes()


# ------------------------------------------------------------------------------------------ the records
@pytest.mark.parametrize('N', [1, 2, 16, 256])
@pytest.mark.parametrize('M', [1, 4, 16])
def test_host_twin_equals_restatement(N, M):
    rng = np.random.RandomState(1000 * N + M)
    for _ in range(3):
        t, c = O.random_table(rng, 11, N)
        _same(B.host_records(t, c, M, INV), O.records(t, c, M, INV))


def test_inv_box_size_is_exact_for_128():
    assert INV == 1 / 128 and B.inv_box_size(128) == float(np.float32(1 / 128))


def test_layout():
    t = np.zeros((3, 4, 5), np.float32)
    t[0, :3] = [[10, 20, 30, 60, 0.5], [0, 0, 8, 4, 0.9], [5, 5, 5, 9, 2.0]]      # the third is degenerate
    t[1, :2] = [[0, 0, np.nan, 1, 1], [1, 1, 3, 3, np.inf]]                        # neither usable
    t[2, :2] = [[0, 0, 2, 2, 0.3], [4, 4, 6, 10, 0.3]]                            # tied scores
    c = np.array([3, 2, 2], np.int32)
    det, valid, count = B.host_records(t, c, 4, INV)
    np.testing.assert_array_equal(count, [2, 0, 2])
    np.testing.assert_array_equal(valid, [[1, 0, 1], [1, 0, 1], [0, 0, 0], [0, 0, 0]])
    np.testing.assert_array_equal(det[0, 0], np.float32([4, 2, 8 / 128, 0.9]))
    np.testing.assert_array_equal(det[1, 0], np.float32([20, 40, 40 / 128, 0.5]))
    for m in (2, 3):                                                  # rows past the count repeat row 0, invalid
        np.testing.assert_array_equal(det[m, 0], det[0, 0])
        np.testing.assert_array_equal(det[m, 2], det[0, 2])
    for m in range(4):                                                # the empty-map record
        np.testing.assert_array_equal(det[m, 1], np.float32([0, 0, 1, -np.inf]))
    np.testing.assert_array_equal(det[0, 2], np.float32([1, 1, 2 / 128, 0.3]))    # the tie goes to the lower index
    np.testing.assert_array_equal(det[1, 2], np.float32([5, 7, 6 / 128, 0.3]))
    # counts are clamped to [0, N]
    _same(B.host_records(t, np.array([-3, 9, 2], np.int32), 4, INV), O.records(t, [0, 4, 2], 4, INV))


def test_kernel_arguments_are_checked():
    t, c = np.zeros((1, 1, 5), np.float32), np.ones(1, np.int32)
    for M, inv in ((0, INV), (17, INV), (1, 0.0), (1, float('inf'))):
        with pytest.raises(_lib.Gen6DLibraryError):
            B.host_records(t, c, M, inv)
    with pytest.raises(_lib.Gen6DLibraryError):
        B.host_records(np.zeros((1, 257, 5), np.float32), c, 1, INV)


# ------------------------------------------------------------------------------------------ boxes.py
def test_input_forms_and_bucket():
    b4 = np.array([[0, 0, 10, 20]], np.float64)
    b5 = np.array([[1, 2, 3, 4, 0.7], [5, 6, 9, 9, 0.1], [0, 0, 1, 1, 0]], np.float32)
    t = B.for_frames([b4, np.zeros((0, 4)), b5], 3, 'x', DEV)
    assert t.N == 4 and t.n_maps == 3
    np.testing.assert_array_equal(t.counts, [1, 0, 3])
    buf = t.host()
    tab, counts = buf[:3 * 4 * 5].reshape(3, 4, 5), buf[3 * 4 * 5:].view(np.int32)
    np.testing.assert_array_equal(counts, [1, 0, 3])
    np.testing.assert_array_equal(tab[0, 0], np.float32([0, 0, 10, 20, 0]))          # [n, 4]: score 0
    np.testing.assert_array_equal(tab[2, :3], b5)
    assert not tab[1].any() and not tab[0, 1:].any()
    for n, N in ((0, 1), (1, 1), (2, 2), (3, 4), (5, 8), (200, 256), (256, 256)):
        assert B.bucket(n) == N
        assert B.for_frames([np.tile(b4, (n, 1))], 1, 'x', DEV).N == N


def test_object_dicts_map_object_major():
    names = ['a', 'b']
    b = lambda k: np.tile(np.array([[0, 0, 4, 4, 1]], np.float32), (k, 1))
    t = B.for_objects([{'a': b(1)}, {'b': b(2), 'a': b(3)}, {}], names, 3, 'x', DEV)
    np.testing.assert_array_equal(t.counts, [1, 3, 0, 0, 2, 0])                       # j = o*qn + f
    with pytest.raises(ValueError, match='not in the set'):
        B.for_objects([{'c': b(1)}, {}, {}], names, 3, 'x', DEV)
    with pytest.raises(ValueError, match='dict'):
        B.for_objects([b(1), {}, {}], names, 3, 'x', DEV)
    t, has = B.for_sequences([None, {'b': b(1)}], 2, 'x', DEV, names)
    np.testing.assert_array_equal(has, [False, True])
    np.testing.assert_array_equal(t.counts, [0, 0, 0, 1])


def test_errors():
    ok = np.array([[0, 0, 1, 1]], np.float32)
    bad = {'non-finite': np.array([[0, 0, np.nan, 1]]), 'inf': np.array([[0, 0, 1, 1, np.inf]]),
           'overflow': np.array([[0, 0, 1e39, 1]]), 'degenerate': np.array([[0, 0, 0, 1]]),
           'negative': np.array([[0, 5, 1, 4]]), 'shape': np.zeros((2, 3)), 'rank': np.zeros(4),
           'too many': np.tile(ok, (257, 1)), 'cpu tensor': torch.zeros(1, 4), 'strings': np.array([['a'] * 4])}
    for name, b in bad.items():
        with pytest.raises(ValueError):
            B.for_frames([b], 1, name, DEV)
    with pytest.raises(ValueError, match='one entry per frame'):
        B.for_frames([ok], 2, 'x', DEV)
    with pytest.raises(ValueError, match='one entry per frame'):
        B.for_frames(None, 1, 'x', DEV)
    B.for_frames([np.tile(ok, (256, 1))], 1, 'x', DEV)


def test_predict_batch_takes_one_box_per_frame():
    for b in (np.zeros(4), np.zeros(5), np.zeros((1, 4)), np.zeros((1, 5))):
        (one,) = B.one_per_frame([b], 1, 'predict_batch')
        assert one.shape == (1, b.shape[-1])
    for b in (np.zeros(3), np.zeros((2, 4)), np.zeros((0, 4)), np.zeros((1, 6))):
        with pytest.raises(ValueError, match='exactly one box'):
            B.one_per_frame([b], 1, 'predict_batch')
    with pytest.raises(ValueError):
        B.one_per_frame([np.zeros(4)], 2, 'predict_batch')


def test_box_graph_names_apart_from_every_existing_name():
    plan = FramePlan([(48, 64), (32, 64)])
    part = PartialStep(6, 1, [4, 1], np.zeros(6, bool), np.ones(6, bool), 1)
    bases = ['predict', 'detect', 'refine', 'full', 'mixed', ('instances', 4, 1, 0.3, None), mixed_name(4, 2), mixed_name(4, (1, 2))]
    wraps = [lambda n: n, part.name, plan.key, plan.device_key, lambda n: plan.device_key(n, True)]
    existing = {w(b) for b in bases for w in wraps}
    boxed = {w(B.graph_name(b, N)) for b in bases + [('instances', 4)] for w in wraps for N in (1, 2, 256)}
    assert not existing & boxed
    assert len(boxed) == len(bases + [1]) * len(wraps) * 3                               # keyed on N


# ------------------------------------------------------------------------------------------ the schedule
@pytest.mark.parametrize('staggered', [False, True])
def test_box_detections_count_as_detector_detections(staggered):
    """Boxes for exactly the due sequences: counters and phases equal the detector schedule's at every step, for S, E in
    1..12; a due sequence without boxes stays due; boxes on a sequence that is not due restart its count at 1."""
    rng = np.random.RandomState(5)
    for S in range(1, 13):
        for E in range(1, 13):
            det, box = Schedule(S, E, staggered), Schedule(S, E, staggered)
            for t in range(30):
                if rng.rand() < 0.1:
                    marked = rng.rand(S) < 0.3
                    det.pending[marked] = box.pending[marked] = True
                stepped = np.flatnonzero(rng.rand(S) < 0.7) if rng.rand() < 0.5 else np.arange(S)
                if not len(stepped):
                    continue
                want_seq, want_kind = det.plan(stepped, len(stepped))
                got_seq, got_kind = box.plan(stepped, len(stepped), box.due()[stepped])
                np.testing.assert_array_equal(got_seq, want_seq)
                assert got_kind == want_kind
                det.advance(stepped)
                box.advance(stepped, got_seq)
                np.testing.assert_array_equal(box.count, det.count)
                np.testing.assert_array_equal(box.pending, det.pending)
            # a due sequence without boxes stays due; a boxed one that is not due restarts at 1
            sch = Schedule(S, E, staggered)
            due = sch.due().copy()
            hit = np.zeros(S, bool)
            hit[S // 2] = True
            det_seq, _ = sch.plan(np.arange(S), S, hit)
            sch.advance(np.arange(S), det_seq)
            np.testing.assert_array_equal(sch.due() & ~hit, due & ~hit)
            assert sch.count[S // 2] == 1 + sch.phase[S // 2]
            hit2 = np.zeros(S, bool)
            if S > 1:
                hit2[0] = True
                sch.advance(np.arange(S), hit2)            # sequence 0 was still pending: a marked detection
                assert sch.count[0] == 1 + sch.phase[0] and not sch.pending[0]
                sch.advance(np.arange(S), hit2)            # now a periodic one
                assert sch.count[0] == 1


class _FakeTracker(InstanceTracker):
    """An InstanceTracker's host planning without a GPU: _run records what it was asked to run."""

    def __init__(self, S, schedule, E=None):
        class Est:
            detector = type('D', (), {'device': DEV})()
            cfg = {'ref_resolution': 128}

            def _generation(self):
                return 0
        self.est, self._gen, self.S, self.M, self.K, self.schedule = Est(), 0, S, 2, 1, schedule
        self.redetect_every = E
        self._pending, self._since = True, 0
        self._schedule = Schedule(S, E, schedule == 'staggered')
        self._drawer, self.runs = None, []

    def _run(self, frames, Ks, out, kind, part=None, det_seq=None, boxes=None):
        self.runs.append((kind, None if det_seq is None else det_seq.copy(), boxes, part))
        b = len(frames)
        return [(np.zeros(b), np.zeros(b), np.zeros(b, np.int64), {})]


def _frames(n):
    return [np.zeros((8, 8, 3), np.uint8)] * n, [np.eye(3)] * n


def test_lockstep_needs_every_entry():
    trk = _FakeTracker(3, 'lockstep', E=5)
    box = np.array([[0, 0, 4, 4]], np.float32)
    with pytest.raises(ValueError, match='every sequence'):
        trk.step(*_frames(3), boxes=[box, None, box])
    with pytest.raises(ValueError, match='one entry per stepped sequence'):
        trk.step(*_frames(3), boxes=[box, box])
    trk._pending, trk._since = False, 2                  # not due: boxes still re-detect, and restart the count
    trk.step(*_frames(3), boxes=[box, np.zeros((0, 4)), box])
    kind, _, table, _ = trk.runs[-1]
    assert kind == 'detect' and trk._since == 1 and not trk._pending
    np.testing.assert_array_equal(table.counts, [1, 0, 1])
    trk.step(*_frames(3))
    assert trk.runs[-1][0] == 'refine' and trk._since == 2


@pytest.mark.parametrize('schedule', ['per_sequence', 'staggered'])
def test_which_sequences_detect(schedule):
    S, box = 4, np.array([[0, 0, 4, 4, 1]], np.float32)
    trk = _FakeTracker(S, schedule, E=3)
    trk.step(*_frames(S), boxes=[box, None, box, None])          # first step: all due, only 0 and 2 detect
    kind, det_seq, table, _ = trk.runs[-1]
    assert kind == 'mixed'
    np.testing.assert_array_equal(det_seq, [True, False, True, False])
    np.testing.assert_array_equal(table.counts, [1, 0, 1, 0])
    np.testing.assert_array_equal(trk.detecting(), [False, True, False, True])     # unboxed due sequences stay due
    trk.step(*_frames(S))                                          # no boxes: the detector takes the due ones
    np.testing.assert_array_equal(trk.runs[-1][1], [False, True, False, True])
    trk.step(*_frames(S), boxes=[None] * S)                        # boxes= with none given: nothing detects
    assert trk.runs[-1][0] == 'refine'
    trk.step(*_frames(S), boxes=[box] * S)
    assert trk.runs[-1][0] == 'detect'
    # a partial step: boxes follow sequences= order, compacted with the frames
    trk.step(*_frames(2), sequences=[3, 1], boxes=[None, box])
    kind, det_seq, table, part = trk.runs[-1]
    np.testing.assert_array_equal(part.seq[:2], [1, 3])
    np.testing.assert_array_equal(det_seq[:2], [True, False])
    assert not det_seq[2:].any()
    np.testing.assert_array_equal(table.counts[:2], [1, 0])
    with pytest.raises(ValueError, match='one entry per stepped sequence'):
        trk.step(*_frames(2), sequences=[3, 1], boxes=[box])


def test_redetect_every_none_never_runs_the_detector_with_boxes():
    S, box = 3, np.array([[0, 0, 4, 4, 1]], np.float32)
    trk = _FakeTracker(S, 'per_sequence', E=None)
    trk.step(*_frames(S), boxes=[box] * S)
    assert trk.runs[-1][0] == 'detect' and trk.runs[-1][2] is not None
    for t in range(10):
        trk.step(*_frames(S), boxes=[box if (t + s) % 4 == 0 else None for s in range(S)])
        kind, det_seq, table, _ = trk.runs[-1]
        assert kind == 'refine' or table is not None
        trk.step(*_frames(S))
        assert trk.runs[-1][0] == 'refine'
