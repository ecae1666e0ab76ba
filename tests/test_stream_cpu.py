"""Tracking a frame stream of unknown length, without a GPU: the in-order merge of `TrackingRunner.stream`, the
trackers and jobs it refuses, a stream of fixed detections end to end, and the ball pipeline's open-end window and
emit tables replayed through a restatement of the ensemble kernel against the reference's ensemble loop."""
import json
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import tracknet as OT
from padel_analytics_b200.engine.tracknet_engine import BallPipeline
from padel_analytics_b200.trackers import BallTracker, KeypointsTracker, TrackingRunner
from padel_analytics_b200.trackers import sv_compat as sv
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from padel_analytics_b200.trackers.runner import FrameMerge
from padel_analytics_b200.trackers.tracker import TrackingResults

VI = sv.VideoInfo(width=8, height=6, fps=30.0, total_frames=None)
COURT = Keypoints([Keypoint(id=i, xy=(10 * i, 20 + i)) for i in range(12)])


# ---- the in-order merge ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_merge_yields_each_frame_once_in_order_when_all_trackers_have_it(seed):
    """Three stub trackers hand over their results in frame order but in bursts of random size at random times, one
    of them lagging behind: every frame comes out once, in order, with each tracker's own result, and only after
    the last tracker to reach it has."""
    rng = np.random.default_rng(seed)
    T = int(rng.integers(0, 60))
    names = ["players", "ball", "court"]
    merge = FrameMerge(names)
    sent = {n: 0 for n in names}
    got = []
    while any(sent[n] < T for n in names):
        n = names[int(rng.integers(0, 3))]
        burst = int(rng.integers(0, 9 if n != "ball" else 3))  # the ball arrives late and in small steps
        for f in range(sent[n], min(T, sent[n] + burst)):
            merge.put(n, f, (n, f))
        sent[n] = min(T, sent[n] + burst)
        for f, entry in merge.ready():
            assert f < min(sent.values()) + 1 and all(sent[k] > f for k in names)
            assert entry == {k: (k, f) for k in names}
            got.append(f)
    assert got == list(range(T))
    assert merge.ready() == []


def test_merge_rejects_results_out_of_order():
    merge = FrameMerge(["a", "b"])
    merge.put("a", 0, "x")
    with pytest.raises(ValueError, match="frame 1 is next"):
        merge.put("a", 2, "y")
    with pytest.raises(ValueError):
        FrameMerge([])


# ---- refusals ----------------------------------------------------------------------------------------------------
def _stub(cls, **attrs):
    t = object.__new__(cls)  # no CUDA here: skip the engine construction, set what is read
    t.results, t.load_path, t.save_path = TrackingResults(), None, None
    for k, v in attrs.items():
        setattr(t, k, v)
    return t


def _court(**kw):
    return _stub(KeypointsTracker, **{"model_type": "yolo", "model": None, "fixed_keypoints_detection": COURT, **kw})


def _frames(T, hw=(6, 8)):
    return (np.full(hw + (3,), i % 256, np.uint8) for i in range(T))


def test_stream_refuses_frames_trackers_cached_trackers_and_world_size(monkeypatch):
    pulled = []

    def frames():
        for f in _frames(5):
            pulled.append(1)
            yield f

    regressor = _stub(KeypointsTracker, model_type="resnet", model=object(), fixed_keypoints_detection=None)
    with pytest.raises(ValueError, match="keypoints_tracker"):
        TrackingRunner([regressor], video_info=VI).stream(frames())
    cached = _stub(BallTracker)
    cached.results.load([object()] * 3)
    with pytest.raises(ValueError, match=r"ball_tracker.*cached predictions"):
        TrackingRunner([_court(), cached], video_info=VI).stream(frames())
    with pytest.raises(ValueError, match="video_info"):
        TrackingRunner([_court()]).stream(frames())

    import torch.distributed as dist

    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda: 2)
    with pytest.raises(ValueError, match="world size 2"):
        TrackingRunner([_court()], video_info=VI).stream(frames())
    assert not pulled, "a refused stream must not pull a frame"


def test_stream_of_fixed_detections_yields_every_frame_and_checks_frame_size(tmp_path):
    """A fixed court needs no device: each frame is yielded as it is pulled, results grow with the frames yielded,
    single frames and batches alike, the predictions are saved once the stream ends (as run() saves them), and a
    frame of another size mid-stream raises ValueError."""
    court = _court(save_path=str(tmp_path / "court.json"))
    runner = TrackingRunner([court], video_info=VI)
    items = [f for f in _frames(3)] + [torch.zeros((4, 6, 8, 3), dtype=torch.uint8)] + [f for f in _frames(2)]
    pulled = [0]

    def counted():
        for it in items:
            pulled[0] += 1
            yield it

    seen = []
    for f, entry in runner.stream(counted()):
        assert entry == {"keypoints_tracker": COURT}
        assert len(court.results) == f + 1
        seen.append((f, pulled[0]))
    assert [f for f, _ in seen] == list(range(9))
    assert [p for _, p in seen] == [1, 2, 3, 4, 4, 4, 4, 5, 6]  # yielded as soon as pulled
    assert court.results.predictions == [COURT] * 9
    assert json.loads((tmp_path / "court.json").read_text()) == json.loads(json.dumps([COURT.serialize()] * 9))

    court.restart()
    bad = [np.zeros((6, 8, 3), np.uint8), np.zeros((6, 9, 3), np.uint8)]
    with pytest.raises(ValueError, match="same frame size"):
        list(runner.stream(iter(bad)))


# ---- the ball pipeline with an open end ---------------------------------------------------------------------------
def _open_pipeline(B):
    """A BallPipeline whose launches are recorded instead of run: (first window, nb, desc, frames pushed then)."""
    pipe = object.__new__(BallPipeline)
    pipe.B, pipe.ring = B, B + 8
    pipe.eng = SimpleNamespace(pred=torch.zeros(1))
    pipe.reset()
    pipe.launches = []

    def launch(key, first_window, row_slot, row_median, desc, want_ens=False):
        assert key == first_window and len(row_slot) == len(row_median)
        pipe.launches.append((first_window, len(row_slot), np.asarray(desc), pipe.n_frames_in))
        return lambda: (key, None)

    pipe._launch_batch = launch
    return pipe


def _ensemble_rows(rows, first_window, desc):
    """numpy restatement of pb_tracknet_ensemble_rows: rows[r] holds window first_window + r"""
    w = OT.ensemble_weight().numpy()
    out = []
    for cw0, tw, n in desc.tolist():
        base = cw0 - first_window
        if tw > n >= 7:
            out.append(np.stack([rows[base + n - 7 + k, 7 - k] * w[k] for k in range(8)]).sum(0, dtype=np.float32))
        else:
            acc = np.zeros(rows.shape[-2:], np.float32)
            for k in range(8):
                if 0 <= n - 7 + k < tw:
                    acc = acc + rows[base + n - 7 + k, 7 - k]
            out.append(acc / (np.float32(n + 1) if n < tw else np.float32(8 - (n - (tw - 1)))))
    return out


def _schedules(T, B):
    yield "batches", [min(B, T - i) for i in range(0, T, B)]
    yield "frames", [1] * T
    rng = np.random.default_rng(T * 31 + B)
    sizes, left = [], T
    while left:
        sizes.append(min(left, int(rng.integers(1, B + 1))))
        left -= sizes[-1]
    yield "ragged", sizes


@pytest.mark.parametrize("B", [1, 4, 9])
def test_open_end_ball_tables_reproduce_the_reference_ensemble(B):
    """Frames pushed in batches, one at a time or in ragged pieces, with the total unknown until `stream_end`: every
    launch keeps the windows it reads inside the heat-map buffer (7 carried + nb new), every frame is emitted exactly
    once, in order, never before frame f+7 has arrived, and the launches replayed through the kernel's restatement
    (with the engine's 7-row carry) equal the reference's stateful ensemble loop bit for bit, head, body and tail."""
    H, W = 8, 64  # an inner size at which torch's reduction over the 8 terms is sequential, as the kernel's
    for T in sorted({0, 1, 7, 8, 9, B, B + 7, 3 * B + 5}):
        g = torch.Generator().manual_seed(T + 100 * B)
        heat = torch.rand((max(0, T - 7), 8, H, W), generator=g)
        if len(heat):
            heat.view(-1)[::7] = 0.5
        every = heat.numpy()
        exp = OT.ensemble_reference_loop(heat, T, B).numpy()
        assert len(exp) == (T if T >= 8 else 0)
        for kind, sizes in _schedules(T, B):
            pipe = _open_pipeline(B)
            for n in sizes:
                assert pipe.n_frames_in + n <= pipe.n_windows + pipe.ring, "ring overflow"
                pipe.n_frames_in += n
                pipe.run_ready_async(None)
                # no window held back: every window whose 8 frames have arrived has run, and emitted its frame
                assert pipe.n_windows == max(0, pipe.n_frames_in - 7), (kind, T)
                assert sum(len(d) for _, _, d, _ in pipe.launches) == pipe.n_windows, (kind, T)
            open_launches = len(pipe.launches)
            pipe.stream_end(T)
            assert len(pipe.launches) - open_launches <= 1, "stream_end: one launch at most after the last push"
            rows = np.zeros((7 + B, 8, H, W), np.float32)
            got = []
            for fw, nb, desc, arrived in pipe.launches:
                assert 0 <= nb <= B and len(desc) <= B + 7
                lo = desc[:, 0] + np.maximum(desc[:, 2] - 7, 0)
                hi = desc[:, 0] + np.minimum(desc[:, 2], desc[:, 1] - 1)
                assert (lo >= fw - 7).all() and (hi < fw + nb).all(), (kind, T, fw, nb, desc)
                assert (desc[:, 2] + 8 <= arrived).all() or arrived == T, "a frame emitted before frame f+7 arrived"
                rows[7:7 + nb] = every[fw:fw + nb]
                got += list(zip(desc[:, 2].tolist(), _ensemble_rows(rows, fw - 7, desc)))
                if nb:
                    rows[:7] = rows[nb:nb + 7].copy()
            assert [f for f, _ in got] == list(range(len(exp))), (kind, T)
            for f, e in got:
                assert np.array_equal(e.view(np.uint32), exp[f].view(np.uint32)), (kind, T, f)
            with pytest.raises(Exception):
                pipe.stream_end(T + 1)  # a total other than the frames pushed


def test_known_total_tables_are_unchanged_by_the_open_end():
    """With the total known from the start (run(), run_clips), the launches are those of before: each batch emits
    its windows' frames and the batch of the last window also the 7 tail frames; stream_end then adds nothing."""
    B, T = 4, 21
    pipe = _open_pipeline(B)
    for i in range(0, T, B):
        pipe.n_frames_in += min(B, T - i)
        pipe.run_ready_async(T)
    got = [(fw, nb, d[:, 2].tolist(), d[:, 1].tolist()) for fw, nb, d, _ in pipe.launches]
    assert got == [(0, 1, [0], [14]), (1, 4, [1, 2, 3, 4], [14] * 4), (5, 4, [5, 6, 7, 8], [14] * 4),
                   (9, 4, [9, 10, 11, 12], [14] * 4), (13, 1, list(range(13, 21)), [14] * 8)]
    pipe.stream_end(T)
    assert len(pipe.launches) == 5
