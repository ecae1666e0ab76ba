"""Tracking a frame stream of unknown length (`TrackingRunner.stream`) against `TrackingRunner.run()` on the same
frames: every yielded entry, the trackers' final results (InpaintNet included), the latency bound of the docstring,
and a frame of another size mid-stream."""
import json

import numpy as np
import pytest
import torch

from oracle import inpaint as OI
from oracle import weights as OW
from padel_analytics_b200 import synth
from padel_analytics_b200.trackers import (BallTracker, KeypointsTracker, PlayerKeypointsTracker, PlayerTracker,
                                           TrackingRunner)
from padel_analytics_b200.trackers import sv_compat as sv
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints

pytestmark = pytest.mark.gpu
H, W = 1080, 1920
B = 4
LENGTHS = sorted({0, 1, 7, 8, 9, B, B + 7, 3 * B + 5})
M = 5  # background from the stream: its first 5 frames
T_LAT = 8 * B + 16  # the latency test's stream


@pytest.fixture(scope="module")
def ckpts():
    return {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
            "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}


@pytest.fixture(scope="module")
def trackers(ckpts):
    """"yolo": the three YOLO trackers and the ball without InpaintNet; "fixed": players, a fixed court and the ball
    with InpaintNet."""
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    court = Keypoints([Keypoint(id=i, xy=(100.0 * i, 50.0 + i)) for i in range(12)])
    groups = {"yolo": [PlayerTracker(ckpts["detect"], poly, batch_size=B),
                         PlayerKeypointsTracker(ckpts["pose13"], 1280, batch_size=B, load_path=None, save_path=None),
                         KeypointsTracker(ckpts["court12"], batch_size=B, model_type="yolo"),
                         BallTracker(ckpts["tracknet"], None, batch_size=B, median_max_sample_num=M)],
                "fixed": [PlayerTracker(ckpts["detect"], poly, batch_size=B),
                          KeypointsTracker(None, batch_size=B, model_type="yolo", fixed_keypoints_detection=court),
                          BallTracker(ckpts["tracknet"], ckpts["inpaint"], batch_size=B, median_max_sample_num=M)]}
    for t in groups["yolo"] + groups["fixed"]:
        t.video_info_post_init(_vi())
    return groups


@pytest.fixture(scope="module")
def video():
    return synth.make_frames(max(LENGTHS + [T_LAT]), H, W, start=3)


def _vi():
    return sv.VideoInfo(width=W, height=H, fps=30.0, total_frames=None)


def _ser(o):
    return json.dumps(o.serialize())


def _ball(tr):
    return next(t for t in tr if isinstance(t, BallTracker))


def _expected(tr, fr, T, med):
    """run() on frames fr[:T] from fresh trackers: {tracker name: [serialised object per frame]}"""
    for t in tr:
        t.restart()
    _ball(tr).median = med
    if T == 0 and med is None:  # no frame to take a background from: nothing to track
        return {str(t): [] for t in tr}
    TrackingRunner(tr, video_info=_vi()).run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
    return {str(t): [_ser(o) for o in t.results.predictions] for t in tr}


def _items(video, T, kind):
    if kind == "host frames":
        return [f.numpy() for f in video[:T]]
    if kind == "device frames":
        return [f for f in video[:T].cuda()]
    return [b for b in video[:T].cuda().split(3)]  # batches of 3 frames: they straddle the pass's chunks of B


@pytest.mark.parametrize("T", LENGTHS)
@pytest.mark.parametrize("which", ["yolo", "fixed"])
def test_stream_equals_run(trackers, video, T, which):
    """Every yielded entry equals run()'s results on the same frames, per tracker and frame (the ball without
    InpaintNet; with it, the yielded ball is TrackNet's and the final results equal run()'s), for host frames,
    device frames and batched device tensors, with the background given and taken from the stream."""
    tr = trackers[which]
    ball = _ball(tr)
    fr = [f.numpy() for f in video[:T]]
    for med in (synth.make_median(H, W).numpy(), None):
        exp = _expected(tr, fr, T, med)
        assert all(len(v) == T for v in exp.values())
        ball.median = None
        for kind in ("host frames", "device frames", "batched device"):
            for t in tr:
                t.restart()
            runner = TrackingRunner(tr, video_info=_vi())
            got = {str(t): [] for t in tr}
            for i, (f, entry) in enumerate(runner.stream(iter(_items(video, T, kind)), median=med)):
                assert f == i and set(entry) == set(got)
                for name, obj in entry.items():
                    got[name].append(_ser(obj))
                assert all(len(t.results) == f + 1 for t in tr)
            for name in got:
                if which == "fixed" and name == "ball_tracker":  # TrackNet per frame, InpaintNet at the end
                    assert len(got[name]) == T
                else:
                    assert got[name] == exp[name], (kind, med is None, name)
                assert [_ser(o) for o in runner.trackers[name].results.predictions] == exp[name], (kind, name)
    if T == max(LENGTHS):
        assert any('"visibility": 1' in s for s in exp["ball_tracker"]), "vacuous: no ball"
        assert any(json.loads(s) for s in exp["players_tracker"]), "vacuous: no players"


@pytest.mark.parametrize("median", [True, False])
def test_stream_latency_bound(trackers, video, median):
    """Once the background exists, the entry of every frame f is yielded before the pass pulls frame f + 2B + 8: at
    most frames 0 .. f + 2B + 7 have been pulled (or the M frames held for the background, when more).  Checked on
    every frame of a stream of 8B + 16 frames, single host frames with the background given and taken from the
    stream, and batches of B device frames with it given."""
    tr = trackers["yolo"]
    med = synth.make_median(H, W).numpy() if median else None
    held = 0 if median else M
    kinds = [("host frames", 1)] + ([("batched device", B)] if median else [])
    for kind, per_item in kinds:
        for t in tr:
            t.restart()
        _ball(tr).median = None
        items = [f.numpy() for f in video[:T_LAT]] if per_item == 1 else list(video[:T_LAT].cuda().split(B))
        pulled = [0]

        def counted():
            for it in items:
                pulled[0] += it.shape[0] if per_item > 1 else 1
                yield it

        at = {f: pulled[0] for f, _ in TrackingRunner(tr, video_info=_vi()).stream(counted(), median=med)}
        assert sorted(at) == list(range(T_LAT))
        for f, p in at.items():
            assert p <= max(held, f + 2 * B + 7), (kind, f, p)
        before_end = [f for f in at if f + 2 * B + 8 < T_LAT]  # frames whose bound is met before the stream ends
        assert len(before_end) >= 4 * B + 8, "vacuous: too few frames under the bound"


def test_stream_rejects_a_frame_of_another_size_mid_stream(trackers, video):
    tr = trackers["yolo"]
    for t in tr:
        t.restart()
    items = [f.numpy() for f in video[:10]] + [np.zeros((720, 1280, 3), np.uint8)]
    with pytest.raises(ValueError, match="same frame size"):
        for _ in TrackingRunner(tr, video_info=_vi()).stream(iter(items), median=synth.make_median(H, W).numpy()):
            pass
    torch.cuda.synchronize()
