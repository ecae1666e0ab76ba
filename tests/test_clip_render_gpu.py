"""GPU: `TrackingRunner.run_clips` with `inference_dir` and `collect_data` against a fresh
`TrackingRunner(..., inference_path=..., collect_data=True).run()` on each clip alone: the decoded frames of every
clip's video, its DataAnalytics and its CSV."""
import hashlib
import json

import numpy as np
import pytest

from oracle import inpaint as OI
from oracle import weights as OW
from padel_analytics_b200 import synth
from padel_analytics_b200.trackers import KeypointsTracker, TrackingRunner
from test_clips_gpu import LENGTHS, H, W, _trackers, _vi
from test_render_gpu import _fixed_court

pytestmark = pytest.mark.gpu
B = 32


def _decoded(path):
    """(fps, (w, h), sha1 of every decoded frame) of a video file."""
    import cv2

    cap = cv2.VideoCapture(str(path))
    assert cap.isOpened(), path
    fps, wh = cap.get(cv2.CAP_PROP_FPS), (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT)))
    hashes = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        hashes.append(hashlib.sha1(np.ascontiguousarray(f).tobytes()).hexdigest())
    cap.release()
    return fps, wh, hashes


def _data(da):
    df = da.into_dataframe(30.0)
    return {"frames": list(da.frames), "columns": list(df.columns), "table": df.to_numpy(np.float64),
            "csv": df.to_csv()}


@pytest.fixture(scope="module")
def frames():
    clips = [synth.make_frames(T, H, W, start=11 * i + 1) for i, T in enumerate(LENGTHS)]
    return {"host": [[f.numpy() for f in c] for c in clips], "device": [c.cuda() for c in clips]}


@pytest.fixture(scope="module")
def ckpts():
    return {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
            "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}


def _make(config, ckpts):
    tr = _trackers(B, synth.make_median(H, W).numpy(), ckpts)
    if config == "fixed_court_no_ball":
        tr = tr[:2] + [KeypointsTracker(None, batch_size=B, fixed_keypoints_detection=_fixed_court())]
    for t in tr:
        t.video_info_post_init(_vi(None))
    return tr


def _per_clip_runs(tr, fr, tmp):
    """What a loop of per-clip run() calls writes: decoded video and data per clip."""
    exp = []
    tmp.mkdir(exist_ok=True)
    for c, T in enumerate(LENGTHS):
        for t in tr:
            t.restart()
        path = tmp / f"ref{c:04d}.mp4"
        run = TrackingRunner(tr, video_info=_vi(T), inference_path=str(path), collect_data=True)
        run.run(frame_source=lambda lo, hi, c=c: iter(fr[c][lo:hi]), total_frames=T)
        exp.append({"video": _decoded(path), **_data(run.data_analytics),
                    "ball": json.dumps([o.serialize() for o in run.trackers["ball_tracker"].results])
                    if "ball_tracker" in run.trackers else ""})
    for t in tr:
        t.restart()
    return exp


def _counting(sources, calls):
    """The sources, each counting in calls[clip] how often it is read."""
    def counted(c, src):
        def read(lo, hi):
            calls[c] += 1
            return src(lo, hi)
        return read
    return [(counted(c, s), T) for c, (s, T) in enumerate(sources)]


def _sources(frames, kind):
    if kind == "host":
        return [(lambda lo, hi, c=c: iter(frames["host"][c][lo:hi]), T) for c, T in enumerate(LENGTHS)]
    dev = frames["device"]
    return [(lambda lo, hi, c=c: (dev[c][i:min(hi, i + 32)] for i in range(lo, hi, 32)), T)
            for c, T in enumerate(LENGTHS)]


def _check_data(runner, exp, save):
    assert len(runner.clips_data_analytics) == len(LENGTHS)
    for c, (da, e) in enumerate(zip(runner.clips_data_analytics, exp)):
        got = _data(da)
        assert got["frames"] == e["frames"] and len(da) == LENGTHS[c], c
        assert got["columns"] == e["columns"]
        assert np.array_equal(got["table"], e["table"], equal_nan=True), c
        assert (save / f"{c:04d}_data.csv").read_text() == e["csv"], c


@pytest.mark.parametrize("config", ["four_trackers", "fixed_court_no_ball"])
def test_run_clips_videos_and_data_equal_per_clip_runs(config, ckpts, frames, tmp_path):
    """Render batches of 8 and 32 frames (so batches span clips), host frames and device batches: each clip's mp4 has
    the clip's frame count, fps and size, and its decoded frames equal those of the per-clip run's file; the data and
    CSV files equal that run's."""
    tr = _make(config, ckpts)
    exp = _per_clip_runs(tr, frames["host"], tmp_path)
    assert any(e["table"][:, 1:9].size and not np.isnan(e["table"][:, 1:9]).all() for e in exp), \
        "vacuous: no projected player"
    if config == "four_trackers":
        assert any('"visibility": 1' in e["ball"] for e in exp), "vacuous: no ball"
    runner = TrackingRunner(tr, video_info=_vi(None))
    combos = [(8, "host"), (32, "device")] if config == "fixed_court_no_ball" else \
        [(8, "host"), (8, "device"), (32, "host"), (32, "device")]
    for rb, kind in combos:
        runner.render_batch_size = rb
        calls = [0] * len(LENGTHS)
        out, save = tmp_path / f"v{rb}{kind}", tmp_path / f"s{rb}{kind}"
        runner.run_clips(_counting(_sources(frames, kind), calls), save_dir=str(save), inference_dir=str(out),
                         collect_data=True)
        assert calls == [2] * len(LENGTHS), "each clip is read once to track and once to render"
        assert all(len(t.results) == 0 for t in tr), "run_clips must leave the trackers' results alone"
        for k in ("", "_decode", "_build", "_upload", "_overlay", "_download", "_encode"):
            assert f"_clips_render{k}" in runner.timings
        for c, T in enumerate(LENGTHS):
            fps, wh, hashes = _decoded(out / f"{c:04d}.mp4")
            assert (fps, wh, len(hashes)) == (pytest.approx(30.0), (W, H), T), (rb, kind, c)
            ref = exp[c]["video"][2]
            bad = [i for i in range(T) if hashes[i] != ref[i]]
            assert not bad, f"render batch {rb}, {kind} frames, clip {c}: frames {bad[:8]} differ"
        _check_data(runner, exp, save)


def test_run_clips_collect_data_reads_no_frame_again(ckpts, frames, tmp_path):
    """collect_data without inference_dir: the same data as the per-clip runs, no video, and no clip read after the
    tracking pass.  A clip of 0 frames gets an empty DataAnalytics and no video."""
    tr = _make("four_trackers", ckpts)
    exp = _per_clip_runs(tr, frames["host"], tmp_path / "ref")
    runner = TrackingRunner(tr, video_info=_vi(None))
    calls = [0] * len(LENGTHS)
    save = tmp_path / "save"
    runner.run_clips(_counting(_sources(frames, "host"), calls), save_dir=str(save), collect_data=True)
    assert calls == [1] * len(LENGTHS)
    assert not list(tmp_path.glob("**/0*.mp4"))
    _check_data(runner, exp, save)
    empty = [(lambda lo, hi: iter([]), 0)] * 2
    runner.run_clips(empty, save_dir=str(save), inference_dir=str(tmp_path / "v"), collect_data=True)
    assert not list((tmp_path / "v").glob("*.mp4"))
    assert [len(da) for da in runner.clips_data_analytics] == [0, 0]
    assert (save / "0001_data.csv").read_text().count("\n") == 1  # the header only
