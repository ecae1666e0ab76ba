"""GPU: the render pass.  pb_render_overlay against the NumPy compositor on random display lists, and
TrackingRunner's rendered frames, video file and collected data against the host restatement of the reference's
drawing loop."""
import numpy as np
import pytest
import torch

from padel_analytics_b200 import _lib as L
from padel_analytics_b200 import synth
from padel_analytics_b200.analytics import DataAnalytics, ProjectedCourt
from padel_analytics_b200.render import composite_numpy, render_frame_cpu
from padel_analytics_b200.trackers import KeypointsTracker, TrackingRunner
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from test_trackers_gpu import H, W, _four_ckpts, _four_trackers, _vi

pytestmark = pytest.mark.gpu


def _random_list(rng, B, Hh, Ww, per_frame):
    rows, sprites, offsets, size = [], [], [0], 0
    for f in range(B):
        n = 0 if f == 1 else per_frame  # frame 1: empty list
        for _ in range(n):
            w, h = int(rng.integers(1, 90)), int(rng.integers(1, 40))
            x0, y0 = int(rng.integers(-w, Ww + 1)), int(rng.integers(-h, Hh + 1))  # clipped at every edge
            if rng.random() < 0.2:
                rows.append((x0, y0, w, h, 0, 0, 0, L.OVERLAY_BLEND))
                continue
            pitch = w + int(rng.integers(0, 3))
            sp = (rng.random((h, pitch)) < 0.5).astype(np.uint8) * rng.integers(1, 256, (h, pitch)).astype(np.uint8)
            rows.append((x0, y0, w, h, size, pitch, int(rng.integers(0, 1 << 24)), L.OVERLAY_STAMP))
            sprites.append(sp.reshape(-1))
            size += sp.size
        offsets.append(len(rows))
    return (np.array(rows, dtype=L.OVERLAY_REC), np.array(offsets, np.int32),
            np.concatenate(sprites) if sprites else np.zeros(1, np.uint8))


@pytest.mark.parametrize("Hh,Ww", [(37, 41), (64, 333), (19, 1279), (1080, 1920)])
def test_overlay_kernel_equals_numpy_compositor(Hh, Ww):
    rng = np.random.default_rng(Hh * 7 + Ww)
    B = 4
    frames = rng.integers(0, 256, (B, Hh, Ww, 3), dtype=np.uint8)
    recs, offsets, atlas = _random_list(rng, B, Hh, Ww, per_frame=60)
    lut = rng.integers(0, 256, 256, dtype=np.uint8)
    exp = composite_numpy(frames.copy(), recs, offsets, atlas, lut)
    dev = torch.from_numpy(frames).cuda()
    d_recs = torch.from_numpy(recs.view(np.uint8)).cuda()
    d_off = torch.from_numpy(offsets).cuda()
    d_atlas = torch.from_numpy(atlas).cuda()
    d_lut = torch.from_numpy(lut).cuda()
    L.check(L.lib().pb_render_overlay(dev.data_ptr(), B, Hh, Ww, d_recs.data_ptr(), d_off.data_ptr(),
                                      d_atlas.data_ptr(), d_lut.data_ptr(), L.stream_ptr()))
    got = dev.cpu().numpy()
    assert np.array_equal(got[1], frames[1])  # empty list: untouched
    if not np.array_equal(got, exp):
        f, y, x, c = np.argwhere(got != exp)[0]
        raise AssertionError(f"{int((got != exp).sum())} bytes differ, first at frame {f} (x, y, c) = ({x}, {y}, {c})")


def _reference_frames(trackers, frames, fixed, data_analytics=None):
    court = ProjectedCourt(_vi(len(frames)))
    return [render_frame_cpu(f, i, trackers, court, data_analytics, fixed) for i, f in enumerate(frames)]


def _fixed_court():
    rng = np.random.default_rng(5)
    base = np.array([[0.29, 0.91], [0.71, 0.91], [0.32, 0.76], [0.5, 0.76], [0.68, 0.76], [0.35, 0.56], [0.65, 0.56],
                     [0.38, 0.41], [0.5, 0.41], [0.62, 0.41], [0.4, 0.31], [0.6, 0.31]]) * [W, H]
    return Keypoints([Keypoint(i, tuple(v)) for i, v in enumerate((base + rng.normal(0, 2, base.shape)).tolist())])


@pytest.mark.parametrize("keypoints,ball", [("model", True), ("model", False), ("fixed", True), ("fixed", False)])
def test_render_frames_equal_the_host_restatement(keypoints, ball):
    T, B = 19, 4
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=5)]
    med = synth.make_median(H, W).numpy()
    tr = _four_trackers(B, med)
    if keypoints == "fixed":
        tr[2] = KeypointsTracker(None, batch_size=B, fixed_keypoints_detection=_fixed_court())
    if not ball:
        tr = tr[:3]
    run = TrackingRunner(tr, video_info=_vi(T))
    run.render_batch_size = 8
    run.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
    assert run.is_fixed_keypoints == (keypoints == "fixed")
    got = list(run.render_frames())
    exp = _reference_frames(run.trackers, fr, run.is_fixed_keypoints)
    assert len(got) == T
    for i in range(T):
        if not np.array_equal(got[i], exp[i]):
            ys, xs = np.nonzero((got[i] != exp[i]).any(-1))
            raise AssertionError(f"frame {i}: {len(ys)} pixels differ, e.g. (x, y) = {list(zip(xs, ys))[:8]}")
    assert any(len(p) for p in run.trackers["players_tracker"].results.predictions), "vacuous: no players"


def test_run_writes_the_video_and_collects_the_data(tmp_path):
    import cv2

    T, B = 21, 4
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=2)]
    tr = _four_trackers(B, synth.make_median(H, W).numpy())
    out = tmp_path / "results.mp4"
    run = TrackingRunner(tr, video_info=_vi(T), inference_path=str(out), collect_data=True)
    run.render_batch_size = 8
    timings = run.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
    assert "_render" in timings
    cap = cv2.VideoCapture(str(out))
    assert cap.isOpened()
    assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (W, H)
    assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(30.0)
    n = 0
    while cap.read()[0]:
        n += 1
    cap.release()
    assert n == T
    da = DataAnalytics()
    _reference_frames(run.trackers, fr, run.is_fixed_keypoints, da)
    da.frames = da.frames[:-1]
    assert len(run.data_analytics) == T and run.data_analytics.frames == da.frames
    got, exp = run.data_analytics.into_dataframe(30.0), da.into_dataframe(30.0)
    assert list(got.columns) == list(exp.columns)
    assert np.array_equal(got.to_numpy(np.float64), exp.to_numpy(np.float64), equal_nan=True)
    # without a video: the same data, no frame rendered
    run2 = TrackingRunner(tr, video_info=_vi(T), collect_data=True)
    run2.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
    assert np.array_equal(run2.data_analytics.into_dataframe(30.0).to_numpy(np.float64), got.to_numpy(np.float64),
                          equal_nan=True)


def test_sharded_run_renders_on_rank_0_like_the_single_process_run(tmp_path):
    import os
    import subprocess
    import sys
    from pathlib import Path

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = Path(__file__).resolve().parents[1]
    cks = _four_ckpts()
    torch.save(cks, tmp_path / "ckpts.pt")
    script = tmp_path / "render2.py"
    script.write_text(f"""
import sys, os
sys.path.insert(0, {str(root)!r}); sys.path.insert(0, {str(root / 'tests')!r})
import numpy as np, torch, torch.distributed as dist
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
from padel_analytics_b200 import synth
from padel_analytics_b200.trackers import TrackingRunner
from test_trackers_gpu import _four_trackers, _vi, H, W
T, B = 23, 4
fr = [f.numpy() for f in synth.make_frames(T, H, W, start=7)]
tr = _four_trackers(B, None, ckpts=torch.load({str(tmp_path / 'ckpts.pt')!r}, weights_only=False), median_max_sample_num=11)
path = {str(tmp_path)!r} + f"/rank{{dist.get_rank()}}.mp4"
run = TrackingRunner(tr, video_info=_vi(T), inference_path=path, collect_data=True)
run.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
if dist.get_rank() == 0:
    np.save({str(tmp_path / 'frames.npy')!r}, np.stack(list(run.render_frames())))
    print("RENDER2_DONE")
dist.destroy_process_group()
""")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541", str(script)], capture_output=True,
                       text=True, env=env, timeout=900)
    assert "RENDER2_DONE" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    assert (tmp_path / "rank0.mp4").exists() and not (tmp_path / "rank1.mp4").exists()
    T, B = 23, 4
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=7)]
    tr = _four_trackers(B, None, ckpts=cks, median_max_sample_num=11)
    run = TrackingRunner(tr, video_info=_vi(T))
    run.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
    assert np.array_equal(np.load(tmp_path / "frames.npy"), np.stack(list(run.render_frames())))
