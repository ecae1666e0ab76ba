"""CPU: the render pass's host side.  Court projection and data collection against the reference's own analytics
code (golden: tests/golden/make_analytics_golden.py), and the display-list decomposition (cv2 calls -> coverage sprites + blend) against whole-frame cv2
drawing, byte for byte, with primitives across every frame border."""
from pathlib import Path
from types import SimpleNamespace

import cv2
import numpy as np
import pytest

from padel_analytics_b200 import _lib as L
from padel_analytics_b200.analytics import DataAnalytics, ProjectedCourt
from padel_analytics_b200.render import (DisplayListBuilder, composite_numpy, pack_display_list,
                                         record_draw_calls, render_frame_cpu)
from padel_analytics_b200.trackers.ball_tracker import Ball
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from padel_analytics_b200.trackers.players_keypoints_tracker import PlayersKeypoints
from padel_analytics_b200.trackers.players_tracker import Player, Players
from padel_analytics_b200.trackers import sv_compat as sv

GOLDEN = Path(__file__).resolve().parent / "golden"


# ---- analytics against the reference -----------------------------------------------------------------------------
@pytest.mark.parametrize("seq", ["fixed", "per_frame", "first_missing"])
def test_projected_court_and_data_analytics_match_the_reference(seq):
    g = np.load(GOLDEN / "analytics_ref.npz")
    kp, present, players, counts, ball = (g[f"{seq}_in_{k}"] for k in ("kp", "kp_present", "players", "counts",
                                                                        "ball"))
    fixed = seq == "fixed"
    T = len(present)
    court = ProjectedCourt(sv.VideoInfo(width=1920, height=1080, fps=25.0))
    da = DataAnalytics()
    fixed_kps = Keypoints([Keypoint(i, tuple(float(v) for v in kp[0, i])) for i in range(12)])
    n_h = 0
    for t in range(T):
        kps = fixed_kps if fixed else Keypoints(
            [Keypoint(i, tuple(float(v) for v in kp[t, i])) for i in range(12)] if present[t] else [])
        H = court.update_homography(kps, fixed)
        if H is None:
            assert np.isnan(g[f"{seq}_H"][t]).all()
            da.step(1)
            continue
        n_h += 1
        np.testing.assert_allclose(H, g[f"{seq}_H"][t], rtol=0, atol=1e-9)
        pls = [SimpleNamespace(feet=(int(x), int(y)), id=int(i)) for x, y, i in players[t, :counts[t]]]
        proj = court.project_players(pls, H, da)
        assert [p.projection for p in proj] == [tuple(v) for v in g[f"{seq}_proj_players"][t, :counts[t]].tolist()]
        b = court.project_ball(SimpleNamespace(asint=lambda b=ball[t]: (int(b[0]), int(b[1]))), H)
        assert b.projection == tuple(g[f"{seq}_proj_ball"][t].tolist())
        da.step(1)
    assert n_h >= T - 3
    da.frames = da.frames[:-1]
    assert da.frames == g[f"{seq}_frames"].tolist() and len(da) == T
    df = da.into_dataframe(25)
    assert list(df.columns) == g[f"{seq}_columns"].tolist()
    ref = g[f"{seq}_table"]
    got = df.to_numpy(dtype=np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    np.testing.assert_allclose(np.nan_to_num(got), np.nan_to_num(ref), rtol=0, atol=1e-9)
    # the dict round trip keeps the positions
    back = DataAnalytics.from_dict(da.into_dict())
    assert back.into_dict() == da.into_dict()


def test_homography_rejects_unhandled_keypoint_counts():
    court = ProjectedCourt(sv.VideoInfo(width=1280, height=720, fps=25.0))
    with pytest.raises(ValueError):
        court.homography_matrix(Keypoints([Keypoint(i, (float(i), float(2 * i))) for i in range(11)]))


def test_data_collection_drops_ids_outside_1_to_4():
    da = DataAnalytics()
    for i, pos in ((7, (1.0, 1.0)), (8, (2.0, 2.0)), (1, (3.0, 3.0)), (5, (4.0, 4.0)), (2, (5.0, 5.0))):
        da.add_player_position(i, pos)
    da.step(1)
    d = da.into_dict()
    assert d["player1_x"] == [3.0] and d["player2_y"] == [5.0] and d["player3_x"] == [None]


# ---- display list == whole-frame cv2 -----------------------------------------------------------------------------
class _Stub:
    """A tracker as the drawing pass sees it: results, draw_kwargs(), object()."""

    def __init__(self, name, obj, preds, kwargs=None):
        self.name, self.obj, self.kwargs = name, obj, kwargs or {}
        self.results = preds

    def object(self):
        return self.obj

    def draw_kwargs(self):
        return self.kwargs

    def __str__(self):
        return self.name


def _court_keypoints(W, H, rng, jitter):
    base = np.array([[0.29, 0.91], [0.71, 0.91], [0.32, 0.76], [0.5, 0.76], [0.68, 0.76], [0.35, 0.56], [0.65, 0.56],
                     [0.38, 0.41], [0.5, 0.41], [0.62, 0.41], [0.4, 0.31], [0.6, 0.31]]) * [W, H]
    return base + rng.normal(0, jitter, base.shape)


def _border_results(W, H, T, seed, fixed_keypoints):
    """T frames of results whose boxes, labels, skeletons, court keypoints and balls straddle all four borders and
    overlap each other."""
    rng = np.random.default_rng(seed)
    players, poses, courts, balls = [], [], [], []
    fixed = Keypoints([Keypoint(i, tuple(xy)) for i, xy in enumerate(_court_keypoints(W, H, rng, 0).tolist())])
    anchors = [(-15, -12), (W - 40, -8), (-30, H - 60), (W - 50, H - 30), (W // 2, 3), (5, H // 2),
               (W - 3, H // 3), (W // 3, H - 2)]
    for t in range(T):
        xyxy, ids = [], []
        for k in range(5):
            ax, ay = anchors[(t + k) % len(anchors)]
            ax, ay = ax + int(rng.integers(-6, 7)), ay + int(rng.integers(-6, 7))
            w, h = int(rng.integers(30, 160)), int(rng.integers(60, 260))
            x1 = ax - w // 2 if ax > W // 2 else ax
            y1 = ay - h // 2 if ay > H // 2 else ay
            xyxy.append([x1, y1, x1 + w, y1 + h])
            ids.append(1 + (t + k) % 6)  # ids 5 and 6 too: drawn, not collected
        xyxy = np.array(xyxy, np.float32) + rng.random((5, 4)).astype(np.float32)
        players.append(Players.from_rows(xyxy, np.array(ids), np.zeros(5, int), rng.random(5).astype(np.float32)))
        pose = np.stack([xyxy[:, :2] + rng.random((5, 13, 2)).transpose(1, 0, 2) * (xyxy[:, 2:] - xyxy[:, :2])
                         for _ in range(1)])[0].transpose(1, 0, 2).astype(np.float64)
        poses.append(PlayersKeypoints.from_xy(pose))
        if fixed_keypoints:
            courts.append(fixed)
        elif t % 4 == 2:
            courts.append(Keypoints([]))  # no keypoints on this frame: homography None
        else:
            xy = _court_keypoints(W, H, rng, 3.0)
            xy[t % 12] = [(W - 2, 2), (1, 3), (W + 3, H - 1), (2, H + 2)][t % 4]  # a keypoint on a corner
            courts.append(Keypoints([Keypoint(i, tuple(v)) for i, v in enumerate(xy.tolist())]))
        bx, by = [(-4, H // 2), (W + 3, 40), (W // 2, -5), (100, H + 4), (W - 1, H - 1), (0, 0)][t % 6]
        balls.append(Ball(frame=t, xy=(float(bx), float(by)), visibility=1))
    vi = sv.VideoInfo(width=W, height=H, fps=25.0, total_frames=T)
    trackers = {"players_tracker": _Stub("players_tracker", Players, players,
                                         {"video_info": vi, "annotator": "rectangle_bounding_box",
                                          "show_confidence": True}),
                "players_keypoints_tracker": _Stub("players_keypoints_tracker", PlayersKeypoints, poses),
                "keypoints_tracker": _Stub("keypoints_tracker", Keypoints, courts),
                "ball_tracker": _Stub("ball_tracker", Ball, balls)}
    return trackers, vi


def _rally_frame(W, H):
    f = cv2.imread(str(GOLDEN / "rally" / "rally_f00_720p.jpg"))
    return f if f.shape[:2] == (H, W) else cv2.resize(f, (W, H), interpolation=cv2.INTER_LINEAR)


@pytest.mark.parametrize("W,H", [(1920, 1080), (1280, 720)])
@pytest.mark.parametrize("fixed", [True, False])
def test_display_list_equals_whole_frame_cv2_across_borders(W, H, fixed):
    T = 8
    trackers, vi = _border_results(W, H, T, seed=W + fixed, fixed_keypoints=fixed)
    frame = _rally_frame(W, H)
    court_ref, court_dev = ProjectedCourt(vi), ProjectedCourt(vi)
    da_ref, da_dev = DataAnalytics(), DataAnalytics()
    builder = DisplayListBuilder((H, W), court_dev)
    per_frame = [builder.frame_records(i, trackers, da_dev, fixed) for i in range(T)]
    recs, offsets, atlas = pack_display_list(per_frame)
    assert (recs["op"] == L.OVERLAY_BLEND).sum() == T
    # every border is crossed by some stamp
    x1, y1 = recs["x0"] + recs["w"], recs["y0"] + recs["h"]
    assert (recs["x0"] == 0).any() and (recs["y0"] == 0).any() and (x1 == W).any() and (y1 == H).any()
    got = composite_numpy(np.repeat(frame[None], T, 0), recs, offsets, atlas, court_dev.blend_lut())
    for i in range(T):
        exp = render_frame_cpu(frame, i, trackers, court_ref, da_ref, fixed)
        if not np.array_equal(got[i], exp):
            ys, xs = np.nonzero((got[i] != exp).any(-1))
            raise AssertionError(f"frame {i}: {len(ys)} pixels differ, e.g. at (x, y) = {list(zip(xs, ys))[:8]}")
    assert da_ref.into_dict() == da_dev.into_dict()
    assert any(v is not None for v in da_dev.into_dict()["player1_x"]), "vacuous: no projected player"


def test_record_draw_calls_sees_each_cv2_call_and_restores_cv2():
    circle = cv2.circle
    p = Player.from_row(np.array([10, 20, 50, 90], np.float32), 3, 0, 0.5)
    calls = record_draw_calls(p.draw, video_info=None)
    assert [c[0] for c in calls] == ["rectangle", "putText"]
    assert calls[0][1]["pt1"] == (10, 20) and calls[1][1]["text"] == "3 0.50"
    p.projection = (100, 100)
    assert [c[0] for c in record_draw_calls(p.draw_projection)] == ["circle", "putText"]
    assert cv2.circle is circle
