"""Generate tests/golden/analytics_ref.npz by running the UNMODIFIED reference analytics package (only possible where
/root/reference exists).

    python tests/golden/make_analytics_golden.py

analytics_ref.npz — the reference's analytics package (ProjectedCourt.draw_projections_and_collect_data,
                DataAnalytics.step / into_dataframe(25)) on seeded court keypoints, players and balls: fixed keypoints,
                per-frame keypoints, and frames without keypoints (also the first ones).  The inputs are stored next to
                the results, so tests/test_render_cpu.py replays them without this script.
"""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))

from oracle import ref_harness  # noqa: E402

OUT = Path(__file__).resolve().parent


def analytics_inputs(seed: int, T: int, fixed: bool, missing_kp=(), W=1920, H=1080):
    """Seeded inputs of one analytics sequence: court keypoints (T,12,2) + present flags, player feet and ids
    (T,5,3) + counts, ball points (T,2)."""
    rng = np.random.default_rng(seed)
    # a court seen in perspective: 4 rows of keypoints (far base line ... near base line), ids ordered like k1..k12
    base = np.array([[560, 980], [1360, 980], [610, 820], [960, 820], [1310, 820], [680, 600], [1240, 600],
                     [730, 440], [960, 440], [1190, 440], [760, 330], [1160, 330]], np.float64)
    kp = np.repeat(base[None], T, 0)
    if not fixed:
        kp = kp + rng.normal(0, 2.0, kp.shape)
    present = np.ones(T, bool)
    present[list(missing_kp)] = False
    players = np.zeros((T, 5, 3), np.int64)
    counts = np.full(T, 4, np.int64)
    start = np.array([[700, 900], [1200, 900], [800, 420], [1100, 420]])
    for t in range(T):
        for p in range(4):
            players[t, p] = [start[p, 0] + 7 * t * (1 if p % 2 else -1) + rng.integers(-3, 4),
                             start[p, 1] + 5 * t * (1 if p < 2 else -1) // 2 + rng.integers(-3, 4), p + 1]
    counts[T // 3] = 3  # a frame where player 4 is missing
    players[T // 2, 4] = [960, 700, 5]  # a fifth id, dropped by the data collection
    counts[T // 2] = 5
    ball = np.stack([200 + 37 * np.arange(T), 300 + 11 * np.arange(T)], 1).astype(np.int64)
    return kp, present, players, counts, ball


ANALYTICS_SEQUENCES = {"fixed": dict(seed=1, T=14, fixed=True, missing_kp=()),
                       "per_frame": dict(seed=2, T=16, fixed=False, missing_kp=(5, 6, 11)),
                       "first_missing": dict(seed=3, T=12, fixed=False, missing_kp=(0, 1, 7))}


def analytics_golden():
    """The reference's own analytics package (ProjectedCourt.draw_projections_and_collect_data, DataAnalytics) over
    the sequences of ANALYTICS_SEQUENCES -> tests/golden/analytics_ref.npz: the homography after every frame (NaN
    when None), the projected players and ball, and into_dataframe(25)."""
    ref_harness.import_reference()
    from trackers.keypoints_tracker.keypoints_tracker import Keypoint, Keypoints
    from analytics import DataAnalytics, ProjectedCourt

    W, H = 1920, 1080
    out = {}
    for name, kw in ANALYTICS_SEQUENCES.items():
        kp, present, players, counts, ball = analytics_inputs(**kw, W=W, H=H)
        T = kw["T"]
        court = ProjectedCourt(SimpleNamespace(width=W, height=H))
        da = DataAnalytics()
        frame = np.zeros((H, W, 3), np.uint8)
        Hs = np.full((T, 3, 3), np.nan)
        proj_p = np.full((T, 5, 2), -1, np.int64)
        proj_b = np.full((T, 2), -1, np.int64)
        fixed_kps = Keypoints([Keypoint(id=i, xy=tuple(float(v) for v in kp[0, i])) for i in range(12)])
        for t in range(T):
            if kw["fixed"]:
                kps = fixed_kps
            else:
                kps = Keypoints([Keypoint(id=i, xy=tuple(float(v) for v in kp[t, i])) for i in range(12)]
                                if present[t] else [])
            pls = [SimpleNamespace(feet=(int(x), int(y)), id=int(i), projection=None,
                                   draw_projection=lambda f: f) for x, y, i in players[t, :counts[t]]]
            bl = SimpleNamespace(asint=(lambda b=ball[t]: (int(b[0]), int(b[1]))), projection=None,
                                 draw_projection=lambda f: f)
            court.draw_projections_and_collect_data(frame, keypoints_detection=kps, players_detection=pls,
                                                    ball_detection=bl, data_analytics=da,
                                                    is_fixed_keypoints=kw["fixed"])
            da.step(1)
            if court.H is not None:
                Hs[t] = court.H
                for j, p in enumerate(pls):
                    proj_p[t, j] = p.projection
                proj_b[t] = bl.projection
        da.frames = da.frames[:-1]
        df = da.into_dataframe(25)
        for k, v in zip(("kp", "kp_present", "players", "counts", "ball"), (kp, present, players, counts, ball)):
            out[f"{name}_in_{k}"] = v
        out[f"{name}_H"] = Hs
        out[f"{name}_proj_players"] = proj_p
        out[f"{name}_proj_ball"] = proj_b
        out[f"{name}_columns"] = np.array(list(df.columns))
        out[f"{name}_table"] = df.to_numpy(dtype=np.float64)
        out[f"{name}_frames"] = np.array(da.frames)
        print(f"analytics_ref {name}: H set on {int(np.isfinite(Hs[:, 0, 0]).sum())}/{T} frames, table {df.shape}")
    np.savez_compressed(OUT / "analytics_ref.npz", **out)


if __name__ == "__main__":
    analytics_golden()
