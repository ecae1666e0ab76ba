"""Frames/s of a list of clips: a Python loop of TrackingRunner(...).run() per clip against one
TrackingRunner.run_clips() call, alternated in one session on the same trackers.

Workload: `--clips` synthetic 1080p clips of 100..330 frames (seeded lengths), all four trackers (seeded checkpoints,
InpaintNet loaded), batch 32, each clip's background computed from its own frames.  The clips are views into one pool
of distinct frames, held either on the device or in pinned host memory (`--where`), so only decode is left out.

    python scripts/clip_times.py --clips 48 --rounds 2 --where device
"""
from __future__ import annotations

import argparse
import json
import sys
import timeit
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from oracle import inpaint as OI  # noqa: E402
from oracle import weights as OW  # noqa: E402
from padel_analytics_b200 import synth  # noqa: E402
from padel_analytics_b200.trackers import (BallTracker, KeypointsTracker, PlayerKeypointsTracker,  # noqa: E402
                                           PlayerTracker, TrackingRunner)
from padel_analytics_b200.trackers import sv_compat as sv  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=48)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--where", choices=("device", "pinned"), default="device")
    ap.add_argument("--min-len", type=int, default=100)
    ap.add_argument("--max-len", type=int, default=330)
    a = ap.parse_args()
    H, W, B = 1080, 1920, a.batch
    rng = np.random.default_rng(0)
    lengths = [int(v) for v in rng.integers(a.min_len, a.max_len + 1, size=a.clips)]
    pool = synth.make_frames(a.max_len + 64, H, W, start=5)
    pool = pool.cuda() if a.where == "device" else pool.pin_memory()
    offs = [int(v) for v in rng.integers(0, 64, size=a.clips)]

    def source(c):
        base = pool[offs[c]:offs[c] + lengths[c]]
        return lambda lo, hi: (base[i:min(hi, i + B)] for i in range(lo, hi, B))

    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    tr = [PlayerTracker(OW.make_yolo("detect"), poly, batch_size=B),
          PlayerKeypointsTracker(OW.make_yolo("pose13", cls_mean=-5.5), 1280, batch_size=B, load_path=None,
                                 save_path=None),
          KeypointsTracker(OW.make_yolo("court12"), batch_size=B, model_type="yolo"),
          BallTracker(OW.make_tracknet(), OI.make_inpaintnet(), batch_size=B)]
    for t in tr:
        t.video_info_post_init(sv.VideoInfo(width=W, height=H, fps=30.0))
    total = sum(lengths)

    def per_clip():
        for c, T in enumerate(lengths):
            for t in tr:
                t.restart()
            TrackingRunner(tr, video_info=sv.VideoInfo(width=W, height=H, fps=30.0, total_frames=T)).run(
                frame_source=source(c), total_frames=T)

    def packed():
        for t in tr:
            t.restart()
        TrackingRunner(tr, video_info=sv.VideoInfo(width=W, height=H, fps=30.0)).run_clips(
            [(source(c), T) for c, T in enumerate(lengths)])

    per_clip()  # warm-up: plans, caches, pinned buffers
    packed()
    res = {"per_clip_run": [], "run_clips": []}
    for _ in range(a.rounds):
        for name, fn in (("per_clip_run", per_clip), ("run_clips", packed)):
            torch.cuda.synchronize()
            t0 = timeit.default_timer()
            fn()
            torch.cuda.synchronize()
            res[name].append(round(total / (timeit.default_timer() - t0), 1))
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "clips": a.clips, "frames": total, "batch": B,
                      "where": a.where, "frames_per_s": res}))


if __name__ == "__main__":
    main()
