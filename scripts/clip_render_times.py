"""Frames/s of tracking AND rendering a list of clips: a Python loop of per-clip
TrackingRunner(..., inference_path=..., collect_data=True).run() against one
TrackingRunner.run_clips(..., inference_dir=..., collect_data=True) call, alternated in one session on the same trackers.

Workload: `--clips` synthetic 1080p clips of 100..330 frames (seeded lengths), all four trackers (seeded checkpoints,
InpaintNet loaded), batch 32 for tracking and rendering, each clip's background computed from its own frames.  The
clips are views into one pool of distinct frames held on the device, so decode is left out of both arms; the videos
go to a temporary directory.  Prints one JSON line: frames/s per arm and round, the render split of each arm's last
round (seconds, summed over clips for the loop), and the card's name and power limit.

    python scripts/clip_render_times.py --clips 16 --rounds 2
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
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


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = ((r.stdout.strip().splitlines() or [", , "])[0].split(", ") + ["", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--min-len", type=int, default=100)
    ap.add_argument("--max-len", type=int, default=330)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "clip_render_times needs a GPU"
    H, W, B, fps = 1080, 1920, a.batch, 30.0
    rng = np.random.default_rng(0)
    lengths = [int(v) for v in rng.integers(a.min_len, a.max_len + 1, size=a.clips)]
    pool = synth.make_frames(a.max_len + 64, H, W, start=5).cuda()
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
        t.video_info_post_init(sv.VideoInfo(width=W, height=H, fps=fps))

    def per_clip(clips, out):
        split = {}
        for c in clips:
            for t in tr:
                t.restart()
            run = TrackingRunner(tr, video_info=sv.VideoInfo(width=W, height=H, fps=fps, total_frames=lengths[c]),
                                 inference_path=str(out / f"{c:04d}.mp4"), collect_data=True)
            run.render_batch_size = B
            run.run(frame_source=source(c), total_frames=lengths[c])
            for k, v in run.timings.items():
                if k.startswith("_render") or k == "_fused_pass":
                    split[k] = split.get(k, 0.0) + v
        return split

    def packed(clips, out):
        for t in tr:
            t.restart()
        run = TrackingRunner(tr, video_info=sv.VideoInfo(width=W, height=H, fps=fps))
        run.render_batch_size = B
        run.run_clips([(source(c), lengths[c]) for c in clips], inference_dir=str(out), collect_data=True)
        return {k: v for k, v in run.timings.items() if k.startswith("_clips")}

    total = sum(lengths)
    print(json.dumps({"frames": total, **card()}), file=sys.stderr, flush=True)
    res = {"per_clip_run": [], "run_clips": []}
    split = {}
    with tempfile.TemporaryDirectory() as td:
        out = Path(td)
        short = [int(np.argmin(lengths))]
        per_clip(short, out)  # warm-up: plans, caches, pinned buffers, the encoder
        packed(short, out)
        for r in range(a.rounds):
            for name, fn in (("per_clip_run", per_clip), ("run_clips", packed)):
                torch.cuda.synchronize()
                t0 = timeit.default_timer()
                split[name] = fn(range(a.clips), out)
                torch.cuda.synchronize()
                res[name].append(round(total / (timeit.default_timer() - t0), 1))
                print(f"round {r} {name}: {res[name][-1]} frames/s", file=sys.stderr, flush=True)
    print(json.dumps({"metric": "clip_list_track_and_render_1080p", "clips": a.clips, "frames": total, "batch": B,
                      "frames_per_s": res,
                      "render_split_s": {n: {k: round(v, 3) for k, v in s.items()} for n, s in split.items()},
                      **card()}))


if __name__ == "__main__":
    main()
