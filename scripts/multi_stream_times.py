"""Frames/s and pull-to-yield latency of `TrackingRunner.stream_many` over S live streams at several batch sizes.

Workload: S synthetic 1080p streams of `--frames` frames each (a pool of `--pool` distinct frames, cycled, each
stream starting at another frame of the pool), pulled round-robin one host HWC uint8 frame at a time, as S cameras
hand them over, through all four trackers (seeded checkpoints, InpaintNet loaded, the backgrounds given).  Per batch
size the trackers are built at that batch and warmed up on a short run; each S is then timed once, with Python's cyclic
garbage collector switched off around the loop (as `run()` does for its pass).  Latency of an entry: from the pass
pulling the frame to the generator yielding its entry.  Frames/s counts every stream's frames, InpaintNet at each
stream's end included; per stream it is the aggregate over S.

Baseline (--baseline S ...): S independent `stream()` generators at batch 1, each with its own tracker set, stepped
round-robin in one process (the next entry of each in turn; each pulls its frames as it needs them).

Prints one JSON line with the card's name, power limit and max SM clock.

    python scripts/multi_stream_times.py --frames 128 --streams 1 2 4 8 16 --batches 4 8 16 --baseline 1 2 4
"""
from __future__ import annotations

import argparse
import gc
import json
import subprocess
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

H, W = 1080, 1920


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = ((r.stdout.strip().splitlines() or [", , "])[0].split(", ") + ["", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def trackers(ck, B: int, vi):
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    tr = [PlayerTracker(ck["detect"], poly, batch_size=B),
          PlayerKeypointsTracker(ck["pose13"], 1280, batch_size=B, load_path=None, save_path=None),
          KeypointsTracker(ck["court12"], batch_size=B, model_type="yolo"),
          BallTracker(ck["tracknet"], ck["inpaint"], batch_size=B)]
    for t in tr:
        t.video_info_post_init(vi)
    return tr


def summary(n: int, seconds: float, S: int, lat: np.ndarray) -> dict:
    return {"frames_per_s": round(n / seconds, 1), "per_stream_frames_per_s": round(n / seconds / S, 1),
            "latency_ms_p50": round(float(np.median(lat)), 2), "latency_ms_max": round(float(lat.max()), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=128, help="frames per stream")
    ap.add_argument("--pool", type=int, default=64)
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 2, 4, 8, 16])
    ap.add_argument("--batches", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--baseline", type=int, nargs="*", default=[1, 2, 4])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_stream_times.py measures on a CUDA device, and none is visible")
    pool = [f.numpy() for f in synth.make_frames(a.pool, H, W, start=5)]
    med = synth.make_median(H, W).numpy()
    ck = {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
          "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}
    vi = sv.VideoInfo(width=W, height=H, fps=30.0)
    out = {"frames_per_stream": a.frames, "resolution": f"{W}x{H}", "source": "host frames, round-robin, one per pull",
           **card(), "stream_many": {}, "baseline_stream_b1": {}}
    for B in a.batches:
        tr = trackers(ck, B, vi)

        def run(S: int, n: int):
            for t in tr:
                t.restart()
            pulled, yielded = {}, {}

            def source():
                for f in range(n):
                    for s in range(S):
                        pulled[(s, f)] = timeit.default_timer()
                        yield s, pool[(f + 7 * s) % len(pool)]

            gc.collect()
            gc.disable()
            try:
                t0 = timeit.default_timer()
                for key, f, _ in TrackingRunner(tr, video_info=vi).stream_many(
                        source(), medians={s: med for s in range(S)}, max_open=max(a.streams)):
                    yielded[(key, f)] = timeit.default_timer()
                torch.cuda.synchronize()
                t1 = timeit.default_timer()
            finally:
                gc.enable()
            lat = np.array([yielded[k] - pulled[k] for k in pulled]) * 1e3
            return summary(S * n, t1 - t0, S, lat)

        run(2, 2 * B + 16)  # warm-up: engines, plans, pinned buffers
        out["stream_many"][B] = {S: run(S, a.frames) for S in a.streams}
        del tr
        torch.cuda.empty_cache()
    for S in a.baseline:
        sets = [trackers(ck, 1, vi) for _ in range(S)]

        def one(S: int, n: int):
            for tr in sets[:S]:
                for t in tr:
                    t.restart()
            pulled, yielded = {}, {}
            feeds = [iter(_Feed(n, s, pulled, pool)) for s in range(S)]
            gens = [TrackingRunner(sets[s], video_info=vi).stream(feeds[s], median=med) for s in range(S)]
            gc.collect()
            gc.disable()
            try:
                t0 = timeit.default_timer()
                live = list(range(S))
                while live:
                    for s in list(live):
                        got = next(gens[s], None)
                        if got is None:
                            live.remove(s)
                        else:
                            yielded[(s, got[0])] = timeit.default_timer()
                torch.cuda.synchronize()
                t1 = timeit.default_timer()
            finally:
                gc.enable()
            lat = np.array([yielded[k] - pulled[k] for k in pulled]) * 1e3
            return summary(S * n, t1 - t0, S, lat)

        one(1, 24)  # warm-up
        out["baseline_stream_b1"][S] = one(S, a.frames)
        del sets
        torch.cuda.empty_cache()
    print(json.dumps(out))


class _Feed:
    """Stream s's frames for `stream()`, stamping each pull."""

    def __init__(self, n: int, s: int, pulled: dict, pool: list):
        self.n, self.s, self.pulled, self.pool = n, s, pulled, pool

    def __iter__(self):
        for f in range(self.n):
            self.pulled[(self.s, f)] = timeit.default_timer()
            yield self.pool[(f + 7 * self.s) % len(self.pool)]


if __name__ == "__main__":
    main()
