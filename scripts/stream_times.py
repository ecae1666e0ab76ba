"""Frames/s and per-frame latency of `TrackingRunner.stream` at several batch sizes.

Workload: `--frames` synthetic 1080p frames (a pool of `--pool` distinct frames, cycled) pulled one at a time as
host HWC uint8 arrays, as a live source hands them over, through all four trackers (seeded checkpoints, InpaintNet
loaded, the background given).  Per batch size the trackers are built at that batch, warmed up on a short stream, and
two streams are timed: one with Python's cyclic garbage collector on (the default) and one with it switched off
around the loop (`gc.disable()`, as `run()` does for its pass).  Latency of frame f: from the pass pulling frame f to
the stream yielding its entry.  Frames/s counts the whole stream, InpaintNet at its end included.  Prints one JSON
line with the card's name, power limit and max SM clock.

    python scripts/stream_times.py --frames 1024 --batches 1 4 8 32
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


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = ((r.stdout.strip().splitlines() or [", , "])[0].split(", ") + ["", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--pool", type=int, default=128)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4, 8, 32])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_times.py measures on a CUDA device, and none is visible")
    H, W = 1080, 1920
    pool = [f.numpy() for f in synth.make_frames(a.pool, H, W, start=5)]
    med = synth.make_median(H, W).numpy()
    ck = {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
          "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    vi = sv.VideoInfo(width=W, height=H, fps=30.0)
    out = {"frames": a.frames, "resolution": f"{W}x{H}", "source": "host frames, one per pull", **card(),
           "batches": {}}
    for B in a.batches:
        tr = [PlayerTracker(ck["detect"], poly, batch_size=B),
              PlayerKeypointsTracker(ck["pose13"], 1280, batch_size=B, load_path=None, save_path=None),
              KeypointsTracker(ck["court12"], batch_size=B, model_type="yolo"),
              BallTracker(ck["tracknet"], ck["inpaint"], batch_size=B)]
        for t in tr:
            t.video_info_post_init(vi)

        def run(n, collector=True):
            for t in tr:
                t.restart()
            pulled = np.zeros(n)
            yielded = np.zeros(n)

            def source():
                for f in range(n):
                    pulled[f] = timeit.default_timer()
                    yield pool[f % len(pool)]

            gc.collect()
            if not collector:
                gc.disable()
            try:
                t0 = timeit.default_timer()
                for f, _ in TrackingRunner(tr, video_info=vi).stream(source(), median=med):
                    yielded[f] = timeit.default_timer()
                torch.cuda.synchronize()
                t1 = timeit.default_timer()
            finally:
                gc.enable()
            return n / (t1 - t0), (yielded - pulled) * 1e3

        run(4 * B + 16)  # warm-up: engines, plans, pinned buffers
        out["batches"][B] = {}
        for name, collector in (("gc_on", True), ("gc_off", False)):
            fps, lat = run(a.frames, collector)
            out["batches"][B][name] = {"frames_per_s": round(fps, 1),
                                       "latency_ms_p50": round(float(np.median(lat)), 2),
                                       "latency_ms_max": round(float(lat.max()), 2)}
        del tr
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
