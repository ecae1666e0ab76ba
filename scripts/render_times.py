"""Render-pass throughput at 1080p: TrackingRunner.draw_and_collect_data() on N synthetic frames, split into decode,
display-list build, upload, pb_render_overlay, download (CUDA events) and encode (writer thread), next to the host
restatement of the reference's loop (decode, whole-frame cv2 drawing with the BGR<->RGB conversions, encode).

    python scripts/render_times.py [--frames 512] [--cpu-frames 128] [--out DIR]

The trackers run first (seeded checkpoints) on the same video; their time is not part of the numbers.  Prints one
JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import timeit
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines() or [", "])[0].split(", ")[:2]
    return {"gpu": name, "power_limit": power}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--cpu-frames", type=int, default=128)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", default=None, help="directory for the videos (default: a temporary one)")
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch

    from padel_analytics_b200 import synth
    from padel_analytics_b200.analytics import DataAnalytics, ProjectedCourt
    from padel_analytics_b200.render import render_frame_cpu
    from padel_analytics_b200.trackers import TrackingRunner
    from padel_analytics_b200.trackers import sv_compat as sv
    from test_trackers_gpu import H, W, _four_trackers

    assert torch.cuda.is_available(), "render_times needs a GPU"
    N, fps = args.frames, 25.0
    with tempfile.TemporaryDirectory() as td:
        out = Path(args.out or td)
        out.mkdir(parents=True, exist_ok=True)
        src_path = out / "source.mp4"
        vw = cv2.VideoWriter(str(src_path), cv2.VideoWriter_fourcc(*"mp4v"), fps, (W, H))
        for a in range(0, N, 32):
            for f in synth.make_frames(min(32, N - a), H, W, start=a, device="cuda").cpu().numpy():
                vw.write(f)
        vw.release()
        vi = sv.VideoInfo.from_video_path(str(src_path))
        assert vi.total_frames == N, vi
        tr = _four_trackers(args.batch, synth.make_median(H, W).numpy())
        run = TrackingRunner(tr, video_path=str(src_path), video_info=vi)
        run.render_batch_size = args.batch
        run.run()  # inference only: no inference_path, no data collection
        # device render pass (twice: the first warms up cv2's writer and the allocations)
        res = {}
        for rep in range(2):
            run.inference_path = str(out / "results.mp4")
            run.data_analytics = DataAnalytics()
            run.timings = {}
            torch.cuda.synchronize()
            t0 = timeit.default_timer()
            run.draw_and_collect_data()
            wall = timeit.default_timer() - t0
            res = {k[len("_render_"):]: round(v, 4) for k, v in run.timings.items() if k.startswith("_render_")}
            res["wall_s"] = round(wall, 4)
            res["frames_per_s"] = round(N / wall, 1)
        cap = cv2.VideoCapture(str(out / "results.mp4"))
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == N
        cap.release()
        # host restatement of the reference's loop over the first cpu_frames frames
        M = min(args.cpu_frames, N)
        court, da = ProjectedCourt(vi), DataAnalytics()
        vw = cv2.VideoWriter(str(out / "results_cpu.mp4"), cv2.VideoWriter_fourcc(*"mp4v"), fps, (W, H))
        t_dec = t_draw = t_enc = 0.0
        t0 = timeit.default_timer()
        for i, f in enumerate(sv.get_video_frames_generator(str(src_path), end=M)):
            t1 = timeit.default_timer()
            img = render_frame_cpu(f, i, run.trackers, court, da, run.is_fixed_keypoints)
            t2 = timeit.default_timer()
            vw.write(img)
            t3 = timeit.default_timer()
            t_dec += t1 - t0
            t_draw += t2 - t1
            t_enc += t3 - t2
            t0 = t3
        vw.release()
        cpu = {"frames": M, "decode_s": round(t_dec, 4), "draw_s": round(t_draw, 4), "encode_s": round(t_enc, 4),
               "frames_per_s": round(M / (t_dec + t_draw + t_enc), 1)}
    print(json.dumps({"metric": "render_pass_1080p", "frames": N, "batch": args.batch, "device_pass": res,
                      "cpu_restatement": cpu, **card()}))


if __name__ == "__main__":
    main()
