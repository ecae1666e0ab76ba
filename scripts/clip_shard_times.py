"""Frames/s of tracking AND rendering a list of clips with `TrackingRunner.run_clips(..., inference_dir=...,
collect_data=True)` sharded over 1, 2 and 4 ranks of a torch.distributed job.

Workload: the clips of `clip_render_times.py` (`--clips` synthetic 1080p clips of 100..330 frames, seeded lengths,
views into one pool of distinct frames held on each rank's device, so decode is left out), all four trackers (seeded
checkpoints, InpaintNet loaded), batch 32 for tracking and rendering, each clip's background from its own frames.  A
world size of 1 is one process without a process group; larger ones are `torch.distributed.run` launches.  Ranks
share one card over gloo when there are fewer GPUs than ranks, and each has its own GPU over NCCL otherwise.  The
world sizes alternate over the rounds.  Each launch warms up on one short clip per rank, then times one run_clips
call over every clip between two barriers (process start-up and engine set-up are outside the timed region).

Prints one JSON line: frames/s per world size and round, the per-rank split of each world size's last round
(seconds: tracking pass, display-list build, encode, exchange, ...), peak device memory per rank (torch allocator,
reserved and allocated; each process's CUDA context comes on top), os.cpu_count(), and the card's name and power
limit.  Every launch gets os.cpu_count() / world OpenMP threads per rank.  A world size that fails is reported under
"failed" and not run again: each rank takes about 21 GiB of device memory at batch 32, so four ranks do not fit on
one 80 GB card.

    python scripts/clip_shard_times.py --ranks 1,2,4 --rounds 2    # a box with 4 GPUs or more
    python scripts/clip_shard_times.py --ranks 1,2,3 --rounds 2    # one 80 GB card
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import timeit
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = ((r.stdout.strip().splitlines() or [", , "])[0].split(", ") + ["", ""])[:3]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def worker(a) -> None:
    """One rank (or the single process): warm up, then time run_clips over every clip; write this rank's record."""
    sys.path.insert(0, str(ROOT))
    import numpy as np
    import torch
    import torch.distributed as dist

    from oracle import inpaint as OI
    from oracle import weights as OW
    from padel_analytics_b200 import synth
    from padel_analytics_b200.trackers import (BallTracker, KeypointsTracker, PlayerKeypointsTracker, PlayerTracker,
                                               TrackingRunner)
    from padel_analytics_b200.trackers import sv_compat as sv

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    ngpu = torch.cuda.device_count()
    dev = torch.device("cuda", rank % ngpu)
    torch.cuda.set_device(dev)
    if world > 1:
        if ngpu >= world:
            dist.init_process_group("nccl", device_id=dev)
        else:
            dist.init_process_group("gloo")
    H, W, B, fps = 1080, 1920, a.batch, 30.0
    rng = np.random.default_rng(0)  # the clips of clip_render_times.py
    lengths = [int(v) for v in rng.integers(a.min_len, a.max_len + 1, size=a.clips)]
    # the frames of clip_render_times.py's pool, made on the device 16 at a time: make_frames' int64 temporaries for
    # the whole pool take tens of GB, once per rank
    n = a.max_len + 64
    pool = torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev)
    for i in range(0, n, 16):
        pool[i:i + 16] = synth.make_frames(min(16, n - i), H, W, start=5 + i, device=dev)
    torch.cuda.empty_cache()
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
    run = TrackingRunner(tr, video_info=sv.VideoInfo(width=W, height=H, fps=fps))
    run.render_batch_size = B
    short = int(np.argmin(lengths))
    with tempfile.TemporaryDirectory() as td:
        run.run_clips([(source(short), lengths[short])] * world, inference_dir=td, collect_data=True)  # warm-up
        run.timings.clear()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        if world > 1:
            dist.barrier()
        t0 = timeit.default_timer()
        run.run_clips([(source(c), lengths[c]) for c in range(a.clips)], inference_dir=td, collect_data=True)
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        seconds = timeit.default_timer() - t0
    rec = {"rank": rank, "seconds": seconds, "frames": sum(lengths),
           "split_s": {k: round(v, 3) for k, v in run.timings.items() if k.startswith("_clips")},
           "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "peak_reserved_gib": round(torch.cuda.max_memory_reserved() / 2 ** 30, 2)}
    with open(os.path.join(a.out, f"rank{rank}.json"), "w") as f:
        json.dump(rec, f)
    if world > 1:
        dist.destroy_process_group()


def launch(a, world: int, out: str, port: int) -> list[dict]:
    args = [str(Path(__file__).resolve()), "--worker", "--out", out, "--clips", str(a.clips), "--batch", str(a.batch),
            "--min-len", str(a.min_len), "--max-len", str(a.max_len)]
    if world == 1:
        cmd = [sys.executable] + args
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
               "--master-addr", "127.0.0.1", "--master-port", str(port)] + args
    # torchrun would give every rank one OpenMP thread; every world size gets an equal share of the host instead
    env = dict(os.environ, OMP_NUM_THREADS=str(max(1, (os.cpu_count() or 1) // world)))
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if r.returncode:
        raise RuntimeError(f"world size {world} failed:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    recs = []
    for rank in range(world):
        with open(os.path.join(out, f"rank{rank}.json")) as f:
            recs.append(json.load(f))
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", default="1,2,4")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--min-len", type=int, default=100)
    ap.add_argument("--max-len", type=int, default=330)
    ap.add_argument("--port", type=int, default=29651)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a)
        return
    import torch

    assert torch.cuda.is_available(), "clip_shard_times needs a GPU"
    worlds = [int(v) for v in a.ranks.split(",")]
    ngpu = torch.cuda.device_count()
    fps = {str(w): [] for w in worlds}
    split, peak, failed = {}, {}, {}
    frames = None
    print(json.dumps({"gpus": ngpu, "cpu_count": os.cpu_count(), **card()}), file=sys.stderr, flush=True)
    for r in range(a.rounds):
        order = worlds if r % 2 == 0 else worlds[::-1]
        for w in order:
            if str(w) in failed:
                continue
            try:
                with tempfile.TemporaryDirectory() as td:
                    recs = launch(a, w, td, a.port + r * 16 + w)
            except RuntimeError as e:  # e.g. too many ranks for one card's memory: reported, not retried
                lines = [ln for ln in str(e).splitlines() if "Error" in ln]
                failed[str(w)] = (lines[-1] if lines else str(e).splitlines()[0])[-400:]
                print(f"round {r} world {w}: failed", file=sys.stderr, flush=True)
                continue
            frames = recs[0]["frames"]
            fps[str(w)].append(round(frames / recs[0]["seconds"], 1))
            split[str(w)] = [rec["split_s"] for rec in recs]
            peak[str(w)] = [{"reserved": rec["peak_reserved_gib"], "allocated": rec["peak_allocated_gib"]}
                            for rec in recs]
            print(f"round {r} world {w}: {fps[str(w)][-1]} frames/s", file=sys.stderr, flush=True)
    print(json.dumps({"metric": "clip_list_track_and_render_1080p_sharded", "clips": a.clips, "frames": frames,
                      "batch": a.batch, "gpus": ngpu,
                      "backend": {str(w): "nccl" if 1 < w <= ngpu else ("gloo, shared card" if w > 1 else "none")
                                  for w in worlds},
                      "frames_per_s": fps, "per_rank_split_s": split, "peak_device_memory_gib": peak, "failed": failed,
                      "cpu_count": os.cpu_count(), **card()}))


if __name__ == "__main__":
    main()
