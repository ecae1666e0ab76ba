"""GPU: `TrackingRunner.run_clips` sharded over the ranks of a torch.distributed job against the single-process call on
the same clips: what every rank returns, which rank reads which clip, every video, JSON and CSV file, and the
DataAnalytics; and the errors every rank raises when one rank fails or two ranks see different frame sizes."""
import os
import pickle
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from padel_analytics_b200 import synth
from padel_analytics_b200.trackers import TrackingRunner
from padel_analytics_b200.trackers.runner import plan_clip_shards
from test_clip_render_gpu import _data, _decoded
from test_clips_gpu import LENGTHS as CLIP_LENGTHS
from test_clips_gpu import H, W, _ser, _trackers, _vi

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
LENGTHS = CLIP_LENGTHS + [0]
B = 32


def _ckpts():
    from oracle import inpaint as OI
    from oracle import weights as OW

    return {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
            "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}


def make_runner(ckpts):
    """All four trackers, InpaintNet, each clip's background from its own first 50 frames."""
    tr = _trackers(B, None, ckpts, median_max_sample_num=50)
    for t in tr:
        t.video_info_post_init(_vi(None))
    return TrackingRunner(tr, video_info=_vi(None))


def clip_sources(calls, lengths=LENGTHS, hw=(H, W), short=None):
    """(frame_source, total_frames) per clip, host frames made on the clip's first read; calls[clip] counts the
    reads.  short = (clip, n): that clip yields only its first n frames."""
    made = {}

    def source(c):
        def read(lo, hi):
            calls[c] += 1
            if c not in made:
                made[c] = [f.numpy() for f in synth.make_frames(lengths[c], *hw, start=11 * c + 1)]
            frames = made[c][:short[1]] if short and short[0] == c else made[c]
            return iter(frames[lo:hi])
        return read

    return [(source(c), T) for c, T in enumerate(lengths)]


def record(runner, got, calls) -> dict:
    return {"results": [{n: _ser(objs) for n, objs in res.items()} for res in got], "calls": list(calls),
            "timings": sorted(runner.timings), "data": [_data(da) for da in runner.clips_data_analytics]}


_SCRIPT = """
import os, pickle, sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import torch, torch.distributed as dist
if {backend!r} == "nccl":
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
else:
    dist.init_process_group("gloo")  # every rank on cuda:0
rank = dist.get_rank()
from test_clip_shards_gpu import LENGTHS, clip_sources, make_runner, record
from padel_analytics_b200.trackers import TrackingRunner
runner = make_runner(torch.load({ckpts!r}, weights_only=False))
calls = [0] * len(LENGTHS)
got = runner.run_clips(clip_sources(calls), save_dir={save!r}, inference_dir={video!r}, collect_data=True)
with open(os.path.join({out!r}, f"rank{{rank}}.pkl"), "wb") as f:
    pickle.dump(record(runner, got, calls), f)
print(f"RUN_OK {{rank}}", flush=True)
court_ball = TrackingRunner(list(runner.trackers.values())[2:], video_info=runner.video_info)
a = clip_sources([0, 0], [9, 9])[0]
b = clip_sources([0, 0], [9, 9], hw=(720, 1280))[1]
try:  # one clip per rank (ranks 0 and 1): each rank sees one frame size
    court_ball.run_clips([a, b])
except ValueError as e:
    assert "same frame size" in str(e), str(e)
    print(f"SIZE_RAISED {{rank}}", flush=True)
try:  # clip 1 is on rank 1 and yields 6 of its 9 frames
    court_ball.run_clips(clip_sources([0, 0], [40, 9], short=(1, 6)), inference_dir={video!r} + "_short")
except ValueError as e:
    assert "rank 1, clip 1" in str(e) and "yielded 6 frames, 9 announced" in str(e), str(e)
    print(f"SHORT_RAISED {{rank}}", flush=True)
dist.destroy_process_group()
"""


@pytest.fixture(scope="module")
def single(tmp_path_factory):
    """The single-process call: its record, videos and saved files."""
    base = tmp_path_factory.mktemp("single")
    ckpts = _ckpts()
    torch.save(ckpts, base / "ckpts.pt")
    runner = make_runner(ckpts)
    calls = [0] * len(LENGTHS)
    got = runner.run_clips(clip_sources(calls), save_dir=str(base / "save"), inference_dir=str(base / "video"),
                           collect_data=True)
    rec = record(runner, got, calls)
    assert any('"visibility": 1' in r["ball_tracker"] for r in rec["results"]), "vacuous: no ball"
    assert any(r["players_tracker"].count('"id"') for r in rec["results"]), "vacuous: no players"
    del runner, got
    torch.cuda.empty_cache()
    return base, rec


@pytest.mark.parametrize("backend,world,port", [("gloo", 2, 29571), ("gloo", 3, 29573), ("nccl", 2, 29577)])
def test_sharded_run_clips_equals_single_process(single, backend, world, port, tmp_path):
    """Every rank returns the single-process list; each clip is read only by the rank the plan gives it, as often as
    the single-process call reads it; every mp4 decodes to the same frames and every JSON and CSV file is byte-equal;
    every rank's clips_data_analytics is equal.  Then a frame-size mismatch between ranks and a short source on
    one rank raise ValueError on every rank."""
    if backend == "nccl" and torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    base, ref = single
    script = tmp_path / "shards.py"
    script.write_text(_SCRIPT.format(root=str(ROOT), tests=str(ROOT / "tests"), backend=backend,
                                     ckpts=str(base / "ckpts.pt"), save=str(tmp_path / "save"),
                                     video=str(tmp_path / "video"), out=str(tmp_path)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)], capture_output=True,
                       text=True, env=env, timeout=900)
    log = r.stdout[-3000:] + r.stderr[-3000:]
    for tag in ("RUN_OK", "SIZE_RAISED", "SHORT_RAISED"):
        for rank in range(world):
            assert f"{tag} {rank}" in r.stdout, (tag, rank, log)
    plan = plan_clip_shards(LENGTHS, world)
    assert all(plan[r] for r in range(world)), plan
    for rank in range(world):
        with open(tmp_path / f"rank{rank}.pkl", "rb") as f:
            rec = pickle.load(f)
        assert rec["results"] == ref["results"], rank
        assert rec["calls"] == [ref["calls"][c] if c in plan[rank] else 0 for c in range(len(LENGTHS))], \
            (rank, rec["calls"], plan)
        assert {"_clips_pass", "_clips_exchange", "_clips_render"} <= set(rec["timings"]), rec["timings"]
        assert len(rec["data"]) == len(LENGTHS)
        for c, (got, exp) in enumerate(zip(rec["data"], ref["data"])):
            assert got["frames"] == exp["frames"] and got["columns"] == exp["columns"] and got["csv"] == exp["csv"]
            assert np.array_equal(got["table"], exp["table"], equal_nan=True), (rank, c)
    for c, T in enumerate(LENGTHS):
        name = f"{c:04d}.mp4"
        assert (tmp_path / "video" / name).exists() == (base / "video" / name).exists() == (T > 0), c
        if T:
            assert _decoded(tmp_path / "video" / name) == _decoded(base / "video" / name), c
    files = sorted(p.name for p in (base / "save").iterdir())
    assert files == sorted(p.name for p in (tmp_path / "save").iterdir())
    assert len(files) == 5 * len(LENGTHS)  # four trackers' JSON and the CSV per clip
    for name in files:
        assert (tmp_path / "save" / name).read_bytes() == (base / "save" / name).read_bytes(), name
