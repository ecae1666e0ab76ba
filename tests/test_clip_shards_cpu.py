"""run_clips over the ranks of a distributed job, without a GPU: the clip assignment (`plan_clip_shards`) over random
clip lists, and the exchange after the pass (status, results as dense arrays, DataAnalytics) over gloo with two
processes."""
import os
import subprocess
import sys
from pathlib import Path

import numpy as np

from padel_analytics_b200.trackers.runner import plan_clip_shards

ROOT = Path(__file__).resolve().parents[1]


def _greedy(lengths, world):
    """The rule restated: longest first (ties: lower clip), to the least loaded rank (ties: lower rank)."""
    load, shards = [0] * world, [[] for _ in range(world)]
    for c in sorted(range(len(lengths)), key=lambda c: (-lengths[c], c)):
        r = min(range(world), key=lambda r: (load[r], r))
        shards[r].append(c)
        load[r] += lengths[c]
    return [sorted(s) for s in shards]


def test_plan_clip_shards_random_lists():
    rng = np.random.default_rng(7)
    cases = 0
    for _ in range(300):
        n = int(rng.integers(0, 25))
        hi = int(rng.choice([1, 10, 400]))
        lengths = [int(v) for v in rng.integers(0, hi, size=n)]
        if n and rng.random() < 0.3:
            lengths[int(rng.integers(0, n))] = 0
        for world in range(1, 10):
            plan = plan_clip_shards(lengths, world)
            assert len(plan) == world
            assert sorted(c for s in plan for c in s) == list(range(n)), (lengths, world, plan)
            assert all(s == sorted(s) for s in plan)
            assert plan == plan_clip_shards(list(lengths), world) == _greedy(lengths, world)
            loads = [sum(lengths[c] for c in s) for s in plan]
            if n:
                assert max(loads) <= sum(lengths) / world + max(lengths), (lengths, world, loads)
            cases += 1
    assert cases == 2700


def test_plan_clip_shards_edges():
    assert plan_clip_shards([], 3) == [[], [], []]
    assert plan_clip_shards([0, 0, 0], 2) == [[0, 1, 2], []]  # 0-frame clips add no load: all to the lowest rank
    assert plan_clip_shards([5, 9], 4) == [[1], [0], [], []]
    assert plan_clip_shards([4, 4, 4, 4], 2) == [[0, 2], [1, 3]]
    assert plan_clip_shards([10, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1], 2) == [[0], list(range(1, 11))]
    assert plan_clip_shards([3, 1], 1) == [[0, 1]]


# ---- the exchange over gloo --------------------------------------------------------------------------------------
_COMMON = """
import sys, json
sys.path.insert(0, {root!r})
import numpy as np, torch.distributed as dist
from padel_analytics_b200.analytics import DataAnalytics
from padel_analytics_b200.trackers import runner as R
from padel_analytics_b200.trackers.ball_tracker import Ball
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from padel_analytics_b200.trackers.players_keypoints_tracker import PlayersKeypoints
from padel_analytics_b200.trackers.players_tracker import Player, Players
dist.init_process_group('gloo')
rank, world = dist.get_rank(), dist.get_world_size()
"""

_ROUND_TRIP = _COMMON + """
LENGTHS = [6, 0, 9, 1, 4, 7]
FIXED = Keypoints([Keypoint(i, (10 * i, 20 + i)) for i in range(12)])  # int coordinates


def players(g, n):
    k = int(g.integers(0, 5))
    xyxy = (g.random((k, 4)) * 1000).astype(np.float32)
    cls, conf = np.zeros(k, int), g.random(k).astype(np.float32)
    form = n % 3
    if form == 0:
        return Players.from_rows(xyxy, g.integers(1, 9, size=k), cls, conf)
    if form == 1:
        return Players.from_rows(xyxy, None, cls, conf)
    return Players([Player.from_row(xyxy[i], None if i % 2 else int(g.integers(1, 9)), 0, conf[i]) for i in range(k)])


def clip(c):
    g = np.random.default_rng(100 + c)
    T = LENGTHS[c]
    res = {{
        "players_tracker": [players(g, n) for n in range(T)],
        "players_keypoints_tracker": [PlayersKeypoints.from_xy(g.random((int(g.integers(0, 4)), 13, 2)) * 900)
                                      for n in range(T)],
        "keypoints_tracker": [Keypoints([Keypoint(id=[10, 11, 1, 0, 7, 9, 8, 5, 6, 2, 4, 3][i], xy=tuple(g.random(2) * 500))
                                         for i in range(12)] if n % 4 else []) for n in range(T)],
        "fixed_court": [FIXED] * T,
        "ball_tracker": [Ball(frame=n, xy=(int(g.integers(0, 1920)), int(g.integers(0, 1080))), visibility=1)
                         if n % 3 else Ball(frame=n, xy=(0.0, 0.0), visibility=0) for n in range(T)],
    }}
    if T > 2:
        res["ball_tracker"][2] = Ball(frame=2, xy=(0, 0), visibility=0)  # a (0, 0) int pair: stays int
    da = DataAnalytics()
    for n in range(T):
        for p in (1, 2, 3, 4):
            if g.random() < 0.7:
                da.add_player_position(p, (float(g.random() * 10), float(g.random() * 20)))
        da.step(1)
    da.frames = da.frames[:-1]
    return res, da


def ser(objs):
    return json.dumps([o.serialize() for o in objs])


plan = R.plan_clip_shards(LENGTHS, world)
mine = plan[rank]
assert all(plan), plan
orig = [clip(c) for c in range(len(LENGTHS))]
names = list(orig[0][0])
hw = R.exchange_clip_status(None, (1080, 1920) if any(LENGTHS[c] for c in mine) else None, mine[0])
assert hw == (1080, 1920), hw
own = {{c: dict(orig[c][0]) for c in mine}}
got = R.exchange_clip_results(own, LENGTHS, names, {{"fixed_court": FIXED}})
assert len(got) == len(LENGTHS)
for c, res in enumerate(got):
    assert list(res) == names, (c, list(res))
    for n in names:
        assert len(res[n]) == LENGTHS[c]
        assert ser(res[n]) == ser(orig[c][0][n]), (rank, c, n)
    if c not in mine:
        assert all(o is FIXED for o in res["fixed_court"])
        assert all(type(a) is type(b) for a, b in zip(res["players_tracker"], orig[c][0]["players_tracker"]))
    else:
        assert res is own[c]
das = R.exchange_clip_data(None, {{c: orig[c][1] for c in mine}})
assert len(das) == len(LENGTHS)
for c, da in enumerate(das):
    ref = orig[c][1]
    assert da.frames == ref.frames and len(da) == len(ref) == LENGTHS[c], c
    a, b = da.into_dataframe(30.0), ref.into_dataframe(30.0)
    assert list(a.columns) == list(b.columns)
    assert np.array_equal(a.to_numpy(np.float64), b.to_numpy(np.float64), equal_nan=True), c
    if c in mine:
        assert da is ref
print(f'ROUND_TRIP_OK {{rank}}', flush=True)
dist.destroy_process_group()
"""

_FAILURE = _COMMON + """
try:
    R.exchange_clip_status((3, "ValueError: clip 3 yielded 5 frames, 9 announced") if rank == 1 else None,
                           (1080, 1920), rank)
except ValueError as e:
    assert "rank 1, clip 3" in str(e) and "yielded 5 frames" in str(e), str(e)
    print(f'FAILED_ON_EVERY_RANK {{rank}}', flush=True)
try:
    R.exchange_clip_status(None, (1080, 1920) if rank == 0 else (720, 1280), 4 * rank + 1)
except ValueError as e:
    assert "same frame size" in str(e) and "clip 5" in str(e), str(e)
    print(f'SIZE_ON_EVERY_RANK {{rank}}', flush=True)
try:
    R.exchange_clip_data((None, "RuntimeError: encoder") if rank == 0 else None, {{}})
except ValueError as e:
    assert "rank 0: RuntimeError: encoder" in str(e), str(e)
    print(f'RENDER_ON_EVERY_RANK {{rank}}', flush=True)
dist.destroy_process_group()
"""


def _launch(tmp_path, name, body, port):
    script = tmp_path / name
    script.write_text(body.format(root=str(ROOT)))
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    return subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script)],
                          capture_output=True, text=True, env=env, timeout=240)


def test_exchange_round_trip_world2_gloo(tmp_path):
    """Two ranks over gloo, each sending only its own clips: every rank gets every clip's results serialising equal
    to the originals (players with ids, without, and with some; pose keypoints; detected court keypoints; fixed court
    keypoints, int coordinates, not sent; balls with int and float pairs; empty clips) and equal DataAnalytics."""
    r = _launch(tmp_path, "round_trip.py", _ROUND_TRIP, 29561)
    assert "ROUND_TRIP_OK 0" in r.stdout and "ROUND_TRIP_OK 1" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_exchange_failure_raises_on_every_rank_world2_gloo(tmp_path):
    """A failure on one rank (after the pass or after the render) and a frame-size mismatch between ranks raise
    ValueError on both ranks; neither is left waiting in a collective (the launch has a timeout)."""
    r = _launch(tmp_path, "failure.py", _FAILURE, 29563)
    for tag in ("FAILED_ON_EVERY_RANK", "SIZE_ON_EVERY_RANK", "RENDER_ON_EVERY_RANK"):
        for rank in (0, 1):
            assert f"{tag} {rank}" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
