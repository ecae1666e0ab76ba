"""CPU: C-ABI surface, host-side tracker logic, sharding maths and the world-size-2 gloo path."""
import json
import math
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from padel_analytics_b200 import _lib as L
from padel_analytics_b200.trackers import runner as R
from padel_analytics_b200.trackers import sv_compat as sv
from padel_analytics_b200.trackers.ball_tracker import Ball
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from padel_analytics_b200.trackers.players_keypoints_tracker import PlayerKeypoint, PlayerKeypoints, PlayersKeypoints
from padel_analytics_b200.trackers.players_tracker import Player, Players
from padel_analytics_b200.trackers.tracker import Tracker, TrackingResults, sampler

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol():
    hdr = (ROOT / "include" / "padel_b200.h").read_text()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(pb_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(L.SIGNATURES), declared ^ set(L.SIGNATURES)
    lib = L.lib()  # loads and binds every symbol (AttributeError if one is missing)
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.pb_version() >= 100
    out = subprocess.run(["nm", "-D", str(L.LIB_PATH)], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (\S+)", out))
    assert declared == exported, declared ^ exported  # the product library exports the header's ABI and nothing else


def test_engines_fail_loudly_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from padel_analytics_b200.engine.tracknet_engine import TrackNetEngine
    from padel_analytics_b200.engine.yolo_engine import YoloEngine

    with pytest.raises(L.PbError):
        TrackNetEngine(None, 1)
    with pytest.raises(L.PbError):
        YoloEngine({"model": {}, "nc": 1, "kpt_shape": None}, 1)


def test_sampler_and_results():
    chunks = list(sampler(iter(range(7)), 3))
    assert chunks == [[0, 1, 2], [3, 4, 5], [6]]  # last partial chunk kept (tracker.py:307-312)
    r = TrackingResults()
    r.update([1, 2])
    r.update([3])
    assert len(r) == 3 and r.counter == 2 and r.sample_predictions == [3] and list(r) == [1, 2, 3]
    r.restart()
    assert len(r) == 0


def test_object_json_round_trips():
    b = Ball(frame=3, xy=(10, 20), visibility=1)
    rt = Ball.from_json(json.loads(json.dumps(b.serialize())))
    assert (rt.frame, tuple(rt.xy), rt.visibility, rt.projection) == (3, (10, 20), 1, None)
    k = Keypoints([Keypoint(id=2, xy=(1.5, 2.5)), Keypoint(id=0, xy=(3.0, 4.0))])
    assert [x["id"] for x in k.serialize()] == [0, 2]
    assert tuple(Keypoints.from_json(json.loads(json.dumps(k.serialize())))[2].xy) == (1.5, 2.5)
    pk = PlayersKeypoints([PlayerKeypoints([PlayerKeypoint(id=i, name=n, xy=(float(i), 1.0))
                                            for i, n in enumerate(PlayerKeypoints.KEYPOINTS_NAMES)])])
    rt = PlayersKeypoints.from_json(json.loads(json.dumps(pk.serialize())))
    assert rt[0]["head"].id == 5 and len(rt[0]) == 13
    det = sv.Detections(xyxy=np.array([[1., 2., 30., 40.]]), confidence=np.array([0.9]), class_id=np.array([0]),
                        tracker_id=np.array([7]))
    p = Players([Player(det)])
    q = Players.from_json(json.loads(json.dumps(p.serialize())))
    assert q[0].id == 7 and q[0].feet == (15, 40) and q[0].class_id == 0


def test_polygon_zone_and_bytetrack_standins():
    if sv.HAVE_SUPERVISION:
        pytest.skip("real supervision installed")
    zone = sv.PolygonZone(np.array([[10, 10], [100, 10], [100, 100], [10, 100]]), frame_resolution_wh=(200, 200))
    det = sv.Detections(xyxy=np.array([[20., 20., 40., 60.], [150., 150., 170., 190.]], dtype=np.float32),
                        confidence=np.array([0.9, 0.8], dtype=np.float32), class_id=np.array([0, 0]))
    assert zone.trigger(det).tolist() == [True, False]
    bt = sv.ByteTrack(frame_rate=30)
    ids = []
    for t in range(5):
        d = sv.Detections(xyxy=np.array([[20. + t, 20., 40. + t, 60.], [100., 100. + t, 130., 160. + t]], np.float32),
                          confidence=np.array([0.9, 0.8], np.float32), class_id=np.array([0, 0]))
        out = bt.update_with_detections(d)
        ids.append(sorted(out.tracker_id.tolist()))
    assert ids[0] == [1, 2] and ids[-1] == [1, 2]


def test_shard_maths():
    for total, world in ((1024, 8), (1000, 3), (10, 4)):
        spans = [R.shard_range(total, r, world) for r in range(world)]
        assert spans[0][0] == 0 and spans[-1][1] == total
        assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
    assert R.ball_shard_frames(100, 0, 25) == (0, 32)
    assert R.ball_shard_frames(100, 25, 50) == (18, 57)
    assert R.ball_shard_frames(100, 75, 100) == (68, 100)


class _Echo(Tracker):
    """Tracker whose 'prediction' for a frame is the frame's first pixel value (stands in for a model on CPU)."""
    batch_size = 3

    def video_info_post_init(self, vi):
        return self

    def object(self):
        return Ball

    def draw_kwargs(self):
        return {}

    def restart(self):
        self.results.restart()

    def __str__(self):
        return "echo"

    def predict_sample(self, sample, **kw):
        return [int(f[0, 0, 0]) for f in sample]

    def predict_frames(self, gen, **kw):
        from padel_analytics_b200.trackers.tracker import NoPredictFrames

        raise NoPredictFrames()


def _frames(lo, hi):
    for i in range(lo, hi):
        yield np.full((2, 2, 3), i, dtype=np.uint8)


def test_runner_single_process():
    t = _Echo()
    R.TrackingRunner([t]).run(frame_source=_frames, total_frames=10)
    assert t.results.predictions == list(range(10))


def _stub(cls, **attrs):
    t = object.__new__(cls)  # no CUDA here: skip the engine construction, set what is read
    for k, v in attrs.items():
        setattr(t, k, v)
    return t


def test_tracker_stages():
    """Each tracker declares how TrackingRunner drives it: "detect" (YOLO model), "fixed", "ball" or "frames"."""
    from padel_analytics_b200.trackers import BallTracker, KeypointsTracker, PlayerKeypointsTracker, PlayerTracker

    def kt(**kw):
        return _stub(KeypointsTracker, **{"model_type": "yolo", "model": object(), "fixed_keypoints_detection": None,
                                          **kw})

    court = Keypoints([Keypoint(id=0, xy=(1.0, 2.0))])
    cases = [(_stub(PlayerTracker), "detect", None), (_stub(PlayerKeypointsTracker), "detect", None),
             (kt(), "detect", None), (kt(fixed_keypoints_detection=court), "fixed", court),
             (kt(model=None, fixed_keypoints_detection=court), "fixed", court), (kt(model=None), "frames", None),
             (kt(model_type="resnet"), "frames", None), (_stub(BallTracker), "ball", None), (_Echo(), "frames", None)]
    for t, stage, fixed in cases:
        assert (t.stage, t.fixed_detection) == (stage, fixed), (type(t).__name__, vars(t))


def test_runner_runs_frames_stage_trackers_in_frame_order():
    """Two trackers of stage "frames" (the echo, and a ResNet court regressor -- here a CPU stand-in for the engine)
    run through predict_and_update; both hold one result per frame, in frame order."""
    from types import SimpleNamespace

    from padel_analytics_b200.trackers import KeypointsTracker

    def regress(chunk):  # (n, 24) in [0, 1]: frame i -> every coordinate i / 16
        return np.array([[f[0, 0, 0] / 16.0] * 24 for f in chunk], dtype=np.float32)

    echo = _Echo()
    kt = KeypointsTracker(None, batch_size=4, model_type="yolo")
    kt.model_type, kt.model = "resnet", SimpleNamespace(predict_frames=regress, to=lambda device: None)
    assert (echo.stage, kt.stage) == ("frames", "frames")
    R.TrackingRunner([echo, kt]).run(frame_source=_frames, total_frames=10)
    assert echo.results.predictions == list(range(10))
    assert [[k.xy for k in p.keypoints] for p in kt.results.predictions] == [[(i / 8, i / 8)] * 12 for i in range(10)]
    assert [[k.id for k in p.keypoints] for p in kt.results.predictions] == [list(range(12))] * 10


def test_runner_world2_gloo(tmp_path):
    """Two processes over gloo: each handles its contiguous shard, rank 0 assembles frame-ordered results."""
    script = tmp_path / "w.py"
    script.write_text(f"""
import sys, json
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import torch.distributed as dist
from test_host_cpu import _Echo, _frames
from padel_analytics_b200.trackers import runner as R
dist.init_process_group('gloo')
t = _Echo()
R.TrackingRunner([t]).run(frame_source=_frames, total_frames=11)
if dist.get_rank() == 0:
    assert t.results.predictions == list(range(11)), t.results.predictions
    print('WORLD2_OK')
else:
    assert t.results.predictions == []
dist.destroy_process_group()
""")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29517", str(script)], capture_output=True,
                       text=True, env=env, timeout=240)
    assert "WORLD2_OK" in r.stdout, r.stdout + r.stderr


def _fake_blocks(frames, kpt_shape, seed=0, per_block=4):
    """Deterministic ragged detections (0..5 per frame) keyed by absolute frame number, as the per-batch ResultBlocks
    of a pass: `per_block` frames each, the last block partial."""
    from padel_analytics_b200.engine.yolo_engine import ResultBlock

    frames = list(frames)
    rowlen = 6 + (kpt_shape[0] * kpt_shape[1] if kpt_shape else 0)
    out = []
    for i in range(0, len(frames), per_block):
        chunk = frames[i:i + per_block]
        rows = np.zeros((len(chunk), 5, rowlen), np.float32)
        counts = np.zeros((len(chunk),), np.int32)
        for j, n in enumerate(chunk):
            g = torch.Generator().manual_seed(1000 * seed + n)
            k = int(torch.randint(0, 6, (1,), generator=g))
            rows[j, :k, :6] = (torch.rand((k, 6), generator=g) * 100 + n).numpy()
            if kpt_shape:
                kp = torch.rand((k,) + tuple(kpt_shape), generator=g) * 50 + n
                rows[j, :k, 6:] = kp.reshape(k, rowlen - 6).numpy()
            counts[j] = k
        out.append(ResultBlock(rows, counts, kpt_shape, {0: "x"}, None))
    return out


def test_runner_world2_gloo_fixed_capacity_block_records(tmp_path):
    """The sharded gather of SURVEY 8(e): ragged per-batch detection blocks -> padded (frames, cap, 6+K*D) blocks +
    counts, all_gather over gloo, rank 0 rebuilds the frame-ordered Results; ball (x, y, vis) int32 records likewise."""
    script = tmp_path / "w2.py"
    script.write_text(f"""
import sys
sys.path.insert(0, {str(ROOT)!r}); sys.path.insert(0, {str(ROOT / 'tests')!r})
import torch, torch.distributed as dist
from types import SimpleNamespace
from test_host_cpu import _fake_blocks
from padel_analytics_b200.trackers import runner as R
dist.init_process_group('gloo')
rank, world, total = dist.get_rank(), dist.get_world_size(), 23
lo, hi = R.shard_range(total, rank, world)
for kpt_shape in (None, (13, 3)):
    trk = SimpleNamespace(model=SimpleNamespace(kpt_shape=kpt_shape, names={{0: 'x'}}))
    rec = R._yolo_records(_fake_blocks(range(lo, hi), kpt_shape), trk)
    parts = R._all_gather_yolo(rec, total, rank, world)
    got = [r for p in parts for r in p.to_results(trk)]
    exp = [r for b in _fake_blocks(range(total), kpt_shape) for r in b]
    assert len(got) == total
    for g, e in zip(got, exp):
        assert torch.equal(g.boxes.data, e.boxes.data)
        if kpt_shape:
            assert torch.equal(g.keypoints.data, e.keypoints.data)
xyv = {{n: (n, 2 * n, n % 2) for n in range(lo, hi) if n % 5}}
ball = R._all_gather_ball(R._ball_records(xyv, lo, hi), total, rank, world)
merged = {{}}
for b in ball:
    merged.update(b.to_dict())
assert merged == {{n: (n, 2 * n, n % 2) for n in range(total) if n % 5}}, merged
if rank == 0:
    print('RECORDS_OK')
dist.destroy_process_group()
""")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29519", str(script)], capture_output=True,
                       text=True, env=env, timeout=240)
    assert "RECORDS_OK" in r.stdout, r.stdout + r.stderr


def test_ball_tracker_inpaint_host_logic_reproduces_reference_golden():
    """BallTracker._inpaint_stage (product host code: mask, sequences, blend, COOR_TH, coordinate ensemble, float32 pixel
    conversion) driven with the CPU oracle network instead of the CUDA kernel must reproduce the golden produced by the
    reference BallTracker's own inpainting branch exactly (tests/golden/inpaint_ref.npz)."""
    from pathlib import Path
    import torch
    from oracle import inpaint as OI
    from padel_analytics_b200.trackers import sv_compat as sv
    from padel_analytics_b200.trackers.ball_tracker import BallTracker

    g = np.load(Path(__file__).resolve().parent / "golden" / "inpaint_ref.npz")
    net = OI.load_inpaintnet(OI.make_inpaintnet())
    bt = object.__new__(BallTracker)  # no CUDA here: skip the engine construction, set what the stage reads
    bt.inpaintnet_seq_len = int(g["seq_len"])
    bt.DELTA_T = 1 / math.sqrt(bt.HEIGHT ** 2 + bt.WIDTH ** 2)  # what __init__ sets (ball_tracker.py:246-247)
    bt.COOR_TH = bt.DELTA_T * 50
    bt.video_info = sv.VideoInfo(width=int(g["W"]), height=int(g["H"]), fps=30.0, total_frames=int(g["T"]))

    def cpu_net(coor, mask):
        with torch.no_grad():
            return net(coor, mask)

    bt.inpaintnet = cpu_net
    res = bt._inpaint_stage(g["x"].tolist(), g["y"].tolist(), g["vis"].tolist())
    n = len(g["X"])
    assert [res[i][0] for i in range(n)] == g["X"].tolist()
    assert [res[i][1] for i in range(n)] == g["Y"].tolist()
    assert [res[i][2] for i in range(n)] == g["V"].tolist()
    # and the mask generator agrees with the oracle's on random trajectories
    rng = np.random.default_rng(3)
    for _ in range(50):
        T = int(rng.integers(5, 80))
        vis = (rng.random(T) > 0.4).astype(int)
        y = rng.integers(0, 1080, T) * vis
        a = BallTracker._generate_inpaint_mask(y.tolist(), vis.tolist(), th_h=54.0)
        b = OI.generate_inpaint_mask(y.tolist(), vis.tolist(), th_h=54.0)
        assert list(a) == list(b)


def test_runner_assemble_applies_inpainting_after_merging_shards():
    """TrackingRunner._assemble: the ball shards are merged first, then the whole-trajectory InpaintNet stage runs once
    (same result as the unsharded BallTracker.predict_frames path, checked against the reference golden)."""
    from pathlib import Path
    import torch
    from oracle import inpaint as OI
    from padel_analytics_b200.trackers import sv_compat as sv
    from padel_analytics_b200.trackers.ball_tracker import BallTracker
    from padel_analytics_b200.trackers.runner import TrackingRunner
    from padel_analytics_b200.trackers.tracker import TrackingResults

    g = np.load(Path(__file__).resolve().parent / "golden" / "inpaint_ref.npz")
    net = OI.load_inpaintnet(OI.make_inpaintnet())
    bt = object.__new__(BallTracker)
    bt.results = TrackingResults()
    bt.inpaintnet_seq_len = int(g["seq_len"])
    bt.DELTA_T = 1 / math.sqrt(bt.HEIGHT ** 2 + bt.WIDTH ** 2)
    bt.COOR_TH = bt.DELTA_T * 50
    bt.video_info = sv.VideoInfo(width=int(g["W"]), height=int(g["H"]), fps=30.0, total_frames=int(g["T"]))
    bt.inpaintnet = lambda c, m: net(c, m).detach()
    T = len(g["x"])
    xyv = {n: (int(g["x"][n]), int(g["y"][n]), int(g["vis"][n])) for n in range(T)}
    parts = [{n: xyv[n] for n in range(0, T // 3)}, {n: xyv[n] for n in range(T // 3, T)}]  # two "ranks"
    TrackingRunner._assemble(bt, parts, T)
    got = bt.results.predictions
    assert [int(b.xy[0]) for b in got] == g["X"].tolist() and [int(b.xy[1]) for b in got] == g["Y"].tolist()
    assert [b.visibility for b in got] == g["V"].tolist()
    # a tracker without an inpainting model keeps the TrackNet trajectory
    bt.inpaintnet = None
    TrackingRunner._assemble(bt, parts, T)
    assert [(int(b.xy[0]), int(b.xy[1]), b.visibility) for b in bt.results.predictions] == [xyv[n] for n in range(T)]


def test_product_package_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under padel_analytics_b200/ may import it (static check)."""
    root = Path(__file__).resolve().parents[1] / "padel_analytics_b200"
    bad = []
    for p in root.rglob("*.py"):
        for i, line in enumerate(p.read_text().splitlines(), 1):
            if re.match(r"\s*(from|import)\s+oracle\b", line):
                bad.append(f"{p.relative_to(root)}:{i}: {line.strip()}")
    assert not bad, bad


def test_yolo_results_scaling_matches_oracle_ops():
    """YoloEngine._results (product host code: un-letterbox, clip, keypoint-confidence zeroing) against the oracle's
    restatement of ultralytics scale_boxes / scale_coords on random detections, several geometries."""
    from oracle import yolov8 as OY
    from padel_analytics_b200.engine.yolo_engine import YoloEngine

    eng = object.__new__(YoloEngine)  # host logic only; no CUDA here
    eng.names = {0: "person"}
    rng = np.random.default_rng(7)
    for kpt_shape, net_hw, orig_hw in [(None, (384, 640), (1080, 1920)), ((13, 3), (1280, 1280), (1280, 1280)),
                                       ((12, 3), (640, 640), (640, 640)), ((13, 3), (384, 640), (2160, 3840)),
                                       (None, (640, 480), (700, 500))]:
        eng.kpt_shape = kpt_shape
        K, D = kpt_shape if kpt_shape else (0, 0)
        n, cap = 3, 9
        rows = np.zeros((n, cap, 6 + K * D), np.float32)
        counts = np.array([cap, 4, 0], np.int32)
        rows[..., 0:4] = rng.uniform(-20, max(net_hw) + 20, (n, cap, 4))
        rows[..., 4] = rng.uniform(0.3, 1, (n, cap))
        if K:
            kp = rng.uniform(-30, max(net_hw) + 30, (n, cap, K, D)).astype(np.float32)
            kp[..., 2] = rng.uniform(0, 1, (n, cap, K))
            rows[..., 6:] = kp.reshape(n, cap, -1)
        res = eng._results(rows, counts, n, net_hw, orig_hw)
        for i in range(n):
            c = counts[i]
            exp_box = OY.scale_boxes(net_hw, torch.from_numpy(rows[i, :c, :4].copy()), orig_hw)
            assert torch.equal(res[i].boxes.xyxy, exp_box), (kpt_shape, net_hw, orig_hw)
            assert torch.equal(res[i].boxes.conf, torch.from_numpy(rows[i, :c, 4]))
            if K:
                k = torch.from_numpy(rows[i, :c, 6:].reshape(c, K, D).copy())
                exp_k = OY.scale_coords(net_hw, k, orig_hw)
                exp_xy = exp_k[..., :2].clone()
                exp_xy[exp_k[..., 2] < 0.5] = 0
                assert torch.equal(res[i].keypoints.xy, exp_xy), (kpt_shape, net_hw, orig_hw)


def test_weight_folding_and_packing_layouts():
    """engine/ops.py host helpers: BN folding is the exact conv+BN(eval) algebra; packed layouts are
    [tap][cout_pad][cin_pad] (with an optional input-channel map) and, for the stem, [filter row][cout_pad][s*4 + c]."""
    import torch.nn as nn
    import torch.nn.functional as F
    from padel_analytics_b200.engine import ops

    g = torch.Generator().manual_seed(0)
    conv = nn.Conv2d(5, 7, 3, padding=1, bias=False)
    bn = nn.BatchNorm2d(7, eps=1e-3).eval()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g))
        bn.weight.copy_(torch.rand(7, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(7, generator=g))
        bn.running_mean.copy_(torch.randn(7, generator=g))
        bn.running_var.copy_(torch.rand(7, generator=g) + 0.5)
        x = torch.randn(2, 5, 9, 11, generator=g)
        w, b = ops.fold_bn(conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, 1e-3)
        assert torch.allclose(F.conv2d(x, w, b, padding=1), bn(conv(x)), atol=1e-5)
    wp, bp = ops.pack_conv_weight(w, b, 16, 16, "cpu")
    assert wp.shape == (9, 16, 16) and wp.dtype == torch.float16 and bp.shape == (16,)
    for r in range(3):
        for s in range(3):
            assert torch.equal(wp[r * 3 + s, :7, :5], w[:, :, r, s].half())
    assert torch.count_nonzero(wp[:, 7:]) == 0 and torch.count_nonzero(wp[:, :, 5:]) == 0
    assert torch.equal(bp[:7], b.float()) and torch.count_nonzero(bp[7:]) == 0
    # input-channel map (concat of individually padded slices): logical channel i lives at cin_map[i]
    cmap = [0, 1, 2, 16, 17]
    wm, _ = ops.pack_conv_weight(w, b, 32, 16, "cpu", cin_map=cmap)
    for i, pos in enumerate(cmap):
        assert torch.equal(wm[4, :7, pos], w[:, i, 1, 1].half())
    assert torch.count_nonzero(wm[:, :, 3:16]) == 0
    # stem: k = s*4 + c over the padded 4-channel pixels, fourth pixel / fourth channel carry zero weights
    ws = torch.randn(6, 3, 3, 3, generator=g)
    sp, sb = ops.pack_stem_weight(ws, torch.arange(6.0), 16, "cpu")
    assert sp.shape == (3, 16, 16)
    for r in range(3):
        for s in range(3):
            for c in range(3):
                assert torch.equal(sp[r, :6, s * 4 + c], ws[:, c, r, s].half())
    assert torch.count_nonzero(sp[:, :, 3::4]) == 0 and torch.count_nonzero(sp[:, :, 12:]) == 0
    assert torch.equal(sb[:6], torch.arange(6.0))


@pytest.mark.parametrize("impl", ["native", "python"])
def test_bytetrack_follows_the_published_algorithm(impl):
    """sv_compat.ByteTrack (C++, pb_bytetrack_*) and ByteTrackPy (numpy): ids from 1, a new track is confirmed at its second frame (immediately on frame 1), an
    occluded track is re-identified from the lost pool through its Kalman prediction, low-score detections only extend
    existing tracks, detections without a track are dropped, reset() restarts the ids."""
    rng = np.random.default_rng(0)
    base = np.array([[100, 100, 160, 260], [400, 120, 470, 300], [800, 500, 880, 700], [1200, 400, 1270, 600]], float)
    bt = (sv.ByteTrack if impl == "native" else sv.ByteTrackPy)(frame_rate=30)
    seen = {}
    for f in range(40):
        b = base + np.array([3 * f, f, 3 * f, f]) + rng.normal(0, 1.5, (4, 4))
        keep = np.ones(4, bool)
        if 10 <= f < 14:
            keep[1] = False  # occlusion of track 2
        conf = np.full(4, 0.8)
        if f == 30:
            conf[2] = 0.2  # low-score detection of an existing track: second association keeps it
        extra = np.array([[50 + f, 900, 90 + f, 1000]]) if f in (20, 21, 22) else np.zeros((0, 4))
        lowonly = np.array([[1500, 100, 1560, 200]]) if f == 5 else np.zeros((0, 4))  # low score, no track: dropped
        xy = np.vstack([b[keep], extra, lowonly])
        cf = np.r_[conf[keep], np.full(len(extra), 0.9), np.full(len(lowonly), 0.2)]
        out = bt.update_with_detections(sv.Detections(xyxy=xy.astype(np.float32), confidence=cf.astype(np.float32),
                                                      class_id=np.zeros(len(xy), int)))
        seen[f] = out.tracker_id.tolist()
    assert seen[0] == [1, 2, 3, 4] and seen[9] == [1, 2, 3, 4]
    assert seen[10] == [1, 3, 4] and seen[13] == [1, 3, 4]
    assert seen[14] == [1, 2, 3, 4]  # re-identified, same id
    assert seen[5] == [1, 2, 3, 4]
    assert seen[20] == [1, 2, 3, 4] and seen[21] == [1, 2, 3, 4, 5] and seen[23] == [1, 2, 3, 4]
    assert seen[30] == [1, 2, 3, 4]
    bt.reset()
    out = bt.update_with_detections(sv.Detections(xyxy=base.astype(np.float32), confidence=np.full(4, 0.9, np.float32),
                                                  class_id=np.zeros(4, int)))
    assert out.tracker_id.tolist() == [1, 2, 3, 4]
    p = Player.from_json({"id": None, "xyxy": [1.0, 2.0, 3.0, 4.0], "projection": None, "class_id": 0, "confidence": 0.5})
    assert p.id is None and Player.from_json(p.serialize()).serialize() == p.serialize()


def test_native_bytetrack_equals_the_python_restatement():
    """pb_bytetrack_update (csrc/bytetrack.cu) vs sv_compat.ByteTrackPy on random multi-object sequences with
    occlusions, low-score and spurious detections: identical kept detections and ids, frame for frame."""
    def seq(seed, T=200):
        rng = np.random.default_rng(seed)
        K = int(rng.integers(3, 14))
        pos, vel, size = rng.uniform(100, 1500, (K, 2)), rng.normal(0, 4, (K, 2)), rng.uniform(40, 220, (K, 2))
        for _ in range(T):
            pos = pos + vel + rng.normal(0, 1.0, (K, 2))
            vis = rng.random(K) > 0.08
            conf = np.clip(rng.normal(0.7, 0.25, K), 0.05, 0.99)
            b = np.hstack([pos - size / 2, pos + size / 2]) + rng.normal(0, 1.5, (K, 4))
            extra = rng.uniform(0, 1800, (int(rng.integers(0, 3)), 2))
            eb = np.hstack([extra, extra + rng.uniform(30, 100, (len(extra), 2))])
            yield (np.vstack([b[vis], eb]).astype(np.float32),
                   np.r_[conf[vis], rng.uniform(0.1, 0.9, len(eb))].astype(np.float32))

    frames = 0
    for seed in range(8):
        a, b = sv.ByteTrackPy(frame_rate=25.08), sv.ByteTrack(frame_rate=25.08)
        for xy, cf in seq(seed):
            mk = lambda: sv.Detections(xyxy=xy.copy(), confidence=cf.copy(), class_id=np.zeros(len(xy), int))
            o1, o2 = a.update_with_detections(mk()), b.update_with_detections(mk())
            assert np.array_equal(o1.tracker_id, o2.tracker_id) and np.array_equal(o1.xyxy, o2.xyxy), (seed, frames)
            frames += 1
    assert frames == 1600


def test_block_postprocess_equals_per_result_postprocess():
    """The dense fast path (ResultBlock -> one polygon test, one pb_bytetrack_update_many call, vectorised ratios) must
    produce exactly what the per-frame loop over ultralytics-style Results produces, for all three YOLO trackers."""
    from types import SimpleNamespace

    from padel_analytics_b200.engine.yolo_engine import ResultBlock
    from padel_analytics_b200.trackers import sv_compat as sv
    from padel_analytics_b200.trackers.keypoints_tracker import KeypointsTracker
    from padel_analytics_b200.trackers.players_keypoints_tracker import PlayerKeypointsTracker
    from padel_analytics_b200.trackers.players_tracker import PlayerTracker

    rng = np.random.default_rng(11)
    F, cap = 90, 7

    def block(kpt_shape):
        K, D = kpt_shape if kpt_shape else (0, 0)
        rows = np.zeros((F, cap, 6 + K * D), np.float32)
        counts = rng.integers(0, cap + 1, F).astype(np.int32)
        counts[:3] = (0, 1, cap)
        # four slowly moving boxes + noise so that ByteTrack keeps, loses and re-finds tracks
        base = rng.uniform(100, 800, (cap, 2))
        for f in range(F):
            xy = base + 3.0 * f + rng.normal(0, 2, (cap, 2))
            rows[f, :, 0:2] = xy
            rows[f, :, 2:4] = xy + rng.uniform(40, 120, (cap, 2))
            rows[f, :, 4] = np.sort(rng.uniform(0.05, 0.95, cap))[::-1]
        if K:
            rows[..., 6:] = rng.uniform(0, 640, (F, cap, K * D)).astype(np.float32)
        rows[np.arange(cap)[None, :] >= counts[:, None]] = 0
        return ResultBlock(rows, counts, kpt_shape, {0: "person"}, (1080, 1920))

    def stub(cls, **attrs):
        t = object.__new__(cls)
        for k, v in attrs.items():
            setattr(t, k, v)
        return t

    poly = np.array([[50, 50], [1500, 60], [1600, 1000], [40, 900]])
    blk = block(None)
    outs = []
    for as_block in (True, False):
        t = stub(PlayerTracker, polygon_zone=sv.PolygonZone(poly, frame_resolution_wh=(1920, 1080)),
                 byte_track=sv.ByteTrack(frame_rate=30))
        outs.append(t.postprocess(blk if as_block else list(blk)))
    assert sum(len(p) for p in outs[0]) > F  # the scenario does track something
    assert len(outs[0]) == len(outs[1]) == F
    for a, b in zip(*outs):
        assert [p.serialize() for p in a] == [p.serialize() for p in b]
    # and split over several calls (the batches of a pass) == one call (rank 0 after the gather)
    t = stub(PlayerTracker, polygon_zone=None, byte_track=sv.ByteTrack(frame_rate=30))
    whole = t.postprocess(blk)
    t = stub(PlayerTracker, polygon_zone=None, byte_track=sv.ByteTrack(frame_rate=30))
    pieces = t.postprocess(blk[:32]) + t.postprocess(blk[32:64]) + t.postprocess(blk[64:])
    assert [[p.serialize() for p in a] for a in whole] == [[p.serialize() for p in a] for a in pieces]

    blk = block((13, 3))
    t = stub(PlayerKeypointsTracker, train_image_size=1280)
    a, b = t.postprocess(blk, (1080, 1920)), t.postprocess(list(blk), (1080, 1920))
    assert [x.serialize() for x in a] == [x.serialize() for x in b]
    blk = block((12, 3))
    t = stub(KeypointsTracker)
    a, b = t.postprocess(blk, (1080, 1920)), t.postprocess(list(blk), (1080, 1920))
    assert [x.serialize() for x in a] == [x.serialize() for x in b]

    # concat pads to the largest count and keeps frame order
    c = ResultBlock.concat([blk[:10], blk[10:11], blk[11:]])
    assert np.array_equal(c.counts, blk.counts) and np.array_equal(c.rows, blk.rows[:, :c.rows.shape[1]])


def test_block_postprocess_handles_empty_blocks_and_empty_shards():
    """A rank may own no frames at all (more ranks than frames) and a batch may hold no detections."""
    from types import SimpleNamespace

    from padel_analytics_b200.engine.yolo_engine import ResultBlock
    from padel_analytics_b200.trackers import runner as R
    from padel_analytics_b200.trackers import sv_compat as sv
    from padel_analytics_b200.trackers.keypoints_tracker import KeypointsTracker
    from padel_analytics_b200.trackers.players_keypoints_tracker import PlayerKeypointsTracker
    from padel_analytics_b200.trackers.players_tracker import PlayerTracker

    def stub(cls, **attrs):
        t = object.__new__(cls)
        for k, v in attrs.items():
            setattr(t, k, v)
        return t

    for ks, cls, extra in ((None, PlayerTracker, dict(polygon_zone=None, byte_track=sv.ByteTrack(frame_rate=30))),
                           ((13, 3), PlayerKeypointsTracker, dict(train_image_size=1280)),
                           ((12, 3), KeypointsTracker, {})):
        trk = stub(cls, model=SimpleNamespace(kpt_shape=ks, names={0: "x"}), **extra)
        rec = R._yolo_records([], trk)  # a shard without frames
        blk = rec.to_results(trk)
        assert len(blk) == 0 and list(blk) == []
        args = () if cls is PlayerTracker else ((1080, 1920),)
        assert trk.postprocess(blk, *args) == []
        rowlen = rec.rows.shape[2]
        none = ResultBlock(np.zeros((4, 1, rowlen), np.float32), np.zeros((4,), np.int32), ks, {0: "x"}, None)
        out = trk.postprocess(ResultBlock.concat([blk, none, blk]), *args)  # frames without detections
        assert len(out) == 4 and all(len(o.serialize()) == 0 for o in out)
