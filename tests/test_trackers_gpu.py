"""Tracker-level parity through the reference-facing API (predict_and_update / predict_frames / runner)."""
import json

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from oracle import tracknet as OT
from oracle import weights as OW
from oracle import yolov8 as OY
from padel_analytics_b200 import synth
from padel_analytics_b200.trackers import (BallTracker, KeypointsTracker, PlayerKeypointsTracker, PlayerTracker,
                                           TrackingRunner)
from padel_analytics_b200.trackers import sv_compat as sv

pytestmark = pytest.mark.gpu
H, W = 1080, 1920


def _vi(total=None):
    return sv.VideoInfo(width=W, height=H, fps=30.0, total_frames=total)


def test_ball_tracker_predict_frames_matches_oracle_and_shards():
    T, B = 27, 8
    ck = OW.make_tracknet()
    frames = synth.make_frames(T, H, W)
    fr = [f.numpy() for f in frames]
    med = synth.make_median(H, W).numpy()
    ora = OT.run_ball_oracle(OW.load_tracknet(ck), fr, med, (W, H), batch_size=B)
    bt = BallTracker(ck, None, batch_size=B, median=med)
    bt.video_info_post_init(_vi(T))
    balls = bt.predict_and_update(iter(fr), total_frames=T).predictions
    assert len(balls) == T and [b.frame for b in balls] == list(range(T))
    # a frame is threshold-stable when the oracle's own answer does not move if 0.5 is shifted by +-eps (eps > the
    # measured heat-map error): on every such frame the tracker's (x, y, visibility) must be IDENTICAL
    eps, scaler = 0.03, (W / 512, H / 288)
    stable = same = 0
    for n, b in enumerate(balls):
        ref = (ora["x"][n], ora["y"][n], ora["vis"][n])
        alts = [tuple(v[0] for v in OT.predict_from_ensemble(ora["ens"][n:n + 1], scaler, threshold=t))
                for t in (0.5 - eps, 0.5 + eps)]
        got = (b.xy[0], b.xy[1], b.visibility)
        if all(a == ref for a in alts):
            stable += 1
            assert got == ref, f"frame {n}: got {got} oracle {ref}"
        same += int(got == ref)
    print(f"ball tracker: identical on {same}/{T} frames; {stable} threshold-stable frames, all identical")
    assert stable >= 3, "vacuous: no stable frames"
    json.dumps([b.serialize() for b in balls])
    # sharded execution (3 contiguous shards, run back to back on this GPU) == unsharded, frame for frame
    full = {n: (b.xy[0], b.xy[1], b.visibility) for n, b in enumerate(balls)}
    from padel_analytics_b200.trackers.runner import ball_shard_frames, shard_range

    merged = {}
    for r in range(3):
        lo, hi = shard_range(T, r, 3)
        flo, fhi = ball_shard_frames(T, lo, hi)
        merged.update(bt.track_xyv(iter(fr[flo:fhi]), T, first_frame=flo, emit_range=(lo, hi)))
    assert merged == full
    # fewer frames than announced: no tail flush, trailing frames are "missing" (ball_tracker.py:423,486,690-698)
    short = bt.predict_frames(iter(fr[:T - 1]), total_frames=T)
    assert [(b.xy, b.visibility) for b in short[-8:]] == [((0.0, 0.0), 0)] * 8


def test_yolo_trackers_api_and_parity():
    B, T = 2, 5
    frames = synth.make_frames(T, H, W, start=3)
    fr = [f.numpy() for f in frames]
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    cks = {k: OW.make_yolo(k) for k in ("detect", "pose13", "court12")}
    pt = PlayerTracker(cks["detect"], poly, batch_size=B)
    pk = PlayerKeypointsTracker(cks["pose13"], 1280, batch_size=B, load_path=None, save_path=None)
    kt = KeypointsTracker(cks["court12"], batch_size=B, model_type="yolo")
    for t in (pt, pk, kt):
        t.video_info_post_init(_vi(T))
        res = t.predict_and_update(iter(fr)).predictions
        assert len(res) == T  # 2+2+1 batches, last partial
        json.dumps([o.serialize() for o in res])
    import parity

    # players: boxes (before ByteTrack) vs oracle through the reference's processing (players_tracker.py:346-359),
    # borderline-exclusion protocol: every non-borderline oracle box needs an IoU >= 0.99 partner, no extras
    net = OW.load_yolo(cks["detect"])
    yolo = OY.YOLO(net)
    yolo.predict([cv2.cvtColor(f, cv2.COLOR_BGR2RGB) for f in fr[:B]], conf=0.5, iou=0.7, imgsz=640, classes=[0])
    got = pt.detect_sample(fr[:B])
    reps = parity.check_batch(net, yolo.last_preprocessed, got, 0.5, 0.7, [0], 300, (H, W), tag="[players tracker]")
    parity.assert_reports(reps, "players tracker", min_sure_frac=0.2, min_tight=0)
    assert all(p.id is not None for p in pt.results.predictions[0])
    # court: the tracker returns 12 keypoints with reference ids (keypoints_tracker.py:214-227)
    k0 = kt.results.predictions[0]
    if len(k0):
        assert sorted(k.id for k in k0) == list(range(12))
    # pose: tracker output (frame pixels, players_keypoints_tracker.py:276-318) vs the oracle's non-borderline players
    net = OW.load_yolo(cks["pose13"])
    yolo = OY.YOLO(net)
    sample = [Image.fromarray(cv2.cvtColor(f, cv2.COLOR_BGR2RGB)).resize((1280, 1280)) for f in fr[:1]]
    yolo.predict(sample, conf=0.25, iou=0.7, imgsz=1280, classes=[0])
    cand = parity.classify_candidates(parity.oracle_predictions(net, yolo.last_preprocessed)[0], 1, 0.25, 0.7, [0], 300)
    _, ck = parity.scale_to_image(cand.boxes, cand.extra, (1280, 1280), (1280, 1280), (13, 3))
    g = pk.results.predictions[0]
    gx = np.array([[kp.xy for kp in player] for player in g], dtype=np.float64).reshape(-1, 13, 2)
    ratio = np.array([W / 1280, H / 1280])
    nsure = 0
    for i in (cand.status == parity.SURE).nonzero().squeeze(1).tolist():
        ek = ck[i].numpy().astype(np.float64)
        stable = np.abs(ek[:, 2] - 0.5) > 0.02  # keypoints whose visibility cut (conf < 0.5 -> (0, 0)) is not borderline
        exy = np.where(ek[:, 2:3] >= 0.5, ek[:, :2], 0.0) * ratio
        d = np.linalg.norm(gx - exy[None], axis=-1)  # (players, 13) frame px
        best = d[:, stable].max(1).min() if len(gx) and stable.any() else 0.0
        assert best < 0.5, f"sure oracle player {i}: nearest tracker player is {best:.3f} px off on a stable keypoint"
        nsure += 1
    print("pose tracker: non-borderline oracle players all matched within 0.5 px:", nsure, "of", int(cand.exact_keep.sum()))
    assert nsure >= 3, "vacuous"


def _four_ckpts():
    return {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
            "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet()}


def _four_trackers(B, med=None, ckpts=None, **ball_kw):
    ck = ckpts or _four_ckpts()
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    return [PlayerTracker(ck["detect"], poly, batch_size=B),
            PlayerKeypointsTracker(ck["pose13"], 1280, batch_size=B, load_path=None, save_path=None),
            KeypointsTracker(ck["court12"], batch_size=B, model_type="yolo"),
            BallTracker(ck["tracknet"], None, batch_size=B, median=med, **ball_kw)]


def _dump(trackers):
    return {str(t): json.dumps([o.serialize() for o in t.results.predictions]) for t in trackers}


def test_runner_fused_default_equals_sequential_reference_loop():
    """TrackingRunner.run() -- the reference's entry point (runner.py:175-236) -- takes the fused single pass by
    default (one decode + upload per batch for all four trackers); its results must be identical, object for object,
    to the reference-style loop of one full pass per tracker (fused=False)."""
    T, B = 21, 4
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=7)]
    med = synth.make_median(H, W).numpy()
    src = lambda lo, hi: iter(fr[lo:hi])
    seq = _four_trackers(B, med)
    t_seq = TrackingRunner(seq, video_info=_vi(T)).run(frame_source=src, total_frames=T, fused=False)
    fus = _four_trackers(B, med)
    run = TrackingRunner(fus, video_info=_vi(T))
    t_fus = run.run(frame_source=src, total_frames=T)
    names = {"players_tracker", "players_keypoints_tracker", "keypoints_tracker", "ball_tracker"}
    assert set(t_seq) == names and names <= set(t_fus) and "_fused_pass" in t_fus
    for t in fus + seq:
        assert len(t.results) == T
    a, b = _dump(seq), _dump(fus)
    for k in names:
        assert a[k] == b[k], k
    assert any(len(p) for p in fus[0].results.predictions), "vacuous: no players"
    # a second run() finds the trackers full and does nothing (cached predictions, runner.py:187-191)
    assert run.run(frame_source=src, total_frames=T) == run.timings


def test_runner_computes_the_background_median_on_device_when_none_is_given():
    """BallTracker(median=None): the runner derives the median from the first median_max_sample_num frames of the
    video (iterable.py:58-73) with the selection kernel; same result as handing np.median's output in."""
    T, B = 20, 4
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=3)]
    src = lambda lo, hi: iter(fr[lo:hi])
    M = 9
    ref_med = np.median(np.array([f[..., ::-1] for f in fr[:M]]), 0).astype("uint8")
    outs = []
    for med, kw in ((ref_med, {}), (None, {"median_max_sample_num": M})):
        tr = _four_trackers(B, med, **kw)[2:]  # court + ball: enough to take the fused path
        TrackingRunner(tr, video_info=_vi(T)).run(frame_source=src, total_frames=T)
        outs.append(_dump(tr)["ball_tracker"])
    assert outs[0] == outs[1]
    # and a later run with a different median at the same resolution must not reuse the cached background
    bt = BallTracker(OW.make_tracknet(), None, batch_size=B, median=ref_med)
    bt.video_info_post_init(_vi(T))
    a = bt.track_xyv(iter(fr), T)
    other = 255 - ref_med
    bt.median = other
    b = bt.track_xyv(iter(fr), T)
    bt2 = BallTracker(OW.make_tracknet(), None, batch_size=B, median=other)
    bt2.video_info_post_init(_vi(T))
    assert b == bt2.track_xyv(iter(fr), T)
    bt.median = ref_med
    assert bt.track_xyv(iter(fr), T) == a


@pytest.mark.parametrize("fused", [None, True, False])
def test_runner_drives_the_resnet_court_regressor_through_predict_frames(fused):
    """KeypointsTracker(model_type="resnet") has no batch model stage (the reference runs it through predict_frames):
    run(), fused or not, gives it the keypoints of predict_and_update alone, and the player tracker beside it the
    results of a run of its own; run_clips refuses it with a ValueError naming it."""
    from oracle import resnet as OR

    T, B = 5, 2
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=4)]
    src = lambda lo, hi: iter(fr[lo:hi])
    sd = OR.make_resnet50_court()
    ck = OW.make_yolo("detect")
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    alone = KeypointsTracker(sd, batch_size=B, model_type="resnet")
    alone.predict_and_update(iter(fr))
    pt_alone = PlayerTracker(ck, poly, batch_size=B)
    TrackingRunner([pt_alone], video_info=_vi(T)).run(frame_source=src, total_frames=T)
    kt = KeypointsTracker(sd, batch_size=B, model_type="resnet")
    pt = PlayerTracker(ck, poly, batch_size=B)
    run = TrackingRunner([pt, kt], video_info=_vi(T))
    run.run(frame_source=src, total_frames=T, fused=fused)
    assert _dump([kt]) == _dump([alone]) and _dump([pt]) == _dump([pt_alone])
    assert len(kt.results) == len(pt.results) == T
    with pytest.raises(ValueError, match="keypoints_tracker"):
        run.run_clips([(src, T)])


def test_runner_sharded_over_nccl_equals_unsharded(tmp_path):
    """World-size-2 NCCL run of TrackingRunner.run (contiguous shards, ball halo, broadcast median, fixed-capacity
    all_gather, rank-0 ByteTrack/objects) == the single-process run.  Needs two GPUs (`gpurun --gpus 2`)."""
    import os
    import subprocess
    import sys
    from pathlib import Path

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = Path(__file__).resolve().parents[1]
    # one set of checkpoints for every process: the seeded factory standardises the heads with CPU convolutions whose
    # last bits depend on the thread count (torchrun sets OMP_NUM_THREADS=1), and the comparison below is exact
    cks = _four_ckpts()
    torch.save(cks, tmp_path / "ckpts.pt")
    script = tmp_path / "nccl2.py"
    script.write_text(f"""
import sys, json, os
sys.path.insert(0, {str(root)!r}); sys.path.insert(0, {str(root / 'tests')!r})
import numpy as np, torch, torch.distributed as dist
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ["LOCAL_RANK"])))
from padel_analytics_b200 import synth
from padel_analytics_b200.trackers import TrackingRunner
from test_trackers_gpu import _four_trackers, _dump, _vi, H, W
T, B = 37, 4
fr = [f.numpy() for f in synth.make_frames(T, H, W, start=7)]
tr = _four_trackers(B, None, ckpts=torch.load({str(tmp_path / 'ckpts.pt')!r}, weights_only=False), median_max_sample_num=11)
run = TrackingRunner(tr, video_info=_vi(T))
t = run.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
if dist.get_rank() == 0:
    open({str(tmp_path / 'sharded.json')!r}, "w").write(json.dumps(_dump(tr)))
    print("NCCL2_DONE", {{k: round(v, 3) for k, v in t.items()}})
dist.destroy_process_group()
""")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29533", str(script)], capture_output=True,
                       text=True, env=env, timeout=900)
    assert "NCCL2_DONE" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    print(r.stdout[-400:])
    T, B = 37, 4
    fr = [f.numpy() for f in synth.make_frames(T, H, W, start=7)]
    tr = _four_trackers(B, None, ckpts=cks, median_max_sample_num=11)
    TrackingRunner(tr, video_info=_vi(T)).run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=T)
    sharded = json.loads((tmp_path / "sharded.json").read_text())
    single = _dump(tr)
    for k in single:
        if sharded[k] != single[k]:  # say where: first differing frame and its two versions
            a, b = json.loads(sharded[k]), json.loads(single[k])
            n = next(i for i in range(max(len(a), len(b))) if i >= min(len(a), len(b)) or a[i] != b[i])
            raise AssertionError(f"{k}: first difference at frame {n} of {len(a)}/{len(b)}\n sharded: "
                                 f"{json.dumps(a[n])[:1500]}\n single : {json.dumps(b[n])[:1500]}")


def test_fused_pass_equals_per_tracker_passes():
    """FusedPass (one upload per batch, all four trackers' device work enqueued together) must give exactly the
    results of the reference-style sequential per-tracker passes."""
    from padel_analytics_b200.trackers.runner import FusedPass

    T, B = 21, 8
    frames = synth.make_frames(T, H, W, start=11)
    fr = [f.numpy() for f in frames]
    med = synth.make_median(H, W).numpy()
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    tr = {"players": PlayerTracker(OW.make_yolo("detect"), poly, batch_size=B),
          "pose": PlayerKeypointsTracker(OW.make_yolo("pose13", cls_mean=-5.5), 1280, batch_size=B, load_path=None,
                                         save_path=None),
          "court": KeypointsTracker(OW.make_yolo("court12"), batch_size=B, model_type="yolo"),
          "ball": BallTracker(OW.make_tracknet(), None, batch_size=B, median=med)}
    for t in tr.values():
        t.video_info_post_init(_vi(T))
    seq = {}
    for k in ("players", "pose", "court"):
        seq[k] = [o.serialize() for o in tr[k].predict_and_update(iter(fr)).predictions]
        tr[k].restart()
    seq["ball"] = [(b.xy[0], b.xy[1], b.visibility) for b in tr["ball"].predict_frames(iter(fr), total_frames=T)]
    host = frames.pin_memory()
    for mode in (0, 1, 2):  # single stream / YOLO chains concurrent / everything concurrent
        for k in ("players", "pose", "court"):
            tr[k].restart()
        fused = FusedPass(tr, (H, W), B, total_frames=T, streams=mode)
        got = {k: [] for k in ("players", "pose", "court")}
        ball = {}
        for out in fused.run(host[i:i + B] for i in range(0, T, B)):
            for k in got:
                got[k] += [o.serialize() for o in out[k]]
            ball.update(out["ball"])
        for k in got:
            assert json.dumps(got[k]) == json.dumps(seq[k]), (k, mode)
        assert [ball.get(n, (0.0, 0.0, 0)) for n in range(T)] == seq["ball"], mode


def test_inpaintnet_kernel_and_stage_match_oracle():
    """InpaintNet fused kernel vs the oracle module, and BallTracker's inpainting stage vs the oracle stage on the
    trajectory of the reference-generated golden (tests/golden/inpaint_ref.npz)."""
    from pathlib import Path
    from oracle import inpaint as OI
    from padel_analytics_b200.engine.inpaint_engine import InpaintNetEngine

    ick = OI.make_inpaintnet()
    net = OI.load_inpaintnet(ick)
    eng = InpaintNetEngine(ick["model"])
    g = torch.Generator().manual_seed(1)
    c = torch.rand((37, 16, 2), generator=g)
    m = (torch.rand((37, 16, 1), generator=g) > 0.6).float()
    with torch.no_grad():
        exp = net(c, m)
    got = eng(c, m).cpu()
    assert (got - exp).abs().max().item() < 2e-5
    gold = np.load(Path(__file__).resolve().parent / "golden" / "inpaint_ref.npz")
    Wv, Hv = int(gold["W"]), int(gold["H"])
    bt = BallTracker(OW.make_tracknet(), ick, batch_size=4, median=synth.make_median(Hv, Wv).numpy())
    bt.video_info_post_init(sv.VideoInfo(width=Wv, height=Hv, fps=30.0, total_frames=int(gold["T"])))
    res = bt._inpaint_stage(gold["x"].tolist(), gold["y"].tolist(), gold["vis"].tolist())
    X, Y, V = gold["X"].tolist(), gold["Y"].tolist(), gold["V"].tolist()
    assert [res[n][2] for n in range(len(X))] == V
    dx = max(abs(res[n][0] - X[n]) for n in range(len(X)))
    dy = max(abs(res[n][1] - Y[n]) for n in range(len(X)))
    assert dx <= 1 and dy <= 1, (dx, dy)  # fp32 kernel vs fp32 CPU convs: integer truncation may move one pixel
    exact = sum(1 for n in range(len(X)) if (res[n][0], res[n][1]) == (X[n], Y[n]))
    assert exact >= len(X) - 3


def test_config0_players_tracker_batch1_on_real_720p_frames():
    """BASELINE.json configs[0]: PlayerTracker only (YOLOv8n-detect), 720p frames of the example clip, batch_size = 1,
    through TrackingRunner.run() (one tracker -> the reference's plain per-tracker loop).  Real video content
    (the committed rally.mp4 frame, shifted to fake motion); detections vs the CPU oracle under the protocol, ids
    from the ByteTrack stage, JSON round trip."""
    import parity
    from fixtures import GOLDEN, glue_ckpt

    base = cv2.imread(str(GOLDEN / "rally" / "rally_f00_720p.jpg"))
    assert base.shape == (720, 1280, 3)
    fr = [np.ascontiguousarray(np.roll(base, 6 * i, axis=1)) for i in range(6)]
    Hh, Ww = 720, 1280
    ck = glue_ckpt("detect")
    poly = sv.PolygonZone(np.array([[0, 0], [Ww, 0], [Ww, Hh], [0, Hh]]), frame_resolution_wh=(Ww, Hh))
    pt = PlayerTracker(ck, poly, batch_size=1)
    run = TrackingRunner([pt], video_info=sv.VideoInfo(width=Ww, height=Hh, fps=25.0, total_frames=len(fr)))
    tm = run.run(frame_source=lambda lo, hi: iter(fr[lo:hi]), total_frames=len(fr))
    assert set(tm) == {"players_tracker"} and len(pt.results) == len(fr)
    json.dumps([o.serialize() for o in pt.results.predictions])
    ids = [p.id for o in pt.results.predictions for p in o]
    assert all(i is not None and i >= 1 for i in ids)
    net = OW.load_yolo(ck)
    yolo = OY.YOLO(net)
    yolo.predict([cv2.cvtColor(f, cv2.COLOR_BGR2RGB) for f in fr[:2]], conf=0.5, iou=0.7, imgsz=640, classes=[0])
    got = []
    for f in fr[:2]:  # batch_size = 1
        got += pt.detect_sample([f])
    reps = parity.check_batch(net, yolo.last_preprocessed, got, 0.5, 0.7, [0], 300, (Hh, Ww), tag="[configs[0] 720p]")
    parity.assert_reports(reps, "configs[0] 720p", min_sure_frac=0.0, min_tight=0)
    assert sum(r.n_ours for r in reps) > 0
