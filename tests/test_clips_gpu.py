"""Tracking a list of clips in one pass: the two multi-clip kernels against a numpy gather and the reference ensemble
loop per clip, and `TrackingRunner.run_clips` against a fresh `TrackingRunner.run()` on each clip alone."""
import json

import numpy as np
import pytest
import torch

from oracle import inpaint as OI
from oracle import tracknet as OT
from oracle import weights as OW
from padel_analytics_b200 import _lib as L
from padel_analytics_b200 import synth
from padel_analytics_b200.engine.clip_plan import plan_clip_batches
from padel_analytics_b200.trackers import (BallTracker, KeypointsTracker, PlayerKeypointsTracker, PlayerTracker,
                                           TrackingRunner)
from padel_analytics_b200.trackers import sv_compat as sv

pytestmark = pytest.mark.gpu
H, W = 1080, 1920


def test_pack_windows_rows_equals_per_row_pack():
    """Every row of one launch over random ring slots and pool medians == the numpy gather of its median and its 8
    ring slots, bit for bit."""
    Hn, Wn, ring, pool, B = 24, 40, 29, 5, 13
    g = torch.Generator().manual_seed(3)
    frames = torch.randint(0, 1 << 15, (ring, Hn, Wn, 4), generator=g, dtype=torch.int16)
    meds = torch.randint(0, 1 << 15, (pool, Hn, Wn, 4), generator=g, dtype=torch.int16)
    slots = torch.randint(0, ring, (B,), generator=g, dtype=torch.int32)
    slots[3] = ring - 1  # a window that wraps the ring
    mids = torch.randint(0, pool, (B,), generator=g, dtype=torch.int32)
    x = torch.full((B, Hn, Wn, 32), 7, dtype=torch.int16, device="cuda")
    fd, md, slots_d, mids_d = frames.cuda(), meds.cuda(), slots.cuda(), mids.cuda()
    L.check(L.lib().pb_tracknet_pack_windows_rows(fd.data_ptr(), ring, slots_d.data_ptr(), md.data_ptr(),
                                                  mids_d.data_ptr(), B, Hn, Wn, x.data_ptr(), L.stream_ptr()))
    got = x.cpu().numpy()
    fr, me = frames.numpy(), meds.numpy()
    for b in range(B):
        chans = [me[mids[b], ..., :3]] + [fr[(int(slots[b]) + f) % ring, ..., :3] for f in range(8)]
        exp = np.concatenate(chans + [np.zeros((Hn, Wn, 5), np.int16)], -1)
        assert np.array_equal(got[b], exp), b


@pytest.mark.parametrize("lengths,batch", [([5, 8, 9, 40, 77, 130], 32), ([8, 9, 8, 15, 3, 23, 8], 4),
                                           ([20, 8, 8, 8, 12], 16), ([30, 2, 30], 1)])
def test_ensemble_rows_equals_per_clip_ensemble(lengths, batch):
    """Every planned batch through pb_tracknet_ensemble_rows, with the engine's pred ring and 7-row carry: each clip's
    frames == oracle/tracknet.py's stateful ensemble loop run on that clip alone (ensemble bit for bit, and the mask
    is its threshold)."""
    Hn, Wn = 288, 512
    g = torch.Generator().manual_seed(len(lengths) * 100 + batch)
    plan = plan_clip_batches(lengths, batch)
    nw = [max(0, t - 7) for t in lengths]
    heat = torch.rand((sum(nw), 8, Hn, Wn), generator=g)
    heat.view(-1)[::5] = 0.5  # many ensembled pixels land on the threshold
    heat_d = heat.cuda()
    pred = torch.zeros((7 + batch, 8, Hn, Wn), device="cuda")
    maxf = 8 * batch
    mask, ens = (torch.empty((maxf, Hn, Wn), dtype=torch.uint8, device="cuda"),
                 torch.empty((maxf, Hn, Wn), device="cuda"))
    got, spans = {}, 0
    for ops in plan.steps:
        for op in ops:
            if op[0] != "run":
                continue
            b = op[1]
            nb, nf = len(b.windows), len(b.frames)
            pred[7:7 + nb] = heat_d[b.first_window:b.first_window + nb]
            desc = torch.tensor(b.desc, dtype=torch.int32).cuda()
            L.check(L.lib().pb_tracknet_ensemble_rows(pred.data_ptr(), b.first_window - 7, desc.data_ptr(), nf, Hn, Wn,
                                                      0.5, mask.data_ptr(), ens.data_ptr(), L.stream_ptr()))
            m, e = mask[:nf].cpu(), ens[:nf].cpu()
            for i, cf in enumerate(b.frames):
                got[cf] = (m[i], e[i])
            spans += len({c for c, _ in b.frames}) > 1
            pred[:7] = pred[nb:nb + 7].clone()
    if batch > 1:  # a one-window batch emits one clip's frames only
        assert spans, "vacuous: no batch emitted frames of two clips"
    w0 = 0
    for c, t in enumerate(lengths):
        exp = OT.ensemble_reference_loop(heat[w0:w0 + nw[c]], t, batch)
        w0 += nw[c]
        assert len(exp) == (t if t >= 8 else 0)
        for f in range(len(exp)):
            m, e = got.pop((c, f))
            assert torch.equal(e, exp[f]), (c, f)
            assert torch.equal(m.bool(), exp[f] > 0.5), (c, f)
    assert not got


# ---- end to end ------------------------------------------------------------------------------------------------------
LENGTHS = [5, 8, 9, 40, 77, 130]


def _trackers(B, med, ckpts, **ball_kw):
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    return [PlayerTracker(ckpts["detect"], poly, batch_size=B),
            PlayerKeypointsTracker(ckpts["pose13"], 1280, batch_size=B, load_path=None, save_path=None),
            KeypointsTracker(ckpts["court12"], batch_size=B, model_type="yolo"),
            BallTracker(ckpts["tracknet"], ckpts["inpaint"], batch_size=B, median=med, **ball_kw)]


def _vi(T):
    return sv.VideoInfo(width=W, height=H, fps=30.0, total_frames=T)


def _ser(objs):
    return json.dumps([o.serialize() for o in objs])


@pytest.fixture(scope="module")
def ckpts():
    return {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
            "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}


@pytest.fixture(scope="module")
def clips():
    return [synth.make_frames(T, H, W, start=11 * i + 1) for i, T in enumerate(LENGTHS)]


@pytest.mark.parametrize("supplied_median", [False, True])
def test_run_clips_equals_run_per_clip(ckpts, clips, supplied_median, tmp_path):
    """run_clips over 6 clips of 5..130 frames, batch 32, all four trackers with InpaintNet, in every stream mode:
    each clip's results == a fresh TrackingRunner.run() on that clip alone (ball x, y, visibility after InpaintNet;
    every YOLO object including ByteTrack ids).  The saved JSON loads back through load_predictions."""
    B = 32
    med = synth.make_median(H, W).numpy() if supplied_median else None
    kw = {} if supplied_median else {"median_max_sample_num": 50}  # clips longer than 50 frames use their first 50
    tr = _trackers(B, med, ckpts, **kw)
    for t in tr:
        t.video_info_post_init(_vi(None))
    fr = [[f.numpy() for f in c] for c in clips]
    expected = []
    for c, T in enumerate(LENGTHS):
        for t in tr:
            t.restart()
        TrackingRunner(tr, video_info=_vi(T)).run(frame_source=lambda lo, hi, c=c: iter(fr[c][lo:hi]), total_frames=T)
        expected.append({str(t): _ser(t.results.predictions) for t in tr})
        assert all(len(t.results) == T for t in tr)
    assert any(json.loads(e["players_tracker"]) != [[]] * T for e, T in zip(expected, LENGTHS)), "vacuous: no players"
    assert any('"visibility": 1' in e["ball_tracker"] for e in expected), "vacuous: no ball"
    for t in tr:
        t.restart()
    host = [c.pin_memory() for c in clips]
    dev = [c.cuda() for c in clips]
    sources = {
        "frames": [(lambda lo, hi, c=c: iter(fr[c][lo:hi]), T) for c, T in enumerate(LENGTHS)],
        "pinned": [(lambda lo, hi, c=c: (host[c][i:min(hi, i + 24)] for i in range(lo, hi, 24)), T)
                   for c, T in enumerate(LENGTHS)],
        "device": [(lambda lo, hi, c=c: (dev[c][i:min(hi, i + 32)] for i in range(lo, hi, 32)), T)
                   for c, T in enumerate(LENGTHS)],
    }
    runner = TrackingRunner(tr, video_info=_vi(None))
    for mode, kind in ((0, "frames"), (1, "pinned"), (2, "device"), (1, "frames")):
        save = tmp_path / f"m{mode}{kind}"
        got = runner.run_clips(sources[kind], save_dir=str(save), streams=mode)
        assert len(got) == len(LENGTHS)
        for c, res in enumerate(got):
            assert set(res) == set(expected[c])
            for name, objs in res.items():
                assert len(objs) == LENGTHS[c]
                assert _ser(objs) == expected[c][name], (mode, kind, c, name)
        assert all(len(t.results) == 0 for t in tr), "run_clips must leave the trackers' results alone"
    for c in range(len(LENGTHS)):  # the saved predictions load back through the trackers' own loader
        for t in tr:
            t.load_path = str(save / f"{c:04d}_{t}.json")
            t.load_predictions()
            assert _ser(t.results.predictions) == expected[c][str(t)]
            t.load_path = None
            t.restart()


def test_run_clips_rejects_mixed_frame_sizes(ckpts):
    tr = _trackers(4, synth.make_median(H, W).numpy(), ckpts)[2:]
    a = [f.numpy() for f in synth.make_frames(9, H, W)]
    b = [f.numpy() for f in synth.make_frames(9, 720, 1280)]
    runner = TrackingRunner(tr, video_info=_vi(None))
    with pytest.raises(ValueError, match="same frame size"):
        runner.run_clips([(lambda lo, hi: iter(a[lo:hi]), 9), (lambda lo, hi: iter(b[lo:hi]), 9)])
