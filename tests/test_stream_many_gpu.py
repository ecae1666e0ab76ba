"""Several live streams in one pass (`TrackingRunner.stream_many`) on the GPU: the table kernels against the row kernels
and the CPU restatement, every stream's entries and final results against `stream()` on its frames alone, and the
latency bound of the docstring."""
import collections
import json

import numpy as np
import pytest
import torch

from oracle import inpaint as OI
from oracle import weights as OW
from padel_analytics_b200 import _lib as L
from padel_analytics_b200 import synth
from padel_analytics_b200.engine.stream_plan import StreamPlanner, ensemble_rule
from padel_analytics_b200.trackers import (BallTracker, KeypointsTracker, PlayerKeypointsTracker, PlayerTracker,
                                           TrackingRunner)
from padel_analytics_b200.trackers import sv_compat as sv
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from test_stream_many_cpu import _interleaving, ensemble_table

pytestmark = pytest.mark.gpu
H, W = 1080, 1920
B = 4
M = 5  # background from the stream: its first 5 frames
T_LAT = 8 * B + 16


def _i32(a):
    return torch.as_tensor(np.asarray(a, dtype=np.int32).reshape(-1)).cuda()


# ---- the table kernels ---------------------------------------------------------------------------------------------
def test_pack_slots_equals_pack_rows_on_video_and_clip_layouts():
    """Slot tables that describe the ring layouts of one video (wrapping) and of a clip list (rows of two clips with
    two medians) give the bytes the row kernel gives."""
    h, w, ring = 16, 32, 20
    g = torch.Generator().manual_seed(1)
    frames = torch.rand((ring, h, w, 4), generator=g).half().cuda()
    medians = torch.rand((2, h, w, 4), generator=g).half().cuda()
    for row_slot, row_median in (([15, 16, 17, 18, 19], [0] * 5), ([3, 4, 13, 14], [0, 0, 1, 1])):
        nb = len(row_slot)
        slots = [[(s + f) % ring for f in range(8)] for s in row_slot]
        a = torch.zeros((nb, h, w, 32), dtype=torch.float16, device="cuda")
        b = torch.ones_like(a)
        rs, rm, st = _i32(row_slot), _i32(row_median), _i32(slots)
        L.check(L.lib().pb_tracknet_pack_windows_rows(frames.data_ptr(), ring, rs.data_ptr(), medians.data_ptr(),
                                                      rm.data_ptr(), nb, h, w, a.data_ptr(), L.stream_ptr()))
        L.check(L.lib().pb_tracknet_pack_windows_slots(frames.data_ptr(), st.data_ptr(), medians.data_ptr(),
                                                       rm.data_ptr(), nb, h, w, b.data_ptr(), L.stream_ptr()))
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def _table_of_desc(desc, first_window):
    """The ensemble table that names, for each (clip window 0, window count, frame) descriptor, the rows
    pb_tracknet_ensemble_rows reads from pred (rows 0..6 = the carry, 7.. = the batch)"""
    out = []
    for cw0, tw, n in desc:
        ws, rule = ensemble_rule(n, tw)
        out.append([-1 if v is None else cw0 + v - (first_window - 7) for v in ws] + [rule])
    return out


@pytest.mark.parametrize("layout", ["video", "clips"])
def test_ensemble_table_equals_ensemble_rows(layout):
    """Tables describing one video's batches (head, body and tail) and a clip list's (a batch spanning two clips of
    another length each) give masks and ens values bit-identical to the row kernel's."""
    h, w, nb = 8, 64, 6
    g = torch.Generator().manual_seed(2)
    pred = torch.rand((7 + nb, 8, h, w), generator=g).cuda()
    pred.view(-1)[::7] = 0.5
    if layout == "video":  # a 20-frame video whose last batch is windows 7..12, after windows 0..6 (head)
        cases = [(7, [(0, 13, n) for n in range(7, 20)]), (7, [(0, 100, n) for n in range(7, 13)])]
    else:  # clip A: windows 0..9 (global), clip B: windows 10..11 (a 9-frame clip), batch = global windows 7..12
        cases = [(7, [(0, 10, n) for n in range(7, 17)] + [(10, 2, n) for n in range(0, 9)] + [(12, 5, 0)])]
    for first_window, desc in cases:
        nf = len(desc)
        d, t = _i32(desc), _i32(_table_of_desc(desc, first_window))
        m1 = torch.zeros((nf, h, w), dtype=torch.uint8, device="cuda")
        m2, e1, e2 = torch.ones_like(m1), torch.zeros((nf, h, w), device="cuda"), torch.ones((nf, h, w), device="cuda")
        L.check(L.lib().pb_tracknet_ensemble_rows(pred.data_ptr(), first_window - 7, d.data_ptr(), nf, h, w, 0.5,
                                                  m1.data_ptr(), e1.data_ptr(), L.stream_ptr()))
        L.check(L.lib().pb_tracknet_ensemble_table(pred.data_ptr(), 7, pred[7:].data_ptr(), t.data_ptr(), nf, h, w,
                                                   0.5, m2.data_ptr(), e2.data_ptr(), L.stream_ptr()))
        assert torch.equal(m1, m2)
        assert torch.equal(e1.view(torch.int32), e2.view(torch.int32))


@pytest.mark.parametrize("Bk", [3, 8])
def test_table_kernels_on_interleaved_streams_equal_the_cpu_restatement(Bk):
    """The planner's tables for a random interleaving of streams, run through the pack, ensemble-table and carry
    kernels on device pools: each row packs the frames of its window, and every emitted frame equals the CPU
    restatement bit for bit (which equals each stream's single-stream ensemble, test_stream_many_cpu)."""
    from padel_analytics_b200.trackers.runner import StreamMux

    h, w = 8, 64
    rng = np.random.default_rng(Bk)
    lengths = [0, 1, 7, 8, 9, 20, 31]
    items = _interleaving(rng, lengths, 3)
    mux = StreamMux(items, Bk, 3, hold_device="cpu")
    plan = StreamPlanner(Bk, 3)
    g = torch.Generator().manual_seed(Bk)
    pix = {k: torch.rand((max(T, 1), h, w, 4), generator=g).half() for k, T in enumerate(lengths)}
    heat = {k: torch.rand((max(T, 1), 8, h, w), generator=g) for k, T in enumerate(lengths)}
    pool = torch.zeros((plan.n_slots, h, w, 4), dtype=torch.float16, device="cuda")
    meds = torch.rand((3, h, w, 4), generator=g).half().cuda()
    carry = torch.zeros((plan.carry_rows, 8, h, w), device="cuda")
    carry_np = np.zeros((plan.carry_rows, 8, h, w), np.float32)
    n_frames = 0
    for _ in mux.pieces():
        while mux.metas:
            runs, ends = mux.metas.popleft()
            st = plan.step([(k, n) for k, _, n in runs], ends)
            chunk = [(k, f0 + i) for k, f0, n in runs for i in range(n)]
            for o, n, slot in st.pushes:
                for i in range(n):
                    k, f = chunk[o + i]
                    pool[slot + i] = pix[k][f].cuda()
            for la in st.launches:
                nb, nf = len(la.rows), len(la.frames)
                fresh = (torch.stack([heat[k][wi] for k, wi in la.rows]) if nb else torch.zeros((1, 8, h, w))).cuda()
                if nb:
                    x = torch.zeros((nb, h, w, 32), dtype=torch.float16, device="cuda")
                    slots, row_median = _i32(la.row_slots), _i32(la.row_median)  # alive until the kernels ran
                    L.check(L.lib().pb_tracknet_pack_windows_slots(pool.data_ptr(), slots.data_ptr(), meds.data_ptr(),
                                                                   row_median.data_ptr(), nb, h, w, x.data_ptr(),
                                                                   L.stream_ptr()))
                    for b, (k, wi) in enumerate(la.rows):
                        exp = torch.cat([meds[la.row_median[b], ..., :3].cpu()] +
                                        [pix[k][wi + f][..., :3] for f in range(8)] +
                                        [torch.zeros((h, w, 5), dtype=torch.float16)], -1)
                        assert torch.equal(x[b].cpu().view(torch.int16), exp.view(torch.int16))
                mask = torch.zeros((nf, h, w), dtype=torch.uint8, device="cuda")
                ens = torch.zeros((nf, h, w), device="cuda")
                table = _i32([r + [rule] for r, rule in zip(la.refs, la.rule)])
                L.check(L.lib().pb_tracknet_ensemble_table(carry.data_ptr(), plan.carry_rows, fresh.data_ptr(),
                                                           table.data_ptr(), nf, h, w, 0.5, mask.data_ptr(),
                                                           ens.data_ptr(), L.stream_ptr()))
                fresh_np = fresh.cpu().numpy()
                for i, (refs, rule) in enumerate(zip(la.refs, la.rule)):
                    e = ensemble_table(carry_np, fresh_np, refs, rule)
                    assert np.array_equal(ens[i].cpu().numpy().view(np.uint32), e.view(np.uint32))
                    assert torch.equal(mask[i].cpu(), torch.from_numpy((e > 0.5).astype(np.uint8)))
                n_frames += nf
                if la.carry:  # a launch of no window (tails only) carries nothing
                    copies = _i32(la.carry)
                    L.check(L.lib().pb_tracknet_carry_rows(carry.data_ptr(), fresh.data_ptr(), copies.data_ptr(),
                                                           len(la.carry), h, w, L.stream_ptr()))
                for dst, src in la.carry:
                    carry_np[dst] = fresh_np[src]
                assert torch.equal(carry.cpu(), torch.from_numpy(carry_np))
    assert n_frames == sum(T for T in lengths if T >= 8)


# ---- stream_many against stream ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ckpts():
    return {"detect": OW.make_yolo("detect"), "pose13": OW.make_yolo("pose13", cls_mean=-5.5),
            "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet(), "inpaint": OI.make_inpaintnet()}


def _vi():
    return sv.VideoInfo(width=W, height=H, fps=30.0, total_frames=None)


@pytest.fixture(scope="module")
def trackers(ckpts):
    """the two tracker groups of test_stream_gpu: "yolo" (three YOLO trackers, the ball without InpaintNet) and "fixed"
    (players, a fixed court, the ball with InpaintNet)"""
    poly = sv.PolygonZone(np.array([[0, 0], [W - 1, 0], [W - 1, H - 1], [0, H - 1]]), frame_resolution_wh=(W, H))
    court = Keypoints([Keypoint(id=i, xy=(100.0 * i, 50.0 + i)) for i in range(12)])
    groups = {"yolo": [PlayerTracker(ckpts["detect"], poly, batch_size=B),
                       PlayerKeypointsTracker(ckpts["pose13"], 1280, batch_size=B, load_path=None, save_path=None),
                       KeypointsTracker(ckpts["court12"], batch_size=B, model_type="yolo"),
                       BallTracker(ckpts["tracknet"], None, batch_size=B, median_max_sample_num=M)],
              "fixed": [PlayerTracker(ckpts["detect"], poly, batch_size=B),
                        KeypointsTracker(None, batch_size=B, model_type="yolo", fixed_keypoints_detection=court),
                        BallTracker(ckpts["tracknet"], ckpts["inpaint"], batch_size=B, median_max_sample_num=M)]}
    for t in groups["yolo"] + groups["fixed"]:
        t.video_info_post_init(_vi())
    return groups


@pytest.fixture(scope="module")
def video():
    return synth.make_frames(T_LAT + 12, H, W, start=3)


def _ser(o):
    return json.dumps(o.serialize())


def _ball(tr):
    return next(t for t in tr if isinstance(t, BallTracker))


# per scenario: (stream key, first video frame, length) and how items are cut
SCENARIOS = {
    "round robin": ([("a", 0, 3 * B + 5), ("b", 2, B + 7), ("c", 5, 9), ("d", 1, 1)], "frames"),
    "bursts": ([("a", 4, 8), ("b", 0, 3 * B + 5), ("c", 3, 7), ("e", 0, 0), ("d", 6, B + 7)], "bursts"),
    "device batches of 3": ([("a", 1, 3 * B + 5), ("b", 7, B + 7), ("c", 0, 9)], "batches"),
}


def _scenario_items(video, streams, cut, rng):
    """(key, frames) items: round-robin over the open streams, "bursts" with random burst sizes, an explicit
    (key, None) for every second stream, and stream d opening only once a has ended"""
    left = {k: [video[o + i] for i in range(T)] for k, o, T in streams}
    order = [k for k, _, _ in streams]
    late = "d" if cut == "bursts" else None
    items, open_ = [], [k for k in order if k != late]
    i = 0
    while open_:
        k = open_[i % len(open_)]
        i += 1
        fr = left[k]
        if not fr:
            open_.remove(k)
            if order.index(k) % 2 == 0 or k == "e":
                items.append((k, None))
            if k == "a" and late:
                open_.append(late)
            continue
        n = {"frames": 1, "bursts": int(rng.integers(1, 6)), "batches": 3}[cut]
        take, left[k] = fr[:n], fr[n:]
        if cut == "frames":
            items.append((k, take[0].numpy()))
        elif cut == "bursts":
            items += [(k, f.numpy()) for f in take] if rng.random() < 0.5 else [(k, torch.stack(take))]
        else:
            items.append((k, torch.stack(take).cuda()))
    return items


@pytest.mark.parametrize("median", ["given", "taken"])
@pytest.mark.parametrize("which", ["yolo", "fixed"])
def test_stream_many_equals_stream_per_stream(trackers, video, which, median):
    """Every stream's yielded entries serialise exactly as `stream()`'s on that stream's frames alone (trackers
    restarted), and `stream_results[key]` equals the trackers' results after that stream (which are run()'s,
    InpaintNet included), for round-robin single frames, bursts with a stream opening after another ended, batches of
    3 device frames, and explicit ends mid-pass; the background given and taken from each stream."""
    tr = trackers[which]
    ball = _ball(tr)
    ball.median = None
    med = synth.make_median(H, W).numpy() if median == "given" else None
    cache = {}
    visible = players = False
    for name, (streams, cut) in SCENARIOS.items():
        exp = {}
        for k, o, T in streams:
            if (o, T) not in cache:
                for t in tr:
                    t.restart()
                got = {str(t): [] for t in tr}
                runner = TrackingRunner(tr, video_info=_vi())
                for f, entry in runner.stream(iter([video[o + i].numpy() for i in range(T)]), median=med):
                    for n_, obj in entry.items():
                        got[n_].append(_ser(obj))
                final = {str(t): [_ser(x) for x in t.results.predictions] for t in tr}
                cache[(o, T)] = (got, final)
            exp[k] = cache[(o, T)]
        for t in tr:
            t.restart()
        runner = TrackingRunner(tr, video_info=_vi())
        items = _scenario_items(video, streams, cut, np.random.default_rng(len(name)))
        got = collections.defaultdict(lambda: {str(t): [] for t in tr})
        meds = None if med is None else {k: med for k, _, _ in streams}
        for key, f, entry in runner.stream_many(iter(items), medians=meds, max_open=4):
            assert f == len(got[key]["ball_tracker"])
            for n_, obj in entry.items():
                got[key][n_].append(_ser(obj))
        for k, _, T in streams:
            assert got.get(k, {str(t): [] for t in tr}) == exp[k][0], (name, k)
            final = {n_: [_ser(x) for x in objs] for n_, objs in runner.stream_results.pop(k).items()}
            assert final == exp[k][1], (name, k)
            visible |= any('"visibility": 1' in s for s in final["ball_tracker"])
            players |= any(json.loads(s) for s in final["players_tracker"])
        assert not runner.stream_results
        assert all(len(t.results) == 0 for t in tr)
    assert visible, "vacuous: no visible ball"
    assert players, "vacuous: no tracked player"


@pytest.mark.parametrize("held", [False, True])
def test_stream_many_latency_bound(trackers, video, held):
    """Three streams of 8B + 16 frames pulled round-robin one host frame at a time, stream b ended explicitly first:
    the entry (s, f) is yielded before the (k + 2B)-th frame is pulled, k the pull of s's frame f + 7, and each
    stream's last 7 entries before the (B + 1)-th frame pulled after its end item.  held: stream c has no background
    and holds its first 3B + 5 frames for it while a and b run; the bound holds for a and b throughout, and for c once
    its background exists."""
    tr = trackers["yolo"]
    for t in tr:
        t.restart()
    ball = _ball(tr)
    hold = 3 * B + 5
    ball.median, ball.median_max_sample_num = None, hold
    med = synth.make_median(H, W).numpy()
    lens = {"a": T_LAT, "b": T_LAT - 12, "c": T_LAT}
    sent = {k: 0 for k in lens}
    pulled = [0]
    pull_of = {}  # (key, frame) -> its 1-based pull count; (key, "end") -> frames pulled when its end item is pulled

    def items():
        while any(sent[k] < T for k, T in lens.items()):
            for k, T in lens.items():
                if sent[k] < T:
                    pulled[0] += 1
                    pull_of[(k, sent[k])] = pulled[0]
                    yield k, video[sent[k] + 3 * " abc".index(k)].numpy()
                    sent[k] += 1
                    if sent[k] == T and k == "b":
                        pull_of[(k, "end")] = pulled[0]
                        yield k, None
        for k in lens:
            pull_of.setdefault((k, "end"), pulled[0])

    medians = {k: med for k in lens if not (held and k == "c")}
    at = {}
    try:
        for key, f, _ in TrackingRunner(tr, video_info=_vi()).stream_many(items(), medians=medians):
            at[(key, f)] = pulled[0]
    finally:
        ball.median_max_sample_num = M
    assert sorted(at) == sorted((k, f) for k, T in lens.items() for f in range(T))
    bg = {k: pull_of[(k, hold - 1)] if k not in medians else 0 for k in lens}  # the pull after which it exists
    checked = 0
    for (k, f), p in at.items():
        if f + 7 < lens[k]:
            if pull_of[(k, f + 7)] > bg[k]:
                assert p < pull_of[(k, f + 7)] + 2 * B, (k, f, p)
                checked += 1
        else:
            assert p <= pull_of[(k, "end")] + B, (k, f, p)
    assert checked >= 2 * (6 * B + 8) + (0 if held else 6 * B + 8), "vacuous: too few frames under the bound"
