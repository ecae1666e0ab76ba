"""Tracking several live streams in one pass, without a GPU: the multi-stream ball planner's tables replayed through a
restatement of the table kernels against each stream's single-stream ensemble, the planner's invariants, the
interleaving of items into upload chunks, the per-stream merge and host state, and the refusals of `stream_many`."""
import collections

import numpy as np
import pytest
import torch

from oracle import tracknet as OT
from padel_analytics_b200.engine.stream_plan import CARRY, StreamPlanner
from padel_analytics_b200.trackers import BallTracker, KeypointsTracker, TrackingRunner
from padel_analytics_b200.trackers import sv_compat as sv
from padel_analytics_b200.trackers.keypoints_tracker import Keypoint, Keypoints
from padel_analytics_b200.trackers.runner import StreamMux, StreamsPass
from padel_analytics_b200.trackers.tracker import TrackingResults

VI = sv.VideoInfo(width=8, height=6, fps=30.0, total_frames=None)
COURT = Keypoints([Keypoint(id=i, xy=(10 * i, 20 + i)) for i in range(12)])
H, W = 4, 8


def ensemble_table(carry, fresh, refs, rule):
    """numpy restatement of pb_tracknet_ensemble_table for one frame: mul then add in k order, or sum then divide"""
    acc = np.zeros(carry.shape[-2:], np.float32)
    for k in range(8):
        r = refs[k]
        if r < 0:
            continue
        row = carry[r] if r < len(carry) else fresh[r - len(carry)]
        if rule == 0:
            acc = acc + row[7 - k] * (np.float32(k + 1 if k < 4 else 8 - k) / np.float32(20))
        else:
            acc = acc + row[7 - k]
    return acc if rule == 0 else acc / np.float32(rule)


def _frame(key, f):
    """a 1x1 frame that names its stream and index (key < 256, f < 65536)"""
    return np.array([[[key, f % 256, f // 256]]], np.uint8)


def _interleaving(rng, lengths, max_open):
    """(key, frames) items: streams opened in key order while fewer than max_open are open, frames pulled from a
    random open stream in single frames or small bursts, each stream ended by (key, None) or by the iterable's end"""
    items, nxt, sent, open_ = [], 0, {}, []
    quiet = int(rng.integers(0, len(lengths)))  # this stream is ended by the iterable's end
    while nxt < len(lengths) or open_:
        if nxt < len(lengths) and len(open_) < max_open and (not open_ or rng.random() < 0.3):
            open_.append(nxt)
            sent[nxt] = 0
            nxt += 1
            continue
        k = open_[int(rng.integers(0, len(open_)))]
        T = lengths[k]
        if sent[k] == T:
            if k == quiet:
                if len(open_) == 1 and nxt == len(lengths):
                    break
                continue
            items.append((k, None))
            open_.remove(k)
            continue
        n = min(T - sent[k], int(rng.integers(1, 4)) if rng.random() < 0.3 else 1)
        if n == 1 and rng.random() < 0.5:
            items.append((k, _frame(k, sent[k])))
        else:
            items.append((k, np.stack([_frame(k, f) for f in range(sent[k], sent[k] + n)])))
        sent[k] += n
    return items


def _replay(items, B, max_open):
    """items -> StreamMux -> StreamPlanner; the tables checked against the pool contents they name, and replayed over
    random heat-maps.  Returns ({key: [(frame, ensemble, frames of the stream pushed then)]}, the heat-maps)."""
    mux = StreamMux(items, B, max_open, hold_device="cpu")
    plan = StreamPlanner(B, max_open)
    heat, emitted = {}, collections.defaultdict(list)
    pool = [None] * plan.n_slots  # (key, frame) per slot
    carry = np.zeros((plan.carry_rows, 8, H, W), np.float32)
    carried = [None] * plan.carry_rows  # (key, window) per carry row
    pushed = collections.Counter()
    rng = np.random.default_rng(7)

    def run(meta):
        runs, ends = meta
        off = 0
        st = plan.step([(k, n) for k, _, n in runs], ends)
        chunk = [(k, f0 + i) for k, f0, n in runs for i in range(n)]
        assert [p[0] for p in st.pushes] == sorted(p[0] for p in st.pushes)
        for o, n, slot in st.pushes:
            assert slot + n <= plan.n_slots
            for i in range(n):
                assert pool[slot + i] is None, "a slot reused while its frame is still read"
                pool[slot + i] = chunk[o + i]
            off += n
        assert off == len(chunk)
        for key, _, n in runs:
            pushed[key] += n
        for launch in st.launches:
            assert len(launch.rows) <= B and len(launch.frames) <= plan.max_frames
            fresh = []
            for (key, w), slots, med in zip(launch.rows, launch.row_slots, launch.row_median):
                assert [pool[s] for s in slots] == [(key, w + f) for f in range(8)]
                assert med == plan.streams[key].lane if key in plan.streams else True
                if key not in heat:
                    heat[key] = rng.random((64, 8, H, W), dtype=np.float32)
                    heat[key].reshape(-1)[::7] = 0.5
                fresh.append(heat[key][w])
            for (key, n), refs, rule in zip(launch.frames, launch.refs, launch.rule):
                for k, r in enumerate(refs):
                    if 0 <= r < plan.carry_rows:
                        assert carried[r] == (key, n - 7 + k), "a carry row that does not hold the window read"
                    elif r >= plan.carry_rows:
                        assert launch.rows[r - plan.carry_rows] == (key, n - 7 + k)
                emitted[key].append((n, ensemble_table(carry, fresh, refs, rule), pushed[key]))
            for dst, src in launch.carry:
                carry[dst] = fresh[src]
                carried[dst] = launch.rows[src]
        for s in st.frees:
            pool[s] = None
        # no ready window held back, and the pool holds at most 7 frames per open stream
        for key, s in plan.streams.items():
            assert s.n_win == max(0, s.n_in - CARRY)
        assert sum(p is not None for p in pool) <= CARRY * len(plan.streams)

    for _ in mux.pieces():
        while mux.metas:
            run(mux.metas.popleft())
    while mux.metas:
        run(mux.metas.popleft())
    assert not plan.streams and all(p is None for p in pool)
    return emitted, heat


@pytest.mark.parametrize("B", [1, 3, 4, 8])
@pytest.mark.parametrize("seed", range(4))
def test_planner_tables_equal_each_streams_single_stream_ensemble(B, seed):
    """Random interleavings of streams of 0-40 frames (including 0, 1, 7, 8 and 9) opening and ending mid-pass with
    max_open reached: every frame of every stream of >= 8 frames is emitted exactly once, in order, none before its
    frame + 7 was pushed (but at the end), and its value equals the single-stream ensemble over that stream's windows
    alone, bit for bit; the rows read the slots that hold their frames, the carry rows hold the windows read."""
    rng = np.random.default_rng(seed * 10 + B)
    lengths = [0, 1, 7, 8, 9] + [int(v) for v in rng.integers(0, 41, 5)]
    rng.shuffle(lengths)
    max_open = 3
    items = _interleaving(rng, lengths, max_open)
    emitted, heat = _replay(items, B, max_open)
    for key, T in enumerate(lengths):
        got = emitted.get(key, [])
        if T < 8:
            assert got == []
            continue
        assert [n for n, _, _ in got] == list(range(T)), (key, T)
        exp = OT.ensemble_reference_loop(torch.from_numpy(heat[key][:T - 7]), T, B).numpy()
        for n, e, at in got:
            assert np.array_equal(e.view(np.uint32), exp[n].view(np.uint32)), (key, T, n)
            assert at >= min(n + 8, T), "a frame emitted before its frame + 7 was pushed"


def test_planner_reaches_max_open_and_the_slot_bound():
    """max_open streams fed round-robin one frame at a time with a batch of B: the live slots reach 7 per stream plus
    the chunk, the bound the pool is sized for, and never more."""
    B, S = 4, 5
    plan = StreamPlanner(B, S)
    peak = 0
    for r in range(30):
        for c in range(S // B + 1):
            keys = [(r * S + i) % S for i in range(c * B, min(S, (c + 1) * B))]
            if not keys:
                continue
            free_before = len(plan._free)
            st = plan.step([(k, 1) for k in keys], [])
            peak = max(peak, plan.n_slots - free_before + len(keys))
            assert len(st.launches) <= 1
    assert peak <= plan.n_slots == CARRY * S + B
    assert peak >= CARRY * S
    with pytest.raises(AssertionError, match="streams in the pass"):
        plan.step([("new", 1)], [])


def test_holding_streams_enter_the_pass_after_their_background():
    """A stream without a background is held for `hold` frames (or until its end), and enters the pass in order after
    its background is taken; the streams around it keep running."""
    taken = []
    items = [("a", _frame(1, 0)), ("b", _frame(2, 0)), ("a", _frame(1, 1)), ("b", _frame(2, 1)), ("a", _frame(1, 2)),
             ("b", _frame(2, 2)), ("c", _frame(3, 0)), ("c", None)]
    mux = StreamMux(items, 2, 4, medians={"b": "given"}, hold=3, background=lambda held: taken.append(len(held)) or "m",
                    hold_device="cpu")
    out = []
    for p in mux.pieces():
        out.append(None if p is None else tuple(int(v) for v in p[:, 0, 0, 0]))
    # a held frame counts as a pull: b's frames do not wait for a second frame of b while a is held
    assert out == [(2,), None, (2,), None, (1,), (1,), (1,), (2,), (3,), None, None]
    assert taken == [3, 1] and mux.medians == {"a": "m", "b": "given", "c": "m"}
    assert list(mux.metas) == [([("b", 0, 1)], []), ([("b", 1, 1)], []), ([("a", 0, 1), ("a", 1, 1)], []),
                               ([("a", 2, 1), ("b", 2, 1)], []), ([("c", 0, 1)], ["c"]), ([], ["a", "b"])]


# ---- stream_many with stub trackers ----------------------------------------------------------------------------------
def _stub(cls, **attrs):
    t = object.__new__(cls)  # no CUDA here: skip the engine construction, set what is read
    t.results, t.load_path, t.save_path = TrackingResults(), None, None
    for k, v in attrs.items():
        setattr(t, k, v)
    return t


def _court(**kw):
    return _stub(KeypointsTracker, **{"model_type": "yolo", "model": None, "fixed_keypoints_detection": COURT, **kw})


def test_stream_many_merges_each_stream_in_order_and_stores_its_results(tmp_path):
    """Fixed detections need no device: each stream's entries come in frame order as its frames are pulled, the
    results of a stream are in `stream_results` before its last entry is yielded, a stream of no frame gets empty
    results, and the tracker's own results and save_path are left alone."""
    court = _court(save_path=str(tmp_path / "court.json"))
    runner = TrackingRunner([court], video_info=VI)
    frame = np.zeros((6, 8, 3), np.uint8)
    items = [("a", frame), ("b", frame), ("a", torch.zeros((3, 6, 8, 3), dtype=torch.uint8)), ("e", None),
             ("b", None), ("c", frame), ("a", frame)]
    seen = []
    for key, f, entry in runner.stream_many(iter(items)):
        assert entry == {"keypoints_tracker": COURT}
        seen.append((key, f))
        if (key, f) == ("b", 0):
            assert "b" not in runner.stream_results
    assert seen == [("a", 0), ("b", 0), ("a", 1), ("a", 2), ("a", 3), ("c", 0), ("a", 4)]
    assert runner.stream_results == {"a": {"keypoints_tracker": [COURT] * 5}, "b": {"keypoints_tracker": [COURT]},
                                     "c": {"keypoints_tracker": [COURT]}, "e": {"keypoints_tracker": []}}
    assert len(court.results) == 0 and not (tmp_path / "court.json").exists()


def test_stream_many_refusals(monkeypatch):
    pulled = []

    def items():
        for k in ("a", "b"):
            pulled.append(k)
            yield k, np.zeros((6, 8, 3), np.uint8)

    regressor = _stub(KeypointsTracker, model_type="resnet", model=object(), fixed_keypoints_detection=None)
    with pytest.raises(ValueError, match="keypoints_tracker"):
        TrackingRunner([regressor], video_info=VI).stream_many(items())
    cached = _stub(BallTracker)
    cached.results.load([object()] * 3)
    with pytest.raises(ValueError, match=r"ball_tracker.*cached predictions"):
        TrackingRunner([_court(), cached], video_info=VI).stream_many(items())
    with pytest.raises(ValueError, match="video_info"):
        TrackingRunner([_court()]).stream_many(items())
    import torch.distributed as dist

    with monkeypatch.context() as m:
        m.setattr(dist, "is_available", lambda: True)
        m.setattr(dist, "is_initialized", lambda: True)
        m.setattr(dist, "get_world_size", lambda: 2)
        with pytest.raises(ValueError, match="world size 2"):
            TrackingRunner([_court()], video_info=VI).stream_many(items())
    assert not pulled, "a refused call must not pull an item"

    runner = TrackingRunner([_court()], video_info=VI)
    f = np.zeros((6, 8, 3), np.uint8)
    with pytest.raises(ValueError, match="stream 'b'.*same frame size"):
        list(runner.stream_many(iter([("a", f), ("b", np.zeros((6, 9, 3), np.uint8))])))
    with pytest.raises(ValueError, match="'a' appears again"):
        list(runner.stream_many(iter([("a", f), ("a", None), ("a", f)])))
    with pytest.raises(ValueError, match="'a' appears again"):
        list(runner.stream_many(iter([("a", None), ("a", None)])))
    with pytest.raises(ValueError, match="max_open is 2"):
        list(runner.stream_many(iter([("a", f), ("b", f), ("c", f)]), max_open=2))
    ok = list(runner.stream_many(iter([("a", f), ("b", f), ("a", None), ("c", f)]), max_open=2))
    assert [(k, i) for k, i, _ in ok] == [("a", 0), ("b", 0), ("c", 0)]


class _Counter:
    """A stub YOLO tracker whose post-processing numbers the frames it has seen since `video_info_post_init`: its
    results tell which host state each run used."""
    stage = "detect"

    def video_info_post_init(self, vi):
        self.byte_track = [0]

    def postprocess(self, res, hw):
        out = []
        for r in res:
            self.byte_track = self.byte_track + [r]
            out.append(len(self.byte_track) - 1)
        return out


def test_streams_pass_runs_each_streams_host_stage_with_its_own_state():
    """Runs of several streams in one batch are post-processed in pull order, each with its stream's own state, fresh
    at the stream's first frame and dropped at its end."""
    t = _Counter()
    sp = object.__new__(StreamsPass)
    sp.hw, sp.video_info, sp.host = (6, 8), VI, {}
    meta1 = ([("a", 0, 2), ("b", 0, 1), ("a", 2, 1)], [])
    meta2 = ([("b", 1, 2), ("a", 3, 1)], ["b"])
    (_, out1) = sp._finish(([("p", t, lambda: ["a0", "a1", "b0", "a2"])], meta1))
    (_, out2) = sp._finish(([("p", t, lambda: ["b1", "b2", "a3"])], meta2))
    assert out1 == {"p": [("a", 0, [1, 2]), ("b", 0, [1]), ("a", 2, [3])]}
    assert out2 == {"p": [("b", 1, [2, 3]), ("a", 3, [4])]}
    assert sp.host["a"]["p"]["byte_track"] == [0, "a0", "a1", "a2", "a3"] and "b" not in sp.host


def _yield_pulls(items, B, hold, given):
    """Replays the mux under a pass with one chunk of look-ahead, as `FusedPass.run` runs: chunk i's results are
    yielded once chunk i + 1 has closed (or the items ended).  Entry (s, f) is final in the chunk that holds s's frame
    f + 7, or the one that ends s.  Returns ({(s, f): frames pulled when it is yielded}, {(s, f): the 1-based pull of
    s's frame f}, {s: frames pulled when its end item was pulled}, {s: frames pulled when its background existed})."""
    pulled, pull_of, end_at, sent = [0], {}, {}, collections.Counter()

    def counted():
        for key, it in items:
            if it is None:
                end_at[key] = pulled[0]
            else:  # an item is pulled whole: each of its frames counts as pulled with its last
                n = it.shape[0] if it.ndim == 4 else 1
                pulled[0] += n
                for _ in range(n):
                    pull_of[(key, sent[key])] = pulled[0]
                    sent[key] += 1
            yield key, it

    mux = StreamMux(counted(), B, 8, medians={k: "given" for k in given}, hold=hold,
                    background=lambda held: "taken", hold_device="cpu")
    closes, n, bg_at = [], 0, {k: 0 for k in given}
    for p in mux.pieces():
        for k in mux.medians:
            bg_at.setdefault(k, pulled[0])
        n += 0 if p is None else p.shape[0]
        assert n <= B
        if p is None or n == B:
            closes.append(pulled[0])
            n = 0
    assert n == 0 and len(closes) == len(mux.metas)
    final, count = {}, collections.Counter()  # entry -> chunk in which it is final
    for i, (runs, ends) in enumerate(mux.metas):
        for key, f0, m in runs:
            for f in range(f0, f0 + m):
                if f >= 7:
                    final[(key, f - 7)] = i
            count[key] = f0 + m
        for key in ends:
            for f in range(max(0, count[key] - 7), count[key]):
                final[(key, f)] = i
    for key in sent:
        end_at.setdefault(key, pulled[0])
    at = {e: closes[i + 1] if i + 1 < len(closes) else pulled[0] for e, i in final.items()}
    return at, pull_of, end_at, bg_at


@pytest.mark.parametrize("B", [1, 4, 8])
@pytest.mark.parametrize("seed", range(3))
def test_latency_bound_holds_while_other_streams_are_held(B, seed):
    """Streams with a given background run beside streams held for theirs (20 frames): the entry (s, f) is yielded
    before the (k + 2B)-th pull, k the pull of s's frame f + 7, whenever s's background existed by then, and a
    stream's last entries no later than B pulls after its end item, in round-robin single frames and random bursts
    (an item of n frames is pulled whole, which moves both bounds by up to n - 1)."""
    rng = np.random.default_rng(seed)
    lengths = [int(v) for v in rng.integers(9, 60, 5)]
    given = [0, 2, 4]
    for burst in (False, True):
        items, sent, live = [], [0] * 5, list(range(5))
        while live:
            k = live[int(rng.integers(0, len(live)))] if burst else live[0]
            n = min(lengths[k] - sent[k], int(rng.integers(1, 4)) if burst else 1)
            items.append((k, np.stack([_frame(k, f) for f in range(sent[k], sent[k] + n)]) if n > 1
                          else _frame(k, sent[k])))
            sent[k] += n
            if sent[k] == lengths[k]:
                live.remove(k)
                if k in (1, 2):
                    items.append((k, None))
            elif not burst:
                live.append(live.pop(0))
        at, pull_of, end_at, bg_at = _yield_pulls(items, B, 20, given)
        slack = 2 if burst else 0
        checked = 0
        for (k, f), p in at.items():
            if f + 7 < lengths[k]:
                if pull_of[(k, f + 7)] > bg_at[k]:
                    assert p < pull_of[(k, f + 7)] + 2 * B + slack, (burst, k, f, p)
                    checked += 1
            else:
                assert p <= end_at[k] + B + slack, (burst, k, f, p)
        assert checked >= 20, "vacuous"
