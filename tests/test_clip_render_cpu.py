"""CPU: the clip-list render pass's host side.  `plan_clip_render` replayed over random clip lists, and
`write_clip_batches` driving real writer threads over a fake encoder that sleeps a random time per frame."""
import queue
import random
import threading
import time

import numpy as np
import pytest

from padel_analytics_b200 import render as R


def _random_lengths(rng):
    n = rng.randint(1, 20)
    out = []
    while len(out) < n:
        if rng.random() < 0.3:  # a run of clips shorter than a batch, empty ones included
            out += [rng.randint(0, 5) for _ in range(rng.randint(2, 12))]
        else:
            out.append(rng.randint(0, 140))
    return out


def _cases(count, seed, max_len=None):
    rng = random.Random(seed)
    cases = [([5, 8, 9, 40, 77, 130], 32, 4), ([5, 8, 9, 40, 77, 130], 8, 4), ([0, 0, 0], 4, 4), ([1] * 70, 32, 4),
             ([3, 0, 1], 1, 1)]
    while len(cases) < count:
        lengths = _random_lengths(rng)
        if max_len is not None:
            lengths = [min(t, max_len) for t in lengths]
        cases.append((lengths, rng.randint(1, 32), rng.choice([1, 2, 3, 4])))
    return cases


def _check_plan(lengths, B, max_open):
    plan = R.plan_clip_render(lengths, B, max_open)
    assert all(len(b.rows) == B for b in plan[:-1]) and (not plan or 0 < len(plan[-1].rows) <= B)
    rows = [r for b in plan for r in b.rows]
    assert rows == [(c, f) for c, T in enumerate(lengths) for f in range(T)]  # every frame once, in order
    got = {c: [] for c in range(len(lengths))}
    state = {}  # clip -> "open" / "finished" / "closed"; writers close as late as the plan allows
    for b in plan:
        assert b.parts, "a batch whose slot no writer would release"
        assert [p.lo for p in b.parts] == [0] + [p.hi for p in b.parts[:-1]] and b.parts[-1].hi == len(b.rows)
        assert len({p.clip for p in b.parts}) == len(b.parts)  # one part per clip: the slot is released len(parts) times
        for p in b.parts:
            assert p.lo < p.hi and b.rows[p.lo:p.hi] == [(p.clip, p.first + j) for j in range(p.hi - p.lo)]
            assert p.open == (p.first == 0) and p.close == (p.first + p.hi - p.lo == lengths[p.clip])
            if p.open:
                assert p.clip not in state
                if p.wait is not None:
                    assert state[p.wait] in ("finished", "closed"), "waiting on a writer that still takes frames"
                    state[p.wait] = "closed"
                state[p.clip] = "open"
                assert sum(s != "closed" for s in state.values()) <= max_open
            else:
                assert p.wait is None and state[p.clip] == "open"
            got[p.clip] += [f for _, f in b.rows[p.lo:p.hi]]
            if p.close:
                state[p.clip] = "finished"
    assert all(got[c] == list(range(T)) for c, T in enumerate(lengths))  # each writer gets its clip's frames
    assert set(state) == {c for c, T in enumerate(lengths) if T} and "open" not in state.values()
    return plan


@pytest.mark.parametrize("seed", range(4))
def test_plan_clip_render_replayed_over_random_clip_lists(seed):
    spans = 0
    for lengths, B, max_open in _cases(100, seed):
        plan = _check_plan(lengths, B, max_open)
        spans += sum(len(b.parts) > 1 for b in plan)
    assert spans, "vacuous: no batch spans two clips"


def test_plan_clip_render_packs_batches_across_clips():
    plan = R.plan_clip_render([5, 8, 9, 40], 32)
    assert [(p.clip, p.lo, p.hi) for p in plan[0].parts] == [(0, 0, 5), (1, 5, 13), (2, 13, 22), (3, 22, 32)]
    assert [p.close for p in plan[0].parts] == [True, True, True, False]
    assert R.plan_clip_render([0, 0], 8) == []
    with pytest.raises(ValueError):
        R.plan_clip_render([3], 0)


class _FakeEncoder:
    """cv2.VideoWriter stand-in: sleeps a random time per frame and records what it was given."""
    lock = threading.Lock()
    opened = {}  # path -> (fps, size, frames, released)
    live = 0
    peak = 0
    fail_path = None

    def __init__(self, path, fourcc, fps, size):
        self.path, self.rng = path, random.Random(path)
        with self.lock:
            assert path not in self.opened
            self.opened[path] = [fps, size, [], False]
            type(self).live += 1
            type(self).peak = max(type(self).peak, type(self).live)

    def isOpened(self):
        return True

    def write(self, f):
        time.sleep(self.rng.random() * 3e-4)
        if self.path == self.fail_path:
            raise RuntimeError("encoder failed")
        self.opened[self.path][2].append(tuple(int(v) for v in f))  # copied now: a reused slot would show here

    def release(self):
        with self.lock:
            self.opened[self.path][3] = True
            type(self).live -= 1


@pytest.fixture
def fake_encoder(monkeypatch):
    import cv2

    monkeypatch.setattr(cv2, "VideoWriter", _FakeEncoder)
    _FakeEncoder.opened, _FakeEncoder.live, _FakeEncoder.peak, _FakeEncoder.fail_path = {}, 0, 0, None
    return _FakeEncoder


def _route(plan, B, fps_of, slots=3, frames=None):
    """Renders `plan` the way OverlayRenderer.run hands out batches (a slot is taken from the queue before each
    batch is filled) and writes it through write_clip_batches.  frames: the first `frames` rows only, as a source
    that ends early leaves them."""
    free = queue.Queue()
    for s in range(slots):
        free.put(s)
    out = [np.full((B, 2), -1, np.int64) for _ in range(slots)]

    def batches():
        left = sum(len(b.rows) for b in plan) if frames is None else frames
        for b in plan:
            if left <= 0:
                return
            slot = free.get(timeout=30)  # a slot that is never released fails here instead of hanging
            buf = out[slot][:min(len(b.rows), left)]
            buf[:] = b.rows[:len(buf)]
            left -= len(buf)
            yield buf, slot

    def open_writer(c, release):
        return R.VideoWriterThread(f"clip{c}", fps_of(c), (1920, 1080), release)

    secs = R.write_clip_batches(plan, batches(), open_writer, free)
    assert sorted(free.get_nowait() for _ in range(slots)) == list(range(slots)) and free.empty()
    return secs


@pytest.mark.parametrize("seed", range(2))
def test_write_clip_batches_routes_each_clip_to_its_writer(seed, fake_encoder):
    for lengths, B, max_open in _cases(14, 100 + seed, max_len=48):
        fake_encoder.opened, fake_encoder.peak = {}, 0
        plan = R.plan_clip_render(lengths, B, max_open)
        secs = _route(plan, B, lambda c: 20.0 + c)
        assert secs >= 0
        assert fake_encoder.live == 0 and fake_encoder.peak <= max_open
        assert set(fake_encoder.opened) == {f"clip{c}" for c, T in enumerate(lengths) if T}
        for c, T in enumerate(lengths):
            if T:
                fps, size, frames, released = fake_encoder.opened[f"clip{c}"]
                assert (fps, size, released) == (20.0 + c, (1920, 1080), True)
                assert frames == [(c, f) for f in range(T)], (lengths, B, c)


def test_write_clip_batches_raises_a_writer_error_after_joining_every_writer(fake_encoder):
    lengths = [5, 8, 9, 40, 2, 2, 2, 30]
    fake_encoder.fail_path = "clip2"
    before = threading.active_count()
    with pytest.raises(RuntimeError, match="encoder failed"):
        _route(R.plan_clip_render(lengths, 8, 2), 8, lambda c: 25.0)
    assert threading.active_count() == before
    assert fake_encoder.live == 0
    assert fake_encoder.opened["clip7"][2] == [(7, f) for f in range(30)]  # the other clips are still written


def test_write_clip_batches_ends_the_writers_where_the_frames_end(fake_encoder):
    lengths = [5, 8, 9, 40]
    for got in (3, 13, 16, 30, 61):
        fake_encoder.opened = {}
        _route(R.plan_clip_render(lengths, 8, 2), 8, lambda c: 25.0, frames=got)
        assert fake_encoder.live == 0
        rows = [(c, f) for c, T in enumerate(lengths) for f in range(T)][:got]
        assert set(fake_encoder.opened) == {f"clip{c}" for c, _ in rows}  # no writer for a clip that got no frame
        for c in {c for c, _ in rows}:
            assert fake_encoder.opened[f"clip{c}"][2:] == [[r for r in rows if r[0] == c], True]
    with pytest.raises(ValueError, match="more than the plan"):
        R.write_clip_batches(R.plan_clip_render([3], 8), iter([(np.zeros((4, 2)), 0)]), None, queue.Queue())
