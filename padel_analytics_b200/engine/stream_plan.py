"""Batch planning for the ball pipeline over several interleaved live streams (pure Python, no device).

Frames of several streams arrive interleaved, in upload chunks of at most `batch` frames, and a stream's length is
known only when it ends.  A TrackNet window is 8 consecutive frames of ONE stream, so the windows of one device batch
are not numbered consecutively and each stream carries its own last 7 windows.  Three device pools replace the
single-stream ring and 7-row carry:

  slot pool    resized frames.  A pushed frame takes a free slot; the slot is freed once the last window that reads
               the frame has been launched (window f for frame f, the stream's last window for its last 7 frames).
  carry pool   7 heat-map rows per open stream: window w of the stream on lane l lives in carry row 7 l + w % 7.
  median pool  one background per open stream, in slot l.

A stream takes a lane (its carry rows and median slot) when its first frame is pushed and gives it back after the step
that ends it.

Each step runs every window that has become computable, in batches of up to `batch` windows, as
`BallPipeline.run_ready_async` does for one stream, so no ready window waits for a later step.  A window emits its own
frame; the step that ends a stream also emits the stream's 7 tail frames, from its last batch or, when no window of
any stream is ready, from a launch of no window that reads the carry pool alone.  Streams shorter than 8 frames have no
window and emit nothing.

Slot bound: after a step every open stream holds at most 7 frames (those of its windows not run yet: all ready windows
ran, so frames n-7..n-1 of a stream of n frames), an ended stream none, and a step pushes at most `batch` frames.  So
7 * max_open + batch slots never run out (`StreamPlanner.n_slots`).
"""
from __future__ import annotations

from dataclasses import dataclass, field

WINDOW = 8
CARRY = WINDOW - 1


def ensemble_rule(n: int, total_windows: int | None) -> tuple[list, int]:
    """The ensemble of frame n of a stream of `total_windows` windows (None: the stream has not ended, and window n
    exists): ([window read at k, or None when it does not exist, for k = 0..7], divisor), divisor 0 for the weighted
    sum of windows n-7..n and d > 0 for the head/tail mean (ball_tracker.py:449-509)."""
    ws = [n - CARRY + k for k in range(WINDOW)]
    if n >= CARRY and (total_windows is None or n < total_windows):
        return ws, 0
    if total_windows is None or n < total_windows:
        return [w if w >= 0 else None for w in ws], n + 1
    return [w if 0 <= w < total_windows else None for w in ws], WINDOW - (n - (total_windows - 1))


@dataclass
class StreamLaunch:
    """One device launch.  Row b runs window `rows[b]` = (stream key, window): its frames are pool slots
    `row_slots[b]` (8), its background median slot `row_median[b]`.  It emits `frames` = (key, frame), frame i
    ensembled from heat-map rows `refs[i]` (8; -1 absent, < carry_rows a carry row, else carry_rows + the batch row)
    by `rule[i]` (0: weighted sum, d > 0: sum / d).  After the ensemble, `carry` = [(carry row, batch row)] keeps each
    stream's newest windows."""
    rows: list = field(default_factory=list)
    row_slots: list = field(default_factory=list)
    row_median: list = field(default_factory=list)
    frames: list = field(default_factory=list)
    refs: list = field(default_factory=list)
    rule: list = field(default_factory=list)
    carry: list = field(default_factory=list)


@dataclass
class StreamStep:
    """What to enqueue for one upload chunk, in order: load `medians` = (key, median slot) for the streams that start,
    resize `pushes` = (offset, n, slot): chunk frames [offset, offset + n) into pool slots slot .. slot + n - 1, run
    `launches`.  `frees`: the slots free again after the launches; `ended`: the streams that ended."""
    medians: list = field(default_factory=list)
    pushes: list = field(default_factory=list)
    launches: list = field(default_factory=list)
    frees: list = field(default_factory=list)
    ended: list = field(default_factory=list)


class _Stream:
    def __init__(self, lane: int):
        self.lane = lane
        self.n_in = 0  # frames pushed
        self.n_win = 0  # windows run
        self.slot = {}  # frame -> pool slot, for the frames still held


class StreamPlanner:
    """Plans the ball pipeline's steps over interleaved streams: `step(segments, ends)` per upload chunk."""

    def __init__(self, batch: int, max_open: int):
        if batch < 1 or max_open < 1:
            raise ValueError("batch and max_open must be >= 1")
        self.batch, self.max_open = batch, max_open
        self.carry_rows = CARRY * max_open
        self.n_slots = CARRY * max_open + batch  # the slot bound of the module docstring
        self.max_frames = batch + CARRY * max_open  # a launch emits its windows' frames and the ending streams' tails
        self._free = list(range(self.n_slots))  # sorted
        self._lanes = list(range(max_open))
        self.streams: dict = {}

    def _alloc(self, n: int) -> list[int]:
        """n free slots: the first run of n consecutive free slots (one resize), else the n lowest."""
        if n == 0:
            return []
        if n > len(self._free):
            raise AssertionError(f"slot pool: {n} frames, {len(self._free)} free slots")
        free = self._free
        for i in range(len(free) - n + 1):
            if free[i + n - 1] - free[i] == n - 1:
                got = free[i:i + n]
                del free[i:i + n]
                return got
        got = free[:n]
        del free[:n]
        return got

    def step(self, segments: list, ends: list) -> StreamStep:
        """segments: [(key, n)]: the chunk's frames, in order, as runs of n consecutive frames of stream `key`; ends:
        the streams that end after this chunk's frames (a key that never pushed a frame is ignored)."""
        st = StreamStep()
        slots = self._alloc(sum(n for _, n in segments))
        off = 0
        for key, n in segments:
            s = self.streams.get(key)
            if s is None:
                if not self._lanes:
                    raise AssertionError(f"more than {self.max_open} streams in the pass")
                s = self.streams[key] = _Stream(self._lanes.pop(0))
                st.medians.append((key, s.lane))
            for i in range(n):
                s.slot[s.n_in] = slots[off + i]
                s.n_in += 1
            off += n
        for i, slot in enumerate(slots):  # resize runs: consecutive chunk frames into consecutive slots
            if st.pushes and st.pushes[-1][2] + st.pushes[-1][1] == slot:
                st.pushes[-1][1] += 1
            else:
                st.pushes.append([i, 1, slot])
        st.pushes = [tuple(p) for p in st.pushes]
        ends = [k for k in ends if k in self.streams]  # a stream that pushed no frame has nothing to end
        ready = [(key, w) for key, s in self.streams.items() for w in range(s.n_win, s.n_in - CARRY)]
        tails = [k for k in ends if self.streams[k].n_in >= WINDOW]
        batches = [ready[i:i + self.batch] for i in range(0, len(ready), self.batch)]
        if not batches and tails:
            batches = [[]]  # the tails alone, from the carry pool
        for i, rows in enumerate(batches):
            st.launches.append(self._launch(rows, tails if i == len(batches) - 1 else [], set(ends)))
        for key, s in self.streams.items():
            done = s.n_in if key in ends else s.n_win  # frame f's last window is window f
            for f in [f for f in s.slot if f < done]:
                st.frees.append(s.slot.pop(f))
        for key in ends:
            self._lanes.append(self.streams.pop(key).lane)
            st.ended.append(key)
        self._lanes.sort()
        self._free = sorted(self._free + st.frees)
        return st

    def _launch(self, rows: list, tails: list, ending: set) -> StreamLaunch:
        L = StreamLaunch(rows=list(rows))
        row_of = {}
        first_new = {}
        for b, (key, w) in enumerate(rows):
            s = self.streams[key]
            row_of[(key, w)] = b
            first_new.setdefault(key, w)
            L.row_slots.append([s.slot[w + f] for f in range(WINDOW)])
            L.row_median.append(s.lane)

        def emit(key, n):
            s = self.streams[key]
            tw = s.n_in - CARRY if key in ending else None
            ws, rule = ensemble_rule(n, tw)
            lo = first_new.get(key, s.n_win)  # the carry holds windows [lo - 7, lo)
            refs = []
            for w in ws:
                if w is None:
                    refs.append(-1)
                elif (key, w) in row_of:
                    refs.append(self.carry_rows + row_of[(key, w)])
                else:
                    if not lo - CARRY <= w < lo:
                        raise AssertionError(f"stream {key!r} frame {n}: window {w} is neither carried nor in the "
                                             "batch")
                    refs.append(CARRY * s.lane + w % CARRY)
            if rule == 0 and -1 in refs:
                raise AssertionError("weighted sum over a missing window")
            L.frames.append((key, n))
            L.refs.append(refs)
            L.rule.append(rule)

        for key, w in rows:
            emit(key, w)
        for key in tails:
            s = self.streams[key]
            for n in range(s.n_in - CARRY, s.n_in):
                emit(key, n)
        for key in first_new:
            s = self.streams[key]
            mine = [w for k, w in rows if k == key]
            for w in mine[-CARRY:]:  # the stream's newest 7 windows; window w's row is window w-7's
                L.carry.append((CARRY * s.lane + w % CARRY, row_of[(key, w)]))
            s.n_win = mine[-1] + 1
        return L
