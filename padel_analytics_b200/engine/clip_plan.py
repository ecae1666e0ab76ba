"""Batch planning for the ball pipeline over a list of clips (pure Python, no device).

The frames of all clips arrive as one stream, in upload chunks of `chunk` frames.  A TrackNet window is 8
consecutive frames of ONE clip, so clip c of T >= 8 frames has T - 7 windows and clips of fewer than 8 frames have
none (their frames never enter the ball ring).  Windows of consecutive clips are numbered consecutively ("global"
windows), which keeps the engine's (7 + B) heat-map buffer and its 7-row carry valid across clip boundaries.

`plan_clip_batches` decides, chunk by chunk, which frames enter the device ring and where, when each clip's
background is loaded into the median pool, and which windows each device batch runs.  Full batches of `batch`
windows run as soon as they are ready; a partial batch runs only when the ring or the median pool would otherwise
overflow, and at the end of the stream.
"""
from __future__ import annotations

from dataclasses import dataclass, field

WINDOW = 8


@dataclass
class ClipBatch:
    """One device batch.  Row b is window `windows[b]` = (clip, window index in the clip); its frames are the ring
    slots (row_slot[b] + f) % ring, f = 0..7, and its background is median pool slot row_median[b].  `first_window`
    is the global index of row 0.  The batch emits `frames` = (clip, frame) in order; `desc` holds the ensemble
    descriptor of each emitted frame: (global index of its clip's window 0, the clip's window count, frame)."""
    first_window: int
    windows: list = field(default_factory=list)
    row_slot: list = field(default_factory=list)
    row_median: list = field(default_factory=list)
    frames: list = field(default_factory=list)
    desc: list = field(default_factory=list)


@dataclass
class ClipPlan:
    """steps[i]: the operations to enqueue when upload chunk i arrives, in order:
      ("median", clip, pool_slot)           load clip's background into the pool
      ("push", offset, n, ring_slot)        resize frames [offset, offset+n) of the chunk into ring slots
                                            ring_slot .. ring_slot+n-1 (never wraps)
      ("run", ClipBatch)                    pack, TrackNet, ensemble, boxes
    """
    lengths: list
    batch: int
    chunk: int
    ring: int
    pool: int
    steps: list
    clip_first_window: list  # global index of each clip's window 0 (clips without windows: where they would start)


def default_ring(batch: int) -> int:
    """Ring of resized frames: room for a batch of pending windows spread over a few clip boundaries."""
    return 4 * batch + 8


def default_pool(ring: int) -> int:
    """Median pool slots: more clips than can have frames in the ring at once (each holds >= 8), so the pool never
    forces a partial batch."""
    return ring // WINDOW + 2


def plan_clip_batches(lengths, batch: int, chunk: int | None = None, ring: int | None = None,
                      pool: int | None = None) -> ClipPlan:
    lengths = [int(t) for t in lengths]
    if any(t < 0 for t in lengths):
        raise ValueError("clip lengths must be >= 0")
    chunk = batch if chunk is None else chunk
    ring = default_ring(batch) if ring is None else ring
    pool = default_pool(ring) if pool is None else pool
    if batch < 1 or chunk < 1:
        raise ValueError("batch and chunk must be >= 1")
    if ring < chunk + WINDOW - 1 or ring < WINDOW:
        raise ValueError(f"ring of {ring} frames cannot take a chunk of {chunk} behind a partial window")
    if pool < 1:
        raise ValueError("the median pool needs a slot")

    nwin = [max(0, t - (WINDOW - 1)) for t in lengths]
    first_win, g = [], 0
    for n in nwin:
        first_win.append(g)
        g += n
    # ring stream position of each clip's first frame (only clips with windows enter the ring)
    ring_pos, p = [], 0
    for t, n in zip(lengths, nwin):
        ring_pos.append(p)
        p += t if n else 0
    total = sum(lengths)

    pending: list = []  # ready windows not yet run: (clip, w)
    nxt = [0, 0]  # next window to become ready: (clip, w) -- clip == len(lengths) when none is left
    pushed = 0  # frames in the ring stream so far
    oldest = [0]  # ring position of the first frame of the oldest window not yet run
    pool_owner: dict[int, int] = {}  # pool slot -> clip
    last_run = [-1]  # global index of the last window run
    ball_rank = {}  # clip -> index among clips with windows
    for c, n in enumerate(nwin):
        if n:
            ball_rank[c] = len(ball_rank)

    def advance_next():
        c, w = nxt
        while c < len(lengths) and w >= nwin[c]:
            c, w = c + 1, 0
        nxt[0], nxt[1] = c, w

    advance_next()

    def update_oldest():
        if pending:
            c, w = pending[0]
        else:
            c, w = nxt
        oldest[0] = ring_pos[c] + w if c < len(lengths) else pushed

    def run(ops, n):
        rows = pending[:n]
        b = ClipBatch(first_window=first_win[rows[0][0]] + rows[0][1])
        for c, w in rows:
            gw = first_win[c] + w
            assert gw == last_run[0] + 1
            last_run[0] = gw
            b.windows.append((c, w))
            b.row_slot.append((ring_pos[c] + w) % ring)
            b.row_median.append(ball_rank[c] % pool)
            emit = [w] + (list(range(nwin[c], lengths[c])) if w == nwin[c] - 1 else [])
            for f in emit:
                b.frames.append((c, f))
                b.desc.append((first_win[c], nwin[c], f))
        del pending[:n]
        update_oldest()
        ops.append(("run", b))

    def flush(ops, until=None):
        """run partial/full batches until `until()` holds (default: nothing pending)"""
        while pending and (until is None or not until()):
            run(ops, min(batch, len(pending)))

    steps = []
    clip_of, clip_lo = [], []
    for c, t in enumerate(lengths):
        clip_of += [c] * t
        clip_lo += list(range(t))
    for start in range(0, total, chunk):
        ops: list = []
        n_chunk = min(chunk, total - start)
        run_start = None  # current contiguous push: [offset, n, slot]
        for off in range(n_chunk):
            c, f = clip_of[start + off], clip_lo[start + off]
            if not nwin[c]:
                continue
            if f == 0:  # the clip's background goes into the slot of a clip whose windows have all run
                slot = ball_rank[c] % pool
                prev = pool_owner.get(slot)
                if prev is not None and (nxt[0] <= prev or any(pc <= prev for pc, _ in pending)):
                    if run_start:
                        ops.append(("push", *run_start))
                        run_start = None
                    flush(ops, lambda: not any(pc <= prev for pc, _ in pending))
                    if nxt[0] <= prev:
                        raise AssertionError("median pool: a clip's windows are not all ready")
                if run_start:
                    ops.append(("push", *run_start))
                    run_start = None
                ops.append(("median", c, slot))
                pool_owner[slot] = c
            if pushed + 1 - oldest[0] > ring:  # the ring is full: run what is pending to free it
                if run_start:
                    ops.append(("push", *run_start))
                    run_start = None
                flush(ops)
                assert pushed + 1 - oldest[0] <= ring
            slot = pushed % ring
            if run_start and run_start[0] + run_start[1] == off and (run_start[2] + run_start[1]) == slot:
                run_start[1] += 1
            else:
                if run_start:
                    ops.append(("push", *run_start))
                run_start = [off, 1, slot]
            pushed += 1
            # windows whose last frame just arrived
            while nxt[0] < len(lengths) and ring_pos[nxt[0]] + nxt[1] + WINDOW <= pushed:
                pending.append((nxt[0], nxt[1]))
                nxt[1] += 1
                advance_next()
            update_oldest()
        if run_start:
            ops.append(("push", *run_start))
        while len(pending) >= batch:
            run(ops, batch)
        if start + n_chunk >= total:
            flush(ops)
        steps.append(ops)
    assert not pending and nxt[0] == len(lengths)
    return ClipPlan(lengths, batch, chunk, ring, pool, steps, first_win)
