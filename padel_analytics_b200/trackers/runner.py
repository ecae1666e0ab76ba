"""TrackingRunner: the per-tracker pass over a video (API of /root/reference/trackers/runner.py:37-236), plus the
multi-GPU sharded variant (SURVEY §8e): one process per GPU, contiguous frame ranges, no per-batch collectives —
detections are gathered once per tracker and the sequential host stages (ByteTrack ids, JSON) run on rank 0.

Every pass reads its frame sources through `frames.py` (`read`, `chunks`, `head`).  After the trackers, `run()`
renders the annotated video to `inference_path` and collects the players' court positions into `data_analytics`
(runner.py:91-173) when either is asked for; the overlays are composited on the device (render.py,
`pb_render_overlay`) and encoding runs on a thread of its own.  `run_clips()` does the same per clip for a list of
clips.  Both draw through one render pass over clips played back to back (`_render_clips`; `run()`'s video is one
clip).  Under torch.distributed `run_clips()` shards whole clips over the ranks (`plan_clip_shards`) and exchanges the
results once after the pass.  `stream()` tracks an iterable of frames of unknown length (a live feed) and yields each
frame's results as soon as every tracker has them (`FrameMerge`).

Documented deviations from reference quirks (SURVEY App. E):
  q7  with collect_data=False the reference's drawing pass ends by trimming `self.data_analytics.frames`, which is
      None, and raises AttributeError; here the trim happens only when data is collected.
  No per-frame prints; `data_analytics` is also filled when no video is written (collect_data=True without an
  inference_path), without rendering any frame.
"""
from __future__ import annotations

import collections
import contextlib
import itertools
import os
import timeit
from typing import Callable, Iterable, Iterator, Optional

import numpy as np
import torch

from . import frames
from . import sv_compat as sv
from ..engine.yolo_engine import ResultBlock
from .ball_tracker import Ball, BallTracker
from .keypoints_tracker import Keypoints
from .players_tracker import Players
from .tracker import Tracker, sampler
from ..analytics import DataAnalytics, ProjectedCourt


def shard_range(total: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous frame range of `rank` (SURVEY §8e): [rank*N/R, (rank+1)*N/R)."""
    return rank * total // world, (rank + 1) * total // world


def plan_clip_shards(lengths: list[int], world: int) -> list[list[int]]:
    """Whole clips per rank for `run_clips` under torch.distributed: longest clip first (ties: lower clip index), each
    to the rank with the fewest frames so far (ties: lower rank); each rank's clips in ascending order.  A pure
    function of its arguments, so every rank computes the same plan without communicating.  Clips of 0 frames are
    assigned too; a rank may get no clip.  The largest load is at most the mean load plus the longest clip."""
    import heapq

    if world < 1:
        raise ValueError(f"world size must be >= 1, got {world}")
    if any(T < 0 for T in lengths):
        raise ValueError("clip lengths must be >= 0")
    heap = [(0, r) for r in range(world)]  # (frames so far, rank): pops the least loaded, lowest rank first
    shards = [[] for _ in range(world)]
    for c in sorted(range(len(lengths)), key=lambda c: (-lengths[c], c)):
        load, r = heapq.heappop(heap)
        shards[r].append(c)
        heapq.heappush(heap, (load + int(lengths[c]), r))
    return [sorted(s) for s in shards]


def ball_shard_frames(total: int, start: int, end: int) -> tuple[int, int]:
    """Frames a ball shard must read to emit frames [start,end): 7 windows of history are recomputed and a window
    spans 8 frames => [start-7, end+7) clipped to the video."""
    return max(0, start - 7), min(total, end + 7)


def _host_state(t: Tracker) -> dict:
    """A tracker's order-dependent host state, as `video_info_post_init` sets it (PlayerTracker: its ByteTrack); put
    back with `t.__dict__.update(state)`."""
    return {k: t.__dict__[k] for k in ("video_info", "byte_track") if k in t.__dict__}


def _batch_trackers(trackers: dict[str, Tracker]) -> dict[str, Tracker]:
    """The trackers a device pass (`FusedPass`, `ClipPass`) feeds: those of stage "detect" or "ball"."""
    return {n: t for n, t in trackers.items() if t.stage in ("detect", "ball")}


class FusedPass:
    """One pass over the video feeding ALL trackers from a single upload per batch (the reference decodes and uploads
    the video once per tracker, runner.py:185-234; SURVEY §8f item 3).  Per batch: the next batch's host->device copy
    runs on a copy stream while this batch computes; the four trackers' device work is enqueued back to back without
    host synchronisation, and each tracker's host post-processing (ByteTrack, result objects) overlaps with the device
    work of the trackers behind it.

    `streams` (default env PADEL_B200_STREAMS, else 1): 0 = every tracker on the caller's stream; 1 = the YOLO trackers
    each on their own stream (their layers are small and latency-bound at batch 32 — many launch fewer CTAs than there
    are SMs — so three independent chains fill the machine), the ball tracker after them on the caller's stream;
    2 = all trackers concurrent.  The kernels and their inputs are the same in every mode, so are the results."""

    def __init__(self, trackers: dict[str, Tracker], frame_hw: tuple[int, int], batch_size: int,
                 total_frames: Optional[int], first_frame: int = 0, emit_range: Optional[tuple[int, int]] = None,
                 streams: Optional[int] = None, raw: bool = False, median=None):
        """raw=True: the YOLO trackers' entries are the engines' raw per-frame Results (no polygon filter / ByteTrack /
        result objects) -- what a shard hands to rank 0, where the order-dependent host stages run once over the
        ordered gather.  median: background for the ball tracker (defaults to BallTracker.median).
        total_frames=None: a stream whose length is known only when `run`'s batches end; `run` then ends with one
        more entry, the ball tracker's last windows and tail frames."""
        self.trackers = trackers
        self.total = total_frames
        self.raw = raw
        self.mode = int(os.environ.get("PADEL_B200_STREAMS", "1")) if streams is None else streams
        # side streams: the YOLO chains at high priority (their CTAs are placed first whenever SMs free up), the ball
        # tracker (mode 2 only) at normal priority
        self.side = {name: torch.cuda.Stream(priority=0 if t.stage == "ball" else -1)
                     for name, t in trackers.items()}
        self.hw = tuple(frame_hw)
        self.B = batch_size
        self.dev = torch.device("cuda")
        self.copy_stream = torch.cuda.Stream()
        self.staging = [torch.empty((batch_size,) + self.hw + (3,), dtype=torch.uint8, device=self.dev)
                        for _ in range(2)]
        self.ready = [torch.cuda.Event(), torch.cuda.Event()]
        self.consumed = [None, None]  # per staging slot: event after the device work that read it
        self._begin_ball(total_frames, first_frame, emit_range, median)

    def _begin_ball(self, total_frames, first_frame, emit_range, median) -> None:
        for t in self.trackers.values():
            if t.stage == "ball":
                t.stream_begin(self.hw, total_frames, first_frame, emit_range, median=median)

    def _upload(self, pieces, slot: int) -> torch.Tensor:
        """pieces: uint8 (n,H,W,3) tensors (pinned host or device) that make up one batch, in order, or one such
        tensor.  A batch of one device tensor is read in place; any other is gathered into the staging slot."""
        if isinstance(pieces, torch.Tensor):
            pieces = [pieces]
        if len(pieces) == 1 and pieces[0].device.type == "cuda":
            return pieces[0]
        n = sum(p.shape[0] for p in pieces)
        main = torch.cuda.current_stream()
        with torch.cuda.stream(self.copy_stream):
            if self.consumed[slot] is not None:  # the batch that last used this slot must have been read
                self.copy_stream.wait_event(self.consumed[slot])
            if any(p.device.type == "cuda" for p in pieces):
                self.copy_stream.wait_stream(main)
            at = 0
            for p in pieces:
                self.staging[slot][at:at + p.shape[0]].copy_(p, non_blocking=True)
                at += p.shape[0]
            self.ready[slot].record(self.copy_stream)
        return self.staging[slot][:n]

    def _process(self, fr: torch.Tensor) -> dict:
        return self._finish(self._launch(fr))

    def _launch(self, fr: torch.Tensor):
        """Enqueue the device work of every tracker for this batch (no host synchronisation)."""
        pending = []
        main = torch.cuda.current_stream()
        forked = []
        order = list(self.trackers.items())
        if self.mode == 1:  # YOLO chains first (concurrent), the ball tracker joins behind them
            order.sort(key=lambda kv: kv[1].stage == "ball")
        for name, t in order:  # enqueue everything first ...
            is_ball = t.stage == "ball"
            own = self.mode == 2 or (self.mode == 1 and not is_ball)
            if own:
                s = self.side[name]
                s.wait_stream(main)
                forked.append(s)
                ctx = torch.cuda.stream(s)
            else:
                if self.mode == 1:
                    for s in forked:
                        main.wait_stream(s)
                ctx = torch.cuda.stream(main)
            with ctx:
                pending.append((name, t, t.stream_push_async(fr) if is_ball else t.detect_sample_async(fr)))
        for s in forked:  # the caller's stream (and the next upload into this staging slot) follows all of them
            main.wait_stream(s)
        pending.sort(key=lambda p: list(self.trackers).index(p[0]))
        return pending, fr.shape[0]

    def _finish(self, launched) -> dict:
        """Wait for each tracker's results in turn and run its host post-processing."""
        pending, _ = launched
        out = {}
        for name, t, fin in pending:  # ... then finish in the same order
            res = fin()
            out[name] = res if t.stage == "ball" or self.raw else t.postprocess(res, self.hw)
        return out

    def run(self, batches: Iterable):
        """batches: iterable of uint8 (n,H,W,3) BGR batches, n <= batch_size, each a pinned host or device tensor or a
        list of such pieces (`frames.chunks`).  Yields one {tracker name: results} dict per batch.

        One batch of look-ahead: batch i+1 is pulled from `batches` and enqueued before batch i's results are yielded.
        A batch (host pieces: copied asynchronously into a staging slot; one device tensor: read in place) must stay
        untouched until ITS OWN results have been yielded, i.e. a producer that reuses buffers needs at least two.

        Without a total (a stream), the ball tracker emits a frame once the frame 7 later has been pushed, and after
        the last batch's dict comes one more, {ball tracker name: results of the last frames} (`_end`)."""
        it = iter(batches)
        main = torch.cuda.current_stream()
        pushed = 0

        def start(batch, i):
            """upload (copy stream) + enqueue all device work of batch i; returns the launch record"""
            nonlocal pushed
            dev = self._upload(batch, i % 2)
            pushed += dev.shape[0]
            staged = dev.data_ptr() == self.staging[i % 2].data_ptr()
            if staged:
                main.wait_event(self.ready[i % 2])
            rec = self._launch(dev)
            if staged:
                ev = torch.cuda.Event()
                ev.record(main)
                self.consumed[i % 2] = ev
            return rec

        cur = next(it, None)
        if cur is None:
            return
        rec, i = start(cur, 0), 0
        while rec is not None:
            # one batch of look-ahead: batch i+1 is uploaded and fully enqueued before batch i's results are collected,
            # so the device never waits for the host post-processing (ByteTrack, result objects) of the batch before
            nxt = next(it, None)
            nrec = start(nxt, i + 1) if nxt is not None else None
            yield self._finish(rec)
            rec, i = nrec, i + 1
        if self.total is None:
            yield self._end(pushed)

    def _end(self, total: int) -> dict:
        """The last step of a stream of `total` frames: the ball tracker's last windows and its 7 tail frames.  They
        are enqueued on the caller's stream, which every tracker's stream has joined after each batch."""
        return {name: t.stream_end_async(total)() for name, t in self.trackers.items() if t.stage == "ball"}


class ClipPass(FusedPass):
    """FusedPass over a list of clips played back to back: upload chunk i holds frames [i*B, (i+1)*B) of the
    concatenated clips, so device batches stay full across clip boundaries.  The ball tracker runs its windows by the
    clip plan (`clip_plan.plan_clip_batches`: a window never spans two clips, each clip has its own background), and
    the order-dependent host stages restart per clip: at a clip's first frame each YOLO tracker gets the clip's
    video_info (PlayerTracker: a fresh ByteTrack at the clip's fps).  Per batch, `run` yields {tracker name:
    [(clip, results of that clip's frames in the batch)]} for the YOLO trackers and [(clip, frame, (x, y, vis))] for
    the ball tracker, whose frames may come late (its partial batches wait for more windows)."""

    def __init__(self, trackers: dict[str, Tracker], frame_hw: tuple[int, int], batch_size: int, lengths: list[int],
                 clip_infos: list, median_of: Callable, streams: Optional[int] = None):
        self.lengths = list(lengths)
        self.clip_infos = clip_infos
        self.median_of = median_of
        self._starts = np.cumsum([0] + self.lengths)
        self._pos = 0
        super().__init__(trackers, frame_hw, batch_size, total_frames=int(self._starts[-1]), streams=streams)

    def _begin_ball(self, total_frames, first_frame, emit_range, median) -> None:
        from ..engine.clip_plan import plan_clip_batches

        for t in self.trackers.values():
            if t.stage == "ball":
                pipe = t.clip_pipeline(self.hw)
                plan = plan_clip_batches(self.lengths, t.batch_size, chunk=self.B, ring=pipe.ring, pool=pipe.pool)
                t.clips_begin(self.hw, plan, self.median_of)

    def _finish(self, launched) -> dict:
        pending, nfr = launched
        base, segs, lo = self._pos, [], self._pos
        while lo < base + nfr:  # (clip, first, end) in the chunk, and the clip frame at `first`
            c = int(np.searchsorted(self._starts, lo, side="right")) - 1
            e = min(base + nfr, int(self._starts[c + 1]))
            segs.append((c, lo - base, e - base, lo - int(self._starts[c])))
            lo = e
        self._pos = base + nfr
        out = {}
        for name, t, fin in pending:
            if t.stage == "ball":
                out[name] = fin()
                continue
            res, parts = fin(), []
            for c, a, b, f0 in segs:
                if f0 == 0:
                    t.video_info_post_init(self.clip_infos[c])
                parts.append((c, t.postprocess(res[a:b], self.hw)))
            out[name] = parts
        return out


class StreamsPass(FusedPass):
    """FusedPass over the frames of several interleaved live streams (`TrackingRunner.stream_many`).  Upload chunk i
    holds the frames `StreamMux` put in it, runs of consecutive frames of one stream each, and may be short or empty
    when a stream ends (its tail is then not held back by frames still to come).  The YOLO engines see one batch of
    frames; their host post-processing runs once per run, in pull order, with that stream's own host state
    (`_host_state`: PlayerTracker gets a fresh ByteTrack at the stream's first frame).  The ball tracker runs its
    windows through the multi-stream planner (`BallTracker.streams_begin`).  Per chunk, `run` yields ((runs
    [(key, first frame, n)], ending keys), {tracker name: results}): [(key, first frame, objects)] for the YOLO
    trackers, [(key, frame, (x, y, vis))] for the ball tracker."""

    def __init__(self, trackers: dict[str, Tracker], frame_hw: tuple[int, int], batch_size: int, max_open: int,
                 metas: collections.deque, median_of: Callable, video_info, streams: Optional[int] = None):
        self.metas = metas  # (runs, ends) per chunk, appended by StreamMux before the chunk is handed over
        self.max_open = max_open
        self.median_of = median_of
        self.video_info = video_info
        self.host: dict = {}  # stream key -> {tracker name: host state}
        self._ball_steps = collections.deque()
        super().__init__(trackers, frame_hw, batch_size, total_frames=None, streams=streams)

    def _begin_ball(self, total_frames, first_frame, emit_range, median) -> None:
        for t in self.trackers.values():
            if t.stage == "ball":
                t.streams_begin(self.hw, self.max_open, self._ball_steps, self.median_of)

    def _launch(self, fr: torch.Tensor):
        meta = self.metas.popleft()
        runs, ends = meta
        balls = {n: t for n, t in self.trackers.items() if t.stage == "ball"}
        if balls:
            self._ball_steps.append(([(key, n) for key, _, n in runs], ends))
        if fr.shape[0]:
            pending, _ = super()._launch(fr)
        else:  # a stream ended at a chunk boundary: its tail alone
            pending = [(name, t, t.stream_push_async(fr)) for name, t in balls.items()]
        return pending, meta

    def _finish(self, launched):
        pending, meta = launched
        runs, ends = meta
        out = {}
        for name, t, fin in pending:
            res = fin()
            if t.stage == "ball":
                out[name] = res
                continue
            parts, a = [], 0
            for key, f0, n in runs:
                if f0 == 0:
                    t.video_info_post_init(self.video_info)
                else:
                    t.__dict__.update(self.host[key][name])
                parts.append((key, f0, t.postprocess(res[a:a + n], self.hw)))
                self.host.setdefault(key, {})[name] = _host_state(t)
                a += n
            out[name] = parts
        for key in ends:
            self.host.pop(key, None)
        return meta, out

    def _end(self, total: int):
        return None  # every stream ended in a chunk of its own


class StreamMux:
    """The (key, frames) items of `TrackingRunner.stream_many` as the pieces of one pass, in pull order: `pieces()`
    yields (n,H,W,3) tensors and None, which closes the upload chunk being filled (`frames.chunks`), and appends to
    `metas`, before handing over the piece that completes it, each chunk's (runs [(key, first frame, n)], keys
    ending after its frames).

    A chunk closes when it holds B frames, when B frames have been pulled since the chunk before it closed (frames
    held for a background count: they are pulled but enter no chunk yet), and at a stream's end, whichever comes
    first.  So a chunk never waits longer than B pulls, however many streams are held, and a stream's tail is not held
    back by frames of other streams still to come.  A chunk may be short, or empty.

    A stream without a background (`medians[key]`, else `default`) has its first `hold` frames copied to the device
    and held; its frames enter the pass when `background(pieces)` has been taken from them (or at its end, from the
    frames it has), and until then the other streams keep running.  ValueError: a frame of another size than the
    first stream's, a key that reappears after its end, more than `max_open` streams open at once."""

    def __init__(self, items: Iterable, batch: int, max_open: int, medians: Optional[dict] = None, default=None,
                 hold: int = 0, background: Optional[Callable] = None, hold_device: str = "cuda"):
        self.items, self.B, self.max_open, self.hold_device = items, batch, max_open, hold_device
        self.medians = dict(medians or {})
        self.default, self.hold, self.background = default, hold, background
        self.metas = collections.deque()
        self.hw = None  # the frame size, fixed by the first frame
        self.count: dict = {}  # per open stream: frames handed to the pass
        self.held: dict = {}  # per open stream waiting for its background: the device copies of its first frames
        self.ended: set = set()
        # the chunk being filled: its runs, the streams ending after it, its frames, the frames pulled since it opened
        self._runs, self._ends, self._n, self._pulls = [], [], 0, 0

    def _put(self, key, t: torch.Tensor, pulled: bool) -> Iterator[Optional[torch.Tensor]]:
        """Hand stream `key`'s frames t to the pass, split at chunk boundaries.  pulled: t was pulled just now, so
        its frames also count toward the chunk's pulls (False for held frames released later)."""
        f0 = self.count[key]
        self.count[key] += t.shape[0]
        while t.shape[0]:
            take = min(self.B - (max(self._n, self._pulls) if pulled else self._n), t.shape[0])
            self._runs.append((key, f0, take))
            f0, self._n = f0 + take, self._n + take
            self._pulls += take if pulled else 0
            part, t = t[:take], t[take:]
            if self._n == self.B:  # full: `frames.chunks` closes it on this piece
                self._close()
                yield part
            elif self._pulls == self.B:
                self._close()
                yield part
                yield None
            else:
                yield part

    def _pull_held(self, n: int) -> Iterator[None]:
        """n frames pulled into a hold: they enter no chunk, but count toward the chunk's pulls."""
        while n:
            take = min(self.B - self._pulls, n)
            self._pulls, n = self._pulls + take, n - take
            if self._pulls == self.B:
                self._close()
                yield None

    def _close(self) -> None:
        self.metas.append((self._runs, self._ends))
        self._runs, self._ends, self._n, self._pulls = [], [], 0, 0

    def _release(self, key) -> Iterator[Optional[torch.Tensor]]:
        """Stream `key`'s held frames, now that its background exists (taken from them when it has any)."""
        held = self.held.pop(key)
        if held and self.background is not None:
            self.medians[key] = self.background(held)
        for t in held:
            yield from self._put(key, t, pulled=False)

    def _end(self, key) -> Iterator[Optional[torch.Tensor]]:
        if key in self.held:
            yield from self._release(key)
        del self.count[key]
        self.ended.add(key)
        self._ends.append(key)

    def pieces(self) -> Iterator[Optional[torch.Tensor]]:
        for key, item in self.items:
            if key in self.ended:
                raise ValueError(f"stream_many: stream {key!r} appears again after its end")
            if item is None:
                if key not in self.count:  # a stream of no frame: nothing to track
                    self.ended.add(key)
                    self._ends.append(key)
                    continue
                yield from self._end(key)
                self._close()
                yield None
                continue
            t = next(frames.tensors([item], self.hw, f"stream {key!r}"))
            self.hw = tuple(t.shape[1:3])
            if key not in self.count:
                if len(self.count) == self.max_open:
                    raise ValueError(f"stream_many: stream {key!r} would be stream {self.max_open + 1} open at once, "
                                     f"max_open is {self.max_open}")
                self.count[key] = 0
                if self.hold and key not in self.medians:
                    if self.default is not None:
                        self.medians[key] = self.default
                    else:
                        self.held[key] = []
            if key in self.held:  # copied: the caller may reuse its buffer once the item is pulled
                held = self.held[key]
                room = self.hold - sum(p.shape[0] for p in held)
                held.append(t[:room].to(self.hold_device, copy=True))
                yield from self._pull_held(min(room, t.shape[0]))
                if room > t.shape[0]:
                    continue
                yield from self._release(key)
                t = t[room:]
                if not t.shape[0]:
                    continue
            yield from self._put(key, t, pulled=True)
        for key in list(self.count):
            yield from self._end(key)
        if self._runs or self._ends:
            self._close()
            yield None


class FrameMerge:
    """In-order merge of per-tracker results for `TrackingRunner.stream`.  Each tracker's results arrive in frame
    order, but the trackers are out of step with one another: a YOLO tracker has a batch's frames when the batch is
    done, the ball tracker has them 7 frames later.  `put` hands over one tracker's result for its next frame; `ready`
    pops, in frame order, every frame that all trackers have."""

    def __init__(self, names: Iterable[str]):
        self.held = {n: collections.deque() for n in names}
        if not self.held:
            raise ValueError("FrameMerge needs at least one tracker")
        self.next = {n: 0 for n in self.held}  # per tracker: the frame its next result is for
        self.frame = 0  # the next frame `ready` pops

    def put(self, name: str, frame: int, obj) -> None:
        if frame != self.next[name]:
            raise ValueError(f"{name}: a result for frame {frame}, but frame {self.next[name]} is next")
        self.held[name].append(obj)
        self.next[name] += 1

    def ready(self) -> list[tuple[int, dict]]:
        """[(frame, {tracker name: result})] of the frames every tracker has now, in frame order."""
        out = []
        for f in range(self.frame, min(self.next.values())):
            out.append((f, {n: q.popleft() for n, q in self.held.items()}))
        self.frame = max(self.frame, min(self.next.values()))
        return out


class TrackingRunner:
    def __init__(self, trackers: dict[str, Tracker] | list[Tracker], video_path: Optional[str] = None,
                 inference_path: Optional[str] = None, start: int = 0, end: Optional[int] = None,
                 collect_data: bool = False, video_info=None):
        if isinstance(trackers, dict):
            trackers = list(trackers.values())
        self.trackers = {str(t): t for t in trackers}
        self.video_path = video_path
        self.inference_path = inference_path
        self.start, self.end = start, end
        if video_info is None and video_path is not None:
            video_info = sv.VideoInfo.from_video_path(video_path)
        self.video_info = video_info
        if video_info is not None:
            total = video_info.total_frames
            self.total_frames = (total if end is None else min(end, total)) - start if total is not None else None
            for t in self.trackers.values():
                t.video_info_post_init(video_info)  # runner.py:61-62
        # runner.py:59-79: fixed court keypoints keep the first homography; the mini court needs the frame size
        self.is_fixed_keypoints = any(t.stage == "fixed" for t in self.trackers.values())
        self.collect_data = collect_data
        self.projected_court = ProjectedCourt(video_info) if video_info is not None else None
        self.data_analytics = DataAnalytics() if collect_data else None
        self.render_batch_size = 32
        self.clips_data_analytics: list[DataAnalytics] = []  # per clip, filled by run_clips(collect_data=True)
        self._source = None  # frame_source of the last run(), for the drawing pass
        self._clip_reading: Optional[int] = None  # run_clips: the clip whose frames the pass read last
        self.timings: dict[str, float] = {}
        self.stream_results: dict = {}  # stream_many: per ended stream, {tracker name: [Object per frame]}

    def restart(self) -> None:
        for t in self.trackers.values():
            t.restart()
        if self.data_analytics:
            self.data_analytics.restart()

    def _frames(self, lo: int, hi: int) -> Iterable[np.ndarray]:
        return sv.get_video_frames_generator(self.video_path, start=self.start + lo, end=self.start + hi)

    def run(self, frame_source: Optional[Callable[[int, int], Iterable[np.ndarray]]] = None,
            total_frames: Optional[int] = None, fused: Optional[bool] = None) -> dict[str, float]:
        """The runner pass (runner.py:185-234).  `frame_source(lo, hi)` yields frames lo..hi-1 (defaults to decoding
        `video_path`).

        fused (default: on when two or more trackers of stage "detect" or "ball" still need inference): ONE pass over
        the frames feeds every such tracker from a single decode + upload per batch (`FusedPass`; the reference decodes
        and uploads once per tracker, runner.py:215-220).  fused=False is the reference's plain loop, one full pass per
        tracker.  Trackers with cached predictions (runner.py:187-191) are skipped; those of stage "fixed" or "frames"
        run through `predict_and_update`.

        Under torch.distributed (world_size > 1) each rank processes its contiguous shard, fixed-capacity detection
        records are all-gathered, and rank 0 runs the order-dependent host stages (polygon filter, ByteTrack ids,
        InpaintNet, result objects) over the ordered frames."""
        import gc

        # The pass creates hundreds of small result objects per frame and keeps them all (the reference's results API);
        # none of them form cycles, so the cyclic collector only costs time (more and more as
        # its generations fill up).  Collection is suspended for the duration of the pass.
        gc_was_on = gc.isenabled()
        gc.disable()
        try:
            timings = self._run(frame_source, total_frames, fused)
        finally:
            if gc_was_on:
                gc.enable()
        import torch.distributed as dist

        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
        if rank == 0 and (self.inference_path or self.data_analytics is not None):  # rank 0 holds every result
            t0 = timeit.default_timer()
            self.draw_and_collect_data()
            timings["_render"] = timeit.default_timer() - t0
        return timings

    def _run(self, frame_source, total_frames, fused) -> dict[str, float]:
        import torch.distributed as dist

        src = frame_source or self._frames
        total = total_frames if total_frames is not None else self.total_frames
        self._source = src
        dist_on = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist_on else (0, 1)
        lo, hi = shard_range(total, rank, world)
        todo = {n: t for n, t in self.trackers.items() if len(t) == 0}  # cached predictions: skipped (runner.py:187-191)
        model = _batch_trackers(todo)
        if fused is None:
            fused = len(model) >= 2 and torch.cuda.is_available()
        if fused and model:
            self._run_fused(model, src, total, lo, hi, rank, world, dist_on)
            todo = {n: t for n, t in todo.items() if n not in model}
        for name, tracker in todo.items():
            tracker.to(tracker.DEVICE)
            t0 = timeit.default_timer()
            if tracker.stage == "ball":
                flo, fhi = ball_shard_frames(total, lo, hi)
                median = self._ball_median(tracker, src, total, rank, dist_on)
                part = tracker.track_xyv(src(flo, fhi), total, first_frame=flo, emit_range=(lo, hi), median=median)
                part = _ball_records(part, lo, hi)
            elif tracker.stage == "detect":
                part, hw = [], None
                for sample in sampler(src(lo, hi), tracker.batch_size):
                    hw = sample[0].shape[:2]
                    part.append(tracker.detect_sample(sample))
                part = (_yolo_records(part, tracker), hw)
            else:  # "frames", and "fixed", whose predict_frames repeats the detection once per frame of the source
                part = list(tracker.predict_and_update(src(lo, hi), total_frames=hi - lo).predictions)
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            self._gather_and_assemble(tracker, part, total, rank, world, dist_on)
            self.timings[name] = timeit.default_timer() - t0
            tracker.to("cpu")
            if rank == 0:
                tracker.save_predictions()
        return self.timings

    # ---- a frame stream of unknown length -------------------------------------------------------------------------
    def stream(self, frames_in: Iterable, median=None) -> Iterator[tuple[int, dict]]:
        """Track a stream of frames whose length is not known in advance (a camera, a broadcast, a long recording):
        a generator of `(frame index, {tracker name: Object})` in frame order, each frame yielded as soon as every
        tracker's result for it is final.

        frames_in: any iterable of HWC uint8 BGR frames or uint8 (n,H,W,3) batches, host or device; the stream ends
        when the iterable does.  Every frame must have the size of the first (ValueError).  Host frames that are not
        pinned are copied as they are pulled; a pinned or device batch is read in place and must stay untouched until
        its frames have been yielded.  The fps (ByteTrack) and the frame size that scales the ball's coordinates come
        from the runner's `video_info`.

        Trackers of stage "detect", "ball" and "fixed" are supported.  A "frames" tracker (the ResNet court regressor),
        a tracker holding cached predictions (a stream has no frame count to match them against) and a torch.distributed
        job of world size > 1 are refused with ValueError, before any frame is pulled.

        Results: while the stream runs, each tracker's `results.predictions` grows by the frames yielded.  The Ball
        yielded per frame is TrackNet's: InpaintNet needs the whole trajectory, so when the stream ends the ball
        tracker's `results` are replaced by `balls(trajectory, frame count)`, which applies InpaintNet.  Then every
        tracker's `results` equal what `run()` gives on the same frames, and, as after `run()`, the model trackers
        are moved to the CPU and every tracker with a `save_path` writes its predictions.  A caller that stops early
        keeps the results of the frames yielded, without InpaintNet, and nothing is saved.

        Unlike `run()`, which switches Python's cyclic garbage collector off for its pass, `stream` leaves it as the
        caller set it: a generator cannot switch it off for its own steps without switching it off for the caller's
        code between them.  The results kept per frame are many small objects that form no cycles, so on a long
        stream each full collection walks more of them; a caller for whom those pauses matter can call
        `gc.disable()` (or `gc.freeze()`) around its loop.

        Background: `median` ((H,W,3) uint8 RGB), else `BallTracker.median`, else the median of the stream's first
        `median_max_sample_num` frames (`run()`'s background), which are held on the device until it is computed.  No
        frame is yielded before the background exists, so that every tracker's entries stay in frame order.

        Latency: with B the pass's batch (the smallest batch_size of the "detect" and "ball" trackers), the entry of
        frame f is yielded before the pass pulls frame f + 2B + 8 from `frames_in` (one batch in flight, one batch of
        look-ahead, the 7 frames the ball ensemble looks ahead), for every f whose frame f + 2B + 8 comes after the
        frames held for the background.  An item of n frames is pulled whole, which moves the bound by up to n - 1
        frames.  A live caller picks a small batch_size."""
        self._check_streamable("stream")
        return self._stream(frames_in, median)

    def _check_streamable(self, what: str) -> None:
        """ValueError for what a stream cannot run: a torch.distributed job, "frames" trackers, cached predictions, no
        video_info."""
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise ValueError(f"{what}: a stream runs in one process, not over a torch.distributed job of world size "
                             f"{dist.get_world_size()}")
        if not self.trackers:
            raise ValueError(f"{what}: no trackers")
        other = sorted(n for n, t in self.trackers.items() if t.stage not in ("detect", "ball", "fixed"))
        if other:
            raise ValueError(f"{what}: trackers {other} have no batch model stage (a YOLO or ball model) and no fixed "
                             "detection")
        cached = sorted(n for n, t in self.trackers.items() if len(t))
        if cached:
            raise ValueError(f"{what}: trackers {cached} hold cached predictions, and a stream has no frame count to "
                             "match them against (restart() them first)")
        if self.video_info is None:
            raise ValueError(f"{what}: the fps and the ball's frame size come from video_info, and this runner has "
                             "none")

    def _stream(self, frames_in: Iterable, median) -> Iterator[tuple[int, dict]]:
        from .ball_tracker import median_background_device

        model = _batch_trackers(self.trackers)
        fixed = {n: t.fixed_detection for n, t in self.trackers.items() if t.stage == "fixed"}
        ball_name, ball = next(((n, t) for n, t in model.items() if t.stage == "ball"), (None, None))
        merge = FrameMerge(self.trackers)
        pieces = frames.tensors(frames_in)
        if ball is not None:
            median = ball.median if median is None else median
            if median is None:  # iterable.py:58-73, as run() does: the first frames, copied as they are pulled
                m, held = ball.median_max_sample_num, [0]

                def own(p):
                    keep = held[0] < m
                    held[0] += p.shape[0]
                    return p.to("cuda", copy=True) if keep else p

                first, pieces = frames.head(map(own, pieces), m)
                if held[0]:
                    median = median_background_device(first)
                pieces = itertools.chain(first, pieces)
        if model:
            B = min(t.batch_size for t in model.values())
            for t in model.values():
                t.to(t.DEVICE)
            sizes = collections.deque()  # frames of each chunk the pass has pulled and not yet finished

            def sized(chunks):
                for c in chunks:
                    sizes.append(sum(p.shape[0] for p in c))
                    yield c

            chunks = frames.chunks(pieces, B)
            first = next(chunks, None)
            if first is None:
                steps = iter(())
            else:
                fp = FusedPass(model, tuple(first[0].shape[1:3]), B, total_frames=None, median=median)
                # after the last chunk, the pass's final entry (the ball's tail) covers no new frame
                steps = ((sizes.popleft() if sizes else 0, out)
                         for out in fp.run(sized(itertools.chain([first], chunks))))
        else:
            steps = ((p.shape[0], {}) for p in pieces)
        total, xyv = 0, {}
        for n, out in steps:
            for name in self.trackers:
                if name == ball_name:
                    for f, (x, y, v) in out.get(name, {}).items():
                        xyv[f] = (x, y, v)
                        merge.put(name, f, Ball(frame=f, xy=(x, y), visibility=v))
                elif name in fixed:
                    for f in range(total, total + n):
                        merge.put(name, f, fixed[name])
                else:
                    for i, o in enumerate(out.get(name, [])):
                        merge.put(name, total + i, o)
            total += n
            yield from self._emit(merge)
        if ball is not None:  # TrackNet gives no frame of a stream shorter than a window: no ball there
            for f in range(merge.next[ball_name], total):
                merge.put(ball_name, f, Ball(frame=f, xy=(0.0, 0.0), visibility=0))
        yield from self._emit(merge)
        if ball is not None:
            ball.results.predictions = ball.balls(xyv, total)  # InpaintNet over the whole trajectory
        for t in self.trackers.values():  # what run() does after its pass
            if t.stage in ("detect", "ball"):
                t.to("cpu")
            t.save_predictions()

    def _emit(self, merge: FrameMerge) -> Iterator[tuple[int, dict]]:
        for f, entry in merge.ready():
            for name, obj in entry.items():
                self.trackers[name].results.predictions.append(obj)
            yield f, entry

    # ---- several live streams in one pass ---------------------------------------------------------------------------
    def stream_many(self, items: Iterable, medians: Optional[dict] = None, max_open: int = 16
                    ) -> Iterator[tuple[object, int, dict]]:
        """Track several live streams (cameras, courts) in one pass whose device batches hold frames of any of them: a
        generator of `(key, frame index, {tracker name: Object})`, each stream's entries in frame order, each entry
        yielded as soon as every tracker's result for it is final.  Each stream gets what `stream()` gives on its
        frames alone.

        items: any iterable of `(key, frames)`: `key` any hashable name of a stream, `frames` one HWC uint8 BGR frame
        or a uint8 (n,H,W,3) batch, host or device, as `stream()` takes them.  `(key, None)` ends stream `key`; every
        open stream ends when the iterable does.  Streams may open and end at any point; a key that ended may not
        appear again (ValueError).  Every frame must have the size of the first (ValueError naming the key), and every
        stream shares the runner's `video_info` (ByteTrack's fps, the ball's coordinate scale).  At most `max_open`
        streams may be open at once (ValueError); the ball stage's device pools are sized for that many (about 42 MB
        per open stream at TrackNet's 288x512, `StreamsBallPipeline`).

        Refused with ValueError before any item is pulled: what `stream()` refuses ("frames" trackers, cached
        predictions, a torch.distributed job of world size > 1, no `video_info`).

        Per stream, the host stages run as if the stream ran alone: YOLO post-processing runs once per run of the
        stream's frames in a batch, in pull order, with the stream's own ByteTrack (PlayerTracker: fresh at its first
        frame).  The yielded Ball is TrackNet's.  When a stream ends, InpaintNet runs over its trajectory and
        `stream_results[key]` = {tracker name: [Object per frame]} holds its final results, equal to `run()`'s on its
        frames, before its last entries are yielded; the caller may pop them.  The trackers' own `results` are left
        untouched and nothing is written to a `save_path`.

        Background per stream: `medians[key]` ((H,W,3) uint8 RGB), else `BallTracker.median`, else the median of the
        stream's first `median_max_sample_num` frames, which are held on the device until it is computed; until then
        the stream's frames do not enter the pass and none of its entries is yielded, while the other streams run.

        Latency: with B the pass's batch (the smallest batch_size of the "detect" and "ball" trackers), count the frames
        of all streams in pull order, those held for a background included; if stream s's frame f + 7 is the k-th frame
        pulled, the entry (s, f) is yielded before the (k + 2B)-th frame is pulled, for every f whose frame f + 7 is
        pulled after s's background exists, whatever the other streams do.  A stream's last 7 entries are yielded
        before the (B + 1)-th frame pulled after its end item.  Both hold because an upload chunk closes once B frames
        have been pulled since the one before it closed, even when held frames left it short or empty, and at every
        end item; the pass keeps one chunk of look-ahead.  An item of n frames is pulled whole, which moves the bounds
        by up to n - 1 frames.

        As `stream()`, this leaves Python's cyclic garbage collector as the caller set it."""
        self._check_streamable("stream_many")
        if max_open < 1:
            raise ValueError("stream_many: max_open must be >= 1")
        return self._stream_many(items, medians, max_open)

    def _stream_many(self, items: Iterable, medians, max_open: int) -> Iterator[tuple[object, int, dict]]:
        from .ball_tracker import median_background_device

        model = _batch_trackers(self.trackers)
        fixed = {n: t.fixed_detection for n, t in self.trackers.items() if t.stage == "fixed"}
        ball_name, ball = next(((n, t) for n, t in model.items() if t.stage == "ball"), (None, None))
        B = min(t.batch_size for t in model.values()) if model else 1
        mux = StreamMux(items, B, max_open, medians, default=None if ball is None else ball.median,
                        hold=0 if ball is None else ball.median_max_sample_num, background=median_background_device)
        merges: dict = {}  # per stream: its FrameMerge
        got: dict = {}  # per stream: {tracker name: objects yielded}
        xyv: dict = {}  # per stream: its TrackNet trajectory
        count: dict = {}  # per stream: frames seen

        def step(meta, out) -> list:
            runs, ends = meta
            for key, f0, n in runs:
                if key not in merges:
                    merges[key], got[key], xyv[key] = FrameMerge(self.trackers), {n_: [] for n_ in self.trackers}, {}
                for name, det in fixed.items():
                    for f in range(f0, f0 + n):
                        merges[key].put(name, f, det)
                count[key] = f0 + n
            for name, parts in out.items():
                if name == ball_name:
                    for key, f, (x, y, v) in parts:
                        xyv[key][f] = (x, y, v)
                        merges[key].put(name, f, Ball(frame=f, xy=(x, y), visibility=v))
                else:
                    for key, f0, objs in parts:
                        for i, o in enumerate(objs):
                            merges[key].put(name, f0 + i, o)
            for key in ends:
                if key not in merges:  # a stream of no frame
                    merges[key], got[key], xyv[key] = FrameMerge(self.trackers), {n_: [] for n_ in self.trackers}, {}
                if ball is not None:  # TrackNet gives no frame of a stream shorter than a window: no ball there
                    for f in range(merges[key].next[ball_name], count.get(key, 0)):
                        merges[key].put(ball_name, f, Ball(frame=f, xy=(0.0, 0.0), visibility=0))
            ready = [(key, f, entry) for key in dict.fromkeys([r[0] for r in runs] + list(merges))
                     for f, entry in merges[key].ready()]
            for key, _, entry in ready:
                for name, obj in entry.items():
                    got[key][name].append(obj)
            for key in ends:
                res = got.pop(key)
                if ball is not None:
                    res[ball_name] = ball.balls(xyv.pop(key), count.pop(key, 0))  # InpaintNet over the trajectory
                self.stream_results[key] = res
                merges.pop(key)
                mux.medians.pop(key, None)
            return ready

        pieces = mux.pieces()
        steps = iter(())
        if model:
            for t in model.values():
                t.to(t.DEVICE)
            chunks = frames.chunks(pieces, B)
            first = next(chunks, None)
            if mux.hw is not None:  # a frame reached the pass
                fp = StreamsPass(model, mux.hw, B, max_open, mux.metas, lambda key: mux.medians[key], self.video_info)
                steps = (r for r in fp.run(itertools.chain([first], chunks)) if r is not None)
            else:
                steps = ((mux.metas.popleft(), {}) for _ in itertools.chain([first], chunks) if _ is not None)
        else:
            def direct():
                for _ in pieces:
                    while mux.metas:
                        yield mux.metas.popleft(), {}
                while mux.metas:
                    yield mux.metas.popleft(), {}

            steps = direct()
        with self._clip_state():
            for meta, out in steps:
                yield from step(meta, out)
        for t in model.values():
            t.to("cpu")

    # ---- drawing pass (runner.py:91-173) -----------------------------------------------------------------------
    def _as_clip(self, frame_source) -> tuple[list, list, list]:
        """The run's video as the one clip of a drawing pass: ([frame source], [video_info], [results]), the clip as
        long as the trackers' results (the frames drawn are fewer if the source ends first)."""
        if self.video_info is None:
            raise ValueError("rendering needs video_info (the frame size of the mini court)")
        vi = self.video_info
        results = {n: t.results for n, t in self.trackers.items()}
        info = sv.VideoInfo(width=vi.width, height=vi.height, fps=vi.fps,
                            total_frames=len(next(iter(results.values()))))
        return [frame_source or self._source or self._frames], [info], [results]

    @contextlib.contextmanager
    def _clip_state(self):
        """Each clip restarts the trackers' order-dependent host stages (`video_info_post_init`: PlayerTracker gets a
        fresh ByteTrack); their `video_info` and ByteTrack are put back on exit, so a later run() finds them as they
        were."""
        saved = {n: _host_state(t) for n, t in self.trackers.items()}
        try:
            yield
        finally:
            for n, t in self.trackers.items():
                t.__dict__.update(saved[n])

    def render_frames(self, frame_source: Optional[Callable[[int, int], Iterable[np.ndarray]]] = None,
                      data_analytics: Optional[DataAnalytics] = None) -> Iterable[np.ndarray]:
        """The run's frames with the drawings of runner.py:114-162 (frame number, every tracker's `draw`, mini
        court, projected players and ball), as uint8 BGR host frames, one per video frame.  `frame_source` is the
        callable `run()` takes (default: the one the last `run()` used, else the video).  Positions go to
        `data_analytics` when one is given.  The overlays are composited on the device in batches."""
        srcs, infos, results = self._as_clip(frame_source)
        with self._clip_state():
            _, _, batches = self._draw_clips(srcs, infos, results, self.projected_court,
                                             None if data_analytics is None else [data_analytics], exact=False)
            for out, _ in batches:
                for f in out:
                    yield f.copy()

    def draw_and_collect_data(self, frame_source=None) -> None:
        """runner.py:91-173: writes the rendered video to `inference_path` (cv2.VideoWriter, mp4v, the video's fps and
        size; encoding on a writer thread, overlapping the next batch) and fills `data_analytics` when collecting."""
        if self.data_analytics is not None:
            self.data_analytics.restart()
        srcs, infos, results = self._as_clip(frame_source)
        with self._clip_state():
            self._render_clips(srcs, infos, results, self.projected_court,
                               None if self.data_analytics is None else [self.data_analytics],
                               [self.inference_path] if self.inference_path else None, exact=False, prefix="_render")

    def _render_clips(self, srcs: list, infos: list, results: list[dict], court: ProjectedCourt,
                      das: Optional[list[DataAnalytics]], paths: Optional[list[str]], exact: bool, prefix: str,
                      clip_ids: Optional[list[int]] = None) -> None:
        """The drawing pass of `_draw_clips` with clip c's video written to paths[c] (mp4v, the clip's fps and frame
        size) by a writer thread of its own (`write_clip_batches`), the render times going to `timings` under
        `prefix`.  paths=None: data only, the positions need no frame (`_collect_positions`).  das: one
        `DataAnalytics` per clip or None; each ends trimmed as the reference trims its one (q7)."""
        import queue

        from ..render import VideoWriterThread, write_clip_batches

        if paths is None:
            for c, vi in enumerate(infos):
                self._collect_positions(results[c], int(vi.total_frames), court, das[c])
        elif sum(int(vi.total_frames) for vi in infos):
            free = queue.Queue()
            for slot in range(3):
                free.put(slot)
            plan, renderer, batches = self._draw_clips(srcs, infos, results, court, das, exact, clip_ids, free)

            def open_writer(c, release):
                return VideoWriterThread(paths[c], infos[c].fps, infos[c].resolution_wh, release)

            self.timings[f"{prefix}_encode"] = write_clip_batches(plan, batches, open_writer, free)
            for k, v in renderer.times.items():
                self.timings[f"{prefix}_{k}"] = v
        if das is not None:
            for da in das:  # q7: the reference trims even when it collects nothing
                da.frames = da.frames[:-1]  # remove the extra frame

    def _draw_clips(self, srcs: list, infos: list, results: list[dict], court: ProjectedCourt,
                    das: Optional[list[DataAnalytics]], exact: bool, clip_ids: Optional[list[int]] = None,
                    free_slots=None):
        """The clips played back to back through one `OverlayRenderer` (one set of pinned buffers, one sprite cache)
        in batches that cross clip boundaries (`plan_clip_render`), each clip's frames read from srcs[c]
        (`frames.read`: exact, or ending where the source ends) and each frame drawn from its clip's results,
        video_info, homography state and das[c].  Every clip starts as a run() of its own would; callers hold
        `_clip_state`.  Returns (plan, renderer, iterator over the rendered (frames, out slot) batches).  clip_ids:
        the clips' numbers in messages (default 0, 1, ...)."""
        from ..render import DisplayListBuilder, OverlayRenderer, plan_clip_render

        lengths = [int(vi.total_frames) for vi in infos]
        hw = (infos[0].height, infos[0].width)
        B = self.render_batch_size
        plan = plan_clip_render(lengths, B)
        builder = DisplayListBuilder(hw, court)
        renderer = OverlayRenderer(hw, B, builder.lut, out_slots=3)

        def build(first, n):
            recs = []
            for c, f in plan[first // B].rows[:n]:  # n < rows: the source ended early
                if f == 0:
                    court.H = None
                    for t in self.trackers.values():
                        t.video_info_post_init(infos[c])
                recs.append(builder.frame_records(f, self.trackers, None if das is None else das[c],
                                                  self.is_fixed_keypoints, results[c]))
            return recs

        batches = _clip_render_batches(srcs, lengths, B, hw, clip_ids, exact)
        return plan, renderer, renderer.run(batches, build, free_slots)

    def _collect_positions(self, results: dict, total: int, court: ProjectedCourt,
                           data_analytics: DataAnalytics) -> None:
        """The players' court positions of frames 0..total-1 into `data_analytics`, without drawing.  results:
        {tracker name: per-frame predictions}."""
        court.H = None
        for i in range(total):
            players = keypoints = None
            for name, t in self.trackers.items():
                if t.object() is Players:
                    players = results[name][i]
                elif t.object() is Keypoints:
                    keypoints = results[name][i]
            H = court.update_homography(keypoints, self.is_fixed_keypoints)
            if H is not None and players:
                court.project_players(players, H, data_analytics)
            data_analytics.step(1)

    # ---- fused single pass -------------------------------------------------------------------------------------
    def _ball_median(self, tracker: BallTracker, src, total: int, rank: int, dist_on: bool):
        """Background median of the ball tracker.  The reference takes it from the first `median_max_sample_num`
        frames of the VIDEO (iterable.py:58-73): under sharding rank 0 computes it from those frames (device
        selection kernel) and broadcasts it, so every shard feeds TrackNet the same background."""
        import torch.distributed as dist

        if tracker.median is not None:
            return tracker.median
        from .ball_tracker import median_background

        med = None
        if rank == 0:
            med = median_background(list(frames.read(src, 0, min(total, tracker.median_max_sample_num))))
        if dist_on:
            dev = _comm_device()
            shape = torch.zeros(3, dtype=torch.int64, device=dev)
            if rank == 0:
                shape = torch.tensor(med.shape, dtype=torch.int64, device=dev)
            dist.broadcast(shape, src=0)
            buf = torch.from_numpy(med).to(dev) if rank == 0 else \
                torch.empty(tuple(int(v) for v in shape.tolist()), dtype=torch.uint8, device=dev)
            dist.broadcast(buf, src=0)
            med = buf.cpu().numpy()
        return med

    def _run_fused(self, model: dict, src, total: int, lo: int, hi: int, rank: int, world: int, dist_on: bool):
        """One pass over this rank's frames for every tracker in `model`.  A ball shard needs 7 frames of history and
        7 of look-ahead (`ball_shard_frames`); the YOLO results of those halo frames are simply dropped."""
        ball = next((t for t in model.values() if t.stage == "ball"), None)
        flo, fhi = ball_shard_frames(total, lo, hi) if ball is not None else (lo, hi)
        B = min(t.batch_size for t in model.values())  # every engine is sized for its own tracker's batch_size
        for t in model.values():
            t.to(t.DEVICE)
        t0 = timeit.default_timer()
        median = self._ball_median(ball, src, total, rank, dist_on) if ball is not None else None
        t_med = timeit.default_timer() - t0
        chunks = frames.chunks(frames.read(src, flo, fhi), B)
        first = next(chunks, None)
        parts = {n: [] for n in model}
        hw = None
        if first is not None:
            hw = tuple(first[0].shape[1:3])
            fp = FusedPass(model, hw, B, total_frames=total, first_frame=flo, emit_range=(lo, hi), raw=dist_on,
                           median=median)
            pos = flo
            for out in fp.run(itertools.chain([first], chunks)):
                for name, t in model.items():
                    res = out[name]
                    if t.stage == "ball":
                        parts[name].append(res)
                    else:  # ResultBlocks under torch.distributed (raw), else post-processed objects
                        a, b = max(lo - pos, 0), min(hi - pos, len(res))  # halo frames of a ball shard are dropped
                        if b > a:
                            parts[name].append(res[a:b])
                pos += B  # every chunk but the last holds B frames
        torch.cuda.synchronize()
        t_pass = timeit.default_timer() - t0
        t1 = timeit.default_timer()
        for name, t in model.items():
            if t.stage == "ball":
                xyv = {}
                for d in parts[name]:
                    xyv.update(d)
                part = _ball_records(xyv, lo, hi)
            elif dist_on:
                part = (_yolo_records(parts[name], t), hw)
            else:
                part = [o for p in parts[name] for o in p]  # already post-processed objects, in frame order
            self._gather_and_assemble(t, part, total, rank, world, dist_on)
            self.timings[name] = t_pass  # one shared pass: per-tracker times are not separable
            t.to("cpu")
            if rank == 0:
                t.save_predictions()
        self.timings["_fused_pass"] = t_pass
        self.timings["_median"] = t_med
        self.timings["_gather_assemble"] = timeit.default_timer() - t1

    def _gather_and_assemble(self, tracker: Tracker, part, total: int, rank: int, world: int, dist_on: bool) -> None:
        if not dist_on:
            if rank == 0:
                self._assemble(tracker, [part], total)
            return
        import torch.distributed as dist

        if isinstance(part, tuple) and isinstance(part[0], YoloRecords):
            gathered = [(r, part[1]) for r in _all_gather_yolo(part[0], total, rank, world)]
        elif isinstance(part, BallRecords):
            gathered = _all_gather_ball(part, total, rank, world)
        else:  # cached / fixed objects: ragged Python lists, gathered as objects
            gathered = [None] * world if rank == 0 else None
            dist.gather_object(part, gathered, dst=0)
        if rank == 0:
            self._assemble(tracker, gathered, total)

    @staticmethod
    def _assemble(tracker: Tracker, parts: list, total: int) -> None:
        if tracker.stage == "ball":
            xyv = {}
            for p in parts:
                xyv.update(p.to_dict() if isinstance(p, BallRecords) else p)
            tracker.results.predictions = tracker.balls(xyv, total)  # InpaintNet: after the shards are merged
        elif parts and isinstance(parts[0], tuple):  # (YoloRecords, frame size) per shard
            hw = next((h for _, h in parts if h), None)
            results = ResultBlock.concat([res.to_results(tracker) for res, _ in parts])
            tracker.results.predictions = tracker.postprocess(results, hw)  # ordered => ByteTrack ids are consistent
        else:
            tracker.results.predictions = [o for p in parts for o in p]

    # ---- a list of clips in one pass ----------------------------------------------------------------------------
    def run_clips(self, clips: list, save_dir: Optional[str] = None, streams: Optional[int] = None,
                  inference_dir: Optional[str] = None, collect_data: bool = False) -> list[dict]:
        """Track a list of clips in one pass and return, per clip, {tracker name: list[Object]}: the results a fresh
        `TrackingRunner(trackers, video_info=<the clip's>).run()` gives on that clip alone.

        clips: video paths, or (frame_source, total_frames) pairs where frame_source(lo, hi) yields the clip's frames
        lo..hi-1 as HWC uint8 BGR frames or (n,H,W,3) uint8 batches (pinned host or device tensors); pairs take
        their fps from this runner's video_info.  Every clip must have the frame size of the first one.

        The clips are played back to back through one `ClipPass` (one upload per batch, one batch of look-ahead, the
        stream modes of FusedPass), so device batches stay full across clip boundaries and the next clip decodes
        while the device works.  Per clip: the ball background is the median of the clip's first
        `median_max_sample_num` frames (unless the BallTracker has a fixed `median`), InpaintNet runs over the clip's
        trajectory, and ByteTrack restarts at the clip's fps.  Trackers with a fixed keypoints detection repeat it.
        With `save_dir`, each clip's predictions are written as `<save_dir>/<clip:04d>_<tracker>.json` in the format
        of `save_predictions`.  The trackers' own `results` are left untouched.

        inference_dir: each clip's annotated video is written to `<inference_dir>/<clip:04d>.mp4` (mp4v, the clip's
        fps and frame size), the frames `TrackingRunner(trackers, video_info=<the clip's>, inference_path=...).run()`
        writes for that clip alone.  collect_data: `clips_data_analytics` holds one `DataAnalytics` per clip, each
        equal to that run's `data_analytics`; with `save_dir` each is also written as `<save_dir>/<clip:04d>_data.csv`
        (`into_dataframe(<clip fps>).to_csv`).  Without `inference_dir` the positions are collected without reading
        a frame again.  A clip of 0 frames gets no video and an empty `DataAnalytics` (no frames).  The clips are
        rendered in one pass after the tracking pass (`_render_clips`).

        Under torch.distributed (world size > 1) the clips are sharded over the ranks (`_run_clips_sharded`): each
        rank tracks and renders only its own clips and writes only their files, and every rank returns every clip's
        results."""
        import gc

        import torch.distributed as dist

        srcs, lengths, fps, hw = self._clip_sources(clips)
        sharded = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        gc_was_on = gc.isenabled()
        gc.disable()
        try:
            with self._clip_state():
                if sharded:
                    return self._run_clips_sharded(srcs, lengths, fps, hw, save_dir, streams, inference_dir,
                                                   collect_data)
                out, hw = self._run_clips(srcs, lengths, fps, hw, streams)
                if inference_dir or collect_data:
                    infos = self._clip_infos(hw, fps, lengths)
                    t0 = timeit.default_timer()
                    self._render_clip_files(srcs, infos, out, inference_dir, collect_data)
                    self.timings["_clips_render"] = timeit.default_timer() - t0
        finally:
            if gc_was_on:
                gc.enable()
        if save_dir is not None:
            self._save_clips(save_dir, range(len(out)), out, self.clips_data_analytics if collect_data else None, fps)
        return out

    def _clip_infos(self, hw, fps: list, lengths: list[int]) -> list:
        if hw is None and lengths:  # no frame was read: (source, length) pairs, fixed detections only
            hw = (self.video_info.height, self.video_info.width)
        return [sv.VideoInfo(width=hw[1], height=hw[0], fps=f, total_frames=T) for f, T in zip(fps, lengths)]

    @staticmethod
    def _save_clips(save_dir: str, which: Iterable[int], results: list[dict], das: Optional[list], fps: list) -> None:
        """Clips `which`: `<clip:04d>_<tracker>.json` (the `save_predictions` format) and, with `das`, `_data.csv`
        (main.py:180-181 per clip)."""
        import json

        os.makedirs(save_dir, exist_ok=True)
        for c in which:
            for name, objs in results[c].items():
                with open(os.path.join(save_dir, f"{c:04d}_{name}.json"), "w") as f:
                    json.dump([o.serialize() for o in objs], f)
            if das is not None:
                das[c].into_dataframe(fps[c]).to_csv(os.path.join(save_dir, f"{c:04d}_data.csv"))

    def _run_clips_sharded(self, srcs: list, lengths: list[int], fps: list, hw, save_dir: Optional[str],
                           streams: Optional[int], inference_dir: Optional[str], collect_data: bool) -> list[dict]:
        """run_clips over the ranks of a torch.distributed job.  `plan_clip_shards` gives each rank whole clips; the
        rank runs every per-clip stage of its own clips (`_run_clips`: background, ByteTrack restart, InpaintNet) and
        never reads another rank's clip.  After the pass the ranks exchange once: first each rank's status (its
        error, the frame size it saw), so that a failure or a frame-size mismatch on any rank raises `ValueError` on
        every rank instead of leaving one blocked in a collective; then every clip's results as dense arrays
        (`exchange_clip_results`).  Each rank renders its own clips (`_render_clip_files`, files named by the global
        clip index) and writes their JSON and CSV files; the ranks are assumed to share `save_dir` and
        `inference_dir`.  The render ends with a second status exchange that also carries the clips' `DataAnalytics`,
        so every rank's `clips_data_analytics` holds every clip's, in clip order."""
        import torch.distributed as dist

        rank, world = dist.get_rank(), dist.get_world_size()
        mine = plan_clip_shards(lengths, world)[rank]
        own = seen = failure = cause = None
        self._clip_reading = None
        try:
            own, seen = self._run_clips([srcs[c] for c in mine], [lengths[c] for c in mine], [fps[c] for c in mine],
                                        hw, streams, clip_ids=mine)
        except Exception as e:  # every rank must reach the status exchange
            failure, cause = (self._clip_reading, f"{type(e).__name__}: {e}"), e
        t0 = timeit.default_timer()
        seen = exchange_clip_status(failure, seen, next((c for c in mine if lengths[c]), None), cause)
        hw = hw if seen is None else seen
        fixed = {n: t.fixed_detection for n, t in self.trackers.items() if t.stage == "fixed"}
        out = exchange_clip_results(dict(zip(mine, own)), lengths, list(self.trackers), fixed)
        self.timings["_clips_exchange"] = timeit.default_timer() - t0
        das = None
        if inference_dir or collect_data:
            infos = self._clip_infos(hw, fps, lengths)
            failure = cause = None
            t0 = timeit.default_timer()
            try:
                self._render_clip_files([srcs[c] for c in mine], [infos[c] for c in mine], own, inference_dir,
                                        collect_data, clip_ids=mine)
            except Exception as e:
                failure, cause = (None, f"{type(e).__name__}: {e}"), e
            self.timings["_clips_render"] = timeit.default_timer() - t0
            t0 = timeit.default_timer()
            own_das = dict(zip(mine, self.clips_data_analytics)) if collect_data and failure is None else {}
            das = exchange_clip_data(failure, own_das, cause)
            if collect_data:
                self.clips_data_analytics = das
            else:
                das = None
            self.timings["_clips_exchange"] += timeit.default_timer() - t0
        if save_dir is not None:
            self._save_clips(save_dir, mine, out, das, fps)
        return out

    def _render_clip_files(self, srcs: list, infos: list, results: list[dict], inference_dir: Optional[str],
                           collect_data: bool, clip_ids: Optional[list[int]] = None) -> None:
        """run_clips' drawing pass (`_render_clips`; a clip that yields fewer frames than announced raises): clip c's
        video to `<inference_dir>/<clip id:04d>.mp4`, one `DataAnalytics` per clip into `clips_data_analytics` when
        collecting.  clip_ids: the clips' numbers in file names and messages (default 0, 1, ...)."""
        ids = list(range(len(infos))) if clip_ids is None else list(clip_ids)
        paths = None
        if inference_dir:
            paths = [os.path.join(inference_dir, f"{c:04d}.mp4") for c in ids]
            if any(vi.total_frames for vi in infos):
                os.makedirs(inference_dir, exist_ok=True)
        das = [DataAnalytics() for _ in infos] if collect_data else None
        court = ProjectedCourt(infos[0]) if infos else None
        self._render_clips(srcs, infos, results, court, das, paths, exact=True, prefix="_clips_render", clip_ids=ids)
        if das is not None:
            self.clips_data_analytics = das

    def _clip_sources(self, clips: list):
        """(frame sources, lengths, fps, frame size or None when only the frames can tell) of the clips."""
        srcs, lengths, fps, hw = [], [], [], None
        for i, clip in enumerate(clips):
            if isinstance(clip, (str, os.PathLike)):
                vi = sv.VideoInfo.from_video_path(str(clip))
                srcs.append((lambda p: lambda lo, hi: sv.get_video_frames_generator(p, start=lo, end=hi))(str(clip)))
                lengths.append(int(vi.total_frames))
                fps.append(vi.fps)
                if hw is None:
                    hw = (vi.height, vi.width)
                elif (vi.height, vi.width) != hw:
                    raise ValueError(f"clip {i} is {vi.width}x{vi.height}, clip 0 is {hw[1]}x{hw[0]}: "
                                     "all clips of one call must have the same frame size")
            else:
                src, total = clip
                if self.video_info is None:
                    raise ValueError("clips given as (frame_source, total_frames) take their fps from the runner's "
                                     "video_info, and this runner has none")
                srcs.append(src)
                lengths.append(int(total))
                fps.append(self.video_info.fps)
        if any(t < 0 for t in lengths):
            raise ValueError("clip lengths must be >= 0")
        return srcs, lengths, fps, hw

    def _run_clips(self, srcs: list, lengths: list[int], fps: list, hw, streams: Optional[int],
                   clip_ids: Optional[list[int]] = None):
        """The tracking pass of run_clips -> (per-clip results, frame size or None when no frame was read).
        clip_ids: the clips' numbers in messages and in `_clip_reading`, the clip whose frames were read last
        (default 0, 1, ...)."""
        from .ball_tracker import median_background_device

        ids = list(range(len(srcs))) if clip_ids is None else list(clip_ids)
        fixed = {n: t for n, t in self.trackers.items() if t.stage == "fixed"}
        model = _batch_trackers(self.trackers)
        other = set(self.trackers) - set(fixed) - set(model)
        if other:
            raise ValueError(f"run_clips: trackers {sorted(other)} have no batch model stage (a YOLO or ball model) "
                             "and no fixed detection")
        out = [{n: [t.fixed_detection] * T for n, t in fixed.items()} for T in lengths]
        if not model or not sum(lengths):
            for res, T in zip(out, lengths):
                res.update({n: [] for n in model})
            return out, hw
        ball_name, ball = next(((n, t) for n, t in model.items() if t.stage == "ball"), (None, None))
        B = min(t.batch_size for t in model.values())
        side = torch.cuda.Stream()  # backgrounds of the clips ahead are computed beside the pass
        meds: dict = {}
        shape = {"hw": hw}

        def clip_pieces(c):
            """clip c's frames as (n,H,W,3) uint8 tensors, after queueing its background when it needs one"""
            self._clip_reading = ids[c]
            it = frames.read(srcs[c], 0, lengths[c], shape["hw"], exact=True, clip=ids[c])
            if ball is not None and lengths[c] >= 8:
                if ball.median is not None:
                    if "fixed" not in meds:
                        meds["fixed"] = (torch.as_tensor(ball.median).to(torch.uint8).cuda(), None)
                    meds[c] = meds["fixed"]
                else:  # iterable.py:58-73 per clip, as TrackingRunner._ball_median does for one video
                    first, it = frames.head(it, min(lengths[c], ball.median_max_sample_num))
                    with torch.cuda.stream(side):
                        med = median_background_device(first)
                        ready = torch.cuda.Event()
                        ready.record(side)
                    meds[c] = (med, ready)
                    it = itertools.chain(first, it)
            for t in it:
                shape["hw"] = tuple(t.shape[1:3])  # the first frames read fix the size every later clip must have
                yield t

        for t in model.values():
            t.to(t.DEVICE)
        t0 = timeit.default_timer()
        gen = frames.chunks((t for c in range(len(srcs)) for t in clip_pieces(c)), B)
        first = next(gen)
        hw = shape["hw"]
        infos = [sv.VideoInfo(width=hw[1], height=hw[0], fps=f, total_frames=T) for f, T in zip(fps, lengths)]
        fp = ClipPass(model, hw, B, lengths, infos, lambda c: meds[c], streams=streams)
        yolo = {n: [[] for _ in lengths] for n in model if n != ball_name}
        xyv = [{} for _ in lengths]
        left = [T if T >= 8 else 0 for T in lengths]
        inpaint_stream = torch.cuda.Stream()

        def finish_ball(c):
            """InpaintNet over the clip's trajectory (on a stream of its own: the pass keeps running) -> Ball list"""
            ball.video_info = infos[c]
            with torch.cuda.stream(inpaint_stream):
                out[c][ball_name] = ball.balls(xyv[c], lengths[c])

        for res in fp.run(itertools.chain([first], gen)):
            for name, parts in res.items():
                if name == ball_name:
                    for c, f, v in parts:
                        xyv[c][f] = v
                        left[c] -= 1
                        if left[c] == 0:
                            finish_ball(c)
                else:
                    for c, objs in parts:
                        yolo[name][c] += objs
        torch.cuda.synchronize()
        if ball is not None:
            for c, T in enumerate(lengths):
                if ball_name not in out[c]:  # clips of fewer than 8 frames have no window
                    finish_ball(c)
        for name, per_clip in yolo.items():
            for c, objs in enumerate(per_clip):
                out[c][name] = objs
        for t in model.values():
            t.to("cpu")
        self.timings["_clips_pass"] = timeit.default_timer() - t0
        return [{n: res[n] for n in self.trackers} for res in out], hw


# ---- fixed-capacity records for the gather (SURVEY §8e) ---------------------------------------------------------
class YoloRecords:
    """Detections of consecutive frames as one dense float32 block (frames, cap, 6 + K*D) + int32 counts: rows are
    [x1, y1, x2, y2, conf, cls, keypoints...] exactly as the engine's ResultBlock holds them."""

    def __init__(self, rows: torch.Tensor, counts: torch.Tensor, kpt_shape):
        self.rows, self.counts, self.kpt_shape = rows, counts, kpt_shape

    def to_results(self, tracker) -> ResultBlock:
        return ResultBlock(self.rows.numpy(), self.counts.numpy(), self.kpt_shape, tracker.model.names, None)


class BallRecords:
    """(x, y, visibility, present) int32 per frame of a contiguous range starting at `first`."""

    def __init__(self, first: int, data: torch.Tensor):
        self.first, self.data = first, data

    def to_dict(self) -> dict:
        return {self.first + i: (int(x), int(y), int(v)) for i, (x, y, v, p) in enumerate(self.data.tolist()) if p}


def _yolo_records(blocks: list, tracker) -> YoloRecords:
    """This rank's frames (a list of per-batch ResultBlocks) as one padded block."""
    kpt_shape = tracker.model.kpt_shape
    rowlen = 6 + (kpt_shape[0] * kpt_shape[1] if kpt_shape else 0)
    empty = ResultBlock(np.zeros((0, 1, rowlen), np.float32), np.zeros((0,), np.int32), kpt_shape, None, None)
    blk = ResultBlock.concat(blocks, like=empty)
    return YoloRecords(torch.from_numpy(blk.rows), torch.from_numpy(blk.counts), kpt_shape)


def _ball_records(xyv: dict, lo: int, hi: int) -> BallRecords:
    data = np.zeros((hi - lo, 4), dtype=np.int32)
    own = [(n - lo, x, y, v) for n, (x, y, v) in xyv.items() if lo <= n < hi]
    if own:
        a = np.asarray(own, dtype=np.int64)
        data[a[:, 0], :3] = a[:, 1:]
        data[a[:, 0], 3] = 1
    return BallRecords(lo, torch.from_numpy(data))


def _clip_render_batches(srcs: list, lengths: list[int], batch_size: int, hw: tuple[int, int],
                         clip_ids: Optional[list[int]] = None, exact: bool = True) -> Iterable[list[torch.Tensor]]:
    """The frames of the clips played back to back, re-read from their sources (`frames.read`: exact, or ending
    where a source ends), in upload batches of `batch_size` that cross clip boundaries (`frames.chunks`).  clip_ids:
    the clips' numbers in messages (default 0, 1, ...)."""
    ids = list(range(len(srcs))) if clip_ids is None else list(clip_ids)
    pieces = (p for c, T in enumerate(lengths) for p in frames.read(srcs[c], 0, T, hw, exact, ids[c]))
    return frames.chunks(pieces, batch_size)


# ---- run_clips over ranks: the exchange after the pass ------------------------------------------------------------
def _all_gather(obj) -> list:
    """Every rank's `obj`, in rank order (all_gather_object: gloo, or NCCL on the current device)."""
    import torch.distributed as dist

    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def _raise_on_failure(failures: list, cause: Optional[BaseException]) -> None:
    """failures: per rank, None or (clip or None, message).  Every rank raises the same ValueError when any failed."""
    bad = [f"rank {r}" + ("" if f[0] is None else f", clip {f[0]}") + f": {f[1]}"
           for r, f in enumerate(failures) if f is not None]
    if bad:
        raise ValueError("run_clips failed on " + "; ".join(bad)) from cause


def exchange_clip_status(failure: Optional[tuple], hw: Optional[tuple], clip: Optional[int],
                         cause: Optional[BaseException] = None) -> Optional[tuple]:
    """The status exchange after a rank's tracking pass: failure = None or (clip or None, message); hw = the frame
    size the rank saw (None if it read no frame), first at `clip`.  Every rank raises ValueError if any rank failed or
    if two ranks saw different frame sizes; otherwise returns the frame size seen (None if no rank read a frame)."""
    statuses = _all_gather((failure, None if hw is None else tuple(hw), clip))
    _raise_on_failure([s[0] for s in statuses], cause)
    sizes = [(c, h) for _, h, c in statuses if h is not None]
    for c, h in sizes[1:]:
        if h != sizes[0][1]:
            raise ValueError(f"clip {c} has {h} frames, clip {sizes[0][0]} {sizes[0][1]}: all clips of one call must "
                             "have the same frame size")
    return sizes[0][1] if sizes else None


def exchange_clip_results(own: dict[int, dict[str, list]], lengths: list[int], names: list[str],
                          fixed: dict[str, object]) -> list[dict[str, list]]:
    """Every clip's results on every rank.  own: {clip: {tracker name: list[Object]}} of this rank's clips (the
    objects are returned as they are); every other clip's are rebuilt from the dense arrays its owner sends
    (`_pack_objects`), `serialize()`-equal to the owner's.  fixed: {tracker name: fixed detection}, repeated per frame
    on every rank rather than sent.  Returns one {tracker name: list[Object]} per clip, in clip order, with the
    trackers in `names` order."""
    packed = {c: {n: _pack_objects(objs) for n, objs in res.items() if n not in fixed} for c, res in own.items()}
    theirs = {}
    for part in _all_gather(packed):
        theirs.update(part)
    out = []
    for c, T in enumerate(lengths):
        if c in own:
            out.append(own[c])
        else:
            out.append({n: [fixed[n]] * T if n in fixed else _unpack_objects(theirs[c][n]) for n in names})
    return out


def exchange_clip_data(failure: Optional[tuple], own: dict[int, DataAnalytics],
                       cause: Optional[BaseException] = None) -> list[DataAnalytics]:
    """The status exchange after a rank's render, carrying its clips' DataAnalytics (as `into_dict` columns).  Every
    rank raises ValueError if any rank failed; otherwise returns the DataAnalytics of every clip any rank sent, in clip
    order (this rank's own objects, the others rebuilt with `from_dict`: equal `frames`, `len()` and
    `into_dataframe`)."""
    statuses = _all_gather((failure, {c: da.into_dict() for c, da in own.items()}))
    _raise_on_failure([s[0] for s in statuses], cause)
    theirs = {c: d for _, part in statuses for c, d in part.items()}
    return [own[c] if c in own else DataAnalytics.from_dict(theirs[c]) for c in sorted(theirs)]


def _pair_is_int(xy) -> bool:
    return isinstance(xy[0], (int, np.integer)) and isinstance(xy[1], (int, np.integer))


def _pair(x: float, y: float, is_int: bool) -> tuple:
    return (int(x), int(y)) if is_int else (float(x), float(y))


def _pack_objects(objs: list) -> tuple:
    """One clip's results of one tracker (the tracking pass's objects, which carry no projection) as (kind, per-frame
    counts, dense per-row arrays).  Coordinates go as float64 with a per-row flag for (int, int) pairs, so the rebuilt
    objects serialise to the same JSON, ints and floats alike."""
    from .keypoints_tracker import Keypoints
    from .players_keypoints_tracker import PlayerKeypoints, PlayersKeypoints

    if not objs:
        return ("empty",)
    first = objs[0]
    if isinstance(first, Players):
        counts, xyxy, ids, has_id, cls, conf = [], [], [], [], [], []
        for p in objs:
            if p._list is None:
                x, i, k, s = p._rows
                n = len(x)
                ids.append(np.zeros(n, np.int64) if i is None else np.asarray(i, np.int64))
                has_id.append(np.full(n, i is not None))
            else:
                pl = p._list
                n = len(pl)
                x, k, s = [q.xyxy for q in pl], [q.class_id for q in pl], [q.confidence for q in pl]
                ids.append(np.array([-1 if q.id is None else q.id for q in pl], np.int64))
                has_id.append(np.array([q.id is not None for q in pl], bool))
            counts.append(n)
            xyxy.append(np.asarray(x).reshape(n, 4))
            cls.append(np.asarray(k, np.int64).reshape(n))
            conf.append(np.asarray(s).reshape(n))
        return ("players", np.asarray(counts, np.int64), np.concatenate(xyxy), np.concatenate(ids),
                np.concatenate(has_id), np.concatenate(cls), np.concatenate(conf))
    if isinstance(first, PlayersKeypoints):
        K = len(PlayerKeypoints.KEYPOINTS_NAMES)
        xy = [np.asarray(p._xy if p._list is None else [[k.xy for k in pk] for pk in p._list], np.float64)
              for p in objs]
        xy = [a.reshape(len(a), K, 2) for a in xy]
        return ("players_keypoints", np.asarray([len(a) for a in xy], np.int64), np.concatenate(xy))
    if isinstance(first, Keypoints):
        kps = [k for o in objs for k in o.keypoints]
        return ("keypoints", np.asarray([len(o.keypoints) for o in objs], np.int64),
                np.asarray([k.id for k in kps], np.int64).reshape(-1),
                np.asarray([k.xy for k in kps], np.float64).reshape(-1, 2),
                np.asarray([_pair_is_int(k.xy) for k in kps], bool).reshape(-1))
    if isinstance(first, Ball):
        return ("ball", np.asarray([b.frame for b in objs], np.int64), np.asarray([b.xy for b in objs], np.float64),
                np.asarray([_pair_is_int(b.xy) for b in objs], bool), np.asarray([b.visibility for b in objs], np.int64))
    raise TypeError(f"no dense form for {type(first).__name__} results")


def _unpack_objects(packed: tuple) -> list:
    """`_pack_objects` inverted: the objects, through the array-backed constructors where there are some."""
    from .keypoints_tracker import Keypoint, Keypoints
    from .players_keypoints_tracker import PlayersKeypoints
    from .players_tracker import Player

    kind = packed[0]
    if kind == "empty":
        return []
    if kind == "ball":
        _, frame, xy, is_int, vis = packed
        return [Ball(frame=f, xy=_pair(x, y, i), visibility=v)
                for f, (x, y), i, v in zip(frame.tolist(), xy.tolist(), is_int.tolist(), vis.tolist())]
    ends = np.cumsum(packed[1]).tolist()
    starts = [0] + ends[:-1]
    if kind == "players":
        _, _, xyxy, ids, has_id, cls, conf = packed
        out = []
        for a, b in zip(starts, ends):
            h = has_id[a:b]
            if h.all():
                out.append(Players.from_rows(xyxy[a:b], ids[a:b], cls[a:b], conf[a:b]))
            elif not h.any():
                out.append(Players.from_rows(xyxy[a:b], None, cls[a:b], conf[a:b]))
            else:  # ids on some players only: only a list of players holds that
                out.append(Players([Player.from_row(xyxy[i], ids[i] if has_id[i] else None, cls[i], conf[i])
                                    for i in range(a, b)]))
        return out
    if kind == "players_keypoints":
        xy = packed[2]
        return [PlayersKeypoints.from_xy(xy[a:b]) for a, b in zip(starts, ends)]
    if kind == "keypoints":
        _, _, ids, xy, is_int = packed
        ids, xy, is_int = ids.tolist(), xy.tolist(), is_int.tolist()
        return [Keypoints([Keypoint(id=ids[i], xy=_pair(*xy[i], is_int[i])) for i in range(a, b)])
                for a, b in zip(starts, ends)]
    raise ValueError(f"unknown packed kind {kind!r}")


def _comm_device() -> torch.device:
    import torch.distributed as dist

    return torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")


def _all_gather_yolo(rec: YoloRecords, total: int, rank: int, world: int) -> list[YoloRecords]:
    """all_gather of padded fixed-capacity blocks: capacity = the global maximum detections per frame (one MAX
    all-reduce), frames padded to the longest shard.  Every rank receives every block; rank 0 uses them."""
    import torch.distributed as dist

    dev = _comm_device()
    npad = max(shard_range(total, r, world)[1] - shard_range(total, r, world)[0] for r in range(world))
    cap = torch.tensor([rec.rows.shape[1]], dtype=torch.int64, device=dev)
    dist.all_reduce(cap, op=dist.ReduceOp.MAX)
    cap = int(cap.item())
    rowlen = rec.rows.shape[2]
    rows = torch.zeros((npad, cap, rowlen), dtype=torch.float32, device=dev)
    counts = torch.zeros((npad,), dtype=torch.int32, device=dev)
    n = rec.rows.shape[0]
    rows[:n, : rec.rows.shape[1]] = rec.rows.to(dev)
    counts[:n] = rec.counts.to(dev)
    all_rows = [torch.empty_like(rows) for _ in range(world)]
    all_counts = [torch.empty_like(counts) for _ in range(world)]
    dist.all_gather(all_rows, rows)
    dist.all_gather(all_counts, counts)
    out = []
    for r in range(world):
        a, b = shard_range(total, r, world)
        out.append(YoloRecords(all_rows[r][: b - a].cpu(), all_counts[r][: b - a].cpu(), rec.kpt_shape))
    return out


def _all_gather_ball(rec: BallRecords, total: int, rank: int, world: int) -> list[BallRecords]:
    import torch.distributed as dist

    dev = _comm_device()
    npad = max(shard_range(total, r, world)[1] - shard_range(total, r, world)[0] for r in range(world))
    data = torch.zeros((npad, 4), dtype=torch.int32, device=dev)
    data[: rec.data.shape[0]] = rec.data.to(dev)
    parts = [torch.empty_like(data) for _ in range(world)]
    dist.all_gather(parts, data)
    out = []
    for r in range(world):
        a, b = shard_range(total, r, world)
        out.append(BallRecords(a, parts[r][: b - a].cpu()))
    return out
