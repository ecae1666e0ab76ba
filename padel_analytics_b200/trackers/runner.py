"""TrackingRunner: the per-tracker pass over a video (API of /root/reference/trackers/runner.py:37-236), plus the
multi-GPU sharded variant (SURVEY §8e): one process per GPU, contiguous frame ranges, no per-batch collectives —
detections are gathered once per tracker and the sequential host stages (ByteTrack ids, JSON) run on rank 0.

Every pass reads its frame sources through `frames.py` (`read`, `chunks`, `head`).  After the trackers, `run()`
renders the annotated video to `inference_path` and collects the players' court positions into `data_analytics`
(runner.py:91-173) when either is asked for; the overlays are composited on the device (render.py,
`pb_render_overlay`) and encoding runs on a thread of its own.  `run_clips()` does the same per clip for a list of
clips.  Both draw through one render pass over clips played back to back (`_render_clips`; `run()`'s video is one
clip).  Under torch.distributed `run_clips()` shards whole clips over the ranks (`plan_clip_shards`) and exchanges the
results once after the pass.

Documented deviations from reference quirks (SURVEY App. E):
  q7  with collect_data=False the reference's drawing pass ends by trimming `self.data_analytics.frames`, which is
      None, and raises AttributeError; here the trim happens only when data is collected.
  No per-frame prints; `data_analytics` is also filled when no video is written (collect_data=True without an
  inference_path), without rendering any frame.
"""
from __future__ import annotations

import contextlib
import itertools
import os
import timeit
from typing import Callable, Iterable, Optional

import numpy as np
import torch

from . import frames
from . import sv_compat as sv
from ..engine.yolo_engine import ResultBlock
from .ball_tracker import Ball, BallTracker
from .keypoints_tracker import Keypoints, KeypointsTracker
from .players_keypoints_tracker import PlayerKeypointsTracker
from .players_tracker import PlayerTracker, Players
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

    def __init__(self, trackers: dict[str, Tracker], frame_hw: tuple[int, int], batch_size: int, total_frames: int,
                 first_frame: int = 0, emit_range: Optional[tuple[int, int]] = None, streams: Optional[int] = None,
                 raw: bool = False, median=None):
        """raw=True: the YOLO trackers' entries are the engines' raw per-frame Results (no polygon filter / ByteTrack /
        result objects) -- what a shard hands to rank 0, where the order-dependent host stages run once over the
        ordered gather.  median: background for the ball tracker (defaults to BallTracker.median)."""
        self.trackers = trackers
        self.raw = raw
        self.mode = int(os.environ.get("PADEL_B200_STREAMS", "1")) if streams is None else streams
        # side streams: the YOLO chains at high priority (their CTAs are placed first whenever SMs free up), the ball
        # tracker (mode 2 only) at normal priority
        self.side = {name: torch.cuda.Stream(priority=0 if isinstance(t, BallTracker) else -1)
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
            if isinstance(t, BallTracker):
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
            order.sort(key=lambda kv: isinstance(kv[1], BallTracker))
        for name, t in order:  # enqueue everything first ...
            if getattr(t, "fixed_keypoints_detection", None) is not None:
                pending.append((name, t, None))
                continue
            is_ball = isinstance(t, BallTracker)
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
        pending, nfr = launched
        out = {}
        for name, t, fin in pending:  # ... then finish in the same order
            if isinstance(t, BallTracker):
                out[name] = fin()
            elif fin is None:
                out[name] = [t.fixed_keypoints_detection] * nfr
            elif self.raw:
                out[name] = fin()
            elif isinstance(t, PlayerTracker):
                out[name] = t.postprocess(fin())
            else:
                out[name] = t.postprocess(fin(), self.hw)
        return out

    def run(self, batches: Iterable):
        """batches: iterable of uint8 (n,H,W,3) BGR batches, n <= batch_size, each a pinned host or device tensor or a
        list of such pieces (`frames.chunks`).  Yields one {tracker name: results} dict per batch.

        One batch of look-ahead: batch i+1 is pulled from `batches` and enqueued before batch i's results are yielded.
        A batch (host pieces: copied asynchronously into a staging slot; one device tensor: read in place) must stay
        untouched until ITS OWN results have been yielded, i.e. a producer that reuses buffers needs at least two."""
        it = iter(batches)
        main = torch.cuda.current_stream()

        def start(batch, i):
            """upload (copy stream) + enqueue all device work of batch i; returns the launch record"""
            dev = self._upload(batch, i % 2)
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
            if isinstance(t, BallTracker):
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
            if isinstance(t, BallTracker):
                out[name] = fin()
                continue
            res, parts = fin(), []
            for c, a, b, f0 in segs:
                if f0 == 0:
                    t.video_info_post_init(self.clip_infos[c])
                piece = res[a:b]
                parts.append((c, t.postprocess(piece) if isinstance(t, PlayerTracker) else t.postprocess(piece, self.hw)))
            out[name] = parts
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
        self.is_fixed_keypoints = any(getattr(t, "fixed_keypoints_detection", None) is not None
                                      for t in self.trackers.values() if isinstance(t, KeypointsTracker))
        self.collect_data = collect_data
        self.projected_court = ProjectedCourt(video_info) if video_info is not None else None
        self.data_analytics = DataAnalytics() if collect_data else None
        self.render_batch_size = 32
        self.clips_data_analytics: list[DataAnalytics] = []  # per clip, filled by run_clips(collect_data=True)
        self._source = None  # frame_source of the last run(), for the drawing pass
        self._clip_reading: Optional[int] = None  # run_clips: the clip whose frames the pass read last
        self.timings: dict[str, float] = {}

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

        fused (default: on when two or more trackers still need inference): ONE pass over the frames feeds every
        such tracker from a single decode + upload per batch (`FusedPass`; the reference decodes and uploads once per
        tracker, runner.py:215-220).  fused=False is the reference's plain loop, one full pass per tracker.
        Trackers with cached predictions (runner.py:187-191) or a fixed keypoints detection never enter the fused set.

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
        model = {n: t for n, t in todo.items() if isinstance(t, (PlayerTracker, PlayerKeypointsTracker, BallTracker))
                 or (isinstance(t, KeypointsTracker) and t.fixed_keypoints_detection is None and t.model is not None)}
        if fused is None:
            fused = len(model) >= 2 and torch.cuda.is_available()
        if fused and model:
            self._run_fused(model, src, total, lo, hi, rank, world, dist_on)
            todo = {n: t for n, t in todo.items() if n not in model}
        for name, tracker in todo.items():
            tracker.to(tracker.DEVICE)
            t0 = timeit.default_timer()
            if isinstance(tracker, BallTracker):
                flo, fhi = ball_shard_frames(total, lo, hi)
                median = self._ball_median(tracker, src, total, rank, dist_on)
                part = tracker.track_xyv(src(flo, fhi), total, first_frame=flo, emit_range=(lo, hi), median=median)
                part = _ball_records(part, lo, hi)
            elif isinstance(tracker, (PlayerTracker, PlayerKeypointsTracker, KeypointsTracker)) and \
                    getattr(tracker, "fixed_keypoints_detection", None) is None:
                part, hw = [], None
                for sample in sampler(src(lo, hi), tracker.batch_size):
                    hw = sample[0].shape[:2]
                    part += tracker.detect_sample(sample)
                part = (_yolo_records(part, tracker), hw)
            else:
                part = list(tracker.predict_and_update(src(lo, hi), total_frames=hi - lo).predictions)
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            self._gather_and_assemble(tracker, part, total, rank, world, dist_on)
            self.timings[name] = timeit.default_timer() - t0
            tracker.to("cpu")
            if rank == 0:
                tracker.save_predictions()
        return self.timings

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
        saved = {n: {k: t.__dict__[k] for k in ("video_info", "byte_track") if k in t.__dict__}
                 for n, t in self.trackers.items()}
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
        ball = next((t for t in model.values() if isinstance(t, BallTracker)), None)
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
                    if isinstance(t, BallTracker):
                        parts[name].append(out[name])
                    else:
                        res = out[name]
                        a, b = max(lo - pos, 0), min(hi - pos, len(res))  # halo frames of a ball shard are dropped
                        if b > a:
                            if isinstance(res, ResultBlock):
                                parts[name].append(res[a:b])
                            else:
                                parts[name] += res[a:b]
                pos += B  # every chunk but the last holds B frames
        torch.cuda.synchronize()
        t_pass = timeit.default_timer() - t0
        t1 = timeit.default_timer()
        for name, t in model.items():
            if isinstance(t, BallTracker):
                xyv = {}
                for d in parts[name]:
                    xyv.update(d)
                part = _ball_records(xyv, lo, hi)
            elif not dist_on or not all(isinstance(p, ResultBlock) for p in parts[name]):
                part = parts[name]  # already post-processed (or fixed) objects, in frame order
            else:
                part = (_yolo_records(parts[name], t), hw)
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
        if isinstance(tracker, BallTracker):
            xyv = {}
            for p in parts:
                xyv.update(p.to_dict() if isinstance(p, BallRecords) else p)
            xyv = tracker.inpaint_xyv(xyv, total)  # whole-trajectory stage: after the shards are merged
            tracker.results.predictions = [
                Ball(frame=n, xy=(xyv[n][0], xyv[n][1]), visibility=xyv[n][2]) if n in xyv
                else Ball(frame=n, xy=(0.0, 0.0), visibility=0) for n in range(total)]
        elif parts and isinstance(parts[0], tuple):
            hw = next((h for _, h in parts if h), None)
            if all(isinstance(res, YoloRecords) for res, _ in parts):  # dense records: stay dense
                results = ResultBlock.concat([res.to_results(tracker) for res, _ in parts])
            else:
                results = []
                for res, _ in parts:
                    results += list(res.to_results(tracker)) if isinstance(res, YoloRecords) else list(res)
            if isinstance(tracker, PlayerTracker):
                tracker.results.predictions = tracker.postprocess(results)  # ordered => ByteTrack ids are consistent
            else:
                tracker.results.predictions = tracker.postprocess(results, hw)
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
        fixed = {n: t.fixed_keypoints_detection for n, t in self.trackers.items()
                 if getattr(t, "fixed_keypoints_detection", None) is not None}
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
        fixed = {n: t for n, t in self.trackers.items() if getattr(t, "fixed_keypoints_detection", None) is not None}
        model = {n: t for n, t in self.trackers.items() if n not in fixed and (
            isinstance(t, (PlayerTracker, PlayerKeypointsTracker, BallTracker)) or
            (isinstance(t, KeypointsTracker) and t.model is not None))}
        other = set(self.trackers) - set(fixed) - set(model)
        if other:
            raise ValueError(f"run_clips: trackers {sorted(other)} have neither a model nor a fixed detection")
        out = [{n: [t.fixed_keypoints_detection] * T for n, t in fixed.items()} for T in lengths]
        if not model or not sum(lengths):
            for res, T in zip(out, lengths):
                res.update({n: [] for n in model})
            return out, hw
        ball_name, ball = next(((n, t) for n, t in model.items() if isinstance(t, BallTracker)), (None, None))
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
                v = ball.inpaint_xyv(xyv[c], lengths[c])
            out[c][ball_name] = [Ball(frame=n, xy=(v[n][0], v[n][1]), visibility=v[n][2]) if n in v
                                 else Ball(frame=n, xy=(0.0, 0.0), visibility=0) for n in range(lengths[c])]

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
    """This rank's frames (a list of per-batch ResultBlocks, or of Results) as one padded block."""
    kpt_shape = tracker.model.kpt_shape
    if blocks and not isinstance(blocks[0], ResultBlock):  # plain Results: one frame each
        rowlen = 6 + (kpt_shape[0] * kpt_shape[1] if kpt_shape else 0)
        one = []
        for r in blocks:
            n = len(r.boxes)
            rows = np.zeros((1, max(n, 1), rowlen), dtype=np.float32)
            rows[0, :n, :6] = r.boxes.data.numpy()
            if kpt_shape and n:
                rows[0, :n, 6:] = r.keypoints.data.numpy().reshape(n, rowlen - 6)
            one.append(ResultBlock(rows, np.array([n], dtype=np.int32), kpt_shape, r.names, r.orig_shape))
        blocks = one
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
