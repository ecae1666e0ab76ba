"""The render pass (the reference's runner.py:91-173): every frame annotated with the trackers' drawings, the
mini court and the projected players and ball, composited on the device.

Each frame's drawing is turned into a display list on the host.  Every primitive the reference draws is an
overwrite-only LINE_8 cv2 call (filled circles, 2-pixel lines and rectangles, Hershey text), so its effect is "these
pixels become this colour".  The host rasterises each call with the same cv2 function onto a small zeroed canvas (the
primitive's bounding box plus a margin, intersected with the frame, so that where cv2 clips, the canvas edge is the
frame edge), and the covered pixels become a coverage sprite.  Sprites are cached by shape and packed into a per-batch
atlas.  The background box is a BLEND record through a 256-entry table computed with the reference's own
cv2.addWeighted.  `pb_render_overlay` applies the records in draw order to the uploaded BGR frames.

The reference draws on an RGB copy and converts back before writing; a colour permutation is all that differs, so the
compositor works on the BGR frame and each record's colour has R and B swapped.
"""
from __future__ import annotations

import functools
import queue
import threading
import timeit
from dataclasses import dataclass
from typing import Callable, Iterable, Optional

import numpy as np

from . import _lib as L
from .analytics import DataAnalytics, ProjectedCourt

FRAME_TEXT_ORG = (20, 50)
FRAME_TEXT_COLOUR = (255, 255, 0)  # RGB

# the cv2 drawing calls a display list can hold, with their parameter names in positional order
_PARAMS = {
    "circle": ("img", "center", "radius", "color", "thickness", "lineType", "shift"),
    "line": ("img", "pt1", "pt2", "color", "thickness", "lineType", "shift"),
    "rectangle": ("img", "pt1", "pt2", "color", "thickness", "lineType", "shift"),
    "putText": ("img", "text", "org", "fontFace", "fontScale", "color", "thickness", "lineType", "bottomLeftOrigin"),
}
_record_lock = threading.Lock()


def record_draw_calls(draw: Callable, *args, **kwargs) -> list[tuple[str, dict]]:
    """Run `draw(frame, *args, **kwargs)` (an object's draw method) with cv2's drawing calls recorded instead of
    executed; returns [(function name, parameters)] in call order.  cv2 is patched for the duration of the call, so no
    other thread may draw with cv2 meanwhile."""
    import cv2

    calls = []
    frame = np.zeros((1, 1, 3), np.uint8)

    def recorder(name):
        names = _PARAMS[name]

        def rec(*a, **kw):
            p = dict(zip(names, a))
            p.update(kw)
            calls.append((name, p))
            return p["img"]
        return rec

    with _record_lock:
        saved = {n: getattr(cv2, n) for n in _PARAMS}
        try:
            for n in _PARAMS:
                setattr(cv2, n, recorder(n))
            draw(frame, *args, **kwargs)
        finally:
            for n, f in saved.items():
                setattr(cv2, n, f)
    return calls


def _pt(p) -> tuple[int, int]:
    return int(p[0]), int(p[1])


def _colour_bgr(c) -> int:
    """cv2 colour of a call on an RGB frame -> packed B | G << 8 | R << 16 of the BGR frame."""
    return _packed_colour(tuple(c) if not np.isscalar(c) else (c,))


@functools.lru_cache(maxsize=256)
def _packed_colour(c: tuple) -> int:
    c = list(c) + [0] * (3 - len(c))
    r, g, b = (int(min(255, max(0, round(float(v))))) for v in c[:3])
    return b | (g << 8) | (r << 16)


def _geometry(name: str, p: dict):
    """(anchor point, shape key, bounding box relative to the anchor as (x0, y0, x1, y1) exclusive) of one call.  The
    box holds every pixel cv2 can touch, with a margin."""
    import cv2

    th = int(p.get("thickness", 1))
    if int(p.get("lineType", cv2.LINE_8)) != cv2.LINE_8 or int(p.get("shift", 0)) != 0:
        raise ValueError(f"display list: cv2.{name} must be LINE_8 without shift")
    m = max(th, 1) + 2
    if name == "circle":
        r = int(p["radius"])
        return _pt(p["center"]), ("circle", r, th), (-r - m, -r - m, r + m + 1, r + m + 1)
    if name in ("line", "rectangle"):
        a, b = _pt(p["pt1"]), _pt(p["pt2"])
        dx, dy = b[0] - a[0], b[1] - a[1]
        return a, (name, dx, dy, th), (min(0, dx) - m, min(0, dy) - m, max(0, dx) + m + 1, max(0, dy) + m + 1)
    if p.get("bottomLeftOrigin", False):
        raise ValueError("display list: putText with bottomLeftOrigin is not supported")
    face, scale = int(p["fontFace"]), float(p["fontScale"])
    (w, h), base = cv2.getTextSize(str(p["text"]), face, scale, th)
    m += int(np.ceil(12 * scale))
    return _pt(p["org"]), ("putText", str(p["text"]), face, scale, th), (-m, -h - m, w + m, base + m)


def _rasterise(name: str, p: dict, ox: int, oy: int, cw: int, ch: int) -> np.ndarray:
    """The call's coverage on a zeroed (ch, cw) canvas whose top-left is frame pixel (ox, oy): the same cv2 call with
    every point moved by (-ox, -oy)."""
    import cv2

    canvas = np.zeros((ch, cw), np.uint8)
    q = {k: v for k, v in p.items() if k != "img"}
    for k in ("center", "pt1", "pt2", "org"):
        if k in q:
            x, y = _pt(q[k])
            q[k] = (x - ox, y - oy)
    q["color"] = 255
    getattr(cv2, name)(canvas, **q)
    return canvas


class DisplayListBuilder:
    """Turns one frame's drawing into records + coverage sprites, in the reference's order (runner.py:114-162)."""

    CACHE_SIZE = 8192

    def __init__(self, frame_hw: tuple[int, int], projected_court: ProjectedCourt):
        self.H, self.W = frame_hw
        self.court = projected_court
        self.lut = projected_court.blend_lut()
        self._sprites: dict = {}  # shape key + canvas relative to the anchor -> coverage (or None: covers nothing)

    def call_record(self, name: str, p: dict):
        """(x0, y0, w, h, sprite, colour) of one cv2 call, or None when it covers no pixel of the frame."""
        (ax, ay), key, (bx0, by0, bx1, by1) = _geometry(name, p)
        x0, y0 = max(0, ax + bx0), max(0, ay + by0)
        x1, y1 = min(self.W, ax + bx1), min(self.H, ay + by1)
        if x0 >= x1 or y0 >= y1:
            return None
        skey = (key, x0 - ax, y0 - ay, x1 - ax, y1 - ay)
        sprite = self._sprites.get(skey, False)
        if sprite is False:
            if len(self._sprites) >= self.CACHE_SIZE:  # per-frame text and skeleton lines: keep memory bounded
                self._sprites.clear()
            sprite = _rasterise(name, p, x0, y0, x1 - x0, y1 - y0)
            sprite = sprite if sprite.any() else None
            self._sprites[skey] = sprite
        if sprite is None:
            return None
        return x0, y0, x1 - x0, y1 - y0, sprite, _colour_bgr(p["color"])

    def frame_records(self, frame_index: int, trackers: dict, data_analytics: Optional[DataAnalytics],
                      is_fixed_keypoints: bool, results: Optional[dict] = None) -> list:
        """Records of one frame: [(x0, y0, w, h, sprite or None (BLEND), colour)].  Updates the court's homography
        and records the players' positions in `data_analytics` as the reference's pass does.  `results` maps each
        tracker's name to the per-frame predictions to draw (default: the tracker's own `results`)."""
        import cv2

        from .trackers.ball_tracker import Ball
        from .trackers.keypoints_tracker import Keypoints
        from .trackers.players_tracker import Players

        calls = [("putText", {"text": f"Frame: {frame_index + 1}", "org": FRAME_TEXT_ORG,
                              "fontFace": cv2.FONT_HERSHEY_SIMPLEX, "fontScale": 1, "color": FRAME_TEXT_COLOUR,
                              "thickness": 1})]
        players = ball = keypoints = None
        for name, t in trackers.items():
            pred = (t.results if results is None else results[name])[frame_index]
            calls += record_draw_calls(pred.draw, **t.draw_kwargs())
            obj = t.object()
            if obj is Players:
                players = pred
            elif obj is Ball:
                ball = pred
            elif obj is Keypoints:
                keypoints = pred
        recs = [r for r in (self.call_record(n, p) for n, p in calls) if r is not None]
        (bx0, by0), (bx1, by1) = self.court.background_position.top_left, self.court.background_position.bottom_right
        x0, y0, x1, y1 = max(0, bx0), max(0, by0), min(self.W, bx1 + 1), min(self.H, by1 + 1)  # filled: inclusive
        if x0 < x1 and y0 < y1:
            recs.append((x0, y0, x1 - x0, y1 - y0, None, 0))
        calls = []
        for centre, colour in self.court.court_keypoints.draw_points():
            calls.append(("circle", {"center": centre, "radius": 5, "color": colour, "thickness": -1}))
        for a, b in self.court.court_keypoints.lines():
            calls.append(("line", {"pt1": a, "pt2": b, "color": (0, 0, 0), "thickness": 2}))
        H = self.court.update_homography(keypoints, is_fixed_keypoints)
        if H is not None and players:
            for p in self.court.project_players(players, H, data_analytics):
                calls += record_draw_calls(p.draw_projection)
        if H is not None and ball:
            calls += record_draw_calls(self.court.project_ball(ball, H).draw_projection)
        recs += [r for r in (self.call_record(n, p) for n, p in calls) if r is not None]
        if data_analytics is not None:
            data_analytics.step(1)
        return recs


def pack_display_list(frames_records: list[list]) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Per-frame record lists -> (records (n,) OVERLAY_REC, offsets int32 (B+1), atlas u8) for pb_render_overlay.
    Each distinct sprite is stored once per batch."""
    offsets = np.zeros(len(frames_records) + 1, np.int32)
    rows, chunks, where, size = [], [], {}, 0
    for f, recs in enumerate(frames_records):
        for x0, y0, w, h, sprite, colour in recs:
            if sprite is None:
                rows.append((x0, y0, w, h, 0, 0, 0, L.OVERLAY_BLEND))
                continue
            off = where.get(id(sprite))
            if off is None:
                off = where[id(sprite)] = size
                chunks.append(sprite.reshape(-1))
                size += sprite.size
            rows.append((x0, y0, w, h, off, sprite.shape[1], colour, L.OVERLAY_STAMP))
        offsets[f + 1] = len(rows)
    recs = np.array(rows, dtype=L.OVERLAY_REC) if rows else np.zeros(0, dtype=L.OVERLAY_REC)
    atlas = np.concatenate(chunks) if chunks else np.zeros(0, np.uint8)
    return recs, offsets, atlas


def composite_numpy(frames: np.ndarray, recs: np.ndarray, offsets: np.ndarray, atlas: np.ndarray,
                    lut: np.ndarray) -> np.ndarray:
    """What pb_render_overlay does, in NumPy, in place on uint8 (B,H,W,3) BGR frames."""
    B, H, W, _ = frames.shape
    for f in range(B):
        for r in recs[offsets[f]:offsets[f + 1]]:
            x0, y0, w, h = int(r["x0"]), int(r["y0"]), int(r["w"]), int(r["h"])
            cx0, cy0, cx1, cy1 = max(x0, 0), max(y0, 0), min(x0 + w, W), min(y0 + h, H)
            if cx0 >= cx1 or cy0 >= cy1:
                continue
            region = frames[f, cy0:cy1, cx0:cx1]
            if int(r["op"]) == L.OVERLAY_BLEND:
                region[:] = lut[region]
                continue
            pitch, off = int(r["pitch"]), int(r["atlas_offset"])
            rows = np.arange(cy0 - y0, cy1 - y0)[:, None] * pitch + np.arange(cx0 - x0, cx1 - x0)[None, :]
            cov = atlas[off + rows] != 0
            c = int(r["colour_bgr"])
            region[cov] = np.array([c & 255, (c >> 8) & 255, (c >> 16) & 255], np.uint8)
    return frames


def render_frame_cpu(frame_bgr: np.ndarray, frame_index: int, trackers: dict, projected_court: ProjectedCourt,
                     data_analytics: Optional[DataAnalytics] = None, is_fixed_keypoints: bool = False) -> np.ndarray:
    """The reference's per-frame loop body (runner.py:114-162) on the host, whole-frame cv2 calls: the yardstick the
    device path is compared with, and its CPU baseline."""
    import cv2

    from .trackers.ball_tracker import Ball
    from .trackers.keypoints_tracker import Keypoints
    from .trackers.players_tracker import Players

    rgb = cv2.cvtColor(frame_bgr, cv2.COLOR_BGR2RGB)
    cv2.putText(rgb, f"Frame: {frame_index + 1}", FRAME_TEXT_ORG, cv2.FONT_HERSHEY_SIMPLEX, 1, FRAME_TEXT_COLOUR, 1)
    players = ball = keypoints = None
    for t in trackers.values():
        pred = t.results[frame_index]
        rgb = pred.draw(rgb, **t.draw_kwargs())
        obj = t.object()
        if obj is Players:
            players = pred
        elif obj is Ball:
            ball = pred
        elif obj is Keypoints:
            keypoints = pred
    out, _ = projected_court.draw_projections_and_collect_data(rgb, keypoints, players, ball, data_analytics,
                                                              is_fixed_keypoints)
    if data_analytics is not None:
        data_analytics.step(1)
    return cv2.cvtColor(out, cv2.COLOR_RGB2BGR)


class OverlayRenderer:
    """Batches of frames through pb_render_overlay: uploaded, composited and copied back into pinned buffers.  Two
    upload slots: while batch i is on the device, batch i+1 is read and its display list built on the host.  Timings
    (seconds) accumulate in `times`: decode, build, upload, overlay, download (the last three from CUDA events)."""

    def __init__(self, frame_hw: tuple[int, int], batch_size: int, lut: np.ndarray, out_slots: int = 2):
        import torch

        H, W = frame_hw
        self.hw, self.B = (H, W), batch_size
        self.dev = torch.device("cuda")
        shape = (batch_size, H, W, 3)
        self.frames = [torch.empty(shape, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.pin_out = [torch.empty(shape, dtype=torch.uint8).pin_memory() for _ in range(out_slots)]
        self.meta_host = [torch.empty(0, dtype=torch.uint8) for _ in range(2)]  # pinned: offsets | records | atlas
        self.meta_dev = [torch.empty(0, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        self.lut = torch.from_numpy(np.ascontiguousarray(lut, dtype=np.uint8)).to(self.dev)
        self.uploaded = [None, None]  # per slot: event after the last upload into it
        self.times = {"decode": 0.0, "build": 0.0, "upload": 0.0, "overlay": 0.0, "download": 0.0}
        self._events = []

    def _stage_meta(self, slot: int, recs, offsets, atlas):
        import torch

        o_rec = (offsets.nbytes + 15) // 16 * 16
        o_atl = o_rec + recs.nbytes
        need = o_atl + atlas.nbytes
        if self.meta_host[slot].numel() < need:
            cap = max(need, 2 * self.meta_host[slot].numel(), 1 << 20)
            self.meta_host[slot] = torch.empty(cap, dtype=torch.uint8).pin_memory()
            self.meta_dev[slot] = torch.empty(cap, dtype=torch.uint8, device=self.dev)
        buf = self.meta_host[slot].numpy()
        buf[:offsets.nbytes] = offsets.view(np.uint8)
        buf[o_rec:o_atl] = recs.view(np.uint8)
        buf[o_atl:need] = atlas
        return need, o_rec, o_atl

    def run(self, batches: Iterable, build: Callable[[int, int], list], free_slots: Optional[queue.Queue] = None):
        """batches: iterable of lists of uint8 (n,H,W,3) BGR tensors (pinned host or device) that add up to at most
        batch_size frames (`trackers.frames.chunks`).  A batch's pieces are uploaded asynchronously: they must stay
        untouched until the batch after next is taken.  build(first_frame, n) -> the batch's per-frame record lists.
        Yields (frames, out_slot): frames an (n,H,W,3) numpy view of pinned out-slot memory.  Without `free_slots` the
        out slots are used in turn and a yielded batch may be overwritten as soon as the generator is advanced; with
        it, a slot is taken from the queue before each download and the consumer puts it back when done with the
        frames."""
        import torch

        lib = L.lib()
        main = torch.cuda.current_stream()
        it = iter(batches)
        pending, i, first = None, 0, 0
        while True:
            t0 = timeit.default_timer()
            s = i % 2
            if self.uploaded[s] is not None:  # the batch before last and this slot's metadata must have been read
                self.uploaded[s].synchronize()
            pieces = next(it, None)
            if pieces is None:
                break
            n = sum(p.shape[0] for p in pieces)
            t1 = timeit.default_timer()
            recs, offsets, atlas = pack_display_list(build(first, n))
            nbytes, o_rec, o_atl = self._stage_meta(s, recs, offsets, atlas)
            t2 = timeit.default_timer()
            self.times["decode"] += t1 - t0
            self.times["build"] += t2 - t1
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            fr = self.frames[s][:n]
            ev[0].record(main)
            at = 0
            for p in pieces:
                fr[at:at + p.shape[0]].copy_(p, non_blocking=True)
                at += p.shape[0]
            meta = self.meta_dev[s]
            meta[:nbytes].copy_(self.meta_host[s][:nbytes], non_blocking=True)
            ev[1].record(main)
            self.uploaded[s] = ev[1]
            base = meta.data_ptr()
            L.check(lib.pb_render_overlay(fr.data_ptr(), n, self.hw[0], self.hw[1], base + o_rec if len(recs) else None,
                                          base, base + o_atl if atlas.size else None, self.lut.data_ptr(),
                                          main.cuda_stream))
            ev[2].record(main)
            o = free_slots.get() if free_slots is not None else i % len(self.pin_out)
            self.pin_out[o][:n].copy_(fr, non_blocking=True)
            ev[3].record(main)
            self._events.append(ev)
            if pending is not None:
                yield self._finish(*pending)
            pending = (ev[3], o, n)
            first += n
            i += 1
        if pending is not None:
            yield self._finish(*pending)
        for ev in self._events:
            self.times["upload"] += ev[0].elapsed_time(ev[1]) / 1e3
            self.times["overlay"] += ev[1].elapsed_time(ev[2]) / 1e3
            self.times["download"] += ev[2].elapsed_time(ev[3]) / 1e3
        self._events = []

    def _finish(self, done, o: int, n: int):
        done.synchronize()
        return self.pin_out[o][:n].numpy(), o


class VideoWriterThread:
    """cv2.VideoWriter on a thread of its own, so that encoding overlaps the next batch.  Batches come in as
    (frames, out_slot); the slot goes back to `free_slots` (anything with `put(slot)`) once its frames are written.
    After `finish()` the thread writes what is queued, releases the writer and sets `closed`."""

    def __init__(self, path: str, fps: float, resolution_wh: tuple[int, int], free_slots: queue.Queue):
        import cv2

        self.writer = cv2.VideoWriter(str(path), cv2.VideoWriter_fourcc(*"mp4v"), float(fps), tuple(resolution_wh))
        if not self.writer.isOpened():
            raise RuntimeError(f"cv2.VideoWriter could not open {path}")
        self.free = free_slots
        self.work: queue.Queue = queue.Queue()
        self.error = None
        self.seconds = 0.0
        self.closed = threading.Event()
        self._finished = False
        self.thread = threading.Thread(target=self._loop, daemon=True)
        self.thread.start()

    def _loop(self):
        while True:
            item = self.work.get()
            if item is None:
                break
            frames, slot = item
            t0 = timeit.default_timer()
            if self.error is None:
                try:
                    for f in frames:
                        self.writer.write(f)
                except Exception as e:  # reported by close(); keep returning slots so the producer never blocks
                    self.error = e
            self.seconds += timeit.default_timer() - t0
            self.free.put(slot)
        try:
            self.writer.release()
        except Exception as e:
            self.error = self.error or e
        self.closed.set()

    def put(self, frames, slot: int):
        self.work.put((frames, slot))

    def finish(self):
        """No more frames: the writer is released once the queued ones are written, without waiting here."""
        if not self._finished:
            self._finished = True
            self.work.put(None)

    def close(self):
        self.finish()
        self.thread.join()
        if self.error is not None:
            raise self.error


# ---- a list of clips through one render pass ---------------------------------------------------------------------
MAX_OPEN_WRITERS = 4  # encoders of consecutive clips that may run at once


@dataclass(frozen=True)
class ClipPart:
    """Rows [lo, hi) of a batch: frames first.. of `clip`, for that clip's writer.  `open`: the writer is opened here
    (the clip's first frame), after the writer of clip `wait` has closed when `wait` is not None.  `close`: the
    clip's last frame, the writer is finished after this part."""
    clip: int
    lo: int
    hi: int
    first: int
    open: bool
    wait: Optional[int]
    close: bool


@dataclass(frozen=True)
class ClipRenderBatch:
    """One render batch of the concatenated clips: (clip, frame in clip) per row, and one part per clip with frames
    in it.  The batch's out slot is free again once every part has been written."""
    rows: list
    parts: list


def plan_clip_render(lengths: list[int], batch_size: int, max_open: int = MAX_OPEN_WRITERS) -> list[ClipRenderBatch]:
    """Batches of `batch_size` frames over the clips played back to back (the last one partial).  Clips of 0 frames
    have no rows and no writer.  A writer opens only after the one opened `max_open` opens before it has closed, so at
    most `max_open` are open at once."""
    if batch_size < 1 or max_open < 1:
        raise ValueError("batch_size and max_open must be >= 1")
    batches, rows, parts, opened = [], [], [], []
    for c, T in enumerate(lengths):
        f = 0
        while f < T:
            take = min(T - f, batch_size - len(rows))
            wait = None
            if f == 0:
                wait = opened[-max_open] if len(opened) >= max_open else None
                opened.append(c)
            parts.append(ClipPart(c, len(rows), len(rows) + take, f, f == 0, wait, f + take == T))
            rows += [(c, f + j) for j in range(take)]
            f += take
            if len(rows) == batch_size:
                batches.append(ClipRenderBatch(rows, parts))
                rows, parts = [], []
    if rows:
        batches.append(ClipRenderBatch(rows, parts))
    return batches


class _SlotRelease:
    """Puts an out slot back on `free` after the last of the parts its batch was split into is written."""

    def __init__(self, free: queue.Queue):
        self.free, self.left, self.lock = free, {}, threading.Lock()

    def expect(self, slot: int, parts: int):
        with self.lock:
            self.left[slot] = parts

    def put(self, slot: int):
        with self.lock:
            self.left[slot] -= 1
            done = self.left[slot] == 0
        if done:
            self.free.put(slot)


def write_clip_batches(plan: list[ClipRenderBatch], batches: Iterable, open_writer: Callable,
                       free_slots: queue.Queue) -> float:
    """Writes the rendered batches ((frames, out slot) pairs, in `plan` order) to one writer per clip.
    open_writer(clip, release) -> a started `VideoWriterThread` that hands slots to `release`.  Each clip's writer is
    finished after its last part, so it drains while later clips render.  Batches that end before the plan does (a
    source that ran short) leave the open writers with the frames they got.  Every writer is closed before this
    returns; the first error is raised after that.  Returns the writers' encode seconds."""
    release = _SlotRelease(free_slots)
    writers: dict = {}
    error = None
    n = 0
    try:
        for frames, slot in batches:
            if n == len(plan) or len(frames) > len(plan[n].rows):
                raise ValueError(f"render batch {n} has {len(frames)} frames, more than the plan")
            parts = [p for p in plan[n].parts if p.lo < len(frames)]
            release.expect(slot, len(parts))
            for p in parts:
                if p.open:
                    if p.wait is not None:
                        writers[p.wait].closed.wait()
                    writers[p.clip] = open_writer(p.clip, release)
                writers[p.clip].put(frames[p.lo:p.hi], slot)
                if p.close:
                    writers[p.clip].finish()
            n += 1
    finally:
        for w in writers.values():
            try:
                w.close()
            except Exception as e:
                error = error or e
    if error is not None:
        raise error
    return sum(w.seconds for w in writers.values())
