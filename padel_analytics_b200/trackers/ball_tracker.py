"""BallTracker on the CUDA engine — API of reference trackers/ball_tracker/ball_tracker.py (Ball :139-206,
BallTracker :208-711).  The TrackNet stage (:373-523) runs fully on device through engine.BallPipeline.

Documented deviations from reference quirks (SURVEY App. E):
  q6  without an InpaintNet the reference dies with KeyError 'Frame' (:675-680); here the Ball list is built from the
      TrackNet x/y/visibility lists directly.
  q2  when `median` is None the reference buffers the first `median_max_sample_num` frames, converts them BGR->RGB
      twice and restarts the sliding window at the buffer boundary; here the median is computed from the same frames
      but every frame is converted once and the window never restarts.
  InpaintNet stage (:525-673): supported — the network runs as one fused CUDA kernel (engine/inpaint_engine.py), the
      surrounding bookkeeping (inpaint mask :100-136, sequence building dataset.py:387-429,493-503, blend, COOR_TH
      thresholds, coordinate ensemble, predict.py:91-147) is restated on the host in `_inpaint_stage`.
"""
from __future__ import annotations

import itertools
import math
from pathlib import Path
from typing import Iterable, Optional, Type

import numpy as np
import torch

from ..engine.inpaint_engine import InpaintNetEngine
from ..engine.tracknet_engine import BallPipeline, ClipBallPipeline, StreamsBallPipeline, TrackNetEngine, bbox_to_xyv
from .tracker import NoPredictSample, Object, Tracker


class Ball(Object):
    def __init__(self, frame: int, xy: tuple[float, float], visibility: int,
                 projection: Optional[tuple[int, int]] = None):
        super().__init__()
        self.frame = frame
        self.xy = xy
        self.visibility = visibility
        self.projection = projection

    @classmethod
    def from_json(cls, x: dict):
        return cls(**x)

    def serialize(self) -> dict:
        return {"frame": self.frame, "xy": self.xy, "visibility": self.visibility, "projection": self.projection}

    def asint(self):
        return tuple(int(v) for v in self.xy)

    def draw(self, frame: np.ndarray) -> np.ndarray:
        import cv2

        cv2.circle(frame, self.asint(), 6, (0, 255, 0), -1)
        return frame

    def draw_projection(self, frame: np.ndarray) -> np.ndarray:
        import cv2

        cv2.circle(frame, self.projection, 6, (255, 255, 0), -1)
        return frame


def median_background(frames_bgr, device="cuda") -> np.ndarray:
    """np.median(frames_rgb, 0).astype('uint8') (iterable.py:58-81) on the device: the frames (a list of HWC uint8 BGR
    frames or (n,H,W,3) uint8 pieces, numpy or torch, host or device) are copied piece by piece into one stack in HBM
    and `pb_median_u8` selects the per-byte median (even counts: mean of the two middle values, truncated like the
    reference's float64 -> uint8 cast), writing RGB order.  Returns the (H,W,3) uint8 RGB median on the host."""
    return median_background_device(frames_bgr, device).cpu().numpy()


def median_background_device(frames_bgr, device="cuda") -> torch.Tensor:
    """`median_background` without the download: the (H,W,3) uint8 RGB median stays on the device, computed on the
    current stream."""
    from .. import _lib as L

    pieces = [p if isinstance(p, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(p)) for p in frames_bgr]
    pieces = [p.unsqueeze(0) if p.dim() == 3 else p for p in pieces]
    if any(p.dtype != torch.uint8 or p.dim() != 4 or p.shape[1:] != pieces[0].shape[1:] or p.shape[-1] != 3
           for p in pieces):
        raise L.PbError("median_background: frames must be uint8 (T,H,W,3)")
    T, H, W, _ = sum(p.shape[0] for p in pieces), *pieces[0].shape[1:]
    stack = torch.empty((T, H, W, 3), dtype=torch.uint8, device=device)
    at = 0
    for p in pieces:
        stack[at:at + p.shape[0]].copy_(p)
        at += p.shape[0]
    out = torch.empty((H, W, 3), dtype=torch.uint8, device=stack.device)
    L.check(L.lib().pb_median_u8(stack.data_ptr(), T, H * W * 3, out.data_ptr(), 1, L.stream_ptr()))
    return out


class BallTracker(Tracker):
    stage = "ball"
    EVAL_MODE: str = "weight"
    TRAJECTORY_LENGTH: int = 8
    HEIGHT: int = 288
    WIDTH: int = 512
    SIGMA: float = 2.5
    IMG_FORMAT = "png"

    def __init__(self, tracking_model_path, inpainting_model_path, batch_size: int,
                 median_max_sample_num: int = 1800, median: Optional[np.ndarray] = None,
                 load_path: Optional[str | Path] = None, save_path: Optional[str | Path] = None):
        super().__init__(load_path=load_path, save_path=save_path)
        self.DELTA_T: float = 1 / math.sqrt(self.HEIGHT ** 2 + self.WIDTH ** 2)
        self.COOR_TH = self.DELTA_T * 50
        ckpt = tracking_model_path if isinstance(tracking_model_path, dict) else \
            torch.load(tracking_model_path, map_location="cpu", weights_only=False)
        self.tracknet_seq_len = ckpt["param_dict"]["seq_len"]
        assert self.tracknet_seq_len == self.TRAJECTORY_LENGTH  # ball_tracker.py:256
        self.bg_mode = ckpt["param_dict"]["bg_mode"]
        if self.bg_mode != "concat":
            raise NotImplementedError("only bg_mode='concat' (what predict_frames hard-codes, :403) is supported")
        self.tracknet = TrackNetEngine(ckpt["model"], max_batch=batch_size, height=self.HEIGHT, width=self.WIDTH)
        if inpainting_model_path:
            ick = inpainting_model_path if isinstance(inpainting_model_path, dict) else \
                torch.load(inpainting_model_path, map_location="cpu", weights_only=False)
            self.inpaintnet_seq_len = ick["param_dict"]["seq_len"]  # ball_tracker.py:270
            self.inpaintnet = InpaintNetEngine(ick["model"])
        else:
            self.inpaintnet = None
        self.batch_size = batch_size
        self.median_max_sample_num = median_max_sample_num
        self.median = median
        self._pipe = None
        self._clip_pipe = None
        self._streams_pipe = None

    def video_info_post_init(self, video_info) -> "BallTracker":
        self.video_info = video_info
        return self

    def object(self) -> Type[Object]:
        return Ball

    def draw_kwargs(self) -> dict:
        return {}

    def __str__(self) -> str:
        return "ball_tracker"

    def restart(self) -> None:
        self.results.restart()

    def to(self, device: str) -> None:
        self.tracknet.to(device)

    def predict_sample(self, sample, **kwargs):
        raise NoPredictSample()

    def _pipeline(self, frame_hw, median_rgb) -> BallPipeline:
        """The pipeline (device rings, resample tables) is cached per frame size; the background median is re-applied
        on every call, as the reference does per predict_frames call (iterable.py:58-81)."""
        if self._pipe is None or (self._pipe.Hs, self._pipe.Ws) != tuple(frame_hw):
            self._pipe = BallPipeline(self.tracknet, frame_hw, median_rgb)
        else:
            self._pipe.set_median(median_rgb)
        return self._pipe

    def track_xyv(self, frame_generator: Iterable[np.ndarray], total_frames: int, first_frame: int = 0,
                  emit_range: Optional[tuple[int, int]] = None, median: Optional[np.ndarray] = None):
        """TrackNet stage on device.  Frames from the generator are absolute frames first_frame, first_frame+1, ...
        Returns dict frame_index -> (x, y, vis) for the frames emitted (restricted to emit_range if given)."""
        it = iter(frame_generator)
        B = self.batch_size
        pending: list[np.ndarray] = []
        median = self.median if median is None else median
        if median is None:  # iterable.py:58-73 (a sharded caller passes the whole-video median instead)
            for f in it:
                pending.append(f)
                if len(pending) == self.median_max_sample_num:
                    break
            if not pending:
                return {}
            median = median_background(pending)
        stream = itertools.chain(pending, it)
        first = next(stream, None)
        if first is None:
            return {}
        self.stream_begin(tuple(first.shape[-3:-1]), total_frames, first_frame, emit_range, median)  # :379-384
        out: dict[int, tuple[int, int, int]] = {}

        def push(frames):
            out.update(self.stream_push_async(frames if isinstance(frames, torch.Tensor) else
                                              torch.from_numpy(np.stack(frames)))())

        if isinstance(first, torch.Tensor) and first.dim() == 4:
            # batched frame source: items are uint8 (n,H,W,3) tensors (pinned host or device), n <= batch_size
            push(first)
            for batch in stream:
                push(batch)
            return out
        chunk = [first]
        for f in stream:
            if len(chunk) == B:
                push(chunk)
                chunk = []
            chunk.append(f)
        if chunk:
            push(chunk)
        return out

    # ---- streaming interface used by the fused single-pass runner (one batch at a time, device work asynchronous) ----
    def stream_begin(self, frame_hw, total_frames: Optional[int] = None, first_frame: int = 0, emit_range=None,
                     median=None):
        """Start a stream of frames first_frame, first_frame+1, ... through the device pipeline.  total_frames=None:
        the stream's length is unknown until `stream_end_async`; until then each push emits only the frames whose
        result cannot depend on where the stream ends (frame f once frame f+7 has arrived).  median: (H,W,3) uint8
        RGB background, host or device (defaults to `self.median`)."""
        median = self.median if median is None else median
        if median is None:
            raise ValueError("stream_begin needs a background median (pass median= to BallTracker or here)")
        pipe = self._pipeline(tuple(frame_hw), median)
        pipe.reset(base=first_frame)
        self._stream = dict(total=total_frames, emit=emit_range,
                            scaler=(self.video_info.width / self.WIDTH, self.video_info.height / self.HEIGHT))
        return pipe

    def clips_begin(self, frame_hw, plan, median_of):
        """Streaming over a list of clips (`TrackingRunner.run_clips`): `plan` is the ClipPlan of the stream
        (`clip_plan.plan_clip_batches` with this tracker's ring and pool, see `clip_pipeline`); `median_of(clip)`
        returns (device (H,W,3) uint8 RGB background, CUDA event after which it is ready, or None).  Each
        `stream_push_async` then takes the next upload chunk and its finish yields [(clip, frame, (x, y, vis))]."""
        pipe = self.clip_pipeline(frame_hw)
        pipe.begin(plan)
        self._stream = dict(clips=plan, step=0, median_of=median_of,
                            scaler=(frame_hw[1] / self.WIDTH, frame_hw[0] / self.HEIGHT))
        return pipe

    def clip_pipeline(self, frame_hw) -> ClipBallPipeline:
        if self._clip_pipe is None or (self._clip_pipe.Hs, self._clip_pipe.Ws) != tuple(frame_hw):
            self._clip_pipe = ClipBallPipeline(self.tracknet, tuple(frame_hw))
        return self._clip_pipe

    def streams_begin(self, frame_hw, max_open: int, steps, median_of):
        """Streaming over several interleaved live streams (`TrackingRunner.stream_many`): `steps` is a deque to which
        the caller appends, before each `stream_push_async`, the chunk's ([(key, frames)] runs, [keys ending]);
        `median_of(key)` returns the stream's (H,W,3) uint8 RGB background.  Each push's finish then yields
        [(key, frame, (x, y, vis))].  Ball coordinates are scaled by `video_info`, shared by every stream."""
        pipe = self._streams_pipe
        if pipe is None or (pipe.Hs, pipe.Ws) != tuple(frame_hw) or pipe.max_open != max_open:
            pipe = self._streams_pipe = StreamsBallPipeline(self.tracknet, tuple(frame_hw), max_open)
        pipe.begin()
        self._stream = dict(streams=steps, median_of=median_of,
                            scaler=(self.video_info.width / self.WIDTH, self.video_info.height / self.HEIGHT))
        return pipe

    def _streams_push_async(self, frames: torch.Tensor):
        s = self._stream
        segments, ends = s["streams"].popleft()
        _, fins = self._streams_pipe.step_async(frames, segments, ends, s["median_of"])
        fin = self._xyv_finish(fins, lambda frames: frames)  # a launch yields its [(key, frame)]
        return lambda: [(k, f, v) for (k, f), v in fin()]

    def _xyv_finish(self, fins, frames_of):
        """A callable that waits for the launches `fins` in turn and returns [(frame, (x, y, vis))] for their boxes;
        frames_of(key) gives the frames of the launch that yields (key, boxes)."""
        scaler = self._stream["scaler"]

        def finish():
            out = []
            for fin in fins:
                key, bbox = fin()
                out += zip(frames_of(key), zip(*bbox_to_xyv(bbox, scaler)))
            return out

        return finish

    def _clips_push_async(self, frames: torch.Tensor):
        pipe, s = self._clip_pipe, self._stream
        ops = s["clips"].steps[s["step"]]
        s["step"] += 1
        fins = []
        for op in ops:
            if op[0] == "median":
                med, ready = s["median_of"](op[1])
                if ready is not None:
                    torch.cuda.current_stream().wait_event(ready)
                pipe.load_median(op[2], med)
            elif op[0] == "push":
                _, off, n, slot = op
                pipe.push_at(frames[off:off + n], slot)
            else:
                fins.append(pipe.run_batch_async(op[1]))
        fin = self._xyv_finish(fins, lambda frames: frames)  # a batch yields its [(clip, frame)]
        return lambda: [(c, f, v) for (c, f), v in fin()]

    def stream_push_async(self, frames: torch.Tensor):
        """frames: uint8 (n,H,W,3) BGR tensor (device or pinned host), n <= batch_size.  Enqueues resize + every
        window that became computable; returns a callable that waits and yields {frame: (x, y, vis)}."""
        if "clips" in self._stream:
            return self._clips_push_async(frames)
        if "streams" in self._stream:
            return self._streams_push_async(frames)
        pipe, s = self._pipe, self._stream
        pipe.push_frames(frames)
        fin = self._xyv_finish(pipe.run_ready_async(s["total"]), itertools.count)  # a launch yields its first frame
        emit = s["emit"]
        return lambda: {n: v for n, v in fin() if emit is None or emit[0] <= n < emit[1]}

    def stream_end_async(self, total_frames: int):
        """End a stream begun without a total at frame `total_frames` (every frame has been pushed): enqueues the
        last windows and the 7 tail frames (`BallPipeline.stream_end`); returns a callable that waits and yields
        {frame: (x, y, vis)} for the frames not emitted yet."""
        self._stream["total"] = total_frames
        fin = self._xyv_finish(self._pipe.stream_end(total_frames), itertools.count)
        return lambda: dict(fin())

    # ---- InpaintNet stage (ball_tracker.py:525-673) -------------------------------------------------------------
    @staticmethod
    def _generate_inpaint_mask(y, vis, th_h: float):
        """ball_tracker.py:100-136."""
        y, vis = np.array(y), np.array(vis)
        mask = np.zeros_like(y)
        i = j = 0
        while j < len(vis):
            while i < len(vis) - 1 and vis[i] == 1:
                i += 1
            j = i
            while j < len(vis) - 1 and vis[j] == 0:
                j += 1
            if j == i:
                break
            elif i == 0 and y[j] > th_h:
                mask[:j] = 1
            elif (i > 1 and y[i - 1] > th_h) and (j < len(vis) and y[j] > th_h):
                mask[i:j] = 1
            i = j
        return mask

    def _inpaint_stage(self, xs, ys, vs):
        """TrackNet per-frame (x, y, vis) lists (every frame 0..T-1 present) -> inpainted lists, as the reference does
        between :525 and :673.  Sequences (stride 1, length L) -> InpaintNet on device -> blend with the mask -> COOR_TH
        threshold -> temporal ensemble over the L windows covering each frame -> threshold -> pixel coordinates."""
        Lq = self.inpaintnet_seq_len
        T = len(xs)
        W_img, H_img = self.video_info.width, self.video_info.height
        mask = self._generate_inpaint_mask(ys, vs, th_h=H_img * 0.05)
        S = T - Lq + 1
        if S <= 0:
            return {}
        sel = np.arange(S)[:, None] + np.arange(Lq)[None, :]
        coor = np.stack([np.asarray(xs, np.float32)[sel], np.asarray(ys, np.float32)[sel]], -1)  # dataset.py:390-420
        coor[:, :, 0] = coor[:, :, 0] / W_img  # dataset.py:499-500
        coor[:, :, 1] = coor[:, :, 1] / H_img
        m = np.asarray(mask, np.float32)[sel][..., None]
        c_t, m_t = torch.from_numpy(coor), torch.from_numpy(m)
        out = self.inpaintnet(c_t, m_t).cpu()
        out = out * m_t + c_t * (1 - m_t)  # :577
        th = (out[:, :, 0] < self.COOR_TH) & (out[:, :, 1] < self.COOR_TH)
        out[th] = 0.0
        # temporal ensemble on coordinates (:584-652): frame n <- windows n-L+1..n, slot L-1-k of window n-L+1+k
        w = torch.ones(Lq)
        for i in range(math.ceil(Lq / 2)):
            w[i] = i + 1
            w[Lq - i - 1] = i + 1
        w = w / w.sum()
        zero = torch.zeros(2)
        ens = torch.zeros((T, 2))
        for n in range(T):
            terms = torch.stack([out[n - (Lq - 1) + k, Lq - 1 - k] if 0 <= n - (Lq - 1) + k < S else zero
                                 for k in range(Lq)])
            if n < S and n >= Lq - 1:
                ens[n] = (terms * w[:, None]).sum(0)
            else:
                ens[n] = terms.sum(0) / ((n + 1) if n < S else (Lq - (n - (S - 1))))
        th = (ens[:, 0] < self.COOR_TH) & (ens[:, 1] < self.COOR_TH)
        ens[th] = 0.0
        scaler = (W_img / self.WIDTH, H_img / self.HEIGHT)
        res = {}
        ens_np = ens.numpy()
        for n in range(T):  # predict.py:125-129 (numpy float32 scalar arithmetic, int() truncation)
            cx = int(ens_np[n][0] * self.WIDTH * scaler[0])
            cy = int(ens_np[n][1] * self.HEIGHT * scaler[1])
            res[n] = (cx, cy, 0 if (cx == 0 and cy == 0) else 1)
        return res

    def inpaint_xyv(self, xyv: dict, total_frames: int) -> dict:
        """Apply the InpaintNet stage to a {frame: (x, y, vis)} trajectory (no-op without an inpainting model); used by
        predict_frames and by the sharded runner on rank 0.  The reference feeds whatever TrackNet produced (frames
        0..T'-1) to the inpainting stage; if fewer frames than announced arrived (CAP_PROP_FRAME_COUNT often
        over-reports: the tail flush never fires and the last 7 frames are missing) the stage runs over the contiguous
        range that is present, with a warning, instead of being skipped."""
        if getattr(self, "inpaintnet", None) is None or not xyv:
            return xyv
        order = sorted(xyv)
        lo, hi = order[0], order[-1]
        if len(order) != hi - lo + 1:
            print(f"{self}: TrackNet results are not a contiguous frame range ({len(order)} frames in [{lo}, {hi}]); "
                  f"InpaintNet stage skipped")
            return xyv
        if len(order) != total_frames:
            print(f"{self}: {len(order)} of {total_frames} announced frames have TrackNet results; "
                  f"inpainting frames {lo}..{hi}")
        res = self._inpaint_stage([xyv[n][0] for n in order], [xyv[n][1] for n in order], [xyv[n][2] for n in order])
        out = dict(xyv)
        out.update({lo + k: v for k, v in res.items()})
        return out

    def balls(self, xyv: dict, total_frames: int) -> list[Ball]:
        """A video's or clip's TrackNet trajectory {frame: (x, y, vis)} -> the InpaintNet stage (`inpaint_xyv`) -> one
        Ball per frame 0..total_frames-1 (ball_tracker.py:675-698: missing frames -> (0,0), visibility 0)."""
        xyv = self.inpaint_xyv(xyv, total_frames)
        return [Ball(frame=n, xy=(xyv[n][0], xyv[n][1]), visibility=xyv[n][2]) if n in xyv
                else Ball(frame=n, xy=(0.0, 0.0), visibility=0) for n in range(total_frames)]

    def predict_frames(self, frame_generator: Iterable[np.ndarray], total_frames: int, **kwargs) -> list[Ball]:
        return self.balls(self.track_xyv(frame_generator, total_frames), total_frames)
