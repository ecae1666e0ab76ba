"""The frame-source format, read in one place.

A frame source is a callable `src(lo, hi)` that yields frames lo..hi-1 of a video, either as HWC uint8 BGR numpy
frames (video decode) or as ready uint8 (n,H,W,3) batches: host tensors (pinned or not) or device tensors.  `read`
turns either into (n,H,W,3) tensors (`tensors` does so for any iterable, such as a stream of unknown length),
`chunks` packs those into upload batches, and `head` splits off the first frames (the ball tracker's background
median).
"""
from __future__ import annotations

import itertools
from typing import Callable, Iterable, Iterator, Optional

import numpy as np
import torch


def read(src: Callable, lo: int, hi: int, hw: Optional[tuple[int, int]] = None, exact: bool = False,
         clip: int = 0) -> Iterator[torch.Tensor]:
    """Frames lo..hi-1 of `src` as uint8 (n,H,W,3) tensors, n >= 1: batches pass through as they are (host, pinned or
    device), an HWC array is wrapped without a copy and gets a leading axis.  The last piece is trimmed to hi - lo
    frames.  Every piece must have the frame size `hw` (default: that of the first piece), else ValueError.  A source
    that ends early raises ValueError with `exact` ("clip {clip} yielded N frames, T announced"), and simply ends
    without: video frame counts over-report (see `BallTracker.inpaint_xyv`)."""
    want, seen = hi - lo, 0
    if want <= 0:
        return
    for t in tensors(src(lo, hi), hw, f"clip {clip}"):
        t = t[:want - seen]
        seen += t.shape[0]
        if t.shape[0]:
            yield t
        if seen == want:
            return
    if exact:
        raise ValueError(f"clip {clip} yielded {seen} frames, {want} announced")


def tensors(items: Iterable, hw: Optional[tuple[int, int]] = None, what: str = "the stream"
            ) -> Iterator[torch.Tensor]:
    """HWC uint8 BGR frames or (n,H,W,3) batches (host or device) as (n,H,W,3) tensors, one per item, pulled one at a
    time: an HWC array is wrapped without a copy and gets a leading axis.  Every item must have the frame size `hw`
    (default: that of the first item), else ValueError naming `what`."""
    for item in items:
        t = item if isinstance(item, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(item))
        if t.dim() == 3:
            t = t.unsqueeze(0)
        if hw is None:
            hw = tuple(t.shape[1:3])
        if tuple(t.shape[1:3]) != tuple(hw):
            raise ValueError(f"{what} has {tuple(t.shape[1:3])} frames, not {tuple(hw)}: all frames of one call "
                             "must have the same frame size")
        yield t


def _pinned(shape: tuple) -> torch.Tensor:
    return torch.empty(shape, dtype=torch.uint8).pin_memory()


def chunks(pieces: Iterable[torch.Tensor], B: int, alloc: Callable[[tuple], torch.Tensor] = _pinned
           ) -> Iterator[list[torch.Tensor]]:
    """Lists of consecutive (n,H,W,3) pieces that add up to B frames (the last list may be short), in order.  Pinned
    and device pieces pass through as slices; host frames that are not pinned are gathered into three (B,H,W,3)
    buffers from `alloc(shape)`, allocated on first need and refilled in turn: a chunk's buffer is refilled three
    chunks later, which a consumer with one chunk of look-ahead (`FusedPass.run`, `OverlayRenderer.run`) has uploaded
    by then.  A piece that is None closes the chunk being filled: it is yielded at once, short or even empty."""
    bufs, out, n, k, run0 = [], [], 0, 0, None  # run0: where the gathered run of the current chunk starts
    for t in pieces:
        if t is None:
            if run0 is not None:
                out.append(bufs[k % 3][run0:n])
            yield out
            out, n, k, run0 = [], 0, k + 1, None
            continue
        while t.shape[0]:
            take = min(B - n, t.shape[0])
            part, t = t[:take], t[take:]
            if part.device.type == "cuda" or part.is_pinned():
                if run0 is not None:
                    out.append(bufs[k % 3][run0:n])
                    run0 = None
                out.append(part)
            else:
                if not bufs:
                    bufs = [alloc((B,) + tuple(part.shape[1:])) for _ in range(3)]
                bufs[k % 3][n:n + take].copy_(part)
                run0 = n if run0 is None else run0
            n += take
            if n == B:
                if run0 is not None:
                    out.append(bufs[k % 3][run0:n])
                yield out
                out, n, k, run0 = [], 0, k + 1, None
    if n:
        if run0 is not None:
            out.append(bufs[k % 3][run0:n])
        yield out


def head(pieces: Iterable[torch.Tensor], m: int) -> tuple[list[torch.Tensor], Iterator[torch.Tensor]]:
    """(the pieces holding the first m frames, an iterator over the rest): a piece that straddles frame m is split, so
    the head holds exactly m frames (fewer if the pieces run out) and chaining the two gives the pieces' frames."""
    it = iter(pieces)
    out, n = [], 0
    while n < m:
        t = next(it, None)
        if t is None:
            break
        take = min(m - n, t.shape[0])
        out.append(t[:take])
        n += take
        if take < t.shape[0]:
            return out, itertools.chain([t[take:]], it)
    return out, it
