"""TrackNet (ball heat-map U-Net) on the wgmma conv kernels + the fused ball pipeline.

Replaces `self.tracknet` of the reference BallTracker (/root/reference/trackers/ball_tracker/ball_tracker.py:260-266,
called at :445-446) and, through `BallPipeline`, the surrounding CPU stages:
  iterable.py:167-199 (PIL resize + window assembly), ball_tracker.py:449-509,523 (temporal ensemble),
  predict.py:7-39,149-221 (threshold + findContours + bbox).
Network definition being replaced: /root/reference/trackers/ball_tracker/models.py:45-74.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .. import _lib as L
from . import ops, resample

H_NET, W_NET = 288, 512

# (block name, n convs, cin, cout) in execution order — models.py:48-54
_BLOCKS = [
    ("down_block_1", 2, 27, 64), ("down_block_2", 2, 64, 128), ("down_block_3", 3, 128, 256),
    ("bottleneck", 3, 256, 512), ("up_block_1", 3, 768, 256), ("up_block_2", 2, 384, 128),
    ("up_block_3", 2, 192, 64),
]


class TrackNetEngine:
    """nn.Module-like: __call__(x (B,27,288,512) f32 cuda) -> (B,8,288,512) f32, .to(), .eval(), .load_state_dict()."""

    def __init__(self, state_dict: dict | None = None, max_batch: int = 8, device: str = "cuda",
                 height: int = H_NET, width: int = W_NET):
        if not torch.cuda.is_available():
            raise L.PbError("TrackNetEngine needs a CUDA device (no CPU fallback)")
        L.lib()
        assert height % 8 == 0 and width % 8 == 0
        self.device = torch.device(device)
        self.B, self.H, self.W = max_batch, height, width
        self._w = {}
        self.prog = None
        self._alloc()
        if state_dict is not None:
            self.load_state_dict(state_dict)

    # -- nn.Module-ish surface the reference touches -------------------------------------------------------
    def to(self, device):
        return self

    def eval(self):
        return self

    def load_state_dict(self, sd: dict):
        """Fold BN (eps=1e-5, torch default; models.py:9) and pack to the kernel layout, then (re)build the program."""
        self._w.clear()
        for name, n, cin, cout in _BLOCKS:
            for i in range(1, n + 1):
                p = f"{name}.conv_{i}"
                ci = cin if i == 1 else cout
                w, b = ops.fold_bn(sd[f"{p}.conv.weight"].float(), sd[f"{p}.bn.weight"].float(),
                                   sd[f"{p}.bn.bias"].float(), sd[f"{p}.bn.running_mean"].float(),
                                   sd[f"{p}.bn.running_var"].float(), 1e-5)
                self._w[p] = ops.pack_conv_weight(w, b, ops.pad16(ci) if ci != 27 else 32, cout, self.device)
        # predictor 1x1 (64 -> 8) + sigmoid.  Default: a 1x1 tensor-core conv (fp16 weights, N = 16) writing the fp32
        # NCHW planes -- HBM-bound.  PADEL_B200_TRACKNET_HEAD=pointwise selects the
        # CUDA-core kernel with fp32 weights instead (308 us: ~800 instructions per 32 pixels, issue-bound).  The
        # fused-epilogue variant of the conv kernel also exists but costs more (512 FMAs per pixel in the epilogue).
        self._head_w = sd["predictor.weight"].float().reshape(8, 64).contiguous().to(self.device)
        self._head_b = sd["predictor.bias"].float().contiguous().to(self.device)
        self._w["predictor"] = ops.pack_conv_weight(sd["predictor.weight"].float().reshape(8, 64, 1, 1),
                                                    sd["predictor.bias"].float(), 64, 16, self.device)
        self._build()
        return self

    # -- buffers + program -----------------------------------------------------------------------------------
    def _alloc(self):
        B, H, W, dev = self.B, self.H, self.W, self.device
        h = lambda hh, ww, c: torch.zeros((B, hh, ww, c), dtype=torch.float16, device=dev)
        self.x = h(H, W, 32)
        self.t1 = h(H, W, 64)
        self.cat3 = h(H, W, 192)  # [up(u2) 128 | x1 64]
        self.p1 = h(H // 2, W // 2, 64)
        self.t2 = h(H // 2, W // 2, 128)
        self.cat2 = h(H // 2, W // 2, 384)  # [up(u1) 256 | x2 128]
        self.p2 = h(H // 4, W // 4, 128)
        self.t3a, self.t3b = h(H // 4, W // 4, 256), h(H // 4, W // 4, 256)
        self.cat1 = h(H // 4, W // 4, 768)  # [up(bottleneck) 512 | x3 256]
        self.p3 = h(H // 8, W // 8, 256)
        self.ba, self.bb = h(H // 8, W // 8, 512), h(H // 8, W // 8, 512)
        self.u1a, self.u1b = h(H // 4, W // 4, 256), h(H // 4, W // 4, 256)
        self.u2a = h(H // 2, W // 2, 128)
        self.u3a, self.u3b = h(H, W, 64), h(H, W, 64)
        # 7 carried windows + B new ones (ball_tracker.py:427-436, :523)
        self.pred = torch.zeros((7 + B, 8, H, W), dtype=torch.float32, device=dev)

    def _build(self):
        # PADEL_B200_BALL_SMS=n: size this program's persistent grids for n SMs (and launch its kernels without
        # programmatic overlap, so a waiting successor never parks on the SMs left free) -- for running beside the YOLO
        # chains of the other trackers (FusedPass streams mode 2) instead of before / after them
        sms = int(os.environ.get("PADEL_B200_BALL_SMS", "0"))
        if sms > 0:
            L.lib().pb_set_plan_options(sms, 0)
        try:
            self._build_program()
        finally:
            L.lib().pb_set_plan_options(0, -1)

    def _build_program(self):
        P = ops.Program()
        W_ = self._w
        R, UP, SIG = L.ACT_RELU, L.OUT_F16_NHWC_UP2, L.ACT_SIGMOID

        def conv(x, coff, cin, name, out, ooff, mode=L.OUT_F16_NHWC, act=R, k=3, store=None, pool=None):
            w, b = W_[name]
            P.conv(ops.make_conv_desc(x, coff, cin, w, b, k, 1, act, out, ooff, mode, store,
                                      out2=None if pool is None else (pool, 0, L.OUT2_POOL2)),
                   cin_real=27 if name == "down_block_1.conv_1" else cin)

        # MaxPool2d of the three encoder blocks (models.py:60,62,64) is a second store of the producing conv
        # (PB_OUT2_POOL2); PADEL_B200_FUSE_OUT2=0 keeps the separate pool launches (A/B)
        fuse = os.environ.get("PADEL_B200_FUSE_OUT2", "1") != "0"

        conv(self.x, 0, 32, "down_block_1.conv_1", self.t1, 0)
        conv(self.t1, 0, 64, "down_block_1.conv_2", self.cat3, 128, pool=self.p1 if fuse else None)
        if not fuse:
            P.maxpool2(self.cat3, 128, 64, self.p1, 0)
        conv(self.p1, 0, 64, "down_block_2.conv_1", self.t2, 0)
        conv(self.t2, 0, 128, "down_block_2.conv_2", self.cat2, 256, pool=self.p2 if fuse else None)
        if not fuse:
            P.maxpool2(self.cat2, 256, 128, self.p2, 0)
        conv(self.p2, 0, 128, "down_block_3.conv_1", self.t3a, 0)
        conv(self.t3a, 0, 256, "down_block_3.conv_2", self.t3b, 0)
        conv(self.t3b, 0, 256, "down_block_3.conv_3", self.cat1, 512, pool=self.p3 if fuse else None)
        if not fuse:
            P.maxpool2(self.cat1, 512, 256, self.p3, 0)
        conv(self.p3, 0, 256, "bottleneck.conv_1", self.ba, 0)
        conv(self.ba, 0, 512, "bottleneck.conv_2", self.bb, 0)
        conv(self.bb, 0, 512, "bottleneck.conv_3", self.cat1, 0, UP)  # nearest x2 fused into the store
        conv(self.cat1, 0, 768, "up_block_1.conv_1", self.u1a, 0)
        conv(self.u1a, 0, 256, "up_block_1.conv_2", self.u1b, 0)
        conv(self.u1b, 0, 256, "up_block_1.conv_3", self.cat2, 0, UP)
        conv(self.cat2, 0, 384, "up_block_2.conv_1", self.u2a, 0)
        conv(self.u2a, 0, 128, "up_block_2.conv_2", self.cat3, 0, UP)
        conv(self.cat3, 0, 192, "up_block_3.conv_1", self.u3a, 0)
        self._pred_new = self.pred[7:]
        conv(self.u3a, 0, 64, "up_block_3.conv_2", self.u3b, 0)
        if os.environ.get("PADEL_B200_TRACKNET_HEAD", "tc") == "tc":
            conv(self.u3b, 0, 64, "predictor", self._pred_new, 0, L.OUT_F32_NCHW, SIG, k=1, store=8)
        else:
            P.pointwise_head(self.u3b, self._head_w, self._head_b, self._pred_new)
        self.prog = P

    # -- execution ---------------------------------------------------------------------------------------------
    def run_packed(self):
        """x (B,H,W,32 fp16, already packed) -> pred[7:7+B]."""
        if self.prog is None:
            raise L.PbError("TrackNetEngine: no weights loaded")
        self.prog.run()

    @torch.no_grad()
    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """Reference-compatible call (ball_tracker.py:445): NCHW fp32 in [0,1] -> (B,8,H,W) fp32 heat-maps."""
        nb = x.shape[0]
        if nb > self.B or tuple(x.shape[1:]) != (27, self.H, self.W):
            raise L.PbError(f"TrackNetEngine: expected (<= {self.B}, 27, {self.H}, {self.W}), got {tuple(x.shape)}")
        self.x[:nb, ..., :27] = x.to(self.device).permute(0, 2, 3, 1).to(torch.float16)
        self.run_packed()
        return self._pred_new[:nb].clone()


def window_desc(w0: int, nb: int, total_frames: int | None) -> np.ndarray:
    """Ensemble descriptors (window 0, window count, frame) of the frames a batch of windows [w0, w0+nb) of one video
    emits: frame w per window w, plus the 7 tail frames (ball_tracker.py:486-509) when the batch runs the video's last
    window.  total_frames=None: the video's end is not known yet (a stream), so the batch emits its windows' own
    frames only, with w0 + nb as their window count.  Any count above a frame selects the same rule for it (head
    below frame 7, else the weighted sum of windows n-7..n) as the true count, which is larger still."""
    tw = w0 + nb if total_frames is None else total_frames - 7
    nframes = nb + (7 if total_frames is not None and w0 + nb == tw else 0)
    desc = np.zeros((nframes, 3), dtype=np.int32)
    desc[:, 1] = tw
    desc[:, 2] = np.arange(w0, w0 + nframes)
    return desc


def tail_desc(total_frames: int) -> np.ndarray:
    """Descriptors of the 7 tail frames of a video of `total_frames` >= 8 frames, for a launch that runs no window:
    the stream's last window already ran while its end was unknown, and the 7-window carry still holds the windows
    these frames read (ball_tracker.py:486-509: frame T-8+i, i = 1..7, is the mean of the 8-i windows that hold it)."""
    tw = total_frames - 7
    desc = np.zeros((7, 3), dtype=np.int32)
    desc[:, 1] = tw
    desc[:, 2] = np.arange(tw, total_frames)
    return desc


def ready_batches(next_window: int, frames_end: int, B: int, total_frames: int | None) -> list[tuple[int, int]]:
    """(first window, window count) of the batches of up to B windows that run every window computable now: window w
    needs frames w..w+7, so the windows [next_window, frames_end - 7) are ready (frames_end: one past the last frame
    that arrived), capped at the video's last window when `total_frames` is known."""
    end = frames_end - 7 if total_frames is None else min(frames_end, total_frames) - 7
    return [(w, min(B, end - w)) for w in range(next_window, end, B)]


class BallPipeline:
    """Frames (BGR u8) -> per-frame ball bbox, entirely on device: PIL-exact resize, window packing, TrackNet,
    temporal ensemble + threshold, connected components.  Mirrors BallTracker.predict_frames' TrackNet stage
    (ball_tracker.py:373-523) including its head/tail ensemble rules (SURVEY App. C).  One video: its background is
    slot 0 of a one-slot median pool, and its windows are numbered from 0 as the one clip of the batch tables.

    The video's length may be unknown while frames arrive (a stream): the launches then emit only frames whose
    ensemble does not depend on where the video ends, and `stream_end` emits the 7 tail frames once it is known."""

    def __init__(self, engine: TrackNetEngine, frame_hw: tuple[int, int], median_rgb: np.ndarray | torch.Tensor):
        self._init_buffers(engine, frame_hw, ring=engine.B + 8, pool=1, max_frames=engine.B + 7)
        self.stage = torch.zeros((self.B + 7, self.Hs, self.Ws, 3), dtype=torch.uint8, device=self.dev)
        self.ens = None
        self._median_src = None
        self.set_median(median_rgb)
        self.reset()

    def _init_buffers(self, engine: TrackNetEngine, frame_hw, ring: int, pool: int, max_frames: int,
                      table_ints: int | None = None):
        """Pillow bicubic tables (frame size -> network size), the ring of `ring` resized frames, a pool of `pool`
        backgrounds, and the per-batch buffers for up to `max_frames` emitted frames and `table_ints` table entries
        (default: the row tables of `_launch_batch`)."""
        self.eng = engine
        self.dev = engine.device
        self.Hs, self.Ws = frame_hw
        B, H, W = engine.B, engine.H, engine.W
        self.B, self.ring, self.pool, self.max_frames = B, ring, pool, max_frames
        bh, kh, self.ksh = resample.pil_bicubic_tables(self.Ws, W)
        bv, kv, self.ksv = resample.pil_bicubic_tables(self.Hs, H)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
        self.bh, self.kh, self.bv, self.kv = up(bh), up(kh), up(bv), up(kv)
        # resized RGB frames and backgrounds as normalised fp16 4-channel pixels (what the window-packing kernel gathers)
        self.small = torch.zeros((ring, H, W, 4), dtype=torch.float16, device=self.dev)
        self.medians = torch.zeros((pool, H, W, 4), dtype=torch.float16, device=self.dev)
        self.tmp = torch.zeros((B + 7, self.Hs, W, 3), dtype=torch.uint8, device=self.dev)
        self.mask = torch.zeros((max_frames, H, W), dtype=torch.uint8, device=self.dev)
        self.scratch = torch.zeros((B + 7, 5, H * W), dtype=torch.int32, device=self.dev)  # boxes run B+7 at a time
        self.bbox = torch.zeros((max_frames, 4), dtype=torch.int32, device=self.dev)
        # a batch's tables on the device: row ring slots (B), row median slots (B), frame descriptors (max_frames, 3)
        self._tables = torch.zeros(2 * B + 3 * max_frames if table_ints is None else table_ints, dtype=torch.int32,
                                   device=self.dev)
        # per launch slot, pinned: the staged tables and the downloaded boxes (see _launch_batch for the slot rule)
        self._stage = [torch.zeros(self._tables.shape, dtype=torch.int32).pin_memory() for _ in range(4)]
        self._host_ring = [torch.zeros((max_frames, 4), dtype=torch.int32).pin_memory() for _ in range(4)]
        self._pending = [None] * 4
        self._turn = 0

    def set_median(self, median_rgb):
        """(Re)apply the background: full-res RGB -> uint8 -> PIL resize (iterable.py:76-81), on device with the same
        kernel as the frames.  A no-op when called again with the very same array object/contents."""
        med = torch.as_tensor(median_rgb)
        if tuple(med.shape[:2]) != (self.Hs, self.Ws):
            raise L.PbError("median must have the frame resolution")
        med = med.to(torch.uint8)
        if self._median_src is not None and self._median_src.shape == med.shape and \
                torch.equal(self._median_src, med.cpu()):
            return
        self._median_src = med.cpu().clone()
        dev_med = med.to(self.dev).contiguous().view(1, self.Hs, self.Ws, 3)
        self._resize(dev_med, 1, self.medians[:1], swap_rb=0)

    def load_median(self, slot: int, median_rgb) -> None:
        """(Hs,Ws,3) uint8 RGB background (host or device) -> resized into pool slot `slot`, as `set_median` does."""
        med = torch.as_tensor(median_rgb).to(self.dev, torch.uint8).contiguous().view(1, self.Hs, self.Ws, 3)
        self._resize(med, 1, self.medians[slot:slot + 1], swap_rb=0)

    def reset(self, base: int = 0):
        """base = absolute index of the first frame that will be pushed (= first window computed); > 0 for shards
        that start mid-video (the 7 windows before the shard are recomputed, SURVEY §8e)."""
        self.base = base
        self.n_frames_in = 0  # frames received
        self.n_windows = 0  # windows processed
        self.tail_emitted = False  # the launch of the video's last window emitted its 7 tail frames
        self.eng.pred.zero_()

    def _resize(self, src, n, dst_f16, swap_rb):
        """Pillow-exact resize of n frames; the vertical pass writes value/255 as fp16 4-channel pixels into dst_f16."""
        L.check(L.lib().pb_pil_resize_u8(src.data_ptr(), n, self.Hs, self.Ws, self.tmp.data_ptr(), None,
                                         self.eng.H, self.eng.W, self.bh.data_ptr(), self.kh.data_ptr(), self.ksh,
                                         self.bv.data_ptr(), self.kv.data_ptr(), self.ksv, swap_rb, dst_f16.data_ptr(),
                                         2, L.stream_ptr()))

    def push_frames(self, frames_bgr: torch.Tensor):
        """frames: (n,Hs,Ws,3) u8 BGR, host (pinned or not) or device; n <= B+7. Resized into the ring."""
        n = frames_bgr.shape[0]
        if n == 0:
            return
        if frames_bgr.device.type != "cuda":
            self.stage[:n].copy_(frames_bgr, non_blocking=True)
            frames_bgr = self.stage[:n]
        if self.n_frames_in + n > self.n_windows + self.ring:
            raise L.PbError("BallPipeline: frame ring overflow (process windows before pushing more frames)")
        frames_bgr = frames_bgr.contiguous()
        start = self.n_frames_in % self.ring
        first = min(n, self.ring - start)  # resize straight into the ring (two runs when it wraps)
        self._resize(frames_bgr[:first], first, self.small[start:start + first], swap_rb=1)
        if first < n:
            self._resize(frames_bgr[first:], n - first, self.small[: n - first], swap_rb=1)
        self.n_frames_in += n

    def windows_ready(self) -> int:
        return max(0, self.n_frames_in - 7) - self.n_windows

    def run_windows(self, nb: int, total_frames: int | None, want_ens: bool = False):
        """Process the next nb windows (nb <= B). Returns (first_frame, host int32 (nframes,4) bboxes) for the frames
        emitted: absolute frames [first_frame, first_frame+nframes)."""
        return self.run_windows_async(nb, total_frames, want_ens)()

    def run_windows_async(self, nb: int, total_frames: int | None, want_ens: bool = False):
        """Enqueue the device work for the next nb windows; returns a callable that waits and yields
        (first_frame, bboxes).  One call in flight.  total_frames=None: the video's length is not known yet
        (`window_desc`)."""
        assert 0 < nb <= self.B and nb <= self.windows_ready()
        w0 = self.base + self.n_windows  # absolute window index
        if total_frames is not None and w0 + nb > total_frames - 7:
            raise L.PbError("BallPipeline: more windows than total_frames allows")
        desc = window_desc(w0, nb, total_frames)  # the video is one clip whose window 0 is window 0
        fin = self._launch_batch(w0, w0, (self.n_windows + np.arange(nb)) % self.ring, np.zeros(nb), desc, want_ens)
        self.n_windows += nb
        self.tail_emitted = len(desc) > nb
        return fin

    def run_ready_async(self, total_frames: int | None) -> list:
        """Enqueue every window that has become computable (`ready_batches`), in batches of up to B, with at most one
        launch in flight (each launch is waited for before the next is enqueued).  Returns the launches' finish
        callables in order."""
        fins = []
        for _, nb in ready_batches(self.base + self.n_windows, self.base + self.n_frames_in, self.B, total_frames):
            if fins:
                res = fins[-1]()
                fins[-1] = lambda res=res: res
            fins.append(self.run_windows_async(nb, total_frames))
        return fins

    def stream_end(self, total_frames: int) -> list:
        """The video ends at frame `total_frames`, the last frame pushed.  Enqueues the windows not run yet, whose last
        batch emits the 7 tail frames, or, when the last window already ran while the end was unknown, a launch of no
        window that emits the tail from the 7 windows carried in the heat-map buffer.  Returns the launches' finish
        callables in order, as `run_ready_async` does."""
        if self.base + self.n_frames_in != total_frames:
            raise L.PbError(f"BallPipeline: stream_end({total_frames}) after {self.base + self.n_frames_in} frames")
        fins = self.run_ready_async(total_frames)
        if total_frames >= 8 and not self.tail_emitted:
            tw = total_frames - 7
            fins.append(self._launch_batch(tw, tw, np.zeros(0), np.zeros(0), tail_desc(total_frames)))
            self.tail_emitted = True
        return fins

    def _launch_batch(self, key, first_window: int, row_slot, row_median, desc, want_ens: bool = False):
        """Enqueue one batch of nb = len(row_slot) windows: pack, TrackNet, ensemble + threshold, boxes, download.
        Row b is global window first_window + b; it gathers the ring slots (row_slot[b] + f) % ring, f = 0..7, and
        median pool slot row_median[b].  desc: per emitted frame, (global index of its clip's window 0, the clip's
        window count, the frame's index in its clip).  Returns a callable that waits and yields (key, host int32
        (nframes, 4) boxes)."""
        eng = self.eng
        nb = len(row_slot)
        desc = np.asarray(desc, dtype=np.int32).reshape(-1, 3)
        nframes = desc.shape[0]
        # pred holds the 7 windows carried from the batch before and this batch's: [first_window - 7, first_window + nb)
        lo = desc[:, 0] + np.maximum(desc[:, 2] - 7, 0)
        hi = desc[:, 0] + np.minimum(desc[:, 2], desc[:, 1] - 1)
        bad = np.flatnonzero((lo < first_window - 7) | (hi >= first_window + nb))
        if bad.size:
            i = bad[0]
            raise L.PbError(f"ensemble: frame {desc[i, 2]} needs windows [{lo[i]},{hi[i]}], the buffer holds "
                            f"[{first_window - 7},{first_window + nb})")
        slot = self._claim_slot()
        stage = self._stage[slot]
        n = 2 * nb + 3 * nframes
        t = stage.numpy()
        t[:nb], t[nb:2 * nb], t[2 * nb:n] = row_slot, row_median, desc.reshape(-1)
        self._tables[:n].copy_(stage[:n], non_blocking=True)
        rows = self._tables.data_ptr()
        if nb:  # nb = 0: a stream's tail, ensembled from the carried windows alone
            L.check(L.lib().pb_tracknet_pack_windows_rows(self.small.data_ptr(), self.ring, rows,
                                                          self.medians.data_ptr(), rows + 4 * nb, nb, eng.H, eng.W,
                                                          eng.x.data_ptr(), L.stream_ptr()))
            eng.run_packed()
        ens_ptr = None
        if want_ens:
            self.ens = torch.empty((nframes, eng.H, eng.W), dtype=torch.float32, device=self.dev)
            ens_ptr = self.ens.data_ptr()
        L.check(L.lib().pb_tracknet_ensemble_rows(eng.pred.data_ptr(), first_window - 7, rows + 8 * nb, nframes, eng.H,
                                                  eng.W, 0.5, self.mask.data_ptr(), ens_ptr, L.stream_ptr()))
        self._boxes(nframes)
        # carry the last 7 windows for the next batch (ball_tracker.py:523), which may start another clip
        if nb:
            carry = eng.pred[nb:nb + 7].clone()
            eng.pred[:7].copy_(carry)
        return self._download(slot, key, nframes)

    def _claim_slot(self) -> int:
        """The next launch slot.  The slot's staged tables and host boxes are rewritten only once its previous launch
        has completed.  That launch was waited for at the end of the launch before this one, unless that launch raised
        midway."""
        slot = self._turn
        self._turn = (slot + 1) % len(self._pending)
        if self._pending[slot] is not None:
            self._pending[slot]()
        return slot

    def _boxes(self, nframes: int) -> None:
        """Boxes of the first `nframes` masks."""
        step = self.scratch.shape[0]
        for f in range(0, nframes, step):  # the scratch holds B+7 frames: several launches for the short-clip case
            m = min(step, nframes - f)
            L.check(L.lib().pb_ccl_bbox(self.mask[f:].data_ptr(), m, self.eng.H, self.eng.W, self.scratch.data_ptr(),
                                        self.bbox[f:].data_ptr(), L.stream_ptr()))

    def _download(self, slot: int, key, nframes: int):
        """Enqueue the download of the first `nframes` boxes into launch slot `slot`; returns the launch's finish."""
        host = self._host_ring[slot]
        host[:nframes].copy_(self.bbox[:nframes], non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        state = {"result": None}

        def finish():
            if state["result"] is None:
                done.synchronize()
                state["result"] = (key, host[:nframes].numpy().copy())
                self._pending[slot] = None
            return state["result"]

        self._pending[slot] = finish
        # the caller may enqueue more batches before collecting this one: the next slot's launch (three launches back),
        # if still uncollected, is waited for now, after this batch is enqueued, so the next launch can reuse its slot
        if self._pending[self._turn] is not None:
            self._pending[self._turn]()
        return finish


class ClipBallPipeline(BallPipeline):
    """BallPipeline over a list of clips in one stream: a device batch may hold the windows of several clips.  The
    host plan (`clip_plan.plan_clip_batches`) says where each frame goes in the ring, when each clip's background is
    loaded into the median pool and which windows every batch runs; each row of a batch gathers from its own ring slot
    and median, and each emitted frame is ensembled over its own clip's windows only.  Per clip the boxes are
    bit-identical to BallPipeline run on that clip alone."""

    def __init__(self, engine: TrackNetEngine, frame_hw: tuple[int, int], ring: int | None = None,
                 pool: int | None = None):
        from .clip_plan import default_pool, default_ring

        ring = default_ring(engine.B) if ring is None else ring
        # a window emits its own frame, plus the 7 tail frames when it ends its clip
        self._init_buffers(engine, frame_hw, ring, default_pool(ring) if pool is None else pool, 8 * engine.B)

    def begin(self, plan) -> None:
        """Start the stream of `plan` (a ClipPlan with this ring and pool)."""
        if plan.ring != self.ring or plan.pool != self.pool or plan.batch > self.B or plan.chunk > self.B:
            raise L.PbError("ClipBallPipeline: the plan was made for another ring, pool or batch size")
        self.eng.pred.zero_()

    def push_at(self, frames_bgr: torch.Tensor, slot: int) -> None:
        """Resize (n,Hs,Ws,3) uint8 BGR device frames into ring slots slot..slot+n-1."""
        n = frames_bgr.shape[0]
        if n and (slot + n > self.ring or n > self.B + 7):
            raise L.PbError("ClipBallPipeline: push outside the ring")
        if n:
            self._resize(frames_bgr.contiguous(), n, self.small[slot:slot + n], swap_rb=1)

    def run_batch_async(self, batch):
        """Enqueue one planned batch; returns a callable that waits and yields (frames [(clip, frame)], host int32
        (nframes, 4) boxes)."""
        return self._launch_batch(batch.frames, batch.first_window, batch.row_slot, batch.row_median, batch.desc)


class StreamsBallPipeline(BallPipeline):
    """BallPipeline over several interleaved live streams in one pass: a device batch may hold windows of any open
    streams, each at its own position.  The host planner (`stream_plan.StreamPlanner`) places each pushed frame in a
    shared pool of resized frames, gives each stream a lane (7 rows of a heat-map carry pool and a median pool slot)
    and names, per launch, each row's 8 frame slots and each emitted frame's 8 heat-map rows.  Per stream the boxes
    are bit-identical to BallPipeline run on that stream alone."""

    def __init__(self, engine: TrackNetEngine, frame_hw: tuple[int, int], max_open: int):
        from .stream_plan import StreamPlanner

        plan = StreamPlanner(engine.B, max_open)
        B, F = engine.B, plan.max_frames
        # tables of a launch: row slots (B, 8), row medians (B), frame refs + rule (F, 9), carry copies (B, 2)
        self._init_buffers(engine, frame_hw, ring=plan.n_slots, pool=max_open, max_frames=F,
                           table_ints=9 * B + 9 * F + 2 * B)
        self.max_open = max_open
        self.carry = torch.zeros((plan.carry_rows, 8, engine.H, engine.W), dtype=torch.float32, device=self.dev)
        self.begin()

    def begin(self) -> None:
        """Start a pass: no stream open, every slot free."""
        from .stream_plan import StreamPlanner

        self.plan = StreamPlanner(self.B, self.max_open)

    def step_async(self, frames_bgr: torch.Tensor, segments: list, ends: list, median_of):
        """One upload chunk: (n,Hs,Ws,3) uint8 BGR device frames made of `segments` = [(key, frames)] runs of one
        stream each, after which the streams `ends` end.  Loads the backgrounds of the streams that start
        (`median_of(key)`: (Hs,Ws,3) uint8 RGB), resizes the frames into their pool slots and enqueues the step's
        launches.  Returns (the planned `StreamStep`, the launches' finish callables, each yielding ([(key, frame)],
        host int32 (nframes, 4) boxes))."""
        st = self.plan.step(segments, ends)
        for key, lane in st.medians:
            self.load_median(lane, median_of(key))
        for off, n, slot in st.pushes:
            self._resize(frames_bgr[off:off + n].contiguous(), n, self.small[slot:slot + n], swap_rb=1)
        return st, [self._launch_table(launch) for launch in st.launches]

    def _launch_table(self, launch):
        """Enqueue one planned launch (`stream_plan.StreamLaunch`): pack, TrackNet, ensemble + threshold, carry
        update, boxes, download."""
        eng = self.eng
        nb, nf, nc = len(launch.rows), len(launch.frames), len(launch.carry)
        slot = self._claim_slot()
        t = self._stage[slot].numpy()
        a, b = 8 * nb, 9 * nb
        c = b + 9 * nf
        d = c + 2 * nc
        if nb:
            t[:a] = np.asarray(launch.row_slots).reshape(-1)
            t[a:b] = launch.row_median
        if nf:
            t[b:c] = np.concatenate([np.asarray(launch.refs), np.asarray(launch.rule)[:, None]], 1).reshape(-1)
        if nc:
            t[c:d] = np.asarray(launch.carry).reshape(-1)
        self._tables[:d].copy_(self._stage[slot][:d], non_blocking=True)
        p = self._tables.data_ptr()
        fresh = eng.pred[7:]
        if nb:  # nb = 0: tails ensembled from the carry pool alone
            L.check(L.lib().pb_tracknet_pack_windows_slots(self.small.data_ptr(), p, self.medians.data_ptr(), p + 4 * a,
                                                           nb, eng.H, eng.W, eng.x.data_ptr(), L.stream_ptr()))
            eng.run_packed()
        L.check(L.lib().pb_tracknet_ensemble_table(self.carry.data_ptr(), self.carry.shape[0], fresh.data_ptr(),
                                                   p + 4 * b, nf, eng.H, eng.W, 0.5, self.mask.data_ptr(), None,
                                                   L.stream_ptr()))
        # after the ensemble: window w's carry row is window w-7's, which frame w reads
        L.check(L.lib().pb_tracknet_carry_rows(self.carry.data_ptr(), fresh.data_ptr(), p + 4 * c, nc, eng.H, eng.W,
                                               L.stream_ptr()))
        self._boxes(nf)
        return self._download(slot, launch.frames, nf)


def bbox_to_xyv(bbox: np.ndarray, img_scaler: tuple[float, float]):
    """predict.py:203-217 on host with Python float arithmetic (bit-identical to the reference's int() truncations)."""
    xs, ys, vs = [], [], []
    for x, y, w, h in bbox.tolist():
        cx, cy = int(x + w / 2), int(y + h / 2)
        cx, cy = int(cx * img_scaler[0]), int(cy * img_scaler[1])
        xs.append(cx), ys.append(cy), vs.append(0 if (cx == 0 and cy == 0) else 1)
    return xs, ys, vs
