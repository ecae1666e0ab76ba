"""The ball pipeline after TrackNet, decision for decision on the device's own heat-maps.

The fp16 TrackNet legitimately differs from the fp32 oracle, but everything after it is exact given its heat-maps: the
windows it read are a gather of fp16 pixels, the temporal ensemble is a fixed sequence of fp32 multiplies and adds
(`ensemble_reference_loop`, the reference's own loop), and the threshold and the component box are integer decisions
(cv2, as the reference).  So every frame is required to match, with no borderline exclusions.  InpaintNet is fp32 end
to end and is checked against a float64 reference with a derived bound (tests/ball_post_ref.py).
"""
import numpy as np
import pytest
import torch

import ball_post_ref as R
from fixtures import rally_frames
from oracle import inpaint as OI
from oracle import tracknet as OT
from oracle import weights as OW
from padel_analytics_b200 import _lib as L
from padel_analytics_b200 import synth
from padel_analytics_b200.engine.tracknet_engine import BallPipeline, TrackNetEngine, bbox_to_xyv
from padel_analytics_b200.trackers.runner import ball_shard_frames

pytestmark = pytest.mark.gpu
DEV = "cuda"
SRC_HW = (360, 640)  # the committed rally crops' size; the synthetic frames use it too
SMALL_HW = (144, 256)  # TrackNet size for the T x batch grid: the post-processing does not depend on the size


def _to16(rgb_u8: np.ndarray) -> torch.Tensor:
    return (torch.from_numpy(rgb_u8).float() * np.float32(1 / 255.0)).half()


def _frames(source: str, T: int) -> list:
    """T BGR frames: the three rally crops rolled a little further each frame (real content, fake motion), or synth."""
    if source == "rally":
        base = rally_frames()
        return [np.ascontiguousarray(np.roll(base[n % 3], (3 * n, 5 * n), (0, 1))) for n in range(T)]
    return [f.numpy() for f in synth.make_frames(T, SRC_HW[0], SRC_HW[1], start=11)]


@pytest.fixture(scope="module")
def tracknet_ckpt():
    return OW.make_tracknet()


_ENGINES = {}


def _engine(ck, B, hw):
    key = (B, hw)
    if key not in _ENGINES:
        _ENGINES[key] = TrackNetEngine(ck["model"], max_batch=B, height=hw[0], width=hw[1])
    return _ENGINES[key]


class Recorder:
    """Hooks a BallPipeline: after each TrackNet launch it snapshots the packed windows eng.x[:nb] and the new
    heat-maps eng.pred[7:7+nb] (optionally overwriting them with planted maps first), and it records each launch's
    first window w0, nb, and (with want_ens) the device ensemble.  Everything is copied on the stream, in order."""

    def __init__(self, pipe: BallPipeline, planted=None):
        self.pipe, self.eng = pipe, pipe.eng
        self.planted = planted  # (total_windows, 8, H, W) device tensor, absolute window index
        self.launches = []
        self._cur = None
        run_packed, run_async = self.eng.run_packed, pipe.run_windows_async

        def hooked_run_packed():
            run_packed()
            w0, nb = self._cur["w0"], self._cur["nb"]
            if self.planted is not None:
                self.eng.pred[7:7 + nb].copy_(self.planted[w0:w0 + nb])
            self._cur["x"] = self.eng.x[:nb].clone()
            self._cur["pred"] = self.eng.pred[7:7 + nb].clone()

        def hooked_run_async(nb, total_frames, want_ens=False):
            self._cur = dict(w0=pipe.base + pipe.n_windows, nb=nb)
            fin = run_async(nb, total_frames, want_ens)
            if want_ens:
                self._cur["ens"] = pipe.ens.clone()
            self.launches.append(self._cur)
            return fin

        self.eng.run_packed = hooked_run_packed
        pipe.run_windows_async = hooked_run_async

    def unhook(self):
        del self.eng.run_packed
        del self.pipe.run_windows_async


def drive(pipe: BallPipeline, frames, T: int, B: int, mode: str, want_ens: bool, base: int = 0, emit=None):
    """Run frames (absolute frames base, base+1, ...) through the pipeline the way BallTracker does:
    'frames'  -- host frames pushed one at a time, every computable window run synchronously (track_xyv's loop);
    'batches' -- device uint8 (n,H,W,3) tensors of B frames, launches asynchronous with one in flight
                 (stream_push_async).  Returns {frame: bbox (4,)}."""
    pipe.reset(base=base)
    out = {}

    def collect(res):
        f0, bbox = res
        for i in range(bbox.shape[0]):
            if emit is None or emit[0] <= f0 + i < emit[1]:
                out[f0 + i] = tuple(int(v) for v in bbox[i])

    def launch():
        fins = []
        while True:
            nb = min(B, pipe.windows_ready(), T - 7 - (pipe.base + pipe.n_windows))
            if nb <= 0:
                return fins
            if fins:
                fins[-1] = fins[-1]()
                fins[-1] = (lambda r: (lambda: r))(fins[-1])
            fins.append(pipe.run_windows_async(nb, T, want_ens))

    if mode == "frames":
        for f in frames:
            pipe.push_frames(torch.from_numpy(f[None]))
            for fin in launch():
                collect(fin())
    else:
        dev = torch.from_numpy(np.stack(frames)).to(DEV)
        prev = []
        for i in range(0, len(frames), B):
            pipe.push_frames(dev[i:i + B])
            for fin in prev:
                collect(fin())
            prev = launch()
        for fin in prev:
            collect(fin())
    return out


def _check_run(rec: Recorder, got: dict, T: int, B: int, frames, base: int, exp_small, med16, want_ens: bool,
               emit=None):
    """Every packed window == the fp16 gather; the snapshots through the reference loop == the device ensemble; every
    emitted frame's box == cv2 on the reference ensemble's mask.  Returns (frames, fg pixels, components, ties)."""
    launches = rec.launches
    w_first = launches[0]["w0"]
    assert w_first == base
    assert [l["w0"] for l in launches] == list(np.cumsum([base] + [l["nb"] for l in launches])[:-1])
    zeros = torch.zeros(exp_small[0].shape[:2] + (5,), dtype=torch.float16)
    for l in launches:
        x = l["x"].cpu()
        for b in range(l["nb"]):
            n = l["w0"] + b  # window n = frames n..n+7
            want = torch.cat([med16] + [exp_small[n + f - base] for f in range(8)] + [zeros], -1)
            assert torch.equal(x[b], want), f"window {n}: packed input differs from the frame gather"
    preds = torch.cat([l["pred"].cpu() for l in launches])
    # the reference loop from the first computed window: for a shard, the windows before `base` are not computed and
    # its first 7 frames are not emitted, so they are left out of the comparison
    if base == 0:
        ens_ref = OT.ensemble_reference_loop(preds, T, B)
        first_frame = 0
    else:
        full = torch.zeros((T - 7,) + preds.shape[1:])
        full[base:base + preds.shape[0]] = preds  # frames before base + 7 or past the shard's end are not compared
        ens_ref = OT.ensemble_reference_loop(full, T, B)
        first_frame = base + 7
    lo, hi = (first_frame, T) if emit is None else emit
    assert sorted(got) == list(range(lo, hi))
    if want_ens:
        dev_ens = {}
        for l in launches:
            for i in range(l["ens"].shape[0]):
                dev_ens[l["w0"] + i] = l["ens"][i]
        for n in range(lo, hi):
            assert torch.equal(dev_ens[n].cpu(), ens_ref[n]), \
                f"frame {n}: ensemble differs by {(dev_ens[n].cpu() - ens_ref[n]).abs().max().item():.3g}"
    frames_checked = fg = comps = ties = 0
    for n in range(lo, hi):
        m = (ens_ref[n] > 0.5).numpy().astype(np.uint8)
        exp = tuple(OT.heatmap_to_bbox(m * 255))
        assert got[n] == exp, f"frame {n}: box {got[n]} vs cv2 {exp}"
        xyv = bbox_to_xyv(np.array([got[n]]), (3.0, 3.0))
        assert tuple(v[0] for v in xyv) == OT.bbox_to_xy(exp, (3.0, 3.0))
        a, c, t = R.component_stats(m)
        frames_checked, fg, comps, ties = frames_checked + 1, fg + a, comps + c, ties + (t >= 2)
    return frames_checked, fg, comps, ties


def _expected_small(frames, pipe):
    """What the ring should hold for each frame: the Pillow resize of its RGB, /255 in fp16."""
    return [_to16(OT.resize_rgb(f[..., ::-1].copy(), pipe.eng.W, pipe.eng.H)) for f in frames]


# ---- a. the pipeline on TrackNet's own heat-maps ---------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 8, 16])
@pytest.mark.parametrize("T", [8, 9, 15, 16, 23, 40, 61])
def test_pipeline_decisions_on_device_heatmaps(tracknet_ckpt, T, B):
    source = "rally" if T % 2 else "synth"
    frames = _frames(source, T)
    eng = _engine(tracknet_ckpt, B, SMALL_HW)
    med = synth.make_median(*SRC_HW).numpy()
    pipe = BallPipeline(eng, SRC_HW, med)
    med16 = _to16(OT.resize_rgb(med, SMALL_HW[1], SMALL_HW[0]))
    exp_small = _expected_small(frames, pipe)
    stats = []
    for mode, want_ens in (("frames", True), ("batches", False)):
        rec = Recorder(pipe)
        got = drive(pipe, frames, T, B, mode, want_ens)
        rec.unhook()
        stats.append(_check_run(rec, got, T, B, frames, 0, exp_small, med16, want_ens))
    n, fg, comps, ties = stats[0]
    print(f"T={T} B={B} {source}: {n} frames, {fg} foreground pixels, {comps} components, {ties} tie frames")


@pytest.mark.parametrize("T,B,shards", [(40, 3, 3), (61, 8, 4)])
def test_pipeline_shards_match_unsharded(tracknet_ckpt, T, B, shards):
    frames = _frames("rally", T)
    eng = _engine(tracknet_ckpt, B, SMALL_HW)
    med = synth.make_median(*SRC_HW).numpy()
    pipe = BallPipeline(eng, SRC_HW, med)
    med16 = _to16(OT.resize_rgb(med, SMALL_HW[1], SMALL_HW[0]))
    exp_small = _expected_small(frames, pipe)
    full = drive(pipe, frames, T, B, "batches", False)
    merged = {}
    for r in range(shards):
        lo, hi = r * T // shards, (r + 1) * T // shards
        flo, fhi = ball_shard_frames(T, lo, hi)
        rec = Recorder(pipe)
        got = drive(pipe, frames[flo:fhi], T, B, "frames", True, base=flo, emit=(lo, hi))
        rec.unhook()
        if fhi - flo >= 8:
            _check_run(rec, got, T, B, frames, flo, exp_small[flo:], med16, True, emit=(lo, hi))
        merged.update(got)
    assert merged == full


# ---- b. planted heat-maps at the shipped size ------------------------------------------------------------------------
def _planted(T: int, H: int, W: int, seed: int) -> torch.Tensor:
    """(T-7, 8, H, W) window heat-maps: window w slot j is frame w+j's map plus per-window jitter.  Most pixels sit on a
    grid of values at and one or two fp32 ulps either side of 0.5 (so the ensemble lands on 0.5 exactly or next to it);
    two blobs move across the frame (crossing batch boundaries), and near the first and last 7 frames a ring of
    near-0.5 pixels outgrows the blobs only under the head / tail mean."""
    g = torch.Generator().manual_seed(seed)
    S = T - 7
    half = torch.tensor(0.5)
    grid = torch.stack([torch.nextafter(half, torch.tensor(d)) if d else half for d in (0.0, 1.0, -1.0)])
    grid = torch.cat([grid, torch.nextafter(grid[1:], torch.tensor([1.0, 0.0]))])  # 0.5, +-1 ulp, +-2 ulp
    base = grid[torch.randint(0, len(grid), (T, H, W), generator=g)]
    base *= (torch.rand((T, H, W), generator=g) > 0.3).float()  # 30% zeros: components stay bounded
    yy, xx = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing="ij")
    for n in range(T):
        for k, (vy, vx) in enumerate(((2.0, 9.0), (-3.0, -7.0))):
            cy, cx = (40 + 100 * k + vy * n) % H, (60 + 200 * k + vx * n) % W
            blob = torch.exp(-((yy - cy) ** 2 / 18 + (xx - cx) ** 2 / 40))
            base[n] = torch.maximum(base[n], blob)
        if n < 7 or n >= T - 7:
            r = ((yy - H / 2) ** 2 + (xx - W / 2) ** 2).sqrt()
            ring = ((r - 60).abs() < 1.5).float() * 0.5004
            base[n] = torch.maximum(base[n], ring)
    win = torch.empty((S, 8, H, W))
    for w in range(S):
        jitter = torch.nextafter(base[w:w + 8], torch.full((8, H, W), float(w % 2)))  # 1 ulp up or down per window
        win[w] = torch.where(torch.rand((8, H, W), generator=g) < 0.5, base[w:w + 8], jitter)
    return win


@pytest.mark.parametrize("T,B", [(23, 8), (16, 8), (8, 1), (24, 16)])
def test_pipeline_decisions_on_planted_heatmaps(tracknet_ckpt, T, B):
    H, W = R.H_NET, R.W_NET
    planted = _planted(T, H, W, seed=T * 31 + B)
    eng = _engine(tracknet_ckpt, B, (H, W))
    frames = _frames("synth", T)
    med = synth.make_median(*SRC_HW).numpy()
    pipe = BallPipeline(eng, SRC_HW, med)
    med16 = _to16(OT.resize_rgb(med, W, H))
    exp_small = _expected_small(frames, pipe)
    for mode, want_ens in (("frames", True), ("batches", False)):
        rec = Recorder(pipe, planted=planted.to(DEV))
        got = drive(pipe, frames, T, B, mode, want_ens)
        rec.unhook()
        n, fg, comps, ties = _check_run(rec, got, T, B, frames, 0, exp_small, med16, want_ens)
    # the ensemble kernel's grid is capped at num_sms * 32 CTAs of 256 threads
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 32 * 256
    most = max(l["nb"] + (7 if l["w0"] + l["nb"] == T - 7 else 0) for l in rec.launches)
    assert most * H * W > cap, "no launch wraps the ensemble's grid-stride loop"
    ens = OT.ensemble_reference_loop(planted, T, B)
    on_half = int((ens == 0.5).sum())
    near = int(((ens - 0.5).abs() <= 2 ** -23).sum())
    print(f"planted T={T} B={B}: {n} frames, {fg} foreground pixels, {comps} components, {ties} tie frames, "
          f"{on_half} ensembled pixels == 0.5, {near} within 1 ulp")
    assert on_half > 0 and near > on_half


# ---- c. pb_ccl_bbox in isolation --------------------------------------------------------------------------------------
def _ccl(masks: np.ndarray, scratch: torch.Tensor) -> np.ndarray:
    n, H, W = masks.shape
    md = torch.from_numpy(masks).to(DEV)
    bbox = torch.full((n, 4), -7, dtype=torch.int32, device=DEV)
    L.check(L.lib().pb_ccl_bbox(md.data_ptr(), n, H, W, scratch.data_ptr(), bbox.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    return bbox.cpu().numpy()


def test_ccl_adversarial_masks_garbage_scratch():
    H, W, n = R.H_NET, R.W_NET, 256 + 7  # B + 7 frames: the engine's largest launch (batch 256)
    names = sorted(R.GENERATORS)
    first = np.stack([R.make_mask(names[i % len(names)], seed=i) for i in range(n)])
    second = np.stack([R.make_mask(names[(i * 7 + 3) % len(names)], seed=1000 + i) for i in range(n)])
    scratch = torch.empty((n, 5, H * W), dtype=torch.int32, device=DEV)
    raw = scratch.view(torch.uint8).view(n, -1)
    raw[0::2] = 0x7F
    raw[1::2] = 0xFF
    ties = 0
    cv2_boxes = {}  # most generators are not seeded: run cv2 once per distinct mask
    for masks in (first, second):  # the second launch reuses the first one's scratch without clearing it
        got = _ccl(masks, scratch)
        for i in range(n):
            key = masks[i].tobytes()
            if key not in cv2_boxes:
                cv2_boxes[key] = tuple(OT.heatmap_to_bbox(masks[i] * 255))
            exp = cv2_boxes[key]
            assert tuple(got[i]) == exp, f"frame {i} ({names[i % len(names)]}): {tuple(got[i])} vs cv2 {exp}"
        ties += sum(R.component_stats(m)[2] >= 2 for m in masks[:len(names)])
    fg = int(first.sum()) + int(second.sum())
    print(f"ccl: {2 * n} frames, {fg} foreground pixels, {ties} tie frames among the generators")


def test_ccl_rejects_bad_shapes_before_launch():
    scratch = torch.zeros((1, 5, 64), dtype=torch.int32, device=DEV)
    bbox = torch.zeros((1, 4), dtype=torch.int32, device=DEV)
    m = torch.zeros((2, 8, 8), dtype=torch.uint8, device=DEV)
    with pytest.raises(L.PbError):
        L.check(L.lib().pb_ccl_bbox(m.data_ptr(), 1, 3, 5, scratch.data_ptr(), bbox.data_ptr(), L.stream_ptr()))
    with pytest.raises(L.PbError):
        L.check(L.lib().pb_ccl_bbox(m.data_ptr() + 1, 1, 8, 8, scratch.data_ptr(), bbox.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()


# ---- d. pb_tracknet_ensemble_rows in isolation ------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["first", "middle", "tail", "single"])
def test_ensemble_batch_positions(case):
    H, W, B = R.H_NET, R.W_NET, 8
    T = {"single": 12, "first": 40, "middle": 40, "tail": 40}[case]
    S = T - 7
    w0 = {"first": 0, "middle": 16, "tail": S - 5, "single": 0}[case]
    nb = {"first": B, "middle": B, "tail": 5, "single": S}[case]
    g = torch.Generator().manual_seed(len(case))
    preds = torch.rand((S, 8, H, W), generator=g) * 0.6 + 0.2
    exp = OT.ensemble_closed_form(preds, T)
    assert torch.equal(exp, OT.ensemble_reference_loop(preds, T, B))
    buf = torch.zeros((7 + nb, 8, H, W))
    for s in range(w0 - 7, w0 + nb):
        if s >= 0:
            buf[s - (w0 - 7)] = preds[s]
    bd = buf.to(DEV)
    nfr = nb + (7 if w0 + nb == S else 0)
    desc = torch.tensor([(0, S, n) for n in range(w0, w0 + nfr)], dtype=torch.int32, device=DEV)  # the video's clip
    masks, ens = [], None
    for want in (True, False):
        mask = torch.full((nfr, H, W), 7, dtype=torch.uint8, device=DEV)
        e = torch.full((nfr, H, W), -1.0, device=DEV) if want else None
        L.check(L.lib().pb_tracknet_ensemble_rows(bd.data_ptr(), w0 - 7, desc.data_ptr(), nfr, H, W, 0.5,
                                                  mask.data_ptr(), L.ptr(e), L.stream_ptr()))
        torch.cuda.synchronize()
        masks.append(mask.cpu())
        ens = e.cpu() if want else ens
    assert torch.equal(ens, exp[w0:w0 + nfr])
    assert torch.equal(masks[0], masks[1])
    assert torch.equal(masks[0].bool(), exp[w0:w0 + nfr] > 0.5)
    print(f"ensemble {case}: frames {w0}..{w0 + nfr - 1} of {T}, {int(masks[0].sum())} foreground pixels")


def test_ensemble_rejects_missing_windows(tracknet_ckpt):
    """A batch whose frames need windows outside the heat-map buffer (the 7 carried windows and the batch's own) is
    refused on the host, before any device work is enqueued."""
    pipe = BallPipeline(_engine(tracknet_ckpt, 8, SMALL_HW), SRC_HW, synth.make_median(*SRC_HW).numpy())
    desc = lambda frame0, nframes: [(0, 33, n) for n in range(frame0, frame0 + nframes)]  # 33 windows (T = 40)
    # a valid batch first: 8 windows from window 0 emit frames 0..7
    pipe._launch_batch(0, 0, list(range(8)), [0] * 8, desc(0, 8))()
    # the same buffers missing the first / last needed window: (buffer rows = 7 + nb, first buffer row's window)
    for S_buf, first_window, frame0, nframes in ((15, 1, 0, 8), (8, 9, 16, 8), (9, 23, 30, 10)):
        nb = S_buf - 7
        launches = L.lib().pb_launch_count()
        with pytest.raises(L.PbError, match="needs windows"):
            pipe._launch_batch(0, first_window + 7, list(range(nb)), [0] * nb, desc(frame0, nframes))
        assert L.lib().pb_launch_count() == launches
    torch.cuda.synchronize()


# ---- e. pb_inpaintnet_forward against the float64 bound ---------------------------------------------------------------
@pytest.fixture(scope="module")
def inpaint_ckpt():
    return OI.make_inpaintnet()


def _scaled(sd, k):
    return {n: (v * k if n.endswith("weight") else v) for n, v in sd.items()}


@pytest.mark.parametrize("scale", [1, 4])
@pytest.mark.parametrize("Lq", [1, 2, 3, 7, 16, 31, 32])
def test_inpaintnet_within_f64_bound(inpaint_ckpt, Lq, scale):
    from padel_analytics_b200.engine.inpaint_engine import InpaintNetEngine

    sd = _scaled(inpaint_ckpt["model"], scale)
    eng = InpaintNetEngine(sd)
    worst = 0.0
    for N in (1, 37, 5000):
        g = torch.Generator().manual_seed(N * 100 + Lq)
        c = torch.rand((N, Lq, 2), generator=g) * 1.2 - 0.1
        m = (torch.rand((N, Lq, 1), generator=g) > 0.5).float()
        got = eng(c, m)
        ref, bound = R.inpaint_forward_f64(sd, c.to(DEV), m.to(DEV))
        r = R.bound_ratio(got, ref, bound)
        assert r <= 1.0, f"N={N}: worst |err|/bound {r:.3g}"
        worst = max(worst, r)
    print(f"inpaintnet L={Lq} x{scale}: worst |err|/bound {worst:.3g}")


def test_inpaintnet_length_limits(inpaint_ckpt):
    from padel_analytics_b200.engine.inpaint_engine import InpaintNetEngine

    eng = InpaintNetEngine(inpaint_ckpt["model"])
    with pytest.raises(L.PbError):
        eng(torch.zeros((2, 33, 2)), torch.zeros((2, 33, 1)))
    out = torch.full((4,), 3.0, device=DEV)
    c = torch.zeros((4,), device=DEV)
    L.check(L.lib().pb_inpaintnet_forward(c.data_ptr(), c.data_ptr(), 0, 16, eng.blob.data_ptr(), out.data_ptr(),
                                          L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.all(out == 3.0)


def _stage_case(name):
    if name == "golden":
        from fixtures import GOLDEN

        gold = np.load(GOLDEN / "inpaint_ref.npz")
        return (int(gold["W"]), int(gold["H"])), gold["x"].tolist(), gold["y"].tolist(), gold["vis"].tolist()
    seed, T, gaps = {"gap_start": (1, 70, [(0, 6)]), "gap_middle": (2, 120, [(20, 27), (50, 52), (80, 95)]),
                     "gap_end": (3, 64, [(40, 44), (58, 64)])}[name]
    wh = (1920, 1080)
    return (wh,) + R.synthetic_trajectory(seed, T, wh, gaps)


@pytest.mark.parametrize("case", ["golden", "gap_start", "gap_middle", "gap_end"])
def test_inpaint_stage_decisions(inpaint_ckpt, case):
    from padel_analytics_b200.engine.inpaint_engine import InpaintNetEngine

    wh, xs, ys, vs = _stage_case(case)
    eng = InpaintNetEngine(inpaint_ckpt["model"])
    Lq = inpaint_ckpt["param_dict"]["seq_len"]
    got, exp, border, ratio = R.stage_decisions(inpaint_ckpt["model"], eng, xs, ys, vs, Lq, wh, device=DEV)
    bad = R.compare_decisions(got, exp, border)
    masked = int(R.stage_tracker(None, Lq, wh)._generate_inpaint_mask(ys, vs, wh[1] * 0.05).sum())
    print(f"inpaint stage {case}: {len(exp)} frames, {masked} inpainted, worst |err|/bound {ratio:.3g}, "
          f"{len(border)} borderline frames")
    assert ratio <= 1.0
    assert not bad, f"frames {bad[:10]}: kernel {[got[n] for n in bad[:3]]} vs reference {[exp[n] for n in bad[:3]]}"
    assert masked > 0, "nothing was inpainted: the case is vacuous"
    assert len(border) <= max(2, len(exp) // 10)
