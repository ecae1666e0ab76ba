"""Device kernels vs the CPU libraries / oracle on identical inputs: integer paths must be bit-exact."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch
from PIL import Image

from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import resample
from oracle import tracknet as OT
from oracle import yolov8 as OY

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _frames(n, h=1080, w=1920, seed=0):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (n, h // 8, w // 8, 3), dtype=np.uint8)
    up = np.stack([cv2.resize(b, (w, h), interpolation=cv2.INTER_CUBIC) for b in base])
    noise = rng.integers(-20, 21, up.shape, dtype=np.int16)
    return np.clip(up.astype(np.int16) + noise, 0, 255).astype(np.uint8)


@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840), (720, 1280)])
def test_letterbox_bit_exact(hw):
    fr = _frames(2, *hw)
    g = resample.letterbox_geometry(hw[0], hw[1], 640)
    xo, xc = resample.cv2_linear_tables(hw[1], g["rw"])
    yo, yc = resample.cv2_linear_tables(hw[0], g["rh"])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    src, xo, xc, yo, yc = t(fr), t(xo), t(xc), t(yo), t(yc)
    dst = torch.zeros((2, g["Hn"], g["Wn"], 16), dtype=torch.float16, device=DEV)
    L.check(L.lib().pb_letterbox_u8_f16(src.data_ptr(), 2, hw[0], hw[1], dst.data_ptr(), g["Hn"], g["Wn"], g["rh"],
                                        g["rw"], g["top"], g["left"], xo.data_ptr(), xc.data_ptr(), yo.data_ptr(),
                                        yc.data_ptr(), 2, 1, 0, 0, L.stream_ptr()))
    dst4 = torch.zeros((2, g["Hn"] + 2, g["Wn"] + 2, 4), dtype=torch.float16, device=DEV)
    L.check(L.lib().pb_letterbox_u8_f16(src.data_ptr(), 2, hw[0], hw[1], dst4.data_ptr(), g["Hn"], g["Wn"], g["rh"],
                                        g["rw"], g["top"], g["left"], xo.data_ptr(), xc.data_ptr(), yo.data_ptr(),
                                        yc.data_ptr(), 2, 1, 0, 1, L.stream_ptr()))
    torch.cuda.synchronize()
    for i in range(2):
        ref = OY.letterbox(fr[i], 640, auto=True)[..., ::-1]  # BGR -> RGB like the predict pipeline
        exp = (torch.from_numpy(np.ascontiguousarray(ref)).float() * np.float32(1.0 / 255.0)).half()
        got = dst[i, ..., :3].cpu()
        assert got.shape == exp.shape
        assert torch.equal(got, exp), f"max diff {(got.float()-exp.float()).abs().max()*255:.3f} levels"
        assert torch.all(dst[i, ..., 3:] == 0)
        assert torch.equal(dst4[i, 1:-1, 1:-1, :3].cpu(), exp)  # PB_IN_STEM4 layout: same values, zero border
        assert float(dst4[i, 0].abs().max()) == 0 and float(dst4[i, :, -1].abs().max()) == 0
        assert float(dst4[i, ..., 3].abs().max()) == 0


@pytest.mark.parametrize("size", [(512, 288), (1280, 1280), (640, 640)])
@pytest.mark.parametrize("hw", [(1080, 1920), (2160, 3840), (542, 954), (1081, 1936)])
def test_pil_resize_bit_exact(size, hw):
    """(1080, 1920) / (2160, 3840) / (1081, 1936: odd row count) take the multi-row horizontal kernel (4 and 2 rows per
    CTA), width 954 (not a multiple of 16) the one-row kernel."""
    fr = _frames(2, *hw, seed=1)
    Wo, Ho = size
    bh, kh, ksh = resample.pil_bicubic_tables(hw[1], Wo)
    bv, kv, ksv = resample.pil_bicubic_tables(hw[0], Ho)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    src, bh, kh, bv, kv = t(fr), t(bh), t(kh), t(bv), t(kv)
    tmp = torch.zeros((2, hw[0], Wo, 3), dtype=torch.uint8, device=DEV)
    dst = torch.zeros((2, Ho, Wo, 3), dtype=torch.uint8, device=DEV)
    f16 = torch.zeros((2, Ho + 2, Wo + 2, 4), dtype=torch.float16, device=DEV)
    L.check(L.lib().pb_pil_resize_u8(src.data_ptr(), 2, hw[0], hw[1], tmp.data_ptr(), dst.data_ptr(), Ho, Wo,
                                     bh.data_ptr(), kh.data_ptr(), ksh, bv.data_ptr(), kv.data_ptr(), ksv, 1,
                                     f16.data_ptr(), 1, L.stream_ptr()))
    torch.cuda.synchronize()
    for i in range(2):
        ref = np.array(Image.fromarray(cv2.cvtColor(fr[i], cv2.COLOR_BGR2RGB)).resize((Wo, Ho)))
        got = dst[i].cpu().numpy()
        assert np.array_equal(got, ref), f"max diff {np.abs(got.astype(int)-ref).max()}"
        exp16 = (torch.from_numpy(ref).float() * np.float32(1.0 / 255.0)).half()
        assert torch.equal(f16[i, 1:-1, 1:-1, :3].cpu(), exp16)  # fused fp16 network-input output (PB_IN_STEM4)
        assert float(f16[i, 0].abs().max()) == 0 and float(f16[i, ..., 3].abs().max()) == 0


def test_tracknet_pack_windows():
    rng = np.random.default_rng(2)
    ring, B, H, W = 12, 4, 32, 64
    frames = rng.integers(0, 256, (ring, H, W, 3), dtype=np.uint8)
    meds = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
    to4 = lambda a: torch.cat([(torch.from_numpy(a).float() * np.float32(1 / 255.0)).half(),
                               torch.zeros(a.shape[:-1] + (1,), dtype=torch.float16)], -1).contiguous().to(DEV)
    x = torch.zeros((B, H, W, 32), dtype=torch.float16, device=DEV)
    slots, mids = [7, 11, 0, 5], [0, 1, 1, 0]  # rows 0 and 1 wrap the ring
    fd, md = to4(frames), to4(meds)
    sd, mdd = (torch.tensor(v, dtype=torch.int32, device=DEV) for v in (slots, mids))
    L.check(L.lib().pb_tracknet_pack_windows_rows(fd.data_ptr(), ring, sd.data_ptr(), md.data_ptr(), mdd.data_ptr(),
                                                  B, H, W, x.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    got = x.cpu().float()
    for b in range(B):
        chans = [meds[mids[b]]] + [frames[(slots[b] + f) % ring] for f in range(8)]
        exp = np.concatenate(chans, -1).astype(np.float64) / 255.0  # iterable.py:186-197
        assert np.abs(got[b, ..., :27].numpy() - exp).max() < 6e-4
        assert torch.all(got[b, ..., 27:] == 0)


@pytest.mark.parametrize("T,bs", [(30, 8), (8, 4), (9, 8), (15, 3), (23, 16)])
def test_ensemble_matches_reference_loop(T, bs):
    H, W = 24, 40
    g = torch.Generator().manual_seed(T)
    S = T - 7
    preds = torch.rand((S, 8, H, W), generator=g)
    exp = OT.ensemble_reference_loop(preds, T, bs)
    buf = torch.zeros((7 + bs, 8, H, W), device=DEV)
    got = []
    w0 = 0
    while w0 < S:
        nb = min(bs, S - w0)
        buf[7:7 + nb] = preds[w0:w0 + nb].to(DEV)
        nfr = nb + (7 if w0 + nb == S else 0)
        desc = torch.tensor([(0, S, n) for n in range(w0, w0 + nfr)], dtype=torch.int32, device=DEV)  # one clip
        mask = torch.zeros((nfr, H, W), dtype=torch.uint8, device=DEV)
        ens = torch.zeros((nfr, H, W), device=DEV)
        L.check(L.lib().pb_tracknet_ensemble_rows(buf.data_ptr(), w0 - 7, desc.data_ptr(), nfr, H, W, 0.5,
                                                  mask.data_ptr(), ens.data_ptr(), L.stream_ptr()))
        torch.cuda.synchronize()
        got.append(ens.cpu())
        assert torch.equal(mask.cpu().bool(), ens.cpu() > 0.5)
        buf[:7] = buf[nb:nb + 7].clone()
        w0 += nb
    got = torch.cat(got)
    assert got.shape == exp.shape
    assert torch.equal(got, exp), f"max diff {(got-exp).abs().max().item():.3e}"


def _blob_mask(rng, H, W, nblobs):
    m = np.zeros((H, W), np.uint8)
    for _ in range(nblobs):
        cy, cx = rng.integers(0, H), rng.integers(0, W)
        ry, rx = rng.integers(1, 6), rng.integers(1, 9)
        yy, xx = np.ogrid[:H, :W]
        m |= (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).astype(np.uint8)
    return m


def test_ccl_bbox_matches_cv2():
    rng = np.random.default_rng(3)
    H, W = 288, 512
    masks = [np.zeros((H, W), np.uint8)]
    masks += [_blob_mask(rng, H, W, n) for n in (1, 2, 3, 5, 8, 13, 40, 120)]
    masks += [(rng.random((H, W)) < d).astype(np.uint8) for d in (0.001, 0.01, 0.1, 0.3, 0.5, 0.7)]
    m = np.ones((H, W), np.uint8); masks.append(m)  # everything foreground
    m = np.zeros((H, W), np.uint8); m[0, 0] = 1; m[H - 1, W - 1] = 1; masks.append(m)  # equal areas -> tie rule
    m = np.zeros((H, W), np.uint8); m[10:20, 10:20] = 1; m[12:18, 12:18] = 0; m[14:16, 14:16] = 1; masks.append(m)
    n = len(masks)
    md = torch.from_numpy(np.stack(masks)).to(DEV)
    scratch = torch.zeros((n, 5, H * W), dtype=torch.int32, device=DEV)
    bbox = torch.zeros((n, 4), dtype=torch.int32, device=DEV)
    L.check(L.lib().pb_ccl_bbox(md.data_ptr(), n, H, W, scratch.data_ptr(), bbox.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    got = bbox.cpu().numpy()
    for i, mk in enumerate(masks):
        exp = tuple(OT.heatmap_to_bbox(mk * 255))
        assert tuple(got[i]) == exp, f"mask {i}: got {tuple(got[i])} expected {exp}"


@pytest.mark.parametrize("nc,kpt,classes,dense", [(80, None, [0], False), (1, (13, 3), None, False),
                                                  (1, (12, 3), None, False), (1, (13, 2), None, False),
                                                  (80, None, [0, 3, 17], False),  # class LIST filter (predict(classes=[...]))
                                                  (80, None, None, False),
                                                  (1, (13, 3), None, True)])  # > 4096 candidates: global-scratch NMS path
def test_decode_nms_matches_oracle(nc, kpt, classes, dense):
    torch.manual_seed(nc + (kpt[0] if kpt else 0))
    B, shapes = 3, [(48, 80), (24, 40), (12, 20)]
    nk = kpt[0] * kpt[1] if kpt else 0
    fC = 64 + nc + nk
    raws = []
    for (h, w) in shapes:
        r = torch.randn(B, fC, h, w)
        r[:, :64] *= 2.0
        r[:, 64:64 + nc] = r[:, 64:64 + nc] * 1.5 - (4.0 if nc > 1 else 2.0) + (6.0 if dense else 0.0)
        raws.append(r)
    head = OY.PoseHead(nc, kpt, (64, 128, 256)) if kpt else OY.DetectHead(nc, (64, 128, 256))
    if kpt:
        y, anc, st = head.decode_boxes(raws)
        kp = torch.cat([r[:, 64 + nc:].reshape(B, nk, -1) for r in raws], 2)
        K, D = kpt
        k = kp.view(B, K, D, -1).clone()
        k[:, :, 0] = (k[:, :, 0] * 2.0 + (anc[0] - 0.5)) * st
        k[:, :, 1] = (k[:, :, 1] * 2.0 + (anc[1] - 0.5)) * st
        if D == 3:
            k[:, :, 2] = k[:, :, 2].sigmoid()
        pred = torch.cat([y, k.view(B, nk, -1)], 1)
    else:
        pred, _, _ = head.decode_boxes(raws)
    conf, iou, max_det = 0.5, 0.7, 300
    exp = OY.non_max_suppression(pred, conf, iou, classes, max_det, nc)

    feats = [r.permute(0, 2, 3, 1).contiguous().to(DEV) for r in raws]
    lv = (L.YoloLevel * 3)()
    for l, (f, (h, w), s) in enumerate(zip(feats, shapes, (8, 16, 32))):
        lv[l].feat, lv[l].h, lv[l].w, lv[l].stride = f.data_ptr(), h, w, s
    cap, rowlen = sum(h * w for h, w in shapes), 6 + nk  # every anchor (5040 here), as the engine sizes it
    cand = torch.zeros((B, cap, rowlen), device=DEV)
    anchor = torch.zeros((B, cap), dtype=torch.int32, device=DEV)
    count = torch.zeros((B,), dtype=torch.int32, device=DEV)
    carr = (C.c_int * len(classes))(*classes) if classes is not None else None
    L.check(L.lib().pb_yolo_decode(lv, 3, B, fC, nc, nk, kpt[1] if kpt else 0, 64, 64 + nc, conf, carr,
                                   len(classes) if classes is not None else 0,
                                   cand.data_ptr(), anchor.data_ptr(), count.data_ptr(), cap, L.stream_ptr()))
    out = torch.zeros((B, max_det, rowlen), device=DEV)
    ocnt = torch.zeros((B,), dtype=torch.int32, device=DEV)
    scratch = torch.empty((max(16, L.lib().pb_yolo_nms_scratch_bytes(B, cap)),), dtype=torch.uint8, device=DEV)
    L.check(L.lib().pb_yolo_nms(cand.data_ptr(), anchor.data_ptr(), count.data_ptr(), B, cap, rowlen, iou, max_det,
                                out.data_ptr(), ocnt.data_ptr(), scratch.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    assert int(count.max()) <= cap
    if dense:
        assert int(count.min()) > 4096, "dense case must exercise the global-scratch path"
    for b in range(B):
        e = exp[b]
        n = int(ocnt[b])
        assert n == e.shape[0], f"image {b}: kept {n} vs oracle {e.shape[0]} (candidates {int(count[b])})"
        assert n > 3, "test is vacuous"
        g = out[b, :n].cpu()
        assert torch.allclose(g, e, rtol=1e-4, atol=2e-3), f"image {b}: max diff {(g-e).abs().max()}"


@pytest.mark.parametrize("T", [1, 2, 7, 8, 255, 300, 401])
def test_median_kernel_matches_numpy(T):
    """pb_median_u8 == np.median(frames_rgb, 0).astype('uint8') (iterable.py:58-81), odd and even counts, counter
    spill past 255 frames, constant / bimodal columns, BGR -> RGB output order."""
    rng = np.random.default_rng(T)
    H, W = 36, 52
    fr = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
    fr[:, 0, 0] = 255
    fr[:, 0, 1] = 0
    fr[: T // 2, 0, 2] = 255
    fr[T // 2:, 0, 2] = 0
    fr[:, 1] = (fr[:, 1] // 64) * 64  # few distinct values: many ties
    ref = np.median(fr[..., ::-1], 0).astype("uint8")  # the reference converts BGR -> RGB first
    src = torch.from_numpy(fr).to(DEV)
    out = torch.zeros((H, W, 3), dtype=torch.uint8, device=DEV)
    L.check(L.lib().pb_median_u8(src.data_ptr(), T, H * W * 3, out.data_ptr(), 1, L.stream_ptr()))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)
    out2 = torch.zeros((H, W, 3), dtype=torch.uint8, device=DEV)
    L.check(L.lib().pb_median_u8(src.data_ptr(), T, H * W * 3, out2.data_ptr(), 0, L.stream_ptr()))
    torch.cuda.synchronize()
    assert np.array_equal(out2.cpu().numpy(), np.median(fr, 0).astype("uint8"))


def test_median_background_full_frames():
    """trackers.ball_tracker.median_background on 1080p frames (list of BGR arrays) == the reference's np.median."""
    from padel_analytics_b200 import synth
    from padel_analytics_b200.trackers.ball_tracker import median_background

    fr = [f.numpy() for f in synth.make_frames(12, 1080, 1920, start=40)]
    ref = np.median(np.array([cv2.cvtColor(f, cv2.COLOR_BGR2RGB) for f in fr]), 0).astype("uint8")
    assert np.array_equal(median_background(fr), ref)
    assert np.array_equal(median_background(fr[:11]), np.median(np.array([f[..., ::-1] for f in fr[:11]]), 0).astype("uint8"))


def test_resamplers_bit_exact_on_natural_frames():
    """LetterBox and the Pillow resize on real video content (the committed rally.mp4 crops + a 720p frame)."""
    from fixtures import GOLDEN, rally_frames

    frames = rally_frames() + [cv2.imread(str(GOLDEN / "rally" / "rally_f00_720p.jpg"))]
    for f in frames:
        Hs, Ws = f.shape[:2]
        fr = np.ascontiguousarray(f[None])
        g = resample.letterbox_geometry(Hs, Ws, 640)
        xo, xc = resample.cv2_linear_tables(Ws, g["rw"])
        yo, yc = resample.cv2_linear_tables(Hs, g["rh"])
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
        src, xo, xc, yo, yc = t(fr), t(xo), t(xc), t(yo), t(yc)
        dst = torch.zeros((1, g["Hn"], g["Wn"], 16), dtype=torch.float16, device=DEV)
        L.check(L.lib().pb_letterbox_u8_f16(src.data_ptr(), 1, Hs, Ws, dst.data_ptr(), g["Hn"], g["Wn"], g["rh"], g["rw"],
                                            g["top"], g["left"], xo.data_ptr(), xc.data_ptr(), yo.data_ptr(),
                                            yc.data_ptr(), 2, 1, 0, 0, L.stream_ptr()))
        ref = OY.letterbox(f, 640, auto=True)[..., ::-1]
        exp = (torch.from_numpy(np.ascontiguousarray(ref)).float() * np.float32(1.0 / 255.0)).half()
        assert torch.equal(dst[0, ..., :3].cpu(), exp)
        for Wo, Ho in ((512, 288), (640, 640)):
            bh, kh, ksh = resample.pil_bicubic_tables(Ws, Wo)
            bv, kv, ksv = resample.pil_bicubic_tables(Hs, Ho)
            bh, kh, bv, kv = t(bh), t(kh), t(bv), t(kv)
            tmp = torch.zeros((1, Hs, Wo, 3), dtype=torch.uint8, device=DEV)
            out = torch.zeros((1, Ho, Wo, 3), dtype=torch.uint8, device=DEV)
            L.check(L.lib().pb_pil_resize_u8(src.data_ptr(), 1, Hs, Ws, tmp.data_ptr(), out.data_ptr(), Ho, Wo,
                                             bh.data_ptr(), kh.data_ptr(), ksh, bv.data_ptr(), kv.data_ptr(), ksv, 1,
                                             None, 0, L.stream_ptr()))
            refp = np.array(Image.fromarray(cv2.cvtColor(f, cv2.COLOR_BGR2RGB)).resize((Wo, Ho)))
            assert np.array_equal(out[0].cpu().numpy(), refp)
