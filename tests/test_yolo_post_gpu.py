"""yolo_decode_kernel and yolo_nms_kernel against the host restatement (yolo_post_ref.py), decision for decision.

NMS: hand-built candidate buffers (decode bypassed) reach every edge directly -- both working-set paths in one launch,
capacities from 1 to 32768, count > cap, slot order, conf ties, IoU exactly float32(t), NaN IoU, class offsets that
overlap, max_det and row lengths.  The kernel must equal the restatement exactly: count, order and row bits; rows from
out_count on keep their fill; a second run is bit-identical.

Decode: random head maps at the engines' geometries (plus 1 and 4 levels, 256 classes with a class filter, a batch
that wraps the grid-stride loop, constructed class ties) against the float64 decode: the candidate set, class and
anchor columns exactly, cand_count exactly, values within the derived bound.  The NMS then runs on the kernel's own
candidates and must equal the restatement on those rows exactly.

Each case prints one line: candidates, kept, NMS path, borderline exclusions and the worst decode error / bound.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import yolo_post_ref as YR
from padel_analytics_b200 import _lib as L

pytestmark = pytest.mark.gpu
DEV = "cuda"
MARK = 0x7FC0DEAD  # a NaN payload: the fill of every output row the kernels must not write
SMEM_CAP = 4096    # kNmsSmemCap: images with more candidates run the NMS on the global scratch area


def _path(counts, cap):
    n = [min(int(c), cap) for c in counts]
    paths = {"smem" if c <= SMEM_CAP else "scratch" for c in n if c > 0}
    return "+".join(sorted(paths)) or "-"


def _run_nms(cand, anchor, count, cap, iou, max_det):
    """pb_yolo_nms on host buffers, twice; returns (out rows as int32 bits (B, max(max_det, 1), rowlen), out_count)."""
    B, _, rowlen = cand.shape
    c, a, n = cand.to(DEV), anchor.to(DEV), count.to(DEV)
    runs = []
    for _ in range(2):
        out = torch.full((B, max(max_det, 1), rowlen), MARK, dtype=torch.int32, device=DEV)
        ocnt = torch.full((B,), -1, dtype=torch.int32, device=DEV)
        scratch = torch.empty((max(16, L.lib().pb_yolo_nms_scratch_bytes(B, cap)),), dtype=torch.uint8, device=DEV)
        L.check(L.lib().pb_yolo_nms(c.data_ptr(), a.data_ptr(), n.data_ptr(), B, cap, rowlen, iou, max_det,
                                    out.data_ptr(), ocnt.data_ptr(), scratch.data_ptr(), L.stream_ptr()))
        torch.cuda.synchronize()
        runs.append((out.cpu(), ocnt.cpu()))
    (o1, n1), (o2, n2) = runs
    assert torch.equal(n1, n2) and torch.equal(o1, o2), "two runs of the NMS kernel differ"
    return o1, n1


def _check_nms(cand, anchor, count, cap, iou, max_det, out, ocnt, tag=""):
    """The kernel's output equals the restatement on the first min(count, cap) slots of every image, bit for bit."""
    kept = []
    for b in range(cand.shape[0]):
        m = min(int(count[b]), cap)
        rows = cand[b, :m]
        k = YR.nms_ref(rows.numpy(), anchor[b, :m].numpy(), iou, max_det)
        n = int(ocnt[b])
        assert n == len(k), f"{tag}image {b}: the kernel kept {n} rows, the restatement {len(k)} (of {m} candidates)"
        exp = rows[torch.from_numpy(k)].contiguous().view(torch.int32)
        got = out[b, :n]
        if not torch.equal(got, exp):
            i = int((got != exp).any(1).nonzero()[0])
            g, e = got[i].view(torch.float32)[:6].tolist(), exp[i].view(torch.float32)[:6].tolist()
            raise AssertionError(f"{tag}image {b}: output row {i} differs: got {g} expected {e}")
        assert (out[b, n:] == MARK).all(), f"{tag}image {b}: rows from out_count {n} on were written"
        kept.append(n)
    return kept


def _buffers(rng, counts, cap, rowlen, nclass=3):
    """Candidate buffers holding random rows in the first min(count, cap) slots of each image."""
    B = len(counts)
    cand = torch.full((B, cap, rowlen), MARK, dtype=torch.int32).view(torch.float32)
    anchor = torch.full((B, cap), -1, dtype=torch.int32)
    for b, n in enumerate(counts):
        m = min(n, cap)
        rows, a = YR.random_candidates(rng, m, rowlen, nclass)
        cand[b, :m] = torch.from_numpy(rows)
        anchor[b, :m] = torch.from_numpy(a)
    return cand, anchor, torch.tensor(counts, dtype=torch.int32)


def _nms_case(tag, cand, anchor, count, cap, iou=0.7, max_det=300):
    out, ocnt = _run_nms(cand, anchor, count, cap, iou, max_det)
    kept = _check_nms(cand, anchor, count, cap, iou, max_det, out, ocnt, tag + ": ")
    print(f"\nnms {tag:28s} candidates {[int(c) for c in count]} cap {cap} kept {kept} path {_path(count, cap)}")
    return kept


# ---- NMS on hand-built candidates ----------------------------------------------------------------------------------
def test_nms_both_paths_one_launch():
    """Shared-memory and scratch images side by side; Pe below and above blockDim (1024)."""
    counts = [0, 1, 2, 1024, 1025, 4096, 4097, 30000]
    cand, anchor, count = _buffers(np.random.default_rng(1), counts, 30000, 6)
    kept = _nms_case("mixed_paths", cand, anchor, count, 30000)
    assert kept[0] == 0 and kept[1] == 1 and min(kept[3:]) > 100


@pytest.mark.parametrize("cap", [1, 2, 3, 4096, 4097, 30000, 32768], ids=lambda c: f"cap{c}")
def test_nms_capacity(cap):
    """count 0, 1, cap / 2, cap and cap + 7 (only the first cap slots count) at every capacity."""
    counts = [0, 1, max(cap // 2, 1), cap, cap + 7]
    cand, anchor, count = _buffers(np.random.default_rng(cap), counts, cap, 6)
    _nms_case(f"cap{cap}", cand, anchor, count, cap)


@pytest.mark.parametrize("n", [3000, 5000])
def test_nms_slot_order_does_not_matter(n):
    """The decode kernel's atomics leave candidates in any slot order: a permutation gives the identical output."""
    rng = np.random.default_rng(n)
    cand, anchor, count = _buffers(rng, [n], n, 45, nclass=1)
    perm = torch.from_numpy(rng.permutation(n))
    out1, c1 = _run_nms(cand, anchor, count, n, 0.7, 300)
    out2, c2 = _run_nms(cand[:, perm].contiguous(), anchor[:, perm].contiguous(), count, n, 0.7, 300)
    assert torch.equal(c1, c2) and torch.equal(out1, out2), "slot order changed the output"
    _check_nms(cand, anchor, count, n, 0.7, 300, out1, c1, f"slot order n={n}: ")


@pytest.mark.parametrize("t", sorted(YR.IOU_FRACTIONS), ids=lambda t: f"iou{t}")
def test_nms_iou_exactly_float_threshold(t):
    """IoU exactly float32(t): torchvision suppresses iff float64(float32(t)) > t (for 0.3, 0.6 and 0.8)."""
    rows = torch.from_numpy(YR.iou_pair_rows(t))
    cand, anchor = rows[None], torch.tensor([[3, 5, 9, 8]], dtype=torch.int32)
    count = torch.tensor([4], dtype=torch.int32)
    out, ocnt = _run_nms(cand, anchor, count, 4, t, 300)
    exp = 2 if YR.SUPPRESSED_AT_FLOAT_T[t] else 4
    assert int(ocnt[0]) == exp, (f"iou={t}: IoU exactly float32({t}): the kernel kept {int(ocnt[0])} of 4 boxes, "
                                 f"torchvision keeps {exp}")
    _check_nms(cand, anchor, count, 4, t, 300, out, ocnt, f"iou={t}: ")


def test_nms_edge_cases():
    """Zero-area boxes (NaN IoU), identical boxes in different classes, class offsets overlapping beyond 7680, conf
    ties at 1.0 -- one image each, in one launch per IoU threshold."""
    for iou in sorted({c[3] for c in YR.edge_case_rows()}):
        cases = [c for c in YR.edge_case_rows() if c[3] == iou]
        cap = max(len(c[1]) for c in cases)
        cand = torch.full((len(cases), cap, 6), MARK, dtype=torch.int32).view(torch.float32)
        anchor = torch.full((len(cases), cap), -1, dtype=torch.int32)
        for b, (_, rows, a, _, _) in enumerate(cases):
            cand[b, :len(rows)] = torch.from_numpy(rows)
            anchor[b, :len(rows)] = torch.from_numpy(a.astype(np.int32))
        count = torch.tensor([len(c[1]) for c in cases], dtype=torch.int32)
        out, ocnt = _run_nms(cand, anchor, count, cap, iou, 300)
        _check_nms(cand, anchor, count, cap, iou, 300, out, ocnt, f"edge cases iou={iou}: ")
        for b, (name, rows, _, _, kept) in enumerate(cases):
            exp = torch.from_numpy(rows[kept]).view(torch.int32)
            assert torch.equal(out[b, :len(kept)], exp), f"{name}: kept rows differ from {kept}"


@pytest.mark.parametrize("max_det", [0, 1, 300, 4001])
def test_nms_max_det(max_det):
    """4001 is more than every image's survivors: the whole greedy pass is emitted."""
    cand, anchor, count = _buffers(np.random.default_rng(max_det), [2500, 800, 4000], 4000, 6)
    kept = _nms_case(f"max_det{max_det}", cand, anchor, count, 4000, 0.7, max_det)
    if max_det == 4001:
        assert max(kept) > 300


@pytest.mark.parametrize("rowlen", [6, 32, 42, 45, 57])
def test_nms_row_length(rowlen):
    """Keypoint payloads of every shipped and ultralytics shape (13x2, 12x3, 13x3, 17x3) are copied bit for bit."""
    cand, anchor, count = _buffers(np.random.default_rng(rowlen), [700, 5000, 0], 5000, rowlen)
    _nms_case(f"rowlen{rowlen}", cand, anchor, count, 5000, 0.45)


# ---- decode ------------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# name: (B, (Hn, Wn), strides, nc, kpt, classes, conf, class-logit shift, extra options)
DECODE_CASES = {
    "det80_384x640_cls0": (3, (384, 640), (8, 16, 32), 80, None, [0], 0.5, 0.0, {}),
    "det80_640": (2, (640, 640), (8, 16, 32), 80, None, None, 0.5, 0.0, {"iou": 0.45}),
    "det80_640_1level": (2, (640, 640), (8,), 80, None, [0, 3, 17], 0.5, 0.0, {}),
    "det256_filter": (2, (640, 640), (8, 16, 32), 256, None, [0, 63, 64, 127, 128, 191, 192, 255], 0.5, 0.0, {}),
    "det256_empty_filter": (2, (640, 640), (8, 16, 32), 256, None, [], 0.5, 0.0, {}),
    "det256": (2, (640, 640), (8, 16, 32), 256, None, None, 0.5, 0.0, {}),
    "pose13x3_1280": (2, (1280, 1280), (8, 16, 32), 1, (13, 3), None, 0.25, 0.0, {}),
    "pose13x3_1280_over_cap": (2, (1280, 1280), (8, 16, 32), 1, (13, 3), None, 0.25, 6.0, {}),
    "court12x3_640_offsets": (2, (640, 640), (8, 16, 32), 1, (12, 3), None, 0.5, 0.0, {"gap": True}),
    "pose13x2_384x640": (3, (384, 640), (8, 16, 32), 1, (13, 2), None, 0.5, 0.0, {}),
    "pose17x3_640_4levels": (2, (640, 640), (8, 16, 32, 64), 1, (17, 3), None, 0.25, 0.0, {}),
    "det1_1280_grid_wrap": (None, (1280, 1280), (8, 16, 32), 1, None, None, 0.5, 0.0, {}),
    "ties": (2, (384, 640), (8, 16, 32), 80, None, None, 0.25, 0.0, {"ties": True}),
    "ties_cls0": (2, (384, 640), (8, 16, 32), 80, None, [0], 0.25, 0.0, {"ties": True}),
}
# (class index -> logit) patterns over a background of -8 at anchors p mod 20 of every level (p = pattern index);
# ultralytics' best class in the comment
TIES = [{0: 20.0, 1: 25.0},   # saturated, distinct logits: 0
        {3: 2.0, 7: 2.0},     # exact tie: 3
        {0: 30.0, 79: 30.0},  # exact and saturated: 0
        {2: 17.5, 5: 40.0}]   # saturated, distinct logits: 2


def _head_maps(seed, B, Hn, Wn, strides, nc, nk, shift, gap, ties):
    g = torch.Generator().manual_seed(seed)
    cls_off = 64 + (8 if gap else 0)
    kpt_off = cls_off + nc + (5 if gap else 0)
    fC = kpt_off + nk + (3 if gap else 0)
    levels = []
    for s in strides:
        h, w = Hn // s, Wn // s
        f = torch.randn(B, h, w, fC, generator=g)
        f[..., :64] *= 2.0
        f[..., cls_off:cls_off + nc] = f[..., cls_off:cls_off + nc] * 1.5 - (4.0 if nc > 1 else 2.0) + shift
        levels.append((f, s))
    if ties:
        for f, _ in levels:
            c = f.view(B, -1, fC)[..., cls_off:cls_off + nc]
            for p, pat in enumerate(TIES):
                sel = c[:, p::20]
                sel.fill_(-8.0)
                for j, v in pat.items():
                    sel[..., j] = v
    return levels, fC, cls_off, kpt_off


@pytest.mark.parametrize("name", list(DECODE_CASES))
def test_decode_then_nms(name):
    B, (Hn, Wn), strides, nc, kpt, classes, conf, shift, opt = DECODE_CASES[name]
    A = sum((Hn // s) * (Wn // s) for s in strides)
    if B is None:  # one more image than the grid-stride loop covers in one pass (32 blocks of 128 per SM)
        B = _sms() * 32 * 128 // A + 1
        assert B * A > _sms() * 32 * 128
    nk, kdim = (kpt[0] * kpt[1], kpt[1]) if kpt else (0, 0)
    levels, fC, cls_off, kpt_off = _head_maps(list(DECODE_CASES).index(name), B, Hn, Wn, strides, nc, nk, shift, opt.get("gap"),
                                              opt.get("ties"))
    cap, rowlen = min(A, 30000), 6 + nk
    feats = [f.to(DEV) for f, _ in levels]
    lv = (L.YoloLevel * len(levels))()
    for l, (f, s) in enumerate(zip(feats, strides)):
        lv[l].feat, lv[l].h, lv[l].w, lv[l].stride = f.data_ptr(), f.shape[1], f.shape[2], s
    cand = torch.full((B, cap, rowlen), MARK, dtype=torch.int32, device=DEV).view(torch.float32)
    anchor = torch.full((B, cap), -1, dtype=torch.int32, device=DEV)
    count = torch.full((B,), -1, dtype=torch.int32, device=DEV)
    carr = (C.c_int * max(len(classes), 1))(*classes) if classes is not None else None
    L.check(L.lib().pb_yolo_decode(lv, len(levels), B, fC, nc, nk, kdim, cls_off, kpt_off, conf, carr,
                                   len(classes) if classes is not None else 0, cand.data_ptr(), anchor.data_ptr(),
                                   count.data_ptr(), cap, L.stream_ptr()))
    torch.cuda.synchronize()
    cand, anchor, count = cand.cpu(), anchor.cpu(), count.cpu()

    ref = YR.decode_ref(levels, nc, nk, kdim, cls_off, kpt_off, conf, classes)
    rep = YR.compare_decode(ref, cand, anchor, count, cap)
    assert rep.ok, f"{name}: decode: " + "; ".join(rep.fails[:4])
    for b in range(B):  # the marker fill past the written slots is untouched
        m = min(int(count[b]), cap)
        assert (cand[b, m:].view(torch.int32) == MARK).all() and (anchor[b, m:] == -1).all(), f"{name}: image {b}"
    if classes == []:
        assert int(count.sum()) == 0
    else:
        assert int(count.min()) > 0, f"{name}: vacuous"
    if shift > 0:
        assert int(count.min()) > cap, f"{name}: the case must overflow the capacity"
    if opt.get("ties"):
        assert all(len(s) for s in ref.sure)

    iou = opt.get("iou", 0.7)
    out, ocnt = _run_nms(cand, anchor, count, cap, iou, 300)
    kept = _check_nms(cand, anchor, count, cap, iou, 300, out, ocnt, f"{name}: nms: ")
    print(f"\ndecode {name:28s} B {B:2d} anchors {A:5d} cap {cap:5d} | candidates {int(count.sum()):6d} "
          f"kept {sum(kept):5d} path {_path(count, cap):12s} | border {rep.border:3d} "
          f"err/bound {rep.max_err_ratio:.3f}")
