"""Self-test of the YOLO post-processing restatement (yolo_post_ref.py): its NMS is torchvision.ops.nms index for
index, decode + NMS reproduce the oracle's ultralytics pipeline, and the decode comparator catches a shifted DFL bin
and swapped box sides."""
import numpy as np
import pytest
import torch
import torchvision

import yolo_post_ref as YR
from oracle import yolov8 as OY


def _tv(boxes, scores, iou):
    return torchvision.ops.nms(torch.from_numpy(boxes), torch.from_numpy(scores), iou).numpy()


def _ref(boxes, scores, iou):
    order = YR.score_order(scores, np.arange(len(scores)))
    return order[YR.greedy_nms(boxes[order], iou)]


@pytest.mark.parametrize("n", [0, 1, 2, 50, 500, 3000])
@pytest.mark.parametrize("iou", [0.3, 0.45, 0.5, 0.6, 0.7, 0.8])
def test_nms_ref_matches_torchvision_random(n, iou):
    rng = np.random.default_rng(n * 10 + int(iou * 100))
    b, s = YR.random_boxes(rng, n)
    exp = _tv(b, s, iou)
    got = _ref(b, s, iou)
    assert np.array_equal(got, exp), f"kept {len(got)} vs torchvision {len(exp)}"
    if n >= 50:
        assert 0 < len(exp) < n, "no suppression: vacuous"


def _tv_rows(rows, anchors, iou):
    """ultralytics' NMS call on the candidates in anchor order (as it hands them over), indices into `rows`."""
    by_anchor = np.argsort(anchors, kind="stable")
    r = rows[by_anchor]
    return by_anchor[_tv(r[:, :4] + r[:, 5:6] * np.float32(YR.MAX_WH), r[:, 4], iou)]


@pytest.mark.parametrize("t", sorted(YR.IOU_FRACTIONS))
def test_nms_ref_iou_exactly_float_threshold(t):
    k, D = YR.IOU_FRACTIONS[t]
    assert np.float32(k) / np.float32(D) == np.float32(t)
    rows = YR.iou_pair_rows(t)
    anchors = np.array([3, 5, 9, 8])
    exp = _tv_rows(rows, anchors, t)
    assert np.array_equal(YR.nms_ref(rows, anchors, t, 300), exp)
    assert exp.tolist() == ([3, 0] if YR.SUPPRESSED_AT_FLOAT_T[t] else [3, 2, 0, 1])


@pytest.mark.parametrize("name,rows,anchors,iou,kept", YR.edge_case_rows(), ids=[c[0] for c in YR.edge_case_rows()])
def test_nms_ref_edge_cases(name, rows, anchors, iou, kept):
    got = YR.nms_ref(rows, anchors, iou, 300)
    assert np.array_equal(got, _tv_rows(rows, anchors, iou))
    assert got.tolist() == kept


def test_nms_ref_max_det():
    rng = np.random.default_rng(7)
    b, s = YR.random_boxes(rng, 800)
    rows = np.concatenate([b, s[:, None], rng.integers(0, 3, (800, 1)).astype(np.float32)], 1)
    a = np.arange(800)
    full = YR.nms_ref(rows, a, 0.7, 10 ** 6)
    assert 300 < len(full) < 800
    for md in (0, 1, 300, len(full) + 5):
        assert np.array_equal(YR.nms_ref(rows, a, 0.7, md), full[:md])


def test_sigmoid_saturates_at_17():
    x = torch.tensor([YR.SATURATED_LOGIT, 20.0, 25.0, 88.0], dtype=torch.float32)
    assert (torch.sigmoid(x) == 1.0).all()
    x = torch.tensor(YR.SATURATED_LOGIT, dtype=torch.float32)
    assert 1.0 / (1.0 + np.exp(np.float32(-x.item()))) == np.float32(1.0)


# ---- decode --------------------------------------------------------------------------------------------------------
SHAPES = [(48, 80), (24, 40), (12, 20)]


def _raws(seed, nc, nk, B=3):
    g = torch.Generator().manual_seed(seed)
    raws = []
    for h, w in SHAPES:
        r = torch.randn(B, 64 + nc + nk, h, w, generator=g)
        r[:, :64] *= 2.0
        r[:, 64:64 + nc] = r[:, 64:64 + nc] * 1.5 - (4.0 if nc > 1 else 2.0)
        raws.append(r)
    return raws


def _levels(raws):
    return [(r.permute(0, 2, 3, 1).contiguous(), s) for r, s in zip(raws, (8, 16, 32))]


def _oracle_pred(raws, nc, kpt):
    B = raws[0].shape[0]
    head = OY.PoseHead(nc, kpt, (64, 128, 256)) if kpt else OY.DetectHead(nc, (64, 128, 256))
    y, anc, st = head.decode_boxes(raws)
    if not kpt:
        return y
    nk = kpt[0] * kpt[1]
    k = torch.cat([r[:, 64 + nc:].reshape(B, nk, -1) for r in raws], 2).view(B, kpt[0], kpt[1], -1).clone()
    k[:, :, 0] = (k[:, :, 0] * 2.0 + (anc[0] - 0.5)) * st
    k[:, :, 1] = (k[:, :, 1] * 2.0 + (anc[1] - 0.5)) * st
    if kpt[1] == 3:
        k[:, :, 2] = k[:, :, 2].sigmoid()
    return torch.cat([y, k.view(B, nk, -1)], 1)


def _oracle_candidates(pred, conf, classes, nc):
    """ultralytics non_max_suppression up to the NMS call: per image the float32 candidate rows and their anchors."""
    out = []
    for x in pred.transpose(-1, -2):
        x = x.clone()
        x[:, :4] = OY.xywh2xyxy(x[:, :4])
        box, cls, mask = x.split((4, nc, x.shape[1] - 4 - nc), 1)
        c, j = cls.max(1, keepdim=True)
        rows = torch.cat((box, c, j.float(), mask), 1)
        keep = c.view(-1) > conf
        if classes is not None:
            keep &= (j == torch.tensor(classes)).any(1)
        out.append((rows[keep].numpy(), torch.nonzero(keep)[:, 0].numpy()))
    return out


CASES = [(80, None, [0]), (80, None, [0, 3, 17]), (80, None, None), (1, (13, 3), None), (1, (12, 3), None),
         (1, (13, 2), None)]


@pytest.mark.parametrize("nc,kpt,classes", CASES)
def test_decode_nms_ref_matches_oracle(nc, kpt, classes):
    nk = kpt[0] * kpt[1] if kpt else 0
    raws = _raws(nc + nk, nc, nk)
    conf, iou, max_det = 0.5, 0.7, 300
    pred = _oracle_pred(raws, nc, kpt)
    exp = OY.non_max_suppression(pred, conf, iou, classes, max_det, nc)
    ref = YR.decode_ref(_levels(raws), nc, nk, kpt[1] if kpt else 0, 64, 64 + nc, conf, classes)
    for b, (orows, oanch) in enumerate(_oracle_candidates(pred, conf, classes, nc)):
        assert len(ref.border[b]) == 0
        # the candidate set and the classes are the oracle's
        assert np.array_equal(ref.sure[b], oanch)
        assert np.array_equal(ref.rows[b, oanch, 5].numpy(), orows[:, 5])
        # NMS restated on the oracle's own candidate rows is the oracle's output, bit for bit
        k = YR.nms_ref(orows, oanch, iou, max_det)
        assert len(k) > 3, "vacuous"
        assert np.array_equal(orows[k].view(np.int32), exp[b].numpy().view(np.int32))
        # decode + NMS restated: the same detections, in the same order, within float32 of the oracle's values
        mine = ref.kernel_rows(b, ref.sure[b]).numpy()
        km = YR.nms_ref(mine, ref.sure[b], iou, max_det)
        assert np.array_equal(ref.sure[b][km], oanch[k])
        np.testing.assert_allclose(mine[km], exp[b].numpy(), rtol=2e-6, atol=2e-4)


def test_decode_ref_best_class_saturated_and_tied():
    """First maximum of the float32 sigmoid, as ultralytics: [20, 25, 0] -> class 0; exact ties -> first index."""
    nc = 3
    f = torch.full((1, 1, 4, 64 + nc), -6.0)
    f[0, 0, 0, 64:] = torch.tensor([20.0, 25.0, 0.0])
    f[0, 0, 1, 64:] = torch.tensor([-1.0, 3.0, 3.0])
    f[0, 0, 2, 64:] = torch.tensor([0.0, 0.0, 40.0])
    f[0, 0, 3, 64:] = torch.tensor([16.0, 16.0 + 2 ** -19, 0.0])  # distinct logits, sigmoids a few ulps apart
    ref = YR.decode_ref([(f, 8)], nc, 0, 0, 64, 0, 0.25)
    assert ref.rows[0, :3, 5].tolist() == [0.0, 1.0, 2.0]
    assert ref.sure[0].tolist() == [0, 1, 2] and ref.border[0].tolist() == [3]
    ref0 = YR.decode_ref([(f, 8)], nc, 0, 0, 64, 0, 0.25, classes=[0])
    assert ref0.sure[0].tolist() == [0]


def _kernel_like(ref, seed=0):
    """Buffers as the decode kernel leaves them, from the reference: rows rounded to float32, slots in random order."""
    B = len(ref.sure)
    cap = max(len(s) for s in ref.sure) + 4
    rowlen = ref.rows.shape[-1]
    cand = torch.full((B, cap, rowlen), float("nan"))
    anchor = torch.full((B, cap), -1, dtype=torch.int32)
    count = torch.zeros(B, dtype=torch.int32)
    rng = np.random.default_rng(seed)
    for b in range(B):
        a = rng.permutation(ref.sure[b])
        cand[b, :len(a)] = ref.kernel_rows(b, a)
        anchor[b, :len(a)] = torch.from_numpy(a.astype(np.int32))
        count[b] = len(a)
    return cand, anchor, count, cap


@pytest.mark.parametrize("mutation", [None, "dfl_bin_shift", "swap_sides", "class", "drop", "extra"])
def test_decode_comparator_catches_mutations(mutation):
    nc, kpt = 1, (13, 3)
    nk = 39
    raws = _raws(5, nc, nk)
    lv = _levels(raws)
    ref = YR.decode_ref(lv, nc, nk, 3, 64, 64 + nc, 0.5)
    if mutation in ("dfl_bin_shift", "swap_sides"):
        mut = []
        for f, s in lv:
            f = f.clone()
            if mutation == "dfl_bin_shift":  # side 0's logits one bin up: dist + ~1
                f[..., 0:16] = torch.roll(f[..., 0:16], 1, -1)
            else:  # left and right distances exchanged
                f[..., 0:16], f[..., 32:48] = f[..., 32:48].clone(), f[..., 0:16].clone()
            mut.append((f, s))
        cand, anchor, count, cap = _kernel_like(YR.decode_ref(mut, nc, nk, 3, 64, 64 + nc, 0.5))
    else:
        cand, anchor, count, cap = _kernel_like(ref)
        if mutation == "class":
            cand[0, 0, 5] = 1.0
        elif mutation == "drop":
            count[1] -= 1
        elif mutation == "extra":
            miss = np.setdiff1d(np.arange(ref.rows.shape[1]), ref.sure[2])[0]
            anchor[2, count[2]] = int(miss)
            cand[2, count[2]] = ref.kernel_rows(2, [miss])[0]
            count[2] += 1
    rep = YR.compare_decode(ref, cand, anchor, count, cap)
    if mutation is None:
        assert rep.ok, rep.fails
        assert rep.rows > 100 and 0.0 < rep.max_err_ratio <= 1.0, rep.row()
    else:
        assert not rep.ok, f"{mutation} not detected: {rep.row()}"
        expect = {"dfl_bin_shift": "values", "swap_sides": "values", "class": "class column",
                  "drop": "candidate set", "extra": "candidate set"}[mutation]
        assert any(expect in f for f in rep.fails), rep.fails
