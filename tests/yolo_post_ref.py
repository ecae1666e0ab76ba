"""Host restatement of the YOLO head decode and NMS (csrc/yolo_post.cu) and the comparator of the decode kernel.

Decode (float64).  For every anchor of the head maps (the pb_yolo_level layout: per level a float32 NHWC map
(B, h, w, fC) with the 64 DFL logits at [0, 64), the class logits at [cls_off, +nc) and the keypoints at [kpt_off, +nk)):
  - best class: ultralytics takes `cls.max(1)` over the float32 *sigmoid* scores, so the first class whose sigmoid
    equals the maximum wins.  Above a logit of ~16.7 every float32 sigmoid is exactly 1.0, so saturated logits tie.
  - conf = sigmoid(best logit); a candidate has conf > `conf` and, with a class filter, its best class in the filter;
  - DFL: per side the softmax expectation over the 16 bins; dist2bbox (xywh) * stride, then xywh -> xyxy;
  - keypoints: (v * 2 + (anchor - 0.5)) * stride, visibility sigmoid(v) when kdim == 3.

Error bound of the kernel's float32 op sequence, first order in u = 2^-24 (the float32 unit roundoff).  Each of
+ - * / rounds once (|rel err| <= u; a fused multiply-add rounds less); CUDA's expf is within 2 ulp (<= 4u relative);
strides are powers of two, so scaling by them and halving are exact.  Per DFL side, R = max - min of its 16 logits:
  - e_j = expf(q_j - max): the subtraction rounds by u|q_j - max| <= uR, expf adds 4u: |rel| <= eta = (4 + R)u;
  - den = sum of 16 positive e_j (15 additions): |rel| <= eta + 15u; num = sum of e_j * j: |rel| <= eta + 16u;
  - dist = num / den: |rel| <= 2 eta + 32u, so E_dist = dist (2 eta + 32u).
  - x1 = a - d0, x2 = a + d2 (a = g + 0.5, exact): E = E_dist + u|x|; S = x1 + x2 and W = x2 - x1:
    E = E_x1 + E_x2 + u|S| (resp. u|W|); cx = S / 2 * stride, hw = W * stride / 2 scale exactly; the outputs
    cx -+ hw: E = E_cx + E_hw + u|out|.
  - conf and visibility, s = 1 / (1 + expf(-x)): expf 4u relative, 1 + e adds u, the division u: E = 6u s.
  - keypoint x, y: v * 2 and a - 0.5 are exact, one rounding of the sum: E = u|out|.
The float64 reference is exact to ~1e-16 relative, far inside these bounds; the comparison allows 2^-10 of slack
for the dropped second-order terms.

Borderline anchors are excluded from the candidate set check and counted: those whose float64 conf is within
BORDER_ULPS float32 ulps of `conf` (the kernel's float conf may fall on either side), and those where a class with a
different logit has a float64 sigmoid within BORDER_ULPS ulps of the best one's, unless both logits are >= 17 (where
every float32 sigmoid is exactly 1.0): there two float32 sigmoid implementations may order the classes differently.

NMS (exact).  Candidates sorted by (conf desc, anchor asc) -- torchvision sorts the scores with a stable sort on the
CPU, and ultralytics hands it the candidates in anchor order -- boxes offset by cls * 7680 in float32, then torchvision's
greedy NMS in its float32 op order: areas (x2 - x1) * (y2 - y1), max / min, max(0, .), inter = w * h,
ovr = inter / (iarea + area_j - inter); a box is suppressed when float64(ovr) > iou (torchvision's threshold is a
double).  At most max_det boxes are emitted.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import torch

U = 2.0 ** -24
MAX_WH = 7680.0
BORDER_ULPS = 8
SATURATED_LOGIT = 17.0  # exp(-17) < 2^-24: 1 + exp(-x) rounds to 1 in float32, even with expf 2 ulp off
SLACK = 1.0 + 2.0 ** -10


def ulp32(x: torch.Tensor) -> torch.Tensor:
    """Spacing of float32 numbers at |x|, in float64."""
    e = torch.frexp(x.abs().to(torch.float64).clamp_min(2.0 ** -140))[1] - 1
    return torch.exp2((e.clamp_min(-126) - 23).to(torch.float64))


# ---- decode ----------------------------------------------------------------------------------------------------
@dataclass
class DecodeRef:
    sure: list    # per image: sorted int64 array of the anchors that are candidates
    border: list  # per image: sorted int64 array of the borderline anchors (candidates or not)
    rows: torch.Tensor   # (B, A, 6 + nk) float64: x1, y1, x2, y2, conf, cls, keypoints of every anchor
    bound: torch.Tensor  # (B, A, 6 + nk) float64 error bound of the kernel's float32 value (cls column: 0)

    def kernel_rows(self, b: int, anchors) -> torch.Tensor:
        """float32 rows as the decode kernel writes them (the reference rounded), for building expected buffers."""
        return self.rows[b, torch.as_tensor(anchors, dtype=torch.long)].to(torch.float32)


def decode_ref(levels, nc: int, nk: int, kdim: int, cls_off: int, kpt_off: int, conf: float, classes=None) -> DecodeRef:
    """levels: [(feat float32 (B, h, w, fC), stride)], anchors numbered level by level, row-major within a level."""
    B = levels[0][0].shape[0]
    f = torch.cat([x.reshape(B, -1, x.shape[-1]) for x, _ in levels], 1)
    gx, gy, st = [], [], []
    for x, s in levels:
        h, w = x.shape[1], x.shape[2]
        assert s > 0 and s & (s - 1) == 0, "the bound assumes power-of-two strides"
        la = torch.arange(h * w)
        gx.append(la % w), gy.append(la // w), st.append(torch.full((h * w,), float(s)))
    gx = torch.cat(gx).to(torch.float64)
    gy = torch.cat(gy).to(torch.float64)
    st = torch.cat(st).to(torch.float64)
    conf = float(np.float32(conf))  # the kernel's argument is a float

    logits = f[..., cls_off:cls_off + nc]
    best = torch.sigmoid(logits).max(-1).indices  # float32 sigmoid, first maximum (ultralytics cls.max(1))
    lbest = logits.gather(-1, best[..., None])
    s64 = torch.sigmoid(logits.to(torch.float64))
    score = s64.gather(-1, best[..., None])[..., 0]
    near = (s64 - score[..., None]).abs() <= BORDER_ULPS * ulp32(score)[..., None]
    clash = near & (logits != lbest) & (torch.minimum(logits, lbest) < SATURATED_LOGIT)
    border = clash.any(-1) | ((score - conf).abs() <= BORDER_ULPS * ulp32(torch.tensor(conf)))
    keep = score > conf
    if classes is not None:
        allowed = torch.zeros(max(nc, 1), dtype=torch.bool)
        for c in classes:
            if c < nc:
                allowed[c] = True
        keep &= allowed[best]
        border &= allowed[best] | clash.any(-1)

    q = f[..., :64].to(torch.float64).reshape(B, -1, 4, 16)
    dist = (torch.softmax(q, -1) * torch.arange(16, dtype=torch.float64)).sum(-1)
    R = q.amax(-1) - q.amin(-1)
    e_dist = dist * (2 * (4 + R) * U + 32 * U) + 1e-30
    ax, ay = gx + 0.5, gy + 0.5
    x1, y1, x2, y2 = ax - dist[..., 0], ay - dist[..., 1], ax + dist[..., 2], ay + dist[..., 3]
    e_x1, e_y1 = e_dist[..., 0] + U * x1.abs(), e_dist[..., 1] + U * y1.abs()
    e_x2, e_y2 = e_dist[..., 2] + U * x2.abs(), e_dist[..., 3] + U * y2.abs()
    cx, cy = (x1 + x2) / 2 * st, (y1 + y2) / 2 * st
    hw, hh = (x2 - x1) * st / 2, (y2 - y1) * st / 2
    e_cx = (e_x1 + e_x2 + U * (x1 + x2).abs()) * st / 2
    e_cy = (e_y1 + e_y2 + U * (y1 + y2).abs()) * st / 2
    e_hw = (e_x1 + e_x2 + U * (x2 - x1).abs()) * st / 2
    e_hh = (e_y1 + e_y2 + U * (y2 - y1).abs()) * st / 2
    box = torch.stack((cx - hw, cy - hh, cx + hw, cy + hh), -1)
    e_box = torch.stack((e_cx + e_hw, e_cy + e_hh, e_cx + e_hw, e_cy + e_hh), -1) + U * box.abs()

    cols = [box, score[..., None], best[..., None].to(torch.float64)]
    errs = [e_box, 6 * U * score[..., None], torch.zeros_like(score)[..., None]]
    K = nk // kdim if kdim else 0
    if K:
        kp = f[..., kpt_off:kpt_off + nk].to(torch.float64).reshape(B, -1, K, kdim)
        kx = (kp[..., 0] * 2 + gx[:, None]) * st[:, None]
        ky = (kp[..., 1] * 2 + gy[:, None]) * st[:, None]
        parts, perr = [kx, ky], [U * kx.abs(), U * ky.abs()]
        if kdim == 3:
            vis = torch.sigmoid(kp[..., 2])
            parts.append(vis), perr.append(6 * U * vis)
        cols.append(torch.stack(parts, -1).reshape(B, -1, nk))
        errs.append(torch.stack(perr, -1).reshape(B, -1, nk))
    rows = torch.cat(cols, -1)
    bound = torch.cat(errs, -1)
    sure = [torch.nonzero(keep[b] & ~border[b])[:, 0].numpy() for b in range(B)]
    bord = [torch.nonzero(border[b])[:, 0].numpy() for b in range(B)]
    return DecodeRef(sure, bord, rows, bound)


@dataclass
class DecodeReport:
    images: int = 0
    rows: int = 0          # candidate rows the kernel wrote (sum of min(cand_count, cap))
    counted: int = 0       # sum of cand_count
    border: int = 0        # borderline anchors excluded from the checks
    max_err_ratio: float = 0.0  # worst |got - ref| / bound over the box, conf and keypoint values
    worst: str = ""
    fails: list = field(default_factory=list)

    @property
    def ok(self) -> bool:
        return not self.fails

    def row(self) -> str:
        return (f"rows {self.rows:6d}  counted {self.counted:6d}  border {self.border:3d}  "
                f"err/bound {self.max_err_ratio:.3f} ({self.worst})")


def compare_decode(ref: DecodeRef, cand: torch.Tensor, anchor: torch.Tensor, count: torch.Tensor, cap: int,
                   rep: DecodeReport | None = None) -> DecodeReport:
    """cand (B, cap, rowlen) float32, anchor (B, cap) int32, count (B,) int32: the decode kernel's outputs (host)."""
    rep = rep or DecodeReport()
    B = cand.shape[0]
    for b in range(B):
        rep.images += 1
        n = int(count[b])
        m = min(n, cap)
        rep.rows += m
        rep.counted += n
        sure, border = ref.sure[b], ref.border[b]
        rep.border += len(border)
        got = anchor[b, :m].to(torch.int64).numpy()
        tag = f"image {b}"
        if len(np.unique(got)) != m:
            rep.fails.append(f"{tag}: an anchor is written twice")
            continue
        if not (len(sure) <= n <= len(sure) + len(border)):
            rep.fails.append(f"{tag}: cand_count {n}, the reference has {len(sure)} candidates "
                             f"(+{len(border)} borderline)")
        A = ref.rows.shape[1]
        if ((got < 0) | (got >= A)).any():
            rep.fails.append(f"{tag}: anchor out of range")
            continue
        got_firm = np.setdiff1d(got, border)
        extra = np.setdiff1d(got_firm, sure)
        if len(extra):
            rep.fails.append(f"{tag}: candidate set: {len(extra)} anchors the reference rejects, first {int(extra[0])}")
        if n <= cap:
            missing = np.setdiff1d(sure, got)
            if len(missing):
                rep.fails.append(f"{tag}: candidate set: {len(missing)} reference candidates missing, "
                                 f"first {int(missing[0])}")
        firm = ~np.isin(got, border)
        if not firm.any():
            continue
        idx = torch.from_numpy(np.nonzero(firm)[0])
        a = torch.from_numpy(got[firm])
        g = cand[b, idx].to(torch.float64)
        r = ref.rows[b, a]
        e = ref.bound[b, a]
        bad_cls = g[:, 5] != r[:, 5]
        if bad_cls.any():
            i = int(bad_cls.nonzero()[0])
            rep.fails.append(f"{tag}: class column: {int(bad_cls.sum())} rows differ, anchor {int(a[i])} got "
                             f"{g[i, 5].item():g} expected {r[i, 5].item():g}")
        if not torch.isfinite(g).all():
            rep.fails.append(f"{tag}: non-finite values")
            continue
        vals = torch.ones(g.shape[1], dtype=torch.bool)
        vals[5] = False
        ratio = ((g - r).abs() / (e * SLACK))[:, vals]
        mx = float(ratio.max())
        if mx > rep.max_err_ratio:
            i, c = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
            col = int(np.nonzero(vals.numpy())[0][c])
            rep.max_err_ratio = mx
            rep.worst = f"image {b} anchor {int(a[i])} col {col}"
        if mx > 1.0:
            i, c = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
            col = int(np.nonzero(vals.numpy())[0][c])
            rep.fails.append(f"{tag}: values: {int((ratio > 1).sum())} outside the bound, worst anchor {int(a[i])} "
                             f"col {col}: got {g[i, col].item()!r} ref {r[i, col].item()!r} "
                             f"bound {e[i, col].item():.3g}")
    return rep


# ---- NMS ---------------------------------------------------------------------------------------------------------
def greedy_nms(boxes: np.ndarray, iou: float, max_det: int | None = None) -> np.ndarray:
    """torchvision.ops.nms's greedy pass over float32 boxes (n, 4) already in score order; returns kept positions."""
    b = np.ascontiguousarray(boxes, dtype=np.float32)
    n = b.shape[0]
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    areas = (x2 - x1) * (y2 - y1)
    supp = np.zeros(n, dtype=bool)
    keep = []
    zero = np.float32(0)
    with np.errstate(invalid="ignore", divide="ignore"):
        for i in range(n):
            if supp[i]:
                continue
            if max_det is not None and len(keep) >= max_det:
                break
            keep.append(i)
            j = slice(i + 1, n)
            w = np.maximum(zero, np.minimum(x2[i], x2[j]) - np.maximum(x1[i], x1[j]))
            h = np.maximum(zero, np.minimum(y2[i], y2[j]) - np.maximum(y1[i], y1[j]))
            inter = w * h
            ovr = inter / (areas[i] + areas[j] - inter)
            supp[j] |= ovr.astype(np.float64) > float(iou)
    return np.asarray(keep, dtype=np.int64)


def score_order(scores: np.ndarray, tiebreak: np.ndarray) -> np.ndarray:
    """Indices by (score desc, tiebreak asc)."""
    return np.lexsort((np.asarray(tiebreak), -np.asarray(scores, dtype=np.float32)))


def nms_ref(rows: np.ndarray, anchors: np.ndarray, iou: float, max_det: int) -> np.ndarray:
    """rows float32 (n, 6 + nk) = x1, y1, x2, y2, conf, cls, ...; returns the indices of the emitted rows, in order."""
    rows = np.asarray(rows, dtype=np.float32)
    order = score_order(rows[:, 4], anchors)
    r = rows[order]
    off = r[:, 5] * np.float32(MAX_WH)
    return order[greedy_nms(r[:, :4] + off[:, None], iou, max_det)]


# ---- hand-built NMS inputs ---------------------------------------------------------------------------------------
def random_boxes(rng, n: int, extent: float = 1280.0):
    """Clustered float32 xyxy boxes (overlaps at every IoU) and scores with exact ties (k/32, 1.0 included)."""
    k = max(1, n // 8)
    cen = rng.uniform(0, extent, (k, 2))
    c = cen[rng.integers(0, k, n)] + rng.normal(0, 6, (n, 2))
    wh = rng.uniform(4, 120, (n, 2))
    b = np.concatenate([c - wh / 2, c + wh / 2], 1).astype(np.float32)
    s = rng.uniform(0.01, 1.0, n).astype(np.float32)
    tie = rng.random(n) < 0.4
    s[tie] = (rng.integers(1, 33, int(tie.sum())) / 32).astype(np.float32)
    return b, s


def random_candidates(rng, n: int, rowlen: int, nclass: int = 3):
    """Candidate rows (n, rowlen) float32 as the decode kernel writes them, and distinct anchors."""
    b, s = random_boxes(rng, n)
    rows = np.empty((n, rowlen), np.float32)
    rows[:, :4], rows[:, 4] = b, s
    rows[:, 5] = rng.integers(0, nclass, n)
    rows[:, 6:] = rng.normal(0, 100, (n, rowlen - 6))
    return rows, rng.choice(1 << 20, n, replace=False).astype(np.int32)


# IoU exactly float32(t): [0,0,D,1] against [0,0,k,1] has inter k, union D, and k / D rounds to float32(t)
IOU_FRACTIONS = {0.3: (3, 10), 0.45: (9, 20), 0.5: (5, 10), 0.6: (6, 10), 0.7: (7, 10), 0.8: (8, 10)}
# torchvision compares float64(ovr) > t: float32(t) rounds above t for 0.3, 0.6 and 0.8
SUPPRESSED_AT_FLOAT_T = {0.3: True, 0.45: False, 0.5: False, 0.6: True, 0.7: False, 0.8: True}


def iou_pair_rows(t: float) -> np.ndarray:
    """Two pairs whose IoU is exactly float32(t): one in class 0 (conf 0.9 / 0.8), one shifted in class 1 (conf 1.0
    twice, so the anchors decide the order)."""
    k, D = IOU_FRACTIONS[t]
    return np.array([[0, 0, D, 1, 0.9, 0], [0, 0, k, 1, 0.8, 0],
                     [100, 0, 100 + k, 1, 1.0, 1], [100, 0, 100 + D, 1, 1.0, 1]], np.float32)


def edge_case_rows():
    """[(name, rows float32 (n, 6), anchors, iou, kept indices)]: hand-built candidate sets of the NMS edges."""
    cases = []
    # zero-area boxes: 0 / 0 = NaN IoU suppresses nothing
    r = np.array([[5, 5, 5, 9, 0.9, 0], [5, 5, 5, 9, 0.8, 0], [3, 3, 3, 3, 0.7, 0], [3, 3, 3, 3, 0.6, 0]], np.float32)
    cases.append(("zero_area", r, np.array([0, 1, 2, 3]), 0.5, [0, 1, 2, 3]))
    # identical boxes in different classes survive; the same class suppresses
    r = np.array([[10, 10, 50, 50, 0.9, 0], [10, 10, 50, 50, 0.8, 1], [10, 10, 50, 50, 0.7, 2],
                  [10, 10, 50, 50, 0.6, 0]], np.float32)
    cases.append(("classes", r, np.array([0, 1, 2, 3]), 0.7, [0, 1, 2]))
    # beyond 7680 the offset boxes of neighbouring classes overlap: class 1 near 0 meets class 0 near 7680, and
    # class 2 at -360 lands on class 0 at 15000
    r = np.array([[7700, 7700, 7800, 7800, 0.9, 0], [30, 30, 130, 130, 0.8, 1], [15000, 15000, 15100, 15100, 0.7, 0],
                  [-360, -360, -260, -260, 0.6, 2]], np.float32)
    cases.append(("beyond_7680", r, np.array([0, 1, 2, 3]), 0.5, [0, 2]))
    # conf ties, 1.0 included: the lower anchor goes first
    r = np.array([[0, 0, 10, 10, 1.0, 0], [0, 0, 10, 10, 1.0, 0], [100, 0, 110, 10, 0.5, 0],
                  [100, 0, 110, 10, 0.5, 0], [100, 0, 110, 10, 0.5, 0]], np.float32)
    cases.append(("conf_ties", r, np.array([9, 4, 7, 2, 5]), 0.5, [1, 3]))
    # the union rounds area_j to float32 before adding iarea: a fused iarea + w_j * h_j moves these IoUs across t
    # (first pair: torchvision's IoU is just above t and suppresses, the fused one is below; second pair: the reverse)
    r = np.array([[394.98663330078125, 221.5212860107422, 515.4710693359375, 414.0947570800781, 0.9, 0],
                  [416.2494201660156, 221.5212860107422, 536.7316284179688, 414.0950927734375, 0.8, 0],
                  [245.85833740234375, 505.31024169921875, 395.59918212890625, 590.181884765625, 0.7, 0],
                  [272.2824401855469, 505.31024169921875, 422.02349853515625, 590.1828002929688, 0.6, 0]], np.float32)
    cases.append(("union_rounding_0.7", r, np.array([0, 1, 2, 3]), 0.7, [0, 2, 3]))
    r = np.array([[25.77671241760254, 268.219482421875, 155.44711303710938, 317.6468505859375, 0.9, 0],
                  [74.96137237548828, 268.219482421875, 204.6324920654297, 317.64630126953125, 0.8, 0],
                  [535.0726928710938, 538.7486572265625, 687.65185546875, 732.108154296875, 0.7, 0],
                  [592.9483032226562, 538.7486572265625, 745.5243530273438, 732.1072998046875, 0.6, 0]], np.float32)
    cases.append(("union_rounding_0.45", r, np.array([0, 1, 2, 3]), 0.45, [0, 2, 3]))
    return cases
