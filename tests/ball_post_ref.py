"""Host references for the ball pipeline's post-processing: adversarial masks for the component-box kernel, and a float64
InpaintNet with a derived per-element error bound plus the inpaint-stage decisions it implies.

The temporal ensemble and the heat-map -> box step are not restated here: the tests use oracle/tracknet.py's
`ensemble_reference_loop` (the reference's own stateful batched loop), `heatmap_to_bbox` (cv2 findContours +
boundingRect, strict `>`) and `bbox_to_xy`.  Given the device's own heat-maps, both are exact: the ensemble is a fixed
sequence of fp32 multiplies and adds, the threshold and the box are integer decisions.

InpaintNet bound.  The kernel runs nine Conv1d(k=3, 'same') layers in fp32; each output is an fp32 FMA chain
acc = b; acc = fma(w, x, acc) over n = 3 * cin taps, followed by LeakyReLU(0.01) (sigmoid on the last layer).  The
reference runs the same layers in float64 on the kernel's exact fp32 inputs and weights; its own error is ~2^-50
relative and ignored.  Let x_l be the reference input of layer l, x~_l the kernel's, |x~_l - x_l| <= e_l
elementwise (e_0 = 0: the inputs are shared).  With u = 2^-24:
    A_l      = |W_l| * (|x_l| + e_l) + |b_l|                          (bounds every partial sum; * is the conv)
    z-error  = sqrt(W_l^2 * e_l^2) + u sqrt(3 cin + 1) * A_l          (inherited + this layer's rounding)
    e_{l+1}  = z-error + 2^-23 |y_l|                                   (LeakyReLU has slope <= 1; the kernel's
                                                                        0.01f * v rounds once and 0.01f != 0.01)
    e_out    = s'(|z| - z-error) z-error + 8 u |y| + 2^-126            (s' = sigmoid's slope at the point of the
                                                                        interval nearest 0, <= 1/4; expf is within
                                                                        2 ulp, 1 + t and the division round once;
                                                                        expf overflows below z = -88.7)
Each of the n = 3 cin + 1 roundings of a chain errs by at most u times its partial sum, itself at most A_l; the
errors of different roundings, and the inherited errors of different inputs, are summed as a root sum of squares,
i.e. as errors of independent sign (the model conv_ref.py uses for the wgmma accumulators).  The worst-case forms,
gamma(n) A_l (Higham, Accuracy and Stability, Lemma 3.1) and |W_l| * e_l, grow by sqrt(n) and by the filter's L1 norm
(20-40 here) per layer: ~10^12 over nine layers, a bound of a pixel or more on every inpainted coordinate, which no
mutation of the network could exceed.  The independent-sign bound keeps a worst-case magnitude for every single
rounding (the typical one is u A / 3 or less); float32 CPU runs of the network stay under 1/13 of it at every
sequence length (tests/test_ball_post_ref_cpu.py) and the CUDA kernel under 1/4 (H100 80GB HBM3; worst at L = 1),
while each mutation listed there exceeds it more than tenfold.
Concatenated inputs (the U-Net's skip connections) carry the bounds of both parts.  The comparator reports
max |got - ref| / bound; a kernel is wrong where that exceeds 1.

Inpaint-stage decisions.  BallTracker._inpaint_stage turns the network outputs into integer pixels through threshold
decisions and truncations: blend with the mask, zero a window slot whose two coordinates are both < COOR_TH, ensemble
the L slots covering each frame, zero a frame whose two coordinates are both < COOR_TH, then
int(c * WIDTH * scale).  `inpaint_decisions` runs those steps in float64 on the reference outputs while carrying the
bound through them (the ensemble's own fp32 rounding adds gamma(L + 2) of its magnitude), and marks a frame
*borderline* when one of its decisions lies within its bound: a slot feeding it within its bound of COOR_TH, an
ensembled coordinate within its bound of COOR_TH, or an ensembled coordinate times the scale within its bound of an
integer.  Every other frame has one possible result, which the kernel's must equal exactly.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24
F32_MIN = 2.0 ** -126  # expf(-v) overflows to inf for v < -88.7: the sigmoid then returns 0 for a value < 2^-126
H_NET, W_NET = 288, 512


# ---- adversarial masks for pb_ccl_bbox (uint8 0/1, (H, W)) -------------------------------------------------------
def serpentine(rng, H=H_NET, W=W_NET):
    """One component filling the frame: full rows joined at alternating ends (union chains of ~H*W/2 links)."""
    m = np.zeros((H, W), np.uint8)
    m[0::2] = 1
    for y in range(1, H, 2):
        m[y, W - 1 if (y // 2) % 2 == 0 else 0] = 1
    return m


def spiral(rng, H=H_NET, W=W_NET):
    """A square spiral of 1-pixel walls 1 pixel apart: one component whose union chain winds to the centre."""
    m = np.zeros((H, W), np.uint8)
    y, x, k = 1, 1, 0
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    m[y, x] = 1
    while True:
        # segment lengths right W-3, down H-3, left W-3, up H-5, right W-5, down H-7, ...
        n = (W - 3 if k == 0 else W - 1 - k) if k % 2 == 0 else H - 2 - k
        if n <= 0:
            break
        dy, dx = dirs[k % 4]
        for _ in range(n):
            y, x = y + dy, x + dx
            m[y, x] = 1
        k += 1
    return m


def checkerboard(rng, H=H_NET, W=W_NET):
    """Half the pixels, one 8-connected component (every link is a diagonal)."""
    return ((np.arange(H)[:, None] + np.arange(W)[None, :]) % 2 == 0).astype(np.uint8)


def diagonal_stripes(rng, H=H_NET, W=W_NET):
    """1-pixel '\\' stripes 4 apart: components connected only through corners, many with equal boxes."""
    return ((np.arange(W)[None, :] - np.arange(H)[:, None]) % 4 == 0).astype(np.uint8)


def antidiagonal_stripes(rng, H=H_NET, W=W_NET):
    """1-pixel '/' stripes 4 apart (the up-right neighbour is the only link)."""
    return ((np.arange(W)[None, :] + np.arange(H)[:, None]) % 4 == 0).astype(np.uint8)


def wrap_left(rng, H=H_NET, W=W_NET):
    """Row y ends with a run at x = W-1, row y+1 starts with a run at x = 0: adjacent in memory (the left neighbour of
    (y+1, 0) is (y, W-1) in a flat index), not in the image.  Run lengths grow down the frame so that a join across
    the wrap would change the winner."""
    m = np.zeros((H, W), np.uint8)
    for k, y in enumerate(range(2, H - 2, 6)):
        m[y, W - 3 - k % 5:] = 1
        m[y + 1, :4 + k % 7] = 1
    m[H - 30:H - 10, 200:205] = 1  # the true winner: 5 x 20
    return m


def wrap_upright(rng, H=H_NET, W=W_NET):
    """Single rows holding a run at x = 0 and one at x = W-1: (y, W-1)'s up-right neighbour in a flat index is (y, 0)
    when the x < W-1 guard is missing (and (y+1, 0)'s up-left one is (y-1, W-1))."""
    m = np.zeros((H, W), np.uint8)
    for k, y in enumerate(range(3, H - 3, 5)):
        m[y, :3 + k % 4] = 1
        m[y, W - 2 - k % 3:] = 1
        m[y + 2, :2] = 1
    m[100:112, 250:253] = 1  # 3 x 12
    return m


def border_touching(rng, H=H_NET, W=W_NET):
    """Components on each border and in each corner; the largest box is clipped by the right border."""
    m = np.zeros((H, W), np.uint8)
    m[0:3, 0:4] = 1
    m[0:2, 100:140] = 1
    m[H - 4:H, 300:330] = 1
    m[50:90, 0:2] = 1
    m[120:200, W - 6:W] = 1
    m[H - 5:H, W - 5:W] = 1
    m[0:4, W - 4:W] = 1
    m[H - 3:H, 0:3] = 1
    return m


def v_comb(rng, H=H_NET, W=W_NET):
    """Shapes whose first raster pixel is not their box's top-left: an inverted V (apex first), a comb with its
    longest tooth in the middle, and a W."""
    m = np.zeros((H, W), np.uint8)
    for t in range(40):  # '^' with apex (20, 100)
        m[20 + t, 100 - t] = m[20 + t, 100 + t] = 1
    m[150, 200:261] = 1  # comb: teeth up, the middle one longest
    for i, x in enumerate(range(200, 261, 6)):
        m[150 - (3 + 2 * min(i, 10 - i)):150, x] = 1
    for t in range(20):  # W
        for x0 in (350, 390):
            m[200 + t, x0 + t] = m[200 + t, x0 + 40 - t] = 1
    return m


def _l_pair(m, y, x, n):
    """Two interlocking equal-box L shapes (a 'Gamma' and its 180-degree rotation): overlapping boxes, n x n each."""
    m[y:y + n, x] = 1
    m[y, x:x + n] = 1
    m[y + 4:y + 4 + n, x + n + 1] = 1
    m[y + 3 + n, x + 2:x + n + 2] = 1


def ties_same_row(rng, H=H_NET, W=W_NET):
    """k equal squares side by side on one row: equal areas, first pixels ordered by x."""
    m = np.zeros((H, W), np.uint8)
    for x in range(20, W - 20, 40):
        m[100:110, x:x + 10] = 1
    m[200:203, 50:53] = 1
    return m


def ties_same_col(rng, H=H_NET, W=W_NET):
    """k equal rectangles stacked in one column."""
    m = np.zeros((H, W), np.uint8)
    for y in range(5, H - 20, 25):
        m[y:y + 12, 300:308] = 1
    return m


def ties_interleaved(rng, H=H_NET, W=W_NET):
    """Equal-box components whose boxes overlap: interlocking L pairs at seeded places, plus an inverted V and a plain
    box of the same 40 x 21 box (apex first vs top-left first)."""
    m = np.zeros((H, W), np.uint8)
    for i in range(4):
        _l_pair(m, 10 + 60 * i + int(rng.integers(0, 5)), 20 + 110 * i + int(rng.integers(0, 5)), 30)
    return m


def ties_apex(rng, H=H_NET, W=W_NET):
    """An inverted V (first pixel at the apex) tied with a rectangle outline whose top row starts further left."""
    m = np.zeros((H, W), np.uint8)
    for t in range(21):  # box x 80..120, y 40..60
        m[40 + t, 100 - t] = m[40 + t, 100 + t] = 1
    m[40, 140:181] = m[60, 140:181] = 1
    m[40:61, 140] = m[40:61, 180] = 1
    m[200, 10:30] = 1
    return m


def island_in_hole(rng, H=H_NET, W=W_NET):
    """A ring with an island in its hole (RETR_EXTERNAL never reports the island) and smaller blobs outside."""
    m = np.zeros((H, W), np.uint8)
    m[50:150, 100:250] = 1
    m[60:140, 110:240] = 0
    m[70:130, 120:230] = 1
    m[80:120, 130:220] = 0
    m[90:110, 140:210] = 1
    m[200:230, 300:340] = 1
    return m


def lattice(rng, H=H_NET, W=W_NET):
    """Isolated pixels on a 2-pixel lattice: (H/2)(W/2) one-pixel components, all tied."""
    m = np.zeros((H, W), np.uint8)
    m[0::2, 0::2] = 1
    return m


def empty(rng, H=H_NET, W=W_NET):
    return np.zeros((H, W), np.uint8)


def full(rng, H=H_NET, W=W_NET):
    return np.ones((H, W), np.uint8)


def random_blobs(rng, H=H_NET, W=W_NET):
    """Seeded ellipses of mixed size (the heat-map shape the engine actually sees), some overlapping."""
    m = np.zeros((H, W), np.uint8)
    yy, xx = np.ogrid[:H, :W]
    for _ in range(int(rng.integers(3, 30))):
        cy, cx = rng.integers(0, H), rng.integers(0, W)
        ry, rx = rng.integers(1, 8), rng.integers(1, 10)
        m |= (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1).astype(np.uint8)
    return m


GENERATORS = {f.__name__: f for f in (
    serpentine, spiral, checkerboard, diagonal_stripes, antidiagonal_stripes, wrap_left, wrap_upright,
    border_touching, v_comb, ties_same_row, ties_same_col, ties_interleaved, ties_apex, island_in_hole, lattice,
    empty, full, random_blobs)}
# generators whose largest box must be shared by >= 2 components
TIE_GENERATORS = ("diagonal_stripes", "antidiagonal_stripes", "ties_same_row", "ties_same_col", "ties_interleaved",
                  "ties_apex", "lattice")
# generators with foreground pairs that a flat-index neighbour test would join across the row wrap
WRAP_GENERATORS = ("wrap_left", "wrap_upright", "serpentine", "border_touching")


def make_mask(name: str, seed: int = 0, H=H_NET, W=W_NET) -> np.ndarray:
    return GENERATORS[name](np.random.default_rng(seed), H, W)


def wrap_pairs(m: np.ndarray) -> int:
    """Foreground pairs that are neighbours in a flat index but not in the image: (y, W-1)-(y+1, 0) (left),
    (y, W-1)-(y, 0) (up-right of (y, W-1) without the x guard) and (y-1, W-1)-(y+1, 0) (up-left of (y+1, 0))."""
    left = int((m[:-1, -1] & m[1:, 0]).sum())
    upright = int((m[:, -1] & m[:, 0]).sum())
    upleft = int((m[:-2, -1] & m[2:, 0]).sum())
    return left + upright + upleft


def component_stats(m: np.ndarray):
    """(foreground pixels, 8-connected components, components sharing the largest box area)."""
    import cv2

    n, lab, st, _ = cv2.connectedComponentsWithStats(m, connectivity=8)
    if n <= 1:
        return int(m.sum()), 0, 0
    areas = st[1:, cv2.CC_STAT_WIDTH].astype(np.int64) * st[1:, cv2.CC_STAT_HEIGHT]
    return int(m.sum()), n - 1, int((areas == areas.max()).sum())


# ---- InpaintNet: float64 reference with an elementwise error bound ---------------------------------------------------
INPAINT_LAYERS = ["down_1.conv", "down_2.conv", "down_3.conv", "buttleneck.conv_1.conv", "buttleneck.conv_2.conv",
                  "up_1.conv", "up_2.conv", "up_3.conv", "predictor"]


def gamma(n: int) -> float:
    return n * U32 / (1 - n * U32)


def inpaint_forward_f64(sd: dict, coor: torch.Tensor, mask: torch.Tensor, device=None):
    """InpaintNet (oracle/inpaint.py's InpaintNetOracle) in float64 on the fp32 values given, with the bound above.
    coor (N, L, 2), mask (N, L, 1) -> (ref (N, L, 2) float64, bound (N, L, 2) float64)."""
    dev = device or coor.device
    W = {k: sd[f"{k}.weight"].to(dev, torch.float64) for k in INPAINT_LAYERS}
    Bi = {k: sd[f"{k}.bias"].to(dev, torch.float64) for k in INPAINT_LAYERS}
    x = torch.cat([coor.to(dev, torch.float64), mask.to(dev, torch.float64)], 2).permute(0, 2, 1).contiguous()
    e = torch.zeros_like(x)

    def layer(k, xs, es, last=False):
        xin, ein = torch.cat(xs, 1), torch.cat(es, 1)
        w, b = W[k], Bi[k]
        z = F.conv1d(xin, w, b, padding=1)
        A = F.conv1d(xin.abs() + ein, w.abs(), b.abs(), padding=1)
        ez = F.conv1d(ein * ein, w * w, None, padding=1).sqrt() + U32 * math.sqrt(3 * w.shape[1] + 1) * A
        if last:
            y = torch.sigmoid(z)
            a = (z.abs() - ez).clamp(min=0)  # the steepest point within the bound
            return y, torch.sigmoid(a) * torch.sigmoid(-a) * ez + 8 * U32 * y.abs() + F32_MIN
        y = F.leaky_relu(z, 0.01)
        return y, ez + 2.0 ** -23 * y.abs()

    x1, e1 = layer("down_1.conv", [x], [e])
    x2, e2 = layer("down_2.conv", [x1], [e1])
    x3, e3 = layer("down_3.conv", [x2], [e2])
    b1, eb1 = layer("buttleneck.conv_1.conv", [x3], [e3])
    b2, eb2 = layer("buttleneck.conv_2.conv", [b1], [eb1])
    u1, eu1 = layer("up_1.conv", [b2, x3], [eb2, e3])
    u2, eu2 = layer("up_2.conv", [u1, x2], [eu1, e2])
    u3, eu3 = layer("up_3.conv", [u2, x1], [eu2, e1])
    y, ey = layer("predictor", [u3], [eu3], last=True)
    return y.permute(0, 2, 1).contiguous(), ey.permute(0, 2, 1).contiguous()


def bound_ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |got - ref| / bound over all elements (> 1: outside the bound)."""
    g = got.to(ref.device, torch.float64)
    return float(((g - ref).abs() / bound).max())


def inpaint_forward_f32(sd: dict, coor, mask, slope=0.01, pad_shift=0, drop_bias=None, transpose_out=False):
    """float32 CPU InpaintNet with optional mutations (for checking that the comparators reject them): LeakyReLU
    `slope`, the 'same' padding shifted by `pad_shift` taps, layer `drop_bias`'s bias left out, and the (L, 2) output
    written channel-major (a (2, L) buffer read as (L, 2))."""
    W = {k: sd[f"{k}.weight"].float() for k in INPAINT_LAYERS}
    Bi = {k: (torch.zeros_like(sd[f"{k}.bias"].float()) if k == drop_bias else sd[f"{k}.bias"].float())
          for k in INPAINT_LAYERS}
    x = torch.cat([coor.float(), mask.float()], 2).permute(0, 2, 1)

    def conv(k, t):
        L = t.shape[-1]
        y = F.conv1d(F.pad(t, (1 + pad_shift, 1 - pad_shift)), W[k], Bi[k])
        return y[..., :L]

    act = lambda t: F.leaky_relu(t, slope)
    x1 = act(conv("down_1.conv", x))
    x2 = act(conv("down_2.conv", x1))
    x3 = act(conv("down_3.conv", x2))
    b = act(conv("buttleneck.conv_2.conv", act(conv("buttleneck.conv_1.conv", x3))))
    u = act(conv("up_1.conv", torch.cat([b, x3], 1)))
    u = act(conv("up_2.conv", torch.cat([u, x2], 1)))
    u = act(conv("up_3.conv", torch.cat([u, x1], 1)))
    y = torch.sigmoid(conv("predictor", u))  # (N, 2, L)
    if transpose_out:
        return y.contiguous().reshape(y.shape[0], -1, 2)
    return y.permute(0, 2, 1).contiguous()


# ---- inpaint-stage decisions ------------------------------------------------------------------------------------------
def coor_th(net_hw=(H_NET, W_NET)) -> float:
    return 50.0 / math.sqrt(net_hw[0] ** 2 + net_hw[1] ** 2)


def inpaint_decisions(ref, bound, coor, mask, T: int, video_wh, host_stage, net_hw=(H_NET, W_NET)):
    """The post-network steps of BallTracker._inpaint_stage in float64 with the bound carried through.
    ref / bound: (S, L, 2) float64 network outputs and their bound; coor (S, L, 2), mask (S, L, 1): the fp32 inputs.
    A frame none of whose L slots is masked does not depend on the network (the blend passes the input through): its
    expected result is `host_stage`'s, the host stage run on the reference outputs, and it is never borderline (an
    unmasked visible frame's coordinate times the scale is its input pixel, an integer up to fp32 rounding, so the
    float64 value cannot decide the truncation).
    Returns (expected {frame: (x, y, vis)}, borderline frame set)."""
    ref = ref.detach().cpu().double().numpy()
    bound = bound.detach().cpu().double().numpy()
    c = coor.detach().cpu().double().numpy()
    m = mask.detach().cpu().double().numpy()
    S, L, _ = ref.shape
    th = coor_th(net_hw)
    th32 = float(np.float32(th))
    tol_th = abs(th - th32) + 2 * U32 * th  # the device compares fp32 values with COOR_TH rounded to fp32
    o = ref * m + c * (1 - m)  # the blend is exact in fp32 for a 0/1 mask
    e = bound * m
    near = (np.abs(o - th) <= e + tol_th).any(-1)  # (S, L): a slot whose zeroing is undecided
    zero = (o < th).all(-1)
    o[zero] = 0.0
    e[zero] = 0.0
    wts = np.ones(L)
    for i in range(math.ceil(L / 2)):
        wts[i] = wts[L - i - 1] = i + 1
    wts = wts / wts.sum()
    W_img, H_img = video_wh
    scale = (W_img / net_hw[1], H_img / net_hw[0])
    exp, border = {}, set()
    for n in range(T):
        ks = [k for k in range(L) if 0 <= n - (L - 1) + k < S]
        slots = [(n - (L - 1) + k, L - 1 - k) for k in ks]
        if not any(m[s, j, 0] for s, j in slots):
            exp[n] = tuple(host_stage[n])
            continue
        if n < S and n >= L - 1:
            coef = np.array([wts[k] for k in ks])
        else:
            coef = np.full(len(ks), 1.0 / ((n + 1) if n < S else (L - (n - (S - 1)))))
        vals = np.array([o[s, j] for s, j in slots])
        errs = np.array([e[s, j] for s, j in slots])
        ens = (coef[:, None] * vals).sum(0)
        err = (coef[:, None] * errs).sum(0) + gamma(L + 2) * (coef[:, None] * np.abs(vals)).sum(0)
        bl = any(near[s, j] for s, j in slots)
        bl |= bool((np.abs(ens - th) <= err + tol_th).any())
        if (ens < th).all():
            xy = (0, 0)
        else:
            xy = []
            for d, (wh, sc) in enumerate(((net_hw[1], scale[0]), (net_hw[0], scale[1]))):
                v = ens[d] * wh * sc
                r = err[d] * wh * sc + 4 * U32 * abs(v) + 1e-9
                if abs(v - round(v)) <= r:
                    bl = True
                xy.append(int(v))
            xy = tuple(xy)
        if bl:
            border.add(n)
        exp[n] = (xy[0], xy[1], 0 if xy == (0, 0) else 1)
    return exp, border


def compare_decisions(got: dict, exp: dict, border: set):
    """Frames (outside `border`) where `got` differs from `exp`."""
    return [n for n in exp if n not in border and tuple(got[n]) != exp[n]]


class RecordingNet:
    """Wraps an InpaintNet callable and keeps the (coor, mask, out) of its last call on the host."""

    def __init__(self, net):
        self.net = net
        self.calls = []

    def __call__(self, coor, mask):
        out = self.net(coor, mask)
        self.calls.append((coor.detach().cpu().clone(), mask.detach().cpu().clone(), out.detach().cpu().clone()))
        return out


def stage_decisions(sd: dict, net, xs, ys, vs, seq_len: int, video_wh, device=None):
    """Run BallTracker._inpaint_stage with `net` as the InpaintNet, then the float64 reference on the exact inputs it
    was given.  Returns (got, expected, borderline frames, worst |err| / bound of the network outputs)."""
    rec = RecordingNet(net)
    got = stage_tracker(rec, seq_len, video_wh)._inpaint_stage(xs, ys, vs)
    (c, m, out), = rec.calls
    ref, bound = inpaint_forward_f64(sd, c.to(device) if device else c, m.to(device) if device else m)
    ref_f32 = ref.float().cpu()
    host = stage_tracker(lambda cc, mm: ref_f32, seq_len, video_wh)._inpaint_stage(xs, ys, vs)
    exp, border = inpaint_decisions(ref, bound, c, m, len(xs), video_wh, host)
    return got, exp, border, bound_ratio(out, ref, bound)


def stage_tracker(net, seq_len: int, video_wh):
    """A BallTracker carrying only what _inpaint_stage reads (the InpaintNet callable, its sequence length and the
    video size), so that the host stage can be run on any network, on the CPU."""
    from padel_analytics_b200.trackers import BallTracker
    from padel_analytics_b200.trackers import sv_compat as sv

    bt = BallTracker.__new__(BallTracker)
    bt.DELTA_T = 1 / math.sqrt(BallTracker.HEIGHT ** 2 + BallTracker.WIDTH ** 2)
    bt.COOR_TH = bt.DELTA_T * 50
    bt.inpaintnet = net
    bt.inpaintnet_seq_len = seq_len
    bt.video_info = sv.VideoInfo(width=video_wh[0], height=video_wh[1], fps=30.0, total_frames=None)
    return bt


def synthetic_trajectory(seed: int, T: int, video_wh, gaps):
    """A bouncing ball's (x, y, vis) pixel lists with visibility gaps [(start, end), ...] (x = y = 0 there)."""
    rng = np.random.default_rng(seed)
    W_img, H_img = video_wh
    xs, ys, vs = [], [], []
    x, y = float(rng.uniform(0.2, 0.8) * W_img), float(rng.uniform(0.3, 0.6) * H_img)
    vx, vy = float(rng.uniform(-12, 12)), float(rng.uniform(-20, -5))
    for n in range(T):
        x, y, vy = x + vx, y + vy, vy + 1.2
        if y > 0.95 * H_img:
            y, vy = 0.95 * H_img, -abs(vy) * 0.8
        if not 0.1 * W_img < x < 0.9 * W_img:
            vx = -vx
        xs.append(int(x)), ys.append(int(y)), vs.append(1)
    for a, b in gaps:
        for n in range(a, min(b, T)):
            xs[n] = ys[n] = vs[n] = 0
    return xs, ys, vs
