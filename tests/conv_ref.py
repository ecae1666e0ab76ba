"""Float64 reference and per-element comparator for one conv op (and the exact references of the pooling ops).

A conv op is checked on exactly the fp16 operands it read -- its input slice, its packed weights
[taps][cout_pad][cin] (stem: [3 filter rows][cout_pad][16], unpacked here) and its fp32 bias -- so the reference does
not depend on BN folding or weight packing.  On the GPU the operands are zero-copy views of the op's own buffers built
from the raw pointers of its descriptor (`conv_views`); the CPU self-test builds the same dictionaries from tensors.

Reference: y = act(conv(x, w) + b [+ res]) [+ res] in float64.  The products of two fp16 values are exact in float64
and a float64 sum of a few thousand of them is exact to ~2^-40 of A, so the reference is the exact result for all
purposes here.  A = conv(|x|, |w|) + |b| + |res| bounds every partial sum the kernel forms.

fp16 outputs: every element must satisfy |got - ref| <= ulp16(ref) + E, with E = 2^-18 * A.
  - The final fp32 -> fp16 rounding (round to nearest) costs at most half an ulp16 of the fp32 value; the other half
    ulp16 absorbs the few-ulp32 errors of the fast SiLU / sigmoid (ex2.approx, rcp.approx: ~2^-21 relative).
  - E bounds the fp32 accumulation error.  The kernel adds K / 16 wgmma k-steps (16 exact products each) into an fp32
    accumulator; each addition rounds or truncates by at most 2^-23 of the running partial sum.  With products of
    mixed sign the partial sums grow like sqrt(k) while A grows like k, so the summed error is about
    2^-23 * (2/3) * sqrt(K / 16) * A: 2^-19.2 * A at K = 9 * 768 (TrackNet's widest layer), and 2^-18 * A holds up
    to K ~ 37000.  SiLU (slope <= 1.1), ReLU (1) and sigmoid (1/4) do not enlarge it by more than the margin.
  - Against the old test tolerance 2e-3 + 2e-3 |y|: ulp16(y) <= 2^-10 |y| < 2e-3 |y|, and E < 2e-3 while A < 2^9
    (an activation sum of a few hundred); an op where any element's bound is not below the old one fails.
fp32 outputs: |got - ref| <= 4 ulp32(ref) + E (no output rounding; the 4 ulps cover expf / fdividef).

Rounding statistics (fp16 outputs): the fraction of elements that differ from the correctly rounded reference
(`mismatch`) and the mean error in ulp16 toward / away from zero (`bias`, signed by the reference) must stay below
MAX_MISMATCH / MAX_BIAS.  A kernel that rounds to nearest mismatches only where its fp32 value and the reference
straddle a rounding midpoint; a store that truncates mismatches on about half the elements and is biased by -1/2 ulp.

Untouched elements: every element of `out` / `out2` outside the op's channel slice is bit-identical to its value
before the op.  Second outputs: PB_OUT2_UP2 / PB_OUT2_POOL2 are exactly the 2x2 replication / 2x2 max of the primary.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

from padel_analytics_b200 import _lib as L

ACC_REL = 2.0 ** -18  # E = ACC_REL * A
F32_ULPS = 4
# Rounding statistics of a round-to-nearest kernel.  On an H100 80GB HBM3 (400 W power limit) the worst op of the
# replayed programs and of the plan sweep showed a mismatch rate of 0.0125 and a bias of -0.0147 ulp (both the
# 768 -> 64 layer with 12 streamed channel blocks); the bounds keep a margin of 3x.  A truncating store sits near 0.5
# / -0.5 (0.25 on ReLU outputs, half of which are exact zeros).  Below MIN_STAT_ELEMENTS elements the statistics are
# not judged: the bias of n round-to-nearest errors has a spread of 0.29 / sqrt(n) ulp.
MAX_MISMATCH = 0.04
MAX_BIAS = 0.05
MIN_STAT_ELEMENTS = 2000


# ---- zero-copy views of device buffers --------------------------------------------------------------------------
class _Cai:
    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"data": (int(ptr), False), "shape": tuple(int(s) for s in shape),
                                         "typestr": typestr, "version": 3, "strides": None}


def view(ptr: int, shape, dtype=torch.float16) -> torch.Tensor:
    """A torch tensor over `prod(shape)` contiguous elements of device memory at `ptr` (no copy)."""
    ts = {torch.float16: "<f2", torch.float32: "<f4"}[dtype]
    return torch.as_tensor(_Cai(ptr, shape, ts), device="cuda")


def out_dims(d):
    s = d.stride
    return d.H // s, d.W // s


def conv_views(d) -> dict:
    """Views of conv op `d`'s buffers: x (whole input tensor), w, b, res (whole residual tensor), out, out2."""
    Ho, Wo = out_dims(d)
    v = {}
    if d.in_layout == L.IN_STEM4:
        v["x"] = view(d.in_, (d.N, d.H + 2, d.W + 2, 4))
        v["w"] = view(d.weight, (3, d.cout_pad, 16))
    else:
        v["x"] = view(d.in_, (d.N, d.H, d.W, d.C))
        v["w"] = view(d.weight, (d.ksize * d.ksize, d.cout_pad, d.cin))
    v["b"] = view(d.bias, (d.cout_pad,), torch.float32)
    v["res"] = view(d.res, (d.N, Ho, Wo, d.res_C)) if d.res else None
    if d.out_mode == L.OUT_F16_NHWC:
        v["out"] = view(d.out, (d.N, Ho, Wo, d.out_C))
    elif d.out_mode == L.OUT_F16_NHWC_UP2:
        v["out"] = view(d.out, (d.N, 2 * Ho, 2 * Wo, d.out_C))
    elif d.out_mode == L.OUT_F32_NHWC:
        v["out"] = view(d.out, (d.N, Ho, Wo, d.out_C), torch.float32)
    elif d.out_mode == L.OUT_F32_NCHW:
        v["out"] = view(d.out, (d.N, d.cout_store, Ho, Wo), torch.float32)
    else:
        raise NotImplementedError(f"out_mode {d.out_mode}")
    if d.head_n:
        raise NotImplementedError("fused 1x1 head")
    v["out2"] = None
    if d.out2_mode == L.OUT2_UP2:
        v["out2"] = view(d.out2, (d.N, 2 * Ho, 2 * Wo, d.out2_C))
    elif d.out2_mode == L.OUT2_POOL2:
        v["out2"] = view(d.out2, (d.N, Ho // 2, Wo // 2, d.out2_C))
    return v


def snapshot(v: dict) -> dict:
    return {k: (None if t is None else t.clone()) for k, t in v.items()}


# ---- reference ----------------------------------------------------------------------------------------------
def unpack_stem_weight(w: torch.Tensor) -> torch.Tensor:
    """[3 filter rows r][cout_pad][16] with k = s * 4 + c -> (cout_pad, 4, 3, 3) over the 4-channel padded input."""
    cout = w.shape[1]
    w4 = w.reshape(3, cout, 4, 4)[:, :, :3, :]  # [r][co][s][c], s < 3
    return w4.permute(1, 3, 0, 2).contiguous()  # [co][c][r][s]


def conv_reference(d, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, res: torch.Tensor | None):
    """float64 (N, Ho, Wo, cout_store) result of conv op `d` on its operands, and A (same shape)."""
    f64 = torch.float64
    if d.in_layout == L.IN_STEM4:
        xi = x.to(f64).permute(0, 3, 1, 2)
        wt = unpack_stem_weight(w).to(f64)
        stride, pad = 2, 0
    else:
        xi = x[..., d.c_in_off:d.c_in_off + d.cin].to(f64).permute(0, 3, 1, 2)
        k = d.ksize
        wt = w.to(f64).reshape(k, k, d.cout_pad, d.cin).permute(2, 3, 0, 1)
        stride, pad = d.stride, k // 2
    acc = F.conv2d(xi, wt, stride=stride, padding=pad).permute(0, 2, 3, 1)
    A = F.conv2d(xi.abs(), wt.abs(), stride=stride, padding=pad).permute(0, 2, 3, 1)
    n = d.cout_store
    acc, A = acc[..., :n], A[..., :n]
    b64 = b[:n].to(f64)
    v = acc + b64
    A = A + b64.abs()
    r = None
    if res is not None:
        r = res[..., d.res_coff:d.res_coff + n].to(f64)
        A = A + r.abs()
    if r is not None and d.res_before_act:
        v = v + r
    if d.act == L.ACT_RELU:
        v = v.clamp_min(0)
    elif d.act == L.ACT_SILU:
        v = v * torch.sigmoid(v)
    elif d.act == L.ACT_SIGMOID:
        v = torch.sigmoid(v)
    if r is not None and not d.res_before_act:
        v = v + r
    return v.contiguous(), A.contiguous()


# ---- comparator ---------------------------------------------------------------------------------------------
def ulp16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp16 numbers at |x| (subnormal spacing 2^-24 below 2^-14), in float64."""
    e = torch.frexp(x.abs().to(torch.float64).clamp_min(2.0 ** -30))[1] - 1  # |x| in [2^e, 2^(e+1))
    return torch.exp2((e.clamp_min(-14) - 10).to(torch.float64))


def ulp32(x: torch.Tensor) -> torch.Tensor:
    e = torch.frexp(x.abs().to(torch.float64).clamp_min(2.0 ** -140))[1] - 1
    return torch.exp2((e.clamp_min(-126) - 23).to(torch.float64))


@dataclass
class ConvReport:
    n: int = 0
    max_ulps: float = 0.0        # max |got - ref| / ulp(ref)
    max_tol_ratio: float = 0.0   # max |got - ref| / tolerance (<= 1 passes)
    max_old_ratio: float = 0.0   # max tolerance / (2e-3 + 2e-3 |ref|): < 1 where this bound is tighter than the old one
    mismatch: float = 0.0        # fraction of fp16 elements != the correctly rounded reference
    bias: float = 0.0            # mean (got - ref) / ulp16(ref), signed by ref (negative: toward zero)
    fails: list = field(default_factory=list)

    @property
    def ok(self) -> bool:
        return not self.fails

    def row(self) -> str:
        return (f"max {self.max_ulps:6.3f} ulp  tol {self.max_tol_ratio:5.3f}  mismatch {self.mismatch:.4f}  "
                f"bias {self.bias:+.4f}  n {self.n}")


def _first_bad(mask: torch.Tensor) -> str:
    idx = mask.nonzero()[0].tolist()
    return f"{int(mask.sum())} elements, first at {idx}"


def compare_values(got: torch.Tensor, ref: torch.Tensor, A: torch.Tensor, rep: ConvReport, what: str = "out"):
    """Per-element bound and rounding statistics of one output (got fp16 or fp32, same shape as ref)."""
    g = got.to(torch.float64)
    err = (g - ref).abs()
    E = ACC_REL * A
    if got.dtype == torch.float16:
        u = ulp16(ref)
        tol = u + E
    else:
        u = ulp32(ref)
        tol = F32_ULPS * u + E
    rep.n += ref.numel()
    if ref.numel() == 0:
        return rep
    if not torch.isfinite(g).all():
        rep.fails.append(f"{what}: non-finite values ({_first_bad(~torch.isfinite(g))})")
        return rep
    rep.max_ulps = max(rep.max_ulps, float((err / u).max()))
    rep.max_tol_ratio = max(rep.max_tol_ratio, float((err / tol).max()))
    old = tol / (2e-3 + 2e-3 * ref.abs())
    rep.max_old_ratio = max(rep.max_old_ratio, float(old.max()))
    if (old >= 1).any():
        rep.fails.append(f"{what}: the bound is not tighter than 2e-3 + 2e-3 |ref| on {_first_bad(old >= 1)} "
                         f"(A too large for ulp + 2^-18 A to mean anything)")
    bad = err > tol
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        rep.fails.append(f"{what}: |got - ref| > ulp + E on {_first_bad(bad)}: got {float(g[i])!r} ref {float(ref[i])!r} "
                         f"tol {float(tol[i]):.3g}")
    if got.dtype == torch.float16:
        # through float32: differs from one correct rounding only within 2^-24 of a midpoint, negligible in a rate
        rn = ref.to(torch.float32).to(torch.float16)
        mism = float((got != rn).double().mean())
        # the bias over the elements whose accumulation error is well below an ulp (near-cancellations would swamp it)
        sharp = E <= u / 4
        bias = float(((g - ref) / u * torch.sign(ref))[sharp].mean()) if sharp.any() else 0.0
        rep.mismatch = max(rep.mismatch, mism)
        rep.bias = bias if abs(bias) > abs(rep.bias) else rep.bias
        if ref.numel() >= MIN_STAT_ELEMENTS and mism > MAX_MISMATCH:
            rep.fails.append(f"{what}: {mism * 100:.2f} % of the elements differ from the correctly rounded result "
                             f"(bound {MAX_MISMATCH * 100:.1f} %)")
        if int(sharp.sum()) >= MIN_STAT_ELEMENTS and abs(bias) > MAX_BIAS:
            rep.fails.append(f"{what}: mean error {bias:+.4f} ulp toward |ref| (bound {MAX_BIAS})")
    return rep


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def check_untouched(before: torch.Tensor, after: torch.Tensor, c0: int, c1: int, rep: ConvReport, what: str):
    """Channels outside [c0, c1) of an NHWC tensor are bit-identical to their value before the op."""
    keep = torch.ones(before.shape[-1], dtype=torch.bool, device=before.device)
    keep[c0:c1] = False
    if keep.any():
        diff = _bits(before[..., keep]) != _bits(after[..., keep])
        if diff.any():
            rep.fails.append(f"{what}: channels outside [{c0}, {c1}) changed: {_first_bad(diff)}")


def check_conv(d, before: dict, after: dict) -> ConvReport:
    """Check conv op `d`: `before` = snapshot of its views (x, w, b, res, out, out2) taken before it ran, `after` =
    out / out2 after it ran."""
    rep = ConvReport()
    ref, A = conv_reference(d, before["x"], before["w"], before["b"], before["res"])
    n = d.cout_store
    out = after["out"]
    c0, c1 = d.out_coff, d.out_coff + n
    if d.out_mode == L.OUT_F32_NCHW:
        compare_values(out, ref.permute(0, 3, 1, 2), A.permute(0, 3, 1, 2), rep)
        prim = None
    elif d.out_mode == L.OUT_F16_NHWC_UP2:
        prim = out[:, 0::2, 0::2, c0:c1]
        compare_values(prim, ref, A, rep)
        for dy in (0, 1):
            for dx in (0, 1):
                if not torch.equal(_bits(out[:, dy::2, dx::2, c0:c1]), _bits(prim)):
                    rep.fails.append(f"out: 2x2 replica ({dy}, {dx}) differs from the pixel it replicates")
        check_untouched(before["out"], out, c0, c1, rep, "out")
    else:
        prim = out[..., c0:c1]
        compare_values(prim, ref, A, rep)
        check_untouched(before["out"], out, c0, c1, rep, "out")
    if d.out2_mode != L.OUT2_NONE:
        o2 = after["out2"]
        a0, a1 = d.out2_coff, d.out2_coff + n
        s2 = o2[..., a0:a1]
        if d.out2_mode == L.OUT2_UP2:
            for dy in (0, 1):
                for dx in (0, 1):
                    if not torch.equal(_bits(s2[:, dy::2, dx::2]), _bits(prim)):
                        rep.fails.append(f"out2: UP2 replica ({dy}, {dx}) is not the primary output")
        else:
            pooled = pool2_exact(prim)
            if not torch.equal(_bits(s2), _bits(pooled)):
                rep.fails.append(f"out2: POOL2 is not the 2x2 max of the primary ({_first_bad(_bits(s2) != _bits(pooled))})")
        check_untouched(before["out2"], o2, a0, a1, rep, "out2")
    return rep


# ---- exact references of the pooling ops ----------------------------------------------------------------------
def pool2_exact(x: torch.Tensor) -> torch.Tensor:
    """2x2 / stride-2 max of an NHWC fp16 tensor (exact: max only selects)."""
    N, H, W, C = x.shape
    return x.reshape(N, H // 2, 2, W // 2, 2, C).amax(dim=(2, 4))


def maxpool_nhwc(x: torch.Tensor, k: int, s: int, p: int) -> torch.Tensor:
    """MaxPool2d(k, s, p) with -inf padding in float64 (exact for fp16 inputs), NHWC in and out."""
    y = F.max_pool2d(x.to(torch.float64).permute(0, 3, 1, 2), k, s, p)
    return y.permute(0, 2, 3, 1).contiguous()


def sppf_reference(x: torch.Tensor) -> list[torch.Tensor]:
    """The three chained MaxPool2d(5, 1, 2) of SPPF."""
    y1 = maxpool_nhwc(x, 5, 1, 2)
    y2 = maxpool_nhwc(y1, 5, 1, 2)
    return [y1, y2, maxpool_nhwc(y2, 5, 1, 2)]


def describe_plan(info) -> str:
    """One-line plan signature of a conv op (pb_op_info)."""
    names = {L.CONV_PER_TAP: "tap", L.CONV_HALO: "halo", L.CONV_HALO_1X1: "halo1x1", L.CONV_HALO_S2: "halo-s2",
             L.CONV_STEM: "stem"}
    s = (f"{names[info.variant]:7s} epi{info.epi} S{info.S} G{info.G} BN{info.BN}x{info.n_ntiles} KB{info.KB}x"
         f"{info.kblocks} a{info.a_stages} b{info.b_stages}")
    if info.variant != L.CONV_PER_TAP:
        s += f" {'res' if info.b_resident else 'str'} {'tma' if info.tma_store else 'lane'}{'+pool' if info.st_pool else ''}"
    return s + f" grid {info.grid}/{info.total_tiles}"


def plan_key(info, d=None) -> dict:
    """The plan axes the coverage test tracks, of one conv op.  Each axis is recorded only for the variants on which
    it is a choice of the set-up: the per-tap kernel reports fixed values on the halo axes (S = G = 1, no resident
    bank, no TMA store), the halo 1x1 / stride-2 / stem set-ups always keep their weights resident, the 1x1 and stem
    plans always use one tap group and stride 2 always nine, and only the 3x3 stride-1 set-up splits N tiles."""
    d = info.desc if d is None else d
    Ho = d.H // d.stride
    v = info.variant
    k = dict(variant=v, epi=info.epi, KB=info.KB, cout_store_lt_pad=d.cout_store < d.cout_pad)
    if v == L.CONV_PER_TAP:
        k["tap_ntiles"] = info.n_ntiles
        return k
    if v == L.CONV_STEM:
        k["stem_BN"] = info.BN
        return k
    k.update(S=info.S, a_stages=info.a_stages, tma_store=info.tma_store, st_pool=info.st_pool,
             tma_S=(info.tma_store, info.S), w_ragged=d.W // d.stride % (8 * info.S) != 0,
             ho16="skip" if 1 <= Ho % 16 <= 8 else "partial" if Ho % 16 else "whole")
    if v == L.CONV_HALO:
        k.update(G=info.G, b_resident=info.b_resident, ntiled=info.n_ntiles > 1,
                 ntile_ragged=info.n_ntiles > 1 and Ho % 16 != 0)
    return k
