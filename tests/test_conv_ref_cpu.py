"""CPU self-test of the conv comparator (tests/conv_ref.py): a CPU emulation of the conv kernels -- an fp32 conv of the
fp16 operands, bias / residual / activation in fp32, round-to-nearest fp16 stores -- passes it at layer shapes with N
tiles, channel slices, residuals, a 2x2-replicated second output, a pooled second output, the stem and an fp32 head;
and each subtly wrong variant of the emulation (a truncating store, a dropped border tap, the wrong N tile's bias, a
skipped channel block, a store one channel outside the slice, the residual on the wrong side of the activation, a
shifted upsample replica) is rejected."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

import conv_ref as R
from padel_analytics_b200 import _lib as L


def _desc(**kw):
    d = dict(N=1, H=12, W=20, C=None, c_in_off=0, cin=32, cout_pad=32, ksize=3, stride=1, act=L.ACT_SILU, res_C=0,
             res_coff=0, out_C=None, out_coff=0, out_mode=L.OUT_F16_NHWC, cout_store=None, head_n=0,
             in_layout=L.IN_NHWC, res_before_act=0, out2_C=0, out2_coff=0, out2_mode=L.OUT2_NONE, res=False)
    d.update(kw)
    d["C"] = d["C"] or d["c_in_off"] + d["cin"]
    d["cout_store"] = d["cout_store"] or d["cout_pad"]
    d["out_C"] = d["out_C"] or d["out_coff"] + d["cout_store"]
    return SimpleNamespace(**d)


CASES = {
    "ntiled": _desc(H=12, W=20, cin=128, cout_pad=256, act=L.ACT_RELU),
    "sliced": _desc(C=96, c_in_off=32, cin=48, cout_pad=48, out_C=96, out_coff=32, act=L.ACT_SILU),
    "residual": _desc(cin=64, cout_pad=64, res=True, res_C=96, res_coff=16, out_C=96, out_coff=16),
    "residual_before_act": _desc(ksize=1, cin=64, cout_pad=128, act=L.ACT_RELU, res=True, res_C=128, res_before_act=1),
    "up2": _desc(ksize=1, cin=64, cout_pad=64, out_C=96, out2_mode=L.OUT2_UP2, out2_C=128, out2_coff=32),
    "pool": _desc(H=16, W=24, cin=64, cout_pad=64, act=L.ACT_RELU, out_C=128, out_coff=64, out2_mode=L.OUT2_POOL2,
                  out2_C=80, out2_coff=16),
    "stem": _desc(H=24, W=32, C=4, cin=16, cout_pad=48, stride=2, in_layout=L.IN_STEM4),
    "f32_head": _desc(ksize=1, cin=64, cout_pad=16, cout_store=8, act=L.ACT_SIGMOID, out_mode=L.OUT_F32_NCHW),
}


def _operands(d, seed=0):
    g = torch.Generator().manual_seed(seed)
    Ho, Wo = d.H // d.stride, d.W // d.stride
    if d.in_layout == L.IN_STEM4:
        x = torch.zeros(d.N, d.H + 2, d.W + 2, 4)
        x[:, 1:-1, 1:-1, :3] = torch.rand(d.N, d.H, d.W, 3, generator=g)
        w = torch.zeros(3, d.cout_pad, 16)
        for s in range(3):
            w[:, :, 4 * s:4 * s + 3] = torch.randn(3, d.cout_pad, 3, generator=g) / 3
    else:
        x = torch.randn(d.N, d.H, d.W, d.C, generator=g)
        w = torch.randn(d.ksize * d.ksize, d.cout_pad, d.cin, generator=g) / (d.ksize * d.ksize * d.cin) ** 0.5
    b = torch.randn(d.cout_pad, generator=g) * 0.2
    t = {"x": x.half(), "w": w.half(), "b": b.float(),
         "res": torch.randn(d.N, Ho, Wo, d.res_C, generator=g).half() if d.res else None}
    if d.out_mode == L.OUT_F32_NCHW:
        t["out"] = torch.full((d.N, d.cout_store, Ho, Wo), 3.0)
    else:
        up = 2 if d.out_mode == L.OUT_F16_NHWC_UP2 else 1
        t["out"] = torch.randn(d.N, Ho * up, Wo * up, d.out_C, generator=g).half()
    t["out2"] = None
    if d.out2_mode == L.OUT2_UP2:
        t["out2"] = torch.randn(d.N, 2 * Ho, 2 * Wo, d.out2_C, generator=g).half()
    elif d.out2_mode == L.OUT2_POOL2:
        t["out2"] = torch.randn(d.N, Ho // 2, Wo // 2, d.out2_C, generator=g).half()
    return t


def _round_toward_zero(v: torch.Tensor) -> torch.Tensor:
    h = v.half()
    up = h.float().abs() > v.abs()  # rounded away from zero: step the magnitude down by one ulp
    bits = h.view(torch.int16).clone()
    bits[up] -= 1
    return bits.view(torch.float16)


def emulate(d, before: dict, mutant: str | None = None) -> dict:
    """The conv op `d` as the kernels compute it (fp32 accumulation, round-to-nearest fp16 stores), optionally with
    one defect."""
    x, w, b = before["x"].float(), before["w"].float(), before["b"].clone()
    if d.in_layout == L.IN_STEM4:
        xi, wt, stride, pad = x.permute(0, 3, 1, 2), R.unpack_stem_weight(w).float(), 2, 0
    else:
        xi = x[..., d.c_in_off:d.c_in_off + d.cin].permute(0, 3, 1, 2)
        wt = w.reshape(d.ksize, d.ksize, d.cout_pad, d.cin).permute(2, 3, 0, 1)
        stride, pad = d.stride, d.ksize // 2
    if mutant == "skip_last_channel_block":
        kb = 64 if d.cin % 64 == 0 else (32 if d.cin % 32 == 0 else 16)
        wt = wt.clone()
        wt[:, d.cin - kb:] = 0
    acc = F.conv2d(xi, wt, stride=stride, padding=pad)
    if mutant == "drop_border_tap":  # the last output column loses filter tap (0, 0)
        t0 = torch.zeros_like(wt)
        t0[:, :, 0, 0] = wt[:, :, 0, 0]
        acc[..., -1] -= F.conv2d(xi, t0, stride=stride, padding=pad)[..., -1]
    acc = acc.permute(0, 2, 3, 1)
    if mutant == "ntile1_uses_ntile0_bias":
        b[128:256] = b[0:128]
    n = d.cout_store
    v = acc[..., :n] + b[:n]
    r = before["res"][..., d.res_coff:d.res_coff + n].float() if d.res else None
    before_act = bool(d.res_before_act) != (mutant == "residual_on_wrong_side")
    if r is not None and before_act:
        v = v + r
    if d.act == L.ACT_RELU:
        v = v.clamp_min(0)
    elif d.act == L.ACT_SILU:
        v = v * torch.sigmoid(v)
    elif d.act == L.ACT_SIGMOID:
        v = torch.sigmoid(v)
    if r is not None and not before_act:
        v = v + r
    after = {"out": before["out"].clone(), "out2": None if before["out2"] is None else before["out2"].clone()}
    if d.out_mode == L.OUT_F32_NCHW:
        after["out"][:] = v.permute(0, 3, 1, 2)
        return after
    h = _round_toward_zero(v) if mutant == "round_toward_zero" else v.half()
    c0, c1 = d.out_coff, d.out_coff + n
    o = after["out"]
    if d.out_mode == L.OUT_F16_NHWC_UP2:
        for dy in (0, 1):
            for dx in (0, 1):
                o[:, dy::2, dx::2, c0:c1] = h
    else:
        o[..., c0:c1] = h
    if mutant == "store_outside_slice":
        o[..., c1] = h[..., -1]
    if d.out2_mode == L.OUT2_UP2:
        a0 = d.out2_coff
        for dy in (0, 1):
            for dx in (0, 1):
                src = h.roll(1, dims=2) if (mutant == "shifted_up2_replica" and (dy, dx) == (1, 1)) else h
                after["out2"][:, dy::2, dx::2, a0:a0 + n] = src
    elif d.out2_mode == L.OUT2_POOL2:
        after["out2"][..., d.out2_coff:d.out2_coff + n] = R.pool2_exact(h)
    return after


@pytest.mark.parametrize("name", list(CASES))
def test_kernel_emulation_passes_the_comparator(name):
    d = CASES[name]
    before = _operands(d)
    rep = R.check_conv(d, before, emulate(d, before))
    print(name, rep.row())
    assert rep.ok, rep.fails
    assert rep.max_tol_ratio <= 1.0 and rep.n > 0


MUTANTS = {
    "round_toward_zero": "ntiled",
    "drop_border_tap": "sliced",
    "ntile1_uses_ntile0_bias": "ntiled",
    "skip_last_channel_block": "ntiled",
    "store_outside_slice": "residual",
    "residual_on_wrong_side": "residual",
    "shifted_up2_replica": "up2",
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_comparator_rejects_a_subtly_wrong_kernel(mutant):
    d = CASES[MUTANTS[mutant]]
    before = _operands(d)
    rep = R.check_conv(d, before, emulate(d, before, mutant))
    print(mutant, rep.row(), rep.fails)
    assert not rep.ok, f"{mutant} passed the comparator: {rep.row()}"


@pytest.mark.parametrize("name", ["sliced", "pool", "stem"])
def test_round_toward_zero_fails_on_the_rounding_statistics_alone(name):
    """A truncating store stays within one ulp of the exact result, so only the rounding statistics can see it."""
    d = CASES[name]
    before = _operands(d, seed=1)
    rep = R.check_conv(d, before, emulate(d, before, "round_toward_zero"))
    assert rep.max_tol_ratio <= 1.0, rep.row()
    assert rep.mismatch > 4 * R.MAX_MISMATCH and rep.bias < -5 * R.MAX_BIAS, rep.row()


def test_ulp16_and_exact_pool_references():
    v = torch.tensor([1.0, 1.999, 2.0, 2.0 ** -14, 2.0 ** -20, 0.0, -65504.0], dtype=torch.float64)
    exp = [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24, 32.0]
    assert R.ulp16(v).tolist() == exp
    x = torch.randn(2, 7, 9, 8).half()
    got = R.sppf_reference(x)
    y = x.double()
    for k in range(3):  # brute force: 5x5 window max with the window clipped to the image
        ref = torch.empty_like(y)
        for i in range(7):
            for j in range(9):
                ref[:, i, j] = y[:, max(i - 2, 0):i + 3, max(j - 2, 0):j + 3].amax(dim=(1, 2))
        assert torch.equal(got[k], ref)
        y = ref


def test_plan_key_records_halo_axes_only_where_the_setup_chooses_them():
    """The per-tap kernel's fixed S = G = 1 / stage count, and the stem's fixed rings, must not count as reached halo
    plan values in the coverage test."""
    d = _desc(H=28, W=20, cin=512, cout_pad=1024, ksize=1)
    info = SimpleNamespace(variant=L.CONV_PER_TAP, epi=2, S=1, G=1, BN=256, n_ntiles=4, KB=64, kblocks=8,
                           b_resident=0, a_stages=4, b_stages=4, tma_store=0, st_pool=0, desc=d)
    k = R.plan_key(info)
    assert k["tap_ntiles"] == 4 and not {"S", "G", "a_stages", "b_resident", "ntiled", "tma_S"} & set(k)
    stem = SimpleNamespace(**{**vars(info), "variant": L.CONV_STEM, "BN": 48, "n_ntiles": 1, "S": 4, "G": 3})
    assert R.plan_key(stem)["stem_BN"] == 48 and "a_stages" not in R.plan_key(stem)
    halo = SimpleNamespace(**{**vars(info), "variant": L.CONV_HALO, "S": 2, "G": 1, "BN": 128, "n_ntiles": 2,
                              "desc": _desc(H=20, W=40, cin=128, cout_pad=256)})
    k = R.plan_key(halo)
    assert (k["G"], k["ntiled"], k["ntile_ragged"], k["ho16"], k["w_ragged"]) == (1, True, True, "skip", True)
    one = SimpleNamespace(**{**vars(halo), "variant": L.CONV_HALO_1X1, "n_ntiles": 1})
    assert "G" not in R.plan_key(one) and "b_resident" not in R.plan_key(one)
