"""wgmma implicit-GEMM conv vs torch fp32 conv2d on the same fp16-rounded operands (and vs the CUDA-core
reference kernel).  Tolerance: fp16 output rounding (rel 2^-10) + fp32 accumulation-order noise."""
import pytest
import torch
import torch.nn.functional as F

from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import ops

pytestmark = pytest.mark.gpu

ACT = {L.ACT_NONE: lambda v: v, L.ACT_RELU: torch.relu, L.ACT_SILU: F.silu, L.ACT_SIGMOID: torch.sigmoid}


def run_case(N, H, W, cin, cout, k, s, act, cin_real=None, c_total=None, c_in_off=0, out_mode=L.OUT_F16_NHWC,
             residual=False, out_coff=0, out_extra=0, seed=0, reference=False, res_first=False):
    g = torch.Generator().manual_seed(seed)
    dev = "cuda"
    cin_real = cin_real or cin
    c_total = c_total or cin
    x = torch.zeros(N, H, W, c_total)
    x[..., c_in_off:c_in_off + cin_real] = torch.randn(N, H, W, cin_real, generator=g)
    x16 = x.half()
    w = torch.randn(cout, cin_real, k, k, generator=g) / (cin_real * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    cout_pad = ops.pad16(cout)
    wp, bp = ops.pack_conv_weight(w, b, cin, cout_pad, dev)
    xd = x16.to(dev)
    Ho, Wo = H // s, W // s
    up = 2 if out_mode == L.OUT_F16_NHWC_UP2 else 1
    if out_mode in (L.OUT_F16_NHWC, L.OUT_F16_NHWC_UP2):
        cs = cout_pad
        out = torch.full((N, Ho * up, Wo * up, cout_pad + out_coff + out_extra), 7.0, dtype=torch.float16, device=dev)
    elif out_mode == L.OUT_F32_NHWC:
        cs = cout
        out = torch.full((N, Ho, Wo, cout + out_coff + out_extra), 7.0, dtype=torch.float32, device=dev)
    else:
        cs = cout
        out = torch.full((N, cout, Ho, Wo), 7.0, dtype=torch.float32, device=dev)
    res = None
    if residual:
        res = torch.randn(N, Ho, Wo, cout_pad, generator=g).half().to(dev)
    d = ops.make_conv_desc(xd, c_in_off, cin, wp, bp, k, s, act, out, out_coff, out_mode, cs, res, 0)
    d.res_before_act = 1 if res_first else 0
    ops.conv2d(d, reference=reference)
    torch.cuda.synchronize()
    # fp32 reference on the fp16-rounded operands
    xr = x16[..., c_in_off:c_in_off + cin_real].float().permute(0, 3, 1, 2)
    wr = w.half().float()
    y = F.conv2d(xr, wr, b, stride=s, padding=k // 2)
    if residual and res_first:  # torchvision ResNet Bottleneck: relu(bn3(conv3(.)) + identity)
        y = y + res.cpu().float()[..., :cout].permute(0, 3, 1, 2)
    y = ACT[act](y)
    if residual and not res_first:
        y = y + res.cpu().float()[..., :cout].permute(0, 3, 1, 2)
    o = out.cpu().float()
    if out_mode == L.OUT_F32_NCHW:
        got = o
    else:
        if up == 2:
            y = F.interpolate(y, scale_factor=2, mode="nearest")
        got = o[..., out_coff:out_coff + cout].permute(0, 3, 1, 2)
        # untouched neighbours keep the fill value
        if out_coff:
            assert torch.all(o[..., :out_coff] == 7.0)
        if out_extra:
            assert torch.all(o[..., out_coff + cs:] == 7.0)
    err = (got - y).abs()
    tol = 2e-3 + 2e-3 * y.abs()
    bad = (err > tol).float().mean().item()
    return bad, err.max().item()


CASES = [
    # N, H, W, cin, cout, k, s, act, kwargs
    dict(N=1, H=16, W=128, cin=64, cout=64, k=1, s=1, act=L.ACT_NONE),
    dict(N=1, H=16, W=128, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),
    dict(N=2, H=36, W=64, cin=128, cout=256, k=3, s=1, act=L.ACT_RELU),
    dict(N=1, H=36, W=64, cin=256, cout=512, k=3, s=1, act=L.ACT_RELU),
    dict(N=2, H=24, W=40, cin=32, cout=32, k=3, s=1, act=L.ACT_SILU),
    dict(N=2, H=24, W=40, cin=16, cout=16, k=3, s=1, act=L.ACT_SILU),
    dict(N=2, H=24, W=40, cin=48, cout=80, k=3, s=1, act=L.ACT_SILU),
    dict(N=2, H=48, W=80, cin=16, cout=32, k=3, s=2, act=L.ACT_SILU),
    dict(N=2, H=48, W=80, cin=64, cout=128, k=3, s=2, act=L.ACT_SILU),
    dict(N=3, H=12, W=20, cin=256, cout=256, k=3, s=1, act=L.ACT_SILU),
    dict(N=4, H=6, W=10, cin=128, cout=64, k=1, s=1, act=L.ACT_SILU),
    dict(N=2, H=24, W=40, cin=32, cout=32, k=3, s=1, act=L.ACT_SILU, residual=True),
    dict(N=2, H=24, W=40, cin=32, cout=32, k=3, s=1, act=L.ACT_SILU, c_total=96, c_in_off=32, out_coff=64,
         out_extra=32),
    dict(N=2, H=16, W=32, cin=32, cout=27, k=1, s=1, act=L.ACT_NONE, cin_real=27, out_mode=L.OUT_F32_NHWC,
         out_coff=64, out_extra=3),
    dict(N=2, H=16, W=32, cin=64, cout=8, k=1, s=1, act=L.ACT_SIGMOID, out_mode=L.OUT_F32_NCHW),
    dict(N=2, H=16, W=32, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU, out_mode=L.OUT_F16_NHWC_UP2),
    dict(N=1, H=72, W=128, cin=768, cout=256, k=3, s=1, act=L.ACT_RELU),
    dict(N=1, H=288, W=512, cin=32, cout=64, k=3, s=1, act=L.ACT_RELU, cin_real=27),
    # ResNet50 court regressor shapes (keypoints_tracker.py:158): identity added BEFORE the ReLU, 1x1 stride-2
    # downsample convs, 2048-wide outputs (8 N tiles)
    dict(N=2, H=14, W=14, cin=256, cout=1024, k=1, s=1, act=L.ACT_RELU, residual=True, res_first=True),
    dict(N=2, H=28, W=28, cin=512, cout=1024, k=1, s=2, act=L.ACT_NONE),
    dict(N=2, H=56, W=56, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),
    dict(N=2, H=28, W=28, cin=128, cout=128, k=3, s=2, act=L.ACT_RELU),
    dict(N=3, H=7, W=7, cin=512, cout=2048, k=1, s=1, act=L.ACT_RELU, residual=True, res_first=True),
    dict(N=2, H=24, W=40, cin=32, cout=32, k=3, s=1, act=L.ACT_RELU, residual=True, res_first=True),
    dict(N=2, H=14, W=14, cin=1024, cout=2048, k=1, s=2, act=L.ACT_NONE),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_reference_kernel_matches_torch(case):
    if case["H"] * case["W"] * case["cin"] * case["cout"] > 2e9:
        pytest.skip("too slow for the CUDA-core kernel")
    bad, mx = run_case(**case, reference=True)
    assert bad == 0.0, f"reference kernel: {bad*100:.3f}% elements out of tolerance (max err {mx})"


HALO_CASES = [
    dict(N=1, H=32, W=64, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),
    dict(N=2, H=36, W=52, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),            # ragged: H % 16, W % 8 != 0
    dict(N=2, H=20, W=12, cin=128, cout=128, k=3, s=1, act=L.ACT_SILU),
    dict(N=1, H=48, W=80, cin=192, cout=64, k=3, s=1, act=L.ACT_RELU),           # 3 channel blocks
    dict(N=2, H=24, W=40, cin=48, cout=80, k=3, s=1, act=L.ACT_SILU),            # KB=16 rows (32B swizzle)
    dict(N=2, H=24, W=40, cin=32, cout=32, k=3, s=1, act=L.ACT_SILU, residual=True, c_total=96, c_in_off=32,
         out_coff=64, out_extra=32),                                             # KB=32 (64B swizzle) + slices
    dict(N=3, H=17, W=9, cin=16, cout=16, k=3, s=1, act=L.ACT_SILU),
    dict(N=1, H=16, W=32, cin=64, cout=128, k=3, s=1, act=L.ACT_RELU, out_mode=L.OUT_F16_NHWC_UP2),
    dict(N=1, H=36, W=64, cin=256, cout=256, k=3, s=1, act=L.ACT_RELU),          # S=1, two accumulator sets
    dict(N=2, H=16, W=32, cin=64, cout=27, k=3, s=1, act=L.ACT_NONE, out_mode=L.OUT_F32_NHWC, out_coff=64,
         out_extra=3),
    # stride-2 halo (pixel-pair rows): 64-byte rows (cin 16) and 128-byte rows (cin 32), ragged tiles, slices
    dict(N=2, H=40, W=56, cin=32, cout=64, k=3, s=2, act=L.ACT_SILU),
    dict(N=3, H=34, W=18, cin=16, cout=16, k=3, s=2, act=L.ACT_SILU, out_coff=16, out_extra=16),
    dict(N=1, H=96, W=160, cin=16, cout=32, k=3, s=2, act=L.ACT_RELU),
    # fast epilogue, fp32 NHWC slice ending mid-chunk (39 = 2 x 16 + 7) at a 32-byte aligned offset
    dict(N=2, H=16, W=32, cin=64, cout=39, k=1, s=1, act=L.ACT_NONE, out_mode=L.OUT_F32_NHWC, out_coff=64,
         out_extra=25),
    dict(N=2, H=24, W=40, cin=64, cout=39, k=3, s=1, act=L.ACT_SILU, out_mode=L.OUT_F32_NHWC, out_coff=8,
         out_extra=1),
    dict(N=2, H=20, W=24, cin=128, cout=256, k=1, s=1, act=L.ACT_RELU, out_mode=L.OUT_F16_NHWC_UP2, out_coff=32),
]


@pytest.mark.parametrize("halo", [0, 1], ids=["pertap", "halo"])
@pytest.mark.parametrize("case", CASES + HALO_CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_tcgen05_conv_matches_torch(case, halo, monkeypatch):
    """Both tensor-core variants (per-tap TMA boxes / shared halo tile; the latter only applies to 3x3 s1)."""
    monkeypatch.setenv("PADEL_B200_CONV_HALO", str(halo))
    bad, mx = run_case(**case)
    assert bad == 0.0, f"tensor-core kernel: {bad*100:.3f}% elements out of tolerance (max err {mx})"


def test_fused_1x1_head_matches_torch():
    """conv3x3+ReLU with the TrackNet predictor (1x1, 8 outputs, sigmoid) fused into the epilogue."""
    g = torch.Generator().manual_seed(5)
    N, H, W, cin, cout = 2, 16, 128, 64, 64
    x = torch.randn(N, H, W, cin, generator=g).half()
    w = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    hw = torch.randn(8, cout, generator=g) * 0.3
    hb = torch.randn(8, generator=g) * 0.1
    wp, bp = ops.pack_conv_weight(w, b, cin, cout, "cuda")
    out = torch.zeros((N, 8, H, W), device="cuda")
    d = ops.make_conv_desc(x.cuda(), 0, cin, wp, bp, 3, 1, L.ACT_RELU, None, 0, L.OUT_NONE,
                           head=(hw.cuda().contiguous(), hb.cuda(), out))
    ops.conv2d(d)
    torch.cuda.synchronize()
    y = torch.relu(F.conv2d(x.float().permute(0, 3, 1, 2), w.half().float(), b, padding=1))
    exp = torch.sigmoid(F.conv2d(y, hw.view(8, cout, 1, 1), hb))
    assert (out.cpu() - exp).abs().max().item() < 2e-3


@pytest.mark.parametrize("shape", [(2, 64, 96, 16), (1, 384, 640, 16), (3, 40, 72, 48)])
def test_stem_conv_padded4_layout(shape):
    """3x3/s2 stem conv reading the padded 4-channel input (PB_IN_STEM4) through one overlapping-row TMA box."""
    N, H, W, cout = shape
    g = torch.Generator().manual_seed(9)
    img = torch.rand(N, H, W, 3, generator=g).half()
    xp = torch.zeros(N, H + 2, W + 2, 4, dtype=torch.float16)
    xp[:, 1:-1, 1:-1, :3] = img
    w = torch.randn(cout, 3, 3, 3, generator=g) / 27 ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    wp, bp = ops.pack_stem_weight(w, b, ops.pad16(cout), "cuda")
    y = F.silu(F.conv2d(img.float().permute(0, 3, 1, 2), w.half().float(), b, stride=2, padding=1))
    for reference in (True, False):
        out = torch.full((N, H // 2, W // 2, ops.pad16(cout)), 7.0, dtype=torch.float16, device="cuda")
        d = ops.make_stem_desc(xp.cuda(), wp, bp, L.ACT_SILU, out)
        ops.conv2d(d, reference=reference)
        torch.cuda.synchronize()
        got = out.cpu().float()[..., :cout].permute(0, 3, 1, 2)
        err = (got - y).abs()
        assert (err > 2e-3 + 2e-3 * y.abs()).float().mean().item() == 0.0, (reference, err.max().item())


PAIR_CASES = [
    dict(N=1, H=32, W=64, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),
    dict(N=2, H=48, W=40, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),             # odd number of 16-row tiles
    dict(N=1, H=64, W=64, cin=192, cout=64, k=3, s=1, act=L.ACT_RELU),
    dict(N=2, H=32, W=32, cin=128, cout=128, k=3, s=1, act=L.ACT_SILU, residual=True),
    dict(N=1, H=32, W=32, cin=32, cout=32, k=3, s=1, act=L.ACT_SILU),
    dict(N=1, H=32, W=64, cin=64, cout=128, k=3, s=1, act=L.ACT_RELU, out_mode=L.OUT_F16_NHWC_UP2),
    dict(N=4, H=288, W=512, cin=64, cout=64, k=3, s=1, act=L.ACT_RELU),
]


@pytest.mark.parametrize("case", PAIR_CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_halo_conv_cta_pair_mode(case, monkeypatch):
    """Halo kernel on deep-K, odd-tile-count and large shapes (those of the former CTA-pair variant)."""
    monkeypatch.setenv("PADEL_B200_CONV_HALO", "1")
    bad, mx = run_case(**case)
    assert bad == 0.0, f"pair-mode kernel: {bad*100:.3f}% elements out of tolerance (max err {mx})"


OUT2_CASES = [
    # YOLO neck: 1x1 conv whose output also feeds nn.Upsample(2) -> concat slice (layers 9->10->11, 12->13->14)
    dict(N=2, H=12, W=20, cin=512, cout=256, k=1, mode=L.OUT2_UP2, act=L.ACT_SILU),
    dict(N=3, H=24, W=40, cin=192, cout=128, k=1, mode=L.OUT2_UP2, act=L.ACT_SILU),
    dict(N=1, H=20, W=20, cin=960, cout=576, k=1, mode=L.OUT2_UP2, act=L.ACT_SILU),  # m scale: 3 N tiles of 192
    dict(N=2, H=16, W=32, cin=64, cout=64, k=3, mode=L.OUT2_UP2, act=L.ACT_RELU),
    # TrackNet encoder: 3x3 conv + MaxPool2d(2) (models.py:58-62); large and ragged tiles
    dict(N=2, H=288, W=512, cin=64, cout=64, k=3, mode=L.OUT2_POOL2, act=L.ACT_RELU),
    dict(N=3, H=144, W=256, cin=128, cout=128, k=3, mode=L.OUT2_POOL2, act=L.ACT_RELU),
    dict(N=2, H=36, W=44, cin=32, cout=48, k=3, mode=L.OUT2_POOL2, act=L.ACT_RELU),
    dict(N=1, H=18, W=10, cin=16, cout=16, k=3, mode=L.OUT2_POOL2, act=L.ACT_SILU),
]


@pytest.mark.parametrize("case", OUT2_CASES, ids=lambda c: "-".join(f"{k}{v}" for k, v in c.items()))
def test_conv_secondary_output_is_the_upsampled_or_pooled_primary(case):
    """PB_OUT2_UP2 / PB_OUT2_POOL2: the second tensor must be EXACTLY nearest-upsample / 2x2 max-pool of the fp16 primary
    output (same rounded values, so bit-exact), inside its channel slice only; the primary equals the plain conv."""
    N, H, W, cin, cout, k, mode, act = (case[q] for q in ("N", "H", "W", "cin", "cout", "k", "mode", "act"))
    g = torch.Generator().manual_seed(5)
    dev = "cuda"
    x = torch.randn(N, H, W, cin, generator=g).half().to(dev)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    wp, bp = ops.pack_conv_weight(w, b, cin, cout, dev)
    off1, off2 = 16, 32
    out = torch.full((N, H, W, cout + off1 + 16), 7.0, dtype=torch.float16, device=dev)
    plain = torch.zeros((N, H, W, cout), dtype=torch.float16, device=dev)
    shape2 = (N, 2 * H, 2 * W) if mode == L.OUT2_UP2 else (N, H // 2, W // 2)
    out2 = torch.full((*shape2, cout + off2 + 16), 5.0, dtype=torch.float16, device=dev)
    ops.conv2d(ops.make_conv_desc(x, 0, cin, wp, bp, k, 1, act, plain, 0))
    ops.conv2d(ops.make_conv_desc(x, 0, cin, wp, bp, k, 1, act, out, off1, out2=(out2, off2, mode)))
    torch.cuda.synchronize()
    prim = out[..., off1:off1 + cout]
    assert torch.equal(prim, plain)
    assert torch.all(out[..., :off1] == 7.0) and torch.all(out[..., off1 + cout:] == 7.0)
    p = prim.permute(0, 3, 1, 2).float()
    want = F.interpolate(p, scale_factor=2, mode="nearest") if mode == L.OUT2_UP2 else F.max_pool2d(p, 2, 2)
    got = out2[..., off2:off2 + cout].permute(0, 3, 1, 2).float()
    assert torch.equal(got, want)
    assert torch.all(out2[..., :off2] == 5.0) and torch.all(out2[..., off2 + cout:] == 5.0)
    # and the plain conv is the usual one
    y = ACT[act](F.conv2d(x.cpu().float().permute(0, 3, 1, 2), w.half().float(), b, padding=k // 2))
    err = (plain.cpu().float().permute(0, 3, 1, 2) - y).abs()
    assert ((err > 2e-3 + 2e-3 * y.abs()).float().mean().item()) == 0
