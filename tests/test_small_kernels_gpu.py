"""The non-conv kernels in isolation, at shapes the shipped programs never produce, against float64 / exact references:
the ResNet stem on ragged output tiles, maxpool3x3s2 on odd sizes, avgpool-fc-sigmoid with more outputs than warps,
pb_u8_normalize_f16 bit for bit, the pointwise head with a grid-stride loop that wraps, sppf on planes narrower than
its window and on the largest plane it accepts, maxpool2 / upsample2 on channel slices."""
import ctypes as C

import pytest
import torch

import conv_ref as R
import test_program_layers_gpu as replay
from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import ops

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("hw", [(36, 50), (18, 34), (2, 2)])
def test_resnet_stem7x7_on_ragged_output_tiles(hw):
    """Output tiles are 8 x 16: H / 2 = 18, 9, 1 and W / 2 = 25, 17, 1 leave partial tiles on both axes."""
    H, W = hw
    g = _gen(H)
    x = torch.randn(2, H, W, 4, generator=g).half().cuda()
    w = (torch.randn(147, 64, generator=g) / 12).cuda()
    b = (torch.randn(64, generator=g) * 0.2).cuda()
    out = torch.full((2, H // 2, W // 2, 64), 7.0, dtype=torch.float16, device="cuda")
    L.check(L.lib().pb_resnet_stem7x7(x.data_ptr(), 2, H, W, w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                      L.stream_ptr()))
    torch.cuda.synchronize()
    rep = replay.check_stem7x7(x, w, b, out)
    print(hw, rep.row())
    assert rep.ok, rep.fails


@pytest.mark.parametrize("hwc", [(7, 9, 8), (13, 1, 16), (1, 5, 24), (112, 112, 64)])
def test_maxpool3x3s2_on_odd_sizes(hwc):
    H, W, Cc = hwc
    x = torch.randn(3, H, W, Cc, generator=_gen(1)).half().cuda()
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out = torch.full((3, Ho, Wo, Cc), 7.0, dtype=torch.float16, device="cuda")
    L.check(L.lib().pb_maxpool3x3s2(x.data_ptr(), 3, H, W, Cc, out.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(out.double(), R.maxpool_nhwc(x, 3, 2, 1))


@pytest.mark.parametrize("hw_c_n", [(49, 2048, 24), (3, 64, 9), (1, 8, 1), (100, 512, 17)])
def test_avgpool_fc_sigmoid_with_more_outputs_than_warps(hw_c_n):
    HW, Cc, n_out = hw_c_n
    g = _gen(HW)
    x = torch.randn(3, HW, Cc, generator=g).half().cuda()
    w = (torch.randn(n_out, Cc, generator=g) / Cc ** 0.5 * 4).cuda()
    b = torch.randn(n_out, generator=g).cuda()
    out = torch.full((3, n_out), 7.0, device="cuda")
    L.check(L.lib().pb_avgpool_fc_sigmoid(x.data_ptr(), 3, HW, Cc, w.data_ptr(), b.data_ptr(), n_out, out.data_ptr(),
                                          L.stream_ptr()))
    torch.cuda.synchronize()
    rep = replay.check_avgpool_fc(x, w, b, out)
    print(hw_c_n, rep.row())
    assert rep.ok, rep.fails


def test_u8_normalize_is_bit_exact_to_the_fp32_formula():
    """((x / 255) - mean) / std in fp32 with IEEE division, rounded to nearest fp16; channel 3 = 0."""
    mean, std = (0.485, 0.465, 0.406), (0.229, 0.224, 0.225)
    src = torch.arange(256, dtype=torch.uint8).repeat(3 * 347).reshape(-1, 3)  # every value in every channel
    src = torch.cat([src, torch.randint(0, 256, (1001, 3), generator=_gen(2), dtype=torch.uint8)])
    npix = src.shape[0]
    dst = torch.full((npix, 4), 7.0, dtype=torch.float16, device="cuda")
    src_d = src.cuda()
    L.check(L.lib().pb_u8_normalize_f16(src_d.data_ptr(), npix, (C.c_float * 3)(*mean), (C.c_float * 3)(*std),
                                        dst.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    m = torch.tensor(mean, dtype=torch.float32)
    s = torch.tensor(std, dtype=torch.float32)
    exp = ((src.float() / torch.tensor(255.0)) - m) / s
    assert torch.equal(dst[:, :3].cpu().view(torch.int16), exp.half().view(torch.int16))
    assert torch.equal(dst[:, 3].cpu(), torch.zeros(npix, dtype=torch.float16))


def _program_check(prog):
    """Run every op of a small program alone through the replay checks."""
    rows, _, _, fails = replay.replay(prog, "small")
    assert not fails, "\n".join(fails)
    return rows


@pytest.mark.parametrize("shape", [(3, 7, 67, 64, 8), (1, 3, 700, 24, 3), (2, 33, 41, 8, 1)])
def test_pointwise_head_when_the_grid_stride_loop_wraps(shape):
    """Built for one SM the head launches at most 5 CTAs of 256 pixels; with more than 5 pixel tiles and npix not a
    multiple of 256 (6, 9 and 11 tiles), the first CTAs take a second tile, and the last, partial tile is reached on a
    later iteration of the grid-stride loop."""
    N, H, W, Cc, n_out = shape
    npix = N * H * W
    assert npix > 5 * 256 and npix % 256 != 0
    g = _gen(W)
    x = torch.randn(N, H, W, Cc, generator=g).half().cuda()
    w = (torch.randn(n_out, Cc, generator=g) / Cc ** 0.5).cuda()
    b = torch.randn(n_out, generator=g).cuda()
    out = torch.full((N, n_out, H, W), 7.0, device="cuda")
    p = ops.Program()
    p.pointwise_head(x, w, b, out)
    p.keep(x, w, b, out)
    L.lib().pb_set_plan_options(1, -1)  # the head sizes its grid when launched
    try:
        _program_check(p)
    finally:
        L.lib().pb_set_plan_options(0, -1)


@pytest.mark.parametrize("hw", [(1, 1), (3, 4), (4, 2), (7, 3), (40, 40), (80, 80)])
def test_sppf_on_planes_narrower_than_the_window_and_the_largest_plane(hw):
    """(80, 80) x 16-byte vectors x 2 buffers = 200 KB: the largest plane the kernel accepts."""
    H, W = hw
    c = 16
    buf = torch.randn(2, H, W, 4 * c + 8, generator=_gen(H * W)).half().cuda()
    p = ops.Program()
    p.sppf_pool(buf, c)
    p.keep(buf)
    _program_check(p)


def test_sppf_rejects_a_plane_that_does_not_fit():
    buf = torch.zeros(1, 81, 80, 32, dtype=torch.float16, device="cuda")
    p = ops.Program()
    p.sppf_pool(buf, 8)
    with pytest.raises(L.PbError, match="does not fit"):
        p.run()


@pytest.mark.parametrize("case", [dict(H=6, W=10, C=48, c_off=16, c=24, out_C=40, out_coff=8),
                                  dict(H=2, W=2, C=8, c_off=0, c=8, out_C=16, out_coff=8),
                                  dict(H=36, W=64, C=384, c_off=256, c=128, out_C=136, out_coff=0)],
                         ids=lambda c: f"{c['H']}x{c['W']}-{c['c_off']}+{c['c']}")
def test_maxpool2_and_upsample2_on_channel_slices(case):
    H, W = case["H"], case["W"]
    x = torch.randn(2, H, W, case["C"], generator=_gen(H)).half().cuda()
    pooled = torch.randn(2, H // 2, W // 2, case["out_C"], generator=_gen(3)).half().cuda()
    up = torch.randn(2, 2 * H, 2 * W, case["out_C"], generator=_gen(4)).half().cuda()
    p = ops.Program()
    p.maxpool2(x, case["c_off"], case["c"], pooled, case["out_coff"])
    p.upsample2(x, case["c_off"], case["c"], up, case["out_coff"])
    p.keep(x, pooled, up)
    _program_check(p)
