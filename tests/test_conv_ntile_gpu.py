"""The halo conv kernel with N tiles (cout > 192 in tiles of 128 channels) and with warpgroups whose eight image rows
lie below the image (72- and 36-row layers): TrackNet's down_block_3 / bottleneck / up_block_1 shapes against torch,
the pooled second store, the TMA-store epilogue against the per-lane stores, and the layers' routing."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import test_conv_gpu as base
from oracle import weights as OW
from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import ops
from padel_analytics_b200.engine.tracknet_engine import TrackNetEngine

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]

NTILE_CASES = [
    dict(N=2, H=72, W=128, cin=128, cout=256, k=3, s=1, act=L.ACT_RELU),  # two N tiles, warpgroup skip
    dict(N=1, H=36, W=64, cin=256, cout=512, k=3, s=1, act=L.ACT_RELU),   # four N tiles
    dict(N=1, H=72, W=128, cin=768, cout=256, k=3, s=1, act=L.ACT_RELU),  # 12 channel blocks
    dict(N=2, H=36, W=64, cin=512, cout=512, k=3, s=1, act=L.ACT_RELU, out_mode=L.OUT_F16_NHWC_UP2),
    dict(N=2, H=36, W=64, cin=128, cout=256, k=3, s=1, act=L.ACT_SILU, c_total=192, c_in_off=64, out_coff=32,
         out_extra=16),                                                   # slices, TMA store
]
_id = lambda c: "-".join(f"{k}{v}" for k, v in c.items())


def _kernel_of(case):
    """Which kernel the default routing gives a layer of this shape."""
    N, H, W, cin, cout = (case[q] for q in ("N", "H", "W", "cin", "cout"))
    x = torch.zeros(N, H, W, cin, dtype=torch.float16, device="cuda")
    wp, bp = ops.pack_conv_weight(torch.zeros(cout, cin, 3, 3), torch.zeros(cout), cin, cout, "cuda")
    out = torch.zeros(N, H, W, cout, dtype=torch.float16, device="cuda")
    p = ops.Program()
    p.conv(ops.make_conv_desc(x, 0, cin, wp, bp, 3, 1, L.ACT_RELU, out, 0))
    return p.op_kernels()[0]


@pytest.mark.parametrize("case", NTILE_CASES, ids=_id)
def test_ntiled_halo_conv_matches_torch(case, monkeypatch):
    monkeypatch.delenv("PADEL_B200_CONV_HALO", raising=False)
    assert _kernel_of(case) == "conv_halo_kernel"
    bad, mx = base.run_case(**case)
    assert bad == 0.0, f"halo kernel: {bad*100:.3f}% elements out of tolerance (max err {mx})"


@pytest.mark.parametrize("case", [dict(N=2, H=72, W=128, cin=256, cout=256, k=3, mode=L.OUT2_POOL2, act=L.ACT_RELU),
                                  dict(N=2, H=36, W=64, cin=128, cout=256, k=3, mode=L.OUT2_POOL2, act=L.ACT_SILU)],
                         ids=_id)
def test_ntiled_pooled_second_store_is_the_maxpool_of_the_primary(case):
    base.test_conv_secondary_output_is_the_upsampled_or_pooled_primary(case)


def test_default_routing_keeps_wasteful_edge_tiles_on_the_per_tap_kernel(monkeypatch):
    """ResNet50's 14x14 and 7x7 3x3 convs would compute 1.31x / 2.6x their output pixels in 16 x 16 halo tiles."""
    monkeypatch.delenv("PADEL_B200_CONV_HALO", raising=False)
    assert _kernel_of(dict(N=2, H=14, W=14, cin=256, cout=256)) == "conv_tc_kernel"
    assert _kernel_of(dict(N=2, H=7, W=7, cin=512, cout=512)) == "conv_tc_kernel"


def test_tracknet_runs_every_3x3_conv_on_the_halo_kernel_and_fuses_every_pool(monkeypatch):
    monkeypatch.delenv("PADEL_B200_CONV_HALO", raising=False)
    monkeypatch.delenv("PADEL_B200_FUSE_OUT2", raising=False)
    prog = TrackNetEngine(OW.make_tracknet()["model"], max_batch=1).prog
    kernels = prog.op_kernels()
    k3 = [kn for kn, d in zip(kernels, prog.descs) if d is not None and d.ksize == 3]
    assert len(k3) == 17 and set(k3) == {"conv_halo_kernel"}, kernels
    assert "maxpool2_kernel" not in kernels, kernels


# N-tiled layers through the TMA-store epilogue: plain slice, 2x2-replicated output, pooled second store (128 -> 256:
# two channel blocks, so the staging tile is used)
CHILD = r"""
import sys, torch
from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import ops
CASES = [
    (2, 36, 64, 128, 256, L.ACT_RELU, L.OUT_F16_NHWC, 0, None),
    (2, 72, 128, 128, 256, L.ACT_SILU, L.OUT_F16_NHWC, 32, None),
    (1, 36, 64, 128, 256, L.ACT_RELU, L.OUT_F16_NHWC_UP2, 0, None),
    (2, 72, 128, 128, 256, L.ACT_RELU, L.OUT_F16_NHWC, 16, L.OUT2_POOL2),
]
res = []
for i, (N, H, W, cin, cout, act, mode, coff, m2) in enumerate(CASES):
    g = torch.Generator().manual_seed(200 + i)
    x = torch.randn(N, H, W, cin, generator=g).half().cuda()
    w = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    wp, bp = ops.pack_conv_weight(w, b, cin, cout, "cuda")
    up = 2 if mode == L.OUT_F16_NHWC_UP2 else 1
    out = torch.full((N, H * up, W * up, cout + coff + 16), 7.0, dtype=torch.float16, device="cuda")
    kw = {}
    if m2 is not None:
        out2 = torch.full((N, H // 2, W // 2, cout + 48), 5.0, dtype=torch.float16, device="cuda")
        kw["out2"] = (out2, 32, m2)
    ops.conv2d(ops.make_conv_desc(x, 0, cin, wp, bp, 3, 1, act, out, coff, mode, cout, None, 0, **kw))
    res.append(out.cpu())
    if m2 is not None:
        res.append(out2.cpu())
torch.cuda.synchronize()
torch.save(res, sys.argv[1])
"""


def _run(tmp_path, on):
    path = tmp_path / f"arm{on}.pt"
    env = dict(os.environ, PADEL_B200_CONV_TMA_STORE=str(on))
    env.pop("PADEL_B200_CONV_HALO", None)
    r = subprocess.run([sys.executable, "-c", CHILD, str(path)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return torch.load(path)


def test_ntiled_tma_store_epilogue_is_bit_identical_to_per_lane_stores(tmp_path):
    a, b = _run(tmp_path, 0), _run(tmp_path, 1)
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16)), f"output {i} differs"
