"""The halo kernel's TMA-store epilogue (PADEL_B200_CONV_TMA_STORE, default on) must write exactly the bits of the
per-lane store epilogue it replaces: same fp32 bias / activation / fp16 rounding, same 2x2 replication and max-pool,
same channel slices.  The switch is read once per process, so each arm runs in a child process."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]

CHILD = r"""
import sys, torch
from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import ops
# N, H, W, cin, cout, k, s, act, out_mode, out_coff, out2 mode
CASES = [
    (2, 40, 72, 64, 64, 3, 1, L.ACT_RELU, L.OUT_F16_NHWC, 0, None),
    (2, 36, 44, 128, 128, 3, 1, L.ACT_SILU, L.OUT_F16_NHWC, 32, None),
    (3, 24, 40, 32, 16, 3, 1, L.ACT_SILU, L.OUT_F16_NHWC, 16, None),
    (2, 24, 40, 48, 32, 3, 1, L.ACT_SIGMOID, L.OUT_F16_NHWC, 8, None),
    (2, 24, 40, 32, 48, 3, 1, L.ACT_NONE, L.OUT_F16_NHWC, 0, None),
    (1, 20, 36, 64, 192, 3, 1, L.ACT_SILU, L.OUT_F16_NHWC, 0, None),
    (2, 32, 48, 64, 128, 3, 1, L.ACT_RELU, L.OUT_F16_NHWC_UP2, 0, None),
    (2, 30, 52, 64, 64, 3, 1, L.ACT_RELU, L.OUT_F16_NHWC, 16, L.OUT2_POOL2),
    (2, 36, 44, 32, 48, 3, 1, L.ACT_RELU, L.OUT_F16_NHWC, 0, L.OUT2_POOL2),
    (2, 16, 32, 64, 64, 3, 1, L.ACT_SILU, L.OUT_F16_NHWC, 0, L.OUT2_UP2),
    (2, 40, 56, 32, 32, 1, 1, L.ACT_SILU, L.OUT_F16_NHWC, 32, None),
    (2, 48, 80, 16, 32, 3, 2, L.ACT_SILU, L.OUT_F16_NHWC, 0, None),
    (2, 48, 80, 32, 64, 3, 2, L.ACT_SILU, L.OUT_F16_NHWC, 0, None),
]
res = []
for i, (N, H, W, cin, cout, k, s, act, mode, coff, m2) in enumerate(CASES):
    g = torch.Generator().manual_seed(100 + i)
    x = torch.randn(N, H, W, cin, generator=g).half().cuda()
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    wp, bp = ops.pack_conv_weight(w, b, cin, cout, "cuda")
    up = 2 if mode == L.OUT_F16_NHWC_UP2 else 1
    out = torch.full((N, H // s * up, W // s * up, cout + coff + 16), 7.0, dtype=torch.float16, device="cuda")
    kw = {}
    if m2 is not None:
        shape2 = (N, 2 * H, 2 * W) if m2 == L.OUT2_UP2 else (N, H // 2, W // 2)
        out2 = torch.full((*shape2, cout + 48), 5.0, dtype=torch.float16, device="cuda")
        kw["out2"] = (out2, 32, m2)
    ops.conv2d(ops.make_conv_desc(x, 0, cin, wp, bp, k, s, act, out, coff, mode, cout, None, 0, **kw))
    res.append(out.cpu())
    if m2 is not None:
        res.append(out2.cpu())
torch.cuda.synchronize()
torch.save(res, sys.argv[1])
"""


def _run(tmp_path, on):
    path = tmp_path / f"arm{on}.pt"
    env = dict(os.environ, PADEL_B200_CONV_TMA_STORE=str(on))
    r = subprocess.run([sys.executable, "-c", CHILD, str(path)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return torch.load(path)


def test_tma_store_epilogue_is_bit_identical_to_per_lane_stores(tmp_path):
    a, b = _run(tmp_path, 0), _run(tmp_path, 1)
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16)), f"output {i} differs"
