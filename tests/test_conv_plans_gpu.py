"""Plan coverage of the conv kernels: a synthetic sweep over the plan edges the shipped programs do not reach, every
case checked with the float64 comparator of tests/conv_ref.py; the union of the plans reached by the sweep and by the
replay of the shipped programs (tests/test_program_layers_gpu.py) must cover a declared set of values on every plan
axis; the sweep holds under the static A/B switches and is bit-identical when built for 1 / 5 SMs or without PDL."""
from __future__ import annotations

import functools
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

import conv_ref as R
import test_program_layers_gpu as replay
from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine import ops

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
RELU, SILU, NONE, SIG = L.ACT_RELU, L.ACT_SILU, L.ACT_NONE, L.ACT_SIGMOID

# name -> layer.  Defaults: N = 1, 3x3 stride 1, SiLU, whole input tensor, output slice at channel 0 of a tensor as
# wide as the layer.  c_total / c_in_off: input tensor width / first channel read; out_C / out_coff: output slice;
# res = (res_C, res_coff); pool / up2 = second output (PB_OUT2_POOL2 / UP2); store = cout_store.
SWEEP = {
    # warpgroup skip (Ho % 16 in 1..8) and partial last tile rows (9..15); Wo % 8S != 0
    "skip8-w20": dict(H=40, W=20, cin=32, cout=32),
    "skip4-w44": dict(H=20, W=44, cin=64, cout=64, act=RELU),
    "skip1": dict(H=17, W=24, cin=16, cout=48),
    "part12-w100": dict(H=12, W=100, cin=32, cout=96, act=RELU),
    "part14": dict(N=2, H=30, W=36, cin=48, cout=16),
    # N tiles on ragged heights / widths
    "ntile-skip": dict(N=2, H=24, W=64, cin=128, cout=256, act=RELU),
    "ntile-part": dict(H=28, W=64, cin=256, cout=512, act=RELU),
    "ntile-s1": dict(H=40, W=40, cin=64, cout=384, act=RELU),
    # resident banks with many channel blocks; deep streamed K (third halo stage)
    "res-7blocks": dict(H=24, W=40, cin=112, cout=48),
    "res-7blocks-a4": dict(H=24, W=40, cin=112, cout=48, res=(48, 0)),
    "res-3blocks": dict(H=32, W=32, cin=192, cout=32, act=RELU),
    "stream-k12": dict(H=20, W=64, cin=768, cout=64, act=RELU),
    "stream-g3": dict(H=24, W=48, cin=128, cout=64),
    "stream-g9": dict(H=24, W=40, cin=128, cout=64, act=RELU),
    "stream-bn192": dict(H=16, W=24, cin=256, cout=192, act=RELU),
    # TMA store at S = 4 / 2 / 1, with and without the pooled second store; UP2 outputs; slices
    "tma-s4": dict(N=2, H=64, W=64, cin=32, cout=64),
    "tma-s4-pool": dict(H=32, W=64, cin=32, cout=64, act=RELU, pool=True),
    "tma-s2": dict(H=48, W=48, cin=64, cout=128, act=RELU),
    "tma-s2-pool": dict(H=36, W=64, cin=64, cout=128, act=RELU, pool=True),
    "tma-s1": dict(H=16, W=24, cin=32, cout=192),
    "tma-s1-pool": dict(H=16, W=16, cin=32, cout=192, act=RELU, pool=True),
    "ntile-pool": dict(H=16, W=16, cin=32, cout=256, act=RELU, pool=True),
    "tma-up2": dict(H=24, W=40, cin=64, cout=64, act=RELU, mode=L.OUT_F16_NHWC_UP2),
    "tma-slices": dict(N=2, H=20, W=28, cin=64, cout=64, c_total=160, c_in_off=64, out_C=192, out_coff=96),
    "many-tiles": dict(N=2, H=160, W=256, cin=64, cout=64, act=RELU),
    # per-lane epilogue: residual after / before the activation, unaligned slices, cout_store < cout_pad
    "silu-res": dict(H=40, W=40, cin=64, cout=64, res=(128, 64)),
    "silu-res-s2": dict(H=20, W=32, cin=64, cout=128, res=(128, 0)),
    "relu-res-first": dict(k=1, H=14, W=14, cin=64, cout=256, act=RELU, res=(256, 0), res_first=True),
    "slice8": dict(H=20, W=20, cin=32, cout=32, out_C=56, out_coff=8),
    "store40": dict(H=20, W=24, cin=32, cout=48, store=40, out_C=40),
    "sigmoid-none": dict(H=16, W=16, cin=32, cout=32, act=SIG),
    "none-act": dict(H=16, W=16, cin=32, cout=32, act=NONE),
    # halo 1x1 (cin <= 32), at W <= 8 (S = 1) and wider; second output UP2
    "1x1-w8": dict(k=1, H=16, W=8, cin=32, cout=64),
    "1x1-w4": dict(k=1, N=2, H=6, W=4, cin=16, cout=32),
    "1x1-wide": dict(k=1, H=40, W=72, cin=32, cout=32),
    "1x1-up2": dict(k=1, H=20, W=20, cin=32, cout=64, up2=True),
    # halo stride 2 (whole C = 16 / 32 tensor)
    "s2-c16": dict(s=2, H=40, W=72, cin=16, cout=32),
    "s2-c32": dict(s=2, H=34, W=50, cin=32, cout=64),
    "s2-c32-wide": dict(s=2, H=32, W=32, cin=32, cout=160),
    # stem (PB_IN_STEM4) at cout 16 .. 128
    "stem16": dict(stem=True, H=34, W=50, cout=16),
    "stem48": dict(stem=True, H=64, W=96, cout=48),
    "stem80": dict(stem=True, H=32, W=40, cout=80),
    "stem128": dict(stem=True, H=36, W=36, cout=128),
    # per-tap kernel: N tiles at cout 1024 / 2048, stride 2, wide 3x3, fp32 1x1 (PB_EPI_F32), fp32 NCHW head
    "tap-1024": dict(k=1, H=14, W=14, cin=256, cout=1024, act=RELU),
    "tap-2048": dict(k=1, s=2, H=14, W=14, cin=512, cout=2048, act=NONE),
    "tap-s2-c64": dict(s=2, H=20, W=36, cin=64, cout=128),
    "tap-3x3-320": dict(H=12, W=20, cin=64, cout=320, act=RELU),
    "tap-1x1-c64": dict(k=1, H=24, W=40, cin=64, cout=96),
    "tap-f32": dict(k=1, H=20, W=20, cin=64, cout=80, act=NONE, mode=L.OUT_F32_NHWC, store=72, out_C=160, out_coff=8),
    "tap-f32-nchw": dict(k=1, H=12, W=20, cin=64, cout=16, act=SIG, mode=L.OUT_F32_NCHW, store=8),
}

# Values every plan axis must reach in the union of the sweep and the shipped programs' replay (conv_ref.plan_key).
REQUIRED = {
    "variant": {L.CONV_PER_TAP, L.CONV_HALO, L.CONV_HALO_1X1, L.CONV_HALO_S2, L.CONV_STEM},
    "epi": {0, 1, 2, 3, 4},
    "S": {1, 2, 4},
    "KB": {16, 32, 64},
    "G": {1, 3, 9},
    "b_resident": {0, 1},
    "a_stages": {2, 3, 4},
    "ntiled": {False, True},
    "tma_store": {0, 1},
    "st_pool": {0, 1},
    "tma_S": {(1, 1), (1, 2), (1, 4), (0, 1), (0, 2), (0, 4)},
    "ho16": {"skip", "partial", "whole"},
    "ntile_ragged": {True},
    "w_ragged": {True},
    "tap_ntiles": {1, 2, 4, 8},
    "stem_BN": {16, 48, 80, 128},
    "cout_store_lt_pad": {True},
}


def build_case(c: dict, seed: int = 0):
    """Tensors and descriptor of sweep case `c` (output buffers pre-filled with a marker)."""
    g = torch.Generator().manual_seed(seed)
    N, H, W, k, s = c.get("N", 1), c["H"], c["W"], c.get("k", 3), c.get("s", 1)
    cout, act = c["cout"], c.get("act", SILU)
    Ho, Wo = H // s, W // s
    if c.get("stem"):
        x = torch.zeros(N, H + 2, W + 2, 4)
        x[:, 1:-1, 1:-1, :3] = torch.rand(N, H, W, 3, generator=g)
        x = x.half().cuda()
        wp, bp = ops.pack_stem_weight(torch.randn(cout, 3, 3, 3, generator=g) / 5, torch.randn(cout, generator=g) * 0.2,
                                      cout, "cuda")
        out = torch.full((N, Ho, Wo, cout), 7.0, dtype=torch.float16, device="cuda")
        return ops.make_stem_desc(x, wp, bp, act, out), [x, wp, bp, out]
    cin = c["cin"]
    C, coff = c.get("c_total", cin), c.get("c_in_off", 0)
    x = (torch.randn(N, H, W, C, generator=g)).half().cuda()
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    wp, bp = ops.pack_conv_weight(w, torch.randn(cout, generator=g) * 0.2, cin, cout, "cuda")
    mode = c.get("mode", L.OUT_F16_NHWC)
    store = c.get("store", cout)
    out_coff = c.get("out_coff", 0)
    out_C = c.get("out_C", out_coff + store)
    if mode == L.OUT_F32_NCHW:
        out = torch.full((N, store, Ho, Wo), 7.0, device="cuda")
    elif mode == L.OUT_F32_NHWC:
        out = torch.full((N, Ho, Wo, out_C), 7.0, device="cuda")
    else:
        up = 2 if mode == L.OUT_F16_NHWC_UP2 else 1
        out = torch.full((N, Ho * up, Wo * up, out_C), 7.0, dtype=torch.float16, device="cuda")
    res = None
    if "res" in c:
        res = torch.randn(N, Ho, Wo, c["res"][0], generator=g).half().cuda()
    out2 = None
    if c.get("pool"):
        out2 = (torch.full((N, Ho // 2, Wo // 2, store + 32), 5.0, dtype=torch.float16, device="cuda"), 16, L.OUT2_POOL2)
    elif c.get("up2"):
        out2 = (torch.full((N, 2 * Ho, 2 * Wo, store + 16), 5.0, dtype=torch.float16, device="cuda"), 16, L.OUT2_UP2)
    d = ops.make_conv_desc(x, coff, cin, wp, bp, k, s, act, out, out_coff, mode, store, res,
                           c["res"][1] if res is not None else 0, res_before_act=c.get("res_first", False), out2=out2)
    keep = [x, wp, bp, out, res, None if out2 is None else out2[0]]
    return d, keep


def run_case(name: str):
    """Build, run and check sweep case `name` as a one-op program: (report, plan info, copies of its outputs)."""
    d, keep = build_case(SWEEP[name])
    p = ops.Program()
    p.conv(d)
    p.keep(*[t for t in keep if t is not None])
    info = p.op_info(0)
    v = R.conv_views(info.desc)
    before = R.snapshot(v)
    p.run()
    rep = R.check_conv(info.desc, before, {"out": v["out"], "out2": v["out2"]})
    outs = [t.clone() for t in replay.op_outputs(info)]
    return rep, info, outs


@functools.cache
def sweep():
    res = {}
    for name in SWEEP:
        rep, info, outs = run_case(name)
        print(f"{name:14s} {R.describe_plan(info):70s} {rep.row()}")
        res[name] = (rep, info, outs)
    torch.cuda.synchronize()
    return res


def test_sweep_cases_match_float64():
    fails = [f"{n}: {f}" for n, (rep, _, _) in sweep().items() for f in rep.fails]
    assert not fails, "\n".join(fails)


def test_sweep_and_shipped_programs_cover_every_plan_axis():
    keys = [R.plan_key(info) for _, info, _ in sweep().values()]
    for name, (_, _, plans, _) in replay.replayed().items():
        keys += [R.plan_key(info) for info in plans]
    reached = {axis: set() for axis in REQUIRED}
    for k in keys:
        for axis in REQUIRED:
            if axis in k:
                reached[axis].add(k[axis])
    for axis in REQUIRED:
        print(f"{axis:18s} {sorted(reached[axis], key=str)}")
    missing = {a: REQUIRED[a] - reached[a] for a in REQUIRED if REQUIRED[a] - reached[a]}
    assert not missing, f"plan values no longer reached (update the sweep table): {missing}"


@pytest.mark.parametrize("opts", [(1, -1), (5, -1), (0, 0)], ids=lambda o: f"sms{o[0]}-pdl{o[1]}")
def test_sweep_outputs_do_not_depend_on_grid_size_or_pdl(opts):
    ref = sweep()
    fails = []
    L.lib().pb_set_plan_options(*opts)
    try:
        for name in SWEEP:
            _, info, outs = run_case(name)
            if (opts[0] > 0 and info.grid > opts[0]) or (opts[1] == 0 and info.pdl != 0):
                fails.append(f"{name}: grid {info.grid} pdl {info.pdl} ignores the plan options {opts}")
            for k, (got, exp) in enumerate(zip(outs, ref[name][2])):
                if not torch.equal(got, exp):
                    fails.append(f"{name}: output {k} differs from the default build")
    finally:
        L.lib().pb_set_plan_options(0, -1)
    assert not fails, "\n".join(fails)


# The static A/B switches are read once per process: each arm runs the sweep in a child process of its own.
AB_ARMS = {"PADEL_B200_CONV_BRES": "0", "PADEL_B200_STEM_RAW": "0", "PADEL_B200_CONV_EPI": "0",
           "PADEL_B200_CONV_HALO1": "2"}


def test_sweep_holds_under_every_static_ab_switch():
    procs = {}
    for var, val in AB_ARMS.items():
        env = dict(os.environ, **{var: val})
        cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", "-s",
               f"tests/{Path(__file__).name}::test_sweep_cases_match_float64"]
        procs[var] = subprocess.Popen(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True)
    fails = []
    try:
        for var, p in procs.items():
            out, _ = p.communicate(timeout=1200)
            print(f"== {var}={AB_ARMS[var]}\n{out[-6000:]}")
            if p.returncode != 0:
                fails.append(f"{var}={AB_ARMS[var]}: exit {p.returncode}\n{out[-3000:]}")
    finally:
        for p in procs.values():  # none outlives the test, whatever happened above
            if p.poll() is None:
                p.kill()
            p.wait()
    assert not fails, "\n".join(fails)
