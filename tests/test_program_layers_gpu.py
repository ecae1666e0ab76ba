"""Layer-by-layer replay of the shipped programs against float64 references, and their grid-size / PDL invariance.

The four programs bench.py measures (players, pose@1280, court@640, TrackNet; built like scripts/layer_table.py) and
the ResNet50 court regressor are built at batch 2 on 1080p frames and run once end to end, so every buffer holds real
activations.  Then every op runs alone (`Program.run(i, i + 1)`) on a snapshot of its inputs:
  - conv ops through the comparator of tests/conv_ref.py (per-element ulp bound, rounding statistics, untouched
    channels, exact second outputs);
  - sppf / maxpool2 / upsample2 exactly against float64 pooling, the pointwise head like an fp32 conv output;
  - the ResNet engine's direct kernels (7x7 stem, 3x3/s2 max-pool, avgpool + fc + sigmoid) the same way.
TrackNet with separate pool launches and the CUDA-core head, and YOLO with separate upsample launches, are replayed
too: they bring maxpool2, upsample2 and the pointwise head in at their real shapes.

Each op's outputs are kept, and every program is rebuilt for 1 and 5 SMs and without PDL: a conv's accumulation order
per output does not depend on which CTA computes it, so every op of the rebuilt program (and the ResNet engine's
direct kernels) must reproduce them bit for bit.
"""
from __future__ import annotations

import functools

import pytest
import torch
import torch.nn.functional as F

import bench
import conv_ref as R
from oracle import resnet as OR
from oracle import tracknet as OT
from oracle import weights as OW
from padel_analytics_b200 import _lib as L
from padel_analytics_b200 import synth
from padel_analytics_b200.engine.resnet_engine import ResNet50Engine
from padel_analytics_b200.engine.tracknet_engine import TrackNetEngine

pytestmark = pytest.mark.gpu

B = 2
KINDS = {0: "conv", 1: "conv", 2: "maxpool2", 3: "upsample2", 4: "sppf", 5: "head"}


# ---- per-op replay ----------------------------------------------------------------------------------------------
def op_outputs(info) -> list[torch.Tensor]:
    """Views of everything op `info` writes."""
    if info.kernel in (0, 1):
        d = info.desc
        v = R.conv_views(d)
        outs = [v["out"] if d.out_mode == L.OUT_F32_NCHW else v["out"][..., d.out_coff:d.out_coff + d.cout_store]]
        if v["out2"] is not None:
            outs.append(v["out2"][..., d.out2_coff:d.out2_coff + d.cout_store])
        return outs
    N, H, W, c = info.N, info.H, info.W, info.c
    if info.kernel == 2:
        return [R.view(info.out, (N, H // 2, W // 2, info.out_C))[..., info.out_coff:info.out_coff + c]]
    if info.kernel == 3:
        return [R.view(info.out, (N, 2 * H, 2 * W, info.out_C))[..., info.out_coff:info.out_coff + c]]
    if info.kernel == 4:
        return [R.view(info.in_, (N, H, W, info.C))[..., c:4 * c]]
    return [R.view(info.out, (N, c, H, W), torch.float32)]


def _exact(got, exp, what, fails):
    if not torch.equal(got.to(torch.float64), exp.to(torch.float64)):
        bad = got.to(torch.float64) != exp.to(torch.float64)
        fails.append(f"{what}: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}")


def _unchanged(before, after, keep, what, fails):
    if keep.any() and not torch.equal(before[..., keep].view(torch.int16), after[..., keep].view(torch.int16)):
        fails.append(f"{what}: channels outside the op's slice changed")


def check_aux(prog, i, info) -> R.ConvReport:
    """Run aux op i alone and check it exactly (pools, upsample) or like an fp32 conv output (pointwise head)."""
    rep = R.ConvReport()
    N, H, W, C, c = info.N, info.H, info.W, info.C, info.c
    if info.kernel == 4:  # sppf: slice 0 of buf is x', slices 1..3 receive the chained pools
        buf = R.view(info.in_, (N, H, W, C))
        before = buf.clone()
        prog.run(i, i + 1)
        for k, y in enumerate(R.sppf_reference(before[..., :c]), start=1):
            _exact(buf[..., k * c:(k + 1) * c], y, f"sppf slice {k}", rep.fails)
        keep = torch.ones(C, dtype=torch.bool, device=buf.device)
        keep[c:4 * c] = False
        _unchanged(before, buf, keep, "sppf", rep.fails)
        rep.n = N * H * W * 3 * c
        return rep
    if info.kernel == 5:  # pointwise head: 1x1 conv C -> c, bias, sigmoid, fp32 NCHW
        x = R.view(info.in_, (N, H, W, C)).clone()
        w = R.view(info.weight, (c, C), torch.float32).to(torch.float64)
        b = R.view(info.bias, (c,), torch.float32).to(torch.float64)
        out = R.view(info.out, (N, c, H, W), torch.float32)
        prog.run(i, i + 1)
        x64 = x.to(torch.float64)
        ref = torch.sigmoid(torch.einsum("nhwc,jc->njhw", x64, w) + b.view(1, c, 1, 1))
        A = torch.einsum("nhwc,jc->njhw", x64.abs(), w.abs()) + b.abs().view(1, c, 1, 1)
        return R.compare_values(out, ref, A, rep)
    x = R.view(info.in_, (N, H, W, C))
    up = info.kernel == 3
    Ho, Wo = (2 * H, 2 * W) if up else (H // 2, W // 2)
    out = R.view(info.out, (N, Ho, Wo, info.out_C))
    xs, before = x[..., info.c_off:info.c_off + c].clone(), out.clone()
    prog.run(i, i + 1)
    exp = xs.repeat_interleave(2, 1).repeat_interleave(2, 2) if up else R.pool2_exact(xs)
    _exact(out[..., info.out_coff:info.out_coff + c], exp, KINDS[info.kernel], rep.fails)
    keep = torch.ones(info.out_C, dtype=torch.bool, device=out.device)
    keep[info.out_coff:info.out_coff + c] = False
    _unchanged(before, out, keep, KINDS[info.kernel], rep.fails)
    rep.n = exp.numel()
    return rep


def replay(prog, label: str):
    """Run every op of `prog` alone and check it.  Returns (rows, outputs, plans): one printable row per op, a copy of
    each op's outputs, and the plan of each conv op."""
    rows, outs, plans, fails = [], [], [], []
    torch.cuda.synchronize()
    for i in range(prog.num_ops):
        info = prog.op_info(i)
        if info.kernel in (0, 1):
            d = info.desc
            v = R.conv_views(d)
            before = R.snapshot(v)
            prog.run(i, i + 1)
            rep = R.check_conv(d, before, {"out": v["out"], "out2": v["out2"]})
            sig = R.describe_plan(info)
            shape = f"{d.H}x{d.W} {d.cin}->{d.cout_pad} k{d.ksize}s{d.stride}"
            plans.append(info)
        else:
            rep = check_aux(prog, i, info)
            sig, shape = KINDS[info.kernel], f"{info.H}x{info.W} c{info.c}"
        outs.append([t.clone() for t in op_outputs(info)])
        rows.append(dict(i=i, shape=shape, plan=sig, rep=rep))
        print(f"{label:9s} {i:3d} {shape:26s} {sig:70s} {rep.row()}")
        fails += [f"{label} op {i} ({shape}, {sig}): {f}" for f in rep.fails]
    torch.cuda.synchronize()
    return rows, outs, plans, fails


def summary(label: str, rows) -> str:
    reps = [r["rep"] for r in rows]
    return (f"{label}: {len(rows)} ops, worst {max(r.max_ulps for r in reps):.2f} ulp, worst tolerance use "
            f"{max(r.max_tol_ratio for r in reps):.3f}, worst mismatch {max(r.mismatch for r in reps):.4f}, "
            f"worst |bias| {max(abs(r.bias) for r in reps):.4f}, worst tolerance / old tolerance "
            f"{max(r.max_old_ratio for r in reps):.3f}")


def replay_same(prog, ref_outs, label: str) -> list[str]:
    """Run `prog` (a rebuild of a replayed program on its own buffers) op by op and compare every op's outputs bit
    for bit with `ref_outs`."""
    fails = []
    for i in range(prog.num_ops):
        prog.run(i, i + 1)
        for k, (got, exp) in enumerate(zip(op_outputs(prog.op_info(i)), ref_outs[i])):
            if not torch.equal(got.view(torch.int16) if got.dtype == torch.float16 else got.view(torch.int32),
                               exp.view(torch.int16) if exp.dtype == torch.float16 else exp.view(torch.int32)):
                fails.append(f"{label}: op {i} output {k} differs from the default build")
                return fails  # later ops read it: their differences would follow from this one
    return fails


# ---- the shipped programs ---------------------------------------------------------------------------------------
@functools.cache
def shipped():
    """The four bench programs and the ResNet50 engine at batch 2, 1080p, after one real forward each."""
    hw = bench.RES["1080p"]
    ckpts = {k: OW.make_yolo(k) for k in ("detect", "pose13", "court12")}
    ckpts["tracknet"] = OW.make_tracknet()
    tr, _ = bench.build_trackers(B, hw, ckpts, "cuda")
    fr = synth.make_frames(B, hw[0], hw[1], device="cuda")
    yolo = {}
    for k in ("players", "pose", "court"):
        tr[k].detect_sample(fr)  # builds the program for the input size and runs it on the frames
        eng = tr[k].model
        key = list(eng._progs)[0]
        yolo[k] = (eng, key)
    tn = tr["ball"].tracknet
    small = synth.make_frames(B + 7, tn.H, tn.W, start=3)
    med = synth.make_median(tn.H, tn.W)
    xw = torch.from_numpy(OT.assemble_windows([f.numpy() for f in small], med.numpy(), tn.W, tn.H))[:B]
    tn(xw.cuda())
    sd = OR.make_resnet50_court()
    rn = ResNet50Engine(sd, max_batch=B)
    rn.predict_frames([f.numpy() for f in synth.make_frames(B, hw[0], hw[1], start=5)])
    torch.cuda.synchronize()
    return dict(yolo=yolo, tracknet=tn, tracknet_ckpt=ckpts["tracknet"], resnet=rn, resnet_sd=sd)


def programs():
    s = shipped()
    progs = {k: eng._progs[key]["prog"] for k, (eng, key) in s["yolo"].items()}
    progs["tracknet"] = s["tracknet"].prog
    progs["resnet"] = s["resnet"].prog
    return progs


def resnet_direct(eng, check: bool, ref_prog_outs=None, label: str = "resnet"):
    """Run the ResNet engine's stem, max-pool, bottleneck program (op by op) and avgpool-fc-sigmoid on eng.x_in; with
    `check`, compare the three direct kernels with float64 references; with `ref_prog_outs`, compare every op of the
    bottleneck program bit for bit with them (replay_same).  Returns ([stem, max-pool, fc outputs], failures)."""
    lib, st, fails = L.lib(), L.stream_ptr(), []
    x = eng.x_in.clone()
    L.check(lib.pb_resnet_stem7x7(eng.x_in.data_ptr(), B, 224, 224, eng.w_stem.data_ptr(), eng.b_stem.data_ptr(),
                                  eng.c1.data_ptr(), st))
    L.check(lib.pb_maxpool3x3s2(eng.c1.data_ptr(), B, 112, 112, 64, eng.p1.data_ptr(), st))
    if ref_prog_outs is not None:
        fails += replay_same(eng.prog, ref_prog_outs, label)
    else:
        for i in range(eng.prog.num_ops):
            eng.prog.run(i, i + 1)
    L.check(lib.pb_avgpool_fc_sigmoid(eng.feat.data_ptr(), B, eng.feat_hw, eng.feat_c, eng.fc_w.data_ptr(),
                                      eng.fc_b.data_ptr(), eng.n_out, eng.out.data_ptr(), st))
    torch.cuda.synchronize()
    if check:
        stem_rep = check_stem7x7(x, eng.w_stem, eng.b_stem, eng.c1)
        fails += [f"resnet stem7x7: {f}" for f in stem_rep.fails]
        _exact(eng.p1, R.maxpool_nhwc(eng.c1, 3, 2, 1), "resnet maxpool3x3s2", fails)
        fc_rep = check_avgpool_fc(eng.feat, eng.fc_w, eng.fc_b, eng.out)
        fails += [f"resnet avgpool_fc_sigmoid: {f}" for f in fc_rep.fails]
        print("resnet stem7x7", stem_rep.row())
        print("resnet avgpool_fc_sigmoid", fc_rep.row())
    return [eng.c1.clone(), eng.p1.clone(), eng.out.clone()], fails


def check_stem7x7(x, w_stem, b_stem, out) -> R.ConvReport:
    """conv 7x7 / s2 / p3 over channels 0..2 of x (fp16) with fp32 weights [(r*7+s)*3+c][64], bias, ReLU."""
    x64 = x[..., :3].to(torch.float64).permute(0, 3, 1, 2)
    w64 = w_stem.to(torch.float64).reshape(7, 7, 3, 64).permute(3, 2, 0, 1)
    b64 = b_stem.to(torch.float64)
    ref = F.conv2d(x64, w64, stride=2, padding=3).permute(0, 2, 3, 1) + b64
    A = F.conv2d(x64.abs(), w64.abs(), stride=2, padding=3).permute(0, 2, 3, 1) + b64.abs()
    return R.compare_values(out, ref.clamp_min(0), A, R.ConvReport())


def check_avgpool_fc(feat, w, b, out) -> R.ConvReport:
    """sigmoid(mean over pixels of feat (N, HW, C) @ w^T + b) in float64."""
    n = feat.shape[0]
    f64 = feat.reshape(n, -1, feat.shape[-1]).to(torch.float64)
    w64, b64 = w.to(torch.float64), b.to(torch.float64)
    ref = torch.sigmoid(f64.mean(1) @ w64.T + b64)
    A = f64.abs().mean(1) @ w64.abs().T + b64.abs()
    return R.compare_values(out, ref, A, R.ConvReport())


@functools.cache
def replayed():
    """Replay every shipped program once: {name: (rows, outs, plans, fails)}."""
    return {name: replay(p, name) for name, p in programs().items()}


# ---- tests ------------------------------------------------------------------------------------------------------
def test_every_layer_of_the_shipped_programs_matches_float64():
    res = replayed()
    fails = [f for v in res.values() for f in v[3]]
    for name, (rows, _, _, _) in res.items():
        print(summary(name, rows))
    _, f2 = resnet_direct(shipped()["resnet"], check=True)
    assert not fails + f2, "\n".join((fails + f2)[:40])


def test_separate_pool_upsample_and_pointwise_head_launches_match_float64(monkeypatch):
    """TrackNet with PADEL_B200_FUSE_OUT2=0 and the CUDA-core head, YOLO with PADEL_B200_FUSE_OUT2=0: maxpool2,
    upsample2 and the pointwise head at their real shapes, on the activations of the shipped programs."""
    s = shipped()
    monkeypatch.setenv("PADEL_B200_FUSE_OUT2", "0")
    monkeypatch.setenv("PADEL_B200_TRACKNET_HEAD", "pointwise")
    tn = TrackNetEngine(s["tracknet_ckpt"]["model"], max_batch=B)
    tn.x.copy_(s["tracknet"].x)
    eng, key = s["yolo"]["players"]
    st = eng._build(*key)
    st["x0"].copy_(eng._progs[key]["x0"])
    fails, kinds = [], set()
    for name, prog in (("tracknet0", tn.prog), ("players0", st["prog"])):
        kinds |= {prog.op_info(i).kernel for i in range(prog.num_ops)}
        rows, _, _, f = replay(prog, name)
        print(summary(name, rows))
        fails += f
    assert {2, 3, 4, 5} <= kinds, kinds
    assert not fails, "\n".join(fails[:40])


def _with_plan_options(sm_limit, pdl, fn):
    """fn() with pb_set_plan_options(sm_limit, pdl) in force: plans capture it when built, and the aux kernels size
    their grids from it when launched."""
    L.lib().pb_set_plan_options(sm_limit, pdl)
    try:
        return fn()
    finally:
        L.lib().pb_set_plan_options(0, -1)


@pytest.mark.parametrize("opts", [(1, -1), (5, -1), (0, 0)], ids=lambda o: f"sms{o[0]}-pdl{o[1]}")
def test_yolo_and_resnet_outputs_do_not_depend_on_grid_size_or_pdl(opts):
    s, ref = shipped(), replayed()
    sms, pdl = opts
    fails = []
    for name, (eng, key) in s["yolo"].items():
        def run():
            st = eng._build(*key)
            st["x0"].copy_(eng._progs[key]["x0"])
            _check_options(st["prog"], sms, pdl, name, fails)
            return replay_same(st["prog"], ref[name][1], f"{name} {opts}")
        fails += _with_plan_options(sms, pdl, run)
    base = s["resnet"]
    base_outs, _ = resnet_direct(base, check=False)

    def run_resnet():
        e = ResNet50Engine(s["resnet_sd"], max_batch=B)
        e.x_in.copy_(base.x_in)
        _check_options(e.prog, sms, pdl, "resnet", fails)
        return resnet_direct(e, check=False, ref_prog_outs=ref["resnet"][1], label=f"resnet {opts}")

    outs, prog_fails = _with_plan_options(sms, pdl, run_resnet)
    fails += prog_fails
    for what, got, exp in zip(("stem7x7", "maxpool3x3s2", "avgpool_fc_sigmoid"), outs, base_outs):
        if not torch.equal(got, exp):
            fails.append(f"resnet {opts}: {what} output differs from the default build")
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("sms", [1, 5])
def test_tracknet_outputs_do_not_depend_on_ball_sms(sms, monkeypatch):
    """PADEL_B200_BALL_SMS=n builds TrackNet for n SMs with PDL off (TrackNetEngine._build sets and resets the plan
    options itself)."""
    s, ref = shipped(), replayed()
    monkeypatch.setenv("PADEL_B200_BALL_SMS", str(sms))
    tn = TrackNetEngine(s["tracknet_ckpt"]["model"], max_batch=B)
    tn.x.copy_(s["tracknet"].x)
    fails = []
    _check_options(tn.prog, sms, 0, "tracknet", fails)
    fails += replay_same(tn.prog, ref["tracknet"][1], f"tracknet BALL_SMS={sms}")
    assert not fails, "\n".join(fails)


def _check_options(prog, sms, pdl, name, fails):
    """The rebuilt program's conv plans did capture the options (grids of at most `sms` CTAs, PDL as asked)."""
    for i in range(prog.num_ops):
        info = prog.op_info(i)
        if info.kernel in (0, 1):
            if (sms > 0 and info.grid > sms) or (pdl == 0 and info.pdl != 0):
                fails.append(f"{name} op {i}: plan grid {info.grid} pdl {info.pdl} ignores the options ({sms}, {pdl})")
                return
