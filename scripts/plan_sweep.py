"""Per-layer conv plan sweep of the four bench programs on the GPU.

The programs are built exactly as bench.build_trackers builds them (players, pose@1280, court@640, TrackNet; the
bench's sparse-head checkpoints), by default at batch 32 on 1080p frames, and run once so every buffer holds real
activations.  Then, for each conv op, every legal plan (pb_conv_list_plans: the router's kernel, the tunable fields
of pb_conv_plan) is built in place of the op's plan and timed alone with CUDA events.  The candidates are interleaved
in a fresh seeded order in each of --reps rounds; a plan's time is the median of its rounds.  Each candidate's
outputs (the whole primary and secondary output tensors and a fused head's output, so channels outside the op's
slice are covered too) must equal the default plan's bit for bit; a plan that differs is reported and never chosen.

Writes one JSON table (--out): the card name, power limit and SM clocks read in the same run, and per conv op its
shape, the default plan and its time, the best plan and its time, and the spread (max - min over the rounds) of both.

    python scripts/plan_sweep.py --batch 32 --out sweep.json [--programs ball,pose] [--max-plans 400]
"""
from __future__ import annotations

import argparse
import json
import random
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bench  # noqa: E402
from oracle import tracknet as OT  # noqa: E402
from oracle import weights as OW  # noqa: E402
from padel_analytics_b200 import _lib as L  # noqa: E402
from padel_analytics_b200 import synth  # noqa: E402


class _Cai:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": tuple(shape), "typestr": typestr, "version": 2}


def _bytes(ptr: int, n: int) -> torch.Tensor:
    return torch.as_tensor(_Cai(ptr, (n,), "|u1"), device="cuda")


def op_buffers(d) -> list[torch.Tensor]:
    """Byte views of every tensor conv op `d` writes: the whole output (and second output) tensor, the head output."""
    s = d.stride
    Ho, Wo = d.H // s, d.W // s
    bufs = []
    if d.out_mode != L.OUT_NONE:
        up = 2 if d.out_mode == L.OUT_F16_NHWC_UP2 else 1
        esz = 4 if d.out_mode in (L.OUT_F32_NHWC, L.OUT_F32_NCHW) else 2
        ch = d.cout_store if d.out_mode == L.OUT_F32_NCHW else d.out_C
        bufs.append(_bytes(d.out, d.N * Ho * up * Wo * up * ch * esz))
    if d.out2_mode == L.OUT2_UP2:
        bufs.append(_bytes(d.out2, d.N * 4 * Ho * Wo * d.out2_C * 2))
    elif d.out2_mode == L.OUT2_POOL2:
        bufs.append(_bytes(d.out2, d.N * (Ho // 2) * (Wo // 2) * d.out2_C * 2))
    if d.head_n:
        bufs.append(_bytes(d.head_out, d.N * d.head_n * Ho * Wo * 4))
    return bufs


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except Exception as e:  # the table stays usable without it; say why
        return {"error": repr(e)}


def build_programs(B: int, res: str, which):
    """The bench's programs at batch B, each run once on real frames."""
    hw = bench.RES[res]
    ckpts = {"detect": OW.make_yolo("detect", cls_mean=-5.0), "pose13": OW.make_yolo("pose13", cls_mean=-5.7),
             "court12": OW.make_yolo("court12"), "tracknet": OW.make_tracknet()}
    tr, _ = bench.build_trackers(B, hw, ckpts, "cuda")
    fr = synth.make_frames(B, hw[0], hw[1], device="cuda")
    progs = {}
    for k in ("players", "pose", "court"):
        if k in which:
            tr[k].detect_sample(fr)
            progs[k] = list(tr[k].model._progs.values())[0]["prog"]
    if "ball" in which:
        tn = tr["ball"].tracknet
        small = synth.make_frames(B + 7, tn.H, tn.W, start=3)
        med = synth.make_median(tn.H, tn.W)
        xw = torch.from_numpy(OT.assemble_windows([f.numpy() for f in small], med.numpy(), tn.W, tn.H))[:B]
        tn(xw.cuda())
        progs["ball"] = tn.prog
    torch.cuda.synchronize()
    return progs, tr


def time_once(prog, i: int, inner: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(inner):
        prog.run(i, i + 1)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / inner


def sweep_op(prog, i: int, reps: int, inner: int, max_plans: int, rng: random.Random, keep_all: bool) -> dict:
    from padel_analytics_b200.engine.ops import plan_of

    info = prog.op_info(i)
    d = info.desc
    default = plan_of(info)
    bufs = op_buffers(d)
    prog.run(i, i + 1)
    torch.cuda.synchronize()
    ref = [b.clone() for b in bufs]
    plans = prog.conv_plans(i)
    n_legal = len(plans)
    keys = [p.key() for p in plans]
    assert default.key() in keys, f"op {i}: default plan {default} is not in the listed set"
    if len(plans) > max_plans:
        others = [p for p in plans if p.key() != default.key()]
        plans = [default] + rng.sample(others, max_plans - 1)
    times = {p.key(): [] for p in plans}
    differs = set()
    for r in range(reps):
        order = list(plans)
        rng.shuffle(order)
        for p in order:
            prog.set_conv_plan(i, p)
            if r == 0:
                prog.run(i, i + 1)  # warm-up, and the exactness check
                torch.cuda.synchronize()
                if not all(torch.equal(a, b) for a, b in zip(bufs, ref)):
                    differs.add(p.key())
                    for a, b in zip(bufs, ref):
                        a.copy_(b)
            times[p.key()].append(time_once(prog, i, inner))
    prog.set_conv_plan(i, None)
    med = {k: statistics.median(v) for k, v in times.items()}
    ok = [k for k in med if k not in differs]
    best = min(ok, key=lambda k: med[k])
    dk = default.key()
    spread = lambda k: max(times[k]) - min(times[k])  # noqa: E731
    by_key = {p.key(): p for p in plans}
    return dict(
        op=i, variant=info.variant,
        shape=f"N{d.N} {d.H}x{d.W} {d.cin}->{d.cout_pad} k{d.ksize}s{d.stride} out{d.out_mode} out2_{d.out2_mode}",
        desc=dict(N=d.N, H=d.H, W=d.W, C=d.C, cin=d.cin, cout_pad=d.cout_pad, ksize=d.ksize, stride=d.stride,
                  out_mode=d.out_mode, out2_mode=d.out2_mode, head_n=d.head_n, res=bool(d.res), epi=info.epi),
        legal=n_legal, timed=len(plans), differ=[repr(by_key[k]) for k in differs],
        old=repr(default), old_ms=med[dk], old_spread_ms=spread(dk),
        best=repr(by_key[best]), best_plan=dict(zip([f for f, _ in L.ConvPlan._fields_], best)),
        best_ms=med[best], best_spread_ms=spread(best),
        gain=(med[dk] - med[best]) / med[dk],
        wins=med[dk] - med[best] > max(spread(dk), spread(best)),
        all_ms={repr(by_key[k]): v for k, v in med.items()} if keep_all else None,
    )


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--res", default="1080p", choices=list(bench.RES))
    ap.add_argument("--programs", default="ball,players,pose,court")
    ap.add_argument("--ops", default="", help="program:op,... to sweep only these conv ops")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--inner", type=int, default=2, help="launches per timed sample")
    ap.add_argument("--max-plans", type=int, default=100000, help="seeded sample of at most this many plans per op")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--all", action="store_true", help="keep every timed plan's median in the table")
    ap.add_argument("--out", default="plan_sweep.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the sweep times plans on the GPU"
    which = args.programs.split(",")
    only = {}
    for item in filter(None, args.ops.split(",")):
        k, v = item.split(":")
        only.setdefault(k, set()).add(int(v))
    rng = random.Random(args.seed)
    info0 = card()
    progs, _keep = build_programs(args.batch, args.res, which)
    rows = []
    for name in which:
        prog = progs[name]
        for i in range(prog.num_ops):
            if prog.op_info(i).kernel not in (0, 1) or (only and i not in only.get(name, ())):
                continue
            row = sweep_op(prog, i, args.reps, args.inner, args.max_plans, rng, args.all)
            row["program"] = name
            rows.append(row)
            print(f"{name:8s} {i:3d} {row['shape']:48s} old {row['old_ms']*1e3:8.1f} us  best {row['best_ms']*1e3:8.1f} us"
                  f"  {100*row['gain']:5.1f} %  {'WIN ' if row['wins'] else '    '} legal {row['legal']} "
                  f"differ {len(row['differ'])}", flush=True)
            if row["wins"]:
                print(f"         old {row['old']}\n         new {row['best']}", flush=True)
    info1 = card()
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(dict(card_before=info0, card_after=info1, batch=args.batch, res=args.res,
                                              reps=args.reps, inner=args.inner, rows=rows), indent=1))
    tot_old = sum(r["old_ms"] for r in rows)
    tot_win = sum(r["old_ms"] - r["best_ms"] for r in rows if r["wins"])
    print(f"card {info0}\nconv total {tot_old:.3f} ms, sum of wins beyond spread {tot_win:.3f} ms")


if __name__ == "__main__":
    main()
