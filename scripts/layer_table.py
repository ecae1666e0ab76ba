"""Per-layer device times of the four bench programs (TrackNet, detect, pose@1280, court@640) at bench shapes.

    python scripts/layer_table.py [--batch 32] [--json OUT.json]

Run from the repository root (the package is imported from the current directory).  Every op is timed with CUDA
events on the launch stream between consecutive ops, median of 5 passes (engine.ops.time_program_ops, the same timing
bench.py's roofline uses).  One row per op: kernel, conv shape, ms, algorithmic TFLOP/s and GB/s.
"""
import argparse
import json
import sys

import torch

sys.path.insert(0, ".")
import bench  # noqa: E402
from oracle import weights as OW  # noqa: E402
from padel_analytics_b200 import synth  # noqa: E402
from padel_analytics_b200.engine import ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json", help="write the table here as JSON")
    args = ap.parse_args()
    B, hw = args.batch, bench.RES["1080p"]
    ckpts = {k: OW.make_yolo(k) for k in ("detect", "pose13", "court12")}
    ckpts["tracknet"] = OW.make_tracknet()
    tr, _ = bench.build_trackers(B, hw, ckpts, "cuda")
    fr = synth.make_frames(B, hw[0], hw[1], device="cuda")
    for k in ("players", "pose", "court"):
        tr[k].detect_sample(fr)  # builds the program for the input size
    progs = {"tracknet": tr["ball"].tracknet.prog}
    for k in ("players", "pose", "court"):
        progs[k] = list(tr[k].model._progs.values())[0]["prog"]
    out = {"device": torch.cuda.get_device_name(0), "batch": B, "programs": {}}
    for name, p in progs.items():
        for _ in range(2):
            p.run()
        torch.cuda.synchronize()
        t = ops.time_program_ops(p, repeats=5)
        kn = p.op_kernels()
        rows = []
        for i, (ms, kd, k, fl, by) in enumerate(zip(t, p.kinds, kn, p.flops, p.bytes)):
            d = p.descs[i]
            shape = ""
            if d is not None and kd == "conv":
                shape = f"{d.H}x{d.W} {d.cin}->{d.cout_pad} k{d.ksize}s{d.stride}"
            rows.append({"i": i, "kind": kd, "kernel": k, "shape": shape, "ms": round(ms, 4),
                         "tflops": round(fl / ms / 1e9, 1) if ms else 0.0, "gbs": round(by / ms / 1e6, 1) if ms else 0.0})
        conv_ms = sum(r["ms"] for r in rows if r["kind"] == "conv")
        halo_ms = sum(r["ms"] for r in rows if r["kernel"] == "conv_halo_kernel")
        out["programs"][name] = {"all_ops_ms": round(sum(t), 3), "conv_ms": round(conv_ms, 3),
                                 "halo_ms": round(halo_ms, 3), "ops": rows}
        print(f"== {name}: {sum(t):.3f} ms, conv {conv_ms:.3f} ms, of which conv_halo_kernel {halo_ms:.3f} ms")
        for r in rows:
            print(f"{r['i']:3d} {r['kernel']:22s} {r['shape']:26s} {r['ms'] * 1e3:9.1f} us {r['tflops']:7.1f} TF/s "
                  f"{r['gbs']:8.1f} GB/s")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
