"""Every legal conv plan computes what the default plan computes, bit for bit.

Each output's accumulation order in both conv kernels is (channel block, tap, k-step): it does not depend on the
fields of pb_conv_plan (S, G, rings, TMA store, N split, pixel tile, grid).  For every conv op of the four bench
programs at batch 2 (built and run once by test_program_layers_gpu.shipped), the default plan must be in the set
pb_conv_list_plans returns, and a seeded sample of that set (the whole set when small) must reproduce the default
plan's outputs bit for bit: the whole primary and second output tensors, so channels outside the op's slice stay
untouched, and a fused head's output.
"""
from __future__ import annotations

import random

import pytest
import torch

import test_program_layers_gpu as T
from padel_analytics_b200 import _lib as L
from padel_analytics_b200.engine.ops import plan_of

pytestmark = pytest.mark.gpu

SAMPLE = 12  # plans per op besides the default one


class _Cai:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"data": (ptr, False), "shape": (n,), "typestr": "|u1", "version": 2}


def _bytes(ptr: int, n: int) -> torch.Tensor:
    return torch.as_tensor(_Cai(ptr, n), device="cuda")


def written(d) -> list[torch.Tensor]:
    """Byte views of every tensor conv op `d` writes, whole."""
    Ho, Wo = d.H // d.stride, d.W // d.stride
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


@pytest.mark.parametrize("name", ["tracknet", "players", "pose", "court"])
def test_every_sampled_plan_reproduces_the_default_plan(name):
    prog = T.programs()[name]
    rng = random.Random(1234)
    fails, n_ops, n_plans = [], 0, 0
    for i in range(prog.num_ops):
        info = prog.op_info(i)
        if info.kernel not in (0, 1):
            continue
        n_ops += 1
        default = plan_of(info)
        plans = prog.conv_plans(i)
        keys = {p.key() for p in plans}
        if default.key() not in keys:
            fails.append(f"op {i}: default plan {default} is not in the legal set ({len(plans)} plans)")
            continue
        others = [p for p in plans if p.key() != default.key()]
        picked = rng.sample(others, min(SAMPLE, len(others)))
        bufs = written(info.desc)
        saved = [b.clone() for b in bufs]  # later ops (and tests) read these buffers: restored below

        def run_marked():
            for b, s in zip(bufs, saved):  # the op's inputs may share a buffer with its outputs: same start each run
                b.copy_(s)
            for b in bufs:  # poison every 7th byte: a plan that skips a store cannot pass on earlier bytes
                b.view(-1)[::7].fill_(0x5A)
            prog.run(i, i + 1)
            torch.cuda.synchronize()

        run_marked()
        ref = [b.clone() for b in bufs]
        for p in picked:
            prog.set_conv_plan(i, p)
            assert plan_of(prog.op_info(i)).key() == p.key(), f"op {i}: built plan differs from {p}"
            run_marked()
            n_plans += 1
            if not all(torch.equal(a, b) for a, b in zip(bufs, ref)):
                fails.append(f"op {i}: {p} differs from the default plan {default}")
        prog.set_conv_plan(i, None)
        assert plan_of(prog.op_info(i)).key() == default.key()
        for b, s in zip(bufs, saved):
            b.copy_(s)
    print(f"{name}: {n_ops} conv ops, {n_plans} forced plans")
    assert n_ops > 0 and not fails, "\n".join(fails[:30])


def test_illegal_plans_are_refused_and_leave_the_op_as_it_was():
    prog = T.programs()["tracknet"]
    i = next(k for k in range(prog.num_ops) if prog.op_info(k).variant == L.CONV_HALO)
    before = plan_of(prog.op_info(i))
    bad = L.ConvPlan.from_buffer_copy(before)
    bad.a_stages = 9  # more halo stages than the kernel has barriers for
    with pytest.raises(L.PbError):
        prog.set_conv_plan(i, bad)
    bad = L.ConvPlan.from_buffer_copy(before)
    bad.grid = 10 ** 6
    with pytest.raises(L.PbError):
        prog.set_conv_plan(i, bad)
    assert plan_of(prog.op_info(i)).key() == before.key()
