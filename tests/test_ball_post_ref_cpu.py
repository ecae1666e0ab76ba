"""The ball post-processing references of tests/ball_post_ref.py checked on the CPU: the adversarial masks are not
vacuous and the union-find restatement agrees with cv2 on them, the InpaintNet float64 bound holds for a float32 run
at every sequence length, and the bound and the inpaint-stage decisions reject mutated networks."""
import numpy as np
import pytest
import torch

import ball_post_ref as R
from oracle import inpaint as OI
from oracle import tracknet as OT


@pytest.mark.parametrize("name", sorted(R.GENERATORS))
def test_restated_component_box_equals_cv2(name):
    m = R.make_mask(name)
    assert m.shape == (R.H_NET, R.W_NET) and m.dtype == np.uint8
    assert tuple(OT.largest_component_bbox(m)) == tuple(OT.heatmap_to_bbox(m * 255))


@pytest.mark.parametrize("name", R.TIE_GENERATORS)
def test_tie_generators_tie(name):
    fg, ncomp, tied = R.component_stats(R.make_mask(name))
    assert tied >= 2, f"{name}: {tied} components share the largest box ({ncomp} components)"


@pytest.mark.parametrize("name", R.WRAP_GENERATORS)
def test_wrap_generators_have_flat_neighbours_across_the_row_end(name):
    assert R.wrap_pairs(R.make_mask(name)) > 0


def test_generators_cover_the_listed_shapes():
    stats = {n: R.component_stats(R.make_mask(n)) for n in R.GENERATORS}
    assert stats["serpentine"][1] == stats["spiral"][1] == stats["checkerboard"][1] == 1
    assert stats["lattice"][1] == (R.H_NET // 2) * (R.W_NET // 2)
    assert stats["empty"] == (0, 0, 0) and stats["full"][0] == R.H_NET * R.W_NET
    assert stats["island_in_hole"][1] >= 3
    v = R.make_mask("v_comb")
    x, y, w, h = OT.heatmap_to_bbox(v * 255)
    ys, xs = np.nonzero(v[y:y + h, x:x + w])
    assert (ys[0], xs[0]) != (0, 0), "the winner's first raster pixel must not be its box's top-left"


def _inputs(L, N=48, seed=0):
    g = torch.Generator().manual_seed(seed * 100 + L)
    c = torch.rand((N, L, 2), generator=g)
    m = (torch.rand((N, L, 1), generator=g) > 0.5).float()
    return c, m


@pytest.fixture(scope="module")
def inpaint_sd():
    return OI.make_inpaintnet()["model"]


def test_f64_reference_is_the_oracle_network(inpaint_sd):
    c, m = _inputs(16)
    net = OI.InpaintNetOracle().double()
    net.load_state_dict(inpaint_sd)
    with torch.no_grad():
        exp = net(c.double(), m.double())
    ref, _ = R.inpaint_forward_f64(inpaint_sd, c, m)
    assert (ref - exp).abs().max().item() < 1e-12


@pytest.mark.parametrize("L", [1, 2, 3, 7, 16, 31, 32])
def test_f32_inpaintnet_within_bound(inpaint_sd, L):
    c, m = _inputs(L)
    ref, bound = R.inpaint_forward_f64(inpaint_sd, c, m)
    r = R.bound_ratio(R.inpaint_forward_f32(inpaint_sd, c, m), ref, bound)
    print(f"L={L}: float32 worst |err|/bound {r:.3g}, bound max {bound.max().item():.3g}")
    assert r <= 1.0
    # the bound is tight enough to mean something: well below the outputs' own scale
    assert bound.max().item() < 1e-2


MUTATIONS = {"slope_0.02": dict(slope=0.02), "pad_shift": dict(pad_shift=1), "bias_dropped": dict(drop_bias="up_2.conv"),
             "transposed_output": dict(transpose_out=True)}


@pytest.mark.parametrize("mut", sorted(MUTATIONS))
def test_bound_rejects_mutated_network(inpaint_sd, mut):
    for L in (2, 16, 32):
        c, m = _inputs(L, seed=1)
        ref, bound = R.inpaint_forward_f64(inpaint_sd, c, m)
        r = R.bound_ratio(R.inpaint_forward_f32(inpaint_sd, c, m, **MUTATIONS[mut]), ref, bound)
        assert r > 10, f"L={L}: mutation {mut} only reaches {r:.3g} of the bound"


def _trajectory_case(seed=3, T=90):
    wh = (1280, 720)
    xs, ys, vs = R.synthetic_trajectory(seed, T, wh, gaps=[(0, 4), (30, 37), (60, 62), (T - 5, T)])
    return wh, xs, ys, vs


def _run_stage(inpaint_sd, net, wh, xs, ys, vs, L=16):
    got, exp, border, _ = R.stage_decisions(inpaint_sd, net, xs, ys, vs, L, wh)
    return got, exp, border


def test_inpaint_decisions_accept_float32_stage(inpaint_sd):
    wh, xs, ys, vs = _trajectory_case()
    got, exp, border = _run_stage(inpaint_sd, lambda c, m: R.inpaint_forward_f32(inpaint_sd, c, m), wh, xs, ys, vs)
    bad = R.compare_decisions(got, exp, border)
    print(f"float32 stage: {len(exp)} frames, {len(border)} borderline, {len(bad)} differ")
    assert not bad
    assert len(border) <= len(exp) // 10
    assert sum(v for _, _, v in exp.values()) > len(exp) // 2  # mostly visible: the test is not about zeros


@pytest.mark.parametrize("mut", sorted(MUTATIONS))
def test_inpaint_decisions_reject_mutated_network(inpaint_sd, mut):
    wh, xs, ys, vs = _trajectory_case()
    net = lambda c, m: R.inpaint_forward_f32(inpaint_sd, c, m, **MUTATIONS[mut])
    got, exp, border = _run_stage(inpaint_sd, net, wh, xs, ys, vs)
    assert R.compare_decisions(got, exp, border), f"mutation {mut} changed no decision"
