"""The clip batch planner (engine/clip_plan.py) and the per-row temporal ensemble it drives, without a GPU.

The planner decides where every frame of a list of clips goes in the device ring, which windows each device batch
packs and which frames it emits; the per-row ensemble is restated in numpy over the concatenated windows and must
equal the oracle's per-clip ensemble bit for bit."""
import numpy as np
import pytest
import torch

from oracle import tracknet as OT
from padel_analytics_b200.engine.clip_plan import WINDOW, plan_clip_batches


def _random_cases(n, seed):
    rng = np.random.default_rng(seed)
    for _ in range(n):
        k = int(rng.integers(1, 9))
        lengths = [int(v) for v in rng.integers(1, 41, size=k)]
        batch = int(rng.integers(1, 33))
        chunk = int(rng.integers(1, batch + 1)) if rng.random() < 0.3 else batch
        ring = None if rng.random() < 0.6 else chunk + WINDOW - 1 + int(rng.integers(0, 2 * batch + 1))
        pool = None if rng.random() < 0.7 else int(rng.integers(1, 4))
        yield lengths, batch, chunk, ring, pool


def _simulate(plan):
    """Replay the plan on the host: a ring of frame ids, a median pool of clip ids, the carried window rows.  Checks
    every invariant and returns the emitted (clip, frame) list and the rows per batch."""
    lengths = plan.lengths
    clip_of = [c for c, t in enumerate(lengths) for _ in range(t)]
    frame_of = [f for t in lengths for f in range(t)]
    ring = [None] * plan.ring
    pool = [None] * plan.pool
    emitted, windows, pos = [], [], 0
    nwin = [max(0, t - 7) for t in lengths]
    for i, ops in enumerate(plan.steps):
        base = i * plan.chunk
        n_chunk = min(plan.chunk, len(clip_of) - base)
        for op in ops:
            if op[0] == "median":
                _, c, slot = op
                pool[slot] = c
            elif op[0] == "push":
                _, off, n, slot = op
                assert 0 <= off and off + n <= n_chunk and slot + n <= plan.ring, "push outside the chunk or ring"
                for j in range(n):
                    ring[slot + j] = (clip_of[base + off + j], frame_of[base + off + j])
            else:
                b = op[1]
                assert 1 <= len(b.windows) <= plan.batch
                for (c, w), s, m in zip(b.windows, b.row_slot, b.row_median):
                    assert [ring[(s + f) % plan.ring] for f in range(WINDOW)] == [(c, w + f) for f in range(WINDOW)], \
                        f"window {(c, w)} does not see its own 8 consecutive frames"
                    assert pool[m] == c, f"window {(c, w)} reads the median of clip {pool[m]}"
                g0 = b.first_window
                assert [plan.clip_first_window[c] + w for c, w in b.windows] == list(range(g0, g0 + len(b.windows)))
                for (c, f), (cw0, tw, fd) in zip(b.frames, b.desc):
                    assert cw0 == plan.clip_first_window[c] and tw == nwin[c] and fd == f
                    lo, hi = cw0 + max(0, f - 7), cw0 + min(f, tw - 1)
                    assert g0 - 7 <= lo and hi < g0 + len(b.windows), "a frame needs a window outside the pred ring"
                windows += b.windows
                emitted += b.frames
    return emitted, windows


@pytest.mark.parametrize("seed", range(8))
def test_planner_random_clip_lists(seed):
    for lengths, batch, chunk, ring, pool in _random_cases(60, seed):
        plan = plan_clip_batches(lengths, batch, chunk=chunk, ring=ring, pool=pool)
        assert len(plan.steps) == -(-sum(lengths) // chunk)
        emitted, windows = _simulate(plan)
        assert windows == [(c, w) for c, t in enumerate(lengths) for w in range(max(0, t - 7))]
        assert emitted == [(c, f) for c, t in enumerate(lengths) if t >= 8 for f in range(t)]


def test_planner_boundary_placements():
    """clips that start, end and sit entirely inside one batch; a clip ending in the batch that holds the next one's
    first windows; clips too short for a window between them; a ring and a pool at their minimum"""
    cases = [([5, 8, 9, 40, 77, 130], 32, None, None), ([8] * 12, 4, None, None), ([9, 3, 8, 1, 20], 5, None, None),
             ([40, 40, 40], 32, 39, 1), ([7, 7, 7, 8], 1, 8, 1), ([33, 8, 8, 8, 2, 50], 8, 15, 2), ([1], 4, None, None),
             ([100], 32, None, None)]
    for lengths, batch, ring, pool in cases:
        plan = plan_clip_batches(lengths, batch, ring=ring, pool=pool)
        emitted, windows = _simulate(plan)
        assert emitted == [(c, f) for c, t in enumerate(lengths) if t >= 8 for f in range(t)], lengths
    # packing: with the default ring every batch but the last is full
    plan = plan_clip_batches([5, 8, 9, 40, 77, 130], 32)
    sizes = [len(op[1].windows) for ops in plan.steps for op in ops if op[0] == "run"]
    assert sizes[:-1] == [32] * (len(sizes) - 1) and sum(sizes) == 1 + 2 + 33 + 70 + 123
    mixed = [op[1] for ops in plan.steps for op in ops if op[0] == "run" and len({c for c, _ in op[1].windows}) > 1]
    assert mixed, "vacuous: no batch spans a clip boundary"


def test_planner_rejects_bad_arguments():
    with pytest.raises(ValueError):
        plan_clip_batches([10], 8, ring=10)
    with pytest.raises(ValueError):
        plan_clip_batches([-1], 8)
    with pytest.raises(ValueError):
        plan_clip_batches([10], 0)


def _ensemble_rows(pred_rows, first_window, desc):
    """numpy restatement of pb_tracknet_ensemble_rows: pred_rows[r] = global window first_window + r"""
    w = OT.ensemble_weight().numpy()
    out = []
    for cw0, tw, n in desc:
        base = cw0 - first_window
        if tw > n >= 7:
            terms = np.stack([pred_rows[base + n - 7 + k, 7 - k] * w[k] for k in range(8)])
            out.append(terms.sum(0, dtype=np.float32))
        else:
            acc = np.zeros(pred_rows.shape[-2:], np.float32)
            for k in range(8):
                if 0 <= n - 7 + k < tw:
                    acc = acc + pred_rows[base + n - 7 + k, 7 - k]
            div = np.float32(n + 1) if n < tw else np.float32(8 - (n - (tw - 1)))
            out.append(acc / div)
    return out


@pytest.mark.parametrize("lengths,batch", [([5, 8, 9, 40, 77, 130], 32), ([8, 9, 8, 15, 16, 3, 23], 4),
                                           ([61, 8, 8, 12], 16), ([30, 2, 30], 1), ([8] * 9, 3)])
def test_row_ensemble_equals_oracle_per_clip(lengths, batch):
    """The per-row ensemble over the planned batches, with the engine's (7 + B) pred ring and 7-row carry, equals
    oracle/tracknet.py's stateful ensemble loop run on each clip alone, bit for bit.  Planted values sit on 0.5."""
    H, W = 8, 64  # an inner size at which torch's reduction over the 8 terms is sequential, as the kernel's
    g = torch.Generator().manual_seed(sum(lengths) + batch)
    preds = [torch.rand((max(0, t - 7), 8, H, W), generator=g) for t in lengths]
    for p in preds:
        if len(p):
            p.view(-1)[::7] = 0.5
    every = torch.cat(preds).numpy() if sum(len(p) for p in preds) else np.zeros((0, 8, H, W), np.float32)
    plan = plan_clip_batches(lengths, batch)
    ring = np.zeros((7 + batch, 8, H, W), np.float32)
    got = {}
    for ops in plan.steps:
        for op in ops:
            if op[0] != "run":
                continue
            b = op[1]
            nb = len(b.windows)
            ring[7:7 + nb] = every[b.first_window:b.first_window + nb]
            for (c, f), e in zip(b.frames, _ensemble_rows(ring, b.first_window - 7, b.desc)):
                got[(c, f)] = e
            ring[:7] = ring[nb:nb + 7].copy()
    for c, t in enumerate(lengths):
        exp = OT.ensemble_reference_loop(preds[c], t, batch).numpy()
        assert len(exp) == (t if t >= 8 else 0)
        for f in range(len(exp)):
            assert np.array_equal(got[(c, f)].view(np.uint32), exp[f].view(np.uint32)), (c, f)
