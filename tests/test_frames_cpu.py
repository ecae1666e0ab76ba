"""CPU: the frame-source reader (`trackers/frames.py`): pieces of HWC frames and host batches, trimmed, checked and
packed into chunks that cross clip boundaries."""
import numpy as np
import pytest
import torch

from padel_analytics_b200.trackers import frames

H, W = 4, 6


def _clips():
    rng = np.random.default_rng(0)
    clips = [rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8) for T in (5, 0, 8, 9, 3)]
    srcs = [lambda lo, hi, c=c: iter(clips[c][lo:hi]) for c in (0, 1, 2)]
    srcs += [lambda lo, hi: (torch.from_numpy(clips[3][i:min(hi, i + 4)]) for i in range(lo, hi, 4)),
             lambda lo, hi: iter([torch.from_numpy(clips[4])])]  # batched host tensors, one longer than the clip
    return clips, srcs


def _host(shape):
    return torch.empty(shape, dtype=torch.uint8)


def test_read_and_chunks_cross_clip_boundaries():
    clips, srcs = _clips()
    lengths = [5, 0, 8, 9, 2]
    pieces = (p for c, T in enumerate(lengths) for p in frames.read(srcs[c], 0, T, (H, W), exact=True, clip=c))
    got = [[p.numpy().copy() for p in b] for b in frames.chunks(pieces, 7, alloc=_host)]  # buffers are reused
    assert [sum(len(p) for p in b) for b in got] == [7, 7, 7, 3]
    flat = np.concatenate([p for b in got for p in b])
    assert np.array_equal(flat, np.concatenate([clips[0], clips[2], clips[3], clips[4][:2]]))
    with pytest.raises(ValueError, match="clip 3 yielded 5 frames, 6 announced"):
        list(frames.chunks(frames.read(srcs[0], 0, 6, exact=True, clip=3), 7, alloc=_host))
    with pytest.raises(ValueError, match="frames"):
        list(frames.read(srcs[0], 0, 5, (H + 1, W)))
    mixed = [np.zeros((H, W, 3), np.uint8), np.zeros((H, W + 1, 3), np.uint8)]
    with pytest.raises(ValueError, match=r"\(4, 7\).*\(4, 6\)"):  # default: the first piece's size
        list(frames.read(lambda lo, hi: iter(mixed), 0, 2))


def test_read_without_exact_ends_with_the_source():
    clips, srcs = _clips()
    assert [len(p) for p in frames.read(srcs[0], 0, 6)] == [1] * 5
    got = [[p.numpy().copy() for p in b] for b in frames.chunks(frames.read(srcs[3], 0, 12), 7, alloc=_host)]
    assert [sum(len(p) for p in b) for b in got] == [7, 2]
    assert np.array_equal(np.concatenate([p for b in got for p in b]), clips[3])
    assert list(frames.read(srcs[0], 0, 0, exact=True)) == []


def test_head_splits_the_piece_at_m():
    clips, srcs = _clips()
    first, rest = frames.head(frames.read(srcs[3], 0, 9), 6)
    assert [len(p) for p in first] == [4, 2]
    assert np.array_equal(torch.cat(first).numpy(), clips[3][:6])
    assert np.array_equal(torch.cat(list(rest)).numpy(), clips[3][6:])
    first, rest = frames.head(frames.read(srcs[0], 0, 5), 8)  # fewer frames than m
    assert len(first) == 5 and list(rest) == []
