"""Device post-path (csrc/post.cu through dg_post_step): SpeakerMap.apply + DelayedAggregation(hamming, loose) + Binarize on
the GPU vs the numpy mirrors of the reference blocks (pinned to the reference in tests/test_oracle_vs_reference.py).
Bit-exact bar: identical segments (float64 times) for every chunk, for latency = step .. duration and ragged batch splits."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib
from diart_b200.blocks.aggregation import DelayedAggregation
from diart_b200.blocks.post import DevicePostPath, post_plan
from diart_b200.blocks.utils import Binarize
from diart_b200.core import SlidingWindow, SlidingWindowFeature

pytestmark = pytest.mark.gpu
F, K, M = 293, 3, 20


def tracks(a):
    return [(s.start, s.end, t, l) for s, t, l in a.itertracks(yield_label=True)]


@pytest.mark.parametrize("latency,splits", [(0.5, [1, 5, 64]), (2.0, [3, 1, 30]), (5.0, [7, 40]), (1.5, [2, 2, 2, 33])])
@pytest.mark.parametrize("F", [293, 292])
def test_device_post_path_equals_reference_blocks(F, latency, splits, cuda_device):
    """F = 292 at latency = step: the first chunk emits F + 1 frames"""
    rng = np.random.default_rng(int(latency * 10) + 1)
    step, tau = 0.5, 0.6
    n = sum(splits)
    seg_all = np.clip(np.cumsum(rng.random((n, F, K)) - 0.5, axis=1) * 0.2 + 0.55, 0, 1).astype(np.float32)
    seg_all[0, :40, 0] = 0.9                                   # a turn that is active from the very first frame
    seg_all[1, -30:, 1] = 0.95                                 # ... and one that is still active at the last frame
    base = rng.permutation(M)[:K]
    map_all = np.stack([base if rng.random() < 0.7 else rng.permutation(M)[:K] for _ in range(n)]).astype(np.int32)
    map_all[rng.random((n, K)) < 0.15] = -1
    starts = [step * i for i in range(n)]
    res = ((0.0 + 80000 * (1 / 16000)) - 0.0) / F
    if (F, latency) == (292, step):
        assert post_plan(np.zeros(1), res, np.zeros(0), np.zeros(0), 1, F, step, latency)[0][0, 2] == F + 1
    agg, binarize = DelayedAggregation(step, latency, "hamming", "loose"), Binarize(tau)
    buf, want = [], []
    for i in range(n):
        permuted = np.zeros((F, M))
        for k, g in enumerate(map_all[i]):
            if g >= 0:
                permuted[:, g] = seg_all[i][:, k]
        buf.append(SlidingWindowFeature(permuted, SlidingWindow(start=starts[i], duration=res, step=res)))
        want.append(binarize(agg(buf)))
        if len(buf) == agg.num_overlapping_windows:
            buf = buf[1:]
    post = DevicePostPath(step, latency, tau, F, K, M, cuda_device)
    got, first = [], 0
    for b in splits:
        seg = torch.from_numpy(seg_all[first:first + b]).to(cuda_device)
        maps = torch.from_numpy(map_all[first:first + b]).to(cuda_device)
        got += post.run(seg, maps, np.array(starts[first:first + b]), res)
        first += b
    lines = 0
    for i, (a, b) in enumerate(zip(want, got)):
        assert tracks(a) == tracks(b), f"chunk {i}"
        lines += len(tracks(a))
    assert lines > n // 4
    # reset: the same stream again gives the same answer (history cleared on both sides)
    post.reset()
    seg = torch.from_numpy(seg_all[:splits[0]]).to(cuda_device)
    maps = torch.from_numpy(map_all[:splits[0]]).to(cuda_device)
    again = post.run(seg, maps, np.array(starts[:splits[0]]), res)
    assert [tracks(a) for a in again] == [tracks(a) for a in want[:splits[0]]]


def test_many_turns_need_a_second_copy(cuda_device):
    """more turns than the prefix that travels with the header (alternating frames on every speaker)"""
    n, tau = 96, 0.5
    seg = np.zeros((n, F, K), np.float32)
    seg[:, ::2, :] = 1.0
    maps = np.tile(np.arange(K, dtype=np.int32), (n, 1))
    post = DevicePostPath(5.0, 5.0, tau, F, K, M, cuda_device)       # step = latency = duration: whole chunks are emitted
    starts = np.arange(n) * 5.0
    res = 5.0 / F
    got = post.run(torch.from_numpy(seg).to(cuda_device), torch.from_numpy(maps).to(cuda_device), starts, res)
    total = sum(len(tracks(a)) for a in got)
    assert total > 16384
    agg, binarize = DelayedAggregation(5.0, 5.0, "hamming", "loose"), Binarize(tau)
    for i in (0, 1, n - 1):
        permuted = np.zeros((F, M))
        permuted[:, :K] = seg[i]
        want = binarize(agg([SlidingWindowFeature(permuted, SlidingWindow(start=starts[i], duration=res, step=res))]))
        assert tracks(want) == tracks(got[i])


def test_plan_rows_a_stream_cannot_have_are_refused(cuda_device):
    """a row with more buffers than latency / step, one whose buffers reach before the stream's first chunk, one with F + 2
    output frames: refused before any launch, and the history is left as it was"""
    lib = _lib.lib()
    step, latency, res = 0.5, 1.5, 5.0 / F
    rng = np.random.default_rng(3)
    seg = torch.from_numpy(rng.random((4, F, K), dtype=np.float32)).to(cuda_device)
    maps = torch.from_numpy(np.tile(np.arange(K, dtype=np.int32), (4, 1))).to(cuda_device)
    starts = np.arange(4) * step
    post = DevicePostPath(step, latency, 0.5, F, K, M, cuda_device)
    plan = np.ascontiguousarray(post_plan(starts, res, np.zeros(0), np.zeros(0), post.nw, F, step, latency)[0])
    wide, early, long_first = plan.copy(), plan.copy(), plan.copy()
    wide[3, 0] = post.nw + 1
    early[1, 0] = 3
    long_first[0, 2] = F + 2
    header, turns = post.buffers(4)
    for name, bad in (("nb > nw", wide), ("before the first chunk", early), ("F + 2 frames", long_first)):
        before = lib.dg_launch_count()
        rc = lib.dg_post_step(post.handle, seg.data_ptr(), maps.data_ptr(), 4, bad.ctypes.data, header.ctypes.data,
                              turns.ctypes.data, len(turns), ctypes.byref(ctypes.c_int()), None)
        assert rc == -1 and lib.dg_launch_count() == before, name
        assert b"dg_post_step: plan row" in lib.dg_last_error(), name
    fresh = DevicePostPath(step, latency, 0.5, F, K, M, cuda_device)
    got, want = post.run(seg, maps, starts, res), fresh.run(seg, maps, starts, res)
    assert [tracks(a) for a in got] == [tracks(a) for a in want] and sum(len(tracks(a)) for a in got) > 0
