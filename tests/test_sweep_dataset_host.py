"""Host half of the dataset sweep (diart_b200.tune.DatasetSweep): concatenated post-path plans, the launch order of the
(file, trial) states, trial groups, reference packing, per-file turn slices and the argument errors.  No GPU needed."""
import ctypes

import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks
from diart_b200.blocks.post import post_plan
from diart_b200.core import Annotation, Segment
from diart_b200.tune import (TRIAL_CHUNKS_PER_LAUNCH, TRIALS_PER_LAUNCH, DatasetSweep, dataset_plan, file_turns,
                             file_windows, pack_references, reference_arrays, seg_resolution, trial_groups)

F = 293


def config(**kw):
    return blocks.SpeakerDiarizationConfig(segmentation=object(), embedding=object(), device=torch.device("cpu"), **kw)


@pytest.mark.parametrize("kw", [{}, {"latency": 2.0}, {"step": 0.3, "latency": 1.2}])
def test_concatenated_plans_equal_the_per_file_plans(kw):
    cfg = config(**kw)
    rng = np.random.default_rng(1)
    fws = [file_windows(rng.standard_normal(int(s * 16000)).astype(np.float32), cfg) for s in (3.2, 9.71, 2.0, 17.3)]
    plan, out_start, out_res = dataset_plan(fws, cfg, F)
    nw = int(round(cfg.latency / cfg.step))
    c0 = 0
    for fw in fws:
        want = post_plan(fw.starts, seg_resolution(cfg, float(fw.starts[0]), F), np.zeros(0), np.zeros(0), nw, F, cfg.step,
                         cfg.latency)
        c1 = c0 + fw.num_windows
        assert np.array_equal(plan[c0:c1], want[0])
        assert np.array_equal(out_start[c0:c1], want[1]) and np.array_equal(out_res[c0:c1], want[2])
        # post.cu: chunk c aggregates chunks c - (nb - 1) .. c; none of them before the file's first chunk
        nb = plan[c0:c1, 0]
        assert np.all(np.arange(c0, c1) - (nb - 1) >= c0)
        assert plan[c0, 0] == 1
        c0 = c1
    assert c0 == len(plan)
    assert fws[0].padding[0] > 0 and fws[0].num_windows == 1


def test_launch_order_is_longest_file_first_and_stable():
    lib = _lib.lib()
    off = np.array([0, 3, 10, 12, 19, 20, 23], np.int32)         # lengths 3, 7, 2, 7, 1, 3
    T = 2
    states = np.full((6 * T, 2), -1, np.int32)
    assert lib.dg_sweep_state_order(6, off.ctypes.data, T, states.ctypes.data) == 0
    files = [1, 3, 0, 5, 2, 4]
    assert states.tolist() == [[f, t] for f in files for t in range(T)]
    assert lib.dg_sweep_state_order(0, off.ctypes.data, T, states.ctypes.data) == -1
    assert b"dg_sweep_state_order" in lib.dg_last_error()
    assert lib.dg_sweep_state_order(6, off.ctypes.data, 0, states.ctypes.data) == -1


@pytest.mark.parametrize("T,N", [(1, 1), (9, 3591), (1024, 3591), (3000, 3591), (5000, 28_000), (7, 4 << 20)])
def test_trial_groups_respect_both_caps_and_cover_every_trial_once(T, N):
    groups = trial_groups(T, N)
    covered = np.concatenate([np.arange(T)[g] for g in groups])
    assert np.array_equal(covered, np.arange(T))
    for g in groups:
        n = g.stop - g.start
        assert 1 <= n <= TRIALS_PER_LAUNCH and n * N <= TRIAL_CHUNKS_PER_LAUNCH
    if T == 1024 and N == 3591:
        assert len(groups) == 1


def test_a_dataset_over_one_launch_is_refused():
    with pytest.raises(ValueError):
        trial_groups(1, TRIAL_CHUNKS_PER_LAUNCH + 1)


def test_references_pack_per_file():
    a = Annotation(uri="a")
    a[Segment(0.0, 2.0), 0] = "x"
    a[Segment(1.0, 3.0), 1] = "y"
    a[Segment(2.5, 4.0), 2] = "x"
    b = Annotation(uri="b")                                   # no segments: zero rows, zero labels
    c = Annotation(uri="c")
    c[Segment(5.0, 6.0), 0] = "z"
    rows, labels, offsets, counts = pack_references([a, b, c])
    assert offsets.tolist() == [0, 3, 3, 4] and counts.tolist() == [2, 0, 1]
    for i, ref in enumerate((a, b, c)):
        r, lab, names = reference_arrays(ref)
        assert np.array_equal(rows[offsets[i]:offsets[i + 1]], r)
        assert np.array_equal(labels[offsets[i]:offsets[i + 1]], lab) and counts[i] == len(names)
    assert rows.dtype == np.float64 and labels.dtype == np.int32 and rows.flags.c_contiguous


def test_file_turns_are_each_files_turns_alone():
    rng = np.random.default_rng(4)
    T, N = 3, 11
    cnt = rng.integers(0, 4, (T, N))
    order = rng.permutation(T * N)                            # the blocks in the order the device's counter leaves them
    header = np.zeros((T, N, 4), np.int32)
    turns, pos = [], 0
    for r in order:
        t, c = divmod(int(r), N)
        header[t, c] = (pos, cnt[t, c], 7, 0)
        turns += [(t << 20) | (c << 10) | k for k in range(cnt[t, c])]
        pos += cnt[t, c]
    turns = np.array(turns, np.uint32)
    h, own, n = file_turns(header, turns, 4, 9)
    assert h.shape == (T, 5, 4) and n == cnt[:, 4:9].sum()
    for t in range(T):
        for j, c in enumerate(range(4, 9)):
            o, k = h[t, j, :2]
            assert own[o:o + k].tolist() == [(t << 20) | (c << 10) | q for q in range(cnt[t, c])]
    assert np.array_equal(h[..., 2], header[:, 4:9, 2])


def test_constructor_argument_errors_without_a_gpu():
    cfg = config()
    with pytest.raises(ValueError):
        DatasetSweep(cfg, [])
    with pytest.raises(ValueError, match="no samples"):
        DatasetSweep(cfg, [("a", np.zeros(16000, np.float32), None), ("b", np.zeros(0, np.float32), None)])


def test_file_entry_points_reject_bad_handles_without_a_gpu():
    lib = _lib.lib()
    off = np.array([0, 1], np.int32)
    n = ctypes.c_int()
    assert lib.dg_sweep_run_files(None, None, None, 1, 1, off.ctypes.data, None, 1, None, None, None, None, None, 0,
                                  ctypes.byref(n), None) == -1
    assert b"dg_sweep_run_files" in lib.dg_last_error()
    assert lib.dg_sweep_score_files(None, None, None, 1, 1, off.ctypes.data, None, 1, None, None, None, None, 0.05, None,
                                    None, None, None, None, None, None, 0, None) == -1
    assert b"dg_sweep_score_files" in lib.dg_last_error()
