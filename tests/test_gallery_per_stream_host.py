"""Per-stream galleries without a GPU: the plan of a tick's grouped gallery search (dg_selftest_gallery_plan_host) against a
numpy model, and the refusals of dg_multi_set_slot_gallery and dg_multi_set_names (dg_selftest_multi_gallery_host)."""
import ctypes as C

import numpy as np
import pytest

from diart_b200 import _lib

TILE_E, TILE_Q = 64, 128


def gallery_splits(G, Qmax):
    """the split count of one gallery searched by Qmax queries: about two CTAs per SM, at most 64, no split empty"""
    tiles, qtiles = -(-G // TILE_E), -(-Qmax // TILE_Q)
    s = min(-(-(2 * 132) // qtiles), 64, tiles)
    per = -(-tiles // s)
    return -(-tiles // per)


def plan(slots, G, thr):
    """slots (n, 3) {slot, key, unnamed} -> (groups (g, 6), segs (n', 2), work (w, 3), splits) from the C planner"""
    slots = np.ascontiguousarray(slots, dtype=np.int32).reshape(-1, 3)
    G = np.ascontiguousarray(G, dtype=np.int32)
    thr = np.ascontiguousarray(thr, dtype=np.float64)
    n = len(slots)
    groups = np.zeros((max(n, 1), 6), dtype=np.int32)
    segs = np.zeros((max(n, 1), 2), dtype=np.int32)
    cap = 1 << 17
    work = np.zeros((cap, 3), dtype=np.int32)
    counts = np.zeros(4, dtype=np.int32)
    _lib.check(_lib.lib().dg_selftest_gallery_plan_host(n, slots.ctypes.data, len(G), G.ctypes.data, thr.ctypes.data,
                                                         groups.ctypes.data, segs.ctypes.data, work.ctypes.data, cap,
                                                         counts.ctypes.data))
    return groups[:counts[0]], segs[:counts[1]], work[:counts[2]], int(counts[3])


def check_plan(slots, G, thr):
    slots = np.asarray(slots, dtype=np.int64).reshape(-1, 3)
    groups, segs, work, splits = plan(slots, G, thr)
    # groups: one per key in order of its first slot, with the sum of its slots' unnamed speakers
    keys = list(dict.fromkeys(int(k) for k in slots[:, 1] if k >= 0))
    assert groups[:, 0].tolist() == keys
    for r, k in enumerate(keys):
        mine = slots[slots[:, 1] == k]
        assert groups[r, 1] == G[k] and groups[r, 5] == mine[:, 2].sum()
        # segments: group by group, slots in order
        assert segs[segs[:, 1] == r, 0].tolist() == mine[:, 0].tolist()
    assert segs[:, 1].tolist() == sorted(segs[:, 1].tolist())
    qtiles = -(-groups[:, 5] // TILE_Q) if len(groups) else np.zeros(0, dtype=np.int64)
    total = int(qtiles.sum())
    if total == 0:
        assert len(work) == 0 and splits == 0
        return groups, work, splits
    s = min(-(-(2 * 132) // total), 64)
    for r in range(len(groups)):
        tiles, per, ns = int(groups[r, 2]), int(groups[r, 3]), int(groups[r, 4])
        assert tiles == -(-G[keys[r]] // TILE_E)
        # the splits partition the group's entry tiles, none empty, at most the tick's split count
        assert 1 <= ns <= min(s, tiles)
        cover = np.concatenate([np.arange(k * per, min(tiles, (k + 1) * per)) for k in range(ns)])
        assert cover.tolist() == list(range(tiles))
        assert all(k * per < tiles for k in range(ns))
        # every query of the group (up to its upper bound) in exactly one work item per split
        mine = work[work[:, 0] == r]
        for k in range(ns):
            t = mine[mine[:, 2] == k, 1]
            assert sorted(t.tolist()) == list(range(int(qtiles[r]))), (r, k)
        assert (mine[:, 2] < ns).all()
    assert splits == max(int(groups[r, 4]) for r in range(len(groups)) if qtiles[r] > 0)
    # split-major, then group, then tile
    order = np.lexsort((work[:, 1], work[:, 0], work[:, 2]))
    assert np.array_equal(order, np.arange(len(work)))
    return groups, work, splits


@pytest.mark.parametrize("G", [1, 63, 64, 65, 1000, 100000])
@pytest.mark.parametrize("n,unnamed", [(1, 1), (3, 20), (50, 20), (4096, 20), (7, 0)])
def test_one_group_is_todays_grid(G, n, unnamed):
    slots = [(2 * a, 0, unnamed) for a in range(n)]
    groups, work, splits = check_plan(slots, [G], [0.5])
    Q = n * unnamed
    if Q == 0:
        assert len(work) == 0
        return
    want = gallery_splits(G, Q)
    qtiles = -(-Q // TILE_Q)
    assert splits == want and groups[0, 4] == want
    assert groups[0, 3] == -(-groups[0, 2] // want)       # the per-split tile count of the single-gallery launch
    # the grid (query tiles, splits) in its linear order: x fastest
    assert work.tolist() == [[0, t, k] for k in range(want) for t in range(qtiles)]


def test_ragged_mixes_of_groups():
    rng = np.random.default_rng(11)
    sizes = [1, 63, 64, 65, 100000, 16, 1000, 12008]
    for trial in range(40):
        n = int(rng.integers(1, 300))
        n_keys = int(rng.integers(1, 9))
        G = rng.choice(sizes, n_keys).astype(np.int32)
        thr = rng.uniform(0.1, 1.0, n_keys)
        key = rng.integers(-1, n_keys, n)
        unnamed = np.where(rng.random(n) < 0.2, 0, rng.integers(0, 33, n))   # some slots fully named
        slots = np.stack([np.sort(rng.choice(4096, n, replace=False)), key, unnamed], axis=1)
        check_plan(slots, G, thr)


def test_one_slot_per_group_and_many_groups():
    n = 4096
    slots = [(a, a, 20) for a in range(n)]
    groups, work, splits = check_plan(slots, [16] * n, [0.3] * n)
    assert len(groups) == n and splits == 1 and len(work) == n
    slots = [(a, a // 64, 20) for a in range(n)]
    groups, work, splits = check_plan(slots, [1000] * 64, [0.5] * 64)
    assert len(groups) == 64 and splits == 1
    # few queries over large galleries: the splits are chosen over the whole list, not per group
    slots = [(a, a, 3) for a in range(4)]
    groups, work, splits = check_plan(slots, [100000, 100000, 65, 1], [0.5] * 4)
    assert splits == 63 and groups[:, 4].tolist() == [63, 63, 2, 1]   # 1 563 tiles in runs of 25


def test_no_slot_with_a_gallery_plans_nothing():
    groups, segs, work, splits = plan([(0, -1, 20), (3, -1, 5)], [64], [0.5])
    assert len(groups) == 0 and len(segs) == 0 and len(work) == 0 and splits == 0


def refusals(ops, slots=4, D=8, M=4, gal=((100, 8, 0), (16, 8, 0), (10, 6, 0), (10, 8, 1))):
    gal = np.ascontiguousarray(gal, dtype=np.int32)
    ops = np.ascontiguousarray(ops, dtype=np.float64)
    result = np.zeros(len(ops), dtype=np.int32)
    msg = C.create_string_buffer(1 << 16)
    lib = _lib.lib()
    before = lib.dg_launch_count()
    _lib.check(lib.dg_selftest_multi_gallery_host(slots, D, M, len(gal), gal.ctypes.data, len(ops), ops.ctypes.data,
                                                  result.ctypes.data, msg, len(msg)))
    assert lib.dg_launch_count() == before
    return result.tolist(), msg.value.decode().split("\n")[:len(ops)]


def test_slot_gallery_refusals():
    OPEN, SET, GIVE, NAMES, TICK, CLOSE = range(6)
    ops = [(SET, 0, 0, 0.5),        # a closed slot
           (OPEN, 0, 0, 0),
           (SET, 0, -1, 0.5),       # a null gallery
           (SET, 0, 2, 0.5),        # another dimension
           (SET, 0, 3, 0.5),        # another device
           (SET, 0, 0, 0.0),        # thresholds outside (0, 2]
           (SET, 0, 0, 2.5),
           (SET, 0, 0, float("nan")),
           (SET, 9, 0, 0.5),        # a slot out of range
           (OPEN, 1, 0, 0),
           (TICK, 1, 0, 0),
           (SET, 1, 0, 0.5),        # after the slot's first tick
           (CLOSE, 1, 0, 0),
           (SET, 1, 0, 0.5)]        # closed again
    result, msgs = refusals(ops)
    for i, (op, rc, m) in enumerate(zip(ops, result, msgs)):
        if op[0] == SET:
            assert rc == -1 and "dg_multi_set_slot_gallery" in m, (i, m)
        else:
            assert rc == 0 and m == "", (i, m)
    assert "not open" in msgs[0] and "null" in msgs[2] and "dimension 6" in msgs[3] and "device 1" in msgs[4]
    assert all("threshold" in msgs[i] for i in (5, 6, 7)) and "first tick" in msgs[11] and "not open" in msgs[13]


def test_names_refusals_check_the_slots_own_gallery():
    OPEN, SET, GIVE, NAMES = range(4)
    ops = [(NAMES, 0, 1, 0),        # a closed slot
           (OPEN, 0, 0, 0),
           (NAMES, 0, 1, 0),        # no gallery (the server has no default)
           (GIVE, 0, 1, 0),         # the slot's own gallery of 16 entries
           (NAMES, 0, 1, 16),       # an entry outside the slot's gallery (inside the other one of 100)
           (NAMES, 0, 1, 99),
           (NAMES, 0, 0, 3),        # a claim by a speaker that is not named
           (NAMES, 0, 1, -2),
           (NAMES, 0, 1 << 5, -1)]  # named speakers beyond max_speakers
    result, msgs = refusals(ops)
    for i, (op, rc, m) in enumerate(zip(ops, result, msgs)):
        if op[0] == NAMES:
            assert rc == -1 and "dg_multi_set_names" in m, (i, m)
        else:
            assert rc == 0, (i, m)
    assert "gallery of 16" in msgs[4] and "gallery of 16" in msgs[5]


def test_null_handles_are_refused():
    lib = _lib.lib()
    assert lib.dg_multi_set_slot_gallery(None, 0, None, 0.5) == -1
    assert b"dg_multi_set_slot_gallery" in lib.dg_last_error()
    assert lib.dg_multi_set_names(None, 0, 0, None) == -1
    assert b"dg_multi_set_names" in lib.dg_last_error()


def test_planning_is_linear_in_slots_and_groups():
    """65 535 streams, each with its own roster gallery: planned far inside a 0.5 s tick, as the tick plans it"""
    n = 65535
    slots = np.stack([np.arange(n), np.arange(n), np.full(n, 20)], axis=1)
    G, thr = [16] * n, [0.3] * n
    best = min(_timed(plan, slots, G, thr) for _ in range(3))
    groups, segs, work, splits = plan(slots, G, thr)
    assert len(groups) == n and len(segs) == n and len(work) == n and splits == 1
    assert best < 0.1, f"{best:.3f} s to plan {n} one-slot groups"
    # and the same number of slots over one gallery costs about as much
    one = min(_timed(plan, np.stack([np.arange(n), np.zeros(n, int), np.full(n, 20)], axis=1), [16], [0.3])
              for _ in range(3))
    assert best < 10 * one + 0.02, (best, one)


def _timed(f, *args):
    import time

    t0 = time.perf_counter()
    f(*args)
    return time.perf_counter() - t0
