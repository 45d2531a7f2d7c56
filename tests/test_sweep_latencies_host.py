"""Host half of the sweeps over several latencies (diart_b200.tune.LatencyUnits, DatasetSweep / VoiceActivitySweep with
``latencies``): the latency argument, the units a file's windows make, the virtual chunk tables, plans, output times and
shifts against file_windows / stream_plan at each latency alone, and the layout checks of the C entry points.  No GPU
needed."""
import numpy as np
import pytest
import torch

from diart_b200 import _lib, blocks
from diart_b200.tune import (DatasetSweep, LatencyUnits, VoiceActivitySweep, at_latency, file_windows, parse_latencies,
                             stream_plan, trial_params)

F = 293


def config(**kw):
    return blocks.SpeakerDiarizationConfig(segmentation=object(), embedding=object(), device=torch.device("cpu"), **kw)


def vad_config(**kw):
    return blocks.VoiceActivityDetectionConfig(segmentation=object(), device=torch.device("cpu"), **kw)


def test_latencies_are_parsed_sorted_and_include_the_config_latency():
    cfg = config(latency=2.0)
    assert parse_latencies(cfg, []) == (2.0,)
    assert parse_latencies(cfg, ["max", 1.0, "min", 2.0, np.float32(3.5), 4]) == (0.5, 1.0, 2.0, 3.5, 4.0, 5.0)
    for bad in (0.2, 5.01, -1.0, float("nan"), "fast", None, True, [1.0]):
        with pytest.raises(ValueError, match="latency"):
            parse_latencies(cfg, [bad])


@pytest.mark.parametrize("make", [lambda cfg, files, lat: DatasetSweep(cfg, files, latencies=lat),
                                  lambda cfg, files, lat: VoiceActivitySweep(vad_config(), files, latencies=lat)])
def test_a_latency_outside_step_duration_is_refused_before_any_model(make):
    # the configs carry no model at all: reaching the network pass would fail with another error
    files = [("a", np.zeros(16000 * 7, np.float32), None)]
    for bad in ([0.49], [5.5], ["none"]):
        with pytest.raises(ValueError, match="latency"):
            make(config(), files, bad)


def test_a_trial_still_cannot_name_the_latency():
    with pytest.raises(ValueError, match="latency"):
        trial_params([{"latency": 2.0}], config())


def test_units_of_a_short_and_a_long_file():
    cfg = config()
    lats = [0.5, 1.0, 2.0, 2.3, 3.0, "max"]
    x_short = np.ones(int(3.2 * 16000), np.float32)
    x_long = np.ones(int(61.3 * 16000), np.float32)
    u = LatencyUnits([x_short, x_long], cfg, lats)
    assert u.latencies == (0.5, 1.0, 2.0, 2.3, 3.0, 5.0)
    # the 3.2 s file: left padding 1.8, 1.3, 0.3 s at 0.5, 1, 2 s and none from 2.3 s on
    lefts = [file_windows(x_short, at_latency(cfg, lat)).padding[0] for lat in u.latencies]
    assert np.allclose(lefts, [1.8, 1.3, 0.3, 0, 0, 0])
    assert np.allclose(u.shifts[:, 0], [-v for v in lefts]) and np.all(u.shifts[:, 1] == 0)
    for li, lat in enumerate(u.latencies):
        for f, x in enumerate((x_short, x_long)):
            assert u.num_windows[li, f] == file_windows(x, at_latency(cfg, lat)).num_windows
    # the short file: a unit per left padding; without left padding, its 1 and 3 windows at 2.3 and 3 s are last batches
    # of fewer than 4 windows (the sinc front end's per-window form), which its 7-window unit at 5 s would compute in a
    # batch of 7: units of their own.  The long file is one unit.
    assert u.num_windows[:, 0].tolist() == [1, 1, 1, 1, 3, 7]
    assert u.unit_of[:, 0].tolist() == [0, 1, 2, 3, 4, 5]
    assert u.unit_of[:, 1].tolist() == [6] * 6
    assert [fw.num_windows for fw in u.unit_windows] == [1, 1, 1, 1, 3, 7, int(u.num_windows[5, 1])]
    assert u.num_chunks == u.unit_offsets[-1] == 14 + u.num_windows[5, 1]


def test_a_last_batch_of_one_to_three_windows_is_a_unit_of_its_own():
    cfg = config()
    x = np.ones(int(132.3 * 16000), np.float32)                # 256 windows at 0.5 s, 257 at 1 s, 258 at 1.5 s, 265 at 5 s
    u = LatencyUnits([x, x[:16000 * 50]], cfg, [1.0, 1.5, "max"])
    assert u.num_windows[:, 0].tolist() == [256, 257, 258, 265]
    assert u.unit_of[:, 0].tolist() == [0, 1, 2, 0]            # 256 windows: one whole batch of the 265-window unit
    assert [fw.num_windows for fw in u.unit_windows[:3]] == [265, 257, 258]
    assert u.num_windows[:, 1].tolist() == [91, 92, 93, 100]    # last batches of 91 .. 100 windows: one unit
    assert u.unit_of[:, 1].tolist() == [3] * 4
    # without the stream form (the VAD sweep's segmentation pass) every batch length gives the same bits: one unit
    assert LatencyUnits([x], cfg, [1.0, 1.5, "max"], stream_form=False).unit_of[:, 0].tolist() == [0] * 4


def check_tables(cfg, waveforms, lats, sel=None):
    u = LatencyUnits(waveforms, cfg, lats)
    unit_fws = list(u.unit_windows)
    u.plan(F)
    assert u.unit_windows == []                                 # the units' audio is dropped once planned
    sel = list(range(len(u.latencies))) if sel is None else sel
    vchunk, voff, plan, out_start, out_res, shifts = u.tables(sel)
    nf = len(waveforms)
    assert len(voff) == len(sel) * nf + 1 and voff[-1] == len(vchunk) == len(plan) == len(out_start) == len(out_res)
    assert plan.shape[1] == 4 + int(round(u.latencies[-1] / cfg.step))
    assert all(a.flags.c_contiguous for a in (vchunk, voff, plan, out_start, out_res, shifts))
    assert vchunk.dtype == np.int32 and voff.dtype == np.int32 and plan.dtype == np.int32
    rc = _lib.lib().dg_sweep_check_latencies(u.num_chunks, len(u.unit_offsets) - 1, u.unit_offsets.ctypes.data, len(vchunk),
                                             len(voff) - 1, vchunk.ctypes.data, voff.ctypes.data, plan.ctypes.data,
                                             plan.shape[1] - 4, F)
    assert rc == 0, _lib.lib().dg_last_error()
    for k, li in enumerate(sel):
        cl = at_latency(cfg, u.latencies[li])
        for f, x in enumerate(waveforms):
            v = k * nf + f
            c0, c1 = int(voff[v]), int(voff[v + 1])
            fw = file_windows(x, cl)
            assert c1 - c0 == fw.num_windows
            # the virtual chunks are the first chunks of one unit, whose windows are those of the file at this latency
            u_idx = int(np.searchsorted(u.unit_offsets, vchunk[c0], side="right")) - 1
            assert vchunk[c0] == u.unit_offsets[u_idx] and u_idx == u.unit_of[li, f]
            assert np.array_equal(vchunk[c0:c1], vchunk[c0] + np.arange(c1 - c0))
            ufw = unit_fws[u_idx]
            for i in {0, fw.num_windows // 2, fw.num_windows - 1}:
                assert np.array_equal(ufw.window(i), fw.window(i)), (li, f, i)
            want = stream_plan(fw.starts, cl, F)
            nw = want[0].shape[1] - 4
            assert np.array_equal(plan[c0:c1, :4 + nw], want[0]) and not plan[c0:c1, 4 + nw:].any()
            assert np.array_equal(out_start[c0:c1], want[1]) and np.array_equal(out_res[c0:c1], want[2])
            assert shifts[v] == -fw.padding[0]
    return u


@pytest.mark.parametrize("seed", range(6))
def test_tables_equal_each_latency_alone_for_random_files_and_latencies(seed):
    rng = np.random.default_rng(seed)
    cfg = config(**({"step": 0.3, "latency": 0.9} if seed == 5 else {}))
    lengths = [rng.uniform(0.3, 4.99), rng.uniform(5.0, 40.0), 3.2, 5.0 + rng.uniform(0, 0.5), rng.uniform(0.05, 20)]
    waveforms = [rng.standard_normal(int(s * 16000) + int(rng.integers(0, 7))).astype(np.float32) for s in lengths]
    grid = np.round(np.arange(cfg.step, cfg.duration + 1e-9, cfg.step), 6)
    lats = list(rng.choice(grid, size=int(rng.integers(1, 6)), replace=False)) + ([rng.uniform(cfg.step, cfg.duration)]
                                                                                  if seed % 2 else ["max"])
    u = check_tables(cfg, waveforms, lats)
    # a selection of the latencies: the same rows for the selected ones
    check_tables(cfg, waveforms, lats, sel=[len(u.latencies) - 1, 0][:len(u.latencies)][::-1])


def layout():
    """two units of 4 and 3 chunks; virtual files: unit 0 (3 chunks), unit 1 (3), unit 0 (4); nw = 3"""
    uoff = np.array([0, 4, 7], np.int32)
    vchunk = np.array([0, 1, 2, 4, 5, 6, 0, 1, 2, 3], np.int32)
    voff = np.array([0, 3, 6, 10], np.int32)
    plan = np.zeros((10, 7), np.int32)
    plan[:, 1] = 10
    plan[:, 0] = [1, 2, 2, 1, 2, 3, 1, 2, 3, 3]
    return uoff, vchunk, voff, plan


def check(uoff, vchunk, voff, plan, nw=3, N=7, frames=20):
    c = np.ascontiguousarray
    uoff, vchunk, voff, plan = c(uoff, np.int32), c(vchunk, np.int32), c(voff, np.int32), c(plan, np.int32)
    return _lib.lib().dg_sweep_check_latencies(N, len(uoff) - 1, uoff.ctypes.data, len(vchunk), len(voff) - 1,
                                               vchunk.ctypes.data, voff.ctypes.data, plan.ctypes.data, nw, frames)


def test_layout_checks():
    lib = _lib.lib()
    uoff, vchunk, voff, plan = layout()
    assert check(uoff, vchunk, voff, plan) == 0
    not_first = vchunk.copy()
    not_first[0:3] = [1, 2, 3]                                  # starts inside unit 0
    inside = vchunk.copy()
    inside[6:10] = [2, 3, 4, 5]
    crosses_end = np.array([0, 1, 2, 4, 5, 6, 4, 5, 6, 7], np.int32)
    gap = vchunk.copy()
    gap[7] = 2
    long_plan = plan.copy()
    long_plan[3, 0] = 2                                         # the first chunk of a virtual file aggregates two buffers
    wide_plan = plan.copy()
    wide_plan[9, 0] = 4                                         # more buffers than the handle's plan width
    no_frames = plan.copy()
    no_frames[5, 1] = 0
    too_many_frames = plan.copy()
    too_many_frames[5, 2] = 1024
    past_shared_memory = plan.copy()
    past_shared_memory[0, 2] = 22                               # frames + 2 output frames: more than the post-path holds
    first_chunk = plan.copy()
    first_chunk[0, 2] = 21                                      # frames + 1: the first chunk of a file may emit that many
    assert check(uoff, vchunk, voff, first_chunk) == 0
    cases = {
        "does not start at the first chunk of a unit": dict(vchunk=not_first),
        "crosses into the next unit": dict(vchunk=np.array([0, 1, 2, 3, 4, 5, 0, 1, 2, 3], np.int32),
                                           uoff=np.array([0, 3, 7], np.int32)),
        "not a run of consecutive chunks": dict(vchunk=gap),
        "starts inside a unit": dict(vchunk=inside),
        "runs past the last chunk": dict(vchunk=crosses_end),
        "plan reaches before the first chunk": dict(plan=long_plan),
        "plan wider than the handle": dict(plan=wide_plan),
        "plan without frames": dict(plan=no_frames),
        "plan over 1023 frames": dict(plan=too_many_frames),
        "plan over frames + 1 output frames": dict(plan=past_shared_memory),
        "virtual file without chunks": dict(voff=np.array([0, 3, 3, 10], np.int32)),
        "virtual offsets not ending at the virtual chunks": dict(voff=np.array([0, 3, 6, 9], np.int32)),
        "unit offsets not ending at N": dict(uoff=np.array([0, 4, 6], np.int32)),
    }
    for name, kw in cases.items():
        args = dict(uoff=uoff, vchunk=vchunk, voff=voff, plan=plan)
        args.update(kw)
        assert check(**args) == -1, name
        assert b"dg_sweep_check_latencies" in lib.dg_last_error(), name
    check(uoff, crosses_end, voff, plan)
    assert b"crosses into the next unit" in lib.dg_last_error()
    check(uoff, not_first, voff, plan)
    assert b"does not start at the first chunk of a unit" in lib.dg_last_error()


def test_latency_entry_points_reject_bad_handles_without_a_gpu():
    lib = _lib.lib()
    uoff, vchunk, voff, plan = layout()
    p = np.array([[0.5, 0.3, 1.0]])
    assert lib.dg_sweep_run_latencies(None, None, None, 7, 2, uoff.ctypes.data, 10, 3, vchunk.ctypes.data, voff.ctypes.data,
                                      p.ctypes.data, 1, plan.ctypes.data, None, None, None, 0, None, None) == -1
    assert b"dg_sweep_run_latencies" in lib.dg_last_error()
    assert lib.dg_sweep_score_latencies(None, None, None, 7, 2, uoff.ctypes.data, 10, 3, vchunk.ctypes.data,
                                        voff.ctypes.data, p.ctypes.data, 1, plan.ctypes.data, None, None, None, 0.05, None,
                                        None, None, None, None, None) == -1
    assert b"dg_sweep_score_latencies" in lib.dg_last_error()
    assert lib.dg_vad_sweep_curve_latencies(None, None, 7, 2, uoff.ctypes.data, 10, 3, vchunk.ctypes.data,
                                            voff.ctypes.data, plan.ctypes.data, None) == -1
    assert b"dg_vad_sweep_curve_latencies" in lib.dg_last_error()
