"""Host side of the sweeps over overlap-aware weightings: building the OSP sets (float32 identity, duplicates, config keys,
non-finite values), mapping trials to (set index, params row), the error messages, and the two C entry points refusing
bad arguments without a device."""
import math

import numpy as np
import pytest

from diart_b200 import _lib
from diart_b200.tune import (MAX_OSP_SETS, osp_dict, osp_index, osp_set, osp_sets, trial_osp_params, trial_osp_sets,
                             trial_params)


class Config:
    gamma, beta, normalize_embedding_weights = 3, 10, False
    tau_active, rho_update, delta_new = 0.6, 0.3, 1.0


CFG = Config()


def test_the_configs_set_comes_first_and_duplicates_collapse():
    sets = osp_sets(CFG, [{"gamma": 2}, {"gamma": 3.0, "beta": 10}, {"beta": 10.0, "gamma": 2.0}, {}, {"beta": 5}])
    assert sets == ((3.0, 10.0, False), (2.0, 10.0, False), (3.0, 5.0, False))
    assert osp_sets(CFG) == ((3.0, 10.0, False),)
    assert osp_sets(CFG, [{"normalize_embedding_weights": True}])[1] == (3.0, 10.0, True)
    assert osp_sets(CFG, [{"normalize_embedding_weights": 1}]) == osp_sets(CFG, [{"normalize_embedding_weights": True}])


def test_equal_float32_values_are_one_set():
    a, b = 2.5, 2.5 + 1e-9                          # distinct float64, one float32
    assert a != b and np.float32(a) == np.float32(b)
    assert len(osp_sets(CFG, [{"gamma": a}, {"gamma": b}])) == 2
    assert osp_set({"gamma": 0.1}, CFG)[0] == float(np.float32(0.1)) != 0.1
    c = float(np.nextafter(np.float32(2.5), np.float32(3)))
    assert len(osp_sets(CFG, [{"gamma": a}, {"gamma": c}])) == 3


@pytest.mark.parametrize("bad", [{"gamma": math.nan}, {"beta": math.inf}, {"beta": -math.inf}])
def test_non_finite_values_are_refused(bad):
    with pytest.raises(ValueError, match="finite"):
        osp_sets(CFG, [bad])


def test_unknown_keys_and_too_many_sets_are_refused():
    with pytest.raises(ValueError, match="unknown keys \\['tau_active'\\]"):
        osp_sets(CFG, [{"tau_active": 0.5}])
    with pytest.raises(ValueError, match="at most 64"):
        osp_sets(CFG, [{"gamma": 0.5 + i} for i in range(MAX_OSP_SETS)])
    assert len(osp_sets(CFG, [{"gamma": 0.5 + i} for i in range(MAX_OSP_SETS - 1)])) == MAX_OSP_SETS


def test_trials_map_to_a_set_index_and_a_params_row():
    sets = osp_sets(CFG, [{"gamma": 2}, {"beta": 5, "normalize_embedding_weights": True}])
    trials = [{}, {"gamma": 2, "tau_active": 0.5}, {"beta": 5.0, "normalize_embedding_weights": True, "delta_new": 0.7},
              {"gamma": 3, "beta": 10, "rho_update": 0.1}]
    index, params = trial_osp_params(trials, CFG, sets)
    assert index.dtype == np.int32 and index.tolist() == [0, 1, 2, 0]
    assert np.array_equal(params, trial_params([{}, {"tau_active": 0.5}, {"delta_new": 0.7}, {"rho_update": 0.1}], CFG))
    assert trial_osp_sets(CFG, trials) == sets
    assert trial_osp_sets(CFG, [{"tau_active": 0.4}]) == osp_sets(CFG)


def test_messages_name_the_trial_and_the_constructed_sets():
    sets = osp_sets(CFG, [{"gamma": 2}])
    with pytest.raises(ValueError) as e:
        trial_osp_params([{}, {"gamma": 4, "tau_active": 0.5}], CFG, sets)
    msg = str(e.value)
    assert msg.startswith("trial 1: OSP set {'gamma': 4.0, 'beta': 10.0, 'normalize_embedding_weights': False} was not "
                          "constructed")
    assert "{'gamma': 2.0, 'beta': 10.0, 'normalize_embedding_weights': False}" in msg
    with pytest.raises(ValueError, match="was not constructed"):
        osp_index(CFG, sets, {"normalize_embedding_weights": True})
    assert osp_index(CFG, sets, {"gamma": 2.0}) == 1
    assert osp_dict(sets[1]) == {"gamma": 2.0, "beta": 10.0, "normalize_embedding_weights": False}
    # the other keys are still trial_params' to refuse
    with pytest.raises(ValueError, match="cannot be swept"):
        trial_osp_params([{"gamma": 2, "latency": 1.0}], CFG, sets)
    with pytest.raises(ValueError, match="at least one trial"):
        trial_osp_params([], CFG, sets)


def test_entry_points_refuse_without_a_device():
    lib = _lib.lib()
    idx = np.zeros(2, np.int32)
    osp = np.array([[3, 10]], np.float32)
    norm = np.zeros(1, np.int32)
    assert lib.dg_sweep_set_trial_sets(None, 1, idx.ctypes.data, 2) == -1
    assert b"null handle" in lib.dg_last_error()
    assert lib.dg_sweep_set_trial_sets(None, 1, None, 2) == -1
    assert lib.dg_sweep_set_trial_sets(None, -1, None, 0) == -1
    bad = np.array([0, 3], np.int32)
    assert lib.dg_sweep_set_trial_sets(None, 2, bad.ctypes.data, 2) == -1
    assert b"outside [0, 2)" in lib.dg_last_error()
    assert lib.dg_pipeline_nets_sets(None, None, 1, 80000, 1, osp.ctypes.data, norm.ctypes.data, None, None, 0, None) == -1
    assert b"dg_pipeline_nets_sets" in lib.dg_last_error()
