"""CPU tier: per-controller horizons and safe-set sizes (lmpc_set_shapes).

The struct and the exported symbols, the Python grid against the instantiated grid of csrc/ftocp_launch.cuh, every refusal of
_native.make_shape_sets, and the argument checks of rollout_mc.run(shape_sets=...), all raised before any device work."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import rollout_mc                                                  # noqa: E402

B = 16
# an LMPC handle of the reference's kind (numSS_it = 4) and an MPC handle
LMPC = dict(N=14, M=96, numSS_it=4)
MPC = dict(N=12, M=0, numSS_it=0)


def _grid_of_header():
    txt = open(os.path.join(ROOT, "racinglmpc_b200", "csrc", "ftocp_launch.cuh")).read()
    body = re.search(r"#define LMPC_FOR_EACH_CASE\(X\)((?:.*\\\n)*.*\n)", txt).group(1)
    return sorted((int(n), int(m)) for n, m in re.findall(r"X\((\d+),\s*(\d+)\)", body))


def test_grid_constant_equals_the_instantiated_grid():
    assert sorted(nat.SHAPE_GRID) == _grid_of_header()
    assert len(set(nat.SHAPE_GRID)) == len(nat.SHAPE_GRID) == 30


def test_library_exports_the_call_and_the_struct_size_matches():
    assert {"lmpc_set_shapes", "lmpc_sizeof_shape_params"} <= set(nat.exported_symbols())
    L = nat.lib()                                 # asserts lmpc_sizeof_shape_params() == sizeof(ShapeParams)
    assert L.lmpc_sizeof_shape_params() == C.sizeof(nat.ShapeParams) == 8
    assert L.lmpc_set_shapes(None, None, 0, None) != 0 and b"null handle" in L.lmpc_last_error()


def test_valid_sets_pack_in_order():
    shapes = [(6, 48), (14, 96), (12, 24), (14, 32)]
    idx = np.arange(B) % 4
    packed, pidx = nat.make_shape_sets(shapes, idx, B, **LMPC)
    assert [(p.N, p.numSS_Points) for p in packed] == shapes
    assert pidx.dtype == np.int32 and np.array_equal(pidx, idx)
    packed, _ = nat.make_shape_sets([(4, 0), (12, 0)], np.arange(B) % 2, B, **MPC)
    assert [(p.N, p.numSS_Points) for p in packed] == [(4, 0), (12, 0)]


@pytest.mark.parametrize("shape", [(13, 48), (14, 40), (48, 96), (16, 24), (12, 16)])
def test_pair_off_the_grid_is_refused(shape):
    with pytest.raises(ValueError, match="not an instantiated"):
        nat.make_shape_sets([shape], np.zeros(B, int), B, N=48, M=96, numSS_it=4)


@pytest.mark.parametrize("shape", [(16, 48), (20, 48), (48, 48)])
def test_shape_above_the_handle_is_refused(shape):
    with pytest.raises(ValueError, match="exceeds"):
        nat.make_shape_sets([shape], np.zeros(B, int), B, **LMPC)


def test_safe_set_size_above_the_handle_is_refused():
    with pytest.raises(ValueError, match="exceeds"):
        nat.make_shape_sets([(12, 64)], np.zeros(B, int), B, N=12, M=48, numSS_it=4)


def test_no_safe_set_on_an_lmpc_handle_and_a_safe_set_on_an_mpc_handle_are_refused():
    with pytest.raises(ValueError, match="exactly when"):
        nat.make_shape_sets([(12, 0)], np.zeros(B, int), B, **LMPC)
    with pytest.raises(ValueError):
        nat.make_shape_sets([(12, 48)], np.zeros(B, int), B, **MPC)


def test_odd_points_per_lap_are_refused():
    # numSS_it = 8: 24 / 8 = 3 points per lap; numSS_it = 5 does not divide 48
    with pytest.raises(ValueError, match="even number"):
        nat.make_shape_sets([(12, 24)], np.zeros(B, int), B, N=14, M=96, numSS_it=8)
    with pytest.raises(ValueError, match="even number"):
        nat.make_shape_sets([(12, 48)], np.zeros(B, int), B, N=14, M=96, numSS_it=5)


@pytest.mark.parametrize("shape", [(12,), (12, 48, 1), "ab", (12.0, 48), (True, 48), None])
def test_malformed_shape_is_refused(shape):
    with pytest.raises(ValueError):
        nat.make_shape_sets([shape], np.zeros(B, int), B, **LMPC)


@pytest.mark.parametrize("index", [np.zeros(B - 1, int), np.zeros(B + 1, int), np.full(B, 2), np.full(B, -1), np.full(B, 0.5), None])
def test_bad_index_is_refused(index):
    with pytest.raises(ValueError):
        nat.make_shape_sets([(12, 48), (14, 96)], index, B, **LMPC)


def test_no_shapes_or_more_than_batch_are_refused():
    with pytest.raises(ValueError):
        nat.make_shape_sets([], np.zeros(B, int), B, **LMPC)
    with pytest.raises(ValueError):
        nat.make_shape_sets([(12, 48)] * (B + 1), np.zeros(B, int), B, **LMPC)


def test_driver_picks_the_smallest_dominating_pair():
    assert rollout_mc.handle_shape(None) == (12, 48)
    assert rollout_mc.handle_shape(([(12, 48)], None)) == (12, 48)
    assert rollout_mc.handle_shape(([(6, 48), (12, 24), (14, 96)], None)) == (14, 96)
    assert rollout_mc.handle_shape(([(6, 48), (14, 64)], None)) == (14, 64)
    assert rollout_mc.handle_shape(([(12, 32), (48, 48)], None)) == (48, 48)
    assert rollout_mc.handle_shape(([(16, 48)], None)) == (16, 48)


def test_driver_refuses_shapes_before_any_device_work():
    idx = np.arange(B) % 2
    with pytest.raises(ValueError, match="dominates"):
        rollout_mc.run(batch=B, shape_sets=([(16, 48), (12, 96)], idx))        # nothing on the grid covers N = 16 and 96 points
    with pytest.raises(ValueError, match="not an instantiated"):
        rollout_mc.run(batch=B, shape_sets=([(13, 48), (12, 48)], idx))
    with pytest.raises(ValueError, match="exactly when"):
        rollout_mc.run(batch=B, shape_sets=([(12, 0), (12, 48)], idx))
    with pytest.raises(ValueError):
        rollout_mc.run(batch=B, shape_sets=([(12, 48), (14, 48)], np.zeros(B - 1, int)))
    with pytest.raises(ValueError, match="warm"):
        rollout_mc.run(batch=B, warm=True, shape_sets=([(12, 48)], np.zeros(B, int)))
    with pytest.raises(ValueError):
        rollout_mc.run(batch=B, shape_sets=([], np.zeros(B, int)))


def test_driver_layout_and_start_follow_the_shapes():
    shapes = ([(6, 48), (14, 96)], np.arange(B) % 2)
    assert rollout_mc.layout(shape_sets=shapes)["N"] == 14 and rollout_mc.layout(shape_sets=shapes)["M"] == 96
    assert rollout_mc.layout() == rollout_mc.layout(shape_sets=([(12, 48)], np.zeros(B, int)))
    start = dict(records=np.zeros((B, 1)), clock=0, steps=8, next_round=1, next_rounds=None, exchanged=[False], exchange_steps=[[]],
                 diverged_step=None, batch=B, laps=3, mode="independent", readiness="batch", poll=8, warm=False, pool_groups=1,
                 layout=rollout_mc.layout(), lap_budget=None,
                 tables=rollout_mc.table_rows(rollout_mc.pack_tables(B, shape_sets=shapes)[0]))
    with pytest.raises(ValueError, match="start records have N"):
        rollout_mc.run(batch=B, laps=5, mode="independent", start=start, shape_sets=shapes)
