"""CPU tier: pool groups of the pooled safe-set exchange (lmpc_set_pool_groups).

The argument rules of the group index (``_native.make_pool_groups``), the numbering of a crossed design's cells
(``sharding.design_groups``), the grouped host ranking (``sharding.pooled_fastest(groups=)``) against a brute-force sort, and
the refusals of ``rollout_mc.run`` that must come before any device work."""
import os
import sys

import numpy as np
import pytest

from racinglmpc_b200 import _native as nat, sharding
from racinglmpc_b200.reference_params import TrackParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 12


def test_library_exports_set_pool_groups():
    assert "lmpc_set_pool_groups" in nat.exported_symbols()
    assert hasattr(nat.lib(), "lmpc_set_pool_groups")


def test_valid_groups_pass_through():
    idx = np.arange(B) % 3
    out = nat.make_pool_groups(idx, 3, B)
    assert out.dtype == np.int32 and out.flags["C_CONTIGUOUS"] and np.array_equal(out, idx)
    assert nat.make_pool_groups(np.zeros(B, int), 1, B).tolist() == [0] * B
    assert nat.make_pool_groups(np.zeros(B, int), 4, B).tolist() == [0] * B        # empty groups are allowed
    assert nat.make_pool_groups(None, 0, B) is None
    big = 200
    assert np.array_equal(nat.make_pool_groups(np.arange(big) % 64, 64, big), np.arange(big) % 64)


@pytest.mark.parametrize("index, ngroups", [
    (np.zeros(B - 1, int), 2), (np.zeros(B + 1, int), 2),      # wrong length
    (np.full(B, 0.5), 2),                                       # not integers
    (np.full(B, 2), 2), (np.full(B, -1), 2),                    # out of range
    (np.zeros(B, int), B + 1),                                  # more groups than controllers
    (np.zeros(B, int), -1),
    (None, 2),                                                  # groups need an index
    (np.zeros(B, int), 0),                                      # one pool takes no index
])
def test_bad_groups_are_a_value_error(index, ngroups):
    with pytest.raises(ValueError):
        nat.make_pool_groups(index, ngroups, B)


def test_more_than_the_group_limit_is_a_value_error():
    big = 200
    assert nat.MAX_POOL_GROUPS == 64
    with pytest.raises(ValueError):
        nat.make_pool_groups(np.arange(big) % 65, 65, big)


def test_design_groups_number_cells_in_first_appearance_order():
    g, G = sharding.design_groups(np.array([2, 0, 2, 1, 0]))
    assert G == 3 and g.dtype == np.int32 and g.tolist() == [0, 1, 0, 2, 1]
    b = np.arange(24)
    tidx, vidx, pidx = b % 3, (b // 3) % 2, (b // 6) % 2
    g, G = sharding.design_groups(tidx, vidx, pidx)
    assert G == 12
    cells = {}
    for i in range(24):
        cells.setdefault((tidx[i], vidx[i], pidx[i]), set()).add(int(g[i]))
    assert all(len(v) == 1 for v in cells.values()) and len({next(iter(v)) for v in cells.values()}) == 12
    first = [int(g[i]) for i in sorted({min(np.nonzero(g == k)[0]) for k in range(G)})]
    assert first == list(range(G))
    g, G = sharding.design_groups(np.zeros(5, int), np.ones(5, int))
    assert G == 1 and not g.any()
    with pytest.raises(ValueError):
        sharding.design_groups(np.zeros(4, int), np.zeros(5, int))


def _brute(lens, groups, k, valid_min=2):
    out = []
    for g in range(int(max(groups)) + 1):
        cand = sorted((int(lens[i]), i) for i in range(len(lens)) if groups[i] == g and lens[i] >= valid_min)
        out.append([i for _, i in cand[:k]])
    return out


def test_grouped_pooled_fastest_equals_a_brute_force_sort():
    rng = np.random.default_rng(3)
    for trial in range(50):
        n = int(rng.integers(1, 40))
        lens = rng.integers(0, 8, n)                        # many ties, and laps shorter than 2 rows (invalid)
        groups = rng.integers(-1, 5, n)
        if groups.max() < 0:
            groups[0] = 0
        k = int(rng.integers(1, 5))
        got = sharding.pooled_fastest(lens, k, groups=groups)
        assert [list(map(int, a)) for a in got] == _brute(lens, groups, k), trial
    # one group is the ungrouped ranking
    lens = rng.integers(0, 8, 30)
    assert np.array_equal(sharding.pooled_fastest(lens, 4, groups=np.zeros(30, int))[0], sharding.pooled_fastest(lens, 4))


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


@pytest.fixture
def no_device(monkeypatch):
    """Any step towards the device fails the test: the refusals must come first."""
    import torch
    rm = _rollout_mc()

    def boom(*a, **k):
        raise AssertionError("device work before the argument check")
    monkeypatch.setattr(torch.cuda, "set_device", boom)
    monkeypatch.setattr(rm, "BatchedController", boom)
    return rm


def test_rollout_mc_refuses_pooled_tracks_before_any_device_work(no_device):
    rm = no_device
    three = [TrackParams.l_shaped(), TrackParams.goggle(), TrackParams.oval()]
    tidx = np.arange(B) % 3
    with pytest.raises(ValueError, match="pool groups"):
        rm.run(batch=B, mode="pooled", track_sets=(three, tidx))
    spans = tidx.copy()
    spans[0] = 1                                            # group 1 holds a controller of track 0
    with pytest.raises(ValueError, match="spans two tracks"):
        rm.run(batch=B, mode="pooled", track_sets=(three, tidx), pool_groups=(spans, 3))
    with pytest.raises(ValueError, match="spans two tracks"):
        rm.run(batch=B, mode="pooled", track_sets=(three, tidx), pool_groups=(np.zeros(B, np.int32), 1))
    # accepted arguments go on to the device (here: the stub)
    with pytest.raises(AssertionError, match="device work"):
        rm.run(batch=B, mode="pooled", track_sets=(three, tidx), pool_groups=sharding.design_groups(tidx))
    with pytest.raises(AssertionError, match="device work"):
        rm.run(batch=B, mode="independent", track_sets=(three, tidx))
