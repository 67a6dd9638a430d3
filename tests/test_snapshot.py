"""CPU tier: the pure-Python side of controller snapshots -- the record header decoder and its layout-mismatch messages on
hand-built headers, the destination and index rules, the tensor checks, and the refusals of rollout_mc.run(capture=, start=)
-- all without a device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from racinglmpc_b200 import _native as nat, reference_params as rp
from racinglmpc_b200.reference_params import TrackParams

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYOUT = dict(N=12, M=48, ncx=2, ncu=4, numSS_it=4, trToUse=4, ss_cap=7, model_cap=5, Tmax=1280, Tcl=1024, warm_start=0,
              bytes=1114240)


def _header(**over):
    h = nat.SnapshotHeader()
    h.magic, h.version, h.bytes = nat.SNAPSHOT_MAGIC, nat.SNAPSHOT_VERSION, LAYOUT["bytes"]
    for f in nat.SNAPSHOT_LAYOUT:
        setattr(h, f, LAYOUT[f])
    h.warm_mode, h.nsect = -1, nat.SNAPSHOT_SECTIONS
    h.sect_off[0], h.sect_bytes[0] = 784, 7 * 1280 * 48
    h.sect_off[3], h.sect_bytes[3] = 784 + 7 * 1280 * 48, 28
    t = TrackParams.l_shaped()
    h.track.nseg = t.seg_table.shape[0]
    h.track.seg[:t.seg_table.size] = list(t.seg_table.ravel())
    h.track.TrackLength = t.TrackLength
    for k, v in over.items():
        setattr(h, k, v)
    return bytes(h)


def test_header_size_and_decode():
    assert C.sizeof(nat.SnapshotHeader) == 784 and C.sizeof(nat.SnapshotHeader) % 16 == 0
    d = nat.decode_snapshot_header(_header())
    assert d["magic"] == nat.SNAPSHOT_MAGIC and d["version"] == nat.SNAPSHOT_VERSION and d["warm_mode"] == -1
    assert {f: d[f] for f in nat.SNAPSHOT_LAYOUT} == {f: LAYOUT[f] for f in nat.SNAPSHOT_LAYOUT}
    assert d["sections"] == {"ss_x": (784, 7 * 1280 * 48), "ss_len": (784 + 7 * 1280 * 48, 28)}
    t = TrackParams.l_shaped()
    assert d["track"]["nseg"] == t.seg_table.shape[0] and np.array_equal(d["track"]["seg"], t.seg_table)
    assert d["track"]["TrackLength"] == t.TrackLength
    # the same bytes as a uint8 array or a CPU tensor, with a record body behind the header
    raw = np.frombuffer(_header() + bytes(64), np.uint8)
    assert nat.decode_snapshot_header(raw)["Tmax"] == 1280
    assert nat.decode_snapshot_header(torch.from_numpy(raw.copy()))["Tcl"] == 1024
    assert len(nat.SNAPSHOT_SECTIONS_NAMES) <= nat.SNAPSHOT_SECTIONS


def test_header_refusals():
    with pytest.raises(ValueError, match="magic"):
        nat.decode_snapshot_header(_header(magic=0x12345678))
    with pytest.raises(ValueError, match="version 2"):
        nat.decode_snapshot_header(_header(version=2))
    with pytest.raises(ValueError, match="784-byte header"):
        nat.decode_snapshot_header(_header()[:100])


@pytest.mark.parametrize("field,value", [("N", 14), ("M", 24), ("Tmax", 1024), ("ss_cap", 6), ("model_cap", 4), ("Tcl", 0),
                                         ("warm_start", 1), ("trToUse", 3), ("numSS_it", 2), ("bytes", 1000000)])
def test_layout_mismatch_names_the_field(field, value):
    d = nat.decode_snapshot_header(_header(**{field: value}))
    msg = nat.snapshot_layout_mismatch(d, LAYOUT)
    assert msg is not None and ("%s is %d in the record and %d in this controller" % (field, value, LAYOUT[field])) in msg
    assert nat.snapshot_layout_mismatch(nat.decode_snapshot_header(_header()), LAYOUT) is None


def test_destination_and_index_rules():
    assert nat.snapshot_indices(None, 8, "inst") is None
    assert nat.snapshot_indices([3, 3, 1], 8, "inst").tolist() == [3, 3, 1]            # repeated sources are allowed
    assert nat.snapshot_indices(np.array([7], np.int64), 8, "inst").dtype == np.int32
    with pytest.raises(ValueError, match="only once"):
        nat.snapshot_indices([1, 2, 1], 8, "inst", unique=True)
    for bad, what in (([8], "out of range"), ([-1], "out of range"), ([], "at least one"), ([1.5], "integer")):
        with pytest.raises(ValueError, match=what):
            nat.snapshot_indices(bad, 8, "inst", unique=True)
    assert nat.snapshot_record_map(None, 3, 5).tolist() == [0, 1, 2]
    assert nat.snapshot_record_map([1, 0, 1, 1], 4, 2).tolist() == [1, 0, 1, 1]        # one record into many controllers
    with pytest.raises(ValueError, match="rec_of"):
        nat.snapshot_record_map(None, 6, 5)
    with pytest.raises(ValueError, match="one integer record index per destination"):
        nat.snapshot_record_map([0, 1], 3, 5)
    with pytest.raises(ValueError, match="out of range"):
        nat.snapshot_record_map([0, 5, 1], 3, 5)


def test_record_tensor_checks():
    cpu = torch.zeros((2, 32), dtype=torch.uint8)
    with pytest.raises(ValueError, match="cuda:0"):
        nat.check_snapshot_tensor(cpu, 0, 32)
    with pytest.raises(ValueError, match="uint8"):
        nat.check_snapshot_tensor(torch.zeros((2, 32), dtype=torch.int32), 0, 32)
    with pytest.raises(ValueError, match="torch tensor"):
        nat.check_snapshot_tensor(np.zeros((2, 32), np.uint8), 0, 32)


def _rollout_mc():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    try:
        import rollout_mc
    finally:
        sys.path.pop(0)
    return rollout_mc


def _capture(**over):
    numSS_it, numSS_Points = rp.lmpc_params(12)[:2]
    cap = dict(records=torch.zeros((16, 32), dtype=torch.uint8), clock=1400, steps=400, next_round=3, next_rounds=None,
               exchanged=[False], exchange_steps=[[200, 320]], diverged_step=None, batch=16, laps=3, mode="pooled",
               readiness="batch", poll=8, warm=False, pool_groups=1, tables={},
               layout=dict(N=12, M=numSS_Points, ncx=2, ncu=4, numSS_it=numSS_it, trToUse=4, ss_cap=7, model_cap=5, Tmax=1280, Tcl=1024,
                           warm_start=0))
    cap.update(over)
    return cap


@pytest.mark.parametrize("over,kw,match", [
    ({}, dict(laps=3), "laps"),
    ({}, dict(laps=2), "laps"),
    ({"batch": 32}, {}, "batch"),
    ({"records": torch.zeros((8, 32), dtype=torch.uint8)}, {}, "records"),
    ({"mode": "independent"}, {}, "mode"),
    ({"readiness": "group"}, {}, "readiness"),
    ({"poll": 16}, {}, "poll"),
    ({"warm": True}, {}, "warm"),
    ({"pool_groups": 3}, {}, "pool groups"),
    ({"layout": dict(_capture()["layout"], Tmax=1024)}, {}, "Tmax"),
    ({"layout": dict(_capture()["layout"], ss_cap=6)}, {}, "ss_cap"),
])
def test_rollout_mc_refuses_a_start_that_does_not_match(over, kw, match):
    rm = _rollout_mc()
    args = dict(batch=16, laps=5, local=0)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        rm.run(start=_capture(**over), **args)


def test_rollout_mc_argument_refusals():
    rm = _rollout_mc()
    with pytest.raises(ValueError, match="lacks"):
        rm.run(batch=16, laps=5, local=0, start={"records": None})
    with pytest.raises(ValueError, match="capture dict"):
        rm.run(batch=16, laps=5, local=0, start=[1, 2])
    with pytest.raises(ValueError, match="capture is a dict"):
        rm.run(batch=16, laps=5, local=0, capture=[])
