"""TrajectoryBuffer host logic against the reference's own class (tests/golden/trajbuf_golden.json, written by
oracle/make_golden_trajbuf.py): the keep decisions of the product's index manager and of oracle/trajbuf.py,
filter_points, the degenerate-grid fix, signatures and exports.  No GPU needed."""
import inspect
import json
import os
import random

import numpy as np
import pytest

from oracle.trajbuf import OracleTrajBuf, grid_filter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = json.load(open(os.path.join(ROOT, "tests", "golden", "trajbuf_golden.json")))
SCEN = {s["name"]: s for s in G["scenarios"]}


def _sums(ep):
    ret = cost = 0
    for r, c in zip(ep["rew"], ep["cost"]):      # python-float accumulation of the f32 values, in time order
        ret += r
        cost += c
    return ret, cost


def _seed(s):
    random.seed(s["seed"])
    np.random.seed(s["seed"])


@pytest.mark.parametrize("name", sorted(SCEN))
def test_index_manager_keeps_the_reference_trajectories(name):
    from fsrl_b200.data.traj_buf import TrajectoryIndex
    s = SCEN[name]
    _seed(s)
    ix = TrajectoryIndex(**s["kwargs"])
    owner = {}
    for k, (ep, want) in enumerate(zip(s["episodes"], s["after"])):
        ret, cost = _sums(ep)
        slot = ix.offer(ret, cost, ep["len"])
        if slot is not None:
            owner[slot] = k
        assert [owner[sl] for sl in ix.slots] == want["kept"], (name, k)
        assert [m.tolist() for m in ix.metrics] == want["metrics"], (name, k)
        assert sum(ix.lens[sl] for sl in ix.slots) == want["n_transitions"]
        assert len(set(ix.slots)) == len(ix.slots)
    # memory follows the kept set: slots are reused, never more than the filter threshold
    bound = ix.filtering_thres if ix.use_grid_filter else ix.max_trajectory
    assert ix.n_slots <= max(bound, ix.max_trajectory)


@pytest.mark.parametrize("name", sorted(SCEN))
def test_oracle_keeps_the_reference_trajectories(name):
    s = SCEN[name]
    _seed(s)
    ob = OracleTrajBuf(**s["kwargs"])
    for k, (ep, want) in enumerate(zip(s["episodes"], s["after"])):
        ret, cost = _sums(ep)
        ob.add({"id": np.array([k])}, ret, cost)
        assert [int(t["id"][0]) for t in ob.trajs] == want["kept"], (name, k)
        assert [m.tolist() for m in ob.metrics] == want["metrics"]


@pytest.mark.parametrize("case", G["filter_points"], ids=lambda c: c["name"])
def test_filter_points_matches_reference(case):
    from fsrl_b200.data import TrajectoryBuffer
    pts = [np.array(p) for p in case["points"]]
    random.seed(case["seed"])
    assert TrajectoryBuffer.filter_points(pts, case["target"]) == case["kept"]
    random.seed(case["seed"])
    assert grid_filter(pts, case["target"]) == case["kept"]


def test_degenerate_grid_is_one_cell():
    """The reference raises on a cloud whose points share one coordinate (zero cell size); here that
    dimension is one cell and the filter returns target_size distinct valid indices."""
    from fsrl_b200.data import TrajectoryBuffer
    d = G["degenerate"]
    assert d["reference_error"] == "cannot convert float NaN to integer"
    pts = [np.array(p) for p in d["points"]]
    random.seed(d["seed"])
    got = TrajectoryBuffer.filter_points(pts, d["target"])
    assert len(got) == d["target"] == len(set(got)) and all(0 <= i < len(pts) for i in got)
    random.seed(d["seed"])
    assert grid_filter(pts, d["target"]) == got
    with pytest.raises(ValueError, match="NaN"):
        grid_filter(pts, d["target"], degenerate_fix=False)
    # every point in one spot: one cell in both dimensions
    random.seed(1)
    same = TrajectoryBuffer.filter_points([np.array([1.0, 2.0])] * 12, 5)
    assert sorted(same) == sorted(set(same)) and len(same) == 5


def test_signatures_match_reference():
    from fsrl_b200.data import BasicCollector, TrajectoryBuffer
    for key, want in G["signatures"].items():
        cname, meth = key.split(".")
        cls = {"TrajectoryBuffer": TrajectoryBuffer, "BasicCollector": BasicCollector}[cname]
        ps = inspect.signature(getattr(cls, meth)).parameters.values()
        got = [[p.name, None if p.default is inspect.Parameter.empty else repr(p.default)] for p in ps]
        assert got == want, key


def test_both_names_exported_and_reachable_through_compat():
    import fsrl_b200.compat
    import fsrl_b200.data as data
    assert {"TrajectoryBuffer", "BasicCollector"} <= set(data.__all__)
    fsrl_b200.compat.install()
    import fsrl.data
    assert fsrl.data.TrajectoryBuffer is data.TrajectoryBuffer and fsrl.data.BasicCollector is data.BasicCollector


def test_replay_buffer_of_one_size_is_one_sub_buffer():
    import fsrl_b200.compat
    fsrl_b200.compat.install()
    from tianshou.data import ReplayBuffer
    b = ReplayBuffer(1000)
    assert (b.buffer_num, b.cap, b.maxsize) == (1, 1000, 1000)
    b = ReplayBuffer(1000, 4)
    assert (b.buffer_num, b.cap) == (4, 250)


def test_grid_filter_frees_slots_and_replacement_reuses_one():
    from fsrl_b200.data.traj_buf import TrajectoryIndex
    random.seed(0)
    np.random.seed(0)
    ix = TrajectoryIndex(max_trajectory=3, use_grid_filter=False)
    slots = [ix.offer(float(i), 0.0, 4) for i in range(3)]
    assert slots == [0, 1, 2]
    s = ix.offer(9.0, 0.0, 7)
    assert s in slots and ix.n_slots == 3 and ix.lens[s] == 7
    assert ix.offer(0.0, float("inf"), 1) is not None and ix.offer(0.0, 0.0, 1) is not None
    rng = TrajectoryIndex(max_trajectory=3, rmax=1.0)
    assert rng.offer(2.0, 0.0, 1) is None and len(rng) == 0
