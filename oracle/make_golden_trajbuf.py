"""Golden vectors for TrajectoryBuffer, produced by the reference's OWN class.

Run in the build container only (needs /root/reference; never on the GPU box):

    python oracle/make_golden_trajbuf.py

``oracle.refrun.bootstrap`` makes ``fsrl`` the reference with stand-ins for the absent packages
(``h5py`` is only needed by ``save()``, which is not driven here).  The one tianshou method the buffer
calls, ``Batch.cat`` over a list, is added as a plain concatenation of each key [UNVERIFIED
restatement of tianshou 0.5; the trajectories it builds are only read back for their ids].

Scripted episodes (seeded) go through ``store()`` one transition at a time.  Every transition's first
observation entry is ``1000 * episode + step``, so a kept trajectory is identified by its first id.
After every finished episode the fixture records the kept episodes in order, the metrics and ``len()``.
``filter_points`` is recorded on fixed point clouds, and the ValueError the reference raises on a cloud
whose points share one coordinate.  Writes tests/golden/trajbuf_golden.json.
"""
from __future__ import annotations

import inspect
import json
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "trajbuf_golden.json")
D, A = 3, 2


def episodes(seed, n, max_len=9):
    """episode k: length, f32 rewards / costs per step, whether it ends terminated (else truncated)"""
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        L = int(g.integers(1, max_len + 1))
        rew = (g.normal(size=L) * 2.0).astype(np.float32)
        cost = (g.integers(0, 3, size=L) * (g.random(L) < 0.4)).astype(np.float32)
        out.append(dict(len=L, rew=[float(x) for x in rew], cost=[float(x) for x in cost],
                        terminal=bool(g.random() < 0.5)))
    return out


def transition(Batch, k, t, ep):
    last = t == ep["len"] - 1
    obs = np.array([[1000 * k + t, k, t]], np.float32)
    return Batch(observations=obs, next_observations=obs + 0.5,
                 actions=np.array([[0.25 * t, -0.5 * k]], np.float32),
                 rewards=np.array([ep["rew"][t]], np.float32), costs=np.array([ep["cost"][t]], np.float32),
                 terminals=np.array([last and ep["terminal"]]), timeouts=np.array([last and not ep["terminal"]]))


def run(Batch, TrajectoryBuffer, name, kw, seed, n_ep):
    random.seed(seed)
    np.random.seed(seed)
    eps = episodes(seed, n_ep)
    buf = TrajectoryBuffer(**kw)
    after = []
    for k, ep in enumerate(eps):
        for t in range(ep["len"]):
            buf.store(transition(Batch, k, t, ep))
        after.append(dict(kept=[int(tr["observations"][0, 0]) // 1000 for tr in buf.buffer],
                          metrics=[[float(m[0]), float(m[1])] for m in buf.metrics], n_transitions=len(buf)))
    return dict(name=name, kwargs=kw, seed=seed, episodes=eps, after=after)


def clouds():
    g = np.random.default_rng(5)
    base = g.normal(size=(5, 2))
    dup = base[g.integers(0, 5, size=30)]
    spread = g.normal(size=(40, 2)) * [3.0, 1.0]
    corner = np.concatenate([g.random((20, 2)), [[1.0, 1.0], [0.0, 0.0], [1.0, 1.0]]])
    integer = g.integers(0, 4, size=(25, 2)).astype(np.float64)
    return [("spread", spread, 10, 1), ("duplicates", dup, 7, 2), ("max_coordinate", corner, 9, 3),
            ("integer_grid", integer, 12, 4), ("spread_small_target", spread, 3, 5)]


def main():
    sys.path.insert(0, ROOT)
    from oracle import refrun
    Batch = refrun.bootstrap(REF)

    def cat(batches):
        full = [b for b in batches if not b.is_empty()]
        return Batch({k: np.concatenate([b[k] for b in full]) for k in full[0].keys()}) if full else Batch()
    Batch.cat = staticmethod(cat)

    from fsrl.data.basic_collector import BasicCollector
    from fsrl.data.traj_buf import TrajectoryBuffer

    scen = [
        run(Batch, TrajectoryBuffer, "grid", dict(max_trajectory=6, filter_interval=1.5), 11, 60),
        run(Batch, TrajectoryBuffer, "grid_interval_2", dict(max_trajectory=5), 12, 50),
        run(Batch, TrajectoryBuffer, "replace", dict(max_trajectory=6, use_grid_filter=False), 13, 50),
        run(Batch, TrajectoryBuffer, "window", dict(max_trajectory=5, filter_interval=1.5, rmin=-3.0, rmax=4.0,
                                                    cmin=0.0, cmax=3.0), 14, 60),
    ]
    pts = []
    for name, p, target, seed in clouds():
        random.seed(seed)
        pts.append(dict(name=name, points=p.tolist(), target=target, seed=seed,
                        kept=[int(i) for i in TrajectoryBuffer.filter_points(list(p), target)]))
    degenerate = np.stack([np.linspace(-2.0, 5.0, 30), np.full(30, 3.0)], axis=1)
    random.seed(6)
    try:
        TrajectoryBuffer.filter_points(list(degenerate), 8)
        err = None
    except ValueError as e:
        err = str(e)
    sig = {}
    for cname, cls, meths in (("TrajectoryBuffer", TrajectoryBuffer, ("__init__", "store", "sample", "get_all", "save",
                                                                      "filter_points", "apply_grid_filter")),
                              ("BasicCollector", BasicCollector, ("__init__", "collect", "reset", "reset_env",
                                                                  "reset_buffer", "reset_stat"))):
        for m in meths:
            ps = inspect.signature(getattr(cls, m)).parameters.values()
            sig[f"{cname}.{m}"] = [[p.name, None if p.default is inspect.Parameter.empty else repr(p.default)] for p in ps]
    out = dict(scenarios=scen, filter_points=pts,
               degenerate=dict(points=degenerate.tolist(), target=8, seed=6, reference_error=err), signatures=sig)
    with open(OUT, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", OUT, "degenerate:", err)


if __name__ == "__main__":
    main()
