"""Plain-numpy restatement of the reference's ``TrajectoryBuffer`` keep rules
(/root/reference/fsrl/data/traj_buf.py:60-161) over whole trajectories -- test infrastructure, written
separately from the product's index manager (fsrl_b200/data/traj_buf.py) so that the two can be
checked against each other and against the reference's own fixture (tests/golden/trajbuf_golden.json).

A trajectory is a dict of numpy arrays; ``add(traj, ret, cost)`` is what ``store()`` does when a
trajectory ends.  Draws: ``random.choice`` for the grid filter, ``np.random.randint`` for replacement,
in the reference's order.  ``degenerate_fix`` selects this project's handling of a zero-width grid
dimension (one cell); without it such a cloud raises ValueError like the reference.
"""
from __future__ import annotations

import math
import random

import numpy as np


def grid_filter(points, target_size, degenerate_fix=True):
    pts = [(float(p[0]), float(p[1])) for p in points]
    side = int(math.ceil(math.sqrt(target_size)))
    cell_of = []
    for d in range(2):
        col = np.array([p[d] for p in pts])
        lo, size = col.min(), (col.max() - col.min()) / side
        if size == 0:
            if not degenerate_fix:
                raise ValueError("cannot convert float NaN to integer")
            cell_of.append([0] * len(pts))
        else:
            cell_of.append([int(np.floor_divide(v - lo, size)) for v in col])
    order, members = [], {}
    for i in range(len(pts)):
        key = (cell_of[0][i], cell_of[1][i])
        if key not in members:
            members[key] = []
            order.append(key)
        members[key].append(i)
    out = []
    for key in order:
        out.append(members[key][-1])
        members[key] = members[key][:-1]
    live = [key for key in order if members[key]]
    while len(out) < target_size:
        key = random.choice(live)
        out.append(members[key][-1])
        members[key] = members[key][:-1]
        if not members[key]:
            live.remove(key)
    return out[:target_size]


class OracleTrajBuf:
    def __init__(self, max_trajectory=99999, use_grid_filter=True, rmin=-np.inf, rmax=np.inf, cmin=-np.inf,
                 cmax=np.inf, filter_interval=2):
        self.max_trajectory, self.use_grid_filter = max_trajectory, use_grid_filter
        self.window = (rmin, rmax, cmin, cmax)
        self.thres = int(filter_interval * max_trajectory) if use_grid_filter else None
        self.trajs, self.metrics = [], []

    def add(self, traj, ret, cost):
        rmin, rmax, cmin, cmax = self.window
        if not (rmin <= ret <= rmax and cmin <= cost <= cmax):
            return
        m = np.array([ret, cost])
        if len(self.trajs) >= self.max_trajectory and not self.use_grid_filter:
            k = np.random.randint(0, len(self.trajs))
            self.trajs[k], self.metrics[k] = traj, m
            return
        full = len(self.trajs) >= self.max_trajectory
        self.trajs.append(traj)
        self.metrics.append(m)
        if full and len(self.trajs) >= self.thres:
            keep = set(grid_filter(self.metrics, self.max_trajectory))
            self.trajs = [t for i, t in enumerate(self.trajs) if i in keep]
            self.metrics = [x for i, x in enumerate(self.metrics) if i in keep]

    def concat(self):
        keys = self.trajs[0].keys()
        return {k: np.concatenate([t[k] for t in self.trajs]) for k in keys}
