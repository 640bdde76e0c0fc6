"""``TrajectoryBuffer`` with the reference's constructor and keep rules
(/root/reference/fsrl/data/traj_buf.py:12-207): finished trajectories whose return and cost lie in
``[rmin, rmax] x [cmin, cmax]`` are kept, up to ``max_trajectory``; past that, either a density grid
filter over the (return, cost) plane thins the kept set back to ``max_trajectory`` once it reaches
``filter_interval * max_trajectory``, or a uniformly drawn kept trajectory is replaced.

The buffer is split in two:

* :class:`TrajectoryIndex` -- pure host bookkeeping: the metrics, the logical order, which arena
  slot holds which trajectory, the filters.  It draws from the global ``random`` (grid filter) and
  ``np.random`` (replacement) exactly as the reference does, so ``seed_all`` gives the same dataset.
* a device arena of fixed-stride slots (one trajectory per slot, stride = the env's
  ``max_episode_steps``) that collectors fill straight from their rollout ring
  (csrc/trajbuf.cu).  A grid filter only rewrites the order list and frees slots; a replacement
  writes one slot.  The arena grows with the number of slots in use, not with ``max_trajectory``.

Deviations from the reference, on purpose:

* ``filter_points`` treats a dimension in which every point has the same value as one cell; the
  reference divides by a zero cell size there and raises ``ValueError`` (cannot convert NaN).
* ``sample(batch_size)`` returns ``batch_size`` transitions; the reference's ``Batch.cat`` call
  with two arguments does not concatenate.
* ``save()`` writes NumPy's compressed ``.npz`` (f32 data, bool flags) instead of HDF5.
"""
from __future__ import annotations

import ctypes
import os
import random
from collections.abc import Sequence
from typing import Dict, List, Optional

import numpy as np
import torch

from .batch import Batch

KEYS = ("observations", "next_observations", "actions", "rewards", "costs", "terminals", "timeouts")


class TrajectoryIndex:
    """Which trajectories the buffer keeps, in which order, and where their data lives.

    ``offer()`` applies the reference's decision for one finished trajectory and returns the arena
    slot its data must be written to, or None when it is not kept.  A slot freed by a later
    decision (grid filter, replacement) may be handed out again at once."""

    def __init__(self, max_trajectory: int = 99999, use_grid_filter: bool = True, rmin: float = -np.inf,
                 rmax: float = np.inf, cmin: float = -np.inf, cmax: float = np.inf, filter_interval: float = 2):
        self.max_trajectory = max_trajectory
        self.rmin, self.rmax, self.cmin, self.cmax = rmin, rmax, cmin, cmax
        self.use_grid_filter = use_grid_filter
        if use_grid_filter:
            assert filter_interval > 1, "the filter interval should be greater than 1"
            self.filtering_thres = int(filter_interval * max_trajectory)
        self.metrics: List[np.ndarray] = []     # logical order
        self.slots: List[int] = []              # logical index -> arena slot
        self.lens: List[int] = []               # arena slot -> trajectory length
        self._free: List[int] = []

    @property
    def n_slots(self) -> int:
        """arena slots handed out so far (the arena must hold this many)"""
        return len(self.lens)

    def _take(self, length: int) -> int:
        if self._free:
            slot = self._free.pop()
            self.lens[slot] = length
        else:
            slot = len(self.lens)
            self.lens.append(length)
        return slot

    def offer(self, rew: float, cost: float, length: int) -> Optional[int]:
        if rew > self.rmax or rew < self.rmin or cost > self.cmax or cost < self.cmin:
            return None
        metric = np.array([rew, cost])
        if len(self.slots) < self.max_trajectory or self.use_grid_filter:
            slot = self._take(length)
            self.slots.append(slot)
            self.metrics.append(metric)
            if len(self.slots) > self.max_trajectory and len(self.slots) >= self.filtering_thres:
                self.apply_grid_filter()
            return slot
        i = np.random.randint(0, len(self.slots))
        self._free.append(self.slots[i])
        slot = self._take(length)
        self.slots[i], self.metrics[i] = slot, metric
        return slot

    def apply_grid_filter(self) -> None:
        keep = set(filter_points(self.metrics, self.max_trajectory))
        slots, metrics = [], []
        for i, (s, m) in enumerate(zip(self.slots, self.metrics)):
            if i in keep:
                slots.append(s)
                metrics.append(m)
            else:
                self._free.append(s)
        self.slots, self.metrics = slots, metrics

    def __len__(self) -> int:
        return len(self.slots)


def filter_points(points, target_size: int) -> list:
    """Indices of at most ``target_size`` of the 2-D ``points`` that keep their spread over the plane.

    The bounding box is cut into ``ceil(sqrt(target_size))`` cells per side (a side of zero width is
    one cell).  Cells are visited in the order their first point appears; each gives up its last
    point, then ``random.choice`` over the cells that still hold points, in that same order, takes
    the last remaining point of the chosen cell until ``target_size`` indices are picked."""
    pts = np.array(points)
    n_side = int(np.ceil(np.sqrt(target_size)))
    lo, hi = pts.min(axis=0), pts.max(axis=0)
    width = (hi - lo) / n_side
    flat = width == 0
    cell_xy = np.floor_divide(pts - lo, np.where(flat, 1.0, width))
    cell_xy[:, flat] = 0
    cells: Dict[tuple, list] = {}
    for i, c in enumerate(map(tuple, cell_xy.astype(np.int64).tolist())):
        cells.setdefault(c, []).append(i)
    picked = [members.pop() for members in cells.values()]
    open_cells = [c for c, members in cells.items() if members]
    while len(picked) < target_size:
        c = random.choice(open_cells)
        picked.append(cells[c].pop())
        if not cells[c]:
            open_cells.remove(c)
    return picked[:target_size]


class _Arena:
    """Fixed-stride device slots: field[k][slot * stride + t]."""

    def __init__(self):
        self.capacity = self.stride = self.D = self.A = 0
        self.device = None
        self.t: Dict[str, torch.Tensor] = {}

    def reserve(self, n_slots: int, stride: int, D: int, A: int, device) -> None:
        device = torch.device(device)
        if self.capacity and (D, A, device) != (self.D, self.A, self.device):
            raise ValueError(f"trajectory arena holds D={self.D}, A={self.A} on {self.device}; "
                             f"got D={D}, A={A} on {device}")
        if n_slots <= self.capacity and stride <= self.stride:
            return
        cap = max(n_slots, 2 * self.capacity, 16)
        stride = max(stride, self.stride)
        new = {}
        for k, (width, dtype) in _fields(D, A).items():
            shape = (cap, stride, width) if width else (cap, stride)
            new[k] = torch.zeros(shape, dtype=dtype, device=device)
            if self.capacity:
                old = self.t[k].view((self.capacity, self.stride) + ((width,) if width else ()))
                new[k][:self.capacity, :self.stride] = old
            new[k] = new[k].view(-1, width) if width else new[k].view(-1)
        self.t, self.capacity, self.stride, self.D, self.A, self.device = new, cap, stride, D, A, device

    def descriptor(self):
        from .. import _lib
        a = _lib.TrajArena()
        t = self.t
        a.obs, a.obs_next, a.act = t["observations"].data_ptr(), t["next_observations"].data_ptr(), t["actions"].data_ptr()
        a.rew, a.cost = t["rewards"].data_ptr(), t["costs"].data_ptr()
        a.term, a.trunc = t["terminals"].data_ptr(), t["timeouts"].data_ptr()
        a.stride, a.n_slots, a.D, a.A = self.stride, self.capacity, self.D, self.A
        return a


def _fields(D: int, A: int):
    f32, u8 = torch.float32, torch.uint8
    return {"observations": (D, f32), "next_observations": (D, f32), "actions": (A, f32), "rewards": (0, f32),
            "costs": (0, f32), "terminals": (0, u8), "timeouts": (0, u8)}


def _packed(n: int, D: int, A: int, device):
    """contiguous output tensors + their arena descriptor (stride 1: one row per transition)"""
    out = {k: torch.empty((n, w) if w else (n,), dtype=dt, device=device) for k, (w, dt) in _fields(D, A).items()}
    arena = _Arena()
    arena.t, arena.capacity, arena.stride, arena.D, arena.A, arena.device = out, n, 1, D, A, torch.device(device)
    return out, arena


def _as_batch(t: Dict[str, torch.Tensor]) -> Batch:
    return Batch({k: (v.bool() if k in ("terminals", "timeouts") else v) for k, v in t.items()})


class _Trajectories(Sequence):
    """``TrajectoryBuffer.buffer``: one Batch of device tensors (views into the arena) per kept trajectory."""

    def __init__(self, owner: "TrajectoryBuffer"):
        self._owner = owner

    def __len__(self) -> int:
        return len(self._owner._index)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        ix, ar = self._owner._index, self._owner._arena
        slot = ix.slots[i]
        lo = slot * ar.stride
        return _as_batch({k: v[lo:lo + ix.lens[slot]] for k, v in ar.t.items()})


class TrajectoryBuffer:
    """Keeps finished trajectories whose return and cost lie in the given window; see the module docstring.

    :param int max_trajectory: number of trajectories to keep. (default=99999)
    :param bool use_grid_filter: thin by density over (return, cost) instead of random replacement.
    :param float rmin, rmax, cmin, cmax: the window a trajectory's return and cost must lie in.
    :param float filter_interval: with the grid filter, it runs when the kept set reaches
        ``int(filter_interval * max_trajectory)`` trajectories. (default=2)
    """

    def __init__(self, max_trajectory: int = 99999, use_grid_filter: bool = True, rmin: float = -np.inf,
                 rmax: float = np.inf, cmin: float = -np.inf, cmax: float = np.inf, filter_interval: float = 2):
        self._index = TrajectoryIndex(max_trajectory, use_grid_filter, rmin, rmax, cmin, cmax, filter_interval)
        self.max_trajectory = max_trajectory
        self.rmin, self.rmax, self.cmin, self.cmax = rmin, rmax, cmin, cmax
        self.use_grid_filter = use_grid_filter
        if use_grid_filter:
            self.filtering_thres = self._index.filtering_thres
        self._arena = _Arena()
        self._open: List[Batch] = []
        self.current_rew, self.current_cost = 0, 0

    filter_points = staticmethod(filter_points)

    @property
    def metrics(self) -> List[np.ndarray]:
        return self._index.metrics

    @property
    def buffer(self) -> Sequence:
        return _Trajectories(self)

    def __len__(self) -> int:
        return int(sum(self._index.lens[s] for s in self._index.slots))

    def apply_grid_filter(self) -> None:
        self._index.apply_grid_filter()

    # ---- per-transition host API (basic_collector.py:238-248) ----------------------------------------
    def store(self, data: Batch) -> None:
        """Append one transition (keys ``observations``, ``next_observations``, ``actions``, ``rewards``,
        ``costs``, ``terminals``, ``timeouts``, each with a leading axis of 1) to the open trajectory; at
        ``terminals or timeouts`` the trajectory is offered to the buffer like a harvested episode."""
        self._open.append(data)
        done = bool(np.asarray(_host(data["terminals"])).item()) or bool(np.asarray(_host(data["timeouts"])).item())
        self.current_rew += np.asarray(_host(data["rewards"])).item()
        self.current_cost += np.asarray(_host(data["costs"])).item()
        if done:
            steps, self._open = self._open, []
            rew, cost = self.current_rew, self.current_cost
            self.current_rew, self.current_cost = 0, 0
            slot = self._index.offer(rew, cost, len(steps))
            if slot is not None:
                self._write_host(slot, steps)

    def _write_host(self, slot: int, steps: List[Batch]) -> None:
        cols = {k: np.concatenate([np.asarray(_host(s[k])).reshape(1, -1) for s in steps]) for k in KEYS}
        D, A = cols["observations"].shape[1], cols["actions"].shape[1]
        device = self._arena.device or torch.device("cuda")
        self._arena.reserve(self._index.n_slots, len(steps), D, A, device)
        lo = slot * self._arena.stride
        for k, (w, dt) in _fields(D, A).items():
            v = torch.from_numpy(np.ascontiguousarray(cols[k] if w else cols[k][:, 0])).to(dt)
            self._arena.t[k][lo:lo + len(steps)].copy_(v)

    # ---- device harvest (csrc/trajbuf.cu) -----------------------------------------------------------------
    def _commit(self, r, rows: np.ndarray, stride: int, D: int, A: int, device, stream: int) -> None:
        """Offer harvested episodes in order; copy the ones still kept at the end straight from the ring."""
        from .. import _lib
        jobs = self._offer_episodes((int(row["env"]), int(row["start"]), int(row["len"]), float(row["ret"]),
                                     float(row["cost"])) for row in rows)
        if not jobs:
            return
        self._arena.reserve(self._index.n_slots, stride, D, A, device)
        jt = torch.tensor(jobs, dtype=torch.int32).to(device)
        a = self._arena.descriptor()
        _lib.check(_lib.lib.fsrl_traj_copy(ctypes.byref(r), ctypes.byref(a), jt.data_ptr(), len(jobs), stream))

    def _offer_episodes(self, episodes) -> List[tuple]:
        """Offer finished episodes (env, ring start, length, return, cost) in order; the copy jobs
        (env, start, length, arena slot) of the ones still kept after the last offer."""
        pending = {}
        for env, start, length, ret, cost in episodes:
            slot = self._index.offer(ret, cost, length)
            if slot is not None:
                pending[slot] = (env, start, length, slot)
        live = set(self._index.slots)
        return [j for s, j in pending.items() if s in live]

    def _copy_host(self, r, jobs: List[tuple], stride: int, D: int, A: int, device, stream: int) -> None:
        """Copy kept episodes from the ring of host-stepped envs (``fsrl_traj_copy_host``); the arena stride grows to
        ``stride`` or the longest of them."""
        from .. import _lib
        if not jobs:
            return
        self._arena.reserve(self._index.n_slots, max([stride] + [j[2] for j in jobs]), D, A, device)
        jt = torch.tensor(jobs, dtype=torch.int32).to(device)
        a = self._arena.descriptor()
        _lib.check(_lib.lib.fsrl_traj_copy_host(ctypes.byref(r), ctypes.byref(a), D, A, jt.data_ptr(), len(jobs),
                                                stream))

    # ---- read-out ----------------------------------------------------------------------------------------------
    def _gather(self, jobs: np.ndarray, n: int, src: "_Arena") -> Dict[str, torch.Tensor]:
        from .. import _lib
        out, packed = _packed(n, src.D, src.A, src.device)
        if len(jobs):
            jt = torch.from_numpy(np.ascontiguousarray(jobs, dtype=np.int64)).to(src.device)
            a, o = src.descriptor(), packed.descriptor()
            with torch.cuda.device(src.device):
                stream = torch.cuda.current_stream().cuda_stream
                _lib.check(_lib.lib.fsrl_traj_gather(ctypes.byref(a), ctypes.byref(o), jt.data_ptr(), len(jobs), stream))
        return out

    def get_all(self) -> Batch:
        """Every kept transition, trajectory after trajectory in the buffer's order, as one Batch of contiguous
        device tensors: observations / next_observations [N, D], actions [N, A] (as the env received them),
        rewards / costs [N] float32, terminals / timeouts [N] bool."""
        if not len(self._index):
            return Batch()
        ix = self._index
        lens = np.array([ix.lens[s] for s in ix.slots], dtype=np.int64)
        first = np.concatenate([[0], np.cumsum(lens)[:-1]])
        jobs = np.stack([np.array(ix.slots, dtype=np.int64), lens, first], axis=1)
        return _as_batch(self._gather(jobs, int(lens.sum()), self._arena))

    def sample(self, batch_size: int) -> Batch:
        """``batch_size`` transitions: a trajectory uniformly (``np.random.randint`` over the kept set), then a
        transition uniformly inside it, drawn in the reference's order."""
        ix, ar = self._index, self._arena
        traj = np.random.randint(0, len(ix), size=batch_size)
        rows = np.empty(batch_size, dtype=np.int64)
        for i in range(batch_size):
            slot = ix.slots[traj[i]]
            rows[i] = slot * ar.stride + np.random.randint(0, ix.lens[slot])
        flat = _Arena()                           # the same storage seen as one-transition slots
        flat.t, flat.capacity, flat.stride, flat.D, flat.A, flat.device = ar.t, ar.capacity * ar.stride, 1, ar.D, ar.A, ar.device
        jobs = np.stack([rows, np.ones(batch_size, np.int64), np.arange(batch_size, dtype=np.int64)], axis=1)
        return _as_batch(self._gather(jobs, batch_size, flat))

    def save(self, log_dir: str, dataset_name: str = "dataset.hdf5") -> None:
        """Write ``get_all()`` to ``<log_dir>/<stem of dataset_name>.npz`` (compressed; the seven keys)."""
        print("Saving dataset...")
        if not os.path.exists(log_dir):
            print(f"Creating saving dir {log_dir}")
            os.makedirs(log_dir)
        path = os.path.join(log_dir, os.path.splitext(dataset_name)[0] + ".npz")
        data = self.get_all()
        np.savez_compressed(path, **{k: data[k].cpu().numpy() for k in KEYS} if len(self._index) else {})
        print(f"Finish saving dataset to {path}!")


def _host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x


# ---- per-collector harvest state ---------------------------------------------------------------------------------
ROW_DTYPE = np.dtype([("env", "<i4"), ("start", "<i4"), ("len", "<i4"), ("finish", "<i4"), ("terminated", "<i4"),
                      ("truncated", "<i4"), ("ret", "<f8"), ("cost", "<f8")])


class TrajectoryHarvest:
    """Device state of the ring scan for one collector's envs (``fsrl_traj_scan_t``)."""

    def __init__(self, env_num: int, device):
        self.E, self.device = int(env_num), torch.device(device)
        i32 = lambda: torch.zeros(self.E, dtype=torch.int32, device=self.device)
        f64 = lambda: torch.zeros(self.E, dtype=torch.float64, device=self.device)
        self.last, self.open, self.open_len, self.steps = i32(), i32(), i32(), i32()
        self.rew, self.cost = f64(), f64()
        self.n_rows = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.rows = torch.zeros(0, dtype=torch.uint8, device=self.device)
        self.row_cap = 0

    def _desc(self, row_cap: int):
        from .. import _lib
        if row_cap > self.row_cap:
            self.rows = torch.zeros(row_cap * ROW_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
            self.row_cap = row_cap
        h = _lib.TrajScan()
        h.last, h.open, h.open_len, h.steps = (t.data_ptr() for t in (self.last, self.open, self.open_len, self.steps))
        h.rew, h.cost, h.rows, h.n_rows = self.rew.data_ptr(), self.cost.data_ptr(), self.rows.data_ptr(), self.n_rows.data_ptr()
        h.row_cap = self.row_cap
        return h

    def begin(self, r, stream: int) -> None:
        from .. import _lib
        h = self._desc(1)
        _lib.check(_lib.lib.fsrl_traj_begin(ctypes.byref(r), ctypes.byref(h), stream))

    def scan(self, r, n_ready: int, window: int, stream: int) -> np.ndarray:
        """Episodes finished since the last scan, in (finish step, env) order.  ``n_ready`` > 0 on the
        one-episode-per-env path (each of the first n_ready envs finishes at most one episode); otherwise at
        most one episode per env and step of the ``window`` steps run since the last scan."""
        from .. import _lib
        cap = n_ready if n_ready > 0 else self.E * window
        h = self._desc(cap)
        _lib.check(_lib.lib.fsrl_traj_scan(ctypes.byref(r), ctypes.byref(h), int(n_ready), stream))
        n = int(self.n_rows.item())
        if n > cap:
            raise RuntimeError(f"trajectory scan: {n} finished episodes, room for {cap}")
        rows = self.rows[:n * ROW_DTYPE.itemsize].cpu().numpy().view(ROW_DTYPE)
        return rows[np.lexsort((rows["env"], rows["finish"]))]
