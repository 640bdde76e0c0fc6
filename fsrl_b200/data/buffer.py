"""Device replay storage with the layout contract of tianshou's ``VectorReplayBuffer`` as the
reference uses it (fsrl/agent/base_agent.py:279; SURVEY.md 2.3 / Appendix A.25):

* ``buffer_num`` sub-buffers of ``ceil(total_size / buffer_num)`` slots, one per env;
* flat index ``p = env * cap + slot``  -> ``sample(0)`` yields every valid transition,
  sub-buffer by sub-buffer in chronological order (the order GAE scans);
* ``unfinished_index()`` = last stored slot of every sub-buffer whose episode is running;
* ``next(idx)`` stays put at a done transition or at the newest slot.

Everything is SoA in HBM; nothing is copied to the host on the training path.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import numpy as np
import torch

from .batch import Batch


class DeviceVectorReplayBuffer:
    def __init__(self, total_size: int, buffer_num: int, device="cuda", **_):
        assert buffer_num > 0
        self.buffer_num = int(buffer_num)
        self.cap = int(math.ceil(total_size / buffer_num))
        self.maxsize = self.cap * self.buffer_num
        self.device = torch.device(device)
        self._allocated = False
        self.D = self.A = 0

    # tianshou allocates on the first add(); we allocate when the collector tells us the dims
    def allocate(self, D: int, A: int, device=None):
        if self._allocated:
            assert (D, A) == (self.D, self.A)
            return
        if device is not None:
            self.device = torch.device(device)
        n, dev = self.maxsize, self.device
        self.D, self.A = D, A
        self.obs = torch.zeros((n, D), dtype=torch.float32, device=dev)
        self.obs_next = torch.zeros((n, D), dtype=torch.float32, device=dev)
        self.act = torch.zeros((n, A), dtype=torch.float32, device=dev)
        self.rew = torch.zeros(n, dtype=torch.float32, device=dev)
        self.cost = torch.zeros(n, dtype=torch.float32, device=dev)
        self.logp = torch.zeros(n, dtype=torch.float32, device=dev)
        self.terminated = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.truncated = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.ptr = torch.zeros(self.buffer_num, dtype=torch.int32, device=dev)
        self.len = torch.zeros(self.buffer_num, dtype=torch.int32, device=dev)
        self._allocated = True

    def fill(self, r) -> None:
        r.b_obs, r.b_obs_next, r.b_act = self.obs.data_ptr(), self.obs_next.data_ptr(), self.act.data_ptr()
        r.b_rew, r.b_cost, r.b_logp = self.rew.data_ptr(), self.cost.data_ptr(), self.logp.data_ptr()
        r.b_term, r.b_trunc = self.terminated.data_ptr(), self.truncated.data_ptr()
        r.b_ptr, r.b_len, r.cap = self.ptr.data_ptr(), self.len.data_ptr(), self.cap

    def reset(self, keep_statistics: bool = False) -> None:
        if self._allocated:
            self.ptr.zero_()
            self.len.zero_()

    def __len__(self) -> int:
        return int(self.len.sum().item()) if self._allocated else 0

    @property
    def done(self) -> torch.Tensor:
        return (self.terminated | self.truncated)

    # ---- index helpers (device tensors, int64) --------------------------------------------------
    def sample_indices(self, batch_size: int) -> torch.Tensor:
        lens = self.len.to(torch.int64)
        if batch_size == 0:
            cap = self.cap
            slot = torch.arange(cap, device=self.device).unsqueeze(0)                 # (1, cap)
            start = torch.where(lens == cap, self.ptr.to(torch.int64), torch.zeros_like(lens))
            order = (start.unsqueeze(1) + slot) % cap                                    # chronological
            flat = order + (torch.arange(self.buffer_num, device=self.device) * cap).unsqueeze(1)
            mask = slot < lens.unsqueeze(1)
            return flat[mask]
        # uniform over all valid transitions (tianshou ReplayBufferManager.sample_indices draws
        # with numpy's global RNG: same here, so host-seeded runs are reproducible)
        lens_h = lens.cpu().numpy()
        total = int(lens_h.sum())
        if total == 0:
            return torch.zeros(0, dtype=torch.int64, device=self.device)
        offsets = np.concatenate([[0], np.cumsum(lens_h)])
        draw = np.random.randint(0, total, size=batch_size)
        env = np.searchsorted(offsets, draw, side="right") - 1
        k = draw - offsets[env]
        ptr_h = self.ptr.cpu().numpy().astype(np.int64)
        start = np.where(lens_h == self.cap, ptr_h, 0)
        slot = (start[env] + k) % self.cap
        return torch.as_tensor(env * self.cap + slot, dtype=torch.int64, device=self.device)

    def last_index(self) -> torch.Tensor:
        """newest stored slot of each non-empty sub-buffer"""
        e = torch.arange(self.buffer_num, device=self.device)
        last = (self.ptr.to(torch.int64) - 1) % self.cap + e * self.cap
        return last[self.len > 0]

    def unfinished_index(self) -> torch.Tensor:
        last = self.last_index()
        return last[self.done[last] == 0]

    def next(self, index: torch.Tensor) -> torch.Tensor:
        index = index.to(torch.int64)
        env = index // self.cap
        nxt = (index % self.cap + 1) % self.cap + env * self.cap
        newest = (self.ptr.to(torch.int64)[env] - 1) % self.cap + env * self.cap
        stay = (self.done[index] != 0) | (index == newest)
        return torch.where(stay, index, nxt)

    def sample(self, batch_size: int) -> Tuple[Batch, torch.Tensor]:
        idx = self.sample_indices(batch_size)
        return self[idx], idx

    def __getitem__(self, idx) -> Batch:
        return Batch(obs=self.obs[idx], act=self.act[idx], rew=self.rew[idx],
                     terminated=self.terminated[idx].bool(), truncated=self.truncated[idx].bool(),
                     done=self.done[idx].bool(), obs_next=self.obs_next[idx],
                     info=Batch(cost=self.cost[idx]), policy=Batch(logp=self.logp[idx]))


# the names the reference imports
VectorReplayBuffer = DeviceVectorReplayBuffer


def ReplayBuffer(size: int, buffer_num: int = 1, **kwargs) -> DeviceVectorReplayBuffer:
    """tianshou's ``ReplayBuffer(size)``: one sub-buffer of ``size`` slots (``BasicCollector``'s buffer,
    basic_collector.py:56; collect_dataset.py:335).  ``ReplayBuffer(size, n)`` keeps meaning n sub-buffers."""
    return DeviceVectorReplayBuffer(size, buffer_num, **kwargs)
