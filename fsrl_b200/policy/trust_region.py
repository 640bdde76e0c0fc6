"""Device machinery shared by the trust-region learners (CPO, TRPO-Lagrangian): resident-batch
engine context, head-gradient / Hessian-vector-product calls (csrc/cpo.cu), conjugate gradients
(reference: fsrl/policy/cpo.py:184-204, trpo_lag.py:261-283) and the critic regression step."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Tuple

import numpy as np
import torch

from .. import _lib
from ..engine import EngineCtx
from .base_policy import DeviceBatch


class TrustRegionMixin:
    _eng: Optional[EngineCtx] = None
    _critic_t = 0
    _l2_reg = 0.0
    _damping_coeff = 0.1

    # ---- engine ----------------------------------------------------------------------------------------
    def _ensure_engine(self, n: int) -> EngineCtx:
        if self._eng is None or self._eng.bmax < n:
            self._eng = EngineCtx(self.arena, n, extra_slots=1, grown_from=self._eng)
            P = self.arena.slots[0].size
            dev = self.device
            self._vec = {k: torch.zeros(P, dtype=torch.float32, device=dev)
                         for k in ("g", "b", "x", "r", "p", "z", "Hinv_g", "Hinv_b", "hv", "theta0", "step")}
            self._v_w2n = torch.zeros(self.arena.slots[0].H ** 2, dtype=torch.float32, device=dev)
            self._sums = torch.zeros(4, dtype=torch.float64, device=dev)
            self._dot = torch.zeros(1, dtype=torch.float64, device=dev)
        return self._eng

    # ---- data parallel (SURVEY.md 8e): the global minibatch is the union of the ranks' minibatches ----
    # Every batch quantity of the trust-region step is a mean over the minibatch, so rank r's local
    # means are combined with the weights n_r / sum(n): sums are all-reduced as sums, gradient /
    # Hessian-vector products as weighted vectors (g, b and each Hv: P floats, ~22 x per update).
    # All ranks then run the SAME conjugate-gradient iterates, dual case analysis and line search.
    _dpw: Optional[float] = None

    def _dp_begin(self, n: int) -> int:
        """Start a minibatch step of n local rows; returns the global row count."""
        dp = getattr(self, "_dp", None)
        if dp is None or dp.world == 1:
            self._dpw = None
            return n
        n_g = int(round(float(dp.all_sum([n])[0])))
        self._dpw = n / n_g
        return n_g

    def _gsums(self) -> np.ndarray:
        sm = self._sums.cpu().numpy()
        return sm if self._dpw is None else self._dp.all_sum(sm)

    def _gscalar(self, x: float) -> float:
        return float(x) if self._dpw is None else float(self._dp.all_sum([x])[0])

    def _gvec(self, t: torch.Tensor) -> None:
        if self._dpw is not None:
            t.mul_(self._dpw)
            self._dp.dist.all_reduce(t)

    def _standardize(self, x: torch.Tensor, n: int) -> None:
        """x <- (x - mean) / std (unbiased) over the whole collect (cpo.py:127-131); under data
        parallelism the moments are those of the union of all ranks' collects."""
        dp = getattr(self, "_dp", None)
        if dp is None or dp.world == 1:
            _lib.check(_lib.lib.fsrl_standardize(x.data_ptr(), n, self._stream()))
            return
        xd = x[:n].double()
        s1, s2, cnt = dp.all_sum([float(xd.sum().item()), float((xd * xd).sum().item()), float(n)])
        mean = s1 / cnt
        var = max((s2 - cnt * mean * mean) / max(cnt - 1.0, 1.0), 0.0)
        x[:n].sub_(mean).div_(float(np.sqrt(var)))

    def _dp_same_count(self, c: int, what: str) -> None:
        dp = getattr(self, "_dp", None)
        if dp is not None and dp.world > 1:
            lo_hi = dp.all_max([c, -c])
            if int(lo_hi[0]) != -int(lo_hi[1]):
                raise RuntimeError(f"data-parallel {what}: ranks disagree ({int(-lo_hi[1])}..{int(lo_hi[0])}); "
                                   "use batch_size >= the per-rank collect size")

    # ---- minibatches and the state-independent Gaussian ------------------------------------------------------
    def _minibatches(self, n_all: int, batch_size: int) -> List[Tuple[torch.Tensor, int]]:
        """tianshou's ``Batch.split(batch_size, shuffle=True, merge_last=True)`` over n_all rows: one
        ``np.random.permutation`` drawn from NumPy's global stream, cut into chunks of batch_size rows, the last
        full chunk absorbing a short tail.  Each chunk as (device int32 row indices, row count)."""
        perm_all = np.random.permutation(n_all)
        merge_last = n_all % batch_size > 0
        chunks = []
        for i in range(0, n_all, batch_size):
            if merge_last and i + 2 * batch_size >= n_all:
                chunks.append(perm_all[i:]); break
            chunks.append(perm_all[i:i + batch_size])
        return [(torch.as_tensor(ch.astype(np.int32), device=self.device), len(ch)) for ch in chunks]

    def _old_dist(self, obs: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(mean, std) of the actor's Gaussian at the current parameters: the mean from one actor pass, squashed
        to max_action * tanh unless unbounded; the state-independent std broadcast over the rows."""
        z = self.net_forward(0, obs)
        mu = self.actor._max * torch.tanh(z) if not self.actor._unbounded else z
        return mu, self.actor.sigma_param.detach().view(1, -1).exp().expand_as(mu)

    def _entropy(self) -> float:
        """Entropy of the state-independent Gaussian: sum over actions of 1/2 + log(2 pi)/2 + log sigma."""
        return float((0.5 + 0.5 * np.log(2 * np.pi) + self.actor.sigma_param.detach().flatten()).sum().item())

    # ---- device helpers -----------------------------------------------------------------------------------
    def _dotp(self, a, b) -> float:
        _lib.check(_lib.lib.fsrl_vec_dot(a.data_ptr(), b.data_ptr(), a.numel(), self._dot.data_ptr(), self._stream()))
        return float(self._dot.item())

    def _descriptor(self, batch: DeviceBatch, perm: Optional[torch.Tensor], n: int) -> "_lib.Cpo":
        eng = self._eng
        a = self.arena.slots[0]
        d = _lib.Cpo()
        d.eng = eng.engine()
        d.actor = eng.netlist([a])
        r = eng.netlist([a])
        r.nets[0].slot = eng.extra_slot(0)
        d.actor_r = r
        d.N, d.ld, d.A = n, batch.adv.shape[1], a.out
        d.bounded, d.max_action = int(not self.actor._unbounded), float(self.actor._max)
        d.obs, d.act, d.logp_old = batch.obs.data_ptr(), batch.act.data_ptr(), batch.logp_old.data_ptr()
        d.mean_old, d.std_old, d.adv = batch.mean_old.data_ptr(), batch.std_old.data_ptr(), batch.adv.data_ptr()
        d.perm = None if perm is None else perm.data_ptr()
        d.out = eng.slot_view(a, "out").data_ptr()
        d.dout = eng.slot_view(a, "dout").data_ptr()
        d.log_sigma = self.arena.extra_ptr(a)
        return d

    def _head(self, d, mode: int):
        _lib.check(_lib.lib.fsrl_cpo_head(ctypes.byref(d), mode, self._sums.data_ptr(), self._stream()))

    def _hvp(self, d, v, out):
        _lib.check(_lib.lib.fsrl_cpo_hvp(ctypes.byref(d), v.data_ptr(), self._v_w2n.data_ptr(), out.data_ptr(),
                                         float(self._damping_coeff), self._stream()))
        self._gvec(out)      # H = sum_r w_r H_r (the damping term carries through: sum_r w_r = 1)

    def _cg(self, d, rhs: torch.Tensor, out: torch.Tensor, nsteps: int = 10, residual_tol: float = 1e-8):
        """cpo.py:184-204.  Single GPU: the whole solve is enqueued by ``fsrl_cg_solve`` -- vectors AND scalars stay on
        the device, no host round trip per iteration.  Data parallel: every Hessian-vector product is all-reduced
        (``_hvp`` -> ``_gvec``), so the loop is driven from the host with two scalar reads per iteration."""
        v = self._vec
        if self._dpw is None:
            n = rhs.numel()
            if getattr(self, "_cg_work", None) is None or self._cg_work.numel() < 4 * n:
                self._cg_work = torch.empty(4 * n, dtype=torch.float32, device=rhs.device)
                self._cg_state = torch.zeros(8, dtype=torch.float64, device=rhs.device)
            _lib.check(_lib.lib.fsrl_cg_solve(ctypes.byref(d), rhs.data_ptr(), out.data_ptr(), self._cg_work.data_ptr(),
                                              self._v_w2n.data_ptr(), self._cg_state.data_ptr(), n, int(nsteps),
                                              float(residual_tol), float(self._damping_coeff), self._stream()))
            return
        x, r, p, z = v["x"], v["r"], v["p"], v["z"]
        x.zero_(); r.copy_(rhs); p.copy_(rhs)
        rs_old = self._dotp(r, r)
        lib, s, n = _lib.lib, self._stream(), rhs.numel()
        for _ in range(nsteps):
            self._hvp(d, p, z)
            alpha = rs_old / self._dotp(p, z)
            _lib.check(lib.fsrl_vec_axpby(alpha, p.data_ptr(), 1.0, x.data_ptr(), n, s))
            _lib.check(lib.fsrl_vec_axpby(-alpha, z.data_ptr(), 1.0, r.data_ptr(), n, s))
            rs_new = self._dotp(r, r)
            if rs_new < residual_tol:
                break
            _lib.check(lib.fsrl_vec_axpby(1.0, r.data_ptr(), rs_new / rs_old, p.data_ptr(), n, s))
            rs_old = rs_new
        out.copy_(x)

    # ---- critic regression (:147-162) ------------------------------------------------------------------------
    def critics_loss(self, batch: DeviceBatch, perm: Optional[torch.Tensor], n: int) -> dict:
        eng = self._eng
        crit = self.arena.slots[1:1 + self.critics_num]
        inp = eng.make_input(batch.obs, perm)
        n_g = self._dp_begin(n)
        eng.forward(crit, inp, n, save=True)
        stats = {}
        for i, s in enumerate(crit):
            self._sums.zero_()
            _lib.check(_lib.lib.fsrl_mse_head(eng.slot_view(s, "out").data_ptr(), batch.ret[i].data_ptr(),
                                              None if perm is None else perm.data_ptr(), n,
                                              eng.slot_view(s, "dout").data_ptr(), self._sums.data_ptr(), self._stream()))
            th = self.arena.theta[s.offset:s.offset + s.size]
            reg = (self._dotp(th, th) * self._l2_reg) if self._l2_reg else 0.0
            stats["loss/vf" + str(i)] = self._gscalar(float(self._sums[0].item())) / n_g + reg
        eng.backward(crit, n)
        eng.wgrad(crit, inp, n)
        if self._dpw is not None:
            for s in crit:
                self._gvec(self.arena.grad[s.offset:s.offset + s.size])
        self._critic_t += 1
        g = self.optim.param_groups[0]
        eng.adam(crit, g["lr"], self._critic_t, betas=g["betas"], eps=g["eps"], l2_reg=self._l2_reg)
        stats["loss/vf_total"] = sum(stats["loss/vf" + str(i)] for i in range(self.critics_num))
        return stats

