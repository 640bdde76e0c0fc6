"""PPO with PID Lagrangian (reference: /root/reference/fsrl/policy/ppo_lag.py).

``process_fn`` = dual GAE on the device (+ the behaviour log-prob, which the rollout kernel
already stored: the reference recomputes it with unchanged weights at :142-149);
``learn`` = for each repeat, draw the minibatch permutation with NumPy's global RNG exactly
like tianshou's ``Batch.split`` (SURVEY.md 2.3), upload it, and run every minibatch of the
repeat as three kernel launches (csrc/ppo.cu) without host synchronisation; the KL early
stop (:251-255) is evaluated once per repeat from the device-side statistics.
"""
from __future__ import annotations

import ctypes
from typing import Any, Dict, List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _lib
from ..nets import ActorProb
from ..optim import FusedAdam
from ..utils.logger import BaseLogger, DummyLogger
from .base_policy import DeviceBatch
from .lagrangian_base import LagrangianPolicy


class PPOLagrangian(LagrangianPolicy):
    def __init__(self, actor, critics, optim, dist_fn=None, logger: BaseLogger = DummyLogger(),
                 target_kl: float = 0.02, vf_coef: float = 0.25,
                 max_grad_norm: Optional[float] = None, gae_lambda: float = 0.95,
                 eps_clip: float = 0.2, dual_clip: Optional[float] = None,
                 value_clip: bool = False, advantage_normalization: bool = True,
                 recompute_advantage: bool = False, use_lagrangian: bool = True,
                 lagrangian_pid: Tuple = (0.05, 0.0005, 0.1),
                 cost_limit: Union[List, float] = np.inf, rescaling: bool = True,
                 gamma: float = 0.99, max_batchsize: int = 99999,
                 reward_normalization: bool = False, deterministic_eval: bool = True,
                 action_scaling: bool = True, action_bound_method: str = "clip",
                 observation_space=None, action_space=None, lr_scheduler=None) -> None:
        super().__init__(actor, critics, dist_fn, logger, use_lagrangian, lagrangian_pid,
                         cost_limit, rescaling, gamma, max_batchsize, reward_normalization,
                         deterministic_eval, action_scaling, action_bound_method,
                         observation_space, action_space, lr_scheduler)
        if not isinstance(optim, FusedAdam):
            # accept a torch.optim.Adam built by reference-style agent code: keep its
            # hyper-parameters, run the update with the fused kernel
            g = optim.param_groups[0]
            optim = FusedAdam(lr=g["lr"], betas=g.get("betas", (0.9, 0.999)), eps=g.get("eps", 1e-8))
        self.optim = optim
        self._lambda = gae_lambda
        self._weight_vf = vf_coef
        self._grad_norm = max_grad_norm
        self._target_kl = target_kl
        self._eps_clip = eps_clip
        assert dual_clip is None or dual_clip > 1.0, \
            "Dual-clip PPO parameter should greater than 1.0."
        self._dual_clip = dual_clip
        self._value_clip = value_clip
        if not self._rew_norm:
            assert not self._value_clip, \
                "value clip is available only when `reward_normalization` is True"
        self._norm_adv = advantage_normalization
        self._recompute_adv = recompute_advantage
        if not isinstance(actor, ActorProb) or actor._c_sigma:
            raise TypeError("PPOLagrangian needs a state-independent-sigma ActorProb")
        assert self.critics_num in (1, 2), "reward critic + at most one cost critic"
        self._scratch = None
        self._bmax = 0
        self._stats_dev = None
        self.last_stats: Dict[str, np.ndarray] = {}

    # -----------------------------------------------------------------------------------------------
    def _ensure_update_state(self, batch_size: int, n_total: int, repeat: int):
        ar = self.arena
        if self.optim.m is None:
            self.optim.attach(ar)
        H = ar.slots[0].H
        n_nets = len(ar.slots)
        bmax = min(max(2 * batch_size, 16), max(n_total, 16))
        bmax = (bmax + 63) // 64 * 64
        if self._scratch is None or bmax > self._bmax:
            self._bmax = bmax
            nfl = _lib.lib.fsrl_ppo_scratch_floats(n_nets, H, bmax)
            self._scratch = torch.zeros(nfl, dtype=torch.float32, device=ar.device)
        if getattr(self, "_w2n", None) is None:
            self._w2n = torch.zeros(n_nets * H * H, dtype=torch.float32, device=ar.device)
            self._norm_sq = torch.zeros(8, dtype=torch.float32, device=ar.device)
            self._mirror_dirty = True
        n_mb = (n_total + batch_size - 1) // batch_size
        need = repeat * n_mb * _lib.PPO_STATS
        if self._stats_dev is None or self._stats_dev.numel() < need:
            self._stats_dev = torch.zeros(need, dtype=torch.float32, device=ar.device)

    def _descriptor(self, batch: DeviceBatch, perm_dev: torch.Tensor) -> "_lib.PpoUpdate":
        ar = self.arena
        u = _lib.PpoUpdate()
        s0 = ar.slots[0]
        u.theta, u.grad = ar.theta.data_ptr(), ar.grad.data_ptr()
        u.adam_m, u.adam_v = self.optim.m.data_ptr(), self.optim.v.data_ptr()
        u.w2n, u.scratch = self._w2n.data_ptr(), self._scratch.data_ptr()
        u.norm_sq, u.stats = self._norm_sq.data_ptr(), self._stats_dev.data_ptr()
        for i, s in enumerate(ar.slots):
            u.net_off[i] = s.offset
        u.n_params = ar.n_params
        u.n_nets, u.D, u.H, u.A, u.C = len(ar.slots), s0.D, s0.H, s0.out, self.critics_num
        u.actor_out, u.bmax = s0.out, self._bmax
        u.obs, u.act, u.logp_old = batch.obs.data_ptr(), batch.act.data_ptr(), batch.logp_old.data_ptr()
        u.adv, u.ret, u.values = batch.adv.data_ptr(), batch.ret.data_ptr(), batch.v.data_ptr()
        u.ld = batch.adv.shape[1]
        u.perm = perm_dev.data_ptr()
        u.eps_clip = self._eps_clip
        u.dual_clip = float(self._dual_clip) if self._dual_clip else 0.0
        u.vf_coef = self._weight_vf
        u.max_grad_norm = float(self._grad_norm) if self._grad_norm else 0.0
        u.max_action = float(self.actor._max)
        lags = self.lagrangians()
        u.lagrangian = lags[0] if (self.use_lagrangian and lags) else 0.0
        u.rescaling = self.rescaling_factor() if self.use_lagrangian else (1.0 if not self.rescaling else 1.0)
        u.bounded = int(not self.actor._unbounded)
        u.norm_adv = int(self._norm_adv)
        u.value_clip = int(self._value_clip)
        u.use_lagrangian = int(self.use_lagrangian and self.critics_num > 1)
        g = self.optim.param_groups[0]
        u.lr, u.beta1, u.beta2, u.adam_eps = g["lr"], g["betas"][0], g["betas"][1], g["eps"]
        need = batch.n * (s0.D + s0.out + 1 + 3 * self.critics_num)
        if getattr(self, "_gather", None) is None or self._gather.numel() < need:
            self._gather = torch.empty(need, dtype=torch.float32, device=ar.device)
        u.gather = self._gather.data_ptr()
        n_mb_max = batch.n // max(int(getattr(self, '_dp_batch', 1)), 1) + 2
        if getattr(self, "_mb_stats", None) is None or self._mb_stats.numel() < 4 * n_mb_max:
            self._mb_stats = torch.zeros(4 * n_mb_max, dtype=torch.float32, device=ar.device)
        u.mb_stats = self._mb_stats.data_ptr()
        u.batch_size = int(getattr(self, '_dp_batch', 0))
        u.barrier = self._norm_sq.data_ptr() + 8
        # persistent wgmma path (csrc/ppo_persist.cu): operand images, partial buffers and flags
        nws = int(_lib.lib.fsrl_ppo_persist_ws_floats(len(ar.slots), s0.D, s0.H))
        if getattr(self, "_persist_ws", None) is None or self._persist_ws.numel() < nws:
            self._persist_ws = torch.zeros(nws, dtype=torch.float32, device=ar.device)
        u.persist_ws, u.persist_ws_floats = self._persist_ws.data_ptr(), self._persist_ws.numel()
        u.persist_off = int(bool(getattr(self, "_persist_off", False)))
        dp = getattr(self, "_dp", None)
        u.world = 1
        if dp is not None and dp.world > 1:
            n_mb = (batch.n + self._dp_batch - 1) // self._dp_batch
            if getattr(self, "_moments", None) is None or self._moments.numel() < 4 * n_mb:
                self._moments = torch.zeros(4 * n_mb, dtype=torch.float64, device=ar.device)
            u.comm, u.world, u.batch_size = dp.comm, dp.world, self._dp_batch
            u.moments_w = u.moments = self._moments.data_ptr()
            dp.fill_p2p(u)
        return u

    # -----------------------------------------------------------------------------------------------
    def process_fn(self, batch, buffer, indices) -> DeviceBatch:
        if self._recompute_adv:
            self._buffer, self._indices = buffer, indices
        batch = self.compute_gae_returns(batch, buffer, indices, self._lambda)     # :141
        # logp_old (:142-149): stored by the rollout kernel under the same weights
        return batch

    def learn(self, batch: DeviceBatch, batch_size: int, repeat: int, **kwargs: Any) -> Dict[str, List[float]]:
        n = batch.n
        ar = self.arena
        self._dp_batch = int(batch_size)
        dp = getattr(self, "_dp", None)
        if dp is not None and dp.world > 1:
            # every rank must run the same number of equally sized minibatches, or the per-step gradient
            # exchanges fall out of step (a hang, or the 20 s peer timeout): fail loudly instead
            lo_hi = dp.all_max([n, -n])
            if int(lo_hi[0]) != -int(lo_hi[1]):
                raise RuntimeError("data-parallel PPO update: ranks hold different batch sizes (%d..%d rows); "
                                   "collect the same number of steps on every rank" % (-int(lo_hi[1]), int(lo_hi[0])))
        self._ensure_update_state(batch_size, n, repeat)
        lib = _lib.lib
        stream = self._stream()
        slot = 0
        self._stats_dev.zero_()
        rows = []
        # staging buffers of the minibatch permutation: allocated once (pinning is a millisecond-scale system call)
        if getattr(self, "_perm_n", -1) != n:
            self._perm_dev = torch.empty(n, dtype=torch.int32, device=ar.device)
            self._perm_host = torch.empty(n, dtype=torch.int32).pin_memory()
            self._perm_n = n
        perm_dev, perm_host = self._perm_dev, self._perm_host
        next_perm = None
        with torch.cuda.device(ar.device):
            if self._mirror_dirty:
                u0 = self._descriptor(batch, perm_dev)
                _lib.check(lib.fsrl_ppo_sync_mirror(ctypes.byref(u0), stream))
                self._mirror_dirty = False
            for step in range(repeat):
                if self._recompute_adv and step > 0:
                    batch = self.compute_gae_returns(batch, self._buffer, self._indices, self._lambda)
                # Batch.split(batch_size, shuffle=True): np.random.permutation (global RNG)
                if next_perm is not None:
                    perm_host.numpy()[:] = next_perm
                    next_perm = None
                else:
                    perm_host.numpy()[:] = self._first_permutation(n)
                perm_dev.copy_(perm_host, non_blocking=True)
                u = self._descriptor(batch, perm_dev)
                n_mb = ctypes.c_int(0)
                _lib.check(lib.fsrl_ppo_lag_epoch(ctypes.byref(u), n, int(batch_size), slot,
                                                  self.optim.step_count, ctypes.byref(n_mb), stream))
                self.optim.step_count += n_mb.value
                self.gradient_steps += n_mb.value
                # while the GPU chews through this repeat, draw the next permutation on the host; if
                # the KL test below stops the loop the draw is rolled back so that the NumPy stream
                # is consumed exactly as in the reference
                rng_state = None
                if step + 1 < repeat:
                    rng_state = np.random.get_state()
                    next_perm = np.random.permutation(n)
                else:
                    self._prefetch_permutation(n)
                st = self._stats_dev[slot * _lib.PPO_STATS:(slot + n_mb.value) * _lib.PPO_STATS] \
                    .view(n_mb.value, _lib.PPO_STATS).cpu().numpy()                    # sync point
                rows.append(st)
                slot += n_mb.value
                approx_kl = float(st[:, 2].sum()) / (n_mb.value + 1e-7)                # :251
                if getattr(self, "_dp", None) is not None:
                    approx_kl = self._dp.mean_scalar(approx_kl)                          # all ranks stop together
                if approx_kl > 1.5 * self._target_kl and rng_state is not None:
                    np.random.set_state(rng_state)
                if approx_kl > 1.5 * self._target_kl:
                    self.logger.print("Early stop at step %d due to reaching max kl." % step)
                    break
        if getattr(self, "_dp", None) is not None:
            self._dp.p2p_check()             # raises if a peer rank never joined a gradient exchange
        self._log_stats(np.concatenate(rows, axis=0), u)
        self.logger.store(gradient_steps=self.gradient_steps, tab="update")

    # ---- first permutation of the NEXT learn call, drawn while the last repeat's launch is still running -----------
    # The global NumPy stream must be consumed exactly as in the reference (one permutation per executed repeat, nothing
    # else), so the draw is speculative: the generator is put back to where it was, and the result is used only if the
    # next learn call finds the generator in that very state (nobody drew from it in between) -- then the generator is
    # advanced to where the draw had left it.
    @staticmethod
    def _same_rng_state(a, b) -> bool:
        return a[0] == b[0] and a[2:] == b[2:] and np.array_equal(a[1], b[1])

    def _prefetch_permutation(self, n: int) -> None:
        before = np.random.get_state()
        perm = np.random.permutation(n)
        self._spec_perm = (n, before, perm, np.random.get_state())
        np.random.set_state(before)

    def _first_permutation(self, n: int) -> np.ndarray:
        spec, self._spec_perm = getattr(self, "_spec_perm", None), None
        if spec is not None and spec[0] == n and self._same_rng_state(np.random.get_state(), spec[1]):
            np.random.set_state(spec[3])
            return spec[2]
        return np.random.permutation(n)

    # ---- the reference's per-piece loss hooks (ppo_lag.py:152-212) ------------------------------------------------
    # ``learn`` never calls these: the persistent launch / kernel chain evaluates both losses, their gradients and the
    # optimiser step fused.  They exist for code written against the reference that calls the pieces itself (custom
    # training loops, examples/customized): eager autograd on the device through the policy's nn.Modules, whose
    # parameters alias the kernels' arena -- so gradients taken from these losses update the same weights.
    def _piece(self, minibatch, name: str, i: int = None) -> torch.Tensor:
        x = getattr(minibatch, name)
        x = x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))
        x = x.to(self.device)
        return x if i is None else x[..., i]

    def critics_loss(self, minibatch):
        """Sum over critics of the (optionally clipped) squared return error; ``(loss, stats)`` like the reference."""
        total, stats = 0.0, {}
        obs = self._piece(minibatch, "obs").float()
        for i, critic in enumerate(self.critics):
            v = critic(obs).flatten()
            target = self._piece(minibatch, "rets", i)
            err = (target - v) ** 2
            if self._value_clip:
                v_old = self._piece(minibatch, "values", i)
                v_lim = v_old + torch.clamp(v - v_old, -self._eps_clip, self._eps_clip)
                err = torch.maximum(err, (target - v_lim) ** 2)
            loss_i = err.mean()
            total = total + loss_i
            stats["loss/vf" + str(i)] = loss_i.item()
        stats["loss/vf_total"] = total.item()
        return total, stats

    def policy_loss(self, batch, dist):
        """Clipped surrogate on the reward advantage + lambda-weighted cost-advantage terms, rescaled by
        1 / (sum(lambda) + 1); advantages are standardised per call, in place, like the reference does."""
        act, logp_old = self._piece(batch, "act"), self._piece(batch, "logp_old")
        logp = dist.log_prob(act)
        ratio = torch.exp(logp - logp_old).float()
        ratio = ratio.reshape(ratio.shape[0], -1).t()
        advs = self._piece(batch, "advs")
        if self._norm_adv:
            for i in range(self.critics_num):
                col = advs[..., i]
                advs[..., i] = (col - col.mean()) / col.std()
        a_r = advs[..., 0]
        unclipped, clipped = ratio * a_r, torch.clamp(ratio, 1.0 - self._eps_clip, 1.0 + self._eps_clip) * a_r
        lower = torch.minimum(unclipped, clipped)
        if self._dual_clip:
            lower = torch.where(a_r < 0, torch.maximum(lower, self._dual_clip * a_r), lower)
        loss_rew = -lower.mean()
        cost_terms = [ratio * advs[..., i] for i in range(1, self.critics_num)] if self.use_lagrangian else []
        loss_safety, stats = self.safety_loss(cost_terms)
        loss = stats["loss/rescaling"] * (loss_rew + loss_safety)
        stats.update({"loss/actor_rew": loss_rew.item(), "loss/actor_total": loss.item(),
                      "loss/kl": (logp_old - logp).mean().item()})
        return loss, stats

    def _log_stats(self, st: np.ndarray, u) -> None:
        """Rebuild the reference's per-minibatch ``loss/*`` keys (ppo_lag.py:169-170,205-211,247;
        lagrangian_base.py:158-165) from the device statistics: one D2H copy per repeat."""
        resc = float(u.rescaling)
        actor_rew, actor_saf, kl = st[:, 0], st[:, 1], st[:, 2]
        vf = st[:, 3:3 + self.critics_num]
        vf_total = vf.sum(axis=1)
        actor_total = resc * (actor_rew + actor_saf)
        total = actor_total + self._weight_vf * vf_total
        out = {"loss/rescaling": np.full(len(st), resc), "loss/actor_rew": actor_rew,
               "loss/actor_total": actor_total, "loss/kl": kl, "loss/vf_total": vf_total,
               "loss/total": total, "loss/entropy": st[:, 5], "loss/grad_norm": st[:, 6]}
        for i in range(self.critics_num):
            out["loss/vf" + str(i)] = vf[:, i]
        if self.use_lagrangian and self.critics_num > 1:
            out["loss/lagrangian"] = np.full(len(st), float(u.lagrangian))
            out["loss/actor_safety"] = actor_saf
        self.last_stats = out
        for k, v in out.items():
            tab, key = k.split("/", 1)
            self.logger.store_many(tab, key, v)
