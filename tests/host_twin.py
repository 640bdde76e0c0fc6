"""The CPU env twins (oracle/) as host envs, for the host-env tests and tools/host_env_collect_time.py.

``TwinEnv`` is env i of a shared twin as a gymnasium env; ``TwinVectorEnv`` puts a whole twin (or any oracle env
with ``reset(ids)`` / ``step(act, ids)`` returning ``(obs, rew, cost, terminated, truncated)``, such as
oracle.trainer_scenario.TerminatingEnv) behind tianshou's vector protocol."""
import numpy as np

from oracle.envs_velocity import OracleVecEnvVel


def _spaces(D, A):
    from fsrl_b200.spaces import Box
    return Box(-np.inf, np.inf, (D,), np.float32), Box(-1.0, 1.0, (A,), np.float32)


class TwinEnv:
    """Env i of a shared CPU twin as a gymnasium env (5-tuple step, (obs, info) reset, cost in info)."""

    def __init__(self, twin, i, task):
        from fsrl_b200.envs import _Spec
        self.twin, self.i = twin, i
        self.observation_space, self.action_space = _spaces(twin.D, twin.A)
        self.spec = _Spec(task, twin.T)

    def reset(self, seed=None, options=None):
        return self.twin.reset([self.i])[0], {}

    def step(self, a):
        o, rew, cost, term, trunc = self.twin.step(np.asarray(a, np.float32)[None], [self.i])
        return o[0], rew[0], bool(term[0]), bool(trunc[0]), {"cost": float(cost[0])}


class TwinVectorEnv:
    """An oracle vector env behind tianshou's vector protocol (len, step(action, id), reset(id)); info is a dict of
    arrays."""

    def __init__(self, inner, task=None, T=None):
        from fsrl_b200.envs import _Spec
        self.inner, self.E = inner, inner.E
        self.observation_space, self.action_space = _spaces(inner.D, inner.A)
        self.spec = _Spec(task, T if T is not None else getattr(inner, "T", None))

    def __len__(self):
        return self.E

    def reset(self, id=None, **kw):
        return self.inner.reset(None if id is None else np.asarray(id)), {}

    def step(self, action, id=None):
        ids = np.arange(self.E) if id is None else np.asarray(id)
        o, rew, cost, term, trunc = self.inner.step(np.asarray(action, np.float32), ids)
        return o, rew, term, trunc, {"cost": cost}


def twin(task, E, seed):
    from fsrl_b200.envs import KINDS
    return OracleVecEnvVel(KINDS[task], E, seed)


def twin_fns(task, E, seed):
    tw = twin(task, E, seed)
    return [lambda i=i: TwinEnv(tw, i, task) for i in range(E)]


def host_twin(task, E, seed, per_env=False):
    """A HostVectorEnv over the twin of `task`: E gymnasium envs (per_env) or the vectorised twin."""
    from fsrl_b200.envs import HostVectorEnv
    if per_env:
        return HostVectorEnv(twin_fns(task, E, seed))
    return HostVectorEnv.from_vector_env(TwinVectorEnv(twin(task, E, seed), task))
