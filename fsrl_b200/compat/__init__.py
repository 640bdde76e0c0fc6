"""Import-compatibility shims so that scripts written against the reference stack
(``fsrl``, ``tianshou``, ``gymnasium``, ``bullet_safety_gym``, ``safety_gymnasium``,
``pyrallis`` -- SURVEY.md 2.3, F10) run on the device engine unchanged:

    import fsrl_b200.compat; fsrl_b200.compat.install()      # before the script's own imports

Only the symbols the reference's ``examples/`` and ``fsrl`` package actually use are provided,
and a shim is installed only when the real package is not importable.
"""
from __future__ import annotations

import argparse
import dataclasses
import importlib
import importlib.util
import sys
import types
from typing import Any, Callable, List


def _mod(name: str, **attrs) -> types.ModuleType:
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__path__ = []          # behave like a package so that `import a.b.c` resolves sub-entries
    sys.modules[name] = m
    return m


def _missing(name: str) -> bool:
    if name in sys.modules:
        return False
    try:
        return importlib.util.find_spec(name) is None
    except (ImportError, ValueError):
        return True


# ---- vector-env factories with tianshou's constructor (a list of env constructors) ------------------
def _vector_env_class(cls_name: str):
    """Registered tasks (DeviceEnv prototypes) become a DeviceVectorEnv; any other env constructor a
    HostVectorEnv stepping those envs in this process."""
    from ..envs import DeviceEnv, DeviceVectorEnv, HostVectorEnv

    class _Vec(DeviceVectorEnv):
        def __new__(cls, env_fns: List[Callable[[], Any]], **kwargs):
            proto = env_fns[0]()
            if isinstance(proto, DeviceEnv):
                self = super().__new__(cls)
                self._proto = proto         # the constructor runs once: __init__ reads the task from it
                return self
            return HostVectorEnv._from_envs([proto] + [fn() for fn in env_fns[1:]],
                                            device=kwargs.get("device", "cuda"), seed=kwargs.get("seed", 0))

        def __init__(self, env_fns: List[Callable[[], Any]], **kwargs):
            super().__init__(self._proto.task, len(env_fns), device=kwargs.get("device", "cuda"),
                             seed=kwargs.get("seed", 0))

    _Vec.__name__ = _Vec.__qualname__ = cls_name
    return _Vec


# ---- pyrallis.wrap: dataclass <- `--field value` CLI flags / `--config file.yaml` --------------------
def _pyrallis_wrap(config_path=None):
    def deco(fn):
        import inspect
        import typing

        def runner(*a, **kw):
            if a or kw:
                return fn(*a, **kw)
            hints = typing.get_type_hints(fn)
            cfg_cls = next(iter(hints.values()))
            ap = argparse.ArgumentParser()
            ap.add_argument("--config", default=config_path)
            for f in dataclasses.fields(cfg_cls):
                ap.add_argument("--" + f.name, default=None)
            ns, _ = ap.parse_known_args()
            values = {}
            if ns.config:
                import yaml
                values.update(yaml.safe_load(open(ns.config)) or {})
            for f in dataclasses.fields(cfg_cls):
                raw = getattr(ns, f.name)
                if raw is not None:
                    import ast
                    try:
                        values[f.name] = ast.literal_eval(raw)
                    except (ValueError, SyntaxError):
                        values[f.name] = raw
            return fn(cfg_cls(**values))

        runner.__wrapped__ = fn
        return runner
    return deco


def install(force: bool = False) -> List[str]:
    """Register the shim modules; returns the names that were installed."""
    import numpy as np
    import torch

    from .. import agent as _agent
    from .. import config as _config
    from .. import data as _data
    from .. import envs as _envs
    from .. import nets as _nets
    from .. import policy as _policy
    from .. import spaces as _spaces
    from .. import trainer as _trainer
    from ..policy.ddpg_lag import GaussianNoise
    from ..utils import exp_util as _exp_util
    from ..utils import logger as _logger
    from ..utils import optim_util as _optim_util
    done = []

    def want(name):
        if force or _missing(name):
            done.append(name)
            return True
        return False

    if want("gymnasium"):
        sp = _mod("gymnasium.spaces", Box=_spaces.Box, Discrete=_spaces.Discrete,
                  MultiBinary=_spaces.MultiBinary, MultiDiscrete=_spaces.MultiDiscrete, Space=_spaces.Space)
        _mod("gymnasium", make=_envs.make, Env=_envs.DeviceEnv, Space=_spaces.Space, spaces=sp)
    for side_effect in ("bullet_safety_gym", "safety_gymnasium"):
        if want(side_effect):
            _mod(side_effect)            # imported only to register tasks; ours are built in
    if want("pyrallis"):
        _mod("pyrallis", wrap=_pyrallis_wrap)
    if want("tianshou"):
        vec = {n: _vector_env_class(n) for n in ("DummyVectorEnv", "ShmemVectorEnv", "SubprocVectorEnv")}
        t_env = _mod("tianshou.env", BaseVectorEnv=_envs.DeviceVectorEnv, VectorEnvNormObs=_envs.VectorEnvNormObs, **vec)
        t_data = _mod("tianshou.data", Batch=_data.Batch, ReplayBuffer=_data.ReplayBuffer,
                      ReplayBufferManager=_data.VectorReplayBuffer, VectorReplayBuffer=_data.VectorReplayBuffer,
                      to_numpy=_data.to_numpy, to_torch_as=_data.to_torch_as)

        RunningMeanStd = _optim_util.RunningMeanStd

        class MovAvg:
            def __init__(self, size=100):
                self.size, self.cache = size, []

            def add(self, x):
                self.cache = (self.cache + list(np.atleast_1d(x)))[-self.size:]
                return self.get()

            def get(self):
                return float(np.mean(self.cache)) if self.cache else 0.0

        class DummyTqdm:
            def __init__(self, total, **kw):
                self.total, self.n = total, 0

            def set_postfix(self, **kw):
                pass

            def update(self, n=1):
                self.n += n

            def __enter__(self):
                return self

            def __exit__(self, *a):
                pass

        t_utils = _mod("tianshou.utils", RunningMeanStd=RunningMeanStd, MovAvg=MovAvg, DummyTqdm=DummyTqdm,
                       MultipleLRSchedulers=object, tqdm_config={"dynamic_ncols": True, "ascii": True},
                       deprecation=lambda msg: None)
        n_common = _mod("tianshou.utils.net.common", Net=_nets.Net, MLP=_nets.MLP)
        n_cont = _mod("tianshou.utils.net.continuous", ActorProb=_nets.ActorProb, Critic=_nets.Critic, Actor=_nets.Actor)
        t_net = _mod("tianshou.utils.net", common=n_common, continuous=n_cont)
        t_utils.net = t_net
        t_expl = _mod("tianshou.exploration", BaseNoise=object, GaussianNoise=GaussianNoise)
        _mod("tianshou", env=t_env, data=t_data, utils=t_utils, exploration=t_expl)
    if want("fsrl"):
        f_net_common = _mod("fsrl.utils.net.common", ActorCritic=_policy.ActorCritic)
        f_net_cont = _mod("fsrl.utils.net.continuous", DoubleCritic=_nets.DoubleCritic, SingleCritic=_nets.SingleCritic)
        f_net = _mod("fsrl.utils.net", common=f_net_common, continuous=f_net_cont)
        f_logger = _mod("fsrl.utils.logger", BaseLogger=_logger.BaseLogger, DummyLogger=_logger.DummyLogger,
                        TensorboardLogger=_logger.TensorboardLogger, WandbLogger=_logger.WandbLogger)
        sys.modules["fsrl.utils.exp_util"] = _exp_util
        sys.modules["fsrl.utils.optim_util"] = _optim_util
        f_utils = _mod("fsrl.utils", BaseLogger=_logger.BaseLogger, DummyLogger=_logger.DummyLogger,
                       TensorboardLogger=_logger.TensorboardLogger, WandbLogger=_logger.WandbLogger,
                       exp_util=_exp_util, optim_util=_optim_util, net=f_net, logger=f_logger)
        cfgs = {}
        for key in ("ppol", "cpo", "sacl", "ddpgl", "trpol", "focops", "focosp", "cvpo"):
            m = getattr(_config, key + "_cfg")
            sys.modules[f"fsrl.config.{key}_cfg"] = m
            cfgs[key + "_cfg"] = m
        f_config = _mod("fsrl.config", **cfgs)
        sys.modules["fsrl.agent"] = _agent
        sys.modules["fsrl.policy"] = _policy
        sys.modules["fsrl.data"] = _data
        sys.modules["fsrl.trainer"] = _trainer
        _mod("fsrl", agent=_agent, policy=_policy, data=_data, trainer=_trainer, utils=f_utils, config=f_config)
    return done
