"""Device-resident vector environments behind the vector-env protocol the reference's
collector consumes (``len(env)``, ``env.action_space``, ``reset``/``step`` --
fsrl/data/fast_collector.py:134,172,286; tianshou BaseVectorEnv).

The dynamics are the analytic models of csrc/envs.cuh (bullet_safety_gym / safety_gymnasium
are absent and irreproducible; SURVEY.md F5).  All state lives in HBM as SoA tensors; the
fused rollout kernel (csrc/rollout.cu) steps every env without host involvement.  ``step`` /
``reset(id)`` give the gym protocol on the same state, for loops that bring their own actions.
A user's own env struct runs on the same path once built into a plugin (:func:`build_device_env`) and
registered under a task name (:func:`register_device_env`; DESIGN §7).  Envs the device cannot run
(gymnasium simulators) go behind :class:`HostVectorEnv` (host_envs.py).
"""
from __future__ import annotations

import ctypes
import hashlib
import os
import re
import subprocess
import sys
import tempfile
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib
from .host_envs import HostVectorEnv, _Spec  # noqa: F401
from .spaces import Box

# task id -> (kind, D, A, S, T).  Registry names follow the reference's examples
# (examples/mlp/train_ppol_agent.py:28-40); BASELINE.json's "SafetyPointGoal1-v0" is an alias
# of the registry name SafetyPointGoal1Gymnasium-v0 (SURVEY.md App. A.20).
KINDS = {
    "SafetyCarCircle-v0": 0, "SafetyCarRun-v0": 1, "SafetyBallCircle-v0": 2, "SafetyBallRun-v0": 3,
    "SafetyAntCircle-v0": 4, "SafetyPointGoal1Gymnasium-v0": 5, "SafetyPointGoal1-v0": 5,
    "SafetyAntRun-v0": 6, "SafetyDroneCircle-v0": 7, "SafetyDroneRun-v0": 8,
    "SafetyPointCircle1Gymnasium-v0": 16, "SafetyPointCircle2Gymnasium-v0": 17,
    "SafetyCarCircle1Gymnasium-v0": 18, "SafetyCarCircle2Gymnasium-v0": 19,
    "SafetyPointGoal2Gymnasium-v0": 20, "SafetyCarGoal1Gymnasium-v0": 21, "SafetyCarGoal2Gymnasium-v0": 22,
    "SafetyPointButton1Gymnasium-v0": 24, "SafetyPointButton2Gymnasium-v0": 25,
    "SafetyCarButton1Gymnasium-v0": 26, "SafetyCarButton2Gymnasium-v0": 27,
    "SafetyPointPush1Gymnasium-v0": 28, "SafetyPointPush2Gymnasium-v0": 29,
    "SafetyCarPush1Gymnasium-v0": 30, "SafetyCarPush2Gymnasium-v0": 31,
    "SafetyHalfCheetahVelocityGymnasium-v1": 33, "SafetyHopperVelocityGymnasium-v1": 34,
    "SafetySwimmerVelocityGymnasium-v1": 35, "SafetyWalker2dVelocityGymnasium-v1": 36,
    "SafetyAntVelocityGymnasium-v1": 37,
}

PLUGIN_KIND_FIRST, PLUGIN_KIND_END = 64, 128   # FSRL_ENV_PLUGIN_FIRST / _END: the kinds of registered plugins


class _Plugin(NamedTuple):
    kind: int
    path: str
    so: ctypes.CDLL       # kept loaded: the library calls its launchers
    renders: bool         # its struct defines draw: render_mode="rgb_array" draws it (DESIGN §7)


PLUGINS = {}   # task -> _Plugin, filled by register_device_env

RENDER_MODES = (None, "rgb_array")
RENDER_MIN, RENDER_MAX = 16, 1024     # frame height and width (fsrl_env_render)


def task_kind(task: str) -> int:
    """The env kind of a built-in or registered task."""
    if task in KINDS:
        return KINDS[task]
    if task in PLUGINS:
        return PLUGINS[task].kind
    raise KeyError(f"unknown task {task!r}; available: {sorted(KINDS) + sorted(PLUGINS)}")


def env_dims(kind: int):
    D, A, S, T = (ctypes.c_int() for _ in range(4))
    _lib.check(_lib.lib.fsrl_env_dims(kind, ctypes.byref(D), ctypes.byref(A), ctypes.byref(S), ctypes.byref(T)))
    return D.value, A.value, S.value, T.value


class DeviceEnv:
    """What ``gym.make(task)`` returns: the spaces + horizon of one env (a descriptor: stepping
    happens only inside a :class:`DeviceVectorEnv`)."""

    def __init__(self, task: str):
        self.task = task
        self.kind = task_kind(task)
        D, A, S, T = env_dims(self.kind)
        self.observation_space = Box(-np.inf, np.inf, (D,), np.float32)
        self.action_space = Box(-1.0, 1.0, (A,), np.float32)
        self.spec = _Spec(task, T)
        self.state_dim = S

    def close(self):
        pass


def make(task: str, **_) -> DeviceEnv:
    return DeviceEnv(task)


class DeviceVectorEnv:
    """E independent envs of one task, resident on one GPU."""

    def __init__(self, task: str, env_num: int, device="cuda", seed: int = 0, render_mode: Optional[str] = None,
                 render_size=(256, 256)):
        if render_mode not in RENDER_MODES:
            raise ValueError(f"render_mode must be one of {RENDER_MODES}, got {render_mode!r}")
        height, width = (int(v) for v in render_size)
        if not (RENDER_MIN <= height <= RENDER_MAX and RENDER_MIN <= width <= RENDER_MAX):
            raise ValueError(f"render_size (height, width) = {(height, width)} outside [{RENDER_MIN}, {RENDER_MAX}]")
        self.render_mode, self.render_size = render_mode, (height, width)
        proto = DeviceEnv(task)
        if render_mode is not None and task in PLUGINS and not PLUGINS[task].renders:
            raise ValueError(f"{task!r} is a user-defined device env whose struct has no draw: it has no renderer, "
                             "so render_mode must be None")
        self.task, self.kind = task, proto.kind
        self.env_num = int(env_num)
        self.device = torch.device(device)
        self.observation_space = proto.observation_space
        self.action_space = proto.action_space
        self.max_episode_steps = proto.spec.max_episode_steps
        self.spec = proto.spec
        self.seed_value = int(seed) & 0xFFFFFFFF
        D, A, S, T = env_dims(self.kind)
        self.D, self.A, self.S = D, A, S
        E, dev = self.env_num, self.device
        self.env_state = torch.zeros((S, E), dtype=torch.float32, device=dev)
        self.obs_cur = torch.zeros((E, D), dtype=torch.float32, device=dev)
        self.env_t = torch.zeros(E, dtype=torch.int32, device=dev)
        self.ep_idx = torch.zeros(E, dtype=torch.int32, device=dev)
        self.act_ctr = torch.zeros(E, dtype=torch.int32, device=dev)
        self.active = torch.zeros(E, dtype=torch.uint8, device=dev)
        self.done_now = torch.zeros(E, dtype=torch.uint8, device=dev)
        self.ep_rew = torch.zeros(E, dtype=torch.float64, device=dev)
        self.ep_len = torch.zeros(E, dtype=torch.int32, device=dev)
        self.stats = torch.zeros(ctypes.sizeof(_lib.CollectStats), dtype=torch.uint8, device=dev)
        self._stats_host = torch.zeros(ctypes.sizeof(_lib.CollectStats), dtype=torch.uint8).pin_memory() \
            if torch.cuda.is_available() else torch.zeros(ctypes.sizeof(_lib.CollectStats), dtype=torch.uint8)
        # rgb_array only: each env's cost of its last step() (0 after a reset), drawn by render()
        self.last_cost = torch.zeros(E, dtype=torch.float32, device=dev) if render_mode == "rgb_array" else None

    def __len__(self):
        return self.env_num

    def seed(self, seed=None):
        if seed is not None:
            self.seed_value = int(seed) & 0xFFFFFFFF
        return [self.seed_value] * self.env_num

    # ---- descriptor shared by every rollout entry point ----------------------------------------
    def fill(self, r: "_lib.Rollout") -> None:
        r.kind, r.E, r.max_steps = self.kind, self.env_num, self.max_episode_steps
        r.seed_env = self.seed_value
        r.env_state, r.obs_cur = self.env_state.data_ptr(), self.obs_cur.data_ptr()
        r.env_t, r.ep_idx, r.act_ctr = self.env_t.data_ptr(), self.ep_idx.data_ptr(), self.act_ctr.data_ptr()
        r.active, r.done_now = self.active.data_ptr(), self.done_now.data_ptr()
        r.ep_rew, r.ep_len = self.ep_rew.data_ptr(), self.ep_len.data_ptr()
        r.stats = self.stats.data_ptr()
        low, high = self.action_space.low, self.action_space.high
        for j in range(self.A):
            r.act_low[j], r.act_high[j] = float(low[j]), float(high[j])

    def _ids(self, id) -> Optional[np.ndarray]:
        """The ``id`` argument of the vector-env protocol as host int32 env ids (None: every env in
        order).  The C ABI checks the range."""
        if id is None:
            return None
        if isinstance(id, torch.Tensor):
            id = id.cpu().numpy()
        ids = np.atleast_1d(np.asarray(id))
        if ids.ndim != 1 or ids.size == 0 or not np.issubdtype(ids.dtype, np.integer):
            raise ValueError(f"env ids must be a non-empty 1-D integer array (got shape {ids.shape}, "
                             f"dtype {ids.dtype})")
        return np.ascontiguousarray(ids, dtype=np.int32)

    def _stream(self) -> int:
        if self.device.type != "cuda":
            raise RuntimeError(f"DeviceVectorEnv steps CUDA devices only (device={self.device})")
        return torch.cuda.current_stream(self.device).cuda_stream

    def reset(self, id=None, **kwargs):
        """Start a fresh episode in every env, or in the envs ``id`` lists (tianshou's
        ``reset(id)``); returns their observations, device tensors, and one empty info dict each.
        A full reset returns the live ``obs_cur``.  ``ids=`` is accepted as another name of ``id``; other
        keywords (gymnasium's ``seed`` / ``options``) are ignored: the reset streams are keyed by the
        vector env's seed."""
        if "ids" in kwargs:
            if id is not None:
                raise TypeError("reset() got both id and ids")
            id = kwargs.pop("ids")
        ids = self._ids(id)
        r = _lib.Rollout()
        self.fill(r)
        r.mode = _lib.MODE_RANDOM
        with torch.cuda.device(self.device):
            stream = self._stream()
            if ids is None:
                _lib.check(_lib.lib.fsrl_env_reset_all(ctypes.byref(r), stream))
                if self.last_cost is not None:
                    self.last_cost.zero_()
                return self.obs_cur, [{} for _ in range(self.env_num)]
            obs = torch.empty((len(ids), self.D), dtype=torch.float32, device=self.device)
            _lib.check(_lib.lib.fsrl_env_reset_ids(ctypes.byref(r), ids.ctypes.data, len(ids), obs.data_ptr(), stream))
            if self.last_cost is not None:
                self.last_cost[torch.from_numpy(ids.astype(np.int64)).to(self.device)] = 0.0
        return obs, [{} for _ in range(len(ids))]

    def read_stats(self) -> "_lib.CollectStats":
        self._stats_host.copy_(self.stats, non_blocking=False)
        return _lib.CollectStats.from_buffer_copy(self._stats_host.numpy().tobytes())

    def step(self, action, id=None):
        """gymnasium's ``step`` over the envs ``id`` lists (all, in order, by default):
        ``action`` is (n, A) in the env's range, a CUDA tensor (used in place) or anything
        ``torch.as_tensor`` takes (uploaded).  Returns ``(obs_next, rew, terminated, truncated,
        info)`` as device tensors with ``info = Batch(cost=..., env_id=...)``.  Envs are not reset
        here: call ``reset(id)`` on the ones that finished.  ``truncated`` is set only when the
        horizon is reached without a termination, as in the collector's buffer.  A listed env must
        appear once."""
        from .data.batch import Batch
        ids = self._ids(id)
        n = self.env_num if ids is None else len(ids)
        act = torch.as_tensor(action, dtype=torch.float32,
                              device=action.device if isinstance(action, torch.Tensor) else None)
        if tuple(act.shape) != (n, self.A):
            raise ValueError(f"action must have shape ({n}, {self.A}), got {tuple(act.shape)}")
        stream = self._stream()
        act = act.to(self.device).contiguous()
        dev = self.device
        obs_next = torch.empty((n, self.D), dtype=torch.float32, device=dev)
        rew = torch.empty(n, dtype=torch.float32, device=dev)
        cost = torch.empty(n, dtype=torch.float32, device=dev)
        term = torch.empty(n, dtype=torch.bool, device=dev)        # written as 0 / 1 bytes
        trunc = torch.empty(n, dtype=torch.bool, device=dev)
        r = _lib.Rollout()
        self.fill(r)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib.fsrl_env_step(ctypes.byref(r), act.data_ptr(), None if ids is None else ids.ctypes.data,
                                              n, obs_next.data_ptr(), rew.data_ptr(), cost.data_ptr(),
                                              term.data_ptr(), trunc.data_ptr(), stream))
        env_id = np.arange(n) if ids is None else ids.astype(np.int64)
        if self.last_cost is not None:
            self.last_cost.index_copy_(0, torch.from_numpy(env_id).to(dev), cost)
        return obs_next, rew, term, trunc, Batch(cost=cost, env_id=env_id)

    def render(self, id=None, **kwargs):
        """With ``render_mode="rgb_array"``: one RGB frame per env (all, or the ones ``id`` lists; an env may be listed
        twice), a contiguous ``uint8`` CUDA tensor of shape ``(n, height, width, 3)``, drawn from the envs' state by
        csrc/render.cuh (views, primitives and palette: DESIGN §7; a user-defined env's scene is its struct's draw).  Robots whose last step cost are drawn in the cost
        colour.  Reads the env state only.  With ``render_mode=None``: ``None``."""
        if self.render_mode is None:
            return None
        ids = self._ids(id)
        n = self.env_num if ids is None else len(ids)
        height, width = self.render_size
        stream = self._stream()
        with torch.cuda.device(self.device):
            out = torch.empty((n, height, width, 3), dtype=torch.uint8, device=self.device)
            r = _lib.Rollout()
            self.fill(r)
            _lib.check(_lib.lib.fsrl_env_render(ctypes.byref(r), None if ids is None else ids.ctypes.data, n, height,
                                                width, self.last_cost.data_ptr(), out.data_ptr(), stream))
        return out

    def close(self):
        pass


# ---- user-defined device envs ------------------------------------------------------------------------------
_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
_INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")


class EnvBuildError(RuntimeError):
    """nvcc rejected a user env header; the message is the compiler's."""


def default_plugin_dir() -> str:
    """Where :func:`build_device_env` caches plugins by default: ``$FSRL_B200_CACHE/env_plugins``, else
    ``~/.cache/fsrl_b200/env_plugins``."""
    root = os.environ.get("FSRL_B200_CACHE") or os.path.join(os.path.expanduser("~"), ".cache", "fsrl_b200")
    return os.path.join(root, "env_plugins")


def _make(*args: str) -> subprocess.CompletedProcess:
    return subprocess.run(["make", "-s", "-C", _CSRC, *args], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                          text=True)


def plugin_path(header: str, out: Optional[str] = None) -> str:
    """The path :func:`build_device_env` gives the plugin of ``header``: ``<stem>-<key>.so`` in ``out``.  The key
    hashes the header's bytes, the library's ABI version, the compiler and flags (csrc/flags.mk) and the library
    sources the plugin is compiled from, so any change to one of them names a new artefact."""
    flags = _make("print-flags")
    if flags.returncode:
        raise EnvBuildError(flags.stdout)
    h = hashlib.sha256()
    parts = [open(header, "rb").read(), str(_lib.lib.fsrl_abi_version()).encode(), flags.stdout.strip().encode()]
    for name in sorted(os.listdir(_CSRC)):
        if name.endswith(".cuh") or name == "env_plugin.cu":
            parts += [name.encode(), open(os.path.join(_CSRC, name), "rb").read()]
    parts.append(open(os.path.join(_INCLUDE, "fsrl_b200.h"), "rb").read())
    for part in parts:
        h.update(len(part).to_bytes(8, "little"))
        h.update(part)
    stem = os.path.splitext(os.path.basename(header))[0]
    return os.path.join(os.path.abspath(out or default_plugin_dir()), f"{stem}-{h.hexdigest()[:20]}.so")


def build_device_env(header: str, out: Optional[str] = None) -> str:
    """Compile the env struct ``UserEnv`` that ``header`` defines into a plugin of the library (csrc/env_plugin.cu,
    with the library's compiler and flags) and return the plugin's path, under ``out`` (default:
    :func:`default_plugin_dir`).  A plugin already built from the same header, ABI, flags and sources is returned
    as it is, without compiling.  Raises ``ValueError`` naming the limit when ``UserEnv`` breaks one of
    1 <= A <= 8, D + A <= 80, 1 <= S <= 32, D >= 1, T >= 1, ``ValueError`` with the contract's text when ``UserEnv``
    defines a ``draw`` that cannot be called with the drawing contract's arguments, and :class:`EnvBuildError` with
    nvcc's message on any other compile error."""
    header = os.path.abspath(header)
    if not os.path.isfile(header):
        raise FileNotFoundError(header)
    path = plugin_path(header, out)
    if os.path.exists(path):
        return path
    os.makedirs(os.path.dirname(path), exist_ok=True)
    fd, tmp = tempfile.mkstemp(suffix=".so", prefix=".build-", dir=os.path.dirname(path))
    os.close(fd)
    try:
        res = _make("plugin", f"PLUGIN_HEADER={header}", f"PLUGIN_OUT={tmp}")
        if res.returncode:
            limits = re.findall(r"env plugin limit: ([^\"\n]+)", res.stdout)
            if limits:
                raise ValueError(f"{header}: UserEnv breaks the limit {limits[0]}")
            contract = re.findall(r"env plugin contract: ([^\"\n]+)", res.stdout)
            if contract:
                raise ValueError(f"{header}: env plugin contract: {contract[0]}")
            raise EnvBuildError(f"building the env plugin of {header} failed:\n{res.stdout}")
        os.replace(tmp + ".ptxas.log", path + ".ptxas.log")
        os.replace(tmp, path)          # atomic: a concurrent build of the same key finds a complete file
    finally:
        for f in (tmp, tmp + ".ptxas.log", tmp + ".o"):
            if os.path.exists(f):
                os.remove(f)
    return path


def _load_plugin(plugin: str):
    so = ctypes.CDLL(os.path.abspath(plugin))
    so.fsrl_env_plugin.restype = ctypes.POINTER(_lib.EnvPlugin)
    so.fsrl_env_plugin.argtypes = []
    return so, so.fsrl_env_plugin()


def _plugin_renderer(so: ctypes.CDLL):
    """The render table of a loaded plugin (its ``fsrl_env_plugin_render()``), or None when its struct has no draw
    or it was built before plugins could render (no such symbol)."""
    try:
        fn = so.fsrl_env_plugin_render
    except AttributeError:
        return None
    fn.restype = ctypes.POINTER(_lib.EnvRenderer)
    fn.argtypes = []
    table = fn()
    return table if table else None


def plugin_dims(plugin: str):
    """(D, A, S, T) of the env a plugin was built from (loads it; needs no GPU)."""
    _, t = _load_plugin(plugin)
    return t.contents.D, t.contents.A, t.contents.S, t.contents.T


def register_device_env(task: str, plugin: str) -> int:
    """Register the plugin ``plugin`` (a path from :func:`build_device_env`) under the task name ``task`` and return
    its env kind.  Afterwards ``task`` works wherever a built-in device task does (``DeviceVectorEnv``, ``make``,
    ``gym.make`` under ``compat.install()``, every collector, wrapper and agent); ``render_mode="rgb_array"`` too when
    the struct defines ``draw`` (DESIGN §7).  A built-in task name is refused, and so is a name already registered from another plugin; registering the same plugin
    under the same name again returns its kind."""
    if task in KINDS:
        raise ValueError(f"{task!r} is a built-in task; register the plugin under another name")
    path = os.path.realpath(plugin)
    if task in PLUGINS:
        if PLUGINS[task].path == path:
            return PLUGINS[task].kind
        raise ValueError(f"{task!r} is already registered from {PLUGINS[task].path}")
    so, table = _load_plugin(path)
    renderer = _plugin_renderer(so)
    kind = ctypes.c_int()
    _lib.check(_lib.lib.fsrl_env_register(table, ctypes.byref(kind)))
    if renderer is not None:
        _lib.check(_lib.lib.fsrl_env_register_renderer(kind.value, renderer))
    PLUGINS[task] = _Plugin(kind.value, path, so, renderer is not None)
    return kind.value


def _main(argv=None) -> int:
    import argparse
    ap = argparse.ArgumentParser(prog="python -m fsrl_b200.envs", description="user-defined device envs")
    sub = ap.add_subparsers(dest="cmd", required=True)
    b = sub.add_parser("build", help="compile a header defining UserEnv into an env plugin; prints its path")
    b.add_argument("header")
    b.add_argument("--out", default=None, help=f"plugin directory (default: {default_plugin_dir()})")
    args = ap.parse_args(argv)
    try:
        print(build_device_env(args.header, args.out))
    except (ValueError, EnvBuildError, FileNotFoundError) as e:
        print(e, file=sys.stderr)
        return 1
    return 0


from .obs_norm import ObsRunningMeanStd, VectorEnvNormObs  # noqa: E402,F401  (obs_norm imports DeviceVectorEnv)


if __name__ == "__main__":
    sys.exit(_main())
