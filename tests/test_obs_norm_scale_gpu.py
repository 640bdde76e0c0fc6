"""Observation normalization (csrc/obsnorm.cu) and the host collect step (csrc/rollout_host.cu) past one tile of envs
and at the benchmarked 2048 envs, against the float64 restatement (tests/obs_norm_twin.py).

obs_rms_partials_kernel reduces each tile of 128 env ids (FSRL_OBS_RMS_TILE) to (count, mean, M2);
obs_rms_apply_kernel merges the tiles in tile order in every CTA of 32 env rows, CTA 0 publishes the statistics and
each CTA normalizes and writes back its own rows.  With 16 envs or fewer there is one tile and one apply CTA, so this
file runs the shapes where the tile merge, the apply CTAs past the first and the ring writes of env ids >= 32 work:
the kernels called directly on synthetic rows (E from 1 to 4097, D up to the widest 80, selections that leave tiles
empty, prior counts past int32, chains of updates, clipped, constant, large-offset and NaN columns), wrapped device
collects of up to 2048 envs whose restarts span several tiles, and the host collect step (one act CTA per
MlpTile<H>::R rows, 256 rows per store CTA) bitwise against the device path at 300 and 2048 envs.

Bounds as tests/test_obs_norm_gpu.py: raw dynamics bit-exact; count exact; mean and var within 1e-9 relative (1e-12
absolute), except the var of a large-offset column, whose bound is derived beside it; every normalized value within 1
float32 ulp of the float64 restatement, clipped values exactly +-clip_max, NaN where the restatement has NaN."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import buffer_to_numpy
from obs_norm_twin import EPS32, OracleObsRms
from test_obs_norm_gpu import (HOPPER, _assert_stats, _assert_successors, _check_host_vs_device,
                               _check_random_collect, _h, _replay_inline, _ulps, _wrapped)

pytestmark = pytest.mark.gpu

TILE = 128                   # FSRL_OBS_RMS_TILE: env ids per partials CTA
CAR_CIRCLE = "SafetyCarCircle-v0"
OFFSET, OFFSET_STD = 1e4, 1.0


# ---- the kernels directly ---------------------------------------------------------------------------------------
def _data(kind, E, D, rng):
    """[E, D] float32 rows: N(0, 1); per-column scales 1e-3 .. 1e3; column 0 constant; the last column at mean 1e4,
    std 1; or N(0, 30^2), most of it beyond +-clip_max once normalized by statistics near (0, 1)."""
    x = rng.standard_normal((E, D)).astype(np.float32)
    if kind == "scales":
        x *= (10.0 ** (np.arange(D) % 7 - 3)).astype(np.float32)
    elif kind == "const":
        x[:, 0] = np.float32(0.7)
    elif kind == "offset":
        x[:, -1] = (OFFSET + OFFSET_STD * rng.standard_normal(E)).astype(np.float32)
    elif kind == "wide":
        x *= np.float32(30.0)
    return x


def _prior(kind, D, rng):
    """(mean, var, count) before the update: the initial state, one observation, or 3e12 (past int32)."""
    if kind == "zero":
        return np.zeros(D), np.ones(D), 0
    if kind == "one":
        return rng.normal(size=D), rng.uniform(0.5, 2.0, D), 1
    return rng.normal(0.0, 0.1, D), rng.uniform(0.8, 1.2, D), 3 * 10 ** 12


def _ids(kind, E, rng):
    """The listed env ids (None: all E without an id list), ascending."""
    e = np.arange(E)
    if kind == "all":
        return None
    if kind == "skip0":              # tile 0 empty: the merge is seeded from tile 1
        return e[e >= TILE]
    if kind == "alt":                # tiles 1, 3, 5, ... empty
        return e[(e // TILE) % 2 == 0]
    if kind == "last":
        return e[-1:]
    if kind == "per_tile":           # one env per tile, at a different lane in each
        t = np.arange(0, E, TILE)
        return np.minimum(t + (37 * np.arange(len(t)) + 5) % TILE, E - 1)
    s = e[rng.random(E) < 0.37]      # a random 37 % subset
    return s if len(s) else e[:1]


def _rms(D, prior, clip_max=10.0, eps=EPS32):
    from fsrl_b200.obs_norm import ObsRunningMeanStd
    rms = ObsRunningMeanStd(D, "cuda", clip_max=clip_max, epsilon=eps)
    rms.copy_from(*prior)
    return rms


def _orms(D, prior, clip_max=10.0, eps=EPS32):
    o = OracleObsRms(D, clip_max, eps)
    o.mean, o.var, o.count = np.array(prior[0], np.float64), np.array(prior[1], np.float64), int(prior[2])
    return o


def _work(E, D):
    from fsrl_b200 import _lib
    return torch.zeros(int(_lib.lib.fsrl_obs_rms_work_bytes(E, D)), dtype=torch.uint8, device="cuda")


def _run(rms, work, x0, ids, update=True):
    """fsrl_obs_rms_rows over x0 (as VectorEnvNormObs._rows calls it): the rows after the call and `out`."""
    from fsrl_b200 import _lib
    E, D = x0.shape
    x = torch.from_numpy(np.ascontiguousarray(x0)).cuda()
    ids32 = None if ids is None else np.ascontiguousarray(ids, np.int32)
    n = E if ids is None else len(ids32)
    out = torch.full((n, D), 1234.5, dtype=torch.float32, device="cuda")
    desc = rms.descriptor(work, update)
    _lib.check(_lib.lib.fsrl_obs_rms_rows(ctypes.byref(desc), x.data_ptr(), E,
                                          None if ids32 is None else ids32.ctypes.data, n, None, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return _h(x), _h(out)


def _state(rms):
    return rms.mean.tobytes(), rms.var.tobytes(), rms.count


def _offset_var_rtol(merges):
    """The var bound of the large-offset column.  Each Chan merge combines means of magnitude `mean` that carry
    float64 rounding of order 2^-52 |mean|, and the squared differences it forms lose up to 2^-52 (mean/std)^2 of
    var relative to the result: 2^-52 * 1e8 = 2.2e-8 per merge (one per non-empty tile, one into the running
    statistics), summed over the merges the value has been through."""
    return merges * 2.0 ** -52 * (OFFSET / OFFSET_STD) ** 2


def _merges(E):
    return -(-E // TILE) + 1


def _assert_rows(E, x0, x1, out, ids, want, clip_max):
    """Unlisted rows bit-unchanged, `out` = the normalized x[ids] bit for bit, <= 1 ulp of the restatement (NaN
    where it has NaN), clipped values exactly +-clip_max."""
    sel = np.arange(E) if ids is None else np.asarray(ids)
    rest = np.ones(E, bool)
    rest[sel] = False
    assert np.array_equal(x1[rest].view(np.int32), x0[rest].view(np.int32))
    assert np.array_equal(out.view(np.int32), x1[sel].view(np.int32))
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(out), nan)
    assert _ulps(out[~nan], want[~nan]) <= 1
    if clip_max:
        at = np.abs(want) == np.float32(clip_max)
        assert np.array_equal(out[at], want[at])


def _assert_rms(rms, o, var_rtol):
    assert rms.count == o.count
    np.testing.assert_allclose(rms.mean, o.mean, rtol=1e-9, atol=1e-12)
    var, want = rms.var, o.var
    assert np.all(np.abs(var - want) <= 1e-12 + var_rtol * np.abs(want)), np.abs(var - want) / np.abs(want)


# E hits the tile edges (128), the apply-CTA edges (32) and last partial tiles of one row; D = 80 is FSRL_ENG_DX_LD.
KERNEL_CASES = [
    # E, D, selection, data, prior, clip_max
    (1, 1, "all", "normal", "zero", 10.0),
    (1, 3, "all", "scales", "one", 10.0),
    (32, 17, "all", "normal", "zero", 10.0),
    (33, 17, "last", "normal", "one", 10.0),
    (33, 3, "rand", "scales", "zero", 10.0),
    (127, 76, "all", "const", "zero", 10.0),
    (128, 80, "all", "normal", "zero", 10.0),
    (128, 1, "rand", "normal", "huge", 10.0),
    (129, 3, "all", "normal", "zero", 10.0),
    (129, 17, "last", "scales", "one", 10.0),
    (129, 80, "skip0", "normal", "zero", 10.0),
    (257, 17, "alt", "offset", "zero", 10.0),
    (257, 76, "per_tile", "normal", "one", 10.0),
    (257, 3, "rand", "wide", "huge", 10.0),
    (1000, 17, "all", "offset", "zero", 10.0),
    (1000, 80, "skip0", "scales", "one", 10.0),
    (1000, 3, "alt", "const", "zero", 10.0),
    (1000, 76, "rand", "wide", "huge", 0.0),
    (2048, 76, "all", "normal", "zero", 10.0),
    (2048, 80, "rand", "scales", "one", 10.0),
    (2048, 17, "per_tile", "wide", "huge", 10.0),
    (2048, 1, "last", "normal", "zero", 10.0),
    (2048, 3, "skip0", "offset", "huge", 10.0),
    (4097, 17, "all", "scales", "zero", 10.0),
    (4097, 3, "last", "offset", "one", 10.0),
    (4097, 80, "skip0", "const", "zero", 10.0),
    (4097, 76, "alt", "normal", "huge", 10.0),
    (4097, 3, "per_tile", "normal", "zero", 10.0),
    (4097, 17, "rand", "wide", "huge", 10.0),
]


@pytest.mark.parametrize("E,D,sel,data,prior,clip_max", KERNEL_CASES)
def test_rows_match_float64(E, D, sel, data, prior, clip_max):
    """One update + normalize of the listed rows against OracleObsRms; the same ids listed shuffled and a second
    identical call give the same bits."""
    rng = np.random.default_rng(E * 1009 + D * 31 + len(sel) + len(data))
    x0, ids, p = _data(data, E, D, rng), _ids(sel, E, rng), _prior(prior, D, rng)
    o = _orms(D, p, clip_max)
    rows = x0 if ids is None else x0[ids]
    o.update(rows)
    want = o.norm(rows)
    rms, work = _rms(D, p, clip_max), _work(E, D)
    x1, out = _run(rms, work, x0, ids)
    var_rtol = np.full(D, 1e-9)
    if data == "offset":
        var_rtol[-1] = _offset_var_rtol(_merges(E))
    _assert_rms(rms, o, var_rtol)
    _assert_rows(E, x0, x1, out, ids, want, clip_max)
    if data == "const":          # a constant column: var exactly 0, every normalized value exactly 0
        assert rms.var[0] == 0.0 and o.var[0] == 0.0
        assert np.all(out[:, 0] == 0.0)
    if data == "wide" and clip_max:
        assert (np.abs(out) == np.float32(clip_max)).mean() > 0.5
    if data == "wide" and not clip_max:
        assert np.abs(out).max() > 50.0
    # the results depend only on which ids hold which rows, not on the order they are listed in
    listed = np.arange(E) if ids is None else ids
    perm = rng.permutation(len(listed))
    rms2 = _rms(D, p, clip_max)
    x2, out2 = _run(rms2, _work(E, D), x0, listed[perm])
    assert _state(rms2) == _state(rms)
    assert np.array_equal(x2.view(np.int32), x1.view(np.int32))
    assert np.array_equal(out2.view(np.int32), out[perm].view(np.int32))
    # and a second identical call gives identical bits
    rms3 = _rms(D, p, clip_max)
    x3, out3 = _run(rms3, work, x0, ids)
    assert _state(rms3) == _state(rms)
    assert np.array_equal(x3.view(np.int32), x1.view(np.int32)) and np.array_equal(out3.view(np.int32),
                                                                                     out.view(np.int32))


def test_chain_of_updates_matches_float64():
    """20 updates of mixed sizes through one workspace from the initial state; the count is exact after each.
    Column 0 is constant throughout (var stays exactly 0), the last column sits at mean 1e4."""
    E, D = 2048, 17
    rng = np.random.default_rng(7)
    rms, work, o = _rms(D, _prior("zero", D, rng)), _work(E, D), OracleObsRms(D)
    sizes = [2048, 1, 129, 37, 2048, 128, 700, 1, 2047, 255, 3, 1500, 64, 2048, 129, 900, 5, 1024, 333, 2048]
    merges, count = 0, 0
    for i, k in enumerate(sizes):
        x0 = _data("offset", E, D, rng)
        x0[:, 0] = np.float32(-3.25)
        ids = None if k == E and i % 2 == 0 else np.sort(rng.choice(E, k, replace=False))
        rows = x0 if ids is None else x0[ids]
        o.update(rows)
        want = o.norm(rows)
        x1, out = _run(rms, work, x0, ids)
        count += k
        merges += len(np.unique((np.arange(E) if ids is None else ids) // TILE)) + 1
        assert rms.count == o.count == count, i
        var_rtol = np.full(D, 1e-9)
        var_rtol[-1] = _offset_var_rtol(merges)
        _assert_rms(rms, o, var_rtol)
        _assert_rows(E, x0, x1, out, ids, want, 10.0)
        assert rms.var[0] == 0.0 and np.all(out[:, 0] == 0.0), i


def test_frozen_rows_leave_statistics_bit_unchanged():
    """update = 0 at E = 2048: the statistics keep their bits, the listed rows are normalized with them."""
    E, D = 2048, 17
    rng = np.random.default_rng(11)
    p = _prior("huge", D, rng)
    p = (p[0], p[1], 123456789)
    rms, o = _rms(D, p), _orms(D, p)
    before = _state(rms)
    for sel in ("all", "rand", "alt"):
        x0, ids = _data("scales", E, D, rng), _ids(sel, E, rng)
        x1, out = _run(rms, _work(E, D), x0, ids, update=False)
        assert _state(rms) == before, sel
        _assert_rows(E, x0, x1, out, ids, o.norm(x0 if ids is None else x0[ids]), 10.0)


def test_nan_observation_poisons_only_its_column():
    """One NaN in column d of an env in tile 2: mean and var of column d become NaN, as in the restatement, and
    every selected row's column d comes back NaN (not -clip_max); the other columns are unaffected."""
    E, D, d = 1000, 17, 5
    rng = np.random.default_rng(3)
    for ids in (None, np.sort(np.concatenate([[300], rng.choice(np.arange(301, E), 200, replace=False)]))):
        x0 = _data("normal", E, D, rng)
        x0[300, d] = np.nan
        p = _prior("one", D, rng)
        o = _orms(D, p)
        rows = x0 if ids is None else x0[ids]
        o.update(rows)
        want = o.norm(rows)
        rms = _rms(D, p)
        x1, out = _run(rms, _work(E, D), x0, ids)
        assert np.isnan(o.mean[d]) and np.isnan(o.var[d])
        np.testing.assert_allclose(rms.mean, o.mean, rtol=1e-9, atol=1e-12, equal_nan=True)
        np.testing.assert_allclose(rms.var, o.var, rtol=1e-9, atol=1e-12, equal_nan=True)
        assert rms.count == o.count
        assert np.isnan(out[:, d]).all()
        _assert_rows(E, x0, x1, out, ids, want, 10.0)


def test_zero_epsilon_constant_column_is_nan():
    """epsilon = 0 with a constant column: (x - mean) / sqrt(0) = 0 / 0 is NaN, as in the restatement."""
    E, D = 300, 3
    rng = np.random.default_rng(5)
    x0 = _data("const", E, D, rng)
    p = _prior("zero", D, rng)
    o = _orms(D, p, eps=0.0)
    o.update(x0)
    with np.errstate(invalid="ignore"):
        want = o.norm(x0)
    rms = _rms(D, p, eps=0.0)
    x1, out = _run(rms, _work(E, D), x0, None)
    assert rms.var[0] == 0.0 and np.isnan(want[:, 0]).all()
    _assert_rms(rms, o, np.full(D, 1e-9))
    _assert_rows(E, x0, x1, out, None, want, 10.0)


# ---- wrapped device-env collects at scale -----------------------------------------------------------------------
class _Record:
    """An oracle vector env that records which envs stepped and the ids of every partial reset (the restarts)."""

    def __init__(self, inner):
        self.inner = inner
        self.stepped = np.zeros(inner.E, bool)
        self.restarts = []

    def __getattr__(self, k):
        return getattr(self.inner, k)

    def step(self, act, ids=None):
        self.stepped[slice(None) if ids is None else np.asarray(ids)] = True
        return self.inner.step(act, ids)

    def reset(self, ids=None):
        if ids is not None:
            self.restarts.append(np.asarray(ids).copy())
        return self.inner.reset(ids)


def _assert_not_vacuous(rec, E, restarts):
    assert rec.stepped[TILE:].any() and rec.stepped[E - 1]
    if restarts:             # a vector step restarted envs of at least two tiles
        assert max(len(np.unique(r // TILE)) for r in rec.restarts) >= 2


@pytest.mark.parametrize("task,E,n_episode,H,restarts", [
    (HOPPER, 129, 129, 64, False),          # inline path, a one-row last tile
    (HOPPER, 300, 451, 64, True),           # resolve path: the surplus rule retires envs, restarts over 3 tiles
    (HOPPER, 2048, 3073, 64, True),
    (CAR_CIRCLE, 2048, 2048, 256, False),   # c2's shape
], ids=["hopper-129-inline", "hopper-300-resolve", "hopper-2048-resolve", "carcircle-2048-c2"])
def test_random_collect_at_scale_matches_twin(task, E, n_episode, H, restarts):
    from fsrl_b200 import envs
    T = envs.make(task).spec.max_episode_steps
    onorm = _check_random_collect(task, E, n_episode, hidden=(H, H), twin=_Record, T=T)
    _assert_not_vacuous(onorm.inner, E, restarts)


@pytest.mark.parametrize("task,E,H", [(HOPPER, 129, 64), (CAR_CIRCLE, 2048, 256)], ids=["hopper-129", "carcircle-2048"])
def test_train_collect_at_scale_replays_through_twin(task, E, H):
    from fsrl_b200 import envs
    T = envs.make(task).spec.max_episode_steps
    policy, venv, norm, buf, col, onorm = _wrapped(task, E, E * T * 2, hidden=(H, H))
    onorm.inner = _Record(onorm.inner)
    policy.train()
    assert col.collect(n_episode=E)["n/ep"] == E
    b = buffer_to_numpy(buf)
    _replay_inline(policy, norm, b, buf.cap, E, onorm)
    _assert_stats(norm.get_obs_rms(), onorm.rms)
    assert np.array_equal(_h(venv.env_state), onorm.inner.st)
    _assert_successors(b, buf.cap, E)
    _assert_not_vacuous(onorm.inner, E, False)


def test_frozen_eval_collect_at_scale():
    """An eval-mode collect of 300 envs with update_obs_rms=False from non-trivial statistics: the statistics keep
    their bits, every stored row is within 1 ulp of the twin's."""
    E = 300
    policy, venv, norm, buf, col, onorm = _wrapped(HOPPER, E, E * 1000 * 2, update=False)
    rng = np.random.default_rng(2)
    D = venv.D
    stats = (rng.normal(0.0, 0.5, D), rng.uniform(0.2, 3.0, D), 98765)
    norm.get_obs_rms().copy_from(*stats)
    onorm.rms.mean, onorm.rms.var, onorm.rms.count = stats[0].copy(), stats[1].copy(), stats[2]
    norm.reset()
    onorm.reset()
    onorm.inner = _Record(onorm.inner)
    before = _state(norm.get_obs_rms())
    policy.eval()
    assert col.collect(n_episode=E)["n/ep"] == E
    assert _state(norm.get_obs_rms()) == before
    b = buffer_to_numpy(buf)
    _replay_inline(policy, norm, b, buf.cap, E, onorm)
    assert _ulps(_h(venv.obs_cur), onorm.observe()) <= 1
    assert np.array_equal(_h(venv.env_state), onorm.inner.st)
    _assert_not_vacuous(onorm.inner, E, False)


# ---- the host collect step at scale, bitwise against the device path ---------------------------------------------
# E = 300 at H = 64: 5 act CTAs (MlpTile<64>::R = 64 rows), 2 store CTAs (256 rows each); E = 2048 at H = 256: 128 act
# CTAs (16 rows), 8 store CTAs.  n_episode is no multiple of E, so restarts and the surplus rule run in both collects.
HOST_SIZES = [(300, 64, 451), (2048, 256, 2349)]


@pytest.mark.parametrize("E,H,n_episode", HOST_SIZES, ids=["E300-H64", "E2048-H256"])
@pytest.mark.parametrize("head", ["ppo", "sac"])
def test_host_step_unwrapped_at_scale_matches_device(E, H, n_episode, head):
    from test_host_env_gpu import COLS, _assert_stats_equal, _collect, _policy

    from fsrl_b200.envs import DeviceVectorEnv
    from host_twin import host_twin
    policy = _policy(head, HOPPER, H)
    cap = 1000 * (n_episode // E + 2)
    sd, rd, cd = _collect(policy, DeviceVectorEnv(HOPPER, E, seed=21), "train", n_episode, cap)
    sh, rh, ch = _collect(policy, host_twin(HOPPER, E, 21), "train", n_episode, cap)
    _assert_stats_equal(sd, sh)
    for k in COLS:
        assert np.array_equal(rd[k], rh[k]), k
    assert np.array_equal(cd, ch)
    assert (rd["len"][TILE:] > 0).any() and ch[E - 1] > 0


@pytest.mark.parametrize("E,H,n_episode", HOST_SIZES, ids=["E300-H64", "E2048-H256"])
def test_host_step_wrapped_at_scale_matches_device(E, H, n_episode):
    _check_host_vs_device(HOPPER, E, n_episode, hidden=(H, H))
