"""The float64 CPU restatement of ``VectorEnvNormObs`` around an oracle vector env (``OracleVecEnv`` and its
subclasses), for the observation-normalization tests.

``OracleNormObs`` has the oracle env's ``step`` / ``reset`` / ``observe`` API, so ``oracle.collector.collect``
runs over it unchanged: ``step`` updates the statistics with the rows it returns and returns them normalized,
``reset`` (all or ``ids``) does the same with the reset rows, and ``observe`` returns each env's current normalized
observation.  The statistics follow tianshou 0.5's RunningMeanStd [UNVERIFIED, restated from memory]: batch mean
and population variance, the parallel update, ``clip((x - mean) / sqrt(var + eps), -clip_max, clip_max)``; here in
float64 with an integer count, each value rounded to float32 once."""
import numpy as np

EPS32 = float(np.finfo(np.float32).eps)


class OracleObsRms:
    def __init__(self, D, clip_max=10.0, eps=EPS32):
        self.mean = np.zeros(D, np.float64)
        self.var = np.ones(D, np.float64)
        self.count = 0
        self.clip_max, self.eps = clip_max, eps

    def update(self, x):
        x = np.asarray(x, np.float64)
        n = len(x)
        if n == 0:
            return
        bm, bv = x.mean(axis=0), x.var(axis=0)
        delta = bm - self.mean
        tot = self.count + n
        m2 = self.var * self.count + bv * n + delta ** 2 * self.count * n / tot
        self.mean = self.mean + delta * n / tot
        self.var = m2 / tot
        self.count = tot

    def norm(self, x):
        y = (np.asarray(x, np.float64) - self.mean) / np.sqrt(self.var + self.eps)
        if self.clip_max:
            y = np.clip(y, -self.clip_max, self.clip_max)
        return y.astype(np.float32)


class OracleNormObs:
    """An oracle vector env with normalized observations (``update``: the statistics take every returned row)."""

    def __init__(self, inner, update=True, rms=None):
        self.inner = inner
        self.E, self.D, self.A = inner.E, inner.D, inner.A
        self.T = getattr(inner, "T", None)
        self.update = update
        self.rms = rms if rms is not None else OracleObsRms(inner.D)
        self.cur = np.zeros((inner.E, inner.D), np.float32)

    def _take(self, ids, raw):
        if self.update:
            self.rms.update(raw)
        o = self.rms.norm(raw)
        self.cur[ids] = o
        return o

    def reset(self, ids=None):
        raw = self.inner.reset(ids)
        return self._take(np.arange(self.E) if ids is None else np.asarray(ids), raw)

    def step(self, act, ids=None):
        obs, rew, cost, term, trunc = self.inner.step(act, ids)
        o = self._take(np.arange(self.E) if ids is None else np.asarray(ids), obs)
        return o, rew, cost, term, trunc

    def observe(self, ids=None):
        return self.cur.copy() if ids is None else self.cur[np.asarray(ids)].copy()
