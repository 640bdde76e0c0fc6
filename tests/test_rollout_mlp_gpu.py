"""The tile MLP forward (csrc/mlpfwd.cu) and the fused rollout step (csrc/rollout.cu) at every hidden
width, env, head and mode, against float64 and the oracle collector, across many CTAs.

A. fsrl_mlp_forward against a float64 forward of the same fp32 parameters and rows: every output must
   satisfy |y - y64| <= 2^-16 m, with the magnitude recursion m1 = |X||W1| + |b1|,
   m2 = m1 |W2| + |b2|, m = m2 |W3| + |b3|, which bounds the error propagated through both ReLU layers.
   Row counts straddle the tile size R = max(4096 / H, 16); rows past n_rows keep a NaN sentinel.
B. The rollout's MLP observed directly: an unbounded GAUSS_INDEP actor in eval mode stores its raw head
   output as the action.  fsrl_mlp_forward on the stored observations, gathered so that every env sits
   at the tile position it had in the rollout, must reproduce it bit for bit (both kernels run the same
   mlp.cuh blocks on the same staged tile), and within the bound of A.  The stored actions replayed
   through the CPU env twin must give bit-identical observations, rewards and costs.
C. The rollout epilogue per head and mode: from the head output (B) and the Philox noise, the stored
   action and log-prob are evaluated in float64 and compared against a first-order error budget of the
   kernel's fp32 operation sequence.
D. Episode bookkeeping at scale.  No env ever terminates (every Env<K>::step sets term = false), so every
   episode truncates at T and which envs finish, retire and reset does not depend on the actions: counts,
   buffer pointers and episode indices are compared as exact integers.  The termination path
   (done_now == 1, b_term) cannot be reached from these envs and is not covered here.
"""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

TOL = 2.0 ** -16               # forward: |err| <= TOL * m
U = 2.0 ** -24                 # unit roundoff of fp32
SENT = 0x7FC0DEAD              # quiet-NaN bit pattern for memory a kernel must not write
HS = (64, 128, 256, 512)
TASKS = ("SafetyCarCircle-v0", "SafetyCarRun-v0", "SafetyBallCircle-v0", "SafetyBallRun-v0",
         "SafetyAntCircle-v0", "SafetyPointGoal1Gymnasium-v0")
LOG_SQRT_2PI = 0.9189385332046727


def _tile_rows(H):
    return max(4096 // H, 16)            # MlpTile<H>::R


def _bits(t):
    return t.contiguous().view(torch.int32)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- networks and the float64 forward ---------------------------------------------------------------------
def _actor(D, H, heads, n_extra=0, seed=0, head_gain=1.0):
    """One net in its own arena.  He-scaled weights and small biases: for O(1) inputs about half the
    ReLUs are active and the outputs are O(1), or O(sqrt(head_gain))."""
    from fsrl_b200.nets import Arena, NetSlot
    gen = torch.Generator().manual_seed(seed)

    def lin(i, o, gain):
        m = nn.Linear(i, o)
        with torch.no_grad():
            m.weight.copy_(torch.randn(o, i, generator=gen) * (gain / i) ** 0.5)
            m.bias.copy_(0.1 * torch.randn(o, generator=gen))
        return m

    extra = nn.Parameter(torch.zeros(n_extra)) if n_extra else None
    slot = NetSlot("actor", None, lin(D, H, 2.0), lin(H, H, 2.0), [lin(H, a, head_gain) for a in heads], extra)
    return Arena([slot], "cuda"), slot


def _ref64(arena, slot, X):
    """float64 forward of the fp32 parameters on the fp32 rows X, and its magnitude recursion"""
    th = arena.theta.detach().double().cpu()
    w1, b1, w2, b2, w3, b3, _ = slot.offsets()
    D, H, out = slot.D, slot.H, slot.out
    W1, B1 = th[w1:w1 + D * H].view(D, H), th[b1:b1 + H]
    W2, B2 = th[w2:w2 + H * H].view(H, H), th[b2:b2 + H]
    W3, B3 = th[w3:w3 + H * out].view(H, out), th[b3:b3 + out]
    X = X.detach().double().cpu()
    h1, m1 = (X @ W1 + B1).clamp_min(0), X.abs() @ W1.abs() + B1.abs()
    h2, m2 = (h1 @ W2 + B2).clamp_min(0), m1 @ W2.abs() + B2.abs()
    return h2 @ W3 + B3, m2 @ W3.abs() + B3.abs()


def _mlp_forward(arena, slot, x, idx, n_rows, y):
    from fsrl_b200 import _lib
    m = arena.mlp3(slot)
    _lib.check(_lib.lib.fsrl_mlp_forward(ctypes.byref(m), x.data_ptr(), None if idx is None else idx.data_ptr(),
                                         n_rows, y.data_ptr(), _stream()))


def _padded_out(n_rows, out, R):
    """an output with R + 3 sentinel rows past n_rows: room for a whole tile written past the end"""
    y = torch.empty(n_rows + R + 3, out, dtype=torch.float32, device="cuda")
    _bits(y).fill_(SENT)
    return y


class Report:
    """largest |err| / scale per quantity; asserts it is <= bound element-wise (an element with scale 0
    must be exact)"""

    def __init__(self, case, bound):
        self.case, self.bound, self.worst = case, bound, {}

    def close(self, name, got, ref, scale):
        got, ref, scale = (a.detach().double().cpu().numpy() if torch.is_tensor(a) else np.asarray(a, np.float64)
                           for a in (got, ref, scale))
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        err = np.where(got == ref, 0.0, np.abs(got - ref))
        assert not np.isnan(err).any(), f"{self.case} {name}: NaN"
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(scale > 0, err / scale, np.where(err > 0, np.inf, 0.0))
        r = float(ratio.max()) if ratio.size else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), r)
        if r > self.bound:
            i = np.unravel_index(int(ratio.argmax()), ratio.shape)
            raise AssertionError(f"{self.case} {name}: |err| / scale = {r:.3g} > {self.bound:.3g} at {i} "
                                 f"(got {got[i]:.9g}, want {ref[i]:.9g}, scale {scale[i]:.3g})")

    def show(self):
        print(f"\n{self.case}: worst ratio (bound {self.bound:.3g}) " +
              " ".join(f"{k}={v:.2e}" for k, v in self.worst.items()))


# ---- A. fsrl_mlp_forward against float64 --------------------------------------------------------------------
DS = (1, 7, 8, 33, 34, 60, 64)
OUTS = (1, 2, 3, 9, 16)


def _fwd_cases():
    out, k = [], 0
    for H in HS:
        R = _tile_rows(H)
        for B in (1, R - 1, R, R + 1, 5 * R + 3, 4097):
            D, o = DS[k % len(DS)], OUTS[k % len(OUTS)]
            out.append(pytest.param(H, D, o, B, id=f"H{H}-D{D}-out{o}-B{B}"))
            k += 1
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("H,D,out,B", _fwd_cases())
def test_mlp_forward_matches_float64(H, D, out, B):
    arena, slot = _actor(D, H, [out], seed=H + 13 * D + B)
    R = _tile_rows(H)
    gen = torch.Generator().manual_seed(7 * B + H)
    rep = Report(f"mlp_forward H={H} D={D} out={out} B={B}", TOL)
    xp = torch.randn(B, D, generator=gen)
    n_src = B // 2 + 5                  # fewer source rows than B: the gather repeats rows, out of order
    xs = torch.randn(n_src, D, generator=gen)
    idx = torch.randint(0, n_src, (B,), generator=gen, dtype=torch.int32)
    idx[-1] = idx[0]
    for mode, x, ii, X in (("plain", xp, None, xp), ("gather", xs, idx, xs[idx.long()])):
        y = _padded_out(B, out, R)
        _mlp_forward(arena, slot, x.cuda(), None if ii is None else ii.cuda(), B, y)
        ref, mag = _ref64(arena, slot, X)
        rep.close(mode, y[:B], ref, mag)
        assert bool((_bits(y[B:]) == SENT).all()), f"{mode}: rows >= n_rows written"
    rep.show()


@pytest.mark.gpu
@pytest.mark.parametrize("H,D,out,B", [(256, 8, 1, 614400), (128, 60, 2, 2048000)],
                         ids=["c2-H256-D8-B614400", "c3-H128-D60-B2048000"])
def test_mlp_forward_bench_sizes(H, D, out, B):
    """the critic pass over a whole benchmark buffer: every row finite, the first and last two tiles and
    ~2000 random rows against float64"""
    arena, slot = _actor(D, H, [out], seed=H + D)
    R = _tile_rows(H)
    x = torch.randn(B, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    y = _padded_out(B, out, R)
    _mlp_forward(arena, slot, x, None, B, y)
    assert bool(torch.isfinite(y[:B]).all()), "non-finite outputs"
    assert bool((_bits(y[B:]) == SENT).all()), "rows >= n_rows written"
    pick = torch.randint(0, B, (2000,), generator=torch.Generator().manual_seed(4))
    rows = torch.cat([torch.arange(2 * R), torch.arange(B - 2 * R, B), pick]).cuda()
    rep = Report(f"mlp_forward H={H} D={D} out={out} B={B}", TOL)
    ref, mag = _ref64(arena, slot, x[rows])
    rep.close("rows", y[rows], ref, mag)
    rep.show()


# ---- rollout rig ----------------------------------------------------------------------------------------------
class _Policy:
    """The policy side of FastCollector: fill_rollout() hands the rollout an arena actor with the head,
    mode and action mapping under test"""

    def __init__(self, arena, slot, head, mode, bounded=False, max_action=1.0, action_bound="clip",
                 action_scaling=True, expl_sigma=0.0, seed=0):
        self.arena, self.slot, self.head, self.mode, self.bounded = arena, slot, head, mode, bounded
        self.max_action, self.action_bound, self.action_scaling = max_action, action_bound, action_scaling
        self.expl_sigma, self.seed = expl_sigma, seed

    def fill_rollout(self, r, exploration_noise=False):
        from fsrl_b200 import _lib
        from fsrl_b200.nets import SIGMA_MAX, SIGMA_MIN
        r.actor = self.arena.mlp3(self.slot)
        r.head = {"indep": _lib.HEAD_GAUSS_INDEP, "cond": _lib.HEAD_GAUSS_COND, "det": _lib.HEAD_DETERMINISTIC}[self.head]
        r.mode = {"train": _lib.MODE_TRAIN, "eval": _lib.MODE_EVAL, "random": _lib.MODE_RANDOM}[self.mode]
        r.bounded = int(self.bounded)
        r.action_bound = {"": _lib.BOUND_NONE, "clip": _lib.BOUND_CLIP, "tanh": _lib.BOUND_TANH}[self.action_bound]
        r.action_scaling = int(self.action_scaling)
        r.max_action, r.expl_sigma = self.max_action, self.expl_sigma
        r.sigma_min, r.sigma_max = SIGMA_MIN, SIGMA_MAX
        r.tanh_eps = float(np.finfo(np.float32).eps)
        r.seed_act = self.seed
        r.log_sigma = self.arena.extra_ptr(self.slot)


def _rig(kind, E, cap_steps=None, seed=0):
    from fsrl_b200.data import VectorReplayBuffer
    from fsrl_b200.envs import DeviceVectorEnv
    venv = DeviceVectorEnv(TASKS[kind], E, device="cuda", seed=seed)
    buf = VectorReplayBuffer(E * (cap_steps or venv.max_episode_steps), E, device="cuda")
    return venv, buf


def _collector(policy, venv, buf):
    from fsrl_b200.data import FastCollector
    col = FastCollector(policy, venv, buf)        # resets every env
    col.reset_buffer()
    return col


def _run_steps(col, n_episode, n):
    """collect_begin and n rollout steps through the collector's descriptor (a collect cut short)"""
    from fsrl_b200 import _lib
    r = col._descriptor(False)
    r.inline_done = int(n_episode <= col.env_num)
    _lib.check(_lib.lib.fsrl_collect_begin(ctypes.byref(r), n_episode, _stream()))
    _lib.check(_lib.lib.fsrl_rollout_steps(ctypes.byref(r), n, _stream()))
    torch.cuda.synchronize()


def _slots(buf, E, t):
    """flat buffer rows of step t of every env (int32, device)"""
    return torch.arange(E, dtype=torch.int32, device="cuda") * buf.cap + t


def _head_out(arena, slot, buf, E, t):
    """fsrl_mlp_forward on the stored observations of step t, one gathered row per env in env order:
    env e sits at row e % R of tile e // R, as in the rollout"""
    y = _padded_out(E, slot.out, _tile_rows(slot.H))
    _mlp_forward(arena, slot, buf.obs, _slots(buf, E, t), E, y)
    assert bool((_bits(y[E:]) == SENT).all())
    return y[:E]


def _map_action(a, bound, scaling):
    """map_action with the kernel's fp32 operations (action space [-1, 1])"""
    f = np.float32
    a = np.asarray(a, f)
    if bound == "clip":
        a = np.minimum(f(1), np.maximum(f(-1), a))
    if scaling:
        low, high = f(-1), f(1)
        a = low + ((high - low) * (a + f(1))) / f(2)
    return a.astype(f)


def _replay(kind, E, seed, buf, n, bound, scaling):
    """the stored actions through the CPU env twin: observations, rewards, costs and truncation flags
    must be bit-identical"""
    from oracle.envs import OracleVecEnv
    rows = (torch.arange(E, device="cuda")[:, None] * buf.cap + torch.arange(n, device="cuda")[None]).reshape(-1)
    g = lambda t: t[rows].cpu().numpy().reshape(E, n, *t.shape[1:])
    b = {k: g(getattr(buf, k)) for k in ("obs", "obs_next", "act", "rew", "cost", "truncated")}
    for k in ("obs", "obs_next", "act", "rew"):
        assert np.isfinite(b[k]).all(), f"non-finite {k}"
    oenv = OracleVecEnv(kind, E, seed)
    obs = oenv.reset()
    for t in range(n):
        assert _same_bits(b["obs"][:, t], obs), f"step {t}: obs"
        obs, rew, cost, term, trunc = oenv.step(_map_action(b["act"][:, t], bound, scaling))
        assert _same_bits(b["obs_next"][:, t], obs), f"step {t}: obs_next"
        assert _same_bits(b["rew"][:, t], rew), f"step {t}: rew"
        assert _same_bits(b["cost"][:, t], cost), f"step {t}: cost"
        assert np.array_equal(b["truncated"][:, t].astype(bool), trunc), f"step {t}: truncated"


# ---- B. the rollout's MLP, observed directly --------------------------------------------------------------------
MAPS = (("clip", True), ("", False), ("clip", False), ("", True))


def _b_cases():
    out = []
    for kind in range(6):
        for hi, H in enumerate(HS):
            E = 3 * _tile_rows(H) + 5           # several CTAs and a partial last tile
            bound, scaling = MAPS[(kind + hi) % 4]
            out.append(pytest.param(kind, H, E, bound, scaling,
                                    id=f"{TASKS[kind].split('-')[0][6:]}-H{H}-E{E}-{bound or 'none'}-{'scaled' if scaling else 'raw'}"))
    # the benchmark shapes
    for kind, H, E, bound, scaling in ((0, 256, 2048, "clip", True), (5, 128, 2048, "clip", True),
                                       (1, 128, 4096, "", True), (4, 512, 1024, "clip", False)):
        out.append(pytest.param(kind, H, E, bound, scaling,
                                id=f"bench-{TASKS[kind].split('-')[0][6:]}-H{H}-E{E}-{bound or 'none'}-{'scaled' if scaling else 'raw'}"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind,H,E,bound,scaling", _b_cases())
def test_rollout_head_output_bitwise_and_env_replay(kind, H, E, bound, scaling):
    """one whole episode of every env; the head output is checked at steps 0, 1, T / 2 and T - 1"""
    from fsrl_b200.envs import env_dims
    D, A, _, T = env_dims(kind)
    # unbounded actions of O(1) reach the envs unclipped without the clip bound, and the feedback through
    # the velocities then overflows some trajectories: keep those actions O(0.2)
    arena, slot = _actor(D, H, [A], n_extra=A, seed=31 * kind + H, head_gain=1.0 if bound == "clip" else 0.05)
    venv, buf = _rig(kind, E, seed=kind + H + E)
    col = _collector(_Policy(arena, slot, "indep", "eval", action_bound=bound, action_scaling=scaling), venv, buf)
    n = T
    _run_steps(col, E, n)
    rep = Report(f"rollout head H={H} {TASKS[kind]} E={E} steps={n}", TOL)
    for t in sorted({0, 1, n // 2, n - 1}):
        rows = _slots(buf, E, t).long()
        y = _head_out(arena, slot, buf, E, t)
        act = buf.act[rows]
        diff = int((_bits(y) != _bits(act)).any(1).sum())
        assert diff == 0, f"step {t}: fsrl_mlp_forward differs from the rollout's head output in {diff} of {E} envs"
        ref, mag = _ref64(arena, slot, buf.obs[rows])
        rep.close(f"t{t}", act, ref, mag)
    _replay(kind, E, venv.seed_value, buf, n, bound, scaling)
    rep.show()


# ---- C. the epilogue per head and mode --------------------------------------------------------------------------
class Ev:
    """A float64 value and a first-order bound on the absolute error of the fp32 kernel computing it: each
    fp32 operation adds c * 2^-24 * |its result| (c = 2 for + - * / fma, 4 for tanhf expf logf log1pf),
    and the error of each operand is carried through the derivative of the operation."""

    def __init__(self, v, e=0.0):
        self.v = np.asarray(v, np.float64)
        self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape)

    def __getitem__(self, k):
        return Ev(self.v[k], self.e[k])


def _c(x):
    return Ev(np.float64(np.float32(x)))


def _add(a, b):
    v = a.v + b.v
    return Ev(v, a.e + b.e + 2 * U * np.abs(v))


def _sub(a, b):
    v = a.v - b.v
    return Ev(v, a.e + b.e + 2 * U * np.abs(v))


def _mul(a, b):
    v = a.v * b.v
    return Ev(v, np.abs(b.v) * a.e + np.abs(a.v) * b.e + 2 * U * np.abs(v))


def _fma(a, b, c):
    v = a.v * b.v + c.v
    return Ev(v, np.abs(b.v) * a.e + np.abs(a.v) * b.e + c.e + 2 * U * np.abs(v))


def _div(a, b):
    v = a.v / b.v
    return Ev(v, a.e / np.abs(b.v) + np.abs(v) * b.e / np.abs(b.v) + 2 * U * np.abs(v))


def _tanh(a):
    v = np.tanh(a.v)
    return Ev(v, (1 - v * v) * a.e + 4 * U * np.abs(v))


def _exp(a):
    v = np.exp(a.v)
    return Ev(v, v * a.e + 4 * U * v)


def _log(a):
    v = np.log(a.v)
    return Ev(v, a.e / np.abs(a.v) + 4 * U * np.abs(v))


def _log1p(a):
    with np.errstate(divide="ignore"):
        v = np.log1p(a.v)
        return Ev(v, a.e / np.abs(1 + a.v) + 4 * U * np.abs(v))


def _epilogue64(o, eps, p, log_sigma):
    """float64 action and log-prob of rollout.cu's epilogue (sampling, log-prob, exploration noise) from
    the fp32 head output o (E, out) and noise eps (E, A); the noise may differ from the kernel's by an
    ulp (its Box-Muller runs in float64 libm on both sides)"""
    from fsrl_b200.nets import SIGMA_MAX, SIGMA_MIN
    E, A = eps.shape
    if p.mode == "random":
        v = Ev(eps)
        if p.action_bound == "tanh":
            v = _mul(_c(0.5), _sub(_log1p(v), _log1p(Ev(-eps))))
        return v, Ev(np.zeros(E))
    z_eps = Ev(eps, 2 * U * np.abs(eps))
    logits = Ev(o[:, :A])
    if p.head == "det" or p.bounded:
        mu = _mul(_c(p.max_action), _tanh(logits))
    else:
        mu = logits
    if p.head == "indep":
        sig = _exp(Ev(np.broadcast_to(log_sigma, (E, A))))
    elif p.head == "cond":
        sig = _exp(Ev(np.clip(o[:, A:2 * A], np.float32(SIGMA_MIN), np.float32(SIGMA_MAX))))
    if p.mode == "eval" or p.head == "det":
        act = mu
    else:
        act = _fma(sig, z_eps, mu)
    acts, lp = [act[:, j] for j in range(A)], Ev(np.zeros(E))
    for j in range(A):
        if p.head == "det":
            break
        if p.head == "cond":
            z = Ev(np.zeros(E)) if p.mode == "eval" else z_eps[:, j]
        else:
            z = _div(_sub(act[:, j], mu[:, j]), sig[:, j])
        lp = _add(lp, _sub(_sub(_mul(_mul(_c(-0.5), z), z), _log(sig[:, j])), _c(LOG_SQRT_2PI)))
        if p.head == "cond":
            sq = _tanh(act[:, j])
            lp = _sub(lp, _log(_add(_sub(_c(1.0), _mul(sq, sq)), _c(np.finfo(np.float32).eps))))
            acts[j] = sq
    if p.head == "det" and p.mode == "train" and p.expl_sigma > 0:
        acts = [_fma(_c(p.expl_sigma), z_eps[:, j], acts[j]) for j in range(A)]
    return Ev(np.stack([a.v for a in acts], 1), np.stack([a.e for a in acts], 1)), lp


C_CASES = [(2, 128), (2, 64), (4, 128), (4, 512)]     # (kind, H): A = 2 and A = 8


@pytest.mark.gpu
@pytest.mark.parametrize("kind,H", C_CASES, ids=[f"{TASKS[k].split('-')[0][6:]}-H{H}" for k, H in C_CASES])
def test_rollout_epilogue_per_head_and_mode(kind, H):
    from fsrl_b200.envs import env_dims
    from oracle.philox import action_noise, action_uniform
    D, A, _, _ = env_dims(kind)
    E = 3 * _tile_rows(H) + 5
    n = 3
    venv, buf = _rig(kind, E, seed=11 + H)
    # one actor per head shape; the conditioned sigma logits straddle both ends of [SIGMA_MIN, SIGMA_MAX]
    indep = _actor(D, H, [A], n_extra=A, seed=H)
    indep[1].extra.data.copy_(torch.linspace(-1.2, 0.4, A))
    cond = _actor(D, H, [A, A], seed=H + 1)
    bias = [-20.3, 2.3] if A == 2 else [-24.0, -20.4, -19.6, -2.0, 0.0, 1.6, 2.4, 6.0]
    cond[1].heads[1].bias.data.copy_(torch.tensor(bias))
    det = _actor(D, H, [A], seed=H + 2)
    nets = {"indep": indep, "cond": cond, "det": det}
    variants = [(h, m, b, s) for m in ("train", "eval")
                for h, b, s in (("indep", False, 0.0), ("indep", True, 0.0), ("cond", False, 0.0),
                                ("cond", True, 0.0), ("det", True, 0.0), ("det", True, 0.1))]
    variants += [("indep", "random", False, 0.0)] * 3
    maps = (("clip", True), ("tanh", False), ("", True), ("tanh", True), ("", False), ("clip", False))
    rep = Report(f"rollout epilogue H={H} {TASKS[kind]} A={A} E={E}", 1.0)
    ctr0 = (torch.arange(E, dtype=torch.int32, device="cuda") * 5 + 1000)
    for i, (head, mode, bounded, expl) in enumerate(variants):
        bound, scaling = maps[i % len(maps)]
        if mode == "random":
            bound = ("clip", "tanh", "")[i % 3]
        arena, slot = nets[head]
        p = _Policy(arena, slot, head, mode, bounded=bounded, max_action=1.5, action_bound=bound,
                    action_scaling=scaling, expl_sigma=expl, seed=1234 + i)
        col = _collector(p, venv, buf)
        venv.act_ctr.copy_(ctr0)
        _run_steps(col, E, n)
        moved = n if mode != "eval" else 0
        assert torch.equal(venv.act_ctr, ctr0 + moved), f"{head} {mode}: act_ctr"
        log_sigma = slot.extra.detach().cpu().numpy() if head == "indep" else None
        tag = f"{head}{'-bounded' if bounded and head != 'det' else ''}{f'-expl{expl}' if expl else ''}-{mode}" + \
            (f"-{bound or 'none'}" if mode == "random" else "")
        for t in range(n):
            rows = _slots(buf, E, t).long()
            o = _head_out(arena, slot, buf, E, t).cpu().numpy()
            ids = np.arange(E)
            ctr = ctr0.cpu().numpy().astype(np.uint32) + np.uint32(t if mode != "eval" else 0)
            if mode == "random":
                eps = action_uniform(p.seed, ids, ctr, A)
            elif mode == "train":
                eps = action_noise(p.seed, ids, ctr, A)
            else:
                eps = np.zeros((E, A), np.float32)
            act, lp = _epilogue64(o, eps, p, log_sigma)
            rep.close(f"{tag}:act", buf.act[rows], act.v, act.e)
            rep.close(f"{tag}:logp", buf.logp[rows], lp.v, lp.e)
        if head == "indep" and mode == "eval" and not bounded:
            assert torch.equal(_bits(buf.act[_slots(buf, E, 0).long()]), _bits(_head_out(arena, slot, buf, E, 0)))
    rep.show()
    # the clamp was hit on both sides
    o = _head_out(*cond, buf, E, 0).cpu().numpy()[:, A:]
    assert (o < -20).any() and (o > 2).any() and ((o > -20) & (o < 2)).any()


# ---- D. bookkeeping at scale (exact integers) ----------------------------------------------------------------
@pytest.mark.gpu
def test_inline_collect_with_idle_tiles():
    """n_episode = 100 of 4096 envs at H = 128 (R = 32): envs 0-99 run one episode each, tile 3 is
    partial and the other 124 tiles take the early-out"""
    kind, E, H, n_ep = 3, 4096, 128, 100
    from fsrl_b200.envs import env_dims
    D, A, _, T = env_dims(kind)
    arena, slot = _actor(D, H, [A], n_extra=A, seed=5)
    venv, buf = _rig(kind, E, cap_steps=T + 5, seed=21)
    col = _collector(_Policy(arena, slot, "indep", "train", seed=99), venv, buf)
    ctr0 = torch.arange(E, dtype=torch.int32, device="cuda") * 7 + 3
    venv.act_ctr.copy_(ctr0)
    floats = (buf.obs, buf.obs_next, buf.act, buf.rew, buf.cost, buf.logp)
    for t in floats:
        _bits(t).fill_(SENT)
    buf.terminated.fill_(0xA5)
    buf.truncated.fill_(0xA5)
    stats = col.collect(n_episode=n_ep)
    assert stats["n/ep"] == n_ep and stats["n/st"] == n_ep * T
    assert stats["truncated"] == 1.0 and stats["terminated"] == 0.0
    cap = buf.cap
    want = torch.zeros(E, dtype=torch.int32)
    want[:n_ep] = T
    assert torch.equal(buf.len.cpu(), want) and torch.equal(buf.ptr.cpu(), want)
    assert torch.equal(venv.act_ctr[:n_ep], ctr0[:n_ep] + T), "act_ctr of the active envs"
    assert torch.equal(venv.act_ctr[n_ep:], ctr0[n_ep:]), "act_ctr of idle envs changed"
    for t in floats:
        v = _bits(t).view(E, cap, -1)
        assert bool((v[:n_ep, :T] != SENT).all()), "a transition of an active env was not stored"
        assert bool((v[:n_ep, T:] == SENT).all()) and bool((v[n_ep:] == SENT).all()), "stored past the episodes"
    tr, te = buf.truncated.view(E, cap), buf.terminated.view(E, cap)
    assert bool((tr[:n_ep, :T - 1] == 0).all() and (tr[:n_ep, T - 1] == 1).all()), "truncation flags"
    assert bool((te[:n_ep, :T] == 0).all())
    assert bool((tr[:n_ep, T:] == 0xA5).all() and (tr[n_ep:] == 0xA5).all() and (te[n_ep:] == 0xA5).all())
    from oracle.envs import OracleVecEnv
    first = buf.obs.view(E, cap, D)[:n_ep, 0].cpu().numpy()
    assert _same_bits(first, OracleVecEnv(kind, E, venv.seed_value).reset()[:n_ep])


@pytest.mark.gpu
@pytest.mark.parametrize("E,surplus", [(1025, 1023), (1025, 1024), (2100, 1025), (2100, 2049), (3000, 1024),
                                       (3000, 2049)])
def test_general_collect_across_resolve_chunks(E, surplus):
    """n_episode = 2E - surplus > E: all E envs truncate together at T, the first `surplus` of them (in env
    order, across the resolve kernel's 1024-env chunks) retire and the others run a second episode"""
    from oracle import collector as ocol
    from oracle.envs import OracleVecEnv
    kind = 3
    n_ep = 2 * E - surplus
    from fsrl_b200.envs import env_dims
    D, A, _, T = env_dims(kind)
    arena, slot = _actor(D, 64, [A], n_extra=A, seed=6)
    venv, buf = _rig(kind, E, cap_steps=2 * T, seed=E + surplus)
    pol = _Policy(arena, slot, "indep", "random", seed=4321)
    col = _collector(pol, venv, buf)
    # a bounded number of steps, rather than collect()'s loop until finished: two episodes, then steps
    # that must do nothing
    _run_steps(col, n_ep, 2 * T + 3)
    st = venv.read_stats()
    assert st.finished == 1, f"not finished after {2 * T + 3} steps: {st.episode_count} of {n_ep} episodes"
    col.reset_env()                  # a collect ends by resetting every env
    stats = {"n/ep": st.episode_count, "n/st": st.step_count}
    oenv = OracleVecEnv(kind, E, venv.seed_value)
    oenv.reset()
    obuf = ocol.OracleBuffer(E * 2 * T, E, D, A)
    ctr = np.zeros(E, np.uint32)
    ost = ocol.collect(oenv, None, n_ep, pol.seed, ctr, obuf, mode="random")
    assert stats["n/ep"] == ost["n/ep"] == n_ep
    assert stats["n/st"] == ost["n/st"] == (2 * E - surplus) * T
    assert np.array_equal(buf.len.cpu().numpy(), obuf.len) and np.array_equal(buf.ptr.cpu().numpy(), obuf.ptr)
    assert np.array_equal(venv.ep_idx.cpu().numpy().astype(np.uint32), oenv.ep_idx)
    assert np.array_equal(venv.act_ctr.cpu().numpy().astype(np.uint32), ctr)
    for k in ("obs", "obs_next", "act", "rew", "cost"):
        assert _same_bits(getattr(buf, k).cpu().numpy(), getattr(obuf, k)), k
    assert np.array_equal(buf.truncated.cpu().numpy().astype(bool), obuf.truncated)
    assert np.array_equal(buf.terminated.cpu().numpy().astype(bool), obuf.terminated)


# ---- E. the oracle's random-mode actions (CPU) -----------------------------------------------------------------
@pytest.mark.parametrize("bound", ["clip", "tanh"])
def test_oracle_random_actions_follow_philox_chunks(bound):
    """random mode: action 4c + j of env e at counter k is usym(philox4x32(e, k, c, 0)[j]), and under the
    tanh bound the stored action is its atanh (rollout.cu, random mode)"""
    from oracle import collector as ocol
    from oracle.envs import OracleVecEnv
    from oracle.philox import KEY_ACT, philox4x32, usym
    kind, E, seed = 4, 3, 77                     # AntCircle: A = 8, two Philox draws per action
    oenv = OracleVecEnv(kind, E, 5)
    oenv.reset()
    T, A = oenv.T, oenv.A
    obuf = ocol.OracleBuffer(E * T, E, oenv.D, A)
    ctr0 = np.array([0, 9, 1000], np.uint32)
    ctr = ctr0.copy()
    ocol.collect(oenv, None, E, seed, ctr, obuf, mode="random", action_bound=bound)
    assert np.array_equal(ctr, ctr0 + np.uint32(T))
    for e in range(E):
        for t in (0, 1, T - 1):
            u = np.zeros(A, np.float32)
            for c in range(2):
                r = philox4x32(e, ctr0[e] + np.uint32(t), c, 0, seed, KEY_ACT)
                for j in range(4):
                    u[4 * c + j] = usym(r[j])
            assert not np.array_equal(u[:4], u[4:])
            if bound == "tanh":
                u = (np.float32(0.5) * (np.log1p(u) - np.log1p(-u))).astype(np.float32)
            assert _same_bits(obuf.act[e * obuf.cap + t], u), (e, t)
