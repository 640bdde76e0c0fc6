"""CPU-side checks of the gym-protocol entry points and of FastCollector's choice of collect path: every refusal
here happens before anything touches a device (the descriptor's state pointers are never dereferenced)."""
import ctypes

import numpy as np
import pytest
import torch

FAKE = 1 << 20


def _descriptor(E=8, kind=0):
    from fsrl_b200 import _lib
    r = _lib.Rollout()
    r.kind, r.E, r.max_steps = kind, E, 300
    for f in ("env_state", "obs_cur", "env_t", "ep_idx", "act_ctr", "active", "done_now", "ep_rew", "ep_len", "stats"):
        setattr(r, f, FAKE)
    return r


def _ids(*v):
    return np.asarray(v, np.int32)


def _step(r, ids, n, act=FAKE, out=FAKE):
    from fsrl_b200 import _lib
    p = None if ids is None else ids.ctypes.data
    return _lib.lib.fsrl_env_step(ctypes.byref(r), act, p, n, out, out, out, out, out, None)


def _reset(r, ids, n):
    from fsrl_b200 import _lib
    p = None if ids is None else ids.ctypes.data
    return _lib.lib.fsrl_env_reset_ids(ctypes.byref(r), p, n, FAKE, None)


@pytest.mark.parametrize("call", [_step, _reset])
def test_bad_n_and_ids_are_rejected(call):
    from fsrl_b200 import _lib
    r = _descriptor()
    for ids, n, msg in [(None, 0, "outside [1, E = 8]"), (None, 9, "outside [1, E = 8]"),
                        (None, 4, "without ids, n must be E"), (_ids(1, 8), 2, "ids[1] = 8 outside"),
                        (_ids(-1), 1, "ids[0] = -1 outside"), (_ids(0, 1, 2), 0, "outside [1, E = 8]")]:
        assert call(r, ids, n) == _lib.FSRL_EINVAL, (ids, n)
        assert msg in _lib.last_error(), (msg, _lib.last_error())


def test_null_pointers_are_rejected():
    from fsrl_b200 import _lib
    r = _descriptor()
    assert _step(r, _ids(0, 1), 2, act=None) == _lib.FSRL_EINVAL and "null action or output" in _lib.last_error()
    assert _step(r, _ids(0, 1), 2, out=None) == _lib.FSRL_EINVAL and "null action or output" in _lib.last_error()
    assert _lib.lib.fsrl_rollout_steps_act(ctypes.byref(r), None, None) == _lib.FSRL_EINVAL
    assert "null action array" in _lib.last_error()
    assert _lib.lib.fsrl_rollout_steps_act(None, FAKE, None) == _lib.FSRL_EINVAL
    r.ep_rew = None
    assert _step(r, _ids(0), 1) == _lib.FSRL_EINVAL and "null state pointer" in _lib.last_error()
    assert _reset(r, _ids(0), 1) == _lib.FSRL_EINVAL
    r = _descriptor(kind=9)
    assert _reset(r, None, 8) == _lib.FSRL_EINVAL and "unknown env kind" in _lib.last_error()


def test_step_refuses_wrong_shapes_and_ids():
    from fsrl_b200.envs import DeviceVectorEnv
    venv = DeviceVectorEnv("SafetyCarCircle-v0", 4, device="cpu")
    for act, id in [(np.zeros((3, 2)), None), (np.zeros((4, 3)), None), (np.zeros(8), None),
                    (np.zeros((2, 2)), [0, 1, 2]), (np.zeros((4, 2)), [[0, 1], [2, 3]]),
                    (np.zeros((1, 2)), [0.5]), (np.zeros((0, 2)), [])]:
        with pytest.raises(ValueError):
            venv.step(act, id)
    with pytest.raises(ValueError, match="env ids"):
        venv.reset(np.zeros((2, 2), np.int64))
    with pytest.raises(ValueError, match="env ids"):          # ids= is the same argument as id
        venv.reset(ids=np.zeros((2, 2), np.int64))
    with pytest.raises(TypeError, match="both id and ids"):
        venv.reset([0], ids=[1])
    with pytest.raises(RuntimeError, match="CUDA devices only"):   # a well-formed call still needs the GPU
        venv.step(np.zeros((2, 2), np.float32), [1, 3])


def _policies():
    from fsrl_b200 import envs, nets
    from fsrl_b200.data import Batch
    from fsrl_b200.policy.base_policy import BasePolicy
    env = envs.make("SafetyCarCircle-v0")
    D, A = env.observation_space.shape[0], env.action_space.shape[0]

    class Plain(BasePolicy):
        def learn(self, batch, **kw):
            return {}

    class OwnForward(Plain):
        def forward(self, batch, state=None, **kw):
            return Batch(act=batch.obs[:, :A])

    class OwnBoth(OwnForward):
        def fill_rollout(self, r, exploration_noise=False):
            pass

    def actor(hidden):
        return nets.ActorProb(nets.Net(D, hidden_sizes=hidden), A)

    kw = dict(observation_space=env.observation_space, action_space=env.action_space)
    critic = nets.Critic(nets.Net(D, hidden_sizes=(64, 64)))
    return dict(
        arena_actor=(Plain(actor((64, 64)), critic, **kw), True),
        own_forward=(OwnForward(actor((64, 64)), critic, **kw), False),
        own_forward_and_fill=(OwnBoth(actor((64, 64)), critic, **kw), True),
        three_layers=(Plain(actor((64, 64, 64)), critic, **kw), False),
        unequal_widths=(Plain(actor((64, 128)), critic, **kw), False),
        three_layer_critic=(Plain(actor((64, 64)), nets.Critic(nets.Net(D, hidden_sizes=(64, 64, 64))), **kw), False),
        torch_module=(torch.nn.Linear(D, A), False),
    )


def test_collect_path_is_chosen_from_the_policy():
    from fsrl_b200.data.fast_collector import _fused_policy

    class FillOnly:
        def fill_rollout(self, r, exploration_noise=False):
            pass

    assert _fused_policy(FillOnly())
    for name, (policy, fused) in _policies().items():
        assert _fused_policy(policy) is fused, name


@pytest.mark.parametrize("name", ["three_layers", "unequal_widths"])
def test_builtin_forward_runs_an_actor_the_arena_cannot_hold(name):
    """BasePolicy.forward with a non-arena actor is the reference's forward on the module itself (no arena, no
    device needed): the bounded mean in eval mode, a sample around it in train mode."""
    from fsrl_b200.data import Batch
    policy, _ = _policies()[name]
    obs = torch.randn(5, 8, generator=torch.Generator().manual_seed(0))
    policy.eval()
    with torch.no_grad():
        (mu, sigma), _ = policy.actor(obs)
        out = policy(Batch(obs=obs))
        assert torch.equal(out.act, mu) and torch.equal(out.logits[1], sigma)
        policy.train()
        torch.manual_seed(1)
        act = policy(Batch(obs=obs)).act
        torch.manual_seed(1)
        assert torch.equal(act, mu + sigma * torch.randn_like(mu))
    assert policy._arena is None
