"""CVPO's host surface without a GPU: the reference's signatures, public attributes, state_dict keys, cvpo_cfg
dataclasses and seeded CVPOAgent parameters (tests/golden/cvpo_*_golden.*, written by tools/make_cvpo_golden.py
from the reference's own classes), the Philox twin of the update's sampling streams, the argument checks of
fsrl_cvpo_steps and the C size of fsrl_cvpo_t."""
import dataclasses
import json
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
KEY_CVPO = 0x4356504F     # csrc/cvpo.cu


def cvpo_noise(seed, rows, A, step, stream):
    """Standard normals of the CVPO update stream: Philox4x32-10 with key (seed, KEY_CVPO) at counter
    (row, step_lo, 8*step_hi + chunk, stream), Box-Muller pairs, chunk c -> action dims 4c..4c+3.
    stream 0: next action of the n-step target (row b); stream 1: E-step particle (row k*B + b)."""
    from oracle.philox import normal_pair, philox4x32
    out = np.zeros((rows, A), np.float32)
    r = np.arange(rows, dtype=np.uint32)
    for c in range((A + 3) // 4):
        x = philox4x32(r, np.uint32(step & 0xFFFFFFFF), np.uint32((step >> 32) * 8 + c), np.uint32(stream), seed, KEY_CVPO)
        n = list(normal_pair(x[0], x[1])) + list(normal_pair(x[2], x[3]))
        for j in range(4):
            if 4 * c + j < A:
                out[:, 4 * c + j] = n[j]
    return out


def _golden():
    return json.load(open(os.path.join(GOLDEN, "cvpo_host_golden.json")))


def _env():
    from fsrl_b200.spaces import Box
    return types.SimpleNamespace(observation_space=Box(low=-np.ones(8, np.float32) * 10, high=np.ones(8, np.float32) * 10),
                                 action_space=Box(low=-np.ones(2, np.float32), high=np.ones(2, np.float32)),
                                 spec=types.SimpleNamespace(max_episode_steps=300))


def _agent(monkeypatch, **kw):
    """CVPOAgent with the device arena patched out (parameters stay the torch modules' own)."""
    from fsrl_b200.policy.base_policy import BasePolicy
    from fsrl_b200.agent import CVPOAgent
    monkeypatch.setattr(BasePolicy, "_build_arena",
                        lambda self, device=None: setattr(self, "_arena", types.SimpleNamespace(device="cpu")) or self._arena)
    return CVPOAgent(_env(), seed=7, hidden_sizes=(16, 16), **kw)


def test_signatures_match_reference():
    from fsrl_b200.agent import CVPOAgent
    from fsrl_b200.policy import CVPO
    import inspect
    g = _golden()["signatures"]
    for key, fn in (("CVPO.__init__", CVPO.__init__), ("CVPOAgent.__init__", CVPOAgent.__init__),
                    ("CVPO.forward", CVPO.forward)):
        got = [[n, str(p.kind)] for n, p in inspect.signature(fn).parameters.items() if n != "self"]
        assert got == [[n, k] for n, k, _ in g[key]], key
        defaults = {n: d for n, _, d in g[key] if not d.startswith("<")}
        for n, p in inspect.signature(fn).parameters.items():
            if n in defaults and n not in ("device", "logger"):
                assert repr(p.default) == defaults[n], (key, n)


@pytest.mark.parametrize("case", ["single", "double"])
def test_state_dict_keys_match_reference(monkeypatch, case):
    agent = _agent(monkeypatch, double_critic=case == "double")
    sd = agent.policy.state_dict()
    want = _golden()["state_dict"][case]["keys"]
    got = {k: (list(v.shape) if torch.is_tensor(v) else "object") for k, v in sd.items()}
    assert got == want
    assert sd["_extra_state"] is None


def test_public_attributes_cover_reference():
    from fsrl_b200.policy import CVPO
    fused = {"critics_loss", "policy_loss"}        # one device launch chain does both
    missing = [n for n in _golden()["public_attrs"] if not hasattr(CVPO, n) and n not in fused
               and n not in ("device", "dtype", "actor", "actor_old", "critics", "critics_old", "actor_optim",
                             "critics_optim", "cost_limit", "qc_thres", "max_episode_steps", "tau", "logger",
                             "dist_fn", "critics_num", "training", "updating", "gradient_steps", "lr_scheduler",
                             "action_space", "observation_space", "action_type", "action_bound_method",
                             "action_scaling", "ret_rms")]
    assert not missing, missing


def test_cvpo_cfg_matches_reference():
    from fsrl_b200.config import cvpo_cfg
    want = _golden()["cvpo_cfg"]
    assert len(want) == 9
    for cn, fields in want.items():
        cls = getattr(cvpo_cfg, cn)
        got = [[f.name, repr(getattr(cls(), f.name))] for f in dataclasses.fields(cls)]
        assert got == fields, cn


def test_agent_initial_parameters_match_reference(monkeypatch):
    raw = np.load(os.path.join(GOLDEN, "cvpo_agent_init_golden.npz"))
    cases = {}
    for k in raw.files:
        c, key = k.split("|", 1)
        cases.setdefault(c, {})[key] = raw[k]
    kws = {"cond_bounded_single": dict(), "cond_unbounded_double": dict(unbounded=True, double_critic=True),
           "indep_bounded_double": dict(conditioned_sigma=False, double_critic=True),
           "indep_unbounded_single": dict(conditioned_sigma=False, unbounded=True),
           "cond_bounded_scaled": dict(last_layer_scale=True)}
    assert set(cases) == set(kws)
    for c, kw in kws.items():
        agent = _agent(monkeypatch, **kw)
        got = {k: v.detach().numpy() for k, v in agent.policy.state_dict().items() if torch.is_tensor(v)}
        assert set(got) == set(cases[c]), c
        for k, v in cases[c].items():
            np.testing.assert_array_equal(got[k], v, err_msg=f"{c} {k}")


def test_philox_twin_layout():
    """The twin draws exactly philox4x32 at the documented counters: rows are independent per stream and step,
    and chunk 1 (dims 4..7) is a different counter from chunk 0."""
    from oracle.philox import normal_pair, philox4x32
    a = cvpo_noise(5, 6, 8, (1 << 32) + 3, 1)
    x = philox4x32(np.array([4], np.uint32), np.uint32(3), np.uint32(8 + 1), np.uint32(1), 5, KEY_CVPO)
    n0, n1 = normal_pair(x[0], x[1])
    np.testing.assert_array_equal(a[4, 4:6], np.array([n0[0], n1[0]], np.float32))
    assert not np.array_equal(cvpo_noise(5, 6, 8, 3, 0), cvpo_noise(5, 6, 8, 3, 1))
    assert not np.array_equal(a[:, :4], a[:, 4:])


def _descriptor():
    from fsrl_b200 import _lib
    fake = 1 << 20
    d = _lib.Cvpo()
    d.off.eng.bmax = 1024
    d.off.D, d.off.A, d.off.C, d.off.n_step = 8, 2, 2, 2
    d.K, d.estep_iters, d.mstep_iters, d.cond_sigma = 16, 1, 1, 1
    for f in ("estep_state", "mstep_state", "particles", "part_idx", "mu_old", "std_old", "comb", "weights"):
        setattr(d, f, fake)
    return d


@pytest.mark.parametrize("field,value,msg", [
    ("world", 2, "single GPU"), ("C", 3, "critic streams"), ("A", 9, "action dim"), ("K", 128, "bmax"),
    ("estep_iters", 0, "estep_iter_num"), ("mstep_iters", 0, "mstep_iter_num"), ("use_alpha", 1, "entropy"),
    ("cond_sigma", 0, "log_sigma")])
def test_cvpo_steps_rejects_bad_arguments(field, value, msg):
    """Invalid descriptors are rejected before anything is enqueued (the fake pointers are never dereferenced)."""
    from fsrl_b200 import _lib
    d = _descriptor()
    setattr(d.off if field in ("world", "C", "A", "use_alpha") else d, field, value)
    rc = _lib.lib.fsrl_cvpo_steps(d, 1 << 20, 1, 64, 0, 0, 0, 1 << 20, None)
    assert rc == _lib.FSRL_EINVAL and msg in _lib.last_error(), _lib.last_error()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="needs a C compiler")
def test_descriptor_size_matches_c(tmp_path):
    from fsrl_b200 import _lib
    import ctypes
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include "fsrl_b200.h"\nint main(void){printf("%zu", sizeof(fsrl_cvpo_t));return 0;}\n')
    exe = tmp_path / "s"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    size = int(subprocess.check_output([str(exe)]))
    assert size == _lib.lib.fsrl_abi_sizeof(10) == ctypes.sizeof(_lib.Cvpo)
    assert _lib.lib.fsrl_abi_version() == 2
