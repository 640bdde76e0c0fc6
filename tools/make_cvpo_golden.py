"""Fixtures of CVPO's host surface, produced by the reference's own classes (on CPU, through the same tianshou /
gymnasium shims as oracle/make_golden_policies.py):

    python tools/make_cvpo_golden.py

writes tests/golden/cvpo_host_golden.json -- the CVPO / CVPOAgent signatures, the public attributes of a CVPO
instance after pre_update_fn, the state_dict keys and shapes with single and double critics, and the nine
cvpo_cfg dataclasses -- and tests/golden/cvpo_agent_init_golden.npz, the seeded initial parameters of CVPOAgent
for conditioned / state-independent sigma, bounded / unbounded means and single / double critics."""
from __future__ import annotations

import dataclasses
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_policies as mg  # noqa: E402

AGENT_CASES = {
    "cond_bounded_single": dict(),
    "cond_unbounded_double": dict(unbounded=True, double_critic=True),
    "indep_bounded_double": dict(conditioned_sigma=False, double_critic=True),
    "indep_unbounded_single": dict(conditioned_sigma=False, unbounded=True),
    "cond_bounded_scaled": dict(last_layer_scale=True),
}


def _env():
    act_space, obs_space = mg._space()
    return types.SimpleNamespace(observation_space=obs_space, action_space=act_space,
                                 spec=types.SimpleNamespace(max_episode_steps=300))


def main():
    mg._bootstrap()
    from fsrl.agent import CVPOAgent
    from fsrl.config import cvpo_cfg
    from fsrl.policy import CVPO
    from fsrl.utils import BaseLogger
    import inspect

    def sig(fn):
        out = []
        for name, p in inspect.signature(fn).parameters.items():
            if name == "self":
                continue
            d = p.default
            if d is inspect.Parameter.empty:
                rep = "<required>"
            elif isinstance(d, (int, float, str, bool, tuple, list, type(None))):
                rep = repr(d)
            else:
                rep = "<object:%s>" % type(d).__name__
            out.append([name, str(p.kind), rep])
        return out

    rec = {"signatures": {"CVPO.__init__": sig(CVPO.__init__), "CVPOAgent.__init__": sig(CVPOAgent.__init__),
                          "CVPO.forward": sig(CVPO.forward)}}
    rec["state_dict"], inits = {}, {}
    for name, double in (("single", False), ("double", True)):
        agent = CVPOAgent(_env(), logger=BaseLogger(), device="cpu", seed=7, hidden_sizes=(mg.H, mg.H),
                          double_critic=double)
        sd = agent.policy.state_dict()
        rec["state_dict"][name] = {"keys": {k: (list(v.shape) if torch.is_tensor(v) else "object") for k, v in sd.items()}}
        if name == "single":
            pol = agent.policy
            pol.pre_update_fn()
            rec["public_attrs"] = sorted(n for n in dir(pol) if not n.startswith("_"))
    rec["cvpo_cfg"] = {}
    for cn in ("TrainCfg", "Bullet1MCfg", "Bullet5MCfg", "Bullet10MCfg", "MujocoBaseCfg", "Mujoco2MCfg", "Mujoco5MCfg",
               "Mujoco20MCfg", "Mujoco10MCfg"):
        cls = getattr(cvpo_cfg, cn)
        rec["cvpo_cfg"][cn] = [[f.name, repr(getattr(cls(), f.name))] for f in dataclasses.fields(cls)]
    for name, kw in AGENT_CASES.items():
        agent = CVPOAgent(_env(), logger=BaseLogger(), device="cpu", seed=7, hidden_sizes=(mg.H, mg.H), **kw)
        for k, v in agent.policy.state_dict().items():
            if torch.is_tensor(v):
                inits[f"{name}|{k}"] = v.detach().numpy().copy()
    path = os.path.join(mg.OUT, "cvpo_host_golden.json")
    with open(path, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(mg.OUT, "cvpo_agent_init_golden.npz"), **inits)
    print("wrote", path, "and cvpo_agent_init_golden.npz", len(inits), "arrays")


if __name__ == "__main__":
    main()
