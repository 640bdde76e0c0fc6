"""Record the digests tests/test_ppo_persist_golden_gpu.py compares with: one repeat of the persistent PPO launch at
D = 8 and D = 40 on synthetic inputs, sha256 of the parameters and Adam moments as int32.
Usage: python tools/persist_golden.py [OUT.json]   (default: tests/golden/ppo_persist_golden.json)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_ppo_persist_golden_gpu import GOLDEN, SHAPES, run_repeat  # noqa: E402

out = {}
for D in sorted(SHAPES):
    active, digests = run_repeat(D)
    assert active, "the persistent launch does not take D = %d" % D
    out["D%d" % D] = digests
    print("D = %d:" % D, digests)
with open(sys.argv[1] if len(sys.argv) > 1 else GOLDEN, "w") as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write("\n")
