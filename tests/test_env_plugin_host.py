"""The env plugin tool without a GPU: building, caching, compile errors, the limits, and the task registry's
refusals (nvcc cross-compiles; loading a plugin and reading its table needs no device)."""
import os
import shutil
import subprocess
import sys

import pytest

from env_plugin_twin import ENV_DIR, PLUGIN_DIR, ROOT, header

GOOD = '''#include "envs.cuh"
struct UserEnv {
    static constexpr int D = %(D)d, A = %(A)d, S = %(S)d, T = 50;
    __device__ static void reset(float* st, uint32_t, uint32_t, uint32_t) {
        for (int i = 0; i < S; ++i) st[i] = 0.0f;
    }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) {
        for (int k = 0; k < D; ++k) o[k] = st[k %% S];
    }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t, float& rew, float& cost,
                                bool& term) {
        st[0] = fsrl::xa(st[0], a[0]);
        rew = st[0]; cost = 0.0f; term = false;
    }
};
'''


def _write(tmp_path, name, text):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def test_build_loads_and_reports_dims():
    """The test env's plugin (build() made it; the tool returns the cached file without compiling) loads and
    reports its widths and horizon."""
    from fsrl_b200 import envs
    path = envs.build_device_env(header("hazard_dash"), out=PLUGIN_DIR)
    assert os.path.dirname(path) == PLUGIN_DIR and path.endswith(".so")
    assert envs.plugin_dims(path) == (19, 3, 32, 200)
    assert envs.plugin_dims(envs.plugin_path(header("car_button1"), PLUGIN_DIR)) == (76, 2, 12, 1000)


def test_cache_hit_and_changed_header(tmp_path):
    from fsrl_b200 import envs
    hdr = _write(tmp_path, "tiny.h", GOOD % dict(D=5, A=1, S=3))
    out = str(tmp_path / "plugins")
    p1 = envs.build_device_env(hdr, out=out)
    assert envs.plugin_dims(p1) == (5, 1, 3, 50)
    mtime = os.stat(p1).st_mtime_ns
    assert envs.build_device_env(hdr, out=out) == p1 and os.stat(p1).st_mtime_ns == mtime
    with open(hdr, "a") as f:
        f.write("// changed\n")
    p2 = envs.build_device_env(hdr, out=out)
    assert p2 != p1 and os.path.exists(p1) and envs.plugin_dims(p2) == (5, 1, 3, 50)
    assert os.path.exists(p2 + ".ptxas.log")
    assert sorted(f for f in os.listdir(out) if f.endswith(".so")) == sorted(os.path.basename(p) for p in (p1, p2))


def test_command_line_builds_the_same_path(tmp_path):
    from fsrl_b200 import envs
    out = subprocess.run([sys.executable, "-m", "fsrl_b200.envs", "build", header("hazard_dash"), "--out", PLUGIN_DIR],
                         cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip().splitlines()[-1] == envs.plugin_path(header("hazard_dash"), PLUGIN_DIR)


def test_syntax_error_reports_the_header_line(tmp_path):
    from fsrl_b200 import envs
    text = GOOD % dict(D=5, A=1, S=3)
    lines = text.splitlines()
    assert "st[i] = 0.0f;" in lines[4]
    lines[4] = lines[4].replace("st[i] = 0.0f;", "st[i] = 0.0f")      # line 5 of the header
    hdr = _write(tmp_path, "broken.h", "\n".join(lines) + "\n")
    with pytest.raises(envs.EnvBuildError) as e:
        envs.build_device_env(hdr, out=str(tmp_path / "plugins"))
    assert "broken.h(5)" in str(e.value) or "broken.h(6)" in str(e.value), str(e.value)
    assert not [f for f in os.listdir(tmp_path / "plugins") if f.endswith(".so")]


@pytest.mark.parametrize("dims,limit", [(dict(D=5, A=9, S=3), "1 <= A <= ENV_MAX_A (8)"),
                                        (dict(D=72, A=9, S=3), "1 <= A <= ENV_MAX_A (8)"),
                                        (dict(D=73, A=8, S=3), "D + A <= FSRL_ENG_DX_LD (80)"),
                                        (dict(D=5, A=2, S=33), "1 <= S <= ENV_MAX_S (32)")])
def test_limits_raise_value_error(tmp_path, dims, limit):
    from fsrl_b200 import envs
    hdr = _write(tmp_path, "big.h", GOOD % dims)
    with pytest.raises(ValueError, match=limit.replace("(", r"\(").replace(")", r"\)").replace("+", r"\+")):
        envs.build_device_env(hdr, out=str(tmp_path / "plugins"))


def test_registry_refusals():
    from fsrl_b200 import envs
    path = envs.plugin_path(header("car_circle"), PLUGIN_DIR)
    with pytest.raises(ValueError, match="built-in task"):
        envs.register_device_env("SafetyCarCircle-v0", path)
    with pytest.raises(KeyError, match="unknown task"):
        envs.DeviceEnv("NotRegistered-v0")
    with pytest.raises(ValueError, match="unknown env kind 100"):
        envs.env_dims(100)


def test_headers_shipped_with_the_tests():
    assert sorted(f for f in os.listdir(ENV_DIR) if f.endswith(".h")) == \
        ["car_button1.h", "car_circle.h", "drone_circle.h", "hazard_dash.h"]
    assert shutil.which("make")
