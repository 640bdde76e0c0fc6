"""Rendering user-defined device envs without a GPU: which plugins export a renderer, the drawing contract's compile
error, the refusals of fsrl_env_register_renderer, and the float32 twins of the drawn test scenes on hand-made
states (nvcc cross-compiles; loading a plugin and registering it needs no device)."""
import ctypes
import os

import numpy as np
import pytest

import render_plugin_twin as rpt
import render_twin as rt
from env_plugin_twin import PLUGIN_DIR
from env_plugin_twin import header as env_header

DRAWN = ("car_circle_drawn", "crowded", "hazard_dash_drawn")
UNDRAWN = ("car_button1", "car_circle", "drone_circle", "hazard_dash")

WRONG_DRAW = '''#include "envs.cuh"
#include "render.cuh"
struct UserEnv {
    static constexpr int D = 1, A = 1, S = 1, T = 10;
    __device__ static void reset(float* st, uint32_t, uint32_t, uint32_t) { st[0] = 0.0f; }
    __device__ static void observe(const float* st, float* o, uint32_t, uint32_t, uint32_t) { o[0] = st[0]; }
    __device__ static void step(float* st, const float* a, uint32_t, uint32_t, uint32_t, float& rew, float& cost,
                                bool& term) {
        st[0] = a[0]; rew = 0.0f; cost = 0.0f; term = false;
    }
    __device__ static void draw(const float* st, fsrl::render::Builder& b) { b.disc(st[0], 0.0f, 0.1f, 1); }
};
'''


def _path(name):
    from fsrl_b200 import envs
    hdr = rpt.header(name) if name in DRAWN else env_header(name)
    path = envs.plugin_path(hdr, PLUGIN_DIR)
    assert os.path.exists(path), f"{path} is missing: build() builds the test env plugins"
    return path


@pytest.mark.parametrize("name", DRAWN + UNDRAWN)
def test_plugins_export_a_renderer_exactly_when_the_struct_draws(name):
    from fsrl_b200 import _lib, envs
    so, _ = envs._load_plugin(_path(name))
    table = envs._plugin_renderer(so)
    if name in DRAWN:
        assert table is not None
        assert table.contents.abi_version == _lib.lib.fsrl_abi_version() and table.contents.render
    else:
        assert table is None


def test_draw_with_the_wrong_signature_names_the_contract(tmp_path):
    from fsrl_b200 import envs
    hdr = tmp_path / "wrong_draw.h"
    hdr.write_text(WRONG_DRAW)
    with pytest.raises(ValueError, match="env plugin contract:") as e:
        envs.build_device_env(str(hdr), out=str(tmp_path / "plugins"))
    assert "draw(const float* st" in str(e.value)
    assert not [f for f in os.listdir(tmp_path / "plugins") if f.endswith(".so")]


def test_register_renderer_refusals():
    from fsrl_b200 import _lib, envs
    reg = _lib.lib.fsrl_env_register_renderer
    so, _ = envs._load_plugin(_path("crowded"))
    good = envs._plugin_renderer(so).contents

    def refused(kind, table, text):
        assert reg(kind, table) == _lib.FSRL_EINVAL
        assert text in _lib.last_error()

    task = "RenderHostCrowded-v0"
    kind = envs.register_device_env(task, _path("crowded"))
    assert envs.PLUGINS[task].renders
    refused(kind, None, "null table")
    no_launcher = _lib.EnvRenderer(good.abi_version, 0, None)
    refused(kind, ctypes.byref(no_launcher), "null table or launcher")
    foreign = _lib.EnvRenderer.from_buffer_copy(good)
    foreign.abi_version = good.abi_version + 1
    refused(kind, ctypes.byref(foreign), "ABI version")
    for k in (0, 5, 37, 63, 127, 128, -1):        # built-in, unregistered and outside the plugin range
        refused(k, ctypes.byref(good), "not a registered plugin kind")
    refused(kind, ctypes.byref(good), "already has a renderer")
    # an undrawn plugin registers without a renderer
    plain = envs.register_device_env("RenderHostCarCircle-v0", _path("car_circle"))
    assert not envs.PLUGINS["RenderHostCarCircle-v0"].renders and plain != kind
    with pytest.raises(ValueError, match="no renderer"):
        envs.DeviceVectorEnv("RenderHostCarCircle-v0", 2, device="cpu", render_mode="rgb_array")


def _hazard_state():
    st = np.zeros(32, np.float32)
    st[0:4] = (-0.5, 0.0, 0.3, 0.4)          # robot at (-0.5, 0) with velocity (0.3, 0.4)
    st[4:6] = (1.0, 1.0)                     # goal
    st[6] = 0.5                              # energy: a quarter of the gauge's scale [0, 2]
    st[8:32] = 1.9                           # every hazard in the corner ...
    st[8:10] = (-1.0, -1.0)                  # ... but the first
    return st


def test_hazard_dash_twin_scene():
    H = W = 128
    st = _hazard_state()
    sc = rpt.scene(rpt.hazard_dash_draw, st, 50, 200)
    assert len(sc.p) == 19 + 1 and sc.p[-1][1] == rt.C_MARK
    assert (sc.x0, sc.x1) == (np.float32(-2.2), np.float32(2.2))
    frame = rt.draw(sc, H, W)
    costed = rt.draw(rpt.scene(rpt.hazard_dash_draw, st, 50, 200, cost=True), H, W)

    def col(img, x, y):
        i, j = rpt.pixel(sc, x, y, H, W)
        return tuple(img[i, j])

    P = {c: tuple(rt.PALETTE[c]) for c in range(len(rt.PALETTE))}
    assert col(frame, 1.0, 1.0) == P[rt.C_GOAL]
    assert col(frame, -1.0, -1.0) == P[rt.C_HAZARD] and col(frame, 1.9, 1.9) == P[rt.C_HAZARD]
    assert col(frame, -1.0, -1.4) == P[rt.C_FLOOR]           # outside the hazard's radius 0.3
    assert col(frame, -0.5 - 0.08, 0.0) == P[rt.C_ROBOT] and col(costed, -0.5 - 0.08, 0.0) == P[rt.C_COST]
    assert col(frame, -0.5 + 0.8 * 0.15, 0.8 * 0.2) == P[rt.C_HEADING]   # the heading: 0.5 s of velocity
    assert col(frame, 2.15, 0.0) == P[rt.C_BG]                # outside the arena
    # the vertical energy gauge along the left edge: filled to a quarter of its length, then its background
    g0, g1 = sc.y0 + (sc.y1 - sc.y0) * np.float32(0.05), sc.y1 - (sc.y1 - sc.y0) * np.float32(0.05)
    gx = sc.x0 + (sc.x1 - sc.x0) * np.float32(0.05)
    assert col(frame, gx, g0 + 0.1 * (g1 - g0)) == P[rt.C_GAUGE]
    assert col(frame, gx, g0 + 0.4 * (g1 - g0)) == P[rt.C_GAUGE_BG]
    assert col(frame, gx, g0 + 0.5 * (g1 - g0)) == P[rt.C_MARK]


def test_crowded_twin_scene_default_window_and_cap():
    H = W = 128
    st = np.array([0.25], np.float32)
    sc = rpt.scene(rpt.crowded_draw, st, 10, 20)
    assert (sc.x0, sc.x1, sc.y0, sc.y1) == (-1, 1, -1, 1)
    assert len(sc.p) == rt.MAX_PRIM and len(sc.p) - 1 == rpt.DRAW_MAX
    frame = rt.draw(sc, H, W)
    costed = rt.draw(rpt.scene(rpt.crowded_draw, st, 10, 20, cost=True), H, W)
    P = {c: tuple(rt.PALETTE[c]) for c in range(len(rt.PALETTE))}
    for k in range(rpt.CROWDED_N):
        i, j = rpt.pixel(sc, rpt.crowded_x(k), 0.25, H, W)
        want = P[rt.C_BG] if k >= rpt.DRAW_MAX else P[rt.C_GOAL] if k % 2 else P[rt.C_HAZARD]
        assert tuple(frame[i, j]) == want, k
    i, j = rpt.pixel(sc, rpt.crowded_x(0), 0.25, H, W)
    assert tuple(costed[i, j]) == P[rt.C_COST]
    i, j = rpt.pixel(sc, -1.0 + 0.01, 1.0 - 0.005, H, W)      # the progress bar: half the width at t / T = 1/2
    assert tuple(frame[i, j]) == P[rt.C_MARK] and tuple(frame[i, W - 2]) == P[rt.C_BG]
