"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol
include/fsrl_b200.h declares (no compute calls -- there is no GPU here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "fsrl_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fsrl_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from fsrl_b200 import _lib
    names = _declared()
    assert len(names) >= 5
    for n in names:
        assert hasattr(_lib.lib, n), f"libfsrl_b200.so does not export {n}"
        assert n in _lib.SIGNATURES, f"{n} declared in the header but not bound in _lib.SIGNATURES"
    for n in _lib.SIGNATURES:
        assert n in names, f"{n} bound in python but not declared in include/fsrl_b200.h"


def test_abi_version_2_and_error_text():
    """Version 2: fsrl_ppo_update_t no longer carries `mask` and `head_indep`, so a binding built against version 1
    would misread every field after `stats`."""
    from fsrl_b200 import _lib
    assert _lib.lib.fsrl_abi_version() == 2
    assert isinstance(_lib.last_error(), str)


def test_argument_validation_needs_no_gpu():
    """EINVAL paths return before touching the device."""
    from fsrl_b200 import _lib
    rc = _lib.lib.fsrl_gae_dual(None, None, None, None, None, None, 0.99, 0.95, None, None,
                                -1, 0, 2, None, 0, None)
    assert rc == _lib.FSRL_EINVAL and "N must be" in _lib.last_error()
    rc = _lib.lib.fsrl_gae_dual(None, None, None, None, None, None, 0.99, 1.5, None, None,
                                8, 8, 2, None, 0, None)
    assert rc == _lib.FSRL_EINVAL and "GAE lambda should be in [0, 1]." in _lib.last_error()
    with pytest.raises(ValueError):
        _lib.check(rc)
    assert _lib.lib.fsrl_gae_dual_workspace_bytes(614400) > 0


def test_ppo_epoch_requires_gather_and_barrier():
    """The PPO epoch driver always gathers the permuted batch and always resets the grid barrier's ticket counter:
    a descriptor without either buffer is rejected before anything is enqueued (the pointers below are never
    dereferenced)."""
    from fsrl_b200 import _lib
    fake = 1 << 20
    u = _lib.PpoUpdate()
    for f in ("theta", "grad", "adam_m", "adam_v", "w2n", "scratch", "norm_sq", "stats",
              "obs", "act", "logp_old", "adv", "ret", "perm", "gather", "barrier"):
        setattr(u, f, fake)
    u.n_nets, u.D, u.H, u.A, u.C, u.actor_out, u.bmax = 3, 8, 256, 2, 2, 2, 1024
    for missing in ("gather", "barrier"):
        setattr(u, missing, None)
        rc = _lib.lib.fsrl_ppo_lag_epoch(u, 1024, 256, 0, 0, None, None)
        assert rc == _lib.FSRL_EINVAL and "gather or barrier" in _lib.last_error()
        setattr(u, missing, fake)


def test_ops_refuse_cpu_tensors():
    import torch
    from fsrl_b200 import ops
    x = torch.zeros(2, 8)
    with pytest.raises(TypeError, match="CUDA tensor"):
        ops.gae_dual(x, x, x[0], x[0], torch.zeros(8, dtype=torch.uint8), None, 0.99, 0.95)


def test_header_is_plain_c99(tmp_path):
    """The drop-in boundary is a C ABI: include/fsrl_b200.h must compile as C99 (no C++, no torch types) and the
    struct sizes a C compiler sees must be the ones the CUDA build reports (what a cgo / JNI / ctypes binding
    relies on)."""
    import shutil
    import subprocess
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "abi.c"
    src.write_text('#include <stdio.h>\n#include "fsrl_b200.h"\n'
                   'int main(void){ printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(fsrl_mlp3_t), '
                   'sizeof(fsrl_collect_stats_t), sizeof(fsrl_rollout_t), sizeof(fsrl_ppo_update_t), sizeof(fsrl_netref_t), '
                   'sizeof(fsrl_netlist_t), sizeof(fsrl_engine_t), sizeof(fsrl_eng_input_t), sizeof(fsrl_offpolicy_t), '
                   'sizeof(fsrl_cpo_t)); return 0; }\n')
    exe = tmp_path / "abi"
    subprocess.check_call([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(root, "include"),
                           "-o", str(exe), str(src)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    from fsrl_b200 import _lib
    assert sizes == [int(_lib.lib.fsrl_abi_sizeof(i)) for i in range(10)]


def test_persistent_exchange_buffers_fit_the_peer_block():
    """Host-side sizing of the persistent PPO launch (no device call): the packet regions of the data-parallel exchange
    (8 source-rank regions + 1 result region per parity, DESIGN.md 6) must fit the peer block `parallel.enable_p2p` is
    willing to allocate, and the workspace must grow with the number of networks."""
    from fsrl_b200 import _lib
    lib = _lib.lib
    sizes = [int(lib.fsrl_ppo_persist_p2p_floats(n)) for n in (1, 2, 3)]
    assert sizes[0] < sizes[1] < sizes[2]
    assert sizes[2] <= 4096 * 1024                      # the bound enable_p2p applies to one parity buffer
    per_net = sizes[1] - sizes[0]
    assert per_net % 9 == 0 and sizes[2] - sizes[1] == per_net
    stride = int(lib.fsrl_p2p_stride(sizes[2]))
    assert stride >= sizes[2] and stride % 64 == 0
    assert int(lib.fsrl_p2p_block_bytes(sizes[2])) >= 2 * 4 * stride
    ws = [int(lib.fsrl_ppo_persist_ws_floats(n, 8, 256)) for n in (1, 2, 3)]
    assert ws[0] < ws[1] < ws[2] and ws[2] - ws[1] == ws[1] - ws[0]
