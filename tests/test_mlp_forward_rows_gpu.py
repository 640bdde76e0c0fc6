"""fsrl_mlp_forward's 64-row persistent kernel (H = 128 and 256) against the 16/32-row kernel it replaces there
(FSRL_MLPFWD_TILED=1), bit for bit: every output element is computed by the same operation sequence in both.

Widths, input and output dims, row counts that straddle the 64-row tile and the persistent grid (132 CTAs x 64 rows
on an H100 at H = 256), and the whole c2 critic pass (614 400 rows), with and without an index gather.  An input
too wide for a 64-row tile falls back to the 16-row kernel.  Rows past n_rows keep a NaN sentinel in both kernels.
"""
import ctypes

import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

SENT = 0x7FC0DEAD              # quiet-NaN bit pattern for memory a kernel must not write


def _net(D, H, out, seed):
    from fsrl_b200.nets import Arena, NetSlot
    gen = torch.Generator().manual_seed(seed)

    def lin(i, o):
        m = nn.Linear(i, o)
        with torch.no_grad():
            m.weight.copy_(torch.randn(o, i, generator=gen) * (2.0 / i) ** 0.5)
            m.bias.copy_(0.1 * torch.randn(o, generator=gen))
        return m

    slot = NetSlot("critic", None, lin(D, H), lin(H, H), [lin(H, out)], None)
    return Arena([slot], "cuda"), slot


def _forward(arena, slot, x, idx, n_rows, tiled, monkeypatch):
    from fsrl_b200 import _lib
    if tiled:
        monkeypatch.setenv("FSRL_MLPFWD_TILED", "1")
    else:
        monkeypatch.delenv("FSRL_MLPFWD_TILED", raising=False)
    y = torch.empty(n_rows + 67, slot.out, dtype=torch.float32, device="cuda")
    y.view(torch.int32).fill_(SENT)
    m = arena.mlp3(slot)
    _lib.check(_lib.lib.fsrl_mlp_forward(ctypes.byref(m), x.data_ptr(), None if idx is None else idx.data_ptr(),
                                         n_rows, y.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return y.view(torch.int32)


def _check(H, D, out, n_rows, gather, monkeypatch, seed=0):
    arena, slot = _net(D, H, out, seed)
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    n_src = n_rows + 5 if gather else n_rows
    x = torch.randn(n_src, D, generator=gen, device="cuda")
    idx = torch.randint(0, n_src, (n_rows,), generator=gen, device="cuda", dtype=torch.int32) if gather else None
    new = _forward(arena, slot, x, idx, n_rows, False, monkeypatch)
    old = _forward(arena, slot, x, idx, n_rows, True, monkeypatch)
    case = f"H={H} D={D} out={out} n_rows={n_rows} gather={gather}"
    assert bool((old[n_rows:] == SENT).all()), f"{case}: 16-row kernel wrote past n_rows"
    assert bool((new[n_rows:] == SENT).all()), f"{case}: 64-row kernel wrote past n_rows"
    assert not bool((new[:n_rows] == SENT).any()), f"{case}: rows left unwritten"
    diff = (new[:n_rows] != old[:n_rows]).any(dim=1).nonzero().flatten()
    assert diff.numel() == 0, f"{case}: {diff.numel()} rows differ, first at {int(diff[0])}"


@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("D", [7, 8, 28, 60])
@pytest.mark.parametrize("out", [1, 2, 16])
@pytest.mark.parametrize("gather", [False, True])
def test_rows_kernel_matches_tiled(H, D, out, gather, monkeypatch):
    for n_rows in (1, 63, 64, 65, 132 * 64 - 1, 132 * 64 + 1, 3 * 132 * 64 + 17):
        _check(H, D, out, n_rows, gather, monkeypatch, seed=n_rows)


@pytest.mark.parametrize("H", [128, 256])
@pytest.mark.parametrize("gather", [False, True])
def test_rows_kernel_c2_critic_pass(H, gather, monkeypatch):
    # SafetyCarCircle-v0 (D = 8), 2048 envs x 300 steps, one value per row
    _check(H, 8, 1, 614400, gather, monkeypatch)


def test_wide_input_takes_tiled_kernel(monkeypatch):
    # 64 rows of a 400-wide input do not fit one CTA's shared memory next to the H = 256 buffers: the call takes
    # the 16-row kernel instead of failing
    _check(256, 400, 2, 65, True, monkeypatch)
