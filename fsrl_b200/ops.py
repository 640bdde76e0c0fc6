"""Thin torch-tensor front end of the C-ABI: validates shapes/dtypes/devices, hands raw device
pointers + the current CUDA stream to libfsrl_b200.so.  torch is plumbing here (device
memory + streams), never the compute path.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import check, lib

_workspaces = {}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError(f"{name} must be a CUDA tensor (fsrl_b200 has no CPU path)")
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    return t


def workspace(nbytes: int, device, tag: str = "default") -> torch.Tensor:
    """Grow-only scratch buffer per (device, tag); caller-owned in the C-ABI sense."""
    key = (torch.device(device).index, tag)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(int(nbytes), 1 << 16), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def gae_dual(v: torch.Tensor, vnext: torch.Tensor, rew: torch.Tensor,
             cost: Optional[torch.Tensor], end_flag: torch.Tensor,
             terminated: Optional[torch.Tensor], gamma: float, gae_lambda: float,
             out: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
             ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Dual GAE over the flat env-major buffer (include/fsrl_b200.h: fsrl_gae_dual).

    v, vnext: (C, N) f32; rew, cost: (N,) f32; end_flag, terminated: (N,) uint8/bool.
    Returns (adv, ret), each (C, N) f32.  Mirrors base_policy.py:384-451 minus the critic
    forward passes."""
    assert 0.0 <= gae_lambda <= 1.0, "GAE lambda should be in [0, 1]."   # base_policy.py:407
    assert 0.0 <= gamma <= 1.0, "discount factor should be in [0, 1]."   # base_policy.py:112
    _req(v, torch.float32, "v"); _req(vnext, torch.float32, "vnext")
    if v.dim() == 1:
        v = v.unsqueeze(0); vnext = vnext.unsqueeze(0)
    C, N = v.shape
    if vnext.shape != v.shape:
        raise ValueError("v and vnext must have the same shape")
    _req(rew, torch.float32, "rew")
    if C == 2:
        if cost is None:
            raise ValueError("cost is required with two critics")
        _req(cost, torch.float32, "cost")
    end_u8 = end_flag.view(torch.uint8) if end_flag.dtype == torch.bool else end_flag
    _req(end_u8, torch.uint8, "end_flag")
    term_u8 = None
    if terminated is not None:
        term_u8 = terminated.view(torch.uint8) if terminated.dtype == torch.bool else terminated
        _req(term_u8, torch.uint8, "terminated")
    for nm, t in (("rew", rew), ("cost", cost), ("end_flag", end_u8), ("terminated", term_u8)):
        if t is not None and t.numel() != N:
            raise ValueError(f"{nm} has {t.numel()} elements, expected {N}")
    if out is None:
        adv = torch.empty_like(v); ret = torch.empty_like(v)
    else:
        adv, ret = out
        _req(adv, torch.float32, "adv"); _req(ret, torch.float32, "ret")
        # the kernel writes C rows of N elements at stride N: a smaller buffer would be written past its end
        for nm, t in (("adv", adv), ("ret", ret)):
            if t.shape != v.shape:
                raise ValueError(f"out {nm} has shape {tuple(t.shape)}, expected {tuple(v.shape)}")
    need = lib.fsrl_gae_dual_workspace_bytes(N)
    ws = workspace(need, v.device, "gae")
    with torch.cuda.device(v.device):
        check(lib.fsrl_gae_dual(_ptr(v), _ptr(vnext), _ptr(rew), _ptr(cost), _ptr(end_u8),
                                _ptr(term_u8), float(gamma), float(gae_lambda), _ptr(adv),
                                _ptr(ret), N, N, C, _ptr(ws), ws.numel(), _stream()))
    return adv, ret
