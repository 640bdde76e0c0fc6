"""Host-side context of the generic MLP engine (csrc/engine.cu): owns the W2 mirror and one
scratch slot per network, and builds the ctypes descriptors (netlists, inputs)."""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence

import torch

from . import _lib
from .nets import Arena, NetSlot

DX_LD = _lib.lib.fsrl_engine_dx_ld()   # row stride of the 'dx' region, and the widest input a net may have


class EngineCtx:
    def __init__(self, arena: Arena, bmax: int, extra_slots: int = 0, grown_from: Optional["EngineCtx"] = None):
        """grown_from: the context this one replaces when a caller needs more rows.  Its Adam moments carry over,
        since the learners' step counters keep counting across the growth."""
        self.arena = arena
        self.bmax = int(bmax)
        dev = arena.device
        H = arena.slots[0].H
        self.H = H
        self.slot_floats = _lib.lib.fsrl_engine_slot_floats(H, self.bmax)
        n = len(arena.slots) + int(extra_slots)
        self._n_base = len(arena.slots)
        self.scratch = torch.zeros(n * self.slot_floats, dtype=torch.float32, device=dev)
        self.w2n = torch.zeros(len(arena.slots) * H * H, dtype=torch.float32, device=dev)
        if grown_from is not None:
            self.adam_m, self.adam_v = grown_from.adam_m, grown_from.adam_v
        else:
            self.adam_m = torch.zeros_like(arena.theta)
            self.adam_v = torch.zeros_like(arena.theta)
        self._index = {id(s): i for i, s in enumerate(arena.slots)}
        self.sync_mirror(arena.slots)

    def extra_slot(self, k: int) -> int:
        return self._n_base + k

    # ---- descriptors ----------------------------------------------------------------------------
    def engine(self) -> "_lib.Engine":
        e = _lib.Engine()
        a = self.arena
        e.theta, e.grad = a.theta.data_ptr(), a.grad.data_ptr()
        e.adam_m, e.adam_v = self.adam_m.data_ptr(), self.adam_v.data_ptr()
        e.w2n, e.scratch, e.bmax = self.w2n.data_ptr(), self.scratch.data_ptr(), self.bmax
        return e

    def netref(self, s: NetSlot) -> "_lib.NetRef":
        i = self._index[id(s)]
        r = _lib.NetRef()
        r.off, r.w2n_off = s.offset, i * self.H * self.H
        r.D, r.H, r.out, r.n_extra, r.slot = s.D, s.H, s.out, s.n_extra, i
        return r

    def netlist(self, slots: Sequence[NetSlot]) -> "_lib.NetList":
        nl = _lib.NetList()
        nl.n = len(slots)
        for i, s in enumerate(slots):
            nl.nets[i] = self.netref(s)
        return nl

    def slot_view(self, s: NetSlot, what: str) -> torch.Tensor:
        """torch view of a scratch region: 'out' / 'dout' [bmax,16], 'dx' [bmax,FSRL_ENG_DX_LD],
        'h1','h2','dz1','dz2' [bmax,H]."""
        i = self._index[id(s)]
        base = i * self.slot_floats
        bh = self.bmax * self.H
        offs = {"h1": 0, "h2": bh, "dz1": 2 * bh, "dz2": 3 * bh, "out": 4 * bh,
                "dout": 4 * bh + self.bmax * 16, "dx": 4 * bh + 2 * self.bmax * 16}
        width = {"out": 16, "dout": 16, "dx": DX_LD}.get(what, self.H)
        o = base + offs[what]
        return self.scratch[o:o + self.bmax * width].view(self.bmax, width)

    @staticmethod
    def make_input(xa: torch.Tensor, ia: Optional[torch.Tensor] = None, xb: Optional[torch.Tensor] = None,
                   ib: Optional[torch.Tensor] = None) -> "_lib.EngInput":
        x = _lib.EngInput()
        x.xa, x.Da = xa.data_ptr(), xa.shape[1]
        x.ia = None if ia is None else ia.data_ptr()
        if xb is not None:
            x.xb, x.Db = xb.data_ptr(), xb.shape[1]
            x.ib = None if ib is None else ib.data_ptr()
        return x

    # ---- thin wrappers -----------------------------------------------------------------------------
    def _stream(self):
        return torch.cuda.current_stream().cuda_stream

    def sync_mirror(self, slots):
        e, nl = self.engine(), self.netlist(slots[:8])
        with torch.cuda.device(self.arena.device):
            for k in range(0, len(slots), 8):
                nl = self.netlist(slots[k:k + 8])
                _lib.check(_lib.lib.fsrl_engine_sync_mirror(ctypes.byref(e), ctypes.byref(nl), self._stream()))

    def forward(self, slots, inp, B, save=False):
        e, nl = self.engine(), self.netlist(slots)
        with torch.cuda.device(self.arena.device):
            _lib.check(_lib.lib.fsrl_engine_forward(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), B, int(save), self._stream()))

    def backward(self, slots, B, want_dx=False):
        e, nl = self.engine(), self.netlist(slots)
        with torch.cuda.device(self.arena.device):
            _lib.check(_lib.lib.fsrl_engine_backward(ctypes.byref(e), ctypes.byref(nl), B, int(want_dx), self._stream()))

    def wgrad(self, slots, inp, B, accumulate=False, norm_sq: Optional[torch.Tensor] = None):
        e, nl = self.engine(), self.netlist(slots)
        with torch.cuda.device(self.arena.device):
            _lib.check(_lib.lib.fsrl_engine_wgrad(ctypes.byref(e), ctypes.byref(nl), ctypes.byref(inp), B,
                                                  int(accumulate), None if norm_sq is None else norm_sq.data_ptr(),
                                                  self._stream()))

    def adam(self, slots, lr, step, betas=(0.9, 0.999), eps=1e-8, grad_scale=1.0, l2_reg=0.0,
             norm_sq: Optional[torch.Tensor] = None, max_grad_norm=0.0):
        e, nl = self.engine(), self.netlist(slots)
        with torch.cuda.device(self.arena.device):
            _lib.check(_lib.lib.fsrl_engine_adam(ctypes.byref(e), ctypes.byref(nl), lr, betas[0], betas[1], eps,
                                                 int(step), grad_scale, l2_reg,
                                                 None if norm_sq is None else norm_sq.data_ptr(),
                                                 float(max_grad_norm or 0.0), self._stream()))

    def polyak(self, dst, src, tau):
        e, d, s = self.engine(), self.netlist(dst), self.netlist(src)
        with torch.cuda.device(self.arena.device):
            _lib.check(_lib.lib.fsrl_engine_polyak(ctypes.byref(e), ctypes.byref(d), ctypes.byref(s), float(tau), self._stream()))
