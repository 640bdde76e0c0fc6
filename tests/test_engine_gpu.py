"""The generic MLP engine (csrc/engine.cu) against float64 references, at every hidden width.

Every case builds its arena straight from NetSlots with seeded weights and recomputes each stage
in float64 on the CPU from the fp32 data that stage read: the input rows, and the activations /
head gradients the previous stage left in the scratch slot.

* forward, backward, wgrad: an output y = sum_i a_i b_i must satisfy |y_dev - y_ref| <= TOL * m,
  m = sum_i |a_i b_i| in float64, with one TOL for every shape.  The largest |err| / m of every
  case is printed.  The head gradient has a non-zero mean, so m is not inflated by cancellation:
  at B = 12325 one dropped 32-row chunk moves a column sum by ~2.6e-3 m, > 100 x TOL.
* single-row probes: with a head gradient that is zero outside one row (0, R - 1, R, 4095, 4096,
  B - 1), dz2 / dz1 / dx carry that row alone and the gradient is that row's outer products.
* sentinels: scratch rows >= B, columns past the head / input width, slots and nets left out of
  the list and the arena's 4-float alignment padding keep their bit patterns.
* adam and polyak are element-wise and are compared in fp32 ulps with torch on the CPU.

Row counts above 4096 make wgrad split the rows over gridDim.z and combine partial tiles with
atomics (nsplit = 2 at 4097, 4 at 3 * 4096 + 37), so those gradients are not bitwise repeatable.
"""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from helpers import adam64, cg64, cg_stop_tol

TOL = 2.0 ** -16
SENT = 0x7FC0DEAD              # quiet-NaN bit pattern for memory a kernel must not write
PAD = 777.0                    # arena alignment padding
HS = (64, 128, 256, 512)
DS = (1, 7, 33, 64)            # 64 = FSRL_ENG_DX_LD; odd widths exercise the zero padding of the input tile
HEADS = ((1, 0), (3, 3), (16, 0), (8, 8))   # (out, n_extra); out + n_extra <= 16
MODES = ("plain", "gather", "critic")
REGIONS = ("h1", "h2", "dz1", "dz2", "out", "dout", "dx")


def _tile_rows(H):
    return max(4096 // H, 16)            # MlpTile<H>::R


def _cases():
    out = []
    for hi, H in enumerate(HS):
        R = _tile_rows(H)
        for bi, B in enumerate((1, R - 1, R + 1, 1000, 4096, 4097, 3 * 4096 + 37)):
            k = hi + bi
            D = DS[k % 4]
            mode = MODES[k % 3]
            if mode == "critic" and D == 1:
                mode = "gather"
            heads = (HEADS[(2 * hi + bi) % 4], HEADS[(2 * hi + bi + 1) % 4])
            out.append(pytest.param(H, D, heads, B, mode, id=f"H{H}-D{D}-B{B}-{mode}"))
    # a full list: 8 nets of one width with every head shape, rows split over 2 CTAs
    out.append(pytest.param(128, 33, HEADS * 2, 4097, "critic", id="H128-D33-B4097-critic-8nets"))
    out.append(pytest.param(512, 7, HEADS * 2, 600, "gather", id="H512-D7-B600-gather-8nets"))
    return out


# ---- arena rig -----------------------------------------------------------------------------------------
def _net(name, D, H, out, n_extra):
    from fsrl_b200.nets import NetSlot
    extra = nn.Parameter(0.3 * torch.randn(n_extra)) if n_extra else None
    return NetSlot(name, None, nn.Linear(D, H), nn.Linear(H, H), [nn.Linear(H, out)], extra)


class Rig:
    """An arena of nets with seeded nn.Linear weights and an engine context with one scratch slot
    per net; the alignment padding of theta / grad / Adam moments holds PAD."""

    def __init__(self, H, shapes, bmax, seed):
        from fsrl_b200.engine import EngineCtx
        from fsrl_b200.nets import Arena
        torch.manual_seed(seed)
        self.slots = [_net(f"n{i}", D, H, out, ne) for i, (D, out, ne) in enumerate(shapes)]
        self.arena = Arena(self.slots, "cuda")
        self.eng = EngineCtx(self.arena, bmax)
        self.H = H
        pad = []
        for i, s in enumerate(self.slots):
            end = self.slots[i + 1].offset if i + 1 < len(self.slots) else self.arena.n_params
            pad += range(s.offset + s.size, end)
        self.pad = torch.tensor(pad, dtype=torch.long, device="cuda")
        for t in (self.arena.theta, self.arena.grad, self.eng.adam_m, self.eng.adam_v):
            t[self.pad] = PAD

    def rng(self, s):
        return slice(s.offset, s.offset + s.size)

    def blocks(self, vec, s):
        """float64 CPU views of one net's blocks inside an arena-layout vector (or a vector of one net)"""
        v = vec.detach().double().cpu()
        if v.numel() != s.size:
            v = v[self.rng(s)]
        D, H, out, ne = s.D, s.H, s.out, s.n_extra
        o = np.cumsum([0, D * H, H, H * H, H, H * out, out, ne])
        return dict(w1t=v[o[0]:o[1]].view(D, H), b1=v[o[1]:o[2]], w2t=v[o[2]:o[3]].view(H, H), b2=v[o[3]:o[4]],
                    w3t=v[o[4]:o[5]].view(H, out), b3=v[o[5]:o[6]], extra=v[o[6]:o[7]])

    def slot_range(self, s):
        i = self.slots.index(s)
        return slice(i * self.eng.slot_floats, (i + 1) * self.eng.slot_floats)

    def view(self, s, what, B=None):
        v = self.eng.slot_view(s, what)
        return v if B is None else v[:B]

    def w2_mirror_ok(self, s):
        i = self.slots.index(s)
        H = self.H
        w2n = self.eng.w2n[i * H * H:(i + 1) * H * H].view(H, H)
        w2t = self.arena.theta[self.rng(s)][s.D * H + H:s.D * H + H + H * H].view(H, H)
        return torch.equal(w2n.view(torch.int32), w2t.t().contiguous().view(torch.int32))


def _bits(t):
    return t.contiguous().view(torch.int32)


def _is_sent(t):
    return bool((_bits(t) == SENT).all())


class Report:
    """largest |err| / m per quantity; asserts |err| <= TOL * m element-wise"""

    def __init__(self, case):
        self.case, self.worst = case, {}

    def close(self, name, got, ref, mag):
        got = got.detach().double().cpu()
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        assert bool(torch.isfinite(got).all()), f"{self.case} {name}: non-finite values"
        err = (got - ref).abs()
        ratio = torch.where(mag > 0, err / mag.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
        r = float(ratio.max()) if ratio.numel() else 0.0
        self.worst[name] = max(self.worst.get(name, 0.0), r)
        if r > TOL:
            i = int(ratio.reshape(-1).argmax())
            raise AssertionError(f"{self.case} {name}: |err| / m = {r:.3g} > {TOL:.3g} at flat index {i} "
                                 f"(got {got.reshape(-1)[i].item():.9g}, want {ref.reshape(-1)[i].item():.9g}, "
                                 f"m {mag.reshape(-1)[i].item():.3g})")

    def show(self):
        print(f"\n{self.case}: max |err|/m (bound {TOL:.3g}) " +
              " ".join(f"{k}={v:.2e}" for k, v in sorted(self.worst.items())))


def _mm(a, b):
    return a @ b, a.abs() @ b.abs()


def _grad_ref(X, h1, h2, dz1, dz2, dout, s):
    """float64 weight gradients (and their term magnitudes) of one net from the stage inputs"""
    G, E = dout[:, :s.out], dout[:, s.out:s.out + s.n_extra]
    ref, mag = {}, {}
    ref["w1t"], mag["w1t"] = _mm(X.t(), dz1)
    ref["w2t"], mag["w2t"] = _mm(h1.t(), dz2)
    ref["w3t"], mag["w3t"] = _mm(h2.t(), G)
    for k, t in (("b1", dz1), ("b2", dz2), ("b3", G), ("extra", E)):
        ref[k], mag[k] = t.sum(0), t.abs().sum(0)
    return ref, mag


def _input(mode, B, D, gen):
    """device input descriptor pieces and the float64 CPU input rows they describe"""
    from fsrl_b200.engine import EngineCtx
    dev = lambda t: t.cuda()
    if mode == "plain":
        xa = torch.randn(B, D, generator=gen)
        keep = (dev(xa),)
        return EngineCtx.make_input(keep[0]), keep, xa.double()
    n_a = B // 2 + 5                     # fewer source rows than B: the gather repeats indices
    if mode == "gather":
        xa = torch.randn(n_a, D, generator=gen)
        ia = torch.randint(0, n_a, (B,), generator=gen, dtype=torch.int32)
        keep = (dev(xa), dev(ia))
        return EngineCtx.make_input(keep[0], keep[1]), keep, xa[ia.long()].double()
    Db = D // 3                           # the SAC critic input concat(obs[ia], act[ib])
    Da = D - Db
    n_b = B // 3 + 2
    xa, xb = torch.randn(n_a, Da, generator=gen), torch.randn(n_b, Db, generator=gen)
    ia = torch.randint(0, n_a, (B,), generator=gen, dtype=torch.int32)
    ib = torch.randint(0, n_b, (B,), generator=gen, dtype=torch.int32)
    keep = (dev(xa), dev(ia), dev(xb), dev(ib))
    return EngineCtx.make_input(*keep), keep, torch.cat([xa[ia.long()], xb[ib.long()]], 1).double()


# ---- forward / backward / wgrad ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("H,D,heads,B,mode", _cases())
def test_forward_backward_wgrad_match_float64(H, D, heads, B, mode):
    from fsrl_b200 import _lib
    # listed nets interleaved with an unlisted one, and listed in reverse arena order
    shapes = [(D, *heads[0]), (D, 1, 0)] + [(D, *h) for h in heads[1:]]
    rig = Rig(H, shapes, bmax=B + 3, seed=H + 7 * B + D)
    eng, arena = rig.eng, rig.arena
    listed = [rig.slots[0]] + rig.slots[2:]
    unlisted = rig.slots[1]
    nets = listed[::-1]
    R = _tile_rows(H)
    rep = Report(f"H={H} D={D} B={B} {mode} nets={len(nets)}")
    gen = torch.Generator().manual_seed(B * 31 + H)
    inp, _keep, X = _input(mode, B, D, gen)
    _bits(eng.scratch).fill_(SENT)
    _bits(arena.grad[rig.rng(unlisted)]).fill_(SENT)
    theta0 = arena.theta.clone()

    # forward without, then with saved activations: the head output must not depend on `save`
    eng.forward(nets, inp, B, save=False)
    out0 = {id(s): rig.view(s, "out", B).clone() for s in listed}
    for s in listed:
        assert _is_sent(rig.view(s, "h1")) and _is_sent(rig.view(s, "h2"))
    eng.forward(nets, inp, B, save=True)
    act = {}
    for s in listed:
        p = rig.blocks(arena.theta, s)
        h1, h2, out = (rig.view(s, k, B).double().cpu() for k in ("h1", "h2", "out"))
        assert torch.equal(_bits(rig.view(s, "out", B)), _bits(out0[id(s)])), "forward output depends on save"
        ref, mag = _mm(X, p["w1t"])
        rep.close("h1", h1, (ref + p["b1"]).clamp_min(0), mag + p["b1"].abs())
        ref, mag = _mm(h1, p["w2t"])
        rep.close("h2", h2, (ref + p["b2"]).clamp_min(0), mag + p["b2"].abs())
        ref, mag = _mm(h2, p["w3t"])
        rep.close("out", out[:, :s.out], ref + p["b3"], mag + p["b3"].abs())
        assert bool((out[:, s.out:] == 0).all()), "forward: columns past the head must be zero"
        act[id(s)] = (h1, h2)

    # seeded head gradients (non-zero mean); columns past out + n_extra keep the sentinel
    douts = {}
    for s in listed:
        w = s.out + s.n_extra
        dd = torch.randn(B, w, generator=gen) + 0.5
        rig.view(s, "dout", B)[:, :w] = dd.cuda()
        douts[id(s)] = dd.double()

    def check_backward(s, want_dx):
        p = rig.blocks(arena.theta, s)
        h1, h2 = act[id(s)]
        dz2, dz1 = (rig.view(s, k, B).double().cpu() for k in ("dz2", "dz1"))
        ref, mag = _mm(douts[id(s)][:, :s.out], p["w3t"].t())
        rep.close("dz2", dz2, ref * (h2 > 0), mag)
        ref, mag = _mm(dz2, p["w2t"].t())
        rep.close("dz1", dz1, ref * (h1 > 0), mag)
        if want_dx:     # dx covers the xb columns of the critic form as well
            ref, mag = _mm(dz1, p["w1t"].t())
            rep.close("dx", rig.view(s, "dx", B)[:, :D], ref, mag)
        return dz1, dz2

    eng.backward(nets, B, want_dx=False)
    saved = {}
    for s in listed:
        assert _is_sent(rig.view(s, "dx")), "backward(want_dx=0) wrote dx"
        saved[id(s)] = check_backward(s, False)
    eng.backward(nets, B, want_dx=True)
    for s in listed:
        dz1, dz2 = check_backward(s, True)
        assert torch.equal(dz1, saved[id(s)][0]) and torch.equal(dz2, saved[id(s)][1]), "dz depends on want_dx"

    # weight gradients: write over a finite prior, accumulate onto it, and into a separate vector
    refs = {}
    for s in listed:
        h1, h2 = act[id(s)]
        dz1, dz2 = saved[id(s)]
        refs[id(s)] = _grad_ref(X, h1, h2, dz1, dz2, douts[id(s)], s)
    prior = {id(s): torch.randn(s.size, generator=gen) for s in listed}
    ns = torch.full((1,), 0.25, dtype=torch.float32, device="cuda")
    for accumulate in (False, True):
        for s in listed:
            arena.grad[rig.rng(s)] = prior[id(s)].cuda()
        ns.fill_(0.25)
        eng.wgrad(nets, inp, B, accumulate=accumulate, norm_sq=ns)
        tot = 0.0
        for s in listed:
            got = rig.blocks(arena.grad, s)
            pb = rig.blocks(prior[id(s)], s)
            ref, mag = refs[id(s)]
            for k in ref:
                r, m = (ref[k] + pb[k], mag[k] + pb[k].abs()) if accumulate else (ref[k], mag[k])
                rep.close(f"g_{k}", got[k], r, m)
            tot += float((arena.grad[rig.rng(s)].double() ** 2).sum())
        # *norm_sq += |final gradient|^2 over the listed nets (fp32 sums of squares)
        assert abs(float(ns.item()) - 0.25 - tot) <= 1e-4 * tot, (accumulate, ns.item() - 0.25, tot)
    grad_before = arena.grad.clone()
    e = eng.engine()
    for s in listed[:2]:
        dst = torch.randn(s.size, generator=gen).cuda()
        _lib.check(_lib.lib.fsrl_engine_wgrad_to(ctypes.byref(e), ctypes.byref(eng.netlist([s])), ctypes.byref(inp),
                                                 B, dst.data_ptr(), torch.cuda.current_stream().cuda_stream))
        got = rig.blocks(dst, s)
        ref, mag = refs[id(s)]
        for k in ref:
            rep.close(f"to_{k}", got[k], ref[k], mag[k])
    assert torch.equal(_bits(arena.grad), _bits(grad_before)), "wgrad_to touched the arena gradient"

    # single-row probes
    for p_row in sorted({r for r in (0, R - 1, R, 4095, 4096, B - 1) if 0 <= r < B}):
        probe = {}
        for s in listed:
            w = s.out + s.n_extra
            dd = torch.zeros(B, w, dtype=torch.float64)
            dd[p_row] = douts[id(s)][p_row]
            rig.view(s, "dout", B)[:, :w] = dd.float().cuda()
            probe[id(s)] = dd
        eng.backward(nets, B, want_dx=True)
        eng.wgrad(nets, inp, B)
        for s in listed:
            dz1, dz2, dx = (rig.view(s, k, B).double().cpu() for k in ("dz1", "dz2", "dx"))
            full1, full2 = saved[id(s)]
            others = torch.ones(B, dtype=torch.bool)
            others[p_row] = False
            assert bool((dz1[others] == 0).all() and (dz2[others] == 0).all() and (dx[others, :D] == 0).all()), \
                f"probe row {p_row}: other rows are not zero"
            assert torch.equal(dz1[p_row], full1[p_row]) and torch.equal(dz2[p_row], full2[p_row]), \
                f"probe row {p_row}: row differs from the full backward"
            h1, h2 = act[id(s)]
            one = slice(p_row, p_row + 1)
            ref, mag = _grad_ref(X[one], h1[one], h2[one], dz1[one], dz2[one], probe[id(s)][one], s)
            got = rig.blocks(arena.grad, s)
            for k in ref:
                rep.close(f"probe_{k}", got[k], ref[k], mag[k])

    # sentinels
    for s in listed:
        for k in REGIONS:
            assert _is_sent(rig.view(s, k)[B:]), f"{k}: rows >= B written"
        assert _is_sent(rig.view(s, "dx", B)[:, D:]), "dx: columns >= D written"
        assert _is_sent(rig.view(s, "dout", B)[:, s.out + s.n_extra:]), "dout columns past the head changed"
    assert _is_sent(eng.scratch[rig.slot_range(unlisted)]), "scratch slot of an unlisted net written"
    assert _is_sent(arena.grad[rig.rng(unlisted)]), "gradient of an unlisted net written"
    assert bool((arena.grad[rig.pad] == PAD).all()), "gradient alignment padding written"
    assert torch.equal(_bits(arena.theta), _bits(theta0)), "parameters changed"
    rep.show()


# ---- Adam --------------------------------------------------------------------------------------------------
# vs torch fp32, in ulps of the largest operand of the update: nvcc contracts to FMA where torch's
# lerp / addcmul / add(alpha) may not
ADAM_ULPS = 4


def _ulp32(*xs):
    """fp32 ulp of the largest magnitude among xs, element-wise (float64 CPU)"""
    big = torch.stack([x.detach().cpu().double().abs() for x in xs]).amax(0)
    return torch.from_numpy(np.spacing(big.float().numpy())).double()


def _ulps(got, want, *terms):
    """|got - want| in ulps of the largest of want and the update's terms: the update p + step (or
    beta m + (1 - beta) g) may cancel, and then one rounding of a term is many ulps of the result"""
    return ((got.detach().cpu().double() - want.detach().cpu().double()).abs() / _ulp32(want, *terms)).max().item()


@pytest.mark.gpu
@pytest.mark.parametrize("opt", ["plain", "scale_l2", "clip"])
@pytest.mark.parametrize("H", HS)
def test_adam_matches_torch(H, opt):
    lr, betas, eps = 3e-3, (0.9, 0.999), 1e-8
    gscale, l2 = (0.37, 1e-3) if opt == "scale_l2" else (1.0, 0.0)
    # nets of different sizes in one list (each has its own plain / W2-tile block split), one left out
    rig = Rig(H, [(17, 3, 3), (5, 1, 0), (64, 16, 0), (1, 8, 8)], bmax=1, seed=H)
    eng, arena = rig.eng, rig.arena
    listed, unlisted = [rig.slots[2], rig.slots[0], rig.slots[3]], rig.slots[1]
    gen = torch.Generator().manual_seed(5 + H)
    eng.adam_m[rig.rng(unlisted)] = 0.5
    eng.adam_v[rig.rng(unlisted)] = 0.25
    _bits(arena.grad[rig.rng(unlisted)]).fill_(SENT)
    keep = {k: t[rig.rng(unlisted)].clone() for k, t in (("theta", arena.theta), ("m", eng.adam_m), ("v", eng.adam_v))}
    params = {id(s): arena.theta[rig.rng(s)].detach().cpu().clone().requires_grad_(True) for s in listed}
    topt = torch.optim.Adam(list(params.values()), lr=lr, betas=betas, eps=eps, weight_decay=2 * l2, foreach=False)
    ns = torch.zeros(1, dtype=torch.float32, device="cuda")
    worst = {"theta": 0.0, "m": 0.0, "v": 0.0, "f64": 0.0}
    for t in (1, 2, 3, 10 ** 6):
        if t == 10 ** 6:
            for st in topt.state.values():
                st["step"] = torch.tensor(float(t - 1))
        grads = {id(s): (torch.randn(s.size, generator=gen) * 0.1).float() for s in listed}
        before = {id(s): (arena.theta[rig.rng(s)].cpu().double(), eng.adam_m[rig.rng(s)].cpu().double(),
                          eng.adam_v[rig.rng(s)].cpu().double()) for s in listed}
        for s in listed:
            arena.grad[rig.rng(s)] = grads[id(s)].cuda()
        max_norm, coef = 0.0, torch.tensor(1.0)
        if opt == "clip":
            nsq = torch.stack([(g.double() ** 2).sum() for g in grads.values()]).sum().float()
            ns.fill_(float(nsq))
            max_norm = 0.3 * float(nsq.sqrt())       # clipping bites: coef ~ 0.3
            # torch.nn.utils.clip_grad_norm_: coef = max_norm / (total_norm + 1e-6), clamped to 1
            coef = (torch.tensor(max_norm, dtype=torch.float32) / (ns.cpu().sqrt()[0] + 1e-6)).clamp(max=1.0)
        eng.adam(listed, lr, t, betas=betas, eps=eps, grad_scale=gscale, l2_reg=l2,
                 norm_sq=ns if opt == "clip" else None, max_grad_norm=max_norm)
        scale = torch.tensor(gscale, dtype=torch.float32) * coef
        for s in listed:
            # torch steps from the device's state, so that each step is compared on its own
            p0, m0, v0 = before[id(s)]
            params[id(s)].data.copy_(p0.float())
            if t > 1:
                topt.state[params[id(s)]]["exp_avg"].copy_(m0.float())
                topt.state[params[id(s)]]["exp_avg_sq"].copy_(v0.float())
            params[id(s)].grad = grads[id(s)] * scale
        topt.step()
        for s in listed:
            tp, st = params[id(s)], topt.state[params[id(s)]]
            p0, m0, v0 = before[id(s)]
            g_eff = grads[id(s)].double() * float(scale) + 2 * l2 * p0
            worst["theta"] = max(worst["theta"], _ulps(arena.theta[rig.rng(s)], tp, p0, tp.double() - p0))
            worst["m"] = max(worst["m"], _ulps(eng.adam_m[rig.rng(s)], st["exp_avg"], m0, g_eff))
            worst["v"] = max(worst["v"], _ulps(eng.adam_v[rig.rng(s)], st["exp_avg_sq"], v0, g_eff * g_eff))
            # one float64 step from the same fp32 state: two roundings of the larger of p and p_new, plus
            # 1e-5 of the step with m replaced by the larger of its terms (m = b1 m0 + (1 - b1) g may cancel)
            p64, _, v64 = adam64(p0, grads[id(s)].double() * float(scale), m0, v0, t, lr, betas, eps, 2 * l2)
            got = arena.theta[rig.rng(s)].cpu().double()
            denom = v64.sqrt() / (1 - betas[1] ** t) ** 0.5 + eps
            step_scale = lr / (1 - betas[0] ** t) * torch.maximum(m0.abs(), g_eff.abs()) / denom
            lim = 2 * _ulp32(p0, p64) + 1e-5 * step_scale
            worst["f64"] = max(worst["f64"], ((got - p64).abs() / lim).max().item())
            assert rig.w2_mirror_ok(s), "W2 mirror is not the transpose of W2 after adam"
    print(f"\nadam H={H} {opt}: max ulps theta={worst['theta']:.0f} m={worst['m']:.0f} v={worst['v']:.0f} "
          f"(bound {ADAM_ULPS}); float64 error / bound {worst['f64']:.2f}")
    assert max(worst["theta"], worst["m"], worst["v"]) <= ADAM_ULPS, worst
    assert worst["f64"] <= 1.0, worst
    for k, t in (("theta", arena.theta), ("m", eng.adam_m), ("v", eng.adam_v)):
        assert torch.equal(t[rig.rng(unlisted)], keep[k]), f"adam changed {k} of an unlisted net"
    assert _is_sent(arena.grad[rig.rng(unlisted)])
    for t in (arena.theta, arena.grad, eng.adam_m, eng.adam_v):
        assert bool((t[rig.pad] == PAD).all()), "adam wrote the alignment padding"


# ---- Polyak and the W2 mirror ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tau", [0.0, 0.005, 1.0])
@pytest.mark.parametrize("H", HS)
def test_polyak_matches_fp32_expression(H, tau):
    shapes = [(9, 3, 3), (9, 1, 0), (9, 3, 3), (9, 1, 0), (9, 1, 0)]
    rig = Rig(H, shapes, bmax=1, seed=3 * H)
    eng, arena = rig.eng, rig.arena
    src, dst, unlisted = rig.slots[0:2], rig.slots[2:4], rig.slots[4]
    theta0, w2n0 = arena.theta.clone(), eng.w2n.clone()
    eng.polyak(dst, src, tau)
    t32 = np.float32(tau)
    omt = np.float32(1.0) - t32
    worst = 0.0
    for d_, s_ in zip(dst, src):
        s_v = theta0[rig.rng(s_)].cpu().numpy()
        d_v = theta0[rig.rng(d_)].cpu().numpy()
        a, b = t32 * s_v, omt * d_v
        want = a + b
        got = arena.theta[rig.rng(d_)].cpu().numpy()
        if tau in (0.0, 1.0):
            assert np.array_equal(got, d_v if tau == 0.0 else s_v), "tau 0 / 1 must copy exactly"
        # two roundings of the larger product (contracted to an FMA or not)
        lim = 2 * np.spacing(np.maximum(np.abs(a), np.abs(b)))
        err = np.abs(got.astype(np.float64) - want)
        worst = max(worst, float((err / lim).max()))
        assert rig.w2_mirror_ok(d_), "W2 mirror of dst is not the transpose after polyak"
    print(f"\npolyak H={H} tau={tau}: max |err| / (2 ulp of the larger term) = {worst:.2f}")
    assert worst <= 1.0
    for s in src + [unlisted]:
        assert torch.equal(_bits(arena.theta[rig.rng(s)]), _bits(theta0[rig.rng(s)])), "polyak changed a source"
    # slots 0, 1 (sources) and 4 (unlisted) keep their mirrors
    assert torch.equal(eng.w2n[:2 * H * H], w2n0[:2 * H * H]), "polyak changed a source mirror"
    assert torch.equal(eng.w2n[4 * H * H:], w2n0[4 * H * H:]), "polyak changed an unlisted mirror"
    assert bool((arena.theta[rig.pad] == PAD).all())


@pytest.mark.gpu
def test_polyak_rejects_different_extra():
    rig = Rig(64, [(9, 3, 3), (9, 3, 0)], bmax=1, seed=1)
    theta0 = rig.arena.theta.clone()
    with pytest.raises(ValueError, match="polyak: shape mismatch"):
        rig.eng.polyak([rig.slots[1]], [rig.slots[0]], 0.5)
    with pytest.raises(ValueError, match="polyak: shape mismatch"):
        rig.eng.polyak([rig.slots[0]], [rig.slots[1]], 0.5)
    assert torch.equal(rig.arena.theta, theta0)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [64, 256])
def test_sync_mirror_more_than_eight_nets(H):
    shapes = [(1 + 5 * i, 1 + i % 16, (3 * i) % (16 - i % 16)) for i in range(11)]
    rig = Rig(H, shapes, bmax=1, seed=11)
    eng = rig.eng
    _bits(eng.w2n).fill_(SENT)
    eng.sync_mirror(rig.slots[2:5])
    for i, s in enumerate(rig.slots):
        if 2 <= i < 5:
            assert rig.w2_mirror_ok(s), i
        else:
            assert _is_sent(eng.w2n[i * H * H:(i + 1) * H * H]), f"mirror of unlisted net {i} written"
    eng.sync_mirror(rig.slots)
    assert all(rig.w2_mirror_ok(s) for s in rig.slots)


# ---- the float64 reference helpers themselves (CPU) ------------------------------------------------------
def test_adam64_matches_torch_adam():
    gen = torch.Generator().manual_seed(0)
    p = torch.randn(50, generator=gen, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([p], lr=1e-2, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.03, foreach=False)
    q, m, v = p.detach().clone(), torch.zeros(50, dtype=torch.float64), torch.zeros(50, dtype=torch.float64)
    for t in (1, 2, 3, 10 ** 6):
        if t == 10 ** 6:
            opt.state[p]["step"] = torch.tensor(float(t - 1))
        g = torch.randn(50, generator=gen, dtype=torch.float64)
        p.grad = g.clone()
        opt.step()
        q, m, v = adam64(q, g, m, v, t, 1e-2, (0.8, 0.99), 1e-6, 0.03)
        torch.testing.assert_close(q, p.detach(), rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(m, opt.state[p]["exp_avg"], rtol=1e-13, atol=1e-15)
        torch.testing.assert_close(v, opt.state[p]["exp_avg_sq"], rtol=1e-13, atol=1e-15)


def test_cg64_solves_and_stops_like_the_reference_loop():
    gen = torch.Generator().manual_seed(1)
    n = 12
    Q = torch.randn(n, n, generator=gen, dtype=torch.float64)
    A = Q @ Q.t() / n + 0.1 * torch.eye(n, dtype=torch.float64)
    b = torch.randn(n, generator=gen, dtype=torch.float64)
    x, res = cg64(lambda v: A @ v, b, nsteps=3 * n, tol=1e-24)
    torch.testing.assert_close(x, torch.linalg.solve(A, b), rtol=1e-9, atol=1e-12)
    assert res[-1] < 1e-24 and all(r >= 1e-24 for r in res[:-1])
    x_full, full = cg64(lambda v: A @ v, b, nsteps=10, tol=0.0)
    k, tol = cg_stop_tol(full)
    assert all(r > tol for r in full[:k]) and full[k] < tol
    x_stop, res_stop = cg64(lambda v: A @ v, b, nsteps=10, tol=tol)
    assert len(res_stop) == k + 1 and res_stop == full[:k + 1]
    # the stopped solve is the unstopped loop's iterate k + 1, and far from its iterate 10
    x_k, _ = cg64(lambda v: A @ v, b, nsteps=k + 1, tol=0.0)
    assert torch.equal(x_stop, x_k)
    assert float((x_stop - x_full).norm()) > 1e-3 * float(x_full.norm())
