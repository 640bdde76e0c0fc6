"""The dual GAE scan (csrc/gae.cu, gae_dual_kernel) past one resident wave of tiles, against the float64 oracle.

fsrl_gae_dual launches a persistent grid of min(tiles, 3 x SMs) CTAs; each CTA keeps claiming 2048-transition tiles
through an atomic ticket, and the carry between tiles comes from decoupled look-back.  At c2's 614 400 transitions
(300 tiles) every CTA of a 132-SM H100 takes exactly one tile; c3's 2 048 000 (1000 tiles) and the benchmark's GAE
sweep run several tiles per CTA.  This file runs that regime: tile counts around and past the wave, segments that
span hundreds of tiles (the look-back composes aggregates instead of stopping at the first predecessor), the scalar
load/store path at scale (misaligned pointers, N % 4 != 0, ld > N), every mode, the parameter edges, back-to-back
calls that re-use the grow-only workspace, and run-to-run repeatability.

Contract (as tests/test_gae_gpu.py): the oracle is oracle.returns.dual_gae (a C port of the reference's numba
gae_return, f64 accumulation, pinned bitwise by tests/golden/returns_golden.npz).  The kernel also accumulates in f64
but re-associates the carry across threads and tiles, so an element may round to the neighbouring f32: <= 1 f32 ulp
everywhere and bit-equality on >= 99.99 % of the elements.  Each case prints its max ulp and bit-equal share."""
import numpy as np
import pytest
import torch

from oracle import returns

pytestmark = pytest.mark.gpu

TILE = 2048                  # GAE_TPB x GAE_ITEMS in csrc/gae.cu


def _wave():
    """Tiles of one resident wave: fsrl_gae_dual launches min(tiles, 3 x SM count) CTAs (__launch_bounds__(256, 3))."""
    return 3 * torch.cuda.get_device_properties(0).multi_processor_count


def _tiles(N):
    return -(-N // TILE)


def _ulp_diff(a, b):
    ai = a.view(np.int32).astype(np.int64)
    bi = b.view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, np.int64(-2**31) - ai, ai)
    bi = np.where(bi < 0, np.int64(-2**31) - bi, bi)
    return np.abs(ai - bi)


def _inputs(N, ends, seed, p_term=0.0, C=2):
    """Env-major buffer of N transitions whose truncations sit at the rows in `ends`, plus terminations at rate
    p_term elsewhere (the synth_gae_inputs distributions, at any N and segment structure)."""
    rng = np.random.default_rng(seed)
    trunc = np.zeros(N, bool)
    trunc[np.asarray(ends, dtype=np.int64)] = True
    term = (rng.random(N) < p_term) & ~trunc
    return dict(v=rng.standard_normal((C, N), dtype=np.float32), vnext=rng.standard_normal((C, N), dtype=np.float32),
                rew=rng.normal(0.5, 1.0, N).astype(np.float32), cost=(rng.random(N) < 0.05).astype(np.float32),
                terminated=term, truncated=trunc, unfinished=np.zeros(N, bool))


def _product(N, T, seed, p_term=0.002, C=2):
    """Collect-like segments: every T-th row is a truncation, rare terminations in between."""
    return _inputs(N, np.arange(T - 1, N, T), seed, p_term, C)


def _oracle(d, gamma, lam, C=2, use_term=True):
    term, trunc = d["terminated"], d["truncated"]
    if not use_term:            # no value mask, but the terminations still end their segments
        term, trunc = np.zeros_like(term), term | trunc
    _, rets, advs = returns.dual_gae(d["v"][:C], d["vnext"][:C], d["rew"], d["cost"], term, trunc, d["unfinished"],
                                     gamma, lam)
    return advs.T, rets.T


def _end(d):
    return (d["terminated"] | d["truncated"] | d["unfinished"]).astype(np.uint8)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _shifted(a, shift):
    """`a` on the device as a contiguous view `shift` elements into a larger allocation."""
    a = np.ascontiguousarray(a)
    flat = torch.from_numpy(a.reshape(-1))
    big = torch.zeros(flat.numel() + shift + 16, dtype=flat.dtype, device="cuda")
    view = big[shift:shift + flat.numel()]
    view.copy_(flat)
    return view.view(a.shape)


def _run(d, gamma, lam, C=2, use_term=True, layout="aligned"):
    """ops.gae_dual on device copies of d.  layout: "aligned" (16-byte aligned contiguous buffers), "float_offset"
    (every float buffer, outputs included, one element into a larger allocation) or "flag_offset" (end_flag /
    terminated one byte in, floats aligned)."""
    from fsrl_b200 import ops
    fshift = 1 if layout == "float_offset" else 0
    bshift = 1 if layout == "flag_offset" else 0
    N = d["rew"].shape[0]
    v, vn = _shifted(d["v"][:C], fshift), _shifted(d["vnext"][:C], fshift)
    rew = _shifted(d["rew"], fshift)
    cost = _shifted(d["cost"], fshift) if C == 2 else None
    end = _shifted(_end(d), bshift)
    term = _shifted(d["terminated"].astype(np.uint8), bshift) if use_term else None
    adv, ret = _shifted(np.zeros((C, N), np.float32), fshift), _shifted(np.zeros((C, N), np.float32), fshift)
    if layout == "float_offset":
        assert all(t.data_ptr() % 16 for t in (v, vn, rew, adv, ret) + ((cost,) if C == 2 else ()))
    if layout == "flag_offset":
        assert end.data_ptr() % 8 and (term is None or term.data_ptr() % 8)
        assert all(t.data_ptr() % 16 == 0 for t in (v, vn, rew, adv, ret))
    ops.gae_dual(v, vn, rew, cost, end, term, gamma, lam, out=(adv, ret))
    torch.cuda.synchronize()
    return adv.cpu().numpy(), ret.cpu().numpy()


def _check(name, d, adv, ret, gamma, lam, C=2, use_term=True):
    want_a, want_r = _oracle(d, gamma, lam, C, use_term)
    N = d["rew"].shape[0]
    for c in range(C):
        ua, ur = _ulp_diff(adv[c], want_a[c]), _ulp_diff(ret[c], want_r[c])
        print("\n%-34s N=%-9d tiles=%-5d critic %d: max ulp adv %d ret %d, bit-equal adv %.6f ret %.6f"
              % (name, N, _tiles(N), c, ua.max(initial=0), ur.max(initial=0), (ua == 0).mean(), (ur == 0).mean()),
              end="")
        assert ua.max(initial=0) <= 1 and ur.max(initial=0) <= 1, (name, c, ua.max(), ur.max(), int(np.argmax(ua)))
        assert (ua == 0).mean() >= 0.9999 and (ur == 0).mean() >= 0.9999, (name, c, (ua == 0).mean(), (ur == 0).mean())


def _several_waves(N):
    W = _wave()
    assert _tiles(N) > W, (N, _tiles(N), W)        # more tiles than CTAs: each CTA claims several tickets


# ---- tile count against the resident wave ----------------------------------------------------------------------------
SIZES = {"wave-1": lambda W: TILE * W - 1, "wave": lambda W: TILE * W, "wave+1": lambda W: TILE * W + 1,
         "2waves+tile+1": lambda W: 2 * TILE * W + TILE + 1, "c3": lambda W: 2048 * 1000, "10M": lambda W: 10_000_000}


@pytest.mark.parametrize("T", [300, 1000])
@pytest.mark.parametrize("size", list(SIZES))
def test_tile_count_against_wave(size, T):
    W = _wave()
    N = SIZES[size](W)
    if size in ("wave+1", "2waves+tile+1", "c3", "10M"):
        _several_waves(N)
    else:
        assert _tiles(N) <= W                       # the boundary itself: one tile per CTA
    d = _product(N, T, seed=N % 100003 + T)
    adv, ret = _run(d, 0.99, 0.95)
    _check(f"{size} T={T}", d, adv, ret, 0.99, 0.95)


# ---- long segments: the look-back composes aggregates across many tiles -------------------------------------------
def _tile_product_nonzero(gl, n_tiles):
    """The f64 A of n_tiles consecutive segment-free tiles, composed as the kernel composes it (per element, then
    per tile)."""
    a = 1.0
    for _ in range(TILE):
        a *= gl
    return a ** n_tiles != 0.0


@pytest.mark.parametrize("gamma,lam", [(1.0, 1.0), (0.999, 0.999)])
def test_one_segment_across_waves(gamma, lam):
    """One env and no end but the final truncation over three waves of tiles.  gamma = lambda = 1 keeps every
    aggregate's A at 1, so a look-back may walk to ticket 0; gamma * lambda = 0.998 gives A ~ 0.017 per tile, non-zero
    in f64 across ~170 tiles.  How far a look-back walks depends on timing; what is asserted is the precondition that
    the segment spans > 100 tiles with a non-zero f64 A."""
    W = _wave()
    N = 3 * TILE * W + 1234
    _several_waves(N)
    d = _inputs(N, [N - 1], seed=21)
    assert d["truncated"].sum() == 1 and not d["terminated"].any()
    assert _tiles(N) > 100 and _tile_product_nonzero(gamma * lam, 101)
    adv, ret = _run(d, gamma, lam)
    _check(f"one segment g={gamma} l={lam}", d, adv, ret, gamma, lam)


def test_mixed_long_segments():
    """Segments of 3 to 30 tiles, their ends at arbitrary offsets inside tiles."""
    W = _wave()
    rng = np.random.default_rng(4)
    N = 2 * TILE * W + 777
    lens = rng.integers(3 * TILE, 30 * TILE, size=N // (3 * TILE) + 1)
    ends = np.cumsum(lens) - 1
    ends = np.append(ends[ends < N - 1], N - 1)
    seg = np.diff(np.concatenate([[-1], ends]))
    assert seg[:-1].min() >= 3 * TILE and seg.max() <= 30 * TILE and len(seg) >= 10
    assert (ends[:-1] % TILE).std() > 0            # the ends do not line up with tile borders
    _several_waves(N)
    d = _inputs(N, ends, seed=5)
    adv, ret = _run(d, 0.999, 0.999)
    _check("mixed 3..30-tile segments", d, adv, ret, 0.999, 0.999)


# ---- layouts: the scalar path at scale ------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["aligned", "float_offset", "flag_offset"])
def test_layouts_multi_wave(layout):
    W = _wave()
    N = 2 * TILE * W + 4096                         # N % 4 == 0: only the pointers decide the path
    _several_waves(N)
    d = _product(N, 300, seed=7)
    adv, ret = _run(d, 0.99, 0.95, layout=layout)
    _check(f"layout {layout}", d, adv, ret, 0.99, 0.95)


def test_n_not_multiple_of_4_multi_wave():
    W = _wave()
    N = 2 * TILE * W + 2049 + 2                     # N % 4 == 3 with aligned pointers: scalar path
    assert N % 4 != 0
    _several_waves(N)
    d = _product(N, 1000, seed=8)
    adv, ret = _run(d, 0.99, 0.95)
    _check("N % 4 != 0", d, adv, ret, 0.99, 0.95)


@pytest.mark.parametrize("pad", [4, 3])
def test_leading_dimension_larger_than_n(pad):
    """[C][ld] buffers through the C-ABI with ld = N + pad (ld % 4 == 0: vector path; otherwise scalar).  Columns
    [N, ld) of adv / ret hold a NaN sentinel that must survive, and NaN in the inputs' padding must not be read."""
    from fsrl_b200 import _lib, ops
    W = _wave()
    N = 2 * TILE * W + 4096
    ld = N + pad
    assert ld > N and (ld % 4 == 0) == (pad == 4)
    _several_waves(N)
    d = _product(N, 300, seed=9)
    nan = float("nan")

    def padded(a):
        t = torch.full((2, ld), nan, dtype=torch.float32, device="cuda")
        t[:, :N] = _cuda(a)
        return t
    v, vn = padded(d["v"]), padded(d["vnext"])
    adv, ret = torch.full((2, ld), nan, device="cuda"), torch.full((2, ld), nan, device="cuda")
    rew, cost = _cuda(d["rew"]), _cuda(d["cost"])
    end, term = _cuda(_end(d)), _cuda(d["terminated"].astype(np.uint8))
    need = _lib.lib.fsrl_gae_dual_workspace_bytes(N)
    ws = ops.workspace(need, v.device, "gae")
    _lib.check(_lib.lib.fsrl_gae_dual(v.data_ptr(), vn.data_ptr(), rew.data_ptr(), cost.data_ptr(), end.data_ptr(),
                                      term.data_ptr(), 0.99, 0.95, adv.data_ptr(), ret.data_ptr(), N, ld, 2,
                                      ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert torch.isnan(adv[:, N:]).all() and torch.isnan(ret[:, N:]).all()
    a, r = adv[:, :N].cpu().numpy(), ret[:, :N].cpu().numpy()
    _check(f"ld = N + {pad}", d, a, r, 0.99, 0.95)


# ---- modes ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["single_critic", "no_terminated", "unfinished_tails"])
def test_modes_multi_wave(mode):
    W = _wave()
    T = 1000
    N = 2 * TILE * W + 3 * T
    _several_waves(N)
    d = _product(N, T, seed=11, p_term=0.003)
    C, use_term = 2, True
    if mode == "single_critic":
        C = 1
    elif mode == "no_terminated":
        use_term = False
        assert d["terminated"].any()
    else:
        # every third env stops mid-episode: its last stored row carries the unfinished flag instead of an end
        last = np.arange(T - 1, N, T)[::3]
        d["truncated"][last] = False
        d["terminated"][last] = False
        d["unfinished"][last] = True
        assert d["unfinished"].sum() == len(last) > 100
    adv, ret = _run(d, 0.99, 0.95, C=C, use_term=use_term)
    _check(f"mode {mode}", d, adv, ret, 0.99, 0.95, C=C, use_term=use_term)


# ---- parameter edges ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma,lam", [(0.99, 0.0), (0.0, 0.95), (1.0, 1.0)])
def test_parameter_edges_multi_wave(gamma, lam):
    W = _wave()
    N = 2 * TILE * W + 2049
    _several_waves(N)
    d = _product(N, 300, seed=12)
    adv, ret = _run(d, gamma, lam)
    _check(f"gamma={gamma} lambda={lam}", d, adv, ret, gamma, lam)


# ---- workspace re-use and repeatability -----------------------------------------------------------------------------
def _dev_inputs(d):
    return (_cuda(d["v"]), _cuda(d["vnext"]), _cuda(d["rew"]), _cuda(d["cost"]), _cuda(_end(d)),
            _cuda(d["terminated"].astype(np.uint8)))


def _every_tile_has_an_end(d):
    """Every tile a look-back can reach holds an end flag, so its carry out is its own aggregate and the carry into
    each tile has one association.  The last tile in memory (ticket 0) is exempt: it publishes its inclusive value
    directly, with no carry in."""
    N = d["rew"].shape[0]
    e = np.zeros(_tiles(N) * TILE, bool)
    e[:N] = _end(d) != 0
    return bool(e.reshape(-1, TILE)[:-1].any(1).all())


def test_workspace_reuse_back_to_back():
    """large -> small -> large on one stream with no synchronisation in between: the grow-only "gae" workspace
    (ticket counter + tile descriptors) is re-zeroed by each call and must not leak state into the next.  Every
    tile holds an end flag, so each call's result is bit-reproducible and must equal a call made on its own."""
    from fsrl_b200 import ops
    W = _wave()
    sizes = [2 * TILE * W + 2049, 5000, 3 * TILE * W + 300]
    _several_waves(sizes[0]); _several_waves(sizes[2])
    ds = [_product(n, 300, seed=30 + k) for k, n in enumerate(sizes)]
    assert all(_every_tile_has_an_end(d) for d in ds)
    ins = [_dev_inputs(d) for d in ds]
    torch.cuda.synchronize()
    chained = [ops.gae_dual(*x, 0.99, 0.95) for x in ins]
    torch.cuda.synchronize()
    for k, (d, x, (adv, ret)) in enumerate(zip(ds, ins, chained)):
        a_alone, r_alone = ops.gae_dual(*x, 0.99, 0.95)
        torch.cuda.synchronize()
        assert torch.equal(adv, a_alone) and torch.equal(ret, r_alone), k
        _check(f"back-to-back call {k}", d, adv.cpu().numpy(), ret.cpu().numpy(), 0.99, 0.95)


def test_repeatable_when_every_tile_holds_an_end():
    """With an end flag in every tile the look-back stops at the first predecessor and the carry has one
    association, so repeated calls are bit-identical.  (Not asserted for segments that span tiles: there the carry
    comes from aggregates or from a predecessor's inclusive value depending on timing, and the two f64 associations
    may round differently; only the ulp bound against the oracle holds on every run.)"""
    W = _wave()
    N = 2048 * 1000
    _several_waves(N)
    d = _product(N, 1000, seed=40)
    assert _every_tile_has_an_end(d)
    runs = [_run(d, 0.99, 0.95) for _ in range(3)]
    for adv, ret in runs[1:]:
        assert np.array_equal(adv.view(np.int32), runs[0][0].view(np.int32))
        assert np.array_equal(ret.view(np.int32), runs[0][1].view(np.int32))
    _check("repeatability", d, *runs[0], 0.99, 0.95)


# ---- front-end validation -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["adv", "ret"])
def test_out_shape_is_validated(which):
    """An `out` buffer smaller than (C, N) is refused before anything is launched.  The undersized tensor is a view
    into a larger allocation with a sentinel tail, so an unchecked launch would write owned memory (and be caught by
    the sentinel) rather than fault."""
    from fsrl_b200 import ops
    N, short, sentinel = 10_000, 9_000, 12345.0
    d = _product(N, 300, seed=50)
    x = _dev_inputs(d)
    bufs = {}
    for nm in ("adv", "ret"):
        if nm == which:
            big = torch.full((2 * N + 64,), sentinel, device="cuda")
            bufs[nm] = (big, big[:2 * short].view(2, short))
        else:
            t = torch.full((2, N), sentinel, device="cuda")
            bufs[nm] = (t, t)
    with pytest.raises(ValueError, match="shape"):
        ops.gae_dual(*x, 0.99, 0.95, out=(bufs["adv"][1], bufs["ret"][1]))
    torch.cuda.synchronize()
    for nm, (owner, _) in bufs.items():
        assert bool((owner == sentinel).all()), nm
