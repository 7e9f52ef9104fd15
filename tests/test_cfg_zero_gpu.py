"""CFG-Zero* guidance on the GPU: the s* reduction in its three forms against fp64, bit-reproducible across launches and
streams; every scaled update bit for bit against a torch fp32 restatement (and at s* = 1 against its unscaled twin); and
the model: sample() against a restatement from the model's own forwards, the number of forwards, the CFG cache, the
first-block cache, GraphedStep and sample_long."""
import ctypes
import math

import numpy as np
import pytest
import torch

import cfg_zero_oracle as Z
from test_cfg_cache_forecast_gpu import PATTERNS, forecast_ref
from test_cfg_cache_gpu import bits, f32, fwd_kw, sampler_inputs, sentinel, small_model, step_ref, t32

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


# 512x512, 480x832 and 512x896 latents of 81 frames (21 latent frames), and small ragged ones
LATENTS = [(1, 21, 16, 64, 64), (1, 21, 16, 60, 104), (1, 21, 16, 64, 112), (1, 3, 16, 5, 7), (1, 1, 16, 1, 1)]
ids = lambda s: "x".join(map(str, s))


def bufs():
    from scail_b200 import ops
    return (torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda"), torch.zeros(4, device="cuda", dtype=torch.float64),
            torch.full((1,), math.nan, device="cuda"))


def corr_pair(shape, seed):
    """A bf16 CFG pair [2, ...] with c correlated with u, as the two branches of a real model are."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.randn(shape[1:], generator=g, device="cuda") * 2.0
    c = 0.8 * u + 0.6 * torch.randn(shape[1:], generator=g, device="cuda")
    return torch.stack([u, c]).to(torch.bfloat16), g


def forecast_slots(shape, coef, c, g):
    """3 delta slots whose forecast is about 0.3 c plus noise; sentinels (NaN and inf encodings) in unread slots."""
    n = math.prod(shape)
    s = sentinel(3, n)
    act = [k for k, cc in enumerate(coef) if cc != 0.0]
    for k in act:
        s[k] = 0.3 * c.float().reshape(-1) / (len(act) * coef[k]) + 0.3 * torch.randn(n, generator=g, device="cuda")
    return s.view(3, *shape)


def check_scale(u, c, out, s):
    """out and s against fp64 sums on the same fp32 u and c: within 1e-6 relative, and s* rounded once from out."""
    u64, c64 = u.double().reshape(-1), c.double().reshape(-1)
    dot, norm = float((c64 * u64).sum()), float((u64 * u64).sum())
    want = Z.optimized_scale(u.reshape(-1).cpu().numpy(), c.reshape(-1).cpu().numpy())
    o, got = out.tolist(), s.item()
    assert abs(o[0] - dot) <= 1e-6 * abs(dot) and abs(o[1] - norm) <= 1e-6 * norm, (o, dot, norm)
    assert o[2] == 0.0 and o[3] == 0.0
    assert abs(got - want) <= 1e-6 * abs(want), (got, want)
    assert got == f32(o[0] / (o[1] + 1e-8))


def reproducible(launch):
    """launch(partials, out, s) twice on this stream and once on another -> identical bits every time."""
    p, o, s = bufs()
    launch(p, o, s)
    first_o, first_s = o.clone(), s.clone()
    launch(p, o, s)
    assert torch.equal(o.view(torch.int64), first_o.view(torch.int64)) and torch.equal(bits(s), bits(first_s))
    side, main = torch.cuda.Stream(), torch.cuda.current_stream()
    p2, o2, s2 = bufs()
    side.wait_stream(main)
    with torch.cuda.stream(side):
        launch(p2, o2, s2)
    main.wait_stream(side)
    assert torch.equal(o2.view(torch.int64), first_o.view(torch.int64)) and torch.equal(bits(s2), bits(first_s))


# ---------------------------------------------------------------- the s* reduction
@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_scale_pair(shape):
    from scail_b200 import ops
    v, _ = corr_pair(shape, 31 + sum(shape))
    p, o, s = bufs()
    assert ops.cfg_zero_scale(v, p, o, s) is s
    check_scale(v[0].float(), v[1].float(), o, s)
    reproducible(lambda p, o, s: ops.cfg_zero_scale(v, p, o, s))


@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_scale_cached(shape):
    from scail_b200 import ops
    v, g = corr_pair(shape, 41 + sum(shape))
    c = v[1:2].contiguous()
    delta = 0.3 * c.float() + 0.4 * torch.randn(shape, generator=g, device="cuda")
    p, o, s = bufs()
    ops.cfg_zero_scale(c, p, o, s, delta=delta)
    check_scale(c.float() - delta, c.float(), o, s)
    reproducible(lambda p, o, s: ops.cfg_zero_scale(c, p, o, s, delta=delta))


@pytest.mark.parametrize("pattern", sorted(PATTERNS))
@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_scale_forecast(shape, pattern):
    from scail_b200 import ops
    v, g = corr_pair(shape, 51 + pattern + sum(shape))
    c = v[1:2].contiguous()
    coef = PATTERNS[pattern]
    slots = forecast_slots(shape, coef, c, g)
    p, o, s = bufs()
    ops.cfg_zero_scale(c, p, o, s, forecast=(slots, coef))
    check_scale(c.float() - forecast_ref(slots, coef), c.float(), o, s)
    reproducible(lambda p, o, s: ops.cfg_zero_scale(c, p, o, s, forecast=(slots, coef)))


def test_scale_zero_u_and_nan():
    from scail_b200 import ops
    shape = (1, 3, 16, 5, 7)
    v, g = corr_pair(shape, 61)
    p, o, s = bufs()
    z = v.clone()
    z[0] = 0
    ops.cfg_zero_scale(z, p, o, s)  # all-zero u: s* = 0 exactly, so the guided velocity is scale * c
    assert s.item() == 0.0 and o[1].item() == 0.0 and o[0].item() == 0.0
    c = v[1:2].contiguous()
    ops.cfg_zero_scale(c, p, o, s, delta=c.float())  # u = c - c = 0 in the cached form
    assert s.item() == 0.0
    ops.cfg_zero_scale(c, p, o, s, forecast=(torch.zeros(3, *shape, device="cuda"), [0.0, 0.0, 0.0]))  # u = c: s* = 1
    assert abs(s.item() - 1.0) <= 1e-6
    nan = v.clone()
    nan[1].view(-1)[5] = math.nan
    ops.cfg_zero_scale(nan, p, o, s)
    assert math.isnan(s.item()) and math.isnan(o[0].item())


# ---------------------------------------------------------------- the scaled updates
S_VALUES = (0.8173, 1.0, 0.0, -1.25)


@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_scaled_euler_kernels(shape):
    """The three scaled Euler steps bit for bit against torch fp32 ops in the stated order: u' = s u; g = u' + scale (c -
    u'); x = x + dsigma g.  At s = 1 the cached forms equal their unscaled kernels."""
    from scail_b200 import ops
    v, g = corr_pair(shape, 71 + sum(shape))
    c = v[1:2].contiguous()
    delta = torch.randn(shape, generator=g, device="cuda")
    x0 = torch.randn(shape, generator=g, device="cuda")
    coef = PATTERNS[2]
    slots = forecast_slots(shape, coef, c, g)
    d_hat = forecast_ref(slots, coef)
    for sv in S_VALUES:
        S = torch.full((1,), f32(sv), device="cuda")
        for scale, dsig in ((4.0, -0.0213), (7.5, -0.0003)):
            sc, ds = f32(scale), f32(dsig)
            combine = lambda u, cc: x0 + t32(ds) * (u + t32(sc) * (cc - u))
            x = x0.clone()
            ops.cfg_euler_(x, v, sc, ds, u_scale=S)
            assert torch.equal(bits(x), bits(combine(S * v[0].float(), v[1].float()))), ("pair", sv, scale)
            for name, run, u in (
                ("cached", lambda x, **k: ops.cfg_euler_cached_(x, c, delta, sc, ds, **k), c.float() - delta),
                ("forecast", lambda x, **k: ops.cfg_euler_cached_forecast_(x, c, slots, coef, sc, ds, **k), c.float() - d_hat),
            ):
                x = x0.clone()
                run(x, u_scale=S)
                assert torch.equal(bits(x), bits(combine(S * u, c.float()))), (name, sv, scale)
                if sv == 1.0:
                    x1 = x0.clone()
                    run(x1)
                    assert torch.equal(bits(x), bits(x1)), (name, "s = 1")
                assert not torch.isnan(x).any(), name


ACTIVE = {1: [0], 2: [0, 2], 3: [0, 1, 2]}


@pytest.mark.parametrize("shape", LATENTS[:4], ids=ids)
def test_scaled_unipc_kernels(shape):
    """The three scaled UniPC steps bit for bit against step_ref on u' = s u, NaN sentinels in slots with zero
    coefficients; at s = 1 each equals its unscaled instantiation."""
    from scail_b200 import ops
    v, g = corr_pair(shape, 81 + sum(shape))
    n = math.prod(shape)
    c = v[1:2].contiguous()
    delta = torch.randn(shape, generator=g, device="cuda")
    dcoef = PATTERNS[3]
    dslots = forecast_slots(shape, dcoef, c, g)
    x0, xl0 = torch.randn(shape, generator=g, device="cuda"), torch.randn(shape, generator=g, device="cuda")
    live = torch.randn(3, n, generator=g, device="cuda") * 0.5
    cf = c.float().reshape(-1)
    forms = {
        "pair": (v[0].float().reshape(-1), v[1].float().reshape(-1),
                 lambda *a, **k: ops.unipc_step_(a[0], a[1], v, *a[2:], **k)),
        "cached": (cf - delta.reshape(-1), cf, lambda *a, **k: ops.unipc_step_cached_(a[0], a[1], c, delta, *a[2:], **k)),
        "forecast": (cf - forecast_ref(dslots, dcoef).reshape(-1), cf,
                     lambda *a, **k: ops.unipc_step_cached_forecast_(a[0], a[1], c, dslots, dcoef, *a[2:], **k)),
    }
    for form, (u, cc, run) in forms.items():
        for n_act, act in ACTIVE.items():
            for correct in (True, False):
                a, b = [0.0] * 3, [0.0] * 3
                for j, s in enumerate(act):
                    a[s] = f32(0.7 - 0.45 * j)
                    b[s] = 0.0 if (j == 0 and n_act > 1) else f32(-0.3 + 0.55 * j)
                coef = [f32(0.93), *a, f32(-0.41), f32(0.88), *b, f32(0.17)]
                before = sentinel(3, n)
                for s in act:
                    before[s] = live[s]
                write, scale, sigma = 2, f32(4.0), f32(0.7312)
                for sv in (0.8173, 1.0):
                    S = torch.full((1,), f32(sv), device="cuda")
                    want = step_ref(x0, xl0, S * u, cc, before, scale, sigma, coef, correct)
                    x, xl, slots = x0.clone(), xl0.clone(), before.clone()
                    run(x, xl, slots, write, scale, sigma, coef, correct, u_scale=S)
                    tag = (form, n_act, correct, sv)
                    assert torch.equal(bits(x.view(-1)), bits(want[0])), tag
                    assert torch.equal(bits(xl.view(-1)), bits(want[1])), tag
                    assert torch.equal(bits(slots[write]), bits(want[2])), tag
                    for s in range(2):
                        assert torch.equal(bits(slots[s]), bits(before[s])), (tag, s)
                    assert not torch.isnan(x).any() and not torch.isnan(xl).any(), tag
                    if sv == 1.0:
                        x1, xl1, slots1 = x0.clone(), xl0.clone(), before.clone()
                        run(x1, xl1, slots1, write, scale, sigma, coef, correct)
                        assert torch.equal(bits(x), bits(x1)) and torch.equal(bits(xl), bits(xl1)), tag
                        assert torch.equal(bits(slots), bits(slots1)), tag


def test_abi_refuses_bad_arguments():
    from scail_b200 import _lib
    n = 64
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    v = torch.zeros(2 * n + 8, device="cuda", dtype=torch.bfloat16)
    x, d, xl = (torch.zeros(n + 8, device="cuda") for _ in range(3))
    slots = torch.zeros(3, n + 8, device="cuda")
    part = torch.zeros(2048, device="cuda")
    out = torch.zeros(4, device="cuda", dtype=torch.float64)
    us = torch.ones(2, device="cuda")
    pv, px, pd, pxl, pp, po, ps = (t.data_ptr() for t in (v, x, d, xl, part, out, us))
    dk = (ctypes.c_float * 3)(0.5, 0.0, 0.0)
    ok = (ctypes.c_float * 10)(*([0.5] * 10))
    scale = lambda **kw: lib.scail_cfg_zero_scale(*[kw.get(k, dv) for k, dv in (
        ("form", 2), ("v", pv), ("d", slots.data_ptr()), ("stride", n + 8), ("n_d", 3), ("dk", ctypes.addressof(dk)),
        ("part", pp), ("plen", 2048), ("out", po), ("s", ps), ("n", n))], st)
    euler = lambda **kw: lib.scail_cfg_euler_scaled(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("v", pv), ("n", n), ("sc", 4.0), ("ds", -0.1), ("s", ps))], st)
    cached = lambda **kw: lib.scail_cfg_euler_cached_scaled(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("c", pv), ("d", pd), ("n", n), ("sc", 4.0), ("ds", -0.1), ("s", ps))], st)
    fcast = lambda **kw: lib.scail_cfg_euler_cached_forecast_scaled(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("c", pv), ("d", slots.data_ptr()), ("stride", n + 8), ("n_d", 3), ("dk", ctypes.addressof(dk)),
        ("n", n), ("sc", 4.0), ("ds", -0.1), ("s", ps))], st)
    unipc = lambda **kw: lib.scail_unipc_step_scaled(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("xl", pxl), ("v", pv), ("slots", slots.data_ptr()), ("stride", n + 8), ("n_slots", 3), ("write", 1),
        ("n", n), ("sc", 4.0), ("sigma", 0.5), ("correct", 1), ("coef", ctypes.addressof(ok)), ("s", ps))], st)
    ucached = lambda **kw: lib.scail_unipc_step_cached_scaled(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("xl", pxl), ("c", pv), ("d", pd), ("slots", slots.data_ptr()), ("stride", n + 8), ("n_slots", 3),
        ("write", 1), ("n", n), ("sc", 4.0), ("sigma", 0.5), ("correct", 1), ("coef", ctypes.addressof(ok)), ("s", ps))], st)
    ufcast = lambda **kw: lib.scail_unipc_step_cached_forecast_scaled(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("xl", pxl), ("c", pv), ("d", slots.data_ptr()), ("dstride", n + 8), ("n_d", 3),
        ("dk", ctypes.addressof(dk)), ("slots", slots.data_ptr()), ("stride", n + 8), ("n_slots", 3), ("write", 1),
        ("n", n), ("sc", 4.0), ("sigma", 0.5), ("correct", 1), ("coef", ctypes.addressof(ok)), ("s", ps))], st)
    for form in (0, 1, 2):
        assert scale(form=form) == 0, lib.scail_last_error()
    assert euler() == 0 and cached() == 0 and fcast() == 0 and unipc() == 0 and ucached() == 0 and ufcast() == 0
    torch.cuda.synchronize()
    cases = [
        (scale, dict(form=3), b"form = 3"), (scale, dict(form=-1), b"form = -1"), (scale, dict(v=None), b"cfg_zero_scale: null"),
        (scale, dict(s=None), b"cfg_zero_scale: null"), (scale, dict(out=None), b"cfg_zero_scale: null"),
        (scale, dict(form=1, d=None), b"null delta"), (scale, dict(dk=None), b"null dcoef"),
        (scale, dict(v=pv + 8), b"16-byte aligned"), (scale, dict(form=1, d=pd + 4), b"16-byte aligned"),
        (scale, dict(s=ps + 2), b"4-byte"), (scale, dict(out=po + 4), b"8-byte"), (scale, dict(part=pp + 2), b"4-byte"),
        (scale, dict(n=6), b"multiple of 4"), (scale, dict(n=0), b"multiple of 4"), (scale, dict(plen=1), b"partials holds"),
        (scale, dict(n_d=4), b"delta slots"), (scale, dict(stride=n - 4), b"slot_stride"),
        (euler, dict(s=None), b"cfg_euler_scaled: null u_scale"), (euler, dict(s=ps + 2), b"u_scale must be 4-byte"),
        (euler, dict(x=px + 4), b"16-byte aligned"), (euler, dict(n=10), b"multiple of 4"),
        (cached, dict(s=None), b"cfg_euler_cached_scaled: null u_scale"), (cached, dict(d=None), b"cfg_euler_cached_scaled: null"),
        (cached, dict(n=6), b"multiple of 4"),
        (fcast, dict(s=None), b"cfg_euler_cached_forecast_scaled: null u_scale"), (fcast, dict(n_d=0), b"delta slots"),
        (unipc, dict(s=None), b"unipc_step_scaled: null u_scale"), (unipc, dict(write=3), b"write_slot"),
        (unipc, dict(n_slots=4), b"n_slots"),
        (ucached, dict(s=None), b"unipc_step_cached_scaled: null u_scale"), (ucached, dict(d=pd + 4), b"16-byte aligned"),
        (ufcast, dict(s=None), b"unipc_step_cached_forecast_scaled: null u_scale"), (ufcast, dict(n_d=4), b"delta slots"),
    ]
    for fn, kw, msg in cases:
        assert fn(**kw) != 0, msg
        assert msg in lib.scail_last_error(), (msg, lib.scail_last_error())
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the model: a small 2-block DiT
def count_forwards(m):
    """Wrap m.forward; the returned list gets the batch size of every forward."""
    calls, f = [], m.forward

    def fwd(x, *a, **kw):
        calls.append(x.shape[0])
        return f(x, *a, **kw)

    m.forward = fwd
    return calls


def restated_sample(m, x0, cond, uc, n, k, solver_order=None, cache_order=None, scale=4.0):
    """sample(..., guidance=CFGZeroStar(k)) restated from the model's own forwards and torch fp32 ops.  Steps 0 .. k-1:
    nothing with Euler, the solver step on u = c = 0 with UniPC.  Later steps: s* from the product's reduction on the u the
    step forms (checked against fp64 above), u' = s* u, then the combine.  With cache_order (0 or 2) the steps after the
    zero-initialised ones follow CFGCache(inf, max_skips=1): two full steps, then conditional-only and full in turn."""
    from scail_b200 import ops, sampler, unipc
    from scail_b200.step_cache import forecast_coefficients
    sig = unipc.check_schedule(sampler.make_flow_timesteps(n, 5.0))
    ctx = sampler.prepare_context(cond, uc)
    kw = fwd_kw(cond)
    x, N = x0.clone(), x0.numel()
    p, o, s = bufs()
    if solver_order is not None:
        x_last, uslots = torch.zeros_like(x0), torch.zeros(solver_order, N, device="cuda")
    if cache_order:
        slots, slot_sigma, n_full = torch.zeros(cache_order + 1, N, device="cuda"), [None] * (cache_order + 1), 0
    for i in range(n):
        j = i - k
        if j < 0:
            if solver_order is None:
                continue
            u = cc = torch.zeros(N, device="cuda")
        elif cache_order is not None and j >= 2 and j % 2 == 0:
            ts = torch.full((1,), sig[i] * 1000.0, device="cuda")
            c16 = m(x, timesteps=ts, context=ctx[1:2], **kw).contiguous()
            cc = c16[0].float().reshape(-1)
            if cache_order == 0:
                d = delta
                ops.cfg_zero_scale(c16, p, o, s, delta=delta.view(x0.shape))
            else:
                fc = forecast_coefficients(sig[i], slot_sigma, n_full, cache_order)
                d = forecast_ref(slots, fc)
                ops.cfg_zero_scale(c16, p, o, s, forecast=(slots, fc))
            u = s.clone() * (cc - d)
        else:
            ts = torch.full((2,), sig[i] * 1000.0, device="cuda")
            v = m(torch.cat([x, x], 0), timesteps=ts, context=ctx, **kw).contiguous()
            u, cc = v[0].float().reshape(-1), v[1].float().reshape(-1)
            if cache_order == 0:
                delta = cc - u
            elif cache_order:
                slots[n_full % (cache_order + 1)] = cc - u
                slot_sigma[n_full % (cache_order + 1)] = sig[i]
                n_full += 1
            ops.cfg_zero_scale(v, p, o, s)
            u = s.clone() * u
        if solver_order is None:
            x = (x.reshape(-1) + t32(f32(sig[i + 1] - sig[i])) * (u + t32(scale) * (cc - u))).view(x0.shape)
            continue
        kk = unipc.step_coefficients(sig, i, solver_order)
        pad = [0.0] * (3 - solver_order)
        coef = [f32(c_) for c_ in [kk.x_last_c, *kk.slot_c, *pad, kk.m_c, kk.y_c, *kk.slot_p, *pad, kk.m_p]]
        z, y, mm = step_ref(x, x_last, u, cc, uslots, scale, sig[i], coef, kk.correct)
        x, x_last = z.view(x0.shape), y.view(x0.shape)
        uslots[kk.write] = mm
    return x


@pytest.mark.parametrize("solver", [None, 1, 2, 3], ids=["euler", "unipc1", "unipc2", "unipc3"])
@pytest.mark.parametrize("k", [0, 1, 2])
def test_sample_against_the_restatement(k, solver):
    from scail_b200 import sampler
    from scail_b200.guidance import CFGZeroStar
    from scail_b200.unipc import UniPC
    m = small_model(20)
    x0, cond, uc = sampler_inputs(20)
    n = 5
    g = CFGZeroStar(k)
    calls = count_forwards(m)
    with torch.no_grad():
        got = sampler.sample(m, x0.clone(), cond, uc, num_steps=n, solver=UniPC(solver) if solver else None, guidance=g)
        assert calls == [2] * (n - k)
        want = restated_sample(m, x0, cond, uc, n, k, solver_order=solver)
    assert g.step_index == n and g.last_scale is not None and math.isfinite(g.last_scale.item())
    assert torch.equal(bits(got), bits(want))
    assert not torch.isnan(got).any()


@pytest.mark.parametrize("solver", [None, 2], ids=["euler", "unipc2"])
@pytest.mark.parametrize("order", [0, 2])
def test_cfg_cache_against_the_restatement(order, solver):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import CFGZeroStar
    from scail_b200.unipc import UniPC
    m = small_model(21)
    x0, cond, uc = sampler_inputs(21)
    n, k = 8, 1
    c = CFGCache(math.inf, max_skips=1, order=order)
    with torch.no_grad():
        got = sampler.sample(m, x0.clone(), cond, uc, num_steps=n, solver=UniPC(solver) if solver else None, cfg_cache=c,
                             guidance=CFGZeroStar(k))
        want = restated_sample(m, x0, cond, uc, n, k, solver_order=solver, cache_order=order)
    # the zero-initialised step is not in the cache's history
    assert [s for _, s in c.history] == [False, False, True, False, True, False, True]
    assert torch.equal(bits(got), bits(want))


def test_first_block_cache_at_zero_equals_no_cache():
    from scail_b200 import sampler
    from scail_b200.guidance import CFGZeroStar
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    m = small_model(22)
    x0, cond, uc = sampler_inputs(22)
    fb = FirstBlockCache(0.0)
    with torch.no_grad():
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, solver=UniPC(2), guidance=CFGZeroStar(1))
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, solver=UniPC(2), guidance=CFGZeroStar(1), step_cache=fb)
    assert torch.equal(bits(cached), bits(plain))
    assert len(fb.history) == 4  # the zero-initialised step ran no head


@pytest.mark.parametrize("how", ["euler", "cfgcache_unipc2"])
def test_graphed_step_is_bit_identical_to_eager(how):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import CFGZeroStar
    from scail_b200.unipc import UniPC
    m = small_model(23)
    x0, cond, uc = sampler_inputs(23)
    n = 7
    sig = sampler.make_flow_timesteps(n, 5.0)
    ge, gg = CFGZeroStar(1), CFGZeroStar(1)
    se = sg = ce = cg = None
    if how != "euler":
        se, sg = UniPC(2), UniPC(2)
        se.begin(sig)
        sg.begin(sig)
        ce, cg = CFGCache(math.inf, max_skips=1), CFGCache(math.inf, max_skips=1)
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, solver=sg, cfg_cache=cg, guidance=gg)
        for i in range(n):
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, solver=se, cfg_cache=ce, guidance=ge)
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(bits(xe), bits(xg)), f"step {i}"
            if i == 0:
                assert torch.equal(bits(xg), bits(x0)) or se is not None  # Euler leaves x as it is on a zero step
    assert ge.step_index == gg.step_index == n
    if ce is not None:
        assert [s for _, s in cg.history] == [False, False, True, False, True, False] and ce.history == cg.history


def test_sample_long_against_a_per_window_restatement():
    from scail_b200 import ops, sampler
    from scail_b200.guidance import CFGZeroStar
    m = small_model(24)
    gen = torch.Generator().manual_seed(24)
    r = lambda *s: torch.randn(*s, generator=gen).to(torch.bfloat16).cuda()
    T, seg, h, w, n, k = 5, 3, 16, 16, 3, 1
    tiles = sampler.make_tile_indices(T, seg, 2)
    x0 = torch.randn(1, T, 16, h, w, generator=gen).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, h, w), image_clip_features=r(1, 257, 1280),
                smpl_tiled=r(1, len(tiles), seg, 16, h // 2, w // 2))
    uc = dict(crossattn=r(1, 20, 64))
    ctx = sampler.prepare_context(cond, uc)
    p, o, s = bufs()
    scales = []

    def denoise(x_tile, sigma, c_k, u_k):  # one window: the b = 2 forward, its own s*, the combine in torch fp32 ops
        x_tile = x_tile.contiguous()
        ts = torch.full((2,), float(sigma) * 1000.0, device="cuda")
        v = m(torch.cat([x_tile, x_tile], 0), timesteps=ts, context=ctx, **fwd_kw(c_k)).contiguous()
        ops.cfg_zero_scale(v, p, o, s)
        scales.append(s.item())
        u, c = s.clone() * v[0].float(), v[1].float()
        return torch.zeros_like(x_tile) + t32(1.0) * (u + t32(4.0) * (c - u))

    with torch.no_grad():
        got = sampler.sample_long(m, x0.clone(), cond, uc, tiles, num_steps=n, guidance=CFGZeroStar(k))
        sig = sampler.make_flow_timesteps(n, 5.0).cuda()
        want = x0.clone()
        for i in range(k, n):
            want = sampler.sampler_step_long(denoise, want, sig[i], sig[i + 1], tiles, cond["smpl_tiled"], dict(cond), dict(uc))
    assert len(scales) == (n - k) * len(tiles) and len(set(scales)) == len(scales)  # every window has its own s*
    assert torch.equal(bits(got), bits(want))
