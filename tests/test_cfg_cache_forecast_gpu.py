"""CFG cache Taylor forecast on the GPU: the three forecast kernels against torch fp32 restatements (bit for bit where the
restatement is exact, 1e-6 of fp64 for the sums), delta planted polynomial in sigma through the cache's own coefficients,
and the model: order 0 against the plain cache, threshold 0 against no cache, forced patterns against a restatement from
the model's own forwards, and GraphedStep against eager."""
import ctypes
import math

import numpy as np
import pytest
import torch

from test_cfg_cache_gpu import bits, f32, fwd_kw, pair, sampler_inputs, sentinel, small_model, step_ref, t32

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
# active slots -> coefficients (each an fp32 value); the other slots are 0 and hold NaN / inf sentinels
PATTERNS = {1: (0.0, 1.3125, 0.0), 2: (-0.75, 0.0, 1.8671875), 3: (0.3330078, -1.1, 1.7)}
PATTERNS = {k: [f32(c) for c in v] for k, v in PATTERNS.items()}


def forecast_ref(slots, coef):
    """delta_hat in torch fp32 ops in the kernel's order: t = c0*S0, then t + c1*S1, then t + c2*S2, zero slots skipped."""
    t = None
    for s, c in enumerate(coef):
        if c != 0.0:
            p = t32(c) * slots[s]
            t = p if t is None else t + p
    return torch.zeros_like(slots[0]) if t is None else t


def live_slots(shape, coef, g):
    """3 slots: random where the coefficient is non-zero, sentinels (NaN and inf encodings) elsewhere."""
    n = math.prod(shape)
    s = sentinel(3, n)
    for k, c in enumerate(coef):
        if c != 0.0:
            s[k] = torch.randn(n, generator=g, device="cuda") * 1.5
    return s.view(3, *shape)


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_delta_forecast_kernel(shape):
    from scail_b200 import ops
    v, g = pair(shape, 21 + sum(shape))
    partials = torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda")
    out = torch.zeros(4, device="cuda", dtype=torch.float64)
    want_new = (v[1].float() - v[0].float()).view(shape)
    for n_act, coef in PATTERNS.items():
        before = live_slots(shape, coef, g)
        t = forecast_ref(before, coef)
        num = float((want_new.double() - t.double()).abs().sum())
        den = float(t.double().abs().sum())
        for write in range(3):  # including a slot the forecast reads: it is read before it is written
            slots = before.clone()
            ops.cfg_cache_delta_forecast(v, slots, write, coef, partials, out)
            tag = (n_act, write)
            assert torch.equal(bits(slots[write]), bits(want_new)), tag
            for s in range(3):
                if s != write:
                    assert torch.equal(bits(slots[s]), bits(before[s])), (tag, s)
            got = out.tolist()
            assert abs(got[0] - num) <= 1e-6 * num and abs(got[1] - den) <= 1e-6 * den, (tag, got, num, den)
            assert got[2] == got[0] / got[1] and got[3] == 0.0
            first = out.clone()
            for _ in range(2):  # repeat launches are bit-identical
                ops.cfg_cache_delta_forecast(v, before.clone(), write, coef, partials, out)
                assert torch.equal(out.view(torch.int64), first.view(torch.int64)), tag
    # c = 1 on one slot alone: cfg_cache_delta's sums with d_ref = that slot, bit for bit
    d_ref = torch.randn(shape, generator=g, device="cuda")
    hold = torch.zeros(4, device="cuda", dtype=torch.float64)
    ops.cfg_cache_delta(v, d_ref, torch.empty(shape, device="cuda"), partials, hold)
    for s in range(3):
        slots = sentinel(3, math.prod(shape)).view(3, *shape)
        slots[s] = d_ref
        coef = [1.0 if k == s else 0.0 for k in range(3)]
        ops.cfg_cache_delta_forecast(v, slots, (s + 1) % 3, coef, partials, out)
        assert torch.equal(out.view(torch.int64), hold.view(torch.int64)), s
    # no active slot (the first full step): den = 0, +inf
    ops.cfg_cache_delta_forecast(v, sentinel(3, math.prod(shape)).view(3, *shape), 0, [0.0] * 3, partials, out)
    num0 = float(want_new.double().abs().sum())
    assert out[1].item() == 0.0 and out[2].item() == math.inf and abs(out[0].item() - num0) <= 1e-6 * num0


@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_cached_euler_forecast_kernel(shape):
    from scail_b200 import ops
    v, g = pair(shape, 31 + sum(shape))
    c = v[1:2].contiguous()
    x0 = torch.randn(shape, generator=g, device="cuda")
    s, ds = f32(4.0), f32(-0.0213)
    for n_act, coef in PATTERNS.items():
        slots = live_slots(shape, coef, g)
        u = c.float() - forecast_ref(slots, coef)
        want = x0 + t32(ds) * (u + t32(s) * (c.float() - u))
        x = x0.clone()
        ops.cfg_euler_cached_forecast_(x, c, slots, coef, s, ds)
        assert torch.equal(bits(x), bits(want)), n_act
        assert not torch.isnan(x).any(), n_act  # the sentinel slots were not read
    delta = torch.randn(shape, generator=g, device="cuda")
    slots = sentinel(3, math.prod(shape)).view(3, *shape)
    slots[0] = delta
    a, b = x0.clone(), x0.clone()
    ops.cfg_euler_cached_(a, c, delta, s, ds)
    ops.cfg_euler_cached_forecast_(b, c, slots, [1.0, 0.0, 0.0], s, ds)
    assert torch.equal(bits(a), bits(b))


@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_cached_unipc_forecast_kernel(shape):
    from scail_b200 import ops
    v, g = pair(shape, 41 + sum(shape))
    n = math.prod(shape)
    c = v[1:2].contiguous()
    x0, xl0 = torch.randn(shape, generator=g, device="cuda"), torch.randn(shape, generator=g, device="cuda")
    live = torch.randn(3, n, generator=g, device="cuda") * 0.5
    a, b = [f32(0.7), 0.0, f32(-0.2)], [f32(0.3), 0.0, f32(0.05)]
    coef = [f32(0.93), *a, f32(-0.41), f32(0.88), *b, f32(0.17)]
    before = sentinel(3, n)
    before[0], before[2] = live[0], live[2]
    scale, sigma = f32(4.0), f32(0.7312)
    for n_act, dcoef in PATTERNS.items():
        dslots = live_slots(shape, dcoef, g)
        u = c.float().reshape(-1) - forecast_ref(dslots, dcoef).reshape(-1)
        for correct in (True, False):
            want = step_ref(x0, xl0, u, c.float().reshape(-1), before, scale, sigma, coef, correct)
            x, xl, slots = x0.clone(), xl0.clone(), before.clone()
            ops.unipc_step_cached_forecast_(x, xl, c, dslots, dcoef, slots, 1, scale, sigma, coef, correct)
            tag = (n_act, correct)
            assert torch.equal(bits(x.view(-1)), bits(want[0])), tag
            assert torch.equal(bits(xl.view(-1)), bits(want[1])), tag
            assert torch.equal(bits(slots[1]), bits(want[2])), tag
            assert torch.equal(bits(slots[0]), bits(before[0])) and torch.equal(bits(slots[2]), bits(before[2])), tag
            assert not torch.isnan(x).any() and not torch.isnan(xl).any(), tag
    # c = (1, 0, 0) is the held-delta step bit for bit
    delta = torch.randn(shape, generator=g, device="cuda")
    dslots = sentinel(3, n).view(3, *shape)
    dslots[0] = delta
    outs = []
    for fc in (False, True):
        x, xl, slots = x0.clone(), xl0.clone(), before.clone()
        if fc:
            ops.unipc_step_cached_forecast_(x, xl, c, dslots, [1.0, 0.0, 0.0], slots, 1, scale, sigma, coef, True)
        else:
            ops.unipc_step_cached_(x, xl, c, delta, slots, 1, scale, sigma, coef, True)
        outs.append((x, xl, slots))
    for p, q in zip(*outs):
        assert torch.equal(bits(p), bits(q))


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("shape", LATENTS[:3], ids=ids)
def test_planted_polynomial_comes_back(shape, order):
    """delta_j = A + B sigma_j (+ C sigma_j^2 at order 2) in the slots, written in the cache's rotation at three full steps
    of a 50-step schedule; the forecast at a later sigma, through the cache's own coefficients and the Euler kernel (c = 0,
    scale 0, dsigma 1, x = 0: x = -delta_hat exactly), must be the polynomial there.
    Bound per element: with S_i = fp32(P(sigma_i)) (one rounding), c_i = fp32 of the fp64 coefficient (one rounding), one
    rounding per product and per sum (at most two sums), the error is at most 5 * 2^-24 * sum_i |c_i S_i| to first order;
    the assert allows 6 * 2^-24 * sum_i |c_i S_i|."""
    from scail_b200 import ops, sampler
    from scail_b200.step_cache import forecast_coefficients
    n = math.prod(shape)
    g = torch.Generator(device="cuda").manual_seed(order + sum(shape))
    A, B, C = (torch.randn(n, generator=g, device="cuda", dtype=torch.float64) for _ in range(3))
    if order == 1:
        C = torch.zeros_like(C)
    P = lambda s: A + B * s + C * s * s
    sig = [float(s) for s in sampler.make_flow_timesteps(50, 5.0)]
    full, at = [20, 22, 24, 26][:order + 2], 27  # order + 2 full steps: the slots have wrapped once
    slots = torch.zeros(order + 1, n, device="cuda")
    slot_sigma = [None] * (order + 1)
    for j, i in enumerate(full):
        slots[j % (order + 1)] = P(sig[i]).float()
        slot_sigma[j % (order + 1)] = sig[i]
    coef = forecast_coefficients(sig[at], slot_sigma, len(full), order)
    assert sum(c != 0.0 for c in coef) == order + 1
    x = torch.zeros(n, device="cuda")
    ops.cfg_euler_cached_forecast_(x, torch.zeros(n, device="cuda", dtype=torch.bfloat16), slots, coef, 0.0, 1.0)
    got = -x.double()
    want = P(sig[at])
    mag = sum(abs(c) * slots[k].double().abs() for k, c in enumerate(coef))
    err = (got - want).abs()
    assert (err <= 6 * 2.0 ** -24 * mag).all(), float((err / mag).max() * 2 ** 24)
    hold = (slots[(len(full) - 1) % (order + 1)].double() - want).abs()
    assert float(hold.max()) > 1e3 * float(err.max()), (float(hold.max()), float(err.max()))


def test_abi_refuses_bad_arguments():
    from scail_b200 import _lib
    n = 64
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    v = torch.zeros(2 * n + 8, device="cuda", dtype=torch.bfloat16)
    x, xl = torch.zeros(n + 8, device="cuda"), torch.zeros(n + 8, device="cuda")
    ds = torch.zeros(3, n + 8, device="cuda")
    us = torch.zeros(3, n + 8, device="cuda")
    part = torch.zeros(2048, device="cuda")
    out = torch.zeros(4, device="cuda", dtype=torch.float64)
    pv, px, pl, pd, pu, pp, po = (t.data_ptr() for t in (v, x, xl, ds, us, part, out))
    three = (ctypes.c_float * 3)(0.5, -0.25, 1.0)
    two = (ctypes.c_float * 3)(0.5, -0.25, 0.0)
    k10 = (ctypes.c_float * 10)(*([0.5] * 10))
    a3, a2, a10 = ctypes.addressof(three), ctypes.addressof(two), ctypes.addressof(k10)
    delta = lambda **kw: lib.scail_cfg_cache_delta_forecast(*[kw.get(k, dv) for k, dv in (
        ("v", pv), ("s", pd), ("stride", n + 8), ("n_slots", 3), ("write", 1), ("coef", a3), ("part", pp), ("plen", 2048),
        ("out", po), ("n", n))], st)
    euler = lambda **kw: lib.scail_cfg_euler_cached_forecast(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("c", pv), ("s", pd), ("stride", n + 8), ("n_slots", 3), ("coef", a3), ("n", n), ("scale", 4.0),
        ("ds", -0.1))], st)
    unipc = lambda **kw: lib.scail_unipc_step_cached_forecast(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("xl", pl), ("c", pv), ("s", pd), ("stride", n + 8), ("n_slots", 3), ("coef", a3), ("us", pu),
        ("ustride", n + 8), ("un", 3), ("write", 1), ("n", n), ("scale", 4.0), ("sigma", 0.5), ("correct", 1),
        ("ucoef", a10))], st)
    assert delta() == 0 and euler() == 0 and unipc() == 0
    torch.cuda.synchronize()
    cases = [
        (delta, dict(v=None), b"cfg_cache_delta_forecast: null"), (delta, dict(coef=None), b"cfg_cache_delta_forecast: null"),
        (delta, dict(s=pd + 4), b"16-byte aligned"), (delta, dict(v=pv + 8), b"16-byte aligned"),
        (delta, dict(part=pp + 2), b"4-byte"), (delta, dict(out=po + 4), b"8-byte"),
        (delta, dict(n=6), b"multiple of 4"), (delta, dict(n=0), b"multiple of 4"), (delta, dict(plen=1), b"partials holds"),
        (delta, dict(n_slots=0), b"1 <= n_slots <= 3"), (delta, dict(n_slots=4), b"1 <= n_slots <= 3"),
        (delta, dict(write=3), b"write_slot = 3"), (delta, dict(write=-1), b"write_slot = -1"),
        (delta, dict(stride=n - 4), b"slot_stride"), (delta, dict(stride=n + 2), b"slot_stride"),
        (delta, dict(n_slots=2, write=0), b"coefficient of delta slot 2 must be 0"),
        (euler, dict(s=None), b"cfg_euler_cached_forecast: null"), (euler, dict(x=px + 4), b"16-byte aligned"),
        (euler, dict(c=pv + 8), b"16-byte aligned"), (euler, dict(n=10), b"multiple of 4"),
        (euler, dict(n_slots=4), b"1 <= n_slots <= 3"), (euler, dict(stride=n - 4), b"slot_stride"),
        (euler, dict(n_slots=1), b"coefficient of delta slot 1 must be 0"),
        (unipc, dict(s=None), b"unipc_step_cached_forecast: null"), (unipc, dict(s=pd + 4), b"16-byte aligned"),
        (unipc, dict(n=6), b"multiple of 4"), (unipc, dict(n_slots=0), b"1 <= n_slots <= 3 delta slots"),
        (unipc, dict(stride=n - 4), b"delta slot_stride"), (unipc, dict(n_slots=2), b"coefficient of delta slot 2"),
        (unipc, dict(un=4), b"n_slots"), (unipc, dict(write=3), b"write_slot"),
    ]
    for fn, kw, msg in cases:
        assert fn(**kw) != 0, msg
        assert msg in lib.scail_last_error(), (msg, lib.scail_last_error())
    assert delta(n_slots=2, write=0, coef=a2) == 0 and euler(n_slots=2, coef=a2) == 0 and unipc(n_slots=2, coef=a2) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the model: a small 2-block DiT
def test_order_zero_is_the_plain_cache():
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    m = small_model(15)
    x0, cond, uc = sampler_inputs(15)
    outs, hists = [], []
    with torch.no_grad():
        for c in (CFGCache(0.3), CFGCache(0.3, order=0)):
            outs.append(sampler.sample(m, x0.clone(), cond, uc, num_steps=8, cfg_cache=c))
            hists.append(c.history)
    assert torch.equal(bits(outs[0]), bits(outs[1])) and hists[0] == hists[1]
    assert any(co for _, co in hists[0]), hists[0]


@pytest.mark.parametrize("solver", [None, 2], ids=["euler", "unipc2"])
@pytest.mark.parametrize("order", [1, 2])
def test_threshold_zero_is_bit_identical_to_no_cache(order, solver):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.unipc import UniPC
    m = small_model(16)
    x0, cond, uc = sampler_inputs(16)
    c = CFGCache(0.0, order=order)
    mk = lambda: UniPC(solver) if solver else None
    with torch.no_grad():
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, solver=mk())
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, solver=mk(), cfg_cache=c)
    assert torch.equal(bits(cached), bits(plain))
    assert [s for _, s in c.history] == [False] * 5 and c.history[0][0] is None and c.history[1][0] == math.inf
    assert all(math.isfinite(i) and i > 0 for i, _ in c.history[2:])


def restated_forecast_sample(m, x0, cond, uc, n, pattern, order, solver_order=None, scale=4.0):
    """sample() with CFGCache(order) restated from the model's own b = 2 and b = 1 forwards and torch fp32 ops: full steps
    keep delta_j = f32(c) - f32(u) in slot j mod (order + 1) with its sigma; conditional-only steps use u = c - delta_hat,
    delta_hat formed from the slots in slot order with forecast_coefficients."""
    from scail_b200 import ops, sampler, unipc
    from scail_b200.step_cache import forecast_coefficients
    sig = unipc.check_schedule(sampler.make_flow_timesteps(n, 5.0))
    ctx = sampler.prepare_context(cond, uc)
    kw = fwd_kw(cond)
    x = x0.clone()
    if solver_order is not None:
        x_last, uslots = torch.zeros_like(x0), torch.zeros(solver_order, x0.numel(), device="cuda")
    slots, slot_sigma, n_full = torch.zeros(order + 1, x0.numel(), device="cuda"), [None] * (order + 1), 0
    for i in range(n):
        if pattern[i]:
            ts = torch.full((1,), sig[i] * 1000.0, device="cuda")
            c = m(x, timesteps=ts, context=ctx[1:2], **kw)[0].float().reshape(-1)
            u = c - forecast_ref(slots, forecast_coefficients(sig[i], slot_sigma, n_full, order))
        else:
            ts = torch.full((2,), sig[i] * 1000.0, device="cuda")
            v = m(torch.cat([x, x], 0), timesteps=ts, context=ctx, **kw).contiguous()
            u, c = v[0].float().reshape(-1), v[1].float().reshape(-1)
            slots[n_full % (order + 1)] = c - u
            slot_sigma[n_full % (order + 1)] = sig[i]
            n_full += 1
        if solver_order is None:
            if pattern[i]:
                x = (x.reshape(-1) + t32(f32(sig[i + 1] - sig[i])) * (u + t32(scale) * (c - u))).view(x0.shape)
            else:
                ops.cfg_euler_(x, v, scale, sig[i + 1] - sig[i])
            continue
        k = unipc.step_coefficients(sig, i, solver_order)
        pad = [0.0] * (3 - solver_order)
        coef = [f32(cc) for cc in [k.x_last_c, *k.slot_c, *pad, k.m_c, k.y_c, *k.slot_p, *pad, k.m_p]]
        z, y, mm = step_ref(x, x_last, u, c, uslots, scale, sig[i], coef, k.correct)
        x, x_last = z.view(x0.shape), y.view(x0.shape)
        uslots[k.write] = mm
    return x


@pytest.mark.parametrize("solver", [None, 2], ids=["euler", "unipc2"])
@pytest.mark.parametrize("how", ["max_skips1", "thresholds"])
@pytest.mark.parametrize("order", [1, 2])
def test_forced_pattern_against_the_restatement(order, how, solver):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.unipc import UniPC
    m = small_model(17)
    x0, cond, uc = sampler_inputs(17)
    n = 9
    if how == "max_skips1":
        c, th = CFGCache(math.inf, max_skips=1, order=order), None
        pattern = [False, False, True, False, True, False, True, False, True]
    else:
        c = CFGCache(0.0, order=order)
        th = [math.inf, math.inf, math.inf, 0.0, 0.0, math.inf, 0.0, math.inf, math.inf]
        pattern = [i >= 2 and t == math.inf for i, t in enumerate(th)]
    sig = sampler.make_flow_timesteps(n, 5.0)
    s = None
    if solver:
        s = UniPC(solver)
        s.begin(sig)
    with torch.no_grad():
        x = x0.clone()
        for i in range(n):
            if th is not None:
                c.threshold = th[i]
            sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, solver=s, cfg_cache=c)
        want = restated_forecast_sample(m, x0, cond, uc, n, pattern, order, solver)
    assert [co for _, co in c.history] == pattern
    assert torch.equal(bits(x), bits(want))


@pytest.mark.parametrize("fast", [False, True], ids=["bf16", "fp8_window1_fbcache_unipc2"])
def test_graphed_step_is_bit_identical_to_eager(fast):
    from scail_b200 import dit, sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    kw = dict(fp8_linear=True, fp8_attention=True, attention_window=1) if fast else {}
    m = small_model(18, **kw)
    x0, cond, uc = sampler_inputs(18)
    n = 8
    sig = sampler.make_flow_timesteps(n, 5.0)
    ce, cg = CFGCache(math.inf, max_skips=1, order=2), CFGCache(math.inf, max_skips=1, order=2)
    se = sg = fe = fg = None
    if fast:
        se, sg = UniPC(2), UniPC(2)
        se.begin(sig)
        sg.begin(sig)
        fe, fg = FirstBlockCache(0.0, order=2), FirstBlockCache(0.0, order=2)
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, step_cache=fg, solver=sg, cfg_cache=cg)
        main = torch.cuda.current_stream().cuda_stream
        ws = {k: b.data_ptr() for k, b in dit._WS.bufs.items() if k[0][1] != main}  # the graphs' workspaces
        slots = None
        for i in range(n):
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=fe, solver=se, cfg_cache=ce)
            if i == 0:  # eager's b = 2 workspace
                ws.update({k: b.data_ptr() for k, b in dit._WS.bufs.items() if k[0][1] == main})
            gs(sig[i], sig[i + 1])
            if i == 0:
                slots = (ce.buffers.slots.data_ptr(), cg.buffers.slots.data_ptr())
            torch.cuda.synchronize()
            assert torch.equal(bits(xe), bits(xg)), f"step {i}"
    pattern = [False, False, True, False, True, False, True, False]
    assert [s for _, s in cg.history] == pattern and ce.history == cg.history
    if fast:  # the first-block cache decides on full steps only
        assert len(fg.history) == pattern.count(False) and fe.history == fg.history
    assert all(k in dit._WS.bufs and dit._WS.bufs[k].data_ptr() == p for k, p in ws.items())
    assert slots == (ce.buffers.slots.data_ptr(), cg.buffers.slots.data_ptr())
    assert ce.buffers.n_full == cg.buffers.n_full == pattern.count(False)
