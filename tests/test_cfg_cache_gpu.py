"""CFG cache on the GPU: the three kernels against torch fp32 restatements, bit for bit; the b = 1 conditional forward
against row 1 of the b = 2 forward in every attention and linear mode; sample() against a restatement built from the
model's own forwards; GraphedStep against eager sampler_step."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def bits(t):
    return t.contiguous().view(torch.int32)


def f32(c):
    return float(np.float32(c))


def t32(c):
    return torch.tensor(c, dtype=torch.float32, device="cuda")


# 512x512, 480x832 and 512x896 latents of 81 frames (21 latent frames), and small ragged ones
LATENTS = [(1, 21, 16, 64, 64), (1, 21, 16, 60, 104), (1, 21, 16, 64, 112), (1, 3, 16, 5, 7), (1, 1, 16, 1, 1)]
ids = lambda s: "x".join(map(str, s))


def pair(shape, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(2, *shape[1:], generator=g, device="cuda") * 2.0).to(torch.bfloat16), g


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_delta_kernel(shape):
    from scail_b200 import ops
    v, g = pair(shape, sum(shape))
    n = math.prod(shape)
    d_ref = torch.randn(shape, generator=g, device="cuda")
    d_new = torch.full(shape, math.nan, device="cuda")
    partials = torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda")
    out = torch.zeros(4, device="cuda", dtype=torch.float64)
    want = v[1].float() - v[0].float()
    ops.cfg_cache_delta(v, d_ref, d_new, partials, out)
    assert torch.equal(bits(d_new), bits(want.view(shape)))
    num = float((want.double() - d_ref[0].double()).abs().sum())
    den = float(d_ref.double().abs().sum())
    got = out.tolist()
    assert abs(got[0] - num) <= 1e-6 * num and abs(got[1] - den) <= 1e-6 * den, (got, num, den)
    assert got[2] == got[0] / got[1] and got[3] == 0.0
    first = out.clone()
    for _ in range(2):  # repeat launches are bit-identical
        ops.cfg_cache_delta(v, d_ref, d_new, partials, out)
        assert torch.equal(out.view(torch.int64), first.view(torch.int64))
    ops.cfg_cache_delta(v, torch.zeros_like(d_ref), d_new, partials, out)  # a zero delta_ref: the first full step
    num0 = float(want.double().abs().sum())
    assert out[2].item() == math.inf and out[1].item() == 0.0 and abs(out[0].item() - num0) <= 1e-6 * num0
    assert n % 4 == 0


@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_cached_euler_kernel(shape):
    from scail_b200 import ops
    v, g = pair(shape, 3 + sum(shape))
    c = v[1:2].contiguous()
    delta = torch.randn(shape, generator=g, device="cuda")
    x0 = torch.randn(shape, generator=g, device="cuda")
    for scale, dsig in ((4.0, -0.0213), (1.0, -1.0), (7.5, -0.0003)):
        s, ds = f32(scale), f32(dsig)
        u = c.float() - delta
        gv = u + t32(s) * (c.float() - u)
        want = x0 + t32(ds) * gv
        x = x0.clone()
        ops.cfg_euler_cached_(x, c, delta, s, ds)
        assert torch.equal(bits(x), bits(want)), (scale, dsig)


def step_ref(x, x_last, u, c, slots, scale, sigma, coef, correct):
    """The UniPC step as separate torch fp32 ops in the kernel's order, from u and c (fp32, flat) -> (z, y, m)."""
    a_x, a, a_m, b_y, b, b_m = coef[0], coef[1:4], coef[4], coef[5], coef[6:9], coef[9]
    g = u + t32(scale) * (c - u)
    m = x.reshape(-1) - t32(sigma) * g
    if correct:
        y = t32(a_x) * x_last.reshape(-1)
        for s in range(slots.shape[0]):
            if a[s] != 0.0:
                y = y + t32(a[s]) * slots[s]
        y = y + t32(a_m) * m
    else:
        y = x.reshape(-1).clone()
    z = t32(b_y) * y
    for s in range(slots.shape[0]):
        if b[s] != 0.0:
            z = z + t32(b[s]) * slots[s]
    z = z + t32(b_m) * m
    return z, y, m


def sentinel(rows, n):
    """A fixed bit pattern with many NaN and inf encodings (compared as bits)."""
    ar = torch.arange(rows * n, device="cuda", dtype=torch.int64)
    pat = ((ar * 2654435761) & 0x7FFFFFFF).to(torch.int32) ^ 0x7F800001
    return pat.view(torch.float32).view(rows, n)


ACTIVE = {1: [0], 2: [0, 2], 3: [0, 1, 2]}


@pytest.mark.parametrize("shape", LATENTS[:4], ids=ids)
def test_cached_unipc_kernel(shape):
    from scail_b200 import ops
    v, g = pair(shape, 7 + sum(shape))
    n = math.prod(shape)
    c = v[1:2].contiguous()
    delta = torch.randn(shape, generator=g, device="cuda")
    x0, xl0 = torch.randn(shape, generator=g, device="cuda"), torch.randn(shape, generator=g, device="cuda")
    live = torch.randn(3, n, generator=g, device="cuda") * 0.5
    u = c.float().reshape(-1) - delta.reshape(-1)
    for n_act, act in ACTIVE.items():
        n_slots = 3
        for correct in (True, False):
            a, b = [0.0] * 3, [0.0] * 3
            for j, s in enumerate(act):
                a[s] = f32(0.7 - 0.45 * j)
                b[s] = 0.0 if (j == 0 and n_act > 1) else f32(-0.3 + 0.55 * j)
            coef = [f32(0.93), *a, f32(-0.41), f32(0.88), *b, f32(0.17)]
            before = sentinel(n_slots, n)  # NaN sentinels in the slots whose coefficients are 0
            for s in act:
                before[s] = live[s]
            write = n_slots - 1
            scale, sigma = f32(4.0), f32(0.7312)
            want = step_ref(x0, xl0, u, c.float().reshape(-1), before, scale, sigma, coef, correct)
            x, xl, slots = x0.clone(), xl0.clone(), before.clone()
            ops.unipc_step_cached_(x, xl, c, delta, slots, write, scale, sigma, coef, correct)
            tag = (n_act, correct)
            assert torch.equal(bits(x.view(-1)), bits(want[0])), tag
            assert torch.equal(bits(xl.view(-1)), bits(want[1])), tag
            assert torch.equal(bits(slots[write]), bits(want[2])), tag
            for s in range(n_slots - 1):
                assert torch.equal(bits(slots[s]), bits(before[s])), (tag, s)
            assert not torch.isnan(x).any() and not torch.isnan(xl).any(), tag


@pytest.mark.parametrize("shape", LATENTS[:4], ids=ids)
def test_cached_unipc_equals_the_pair_step_where_delta_is_exact(shape):
    from scail_b200 import ops
    v, g = pair(shape, 11 + sum(shape))
    n = math.prod(shape)
    # planted elements whose bf16 c and u differ by more than 2^16 in magnitude: f32(c) - f32(u) rounds there
    planted = torch.arange(0, n, max(1, n // 7), device="cuda")[:6]
    vf = v.view(2, -1)
    vf[0, planted] = torch.tensor([1.0, -3.0, 2.0 ** -20, 5.5, -1.0, 0.75], device="cuda").to(torch.bfloat16)[:planted.numel()]
    vf[1, planted] = torch.tensor([2.0 ** 20, 2.0 ** 18 * 1.5, 3.0, -2.0 ** 24, 2.0 ** 25, -2.0 ** 17], device="cuda"
                                  ).to(torch.bfloat16)[:planted.numel()]
    u, c = vf[0].float(), vf[1].float()
    delta = torch.empty(shape, device="cuda")
    ops.cfg_cache_delta(v, torch.zeros_like(delta), delta, torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda"),
                        torch.zeros(4, device="cuda", dtype=torch.float64))
    exact = (c - delta.view(-1)) == u
    inexact = (~exact).nonzero().view(-1)
    big = (c.abs() > u.abs() * 2.0 ** 16) | (u.abs() > c.abs() * 2.0 ** 16)
    assert big[inexact].all(), "the only elements where c - (c - u) != u are those with |c| and |u| 2^16 apart"
    assert inexact.numel() >= 1
    x0, xl0 = torch.randn(shape, generator=g, device="cuda"), torch.randn(shape, generator=g, device="cuda")
    slots0 = torch.randn(2, n, generator=g, device="cuda")
    coef = [f32(0.93), f32(0.3), f32(-0.2), 0.0, f32(-0.41), f32(0.88), f32(0.1), f32(0.05), 0.0, f32(0.17)]
    outs = []
    for cached in (False, True):
        x, xl, sl = x0.clone(), xl0.clone(), slots0.clone()
        if cached:
            ops.unipc_step_cached_(x, xl, v[1:2].contiguous(), delta, sl, 1, 4.0, 0.61, coef, True)
        else:
            ops.unipc_step_(x, xl, v, sl, 1, 4.0, 0.61, coef, True)
        outs.append((x.view(-1), xl.view(-1), sl[1]))
    for p, q in zip(*outs):  # x, x_last and the written slot agree wherever delta was exact
        assert (bits(p) == bits(q))[exact].all()


def test_abi_refuses_bad_arguments():
    import ctypes
    from scail_b200 import _lib
    n = 64
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    v = torch.zeros(2 * n + 8, device="cuda", dtype=torch.bfloat16)
    x, d0, d1 = (torch.zeros(n + 8, device="cuda") for _ in range(3))
    part = torch.zeros(2048, device="cuda")
    out = torch.zeros(4, device="cuda", dtype=torch.float64)
    pv, px, p0, p1, pp, po = (t.data_ptr() for t in (v, x, d0, d1, part, out))
    delta = lambda **kw: lib.scail_cfg_cache_delta(*[kw.get(k, dv) for k, dv in (
        ("v", pv), ("ref", p0), ("new", p1), ("part", pp), ("plen", 2048), ("out", po), ("n", n))], st)
    euler = lambda **kw: lib.scail_cfg_euler_cached(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("c", pv), ("d", p0), ("n", n), ("s", 4.0), ("ds", -0.1))], st)
    slots = torch.zeros(3, n + 8, device="cuda")
    ok = (ctypes.c_float * 10)(*([0.5] * 10))
    two = (ctypes.c_float * 10)(*([0.5] * 3 + [0.0] + [0.5] * 4 + [0.0, 0.5]))
    unipc = lambda **kw: lib.scail_unipc_step_cached(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("xl", p1), ("c", pv), ("d", p0), ("s", slots.data_ptr()), ("stride", n + 8), ("n_slots", 3), ("write", 1),
        ("n", n), ("scale", 4.0), ("sigma", 0.5), ("correct", 1), ("coef", ctypes.addressof(ok)))], st)
    assert delta() == 0 and euler() == 0 and unipc() == 0
    torch.cuda.synchronize()
    cases = [
        (delta, dict(v=None), b"cfg_cache_delta: null"), (delta, dict(out=None), b"cfg_cache_delta: null"),
        (delta, dict(ref=p0 + 4), b"16-byte aligned"), (delta, dict(v=pv + 8), b"16-byte aligned"),
        (delta, dict(part=pp + 2), b"4-byte"), (delta, dict(out=po + 4), b"8-byte"),
        (delta, dict(n=6), b"multiple of 4"), (delta, dict(n=0), b"multiple of 4"), (delta, dict(plen=1), b"partials holds"),
        (euler, dict(d=None), b"cfg_euler_cached: null"), (euler, dict(x=px + 4), b"16-byte aligned"),
        (euler, dict(c=pv + 8), b"16-byte aligned"), (euler, dict(n=10), b"multiple of 4"),
        (unipc, dict(d=None), b"unipc_step_cached: null"), (unipc, dict(d=p0 + 4), b"16-byte aligned"),
        (unipc, dict(n=6), b"multiple of 4"), (unipc, dict(n_slots=4), b"n_slots"), (unipc, dict(write=3), b"write_slot"),
        (unipc, dict(stride=n - 4), b"slot_stride"), (unipc, dict(n_slots=2), b"coefficients of slot 2"),
    ]
    for fn, kw, msg in cases:
        assert fn(**kw) != 0, msg
        assert msg in lib.scail_last_error(), (msg, lib.scail_last_error())
    assert unipc(n_slots=2, write=1, coef=ctypes.addressof(two)) == 0
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the model: a small 2-block DiT
CFG = dict(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=2, text_dim=64, time_embed_dim=256)


def small_model(seed=0, **kw):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(seed)
    m = DiffusionTransformer(**CFG, **kw).to(torch.bfloat16).cuda().eval()
    with torch.no_grad():
        for _, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    return m


def sampler_inputs(seed=2, t=5, h=32, w=32):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16).cuda()
    x0 = torch.randn(1, t, 16, h, w, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, h, w), concat_smpl_render=r(1, t, 16, h // 2, w // 2),
                image_clip_features=r(1, 257, 1280))
    uc = dict(crossattn=r(1, 20, 64))  # shorter than the cond prompt: prepare_context pads it
    return x0, cond, uc


def fwd_kw(cond):
    return dict(y=None, ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
                image_clip_features=cond["image_clip_features"], concat_images=None)


MODES = {
    "bf16": {},
    "fp8_linear_fp8_attention": dict(fp8_linear=True, fp8_attention=True),
    "window1": dict(attention_window=1),
    "adaptive0.9": "adaptive",
    "fp8_window1": dict(fp8_linear=True, fp8_attention=True, attention_window=1),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_cond_forward_equals_row_1_of_the_pair(mode):
    from scail_b200 import sampler, sparse
    kw = MODES[mode]
    if kw == "adaptive":
        kw = dict(attention_adaptive=sparse.AdaptiveTiles(0.9))
    m = small_model(1, **kw)
    x0, cond, uc = sampler_inputs(3, t=5, h=32, w=48)
    ctx = sampler.prepare_context(cond, uc)
    with torch.no_grad():
        ts = torch.full((2,), 731.0, device="cuda")
        v2 = m(torch.cat([x0, x0], 0), timesteps=ts, context=ctx, **fwd_kw(cond))
        v1 = m(x0, timesteps=ts[1:], context=ctx[1:2], **fwd_kw(cond))
    assert v1.shape == (1, *v2.shape[1:])
    assert torch.equal(bits(v1[0].float()), bits(v2[1].float())), mode


def test_cond_forward_reuses_the_cached_conditioning_row():
    from scail_b200 import ops, sampler
    m = small_model(2)
    x0, cond, uc = sampler_inputs(4)
    ctx = sampler.prepare_context(cond, uc)
    ts = torch.full((2,), 512.0, device="cuda")
    with torch.no_grad():
        v2 = m(torch.cat([x0, x0], 0), timesteps=ts, context=ctx, **fwd_kw(cond))
        n0 = ops.LAUNCHES
        plain = m(x0, timesteps=ts[1:], context=ctx[1:2], **fwd_kw(cond))
        n_plain = ops.LAUNCHES - n0
        m.set_conditioning(ctx, cond["image_clip_features"], batch=2)
        try:
            n0 = ops.LAUNCHES
            cached = m(x0, timesteps=ts[1:], context=ctx[1:2], **fwd_kw(cond))
            n_cached = ops.LAUNCHES - n0
        finally:
            m.clear_conditioning()
    # text embedding (2 GEMMs), CLIP projection (2 LNs, 2 GEMMs) and per layer the text and CLIP K/V (2 GEMMs, 2 RMSNorms)
    assert n_plain - n_cached == 6 + 4 * CFG["num_layers"], (n_plain, n_cached)
    assert torch.equal(bits(cached.float()), bits(plain.float()))
    assert torch.equal(bits(cached[0].float()), bits(v2[1].float()))


def restated_sample(m, x0, cond, uc, n, pattern, scale=4.0, order=None):
    """sample() restated from the model's own b = 2 and b = 1 forwards: full steps update with the pair (cfg_euler_, or the
    UniPC step in torch ops with the product's coefficients), conditional-only steps with u = c - delta in torch ops."""
    from scail_b200 import ops, sampler, unipc
    sig = unipc.check_schedule(sampler.make_flow_timesteps(n, 5.0))
    ctx = sampler.prepare_context(cond, uc)
    kw = fwd_kw(cond)
    x = x0.clone()
    if order is not None:
        x_last, slots = torch.zeros_like(x0), torch.zeros(order, x0.numel(), device="cuda")
    delta = None
    for i in range(n):
        if pattern[i]:
            ts = torch.full((1,), sig[i] * 1000.0, device="cuda")
            c = m(x, timesteps=ts, context=ctx[1:2], **kw)[0].float().reshape(-1)
            u = c - delta
        else:
            ts = torch.full((2,), sig[i] * 1000.0, device="cuda")
            v = m(torch.cat([x, x], 0), timesteps=ts, context=ctx, **kw).contiguous()
            u, c = v[0].float().reshape(-1), v[1].float().reshape(-1)
            delta = c - u
        if order is None:
            if pattern[i]:
                x = (x.reshape(-1) + t32(f32(sig[i + 1] - sig[i])) * (u + t32(scale) * (c - u))).view(x0.shape)
            else:
                ops.cfg_euler_(x, v, scale, sig[i + 1] - sig[i])
            continue
        k = unipc.step_coefficients(sig, i, order)
        pad = [0.0] * (3 - order)
        coef = [f32(cc) for cc in [k.x_last_c, *k.slot_c, *pad, k.m_c, k.y_c, *k.slot_p, *pad, k.m_p]]
        z, y, mm = step_ref(x, x_last, u, c, slots, scale, sig[i], coef, k.correct)
        x, x_last = z.view(x0.shape), y.view(x0.shape)
        slots[k.write] = mm
    return x


@pytest.mark.parametrize("solver", [None, 2], ids=["euler", "unipc2"])
def test_threshold_zero_is_bit_identical_to_no_cache(solver):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.unipc import UniPC
    m = small_model(5)
    x0, cond, uc = sampler_inputs(5)
    c = CFGCache(0.0)
    mk = lambda: UniPC(solver) if solver else None
    with torch.no_grad():
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, solver=mk())
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, solver=mk(), cfg_cache=c)
    assert torch.equal(bits(cached), bits(plain))
    assert [s for _, s in c.history] == [False] * 5 and c.history[0][0] is None and c.history[1][0] == math.inf
    assert all(math.isfinite(i) and i > 0 for i, _ in c.history[2:])


@pytest.mark.parametrize("solver", [None, 2], ids=["euler", "unipc2"])
@pytest.mark.parametrize("how", ["max_skips1", "thresholds"])
def test_forced_pattern_against_the_restatement(solver, how):
    from scail_b200 import dit, sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.unipc import UniPC
    m = small_model(6)
    x0, cond, uc = sampler_inputs(6)
    n = 7
    if how == "max_skips1":
        c, th = CFGCache(math.inf, max_skips=1), None
        pattern = [False, False, True, False, True, False, True]
    else:
        c = CFGCache(0.0)
        th = [math.inf, math.inf, math.inf, 0.0, math.inf, math.inf, 0.0]
        pattern = [i >= 2 and t == math.inf for i, t in enumerate(th)]
    sig = sampler.make_flow_timesteps(n, 5.0)
    s = None
    if solver:
        s = UniPC(solver)
        s.begin(sig)
    ctx = sampler.prepare_context(cond, uc)
    main = torch.cuda.current_stream().cuda_stream
    with torch.no_grad():
        x = x0.clone()
        ws = None
        for i in range(n):
            if th is not None:
                c.threshold = th[i]
            sampler.sampler_step(m, x, sig[i], sig[i + 1], cond, uc, 4.0, _ctx=ctx, solver=s, cfg_cache=c)
            if i == 0:  # the b = 2 workspace of the caller's stream
                ws = {k: b.data_ptr() for k, b in dit._WS.bufs.items() if k[0][1] == main}
        # the b = 1 forwards ran on the cache's stream: the caller's b = 2 workspace was never reallocated
        assert all(k in dit._WS.bufs and dit._WS.bufs[k].data_ptr() == p for k, p in ws.items())
        want = restated_sample(m, x0, cond, uc, n, pattern, order=solver)  # (its b = 1 forwards run on this stream)
    assert [co for _, co in c.history] == pattern
    assert torch.equal(bits(x), bits(want))


def test_sample_with_cache_cross_kv_is_bit_identical():
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    m = small_model(7)
    x0, cond, uc = sampler_inputs(7)
    with torch.no_grad():
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=6, cfg_cache=CFGCache(math.inf, max_skips=1))
        m.mixins["adaln_layer"].cache_cross_kv = True
        c = CFGCache(math.inf, max_skips=1)
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=6, cfg_cache=c)
    assert [s for _, s in c.history] == [False, False, True, False, True, False]
    assert torch.equal(bits(cached), bits(plain))


@pytest.mark.parametrize("fast", [False, True], ids=["bf16", "fp8_window1_fbcache_unipc2"])
def test_graphed_step_is_bit_identical_to_eager(fast):
    from scail_b200 import dit, sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    kw = dict(fp8_linear=True, fp8_attention=True, attention_window=1) if fast else {}
    m = small_model(8, **kw)
    x0, cond, uc = sampler_inputs(8)
    n = 8
    sig = sampler.make_flow_timesteps(n, 5.0)
    ce, cg = CFGCache(math.inf, max_skips=1), CFGCache(math.inf, max_skips=1)
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
        for i in range(n):
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=fe, solver=se, cfg_cache=ce)
            if i == 0:  # eager's b = 2 workspace
                ws.update({k: b.data_ptr() for k, b in dit._WS.bufs.items() if k[0][1] == main})
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(bits(xe), bits(xg)), f"step {i}"
    pattern = [False, False, True, False, True, False, True, False]
    assert [s for _, s in cg.history] == pattern and ce.history == cg.history
    if fast:  # the first-block cache decides on full steps only
        assert len(fg.history) == pattern.count(False) and fe.history == fg.history
    assert all(k in dit._WS.bufs and dit._WS.bufs[k].data_ptr() == p for k, p in ws.items())


def test_graphed_steps_at_two_sizes_with_eager_at_a_third_in_between():
    """Two GraphedSteps with a CFG cache at two latent sizes and eager cfg-cache sampling at a third, interleaved: each b = 1
    graph keeps its own workspace, so every step stays bit-identical to eager sampler_step at its size."""
    import gc
    from scail_b200 import dit, sampler
    from scail_b200.cfg_cache import CFGCache
    m = small_model(9)
    n = 6
    sig = sampler.make_flow_timesteps(n, 5.0)
    runs = []
    with torch.no_grad():
        for seed, (h, w) in ((10, (32, 32)), (11, (32, 48))):
            x0, cond, uc = sampler_inputs(seed, t=5, h=h, w=w)
            xg, xe = x0.clone(), x0.clone()
            cg, ce = CFGCache(math.inf, max_skips=1), CFGCache(math.inf, max_skips=1)
            runs.append((sampler.GraphedStep(m, xg, cond, uc, 4.0, cfg_cache=cg), xg, xe, cond, uc, cg, ce))
        x3, cond3, uc3 = sampler_inputs(12, t=3, h=24, w=40)
        for i in range(n):
            for g, xg, xe, cond, uc, cg, ce in runs:
                g(sig[i], sig[i + 1])
                sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, cfg_cache=ce)
                c3 = CFGCache(math.inf, max_skips=1)  # a third size on yet another cache, between every two steps
                sampler.sample(m, x3.clone(), cond3, uc3, num_steps=3, cfg_cache=c3)
                assert [s for _, s in c3.history] == [False, False, True]
                del c3
                gc.collect()
            torch.cuda.synchronize()
            for g, xg, xe, cond, uc, cg, ce in runs:
                assert torch.equal(bits(xg), bits(xe)), f"step {i}"
    for g, xg, xe, cond, uc, cg, ce in runs:
        assert [s for _, s in cg.history] == [False, False, True, False, True, False] and ce.history == cg.history
    # a collected cache takes the b = 1 workspace of its stream with it
    c = CFGCache(math.inf)
    x0, cond, uc = sampler_inputs(13)
    with torch.no_grad():
        sampler.sample(m, x0, cond, uc, num_steps=3, cfg_cache=c)
    h = c.stream(x0.device).cuda_stream
    assert any(k[0][1] == h for k in dit._WS.bufs)
    del c
    gc.collect()
    assert not any(k[0][1] == h for k in dit._WS.bufs)
