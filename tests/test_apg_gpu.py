"""APG guidance on the GPU: the reduce / finish / update kernels in their three forms against the fp64 oracle at the real
latents, element by element; bit-reproducibility across launches and streams; the UniPC data-prediction step; the model:
sample() step by step against the oracle, reset(), GraphedStep, both caches and UniPC 1-3; and the kernels that
guidance=None and CFGZeroStar launch, unchanged."""
import ctypes
import math

import pytest
import torch

import apg_oracle as A
from kernel_check import recording
from test_cfg_cache_forecast_gpu import PATTERNS, forecast_ref
from test_cfg_cache_gpu import bits, f32, sampler_inputs, sentinel, small_model

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24  # fp32 unit roundoff


@pytest.fixture(autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


@pytest.fixture(autouse=True, scope="module")
def leave_workspaces_as_found():
    """Drop the DiT workspaces this module's forwards created (GraphedStep and CFGCache streams): stream handles recur, and
    a later test may hold the workspace of a recurring handle."""
    from scail_b200 import dit
    before = set(dit._WS.bufs)
    yield
    torch.cuda.synchronize()
    for k in [k for k in dit._WS.bufs if k not in before]:
        del dit._WS.bufs[k]


# 512x512, 480x832 and 512x896 latents of 81 frames (21 latent frames), and a small ragged one
LATENTS = [(1, 21, 16, 64, 64), (1, 21, 16, 60, 104), (1, 21, 16, 64, 112), (1, 3, 16, 5, 7)]
ids = lambda s: "x".join(map(str, s))


def _frames(t, T):
    return t.reshape(T, -1)


def _bcast(v, T):
    return v.view(1, T, 1, 1, 1)


def bounds(x, u, c, sigma, scale, eta, momentum, avg_old, parts, raw):
    """Per-element bound on |D_g(device) - D_g(fp64)| and the per-frame bounds (df, dp) on the factors, all fp64.

    a = |x| + sigma (|c| + |u|) (+ |momentum avg|) bounds every term that forms D_c, D_u, diff and the average.  The device
    rounds each of its dozen or so fp32 products and sums once, each within EPS of its own terms, so 16 EPS of the terms'
    magnitudes covers the per-element arithmetic.  f and p come from fp32 sums per (frame, CTA): a thread adds at most a few
    dozen products, then 5 shuffle and 8 warp levels, so each sum is within 64 EPS of the sum of |terms|, which by
    Cauchy-Schwarz is at most the product of the two vectors' norms (plus |a|'s share of the device's own rounding of D_c
    and diff).  Hence |df| <= 64 EPS f (1 + |a| / |diff|) and |dp| <= 64 EPS (|p| (1 + |a| / |diff|) + f (|diff| + |a|) /
    |D_c| + 2 |p| (1 + |a| / |D_c|)) per frame, which enter D_g through (w - 1) (df |diff| + (1 + |eta|) dp |D_c|)."""
    T = x.shape[1]
    a = x.double().abs() + sigma * (c.double().abs() + u.double().abs())
    if momentum:
        a = a + abs(momentum) * avg_old.double().abs()
    wm1 = abs(scale - 1.0)
    f, p = parts["f"], parts["p"]
    rawd, dc = raw["diff"], parts["D_c"]
    na, nd, nc = (_frames(t, T).norm(dim=1) for t in (a, rawd, dc))
    ra = torch.where(nd > 0, na / nd, torch.zeros_like(nd))
    df = 64 * EPS * f * (1 + ra)
    dp = 64 * EPS * (p.abs() * (1 + ra) + torch.where(nc > 0, (f * (nd + na) + 2 * p.abs() * (nc + na)) / nc,
                                                        torch.zeros_like(nc)))
    elem = 16 * EPS * (a + wm1 * (_bcast(f, T) * (a + rawd.abs()) + (1 + abs(eta)) * _bcast(p.abs(), T) * a))
    frame = wm1 * (_bcast(df, T) * rawd.abs() + (1 + abs(eta)) * _bcast(dp, T) * dc.abs())
    return elem + frame, df, dp


def euler_bound(x, d_g, bdg, sigma, next_sigma):
    """|x'(device) - x'(fp64)| for x' = x + k (x - D_g): k rounded once, then one difference, product and sum, each within
    EPS of its terms, plus k times D_g's own bound."""
    k = abs((next_sigma - sigma) / sigma)
    return k * bdg + 4 * EPS * (x.double().abs() + k * (x.double().abs() + d_g.abs()))


def assert_within(got, want, bound, what):
    d = (got.double() - want).abs()
    bad = ~(d <= bound)
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {d.numel()} elements outside the bound; worst |d| / bound "
                                 f"= {float((d / bound.clamp_min(1e-300)).max()):.3g}")


# ---------------------------------------------------------------- kernels
def make_case(shape, form, seed, sigma):
    """x (fp32), v (the pair, or c alone), the form's kwargs, and the fp64 (u, c) the oracle sees.  Frame 0 has D_c = 0,
    frame 1 has diff = 0 (u = c, and a zero average), frame 2 is planted 1024 times larger."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    T = shape[1]
    u = torch.randn(shape, generator=g, device="cuda") * 2.0
    c = 0.8 * u + 0.6 * torch.randn(shape, generator=g, device="cuda")
    u[0, 1] = c[0, 1]
    u[0, 2] *= 1024.0
    c[0, 2] *= 1024.0
    pair = torch.cat([u, c]).to(torch.bfloat16)
    cf = pair[1:2].float()
    x = torch.randn(shape, generator=g, device="cuda")
    x[0, 0] = sigma * cf[0, 0]  # exact in fp32: D_c = 0
    avg = torch.randn(shape, generator=g, device="cuda")
    avg[0, 1] = 0.0
    if form == "pair":
        return x, pair, {}, pair[0:1].double(), cf.double(), avg
    c1 = pair[1:2].contiguous()
    if form == "cached":
        delta = cf - pair[0:1].float() + 0.01 * torch.randn(shape, generator=g, device="cuda")
        delta[0, 1] = 0.0
        return x, c1, dict(delta=delta), cf.double() - delta.double(), cf.double(), avg
    coef = PATTERNS[3]
    n = math.prod(shape)
    slots = sentinel(3, n).view(3, *shape)
    for k in range(3):
        slots[k] = (cf - pair[0:1].float()) / (3 * coef[k]) + 0.01 * torch.randn(shape, generator=g, device="cuda")
        slots[k, 0, 1] = 0.0
    d_hat = forecast_ref(slots, coef)  # the cache's fp32 forecast, as the kernels form it
    return x, c1, dict(forecast=(slots, coef)), cf.double() - d_hat.double(), cf.double(), avg


def apg_buffers(T):
    from scail_b200 import ops
    return (torch.full((ops.apg_partials_len(T),), math.nan, device="cuda"),
            torch.full((T, 4), math.nan, device="cuda", dtype=torch.float64), torch.full((T, 2), math.nan, device="cuda"))


CASES = {"vanilla": (1.0, 0.0, 0.0), "thresholded_momentum": (0.3, "auto", -0.5)}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("form", ["pair", "cached", "forecast"])
@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_kernels_against_the_oracle(shape, form, case):
    from scail_b200 import ops
    T, n = shape[1], math.prod(shape)
    sigma, next_sigma, scale = 0.5, 0.4375, 5.0
    x, v, kw, u64, c64, avg_old = make_case(shape, form, 7 + sum(shape) + len(form), sigma)
    eta, r, beta = CASES[case]
    raw = A.apg_parts(x, u64, c64, sigma, scale, eta, 0.0, beta, avg_old)  # before the threshold
    if r == "auto":  # the planted frame is cut to r, frames of ordinary size are not
        norms = _frames(raw["diff"], T).norm(dim=1)
        r = 1.5 * float(norms[[t for t in range(T) if t != 2]].max())
    parts = A.apg_parts(x, u64, c64, sigma, scale, eta, r, beta, avg_old)
    bdg, df, dp = bounds(x, u64, c64, sigma, scale, eta, beta, avg_old, parts, raw)
    partials, sums, factors = apg_buffers(T)
    avg = avg_old.clone() if beta else None
    ops.apg_reduce(x, v, sigma, partials, avg, beta, **kw)
    ops.apg_finish(partials, sums, factors, r, T, n)
    # the sums: within 64 EPS of the sum of |terms| (see bounds), which Cauchy-Schwarz bounds by the norms
    a = _frames(x.double().abs() + sigma * (c64.abs() + u64.abs()) + (abs(beta) * avg_old.double().abs() if beta else 0), T)
    na = a.norm(dim=1)
    d, pc = _frames(raw["diff"], T), _frames(raw["D_c"], T)
    nd, nc = d.norm(dim=1), pc.norm(dim=1)
    for k, (want, b) in enumerate((((d * d).sum(1), nd * (nd + 2 * na)), ((d * pc).sum(1), nd * nc + na * (nd + nc)),
                                   ((pc * pc).sum(1), nc * (nc + 2 * na)))):
        assert bool(((sums[:, k] - want).abs() <= 64 * EPS * b).all()), (k, sums[:, k], want)
    assert bool((sums[:, 3] == 0).all())
    assert sums[0, 2].item() == 0.0 and sums[1, 0].item() == 0.0  # the zero frames are exactly zero
    assert factors[0, 1].item() == 0.0 and factors[1, 0].item() == 1.0 and factors[1, 1].item() == 0.0
    assert bool(((factors[:, 0].double() - parts["f"]).abs() <= df + EPS * parts["f"]).all()), (factors[:, 0], parts["f"])
    assert bool(((factors[:, 1].double() - parts["p"]).abs() <= dp + EPS * parts["p"].abs()).all()), (factors[:, 1], parts["p"])
    if r:
        assert factors[2, 0].item() < 1e-2 and int((factors[:, 0] == 1.0).sum()) == T - 1  # cut and uncut frames
    if beta:  # pass 1 wrote the average: one difference, one product and one sum of at most |a|
        assert_within(avg, parts["avg"], 8 * EPS * a.view(shape), "average")
    # the data prediction into a buffer: x untouched
    out = torch.full(shape, math.nan, device="cuda")
    x0 = x.clone()
    assert ops.apg_update_(x, v, factors, scale, eta, sigma, out=out, avg=avg, **kw) is out
    assert torch.equal(bits(x), bits(x0))
    assert_within(out, parts["D_g"], bdg, "D_g")
    assert float(out[0, 1].double().sub(parts["D_c"][0, 1]).abs().max()) <= float(bdg[0, 1].max())  # diff = 0: D_g = D_c
    # the Euler step in place
    assert ops.apg_update_(x, v, factors, scale, eta, sigma, next_sigma, avg=avg, **kw) is x
    want = A.euler(x0, parts["D_g"], sigma, next_sigma)
    assert_within(x, want, euler_bound(x0, parts["D_g"], bdg, sigma, next_sigma), "Euler")
    if case == "vanilla":  # eta = 1, r = 0, beta = 0: vanilla CFG in exact arithmetic
        assert_within(x, A.vanilla_cfg_euler(x0, u64, c64, scale, sigma, next_sigma),
                      euler_bound(x0, parts["D_g"], bdg, sigma, next_sigma) + 1e-12 * want.abs(), "vanilla")


def test_nan_stays_in_its_frame():
    from scail_b200 import ops
    shape = (1, 3, 16, 5, 7)
    x, v, _, _, _, _ = make_case(shape, "pair", 5, 0.5)
    v[1, 2, 0, 0, 0] = math.nan
    partials, sums, factors = apg_buffers(3)
    ops.apg_reduce(x, v, 0.5, partials)
    ops.apg_finish(partials, sums, factors, 1.0, 3, x.numel())
    ops.apg_update_(x, v, factors, 4.0, 0.5, 0.5, 0.4)
    assert torch.isnan(x[0, 2]).all() and not torch.isnan(x[0, :2]).any()
    assert math.isnan(factors[2, 1].item())


def test_repeated_launches_and_streams_are_bit_identical():
    from scail_b200 import ops
    shape = LATENTS[2]
    T = shape[1]
    x, v, kw, _, _, avg_old = make_case(shape, "forecast", 11, 0.5)

    def run():
        partials, sums, factors = apg_buffers(T)
        avg, xe, m = avg_old.clone(), x.clone(), torch.empty_like(x)
        ops.apg_reduce(xe, v, 0.5, partials, avg, -0.7, **kw)
        ops.apg_finish(partials, sums, factors, 30.0, T, xe.numel())
        ops.apg_update_(xe, v, factors, 4.5, 0.2, 0.5, out=m, avg=avg, **kw)
        ops.apg_update_(xe, v, factors, 4.5, 0.2, 0.5, 0.41, avg=avg, **kw)
        return [bits(partials), sums.view(torch.int64), bits(factors), bits(avg), bits(xe), bits(m)]

    first = run()
    for _ in range(2):
        assert all(torch.equal(a, b) for a, b in zip(first, run()))
    side, main = torch.cuda.Stream(), torch.cuda.current_stream()
    side.wait_stream(main)
    with torch.cuda.stream(side):
        other = run()
    main.wait_stream(side)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(first, other))


def solver_ref(x, x_last, m, slots, coef, correct):
    """The UniPC step after m, as separate torch fp32 ops in the kernel's order -> (z, y), flat."""
    t = lambda c_: torch.tensor(c_, dtype=torch.float32, device="cuda")
    a_x, a, a_m, b_y, b, b_m = coef[0], coef[1:4], coef[4], coef[5], coef[6:9], coef[9]
    m = m.reshape(-1)
    if correct:
        y = t(a_x) * x_last.reshape(-1)
        for s in range(slots.shape[0]):
            if a[s] != 0.0:
                y = y + t(a[s]) * slots[s]
        y = y + t(a_m) * m
    else:
        y = x.reshape(-1).clone()
    z = t(b_y) * y
    for s in range(slots.shape[0]):
        if b[s] != 0.0:
            z = z + t(b[s]) * slots[s]
    return z + t(b_m) * m, y


@pytest.mark.parametrize("shape", LATENTS, ids=ids)
def test_unipc_data_prediction_kernel(shape):
    """unipc_step_dpred_ bit for bit against the solver's algebra on the given m, NaN sentinels in zero-coefficient slots."""
    from scail_b200 import ops
    n = math.prod(shape)
    g = torch.Generator(device="cuda").manual_seed(3 + sum(shape))
    x0, xl0, m = (torch.randn(shape, generator=g, device="cuda") for _ in range(3))
    live = torch.randn(3, n, generator=g, device="cuda")
    for act in ([0], [0, 2], [0, 1, 2]):
        for correct in (True, False):
            a, b = [0.0] * 3, [0.0] * 3
            for j, s in enumerate(act):
                a[s], b[s] = f32(0.7 - 0.45 * j), f32(-0.3 + 0.55 * j)
            coef = [f32(0.93), *a, f32(-0.41), f32(0.88), *b, f32(0.17)]
            before = sentinel(3, n)
            for s in act:
                before[s] = live[s]
            x, xl, slots = x0.clone(), xl0.clone(), before.clone()
            ops.unipc_step_dpred_(x, xl, m, slots, 1, coef, correct)
            z, y = solver_ref(x0, xl0, m, before, coef, correct)
            assert torch.equal(bits(x.view(-1)), bits(z)) and torch.equal(bits(xl.view(-1)), bits(y)), (act, correct)
            assert torch.equal(bits(slots[1]), bits(m.view(-1)))
            for s in (0, 2):
                assert torch.equal(bits(slots[s]), bits(before[s]))


def test_abi_refuses_bad_arguments():
    from scail_b200 import _lib
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    T, n = 2, 128
    x, avg, m = (torch.zeros(n + 8, device="cuda") for _ in range(3))
    slots = torch.zeros(2, n, device="cuda")
    v = torch.zeros(2 * n + 8, device="cuda", dtype=torch.bfloat16)
    part = torch.zeros(3 * T * 32, device="cuda")
    sums = torch.zeros(T, 4, device="cuda", dtype=torch.float64)
    fac = torch.zeros(T + 1, 2, device="cuda")
    px, pa, pm, pv, pp, ps, pf = (t.data_ptr() for t in (x, avg, m, v, part, sums, fac))
    coef = (ctypes.c_float * 10)(0.5, 0.5, 0.5, 0.0, 0.5, 0.5, 0.5, 0.5, 0.0, 0.5)  # slot 2 unused with n_slots = 2
    red = lambda **kw: lib.scail_apg_reduce(*[kw.get(k, dv) for k, dv in (
        ("form", 0), ("x", px), ("v", pv), ("d", None), ("ds", 0), ("nd", 0), ("dk", None), ("avg", pa), ("sigma", 0.5),
        ("beta", -0.5), ("part", pp), ("plen", 3 * T * 32), ("T", T), ("n", n))], st)
    fin = lambda **kw: lib.scail_apg_finish(*[kw.get(k, dv) for k, dv in (
        ("part", pp), ("plen", 3 * T * 32), ("sums", ps), ("fac", pf), ("r", 1.0), ("T", T), ("n", n))], st)
    upd = lambda **kw: lib.scail_apg_update(*[kw.get(k, dv) for k, dv in (
        ("form", 0), ("x", px), ("v", pv), ("d", None), ("ds", 0), ("nd", 0), ("dk", None), ("avg", pa), ("fac", pf),
        ("m", pm), ("sigma", 0.5), ("wm1", 3.0), ("eta", 0.5), ("k", -0.1), ("T", T), ("n", n))], st)
    dpr = lambda **kw: lib.scail_unipc_step_dpred(*[kw.get(k, dv) for k, dv in (
        ("x", px), ("xl", pa), ("m", pm), ("slots", slots.data_ptr()), ("stride", n), ("n_slots", 2), ("write", 1), ("n", n),
        ("correct", 1), ("coef", ctypes.addressof(coef)))], st)
    assert red() == 0 and fin() == 0 and upd() == 0 and upd(m=None) == 0 and dpr() == 0, lib.scail_last_error()
    torch.cuda.synchronize()
    cases = [
        (red, dict(form=3), b"form = 3"), (red, dict(x=None), b"apg_reduce: null operand"),
        (red, dict(form=1), b"null delta"), (red, dict(form=2, d=px), b"null dcoef"),
        (red, dict(x=px + 4), b"16-byte aligned"), (red, dict(avg=pa + 4), b"avg 16-byte"),
        (red, dict(n=n + 4), b"multiple of 4 * frames"), (red, dict(T=0), b"frames"), (red, dict(plen=5), b"partials holds"),
        (red, dict(part=None), b"null partials"),
        (fin, dict(r=-1.0), b"norm_threshold"), (fin, dict(r=math.inf), b"norm_threshold"), (fin, dict(fac=pf + 4), b"8-byte"),
        (fin, dict(plen=5), b"partials holds"), (fin, dict(sums=None), b"apg_finish: null"), (fin, dict(n=6), b"multiple"),
        (upd, dict(fac=None), b"null factors"), (upd, dict(m=pm + 4), b"16-byte"), (upd, dict(form=-1), b"form = -1"),
        (upd, dict(v=pv + 8), b"16-byte aligned"),
        (dpr, dict(m=None), b"unipc_step_dpred: null"), (dpr, dict(write=2), b"write_slot"), (dpr, dict(m=pm + 4), b"16-byte"),
    ]
    for fn, kw, msg in cases:
        assert fn(**kw) != 0, msg
        assert msg in lib.scail_last_error(), (msg, lib.scail_last_error())
    torch.cuda.synchronize()


# ---------------------------------------------------------------- the model: a small 2-block DiT
def record_forwards(m):
    """Wrap m.forward: the returned list gets (input latent, output) of every forward, cloned."""
    calls, f = [], m.forward

    def fwd(x, *a, **kw):
        out = f(x, *a, **kw)
        calls.append((x.detach().clone(), out.detach().clone()))
        return out

    m.forward = fwd
    return calls


def oracle_check(x_in, v, x_out, sigma, next_sigma, scale, g, avg, delta_hat=None, m_dev=None):
    """One product step against the oracle: the Euler result x_out (or, with m_dev, the solver's data prediction) within
    the bound of `bounds`.  delta_hat (fp32) marks a conditional-only step: v is c alone and u = c - delta_hat.  Returns the
    oracle's momentum average after the step."""
    if delta_hat is None:
        u, c = v[0:1].double(), v[1:2].double()
    else:
        c = v[0:1].double()
        u = c - delta_hat.double()
    eta, r, beta = g.eta, g.norm_threshold, g.momentum
    raw = A.apg_parts(x_in, u, c, sigma, scale, eta, 0.0, beta, avg)
    parts = A.apg_parts(x_in, u, c, sigma, scale, eta, r, beta, avg)
    bdg, _, _ = bounds(x_in, u, c, sigma, scale, eta, beta, avg if avg is not None else torch.zeros_like(x_in), parts, raw)
    if m_dev is not None:
        assert_within(m_dev.view(x_in.shape), parts["D_g"], bdg, "data prediction")
    else:
        assert_within(x_out, A.euler(x_in, parts["D_g"], sigma, next_sigma),
                      euler_bound(x_in, parts["D_g"], bdg, sigma, next_sigma), "Euler step")
    return parts["avg"]


def test_sample_apg_1_0_0_is_vanilla_cfg_step_by_step():
    """APG(1, 0, 0) over 4 steps: each step, from the latent and the pair the model gave, within the stated bound of the
    fp64 vanilla step, and of what guidance=None's kernel makes of the same inputs."""
    from scail_b200 import ops, sampler
    from scail_b200.guidance import APG
    m = small_model(40)
    x0, cond, uc = sampler_inputs(40)
    n, scale = 4, 4.0
    calls = record_forwards(m)
    with torch.no_grad():
        got = sampler.sample(m, x0.clone(), cond, uc, num_steps=n, scale=scale, guidance=APG(1.0))
    sig = [float(s) for s in sampler.make_flow_timesteps(n, 5.0)]
    assert len(calls) == n
    xs = [cl[0][0:1] for cl in calls] + [got]
    g = APG(1.0)
    for i in range(n):
        v = calls[i][1]
        oracle_check(xs[i], v, xs[i + 1], sig[i], sig[i + 1], scale, g, None)
        none = ops.cfg_euler_(xs[i].clone(), v.contiguous(), scale, sig[i + 1] - sig[i])
        # the vanilla kernel's own error: one difference, product and sum per term, within 4 EPS of the terms
        dsig = abs(sig[i + 1] - sig[i])
        u, c = v[0:1].double(), v[1:2].double()
        b_none = 4 * EPS * (xs[i].double().abs() + dsig * (u.abs() + scale * (c.abs() + u.abs())))
        raw = A.apg_parts(xs[i], u, c, sig[i], scale, 1.0)
        bdg, _, _ = bounds(xs[i], u, c, sig[i], scale, 1.0, 0.0, None, raw, raw)
        assert_within(xs[i + 1], none.double(), euler_bound(xs[i], raw["D_g"], bdg, sig[i], sig[i + 1]) + b_none,
                      f"APG(1, 0, 0) against guidance=None, step {i}")


@pytest.mark.parametrize("solver", [None, 1, 2, 3], ids=["euler", "unipc1", "unipc2", "unipc3"])
def test_sample_against_the_oracle_step_by_step(solver):
    """APG(0.4, r, -0.5) with r > 0: every step against the oracle carrying its own fp64 momentum; with UniPC the solver's
    data prediction within the bound and the rest of its step bit for bit from it.  Then reset() clears the momentum: a
    second sample() with the same object is bit-identical to the first and to a fresh object's."""
    from scail_b200 import sampler, unipc
    from scail_b200.guidance import APG
    from scail_b200.unipc import UniPC
    mdl = small_model(41)
    x0, cond, uc = sampler_inputs(41)
    n, scale = 4, 5.0
    g = APG(0.4, 1e-2, -0.5)
    sig = sampler.make_flow_timesteps(n, 5.0)
    sl = [float(s) for s in sig]
    s = UniPC(solver) if solver else None
    if s is not None:
        s.begin(sig)
    calls = record_forwards(mdl)
    x, avg = x0.clone(), None
    with torch.no_grad():
        for i in range(n):
            x_in = x.clone()
            if s is not None:
                xl0 = s.x_last.clone() if i else torch.zeros_like(x)
                slots0 = s.slots.clone() if i else torch.zeros(solver, x.numel(), device="cuda")
            sampler.sampler_step(mdl, x, sig[i], sig[i + 1], cond, uc, scale, solver=s, guidance=g)
            v = calls[-1][1]
            if s is None:
                avg = oracle_check(x_in, v, x, sl[i], sl[i + 1], scale, g, avg)
                continue
            k = unipc.step_coefficients(sl, i, solver)
            avg = oracle_check(x_in, v, None, sl[i], sl[i + 1], scale, g, avg, m_dev=s.slots[k.write])
            pad = [0.0] * (3 - solver)
            coef = [f32(c_) for c_ in [k.x_last_c, *k.slot_c, *pad, k.m_c, k.y_c, *k.slot_p, *pad, k.m_p]]
            z, y = solver_ref(x_in, xl0, s.slots[k.write], slots0, coef, k.correct)
            assert torch.equal(bits(x.view(-1)), bits(z)) and torch.equal(bits(s.x_last.view(-1)), bits(y)), i
        assert g.step_index == n and bool((g.last_factors[:, 0] < 1).all())  # the threshold was active
        again = sampler.sample(mdl, x0.clone(), cond, uc, num_steps=n, scale=scale, solver=UniPC(solver) if solver else None,
                               guidance=g)
        fresh = sampler.sample(mdl, x0.clone(), cond, uc, num_steps=n, scale=scale, solver=UniPC(solver) if solver else None,
                               guidance=APG(0.4, 1e-2, -0.5))
    assert torch.equal(bits(again), bits(x)) and torch.equal(bits(fresh), bits(x))


@pytest.mark.parametrize("solver", [None, 2], ids=["euler", "unipc2"])
def test_cfg_cache_forecast_against_the_oracle(solver):
    """CFGCache(inf, max_skips=1, order=2): full and conditional-only steps in turn; a conditional-only step's u is f32(c)
    - the cache's forecast, and the momentum advances on every step."""
    from scail_b200 import sampler, unipc
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import APG
    from scail_b200.unipc import UniPC
    mdl = small_model(42)
    x0, cond, uc = sampler_inputs(42)
    n, scale = 7, 4.0
    g, cc = APG(0.0, 0.5, -0.75), CFGCache(math.inf, max_skips=1, order=2)
    sig = sampler.make_flow_timesteps(n, 5.0)
    sl = [float(s_) for s_ in sig]
    s = UniPC(solver) if solver else None
    if s is not None:
        s.begin(sig)
    calls = record_forwards(mdl)
    x, avg = x0.clone(), None
    with torch.no_grad():
        for i in range(n):
            x_in = x.clone()
            sampler.sampler_step(mdl, x, sig[i], sig[i + 1], cond, uc, scale, solver=s, cfg_cache=cc, guidance=g)
            v = calls[-1][1]
            d_hat = forecast_ref(cc.buffers.slots, cc.forecast()) if v.shape[0] == 1 else None
            m_dev = None if s is None else s.slots[unipc.step_coefficients(sl, i, solver).write]
            avg = oracle_check(x_in, v, x, sl[i], sl[i + 1], scale, g, avg, delta_hat=d_hat, m_dev=m_dev)
    assert [c_ for _, c_ in cc.history] == [False, False, True, False, True, False, True]
    assert g.step_index == n


def test_caches_at_threshold_zero_are_bit_identical_to_none():
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import APG
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    m = small_model(43)
    x0, cond, uc = sampler_inputs(43)
    with torch.no_grad():
        for solver in (None, 2):
            mk = lambda: dict(solver=UniPC(solver) if solver else None, guidance=APG(0.5, 1.0, -0.5))
            plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, **mk())
            cfgc = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, cfg_cache=CFGCache(0.0), **mk())
            fb = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, step_cache=FirstBlockCache(0.0), **mk())
            assert torch.equal(bits(cfgc), bits(plain)) and torch.equal(bits(fb), bits(plain)), solver


@pytest.mark.parametrize("how", ["euler", "cfgcache_unipc2"])
def test_graphed_step_is_bit_identical_to_eager(how):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import APG
    from scail_b200.unipc import UniPC
    m = small_model(44)
    x0, cond, uc = sampler_inputs(44)
    n = 6
    sig = sampler.make_flow_timesteps(n, 5.0)
    ge, gg = APG(0.5, 1.0, -0.5), APG(0.5, 1.0, -0.5)
    se = sg = ce = cg = None
    if how != "euler":
        se, sg = UniPC(2), UniPC(2)
        se.begin(sig)
        sg.begin(sig)
        ce, cg = CFGCache(math.inf, max_skips=1, order=2), CFGCache(math.inf, max_skips=1, order=2)
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, solver=sg, cfg_cache=cg, guidance=gg)
        for i in range(n):
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, solver=se, cfg_cache=ce, guidance=ge)
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(bits(xe), bits(xg)), f"step {i}"
    assert ge.step_index == gg.step_index == n
    if ce is not None:
        assert [s for _, s in cg.history] == [False, False, True, False, True, False] and ce.history == cg.history


UPDATE_OPS = ["cfg_euler_", "unipc_step_", "cfg_cache_delta", "cfg_euler_cached_", "unipc_step_cached_",
              "cfg_cache_delta_forecast", "cfg_euler_cached_forecast_", "unipc_step_cached_forecast_", "cfg_zero_scale",
              "apg_reduce", "apg_finish", "apg_update_", "unipc_step_dpred_"]


def test_none_and_cfg_zero_star_launch_what_they_launched_before():
    """The update-side launches of guidance=None and CFGZeroStar, in order, are those of the code before APG existed: no
    APG or data-prediction op runs, and the others run with the same (un)scaled forms."""
    from scail_b200 import ops, sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import CFGZeroStar
    from scail_b200.unipc import UniPC
    m = small_model(45)
    x0, cond, uc = sampler_inputs(45)
    E, Es, Z, D = ("cfg_euler_", False), ("cfg_euler_", True), ("cfg_zero_scale", False), ("cfg_cache_delta", False)
    U, Us = ("unipc_step_", False), ("unipc_step_", True)
    Ec, Ecs = ("cfg_euler_cached_", False), ("cfg_euler_cached_", True)
    expected = {
        "none_euler": (dict(), [E] * 4),
        "none_unipc2": (dict(solver=2), [U] * 4),
        "cfgzero1_euler": (dict(guidance=1), [Z, Es] * 3),
        "cfgzero1_unipc2": (dict(solver=2, guidance=1), [U] + [Z, Us] * 3),
        "none_cfgcache": (dict(cache=True), [D, E, D, E, Ec, D, E]),
        "cfgzero0_cfgcache": (dict(cache=True, guidance=0), [D, Z, Es, D, Z, Es, Z, Ecs, D, Z, Es]),
    }
    for name, (cfg, want) in expected.items():
        seq = []

        def fields(op, args):  # (op, scaled update): cfg_zero_scale's own u_scale is its output
            seq.append((op, op != "cfg_zero_scale" and args.get("u_scale") is not None))
            return {}, 0

        with torch.no_grad(), recording(ops, UPDATE_OPS, fields):
            sampler.sample(m, x0.clone(), cond, uc, num_steps=4, solver=UniPC(cfg["solver"]) if "solver" in cfg else None,
                           cfg_cache=CFGCache(math.inf, max_skips=1) if cfg.get("cache") else None,
                           guidance=CFGZeroStar(cfg["guidance"]) if "guidance" in cfg else None)
        assert seq == want, (name, seq)
