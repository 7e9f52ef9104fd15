"""Taylor forecast of the first-block residual cache on the GPU: the two forecast kernels against torch restatements
(tests/forecast_oracle.py), exact recovery of polynomial residuals through the cache's own slot and coefficient logic, the
cached model against a restatement built from its own hooks, and GraphedStep against eager sampler_step."""
import math

import numpy as np
import pytest
import torch

from forecast_oracle import RestatedForecastCache, apply_forecast_ref
from step_cache_oracle import apply_ref, update_ref

pytestmark = pytest.mark.gpu


def rnd(*shape, scale=1.0, seed=0, dtype=torch.bfloat16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def bits(t):
    return t.view(torch.int32)


# ---------------------------------------------------------------- 1. update_slot
# (B, N, d, n_ref, n_seq): small ragged shapes with odd n_ref, then b = 2 at 512x512, 480x832 and 512x896 (21 frames)
SHAPES = [(1, 200, 256, 41, 100), (2, 333, 136, 77, 211), (3, 91, 8, 3, 80), (2, 1856, 264, 257, 1280),
          (2, 27904, 5120, 1024, 21504), (2, 42510, 5120, 1560, 32760), (2, 48832, 5120, 1792, 37632)]
SMALL = SHAPES[:4]


def sentinel_slots(n_slots, B, n_seq, d):
    """Slots filled with a fixed bit pattern that includes NaNs and infinities (compared as bits)."""
    ar = torch.arange(n_slots * B * n_seq * d, device="cuda", dtype=torch.int64)
    pat = ((ar * 2654435761) & 0x7FFFFFFF).to(torch.int32) ^ 0x7F800001  # many of these are NaN or inf patterns
    return pat.view(torch.float32).view(n_slots, B, n_seq, d)


def slot_tensor(s):
    return torch.tensor([s], device="cuda", dtype=torch.int32)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_update_slot_writes_one_slot_bit_exact(shape):
    from scail_b200 import ops
    B, N, d, n_ref, n_seq = shape
    h1c = rnd(B, n_seq, d, seed=3)
    h = rnd(B, N, d, scale=4.0, seed=4)
    h[0, n_ref, :4] = torch.tensor([1e6, 3e-5, -7e4, 0.0], device="cuda", dtype=torch.bfloat16)
    want = update_ref(h, h1c, n_ref)
    n_slots = 3 if N < 40000 or d < 5120 else 2  # keep the largest case's slots within a few GB
    before = sentinel_slots(n_slots, B, n_seq, d)
    for s in list(range(n_slots)) + [-1, n_slots, 1 << 20]:
        R = before.clone()
        ops.step_cache_update_slot(h, h1c, R, slot_tensor(s), n_ref)
        for k in range(n_slots):
            if k == s:
                assert torch.equal(R[k], want), (s, k)
            else:
                assert torch.equal(bits(R[k]), bits(before[k])), (s, k)  # other slots, and all for an out-of-range index
        del R
    del before
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- 2. apply_forecast
COEFS = [(-0.3125, 0.0, 0.0), (0.0, 2.5, -1.5), (3.0, -3.0, 1.0), (0.1, 0.0, 0.9), (1.7000000476837158, -0.7, 0.0)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_apply_forecast_bit_exact(shape):
    from scail_b200 import ops
    B, N, d, n_ref, n_seq = shape
    R = rnd(3, B, n_seq, d, scale=0.5, seed=11, dtype=torch.float32)
    R[0, 0, 0, :3] = torch.tensor([3e38, -1e-30, 7.0], device="cuda")  # an overflowing product and a tiny one
    h0 = rnd(B, N, d, scale=2.0, seed=12)
    outside = torch.ones(N, dtype=torch.bool)
    outside[n_ref:n_ref + n_seq] = False
    big = N * d > 10 ** 8
    for coef in (COEFS[1:3] if big else COEFS):
        c = torch.tensor([np.float32(x) for x in coef], device="cuda", dtype=torch.float32)
        cf = [float(x) for x in c.tolist()]
        want = apply_forecast_ref(h0, R, cf, n_ref)
        got = h0.clone()
        ops.step_cache_apply_forecast(got, R, c, n_ref)
        assert torch.equal(got, want), coef
        assert torch.equal(got[:, outside], h0[:, outside])  # ref and pose rows untouched
        again = h0.clone()
        ops.step_cache_apply_forecast(again, R, c, n_ref)
        assert torch.equal(again, got)  # repeat launches are bit-identical
    # c = (1, 0, 0) is step_cache_apply bit for bit, whichever slot holds the 1
    for s in range(3):
        c = torch.zeros(3, device="cuda")
        c[s] = 1.0
        got = h0.clone()
        ops.step_cache_apply_forecast(got, R, c, n_ref)
        assert torch.equal(got, apply_ref(h0, R[s], n_ref)), s
        plain = h0.clone()
        ops.step_cache_apply(plain, R[s].contiguous(), n_ref)
        assert torch.equal(got, plain), s
    # no active slot: h unchanged
    got = h0.clone()
    ops.step_cache_apply_forecast(got, R, torch.zeros(3, device="cuda"), n_ref)
    assert torch.equal(got, h0)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("shape", SMALL, ids=lambda s: "x".join(map(str, s)))
def test_apply_forecast_does_not_read_a_zero_coefficient_slot(shape):
    from scail_b200 import ops
    B, N, d, n_ref, n_seq = shape
    R = rnd(3, B, n_seq, d, seed=21, dtype=torch.float32)
    h0 = rnd(B, N, d, seed=22)
    for dead in range(3):
        Rn = R.clone()
        Rn[dead] = math.nan
        coef = [0.5, -1.25, 1.75]
        coef[dead] = 0.0
        want = apply_forecast_ref(h0, R, coef, n_ref)
        got = h0.clone()
        ops.step_cache_apply_forecast(got, Rn, torch.tensor(coef, device="cuda"), n_ref)
        assert torch.equal(got, want), dead
    # fewer slots than coefficients: only the first n_slots coefficients are read
    got = h0.clone()
    ops.step_cache_apply_forecast(got, R[:2].contiguous(), torch.tensor([0.5, 0.5, math.nan], device="cuda"), n_ref)
    assert torch.equal(got, apply_forecast_ref(h0, R[:2], [0.5, 0.5], n_ref))


def test_forecast_abi_refuses_bad_arguments():
    from scail_b200 import _lib
    B, N, d, n_ref, n_seq = 2, 40, 16, 8, 24
    h = torch.zeros(B, N, d, device="cuda", dtype=torch.bfloat16)
    h1c = torch.zeros(B, n_seq, d, device="cuda", dtype=torch.bfloat16)
    n = B * n_seq * d
    R = torch.zeros(3, n + 4, device="cuda")  # padded slots: slot_stride = n + 4
    slot, coef = slot_tensor(1), torch.tensor([0.0, 1.0, 0.0], device="cuda")
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    ph, pc, pR, ps, pk = h.data_ptr(), h1c.data_ptr(), R.data_ptr(), slot.data_ptr(), coef.data_ptr()
    upd = lambda *a: lib.scail_step_cache_update_slot(*a, st)
    app = lambda *a: lib.scail_step_cache_apply_forecast(*a, st)
    assert upd(ph, pc, pR, n + 4, 3, ps, B, N, d, n_ref, n_seq) == 0
    assert app(ph, pR, n + 4, 3, pk, B, N, d, n_ref, n_seq) == 0
    torch.cuda.synchronize()
    for call, msg in ((lambda: upd(None, pc, pR, n, 3, ps, B, N, d, n_ref, n_seq), b"null"),
                      (lambda: upd(ph, pc, pR, n, 3, None, B, N, d, n_ref, n_seq), b"null"),
                      (lambda: app(ph, pR, n, 3, None, B, N, d, n_ref, n_seq), b"null"),
                      (lambda: upd(ph + 2, pc, pR, n, 3, ps, B, N, d, n_ref, n_seq), b"16-byte aligned"),
                      (lambda: app(ph, pR + 4, n, 3, pk, B, N, d, n_ref, n_seq), b"16-byte aligned"),
                      (lambda: upd(ph, pc, pR, n, 3, ps + 2, B, N, d, n_ref, n_seq), b"slot must be 4-byte aligned"),
                      (lambda: app(ph, pR, n, 3, pk + 1, B, N, d, n_ref, n_seq), b"coef must be 4-byte aligned"),
                      (lambda: upd(ph, pc, pR, n, 3, ps, B, N, 12, n_ref, n_seq), b"multiple of 8"),
                      (lambda: app(ph, pR, n, 0, pk, B, N, d, n_ref, n_seq), b"n_slots"),
                      (lambda: upd(ph, pc, pR, n, 4, ps, B, N, d, n_ref, n_seq), b"n_slots"),
                      (lambda: app(ph, pR, n - 8, 3, pk, B, N, d, n_ref, n_seq), b"slot_stride"),
                      (lambda: upd(ph, pc, pR, n + 2, 3, ps, B, N, d, n_ref, n_seq), b"multiple of 4"),
                      (lambda: app(ph, pR, n, 3, pk, B, N, d, 20, n_seq), b"noise rows"),
                      (lambda: upd(ph, pc, pR, 1 << 40, 3, ps, B, 1 << 28, 5120, 0, 1), b"2^31")):
        assert call() != 0, msg
        assert msg in lib.scail_last_error(), (msg, lib.scail_last_error())


# ---------------------------------------------------------------- 3. polynomial recovery through the cache's own logic
@pytest.mark.parametrize("order", [1, 2])
def test_forecast_recovers_polynomial_residuals(order):
    """Residuals exactly polynomial of degree `order` in sigma (built in fp64, stored in fp32) are written into the slots the
    cache names; the cache's coefficients must then reproduce the polynomial at the skipped step's sigma."""
    from scail_b200 import ops, sampler
    from scail_b200.step_cache import FirstBlockCache
    B, N, d, n_ref, n_seq = 2, 333, 136, 77, 211
    sig = [float(s) for s in sampler.make_flow_timesteps(50, 5.0)]
    g = torch.Generator(device="cuda").manual_seed(order)
    a = [torch.randn(B, n_seq, d, generator=g, device="cuda", dtype=torch.float64) * 2.0 ** e for e in (0, 2, 3)]
    poly = lambda s: a[0] + a[1] * s + (a[2] * s * s if order == 2 else 0.0)
    # computed at uneven intervals, more computed steps than slots (so the slots wrap), then skipped steps
    schedule = [(10, False), (11, False), (13, False), (14, False), (16, True), (17, True), (18, False), (19, False),
                (22, False), (25, True)]
    results = {}
    for o in (order, 0):
        c = FirstBlockCache(math.inf, order=o)
        bufs = c.workspace(B, N, d, n_ref, n_seq, "cuda")
        worst = 0.0
        for i, skip in schedule:
            c.set_sigma(sig[i])
            c.begin()
            c.threshold = math.inf if skip else 0.0
            assert c.decide(0.5) is skip
            c.stage(skip)
            R = poly(sig[i]).float()
            if not skip:
                if o == 0:
                    bufs.R.copy_(R)
                else:
                    s = int(bufs.ctl_slot.item())  # the slot the cache's update kernel would write
                    assert 0 <= s <= o
                    bufs.R_slots[s].copy_(R)
                c.computed()
                continue
            h = torch.zeros(B, N, d, device="cuda", dtype=torch.bfloat16)
            if o == 0:
                ops.step_cache_apply(h, bufs.R, n_ref)
                absum = bufs.R.double().abs()
            else:
                ops.step_cache_apply_forecast(h, bufs.R_slots, bufs.ctl_coef, n_ref)
                coef = bufs.ctl_coef.tolist()
                absum = sum(abs(cc) * bufs.R_slots[k].double().abs() for k, cc in enumerate(coef) if cc != 0.0)
            got = h[:, n_ref:n_ref + n_seq].double()
            exact = poly(sig[i])
            want = exact.to(torch.bfloat16).double()
            # Bound: the fp32 sum t differs from the exact polynomial by at most 5 roundings of 2^-24 relative to
            # sum|c_i R_i|: the fp32 residuals R_i, the fp32 coefficients c_i (fp64 evaluation error is far below that), each
            # product, and at most two sums (the final h + t is exact at h = 0).  bf16 rounding of t and of the exact value
            # then differ by at most one bf16 ulp at the larger magnitude (2^-7 relative to the binade's power of two).
            mag = torch.maximum(got.abs(), want.abs())
            ulp = torch.exp2(torch.floor(torch.log2(mag.clamp_min(2.0 ** -126))) - 7)
            bound = ulp + 5 * 2.0 ** -24 * absum
            worst = max(worst, float(((got - want).abs() / bound).max()))
        results[o] = worst
    print(f"order {order}: worst |forecast - bf16(exact)| / bound = {results[order]:.3f}; order 0 (hold): {results[0]:.1f}")
    assert results[order] <= 1.0
    assert results[0] > 10.0  # the hold misses the polynomial by far more than the rounding bound


# ---------------------------------------------------------------- 4. the model (small 2-layer config)
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
    uc = dict(crossattn=r(1, 24, 64))
    return x0, cond, uc


HOLD_PATTERN = [0.0, math.inf, math.inf, 0.0, math.inf]  # the order-0 forced pattern
FORECAST_PATTERN = [0.0, 0.0, 0.0, math.inf, math.inf, 0.0, math.inf, math.inf]


def test_order_0_is_bit_identical_to_the_plain_cache():
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(1)
    x0, cond, uc = sampler_inputs(1)
    sig = sampler.make_flow_timesteps(50, 5.0)
    a, b = FirstBlockCache(0.0), FirstBlockCache(0.0, order=0, max_skips=None)
    with torch.no_grad():
        xa, xb = x0.clone(), x0.clone()
        for i, thr in enumerate(HOLD_PATTERN):
            a.threshold = b.threshold = thr
            sampler.sampler_step(m, xa, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=a)
            sampler.sampler_step(m, xb, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=b)
            assert torch.equal(xa, xb), i
    assert a.history == b.history and [s for _, s in b.history] == [False, True, True, False, True]


@pytest.mark.parametrize("order", [1, 2])
def test_threshold_zero_is_bit_identical_to_no_cache(order):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(2)
    x0, cond, uc = sampler_inputs(2)
    c = FirstBlockCache(0.0, order=order)
    with torch.no_grad():
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=5)
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, step_cache=c)
    assert torch.equal(cached, plain)
    assert [s for _, s in c.history] == [False] * 5 and c.buffers.n_computed == 5


@pytest.mark.parametrize("order", [1, 2])
def test_forced_pattern_against_the_restatement(order):
    from scail_b200 import ops, sampler
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(3)
    x0, cond, uc = sampler_inputs(3)
    sig = sampler.make_flow_timesteps(50, 5.0)
    c, want = FirstBlockCache(0.0, order=order), RestatedForecastCache(m, order)
    ctx = sampler.prepare_context(cond, uc)
    kw = dict(ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
              image_clip_features=cond["image_clip_features"], concat_images=None)
    with torch.no_grad():
        x = x0.clone()
        for i, thr in enumerate(FORECAST_PATTERN):
            c.threshold = thr
            ts = torch.full((2,), float(sig[i]) * 1000.0, device="cuda")
            x2 = torch.cat([x, x])
            c.set_sigma(sig[i])
            v = m(x2, timesteps=ts, context=ctx, _step_cache=c, **kw).clone()
            vw = want.forward(thr, sig[i], x2, timesteps=ts, context=ctx, **kw)
            torch.cuda.synchronize()
            assert torch.equal(v, vw), f"step {i}"
            ops.cfg_euler_(x, v.contiguous(), 4.0, float(sig[i + 1]) - float(sig[i]))
    skipped = [thr == math.inf for thr in FORECAST_PATTERN]
    assert [s for _, s in c.history] == skipped == [s for _, s in want.history]
    for (a, _), (b, _) in zip(c.history, want.history):
        assert a == b or abs(a - b) <= 1e-6 * b, (a, b)
    assert c.buffers.n_computed == 4 and c.buffers.slot_sigma.count(None) == 0


@pytest.mark.parametrize("order", [0, 1, 2])
def test_max_skips_one_alternates(order):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(4)
    x0, cond, uc = sampler_inputs(4)
    c = FirstBlockCache(math.inf, order=order, max_skips=1)
    with torch.no_grad():
        sampler.sample(m, x0.clone(), cond, uc, num_steps=6, step_cache=c)
    assert [s for _, s in c.history] == [False, True] * 3


# ---------------------------------------------------------------- 5. graphs
@pytest.mark.parametrize("fast", [False, True], ids=["bf16", "fp8_window1"])
def test_graphed_step_is_bit_identical_to_eager(fast):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    kw = dict(fp8_linear=True, fp8_attention=True, attention_window=1) if fast else {}
    m = small_model(6, **kw)
    x0, cond, uc = sampler_inputs(7)
    sig = sampler.make_flow_timesteps(50, 5.0)
    ce, cg = FirstBlockCache(0.0, order=2), FirstBlockCache(0.0, order=2)
    pattern = FORECAST_PATTERN + [0.0, math.inf]
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, step_cache=cg)
        assert gs.kernels_in_graph > 20
        for i, thr in enumerate(pattern):
            if i == len(FORECAST_PATTERN):  # a new run with the same objects: the graphs are captured again
                ce.reset()
                cg.reset()
            ce.threshold = cg.threshold = thr
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=ce)
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(xe, xg), f"step {i}"
    assert ce.history == cg.history
    assert [s for _, s in cg.history] == [False, True]
