"""CFG cache Taylor forecast (CFGCache(order >= 1)): validation, the sigma requirement, the coefficients the cache hands to
each full and conditional-only step, slot rotation and the unchanged decision rule, without a GPU.  The kernel launchers
are replaced by recorders, so the host policy runs on CPU tensors."""
import math
import types

import numpy as np
import pytest
import torch

from test_cfg_cache_cpu import run

SHAPE = (1, 1, 16, 1, 2)


def test_order_validation():
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.step_cache import check_order
    assert CFGCache(0.1).order == 0
    for ok in (0, 1, 2, np.int64(2)):
        c = CFGCache(0.1, order=ok)
        assert c.order == int(ok) and type(c.order) is int
    for bad in (True, False, 1.0, "1", None, [1]):
        with pytest.raises(TypeError, match="cfg_cache order"):
            CFGCache(0.1, order=bad)
    for bad in (-1, 3, 7):
        with pytest.raises(ValueError, match="cfg_cache order must be 0, 1 or 2"):
            CFGCache(0.1, order=bad)
    # the default message is the first-block cache's, as before
    with pytest.raises(TypeError, match="^step cache order must be an int"):
        check_order(True)
    with pytest.raises(ValueError, match="^step cache order must be 0, 1 or 2"):
        check_order(3)


class Recorder:
    """Stands in for the kernel launchers: records what the cache hands them and sets the sums a full step reads back:
    num = `next_num`, and den = 1, or 0 where the kernel's reference is zero (the first full step)."""

    def __init__(self, monkeypatch):
        from scail_b200 import ops
        self.calls, self.next_num = [], 0.5

        def delta(v, d_ref, d_new, partials, out):
            first = not any(k[0] == "delta" for k in self.calls)
            self.calls.append(("delta",))
            out[:2] = torch.tensor([self.next_num, 0.0 if first else 1.0], dtype=torch.float64)

        def delta_forecast(v, slots, write_slot, coef, partials, out):
            assert slots.shape == (len(coef), *SHAPE)
            self.calls.append(("delta_forecast", write_slot, list(coef)))
            out[:2] = torch.tensor([self.next_num, 1.0 if any(coef) else 0.0], dtype=torch.float64)

        def euler_cached(x, c, delta, scale, dsigma):
            self.calls.append(("euler_cached",))

        def euler_forecast(x, c, slots, coef, scale, dsigma):
            self.calls.append(("euler_forecast", list(coef)))

        def unipc_forecast(x, x_last, c, dslots, dcoef, slots, write, scale, sigma, coef, correct):
            self.calls.append(("unipc_forecast", list(dcoef)))

        def unipc_pair(x, x_last, v, slots, write, scale, sigma, coef, correct):
            pass

        for name, fn in (("cfg_cache_delta", delta), ("cfg_cache_delta_forecast", delta_forecast),
                         ("cfg_euler_cached_", euler_cached), ("cfg_euler_cached_forecast_", euler_forecast),
                         ("unipc_step_cached_forecast_", unipc_forecast), ("unipc_step_", unipc_pair)):
            monkeypatch.setattr(ops, name, fn)


def drive(cache, sigmas, thresholds=None, solver=None):
    """The sampler's use of the cache over len(sigmas) - 1 steps on a CPU latent -> the cond_only pattern."""
    x = torch.zeros(SHAPE)
    v = torch.zeros(2, *SHAPE[1:], dtype=torch.bfloat16)
    pattern = []
    for i in range(len(sigmas) - 1):
        if thresholds is not None:
            cache.threshold = thresholds[i]
        co = cache.begin_step(x, sigmas[i])
        pattern.append(co)
        if co:
            cache.cond_update(x, v[1:2], 4.0, sigmas[i], sigmas[i + 1], solver)
        else:
            cache.full_step(v)
            if solver is not None:
                solver.step(x, v, 4.0, sigmas[i], sigmas[i + 1])
    return pattern


def lagrange(points, sigma, n_slots):
    """numpy's fp64 interpolating polynomial through points [(sigma_k, slot_k)]: the weight of each slot in its value at
    sigma (the polynomial through e_k at point k, evaluated at sigma)."""
    coef = [0.0] * n_slots
    if not points:
        return coef
    xs = np.array([p[0] for p in points], dtype=np.float64)
    for k, (_, slot) in enumerate(points):
        e = np.zeros(len(points))
        e[k] = 1.0
        coef[slot] = float(np.polyval(np.polyfit(xs, e, len(points) - 1), sigma))
    return coef


def expected(full, sigma, order):
    """The points a forecast at sigma goes through, given the full steps so far [(sigma_j, slot_j)]: the min(order + 1, j)
    most recent ones, fewer while their sigmas repeat."""
    m = min(order, len(full) - 1)
    while m > 0 and len({s for s, _ in full[-(m + 1):]}) < m + 1:
        m -= 1
    return full[-(m + 1):] if full else []


def close(got, want):
    """Each coefficient within one fp32 rounding (and numpy's fp64 noise) of numpy's; slots numpy does not use exactly 0."""
    return len(got) == len(want) and all(abs(g - w) <= 4e-7 * max(1.0, abs(w)) for g, w in zip(got, want)) and \
        all(g == 0.0 for g, w in zip(got, want) if w == 0.0)


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("max_skips", [1, 2])
def test_coefficients_handed_to_each_step(monkeypatch, order, max_skips):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    rec = Recorder(monkeypatch)
    sig = [float(s) for s in sampler.make_flow_timesteps(14, 5.0)]
    c = CFGCache(math.inf, max_skips=max_skips, order=order)
    pattern = drive(c, sig)
    assert pattern[:2] == [False, False] and any(pattern)
    full = []  # (sigma, slot) of every full step so far
    calls = iter(rec.calls)
    for i, co in enumerate(pattern):
        call = next(calls)
        pts = expected(full, sig[i], order)
        want = lagrange(pts, sig[i], order + 1)
        if co:
            assert call[0] == "euler_forecast" and close(call[1], want), (i, call, want)
            assert all(np.float32(x) == x for x in call[1])  # each an fp32 value
        else:
            slot = len(full) % (order + 1)
            assert call[0] == "delta_forecast" and call[1] == slot, (i, call)
            assert close(call[2], want), (i, call, want)
            if len(full) == 0:
                assert call[2] == [0.0] * (order + 1)  # the first full step: +inf indicator
            if len(full) == 1:
                assert call[2] == [1.0 if s == 0 else 0.0 for s in range(order + 1)]  # the hold: cfg_cache_delta's sums
            full.append((sig[i], slot))
    assert next(calls, None) is None
    assert c.buffers.slot_sigma == [next((s for s, sl in reversed(full) if sl == k), None) for k in range(order + 1)]


def test_forecast_goes_through_the_solver(monkeypatch):
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.unipc import UniPC
    rec = Recorder(monkeypatch)
    sig = [float(s) for s in sampler.make_flow_timesteps(6, 5.0)]
    s = UniPC(2)
    s.begin(sig)
    c = CFGCache(math.inf, max_skips=1, order=2)
    assert drive(c, sig, solver=s) == [False, False, True, False, True, False]
    kinds = [k[0] for k in rec.calls]
    assert kinds == ["delta_forecast", "delta_forecast", "unipc_forecast", "delta_forecast", "unipc_forecast", "delta_forecast"]
    assert close(rec.calls[2][1], lagrange([(sig[0], 0), (sig[1], 1)], sig[2], 3))
    assert close(rec.calls[4][1], lagrange([(sig[0], 0), (sig[1], 1), (sig[3], 2)], sig[4], 3))
    with pytest.raises(ValueError, match="delta or forecast"):
        s.step(torch.zeros(SHAPE), None, 4.0, sig[5], sig[6], delta=torch.zeros(SHAPE), forecast=(None, [1.0]))


def test_order_zero_runs_the_hold_kernels(monkeypatch):
    from scail_b200.cfg_cache import CFGCache
    rec = Recorder(monkeypatch)
    c = CFGCache(math.inf, max_skips=1)
    assert drive(c, [0.9, 0.8, 0.7, 0.6, 0.5]) == [False, False, True, False]
    assert [k[0] for k in rec.calls] == ["delta", "delta", "euler_cached", "delta"]
    assert c.buffers.slots is None and c.buffers.d_ref is c.delta
    assert c.buffers.nbytes() == 2 * 4 * math.prod(SHAPE)
    c2 = CFGCache(math.inf, order=2)
    drive(c2, [0.9, 0.8])
    assert c2.buffers.nbytes() == 3 * 4 * math.prod(SHAPE) and c2.buffers.d_ref is None


@pytest.mark.parametrize("order", [1, 2])
def test_degree_reduction_on_repeated_sigma(monkeypatch, order):
    from scail_b200.cfg_cache import CFGCache
    rec = Recorder(monkeypatch)
    c = CFGCache(0.0, order=order)
    sig = [0.9, 0.9, 0.9, 0.8, 0.8, 0.7, 0.6]
    drive(c, sig)
    got = [k[2] for k in rec.calls]
    n = order + 1
    e = lambda *pairs: [dict(pairs).get(s, 0.0) for s in range(n)]
    assert got[0] == [0.0] * n
    assert got[1] == e((0, 1.0))  # one point: the hold
    assert got[2] == e((1, 1.0))  # two points at one sigma: reduced to the newest
    want3 = e((2 % n, 1.0))  # the newest two (and three) share sigma 0.9: the hold of the newest
    assert got[3] == want3
    # step 4 at 0.8: points 0.8 (step 3), 0.9 (step 2)[, 0.9 (step 1)]: degree 1 at most
    assert close(got[4], lagrange([(0.9, 2 % n), (0.8, 3 % n)], 0.8, n))
    # step 5 at 0.7: newest two share sigma 0.8: degree 0, the hold of step 4
    assert got[5] == e((4 % n, 1.0))


@pytest.mark.parametrize("order", [1, 2])
def test_slots_rotate_and_reset_drops_them(monkeypatch, order):
    from scail_b200.cfg_cache import CFGCache
    rec = Recorder(monkeypatch)
    c = CFGCache(0.0, order=order)
    sig = [1.0 - 0.05 * i for i in range(12)]
    drive(c, sig)
    n = order + 1
    assert [k[1] for k in rec.calls] == [j % n for j in range(11)]
    assert c.buffers.n_full == 11
    assert c.buffers.slot_sigma == [sig[max(j for j in range(11) if j % n == s)] for s in range(n)]
    assert c.delta.data_ptr() == c.buffers.slots[10 % n].data_ptr()
    c.reset()
    assert c.buffers is None and c.delta is None and c.history == []
    rec.calls.clear()
    drive(c, sig[:3])
    assert [k[1] for k in rec.calls] == [0, 1 % n] and rec.calls[0][2] == [0.0] * n
    # a latent of another shape drops the slots and their sigmas
    x2 = torch.zeros(1, 2, 16, 1, 2)
    c.begin_step(x2, 0.5)
    assert c.buffers is None


def test_sigma_is_required_at_order_one_and_two():
    from scail_b200.cfg_cache import CFGCache
    x = torch.zeros(SHAPE)
    for order in (1, 2):
        c = CFGCache(math.inf, order=order)
        with pytest.raises(ValueError, match="cfg_cache.*sigma"):
            c.begin_step(x)
        assert c.history == [] and c.buffers is None  # nothing was recorded
        with pytest.raises(ValueError, match="cfg_cache sigma must be finite"):
            c.begin_step(x, math.nan)
        with pytest.raises(TypeError, match="cfg_cache sigma"):
            c.begin_step(x, True)
        assert c.history == []
        assert c.begin_step(x, torch.tensor(0.5)) is False and c.history == [(None, False)]
    c0 = CFGCache(math.inf)
    assert c0.begin_step(x) is False  # order 0 needs no sigma, as before


def test_sampler_and_graphed_step_pass_sigma(monkeypatch):
    """sampler_step hands the cache its sigma (the override when one is given) before anything runs."""
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    seen = []
    c = CFGCache(math.inf, order=1)

    def begin_step(x, sigma=None):
        seen.append(float(sigma))
        raise RuntimeError("stop")

    monkeypatch.setattr(c, "begin_step", begin_step)
    model = types.SimpleNamespace()
    x = torch.zeros(SHAPE)
    cond = dict(crossattn=torch.zeros(1, 4, 64), ref_concat=None, concat_smpl_render=None, image_clip_features=None)
    for kw, want in ((dict(), 0.75), (dict(_sigma_override=0.3), 0.3)):
        with pytest.raises(RuntimeError, match="stop"):
            sampler.sampler_step(model, x, torch.tensor(0.75), 0.5, cond, dict(crossattn=torch.zeros(1, 4, 64)),
                                 cfg_cache=c, **kw)
        assert seen[-1] == pytest.approx(want)
    import inspect
    src = inspect.getsource(sampler.GraphedStep.__call__)
    assert "cc.begin_step(self.x, sigma)" in src


@pytest.mark.parametrize("order", [0, 1, 2])
def test_decision_sequences_and_history_unchanged(order):
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(math.inf, order=order)
    assert run(c, [math.inf, 0.3], 8) == [False, False] + [True] * 6
    assert c.history == [(None, False), (math.inf, False)] + [(0.3, True)] * 6
    c = CFGCache(0.0, order=order)
    assert run(c, [math.inf, 0.0, 1e-12, 0.5, 0.0, 0.0], 6) == [False] * 6
    c = CFGCache(math.inf, order=order)
    assert run(c, [math.inf, math.nan, math.nan, 0.1], 6) == [False, False, False, False, True, True]
    assert run(CFGCache(math.inf, max_skips=0, order=order), [math.inf] + [0.1] * 10, 8) == [False] * 8
    assert run(CFGCache(math.inf, max_skips=1, order=order), [math.inf] + [0.1] * 10, 9) == \
        [False, False, True, False, True, False, True, False, True]
    c = CFGCache(0.0, order=order)
    th = [0.0, 0.0, 0.0, 0.5, 0.5, 0.05, 0.5, math.inf]
    assert run(c, [math.inf, 0.2, 0.1, 0.3], 8, th) == [False, False, False, True, True, False, True, True]
    assert all(isinstance(h, tuple) and len(h) == 2 and type(h[1]) is bool for h in c.history)


@pytest.mark.parametrize("order", [1, 2])
def test_driven_history_matches_order_zero(monkeypatch, order):
    """The same indicators through the whole begin_step / full_step cycle give the same history at every order."""
    from scail_b200.cfg_cache import CFGCache
    rec = Recorder(monkeypatch)
    sig = [1.0 - 0.07 * i for i in range(11)]
    th = [math.inf, math.inf, 0.6, 0.4, math.inf, 0.0, math.inf, 0.6, 0.6, 0.6]
    hist = []
    for o in (0, order):
        rec.next_num = 0.5
        c = CFGCache(0.0, max_skips=2, order=o)
        drive(c, sig, th)
        hist.append(c.history)
    assert hist[0] == hist[1]
    assert [co for _, co in hist[0]] == [False, False, True, False, True, False, True, True, False, True]
