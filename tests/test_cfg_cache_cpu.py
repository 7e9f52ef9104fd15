"""CFG cache: the host-side policy (scail_b200.cfg_cache), the conditioning row lookup and the refusals, without a GPU."""
import math
import types

import pytest
import torch


def test_threshold_validation():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(0)
    assert c.threshold == 0.0 and isinstance(c.threshold, float)
    for ok in (0.0, 0.05, 3, math.inf, float("inf")):
        c.threshold = ok
        assert c.threshold == float(ok)
    for bad in (True, False, "0.1", None, [0.1], 1j):
        with pytest.raises(TypeError, match="cfg_cache threshold"):
            CFGCache(bad)
        with pytest.raises(TypeError, match="cfg_cache threshold"):
            c.threshold = bad
    for bad in (-1e-9, -1, -math.inf, math.nan):
        with pytest.raises(ValueError, match="cfg_cache threshold"):
            CFGCache(bad)
        with pytest.raises(ValueError, match="cfg_cache threshold"):
            c.threshold = bad
    assert c.threshold == math.inf  # a refused value leaves the last good one


def test_max_skips_validation():
    from scail_b200.cfg_cache import CFGCache
    assert CFGCache(0.1).max_skips is None
    for ok in (0, 1, 7):
        assert CFGCache(0.1, max_skips=ok).max_skips == ok
    for bad in (True, 1.0, "1", [1]):
        with pytest.raises(TypeError, match="cfg_cache max_skips"):
            CFGCache(0.1, max_skips=bad)
    with pytest.raises(ValueError, match="cfg_cache max_skips"):
        CFGCache(0.1, max_skips=-1)


def run(c, full_indicators, n, thresholds=None):
    """The sampler's use of the policy over n steps: before each step decide on the indicator of the last full step (None
    until one ran); each full step yields the next value of `full_indicators`.  -> the cond_only pattern."""
    it = iter(full_indicators)
    ind, out = None, []
    for i in range(n):
        if thresholds is not None:
            c.threshold = thresholds[i]
        co = c.decide(ind)
        out.append(co)
        if not co:
            ind = next(it)
    return out


def test_two_full_steps_then_threshold_inf_skips_every_later_step():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(math.inf)
    # a zero-filled delta_ref makes the first full step's indicator +inf, which is never < inf
    assert run(c, [math.inf, 0.3], 8) == [False, False] + [True] * 6
    assert c.history == [(None, False), (math.inf, False)] + [(0.3, True)] * 6


def test_threshold_zero_never_skips():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(0.0)
    assert run(c, [math.inf, 0.0, 1e-12, 0.5, 0.0, 0.0], 6) == [False] * 6
    assert [i for i, _ in c.history] == [None, math.inf, 0.0, 1e-12, 0.5, 0.0]


def test_nan_never_skips():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(math.inf)
    assert run(c, [math.inf, math.nan, math.nan, 0.1], 6) == [False, False, False, False, True, True]
    assert math.isnan(c.history[2][0]) and c.history[2][1] is False


def test_max_skips_zero_and_one():
    from scail_b200.cfg_cache import CFGCache
    assert run(CFGCache(math.inf, max_skips=0), [math.inf] + [0.1] * 10, 8) == [False] * 8
    c = CFGCache(math.inf, max_skips=1)
    assert run(c, [math.inf] + [0.1] * 10, 9) == [False, False, True, False, True, False, True, False, True]
    assert run(CFGCache(math.inf, max_skips=2), [math.inf] + [0.1] * 10, 8) == [False, False, True, True, False, True, True,
                                                                                 False]


def test_threshold_changed_between_steps():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(0.0)
    th = [0.0, 0.0, 0.0, 0.5, 0.5, 0.05, 0.5, math.inf]
    got = run(c, [math.inf, 0.2, 0.1, 0.3], 8, th)
    # step 3 decides on 0.1 (step 2's) < 0.5; step 5 on 0.1 against 0.05: full -> 0.3; step 6: 0.3 < 0.5; step 7: inf
    assert got == [False, False, False, True, True, False, True, True]
    assert [i for i, _ in c.history] == [None, math.inf, 0.2, 0.1, 0.1, 0.1, 0.3, 0.3]


def test_reset_drops_state_and_history():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(math.inf, max_skips=1)
    run(c, [math.inf, 0.1, 0.1], 4)
    c.buffers = object()
    c._pending = True
    c.reset()
    assert c.history == [] and c.buffers is None and c.delta is None and not c._pending
    assert run(c, [math.inf, 0.1], 3) == [False, False, True]  # the two-full-steps start again, the skip run restarted
    assert c.history[0] == (None, False)


def test_history_format():
    from scail_b200.cfg_cache import CFGCache
    c = CFGCache(0.5)
    run(c, [math.inf, 0.25], 3)
    assert all(isinstance(h, tuple) and len(h) == 2 and type(h[1]) is bool for h in c.history)
    assert c.history == [(None, False), (math.inf, False), (0.25, True)]


def test_conditioning_row_lookup():
    from scail_b200.dit import Conditioning
    Lt, Lc, d = 3, 5, 8
    ctx, clip_feats = torch.randn(2, Lt, 16), torch.randn(1, 257, 32)
    cond = Conditioning(ctx, clip_feats, 2)
    cond.text, cond.clip = torch.randn(2, Lt, d), torch.randn(2, Lc, d)
    cond.xkv = [(torch.randn(2 * Lt, 2 * d), torch.randn(2 * Lc, 2 * d)) for _ in range(3)]
    assert cond.lookup(ctx, clip_feats, 2) is cond
    r = cond.lookup(ctx[1:2], clip_feats, 1)
    assert r is not None and r is cond.lookup(ctx[1:2], clip_feats, 1)  # one handle per row
    assert torch.equal(r.text, cond.text[1:2]) and torch.equal(r.clip, cond.clip[1:2])
    assert r.text.data_ptr() == cond.text[1].data_ptr()  # views: nothing copied
    for (tk, ck), (rt, rc) in zip(cond.xkv, r.xkv):
        assert torch.equal(rt, tk[Lt:]) and torch.equal(rc, ck[Lc:]) and rt.data_ptr() == tk[Lt].data_ptr()
    r0 = cond.lookup(ctx[0:1], clip_feats, 1)
    assert torch.equal(r0.text, cond.text[:1]) and torch.equal(r0.xkv[0][1], cond.xkv[0][1][:Lc])
    assert cond.lookup(ctx[1:2].clone(), clip_feats, 1) is None  # another tensor object: never matched by address
    assert cond.lookup(ctx[1:2], clip_feats.clone(), 1) is None
    assert cond.lookup(ctx[1:2], clip_feats, 2) is None
    assert cond.lookup(ctx[:, :2], clip_feats, 1) is None  # not a batch row
    assert cond.lookup(ctx[1:2, :, :8], clip_feats, 1) is None
    ctx.add_(1.0)  # an edited prompt tensor is stale for the handle and its rows
    assert cond.lookup(ctx[1:2], clip_feats, 1) is None and cond.lookup(ctx, clip_feats, 2) is None


def _tiny_model():
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    return DiffusionTransformer(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=2, text_dim=64,
                                time_embed_dim=256).eval()


def _inputs(t=1, h=8, w=8):
    x = torch.zeros(1, t, 16, h, w)
    cond = dict(crossattn=torch.zeros(1, 4, 64), ref_concat=torch.zeros(1, 1, 16, h, w),
                concat_smpl_render=torch.zeros(1, t, 16, h // 2, w // 2), image_clip_features=torch.zeros(1, 257, 1280))
    return x, cond, dict(crossattn=torch.zeros(1, 4, 64))


def test_refusals_before_anything_runs():
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache, check_supported
    c = CFGCache(0.1)
    m = _tiny_model()
    x, cond, uc = _inputs()
    ad = m.mixins["adaln_layer"]
    ad.cp = types.SimpleNamespace(size=2, rank=0)
    with pytest.raises(NotImplementedError, match="cfg_cache"):
        sampler.sample(m, x, cond, uc, num_steps=1, cfg_cache=c)
    with pytest.raises(NotImplementedError, match="cfg_cache"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, cfg_cache=c)
    with pytest.raises(NotImplementedError, match="cfg_cache"):
        sampler.GraphedStep(m, x, cond, uc, cfg_cache=c)
    ad.cp = types.SimpleNamespace(size=1, rank=0)  # a group of one is a single GPU
    check_supported(ad.cp)
    ad.cp = None
    plan = types.SimpleNamespace(branch=1)
    with pytest.raises(NotImplementedError, match="cfg_cache.*HybridParallel"):
        sampler.sample(m, x, cond, uc, num_steps=1, plan=plan, cfg_cache=c)
    with pytest.raises(NotImplementedError, match="cfg_cache.*HybridParallel"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, plan=plan, cfg_cache=c)
    with pytest.raises(NotImplementedError, match="cfg_cache.*chunk_dim"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, cfg_cache=c, chunk_dim=3)
    with pytest.raises(NotImplementedError, match="cfg_cache.*_num_layers"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, cfg_cache=c, _num_layers=1)
    with pytest.raises(TypeError, match="cfg_cache"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, cfg_cache=0.1)
    with pytest.raises(TypeError, match="cfg_cache"):
        sampler.sample(m, x, cond, uc, num_steps=1, cfg_cache="on")
    assert c.history == [] and c.buffers is None  # nothing ran


def test_solver_validation_precedes_the_decision():
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.unipc import UniPC
    c, s = CFGCache(math.inf), UniPC(2)
    s.begin(sampler.make_flow_timesteps(4, 5.0))
    x, cond, uc = _inputs()
    with pytest.raises(ValueError, match="solver"):
        sampler.sampler_step(_tiny_model(), x, 0.5, 0.25, cond, uc, solver=s, cfg_cache=c)
    assert c.history == []


def test_sample_long_does_not_take_it():
    import inspect
    from scail_b200 import sampler
    assert "cfg_cache" not in inspect.signature(sampler.sample_long).parameters
    for f in (sampler.sample, sampler.sampler_step, sampler.GraphedStep):
        assert inspect.signature(f).parameters["cfg_cache"].default is None
