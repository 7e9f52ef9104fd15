"""First-block residual cache: the host-side policy (scail_b200.step_cache) and the refusals, without a GPU."""
import math
import types

import pytest
import torch


def test_threshold_validation():
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(0)
    assert c.threshold == 0.0 and isinstance(c.threshold, float)
    for ok in (0.0, 0.05, 3, math.inf, float("inf")):
        c.threshold = ok
        assert c.threshold == float(ok)
    for bad in (True, False, "0.1", None, [0.1], 1j):
        with pytest.raises(TypeError):
            FirstBlockCache(bad)
        with pytest.raises(TypeError):
            c.threshold = bad
    for bad in (-1e-9, -1, -math.inf, math.nan):
        with pytest.raises(ValueError):
            FirstBlockCache(bad)
        with pytest.raises(ValueError):
            c.threshold = bad
    assert c.threshold == math.inf  # a refused value leaves the last good one


def test_indicator_from_sums():
    from scail_b200.step_cache import indicator
    assert indicator(1.0, 4.0) == 0.25
    assert indicator(0.0, 4.0) == 0.0
    assert indicator(1.0, 0.0) == math.inf
    assert indicator(0.0, 0.0) == math.inf  # zero denominator, even with a zero numerator
    assert math.isnan(indicator(math.nan, 1.0))
    assert math.isnan(indicator(math.inf, math.inf))
    assert indicator(math.inf, 1.0) == math.inf


def _geometry(c, B=2, N=40, d=16, n_ref=8, n_seq=24):
    return c.workspace(B, N, d, n_ref, n_seq, "cpu")


def test_decision_rule_over_scripted_indicators():
    from scail_b200.step_cache import FirstBlockCache, indicator
    c = FirstBlockCache(0.1)
    b = _geometry(c)
    assert b.r_ref.abs().sum() == 0 and b.h1.shape == (2, 40, 16) and b.R.shape == (2, 24, 16) and b.R.dtype == torch.float32
    assert not c.decide(0.0)  # no state yet: computes, however small the indicator
    c.computed()
    script = [(0.05, 0.1, True), (0.1, 0.1, False), (0.099, 0.1, True), (math.nan, 0.1, False), (math.nan, math.inf, False),
              (indicator(1.0, 0.0), 0.1, False), (indicator(1.0, 0.0), math.inf, False), (1e30, math.inf, True),
              (0.0, 0.0, False), (1e-12, 0.0, False), (0.0, 1e-12, True)]
    for ind, thr, want in script:
        c.threshold = thr
        assert c.decide(ind) is want, (ind, thr)
    hist = c.history[1:]
    assert len(c.history) == 1 + len(script)
    assert [s for _, s in hist] == [w for _, _, w in script]
    assert c.history[0] == (0.0, False)


def test_skip_updates_nothing_and_compute_swaps_buffers():
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(math.inf)
    b = _geometry(c)
    r0, r1 = b.r_ref, b.r_new
    assert not c.decide(1.0)
    c.computed()
    assert b.r_ref is r1 and b.r_new is r0 and c.has_state
    assert c.decide(5.0)  # a skip: no swap, no state change
    assert b.r_ref is r1 and b.r_new is r0
    c.threshold = 0
    assert not c.decide(5.0)
    c.computed()
    assert b.r_ref is r0 and b.r_new is r1


def test_reset_and_geometry_or_batch_change_invalidate_state():
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(math.inf)
    b = _geometry(c)
    c.decide(1.0)
    c.computed()
    assert _geometry(c) is b and c.decide(1.0)  # same key: state kept
    c.reset()
    assert c.buffers is None and c.history == [] and not c.has_state
    b = _geometry(c)
    assert not c.decide(1.0)  # after a reset the next forward computes
    c.computed()
    for change in (dict(B=1), dict(N=48), dict(d=32), dict(n_ref=4), dict(n_seq=20)):
        b2 = _geometry(c, **change)
        assert b2 is not b and not c.has_state
        assert not c.decide(0.0), change  # a new geometry or batch computes first
        c.computed()
        assert c.decide(0.0)
        b = _geometry(c)  # back to the default key: also new
        assert not c.has_state
        c.decide(1.0)
        c.computed()
    assert len(c.history) == 1 + 3 * 5  # history runs across geometry changes: only reset() clears it


def test_workspace_memory_at_14b_width():
    """Bytes of h1, r_ref, r_new (bf16 [B, N, d]), h1c (bf16) and R (fp32) over the noise rows, as DESIGN §3.4 states them."""
    def nbytes(B, N, d, n_seq):
        return 3 * B * N * d * 2 + B * n_seq * d * (2 + 4)
    assert round(nbytes(2, 27904, 5120, 21 * 1024) / 1e9, 2) == 3.04
    assert round(nbytes(2, 48832, 5120, 21 * 1792) / 1e9, 2) == 5.31
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(0)
    assert _geometry(c, B=2, N=40, d=16, n_seq=24).nbytes() == nbytes(2, 40, 16, 24)


# ---------------------------------------------------------------- refusals (raised before anything touches a device)
def _tiny_model():
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    return DiffusionTransformer(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=2, text_dim=64,
                                time_embed_dim=256).eval()


def _inputs(b=2, t=1, h=8, w=8):
    x = torch.zeros(b, t, 16, h, w)
    kw = dict(timesteps=torch.zeros(b), context=torch.zeros(b, 4, 64), ref_concat=torch.zeros(1, 1, 16, h, w),
              concat_smpl_render=torch.zeros(1, t, 16, h // 2, w // 2), image_clip_features=torch.zeros(1, 257, 1280))
    return x, kw


def test_refusals():
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache, check_supported
    c = FirstBlockCache(0.1)
    m = _tiny_model()
    x, kw = _inputs()
    with pytest.raises(NotImplementedError, match="step_cache"):
        m(x, _step_cache=c, chunk_dim=3, **kw)
    with pytest.raises(NotImplementedError, match="step_cache"):
        m(x, _step_cache=c, _num_layers=1, **kw)
    m.mixins["adaln_layer"].cp = types.SimpleNamespace(size=2, rank=0)
    with pytest.raises(NotImplementedError, match="step_cache"):
        m(x, _step_cache=c, **kw)
    cond = dict(crossattn=torch.zeros(1, 4, 64), ref_concat=kw["ref_concat"], concat_smpl_render=kw["concat_smpl_render"],
                image_clip_features=kw["image_clip_features"])
    uc = dict(crossattn=torch.zeros(1, 4, 64))
    with pytest.raises(NotImplementedError, match="step_cache"):
        sampler.sample(m, x[:1], cond, uc, num_steps=1, step_cache=c)
    m.mixins["adaln_layer"].cp = types.SimpleNamespace(size=1, rank=0)  # a group of one is a single GPU
    check_supported(m.mixins["adaln_layer"].cp)
    plan = types.SimpleNamespace(branch=0)
    with pytest.raises(NotImplementedError, match="step_cache"):
        sampler.sample(m, x[:1], cond, uc, num_steps=1, plan=plan, step_cache=c)
    with pytest.raises(NotImplementedError, match="step_cache"):
        sampler.sampler_step(m, x[:1], 1.0, 0.9, cond, uc, plan=plan, step_cache=c)
    assert c.history == [] and c.buffers is None  # nothing ran
    with pytest.raises(NotImplementedError, match="step_cache"):
        sampler.GraphedStep(_with_cp(m), x[:1], cond, uc, step_cache=c)
    # without a cache, the CPU forward still refuses for want of CUDA, as before
    m.mixins["adaln_layer"].cp = None
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x, **kw)


def _with_cp(m):
    m.mixins["adaln_layer"].cp = types.SimpleNamespace(size=2, rank=0)
    return m
