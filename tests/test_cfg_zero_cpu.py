"""CFG-Zero* guidance without a GPU: argument validation, the step-counting rule, the refusals, zero-initialised steps that
run no forward and tell no cache, sample_long's skipped steps, and the fp64 oracle's own properties."""
import inspect
import math
import types

import numpy as np
import pytest
import torch

import cfg_zero_oracle as Z


def test_zero_init_steps_validation():
    from scail_b200.guidance import CFGZeroStar
    for bad in (True, False, 1.0, 0.5, -1, "1", None):
        with pytest.raises(ValueError, match="zero_init_steps"):
            CFGZeroStar(bad)
    for ok in (0, 1, 2, 7, np.int64(3)):
        assert CFGZeroStar(ok).zero_init_steps == int(ok)
    assert CFGZeroStar().zero_init_steps == 1


@pytest.mark.parametrize("k", [0, 1, 2, 5])
def test_step_counting_across_reset(k):
    from scail_b200.guidance import CFGZeroStar
    g = CFGZeroStar(k)
    for _ in range(2):
        got = [g.begin_step() for _ in range(7)]
        assert got == [Z.zero_init(i, k) for i in range(7)]
        assert g.step_index == 7
        g.reset()
        assert g.step_index == 0 and g.last_scale is None


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
    from scail_b200.guidance import CFGZeroStar, check_supported
    g = CFGZeroStar(1)
    m = _tiny_model()
    x, cond, uc = _inputs()
    ad = m.mixins["adaln_layer"]
    ad.cp = types.SimpleNamespace(size=2, rank=0)
    with pytest.raises(NotImplementedError, match="guidance.*context parallelism"):
        sampler.sample(m, x, cond, uc, num_steps=1, guidance=g)
    with pytest.raises(NotImplementedError, match="guidance.*context parallelism"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, guidance=g)
    with pytest.raises(NotImplementedError, match="guidance.*context parallelism"):
        sampler.GraphedStep(m, x, cond, uc, guidance=g)
    with pytest.raises(NotImplementedError, match="guidance.*context parallelism"):
        sampler.guided_velocity(m, x, 0.5, cond, uc, guidance=g)
    with pytest.raises(NotImplementedError, match="guidance.*context parallelism"):
        sampler.sample_long(m, x, dict(cond, smpl_tiled=None), uc, [[0]], num_steps=1, guidance=g)
    ad.cp = types.SimpleNamespace(size=1, rank=0)  # a group of one is a single GPU
    check_supported(ad.cp)
    ad.cp = None
    with pytest.raises(NotImplementedError, match="guidance.*chunk_dim"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, guidance=g, chunk_dim=3)
    with pytest.raises(TypeError, match="guidance"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, guidance=0)
    with pytest.raises(TypeError, match="guidance"):
        sampler.sample(m, x, cond, uc, num_steps=1, guidance="cfg-zero*")
    assert g.step_index == 0 and g.last_scale is None  # nothing ran


def test_every_entry_point_takes_it_with_default_none():
    from scail_b200 import cfg_cache, sampler
    for f in (sampler.sample, sampler.sampler_step, sampler.GraphedStep, sampler.sample_long, sampler.guided_velocity,
              cfg_cache.CFGCache.cond_update):
        assert inspect.signature(f).parameters["guidance"].default is None, f


class _NoForward:
    """A model stand-in that fails if a forward is attempted."""
    calls = 0

    def __call__(self, *a, **kw):
        _NoForward.calls += 1
        raise AssertionError("a zero-initialised step ran a forward")


def test_zero_initialised_step_runs_nothing_and_tells_no_cache():
    from scail_b200 import sampler
    from scail_b200.cfg_cache import CFGCache
    from scail_b200.guidance import CFGZeroStar
    from scail_b200.step_cache import FirstBlockCache
    g, cc, fb = CFGZeroStar(2), CFGCache(math.inf), FirstBlockCache(0.1)
    x, cond, uc = _inputs()
    x.normal_()
    before = x.clone()
    for i in range(2):
        out = sampler.sampler_step(_NoForward(), x, 0.9 - 0.1 * i, 0.8 - 0.1 * i, cond, uc, guidance=g, cfg_cache=cc,
                                   step_cache=fb)
        assert out is x
    assert torch.equal(x, before) and _NoForward.calls == 0
    assert cc.history == [] and cc.buffers is None and fb.history == []
    assert g.step_index == 2 and g.last_scale is None
    with pytest.raises(AssertionError, match="zero-initialised"):  # step 2 is guided: it needs the forward
        sampler.sampler_step(_NoForward(), x, 0.7, 0.6, cond, uc, guidance=g)


@pytest.mark.parametrize("k", [0, 1, 2])
def test_sample_long_skips_zero_initialised_steps(k):
    """sample_long with a denoise override: steps 0 .. k-1 run no window and leave x as it is; the other steps are the plain
    loop's steps."""
    from scail_b200 import sampler
    from scail_b200.guidance import CFGZeroStar
    gen = torch.Generator().manual_seed(3)
    T, seg, h, w, n = 5, 3, 4, 4, 4
    tiles = sampler.make_tile_indices(T, seg, 2)
    x0 = torch.randn(1, T, 16, h, w, generator=gen)
    cond = dict(crossattn=torch.zeros(1, 2, 8), smpl_tiled=torch.randn(1, len(tiles), seg, 16, h // 2, w // 2, generator=gen))
    uc = dict(crossattn=torch.zeros(1, 2, 8))
    seen = []

    def denoise(x_tile, sigma, c_k, u_k):
        seen.append(float(sigma))
        return 0.5 * x_tile - c_k["concat_smpl_render"].mean() * float(sigma)

    g = CFGZeroStar(k)
    got = sampler.sample_long(None, x0.clone(), cond, uc, tiles, num_steps=n, denoise=denoise, guidance=g)
    sig = sampler.make_flow_timesteps(n, 5.0)
    assert seen == [float(sig[i]) for i in range(k, n) for _ in tiles]
    want = x0.clone()
    for i in range(k, n):
        want = sampler.sampler_step_long(denoise, want, sig[i], sig[i + 1], tiles, cond["smpl_tiled"], dict(cond), dict(uc))
    assert torch.equal(got, want)
    assert g.step_index == n


def test_oracle_scale_is_the_least_squares_projection():
    rng = np.random.default_rng(0)
    u = rng.standard_normal(1000)
    c = 0.7 * u + 0.2 * rng.standard_normal(1000)
    s = Z.optimized_scale(u, c)
    err = lambda t: np.sum((c - t * u) ** 2)
    assert err(s) <= min(err(s * (1 + 1e-6)), err(s * (1 - 1e-6)))
    assert Z.optimized_scale(np.zeros(8), c[:8]) == 0.0
    assert np.array_equal(Z.guided_velocity(np.zeros(8), c[:8], 4.0, 0.0), 4.0 * c[:8])
    assert np.allclose(Z.guided_velocity(u, c, 4.0, 1.0), u + 4.0 * (c - u), rtol=0, atol=1e-12)
    assert math.isnan(Z.optimized_scale(u, np.where(np.arange(1000) == 5, np.nan, c)))
