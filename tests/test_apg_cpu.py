"""APG guidance without a GPU: the fp64 oracle's own properties (vanilla CFG as a special case, orthogonality, the norm
threshold, the momentum recurrence), argument validation, the refusals, and the ops' lack of a CPU path."""
import inspect
import math
import types

import numpy as np
import pytest
import torch

import apg_oracle as A


def _pair(T=4, h=3, w=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(1, T, 16, h, w, generator=g, dtype=torch.float64)
    u = torch.randn(1, T, 16, h, w, generator=g, dtype=torch.float64)
    c = 0.8 * u + 0.5 * torch.randn(1, T, 16, h, w, generator=g, dtype=torch.float64)
    return x, u, c


def test_oracle_is_vanilla_cfg_at_eta_1():
    x, u, c = _pair()
    for sigma, nxt, scale in ((0.9, 0.85, 4.0), (0.3, 0.0, 7.5), (0.05, 0.01, 1.0)):
        parts = A.apg_parts(x, u, c, sigma, scale, 1.0)
        got = A.euler(x, parts["D_g"], sigma, nxt)
        want = A.vanilla_cfg_euler(x, u, c, scale, sigma, nxt)
        assert torch.allclose(got, want, rtol=0, atol=1e-12 * float(want.abs().max())), float((got - want).abs().max())
        # and the data prediction itself: D_c + (w - 1) (D_c - D_u)
        dg = x - sigma * c + (scale - 1.0) * (sigma * (u - c))
        assert torch.allclose(parts["D_g"], dg, rtol=0, atol=1e-12 * float(dg.abs().max()))


def test_oracle_projection_is_orthogonal_per_frame():
    x, u, c = _pair(T=5)
    c[0, 3] *= 1000.0  # a large frame: per-frame sums must not see it elsewhere
    parts = A.apg_parts(x, u, c, 0.7, 5.0, 0.0, norm_threshold=3.0)
    T = x.shape[1]
    orth, dc, par = (parts[k].reshape(T, -1) for k in ("orth", "D_c", "par"))
    for t in range(T):
        cos = float(orth[t] @ dc[t]) / (float(orth[t].norm()) * float(dc[t].norm()))
        assert abs(cos) < 1e-12, (t, cos)
        assert torch.allclose(orth[t] + par[t], parts["diff"].reshape(T, -1)[t], rtol=0, atol=1e-12)
    # eta = 0 drops the parallel part: D_g - D_c = (w - 1) orth
    assert torch.allclose(parts["D_g"] - parts["D_c"], 4.0 * parts["orth"], rtol=0, atol=1e-9)


def test_oracle_norm_threshold_per_frame():
    x, u, c = _pair(T=6)
    u[0, 2] = c[0, 2]  # diff = 0: the factor is 1
    raw = A.apg_parts(x, u, c, 0.6, 4.0, 0.5)["diff"].reshape(6, -1).norm(dim=1)
    r = float(raw[raw > 0].median())  # some frames above r, some at or below it
    parts = A.apg_parts(x, u, c, 0.6, 4.0, 0.5, norm_threshold=r)
    norms = parts["diff"].reshape(6, -1).norm(dim=1)
    assert bool((norms <= r * (1 + 1e-12)).all()), norms
    for t in range(6):
        want = 1.0 if raw[t] <= r else r / float(raw[t])
        assert abs(float(parts["f"][t]) - want) <= 1e-15, t
    assert float(parts["f"][2]) == 1.0 and float(raw[2]) == 0.0
    assert bool((raw > r).any()) and bool(((raw > 0) & (raw <= r)).any())


def test_oracle_zero_norm_frames_and_nan():
    x, u, c = _pair(T=3)
    sigma = 0.5
    x[0, 0] = sigma * c[0, 0]  # D_c = 0: par = 0
    parts = A.apg_parts(x, u, c, sigma, 4.0, 0.7)
    assert float(parts["p"][0]) == 0.0 and float(parts["par"][0, 0].abs().max()) == 0.0
    c[0, 1, 0, 0, 0] = math.nan
    parts = A.apg_parts(x, u, c, sigma, 4.0, 0.7, norm_threshold=1.0)
    assert torch.isnan(parts["D_g"][0, 1]).all() and not torch.isnan(parts["D_g"][0, 2]).any()


def test_oracle_momentum_matches_the_unrolled_sum():
    beta = -0.75
    x, u, c = _pair(T=3, seed=1)
    diffs, avg = [], None
    for k in range(3):
        sigma = 0.9 - 0.2 * k
        xk, uk, ck = x + 0.1 * k, u * (1 + 0.3 * k), c - 0.2 * k
        diffs.append((xk - sigma * ck) - (xk - sigma * uk))
        parts = A.apg_parts(xk, uk, ck, sigma, 4.0, 0.0, momentum=beta, avg=avg)
        avg = parts["avg"]
    want = diffs[2] + beta * diffs[1] + beta ** 2 * diffs[0]
    assert torch.allclose(avg, want, rtol=0, atol=1e-12)
    assert torch.allclose(parts["diff"], want, rtol=0, atol=1e-12)  # no threshold: diff is the average


def test_validation():
    from scail_b200.guidance import APG
    for name, kw in (("eta", dict(eta=True)), ("eta", dict(eta=math.nan)), ("eta", dict(eta=math.inf)), ("eta", dict(eta="1")),
                     ("eta", dict(eta=None)), ("norm_threshold", dict(eta=1.0, norm_threshold=-0.5)),
                     ("norm_threshold", dict(eta=1.0, norm_threshold=False)),
                     ("norm_threshold", dict(eta=1.0, norm_threshold=math.inf)), ("momentum", dict(eta=1.0, momentum=True)),
                     ("momentum", dict(eta=1.0, momentum=-math.inf)), ("momentum", dict(eta=1.0, momentum=math.nan))):
        with pytest.raises(ValueError, match=name):
            APG(**kw)
    with pytest.raises(TypeError):
        APG()  # eta has no default
    g = APG(0, 2, -0.5)
    assert (g.eta, g.norm_threshold, g.momentum) == (0.0, 2.0, -0.5)
    g = APG(np.float32(0.25))
    assert (g.eta, g.norm_threshold, g.momentum) == (0.25, 0.0, 0.0)
    assert [g.begin_step() for _ in range(3)] == [False] * 3 and g.step_index == 3
    g.reset()
    assert g.step_index == 0 and g.last_factors is None
    with pytest.raises(ValueError, match="sigma > 0"):
        g.update(torch.zeros(1, 1, 16, 2, 2), torch.zeros(2, 1, 16, 2, 2), 4.0, 0.0, 0.0)


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
    from scail_b200.guidance import APG
    g = APG(0.0, 1.0, -0.5)
    m = _tiny_model()
    x, cond, uc = _inputs()
    ad = m.mixins["adaln_layer"]
    ad.cp = types.SimpleNamespace(size=2, rank=0)
    for call in (lambda: sampler.sample(m, x, cond, uc, num_steps=1, guidance=g),
                 lambda: sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, guidance=g),
                 lambda: sampler.GraphedStep(m, x, cond, uc, guidance=g)):
        with pytest.raises(NotImplementedError, match="guidance.*context parallelism.*APG"):
            call()
    ad.cp = None
    with pytest.raises(NotImplementedError, match="guidance.*chunk_dim"):
        sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, guidance=g, chunk_dim=3)
    with pytest.raises(NotImplementedError, match="sample_long.*APG.*per window"):
        sampler.sample_long(m, x, dict(cond, smpl_tiled=None), uc, [[0]], num_steps=1, guidance=g)
    with pytest.raises(NotImplementedError, match="guided_velocity.*APG"):
        sampler.guided_velocity(m, x, 0.5, cond, uc, guidance=g)
    for bad in (0, "apg", 1.0, object()):
        with pytest.raises(TypeError, match="guidance.*APG"):
            sampler.sampler_step(m, x, 1.0, 0.9, cond, uc, guidance=bad)
    assert g.step_index == 0 and g.last_factors is None  # nothing ran


def test_sample_long_keeps_accepting_cfg_zero_star():
    from scail_b200 import sampler
    from scail_b200.guidance import CFGZeroStar
    x = torch.zeros(1, 3, 16, 2, 2)
    cond = dict(crossattn=torch.zeros(1, 2, 8), smpl_tiled=torch.zeros(1, 1, 3, 16, 1, 1))
    out = sampler.sample_long(None, x, cond, dict(cond), [[0, 1, 2]], num_steps=1, guidance=CFGZeroStar(1),
                              denoise=lambda *a: None)  # the one step is zero-initialised: no window runs
    assert out is x


def test_entry_points_take_it():
    from scail_b200 import cfg_cache, sampler, unipc
    for f in (sampler.sample, sampler.sampler_step, sampler.GraphedStep, cfg_cache.CFGCache.cond_update):
        assert inspect.signature(f).parameters["guidance"].default is None, f
    assert inspect.signature(unipc.UniPC.step).parameters["m"].default is None


def test_ops_need_cuda():
    from scail_b200 import ops
    x = torch.zeros(1, 2, 16, 2, 2)
    v = torch.zeros(2, 2, 16, 2, 2, dtype=torch.bfloat16)
    part = torch.zeros(ops.apg_partials_len(2))
    factors = torch.zeros(2, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.apg_reduce(x, v, 0.5, part)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.apg_finish(part, torch.zeros(2, 4, dtype=torch.float64), factors, 0.0, 2, x.numel())
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.apg_update_(x, v, factors, 4.0, 1.0, 0.5, 0.4)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.unipc_step_dpred_(x, x.clone(), x.clone(), torch.zeros(2, x.numel()), 0, [0.0] * 10, False)
    from scail_b200.guidance import APG
    with pytest.raises(RuntimeError, match="CUDA"):
        APG(1.0).update(x, v, 4.0, 0.5, 0.4)
