"""First-block residual cache on the GPU: the three kernels against torch restatements, the cached model against a
restatement built from its own hooks (tests/step_cache_oracle.py), and GraphedStep against eager sampler_step."""
import math

import pytest
import torch

from step_cache_oracle import RestatedCache, apply_ref, indicator_sums, update_ref

pytestmark = pytest.mark.gpu


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm())


# ---------------------------------------------------------------- 1. kernels
# (B, N, d, n_ref, n_seq): row counts that are not multiples of 128, b = 1 and 2, and one 14B-width case (512x512, 21 frames)
SHAPES = [(1, 200, 256, 40, 100), (2, 333, 136, 77, 211), (2, 1856, 256, 256, 1280), (1, 1, 8, 0, 1),
          (2, 27904, 5120, 1024, 21504)]


def operands(B, N, d, seed):
    h0 = rnd(B, N, d, seed=seed)
    h1 = (h0.float() + rnd(B, N, d, scale=0.3, seed=seed + 1).float()).to(torch.bfloat16)
    r_ref = ((h1.float() - h0.float()) * (1 + 0.05 * rnd(B, N, d, seed=seed + 2).float())).to(torch.bfloat16)
    return h0, h1, r_ref


def scratch(B, N, d, n_seq):
    from scail_b200 import ops
    return (torch.empty(B, N, d, device="cuda", dtype=torch.bfloat16), torch.empty(B, n_seq, d, device="cuda", dtype=torch.bfloat16),
            torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda", dtype=torch.float32),
            torch.empty(4, device="cuda", dtype=torch.float64))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_indicator_kernel_against_fp64(shape):
    from scail_b200 import ops
    B, N, d, n_ref, n_seq = shape
    h0, h1, r_ref = operands(B, N, d, seed=N)
    r_new, h1c, partials, out = scratch(B, N, d, n_seq)
    ops.step_cache_indicator(h0, h1, r_ref, r_new, h1c, n_ref, partials, out)
    r, num, den = indicator_sums(h0, h1, r_ref)
    assert torch.equal(r_new, r)
    assert torch.equal(h1c, h1[:, n_ref:n_ref + n_seq])
    got = out.tolist()
    assert abs(got[0] - num) <= 1e-6 * num and abs(got[1] - den) <= 1e-6 * den, (got, num, den)
    assert got[2] == got[0] / got[1] and got[3] == 0.0
    assert abs(got[2] - num / den) <= 2e-6 * (num / den)
    # repeat launches, also from another stream, give bit-identical sums
    first = out.clone()
    for st in (torch.cuda.current_stream(), torch.cuda.Stream()):
        with torch.cuda.stream(st):
            out.zero_()
            ops.step_cache_indicator(h0, h1, r_ref, r_new, h1c, n_ref, partials, out)
        torch.cuda.synchronize()
        assert torch.equal(out, first)


def test_indicator_zero_denominator_and_zero_numerator():
    from scail_b200 import ops
    B, N, d, n_ref, n_seq = 2, 333, 136, 77, 211
    h0, h1, _ = operands(B, N, d, seed=7)
    r_new, h1c, partials, out = scratch(B, N, d, n_seq)
    ops.step_cache_indicator(h0, h1, torch.zeros_like(h0), r_new, h1c, n_ref, partials, out)
    assert out[1].item() == 0.0 and out[0].item() > 0 and out[2].item() == math.inf
    r = r_new.clone()
    ops.step_cache_indicator(h0, h1, r, r_new, h1c, n_ref, partials, out)
    assert out[0].item() == 0.0 and out[1].item() > 0 and out[2].item() == 0.0
    ops.step_cache_indicator(h0, h0, torch.zeros_like(h0), r_new, h1c, n_ref, partials, out)
    assert out.tolist()[:3] == [0.0, 0.0, math.inf]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_update_and_apply_bit_exact(shape):
    from scail_b200 import ops
    B, N, d, n_ref, n_seq = shape
    h1c = rnd(B, n_seq, d, seed=3)
    h = rnd(B, N, d, scale=4.0, seed=4)
    h[0, n_ref, :4] = torch.tensor([1e6, 3e-5, -7e4, 0.0], device="cuda", dtype=torch.bfloat16)  # exponent gaps past 2^16 against h1c
    R = torch.empty(B, n_seq, d, device="cuda", dtype=torch.float32)
    ops.step_cache_update(h, h1c, R, n_ref)
    want_R = update_ref(h, h1c, n_ref)
    assert torch.equal(R, want_R)
    hb = rnd(B, N, d, seed=5)
    want = apply_ref(hb, R, n_ref)
    ops.step_cache_apply(hb, R, n_ref)
    assert torch.equal(hb, want)
    outside = torch.ones(N, dtype=torch.bool)
    outside[n_ref:n_ref + n_seq] = False
    assert torch.equal(hb[:, outside], rnd(B, N, d, seed=5)[:, outside])  # ref and pose rows untouched


def test_abi_refuses_bad_shapes_and_pointers():
    from scail_b200 import _lib, ops
    h = torch.zeros(2, 40, 16, device="cuda", dtype=torch.bfloat16)
    R = torch.zeros(2, 24, 16, device="cuda", dtype=torch.float32)
    lib, p = _lib.lib(), h.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    assert lib.scail_step_cache_apply(p, R.data_ptr(), 2, 40, 16, 8, 24, st) == 0
    assert lib.scail_step_cache_apply(None, R.data_ptr(), 2, 40, 16, 8, 24, st) != 0
    assert b"null" in lib.scail_last_error()
    assert lib.scail_step_cache_apply(p + 2, R.data_ptr(), 2, 40, 16, 8, 24, st) != 0
    assert b"aligned" in lib.scail_last_error()
    assert lib.scail_step_cache_update(p, p, R.data_ptr(), 2, 40, 12, 8, 24, st) != 0
    assert b"multiple of 8" in lib.scail_last_error()
    assert lib.scail_step_cache_update(p, p, R.data_ptr(), 2, 40, 16, 20, 24, st) != 0
    assert b"noise rows" in lib.scail_last_error()
    assert lib.scail_step_cache_apply(p, R.data_ptr(), 2, 1 << 28, 5120, 0, 1, st) != 0
    assert b"2^31" in lib.scail_last_error()
    small = torch.zeros(4, device="cuda", dtype=torch.float32)
    out = torch.zeros(4, device="cuda", dtype=torch.float64)
    assert lib.scail_step_cache_indicator(p, p, p, p, p, small.data_ptr(), 1, out.data_ptr(), 2, 40, 16, 8, 24, st) != 0
    assert b"partials" in lib.scail_last_error()
    with pytest.raises(AssertionError):
        ops.step_cache_apply(h, torch.zeros(2, 20, 16, device="cuda"), 30)  # noise rows past N


# ---------------------------------------------------------------- 2. the model (small config)
CFG = dict(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=3, text_dim=64, time_embed_dim=256)


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


PATTERN = [0.0, math.inf, math.inf, 0.0, math.inf]  # computed, skipped, skipped, computed, skipped


@pytest.mark.parametrize("cross_kv", [False, True])
def test_threshold_zero_is_bit_identical_to_no_cache(cross_kv):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(1)
    m.mixins["adaln_layer"].cache_cross_kv = cross_kv
    x0, cond, uc = sampler_inputs()
    c = FirstBlockCache(0.0)
    with torch.no_grad():
        plain = sampler.sample(m, x0.clone(), cond, uc, num_steps=5)
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=5, step_cache=c)
    assert torch.equal(cached, plain)
    assert [s for _, s in c.history] == [False] * 5
    assert c.history[0][0] == math.inf and all(0 < i < math.inf for i, _ in c.history[1:])


def test_forced_pattern_against_the_restatement():
    from scail_b200 import ops, sampler
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(2)
    x0, cond, uc = sampler_inputs(3)
    sig = sampler.make_flow_timesteps(50, 5.0)
    c, want = FirstBlockCache(0.0), RestatedCache(m)
    ctx = sampler.prepare_context(cond, uc)
    kw = dict(ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
              image_clip_features=cond["image_clip_features"], concat_images=None)
    with torch.no_grad():
        xg, xw = x0.clone(), x0.clone()
        for i, thr in enumerate(PATTERN):
            c.threshold = thr
            sampler.sampler_step(m, xg, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=c)
            ts = torch.full((2,), float(sig[i]) * 1000.0, device="cuda")
            v = want.forward(thr, torch.cat([xw, xw]), timesteps=ts, context=ctx, **kw)
            ops.cfg_euler_(xw, v.contiguous(), 4.0, float(sig[i + 1]) - float(sig[i]))
            torch.cuda.synchronize()
            assert torch.equal(xg, xw), f"step {i}"
    assert [s for _, s in c.history] == [False, True, True, False, True] == [s for _, s in want.history]
    for (a, _), (b, _) in zip(c.history, want.history):
        assert a == b or abs(a - b) <= 1e-6 * b, (a, b)


def test_identical_inputs_indicator_zero_and_skip_matches_compute():
    from scail_b200.step_cache import FirstBlockCache
    m = small_model(4)
    from scail_b200 import sampler
    x0, cond, uc = sampler_inputs(5)
    x2 = torch.cat([x0, x0]).to(torch.bfloat16)
    kw = dict(timesteps=torch.full((2,), 700.0, device="cuda"), context=sampler.prepare_context(cond, uc),
              ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
              image_clip_features=cond["image_clip_features"])
    c = FirstBlockCache(1e-3)
    with torch.no_grad():
        computed = m(x2, _step_cache=c, **kw).clone()
        bufs = c.buffers
        n_ref, n_seq = bufs.n_ref, bufs.h1c.shape[1]
        h_L = bufs.h1[:, n_ref:n_ref + n_seq].clone()
        h1 = bufs.h1c.clone()
        skipped = m(x2, _step_cache=c, **kw).clone()
        applied = bufs.h1[:, n_ref:n_ref + n_seq].clone()
        plain = m(x2, **kw)
    assert c.history[0] == (math.inf, False) and c.history[1] == (0.0, True)
    assert torch.equal(computed, plain)
    # The skipped step feeds bf16(f32(h1) + R), R = f32(h_L) - f32(h1), to the final layer instead of h_L.  Both are bf16
    # (8-bit significands), so h_L - h1 is exact in fp32 unless their magnitudes are more than 2^16 apart; only there can the
    # rounded R fail to return h_L.  Everything else is bit-identical, hence the tight bound on the velocity.
    differ = applied != h_L
    a, b = h_L[differ].float().abs(), h1[differ].float().abs()
    assert bool(((a > 2.0 ** 16 * b) | (b > 2.0 ** 16 * a)).all()), int(differ.sum())
    e = rel(skipped, computed)
    print(f"skipped vs computed on identical inputs: {int(differ.sum())} of {differ.numel()} noise-row values differ, "
          f"velocity rel-L2 {e:.2e}")
    assert e <= 1e-5


# ---------------------------------------------------------------- 3. graphs
@pytest.mark.parametrize("fast", [False, True], ids=["bf16", "fp8_window1"])
def test_graphed_step_is_bit_identical_to_eager(fast):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    kw = dict(fp8_linear=True, fp8_attention=True, attention_window=1) if fast else {}
    m = small_model(6, **kw)
    x0, cond, uc = sampler_inputs(7)
    sig = sampler.make_flow_timesteps(50, 5.0)
    ce, cg = FirstBlockCache(0.0), FirstBlockCache(0.0)
    pattern = PATTERN + [0.0, math.inf]
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, step_cache=cg)
        assert gs.kernels_in_graph > 20
        for i, thr in enumerate(pattern):
            if i == len(PATTERN):  # a new run with the same objects: the graphs are captured again for the new buffers
                ce.reset()
                cg.reset()
            ce.threshold = cg.threshold = thr
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=ce)
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(xe, xg), f"step {i}"
    assert ce.history == cg.history
    assert [s for _, s in cg.history] == [False, True]
