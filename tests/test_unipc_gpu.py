"""UniPC flow solver on the GPU: the fused step kernel bit-exact against separate torch fp32 ops in the stated order, the
sampler against a restatement that calls the model and applies those ops with the product's coefficients (and against
the fp64 oracle, tests/unipc_oracle.py, driven by the same velocities), GraphedStep against eager sampler_step, and the
composition with the first-block cache."""
import math

import numpy as np
import pytest
import torch

import unipc_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def bits(t):
    return t.view(torch.int32)


def f32(c):
    return float(np.float32(c))


def step_ref(x, x_last, v, slots, scale, sigma, coef, correct):
    """Separate torch fp32 ops in the kernel's order -> (z, y, m), flat.  Slot terms with a zero coefficient are skipped."""
    t = lambda c: torch.tensor(c, dtype=torch.float32, device=x.device)
    a_x, a, a_m, b_y, b, b_m = coef[0], coef[1:4], coef[4], coef[5], coef[6:9], coef[9]
    u, c = v[0].float().reshape(-1), v[1].float().reshape(-1)
    g = u + t(scale) * (c - u)
    m = x.reshape(-1) - t(sigma) * g
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
    z = z + t(b_m) * m
    return z, y, m


def sentinel(rows, n):
    """A fixed bit pattern with many NaN and inf encodings (compared as bits)."""
    ar = torch.arange(rows * n, device="cuda", dtype=torch.int64)
    pat = ((ar * 2654435761) & 0x7FFFFFFF).to(torch.int32) ^ 0x7F800001
    return pat.view(torch.float32).view(rows, n)


# 512x512, 480x832 and 512x896 latents of 81 frames (21 latent frames), and a small one with odd t, h and w
LATENTS = [(1, 21, 16, 64, 64), (1, 21, 16, 60, 104), (1, 21, 16, 64, 112), (1, 3, 16, 5, 7)]
ACTIVE = {1: [0], 2: [0, 2], 3: [0, 1, 2]}  # n_slots runs from the last active slot + 1 to 3


@pytest.mark.parametrize("shape", LATENTS, ids=lambda s: "x".join(map(str, s)))
def test_kernel_bit_exact(shape):
    from scail_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    n = math.prod(shape)
    x0, xl0 = rn(*shape), rn(*shape)
    v = (rn(2, *shape[1:]) * 2.0).to(torch.bfloat16)
    x0.view(-1)[:3] = torch.tensor([3e38, -1e-30, 0.0], device="cuda")  # an overflowing product and a tiny one
    live = rn(3, n) * 0.5
    for n_act, act in ACTIVE.items():
        for n_slots in sorted({max(act) + 1, 3}):
            for write in sorted({0, n_slots - 1}):
                for correct in (True, False):
                    a, b = [0.0] * 3, [0.0] * 3
                    for j, s in enumerate(act):
                        a[s] = f32(0.7 - 0.45 * j)
                        b[s] = 0.0 if (j == 0 and n_act > 1) else f32(-0.3 + 0.55 * j)  # the oldest only in the corrector
                    coef = [f32(0.93), *a, f32(-0.41), f32(0.88), *b, f32(0.17)]
                    before = sentinel(n_slots, n)
                    for s in act:
                        if s < n_slots:
                            before[s] = live[s]
                    scale, sigma = f32(4.0), f32(0.7312)
                    want = step_ref(x0, xl0, v, before, scale, sigma, coef, correct)
                    outs = []
                    for _ in range(2):  # repeat launches are bit-identical
                        x, xl, slots = x0.clone(), xl0.clone(), before.clone()
                        ops.unipc_step_(x, xl, v, slots, write, scale, sigma, coef, correct)
                        outs.append((x, xl, slots))
                        tag = (n_act, n_slots, write, correct)
                        assert torch.equal(bits(x.view(-1)), bits(want[0])), tag
                        assert torch.equal(bits(xl.view(-1)), bits(want[1])), tag
                        assert torch.equal(bits(slots[write]), bits(want[2])), tag
                        for s in range(n_slots):
                            if s != write:  # unwritten slots keep their bits, NaN sentinels included
                                assert torch.equal(bits(slots[s]), bits(before[s])), (tag, s)
                        assert not torch.isnan(x.view(-1)[3:]).any() and not torch.isnan(xl.view(-1)[3:]).any(), tag
                    assert all(torch.equal(bits(p), bits(q)) for p, q in zip(outs[0], outs[1]))
    torch.cuda.empty_cache()


def test_abi_refuses_bad_arguments():
    import ctypes
    from scail_b200 import _lib
    n = 64
    x, xl, sl = (torch.zeros(n + 8, device="cuda") for _ in range(3))
    slots = torch.zeros(3, n + 8, device="cuda")
    v = torch.zeros(2 * n + 8, device="cuda", dtype=torch.bfloat16)
    ok = (ctypes.c_float * 10)(*([0.5] * 10))
    two = (ctypes.c_float * 10)(*([0.5] * 3 + [0.0] + [0.5] * 4 + [0.0, 0.5]))
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    px, pl, pv, ps = x.data_ptr(), xl.data_ptr(), v.data_ptr(), slots.data_ptr()
    call = lambda *a: lib.scail_unipc_step(*a, st)
    args = lambda **kw: [kw.get(k, d) for k, d in (("x", px), ("xl", pl), ("v", pv), ("s", ps), ("stride", n + 8),
                                                    ("n_slots", 3), ("write", 1), ("n", n), ("scale", 4.0),
                                                    ("sigma", 0.5), ("correct", 1), ("coef", ctypes.addressof(ok)))]
    assert call(*args()) == 0
    assert call(*args(n_slots=2, coef=ctypes.addressof(two))) == 0
    torch.cuda.synchronize()
    for kw, msg in ((dict(x=None), b"null"), (dict(s=None), b"null"), (dict(coef=None), b"null"),
                    (dict(x=px + 4), b"16-byte aligned"), (dict(v=pv + 8), b"16-byte aligned"),
                    (dict(s=ps + 4), b"16-byte aligned"), (dict(n=6), b"multiple of 4"), (dict(n=0), b"multiple of 4"),
                    (dict(n_slots=0), b"n_slots"), (dict(n_slots=4), b"n_slots"), (dict(write=3), b"write_slot"),
                    (dict(write=-1), b"write_slot"), (dict(n_slots=2, write=2, coef=ctypes.addressof(two)), b"write_slot"),
                    (dict(stride=n - 4), b"slot_stride"), (dict(stride=n + 2), b"slot_stride"),
                    (dict(n_slots=2), b"coefficients of slot 2")):
        assert call(*args(**kw)) != 0, msg
        assert msg in lib.scail_last_error(), (msg, lib.scail_last_error())


# ---------------------------------------------------------------- the sampler on a small 2-block model
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


def restated_sample(m, x0, cond, uc, num_steps, shift, scale, order):
    """The model forward as sampler_step calls it, then step_ref with the product's coefficients -> (x, guided velocities
    in fp64, flat)."""
    from scail_b200 import sampler, unipc
    sig = unipc.check_schedule(sampler.make_flow_timesteps(num_steps, shift))
    ctx = sampler.prepare_context(cond, uc)
    kw = dict(y=None, ref_concat=cond["ref_concat"], concat_smpl_render=cond["concat_smpl_render"],
              image_clip_features=cond["image_clip_features"], concat_images=None)
    x, x_last = x0.clone(), torch.zeros_like(x0)
    slots = torch.zeros(order, x0.numel(), device="cuda")
    G = []
    for i in range(num_steps):
        ts = torch.full((2,), sig[i] * 1000.0, device="cuda", dtype=torch.float32)
        v = m(torch.cat([x, x], 0), timesteps=ts, context=ctx, **kw).contiguous()
        u, c = v[0].double().reshape(-1), v[1].double().reshape(-1)
        G.append((u + scale * (c - u)).cpu().numpy())
        k = unipc.step_coefficients(sig, i, order)
        pad = [0.0] * (3 - order)
        coef = [f32(cc) for cc in [k.x_last_c, *k.slot_c, *pad, k.m_c, k.y_c, *k.slot_p, *pad, k.m_p]]
        z, y, mm = step_ref(x, x_last, v, slots, scale, sig[i], coef, k.correct)
        x, x_last = z.view(x0.shape), y.view(x0.shape)
        slots[k.write] = mm
    return x, G, sig


@pytest.mark.parametrize("order", [1, 2, 3])
def test_sample_against_the_restatement_and_the_oracle(order):
    from scail_b200 import sampler
    from scail_b200.unipc import UniPC
    m = small_model(order)
    x0, cond, uc = sampler_inputs(order)
    n = 10
    with torch.no_grad():
        got = sampler.sample(m, x0.clone(), cond, uc, num_steps=n, shift_scale=5.0, scale=4.0, solver=UniPC(order))
        want, G, sig = restated_sample(m, x0, cond, uc, n, 5.0, 4.0, order)
        euler = sampler.sample(m, x0.clone(), cond, uc, num_steps=n, shift_scale=5.0, scale=4.0)
    assert torch.equal(got, want)
    oracle = O.sample(x0.double().cpu().numpy().reshape(-1), sig, order, lambda x, s, i: G[i])
    err = float(np.linalg.norm(got.double().cpu().numpy().reshape(-1) - oracle) / np.linalg.norm(oracle))
    print(f"order {order}: final latent rel-L2 vs the fp64 oracle with the same velocities = {err:.2e}")
    assert err < 1e-5
    assert not torch.equal(got, euler)


@pytest.mark.parametrize("fast", [False, True], ids=["bf16", "fp8_window1_cache"])
def test_graphed_step_is_bit_identical_to_eager(fast):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    kw = dict(fp8_linear=True, fp8_attention=True, attention_window=1) if fast else {}
    m = small_model(6, **kw)
    x0, cond, uc = sampler_inputs(7)
    n = 8
    sig = sampler.make_flow_timesteps(n, 5.0)
    se, sg = UniPC(2), UniPC(2)
    se.begin(sig)
    sg.begin(sig)
    ce = cg = None
    pattern = [0.0, 0.0, 0.0, math.inf, math.inf, 0.0, math.inf, 0.0]  # forced skips of the cache
    if fast:
        ce, cg = FirstBlockCache(0.0, order=2), FirstBlockCache(0.0, order=2)
    with torch.no_grad():
        xe, xg = x0.clone(), x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0, step_cache=cg, solver=sg)
        with pytest.raises(ValueError, match="solver"):  # refused before the graph runs: x is untouched
            gs(sig[0], sig[2])
        assert torch.equal(xg, x0)
        for i in range(n):
            if fast:
                ce.threshold = cg.threshold = pattern[i]
            sampler.sampler_step(m, xe, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=ce, solver=se)
            gs(sig[i], sig[i + 1])
            torch.cuda.synchronize()
            assert torch.equal(xe, xg), f"step {i}"
    if fast:
        assert ce.history == cg.history and any(s for _, s in cg.history)


def test_first_block_cache_at_zero_is_bit_identical_to_the_solver_alone():
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    from scail_b200.unipc import UniPC
    m = small_model(8)
    x0, cond, uc = sampler_inputs(8)
    c = FirstBlockCache(0.0)
    with torch.no_grad():
        alone = sampler.sample(m, x0.clone(), cond, uc, num_steps=6, solver=UniPC(3))
        cached = sampler.sample(m, x0.clone(), cond, uc, num_steps=6, step_cache=c, solver=UniPC(3))
    assert torch.equal(cached, alone)
    assert [s for _, s in c.history] == [False] * 6
