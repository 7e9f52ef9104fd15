"""Taylor forecast of the first-block residual cache (FirstBlockCache(order >= 1)): the host-side policy without a GPU --
coefficients, effective degree, slot rotation, max_skips, validation, the missing-sigma error and the unchanged refusals."""
import math
import types

import numpy as np
import pytest
import torch


def _geometry(c, B=2, N=40, d=16, n_ref=8, n_seq=24):
    return c.workspace(B, N, d, n_ref, n_seq, "cpu")


def _sigmas():
    from scail_b200.sampler import make_flow_timesteps
    return [float(s) for s in make_flow_timesteps(50, 5)]


def _numpy_coefficients(sig_pts, sigma):
    """Independent fp64 evaluation: the polynomial through (sig_pts, e_i) evaluated at sigma is the coefficient of point i."""
    out = []
    for i in range(len(sig_pts)):
        e = np.zeros(len(sig_pts))
        e[i] = 1.0
        if len(sig_pts) == 1:
            out.append(1.0)
            continue
        p = np.polyfit(np.asarray(sig_pts, dtype=np.float64), e, len(sig_pts) - 1)
        out.append(float(np.polyval(p, sigma)))
    return out


def _run(c, sigmas, skips):
    """Drive the cache's host side over a schedule (no kernels): -> the (slot, coefficients) staged for every step."""
    staged = []
    for sigma, want_skip in zip(sigmas, skips):
        c.set_sigma(sigma)
        c.begin()
        skip = c.decide(0.0 if want_skip else math.inf)
        staged.append(c.control(skip))
        c.stage(skip)
        if not skip:
            c.computed()
    return staged


@pytest.mark.parametrize("order", [1, 2])
def test_coefficients_against_numpy_fp64(order):
    from scail_b200.step_cache import forecast_coefficients
    sig = _sigmas()
    for start in (0, 5, 20, 40, 45):
        pts = sig[start:start + order + 1]
        for target in (sig[start + order + 1], sig[start + order + 2] if start + order + 2 < len(sig) else 0.0):
            slot_sigma = pts[:]  # computed step j went to slot j
            got = forecast_coefficients(target, slot_sigma, order + 1, order)
            want = _numpy_coefficients(pts, target)
            for g, w in zip(got, want):
                assert g == float(np.float32(g))  # exactly an fp32 value
                assert abs(g - w) <= 2.0 ** -23 * abs(w) + 1e-12, (start, target, got, want)
            # the coefficients of a Lagrange basis sum to one and reproduce sigma itself (degree >= 1)
            assert abs(sum(got) - 1.0) <= 1e-6
            assert abs(sum(g * s for g, s in zip(got, pts)) - target) <= 1e-6


def test_effective_degree_grows_with_computed_steps():
    from scail_b200.step_cache import forecast_coefficients
    sig = _sigmas()
    assert forecast_coefficients(sig[1], [None] * 3, 0, 2) == [0.0, 0.0, 0.0]  # nothing computed: nothing applied
    assert forecast_coefficients(sig[1], [sig[0], None, None], 1, 2) == [1.0, 0.0, 0.0]  # one point: the hold
    c2 = forecast_coefficients(sig[2], [sig[0], sig[1], None], 2, 2)  # two points: the line
    assert c2[2] == 0.0 and c2 == [float(np.float32(x)) for x in _numpy_coefficients(sig[:2], sig[2])] + [0.0]
    c3 = forecast_coefficients(sig[3], sig[:3], 3, 2)
    assert all(x != 0.0 for x in c3)
    # order 1 never uses more than the two most recent steps
    assert forecast_coefficients(sig[5], [sig[4], sig[3]], 4, 1) == forecast_coefficients(sig[5], [sig[4], sig[3]], 2, 1)


def test_duplicate_sigma_reduces_the_degree():
    from scail_b200.step_cache import forecast_coefficients
    # slots hold steps j = 0, 1, 2 (sigma 0.9, 0.8, 0.8); the two newest coincide -> the hold of the newest (slot 2)
    assert forecast_coefficients(0.7, [0.9, 0.8, 0.8], 3, 2) == [0.0, 0.0, 1.0]
    # newest two distinct, the third equal to the newest: degree 1 through slots 2 and 1
    got = forecast_coefficients(0.7, [0.8, 0.9, 0.8], 3, 2)
    assert got[0] == 0.0 and got[1:] == [float(np.float32(x)) for x in _numpy_coefficients([0.9, 0.8], 0.7)]
    assert forecast_coefficients(0.7, [0.8, 0.8], 2, 1) == [0.0, 1.0]


def test_slot_rotation_and_staged_control():
    from scail_b200.step_cache import FirstBlockCache
    sig = _sigmas()
    c = FirstBlockCache(math.inf, order=2)
    b = _geometry(c)
    assert b.R is None and b.R_slots.shape == (3, 2, 24, 16) and b.R_slots.dtype == torch.float32
    assert b.R_slots.abs().sum() == 0 and b.slot_sigma == [None] * 3
    assert b.ctl.tolist() == [-1, 0, 0, 0]
    pattern = [False, False, False, True, False, True, True, False, False]
    staged = _run(c, sig, pattern)
    writes = [slot for (slot, _), s in zip(staged, pattern) if not s]
    assert writes == [0, 1, 2, 0, 1, 2]  # the j-th computed step writes slot j mod 3
    assert all(slot == -1 for (slot, _), s in zip(staged, pattern) if s)
    computed = [i for i, s in enumerate(pattern) if not s]
    assert b.n_computed == 6
    assert b.slot_sigma == [sig[computed[3]], sig[computed[4]], sig[computed[5]]]
    # the skip at step 3 used steps 0, 1, 2 (slots 0, 1, 2); at step 5 steps 1, 2, 4 (slots 1, 2, 0)
    want3 = _numpy_coefficients([sig[0], sig[1], sig[2]], sig[3])
    assert staged[3][1] == [float(np.float32(x)) for x in want3]
    w5 = _numpy_coefficients([sig[4], sig[1], sig[2]], sig[5])  # slot order: 0 holds step 4, 1 step 1, 2 step 2
    assert staged[5][1] == [float(np.float32(x)) for x in w5]
    # the control block holds the last staged step: a computed step writing slot 2
    assert b.ctl.tolist()[0] == 2
    # skip after a computed step: its coefficients go into the control block as fp32 bits
    c.set_sigma(sig[9])
    c.begin()
    assert c.decide(0.0)
    c.stage(True)
    slot, coef = c.control(True)
    assert b.ctl_slot.tolist() == [-1] and b.ctl_coef.tolist() == coef


def test_order_1_pads_the_control_block_to_three_coefficients():
    from scail_b200.step_cache import FirstBlockCache
    sig = _sigmas()
    c = FirstBlockCache(math.inf, order=1)
    b = _geometry(c)
    assert b.R_slots.shape[0] == 2
    _run(c, sig, [False, False, True])
    assert b.ctl_coef.tolist()[2] == 0.0 and b.ctl_coef.tolist()[:2] == c.control(True)[1]


@pytest.mark.parametrize("order", [0, 1, 2])
def test_max_skips_patterns(order):
    from scail_b200.step_cache import FirstBlockCache
    sig = _sigmas()
    for max_skips, want in ((None, [False] + [True] * 7), (0, [False] * 8), (1, [False, True] * 4),
                            (2, [False, True, True] * 2 + [False, True]), (3, [False, True, True, True] * 2)):
        c = FirstBlockCache(math.inf, order=order, max_skips=max_skips)
        _geometry(c)
        for i in range(8):
            c.set_sigma(sig[i])
            c.begin()
            s = c.decide(0.5)
            c.stage(s)
            if not s:
                c.computed()
        assert [s for _, s in c.history] == want, max_skips
        assert all(h == (0.5, s) for h, s in zip(c.history, want))  # the history tuple is unchanged: (indicator, skipped)
    # a step that would compute anyway resets the run; the cap can change between steps
    c = FirstBlockCache(0.1, order=order, max_skips=2)
    _geometry(c)
    got = []
    for i, ind in enumerate([1.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0]):
        c.set_sigma(sig[i])
        c.begin()
        got.append(c.decide(ind))
        if not got[-1]:
            c.computed()
    assert got == [False, True, False, True, True, False, True]
    c.max_skips = None
    c.set_sigma(sig[8])
    c.begin()
    assert c.decide(0.0)


def test_reset_drops_slots_and_sigmas():
    from scail_b200.step_cache import FirstBlockCache
    sig = _sigmas()
    c = FirstBlockCache(math.inf, order=2, max_skips=1)
    b = _geometry(c)
    _run(c, sig, [False, False, True])
    assert b.n_computed == 2 and c._run == 1
    c.reset()
    assert c.buffers is None and c.history == [] and not c.has_state and c._run == 0
    b2 = _geometry(c)
    assert b2 is not b and b2.n_computed == 0 and b2.slot_sigma == [None] * 3 and b2.R_slots.abs().sum() == 0
    staged = _run(c, sig[10:], [False, True])
    assert staged == [(0, [0.0, 0.0, 0.0]), (-1, [1.0, 0.0, 0.0])]
    # another geometry also starts from empty slots
    _run(c, sig[12:], [False])
    b3 = _geometry(c, N=48)
    assert b3 is not b2 and b3.n_computed == 0 and not c.has_state


def test_argument_validation():
    from scail_b200.step_cache import FirstBlockCache
    for order in (0, 1, 2, np.int64(2)):
        assert FirstBlockCache(0.1, order=order).order == int(order)
    for bad in (True, False, 1.0, 2.0, "1", None, [1]):
        with pytest.raises(TypeError):
            FirstBlockCache(0.1, order=bad)
    for bad in (-1, 3, 10):
        with pytest.raises(ValueError):
            FirstBlockCache(0.1, order=bad)
    c = FirstBlockCache(0.1, order=1)
    with pytest.raises(AttributeError):
        c.order = 2  # the slots are sized by the order: fixed at construction
    for ok in (None, 0, 1, 50, np.int32(4)):
        assert FirstBlockCache(0.1, max_skips=ok).max_skips == (None if ok is None else int(ok))
    for bad in (True, 1.0, "2", math.inf):
        with pytest.raises(TypeError):
            FirstBlockCache(0.1, max_skips=bad)
        with pytest.raises(TypeError):
            c.max_skips = bad
    for bad in (-1, -5):
        with pytest.raises(ValueError):
            FirstBlockCache(0.1, max_skips=bad)
    with pytest.raises(TypeError):
        FirstBlockCache(True, order=1)  # the threshold's own validation is unchanged
    for bad in (math.nan, math.inf, -math.inf):
        with pytest.raises(ValueError):
            c.set_sigma(bad)
    with pytest.raises(TypeError):
        c.set_sigma(True)
    c.set_sigma(torch.tensor(0.5))  # the sampler's sigmas are one-element tensors
    c.begin()
    assert c._step_sigma == 0.5


def test_defaults_keep_the_order_0_buffers():
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(0.1)
    assert c.order == 0 and c.max_skips is None
    b = _geometry(c)
    assert b.R is not None and b.R.shape == (2, 24, 16) and b.R_slots is None and b.ctl is None
    c.begin()  # order 0 needs no sigma
    assert not c.decide(0.0)
    c.stage(False)  # nothing to stage at order 0
    c.computed()
    assert c.decide(0.0) and c.history == [(0.0, False), (0.0, True)]


def test_workspace_memory_of_the_slots():
    """order + 1 fp32 slots replace R: each order adds B * n_seq * d * 4 bytes (DESIGN §3.4)."""
    assert round(2 * 21 * 1024 * 5120 * 4 / 1e9, 2) == 0.88  # 512x512, b = 2
    assert round(2 * 21 * 1792 * 5120 * 4 / 1e9, 2) == 1.54  # 512x896
    from scail_b200.step_cache import FirstBlockCache
    base = _geometry(FirstBlockCache(0)).nbytes()
    for order in (1, 2):
        assert _geometry(FirstBlockCache(0, order=order)).nbytes() == base + order * 2 * 24 * 16 * 4


# ---------------------------------------------------------------- the forward: missing sigma, refusals (no device needed)
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


@pytest.mark.parametrize("order", [1, 2])
def test_missing_sigma_is_refused(order):
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(0.1, order=order)
    m = _tiny_model()
    x, kw = _inputs()
    with pytest.raises(ValueError, match=r"step_cache.*sigma"):
        m(x, _step_cache=c, **kw)
    assert c.history == [] and c.buffers is None  # refused before anything ran
    c.set_sigma(0.5)
    with pytest.raises(RuntimeError, match="CUDA"):  # with a sigma the forward goes on (and needs CUDA here)
        m(x, _step_cache=c, **kw)
    with pytest.raises(ValueError, match=r"step_cache.*sigma"):  # the sigma was consumed by that forward
        m(x, _step_cache=c, **kw)


@pytest.mark.parametrize("order", [1, 2])
def test_refusals_are_unchanged(order):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    c = FirstBlockCache(0.1, order=order, max_skips=2)
    m = _tiny_model()
    x, kw = _inputs()
    c.set_sigma(0.5)
    with pytest.raises(NotImplementedError, match="step_cache is not implemented with chunk_dim"):
        m(x, _step_cache=c, chunk_dim=3, **kw)
    c.set_sigma(0.5)
    with pytest.raises(NotImplementedError, match="step_cache is not implemented with _num_layers"):
        m(x, _step_cache=c, _num_layers=1, **kw)
    m.mixins["adaln_layer"].cp = types.SimpleNamespace(size=2, rank=0)
    c.set_sigma(0.5)
    with pytest.raises(NotImplementedError, match="step_cache is not implemented under context parallelism"):
        m(x, _step_cache=c, **kw)
    cond = dict(crossattn=torch.zeros(1, 4, 64), ref_concat=kw["ref_concat"], concat_smpl_render=kw["concat_smpl_render"],
                image_clip_features=kw["image_clip_features"])
    uc = dict(crossattn=torch.zeros(1, 4, 64))
    with pytest.raises(NotImplementedError, match="step_cache is not implemented under context parallelism"):
        sampler.sample(m, x[:1], cond, uc, num_steps=1, step_cache=c)
    with pytest.raises(NotImplementedError, match="step_cache is not implemented under context parallelism"):
        sampler.GraphedStep(m, x[:1], cond, uc, step_cache=c)
    m.mixins["adaln_layer"].cp = None
    plan = types.SimpleNamespace(branch=0)
    with pytest.raises(NotImplementedError, match="step_cache is not implemented with a HybridParallel plan"):
        sampler.sample(m, x[:1], cond, uc, num_steps=1, plan=plan, step_cache=c)
    with pytest.raises(NotImplementedError, match="step_cache is not implemented with a HybridParallel plan"):
        sampler.sampler_step(m, x[:1], 1.0, 0.9, cond, uc, plan=plan, step_cache=c)
    assert c.history == [] and c.buffers is None  # nothing ran
