"""UniPC flow solver on the host: the product's composed fp64 coefficients against the step-by-step restatement
(tests/unipc_oracle.py), convergence on Gaussian data whose ODE solution is known, the edge rules, and validation.  The
solver's launches are replaced by an fp64 CPU restatement of the kernel, so the policy runs end to end without a GPU."""
import math

import numpy as np
import pytest
import torch

import unipc_oracle as O
from scail_b200 import sampler, unipc
from scail_b200.unipc import UniPC, step_coefficients


def apply_coefficients(x, sigmas, order, velocity):
    """The product's per-step linear combination (step_coefficients), applied in fp64 in the kernel's dataflow: m_i into
    slot i mod order, y into x_last, z into x."""
    sig = unipc.check_schedule(sigmas)
    x = np.asarray(x, dtype=np.float64).copy()
    slots, x_last = [None] * order, None
    for i in range(len(sig) - 1):
        k = step_coefficients(sig, i, order)
        m = x - sig[i] * velocity(x, sig[i], i)
        if k.correct:
            y = k.x_last_c * x_last
            for s, c in enumerate(k.slot_c):
                if c != 0.0:
                    y = y + c * slots[s]
            y = y + k.m_c * m
        else:
            y = x
        z = k.y_c * y
        for s, c in enumerate(k.slot_p):
            if c != 0.0:
                z = z + c * slots[s]
        x = z + k.m_p * m
        slots[k.write], x_last = m, y
    return x


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def all_coefficients(k):
    return [k.x_last_c, *k.slot_c, k.m_c, k.y_c, *k.slot_p, k.m_p]


@pytest.mark.parametrize("order", [1, 2, 3])
@pytest.mark.parametrize("shift", [1.0, 3.0, 5.0])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 10, 20, 50])
def test_coefficients_match_the_oracle(n, shift, order):
    sig = sampler.make_flow_timesteps(n, shift)
    rng = np.random.default_rng(n * 100 + int(shift) * 10 + order)
    x0 = rng.standard_normal(4096)
    G = rng.standard_normal((n, 4096)) * np.exp(rng.normal(0.0, 1.0, (n, 1)))
    vel = lambda x, s, i: G[i]
    want = O.sample(x0, sig, order, vel)
    got = apply_coefficients(x0, sig, order, vel)
    assert rel(got, want) < 1e-12
    s = unipc.check_schedule(sig)
    for i in range(n):
        k = step_coefficients(s, i, order)
        assert all(math.isfinite(c) for c in all_coefficients(k)), (i, k)
        assert k.correct == (i >= 1) and k.write == i % order
        if not k.correct:
            assert k.x_last_c == k.m_c == 0.0 and k.slot_c == [0.0] * order


@pytest.mark.parametrize("order", [1, 2, 3])
def test_coefficients_on_a_schedule_that_starts_below_one(order):
    """sigma_0 < 1: lambda_0 is finite, so the first older point is used (no stop at sigma = 1)."""
    sig = [0.9, 0.7, 0.45, 0.3, 0.2, 0.1, 0.0]
    rng = np.random.default_rng(order)
    x0, G = rng.standard_normal(512), rng.standard_normal((6, 512))
    vel = lambda x, s, i: G[i]
    assert rel(apply_coefficients(x0, sig, order, vel), O.sample(x0, sig, order, vel)) < 1e-12


def test_edge_rules():
    for n, shift in ((1, 5.0), (7, 1.0), (50, 5.0)):
        s = unipc.check_schedule(sampler.make_flow_timesteps(n, shift))
        for order in (1, 2, 3):
            # the last step predicts at order 1 to sigma = 0: x_n = m_{n-1} exactly
            k = step_coefficients(s, n - 1, order)
            assert k.y_c == 0.0 and k.m_p == 1.0 and k.slot_p == [0.0] * order
            # step 0 starts at sigma = 1: x_1 = sigma_1 x + alpha_1 m_0, which is Euler
            k = step_coefficients(s, 0, order)
            if n > 1:
                assert k.y_c == s[1] and k.m_p == 1.0 - s[1] and k.slot_p == [0.0] * order
    # the order-1 predictor is Euler: z = x + (sigma_t - sigma_s) g, also from sigma_s < 1
    s = [0.8, 0.5, 0.0]
    k = step_coefficients(s, 0, 1)
    assert k.y_c + k.m_p == pytest.approx(1.0, abs=1e-15)
    assert -k.m_p * s[0] == pytest.approx(s[1] - s[0], abs=1e-15)
    # an older point at sigma = 1 lowers the order: step 1's predictor at order 3 uses no older output, step 2's one
    s = unipc.check_schedule(sampler.make_flow_timesteps(10, 5.0))
    assert step_coefficients(s, 1, 3).slot_p == [0.0, 0.0, 0.0]
    assert sum(c != 0.0 for c in step_coefficients(s, 2, 3).slot_p) == 1
    assert sum(c != 0.0 for c in step_coefficients(s, 3, 3).slot_p) == 2


# ---------------------------------------------------------------- convergence on Gaussian data
def gaussian_problem(seed=0, size=1000):
    rng = np.random.default_rng(seed)
    mu = rng.standard_normal(size)
    s = np.exp(rng.normal(0.0, 0.7, size))  # log s ~ N(0, 0.49)
    eps = rng.standard_normal(size)
    return O.gaussian_velocity(mu, s), eps, mu + s * eps


def errors(shift, n):
    v, eps, want = gaussian_problem()
    sig = sampler.make_flow_timesteps(n, shift)
    return rel(O.euler(eps, sig, v), want), [rel(apply_coefficients(eps, sig, p, v), want) for p in (1, 2, 3)]


@pytest.mark.parametrize("shift", [1.0, 3.0, 5.0])
def test_unipc_beats_euler_on_gaussian_data(shift):
    for n in (5, 8, 10, 20, 40, 80):
        e, u = errors(shift, n)
        assert all(x < e for x in u), (n, e, u)


def test_observed_order_at_shift_1():
    e40, u40 = errors(1.0, 40)
    e80, u80 = errors(1.0, 80)
    assert math.log2(e40 / e80) == pytest.approx(1.0, abs=0.1)  # Euler is first order
    for p in (1, 2, 3):
        assert math.log2(u40[p - 1] / u80[p - 1]) >= p + 0.4, (p, u40, u80)


@pytest.mark.parametrize("shift,n,want", [(1.0, 40, (4.08e-2, 4.21e-3, 7.97e-4, 6.13e-4)),
                                          (1.0, 80, (2.07e-2, 1.08e-3, 1.26e-4, 5.42e-5)),
                                          (5.0, 20, (7.54e-2, 4.47e-2, 1.99e-2, 1.89e-2)),
                                          (5.0, 40, (3.87e-2, 1.68e-2, 4.99e-3, 4.31e-3))])
def test_gaussian_errors_match_the_recorded_values(shift, n, want):
    e, u = errors(shift, n)
    np.testing.assert_allclose([e, *u], want, rtol=6e-3)  # the table gives 3 significant digits


def test_order_2_at_20_steps_beats_euler_at_40_at_shift_5():
    assert errors(5.0, 20)[1][1] < errors(5.0, 40)[0]


# ---------------------------------------------------------------- validation
def test_order_is_validated():
    for bad in (True, False, 2.0, "2", None):
        with pytest.raises(TypeError, match="order"):
            UniPC(bad)
    for bad in (0, 4, -1):
        with pytest.raises(ValueError, match="order"):
            UniPC(bad)
    assert [UniPC(p).order for p in (1, 2, 3)] == [1, 2, 3] and UniPC().order == 2
    assert UniPC(np.int64(3)).order == 3


@pytest.mark.parametrize("bad", [[1.0], [[1.0, 0.0]], [1.0, 0.5, 0.5, 0.0], [1.0, 0.6, 0.7, 0.0], [1.5, 0.5, 0.0],
                                 [1.0, 0.5, 0.1], [1.0, math.nan, 0.0], [math.inf, 0.5, 0.0], [1.0, 0.5, -0.1]])
def test_schedule_is_validated(bad):
    with pytest.raises(ValueError, match="schedule"):
        UniPC().begin(bad)


def test_schedule_accepts_the_sampler_schedule():
    sig = sampler.make_flow_timesteps(12, 5.0)
    u = UniPC(3)
    u.begin(sig)
    assert u.sigmas == [float(s) for s in sig]
    u.begin([0.9, 0.5, 0.0])
    assert u.sigmas == [0.9, 0.5, 0.0]


def kernel_on_cpu(calls):
    """A CPU restatement of ops.unipc_step_ for host tests, in fp64 on the stored fp32 values."""
    def run(x, x_last, v, slots, write, scale, sigma, coef, correct):
        calls.append((write, sigma, list(coef), bool(correct)))
        d = lambda t: t.double().reshape(-1)
        u, c = d(v[0]), d(v[1])
        m = d(x) - sigma * (u + scale * (c - u))
        a_x, a, a_m, b_y, b, b_m = coef[0], coef[1:4], coef[4], coef[5], coef[6:9], coef[9]
        M = [d(slots[s]) if s < slots.shape[0] else None for s in range(3)]
        y = a_x * d(x_last) + sum(a[s] * M[s] for s in range(3) if a[s] != 0.0) + a_m * m if correct else d(x)
        z = b_y * y + sum(b[s] * M[s] for s in range(3) if b[s] != 0.0) + b_m * m
        x.copy_(z.view(x.shape)), x_last.copy_(y.view(x.shape)), slots[write].copy_(m)
        return x
    return run


class FakeModel:
    """Returns a fixed CFG pair; counts its forwards."""

    def __init__(self, shape, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.v = torch.randn(2, *shape[1:], generator=g).to(torch.bfloat16)
        self.calls = 0

    def __call__(self, x2, **kw):
        self.calls += 1
        return self.v


COND = dict(crossattn=torch.zeros(1, 4, 8), ref_concat=None, concat_smpl_render=None, image_clip_features=None)
UC = dict(crossattn=torch.zeros(1, 4, 8))


def test_sampler_runs_the_policy(monkeypatch):
    calls = []
    monkeypatch.setattr(unipc.ops, "unipc_step_", kernel_on_cpu(calls))
    shape = (1, 3, 16, 4, 6)
    model = FakeModel(shape)
    x0 = torch.randn(shape, generator=torch.Generator().manual_seed(1))
    u = UniPC(3)
    n = 8
    got = sampler.sample(model, x0.clone(), COND, UC, num_steps=n, shift_scale=5.0, scale=3.0, solver=u)
    assert model.calls == n and len(calls) == n and u.step_index == n
    sig = u.sigmas
    assert [c[0] for c in calls] == [i % 3 for i in range(n)] and [c[1] for c in calls] == sig[:n]
    assert [c[3] for c in calls] == [False] + [True] * (n - 1)
    for i, c in enumerate(calls):  # each coefficient rounded once to fp32; absent slots get exactly 0
        k = step_coefficients(sig, i, 3)
        want = [k.x_last_c, *k.slot_c, k.m_c, k.y_c, *k.slot_p, k.m_p]
        assert c[2] == [float(np.float32(w)) for w in want]
    vf = model.v.double()
    g = (vf[0] + 3.0 * (vf[1] - vf[0])).numpy().reshape(-1)
    want = O.sample(x0.double().numpy().reshape(-1), sig, 3, lambda x, s, i: g)
    assert rel(got.double().numpy().reshape(-1), want) < 1e-5
    # a second run reuses the buffers and starts again at step 0
    slots = u.slots
    sampler.sample(model, x0.clone(), COND, UC, num_steps=4, solver=u)
    assert u.slots is slots and u.step_index == 4


def test_step_is_validated_before_anything_runs(monkeypatch):
    calls = []
    monkeypatch.setattr(unipc.ops, "unipc_step_", kernel_on_cpu(calls))
    shape = (1, 2, 16, 4, 4)
    model = FakeModel(shape)
    x = torch.zeros(shape)
    sig = sampler.make_flow_timesteps(3, 5.0)
    u = UniPC(2)
    step = lambda xx, i, j: sampler.sampler_step(model, xx, sig[i], sig[j], COND, UC, solver=u)
    with pytest.raises(ValueError, match="solver.*no sigma schedule"):
        step(x, 0, 1)
    u.begin(sig)
    with pytest.raises(ValueError, match="solver.*step 0"):
        step(x, 1, 2)
    with pytest.raises(ValueError, match="solver.*step 0"):
        sampler.sampler_step(model, x, float(sig[0]), 0.5, COND, UC, solver=u)
    assert model.calls == 0 and not calls
    step(x, 0, 1)
    with pytest.raises(ValueError, match="solver.*latent"):
        step(torch.zeros(1, 2, 16, 4, 8), 1, 2)
    with pytest.raises(ValueError, match="solver.*latent"):
        step(torch.zeros(shape, dtype=torch.float64), 1, 2)
    assert model.calls == 1 and len(calls) == 1
    step(x, 1, 2)
    step(x, 2, 3)
    with pytest.raises(ValueError, match="solver.*all 3 steps"):
        step(x, 2, 3)
    u.reset()
    step(x, 0, 1)  # reset() starts the bound schedule again
    assert model.calls == 4
    assert sampler.sample.__defaults__[-1] is None  # the default sampler stays Euler
