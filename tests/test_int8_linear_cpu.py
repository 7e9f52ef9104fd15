"""fp8_linear="int8" on the CPU: the mode is accepted by both constructors and as the plain attribute, every other value keeps
its old meaning, the entry points open no CPU path, and the torch restatement the GPU tests pin the kernels to has the
format's edge cases: round-half-even, saturation at +-127 and an all-zero row."""
import argparse

import pytest
import torch

import int8_linear_oracle as R

SMALL = dict(hidden_size=128, num_attention_heads=1, inner_hidden_size=256, num_layers=2, text_dim=32, time_embed_dim=128)


def model(mode):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    return DiffusionTransformer(fp8_linear=mode, **SMALL)


def test_constructors_and_attribute_take_int8():
    from scail_b200.dit import FP8_LINEAR_INT8, AdaLNMixin
    assert FP8_LINEAR_INT8 == "int8"
    ad = model("int8").mixins["adaln_layer"]
    assert ad.fp8_linear == "int8"
    targs = argparse.Namespace(layernorm_epsilon=1e-6, num_attention_heads=1, is_gated_mlp=False)
    kw = dict(qk_ln=True, hidden_size_head=64, share_adaln=True, use_i2v_clip=True)
    assert AdaLNMixin(64, 1, 64, 3, targs, fp8_linear="int8", **kw).fp8_linear == "int8"
    for mode in (False, True, "int8", None):  # a plain attribute, set between forwards
        ad.fp8_linear = mode
        assert ad.fp8_linear is mode


def test_only_the_exact_string_int8_is_new():
    """Falsy values stay bf16 and every other truthy value stays e4m3, including the strings that only read as e4m3 by their
    truth (the attribute has never been validated, and is not now)."""
    from scail_b200 import ops
    from scail_b200.dit import linear_format
    assert linear_format("int8") is ops.INT8
    for mode in (False, None, 0, ""):
        assert linear_format(mode) is None, mode
    for mode in (True, 1, "INT8", "int8 ", "e4m3", "fp8", "int4", 2.0):
        assert linear_format(mode) is ops.FP8, mode


def test_state_dict_identical_in_int8_mode():
    a, b = model("int8"), model(False)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(torch.equal(sa[k], sb[k]) for k in sa)


def test_int8_forward_still_needs_cuda():
    m = model("int8")
    x = torch.zeros(1, 1, 16, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x, timesteps=torch.zeros(1), context=torch.zeros(1, 4, 32), ref_concat=torch.zeros(1, 1, 16, 8, 8),
          concat_smpl_render=torch.zeros(1, 1, 16, 4, 4), image_clip_features=torch.zeros(1, 257, 1280))


def test_int8_entry_points_have_no_cpu_path():
    from scail_b200 import ops
    q = torch.zeros(4, 32, dtype=torch.int8)
    s = torch.ones(4)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.gemm_fp8(q, s, q, s)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.quant_rows_fp8(torch.zeros(4, 32, dtype=torch.bfloat16), q, s)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.ln_modulate(torch.zeros(1, 4, 32, dtype=torch.bfloat16), out_fp8=(q, s))


def test_gemm_refuses_mixed_operand_dtypes():
    from scail_b200 import ops
    i8 = torch.zeros(4, 32, dtype=torch.int8)
    e4 = torch.zeros(4, 32, dtype=ops.FP8)
    s = torch.ones(4)
    for a, w in ((i8, e4), (e4, i8)):
        with pytest.raises(TypeError, match="both"):
            ops.gemm_fp8(a, s, w, s)


# ---------------------------------------------------------------- the restatement's edge cases
def test_round_half_even():
    s = torch.ones(1)
    x = torch.tensor([[0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5, -126.5, 0.49999997, 1.5000001]])
    assert R.codes(x, s).tolist() == [[0, 2, 2, 0, -2, -2, 126, -126, 0, 2]]


def test_saturation_at_127():
    s = torch.ones(1)
    x = torch.tensor([[127.4, 127.5, 128.0, 1e30, -127.5, -1e30, float("inf"), float("-inf")]])
    assert R.codes(x, s).tolist() == [[127, 127, 127, 127, -127, -127, 127, -127]]
    # the row's amax maps to +-127, with s the fp32 quotient amax / 127
    q, sc = R.quant(torch.tensor([[3.0, -3.0, 1.0]]).to(torch.bfloat16))
    assert q.tolist() == [[127, -127, 42]] and torch.equal(sc, torch.tensor([3.0]) / torch.tensor([127.0]))


def test_all_zero_row():
    x = torch.zeros(3, 48, dtype=torch.bfloat16)
    x[1, 5] = -2.0
    q, s = R.quant(x)
    assert s.tolist()[0] == 1.0 and s.tolist()[2] == 1.0 and not q[0].any() and not q[2].any()
    assert q[1, 5] == -127 and q[1].count_nonzero() == 1


def test_restated_chain_on_the_cpu():
    """The chain in fp64 codes and fp32 epilogue against a direct computation, for every epilogue."""
    g = torch.Generator().manual_seed(0)
    M, N, K = 70, 24, 96
    aq = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8)
    wq = torch.randint(-127, 128, (N, K), generator=g, dtype=torch.int8)
    sa, sw = torch.rand(M, generator=g) / 100, torch.rand(N, generator=g) / 100
    bias = torch.randn(N, generator=g).to(torch.bfloat16)
    res = torch.randn(M, N, generator=g).to(torch.bfloat16)
    gate = torch.randn(3, N, generator=g).to(torch.bfloat16)
    acc = (aq.long() @ wq.long().T).float()
    f = acc * sa[:, None] * sw[None, :] + bias.float()
    assert torch.equal(R.accumulate(aq, wq), (aq.long() @ wq.long().T).double())
    assert torch.equal(R.gemm(aq, sa, wq, sw, bias, chunk=16), f)
    assert torch.equal(R.gemm(aq, sa, wq, sw, bias, "BIAS_RES", res=res, chunk=16), f + res.float())
    want = f * gate.float().repeat_interleave(30, 0)[:M] + res.float()
    assert torch.equal(R.gemm(aq, sa, wq, sw, bias, "BIAS_GATE_RES", gate, 30, res, chunk=16), want)
    assert torch.allclose(R.gemm(aq, sa, wq, sw, bias, "BIAS_GELU"), torch.nn.functional.gelu(f, approximate="tanh"))
