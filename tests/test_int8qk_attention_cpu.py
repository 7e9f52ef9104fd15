"""fp8_attention="int8_qk" on the CPU: the mode's validation at construction and at forward time, the context-parallel
refusal, that the state_dict does not change, and that neither the forward nor any of the new ops opens a CPU path."""
import argparse

import pytest
import torch

SMALL = dict(hidden_size=128, num_attention_heads=1, inner_hidden_size=256, num_layers=2, text_dim=32, time_embed_dim=128)


def model(**kw):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    return DiffusionTransformer(**SMALL, **kw)


def inputs():
    return torch.zeros(1, 1, 16, 8, 8), dict(timesteps=torch.zeros(1), context=torch.zeros(1, 4, 32),
                                             ref_concat=torch.zeros(1, 1, 16, 8, 8),
                                             concat_smpl_render=torch.zeros(1, 1, 16, 4, 4),
                                             image_clip_features=torch.zeros(1, 257, 1280))


def test_both_constructors_take_the_mode():
    from scail_b200.dit import AdaLNMixin
    assert model(fp8_attention="int8_qk").mixins["adaln_layer"].fp8_attention == "int8_qk"
    both = model(fp8_attention="int8_qk", fp8_linear=True).mixins["adaln_layer"]
    assert both.fp8_attention == "int8_qk" and both.fp8_linear is True
    targs = argparse.Namespace(layernorm_epsilon=1e-6, num_attention_heads=1, is_gated_mlp=False)
    kw = dict(qk_ln=True, hidden_size_head=64, share_adaln=True, use_i2v_clip=True)
    assert AdaLNMixin(64, 1, 64, 3, targs, fp8_attention="int8_qk", **kw).fp8_attention == "int8_qk"
    # False and True keep their meaning and their identity
    assert model(fp8_attention=True).mixins["adaln_layer"].fp8_attention is True
    assert model().mixins["adaln_layer"].fp8_attention is False


@pytest.mark.parametrize("bad", ["INT8_QK", "int8", "fp8", "", "true", "int8_qk "])
def test_any_other_string_is_refused_naming_the_option(bad):
    with pytest.raises(ValueError, match="fp8_attention"):
        model(fp8_attention=bad)
    from scail_b200.dit import check_fp8_attention
    with pytest.raises(ValueError, match="fp8_attention"):
        check_fp8_attention(bad)


def test_attribute_set_to_a_bad_string_is_refused_before_any_launch():
    """forward() checks the mode (and the context-parallel refusals) on the mixin before its first launch; on the CPU the
    forward stops earlier, at its CUDA check, so the check itself is called here."""
    ad = model().mixins["adaln_layer"]
    ad.fp8_attention = "int4"
    with pytest.raises(ValueError, match="fp8_attention"):
        ad._refuse_fp8_attention_cp()
    ad.fp8_attention = "int8_qk"
    ad._refuse_fp8_attention_cp()


def test_state_dict_identical_with_and_without_the_mode():
    a, b = model(fp8_attention="int8_qk"), model()
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(sa[k].shape == sb[k].shape and torch.equal(sa[k], sb[k]) for k in sa)
    a.load_state_dict(sb, strict=True)


def test_context_parallel_of_size_two_is_refused():
    class StubCP:
        size, rank = 2, 0

    ad = model(fp8_attention="int8_qk").mixins["adaln_layer"]
    ad.cp = StubCP()
    with pytest.raises(NotImplementedError, match="fp8_attention"):
        ad._refuse_fp8_attention_cp()
    ad.cp.size = 1  # a group of one is no context parallelism
    ad._refuse_fp8_attention_cp()


def test_forward_still_needs_cuda():
    m = model(fp8_attention="int8_qk")
    x, kw = inputs()
    with pytest.raises(RuntimeError, match="CUDA"), torch.no_grad():
        m(x, **kw)


def test_ops_have_no_cpu_path():
    from scail_b200 import ops
    B, H, L = 1, 1, 130
    d = 128 * H
    qkv = torch.zeros(B * L, 3 * d, dtype=torch.bfloat16)
    w = torch.ones(d, dtype=torch.bfloat16)
    q8, k8 = torch.zeros(B * L, d, dtype=torch.int8), torch.zeros(B * L, d, dtype=torch.int8)
    sc = torch.ones(B, H, 256)
    vt, vs = torch.zeros(B, H, 128, 256, dtype=torch.uint8).view(torch.float8_e4m3fn), torch.ones(B, H, 128)
    out = torch.empty(B * L, d, dtype=torch.bfloat16)
    calls = [
        lambda: ops.rmsnorm_rope_int8q(qkv, L, d, [(0, w), (d, w)], q8, sc),
        lambda: ops.quant_k_int8(qkv[:, d:2 * d], B, H, L),
        lambda: ops.attention_int8qk(q8, sc, k8, sc, vt, vs, out, B, H, L),
        lambda: ops.tile_pool(q8, B, H, L, x_scale=sc),
    ]
    for call in calls:
        with pytest.raises(RuntimeError, match="CUDA"):
            call()


def test_partial_workspace_length():
    from scail_b200 import ops
    # one fp64 sum per (batch, 256-key chunk, channel)
    assert ops.quant_k_int8_partial_len(2, 40, 27904) == 2 * 109 * 5120
    assert ops.quant_k_int8_partial_len(1, 1, 256) == 128
    assert ops.quant_k_int8_partial_len(1, 1, 257) == 256
