"""The fp8_attention switch on the CPU: both constructors take it (off by default), it leaves the state_dict exactly as it is,
and it does not open a CPU path."""
import argparse

import pytest
import torch

SMALL = dict(hidden_size=128, num_attention_heads=1, inner_hidden_size=256, num_layers=2, text_dim=32, time_embed_dim=128)


def model(**kw):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    return DiffusionTransformer(**SMALL, **kw)


def test_both_constructors_take_the_kwarg():
    from scail_b200.dit import AdaLNMixin
    assert model(fp8_attention=True).mixins["adaln_layer"].fp8_attention is True
    assert model().mixins["adaln_layer"].fp8_attention is False  # off by default
    both = model(fp8_attention=True, fp8_linear=True).mixins["adaln_layer"]
    assert both.fp8_attention is True and both.fp8_linear is True
    targs = argparse.Namespace(layernorm_epsilon=1e-6, num_attention_heads=1, is_gated_mlp=False)
    kw = dict(qk_ln=True, hidden_size_head=64, share_adaln=True, use_i2v_clip=True)
    assert AdaLNMixin(64, 1, 64, 3, targs, fp8_attention=True, **kw).fp8_attention is True
    assert AdaLNMixin(64, 1, 64, 3, targs, **kw).fp8_attention is False


def test_state_dict_identical_with_and_without_fp8_attention():
    a, b = model(fp8_attention=True), model()
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(sa[k].shape == sb[k].shape and torch.equal(sa[k], sb[k]) for k in sa)
    a.load_state_dict(sb, strict=True)


def test_fp8_attention_forward_still_needs_cuda():
    m = model(fp8_attention=True)
    x = torch.zeros(1, 1, 16, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x, timesteps=torch.zeros(1), context=torch.zeros(1, 4, 32), ref_concat=torch.zeros(1, 1, 16, 8, 8),
          concat_smpl_render=torch.zeros(1, 1, 16, 4, 4), image_clip_features=torch.zeros(1, 257, 1280))
