"""The fp8_linear switch on the CPU: it is accepted by both constructors, leaves the state_dict exactly as it is, and does
not open a CPU path."""
import argparse

import pytest
import torch

SMALL = dict(hidden_size=128, num_attention_heads=1, inner_hidden_size=256, num_layers=2, text_dim=32, time_embed_dim=128)


def model(fp8):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(0)
    return DiffusionTransformer(fp8_linear=fp8, **SMALL)


def test_state_dict_identical_with_and_without_fp8():
    a, b = model(True), model(False)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    assert all(sa[k].shape == sb[k].shape and torch.equal(sa[k], sb[k]) for k in sa)
    a.load_state_dict(sb, strict=True)


def test_both_constructors_take_the_kwarg():
    from scail_b200.dit import AdaLNMixin
    assert model(True).mixins["adaln_layer"].fp8_linear is True
    assert model(False).mixins["adaln_layer"].fp8_linear is False
    targs = argparse.Namespace(layernorm_epsilon=1e-6, num_attention_heads=1, is_gated_mlp=False)
    kw = dict(qk_ln=True, hidden_size_head=64, share_adaln=True, use_i2v_clip=True)
    assert AdaLNMixin(64, 1, 64, 3, targs, fp8_linear=True, **kw).fp8_linear is True
    assert AdaLNMixin(64, 1, 64, 3, targs, **kw).fp8_linear is False  # off by default


def test_fp8_forward_still_needs_cuda():
    m = model(True)
    x = torch.zeros(1, 1, 16, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x, timesteps=torch.zeros(1), context=torch.zeros(1, 4, 32), ref_concat=torch.zeros(1, 1, 16, 8, 8),
          concat_smpl_render=torch.zeros(1, 1, 16, 4, 4), image_clip_features=torch.zeros(1, 257, 1280))
