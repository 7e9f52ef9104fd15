"""Hopper-native (sm_90a) SCAIL DiT: drop-in replacements for the reference's SAT mixins plus a standalone
`DiffusionTransformer` with the reference's constructor kwargs, forward signature and state_dict names.

Reference surface mirrored here (paths relative to /root/reference):
  * mixins  ImagePatchEmbeddingMixin / Rotary3DPositionEmbeddingMixin / AdaLNMixin / FinalLayerMixin /
            UlyessAttentionMixin  — dit_video_crossattn_sc_xc.py:76-130, 351-757, 787-835, 844-1203;
            same hook names and signatures as collected by BaseModel.collect_hooks_
            (sat/model/base_model.py:140-176), so the YAML `target:` strings of
            configs/video_model/Wan2.1-i2v-14Bsc-pose-xc-latent.yaml:55-75 can point at this module and
            the reference's own DiffusionTransformer / BaseTransformer call into it unchanged.
  * DiffusionTransformer — dit_video_crossattn_sc_xc.py:1209-1587, usable without SAT (the GPU box has no
            /root/reference): it owns `mixins` and `transformer.layers[...]` with identical parameter names
            (SURVEY.md §8b) and runs the same hook sequence as BaseTransformer.forward
            (sat/model/transformer.py:572-746).

Every per-step op is a kernel of libscail_b200.so (scail_b200.ops); PyTorch only allocates buffers and
sequences launches.  There is no CPU path: calling forward without CUDA raises.
"""
import argparse
import math
import weakref
from functools import reduce
from operator import mul

import torch
from torch import nn

from . import ops, rope

try:  # when SAT is importable (reference present) be a real BaseMixin so add_mixin / collect_hooks_ accept us
    from sat.model.mixins import BaseMixin as _SatBaseMixin  # type: ignore
    from sat.model.base_model import non_conflict  # type: ignore
except Exception:  # standalone (GPU box)
    _SatBaseMixin = None

    def non_conflict(func):
        func.non_conflict = True
        return func


class BaseMixin(_SatBaseMixin if _SatBaseMixin is not None else nn.Module):
    """sat/model/mixins.py BaseMixin when available, else a minimal stand-in (an nn.Module whose
    `transformer` back-pointer is set without registering it as a submodule)."""

    def __init__(self):
        super().__init__()

    def reinit(self, parent_model=None):
        pass


def _set_transformer(mixin, transformer):
    object.__setattr__(mixin, "transformer", transformer)


# ------------------------------------------------------------------------------------------------
# parameter containers with the reference's names / layouts ([out, in] row-major)
# ------------------------------------------------------------------------------------------------


class _Linear(nn.Module):
    """Weight holder for ColumnParallelLinear / RowParallelLinear / nn.Linear (sat/mpu/layers.py:171-485)."""

    def __init__(self, in_features, out_features, bias=True, std=0.02):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_features, in_features) * std)
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None

    def __getstate__(self):  # the e4m3 copy (AdaLNMixin.fp8_weight) is derived data holding a weakref: not pickled
        state = self.__dict__.copy()
        state.pop("_fp8_cache", None)
        return state


class _Norm(nn.Module):
    def __init__(self, dim, bias=False):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))
        if bias:
            self.bias = nn.Parameter(torch.zeros(dim))


class _SelfAttention(nn.Module):  # sat/model/transformer.py:34-118
    def __init__(self, hidden):
        super().__init__()
        self.query_key_value = _Linear(hidden, 3 * hidden)
        self.dense = _Linear(hidden, hidden)


class _CrossAttention(nn.Module):  # sat/model/transformer.py:120-198
    def __init__(self, hidden):
        super().__init__()
        self.query = _Linear(hidden, hidden)
        self.key_value = _Linear(hidden, 2 * hidden)
        self.dense = _Linear(hidden, hidden)


class _MLP(nn.Module):  # sat/model/transformer.py:201-311 (is_gated_mlp=False, F1)
    def __init__(self, hidden, inner):
        super().__init__()
        self.dense_h_to_4h = _Linear(hidden, inner)
        self.dense_4h_to_h = _Linear(inner, hidden)


class _Layer(nn.Module):  # sat/model/transformer.py BaseTransformerLayer (is_decoder=True, no-affine pre-LNs)
    def __init__(self, hidden, inner):
        super().__init__()
        self.attention = _SelfAttention(hidden)
        self.cross_attention = _CrossAttention(hidden)
        self.post_cross_attention_layernorm = _Norm(hidden, bias=True)
        self.mlp = _MLP(hidden, inner)


class _Transformer(nn.Module):
    def __init__(self, num_layers, hidden, inner, num_heads, layernorm_epsilon):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(hidden, inner) for _ in range(num_layers)])
        self.hidden_size = hidden
        self.num_attention_heads = num_heads
        self.layernorm_epsilon = layernorm_epsilon
        self.layernorm_order = "pre"
        self.is_decoder = True
        self.hooks = {}


# ------------------------------------------------------------------------------------------------
# workspace: caller-owned PyTorch buffers reused across layers and steps (stable pointers => TMA
# descriptors are encoded once)
# ------------------------------------------------------------------------------------------------


class _Workspace:
    def __init__(self):
        self.bufs = {}

    def get(self, name, shape, device, dtype=torch.bfloat16):
        # one buffer set per CUDA stream: the context-parallel path runs the two CFG branches on two streams
        name = (name, torch.cuda.current_stream(device).cuda_stream)
        key = (name, tuple(shape), str(device), dtype)
        b = self.bufs.get(key)
        if b is None:
            for k in [k for k in self.bufs if k[0] == name]:
                del self.bufs[k]
            b = torch.empty(shape, device=device, dtype=dtype)
            self.bufs[key] = b
        return b


_WS = _Workspace()


class Conditioning:
    """Step-invariant conditioning of one sample (SURVEY §8f rank 1): text / CLIP embeddings and every layer's
    cross-attention K,V, computed ONCE by `DiffusionTransformer.set_conditioning` with the same kernels the per-step path
    uses (bit-identical).  It holds references to the caller's `context` / `image_clip_features` tensors and is used only
    while forward() is called with those very tensor OBJECTS at the same `_version` — never matched by address, so a new
    prompt living at a recycled address cannot hit a stale entry (ADVICE r1)."""

    def __init__(self, context, clip_feats, batch):
        self.context, self.clip_feats, self.batch = context, clip_feats, batch
        self.versions = (context._version, clip_feats._version)
        self.text = self.clip = None
        self.xkv = []  # per layer: (tkv [B*Lt, 2d], ckv [B*Lc, 2d])

    def matches(self, context, clip_feats, batch):
        return (context is self.context and clip_feats is self.clip_feats and batch == self.batch
                and (context._version, clip_feats._version) == self.versions)


def _need_cuda(t):
    if not t.is_cuda:
        raise RuntimeError("scail_b200 has no CPU path: tensors must live on a CUDA (sm_90a) device")


# ------------------------------------------------------------------------------------------------
# mixins
# ------------------------------------------------------------------------------------------------


class UlyessAttentionMixin(BaseMixin):
    """Placeholder for the reference's Ulysses wrapper (dit_video_crossattn_sc_xc.py:351-379).  Sequence
    parallelism here is token-sharded context parallelism with one K/V all-gather per block
    (scail_b200.parallel), handled inside AdaLNMixin.layer_forward; no attention_fn hook is installed."""

    def __init__(self):
        super().__init__()


class Rotary3DPositionEmbeddingMixin(BaseMixin):
    """dit_video_crossattn_sc_xc.py:382-757.  Tables are produced by scail_b200.rope (same op order as the
    reference ctor) and consumed by the fused RMSNorm+RoPE kernel inside AdaLNMixin.attention_forward."""

    def __init__(self, height, width, compressed_num_frames, hidden_size, hidden_size_head, theta=10000,
                 rot_v=False, pnp=False, height_interpolation=1.0, width_interpolation=1.0, time_interpolation=1.0,
                 learnable_pos_embed=False, patch_size=None, interleaved_rope=False):
        super().__init__()
        if not interleaved_rope or rot_v or pnp:
            raise NotImplementedError("scail_b200 implements the SCAIL config: interleaved_rope=True, rot_v=False, pnp=False")
        if hidden_size_head != 128:
            raise NotImplementedError("attention kernel is specialised for head_dim 128")
        self.height, self.width, self.compressed_num_frames = height, width, compressed_num_frames
        self.hidden_size_head = hidden_size_head
        self.theta = float(theta)

    def tables(self, device, **kw):
        T, H, W = kw["rope_T"], kw["rope_H"], kw["rope_W"]
        if T > self.compressed_num_frames or H + kw.get("rope_H_shift", 0) > self.height or \
                W + kw.get("rope_W_shift", 0) > self.width:
            raise ValueError("latent geometry exceeds the RoPE grid of the reference ctor (:424-426)")
        return rope.build_tables(device, self.hidden_size_head, T, H, W, kw.get("rope_H_shift", 0),
                                 kw.get("rope_W_shift", 0), kw.get("global_rope_H", 0), kw.get("global_rope_W", 120),
                                 self.theta)

    def position_embedding_forward(self, position_ids, **kwargs):  # :650-651
        return None

    def reinit(self, parent_model=None):
        if hasattr(self.transformer, "position_embeddings"):
            del self.transformer.position_embeddings


class ImagePatchEmbeddingMixin(BaseMixin):
    """dit_video_crossattn_sc_xc.py:76-135: two Conv3d(k=s=(1,2,2)) == patch gather + GEMM (K = 20*4 = 80)."""

    def __init__(self, in_channels, hidden_size, patch_size, bias=True, use_conv=True):
        super().__init__()
        if not use_conv or tuple(patch_size) != (1, 2, 2) or in_channels != 20:
            raise NotImplementedError("scail_b200 implements in_channels=20, patch_size=(1,2,2), use_conv=True")
        self.patch_size = patch_size
        self.use_conv = use_conv
        self.proj = nn.Conv3d(in_channels, hidden_size, kernel_size=tuple(patch_size), stride=tuple(patch_size), bias=bias)
        self.proj_pose = nn.Conv3d(in_channels, hidden_size, kernel_size=tuple(patch_size), stride=tuple(patch_size), bias=bias)

    def reinit(self, parent_model=None):  # dit_video_crossattn_sc_xc.py:132-136
        w = self.proj.weight.data
        nn.init.xavier_uniform_(w.view([w.shape[0], -1]))
        nn.init.constant_(self.proj.bias, 0)
        if hasattr(self.transformer, "word_embeddings"):
            del self.transformer.word_embeddings

    def word_embedding_forward(self, input_ids, **kwargs):
        images, ref, pose = kwargs["images"], kwargs["ref_concat"], kwargs["concat_smpl_render"]
        _need_cuda(images)
        bf = torch.bfloat16
        images, ref, pose = images.to(bf).contiguous(), ref.to(bf).contiguous(), pose.to(bf).contiguous()
        B = images.shape[0]
        a_main, a_pose = ops.patchify(images, ref, pose)
        n_main, n_pose = a_main.shape[1], a_pose.shape[1]
        d = self.proj.weight.shape[0]
        hidden = kwargs.get("_hidden_out")
        if hidden is None:
            hidden = torch.empty(B, n_main + n_pose, d, device=images.device, dtype=bf)
        w_main, w_pose = self.proj.weight.view(d, -1), self.proj_pose.weight.view(d, -1)
        for b in range(B):  # token order ref || noise || pose per batch element (:118-124)
            ops.gemm(a_main[b], w_main, self.proj.bias, out=hidden[b, :n_main])
            ops.gemm(a_pose[b], w_pose, self.proj_pose.bias, out=hidden[b, n_main:])
        return hidden


class FinalLayerMixin(BaseMixin):
    """dit_video_crossattn_sc_xc.py:787-841 (share_adaln=True): LN + modulate + Linear(d -> 64) on the noise
    tokens only, then unpatchify (:764-784)."""

    def __init__(self, hidden_size, time_embed_dim, patch_size, out_channels, elementwise_affine, layernorm_epsilon,
                 share_adaln):
        super().__init__()
        if not share_adaln or elementwise_affine or tuple(patch_size) != (1, 2, 2) or out_channels != 16:
            raise NotImplementedError("scail_b200 implements share_adaln=True, elementwise_affine=False, patch (1,2,2), 16 ch")
        self.hidden_size, self.patch_size, self.out_channels = hidden_size, patch_size, out_channels
        self.layernorm_epsilon = layernorm_epsilon
        self.share_adaln = share_adaln
        self.linear = nn.Linear(hidden_size, reduce(mul, patch_size) * out_channels, bias=True)
        self.adaLN_modulation = nn.Parameter(torch.randn(1, 2, hidden_size) / hidden_size ** 0.5)

    def final_forward(self, logits, **kwargs):
        x, emb = logits, kwargs["final_layer_emb"]
        _need_cuda(x)
        B, N, d = x.shape
        n_ref, n_seq = kwargs["ref_length"], kwargs["seq_length"]
        # shift, scale = (emb + adaLN_modulation[0, {0, 1}])  (:823): two launches of the library kernel, no eager torch op
        emb = emb.contiguous()
        shift = ops.adaln_modulation(emb, self.adaLN_modulation[0, 0])
        scale = ops.adaln_modulation(emb, self.adaLN_modulation[0, 1])
        xin = ops.ln_modulate(x.contiguous(), shift=shift, scale=scale, eps=self.layernorm_epsilon,
                              rows_out=n_seq, row_offset=n_ref)
        lin = ops.gemm(xin.view(B * n_seq, d), self.linear.weight, self.linear.bias)
        return ops.unpatchify(lin, B, kwargs["rope_T"], kwargs["rope_H"], kwargs["rope_W"])


class AdaLNMixin(BaseMixin):
    """dit_video_crossattn_sc_xc.py:844-1203.  `layer_forward` runs one whole DiT block as ~18 kernel launches:
    adaLN vectors -> LN+modulate -> QKV GEMM -> RMSNorm+RoPE -> flash attention -> out-proj GEMM with fused
    bias/gate/residual -> LN(affine) -> cross q GEMM + RMSNorm -> text / CLIP K,V GEMMs + RMSNorm -> two
    attention passes (second accumulates) -> out-proj GEMM with fused bias/residual -> LN+modulate -> fc1 GEMM
    with fused bias+GELU-tanh -> fc2 GEMM with fused bias/gate/residual."""

    def __init__(self, hidden_size, num_layers, time_embed_dim, compressed_num_frames, transformer_args, qk_ln=True,
                 qk_ln_affine=None, hidden_size_head=None, params_dtype=torch.float, device=torch.device("cpu"),
                 elementwise_affine=True, share_adaln=False, use_i2v_clip=False, fp8_linear=False):
        super().__init__()
        if not (qk_ln and share_adaln and use_i2v_clip) or hidden_size_head != hidden_size:
            raise NotImplementedError("scail_b200 implements qk_ln=True over the full hidden width, share_adaln=True, use_i2v_clip=True")
        if getattr(transformer_args, "is_gated_mlp", False):
            raise NotImplementedError("gated MLP is not part of the SCAIL-14B config (use_SwiGLU: False)")
        self.num_layers = num_layers
        self.hidden_size = hidden_size
        self.layernorm_epsilon = transformer_args.layernorm_epsilon
        self.num_attention_heads = transformer_args.num_attention_heads
        self.share_adaln, self.use_i2v_clip, self.qk_ln = share_adaln, use_i2v_clip, qk_ln
        self.adaLN_modulations = nn.ParameterList(
            [nn.Parameter(torch.randn(1, 6, hidden_size) / hidden_size ** 0.5) for _ in range(num_layers)])
        mk = lambda: nn.ModuleList([_Norm(hidden_size) for _ in range(num_layers)])
        self.query_layernorm_list, self.key_layernorm_list = mk(), mk()
        self.cross_query_layernorm_list, self.cross_key_layernorm_list = mk(), mk()
        self.clip_feature_key_layernorm_list = mk()
        self.clip_feature_key_value_list = nn.ModuleList(
            [_Linear(hidden_size, 2 * hidden_size) for _ in range(num_layers)])
        self.cp = None  # scail_b200.parallel.ContextParallel or None
        # SURVEY §8f rank 1 (opt-in): text / CLIP K,V of every layer depend only on the prompt and the reference image,
        # yet the reference recomputes them in all 40 blocks of all 50 steps (dit_video_crossattn_sc_xc.py:1117-1130).
        # With cache_cross_kv=True, sampler.sample() precomputes them once per call (DiffusionTransformer.set_conditioning,
        # an explicit handle — nothing is keyed on tensor addresses) and every step reuses them: numerically identical.
        # bench.py keeps it OFF so that the timed step does the reference's full work.
        self.cache_cross_kv = False
        # Opt-in: the six per-block linears over all tokens (QKV, self-attention out, cross q, cross-attention out, fc1, fc2) run
        # as e4m3 GEMMs with one scale per token and per output channel (scail_gemm_fp8); everything else stays bf16.  The
        # e4m3 weights are derived on the GPU on first use and are not part of the state_dict.  A plain attribute: it can be
        # toggled between forwards.
        self.fp8_linear = fp8_linear

    # -- fp8 linears ---------------------------------------------------------------------------
    FP8_LINEARS = ("attention.query_key_value", "attention.dense", "cross_attention.query", "cross_attention.dense",
                   "mlp.dense_h_to_4h", "mlp.dense_4h_to_h")

    def fp8_weight(self, lin, streams=()):
        """(q e4m3 [out, in], scale fp32 [out]) of `lin.weight`, quantised on the current stream on first use and again
        whenever the parameter object, its storage or its version has changed (a checkpoint loaded after construction, an
        in-place edit), so a stale copy is never used.  The copy lives on `lin` (not in the state_dict) with only a weak
        reference to the weight: a replaced parameter is neither kept alive nor served.  A changed weight of the same shape
        is re-derived into the same buffers, so the pointers a CUDA graph captured stay valid.  Newly allocated buffers are
        recorded on `streams`, the other streams that will read them."""
        w = lin.weight
        tag = (w.data_ptr(), w._version)
        c = getattr(lin, "_fp8_cache", None)
        if c is not None and c[0]() is w and c[1] == tag:
            return c[2], c[3]
        if c is not None and c[2].shape == w.shape and c[2].device == w.device:
            q, sc = ops.quant_rows_fp8(w.detach(), c[2], c[3])
        else:
            lin._fp8_cache = None  # free the old copy before allocating the new one
            q, sc = ops.quant_rows_fp8(w.detach())
            for st in streams:
                q.record_stream(st)
                sc.record_stream(st)
        lin._fp8_cache = (weakref.ref(w), tag, q, sc)
        return q, sc

    def prepare_fp8_weights(self, num_layers=None, streams=()):
        """Bring the e4m3 copies of the first `num_layers` blocks' six linears up to date on the current stream.  Work that
        reads them on other streams must be ordered after this (DiffusionTransformer.forward does it before the context-parallel
        branch streams fork).  Returns the copies."""
        out = []
        for layer in list(self.transformer.layers)[:num_layers]:
            for name in self.FP8_LINEARS:
                out.extend(self.fp8_weight(layer.get_submodule(name), streams))
        return out

    def _fp8_act(self, x2, name):
        """x2 bf16 [M, K] -> its e4m3 rows and scales, in the per-stream workspace `name`."""
        M, K = x2.shape
        q = _WS.get(name, (M, K), x2.device, ops.FP8)
        sc = _WS.get(name + "_scale", (M,), x2.device, torch.float32)
        return ops.quant_rows_fp8(x2, q, sc)

    def _linear(self, x2, lin, x_scale=None, out=None, name="act8", **kw):
        """epilogue(x2 @ lin.weight^T + lin.bias) into `out`.  bf16 GEMM unless fp8_linear; then the e4m3 GEMM, on x2 itself when
        it is already e4m3 (with its row scales x_scale), else on x2 quantised into workspace `name`."""
        if not self.fp8_linear:
            return ops.gemm(x2, lin.weight, lin.bias, out=out, **kw)
        if x2.dtype != ops.FP8:
            x2, x_scale = self._fp8_act(x2, name)
        wq, ws = self.fp8_weight(lin)
        return ops.gemm_fp8(x2, x_scale, wq, ws, lin.bias, out=out, **kw)

    # -- hooks ---------------------------------------------------------------------------------
    def layer_forward(self, hidden_states, mask, *args, **kwargs):
        """One DiT block (:1009-1051).  IN-PLACE contract: when `hidden_states` is a contiguous bf16 tensor (what
        word_embedding_forward / the previous layer_forward return) the residual stream is updated in that very buffer by the
        fused `x + gate * (acc + bias)` GEMM epilogues and the same tensor is returned — the reference's out-of-place
        `hidden_states = hidden_states + ...` semantics are preserved for its caller (BaseTransformer.forward rebinds the name,
        sat/model/transformer.py:712-722), but a caller that keeps its own reference to the input sees it change.  Any other
        dtype / layout is first copied to a fresh bf16 buffer."""
        _need_cuda(hidden_states)
        l = int(kwargs["layer_id"])
        layer = self.transformer.layers[l]
        x = hidden_states
        if x.dtype != torch.bfloat16 or not x.is_contiguous():
            x = x.to(torch.bfloat16).contiguous()
        B, N, d = x.shape
        dev = x.device
        eps = self.layernorm_epsilon
        x2 = x.view(B * N, d)
        mod = ops.adaln_modulation(kwargs["emb"], self.adaLN_modulations[l].view(-1)).view(B, 6, d)  # :1025-1028
        fp8 = self.fp8_linear
        if fp8:
            ln8 = (_WS.get("ln8", (B * N, d), dev, ops.FP8), _WS.get("ln8_scale", (B * N,), dev, torch.float32))
        else:
            lnb = _WS.get("ln", (B, N, d), dev)

        def ln(**kw):
            """The block's LNs feed linears only: with fp8_linear they write e4m3 rows + scales.  -> (rows [B, N, d], scales)"""
            if fp8:
                ops.ln_modulate(x, eps=eps, out_fp8=ln8, **kw)
                return ln8[0].view(B, N, d), ln8[1]
            return ops.ln_modulate(x, out=lnb, eps=eps, **kw), None

        # ---- self attention (:1031-1036) ----
        h, hs = ln(shift=mod[:, 0], scale=mod[:, 1])
        ctx = _WS.get("ctx", (B * N, d), dev)
        self.attention_forward(h, mask, _ctx_out=ctx, _fp8_scale=hs, **kwargs)  # leaves merged-head context in ctx
        a = layer.attention
        self._linear(ctx, a.dense, out=x2, name="ctx8", epilogue=ops.EPI_BIAS_GATE_RES, gate=mod[:, 2], residual=x2,
                     rows_per_batch=N)

        # ---- cross attention (:1039-1042) ----
        pl = layer.post_cross_attention_layernorm
        h, hs = ln(gamma=pl.weight, beta=pl.bias)
        xkv_all = kwargs.get("_xkv_layers")
        self.cross_attention_forward(h, kwargs.get("cross_attention_mask"), kwargs["encoder_outputs"], _ctx_out=ctx,
                                     _xkv=xkv_all[l] if xkv_all is not None else None, _fp8_scale=hs,
                                     **{k: v for k, v in kwargs.items() if k not in ("cross_attention_mask", "encoder_outputs")})
        c = layer.cross_attention
        self._linear(ctx, c.dense, out=x2, name="ctx8", epilogue=ops.EPI_BIAS_RES, residual=x2)

        # ---- MLP (:1045-1050) ----
        h, hs = ln(shift=mod[:, 3], scale=mod[:, 4])
        m = layer.mlp
        inner = m.dense_h_to_4h.weight.shape[0]
        h1 = _WS.get("mlp", (B * N, inner), dev)
        self._linear(h.view(B * N, d), m.dense_h_to_4h, hs, out=h1, epilogue=ops.EPI_BIAS_GELU)
        self._linear(h1, m.dense_4h_to_h, out=x2, name="mlp8", epilogue=ops.EPI_BIAS_GATE_RES, gate=mod[:, 5], residual=x2,
                     rows_per_batch=N)
        return x

    def attention_forward(self, hidden_states, mask, _ctx_out=None, _fp8_scale=None, **kw_args):
        """:1058-1105.  Returns the out-projected attention output unless `_ctx_out` is given (then the
        merged-head context is left there for the fused out-proj epilogue of layer_forward).  hidden_states may be e4m3 rows
        with their scales in `_fp8_scale` (fp8_linear)."""
        l = int(kw_args["layer_id"])
        a = self.transformer.layers[l].attention
        B, N, d = hidden_states.shape
        dev = hidden_states.device
        H = self.num_attention_heads
        cos, sin = self._rope_tables(dev, **kw_args)
        h2 = hidden_states.view(B * N, d)
        if self.fp8_linear and h2.dtype != ops.FP8:
            h2, _fp8_scale = self._fp8_act(h2, "ln8")
        ctx = _ctx_out if _ctx_out is not None else torch.empty(B * N, d, device=dev, dtype=torch.bfloat16)
        wq, wk = self.query_layernorm_list[l].weight, self.key_layernorm_list[l].weight
        if self.cp is None or self.cp.size == 1:
            qkv = _WS.get("qkv", (B * N, 3 * d), dev)
            self._linear(h2, a.query_key_value, _fp8_scale, out=qkv)
            ops.rmsnorm_rope(qkv, N, d, [(0, wq), (d, wk)], cos, sin, eps=self.layernorm_epsilon)
            ops.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], ctx, B, H, N, N)
        else:
            # engine-style sequence parallelism (diffusion_video.py:495-552): the latents arrive pre-chunked on H or W, so the
            # RoPE tables built from rope_H/W_shift are already this rank's; otherwise tokens were sharded by shard_tokens()
            self.cp.self_attention(self, a, h2, B, N, d, H, wq, wk, cos, sin, ctx,
                                   tables_local=kw_args.get("chunk_dim") is not None, h_scale=_fp8_scale)
        if _ctx_out is not None:
            return None
        return self._linear(ctx, a.dense, name="ctx8").view(B, N, d)

    def cross_attention_forward(self, hidden_states, cross_attention_mask, encoder_outputs, _ctx_out=None, _fp8_scale=None,
                                **kw_args):
        """:1107-1203: text K/V and CLIP K/V are two separate softmaxes whose outputs are summed (F4).  hidden_states may be
        e4m3 rows with their scales in `_fp8_scale` (fp8_linear)."""
        l = int(kw_args["layer_id"])
        c = self.transformer.layers[l].cross_attention
        B, N, d = hidden_states.shape
        dev = hidden_states.device
        H = self.num_attention_heads
        eps = self.layernorm_epsilon
        bf = torch.bfloat16
        text = encoder_outputs.to(bf).contiguous()
        clip = kw_args["image_clip_features"].to(bf).contiguous()
        Lt, Lc = text.shape[1], clip.shape[1]
        xq = _WS.get("xq", (B * N, d), dev)
        self._linear(hidden_states.view(B * N, d), c.query, _fp8_scale, out=xq, name="ln8")
        ops.rmsnorm_rope(xq, N, d, [(0, self.cross_query_layernorm_list[l].weight)], eps=eps)
        pre = kw_args.get("_xkv")  # (tkv, ckv) of this layer from a Conditioning handle (rows of this call's batch elements)
        if pre is not None:
            tkv, ckv = pre
        else:
            tkv, ckv = self.cross_kv(l, text, clip)
        ctx = _ctx_out if _ctx_out is not None else torch.empty(B * N, d, device=dev, dtype=bf)
        ops.attention(xq, tkv[:, :d], tkv[:, d:], ctx, B, H, N, Lt)
        ops.attention(xq, ckv[:, :d], ckv[:, d:], ctx, B, H, N, Lc, accumulate=True)
        if _ctx_out is not None:
            return None
        return self._linear(ctx, c.dense, name="ctx8").view(B, N, d)

    def cross_kv(self, l, text, clip, keep=False):
        """Text and CLIP K,V of layer l (:1117-1130): K/V projection + K RMSNorm.  keep=True allocates fresh buffers (for a
        Conditioning handle) instead of the per-stream workspace."""
        c = self.transformer.layers[l].cross_attention
        B, Lt, d = text.shape
        Lc = clip.shape[1]
        dev, bf, eps = text.device, torch.bfloat16, self.layernorm_epsilon
        tkv = torch.empty(B * Lt, 2 * d, device=dev, dtype=bf) if keep else _WS.get("tkv", (B * Lt, 2 * d), dev)
        ops.gemm(text.view(B * Lt, d), c.key_value.weight, c.key_value.bias, out=tkv)
        ops.rmsnorm_rope(tkv, Lt, d, [(0, self.cross_key_layernorm_list[l].weight)], eps=eps)
        ckv_lin = self.clip_feature_key_value_list[l]
        ckv = torch.empty(B * Lc, 2 * d, device=dev, dtype=bf) if keep else _WS.get("ckv", (B * Lc, 2 * d), dev)
        ops.gemm(clip.view(B * Lc, d), ckv_lin.weight, ckv_lin.bias, out=ckv)
        ops.rmsnorm_rope(ckv, Lc, d, [(0, self.clip_feature_key_layernorm_list[l].weight)], eps=eps)
        return tkv, ckv

    def _rope_tables(self, dev, **kw):
        pe = getattr(self, "_pos_embed", None)
        if pe is not None:
            return pe.tables(dev, **kw)
        return rope.build_tables(dev, 128, kw["rope_T"], kw["rope_H"], kw["rope_W"], kw.get("rope_H_shift", 0),
                                 kw.get("rope_W_shift", 0), kw.get("global_rope_H", 0), kw.get("global_rope_W", 120))


# ------------------------------------------------------------------------------------------------
# standalone model
# ------------------------------------------------------------------------------------------------


class _MLPProj(nn.Module):  # dit_video_crossattn_sc_xc.py:31-45
    def __init__(self, in_dim, out_dim):
        super().__init__()
        self.proj = nn.Sequential(nn.LayerNorm(in_dim), nn.Linear(in_dim, in_dim), nn.GELU(),
                                  nn.Linear(in_dim, out_dim), nn.LayerNorm(out_dim))


class DiffusionTransformer(nn.Module):
    """Same ctor kwargs / forward signature / state_dict names as the reference class
    (dit_video_crossattn_sc_xc.py:1209-1587); SAT-free."""

    def __init__(self, transformer_args=None, num_frames=81, time_compressed_rate=4, latent_width=300,
                 latent_height=300, patch_size=(1, 2, 2), in_channels=20, out_channels=16, hidden_size=5120,
                 text_dim=4096, num_layers=40, num_attention_heads=40, elementwise_affine=False, time_freq_dim=256,
                 time_embed_dim=None, modules=None, share_adaln=True, use_SwiGLU=False, use_RMSNorm=False,
                 layernorm_epsilon=1e-6, inner_hidden_size=None, use_i2v_clip=True, dtype="bf16", fp8_linear=False, **kwargs):
        super().__init__()
        if use_SwiGLU or use_RMSNorm:
            raise NotImplementedError("SCAIL-14B uses the non-gated GELU-tanh MLP and LayerNorm (yaml:42-43)")
        self.patch_size = list(patch_size)
        self.num_frames, self.time_compressed_rate = num_frames, time_compressed_rate
        self.latent_width, self.latent_height = latent_width, latent_height
        self.in_channels, self.out_channels = in_channels, out_channels
        self.hidden_size, self.text_dim = hidden_size, text_dim
        self.time_embed_dim = time_embed_dim if time_embed_dim is not None else hidden_size
        self.time_freq_dim = time_freq_dim if time_freq_dim is not None else self.time_embed_dim
        self.num_layers, self.num_attention_heads = num_layers, num_attention_heads
        self.inner_hidden_size = inner_hidden_size if inner_hidden_size is not None else hidden_size * 4
        self.layernorm_epsilon = layernorm_epsilon
        self.share_adaln, self.use_i2v_clip = share_adaln, use_i2v_clip
        self.dtype = torch.bfloat16
        d = hidden_size
        targs = argparse.Namespace(layernorm_epsilon=layernorm_epsilon, num_attention_heads=num_attention_heads,
                                   inner_hidden_size=self.inner_hidden_size, is_gated_mlp=False,
                                   num_multi_query_heads=0, cross_num_multi_query_heads=0)
        self.transformer = _Transformer(num_layers, d, self.inner_hidden_size, num_attention_heads, layernorm_epsilon)
        self.time_embed = nn.Sequential(nn.Linear(self.time_freq_dim, self.time_embed_dim), nn.SiLU(),
                                        nn.Linear(self.time_embed_dim, self.time_embed_dim))
        self.adaln_projection = nn.Sequential(nn.SiLU(), nn.Linear(self.time_embed_dim, d * 6))
        self.text_embedding = nn.Sequential(nn.Linear(text_dim, d), nn.GELU(approximate="tanh"), nn.Linear(d, d))
        self.clip_proj = _MLPProj(1280, d)
        frames = (num_frames - 1) // time_compressed_rate + 1
        self.mixins = nn.ModuleDict()
        self.add_mixin("ulysse", UlyessAttentionMixin())
        self.add_mixin("pos_embed", Rotary3DPositionEmbeddingMixin(
            latent_height // self.patch_size[1], latent_width // self.patch_size[2], frames, d,
            d // num_attention_heads, interleaved_rope=True, patch_size=self.patch_size))
        self.add_mixin("patch_embed", ImagePatchEmbeddingMixin(in_channels, d, self.patch_size))
        self.add_mixin("adaln_layer", AdaLNMixin(d, num_layers, self.time_embed_dim, frames, targs, qk_ln=True,
                                                 qk_ln_affine=True, hidden_size_head=d, elementwise_affine=elementwise_affine,
                                                 share_adaln=True, use_i2v_clip=True, fp8_linear=fp8_linear))
        self.add_mixin("final_layer", FinalLayerMixin(d, self.time_embed_dim, self.patch_size, out_channels,
                                                      elementwise_affine, layernorm_epsilon, True))
        object.__setattr__(self.mixins["adaln_layer"], "_pos_embed", self.mixins["pos_embed"])

    def add_mixin(self, name, mixin, reinit=False):  # sat/model/base_model.py add_mixin
        self.mixins[name] = mixin
        _set_transformer(mixin, self.transformer)

    def get_mixin(self, name):
        return self.mixins[name]

    # -- per-step embeddings (dit_video_crossattn_sc_xc.py:1505-1555) -----------------------------
    def _text_clip_embeddings(self, context, clip_feats, B):
        """text_embedding (:1505) and clip_proj (:1507-1515): depend on the prompt / reference image only."""
        bf = torch.bfloat16
        dev = context.device
        d = self.hidden_size
        te = self.text_embedding
        Lt = context.shape[1]
        c2 = context.to(bf).contiguous().view(-1, self.text_dim)
        t1 = ops.gemm(c2, te[0].weight, te[0].bias, epilogue=ops.EPI_BIAS_GELU)
        text = ops.gemm(t1, te[2].weight, te[2].bias).view(context.shape[0], Lt, d)
        p = self.clip_proj.proj
        cf = clip_feats.to(device=dev, dtype=bf).contiguous()
        Bc, Lc, dc = cf.shape
        c0 = ops.ln_modulate(cf, gamma=p[0].weight, beta=p[0].bias, eps=p[0].eps)
        c1 = ops.gemm(c0.view(Bc * Lc, dc), p[1].weight, p[1].bias, epilogue=ops.EPI_BIAS_GELU_ERF)
        c3 = ops.gemm(c1, p[3].weight, p[3].bias).view(Bc, Lc, d)
        clip = ops.ln_modulate(c3, gamma=p[4].weight, beta=p[4].bias, eps=p[4].eps)
        if Bc != B:
            clip = clip.repeat(B // Bc, 1, 1)  # :1512-1515
        return text, clip

    def set_conditioning(self, context, image_clip_features, batch=None):
        """Precompute the step-invariant conditioning for `context` [b,L,text_dim] / `image_clip_features` [1|b,257,1280]
        (SURVEY §8f rank 1).  Subsequent forward() calls that pass these SAME tensor objects skip text_embedding, clip_proj
        and all 40 layers' text/CLIP K,V projections.  Returns the handle; clear_conditioning() drops it."""
        _need_cuda(context)
        B = batch if batch is not None else context.shape[0]
        cond = Conditioning(context, image_clip_features, B)
        cond.text, cond.clip = self._text_clip_embeddings(context, image_clip_features, B)
        ad = self.mixins["adaln_layer"]
        cond.xkv = [ad.cross_kv(l, cond.text, cond.clip, keep=True) for l in range(self.num_layers)]
        self._conditioning = cond
        return cond

    def clear_conditioning(self):
        self._conditioning = None

    def _embeddings(self, timesteps, context, clip_feats, B, cond=None):
        dev = context.device
        if cond is not None:
            text, clip = cond.text, cond.clip
        else:
            text, clip = self._text_clip_embeddings(context, clip_feats, B)
        t_emb = ops.timestep_embedding(timesteps.to(device=dev, dtype=torch.float32).contiguous(), self.time_freq_dim)
        e1 = ops.gemm(t_emb, self.time_embed[0].weight, self.time_embed[0].bias, epilogue=ops.EPI_BIAS_SILU)
        emb = ops.gemm(e1, self.time_embed[2].weight, self.time_embed[2].bias)
        adaln = ops.gemm(ops.silu(emb), self.adaln_projection[1].weight, self.adaln_projection[1].bias)
        return text, clip, emb, adaln

    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        """x [b,t,16,h,w]; kwargs: ref_concat [1|b,1,16,h,w], concat_smpl_render [1|b,t,16,h/2,w/2],
        image_clip_features [1|b,257,1280], concat_images (gate only, F12), history_mask [1|b,t,4,h,w] (optional: the mask
        channels of x, :1462-1467), chunk_dim (3 | 4 | None: the engine's pre-chunked sequence parallelism,
        diffusion_video.py:495-552).  Returns [b,t,16,h,w] bf16 (the local chunk when chunk_dim is set)."""
        _need_cuda(x)
        assert y is None, "SCAIL's DiT is not class-conditional (num_classes is None)"
        assert kwargs.get("ref_concat") is not None, "must specify ref_concat"
        b, t, c, h, w = x.shape
        bf = torch.bfloat16
        xb = ops.cast_bf16(x.contiguous()) if x.dtype == torch.float32 else x.to(bf).contiguous()
        ref = kwargs["ref_concat"].to(bf).contiguous()
        pose = kwargs["concat_smpl_render"].to(bf).contiguous()
        hm = kwargs.get("history_mask")
        if hm is not None:
            # non-zero mask channels: assemble the 20-channel inputs explicitly, exactly as :1462-1503 does
            rep = lambda a: a.to(bf).repeat(b // a.shape[0], 1, 1, 1, 1)
            xb = torch.cat([xb, rep(hm)], 2).contiguous()
            ref = torch.cat([rep(ref), torch.ones(b, 1, 4, h, w, device=x.device, dtype=bf)], 2).contiguous()
            pose = torch.cat([rep(pose), torch.ones(b, t, 4, h // 2, w // 2, device=x.device, dtype=bf)], 2).contiguous()
        cond = getattr(self, "_conditioning", None)
        if cond is not None and not cond.matches(context, kwargs["image_clip_features"], b):
            cond = None  # different prompt / image tensors: compute everything (never reuse by address)
        text, clip, emb, adaln = self._embeddings(timesteps, context, kwargs["image_clip_features"], b, cond)
        pp = reduce(mul, self.patch_size)
        kw = dict(seq_length=t * h * w // pp, pose_length=t * (h // 2) * (w // 2) // pp, ref_length=h * w // pp,
                  emb=adaln, final_layer_emb=emb, encoder_outputs=text, image_clip_features=clip,
                  cross_attention_mask=None, rope_T=t // self.patch_size[0], rope_H=h // self.patch_size[1],
                  rope_W=w // self.patch_size[2], global_rope_H=0, global_rope_W=120, rope_H_shift=0, rope_W_shift=0,
                  _xkv_layers=cond.xkv if cond is not None else None)
        ad = self.mixins["adaln_layer"]
        cp = ad.cp
        chunk_dim = kwargs.get("chunk_dim")
        if chunk_dim is not None:  # :1578-1585
            if cp is None or cp.size == 1:
                raise RuntimeError("chunk_dim is set but no ContextParallel group is attached (adaln_layer.cp)")
            if chunk_dim == 3:
                kw["rope_H_shift"] = cp.rank * kw["rope_H"]
            elif chunk_dim == 4:
                kw["rope_W_shift"] = cp.rank * kw["rope_W"]
            else:
                raise NotImplementedError("chunk_dim must be 3 (H) or 4 (W)")
            kw["chunk_dim"] = chunk_dim
        N = kw["ref_length"] + kw["seq_length"] + kw["pose_length"]
        hidden = _WS.get("hidden", (b, N, self.hidden_size), x.device)
        # the 16-channel inputs go straight to the gather kernel, which synthesises the mask channels
        hidden = self.mixins["patch_embed"].word_embedding_forward(None, images=xb, ref_concat=ref,
                                                                   concat_smpl_render=pose, _hidden_out=hidden)
        n_layers = int(kwargs.get("_num_layers") or self.num_layers)  # verification hook (bench.py cp_check_rel): first k blocks only
        if cp is None or cp.size == 1:
            for l in range(n_layers):
                hidden = ad.layer_forward(hidden, None, layer_id=l, **kw)
            return self.mixins["final_layer"].final_forward(hidden, **kw)
        # ---- context parallel: the CFG branches (independent batch elements) run on separate streams so that one
        # branch's K/V all-gather overlaps the other branch's GEMMs / attention.  Tokens are either sharded here
        # (replicated inputs) or already local (chunk_dim: the engine chunked the latents on H/W per rank) ----
        local = hidden if chunk_dim is not None else cp.shard_tokens(hidden)
        main = torch.cuda.current_stream()
        streams = cp.branch_streams(b, x.device)
        if ad.fp8_linear:  # every branch reads the same e4m3 weights: derive them here, before the branch streams wait on main
            ad.prepare_fp8_weights(n_layers, streams)
        per = []
        for i in range(b):
            kwi = dict(kw, emb=adaln[i:i + 1], encoder_outputs=text[i:i + 1], image_clip_features=clip[i:i + 1])
            if cond is not None:
                Lt, Lc = text.shape[1], clip.shape[1]
                kwi["_xkv_layers"] = [(tk[i * Lt:(i + 1) * Lt], ck[i * Lc:(i + 1) * Lc]) for tk, ck in cond.xkv]
            per.append([local[i:i + 1].contiguous(), kwi])
            streams[i].wait_stream(main)
        for l in range(n_layers):
            for i in range(b):
                with torch.cuda.stream(streams[i]):
                    per[i][0] = ad.layer_forward(per[i][0], None, layer_id=l, **per[i][1])
        for i in range(b):
            main.wait_stream(streams[i])
        hidden = torch.cat([h_ for h_, _ in per], 0)
        if chunk_dim is None:
            hidden = cp.gather_tokens(hidden, N)
        return self.mixins["final_layer"].final_forward(hidden, **kw)
