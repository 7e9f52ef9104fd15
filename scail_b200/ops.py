"""Thin torch-tensor wrappers over the C ABI (one function per entry point).  All tensors must be
CUDA tensors; there is no CPU path.  Launches go to torch.cuda.current_stream()."""
import math

import torch

from . import _lib

EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_BIAS_RES, EPI_BIAS_SILU, EPI_BIAS_GELU_ERF = range(6)

LAUNCHES = 0  # number of library kernels launched through this module (bench.py reports it)
ATTN_EVENTS = None  # bench.py sets this to a list to collect (start, end) CUDA events of self-attention launches


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _req(t, dtype=torch.bfloat16):
    if not t.is_cuda:
        raise RuntimeError("scail_b200 ops need CUDA tensors: there is no CPU fallback")
    if t.dtype != dtype:
        raise TypeError(f"expected {dtype}, got {t.dtype}")
    return t


def _count(n=1):
    global LAUNCHES
    LAUNCHES += n


def gemm(a, w, bias=None, out=None, epilogue=EPI_BIAS, gate=None, residual=None, rows_per_batch=0, out_fp32=False):
    """out[M,N] = epilogue(a[M,K] @ w[N,K]^T).  a/out may be row-strided 2-D views (stride(1)==1)."""
    _req(a), _req(w)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and a.stride(1) == 1 and w.stride(1) == 1
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    assert out.shape == (M, N) and out.stride(1) == 1
    gs = gate.stride(0) if gate is not None else 0
    _lib.check(_lib.lib().scail_gemm_bf16(
        _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(bias), _ptr(out), out.stride(0), M, N, K, epilogue,
        _ptr(gate), gs, rows_per_batch, _ptr(residual), residual.stride(0) if residual is not None else 0,
        1 if out.dtype == torch.float32 else 0, _stream()), "scail_gemm_bf16")
    _count()
    return out


FP8 = torch.float8_e4m3fn


def gemm_fp8(a, a_scale, w, w_scale, bias=None, out=None, epilogue=EPI_BIAS, gate=None, residual=None, rows_per_batch=0):
    """out[M,N] (bf16) = epilogue((a[M,K] @ w[N,K]^T) * a_scale[m] * w_scale[n]); a, w e4m3 with fp32 per-row scales (as
    quant_rows_fp8 makes them).  a/out may be row-strided 2-D views (stride(1)==1), K % 16 == 0."""
    _req(a, FP8), _req(w, FP8), _req(a_scale, torch.float32), _req(w_scale, torch.float32)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and a.stride(1) == 1 and w.stride(1) == 1
    assert a_scale.shape == (M,) and w_scale.shape == (N,) and a_scale.stride(0) == 1 and w_scale.stride(0) == 1
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.bfloat16)
    _req(out)
    assert out.shape == (M, N) and out.stride(1) == 1
    gs = gate.stride(0) if gate is not None else 0
    _lib.check(_lib.lib().scail_gemm_fp8(
        _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(bias), _ptr(out), out.stride(0), M, N, K, epilogue,
        _ptr(gate), gs, rows_per_batch, _ptr(residual), residual.stride(0) if residual is not None else 0, 0,
        _ptr(a_scale), _ptr(w_scale), _stream()), "scail_gemm_fp8")
    _count()
    return out


def quant_rows_fp8(x, q=None, scale=None):
    """Row-wise e4m3: x bf16 [M, K] (row-strided 2-D view) -> (q e4m3 [M, K], scale fp32 [M]) with scale = amax(|row|) / 448
    (1 for an all-zero row) and q = satfinite_rn(x / scale)."""
    _req(x)
    assert x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    if q is None:
        q = torch.empty(M, K, device=x.device, dtype=FP8)
    if scale is None:
        scale = torch.empty(M, device=x.device, dtype=torch.float32)
    _req(q, FP8), _req(scale, torch.float32)
    assert q.shape == (M, K) and q.is_contiguous() and scale.shape == (M,) and scale.is_contiguous()
    _lib.check(_lib.lib().scail_quant_rows_fp8(_ptr(x), x.stride(0), _ptr(q), _ptr(scale), M, K, _stream()),
               "scail_quant_rows_fp8")
    _count()
    return q, scale


def ln_modulate(x, out=None, gamma=None, beta=None, shift=None, scale=None, eps=1e-6, rows_out=None, row_offset=0,
                out_fp8=None):
    """x [B, Nin, D] -> out [B, rows_out, D] = modulate(LN(x[:, row_offset:row_offset+rows_out])).
    out_fp8=(q, s): write that result quantised instead, q e4m3 [B*rows_out, D] and s fp32 [B*rows_out] (bit for bit
    quant_rows_fp8 of the bf16 result), and return (q, s)."""
    _req(x)
    B, n_in, D = x.shape
    rows_out = n_in if rows_out is None else rows_out
    assert x.is_contiguous()
    ms = shift.stride(0) if shift is not None else 0
    if shift is not None:
        assert shift.stride(-1) == 1 and scale.stride(-1) == 1 and scale.stride(0) == ms
    if out_fp8 is not None:
        assert out is None
        q, s = out_fp8
        _req(q, FP8), _req(s, torch.float32)
        assert q.is_contiguous() and q.numel() == B * rows_out * D and s.is_contiguous() and s.numel() == B * rows_out
        _lib.check(_lib.lib().scail_ln_modulate_fp8(_ptr(x), _ptr(q), _ptr(s), _ptr(gamma), _ptr(beta), _ptr(shift),
                                                    _ptr(scale), ms, B, rows_out, n_in, row_offset, D, eps, _stream()),
                   "scail_ln_modulate_fp8")
        _count()
        return out_fp8
    if out is None:
        out = torch.empty(B, rows_out, D, device=x.device, dtype=torch.bfloat16)
    assert out.is_contiguous()
    _lib.check(_lib.lib().scail_ln_modulate(_ptr(x), _ptr(out), _ptr(gamma), _ptr(beta), _ptr(shift), _ptr(scale), ms,
                                            B, rows_out, n_in, row_offset, D, eps, _stream()), "scail_ln_modulate")
    _count()
    return out


def rmsnorm_rope(buf, rows_per_batch, D, slabs, cos=None, sin=None, eps=1e-6):
    """In-place RMSNorm(+RoPE) on column slabs [(col_offset, weight), ...] of the 2-D bf16 matrix buf."""
    _req(buf)
    assert buf.dim() == 2 and buf.stride(1) == 1 and 1 <= len(slabs) <= 2
    (o0, w0) = slabs[0]
    (o1, w1) = slabs[1] if len(slabs) == 2 else (0, None)
    _lib.check(_lib.lib().scail_rmsnorm_rope(_ptr(buf), buf.stride(0), buf.shape[0], rows_per_batch, D, len(slabs),
                                             o0, _ptr(w0), o1, _ptr(w1), _ptr(cos), _ptr(sin), eps, _stream()),
               "scail_rmsnorm_rope")
    _count()
    return buf


def attention(q, k, v, out, B, H, q_len, kv_len, q_batch_rows=None, kv_batch_rows=None, scale=None, accumulate=False):
    """q/k/v/out: 2-D row-strided bf16 views [rows, H*128] (stride(1)==1); head h = columns h*128..h*128+127."""
    for t in (q, k, v, out):
        _req(t)
        assert t.dim() == 2 and t.stride(1) == 1
    q_batch_rows = q_len if q_batch_rows is None else q_batch_rows
    kv_batch_rows = kv_len if kv_batch_rows is None else kv_batch_rows
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and kv_len > 1024:  # self-attention launches only
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    _lib.check(_lib.lib().scail_attention(_ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
                                          out.stride(0), B, H, q_len, kv_len, q_batch_rows, kv_batch_rows, q.shape[0],
                                          k.shape[0], scale, 1 if accumulate else 0, _stream()), "scail_attention")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()
    return out


def attention_partial(q, k, v, o32, state, B, H, q_len, ranges, q_batch_rows=None, kv_batch_rows=None, scale=None):
    """Attention of q over the key rows `ranges` = [(off0, len0)] or [(off0, len0), (off1, len1)] of every batch (offsets inside a
    batch of kv_batch_rows rows).  o32: fp32 [rows, H*128] (normalised partial result), state: fp32 [rows, H, 2] = (max, sum)."""
    for t in (q, k, v):
        _req(t)
        assert t.dim() == 2 and t.stride(1) == 1
    _req(o32, torch.float32), _req(state, torch.float32)
    assert o32.dim() == 2 and o32.stride(1) == 1 and state.is_contiguous() and state.numel() == o32.shape[0] * H * 2
    (o0, l0) = ranges[0]
    (o1, l1) = ranges[1] if len(ranges) > 1 else (0, 0)
    q_batch_rows = q_len if q_batch_rows is None else q_batch_rows
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and l0 + l1 > 1024:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    _lib.check(_lib.lib().scail_attention_partial(_ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(o32),
                                                  o32.stride(0), _ptr(state), B, H, q_len, o0, l0, o1, l1, q_batch_rows,
                                                  kv_batch_rows, q.shape[0], k.shape[0], scale, _stream()), "scail_attention_partial")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()


def attention_merge(o32_a, state_a, o32_b, state_b, out, H):
    """out (bf16 [rows, H*128]) = merge of two partial attention results over disjoint key sets (see attention_partial)."""
    _req(out)
    rows = out.shape[0]
    assert o32_a.shape == o32_b.shape and o32_a.stride(0) == o32_b.stride(0) and out.stride(1) == 1
    _lib.check(_lib.lib().scail_attention_merge(_ptr(o32_a), _ptr(state_a), _ptr(o32_b), _ptr(state_b), _ptr(out), o32_a.stride(0),
                                                out.stride(0), rows, H, _stream()), "scail_attention_merge")
    _count()
    return out


def adaln_modulation(emb, param, out=None):
    _req(emb), _req(param)
    B, n = emb.shape
    assert param.numel() == n
    if out is None:
        out = torch.empty_like(emb)
    _lib.check(_lib.lib().scail_adaln_modulation(_ptr(emb), _ptr(param), _ptr(out), B, n, _stream()), "scail_adaln_modulation")
    _count()
    return out


def silu(x):
    _req(x)
    out = torch.empty_like(x)
    _lib.check(_lib.lib().scail_silu(_ptr(x), _ptr(out), x.numel(), _stream()), "scail_silu")
    _count()
    return out


def timestep_embedding(t, dim):
    _req(t, torch.float32)
    out = torch.empty(t.shape[0], dim, device=t.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_timestep_embedding(_ptr(t), _ptr(out), t.shape[0], dim, _stream()), "scail_timestep_embedding")
    _count()
    return out


def patchify(x, ref, pose):
    """x [B,T,C,H,W], ref [Br,1,C,H,W], pose [Bp,T,C,H/2,W/2] (bf16, C = 16 or 20)
    -> (a_main [B,n_main,80], a_pose [B,n_pose,80]).  C == 16: mask channels are synthesised."""
    _req(x), _req(ref), _req(pose)
    B, T, C, H, W = x.shape
    assert C in (16, 20) and ref.shape[2] == C and pose.shape[2] == C
    assert x.is_contiguous() and ref.is_contiguous() and pose.is_contiguous()
    n_main = (1 + T) * (H // 2) * (W // 2)
    n_pose = T * (H // 4) * (W // 4)
    a_main = torch.empty(B, n_main, 80, device=x.device, dtype=torch.bfloat16)
    a_pose = torch.empty(B, n_pose, 80, device=x.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_patchify(_ptr(x), _ptr(ref), _ptr(pose), _ptr(a_main), _ptr(a_pose), B, ref.shape[0],
                                         pose.shape[0], T, H, W, C, _stream()), "scail_patchify")
    _count()
    return a_main, a_pose


def unpatchify(lin, B, T, Hp, Wp):
    _req(lin)
    assert lin.is_contiguous() and lin.numel() == B * T * Hp * Wp * 64
    out = torch.empty(B, T, 16, 2 * Hp, 2 * Wp, device=lin.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_unpatchify(_ptr(lin), _ptr(out), B, T, Hp, Wp, _stream()), "scail_unpatchify")
    _count()
    return out


def cfg_euler_(x, v, scale, dsigma):
    """x (fp32, [1,...]) += dsigma * (v[0] + scale * (v[1] - v[0])); v bf16 [2, ...]."""
    _req(x, torch.float32), _req(v)
    assert x.is_contiguous() and v.is_contiguous() and v.numel() == 2 * x.numel()
    _lib.check(_lib.lib().scail_cfg_euler(_ptr(x), _ptr(v), x.numel(), float(scale), float(dsigma), _stream()), "scail_cfg_euler")
    _count()
    return x


def cast_bf16(x):
    _req(x, torch.float32)
    out = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_cast_f32_bf16(_ptr(x.contiguous()), _ptr(out), x.numel(), _stream()), "scail_cast_f32_bf16")
    _count()
    return out


# ---------------------------------------------------------------- Wan2.1 VAE decode ops (channels-last)
CONV_EPI_BIAS, CONV_EPI_BIAS_RES, CONV_EPI_HEAD_CLAMP = range(3)


def conv3d_fusable(x, kh, kw, cout):
    """True when conv3d_cl can also emit SiLU(RMS_norm(out) * gamma) from its epilogue (row-tile kernel, Cout == 96)."""
    return kh == 3 and kw == 3 and x.shape[2] >= 128 and cout == 96


def _hist_arg(hist, x, kt):
    """(pointer, frames) of an optional causal history [T_hist, H, W, Cin] for the conv input x (scail_conv3d_cl_hist)."""
    if hist is None or hist.shape[0] == 0:
        return None, 0
    _req(hist)
    assert hist.is_contiguous() and hist.shape[1:] == x.shape[1:] and hist.shape[0] <= kt - 1, (tuple(hist.shape), tuple(x.shape), kt)
    return _ptr(hist), hist.shape[0]


def conv3d_cl(x, w2, bias, kt, kh, kw, cout, out=None, residual=None, fmul=1, ocols=None, head=False, norm_gamma=None,
              want_raw=True, *, hist=None, out_frame_offset=0):
    """x [T,H,W,Cin] bf16 channels-last; w2 [cout, kt*kh*kw*Cin] bf16.  Returns out [T*fmul,H,W,ocols] bf16
    (or fp32 planes [cout,T,H,W] when head=True).  With norm_gamma (see conv3d_fusable) returns (out, out2) where
    out2 = SiLU(RMS_norm(out) * gamma) comes from the same epilogue; want_raw=False skips writing `out` (returned None).
    hist [T_hist <= kt-1, H, W, Cin]: the input frames preceding x[0] (causal history of a chunked run) instead of zero
    padding.  head=True with out_frame_offset: write frames [out_frame_offset, out_frame_offset + T) of a given fp32
    out [cout, T_total, H, W]."""
    _req(x), _req(w2)
    T, H, W, Cin = x.shape
    assert x.is_contiguous() and w2.is_contiguous() and w2.shape == (cout, kt * kh * kw * Cin)
    hp, th = _hist_arg(hist, x, kt)
    ocols = cout if ocols is None else ocols
    out2 = None
    plane = 0
    if head:
        if out is None:
            assert out_frame_offset == 0, "out_frame_offset needs an output tensor"
            out = torch.empty(cout, T, H, W, device=x.device, dtype=torch.float32)
        _req(out, torch.float32)
        assert out.is_contiguous() and out.shape[0] == cout and out.shape[2:] == (H, W)
        assert 0 <= out_frame_offset and out_frame_offset + T <= out.shape[1]
        epi, ldo, plane = CONV_EPI_HEAD_CLAMP, 0, out.stride(0)
    else:
        assert out_frame_offset == 0, "out_frame_offset is for the head epilogue"
        if norm_gamma is not None:
            assert conv3d_fusable(x, kh, kw, cout) and fmul == 1
            out2 = torch.empty(T, H, W, cout, device=x.device, dtype=torch.bfloat16)
        if out is None and (want_raw or norm_gamma is None):
            out = torch.empty(T * fmul, H, W, ocols, device=x.device, dtype=torch.bfloat16)
        epi, ldo = (CONV_EPI_BIAS_RES if residual is not None else CONV_EPI_BIAS), (out.shape[-1] if out is not None else cout)
        assert out is None or out.is_contiguous()
    _lib.check(_lib.lib().scail_conv3d_cl_hist(_ptr(x), T, H, W, Cin, _ptr(w2), cout, kt, kh, kw, _ptr(bias), _ptr(residual),
                                               residual.shape[-1] if residual is not None else 0, _ptr(out), ldo, ocols, fmul,
                                               epi, _ptr(norm_gamma), _ptr(out2), hp, th, plane, out_frame_offset, _stream()),
               "scail_conv3d_cl_hist")
    _count()
    return (out, out2) if norm_gamma is not None else out


def conv3d_strided_cl(x, w2, bias, kt, kh, kw, cout, out_shape, sstride=1, pad_h=0, pad_w=0, tstride=1, toff=0, out=None, *,
                      hist=None):
    """Strided conv for the VAE encoder: x [T,H,W,Cin] -> out [T_out,H_out,W_out,cout] (see scail_conv3d_strided_cl);
    hist [T_hist <= kt-1, H, W, Cin]: input frames preceding x[0], read for the taps at frames < 0 (scail_conv3d_strided_cl_hist)."""
    _req(x), _req(w2)
    T, H, W, Cin = x.shape
    assert x.is_contiguous() and w2.is_contiguous() and w2.shape == (cout, kt * kh * kw * Cin)
    hp, th = _hist_arg(hist, x, kt)
    To, Ho, Wo = out_shape
    if out is None:
        out = torch.empty(To, Ho, Wo, cout, device=x.device, dtype=torch.bfloat16)
    assert out.is_contiguous() and out.shape[-1] == cout
    _lib.check(_lib.lib().scail_conv3d_strided_cl_hist(_ptr(x), T, H, W, Cin, _ptr(w2), cout, kt, kh, kw, _ptr(bias), _ptr(out),
                                                       cout, To, Ho, Wo, sstride, pad_h, pad_w, tstride, toff, hp, th, _stream()),
               "scail_conv3d_strided_cl_hist")
    _count()
    return out


def rmsnorm_cl(x, gamma, silu=True, out=None):
    _req(x), _req(gamma)
    C = x.shape[-1]
    assert x.is_contiguous() and gamma.numel() == C
    if out is None:
        out = torch.empty_like(x)
    _lib.check(_lib.lib().scail_rmsnorm_cl(_ptr(x), _ptr(gamma), _ptr(out), x.numel() // C, C, 1 if silu else 0, _stream()),
               "scail_rmsnorm_cl")
    _count()
    return out


def upsample2x_cl(x):
    _req(x)
    Fr, H, W, C = x.shape
    assert x.is_contiguous()
    out = torch.empty(Fr, 2 * H, 2 * W, C, device=x.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_upsample2x_cl(_ptr(x), _ptr(out), Fr, H, W, C, _stream()), "scail_upsample2x_cl")
    _count()
    return out


def vae_latent_to_cl(z, mean, inv_std):
    """z [16,T,h,w] bf16 -> [T,h,w,16] bf16 = z / inv_std + mean."""
    _req(z), _req(mean, torch.float32), _req(inv_std, torch.float32)
    C, T, h, w = z.shape
    assert C == 16 and z.is_contiguous()
    out = torch.empty(T, h, w, 16, device=z.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_vae_latent_to_cl(_ptr(z), _ptr(mean), _ptr(inv_std), _ptr(out), T, h, w, _stream()),
               "scail_vae_latent_to_cl")
    _count()
    return out


def softmax_rows(s, scale, out=None):
    _req(s, torch.float32)
    rows, cols = s.shape
    assert s.is_contiguous()
    if out is None:
        out = torch.empty(rows, cols, device=s.device, dtype=torch.bfloat16)
    _lib.check(_lib.lib().scail_softmax_rows(_ptr(s), _ptr(out), rows, cols, float(scale), _stream()), "scail_softmax_rows")
    _count()
    return out
