"""Thin torch-tensor wrappers over the C ABI (one function per entry point).  All tensors must be
CUDA tensors; there is no CPU path.  Launches go to torch.cuda.current_stream()."""
import ctypes
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
INT8 = torch.int8


def gemm_fp8(a, a_scale, w, w_scale, bias=None, out=None, epilogue=EPI_BIAS, gate=None, residual=None, rows_per_batch=0):
    """out[M,N] (bf16) = epilogue((a[M,K] @ w[N,K]^T) * a_scale[m] * w_scale[n]); a, w e4m3 with fp32 per-row scales (as
    quant_rows_fp8 makes them).  a/out may be row-strided 2-D views (stride(1)==1), K % 16 == 0.
    a and w both int8 (torch.int8 codes in the INT8 row format, quant_rows_fp8 with an int8 q): the INT8 GEMM
    (scail_gemm_int8), the product exact in s32, K <= 131072.  Mixed operand dtypes raise TypeError."""
    int8 = a.dtype == INT8
    if int8 != (w.dtype == INT8):
        raise TypeError(f"gemm_fp8: a and w must both be e4m3 or both be int8, got {a.dtype} and {w.dtype}")
    _req(a, INT8 if int8 else FP8), _req(w, INT8 if int8 else FP8), _req(a_scale, torch.float32), _req(w_scale, torch.float32)
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and a.stride(1) == 1 and w.stride(1) == 1
    assert a_scale.shape == (M,) and w_scale.shape == (N,) and a_scale.stride(0) == 1 and w_scale.stride(0) == 1
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.bfloat16)
    _req(out)
    assert out.shape == (M, N) and out.stride(1) == 1
    gs = gate.stride(0) if gate is not None else 0
    name = "scail_gemm_int8" if int8 else "scail_gemm_fp8"
    _lib.check(getattr(_lib.lib(), name)(
        _ptr(a), a.stride(0), _ptr(w), w.stride(0), _ptr(bias), _ptr(out), out.stride(0), M, N, K, epilogue,
        _ptr(gate), gs, rows_per_batch, _ptr(residual), residual.stride(0) if residual is not None else 0, 0,
        _ptr(a_scale), _ptr(w_scale), _stream()), name)
    _count()
    return out


def quant_rows_fp8(x, q=None, scale=None):
    """Row-wise e4m3: x bf16 [M, K] (row-strided 2-D view) -> (q e4m3 [M, K], scale fp32 [M]) with scale = amax(|row|) / 448
    (1 for an all-zero row) and q = satfinite_rn(x / scale).  An int8 q selects the INT8 row format (scail_quant_rows_int8):
    scale = amax(|row|) / 127 (1 for an all-zero row) and q = round-half-even(x / scale) saturated to [-127, 127]."""
    _req(x)
    assert x.dim() == 2 and x.stride(1) == 1
    M, K = x.shape
    if q is None:
        q = torch.empty(M, K, device=x.device, dtype=FP8)
    if scale is None:
        scale = torch.empty(M, device=x.device, dtype=torch.float32)
    int8 = q.dtype == INT8
    _req(q, INT8 if int8 else FP8), _req(scale, torch.float32)
    assert q.shape == (M, K) and q.is_contiguous() and scale.shape == (M,) and scale.is_contiguous()
    name = "scail_quant_rows_int8" if int8 else "scail_quant_rows_fp8"
    _lib.check(getattr(_lib.lib(), name)(_ptr(x), x.stride(0), _ptr(q), _ptr(scale), M, K, _stream()), name)
    _count()
    return q, scale


def ln_modulate(x, out=None, gamma=None, beta=None, shift=None, scale=None, eps=1e-6, rows_out=None, row_offset=0,
                out_fp8=None):
    """x [B, Nin, D] -> out [B, rows_out, D] = modulate(LN(x[:, row_offset:row_offset+rows_out])).
    out_fp8=(q, s): write that result quantised instead, q e4m3 [B*rows_out, D] and s fp32 [B*rows_out] (bit for bit
    quant_rows_fp8 of the bf16 result), and return (q, s).  An int8 q writes the INT8 row format instead
    (scail_ln_modulate_int8, bit for bit quant_rows_fp8 of the bf16 result into an int8 q)."""
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
        int8 = q.dtype == INT8
        _req(q, INT8 if int8 else FP8), _req(s, torch.float32)
        assert q.is_contiguous() and q.numel() == B * rows_out * D and s.is_contiguous() and s.numel() == B * rows_out
        name = "scail_ln_modulate_int8" if int8 else "scail_ln_modulate_fp8"
        _lib.check(getattr(_lib.lib(), name)(_ptr(x), _ptr(q), _ptr(s), _ptr(gamma), _ptr(beta), _ptr(shift),
                                             _ptr(scale), ms, B, rows_out, n_in, row_offset, D, eps, _stream()), name)
        _count()
        return out_fp8
    if out is None:
        out = torch.empty(B, rows_out, D, device=x.device, dtype=torch.bfloat16)
    assert out.is_contiguous()
    _lib.check(_lib.lib().scail_ln_modulate(_ptr(x), _ptr(out), _ptr(gamma), _ptr(beta), _ptr(shift), _ptr(scale), ms,
                                            B, rows_out, n_in, row_offset, D, eps, _stream()), "scail_ln_modulate")
    _count()
    return out


def fp8_pad(L):
    """L_pad of the fp8 self-attention operands: L rounded up to the 128-key tile."""
    return (L + 127) // 128 * 128


def rmsnorm_rope(buf, rows_per_batch, D, slabs, cos=None, sin=None, eps=1e-6, out_fp8=None):
    """In-place RMSNorm(+RoPE) on column slabs [(col_offset, weight), ...] of the 2-D bf16 matrix buf.
    out_fp8=[(q8, s8) per slab]: write the result quantised instead (buf is left as it is) for attention_fp8: q8 e4m3
    [rows, D] (2-D, stride(1)==1) and s8 fp32 [B, D/128, L_pad] (one scale per token and 128-wide head, zeros past
    rows_per_batch); bit for bit quant_rows_fp8 of the bf16 result viewed as [rows * D/128, 128].  Returns out_fp8."""
    _req(buf)
    assert buf.dim() == 2 and buf.stride(1) == 1 and 1 <= len(slabs) <= 2
    (o0, w0) = slabs[0]
    (o1, w1) = slabs[1] if len(slabs) == 2 else (0, None)
    if out_fp8 is not None:
        assert len(out_fp8) == len(slabs)
        rows = buf.shape[0]
        q8s = [q for q, _ in out_fp8]
        for q, s in out_fp8:
            _req(q, FP8), _req(s, torch.float32)
            assert q.dim() == 2 and q.shape == (rows, D) and q.stride(1) == 1 and q.stride(0) == q8s[0].stride(0)
            assert s.is_contiguous() and s.shape == (rows // rows_per_batch, D // 128, s.shape[-1])
        (qa, sa) = out_fp8[0]
        (qb, sb) = out_fp8[1] if len(out_fp8) == 2 else (None, None)
        _lib.check(_lib.lib().scail_rmsnorm_rope_fp8(
            _ptr(buf), buf.stride(0), rows, rows_per_batch, D, len(slabs), o0, _ptr(w0), o1, _ptr(w1), _ptr(cos), _ptr(sin), eps,
            _ptr(qa), _ptr(sa), _ptr(qb), _ptr(sb), qa.stride(0), sa.shape[-1], _stream()), "scail_rmsnorm_rope_fp8")
        _count()
        return out_fp8
    _lib.check(_lib.lib().scail_rmsnorm_rope(_ptr(buf), buf.stride(0), buf.shape[0], rows_per_batch, D, len(slabs),
                                             o0, _ptr(w0), o1, _ptr(w1), _ptr(cos), _ptr(sin), eps, _stream()),
               "scail_rmsnorm_rope")
    _count()
    return buf


def rmsnorm_rope_int8q(buf, rows_per_batch, D, slabs, q8, q_scale, cos=None, sin=None, eps=1e-6):
    """fp8_attention="int8_qk" form of rmsnorm_rope over the two slabs [(q_offset, wq), (k_offset, wk)] of the 2-D bf16 buf:
    Q goes to INT8 rows q8 [rows, D] (2-D, stride(1)==1) with scales q_scale fp32 [B, D/128, L_pad] (s = amax / 127, q =
    round-half-even(x / s) clamped to [-127, 127], one per token and 128-wide head, zeros past rows_per_batch), bit for bit
    the quantised bf16 result; K is normalised in place in bf16 exactly as rmsnorm_rope writes it.  Returns (q8, q_scale)."""
    _req(buf), _req(q8, INT8), _req(q_scale, torch.float32)
    assert buf.dim() == 2 and buf.stride(1) == 1 and len(slabs) == 2
    (o0, w0), (o1, w1) = slabs
    rows = buf.shape[0]
    assert q8.dim() == 2 and q8.shape == (rows, D) and q8.stride(1) == 1
    assert q_scale.is_contiguous() and q_scale.shape == (rows // rows_per_batch, D // 128, q_scale.shape[-1])
    _lib.check(_lib.lib().scail_rmsnorm_rope_int8q(
        _ptr(buf), buf.stride(0), rows, rows_per_batch, D, 2, o0, _ptr(w0), o1, _ptr(w1), _ptr(cos), _ptr(sin), eps,
        _ptr(q8), _ptr(q_scale), q8.stride(0), q_scale.shape[-1], _stream()), "scail_rmsnorm_rope_int8q")
    _count()
    return q8, q_scale


KMEAN_ROWS = 256  # keys per fp64 partial sum of quant_k_int8


def quant_k_int8_partial_len(B, H, L):
    """fp64 entries of quant_k_int8's partial-sum workspace: B ceil(L / 256) H 128."""
    return B * -(-int(L) // KMEAN_ROWS) * H * 128


def quant_k_int8(k, B, H, L, k8=None, scale=None, kbar=None, partial=None):
    """K operand of attention_int8qk: k bf16 [B*L, H*128] (2-D row-strided view) -> (k8 int8 [B*L, H*128], scale fp32
    [B, H, L_pad], kbar fp32 [B, H*128]).  kbar is the per-(batch, channel) mean over the L keys (fp64 sums over fixed
    256-key chunks, added in order, divided by L in fp64, rounded once); k8 and scale quantise K' = f32(k) - kbar (one fp32
    rounding) per token and head in the INT8 row format of rmsnorm_rope_int8q.  partial: fp64 workspace of
    quant_k_int8_partial_len(B, H, L) entries (allocated when None).  Bit-reproducible, no host reads."""
    _req(k)
    assert k.dim() == 2 and k.stride(1) == 1 and k.shape == (B * L, H * 128)
    Lp = fp8_pad(L)
    dev = k.device
    k8 = torch.empty(B * L, H * 128, device=dev, dtype=INT8) if k8 is None else k8
    scale = torch.empty(B, H, Lp, device=dev, dtype=torch.float32) if scale is None else scale
    kbar = torch.empty(B, H * 128, device=dev, dtype=torch.float32) if kbar is None else kbar
    n = quant_k_int8_partial_len(B, H, L)
    partial = torch.empty(n, device=dev, dtype=torch.float64) if partial is None else partial
    _req(k8, INT8), _req(scale, torch.float32), _req(kbar, torch.float32), _req(partial, torch.float64)
    assert k8.dim() == 2 and k8.shape == (B * L, H * 128) and k8.stride(1) == 1
    assert scale.is_contiguous() and scale.shape == (B, H, Lp) and kbar.is_contiguous() and kbar.shape == (B, H * 128)
    assert partial.is_contiguous()
    _lib.check(_lib.lib().scail_quant_k_int8(_ptr(k), k.stride(0), _ptr(k8), k8.stride(0), _ptr(scale), _ptr(kbar),
                                             _ptr(partial), partial.numel(), B, H, L, Lp, _stream()), "scail_quant_k_int8")
    _count(3)
    return k8, scale, kbar


def attention_int8qk(q8, q_scale, k8, k_scale, vt, v_scale, out, B, H, L, scale=None, tiles=None, bh_maps=None):
    """Self-attention with INT8 Q and K (q_len == kv_len == L): q8 and its scales from rmsnorm_rope_int8q, k8 and its scales
    from quant_k_int8 (smoothed K), (vt, v_scale) from quant_vt_fp8; out bf16 [B*L, H*128] merged heads.  S = Q K^T is
    exact in s32; V, P and the softmax are attention_fp8's.  tiles: one block-sparse map for every (batch, head), as for
    attention_sparse; bh_maps=(ptr, idx): per-(batch, head) maps as for attention_sparse_bh.  At most one of the two."""
    if tiles is not None and bh_maps is not None:
        raise ValueError("attention_int8qk: give tiles or bh_maps, not both")
    m = _tile_map(tiles, L) if tiles is not None else None
    for t in (q8, k8):
        _req(t, INT8)
        assert t.dim() == 2 and t.stride(1) == 1 and t.shape == (B * L, H * 128)
    Lp = fp8_pad(L)
    for s in (q_scale, k_scale):
        _req(s, torch.float32)
        assert s.is_contiguous() and s.shape == (B, H, Lp)
    _req(vt, FP8), _req(v_scale, torch.float32), _req(out)
    assert vt.is_contiguous() and vt.shape == (B, H, 128, Lp) and v_scale.is_contiguous() and v_scale.shape == (B, H, 128)
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (B * L, H * 128)
    ptr = idx = None
    ps = ids = 0
    if m is not None:
        m._check_for(L, q8.device)
        ptr, idx = m.ptr, m.idx
    elif bh_maps is not None:
        ptr, idx = bh_maps
        ps, ids = _bh_maps(ptr, idx, B, H, L, q8.device)
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and L > 1024:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    _lib.check(_lib.lib().scail_attention_int8qk(_ptr(q8), q8.stride(0), _ptr(q_scale), _ptr(k8), k8.stride(0), _ptr(k_scale),
                                                 _ptr(vt), _ptr(v_scale), _ptr(out), out.stride(0), B, H, 128, L, Lp, scale,
                                                 _ptr(ptr), ps, _ptr(idx), ids, _stream()), "scail_attention_int8qk")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()
    return out


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


ATT_TILE = 128  # query rows and keys per attention tile


def check_tile_map(kv_tile_ptr, kv_tile_idx, q_len, kv_len):
    """Validate a block-sparse attention map on the host (array-likes of ints): kv_tile_ptr [ceil(q_len/128) + 1] with
    ptr[0] == 0 and ptr[-1] == len(kv_tile_idx); every row ptr[q]..ptr[q+1] non-empty, strictly ascending, each index in
    [0, ceil(kv_len/128)).  Raises ValueError naming the first violation."""
    import numpy as np
    ptr = np.asarray(kv_tile_ptr)
    idx = np.asarray(kv_tile_idx)
    n_q, n_kv = -(-int(q_len) // ATT_TILE), -(-int(kv_len) // ATT_TILE)
    if q_len <= 0 or kv_len <= 0:
        raise ValueError(f"tile map: q_len={q_len} and kv_len={kv_len} must be positive")
    if ptr.ndim != 1 or idx.ndim != 1 or not np.issubdtype(ptr.dtype, np.integer) or not np.issubdtype(idx.dtype, np.integer):
        raise ValueError("tile map: kv_tile_ptr and kv_tile_idx must be 1-D integer arrays")
    if ptr.size != n_q + 1:
        raise ValueError(f"tile map: kv_tile_ptr has {ptr.size} entries, want n_q_tiles + 1 = {n_q + 1}")
    if ptr[0] != 0 or ptr[-1] != idx.size:
        raise ValueError(f"tile map: kv_tile_ptr must run from 0 to nnz = {idx.size} (got {ptr[0]} .. {ptr[-1]})")
    counts = np.diff(ptr.astype(np.int64))
    if (counts <= 0).any():
        raise ValueError(f"tile map: query tile {int(np.argmax(counts <= 0))} has no key tiles (rows must be non-empty)")
    if idx.size and (idx.min() < 0 or idx.max() >= n_kv):
        raise ValueError(f"tile map: key tile indices must lie in [0, {n_kv})")
    step = np.diff(idx.astype(np.int64))
    row_start = np.zeros(idx.size, dtype=bool)
    row_start[ptr[:-1]] = True
    if (step <= 0)[~row_start[1:]].any():
        raise ValueError("tile map: every row's key tiles must be strictly ascending")


class TileMap:
    """A validated block-sparse self-attention map on one device: for query tile q (rows [128 q, 128 q + 128)) the key tiles
    kv_tile_idx[kv_tile_ptr[q] : kv_tile_ptr[q + 1]] (keys [128 k, 128 k + 128)), int32.  One map serves every (batch,
    head).  device=None keeps the validated host arrays only."""

    def __init__(self, kv_tile_ptr, kv_tile_idx, q_len, kv_len, device=None, checked=False):
        import numpy as np
        ptr = np.asarray(kv_tile_ptr.cpu() if isinstance(kv_tile_ptr, torch.Tensor) else kv_tile_ptr)
        idx = np.asarray(kv_tile_idx.cpu() if isinstance(kv_tile_idx, torch.Tensor) else kv_tile_idx)
        if not checked:
            check_tile_map(ptr, idx, q_len, kv_len)
        self.q_len, self.kv_len = int(q_len), int(kv_len)
        self.n_q_tiles, self.n_kv_tiles, self.nnz = ptr.size - 1, -(-self.kv_len // ATT_TILE), int(idx.size)
        self.density = self.nnz / float(self.n_q_tiles * self.n_kv_tiles)
        self.ptr = self.idx = None
        if device is not None:
            self.ptr = torch.from_numpy(ptr.astype(np.int32)).to(device)
            self.idx = torch.from_numpy(idx.astype(np.int32)).to(device)

    def _check_for(self, L, device):
        if self.q_len != L or self.kv_len != L:
            raise ValueError(f"tile map built for q_len={self.q_len}, kv_len={self.kv_len}; this launch has L={L}")
        if self.ptr is None or self.ptr.device != device:
            raise ValueError(f"tile map lives on {None if self.ptr is None else self.ptr.device}, the operands on {device}")


def _tile_map(tiles, L):
    """A TileMap, or a (kv_tile_ptr, kv_tile_idx) pair validated and uploaded here (once per call)."""
    if isinstance(tiles, TileMap):
        return tiles
    ptr, idx = tiles
    host = [t.cpu() if isinstance(t, torch.Tensor) else t for t in (ptr, idx)]
    check_tile_map(*host, L, L)  # before anything touches a device
    dev = ptr.device if isinstance(ptr, torch.Tensor) and ptr.is_cuda else torch.device("cuda", torch.cuda.current_device())
    return TileMap(*host, L, L, device=dev, checked=True)


def attention_sparse(q, k, v, out, B, H, L, tiles, q_batch_rows=None, kv_batch_rows=None, scale=None, accumulate=False):
    """Block-sparse bf16 self-attention (q_len == kv_len == L): as attention(), but query tile t attends only to the keys of
    the key tiles `tiles` lists for it (a TileMap, or a (kv_tile_ptr, kv_tile_idx) pair: see check_tile_map)."""
    m = _tile_map(tiles, L)
    for t in (q, k, v, out):
        _req(t)
        assert t.dim() == 2 and t.stride(1) == 1
    m._check_for(L, q.device)
    q_batch_rows = L if q_batch_rows is None else q_batch_rows
    kv_batch_rows = L if kv_batch_rows is None else kv_batch_rows
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and L > 1024:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    _lib.check(_lib.lib().scail_attention_sparse(_ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
                                                 out.stride(0), B, H, L, L, q_batch_rows, kv_batch_rows, q.shape[0],
                                                 k.shape[0], scale, 1 if accumulate else 0, _ptr(m.ptr), _ptr(m.idx), m.nnz,
                                                 _stream()), "scail_attention_sparse")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()
    return out


def quant_vt_fp8(v, B, H, L, vt=None, scale=None, work=None):
    """V operand of attention_fp8: v bf16 [B*L, H*128] (2-D row-strided view) -> (vt e4m3 [B, H, 128, L_pad], scale fp32
    [B, H, 128]): Vt's rows are the channels over the keys in the e4m3 row format, zero past L, and inside every 16-key group
    logical column k holds key 2*((k%16)//4) + k%2 + 8*((k%4)//2) (attention_fp8's P fragment order).  work: int32 [B, H*128] workspace (allocated when None)."""
    _req(v)
    assert v.dim() == 2 and v.stride(1) == 1 and v.shape == (B * L, H * 128)
    Lp = fp8_pad(L)
    if vt is None:
        vt = torch.empty(B, H, 128, Lp, device=v.device, dtype=FP8)
    if scale is None:
        scale = torch.empty(B, H, 128, device=v.device, dtype=torch.float32)
    if work is None:
        work = torch.empty(B, H * 128, device=v.device, dtype=torch.int32)
    _req(vt, FP8), _req(scale, torch.float32), _req(work, torch.int32)
    assert vt.is_contiguous() and vt.shape == (B, H, 128, Lp) and scale.is_contiguous() and scale.shape == (B, H, 128)
    assert work.is_contiguous() and work.numel() >= B * H * 128
    _lib.check(_lib.lib().scail_quant_vt_fp8(_ptr(v), v.stride(0), _ptr(vt), _ptr(scale), _ptr(work), B, H, 128, L, Lp,
                                             _stream()), "scail_quant_vt_fp8")
    _count(2)
    return vt, scale


def attention_fp8(q8, q_scale, k8, k_scale, vt, v_scale, out, B, H, L, scale=None, tiles=None):
    """FP8 self-attention (q_len == kv_len == L): q8/k8 e4m3 [B*L, H*128] (2-D row-strided) with scales [B, H, L_pad] as
    rmsnorm_rope(out_fp8=...) writes them, (vt, v_scale) from quant_vt_fp8; out bf16 [B*L, H*128] merged heads.
    tiles (attention_fp8_sparse): a block-sparse map as for attention_sparse."""
    m = _tile_map(tiles, L) if tiles is not None else None
    for t in (q8, k8):
        _req(t, FP8)
        assert t.dim() == 2 and t.stride(1) == 1 and t.shape == (B * L, H * 128)
    Lp = fp8_pad(L)
    for s in (q_scale, k_scale):
        _req(s, torch.float32)
        assert s.is_contiguous() and s.shape == (B, H, Lp)
    _req(vt, FP8), _req(v_scale, torch.float32), _req(out)
    assert vt.is_contiguous() and vt.shape == (B, H, 128, Lp) and v_scale.is_contiguous() and v_scale.shape == (B, H, 128)
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (B * L, H * 128)
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and L > 1024:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    if m is None:
        _lib.check(_lib.lib().scail_attention_fp8(_ptr(q8), q8.stride(0), _ptr(q_scale), _ptr(k8), k8.stride(0),
                                                  _ptr(k_scale), _ptr(vt), _ptr(v_scale), _ptr(out), out.stride(0), B, H, 128, L,
                                                  Lp, scale, _stream()), "scail_attention_fp8")
    else:
        m._check_for(L, q8.device)
        _lib.check(_lib.lib().scail_attention_fp8_sparse(_ptr(q8), q8.stride(0), _ptr(q_scale), _ptr(k8), k8.stride(0),
                                                         _ptr(k_scale), _ptr(vt), _ptr(v_scale), _ptr(out), out.stride(0), B, H,
                                                         128, L, Lp, scale, _ptr(m.ptr), _ptr(m.idx), m.nnz, _stream()),
                   "scail_attention_fp8_sparse")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()
    return out


def attention_fp8_sparse(q8, q_scale, k8, k_scale, vt, v_scale, out, B, H, L, tiles, scale=None):
    """Block-sparse FP8 self-attention: attention_fp8 over the key tiles `tiles` lists for each query tile (see
    attention_sparse)."""
    return attention_fp8(q8, q_scale, k8, k_scale, vt, v_scale, out, B, H, L, scale=scale, tiles=tiles)


def _bh_maps(ptr, idx, B, H, L, device):
    """(ptr_stride, idx_stride) of per-(batch, head) maps: int32 ptr [B, H, >= n + 1] and idx [B, H, >= n * n], contiguous."""
    n = -(-int(L) // ATT_TILE)
    for t, want, what in ((ptr, n + 1, "kv_tile_ptr"), (idx, n * n, "kv_tile_idx")):
        _req(t, torch.int32)
        if t.dim() != 3 or tuple(t.shape[:2]) != (B, H) or t.shape[2] < want or not t.is_contiguous():
            raise ValueError(f"per-(batch, head) {what} must be a contiguous int32 [B={B}, H={H}, >= {want}], got "
                             f"{tuple(t.shape)}")
        if t.device != device:
            raise ValueError(f"{what} lives on {t.device}, the operands on {device}")
    return ptr.shape[2], idx.shape[2]


def attention_sparse_bh(q, k, v, out, B, H, L, ptr, idx, q_batch_rows=None, kv_batch_rows=None, scale=None):
    """Block-sparse bf16 self-attention with one map per (batch, head): (b, h) attends as attention_sparse under the CSR map
    ptr[b, h] (int32 [B, H, >= n + 1], n = ceil(L / 128)) and idx[b, h] (int32 [B, H, >= n * n]).  The maps' contents are
    not read on the host (select_tiles builds them on the device)."""
    for t in (q, k, v, out):
        _req(t)
        assert t.dim() == 2 and t.stride(1) == 1
    ps, ids = _bh_maps(ptr, idx, B, H, L, q.device)
    q_batch_rows = L if q_batch_rows is None else q_batch_rows
    kv_batch_rows = L if kv_batch_rows is None else kv_batch_rows
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and L > 1024:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    _lib.check(_lib.lib().scail_attention_sparse_bh(_ptr(q), q.stride(0), _ptr(k), k.stride(0), _ptr(v), v.stride(0), _ptr(out),
                                                    out.stride(0), B, H, L, q_batch_rows, kv_batch_rows, q.shape[0], k.shape[0],
                                                    scale, _ptr(ptr), ps, _ptr(idx), ids, _stream()), "scail_attention_sparse_bh")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()
    return out


def attention_fp8_sparse_bh(q8, q_scale, k8, k_scale, vt, v_scale, out, B, H, L, ptr, idx, scale=None):
    """FP8 self-attention (operands as attention_fp8) with one block-sparse map per (batch, head), as attention_sparse_bh."""
    for t in (q8, k8):
        _req(t, FP8)
        assert t.dim() == 2 and t.stride(1) == 1 and t.shape == (B * L, H * 128)
    Lp = fp8_pad(L)
    for s in (q_scale, k_scale):
        _req(s, torch.float32)
        assert s.is_contiguous() and s.shape == (B, H, Lp)
    _req(vt, FP8), _req(v_scale, torch.float32), _req(out)
    assert vt.is_contiguous() and vt.shape == (B, H, 128, Lp) and v_scale.is_contiguous() and v_scale.shape == (B, H, 128)
    assert out.dim() == 2 and out.stride(1) == 1 and out.shape == (B * L, H * 128)
    ps, ids = _bh_maps(ptr, idx, B, H, L, q8.device)
    scale = 1.0 / math.sqrt(128) if scale is None else scale
    ev = None
    if ATTN_EVENTS is not None and L > 1024:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    _lib.check(_lib.lib().scail_attention_fp8_sparse_bh(_ptr(q8), q8.stride(0), _ptr(q_scale), _ptr(k8), k8.stride(0),
                                                        _ptr(k_scale), _ptr(vt), _ptr(v_scale), _ptr(out), out.stride(0), B, H, 128,
                                                        L, Lp, scale, _ptr(ptr), ps, _ptr(idx), ids, _stream()),
               "scail_attention_fp8_sparse_bh")
    if ev is not None:
        ev[1].record()
        ATTN_EVENTS.append(ev)
    _count()
    return out


def tile_pool(x, B, H, L, out=None, x_scale=None):
    """Tile means of one self-attention operand: x [B*L, H*128] (2-D row-strided view) bf16, or e4m3 or int8 with its
    per-token scales x_scale [B, H, L_pad] -> out fp32 [B, H, ceil(L/128), 128], the mean of each 128-row tile's valid rows
    (of x * scale for e4m3 and int8).  Bit-reproducible."""
    fp8 = x_scale is not None
    int8 = fp8 and x.dtype == INT8
    _req(x, (INT8 if int8 else FP8) if fp8 else torch.bfloat16)
    assert x.dim() == 2 and x.stride(1) == 1 and x.shape == (B * L, H * 128)
    n = -(-L // ATT_TILE)
    Lp = fp8_pad(L)
    if fp8:
        _req(x_scale, torch.float32)
        assert x_scale.is_contiguous() and x_scale.shape == (B, H, Lp)
    if out is None:
        out = torch.empty(B, H, n, 128, device=x.device, dtype=torch.float32)
    _req(out, torch.float32)
    assert out.is_contiguous() and out.shape == (B, H, n, 128)
    if int8:
        _lib.check(_lib.lib().scail_attention_tile_pool_int8(_ptr(x), x.stride(0), _ptr(x_scale), _ptr(out), B, H, L, Lp,
                                                             _stream()), "scail_attention_tile_pool_int8")
    else:
        _lib.check(_lib.lib().scail_attention_tile_pool(_ptr(x), x.stride(0), _ptr(x_scale), 1 if fp8 else 0, _ptr(out), B, H,
                                                        L, Lp if fp8 else 0, _stream()), "scail_attention_tile_pool")
    _count()
    return out


def select_scratch_len(B, H, L):
    """int32 entries of the scratch select_tiles needs: B H n (1 + ceil(n / 32)), n = ceil(L / 128)."""
    n = -(-int(L) // ATT_TILE)
    return B * H * n * (1 + -(-n // 32))


def select_tiles(qbar, kbar, B, H, L, n_ref, mass, max_tiles, ptr, idx, scratch):
    """Per-(batch, head) tile maps chosen on the device from the tile means qbar, kbar (fp32 [B, H, n, 128], tile_pool):
    query tile q lists its diagonal tile, every key tile holding one of the n_ref reference tokens, then the key tiles of
    largest estimated softmax mass e_k = n_k exp(s_k - max s), s_k = qbar_q . kbar_k / sqrt(128) (ties: lower index), until
    the listed mass reaches `mass` of the total or max_tiles (None: no cap) were taken that way.  Writes ptr, idx (int32
    [B, H, n + 1] and [B, H, n * n] or wider); scratch int32 [>= select_scratch_len(B, H, L)].  No host synchronisation."""
    n = -(-int(L) // ATT_TILE)
    for t in (qbar, kbar):
        _req(t, torch.float32)
        assert t.is_contiguous() and t.shape == (B, H, n, 128)
    ps, ids = _bh_maps(ptr, idx, B, H, L, qbar.device)
    _req(scratch, torch.int32)
    assert scratch.is_contiguous()
    _lib.check(_lib.lib().scail_attention_select_tiles(_ptr(qbar), _ptr(kbar), B, H, L, n_ref, float(mass),
                                                       -1 if max_tiles is None else int(max_tiles), _ptr(ptr), ps, _ptr(idx),
                                                       ids, _ptr(scratch), scratch.numel(), _stream()),
               "scail_attention_select_tiles")
    _count(2)
    return ptr, idx


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


def _u_scale(u_scale):
    """The CFG-Zero* scale operand of a scaled update: a one-element fp32 device tensor (scail_b200.guidance)."""
    _req(u_scale, torch.float32)
    assert u_scale.numel() == 1, tuple(u_scale.shape)
    return _ptr(u_scale)


def cfg_euler_(x, v, scale, dsigma, u_scale=None):
    """x (fp32, [1,...]) += dsigma * (v[0] + scale * (v[1] - v[0])); v bf16 [2, ...].
    With u_scale (fp32 [1] on the device, CFG-Zero*'s s), another kernel, per element in this order with each product and
    sum rounded on its own: u' = s*v[0]; g = u' + scale*(v[1] - u'); x = x + dsigma*g (x.numel() % 4 == 0).  Returns x."""
    _req(x, torch.float32), _req(v)
    assert x.is_contiguous() and v.is_contiguous() and v.numel() == 2 * x.numel()
    if u_scale is None:
        _lib.check(_lib.lib().scail_cfg_euler(_ptr(x), _ptr(v), x.numel(), float(scale), float(dsigma), _stream()),
                   "scail_cfg_euler")
    else:
        _lib.check(_lib.lib().scail_cfg_euler_scaled(_ptr(x), _ptr(v), x.numel(), float(scale), float(dsigma),
                                                     _u_scale(u_scale), _stream()), "scail_cfg_euler_scaled")
    _count()
    return x


def unipc_step_(x, x_last, v, slots, write_slot, scale, sigma, coef, correct, u_scale=None):
    """One fused UniPC step (scail_b200.unipc), in place: g = v[0] + scale*(v[1] - v[0]); m = x - sigma*g; y = a_x*x_last +
    a_k*slots[k] (slot order) + a_m*m if `correct`, else y = x; x = b_y*y + b_k*slots[k] + b_m*m; x_last = y;
    slots[write_slot] = m.  Each product and sum rounded on its own; slots with zero coefficients are not read.
    x, x_last fp32 (same shape, contiguous), v bf16 [2, ...], slots fp32 [n_slots, x.numel()]; coef: 10 floats
    (a_x, a_0, a_1, a_2, a_m, b_y, b_0, b_1, b_2, b_m), passed by value.  With u_scale (fp32 [1] on the device, CFG-Zero*'s
    s), u = s*v[0] (one rounded product) comes first and every later instruction is the same: s = 1 gives the unscaled
    step bit for bit.  Returns x."""
    _req(x, torch.float32), _req(x_last, torch.float32), _req(v), _req(slots, torch.float32)
    assert x.is_contiguous() and x_last.is_contiguous() and x_last.shape == x.shape
    assert v.is_contiguous() and v.numel() == 2 * x.numel()
    assert slots.dim() == 2 and slots.is_contiguous() and slots.shape[1] == x.numel(), tuple(slots.shape)
    assert len(coef) == 10
    c = (ctypes.c_float * 10)(*coef)
    args = (_ptr(x), _ptr(x_last), _ptr(v), _ptr(slots), slots.stride(0), slots.shape[0], int(write_slot), x.numel(),
            float(scale), float(sigma), int(bool(correct)), ctypes.addressof(c))
    if u_scale is None:
        _lib.check(_lib.lib().scail_unipc_step(*args, _stream()), "scail_unipc_step")
    else:
        _lib.check(_lib.lib().scail_unipc_step_scaled(*args, _u_scale(u_scale), _stream()), "scail_unipc_step_scaled")
    _count()
    return x


# ---------------------------------------------------------------- CFG cache (scail_b200.cfg_cache)
def cfg_cache_delta(v, d_ref, d_new, partials, out):
    """d_new = f32(v[1]) - f32(v[0]) (fp32, one subtraction rounded once) and out (fp64 [4]) = (sum |d_new - d_ref|,
    sum |d_ref|, their ratio (+inf for a zero denominator), 0); v bf16 [2, ...] (the CFG pair as cfg_euler_ reads it),
    d_ref, d_new fp32 with v[0]'s element count, partials fp32 [>= STEP_CACHE_PARTIALS] scratch.  Bit-reproducible.
    Returns out."""
    _req(v), _req(d_ref, torch.float32), _req(d_new, torch.float32), _req(partials, torch.float32), _req(out, torch.float64)
    n = d_new.numel()
    assert v.is_contiguous() and v.numel() == 2 * n and d_ref.is_contiguous() and d_new.is_contiguous() and d_ref.numel() == n
    assert partials.is_contiguous() and out.is_contiguous() and out.numel() >= 4
    _lib.check(_lib.lib().scail_cfg_cache_delta(_ptr(v), _ptr(d_ref), _ptr(d_new), _ptr(partials), partials.numel(), _ptr(out),
                                                n, _stream()), "scail_cfg_cache_delta")
    _count(2)
    return out


def cfg_euler_cached_(x, c, delta, scale, dsigma, u_scale=None):
    """The conditional-only Euler step, in place on x (fp32): u = c - delta; g = u + scale*(c - u); x = x + dsigma*g, each
    product and sum rounded on its own.  c bf16 (the conditional output alone), delta fp32, both with x's element count.
    With u_scale (fp32 [1] on the device, CFG-Zero*'s s), u = s*u (one rounded product) right after u is formed; s = 1
    gives the unscaled step bit for bit."""
    _req(x, torch.float32), _req(c), _req(delta, torch.float32)
    assert x.is_contiguous() and c.is_contiguous() and delta.is_contiguous() and c.numel() == x.numel() == delta.numel()
    args = (_ptr(x), _ptr(c), _ptr(delta), x.numel(), float(scale), float(dsigma))
    if u_scale is None:
        _lib.check(_lib.lib().scail_cfg_euler_cached(*args, _stream()), "scail_cfg_euler_cached")
    else:
        _lib.check(_lib.lib().scail_cfg_euler_cached_scaled(*args, _u_scale(u_scale), _stream()),
                   "scail_cfg_euler_cached_scaled")
    _count()
    return x


def unipc_step_cached_(x, x_last, c, delta, slots, write_slot, scale, sigma, coef, correct, u_scale=None):
    """unipc_step_ with u = f32(c) - delta in place of the pair's u: c bf16 (the conditional output alone), delta fp32, both
    with x's element count; everything else (u_scale included) as unipc_step_.  Returns x."""
    _req(x, torch.float32), _req(x_last, torch.float32), _req(c), _req(delta, torch.float32), _req(slots, torch.float32)
    assert x.is_contiguous() and x_last.is_contiguous() and x_last.shape == x.shape
    assert c.is_contiguous() and delta.is_contiguous() and c.numel() == x.numel() == delta.numel()
    assert slots.dim() == 2 and slots.is_contiguous() and slots.shape[1] == x.numel(), tuple(slots.shape)
    assert len(coef) == 10
    k = (ctypes.c_float * 10)(*coef)
    args = (_ptr(x), _ptr(x_last), _ptr(c), _ptr(delta), _ptr(slots), slots.stride(0), slots.shape[0], int(write_slot),
            x.numel(), float(scale), float(sigma), int(bool(correct)), ctypes.addressof(k))
    if u_scale is None:
        _lib.check(_lib.lib().scail_unipc_step_cached(*args, _stream()), "scail_unipc_step_cached")
    else:
        _lib.check(_lib.lib().scail_unipc_step_cached_scaled(*args, _u_scale(u_scale), _stream()),
                   "scail_unipc_step_cached_scaled")
    _count()
    return x


def _delta_forecast(slots, coef, n):
    """The delta slots (fp32 [n_slots, n], contiguous) and their forecast coefficients (n_slots floats, padded with zeros to
    the kernels' 3) -> (slot stride, n_slots, the ctypes float[3])."""
    assert slots.dim() >= 2 and slots.is_contiguous() and slots[0].numel() == n, tuple(slots.shape)
    assert len(coef) == slots.shape[0]
    return slots.stride(0), slots.shape[0], (ctypes.c_float * 3)(*coef, *[0.0] * (3 - len(coef)))


def cfg_cache_delta_forecast(v, slots, write_slot, coef, partials, out):
    """cfg_cache_delta against a forecast: slots[write_slot] = f32(v[1]) - f32(v[0]) and out = (sum |d_new - t|, sum |t|,
    their ratio, 0) with t = c0*S0, then t + c1*S1, then t + c2*S2 (each product and sum rounded on its own; a slot whose
    coefficient is 0 is not read).  slots fp32 [n_slots, ...] with v[0]'s element count per slot, coef n_slots fp32 values.
    Bit-reproducible.  Returns out."""
    _req(v), _req(slots, torch.float32), _req(partials, torch.float32), _req(out, torch.float64)
    n = v.numel() // 2
    assert v.is_contiguous() and partials.is_contiguous() and out.is_contiguous() and out.numel() >= 4
    stride, n_slots, k = _delta_forecast(slots, coef, n)
    _lib.check(_lib.lib().scail_cfg_cache_delta_forecast(_ptr(v), _ptr(slots), stride, n_slots, int(write_slot),
                                                         ctypes.addressof(k), _ptr(partials), partials.numel(), _ptr(out), n,
                                                         _stream()), "scail_cfg_cache_delta_forecast")
    _count(2)
    return out


def cfg_euler_cached_forecast_(x, c, slots, coef, scale, dsigma, u_scale=None):
    """cfg_euler_cached_ (u_scale included) with delta = the forecast of the delta slots (as cfg_cache_delta_forecast forms
    it)."""
    _req(x, torch.float32), _req(c), _req(slots, torch.float32)
    assert x.is_contiguous() and c.is_contiguous() and c.numel() == x.numel()
    stride, n_slots, k = _delta_forecast(slots, coef, x.numel())
    args = (_ptr(x), _ptr(c), _ptr(slots), stride, n_slots, ctypes.addressof(k), x.numel(), float(scale), float(dsigma))
    if u_scale is None:
        _lib.check(_lib.lib().scail_cfg_euler_cached_forecast(*args, _stream()), "scail_cfg_euler_cached_forecast")
    else:
        _lib.check(_lib.lib().scail_cfg_euler_cached_forecast_scaled(*args, _u_scale(u_scale), _stream()),
                   "scail_cfg_euler_cached_forecast_scaled")
    _count()
    return x


def unipc_step_cached_forecast_(x, x_last, c, dslots, dcoef, slots, write_slot, scale, sigma, coef, correct, u_scale=None):
    """unipc_step_cached_ with delta = the forecast of the delta slots dslots with the coefficients dcoef (as
    cfg_cache_delta_forecast forms it); everything else (u_scale included) as unipc_step_.  Returns x."""
    _req(x, torch.float32), _req(x_last, torch.float32), _req(c), _req(dslots, torch.float32), _req(slots, torch.float32)
    assert x.is_contiguous() and x_last.is_contiguous() and x_last.shape == x.shape
    assert c.is_contiguous() and c.numel() == x.numel()
    assert slots.dim() == 2 and slots.is_contiguous() and slots.shape[1] == x.numel(), tuple(slots.shape)
    assert len(coef) == 10
    dstride, n_d, dk = _delta_forecast(dslots, dcoef, x.numel())
    k = (ctypes.c_float * 10)(*coef)
    args = (_ptr(x), _ptr(x_last), _ptr(c), _ptr(dslots), dstride, n_d, ctypes.addressof(dk), _ptr(slots), slots.stride(0),
            slots.shape[0], int(write_slot), x.numel(), float(scale), float(sigma), int(bool(correct)), ctypes.addressof(k))
    if u_scale is None:
        _lib.check(_lib.lib().scail_unipc_step_cached_forecast(*args, _stream()), "scail_unipc_step_cached_forecast")
    else:
        _lib.check(_lib.lib().scail_unipc_step_cached_forecast_scaled(*args, _u_scale(u_scale), _stream()),
                   "scail_unipc_step_cached_forecast_scaled")
    _count()
    return x


# ---------------------------------------------------------------- CFG-Zero* guidance (scail_b200.guidance)
def cfg_zero_scale(v, partials, out, u_scale, delta=None, forecast=None):
    """CFG-Zero*'s optimised scale s = <c, u> / (|u|^2 + 1e-8) over all elements, on the device: u_scale (fp32 [1]) = s,
    computed in fp64 and rounded once, and out (fp64 [4]) = (<c, u>, |u|^2, 0, 0).  u and c come from
      v alone:        v bf16 [2, ...], the CFG pair (u, c) as cfg_euler_ reads it;
      delta:          v = c alone (bf16 [1, ...]) and u = f32(c) - delta (fp32), as cfg_euler_cached_ forms it;
      forecast:       v = c alone and u = f32(c) - delta_hat with forecast = (slots, coefficients), as
                      cfg_euler_cached_forecast_ forms it.
    Pass 1 adds f32(c)*u and u*u per CTA in fp32 (each product and sum rounded on its own) over a partition fixed by the
    size; pass 2 adds the CTA sums in fp64 in a fixed order.  Bit-reproducible; partials fp32 [>= STEP_CACHE_PARTIALS]
    scratch.  Returns u_scale."""
    if delta is not None and forecast is not None:
        raise ValueError("cfg_zero_scale: pass delta or forecast, not both")
    _req(v), _req(partials, torch.float32), _req(out, torch.float64)
    assert v.is_contiguous() and partials.is_contiguous() and out.is_contiguous() and out.numel() >= 4
    up = _u_scale(u_scale)
    dptr, dstride, n_d, dk = None, 0, 0, None
    if forecast is not None:
        n = v.numel()
        _req(forecast[0], torch.float32)
        dstride, n_d, dk = _delta_forecast(forecast[0], forecast[1], n)
        form, dptr = 2, _ptr(forecast[0])
    elif delta is not None:
        n = v.numel()
        _req(delta, torch.float32)
        assert delta.is_contiguous() and delta.numel() == n
        form, dptr = 1, _ptr(delta)
    else:
        n = v.numel() // 2
        form = 0
    _lib.check(_lib.lib().scail_cfg_zero_scale(form, _ptr(v), dptr, dstride, n_d, None if dk is None else ctypes.addressof(dk),
                                               _ptr(partials), partials.numel(), _ptr(out), up, n, _stream()),
               "scail_cfg_zero_scale")
    _count(2)
    return u_scale


# ---------------------------------------------------------------- APG guidance (scail_b200.guidance)
APG_MAX_CTAS_PER_FRAME = 32  # pass 1 of apg_reduce runs at most this many CTAs per latent frame


def apg_partials_len(frames):
    """fp32 partials apg_reduce needs for a latent of `frames` frames: 3 sums per CTA."""
    return 3 * frames * APG_MAX_CTAS_PER_FRAME


def _apg_operands(x, v, delta, forecast):
    """(form, delta pointer, delta stride, n_dslots, ctypes coefficients or None, frames) of an APG launch on x [1, T, ...]
    fp32 with u and c as cfg_zero_scale takes them: v the pair, or c alone with delta or forecast = (slots, coefficients)."""
    if delta is not None and forecast is not None:
        raise ValueError("apg: pass delta or forecast, not both")
    _req(x, torch.float32), _req(v)
    assert x.is_contiguous() and v.is_contiguous() and x.dim() >= 2 and x.shape[0] == 1, tuple(x.shape)
    n = x.numel()
    if forecast is not None:
        _req(forecast[0], torch.float32)
        assert v.numel() == n
        stride, n_d, dk = _delta_forecast(forecast[0], forecast[1], n)
        return 2, _ptr(forecast[0]), stride, n_d, dk, x.shape[1]
    if delta is not None:
        _req(delta, torch.float32)
        assert v.numel() == n and delta.is_contiguous() and delta.numel() == n
        return 1, _ptr(delta), 0, 0, None, x.shape[1]
    assert v.numel() == 2 * n
    return 0, None, 0, 0, None, x.shape[1]


def apg_reduce(x, v, sigma, partials, avg=None, momentum=0.0, delta=None, forecast=None):
    """APG pass 1 on the latent x (fp32 [1, T, ...], one frame per x[0, t]) at the step's sigma: D_c = x - sigma*c,
    diff = D_c - (x - sigma*u), each product and sum rounded on its own; u and c from the pair v, or from c = v alone with
    delta or forecast, as cfg_zero_scale forms them.  With avg (fp32, x's shape) avg = diff + momentum*avg in place, and
    diff = avg.  fp32 partial sums of diff*diff, diff*D_c and D_c*D_c per (frame, CTA) over a partition fixed by the shape
    -> partials (fp32, at least apg_partials_len(T)).  Bit-reproducible.  Returns partials."""
    form, dptr, dstride, n_d, dk, frames = _apg_operands(x, v, delta, forecast)
    _req(partials, torch.float32)
    assert partials.is_contiguous()
    if avg is not None:
        _req(avg, torch.float32)
        assert avg.is_contiguous() and avg.numel() == x.numel()
    _lib.check(_lib.lib().scail_apg_reduce(form, _ptr(x), _ptr(v), dptr, dstride, n_d,
                                           None if dk is None else ctypes.addressof(dk), _ptr(avg), float(sigma),
                                           float(momentum), _ptr(partials), partials.numel(), frames, x.numel(), _stream()),
               "scail_apg_reduce")
    _count()
    return partials


def apg_finish(partials, sums, factors, norm_threshold, frames, n):
    """APG pass 2: per frame, the partials of apg_reduce on a latent of n elements in `frames` frames added in fp64 in a fixed
    order -> sums (fp64 [frames, 4]) = (|diff|^2, <diff, D_c>, |D_c|^2, 0) and factors (fp32 [frames, 2]) = (f, p), computed
    in fp64 and rounded once: f = r / |diff| if r = norm_threshold > 0 and |diff| > r, else 1; p = f <diff, D_c> / |D_c|^2,
    0 for |D_c| = 0.  Returns factors."""
    _req(partials, torch.float32), _req(sums, torch.float64), _req(factors, torch.float32)
    assert sums.is_contiguous() and sums.numel() >= 4 * frames and factors.is_contiguous() and factors.numel() >= 2 * frames
    _lib.check(_lib.lib().scail_apg_finish(_ptr(partials), partials.numel(), _ptr(sums), _ptr(factors), float(norm_threshold),
                                           int(frames), int(n), _stream()), "scail_apg_finish")
    _count()
    return factors


def apg_update_(x, v, factors, scale, eta, sigma, next_sigma=None, out=None, avg=None, delta=None, forecast=None):
    """The APG update of x (fp32 [1, T, ...]) with the per-frame factors (f, p) of apg_finish: D_c and diff as apg_reduce
    forms them (diff = avg, the average apg_reduce wrote, when avg is given); par = p*D_c; orth = f*diff - par; D_g = D_c +
    (scale - 1)*(orth + eta*par), each product and sum rounded on its own.  With out (fp32, x's shape) D_g -> out and x is
    left as it is; else the Euler step x = x + k*(x - D_g) in place, k = (next_sigma - sigma) / sigma (fp64, rounded once).
    scale - 1 is likewise formed in fp64 and rounded once.  Returns out, or x."""
    form, dptr, dstride, n_d, dk, frames = _apg_operands(x, v, delta, forecast)
    _req(factors, torch.float32)
    assert factors.is_contiguous() and factors.numel() >= 2 * frames
    if avg is not None:
        _req(avg, torch.float32)
        assert avg.is_contiguous() and avg.numel() == x.numel()
    if out is not None:
        _req(out, torch.float32)
        assert out.is_contiguous() and out.numel() == x.numel()
        k = 0.0
    else:
        k = (float(next_sigma) - float(sigma)) / float(sigma)
    _lib.check(_lib.lib().scail_apg_update(form, _ptr(x), _ptr(v), dptr, dstride, n_d,
                                           None if dk is None else ctypes.addressof(dk), _ptr(avg), _ptr(factors), _ptr(out),
                                           float(sigma), float(scale) - 1.0, float(eta), k, frames, x.numel(), _stream()),
               "scail_apg_update")
    _count()
    return x if out is None else out


def unipc_step_dpred_(x, x_last, m, slots, write_slot, coef, correct):
    """unipc_step_ with the data prediction m (fp32, x's shape: APG's D_g) read in place of x - sigma*g; every later
    instruction is the same.  Returns x."""
    _req(x, torch.float32), _req(x_last, torch.float32), _req(m, torch.float32), _req(slots, torch.float32)
    assert x.is_contiguous() and x_last.is_contiguous() and x_last.shape == x.shape
    assert m.is_contiguous() and m.numel() == x.numel()
    assert slots.dim() == 2 and slots.is_contiguous() and slots.shape[1] == x.numel(), tuple(slots.shape)
    assert len(coef) == 10
    c = (ctypes.c_float * 10)(*coef)
    _lib.check(_lib.lib().scail_unipc_step_dpred(_ptr(x), _ptr(x_last), _ptr(m), _ptr(slots), slots.stride(0), slots.shape[0],
                                                 int(write_slot), x.numel(), int(bool(correct)), ctypes.addressof(c),
                                                 _stream()), "scail_unipc_step_dpred")
    _count()
    return x


# ---------------------------------------------------------------- first-block residual cache (scail_b200.step_cache)
STEP_CACHE_PARTIALS = 2048  # fp32 partial sums of step_cache_indicator: 2 per CTA, at most 1024 CTAs


def _noise_rows(h, t, n_ref, dtype):
    """(B, N, d, n_seq) of a contiguous bf16 h [B, N, d] and its contiguous noise-row tensor t [B, n_seq, d] of `dtype`."""
    _req(h), _req(t, dtype)
    assert h.dim() == 3 and t.dim() == 3 and h.is_contiguous() and t.is_contiguous()
    B, N, d = h.shape
    n_seq = t.shape[1]
    assert t.shape == (B, n_seq, d) and 0 <= n_ref and n_ref + n_seq <= N, (tuple(h.shape), tuple(t.shape), n_ref)
    return B, N, d, n_seq


def step_cache_indicator(h0, h1, r_ref, r_new, h1c, n_ref, partials, out):
    """r_new = bf16_rn(f32(h1) - f32(h0)), h1c = h1[:, n_ref:n_ref + n_seq], and out (fp64 [4]) = (sum |r_new - r_ref|,
    sum |r_ref|, their ratio (+inf for a zero denominator), 0) over all B*N*d elements; h0, h1, r_ref, r_new bf16 [B, N, d],
    h1c bf16 [B, n_seq, d], partials fp32 [>= STEP_CACHE_PARTIALS] scratch.  Bit-reproducible.  Returns out."""
    B, N, d, n_seq = _noise_rows(h1, h1c, n_ref, torch.bfloat16)
    for t in (h0, r_ref, r_new):
        _req(t)
        assert t.shape == h1.shape and t.is_contiguous()
    _req(partials, torch.float32), _req(out, torch.float64)
    assert partials.is_contiguous() and out.is_contiguous() and out.numel() >= 4
    _lib.check(_lib.lib().scail_step_cache_indicator(_ptr(h0), _ptr(h1), _ptr(r_ref), _ptr(r_new), _ptr(h1c), _ptr(partials),
                                                     partials.numel(), _ptr(out), B, N, d, n_ref, n_seq, _stream()),
               "scail_step_cache_indicator")
    _count(2)
    return out


def step_cache_update(h, h1c, R, n_ref):
    """R (fp32 [B, n_seq, d]) = f32(h[:, n_ref:n_ref + n_seq]) - f32(h1c); h bf16 [B, N, d], h1c bf16 [B, n_seq, d]."""
    B, N, d, n_seq = _noise_rows(h, R, n_ref, torch.float32)
    _req(h1c)
    assert h1c.shape == R.shape and h1c.is_contiguous()
    _lib.check(_lib.lib().scail_step_cache_update(_ptr(h), _ptr(h1c), _ptr(R), B, N, d, n_ref, n_seq, _stream()),
               "scail_step_cache_update")
    _count()
    return R


def step_cache_apply(h, R, n_ref):
    """In place: h[:, n_ref:n_ref + n_seq] = bf16_rn(f32(h[:, n_ref:n_ref + n_seq]) + R); h bf16 [B, N, d], R fp32
    [B, n_seq, d].  Returns h."""
    B, N, d, n_seq = _noise_rows(h, R, n_ref, torch.float32)
    _lib.check(_lib.lib().scail_step_cache_apply(_ptr(h), _ptr(R), B, N, d, n_ref, n_seq, _stream()), "scail_step_cache_apply")
    _count()
    return h


def _slots(h, R_slots, n_ref):
    """(B, N, d, n_seq, n_slots, slot_stride) of h bf16 [B, N, d] and its forecast slots R_slots fp32 [n_slots, B, n_seq, d]."""
    _req(R_slots, torch.float32)
    assert R_slots.dim() == 4 and R_slots.is_contiguous() and 1 <= R_slots.shape[0] <= 3, tuple(R_slots.shape)
    B, N, d, n_seq = _noise_rows(h, R_slots[0], n_ref, torch.float32)
    return B, N, d, n_seq, R_slots.shape[0], R_slots[0].numel()


def step_cache_update_slot(h, h1c, R_slots, slot, n_ref):
    """R_slots[slot] (fp32 [B, n_seq, d]) = f32(h[:, n_ref:n_ref + n_seq]) - f32(h1c), where slot is an int32 device tensor
    (read by the kernel when it runs; a slot outside [0, n_slots) writes nothing); R_slots fp32 [n_slots, B, n_seq, d]."""
    B, N, d, n_seq, n_slots, stride = _slots(h, R_slots, n_ref)
    _req(h1c), _req(slot, torch.int32)
    assert h1c.shape == (B, n_seq, d) and h1c.is_contiguous() and slot.numel() >= 1
    _lib.check(_lib.lib().scail_step_cache_update_slot(_ptr(h), _ptr(h1c), _ptr(R_slots), stride, n_slots, _ptr(slot), B, N, d,
                                                       n_ref, n_seq, _stream()), "scail_step_cache_update_slot")
    _count()
    return R_slots


def step_cache_apply_forecast(h, R_slots, coef, n_ref):
    """In place on h[:, n_ref:n_ref + n_seq]: t = c0*R0, t = t + c1*R1, t = t + c2*R2 (each product and sum rounded on its own;
    slots with c == 0 are not read), h = bf16_rn(f32(h) + t).  coef: fp32 device tensor of n_slots coefficients, read by the
    kernel when it runs; R_slots fp32 [n_slots, B, n_seq, d].  Returns h."""
    B, N, d, n_seq, n_slots, stride = _slots(h, R_slots, n_ref)
    _req(coef, torch.float32)
    assert coef.numel() >= n_slots and coef.is_contiguous()
    _lib.check(_lib.lib().scail_step_cache_apply_forecast(_ptr(h), _ptr(R_slots), stride, n_slots, _ptr(coef), B, N, d, n_ref,
                                                          n_seq, _stream()), "scail_step_cache_apply_forecast")
    _count()
    return h


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
