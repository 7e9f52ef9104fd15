"""GPU parity tests of the individual sm_90a kernels, called through the C ABI (scail_b200.ops ->
ctypes -> libscail_b200.so) and compared with the oracle restatement (oracle/dit_oracle.py, fp32) on the
same seeded inputs.  Tolerances: bf16 outputs -> rel-L2 vs the fp32 oracle <= 4e-3 (one bf16 ulp is
2^-8 = 3.9e-3; SURVEY §0 F10), stated per test."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-12))


def rnd(*shape, scale=1.0, seed=0, dev="cuda"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(dev)


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 256), (384, 768, 256), (300, 64, 80), (2, 1536, 256),
                                   (1000, 1280, 1280), (27904 // 8, 5120, 5120)])
def test_gemm_bias(M, N, K):
    from scail_b200 import ops
    a, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    out = ops.gemm(a, w, b)
    ref = a.float() @ w.float().t() + b.float()
    torch.cuda.synchronize()
    assert rel(out, ref) < 4e-3, rel(out, ref)


@pytest.mark.parametrize("epi", ["gelu", "silu", "gelu_erf", "gate_res", "res", "fp32"])
def test_gemm_epilogues(epi):
    from scail_b200 import ops
    import torch.nn.functional as F
    B, n, N, K = 2, 192, 512, 256
    M = B * n
    a, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    acc = a.float() @ w.float().t() + b.float()
    if epi == "gelu":
        out, ref = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GELU), F.gelu(acc, approximate="tanh")
    elif epi == "silu":
        out, ref = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_SILU), F.silu(acc)
    elif epi == "gelu_erf":
        out, ref = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GELU_ERF), F.gelu(acc)
    elif epi == "gate_res":
        mod = rnd(B, 6, N, seed=4)
        res = rnd(M, N, seed=5)
        out = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GATE_RES, gate=mod[:, 2], residual=res, rows_per_batch=n)
        ref = res.float() + mod[:, 2].float().repeat_interleave(n, 0) * acc
    elif epi == "res":
        res = rnd(M, N, seed=5)
        out, ref = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_RES, residual=res), res.float() + acc
    else:
        out, ref = ops.gemm(a, w, b, out_fp32=True), acc
        assert out.dtype == torch.float32
        assert rel(out, ref) < 1e-5
    torch.cuda.synchronize()
    assert rel(out, ref) < 4e-3, rel(out, ref)


def test_gemm_strided_views():
    """A and C as column slabs of wider matrices (how q-proj / QKV consumers address the fused buffers)."""
    from scail_b200 import ops
    M, N, K = 256, 256, 256
    big_a, w = rnd(M, 3 * K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    big_c = torch.zeros(M, 2 * N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(big_a[:, K:2 * K], w, None, out=big_c[:, N:])
    ref = big_a[:, K:2 * K].float() @ w.float().t()
    assert rel(big_c[:, N:], ref) < 4e-3
    assert float(big_c[:, :N].abs().max()) == 0.0


@pytest.mark.parametrize("D", [256, 1280, 5120])
def test_ln_modulate(D):
    from oracle import dit_oracle as O
    from scail_b200 import ops
    B, n = 2, 77
    x = rnd(B, n, D, seed=1)
    mod = rnd(B, 6, D, scale=0.5, seed=2)
    g, b = rnd(D, seed=3), rnd(D, seed=4)
    out = ops.ln_modulate(x, shift=mod[:, 0], scale=mod[:, 1])
    ref = O.modulate(O.layernorm(x.float()), mod[:, 0:1].float(), mod[:, 1:2].float())
    assert rel(out, ref) < 4e-3
    out = ops.ln_modulate(x, gamma=g, beta=b, eps=1e-5)
    assert rel(out, O.layernorm(x.float(), g.float(), b.float(), eps=1e-5)) < 4e-3
    out = ops.ln_modulate(x, shift=mod[:, 3], scale=mod[:, 4], rows_out=30, row_offset=11)
    ref = O.modulate(O.layernorm(x.float()[:, 11:41]), mod[:, 3:4].float(), mod[:, 4:5].float())
    assert out.shape == (B, 30, D) and rel(out, ref) < 4e-3


@pytest.mark.parametrize("D,heads", [(256, 2), (5120, 40)])
def test_rmsnorm_rope(D, heads):
    from oracle import dit_oracle as O
    from scail_b200 import ops
    B, t, h, w = 2, 2, 8, 8
    n_ref, n_seq, n_pose = O.segment_lengths(t, h, w)
    n = n_ref + n_seq + n_pose
    qkv = rnd(B * n, 3 * D, seed=1)
    wq, wk = rnd(D, seed=2) * 0.1 + 1, rnd(D, seed=3) * 0.1 + 1
    cos, sin = O.rope_tables(128, t, h // 2, w // 2, 21, 150, 150)
    cos, sin = cos.cuda(), sin.cuda()
    ref_q = O.rmsnorm(qkv[:, :D].float(), wq.float()).view(B, n, heads, 128)
    ref_k = O.rmsnorm(qkv[:, D:2 * D].float(), wk.float()).view(B, n, heads, 128)
    c, s = cos[None, :, None, :], sin[None, :, None, :]
    ref_q = ref_q * c + O.rotate_half(ref_q) * s
    ref_k = ref_k * c + O.rotate_half(ref_k) * s
    v_before = qkv[:, 2 * D:].clone()
    ops.rmsnorm_rope(qkv, n, D, [(0, wq), (D, wk)], cos, sin)
    assert rel(qkv[:, :D].view(B, n, heads, 128), ref_q) < 4e-3
    assert rel(qkv[:, D:2 * D].view(B, n, heads, 128), ref_k) < 4e-3
    assert torch.equal(qkv[:, 2 * D:], v_before)


@pytest.mark.parametrize("M,N,K,epi", [(2048, 2560, 512, 0), (2176, 2304, 640, 2), (4100, 1288, 256, 1), (256, 18944, 128, 3)])
def test_gemm_cta_pair_kernel(M, N, K, epi):
    """Shapes with more 128 x 256 output tiles (148 to 198) than the H100 has SMs, so the persistent CTAs each loop over
    more than one tile: ragged M / N edges (M = 4100, N = 1288), a gate that changes batch every 1024 rows, and the bias,
    GELU-tanh, gate+residual and residual epilogues, against an fp32 reference."""
    from scail_b200 import ops
    a, w, b = rnd(M, K, seed=1), rnd(N, K, seed=2) * 0.05, rnd(N, seed=3)
    ref = a.float() @ w.float().t() + b.float()
    kw = {}
    rpb = 1024
    if epi == 1:
        ref = torch.nn.functional.gelu(ref, approximate="tanh")
    if epi in (2, 3):
        res = rnd(M, N, seed=4)
        kw = dict(residual=res.clone())
        if epi == 2:
            gate = rnd((M + rpb - 1) // rpb, N, seed=5)
            kw.update(gate=gate, rows_per_batch=rpb)
            ref = ref * gate.float().repeat_interleave(rpb, 0)[:M]
        ref = ref + res.float()
    out = ops.gemm(a, w, b, epilogue=epi, **kw)
    torch.cuda.synchronize()
    assert rel(out, ref) < 4e-3, rel(out, ref)


@pytest.mark.parametrize("B,H,nq,nkv", [(1, 1, 256, 128), (1, 2, 256, 256), (2, 2, 384, 384), (1, 2, 300, 257),
                                        (2, 3, 512, 1000), (1, 1, 128, 4096), (1, 1, 128, 64), (1, 2, 256, 40),
                                        (1, 1, 256, 191), (2, 1, 130, 193), (1, 2, 256, 320)])
def test_attention(B, H, nq, nkv):
    from oracle import dit_oracle as O
    from scail_b200 import ops
    D = H * 128
    q, k, v = rnd(B * nq, D, seed=1), rnd(B * nkv, D, seed=2), rnd(B * nkv, D, seed=3)
    out = torch.zeros(B * nq, D, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, out, B, H, nq, nkv)
    torch.cuda.synchronize()
    hq = O.heads(q.float().view(B, nq, D), H)
    ref = O.merge_heads(O.sdpa(hq, O.heads(k.float().view(B, nkv, D), H), O.heads(v.float().view(B, nkv, D), H)))
    assert rel(out.view(B, nq, D), ref) < 6e-3, rel(out.view(B, nq, D), ref)


def test_attention_fused_qkv_layout_and_accumulate():
    """Q/K/V read as column slabs of the fused QKV matrix; second call accumulates (cross-attn text+CLIP sum)."""
    from oracle import dit_oracle as O
    from scail_b200 import ops
    B, H, n = 2, 2, 256
    D = H * 128
    qkv = rnd(B * n, 3 * D, seed=1)
    out = torch.zeros(B * n, D, device="cuda", dtype=torch.bfloat16)
    ops.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], out, B, H, n, n)
    f = qkv.float().view(B, n, 3 * D)
    ref = O.merge_heads(O.sdpa(O.heads(f[..., :D], H), O.heads(f[..., D:2 * D], H), O.heads(f[..., 2 * D:], H)))
    assert rel(out.view(B, n, D), ref) < 6e-3
    kv2 = rnd(B * 257, 2 * D, seed=5)
    ops.attention(qkv[:, :D], kv2[:, :D], kv2[:, D:], out, B, H, n, 257, accumulate=True)
    f2 = kv2.float().view(B, 257, 2 * D)
    ref2 = ref + O.merge_heads(O.sdpa(O.heads(f[..., :D], H), O.heads(f2[..., :D], H), O.heads(f2[..., D:], H)))
    assert rel(out.view(B, n, D), ref2) < 8e-3


@pytest.mark.parametrize("P,n_local,rank", [(4, 200, 1), (2, 384, 0), (4, 328, 3), (8, 100, 5)])
def test_attention_partial_and_merge(P, n_local, rank):
    """Context-parallel split: partial over the local key shard + partial over every other shard (two row ranges, not
    tile-aligned), merged with their softmax statistics, equals attention over all keys."""
    from oracle import dit_oracle as O
    from scail_b200 import ops
    B, H = 2, 2
    D = H * 128
    nkv = P * n_local
    q, k, v = rnd(B * n_local, D, seed=1), rnd(B * nkv, D, seed=2), rnd(B * nkv, D, seed=3)
    full = torch.zeros(B * n_local, D, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, full, B, H, n_local, nkv)
    oa = torch.empty(B * n_local, D, device="cuda", dtype=torch.float32)
    ob = torch.empty_like(oa)
    sa = torch.empty(B * n_local, H, 2, device="cuda", dtype=torch.float32)
    sb = torch.empty_like(sa)
    ops.attention_partial(q, k, v, oa, sa, B, H, n_local, [(rank * n_local, n_local)], kv_batch_rows=nkv)
    remote = [(o, l) for (o, l) in ((0, rank * n_local), ((rank + 1) * n_local, (P - 1 - rank) * n_local)) if l > 0]
    ops.attention_partial(q, k, v, ob, sb, B, H, n_local, remote, kv_batch_rows=nkv)
    out = torch.zeros_like(full)
    ops.attention_merge(oa, sa, ob, sb, out, H)
    torch.cuda.synchronize()
    ref = O.merge_heads(O.sdpa(O.heads(q.float().view(B, n_local, D), H), O.heads(k.float().view(B, nkv, D), H),
                               O.heads(v.float().view(B, nkv, D), H)))
    assert rel(out.view(B, n_local, D), ref) < 6e-3
    assert rel(out, full) < 3e-3  # vs the single pass: only rounding-order differences
    # the local partial alone is attention over the local shard
    kl = k.view(B, nkv, D)[:, rank * n_local:(rank + 1) * n_local].float()
    vl = v.view(B, nkv, D)[:, rank * n_local:(rank + 1) * n_local].float()
    ref_l = O.merge_heads(O.sdpa(O.heads(q.float().view(B, n_local, D), H), O.heads(kl, H), O.heads(vl, H)))
    assert rel(oa.view(B, n_local, D), ref_l) < 6e-3


def test_attention_large_scores_rescale_path():
    """Scores with a growing row max force the lazy O-rescale branch (max grows by > 2^8 between tiles)."""
    from oracle import dit_oracle as O
    from scail_b200 import ops
    H, nq, nkv = 1, 128, 1024
    q = rnd(nq, 128, seed=1)
    k = rnd(nkv, 128, seed=2) * torch.linspace(0.2, 6.0, nkv, device="cuda")[:, None].to(torch.bfloat16)
    v = rnd(nkv, 128, seed=3)
    out = torch.zeros(nq, 128, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, out, 1, H, nq, nkv)
    ref = O.sdpa(q.float()[None, None], k.float()[None, None], v.float()[None, None])[0, 0]
    assert rel(out, ref) < 8e-3


def test_small_ops():
    from oracle import dit_oracle as O
    from scail_b200 import ops
    import torch.nn.functional as F
    t = torch.tensor([500.0, 37.5], device="cuda")
    assert rel(ops.timestep_embedding(t, 256), O.timestep_embedding(t.cpu(), 256).cuda()) < 4e-3
    x = rnd(2, 1536, seed=1)
    assert rel(ops.silu(x), F.silu(x.float())) < 4e-3
    p = rnd(1, 6, 256, seed=2)
    assert rel(ops.adaln_modulation(x, p), x.float() + p.float().view(1, -1)) < 4e-3
    lat = torch.randn(1, 4, 16, 8, 8, device="cuda")
    v = rnd(2, 4, 16, 8, 8, seed=3)
    want = O.cfg_euler_step(lat, v[:1].float(), v[1:].float(), 0.9, 0.8, 4.0)
    got = ops.cfg_euler_(lat.clone(), v, 4.0, 0.8 - 0.9)
    assert float((got - want).abs().max()) < 1e-5
    assert torch.equal(ops.cast_bf16(lat), lat.to(torch.bfloat16))


def test_patchify_unpatchify_index_exact():
    """Integer-coded patch order / unpatchify scatter against the golden maps produced by the reference
    (tests/golden/dit_index.pt): bit-exact."""
    import os
    from scail_b200 import ops
    ix = torch.load(os.path.join(os.path.dirname(__file__), "golden", "dit_index.pt"))
    t, h, w = ix["geom"]["t"], ix["geom"]["h"], ix["geom"]["w"]
    # values < 256 are exact in bf16: encode ids modulo 251 in channel 0, zeros elsewhere
    def ids(tt, hh, ww, base):
        return ((base + torch.arange(tt * hh * ww)) % 251).float().reshape(1, tt, 1, hh, ww)
    def full(a):
        return torch.cat([a, torch.zeros(a.shape[0], a.shape[1], 15, *a.shape[3:])], 2).to(torch.bfloat16).cuda().contiguous()
    a_main, a_pose = ops.patchify(full(ids(t, h, w, 0)), full(ids(1, h, w, 100000)), full(ids(t, h // 2, w // 2, 200000)))
    got = torch.cat([a_main[0, :, :4], a_pose[0, :, :4]], 0).float().cpu()  # channel 0: (p,q) = 4 values
    want = (ix["tok_ids"][0] % 251).float()
    assert torch.equal(got, want)
    # mask channels: x -> 0, ref -> 1, pose -> 1 (dit_video_crossattn_sc_xc.py:1468-1503)
    n_ref = h * w // 4
    assert float(a_main[0, :n_ref, 64:].min()) == 1.0 and float(a_main[0, n_ref:, 64:].abs().max()) == 0.0
    assert float(a_pose[0, :, 64:].min()) == 1.0
    n_seq = t * h * w // 4
    N = ix["tok_ids"].shape[1]
    code = ((torch.arange(N)[:, None] * 64 + torch.arange(64)[None]) % 251)
    lin = code[n_ref:n_ref + n_seq].to(torch.bfloat16).cuda().contiguous()[None]
    got = ops.unpatchify(lin, 1, t, h // 2, w // 2).float().cpu()
    assert torch.equal(got, (ix["unpatchify"] % 251).float())


def test_error_paths_return_codes_not_crashes():
    """Bad arguments must come back as a negative return code + message (never exit / crash / silent fallback)."""
    from scail_b200 import _lib, ops
    a, w = rnd(16, 24), rnd(8, 24)
    with pytest.raises(RuntimeError, match="multiples of 8"):
        ops.gemm(a[:, :20].contiguous(), w[:, :20].contiguous())  # K = 20
    with pytest.raises(RuntimeError, match="unknown epilogue"):
        ops.gemm(a, w, epilogue=17)
    with pytest.raises(RuntimeError, match="gate/residual required"):
        ops.gemm(a, w, epilogue=ops.EPI_BIAS_GATE_RES)
    with pytest.raises(RuntimeError, match="16-byte aligned"):  # ADVICE r1: the epilogue uses 16-byte accesses
        ops.gemm(a, w, rnd(w.shape[0] + 8)[4:4 + w.shape[0]])      # bias view at an 8-byte offset
    with pytest.raises(RuntimeError, match="multiples of 8"):
        big = torch.empty(a.shape[0], w.shape[0] + 4, device="cuda", dtype=torch.bfloat16)
        ops.gemm(a, w, out=big[:, :w.shape[0]])                    # bf16 output with ldc % 8 == 4
    x = rnd(2, 4, 388)
    with pytest.raises(RuntimeError, match="multiple of 8"):
        ops.ln_modulate(x)
    with pytest.raises(RuntimeError, match="unsupported channel count"):
        ops.rmsnorm_cl(rnd(4, 40), rnd(40))
    h = _lib.lib()
    assert h.scail_attention(None, 0, None, 0, None, 0, None, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1.0, 0, None) < 0
    assert b"null operand" in h.scail_last_error()
    # the library is still healthy afterwards
    out = ops.gemm(rnd(128, 64), rnd(256, 64))
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
