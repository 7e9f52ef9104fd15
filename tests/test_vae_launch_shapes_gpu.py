"""The Wan VAE kernels at the shapes SCAIL's inference launches them, against fp32.

SCAIL runs the VAE three ways: it decodes the 81-frame result, encodes the reference image as a single frame, and
encodes the 81-frame pose render (often at half resolution) and the reference image followed by zero frames.  At
512x896 and 480x832 the kernels meet channel widths, N blocks and ragged edges that small test shapes never reach
(480x832 is ragged for the conv tiles at every stage: H = 60, W = 104 / 208 / 416 / 832).

test_every_vae_launch_matches_fp32: a random-weight WanVAE(dim=96) runs those geometries with the conv / GEMM / norm /
softmax / upsample entry points of scail_b200.ops wrapped by recorders.  Each distinct launch (every argument except
the frame count) is re-run on fresh random data at <= 3 frames plus its causal history, and compared with an fp32
reference on the GPU (TF32 off) by kernel_check.assert_close_bf16: rel-L2 <= 4e-3 and an elementwise bound that one
wrong pixel trips.  GEMMs keep their recorded M, since the tile order depends on it.

The rest compares whole paths with the fp32 oracle (oracle/vae_oracle.py, pinned to the reference by
test_oracle_golden.py): the full-width encoder on a single 480x832 frame, on 5 frames whose stages are >= 128 px wide
(row-tile kernel at 96 / 192 / 384 channels) and on one frame followed by zero frames; a single-frame decode (the
upsample3d T = 1 branch); and the mid-block attention at 64x112 = 7168 tokens."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from kernel_check import assert_close_bf16, recording

pytestmark = pytest.mark.gpu

OPS = ("conv3d_cl", "conv3d_strided_cl", "gemm", "rmsnorm_cl", "softmax_rows", "upsample2x_cl")
DECODE_LATENTS = [(2, 64, 112), (2, 60, 104), (1, 64, 112)]  # -> 5x512x896, 5x480x832, 1x512x896
ENCODE_VIDEOS = [(5, 512, 896), (1, 512, 896), (5, 256, 448), (5, 480, 832)]
CHUNKED_DECODE = (3, 64, 112)  # chunk_frames=1: every causal conv with a history, the head at a frame offset
CHUNKED_ENCODE = (9, 256, 448)  # chunk_frames=1: also the stride-2 time_conv at toff = -1 with a 1-frame history

# End-to-end bound per element: 40 bf16 layers do not keep one-rounding accuracy, but no element may be off by more
# than 1/16 of its value plus 1/16 of the largest output (an unwritten or misplaced tile, a wrong frame).
E2E_ELEM = dict(elem_rel=2.0 ** -4, elem_abs=2.0 ** -4)


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


def _randomize_(module, seed):
    """Fan-in scaled weights, gammas near 1, small biases (as in test_vae_gpu.py)."""
    torch.manual_seed(seed)
    with torch.no_grad():
        for n, p in module.named_parameters():
            if "gamma" in n:
                p.copy_(1 + 0.1 * torch.randn_like(p))
            elif p.dim() >= 2 and p.numel() > p.shape[0]:
                p.copy_(torch.randn_like(p) / p[0].numel() ** 0.5)
            else:
                p.copy_(0.02 * torch.randn_like(p))
    return module


@contextlib.contextmanager
def _oracle_on_gpu():
    """fp32 oracle on the GPU, TF32 off, convolutions without cuDNN: its fp32 algorithms take tens of GB of workspace at
    512x896 when the card has it free."""
    with torch.device("cuda"), torch.backends.cudnn.flags(enabled=False, allow_tf32=False):
        yield


def _random_vae(seed):
    from scail_b200.wan_vae import WanVAE
    vae = WanVAE(dim=96)
    _randomize_(vae.model, seed)
    return vae


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _pack(w):
    """[Cout, Cin, kt, kh, kw] -> [Cout, kt*kh*kw*Cin] (tap-major, channel-minor)."""
    return w.permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1).contiguous()


def _ncthw(x):
    """Channels-last [T, H, W, C] -> fp32 [1, C, T, H, W]."""
    return x.float().permute(3, 0, 1, 2)[None]


def _conv_frames(xin, w, b, n, tstride=1, sstride=1):
    """fp32 F.conv3d over the already padded xin [1, Cin, *, H, W], one output frame at a time (output j reads frames
    j*tstride ..): cuDNN's workspace for a whole 3-frame 512x896 conv would dominate the test's memory."""
    kt = w.shape[2]
    return torch.cat([F.conv3d(xin[:, :, j * tstride:j * tstride + kt], w, b, stride=(1, sstride, sstride))
                      for j in range(n)], 2)


# ---------------------------------------------------------------- recording
def _fields(name, a):
    """(fields that select the kernel and its edges, frame count) of one call; `a` holds the bound arguments."""
    if name == "conv3d_cl":
        T, H, W, Cin = a["x"].shape
        assert a["norm_gamma"] is None  # wan_vae.py does not use the fused norm output
        return dict(H=H, W=W, Cin=Cin, cout=a["cout"], taps=(a["kt"], a["kh"], a["kw"]), fmul=a["fmul"],
                    ocols=a["ocols"] or a["cout"], head=a["head"], residual=a["residual"] is not None,
                    hist=0 if a["hist"] is None else a["hist"].shape[0], offset=a["out_frame_offset"] > 0), T
    if name == "conv3d_strided_cl":
        _, H, W, Cin = a["x"].shape
        To, Ho, Wo = a["out_shape"]
        return dict(H=H, W=W, Cin=Cin, cout=a["cout"], taps=(a["kt"], a["kh"], a["kw"]), out_hw=(Ho, Wo),
                    sstride=a["sstride"], pad=(a["pad_h"], a["pad_w"]), tstride=a["tstride"], toff=a["toff"],
                    hist=0 if a["hist"] is None else a["hist"].shape[0]), To
    if name == "gemm":
        x, w, out, res = a["a"], a["w"], a["out"], a["residual"]
        assert a["gate"] is None
        return dict(M=x.shape[0], N=w.shape[0], K=x.shape[1], lda=x.stride(0), ldw=w.stride(0),
                    ldc=w.shape[0] if out is None else out.stride(0),
                    fp32=a["out_fp32"] if out is None else out.dtype == torch.float32, bias=a["bias"] is not None,
                    epilogue=a["epilogue"], ldr=0 if res is None else res.stride(0), rows_per_batch=a["rows_per_batch"]), 1
    if name == "rmsnorm_cl":
        return dict(shape=tuple(a["x"].shape[1:]), silu=a["silu"]), a["x"].shape[0]
    if name == "softmax_rows":
        return dict(rows=a["s"].shape[0], cols=a["s"].shape[1], scale=float(a["scale"])), 1
    if name == "upsample2x_cl":
        return dict(shape=tuple(a["x"].shape[1:])), a["x"].shape[0]
    raise KeyError(name)


@pytest.fixture(scope="module")
def launches():
    """[(op, fields, frames)] of every distinct launch at the production geometries, in first-call order."""
    from scail_b200 import ops
    vae = _random_vae(0)
    g = torch.Generator(device="cuda").manual_seed(0)
    video = lambda T, H, W: torch.rand(3, T, H, W, device="cuda", generator=g) * 2 - 1
    with recording(ops, OPS, _fields) as seen:
        for T, h, w in DECODE_LATENTS:
            vae.decode([torch.randn(16, T, h, w, device="cuda", generator=g)])
        vae.decode([torch.randn(16, *CHUNKED_DECODE, device="cuda", generator=g)], chunk_frames=1)
        for T, H, W in ENCODE_VIDEOS:
            vae.encode([video(T, H, W)])
        vae.encode([video(*CHUNKED_ENCODE)], chunk_frames=1)
    torch.cuda.synchronize()
    return [(name, dict(f), T) for (name, f), T in seen.items()]


# ---------------------------------------------------------------- one launch vs fp32
def check_conv3d_cl(ops, f, T, g):
    H, W, Cin, cout, (kt, kh, kw), fmul, ocols, th = (f[k] for k in ("H", "W", "Cin", "cout", "taps", "fmul", "ocols", "hist"))
    T = min(T, 3)
    x, hist = _rand(g, T, H, W, Cin), (_rand(g, th, H, W, Cin) if th else None)
    # head: output std ~0.4, so that about 1 % of the outputs reach the clamp at +-1 (checked below); a value clamped on
    # both sides would hide an error
    fan_in = Cin * kt * kh * kw
    w = _rand(g, cout, Cin, kt, kh, kw, scale=(0.4 if f["head"] else 1.0) * fan_in ** -0.5)
    b = _rand(g, cout, scale=0.05 if f["head"] else 1.0)
    xin = F.pad(_ncthw(x if hist is None else torch.cat([hist, x])), (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    y = _conv_frames(xin[:, :, th:], w.float(), b.float(), T)[0]  # the output frames of x
    if f["head"]:  # fp32 planes [cout, T, H, W], clamped; with an offset, into frames [off, off + T) of a larger output
        off = 1 if f["offset"] else 0
        out = torch.full((cout, T + 2, H, W), 7.0, device="cuda") if off else None
        got = ops.conv3d_cl(x, _pack(w), b, kt, kh, kw, cout, head=True, out=out, out_frame_offset=off, hist=hist)
        if off:
            assert bool((got[:, :off] == 7).all() and (got[:, off + T:] == 7).all()), "head wrote outside its frames"
            got = got[:, off:off + T]
        clamped = float((y.abs() >= 1).float().mean())
        assert clamped < 0.03, f"head test data: {clamped:.1%} of the reference outputs are clamped"
        return got, y.clamp(-1, 1)
    y = y.permute(1, 2, 3, 0)
    if fmul > 1:  # upsample3d time_conv: channel block i of frame t is output frame fmul * t + i
        y = y.reshape(T, H, W, fmul, ocols).permute(0, 3, 1, 2, 4).reshape(T * fmul, H, W, ocols)
    res = _rand(g, T * fmul, H, W, ocols) if f["residual"] else None
    got = ops.conv3d_cl(x, _pack(w), b, kt, kh, kw, cout, residual=res, fmul=fmul, ocols=ocols, hist=hist)
    return got, y if res is None else y + res.float()


def check_conv3d_strided_cl(ops, f, To, g):
    H, W, Cin, cout, (kt, kh, kw), (Ho, Wo), s, (ph, pw), ts, toff, th = (
        f[k] for k in ("H", "W", "Cin", "cout", "taps", "out_hw", "sstride", "pad", "tstride", "toff", "hist"))
    To = min(To, 3 if ts == 1 else 2)
    T = (To - 1) * ts + toff + kt  # input frames up to the last one the last output reads
    x, hist = _rand(g, T, H, W, Cin), (_rand(g, th, H, W, Cin) if th else None)
    w, b = _rand(g, cout, Cin, kt, kh, kw, scale=(Cin * kt * kh * kw) ** -0.5), _rand(g, cout)
    got = ops.conv3d_strided_cl(x, _pack(w), b, kt, kh, kw, cout, (To, Ho, Wo), sstride=s, pad_h=ph, pad_w=pw, tstride=ts,
                                toff=toff, hist=hist)
    # output frame j reads frames j*ts + toff .. of x (negative: the history, then zeros); spatially the ZeroPad2d
    # convention: pad_h / pad_w zeros before, and zeros past the bottom / right edge as far as the last output reads
    xin = _ncthw(x if hist is None else torch.cat([hist, x]))
    f0 = toff + th
    xin = F.pad(xin, (pw, max(0, (Wo - 1) * s + kw - pw - W), ph, max(0, (Ho - 1) * s + kh - ph - H), max(0, -f0), 0))
    want = _conv_frames(xin[:, :, max(0, f0):], w.float(), b.float(), To, ts, s)[0, :, :, :Ho, :Wo]
    return got, want.permute(1, 2, 3, 0)


def check_gemm(ops, f, _, g):
    M, N, K = f["M"], f["N"], f["K"]
    assert f["epilogue"] in (ops.EPI_BIAS, ops.EPI_BIAS_RES), f["epilogue"]
    a = _rand(g, M, f["lda"])[:, :K]
    w = _rand(g, N, f["ldw"], scale=K ** -0.5)[:, :K]
    bias = _rand(g, N) if f["bias"] else None
    res = _rand(g, M, f["ldr"])[:, :N] if f["ldr"] else None
    out = torch.empty(M, f["ldc"], device="cuda", dtype=torch.float32 if f["fp32"] else torch.bfloat16)[:, :N]
    got = ops.gemm(a, w, bias, out=out, epilogue=f["epilogue"], residual=res, rows_per_batch=f["rows_per_batch"])
    want = a.float() @ w.float().T
    if bias is not None:
        want += bias.float()
    if res is not None:
        want += res.float()
    return got, want


def check_rmsnorm_cl(ops, f, T, g):
    x = _rand(g, min(T, 3), *f["shape"])
    C = x.shape[-1]
    gamma = (1 + 0.1 * torch.randn(C, device="cuda", generator=g)).to(torch.bfloat16)
    want = F.normalize(x.float(), dim=-1) * C ** 0.5 * gamma.float()
    return ops.rmsnorm_cl(x, gamma, silu=f["silu"]), F.silu(want) if f["silu"] else want


def check_softmax_rows(ops, f, _, g):
    scale = f["scale"]
    s = torch.randn(f["rows"], f["cols"], device="cuda", generator=g) * (3.0 / scale)  # scaled logits with std 3
    return ops.softmax_rows(s, scale), torch.softmax(s * scale, -1)


def check_upsample2x_cl(ops, f, T, g):
    x = _rand(g, min(T, 3), *f["shape"])
    return ops.upsample2x_cl(x), x.repeat_interleave(2, 1).repeat_interleave(2, 2)


CHECKS = {name: globals()["check_" + name] for name in OPS}


def _describe(name, f):
    return name + " " + " ".join(f"{k}={v}" for k, v in f.items())


def test_every_vae_launch_matches_fp32(launches):
    from scail_b200 import ops
    failures = []
    print(f"\n{len(launches)} distinct VAE launches (frames: as recorded; re-run at <= 3 plus the history)")
    for i, (name, f, T) in enumerate(launches):
        what = f"{_describe(name, f)} T={T}"
        g = torch.Generator(device="cuda").manual_seed(1000 + i)
        torch.cuda.reset_peak_memory_stats()
        try:
            got, want = CHECKS[name](ops, f, T, g)
            if name == "upsample2x_cl":
                assert torch.equal(got, want), f"{what}: not bit-exact"
                result = "exact"
            else:
                c = assert_close_bf16(got, want, what)
                result = (f"rel-L2 {c.rel_l2:.2e}, worst |d|/bound {c.worst_ratio:.2f} "
                          f"(|d| {abs(c.got_at_worst - c.want_at_worst):.2e} at {c.worst_index})")
            print(f"{what}: {result}, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")
        except AssertionError as e:
            print(f"FAIL {e}")
            failures.append(str(e))
        got = want = None
    assert not failures, f"{len(failures)} of {len(launches)} launches failed:\n" + "\n".join(failures)


def test_recorded_launches_cover_the_production_cases(launches):
    def has(name, **want):
        return any(n == name and all(v(f[k]) if callable(v) else f[k] == v for k, v in want.items()) for n, f, _ in launches)

    cases = {
        "encoder conv1 (RGB zero-padded to Cin = 8) at 896 and 832 px": has("conv3d_cl", Cin=8, W=896) and has("conv3d_cl", Cin=8, W=832),
        "3x3 stride-2 conv at C = 96 / 192 / 384": all(has("conv3d_strided_cl", sstride=2, Cin=c, cout=c) for c in (96, 192, 384)),
        "upsample3d time_conv, 768 wide, fmul = 2": has("conv3d_cl", taps=(3, 1, 1), cout=768, fmul=2),
        "ragged H = 60, W = 104 conv": has("conv3d_cl", H=60, W=104),
        "ragged 128-px row tiles, W = 208 / 416 / 832": all(has("conv3d_cl", W=w, taps=(3, 3, 3)) for w in (208, 416, 832)),
        "conv3d_cl with a causal history": has("conv3d_cl", hist=lambda n: n > 0),
        "conv3d_cl with a history at >= 128 px": has("conv3d_cl", hist=lambda n: n > 0, W=lambda w: w >= 128),
        "time_conv with a history": has("conv3d_cl", fmul=2, hist=lambda n: n > 0),
        "strided time_conv at toff = -1 with a history": has("conv3d_strided_cl", tstride=2, toff=-1, hist=1),
        "head at a frame offset": has("conv3d_cl", head=True, offset=True),
        "softmax over 7168-token rows": has("softmax_rows", cols=7168),
    }
    print("\n" + "\n".join(f"{'ok' if ok else 'MISSING'}: {what}" for what, ok in cases.items()))
    assert all(cases.values()), [what for what, ok in cases.items() if not ok]


# ---------------------------------------------------------------- whole paths vs the fp32 oracle
@pytest.mark.parametrize("frames,H,W,zero_tail", [(1, 480, 832, False), (5, 64, 512, False), (5, 64, 256, True)],
                         ids=["single_480x832", "5x64x512", "image_then_zeros_64x256"])
def test_full_width_encode_vs_oracle(frames, H, W, zero_tail):
    from oracle import vae_oracle as V
    vae = _random_vae(11)
    sd = {k: v.float() for k, v in vae.model.state_dict().items()}
    g = torch.Generator(device="cuda").manual_seed(12)
    video = (torch.rand(3, frames, H, W, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16).float()
    if zero_tail:  # SCAIL's `image` input: the reference image followed by zero frames
        video[:, 1:] = 0
    got = vae.encode([video])
    with _oracle_on_gpu():
        want = V.encode(sd, video[None])
    c = assert_close_bf16(got, want, f"encode {frames}x{H}x{W}", rel_l2=2e-2, **E2E_ELEM)  # as the encode golden tests
    print(f"\nencode {frames}x{H}x{W} (dim 96) vs fp32 oracle: rel-L2 {c.rel_l2:.3e}, worst |d|/bound {c.worst_ratio:.2f}")


def test_single_frame_decode_vs_oracle():
    """One latent frame: upsample3d takes its T = 1 branch (no time_conv)."""
    from oracle import vae_oracle as V
    vae = _random_vae(13)
    sd = {k: v.float() for k, v in vae.model.state_dict().items()}
    z = _rand(torch.Generator(device="cuda").manual_seed(14), 16, 1, 64, 112)
    got = vae.decode([z])
    with _oracle_on_gpu():
        want = V.decode(sd, z[None].float())
    c = assert_close_bf16(got, want, "decode 1x64x112", rel_l2=1.5e-2, **E2E_ELEM)  # as the dim-96 decode in test_scale_gpu
    print(f"\ndecode 1x64x112 -> 1x512x896 (dim 96) vs fp32 oracle: rel-L2 {c.rel_l2:.3e}, worst |d|/bound {c.worst_ratio:.2f}")


def test_mid_block_attention_at_7168_tokens_vs_oracle():
    from torch.nn.attention import SDPBackend, sdpa_kernel

    from oracle import vae_oracle as V
    from scail_b200.wan_vae import AttentionBlock
    C = 384
    blk = _randomize_(AttentionBlock(C), 15).cuda().to(torch.bfloat16)
    with torch.no_grad():  # q, k x1.6: scaled logits with std ~2.5, so some 14 tokens carry each row and the attention
        blk.to_qkv.weight[:2 * C] *= 1.6  # term is not swamped by the residual
    x = _rand(torch.Generator(device="cuda").manual_seed(16), 1, 64, 112, C)
    got = blk.run(x)
    sd = {"a." + k: v.float() for k, v in blk.state_dict().items()}
    with _oracle_on_gpu(), sdpa_kernel(SDPBackend.MATH):
        want = V.attention_block(sd, "a", _ncthw(x))[0].permute(1, 2, 3, 0)
    # six bf16 roundings in series (normed x, q / k, P, V^T, O, output): looser than one rounding per element
    c = assert_close_bf16(got, want, "attention block", rel_l2=1e-2, elem_rel=2.0 ** -6, elem_abs=2.0 ** -8)
    # the residual x passes through exactly, so the whole output hides most of an attention error; the block's own
    # contribution is the difference, which also carries the output's rounding at the scale of |x|
    d = assert_close_bf16(got.float() - x.float(), want - x.float(), "attention term", rel_l2=2e-2, **E2E_ELEM)
    print(f"\nattention block, 7168 tokens x 384: rel-L2 {c.rel_l2:.3e} (worst |d|/bound {c.worst_ratio:.2f}); "
          f"attention term alone {d.rel_l2:.3e}")
