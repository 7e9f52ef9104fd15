"""fp8_linear="int8": the INT8 quantiser and the fused LN bit for bit against the restatement (int8_linear_oracle), the INT8
GEMM through ops.gemm_fp8 on int8 operands in all six epilogues (bias, residual and gate bit for bit against the restated
chain; the activations to the bf16 bound), and the model-level guarantees: toggling between the three modes, a GraphedStep
that follows in-place weight edits, and context-parallel ranks bit-identical to the one-GPU forward.  TF32 is off
throughout."""
import pytest
import torch

import int8_linear_oracle as R
from kernel_check import assert_close_bf16

pytestmark = pytest.mark.gpu
I8 = torch.int8
BF = torch.bfloat16
GELU_TANH_ABS = 2.0 ** -11  # tanh.approx slack, as in test_gemm_tiles_gpu.py
EPIS = ("BIAS", "BIAS_GELU", "BIAS_GATE_RES", "BIAS_RES", "BIAS_SILU", "BIAS_GELU_ERF")
EXACT = ("BIAS", "BIAS_GATE_RES", "BIAS_RES")


@pytest.fixture(autouse=True)
def _no_tf32():
    a, b = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = a, b


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(BF)


def quant8(x):
    """ops.quant_rows_fp8 into an int8 q: the INT8 row format on the GPU."""
    from scail_b200 import ops
    q = torch.empty(x.shape, device="cuda", dtype=I8)
    return ops.quant_rows_fp8(x, q, torch.empty(x.shape[0], device="cuda"))


# ---------------------------------------------------------------- 1. quantiser
@pytest.mark.parametrize("K", [5120, 13824, 15360])
def test_quant_rows_int8_bit_exact(K):
    M = 333  # ragged: not a multiple of anything the kernels tile by
    big = rnd(M, K + 96, seed=K)
    x = big[:, 48:48 + K]  # a column slab of a wider buffer
    x[5] = 0                                       # all-zero row
    x[7, 100] = 3.0e4                              # one large outlier
    x[9] = (x[9].float() * 1e-30).to(BF)           # tiny magnitudes
    x[11, :] = 0
    x[11, K - 1] = -2.0                            # a single non-zero at the row's end
    x[13] = torch.tensor([0.5, 1.5, 2.5, -2.5], device="cuda").repeat(K // 4).to(BF)
    x[13, 0] = 127.0                               # s = 1: exact ties x.5, rounded half to even
    q, s = quant8(x)
    qr, sr = R.quant(x)
    assert torch.equal(s, sr)
    assert torch.equal(q, qr)
    assert float(s[5]) == 1.0 and not q[5].any()
    assert int(q[11, K - 1]) == -127 and q[13, 1:4].tolist() == [2, 2, -2]


# ---------------------------------------------------------------- 2. fused LN
@pytest.mark.parametrize("form", ["modulate", "affine"])
@pytest.mark.parametrize("rows", ["all", "offset"])
def test_ln_modulate_int8_bit_exact(form, rows):
    from scail_b200 import ops
    B, N, d = 2, 1000, 5120
    x = rnd(B, N, d, seed=1) + rnd(B, N, 1, seed=5)
    if form == "modulate":  # per-batch shift / scale: slices of the block's [B, 6, d] adaLN vectors
        mod = rnd(B, 6, d, scale=0.5, seed=2)
        kw = dict(shift=mod[:, 3], scale=mod[:, 4])
    else:
        kw = dict(gamma=rnd(d, seed=3) + 1, beta=rnd(d, scale=0.1, seed=4))
    if rows == "offset":  # the final layer's form: rows [row_offset, row_offset + rows_out) of each batch
        kw.update(rows_out=700, row_offset=257)
    n = kw.get("rows_out", N)
    ref = ops.ln_modulate(x, eps=1e-6, **kw)
    q = torch.full((B * n, d), 99, device="cuda", dtype=I8)
    s = torch.full((B * n,), 7.0, device="cuda")
    got = ops.ln_modulate(x, eps=1e-6, out_fp8=(q, s), **kw)
    assert got[0] is q and got[1] is s
    qr, sr = R.quant(ref.view(B * n, d))
    assert torch.equal(s, sr)
    assert torch.equal(q, qr)
    qk, sk = quant8(ref.view(B * n, d))  # and the quantiser kernel of the bf16 result
    assert torch.equal(q, qk) and torch.equal(s, sk)


# ---------------------------------------------------------------- 3. GEMM
def run_int8(epi, M, N, K, rows_per_batch=0, out=None, in_place=False, a_slab=False, seed=0, codes=None):
    """ops.gemm_fp8 on int8 operands with epilogue `epi` -> (got, restated fp32 chain).  codes: (aq, wq) to use instead of
    quantised random operands."""
    from scail_b200 import ops
    b = rnd(N, seed=seed + 3)
    if codes is None:
        (aq, sa), (wq, sw) = R.quant(rnd(M, K, seed=seed + 1)), R.quant(rnd(N, K, scale=K ** -0.5, seed=seed + 2))
    else:
        aq, wq = codes
        sa = torch.rand(M, device="cuda") * 1e-4
        sw = torch.rand(N, device="cuda") * 1e-4
    if a_slab:  # A as a column slab of a wider int8 buffer
        big = torch.full((M, 3 * K), 55, device="cuda", dtype=I8)
        big[:, K:2 * K] = aq
        aq = big[:, K:2 * K]
    kw, gate, res = {}, None, None
    rpb = rows_per_batch or M
    if epi in ("BIAS_GATE_RES", "BIAS_RES"):
        res = rnd(M, N, seed=seed + 7)
        if epi == "BIAS_GATE_RES":
            gate = rnd(-(-M // rpb), 3, N, seed=seed + 8)[:, 1]  # rows gate_stride = 3 N apart, like mod[:, k]
            kw.update(gate=gate, rows_per_batch=rpb)
        if in_place:
            if out is None:
                out = torch.empty(M, N, device="cuda", dtype=BF)
            out.copy_(res)
            res = out
        kw["residual"] = res
    want = R.gemm(aq, sa, wq, sw, b, epi, gate, rpb, None if res is None else res.clone())
    got = ops.gemm_fp8(aq, sa, wq, sw, b, out=out, epilogue=getattr(ops, "EPI_" + epi), **kw)
    torch.cuda.synchronize()
    return got, want


def check(got, want, epi, what):
    if epi in EXACT:
        bad = int((got != want.to(BF)).sum())
        assert bad == 0, f"{what}: {bad} of {got.numel()} elements differ from the restated chain"
        print(f"{what}: bit-exact")
    else:
        c = assert_close_bf16(got, want, what, elem_abs=GELU_TANH_ABS if epi == "BIAS_GELU" else 2.0 ** -12)
        print(f"{what}: rel-L2 {c.rel_l2:.2e}, worst |d|/bound {c.worst_ratio:.2f}")


LINEARS = [("qkv", 3 * 5120, 5120, "BIAS"), ("attn_out", 5120, 5120, "BIAS_GATE_RES"), ("cross_q", 5120, 5120, "BIAS"),
           ("cross_out", 5120, 5120, "BIAS_RES"), ("fc1", 13824, 5120, "BIAS_GELU"), ("fc2", 5120, 13824, "BIAS_GATE_RES")]


@pytest.mark.parametrize("name,N,K,epi", LINEARS)
def test_gemm_int8_at_the_six_linears(name, N, K, epi):
    """The six per-block linears' (N, K) at a ragged M = 4000 with two batches; gate and residual in place, as the block
    runs them."""
    got, want = run_int8(epi, 4000, N, K, rows_per_batch=2000, in_place=True, seed=N + K)
    check(got, want, epi, name)


@pytest.mark.parametrize("epi", ["BIAS_SILU", "BIAS_GELU_ERF"])
def test_gemm_int8_other_epilogues(epi):
    got, want = run_int8(epi, 1000, 5120, 5120, seed=11)
    check(got, want, epi, epi)


@pytest.mark.parametrize("M", [2, 130, 1000])
@pytest.mark.parametrize("N", [72, 200])
@pytest.mark.parametrize("epi", EPIS)
def test_gemm_int8_ragged(epi, N, M):
    """M and N not multiples of the 128 x 256 tile, K = 144 not a multiple of the 128-wide k-block."""
    got, want = run_int8(epi, M, N, 144, rows_per_batch=max(M // 2, 1))
    check(got, want, epi, f"{epi} M={M} N={N}")


@pytest.mark.parametrize("rows_per_batch", [1000, 100])
@pytest.mark.parametrize("in_place", [False, True])
def test_gemm_int8_gate_rows_inside_tile(rows_per_batch, in_place):
    """rows_per_batch = 100: most 128-row tiles straddle a batch boundary, some span three batches."""
    got, want = run_int8("BIAS_GATE_RES", 3000, 512, 256, rows_per_batch=rows_per_batch, in_place=in_place)
    check(got, want, "BIAS_GATE_RES", f"gate rows_per_batch={rows_per_batch} in_place={in_place}")


@pytest.mark.parametrize("epi", EPIS)
def test_gemm_int8_column_slabs(epi):
    """A and C as column slabs of wider buffers at ragged M and N: everything beside C is bit for bit unchanged."""
    M, N, K = 300, 200, 192
    big_c = rnd(M + 3, 512, seed=9)
    before = big_c.clone()
    c = big_c[:M, 136:136 + N]
    got, want = run_int8(epi, M, N, K, rows_per_batch=128, out=c, in_place=epi in ("BIAS_RES", "BIAS_GATE_RES"),
                         a_slab=True)
    assert got.data_ptr() == c.data_ptr()
    check(c, want, epi, f"{epi} slab")
    assert torch.equal(big_c[:, :136], before[:, :136])
    assert torch.equal(big_c[:, 136 + N:], before[:, 136 + N:])
    assert torch.equal(big_c[M:], before[M:])


def test_gemm_int8_worst_case_magnitude():
    """All codes +-127 at K = 13 824: |acc| reaches 13 824 * 127^2 = 2.23e8 (row 0 against column 0: every product +16 129),
    far past fp32's 2^24, so the one conversion to fp32 rounds; the s32 sum itself must not wrap or lose a bit."""
    M, N, K = 300, 264, 13824
    g = torch.Generator(device="cuda").manual_seed(12)
    aq = (torch.randint(0, 2, (M, K), device="cuda", generator=g, dtype=I8) * 2 - 1) * 127
    wq = (torch.randint(0, 2, (N, K), device="cuda", generator=g, dtype=I8) * 2 - 1) * 127
    aq[0], wq[0], wq[1] = 127, 127, -127
    for epi in ("BIAS", "BIAS_GATE_RES"):
        got, want = run_int8(epi, M, N, K, rows_per_batch=M, codes=(aq, wq))
        check(got, want, epi, f"{epi} all codes +-127")
    assert float(R.accumulate(aq[:1], wq[:2]).abs().max()) == K * 127 * 127


def test_gemm_int8_refusals():
    from scail_b200 import _lib, ops
    aq, sa = quant8(rnd(64, 144))
    wq, sw = quant8(rnd(64, 144))
    out = torch.empty(64, 64, device="cuda", dtype=torch.float32)
    f = _lib.lib().scail_gemm_int8
    rc = f(aq.data_ptr(), 144, wq.data_ptr(), 144, None, out.data_ptr(), 64, 64, 64, 144, 0, None, 0, 0, None, 0, 1,
           sa.data_ptr(), sw.data_ptr(), None)
    assert rc == -1 and b"bf16" in _lib.lib().scail_last_error()
    rc = f(aq.data_ptr(), 144, wq.data_ptr(), 144, None, out.data_ptr(), 64, 64, 64, 136, 0, None, 0, 0, None, 0, 0,
           sa.data_ptr(), sw.data_ptr(), None)
    assert rc == -1 and b"multiples of 16" in _lib.lib().scail_last_error()
    rc = f(aq.data_ptr(), 144, wq.data_ptr(), 144, None, out.data_ptr(), 64, 64, 64, 131072 + 16, 0, None, 0, 0, None, 0, 0,
           sa.data_ptr(), sw.data_ptr(), None)
    assert rc == -1 and b"131072" in _lib.lib().scail_last_error()
    with pytest.raises(TypeError, match="both"):
        ops.gemm_fp8(aq, sa, ops.quant_rows_fp8(rnd(64, 144))[0], sw)


# ---------------------------------------------------------------- 4. the model: modes, graphs, context parallelism
SMALL = dict(hidden_size=256, num_attention_heads=2, inner_hidden_size=512, num_layers=2, text_dim=64, time_embed_dim=256)


def small_model(seed=0, mode="int8"):
    from scail_b200.dit import DiffusionTransformer
    torch.manual_seed(seed)
    m = DiffusionTransformer(fp8_linear=mode, **SMALL).to(BF).cuda().eval()
    with torch.no_grad():
        for _, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
    return m


def small_inputs(seed=1, t=3, h=16, w=16, b=2):
    """N = 4 * 64 + 3 * 16 = 304 tokens at the default size."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(BF).cuda()
    x, ref, pose = r(b, t, 16, h, w), r(1, 1, 16, h, w), r(1, t, 16, h // 2, w // 2)
    return dict(x=x, timesteps=torch.full((b,), 400.0, device="cuda"), context=r(b, 24, 64), ref_concat=ref,
                concat_smpl_render=pose, image_clip_features=r(1, 257, 1280))


def test_toggling_modes_matches_fresh_models():
    """False -> "int8" -> True -> False between forwards of one model: each forward gives the bits of a fresh model built in
    that mode, so no mode leaves state (weight copies, workspaces) that changes another's result."""
    inp = small_inputs(5)
    m = small_model(6, False)
    got = {}
    with torch.no_grad():
        for i, mode in enumerate((False, "int8", True, False)):
            m.mixins["adaln_layer"].fp8_linear = mode
            got[i] = m(**inp).clone()
        fresh = {mode: small_model(6, mode)(**inp).clone() for mode in (False, "int8", True)}
    torch.cuda.synchronize()
    assert torch.equal(got[0], fresh[False]) and torch.equal(got[3], fresh[False])
    assert torch.equal(got[1], fresh["int8"]) and torch.equal(got[2], fresh[True])
    assert not torch.equal(got[1], got[0]) and not torch.equal(got[1], got[2])
    lin = m.transformer.layers[0].mlp.dense_h_to_4h
    assert lin._int8_cache[2].dtype == I8 and lin._fp8_cache[2].dtype == torch.float8_e4m3fn


def test_int8_composes_with_every_fp8_attention_mode():
    """fp8_linear="int8" composes with the three fp8_attention values: each forward matches a fresh model in that pair of
    modes bit for bit."""
    inp = small_inputs(7)
    m = small_model(8)
    with torch.no_grad():
        for att in (False, True, "int8_qk"):
            m.mixins["adaln_layer"].fp8_attention = att
            got = m(**inp).clone()
            f = small_model(8)
            f.mixins["adaln_layer"].fp8_attention = att
            assert torch.equal(got, f(**inp)), att


def test_graphed_step_follows_in_place_weight_edits_in_int8():
    """GraphedStep in INT8 mode replays the bits of sampler_step, also after an in-place edit of a weight after capture (the
    int8 copy is re-derived into the buffers the graph holds)."""
    from scail_b200 import sampler
    m = small_model(16)
    g = torch.Generator().manual_seed(3)
    r = lambda *s: torch.randn(*s, generator=g).to(BF).cuda()
    x0 = torch.randn(1, 3, 16, 8, 8, generator=g).cuda()
    cond = dict(crossattn=r(1, 24, 64), ref_concat=r(1, 1, 16, 8, 8), concat_smpl_render=r(1, 3, 16, 4, 4),
                image_clip_features=r(1, 257, 1280))
    uc = dict(crossattn=r(1, 24, 64))
    sig = sampler.make_flow_timesteps(50, 5.0)
    edit = lambda model: model.transformer.layers[1].mlp.dense_4h_to_h.weight.mul_(0.5)
    with torch.no_grad():
        xg = x0.clone()
        gs = sampler.GraphedStep(m, xg, cond, uc, 4.0)
        held = m.transformer.layers[1].mlp.dense_4h_to_h._int8_cache[2]
        gs(sig[0], sig[1])
        gs(sig[1], sig[2])
        edit(m)
        gs(sig[2], sig[3])
        assert m.transformer.layers[1].mlp.dense_4h_to_h._int8_cache[2] is held  # re-derived in place
        e = small_model(16)
        xe = x0.clone()
        sampler.sampler_step(e, xe, sig[0], sig[1], cond, uc, 4.0)
        sampler.sampler_step(e, xe, sig[1], sig[2], cond, uc, 4.0)
        edit(e)
        sampler.sampler_step(e, xe, sig[2], sig[3], cond, uc, 4.0)
    torch.cuda.synchronize()
    assert torch.equal(xe, xg)


@pytest.mark.parametrize("b", [2, 1])
def test_context_parallel_ranks_match_one_gpu_int8(b):
    """Token-sharded ranks 0, 1 and P - 1 (P = 4, 76 tokens each) through the in-process stand-in rank: every block output
    and the output rows bit-identical to the one-GPU INT8 forward, at b = 2 (the CFG branches on two streams) and b = 1."""
    from test_cp_launch_shapes_gpu import compare_rank, reference, run_rank
    from scail_b200 import dit
    m = small_model(21)
    inp = small_inputs(22, b=b)
    P = 4
    with torch.no_grad():
        ref = reference(m, inp)
        for rank in (0, 1, P - 1):
            dit._WS.bufs.clear()
            out, blocks, index = run_rank(m, inp, ref, P, rank)
            res = compare_rank(out, blocks, ref, P, rank, index)
            assert all(same for same, _ in res.values()), (rank, res)
    lin = m.transformer.layers[0].attention.query_key_value
    assert lin._int8_cache is not None and getattr(lin, "_fp8_cache", None) is None
