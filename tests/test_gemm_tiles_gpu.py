"""The GEMM's staged epilogue, element by element: every epilogue at ragged M and N, gate rows that change inside a
128-row tile, the DiT's in-place residual at the bench shapes, and A / C as column slabs of wider buffers.

The epilogue writes each 128 x 256 tile into a swizzled shared-memory buffer and stores it with TMA, which clips to
[M, N].  A misplaced column chunk, a wrong swizzle row or a store past N changes a few elements or writes a neighbour,
which rel-L2 barely sees; so every result goes through kernel_check.assert_close_bf16 against an fp32 reference computed
on the GPU with TF32 off, and slab neighbours are compared bit for bit."""
import pytest
import torch

from kernel_check import assert_close_bf16

pytestmark = pytest.mark.gpu

# tanh.approx.f32 has a relative error of about 2^-11, so gelu_tanh(x) = 0.5 x (1 + tanh(u)) is off by up to
# 0.5 |x| 2^-11 = |x| 2^-12 before rounding.  Where 1 + tanh(u) is near 0 (x very negative) that is not small relative
# to the output, so the absolute slack is doubled to 2^-11 max|want|: max|want| ~ max x for GELU, which covers |x| 2^-12.
GELU_TANH_ABS = 2.0 ** -11


@pytest.fixture(autouse=True)
def _no_tf32():
    a = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = a


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


EPIS = ["bias", "gelu", "silu", "gelu_erf", "gate_res", "res", "fp32"]


def run_epilogue(epi, a, w, b, rows_per_batch=0, out=None, in_place=False, seed=7):
    """Run ops.gemm with epilogue `epi`; return (got, fp32 reference, elem_abs)."""
    from scail_b200 import ops
    import torch.nn.functional as F
    M, N = a.shape[0], w.shape[0]
    acc = a.float() @ w.float().t() + b.float()
    code = {"bias": ops.EPI_BIAS, "gelu": ops.EPI_BIAS_GELU, "silu": ops.EPI_BIAS_SILU, "gelu_erf": ops.EPI_BIAS_GELU_ERF,
            "gate_res": ops.EPI_BIAS_GATE_RES, "res": ops.EPI_BIAS_RES, "fp32": ops.EPI_BIAS}[epi]
    kw, elem_abs = {}, 2.0 ** -12
    if epi in ("gate_res", "res"):
        res = rnd(M, N, seed=seed)
        ref = acc
        if epi == "gate_res":
            rpb = rows_per_batch or M
            gate = rnd((M + rpb - 1) // rpb, 3, N, seed=seed + 1)[:, 1]  # rows gate_stride = 3 N apart, like mod[:, k]
            kw.update(gate=gate, rows_per_batch=rpb)
            ref = ref * gate.float().repeat_interleave(rpb, 0)[:M]
        ref = ref + res.float()
        if in_place:
            if out is None:
                out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
            out.copy_(res)
            res = out
        kw["residual"] = res
    elif epi == "gelu":
        ref, elem_abs = F.gelu(acc, approximate="tanh"), GELU_TANH_ABS
    elif epi == "silu":
        ref = F.silu(acc)
    elif epi == "gelu_erf":
        ref = F.gelu(acc)
    else:
        ref = acc
    if epi == "fp32" and out is None:
        out = torch.empty(M, N, device="cuda", dtype=torch.float32)
    got = ops.gemm(a, w, b, out=out, epilogue=code, **kw)
    torch.cuda.synchronize()
    assert got.dtype == (torch.float32 if epi == "fp32" else torch.bfloat16)
    return got, ref, elem_abs


def check(got, ref, what, elem_abs):
    if got.dtype == torch.float32:  # no rounding at all: only the fp32 summation order differs
        d = (got - ref).abs().max().item()
        assert d <= 2.0 ** -16 * ref.abs().max().item(), f"{what}: max |diff| {d:.3g}"
    else:
        assert_close_bf16(got, ref, what, elem_abs=elem_abs)


@pytest.mark.parametrize("name,N,K,epi", [("qkv", 3 * 5120, 5120, "bias"), ("attn_out", 5120, 5120, "gate_res"),
                                          ("fc1", 13824, 5120, "gelu"), ("fc2", 5120, 13824, "gate_res")])
def test_gemm_bench_shapes(name, N, K, epi):
    """The four per-block GEMMs at M = 2 x 27904; gate+residual in place (residual is out), as the DiT calls them."""
    M = 2 * 27904
    a, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    got, ref, elem_abs = run_epilogue(epi, a, w, b, rows_per_batch=27904, in_place=True)
    check(got, ref, name, elem_abs)


@pytest.mark.parametrize("M", [2, 130, 1000])
@pytest.mark.parametrize("N", [72, 200])
@pytest.mark.parametrize("epi", EPIS)
def test_gemm_epilogue_ragged(epi, N, M):
    """Every epilogue with M and N not multiples of the 128 x 256 tile (N = 72: only part of the first 64-column chunk)."""
    K = 136
    a, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    got, ref, elem_abs = run_epilogue(epi, a, w, b, rows_per_batch=max(M // 2, 1))
    check(got, ref, f"{epi} M={M} N={N}", elem_abs)


@pytest.mark.parametrize("rows_per_batch", [1000, 100])
@pytest.mark.parametrize("in_place", [False, True])
def test_gemm_gate_rows_inside_tile(rows_per_batch, in_place):
    """rows_per_batch = 1000: tiles 7 and 15 hold rows of two batches.  100: every tile spans two or three batches."""
    M, N, K = 3000, 512, 256
    a, w, b = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    got, ref, elem_abs = run_epilogue("gate_res", a, w, b, rows_per_batch=rows_per_batch, in_place=in_place)
    check(got, ref, f"gate rows_per_batch={rows_per_batch}", elem_abs)


@pytest.mark.parametrize("epi", ["bias", "gelu", "res", "gate_res", "fp32"])
def test_gemm_column_slabs(epi):
    """A and C as column slabs of wider buffers at ragged N (and M): the columns beside C are bit for bit unchanged."""
    M, N, K = 300, 200, 192
    big_a = rnd(M, 3 * K, seed=1)
    a = big_a[:, K:2 * K]
    w, b = rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3)
    dtype = torch.float32 if epi == "fp32" else torch.bfloat16
    big_c = rnd(M + 3, 512, seed=9).to(dtype)  # rows past M and columns around the slab hold sentinel data
    before = big_c.clone()
    c = big_c[:M, 136:136 + N]
    got, ref, elem_abs = run_epilogue(epi, a, w, b, rows_per_batch=128, out=c, in_place=epi in ("res", "gate_res"))
    assert got.data_ptr() == c.data_ptr()
    check(c, ref, f"{epi} slab", elem_abs)
    assert torch.equal(big_c[:, :136], before[:, :136])
    assert torch.equal(big_c[:, 136 + N:], before[:, 136 + N:])
    assert torch.equal(big_c[M:], before[M:])
    assert torch.equal(big_a, rnd(M, 3 * K, seed=1))
