"""Restatement of the INT8 linears of fp8_linear="int8" (DESIGN §3.1.1) in torch, for the tests to pin the kernels to.

Row format (quant_rows_int8_kernel, ln_modulate_kernel<false, true>): s = amax(|row|) / 127 as an IEEE fp32 division (1 for
an all-zero row), q = round-half-even(x / s) saturated to [-127, 127].

GEMM (gemm_int8_kernel): the s32 accumulator is exact, and so is an fp64 GEMM of the codes (every product is at most
127^2 = 16 129 and every partial sum stays below 2^53), so `a.double() @ w.double().T` is the accumulator bit for bit.  The
epilogue then restates in fp32 in the kernel's order, every step one IEEE rounding:
  f = (f32(acc) * s_a[m]) * s_w[n] + bias[n];  f = act(f);  f = f * gate[b(m), n];  f = f + res[m, n];  C = bf16(f).
Eager torch runs each of those as its own elementwise kernel (no contraction into an FMA), so the restated chain is exact
for the bias, residual and gate epilogues; the activations (tanh.approx, __expf, erff in the kernel) are only close."""
import torch
import torch.nn.functional as F

QMAX = 127.0


def codes(xf, s):
    """round-half-even(x / s) saturated to +-127, as int8 (xf fp32 [M, K], s fp32 [M])."""
    return torch.round(xf / s[:, None]).clamp_(-QMAX, QMAX).to(torch.int8)


def quant(x):
    """The INT8 row format of x [M, K] -> (q int8 [M, K], s fp32 [M]).  The divisor is a tensor: torch evaluates
    `tensor / python_float` as a multiplication by the reciprocal, not as the IEEE division the kernels do."""
    xf = x.float()
    amax = xf.abs().amax(1)
    s = torch.where(amax > 0, amax / torch.full_like(amax, QMAX), torch.ones_like(amax))
    return codes(xf, s), s


def accumulate(aq, wq):
    """The exact s32 accumulator of int8 codes a [M, K] and w [N, K], as fp64 [M, N]."""
    return aq.double() @ wq.double().T


def pre_activation(acc, sa, sw, bias=None):
    """(f32(acc) * s_a) * s_w (+ bias), fp32 [M, N]."""
    f = acc.float().mul_(sa[:, None]).mul_(sw[None, :])
    return f.add_(bias.float()) if bias is not None else f


def activation(f, epi):
    """The activation of epilogue `epi` (the name of scail_b200.ops's EPI_* constant without the prefix) in fp32."""
    if epi == "BIAS_GELU":
        return F.gelu(f, approximate="tanh")
    if epi == "BIAS_SILU":
        return F.silu(f)
    if epi == "BIAS_GELU_ERF":
        return F.gelu(f)
    return f


def epilogue(f, epi, gate_rows=None, res=None):
    """The rest of the chain on the fp32 pre-activation f [M, N]: the activation, the gate (gate_rows [M, N]: row m's gate
    row) and the residual -> fp32 before the bf16 rounding."""
    f = activation(f, epi)
    if epi == "BIAS_GATE_RES":
        f = f.mul_(gate_rows.float())
    if epi in ("BIAS_GATE_RES", "BIAS_RES"):
        f = f.add_(res.float())
    return f


def gemm(aq, sa, wq, sw, bias=None, epi="BIAS", gate=None, rows_per_batch=None, res=None, chunk=8192):
    """The whole chain -> fp32 [M, N] before the bf16 rounding (bf16 of it is the kernel's output for the bias, residual and
    gate epilogues).  gate [B, N]: row m reads gate[m // rows_per_batch].  Rows in chunks, so that the fp64 accumulator of a
    14B-width launch stays small."""
    M = aq.shape[0]
    rpb = rows_per_batch or M
    out = torch.empty(M, wq.shape[0], device=aq.device, dtype=torch.float32)
    for r0 in range(0, M, chunk):
        r1 = min(M, r0 + chunk)
        f = pre_activation(accumulate(aq[r0:r1], wq), sa[r0:r1], sw, bias)
        g = None if gate is None else gate[torch.arange(r0, r1, device=gate.device) // rpb]
        out[r0:r1] = epilogue(f, epi, g, None if res is None else res[r0:r1])
    return out
