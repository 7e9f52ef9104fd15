"""The INT8 linear launches of the 14B DiT step (fp8_linear="int8") against their restatement, element by element.

test_every_int8_linear_launch_matches_the_restatement: the full-width two-block random model of test_dit_launch_shapes_gpu.py
runs with fp8_linear="int8" at 21x64x64, 21x60x104 and 21x64x112 (N = 27 904 / 42 510 / 48 832): one sampler.sampler_step
(CFG batch b = 2) and the conditional row alone (b = 1, as CFGCache and a HybridParallel rank call it), each once with every
fp8_attention value (False, True, "int8_qk").  gemm_fp8, quant_rows_fp8 and ln_modulate are recorded by
kernel_check.recording, and each distinct INT8 launch (int8 operands, an int8 q, an int8 out_fp8) is re-run on fresh seeded
data inside sentinel buffers (test_dit_launch_shapes_gpu.Slab) against int8_linear_oracle, by the rules of
test_int8_linear_gpu.py: the quantisers and the bias, residual and gate epilogues bit for bit, GELU-tanh to the bf16 bound.
The bf16 and e4m3 launches of these entry points are test_dit_launch_shapes_gpu.py's.

test_full_width_block_at_480x832_int8_linears_vs_oracle: one full-width block at 21x60x104, b = 2, with INT8 linears and
with e4m3 linears on the same inputs, against oracle/dit_oracle.py in fp32; the INT8 block must be the closer one."""
import time

import pytest
import torch

import int8_linear_oracle as R
from kernel_check import assert_close_bf16, recording
from test_dit_launch_shapes_gpu import (BF, GEOMETRIES, GELU_TANH_ABS, Slab, _describe, _exact, _fields, _no_tf32, _rand,
                                        _view, full_width_model, rel, step_inputs)
from test_scale_gpu import sdpa_fp32_chunked

pytestmark = pytest.mark.gpu
_no_tf32 = _no_tf32  # autouse: TF32 off in every test of this module

OPS = ("gemm_fp8", "quant_rows_fp8", "ln_modulate")
ATTENTION = (False, True, "int8_qk")
I8 = torch.int8


def _fields_int8(name, a):
    """_fields of test_dit_launch_shapes_gpu plus whether the launch is the INT8 form."""
    key, v = _fields(name, a)
    if name == "gemm_fp8":
        key["int8"] = a["a"].dtype == I8
    elif name == "quant_rows_fp8":
        key.update(int8=a["q"] is not None and a["q"].dtype == I8, q=None if a["q"] is None else _view(a["q"]))
    else:
        key["int8"] = a["out_fp8"] is not None and a["out_fp8"][0].dtype == I8
    return key, v


@pytest.fixture(scope="module")
def launches():
    """[(op, key)] of every distinct INT8 launch of the cases in the module docstring, in first-call order."""
    from scail_b200 import dit, ops, sampler
    m = full_width_model(2)
    ad = m.mixins["adaln_layer"]
    ad.fp8_linear = "int8"
    sig = sampler.make_flow_timesteps(50, 5.0)
    with torch.no_grad(), recording(ops, OPS, _fields_int8) as seen:
        for i, (geo, (t, h, w)) in enumerate(GEOMETRIES.items()):
            x0, cond, uc = step_inputs(10 + i, t, h, w)
            ctx = sampler.prepare_context(cond, uc)[1:2]
            ts = torch.full((1,), float(sig[2]) * 1000.0, device="cuda")
            for att in ATTENTION:
                ad.fp8_attention = att
                sampler.sampler_step(m, x0.clone(), sig[0], sig[1], cond, uc, 4.0)
                m(x0.clone(), timesteps=ts, context=ctx, y=None, ref_concat=cond["ref_concat"],
                  concat_smpl_render=cond["concat_smpl_render"], image_clip_features=cond["image_clip_features"],
                  concat_images=None)
    torch.cuda.synchronize()
    del m, ad
    dit._WS.bufs.clear()
    torch.cuda.empty_cache()
    return [(name, dict(k)) for (name, k) in seen if dict(k)["int8"]]


# ---------------------------------------------------------------- one launch vs the restatement
def _quantised(g, rows, cols, scale=1.0):
    return R.quant(_rand(g, rows, cols, scale=scale))


def check_gemm_fp8(ops, f, g):
    M, N, K, epi = f["M"], f["N"], f["K"], f["epilogue"]
    name = {getattr(ops, "EPI_" + e): e for e in ("BIAS", "BIAS_GELU", "BIAS_GATE_RES", "BIAS_RES", "BIAS_SILU",
                                                  "BIAS_GELU_ERF")}[epi]
    assert not f["fp32"]
    aq, sa = _quantised(g, M, K)
    wq, sw = _quantised(g, N, K, scale=K ** -0.5)
    A, W = Slab(aq, f["a"]), Slab(wq, (f["ldw"], 0, False))
    bias = _rand(g, N) if f["bias"] else None
    slabs, kw = [A, W], {}
    res = _rand(g, M, N) if f["residual"] is not None else None
    out = Slab(res if f["residual"] == "out" else torch.zeros(M, N, device="cuda", dtype=BF), f["out"])
    slabs.append(out)
    if f["residual"] is not None:
        if f["residual"] == "out":
            kw["residual"] = out.v
        else:
            Rs = Slab(res, f["residual"])
            slabs.append(Rs)
            kw["residual"] = Rs.v
    gate, rpb = None, f["rows_per_batch"] or M
    if name == "BIAS_GATE_RES":
        G = Slab(_rand(g, -(-M // rpb), N), f["gate"])
        slabs.append(G)
        gate = G.v
        kw.update(gate=gate, rows_per_batch=rpb)
    want = R.gemm(aq, sa, wq, sw, bias, name, gate, rpb, res)
    del aq, wq
    ops.gemm_fp8(A.v, sa, W.v, sw, bias, out=out.v, epilogue=epi, **kw)
    torch.cuda.synchronize()
    for s in slabs:
        s.check("gemm_fp8 int8")
    if name in ("BIAS", "BIAS_RES", "BIAS_GATE_RES"):
        return f"{name}: " + _exact(out.v, want.to(BF), "gemm_fp8 int8"), 0.0
    c = assert_close_bf16(out.v, want, "gemm_fp8 int8", elem_abs=GELU_TANH_ABS if name == "BIAS_GELU" else 2.0 ** -12)
    return f"{name}: rel-L2 {c.rel_l2:.2e}, worst |d|/bound {c.worst_ratio:.2f}", c.worst_ratio


def check_quant_rows_fp8(ops, f, g):
    M, K = f["M"], f["K"]
    x = _rand(g, M, K, scale=3.0)
    x[M // 2] = 0  # an all-zero row: scale 1
    X = Slab(x, f["x"])
    Q = Slab(torch.zeros(M, K, device="cuda", dtype=I8), f["q"])
    S = Slab(torch.zeros(M, 1, device="cuda"), (1, 0, True))
    ops.quant_rows_fp8(X.v, Q.v, S.v.view(-1))
    torch.cuda.synchronize()
    for s in (X, Q, S):
        s.check("quant_rows_fp8 int8")
    qr, sr = R.quant(x)
    _exact(S.v.view(-1), sr, "quant_rows_fp8 int8 scales")
    return _exact(Q.v, qr, "quant_rows_fp8 int8 codes"), 0.0


def check_ln_modulate(ops, f, g):
    B, n_in, D, rows, off, eps = f["B"], f["n_in"], f["D"], f["rows_out"], f["row_offset"], f["eps"]
    x = _rand(g, B, n_in, D, scale=2.0) + _rand(g, B, n_in, 1)  # rows with a mean of their own
    kw = dict(eps=eps, rows_out=rows, row_offset=off)
    if f["gamma"]:
        kw["gamma"] = 1 + _rand(g, D, scale=0.1)
    if f["beta"]:
        kw["beta"] = _rand(g, D, scale=0.1)
    if f["mod_stride"] is not None:  # shift, scale: rows of the block's adaLN vectors (mod[:, k], stride 6 d)
        assert f["mod_stride"] >= 2 * D
        mod = _rand(g, B, f["mod_stride"], scale=0.5)
        kw.update(shift=mod[:, :D], scale=mod[:, D:2 * D])
    q = Slab(torch.zeros(B * rows, D, device="cuda", dtype=I8), (D, 0, True))
    s = Slab(torch.zeros(B * rows, 1, device="cuda"), (1, 0, True))
    ops.ln_modulate(x, out_fp8=(q.v, s.v.view(-1)), **kw)
    torch.cuda.synchronize()
    q.check("ln_modulate int8 codes"), s.check("ln_modulate int8 scales")
    ref = ops.ln_modulate(x, **kw)  # the bf16 form, pinned to fp32 by test_dit_launch_shapes_gpu at the same shapes
    qr, sr = R.quant(ref.view(B * rows, D))
    _exact(s.v.view(-1), sr, "ln_modulate int8 scales")
    return _exact(q.v, qr, "ln_modulate int8 codes"), 0.0


CHECKS = {name: globals()["check_" + name] for name in OPS}


def test_every_int8_linear_launch_matches_the_restatement(launches):
    from scail_b200 import ops
    failures, worst = [], {}
    t0 = time.time()
    print(f"\n{len(launches)} distinct INT8 launches")
    for i, (name, f) in enumerate(launches):
        what = _describe(name, f)
        g = torch.Generator(device="cuda").manual_seed(5000 + i)
        try:
            result, ratio = CHECKS[name](ops, f, g)
            worst[name] = max(worst.get(name, 0.0), ratio)
            print(f"{what}: {result}")
        except AssertionError as e:
            print(f"FAIL {what}: {e}")
            failures.append(f"{what}: {e}")
        torch.cuda.empty_cache()
    print("worst |d|/bound per op (0 = bit-exact): " + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))
    print(f"{len(launches)} launches checked in {time.time() - t0:.0f} s")
    assert not failures, f"{len(failures)} of {len(launches)} launches failed:\n" + "\n".join(failures)


def test_recorded_int8_launches_cover_the_cases(launches):
    """The six linears at b = 2 and b = 1 at every geometry, the LN forms feeding them, and the quantisers of the contexts
    (self- and cross-attention out) and of the fc1 output."""
    from scail_b200 import ops
    d, inner = 5120, 13824

    def has(name, **want):
        return any(n == name and all(f[k] == v for k, v in want.items()) for n, f in launches)

    cases = {}
    for geo, (t, h, w) in GEOMETRIES.items():
        N = (1 + t) * (h // 2) * (w // 2) + t * (h // 4) * (w // 4)
        for b in (2, 1):
            M = b * N
            gate = dict(epilogue=ops.EPI_BIAS_GATE_RES, rows_per_batch=N, residual="out")
            cases[f"{geo}, b = {b}"] = all((
                has("gemm_fp8", M=M, N=3 * d, K=d, epilogue=ops.EPI_BIAS),
                has("gemm_fp8", M=M, N=d, K=d, **gate),
                has("gemm_fp8", M=M, N=d, K=d, epilogue=ops.EPI_BIAS),
                has("gemm_fp8", M=M, N=d, K=d, epilogue=ops.EPI_BIAS_RES, residual="out"),
                has("gemm_fp8", M=M, N=inner, K=d, epilogue=ops.EPI_BIAS_GELU),
                has("gemm_fp8", M=M, N=d, K=inner, **gate),
                has("ln_modulate", B=b, n_in=N, gamma=False), has("ln_modulate", B=b, n_in=N, gamma=True),
                has("quant_rows_fp8", M=M, K=d), has("quant_rows_fp8", M=M, K=inner)))
    print("\n" + "\n".join(f"{'ok' if ok else 'MISSING'}: {what}" for what, ok in cases.items()))
    assert all(cases.values()), [what for what, ok in cases.items() if not ok]


# ---------------------------------------------------------------- the whole block vs the fp32 oracle
def test_full_width_block_at_480x832_int8_linears_vs_oracle():
    """One 14B-width block plus the embeddings and the final layer at latent 21x60x104 (N = 42 510), b = 2 (two different
    text contexts), bf16 attention, with INT8 and with e4m3 linears, against the fp32 oracle."""
    import oracle.dit_oracle as O
    m = full_width_model(1, seed=5)
    x0, cond, uc = step_inputs(6, *GEOMETRIES["480x832"])
    x = torch.cat([x0, x0]).to(BF)
    ctx = torch.cat([uc["crossattn"], cond["crossattn"]])
    ref, pose, clip = cond["ref_concat"], cond["concat_smpl_render"], cond["image_clip_features"]
    ts = torch.full((2,), 500.0, device="cuda")
    ad = m.mixins["adaln_layer"]
    orig = ad.layer_forward
    cap, got = {}, {}

    def lf(hid, mask, **kw):
        o = orig(hid, mask, **kw)
        cap["block"] = o.clone()
        return o

    ad.layer_forward = lf
    with torch.no_grad():
        for mode in ("int8", True, False):
            ad.fp8_linear = mode
            out = m(x, timesteps=ts, context=ctx, ref_concat=ref, concat_smpl_render=pose, image_clip_features=clip).float()
            got[mode] = (cap["block"].float(), out)
    torch.cuda.synchronize()
    sd = {k: v.float() for k, v in m.state_dict().items()}
    del m, ad, orig
    old_sdpa = O.sdpa
    O.sdpa = lambda q, k, v: sdpa_fp32_chunked(q, k, v) if q.dtype == torch.float32 else old_sdpa(q, k, v)
    try:
        with torch.no_grad(), torch.device("cuda"):
            want, hid = O.dit_forward(sd, x.float(), ts, ctx.float(), ref.float(), pose.float(), clip.float(), 40, 1,
                                      return_hidden=True)
            hid = hid[1]
    finally:
        O.sdpa = old_sdpa
    for b, branch in enumerate(("uncond", "cond")):
        e = {mode: (rel(blk[b], hid[b]), rel(out[b], want[b])) for mode, (blk, out) in got.items()}
        (i_blk, i_out), (f_blk, f_out), (b_blk, b_out) = e["int8"], e[True], e[False]
        print(f"480x832 block, b = 2, {branch} branch vs the fp32 oracle: int8 linears block {i_blk:.3e} out {i_out:.3e} | "
              f"e4m3 linears block {f_blk:.3e} out {f_out:.3e} | bf16 block {b_blk:.3e} out {b_out:.3e} | int8 / e4m3: "
              f"block {i_blk / f_blk:.3f} out {i_out / f_out:.3f}")
        assert i_blk < f_blk and i_out < f_out, (branch, e)
