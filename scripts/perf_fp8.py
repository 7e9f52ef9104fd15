"""FP8 (e4m3) linears against bf16, in one process, alternating.  Prints one JSON line per result with the card's name and
power limit.

  1. The six per-block GEMMs at b = 2, N = 27 904 (M = 55 808): our bf16 GEMM; our fp8 GEMM alone and together with the
     quantisation of its activation (quant_rows_fp8 for the out-projections and fc2, the fp8 LayerNorm for QKV, cross q
     and fc1, timed against the bf16 LayerNorm it replaces); torch._scaled_mm with row-wise scales on the same operands.
  2. Sampler steps/s of the 40-block 14B model (bench.py's model and inputs) with fp8_linear on and off on the same
     instance, and the rel-L2 of the fp8 CFG velocity against the bf16 one.
ITERS (default 20) launches per GEMM timing, REPS (default 2) alternating rounds, STEPS (default 2) timed sampler steps."""
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scail_b200 import ops  # noqa: E402

d, f, n = 5120, 13824, 27904
M = 2 * n
# name: (N, K, epilogue, activation quantiser: "ln" = fused fp8 LayerNorm, "rows" = quant_rows_fp8)
SHAPES = {"qkv": (3 * d, d, ops.EPI_BIAS, "ln"), "attn_out": (d, d, ops.EPI_BIAS_GATE_RES, "rows"),
          "cross_q": (d, d, ops.EPI_BIAS, "ln"), "cross_out": (d, d, ops.EPI_BIAS_RES, "rows"),
          "fc1": (f, d, ops.EPI_BIAS_GELU, "ln"), "fc2": (d, f, ops.EPI_BIAS_GATE_RES, "rows")}
ITERS = int(os.environ.get("ITERS", 20))
REPS = int(os.environ.get("REPS", 2))
STEPS = int(os.environ.get("STEPS", 2))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q}


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(ITERS):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / ITERS


def gemm_shape(name):
    N, K, epi, quant = SHAPES[name]
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * K ** -0.5
    b = torch.randn(N, device="cuda", dtype=torch.bfloat16)
    out = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    kw = {}
    if epi == ops.EPI_BIAS_GATE_RES:
        kw = dict(gate=torch.randn(2, N, device="cuda", dtype=torch.bfloat16), residual=out, rows_per_batch=n)
    elif epi == ops.EPI_BIAS_RES:
        kw = dict(residual=out)
    wq, ws = ops.quant_rows_fp8(w)
    aq, sa = ops.quant_rows_fp8(a)
    x3 = a.view(2, n, K)  # LayerNorm input for the "ln" shapes (K = d)
    mod = torch.randn(2, 6, K, device="cuda", dtype=torch.bfloat16) * 0.1
    ln_kw = dict(shift=mod[:, 0], scale=mod[:, 1])
    lnb = torch.empty(2, n, K, device="cuda", dtype=torch.bfloat16)

    def quantise():
        if quant == "ln":
            ops.ln_modulate(x3, eps=1e-6, out_fp8=(aq, sa), **ln_kw)
        else:
            ops.quant_rows_fp8(a, aq, sa)

    def bf16_producer():  # what the bf16 path runs in the quantiser's place: the bf16 LayerNorm (nothing for "rows")
        if quant == "ln":
            ops.ln_modulate(x3, out=lnb, eps=1e-6, **ln_kw)

    arms = {
        "ours_bf16": lambda: ops.gemm(a, w, b, out=out, epilogue=epi, **kw),
        "ours_fp8": lambda: ops.gemm_fp8(aq, sa, wq, ws, b, out=out, epilogue=epi, **kw),
        "ours_fp8_with_quant": lambda: (quantise(), ops.gemm_fp8(aq, sa, wq, ws, b, out=out, epilogue=epi, **kw)),
        "ours_bf16_with_ln": lambda: (bf16_producer(), ops.gemm(a, w, b, out=out, epilogue=epi, **kw)),
        "quant_only": quantise,
        "torch_scaled_mm_rowwise": lambda: torch._scaled_mm(aq, wq.t(), scale_a=sa[:, None], scale_b=ws[None, :],
                                                            out_dtype=torch.bfloat16),
    }
    res = {k: [] for k in arms}
    for _ in range(REPS):
        for k, fn in arms.items():
            res[k].append(round(timed(fn), 3))
    flops = 2.0 * M * N * K
    line = {"gemm": name, "M": M, "N": N, "K": K, "ms": res,
            "tflops_fp8_alone": round(flops / min(res["ours_fp8"]) / 1e9, 1),
            "tflops_bf16": round(flops / min(res["ours_bf16"]) / 1e9, 1),
            "quant_bytes": M * K * 3 + 4 * M if quant == "rows" else None, **card()}
    print(json.dumps(line), flush=True)
    del a, w, out, wq, aq, lnb
    torch.cuda.empty_cache()


def steps():
    import bench
    from scail_b200 import sampler
    m = bench.build_model("cuda")
    h = bench.synthetic_inputs()
    dv = {k: v.cuda() for k, v in h.items()}
    cond = dict(crossattn=dv["context_cond"], ref_concat=dv["ref_concat"], concat_smpl_render=dv["concat_smpl_render"],
                image_clip_features=dv["image_clip_features"])
    uc = dict(crossattn=dv["context_uncond"])
    sig = sampler.make_flow_timesteps(50, 5.0)
    ad = m.mixins["adaln_layer"]
    res, vel = {"bf16": [], "fp8": []}, {}
    with torch.no_grad():
        for rep in range(REPS):
            for mode in ("bf16", "fp8"):
                ad.fp8_linear = mode == "fp8"
                vel[mode] = sampler.guided_velocity(m, dv["x"], float(sig[10]), cond, uc, 4.0)  # warm-up (fp8: quantises weights)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(STEPS):
                    sampler.sampler_step(m, dv["x"].clone(), sig[10 + i], sig[11 + i], cond, uc, 4.0)
                torch.cuda.synchronize()
                res[mode].append(round(STEPS / (time.perf_counter() - t0), 4))
    v16, v8 = vel["bf16"].float(), vel["fp8"].float()
    rel = float((v8 - v16).norm() / v16.norm())
    print(json.dumps({"sampler_steps_per_s": res, "steps_per_rep": STEPS,
                      "velocity_rel_l2_fp8_vs_bf16": rel, "workload": "SCAIL-14B, 40 blocks, latent 21x64x64, CFG batch 2",
                      **card()}), flush=True)


if __name__ == "__main__":
    torch.manual_seed(0)
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "gemm"):
        for name in SHAPES:
            gemm_shape(name)
    if which in ("all", "steps"):
        steps()
