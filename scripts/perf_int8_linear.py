"""INT8 linears (fp8_linear="int8") against e4m3 and bf16, in one process, alternating.  Prints one JSON line per result with
the card's name, power limit and maximum SM clock as nvidia-smi reads them (nothing is set).

  1. The six per-block GEMMs at b = 2, N = 27 904 (M = 55 808), CUDA events over ITERS launches each: our bf16 GEMM, the
     e4m3 GEMM, the INT8 GEMM alone and together with the quantisation of its activation (quant_rows_fp8 into an int8 q
     for the out-projections and fc2, the INT8 LayerNorm for QKV, cross q and fc1), the e4m3 GEMM with its quantisation,
     and the bf16 GEMM with the bf16 LayerNorm the quantised forms replace.
  2. Sampler steps/s of the 40-block 14B model (bench.py's model and inputs) with the same instance toggled bf16 / e4m3 /
     INT8 linears, and the rel-L2 of each 8-bit mode's CFG velocity against the bf16 one.
ITERS (default 20) launches per GEMM timing, REPS (default 2) alternating rounds, STEPS (default 2) timed sampler steps."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from perf_fp8 import SHAPES, M, card, d, n, timed  # noqa: E402
from scail_b200 import ops  # noqa: E402

REPS = int(os.environ.get("REPS", 2))
STEPS = int(os.environ.get("STEPS", 2))


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
    i8 = lambda rows, cols: (torch.empty(rows, cols, device="cuda", dtype=ops.INT8), torch.empty(rows, device="cuda"))
    wq, ws = ops.quant_rows_fp8(w)
    aq, sa = ops.quant_rows_fp8(a)
    wi, wis = ops.quant_rows_fp8(w, *i8(N, K))
    ai, ais = ops.quant_rows_fp8(a, *i8(M, K))
    x3 = a.view(2, n, K)  # LayerNorm input for the "ln" shapes (K = d)
    mod = torch.randn(2, 6, K, device="cuda", dtype=torch.bfloat16) * 0.1
    ln_kw = dict(shift=mod[:, 0], scale=mod[:, 1])
    lnb = torch.empty(2, n, K, device="cuda", dtype=torch.bfloat16)

    def quantise(q, s):
        if quant == "ln":
            ops.ln_modulate(x3, eps=1e-6, out_fp8=(q, s), **ln_kw)
        else:
            ops.quant_rows_fp8(a, q, s)

    def bf16_producer():  # what the bf16 path runs in the quantiser's place: the bf16 LayerNorm (nothing for "rows")
        if quant == "ln":
            ops.ln_modulate(x3, out=lnb, eps=1e-6, **ln_kw)

    arms = {
        "bf16": lambda: ops.gemm(a, w, b, out=out, epilogue=epi, **kw),
        "e4m3": lambda: ops.gemm_fp8(aq, sa, wq, ws, b, out=out, epilogue=epi, **kw),
        "int8": lambda: ops.gemm_fp8(ai, ais, wi, wis, b, out=out, epilogue=epi, **kw),
        "int8_with_quant": lambda: (quantise(ai, ais), ops.gemm_fp8(ai, ais, wi, wis, b, out=out, epilogue=epi, **kw)),
        "e4m3_with_quant": lambda: (quantise(aq, sa), ops.gemm_fp8(aq, sa, wq, ws, b, out=out, epilogue=epi, **kw)),
        "bf16_with_ln": lambda: (bf16_producer(), ops.gemm(a, w, b, out=out, epilogue=epi, **kw)),
    }
    res = {k: [] for k in arms}
    for _ in range(REPS):
        for k, fn in arms.items():
            res[k].append(round(timed(fn), 3))
    flops = 2.0 * M * N * K
    tops = {k: round(flops / min(v) / 1e9, 1) for k, v in res.items() if k in ("bf16", "e4m3", "int8")}
    print(json.dumps({"gemm": name, "M": M, "N": N, "K": K, "ms": res, "tera_ops_per_s": tops, **card()}), flush=True)
    del a, w, out, wq, aq, wi, ai, lnb
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
    modes = {"bf16": False, "e4m3": True, "int8": "int8"}
    res, vel = {k: [] for k in modes}, {}
    with torch.no_grad():
        for rep in range(REPS):
            for mode, lin in modes.items():
                ad.fp8_linear = lin
                vel[mode] = sampler.guided_velocity(m, dv["x"], float(sig[10]), cond, uc, 4.0)  # warm-up (quantises weights)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(STEPS):
                    sampler.sampler_step(m, dv["x"].clone(), sig[10 + i], sig[11 + i], cond, uc, 4.0)
                torch.cuda.synchronize()
                res[mode].append(round(STEPS / (time.perf_counter() - t0), 4))
    v16 = vel["bf16"].float()
    rel = {k: float((v.float() - v16).norm() / v16.norm()) for k, v in vel.items() if k != "bf16"}
    print(json.dumps({"sampler_steps_per_s": res, "steps_per_rep": STEPS, "velocity_rel_l2_vs_bf16": rel,
                      "allocated_gib_with_both_weight_copies": round(torch.cuda.memory_allocated() / 2 ** 30, 1),
                      "workload": f"SCAIL-14B, 40 blocks, latent 21x64x64, CFG batch 2, d = {d}", **card()}), flush=True)


if __name__ == "__main__":
    torch.manual_seed(0)
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "gemm"):
        for name in SHAPES:
            gemm_shape(name)
    if which in ("all", "steps"):
        steps()
