"""fp8_attention="int8_qk" against the e4m3 self-attention (fp8_attention=True) on the SCAIL-14B shape (b = 2, 40 heads).

  kernels: ms per launch at N = 27 904 and 48 832 of every kernel of both arms and of each arm's total, the int8 and e4m3
           arms alternating in this process, best of REPS (default 3) rounds of ITERS (default 5) launches each:
             e4m3 : rmsnorm_rope(out_fp8) + quant_vt_fp8 + attention_fp8
             int8 : rmsnorm_rope_int8q + quant_k_int8 + quant_vt_fp8 + attention_int8qk
  steps:   sampler steps/s of bench.py's 40-block model and inputs at 512x512 for bf16, fp8 attention and int8_qk on the same
           instance (STEPS, default 2, timed steps per round, REPS rounds alternating), and each mode's guided-velocity
           rel-L2 from bf16 in the same run.
Prints one JSON line per part with the card's name, power limit and max SM clock."""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scail_b200 import ops  # noqa: E402

B, H, d = 2, 40, 5120
REPS = int(os.environ.get("REPS", 3))
ITERS = int(os.environ.get("ITERS", 5))
STEPS = int(os.environ.get("STEPS", 2))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q}


def timed(fn):
    fn()
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(ITERS):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / ITERS


def kernels(N):
    torch.manual_seed(0)
    Lp = ops.fp8_pad(N)
    qkv = torch.randn(B * N, 3 * d, device="cuda", dtype=torch.bfloat16)
    out = torch.empty(B * N, d, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(2, d, device="cuda", dtype=torch.bfloat16) * 0.1 + 1
    ang = torch.rand(N, 128, device="cuda") * 6.3
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    slabs = [(0, w[0]), (d, w[1])]
    f32 = torch.float32
    q8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
    k8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
    qi = (torch.empty(B * N, d, device="cuda", dtype=ops.INT8), torch.empty(B, H, Lp, device="cuda"))
    ki = (torch.empty(B * N, d, device="cuda", dtype=ops.INT8), torch.empty(B, H, Lp, device="cuda"))
    kbar = torch.empty(B, d, device="cuda", dtype=f32)
    part = torch.empty(ops.quant_k_int8_partial_len(B, H, N), device="cuda", dtype=torch.float64)
    vt = torch.empty(B, H, 128, Lp, device="cuda", dtype=ops.FP8)
    vs = torch.empty(B, H, 128, device="cuda")
    work = torch.empty(B, d, device="cuda", dtype=torch.int32)
    qkv_i8 = qkv.clone()  # the int8 form normalises K in place: on a copy, refreshed before each int8 arm
    vt8 = lambda: ops.quant_vt_fp8(qkv[:, 2 * d:], B, H, N, vt, vs, work)
    rope8 = lambda: ops.rmsnorm_rope(qkv, N, d, slabs, cos, sin, out_fp8=[q8, k8])
    att8 = lambda: ops.attention_fp8(q8[0], q8[1], k8[0], k8[1], vt, vs, out, B, H, N)
    ropei = lambda: ops.rmsnorm_rope_int8q(qkv_i8, N, d, slabs, qi[0], qi[1], cos, sin)
    quantk = lambda: ops.quant_k_int8(qkv_i8[:, d:2 * d], B, H, N, ki[0], ki[1], kbar, part)
    atti = lambda: ops.attention_int8qk(qi[0], qi[1], ki[0], ki[1], vt, vs, out, B, H, N)
    arms = {"fp8_rmsnorm_rope": rope8, "fp8_quant_vt": vt8, "fp8_attention": att8, "fp8_total": lambda: (rope8(), vt8(), att8()),
            "int8_rmsnorm_rope": ropei, "int8_quant_k": quantk, "int8_quant_vt": vt8, "int8_attention": atti,
            "int8_total": lambda: (ropei(), quantk(), vt8(), atti())}
    ms = {k: [] for k in arms}
    for _ in range(REPS):
        for k, fn in arms.items():
            if k.startswith("int8"):
                qkv_i8.copy_(qkv)
            ms[k].append(round(timed(fn), 3))
    best = {k: min(v) for k, v in ms.items()}
    fl = 4 * B * H * N * N * 128
    return dict(part="kernels", B=B, H=H, N=N, ms=ms, best=best,
                attention_int8_over_fp8=round(best["int8_attention"] / best["fp8_attention"], 4),
                total_int8_over_fp8=round(best["int8_total"] / best["fp8_total"], 4),
                int8_attention_tflops=round(fl / best["int8_attention"] / 1e9, 1),
                fp8_attention_tflops=round(fl / best["fp8_attention"] / 1e9, 1), **card())


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
    modes = {"bf16": False, "fp8_attention": True, "int8_qk": "int8_qk"}
    res, vel = {k: [] for k in modes}, {}
    with torch.no_grad():
        for _ in range(max(1, REPS - 1)):
            for mode, att in modes.items():
                ad.fp8_attention = att
                vel[mode] = sampler.guided_velocity(m, dv["x"], float(sig[10]), cond, uc, 4.0)  # also the warm-up
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for i in range(STEPS):
                    sampler.sampler_step(m, dv["x"].clone(), sig[10 + i], sig[11 + i], cond, uc, 4.0)
                torch.cuda.synchronize()
                res[mode].append(round(STEPS / (time.perf_counter() - t0), 4))
    ad.fp8_attention = False
    v16 = vel["bf16"].float()
    rel = {k: float((v.float() - v16).norm() / v16.norm()) for k, v in vel.items() if k != "bf16"}
    return dict(part="steps", sampler_steps_per_s=res, steps_per_rep=STEPS, velocity_rel_l2_vs_bf16=rel,
                workload="SCAIL-14B, 40 blocks, latent 21x64x64, CFG batch 2", **card())


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "kernels"):
        for N in (27904, 48832):
            print(json.dumps(kernels(N)), flush=True)
            torch.cuda.empty_cache()
    if which in ("all", "steps"):
        print(json.dumps(steps()), flush=True)
