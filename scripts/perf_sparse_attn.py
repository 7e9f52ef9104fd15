"""Block-sparse (frame-window) self-attention against dense, on one GPU.  Prints one JSON line with the card's name and power
limit; OUT=<dir> also appends it to <dir>/perf_sparse_attn.jsonl (nothing is written otherwise).

  kernels: ms per launch of the dense kernel and of the sparse kernel at windows 1, 2, 3 and 5, at b = 2, 40 heads and
           N = 27 904 (512 x 512) and 48 832 (512 x 896), bf16 (scail_attention) and fp8 (scail_attention_fp8).  The arms
           alternate inside each round; each number is the best of REPS rounds (default 3) of 5 timed launches.
  steps:   sampler steps/s of bench.py's 14B model and inputs (512 x 512), the same instance toggled dense / window 2
           (STEP_WINDOW), alternated ROUNDS times (default 2), and the rel-L2 of the window's guided velocity against the
           dense one on those random weights (not a statement about visual quality: there are no real weights here).
PARTS=kernels or PARTS=steps runs one part only."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from scail_b200 import ops, sparse  # noqa: E402

WINDOWS = (1, 2, 3, 5)
REPS = int(os.environ.get("REPS", 3))


def timeit(fn, iters=5):
    fn(); fn(); torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def geometry(t, h, w):
    """bench.py's token layout for a t x h x w latent (patch 1 x 2 x 2)."""
    H, W = h // 2, w // 2
    return sparse.geometry(H * W, t * H * W, t * (h // 2) * (w // 2) // 4, t, H, W)


def kernels():
    B, H, d = 2, 40, 5120
    res = []
    for t, h, w in ((21, 64, 64), (21, 64, 112)):
        g = geometry(t, h, w)
        N = g.ref_length + g.seq_length + g.pose_length
        torch.manual_seed(0)
        qkv = torch.randn(B * N, 3 * d, device="cuda", dtype=torch.bfloat16)
        out = torch.empty(B * N, d, device="cuda", dtype=torch.bfloat16)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        maps = {wd: sparse.tile_map(g, wd, "cuda") for wd in WINDOWS}
        Lp = ops.fp8_pad(N)
        q8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
        k8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
        w1 = torch.ones(d, device="cuda", dtype=torch.bfloat16)
        ops.rmsnorm_rope(qkv, N, d, [(0, w1), (d, w1)], out_fp8=[q8, k8])
        vt, vs = ops.quant_vt_fp8(v, B, H, N)
        arms = {"bf16_dense": lambda: ops.attention(q, k, v, out, B, H, N, N),
                "fp8_dense": lambda: ops.attention_fp8(q8[0], q8[1], k8[0], k8[1], vt, vs, out, B, H, N)}
        for wd, m in maps.items():
            arms[f"bf16_w{wd}"] = lambda m=m: ops.attention_sparse(q, k, v, out, B, H, N, m)
            arms[f"fp8_w{wd}"] = lambda m=m: ops.attention_fp8_sparse(q8[0], q8[1], k8[0], k8[1], vt, vs, out, B, H, N, m)
        ms = {a: [] for a in arms}
        for _ in range(REPS):
            for a, fn in arms.items():
                ms[a].append(round(timeit(fn), 3))
        best = {a: min(x) for a, x in ms.items()}
        row = dict(N=N, latent=f"{t}x{h}x{w}", n_tiles=maps[1].n_q_tiles, ms=ms, best_ms=best,
                   density={wd: round(m.density, 4) for wd, m in maps.items()})
        for dt in ("bf16", "fp8"):
            row[f"{dt}_time_over_dense"] = {wd: round(best[f"{dt}_w{wd}"] / best[f"{dt}_dense"], 3) for wd in WINDOWS}
            # time per listed tile pair relative to dense: 1.0 means the sparse launch runs as fast per tile as the dense one
            row[f"{dt}_time_over_density"] = {wd: round(best[f"{dt}_w{wd}"] / best[f"{dt}_dense"] / maps[wd].density, 3)
                                              for wd in WINDOWS}
        res.append(row)
        del qkv, out, q8, k8, vt, vs, arms
        torch.cuda.empty_cache()
    return res


def steps():
    import bench
    from scail_b200 import sampler
    window = int(os.environ.get("STEP_WINDOW", 2))
    dev = torch.device("cuda", torch.cuda.current_device())
    model = bench.build_model(dev)
    ad = model.mixins["adaln_layer"]
    host = bench.synthetic_inputs()
    d = {k: v.to(dev) for k, v in host.items()}
    cond = dict(crossattn=d["context_cond"], ref_concat=d["ref_concat"], concat_smpl_render=d["concat_smpl_render"],
                image_clip_features=d["image_clip_features"])
    uc = dict(crossattn=d["context_uncond"])
    sig = sampler.make_flow_timesteps(50, 5.0)
    x = d["x"].clone()
    n_steps = int(os.environ.get("STEPS", 2))
    sps = {"dense": [], f"window{window}": []}
    with torch.no_grad():
        vel = {}
        for name, wd in (("dense", None), (f"window{window}", window)):
            ad.attention_window = wd
            vel[name] = sampler.guided_velocity(model, d["x"], sig[10], cond, uc, 4.0).clone()
            sampler.sampler_step(model, x, sig[0], sig[1], cond, uc, 4.0)  # warm-up of this mode
        for _ in range(int(os.environ.get("ROUNDS", 2))):
            for name, wd in (("dense", None), (f"window{window}", window)):
                ad.attention_window = wd
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(n_steps):
                    sampler.sampler_step(model, x, sig[i], sig[i + 1], cond, uc, 4.0)
                e1.record(); torch.cuda.synchronize()
                sps[name].append(round(1000.0 * n_steps / e0.elapsed_time(e1), 4))
        ad.attention_window = None
    a, b = vel["dense"].double(), vel[f"window{window}"].double()
    return dict(latent=f"{bench.T_LAT}x{bench.H_LAT}x{bench.W_LAT}", steps_per_round=n_steps, steps_per_s=sps,
                speedup=round(max(sps[f"window{window}"]) / max(sps["dense"]), 3),
                guided_velocity_rel_l2=float((b - a).norm() / a.norm()))


def main():
    assert torch.cuda.is_available(), "perf_sparse_attn.py needs a CUDA device"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = ""
    parts = os.environ.get("PARTS", "kernels,steps").split(",")
    res = dict(gpu=torch.cuda.get_device_name(), nvidia_smi=smi)
    if "kernels" in parts:
        res["kernels"] = kernels()
    if "steps" in parts:
        res["steps"] = steps()
    line = json.dumps(res)
    print(line, flush=True)
    if os.environ.get("OUT"):
        os.makedirs(os.environ["OUT"], exist_ok=True)
        with open(os.path.join(os.environ["OUT"], "perf_sparse_attn.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
