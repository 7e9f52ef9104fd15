"""UniPC flow solver (scail_b200.unipc): kernel cost, sampler cost and final-latent error.  Prints one JSON line per result
with the card's name and power limit; OUT=<dir> also appends them to <dir>/perf_unipc.jsonl (nothing is written otherwise).

  kernels: ms and GB/s of unipc_step_ at the 512x512, 480x832 and 512x896 latents (21 latent frames), for orders 1, 2 and 3
           with the coefficients of a step in the middle of a 50-step schedule (every slot of the order in use), against
           3.35 TB/s; each launch timed after an L2 flush, best of ROUNDS rounds of ITERS launches.  Bytes: x, the bf16 pair, x_last and the active slots read;
           x, x_last and one slot written.
  steps:   steps/s of bench.py's 14B model at 512x512 (40 blocks, CFG batch 2) over a 10-step sample(), Euler against
           UniPC order 2, the two arms alternating in each of ROUNDS rounds.
  error:   the final latent of Euler and of UniPC orders 1-3 at 10, 20 and 30 steps, rel-L2 against a 200-step Euler run, on
           the small random-weight model of perf_forecast_cache.py.  Random weights: a report, not a quality claim.
PARTS=kernels,error,steps selects parts (default all three)."""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from perf_fp8 import card  # noqa: E402
from perf_forecast_cache import small_model  # noqa: E402
from scail_b200 import ops, sampler, unipc  # noqa: E402

ROUNDS = int(os.environ.get("ROUNDS", 3))
ITERS = int(os.environ.get("ITERS", 50))
PARTS = os.environ.get("PARTS", "kernels,error,steps").split(",")
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
LATENTS = {"512x512": (1, 21, 16, 64, 64), "480x832": (1, 21, 16, 60, 104), "512x896": (1, 21, 16, 64, 112)}
NOTE = "random weights: a report of the solver's error against a fine Euler run, not a claim about visual quality"


def emit(line):
    line = {**line, **card()}
    print(json.dumps(line), flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "perf_unipc.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def cold_ms(fn):
    """Each launch timed on its own with events, after a 256 MB write that evicts the 50 MB L2: HBM-cold, as in a
    sampler step, where the forward in between evicts the latent.  Best of ROUNDS rounds of the mean over ITERS."""
    flush = torch.empty(64 << 20, device="cuda", dtype=torch.float32)
    res = []
    for _ in range(ROUNDS):
        fn()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(ITERS)]
        for s, e in ev:
            flush.zero_()
            s.record()
            fn()
            e.record()
        torch.cuda.synchronize()
        res.append(sum(s.elapsed_time(e) for s, e in ev) / ITERS)
    return min(res), res


def kernels():
    sig = unipc.check_schedule(sampler.make_flow_timesteps(50, 5.0))
    for name, shape in LATENTS.items():
        n = 1
        for s in shape:
            n *= s
        for order in (1, 2, 3):
            i = 25
            k = unipc.step_coefficients(sig, i, order)
            pad = [0.0] * (3 - order)
            coef = [float(c) for c in torch.tensor([k.x_last_c, *k.slot_c, *pad, k.m_c, k.y_c, *k.slot_p, *pad, k.m_p])]
            active = sum(1 for a, b in zip(k.slot_c, k.slot_p) if a != 0.0 or b != 0.0)
            x, xl = torch.randn(shape, device="cuda"), torch.randn(shape, device="cuda")
            v = torch.randn(2, *shape[1:], device="cuda").to(torch.bfloat16)
            slots = torch.randn(order, n, device="cuda")
            # repeated in place: the values may grow to inf over the launches, which costs the same as finite values
            ms, rounds = cold_ms(lambda: ops.unipc_step_(x, xl, v, slots, k.write, 4.0, sig[i], coef, True))
            nbytes = n * (4 + 4 + 4 + 4 * active) + n * 12
            emit({"part": "kernels", "latent": name, "shape": list(shape), "order": order, "active_slots": active,
                  "ms_best": round(ms, 4), "ms_rounds": [round(r, 4) for r in rounds], "bytes": nbytes,
                  "GB_per_s": round(nbytes / ms / 1e6, 1), "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)})
            del x, xl, v, slots
        torch.cuda.empty_cache()


def error():
    m, x0, cond, uc = small_model()
    ref = sampler.sample(m, x0.clone(), cond, uc, num_steps=200)
    rel = lambda x: round(float((x - ref).norm() / ref.norm()), 6)
    out = {}
    for n in (10, 20, 30):
        row = {"euler": rel(sampler.sample(m, x0.clone(), cond, uc, num_steps=n))}
        for order in (1, 2, 3):
            row[f"unipc_{order}"] = rel(sampler.sample(m, x0.clone(), cond, uc, num_steps=n, solver=unipc.UniPC(order)))
        out[f"{n}_steps"] = row
    emit({"part": "error", "model": "small: 4 blocks, hidden 512, latent 5x32x32", "shift": 5.0, "scale": 4.0,
          "reference": "Euler, 200 steps", "final_latent_rel_l2": out, "note": NOTE})
    del m
    torch.cuda.empty_cache()


def steps():
    import bench
    m = bench.build_model("cuda")
    h = bench.synthetic_inputs()
    dv = {k: v.cuda() for k, v in h.items()}
    cond = dict(crossattn=dv["context_cond"], ref_concat=dv["ref_concat"], concat_smpl_render=dv["concat_smpl_render"],
                image_clip_features=dv["image_clip_features"])
    uc = dict(crossattn=dv["context_uncond"])
    n = 10
    arms = {"euler": None, "unipc_2": unipc.UniPC(2)}
    sampler.sample(m, dv["x"].clone(), cond, uc, num_steps=2)  # warm-up of both update paths
    sampler.sample(m, dv["x"].clone(), cond, uc, num_steps=2, solver=unipc.UniPC(2))
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for name, solver in arms.items():
            x = dv["x"].clone()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sampler.sample(m, x, cond, uc, num_steps=n, solver=solver)
            torch.cuda.synchronize()
            res[name].append(round(n / (time.perf_counter() - t0), 5))
    med = {k: statistics.median(v) for k, v in res.items()}
    emit({"part": "steps", "workload": "SCAIL-14B, 40 blocks, latent 21x64x64 (512x512), CFG batch 2, eager sample()",
          "steps": n, "rounds": ROUNDS, "steps_per_s": res, "median_steps_per_s": med,
          "unipc_2_over_euler_median": round(med["unipc_2"] / med["euler"] - 1, 5),
          "spread": {k: round((max(v) - min(v)) / min(v), 5) for k, v in res.items()}})


if __name__ == "__main__":
    assert torch.cuda.is_available(), "perf_unipc.py measures on a CUDA device"
    torch.manual_seed(0)
    with torch.no_grad():
        if "kernels" in PARTS:
            kernels()
        if "error" in PARTS:
            error()
        if "steps" in PARTS:
            steps()
