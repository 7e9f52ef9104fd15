"""CFG-Zero* guidance (scail_b200.guidance): kernel cost and sampler cost.  Prints one JSON line per result with the card's
name and power limit; OUT=<dir> also appends them to <dir>/perf_cfg_zero.jsonl (nothing is written otherwise).

  kernels: ms and GB/s at the 512x512, 480x832 and 512x896 latents (21 latent frames) against 3.35 TB/s, each launch timed
           after an L2 flush, best of ROUNDS rounds of the mean over ITERS launches (perf_unipc.cold_ms):
             scale       the s* reduction on the CFG pair, pass 1 + pass 2 (reads the bf16 pair);
             euler       cfg_euler_ (reads x and the pair, writes x) against its scaled form (also reads s*);
             unipc_2     unipc_step_ at order 2, both slots in use (reads x, x_last, the pair and 2 slots; writes x, x_last
                         and one slot), against its scaled form.
  steps:   steps/s of bench.py's 14B model at 512x512 (40 blocks, CFG batch 2) over a 10-step eager sample(), guidance=None
           against CFGZeroStar(0) and CFGZeroStar(1), the three arms alternating in each of ROUNDS rounds.  Expected, not
           measured here: CFGZeroStar(0) costs what None costs within the spread, and CFGZeroStar(1) saves about one
           forward in ten.
PARTS=kernels,steps selects parts (default both)."""
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import perf_unipc  # noqa: E402
from perf_fp8 import card  # noqa: E402
from scail_b200 import ops, sampler, unipc  # noqa: E402
from scail_b200.guidance import CFGZeroStar  # noqa: E402

ROUNDS = int(os.environ.get("ROUNDS", 3))
PARTS = os.environ.get("PARTS", "kernels,steps").split(",")
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
LATENTS = perf_unipc.LATENTS


def emit(line):
    line = {**line, **card()}
    print(json.dumps(line), flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "perf_cfg_zero.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def _row(name, shape, kernel, nbytes, ms, rounds):
    return {"part": "kernels", "latent": name, "shape": list(shape), "kernel": kernel, "ms_best": round(ms, 4),
            "ms_rounds": [round(r, 4) for r in rounds], "bytes": nbytes, "GB_per_s": round(nbytes / ms / 1e6, 1),
            "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)}


def kernels():
    sig = unipc.check_schedule(sampler.make_flow_timesteps(50, 5.0))
    i = 25
    k = unipc.step_coefficients(sig, i, 2)
    coef = [float(c) for c in torch.tensor([k.x_last_c, *k.slot_c, 0.0, k.m_c, k.y_c, *k.slot_p, 0.0, k.m_p])]
    for name, shape in LATENTS.items():
        n = 1
        for s in shape:
            n *= s
        x, xl = torch.randn(shape, device="cuda"), torch.randn(shape, device="cuda")
        v = torch.randn(2, *shape[1:], device="cuda").to(torch.bfloat16)
        slots = torch.randn(2, n, device="cuda")
        g = CFGZeroStar(0)
        s = g.scale(v)
        ms, r = perf_unipc.cold_ms(lambda: g.scale(v))
        emit(_row(name, shape, "scale (pass 1 + pass 2)", n * 4, ms, r))
        # x grows over the repeated in-place launches; finite or not, the cost is the same
        for kern, fn in (("euler", lambda: ops.cfg_euler_(x, v, 4.0, -0.02)),
                         ("euler_scaled", lambda: ops.cfg_euler_(x, v, 4.0, -0.02, u_scale=s))):
            ms, r = perf_unipc.cold_ms(fn)
            emit(_row(name, shape, kern, n * 12, ms, r))
        for kern, fn in (("unipc_2", lambda: ops.unipc_step_(x, xl, v, slots, k.write, 4.0, sig[i], coef, True)),
                         ("unipc_2_scaled", lambda: ops.unipc_step_(x, xl, v, slots, k.write, 4.0, sig[i], coef, True,
                                                                    u_scale=s))):
            ms, r = perf_unipc.cold_ms(fn)
            emit(_row(name, shape, kern, n * (4 + 4 + 4 + 4 * 2) + n * 12, ms, r))
        del x, xl, v, slots, g, s
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
    arms = {"none": None, "cfg_zero_star_0": CFGZeroStar(0), "cfg_zero_star_1": CFGZeroStar(1)}
    for g in arms.values():  # warm-up of every update path
        sampler.sample(m, dv["x"].clone(), cond, uc, num_steps=2, guidance=g)
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for name, g in arms.items():
            x = dv["x"].clone()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sampler.sample(m, x, cond, uc, num_steps=n, guidance=g)
            torch.cuda.synchronize()
            res[name].append(round(n / (time.perf_counter() - t0), 5))
    med = {k: statistics.median(v) for k, v in res.items()}
    emit({"part": "steps", "workload": "SCAIL-14B, 40 blocks, latent 21x64x64 (512x512), CFG batch 2, eager sample()",
          "steps": n, "rounds": ROUNDS, "steps_per_s": res, "median_steps_per_s": med,
          "k0_over_none_median": round(med["cfg_zero_star_0"] / med["none"] - 1, 5),
          "k1_over_none_median": round(med["cfg_zero_star_1"] / med["none"] - 1, 5),
          "spread": {k: round((max(v) - min(v)) / min(v), 5) for k, v in res.items()}})


if __name__ == "__main__":
    assert torch.cuda.is_available(), "perf_cfg_zero.py measures on a CUDA device"
    torch.manual_seed(0)
    with torch.no_grad():
        if "kernels" in PARTS:
            kernels()
        if "steps" in PARTS:
            steps()
