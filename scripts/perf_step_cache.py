"""First-block residual cache (scail_b200.step_cache) on bench.py's 14B model and inputs (512 x 512, 40 blocks, CFG batch 2).
Prints one JSON line per result with the card's name and power limit; OUT=<dir> also appends them to
<dir>/perf_step_cache.jsonl (nothing is written otherwise).

  steps:   ms per sampler step, dense bf16 and window 2, each eager (sampler_step) and with GraphedStep, for
           (a) no cache, (b) threshold 0 (a computed step with the cache) and (c) threshold inf after one computed step (a
           skipped step).  The three arms alternate inside each of ROUNDS rounds (default 3), STEPS timed steps each (default
           2); best and median over rounds.  Also whether the latents of (a) and (b) are bit-identical.
  kernels: ms and GB/s of the three cache kernels at b = 2, N = 27 904, d = 5120 against 3.35 TB/s (ITERS launches).
  trace:   the indicator of a 50-step sample at threshold 0 (window 2, GraphedStep).  The weights are random, so this says
           nothing about the skip rate real weights would give.
PARTS=steps,kernels,trace selects parts."""
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
from scail_b200 import ops  # noqa: E402

ROUNDS = int(os.environ.get("ROUNDS", 3))
STEPS = int(os.environ.get("STEPS", 2))
ITERS = int(os.environ.get("ITERS", 20))
PARTS = os.environ.get("PARTS", "steps,kernels,trace").split(",")
HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
WORKLOAD = "SCAIL-14B, 40 blocks, latent 21x64x64 (512x512), CFG batch 2"


def emit(line):
    line = {**line, **card()}
    print(json.dumps(line), flush=True)
    out = os.environ.get("OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "perf_step_cache.jsonl"), "a") as f:
            f.write(json.dumps(line) + "\n")


def setup():
    import bench
    from scail_b200 import sampler
    m = bench.build_model("cuda")
    h = bench.synthetic_inputs()
    dv = {k: v.cuda() for k, v in h.items()}
    cond = dict(crossattn=dv["context_cond"], ref_concat=dv["ref_concat"], concat_smpl_render=dv["concat_smpl_render"],
                image_clip_features=dv["image_clip_features"])
    uc = dict(crossattn=dv["context_uncond"])
    return m, dv["x"], cond, uc, sampler.make_flow_timesteps(50, 5.0)


def steps(m, x0, cond, uc, sig):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    ad = m.mixins["adaln_layer"]
    for window in (None, 2):
        ad.attention_window = window
        for graphed in (False, True):
            c = FirstBlockCache(0.0)
            xa, xb = x0.clone(), x0.clone()
            if graphed:
                g_plain = sampler.GraphedStep(m, xa, cond, uc, 4.0)
                g_cache = sampler.GraphedStep(m, xb, cond, uc, 4.0, step_cache=c)
                run_a = lambda i: g_plain(sig[i], sig[i + 1])
                run_c = lambda i: g_cache(sig[i], sig[i + 1])
            else:
                run_a = lambda i: sampler.sampler_step(m, xa, sig[i], sig[i + 1], cond, uc, 4.0)
                run_c = lambda i: sampler.sampler_step(m, xb, sig[i], sig[i + 1], cond, uc, 4.0, step_cache=c)
            # (a) and (b) take the same steps from the same latent: their latents must stay bit-identical.  (c) continues from
            # (b)'s state with threshold inf, then (b)'s next round computes again (threshold 0).
            res = {"a_no_cache": [], "b_threshold_0": [], "c_threshold_inf": []}
            c.threshold = 0.0
            run_a(10), run_c(10)  # warm-up; gives the cache its first computed step
            torch.cuda.synchronize()
            equal, i = True, 11
            for _ in range(ROUNDS):
                for arm, thr in (("a_no_cache", None), ("b_threshold_0", 0.0), ("c_threshold_inf", float("inf"))):
                    if thr is not None:
                        c.threshold = thr
                    t0 = time.perf_counter()
                    for k in range(STEPS):
                        (run_a if thr is None else run_c)(i + k)
                    torch.cuda.synchronize()
                    res[arm].append(round((time.perf_counter() - t0) * 1000.0 / STEPS, 2))
                    if arm == "b_threshold_0":
                        equal = equal and torch.equal(xa, xb)
                        xb.copy_(xa)  # (c) then starts from the same latent; the cache state is (b)'s last computed step
                i += STEPS
                xb.copy_(xa)
            skipped = [s for _, s in c.history]
            assert skipped.count(True) == ROUNDS * STEPS, skipped
            best = {k: min(v) for k, v in res.items()}
            med = {k: statistics.median(v) for k, v in res.items()}
            emit({"part": "steps", "attention_window": window, "graphed": graphed, "ms_per_step": res, "best_ms": best,
                  "median_ms": med, "overhead_b_over_a_best": round(best["b_threshold_0"] / best["a_no_cache"] - 1, 5),
                  "overhead_b_over_a_median": round(med["b_threshold_0"] / med["a_no_cache"] - 1, 5),
                  "a_spread": round((max(res["a_no_cache"]) - min(res["a_no_cache"])) / min(res["a_no_cache"]), 5),
                  "skip_cost_c_over_b_best": round(best["c_threshold_inf"] / best["b_threshold_0"], 5),
                  "latents_a_b_bit_identical": bool(equal), "rounds": ROUNDS, "steps_per_round": STEPS, "workload": WORKLOAD})
            del c
            if graphed:
                del g_plain, g_cache
            torch.cuda.empty_cache()
    ad.attention_window = None


def kernels():
    B, N, d, n_ref, n_seq = 2, 27904, 5120, 1024, 21504
    bf = torch.bfloat16
    h0 = torch.randn(B, N, d, device="cuda", dtype=bf)
    h1 = torch.randn(B, N, d, device="cuda", dtype=bf)
    r_ref = torch.randn(B, N, d, device="cuda", dtype=bf)
    r_new, h1c = torch.empty_like(h0), torch.empty(B, n_seq, d, device="cuda", dtype=bf)
    R = torch.empty(B, n_seq, d, device="cuda", dtype=torch.float32)
    partials = torch.empty(ops.STEP_CACHE_PARTIALS, device="cuda", dtype=torch.float32)
    out = torch.empty(4, device="cuda", dtype=torch.float64)
    E, En = B * N * d, B * n_seq * d
    arms = {  # name: (launch, bytes moved)
        "indicator": (lambda: ops.step_cache_indicator(h0, h1, r_ref, r_new, h1c, n_ref, partials, out), 3 * E * 2 + E * 2 + En * 2),
        "update": (lambda: ops.step_cache_update(h1, h1c, R, n_ref), En * 2 * 2 + En * 4),
        "apply": (lambda: ops.step_cache_apply(h1, R, n_ref), En * 2 * 2 + En * 4),
    }
    res = {k: [] for k in arms}
    for _ in range(ROUNDS):
        for k, (fn, _) in arms.items():
            fn(); fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(ITERS):
                fn()
            e.record()
            torch.cuda.synchronize()
            res[k].append(s.elapsed_time(e) / ITERS)
    for k, (_, nbytes) in arms.items():
        ms = min(res[k])
        emit({"part": "kernels", "kernel": k, "B": B, "N": N, "d": d, "n_seq": n_seq, "ms_best": round(ms, 4),
              "ms_rounds": [round(v, 4) for v in res[k]], "bytes": nbytes, "GB_per_s": round(nbytes / ms / 1e6, 1),
              "fraction_of_3.35TB_per_s": round(nbytes / ms / 1e-3 / HBM_PEAK, 3)})


def trace(m, x0, cond, uc, sig):
    from scail_b200 import sampler
    from scail_b200.step_cache import FirstBlockCache
    m.mixins["adaln_layer"].attention_window = 2
    c = FirstBlockCache(0.0)
    x = x0.clone()
    g = sampler.GraphedStep(m, x, cond, uc, 4.0, step_cache=c)
    t0 = time.perf_counter()
    for i in range(50):
        g(sig[i], sig[i + 1])
    torch.cuda.synchronize()
    emit({"part": "trace", "attention_window": 2, "threshold": 0.0, "indicator": [round(v, 6) for v, _ in c.history],
          "s_total": round(time.perf_counter() - t0, 2), "note": "random weights: says nothing about the skip rate of real weights",
          "workload": WORKLOAD})
    m.mixins["adaln_layer"].attention_window = None


if __name__ == "__main__":
    assert torch.cuda.is_available(), "perf_step_cache.py measures on a CUDA device"
    torch.manual_seed(0)
    with torch.no_grad():
        if "kernels" in PARTS:
            kernels()
            torch.cuda.empty_cache()
        if "steps" in PARTS or "trace" in PARTS:
            args = setup()
            if "steps" in PARTS:
                steps(*args)
            if "trace" in PARTS:
                trace(*args)
