"""GEMM timing at the 14B step's shapes (M = 2 x 27904), CUDA events over `ITERS` back-to-back launches (default 40: long
enough for the power cap to settle).  Prints one JSON line per result, with the card's name and power limit.

  SHAPE=qkv|attn_out|cross_q|cross_out|fc1|fc2   one per-block GEMM, ours and F.linear alternating (REPS rounds)
  SHAPE=all                                       the six per-block GEMMs, then the K sweep
  SHAPE=ksweep                                    out-projection N and epilogue at K = 5120 and 13824: fits the cost of a
                                                  k-block and the per-tile cost that does not depend on K
Knob: SCAIL_GEMM_GROUP_M (rasterisation group).  SCAIL_LIB_VARIANT picks another build of the library (A/B runs)."""
import json, os, subprocess, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scail_b200 import ops

d, f, n = 5120, 13824, 27904
M = 2 * n
SHAPES = {"qkv": (3 * d, d, ops.EPI_BIAS), "attn_out": (d, d, ops.EPI_BIAS_GATE_RES), "cross_q": (d, d, ops.EPI_BIAS),
          "cross_out": (d, d, ops.EPI_BIAS_RES), "fc1": (f, d, ops.EPI_BIAS_GELU), "fc2": (d, f, ops.EPI_BIAS_GATE_RES)}
ITERS = int(os.environ.get("ITERS", 40))
REPS = int(os.environ.get("REPS", 2))
TILE_M, TILE_N = 128, 256


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q, "variant": os.environ.get("SCAIL_LIB_VARIANT", "")}


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


def operands(N, K, epi):
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    w = torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * K ** -0.5
    b = torch.randn(N, device="cuda", dtype=torch.bfloat16)
    out = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    kw = {}
    if epi == ops.EPI_BIAS_GATE_RES:
        kw = dict(gate=torch.randn(2, N, device="cuda", dtype=torch.bfloat16), residual=out, rows_per_batch=n)
    elif epi == ops.EPI_BIAS_RES:
        kw = dict(residual=out)
    return a, w, b, out, kw


def shape(name):
    N, K, epi = SHAPES[name]
    a, w, b, out, kw = operands(N, K, epi)
    ours, lib = [], []
    for _ in range(REPS):  # alternate, so that clock and neighbour drift hit both alike
        ours.append(timed(lambda: ops.gemm(a, w, b, out=out, epilogue=epi, **kw)))
        lib.append(timed(lambda: torch.nn.functional.linear(a, w, b)))
    ms, ms_t = min(ours), min(lib)
    return dict(shape=name, M=M, N=N, K=K, epilogue=epi, ours_ms=[round(x, 3) for x in ours],
                cublas_ms=[round(x, 3) for x in lib], ours_tflops=round(2 * M * N * K / ms / 1e9, 1),
                ours_over_cublas=round(ms_t / ms, 3))


def ksweep():
    """Same N, epilogue and tile count at two K: per wave, time = intercept + k_blocks * per_k_block."""
    N, _, epi = SHAPES["attn_out"]
    waves = -(-M // TILE_M) * -(-N // TILE_N) / torch.cuda.get_device_properties(0).multi_processor_count
    per_wave = {}
    for K in (d, f):
        a, w, b, out, kw = operands(N, K, epi)
        per_wave[K] = min(timed(lambda: ops.gemm(a, w, b, out=out, epilogue=epi, **kw)) for _ in range(REPS)) / waves * 1e3
        del a, w, b, out, kw
    kb1, kb2 = d // 64, f // 64
    slope = (per_wave[f] - per_wave[d]) / (kb2 - kb1)
    return dict(shape="ksweep", N=N, epilogue=epi, waves=round(waves, 2),
                per_wave_us={str(k): round(v, 1) for k, v in per_wave.items()},
                per_k_block_us=round(slope, 3), per_tile_intercept_us=round(per_wave[d] - kb1 * slope, 1))


def main():
    which = os.environ.get("SHAPE", "qkv")
    info = card()
    names = list(SHAPES) + ["ksweep"] if which == "all" else [which]
    for name in names:
        res = ksweep() if name == "ksweep" else shape(name)
        res.update(info)
        print(json.dumps(res), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
