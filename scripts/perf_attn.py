"""Self-attention at the SCAIL-14B shape (b=2, 40 heads, N=27904 by default; N=... env for config B): CUDA-event timing of
scail_attention, torch SDPA (cuDNN/flash) beside it, and the relL2 between the two outputs.  SCAIL_LIB_VARIANT picks an
A/B build of the library (scripts/build_variants.sh).
FP8=1: instead, the fp8 self-attention against bf16, alternated REPS times in this process: the bf16 arm is
rmsnorm_rope + scail_attention, the fp8 arm rmsnorm_rope(out_fp8) + quant_vt_fp8 + attention_fp8; each kernel is also timed
alone.  Prints the card's name and power limit and TFLOP/s against the 1979 (e4m3) / 989 (bf16) TFLOP/s data-sheet peaks."""
import json, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scail_b200 import ops
B, H, N, d = int(os.environ.get("B", 2)), 40, int(os.environ.get("N", 27904)), 5120
torch.manual_seed(0)
qkv = torch.randn(B * N, 3 * d, device="cuda", dtype=torch.bfloat16)
out = torch.empty(B * N, d, device="cuda", dtype=torch.bfloat16)
f = lambda: ops.attention(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], out, B, H, N, N)


def timeit(fn, iters=5):
    fn(); fn(); torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / iters




def fp8_arms():
    import subprocess
    Lp = ops.fp8_pad(N)
    w = torch.randn(2, d, device="cuda", dtype=torch.bfloat16) * 0.1 + 1
    ang = torch.rand(N, 128, device="cuda") * 6.3
    cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
    q8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
    k8 = (torch.empty(B * N, d, device="cuda", dtype=ops.FP8), torch.empty(B, H, Lp, device="cuda"))
    vt = torch.empty(B, H, 128, Lp, device="cuda", dtype=ops.FP8)
    vs = torch.empty(B, H, 128, device="cuda")
    work = torch.empty(B, d, device="cuda", dtype=torch.int32)
    slabs = [(0, w[0]), (d, w[1])]
    rope8 = lambda: ops.rmsnorm_rope(qkv, N, d, slabs, cos, sin, out_fp8=[q8, k8])
    vt8 = lambda: ops.quant_vt_fp8(qkv[:, 2 * d:], B, H, N, vt, vs, work)
    att8 = lambda: ops.attention_fp8(q8[0], q8[1], k8[0], k8[1], vt, vs, out, B, H, N)
    qkv_copy = qkv.clone()  # the bf16 RMSNorm+RoPE works in place: on a copy, so every round sees the same inputs
    rope16 = lambda: ops.rmsnorm_rope(qkv_copy, N, d, slabs, cos, sin)
    arms = {"bf16_rmsnorm_rope": rope16, "bf16_attention": f, "bf16_total": lambda: (rope16(), f()),
            "fp8_rmsnorm_rope": rope8, "fp8_quant_vt": vt8, "fp8_attention": att8, "fp8_total": lambda: (rope8(), vt8(), att8())}
    ms = {k: [] for k in arms}
    for _ in range(int(os.environ.get("REPS", 3))):
        for k, fn in arms.items():
            ms[k].append(round(timeit(fn), 3))
    best = {k: min(v) for k, v in ms.items()}
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = ""
    fl = 4 * B * H * N * N * 128
    return dict(B=B, N=N, ms=ms, fp8_over_bf16_total=round(best["fp8_total"] / best["bf16_total"], 3),
                fp8_attention_tflops=round(fl / best["fp8_attention"] / 1e9, 1),
                fp8_attention_share_of_e4m3_peak=round(fl / best["fp8_attention"] / 1e9 / 1979, 3),
                bf16_attention_tflops=round(fl / best["bf16_attention"] / 1e9, 1),
                gpu=torch.cuda.get_device_name(), nvidia_smi=smi)


def bf16_arm():
    ms = timeit(f)
    fl = 4 * B * H * N * N * 128
    res = dict(variant=os.environ.get("SCAIL_LIB_VARIANT", "product"), B=B, N=N, ms=round(ms, 3), tflops=round(fl / ms / 1e9, 1))
    if os.environ.get("SDPA", "1") == "1":
        q4 = qkv.view(B, N, 3, H, 128)
        qh, kh, vh = (q4[:, :, i].transpose(1, 2) for i in range(3))
        g = lambda: torch.nn.functional.scaled_dot_product_attention(qh, kh, vh)
        ms_t = timeit(g, 3)
        ref = g().transpose(1, 2).reshape(B * N, d)
        f(); torch.cuda.synchronize()
        rel = float((out.float() - ref.float()).norm() / ref.float().norm())
        res.update(torch_sdpa_ms=round(ms_t, 3), torch_sdpa_tflops=round(fl / ms_t / 1e9, 1), rel_vs_sdpa=rel)
    return res


res = fp8_arms() if os.environ.get("FP8") == "1" else bf16_arm()
print(json.dumps(res), flush=True)
os.makedirs("gpurun_out", exist_ok=True)
open("gpurun_out/perf_attn.jsonl", "a").write(json.dumps(res) + "\n")
