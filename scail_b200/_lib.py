"""ctypes binding of libscail_b200.so (C ABI: include/scail_b200.h).

Follows the reference's only ctypes-kernel precedent (sat/quantization/kernels.py:70-121):
outputs are allocated by the caller with torch.empty, pointers are passed as c_void_p(data_ptr),
kernels launch on torch.cuda.current_stream().
"""
import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
# SCAIL_LIB_VARIANT=<tag> loads libscail_b200_<tag>.so instead (kernel A/B experiments under scripts/; never set in product use)
_VARIANT = os.environ.get("SCAIL_LIB_VARIANT", "")
LIB_PATH = os.path.join(_HERE, f"libscail_b200_{_VARIANT}.so" if _VARIANT else "libscail_b200.so")
CSRC = os.path.join(_HERE, "csrc")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]

c_p, c_i64, c_int, c_f = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float

# name -> argtypes; must list every symbol declared in include/scail_b200.h (tests check this)
SIGNATURES = {
    "scail_version": [],
    "scail_device_sm_count": [c_int],
    "scail_gemm_bf16": [c_p, c_i64, c_p, c_i64, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_int, c_p, c_i64, c_i64, c_p,
                        c_i64, c_int, c_p],
    "scail_gemm_fp8": [c_p, c_i64, c_p, c_i64, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_int, c_p, c_i64, c_i64, c_p,
                       c_i64, c_int, c_p, c_p, c_p],
    "scail_quant_rows_fp8": [c_p, c_i64, c_p, c_p, c_i64, c_i64, c_p],
    "scail_ln_modulate": [c_p, c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_f, c_p],
    "scail_ln_modulate_fp8": [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_f, c_p],
    "scail_rmsnorm_rope": [c_p, c_i64, c_i64, c_i64, c_i64, c_int, c_i64, c_p, c_i64, c_p, c_p, c_p, c_f, c_p],
    "scail_attention": [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                        c_i64, c_i64, c_f, c_int, c_p],
    "scail_attention_partial": [c_p, c_i64, c_p, c_i64, c_p, c_i64, c_p, c_i64, c_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                                c_i64, c_i64, c_i64, c_i64, c_i64, c_f, c_p],
    "scail_attention_merge": [c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_p],
    "scail_cp_unique_id": [c_p, ctypes.c_char_p],
    "scail_cp_init": [c_p, c_int, c_int, ctypes.c_char_p],
    "scail_cp_allgather": [c_int, c_p, c_p, c_i64, c_p],
    "scail_cp_wait": [c_int, c_p],
    "scail_cp_destroy": [c_int],
    "scail_adaln_modulation": [c_p, c_p, c_p, c_i64, c_i64, c_p],
    "scail_silu": [c_p, c_p, c_i64, c_p],
    "scail_timestep_embedding": [c_p, c_p, c_i64, c_i64, c_p],
    "scail_patchify": [c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_p],
    "scail_unpatchify": [c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_p],
    "scail_cfg_euler": [c_p, c_p, c_i64, c_f, c_f, c_p],
    "scail_cast_f32_bf16": [c_p, c_p, c_i64, c_p],
    "scail_conv3d_cl": [c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_i64, c_int, c_int, c_int, c_p, c_p, c_i64, c_p, c_i64,
                        c_i64, c_int, c_int, c_p, c_p, c_p],
    "scail_conv3d_strided_cl": [c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_i64, c_int, c_int, c_int, c_p, c_p, c_i64, c_i64,
                                c_i64, c_i64, c_int, c_int, c_int, c_int, c_int, c_p],
    "scail_conv3d_cl_hist": [c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_i64, c_int, c_int, c_int, c_p, c_p, c_i64, c_p, c_i64,
                             c_i64, c_int, c_int, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_p],
    "scail_conv3d_strided_cl_hist": [c_p, c_i64, c_i64, c_i64, c_i64, c_p, c_i64, c_int, c_int, c_int, c_p, c_p, c_i64, c_i64,
                                     c_i64, c_i64, c_int, c_int, c_int, c_int, c_int, c_p, c_i64, c_p],
    "scail_rmsnorm_cl": [c_p, c_p, c_p, c_i64, c_i64, c_int, c_p],
    "scail_upsample2x_cl": [c_p, c_p, c_i64, c_i64, c_i64, c_i64, c_p],
    "scail_vae_latent_to_cl": [c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_p],
    "scail_softmax_rows": [c_p, c_p, c_i64, c_i64, c_f, c_p],
}


def sources():
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))]


def needs_build():
    if _VARIANT:
        return False
    if not os.path.isfile(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    hdr = os.path.join(os.path.dirname(_HERE), "include", "scail_b200.h")
    return any(os.path.getmtime(s) > t for s in sources() + [hdr])


def build(force=False, verbose=False):
    """Compile the CUDA extension in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    if not force and not needs_build():
        return LIB_PATH
    extra = os.environ.get("SCAIL_NVCC_EXTRA", "").split()  # extra nvcc flags for experiments, e.g. -DSCAIL_MBAR_DEBUG
    cmd = ["nvcc", *NVCC_FLAGS, *extra, "-o", LIB_PATH, os.path.join(CSRC, "api.cu"), "-lcudart", "-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB_PATH


_lib = None


def lib():
    """Load the library (building it first if sources are newer and nvcc exists). Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if needs_build():
        try:
            build()
        except FileNotFoundError as e:  # no nvcc
            if not os.path.isfile(LIB_PATH):
                raise RuntimeError("libscail_b200.so is missing and nvcc is not available to build it") from e
    h = ctypes.CDLL(LIB_PATH)
    h.scail_last_error.restype = ctypes.c_char_p
    h.scail_last_error.argtypes = []
    for name, args in SIGNATURES.items():
        if _VARIANT and not hasattr(h, name):
            continue  # experiment builds (scripts/build_variants.sh) may predate an entry point
        fn = getattr(h, name)
        fn.argtypes = args
        fn.restype = c_int
    _lib = h
    return h


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"{what} failed ({rc}): {lib().scail_last_error().decode()}")
