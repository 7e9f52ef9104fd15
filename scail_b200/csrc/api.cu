// C ABI of libscail_b200.so (see include/scail_b200.h).  Host-side launch code: argument checks,
// TMA descriptor cache, kernel launches on the caller's stream.  No CPU fallback anywhere.
#include <cuda.h>
#include <cuda_runtime.h>

#include <dlfcn.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "../../include/scail_b200.h"
#include "adaptive.cuh"
#include "apg.cuh"
#include "attention.cuh"
#include "cfg_cache.cuh"
#include "cfg_zero.cuh"
#include "conv.cuh"
#include "gemm.cuh"
#include "rowops.cuh"
#include "solver.cuh"
#include "step_cache.cuh"

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

#define SCAIL_CHECK_CUDA(expr)                                                              \
    do {                                                                                    \
        cudaError_t _e = (expr);                                                            \
        if (_e != cudaSuccess) return fail(-2, "%s: %s", #expr, cudaGetErrorString(_e));   \
    } while (0)

#define SCAIL_REQUIRE(cond, ...)                   \
    do {                                           \
        if (!(cond)) return fail(-1, __VA_ARGS__); \
    } while (0)

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

struct MapKey {
    const void* ptr;
    uint64_t rows, cols, ld;
    uint32_t box_rows, box_cols;
    uint32_t esize;
    bool operator==(const MapKey& o) const {
        return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows &&
               box_cols == o.box_cols && esize == o.esize;
    }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = reinterpret_cast<size_t>(k.ptr);
        auto mix = [&](uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix(k.rows); mix(k.cols); mix(k.ld); mix(k.box_rows); mix(k.box_cols); mix(k.esize);
        return h;
    }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// 2-D row-major [rows, cols] with leading dimension ld (elements) of bf16 (esize 2), fp32 (4) or bytes (1: e4m3);
// box = [box_rows, box_cols], box_cols * esize == 128 bytes (SWIZZLE_128B).  Out-of-bounds elements are zero-filled on loads
// and not written by stores.
int make_tmap_2d(const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, uint32_t box_cols,
                 CUtensorMap* out, uint32_t esize = 2) {
    MapKey key{ptr, rows, cols, ld, box_rows, box_cols, esize};
    const CUtensorMapDataType dtype = esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                      : esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        auto it = g_maps.find(key);
        if (it != g_maps.end()) {
            *out = it->second;
            return 0;
        }
    }
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return fail(-3, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * esize) & 15)) return fail(-1, "TMA operand must be 16-byte aligned (ptr=%p ld=%llu)", ptr, (unsigned long long)ld);
    cuuint64_t gdim[2] = {cols, rows};
    cuuint64_t gstride[1] = {ld * esize};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, dtype, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(-3, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu ld=%llu box=%ux%u", (int)r,
                                        (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld, box_rows, box_cols);
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        if (g_maps.size() > 8192) g_maps.clear();
        g_maps[key] = m;
    }
    *out = m;
    return 0;
}

// 4-D bf16 channels-last activation [T, H, W, C]: dims (C, W, H, T), box (64, 16, 8, 1), SWIZZLE_128B.
// Out-of-bounds box elements (channel tail, spatial halo, t < 0) are zero-filled.
struct Map4Key {
    const void* ptr; uint64_t T, H, W, C; uint32_t bw, bh, es;
    bool operator==(const Map4Key& o) const { return ptr == o.ptr && T == o.T && H == o.H && W == o.W && C == o.C && bw == o.bw && bh == o.bh && es == o.es; }
};
struct Map4KeyHash {
    size_t operator()(const Map4Key& k) const {
        size_t h = reinterpret_cast<size_t>(k.ptr);
        auto mix = [&](uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
        mix(k.T); mix(k.H); mix(k.W); mix(k.C); mix(k.bw); mix(k.bh); mix(k.es);
        return h;
    }
};
std::unordered_map<Map4Key, CUtensorMap, Map4KeyHash> g_maps4;

int make_tmap_cl4d(const void* ptr, uint64_t T, uint64_t H, uint64_t W, uint64_t C, CUtensorMap* out, uint32_t box_w = 16,
                   uint32_t box_h = 8, uint32_t estride = 1) {
    // estride = 2: the box spans box_w x box_h input pixels but only every second one is fetched (stride-2 conv)
    Map4Key key{ptr, T, H, W, C, box_w, box_h, estride};
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        auto it = g_maps4.find(key);
        if (it != g_maps4.end()) { *out = it->second; return 0; }
    }
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) return fail(-3, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (C % 8)) return fail(-1, "conv input must be 16-byte aligned with C %% 8 == 0");
    cuuint64_t gdim[4] = {C, W, H, T};
    cuuint64_t gstride[3] = {C * 2, W * C * 2, H * W * C * 2};
    cuuint32_t box[4] = {64, box_w, box_h, 1};
    cuuint32_t estr[4] = {1, estride, estride, 1};
    CUtensorMap m;
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), gdim, gstride, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(-3, "cuTensorMapEncodeTiled(4d) failed (%d) T=%llu H=%llu W=%llu C=%llu", (int)r,
                                        (unsigned long long)T, (unsigned long long)H, (unsigned long long)W, (unsigned long long)C);
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        if (g_maps4.size() > 4096) g_maps4.clear();
        g_maps4[key] = m;
    }
    *out = m;
    return 0;
}

constexpr int MAX_DEVICES = 64;
int g_sm_count[MAX_DEVICES] = {0};  // per device: a process may drive several GPUs
int sm_count() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEVICES) return 0;
    if (g_sm_count[dev] == 0) cudaDeviceGetAttribute(&g_sm_count[dev], cudaDevAttrMultiProcessorCount, dev);
    return g_sm_count[dev];
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

struct SmemKey {
    const void* fn; int dev;
    bool operator==(const SmemKey& o) const { return fn == o.fn && dev == o.dev; }
};
struct SmemKeyHash {
    size_t operator()(const SmemKey& k) const { return reinterpret_cast<size_t>(k.fn) * 31u + static_cast<size_t>(k.dev); }
};
std::unordered_map<SmemKey, cudaError_t, SmemKeyHash> g_smem_done;  // MaxDynamicSharedMemorySize is a per-device function attribute
template <typename K>
int set_smem(K kernel, int bytes) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(-2, "no current CUDA device");
    const SmemKey key{reinterpret_cast<const void*>(kernel), dev};
    cudaError_t err;
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        auto it = g_smem_done.find(key);
        if (it == g_smem_done.end()) {
            err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
            g_smem_done[key] = err;
        } else {
            err = it->second;
        }
    }
    return err == cudaSuccess ? 0 : fail(-2, "cudaFuncSetAttribute(smem=%d): %s", bytes, cudaGetErrorString(err));
}

inline int blocks_for(int64_t n, int per) { return static_cast<int>((n + per - 1) / per); }

template <int BN>
static int launch_conv(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& th, const scail::ConvParams& p,
                       cudaStream_t st) {
    using namespace scail;
    int rc;
    if ((rc = set_smem(conv3d_kernel<BN>, ConvCfg<BN>::SMEM_BYTES))) return rc;
    const int tiles = p.T * blocks_for(p.H, CONV_PH) * blocks_for(p.W, CONV_PW) * blocks_for(p.Cout, BN);
    const int sms = sm_count();
    if (sms <= 0) return fail(-2, "conv3d: no CUDA device");
    conv3d_kernel<BN><<<tiles < sms ? tiles : sms, CONV_THREADS, ConvCfg<BN>::SMEM_BYTES, st>>>(tx, tw, th, p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int EPI, bool F32>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tc, const CUtensorMap& tr,
                       const scail::GemmParams& p, int grid, cudaStream_t st) {
    using namespace scail;
    int rc;
    if ((rc = set_smem(gemm_bf16_kernel<EPI, F32>, GEMM_SMEM_BYTES))) return rc;
    gemm_bf16_kernel<EPI, F32><<<grid, GEMM_THREADS, GEMM_SMEM_BYTES, st>>>(ta, tw, tc, tr, p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// OP: GEMM_OP_E4M3 (gemm_fp8_kernel) or GEMM_OP_INT8 (gemm_int8_kernel)
template <int OP, int EPI>
static int launch_gemm_scaled(const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tc, const CUtensorMap& tr,
                              const scail::GemmParams& p, int grid, cudaStream_t st) {
    using namespace scail;
    constexpr int smem = GemmCfg<OP>::SMEM_BYTES;
    auto kernel = OP == GEMM_OP_INT8 ? gemm_int8_kernel<EPI> : gemm_fp8_kernel<EPI>;
    int rc;
    if ((rc = set_smem(kernel, smem))) return rc;
    kernel<<<grid, GEMM_THREADS, smem, st>>>(ta, tw, tc, tr, p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int LP, int VPL>
static int launch_rmsnorm_cl(const void* x, const void* gamma, void* out, int64_t npix, int C, int silu, cudaStream_t st) {
    const int pix_per_block = 8 * (32 / LP);
    const int grid = blocks_for(npix, pix_per_block);
    auto xp = static_cast<const __nv_bfloat16*>(x);
    auto gp = static_cast<const __nv_bfloat16*>(gamma);
    auto op = static_cast<__nv_bfloat16*>(out);
    if (silu) scail::rmsnorm_cl_kernel<true, LP, VPL><<<grid, 256, 0, st>>>(xp, gp, op, npix, C);
    else scail::rmsnorm_cl_kernel<false, LP, VPL><<<grid, 256, 0, st>>>(xp, gp, op, npix, C);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace

extern "C" {

const char* scail_last_error(void) { return g_err; }
int scail_version(void) { return 100; }

int scail_device_sm_count(int device) {
    int n = 0;
    cudaError_t e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
    if (e != cudaSuccess) return fail(-2, "no usable CUDA device: %s", cudaGetErrorString(e));
    return n;
}

int scail_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                    int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                    int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(A && W && C, "gemm: null operand");
    SCAIL_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
    SCAIL_REQUIRE(N % 8 == 0 && K % 8 == 0 && lda % 8 == 0 && ldw % 8 == 0 && ldc % (c_fp32 ? 4 : 8) == 0,
                  "gemm: N, K, lda, ldw (and ldc for a bf16 output; ldc %% 4 for fp32) must be multiples of 8");
    SCAIL_REQUIRE(aligned16(C) && aligned16(bias) && aligned16(gate) && aligned16(residual),
                  "gemm: C, bias, gate and residual must be 16-byte aligned (the epilogue uses 16-byte accesses)");
    SCAIL_REQUIRE(epilogue >= 0 && epilogue <= 5, "gemm: unknown epilogue %d", epilogue);
    if (epilogue == EPI_BIAS_GATE_RES) SCAIL_REQUIRE(gate && residual && gate_stride % 8 == 0, "gemm: gate/residual required");
    if (epilogue == EPI_BIAS_RES) SCAIL_REQUIRE(residual, "gemm: residual required");
    if (residual) SCAIL_REQUIRE(ldr % 8 == 0, "gemm: ldr must be a multiple of 8");
    const bool res_epi = epilogue == EPI_BIAS_GATE_RES || epilogue == EPI_BIAS_RES;
    SCAIL_REQUIRE(!(c_fp32 && res_epi), "gemm: the residual epilogues write a bf16 output");
    CUtensorMap ta, tw, tc, tr;
    int rc;
    GemmParams p;
    p.M = (int)M; p.N = (int)N; p.K = (int)K;
    p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.gate = static_cast<const __nv_bfloat16*>(gate);
    p.gate_stride = gate_stride;
    p.rows_per_batch = rows_per_batch > 0 ? (int)rows_per_batch : (int)M;
    static const int gm_env = getenv("SCAIL_GEMM_GROUP_M") ? atoi(getenv("SCAIL_GEMM_GROUP_M")) : 0;
    const int sms = sm_count();
    SCAIL_REQUIRE(sms > 0, "gemm: no CUDA device");
    if ((rc = make_tmap_2d(A, M, K, lda, GEMM_BM, GEMM_BK, &ta))) return rc;
    if ((rc = make_tmap_2d(W, N, K, ldw, GEMM_BN, GEMM_BK, &tw))) return rc;
    // C (and the residual) in 64-row boxes of 128 bytes: one box per warpgroup and staging column chunk
    if ((rc = make_tmap_2d(C, M, N, ldc, 64, c_fp32 ? 32 : 64, &tc, c_fp32 ? 4 : 2))) return rc;
    if (res_epi) {
        if ((rc = make_tmap_2d(residual, M, N, ldr, 64, 64, &tr))) return rc;
    } else {
        tr = tc;  // unused
    }
    p.group_m = gm_env > 0 ? gm_env : 16;
    const int num_tiles = blocks_for(M, GEMM_BM) * blocks_for(N, GEMM_BN);
    const int grid = num_tiles < sms ? num_tiles : sms;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (epilogue) {
        case EPI_BIAS:
            return c_fp32 ? launch_gemm<EPI_BIAS, true>(ta, tw, tc, tr, p, grid, st)
                          : launch_gemm<EPI_BIAS, false>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GELU:
            return c_fp32 ? launch_gemm<EPI_BIAS_GELU, true>(ta, tw, tc, tr, p, grid, st)
                          : launch_gemm<EPI_BIAS_GELU, false>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_SILU:
            return c_fp32 ? launch_gemm<EPI_BIAS_SILU, true>(ta, tw, tc, tr, p, grid, st)
                          : launch_gemm<EPI_BIAS_SILU, false>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GELU_ERF:
            return c_fp32 ? launch_gemm<EPI_BIAS_GELU_ERF, true>(ta, tw, tc, tr, p, grid, st)
                          : launch_gemm<EPI_BIAS_GELU_ERF, false>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GATE_RES: return launch_gemm<EPI_BIAS_GATE_RES, false>(ta, tw, tc, tr, p, grid, st);
        default: return launch_gemm<EPI_BIAS_RES, false>(ta, tw, tc, tr, p, grid, st);
    }
}

}  // extern "C"

// scail_gemm_fp8 and scail_gemm_int8: the same checks and launch on 1-byte operands; `what` names the entry point
template <int OP>
static int gemm_scaled_impl(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                            int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                            int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, const float* scale_a,
                            const float* scale_w, scail_stream_t stream, const char* what) {
    using namespace scail;
    using Cfg = GemmCfg<OP>;
    SCAIL_REQUIRE(A && W && C && scale_a && scale_w, "%s: null operand", what);
    SCAIL_REQUIRE(!c_fp32, "%s: the output is bf16 (c_fp32 must be 0)", what);
    SCAIL_REQUIRE(M > 0 && N > 0 && K > 0, "%s: bad shape M=%lld N=%lld K=%lld", what, (long long)M, (long long)N, (long long)K);
    SCAIL_REQUIRE(K % 16 == 0 && lda % 16 == 0 && ldw % 16 == 0,
                  "%s: K, lda and ldw must be multiples of 16 (16-byte %s row pitch)", what, OP == GEMM_OP_INT8 ? "int8" : "e4m3");
    // int8: the s32 accumulator is exact while K * 127^2 < 2^31
    if (OP == GEMM_OP_INT8) SCAIL_REQUIRE(K <= 131072, "%s: K=%lld exceeds 131072 (s32 accumulator range)", what, (long long)K);
    SCAIL_REQUIRE(N % 8 == 0 && ldc % 8 == 0, "%s: N and ldc must be multiples of 8", what);
    SCAIL_REQUIRE(aligned16(C) && aligned16(bias) && aligned16(gate) && aligned16(residual),
                  "%s: C, bias, gate and residual must be 16-byte aligned (the epilogue uses 16-byte accesses)", what);
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(scale_a) & 3) == 0 && (reinterpret_cast<uintptr_t>(scale_w) & 3) == 0,
                  "%s: scales must be 4-byte aligned float32", what);
    SCAIL_REQUIRE(epilogue >= 0 && epilogue <= 5, "%s: unknown epilogue %d", what, epilogue);
    if (epilogue == EPI_BIAS_GATE_RES) SCAIL_REQUIRE(gate && residual && gate_stride % 8 == 0, "%s: gate/residual required", what);
    if (epilogue == EPI_BIAS_RES) SCAIL_REQUIRE(residual, "%s: residual required", what);
    if (residual) SCAIL_REQUIRE(ldr % 8 == 0, "%s: ldr must be a multiple of 8", what);
    const bool res_epi = epilogue == EPI_BIAS_GATE_RES || epilogue == EPI_BIAS_RES;
    CUtensorMap ta, tw, tc, tr;
    int rc;
    GemmParams p;
    p.M = (int)M; p.N = (int)N; p.K = (int)K;
    p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.gate = static_cast<const __nv_bfloat16*>(gate);
    p.gate_stride = gate_stride;
    p.rows_per_batch = rows_per_batch > 0 ? (int)rows_per_batch : (int)M;
    p.group_m = 16;
    p.scale_a = scale_a;
    p.scale_w = scale_w;
    const int sms = sm_count();
    SCAIL_REQUIRE(sms > 0, "%s: no CUDA device", what);
    if ((rc = make_tmap_2d(A, M, K, lda, Cfg::BM, Cfg::BK, &ta, 1))) return rc;
    if ((rc = make_tmap_2d(W, N, K, ldw, Cfg::BN, Cfg::BK, &tw, 1))) return rc;
    if ((rc = make_tmap_2d(C, M, N, ldc, 64, 64, &tc))) return rc;
    if (res_epi) {
        if ((rc = make_tmap_2d(residual, M, N, ldr, 64, 64, &tr))) return rc;
    } else {
        tr = tc;  // unused
    }
    const int num_tiles = blocks_for(M, Cfg::BM) * blocks_for(N, Cfg::BN);
    const int grid = num_tiles < sms ? num_tiles : sms;
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (epilogue) {
        case EPI_BIAS: return launch_gemm_scaled<OP, EPI_BIAS>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GELU: return launch_gemm_scaled<OP, EPI_BIAS_GELU>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_SILU: return launch_gemm_scaled<OP, EPI_BIAS_SILU>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GELU_ERF: return launch_gemm_scaled<OP, EPI_BIAS_GELU_ERF>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GATE_RES: return launch_gemm_scaled<OP, EPI_BIAS_GATE_RES>(ta, tw, tc, tr, p, grid, st);
        default: return launch_gemm_scaled<OP, EPI_BIAS_RES>(ta, tw, tc, tr, p, grid, st);
    }
}

template <bool INT8>
static int quant_rows_impl(const void* x, int64_t ldx, void* q, float* scale, int64_t M, int64_t K, scail_stream_t stream,
                           const char* what) {
    using namespace scail;
    SCAIL_REQUIRE(x && q && scale, "%s: null operand", what);
    SCAIL_REQUIRE(M > 0 && K > 0 && K % 16 == 0 && ldx % 8 == 0 && aligned16(x) && aligned16(q),
                  "%s: K must be a multiple of 16, ldx of 8, x and q 16-byte aligned", what);
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(scale) & 3) == 0, "%s: scale must be 4-byte aligned float32", what);
    auto xp = static_cast<const __nv_bfloat16*>(x);
    auto qp = static_cast<uint8_t*>(q);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int vpt = blocks_for(K / 8, ROW_THREADS);  // 16-byte vectors per thread
    auto k4 = INT8 ? quant_rows_int8_kernel<4> : quant_rows_fp8_kernel<4>;
    auto k8 = INT8 ? quant_rows_int8_kernel<8> : quant_rows_fp8_kernel<8>;
    auto k16 = INT8 ? quant_rows_int8_kernel<16> : quant_rows_fp8_kernel<16>;
    if (vpt <= 4) k4<<<(unsigned)M, ROW_THREADS, 0, st>>>(xp, ldx, qp, scale, (int)K);
    else if (vpt <= 8) k8<<<(unsigned)M, ROW_THREADS, 0, st>>>(xp, ldx, qp, scale, (int)K);
    else if (vpt <= 16) k16<<<(unsigned)M, ROW_THREADS, 0, st>>>(xp, ldx, qp, scale, (int)K);
    else return fail(-1, "%s: K=%lld exceeds %d", what, (long long)K, 16 * ROW_THREADS * 8);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

extern "C" {

int scail_gemm_fp8(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                   int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                   int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, const float* scale_a,
                   const float* scale_w, scail_stream_t stream) {
    return gemm_scaled_impl<scail::GEMM_OP_E4M3>(A, lda, W, ldw, bias, C, ldc, M, N, K, epilogue, gate, gate_stride,
                                                 rows_per_batch, residual, ldr, c_fp32, scale_a, scale_w, stream, "gemm_fp8");
}

int scail_gemm_int8(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                    int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                    int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, const float* scale_a,
                    const float* scale_w, scail_stream_t stream) {
    return gemm_scaled_impl<scail::GEMM_OP_INT8>(A, lda, W, ldw, bias, C, ldc, M, N, K, epilogue, gate, gate_stride,
                                                 rows_per_batch, residual, ldr, c_fp32, scale_a, scale_w, stream, "gemm_int8");
}

int scail_quant_rows_fp8(const void* x, int64_t ldx, void* q, float* scale, int64_t M, int64_t K, scail_stream_t stream) {
    return quant_rows_impl<false>(x, ldx, q, scale, M, K, stream, "quant_rows_fp8");
}

int scail_quant_rows_int8(const void* x, int64_t ldx, void* q, float* scale, int64_t M, int64_t K, scail_stream_t stream) {
    return quant_rows_impl<true>(x, ldx, q, scale, M, K, stream, "quant_rows_int8");
}

// int8: out_q takes INT8 rows instead of e4m3 ones
static int ln_modulate_impl(const void* x, void* out, void* out_q, float* out_scale, const void* gamma, const void* beta,
                            const void* shift, const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out,
                            int64_t in_batch_rows, int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream,
                            bool int8 = false) {
    using namespace scail;
    SCAIL_REQUIRE(D % 8 == 0 && D <= ROW_MAXV * ROW_THREADS * 8, "ln_modulate: D=%lld must be a multiple of 8 and <= %d", (long long)D, ROW_MAXV * ROW_THREADS * 8);
    SCAIL_REQUIRE((gamma == nullptr) == (beta == nullptr) && (shift == nullptr) == (scale == nullptr), "ln_modulate: gamma/beta and shift/scale come in pairs");
    LnModParams p;
    p.x = static_cast<const __nv_bfloat16*>(x); p.out = static_cast<__nv_bfloat16*>(out);
    p.out_q = static_cast<uint8_t*>(out_q); p.out_scale = out_scale;
    p.gamma = static_cast<const __nv_bfloat16*>(gamma); p.beta = static_cast<const __nv_bfloat16*>(beta);
    p.shift = static_cast<const __nv_bfloat16*>(shift); p.scale = static_cast<const __nv_bfloat16*>(scale);
    p.mod_stride = mod_stride; p.D = (int)D; p.rows_out = (int)rows_out; p.in_batch_rows = (int)in_batch_rows;
    p.in_row_offset = (int)in_row_offset; p.total_rows = (int)(B * rows_out); p.eps = eps;
    if (out_q && int8) ln_modulate_kernel<false, true><<<p.total_rows, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    else if (out_q) ln_modulate_kernel<true><<<p.total_rows, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    else ln_modulate_kernel<false><<<p.total_rows, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_ln_modulate(const void* x, void* out, const void* gamma, const void* beta, const void* shift,
                      const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out, int64_t in_batch_rows,
                      int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out, "ln_modulate: null operand");
    return ln_modulate_impl(x, out, nullptr, nullptr, gamma, beta, shift, scale, mod_stride, B, rows_out, in_batch_rows,
                            in_row_offset, D, eps, stream);
}

int scail_ln_modulate_fp8(const void* x, void* out_q, float* out_scale, const void* gamma, const void* beta, const void* shift,
                          const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out, int64_t in_batch_rows,
                          int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out_q && out_scale, "ln_modulate_fp8: null operand");
    SCAIL_REQUIRE(D % 16 == 0 && aligned16(out_q) && (reinterpret_cast<uintptr_t>(out_scale) & 3) == 0,
                  "ln_modulate_fp8: D must be a multiple of 16, out_q 16-byte aligned, out_scale 4-byte aligned");
    return ln_modulate_impl(x, nullptr, out_q, out_scale, gamma, beta, shift, scale, mod_stride, B, rows_out, in_batch_rows,
                            in_row_offset, D, eps, stream);
}

int scail_ln_modulate_int8(const void* x, void* out_q, float* out_scale, const void* gamma, const void* beta, const void* shift,
                           const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out, int64_t in_batch_rows,
                           int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out_q && out_scale, "ln_modulate_int8: null operand");
    SCAIL_REQUIRE(D % 16 == 0 && aligned16(out_q) && (reinterpret_cast<uintptr_t>(out_scale) & 3) == 0,
                  "ln_modulate_int8: D must be a multiple of 16, out_q 16-byte aligned, out_scale 4-byte aligned");
    return ln_modulate_impl(x, nullptr, out_q, out_scale, gamma, beta, shift, scale, mod_stride, B, rows_out, in_batch_rows,
                            in_row_offset, D, eps, stream, true);
}

int scail_rmsnorm_rope(void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                       int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                       const float* cos, const float* sin, float eps, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(buf && weight0 && (nslabs == 1 || (nslabs == 2 && weight1)), "rmsnorm_rope: null operand");
    SCAIL_REQUIRE(D % 8 == 0 && D <= ROW_MAXV * ROW_THREADS * 8 && ld % 8 == 0 && col_offset0 % 8 == 0 && col_offset1 % 8 == 0, "rmsnorm_rope: bad D/ld/offset");
    SCAIL_REQUIRE(!cos || D % 128 == 0, "rmsnorm_rope: RoPE needs D to be a multiple of the 128-wide head");
    SCAIL_REQUIRE(rows > 0 && rows_per_batch > 0, "rmsnorm_rope: bad row counts");
    SCAIL_REQUIRE((cos == nullptr) == (sin == nullptr), "rmsnorm_rope: cos/sin come in pairs");
    RmsRopeParams p;
    p.buf = static_cast<__nv_bfloat16*>(buf); p.ld = ld;
    p.col_offset[0] = (int)col_offset0; p.col_offset[1] = (int)col_offset1;
    p.weight[0] = static_cast<const __nv_bfloat16*>(weight0); p.weight[1] = static_cast<const __nv_bfloat16*>(weight1);
    p.nslabs = nslabs; p.D = (int)D; p.rows = (int)rows; p.rows_per_batch = (int)rows_per_batch;
    p.cos = cos; p.sin = sin; p.eps = eps;
    dim3 grid((unsigned)rows, nslabs);
    rmsnorm_rope_kernel<false><<<grid, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }

int scail_rmsnorm_rope_fp8(const void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                           int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                           const float* cos, const float* sin, float eps, void* q8_0, float* s8_0, void* q8_1, float* s8_1,
                           int64_t ld8, int64_t L_pad, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(buf && weight0 && q8_0 && s8_0 && (nslabs == 1 || (nslabs == 2 && weight1 && q8_1 && s8_1)),
                  "rmsnorm_rope_fp8: null operand");
    SCAIL_REQUIRE(D % 128 == 0 && D <= ROW_MAXV * ROW_THREADS * 8, "rmsnorm_rope_fp8: D=%lld must be a multiple of the 128-wide head and <= %d",
                  (long long)D, ROW_MAXV * ROW_THREADS * 8);
    SCAIL_REQUIRE(ld % 8 == 0 && col_offset0 % 8 == 0 && col_offset1 % 8 == 0 && aligned16(buf), "rmsnorm_rope_fp8: bad ld/offset");
    SCAIL_REQUIRE(ld8 % 16 == 0 && ld8 >= D && aligned16(q8_0) && aligned16(q8_1) && aligned4(s8_0) && aligned4(s8_1),
                  "rmsnorm_rope_fp8: ld8 must be a multiple of 16 and >= D, q8 16-byte and s8 4-byte aligned");
    SCAIL_REQUIRE(rows > 0 && rows_per_batch > 0 && rows % rows_per_batch == 0, "rmsnorm_rope_fp8: bad row counts");
    SCAIL_REQUIRE(L_pad % 128 == 0 && rows_per_batch <= L_pad, "rmsnorm_rope_fp8: L_pad=%lld must be a multiple of 128 and >= L=%lld",
                  (long long)L_pad, (long long)rows_per_batch);
    SCAIL_REQUIRE((cos == nullptr) == (sin == nullptr), "rmsnorm_rope_fp8: cos/sin come in pairs");
    RmsRopeParams p;
    p.buf = const_cast<__nv_bfloat16*>(static_cast<const __nv_bfloat16*>(buf)); p.ld = ld;
    p.col_offset[0] = (int)col_offset0; p.col_offset[1] = (int)col_offset1;
    p.weight[0] = static_cast<const __nv_bfloat16*>(weight0); p.weight[1] = static_cast<const __nv_bfloat16*>(weight1);
    p.nslabs = nslabs; p.D = (int)D; p.rows = (int)rows; p.rows_per_batch = (int)rows_per_batch;
    p.cos = cos; p.sin = sin; p.eps = eps;
    p.q8[0] = static_cast<uint8_t*>(q8_0); p.q8[1] = static_cast<uint8_t*>(q8_1);
    p.s8[0] = s8_0; p.s8[1] = s8_1; p.ld8 = ld8; p.L_pad = (int)L_pad;
    dim3 grid((unsigned)rows, nslabs);
    rmsnorm_rope_kernel<true><<<grid, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_rmsnorm_rope_int8q(void* buf, int64_t ld, int64_t rows, int64_t rows_per_batch, int64_t D, int nslabs,
                             int64_t col_offset0, const void* weight0, int64_t col_offset1, const void* weight1,
                             const float* cos, const float* sin, float eps, void* q8, float* q_scale, int64_t ld8, int64_t L_pad,
                             scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(nslabs == 2, "rmsnorm_rope_int8q: nslabs=%d must be 2 (slab 0 = Q, slab 1 = K)", nslabs);
    SCAIL_REQUIRE(buf && weight0 && weight1 && q8 && q_scale, "rmsnorm_rope_int8q: null operand");
    SCAIL_REQUIRE(D % 128 == 0 && D <= ROW_MAXV * ROW_THREADS * 8, "rmsnorm_rope_int8q: D=%lld must be a multiple of the 128-wide head and <= %d",
                  (long long)D, ROW_MAXV * ROW_THREADS * 8);
    SCAIL_REQUIRE(ld % 8 == 0 && col_offset0 % 8 == 0 && col_offset1 % 8 == 0 && aligned16(buf), "rmsnorm_rope_int8q: bad ld/offset");
    SCAIL_REQUIRE(ld8 % 16 == 0 && ld8 >= D && aligned16(q8) && aligned4(q_scale),
                  "rmsnorm_rope_int8q: ld8 must be a multiple of 16 and >= D, q8 16-byte and q_scale 4-byte aligned");
    SCAIL_REQUIRE(rows > 0 && rows_per_batch > 0 && rows % rows_per_batch == 0, "rmsnorm_rope_int8q: bad row counts");
    SCAIL_REQUIRE(L_pad % 128 == 0 && rows_per_batch <= L_pad, "rmsnorm_rope_int8q: L_pad=%lld must be a multiple of 128 and >= L=%lld",
                  (long long)L_pad, (long long)rows_per_batch);
    SCAIL_REQUIRE((cos == nullptr) == (sin == nullptr), "rmsnorm_rope_int8q: cos/sin come in pairs");
    RmsRopeParams p;
    p.buf = static_cast<__nv_bfloat16*>(buf); p.ld = ld;
    p.col_offset[0] = (int)col_offset0; p.col_offset[1] = (int)col_offset1;
    p.weight[0] = static_cast<const __nv_bfloat16*>(weight0); p.weight[1] = static_cast<const __nv_bfloat16*>(weight1);
    p.nslabs = 2; p.D = (int)D; p.rows = (int)rows; p.rows_per_batch = (int)rows_per_batch;
    p.cos = cos; p.sin = sin; p.eps = eps;
    p.q8[0] = static_cast<uint8_t*>(q8); p.q8[1] = nullptr;
    p.s8[0] = q_scale; p.s8[1] = nullptr; p.ld8 = ld8; p.L_pad = (int)L_pad;
    dim3 grid((unsigned)rows, 2);
    rmsnorm_rope_kernel<false, true><<<grid, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_quant_k_int8(const void* k, int64_t ldk, void* k8, int64_t ld8, float* k_scale, float* kbar, double* partial,
                       int64_t partial_len, int64_t B, int64_t H, int64_t L, int64_t L_pad, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(k && k8 && k_scale && kbar && partial, "quant_k_int8: null operand");
    const int64_t need = B * ((L + KMEAN_ROWS - 1) / KMEAN_ROWS) * H * ATT_D;
    SCAIL_REQUIRE(partial_len >= need, "quant_k_int8: partial_len=%lld must be >= B*ceil(L/256)*H*128 = %lld", (long long)partial_len,
                  (long long)need);
    SCAIL_REQUIRE(B > 0 && H > 0 && L > 0 && L_pad % 128 == 0 && L <= L_pad && B <= 65535,
                  "quant_k_int8: bad shape B=%lld H=%lld L=%lld L_pad=%lld (L <= L_pad, L_pad %% 128 == 0)", (long long)B,
                  (long long)H, (long long)L, (long long)L_pad);
    SCAIL_REQUIRE(H * ATT_D <= ROW_MAXV * ROW_THREADS * 8, "quant_k_int8: H*128=%lld must be <= %d", (long long)(H * ATT_D),
                  ROW_MAXV * ROW_THREADS * 8);
    SCAIL_REQUIRE(ldk % 8 == 0 && ldk >= H * ATT_D && ld8 % 16 == 0 && ld8 >= H * ATT_D,
                  "quant_k_int8: ldk must be a multiple of 8 and ld8 of 16, both >= H*128");
    SCAIL_REQUIRE(aligned16(k) && aligned16(k8) && aligned16(kbar) && aligned4(k_scale) && (reinterpret_cast<uintptr_t>(partial) & 7) == 0,
                  "quant_k_int8: k, k8 and kbar must be 16-byte aligned, k_scale 4-byte, partial 8-byte");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int D = (int)(H * ATT_D);
    const unsigned n_chunks = blocks_for(L, KMEAN_ROWS);
    dim3 gp(n_chunks, (unsigned)B, blocks_for(D, 128 * 8));
    k_mean_partial_kernel<<<gp, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(k), ldk, partial, (int)L, D);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    dim3 gf(blocks_for(D, 128), (unsigned)B);
    k_mean_finish_kernel<<<gf, 128, 0, st>>>(partial, kbar, (int)n_chunks, (int)L, D);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    quant_k_int8_kernel<<<(unsigned)(B * L), ROW_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(k), ldk, kbar,
                                                                    static_cast<int8_t*>(k8), ld8, k_scale, (int)L, (int)L_pad, D);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_quant_vt_fp8(const void* v, int64_t ldv, void* vt, float* v_scale, void* amax_work, int64_t B, int64_t H,
                       int64_t head_dim, int64_t L, int64_t L_pad, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(v && vt && v_scale && amax_work, "quant_vt_fp8: null operand");
    SCAIL_REQUIRE(head_dim == ATT_D, "quant_vt_fp8: head_dim=%lld, only 128 is supported", (long long)head_dim);
    SCAIL_REQUIRE(B > 0 && H > 0 && L > 0 && L_pad % 128 == 0 && L <= L_pad,
                  "quant_vt_fp8: bad shape B=%lld H=%lld L=%lld L_pad=%lld (L <= L_pad, L_pad %% 128 == 0)", (long long)B,
                  (long long)H, (long long)L, (long long)L_pad);
    SCAIL_REQUIRE(ldv % 8 == 0 && ldv >= H * ATT_D && aligned16(v) && aligned16(vt) && aligned4(v_scale) && aligned4(amax_work),
                  "quant_vt_fp8: ldv must be a multiple of 8 and >= H*128, v and vt 16-byte aligned, v_scale and amax_work 4-byte aligned");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int D = (int)(H * ATT_D);
    SCAIL_CHECK_CUDA(cudaMemsetAsync(amax_work, 0, sizeof(unsigned) * B * D, st));
    dim3 ga(blocks_for(L, VT_AMAX_ROWS), (unsigned)B, blocks_for(D, 128 * 8));
    quant_vt_amax_kernel<<<ga, 128, 0, st>>>(static_cast<const __nv_bfloat16*>(v), ldv, static_cast<unsigned*>(amax_work),
                                             (int)L, D);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    dim3 gt((unsigned)(L_pad / VT_KEYS), (unsigned)H, (unsigned)B);
    quant_vt_fp8_kernel<<<gt, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(v), ldv, static_cast<const unsigned*>(amax_work),
                                            static_cast<uint8_t*>(vt), v_scale, (int)L, (int)L_pad, (int)H);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Host checks of a block-sparse map (the contents live on the device: the Python wrapper validates them when it builds
// the map).  `what` names the entry point in the message.
static int check_tile_map(const char* what, const int32_t* kv_tile_ptr, const int32_t* kv_tile_idx, int64_t nnz, int64_t q_len,
                          int64_t kv_len) {
    SCAIL_REQUIRE(kv_tile_ptr && kv_tile_idx, "%s: null tile map", what);
    SCAIL_REQUIRE(aligned4(kv_tile_ptr) && aligned4(kv_tile_idx), "%s: kv_tile_ptr and kv_tile_idx must be 4-byte aligned int32", what);
    const int64_t n_q_tiles = (q_len + scail::ATT_BQ - 1) / scail::ATT_BQ, n_kv_tiles = (kv_len + scail::ATT_BKV - 1) / scail::ATT_BKV;
    SCAIL_REQUIRE(nnz >= n_q_tiles && nnz <= n_q_tiles * n_kv_tiles,
                  "%s: nnz=%lld must lie in [n_q_tiles, n_q_tiles * n_kv_tiles] = [%lld, %lld] (every row non-empty, no repeats)",
                  what, (long long)nnz, (long long)n_q_tiles, (long long)(n_q_tiles * n_kv_tiles));
    return 0;
}

// attention_fp8_kernel<sparse, int8qk>, one of its four instantiations
static int launch_attention_fp8(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const scail::Attn8Params& p,
                                dim3 grid, bool sparse, bool int8qk, cudaStream_t st) {
    using namespace scail;
    int rc;
    auto kernel = sparse ? (int8qk ? attention_fp8_kernel<true, true> : attention_fp8_kernel<true, false>)
                         : (int8qk ? attention_fp8_kernel<false, true> : attention_fp8_kernel<false, false>);
    if ((rc = set_smem(kernel, ATT8_SMEM_BYTES))) return rc;
    kernel<<<grid, ATT_THREADS, ATT8_SMEM_BYTES, st>>>(tq, tk, tv, p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// int8qk: Q and K are INT8 (attention_fp8_kernel<., true>); `what` names the entry point in the messages
static int attention_fp8_impl(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                              const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H,
                              int64_t head_dim, int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr,
                              const int32_t* kv_tile_idx, scail_stream_t stream, int64_t ptr_stride = 0, int64_t idx_stride = 0,
                              bool int8qk = false, const char* what = "attention_fp8") {
    using namespace scail;
    SCAIL_REQUIRE(Q && q_scale && K && k_scale && vt && v_scale && out, "%s: null operand", what);
    SCAIL_REQUIRE(head_dim == ATT_D, "%s: head_dim=%lld, only 128 is supported", what, (long long)head_dim);
    SCAIL_REQUIRE(B > 0 && H > 0 && L > 0 && L_pad % 128 == 0 && L <= L_pad,
                  "%s: bad shape B=%lld H=%lld L=%lld L_pad=%lld (L <= L_pad, L_pad %% 128 == 0)", what, (long long)B,
                  (long long)H, (long long)L, (long long)L_pad);
    SCAIL_REQUIRE(ldq % 16 == 0 && ldk % 16 == 0 && ldq >= H * ATT_D && ldk >= H * ATT_D && ldo % 8 == 0 && ldo >= H * ATT_D,
                  "%s: ldq and ldk must be multiples of 16, ldo of 8, all >= H*128", what);
    SCAIL_REQUIRE(aligned16(Q) && aligned16(K) && aligned16(vt) && aligned16(out) && aligned16(k_scale) && aligned4(q_scale) &&
                      (reinterpret_cast<uintptr_t>(v_scale) & 7) == 0,
                  "%s: Q, K, vt, out and k_scale must be 16-byte aligned, v_scale 8-byte, q_scale 4-byte", what);
    CUtensorMap tq, tk, tv;
    int rc;
    const uint64_t cols = (uint64_t)H * ATT_D;
    if ((rc = make_tmap_2d(Q, B * L, cols, ldq, ATT_BQ, 128, &tq, 1))) return rc;
    if ((rc = make_tmap_2d(K, B * L, cols, ldk, ATT_BKV, 128, &tk, 1))) return rc;
    if ((rc = make_tmap_2d(vt, B * H * ATT_D, L_pad, L_pad, ATT_D, 128, &tv, 1))) return rc;
    Attn8Params p;
    p.out = static_cast<__nv_bfloat16*>(out); p.ldo = ldo;
    p.q_scale = q_scale; p.k_scale = k_scale; p.v_scale = v_scale;
    p.L = (int)L; p.L_pad = (int)L_pad; p.heads = (int)H;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.kv_tile_ptr = kv_tile_ptr; p.kv_tile_idx = kv_tile_idx;
    p.ptr_stride = ptr_stride; p.idx_stride = idx_stride;
    dim3 grid((unsigned)(L_pad / ATT_BQ), (unsigned)H, (unsigned)B);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    return launch_attention_fp8(tq, tk, tv, p, grid, kv_tile_ptr != nullptr, int8qk, st);
}

int scail_attention_fp8(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                        const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H, int64_t head_dim,
                        int64_t L, int64_t L_pad, float scale, scail_stream_t stream) {
    return attention_fp8_impl(Q, ldq, q_scale, K, ldk, k_scale, vt, v_scale, out, ldo, B, H, head_dim, L, L_pad, scale, nullptr,
                              nullptr, stream);
}

int scail_attention_fp8_sparse(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                               const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H,
                               int64_t head_dim, int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr,
                               const int32_t* kv_tile_idx, int64_t nnz, scail_stream_t stream) {
    int rc;
    if ((rc = check_tile_map("attention_fp8_sparse", kv_tile_ptr, kv_tile_idx, nnz, L, L))) return rc;
    return attention_fp8_impl(Q, ldq, q_scale, K, ldk, k_scale, vt, v_scale, out, ldo, B, H, head_dim, L, L_pad, scale,
                              kv_tile_ptr, kv_tile_idx, stream);
}

static int attention_impl(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                          int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_off0, int64_t kv_len0, int64_t kv_off1,
                          int64_t kv_len1, int64_t q_batch_rows, int64_t kv_batch_rows, int64_t q_rows_total,
                          int64_t kv_rows_total, float scale, int accumulate, float* o32, int64_t ldo32, void* state,
                          const int32_t* kv_tile_ptr, const int32_t* kv_tile_idx, scail_stream_t stream,
                          int64_t ptr_stride = 0, int64_t idx_stride = 0) {
    using namespace scail;
    SCAIL_REQUIRE(Q && K && V && (out || o32), "attention: null operand");
    SCAIL_REQUIRE(B > 0 && H > 0 && q_len > 0 && kv_len0 > 0 && kv_len1 >= 0 && kv_off0 >= 0 && kv_off1 >= 0, "attention: bad shape");
    SCAIL_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "attention: leading dims must be multiples of 8");
    SCAIL_REQUIRE(aligned16(out) && aligned16(o32), "attention: out must be 16-byte aligned");
    SCAIL_REQUIRE((o32 == nullptr) == (state == nullptr) && (!o32 || (ldo32 % 4 == 0 && !accumulate)), "attention: o32 and state come together (ldo32 %% 4 == 0, no accumulate)");
    SCAIL_REQUIRE(q_len <= q_batch_rows && kv_off0 + kv_len0 <= kv_batch_rows && kv_off1 + kv_len1 <= kv_batch_rows &&
                      B * q_batch_rows <= q_rows_total + (q_batch_rows - q_len) &&
                      (B - 1) * kv_batch_rows + (kv_len1 > 0 ? kv_off1 + kv_len1 : kv_off0 + kv_len0) <= kv_rows_total,
                  "attention: row extents inconsistent");
    CUtensorMap tq, tk, tv;
    int rc;
    const uint64_t cols = (uint64_t)H * ATT_D;
    if ((rc = make_tmap_2d(Q, q_rows_total, cols, ldq, ATT_BQ, 64, &tq))) return rc;
    if ((rc = make_tmap_2d(K, kv_rows_total, cols, ldk, ATT_BKV, 64, &tk))) return rc;
    if ((rc = make_tmap_2d(V, kv_rows_total, cols, ldv, ATT_BKV, 64, &tv))) return rc;
    AttnParams p;
    p.out = static_cast<__nv_bfloat16*>(out); p.ldo = ldo;
    p.q_len = (int)q_len; p.kv_len = (int)kv_len0; p.kv_off = (int)kv_off0; p.kv_off1 = (int)kv_off1; p.kv_len1 = (int)kv_len1;
    p.q_batch_rows = (int)q_batch_rows; p.kv_batch_rows = (int)kv_batch_rows;
    p.o32 = o32; p.ldo32 = ldo32; p.state = static_cast<float2*>(state); p.heads = (int)H;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.accumulate = accumulate;
    p.kv_tile_ptr = kv_tile_ptr; p.kv_tile_idx = kv_tile_idx;
    p.ptr_stride = ptr_stride; p.idx_stride = idx_stride;
    dim3 grid(blocks_for(q_len, ATT_BQ), (unsigned)H, (unsigned)B);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (kv_tile_ptr) {
        if ((rc = set_smem(attention_fwd_kernel<true>, ATT_SMEM_BYTES))) return rc;
        attention_fwd_kernel<true><<<grid, ATT_THREADS, ATT_SMEM_BYTES, st>>>(tq, tk, tv, p);
    } else {
        if ((rc = set_smem(attention_fwd_kernel<false>, ATT_SMEM_BYTES))) return rc;
        attention_fwd_kernel<false><<<grid, ATT_THREADS, ATT_SMEM_BYTES, st>>>(tq, tk, tv, p);
    }
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_attention(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                    int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_len, int64_t q_batch_rows,
                    int64_t kv_batch_rows, int64_t q_rows_total, int64_t kv_rows_total, float scale, int accumulate,
                    scail_stream_t stream) {
    return attention_impl(Q, ldq, K, ldk, V, ldv, out, ldo, B, H, q_len, 0, kv_len, 0, 0, q_batch_rows, kv_batch_rows, q_rows_total,
                          kv_rows_total, scale, accumulate, nullptr, 0, nullptr, nullptr, nullptr, stream);
}

int scail_attention_sparse(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                           int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_len, int64_t q_batch_rows,
                           int64_t kv_batch_rows, int64_t q_rows_total, int64_t kv_rows_total, float scale, int accumulate,
                           const int32_t* kv_tile_ptr, const int32_t* kv_tile_idx, int64_t nnz, scail_stream_t stream) {
    SCAIL_REQUIRE(q_len == kv_len, "attention_sparse: self-attention only (q_len=%lld != kv_len=%lld)", (long long)q_len,
                  (long long)kv_len);
    int rc;
    if ((rc = check_tile_map("attention_sparse", kv_tile_ptr, kv_tile_idx, nnz, q_len, kv_len))) return rc;
    return attention_impl(Q, ldq, K, ldk, V, ldv, out, ldo, B, H, q_len, 0, kv_len, 0, 0, q_batch_rows, kv_batch_rows, q_rows_total,
                          kv_rows_total, scale, accumulate, nullptr, 0, nullptr, kv_tile_ptr, kv_tile_idx, stream);
}

// Host checks of per-(batch, head) maps (scail_attention_sparse_bh, scail_attention_select_tiles): pointers, alignment and
// strides that give every (b, h) a slot of n_q + 1 row pointers and n_q * n_kv indices.
static int check_bh_maps(const char* what, const void* kv_tile_ptr, int64_t ptr_stride, const void* kv_tile_idx,
                         int64_t idx_stride, int64_t L) {
    SCAIL_REQUIRE(kv_tile_ptr && kv_tile_idx, "%s: null tile map", what);
    SCAIL_REQUIRE(aligned4(kv_tile_ptr) && aligned4(kv_tile_idx), "%s: kv_tile_ptr and kv_tile_idx must be 4-byte aligned int32", what);
    SCAIL_REQUIRE(L > 0, "%s: L=%lld must be positive", what, (long long)L);
    const int64_t n = (L + scail::ATT_BKV - 1) / scail::ATT_BKV;
    SCAIL_REQUIRE(ptr_stride >= n + 1, "%s: ptr_stride=%lld must be >= n_q_tiles + 1 = %lld", what, (long long)ptr_stride,
                  (long long)(n + 1));
    SCAIL_REQUIRE(idx_stride >= n * n, "%s: idx_stride=%lld must be >= n_q_tiles * n_kv_tiles = %lld", what, (long long)idx_stride,
                  (long long)(n * n));
    return 0;
}

int scail_attention_sparse_bh(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                              int64_t ldo, int64_t B, int64_t H, int64_t L, int64_t q_batch_rows, int64_t kv_batch_rows,
                              int64_t q_rows_total, int64_t kv_rows_total, float scale, const int32_t* kv_tile_ptr,
                              int64_t ptr_stride, const int32_t* kv_tile_idx, int64_t idx_stride, scail_stream_t stream) {
    int rc;
    if ((rc = check_bh_maps("attention_sparse_bh", kv_tile_ptr, ptr_stride, kv_tile_idx, idx_stride, L))) return rc;
    return attention_impl(Q, ldq, K, ldk, V, ldv, out, ldo, B, H, L, 0, L, 0, 0, q_batch_rows, kv_batch_rows, q_rows_total,
                          kv_rows_total, scale, 0, nullptr, 0, nullptr, kv_tile_ptr, kv_tile_idx, stream, ptr_stride, idx_stride);
}

int scail_attention_fp8_sparse_bh(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk,
                                  const float* k_scale, const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B,
                                  int64_t H, int64_t head_dim, int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr,
                                  int64_t ptr_stride, const int32_t* kv_tile_idx, int64_t idx_stride, scail_stream_t stream) {
    int rc;
    if ((rc = check_bh_maps("attention_fp8_sparse_bh", kv_tile_ptr, ptr_stride, kv_tile_idx, idx_stride, L))) return rc;
    return attention_fp8_impl(Q, ldq, q_scale, K, ldk, k_scale, vt, v_scale, out, ldo, B, H, head_dim, L, L_pad, scale,
                              kv_tile_ptr, kv_tile_idx, stream, ptr_stride, idx_stride);
}

int scail_attention_int8qk(const void* Q, int64_t ldq, const float* q_scale, const void* K, int64_t ldk, const float* k_scale,
                           const void* vt, const float* v_scale, void* out, int64_t ldo, int64_t B, int64_t H, int64_t head_dim,
                           int64_t L, int64_t L_pad, float scale, const int32_t* kv_tile_ptr, int64_t ptr_stride,
                           const int32_t* kv_tile_idx, int64_t idx_stride, scail_stream_t stream) {
    int rc;
    if (kv_tile_ptr || kv_tile_idx) {
        SCAIL_REQUIRE(kv_tile_ptr && kv_tile_idx, "attention_int8qk: kv_tile_ptr and kv_tile_idx come together (both null: dense)");
        SCAIL_REQUIRE((ptr_stride == 0) == (idx_stride == 0), "attention_int8qk: ptr_stride and idx_stride are both 0 (one shared map) or both set");
        if (ptr_stride != 0) {
            if ((rc = check_bh_maps("attention_int8qk", kv_tile_ptr, ptr_stride, kv_tile_idx, idx_stride, L))) return rc;
        } else {
            SCAIL_REQUIRE(aligned4(kv_tile_ptr) && aligned4(kv_tile_idx), "attention_int8qk: kv_tile_ptr and kv_tile_idx must be 4-byte aligned int32");
        }
    }
    return attention_fp8_impl(Q, ldq, q_scale, K, ldk, k_scale, vt, v_scale, out, ldo, B, H, head_dim, L, L_pad, scale,
                              kv_tile_ptr, kv_tile_idx, stream, ptr_stride, idx_stride, true, "attention_int8qk");
}

int scail_attention_tile_pool(const void* x, int64_t ldx, const float* x_scale, int fp8, float* out, int64_t B, int64_t H,
                              int64_t L, int64_t L_pad, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(x && out, "attention_tile_pool: null operand");
    SCAIL_REQUIRE(fp8 == 0 || fp8 == 1, "attention_tile_pool: fp8=%d must be 0 (bf16) or 1 (e4m3 with scales)", fp8);
    SCAIL_REQUIRE(fp8 == (x_scale != nullptr), "attention_tile_pool: x_scale must be given exactly when fp8 == 1");
    SCAIL_REQUIRE(B > 0 && H > 0 && L > 0 && B <= 65535 && H <= 65535,
                  "attention_tile_pool: bad shape B=%lld H=%lld L=%lld", (long long)B, (long long)H, (long long)L);
    SCAIL_REQUIRE(ldx >= H * ATT_D, "attention_tile_pool: ldx=%lld must be >= H*128 = %lld", (long long)ldx, (long long)(H * ATT_D));
    SCAIL_REQUIRE(!fp8 || (L_pad % 128 == 0 && L <= L_pad), "attention_tile_pool: L_pad=%lld must be a multiple of 128 and >= L=%lld",
                  (long long)L_pad, (long long)L);
    SCAIL_REQUIRE(aligned4(out) && aligned4(x_scale) && (fp8 || (reinterpret_cast<uintptr_t>(x) & 1) == 0),
                  "attention_tile_pool: out and x_scale must be 4-byte aligned, a bf16 x 2-byte aligned");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid(blocks_for(L, ATT_BKV), (unsigned)H, (unsigned)B);
    if (fp8) tile_pool_kernel<true><<<grid, ATT_D, 0, st>>>(x, ldx, x_scale, out, (int)L, (int)L_pad, (int)H);
    else tile_pool_kernel<false><<<grid, ATT_D, 0, st>>>(x, ldx, nullptr, out, (int)L, 0, (int)H);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_attention_tile_pool_int8(const void* x, int64_t ldx, const float* x_scale, float* out, int64_t B, int64_t H, int64_t L,
                                   int64_t L_pad, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(x && x_scale && out, "attention_tile_pool_int8: null operand");
    SCAIL_REQUIRE(B > 0 && H > 0 && L > 0 && B <= 65535 && H <= 65535,
                  "attention_tile_pool_int8: bad shape B=%lld H=%lld L=%lld", (long long)B, (long long)H, (long long)L);
    SCAIL_REQUIRE(ldx >= H * ATT_D, "attention_tile_pool_int8: ldx=%lld must be >= H*128 = %lld", (long long)ldx, (long long)(H * ATT_D));
    SCAIL_REQUIRE(L_pad % 128 == 0 && L <= L_pad, "attention_tile_pool_int8: L_pad=%lld must be a multiple of 128 and >= L=%lld",
                  (long long)L_pad, (long long)L);
    SCAIL_REQUIRE(aligned4(out) && aligned4(x_scale), "attention_tile_pool_int8: out and x_scale must be 4-byte aligned");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    dim3 grid(blocks_for(L, ATT_BKV), (unsigned)H, (unsigned)B);
    tile_pool_kernel<false, true><<<grid, ATT_D, 0, st>>>(x, ldx, x_scale, out, (int)L, (int)L_pad, (int)H);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_attention_select_tiles(const float* qbar, const float* kbar, int64_t B, int64_t H, int64_t L, int64_t n_ref, double mass,
                                 int64_t max_tiles, int32_t* kv_tile_ptr, int64_t ptr_stride, int32_t* kv_tile_idx,
                                 int64_t idx_stride, int32_t* scratch, int64_t scratch_len, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(qbar && kbar && scratch, "attention_select_tiles: null operand");
    SCAIL_REQUIRE(aligned16(qbar) && aligned16(kbar) && aligned4(scratch),
                  "attention_select_tiles: qbar and kbar must be 16-byte aligned, scratch 4-byte aligned");
    int rc;
    if ((rc = check_bh_maps("attention_select_tiles", kv_tile_ptr, ptr_stride, kv_tile_idx, idx_stride, L))) return rc;
    const int64_t n = (L + ATT_BKV - 1) / ATT_BKV, words = (n + 31) / 32;
    SCAIL_REQUIRE(B > 0 && H > 0 && B <= 65535 && H <= 65535 && B * H <= 65535 && n <= ADA_MAX_TILES,
                  "attention_select_tiles: bad shape B=%lld H=%lld L=%lld (B*H <= 65535, ceil(L/128) <= %d)", (long long)B,
                  (long long)H, (long long)L, ADA_MAX_TILES);
    SCAIL_REQUIRE(n_ref >= 0 && n_ref <= L, "attention_select_tiles: n_ref=%lld must lie in [0, L=%lld]", (long long)n_ref, (long long)L);
    SCAIL_REQUIRE(mass >= 0.0 && mass <= 1.0, "attention_select_tiles: mass=%g must lie in [0, 1]", mass);
    SCAIL_REQUIRE(max_tiles >= -1, "attention_select_tiles: max_tiles=%lld must be >= 0, or -1 for no cap", (long long)max_tiles);
    SCAIL_REQUIRE(scratch_len >= B * H * n * (1 + words), "attention_select_tiles: scratch holds %lld int32, this shape needs %lld",
                  (long long)scratch_len, (long long)(B * H * n * (1 + words)));
    SelectParams p;
    p.qbar = qbar; p.kbar = kbar;
    p.heads = (int)H; p.L = (int)L; p.n_t = (int)n; p.n_ref_tiles = (int)((n_ref + ATT_BKV - 1) / ATT_BKV);
    p.mass = mass; p.max_tiles = (int)(max_tiles < n ? max_tiles : n); p.words = (int)words;
    p.counts = scratch; p.bits = reinterpret_cast<uint32_t*>(scratch + B * H * n);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int smem = (int)n * (2 * sizeof(double) + sizeof(int));
    select_tiles_kernel<<<dim3((unsigned)n, (unsigned)H, (unsigned)B), ADA_SELECT_THREADS, smem, st>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    compact_tiles_kernel<<<dim3((unsigned)n, (unsigned)(B * H)), 32, 0, st>>>(scratch, p.bits, (int)n, (int)words, kv_tile_ptr,
                                                                              ptr_stride, kv_tile_idx, idx_stride);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_attention_partial(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, float* o32,
                            int64_t ldo32, void* state, int64_t B, int64_t H, int64_t q_len, int64_t kv_off0, int64_t kv_len0,
                            int64_t kv_off1, int64_t kv_len1, int64_t q_batch_rows, int64_t kv_batch_rows, int64_t q_rows_total,
                            int64_t kv_rows_total, float scale, scail_stream_t stream) {
    SCAIL_REQUIRE(o32 && state, "attention_partial: null operand");
    return attention_impl(Q, ldq, K, ldk, V, ldv, nullptr, 8, B, H, q_len, kv_off0, kv_len0, kv_off1, kv_len1, q_batch_rows,
                          kv_batch_rows, q_rows_total, kv_rows_total, scale, 0, o32, ldo32, state, nullptr, nullptr, stream);
}

int scail_attention_merge(const float* o32_a, const void* state_a, const float* o32_b, const void* state_b, void* out,
                          int64_t ldo32, int64_t ldo, int64_t rows, int64_t H, scail_stream_t stream) {
    SCAIL_REQUIRE(o32_a && state_a && o32_b && state_b && out && rows > 0 && H > 0, "attention_merge: bad args");
    SCAIL_REQUIRE(ldo32 % 4 == 0 && ldo % 4 == 0 && aligned16(o32_a) && aligned16(o32_b) && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
                  "attention_merge: alignment");
    const int64_t warps = rows * H;
    scail::attn_merge_kernel<<<blocks_for(warps, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        o32_a, static_cast<const float2*>(state_a), o32_b, static_cast<const float2*>(state_b), static_cast<__nv_bfloat16*>(out),
        ldo32, ldo, rows, (int)H);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_adaln_modulation(const void* emb, const void* param, void* out, int64_t B, int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(emb && param && out, "adaln_modulation: null operand");
    scail::adaln_modulation_kernel<<<blocks_for(B * n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(emb), static_cast<const __nv_bfloat16*>(param), static_cast<__nv_bfloat16*>(out), (int)B, (int)n);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_silu(const void* x, void* out, int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out, "silu: null operand");
    scail::silu_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(x), static_cast<__nv_bfloat16*>(out), (int)n);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_timestep_embedding(const float* t, void* out, int64_t B, int64_t dim, scail_stream_t stream) {
    SCAIL_REQUIRE(t && out && dim % 2 == 0, "timestep_embedding: bad args");
    scail::timestep_embedding_kernel<<<blocks_for(B * dim / 2, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        t, static_cast<__nv_bfloat16*>(out), (int)B, (int)dim);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_patchify(const void* x, const void* ref, const void* pose, void* a_main, void* a_pose, int64_t B,
                   int64_t Br, int64_t Bp, int64_t T, int64_t H, int64_t W, int64_t cin, scail_stream_t stream) {
    SCAIL_REQUIRE(x && ref && pose && a_main && a_pose, "patchify: null operand");
    SCAIL_REQUIRE(cin == 16 || cin == 20, "patchify: cin must be 16 or 20");
    SCAIL_REQUIRE(H % 4 == 0 && W % 4 == 0 && Br >= 1 && Bp >= 1, "patchify: H, W must be multiples of 4");
    scail::PatchifyParams p;
    p.x = static_cast<const __nv_bfloat16*>(x); p.ref = static_cast<const __nv_bfloat16*>(ref);
    p.pose = static_cast<const __nv_bfloat16*>(pose); p.a_main = static_cast<__nv_bfloat16*>(a_main);
    p.a_pose = static_cast<__nv_bfloat16*>(a_pose);
    p.B = (int)B; p.Br = (int)Br; p.Bp = (int)Bp; p.T = (int)T; p.H = (int)H; p.W = (int)W; p.cin = (int)cin;
    const int64_t total = B * ((1 + T) * (H / 2) * (W / 2) + T * (H / 4) * (W / 4)) * 20;
    scail::patchify_kernel<<<blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_unpatchify(const void* lin, void* out, int64_t B, int64_t T, int64_t Hp, int64_t Wp, scail_stream_t stream) {
    SCAIL_REQUIRE(lin && out, "unpatchify: null operand");
    const int64_t total = B * T * 16 * 4 * Hp * Wp;
    scail::unpatchify_kernel<<<blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(lin), static_cast<__nv_bfloat16*>(out), (int)B, (int)T, (int)Hp, (int)Wp);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_cfg_euler(float* x, const void* v, int64_t n, float scale, float dsigma, scail_stream_t stream) {
    SCAIL_REQUIRE(x && v, "cfg_euler: null operand");
    scail::cfg_euler_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<const __nv_bfloat16*>(v), n, scale, dsigma);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Slot and coefficient checks shared by the two UniPC entry points; fills k.  Returns 0 or the fail() code.
static int unipc_coef(const char* what, int64_t slot_stride, int64_t n_slots, int64_t write_slot, int64_t n,
                      const float* coef, scail::UnipcCoef* k) {
    SCAIL_REQUIRE(n >= 4 && n % 4 == 0, "%s: need n a positive multiple of 4 (got n=%lld)", what, (long long)n);
    SCAIL_REQUIRE(n_slots >= 1 && n_slots <= scail::UNIPC_MAX_SLOTS, "%s: need 1 <= n_slots <= %d (got %lld)", what,
                  scail::UNIPC_MAX_SLOTS, (long long)n_slots);
    SCAIL_REQUIRE(write_slot >= 0 && write_slot < n_slots, "%s: write_slot = %lld must be in [0, n_slots = %lld)", what,
                  (long long)write_slot, (long long)n_slots);
    SCAIL_REQUIRE(slot_stride >= n && slot_stride % 4 == 0, "%s: slot_stride = %lld floats must be >= n = %lld and a "
                  "multiple of 4 so that every slot is whole and 16-byte aligned", what, (long long)slot_stride, (long long)n);
    k->a_x = coef[0];
    k->a_m = coef[4];
    k->b_y = coef[5];
    k->b_m = coef[9];
    for (int s = 0; s < scail::UNIPC_MAX_SLOTS; ++s) {
        k->a[s] = coef[1 + s];
        k->b[s] = coef[6 + s];
        SCAIL_REQUIRE(s < n_slots || (k->a[s] == 0.f && k->b[s] == 0.f),
                      "%s: the coefficients of slot %d must be 0 with n_slots = %lld", what, s, (long long)n_slots);
    }
    return 0;
}

// Checks shared by the forecast entry points of the CFG cache's delta slots; fills k.  Returns 0 or the fail() code.
static int delta_forecast_coef(const char* what, int64_t slot_stride, int64_t n_slots, int64_t n, const float* coef,
                               scail::DeltaForecast* k) {
    SCAIL_REQUIRE(n >= 4 && n % 4 == 0, "%s: need n a positive multiple of 4 (got n=%lld)", what, (long long)n);
    SCAIL_REQUIRE(n_slots >= 1 && n_slots <= scail::DELTA_MAX_SLOTS, "%s: need 1 <= n_slots <= %d delta slots (got %lld)",
                  what, scail::DELTA_MAX_SLOTS, (long long)n_slots);
    SCAIL_REQUIRE(slot_stride >= n && slot_stride % 4 == 0, "%s: delta slot_stride = %lld floats must be >= n = %lld and a "
                  "multiple of 4 so that every slot is whole and 16-byte aligned", what, (long long)slot_stride, (long long)n);
    for (int s = 0; s < scail::DELTA_MAX_SLOTS; ++s) {
        k->c[s] = coef[s];
        SCAIL_REQUIRE(s < n_slots || k->c[s] == 0.f, "%s: the forecast coefficient of delta slot %d must be 0 with n_slots = %lld",
                      what, s, (long long)n_slots);
    }
    return 0;
}

// The u_scale check of every scaled entry point (CFG-Zero*): a non-null, 4-byte aligned device scalar.
static int check_u_scale(const char* what, const float* u_scale) {
    SCAIL_REQUIRE(u_scale, "%s: null u_scale", what);
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(u_scale) & 3) == 0, "%s: u_scale must be 4-byte aligned", what);
    return 0;
}

// The three UniPC step forms, unscaled (u_scale == nullptr) or scaled.  cached: c alone with delta (one fp32 tensor, or
// with dcoef the forecast of n_dslots slots at stride dslot_stride); else v is the pair and delta is not read.
static int unipc_launch(const char* what, float* x, float* x_last, const void* v, bool cached, const float* delta,
                        int64_t dslot_stride, int64_t n_dslots, const float* dcoef, float* slots, int64_t slot_stride,
                        int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                        const float* u_scale, cudaStream_t st) {
    scail::UnipcCoef k;
    if (int rc = unipc_coef(what, slot_stride, n_slots, write_slot, n, coef, &k)) return rc;
    scail::DeltaForecast dk{};
    if (dcoef)
        if (int rc = delta_forecast_coef(what, dslot_stride, n_dslots, n, dcoef, &dk)) return rc;
    const int64_t nvec = n / 4;
    const int grid = static_cast<int>(blocks_for(nvec, scail::UNIPC_THREADS));
    float4* x4 = reinterpret_cast<float4*>(x);
    float4* xl4 = reinterpret_cast<float4*>(x_last);
    const uint2* v2 = static_cast<const uint2*>(v);
    const float4* d4 = reinterpret_cast<const float4*>(delta);
    const int64_t ds = dcoef ? dslot_stride : 0;
    const int corr = correct ? 1 : 0;
#define SCAIL_UNIPC_LAUNCH(...)                                                                                          \
    scail::unipc_step_kernel<__VA_ARGS__><<<grid, scail::UNIPC_THREADS, 0, st>>>(x4, xl4, v2, slots, slot_stride,      \
                                                                                 (int)n_slots, (int)write_slot, nvec,  \
                                                                                 scale, sigma, corr, k, d4, ds, dk, u_scale,  \
                                                                                 nullptr)
    if (!cached)
        u_scale ? SCAIL_UNIPC_LAUNCH(false, false, true) : SCAIL_UNIPC_LAUNCH(false);
    else if (!dcoef)
        u_scale ? SCAIL_UNIPC_LAUNCH(true, false, true) : SCAIL_UNIPC_LAUNCH(true);
    else
        u_scale ? SCAIL_UNIPC_LAUNCH(true, true, true) : SCAIL_UNIPC_LAUNCH(true, true);
#undef SCAIL_UNIPC_LAUNCH
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_unipc_step(float* x, float* x_last, const void* v, float* slots, int64_t slot_stride, int64_t n_slots,
                     int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                     scail_stream_t stream) {
    SCAIL_REQUIRE(x && x_last && v && slots && coef, "unipc_step: null operand");
    SCAIL_REQUIRE(aligned16(x) && aligned16(x_last) && aligned16(v) && aligned16(slots),
                  "unipc_step: x, x_last, v and slots must be 16-byte aligned");
    return unipc_launch("unipc_step", x, x_last, v, false, nullptr, 0, 0, nullptr, slots, slot_stride, n_slots, write_slot, n,
                        scale, sigma, correct, coef, nullptr, static_cast<cudaStream_t>(stream));
}

int scail_unipc_step_scaled(float* x, float* x_last, const void* v, float* slots, int64_t slot_stride, int64_t n_slots,
                            int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                            const float* u_scale, scail_stream_t stream) {
    SCAIL_REQUIRE(x && x_last && v && slots && coef, "unipc_step_scaled: null operand");
    SCAIL_REQUIRE(aligned16(x) && aligned16(x_last) && aligned16(v) && aligned16(slots),
                  "unipc_step_scaled: x, x_last, v and slots must be 16-byte aligned");
    if (int rc = check_u_scale("unipc_step_scaled", u_scale)) return rc;
    return unipc_launch("unipc_step_scaled", x, x_last, v, false, nullptr, 0, 0, nullptr, slots, slot_stride, n_slots,
                        write_slot, n, scale, sigma, correct, coef, u_scale, static_cast<cudaStream_t>(stream));
}

static int unipc_cached(const char* what, float* x, float* x_last, const void* c, const float* delta, float* slots,
                        int64_t slot_stride, int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma,
                        int correct, const float* coef, const float* u_scale, scail_stream_t stream) {
    SCAIL_REQUIRE(x && x_last && c && delta && slots && coef, "%s: null operand", what);
    SCAIL_REQUIRE(aligned16(x) && aligned16(x_last) && aligned16(c) && aligned16(delta) && aligned16(slots),
                  "%s: x, x_last, c, delta and slots must be 16-byte aligned", what);
    return unipc_launch(what, x, x_last, c, true, delta, 0, 0, nullptr, slots, slot_stride, n_slots, write_slot, n, scale,
                        sigma, correct, coef, u_scale, static_cast<cudaStream_t>(stream));
}

int scail_unipc_step_cached(float* x, float* x_last, const void* c, const float* delta, float* slots, int64_t slot_stride,
                            int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma, int correct,
                            const float* coef, scail_stream_t stream) {
    return unipc_cached("unipc_step_cached", x, x_last, c, delta, slots, slot_stride, n_slots, write_slot, n, scale, sigma,
                        correct, coef, nullptr, stream);
}

int scail_unipc_step_cached_scaled(float* x, float* x_last, const void* c, const float* delta, float* slots,
                                   int64_t slot_stride, int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma,
                                   int correct, const float* coef, const float* u_scale, scail_stream_t stream) {
    if (int rc = check_u_scale("unipc_step_cached_scaled", u_scale)) return rc;
    return unipc_cached("unipc_step_cached_scaled", x, x_last, c, delta, slots, slot_stride, n_slots, write_slot, n, scale,
                        sigma, correct, coef, u_scale, stream);
}

int scail_cfg_cache_delta_forecast(const void* v, float* slots, int64_t slot_stride, int64_t n_slots, int64_t write_slot,
                                   const float* coef, float* partials, int64_t partials_len, double* out, int64_t n,
                                   scail_stream_t stream) {
    SCAIL_REQUIRE(v && slots && coef && partials && out, "cfg_cache_delta_forecast: null operand");
    SCAIL_REQUIRE(aligned16(v) && aligned16(slots), "cfg_cache_delta_forecast: v and slots must be 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(partials) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
                  "cfg_cache_delta_forecast: partials must be 4-byte and out 8-byte aligned");
    scail::DeltaForecast k;
    if (int rc = delta_forecast_coef("cfg_cache_delta_forecast", slot_stride, n_slots, n, coef, &k)) return rc;
    SCAIL_REQUIRE(write_slot >= 0 && write_slot < n_slots,
                  "cfg_cache_delta_forecast: write_slot = %lld must be in [0, n_slots = %lld)", (long long)write_slot,
                  (long long)n_slots);
    const int64_t nvec = n / 4;
    const int ctas = static_cast<int>(std::min<int64_t>(scail::SC_MAX_CTAS, (nvec + scail::SC_THREADS - 1) / scail::SC_THREADS));
    SCAIL_REQUIRE(partials_len >= 2 * ctas, "cfg_cache_delta_forecast: partials holds %lld floats, this size needs %d",
                  (long long)partials_len, 2 * ctas);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    scail::cfg_cache_delta_forecast_kernel<<<ctas, scail::SC_THREADS, 0, st>>>(static_cast<const uint2*>(v), slots, slot_stride,
                                                                               (int)write_slot, k, partials, nvec);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    scail::step_cache_finish_kernel<<<1, scail::SC_THREADS, 0, st>>>(partials, ctas, out);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int cfg_euler_cached_forecast(const char* what, float* x, const void* c, const float* slots, int64_t slot_stride,
                                     int64_t n_slots, const float* coef, int64_t n, float scale, float dsigma,
                                     const float* u_scale, scail_stream_t stream) {
    SCAIL_REQUIRE(x && c && slots && coef, "%s: null operand", what);
    SCAIL_REQUIRE(aligned16(x) && aligned16(c) && aligned16(slots), "%s: x, c and slots must be 16-byte aligned", what);
    scail::DeltaForecast k;
    if (int rc = delta_forecast_coef(what, slot_stride, n_slots, n, coef, &k)) return rc;
    const int64_t nvec = n / 4;
    const int grid = static_cast<int>(blocks_for(nvec, scail::CFGC_THREADS));
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float4* x4 = reinterpret_cast<float4*>(x);
    const uint2* c2 = static_cast<const uint2*>(c);
    if (u_scale)
        scail::cfg_euler_cached_forecast_kernel<true><<<grid, scail::CFGC_THREADS, 0, st>>>(x4, c2, slots, slot_stride, k, nvec,
                                                                                           scale, dsigma, u_scale);
    else
        scail::cfg_euler_cached_forecast_kernel<false><<<grid, scail::CFGC_THREADS, 0, st>>>(x4, c2, slots, slot_stride, k, nvec,
                                                                                            scale, dsigma, nullptr);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_cfg_euler_cached_forecast(float* x, const void* c, const float* slots, int64_t slot_stride, int64_t n_slots,
                                    const float* coef, int64_t n, float scale, float dsigma, scail_stream_t stream) {
    return cfg_euler_cached_forecast("cfg_euler_cached_forecast", x, c, slots, slot_stride, n_slots, coef, n, scale, dsigma,
                                     nullptr, stream);
}

int scail_cfg_euler_cached_forecast_scaled(float* x, const void* c, const float* slots, int64_t slot_stride, int64_t n_slots,
                                           const float* coef, int64_t n, float scale, float dsigma, const float* u_scale,
                                           scail_stream_t stream) {
    if (int rc = check_u_scale("cfg_euler_cached_forecast_scaled", u_scale)) return rc;
    return cfg_euler_cached_forecast("cfg_euler_cached_forecast_scaled", x, c, slots, slot_stride, n_slots, coef, n, scale,
                                     dsigma, u_scale, stream);
}

static int unipc_cached_forecast(const char* what, float* x, float* x_last, const void* c, const float* dslots,
                                 int64_t dslot_stride, int64_t n_dslots, const float* dcoef, float* slots, int64_t slot_stride,
                                 int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma, int correct,
                                 const float* coef, const float* u_scale, scail_stream_t stream) {
    SCAIL_REQUIRE(x && x_last && c && dslots && dcoef && slots && coef, "%s: null operand", what);
    SCAIL_REQUIRE(aligned16(x) && aligned16(x_last) && aligned16(c) && aligned16(dslots) && aligned16(slots),
                  "%s: x, x_last, c, dslots and slots must be 16-byte aligned", what);
    return unipc_launch(what, x, x_last, c, true, dslots, dslot_stride, n_dslots, dcoef, slots, slot_stride, n_slots, write_slot,
                        n, scale, sigma, correct, coef, u_scale, static_cast<cudaStream_t>(stream));
}

int scail_unipc_step_cached_forecast(float* x, float* x_last, const void* c, const float* dslots, int64_t dslot_stride,
                                     int64_t n_dslots, const float* dcoef, float* slots, int64_t slot_stride, int64_t n_slots,
                                     int64_t write_slot, int64_t n, float scale, float sigma, int correct, const float* coef,
                                     scail_stream_t stream) {
    return unipc_cached_forecast("unipc_step_cached_forecast", x, x_last, c, dslots, dslot_stride, n_dslots, dcoef, slots,
                                 slot_stride, n_slots, write_slot, n, scale, sigma, correct, coef, nullptr, stream);
}

int scail_unipc_step_cached_forecast_scaled(float* x, float* x_last, const void* c, const float* dslots, int64_t dslot_stride,
                                            int64_t n_dslots, const float* dcoef, float* slots, int64_t slot_stride,
                                            int64_t n_slots, int64_t write_slot, int64_t n, float scale, float sigma,
                                            int correct, const float* coef, const float* u_scale, scail_stream_t stream) {
    if (int rc = check_u_scale("unipc_step_cached_forecast_scaled", u_scale)) return rc;
    return unipc_cached_forecast("unipc_step_cached_forecast_scaled", x, x_last, c, dslots, dslot_stride, n_dslots, dcoef,
                                 slots, slot_stride, n_slots, write_slot, n, scale, sigma, correct, coef, u_scale, stream);
}

int scail_cfg_cache_delta(const void* v, const float* d_ref, float* d_new, float* partials, int64_t partials_len, double* out,
                          int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(v && d_ref && d_new && partials && out, "cfg_cache_delta: null operand");
    SCAIL_REQUIRE(aligned16(v) && aligned16(d_ref) && aligned16(d_new),
                  "cfg_cache_delta: v, d_ref and d_new must be 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(partials) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
                  "cfg_cache_delta: partials must be 4-byte and out 8-byte aligned");
    SCAIL_REQUIRE(n >= 4 && n % 4 == 0, "cfg_cache_delta: need n a positive multiple of 4 (got n=%lld)", (long long)n);
    const int64_t nvec = n / 4;
    const int ctas = static_cast<int>(std::min<int64_t>(scail::SC_MAX_CTAS, (nvec + scail::SC_THREADS - 1) / scail::SC_THREADS));
    SCAIL_REQUIRE(partials_len >= 2 * ctas, "cfg_cache_delta: partials holds %lld floats, this size needs %d",
                  (long long)partials_len, 2 * ctas);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    scail::cfg_cache_delta_kernel<<<ctas, scail::SC_THREADS, 0, st>>>(
        static_cast<const uint2*>(v), reinterpret_cast<const float4*>(d_ref), reinterpret_cast<float4*>(d_new), partials, nvec);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    scail::step_cache_finish_kernel<<<1, scail::SC_THREADS, 0, st>>>(partials, ctas, out);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int cfg_euler_cached(const char* what, float* x, const void* c, const float* delta, int64_t n, float scale,
                            float dsigma, const float* u_scale, scail_stream_t stream) {
    SCAIL_REQUIRE(x && c && delta, "%s: null operand", what);
    SCAIL_REQUIRE(aligned16(x) && aligned16(c) && aligned16(delta), "%s: x, c and delta must be 16-byte aligned", what);
    SCAIL_REQUIRE(n >= 4 && n % 4 == 0, "%s: need n a positive multiple of 4 (got n=%lld)", what, (long long)n);
    const int64_t nvec = n / 4;
    const int grid = static_cast<int>(blocks_for(nvec, scail::CFGC_THREADS));
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float4* x4 = reinterpret_cast<float4*>(x);
    const uint2* c2 = static_cast<const uint2*>(c);
    const float4* d4 = reinterpret_cast<const float4*>(delta);
    if (u_scale)
        scail::cfg_euler_cached_kernel<true><<<grid, scail::CFGC_THREADS, 0, st>>>(x4, c2, d4, nvec, scale, dsigma, u_scale);
    else
        scail::cfg_euler_cached_kernel<false><<<grid, scail::CFGC_THREADS, 0, st>>>(x4, c2, d4, nvec, scale, dsigma, nullptr);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_cfg_euler_cached(float* x, const void* c, const float* delta, int64_t n, float scale, float dsigma,
                           scail_stream_t stream) {
    return cfg_euler_cached("cfg_euler_cached", x, c, delta, n, scale, dsigma, nullptr, stream);
}

int scail_cfg_euler_cached_scaled(float* x, const void* c, const float* delta, int64_t n, float scale, float dsigma,
                                  const float* u_scale, scail_stream_t stream) {
    if (int rc = check_u_scale("cfg_euler_cached_scaled", u_scale)) return rc;
    return cfg_euler_cached("cfg_euler_cached_scaled", x, c, delta, n, scale, dsigma, u_scale, stream);
}

int scail_cfg_euler_scaled(float* x, const void* v, int64_t n, float scale, float dsigma, const float* u_scale,
                           scail_stream_t stream) {
    SCAIL_REQUIRE(x && v, "cfg_euler_scaled: null operand");
    if (int rc = check_u_scale("cfg_euler_scaled", u_scale)) return rc;
    SCAIL_REQUIRE(aligned16(x) && aligned16(v), "cfg_euler_scaled: x and v must be 16-byte aligned");
    SCAIL_REQUIRE(n >= 4 && n % 4 == 0, "cfg_euler_scaled: need n a positive multiple of 4 (got n=%lld)", (long long)n);
    const int64_t nvec = n / 4;
    scail::cfg_euler_scaled_kernel<<<blocks_for(nvec, scail::CFGC_THREADS), scail::CFGC_THREADS, 0,
                                     static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<float4*>(x),
                                                                          static_cast<const uint2*>(v), nvec, scale, dsigma,
                                                                          u_scale);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_cfg_zero_scale(int form, const void* v, const float* delta, int64_t delta_stride, int64_t n_dslots, const float* dcoef,
                         float* partials, int64_t partials_len, double* out, float* u_scale, int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(form >= scail::CFGZ_PAIR && form <= scail::CFGZ_FORECAST,
                  "cfg_zero_scale: form = %d must be 0 (pair), 1 (cached) or 2 (forecast)", form);
    SCAIL_REQUIRE(v && partials && out && u_scale, "cfg_zero_scale: null operand");
    SCAIL_REQUIRE(form == scail::CFGZ_PAIR || delta, "cfg_zero_scale: null delta with form %d", form);
    SCAIL_REQUIRE(form != scail::CFGZ_FORECAST || dcoef, "cfg_zero_scale: null dcoef with form 2");
    SCAIL_REQUIRE(aligned16(v) && (form == scail::CFGZ_PAIR || aligned16(delta)),
                  "cfg_zero_scale: v and delta must be 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(partials) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0 &&
                      (reinterpret_cast<uintptr_t>(u_scale) & 3) == 0,
                  "cfg_zero_scale: partials and u_scale must be 4-byte and out 8-byte aligned");
    SCAIL_REQUIRE(n >= 4 && n % 4 == 0, "cfg_zero_scale: need n a positive multiple of 4 (got n=%lld)", (long long)n);
    scail::DeltaForecast dk{};
    if (form == scail::CFGZ_FORECAST)
        if (int rc = delta_forecast_coef("cfg_zero_scale", delta_stride, n_dslots, n, dcoef, &dk)) return rc;
    const int64_t nvec = n / 4;
    const int ctas = static_cast<int>(std::min<int64_t>(scail::SC_MAX_CTAS, (nvec + scail::SC_THREADS - 1) / scail::SC_THREADS));
    SCAIL_REQUIRE(partials_len >= 2 * ctas, "cfg_zero_scale: partials holds %lld floats, this size needs %d",
                  (long long)partials_len, 2 * ctas);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint2* v2 = static_cast<const uint2*>(v);
    const int64_t ds = form == scail::CFGZ_FORECAST ? delta_stride : 0;
    if (form == scail::CFGZ_PAIR)
        scail::cfg_zero_dot_kernel<scail::CFGZ_PAIR><<<ctas, scail::SC_THREADS, 0, st>>>(v2, nullptr, 0, dk, partials, nvec);
    else if (form == scail::CFGZ_CACHED)
        scail::cfg_zero_dot_kernel<scail::CFGZ_CACHED><<<ctas, scail::SC_THREADS, 0, st>>>(v2, delta, 0, dk, partials, nvec);
    else
        scail::cfg_zero_dot_kernel<scail::CFGZ_FORECAST><<<ctas, scail::SC_THREADS, 0, st>>>(v2, delta, ds, dk, partials, nvec);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    scail::cfg_zero_finish_kernel<<<1, scail::SC_THREADS, 0, st>>>(partials, ctas, out, u_scale);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---- APG (scail_b200/guidance.py, csrc/apg.cuh)

// Checks shared by the APG entry points: the form and its operands, and the latent's frames; fills dk and the frame's
// vector count.  Returns 0 or the fail() code.
static int apg_operands(const char* what, int form, const float* x, const void* v, const float* delta, int64_t delta_stride,
                        int64_t n_dslots, const float* dcoef, int64_t frames, int64_t n, scail::DeltaForecast* dk,
                        int64_t* fvec) {
    SCAIL_REQUIRE(form >= scail::CFGZ_PAIR && form <= scail::CFGZ_FORECAST,
                  "%s: form = %d must be 0 (pair), 1 (cached) or 2 (forecast)", what, form);
    SCAIL_REQUIRE(x && v, "%s: null operand", what);
    SCAIL_REQUIRE(form == scail::CFGZ_PAIR || delta, "%s: null delta with form %d", what, form);
    SCAIL_REQUIRE(form != scail::CFGZ_FORECAST || dcoef, "%s: null dcoef with form 2", what);
    SCAIL_REQUIRE(aligned16(x) && aligned16(v) && (form == scail::CFGZ_PAIR || aligned16(delta)),
                  "%s: x, v and delta must be 16-byte aligned", what);
    SCAIL_REQUIRE(frames >= 1 && frames <= 65535, "%s: need 1 <= frames <= 65535 (got %lld)", what, (long long)frames);
    SCAIL_REQUIRE(n >= 4 && n % (4 * frames) == 0 && n / 4 <= 0xffffffffll,
                  "%s: need n a positive multiple of 4 * frames below 2^34 (got n=%lld, frames=%lld)", what, (long long)n,
                  (long long)frames);
    *dk = scail::DeltaForecast{};
    if (form == scail::CFGZ_FORECAST)
        if (int rc = delta_forecast_coef(what, delta_stride, n_dslots, n, dcoef, dk)) return rc;
    *fvec = n / 4 / frames;
    return 0;
}

int scail_apg_reduce(int form, const float* x, const void* v, const float* delta, int64_t delta_stride, int64_t n_dslots,
                     const float* dcoef, float* avg, float sigma, float momentum, float* partials, int64_t partials_len,
                     int64_t frames, int64_t n, scail_stream_t stream) {
    scail::DeltaForecast dk;
    int64_t fvec;
    if (int rc = apg_operands("apg_reduce", form, x, v, delta, delta_stride, n_dslots, dcoef, frames, n, &dk, &fvec)) return rc;
    SCAIL_REQUIRE(partials, "apg_reduce: null partials");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(partials) & 3) == 0 && (!avg || aligned16(avg)),
                  "apg_reduce: partials must be 4-byte and avg 16-byte aligned");
    const int parts = scail::apg_ctas_per_frame(fvec);
    SCAIL_REQUIRE(partials_len >= 3 * frames * parts, "apg_reduce: partials holds %lld floats, this size needs %lld",
                  (long long)partials_len, (long long)(3 * frames * parts));
    const dim3 grid(parts, static_cast<unsigned>(frames));
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const uint2* v2 = static_cast<const uint2*>(v);
    const int64_t ds = form == scail::CFGZ_FORECAST ? delta_stride : 0;
    float4* a4 = reinterpret_cast<float4*>(avg);
#define SCAIL_APG_REDUCE(F, M) \
    scail::apg_reduce_kernel<F, M><<<grid, scail::APG_THREADS, 0, st>>>(x4, v2, delta, ds, dk, a4, sigma, momentum, partials, fvec)
    if (form == scail::CFGZ_PAIR)
        avg ? SCAIL_APG_REDUCE(scail::CFGZ_PAIR, true) : SCAIL_APG_REDUCE(scail::CFGZ_PAIR, false);
    else if (form == scail::CFGZ_CACHED)
        avg ? SCAIL_APG_REDUCE(scail::CFGZ_CACHED, true) : SCAIL_APG_REDUCE(scail::CFGZ_CACHED, false);
    else
        avg ? SCAIL_APG_REDUCE(scail::CFGZ_FORECAST, true) : SCAIL_APG_REDUCE(scail::CFGZ_FORECAST, false);
#undef SCAIL_APG_REDUCE
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_apg_finish(const float* partials, int64_t partials_len, double* sums, float* factors, double norm_threshold,
                     int64_t frames, int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(partials && sums && factors, "apg_finish: null operand");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(partials) & 3) == 0 && (reinterpret_cast<uintptr_t>(sums) & 7) == 0 &&
                      (reinterpret_cast<uintptr_t>(factors) & 7) == 0,
                  "apg_finish: partials must be 4-byte and sums and factors 8-byte aligned");
    SCAIL_REQUIRE(frames >= 1 && frames <= 65535 && n >= 4 && n % (4 * frames) == 0,
                  "apg_finish: need 1 <= frames <= 65535 and n a positive multiple of 4 * frames (got n=%lld, frames=%lld)",
                  (long long)n, (long long)frames);
    SCAIL_REQUIRE(std::isfinite(norm_threshold) && norm_threshold >= 0.0,
                  "apg_finish: norm_threshold must be finite and >= 0 (got %g)", norm_threshold);
    const int parts = scail::apg_ctas_per_frame(n / 4 / frames);
    SCAIL_REQUIRE(partials_len >= 3 * frames * parts, "apg_finish: partials holds %lld floats, this size needs %lld",
                  (long long)partials_len, (long long)(3 * frames * parts));
    scail::apg_finish_kernel<<<static_cast<unsigned>(frames), 32, 0, static_cast<cudaStream_t>(stream)>>>(
        partials, parts, norm_threshold, sums, factors);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_apg_update(int form, float* x, const void* v, const float* delta, int64_t delta_stride, int64_t n_dslots,
                     const float* dcoef, const float* avg, const float* factors, float* m, float sigma, float wm1, float eta,
                     float k_euler, int64_t frames, int64_t n, scail_stream_t stream) {
    scail::DeltaForecast dk;
    int64_t fvec;
    if (int rc = apg_operands("apg_update", form, x, v, delta, delta_stride, n_dslots, dcoef, frames, n, &dk, &fvec)) return rc;
    SCAIL_REQUIRE(factors, "apg_update: null factors");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(factors) & 7) == 0 && (!avg || aligned16(avg)) && (!m || aligned16(m)),
                  "apg_update: factors must be 8-byte and avg and m 16-byte aligned");
    const int64_t nvec = n / 4;
    const int grid = blocks_for(nvec, scail::APG_THREADS);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    float4* x4 = reinterpret_cast<float4*>(x);
    const uint2* v2 = static_cast<const uint2*>(v);
    const int64_t ds = form == scail::CFGZ_FORECAST ? delta_stride : 0;
    const float4* a4 = reinterpret_cast<const float4*>(avg);
    const float2* f2 = reinterpret_cast<const float2*>(factors);
    float4* m4 = reinterpret_cast<float4*>(m);
    const unsigned fv = static_cast<unsigned>(fvec);
#define SCAIL_APG_UPDATE(F, M, D)                                                                                           \
    scail::apg_update_kernel<F, M, D><<<grid, scail::APG_THREADS, 0, st>>>(x4, v2, delta, ds, dk, a4, f2, m4, sigma, wm1, eta, \
                                                                          k_euler, nvec, fv)
#define SCAIL_APG_UPDATE_OUT(F, M) m ? SCAIL_APG_UPDATE(F, M, true) : SCAIL_APG_UPDATE(F, M, false)
    if (avg)  // the diff is the average pass 1 wrote: the form only says where c is
        form == scail::CFGZ_PAIR ? SCAIL_APG_UPDATE_OUT(scail::CFGZ_PAIR, true) : SCAIL_APG_UPDATE_OUT(scail::CFGZ_CACHED, true);
    else if (form == scail::CFGZ_PAIR)
        SCAIL_APG_UPDATE_OUT(scail::CFGZ_PAIR, false);
    else if (form == scail::CFGZ_CACHED)
        SCAIL_APG_UPDATE_OUT(scail::CFGZ_CACHED, false);
    else
        SCAIL_APG_UPDATE_OUT(scail::CFGZ_FORECAST, false);
#undef SCAIL_APG_UPDATE_OUT
#undef SCAIL_APG_UPDATE
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_unipc_step_dpred(float* x, float* x_last, const float* m, float* slots, int64_t slot_stride, int64_t n_slots,
                           int64_t write_slot, int64_t n, int correct, const float* coef, scail_stream_t stream) {
    SCAIL_REQUIRE(x && x_last && m && slots && coef, "unipc_step_dpred: null operand");
    SCAIL_REQUIRE(aligned16(x) && aligned16(x_last) && aligned16(m) && aligned16(slots),
                  "unipc_step_dpred: x, x_last, m and slots must be 16-byte aligned");
    scail::UnipcCoef k;
    if (int rc = unipc_coef("unipc_step_dpred", slot_stride, n_slots, write_slot, n, coef, &k)) return rc;
    const int64_t nvec = n / 4;
    scail::unipc_step_kernel<false, false, false, true>
        <<<blocks_for(nvec, scail::UNIPC_THREADS), scail::UNIPC_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<float4*>(x), reinterpret_cast<float4*>(x_last), nullptr, slots, slot_stride, (int)n_slots,
            (int)write_slot, nvec, 0.f, 0.f, correct ? 1 : 0, k, nullptr, 0, scail::DeltaForecast{}, nullptr,
            reinterpret_cast<const float4*>(m));
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_cast_f32_bf16(const float* x, void* out, int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out, "cast: null operand");
    scail::cast_f32_to_bf16_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<__nv_bfloat16*>(out), n);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Shape checks shared by the three step-cache entry points; returns 0 or the fail() code.
static int step_cache_shape(const char* what, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq) {
    SCAIL_REQUIRE(B >= 1 && N >= 1 && d >= 8 && d % 8 == 0, "%s: need B >= 1, N >= 1 and d a positive multiple of 8 (got B=%lld, "
                  "N=%lld, d=%lld)", what, (long long)B, (long long)N, (long long)d);
    SCAIL_REQUIRE(n_ref >= 0 && n_seq >= 1 && n_ref + n_seq <= N, "%s: noise rows [n_ref, n_ref + n_seq) = [%lld, %lld) must lie "
                  "inside the N = %lld rows of a batch element", what, (long long)n_ref, (long long)(n_ref + n_seq), (long long)N);
    SCAIL_REQUIRE(B * N * (d / 8) < (int64_t(1) << 31), "%s: B * N * d / 8 must be < 2^31 (got %lld)", what,
                  (long long)(B * N * (d / 8)));
    return 0;
}

int scail_step_cache_indicator(const void* h0, const void* h1, const void* r_ref, void* r_new, void* h1c, float* partials,
                               int64_t partials_len, double* out, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq,
                               scail_stream_t stream) {
    SCAIL_REQUIRE(h0 && h1 && r_ref && r_new && h1c && partials && out, "step_cache_indicator: null operand");
    SCAIL_REQUIRE(aligned16(h0) && aligned16(h1) && aligned16(r_ref) && aligned16(r_new) && aligned16(h1c),
                  "step_cache_indicator: h0, h1, r_ref, r_new and h1c must be 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(partials) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0,
                  "step_cache_indicator: partials must be 4-byte and out 8-byte aligned");
    if (int rc = step_cache_shape("step_cache_indicator", B, N, d, n_ref, n_seq)) return rc;
    const int64_t nvec = B * N * (d / 8);
    const int ctas = static_cast<int>(std::min<int64_t>(scail::SC_MAX_CTAS, (nvec + scail::SC_THREADS - 1) / scail::SC_THREADS));
    SCAIL_REQUIRE(partials_len >= 2 * ctas, "step_cache_indicator: partials holds %lld floats, this shape needs %d",
                  (long long)partials_len, 2 * ctas);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    scail::step_cache_indicator_kernel<<<ctas, scail::SC_THREADS, 0, st>>>(
        static_cast<const uint4*>(h0), static_cast<const uint4*>(h1), static_cast<const uint4*>(r_ref), static_cast<uint4*>(r_new),
        static_cast<uint4*>(h1c), partials, nvec, static_cast<unsigned>(d / 8), static_cast<unsigned>(N), (int)n_ref, (int)n_seq);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    scail::step_cache_finish_kernel<<<1, scail::SC_THREADS, 0, st>>>(partials, ctas, out);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_step_cache_update(const void* h, const void* h1c, float* R, int64_t B, int64_t N, int64_t d, int64_t n_ref,
                            int64_t n_seq, scail_stream_t stream) {
    SCAIL_REQUIRE(h && h1c && R, "step_cache_update: null operand");
    SCAIL_REQUIRE(aligned16(h) && aligned16(h1c) && aligned16(R), "step_cache_update: h, h1c and R must be 16-byte aligned");
    if (int rc = step_cache_shape("step_cache_update", B, N, d, n_ref, n_seq)) return rc;
    const int64_t nvec = B * n_seq * (d / 8);
    scail::step_cache_update_kernel<<<blocks_for(nvec, scail::SC_THREADS), scail::SC_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(h), static_cast<const uint4*>(h1c), reinterpret_cast<float4*>(R), nvec, (int)(d / 8), (int)N,
        (int)n_ref, (int)n_seq);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_step_cache_apply(void* h, const float* R, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq,
                           scail_stream_t stream) {
    SCAIL_REQUIRE(h && R, "step_cache_apply: null operand");
    SCAIL_REQUIRE(aligned16(h) && aligned16(R), "step_cache_apply: h and R must be 16-byte aligned");
    if (int rc = step_cache_shape("step_cache_apply", B, N, d, n_ref, n_seq)) return rc;
    const int64_t nvec = B * n_seq * (d / 8);
    scail::step_cache_apply_kernel<<<blocks_for(nvec, scail::SC_THREADS), scail::SC_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<uint4*>(h), reinterpret_cast<const float4*>(R), nvec, (int)(d / 8), (int)N, (int)n_ref, (int)n_seq);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Slot checks shared by the two forecast entry points: 1 <= n_slots <= 3, and every slot is a whole, 16-byte aligned
// [B, n_seq, d] fp32 tensor that does not overlap the next one.
static int step_cache_slots(const char* what, int64_t slot_stride, int64_t n_slots, int64_t B, int64_t n_seq, int64_t d) {
    SCAIL_REQUIRE(n_slots >= 1 && n_slots <= scail::SC_MAX_SLOTS, "%s: need 1 <= n_slots <= %d (got %lld)", what,
                  scail::SC_MAX_SLOTS, (long long)n_slots);
    SCAIL_REQUIRE(slot_stride >= B * n_seq * d, "%s: slot_stride = %lld floats must be >= B * n_seq * d = %lld", what,
                  (long long)slot_stride, (long long)(B * n_seq * d));
    SCAIL_REQUIRE(slot_stride % 4 == 0, "%s: slot_stride = %lld floats must be a multiple of 4 so that every slot is 16-byte "
                  "aligned", what, (long long)slot_stride);
    return 0;
}

int scail_step_cache_update_slot(const void* h, const void* h1c, float* R_slots, int64_t slot_stride, int64_t n_slots,
                                 const int* slot, int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq,
                                 scail_stream_t stream) {
    SCAIL_REQUIRE(h && h1c && R_slots && slot, "step_cache_update_slot: null operand");
    SCAIL_REQUIRE(aligned16(h) && aligned16(h1c) && aligned16(R_slots),
                  "step_cache_update_slot: h, h1c and R_slots must be 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(slot) & 3) == 0, "step_cache_update_slot: slot must be 4-byte aligned");
    if (int rc = step_cache_shape("step_cache_update_slot", B, N, d, n_ref, n_seq)) return rc;
    if (int rc = step_cache_slots("step_cache_update_slot", slot_stride, n_slots, B, n_seq, d)) return rc;
    const int64_t nvec = B * n_seq * (d / 8);
    scail::step_cache_update_slot_kernel<<<blocks_for(nvec, scail::SC_THREADS), scail::SC_THREADS, 0,
                                           static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(h), static_cast<const uint4*>(h1c), R_slots, slot_stride, (int)n_slots, slot, nvec,
        (int)(d / 8), (int)N, (int)n_ref, (int)n_seq);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_step_cache_apply_forecast(void* h, const float* R_slots, int64_t slot_stride, int64_t n_slots, const float* coef,
                                    int64_t B, int64_t N, int64_t d, int64_t n_ref, int64_t n_seq, scail_stream_t stream) {
    SCAIL_REQUIRE(h && R_slots && coef, "step_cache_apply_forecast: null operand");
    SCAIL_REQUIRE(aligned16(h) && aligned16(R_slots), "step_cache_apply_forecast: h and R_slots must be 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(coef) & 3) == 0, "step_cache_apply_forecast: coef must be 4-byte aligned");
    if (int rc = step_cache_shape("step_cache_apply_forecast", B, N, d, n_ref, n_seq)) return rc;
    if (int rc = step_cache_slots("step_cache_apply_forecast", slot_stride, n_slots, B, n_seq, d)) return rc;
    const int64_t nvec = B * n_seq * (d / 8);
    scail::step_cache_apply_forecast_kernel<<<blocks_for(nvec, scail::SC_THREADS), scail::SC_THREADS, 0,
                                              static_cast<cudaStream_t>(stream)>>>(
        static_cast<uint4*>(h), R_slots, slot_stride, (int)n_slots, coef, nvec, (int)(d / 8), (int)N, (int)n_ref, (int)n_seq);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_conv3d_cl(const void* x, int64_t T, int64_t H, int64_t W, int64_t Cin, const void* w2, int64_t Cout, int KT,
                    int KH, int KW, const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo,
                    int64_t ocols, int fmul, int epilogue, const void* norm_gamma, void* out2, scail_stream_t stream) {
    return scail_conv3d_cl_hist(x, T, H, W, Cin, w2, Cout, KT, KH, KW, bias, residual, ldr, out, ldo, ocols, fmul, epilogue,
                                norm_gamma, out2, nullptr, 0, 0, 0, stream);
}

int scail_conv3d_cl_hist(const void* x, int64_t T, int64_t H, int64_t W, int64_t Cin, const void* w2, int64_t Cout, int KT,
                         int KH, int KW, const void* bias, const void* residual, int64_t ldr, void* out, int64_t ldo,
                         int64_t ocols, int fmul, int epilogue, const void* norm_gamma, void* out2, const void* hist,
                         int64_t T_hist, int64_t out_plane_stride, int64_t out_frame_offset, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(x && w2 && (out || (norm_gamma && out2)), "conv3d: null operand");
    SCAIL_REQUIRE((norm_gamma == nullptr) == (out2 == nullptr), "conv3d: norm_gamma and out2 come together");
    if (norm_gamma) SCAIL_REQUIRE(KH == 3 && KW == 3 && W >= 128 && Cout == 96 && epilogue != CONV_EPI_HEAD_CLAMP && fmul <= 1,
                                  "conv3d: the fused RMS_norm+SiLU output needs the row-tile kernel with Cout == 96 (3x3 taps, W >= 128)");
    SCAIL_REQUIRE(T > 0 && H > 0 && W > 0 && Cin % 8 == 0 && Cout > 0, "conv3d: bad shape");
    SCAIL_REQUIRE(KT >= 1 && KT <= 3 && KH >= 1 && KH <= 3 && KW >= 1 && KW <= 3 && (KH & 1) && (KW & 1), "conv3d: taps must be 1 or 3");
    SCAIL_REQUIRE(epilogue >= 0 && epilogue <= 2, "conv3d: unknown epilogue");
    if (epilogue == CONV_EPI_BIAS_RES) SCAIL_REQUIRE(residual && ldr % 8 == 0, "conv3d: residual required");
    SCAIL_REQUIRE(aligned16(out) && aligned16(bias) && aligned16(residual) && aligned16(out2), "conv3d: out, bias, residual must be 16-byte aligned");
    if (epilogue == CONV_EPI_HEAD_CLAMP) SCAIL_REQUIRE(bias && Cout <= 16, "conv3d: head epilogue needs bias and Cout <= 16");
    else SCAIL_REQUIRE(Cout % 8 == 0 && ldo % 8 == 0 && ocols > 0 && ocols % 8 == 0, "conv3d: Cout, ldo, ocols must be multiples of 8");
    SCAIL_REQUIRE(T_hist >= 0 && T_hist <= KT - 1, "conv3d: T_hist=%lld must be in [0, KT-1=%d]", (long long)T_hist, KT - 1);
    SCAIL_REQUIRE(T_hist == 0 || (hist && aligned16(hist)), "conv3d: a history of T_hist > 0 frames needs a 16-byte aligned hist");
    const int64_t plane = out_plane_stride > 0 ? out_plane_stride : T * H * W;
    if (epilogue == CONV_EPI_HEAD_CLAMP)
        SCAIL_REQUIRE(out_frame_offset >= 0 && out_plane_stride >= 0 && plane >= (out_frame_offset + T) * H * W,
                      "conv3d: head output planes of %lld elements cannot hold frames [%lld, %lld)", (long long)plane,
                      (long long)out_frame_offset, (long long)(out_frame_offset + T));
    else SCAIL_REQUIRE(out_plane_stride == 0 && out_frame_offset == 0, "conv3d: out_plane_stride / out_frame_offset are head-epilogue only");
    const int taps = KT * KH * KW;
    CUtensorMap tx, tw, th;
    int rc;
    if ((rc = make_tmap_cl4d(x, T, H, W, Cin, &tx))) return rc;
    th = tx;  // not read when T_hist == 0
    if (T_hist > 0 && (rc = make_tmap_cl4d(hist, T_hist, H, W, Cin, &th))) return rc;
    const int BN = Cout <= 16 ? 16 : (Cout <= 96 ? 96 : 192);
    if ((rc = make_tmap_2d(w2, Cout, (uint64_t)taps * Cin, (uint64_t)taps * Cin, BN, 64, &tw))) return rc;
    ConvParams p;
    p.T = (int)T; p.H = (int)H; p.W = (int)W; p.Cin = (int)Cin; p.Cout = (int)Cout; p.KT = KT; p.KH = KH; p.KW = KW;
    p.bias = static_cast<const __nv_bfloat16*>(bias); p.residual = static_cast<const __nv_bfloat16*>(residual);
    p.out = out; p.ldo = ldo; p.ldr = ldr; p.ocols = (int)(ocols > 0 ? ocols : Cout); p.fmul = fmul > 0 ? fmul : 1;
    p.epilogue = epilogue;
    p.norm_gamma = static_cast<const __nv_bfloat16*>(norm_gamma); p.out2 = static_cast<__nv_bfloat16*>(out2);
    p.sstride = 1; p.pad_h = KH / 2; p.pad_w = KW / 2; p.tstride = 1; p.toff = -(KT - 1);
    p.T_hist = (int)T_hist;
    if (epilogue == CONV_EPI_HEAD_CLAMP) {  // plane stride in ldo; `out` starts at frame out_frame_offset of every plane
        p.ldo = plane;
        p.out = static_cast<float*>(out) + out_frame_offset * H * W;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    static const bool row_ok_env = !(getenv("SCAIL_CONV_ROW") && atoi(getenv("SCAIL_CONV_ROW")) == 0);
    const bool row_head = epilogue == CONV_EPI_HEAD_CLAMP && Cout <= 16;
    if (norm_gamma) SCAIL_REQUIRE(row_ok_env, "conv3d: fused norm output requested but SCAIL_CONV_ROW=0");
    if (row_ok_env && KH == 3 && KW == 3 && W >= 128 && (Cout % 96 == 0 || row_head) && fmul <= 1 && (ocols <= 0 || ocols == Cout)) {
        // row-tile kernel: 2 output rows x 128 pixels x BN channels per iteration, taps as shifted smem views
        const int RBN = row_head ? 16 : 96;
        CUtensorMap txr, twr, thr;
        if ((rc = make_tmap_cl4d(x, T, H, W, Cin, &txr, CROW_A_ROWS, 2))) return rc;
        if ((rc = make_tmap_2d(w2, Cout, (uint64_t)taps * Cin, (uint64_t)taps * Cin, RBN, 64, &twr))) return rc;
        thr = txr;
        if (T_hist > 0 && (rc = make_tmap_cl4d(hist, T_hist, H, W, Cin, &thr, CROW_A_ROWS, 2))) return rc;
        const int tiles = (int)(T * ((H + 1) / 2) * blocks_for(W, CROW_PW) * blocks_for(Cout, RBN));
        const int sms = sm_count();
        SCAIL_REQUIRE(sms > 0, "conv3d: no CUDA device");
        const int grid = tiles < sms ? tiles : sms;
        if (row_head) {
            if ((rc = set_smem(conv3d_row_kernel<16>, ConvRowCfg<16>::SMEM_BYTES))) return rc;
            conv3d_row_kernel<16><<<grid, CONV_THREADS, ConvRowCfg<16>::SMEM_BYTES, st>>>(txr, twr, thr, p);
        } else {
            if ((rc = set_smem(conv3d_row_kernel<96>, ConvRowCfg<96>::SMEM_BYTES))) return rc;
            conv3d_row_kernel<96><<<grid, CONV_THREADS, ConvRowCfg<96>::SMEM_BYTES, st>>>(txr, twr, thr, p);
        }
        SCAIL_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    if (BN == 16) return launch_conv<16>(tx, tw, th, p, st);
    if (BN == 96) return launch_conv<96>(tx, tw, th, p, st);
    return launch_conv<192>(tx, tw, th, p, st);
}

int scail_conv3d_strided_cl(const void* x, int64_t T_in, int64_t H_in, int64_t W_in, int64_t Cin, const void* w2, int64_t Cout,
                            int KT, int KH, int KW, const void* bias, void* out, int64_t ldo, int64_t T_out, int64_t H_out,
                            int64_t W_out, int sstride, int pad_h, int pad_w, int tstride, int toff, scail_stream_t stream) {
    return scail_conv3d_strided_cl_hist(x, T_in, H_in, W_in, Cin, w2, Cout, KT, KH, KW, bias, out, ldo, T_out, H_out, W_out,
                                        sstride, pad_h, pad_w, tstride, toff, nullptr, 0, stream);
}

int scail_conv3d_strided_cl_hist(const void* x, int64_t T_in, int64_t H_in, int64_t W_in, int64_t Cin, const void* w2,
                                 int64_t Cout, int KT, int KH, int KW, const void* bias, void* out, int64_t ldo, int64_t T_out,
                                 int64_t H_out, int64_t W_out, int sstride, int pad_h, int pad_w, int tstride, int toff,
                                 const void* hist, int64_t T_hist, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(x && w2 && out, "conv3d_strided: null operand");
    SCAIL_REQUIRE(Cin % 8 == 0 && Cout % 8 == 0 && ldo % 8 == 0, "conv3d_strided: channels must be multiples of 8");
    SCAIL_REQUIRE((sstride == 1 || sstride == 2) && (tstride == 1 || tstride == 2), "conv3d_strided: strides must be 1 or 2");
    SCAIL_REQUIRE(KT >= 1 && KT <= 3 && KH >= 1 && KH <= 3 && KW >= 1 && KW <= 3, "conv3d_strided: taps must be 1..3");
    SCAIL_REQUIRE(T_hist >= 0 && T_hist <= KT - 1, "conv3d_strided: T_hist=%lld must be in [0, KT-1=%d]", (long long)T_hist, KT - 1);
    SCAIL_REQUIRE(T_hist == 0 || (hist && aligned16(hist)), "conv3d_strided: a history of T_hist > 0 frames needs a 16-byte aligned hist");
    const int taps = KT * KH * KW;
    CUtensorMap tx, tw, th;
    int rc;
    if ((rc = make_tmap_cl4d(x, T_in, H_in, W_in, Cin, &tx, 16 * sstride, 8 * sstride, sstride))) return rc;
    th = tx;  // not read when T_hist == 0
    if (T_hist > 0 && (rc = make_tmap_cl4d(hist, T_hist, H_in, W_in, Cin, &th, 16 * sstride, 8 * sstride, sstride))) return rc;
    const int BN = Cout <= 16 ? 16 : (Cout <= 96 ? 96 : 192);
    if ((rc = make_tmap_2d(w2, Cout, (uint64_t)taps * Cin, (uint64_t)taps * Cin, BN, 64, &tw))) return rc;
    ConvParams p;
    p.T = (int)T_out; p.H = (int)H_out; p.W = (int)W_out; p.Cin = (int)Cin; p.Cout = (int)Cout; p.KT = KT; p.KH = KH; p.KW = KW;
    p.bias = static_cast<const __nv_bfloat16*>(bias); p.residual = nullptr; p.out = out; p.ldo = ldo; p.ldr = 0;
    p.ocols = (int)Cout; p.fmul = 1; p.epilogue = CONV_EPI_BIAS; p.norm_gamma = nullptr; p.out2 = nullptr;
    p.sstride = sstride; p.pad_h = pad_h; p.pad_w = pad_w; p.tstride = tstride; p.toff = toff;
    p.T_hist = (int)T_hist;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (BN == 16) return launch_conv<16>(tx, tw, th, p, st);
    if (BN == 96) return launch_conv<96>(tx, tw, th, p, st);
    return launch_conv<192>(tx, tw, th, p, st);
}

int scail_rmsnorm_cl(const void* x, const void* gamma, void* out, int64_t npix, int64_t C, int silu, scail_stream_t stream) {
    SCAIL_REQUIRE(x && gamma && out, "rmsnorm_cl: null operand");
    auto st = static_cast<cudaStream_t>(stream);
    switch (C) {  // C = 8 * LP * VPL
        case 16:  return launch_rmsnorm_cl<2, 1>(x, gamma, out, npix, 16, silu, st);
        case 32:  return launch_rmsnorm_cl<4, 1>(x, gamma, out, npix, 32, silu, st);
        case 64:  return launch_rmsnorm_cl<8, 1>(x, gamma, out, npix, 64, silu, st);
        case 96:  return launch_rmsnorm_cl<4, 3>(x, gamma, out, npix, 96, silu, st);
        case 128: return launch_rmsnorm_cl<16, 1>(x, gamma, out, npix, 128, silu, st);
        case 192: return launch_rmsnorm_cl<8, 3>(x, gamma, out, npix, 192, silu, st);
        case 256: return launch_rmsnorm_cl<16, 2>(x, gamma, out, npix, 256, silu, st);
        case 384: return launch_rmsnorm_cl<16, 3>(x, gamma, out, npix, 384, silu, st);
        case 512: return launch_rmsnorm_cl<16, 4>(x, gamma, out, npix, 512, silu, st);
        default:  return fail(-1, "rmsnorm_cl: unsupported channel count %lld (supported: 16,32,64,96,128,192,256,384,512)", (long long)C);
    }
}

int scail_upsample2x_cl(const void* x, void* out, int64_t frames, int64_t H, int64_t W, int64_t C, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out && C % 8 == 0, "upsample2x_cl: bad args");
    const int64_t total = frames * 4 * H * W * (C / 8);
    scail::upsample2x_cl_kernel<<<blocks_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint4*>(x), static_cast<uint4*>(out), frames, (int)H, (int)W, (int)(C / 8));
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_vae_latent_to_cl(const void* z, const float* mean, const float* inv_std, void* out, int64_t T, int64_t h,
                           int64_t w, scail_stream_t stream) {
    SCAIL_REQUIRE(z && mean && inv_std && out, "vae_latent_to_cl: null operand");
    scail::vae_latent_to_cl_kernel<<<blocks_for(T * h * w * 16, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(z), mean, inv_std, static_cast<__nv_bfloat16*>(out), (int)T, (int)h, (int)w);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_softmax_rows(const float* s, void* p, int64_t rows, int64_t cols, float scale, scail_stream_t stream) {
    SCAIL_REQUIRE(s && p && rows > 0 && cols > 0, "softmax_rows: bad args");
    scail::softmax_rows_kernel<<<blocks_for(rows, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        s, static_cast<__nv_bfloat16*>(p), (int)rows, (int)cols, scale);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// Context-parallel collective (SURVEY.md 8b "collective"): the one exchange step of the path -- the per-block K/V all-gather
// over the sequence-parallel group -- behind the C ABI, on a library-owned communication stream with event hand-off.
// NCCL is bound at run time (dlopen of the libnccl.so.2 the process already uses, i.e. PyTorch's): no link-time dependency,
// and nothing here exists without it (no fallback: scail_cp_init fails loudly).
namespace {

struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
struct UniqueId { char b[128]; };
typedef int (*CommInitRankFn)(void**, int, UniqueId, int);
NcclApi g_nccl;
CommInitRankFn g_nccl_init = nullptr;

int load_nccl(const char* path) {
    if (g_nccl.lib) return 0;
    const char* names[] = {path, "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
        if (!n || !*n) continue;
        g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
        if (g_nccl.lib) break;
    }
    if (!g_nccl.lib) return fail(-4, "cp: cannot dlopen libnccl (%s)", dlerror());
    g_nccl.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(g_nccl.lib, "ncclGetUniqueId"));
    g_nccl_init = reinterpret_cast<CommInitRankFn>(dlsym(g_nccl.lib, "ncclCommInitRank"));
    g_nccl.AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(dlsym(g_nccl.lib, "ncclAllGather"));
    g_nccl.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(g_nccl.lib, "ncclCommDestroy"));
    g_nccl.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(g_nccl.lib, "ncclGetErrorString"));
    if (!g_nccl.GetUniqueId || !g_nccl_init || !g_nccl.AllGather || !g_nccl.CommDestroy) {
        g_nccl.lib = nullptr;
        return fail(-4, "cp: libnccl lacks a required symbol");
    }
    return 0;
}

struct CpGroup {
    void* comm = nullptr;
    int rank = 0, nranks = 0;
    cudaStream_t stream = nullptr;   // library-owned communication stream
    cudaEvent_t ready = nullptr;     // recorded on the caller's stream before a collective
    cudaEvent_t done = nullptr;      // recorded on the communication stream after the last collective
};
constexpr int MAX_CP_GROUPS = 16;
CpGroup g_cp[MAX_CP_GROUPS];

#define SCAIL_CHECK_NCCL(expr)                                                                                       \
    do {                                                                                                             \
        int _r = (expr);                                                                                             \
        if (_r != 0) return fail(-4, "%s: %s", #expr, g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "nccl error"); \
    } while (0)

}  // namespace

/* 128-byte NCCL unique id for a new group (call on one rank, ship to the others with any host-side channel). */
int scail_cp_unique_id(void* out128, const char* nccl_path) {
    SCAIL_REQUIRE(out128, "cp_unique_id: null");
    int rc;
    if ((rc = load_nccl(nccl_path))) return rc;
    SCAIL_CHECK_NCCL(g_nccl.GetUniqueId(out128));
    return 0;
}

/* Join the group; the current CUDA device is the rank's GPU.  Returns a handle >= 0. */
int scail_cp_init(const void* unique_id128, int rank, int nranks, const char* nccl_path) {
    SCAIL_REQUIRE(unique_id128 && nranks >= 1 && rank >= 0 && rank < nranks, "cp_init: bad args");
    int rc;
    if ((rc = load_nccl(nccl_path))) return rc;
    int h = -1;
    {
        std::lock_guard<std::mutex> lk(g_map_mu);
        for (int i = 0; i < MAX_CP_GROUPS; ++i)
            if (!g_cp[i].comm) { h = i; break; }
    }
    SCAIL_REQUIRE(h >= 0, "cp_init: too many groups");
    UniqueId id;
    memcpy(id.b, unique_id128, 128);
    CpGroup g;
    g.rank = rank; g.nranks = nranks;
    SCAIL_CHECK_NCCL(g_nccl_init(&g.comm, nranks, id, rank));
    int lo = 0, hi = 0;
    SCAIL_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    SCAIL_CHECK_CUDA(cudaStreamCreateWithPriority(&g.stream, cudaStreamNonBlocking, hi));  // highest priority: gathers first
    SCAIL_CHECK_CUDA(cudaEventCreateWithFlags(&g.ready, cudaEventDisableTiming));
    SCAIL_CHECK_CUDA(cudaEventCreateWithFlags(&g.done, cudaEventDisableTiming));
    std::lock_guard<std::mutex> lk(g_map_mu);
    g_cp[h] = g;
    return h;
}

/* In-place-capable all-gather of `bytes_per_rank` bytes: recv holds nranks consecutive slots, rank r's slot is
 * recv + r * bytes_per_rank (send may alias this rank's slot).  Ordered after everything already enqueued on
 * `compute_stream`; runs on the group's own stream; returns immediately (scail_cp_wait joins). */
int scail_cp_allgather(int handle, const void* send, void* recv, int64_t bytes_per_rank, scail_stream_t compute_stream) {
    SCAIL_REQUIRE(handle >= 0 && handle < MAX_CP_GROUPS && g_cp[handle].comm, "cp_allgather: bad handle");
    SCAIL_REQUIRE(send && recv && bytes_per_rank > 0, "cp_allgather: bad args");
    CpGroup& g = g_cp[handle];
    SCAIL_CHECK_CUDA(cudaEventRecord(g.ready, static_cast<cudaStream_t>(compute_stream)));
    SCAIL_CHECK_CUDA(cudaStreamWaitEvent(g.stream, g.ready, 0));
    SCAIL_CHECK_NCCL(g_nccl.AllGather(send, recv, static_cast<size_t>(bytes_per_rank), /*ncclInt8*/ 0, g.comm, g.stream));
    SCAIL_CHECK_CUDA(cudaEventRecord(g.done, g.stream));
    return 0;
}

/* Make `compute_stream` wait for every collective enqueued on the group so far (device-side, no host sync). */
int scail_cp_wait(int handle, scail_stream_t compute_stream) {
    SCAIL_REQUIRE(handle >= 0 && handle < MAX_CP_GROUPS && g_cp[handle].comm, "cp_wait: bad handle");
    SCAIL_CHECK_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(compute_stream), g_cp[handle].done, 0));
    return 0;
}

int scail_cp_destroy(int handle) {
    SCAIL_REQUIRE(handle >= 0 && handle < MAX_CP_GROUPS && g_cp[handle].comm, "cp_destroy: bad handle");
    CpGroup g = g_cp[handle];
    cudaStreamSynchronize(g.stream);
    g_nccl.CommDestroy(g.comm);
    cudaEventDestroy(g.ready);
    cudaEventDestroy(g.done);
    cudaStreamDestroy(g.stream);
    std::lock_guard<std::mutex> lk(g_map_mu);
    g_cp[handle] = CpGroup();
    return 0;
}

}  // extern "C"
