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
#include "attention.cuh"
#include "conv.cuh"
#include "gemm.cuh"
#include "rowops.cuh"

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

template <int EPI>
static int launch_gemm_fp8(const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tc, const CUtensorMap& tr,
                           const scail::GemmParams& p, int grid, cudaStream_t st) {
    using namespace scail;
    constexpr int smem = GemmCfg<true>::SMEM_BYTES;
    int rc;
    if ((rc = set_smem(gemm_fp8_kernel<EPI>, smem))) return rc;
    gemm_fp8_kernel<EPI><<<grid, GEMM_THREADS, smem, st>>>(ta, tw, tc, tr, p);
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

int scail_gemm_fp8(const void* A, int64_t lda, const void* W, int64_t ldw, const void* bias, void* C, int64_t ldc,
                   int64_t M, int64_t N, int64_t K, int epilogue, const void* gate, int64_t gate_stride,
                   int64_t rows_per_batch, const void* residual, int64_t ldr, int c_fp32, const float* scale_a,
                   const float* scale_w, scail_stream_t stream) {
    using namespace scail;
    using Cfg = GemmCfg<true>;
    SCAIL_REQUIRE(A && W && C && scale_a && scale_w, "gemm_fp8: null operand");
    SCAIL_REQUIRE(!c_fp32, "gemm_fp8: the output is bf16 (c_fp32 must be 0)");
    SCAIL_REQUIRE(M > 0 && N > 0 && K > 0, "gemm_fp8: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
    SCAIL_REQUIRE(K % 16 == 0 && lda % 16 == 0 && ldw % 16 == 0,
                  "gemm_fp8: K, lda and ldw must be multiples of 16 (16-byte e4m3 row pitch)");
    SCAIL_REQUIRE(N % 8 == 0 && ldc % 8 == 0, "gemm_fp8: N and ldc must be multiples of 8");
    SCAIL_REQUIRE(aligned16(C) && aligned16(bias) && aligned16(gate) && aligned16(residual),
                  "gemm_fp8: C, bias, gate and residual must be 16-byte aligned (the epilogue uses 16-byte accesses)");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(scale_a) & 3) == 0 && (reinterpret_cast<uintptr_t>(scale_w) & 3) == 0,
                  "gemm_fp8: scales must be 4-byte aligned float32");
    SCAIL_REQUIRE(epilogue >= 0 && epilogue <= 5, "gemm_fp8: unknown epilogue %d", epilogue);
    if (epilogue == EPI_BIAS_GATE_RES) SCAIL_REQUIRE(gate && residual && gate_stride % 8 == 0, "gemm_fp8: gate/residual required");
    if (epilogue == EPI_BIAS_RES) SCAIL_REQUIRE(residual, "gemm_fp8: residual required");
    if (residual) SCAIL_REQUIRE(ldr % 8 == 0, "gemm_fp8: ldr must be a multiple of 8");
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
    SCAIL_REQUIRE(sms > 0, "gemm_fp8: no CUDA device");
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
        case EPI_BIAS: return launch_gemm_fp8<EPI_BIAS>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GELU: return launch_gemm_fp8<EPI_BIAS_GELU>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_SILU: return launch_gemm_fp8<EPI_BIAS_SILU>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GELU_ERF: return launch_gemm_fp8<EPI_BIAS_GELU_ERF>(ta, tw, tc, tr, p, grid, st);
        case EPI_BIAS_GATE_RES: return launch_gemm_fp8<EPI_BIAS_GATE_RES>(ta, tw, tc, tr, p, grid, st);
        default: return launch_gemm_fp8<EPI_BIAS_RES>(ta, tw, tc, tr, p, grid, st);
    }
}

int scail_quant_rows_fp8(const void* x, int64_t ldx, void* q, float* scale, int64_t M, int64_t K, scail_stream_t stream) {
    using namespace scail;
    SCAIL_REQUIRE(x && q && scale, "quant_rows_fp8: null operand");
    SCAIL_REQUIRE(M > 0 && K > 0 && K % 16 == 0 && ldx % 8 == 0 && aligned16(x) && aligned16(q),
                  "quant_rows_fp8: K must be a multiple of 16, ldx of 8, x and q 16-byte aligned");
    SCAIL_REQUIRE((reinterpret_cast<uintptr_t>(scale) & 3) == 0, "quant_rows_fp8: scale must be 4-byte aligned float32");
    auto xp = static_cast<const __nv_bfloat16*>(x);
    auto qp = static_cast<uint8_t*>(q);
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int vpt = blocks_for(K / 8, ROW_THREADS);  // 16-byte vectors per thread
    if (vpt <= 4) quant_rows_fp8_kernel<4><<<(unsigned)M, ROW_THREADS, 0, st>>>(xp, ldx, qp, scale, (int)K);
    else if (vpt <= 8) quant_rows_fp8_kernel<8><<<(unsigned)M, ROW_THREADS, 0, st>>>(xp, ldx, qp, scale, (int)K);
    else if (vpt <= 16) quant_rows_fp8_kernel<16><<<(unsigned)M, ROW_THREADS, 0, st>>>(xp, ldx, qp, scale, (int)K);
    else return fail(-1, "quant_rows_fp8: K=%lld exceeds %d", (long long)K, 16 * ROW_THREADS * 8);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int ln_modulate_impl(const void* x, void* out, void* out_q, float* out_scale, const void* gamma, const void* beta,
                            const void* shift, const void* scale, int64_t mod_stride, int64_t B, int64_t rows_out,
                            int64_t in_batch_rows, int64_t in_row_offset, int64_t D, float eps, scail_stream_t stream) {
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
    if (out_q) ln_modulate_kernel<true><<<p.total_rows, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
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
    rmsnorm_rope_kernel<<<grid, ROW_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

static int attention_impl(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                          int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_off0, int64_t kv_len0, int64_t kv_off1,
                          int64_t kv_len1, int64_t q_batch_rows, int64_t kv_batch_rows, int64_t q_rows_total,
                          int64_t kv_rows_total, float scale, int accumulate, float* o32, int64_t ldo32, void* state,
                          scail_stream_t stream) {
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
    if ((rc = set_smem(attention_fwd_kernel, ATT_SMEM_BYTES))) return rc;
    dim3 grid(blocks_for(q_len, ATT_BQ), (unsigned)H, (unsigned)B);
    attention_fwd_kernel<<<grid, ATT_THREADS, ATT_SMEM_BYTES, static_cast<cudaStream_t>(stream)>>>(tq, tk, tv, p);
    SCAIL_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scail_attention(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, void* out,
                    int64_t ldo, int64_t B, int64_t H, int64_t q_len, int64_t kv_len, int64_t q_batch_rows,
                    int64_t kv_batch_rows, int64_t q_rows_total, int64_t kv_rows_total, float scale, int accumulate,
                    scail_stream_t stream) {
    return attention_impl(Q, ldq, K, ldk, V, ldv, out, ldo, B, H, q_len, 0, kv_len, 0, 0, q_batch_rows, kv_batch_rows, q_rows_total,
                          kv_rows_total, scale, accumulate, nullptr, 0, nullptr, stream);
}

int scail_attention_partial(const void* Q, int64_t ldq, const void* K, int64_t ldk, const void* V, int64_t ldv, float* o32,
                            int64_t ldo32, void* state, int64_t B, int64_t H, int64_t q_len, int64_t kv_off0, int64_t kv_len0,
                            int64_t kv_off1, int64_t kv_len1, int64_t q_batch_rows, int64_t kv_batch_rows, int64_t q_rows_total,
                            int64_t kv_rows_total, float scale, scail_stream_t stream) {
    SCAIL_REQUIRE(o32 && state, "attention_partial: null operand");
    return attention_impl(Q, ldq, K, ldk, V, ldv, nullptr, 8, B, H, q_len, kv_off0, kv_len0, kv_off1, kv_len1, q_batch_rows,
                          kv_batch_rows, q_rows_total, kv_rows_total, scale, 0, o32, ldo32, state, stream);
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

int scail_cast_f32_bf16(const float* x, void* out, int64_t n, scail_stream_t stream) {
    SCAIL_REQUIRE(x && out, "cast: null operand");
    scail::cast_f32_to_bf16_kernel<<<blocks_for(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, static_cast<__nv_bfloat16*>(out), n);
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
