// UniPC multistep flow solver (scail_b200/unipc.py): one fused pass over the fp32 latent per sampler step.  The host
// composes the step's linear combination in fp64 and passes each coefficient, rounded once to fp32, by value.  Every thread
// moves 4 elements: 16-byte vectors of the fp32 tensors and 8-byte vectors of the bf16 CFG pair.
#pragma once
#include <cuda_bf16.h>

namespace scail {

constexpr int UNIPC_THREADS = 256;
constexpr int UNIPC_MAX_SLOTS = 3;

// a_x * x_last + sum a[k] * M_k + a_m * m  (corrector), then  b_y * y + sum b[k] * M_k + b_m * m  (predictor)
struct UnipcCoef {
    float a_x, a[UNIPC_MAX_SLOTS], a_m, b_y, b[UNIPC_MAX_SLOTS], b_m;
};

__device__ __forceinline__ void unipc_unpack4(const uint2& u, float (&f)[4]) {
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&u);
    const float2 lo = __bfloat1622float2(p[0]), hi = __bfloat1622float2(p[1]);
    f[0] = lo.x; f[1] = lo.y; f[2] = hi.x; f[3] = hi.y;
}

__device__ __forceinline__ void unipc_load(const float4* p, int64_t i, float (&f)[4]) {
    const float4 t = p[i];
    f[0] = t.x; f[1] = t.y; f[2] = t.z; f[3] = t.w;
}

// acc = acc + c * M (or acc = c * M when `first`), each product and sum rounded on its own.
__device__ __forceinline__ void unipc_axpy(float (&acc)[4], float c, const float (&M)[4], bool first) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float p = __fmul_rn(c, M[j]);
        acc[j] = first ? p : __fadd_rn(acc[j], p);
    }
}

// The CFG cache's forecast of delta = c - u (scail_b200/cfg_cache.py, order >= 1): the host's fp32 coefficient of each of
// up to DELTA_MAX_SLOTS fp32 slots of delta, slot s at `slots + s * slot_stride` floats.
constexpr int DELTA_MAX_SLOTS = 3;
struct DeltaForecast {
    float c[DELTA_MAX_SLOTS];
};

// t = c0*S0, then t = t + c1*S1, then t = t + c2*S2 at vector i, each product and sum rounded on its own (no FMA).  A slot
// whose coefficient is exactly 0 is neither read nor added, so stale or NaN slots cannot leak, and c = (1, 0, 0) gives S0
// bit for bit; with no active slot t = 0.
__device__ __forceinline__ void delta_forecast4(const float* slots, int64_t slot_stride, const DeltaForecast& k, int64_t i,
                                                float (&t)[4]) {
    bool first = true;
#pragma unroll
    for (int s = 0; s < DELTA_MAX_SLOTS; ++s) {
        if (k.c[s] == 0.f) continue;
        float S[4];
        unipc_load(reinterpret_cast<const float4*>(slots + s * slot_stride), i, S);
        unipc_axpy(t, k.c[s], S, first);
        first = false;
    }
    if (first) {
#pragma unroll
        for (int j = 0; j < 4; ++j) t[j] = 0.f;
    }
}

// In fixed order, per element: g = u + s*(c - u); m = x - sigma*g; y = a_x*x_last + a[k]*M_k (slot order) + a_m*m when
// `correct`, else y = x; z = b_y*y + b[k]*M_k (slot order) + b_m*m.  Writes x = z, x_last = y and slot `write_slot` = m.
// A slot whose a[k] and b[k] are both exactly 0 is not read, and a term with a zero slot coefficient is not added, so stale
// or NaN slots cannot leak.  Every thread reads all it needs before it writes, so the write slot may be one it reads.
// kCached = false: v is the bf16 CFG pair [2, nvec * 4] and `delta` is not read.  kCached = true (the CFG cache's
// conditional-only step, scail_b200/cfg_cache.py): v is the conditional output alone [nvec * 4] and u = f32(c) - delta;
// every instruction after that is shared.  kForecast (with kCached; CFGCache(order >= 1)): delta is the forecast
// delta_forecast4 of the slots at `delta` (stride delta_stride floats) with the coefficients dk, in place of one held
// delta.  `delta`, delta_stride and dk are the last parameters, so the other parameters keep their offsets.
// kScaled (CFG-Zero*, scail_b200/guidance.py): u = (*u_scale) * u, one rounded product, once u is formed; the rest is
// unchanged, so *u_scale == 1 gives the unscaled step bit for bit.  u_scale is not read otherwise.
// kDataPred (APG, scail_b200/guidance.py): m is read from `mpred` (fp32, the guidance's data prediction) in place of
// x - sigma*g, and v, delta, u_scale, scale and sigma are not read; every instruction after m is shared.  mpred is the last
// parameter and is not read otherwise.
template <bool kCached, bool kForecast = false, bool kScaled = false, bool kDataPred = false>
__global__ void __launch_bounds__(UNIPC_THREADS) unipc_step_kernel(float4* __restrict__ x, float4* __restrict__ x_last,
                                                                   const uint2* __restrict__ v, float* __restrict__ slots,
                                                                   int64_t slot_stride, int n_slots, int write_slot,
                                                                   int64_t nvec, float scale, float sigma, int correct,
                                                                   UnipcCoef k, const float4* __restrict__ delta,
                                                                   int64_t delta_stride, DeltaForecast dk,
                                                                   const float* __restrict__ u_scale,
                                                                   const float4* __restrict__ mpred) {
    static_assert(kCached || !kForecast, "the forecast form is a cached step");
    static_assert(!kDataPred || (!kCached && !kScaled), "the data-prediction form reads m alone");
    const int64_t i = static_cast<int64_t>(blockIdx.x) * UNIPC_THREADS + threadIdx.x;
    if (i >= nvec) return;
    float fx[4], fu[4], fc[4], m[4], y[4], z[4];
    unipc_load(x, i, fx);
    if constexpr (kDataPred) {
        unipc_load(mpred, i, m);
    } else if constexpr (kCached) {
        float fd[4];
        unipc_unpack4(v[i], fc);
        if constexpr (kForecast)
            delta_forecast4(reinterpret_cast<const float*>(delta), delta_stride, dk, i, fd);
        else
            unipc_load(delta, i, fd);
#pragma unroll
        for (int j = 0; j < 4; ++j) fu[j] = __fsub_rn(fc[j], fd[j]);
    } else {
        unipc_unpack4(v[i], fu);
        unipc_unpack4(v[nvec + i], fc);
    }
    if constexpr (kScaled) {
        const float su = *u_scale;
#pragma unroll
        for (int j = 0; j < 4; ++j) fu[j] = __fmul_rn(su, fu[j]);
    }
    float M[UNIPC_MAX_SLOTS][4];
#pragma unroll
    for (int s = 0; s < UNIPC_MAX_SLOTS; ++s)
        if (s < n_slots && (k.a[s] != 0.f || k.b[s] != 0.f))
            unipc_load(reinterpret_cast<const float4*>(slots + s * slot_stride), i, M[s]);
    if constexpr (!kDataPred) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float g = __fadd_rn(fu[j], __fmul_rn(scale, __fsub_rn(fc[j], fu[j])));
            m[j] = __fsub_rn(fx[j], __fmul_rn(sigma, g));
        }
    }
    if (correct) {
        float xl[4];
        unipc_load(x_last, i, xl);
        unipc_axpy(y, k.a_x, xl, true);
#pragma unroll
        for (int s = 0; s < UNIPC_MAX_SLOTS; ++s)
            if (s < n_slots && k.a[s] != 0.f) unipc_axpy(y, k.a[s], M[s], false);
        unipc_axpy(y, k.a_m, m, false);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = fx[j];
    }
    unipc_axpy(z, k.b_y, y, true);
#pragma unroll
    for (int s = 0; s < UNIPC_MAX_SLOTS; ++s)
        if (s < n_slots && k.b[s] != 0.f) unipc_axpy(z, k.b[s], M[s], false);
    unipc_axpy(z, k.b_m, m, false);
    x[i] = make_float4(z[0], z[1], z[2], z[3]);
    x_last[i] = make_float4(y[0], y[1], y[2], y[3]);
    reinterpret_cast<float4*>(slots + write_slot * slot_stride)[i] = make_float4(m[0], m[1], m[2], m[3]);
}

}  // namespace scail
