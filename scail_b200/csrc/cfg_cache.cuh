// CFG cache (scail_b200/cfg_cache.py): the two HBM-bound passes around a conditional-only sampler step.  A full step keeps
// delta = f32(c) - f32(u) of its CFG pair (fp32, one subtraction rounded once) and measures how far it moved since the last
// full step; a conditional-only step rebuilds u = f32(c) - delta.  Every thread moves 4 elements: 16-byte vectors of the
// fp32 tensors and 8-byte vectors of bf16, as the UniPC step does.
#pragma once
#include <cuda_bf16.h>

#include "solver.cuh"      // unipc_unpack4, unipc_load, DeltaForecast, delta_forecast4
#include "step_cache.cuh"  // SC_THREADS, SC_MAX_CTAS, sc_write_partials, step_cache_finish_kernel

namespace scail {

constexpr int CFGC_THREADS = 256;

// Pass 1 of the delta.  d_new = f32(c) - f32(u) from the pair v = [u; c] (bf16 [2, nvec * 4], cfg_euler's layout); this
// CTA's fp32 partial sums of |d_new - d_ref| and |d_ref| -> partials[blockIdx.x] and partials[gridDim.x + blockIdx.x].  The
// grid is a function of the size only and every thread walks the same grid-stride vectors in the same order, so the
// partials do not depend on the device, the stream or timing.  Pass 2 is step_cache_finish_kernel.
__global__ void __launch_bounds__(SC_THREADS) cfg_cache_delta_kernel(const uint2* __restrict__ v, const float4* __restrict__ d_ref,
                                                                     float4* __restrict__ d_new, float* __restrict__ partials,
                                                                     int64_t nvec) {
    float s_diff = 0.f, s_ref = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * SC_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x; i < nvec; i += stride) {
        float fu[4], fc[4], fr[4], fd[4];
        unipc_unpack4(v[i], fu);
        unipc_unpack4(v[nvec + i], fc);
        unipc_load(d_ref, i, fr);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            fd[j] = __fsub_rn(fc[j], fu[j]);
            s_diff = __fadd_rn(s_diff, fabsf(__fsub_rn(fd[j], fr[j])));
            s_ref = __fadd_rn(s_ref, fabsf(fr[j]));
        }
        d_new[i] = make_float4(fd[0], fd[1], fd[2], fd[3]);
    }
    sc_write_partials(s_diff, s_ref, partials);
}

// The conditional-only Euler step, per element in this order, each product and sum rounded on its own (no FMA):
// u = c - delta; g = u + scale*(c - u); x = x + dsigma*g.  c is the conditional output alone (bf16 [nvec * 4]).
// kScaled (CFG-Zero*, scail_b200/guidance.py): u = (*u_scale) * u, one rounded product, right after u is formed; with
// *u_scale == 1 the step is the unscaled one bit for bit.  u_scale is not read otherwise.
template <bool kScaled = false>
__global__ void __launch_bounds__(CFGC_THREADS) cfg_euler_cached_kernel(float4* __restrict__ x, const uint2* __restrict__ c,
                                                                        const float4* __restrict__ delta, int64_t nvec,
                                                                        float scale, float dsigma,
                                                                        const float* __restrict__ u_scale) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * CFGC_THREADS + threadIdx.x;
    if (i >= nvec) return;
    float fx[4], fc[4], fd[4];
    unipc_load(x, i, fx);
    unipc_unpack4(c[i], fc);
    unipc_load(delta, i, fd);
    const float su = kScaled ? *u_scale : 1.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float u = __fsub_rn(fc[j], fd[j]);
        if constexpr (kScaled) u = __fmul_rn(su, u);
        const float g = __fadd_rn(u, __fmul_rn(scale, __fsub_rn(fc[j], u)));
        fx[j] = __fadd_rn(fx[j], __fmul_rn(dsigma, g));
    }
    x[i] = make_float4(fx[0], fx[1], fx[2], fx[3]);
}

// ---- Taylor forecast (CFGCache(order >= 1)): n_slots fp32 delta slots of nvec * 4 floats, slot s at slots + s * slot_stride,
// and the host's coefficients by value (delta_forecast4 in solver.cuh: slots with a zero coefficient are not read).

// cfg_cache_delta_kernel against a forecast: slot write_slot = f32(c) - f32(u), and the partial sums of |d_new - t| and |t|
// with t = delta_forecast4(k) in place of d_ref, in the same partition and order (so with c = (1, 0, 0) on the slot that
// d_ref was, the partials are cfg_cache_delta_kernel's bit for bit).  Every thread reads all slots of its vector before it
// writes, so the write slot may be one the forecast reads.
__global__ void __launch_bounds__(SC_THREADS) cfg_cache_delta_forecast_kernel(const uint2* __restrict__ v,
                                                                              float* __restrict__ slots, int64_t slot_stride,
                                                                              int write_slot, DeltaForecast k,
                                                                              float* __restrict__ partials, int64_t nvec) {
    float s_diff = 0.f, s_ref = 0.f;
    float4* d_new = reinterpret_cast<float4*>(slots + write_slot * slot_stride);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * SC_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x; i < nvec; i += stride) {
        float fu[4], fc[4], fr[4], fd[4];
        unipc_unpack4(v[i], fu);
        unipc_unpack4(v[nvec + i], fc);
        delta_forecast4(slots, slot_stride, k, i, fr);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            fd[j] = __fsub_rn(fc[j], fu[j]);
            s_diff = __fadd_rn(s_diff, fabsf(__fsub_rn(fd[j], fr[j])));
            s_ref = __fadd_rn(s_ref, fabsf(fr[j]));
        }
        d_new[i] = make_float4(fd[0], fd[1], fd[2], fd[3]);
    }
    sc_write_partials(s_diff, s_ref, partials);
}

// cfg_euler_cached_kernel with delta = delta_forecast4(k): with c = (1, 0, 0) it is cfg_euler_cached_kernel bit for bit.
template <bool kScaled = false>
__global__ void __launch_bounds__(CFGC_THREADS) cfg_euler_cached_forecast_kernel(float4* __restrict__ x,
                                                                                 const uint2* __restrict__ c,
                                                                                 const float* __restrict__ slots,
                                                                                 int64_t slot_stride, DeltaForecast k,
                                                                                 int64_t nvec, float scale, float dsigma,
                                                                                 const float* __restrict__ u_scale) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * CFGC_THREADS + threadIdx.x;
    if (i >= nvec) return;
    float fx[4], fc[4], fd[4];
    unipc_load(x, i, fx);
    unipc_unpack4(c[i], fc);
    delta_forecast4(slots, slot_stride, k, i, fd);
    const float su = kScaled ? *u_scale : 1.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float u = __fsub_rn(fc[j], fd[j]);
        if constexpr (kScaled) u = __fmul_rn(su, u);
        const float g = __fadd_rn(u, __fmul_rn(scale, __fsub_rn(fc[j], u)));
        fx[j] = __fadd_rn(fx[j], __fmul_rn(dsigma, g));
    }
    x[i] = make_float4(fx[0], fx[1], fx[2], fx[3]);
}

}  // namespace scail
