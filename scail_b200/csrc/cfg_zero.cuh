// CFG-Zero* guidance (scail_b200/guidance.py): the optimised scale s* = <c, u> / (|u|^2 + 1e-8) of the unconditional output,
// one scalar over the whole latent, reduced on the device in two passes; the update kernels read it through a device
// pointer (u_scale), so it never goes to the host.  The scaled cached and UniPC updates are the kScaled instantiations in
// cfg_cache.cuh and solver.cuh; the scaled Euler step on the pair is below.  Every thread moves 4 elements.
#pragma once
#include <cuda_bf16.h>

#include "cfg_cache.cuh"   // CFGC_THREADS
#include "solver.cuh"      // unipc_unpack4, unipc_load, DeltaForecast, delta_forecast4
#include "step_cache.cuh"  // SC_THREADS, sc_write_partials, sc_sum_partials

namespace scail {

// Where pass 1 takes u from, matching the update it feeds.
enum CfgZeroForm : int {
    CFGZ_PAIR = 0,      // v = [u; c], the bf16 CFG pair [2, nvec * 4]
    CFGZ_CACHED = 1,    // v = c alone (bf16 [nvec * 4]); u = f32(c) - delta, delta fp32 [nvec * 4]
    CFGZ_FORECAST = 2,  // v = c alone; u = f32(c) - delta_forecast4(delta slots, dk)
};

// Pass 1: this CTA's fp32 partial sums of f32(c)*u and u*u (each product and sum rounded on its own) -> partials[blockIdx.x]
// and partials[gridDim.x + blockIdx.x].  u is formed exactly as the update kernels of the same form form it.  The grid is a
// function of the size only and every thread walks the same grid-stride vectors in the same order (cfg_cache_delta_kernel's
// rule), so the partials do not depend on the device, the stream or timing.
template <int kForm>
__global__ void __launch_bounds__(SC_THREADS) cfg_zero_dot_kernel(const uint2* __restrict__ v, const float* __restrict__ delta,
                                                                  int64_t delta_stride, DeltaForecast dk,
                                                                  float* __restrict__ partials, int64_t nvec) {
    float s_dot = 0.f, s_uu = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * SC_THREADS;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * SC_THREADS + threadIdx.x; i < nvec; i += stride) {
        float fu[4], fc[4];
        if constexpr (kForm == CFGZ_PAIR) {
            unipc_unpack4(v[i], fu);
            unipc_unpack4(v[nvec + i], fc);
        } else {
            float fd[4];
            unipc_unpack4(v[i], fc);
            if constexpr (kForm == CFGZ_FORECAST)
                delta_forecast4(delta, delta_stride, dk, i, fd);
            else
                unipc_load(reinterpret_cast<const float4*>(delta), i, fd);
#pragma unroll
            for (int j = 0; j < 4; ++j) fu[j] = __fsub_rn(fc[j], fd[j]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            s_dot = __fadd_rn(s_dot, __fmul_rn(fc[j], fu[j]));
            s_uu = __fadd_rn(s_uu, __fmul_rn(fu[j], fu[j]));
        }
    }
    sc_write_partials(s_dot, s_uu, partials);
}

// Pass 2: one CTA sums the n_parts partials in fp64 in step_cache_finish_kernel's fixed order -> out = {dot, norm, 0, 0} and
// *u_scale = dot / (norm + 1e-8), computed in fp64 and rounded once to fp32 (0 for an all-zero u; NaN propagates).
__global__ void __launch_bounds__(SC_THREADS) cfg_zero_finish_kernel(const float* __restrict__ partials, int n_parts,
                                                                     double* __restrict__ out, float* __restrict__ u_scale) {
    __shared__ double red[2][SC_THREADS];
    sc_sum_partials(partials, n_parts, red);
    if (threadIdx.x == 0) {
        const double dot = red[0][0], norm = red[1][0];
        out[0] = dot;
        out[1] = norm;
        out[2] = 0.0;
        out[3] = 0.0;
        *u_scale = static_cast<float>(dot / (norm + 1e-8));
    }
}

// The scaled Euler step from the CFG pair v = [u; c] (bf16 [2, nvec * 4]), per element in this order, each product and sum
// rounded on its own (no FMA): u' = s*u; g = u' + scale*(c - u'); x = x + dsigma*g, with s = *u_scale.  (cfg_euler_kernel,
// the unscaled step, is left to the compiler's contraction; this kernel is not its bit-twin at s = 1.)
__global__ void __launch_bounds__(CFGC_THREADS) cfg_euler_scaled_kernel(float4* __restrict__ x, const uint2* __restrict__ v,
                                                                        int64_t nvec, float scale, float dsigma,
                                                                        const float* __restrict__ u_scale) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * CFGC_THREADS + threadIdx.x;
    if (i >= nvec) return;
    float fx[4], fu[4], fc[4];
    unipc_load(x, i, fx);
    unipc_unpack4(v[i], fu);
    unipc_unpack4(v[nvec + i], fc);
    const float su = *u_scale;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float u = __fmul_rn(su, fu[j]);
        const float g = __fadd_rn(u, __fmul_rn(scale, __fsub_rn(fc[j], u)));
        fx[j] = __fadd_rn(fx[j], __fmul_rn(dsigma, g));
    }
    x[i] = make_float4(fx[0], fx[1], fx[2], fx[3]);
}

}  // namespace scail
