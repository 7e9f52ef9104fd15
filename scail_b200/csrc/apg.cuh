// Adaptive projected guidance, APG (scail_b200/guidance.py): the guidance rule of Sadat, Hilliges and Weber (ICLR 2025) on
// data predictions, with its projection and norm threshold reduced per latent frame on the device.  The latent x is fp32
// [T, F] (one frame = F = 16*h*w contiguous elements, F % 4 == 0); the step goes from sigma with guidance scale w:
//   D_c = x - sigma*c, D_u = x - sigma*u, diff = D_c - D_u;  with momentum beta: avg = diff + beta*avg, diff = avg;
//   per frame t:  f_t = min(1, r / |diff_t|) (1 when r = 0 or |diff_t| = 0),  p_t = f_t <diff_t, D_c,t> / |D_c,t|^2 (0 when
//                 |D_c,t| = 0);
//   D_g = D_c + (w - 1)*(orth + eta*par)  with  par = p_t*D_c, orth = f_t*diff - par.
// Three passes: apg_reduce_kernel (per-(frame, CTA) fp32 partials), apg_finish_kernel (fp64 per frame -> factors [T, 2] =
// {f_t, p_t}), apg_update_kernel (the rule, then the Euler step in place on x or D_g to a buffer for the solver).  Every
// thread moves 4 elements: 16-byte vectors of the fp32 tensors and 8-byte vectors of bf16.  Each product and sum is rounded
// on its own (no FMA), so pass 1 and the update form D_c, D_u and diff with the same bits.
#pragma once
#include <cuda_bf16.h>

#include "adaptive.cuh"    // warp_sum_f64
#include "cfg_zero.cuh"    // CfgZeroForm: where u comes from
#include "rowops.cuh"      // warp_sum
#include "solver.cuh"      // unipc_unpack4, unipc_load, DeltaForecast, delta_forecast4

namespace scail {

constexpr int APG_THREADS = 256;
constexpr int APG_MAX_CTAS_PER_FRAME = 32;  // partials hold 3 * T * APG_MAX_CTAS_PER_FRAME floats

// The CTAs of pass 1 per frame: a function of the frame's vector count only.
__host__ __device__ __forceinline__ int apg_ctas_per_frame(int64_t fvec) {
    const int64_t c = (fvec + APG_THREADS - 1) / APG_THREADS;
    return static_cast<int>(c < APG_MAX_CTAS_PER_FRAME ? c : APG_MAX_CTAS_PER_FRAME);
}

// x, c and (by kForm) u at vector i of the latent (nvec vectors; the pair holds u at vector i and c at nvec + i, the
// cached forms hold c alone at i), then D_c and diff = D_c - D_u.  u is formed exactly as the CFG-Zero* reduction and the
// cached updates of the same form form it.
template <int kForm>
__device__ __forceinline__ void apg_diff4(const float4* __restrict__ x, const uint2* __restrict__ v, const float* delta,
                                          int64_t delta_stride, const DeltaForecast& dk, int64_t i, int64_t nvec, float sigma,
                                          float (&fx)[4], float (&dc)[4], float (&diff)[4]) {
    float fu[4], fc[4];
    unipc_load(x, i, fx);
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
        dc[j] = __fsub_rn(fx[j], __fmul_rn(sigma, fc[j]));
        diff[j] = __fsub_rn(dc[j], __fsub_rn(fx[j], __fmul_rn(sigma, fu[j])));
    }
}

// Pass 1.  Grid (ctas_per_frame, T): CTA (b, t) walks the vectors b*APG_THREADS + threadIdx.x + k*ctas_per_frame*APG_THREADS
// of frame t, so the partition is a function of the shape only and the partials do not depend on the device, the stream or
// timing.  With kMomentum it reads avg once and writes avg = diff + beta*avg once (this pass owns the momentum write; the
// update reads the new avg as diff).  This CTA's fp32 sums of diff*diff, diff*D_c and D_c*D_c (each product and sum rounded
// on its own, then the CTA in a fixed order) -> partials[(s*T + t)*ctas_per_frame + b] for s = 0, 1, 2.
template <int kForm, bool kMomentum>
__global__ void __launch_bounds__(APG_THREADS) apg_reduce_kernel(const float4* __restrict__ x, const uint2* __restrict__ v,
                                                                 const float* __restrict__ delta, int64_t delta_stride,
                                                                 DeltaForecast dk, float4* __restrict__ avg, float sigma,
                                                                 float beta, float* __restrict__ partials, int64_t fvec) {
    const int64_t t = blockIdx.y, nvec = fvec * gridDim.y;
    float s_dd = 0.f, s_dp = 0.f, s_pp = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * APG_THREADS;
    for (int64_t k = static_cast<int64_t>(blockIdx.x) * APG_THREADS + threadIdx.x; k < fvec; k += stride) {
        const int64_t i = t * fvec + k;
        float fx[4], dc[4], diff[4];
        apg_diff4<kForm>(x, v, delta, delta_stride, dk, i, nvec, sigma, fx, dc, diff);
        if constexpr (kMomentum) {
            float a[4];
            unipc_load(avg, i, a);
#pragma unroll
            for (int j = 0; j < 4; ++j) diff[j] = __fadd_rn(diff[j], __fmul_rn(beta, a[j]));
            avg[i] = make_float4(diff[0], diff[1], diff[2], diff[3]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            s_dd = __fadd_rn(s_dd, __fmul_rn(diff[j], diff[j]));
            s_dp = __fadd_rn(s_dp, __fmul_rn(diff[j], dc[j]));
            s_pp = __fadd_rn(s_pp, __fmul_rn(dc[j], dc[j]));
        }
    }
    __shared__ float red[3][APG_THREADS / 32];
    s_dd = warp_sum(s_dd);
    s_dp = warp_sum(s_dp);
    s_pp = warp_sum(s_pp);
    if ((threadIdx.x & 31) == 0) {
        red[0][threadIdx.x >> 5] = s_dd;
        red[1][threadIdx.x >> 5] = s_dp;
        red[2][threadIdx.x >> 5] = s_pp;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < APG_THREADS / 32; ++w) s += red[threadIdx.x][w];
        partials[(threadIdx.x * gridDim.y + t) * gridDim.x + blockIdx.x] = s;
    }
}

// Pass 2.  One warp per frame t: lane b takes partial b of each sum in fp64 (b < n_parts <= 32), a fixed shuffle tree adds
// them, then in fp64: f = r / |diff| when r > 0 and |diff| > r, else 1; p = f * dot / |D_c|^2, 0 when |D_c|^2 = 0 (NaN
// propagates through p, and through diff itself when f = 1).  -> sums[4t..4t+3] = {|diff|^2, dot, |D_c|^2, 0} (fp64) and
// factors[2t] = f, factors[2t + 1] = p, each rounded once to fp32.
__global__ void __launch_bounds__(32) apg_finish_kernel(const float* __restrict__ partials, int n_parts, double norm_threshold,
                                                        double* __restrict__ sums, float* __restrict__ factors) {
    const int t = blockIdx.x, T = gridDim.x, lane = threadIdx.x;
    double s[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
        s[k] = warp_sum_f64(lane < n_parts ? static_cast<double>(partials[(k * T + t) * n_parts + lane]) : 0.0);
    if (lane == 0) {
        const double nd = s[0], dot = s[1], nc = s[2], norm = sqrt(nd);
        const double f = (norm_threshold > 0.0 && norm > norm_threshold) ? norm_threshold / norm : 1.0;
        const double p = nc == 0.0 ? 0.0 : f * dot / nc;
        sums[4 * t] = nd;
        sums[4 * t + 1] = dot;
        sums[4 * t + 2] = nc;
        sums[4 * t + 3] = 0.0;
        factors[2 * t] = static_cast<float>(f);
        factors[2 * t + 1] = static_cast<float>(p);
    }
}

// The update, per element in this order with each product and sum rounded on its own: D_c and diff as pass 1 forms them
// (kMomentum: diff = avg, the average pass 1 wrote; else apg_diff4 again, the same instructions); then with {f, p} of the
// element's frame: par = p*D_c; orth = f*diff - par; D_g = D_c + wm1*(orth + eta*par).  kDataPred: D_g -> m (fp32, the
// solver's data prediction) and x is only read; else the Euler step in place, x = x + k_euler*(x - D_g) with k_euler =
// (sigma' - sigma) / sigma from the host.
template <int kForm, bool kMomentum, bool kDataPred>
__global__ void __launch_bounds__(APG_THREADS) apg_update_kernel(float4* __restrict__ x, const uint2* __restrict__ v,
                                                                 const float* __restrict__ delta, int64_t delta_stride,
                                                                 DeltaForecast dk, const float4* __restrict__ avg,
                                                                 const float2* __restrict__ factors, float4* __restrict__ m,
                                                                 float sigma, float wm1, float eta, float k_euler,
                                                                 int64_t nvec, unsigned fvec) {
    const int64_t i = static_cast<int64_t>(blockIdx.x) * APG_THREADS + threadIdx.x;
    if (i >= nvec) return;
    float fx[4], dc[4], diff[4];
    if constexpr (kMomentum) {
        float fc[4];
        unipc_load(x, i, fx);
        unipc_unpack4(v[kForm == CFGZ_PAIR ? nvec + i : i], fc);
        unipc_load(avg, i, diff);
#pragma unroll
        for (int j = 0; j < 4; ++j) dc[j] = __fsub_rn(fx[j], __fmul_rn(sigma, fc[j]));
    } else {
        apg_diff4<kForm>(x, v, delta, delta_stride, dk, i, nvec, sigma, fx, dc, diff);
    }
    const float2 fp = factors[static_cast<unsigned>(i) / fvec];
    float g[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float par = __fmul_rn(fp.y, dc[j]);
        const float orth = __fsub_rn(__fmul_rn(fp.x, diff[j]), par);
        g[j] = __fadd_rn(dc[j], __fmul_rn(wm1, __fadd_rn(orth, __fmul_rn(eta, par))));
    }
    if constexpr (kDataPred) {
        m[i] = make_float4(g[0], g[1], g[2], g[3]);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) fx[j] = __fadd_rn(fx[j], __fmul_rn(k_euler, __fsub_rn(fx[j], g[j])));
        x[i] = make_float4(fx[0], fx[1], fx[2], fx[3]);
    }
}

}  // namespace scail
