// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epi(A[M,K] * W[N,K]^T)
//   * one producer warp streams A/W tiles with TMA (SWIZZLE_128B) into a 4-deep shared-memory ring,
//   * two consumer warpgroups each own 64 rows of the 128 x 256 tile: wgmma m64n256k16 with fp32 accumulators in registers,
//     one wgmma group kept in flight so that a ring stage is released as soon as the MMAs that read it have retired,
//   * the epilogue (bias / activation / gate / residual, one bf16 rounding) runs on the accumulator registers while the
//     producer already fills the ring with the next tile's operands.
// Replaces the reference's F.linear calls (sat/mpu/layers.py:230-243, :425-444) together with
// the elementwise ops that follow them (bias, GELU-tanh, gate*out + residual).
#pragma once
#include "sm90.cuh"

namespace scail {

enum GemmEpilogue : int {
    EPI_BIAS = 0,           // C = acc + bias
    EPI_BIAS_GELU = 1,      // C = gelu_tanh(acc + bias)            (sat/transformer_defaults.py:173-174)
    EPI_BIAS_GATE_RES = 2,  // C = res + gate[b] * (acc + bias)     (dit_video_crossattn_sc_xc.py:1036,1050)
    EPI_BIAS_RES = 3,       // C = res + (acc + bias)               (dit_video_crossattn_sc_xc.py:1042)
    EPI_BIAS_SILU = 4,      // C = silu(acc + bias)
    EPI_BIAS_GELU_ERF = 5,  // C = gelu(acc + bias), exact erf form (MLPProj, dit_video_crossattn_sc_xc.py:38)
};

struct GemmParams {
    int M, N, K;
    const __nv_bfloat16* bias;      // [N] or null
    const __nv_bfloat16* gate;      // [B, gate_stride] (row b = m / rows_per_batch) or null
    const __nv_bfloat16* residual;  // [M, ldr] or null
    __nv_bfloat16* C;               // [M, ldc]
    float* C32;                     // optional fp32 output instead of bf16
    int64_t ldc, ldr, gate_stride;
    int rows_per_batch;
    int epilogue;
    int group_m;  // rasterisation: m-blocks per L2 group
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BN = 256;
constexpr int GEMM_BK = 64;
constexpr int GEMM_STAGES = 4;
constexpr int GEMM_A_BYTES = GEMM_BM * GEMM_BK * 2;  // 16 KB
constexpr int GEMM_B_BYTES = GEMM_BN * GEMM_BK * 2;  // 32 KB
constexpr int GEMM_STAGE_BYTES = GEMM_A_BYTES + GEMM_B_BYTES;
constexpr int GEMM_SMEM_BYTES = GEMM_STAGES * GEMM_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int GEMM_THREADS = 384;  // warpgroup 0: producer; warpgroups 1, 2: consumers
static_assert(GEMM_SMEM_BYTES <= 232448, "gemm: shared memory budget");

__device__ __forceinline__ void gemm_tile_coords(int tile, int num_m, int num_n, int group_m, int& m_blk, int& n_blk) {
    int per_group = group_m * num_n;
    int g = tile / per_group;
    int first_m = g * group_m;
    int gsize = min(group_m, num_m - first_m);
    int r = tile - g * per_group;
    n_blk = r / gsize;
    m_blk = first_m + (r - n_blk * gsize);
}

__device__ __forceinline__ float epi_act(float v, int epilogue) {
    if (epilogue == EPI_BIAS_GELU) return gelu_tanh(v);
    if (epilogue == EPI_BIAS_SILU) return v / (1.0f + __expf(-v));
    if (epilogue == EPI_BIAS_GELU_ERF) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    return v;
}

// Epilogue of one column pair (col, col + 1) of one row: bias, activation, gate, residual in fp32, one rounding.
__device__ __forceinline__ void gemm_epilogue_pair(const GemmParams& p, int row, int col, float f0, float f1) {
    if (row >= p.M || col >= p.N) return;
    if (p.bias) {
        const float2 b2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
        f0 += b2.x;
        f1 += b2.y;
    }
    if (p.epilogue == EPI_BIAS_GELU || p.epilogue == EPI_BIAS_SILU || p.epilogue == EPI_BIAS_GELU_ERF) {
        f0 = epi_act(f0, p.epilogue);
        f1 = epi_act(f1, p.epilogue);
    }
    if (p.epilogue == EPI_BIAS_GATE_RES) {
        const int bidx = row / p.rows_per_batch;
        const float2 g2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.gate + bidx * p.gate_stride + col));
        f0 *= g2.x;
        f1 *= g2.y;
    }
    if (p.epilogue == EPI_BIAS_GATE_RES || p.epilogue == EPI_BIAS_RES) {
        const float2 r2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.residual + static_cast<int64_t>(row) * p.ldr + col));
        f0 += r2.x;
        f1 += r2.y;
    }
    if (p.C32) *reinterpret_cast<float2*>(p.C32 + static_cast<int64_t>(row) * p.ldc + col) = make_float2(f0, f1);
    else *reinterpret_cast<uint32_t*>(p.C + static_cast<int64_t>(row) * p.ldc + col) = pack_bf16(f0, f1);
}

__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const GemmParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + GEMM_STAGES * GEMM_STAGE_BYTES;
    // barrier layout (8 B each): full[S], empty[S]
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (GEMM_STAGES + s); };

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_m = (p.M + GEMM_BM - 1) / GEMM_BM;
    const int num_n = (p.N + GEMM_BN - 1) / GEMM_BN;
    const int num_tiles = num_m * num_n;
    const int num_k = (p.K + GEMM_BK - 1) / GEMM_BK;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_w);
        for (int s = 0; s < GEMM_STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int m_blk, n_blk;
                gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
                for (int kb = 0; kb < num_k; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1, 1);
                    const uint32_t sa = smem_base + stage * GEMM_STAGE_BYTES;
                    mbar_expect_tx(full_bar(stage), GEMM_STAGE_BYTES);
                    tma_load_2d(sa, &tmap_a, full_bar(stage), kb * GEMM_BK, m_blk * GEMM_BM);
                    tma_load_2d(sa + GEMM_A_BYTES, &tmap_w, full_bar(stage), kb * GEMM_BK, n_blk * GEMM_BN);
                    if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ===================== consumer warpgroups =====================
        setmaxnreg_inc<232>();
        const int wg = (warp >> 2) - 1;  // 0 or 1: rows [64 wg, 64 wg + 64) of the tile
        const int t = threadIdx.x & 127;
        const bool releaser = t == 0;
        int stage = 0;
        uint32_t phase = 0;
        float acc[GEMM_BN / 2];
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int m_blk, n_blk;
            gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
#pragma unroll
            for (int i = 0; i < GEMM_BN / 2; ++i) acc[i] = 0.f;
            int prev_stage = -1;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(full_bar(stage), phase, 3);
                const uint32_t sa = smem_base + stage * GEMM_STAGE_BYTES;
                const uint64_t da = wgmma_desc_kmajor_sw128(sa + wg * (64 * 128));
                const uint64_t db = wgmma_desc_kmajor_sw128(sa + GEMM_A_BYTES);
                fence_regs(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<GEMM_BN>(acc, da + 2 * k, db + 2 * k, 1);
                wgmma_commit();
                wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
                fence_regs(acc);
                if (prev_stage >= 0 && releaser) mbar_arrive(empty_bar(prev_stage));
                prev_stage = stage;
                if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (prev_stage >= 0 && releaser) mbar_arrive(empty_bar(prev_stage));
            // ---- epilogue straight from the accumulator fragments ----
            const int row0 = m_blk * GEMM_BM + wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
            const int colb = n_blk * GEMM_BN + 2 * (t & 3);
#pragma unroll
            for (int j = 0; j < GEMM_BN / 8; ++j) {
                gemm_epilogue_pair(p, row0, colb + 8 * j, acc[4 * j], acc[4 * j + 1]);
                gemm_epilogue_pair(p, row0 + 8, colb + 8 * j, acc[4 * j + 2], acc[4 * j + 3]);
            }
        }
    }
}

}  // namespace scail
