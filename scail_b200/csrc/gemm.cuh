// Persistent warp-specialised bf16 GEMM for sm_90a:  C[M,N] = epi(A[M,K] * W[N,K]^T)
//   * one producer warp streams A/W tiles with TMA (SWIZZLE_128B) into a 3-deep shared-memory ring,
//   * a second producer warp loads what the epilogue shares per tile: the tile's 256 bias values and gate rows into
//     shared memory and, for the residual epilogues, the 128 x 256 residual tile by TMA into the output staging buffer,
//     while the consumers are still in the main loop,
//   * two consumer warpgroups each own 64 rows of the 128 x 256 tile: wgmma m64n256k16 with fp32 accumulators in registers,
//     one wgmma group kept in flight so that a ring stage is released as soon as the MMAs that read it have retired,
//   * the epilogue (chosen at compile time: bias / activation / gate / residual in fp32, one bf16 rounding) writes the
//     tile into the swizzled staging buffer and one thread per warpgroup stores it with TMA; the store drains while the
//     next tile's main loop runs.  TMA clips the store to [M, N], so ragged edges and C as a column slab of a wider
//     buffer never write outside the output.
// Replaces the reference's F.linear calls (sat/mpu/layers.py:230-243, :425-444) together with
// the elementwise ops that follow them (bias, GELU-tanh, gate*out + residual).
//
// gemm_fp8_kernel is the same kernel on e4m3 operands with one fp32 scale per row of A and per row of W:
//   C = epi((sum_k A_q W_q) * s_a[m] * s_w[n]).  A 128-element fp8 k-block is a 128-byte row, so the TMA boxes, the swizzle and
//   the descriptor steps are the bf16 kernel's.  Hopper's fp8 wgmma keeps only about 14 bits of its fp32 accumulator, so each
//   k-block's MMAs go into a fresh accumulator that is then added into an fp32 register accumulator (promotion).  ptxas
//   allocates every warp against the 168 registers of the 384-thread launch bound (setmaxnreg only moves the budget at run
//   time), so the two accumulators fit at 64 x 128 per warpgroup (64 x 192 spills): the fp8 tile is 128 x 128.  The loader warp also brings the tile's
//   s_w columns and s_a rows; the scales multiply the accumulator first, then the epilogue runs exactly as for bf16.
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

// C and the residual are addressed through tensor maps; these are the operands the epilogue reads directly.
struct GemmParams {
    int M, N, K;
    const __nv_bfloat16* bias;  // [N] or null
    const __nv_bfloat16* gate;  // [B, gate_stride] (row b = m / rows_per_batch) or null
    int64_t gate_stride;
    int rows_per_batch;
    int group_m;  // rasterisation: m-blocks per L2 group
    const float* scale_a;  // fp8 only: [M] scale of each row of A
    const float* scale_w;  // fp8 only: [N] scale of each row of W
};

constexpr int GEMM_THREADS = 384;  // warpgroup 0: producer; warpgroups 1, 2: consumers
// Output staging: BN / 64 column chunks of [128 rows][128 B] (64 bf16 or 32 fp32 columns), TMA SWIZZLE_128B layout.
// Warpgroup w owns rows [64 w, 64 w + 64) of every chunk, so each warpgroup stores 64-row boxes of its own.
constexpr int GEMM_OUT_CHUNK_BYTES = 128 * 128;  // 16 KB

// Every k-block row is 128 bytes (64 bf16 or 128 e4m3 elements).
template <bool FP8>
struct GemmCfg {
    static constexpr int BM = 128;
    static constexpr int BN = FP8 ? 128 : 256;
    static constexpr int BK = FP8 ? 128 : 64;
    // bf16: 3 stages, the 64 KB output staging tile does not fit beside a 4th 48 KB stage in 227 KB.
    // fp8: 5 stages of 32 KB beside a 32 KB staging tile.
    static constexpr int STAGES = FP8 ? 5 : 3;
    static constexpr int A_BYTES = BM * 128;
    static constexpr int B_BYTES = BN * 128;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int OUT_CHUNKS = BN / 64;
    static constexpr int OUT_OFF = STAGES * STAGE_BYTES;
    static constexpr int BIAS_OFF = OUT_OFF + OUT_CHUNKS * GEMM_OUT_CHUNK_BYTES;  // fp32 [BN], zeros without a bias
    static constexpr int GATE_OFF = BIAS_OFF + BN * 4;           // bf16 [2][BN]: the gate rows of the tile's first two batches
    static constexpr int SCALE_OFF = GATE_OFF + 2 * BN * 2;      // fp8: fp32 s_w [BN], then s_a [BM]
    static constexpr int BAR_OFF = SCALE_OFF + (FP8 ? (BN + BM) * 4 : 0);
    static constexpr int SMEM_BYTES = BAR_OFF + 128 /*barriers*/ + 1024 /*align*/;
    static_assert(SMEM_BYTES <= 232448, "gemm: shared memory budget");
    static_assert(OUT_OFF % 1024 == 0 && A_BYTES % 1024 == 0 && STAGE_BYTES % 1024 == 0,
                  "gemm: TMA SWIZZLE_128B destinations must be 1024-B aligned");
};
constexpr int GEMM_BM = GemmCfg<false>::BM;
constexpr int GEMM_BN = GemmCfg<false>::BN;
constexpr int GEMM_BK = GemmCfg<false>::BK;
constexpr int GEMM_SMEM_BYTES = GemmCfg<false>::SMEM_BYTES;

__device__ __forceinline__ void gemm_tile_coords(int tile, int num_m, int num_n, int group_m, int& m_blk, int& n_blk) {
    int per_group = group_m * num_n;
    int g = tile / per_group;
    int first_m = g * group_m;
    int gsize = min(group_m, num_m - first_m);
    int r = tile - g * per_group;
    n_blk = r / gsize;
    m_blk = first_m + (r - n_blk * gsize);
}

template <int EPI>
__device__ __forceinline__ float epi_act(float v) {
    if constexpr (EPI == EPI_BIAS_GELU) return gelu_tanh(v);
    else if constexpr (EPI == EPI_BIAS_SILU) return v / (1.0f + __expf(-v));
    else if constexpr (EPI == EPI_BIAS_GELU_ERF) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    else return v;
}

// F32: fp32 output (no residual epilogues, bf16 only).  The fp32 tile is twice the staging buffer, so it is stored in two
// 128-column passes.  FP8: e4m3 operands with per-row scales (gemm_fp8_kernel).
template <int EPI, bool F32, bool FP8>
__device__ __forceinline__ void gemm_body(const CUtensorMap& tmap_a, const CUtensorMap& tmap_w, const CUtensorMap& tmap_c,
                                          const CUtensorMap& tmap_r, const GemmParams& p) {
    using C = GemmCfg<FP8>;
    constexpr int GEMM_BN = C::BN, GEMM_BK = C::BK, GEMM_STAGES = C::STAGES;
    constexpr int GEMM_A_BYTES = C::A_BYTES, GEMM_STAGE_BYTES = C::STAGE_BYTES;
    constexpr bool RES = EPI == EPI_BIAS_GATE_RES || EPI == EPI_BIAS_RES;
    constexpr bool GATE = EPI == EPI_BIAS_GATE_RES;
    static_assert(!(F32 && RES), "gemm: the residual epilogues write bf16");
    static_assert(!(F32 && FP8), "gemm: the fp8 GEMM writes bf16");
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (smem_base - smem_u32(smem_raw));
    const uint32_t out_base = smem_base + C::OUT_OFF;
    const uint32_t bias_base = smem_base + C::BIAS_OFF;
    const uint32_t scale_base = smem_base + C::SCALE_OFF;  // fp8: s_w [BN] then s_a [BM]
    const uint32_t bar_base = smem_base + C::BAR_OFF;
    // barrier layout (8 B each): full[S], empty[S], epi_full, epi_empty, res_full, out_free
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (GEMM_STAGES + s); };
    const uint32_t epi_full = bar_base + 16u * GEMM_STAGES;  // bias / gate (/ scales) of the tile are in shared memory
    const uint32_t epi_empty = epi_full + 8;                 // both warpgroups are done reading them
    const uint32_t res_full = epi_full + 16;                 // the residual tile has landed in the staging buffer
    const uint32_t out_free = epi_full + 24;                 // both warpgroups' previous stores have read the staging buffer

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_m = (p.M + GEMM_BM - 1) / GEMM_BM;
    const int num_n = (p.N + GEMM_BN - 1) / GEMM_BN;
    const int num_tiles = num_m * num_n;
    const int num_k = (p.K + GEMM_BK - 1) / GEMM_BK;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_w);
        tma_prefetch_desc(&tmap_c);
        if (RES) tma_prefetch_desc(&tmap_r);
        for (int s = 0; s < GEMM_STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);  // one arrive per consumer warpgroup
        }
        mbar_init(epi_full, 32);  // every lane of the epilogue loader warp
        mbar_init(epi_empty, 2);
        mbar_init(res_full, 1);
        mbar_init(out_free, 2);
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
        } else if (warp == 1) {
            // ---- epilogue loader: per-tile bias and gate rows, and the residual tile ----
            float* bias_s = reinterpret_cast<float*>(smem + C::BIAS_OFF);
            __nv_bfloat16* gate_s = reinterpret_cast<__nv_bfloat16*>(smem + C::GATE_OFF);
            int it = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
                int m_blk, n_blk;
                gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
                const int m0 = m_blk * GEMM_BM, n0 = n_blk * GEMM_BN;
                const int c = 8 * lane, col = n0 + c;  // N % 8 == 0: an 8-column group is wholly inside or outside
                mbar_wait(epi_empty, (it & 1) ^ 1, 4);
                if (GEMM_BN == 32 * 8 || c < GEMM_BN) {  // 32 lanes x 8 columns span the bf16 tile; half of them the fp8 one
                    uint4 braw = make_uint4(0, 0, 0, 0);
                    if (p.bias && col < p.N) braw = *reinterpret_cast<const uint4*>(p.bias + col);
                    const float2 b01 = unpack_bf16(braw.x), b23 = unpack_bf16(braw.y);
                    const float2 b45 = unpack_bf16(braw.z), b67 = unpack_bf16(braw.w);
                    *reinterpret_cast<float4*>(bias_s + c) = make_float4(b01.x, b01.y, b23.x, b23.y);
                    *reinterpret_cast<float4*>(bias_s + c + 4) = make_float4(b45.x, b45.y, b67.x, b67.y);
                    if constexpr (GATE) {
                        const int b0 = m0 / p.rows_per_batch;
#pragma unroll
                        for (int s = 0; s < 2; ++s) {
                            uint4 g = make_uint4(0, 0, 0, 0);
                            const int b = b0 + s;
                            if (col < p.N && static_cast<int64_t>(b) * p.rows_per_batch < p.M)
                                g = *reinterpret_cast<const uint4*>(p.gate + b * p.gate_stride + col);
                            *reinterpret_cast<uint4*>(gate_s + s * GEMM_BN + c) = g;
                        }
                    }
                }
                if constexpr (FP8) {  // zeros outside [M, N]: those rows and columns are clipped by the store anyway
                    float* sw_s = reinterpret_cast<float*>(smem + C::SCALE_OFF);
                    float* sa_s = sw_s + GEMM_BN;
                    for (int i = lane; i < GEMM_BN; i += 32) sw_s[i] = n0 + i < p.N ? p.scale_w[n0 + i] : 0.f;
                    for (int i = lane; i < C::BM; i += 32) sa_s[i] = m0 + i < p.M ? p.scale_a[m0 + i] : 0.f;
                }
                mbar_arrive(epi_full);
                if constexpr (RES) {
                    if (lane == 0) {
                        mbar_wait(out_free, it & 1, 5);
                        uint32_t bytes = 0;
                        for (int h = 0; h < 2; ++h)
                            for (int cc = 0; cc < C::OUT_CHUNKS; ++cc)
                                if (m0 + 64 * h < p.M && n0 + 64 * cc < p.N) bytes += GEMM_OUT_CHUNK_BYTES / 2;
                        mbar_expect_tx(res_full, bytes);
                        for (int h = 0; h < 2; ++h)
                            for (int cc = 0; cc < C::OUT_CHUNKS; ++cc)
                                if (m0 + 64 * h < p.M && n0 + 64 * cc < p.N)
                                    tma_load_2d(out_base + cc * GEMM_OUT_CHUNK_BYTES + h * (GEMM_OUT_CHUNK_BYTES / 2), &tmap_r,
                                                res_full, n0 + 64 * cc, m0 + 64 * h);
                    }
                    __syncwarp();
                }
            }
        }
    } else {
        // ===================== consumer warpgroups =====================
        setmaxnreg_inc<232>();
        const int wg = (warp >> 2) - 1;  // 0 or 1: rows [64 wg, 64 wg + 64) of the tile
        const int t = threadIdx.x & 127;
        const bool leader = t == 0;  // releases ring stages, issues and waits for this warpgroup's stores
        // accumulator fragment: rows r0 (acc[4j], acc[4j+1]) and r0 + 8 (acc[4j+2], acc[4j+3]), columns 8 j + 2 q (+1)
        const int r0 = (t >> 5) * 16 + ((t & 31) >> 2);
        const int q = t & 3;
        const uint32_t sw = static_cast<uint32_t>(r0 & 7);  // SWIZZLE_128B: 16-B unit u of row r sits at u ^ (r & 7)
        const uint32_t out_rows = out_base + wg * (GEMM_OUT_CHUNK_BYTES / 2) + r0 * 128;
        // shared address of columns (8 j + 2 q, +1), row r0 (+ 8 rows = + 1024 B)
        auto out_addr = [&](int j) -> uint32_t {
            if constexpr (F32) {
                const int jp = j & 15;  // column 8 j + 2 q of the 128-column pass
                return out_rows + (jp >> 2) * GEMM_OUT_CHUNK_BYTES + (((2u * (jp & 3) + (q >> 1)) ^ sw) << 4) + 8 * (q & 1);
            } else {
                return out_rows + (j >> 3) * GEMM_OUT_CHUNK_BYTES + (((j & 7) ^ sw) << 4) + 4 * q;
            }
        };
        int stage = 0;
        uint32_t phase = 0;
        float acc[GEMM_BN / 2];
        [[maybe_unused]] float part[FP8 ? GEMM_BN / 2 : 1];  // fp8: one k-block's wgmma accumulator
        int it = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
            int m_blk, n_blk;
            gemm_tile_coords(tile, num_m, num_n, p.group_m, m_blk, n_blk);
            const int m0 = m_blk * GEMM_BM, n0 = n_blk * GEMM_BN;
#pragma unroll
            for (int i = 0; i < GEMM_BN / 2; ++i) acc[i] = 0.f;
            int prev_stage = -1;
            const int kb_free = num_k > 1 ? 1 : 0;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(full_bar(stage), phase, 3);
                const uint32_t sa = smem_base + stage * GEMM_STAGE_BYTES;
                const uint64_t da = wgmma_desc_kmajor_sw128(sa + wg * (64 * 128));
                const uint64_t db = wgmma_desc_kmajor_sw128(sa + GEMM_A_BYTES);
                if constexpr (FP8) {
                    fence_regs(part);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < GEMM_BK / 32; ++k) wgmma_ss_e4m3<GEMM_BN>(part, da + 2 * k, db + 2 * k, k > 0);
                    wgmma_commit();
                    wgmma_wait<0>();
                    fence_regs(part);
                    if (leader) mbar_arrive(empty_bar(stage));
#pragma unroll
                    for (int i = 0; i < GEMM_BN / 2; ++i) acc[i] = __fadd_rn(acc[i], part[i]);  // promotion to fp32
                } else {
                    fence_regs(acc);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<GEMM_BN>(acc, da + 2 * k, db + 2 * k, 1);
                    wgmma_commit();
                    wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
                    fence_regs(acc);
                    if (prev_stage >= 0 && leader) mbar_arrive(empty_bar(prev_stage));
                }
                prev_stage = stage;
                if (++stage == GEMM_STAGES) { stage = 0; phase ^= 1; }
                // early in the tile: once the previous tile's store has read the staging buffer, hand it to the
                // loader (residual) or to this warpgroup's epilogue
                if (kb == kb_free && leader) {
                    bulk_wait_read_all();
                    mbar_arrive(out_free);
                }
            }
            if constexpr (!FP8) {
                wgmma_wait<0>();
                fence_regs(acc);
                if (prev_stage >= 0 && leader) mbar_arrive(empty_bar(prev_stage));
            }

            // ---- epilogue: fp32 in registers, one rounding, into the staging buffer ----
            mbar_wait(epi_full, it & 1, 6);
            if constexpr (RES) mbar_wait(res_full, it & 1, 7);
            else named_bar_sync(1 + wg, 128);  // the leader has seen the previous store finish reading the buffer
            const __nv_bfloat16* grow[2];
            int gmax[2];
            if constexpr (GATE) {
                const int b0 = m0 / p.rows_per_batch;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int b = min(m0 + wg * 64 + r0 + 8 * h, p.M - 1) / p.rows_per_batch;
                    if (b - b0 < 2) {
                        grow[h] = reinterpret_cast<const __nv_bfloat16*>(smem + C::GATE_OFF) + (b - b0) * GEMM_BN;
                        gmax[h] = GEMM_BN - 2;
                    } else {  // rows_per_batch < 128: a tile spanning more than two batches reads the gate in place
                        grow[h] = p.gate + b * p.gate_stride + n0;
                        gmax[h] = p.N - 2 - n0;
                    }
                }
            }
            [[maybe_unused]] float srow[2];  // fp8: s_a of rows r0 and r0 + 8
            if constexpr (FP8) {
#pragma unroll
                for (int h = 0; h < 2; ++h) srow[h] = lds_f1(scale_base + 4 * (GEMM_BN + wg * 64 + r0 + 8 * h));
            }
            auto issue_store = [&](int pass) {
                fence_proxy_async_smem();
                named_bar_sync(1 + wg, 128);
                if (leader) {
                    const int rows = m0 + wg * 64;
                    constexpr int chunk_cols = F32 ? 32 : 64;
#pragma unroll
                    for (int c = 0; c < C::OUT_CHUNKS; ++c) {
                        const int col = n0 + pass * 128 + c * chunk_cols;
                        if (rows < p.M && col < p.N)
                            tma_store_2d(&tmap_c, out_base + c * GEMM_OUT_CHUNK_BYTES + wg * (GEMM_OUT_CHUNK_BYTES / 2), col, rows);
                    }
                    bulk_commit();
                }
            };
            // G accumulator column groups (8 G columns) at a time: their shared-memory loads are issued together
            constexpr int G = F32 ? 4 : 8;  // fewer live registers where the fp32 stores need them (no spills)
#pragma unroll
            for (int cc = 0; cc < GEMM_BN / 8 / G; ++cc) {
                if constexpr (F32) {
                    if (cc == 16 / G) {  // first 128 columns are staged: store them, wait until they are read
                        issue_store(0);
                        if (leader) bulk_wait_read_all();
                        named_bar_sync(1 + wg, 128);
                    }
                }
                float2 bb[G];
                [[maybe_unused]] float2 ss[G];
                uint32_t gg[2 * G], rr[2 * G];
#pragma unroll
                for (int jj = 0; jj < G; ++jj) {
                    const int j = G * cc + jj;
                    bb[jj] = lds_f2(bias_base + 4 * (8 * j + 2 * q));
                    if constexpr (FP8) ss[jj] = lds_f2(scale_base + 4 * (8 * j + 2 * q));
                    if constexpr (GATE) {
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            gg[2 * jj + h] = *reinterpret_cast<const uint32_t*>(grow[h] + min(8 * j + 2 * q, gmax[h]));
                    }
                    if constexpr (RES) {
                        rr[2 * jj] = lds_u32(out_addr(j));
                        rr[2 * jj + 1] = lds_u32(out_addr(j) + 1024);
                    }
                }
#pragma unroll
                for (int jj = 0; jj < G; ++jj) {
                    const int j = G * cc + jj;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float a0 = acc[4 * j + 2 * h], a1 = acc[4 * j + 2 * h + 1];
                        if constexpr (FP8) {  // (acc * s_a) * s_w, then the bf16 kernel's epilogue
                            a0 = __fmul_rn(__fmul_rn(a0, srow[h]), ss[jj].x);
                            a1 = __fmul_rn(__fmul_rn(a1, srow[h]), ss[jj].y);
                        }
                        float f0 = __fadd_rn(a0, bb[jj].x);
                        float f1 = __fadd_rn(a1, bb[jj].y);
                        f0 = epi_act<EPI>(f0);
                        f1 = epi_act<EPI>(f1);
                        if constexpr (GATE) {
                            const float2 g2 = unpack_bf16(gg[2 * jj + h]);
                            f0 = __fmul_rn(f0, g2.x);
                            f1 = __fmul_rn(f1, g2.y);
                        }
                        if constexpr (RES) {
                            const float2 r2 = unpack_bf16(rr[2 * jj + h]);
                            f0 = __fadd_rn(f0, r2.x);
                            f1 = __fadd_rn(f1, r2.y);
                        }
                        if constexpr (F32) sts_f2(out_addr(j) + 1024 * h, f0, f1);
                        else sts_u32(out_addr(j) + 1024 * h, pack_bf16(f0, f1));
                    }
                }
            }
            issue_store(F32 ? 1 : 0);
            if (leader) mbar_arrive(epi_empty);  // bias and gate reads are behind the barrier in issue_store
        }
        if (leader) bulk_wait_all();
    }
}

template <int EPI, bool F32>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                 const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r,
                 const GemmParams p) {
    gemm_body<EPI, F32, false>(tmap_a, tmap_w, tmap_c, tmap_r, p);
}

template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_r,
                const GemmParams p) {
    gemm_body<EPI, false, true>(tmap_a, tmap_w, tmap_c, tmap_r, p);
}

}  // namespace scail
