// Implicit-GEMM causal 3-D convolution on wgmma for the Wan2.1 VAE decoder (sgm/models/wan_vae.py:17-36,
// CausalConv3d; :186-220 ResidualBlock; :101-160 Resample).
//
// Activations are channels-last bf16 [T, H, W, C].  One M tile = an 8x16 patch of output pixels of one frame.
// For every filter tap (dt, dh, dw) and every 64-channel slice, TMA fetches the SHIFTED 8x16x64 input box
// (4-D tensor map; out-of-bounds coordinates — spatial zero padding and the causal t < 0 frames — are
// zero-filled by the hardware), which lands in shared memory exactly like a 128 x 64 K-major GEMM A tile.
// B = weights repacked to [Cout, taps * Cin] (tap-major, channel-minor).  The rest is the GEMM pipeline of
// gemm.cuh: one TMA producer warp, two consumer warpgroups (wgmma m64 x BN x 16 each, fp32 accumulators in registers).
//
// Chunked (temporally tiled) VAE runs pass a second activation map, the causal history [T_hist, H, W, Cin]: the last
// frames of the previous chunk's input.  A box whose frame ct is < 0 is then fetched from the history at frame
// ct + T_hist instead (and is zero-filled as before when that is still < 0).  Same box shape and byte count, same
// tap / channel-slice order, so a chunk computes exactly what the whole sequence computes for its frames.
#pragma once
#include "sm90.cuh"

namespace scail {

// TMA load of one activation box at frame t: from the history map when t < 0 and there is a history, else from x.
__device__ __forceinline__ void conv_load_act(uint32_t dst, const CUtensorMap* tmap_x, const CUtensorMap* tmap_h, int T_hist,
                                              uint32_t bar, int c, int w, int h, int t) {
    if (t < 0 && T_hist > 0) tma_load_4d(dst, tmap_h, bar, c, w, h, t + T_hist);
    else tma_load_4d(dst, tmap_x, bar, c, w, h, t);
}

enum ConvEpilogue : int {
    CONV_EPI_BIAS = 0,       // out = acc + bias
    CONV_EPI_BIAS_RES = 1,   // out = acc + bias + residual   (ResidualBlock: x + h, wan_vae.py:220)
    CONV_EPI_HEAD_CLAMP = 2  // fp32 NCTHW planes, clamp(-1,1), first 3 channels (wan_vae.py:662-664)
};

struct ConvParams {
    int T, H, W;          // output (= input) extent
    int Cin, Cout;        // Cout = valid output channels (weights are zero-padded up to a multiple of BN)
    int KT, KH, KW;       // filter taps; temporal padding is causal (KT-1 on the left), spatial is "same"
    const __nv_bfloat16* bias;      // [Cout]
    const __nv_bfloat16* residual;  // channels-last [T, H, W, ldr]
    void* out;                      // bf16 channels-last [*, H, W, ldo]  or  fp32 [3, *, H, W] (head)
    int64_t ldo, ldr;               // head: ldo = elements per output channel plane (the host may offset `out` by frames)
    int sstride, pad_h, pad_w;  // input coordinate of tap (dh,dw) for output (h,w): (h*sstride + dh - pad_h, w*sstride + dw - pad_w)
    int tstride, toff;          // input frame of tap dt for output frame t: t*tstride + dt + toff (causal stride 1: toff = -(KT-1))
    const __nv_bfloat16* norm_gamma;  // row-tile kernel, Cout == 96 only: also emit out2 = SiLU(RMS_norm(value) * gamma)
    __nv_bfloat16* out2;              //   (the next conv's input, wan_vae.py:194-198) ; `out` may then be null
    int ocols;            // output column c lands in frame t*fmul + c / ocols, channel c % ocols
    int fmul;             // (time_conv of upsample3d interleaves its two channel halves as two frames)
    int epilogue;
    int T_hist;           // frames of the causal history map: a tap at input frame ct < 0 reads history frame ct + T_hist
                          // (still < 0: zero-filled); 0 = no history, t < 0 is zero padding (CausalConv3d cache_x, wan_vae.py:28-36)
};
// 128 bytes: T_hist fills the tail padding.  A larger struct measurably changes the code nvcc generates for the
// epilogues (more parameter reloads and branches; 9 % slower VAE decode on H100), so keep new fields out of it.
static_assert(sizeof(ConvParams) == 128, "ConvParams: keep the kernel parameter struct at 128 bytes");

constexpr int CONV_BM = 128, CONV_BK = 64, CONV_PH = 8, CONV_PW = 16;
constexpr int CONV_A_BYTES = CONV_BM * CONV_BK * 2;
constexpr int CONV_THREADS = 384;  // warpgroup 0: producer; warpgroups 1, 2: consumers

template <int BN>
struct ConvCfg {
    static constexpr int B_BYTES = BN * CONV_BK * 2;
    static constexpr int STAGE_BYTES = CONV_A_BYTES + B_BYTES;
    static constexpr int STAGES = (BN <= 128) ? 6 : 4;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
    static_assert(SMEM_BYTES <= 232448, "conv: shared memory budget");
};

// Epilogue of one channel pair (col, col + 1) of output pixel (t, h, w); the caller checks the pixel.
__device__ __forceinline__ void conv_store_pair(const ConvParams& p, int t, int h, int w, int col, float f0, float f1) {
    if (p.epilogue == CONV_EPI_HEAD_CLAMP) {  // fp32 planes [Cout, *, H, W], clamp(-1, 1), first 3 channels
        float* o = static_cast<float*>(p.out);
        const int64_t plane = p.ldo;
        const int64_t pix = (static_cast<int64_t>(t) * p.H + h) * p.W + w;
        if (col < 3 && col < p.Cout) o[col * plane + pix] = fminf(fmaxf(f0 + __bfloat162float(p.bias[col]), -1.0f), 1.0f);
        if (col + 1 < 3 && col + 1 < p.Cout)
            o[(col + 1) * plane + pix] = fminf(fmaxf(f1 + __bfloat162float(p.bias[col + 1]), -1.0f), 1.0f);
        return;
    }
    if (col >= p.Cout) return;
    const int fr = t * p.fmul + col / p.ocols;
    const int64_t pix = (static_cast<int64_t>(fr) * p.H + h) * p.W + w;
    if (p.bias) {
        const float2 b2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
        f0 += b2.x;
        f1 += b2.y;
    }
    if (p.epilogue == CONV_EPI_BIAS_RES) {
        const float2 r2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.residual + pix * p.ldr + col % p.ocols));
        f0 += r2.x;
        f1 += r2.y;
    }
    *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(p.out) + pix * p.ldo + col % p.ocols) = pack_bf16(f0, f1);
}

template <int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3d_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
              const __grid_constant__ CUtensorMap tmap_h, const ConvParams p) {
    using Cfg = ConvCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + STAGES * Cfg::STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_h = (p.H + CONV_PH - 1) / CONV_PH, tiles_w = (p.W + CONV_PW - 1) / CONV_PW;
    const int num_m = p.T * tiles_h * tiles_w;
    const int num_n = (p.Cout + BN - 1) / BN;
    const int num_tiles = num_m * num_n;
    const int kc_per_tap = (p.Cin + CONV_BK - 1) / CONV_BK;
    const int taps = p.KT * p.KH * p.KW;
    const int num_k = taps * kc_per_tap;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_x);
        tma_prefetch_desc(&tmap_w);
        if (p.T_hist > 0) tma_prefetch_desc(&tmap_h);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);
        }
        fence_barrier_init();
    }
    __syncthreads();

    auto tile_coords = [&](int tile, int& t, int& h0, int& w0, int& n_blk) {
        n_blk = tile % num_n;
        int m = tile / num_n;
        w0 = (m % tiles_w) * CONV_PW;
        m /= tiles_w;
        h0 = (m % tiles_h) * CONV_PH;
        t = m / tiles_h;
    };

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int t, h0, w0, n_blk;
                tile_coords(tile, t, h0, w0, n_blk);
                for (int tap = 0; tap < taps; ++tap) {
                    const int dw = tap % p.KW, dh = (tap / p.KW) % p.KH, dt = tap / (p.KW * p.KH);
                    const int ct = t * p.tstride + dt + p.toff, ch = h0 * p.sstride + dh - p.pad_h, cw = w0 * p.sstride + dw - p.pad_w;
                    for (int kc = 0; kc < kc_per_tap; ++kc) {
                        mbar_wait(empty_bar(stage), phase ^ 1, 51);
                        const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
                        mbar_expect_tx(full_bar(stage), Cfg::STAGE_BYTES);
                        conv_load_act(sa, &tmap_x, &tmap_h, p.T_hist, full_bar(stage), kc * CONV_BK, cw, ch, ct);
                        tma_load_2d(sa + CONV_A_BYTES, &tmap_w, full_bar(stage), tap * p.Cin + kc * CONV_BK, n_blk * BN);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const int wg = (warp >> 2) - 1;  // pixel rows [64 wg, 64 wg + 64) of the 128-pixel tile
        const int tid = threadIdx.x & 127;
        const bool releaser = tid == 0;
        int stage = 0;
        uint32_t phase = 0;
        float acc[BN / 2];
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int t, h0, w0, n_blk;
            tile_coords(tile, t, h0, w0, n_blk);
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            int prev_stage = -1;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(full_bar(stage), phase, 53);
                const uint32_t sa = smem_base + stage * Cfg::STAGE_BYTES;
                const uint64_t da = wgmma_desc_kmajor_sw128(sa + wg * (64 * 128));
                const uint64_t db = wgmma_desc_kmajor_sw128(sa + CONV_A_BYTES);
                fence_regs(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < CONV_BK / 16; ++k) wgmma_ss<BN>(acc, da + 2 * k, db + 2 * k, 1);
                wgmma_commit();
                wgmma_wait<1>();
                fence_regs(acc);
                if (prev_stage >= 0 && releaser) mbar_arrive(empty_bar(prev_stage));
                prev_stage = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (prev_stage >= 0 && releaser) mbar_arrive(empty_bar(prev_stage));
            const int colb = n_blk * BN + 2 * (tid & 3);
#pragma unroll
            for (int h8 = 0; h8 < 2; ++h8) {
                const int r = wg * 64 + (tid >> 5) * 16 + ((tid & 31) >> 2) + 8 * h8;
                const int h = h0 + r / CONV_PW, w = w0 + r % CONV_PW;
                if (h >= p.H || w >= p.W) continue;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) conv_store_pair(p, t, h, w, colb + 8 * j, acc[4 * j + 2 * h8], acc[4 * j + 2 * h8 + 1]);
            }
        }
    }
}

// ------------------------------------------------------------------ row-tile variant (3x3 spatial taps, W >= 128)
// The generic kernel above re-fetches the input patch from L2 for each of the 27 taps and the weight slice for every
// 128-pixel tile; with 96 output channels that makes it L2-bound.
// Here one CTA iteration produces TWO output rows (h0, h0+1) x 128 pixels x 96 channels (consumer warpgroup i owns row h0+i).
// Per (dt, dh, 64-channel slice) ONE TMA box [2 rows x 130 pixels x 64 ch] is staged (input rows h0+dh-1, h0+dh with a
// one-pixel halo on both sides); the three dw taps of both output rows are row-shifted views of it: the wgmma descriptor
// start address is simply advanced by whole 128-byte rows (the 128B swizzle is a function of the absolute shared memory
// address, exactly as TMA wrote it), and the three weight slices of the stage are shared by both rows.
constexpr int CROW_PW = 128;
constexpr int CROW_A_ROWS = CROW_PW + 2;                                       // 130 pixels per input row
constexpr int CROW_A_BYTES = ((2 * CROW_A_ROWS * 128 + 1023) / 1024) * 1024;   // 33280 -> 33792
template <int BN>
struct ConvRowCfg {  // BN = 96 (residual / resample convs) or 16 (head conv 96 -> 3, L2-bound: the MMAs are almost free)
    static constexpr int B_BYTES = BN * CONV_BK * 2;                               // per dw tap
    static constexpr int STAGE_BYTES = CROW_A_BYTES + ((3 * B_BYTES + 1023) / 1024) * 1024;
    static constexpr int STAGES = BN > 16 ? 3 : 5;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
    static constexpr uint32_t TX_BYTES = 2 * CROW_A_ROWS * 128 + 3 * B_BYTES;      // bytes the TMA engine reports per stage
    static_assert(SMEM_BYTES <= 232448, "conv row kernel: shared memory budget");
};

template <int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1)
conv3d_row_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                  const __grid_constant__ CUtensorMap tmap_h, const ConvParams p) {
    using Cfg = ConvRowCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int CROW_STAGE_BYTES = Cfg::STAGE_BYTES, CROW_B_BYTES = Cfg::B_BYTES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + STAGES * CROW_STAGE_BYTES;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_h = (p.H + 1) / 2, tiles_w = (p.W + CROW_PW - 1) / CROW_PW;
    const int num_m = p.T * tiles_h * tiles_w;
    const int num_n = (p.Cout + BN - 1) / BN;
    const int num_tiles = num_m * num_n;
    const int kc_per_tap = (p.Cin + CONV_BK - 1) / CONV_BK;
    const int num_k = p.KT * 3 * kc_per_tap;  // stages per tile: (dt, dh, kc)

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_x);
        tma_prefetch_desc(&tmap_w);
        if (p.T_hist > 0) tma_prefetch_desc(&tmap_h);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), 2);
        }
        fence_barrier_init();
    }
    __syncthreads();

    auto tile_coords = [&](int tile, int& t, int& h0, int& w0, int& n_blk) {
        n_blk = tile % num_n;
        int m = tile / num_n;
        w0 = (m % tiles_w) * CROW_PW;
        m /= tiles_w;
        h0 = (m % tiles_h) * 2;
        t = m / tiles_h;
    };

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                int t, h0, w0, n_blk;
                tile_coords(tile, t, h0, w0, n_blk);
                for (int dt = 0; dt < p.KT; ++dt)
                    for (int dh = 0; dh < 3; ++dh)
                        for (int kc = 0; kc < kc_per_tap; ++kc) {
                            mbar_wait(empty_bar(stage), phase ^ 1, 61);
                            const uint32_t sa = smem_base + stage * CROW_STAGE_BYTES;
                            mbar_expect_tx(full_bar(stage), Cfg::TX_BYTES);
                            conv_load_act(sa, &tmap_x, &tmap_h, p.T_hist, full_bar(stage), kc * CONV_BK, w0 - 1, h0 + dh - 1,
                                          t + dt + p.toff);
                            const int tap0 = (dt * 3 + dh) * 3;
#pragma unroll
                            for (int dw = 0; dw < 3; ++dw)
                                tma_load_2d(sa + CROW_A_BYTES + dw * CROW_B_BYTES, &tmap_w, full_bar(stage),
                                            (tap0 + dw) * p.Cin + kc * CONV_BK, n_blk * BN);
                            if (++stage == STAGES) { stage = 0; phase ^= 1; }
                        }
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const int i = (warp >> 2) - 1;  // output row h0 + i reads input row slot i of the box
        const int tid = threadIdx.x & 127;
        const bool releaser = tid == 0;
        int stage = 0;
        uint32_t phase = 0;
        float acc[2][BN / 2];  // pixels [0, 64) and [64, 128) of the row
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            int t, h0, w0, n_blk;
            tile_coords(tile, t, h0, w0, n_blk);
#pragma unroll
            for (int half = 0; half < 2; ++half)
#pragma unroll
                for (int k = 0; k < BN / 2; ++k) acc[half][k] = 0.f;
            int prev_stage = -1;
            for (int kb = 0; kb < num_k; ++kb) {
                mbar_wait(full_bar(stage), phase, 63);
                const uint32_t sa = smem_base + stage * CROW_STAGE_BYTES;
                fence_regs(acc[0]);
                fence_regs(acc[1]);
                wgmma_fence();
#pragma unroll
                for (int dw = 0; dw < 3; ++dw) {
                    const uint64_t db = wgmma_desc_kmajor_sw128(sa + CROW_A_BYTES + dw * CROW_B_BYTES);
#pragma unroll
                    for (int half = 0; half < 2; ++half) {
                        const uint64_t da = wgmma_desc_kmajor_sw128(sa + (i * CROW_A_ROWS + dw + 64 * half) * 128);
#pragma unroll
                        for (int k = 0; k < CONV_BK / 16; ++k) wgmma_ss<BN>(acc[half], da + 2 * k, db + 2 * k, 1);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                fence_regs(acc[0]);
                fence_regs(acc[1]);
                if (prev_stage >= 0 && releaser) mbar_arrive(empty_bar(prev_stage));
                prev_stage = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            fence_regs(acc[0]);
            fence_regs(acc[1]);
            if (prev_stage >= 0 && releaser) mbar_arrive(empty_bar(prev_stage));
            const int h = h0 + i;
            const int quad = tid & 3;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
#pragma unroll
                for (int h8 = 0; h8 < 2; ++h8) {
                    const int w = w0 + half * 64 + (tid >> 5) * 16 + ((tid & 31) >> 2) + 8 * h8;
                    const bool pix_ok = h < p.H && w < p.W;
                    if constexpr (BN == 96) {
                        if (p.norm_gamma != nullptr) {
                            // Fused RMS_norm + SiLU of the NEXT conv's input: the quad of lanes holds all 96 channels of the pixel.
                            const int64_t pix = (static_cast<int64_t>(t) * p.H + h) * p.W + w;
                            float v[BN / 4];
                            float ss = 0.f;
#pragma unroll
                            for (int j = 0; j < BN / 8; ++j) {
                                const int col = 8 * j + 2 * quad;
                                float f0 = acc[half][4 * j + 2 * h8], f1 = acc[half][4 * j + 2 * h8 + 1];
                                if (p.bias) {
                                    const float2 b2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.bias + col));
                                    f0 += b2.x;
                                    f1 += b2.y;
                                }
                                if (p.epilogue == CONV_EPI_BIAS_RES && pix_ok) {
                                    const float2 r2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.residual + pix * p.ldr + col));
                                    f0 += r2.x;
                                    f1 += r2.y;
                                }
                                v[2 * j] = f0;
                                v[2 * j + 1] = f1;
                                ss += f0 * f0 + f1 * f1;
                                if (p.out && pix_ok)
                                    *reinterpret_cast<uint32_t*>(static_cast<__nv_bfloat16*>(p.out) + pix * p.ldo + col) = pack_bf16(f0, f1);
                            }
                            ss += __shfl_xor_sync(0xffffffffu, ss, 1);
                            ss += __shfl_xor_sync(0xffffffffu, ss, 2);
                            if (!pix_ok) continue;
                            const float inv = 9.797958971132712f / fmaxf(sqrtf(ss), 1e-12f);  // sqrt(96) / max(||x||, eps)
#pragma unroll
                            for (int j = 0; j < BN / 8; ++j) {
                                const int col = 8 * j + 2 * quad;
                                const float2 g2 = unpack_bf16(*reinterpret_cast<const uint32_t*>(p.norm_gamma + col));
                                float a = v[2 * j] * inv * g2.x, b = v[2 * j + 1] * inv * g2.y;
                                a = a / (1.0f + __expf(-a));
                                b = b / (1.0f + __expf(-b));
                                *reinterpret_cast<uint32_t*>(p.out2 + pix * 96 + col) = pack_bf16(a, b);
                            }
                            continue;
                        }
                    }
                    if (!pix_ok) continue;
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
                        conv_store_pair(p, t, h, w, n_blk * BN + 8 * j + 2 * quad, acc[half][4 * j + 2 * h8], acc[half][4 * j + 2 * h8 + 1]);
                }
            }
        }
    }
}

// ------------------------------------------------------------------ VAE elementwise kernels (channels-last)

// RMS_norm over channels (F.normalize(x, dim=C) * sqrt(C) * gamma, wan_vae.py:39-54) followed by SiLU.
// x, out: [npix, C] bf16, C = 8 * LP * VPL.  LP lanes (a power of two) share one pixel, each holding VPL 16-byte
// vectors; the sum of squares is reduced with xor-shuffles inside the LP-lane group — no shared memory, no
// block barrier, fully coalesced 16-byte accesses (a warp covers 32/LP consecutive pixels).
template <bool SILU, int LP, int VPL>
__global__ void __launch_bounds__(256) rmsnorm_cl_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                                                         __nv_bfloat16* __restrict__ out, int64_t npix, int C) {
    constexpr int G = LP * VPL;  // vectors per pixel
    const int lane = threadIdx.x & 31;
    const int sub = lane % LP;   // lane within the pixel group
    const int64_t warp = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int64_t pix = warp * (32 / LP) + lane / LP;
    const bool ok = pix < npix;
    const uint4* xin = reinterpret_cast<const uint4*>(x) + pix * G;
    uint4 v[VPL];
    float ss = 0.f;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        v[k] = ok ? xin[k * LP + sub] : make_uint4(0, 0, 0, 0);
        const uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 f = unpack_bf16(w[j]);
            ss += f.x * f.x + f.y * f.y;
        }
    }
#pragma unroll
    for (int o = LP / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if (!ok) return;
    const float inv = sqrtf(static_cast<float>(C)) / fmaxf(sqrtf(ss), 1e-12f);
    uint4* o4 = reinterpret_cast<uint4*>(out) + pix * G;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
        const int vi = k * LP + sub;
        uint4 g = *reinterpret_cast<const uint4*>(gamma + vi * 8);
        const uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w}, gw[4] = {g.x, g.y, g.z, g.w};
        uint32_t r[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 f = unpack_bf16(w[j]), g2 = unpack_bf16(gw[j]);
            float a = f.x * inv * g2.x, b = f.y * inv * g2.y;
            if (SILU) {
                a = a / (1.0f + __expf(-a));
                b = b / (1.0f + __expf(-b));
            }
            r[j] = pack_bf16(a, b);
        }
        o4[vi] = make_uint4(r[0], r[1], r[2], r[3]);
    }
}

// nearest-exact 2x spatial upsample (wan_vae.py:57-63, 77-83), channels-last: [F, H, W, C] -> [F, 2H, 2W, C]
__global__ void upsample2x_cl_kernel(const uint4* x, uint4* out, int64_t frames, int H, int W, int G) {
    const int64_t total = frames * (2 * H) * (2 * W) * G;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int g = i % G;
    int64_t pix = i / G;
    const int xo = pix % (2 * W);
    pix /= (2 * W);
    const int yo = pix % (2 * H);
    const int64_t f = pix / (2 * H);
    out[i] = x[((f * H + (yo >> 1)) * W + (xo >> 1)) * G + g];
}

// z [16, T, h, w] (any float) * std + mean per channel -> channels-last bf16 [T, h, w, 16]
// (WanVAE_.decode un-scaling, wan_vae.py:547-551, with scale = [mean, 1/std] from :630-640)
__global__ void vae_latent_to_cl_kernel(const __nv_bfloat16* z, const float* mean, const float* inv_std,
                                        __nv_bfloat16* out, int T, int h, int w) {
    const int64_t total = static_cast<int64_t>(T) * h * w * 16;
    const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = i % 16;
    const int64_t pix = i / 16;  // (t, y, x)
    const float v = __bfloat162float(z[static_cast<int64_t>(c) * T * h * w + pix]);
    out[i] = __float2bfloat16(v / inv_std[c] + mean[c]);
}

// row softmax of fp32 scores -> bf16 probabilities (mid-block attention, wan_vae.py:252-256); one warp per row
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* s, __nv_bfloat16* p, int rows, int cols,
                                                           float scale) {
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* in = s + static_cast<int64_t>(row) * cols;
    float mx = -INFINITY;
    for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, in[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int c = lane; c < cols; c += 32) sum += __expf((in[c] - mx) * scale);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.0f / sum;
    __nv_bfloat16* out = p + static_cast<int64_t>(row) * cols;
    for (int c = lane; c < cols; c += 32) out[c] = __float2bfloat16(__expf((in[c] - mx) * scale) * inv);
}

}  // namespace scail
