// Persistent ping-pong wgmma GEMM (sm_90a) for the plain bias / activation GEMMs:
//   * three warpgroups, one CTA per SM: warpgroup 0 is the TMA producer (one thread, registers handed back with setmaxnreg.dec),
//     warpgroups 1 and 2 are consumers (setmaxnreg.inc) that each own a WHOLE 128 x BLOCK_N output tile -- two m64nBLOCK_Nk16
//     per k step, BLOCK_N fp32 accumulators per thread;
//   * the CTA walks the same tile list as gemm_persistent_kernel (tile b, b + grid, ..., N index fastest); consumer w takes every
//     other tile of it, and a pair of ordering barriers lets consumer w start its mainloop only after the other consumer has issued
//     the last MMA of the previous tile.  The tensor pipe sees back-to-back mainloops while each consumer's epilogue runs under
//     the other's MMAs (gemm_persistent_kernel leaves the tensor pipe idle during its epilogue);
//   * the producer fills the ring in tile order and runs ahead across tiles; a stage is released by the warpgroup that read it;
//   * the epilogue works on the accumulator fragments directly (no fp32 deposit of the tile): bias from a per-warpgroup slice, the
//     activation, the 16-bit / fp32 conversion -- the same element operations in the same order as gemm_persistent_kernel's
//     bias_act32 / store16_sw / store_f32_sw, so the outputs are bit-identical -- into a per-warpgroup SWIZZLE_128B staging tile
//     that leaves through TMA stores (rows past M are clipped by the TMA).  fp32 outputs leave in 64-column halves.
//   Requirements (checked by the launcher): no residual, no LayerNorm, no pooled product, not the fp32-parity mode, N a multiple
//   of BLOCK_N, and a TMA output map for every output.
#pragma once
#include "gemm_persistent.cuh"

namespace vb {
namespace ppgemm {

using pgemm::kBlockK;
using pgemm::kBlockM;
using pgemm::kMmaK;

template <int BLOCK_N>
struct PPCfg {
    static_assert(BLOCK_N == 64 || BLOCK_N == 128, "ping-pong tile widths: 64 / 128");
    static constexpr int kStageBytesA = kBlockM * kBlockK * 2;
    static constexpr int kStageBytesB = BLOCK_N * kBlockK * 2;
    static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
    static constexpr int kThreads = 384;                 // producer warpgroup + two consumer warpgroups
    static constexpr int kMinBlocks = 1;
    static constexpr int kProducerRegs = 40;
    static constexpr int kConsumerRegs = 232;            // 128 x 40 + 256 x 232 <= 64 K registers
    // per-consumer staging tile: 128 rows x 256 bytes = two 16 KB slabs of 128 rows x 128 bytes (the TMA store box), i.e. a
    // 128 x 128 16-bit tile or a 64-column half of an fp32 one
    static constexpr int kSlabBytes = kBlockM * 128;
    static constexpr int kStagingBytes = 2 * kSlabBytes;
    static constexpr int kBiasBytes = 2 * BLOCK_N * 4;
    static constexpr int kFit = (232448 - 2 * kStagingBytes - kBiasBytes - 16 * 8) / kStageBytes;
    static constexpr int kStages = kFit > 8 ? 8 : kFit;
    static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kStagingBytes + kBiasBytes + 2 * kStages * 8;
    static_assert(kStages >= 4 && kSmemBytes <= 232448, "shared memory budget (227 KB per block)");
};

// named barriers (0 is __syncthreads): 1 + w = consumer w alone, 3 + w = "consumer w may start its next mainloop"
__device__ __forceinline__ void wg_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void order_wait(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void order_signal(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v)); }
__device__ __forceinline__ void st_shared_f32x2(uint32_t a, float x, float y) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y));
}

template <int ACT>
__device__ __forceinline__ float act1(float x) {            // bias_act32's per-element activation
    if (ACT == kActGelu) return gelu_erf(x);
    if (ACT == kActRelu) return fmaxf(x, 0.0f);
    return x;
}

// acc = act(acc + bias) for one m64 half; fragment d[4j + {0,1}] -> columns 8j + cq + {0,1}, d[4j + {2,3}] the same 8 rows lower
template <int BLOCK_N, int ACT>
__device__ __forceinline__ void bias_act_frag(float (&d)[BLOCK_N / 2], const float* bias_s, int cq) {
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
        const float2 b = *reinterpret_cast<const float2*>(bias_s + 8 * j + cq);
        d[4 * j + 0] = act1<ACT>(d[4 * j + 0] + b.x);
        d[4 * j + 1] = act1<ACT>(d[4 * j + 1] + b.y);
        d[4 * j + 2] = act1<ACT>(d[4 * j + 2] + b.x);
        d[4 * j + 3] = act1<ACT>(d[4 * j + 3] + b.y);
    }
}
// 16-bit: slab j / 8 holds columns [64 (j / 8), +64); 16-byte unit u of row r sits at u ^ (r & 7) (SWIZZLE_128B)
template <int BLOCK_N, bool F16>
__device__ __forceinline__ void stage16(uint32_t stg, const float (&d)[BLOCK_N / 2], int r, int cq) {
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
        const uint32_t a = stg + (j >> 3) * PPCfg<BLOCK_N>::kSlabBytes + r * 128 + ((((j & 7) ^ (r & 7))) << 4) + cq * 2;
        st_shared_u32(a, F16 ? pack16x2_rt(d[4 * j], d[4 * j + 1], 1) : pack_bf16x2(d[4 * j], d[4 * j + 1]));
        st_shared_u32(a + 8 * 128, F16 ? pack16x2_rt(d[4 * j + 2], d[4 * j + 3], 1) : pack_bf16x2(d[4 * j + 2], d[4 * j + 3]));
    }
}
// fp32, 64-column half H: slab (j % 8) / 4 holds 32 columns; column 8j + cq is unit 2 (j % 4) + cq / 4, byte 4 (cq % 4)
template <int BLOCK_N, int H>
__device__ __forceinline__ void stage32(uint32_t stg, const float (&d)[BLOCK_N / 2], int r, int cq) {
#pragma unroll
    for (int j = 8 * H; j < 8 * H + 8; ++j) {
        const int u = 2 * (j & 3) + (cq >> 2);
        const uint32_t a = stg + ((j & 7) >> 2) * PPCfg<BLOCK_N>::kSlabBytes + r * 128 + ((u ^ (r & 7)) << 4) + (cq & 3) * 4;
        st_shared_f32x2(a, d[4 * j], d[4 * j + 1]);
        st_shared_f32x2(a + 8 * 128, d[4 * j + 2], d[4 * j + 3]);
    }
}

// MODE 0: every M tile.  MODE 6: the tile list ends at the device row count *p.m_rows (packed batches), as in gemm_persistent_kernel.
template <int BLOCK_N, int ACT, bool F16, int MODE>
__global__ void __launch_bounds__(PPCfg<BLOCK_N>::kThreads, PPCfg<BLOCK_N>::kMinBlocks)
gemm_pingpong_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                     const __grid_constant__ CUtensorMap tmap_c16, const __grid_constant__ CUtensorMap tmap_c32,
                     const GemmEpilogue p, const int num_m_tiles, const int num_n_tiles) {
    using Cfg = PPCfg<BLOCK_N>;
    constexpr int kStages = Cfg::kStages;
    static_assert(MODE == 0 || MODE == 6, "plain and device-row-count variants only");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();    // SWIZZLE_128B atoms; no printf in a kernel that issues wgmma (C7510)
    uint8_t* ring = smem_raw;
    uint8_t* staging = ring + kStages * Cfg::kStageBytes;                          // [2][kStagingBytes]
    float* s_bias = reinterpret_cast<float*>(staging + 2 * Cfg::kStagingBytes);    // [2][BLOCK_N]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_bias + 2 * BLOCK_N);
    uint64_t* empty_bar = full_bar + kStages;

    const int wg = threadIdx.x >> 7;
    const int num_kb = (p.K + kBlockK - 1) / kBlockK;
    // profiling stamps (vb200_timeline): 0 clock64 at entry, 8 / 9 globaltimer at entry / exit, 10 last tile accumulated,
    // 11 tiles walked, 12 SM id, 13 clock64 at exit
    long long* stamps = p.timing ? p.timing + 16 * static_cast<size_t>(blockIdx.x) : nullptr;
    if (stamps && threadIdx.x == 0) {
        stamps[0] = clock64();
        unsigned long long gt;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        stamps[8] = static_cast<long long>(gt);
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        stamps[12] = smid;
    }

    int run_m_tiles = num_m_tiles;
    if constexpr (MODE == 6) {                           // written before the graph starts: read ahead of griddepcontrol.wait
        const int mr = max(0, min(*p.m_rows, p.M));
        run_m_tiles = min(num_m_tiles, (mr + kBlockM - 1) / kBlockM);
    }
    const int total_tiles = run_m_tiles * num_n_tiles;
    const int first_tile = static_cast<int>(blockIdx.x);
    const int tile_stride = static_cast<int>(gridDim.x);
    const int n_local = first_tile < total_tiles ? (total_tiles - first_tile + tile_stride - 1) / tile_stride : 0;
    if (stamps && threadIdx.x == 0) stamps[11] = n_local;

    // ---------------------------------------------------------------- setup (as gemm_persistent_kernel)
    int early = 0;
    bool early_a = false;
    const bool producer_thread = threadIdx.x == 0;
    if (producer_thread) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        if (p.out_bf16 != nullptr) tma_prefetch_desc(&tmap_c16);
        if (p.out_f32 != nullptr) tma_prefetch_desc(&tmap_c32);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 4);                 // one arrival per warp of the consumer warpgroup that read the stage
        }
        mbar_fence_init();
        if (n_local > 0 && p.pdl != 1) {
            early_a = p.pdl != 5;
            const int m0 = (first_tile / num_n_tiles) * kBlockM, n0 = (first_tile % num_n_tiles) * BLOCK_N;
            early = min(kStages, num_kb);
            for (int i = 0; i < early; ++i) {
                uint8_t* sa = ring + i * Cfg::kStageBytes;
                mbar_arrive_expect_tx(&full_bar[i], Cfg::kStageBytes);
                if (early_a) tma_load_2d(sa, &tmap_a, &full_bar[i], i * kBlockK, m0);
                tma_load_2d(sa + Cfg::kStageBytesA, &tmap_b, &full_bar[i], i * kBlockK, n0);
            }
        }
    }
    __syncthreads();
    if (p.pdl && !(p.pdl == 5 && producer_thread)) pdl_wait();

    if (wg == 0) {
        // ============================================================ TMA producer
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Cfg::kProducerRegs));
        if (producer_thread) {
            int s = 0;
            uint32_t phase = 0;
            if (p.pdl == 5) pdl_wait();
            for (int tile = first_tile; tile < total_tiles; tile += tile_stride) {
                const int m0 = (tile / num_n_tiles) * kBlockM, n0 = (tile % num_n_tiles) * BLOCK_N;
                for (int kb = 0; kb < num_kb; ++kb) {
                    uint8_t* sa = ring + s * Cfg::kStageBytes;
                    if (early > 0) {
                        --early;
                        if (!early_a) tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kBlockK, m0);
                    } else {
                        mbar_wait_nocall(&empty_bar[s], phase ^ 1u);
                        mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
                        tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kBlockK, m0);
                        tma_load_2d(sa + Cfg::kStageBytesA, &tmap_b, &full_bar[s], kb * kBlockK, n0);
                    }
                    if (++s == kStages) { s = 0; phase ^= 1u; }
                }
            }
        }
    } else {
        // ============================================================ consumers: whole tiles, alternating
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Cfg::kConsumerRegs));
        constexpr uint64_t kDescStage = static_cast<uint64_t>(Cfg::kStageBytes >> 4);
        constexpr uint64_t kDescHalf = static_cast<uint64_t>((64 * 128) >> 4);        // rows 64..127 of the A box
        const int cw = wg - 1;
        const int ct = threadIdx.x & 127;
        const int lane = ct & 31;
        const uint64_t da0 = gmma_desc_kmajor_sw128(smem_u32(ring));
        const uint64_t db0 = gmma_desc_kmajor_sw128(smem_u32(ring + Cfg::kStageBytesA));
        float* my_bias = s_bias + cw * BLOCK_N;
        const uint32_t stg = smem_u32(staging + cw * Cfg::kStagingBytes);
        uint8_t* stg_ptr = staging + cw * Cfg::kStagingBytes;
        const int r0 = 16 * (ct >> 5) + (lane >> 2);     // fragment row (plus 8, plus 64 for the second m64 half)
        const int cq = 2 * (lane & 3);                   // fragment column offset within each 8-column group
        int ks = 0;
        uint32_t kphase = 0;
        auto skip_tile = [&]() __attribute__((always_inline)) {     // the other consumer's tile: its k-blocks are not ours
            ks += num_kb;
            while (ks >= kStages) { ks -= kStages; kphase ^= 1u; }
        };
        if (cw == 1) skip_tile();
        for (int li = cw; li < n_local; li += 2) {
            const int tile = first_tile + li * tile_stride;
            const int m0 = (tile / num_n_tiles) * kBlockM, n0 = (tile % num_n_tiles) * BLOCK_N;
            // staging tile and bias slice are free once the previous tile's TMA stores have read the staging tile (thread 0
            // issued them) and every thread is past the barrier below
            if (ct == 0) tma_store_wait_read();
            if (ct < BLOCK_N) my_bias[ct] = p.bias ? p.bias[n0 + ct] : 0.0f;
            wg_bar_sync(1 + cw);
            if (li > 0) order_wait(3 + cw);

            float d0[BLOCK_N / 2], d1[BLOCK_N / 2];
            int prev = -1;
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait_nocall(&full_bar[ks], kphase);
                const uint64_t da = da0 + kDescStage * static_cast<uint64_t>(ks);
                const uint64_t db = db0 + kDescStage * static_cast<uint64_t>(ks);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < kBlockK / kMmaK; ++k) {
                    const uint32_t scale = (kb == 0 && k == 0) ? 0u : 1u;
                    Wgmma<BLOCK_N, F16>::mma(d0, da + 2u * k, db + 2u * k, scale);
                    Wgmma<BLOCK_N, F16>::mma(d1, da + kDescHalf + 2u * k, db + 2u * k, scale);
                }
                wgmma_commit();
                if (prev >= 0) {
                    wgmma_wait<1>();                                     // k-block kb - 1 has read its stage
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = ks;
                if (++ks == kStages) { ks = 0; kphase ^= 1u; }
            }
            if (li + 1 < n_local) order_signal(3 + (1 - cw));           // every MMA of this tile is issued: the other consumer goes
            wgmma_wait<0>();
            if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
            if (li == n_local - 1) {                                     // this CTA's last tile is accumulated
                if (p.pdl && ct == 0) pdl_launch_dependents();
                if (stamps && ct == 0) stamps[10] = clock64();
            }

            // ---- epilogue from the fragments
            bias_act_frag<BLOCK_N, ACT>(d0, my_bias, cq);
            bias_act_frag<BLOCK_N, ACT>(d1, my_bias, cq);
            bool staged = false;                         // the staging tile holds a pass whose TMA store may still read it
            auto flush = [&](const CUtensorMap* map, int ncols_slab, int c0) __attribute__((always_inline)) {
                fence_proxy_async_smem();                // my st.shared -> visible to the TMA
                wg_bar_sync(1 + cw);                     // ... and everybody's
                if (ct == 0) {
                    tma_store_2d(map, stg_ptr, c0, m0);
                    tma_store_2d(map, stg_ptr + Cfg::kSlabBytes, c0 + ncols_slab, m0);
                    tma_store_commit();
                }
                staged = true;
            };
            auto reuse = [&]() __attribute__((always_inline)) {
                if (staged) {
                    if (ct == 0) tma_store_wait_read();
                    wg_bar_sync(1 + cw);
                }
            };
            if (p.out_bf16 != nullptr) {
                stage16<BLOCK_N, F16>(stg, d0, r0, cq);
                stage16<BLOCK_N, F16>(stg, d1, r0 + 64, cq);
                if (BLOCK_N == 128) {
                    flush(&tmap_c16, 64, n0);
                } else {                                 // one 16 KB slab
                    fence_proxy_async_smem();
                    wg_bar_sync(1 + cw);
                    if (ct == 0) { tma_store_2d(&tmap_c16, stg_ptr, n0, m0); tma_store_commit(); }
                    staged = true;
                }
            }
            if (p.out_f32 != nullptr) {
                reuse();
                stage32<BLOCK_N, 0>(stg, d0, r0, cq);
                stage32<BLOCK_N, 0>(stg, d1, r0 + 64, cq);
                flush(&tmap_c32, 32, n0);
                if constexpr (BLOCK_N == 128) {
                    reuse();
                    stage32<BLOCK_N, 1>(stg, d0, r0, cq);
                    stage32<BLOCK_N, 1>(stg, d1, r0 + 64, cq);
                    flush(&tmap_c32, 32, n0 + 64);
                }
            }
            if (li + 1 < n_local) skip_tile();
        }
        if (ct == 0) tma_store_wait_read();              // shared memory stays valid until the TMA has read it
    }

    __syncthreads();
    if (stamps && threadIdx.x == 0) {
        unsigned long long gt;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        stamps[9] = static_cast<long long>(gt);
        stamps[13] = clock64();
    }
}

}  // namespace ppgemm
}  // namespace vb
