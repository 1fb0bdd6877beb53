// Persistent, warp-specialised wgmma GEMM (sm_90a):
//   * each CTA loops over output tiles, so barrier init, descriptor prefetch and the TMA/L2 latency of the first k-block are paid
//     once per kernel, not once per tile;
//   * one TMA producer warp runs ahead across tile boundaries (the shared-memory ring never drains);
//   * two consumer warpgroups accumulate the 128 x BLOCK_N tile in registers (64 rows each, one k-block of wgmma in flight while
//     the previous stage is handed back), deposit it in a padded fp32 shared-memory tile and then, as eight epilogue warps, read
//     it back one row per thread in 32-column chunks -- meanwhile the producer already fills the ring for the next tile;
//   * epilogue code is specialised OUTSIDE the per-element loops (activation, 16-bit format); outputs are transposed through a
//     swizzled 2 KB per-warp buffer so that a store instruction writes 8 rows x 64 bytes; GELU through a polynomial erf;
//   * launched programmatically (GemmEpilogue::pdl) the producer issues the weight tiles of the first ring pass before
//     griddepcontrol.wait; every kernel triggers its dependents once its last tile is accumulated.
// A residual LayerNorm is not part of this kernel: the GEMM writes fp32 and the row kernel of layernorm.cu normalises.
//
//   D[M,N] = epilogue( A[M,K] (16-bit, row-major)  x  W[N,K]^T (16-bit, nn.Linear layout = K-major) ), fp32 accumulate.
#pragma once
#include <algorithm>
#include <cstdlib>
#include "kernels.h"
#include "wgmma.cuh"

namespace vb {

namespace pgemm {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kMmaK = 16;

// MODE 0: default.  MODE 3: the same kernel with the fp32-parity mode's hi | lo | hi 16-bit output (a compile-time variant so the
// default kernel's register budget is untouched).  MODE 7: MODE 3 summing each k-block's wgmma result in round-to-nearest fp32 on
// the CUDA cores (GemmEpilogue::split_acc, the engine's fp32-parity GEMMs; 64-wide tiles).  MODE 6 ("ROWS"): MODE 0 whose tile list ends at a device row count
// (GemmEpilogue::m_rows, packed batches) -- a variant of its own so that MODE 0 keeps its register allocation.
// MODE 0 and 6 also come 192 wide (96 accumulators per consumer thread, a 2-stage ring): 128 x 192 tiles cover an N = 3072 GEMM in
// 16 column tiles instead of 24.
// One CTA per SM: each consumer thread holds BLOCK_N / 2 fp32 accumulators, and the deposited tile plus a ring deep enough to
// cover the L2 latency take most of the 227 KB of shared memory.
template <int BLOCK_N, int MODE = 0>
struct PCfg {
    static_assert(BLOCK_N == 64 || BLOCK_N == 128 || ((MODE == 0 || MODE == 6) && BLOCK_N == 192),
                  "tile widths: 64 / 128 (MODE 0 and 6 also 192)");
    static constexpr int kStageBytesA = kBlockM * kBlockK * 2;
    static constexpr int kStageBytesB = BLOCK_N * kBlockK * 2;
    static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
    static constexpr int kNumChunks = BLOCK_N / 32;
    // warps 0-7: two consumer warpgroups (wgmma wants whole, aligned warpgroups; each owns 64 rows of the tile and then works as
    // four of the eight epilogue warps), warp 8: TMA producer.  Nine warps leave up to 168 registers per thread.
    static constexpr int kConsumerWarps = 8;
    static constexpr int kProducerWarp = 8;
    static constexpr int kEpiWarps = 8;
    static constexpr int kEpiThreads = 32 * kEpiWarps;
    static constexpr int kThreads = 32 * (kConsumerWarps + 1);
    static constexpr int kMinBlocks = 1;
    // Deposited accumulator tile: [128][BLOCK_N + 4] fp32.  The pad makes both the row-per-thread float4 reads of the epilogue
    // and the fragment-layout float2 writes of the consumer warpgroups (at most) two-way bank conflicted.
    static constexpr int kAccLd = BLOCK_N + 4;
    static constexpr int kAccBytes = kBlockM * kAccLd * 4;
    // Per-epilogue-warp transpose buffer so global stores are row-contiguous: 32 rows x 64 bytes, XOR-swizzled
    // (store16_sw / store_f32_sw).
    static constexpr int kXposeBytesPerWarp = 2048;
    static constexpr int kXposeBytes = kEpiWarps * kXposeBytesPerWarp;
    // ONE bias slice (the tile-end barrier of the epilogue warps protects it)
    static constexpr int kBiasFloats = BLOCK_N;
    static constexpr int kBarBytes = 2 * 8 * 8 + 16;
    static constexpr int kFit = (232448 - kAccBytes - kXposeBytes - kBiasFloats * 4 - kBarBytes) / kStageBytes;
    static constexpr int kStages = kFit > 8 ? 8 : kFit;
    static constexpr int kNumBars = 2 * kStages;
    static constexpr int kSmemAux = kBiasFloats * 4 + kNumBars * 8 + 16 + kXposeBytes;
    // no alignment slack: the dynamic shared-memory window starts 1024-aligned (checked at kernel entry)
    static constexpr int kSmemBytes = kStages * kStageBytes + kAccBytes + kSmemAux;
    static_assert(kStages >= 2 && kSmemBytes <= 232448, "shared memory budget (227 KB per block)");
};

template <int kThreadsInBar>
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kThreadsInBar) : "memory"); }

// ---- one row's 32 consecutive accumulator columns from the deposited tile
__device__ __forceinline__ void acc_ld32(const float* src, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 f = reinterpret_cast<const float4*>(src)[j];
        v[4 * j] = f.x; v[4 * j + 1] = f.y; v[4 * j + 2] = f.z; v[4 * j + 3] = f.w;
    }
}

// ---- consumer warpgroup wg: rows [64 wg, 64 wg + 64) of the 128 x BLOCK_N accumulator, one k-block (four k steps)
template <int BLOCK_N, bool F16>
__device__ __forceinline__ void mma_kblock(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db, bool first) {
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBlockK / kMmaK; ++k) Wgmma<BLOCK_N, F16>::mma(d, da + 2u * k, db + 2u * k, (first && k == 0) ? 0u : 1u);
    wgmma_commit();
}
// Fragment layout of m64nNk16 (thread t of the consumer threads, t / 128 = warpgroup): d[4j + {0,1}] -> row 16 (t / 32) + (t % 32) / 4,
// columns 8j + 2 (t % 4) + {0,1}; d[4j + {2,3}] -> the same columns 8 rows further down.
template <int BLOCK_N>
__device__ __forceinline__ void acc_deposit(float* s_acc, const float (&d)[BLOCK_N / 2], int t) {
    constexpr int ld = BLOCK_N + 4;
    const int r0 = 16 * (t >> 5) + ((t & 31) >> 2), c0 = 2 * (t & 3);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
        float* o = s_acc + r0 * ld + 8 * j + c0;
        *reinterpret_cast<float2*>(o) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2*>(o + 8 * ld) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}

// ---- straight-line per-chunk epilogue pieces (all flags resolved outside the element loops)
template <int ACT>
__device__ __forceinline__ void bias_act32(float (&v)[32], const float* bias_s) {
#pragma unroll
    for (int j4 = 0; j4 < 8; ++j4) {
        const float4 b = reinterpret_cast<const float4*>(bias_s)[j4];     // smem broadcast, 16-byte reads
        float x0 = v[4 * j4 + 0] + b.x, x1 = v[4 * j4 + 1] + b.y, x2 = v[4 * j4 + 2] + b.z, x3 = v[4 * j4 + 3] + b.w;
        if (ACT == kActGelu) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); x2 = gelu_erf(x2); x3 = gelu_erf(x3); }
        if (ACT == kActGeluExact) { x0 = gelu_erf_as(x0); x1 = gelu_erf_as(x1); x2 = gelu_erf_as(x2); x3 = gelu_erf_as(x3); }
        if (ACT == kActRelu) { x0 = fmaxf(x0, 0.0f); x1 = fmaxf(x1, 0.0f); x2 = fmaxf(x2, 0.0f); x3 = fmaxf(x3, 0.0f); }
        v[4 * j4 + 0] = x0; v[4 * j4 + 1] = x1; v[4 * j4 + 2] = x2; v[4 * j4 + 3] = x3;
    }
}
template <bool F16>
__device__ __forceinline__ void store16x32(__nv_bfloat16* op, const float (&v)[32]) {   // 64 contiguous bytes, 16-byte aligned
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint4 u;
        u.x = F16 ? pack16x2_rt(v[8 * j + 0], v[8 * j + 1], 1) : pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
        u.y = F16 ? pack16x2_rt(v[8 * j + 2], v[8 * j + 3], 1) : pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
        u.z = F16 ? pack16x2_rt(v[8 * j + 4], v[8 * j + 5], 1) : pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
        u.w = F16 ? pack16x2_rt(v[8 * j + 6], v[8 * j + 7], 1) : pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
        reinterpret_cast<uint4*>(op)[j] = u;
    }
}
__device__ __forceinline__ void store_f32x32(float* op, const float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) reinterpret_cast<float4*>(op)[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
}
// general (ragged N / unaligned ld) path
__device__ __noinline__ static void store_chunk_slow(const GemmEpilogue& p, int m, int nc, const float* v) {
    if (p.out_bf16 != nullptr) {
        uint16_t* op = reinterpret_cast<uint16_t*>(p.out_bf16) + static_cast<size_t>(m) * p.ld_bf16 + nc;
#pragma unroll
        for (int j = 0; j < 32; ++j) if (nc + j < p.N) op[j] = cvt16_rt(v[j], p.out_f16);
    }
    if (p.out_f32 != nullptr) {
        float* op = p.out_f32 + static_cast<size_t>(m) * p.ld_f32 + nc;
#pragma unroll
        for (int j = 0; j < 32; ++j) if (nc + j < p.N) op[j] = v[j];
    }
}
template <bool F16>
__device__ __forceinline__ void store_chunk(const GemmEpilogue& p, int m, int nc, bool fast, const float (&v)[32]) {
    if (fast) {
        if (p.out_bf16 != nullptr) store16x32<F16>(p.out_bf16 + static_cast<size_t>(m) * p.ld_bf16 + nc, v);
        if (p.out_f32 != nullptr) store_f32x32(p.out_f32 + static_cast<size_t>(m) * p.ld_f32 + nc, v);
    } else {
        float tmp[32];                       // only this (ragged N / odd stride) path touches local memory
#pragma unroll
        for (int j = 0; j < 32; ++j) tmp[j] = v[j];
        store_chunk_slow(p, m, nc, tmp);
    }
}

// ---- row-contiguous stores through a per-warp 2 KB shared-memory transpose (32 rows x 64 bytes, XOR-swizzled)
// Row r keeps its four 16-byte units j at position j ^ ((r >> 1) & 3): the row-per-lane writes (one unit per instruction) and
// the 8-rows-per-instruction reads (lane -> row it*8 + lane/4, unit lane%4) are both bank-conflict free, and every global
// store instruction writes 8 rows x 64 contiguous bytes.  The epilogue is bound by LSU wavefronts (one per 128-byte line
// touched per instruction): 32-byte row pieces cost twice as many as these 64-byte ones.
__device__ __forceinline__ int sw_unit(int r, int j) { return r * 4 + (j ^ ((r >> 1) & 3)); }     // in 16-byte units
template <bool F16>
__device__ __forceinline__ void store16_sw(uint4* st, __nv_bfloat16* out, int ld, int m_warp, int M, int ncol,
                                           const float (&v)[32], int lane) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint4 u;
        u.x = F16 ? pack16x2_rt(v[8 * j + 0], v[8 * j + 1], 1) : pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
        u.y = F16 ? pack16x2_rt(v[8 * j + 2], v[8 * j + 3], 1) : pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
        u.z = F16 ? pack16x2_rt(v[8 * j + 4], v[8 * j + 5], 1) : pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
        u.w = F16 ? pack16x2_rt(v[8 * j + 6], v[8 * j + 7], 1) : pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
        st[sw_unit(lane, j)] = u;
    }
    __syncwarp();
    const int j = lane & 3;
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const int r = it * 8 + (lane >> 2);
        const uint4 u = st[sw_unit(r, j)];
        if (m_warp + r < M) *reinterpret_cast<uint4*>(out + static_cast<size_t>(m_warp + r) * ld + ncol + j * 8) = u;
    }
    __syncwarp();                                          // staging buffer is reused by the next chunk
}
// fp32, 16 columns per pass; nvalid = columns of this chunk that exist (N - ncol): a ragged last chunk (the 3129-wide VQA
// head) is finished with scalar stores from the same transposed layout.
__device__ __forceinline__ void store_f32_sw(uint4* st, float* out, int ld, int m_warp, int M, int ncol, const float (&v)[32],
                                             int lane, int nvalid = 32) {
    const int j = lane & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const float4 f = make_float4(v[16 * h + 4 * jj], v[16 * h + 4 * jj + 1], v[16 * h + 4 * jj + 2], v[16 * h + 4 * jj + 3]);
            st[sw_unit(lane, jj)] = *reinterpret_cast<const uint4*>(&f);
        }
        __syncwarp();
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int r = it * 8 + (lane >> 2);
            const uint4 u = st[sw_unit(r, j)];
            const float4 f = *reinterpret_cast<const float4*>(&u);
            const int c0 = 16 * h + 4 * j;
            if (m_warp + r < M) {
                float* o4 = out + static_cast<size_t>(m_warp + r) * ld + ncol + c0;
                if (c0 + 4 <= nvalid) {
                    *reinterpret_cast<float4*>(o4) = f;
                } else {
                    if (c0 + 0 < nvalid) o4[0] = f.x;
                    if (c0 + 1 < nvalid) o4[1] = f.y;
                    if (c0 + 2 < nvalid) o4[2] = f.z;
                }
            }
        }
        __syncwarp();
    }
}

template <int BLOCK_N, int ACT, bool F16, int MODE = 0>
__global__ void __launch_bounds__(PCfg<BLOCK_N, MODE>::kThreads, PCfg<BLOCK_N, MODE>::kMinBlocks)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_c, const GemmEpilogue p, const int num_m_tiles,
                       const int num_n_tiles) {
    using Cfg = PCfg<BLOCK_N, MODE>;
    constexpr int kStages = Cfg::kStages;
    constexpr int kNC = Cfg::kNumChunks;
    constexpr int kEpiThreads = Cfg::kEpiThreads;
    static_assert(BLOCK_N % 32 == 0 && BLOCK_N >= 64 && BLOCK_N <= 256, "epilogue works in 32-column chunks");

    // 1024-byte alignment (SWIZZLE_128B atoms) by pointer arithmetic on the shared array: an integer round trip would turn every
    // later access into a GENERIC load/store (LD.E / ST.E instead of LDS / STS in the epilogue -- seen in the SASS)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    if ((smem_u32(smem_raw) & 1023u) != 0u) {            // SWIZZLE_128B atoms need it; the budget has no slack to re-align
        if (threadIdx.x == 0) printf("vb: dynamic shared memory base %u not 1024-byte aligned\n", smem_u32(smem_raw));
        __trap();
    }
    uint8_t* ring = smem_raw;
    float* s_acc = reinterpret_cast<float*>(ring + kStages * Cfg::kStageBytes);    // [128][kAccLd] deposited accumulator
    float* s_bias = s_acc + kBlockM * Cfg::kAccLd;                                  // [BLOCK_N]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_bias + Cfg::kBiasFloats);
    uint64_t* empty_bar = full_bar + kStages;
    uint8_t* s_xpose = reinterpret_cast<uint8_t*>(empty_bar + kStages) + 16;       // [kEpiWarps][kXposeBytesPerWarp]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_kb = (p.K + kBlockK - 1) / kBlockK;
    // profiling stamps (first tile of each CTA): 0 entry, 1 setup done, 2 first k-block landed, 3 last k-block accumulated,
    // 4 accumulator ready, 5 and 7 epilogue done, 6 producer past griddepcontrol.wait (VB200_STAMPS builds)
    long long* stamps = p.timing ? p.timing + 16 * (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
    if (stamps && threadIdx.x == 0) {
        stamps[0] = clock64();
        unsigned long long gt;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        stamps[8] = static_cast<long long>(gt);                                    // ns, for launch-ramp analysis
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        stamps[12] = smid;                                                         // per-SM occupancy (scripts/step_timeline.py)
    }

    // ---- tile assignment.  CTA b takes tiles b, b+grid, ... with the N index fastest (CTAs that run together share an A row-panel
    // in L2).
    // Packed batches (p.m_rows): the producer and the consumers derive the same, shorter tile list from the device row count --
    // M tiles whose first row is at or past it do not exist for this launch.  The count is written before the graph starts.  A CTA
    // left without a tile triggers its dependents by exiting.
    int run_m_tiles = num_m_tiles;
    if constexpr (MODE == 6) {
        const int mr = max(0, min(*p.m_rows, p.M));
        run_m_tiles = min(num_m_tiles, (mr + kBlockM - 1) / kBlockM);
    }
    const int total_tiles = run_m_tiles * num_n_tiles;
    const int first_tile = static_cast<int>(blockIdx.x);
    const int tile_stride = static_cast<int>(gridDim.x);
    auto tile_m0 = [&](int tile) { return (tile / num_n_tiles) * kBlockM; };
    auto tile_n0 = [&](int tile) { return (tile % num_n_tiles) * BLOCK_N; };

    // ---------------------------------------------------------------- one-time setup
    // The producer thread does not wait for the CTA-wide setup barrier: as soon as ITS barriers exist it puts the first ring
    // pass of the first tile in flight -- activations and weights when the kernel has no programmatic dependency (pdl 0),
    // only the weights (they do not depend on the previous kernel) when it was launched programmatically with pdl == 5; the
    // activation tiles then follow after griddepcontrol.wait.
    int early = 0;                 // k-blocks of the first tile already (partly) in flight     } producer thread only
    bool early_a = false;          // ... including their activation tiles                       }
    if (warp == Cfg::kProducerWarp && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        if (p.tma_store) tma_prefetch_desc(&tmap_c);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], Cfg::kConsumerWarps);                   // one arrival per consumer warp
        }
        mbar_fence_init();
#ifdef VB200_DECOMPOSE
        const bool early_ok = !(p.debug & 4);
#else
        constexpr bool early_ok = true;
#endif
        if (first_tile < total_tiles && p.pdl != 1 && early_ok) {
            early_a = p.pdl != 5;
            const int m0 = (first_tile / num_n_tiles) * kBlockM, n0 = (first_tile % num_n_tiles) * BLOCK_N;
            early = min(kStages, num_kb);
            for (int i = 0; i < early; ++i) {                  // fresh barriers: every slot is free
                uint8_t* sa = ring + i * Cfg::kStageBytes;
                mbar_arrive_expect_tx(&full_bar[i], Cfg::kStageBytes);
                if (early_a) tma_load_2d(sa, &tmap_a, &full_bar[i], i * kBlockK, m0);
                tma_load_2d(sa + Cfg::kStageBytesA, &tmap_b, &full_bar[i], i * kBlockK, n0);
            }
        }
    }
    __syncthreads();
    if (stamps && threadIdx.x == 0) stamps[1] = clock64();

    // Programmatic dependent launch: everything above overlapped the previous kernel's tail; its outputs are visible after the
    // wait.  (The producer thread of a pdl == 5 kernel waits inside its own branch, right before the first activation tile.)
    const bool producer_thread = warp == Cfg::kProducerWarp && lane == 0;
    if (p.pdl && !(p.pdl == 5 && producer_thread)) pdl_wait();

    if (warp == Cfg::kProducerWarp) {
        // ============================================================ TMA producer
        if (lane == 0) {
            int s = 0;
            uint32_t phase = 0;
            if (p.pdl == 5) pdl_wait();
#ifdef VB200_STAMPS
            if (stamps) stamps[6] = clock64();                         // producer past griddepcontrol.wait
#endif
            for (int tile = first_tile; tile < total_tiles; tile += tile_stride) {
                const int m0 = tile_m0(tile), n0 = tile_n0(tile);
                for (int kb = 0; kb < num_kb; ++kb) {
                    uint8_t* sa = ring + s * Cfg::kStageBytes;
                    uint8_t* sb = sa + Cfg::kStageBytesA;
                    if (early > 0) {                           // first ring pass of the first tile: already (partly) in flight
                        --early;
                        if (!early_a) tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kBlockK, m0);
                    } else {
                        mbar_wait_nocall(&empty_bar[s], phase ^ 1u);
#ifdef VB200_DECOMPOSE
                        if (p.debug & 4) {
                            mbar_arrive(&full_bar[s]);                 // timing decomposition: MMAs on stale shared memory
                        } else
#endif
                        {
                            mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
                            tma_load_2d(sa, &tmap_a, &full_bar[s], kb * kBlockK, m0);
                            tma_load_2d(sb, &tmap_b, &full_bar[s], kb * kBlockK, n0);
                        }
                    }
                    if (++s == kStages) { s = 0; phase ^= 1u; }
                }
            }
        }
        __syncwarp();
    } else {
        // ============================================================ consumer warpgroups: MMA, then epilogue
        // One k-block's wgmma group stays in flight while the stage of the previous one is handed back to the producer.
        constexpr uint64_t kDescStage = static_cast<uint64_t>(Cfg::kStageBytes >> 4);       // descriptor address units (16 B)
        const int wg = warp >> 2;
        const uint64_t da0 = gmma_desc_kmajor_sw128(smem_u32(ring + wg * 64 * 128));         // this warpgroup's 64 rows of A
        const uint64_t db0 = gmma_desc_kmajor_sw128(smem_u32(ring + Cfg::kStageBytesA));
        int ks = 0;
        uint32_t kphase = 0;
        // a stage is free once this warp's wgmma have read it
        auto release = [&](int st) __attribute__((always_inline)) {
            if (lane == 0) mbar_arrive(&empty_bar[st]);
        };
        // accumulate tile `tile` and deposit it in s_acc; returns once all 128 rows are there
        auto mma_tile = [&](int tile, uint32_t it) __attribute__((always_inline)) {
            float d[BLOCK_N / 2];
            int prev = -1;
            if constexpr (MODE == 7) {
                // fp32-parity mode (GemmEpilogue::split_acc): every k-block (one of hi.hi, lo.hi, hi.lo over 64 columns) starts from zero in the wgmma
                // accumulator and is added to `sum` on the CUDA cores, round to nearest.  Accumulating all K' = 3K products in the
                // wgmma accumulator loses bits at every k step instead, an error that grows with K: on the 268 M model (K = 768 ...
                // 3072) it put the forward ~15x further from fp64 than fp32 arithmetic is.  One k-block in flight at a time.
                float sum[BLOCK_N / 2];
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait_nocall(&full_bar[ks], kphase);
                    const uint64_t da = da0 + kDescStage * static_cast<uint64_t>(ks);
                    const uint64_t db = db0 + kDescStage * static_cast<uint64_t>(ks);
                    mma_kblock<BLOCK_N, F16>(d, da, db, true);
                    wgmma_wait<0>();
                    release(ks);
                    if (++ks == kStages) { ks = 0; kphase ^= 1u; }
#pragma unroll
                    for (int j = 0; j < BLOCK_N / 2; ++j) sum[j] = kb == 0 ? d[j] : __fadd_rn(sum[j], d[j]);
                }
                if (p.pdl && threadIdx.x == 0 && tile + tile_stride >= total_tiles) pdl_launch_dependents();
                acc_deposit<BLOCK_N>(s_acc, sum, threadIdx.x);
                epi_bar_sync<kEpiThreads>();
                return;
            }
            for (int kb = 0; kb < num_kb; ++kb) {
                mbar_wait_nocall(&full_bar[ks], kphase);
#ifdef VB200_STAMPS
                if (stamps && threadIdx.x == 0 && it == 0 && kb == 0) stamps[2] = clock64();
#endif
                const uint64_t da = da0 + kDescStage * static_cast<uint64_t>(ks);
                const uint64_t db = db0 + kDescStage * static_cast<uint64_t>(ks);
#ifdef VB200_DECOMPOSE
                if (!(p.debug & 1))
#endif
                    mma_kblock<BLOCK_N, F16>(d, da, db, kb == 0);
                if (prev >= 0) {
                    wgmma_wait<1>();                                     // k-block kb - 1 has read its stage
                    release(prev);
                }
                prev = ks;
                if (++ks == kStages) { ks = 0; kphase ^= 1u; }
            }
            wgmma_wait<0>();
            if (prev >= 0) release(prev);
#ifdef VB200_STAMPS
            if (stamps && threadIdx.x == 0 && it == 0) stamps[3] = clock64();
#endif
            // This CTA's tensor work is done: let the next kernel's CTAs come up while the epilogue drains (their
            // griddepcontrol.wait still holds them until this whole grid has finished).
            if (p.pdl && threadIdx.x == 0 && tile + tile_stride >= total_tiles) pdl_launch_dependents();
            acc_deposit<BLOCK_N>(s_acc, d, threadIdx.x);
            epi_bar_sync<kEpiThreads>();                                 // the whole tile is deposited
        };
        const int ew = warp;                          // 0..kEpiWarps-1
        const int q = ew & 3;                         // row quarter of the tile this warp owns
        const int row = q * 32 + lane;
        const int et = threadIdx.x;
        const bool st_fast = (p.out_bf16 == nullptr || (p.ld_bf16 & 7) == 0) && (p.out_f32 == nullptr || (p.ld_f32 & 3) == 0);
        uint32_t it = 0;
        for (int tile = first_tile; tile < total_tiles; tile += tile_stride, ++it) {
            const int m0 = tile_m0(tile), n0 = tile_n0(tile);
            const int m = m0 + row;
            const bool m_ok = m < p.M;
            const float* acc_row = s_acc + row * Cfg::kAccLd;
            const bool stamp = stamps && it == 0 && et == 0;

            // ------------------------------------------------ epilogue: 8 warps, one 32-column chunk at a time
            const float* bias_t = s_bias;
            // per-tile bias slice; the barrier below orders it before the reads, the one at the end of the tile orders
            // the reads before the next tile's writes
            for (int i = et; i < BLOCK_N; i += kEpiThreads) s_bias[i] = (p.bias && n0 + i < p.N) ? p.bias[n0 + i] : 0.0f;
            epi_bar_sync<kEpiThreads>();
            mma_tile(tile, it);
            if (stamp) stamps[4] = clock64();
            float* const out_f32 = p.out_f32;
            // TMA-store path (CTA-uniform): this is the CTA's last tile, so no operand load is or will be in flight and
            // every MMA that read the ring has completed (mma_tile above)
            constexpr bool kF32SlabsFit = (BLOCK_N / 32) * (kBlockM * 128) <= kStages * Cfg::kStageBytes;
            const bool use_tma = p.tma_store != 0 && st_fast && tile + tile_stride >= total_tiles &&
                                 (p.tma_store == 1 || kF32SlabsFit) &&
                                 (p.tma_store == 1 ? (p.out_bf16 != nullptr && p.out_f32 == nullptr)
                                                   : (p.out_f32 != nullptr && p.out_bf16 == nullptr));
            auto finish_chunk = [&](float (&v)[32], int nc) __attribute__((always_inline)) {
                bias_act32<ACT>(v, bias_t + (nc - n0));
#ifdef VB200_DECOMPOSE
                if ((p.debug & 2) && __float_as_uint(v[0]) != 0x7fc12345u) return;     // timing decomposition: no stores
#endif
                if (p.mul != nullptr && m_ok) {
                    const float* mp = p.mul + static_cast<size_t>(m) * p.ld_mul + nc;
                    if ((p.ld_mul & 3) == 0 && nc + 32 <= p.N) {          // 8 x 16-byte loads instead of 32 scalar ones
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float4 f = reinterpret_cast<const float4*>(mp)[j];
                            v[4 * j] *= f.x; v[4 * j + 1] *= f.y; v[4 * j + 2] *= f.z; v[4 * j + 3] *= f.w;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j) if (nc + j < p.N) v[j] *= mp[j];
                    }
                }
                if (use_tma) {
                    // last tile of this CTA: the operand ring is idle -> stage the tile there in the TMA's SWIZZLE_128B
                    // layout (16-byte unit u of row r at u ^ (r & 7): row-per-lane writes are bank-conflict free)
                    const int cl = nc - n0;
                    if (p.tma_store == 1) {                              // 16-bit: slabs of 64 columns x 128 rows (16 KB)
                        uint4* slab = reinterpret_cast<uint4*>(ring + (cl >> 6) * (kBlockM * 128)) + row * 8;
                        const int u0 = (cl & 32) ? 4 : 0;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            uint4 u;
                            u.x = F16 ? pack16x2_rt(v[8 * j + 0], v[8 * j + 1], 1) : pack_bf16x2(v[8 * j + 0], v[8 * j + 1]);
                            u.y = F16 ? pack16x2_rt(v[8 * j + 2], v[8 * j + 3], 1) : pack_bf16x2(v[8 * j + 2], v[8 * j + 3]);
                            u.z = F16 ? pack16x2_rt(v[8 * j + 4], v[8 * j + 5], 1) : pack_bf16x2(v[8 * j + 4], v[8 * j + 5]);
                            u.w = F16 ? pack16x2_rt(v[8 * j + 6], v[8 * j + 7], 1) : pack_bf16x2(v[8 * j + 6], v[8 * j + 7]);
                            slab[(u0 + j) ^ (row & 7)] = u;
                        }
                    } else {                                             // fp32: slabs of 32 columns x 128 rows (16 KB)
                        uint4* slab = reinterpret_cast<uint4*>(ring + (cl >> 5) * (kBlockM * 128)) + row * 8;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float4 f = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                            slab[j ^ (row & 7)] = *reinterpret_cast<const uint4*>(&f);
                        }
                    }
                    return;
                }
                uint4* xb = reinterpret_cast<uint4*>(s_xpose + ew * Cfg::kXposeBytesPerWarp);
                const int nvalid = p.N - nc;                                   // < 32 in a ragged last chunk, <= 0 beyond N
                const bool fast16 = st_fast && nvalid >= 32 && p.out_bf16 != nullptr;
                const bool fast32 = st_fast && nvalid > 0 && p.out_f32 != nullptr;                 // all warp-uniform
                if (fast32) store_f32_sw(xb, out_f32, p.ld_f32, m0 + q * 32, p.M, nc, v, lane, nvalid);
                if (fast16) {
                    if constexpr (MODE == 3 || MODE == 7) {
                        // fp32-parity mode: the 16-bit operand is written as fp16 hi | lo | hi per 64 columns (split_col),
                        // so the consuming GEMM's K' = 3K contraction against W' = hi | hi | lo adds hi.hi + lo.hi + hi.lo
                        const int c3 = split_col(nc);
                        store16_sw<F16>(xb, p.out_bf16, p.ld_bf16, m0 + q * 32, p.M, c3, v, lane);
                        store16_sw<F16>(xb, p.out_bf16, p.ld_bf16, m0 + q * 32, p.M, c3 + 128, v, lane);
#pragma unroll
                        for (int j = 0; j < 32; ++j) v[j] = split_lo(v[j]);
                        store16_sw<F16>(xb, p.out_bf16, p.ld_bf16, m0 + q * 32, p.M, c3 + 64, v, lane);
                    } else {
                        store16_sw<F16>(xb, p.out_bf16, p.ld_bf16, m0 + q * 32, p.M, nc, v, lane);
                    }
                }
                if (m_ok && nvalid > 0 && ((p.out_f32 != nullptr && !fast32) || (p.out_bf16 != nullptr && !fast16))) {
                    GemmEpilogue ps = p;                       // per-lane (ragged 16-bit / odd stride) remainder
                    ps.out_f32 = out_f32;
                    if (fast32) ps.out_f32 = nullptr;
                    if (fast16) ps.out_bf16 = nullptr;
                    store_chunk<F16>(ps, m, nc, false, v);
                }
            };
            {
                // eight warps: column group g = ew / 4 takes chunks [g * kNC/2, (g+1) * kNC/2)
                constexpr int kCPG = kNC / 2;
                const int g = ew >> 2;
#pragma unroll
                for (int ci = 0; ci < kCPG; ++ci) {
                    const int c = g * kCPG + ci;
                    float v[32];
                    acc_ld32(acc_row + c * 32, v);
                    if (stamp && ci == 0) stamps[14] = clock64();         // first chunk in registers
                    finish_chunk(v, n0 + c * 32);
                    if (stamp && ci == 0) stamps[15] = clock64();         // first chunk stored
                }
            }
            if (use_tma) {
                fence_proxy_async_smem();                        // my staged rows -> visible to the TMA
                epi_bar_sync<kEpiThreads>();                     // ... and everybody else's
                if (et == 0) {
                    if (p.tma_store == 1) {
                        for (int sl = 0; sl < BLOCK_N / 64; ++sl)
                            if (n0 + sl * 64 < p.N) tma_store_2d(&tmap_c, ring + sl * (kBlockM * 128), n0 + sl * 64, m0);
                    } else {
                        for (int sl = 0; sl < BLOCK_N / 32; ++sl)
                            if (n0 + sl * 32 < p.N) tma_store_2d(&tmap_c, ring + sl * (kBlockM * 128), n0 + sl * 32, m0);
                    }
                    tma_store_commit_and_wait_read();            // the ring is read before this CTA tears down
                }
            }
            if (stamp) { stamps[5] = clock64(); stamps[7] = clock64(); }
            if (tile + tile_stride < total_tiles) epi_bar_sync<kEpiThreads>();   // bias slice and s_acc free for the next tile
        }
    }

    // ---------------------------------------------------------------- teardown
    __syncthreads();
    if (stamps && threadIdx.x == 0) {
        unsigned long long gt;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        stamps[9] = static_cast<long long>(gt);
        stamps[13] = clock64();
    }
}


// --------------------------------------------------------------------------------------------- host side (shared)
inline int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

template <typename Cfg>
void fill_cfg(cudaLaunchConfig_t& cfg, cudaLaunchAttribute* attrs, dim3 grid, int pdl, cudaStream_t st) {
    cfg = cudaLaunchConfig_t{};
    cfg.gridDim = grid;
    cfg.blockDim = dim3(Cfg::kThreads, 1, 1);
    cfg.dynamicSmemBytes = Cfg::kSmemBytes;
    cfg.stream = st;
    unsigned na = 0;
    if (pdl) {
        attrs[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attrs[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attrs;
    cfg.numAttrs = na;
}

// Persistent grid of a plain kernel with one CTA per SM: every SM by default.  VB200_GRID_PCT caps it at that percentage of the
// SMs, leaving room for kernels of the other ViLBERT stream / the other in-flight batch; grid_pct (10..100) overrides it per launch
// (profiling: timed alone).
inline int persistent_grid(int tiles, int grid_pct) {
    static const int env_pct = [] { const char* e = getenv("VB200_GRID_PCT"); const int v = e ? atoi(e) : 100; return (v >= 10 && v <= 100) ? v : 100; }();
    const int pct = (grid_pct >= 10 && grid_pct <= 100) ? grid_pct : env_pct;
    const int slots = std::max(1, num_sms() * pct / 100);
    // balanced walk: every CTA gets the same number of tiles (+-1): tiles = 288, cap 132 -> 96 CTAs x 3 instead of 24 x 3 + 108 x 2
    static const bool balance = [] { const char* e = getenv("VB200_GRID_BALANCE"); return e == nullptr || atoi(e) != 0; }();
    int g = std::min(tiles, slots);
    if (balance && tiles > slots) { const int per = (tiles + slots - 1) / slots; g = (tiles + per - 1) / per; }
    return g;
}

template <int BLOCK_N, int ACT, bool F16, int MODE = 0>
cudaError_t launch_p(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const GemmEpilogue& ep, int grid_pct,
                     cudaStream_t st) {
    using Cfg = PCfg<BLOCK_N, MODE>;
    auto kern = gemm_persistent_kernel<BLOCK_N, ACT, F16, MODE>;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return e;
    const int n_tiles = (ep.N + BLOCK_N - 1) / BLOCK_N;
    const int m_tiles = (ep.M + kBlockM - 1) / kBlockM;
    static_assert(Cfg::kMinBlocks == 1, "persistent_grid assumes one CTA per SM");
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attrs[1];
    fill_cfg<Cfg>(cfg, attrs, dim3(persistent_grid(m_tiles * n_tiles, grid_pct), 1, 1), ep.pdl == 1 || ep.pdl == 5, st);
    GemmEpilogue e2 = ep;
    if (tc == nullptr) { e2.tma_store = 0; tc = &ta; }                             // &ta: any valid map for the unused slot
    return cudaLaunchKernelEx(&cfg, kern, ta, tb, *tc, e2, m_tiles, n_tiles);
}

}  // namespace pgemm
}  // namespace vb
