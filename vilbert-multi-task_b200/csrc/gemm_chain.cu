// Two dependent GEMMs in ONE persistent launch (VERDICT r1 item 2(ii)): the FFN of a BertLayer / BertImageLayer / connection layer,
//     H = act(X W1^T + b1)   (16-bit, [M, N1])          Y = H W2^T + b2   ([M, N2], fp32 for the LayerNorm that follows)
// ([UPSTREAM] BertIntermediate + BertOutput.dense, vilbert/vilbert.py; anchor worker.py:286-289).
//
// Why: at batch 64 a GEMM launch is dominated by per-CTA fixed cost and every CTA owns one or two tiles.
// Here the CTAs of one grid pull tiles of BOTH GEMMs from one ordered list (chain_decode) -- the second GEMM's tiles of a row panel
// become available right after the first GEMM's tiles of the NEXT panel -- so there is no launch gap and no second prologue, the
// producer fills the ring for the next tile while the consumers run an epilogue, and the long-K second GEMM (96 tiles at batch
// 64) no longer leaves a third of the SMs idle.
//
// Dependency: tile (m, n) of GEMM 2 reads rows [128 m, 128 m + 128) of H, i.e. ALL N1 / 128 tiles of panel m of GEMM 1.  Every GEMM-1
// tile, once its stores are globally visible (membar + release), increments panel_done[m]; the TMA producer of a GEMM-2 tile
// spins on panel_done[m] == N1 / 128 (acquire) before its first load of H.  No deadlock: list positions are handed out in increasing
// order and every dependency of a position is a smaller position, so the smallest unfinished position never waits on anything
// (the grid is persistent: at most the resident CTA slots; programmatic dependents cannot occupy slots before every CTA of this grid
// has triggered).  The last CTA to finish resets the counters, so a CUDA graph can replay the launch.
// Same tiles, same accumulation order as two separate launches: results are bit-identical (tests/test_gpu_ops.py::test_gemm_chain).
#include <cstdlib>
#include "gemm_persistent.cuh"

namespace vb {
namespace pgemm {

struct ChainParams {
    GemmEpilogue p[2];
    int m_tiles;            // row panels (shared by both GEMMs)
    int n_tiles[2];
    int* sync;              // [m_tiles] GEMM-1 tiles finished per panel | [m_tiles] next list position | [m_tiles + 1] CTAs finished
};

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
    asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Tile list (position -> work item).  P row panels; block 0 = the GEMM-1 tiles of panel 0, block b = [GEMM-1 tiles of panel b |
// GEMM-2 tiles of panel b - 1], last block = the GEMM-2 tiles of panel P - 1: a panel's second-GEMM tiles are handed out one panel's
// worth of first-GEMM tiles after its own -- by the time a CTA fetches one, its inputs are (nearly) complete, and the long-K
// second-GEMM tiles are spread over the whole launch instead of forming its tail.  Every dependency of a position lies at a smaller
// position, and positions are handed out in order (atomic counter): the smallest unfinished position can always make progress.
struct ChainTile { int g, m_t, n_t; };
__device__ __forceinline__ ChainTile chain_decode(int pos, int P, int n0, int n1) {
    ChainTile t;
    if (pos < n0) { t.g = 0; t.m_t = 0; t.n_t = pos; return t; }
    const int q = pos - n0, S = n0 + n1;
    const int b = q / S + 1, r = q - (b - 1) * S;
    if (b < P && r < n0) { t.g = 0; t.m_t = b; t.n_t = r; }
    else { t.g = 1; t.m_t = b - 1; t.n_t = b < P ? r - n0 : r; }      // (b == P: only the n1 tiles of the last panel remain)
    return t;
}

// the plain kernel's layout plus two tile_done barriers
constexpr int kChainSmemBytes = PCfg<128, false, 0>::kSmemBytes + 16;
static_assert(kChainSmemBytes <= 232448, "shared memory budget");

template <bool F16>
__global__ void __launch_bounds__(PCfg<128, false, 0>::kThreads, 1)
gemm_chain_kernel(const __grid_constant__ CUtensorMap ta0, const __grid_constant__ CUtensorMap tb0,
                  const __grid_constant__ CUtensorMap ta1, const __grid_constant__ CUtensorMap tb1, const ChainParams cp) {
    using Cfg = PCfg<128, false, 0>;
    constexpr int BLOCK_N = 128;
    constexpr int kStages = Cfg::kStages;
    constexpr int kNC = Cfg::kNumChunks;
    constexpr int kEpiThreads = Cfg::kEpiThreads;

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    if ((smem_u32(smem_raw) & 1023u) != 0u) __trap();
    uint8_t* ring = smem_raw;
    float* s_acc = reinterpret_cast<float*>(ring + kStages * Cfg::kStageBytes);
    float* s_bias = s_acc + kBlockM * Cfg::kAccLd;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_bias + Cfg::kBiasFloats);
    uint64_t* empty_bar = full_bar + kStages;
    uint64_t* sched_full = empty_bar + kStages;                       // [2] position published in s_tile[i & 1]
    uint64_t* tile_done = sched_full + 2;                             // [2] the consumers have finished the tile of slot i & 1
    volatile int* s_tile = reinterpret_cast<volatile int*>(tile_done + 2);
    uint8_t* s_xpose = reinterpret_cast<uint8_t*>(tile_done + 2) + 16;   // kChainSmemBytes: 16 bytes more than the plain kernel

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int P = cp.m_tiles, n0t = cp.n_tiles[0], n1t = cp.n_tiles[1];
    const int total = P * (n0t + n1t);
    const int pdl = cp.p[0].pdl;
    int* panel_done = cp.sync;
    int* next_pos = cp.sync + P;
    int* fin = cp.sync + P + 1;

    if (warp == Cfg::kProducerWarp && lane == 0) {
        tma_prefetch_desc(&ta0); tma_prefetch_desc(&tb0); tma_prefetch_desc(&ta1); tma_prefetch_desc(&tb1);
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], Cfg::kConsumerWarps); }
        for (int a = 0; a < 2; ++a) { mbar_init(&sched_full[a], 1); mbar_init(&tile_done[a], 1); }
        mbar_fence_init();
    }
    __syncthreads();
    if (pdl) pdl_wait();

    // Dynamic tile scheduler.  The producer thread fetches list positions (atomicAdd) and publishes position i of this CTA in
    // s_tile[i & 1] / sched_full[i & 1]; it rewrites a slot for position i + 2 only after the consumers have finished tile i
    // (tile_done[i & 1]).
    if (warp == Cfg::kProducerWarp) {
        // ============================================================ TMA producer + scheduler
        if (lane == 0) {
            int s = 0;
            uint32_t phase = 0, it = 0;
            while (true) {
                const int pos = atomicAdd(next_pos, 1);
                if (it >= 2) mbar_wait_nocall(&tile_done[it & 1u], ((it >> 1) & 1u) ^ 1u);   // tile it - 2 finished: slot reusable
                s_tile[it & 1u] = pos;
                mbar_arrive(&sched_full[it & 1u]);                     // release: the consumers' try_wait acquires
                if (pos >= total) break;
                const ChainTile t = chain_decode(pos, P, n0t, n1t);
                const CUtensorMap* ta = t.g ? &ta1 : &ta0;
                const CUtensorMap* tb = t.g ? &tb1 : &tb0;
                const int num_kb = (cp.p[t.g].K + kBlockK - 1) / kBlockK;
                if (t.g == 1) {
                    // rows of H this tile reads come from the N1 / 128 GEMM-1 tiles of panel m_t, written by other CTAs
                    uint32_t spins = 0;
                    while (ld_acquire_gpu(panel_done + t.m_t) < n0t) {
                        if (++spins > VB_SPIN_LIMIT) __trap();          // no printf: a call here would serialise the wgmma (C7510)
                    }
                    fence_proxy_async_all();           // generic-proxy observation -> the async-proxy (TMA) reads that follow
                }
                for (int kb = 0; kb < num_kb; ++kb) {
                    uint8_t* sa = ring + s * Cfg::kStageBytes;
                    mbar_wait_nocall(&empty_bar[s], phase ^ 1u);
                    mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
                    tma_load_2d(sa, ta, &full_bar[s], kb * kBlockK, t.m_t * kBlockM);
                    tma_load_2d(sa + Cfg::kStageBytesA, tb, &full_bar[s], kb * kBlockK, t.n_t * BLOCK_N);
                    if (++s == kStages) { s = 0; phase ^= 1u; }
                }
                ++it;
            }
        }
        __syncwarp();
    } else {
        // ============================================================ consumer warpgroups: MMA, then epilogue
        constexpr uint64_t kDescStage = static_cast<uint64_t>(Cfg::kStageBytes >> 4);
        const int wg = warp >> 2;
        const uint64_t da0 = gmma_desc_kmajor_sw128(smem_u32(ring + wg * 64 * 128));
        const uint64_t db0 = gmma_desc_kmajor_sw128(smem_u32(ring + Cfg::kStageBytesA));
        const int ew = warp, q = warp & 3, et = threadIdx.x;
        const int row = q * 32 + lane;
        const float* acc_row = s_acc + row * Cfg::kAccLd;
        int ks = 0;
        uint32_t kphase = 0;
        for (uint32_t it = 0;; ++it) {
            mbar_wait_nocall(&sched_full[it & 1u], (it >> 1) & 1u);
            const int pos = s_tile[it & 1u];
            if (pos >= total) break;
            const ChainTile t = chain_decode(pos, P, n0t, n1t);
            const GemmEpilogue& p = cp.p[t.g];
            const int num_kb = (p.K + kBlockK - 1) / kBlockK;
            const int m0 = t.m_t * kBlockM, n0 = t.n_t * BLOCK_N;
            for (int i = et; i < BLOCK_N; i += kEpiThreads) s_bias[i] = (p.bias && n0 + i < p.N) ? p.bias[n0 + i] : 0.0f;
            {
                float d[BLOCK_N / 2];
                int prev = -1;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait_nocall(&full_bar[ks], kphase);
                    mma_kblock<BLOCK_N, F16>(d, da0 + kDescStage * static_cast<uint64_t>(ks), db0 + kDescStage * static_cast<uint64_t>(ks), kb == 0);
                    if (prev >= 0) {
                        wgmma_wait<1>();
                        if (lane == 0) mbar_arrive(&empty_bar[prev]);
                    }
                    prev = ks;
                    if (++ks == kStages) { ks = 0; kphase ^= 1u; }
                }
                wgmma_wait<0>();
                if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
                acc_deposit<BLOCK_N>(s_acc, d, threadIdx.x);
            }
            epi_bar_sync<kEpiThreads>();                               // tile deposited, bias slice written
            constexpr int kCPG = kNC / 2;
            const int cg = ew >> 2;
#pragma unroll
            for (int ci = 0; ci < kCPG; ++ci) {
                const int c = cg * kCPG + ci;
                const int nc = n0 + c * 32;
                float v[32];
                acc_ld32(acc_row + c * 32, v);
                const float* bs = s_bias + c * 32;
                if (p.act == kActGelu) bias_act32<kActGelu>(v, bs);
                else if (p.act == kActRelu) bias_act32<kActRelu>(v, bs);
                else bias_act32<kActNone>(v, bs);
                if (nc < p.N) {                                         // host: N % 32 == 0, aligned strides
                    uint4* xb = reinterpret_cast<uint4*>(s_xpose + ew * Cfg::kXposeBytesPerWarp);
                    if (p.out_f32 != nullptr) store_f32_sw(xb, p.out_f32, p.ld_f32, m0 + q * 32, p.M, nc, v, lane, 32);
                    if (p.out_bf16 != nullptr) store16_sw<F16>(xb, p.out_bf16, p.ld_bf16, m0 + q * 32, p.M, nc, v, lane);
                }
            }
            // this tile of H is complete once every consumer thread's stores are visible device-wide; the barrier also frees
            // s_acc and the bias slice for the next tile
            if (t.g == 0) __threadfence();
            epi_bar_sync<kEpiThreads>();
            if (et == 0) {
                if (t.g == 0) red_release_gpu_add(panel_done + t.m_t, 1);
                mbar_arrive(&tile_done[it & 1u]);
            }
        }
        if (pdl && threadIdx.x == 0) pdl_launch_dependents();
    }

    __syncthreads();
    // the last CTA to leave zeroes the counters: the launch can be replayed (CUDA graph) without a memset node
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(fin, 1) == static_cast<int>(gridDim.x) - 1) {
            for (int i = 0; i < P + 2; ++i) cp.sync[i] = 0;
            __threadfence();
        }
    }
}

}  // namespace pgemm

// ep0: X -> H (16-bit output only); ep1: H -> Y.  Both with 128-wide tiles; sync: (m_tiles + 2) zeroed ints owned by this launch site.
cudaError_t launch_gemm_chain(const CUtensorMap& ta0, const CUtensorMap& tb0, const GemmEpilogue& ep0, const CUtensorMap& ta1,
                              const CUtensorMap& tb1, const GemmEpilogue& ep1, int* sync, cudaStream_t st) {
    using namespace pgemm;
    using Cfg = PCfg<128, false, 0>;
    if (ep0.M != ep1.M || ep0.M < 1 || ep0.N < 1 || ep1.N < 1 || ep0.K < 1 || ep1.K < 1 || sync == nullptr) return cudaErrorInvalidValue;
    if (ep0.a_f16 != ep1.a_f16 || ep0.a_f16 != ep0.out_f16 || ep1.a_f16 != ep1.out_f16) return cudaErrorInvalidValue;
    for (const GemmEpilogue* e : {&ep0, &ep1}) {
        if (e->res || e->mul || e->gamma || e->split16 || e->ln_mode || (e->N & 31) || (e->out_bf16 && (e->ld_bf16 & 7)) ||
            (e->out_f32 && (e->ld_f32 & 3)) || (!e->out_bf16 && !e->out_f32) || e->act == kActGeluExact)
            return cudaErrorInvalidValue;
    }
    if (ep0.out_bf16 == nullptr) return cudaErrorInvalidValue;                            // H is GEMM 2's A operand
    auto kern = ep0.a_f16 ? gemm_chain_kernel<true> : gemm_chain_kernel<false>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmemBytes);
    if (e != cudaSuccess) return e;
    ChainParams cp{};
    cp.p[0] = ep0; cp.p[1] = ep1;
    cp.p[0].tma_store = cp.p[1].tma_store = 0;
    cp.m_tiles = (ep0.M + kBlockM - 1) / kBlockM;
    cp.n_tiles[0] = (ep0.N + 127) / 128; cp.n_tiles[1] = (ep1.N + 127) / 128;
    cp.sync = sync;
    const int tiles = cp.m_tiles * (cp.n_tiles[0] + cp.n_tiles[1]);
    static const int env_pct = [] { const char* v = getenv("VB200_CHAIN_GRID_PCT"); const int x = v ? atoi(v) : 100; return (x >= 10 && x <= 100) ? x : 100; }();
    const int slots = std::max(1, num_sms() * Cfg::kMinBlocks * env_pct / 100);
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attrs[2];
    fill_cfg<Cfg, false>(cfg, attrs, dim3(std::min(tiles, slots), 1, 1), 1, ep0.pdl == 1 || ep0.pdl == 5, st);
    cfg.dynamicSmemBytes = kChainSmemBytes;
    return cudaLaunchKernelEx(&cfg, kern, ta0, tb0, ta1, tb1, cp);
}

}  // namespace vb
