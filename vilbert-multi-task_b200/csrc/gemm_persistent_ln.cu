// LayerNorm-fused (cluster) instantiations of the persistent wgmma GEMM; see gemm_persistent.cuh.
#include <cstdlib>
#include "gemm_persistent.cuh"

namespace vb {
using namespace pgemm;

// How many clusters of `cluster` CTAs of the LN kernel can be resident at once (0 = that cluster size cannot launch).
template <int BLOCK_N>
static int max_clusters(int cluster) {
    using Cfg = PCfg<BLOCK_N, true>;
    static int cache[kMaxCluster + 1] = {};   // 0 unknown, -1 unsupported
    if (cluster < 1 || cluster > kMaxCluster) return 0;
    if (cache[cluster] != 0) return cache[cluster] < 0 ? 0 : cache[cluster];
    auto kern = gemm_persistent_kernel<BLOCK_N, true, kActNone, true>;
    int n = 0;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes) == cudaSuccess &&
        cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess) {
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute attrs[2];
        fill_cfg<Cfg, true>(cfg, attrs, dim3(cluster, 1, 1), cluster, 0, nullptr);
        if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) n = 0;
    }
    cudaGetLastError();
    cache[cluster] = n > 0 ? n : -1;
    return n > 0 ? n : 0;
}

int num_sms_host() { return pgemm::num_sms(); }

int gemm_p_max_clusters(int block_n, int cluster) {
    switch (block_n) {
        case 64: return max_clusters<64>(cluster);
        case 96: return max_clusters<96>(cluster);
        case 128: return max_clusters<128>(cluster);
    }
    return 0;
}

int gemm_p_pick_block_n(int N, bool ln) {
    if (!ln) {
        static const int forced = [] { const char* e = getenv("VB200_BN"); return e ? atoi(e) : 0; }();   // A/B switch
        if ((forced == 64 || forced == 128) && N % forced == 0) return forced;
        return N <= 64 ? 64 : 128;
    }
    static const int first = [] { const char* e = getenv("VB200_LN_BN"); return e ? atoi(e) : 128; }();   // A/B: preferred width
    const int cands[4] = {first, 128, 96, 64};
    for (int ci = 0; ci < 4; ++ci) {
        const int bn = cands[ci];
        if (bn != 64 && bn != 96 && bn != 128) continue;
        if (N % bn != 0 || N / bn > kMaxCluster) continue;
        if (gemm_p_max_clusters(bn, N / bn) > 0) return bn;
    }
    return 0;
}

template <int BN>
static cudaError_t dispatch_ln(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, cudaStream_t st) {
    const bool f16 = ep.a_f16 != 0;
    const int resident = max_clusters<BN>(ep.N / BN);
    switch (ep.act) {
        case kActNone: return f16 ? launch_p<BN, true, kActNone, true>(ta, tb, ep, resident, st) : launch_p<BN, true, kActNone, false>(ta, tb, ep, resident, st);
        case kActGelu: return f16 ? launch_p<BN, true, kActGelu, true>(ta, tb, ep, resident, st) : launch_p<BN, true, kActGelu, false>(ta, tb, ep, resident, st);
    }
    return cudaErrorInvalidValue;     // ReLU + LayerNorm does not occur on the ViLBERT path
}

cudaError_t launch_gemm_persistent(const CUtensorMap& ta, const CUtensorMap& tb, const GemmEpilogue& ep, int block_n,
                                   bool ln, cudaStream_t st) {
    if (ep.M < 1 || ep.N < 1 || ep.K < 1) return cudaErrorInvalidValue;
    if (!ln) return launch_gemm_persistent_plain(ta, tb, ep, block_n, st);
    if (ep.N % block_n != 0 || ep.N / block_n > kMaxCluster || ep.gamma == nullptr || ep.beta == nullptr ||
        (ep.out_bf16 && (ep.ld_bf16 & 7)) || (ep.out_f32 && (ep.ld_f32 & 3)) || (ep.res && (ep.ld_res & 3)) ||
        ep.mul != nullptr || ep.a_f16 != ep.out_f16)
        return cudaErrorInvalidValue;
    switch (block_n) {
        case 64: return dispatch_ln<64>(ta, tb, ep, st);
        case 96: return dispatch_ln<96>(ta, tb, ep, st);
        case 128: return dispatch_ln<128>(ta, tb, ep, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace vb
