// Instantiations and launcher of the ping-pong wgmma GEMM; see gemm_pingpong.cuh.
#include "gemm_pingpong.cuh"

namespace vb {
using namespace ppgemm;

template <int BN, int ACT, bool F16, int MODE>
static cudaError_t launch_pp(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc16, const CUtensorMap& tc32,
                             const GemmEpilogue& ep, int pct, cudaStream_t st) {
    using Cfg = PPCfg<BN>;
    auto kern = gemm_pingpong_kernel<BN, ACT, F16, MODE>;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes);
    if (e != cudaSuccess) return e;
    const int n_tiles = ep.N / BN;
    const int m_tiles = (ep.M + kBlockM - 1) / kBlockM;
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute attrs[1];
    pgemm::fill_cfg<Cfg>(cfg, attrs, dim3(pgemm::persistent_grid(m_tiles * n_tiles, pct), 1, 1), ep.pdl == 1 || ep.pdl == 5, st);
    return cudaLaunchKernelEx(&cfg, kern, ta, tb, tc16, tc32, ep, m_tiles, n_tiles);
}

template <int BN, int MODE>
static cudaError_t dispatch_pp(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc16, const CUtensorMap& tc32,
                               const GemmEpilogue& ep, int pct, cudaStream_t st) {
    const bool f16 = ep.a_f16 != 0;
    switch (ep.act) {
        case kActNone: return f16 ? launch_pp<BN, kActNone, true, MODE>(ta, tb, tc16, tc32, ep, pct, st) : launch_pp<BN, kActNone, false, MODE>(ta, tb, tc16, tc32, ep, pct, st);
        case kActGelu: return f16 ? launch_pp<BN, kActGelu, true, MODE>(ta, tb, tc16, tc32, ep, pct, st) : launch_pp<BN, kActGelu, false, MODE>(ta, tb, tc16, tc32, ep, pct, st);
        case kActRelu: return f16 ? launch_pp<BN, kActRelu, true, MODE>(ta, tb, tc16, tc32, ep, pct, st) : launch_pp<BN, kActRelu, false, MODE>(ta, tb, tc16, tc32, ep, pct, st);
    }
    return cudaErrorInvalidValue;
}

bool gemm_pingpong_supports(const GemmEpilogue& ep, int block_n) {
    return (block_n == 64 || block_n == 128) && ep.M >= 1 && ep.K >= 1 && ep.N >= block_n && ep.N % block_n == 0 &&
           ep.mul == nullptr && !ep.split16 && ep.a_f16 == ep.out_f16 &&
           (ep.act == kActNone || ep.act == kActGelu || ep.act == kActRelu) && (ep.out_bf16 != nullptr || ep.out_f32 != nullptr);
}

cudaError_t launch_gemm_pingpong(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc16, const CUtensorMap* tc32,
                                 const GemmEpilogue& ep, int block_n, int pct, cudaStream_t st) {
    if (!gemm_pingpong_supports(ep, block_n) || (ep.out_bf16 != nullptr && tc16 == nullptr) ||
        (ep.out_f32 != nullptr && tc32 == nullptr))
        return cudaErrorInvalidValue;
    const CUtensorMap& c16 = tc16 ? *tc16 : ta;        // &ta: any valid map for an unused slot
    const CUtensorMap& c32 = tc32 ? *tc32 : ta;
    const bool rows = ep.m_rows != nullptr;
    if (block_n == 64) return rows ? dispatch_pp<64, 6>(ta, tb, c16, c32, ep, pct, st) : dispatch_pp<64, 0>(ta, tb, c16, c32, ep, pct, st);
    return rows ? dispatch_pp<128, 6>(ta, tb, c16, c32, ep, pct, st) : dispatch_pp<128, 0>(ta, tb, c16, c32, ep, pct, st);
}

}  // namespace vb
