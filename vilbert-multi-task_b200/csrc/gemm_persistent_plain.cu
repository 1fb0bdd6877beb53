// Instantiations (bias / GELU / ReLU / pooled-product) and launcher of the persistent wgmma GEMM; see gemm_persistent.cuh.
#include "gemm_persistent.cuh"

namespace vb {
using namespace pgemm;

int num_sms_host() { return pgemm::num_sms(); }

int gemm_p_pick_block_n(int N) { return N <= 64 ? 64 : 128; }

template <int BN, int MODE>
static cudaError_t dispatch_act(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const GemmEpilogue& ep, int pct,
                                cudaStream_t st) {
    const bool f16 = ep.a_f16 != 0;
    switch (ep.act) {
        case kActNone: return f16 ? launch_p<BN, kActNone, true, MODE>(ta, tb, tc, ep, pct, st) : launch_p<BN, kActNone, false, MODE>(ta, tb, tc, ep, pct, st);
        case kActGelu: return f16 ? launch_p<BN, kActGelu, true, MODE>(ta, tb, tc, ep, pct, st) : launch_p<BN, kActGelu, false, MODE>(ta, tb, tc, ep, pct, st);
        case kActRelu: return f16 ? launch_p<BN, kActRelu, true, MODE>(ta, tb, tc, ep, pct, st) : launch_p<BN, kActRelu, false, MODE>(ta, tb, tc, ep, pct, st);
    }
    return cudaErrorInvalidValue;
}

// fp32-parity mode (fp16 hi/lo operands, K' = 3K): PCfg MODE 3 writes the 16-bit output as hi | lo | hi; GELU with the 1.5e-7 erf.
// MODE 7 is MODE 3 whose k-blocks are summed with round-to-nearest fp32 adds (GemmEpilogue::split_acc).
template <int BN, int MODE>
static cudaError_t dispatch_split(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const GemmEpilogue& ep, int pct,
                                cudaStream_t st) {
    switch (ep.act) {
        case kActNone: return launch_p<BN, kActNone, true, MODE>(ta, tb, tc, ep, pct, st);
        case kActGelu:
        case kActGeluExact: return launch_p<BN, kActGeluExact, true, MODE>(ta, tb, tc, ep, pct, st);
        case kActRelu: return launch_p<BN, kActRelu, true, MODE>(ta, tb, tc, ep, pct, st);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_gemm_persistent_plain(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap* tc, const GemmEpilogue& ep,
                                         int block_n, int pct, cudaStream_t st) {
    if (ep.M < 1 || ep.N < 1 || ep.K < 1 || ep.a_f16 != ep.out_f16) return cudaErrorInvalidValue;
    if (ep.split16 || ep.split_acc || ep.act == kActGeluExact) {
        // hi | lo | hi output: fp16, whole 64-column groups, no TMA store; narrow tiles only (the mode is for parity, not speed).
        // The k-block sums of MODE 7 take 64-wide tiles only (128-wide ones spill).
        if (!ep.a_f16 || (ep.split16 && (ep.out_bf16 == nullptr || (ep.N & 63) || (ep.ld_bf16 & 7))) || ep.tma_store == 1 ||
            (ep.split_acc && block_n != 64))
            return cudaErrorInvalidValue;
        if (ep.split_acc) return dispatch_split<64, 7>(ta, tb, tc, ep, pct, st);
        return block_n == 64 ? dispatch_split<64, 3>(ta, tb, tc, ep, pct, st) : dispatch_split<128, 3>(ta, tb, tc, ep, pct, st);
    }
    const bool rows = ep.m_rows != nullptr;          // MODE 6: the tile list ends at a device row count (packed batches)
    switch (block_n) {
        case 64: return rows ? dispatch_act<64, 6>(ta, tb, tc, ep, pct, st) : dispatch_act<64, 0>(ta, tb, tc, ep, pct, st);
        case 128: return rows ? dispatch_act<128, 6>(ta, tb, tc, ep, pct, st) : dispatch_act<128, 0>(ta, tb, tc, ep, pct, st);
        case 192:                                    // 128x192 tiles, 2-stage ring
            if (ep.N % 192 != 0) return cudaErrorInvalidValue;
            return rows ? dispatch_act<192, 6>(ta, tb, tc, ep, pct, st) : dispatch_act<192, 0>(ta, tb, tc, ep, pct, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace vb
