// Host side of the vilbert_b200 engine: BertConfig JSON, state_dict audit + weight repack, per-shape plans
// (workspace, TMA descriptors, launch list, CUDA graph) and the C ABI of include/vilbert_b200.h.
//
// Mirrors what the reference does at worker.py:495-536 (config + from_pretrained + cuda)
// and worker.py:286-289 (the forward call); the layer schedule and module wiring follow the [UPSTREAM]
// vilbert/vilbert.py restated in SURVEY.md section 3C / 8a.
#include "../../include/vilbert_b200.h"

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <numeric>
#include <stdexcept>
#include <string>
#include <utility>
#include <variant>
#include <vector>

#include <nvtx3/nvToolsExt.h>      // header-only NVTX v3: ranges per layer / per forward for nsys and ncu --nvtx (SURVEY.md section 5)

#include "kernels.h"

namespace {

using vb::GemmEpilogue;
typedef __nv_bfloat16 bf16;

struct VbError : std::runtime_error {
    int status;
    VbError(int s, const std::string& m) : std::runtime_error(m), status(s) {}
};

[[noreturn]] void fail(int status, const char* fmt, ...) {
    char buf[2048];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    throw VbError(status, buf);
}

#define CUDA_CHECK(expr)                                                                                    \
    do {                                                                                                    \
        cudaError_t _e = (expr);                                                                            \
        if (_e != cudaSuccess) fail(VB200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                                    __FILE__, __LINE__);                                                    \
    } while (0)

std::string g_create_error;   // last failed vb200_create (no handle to hang it on)

// ------------------------------------------------------------------------------------------ tiny JSON
struct JVal {
    enum Kind { NUM, STR, BOOL, ARR, NUL, OBJ } kind = NUL;
    double num = 0;
    bool b = false;
    std::string str;
    std::vector<double> arr;
};

struct JsonParser {
    const char* p;
    explicit JsonParser(const char* s) : p(s) {}
    void ws() { while (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r') ++p; }
    std::string parse_string() {
        if (*p != '"') fail(VB200_ERR_CONFIG, "config JSON: expected string");
        ++p;
        std::string s;
        while (*p && *p != '"') {
            if (*p != '\\') { s.push_back(*p++); continue; }
            ++p;                                                   // escape sequence (RFC 8259 section 7)
            switch (*p) {
                case 'n': s.push_back('\n'); break;
                case 't': s.push_back('\t'); break;
                case 'r': s.push_back('\r'); break;
                case 'b': s.push_back('\b'); break;
                case 'f': s.push_back('\f'); break;
                case 'u': {                                        // \uXXXX -> UTF-8 (basic multilingual plane; surrogates kept as-is)
                    unsigned cp = 0;
                    for (int i = 1; i <= 4; ++i) {
                        const char c = p[i];
                        const int d = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : (c >= 'A' && c <= 'F') ? c - 'A' + 10 : -1;
                        if (d < 0) fail(VB200_ERR_CONFIG, "config JSON: bad \\u escape");
                        cp = cp * 16 + static_cast<unsigned>(d);
                    }
                    p += 4;
                    if (cp < 0x80) s.push_back(static_cast<char>(cp));
                    else if (cp < 0x800) { s.push_back(static_cast<char>(0xC0 | (cp >> 6))); s.push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
                    else { s.push_back(static_cast<char>(0xE0 | (cp >> 12))); s.push_back(static_cast<char>(0x80 | ((cp >> 6) & 0x3F))); s.push_back(static_cast<char>(0x80 | (cp & 0x3F))); }
                    break;
                }
                case '\0': fail(VB200_ERR_CONFIG, "config JSON: unterminated string");
                default: s.push_back(*p);                          // \" \\ \/
            }
            ++p;
        }
        if (*p != '"') fail(VB200_ERR_CONFIG, "config JSON: unterminated string");
        ++p;
        return s;
    }
    void skip_value();
    JVal parse_value() {
        ws();
        JVal v;
        if (*p == '"') { v.kind = JVal::STR; v.str = parse_string(); }
        else if (*p == '[') {
            v.kind = JVal::ARR;
            ++p; ws();
            while (*p && *p != ']') {
                JVal e = parse_value();
                if (e.kind == JVal::NUM) v.arr.push_back(e.num);
                ws();
                if (*p == ',') { ++p; ws(); }
            }
            if (*p != ']') fail(VB200_ERR_CONFIG, "config JSON: unterminated array");
            ++p;
        } else if (*p == '{') {            // nested objects are skipped (none carry model dimensions)
            v.kind = JVal::OBJ;
            int depth = 0;
            do {
                if (*p == '"') { parse_string(); continue; }
                if (*p == '{') ++depth;
                if (*p == '}') --depth;
                ++p;
            } while (*p && depth > 0);
        } else if (!strncmp(p, "true", 4)) { v.kind = JVal::BOOL; v.b = true; p += 4; }
        else if (!strncmp(p, "false", 5)) { v.kind = JVal::BOOL; v.b = false; p += 5; }
        else if (!strncmp(p, "null", 4)) { v.kind = JVal::NUL; p += 4; }
        else {
            char* end = nullptr;
            v.num = strtod(p, &end);
            if (end == p) fail(VB200_ERR_CONFIG, "config JSON: unexpected character '%c'", *p);
            v.kind = JVal::NUM;
            p = end;
        }
        return v;
    }
    std::map<std::string, JVal> parse_object() {
        std::map<std::string, JVal> m;
        ws();
        if (*p != '{') fail(VB200_ERR_CONFIG, "config JSON: expected '{'");
        ++p; ws();
        while (*p && *p != '}') {
            std::string k = parse_string();
            ws();
            if (*p != ':') fail(VB200_ERR_CONFIG, "config JSON: expected ':' after \"%s\"", k.c_str());
            ++p;
            m[k] = parse_value();
            ws();
            if (*p == ',') { ++p; ws(); }
        }
        if (*p != '}') fail(VB200_ERR_CONFIG, "config JSON: unterminated object");
        return m;
    }
};

struct Config {
    int hidden = 768, layers = 12, heads = 12, inter = 3072, max_pos = 512, type_vocab = 2, vocab = 30522;
    int v_feat = 2048, v_target = 1601, v_hidden = 1024, v_layers = 6, v_heads = 8, v_inter = 1024;
    int bi_hidden = 1024, bi_heads = 8;
    int task_tokens = 1, n_task = 20;
    int visual_target = 0, predict_feature = 0;   // pre-training options: read here, accepted only at 0 by vb200_create_pretraining
    std::vector<int> v_bi_id{0, 1, 2, 3, 4, 5}, t_bi_id{6, 7, 8, 9, 10, 11};
    std::string hidden_act = "gelu", v_hidden_act = "gelu", fusion = "mul";
    float ln_eps = 1e-12f;
};

Config parse_config(const char* json) {
    Config c;
    if (json == nullptr) fail(VB200_ERR_CONFIG, "config JSON is NULL");
    JsonParser jp(json);
    auto m = jp.parse_object();
    auto geti = [&](const char* k, int& dst) {
        auto it = m.find(k);
        if (it == m.end()) return;
        if (it->second.kind == JVal::NUM) dst = static_cast<int>(it->second.num);
        else if (it->second.kind == JVal::BOOL) dst = it->second.b ? 1 : 0;
    };
    geti("hidden_size", c.hidden); geti("num_hidden_layers", c.layers); geti("num_attention_heads", c.heads);
    geti("intermediate_size", c.inter); geti("max_position_embeddings", c.max_pos);
    geti("type_vocab_size", c.type_vocab); geti("vocab_size", c.vocab); geti("v_feature_size", c.v_feat);
    geti("v_target_size", c.v_target); geti("v_hidden_size", c.v_hidden); geti("v_num_hidden_layers", c.v_layers);
    geti("v_num_attention_heads", c.v_heads); geti("v_intermediate_size", c.v_inter);
    geti("bi_hidden_size", c.bi_hidden); geti("bi_num_attention_heads", c.bi_heads);
    geti("task_specific_tokens", c.task_tokens); geti("num_task_tokens", c.n_task);
    geti("visual_target", c.visual_target); geti("predict_feature", c.predict_feature);
    auto geta = [&](const char* k, std::vector<int>& dst) {
        auto it = m.find(k);
        if (it == m.end() || it->second.kind != JVal::ARR) return;
        dst.clear();
        for (double d : it->second.arr) dst.push_back(static_cast<int>(d));
    };
    geta("v_biattention_id", c.v_bi_id); geta("t_biattention_id", c.t_bi_id);
    auto gets = [&](const char* k, std::string& dst) {
        auto it = m.find(k);
        if (it != m.end() && it->second.kind == JVal::STR) dst = it->second.str;
    };
    gets("hidden_act", c.hidden_act); gets("v_hidden_act", c.v_hidden_act); gets("fusion_method", c.fusion);
    int dyn = 0;
    geti("dynamic_attention", dyn);
    // ---- what this engine implements (everything the worker configures, worker.py:509-522)
    if (dyn) fail(VB200_ERR_CONFIG, "dynamic_attention=true is not supported (worker.py:484 sets it false)");
    if (c.hidden_act != "gelu" || c.v_hidden_act != "gelu") fail(VB200_ERR_CONFIG, "only hidden_act = gelu is supported");
    if (c.fusion != "mul") fail(VB200_ERR_CONFIG, "only fusion_method = mul is supported");
    if (c.v_bi_id.size() != c.t_bi_id.size()) fail(VB200_ERR_CONFIG, "v_biattention_id / t_biattention_id length mismatch");
    // Connection layer i runs after the stream layers below ids[i]: every id must lie in [0, the stream's layer count] and no id
    // may be below the one before it (equal neighbours are back-to-back connection layers).  Anything else would index past the
    // layer lists when a plan is built, or leave checkpoint layers that never run.
    auto ids_ok = [](const char* field, const std::vector<int>& ids, int n_layers, const char* n_field) {
        for (size_t i = 0; i < ids.size(); ++i) {
            if (ids[i] < 0 || ids[i] > n_layers)
                fail(VB200_ERR_CONFIG, "%s[%zu] = %d is outside [0, %s = %d]", field, i, ids[i], n_field, n_layers);
            if (i > 0 && ids[i] < ids[i - 1])
                fail(VB200_ERR_CONFIG, "%s[%zu] = %d is below %s[%zu] = %d: the ids must not decrease", field, i, ids[i], field, i - 1,
                     ids[i - 1]);
        }
    };
    ids_ok("t_biattention_id", c.t_bi_id, c.layers, "num_hidden_layers");
    ids_ok("v_biattention_id", c.v_bi_id, c.v_layers, "v_num_hidden_layers");
    auto head_ok = [](int hid, int heads) { return heads > 0 && hid % heads == 0 && (hid / heads == 64 || hid / heads == 128); };
    if (!head_ok(c.hidden, c.heads) || !head_ok(c.v_hidden, c.v_heads) || !head_ok(c.bi_hidden, c.bi_heads))
        fail(VB200_ERR_CONFIG, "attention head size must be 64 or 128");
    for (int d : {c.hidden, c.v_hidden, c.bi_hidden, c.inter, c.v_inter})
        if (d % 128 != 0) fail(VB200_ERR_CONFIG, "hidden/intermediate sizes must be multiples of 128 (got %d)", d);
    if (c.hidden > 1024 || c.v_hidden > 1024 || c.bi_hidden > 1024)
        fail(VB200_ERR_CONFIG, "hidden sizes above 1024 are not supported");
    if (c.v_feat % 8 != 0) fail(VB200_ERR_CONFIG, "v_feature_size must be a multiple of 8");
    return c;
}

// ------------------------------------------------------------------------------------------ device memory
struct Arena {   // owns every device allocation of an engine / plan
    std::vector<void*> ptrs;
    size_t total = 0;
    void* alloc(size_t bytes) {
        void* p = nullptr;
        bytes = (bytes + 255) & ~size_t(255);
        CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 256));
        ptrs.push_back(p);
        total += bytes;
        return p;
    }
    template <typename T> T* alloc_n(size_t n) { return static_cast<T*>(alloc(n * sizeof(T))); }
    ~Arena() { for (void* p : ptrs) cudaFree(p); }
};

// Owners of the runtime's handles.  A stream is drained before it is destroyed: a launch list that throws midway leaves kernels
// that still read the workspace its plan is about to free.
struct EventDel { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct StreamDel { void operator()(cudaStream_t s) const { cudaStreamSynchronize(s); cudaStreamDestroy(s); } };
struct GraphDel { void operator()(cudaGraph_t g) const { cudaGraphDestroy(g); } };
struct GraphExecDel { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
struct PinnedDel { void operator()(char* p) const { cudaFreeHost(p); } };
using Event = std::unique_ptr<CUevent_st, EventDel>;
using Stream = std::unique_ptr<CUstream_st, StreamDel>;
using Graph = std::unique_ptr<CUgraph_st, GraphDel>;
using GraphExec = std::unique_ptr<CUgraphExec_st, GraphExecDel>;

Event make_event(unsigned flags = cudaEventDisableTiming) {
    cudaEvent_t e;
    CUDA_CHECK(cudaEventCreateWithFlags(&e, flags));
    return Event(e);
}
Stream make_stream() {
    cudaStream_t s;
    CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return Stream(s);
}
// What `enqueue` launches on st, as a graph.  A throw from enqueue ends the capture it aborted before it propagates.
Graph capture_graph(cudaStream_t st, const std::function<void()>& enqueue) {
    CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    cudaGraph_t g = nullptr;
    try {
        enqueue();
    } catch (...) {
        cudaStreamEndCapture(st, &g);
        Graph partial(g);
        throw;
    }
    const cudaError_t e = cudaStreamEndCapture(st, &g);
    Graph owned(g);
    CUDA_CHECK(e);
    return owned;
}
GraphExec instantiate(cudaGraph_t g) {
    cudaGraphExec_t x;
    CUDA_CHECK(cudaGraphInstantiate(&x, g, 0));
    return GraphExec(x);
}

// What a call builds on the host (a packed forward's row layout, the descriptors of the calls beside the forward) reaches the device
// through two owners.  Both grow on demand to at least twice their last size (and kMinGrowBytes), and set the pointer and the size
// together, once the allocation has succeeded.
//   Staging: a pinned host buffer and `copied`, recorded once the call's copies out of it are enqueued.  stage() waits on the host
//     until the previous call's copies have left the buffer, grows it, and lets the caller fill it and put its parts on the device.
//   Workspace: a device buffer and `done`, which the call records (release) after its last kernel that reads the buffer.  acquire()
//     makes the call's stream wait for the previous call's `done` before anything writes the buffer, so growth is stream-ordered
//     (cudaFreeAsync / cudaMallocAsync on that stream) and never blocks the host.
// Their events are created with the engine (a plan's Staging with its plan), never in the audit pass.
constexpr size_t kMinGrowBytes = 4096;
inline size_t grown(size_t have, size_t need) { return std::max({need, 2 * have, kMinGrowBytes}); }

struct Staging {
    Event copied;
    std::unique_ptr<char, PinnedDel> buf;
    size_t size = 0;
    ~Staging() { if (copied) cudaEventSynchronize(copied.get()); }
    void reserve(size_t bytes) {
        if (bytes <= size) return;
        char* p;
        CUDA_CHECK(cudaMallocHost(&p, bytes));
        buf.reset(p);
        size = bytes;
    }
    // fill(h, put): h holds `bytes`; put(dst, at, n) copies bytes [at, at + n) of h to the device at dst on st
    template <typename Fill> void stage(size_t bytes, cudaStream_t st, Fill&& fill) {
        CUDA_CHECK(cudaEventSynchronize(copied.get()));
        if (bytes > size) reserve(grown(size, bytes));
        char* h = buf.get();
        fill(h, [&](void* dst, size_t at, size_t n) { CUDA_CHECK(cudaMemcpyAsync(dst, h + at, n, cudaMemcpyHostToDevice, st)); });
        CUDA_CHECK(cudaEventRecord(copied.get(), st));
    }
};

struct Workspace {
    Event done;
    char* p = nullptr;
    size_t size = 0;
    ~Workspace() {
        if (done) cudaEventSynchronize(done.get());
        if (p) cudaFree(p);
    }
    char* acquire(size_t bytes, cudaStream_t st) {
        CUDA_CHECK(cudaStreamWaitEvent(st, done.get(), 0));
        if (bytes > size) {
            const size_t n = grown(size, bytes);
            void* q;
            CUDA_CHECK(cudaMallocAsync(&q, n, st));
            char* old = std::exchange(p, static_cast<char*>(q));
            size = n;
            if (old) CUDA_CHECK(cudaFreeAsync(old, st));
        }
        return p;
    }
    void release(cudaStream_t st) { CUDA_CHECK(cudaEventRecord(done.get(), st)); }
};

inline uint16_t f32_to_f16_bits(float f) {          // IEEE half, round to nearest even, saturating to +-65504
    const __half h = __float2half_rn(f);            // host-callable conversion from cuda_fp16.h
    uint16_t b;
    memcpy(&b, &h, 2);
    if ((b & 0x7fffu) == 0x7c00u) b = static_cast<uint16_t>((b & 0x8000u) | 0x7bffu);
    return b;
}
inline uint16_t f32_to_bf16_bits(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);   // NaN
    u += 0x7fffu + ((u >> 16) & 1u);                                                          // round to nearest even
    return static_cast<uint16_t>(u >> 16);
}
inline float bf16_bits_to_f32(uint16_t h) { uint32_t u = static_cast<uint32_t>(h) << 16; float f; memcpy(&f, &u, 4); return f; }
inline float half_bits_to_f32(uint16_t h) {
    const uint32_t sign = (h & 0x8000u) << 16, exp = (h >> 10) & 0x1f, man = h & 0x3ff;
    uint32_t u;
    if (exp == 0) {
        if (man == 0) u = sign;
        else {
            int e = -1; uint32_t m = man;
            do { ++e; m <<= 1; } while (!(m & 0x400));
            u = sign | ((127 - 15 - e) << 23) | ((m & 0x3ff) << 13);
        }
    } else if (exp == 31) u = sign | 0x7f800000u | (man << 13);
    else u = sign | ((exp + 112) << 23) | (man << 13);
    float f; memcpy(&f, &u, 4); return f;
}

struct HostTensor {
    int dtype = 0, ndim = 0;
    int64_t shape[2] = {0, 0};
    const void* data = nullptr;
    bool used = false;
    int64_t numel() const { return ndim == 1 ? shape[0] : shape[0] * shape[1]; }
    float at(int64_t i) const {
        switch (dtype) {
            case VB200_F32: return static_cast<const float*>(data)[i];
            case VB200_F16: return half_bits_to_f32(static_cast<const uint16_t*>(data)[i]);
            default: { uint32_t u = static_cast<uint32_t>(static_cast<const uint16_t*>(data)[i]) << 16; float f; memcpy(&f, &u, 4); return f; }
        }
    }
};

struct LinearW {            // nn.Linear [N, K] -> bf16 [N, ldw] (K zero-padded to a multiple of 64), fp32 bias
    bf16* w = nullptr;
    float* bias = nullptr;
    int N = 0, K = 0, ldw = 0;
};
struct LNW { float* g = nullptr; float* b = nullptr; int n = 0; };
struct RowW { float* w = nullptr; float* b = nullptr; int n_out = 0, K = 0; };   // narrow fp32 heads
struct LayerW { LinearW qkv, attn_out, inter, out; LNW ln1, ln2; };
struct ConnW { LinearW qkv_img, qkv_txt, dense1, dense2, v_inter, v_out, t_inter, t_out; LNW ln1, ln2, v_ln, t_ln; };
struct ClsW { LinearW fc0, fc3; LNW ln; RowW fc3_row; };

// ------------------------------------------------------------------------------------------ TMA descriptors
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
    if (qr != cudaDriverEntryPointSuccess || p == nullptr) fail(VB200_ERR_CUDA, "cuTensorMapEncodeTiled not available in this driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
    return fn;
}
// bf16 matrix [rows, cols] with row stride ld (elements); box = 64 columns x box_rows rows, 128-byte swizzle,
// out-of-bounds elements read as zero.
CUtensorMap make_tmap(const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, bool f16 = false) {
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld * 2) % 16 != 0)
        fail(VB200_ERR_INVALID, "TMA operand must be 16-byte aligned with a 16-byte-multiple row stride (ld=%lld)", (long long)ld);
    if (box_rows < 1 || box_rows > 256) fail(VB200_ERR_INVALID, "TMA box rows %d out of range", box_rows);
    CUtensorMap m;
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
    cuuint32_t box[2] = {64, static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode_fn()(&m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box,
                                 estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) fail(VB200_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld cols=%lld ld=%lld box_rows=%d)",
                                (int)r, (long long)rows, (long long)cols, (long long)ld, box_rows);
    return m;
}

// Output tile map for the TMA-store epilogue: [rows, cols] row-major with leading dimension ld (elements), boxes of 128 rows x
// 128 bytes (64 16-bit or 32 fp32 columns), SWIZZLE_128B.  Returns false when the buffer does not meet the TMA's alignment rules.
bool make_tmap_out(CUtensorMap* m, const void* base, int64_t rows, int64_t cols, int64_t ld, bool fp32, bool f16) {
    const int esz = fp32 ? 4 : 2;
    if (base == nullptr || (reinterpret_cast<uintptr_t>(base) & 15) || (ld * esz) % 16 != 0 || rows < 1 || cols < 1) return false;
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * esz};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(128 / esz), 128};
    cuuint32_t estr[2] = {1, 1};
    const CUtensorMapDataType dt = fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                        : (f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    return get_encode_fn()(m, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// Which kernel takes the plain GEMMs it supports: 1 ping-pong (default), 0 the cooperative gemm_persistent_kernel.
// VB200_GEMM=coop|pingpong is the A/B switch; vb200_set_option("gemm_kernel") changes it per engine.
int default_gemm_kernel() {
    static const int v = [] { const char* e = getenv("VB200_GEMM"); return (e && strcmp(e, "coop") == 0) ? 0 : 1; }();
    return v;
}

// One GEMM launch: operand maps, output maps, epilogue, tile width and kernel (make_gemm).
struct GemmCall {
    CUtensorMap ta{}, tb{};
    CUtensorMap tc16{}, tc32{};    // output maps of the TMA store: 16-bit and fp32 output (cooperative kernel: the one ep.tma_store names)
    GemmEpilogue ep{};
    int block_n = 128;
    bool pingpong = false;         // the ping-pong kernel (gemm_pingpong.cuh), else the cooperative one (gemm_persistent.cuh)
    // grid_pct: 0 the default persistent grid, 10..100 this percentage of the SMs (vb200_profile_ops)
    cudaError_t launch(cudaStream_t st, int grid_pct = 0) const {
        if (pingpong) return vb::launch_gemm_pingpong(ta, tb, &tc16, &tc32, ep, block_n, grid_pct, st);
        const CUtensorMap* tc = ep.tma_store == 1 ? &tc16 : (ep.tma_store == 2 ? &tc32 : nullptr);
        return vb::launch_gemm_persistent_plain(ta, tb, tc, ep, block_n, grid_pct, st);
    }
};
// What a caller fixes of a GEMM launch: the tile width (0: gemm_p_pick_block_n(N)) and the kernel -- 0 the cooperative one, 1 the
// ping-pong one wherever it takes the GEMM and the TMA can store every output (else the cooperative one), -1 as 1 or 0 by the process
// default (default_gemm_kernel).
struct GemmSpec { int block_n = 0; int kernel = -1; };
// A = [ep.M, ep.K] with row stride lda, W = [ep.N, ep.K] with row stride ldw (elements); ep names the outputs, activation and the
// rest of the epilogue but not the TMA store, which is decided here: ping-pong outputs all leave through the TMA, a cooperative
// GEMM with exactly one aligned output and no hi | lo | hi split stores its last tile through it.
GemmCall make_gemm(const void* A, int64_t lda, const void* W, int64_t ldw, const GemmEpilogue& ep, GemmSpec spec = {}) {
    GemmCall g;
    g.ep = ep;
    g.ep.tma_store = 0;
    g.block_n = spec.block_n > 0 ? spec.block_n : vb::gemm_p_pick_block_n(ep.N);
    g.ta = make_tmap(A, ep.M, ep.K, lda, 128, ep.a_f16 != 0);
    g.tb = make_tmap(W, ep.N, ep.K, ldw, g.block_n, ep.a_f16 != 0);
    auto out16 = [&](CUtensorMap* m) { return make_tmap_out(m, ep.out_bf16, ep.M, ep.N, ep.ld_bf16, false, ep.out_f16 != 0); };
    auto out32 = [&](CUtensorMap* m) { return make_tmap_out(m, ep.out_f32, ep.M, ep.N, ep.ld_f32, true, false); };
    const int kernel = spec.kernel < 0 ? default_gemm_kernel() : spec.kernel;
    g.pingpong = kernel == 1 && vb::gemm_pingpong_supports(ep, g.block_n) && (ep.out_bf16 == nullptr || out16(&g.tc16)) &&
                 (ep.out_f32 == nullptr || out32(&g.tc32));
    if (!g.pingpong && !ep.split16) {
        if (ep.out_bf16 != nullptr && ep.out_f32 == nullptr && out16(&g.tc16)) g.ep.tma_store = 1;
        else if (ep.out_f32 != nullptr && ep.out_bf16 == nullptr && out32(&g.tc32)) g.ep.tma_store = 2;
    }
    return g;
}

// ------------------------------------------------------------------------------------------ launch list
// Rows per sample: up to kStagedAttnRows a plan's attention stages whole (sample, head) tiles in shared memory (attention.cu), above
// it it streams K / V in key blocks.  kMaxRowsPerSample caps vb200_set_option("max_rows_per_sample"): region selection ranks at most
// 2048 proposals and the fp32 attention kernel holds 8 probability rows of up to 1024 keys in shared memory.
constexpr int kStagedAttnRows = 256;
constexpr int kMaxRowsPerSample = 1024;
// What a rejection above the bound names: the default bound is the staged kernels' limit, a raised one the engine's option.
inline const char* bound_name(int max_rows) {
    return max_rows == kStagedAttnRows ? "the small-sequence attention kernels" : "this engine's max_rows_per_sample";
}
// Launch-list entries.  Each kind's arguments are the named arguments of its launcher (kernels.h); packed plans add the device row
// count of the rows an op computes (m_rows) and the per-sample row offsets of the attention operands (offs*).
struct SelfAttnArgs {
    const bf16* qkv; int ld_qkv, hidden; const float* mask; bf16* ctx; int ld_ctx, B, L, heads, head_dim; const int* offs;
    bool stream_kv;                // the streaming kernel (more than kStagedAttnRows rows per sample)
    vb::HeadGate gate;             // gated packed plans: the entry's column of the plan's gate table
};
struct CoAttnArgs {
    const bf16 *qkv_img, *qkv_txt; int ld_img, ld_txt, hidden; const float *img_mask, *txt_mask;
    bf16 *ctx_txt, *ctx_img; int ld_ctx_txt, ld_ctx_img, B, T, V, heads, head_dim; const int *offs_t, *offs_v;
    bool stream_kv;                // the streaming kernel (either stream above kStagedAttnRows rows per sample)
    vb::HeadGate gate;             // gated packed plans: the text-query entry's column, the image-query one at gate.next
};
struct RowdotArgs { const float *x, *W, *bias, *add; float* out; int ld_x, ld_out, M, K, n_out; const int* m_rows; };
struct LayerNormArgs {             // out = LN(y + res)
    const float *y, *res, *gamma, *beta; int ld_y, ld_res; float* out_f32; int ld_f32; bf16* out16; int ld16, M, N; const int* m_rows;
};
// fp32 attention (attention_f32.cu): fp32-parity mode and the attention-probability output; packed: probabilities per sample (pk)
struct AttnF32Args {
    const void *q, *k, *v; int ld_q, ld_kv, in_kind; const float* mask; int B, Lq, Lk, heads, head_dim;
    bf16* ctx; int ld_ctx, ctx_mode; float* probs; bool packed; vb::PackedProbs pk;
    bool mean;                     // the head-mean kernel: maps only, [B, Lq, Lk] (packed: heads factor 1)
};
// Row offs[b] of src16 (ld16 wide) -> row b of dst16, b < B, clamped to n_src rows; with src_f32 the same row (`hidden` wide) -> dst_f32.
struct GatherArgs { const int* offs; int n_src, B; const bf16* src16; bf16* dst16; int ld16; const float* src_f32; float* dst_f32; int hidden; };

struct Op {
    // the index of the alternative is the kind number vb200_profile_ops reports
    std::variant<GemmCall, SelfAttnArgs, CoAttnArgs, RowdotArgs, LayerNormArgs, AttnF32Args, GatherArgs, vb::StateArgs> args;
    int stream = 0;                // 0 main, 1 side (image branch) inside the captured graph
    double flops = 0;
    enum Sync { NONE, FORK, JOIN } sync = NONE;   // fork/join markers for the two-stream graph
    const char* tag = nullptr;     // layer this launch belongs to ("T3", "V0", "C2", "embed", "heads"): NVTX range name
};
template <class... F> struct Overloaded : F... { using F::operator()...; };
template <class... F> Overloaded(F...) -> Overloaded<F...>;

struct OutBuf { float* p = nullptr; int rows = 0, cols = 0, ld = 0; };
// The twelve outputs of a forward, in vb200_outputs' order: per slot its field, the plan-key bit of a call that reads it -- a head's
// select bit, kTextRows / kImageRows (above the public bits) for a sequence tap, none for pooled_output, which every suffix plan
// writes -- what its rows are and its name in messages.  A packed plan holds its per-row outputs at the call's row totals.
constexpr uint32_t kTextRows = 1u << 30, kImageRows = 1u << 31;
enum OutRows { kPerSample, kPerPair, kTextRow, kImageRow };   // kPerPair: B / 2 rows, B at an odd batch
using OutField = float* vb200_outputs::*;
struct OutSlot { OutField field; uint32_t bit; OutRows rows; const char* name; };
enum { kOutVqa, kOutGqa, kOutVilLogit, kOutBinary, kOutTri, kOutVisionPred, kOutVisionLogit, kOutLingPred, kOutLingLogit, kOutSeqT,
       kOutSeqV, kOutPooled, kNumOuts };
constexpr OutSlot kOutSlots[kNumOuts] = {
    {&vb200_outputs::vil_prediction, VB200_OUT_VIL_PREDICTION, kPerSample, "vil_prediction (VB200_OUT_VIL_PREDICTION)"},
    {&vb200_outputs::vil_prediction_gqa, VB200_OUT_VIL_PREDICTION_GQA, kPerSample, "vil_prediction_gqa (VB200_OUT_VIL_PREDICTION_GQA)"},
    {&vb200_outputs::vil_logit, VB200_OUT_VIL_LOGIT, kPerSample, "vil_logit (VB200_OUT_VIL_LOGIT)"},
    {&vb200_outputs::vil_binary_prediction, VB200_OUT_VIL_BINARY_PREDICTION, kPerPair, "vil_binary_prediction (VB200_OUT_VIL_BINARY_PREDICTION)"},
    {&vb200_outputs::vil_tri_prediction, VB200_OUT_VIL_TRI_PREDICTION, kPerSample, "vil_tri_prediction (VB200_OUT_VIL_TRI_PREDICTION)"},
    {&vb200_outputs::vision_prediction, VB200_OUT_VISION_PREDICTION, kImageRow, "vision_prediction (VB200_OUT_VISION_PREDICTION)"},
    {&vb200_outputs::vision_logit, VB200_OUT_VISION_LOGIT, kImageRow, "vision_logit (VB200_OUT_VISION_LOGIT)"},
    {&vb200_outputs::linguisic_prediction, VB200_OUT_LINGUISIC_PREDICTION, kTextRow, "linguisic_prediction (VB200_OUT_LINGUISIC_PREDICTION)"},
    {&vb200_outputs::linguisic_logit, VB200_OUT_LINGUISIC_LOGIT, kTextRow, "linguisic_logit (VB200_OUT_LINGUISIC_LOGIT)"},
    {&vb200_outputs::sequence_output_t, kTextRows, kTextRow, "sequence_output_t"},
    {&vb200_outputs::sequence_output_v, kImageRows, kImageRow, "sequence_output_v"},
    {&vb200_outputs::pooled_output, 0, kPerSample, "pooled_output"},
};
// the plan-key bits of the outputs whose rows are `rows`
constexpr uint32_t out_bits(OutRows rows) {
    uint32_t m = 0;
    for (const OutSlot& o : kOutSlots) if (o.rows == rows) m |= o.bit;
    return m;
}

// ------------------------------------------------------------------------------------------ packed batches
// The d_meta format of a packed plan, in ints: text row offsets [B + 1] | image row offsets [B + 1]; with `src` (a packed pair suffix)
// then the pairs' first rows in the cached text states [B] | image states [B]; with n_entries > 0 (the packed attention
// probabilities, VB200_OUT_ATTENTION_PACKED) then, 8-byte aligned, the int64 destination pointer | entry float offsets [n_entries] |
// per-sample prefix sums [3][B + 1] (sum T_b'^2, sum V_b'^2, sum T_b' V_b' over b' < b); with n_states > 0 (the layer states,
// VB200_OUT_LAYER_STATES, which dense plans stage in the same format) then, 8-byte aligned, one int64 destination pointer per selected
// state entry.  A stream's row total, which bounds its GEMM, LayerNorm and rowdot rows, is its last offset.
struct MetaLayout {
    size_t B = 0, n_entries = 0;
    bool src = false;
    size_t n_states = 0;
    size_t offs_t() const { return 0; }
    size_t offs_v() const { return B + 1; }
    size_t rows_t() const { return offs_t() + B; }
    size_t rows_v() const { return offs_v() + B; }
    size_t src_t() const { return 2 * (B + 1); }
    size_t src_v() const { return src_t() + B; }
    size_t rows_end() const { return src ? src_v() + B : src_t(); }
    size_t probs_dst() const { return (rows_end() + 1) & ~static_cast<size_t>(1); }
    size_t probs_entry(size_t e) const { return probs_dst() + 2 * (1 + e); }
    size_t probs_prefix(int k) const { return probs_entry(n_entries) + 2 * static_cast<size_t>(k) * (B + 1); }
    size_t probs_end() const { return n_entries ? probs_prefix(3) : rows_end(); }
    size_t state_dst(size_t e) const { return ((probs_end() + 1) & ~static_cast<size_t>(1)) + 2 * e; }
    size_t size() const { return n_states ? state_dst(n_states) : probs_end(); }
};

// Which attention maps a forward writes (vb200_set_option "attention_entries" / "attention_heads"): bit e of `mask` selects entry e
// of the full list (execution order; a configuration with more than 63 entries always writes every entry), `mean` writes each
// selected entry averaged over heads (heads 1 in the layouts).  The default is every entry, every head.
struct AttnSelect {
    uint64_t mask = ~0ull;
    bool mean = false;
    bool has(int e) const { return e > 63 || ((mask >> e) & 1); }
    int heads(int h) const { return mean ? 1 : h; }
};
// The full list's entries in execution order: kinds 0 text layer, 1 image layer, 2 / 3 the two directions of a connection layer.
std::vector<int> attention_kinds(const std::vector<std::string>& schedule) {
    std::vector<int> k;
    for (const std::string& step : schedule) {
        if (step[0] == 'T') k.push_back(0);
        else if (step[0] == 'V') k.push_back(1);
        else { k.push_back(2); k.push_back(3); }
    }
    return k;
}

// Which layer states a forward writes (vb200_set_option "state_entries" / "state_rows"): bit e of `mask` selects entry e of the full
// list (state_kinds; a configuration with more than 63 entries always writes every entry), `rows` 0 every row, 1 each sample's first
// row, 2 each sample's mean over its real rows.  The default is every entry, every row.
struct StateSelect {
    uint64_t mask = ~0ull;
    int rows = 0;
    bool has(int e) const { return e > 63 || ((mask >> e) & 1); }
    int index(int e) const { return e > 63 ? e : __builtin_popcountll(mask & ((1ull << e) - 1)); }   // e's place in the layouts
};
// The full layer-state list in execution order, 0 a text state and 1 an image state: the text and the image embedding, then per
// schedule step the state of each stream it writes, text first.  Built next to attention_kinds so both lists follow the schedule.
std::vector<int> state_kinds(const std::vector<std::string>& schedule) {
    std::vector<int> k{0, 1};
    for (const std::string& step : schedule) {
        if (step[0] != 'V') k.push_back(0);
        if (step[0] != 'T') k.push_back(1);
    }
    return k;
}
// Layout of vb200_outputs.layer_states: the selected entries in execution order, each `rows` x width floats back to back.  rows_t /
// rows_v are a stream's rows under state_rows 0 (dense: B x T / B x V, packed: the call's row totals); state_rows 1 and 2 give B.
struct StateLayout {
    std::vector<int32_t> kind, rows, width;
    std::vector<int64_t> offset;
    int64_t total = 0;
};
StateLayout state_layout(const Config& c, const std::vector<std::string>& schedule, const StateSelect& sel, int B, int64_t rows_t,
                         int64_t rows_v) {
    StateLayout l;
    const std::vector<int> kinds = state_kinds(schedule);
    for (int e = 0; e < static_cast<int>(kinds.size()); ++e) {
        if (!sel.has(e)) continue;
        const int kind = kinds[e], width = kind == 0 ? c.hidden : c.v_hidden;
        const int64_t rows = sel.rows == 0 ? (kind == 0 ? rows_t : rows_v) : B;
        l.kind.push_back(kind);
        l.rows.push_back(static_cast<int32_t>(rows));
        l.width.push_back(width);
        l.offset.push_back(l.total);
        l.total += rows * width;
    }
    return l;
}
// Each selected entry's destination (dst + its offset) into meta, in the layout's state section (resized to hold it)
void put_state_dsts(MetaLayout& layout, std::vector<int>& meta, const StateLayout& l, float* dst) {
    layout.n_states = l.offset.size();
    meta.resize(layout.size(), 0);
    for (size_t e = 0; e < l.offset.size(); ++e) {
        const int64_t p = static_cast<int64_t>(reinterpret_cast<uintptr_t>(dst + l.offset[e]));
        memcpy(meta.data() + layout.state_dst(e), &p, sizeof(p));
    }
}
// A forward with VB200_OUT_LAYER_STATES needs the caller's buffer, 16-byte aligned: the state kernels write it with 16-byte stores.
void check_state_buffer(const char* api, const float* states) {
    if (states == nullptr) fail(VB200_ERR_INVALID, "%s: VB200_OUT_LAYER_STATES needs vb200_outputs.layer_states (NULL)", api);
    if (reinterpret_cast<uintptr_t>(states) & 15) fail(VB200_ERR_INVALID, "%s: vb200_outputs.layer_states is not 16-byte aligned", api);
}
// The layer states exist for the dense and packed device-pointer forwards only; every other entry point rejects their select bit.
void reject_layer_states(uint32_t select, const char* api) {
    if (select & VB200_OUT_LAYER_STATES)
        fail(VB200_ERR_INVALID, "%s: VB200_OUT_LAYER_STATES is only supported by vb200_forward, vb200_forward_slot, vb200_forward_regions, "
             "vb200_forward_packed and vb200_forward_regions_packed", api);
}

// Layout of the packed attention probabilities (VB200_OUT_ATTENTION_PACKED) from the two streams' row offsets [B + 1]: the selected
// entries in execution order (the order get_plan adds the probability ops in), each holding sample b's [heads, Lq_b, Lk_b] block at
// heads * prefix[b] (heads 1 under the head mean); prefix = sum over b' < b of T_b'^2 (text layers), V_b'^2 (image layers) or
// T_b' V_b' (both directions of a connection layer).  int64 throughout: at batch 512 with 256 rows per sample one call holds more than 2^31 floats.
struct PackedAttnLayout {
    std::vector<int32_t> heads, kind;
    std::vector<int64_t> offset;
    std::vector<int64_t> prefix;       // [3][B + 1]
    int64_t total = 0;
};
PackedAttnLayout packed_attn_layout(const Config& c, const std::vector<std::string>& schedule, const AttnSelect& sel, int B,
                                    const int* offs_t, const int* offs_v) {
    PackedAttnLayout l;
    const size_t n = static_cast<size_t>(B) + 1;
    l.prefix.assign(3 * n, 0);
    for (int b = 0; b < B; ++b) {
        const int64_t T = offs_t[b + 1] - offs_t[b], V = offs_v[b + 1] - offs_v[b];
        l.prefix[b + 1] = l.prefix[b] + T * T;
        l.prefix[n + b + 1] = l.prefix[n + b] + V * V;
        l.prefix[2 * n + b + 1] = l.prefix[2 * n + b] + T * V;
    }
    const std::vector<int> kinds = attention_kinds(schedule);
    for (int e = 0; e < static_cast<int>(kinds.size()); ++e) {
        if (!sel.has(e)) continue;
        const int kind = kinds[e], heads = sel.heads(kind == 0 ? c.heads : kind == 1 ? c.v_heads : c.bi_heads);
        l.heads.push_back(heads);
        l.kind.push_back(kind);
        l.offset.push_back(l.total);
        l.total += heads * l.prefix[(kind < 2 ? kind : 2) * n + B];
    }
    return l;
}
// The packed probability layout exists for the two packed forwards only; every other forward rejects its select bit.
void reject_packed_attention(uint32_t select, const char* api) {
    if (select & VB200_OUT_ATTENTION_PACKED)
        fail(VB200_ERR_INVALID, "%s: VB200_OUT_ATTENTION_PACKED is only supported by vb200_forward_packed and vb200_forward_regions_packed",
             api);
}

// Host lengths of one packed call.  Text lengths count tokens without the task token; a capacity (rows per item, 0: the call's
// longest) only sizes the plan.  A stream without lengths (the retrieval prefixes) is not part of the call: its offsets stay zero.
struct PackedLengths {
    const char* item;                                   // what one entry of the batch is called in messages
    int B;
    const int32_t* n_tokens; int max_tokens;
    const int32_t* n_regions; int max_regions;
    const int32_t* src_t = nullptr;                     // packed pair suffix: each pair's first row in the cached text states
    const int32_t* src_v = nullptr;                     //   and in the cached image states
};
// One packed call's rows: the plan's per-sample capacities and the d_meta contents (in `layout`) its kernels read.
struct PackedBatch {
    int Tin = 1, V = 1;              // plan capacities: T = Tin + task token and V rounded up to 16 rows; 1 for a stream not in the call
    MetaLayout layout;
    std::vector<int> meta;
    const int* offs_t() const { return meta.data() + layout.offs_t(); }
    const int* offs_v() const { return meta.data() + layout.offs_v(); }
    int rows_t() const { return meta[layout.rows_t()]; }
    int rows_v() const { return meta[layout.rows_v()]; }
};
// Validates a packed call's lengths and lays out its rows: offs[i + 1] = offs[i] + rows_i per stream (text: T_i = Tin_i + task
// token).  Rejects a batch < 1, a negative capacity, a length < 1 or above a non-zero capacity, more than max_rows rows per sample
// (the engine's max_rows_per_sample) and Tin_i > max_position_embeddings.  maps (non-null): where the plan's kernels write the packed
// attention probabilities of the entries `sel` selects, whose layout then joins the meta; states (non-null): the same for the layer
// states `ssel` selects.
PackedBatch pack_batch(const char* api, const Config& c, const std::vector<std::string>& schedule, const PackedLengths& in, float* maps,
                       int max_rows, const AttnSelect& sel = {}, float* states = nullptr, const StateSelect& ssel = {}) {
    if (in.B < 1) fail(VB200_ERR_INVALID, "%s: batch must be positive", api);
    if (in.max_tokens < 0) fail(VB200_ERR_INVALID, "%s: negative capacity max_tokens %d", api, in.max_tokens);
    if (in.max_regions < 0) fail(VB200_ERR_INVALID, "%s: negative capacity max_regions %d", api, in.max_regions);
    const int task = c.task_tokens ? 1 : 0;
    PackedBatch b;
    b.layout = MetaLayout{static_cast<size_t>(in.B), 0, in.src_t != nullptr};
    b.meta.assign(b.layout.size(), 0);
    auto pack = [&](bool text, const int32_t* len, int cap, size_t at) {      // one stream's offsets; returns its plan capacity
        const char* name = text ? "n_tokens" : "n_regions";
        const int extra = text ? task : 0;
        int* offs = b.meta.data() + at;
        int longest = 0;
        for (int i = 0; i < in.B; ++i) {
            const int l = len[i];
            if (l < 1) fail(VB200_ERR_INVALID, "%s: %s %d has %s %d (must be >= 1)", api, in.item, i, name, l);
            if (cap > 0 && l > cap) fail(VB200_ERR_INVALID, "%s: %s %d has %s %d, above the capacity %d", api, in.item, i, name, l, cap);
            if (l + extra > max_rows)
                fail(VB200_ERR_INVALID, "%s: %s %d too long for %s (%s=%d, max %d)", api, in.item, i, bound_name(max_rows),
                     text ? "T" : "V", l + extra, max_rows);
            if (text && l > c.max_pos)
                fail(VB200_ERR_INVALID, "%s: %s %d has n_tokens %d > max_position_embeddings %d", api, in.item, i, l, c.max_pos);
            offs[i + 1] = offs[i] + l + extra;
            longest = std::max(longest, l);
        }
        const int rows = (cap > 0 ? cap : longest) + extra;                     // rounded up to the attention kernels' 16-row buckets
        if (rows > max_rows)
            fail(VB200_ERR_INVALID, "%s: capacity above %d rows per sample (%s=%d)", api, max_rows, text ? "T" : "V", rows);
        return (rows + 15) / 16 * 16;
    };
    if (in.n_tokens) b.Tin = pack(true, in.n_tokens, in.max_tokens, b.layout.offs_t()) - task;
    if (in.n_regions) b.V = pack(false, in.n_regions, in.max_regions, b.layout.offs_v());
    if (b.layout.src) {
        std::copy(in.src_t, in.src_t + in.B, b.meta.begin() + b.layout.src_t());
        std::copy(in.src_v, in.src_v + in.B, b.meta.begin() + b.layout.src_v());
    }
    if (maps) {
        const PackedAttnLayout l = packed_attn_layout(c, schedule, sel, in.B, b.offs_t(), b.offs_v());
        const int64_t dst = static_cast<int64_t>(reinterpret_cast<uintptr_t>(maps));
        b.layout.n_entries = l.offset.size();
        b.meta.resize(b.layout.size(), 0);
        memcpy(b.meta.data() + b.layout.probs_dst(), &dst, sizeof(dst));
        memcpy(b.meta.data() + b.layout.probs_entry(0), l.offset.data(), l.offset.size() * sizeof(int64_t));
        memcpy(b.meta.data() + b.layout.probs_prefix(0), l.prefix.data(), l.prefix.size() * sizeof(int64_t));
    }
    if (states) put_state_dsts(b.layout, b.meta, state_layout(c, schedule, ssel, in.B, b.rows_t(), b.rows_v()), states);
    return b;
}
// Detector box counts of a packed region call -> regions per image, V_i = n_boxes_i + 1 (the boxes and the global mean row), and
// the region capacity (max_boxes + 1, or 0: the call's longest).  Checked in the caller's units before pack_batch sees V_i.
struct BoxRows { std::vector<int32_t> v; int max_regions; };
BoxRows box_rows(const char* api, int n, const int32_t* n_boxes, int max_boxes, int max_rows) {
    if (max_boxes < 0) fail(VB200_ERR_INVALID, "%s: negative capacity max_boxes %d", api, max_boxes);
    if (max_boxes > max_rows - 1)
        fail(VB200_ERR_INVALID, "%s: capacity max_boxes %d above %d (V = boxes + 1 <= %d)", api, max_boxes, max_rows - 1, max_rows);
    BoxRows r{{}, max_boxes > 0 ? max_boxes + 1 : 0};
    for (int i = 0; i < n; ++i) {
        const int k = n_boxes[i];
        if (k < 1) fail(VB200_ERR_INVALID, "%s: image %d has n_boxes %d (must be >= 1)", api, i, k);
        if (max_boxes > 0 && k > max_boxes)
            fail(VB200_ERR_INVALID, "%s: image %d has n_boxes %d, above the capacity max_boxes %d", api, i, k, max_boxes);
        if (k + 1 > max_rows) fail(VB200_ERR_INVALID, "%s: image %d has n_boxes %d (V = n_boxes + 1 must be <= %d)", api, i, k, max_rows);
        r.v.push_back(k + 1);
    }
    return r;
}

struct Plan {
    int B = 0, Tin = 0, T = 0, V = 0;
    Arena mem;
    // input-side buffers
    bf16* img_a = nullptr; int kp = 0;
    float *mask_t = nullptr, *mask_v = nullptr;
    float* t_f32[2]; bf16* t_b16[2];              // each stream's state: [0] between layers, [1] a layer's attention LayerNorm output
    float* v_f32[2]; bf16* v_b16[2];
    std::vector<Op> ops;
    OutBuf outs[kNumOuts];
    struct AttnOut { float* p; int heads, Lq, Lk; };   // attention probabilities [B, heads, Lq, Lk] in schedule order
    std::vector<AttnOut> attn;                         //   (T / V layers: one entry; connection layers: text->image, image->text)
    uint64_t last_use = 0;                             // plan-cache LRU stamp
    long long* timeline = nullptr;                     // profiling (set_option "timeline"): [GEMM op][kTimelineCtas][16] stamps of the LAST replay
    double flops = 0;
    Graph graph;
    GraphExec exec;
    // host-API staging (device copies of the inputs)
    int64_t *d_q = nullptr, *d_seg = nullptr, *d_mask = nullptr, *d_task = nullptr;
    float *d_feat = nullptr, *d_loc = nullptr;
    uint8_t* d_imask = nullptr;
    float* d_out[12] = {nullptr};
    // packed plans (the packed forwards and retrieval calls): d_meta in the format `layout` describes, filled per call through
    // `meta` (stage_meta), reserved at plan build so that a forward never allocates
    bool packed = false;
    MetaLayout layout;
    int* d_meta = nullptr;
    Staging meta;
    const int* offs_t() const { return d_meta + layout.offs_t(); }
    const int* offs_v() const { return d_meta + layout.offs_v(); }
    const int* rows_t() const { return d_meta + layout.rows_t(); }
    const int* rows_v() const { return d_meta + layout.rows_v(); }
    const int* src_t() const { return d_meta + layout.src_t(); }
    const int* src_v() const { return d_meta + layout.src_v(); }
    const int64_t* meta64(size_t at) const { return reinterpret_cast<const int64_t*>(d_meta + at); }
    // gated packed plans (vb200_forward_packed_gated): the head gate table [B, n_entries, max_heads] fp32, written per call ahead of
    // the plan's kernels; every attention launch reads its entry's column
    float* gate = nullptr;
    int gate_entries = 0, gate_heads = 0;
    vb::HeadGate gate_at(int e) const {
        if (gate == nullptr) return {};
        return vb::HeadGate{gate + static_cast<size_t>(e) * gate_heads, gate_entries * gate_heads, gate_heads};
    }
};

// One pre-training head at one bucket of M listed rows (vb200_pretraining_heads): the device row list (the call's count first, which
// bounds the GEMM, LayerNorm and rowdot rows), the gathered operand, the forward's launch list for that head built by PlanBuilder
// at M rows (TMA descriptors included) and its fp32 logits.  Built once per bucket and kept, apart from the forward plans:
// never captured, counted against max_plans or evicted.
enum { kHeadText = 0, kHeadImage = 1, kHeadPair = 2 };
constexpr int kMaxHeadRows = 1 << 20;   // rows per list of one call (the largest bucket's logits: 1M x 30522 fp32 = 125 GB is already
                                        // past any device; the bound keeps the bucket arithmetic in int)
struct RowHeads {
    Plan pl;                       // workspace (pl.mem) and launch list (pl.ops)
    int M = 0;
    int* d_rows = nullptr;         // [1 + 2M]: count, then the rows, then (vb200_pretraining_objectives) their labels
    void* a = nullptr;             // [M, width]: 16-bit operand (x3: hi | lo | hi) of the transform GEMM, fp32 pooled rows (pair head)
    OutBuf logits;                 // [M, N] fp32, row stride logits.ld
    float* loss = nullptr;         // [M]: each listed row's objective (vb200_pretraining_objectives)
};

}  // namespace

// =========================================================================================== engine
struct vb200_engine {
    Config cfg;
    vb200_options opt{};
    int num_labels = 0, gqa_labels = 0;
    // vb200_create_pretraining: the checkpoint holds the encoder and the `cls` heads only.  No task head is loaded, and asking for one
    // (a select bit, a decode family) is VB200_ERR_INVALID; num_labels and gqa_labels stay 0.
    bool pretraining = false;
    bool dry = false;          // audit pass: check names / shapes / dtypes only, touch no device
    int lone_rows = 320;       // VB200_LONE_ROWS (0 = off): forwards with at most this many rows in either stream (batch <= 8 at the default
                               // shapes) run their plain GEMMs with 64-wide tiles while those still fit one CTA per SM
    // vb200_set_option("max_rows_per_sample"), 256..1024: the longest text (T = Tin + task token) or image (V) sequence a call may
    // bring.  Validation only -- a plan's attention kernels follow from its shape (streaming above 256 rows), so no plan is dropped.
    int max_rows = 256;
    AttnSelect attn_sel;       // vb200_set_option("attention_entries" / "attention_heads"): the maps a forward with the map bit writes
    StateSelect state_sel;     // vb200_set_option("state_entries" / "state_rows"): the layer states a forward with the state bit writes
    bool x3 = false;           // fp32-parity mode (vb200_options::split_fp32): fp16 hi/lo split operands, K' = 3K GEMMs, fp32 attention
    // Programmatic dependent launch (opt.use_pdl): every kernel triggers its dependents once its main work is issued, and a
    // dependent GEMM's producer puts its first weight tiles in flight before griddepcontrol.wait.  On by default;
    // VB200_PDL=off|full, use_pdl < 0 = off.
    int gemm_kernel = 1;       // default_gemm_kernel(): 1 = plain GEMMs the ping-pong kernel supports run on it, 0 = all on the cooperative one
    Arena weights;
    std::string last_error;
    // embeddings
    float *word = nullptr, *pos = nullptr, *type = nullptr, *task = nullptr;
    bf16* word_b16 = nullptr;   // tied LM decoder operand
    LNW emb_ln, vemb_ln;
    LinearW img_emb;            // [v_hidden, v_feat + 64]: image_embeddings | image_location_embeddings | 0, bias = b_img + b_loc
    std::vector<LayerW> t_layers, v_layers;
    std::vector<ConnW> c_layers;
    LinearW t_pool, v_pool;
    ClsW vqa, gqa, binary;
    RowW vil_logit, vil_tri, vision_logit, ling_logit, seq_rel;
    // pre-training heads
    LinearW lm_transform, img_transform, img_decoder, lm_decoder;
    LNW lm_ln, img_ln;
    float* lm_bias = nullptr;
    std::map<std::string, HostTensor> sd;
    std::map<std::vector<int64_t>, std::unique_ptr<Plan>> plans;
    bool timeline = false;          // vb200_set_option("timeline", 1): plans built from now on record per-CTA stamps (vb200_timeline)
    int profile_grid_pct = 0;       // vb200_set_option("profile_grid_pct"): persistent-grid override for vb200_profile_ops only
    uint64_t use_clock = 0;         // LRU clock of the plan cache
    size_t max_plans = 24;          // VB200_MAX_PLANS: least-recently-used plans beyond this are destroyed (workspace + graph)
    std::vector<std::string> schedule;
    // pre-training heads at chosen rows (vb200_pretraining_heads): per head (kHeadText / kHeadImage / kHeadPair) the RowHeads of every
    // bucket seen so far
    std::map<int, std::unique_ptr<RowHeads>> row_heads[3];
    // Members are destroyed in reverse order: the owners below go before the plans and RowHeads above, and each Staging waits for
    // its copies before the workspaces they fill are freed.
    // The calls beside the forward: answer decode's descriptors (pretraining_heads' top-k ones too) and vb200_decode_answers_host's
    // device answers, attention relevance's entry and sample descriptors, region selection's descriptors and workspace (device
    // descriptors, row stats, boxes, bitmasks, max_conf, keep lists), and pre-training's row lists, staged into the RowHeads' d_rows.
    // The RowHeads never grow, so pre_done alone orders those calls, as a Workspace's `done` does.  Answer and message ablation:
    // the sample and segment descriptors (staged through abl_in) and the samples' text ids.
    Workspace dec_ws, ans_ws, rel_ws, sel_ws, abl_ws;
    Staging dec_in, rel_in, sel_in, pre_in, abl_in;
    Event pre_done;
    Stream side_stream;
    Event ev_fork, ev_join;

    // ---------------------------------------------------------------- checkpoint ingestion
    HostTensor& need(const std::string& name, int ndim, int64_t d0, int64_t d1 = 0) {
        auto it = sd.find(name);
        if (it == sd.end()) fail(VB200_ERR_CHECKPOINT, "checkpoint is missing key \"%s\"", name.c_str());
        HostTensor& t = it->second;
        if (t.ndim != ndim || t.shape[0] != d0 || (ndim == 2 && t.shape[1] != d1))
            fail(VB200_ERR_CHECKPOINT, "checkpoint key \"%s\" has shape [%lld,%lld] (ndim %d), expected [%lld,%lld] (ndim %d)",
                 name.c_str(), (long long)t.shape[0], (long long)t.shape[1], t.ndim, (long long)d0, (long long)d1, ndim);
        t.used = true;
        return t;
    }
    float* upload_f32(const std::vector<float>& h) {
        if (dry) return nullptr;
        float* d = weights.alloc_n<float>(h.size());
        CUDA_CHECK(cudaMemcpy(d, h.data(), h.size() * 4, cudaMemcpyHostToDevice));
        return d;
    }
    float* load_vec(const std::string& name, int64_t n) {
        HostTensor& t = need(name, 1, n);
        if (dry) return nullptr;
        std::vector<float> h(n);
        for (int64_t i = 0; i < n; ++i) h[i] = t.at(i);
        return upload_f32(h);
    }
    float* load_mat_f32(const std::string& name, int64_t r, int64_t c) {
        HostTensor& t = need(name, 2, r, c);
        if (dry) return nullptr;
        std::vector<float> h(r * c);
        if (t.dtype == VB200_F32) memcpy(h.data(), t.data, h.size() * 4);
        else for (int64_t i = 0; i < r * c; ++i) h[i] = t.at(i);
        return upload_f32(h);
    }
    LNW load_ln(const std::string& prefix, int n) {
        LNW l; l.n = n;
        l.g = load_vec(prefix + ".weight", n);
        l.b = load_vec(prefix + ".bias", n);
        return l;
    }
    // one or several nn.Linear stacked along N (fused QKV), optional extra K columns from a second weight
    LinearW load_linear(const std::vector<std::string>& prefixes, int64_t n_each, int64_t k,
                        const std::string& extra_k_prefix = "", int64_t extra_k = 0) {
        LinearW L;
        L.N = static_cast<int>(n_each * prefixes.size());
        L.K = static_cast<int>(k + (extra_k ? 64 : 0));
        L.ldw = (L.K + 63) / 64 * 64;
        if (dry) {
            for (const std::string& p : prefixes) { need(p + ".weight", 2, n_each, k); need(p + ".bias", 1, n_each); }
            if (extra_k) { need(extra_k_prefix + ".weight", 2, n_each, extra_k); need(extra_k_prefix + ".bias", 1, n_each); }
            return L;
        }
        const bool f16 = opt.act_fp16 != 0;     // weights are stored in the same 16-bit format as the activations
        if (x3) { load_linear_split(L, prefixes, n_each, k, extra_k_prefix, extra_k); return L; }
        std::vector<uint16_t> h(static_cast<size_t>(L.N) * L.ldw, 0);
        std::vector<float> hb(L.N, 0.0f);
        for (size_t pi = 0; pi < prefixes.size(); ++pi) {
            HostTensor& w = need(prefixes[pi] + ".weight", 2, n_each, k);
            HostTensor& b = need(prefixes[pi] + ".bias", 1, n_each);
            for (int64_t n = 0; n < n_each; ++n) {
                uint16_t* dst = &h[(pi * n_each + n) * L.ldw];
                if (w.dtype == VB200_F32) {
                    const float* src = static_cast<const float*>(w.data) + n * k;
                    if (f16) for (int64_t j = 0; j < k; ++j) dst[j] = f32_to_f16_bits(src[j]);
                    else for (int64_t j = 0; j < k; ++j) dst[j] = f32_to_bf16_bits(src[j]);
                } else {
                    for (int64_t j = 0; j < k; ++j) dst[j] = cvt16(w.at(n * k + j));
                }
                hb[pi * n_each + n] = b.at(n);
            }
        }
        if (extra_k) {
            HostTensor& w = need(extra_k_prefix + ".weight", 2, n_each, extra_k);
            HostTensor& b = need(extra_k_prefix + ".bias", 1, n_each);
            for (int64_t n = 0; n < n_each; ++n) {
                for (int64_t j = 0; j < extra_k; ++j) h[n * L.ldw + k + j] = cvt16(w.at(n * extra_k + j));
                hb[n] += b.at(n);
            }
        }
        L.w = weights.alloc_n<bf16>(h.size());
        CUDA_CHECK(cudaMemcpy(L.w, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
        L.bias = upload_f32(hb);
        return L;
    }
    uint16_t cvt16(float f) const { return opt.act_fp16 ? f32_to_f16_bits(f) : f32_to_bf16_bits(f); }
    // fp32-parity mode: every weight is stored as fp16 hi | hi | lo per 64 columns of K (activations are hi | lo | hi), so the
    // K' = 3K GEMM adds hi.hi + lo.hi + hi.lo; physical row stride 3 * ldw.
    static void put_split_w(uint16_t* row, int64_t j, float w) {
        const uint16_t hi = f32_to_f16_bits(w);
        const uint16_t lo = f32_to_f16_bits(w - half_bits_to_f32(hi));
        uint16_t* d = row + (j >> 6) * 192 + (j & 63);
        d[0] = hi; d[64] = hi; d[128] = lo;
    }
    void load_linear_split(LinearW& L, const std::vector<std::string>& prefixes, int64_t n_each, int64_t k,
                           const std::string& extra_k_prefix, int64_t extra_k) {
        std::vector<uint16_t> h(static_cast<size_t>(L.N) * L.ldw * 3, 0);
        std::vector<float> hb(L.N, 0.0f);
        for (size_t pi = 0; pi < prefixes.size(); ++pi) {
            HostTensor& w = need(prefixes[pi] + ".weight", 2, n_each, k);
            HostTensor& b = need(prefixes[pi] + ".bias", 1, n_each);
            for (int64_t n = 0; n < n_each; ++n) {
                uint16_t* dst = &h[(pi * n_each + n) * L.ldw * 3];
                for (int64_t j = 0; j < k; ++j) put_split_w(dst, j, w.at(n * k + j));
                hb[pi * n_each + n] = b.at(n);
            }
        }
        if (extra_k) {
            HostTensor& w = need(extra_k_prefix + ".weight", 2, n_each, extra_k);
            HostTensor& b = need(extra_k_prefix + ".bias", 1, n_each);
            for (int64_t n = 0; n < n_each; ++n) {
                for (int64_t j = 0; j < extra_k; ++j) put_split_w(&h[n * L.ldw * 3], k + j, w.at(n * extra_k + j));
                hb[n] += b.at(n);
            }
        }
        L.w = weights.alloc_n<bf16>(h.size());
        CUDA_CHECK(cudaMemcpy(L.w, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
        L.bias = upload_f32(hb);
    }
    LinearW load_linear1(const std::string& prefix, int64_t n, int64_t k) { return load_linear({prefix}, n, k); }
    RowW load_row(const std::string& prefix, int n_out, int k) {
        RowW r; r.n_out = n_out; r.K = k;
        r.w = load_mat_f32(prefix + ".weight", n_out, k);
        r.b = load_vec(prefix + ".bias", n_out);
        return r;
    }
    LayerW load_layer(const std::string& p, int hid, int inter) {
        LayerW L;
        L.ln1 = load_ln(p + ".attention.output.LayerNorm", hid);
        L.ln2 = load_ln(p + ".output.LayerNorm", hid);
        L.qkv = load_linear({p + ".attention.self.query", p + ".attention.self.key", p + ".attention.self.value"}, hid, hid);
        L.attn_out = load_linear1(p + ".attention.output.dense", hid, hid);
        L.inter = load_linear1(p + ".intermediate.dense", inter, hid);
        L.out = load_linear1(p + ".output.dense", hid, inter);
        return L;
    }
    ClsW load_cls(const std::string& p, int in_dim, int hid, int out_dim, bool narrow) {
        ClsW c;
        c.fc0 = load_linear1(p + ".logit_fc.0", hid, in_dim);
        c.ln = load_ln(p + ".logit_fc.2", hid);
        if (narrow) c.fc3_row = load_row(p + ".logit_fc.3", out_dim, hid);
        else c.fc3 = load_linear1(p + ".logit_fc.3", out_dim, hid);
        return c;
    }

    void ingest(int64_t n_tensors, const vb200_tensor* tensors) {
        for (int64_t i = 0; i < n_tensors; ++i) {
            const vb200_tensor& t = tensors[i];
            if (t.name == nullptr || t.data == nullptr) fail(VB200_ERR_CHECKPOINT, "state_dict entry %lld has a NULL name or data pointer", (long long)i);
            if (t.ndim < 1 || t.ndim > 2 || t.dtype < 0 || t.dtype > 2)
                fail(VB200_ERR_CHECKPOINT, "state_dict entry \"%s\": unsupported ndim %d / dtype %d", t.name, t.ndim, t.dtype);
            std::string name = t.name;
            if (name.rfind("module.", 0) == 0) name = name.substr(7);          // DataParallel prefix
            // old checkpoints: LayerNorm gamma/beta -> weight/bias
            auto ends = [&](const char* s) { size_t n = strlen(s); return name.size() >= n && name.compare(name.size() - n, n, s) == 0; };
            if (ends(".gamma")) name = name.substr(0, name.size() - 6) + ".weight";
            else if (ends(".beta")) name = name.substr(0, name.size() - 5) + ".bias";
            HostTensor h; h.dtype = t.dtype; h.ndim = t.ndim; h.shape[0] = t.shape[0]; h.shape[1] = t.ndim == 2 ? t.shape[1] : 0; h.data = t.data;
            sd[name] = h;
        }
        const Config& c = cfg;
        // vil_prediction width comes from the checkpoint unless the caller pins it (worker.py:523 passes 3129)
        if (!pretraining) {
            auto it = sd.find("vil_prediction.logit_fc.3.weight");
            if (it == sd.end()) fail(VB200_ERR_CHECKPOINT, "checkpoint is missing key \"vil_prediction.logit_fc.3.weight\"");
            const int ck = static_cast<int>(it->second.shape[0]);
            if (opt.num_labels > 0 && opt.num_labels != ck)
                fail(VB200_ERR_CHECKPOINT, "num_labels=%d but the checkpoint's vil_prediction head has %d outputs", opt.num_labels, ck);
            num_labels = ck;
            auto ig = sd.find("vil_prediction_gqa.logit_fc.3.weight");
            if (ig == sd.end()) fail(VB200_ERR_CHECKPOINT, "checkpoint is missing key \"vil_prediction_gqa.logit_fc.3.weight\"");
            gqa_labels = static_cast<int>(ig->second.shape[0]);
        }
        word = load_mat_f32("bert.embeddings.word_embeddings.weight", c.vocab, c.hidden);
        pos = load_mat_f32("bert.embeddings.position_embeddings.weight", c.max_pos, c.hidden);
        type = load_mat_f32("bert.embeddings.token_type_embeddings.weight", c.type_vocab, c.hidden);
        if (c.task_tokens) task = load_mat_f32("bert.embeddings.task_embeddings.weight", c.n_task, c.hidden);
        emb_ln = load_ln("bert.embeddings.LayerNorm", c.hidden);
        img_emb = load_linear({"bert.v_embeddings.image_embeddings"}, c.v_hidden, c.v_feat,
                              "bert.v_embeddings.image_location_embeddings", 5);
        vemb_ln = load_ln("bert.v_embeddings.LayerNorm", c.v_hidden);
        // [UPSTREAM] BertEncoder.forward schedule
        {
            int v_start = 0, t_start = 0;
            for (size_t i = 0; i < c.v_bi_id.size(); ++i) {
                const int v_end = c.v_bi_id[i], t_end = c.t_bi_id[i];
                for (int k = t_start; k < t_end; ++k) schedule.push_back("T" + std::to_string(k));
                for (int k = v_start; k < v_end; ++k) schedule.push_back("V" + std::to_string(k));
                schedule.push_back("C" + std::to_string(i));
                v_start = v_end; t_start = t_end;
            }
            for (int k = v_start; k < c.v_layers; ++k) schedule.push_back("V" + std::to_string(k));
            for (int k = t_start; k < c.layers; ++k) schedule.push_back("T" + std::to_string(k));
        }
        for (int i = 0; i < c.layers; ++i)
            t_layers.push_back(load_layer("bert.encoder.layer." + std::to_string(i), c.hidden, c.inter));
        for (int i = 0; i < c.v_layers; ++i)
            v_layers.push_back(load_layer("bert.encoder.v_layer." + std::to_string(i), c.v_hidden, c.v_inter));
        for (size_t i = 0; i < c.v_bi_id.size(); ++i) {
            const std::string p = "bert.encoder.c_layer." + std::to_string(i);
            ConnW w;
            w.ln1 = load_ln(p + ".biOutput.LayerNorm1", c.v_hidden);
            w.ln2 = load_ln(p + ".biOutput.LayerNorm2", c.hidden);
            w.v_ln = load_ln(p + ".v_output.LayerNorm", c.v_hidden);
            w.t_ln = load_ln(p + ".t_output.LayerNorm", c.hidden);
            w.qkv_img = load_linear({p + ".biattention.query1", p + ".biattention.key1", p + ".biattention.value1"}, c.bi_hidden, c.v_hidden);
            w.qkv_txt = load_linear({p + ".biattention.query2", p + ".biattention.key2", p + ".biattention.value2"}, c.bi_hidden, c.hidden);
            w.dense1 = load_linear1(p + ".biOutput.dense1", c.v_hidden, c.bi_hidden);
            w.dense2 = load_linear1(p + ".biOutput.dense2", c.hidden, c.bi_hidden);
            w.v_inter = load_linear1(p + ".v_intermediate.dense", c.v_inter, c.v_hidden);
            w.v_out = load_linear1(p + ".v_output.dense", c.v_hidden, c.v_inter);
            w.t_inter = load_linear1(p + ".t_intermediate.dense", c.inter, c.hidden);
            w.t_out = load_linear1(p + ".t_output.dense", c.hidden, c.inter);
            c_layers.push_back(w);
            // [UPSTREAM] present in the checkpoint, never applied in forward
            for (const char* u : {".biOutput.q_dense1.weight", ".biOutput.q_dense1.bias", ".biOutput.q_dense2.weight", ".biOutput.q_dense2.bias"}) {
                auto it = sd.find(p + u);
                if (it != sd.end()) it->second.used = true;
            }
        }
        t_pool = load_linear1("bert.t_pooler.dense", c.bi_hidden, c.hidden);
        v_pool = load_linear1("bert.v_pooler.dense", c.bi_hidden, c.v_hidden);
        if (!pretraining) {   // task heads; on a pre-training engine their keys are unexpected ones (strict) like any other
            vqa = load_cls("vil_prediction", c.bi_hidden, 2 * c.bi_hidden, num_labels, false);
            gqa = load_cls("vil_prediction_gqa", c.bi_hidden, 2 * c.bi_hidden, gqa_labels, false);
            binary = load_cls("vil_binary_prediction", 2 * c.bi_hidden, 2 * c.bi_hidden, 2, true);
            vil_logit = load_row("vil_logit", 1, c.bi_hidden);
            vil_tri = load_row("vil_tri_prediction", 3, c.bi_hidden);
            vision_logit = load_row("vision_logit", 1, c.v_hidden);
            ling_logit = load_row("linguisic_logit", 1, c.hidden);
        }
        seq_rel = load_row("cls.bi_seq_relationship", 2, c.bi_hidden);
        lm_transform = load_linear1("cls.predictions.transform.dense", c.hidden, c.hidden);
        lm_ln = load_ln("cls.predictions.transform.LayerNorm", c.hidden);
        lm_bias = load_vec("cls.predictions.bias", c.vocab);
        img_transform = load_linear1("cls.imagePredictions.transform.dense", c.v_hidden, c.v_hidden);
        img_ln = load_ln("cls.imagePredictions.transform.LayerNorm", c.v_hidden);
        img_decoder = load_linear1("cls.imagePredictions.decoder", c.v_target, c.v_hidden);
        {   // tied LM decoder: bf16 copy of the word-embedding table as a [vocab, hidden] GEMM operand
            HostTensor& w = need("bert.embeddings.word_embeddings.weight", 2, c.vocab, c.hidden);
            if (!dry) {
                std::vector<uint16_t> h(static_cast<size_t>(c.vocab) * c.hidden * (x3 ? 3 : 1));
                if (x3) {
                    for (int64_t n = 0; n < c.vocab; ++n)
                        for (int64_t j = 0; j < c.hidden; ++j) put_split_w(&h[static_cast<size_t>(n) * c.hidden * 3], j, w.at(n * c.hidden + j));
                } else {
                    for (size_t i = 0; i < h.size(); ++i) h[i] = cvt16(w.at(i));
                }
                word_b16 = weights.alloc_n<bf16>(h.size());
                CUDA_CHECK(cudaMemcpy(word_b16, h.data(), h.size() * 2, cudaMemcpyHostToDevice));
            }
            lm_decoder.w = word_b16; lm_decoder.bias = lm_bias; lm_decoder.N = c.vocab; lm_decoder.K = c.hidden; lm_decoder.ldw = c.hidden;
            auto it = sd.find("cls.predictions.decoder.weight");   // tied duplicate of the word table
            if (it != sd.end()) it->second.used = true;
            auto ip = sd.find("bert.embeddings.position_ids");
            if (ip != sd.end()) ip->second.used = true;
        }
        if (opt.strict) {
            std::string extra;
            int n = 0;
            for (auto& kv : sd) if (!kv.second.used) { if (n++ < 8) extra += " \"" + kv.first + "\""; }
            if (n) fail(VB200_ERR_CHECKPOINT, "checkpoint has %d unexpected key(s):%s%s", n, extra.c_str(), n > 8 ? " ..." : "");
        }
        sd.clear();   // host pointers are the caller's; do not keep them
    }

    // ---------------------------------------------------------------- plan construction
    // One ViLBERT stream of a forward plan under construction: every layer kind and the heads read the stream's facts from here.
    struct StreamRec {
        float** f32; bf16** b16;            // the plan's t_f32 / t_b16 or v_f32 / v_b16
        int hid, seq, rows;                 // width, rows per sample (a packed plan's capacity), B x seq
        int branch, prefix;                 // graph branch of its layers; prefix sums of its packed self-attention maps (0 T^2, 1 V^2)
        const float* mask;
        uint8_t* qkv; bf16* ctx; bf16* inter;   // scratch: Q | K | V projections, attention context, FFN intermediate
        const int* m_rows; const int* offs;     // packed plans: device row count and per-sample row offsets
        bf16* tail;                         // pruned tail: its last layer's compact 16-bit output [B, hid], each sample's first row
    };
    // One nn.Linear's arguments (PlanBuilder::linear): the weight and the operand [rows, w.K] at row stride lda are fixed, the rest
    // named.  All sizes are LOGICAL (elements of the mathematical matrices).  Over a stream: every row of it, on its branch.
    struct LinearArgs {
        const LinearW& w; const bf16* a; int64_t lda, rows;
        int act = vb::kActNone;
        bf16* out16 = nullptr; int ld16 = 0;
        float* out32 = nullptr; int ld32 = 0;
        const LNW* ln = nullptr; const float* res = nullptr; int ld_res = 0;   // LayerNorm(GEMM + res): the row kernel writes the outputs
        const float* mul = nullptr; int ld_mul = 0;                           // epilogue product operand (the pooled product)
        const int* m_rows = nullptr;                                          // packed plans: device count of the rows computed
        int branch = 0;                                                       // graph branch: 0 main, 1 side (image)
        Op::Sync sync = Op::NONE;
        LinearArgs(const LinearW& w_, const bf16* a_, int64_t lda_, int64_t rows_) : w(w_), a(a_), lda(lda_), rows(rows_) {}
        LinearArgs(const StreamRec& s, const LinearW& w_, const bf16* a_, int64_t lda_)
            : w(w_), a(a_), lda(lda_), rows(s.rows), m_rows(s.m_rows), branch(s.branch) {}
    };
    // Builds one launch list into `pl` (get_plan, row_heads_for) and holds what only construction needs.  Every op it adds takes the
    // current tag: the NVTX range name, also named by a failed GEMM launch's message.
    struct PlanBuilder {
        vb200_engine& eng;
        Plan& pl;
        int lone_m;                         // the rows the lone-rows tile rule compares: a forward's larger stream, a RowHeads bucket
        const char* tag;
        float* y[2] = {nullptr, nullptr};   // per-branch fp32 GEMM output feeding the row LayerNorm kernel
        StreamRec t{}, v{};
        bool maps = false;                  // the forward writes the attention maps attn_sel selects
        int entry = 0;                      // the current schedule step's first attention-map entry in the full list
        int n_probs = 0;                    // packed attention-probability ops added so far (their entry index)
        bool states = false;                // the forward writes the layer states state_sel selects

        // Physical width factor of the 16-bit operand buffers: in fp32-parity mode (x3) each is 3x as wide (fp16 hi | lo | hi per 64
        // columns).  buf16 sizes them, linear and gather scale their strides and K; nothing else applies it.
        int S() const { return eng.x3 ? 3 : 1; }
        bf16* buf16(size_t rows, size_t width) { return pl.mem.alloc_n<bf16>(rows * width * S()); }
        float* buf32(size_t rows, size_t width) { return pl.mem.alloc_n<float>(rows * width); }
        void push(Op op) { op.tag = tag; pl.ops.push_back(op); }
        OutBuf make_out(int rows, int cols) { const int ld = (cols + 3) / 4 * 4; return OutBuf{buf32(rows, ld), rows, cols, ld}; }
        // output slot `slot` of a forward, `cols` wide, at the rows kOutSlots gives it
        const OutBuf& out(int slot, int cols) {
            const int B = pl.B, r = kOutSlots[slot].rows;
            const int rows = r == kPerSample ? B : r == kPerPair ? (B % 2 == 0 ? B / 2 : B) : r == kTextRow ? t.rows : v.rows;
            return pl.outs[slot] = make_out(rows, cols);
        }

        // One nn.Linear (+ activation, + residual LayerNorm) -> one or two launch-list entries on a.branch: the GEMM (+bias,
        // +activation), and with a.ln it writes fp32 to the branch's scratch and the row LayerNorm kernel (adds the residual) follows.
        void linear(const LinearArgs& a) {
            const LinearW& W = a.w;
            const int S = this->S();
            GemmEpilogue e{};
            e.M = static_cast<int>(a.rows); e.N = W.N; e.K = W.ldw * S;
            e.bias = W.bias; e.mul = a.mul; e.ld_mul = a.ld_mul; e.act = eng.x3 && a.act == vb::kActGelu ? vb::kActGeluExact : a.act;
            e.pdl = eng.opt.use_pdl ? 5 : 0;
            e.a_f16 = eng.opt.act_fp16; e.out_f16 = eng.opt.act_fp16;
            e.m_rows = a.m_rows;
            e.split_acc = eng.x3 ? 1 : 0;
            if (a.ln) {
                e.out_f32 = y[a.branch]; e.ld_f32 = W.N;
            } else {
                e.out_bf16 = a.out16; e.ld_bf16 = a.ld16 * S; e.out_f32 = a.out32; e.ld_f32 = a.ld32;
                e.split16 = (eng.x3 && a.out16 != nullptr) ? 1 : 0;
                if (e.split16 && (W.N & 63)) fail(VB200_ERR_INVALID, "fp32-parity mode: 16-bit GEMM output of width %d is not a multiple of 64", W.N);
            }
            // Small forwards (<= lone_rows rows in either stream, batch <= 8): 64-wide tiles while they still fit one CTA per SM -- twice
            // the CTAs, half the epilogue each.  The tile width never changes an element's accumulation order.  RowHeads plans compare
            // their bucket M.
            int block_n = eng.x3 ? 64 : vb::gemm_p_pick_block_n(W.N);      // the fp32-parity kernel runs 64-wide tiles only
            if (eng.lone_rows > 0 && !eng.x3 && block_n == 128 && W.N % 64 == 0 && lone_m <= eng.lone_rows &&
                ((a.rows + 127) / 128) * (W.N / 64) <= vb::num_sms_host())
                block_n = 64;
            // Ping-pong kernel: each consumer warpgroup's epilogue runs under the other's mainloop.  It takes every plain GEMM it
            // supports (not the fp32-parity, pooled-product or ragged-N ones) whose outputs the TMA can store.
            // It takes the tile width chosen above, 128 even where that leaves one tile per CTA: 64-wide ping-pong tiles measured slower on H100 SXM
            // (700 W, bf16, 16-bit output, scripts/kernel_bench.py) at 1984x768x768 (9.74 vs 8.20 us), 1984x768x3072 (29.19 vs 20.32) and
            // 2304x1024x1024 (16.71 vs 15.88), and only 4 % faster with GELU at 2304x1024x1024 (18.04 vs 18.81).  The single-panel
            // launches of a batch-64 forward (poolers, fc0, the pruned tails) keep 128 too: 64-wide was slower at 64x768x768 (8.71 vs
            // 8.45 / 8.41 us, two 128-wide runs), 64x3072x768 GELU (9.54 vs 9.13 / 9.07), 64x1024x1024 (10.18 vs 10.04 / 9.97; GELU 10.40
            // vs 10.21 / 10.10), 64x1024x768 ReLU (8.53 vs 8.08 / 8.05) and 64x2048x1024 GELU (10.57 vs 10.47 / 10.42), and 2 % faster
            // only at 64x768x3072 (20.74 vs 21.23 / 21.12); same card, bf16.
            const GemmCall g = make_gemm(a.a, a.lda * S, W.w, static_cast<int64_t>(W.ldw) * S, e, {block_n, eng.x3 ? 0 : eng.gemm_kernel});
            push({g, a.branch, 2.0 * a.rows * W.N * W.K, a.sync});
            if (a.ln) {
                LayerNormArgs l{};
                l.y = y[a.branch]; l.ld_y = W.N; l.res = a.res; l.ld_res = a.ld_res; l.gamma = a.ln->g; l.beta = a.ln->b;
                l.out_f32 = a.out32; l.ld_f32 = a.out32 ? a.ld32 : 0; l.out16 = a.out16; l.ld16 = a.out16 ? a.ld16 * S : 0;
                l.M = static_cast<int>(a.rows); l.N = W.N; l.m_rows = a.m_rows;
                push({l, a.branch});
            }
        }
        // Row offs[b] of stream s's src16 (and src32) -> row b of the compact [B, hid] dst16 (and dst32): each sample's first row.
        void gather(const StreamRec& s, int branch, Op::Sync sync, const bf16* src16, bf16* dst16, const float* src32 = nullptr,
                    float* dst32 = nullptr) {
            GatherArgs g{};
            g.offs = s.offs; g.n_src = s.rows; g.B = pl.B; g.src16 = src16; g.dst16 = dst16; g.ld16 = s.hid * S();
            g.src_f32 = src32; g.dst_f32 = dst32; g.hidden = src32 ? s.hid : 0;
            push({g, branch, 0.0, sync});
        }
        void rowdot(const float* x, int ld_x, const RowW& w, const float* add, const OutBuf& o, const int* m_rows = nullptr) {
            push({RowdotArgs{x, w.w, w.b, add, o.p, ld_x, o.ld, o.rows, w.K, w.n_out, m_rows}, 0, 2.0 * o.rows * w.K * w.n_out});
        }
        // Q | K | V of stream s (w: 3 x its attention width): 16-bit for the tensor-core attention kernels, fp32 in fp32-parity mode
        void qkv(const StreamRec& s, const LinearW& w) {
            LinearArgs g(s, w, s.b16[0], s.hid);
            g.out16 = eng.x3 ? nullptr : reinterpret_cast<bf16*>(s.qkv); g.ld16 = w.N;
            g.out32 = eng.x3 ? reinterpret_cast<float*>(s.qkv) : nullptr; g.ld32 = w.N;
            linear(g);
        }
        // softmax(Q K^T / sqrt(d) + mask) V of stream q's queries over stream kv's keys and values (Q | K | V projections hid wide).
        // A self-attention (q == kv) runs on its stream's branch, both directions of a connection layer on the main one.  Default:
        // the tensor-core kernel writes the context (callers push that op themselves); this adds the fp32 kernel -- as THE attention
        // in fp32-parity mode (context out as hi | lo | hi; `sync` is that launch's), and/or as the producer of the attention-probability
        // output.  Packed plans: the probabilities of every sample at its own lengths straight into the caller's buffer, at the entry's
        // offset and the sample's prefix sum (0 T^2, 1 V^2, 2 T V) of the plan's probability meta.  The entry is written when it is
        // selected (attn_sel); under the head mean its maps come from a maps-only head-mean launch, after the fp32-parity mode's context
        // launch.  Adds nothing outside fp32-parity mode for an entry that is not selected.
        void attention_f32(const StreamRec& q, const StreamRec& kv, int hid, int heads, int entry, Op::Sync sync = Op::NONE) {
            const bool self = &q == &kv, want_probs = maps && eng.attn_sel.has(entry), mean = want_probs && eng.attn_sel.mean;
            const int branch = self ? q.branch : 0;
            const size_t qe = eng.x3 ? 4 : 2;
            AttnF32Args a{};
            a.q = q.qkv; a.k = kv.qkv + hid * qe; a.v = kv.qkv + 2 * hid * qe; a.ld_q = 3 * hid; a.ld_kv = 3 * hid; a.mask = kv.mask;
            a.Lq = q.seq; a.Lk = kv.seq;
            a.in_kind = eng.x3 ? 0 : (eng.opt.act_fp16 ? 1 : 2);
            a.B = pl.B; a.heads = heads; a.head_dim = hid / heads;
            if (eng.x3) {
                AttnF32Args c = a;
                c.ctx = q.ctx; c.ctx_mode = 3; c.ld_ctx = 3 * hid;
                if (want_probs && !mean) c.probs = attn_out(heads, a.Lq, a.Lk);
                push({c, branch, 4.0 * pl.B * heads * a.Lq * a.Lk * (hid / heads), sync});
            }
            if (!want_probs || (eng.x3 && !mean)) return;
            a.mean = mean;
            if (pl.packed) {
                const MetaLayout& m = pl.layout;
                a.packed = true;
                a.pk = vb::PackedProbs{q.offs, kv.offs, pl.meta64(m.probs_dst()), pl.meta64(m.probs_entry(n_probs)),
                                       pl.meta64(m.probs_prefix(self ? q.prefix : 2)), pl.gate_at(entry)};
                ++n_probs;
            } else {
                a.probs = attn_out(mean ? 1 : heads, a.Lq, a.Lk);
            }
            push({a, branch, 0.0});
        }
        // Layer-state entry e of the full list (state_kinds), stream s's fp32 state, when the forward writes it and state_sel selects
        // it: one launch on s's branch, added right after the op that wrote the state, so the stream's next layer cannot overwrite it
        // first.  Its destination is the entry's pointer in the plan's staged meta.
        void state(const StreamRec& s, int e) {
            if (!states || !eng.state_sel.has(e)) return;
            const vb::StateArgs a{s.f32[0], s.offs, s.m_rows, pl.packed ? nullptr : s.mask,
                                  pl.meta64(pl.layout.state_dst(eng.state_sel.index(e))), pl.B, s.seq, s.hid, eng.state_sel.rows};
            push({a, s.branch, 0.0});
        }
        // a dense plan's next attention-probability output [B, heads, Lq, Lk]
        float* attn_out(int heads, int Lq, int Lk) {
            float* p = pl.mem.alloc_n<float>(static_cast<size_t>(pl.B) * heads * Lq * Lk);
            pl.attn.push_back(Plan::AttnOut{p, heads, Lq, Lk});
            return p;
        }
        // A layer's row-local half on stream s: the attention output (ctx, ctx_w wide) + LayerNorm with the layer input -> [1], the
        // FFN and its LayerNorm with that output -> [0].  `sync` is the first GEMM's.
        void row_local(StreamRec& s, int ctx_w, const LinearW& wo, const LNW& ln1, const LinearW& wi, const LinearW& wf, const LNW& ln2,
                       Op::Sync sync) {
            auto ln_linear = [&](const bf16* a, int64_t lda, const LinearW& w, const LNW& ln, int from, int to, Op::Sync sy) {
                LinearArgs g(s, w, a, lda);
                g.ln = &ln; g.res = s.f32[from]; g.ld_res = s.hid; g.sync = sy;
                g.out16 = s.b16[to]; g.ld16 = s.hid; g.out32 = s.f32[to]; g.ld32 = s.hid;
                linear(g);
            };
            ln_linear(s.ctx, ctx_w, wo, ln1, 0, 1, sync);
            LinearArgs g(s, wi, s.b16[1], s.hid);
            g.act = vb::kActGelu; g.out16 = s.inter; g.ld16 = wi.N;
            linear(g);
            ln_linear(s.inter, wi.N, wf, ln2, 1, 0, Op::NONE);
        }
        // One BertLayer / BertImageLayer.  `tail` (the pruned tail): Q, K, V and the attention on every row (each is a key and a
        // value), the rest on each sample's first row -- read at stride seq rows on dense plans, gathered from the sample offsets on
        // packed ones -- into compact [B, hid] rows, s.tail.
        void layer(const LayerW& L, StreamRec& s, int heads, bool tail) {
            const int hid = s.hid, B = pl.B;
            qkv(s, L.qkv);
            if (!eng.x3) {
                SelfAttnArgs a{};
                a.qkv = reinterpret_cast<bf16*>(s.qkv); a.ld_qkv = 3 * hid; a.hidden = hid; a.mask = s.mask; a.ctx = s.ctx; a.ld_ctx = hid;
                a.B = B; a.L = s.seq; a.heads = heads; a.head_dim = hid / heads; a.offs = s.offs;
                a.stream_kv = s.seq > kStagedAttnRows;
                a.gate = pl.gate_at(entry);
                push({a, s.branch, 4.0 * B * heads * s.seq * s.seq * (hid / heads)});
            }
            if (eng.x3 || maps) attention_f32(s, s, hid, heads, entry);
            if (!tail) {
                row_local(s, hid, L.attn_out, L.ln1, L.inter, L.out, L.ln2, Op::NONE);
                return;
            }
            const bf16* ctx = s.ctx;
            const float* res = s.f32[0];
            int ld = s.seq * hid;
            if (pl.packed) {
                bf16* ctx_c = buf16(B, hid);
                float* res_c = buf32(B, hid);
                gather(s, s.branch, Op::NONE, s.ctx, ctx_c, res, res_c);
                ctx = ctx_c; res = res_c; ld = hid;
            }
            float* ln1_f = buf32(B, hid);
            bf16* ln1_b = buf16(B, hid);
            s.tail = buf16(B, hid);
            LinearArgs o(L.attn_out, ctx, ld, B);
            o.ln = &L.ln1; o.res = res; o.ld_res = ld; o.out16 = ln1_b; o.ld16 = hid; o.out32 = ln1_f; o.ld32 = hid; o.branch = s.branch;
            linear(o);
            LinearArgs i(L.inter, ln1_b, hid, B);
            i.act = vb::kActGelu; i.out16 = s.inter; i.ld16 = L.inter.N; i.branch = s.branch;
            linear(i);
            LinearArgs f(L.out, s.inter, L.inter.N, B);     // no fp32 copy: nothing reads the pruned stream's final fp32 rows
            f.ln = &L.ln2; f.res = ln1_f; f.ld_res = hid; f.out16 = s.tail; f.ld16 = hid; f.branch = s.branch;
            linear(f);
        }
        // One connection layer: both projections, the co-attention after joining the image branch, then the image branch's row-local
        // half on the side stream (forking from the co-attention) and the text branch's on the main one.
        void connection(const ConnW& W) {
            const int B = pl.B, Hb = eng.cfg.bi_hidden, heads = eng.cfg.bi_heads;
            qkv(v, W.qkv_img);
            qkv(t, W.qkv_txt);
            if (!eng.x3) {
                CoAttnArgs a{};
                a.qkv_img = reinterpret_cast<bf16*>(v.qkv); a.ld_img = 3 * Hb; a.qkv_txt = reinterpret_cast<bf16*>(t.qkv); a.ld_txt = 3 * Hb;
                a.hidden = Hb; a.img_mask = v.mask; a.txt_mask = t.mask; a.ctx_txt = t.ctx; a.ld_ctx_txt = Hb; a.ctx_img = v.ctx; a.ld_ctx_img = Hb;
                a.B = B; a.T = t.seq; a.V = v.seq; a.heads = heads; a.head_dim = Hb / heads; a.offs_t = t.offs; a.offs_v = v.offs;
                a.stream_kv = t.seq > kStagedAttnRows || v.seq > kStagedAttnRows;
                a.gate = pl.gate_at(entry);
                push({a, 0, 8.0 * B * heads * t.seq * v.seq * (Hb / heads), Op::JOIN});
            }
            if (eng.x3 || maps) {
                // text queries (Q2) over image keys / values (K1, V1) -> text context; then image queries (Q1) over K2, V2
                attention_f32(t, v, Hb, heads, entry, Op::JOIN);
                attention_f32(v, t, Hb, heads, entry + 1);
            }
            row_local(v, Hb, W.dense1, W.ln1, W.v_inter, W.v_out, W.v_ln, Op::FORK);
            row_local(t, Hb, W.dense2, W.ln2, W.t_inter, W.t_out, W.t_ln, Op::NONE);
        }
        // A two-GEMM head on `rows` rows of a (row stride lda): the transform (GELU, LayerNorm) into hid16, the decoder's logits into
        // a new *logits -- a task head's logit_fc, a pre-training prediction head.
        void predict(const LinearW& transform, const LNW& ln, const LinearW& decoder, const bf16* a, int lda, bf16* hid16, int rows,
                     const int* m_rows, OutBuf* logits) {
            LinearArgs g0(transform, a, lda, rows);
            g0.act = vb::kActGelu; g0.ln = &ln; g0.out16 = hid16; g0.ld16 = transform.N; g0.m_rows = m_rows;
            linear(g0);
            *logits = make_out(rows, decoder.N);
            LinearArgs g1(decoder, hid16, transform.N, rows);
            g1.out32 = logits->p; g1.ld32 = logits->ld; g1.m_rows = m_rows;
            linear(g1);
        }
        // ---- poolers + heads (main stream, after joining the image branch)
        void heads(uint32_t select) {
            const vb200_engine& E = eng;
            const int B = pl.B, Hb = E.cfg.bi_hidden;
            float* pooled_t = buf32(B, Hb);
            float* pooled = buf32(B, Hb);
            bf16* pooled_b = buf16(B, Hb);
            Op::Sync join = Op::JOIN;       // the heads' first launch waits for the image branch
            // The poolers' operand, each sample's first row of a final state: a pruned tail's compact rows, the full state at stride
            // seq rows on dense plans, or on packed plans (a sample's first row sits at a per-call offset) the B first rows gathered
            // into compact [B, hid] rows.  Returns the operand and its row stride.
            auto first_rows = [&](const StreamRec& s) -> std::pair<const bf16*, int64_t> {
                if (s.tail != nullptr) return {s.tail, s.hid};
                if (!pl.packed) return {s.b16[0], static_cast<int64_t>(s.seq) * s.hid};
                bf16* first = buf16(B, s.hid);
                gather(s, 0, std::exchange(join, Op::NONE), s.b16[0], first);
                return {first, s.hid};
            };
            const auto first_t = first_rows(t);
            const auto first_v = first_rows(v);
            LinearArgs pt(E.t_pool, first_t.first, first_t.second, B);
            pt.act = vb::kActRelu; pt.out32 = pooled_t; pt.ld32 = Hb; pt.sync = join;
            linear(pt);
            LinearArgs pv(E.v_pool, first_v.first, first_v.second, B);
            pv.act = vb::kActRelu; pv.out16 = pooled_b; pv.ld16 = Hb; pv.out32 = pooled; pv.ld32 = Hb; pv.mul = pooled_t; pv.ld_mul = Hb;
            linear(pv);
            pl.outs[kOutPooled] = OutBuf{pooled, B, Hb, Hb};
            auto cls_head = [&](const ClsW& w, int slot) { predict(w.fc0, w.ln, w.fc3, pooled_b, Hb, buf16(B, 2 * Hb), B, nullptr, &pl.outs[slot]); };
            if (select & VB200_OUT_VIL_PREDICTION) cls_head(E.vqa, kOutVqa);
            if (select & VB200_OUT_VIL_PREDICTION_GQA) cls_head(E.gqa, kOutGqa);
            if (select & VB200_OUT_VIL_LOGIT) rowdot(pooled, Hb, E.vil_logit, nullptr, out(kOutVilLogit, 1));
            if (select & VB200_OUT_VIL_BINARY_PREDICTION) {
                if (B % 2 == 0) {
                    // pooled.view(-1, 2*bi_hidden): adjacent samples form one NLVR2 pair (worker.py:266-276)
                    float* hid = buf32(B / 2, 2 * Hb);
                    LinearArgs g0(E.binary.fc0, pooled_b, 2 * Hb, B / 2);
                    g0.act = vb::kActGelu; g0.ln = &E.binary.ln; g0.out32 = hid; g0.ld32 = 2 * Hb;
                    linear(g0);
                    rowdot(hid, 2 * Hb, E.binary.fc3_row, nullptr, out(kOutBinary, 2));
                } else {
                    // [UPSTREAM] odd batch: element 3 stays the pre-training bi_seq_relationship score
                    rowdot(pooled, Hb, E.seq_rel, nullptr, out(kOutBinary, 2));
                }
            }
            if (select & VB200_OUT_VIL_TRI_PREDICTION) rowdot(pooled, Hb, E.vil_tri, nullptr, out(kOutTri, 3));
            if (select & VB200_OUT_VISION_PREDICTION)
                predict(E.img_transform, E.img_ln, E.img_decoder, v.b16[0], v.hid, buf16(v.rows, v.hid), v.rows, v.m_rows, &pl.outs[kOutVisionPred]);
            if (select & VB200_OUT_VISION_LOGIT) rowdot(v.f32[0], v.hid, E.vision_logit, v.mask, out(kOutVisionLogit, 1), v.m_rows);
            if (select & VB200_OUT_LINGUISIC_PREDICTION)
                predict(E.lm_transform, E.lm_ln, E.lm_decoder, t.b16[0], t.hid, buf16(t.rows, t.hid), t.rows, t.m_rows, &pl.outs[kOutLingPred]);
            if (select & VB200_OUT_LINGUISIC_LOGIT) rowdot(t.f32[0], t.hid, E.ling_logit, nullptr, out(kOutLingLogit, 1), t.m_rows);
        }
    };
    // attention-probability entries one forward with maps writes: the selected ones of the full list (one per text / image layer,
    // two per connection layer)
    int selected_entries() const {
        const int all = static_cast<int>(attention_kinds(schedule).size());
        int n = 0;
        for (int e = 0; e < all; ++e) n += attn_sel.has(e) ? 1 : 0;
        return n;
    }

    // layer-state entries one forward with states writes
    int selected_states() const {
        const int all = static_cast<int>(state_kinds(schedule).size());
        int n = 0;
        for (int e = 0; e < all; ++e) n += state_sel.has(e) ? 1 : 0;
        return n;
    }

    // Plan modes.  FULL is the reference's forward (worker.py:286-289).  The other three split it at the first connection layer
    // for caption-image retrieval (SURVEY.md section 8e): everything before it depends on the caption alone (text embeddings +
    // the text layers scheduled ahead of C0) or on the image alone (image embedding + any image layer ahead of C0), so a
    // 1000 x 1000 score matrix computes those once per caption / per image and runs only the SUFFIX per pair -- the same kernels on
    // the same rows, hence bit-identical scores.
    // PACKED runs FULL's schedule on a packed variable-length batch (vb200_forward_packed): Tin + task tokens and V are the plan's
    // per-sample capacities (multiples of 16), every buffer holds B x capacity rows, and the kernels take the call's row offsets and
    // row totals from the plan's d_meta -- GEMMs skip the tiles past the totals, attention runs each sample at its own length.
    // PACKED_TEXT_PREFIX, PACKED_IMAGE_PREFIX and PACKED_SUFFIX are the retrieval split of PACKED: captions, images and pairs
    // stored back to back at their own lengths (mode = PACKED + the dense mode).
    enum PlanMode { FULL = 0, TEXT_PREFIX = 1, IMAGE_PREFIX = 2, SUFFIX = 3, PACKED = 4,
                    PACKED_TEXT_PREFIX = 5, PACKED_IMAGE_PREFIX = 6, PACKED_SUFFIX = 7 };

    // The plan-key bits of the taps a call reads (kTextRows / kImageRows): a forward whose select and taps read no final row of a
    // stream prunes that stream's tail (get_plan).
    static uint32_t rows_read(const vb200_outputs* out) {
        uint32_t r = 0;
        for (const OutSlot& o : kOutSlots) r |= out != nullptr && out->*o.field ? o.bit & (kTextRows | kImageRows) : 0;
        return r;
    }

    // A pre-training engine has no task head: every select bit of VB200_OUT_TASK_HEADS is rejected, naming the head.
    static void reject_task_heads(uint32_t select) {
        for (const OutSlot& h : kOutSlots)
            if (select & h.bit & VB200_OUT_TASK_HEADS)
                fail(VB200_ERR_INVALID, "the task head %s is not part of a pre-training engine (select only the pre-training heads, "
                     "taps or attention maps)", h.name);
    }

    // The plan-key bits of the final rows a layer-state selection reads: a selected last entry of a stream keeps its tail unpruned.
    uint32_t states_read() const {
        const std::vector<int> k = state_kinds(schedule);
        int last[2] = {0, 0};
        for (int e = 0; e < static_cast<int>(k.size()); ++e) last[k[e]] = e;
        return (state_sel.has(last[0]) ? kTextRows : 0) | (state_sel.has(last[1]) ? kImageRows : 0);
    }
    // The head gate table's shape: every entry of the full attention list, the configuration's largest head count.
    int gate_entries() const { return static_cast<int>(attention_kinds(schedule).size()); }
    int gate_heads() const { return std::max({cfg.heads, cfg.v_heads, cfg.bi_heads}); }

    // gated (PACKED plans only): the plan owns a head gate table and its attention launches read it
    Plan* get_plan(int B, int Tin, int V, uint32_t select, int slot = 0, int mode = FULL, bool want_attn = false, bool want_states = false,
                   bool gated = false) {
        if (slot < 0 || slot > 15) fail(VB200_ERR_INVALID, "slot %d out of range (0..15)", slot);
        if (slot > 0 && !opt.use_cuda_graph) fail(VB200_ERR_INVALID, "concurrent slots need CUDA-graph plans (use_cuda_graph)");
        const bool packed = mode >= PACKED;
        const int schedule_mode = packed ? mode - PACKED : mode;     // which part of the schedule: FULL, a prefix or the suffix
        if (schedule_mode == TEXT_PREFIX || schedule_mode == IMAGE_PREFIX) { select = 0; want_attn = false; want_states = false; }
        if (want_states) select |= states_read();
        if (pretraining) reject_task_heads(select);
        const int T = Tin + (cfg.task_tokens ? 1 : 0);
        // ahead of the cache: a plan built under a higher max_rows_per_sample must not outlive the bound being lowered.  Packed
        // capacities are the call's longest rows rounded up to 16 (pack_batch has checked the rows themselves against the bound)
        const int cap = mode >= PACKED ? (max_rows + 15) / 16 * 16 : max_rows;
        if (T > cap || V > cap)
            fail(VB200_ERR_INVALID, "sequence too long for %s (T=%d, V=%d, max %d)", bound_name(max_rows), T, V, cap);
        // the map selection is part of the key of a plan with maps: a call never replays a plan built for another selection
        // and so is the state selection of a plan with layer states
        std::vector<int64_t> key{B, Tin, V, static_cast<int64_t>(select), slot, mode, want_attn ? 1 : 0,
                                 want_attn ? static_cast<int64_t>(attn_sel.mask) : 0, want_attn && attn_sel.mean ? 1 : 0,
                                 want_states ? 1 : 0, want_states ? static_cast<int64_t>(state_sel.mask) : 0,
                                 want_states ? state_sel.rows : 0, gated ? 1 : 0};
        auto it = plans.find(key);
        if (it != plans.end()) { it->second->last_use = ++use_clock; return it->second.get(); }
        std::unique_ptr<Plan> up(new Plan());
        Plan& pl = *up;
        const Config& c = cfg;
        // The build's stream: the zero fills below and the validation pass.  A plain cudaMemset would go to the legacy default
        // stream, which a non-blocking stream (this one, and a caller's) does not wait for, so the validation pass could read what an
        // evicted plan left in the same memory.  The build synchronises it before the plan is used on any other stream.
        const Stream ws = make_stream();
        if (B < 1 || Tin < 1 || V < 1) fail(VB200_ERR_INVALID, "batch, n_tokens and n_regions must be positive");
        if (Tin > c.max_pos && !packed) fail(VB200_ERR_INVALID, "n_tokens %d exceeds max_position_embeddings %d", Tin, c.max_pos);
        pl.B = B; pl.Tin = Tin; pl.T = T; pl.V = V;
        if (packed || want_states) {
            // zero offsets and destinations until the first call: the validation pass and the capture below then touch no row and
            // write no state.  Dense plans hold only the layer states' destinations.
            pl.packed = packed;
            pl.layout = MetaLayout{static_cast<size_t>(B), packed && want_attn ? static_cast<size_t>(selected_entries()) : 0,
                                   mode == PACKED_SUFFIX, want_states ? static_cast<size_t>(selected_states()) : 0};
            const size_t n_meta = pl.layout.size();
            pl.d_meta = pl.mem.alloc_n<int>(n_meta);
            CUDA_CHECK(cudaMemsetAsync(pl.d_meta, 0, n_meta * sizeof(int), ws.get()));
            pl.meta.copied = make_event();
            pl.meta.reserve(n_meta * sizeof(int));
        }
        if (gated) {
            if (mode != PACKED) fail(VB200_ERR_INVALID, "head gates exist for the PACKED forwards only");
            pl.gate_entries = gate_entries();
            pl.gate_heads = gate_heads();
            pl.gate = pl.mem.alloc_n<float>(static_cast<size_t>(B) * pl.gate_entries * pl.gate_heads);
        }
        const int Mt = B * T, Mv = B * V, H = c.hidden, Hv = c.v_hidden, Hb = c.bi_hidden;
        const bool full = schedule_mode == FULL;
        const bool do_t = full || schedule_mode == TEXT_PREFIX, do_v = full || schedule_mode == IMAGE_PREFIX;
        const bool do_s = full || schedule_mode == SUFFIX;
        // Pruned tail: the poolers read one row per sample of each final state.  A stream no per-row head and no tap reads runs its
        // last layer's row-local half (everything after the self-attention) on those B rows only; bit-identical rows, since no
        // kernel's per-element result depends on M.  A stream whose last layer is a connection layer keeps its full rows.
        const bool prune_t = do_s && !(select & out_bits(kTextRow));
        const bool prune_v = do_s && !(select & out_bits(kImageRow));
        size_t last_t = 0, last_v = 0;                 // the last schedule step writing each stream
        for (size_t i = 0; i < schedule.size(); ++i) {
            if (schedule[i][0] != 'V') last_t = i;
            if (schedule[i][0] != 'T') last_v = i;
        }
        PlanBuilder b{*this, pl, std::max(Mt, Mv), "embed"};
        pl.kp = img_emb.ldw;
        pl.img_a = b.buf16(Mv, pl.kp);
        pl.mask_t = pl.mem.alloc_n<float>(Mt);
        pl.mask_v = pl.mem.alloc_n<float>(Mv);
        if (mode == PACKED_SUFFIX) {
            // the attention kernels read the additive key masks in packed plans too, and every packed row is real: all zero, for good
            // (no embedding kernel of a packed suffix writes them)
            CUDA_CHECK(cudaMemsetAsync(pl.mask_t, 0, static_cast<size_t>(Mt) * sizeof(float), ws.get()));
            CUDA_CHECK(cudaMemsetAsync(pl.mask_v, 0, static_cast<size_t>(Mv) * sizeof(float), ws.get()));
        }
        for (int i = 0; i < 2; ++i) {
            pl.t_f32[i] = b.buf32(Mt, H);
            pl.t_b16[i] = b.buf16(Mt, H);
            pl.v_f32[i] = b.buf32(Mv, Hv);
            pl.v_b16[i] = b.buf16(Mv, Hv);
        }
        b.y[0] = pl.mem.alloc_n<float>(std::max({static_cast<size_t>(Mt) * H, static_cast<size_t>(Mv) * Hv, static_cast<size_t>(B) * 2 * Hb}));
        b.y[1] = b.buf32(Mv, Hv);
        // Q | K | V projections: 16-bit for the tensor-core attention kernel, fp32 in fp32-parity mode
        const size_t qe = x3 ? 4 : 2;
        uint8_t* qkv_t = static_cast<uint8_t*>(pl.mem.alloc(static_cast<size_t>(Mt) * 3 * std::max(H, Hb) * qe));
        uint8_t* qkv_v = static_cast<uint8_t*>(pl.mem.alloc(static_cast<size_t>(Mv) * 3 * std::max(Hv, Hb) * qe));
        bf16* ctx_t = b.buf16(Mt, std::max(H, Hb));
        bf16* ctx_v = b.buf16(Mv, std::max(Hv, Hb));
        bf16* inter_t = b.buf16(Mt, c.inter);
        bf16* inter_v = b.buf16(Mv, c.v_inter);
        b.t = StreamRec{pl.t_f32, pl.t_b16, H, T, Mt, 0, 0, pl.mask_t, qkv_t, ctx_t, inter_t, packed ? pl.rows_t() : nullptr,
                        packed ? pl.offs_t() : nullptr, nullptr};
        b.v = StreamRec{pl.v_f32, pl.v_b16, Hv, V, Mv, 1, 1, pl.mask_v, qkv_v, ctx_v, inter_v, packed ? pl.rows_v() : nullptr,
                        packed ? pl.offs_v() : nullptr, nullptr};
        b.maps = want_attn;
        b.states = want_states;

        // image embedding: LayerNorm(feat.W_img^T + loc.W_loc^T + b) as ONE GEMM over K = v_feat + 64, on the side stream: it
        // overlaps the text layers ahead of the first co-attention
        if (do_v) {
            LinearArgs g(b.v, img_emb, pl.img_a, pl.kp);
            g.ln = &vemb_ln; g.out16 = pl.v_b16[0]; g.ld16 = Hv; g.out32 = pl.v_f32[0]; g.ld32 = Hv;
            b.linear(g);
        }
        // layer states (FULL and PACKED plans only): the embeddings are entries 0 (text, written by the input kernels ahead of the
        // plan) and 1, then each step's text state before its image state
        b.state(b.v, 1);
        b.state(b.t, 0);
        int state_e = 2;
        bool in_suffix = false;
        for (size_t si = 0; si < schedule.size(); ++si) {
            const std::string& step = schedule[si];
            const int idx = atoi(step.c_str() + 1);
            b.tag = step.c_str();          // engine.schedule outlives every plan
            if (step[0] == 'C') in_suffix = true;
            if (step[0] == 'T') {
                if (in_suffix ? do_s : do_t) b.layer(t_layers[idx], b.t, c.heads, prune_t && si == last_t);
            } else if (step[0] == 'V') {
                if (in_suffix ? do_s : do_v) b.layer(v_layers[idx], b.v, c.v_heads, prune_v && si == last_v);
            } else if (do_s) {
                b.connection(c_layers[idx]);
            }
            if (step[0] != 'V') b.state(b.t, state_e++);
            if (step[0] != 'T') b.state(b.v, state_e++);
            b.entry += step[0] == 'C' ? 2 : 1;
        }
        if (b.t.tail == nullptr) pl.outs[kOutSeqT] = OutBuf{pl.t_f32[0], Mt, H, H};
        if (b.v.tail == nullptr) pl.outs[kOutSeqV] = OutBuf{pl.v_f32[0], Mv, Hv, Hv};
        b.tag = "heads";
        if (do_s) b.heads(select);
        for (const Op& op : pl.ops) pl.flops += op.flops;

        if (timeline) attach_timeline(pl, ws.get());
        // One eager pass first: opts kernels into their shared-memory sizes and surfaces launch-configuration
        // errors with a real message (errors inside a capture only invalidate the capture).
        if (!pl.ops.empty()) run_ops(pl, ws.get());
        CUDA_CHECK(cudaStreamSynchronize(ws.get()));
        if (!pl.ops.empty() && opt.use_cuda_graph) capture(pl);
        Plan* raw = up.get();
        raw->last_use = ++use_clock;
        plans[key] = std::move(up);
        evict_plans(raw);
        return raw;
    }

    // Profiling: every plain persistent GEMM of the plan writes its per-CTA stamps (gemm_persistent.cuh: entry / exit %globaltimer, SM id,
    // clock64 at setup done, first k-block landed, last MMA committed, epilogue done) into a plan-owned buffer; a replay overwrites the
    // previous one, so after a run the buffer holds the LAST forward of this plan (scripts/step_timeline.py reads two slots' worth).
    static constexpr int kTimelineCtas = 304;
    void attach_timeline(Plan& pl, cudaStream_t st) {
        size_t n = 0;
        for (const Op& op : pl.ops) n += std::holds_alternative<GemmCall>(op.args);
        if (n == 0) return;
        pl.timeline = pl.mem.alloc_n<long long>(n * kTimelineCtas * 16);
        CUDA_CHECK(cudaMemsetAsync(pl.timeline, 0, n * kTimelineCtas * 16 * sizeof(long long), st));
        size_t i = 0;
        for (Op& op : pl.ops)
            if (GemmCall* g = std::get_if<GemmCall>(&op.args)) g->ep.timing = pl.timeline + (i++) * kTimelineCtas * 16;
    }

    // Plan cache bound (a MicroBatchWorker produces many (batch, length, regions) combinations): beyond max_plans the least
    // recently used plan -- its workspace (about 1 MB per pair) and CUDA graph -- is destroyed.  Rare, so the device is drained
    // first: a plan may still be executing on some stream.
    void evict_plans(const Plan* keep) {
        while (plans.size() > max_plans) {
            auto victim = plans.end();
            for (auto it = plans.begin(); it != plans.end(); ++it)
                if (it->second.get() != keep && (victim == plans.end() || it->second->last_use < victim->second->last_use)) victim = it;
            if (victim == plans.end()) break;
            cudaDeviceSynchronize();
            plans.erase(victim);
        }
    }

    // ---------------------------------------------------------------- execution
    void launch_op(const Op& op, cudaStream_t st) {
        const int pdl = opt.use_pdl, f16 = opt.act_fp16;
        std::visit(Overloaded{
            [&](const GemmCall& g) {
                const cudaError_t le = g.launch(st, profile_grid_pct);   // profile_grid_pct: 0 outside vb200_profile_ops
                const GemmEpilogue& e = g.ep;
                if (le != cudaSuccess)
                    fail(VB200_ERR_CUDA, "GEMM launch failed: %s (layer %s, M=%d N=%d K=%d act=%d block_n=%d split16=%d tma_store=%d)",
                         cudaGetErrorString(le), op.tag ? op.tag : "?", e.M, e.N, e.K, e.act, g.block_n, e.split16, e.tma_store);
            },
            [&](const SelfAttnArgs& a) {
                CUDA_CHECK((a.stream_kv ? vb::launch_self_attention_stream : vb::launch_self_attention)(
                    a.qkv, a.ld_qkv, a.hidden, a.mask, a.ctx, a.ld_ctx, a.B, a.L, a.heads, a.head_dim, pdl, f16, st, a.offs, a.gate));
            },
            [&](const CoAttnArgs& a) {
                CUDA_CHECK((a.stream_kv ? vb::launch_co_attention_stream : vb::launch_co_attention)(
                    a.qkv_img, a.ld_img, a.qkv_txt, a.ld_txt, a.hidden, a.img_mask, a.txt_mask, a.ctx_txt, a.ld_ctx_txt, a.ctx_img,
                    a.ld_ctx_img, a.B, a.T, a.V, a.heads, a.head_dim, pdl, f16, st, a.offs_t, a.offs_v, a.gate));
            },
            [&](const RowdotArgs& a) {
                CUDA_CHECK(vb::launch_rowdot(a.x, a.ld_x, a.W, a.bias, a.add, a.out, a.ld_out, a.M, a.K, a.n_out, pdl, st, a.m_rows));
            },
            [&](const LayerNormArgs& a) {
                CUDA_CHECK(vb::launch_ln_residual(a.y, a.ld_y, a.res, a.ld_res, a.gamma, a.beta, cfg.ln_eps, a.out_f32, a.ld_f32, a.out16,
                                                  a.ld16, a.M, a.N, f16, x3 ? 1 : 0, pdl, st, a.m_rows));
            },
            [&](const AttnF32Args& a) {
                if (a.mean) {
                    CUDA_CHECK(vb::launch_attention_f32_mean(a.q, a.ld_q, a.k, a.ld_kv, a.in_kind, a.mask, a.B, a.Lq, a.Lk, a.heads,
                                                             a.head_dim, a.probs, pdl, st, a.packed ? &a.pk : nullptr));
                    return;
                }
                CUDA_CHECK(vb::launch_attention_f32(a.q, a.ld_q, a.k, a.v, a.ld_kv, a.in_kind, a.mask, a.B, a.Lq, a.Lk, a.heads,
                                                    a.head_dim, a.ctx, a.ld_ctx, a.ctx_mode, a.probs, pdl, st,
                                                    a.packed ? &a.pk : nullptr));
            },
            [&](const GatherArgs& a) {
                CUDA_CHECK(vb::launch_gather_state(a.offs, a.n_src, a.src_f32, a.src16, nullptr, a.dst_f32, a.dst16, nullptr, a.B, 1,
                                                   a.hidden, a.ld16, st));
            },
            [&](const vb::StateArgs& a) { CUDA_CHECK(vb::launch_layer_state(a, pdl, st)); },
        }, op.args);
    }
    // vb200_profile_ops' dims of a launch-list entry
    static std::array<int, 4> op_dims(const Op& op) {
        return std::visit(Overloaded{
            [](const GemmCall& g) { return std::array<int, 4>{g.ep.M, g.ep.N, g.ep.K, g.ep.act}; },
            [](const SelfAttnArgs& a) { return std::array<int, 4>{a.B, a.L, 0, a.heads}; },
            [](const CoAttnArgs& a) { return std::array<int, 4>{a.B, a.T, a.V, a.heads}; },
            [](const RowdotArgs&) { return std::array<int, 4>{0, 0, 0, 0}; },
            [](const LayerNormArgs& a) { return std::array<int, 4>{a.M, a.N, 0, 0}; },
            [](const AttnF32Args& a) { return std::array<int, 4>{a.B, 0, 0, a.heads}; },
            [](const GatherArgs& a) { return std::array<int, 4>{a.B, 0, 0, 0}; },
            [](const vb::StateArgs& a) { return std::array<int, 4>{a.B, a.L, a.H, 0}; },
        }, op.args);
    }
    // Text-stream ops go to `st`, image-stream ops to the side stream so the two ViLBERT streams overlap
    // (T_k || V_k between co-attentions, and the two halves of a connection layer).  Dependencies across the
    // two are explicit: a side op marked FORK (and the first side op) waits for everything enqueued on `st`
    // so far; a main op marked JOIN waits for the side stream.  Under capture these become graph edges.
    void run_ops(Plan& pl, cudaStream_t st) {
        bool side_started = false, side_dirty = false;
        const char* open_tag = nullptr;
        struct RangeGuard { const char*& t; ~RangeGuard() { if (t) nvtxRangePop(); } } guard{open_tag};
        for (const Op& op : pl.ops) {
            if (op.tag != open_tag) {              // one NVTX range per layer of the schedule (enqueue side)
                if (open_tag) nvtxRangePop();
                open_tag = op.tag;
                if (open_tag) nvtxRangePushA(open_tag);
            }
            if (op.stream == 1) {
                if (!side_started || op.sync == Op::FORK) {
                    CUDA_CHECK(cudaEventRecord(ev_fork.get(), st));
                    CUDA_CHECK(cudaStreamWaitEvent(side_stream.get(), ev_fork.get(), 0));
                    side_started = true;
                }
                launch_op(op, side_stream.get());
                side_dirty = true;
            } else {
                if (op.sync == Op::JOIN && side_dirty) {
                    CUDA_CHECK(cudaEventRecord(ev_join.get(), side_stream.get()));
                    CUDA_CHECK(cudaStreamWaitEvent(st, ev_join.get(), 0));
                    side_dirty = false;
                }
                launch_op(op, st);
            }
        }
        if (side_dirty) {
            CUDA_CHECK(cudaEventRecord(ev_join.get(), side_stream.get()));
            CUDA_CHECK(cudaStreamWaitEvent(st, ev_join.get(), 0));
        }
    }
    // Per-op device time: each launch-list entry is captured `kRep` times into its own CUDA graph and the graph replayed
    // between two CUDA events on the launching stream, so the number is the kernel's duration (incl. the grid launch
    // latency every launch pays inside the captured forward as well) without host launch gaps.  Every op is idempotent on
    // the plan's workspace, which must hold a previous forward's data.  Used by bench.py for the per-kernel roofline.
    void profile_ops(Plan& pl, int iters, std::vector<double>& ms_out) {
        constexpr int kRep = 8;
        const Stream owned = make_stream();
        const cudaStream_t st = owned.get();
        const Event e0 = make_event(cudaEventDefault), e1 = make_event(cudaEventDefault);
        const size_t n = pl.ops.size();
        ms_out.assign(n, 0.0);
        for (size_t i = 0; i < n; ++i) {
            const Graph g = capture_graph(st, [&] { for (int r = 0; r < kRep; ++r) launch_op(pl.ops[i], st); });
            const GraphExec ge = instantiate(g.get());
            CUDA_CHECK(cudaGraphLaunch(ge.get(), st));                  // warm-up
            CUDA_CHECK(cudaEventRecord(e0.get(), st));
            for (int it = 0; it < iters; ++it) CUDA_CHECK(cudaGraphLaunch(ge.get(), st));
            CUDA_CHECK(cudaEventRecord(e1.get(), st));
            CUDA_CHECK(cudaStreamSynchronize(st));
            float ms = 0.0f;
            CUDA_CHECK(cudaEventElapsedTime(&ms, e0.get(), e1.get()));
            ms_out[i] = ms / (static_cast<double>(iters) * kRep);
        }
    }

    void capture(Plan& pl) {
        const Stream cs = make_stream();
        pl.graph = capture_graph(cs.get(), [&] { run_ops(pl, cs.get()); });
        pl.exec = instantiate(pl.graph.get());
    }

    void check_inputs(const vb200_inputs& in) const {
        if (!in.question || !in.features || !in.spatials || !in.segment_ids || !in.input_mask || !in.image_mask ||
            (cfg.task_tokens && !in.task_tokens))
            fail(VB200_ERR_INVALID, "vb200_inputs has a NULL required pointer");
    }
    // the dense forward's input kernels, on inputs check_inputs has accepted
    void embed_inputs(Plan& pl, const vb200_inputs& in, cudaStream_t st) {
        embed_text(pl, in.question, in.segment_ids, in.input_mask, in.task_tokens, pl.B * pl.T, st);
        pack_image(pl, in.features, in.spatials, in.image_mask, pl.B * pl.V, st);
    }
    // The input kernels of every plan.  `rows`: the text / image rows of the call -- B x T / B x V on dense plans (padding from the
    // masks), the call's row totals on packed plans (no masks: every row is real; the rows up to the next 128-row GEMM tile are
    // zeroed, the only rows past the totals a GEMM loads).
    void embed_text(Plan& pl, const int64_t* q, const int64_t* seg, const int64_t* input_mask, const int64_t* tk, int rows, cudaStream_t st) {
        const Config& c = cfg;
        CUDA_CHECK(vb::launch_text_embed(q, seg, input_mask, tk, word, pos, type, task, emb_ln.g, emb_ln.b, c.ln_eps, pl.t_f32[0], pl.t_b16[0],
                                         pl.mask_t, pl.B, pl.Tin, c.hidden, c.vocab, c.max_pos, c.type_vocab, c.n_task, c.task_tokens,
                                         opt.act_fp16, x3 ? 1 : 0, st, pl.packed ? pl.offs_t() : nullptr, rows));
        if (pl.packed) zero_tail(pl.t_b16[0], rows, pl.B * pl.T, c.hidden, st);
    }
    void pack_image(Plan& pl, const float* feats, const float* loc, const uint8_t* image_mask, int rows, cudaStream_t st) {
        CUDA_CHECK(vb::launch_image_pack(feats, loc, image_mask, pl.img_a, pl.mask_v, rows, cfg.v_feat, pl.kp, opt.act_fp16, x3 ? 1 : 0, st));
        if (pl.packed) zero_tail(pl.img_a, rows, pl.B * pl.V, pl.kp, st);
    }
    // zero the 16-bit operand rows [rows, next 128-row boundary) of a buffer with `cap` rows
    static void zero_tail(bf16* buf, int rows, int cap, size_t width, cudaStream_t st) {
        const int end = std::min(cap, (rows + 127) / 128 * 128);
        if (end > rows) CUDA_CHECK(cudaMemsetAsync(buf + static_cast<size_t>(rows) * width, 0, static_cast<size_t>(end - rows) * width * 2, st));
    }
    void run_plan(Plan& pl, cudaStream_t st) {
        if (pl.ops.empty()) return;
        struct R { R(const Plan& p) { char b[96]; snprintf(b, sizeof(b), "vb200 forward B=%d T=%d V=%d", p.B, p.T, p.V); nvtxRangePushA(b); }
                   ~R() { nvtxRangePop(); } } range(pl);
        if (pl.exec) CUDA_CHECK(cudaGraphLaunch(pl.exec.get(), st));
        else run_ops(pl, st);
    }
    // worker.py:422-455 on the device: detector output -> operand rows / masks for the same plan as the dense forward
    void embed_regions(Plan& pl, const vb200_region_inputs& in, cudaStream_t st) {
        const Config& c = cfg;
        if (!in.question || !in.segment_ids || !in.input_mask || (c.task_tokens && !in.task_tokens) || !in.box_features || !in.boxes ||
            !in.image_wh)
            fail(VB200_ERR_INVALID, "vb200_region_inputs has a NULL required pointer");
        embed_text(pl, in.question, in.segment_ids, in.input_mask, in.task_tokens, pl.B * pl.T, st);
        CUDA_CHECK(vb::launch_region_pack(in.box_features, in.boxes, in.image_wh, in.num_boxes, pl.img_a, pl.mask_v, in.spatials_out,
                                          pl.B, pl.V - 1, c.v_feat, pl.kp, opt.act_fp16, x3 ? 1 : 0, st));
    }
    // ---- packed batches (run_packed has staged the call's d_meta ahead of these, in stream order)
    // Packed detector output: the region-pack kernel writes every image's mean row and boxes at the plan's image offsets (the same
    // rows embed_regions writes for that image alone)
    // (src / kept: the ablation calls' per-image sources and kept-box lists, see launch_region_pack)
    void pack_regions_packed(Plan& pl, const float* box_feats, const float* boxes, const float* image_wh, float* spatials_out, int rows,
                             cudaStream_t st, const vb::RegionSrc* src = nullptr, const int32_t* kept = nullptr) {
        CUDA_CHECK(vb::launch_region_pack(box_feats, boxes, image_wh, nullptr, pl.img_a, pl.mask_v, spatials_out, pl.B, 0, cfg.v_feat,
                                          pl.kp, opt.act_fp16, 0, st, pl.offs_v(), src, kept));
        zero_tail(pl.img_a, rows, pl.B * pl.V, pl.kp, st);
    }
    // packed pair suffix: every pair's rows are gathered from the packed caption / image states into the plan's packed buffers
    void gather_packed_state(Plan& pl, const vb200_packed_pairs& in, const PackedBatch& b, cudaStream_t st) {
        const Config& c = cfg;
        const vb::PackedStateCopy text{pl.offs_t(), pl.src_t(), in.text_f32, in.text_16, pl.t_f32[0], pl.t_b16[0], c.hidden / 4, c.hidden / 8};
        const vb::PackedStateCopy image{pl.offs_v(), pl.src_v(), in.image_f32, in.image_16, pl.v_f32[0], pl.v_b16[0], c.v_hidden / 4,
                                        c.v_hidden / 8};
        CUDA_CHECK(vb::launch_gather_packed_state(text, image, pl.B, st));
        zero_tail(pl.t_b16[0], b.rows_t(), pl.B * pl.T, c.hidden, st);
        zero_tail(pl.v_b16[0], b.rows_v(), pl.B * pl.V, c.v_hidden, st);
    }
    // ---- retrieval reuse (PlanMode): per-caption / per-image prefixes and the pair suffix.  A prefix leaves its stream's state after
    // the layers ahead of the first connection layer in the caller's buffers: B x T / B x V rows with the mask on dense plans, the
    // call's rows back to back and no mask (mask null) on packed plans
    struct PrefixState { float* f32; void* b16; float* mask; };
    void copy_state(const Plan& pl, bool text, size_t rows, const PrefixState& to, cudaStream_t st) {
        const size_t H = text ? cfg.hidden : cfg.v_hidden, S = x3 ? 3 : 1;
        const float* f32 = text ? pl.t_f32[0] : pl.v_f32[0];
        const bf16* b16 = text ? pl.t_b16[0] : pl.v_b16[0];
        CUDA_CHECK(cudaMemcpyAsync(to.f32, f32, rows * H * 4, cudaMemcpyDeviceToDevice, st));
        CUDA_CHECK(cudaMemcpyAsync(to.b16, b16, rows * H * S * 2, cudaMemcpyDeviceToDevice, st));
        if (to.mask != nullptr) CUDA_CHECK(cudaMemcpyAsync(to.mask, text ? pl.mask_t : pl.mask_v, rows * 4, cudaMemcpyDeviceToDevice, st));
    }
    void gather_state(Plan& pl, const int32_t* t_idx, int n_text, const float* t_f32, const void* t_16, const float* t_mask,
                      const int32_t* v_idx, int n_img, const float* v_f32, const void* v_16, const float* v_mask, cudaStream_t st) {
        const Config& c = cfg;
        if (!t_idx || !t_f32 || !t_16 || !t_mask || !v_idx || !v_f32 || !v_16 || !v_mask) fail(VB200_ERR_INVALID, "vb200_forward_cached: NULL pointer");
        const int S = x3 ? 3 : 1;
        CUDA_CHECK(vb::launch_gather_state(t_idx, n_text, t_f32, t_16, t_mask, pl.t_f32[0], pl.t_b16[0], pl.mask_t, pl.B, pl.T,
                                           c.hidden, c.hidden * S, st));
        CUDA_CHECK(vb::launch_gather_state(v_idx, n_img, v_f32, v_16, v_mask, pl.v_f32[0], pl.v_b16[0], pl.mask_v, pl.B, pl.V,
                                           c.v_hidden, c.v_hidden * S, st));
    }
    // What every dense entry point shares once it has checked its own inputs: the packed-map rejection, the call's plan, its input
    // kernels (`input`), the plan and then the forward's outputs (out != null, copied with `kind`) or the prefix's state (`state`).
    void run_dense(const char* api, int B, int Tin, int V, uint32_t select, int slot, int mode, const vb200_outputs* out,
                   const PrefixState& state, cudaMemcpyKind kind, void* cuda_stream, const std::function<void(Plan&, cudaStream_t)>& input) {
        reject_packed_attention(select, api);
        if (mode != FULL || kind != cudaMemcpyDeviceToDevice) reject_layer_states(select, api);
        const bool states = (select & VB200_OUT_LAYER_STATES) != 0;
        if (states) check_state_buffer(api, out->layer_states);
        CUDA_CHECK(cudaSetDevice(opt.device));
        Plan& pl = *get_plan(B, Tin, V, (select & VB200_OUT_ALL) | rows_read(out), slot, mode, (select & VB200_OUT_ATTENTION) != 0, states);
        const cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
        if (states) {
            MetaLayout layout{static_cast<size_t>(pl.B)};
            std::vector<int> meta(layout.size(), 0);
            put_state_dsts(layout, meta, state_layout(cfg, schedule, state_sel, pl.B, static_cast<int64_t>(pl.B) * pl.T,
                                                      static_cast<int64_t>(pl.B) * pl.V), out->layer_states);
            stage_meta(pl, meta, st);
        }
        input(pl, st);
        run_plan(pl, st);
        if (out != nullptr) copy_outputs(pl, *out, st, kind);
        else copy_state(pl, mode == TEXT_PREFIX, mode == TEXT_PREFIX ? pl.B * pl.T : pl.B * pl.V, state, st);
    }
    // What every packed entry point shares once it has checked its own inputs: the engine-wide rejections, the call's rows
    // (pack_batch), its plan, the d_meta staged ahead of `input` (the call's input kernels), the plan and then, for the forwards
    // (out != null), the outputs at the call's row totals or, for the prefixes, the state of the call's rows.  Returns the plan,
    // whose outputs stay valid in stream order until the plan's next run.  head_mask (DEVICE [B, gate_entries, gate_heads], the gated
    // forwards): the call runs the gated plan, and one copy puts the mask into the plan's gate table ahead of `input`.  gated without
    // a head_mask (head ablation): the gated plan, whose table `input` writes.
    Plan& run_packed(const char* api, int mode, const PackedLengths& len, uint32_t select, int slot, const vb200_outputs* out,
                     const PrefixState& state, void* cuda_stream, const std::function<void(Plan&, const PackedBatch&, cudaStream_t)>& input,
                     const float* head_mask = nullptr, bool gated = false) {
        if (select & VB200_OUT_ATTENTION)
            fail(VB200_ERR_INVALID, "%s: the attention-probability output (VB200_OUT_ATTENTION) is not supported", api);
        if (mode != PACKED) reject_packed_attention(select, api);
        if (mode != PACKED) reject_layer_states(select, api);
        const bool maps = (select & VB200_OUT_ATTENTION_PACKED) != 0;
        if (maps && out->attention_probs == nullptr)
            fail(VB200_ERR_INVALID, "%s: VB200_OUT_ATTENTION_PACKED needs vb200_outputs.attention_probs (NULL)", api);
        if (x3) fail(VB200_ERR_INVALID, "%s: packed batches are not supported in split_fp32 (fp32x) mode", api);
        const bool states = (select & VB200_OUT_LAYER_STATES) != 0;
        if (states) check_state_buffer(api, out->layer_states);
        const PackedBatch b = pack_batch(api, cfg, schedule, len, maps ? out->attention_probs : nullptr, max_rows, attn_sel,
                                         states ? out->layer_states : nullptr, state_sel);
        CUDA_CHECK(cudaSetDevice(opt.device));
        Plan& pl = *get_plan(len.B, b.Tin, b.V, (select & VB200_OUT_ALL) | rows_read(out), slot, mode, maps, states,
                             gated || head_mask != nullptr);
        const cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
        stage_meta(pl, b.meta, st);
        if (head_mask != nullptr)
            CUDA_CHECK(cudaMemcpyAsync(pl.gate, head_mask, static_cast<size_t>(pl.B) * pl.gate_entries * pl.gate_heads * sizeof(float),
                                       cudaMemcpyDeviceToDevice, st));
        input(pl, b, st);
        run_plan(pl, st);
        if (out != nullptr) copy_outputs(pl, *out, st, cudaMemcpyDeviceToDevice, b.rows_t(), b.rows_v());
        else copy_state(pl, mode == PACKED_TEXT_PREFIX, mode == PACKED_TEXT_PREFIX ? b.rows_t() : b.rows_v(), state, st);
        return pl;
    }
    // meta (host, in the plan's d_meta layout) -> d_meta, in stream order ahead of the plan's kernels
    void stage_meta(Plan& pl, const std::vector<int>& meta, cudaStream_t st) {
        const size_t bytes = meta.size() * sizeof(int);
        pl.meta.stage(bytes, st, [&](char* h, const auto& put) { memcpy(h, meta.data(), bytes); put(pl.d_meta, 0, bytes); });
    }
    // ---- answer decode: every descriptor is resolved and bounds-checked before anything is enqueued
    std::vector<vb::DecodeDesc> decode_descs(const char* api, const vb200_decode_msg* msgs, int n, const vb200_outputs* out, int batch,
                                             int vision_rows, const float* spatials) const {
        if (n < 1) fail(VB200_ERR_INVALID, "%s: n must be positive (n = %d)", api, n);
        if (msgs == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "%s: msgs / out is NULL", api);
        if (batch < 0 || vision_rows < 0) fail(VB200_ERR_INVALID, "%s: negative batch %d or vision_rows %d", api, batch, vision_rows);
        std::vector<vb::DecodeDesc> d(n);
        for (int i = 0; i < n; ++i) {
            const vb200_decode_msg& m = msgs[i];
            const char* field = nullptr;
            const float* src = nullptr;
            int64_t rows = batch, width = 1;
            switch (m.family) {
                case VB200_DECODE_VQA: field = "vil_prediction"; src = out->vil_prediction; width = num_labels; break;
                case VB200_DECODE_GQA: field = "vil_prediction_gqa"; src = out->vil_prediction_gqa; width = gqa_labels; break;
                case VB200_DECODE_NLVR2:
                    field = "vil_binary_prediction"; src = out->vil_binary_prediction; width = 2; rows = batch % 2 == 0 ? batch / 2 : batch;
                    break;
                case VB200_DECODE_SNLI_VE: field = "vil_tri_prediction"; src = out->vil_tri_prediction; width = 3; break;
                case VB200_DECODE_RETRIEVAL: field = "vil_logit"; src = out->vil_logit; break;
                case VB200_DECODE_GROUNDING: field = "vision_logit"; src = out->vision_logit; rows = vision_rows; break;
                default: fail(VB200_ERR_INVALID, "%s: message %d has unknown family %d", api, i, m.family);
            }
            if (pretraining)
                fail(VB200_ERR_INVALID, "%s: message %d (family %d) reads the task head %s, which is not part of a pre-training engine", api,
                     i, m.family, field);
            if (src == nullptr) fail(VB200_ERR_INVALID, "%s: message %d (family %d) reads vb200_outputs.%s, which is NULL", api, i, m.family, field);
            const bool grounding = m.family == VB200_DECODE_GROUNDING;
            if (grounding && spatials == nullptr) fail(VB200_ERR_INVALID, "%s: message %d is a grounding message and spatials is NULL", api, i);
            if (m.count < 1 || m.first < 0 || static_cast<int64_t>(m.first) + m.count > rows)
                fail(VB200_ERR_INVALID, "%s: message %d has rows [%d, %lld) outside %s's %lld rows", api, i, m.first,
                     static_cast<long long>(static_cast<int64_t>(m.first) + m.count), field, static_cast<long long>(rows));
            const int64_t len = static_cast<int64_t>(m.count) * width;
            if (len > INT32_MAX) fail(VB200_ERR_INVALID, "%s: message %d has a segment of %lld logits", api, i, static_cast<long long>(len));
            if (m.top_n < 1 || m.top_n > VB200_DECODE_MAX_TOP || m.top_n > len)
                fail(VB200_ERR_INVALID, "%s: message %d has top_n %d outside [1, %lld] (segment of %lld logits, at most %d)", api, i, m.top_n,
                     static_cast<long long>(std::min<int64_t>(len, VB200_DECODE_MAX_TOP)), static_cast<long long>(len), VB200_DECODE_MAX_TOP);
            d[i].src = src + static_cast<size_t>(m.first) * width;
            d[i].spatials = grounding ? spatials + static_cast<size_t>(m.first) * 5 : nullptr;
            d[i].image_w = m.image_w;
            d[i].image_h = m.image_h;
            d[i].len = static_cast<int>(len);
            d[i].top_n = m.top_n;
        }
        return d;
    }
    // descriptors -> dec_ws through dec_in (in stream order), then the decode kernel writes answers [n]
    void decode_answers(const std::vector<vb::DecodeDesc>& d, vb200_answer* answers, cudaStream_t st) {
        CUDA_CHECK(vb::launch_answer_decode(stage_decode(d, st), static_cast<int>(d.size()), answers, st));
        dec_ws.release(st);
    }
    // the caller releases dec_ws after its last decode kernel
    template <typename Desc>
    const Desc* stage_decode(const std::vector<Desc>& d, cudaStream_t st) {
        const size_t bytes = d.size() * sizeof(Desc);
        char* dst = dec_ws.acquire(bytes, st);
        dec_in.stage(bytes, st, [&](char* h, const auto& put) { memcpy(h, d.data(), bytes); put(dst, 0, bytes); });
        return reinterpret_cast<const Desc*>(dst);
    }
    // ---- attention relevance: lengths and the map selection are checked, and the descriptors built, before anything is enqueued
    void attention_relevance(const float* maps, int batch, const int32_t* n_tokens, const int32_t* n_regions, int packed,
                             float* relevance, cudaStream_t st) {
        const char* api = "vb200_attention_relevance";
        if (maps == nullptr || relevance == nullptr) fail(VB200_ERR_INVALID, "%s: attention_probs / relevance is NULL", api);
        if (n_tokens == nullptr || n_regions == nullptr) fail(VB200_ERR_INVALID, "%s: n_tokens / n_regions is NULL", api);
        if (packed != 0 && packed != 1) fail(VB200_ERR_INVALID, "%s: packed must be 0 or 1 (got %d)", api, packed);
        if (batch < 1) fail(VB200_ERR_INVALID, "%s: batch must be positive", api);
        const std::vector<int> kinds = attention_kinds(schedule);
        for (int e = 0; e < static_cast<int>(kinds.size()); ++e)
            if (!attn_sel.has(e))
                fail(VB200_ERR_INVALID, "%s: attention entry %d is not selected (\"attention_entries\"); the rollout needs every entry", api, e);
        // a dense batch is a packed one whose samples all have the padded lengths: the same validation, and the same layout
        // (entry e's offset sum_{e' < e} B heads Lq Lk, sample b's block at heads * b Lq Lk)
        std::vector<int32_t> tin, nv;
        if (!packed) { tin.assign(batch, *n_tokens); nv.assign(batch, *n_regions); }
        const PackedBatch b = pack_batch(api, cfg, schedule, {"sample", batch, packed ? n_tokens : tin.data(), 0,
                                                              packed ? n_regions : nv.data(), 0}, nullptr, max_rows);
        const PackedAttnLayout l = packed_attn_layout(cfg, schedule, attn_sel, batch, b.offs_t(), b.offs_v());
        const size_t n = l.offset.size(), n1 = static_cast<size_t>(batch) + 1;
        std::vector<vb::RelevanceEntry> ents(n);
        for (size_t e = 0; e < n; ++e) ents[e] = {l.offset[e], l.kind[e], l.heads[e]};
        std::vector<vb::RelevanceSample> smp(batch);
        int64_t out = 0;
        int max_cols = 0;
        for (int i = 0; i < batch; ++i) {
            const int T = b.offs_t()[i + 1] - b.offs_t()[i], V = b.offs_v()[i + 1] - b.offs_v()[i];
            smp[i] = {{l.prefix[i], l.prefix[n1 + i], l.prefix[2 * n1 + i]}, out, T, V};
            out += 2 * static_cast<int64_t>(T + V);
            max_cols = std::max(max_cols, T + V);
        }
        // stage entries then samples (both 8-byte aligned) in one copy, in stream order
        const size_t eb = n * sizeof(vb::RelevanceEntry), bytes = eb + smp.size() * sizeof(vb::RelevanceSample);
        char* dst = rel_ws.acquire(bytes, st);
        rel_in.stage(bytes, st, [&](char* h, const auto& put) {
            memcpy(h, ents.data(), eb);
            memcpy(h + eb, smp.data(), bytes - eb);
            put(dst, 0, bytes);
        });
        CUDA_CHECK(vb::launch_attention_relevance(maps, reinterpret_cast<const vb::RelevanceEntry*>(dst), static_cast<int>(n),
                                                  reinterpret_cast<const vb::RelevanceSample*>(dst + eb), batch, max_cols, relevance, st));
        rel_ws.release(st);
    }
    // ---- answer, message, head and coalition ablation.  Every entry point converts its messages to AblMsgs, ablation_layout
    // describes every variant (AblLayout) and run_ablation runs them: one packed forward of every variant's samples, one segment
    // gather, one scoring.
    // The rejections every ablation call shares: the batch's pointers, mask_token, slot and the length rules of
    // vb200_forward_regions_packed on the samples (every variant is no longer than its samples).  Returns the region capacity.
    int check_ablation_inputs(const char* api, const vb200_packed_region_inputs* in, int64_t mask_token, int slot) const {
        const int task = cfg.task_tokens ? 1 : 0;
        if (!in->n_tokens || !in->n_boxes || !in->question || !in->segment_ids || !in->box_features || !in->boxes || !in->image_wh ||
            (task && !in->task_tokens))
            fail(VB200_ERR_INVALID, "%s: vb200_packed_region_inputs has a NULL required pointer", api);
        if (reinterpret_cast<uintptr_t>(in->box_features) & 15) fail(VB200_ERR_INVALID, "%s: box_features is not 16-byte aligned", api);
        if (mask_token < 0 || mask_token >= cfg.vocab)
            fail(VB200_ERR_INVALID, "%s: mask_token %lld outside [0, %d)", api, static_cast<long long>(mask_token), cfg.vocab);
        if (slot < 0 || slot > 15) fail(VB200_ERR_INVALID, "%s: slot %d out of range (0..15)", api, slot);
        if (slot > 0 && !opt.use_cuda_graph) fail(VB200_ERR_INVALID, "%s: concurrent slots need CUDA-graph plans (use_cuda_graph)", api);
        const BoxRows v = box_rows(api, in->batch, in->n_boxes, in->max_boxes, max_rows);
        for (int i = 0; i < in->batch; ++i)
            if (in->n_tokens[i] + task > max_rows)
                fail(VB200_ERR_INVALID, "%s: image %d has n_tokens %d (T = n_tokens + 1 must be <= %d)", api, i, in->n_tokens[i], max_rows);
        pack_batch(api, cfg, schedule, {"image", in->batch, in->n_tokens, in->max_tokens, v.v.data(), v.max_regions}, nullptr, max_rows);
        return v.max_regions;
    }
    // One variant: its layout record, where its segment is gathered from (seg.dst = rec.offset), and its score -- against the
    // message's unablated variant `base`, index `column`, without segment row `drop` (-1: none).
    struct AblVariant { vb200_ablation_variant rec; vb::SegmentDesc seg; int base, column, drop; };
    // The variants in layout order and the forward samples they run: text and image sources, lengths.  NLVR2 variants take the first
    // samples, two each, so every pair starts on an even sample with no filler.
    struct AblLayout {
        std::vector<AblVariant> v;
        std::vector<vb::TextSrc> text;
        std::vector<vb::RegionSrc> img;
        std::vector<uint32_t> mask;    // masked-position bitmaps, one word-aligned run per masked question (TextSrc::masked)
        std::vector<int32_t> kept;     // kept-box lists, one run per reduced image (RegionSrc::kept)
        std::vector<int32_t> tin, nv;
        std::vector<int32_t> gate;     // head ablation: per sample the gate table element (entry * gate_heads + head) set to 0, or -1
        int64_t n_floats = 0;
        bool grounding = false;
        bool gated = false;            // head ablation: the samples run the gated plan
    };
    // One message of any ablation kind: its family, images and answer; the positions [token_begin, token_end) and boxes [box_begin,
    // box_end) it masks and drops one at a time (answer and message ablation); the attention entries [entry_begin, entry_end) whose
    // heads it gates one at a time (head ablation); and its units and coalitions (coalition ablation, else null).
    struct AblMsg {
        int family, image_begin, n_images, answer;
        int token_begin, token_end, box_begin, box_end;
        int entry_begin, entry_end;
        const vb200_coalition_message* coal;
    };
    static AblMsg abl_msg(int family, int sample, const vb200_ablation_msg& a) {
        return {family, sample, 1, a.answer, a.token_begin, a.token_end, a.box_begin, a.box_end, 0, 0, nullptr};
    }
    static AblMsg abl_msg(const vb200_ablation_message& m) {
        return {m.family, m.image_begin, m.n_images, m.answer, m.token_begin, m.token_end, m.box_begin, m.box_end, 0, 0, nullptr};
    }
    static AblMsg abl_msg(const vb200_head_ablation_message& m) {
        return {m.family, m.image_begin, m.n_images, m.answer, 0, 0, 0, 0, m.entry_begin, m.entry_end, nullptr};
    }
    static AblMsg abl_msg(const vb200_coalition_message& m) { return {m.family, m.image_begin, m.n_images, m.answer, 0, 0, 0, 0, 0, 0, &m}; }
    template <typename M>
    static std::vector<AblMsg> abl_msgs(const char* api, const M* msgs, int n_msgs) {
        if (msgs == nullptr) fail(VB200_ERR_INVALID, "%s: msgs is NULL", api);
        if (n_msgs < 1) fail(VB200_ERR_INVALID, "%s: n_msgs must be positive (n_msgs = %d)", api, n_msgs);
        std::vector<AblMsg> m;
        for (int i = 0; i < n_msgs; ++i) m.push_back(abl_msg(msgs[i]));
        return m;
    }
    // Coalition message i's units and coalitions checked against its question length T and box count nb; pos_unit / box_unit get
    // each position's and box's unit (-1: in none).
    static void check_coalitions(const char* api, int i, const vb200_coalition_message& c, int T, int nb, std::vector<int>& pos_unit,
                                 std::vector<int>& box_unit) {
        if (c.family == VB200_DECODE_GROUNDING)
            fail(VB200_ERR_INVALID, "%s: message %d is a grounding message (its answer is a box, which a coalition would renumber)", api, i);
        if (c.n_units < 1 || c.n_units > VB200_COALITION_MAX_UNITS)
            fail(VB200_ERR_INVALID, "%s: message %d has n_units %d outside [1, %d]", api, i, c.n_units, VB200_COALITION_MAX_UNITS);
        if (c.n_coalitions < 0) fail(VB200_ERR_INVALID, "%s: message %d has n_coalitions %d (must be >= 0)", api, i, c.n_coalitions);
        if (!c.position_offsets || !c.box_offsets || (c.n_coalitions > 0 && !c.coalitions))
            fail(VB200_ERR_INVALID, "%s: message %d has a NULL position_offsets / box_offsets / coalitions array", api, i);
        pos_unit.assign(T, -1);
        box_unit.assign(nb, -1);
        for (int pass = 0; pass < 2; ++pass) {
            const bool text = pass == 0;
            const int32_t* offs = text ? c.position_offsets : c.box_offsets;
            const int32_t* item = text ? c.positions : c.boxes;
            std::vector<int>& owner = text ? pos_unit : box_unit;
            const char* what = text ? "position" : "box";
            if (offs[0] != 0) fail(VB200_ERR_INVALID, "%s: message %d: %s_offsets[0] is %d (must be 0)", api, i, what, offs[0]);
            for (int u = 0; u < c.n_units; ++u) {
                if (offs[u + 1] < offs[u])
                    fail(VB200_ERR_INVALID, "%s: message %d unit %d: %s_offsets decrease (%d after %d)", api, i, u, what, offs[u + 1], offs[u]);
                if (offs[u + 1] > offs[u] && item == nullptr)
                    fail(VB200_ERR_INVALID, "%s: message %d unit %d lists %ss, but the %ss array is NULL", api, i, u, what, what);
                for (int32_t k = offs[u]; k < offs[u + 1]; ++k) {
                    const int x = item[k], lim = text ? T : nb;
                    if (x < 0 || x >= lim)
                        fail(VB200_ERR_INVALID, "%s: message %d unit %d has %s %d outside [0, %d)", api, i, u, what, x, lim);
                    if (owner[x] >= 0)
                        fail(VB200_ERR_INVALID, "%s: message %d unit %d has %s %d, which unit %d already holds", api, i, u, what, x, owner[x]);
                    owner[x] = u;
                }
            }
        }
        for (int u = 0; u < c.n_units; ++u)
            if (c.position_offsets[u + 1] == c.position_offsets[u] && c.box_offsets[u + 1] == c.box_offsets[u])
                fail(VB200_ERR_INVALID, "%s: message %d unit %d is empty (no position and no box)", api, i, u);
        const size_t W = (static_cast<size_t>(c.n_units) + 63) / 64;
        const uint64_t past = c.n_units % 64 ? ~0ull << (c.n_units % 64) : 0ull;
        for (int s = 0; s < c.n_coalitions; ++s)
            if (c.coalitions[s * W + W - 1] & past)
                fail(VB200_ERR_INVALID, "%s: message %d coalition %d sets a bit at or past n_units %d", api, i, s, c.n_units);
    }
    // The messages checked against the batch's lengths and laid out; no sample cap (run_ablation applies it).  After its token and
    // box variants, each message gets one variant per head of every entry in its entry range (kind 3, unit entry * gate_heads +
    // head): the message's samples, unablated, with that one gate at 0.  A coalition message (token and box ranges empty) gets after
    // the full input one variant per coalition (kind 4, unit = its index): every sample of the message with the coalition's absent
    // units removed.  gated: the samples run the gated plan (head ablation).
    AblLayout ablation_layout(const char* api, int batch, const int32_t* n_tokens, const int32_t* n_boxes, const std::vector<AblMsg>& msgs,
                              bool gated) const {
        if (n_tokens == nullptr || n_boxes == nullptr) fail(VB200_ERR_INVALID, "%s: n_tokens / n_boxes is NULL", api);
        if (batch < 1) fail(VB200_ERR_INVALID, "%s: batch must be positive (batch = %d)", api, batch);
        const int n_msgs = static_cast<int>(msgs.size());
        std::vector<int> tok0(batch + 1, 0), box0(batch + 1, 0);
        for (int i = 0; i < batch; ++i) {
            if (n_tokens[i] < 1 || n_boxes[i] < 1)
                fail(VB200_ERR_INVALID, "%s: image %d has n_tokens %d / n_boxes %d (both must be >= 1)", api, i, n_tokens[i], n_boxes[i]);
            if (tok0[i] > INT32_MAX - n_tokens[i] || box0[i] > INT32_MAX - n_boxes[i])
                fail(VB200_ERR_INVALID, "%s: the batch's tokens or boxes overflow int32", api);
            tok0[i + 1] = tok0[i] + n_tokens[i];
            box0[i + 1] = box0[i] + n_boxes[i];
        }
        AblLayout L;
        L.gated = gated;
        std::vector<std::vector<AblVariant>> per(n_msgs);
        std::vector<int> entry_heads;
        for (int kind : attention_kinds(schedule)) entry_heads.push_back(kind == 0 ? cfg.heads : kind == 1 ? cfg.v_heads : cfg.bi_heads);
        std::vector<std::vector<int>> pos_unit(n_msgs), box_unit(n_msgs);   // a coalition message's owning units, -1: none
        // one sample: message m's question with the positions of bitmap run `masked` replaced (-1: none), image `image` with the
        // nbox boxes of kept-list run `kept` (-1: all its boxes)
        auto sample = [&](const AblMsg& m, int masked, int image, int kept = -1, int nbox = -1, int gate = -1) {
            L.gate.push_back(gate);
            L.text.push_back({tok0[m.image_begin], n_tokens[m.image_begin], masked, m.image_begin});
            L.img.push_back({image, box0[image], kept});
            L.tin.push_back(n_tokens[m.image_begin]);
            L.nv.push_back((kept < 0 ? n_boxes[image] : nbox) + 1);
            return static_cast<int>(L.text.size()) - 1;
        };
        auto mask_run = [&](int tin, const std::vector<int>& pos) {          // a bitmap run of tin bits, `pos` set
            if (pos.empty()) return -1;
            const int at = static_cast<int>(L.mask.size());
            L.mask.resize(L.mask.size() + (tin + 31) / 32, 0u);
            for (int p : pos) L.mask[at + p / 32] |= 1u << (p % 32);
            return at;
        };
        auto reduced = [&](const AblMsg& m, int masked, int image, const std::vector<int32_t>& rows) {   // `rows` kept
            if (static_cast<int>(rows.size()) == n_boxes[image]) return sample(m, masked, image);
            const int at = static_cast<int>(L.kept.size());
            L.kept.insert(L.kept.end(), rows.begin(), rows.end());
            return sample(m, masked, image, at, static_cast<int>(rows.size()));
        };
        auto without = [&](const AblMsg& m, int image, int skip) {   // image without box `skip`
            std::vector<int32_t> rows;
            for (int r = 0; r < n_boxes[image]; ++r)
                if (r != skip) rows.push_back(r);
            return reduced(m, -1, image, rows);
        };
        for (int pass = 0; pass < 2; ++pass)
            for (int i = 0; i < n_msgs; ++i) {
                const AblMsg& m = msgs[i];
                const int f = m.family, K = m.n_images, ib = m.image_begin;
                int head = 0, width = 0, images = 1;
                switch (f) {
                    case VB200_DECODE_VQA: head = kOutVqa; width = num_labels; break;
                    case VB200_DECODE_GQA: head = kOutGqa; width = gqa_labels; break;
                    case VB200_DECODE_SNLI_VE: head = kOutTri; width = 3; break;
                    case VB200_DECODE_NLVR2: head = kOutBinary; width = 2; images = 2; break;
                    case VB200_DECODE_RETRIEVAL: head = kOutVilLogit; width = K; images = 0; break;
                    case VB200_DECODE_GROUNDING: head = kOutVisionLogit; break;
                    default: fail(VB200_ERR_INVALID, "%s: message %d has unknown family %d", api, i, f);
                }
                if (pass == 0) {               // every message is checked before any sample is laid out
                    if (images ? K != images : K < 1)
                        fail(VB200_ERR_INVALID, "%s: message %d (family %d) has n_images %d (the family reads %s)", api, i, f, K,
                             images == 2 ? "2" : images ? "1" : ">= 1");
                    if (ib < 0 || ib > batch - K)
                        fail(VB200_ERR_INVALID, "%s: message %d has images [%d, %lld) outside the batch of %d", api, i, ib,
                             static_cast<long long>(ib) + K, batch);
                    const int len = f == VB200_DECODE_GROUNDING ? n_boxes[ib] + 1 : width;
                    if (len < 1) fail(VB200_ERR_INVALID, "%s: message %d: family %d's head has no columns on this engine", api, i, f);
                    if (m.answer < -1 || m.answer >= len)
                        fail(VB200_ERR_INVALID, "%s: message %d has answer %d outside [-1, %d)", api, i, m.answer, len);
                    const int T = n_tokens[ib], nb = box0[ib + K] - box0[ib];
                    if (m.token_begin < 0 || m.token_begin > m.token_end || m.token_end > T)
                        fail(VB200_ERR_INVALID, "%s: message %d has the token range [%d, %d), reversed or outside [0, %d]", api, i,
                             m.token_begin, m.token_end, T);
                    if (m.box_begin < 0 || m.box_begin > m.box_end || m.box_end > nb)
                        fail(VB200_ERR_INVALID, "%s: message %d has the box range [%d, %d), reversed or outside [0, %d]", api, i,
                             m.box_begin, m.box_end, nb);
                    for (int k = 0; k < K; ++k)
                        if (n_boxes[ib + k] < 2 && m.box_begin < box0[ib + k + 1] - box0[ib] && m.box_end > box0[ib + k] - box0[ib])
                            fail(VB200_ERR_INVALID, "%s: message %d drops a box of its image %d, which has %d box (box ablation needs >= 2)",
                                 api, i, k, n_boxes[ib + k]);
                    if (m.entry_begin < 0 || m.entry_begin > m.entry_end || m.entry_end > static_cast<int>(entry_heads.size()))
                        fail(VB200_ERR_INVALID, "%s: message %d has the entry range [%d, %d), reversed or outside [0, %d]", api, i,
                             m.entry_begin, m.entry_end, static_cast<int>(entry_heads.size()));
                    if (m.coal != nullptr) check_coalitions(api, i, *m.coal, T, nb, pos_unit[i], box_unit[i]);
                }
                if ((f == VB200_DECODE_NLVR2) != (pass == 0)) continue;
                std::vector<AblVariant>& out = per[i];
                // kind, unit, samples, segment (row: the first sample's head row; a grounding one's vision row is set below), drop
                auto variant = [&](int kind, int unit, int samples, vb::SegmentDesc seg, int drop) {
                    out.push_back({{i, kind, unit, samples, 0, seg.len}, seg, 0, m.answer, drop});
                };
                auto seg = [&](int first) -> vb::SegmentDesc {
                    if (f == VB200_DECODE_NLVR2) return {head, first / 2, 2, -1, 0, 0};
                    if (f == VB200_DECODE_GROUNDING) return {head, first, L.nv[first], -1, 0, 0};
                    return {head, first, width, -1, 0, 0};
                };
                auto all_images = [&](int masked, int gate = -1) {
                    const int first = sample(m, masked, ib, -1, -1, gate);
                    for (int k = 1; k < K; ++k) sample(m, masked, ib + k, -1, -1, gate);
                    return first;
                };
                const int base = all_images(-1);
                variant(0, -1, K, seg(base), -1);
                for (int p = m.token_begin; p < m.token_end; ++p) {
                    const int first = all_images(mask_run(n_tokens[ib], {p}));
                    variant(1, p, K, seg(first), -1);
                }
                for (int u = m.box_begin; u < m.box_end; ++u) {
                    int k = 0;
                    while (box0[ib + k + 1] - box0[ib] <= u) ++k;
                    const int j = u - (box0[ib + k] - box0[ib]);
                    if (f == VB200_DECODE_NLVR2) {
                        const int first = k == 0 ? without(m, ib, j) : sample(m, -1, ib);
                        if (k == 1) without(m, ib + 1, j); else sample(m, -1, ib + 1);
                        variant(2, u, 2, seg(first), -1);
                    } else if (f == VB200_DECODE_RETRIEVAL) {     // the unablated segment, element k from the changed image alone
                        vb::SegmentDesc s = seg(base);
                        s.sub = k;
                        s.sub_row = without(m, ib + k, j);
                        variant(2, u, 1, s, -1);
                    } else {
                        const int first = without(m, ib, j);
                        variant(2, u, 1, seg(first), f == VB200_DECODE_GROUNDING ? j + 1 : -1);
                    }
                }
                for (int e = m.entry_begin; e < m.entry_end; ++e)
                    for (int h = 0; h < entry_heads[e]; ++h) {
                        const int unit = e * gate_heads() + h;
                        variant(3, unit, K, seg(all_images(-1, unit)), -1);
                    }
                if (m.coal != nullptr) {
                    const vb200_coalition_message& c = *m.coal;
                    const size_t W = (static_cast<size_t>(c.n_units) + 63) / 64;
                    for (int s = 0; s < c.n_coalitions; ++s) {
                        const uint64_t* bits = c.coalitions + s * W;
                        auto absent = [&](int unit) { return unit >= 0 && !((bits[unit >> 6] >> (unit & 63)) & 1u); };
                        std::vector<int> masked;
                        for (int t = 0; t < n_tokens[ib]; ++t)
                            if (absent(pos_unit[i][t])) masked.push_back(t);
                        const int mw = mask_run(n_tokens[ib], masked);
                        int first = -1;
                        for (int k = 0; k < K; ++k) {
                            const int b0 = box0[ib + k] - box0[ib];
                            std::vector<int32_t> rows;
                            for (int r = 0; r < n_boxes[ib + k]; ++r)
                                if (!absent(box_unit[i][b0 + r])) rows.push_back(r);
                            const int x = reduced(m, mw, ib + k, rows);
                            if (k == 0) first = x;
                        }
                        variant(4, s, K, seg(first), -1);
                    }
                }
                L.grounding |= f == VB200_DECODE_GROUNDING;
            }
        std::vector<int64_t> vrow(L.nv.size() + 1, 0);       // each sample's first vision_logit row
        for (size_t s = 0; s < L.nv.size(); ++s) vrow[s + 1] = vrow[s] + L.nv[s];
        for (int i = 0; i < n_msgs; ++i) {
            const int base = static_cast<int>(L.v.size());
            for (AblVariant a : per[i]) {
                if (msgs[i].family == VB200_DECODE_GROUNDING) a.seg.row = static_cast<int32_t>(vrow[a.seg.row]);
                a.rec.offset = a.seg.dst = L.n_floats;
                a.base = base;
                L.n_floats += a.rec.length;
                L.v.push_back(a);
            }
        }
        return L;
    }
    // Every sample of L as one PACKED forward (rounded up to a multiple of 64 with fillers: sample 0's first token and box), each
    // variant's segment gathered into variant_logits, and with scores one score per variant.  abl_ws holds the sample and segment
    // descriptors (staged through abl_in) and the samples' text ids.
    void run_ablation(const char* api, const vb200_packed_region_inputs* in, AblLayout L, int max_regions, int64_t mask_token,
                      float* variant_logits, vb200_ablation_score* scores, int slot, cudaStream_t st) {
        const int64_t count = static_cast<int64_t>(L.text.size());
        if (count > VB200_ABLATION_MAX_VARIANTS)
            fail(VB200_ERR_INVALID, "%s: the variants run %lld forward samples, above %d (split the messages across calls)", api,
                 static_cast<long long>(count), VB200_ABLATION_MAX_VARIANTS);
        const int task = cfg.task_tokens ? 1 : 0;
        const int n_pad = static_cast<int>((count + 63) / 64 * 64), n_var = static_cast<int>(L.v.size());
        for (int64_t s = count; s < n_pad; ++s) {
            L.text.push_back({0, 1, -1, 0});
            L.img.push_back({0, 0, -1});
            L.tin.push_back(1);
            L.nv.push_back(2);
            L.gate.push_back(-1);
        }
        std::vector<vb::SegmentDesc> seg(n_var);
        for (int k = 0; k < n_var; ++k) seg[k] = L.v[k].seg;
        const int64_t sum_tin = std::accumulate(L.tin.begin(), L.tin.end(), int64_t{0});

        size_t at = 0;
        auto carve = [&](size_t bytes) { const size_t a = at; at += (bytes + 255) / 256 * 256; return a; };
        const size_t o_text = carve(n_pad * sizeof(vb::TextSrc)), o_img = carve(n_pad * sizeof(vb::RegionSrc));
        const size_t o_seg = carve(n_var * sizeof(vb::SegmentDesc));
        const size_t o_gate = L.gated ? carve(n_pad * sizeof(int32_t)) : 0;
        const size_t o_mask = carve(L.mask.size() * sizeof(uint32_t)), o_kept = carve(L.kept.size() * sizeof(int32_t)), staged = at;
        const size_t o_q = carve(sum_tin * 8), o_ids = carve(sum_tin * 8), o_task = carve(static_cast<size_t>(n_pad) * 8);
        CUDA_CHECK(cudaSetDevice(opt.device));
        char* ws = abl_ws.acquire(at, st);
        abl_in.stage(staged, st, [&](char* h, const auto& put) {
            memcpy(h + o_text, L.text.data(), n_pad * sizeof(vb::TextSrc));
            memcpy(h + o_img, L.img.data(), n_pad * sizeof(vb::RegionSrc));
            memcpy(h + o_seg, seg.data(), n_var * sizeof(vb::SegmentDesc));
            if (L.gated) memcpy(h + o_gate, L.gate.data(), n_pad * sizeof(int32_t));
            if (!L.mask.empty()) memcpy(h + o_mask, L.mask.data(), L.mask.size() * sizeof(uint32_t));
            if (!L.kept.empty()) memcpy(h + o_kept, L.kept.data(), L.kept.size() * sizeof(int32_t));
            put(ws, 0, staged);
        });
        const auto* text_d = reinterpret_cast<const vb::TextSrc*>(ws + o_text);
        const auto* img_d = reinterpret_cast<const vb::RegionSrc*>(ws + o_img);
        int64_t *q = reinterpret_cast<int64_t*>(ws + o_q), *ids = reinterpret_cast<int64_t*>(ws + o_ids);
        int64_t* tk = reinterpret_cast<int64_t*>(ws + o_task);
        // the pooled task heads always, vision_logit for a grounding message: at most two plans per bucket and capacities
        const uint32_t select = VB200_OUT_VIL_PREDICTION | VB200_OUT_VIL_PREDICTION_GQA | VB200_OUT_VIL_LOGIT | VB200_OUT_VIL_BINARY_PREDICTION |
                                VB200_OUT_VIL_TRI_PREDICTION | (L.grounding ? VB200_OUT_VISION_LOGIT : 0u);
        const vb200_outputs none{};                   // the segments are gathered from the plan's heads, not copied out
        const Plan& pl = run_packed(api, PACKED, {"variant", n_pad, L.tin.data(), in->max_tokens, L.nv.data(), max_regions}, select, slot,
                                    &none, {}, st, [&](Plan& p, const PackedBatch& b, cudaStream_t s) {
            CUDA_CHECK(vb::launch_variant_text(text_d, n_pad, p.offs_t(), task, in->question, in->segment_ids, in->task_tokens, mask_token,
                                               q, ids, tk, s, reinterpret_cast<const uint32_t*>(ws + o_mask)));
            embed_text(p, q, ids, nullptr, tk, b.rows_t(), s);
            pack_regions_packed(p, in->box_features, in->boxes, in->image_wh, nullptr, b.rows_v(), s, img_d,
                                reinterpret_cast<const int32_t*>(ws + o_kept));
            if (L.gated)
                CUDA_CHECK(vb::launch_gate_rows(reinterpret_cast<const int32_t*>(ws + o_gate), n_pad, p.gate_entries * p.gate_heads, p.gate, s));
        }, nullptr, L.gated);
        vb::SegmentHeads heads{};
        for (int h = 0; h < vb::kSegmentHeads; ++h) {
            heads.p[h] = pl.outs[h].p;
            heads.ld[h] = pl.outs[h].ld;
            heads.cols[h] = pl.outs[h].cols;
        }
        CUDA_CHECK(vb::launch_segment_gather(reinterpret_cast<const vb::SegmentDesc*>(ws + o_seg), n_var, heads, variant_logits, st));
        abl_ws.release(st);
        if (scores != nullptr) {
            std::vector<vb::DecodeDesc> d(n_var);
            for (int k = 0; k < n_var; ++k) {
                const AblVariant& a = L.v[k];
                d[k].src = variant_logits + a.rec.offset;
                d[k].len = a.rec.length;
                d[k].top_n = 1;
                d[k].ref = variant_logits + L.v[a.base].rec.offset;
                d[k].score = scores + k;
                d[k].column = a.column;
                d[k].drop = a.drop;
            }
            CUDA_CHECK(vb::launch_answer_decode(stage_decode(d, st), n_var, nullptr, st));
            dec_ws.release(st);
        }
    }
    // The four run entry points: the rejections they share, then the call's messages (messages(), which checks them in the entry
    // point's own terms where it has any), laid out and run.
    template <typename Messages>
    void ablate(const char* api, const vb200_packed_region_inputs* in, const void* msgs, bool gated, int64_t mask_token, float* variant_logits,
                vb200_ablation_score* scores, int slot, cudaStream_t st, Messages messages) {
        if (in == nullptr || msgs == nullptr || variant_logits == nullptr) fail(VB200_ERR_INVALID, "%s: in / msgs / variant_logits is NULL", api);
        if (x3) fail(VB200_ERR_INVALID, "%s: packed batches are not supported in split_fp32 (fp32x) mode", api);
        if (pretraining) fail(VB200_ERR_INVALID, "%s: a pre-training engine has no task head to attribute an answer of", api);
        if (reinterpret_cast<uintptr_t>(variant_logits) & 3) fail(VB200_ERR_INVALID, "%s: variant_logits is not 4-byte aligned", api);
        if (reinterpret_cast<uintptr_t>(scores) & 3) fail(VB200_ERR_INVALID, "%s: scores is not 4-byte aligned", api);
        const int max_regions = check_ablation_inputs(api, in, mask_token, slot);
        run_ablation(api, in, ablation_layout(api, in->batch, in->n_tokens, in->n_boxes, messages(), gated), max_regions, mask_token,
                     variant_logits, scores, slot, st);
    }
    // The three layout entry points: the layout's records (variants NULL: none) and totals.
    template <typename M>
    void layout(const char* api, int batch, const int32_t* n_tokens, const int32_t* n_boxes, const M* msgs, int n_msgs, bool gated,
                vb200_ablation_variant* variants, int64_t* n_variants, int64_t* n_floats, int64_t* n_samples) const {
        if (n_variants == nullptr || n_floats == nullptr || n_samples == nullptr)
            fail(VB200_ERR_INVALID, "%s: n_variants / n_floats / n_samples is NULL", api);
        if (pretraining) fail(VB200_ERR_INVALID, "%s: a pre-training engine has no task head to attribute an answer of", api);
        const AblLayout L = ablation_layout(api, batch, n_tokens, n_boxes, abl_msgs(api, msgs, n_msgs), gated);
        if (variants != nullptr)
            for (size_t k = 0; k < L.v.size(); ++k) variants[k] = L.v[k].rec;
        *n_variants = static_cast<int64_t>(L.v.size());
        *n_floats = L.n_floats;
        *n_samples = static_cast<int64_t>(L.text.size());
    }
    // vb200_answer_ablation: one single-image message of `family` per sample, checked in the samples' terms first
    void answer_ablation(const vb200_packed_region_inputs* in, const vb200_ablation_msg* msgs, int family, int64_t mask_token,
                         float* variant_logits, vb200_ablation_score* scores, int slot, cudaStream_t st) {
        const char* api = "vb200_answer_ablation";
        ablate(api, in, msgs, false, mask_token, variant_logits, scores, slot, st, [&] {
            int width = 0;
            switch (family) {
                case VB200_DECODE_VQA: width = num_labels; break;
                case VB200_DECODE_GQA: width = gqa_labels; break;
                case VB200_DECODE_SNLI_VE: width = 3; break;
                case VB200_DECODE_NLVR2: fail(VB200_ERR_INVALID, "%s: family NLVR2 is not supported (an answer reads two images)", api);
                case VB200_DECODE_RETRIEVAL:
                    fail(VB200_ERR_INVALID, "%s: family retrieval is not supported (an answer ranks many images)", api);
                case VB200_DECODE_GROUNDING:
                    fail(VB200_ERR_INVALID, "%s: family grounding is not supported (the answer is a box a variant may remove)", api);
                default: fail(VB200_ERR_INVALID, "%s: unknown family %d", api, family);
            }
            if (width < 1) fail(VB200_ERR_INVALID, "%s: family %d's head has no columns on this engine", api, family);
            std::vector<AblMsg> m;
            int64_t count = 0;
            for (int i = 0; i < in->batch; ++i) {
                const vb200_ablation_msg& a = msgs[i];
                const int T = in->n_tokens[i], nb = in->n_boxes[i];
                if (a.answer < -1 || a.answer >= width)
                    fail(VB200_ERR_INVALID, "%s: sample %d has answer %d outside [-1, %d)", api, i, a.answer, width);
                if (a.token_begin < 0 || a.token_begin > a.token_end || a.token_end > T)
                    fail(VB200_ERR_INVALID, "%s: sample %d has the token range [%d, %d), reversed or outside [0, %d]", api, i,
                         a.token_begin, a.token_end, T);
                if (a.box_begin < 0 || a.box_begin > a.box_end || a.box_end > nb)
                    fail(VB200_ERR_INVALID, "%s: sample %d has the box range [%d, %d), reversed or outside [0, %d]", api, i, a.box_begin,
                         a.box_end, nb);
                if (a.box_end > a.box_begin && nb < 2)
                    fail(VB200_ERR_INVALID, "%s: sample %d drops a box of an image with %d box (box ablation needs >= 2)", api, i, nb);
                count += 1 + (a.token_end - a.token_begin) + (a.box_end - a.box_begin);
                if (count > VB200_ABLATION_MAX_VARIANTS)
                    fail(VB200_ERR_INVALID, "%s: the variants of samples 0..%d number %lld, above %d (split the ranges across calls)", api,
                         i, static_cast<long long>(count), VB200_ABLATION_MAX_VARIANTS);
                m.push_back(abl_msg(family, i, a));
            }
            return m;
        });
    }
    void message_ablation(const vb200_packed_region_inputs* in, const vb200_ablation_message* msgs, int n_msgs, int64_t mask_token,
                          float* variant_logits, vb200_ablation_score* scores, int slot, cudaStream_t st) {
        const char* api = "vb200_message_ablation";
        ablate(api, in, msgs, false, mask_token, variant_logits, scores, slot, st, [&] { return abl_msgs(api, msgs, n_msgs); });
    }
    void message_ablation_layout(int batch, const int32_t* n_tokens, const int32_t* n_boxes, const vb200_ablation_message* msgs, int n_msgs,
                                 vb200_ablation_variant* variants, int64_t* n_variants, int64_t* n_floats, int64_t* n_samples) const {
        layout("vb200_message_ablation_layout", batch, n_tokens, n_boxes, msgs, n_msgs, false, variants, n_variants, n_floats, n_samples);
    }
    // head ablation masks no position: mask_token 0 is any valid token id
    void head_ablation(const vb200_packed_region_inputs* in, const vb200_head_ablation_message* msgs, int n_msgs, float* variant_logits,
                       vb200_ablation_score* scores, int slot, cudaStream_t st) {
        const char* api = "vb200_head_ablation";
        ablate(api, in, msgs, true, 0, variant_logits, scores, slot, st, [&] { return abl_msgs(api, msgs, n_msgs); });
    }
    void head_ablation_layout(int batch, const int32_t* n_tokens, const int32_t* n_boxes, const vb200_head_ablation_message* msgs, int n_msgs,
                              vb200_ablation_variant* variants, int64_t* n_variants, int64_t* n_floats, int64_t* n_samples) const {
        layout("vb200_head_ablation_layout", batch, n_tokens, n_boxes, msgs, n_msgs, true, variants, n_variants, n_floats, n_samples);
    }
    void coalition_ablation(const vb200_packed_region_inputs* in, const vb200_coalition_message* msgs, int n_msgs, int64_t mask_token,
                            float* variant_logits, vb200_ablation_score* scores, int slot, cudaStream_t st) {
        const char* api = "vb200_coalition_ablation";
        ablate(api, in, msgs, false, mask_token, variant_logits, scores, slot, st, [&] { return abl_msgs(api, msgs, n_msgs); });
    }
    void coalition_ablation_layout(int batch, const int32_t* n_tokens, const int32_t* n_boxes, const vb200_coalition_message* msgs, int n_msgs,
                                   vb200_ablation_variant* variants, int64_t* n_variants, int64_t* n_floats, int64_t* n_samples) const {
        layout("vb200_coalition_ablation_layout", batch, n_tokens, n_boxes, msgs, n_msgs, false, variants, n_variants, n_floats, n_samples);
    }
    // vb200_shapley_values: every descriptor is checked before anything is enqueued
    void shapley_values(const vb200_shapley_message* msgs, int n_msgs, const int32_t* perm, const float* values, float* phi, float* se,
                        cudaStream_t st) {
        const char* api = "vb200_shapley_values";
        if (msgs == nullptr || perm == nullptr || values == nullptr || phi == nullptr || se == nullptr)
            fail(VB200_ERR_INVALID, "%s: msgs / perm / values / phi / stderr is NULL", api);
        if (n_msgs < 1) fail(VB200_ERR_INVALID, "%s: n_msgs must be positive (n_msgs = %d)", api, n_msgs);
        if ((reinterpret_cast<uintptr_t>(perm) | reinterpret_cast<uintptr_t>(values) | reinterpret_cast<uintptr_t>(phi) |
             reinterpret_cast<uintptr_t>(se)) & 3)
            fail(VB200_ERR_INVALID, "%s: perm / values / phi / stderr is not 4-byte aligned", api);
        std::vector<vb::ShapleyDesc> d(n_msgs);
        for (int i = 0; i < n_msgs; ++i) {
            const vb200_shapley_message& m = msgs[i];
            if (m.n_units < 1 || m.n_units > VB200_COALITION_MAX_UNITS)
                fail(VB200_ERR_INVALID, "%s: message %d has n_units %d outside [1, %d]", api, i, m.n_units, VB200_COALITION_MAX_UNITS);
            if (m.n_perm < 1) fail(VB200_ERR_INVALID, "%s: message %d has n_perm %d (must be >= 1)", api, i, m.n_perm);
            if (m.group != 1 && m.group != 2) fail(VB200_ERR_INVALID, "%s: message %d has group %d (1 or 2)", api, i, m.group);
            if (m.n_perm % m.group) fail(VB200_ERR_INVALID, "%s: message %d has n_perm %d, not a multiple of group %d", api, i, m.n_perm, m.group);
            if (m.perm_offset < 0 || m.value_offset < 0 || m.out_offset < 0)
                fail(VB200_ERR_INVALID, "%s: message %d has a negative offset", api, i);
            d[i] = {perm + m.perm_offset, values + m.value_offset, phi + m.out_offset, se + m.out_offset, m.n_units, m.n_perm, m.group};
        }
        CUDA_CHECK(cudaSetDevice(opt.device));
        CUDA_CHECK(vb::launch_shapley_values(stage_decode(d, st), n_msgs, st));
        dec_ws.release(st);
    }
    // vb200_interaction_values: every descriptor and pair is checked before anything is enqueued; the pairs follow the descriptors in
    // one staged copy
    void interaction_values(const vb200_interaction_message* msgs, int n_msgs, const int32_t* perm, const float* values, float* inter,
                            float* se, cudaStream_t st) {
        const char* api = "vb200_interaction_values";
        if (msgs == nullptr || perm == nullptr || values == nullptr || inter == nullptr || se == nullptr)
            fail(VB200_ERR_INVALID, "%s: msgs / perm / values / inter / stderr is NULL", api);
        if (n_msgs < 1) fail(VB200_ERR_INVALID, "%s: n_msgs must be positive (n_msgs = %d)", api, n_msgs);
        if ((reinterpret_cast<uintptr_t>(perm) | reinterpret_cast<uintptr_t>(values) | reinterpret_cast<uintptr_t>(inter) |
             reinterpret_cast<uintptr_t>(se)) & 3)
            fail(VB200_ERR_INVALID, "%s: perm / values / inter / stderr is not 4-byte aligned", api);
        std::vector<vb::InteractionDesc> d(n_msgs);
        int64_t total = 0;
        int max_pairs = 0;
        for (int i = 0; i < n_msgs; ++i) {
            const vb200_interaction_message& m = msgs[i];
            if (m.n_units < 2 || m.n_units > VB200_COALITION_MAX_UNITS)
                fail(VB200_ERR_INVALID, "%s: message %d has n_units %d outside [2, %d]", api, i, m.n_units, VB200_COALITION_MAX_UNITS);
            if (m.n_perm < 1) fail(VB200_ERR_INVALID, "%s: message %d has n_perm %d (must be >= 1)", api, i, m.n_perm);
            if (m.group != 1 && m.group != 2) fail(VB200_ERR_INVALID, "%s: message %d has group %d (1 or 2)", api, i, m.group);
            if (m.n_perm % m.group) fail(VB200_ERR_INVALID, "%s: message %d has n_perm %d, not a multiple of group %d", api, i, m.n_perm, m.group);
            if (m.perm_offset < 0 || m.value_offset < 0 || m.out_offset < 0)
                fail(VB200_ERR_INVALID, "%s: message %d has a negative offset", api, i);
            if (m.n_pairs < 1) fail(VB200_ERR_INVALID, "%s: message %d has n_pairs %d (must be >= 1)", api, i, m.n_pairs);
            if (m.pairs == nullptr) fail(VB200_ERR_INVALID, "%s: message %d has NULL pairs", api, i);
            total += m.n_pairs;
            if (total > VB200_INTERACTION_MAX_PAIRS)
                fail(VB200_ERR_INVALID, "%s: the pairs of messages 0..%d number %lld, above %d (split the messages across calls)", api, i,
                     static_cast<long long>(total), VB200_INTERACTION_MAX_PAIRS);
            for (int q = 0; q < m.n_pairs; ++q) {
                const int a = m.pairs[2 * q], b = m.pairs[2 * q + 1];
                if (a < 0 || a >= m.n_units || b < 0 || b >= m.n_units)
                    fail(VB200_ERR_INVALID, "%s: message %d pair %d (%d, %d) has a unit outside [0, %d)", api, i, q, a, b, m.n_units);
                if (a == b) fail(VB200_ERR_INVALID, "%s: message %d pair %d pairs unit %d with itself", api, i, q, a);
            }
            max_pairs = std::max(max_pairs, static_cast<int>(m.n_pairs));
            d[i] = {perm + m.perm_offset, values + m.value_offset, nullptr, inter + m.out_offset, se + m.out_offset, m.n_units, m.n_perm,
                    m.group, m.n_pairs};
        }
        CUDA_CHECK(cudaSetDevice(opt.device));
        const size_t desc_bytes = d.size() * sizeof(vb::InteractionDesc), bytes = desc_bytes + static_cast<size_t>(total) * 8;
        char* dst = dec_ws.acquire(bytes, st);
        dec_in.stage(bytes, st, [&](char* h, const auto& put) {
            size_t at = desc_bytes;
            for (int i = 0; i < n_msgs; ++i) {
                d[i].pairs = reinterpret_cast<const int32_t*>(dst + at);
                memcpy(h + at, msgs[i].pairs, static_cast<size_t>(msgs[i].n_pairs) * 8);
                at += static_cast<size_t>(msgs[i].n_pairs) * 8;
            }
            memcpy(h, d.data(), desc_bytes);
            put(dst, 0, bytes);
        });
        CUDA_CHECK(vb::launch_interaction_values(reinterpret_cast<const vb::InteractionDesc*>(dst), n_msgs, max_pairs, st));
        dec_ws.release(st);
    }
    // ---- region selection: every descriptor is checked before anything is enqueued
    void select_regions(const vb200_detections* imgs, int n, const vb200_select_params* p, const vb200_selected* out, cudaStream_t st) {
        const char* api = "vb200_select_regions";
        if (imgs == nullptr || p == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "%s: imgs / p / out is NULL", api);
        if (n < 1 || n > 65535) fail(VB200_ERR_INVALID, "%s: n = %d outside [1, 65535]", api, n);
        const int C = p->n_classes, F = p->feature_size, K = p->max_boxes;
        if (C < 2 || C > 2048) fail(VB200_ERR_INVALID, "%s: n_classes = %d outside [2, 2048]", api, C);
        if (F < 4 || F % 4 != 0) fail(VB200_ERR_INVALID, "%s: feature_size = %d is not a positive multiple of 4", api, F);
        if (K < 1 || K > max_rows - 1) fail(VB200_ERR_INVALID, "%s: max_boxes = %d outside [1, %d]", api, K, max_rows - 1);
        if (!(p->nms_iou > 0.f && p->nms_iou <= 1.f)) fail(VB200_ERR_INVALID, "%s: nms_iou = %g outside (0, 1]", api, p->nms_iou);
        if (std::isnan(p->conf_thresh)) fail(VB200_ERR_INVALID, "%s: conf_thresh is NaN", api);
        if (p->background != 0 && p->background != 1) fail(VB200_ERR_INVALID, "%s: background = %d is not 0 or 1", api, p->background);
        if (p->out_rows < 1) fail(VB200_ERR_INVALID, "%s: out_rows = %d", api, p->out_rows);
        if (out->box_features == nullptr || out->boxes == nullptr || out->num_boxes == nullptr)
            fail(VB200_ERR_INVALID, "%s: box_features, boxes and num_boxes are required", api);
        if (reinterpret_cast<uintptr_t>(out->box_features) % 16 != 0) fail(VB200_ERR_INVALID, "%s: box_features is not 16-byte aligned", api);
        if (reinterpret_cast<uintptr_t>(out->boxes) % 16 != 0) fail(VB200_ERR_INVALID, "%s: boxes is not 16-byte aligned", api);
        std::vector<vb::SelectDesc> d(n);
        std::vector<std::pair<int, int>> ranges(n);        // (dst_row, image)
        size_t rows = 0, words = 0;
        int max_n = 0, max_npad = 32;
        for (int i = 0; i < n; ++i) {
            const vb200_detections& m = imgs[i];
            if (m.n_proposals < 1 || m.n_proposals > vb::kSelectMaxProposals)
                fail(VB200_ERR_INVALID, "%s: image %d has %d proposals, outside [1, %d]", api, i, m.n_proposals, vb::kSelectMaxProposals);
            if (m.proposals == nullptr || m.scores == nullptr || m.features == nullptr)
                fail(VB200_ERR_INVALID, "%s: image %d has a NULL proposals / scores / features pointer", api, i);
            if (reinterpret_cast<uintptr_t>(m.features) % 16 != 0) fail(VB200_ERR_INVALID, "%s: image %d's features are not 16-byte aligned", api, i);
            if (!(m.im_scale > 0.0) || !std::isfinite(static_cast<float>(m.im_scale)))
                fail(VB200_ERR_INVALID, "%s: image %d has im_scale %g", api, i, m.im_scale);
            const int k = std::min(K, m.n_proposals);
            if (m.dst_row < 0 || static_cast<int64_t>(m.dst_row) + k > p->out_rows)
                fail(VB200_ERR_INVALID, "%s: image %d's rows [%d, %lld) fall outside out_rows %d", api, i, m.dst_row,
                     static_cast<long long>(static_cast<int64_t>(m.dst_row) + k), p->out_rows);
            int npad = 32;
            while (npad < m.n_proposals) npad <<= 1;
            vb::SelectDesc& s = d[i];
            s.proposals = m.proposals;
            s.scores = m.scores;
            s.features = m.features;
            s.row0 = rows;
            s.mask0 = words;
            s.im_scale = static_cast<float>(m.im_scale);
            s.n = m.n_proposals;
            s.npad = npad;
            s.nw = (m.n_proposals + 31) / 32;
            s.dst_row = m.dst_row;
            s.k = k;
            rows += m.n_proposals;
            words += static_cast<size_t>(m.n_proposals) * s.nw;
            max_n = std::max(max_n, m.n_proposals);
            max_npad = std::max(max_npad, npad);
            ranges[i] = {m.dst_row, i};
        }
        std::sort(ranges.begin(), ranges.end());
        for (int r = 1; r < n; ++r) {
            const vb::SelectDesc& a = d[ranges[r - 1].second];
            if (a.dst_row + a.k > ranges[r].first)
                fail(VB200_ERR_INVALID, "%s: image %d's rows [%d, %d) overlap image %d's rows starting at %d", api, ranges[r].second,
                     ranges[r].first, ranges[r].first + d[ranges[r].second].k, ranges[r - 1].second, a.dst_row);
        }
        // workspace layout: descriptors, stats [rows] float2, dbox [rows] float4, max_conf [rows], keep [n, K], mask [words]
        auto up = [](size_t b) { return (b + 255) & ~static_cast<size_t>(255); };
        const size_t o_desc = 0, o_stats = up(o_desc + n * sizeof(vb::SelectDesc)), o_box = up(o_stats + rows * 8),
                     o_conf = up(o_box + rows * 16), o_keep = up(o_conf + rows * 4), o_mask = up(o_keep + static_cast<size_t>(n) * K * 4),
                     need = up(o_mask + words * 4);
        char* ws = sel_ws.acquire(need, st);
        vb::SelectArgs a{};
        a.C = C; a.F = F; a.K = K; a.start = p->background ? 0 : 1;
        a.thr = std::max(p->conf_thresh, 0.f);
        a.nms_iou = p->nms_iou;
        a.stats = reinterpret_cast<float2*>(ws + o_stats);
        a.dbox = reinterpret_cast<float*>(ws + o_box);
        a.max_conf = reinterpret_cast<unsigned*>(ws + o_conf);
        a.keep = reinterpret_cast<int*>(ws + o_keep);
        a.mask = reinterpret_cast<unsigned*>(ws + o_mask);
        a.box_features = out->box_features;
        a.boxes = out->boxes;
        a.num_boxes = out->num_boxes;
        a.keep_index = out->keep_index;
        a.max_conf_out = out->max_conf;
        a.cls_prob = out->cls_prob;
        a.objects = out->objects;
        const size_t db = n * sizeof(vb::SelectDesc);
        sel_in.stage(db, st, [&](char* h, const auto& put) { memcpy(h, d.data(), db); put(ws + o_desc, 0, db); });
        CUDA_CHECK(cudaMemsetAsync(a.max_conf, 0, rows * 4, st));
        CUDA_CHECK(vb::launch_select_regions(reinterpret_cast<const vb::SelectDesc*>(ws + o_desc), n, max_n, max_npad, a, st));
        sel_ws.release(st);
    }
    // ---- pre-training heads at chosen rows
    // The RowHeads of `head` for n rows: bucket M = 128 * 2^k >= n, built on its first use with the forward's head launches
    // (PlanBuilder::heads) at M rows and the device row count as their m_rows.
    RowHeads& row_heads_for(int head, int n) {
        int M = 128;
        while (M < n) M *= 2;
        std::unique_ptr<RowHeads>& slot = row_heads[head][M];
        if (slot) return *slot;
        std::unique_ptr<RowHeads> r(new RowHeads());
        Plan& pl = r->pl;
        PlanBuilder b{*this, pl, M, "pretraining heads"};
        r->M = M;
        r->d_rows = pl.mem.alloc_n<int>(2 * static_cast<size_t>(M) + 1);
        r->loss = pl.mem.alloc_n<float>(M);
        const int* count = r->d_rows;
        if (head == kHeadPair) {
            const int Hb = cfg.bi_hidden;
            float* a = b.buf32(M, Hb);
            r->a = a;
            r->logits = b.make_out(M, 2);
            b.rowdot(a, Hb, seq_rel, nullptr, r->logits, count);
        } else {
            const bool text = head == kHeadText;
            const int H = text ? cfg.hidden : cfg.v_hidden;
            const LinearW& transform = text ? lm_transform : img_transform;
            const LinearW& decoder = text ? lm_decoder : img_decoder;
            bf16* a = b.buf16(M, H);
            bf16* hid = b.buf16(M, H);
            r->a = a;
            b.y[0] = b.buf32(M, H);
            b.predict(transform, text ? lm_ln : img_ln, decoder, a, H, hid, M, count, &r->logits);
        }
        slot = std::move(r);
        return *slot;
    }
    // One head's list of a vb200_pretraining_heads / vb200_pretraining_objectives call: the fp32 state it gathers from, the rows, the
    // head's logits per row, the objectives' HOST labels (staged after the rows: token and pair heads) and whether any output reads it.
    struct HeadGroup {
        const char* list; const char* state; const float* src; int src_rows, width, n; const int32_t* rows; int N;
        const int32_t* labels; bool run;
    };
    HeadGroup head_group(int head, const vb200_pretrain_rows& in) const {
        if (head == kHeadText)
            return {"text_rows", "text_state", in.text_state, in.t_rows, cfg.hidden, in.n_t, in.text_rows, cfg.vocab, nullptr, false};
        if (head == kHeadImage)
            return {"image_rows", "image_state", in.image_state, in.v_rows, cfg.v_hidden, in.n_v, in.image_rows, cfg.v_target, nullptr, false};
        return {"pair_rows", "pooled_state", in.pooled_state, in.p_rows, cfg.bi_hidden, in.n_p, in.pair_rows, 2, nullptr, false};
    }
    static void check_group(const char* api, const HeadGroup& x) {
        if (x.n < 0 || x.n > kMaxHeadRows) fail(VB200_ERR_INVALID, "%s: %s has a count of %d (must be in [0, %d])", api, x.list, x.n, kMaxHeadRows);
        if (x.n == 0) return;
        if (x.rows == nullptr) fail(VB200_ERR_INVALID, "%s: %s is NULL for %d rows", api, x.list, x.n);
        if (x.src == nullptr) fail(VB200_ERR_INVALID, "%s: %s is NULL for a non-empty %s", api, x.state, x.list);
        if (reinterpret_cast<uintptr_t>(x.src) & 15) fail(VB200_ERR_INVALID, "%s: %s is not 16-byte aligned", api, x.state);
        for (int i = 0; i < x.n; ++i)
            if (x.rows[i] < 0 || x.rows[i] >= x.src_rows)
                fail(VB200_ERR_INVALID, "%s: %s[%d] = %d is outside the %d rows of %s", api, x.list, i, x.rows[i], x.src_rows, x.state);
    }
    // The RowHeads of every group that runs, with its count, rows and labels staged through pre_in into rh->d_rows, in stream order
    // after the previous call (any stream) is done with them.  The caller records pre_done.
    void stage_rows(const HeadGroup (&g)[3], RowHeads* (&rh)[3], cudaStream_t st) {
        size_t staged = 0;
        for (int i = 0; i < 3; ++i) {
            if (!g[i].run) continue;
            rh[i] = &row_heads_for(i, g[i].n);
            staged += 1 + static_cast<size_t>(g[i].n) * (g[i].labels ? 2 : 1);
        }
        CUDA_CHECK(cudaStreamWaitEvent(st, pre_done.get(), 0));
        pre_in.stage(staged * sizeof(int32_t), st, [&](char* hb, const auto& put) {
            int32_t* h = reinterpret_cast<int32_t*>(hb);
            size_t at = 0;
            for (int i = 0; i < 3; ++i) {
                if (rh[i] == nullptr) continue;
                const size_t n = static_cast<size_t>(g[i].n), len = 1 + n * (g[i].labels ? 2 : 1);
                h[at] = g[i].n;
                memcpy(h + at + 1, g[i].rows, n * sizeof(int32_t));
                if (g[i].labels) memcpy(h + at + 1 + n, g[i].labels, n * sizeof(int32_t));
                put(rh[i]->d_rows, at * sizeof(int32_t), len * sizeof(int32_t));
                at += len;
            }
        });
    }
    // One running group's gather and the forward's head launches: its logits land in r.logits.
    void run_row_heads(int head, const HeadGroup& x, RowHeads& r, cudaStream_t st) {
        const int rows_out = (x.n + 127) / 128 * 128;                // the rest of the last 128-row tile is zeroed
        const int mode = head == kHeadPair ? 3 : (x3 ? 2 : (opt.act_fp16 ? 1 : 0));
        const int ld = head == kHeadPair ? x.width : x.width * (x3 ? 3 : 1);
        CUDA_CHECK(vb::launch_gather_rows(x.src, r.d_rows + 1, x.n, rows_out, x.width, r.a, ld, mode, st));
        for (const Op& op : r.pl.ops) launch_op(op, st);
    }
    void pretraining_heads(const vb200_pretrain_rows* in, const vb200_pretrain_out* out, cudaStream_t st) {
        const char* api = "vb200_pretraining_heads";
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "%s: in / out is NULL", api);
        const int k = in->top_k;
        if (k < 0 || k > VB200_DECODE_MAX_TOP) fail(VB200_ERR_INVALID, "%s: top_k %d outside [0, %d]", api, k, VB200_DECODE_MAX_TOP);
        float* logits[3] = {out->token_logits, out->region_logits, out->alignment};
        vb200_answer* top[3] = {out->token_top, out->region_top, nullptr};
        const char* top_name[3] = {"token_top", "region_top", nullptr};
        HeadGroup g[3];
        bool any = false;
        for (int i = 0; i < 3; ++i) {
            g[i] = head_group(i, *in);
            if (top[i] != nullptr && k == 0) fail(VB200_ERR_INVALID, "%s: %s is requested with top_k = 0", api, top_name[i]);
            if (top[i] != nullptr && k > g[i].N)
                fail(VB200_ERR_INVALID, "%s: top_k %d is above the %d logits of a %s row", api, k, g[i].N, top_name[i]);
            check_group(api, g[i]);
            g[i].run = g[i].n > 0 && (logits[i] != nullptr || top[i] != nullptr);
            any = any || g[i].run;
        }
        if (!any) return;
        CUDA_CHECK(cudaSetDevice(opt.device));
        RowHeads* rh[3] = {nullptr, nullptr, nullptr};
        stage_rows(g, rh, st);
        std::vector<vb::DecodeDesc> descs;
        for (int i = 0; i < 3; ++i)
            if (rh[i] != nullptr && top[i] != nullptr)
                for (int r = 0; r < g[i].n; ++r)
                    descs.push_back(vb::DecodeDesc{rh[i]->logits.p + static_cast<size_t>(r) * rh[i]->logits.ld, nullptr, 0.0, 0.0, g[i].N, k});
        const vb::DecodeDesc* dd = descs.empty() ? nullptr : stage_decode(descs, st);
        for (int i = 0; i < 3; ++i) {
            if (rh[i] == nullptr) continue;
            const HeadGroup& x = g[i];
            run_row_heads(i, x, *rh[i], st);
            if (logits[i] != nullptr)
                CUDA_CHECK(cudaMemcpy2DAsync(logits[i], static_cast<size_t>(x.N) * 4, rh[i]->logits.p,
                                             static_cast<size_t>(rh[i]->logits.ld) * 4, static_cast<size_t>(x.N) * 4, x.n,
                                             cudaMemcpyDeviceToDevice, st));
            if (top[i] != nullptr) {
                CUDA_CHECK(vb::launch_answer_decode(dd, x.n, top[i], st));
                dd += x.n;
            }
        }
        if (!descs.empty()) dec_ws.release(st);
        CUDA_CHECK(cudaEventRecord(pre_done.get(), st));
    }
    // The three pre-training objectives at the listed rows: the heads of pretraining_heads, then one CTA per listed row computes its
    // loss from the compact logits and one CTA reduces each list in a fixed order.
    void pretraining_objectives(const vb200_pretrain_rows* in, const vb200_pretrain_targets* tg, const vb200_pretrain_losses* out,
                                cudaStream_t st) {
        const char* api = "vb200_pretraining_objectives";
        if (in == nullptr || tg == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "%s: in / targets / out is NULL", api);
        if (in->top_k != 0) fail(VB200_ERR_INVALID, "%s: top_k %d (the objectives rank nothing: it must be 0)", api, in->top_k);
        if (reinterpret_cast<uintptr_t>(out->reduced) & 3) fail(VB200_ERR_INVALID, "%s: reduced is not 4-byte aligned", api);
        float* per_row[3] = {out->token_loss, out->region_loss, out->pair_loss};
        HeadGroup g[3];
        for (int i = 0; i < 3; ++i) {
            g[i] = head_group(i, *in);
            check_group(api, g[i]);
            g[i].run = g[i].n > 0 && (per_row[i] != nullptr || out->reduced != nullptr);
        }
        const HeadGroup& t = g[kHeadText];
        const HeadGroup& v = g[kHeadImage];
        const HeadGroup& p = g[kHeadPair];
        if (t.n > 0) {
            if (tg->token_labels == nullptr) fail(VB200_ERR_INVALID, "%s: token_labels is NULL for %d text rows", api, t.n);
            for (int i = 0; i < t.n; ++i)
                if (tg->token_labels[i] < 0 || tg->token_labels[i] >= cfg.vocab)
                    fail(VB200_ERR_INVALID, "%s: token_labels[%d] = %d is outside [0, %d)", api, i, tg->token_labels[i], cfg.vocab);
        }
        if (v.n > 0) {
            if (tg->image_targets == nullptr) fail(VB200_ERR_INVALID, "%s: image_targets is NULL for %d image rows", api, v.n);
            if (reinterpret_cast<uintptr_t>(tg->image_targets) & 3) fail(VB200_ERR_INVALID, "%s: image_targets is not 4-byte aligned", api);
        }
        if (p.n > 0) {
            if (tg->pair_labels == nullptr) fail(VB200_ERR_INVALID, "%s: pair_labels is NULL for %d pair rows", api, p.n);
            for (int i = 0; i < p.n; ++i)
                if (tg->pair_labels[i] != 0 && tg->pair_labels[i] != 1)
                    fail(VB200_ERR_INVALID, "%s: pair_labels[%d] = %d is not 0 or 1", api, i, tg->pair_labels[i]);
        }
        if (!t.run && !v.run && !p.run && out->reduced == nullptr) return;
        g[kHeadText].labels = tg->token_labels;
        g[kHeadPair].labels = tg->pair_labels;
        CUDA_CHECK(cudaSetDevice(opt.device));
        RowHeads* rh[3] = {nullptr, nullptr, nullptr};
        stage_rows(g, rh, st);
        vb::LossRows rows[3] = {};
        for (int i = 0; i < 3; ++i) {
            if (rh[i] == nullptr) continue;
            run_row_heads(i, g[i], *rh[i], st);
            rows[i] = vb::LossRows{rh[i]->logits.p, rh[i]->logits.ld, g[i].N, g[i].n,
                                   g[i].labels ? rh[i]->d_rows + 1 + g[i].n : nullptr, i == kHeadImage ? tg->image_targets : nullptr,
                                   rh[i]->loss};
        }
        CUDA_CHECK(vb::launch_pretrain_losses(rows, out->reduced, st));
        for (int i = 0; i < 3; ++i)
            if (rh[i] != nullptr && per_row[i] != nullptr)
                CUDA_CHECK(cudaMemcpyAsync(per_row[i], rh[i]->loss, static_cast<size_t>(g[i].n) * 4, cudaMemcpyDeviceToDevice, st));
        CUDA_CHECK(cudaEventRecord(pre_done.get(), st));
    }
    // rows_t / rows_v (packed plans): the call's row totals -- the per-row outputs hold that many packed rows
    void copy_outputs(Plan& pl, const vb200_outputs& out, cudaStream_t st, cudaMemcpyKind kind, int rows_t = 0, int rows_v = 0) {
        for (int s = 0; s < kNumOuts; ++s) {
            float* dst = out.*kOutSlots[s].field;
            const OutBuf& o = pl.outs[s];
            if (dst == nullptr) continue;
            if (o.p == nullptr) fail(VB200_ERR_INVALID, "output slot %d requested but not selected in the `select` mask", s);
            int rows = o.rows;
            if (pl.packed && kOutSlots[s].rows == kImageRow) rows = rows_v;
            if (pl.packed && kOutSlots[s].rows == kTextRow) rows = rows_t;
            CUDA_CHECK(cudaMemcpy2DAsync(dst, static_cast<size_t>(o.cols) * 4, o.p, static_cast<size_t>(o.ld) * 4,
                                         static_cast<size_t>(o.cols) * 4, rows, kind, st));
        }
        // packed probabilities (layout entries) were written into out.attention_probs by the plan's kernels: nothing to copy
        if (out.attention_probs != nullptr && pl.layout.n_entries == 0) {
            if (pl.attn.empty()) fail(VB200_ERR_INVALID, "attention_probs requested but VB200_OUT_ATTENTION is not set in `select`");
            float* dst = out.attention_probs;
            for (const Plan::AttnOut& a : pl.attn) {
                const size_t n = static_cast<size_t>(pl.B) * a.heads * a.Lq * a.Lk;
                CUDA_CHECK(cudaMemcpyAsync(dst, a.p, n * 4, kind, st));
                dst += n;
            }
        }
    }
};

namespace {
int guard(vb200_handle h, const std::function<void()>& body) {
    try {
        body();
        return VB200_OK;
    } catch (const VbError& e) {
        if (h) h->last_error = e.what(); else g_create_error = e.what();
        return e.status;
    } catch (const std::exception& e) {
        if (h) h->last_error = e.what(); else g_create_error = e.what();
        return VB200_ERR_INVALID;
    }
}

void require_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        fail(VB200_ERR_NO_DEVICE, "no CUDA device visible (%s); vilbert_b200 has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= n) fail(VB200_ERR_INVALID, "device ordinal %d out of range (0..%d)", device, n - 1);
    cudaDeviceProp p;
    CUDA_CHECK(cudaGetDeviceProperties(&p, device));
    if (p.major != 9 || p.minor != 0) fail(VB200_ERR_NO_DEVICE, "device %d is sm_%d%d; the kernels are built for sm_90a only", device, p.major, p.minor);
    CUDA_CHECK(cudaSetDevice(device));
}

}  // namespace

// =========================================================================================== C ABI
extern "C" {

int vb200_abi_version(void) { return VB200_ABI_VERSION; }

}  // extern "C"

namespace {
// vb200_create (multi-task checkpoint, every task head) and vb200_create_pretraining (encoder + `cls` heads): the same options, audit and
// ingestion; `pretraining` selects the key set.
int create_engine(const char* api, bool pretraining, const char* config_json, int64_t n_tensors, const vb200_tensor* tensors,
                  const vb200_options* opt, vb200_handle* out) {
    if (out == nullptr) { g_create_error = std::string(api) + ": out handle pointer is NULL"; return VB200_ERR_INVALID; }
    *out = nullptr;
    std::unique_ptr<vb200_engine> eng;
    int rc = guard(nullptr, [&] {
        if (tensors == nullptr || n_tensors <= 0) fail(VB200_ERR_CHECKPOINT, "empty state_dict");
        vb200_options o{};
        if (opt) o = *opt;
        if (pretraining && o.num_labels != 0)
            fail(VB200_ERR_INVALID, "%s: num_labels must be 0 (a pre-training checkpoint has no vil_prediction head)", api);
        if (o.ln_fold != 0) fail(VB200_ERR_INVALID, "vb200_options: the LayerNorm fold was removed (its reserved field must be 0)");
        if (o.fused_layernorm > 0)
            fail(VB200_ERR_INVALID, "vb200_options: the cluster-LayerNorm GEMM epilogue was removed (fused_layernorm must be 0 or negative)");
        // tri-state flags: 0 = default, 1 = on, -1 = off
        o.use_cuda_graph = o.use_cuda_graph >= 0 ? 1 : 0;
        o.strict = o.strict >= 0 ? 1 : 0;
        const int pdl_req = o.use_pdl;
        o.use_pdl = o.use_pdl > 0 ? 1 : 0;
        o.split_fp32 = o.split_fp32 > 0 ? 1 : 0;
        o.act_fp16 = (o.act_fp16 >= 0 || o.split_fp32) ? 1 : 0;
        Config c = parse_config(config_json);
        if (pretraining && c.visual_target != 0)
            fail(VB200_ERR_CONFIG, "visual_target=%d is not supported (the masked-region head is the KL objective over v_target_size "
                 "classes, visual_target 0)", c.visual_target);
        if (pretraining && c.predict_feature) fail(VB200_ERR_CONFIG, "predict_feature=true is not supported (visual_target 0 only)");
        {   // audit the state_dict (names, shapes, dtypes, strictness) before touching any device
            vb200_engine audit;
            audit.cfg = c; audit.opt = o; audit.dry = true; audit.x3 = o.split_fp32 != 0; audit.pretraining = pretraining;
            audit.ingest(n_tensors, tensors);
        }
        require_device(o.device);
        eng.reset(new vb200_engine());
        eng->cfg = c;
        eng->opt = o;
        eng->pretraining = pretraining;
        eng->x3 = o.split_fp32 != 0;
        if (const char* v = getenv("VB200_LONE_ROWS")) eng->lone_rows = std::max(0, atoi(v));
        eng->max_plans = o.max_plans > 0 ? static_cast<size_t>(o.max_plans) : 24;
        if (const char* v = getenv("VB200_MAX_PLANS")) { const int n = atoi(v); if (n > 0) eng->max_plans = static_cast<size_t>(n); }
        if (pdl_req == 0) eng->opt.use_pdl = 1;               // default: full
        if (const char* v = getenv("VB200_PDL")) {
            if (strcmp(v, "full") == 0) eng->opt.use_pdl = 1;
            if (strcmp(v, "off") == 0) eng->opt.use_pdl = 0;
        }
        eng->gemm_kernel = default_gemm_kernel();
        eng->side_stream = make_stream();
        for (Event* e : {&eng->ev_fork, &eng->ev_join, &eng->pre_done}) *e = make_event();
        for (Staging* s : {&eng->dec_in, &eng->rel_in, &eng->sel_in, &eng->pre_in, &eng->abl_in}) s->copied = make_event();
        for (Workspace* w : {&eng->dec_ws, &eng->ans_ws, &eng->rel_ws, &eng->sel_ws, &eng->abl_ws}) w->done = make_event();
        eng->ingest(n_tensors, tensors);
        CUDA_CHECK(cudaDeviceSynchronize());
    });
    if (rc != VB200_OK) return rc;
    *out = eng.release();
    return VB200_OK;
}
}  // namespace

extern "C" {

int vb200_create(const char* config_json, int64_t n_tensors, const vb200_tensor* tensors, const vb200_options* opt,
                 vb200_handle* out) {
    return create_engine("vb200_create", false, config_json, n_tensors, tensors, opt, out);
}

int vb200_create_pretraining(const char* config_json, int64_t n_tensors, const vb200_tensor* tensors, const vb200_options* opt,
                             vb200_handle* out) {
    return create_engine("vb200_create_pretraining", true, config_json, n_tensors, tensors, opt, out);
}

int vb200_destroy(vb200_handle h) {
    if (h == nullptr) return VB200_OK;
    cudaSetDevice(h->opt.device);
    cudaDeviceSynchronize();
    delete h;
    return VB200_OK;
}

const char* vb200_last_error(vb200_handle h) { return h ? h->last_error.c_str() : g_create_error.c_str(); }

int vb200_forward(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, void* cuda_stream) {
    return vb200_forward_slot(h, in, out, select, 0, cuda_stream);
}

int vb200_forward_slot(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                       void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "inputs/outputs struct is NULL");
        h->run_dense("vb200_forward", in->batch, in->n_tokens, in->n_regions, select, slot, vb200_engine::FULL, out, {},
                     cudaMemcpyDeviceToDevice, cuda_stream, [&](Plan& pl, cudaStream_t st) {
                         h->check_inputs(*in);
                         h->embed_inputs(pl, *in, st);
                     });
    });
}

namespace {
// vb200_forward_packed and its gated form (head_mask non-null; `api` names the entry point)
int forward_packed(vb200_handle h, const char* api, const vb200_packed_inputs* in, const float* head_mask, const vb200_outputs* out,
                   uint32_t select, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "inputs/outputs struct is NULL");
        if (!in->n_tokens || !in->n_regions || !in->question || !in->segment_ids || !in->features || !in->spatials ||
            (h->cfg.task_tokens && !in->task_tokens))
            fail(VB200_ERR_INVALID, "vb200_packed_inputs has a NULL required pointer");
        h->run_packed(api, vb200_engine::PACKED,
                      {"sample", in->batch, in->n_tokens, in->max_tokens, in->n_regions, in->max_regions}, select, slot, out, {},
                      cuda_stream, [&](Plan& pl, const PackedBatch& b, cudaStream_t st) {
                          h->embed_text(pl, in->question, in->segment_ids, nullptr, in->task_tokens, b.rows_t(), st);
                          h->pack_image(pl, in->features, in->spatials, nullptr, b.rows_v(), st);
                      }, head_mask);
    });
}

// vb200_forward_regions_packed and its gated form (head_mask non-null)
int forward_regions_packed(vb200_handle h, const char* api, const vb200_packed_region_inputs* in, const float* head_mask,
                           const vb200_outputs* out, uint32_t select, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "inputs/outputs struct is NULL");
        const int task = h->cfg.task_tokens ? 1 : 0;
        if (!in->n_tokens || !in->n_boxes || !in->question || !in->segment_ids || !in->box_features || !in->boxes || !in->image_wh ||
            (task && !in->task_tokens))
            fail(VB200_ERR_INVALID, "vb200_packed_region_inputs has a NULL required pointer");
        const BoxRows v = box_rows(api, in->batch, in->n_boxes, in->max_boxes, h->max_rows);
        // named in the caller's field before pack_batch sees T_i
        for (int i = 0; i < in->batch; ++i)
            if (in->n_tokens[i] + task > h->max_rows)
                fail(VB200_ERR_INVALID, "%s: image %d has n_tokens %d (T = n_tokens + 1 must be <= %d)", api, i, in->n_tokens[i], h->max_rows);
        h->run_packed(api, vb200_engine::PACKED, {"image", in->batch, in->n_tokens, in->max_tokens, v.v.data(), v.max_regions}, select,
                      slot, out, {}, cuda_stream, [&](Plan& pl, const PackedBatch& b, cudaStream_t st) {
                          h->embed_text(pl, in->question, in->segment_ids, nullptr, in->task_tokens, b.rows_t(), st);
                          h->pack_regions_packed(pl, in->box_features, in->boxes, in->image_wh, in->spatials_out, b.rows_v(), st);
                      }, head_mask);
    });
}
// the gated forwards' own rejection, ahead of everything else: a gated call without a gate table
int reject_null_mask(vb200_handle h, const char* api, const float* head_mask) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { if (head_mask == nullptr) fail(VB200_ERR_INVALID, "%s: head_mask is NULL", api); });
}
}  // namespace

int vb200_forward_packed(vb200_handle h, const vb200_packed_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                         void* cuda_stream) {
    return forward_packed(h, "vb200_forward_packed", in, nullptr, out, select, slot, cuda_stream);
}

int vb200_forward_packed_gated(vb200_handle h, const vb200_packed_inputs* in, const float* head_mask, const vb200_outputs* out,
                               uint32_t select, int32_t slot, void* cuda_stream) {
    const char* api = "vb200_forward_packed_gated";
    const int r = reject_null_mask(h, api, head_mask);
    return r != VB200_OK ? r : forward_packed(h, api, in, head_mask, out, select, slot, cuda_stream);
}

int vb200_forward_regions_packed(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_outputs* out, uint32_t select,
                                 int32_t slot, void* cuda_stream) {
    return forward_regions_packed(h, "vb200_forward_regions_packed", in, nullptr, out, select, slot, cuda_stream);
}

int vb200_forward_regions_packed_gated(vb200_handle h, const vb200_packed_region_inputs* in, const float* head_mask,
                                       const vb200_outputs* out, uint32_t select, int32_t slot, void* cuda_stream) {
    const char* api = "vb200_forward_regions_packed_gated";
    const int r = reject_null_mask(h, api, head_mask);
    return r != VB200_OK ? r : forward_regions_packed(h, api, in, head_mask, out, select, slot, cuda_stream);
}

int vb200_forward_regions(vb200_handle h, const vb200_region_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                          void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "inputs/outputs struct is NULL");
        if (in->n_boxes < 1) fail(VB200_ERR_INVALID, "n_boxes must be positive");
        h->run_dense("vb200_forward_regions", in->batch, in->n_tokens, in->n_boxes + 1, select, slot, vb200_engine::FULL, out, {},
                     cudaMemcpyDeviceToDevice, cuda_stream, [&](Plan& pl, cudaStream_t st) { h->embed_regions(pl, *in, st); });
    });
}

int vb200_encode_text(vb200_handle h, int32_t n, int32_t n_tokens, const int64_t* question, const int64_t* segment_ids,
                      const int64_t* input_mask, const int64_t* task_tokens, float* state_f32, void* state_16, float* state_mask,
                      void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (!question || !segment_ids || !input_mask || (h->cfg.task_tokens && !task_tokens) || !state_f32 || !state_16 || !state_mask)
            fail(VB200_ERR_INVALID, "vb200_encode_text: NULL pointer");
        h->run_dense("vb200_encode_text", n, n_tokens, 1, 0, 0, vb200_engine::TEXT_PREFIX, nullptr, {state_f32, state_16, state_mask},
                     cudaMemcpyDeviceToDevice, cuda_stream, [&](Plan& pl, cudaStream_t st) {
                         h->embed_text(pl, question, segment_ids, input_mask, task_tokens, pl.B * pl.T, st);
                     });
    });
}

int vb200_encode_image(vb200_handle h, int32_t n, int32_t n_regions, const float* features, const float* spatials,
                       const uint8_t* image_mask, float* state_f32, void* state_16, float* state_mask, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (!features || !spatials || !image_mask || !state_f32 || !state_16 || !state_mask)
            fail(VB200_ERR_INVALID, "vb200_encode_image: NULL pointer");
        h->run_dense("vb200_encode_image", n, 1, n_regions, 0, 0, vb200_engine::IMAGE_PREFIX, nullptr, {state_f32, state_16, state_mask},
                     cudaMemcpyDeviceToDevice, cuda_stream, [&](Plan& pl, cudaStream_t st) {
                         h->pack_image(pl, features, spatials, image_mask, pl.B * pl.V, st);
                     });
    });
}

int vb200_forward_cached(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, const int32_t* text_index,
                         int32_t n_text, const float* text_f32, const void* text_16, const float* text_mask,
                         const int32_t* image_index, int32_t n_image, const float* image_f32, const void* image_16,
                         const float* image_mask, const vb200_outputs* out, uint32_t select, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (out == nullptr) fail(VB200_ERR_INVALID, "outputs struct is NULL");
        if (n_text < 1 || n_image < 1) fail(VB200_ERR_INVALID, "cached state counts must be positive");
        h->run_dense("vb200_forward_cached", batch, n_tokens, n_regions, select, slot, vb200_engine::SUFFIX, out, {},
                     cudaMemcpyDeviceToDevice, cuda_stream, [&](Plan& pl, cudaStream_t st) {
                         h->gather_state(pl, text_index, n_text, text_f32, text_16, text_mask, image_index, n_image, image_f32, image_16,
                                         image_mask, st);
                     });
    });
}

int vb200_encode_text_packed(vb200_handle h, int32_t n, int32_t max_tokens, const int32_t* n_tokens, const int64_t* question,
                             const int64_t* segment_ids, const int64_t* task_tokens, float* state_f32, void* state_16, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_encode_text_packed";
        if (!n_tokens || !question || !segment_ids || (h->cfg.task_tokens && !task_tokens) || !state_f32 || !state_16)
            fail(VB200_ERR_INVALID, "%s: NULL pointer", api);
        h->run_packed(api, vb200_engine::PACKED_TEXT_PREFIX, {"caption", n, n_tokens, max_tokens, nullptr, 0}, 0, 0, nullptr,
                      {state_f32, state_16, nullptr}, cuda_stream, [&](Plan& pl, const PackedBatch& b, cudaStream_t st) {
                          h->embed_text(pl, question, segment_ids, nullptr, task_tokens, b.rows_t(), st);
                      });
    });
}

int vb200_encode_image_packed(vb200_handle h, int32_t n, int32_t max_regions, const int32_t* n_regions, const float* features,
                              const float* spatials, float* state_f32, void* state_16, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_encode_image_packed";
        if (!n_regions || !features || !spatials || !state_f32 || !state_16) fail(VB200_ERR_INVALID, "%s: NULL pointer", api);
        h->run_packed(api, vb200_engine::PACKED_IMAGE_PREFIX, {"image", n, nullptr, 0, n_regions, max_regions}, 0, 0, nullptr,
                      {state_f32, state_16, nullptr}, cuda_stream, [&](Plan& pl, const PackedBatch& b, cudaStream_t st) {
                          h->pack_image(pl, features, spatials, nullptr, b.rows_v(), st);
                      });
    });
}

int vb200_encode_regions_packed(vb200_handle h, int32_t n, int32_t max_boxes, const int32_t* n_boxes, const float* box_features,
                                const float* boxes, const float* image_wh, float* state_f32, void* state_16, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_encode_regions_packed";
        if (!n_boxes || !box_features || !boxes || !image_wh || !state_f32 || !state_16) fail(VB200_ERR_INVALID, "%s: NULL pointer", api);
        const BoxRows v = box_rows(api, n, n_boxes, max_boxes, h->max_rows);
        // the PACKED_IMAGE_PREFIX plan of vb200_encode_image_packed at max_regions = max_boxes + 1, fed by the region pack of
        // vb200_forward_regions_packed: each image's rows are the rows that forward writes for it
        h->run_packed(api, vb200_engine::PACKED_IMAGE_PREFIX, {"image", n, nullptr, 0, v.v.data(), v.max_regions}, 0, 0, nullptr,
                      {state_f32, state_16, nullptr}, cuda_stream, [&](Plan& pl, const PackedBatch& b, cudaStream_t st) {
                          h->pack_regions_packed(pl, box_features, boxes, image_wh, nullptr, b.rows_v(), st);
                      });
    });
}

int vb200_forward_cached_packed(vb200_handle h, const vb200_packed_pairs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                                void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_forward_cached_packed";
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "inputs/outputs struct is NULL");
        if (in->n_text < 1 || in->n_image < 1) fail(VB200_ERR_INVALID, "%s: n_text and n_image must be positive", api);
        if (!in->text_index || !in->image_index || !in->text_offsets || !in->image_offsets || !in->text_f32 || !in->text_16 ||
            !in->image_f32 || !in->image_16)
            fail(VB200_ERR_INVALID, "%s: vb200_packed_pairs has a NULL required pointer", api);
        auto check_offsets = [&](const int32_t* offs, int n, const char* what) {
            if (offs[0] < 0) fail(VB200_ERR_INVALID, "%s: %s_offsets[0] = %d is negative", api, what, offs[0]);
            for (int i = 0; i < n; ++i)
                if (offs[i + 1] <= offs[i])
                    fail(VB200_ERR_INVALID, "%s: %s state %d has %d rows (the offsets must increase)", api, what, i, offs[i + 1] - offs[i]);
        };
        check_offsets(in->text_offsets, in->n_text, "text");
        check_offsets(in->image_offsets, in->n_image, "image");
        // each pair's lengths and first rows in the cached states
        const int task = h->cfg.task_tokens ? 1 : 0;
        std::vector<int32_t> tin, nv, src_t, src_v;
        for (int b = 0; b < in->batch; ++b) {
            const int ti = in->text_index[b], vi = in->image_index[b];
            if (ti < 0 || ti >= in->n_text) fail(VB200_ERR_INVALID, "%s: pair %d: text_index %d outside [0, %d)", api, b, ti, in->n_text);
            if (vi < 0 || vi >= in->n_image) fail(VB200_ERR_INVALID, "%s: pair %d: image_index %d outside [0, %d)", api, b, vi, in->n_image);
            tin.push_back(in->text_offsets[ti + 1] - in->text_offsets[ti] - task);
            nv.push_back(in->image_offsets[vi + 1] - in->image_offsets[vi]);
            src_t.push_back(in->text_offsets[ti]);
            src_v.push_back(in->image_offsets[vi]);
        }
        h->run_packed(api, vb200_engine::PACKED_SUFFIX,
                      {"pair", in->batch, tin.data(), in->max_tokens, nv.data(), in->max_regions, src_t.data(), src_v.data()}, select, slot,
                      out, {}, cuda_stream, [&](Plan& pl, const PackedBatch& b, cudaStream_t st) { h->gather_packed_state(pl, *in, b, st); });
    });
}

int vb200_decode_answers(vb200_handle h, const vb200_decode_msg* msgs, int32_t n, const vb200_outputs* out, int32_t batch,
                         int32_t vision_rows, const float* spatials, vb200_answer* answers, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_decode_answers";
        const std::vector<vb::DecodeDesc> d = h->decode_descs(api, msgs, n, out, batch, vision_rows, spatials);
        if (answers == nullptr) fail(VB200_ERR_INVALID, "%s: answers is NULL", api);
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        h->decode_answers(d, answers, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_decode_answers_host(vb200_handle h, const vb200_decode_msg* msgs, int32_t n, const vb200_outputs* out, int32_t batch,
                              int32_t vision_rows, const float* spatials, vb200_answer* answers, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_decode_answers_host";
        const std::vector<vb::DecodeDesc> d = h->decode_descs(api, msgs, n, out, batch, vision_rows, spatials);
        if (answers == nullptr) fail(VB200_ERR_INVALID, "%s: answers is NULL", api);
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
        const size_t bytes = d.size() * sizeof(vb200_answer);
        vb200_answer* dev = reinterpret_cast<vb200_answer*>(h->ans_ws.acquire(bytes, st));
        h->decode_answers(d, dev, st);
        CUDA_CHECK(cudaMemcpyAsync(answers, dev, bytes, cudaMemcpyDeviceToHost, st));
        h->ans_ws.release(st);
        CUDA_CHECK(cudaStreamSynchronize(st));
    });
}

int vb200_attention_relevance(vb200_handle h, const float* attention_probs, int32_t batch, const int32_t* n_tokens,
                              const int32_t* n_regions, int32_t packed, float* relevance, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        h->attention_relevance(attention_probs, batch, n_tokens, n_regions, packed, relevance, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_answer_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_ablation_msg* msgs, int32_t family,
                          int64_t mask_token, float* variant_logits, vb200_ablation_score* scores, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        h->answer_ablation(in, msgs, family, mask_token, variant_logits, scores, slot, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_message_ablation_layout(vb200_handle h, int32_t batch, const int32_t* n_tokens, const int32_t* n_boxes,
                                  const vb200_ablation_message* msgs, int32_t n_msgs, vb200_ablation_variant* variants, int64_t* n_variants,
                                  int64_t* n_floats, int64_t* n_samples) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->message_ablation_layout(batch, n_tokens, n_boxes, msgs, n_msgs, variants, n_variants, n_floats, n_samples); });
}

int vb200_head_ablation_layout(vb200_handle h, int32_t batch, const int32_t* n_tokens, const int32_t* n_boxes,
                               const vb200_head_ablation_message* msgs, int32_t n_msgs, vb200_ablation_variant* variants, int64_t* n_variants,
                               int64_t* n_floats, int64_t* n_samples) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->head_ablation_layout(batch, n_tokens, n_boxes, msgs, n_msgs, variants, n_variants, n_floats, n_samples); });
}

int vb200_coalition_ablation_layout(vb200_handle h, int32_t batch, const int32_t* n_tokens, const int32_t* n_boxes,
                                    const vb200_coalition_message* msgs, int32_t n_msgs, vb200_ablation_variant* variants,
                                    int64_t* n_variants, int64_t* n_floats, int64_t* n_samples) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->coalition_ablation_layout(batch, n_tokens, n_boxes, msgs, n_msgs, variants, n_variants, n_floats, n_samples); });
}

int vb200_coalition_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_coalition_message* msgs, int32_t n_msgs,
                             int64_t mask_token, float* variant_logits, vb200_ablation_score* scores, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        h->coalition_ablation(in, msgs, n_msgs, mask_token, variant_logits, scores, slot, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_shapley_values(vb200_handle h, const vb200_shapley_message* msgs, int32_t n_msgs, const int32_t* perm, const float* values,
                         float* phi, float* stderr_out, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->shapley_values(msgs, n_msgs, perm, values, phi, stderr_out, static_cast<cudaStream_t>(cuda_stream)); });
}

int vb200_interaction_values(vb200_handle h, const vb200_interaction_message* msgs, int32_t n_msgs, const int32_t* perm,
                             const float* values, float* inter, float* stderr_out, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->interaction_values(msgs, n_msgs, perm, values, inter, stderr_out, static_cast<cudaStream_t>(cuda_stream)); });
}

int vb200_head_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_head_ablation_message* msgs, int32_t n_msgs,
                        float* variant_logits, vb200_ablation_score* scores, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        h->head_ablation(in, msgs, n_msgs, variant_logits, scores, slot, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_message_ablation(vb200_handle h, const vb200_packed_region_inputs* in, const vb200_ablation_message* msgs, int32_t n_msgs,
                           int64_t mask_token, float* variant_logits, vb200_ablation_score* scores, int32_t slot, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        h->message_ablation(in, msgs, n_msgs, mask_token, variant_logits, scores, slot, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_select_regions(vb200_handle h, const vb200_detections* imgs, int32_t n, const vb200_select_params* p, const vb200_selected* out,
                         void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        h->select_regions(imgs, n, p, out, static_cast<cudaStream_t>(cuda_stream));
    });
}

int vb200_pretraining_heads(vb200_handle h, const vb200_pretrain_rows* in, const vb200_pretrain_out* out, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->pretraining_heads(in, out, static_cast<cudaStream_t>(cuda_stream)); });
}

int vb200_pretraining_objectives(vb200_handle h, const vb200_pretrain_rows* in, const vb200_pretrain_targets* targets,
                                 const vb200_pretrain_losses* out, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] { h->pretraining_objectives(in, targets, out, static_cast<cudaStream_t>(cuda_stream)); });
}

int vb200_attention_layout(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, int32_t max_entries,
                           int32_t* n_entries, int32_t* dims, int64_t* offsets, int64_t* total_floats) {
    if (h == nullptr || n_entries == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        // derived from the layer schedule and the map selection alone (no plan is built): the order get_plan's builder
        // calls PlanBuilder::attention_f32 in
        const Config& c = h->cfg;
        const int T = n_tokens + (c.task_tokens ? 1 : 0), V = n_regions;
        const std::vector<int> kinds = attention_kinds(h->schedule);
        int n = 0;
        int64_t off = 0;
        for (int e = 0; e < static_cast<int>(kinds.size()); ++e) {
            if (!h->attn_sel.has(e)) continue;
            const int kind = kinds[e], heads = h->attn_sel.heads(kind == 0 ? c.heads : kind == 1 ? c.v_heads : c.bi_heads);
            const int lq = kind == 0 || kind == 2 ? T : V, lk = kind == 0 || kind == 3 ? T : V;
            if (n < max_entries) {
                if (dims) { dims[4 * n] = heads; dims[4 * n + 1] = lq; dims[4 * n + 2] = lk; dims[4 * n + 3] = kind; }
                if (offsets) offsets[n] = off;
            }
            off += static_cast<int64_t>(batch) * heads * lq * lk;
            ++n;
        }
        *n_entries = n;
        if (total_floats) *total_floats = off;
    });
}

int vb200_attention_layout_packed(vb200_handle h, int32_t batch, const int32_t* n_tokens, const int32_t* n_regions, int32_t max_entries,
                                  int32_t* n_entries, int32_t* dims, int64_t* offsets, int64_t* total_floats) {
    if (h == nullptr || n_entries == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        // from the lengths and the layer schedule alone (no plan is built), validated as the packed forwards validate them
        const char* api = "vb200_attention_layout_packed";
        if (!n_tokens || !n_regions) fail(VB200_ERR_INVALID, "%s: NULL length array", api);
        const PackedBatch b = pack_batch(api, h->cfg, h->schedule, {"sample", batch, n_tokens, 0, n_regions, 0}, nullptr, h->max_rows);
        const PackedAttnLayout l = packed_attn_layout(h->cfg, h->schedule, h->attn_sel, batch, b.offs_t(), b.offs_v());
        const int n = static_cast<int>(l.heads.size());
        for (int e = 0; e < n && e < max_entries; ++e) {
            if (dims) { dims[2 * e] = l.heads[e]; dims[2 * e + 1] = l.kind[e]; }
            if (offsets) offsets[e] = l.offset[e];
        }
        *n_entries = n;
        if (total_floats) *total_floats = l.total;
    });
}

int vb200_attention_selection(vb200_handle h, int32_t max_entries, int32_t* n_entries, int32_t* kinds, int32_t* layout_entry) {
    if (h == nullptr || n_entries == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const std::vector<int> k = attention_kinds(h->schedule);
        int selected = 0;
        for (int e = 0; e < static_cast<int>(k.size()); ++e) {
            const bool has = h->attn_sel.has(e);
            if (e < max_entries) {
                if (kinds) kinds[e] = k[e];
                if (layout_entry) layout_entry[e] = has ? selected : -1;
            }
            selected += has ? 1 : 0;
        }
        *n_entries = static_cast<int32_t>(k.size());
    });
}

}  // extern "C"

namespace {
// the arrays of vb200_state_layout / vb200_state_layout_packed
void put_state_layout(const StateLayout& l, int32_t max_entries, int32_t* n_entries, int32_t* kinds, int32_t* dims, int64_t* offsets,
                      int64_t* total_floats) {
    const int n = static_cast<int>(l.offset.size());
    for (int e = 0; e < n && e < max_entries; ++e) {
        if (kinds) kinds[e] = l.kind[e];
        if (dims) { dims[2 * e] = l.rows[e]; dims[2 * e + 1] = l.width[e]; }
        if (offsets) offsets[e] = l.offset[e];
    }
    *n_entries = n;
    if (total_floats) *total_floats = l.total;
}
}  // namespace

extern "C" {

int vb200_state_layout(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, int32_t max_entries, int32_t* n_entries,
                       int32_t* kinds, int32_t* dims, int64_t* offsets, int64_t* total_floats) {
    if (h == nullptr || n_entries == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (batch < 1 || n_tokens < 1 || n_regions < 1) fail(VB200_ERR_INVALID, "vb200_state_layout: batch, n_tokens and n_regions must be positive");
        const int64_t T = n_tokens + (h->cfg.task_tokens ? 1 : 0);
        put_state_layout(state_layout(h->cfg, h->schedule, h->state_sel, batch, batch * T, static_cast<int64_t>(batch) * n_regions),
                         max_entries, n_entries, kinds, dims, offsets, total_floats);
    });
}

int vb200_state_layout_packed(vb200_handle h, int32_t batch, const int32_t* n_tokens, const int32_t* n_regions, int32_t max_entries,
                              int32_t* n_entries, int32_t* kinds, int32_t* dims, int64_t* offsets, int64_t* total_floats) {
    if (h == nullptr || n_entries == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const char* api = "vb200_state_layout_packed";
        if (!n_tokens || !n_regions) fail(VB200_ERR_INVALID, "%s: NULL length array", api);
        const PackedBatch b = pack_batch(api, h->cfg, h->schedule, {"sample", batch, n_tokens, 0, n_regions, 0}, nullptr, h->max_rows);
        put_state_layout(state_layout(h->cfg, h->schedule, h->state_sel, batch, b.rows_t(), b.rows_v()), max_entries, n_entries, kinds,
                         dims, offsets, total_floats);
    });
}

int vb200_state_selection(vb200_handle h, int32_t max_entries, int32_t* n_entries, int32_t* kinds, int32_t* layout_entry) {
    if (h == nullptr || n_entries == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const std::vector<int> k = state_kinds(h->schedule);
        for (int e = 0; e < static_cast<int>(k.size()) && e < max_entries; ++e) {
            if (kinds) kinds[e] = k[e];
            if (layout_entry) layout_entry[e] = h->state_sel.has(e) ? h->state_sel.index(e) : -1;
        }
        *n_entries = static_cast<int32_t>(k.size());
    });
}

int vb200_forward_host(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, void* cuda_stream) {
    return vb200_forward_host_slot(h, in, out, select, 0, 1, cuda_stream);
}

int vb200_forward_host_slot(vb200_handle h, const vb200_inputs* in, const vb200_outputs* out, uint32_t select, int32_t slot,
                            int32_t synchronize, void* cuda_stream) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        if (in == nullptr || out == nullptr) fail(VB200_ERR_INVALID, "inputs/outputs struct is NULL");
        h->run_dense("vb200_forward_host", in->batch, in->n_tokens, in->n_regions, select, slot, vb200_engine::FULL, out, {},
                     cudaMemcpyDeviceToHost, cuda_stream, [&](Plan& pl, cudaStream_t st) {
            const size_t B = pl.B, Tin = pl.Tin, V = pl.V, F = h->cfg.v_feat;
            if (pl.d_q == nullptr) {
                pl.d_q = pl.mem.alloc_n<int64_t>(B * Tin); pl.d_seg = pl.mem.alloc_n<int64_t>(B * Tin);
                pl.d_mask = pl.mem.alloc_n<int64_t>(B * Tin); pl.d_task = pl.mem.alloc_n<int64_t>(B);
                pl.d_feat = pl.mem.alloc_n<float>(B * V * F); pl.d_loc = pl.mem.alloc_n<float>(B * V * 5);
                pl.d_imask = pl.mem.alloc_n<uint8_t>(B * V);
            }
            h->check_inputs(*in);
            CUDA_CHECK(cudaMemcpyAsync(pl.d_q, in->question, B * Tin * 8, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(pl.d_seg, in->segment_ids, B * Tin * 8, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(pl.d_mask, in->input_mask, B * Tin * 8, cudaMemcpyHostToDevice, st));
            if (in->task_tokens) CUDA_CHECK(cudaMemcpyAsync(pl.d_task, in->task_tokens, B * 8, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(pl.d_feat, in->features, B * V * F * 4, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(pl.d_loc, in->spatials, B * V * 5 * 4, cudaMemcpyHostToDevice, st));
            CUDA_CHECK(cudaMemcpyAsync(pl.d_imask, in->image_mask, B * V, cudaMemcpyHostToDevice, st));
            vb200_inputs dev = *in;
            dev.question = pl.d_q; dev.segment_ids = pl.d_seg; dev.input_mask = pl.d_mask; dev.task_tokens = pl.d_task;
            dev.features = pl.d_feat; dev.spatials = pl.d_loc; dev.image_mask = pl.d_imask; dev.co_attention_mask = nullptr;
            h->embed_inputs(pl, dev, st);
        });
        if (synchronize) CUDA_CHECK(cudaStreamSynchronize(static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_plan_info(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, uint32_t select,
                    int64_t* n_launches, double* flops) {
    if (h == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        Plan* pl = h->get_plan(batch, n_tokens, n_regions, select & VB200_OUT_ALL, 0, vb200_engine::FULL,
                               (select & VB200_OUT_ATTENTION) != 0, (select & VB200_OUT_LAYER_STATES) != 0);
        if (n_launches) *n_launches = static_cast<int64_t>(pl->ops.size()) + 2;   // + text-embed + image-pack
        if (flops) *flops = pl->flops;
    });
}

int vb200_profile_ops(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, uint32_t select, int32_t iters,
                      int32_t max_ops, int32_t* n_ops, int32_t* kinds, double* ms, double* flops, int32_t* dims) {
    if (h == nullptr || n_ops == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        Plan* pl = h->get_plan(batch, n_tokens, n_regions, select & VB200_OUT_ALL);
        std::vector<double> t;
        struct Reset { vb200_engine* e; int keep; ~Reset() { e->profile_grid_pct = keep; } } reset{h, h->profile_grid_pct};
        h->profile_ops(*pl, iters < 1 ? 1 : iters, t);
        h->profile_grid_pct = 0;          // the override never leaks into forwards (plans are captured without it anyway)
        reset.keep = 0;
        const int n = static_cast<int>(pl->ops.size());
        *n_ops = n;
        for (int i = 0; i < n && i < max_ops; ++i) {
            const Op& op = pl->ops[i];
            if (kinds) kinds[i] = static_cast<int>(op.args.index());
            if (ms) ms[i] = t[i];
            if (flops) flops[i] = op.flops;
            if (dims) {
                const std::array<int, 4> d = vb200_engine::op_dims(op);
                std::copy(d.begin(), d.end(), dims + 4 * i);
            }
        }
    });
}

int vb200_set_option(vb200_handle h, const char* key, int64_t value) {
    if (h == nullptr || key == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const std::string k = key;
        if (k == "profile_grid_pct") {
            if (value != 0 && (value < 10 || value > 100)) fail(VB200_ERR_INVALID, "profile_grid_pct must be 0 or 10..100");
            h->profile_grid_pct = static_cast<int>(value);
        } else if (k == "max_plans") {
            if (value < 1) fail(VB200_ERR_INVALID, "max_plans must be positive");
            h->max_plans = static_cast<size_t>(value);
        } else if (k == "timeline") {
            if ((value != 0) != h->timeline) {
                CUDA_CHECK(cudaDeviceSynchronize());
                h->plans.clear();
                h->timeline = value != 0;
            }
        } else if (k == "gemm_kernel") {
            if (value != 0 && value != 1) fail(VB200_ERR_INVALID, "gemm_kernel must be 0 (cooperative) or 1 (ping-pong)");
            if (value != h->gemm_kernel) {              // the kernel is chosen when a plan is built
                CUDA_CHECK(cudaDeviceSynchronize());
                h->plans.clear();
                for (auto& m : h->row_heads) m.clear();
                h->gemm_kernel = static_cast<int>(value);
            }
        } else if (k == "max_rows_per_sample") {
            if (value < kStagedAttnRows || value > kMaxRowsPerSample)
                fail(VB200_ERR_INVALID, "max_rows_per_sample must be in [%d, %d]", kStagedAttnRows, kMaxRowsPerSample);
            h->max_rows = static_cast<int>(value);       // validation only: every cached plan stays valid
        } else if (k == "attention_entries") {
            // the selection is part of the plan key of a plan with maps: no cached plan is dropped
            const int n = static_cast<int>(attention_kinds(h->schedule).size());
            if (n > 63)
                fail(VB200_ERR_INVALID, "attention_entries: this configuration has %d attention entries, more than the 63 a mask holds", n);
            const uint64_t full = (1ull << n) - 1;
            if (value == 0 || (static_cast<uint64_t>(value) & ~full) != 0)
                fail(VB200_ERR_INVALID, "attention_entries: mask 0x%llx must be non-zero and select only entries 0..%d",
                     (unsigned long long)value, n - 1);
            h->attn_sel.mask = static_cast<uint64_t>(value) == full ? ~0ull : static_cast<uint64_t>(value);
        } else if (k == "attention_heads") {
            if (value != 0 && value != 1)
                fail(VB200_ERR_INVALID, "attention_heads must be 0 (every head) or 1 (the mean over heads), got %lld", (long long)value);
            h->attn_sel.mean = value == 1;
        } else if (k == "state_entries") {
            // part of the plan key of a plan with states: no cached plan is dropped
            const int n = static_cast<int>(state_kinds(h->schedule).size());
            if (n > 63) fail(VB200_ERR_INVALID, "state_entries: this configuration has %d state entries, more than the 63 a mask holds", n);
            const uint64_t full = (1ull << n) - 1;
            if (value == 0 || (static_cast<uint64_t>(value) & ~full) != 0)
                fail(VB200_ERR_INVALID, "state_entries: mask 0x%llx must be non-zero and select only entries 0..%d", (unsigned long long)value,
                     n - 1);
            h->state_sel.mask = static_cast<uint64_t>(value) == full ? ~0ull : static_cast<uint64_t>(value);
        } else if (k == "state_rows") {
            if (value < 0 || value > 2)
                fail(VB200_ERR_INVALID, "state_rows must be 0 (every row), 1 (each sample's first row) or 2 (each sample's mean), got %lld",
                     (long long)value);
            h->state_sel.rows = static_cast<int>(value);
        } else fail(VB200_ERR_INVALID, "unknown option \"%s\"", key);
    });
}

int vb200_timeline(vb200_handle h, int32_t batch, int32_t n_tokens, int32_t n_regions, uint32_t select, int32_t slot, int32_t max_ops,
                   int32_t* n_ops, int32_t* dims, int64_t* stamps) {
    if (h == nullptr || n_ops == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        CUDA_CHECK(cudaSetDevice(h->opt.device));
        if (!h->timeline) fail(VB200_ERR_INVALID, "vb200_timeline: set_option(\"timeline\", 1) first");
        Plan* pl = h->get_plan(batch, n_tokens, n_regions, select & VB200_OUT_ALL, slot);
        CUDA_CHECK(cudaDeviceSynchronize());
        int n = 0;
        for (const Op& op : pl->ops) {
            const GemmCall* g = std::get_if<GemmCall>(&op.args);
            if (g == nullptr || g->ep.timing == nullptr) continue;
            if (n < max_ops) {
                if (dims) { dims[4 * n] = g->ep.M; dims[4 * n + 1] = g->ep.N; dims[4 * n + 2] = g->ep.K; dims[4 * n + 3] = op.stream; }
                if (stamps) CUDA_CHECK(cudaMemcpy(stamps + static_cast<size_t>(n) * vb200_engine::kTimelineCtas * 16, g->ep.timing,
                                                  sizeof(long long) * vb200_engine::kTimelineCtas * 16, cudaMemcpyDeviceToHost));
            }
            ++n;
        }
        *n_ops = n;
    });
}

int vb200_model_dim(vb200_handle h, const char* key, int64_t* value) {
    if (h == nullptr || key == nullptr || value == nullptr) return VB200_ERR_INVALID;
    return guard(h, [&] {
        const Config& c = h->cfg;
        const std::string k = key;
        if (k == "hidden_size") *value = c.hidden; else if (k == "v_hidden_size") *value = c.v_hidden;
        else if (k == "bi_hidden_size") *value = c.bi_hidden; else if (k == "vocab_size") *value = c.vocab;
        else if (k == "v_target_size") *value = c.v_target; else if (k == "v_feature_size") *value = c.v_feat;
        else if (k == "num_labels") *value = h->num_labels; else if (k == "gqa_labels") *value = h->gqa_labels;
        else if (k == "task_specific_tokens") *value = c.task_tokens;
        else if (k == "weight_bytes") *value = static_cast<int64_t>(h->weights.total);
        else if (k == "operand_width_factor") *value = h->x3 ? 3 : 1;
        else if (k == "n_plans") *value = static_cast<int64_t>(h->plans.size());
        else if (k == "n_layers_scheduled") *value = static_cast<int64_t>(h->schedule.size());
        else if (k == "max_rows_per_sample") *value = h->max_rows;
        else if (k == "head_mask_entries") *value = h->gate_entries();
        else if (k == "head_mask_heads") *value = h->gate_heads();
        else if (k == "attention_entries") {
            const size_t n = attention_kinds(h->schedule).size();
            *value = n > 63 ? -1 : static_cast<int64_t>(h->attn_sel.mask & ((1ull << n) - 1));
        } else if (k == "attention_heads") *value = h->attn_sel.mean ? 1 : 0;
        else if (k == "state_entries") {
            const size_t n = state_kinds(h->schedule).size();
            *value = n > 63 ? -1 : static_cast<int64_t>(h->state_sel.mask & ((1ull << n) - 1));
        } else if (k == "state_rows") *value = h->state_sel.rows;
        else fail(VB200_ERR_INVALID, "unknown model dimension \"%s\"", key);
    });
}

// ---------------------------------------------------------------- kernel-level entry points
static std::string g_op_error;
static int op_guard(const std::function<void()>& body) {
    try { body(); return VB200_OK; }
    catch (const VbError& e) { g_create_error = e.what(); return e.status; }
    catch (const std::exception& e) { g_create_error = e.what(); return VB200_ERR_INVALID; }
}

int vb200_linear(const void* x_bf16, int64_t ld_x, const void* w_bf16, int64_t ld_w, const float* bias,
                 const float* residual, int64_t ld_res, const float* gamma, const float* beta, float eps, int32_t act,
                 void* y_bf16, int64_t ld_y_bf16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K,
                 int32_t block_n, int32_t use_pdl, int32_t act_fp16, int32_t variant, long long* timing, void* cuda_stream) {
    return op_guard([&] {
        // LayerNorm is the row kernel's job (vb200_layernorm on the fp32 output); eps is ignored
        if (residual != nullptr || gamma != nullptr || beta != nullptr)
            fail(VB200_ERR_INVALID, "vb200_linear: residual, gamma and beta must be NULL (the cluster-LayerNorm GEMM epilogue was "
                                    "removed; run vb200_layernorm on the fp32 output)");
        // Variant 2 named the Blackwell CTA-pair kernel, variants 3 and 4 Blackwell occupancy configurations of the persistent kernel
        // (three CTAs per SM; one CTA with a 6-stage ring); ABI version 2 keeps accepting them, and on sm_90a they select the
        // persistent kernel itself.  block_n 256 (the Blackwell 256-wide tile) runs as 128-wide tiles, which give the same bits: the
        // tile width never changes an element's accumulation order.
        if (variant < 0 || variant == 1 || variant > 5)
            fail(VB200_ERR_INVALID, "vb200_linear: variant %d does not exist (0 persistent, 2 / 3 / 4 = 0, 5 ping-pong)", variant);
        GemmEpilogue e{};
        e.M = (int)M; e.N = (int)N; e.K = (int)K; e.bias = bias; e.out_bf16 = static_cast<bf16*>(y_bf16); e.ld_bf16 = (int)ld_y_bf16;
        e.out_f32 = y_f32; e.ld_f32 = (int)ld_y_f32; e.act = act; e.pdl = use_pdl;
        e.a_f16 = act_fp16 ? 1 : 0; e.out_f16 = e.a_f16; e.timing = timing;
        const cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
        int bn = block_n > 0 ? block_n : vb::gemm_p_pick_block_n(static_cast<int>(N));
        if (variant == 5) {
            const GemmCall g = make_gemm(x_bf16, ld_x, w_bf16, ld_w, e, {bn, 1});
            if (!g.pingpong)
                fail(VB200_ERR_INVALID, "vb200_linear: variant 5 (ping-pong) takes plain GEMMs with N a multiple of block_n 64 / 128 and "
                                        "TMA-storable outputs (N=%lld block_n=%d)", (long long)N, bn);
            CUDA_CHECK(g.launch(st));
            return;
        }
        if (bn == 256) bn = 128;
        if (bn != 64 && bn != 128 && bn != 192)
            fail(VB200_ERR_INVALID, "vb200_linear: block_n %d (plain tiles are 64, 128, 192 or 256 wide)", bn);
        if (variant >= 2 && bn != 128 && !(variant == 4 && bn == 64))
            fail(VB200_ERR_INVALID, "vb200_linear: variants 2 and 3 are the plain 128-wide tile, variant 4 the 128- or 64-wide one");
        if (const char* dbg = getenv("VB200_DEBUG")) e.debug = atoi(dbg);          // timing decomposition (kernels.h), op entry only
        CUDA_CHECK(make_gemm(x_bf16, ld_x, w_bf16, ld_w, e, {bn, 0}).launch(st));
    });
}

int vb200_linear_rows(const void* x16, int64_t ld_x, const void* w16, int64_t ld_w, const float* bias, int32_t act, void* y16,
                      int64_t ld_y16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K, int32_t block_n, int32_t act_fp16,
                      const int32_t* m_rows, void* cuda_stream) {
    return op_guard([&] {
        if (m_rows == nullptr) fail(VB200_ERR_INVALID, "vb200_linear_rows: m_rows is NULL");
        const int bn = block_n > 0 ? block_n : vb::gemm_p_pick_block_n(static_cast<int>(N));
        if (bn != 64 && bn != 128 && bn != 192) fail(VB200_ERR_INVALID, "vb200_linear_rows: block_n %d (plain tiles are 64, 128 or 192 wide)", bn);
        GemmEpilogue e{};
        e.M = (int)M; e.N = (int)N; e.K = (int)K; e.bias = bias; e.act = act; e.a_f16 = act_fp16 ? 1 : 0; e.out_f16 = e.a_f16;
        e.out_bf16 = static_cast<bf16*>(y16); e.ld_bf16 = (int)ld_y16; e.out_f32 = y_f32; e.ld_f32 = (int)ld_y_f32; e.m_rows = m_rows;
        CUDA_CHECK(make_gemm(x16, ld_x, w16, ld_w, e, {bn, -1}).launch(static_cast<cudaStream_t>(cuda_stream)));   // as the engine
    });
}

int vb200_layernorm(const float* y, int64_t ld_y, const float* residual, int64_t ld_res, const float* gamma, const float* beta,
                    float eps, float* out_f32, int64_t ld_f32, void* out_16, int64_t ld_16, int64_t M, int64_t N,
                    int32_t act_fp16, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_ln_residual(y, (int)ld_y, residual, (int)ld_res, gamma, beta, eps, out_f32, (int)ld_f32,
                                          static_cast<bf16*>(out_16), (int)ld_16, (int)M, (int)N, act_fp16 ? 1 : 0, 0, 0,
                                          static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_layernorm_split(const float* y, int64_t ld_y, const float* residual, int64_t ld_res, const float* gamma, const float* beta,
                          float eps, float* out_f32, int64_t ld_f32, void* out_16, int64_t ld_16, int64_t M, int64_t N, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_ln_residual(y, (int)ld_y, residual, (int)ld_res, gamma, beta, eps, out_f32, (int)ld_f32,
                                          static_cast<bf16*>(out_16), (int)ld_16, (int)M, (int)N, 1, 1, 0,
                                          static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_linear_split(const void* x16, int64_t ld_x, const void* w16, int64_t ld_w, const float* bias, int32_t act, void* y16,
                       int64_t ld_y16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K3, void* cuda_stream) {
    return op_guard([&] {
        if (K3 % 192 != 0) fail(VB200_ERR_INVALID, "vb200_linear_split: K3 = %lld is not 3 x a multiple of 64", (long long)K3);
        GemmEpilogue e{};
        e.M = (int)M; e.N = (int)N; e.K = (int)K3; e.bias = bias; e.out_bf16 = static_cast<bf16*>(y16);
        e.ld_bf16 = (int)ld_y16; e.out_f32 = y_f32; e.ld_f32 = (int)ld_y_f32; e.act = act; e.a_f16 = 1; e.out_f16 = 1;
        e.split16 = y16 != nullptr ? 1 : 0;
        e.split_acc = 1;
        // as the engine's fp32-parity GEMMs: the cooperative kernel at 64-wide tiles, the TMA store for an fp32-only output
        CUDA_CHECK(make_gemm(x16, ld_x, w16, ld_w, e, {64, 0}).launch(static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_attention_f32(const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv, int32_t in_kind,
                        const float* key_mask_add, int32_t B, int32_t Lq, int32_t Lk, int32_t heads, int32_t head_dim, void* ctx,
                        int64_t ld_ctx, int32_t ctx_mode, float* probs, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_attention_f32(q, (int)ld_q, k, v, (int)ld_kv, in_kind, key_mask_add, B, Lq, Lk, heads, head_dim,
                                            static_cast<bf16*>(ctx), (int)ld_ctx, ctx_mode, probs, 0,
                                            static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_self_attention(const void* qkv_bf16, int64_t ld_qkv, int32_t hidden, const float* mask_add, void* ctx_bf16,
                         int64_t ld_ctx, int32_t B, int32_t L, int32_t heads, int32_t head_dim, int32_t act_fp16,
                         void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_self_attention(static_cast<const bf16*>(qkv_bf16), (int)ld_qkv, hidden, mask_add,
                                             static_cast<bf16*>(ctx_bf16), (int)ld_ctx, B, L, heads, head_dim, 0,
                                             act_fp16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_co_attention(const void* qkv_img_bf16, int64_t ld_img, const void* qkv_txt_bf16, int64_t ld_txt,
                       int32_t hidden, const float* img_mask_add, const float* txt_mask_add, void* ctx_txt_bf16,
                       int64_t ld_ctx_txt, void* ctx_img_bf16, int64_t ld_ctx_img, int32_t B, int32_t T, int32_t V,
                       int32_t heads, int32_t head_dim, int32_t act_fp16, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_co_attention(static_cast<const bf16*>(qkv_img_bf16), (int)ld_img,
                                           static_cast<const bf16*>(qkv_txt_bf16), (int)ld_txt, hidden, img_mask_add,
                                           txt_mask_add, static_cast<bf16*>(ctx_txt_bf16), (int)ld_ctx_txt,
                                           static_cast<bf16*>(ctx_img_bf16), (int)ld_ctx_img, B, T, V, heads, head_dim, 0,
                                           act_fp16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_self_attention_packed(const void* qkv16, int64_t ld_qkv, int32_t hidden, const float* mask_add, void* ctx16, int64_t ld_ctx,
                                int32_t B, int32_t L_cap, int32_t heads, int32_t head_dim, int32_t act_fp16, const int32_t* offs,
                                void* cuda_stream) {
    return op_guard([&] {
        if (offs == nullptr) fail(VB200_ERR_INVALID, "vb200_self_attention_packed: offs is NULL");
        CUDA_CHECK(vb::launch_self_attention(static_cast<const bf16*>(qkv16), (int)ld_qkv, hidden, mask_add, static_cast<bf16*>(ctx16),
                                             (int)ld_ctx, B, L_cap, heads, head_dim, 0, act_fp16 ? 1 : 0,
                                             static_cast<cudaStream_t>(cuda_stream), offs));
    });
}

int vb200_co_attention_packed(const void* qkv_img16, int64_t ld_img, const void* qkv_txt16, int64_t ld_txt, int32_t hidden,
                              const float* img_mask_add, const float* txt_mask_add, void* ctx_txt16, int64_t ld_ctx_txt, void* ctx_img16,
                              int64_t ld_ctx_img, int32_t B, int32_t T_cap, int32_t V_cap, int32_t heads, int32_t head_dim,
                              int32_t act_fp16, const int32_t* offs_t, const int32_t* offs_v, void* cuda_stream) {
    return op_guard([&] {
        if (offs_t == nullptr || offs_v == nullptr) fail(VB200_ERR_INVALID, "vb200_co_attention_packed: offs_t / offs_v is NULL");
        CUDA_CHECK(vb::launch_co_attention(static_cast<const bf16*>(qkv_img16), (int)ld_img, static_cast<const bf16*>(qkv_txt16),
                                           (int)ld_txt, hidden, img_mask_add, txt_mask_add, static_cast<bf16*>(ctx_txt16),
                                           (int)ld_ctx_txt, static_cast<bf16*>(ctx_img16), (int)ld_ctx_img, B, T_cap, V_cap, heads,
                                           head_dim, 0, act_fp16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream), offs_t, offs_v));
    });
}

int vb200_self_attention_stream(const void* qkv16, int64_t ld_qkv, int32_t hidden, const float* mask_add, void* ctx16, int64_t ld_ctx,
                                int32_t B, int32_t L_cap, int32_t heads, int32_t head_dim, int32_t act_fp16, const int32_t* offs,
                                void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_self_attention_stream(static_cast<const bf16*>(qkv16), (int)ld_qkv, hidden, mask_add,
                                                    static_cast<bf16*>(ctx16), (int)ld_ctx, B, L_cap, heads, head_dim, 0,
                                                    act_fp16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream), offs));
    });
}

int vb200_co_attention_stream(const void* qkv_img16, int64_t ld_img, const void* qkv_txt16, int64_t ld_txt, int32_t hidden,
                              const float* img_mask_add, const float* txt_mask_add, void* ctx_txt16, int64_t ld_ctx_txt, void* ctx_img16,
                              int64_t ld_ctx_img, int32_t B, int32_t T_cap, int32_t V_cap, int32_t heads, int32_t head_dim,
                              int32_t act_fp16, const int32_t* offs_t, const int32_t* offs_v, void* cuda_stream) {
    return op_guard([&] {
        if ((offs_t == nullptr) != (offs_v == nullptr))
            fail(VB200_ERR_INVALID, "vb200_co_attention_stream: offs_t and offs_v must both be NULL (dense) or both be set (packed)");
        CUDA_CHECK(vb::launch_co_attention_stream(static_cast<const bf16*>(qkv_img16), (int)ld_img, static_cast<const bf16*>(qkv_txt16),
                                                  (int)ld_txt, hidden, img_mask_add, txt_mask_add, static_cast<bf16*>(ctx_txt16),
                                                  (int)ld_ctx_txt, static_cast<bf16*>(ctx_img16), (int)ld_ctx_img, B, T_cap, V_cap,
                                                  heads, head_dim, 0, act_fp16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream), offs_t,
                                                  offs_v));
    });
}

int vb200_linear_product(const void* x16, int64_t ld_x, const void* w16, int64_t ld_w, const float* bias, int32_t act, const float* mul,
                         int64_t ld_mul, void* y16, int64_t ld_y16, float* y_f32, int64_t ld_y_f32, int64_t M, int64_t N, int64_t K,
                         int32_t block_n, int32_t act_fp16, void* cuda_stream) {
    return op_guard([&] {
        if (mul == nullptr) fail(VB200_ERR_INVALID, "vb200_linear_product: mul is NULL");
        // as PlanBuilder::linear builds the pooled product: the cooperative kernel (ping-pong takes no product), its tile width, its TMA store
        const int bn = block_n > 0 ? block_n : vb::gemm_p_pick_block_n(static_cast<int>(N));
        if (bn != 64 && bn != 128 && bn != 192) fail(VB200_ERR_INVALID, "vb200_linear_product: block_n %d (plain tiles are 64, 128 or 192 wide)", bn);
        GemmEpilogue e{};
        e.M = (int)M; e.N = (int)N; e.K = (int)K; e.bias = bias; e.act = act; e.mul = mul; e.ld_mul = (int)ld_mul;
        e.a_f16 = act_fp16 ? 1 : 0; e.out_f16 = e.a_f16;
        e.out_bf16 = static_cast<bf16*>(y16); e.ld_bf16 = (int)ld_y16; e.out_f32 = y_f32; e.ld_f32 = (int)ld_y_f32;
        CUDA_CHECK(make_gemm(x16, ld_x, w16, ld_w, e, {bn, -1}).launch(static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_text_embed(const int64_t* ids, const int64_t* seg, const int64_t* input_mask, const int64_t* task, const float* word,
                     const float* pos, const float* type, const float* task_tab, const float* gamma, const float* beta, float eps,
                     float* out_f32, void* out16, float* mask_add, int32_t B, int32_t Tin, int32_t H, int32_t vocab, int32_t max_pos,
                     int32_t n_type, int32_t n_task, int32_t task_tokens, int32_t act_fp16, int32_t split16, const int32_t* offs,
                     int32_t rows, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_text_embed(ids, seg, input_mask, task, word, pos, type, task_tab, gamma, beta, eps, out_f32,
                                         static_cast<bf16*>(out16), mask_add, B, Tin, H, vocab, max_pos, n_type, n_task, task_tokens,
                                         act_fp16 ? 1 : 0, split16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream), offs, rows));
    });
}

int vb200_image_pack(const float* feats, const float* loc, const uint8_t* image_mask, void* a_out, float* mask_add, int32_t rows,
                     int32_t F, int32_t Kp, int32_t act_fp16, int32_t split16, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_image_pack(feats, loc, image_mask, static_cast<bf16*>(a_out), mask_add, rows, F, Kp, act_fp16 ? 1 : 0,
                                         split16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_region_pack(const float* box_feats, const float* boxes, const float* image_wh, const int32_t* num_boxes, void* a_out,
                      float* mask_add, float* spatials_out, int32_t B, int32_t n, int32_t F, int32_t Kp, int32_t act_fp16, int32_t split16,
                      const int32_t* offs, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_region_pack(box_feats, boxes, image_wh, num_boxes, static_cast<bf16*>(a_out), mask_add, spatials_out, B, n,
                                          F, Kp, act_fp16 ? 1 : 0, split16 ? 1 : 0, static_cast<cudaStream_t>(cuda_stream), offs));
    });
}

int vb200_rowdot(const float* x, int64_t ld_x, const float* w, const float* bias, const float* add, float* out, int64_t ld_out,
                 int64_t M, int64_t K, int32_t n_out, const int32_t* m_rows, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_rowdot(x, (int)ld_x, w, bias, add, out, (int)ld_out, (int)M, (int)K, n_out, 0,
                                     static_cast<cudaStream_t>(cuda_stream), m_rows));
    });
}

int vb200_gather_state(const int32_t* idx, int32_t n_src, const float* src_f32, const void* src16, const float* src_mask, float* dst_f32,
                       void* dst16, float* dst_mask, int32_t B, int32_t L, int32_t H, int32_t H16, void* cuda_stream) {
    return op_guard([&] {
        CUDA_CHECK(vb::launch_gather_state(idx, n_src, src_f32, src16, src_mask, dst_f32, dst16, dst_mask, B, L, H, H16,
                                           static_cast<cudaStream_t>(cuda_stream)));
    });
}

int vb200_gather_packed_state(int32_t B, const int32_t* t_dst_offs, const int32_t* t_src_offs, const float* t_src_f32, const void* t_src16,
                              float* t_dst_f32, void* t_dst16, int32_t t_n32, int32_t t_n16, const int32_t* i_dst_offs,
                              const int32_t* i_src_offs, const float* i_src_f32, const void* i_src16, float* i_dst_f32, void* i_dst16,
                              int32_t i_n32, int32_t i_n16, void* cuda_stream) {
    return op_guard([&] {
        const vb::PackedStateCopy text{t_dst_offs, t_src_offs, t_src_f32, t_src16, t_dst_f32, t_dst16, t_n32, t_n16};
        const vb::PackedStateCopy image{i_dst_offs, i_src_offs, i_src_f32, i_src16, i_dst_f32, i_dst16, i_n32, i_n16};
        CUDA_CHECK(vb::launch_gather_packed_state(text, image, B, static_cast<cudaStream_t>(cuda_stream)));
    });
}

}  // extern "C"
