// audiodec_b200 host side: model plans, weight ingest/packing, the C ABI (include/audiodec_b200.h).
//
// The reference builds torch modules from config.yml and runs ~60 nn.Conv1d calls per encode/decode,
// each preceded by a torch.cat of its pad_buffer (layers/conv_layer.py:153-156).  Here a model is a
// flat list of `Op`s over three ping-pong activation buffers in HBM (channels-last), each Op one
// kernel launch that reads its causal history from a per-stream state buffer and writes the next one.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "../../include/audiodec_b200.h"
#include "kernels.cuh"
#include "wg_conv.cuh"
#include <cuda_fp16.h>
#include <cuda_bf16.h>

using namespace adec;

namespace {
thread_local std::string g_create_error;

std::string fmt(const char* f, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, f);
    vsnprintf(buf, sizeof buf, f, ap);
    va_end(ap);
    return buf;
}

struct HostTensor {
    std::vector<int64_t> shape;
    std::vector<float> data;
    int64_t numel() const { int64_t n = 1; for (auto s : shape) n *= s; return n; }
};

int round_up(int v, int m) { return (v + m - 1) / m * m; }
bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }
int ilog2(int v) { int l = 0; while ((1 << l) < v) ++l; return l; }

// ------------------------------------------------------------------------------------------------
// kernel dispatch table
// ------------------------------------------------------------------------------------------------
typedef cudaError_t (*ConvLaunchFn)(const ConvArgs&, dim3, int, cudaStream_t);

template <int CW, int CO, int TT, int KC, bool F>
cudaError_t launch_conv(const ConvArgs& a, dim3 grid, int window_rows, cudaStream_t s) {
    using Cfg = ConvCfg<CW, CO, TT, KC>;
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    auto kern = conv_gemm_kernel<CW, CO, TT, KC, F>;
    if (dev < 64 && !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return e;
        configured[dev] = true;
    }
    const size_t smem = Cfg::smem_bytes(window_rows);
    if (smem > 227 * 1024) return cudaErrorInvalidConfiguration;
    kern<<<grid, Cfg::NTHREADS, smem, s>>>(a);
    return cudaGetLastError();
}

struct ConvKernelCfg { int CW, CO, TT, KC; bool fuse; ConvLaunchFn fn; };

#define ADEC_PLAIN(CW) \
    {CW, 256, 64, 8, false, launch_conv<CW, 256, 64, 8, false>}, \
    {CW, 128, 64, 16, false, launch_conv<CW, 128, 64, 16, false>}, \
    {CW, 64, 128, 32, false, launch_conv<CW, 64, 128, 32, false>}, \
    {CW, 32, 256, 32, false, launch_conv<CW, 32, 256, 32, false>}

const ConvKernelCfg kConvKernels[] = {
    ADEC_PLAIN(32), ADEC_PLAIN(64), ADEC_PLAIN(96), ADEC_PLAIN(128), ADEC_PLAIN(256),
    {32, 32, 256, 32, true, launch_conv<32, 32, 256, 32, true>},
    {64, 64, 128, 32, true, launch_conv<64, 64, 128, 32, true>},
    {128, 128, 64, 16, true, launch_conv<128, 128, 64, 16, true>},
    {256, 256, 64, 8, true, launch_conv<256, 256, 64, 8, true>},
};

const ConvKernelCfg* find_conv_kernel(int CW, int CO, bool fuse) {
    for (const auto& k : kConvKernels)
        if (k.CW == CW && k.CO == CO && k.fuse == fuse) return &k;
    return nullptr;
}

// tensor-core engine (wg_conv.cuh): PREC_F16 = two fp16 pieces per operand, three products (fp32-grade, default); PREC_TF32 = 3xTF32
// (ADEC_CONV_PATH=tf32); PREC_BF16 = bf16 operands, one product (the bf16 modes of the vocoder and the symAD decoder-only handle;
// BST = bf16 activations in HBM as well).
// Persistent: one CTA per SM loops over (time tile, channel tile, stream) tiles.
typedef cudaError_t (*TcPersistFn)(const ConvArgs&, int, int, int, int, int, cudaStream_t);
template <int NT, bool F, int PRE, int PREC, bool BST, bool VL, bool PAIR = false>
cudaError_t launch_wg(const ConvArgs& a, int n_xtiles, int n_ytiles, int n_tiles, int n_ctas, int smem_bytes, cudaStream_t s) {
    static bool configured[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    auto kern = wg_conv_kernel<NT, F, PRE, PREC, BST, VL, PAIR>;
    constexpr int kMaxDyn = 227 * 1024;
    if (dev < 64 && !configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDyn);
        if (e != cudaSuccess) return e;
        configured[dev] = true;
    }
    if (smem_bytes > kMaxDyn) return cudaErrorInvalidConfiguration;
    // Programmatic dependent launch: the next launch's CTAs may start (barrier init, first weight stages - weights are constants) while
    // the tail of the previous kernel of the stream is still running; its producer and consumer warps execute griddepcontrol.wait
    // before they touch any activation or state (wg_conv.cuh), which blocks until the previous grid has completed.
    static const bool pdl = [] { const char* e = getenv("ADEC_PDL"); return !e || atoi(e) != 0; }();
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)n_ctas);
    cfg.blockDim = dim3((unsigned)WgCfg<NT, PREC>::THREADS);
    cfg.dynamicSmemBytes = (size_t)smem_bytes;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, a, n_xtiles, n_ytiles, n_tiles);
}
typedef size_t (*TcSmemFn)(int, bool, bool, int);
typedef int (*TcWbufFn)(int, bool, bool, int);
// the paired instantiation (two output rows per MMA row): built for the fused fp16-split RU(32) only
template <int NT, bool F, int PRE, int PREC, bool BST>
constexpr TcPersistFn pair_fn() {
    if constexpr (NT == 32 && F && PREC == PREC_F16 && !BST) return launch_wg<NT, F, PRE, PREC, BST, false, true>;
    else return nullptr;
}
// pfn_vl: the varlen instantiation (adec_*_offline_varlen); pfn_pair: the paired one, or nullptr
struct TcKernelCfg { int NT; bool fuse; int pre, prec; bool bst; int tap_bytes; TcPersistFn pfn, pfn_vl, pfn_pair; TcSmemFn smem; TcWbufFn n_wbuf; };
#define ADEC_TC1(NT, F, PRE, PREC, BST) \
    {NT, F, PRE, PREC, BST, WgCfg<NT, PREC>::TAP_BYTES, launch_wg<NT, F, PRE, PREC, BST, false>, launch_wg<NT, F, PRE, PREC, BST, true>, \
     pair_fn<NT, F, PRE, PREC, BST>(), WgCfg<NT, PREC>::smem_bytes, WgCfg<NT, PREC>::n_wbuf}
#define ADEC_TC_FP32(NT, PREC) \
    ADEC_TC1(NT, true, ACT_ELU, PREC, false), ADEC_TC1(NT, false, ACT_NONE, PREC, false), ADEC_TC1(NT, false, ACT_ELU, PREC, false), \
    ADEC_TC1(NT, false, ACT_LRELU, PREC, false), ADEC_TC1(NT, false, ACT_NORM, PREC, false)
// bf16: the vocoder's layers (none / LeakyReLU / norm) and the symAD decoder's (fused residual unit, ELU before the split unit's
// launches and symAAD's transposed convs)
#define ADEC_TC_BF16(NT, BST) \
    ADEC_TC1(NT, false, ACT_NONE, PREC_BF16, BST), ADEC_TC1(NT, false, ACT_LRELU, PREC_BF16, BST), ADEC_TC1(NT, false, ACT_NORM, PREC_BF16, BST), \
    ADEC_TC1(NT, true, ACT_ELU, PREC_BF16, BST), ADEC_TC1(NT, false, ACT_ELU, PREC_BF16, BST)
#define ADEC_TC(NT) ADEC_TC_FP32(NT, PREC_F16), ADEC_TC_FP32(NT, PREC_TF32), ADEC_TC_BF16(NT, false), ADEC_TC_BF16(NT, true)
const TcKernelCfg kTcKernels[] = {ADEC_TC(128), ADEC_TC(64), ADEC_TC(32)};

const TcKernelCfg* find_tc_kernel(int NT, bool fuse, int pre, int prec, bool bst) {
    for (const auto& k : kTcKernels)
        if (k.NT == NT && k.fuse == fuse && k.pre == pre && k.prec == prec && k.bst == bst) return &k;
    return nullptr;
}

uint16_t half_bits(float x) { const __half h = __float2half_rn(x); uint16_t u; memcpy(&u, &h, 2); return u; }
float half_value(uint16_t u) { __half h; memcpy(&h, &u, 2); return __half2float(h); }
uint16_t bf16_bits(float x) { const __nv_bfloat16 h = __float2bfloat16_rn(x); uint16_t u; memcpy(&u, &h, 2); return u; }

float tf32_round_host(float x) {   // cvt.rna.tf32.f32: round to nearest (ties away), 10-bit mantissa
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7F800000u) == 0x7F800000u) return x;
    u = (u + 0x1000u) & 0xFFFFE000u;
    float r;
    memcpy(&r, &u, 4);
    return r;
}

// ------------------------------------------------------------------------------------------------
// Op: one kernel launch of the plan
// ------------------------------------------------------------------------------------------------
enum OpKind { OP_STEM, OP_CONV, OP_HEAD };
enum { BUF_EXT_IN = -10, BUF_EXT_OUT = -11, BUF_NONE = -1 };

// One reference pad_buffer an op's causal state holds (the state map, adec_state_entry): the key (1, C, P) channels-first is rows
// [zrows, zrows + P) of the op's (P_op, st_C) channels-last state, its channel g * cg + c at column col0 + g * gstride + c.
//   plain layers:       groups 1, col0 0, zrows 0
//   MultiGroupConv1d:   groups G; convs1.0 reads one shared input, so its key holds G copies of it (x.repeat, multi_fusion.py:134):
//                       gstride 0, export writes every copy, import reads copy 0
//   AD v0 (synthesize_mrf_as_groups): one key per block b with kernel k_b; the op keeps (K - 1) dil rows, the key the last
//                       (k_b - 1) dil of them (zrows = (K - k_b) dil) in group b (col0 = b Cin).  Import zeroes the older rows, which
//                       only meet zero taps.  convs1.0's blocks share one input: only the block with the largest kernel is imported.
struct StKey {
    std::string key;
    int C = 0, P = 0, groups = 1, cg = 0, col0 = 0, gstride = 0, zrows = 0;
    bool import = true;
};

struct Op {
    OpKind kind = OP_CONV;
    std::string name;
    // logical description (per group, after channel padding)
    int G = 1, Cin = 0, Cin_eff = 0, Cout = 0, Ktaps = 1, dil = 1, RG = 1;
    int P = 0;        // history rows (of x~)
    int down = 1;     // Tout = (T-1)/down + 1
    int up = 1;       // rows after reinterpretation = Tout*up (transposed conv)
    bool fuse = false, shared_in = false, out_nct = false, post_tanh = false;
    int pre_act = ACT_NONE, mid_act = ACT_NONE;
    float slope = 0.f;
    // host weights until finalize
    std::vector<float> weff;    // [G][Ktaps][Cin_eff][Cout]
    std::vector<float> weff2;   // fuse: [Cout][Cout] as [ci][co]
    std::vector<float> hbias;   // [G*Cout] or empty
    std::vector<float> hstate;  // initial state (P, st_C) or empty (zeros)
    // kernel config
    const ConvKernelCfg* kc = nullptr;
    const TcKernelCfg* tc = nullptr;   // tensor-core path; kc = FFMA path
    int n_pieces = 1, n_co_tiles = 1;
    // device
    float *w = nullptr, *w2 = nullptr, *bias = nullptr;
    float* cscale = nullptr;   // fp16-split engine: 2^-p of each output column, [G*Cout] as the bias (fuse: then [Cout] of w2)
    float* w_pair = nullptr;   // the fused RU(32): paired taps [W_j | W_j-1] for the paired kernel (TcKernelCfg::pfn_pair)
    const float *mean = nullptr, *scale = nullptr;
    float head_bias = 0.f;
    long long w_tile_floats = 0;
    int st_C = 0, st_groups = 1;
    float* st[2] = {nullptr, nullptr};
    int cur = 0;
    std::vector<StKey> keys;    // the reference pad_buffers this op's state holds
    // wiring
    int in_buf = BUF_NONE, out_buf = BUF_NONE, res_buf = BUF_NONE;
    int ldx = 0, x_goff = 0, ldy = 0, y_goff = 0, ldr = 0, r_goff = 0;
};

struct DevBuf {
    float* p = nullptr;
    size_t cap = 0;
};

// Stream slots of one op list (encoder or decoder): bit[s] = 1 when stream s's current state is in st[cur ^ 1] of every stateful op
// of the list rather than st[cur].  Slot calls advance a subset of streams without flipping op.cur: they flip the bits of the streams
// they advance instead.  Calls that know nothing of slots (uniform encode / decode, adec_set_streams) first copy the flipped streams
// back into st[cur] (only when a slot call has happened since the last time: `dirty`).
struct SlotBits {
    std::vector<uint8_t> bit;
    bool dirty = false;
};

}  // namespace

struct adec_handle {
    adec_config cfg{};
    int device = 0;
    bool finalized = false;
    std::string err;
    std::map<std::string, HostTensor> tensors;
    std::set<std::string> consumed;
    std::vector<Op> enc_ops, dec_ops;
    int n_streams = 1;
    int st_cap = 1;        // streams the state buffers were allocated for
    int engine = 2;               // ADEC_CONV_PATH: 2 = f16 (fp16-split wgmma, default), 1 = tf32 (3xTF32 wgmma), 0 = ffma (CUDA cores)
    int tc_max_fuse = 128;        // ADEC_TC_MAXFUSE: residual units wider than this run as two launches on the tensor-core engines
    bool bf16 = false;            // cfg.compute_dtype >= 1: bf16 operands (HiFi-GAN vocoder and symAD decoder-only, f16 engine only)
    bool act_bf16 = false;        // cfg.compute_dtype == 2: bf16 activations, causal state and decode I/O as well
    int act_bytes() const { return act_bf16 ? 2 : 4; }   // bytes per stored activation / state element
    bool stack_rows = true;       // ADEC_STACK_ROWS=0: never stack several streams' rows into one tile (A/B)
    unsigned long long* d_ktrace = nullptr;   // ADEC_KTRACE=1: per-launch {start ns, end ns, SM cycles} records (diagnostics)
    int ktrace_n = 0;
    int n_sms = 132;
    DevBuf ws[3];
    // bumped by every reallocation a captured stream step bakes in (ws[*] growth, state buffers in resize_state): a graph captured
    // at another generation re-captures before its next launch (adec_graph_launch)
    uint64_t gen = 0;
    std::vector<void*> owned;     // device allocations freed in destroy
    // rvq
    float *d_embed = nullptr, *d_e2 = nullptr, *d_codebook = nullptr;
    float *d_mean = nullptr, *d_scale = nullptr;
    int* d_err = nullptr;
    int64_t launches = 0;
    bool profiling = false;       // per-op CUDA-event timing (adec_profile)
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
    std::vector<std::string> prof_names;
    std::vector<double> prof_bytes;   // algorithmic bytes of each recorded launch (SURVEY 8(d) per-layer model)
    // host-path scratch
    DevBuf hx, hz, hzq, hy;
    DevBuf vl_tab;                // varlen row tables of the last call (ints)
    DevBuf mom_tab;               // row offsets of the last adec_zq_moments call (ints)
    DevBuf conceal_tab;           // row descriptors of the last adec_lookup_packed_conceal call (adec_conceal_row)
    DevBuf playout_tab;           // row descriptors of the last adec_lookup_packed_playout / _timescale call (adec_playout_row)
    SlotBits enc_slots, dec_slots;
    DevBuf slot_tab;              // stream pairs of the last state copy (ints)
    // the state map: every reference pad_buffer the handle runs, in plan order (encoder ops, then decoder ops), one stream's exported
    // vector holding them one after the other; st_tiles: the 32 x 32 tiles of the export / import kernels (adec_get_stream_state)
    struct StMapEntry { int list, op, k; long long off; };
    std::vector<StMapEntry> st_map;
    std::vector<int4> st_tiles;
    long long st_elems = 0;
    DevBuf st_tab;                // entries, tiles and streams of the last export / import
    long long* hidx = nullptr;
    size_t hidx_cap = 0;
    std::vector<int>* launch_log = nullptr;   // run_ops appends one ADEC_TEST_REC record per launch here (adec_record_launches)
    std::vector<int> launch_rec;

    int fail(const std::string& m) { err = m; return 1; }
};

namespace {

#define CK(h, call)                                                                        \
    do {                                                                                   \
        cudaError_t e_ = (call);                                                           \
        if (e_ != cudaSuccess) return (h)->fail(fmt("%s failed: %s", #call, cudaGetErrorString(e_))); \
    } while (0)

int dev_alloc(adec_handle* h, float** p, size_t n_floats) {
    CK(h, cudaMalloc((void**)p, std::max<size_t>(n_floats, 4) * sizeof(float)));
    h->owned.push_back(*p);
    return 0;
}

int dev_upload(adec_handle* h, float** p, const std::vector<float>& v) {
    if (dev_alloc(h, p, v.size())) return 1;
    if (!v.empty()) CK(h, cudaMemcpy(*p, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}

int ensure(adec_handle* h, DevBuf& b, size_t n_floats) {
    if (b.cap >= n_floats) return 0;
    if (b.p) CK(h, cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    CK(h, cudaMalloc((void**)&b.p, n_floats * sizeof(float)));
    b.cap = n_floats;
    if (&b >= h->ws && &b < h->ws + 3) ++h->gen;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// weight access (state-dict keys), weight-norm folding
// ------------------------------------------------------------------------------------------------
const HostTensor* find(adec_handle* h, const std::string& key) {
    auto it = h->tensors.find(key);
    if (it == h->tensors.end()) return nullptr;
    h->consumed.insert(key);
    return &it->second;
}

// returns the effective weight for "<prefix>.weight" or folds "<prefix>.weight_g/_v"
// (torch.nn.utils.weight_norm, dim=0: w = v * (g / ||v||), norm over all dims but 0; HiFiGAN.py:193-203)
int get_weight(adec_handle* h, const std::string& prefix, HostTensor* out) {
    if (const HostTensor* w = find(h, prefix + ".weight")) { *out = *w; return 0; }
    const HostTensor* g = find(h, prefix + ".weight_g");
    const HostTensor* v = find(h, prefix + ".weight_v");
    if (!g || !v) return h->fail("missing key " + prefix + ".weight (or .weight_g/.weight_v)");
    const int64_t n0 = v->shape[0], inner = v->numel() / n0;
    if (g->numel() != n0) return h->fail("bad weight_g shape for " + prefix);
    *out = *v;
    for (int64_t i = 0; i < n0; ++i) {
        double ss = 0;
        for (int64_t j = 0; j < inner; ++j) ss += (double)v->data[i * inner + j] * v->data[i * inner + j];
        const float scale = g->data[i] / (float)std::sqrt(ss);
        for (int64_t j = 0; j < inner; ++j) out->data[i * inner + j] = v->data[i * inner + j] * scale;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Op builders
// ------------------------------------------------------------------------------------------------
// causal conv, weight (Cout_total, Cin_g, K)  (layers/conv_layer.py:118-156)
int make_conv_op(adec_handle* h, Op* op, const std::string& name, const HostTensor& W, const HostTensor* bias,
                 int stride, int dil, int groups, int pre_act, float slope, bool shared_in) {
    if (W.shape.size() != 3) return h->fail("conv weight must be 3-D: " + name);
    const int cout_t = (int)W.shape[0], cin_g = (int)W.shape[1], K = (int)W.shape[2];
    if (cout_t % groups) return h->fail("Cout not divisible by groups: " + name);
    const int cout_g = cout_t / groups;
    op->kind = OP_CONV;
    op->name = name;
    op->G = groups;
    op->pre_act = pre_act;
    op->slope = slope;
    op->shared_in = shared_in;
    op->Cout = round_up(cout_g, 32);
    if (stride == 1) {
        op->RG = 1; op->Ktaps = K; op->dil = dil; op->P = (K - 1) * dil; op->down = 1;
        op->Cin = round_up(cin_g, 32);
        op->Cin_eff = op->Cin;
    } else {
        // k = 2s strided conv (encoder.py:62-68) -> 2-tap conv over s-row groups
        if (K != 2 * stride || dil != 1) return h->fail(fmt("%s: strided conv needs kernel=2*stride, dilation 1", name.c_str()));
        if (!is_pow2(cin_g) || cin_g < 4) return h->fail(fmt("%s: strided conv needs power-of-two Cin>=4", name.c_str()));
        op->RG = stride; op->Ktaps = 2; op->dil = 1; op->P = K - 1; op->down = stride;
        op->Cin = cin_g;
        op->Cin_eff = round_up(stride * cin_g, 32);
    }
    op->weff.assign((size_t)groups * op->Ktaps * op->Cin_eff * op->Cout, 0.f);
    for (int g = 0; g < groups; ++g)
        for (int co = 0; co < cout_g; ++co)
            for (int ci = 0; ci < cin_g; ++ci)
                for (int k = 0; k < K; ++k) {
                    const float v = W.data[((size_t)(g * cout_g + co) * cin_g + ci) * K + k];
                    int tap, q;
                    if (stride == 1) { tap = k; q = ci; }
                    else { tap = k / stride; q = (k % stride) * cin_g + ci; }
                    op->weff[(((size_t)g * op->Ktaps + tap) * op->Cin_eff + q) * op->Cout + co] = v;
                }
    if (bias) {
        op->hbias.assign((size_t)groups * op->Cout, 0.f);
        for (int g = 0; g < groups; ++g)
            for (int co = 0; co < cout_g; ++co) op->hbias[(size_t)g * op->Cout + co] = bias->data[g * cout_g + co];
    }
    op->st_groups = shared_in ? 1 : groups;
    op->st_C = op->st_groups * op->Cin;
    return 0;
}

// causal transposed conv, weight (Cin, Cout, 2s)  (layers/conv_layer.py:162-197)
//   y[j*s+r] = b + W[:,:,r]^T x[j] + W[:,:,s+r]^T x[j-1]      (x[j-1] = tap 0, x[j] = tap 1)
int make_convtr_op(adec_handle* h, Op* op, const std::string& name, const HostTensor& W, const HostTensor* bias,
                   int stride, int pre_act, float slope) {
    if (W.shape.size() != 3 || W.shape[2] != 2 * stride) return h->fail(name + ": transposed conv needs kernel = 2*stride");
    const int cin = (int)W.shape[0], cout = (int)W.shape[1], K = 2 * stride;
    op->kind = OP_CONV;
    op->name = name;
    op->G = 1; op->RG = 1; op->Ktaps = 2; op->dil = 1; op->P = 1; op->down = 1; op->up = stride;
    op->pre_act = pre_act; op->slope = slope;
    op->Cin = round_up(cin, 32);
    op->Cin_eff = op->Cin;
    op->Cout = round_up(stride * cout, 32);
    op->weff.assign((size_t)2 * op->Cin_eff * op->Cout, 0.f);
    for (int ci = 0; ci < cin; ++ci)
        for (int co = 0; co < cout; ++co)
            for (int r = 0; r < stride; ++r) {
                op->weff[((size_t)0 * op->Cin_eff + ci) * op->Cout + r * cout + co] = W.data[((size_t)ci * cout + co) * K + stride + r];
                op->weff[((size_t)1 * op->Cin_eff + ci) * op->Cout + r * cout + co] = W.data[((size_t)ci * cout + co) * K + r];
            }
    if (bias) {
        op->hbias.assign(op->Cout, 0.f);
        for (int r = 0; r < stride; ++r)
            for (int co = 0; co < cout; ++co) op->hbias[r * cout + co] = bias->data[co];
    }
    op->st_groups = 1;
    op->st_C = op->Cin;
    return 0;
}

// residual unit (models/autoencoder/modules/residual_unit.py:49-81): x + W2 * act(conv_k7_dil(act(x)))
int make_ru_op(adec_handle* h, Op* op, const std::string& name, const HostTensor& W1, const HostTensor& W2, int dil, int act) {
    if (make_conv_op(h, op, name, W1, nullptr, 1, dil, 1, act, 0.f, false)) return 1;
    const int c = (int)W1.shape[0];
    if (W1.shape[1] != c || W2.shape[0] != c || W2.shape[1] != c || W2.shape[2] != 1 || c != op->Cout)
        return h->fail(name + ": residual unit needs square weights with C % 32 == 0");
    op->fuse = true;
    op->mid_act = act;
    op->weff2.assign((size_t)c * c, 0.f);
    for (int co = 0; co < c; ++co)
        for (int ci = 0; ci < c; ++ci) op->weff2[(size_t)ci * c + co] = W2.data[(size_t)co * c + ci];
    return 0;
}

// Tensor-core path, C > 128: the fused unit would need 2*C > 256 accumulator registers per drain thread, so it runs
// as two launches: k7 dilated conv (ELU on load) -> mid, then 1x1 conv (ELU on load) + skip.
void split_ru_op(const Op& ru, Op* conv, Op* pw) {
    *conv = ru;
    conv->fuse = false;
    conv->weff2.clear();
    conv->mid_act = ACT_NONE;
    *pw = Op();
    pw->kind = OP_CONV;
    pw->name = ru.name + ".conv2";
    pw->G = 1; pw->Cin = ru.Cout; pw->Cin_eff = ru.Cout; pw->Cout = ru.Cout; pw->Ktaps = 1; pw->dil = 1; pw->RG = 1; pw->P = 0;
    pw->pre_act = ru.mid_act; pw->slope = ru.slope;
    pw->weff = ru.weff2;            // [ci][co] == [1 tap][Cin_eff][Cout]
    pw->st_groups = 1; pw->st_C = ru.Cout;
}

int pick_piece_width(const Op& op) {
    static const int cands[] = {256, 128, 96, 64, 32};
    for (int cw : cands) {
        if (op.Cin_eff % cw) continue;
        if (op.RG > 1 && !(cw % op.Cin == 0 || op.Cin % cw == 0)) continue;
        return cw;
    }
    return 0;
}

// wgmma engines (wg_conv.cuh): weights in K-major, no-swizzle blocks of 16 bytes, the layout WgCfg streams:
//   [group g][co tile][piece][tap][plane][kb = 16-byte K block][ntw columns][16 B]
// ntw: columns per tile (NT; 2 NT for the paired taps); one (piece, tap) at ntw = NT is TAP_BYTES.  The planes of a weight w:
// 3xTF32 hi | lo (4 bytes each), fp16 hi | lo | hi * 2^-11 of w * 2^p (2 bytes each), or one bf16 plane.  p: [G * cout], the power
// of two of each output column (fp16 only).
std::vector<float> pack_wg(int prec, const float* weff, int G, int ntiles, int pieces, int taps, int cin_eff, int cout,
                           const std::vector<int>& p, int ntw) {
    const int eb = prec == PREC_TF32 ? 4 : 2, npl = prec == PREC_F16 ? 3 : prec == PREC_TF32 ? 2 : 1;
    const int epb = 16 / eb, KB = TC_CP / epb;     // elements per block, K blocks per piece
    const size_t plane = (size_t)KB * ntw * epb;    // elements
    std::vector<uint8_t> img((size_t)G * ntiles * pieces * taps * npl * plane * eb, 0);
    size_t o = 0;     // in elements
    for (int g = 0; g < G; ++g)
        for (int nt = 0; nt < ntiles; ++nt)
            for (int pc = 0; pc < pieces; ++pc)
                for (int tap = 0; tap < taps; ++tap) {
                    for (int kb = 0; kb < KB; ++kb)
                        for (int n = 0; n < ntw; ++n)
                            for (int e = 0; e < epb; ++e) {
                                const int k = pc * TC_CP + kb * epb + e;
                                const float w = nt * ntw + n < cout ? weff[(((size_t)g * taps + tap) * cin_eff + k) * cout + nt * ntw + n] : 0.f;
                                uint32_t v[3];
                                if (prec == PREC_TF32) {
                                    const float hi = tf32_round_host(w), lo = tf32_round_host(w - hi);
                                    memcpy(&v[0], &hi, 4);
                                    memcpy(&v[1], &lo, 4);
                                } else if (prec == PREC_F16) {
                                    const float ws = nt * ntw + n < cout ? std::ldexp(w, p[(size_t)g * cout + nt * ntw + n]) : 0.f;
                                    v[0] = half_bits(ws);
                                    v[1] = half_bits(ws - half_value(v[0]));
                                    v[2] = half_bits(half_value(v[0]) * (1.0f / 2048.0f));
                                } else {
                                    v[0] = bf16_bits(w);
                                }
                                for (int pl = 0; pl < npl; ++pl) {
                                    uint8_t* at = img.data() + (o + pl * plane + ((size_t)kb * ntw + n) * epb + e) * eb;
                                    for (int i = 0; i < eb; ++i) at[i] = (uint8_t)(v[pl] >> (8 * i));    // little-endian, as the device reads it
                                }
                            }
                    o += npl * plane;
                }
    std::vector<float> out(img.size() / 4);
    memcpy(out.data(), img.data(), img.size());
    return out;
}

// wgmma engines: choose the kernel instantiation and the weight scales, pack and upload the weights
int finalize_op_wg(adec_handle* h, Op* op) {
    int NT = op->Cout % 128 == 0 ? 128 : op->Cout % 64 == 0 ? 64 : 32;
    // 96 outputs (transposed conv 64 -> 3*32): one zero-padded 128-wide tile beats three 32-wide tiles that each rebuild the
    // same activation window (the epilogue masks per column pair)
    const bool pad_tile = !op->fuse && NT == 32 && op->Cout > 64 && op->Cout < 128;
    if (pad_tile) NT = 128;
    const int prec = h->engine == 1 ? PREC_TF32 : h->bf16 ? PREC_BF16 : PREC_F16;
    // bf16 storage reads a window row as whole 16-byte vectors of one s * Cin row: no 4-channel strided convs
    if (h->act_bf16 && op->RG > 1 && op->Cin < 8) return h->fail(op->name + ": bf16 activations need strided convs with Cin >= 8");
    op->tc = find_tc_kernel(NT, op->fuse, op->pre_act, prec, h->act_bf16);
    if (!op->tc || (op->fuse && (NT != op->Cout || op->mid_act != op->pre_act))) return h->fail(op->name + ": no tensor-core kernel");
    op->n_pieces = op->Cin_eff / TC_CP;
    op->n_co_tiles = pad_tile ? 1 : op->Cout / NT;
    op->w_tile_floats = (long long)((size_t)op->n_pieces * op->Ktaps * op->tc->tap_bytes / 4);
    // fp16 planes hold the weights of output column c times 2^p_c, max |w * 2^p_c| over the column in [4096, 8192), so that a column
    // far below the op's largest weight keeps its W_lo plane normal; the kernel scales column c's sums back by 2^-p_c (cscale).
    // p_c stays in [-127, 126]: 2^-p_c is a normal float.  A zero or non-finite column: p_c = 0.  The other precisions: p = 0
    // (w: [G][taps][cin][cols], column g * cols + co)
    auto pow2_scales = [prec](const std::vector<float>& w, int G, int cols) {
        std::vector<float> wmax((size_t)G * cols, 0.f);
        const size_t per_g = w.size() / G;
        for (size_t i = 0; i < w.size(); ++i) {
            float& m = wmax[i / per_g * cols + i % cols];
            m = std::max(m, std::fabs(w[i]));
        }
        std::vector<int> p(wmax.size(), 0);
        for (size_t c = 0; c < p.size(); ++c)
            if (prec == PREC_F16 && wmax[c] > 0.f && std::isfinite(wmax[c])) {
                while (p[c] < 126 && std::ldexp(wmax[c], p[c]) < 4096.f) ++p[c];
                while (p[c] > -127 && std::ldexp(wmax[c], p[c]) >= 8192.f) --p[c];
            }
        return p;
    };
    std::vector<int> p1 = pow2_scales(op->weff, op->G, op->Cout), p2;
    if (op->fuse) p2 = pow2_scales(op->weff2, 1, op->Cout);
    if (prec == PREC_F16) {
        std::vector<float> cs;
        for (int p : p1) cs.push_back(std::ldexp(1.0f, -p));
        for (int p : p2) cs.push_back(std::ldexp(1.0f, -p));
        if (dev_upload(h, &op->cscale, cs)) return 1;
    }
    if (dev_upload(h, &op->w, pack_wg(prec, op->weff.data(), op->G, op->n_co_tiles, op->n_pieces, op->Ktaps, op->Cin_eff, op->Cout, p1, NT)))
        return 1;
    if (op->tc->pfn_pair && op->Ktaps % 2 == 1) {
        // the paired kernel's K + 1 taps [W_j | W_j-1] (W_-1 = W_K = 0), 2 NT columns each, both halves with column co's scale;
        // uniform rows run it, stacked and varlen rows the unpaired kernel with the same one-tap groups (WgCfg::tpg), so both give the
        // same sums
        const int C = op->Cout, Ci = op->Cin_eff, K = op->Ktaps;
        std::vector<float> wp((size_t)(K + 1) * Ci * 2 * C, 0.f);
        for (int j = 0; j <= K; ++j)
            for (int ci = 0; ci < Ci; ++ci)
                for (int co = 0; co < C; ++co) {
                    float* row = wp.data() + ((size_t)j * Ci + ci) * 2 * C;
                    if (j < K) row[co] = op->weff[((size_t)j * Ci + ci) * C + co];
                    if (j > 0) row[C + co] = op->weff[((size_t)(j - 1) * Ci + ci) * C + co];
                }
        std::vector<int> pp(p1);
        pp.insert(pp.end(), p1.begin(), p1.end());
        if (dev_upload(h, &op->w_pair, pack_wg(prec, wp.data(), 1, 1, op->n_pieces, K + 1, Ci, 2 * C, pp, 2 * NT))) return 1;
    }
    if (op->fuse && dev_upload(h, &op->w2, pack_wg(prec, op->weff2.data(), 1, 1, op->Cout / TC_CP, 1, op->Cout, op->Cout, p2, NT)))
        return 1;
    return 0;
}

// FFMA engine (conv_gemm_kernel): choose the kernel instantiation, pack and upload the weights
int finalize_op_ffma(adec_handle* h, Op* op) {
    int CW, CO;
    if (op->fuse) {
        CW = CO = op->Cout;
    } else {
        CW = pick_piece_width(*op);
        CO = op->Cout % 256 == 0 ? 256 : op->Cout % 128 == 0 ? 128 : op->Cout % 64 == 0 ? 64 : 32;
    }
    op->kc = CW ? find_conv_kernel(CW, CO, op->fuse) : nullptr;
    if (!op->kc) return h->fail(fmt("%s: no kernel for Cin_eff=%d Cout=%d fuse=%d", op->name.c_str(), op->Cin_eff, op->Cout, (int)op->fuse));
    op->n_pieces = op->Cin_eff / CW;
    op->n_co_tiles = op->Cout / CO;
    const int KC = op->kc->KC, nkc = CW / KC;
    op->w_tile_floats = (long long)op->Ktaps * op->Cin_eff * CO;
    std::vector<float> packed((size_t)op->G * op->n_co_tiles * op->w_tile_floats);
    size_t o = 0;
    for (int g = 0; g < op->G; ++g)
        for (int ct = 0; ct < op->n_co_tiles; ++ct)
            for (int pc = 0; pc < op->n_pieces; ++pc)
                for (int tap = 0; tap < op->Ktaps; ++tap)
                    for (int kcc = 0; kcc < nkc; ++kcc)
                        for (int k = 0; k < KC; ++k) {
                            const int q = pc * CW + kcc * KC + k;
                            const float* src = &op->weff[(((size_t)g * op->Ktaps + tap) * op->Cin_eff + q) * op->Cout + ct * CO];
                            for (int co = 0; co < CO; ++co) packed[o++] = src[co];
                        }
    if (dev_upload(h, &op->w, packed)) return 1;
    if (op->fuse && dev_upload(h, &op->w2, op->weff2)) return 1;   // [ci][co] == [chunk][kc][co] for CO == C
    return 0;
}

int finalize_op(adec_handle* h, Op* op) {
    if (op->kind != OP_CONV) return 0;
    if (h->engine != 0 ? finalize_op_wg(h, op) : finalize_op_ffma(h, op)) return 1;
    if (!op->hbias.empty() && dev_upload(h, &op->bias, op->hbias)) return 1;
    std::vector<float>().swap(op->weff);
    std::vector<float>().swap(op->weff2);
    return 0;
}

int alloc_state(adec_handle* h, Op* op, int n_streams) {
    const size_t per = (size_t)op->P * op->st_C, eb = h->act_bytes();
    if (per == 0) return 0;
    for (int i = 0; i < 2; ++i) {
        CK(h, cudaMalloc((void**)&op->st[i], per * n_streams * eb));     // owned by the op: freed on resize / destroy
        CK(h, cudaMemset(op->st[i], 0, per * n_streams * eb));
    }
    op->cur = 0;
    if (!op->hstate.empty()) {
        std::vector<uint16_t> hb;       // bf16 activations: the checkpoint's pad_buffer rounded once, like `.to(torch.bfloat16)`
        if (h->act_bf16) for (float v : op->hstate) hb.push_back(bf16_bits(v));
        const void* src = h->act_bf16 ? (const void*)hb.data() : (const void*)op->hstate.data();
        for (int s = 0; s < n_streams; ++s)
            CK(h, cudaMemcpy((char*)op->st[0] + s * per * eb, src, per * eb, cudaMemcpyHostToDevice));
    }
    return 0;
}

// Register reference key `key` of op `op` (see StKey; the key's reference shape is (1, groups * cg, P)) and load it from the state dict
// as the op's initial state.  The reference stores in pad_buffer the tail of what it feeds to conv.inference, i.e. values AFTER the
// pre-activation / normalisation (residual_unit.py:79 `conv1.inference(self.activation(x))`, HiFiGAN.py:276-284,288), and the kernels keep
// exactly that: state rows are never activated again (only chunk rows are, while the window is written), so checkpoint values are copied as
// they are.  A batched (B, C, P) buffer loads its row 0 here; the Python layer imports every row per stream (load_state_dict).
void add_pad_buffer(adec_handle* h, Op* op, StKey k) {
    if (!k.P) k.P = op->P - k.zrows;
    if (!k.C) k.C = k.groups * k.cg;
    const HostTensor* pb = find(h, k.key);
    op->keys.push_back(k);
    if (!k.import || !pb || pb->shape.size() != 3 || op->P == 0) return;
    const int C = (int)pb->shape[1], P = (int)pb->shape[2];
    if (P != k.P) return;
    bool any = false;
    for (int64_t i = 0; i < (int64_t)C * P && i < pb->numel(); ++i) any |= (pb->data[i] != 0.f);
    if (!any) return;
    if (op->hstate.empty()) op->hstate.assign((size_t)op->P * op->st_C, 0.f);
    const int groups = k.gstride ? k.groups : 1;      // a shared input: copy 0
    for (int g = 0; g < groups; ++g)
        for (int c = 0; c < k.cg && g * k.cg + c < C; ++c)
            for (int p = 0; p < P; ++p)
                op->hstate[(size_t)(k.zrows + p) * op->st_C + k.col0 + g * k.gstride + c] = pb->data[((size_t)(g * k.cg + c)) * P + p];
}

// a plain layer, or a MultiGroupConv1d conv (op->G groups of c_real channels; shared_in: copies of one input)
void load_pad_buffer(adec_handle* h, Op* op, const std::string& key, int c_real) {
    StKey k;
    k.key = key; k.cg = c_real;
    k.groups = op->kind == OP_CONV ? op->G : 1;
    k.gstride = op->shared_in ? 0 : op->Cin;
    add_pad_buffer(h, op, k);
}

// ------------------------------------------------------------------------------------------------
// plan execution
// ------------------------------------------------------------------------------------------------
// What a codec call runs over, and so what it does to the causal state (run_call):
//   CALL_STREAM   B = n_streams uniform streams, each advanced by T rows                       (adec_encode / adec_decode)
//   CALL_OFFLINE  B uniform utterances from zero history; transposed convs replicate their first input row instead of reading state
//   CALL_VARLEN   CALL_OFFLINE over B utterances of their own lengths, concatenated along time  (adec_*_offline_varlen)
//   CALL_SLOTS    B distinct streams of the handle, each advanced by a chunk of its own length  (adec_*_streams)
enum CallMode { CALL_STREAM, CALL_OFFLINE, CALL_VARLEN, CALL_SLOTS };

struct RunCtx {
    int B;
    const float* ext_in;
    float* ext_out;
    cudaStream_t stream;
    CallMode mode = CALL_STREAM;
    const int* lengths = nullptr;  // CALL_VARLEN / CALL_SLOTS: HOST lengths of the B utterances, concatenated along time in ext_in / ext_out
    const int* slots = nullptr;    // CALL_SLOTS: HOST stream slot of each utterance
    const char* what = "";         // entry point, for messages
    bool varlen() const { return mode == CALL_VARLEN || mode == CALL_SLOTS; }
};

SlotBits* slot_bits(adec_handle* h, const std::vector<Op>& ops) {
    return &ops == &h->enc_ops ? &h->enc_slots : &ops == &h->dec_ops ? &h->dec_slots : nullptr;
}

// Copy per-stream state rows of every stateful op of `ops`: pair j copies stream pairs[2j] of st[cur ^ src_sel] to stream pairs[2j + 1]
// of st[cur ^ dst_sel].  The pairs go up in one copy on `stream`.
int slot_copy(adec_handle* h, std::vector<Op>& ops, const std::vector<int>& pairs, int src_sel, int dst_sel, cudaStream_t stream) {
    const int n = (int)pairs.size() / 2;
    if (n == 0) return 0;
    if (ensure(h, h->slot_tab, pairs.size())) return 1;
    CK(h, cudaMemcpyAsync(h->slot_tab.p, pairs.data(), pairs.size() * sizeof(int), cudaMemcpyHostToDevice, stream));
    for (Op& op : ops) {
        const long long per = (long long)op.P * op.st_C * h->act_bytes() / 4;     // words per stream (see resize_state)
        if (!per) continue;
        const long long tot = per * n;
        slot_copy_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(op.st[op.cur ^ dst_sel], op.st[op.cur ^ src_sel], per,
                                                                          reinterpret_cast<const int*>(h->slot_tab.p), n);
        CK(h, cudaGetLastError());
        ++h->launches;
    }
    return 0;
}

// Put every stream's current state back into st[cur] (the layout the uniform calls and adec_set_streams know): one copy of the streams
// whose bit is set, and only if a slot call has happened since the last time.
int slot_fixup(adec_handle* h, std::vector<Op>& ops, cudaStream_t stream) {
    SlotBits* sb = slot_bits(h, ops);
    if (!sb || !sb->dirty) return 0;
    std::vector<int> pairs;
    for (int s = 0; s < (int)sb->bit.size(); ++s)
        if (sb->bit[s]) { pairs.push_back(s); pairs.push_back(s); }
    if (slot_copy(h, ops, pairs, 1, 0, stream)) return 1;
    std::fill(sb->bit.begin(), sb->bit.end(), 0);
    sb->dirty = false;
    return 0;
}

// varlen row spaces must stay inside the kernels' 32-bit row indices, with room for a tile and its halo past the end
constexpr long long kVlMaxRows = (1ll << 31) - 4096;

// Per-op row tables of a varlen call: utterance b's input rows [in[b], in[b + 1]) and output rows [out[b], out[b + 1]) of every op,
// the arithmetic of the uniform path (Tout = (T - 1) / down + 1, then T = Tout * up) applied per utterance.  Fails on a row space
// that does not fit the kernels' 32-bit row indices.
struct VlPlan {
    std::vector<int> tab;                 // per op: in (B + 1) | out (B + 1)
    std::vector<long long> T, Tout;       // per op: total input / output rows
};
int plan_varlen(adec_handle* h, const std::vector<Op>& ops, const RunCtx& rc, VlPlan* pl) {
    const int B = rc.B;
    std::vector<long long> len(rc.lengths, rc.lengths + B);
    pl->tab.assign(ops.size() * 2 * (B + 1), 0);
    for (size_t k = 0; k < ops.size(); ++k) {
        const Op& op = ops[k];
        const long long halo = op.kind == OP_CONV ? (long long)(op.Ktaps - 1) * op.dil : 0;
        int* in = pl->tab.data() + k * 2 * (B + 1);
        int* out = in + B + 1;
        long long si = 0, so = 0;
        for (int b = 0; b < B; ++b) {
            const long long tout = (len[b] - 1) / op.down + 1;
            si += len[b];
            so += tout;
            if (si > kVlMaxRows || so * op.up > kVlMaxRows || so + (b + 1) * halo > kVlMaxRows)
                return h->fail(fmt("%s: the batch needs more than %lld rows at %s, beyond the kernels' 32-bit row indexing; split it",
                                   rc.what, kVlMaxRows, op.name.c_str()));
            in[b + 1] = (int)si;
            out[b + 1] = (int)so;
            len[b] = tout * op.up;
        }
        pl->T.push_back(si);
        pl->Tout.push_back(so);
    }
    return 0;
}

// Grow the activation workspaces to what `ops` need over B uniform streams of T_in rows, or over the varlen row tables `pl`
int size_ws(adec_handle* h, const std::vector<Op>& ops, int B, int T_in, const VlPlan* pl) {
    size_t need[3] = {0, 0, 0};
    int T = T_in;
    for (size_t k = 0; k < ops.size(); ++k) {
        const Op& op = ops[k];
        const int Tout = (T - 1) / op.down + 1;
        const size_t rows = pl ? (size_t)pl->Tout[k] : (size_t)B * Tout;
        if (op.out_buf >= 0) need[op.out_buf] = std::max(need[op.out_buf], rows * op.ldy);
        T = Tout * op.up;
    }
    for (int i = 0; i < 3; ++i)     // need[] counts elements; the buffers are sized in floats
        if (need[i] && ensure(h, h->ws[i], (need[i] * h->act_bytes() + 3) / 4)) return 1;
    return 0;
}

// The launches of one call.  Reads each stateful op's history from st[cur] (slot calls: from the buffer the stream's slot bit names)
// and writes the new state to the other buffer; what that does to `cur` and the slot bits is the caller's (run_call).
int run_ops(adec_handle* h, std::vector<Op>& ops, const RunCtx& rc, int T_in, int* T_out_final) {
    // pass 1: workspace sizes (varlen: the row tables, uploaded in one copy on the call's stream)
    const bool vl = rc.varlen();
    VlPlan pl;
    if (vl) {
        if (plan_varlen(h, ops, rc, &pl)) return 1;
        for (const Op& op : ops)
            if (op.kind == OP_CONV && !op.tc)
                return h->fail(fmt("%s: the FFMA engine (ADEC_CONV_PATH=ffma) has no varlen kernels; use the f16 or tf32 tensor-core engine",
                                   rc.what));
    }
    if (size_ws(h, ops, rc.B, T_in, vl ? &pl : nullptr)) return 1;
    if (!vl && rc.B != h->n_streams) return h->fail(fmt("batch %d != n_streams %d (call adec_set_streams)", rc.B, h->n_streams));
    const int* vl_tab = nullptr;
    const int* vl_slot = nullptr;
    if (vl) {
        size_t at = 0;
        if (rc.mode == CALL_SLOTS) {
            // the slot table (2 * slot + bit per utterance, the same for every op) follows the row tables in the one copy
            for (const Op& op : ops)      // the conv kernels address a slot's history rows with 32-bit element offsets
                if ((long long)h->n_streams * op.P * op.st_C >= (1ll << 31))
                    return h->fail(fmt("%s: %d streams of %s state exceed 2^31 elements per buffer; use fewer streams per handle", rc.what,
                                       h->n_streams, op.name.c_str()));
            const SlotBits* sb = slot_bits(h, ops);
            at = pl.tab.size();
            for (int b = 0; b < rc.B; ++b) pl.tab.push_back(2 * rc.slots[b] + sb->bit[rc.slots[b]]);
        }
        if (ensure(h, h->vl_tab, pl.tab.size())) return 1;
        CK(h, cudaMemcpyAsync(h->vl_tab.p, pl.tab.data(), pl.tab.size() * sizeof(int), cudaMemcpyHostToDevice, rc.stream));
        vl_tab = reinterpret_cast<const int*>(h->vl_tab.p);
        if (rc.mode == CALL_SLOTS) vl_slot = vl_tab + at;
    }

    int T = T_in;
    for (size_t k = 0; k < ops.size(); ++k) {
        Op& op = ops[k];
        int Tout = (T - 1) / op.down + 1;
        const int* vl_in = vl ? vl_tab + k * 2 * (rc.B + 1) : nullptr;
        const int* vl_out = vl ? vl_in + rc.B + 1 : nullptr;
        if (vl) { T = (int)pl.T[k]; Tout = (int)pl.Tout[k]; }
        const int nb = vl ? 1 : rc.B;                        // varlen: one row space of concatenated utterances
        const float* xin = op.in_buf == BUF_EXT_IN ? rc.ext_in : h->ws[op.in_buf].p;
        float* yout = op.out_buf == BUF_EXT_OUT ? rc.ext_out : h->ws[op.out_buf].p;
        const float* st_in = op.st[op.cur];
        float* st_out = op.st[op.cur ^ 1];
        cudaError_t e = cudaSuccess;
        cudaEvent_t ev0 = nullptr, ev1 = nullptr;
        if (h->profiling) {
            cudaEventCreate(&ev0); cudaEventCreate(&ev1);
            cudaEventRecord(ev0, rc.stream);
        }
        if (op.kind == OP_STEM) {
            StemArgs a{};
            a.x = xin; a.x_bs = T; a.st_in = st_in; a.st_out = st_out; a.T = T;
            a.w = op.w; a.bias = op.bias; a.y = yout; a.y_bs = (long long)T * op.ldy;
            a.vl_off = vl_in; a.vl_B = rc.B; a.vl_slot = vl_slot;
            dim3 grid((T + 1023) / 1024, nb);
            if (vl && h->act_bf16) stem_kernel<32, 7, true, true><<<grid, 256, 0, rc.stream>>>(a);
            else if (vl) stem_kernel<32, 7, true><<<grid, 256, 0, rc.stream>>>(a);
            else if (h->act_bf16) stem_kernel<32, 7, false, true><<<grid, 256, 0, rc.stream>>>(a);
            else stem_kernel<32, 7><<<grid, 256, 0, rc.stream>>>(a);
            e = cudaGetLastError();
        } else if (op.kind == OP_HEAD) {
            HeadArgs a{};
            a.x = xin; a.x_bs = (long long)T * op.ldx; a.ldx = op.ldx; a.st_in = st_in; a.st_out = st_out; a.T = T;
            a.w = op.w; a.bias = op.head_bias; a.pre_act = op.pre_act; a.slope = op.slope; a.post_tanh = op.post_tanh;
            a.y = yout; a.y_bs = T;
            a.vl_off = vl_in; a.vl_B = rc.B; a.vl_slot = vl_slot;
            dim3 grid((T + 255) / 256, nb);
            if (vl && h->act_bf16) head_kernel<32, 7, true, true><<<grid, 256, 0, rc.stream>>>(a);
            else if (vl) head_kernel<32, 7, false, true><<<grid, 256, 0, rc.stream>>>(a);
            else if (h->act_bf16) head_kernel<32, 7, true><<<grid, 256, 0, rc.stream>>>(a);
            else head_kernel<32, 7, false><<<grid, 256, 0, rc.stream>>>(a);
            e = cudaGetLastError();
        } else {
            ConvArgs a{};
            a.x = xin; a.x_bs = (long long)T * op.ldx; a.ldx = op.ldx; a.x_goff = op.x_goff;
            a.st_in = st_in; a.st_out = st_out; a.st_ld = op.st_C; a.st_goff = op.shared_in ? 0 : op.Cin; a.st_groups = op.st_groups;
            a.P = op.P; a.T = T; a.Tout = Tout;
            a.Ktaps = op.Ktaps; a.dil = op.dil; a.RG = op.RG; a.lgCin = ilog2(op.Cin); a.Cin = op.Cin;
            a.n_pieces = op.n_pieces; a.pre_act = op.pre_act; a.slope = op.slope; a.mean = op.mean; a.scale = op.scale;
            a.w = op.w; a.w2 = op.w2; a.bias = op.bias; a.n_co_tiles = op.n_co_tiles; a.Cout_g = op.Cout;
            a.w_tile_floats = op.w_tile_floats;
            if (op.fuse) { a.res = xin; a.res_bs = a.x_bs; a.ldr = op.ldx; a.r_goff = 0; }
            else if (op.res_buf >= 0) { a.res = h->ws[op.res_buf].p; a.res_bs = (long long)Tout * op.ldr; a.ldr = op.ldr; a.r_goff = op.r_goff; }
            a.y = yout; a.ldy = op.ldy; a.y_goff = op.y_goff; a.out_nct = op.out_nct;
            a.y_bs = op.out_nct ? (long long)op.G * op.Cout * Tout : (long long)Tout * op.ldy;
            a.mid_act = op.mid_act;
            a.hist_rep = ((rc.mode == CALL_OFFLINE || rc.mode == CALL_VARLEN) && op.up > 1) ? 1 : 0;
            a.cscale = op.cscale; a.err = h->d_err;
            if (h->d_ktrace && h->ktrace_n < 4096) a.dbg = h->d_ktrace + KT_REC * (size_t)(h->ktrace_n++);
            if (op.tc) {
                // persistent tensor-core kernels: one CTA per SM loops over (time tile, channel tile, stream) tiles
                int wrows = TC_TT + (op.Ktaps - 1) * op.dil;
                dim3 grid((Tout + TC_TT - 1) / TC_TT, op.G * op.n_co_tiles, rc.B);
                a.n_streams = rc.B;
                if (vl) {
                    // one stacked row space: utterance b owns Tout_b + halo rows (ConvArgs::vl_in / vl_out)
                    const long long rows = (long long)Tout + (long long)rc.B * (op.Ktaps - 1) * op.dil;
                    grid = dim3((unsigned)((rows + TC_TT - 1) / TC_TT), grid.y, 1);
                    a.n_streams = 1;
                    a.vl_in = vl_in; a.vl_out = vl_out; a.vl_B = rc.B; a.vl_slot = vl_slot;
                } else if (h->stack_rows) {
                    // fill the 128-row tiles across streams when that needs fewer tiles (short chunks: 256 streams x 5..25 rows per layer)
                    const long long L = (long long)Tout + (long long)(op.Ktaps - 1) * op.dil;
                    const long long stacked = (rc.B * L + TC_TT - 1) / TC_TT;
                    // (stacked tiles take the per-row edge path in the producers: only worth it when at least a quarter of the tiles go away)
                    if (stacked * 4 <= (long long)grid.x * rc.B * 3 && rc.B * L < (1ll << 30)) {
                        a.stack_L = (int)L;
                        grid = dim3((unsigned)stacked, grid.y, 1);
                    }
                }
                // uniform rows of the fused RU(32): the paired kernel, tiles of pair_tt(dil) rows, its window stored as two arrays
                const bool pair = op.w_pair && !vl && !a.stack_L;
                if (pair) {
                    a.w = op.w_pair;
                    wrows = 2 * pair_rows(op.Ktaps, op.dil);
                    grid.x = (unsigned)((Tout + pair_tt(op.dil) - 1) / pair_tt(op.dil));
                }
                const long long n_tiles = (long long)grid.x * grid.y * grid.z;
                const int n_ctas = (int)std::min<long long>(n_tiles, h->n_sms);
                // the fp16-split engine's per-column scales (Op::cscale) live in shared memory during the launch
                const int sbytes = op.cscale ? (int)(((size_t)(op.G + (op.fuse ? 1 : 0)) * op.Cout * sizeof(float) + 15) / 16 * 16) : 0;
                const size_t psmem = op.tc->smem(wrows, op.fuse, pair, sbytes);
                a.n_wbuf = op.tc->n_wbuf(wrows, op.fuse, pair, sbytes);
                if (a.n_wbuf < 1) return h->fail(fmt("%s: window of %d rows does not fit in shared memory", op.name.c_str(), wrows));
                e = (vl ? op.tc->pfn_vl : pair ? op.tc->pfn_pair : op.tc->pfn)(a, (int)grid.x, (int)grid.y, (int)n_tiles, n_ctas, (int)psmem, rc.stream);
                if (h->launch_log)
                    h->launch_log->insert(h->launch_log->end(), {ADEC_TEST_LAUNCH_TC, op.tc->NT, op.tc->fuse, op.tc->pre, op.tc->prec, vl, pair,
                                                                 a.stack_L > 0, op.tc->bst});
            } else {
                const int TT = op.kc->TT;
                dim3 grid((Tout + TT - 1) / TT, op.G * op.n_co_tiles, rc.B);
                e = op.kc->fn(a, grid, TT + (op.Ktaps - 1) * op.dil, rc.stream);
                if (h->launch_log)
                    h->launch_log->insert(h->launch_log->end(), {ADEC_TEST_LAUNCH_FFMA, op.kc->CO, op.kc->fuse, op.pre_act, 0, 0, 0, 0, 0});
            }
        }
        if (h->launch_log && op.kind != OP_CONV)
            h->launch_log->insert(h->launch_log->end(), {op.kind == OP_STEM ? ADEC_TEST_LAUNCH_STEM : ADEC_TEST_LAUNCH_HEAD, 0, 0, op.pre_act,
                                                         0, vl, 0, 0, h->act_bf16});
        if (e != cudaSuccess) return h->fail(fmt("launch of %s failed: %s", op.name.c_str(), cudaGetErrorString(e)));
        ++h->launches;
        if (h->profiling) {
            cudaEventRecord(ev1, rc.stream);
            h->prof_events.emplace_back(ev0, ev1);
            h->prof_names.push_back(op.name);
            // algorithmic bytes: eb*(Cin*Tin + Cout*Tout [+ Cout*Tout residual]) per stream (fused unit: its two convs + skip), eb = 4 for
            // fp32 activations, 2 for bf16
            const double cin = op.kind == OP_STEM ? 1 : (double)op.G * op.Cin_eff / std::max(1, op.RG) * (op.shared_in ? 1.0 / op.G : 1.0);
            const double cout = op.kind == OP_HEAD ? 1 : (double)op.G * op.Cout;
            const double eb = h->act_bytes();
            double bytes = eb * nb * (cin * T + cout * Tout);
            if (op.fuse) bytes += eb * nb * (3.0 * cout * Tout);      // mid write+read (1x1 conv in/out) and the skip read
            else if (op.res_buf >= 0) bytes += eb * nb * cout * Tout;
            h->prof_bytes.push_back(bytes);
        }
        T = Tout * op.up;
    }
    if (T_out_final) *T_out_final = T;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// model builders
// ------------------------------------------------------------------------------------------------
int need_tensor(adec_handle* h, const std::string& key, const HostTensor** out) {
    *out = find(h, key);
    if (!*out) return h->fail("missing key " + key);
    return 0;
}

int build_stem(adec_handle* h, Op* op, const std::string& prefix, int cout) {
    HostTensor Wt;
    if (get_weight(h, prefix + ".conv", &Wt)) return 1;
    const HostTensor* W = &Wt;
    if (W->shape[0] != 32 || W->shape[1] != 1 || W->shape[2] != 7 || cout != 32)
        return h->fail("stem conv: only input_channels=1, encode_channels=32, kernel 7 is built");
    op->kind = OP_STEM; op->name = prefix; op->P = 6; op->st_C = 1; op->Cin = 1; op->Cout = 32;
    std::vector<float> w(7 * 32);
    for (int co = 0; co < 32; ++co)
        for (int k = 0; k < 7; ++k) w[k * 32 + co] = W->data[co * 7 + k];
    if (dev_upload(h, &op->w, w)) return 1;
    if (const HostTensor* b = find(h, prefix + ".conv.bias")) { if (dev_upload(h, &op->bias, b->data)) return 1; }
    load_pad_buffer(h, op, prefix + ".pad_buffer", 1);
    return 0;
}

int build_head(adec_handle* h, Op* op, const std::string& prefix, int pre_act, float slope, bool tanh_out) {
    HostTensor W;
    if (get_weight(h, prefix + ".conv", &W)) return 1;
    if (W.shape[0] != 1 || W.shape[1] != 32 || W.shape[2] != 7)
        return h->fail("head conv: only 32 -> 1 channels, kernel 7 is built");
    op->kind = OP_HEAD; op->name = prefix; op->P = 6; op->st_C = 32; op->Cin = 32; op->Cout = 1;
    op->pre_act = pre_act; op->slope = slope; op->post_tanh = tanh_out;
    std::vector<float> w(7 * 32);
    for (int ci = 0; ci < 32; ++ci)
        for (int k = 0; k < 7; ++k) w[k * 32 + ci] = W.data[ci * 7 + k];
    if (dev_upload(h, &op->w, w)) return 1;
    if (const HostTensor* b = find(h, prefix + ".conv.bias")) op->head_bias = b->data[0];
    op->st_groups = 1;
    load_pad_buffer(h, op, prefix + ".pad_buffer", 32);
    return 0;
}

// wiring helper: ops read `cur` and write another workspace buffer
struct Wire {
    int cur = BUF_EXT_IN;
    int cur_ld = 0;
    int pick(int avoid1 = -99, int avoid2 = -99) const {
        for (int i = 0; i < 3; ++i)
            if (i != cur && i != avoid1 && i != avoid2) return i;
        return 0;
    }
};

void chain(Op* op, Wire* w, int out_ld) {
    op->in_buf = w->cur; op->ldx = w->cur_ld; op->x_goff = op->shared_in ? 0 : op->Cin;
    op->out_buf = w->pick(); op->ldy = out_ld; op->y_goff = op->Cout;
    w->cur = op->out_buf; w->cur_ld = out_ld;
}

// append a residual unit to `ops`: one fused launch, or (tensor-core path, C > 128) conv + 1x1 launches
int push_ru(adec_handle* h, std::vector<Op>* ops, Wire* w, const std::string& ru, int dil, int ch) {
    HostTensor W1, W2;
    if (get_weight(h, ru + ".conv1.conv", &W1) || get_weight(h, ru + ".conv2", &W2)) return 1;
    Op op;
    if (make_ru_op(h, &op, ru, W1, W2, dil, ACT_ELU)) return 1;
    load_pad_buffer(h, &op, ru + ".conv1.pad_buffer", ch);
    if (h->engine != 0 && op.Cout > h->tc_max_fuse) {
        Op conv, pw;
        split_ru_op(op, &conv, &pw);
        const int x_buf = w->cur;
        chain(&conv, w, ch);
        pw.in_buf = w->cur; pw.ldx = ch; pw.x_goff = pw.Cin;
        pw.res_buf = x_buf; pw.ldr = ch; pw.r_goff = 0;
        pw.out_buf = w->pick(x_buf); pw.ldy = ch; pw.y_goff = pw.Cout;
        w->cur = pw.out_buf; w->cur_ld = ch;
        ops->push_back(std::move(conv));
        ops->push_back(std::move(pw));
    } else {
        chain(&op, w, ch);
        ops->push_back(std::move(op));
    }
    return 0;
}

constexpr int kRuDils[3] = {1, 3, 9};     // encoder.py:33, decoder.py:30

int check_symad_cfg(adec_handle* h) {
    const adec_config& c = h->cfg;
    if (c.input_channels != 1 || c.output_channels != 1) return h->fail("symAD: only mono (input/output_channels=1) is built");
    if (c.code_dim != 64) return h->fail("symAD: only code_dim=64 is built");
    return 0;
}

// ---- decoder (models/autoencoder/modules/decoder.py:84-148): what a full symAD handle and a decoder-only one (ADEC_MODEL_SYMAD_DECODER)
// both decode with
int build_symad_decoder(adec_handle* h) {
    const adec_config& c = h->cfg;
    Wire d; d.cur = BUF_EXT_IN; d.cur_ld = c.code_dim;
    {
        HostTensor W;
        if (get_weight(h, "decoder.conv1.conv", &W)) return 1;
        Op op;
        if (make_conv_op(h, &op, "decoder.conv1", W, find(h, "decoder.conv1.conv.bias"), 1, 1, 1, ACT_NONE, 0.f, false)) return 1;
        load_pad_buffer(h, &op, "decoder.conv1.pad_buffer", c.code_dim);
        chain(&op, &d, op.Cout);
        h->dec_ops.push_back(std::move(op));
    }
    for (int i = 0; i < c.n_dec; ++i) {
        // symAAD wraps each block as Sequential(ELU, DecoderBlock) -> keys "...conv_blocks.i.1.*" (decoder.py:183-195)
        const std::string pre = fmt(c.codec_activate ? "decoder.conv_blocks.%d.1" : "decoder.conv_blocks.%d", i);
        const int cin = c.decode_channels * c.dec_ratios[i];
        const int cout = i < c.n_dec - 1 ? c.decode_channels * c.dec_ratios[i + 1] : c.decode_channels;
        HostTensor W;
        if (get_weight(h, pre + ".conv.deconv", &W)) return 1;
        Op op;
        if (make_convtr_op(h, &op, pre + ".conv", W, find(h, pre + ".conv.deconv.bias"), c.dec_strides[i],
                           c.codec_activate ? ACT_ELU : ACT_NONE, 0.f)) return 1;
        if (op.Cout != c.dec_strides[i] * cout) return h->fail(pre + ": stride*Cout must be a multiple of 32");
        load_pad_buffer(h, &op, pre + ".conv.pad_buffer", cin);
        chain(&op, &d, op.Cout);
        d.cur_ld = cout;   // (T, s*Cout) is (T*s, Cout)
        h->dec_ops.push_back(std::move(op));
        for (int j = 0; j < 3; ++j)
            if (push_ru(h, &h->dec_ops, &d, pre + fmt(".res_units.%d", j), kRuDils[j], cout)) return 1;
    }
    {
        Op op;
        if (build_head(h, &op, "decoder.conv2", c.codec_activate ? ACT_ELU : ACT_NONE, 0.f, c.codec_activate != 0)) return 1;   // decoder.py:209-211
        op.in_buf = d.cur; op.ldx = d.cur_ld; op.out_buf = BUF_EXT_OUT; op.ldy = 1;
        h->dec_ops.push_back(std::move(op));
    }
    return 0;
}

// The decoder-only handle loads a full generator state dict: the encoder, projector and RVQ keys are accepted and ignored.
int build_symad_decoder_only(adec_handle* h) {
    if (check_symad_cfg(h) || build_symad_decoder(h)) return 1;
    for (const auto& kv : h->tensors)
        for (const char* pre : {"encoder.", "projector.", "quantizer."})
            if (kv.first.compare(0, strlen(pre), pre) == 0) h->consumed.insert(kv.first);
    return 0;
}

// ---- encoder (models/autoencoder/modules/encoder.py:84-142) and projector: what a full symAD handle and an encoder-only one
// (ADEC_MODEL_SYMAD_ENCODER) both encode with
int build_symad_encoder(adec_handle* h) {
    const adec_config& c = h->cfg;
    Wire w; w.cur = BUF_EXT_IN; w.cur_ld = 1;
    {
        Op op;
        if (build_stem(h, &op, "encoder.conv", c.encode_channels)) return 1;
        op.in_buf = BUF_EXT_IN; op.ldx = 1; op.out_buf = 0; op.ldy = 32;
        w.cur = 0; w.cur_ld = 32;
        h->enc_ops.push_back(std::move(op));
    }
    int ch = c.encode_channels;
    for (int i = 0; i < c.n_enc; ++i) {
        const std::string pre = fmt("encoder.conv_blocks.%d", i);
        for (int j = 0; j < 3; ++j)
            if (push_ru(h, &h->enc_ops, &w, pre + fmt(".res_units.%d", j), kRuDils[j], ch)) return 1;
        HostTensor W;
        if (get_weight(h, pre + ".conv.conv", &W)) return 1;
        const HostTensor* b = find(h, pre + ".conv.conv.bias");
        Op op;
        if (make_conv_op(h, &op, pre + ".conv", W, b, c.enc_strides[i], 1, 1, ACT_NONE, 0.f, false)) return 1;
        load_pad_buffer(h, &op, pre + ".conv.pad_buffer", ch);
        ch = c.encode_channels * c.enc_ratios[i];
        chain(&op, &w, ch);
        h->enc_ops.push_back(std::move(op));
    }
    {   // projector (projector.py:40,52-54): k=3, no bias; writes z channels-first (B,64,F)
        HostTensor W;
        if (get_weight(h, "projector.project.conv", &W)) return 1;
        Op op;   // symAAD: the encoder's trailing ELU (encoder.py:174-175) is this conv's pre-activation
        if (make_conv_op(h, &op, "projector.project", W, find(h, "projector.project.conv.bias"), 1, 1, 1,
                         c.codec_activate ? ACT_ELU : ACT_NONE, 0.f, false)) return 1;
        load_pad_buffer(h, &op, "projector.project.pad_buffer", ch);
        op.in_buf = w.cur; op.ldx = w.cur_ld; op.x_goff = op.Cin;
        op.out_buf = BUF_EXT_OUT; op.out_nct = true; op.ldy = op.Cout; op.y_goff = op.Cout;
        if (op.Cout != c.code_dim) return h->fail("projector: code_dim must be a multiple of 32");
        h->enc_ops.push_back(std::move(op));
    }
    return 0;
}

// ---- residual VQ (layers/vq_module.py): the codebooks of a full symAD handle and of an encoder-only one
int build_symad_rvq(adec_handle* h) {
    const adec_config& c = h->cfg;
    const int nq = c.codebook_num, D = c.code_dim, N = c.codebook_size;
    if (N != 1024) return h->fail("RVQ: only codebook_size=1024 is built");
    std::vector<float> embed((size_t)nq * D * N), e2((size_t)nq * N), cb((size_t)nq * N * D);
    for (int i = 0; i < nq; ++i) {
        const HostTensor* E;
        if (need_tensor(h, fmt("quantizer.codebook.layers.%d.embed", i), &E)) return 1;
        if (E->shape.size() != 2 || E->shape[0] != D || E->shape[1] != N) return h->fail("bad embed shape");
        std::copy(E->data.begin(), E->data.end(), embed.begin() + (size_t)i * D * N);
        for (int cdx = 0; cdx < N; ++cdx) {
            // embed.pow(2).sum(0) in torch's order: cascade sum over blocks of 16 rows (see oracle/rvq_oracle.c)
            float total = 0.f;
            for (int bk = 0; bk < D; bk += 16) {
                float part = 0.f;
                for (int k = bk; k < bk + 16 && k < D; ++k) {
                    volatile float sq = E->data[(size_t)k * N + cdx] * E->data[(size_t)k * N + cdx];
                    part = part + sq;
                }
                total = bk == 0 ? part : total + part;
            }
            e2[(size_t)i * N + cdx] = total;
            for (int k = 0; k < D; ++k) cb[((size_t)i * N + cdx) * D + k] = E->data[(size_t)k * N + cdx];   // vq_module.py:151-157
        }
        find(h, fmt("quantizer.codebook.layers.%d.cluster_size", i));
        find(h, fmt("quantizer.codebook.layers.%d.embed_avg", i));
    }
    if (dev_upload(h, &h->d_embed, embed) || dev_upload(h, &h->d_e2, e2) || dev_upload(h, &h->d_codebook, cb)) return 1;
    return 0;
}

int build_symad(adec_handle* h) {
    return check_symad_cfg(h) || build_symad_encoder(h) || build_symad_decoder(h) || build_symad_rvq(h);
}

// The encoder-only handle loads a full generator state dict: the decoder keys are accepted and ignored.
int build_symad_encoder_only(adec_handle* h) {
    if (check_symad_cfg(h) || build_symad_encoder(h) || build_symad_rvq(h)) return 1;
    for (const auto& kv : h->tensors)
        if (kv.first.compare(0, 8, "decoder.") == 0) h->consumed.insert(kv.first);
    return 0;
}

// AD v0 (MultiReceptiveField, multi_fusion.py:23-79): the mean of one residual block per kernel size.  A causal conv with
// kernel k equals one with kernel K >= k whose first K-k taps are zero, so the three blocks are expressed as ONE grouped
// conv stack with the largest kernel (zero-padded taps) followed by a 1x1 "conv_out" holding [I/3 I/3 I/3] - exactly
// the MultiGroupConv1d graph the kernels already run.
int synthesize_mrf_as_groups(adec_handle* h, int stage, int C, HostTensor W1[], HostTensor B1[], HostTensor W2[], HostTensor B2[],
                             HostTensor* Wout) {
    const adec_config& c = h->cfg;
    const int nb = c.n_resblocks;
    int K = 0;
    for (int b = 0; b < nb; ++b) K = std::max(K, c.resblock_kernel_sizes[b]);
    for (int j = 0; j < c.n_dil; ++j)
        for (int which = 0; which < 2; ++which) {
            HostTensor& W = which ? W2[j] : W1[j];
            HostTensor& Bt = which ? B2[j] : B1[j];
            W.shape = {nb * C, C, K};
            W.data.assign((size_t)nb * C * C * K, 0.f);
            Bt.shape = {nb * C};
            Bt.data.assign((size_t)nb * C, 0.f);
            for (int b = 0; b < nb; ++b) {
                const int kb = c.resblock_kernel_sizes[b];
                const std::string pre = fmt("blocks.%d.blocks.%d.convs%d.%d", stage, b, which + 1, j);
                HostTensor w;
                if (get_weight(h, pre + ".conv", &w)) return 1;
                if (w.shape.size() != 3 || w.shape[0] != C || w.shape[1] != C || w.shape[2] != kb) return h->fail("bad shape: " + pre);
                for (int co = 0; co < C; ++co)
                    for (int ci = 0; ci < C; ++ci)
                        for (int k = 0; k < kb; ++k)
                            W.data[((size_t)(b * C + co) * C + ci) * K + (K - kb) + k] = w.data[((size_t)co * C + ci) * kb + k];
                if (const HostTensor* bb = find(h, pre + ".conv.bias"))
                    for (int co = 0; co < C; ++co) Bt.data[b * C + co] = bb->data[co];
            }
        }
    Wout->shape = {C, nb * C, 1};
    Wout->data.assign((size_t)C * nb * C, 0.f);
    for (int co = 0; co < C; ++co)
        for (int b = 0; b < nb; ++b) Wout->data[(size_t)co * nb * C + b * C + co] = 1.0f / nb;
    return 0;
}

int build_hifigan(adec_handle* h) {
    const adec_config& c = h->cfg;
    if (c.out_channels != 1) return h->fail("HiFi-GAN: only out_channels=1 is built");
    const bool mrf = c.n_resblocks > 0;       // AD v0
    if (!mrf && c.groups < 2) return h->fail("HiFi-GAN: groups must be > 1 for the MultiGroupConv1d variant");
    if (mrf && c.groups != 1) return h->fail("HiFi-GAN: MultiReceptiveField needs groups = 1");
    const float slope = c.negative_slope;
    if (c.has_stats) {
        const HostTensor *m, *s;
        if (need_tensor(h, "mean", &m) || need_tensor(h, "scale", &s)) return 1;
        std::vector<float> mp(round_up(c.in_channels, 32), 0.f), sp(round_up(c.in_channels, 32), 1.f);
        std::copy(m->data.begin(), m->data.end(), mp.begin());
        std::copy(s->data.begin(), s->data.end(), sp.begin());
        if (dev_upload(h, &h->d_mean, mp) || dev_upload(h, &h->d_scale, sp)) return 1;
    }
    Wire w; w.cur = BUF_EXT_IN; w.cur_ld = c.in_channels;
    {   // input_conv (HiFiGAN.py:84-89, :282-284); decode_norm folded into its window load (:276-279)
        HostTensor W;
        if (get_weight(h, "input_conv.conv", &W)) return 1;
        Op op;
        if (make_conv_op(h, &op, "input_conv", W, find(h, "input_conv.conv.bias"), 1, 1, 1, c.has_stats ? ACT_NORM : ACT_NONE, 0.f, false)) return 1;
        op.mean = h->d_mean; op.scale = h->d_scale;
        load_pad_buffer(h, &op, "input_conv.pad_buffer", c.in_channels);
        chain(&op, &w, op.Cout);
        h->dec_ops.push_back(std::move(op));
    }
    for (int i = 0; i < c.n_up; ++i) {
        const int cin = c.channels >> i, cout = c.channels >> (i + 1), s = c.upsample_scales[i];
        if (c.upsample_kernel_sizes[i] != 2 * s) return h->fail("HiFi-GAN: upsample kernel must be 2*scale (HiFiGAN.py:95)");
        {
            HostTensor W;
            const std::string pre = fmt("upsamples.%d", i);
            if (get_weight(h, pre + ".deconv", &W)) return 1;
            Op op;
            if (make_convtr_op(h, &op, pre, W, find(h, pre + ".deconv.bias"), s, ACT_LRELU, slope)) return 1;
            if (op.Cout != s * cout) return h->fail(pre + ": scale*Cout must be a multiple of 32");
            load_pad_buffer(h, &op, pre + ".pad_buffer", cin);
            chain(&op, &w, op.Cout);
            w.cur_ld = cout;
            h->dec_ops.push_back(std::move(op));
        }
        // MultiGroupConv1d (multi_fusion.py:82-141): x.repeat folded away (shared_in on the first conv)
        const int G = mrf ? c.n_resblocks : c.groups, C3 = G * cout;
        HostTensor mW1[ADEC_MAX_STAGES], mB1[ADEC_MAX_STAGES], mW2[ADEC_MAX_STAGES], mB2[ADEC_MAX_STAGES], mWout;
        if (mrf && synthesize_mrf_as_groups(h, i, cout, mW1, mB1, mW2, mB2, &mWout)) return 1;
        const int A = w.cur;                 // c (T, cout)
        const int Bb = w.pick();             // xt
        const int Cc = w.pick(Bb);           // x (T, 3C)
        for (int j = 0; j < c.n_dil; ++j) {
            const std::string p1 = fmt("blocks.%d.convs1.%d", i, j), p2 = fmt("blocks.%d.convs2.%d", i, j);
            HostTensor W1, W2;
            const HostTensor *b1 = nullptr, *b2 = nullptr;
            if (mrf) {
                W1 = mW1[j]; W2 = mW2[j]; b1 = &mB1[j]; b2 = &mB2[j];
            } else {
                if (get_weight(h, p1 + ".conv", &W1) || get_weight(h, p2 + ".conv", &W2)) return 1;
                b1 = find(h, p1 + ".conv.bias"); b2 = find(h, p2 + ".conv.bias");
            }
            Op o1, o2;
            if (make_conv_op(h, &o1, p1, W1, b1, 1, c.resblock_dilations[j], G, ACT_LRELU, slope, j == 0)) return 1;
            if (make_conv_op(h, &o2, p2, W2, b2, 1, 1, G, ACT_LRELU, slope, false)) return 1;
            if (o1.Cout != cout || o1.Cin != cout) return h->fail(p1 + ": channels must be a multiple of 32");
            if (!mrf) {
                load_pad_buffer(h, &o1, p1 + ".pad_buffer", cout);
                load_pad_buffer(h, &o2, p2 + ".pad_buffer", cout);
            } else {
                // one key per block: the tail of the block's group (convs1.0: of the shared input, read from the largest kernel's block)
                int kmax = 0;
                for (int b = 1; b < G; ++b) if (c.resblock_kernel_sizes[b] > c.resblock_kernel_sizes[kmax]) kmax = b;
                for (int which = 0; which < 2; ++which) {
                    Op& o = which ? o2 : o1;
                    for (int b = 0; b < G; ++b) {
                        StKey k;
                        k.key = fmt("blocks.%d.blocks.%d.convs%d.%d.pad_buffer", i, b, which + 1, j);
                        k.cg = cout;
                        k.P = (c.resblock_kernel_sizes[b] - 1) * o.dil;
                        k.zrows = o.P - k.P;
                        k.col0 = o.shared_in ? 0 : b * o.Cin;
                        k.import = !o.shared_in || b == kmax;
                        add_pad_buffer(h, &o, k);
                    }
                }
            }
            o1.in_buf = j == 0 ? A : Cc; o1.ldx = j == 0 ? cout : C3; o1.x_goff = j == 0 ? 0 : cout;
            o1.out_buf = Bb; o1.ldy = C3; o1.y_goff = cout;
            o2.in_buf = Bb; o2.ldx = C3; o2.x_goff = cout;
            o2.res_buf = j == 0 ? A : Cc; o2.ldr = j == 0 ? cout : C3; o2.r_goff = j == 0 ? 0 : cout;
            o2.out_buf = Cc; o2.ldy = C3; o2.y_goff = cout;     // j>0: in place over the residual (element-wise safe)
            h->dec_ops.push_back(std::move(o1));
            h->dec_ops.push_back(std::move(o2));
        }
        {
            HostTensor W;
            const std::string po = fmt("blocks.%d.conv_out", i);
            if (mrf) W = mWout;
            else if (get_weight(h, po, &W)) return 1;
            Op op;
            if (make_conv_op(h, &op, po, W, find(h, po + ".bias"), 1, 1, 1, ACT_NONE, 0.f, false)) return 1;
            op.in_buf = Cc; op.ldx = C3; op.x_goff = op.Cin;
            op.out_buf = A; op.ldy = cout; op.y_goff = op.Cout;
            w.cur = A; w.cur_ld = cout;
            h->dec_ops.push_back(std::move(op));
        }
    }
    {   // output: LeakyReLU(0.01) -> conv -> tanh (HiFiGAN.py:116-123, :294-296)
        Op op;
        if (build_head(h, &op, "output_conv", ACT_LRELU, 0.01f, true)) return 1;
        op.in_buf = w.cur; op.ldx = w.cur_ld; op.out_buf = BUF_EXT_OUT; op.ldy = 1;
        h->dec_ops.push_back(std::move(op));
    }
    return 0;
}

int hop_of(const adec_handle* h) {
    int hop = 1;
    const int mt = h->cfg.model_type;
    if (mt == ADEC_MODEL_SYMAD || mt == ADEC_MODEL_SYMAD_ENCODER) for (int i = 0; i < h->cfg.n_enc; ++i) hop *= h->cfg.enc_strides[i];
    else if (mt == ADEC_MODEL_SYMAD_DECODER) for (int i = 0; i < h->cfg.n_dec; ++i) hop *= h->cfg.dec_strides[i];
    else for (int i = 0; i < h->cfg.n_up; ++i) hop *= h->cfg.upsample_scales[i];
    return hop;
}

int fail_encoder_only(adec_handle* h, const std::string& what) {
    return h->fail(what + ": a symAD encoder-only handle (ADEC_MODEL_SYMAD_ENCODER) has no decoder, lookup or unpack; use a full symAD "
                          "handle (ADEC_MODEL_SYMAD) or a decoder handle");
}

// The entry points that need the encoder, projector or the RVQ's nearest-codeword search (encode, quantize, pack): a full symAD handle
// or an encoder-only one
int need_symad_tx(adec_handle* h, const std::string& what) {
    if (h->cfg.model_type == ADEC_MODEL_SYMAD || h->cfg.model_type == ADEC_MODEL_SYMAD_ENCODER) return 0;
    if (h->cfg.model_type == ADEC_MODEL_SYMAD_DECODER)
        return h->fail(what + ": a symAD decoder-only handle (ADEC_MODEL_SYMAD_DECODER) has no encoder, projector or RVQ; use a full symAD "
                              "handle (ADEC_MODEL_SYMAD)");
    return h->fail(what + ": not a symAD handle");
}

// The entry points of a full symAD handle only: lookup, unpack, the RVQ's forward sum and its moments
int need_full_symad(adec_handle* h, const std::string& what) {
    if (h->cfg.model_type == ADEC_MODEL_SYMAD_ENCODER) return fail_encoder_only(h, what);
    return need_symad_tx(h, what);
}

// The state map from the ops' keys, and the 32 x 32 (channel, row) tiles the export / import kernels run over
void build_state_map(adec_handle* h) {
    h->st_map.clear();
    h->st_tiles.clear();
    h->st_elems = 0;
    for (int list = 0; list < 2; ++list) {
        const std::vector<Op>& ops = list ? h->dec_ops : h->enc_ops;
        for (int o = 0; o < (int)ops.size(); ++o)
            for (int k = 0; k < (int)ops[o].keys.size(); ++k) {
                const StKey& key = ops[o].keys[k];
                const int e = (int)h->st_map.size();
                h->st_map.push_back({list, o, k, h->st_elems});
                h->st_elems += (long long)key.C * key.P;
                for (int c0 = 0; c0 < key.C; c0 += 32)
                    for (int r0 = 0; r0 < key.zrows + key.P; r0 += 32) h->st_tiles.push_back(make_int4(e, c0, r0, 0));
            }
    }
}

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

}  // namespace

// ==================================================================================================
// C ABI
// ==================================================================================================
extern "C" {

int adec_create(const adec_config* cfg, int device, adec_handle** out) {
    if (!cfg || !out) { g_create_error = "null argument"; return 1; }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device < 0 || device >= ndev) {
        g_create_error = fmt("no usable CUDA device %d (%s); audiodec_b200 has no CPU fallback", device,
                             e == cudaSuccess ? "out of range" : cudaGetErrorString(e));
        return 1;
    }
    if (cfg->n_enc > ADEC_MAX_STAGES || cfg->n_dec > ADEC_MAX_STAGES || cfg->n_up > ADEC_MAX_STAGES || cfg->n_dil > ADEC_MAX_STAGES) {
        g_create_error = "too many stages";
        return 1;
    }
    auto* h = new adec_handle();
    h->cfg = *cfg;
    h->device = device;
    if (const char* pth = getenv("ADEC_CONV_PATH")) {
        if (!strcmp(pth, "ffma")) h->engine = 0;
        else if (!strcmp(pth, "tf32")) h->engine = 1;
        else if (!strcmp(pth, "f16") || !strcmp(pth, "tc") || !*pth) h->engine = 2;
        else { g_create_error = std::string("ADEC_CONV_PATH must be f16, tf32 or ffma, not ") + pth; delete h; return 1; }
    }
    if (const char* sr = getenv("ADEC_STACK_ROWS")) h->stack_rows = atoi(sr) != 0;
    if (const char* mf = getenv("ADEC_TC_MAXFUSE")) h->tc_max_fuse = atoi(mf);
    if (const char* kt = getenv("ADEC_KTRACE")) {
        if (atoi(kt)) {
            DeviceGuard dgk(device);
            if (cudaMalloc((void**)&h->d_ktrace, 4096 * KT_REC * sizeof(unsigned long long)) == cudaSuccess)
                cudaMemset(h->d_ktrace, 0, 4096 * KT_REC * sizeof(unsigned long long));    // the phase counters accumulate
        }
    }
    h->bf16 = cfg->compute_dtype == 1 || cfg->compute_dtype == 2;
    h->act_bf16 = cfg->compute_dtype == 2;
    if (cfg->compute_dtype < 0 || cfg->compute_dtype > 2) {
        g_create_error = "compute_dtype must be 0 (fp32), 1 (bf16 operands) or 2 (bf16 operands and activations)";
        delete h;
        return 1;
    }
    const bool enc_only = cfg->model_type == ADEC_MODEL_SYMAD_ENCODER;
    if (h->bf16 && ((cfg->model_type != ADEC_MODEL_HIFIGAN && cfg->model_type != ADEC_MODEL_SYMAD_DECODER && !enc_only) || h->engine != 2)) {
        g_create_error = "compute_dtype = bf16 is built for the decoder handles - the HiFi-GAN vocoder and the symAD decoder-only handle "
                         "(ADEC_MODEL_SYMAD_DECODER) - and for the symAD encoder-only handle (ADEC_MODEL_SYMAD_ENCODER), on the f16 "
                         "tensor-core engine only (the encoder, projector and RVQ of a full symAD handle must stay fp32-grade for "
                         "bit-identical indices)";
        delete h;
        return 1;
    }
    const bool symad_part = cfg->model_type == ADEC_MODEL_SYMAD_DECODER || enc_only;
    const int zq_dim = symad_part ? cfg->code_dim : cfg->in_channels;
    if (h->act_bf16 && zq_dim % 8) {      // a bf16 zq row must be whole 16-byte vectors
        g_create_error = symad_part ? "compute_dtype = 2 needs code_dim to be a multiple of 8"
                                                                     : "compute_dtype = 2 needs in_channels to be a multiple of 8";
        delete h;
        return 1;
    }
    cudaDeviceGetAttribute(&h->n_sms, cudaDevAttrMultiProcessorCount, device);
    DeviceGuard dg(device);
    if (cudaMalloc((void**)&h->d_err, sizeof(int)) != cudaSuccess || cudaMemset(h->d_err, 0, sizeof(int)) != cudaSuccess) {
        g_create_error = "cudaMalloc failed";
        delete h;
        return 1;
    }
    *out = h;
    return 0;
}

void adec_destroy(adec_handle* h) {
    if (!h) return;
    DeviceGuard dg(h->device);
    for (void* p : h->owned) cudaFree(p);
    for (auto* ops : {&h->enc_ops, &h->dec_ops})
        for (Op& op : *ops)
            for (int i = 0; i < 2; ++i) if (op.st[i]) cudaFree(op.st[i]);
    for (auto& b : h->ws) if (b.p) cudaFree(b.p);
    for (DevBuf* b : {&h->hx, &h->hz, &h->hzq, &h->hy, &h->vl_tab, &h->mom_tab, &h->conceal_tab, &h->playout_tab,
                      &h->slot_tab, &h->st_tab}) if (b->p) cudaFree(b->p);
    if (h->hidx) cudaFree(h->hidx);
    if (h->d_err) cudaFree(h->d_err);
    if (h->d_ktrace) cudaFree(h->d_ktrace);
    delete h;
}

const char* adec_last_error(const adec_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int adec_set_tensor(adec_handle* h, const char* key, const float* data, const int64_t* shape, int ndim) {
    if (!h || !key || !data || ndim < 0 || ndim > 4) return h ? h->fail("bad argument to adec_set_tensor") : 1;
    if (h->finalized) return h->fail("adec_set_tensor after adec_finalize");
    HostTensor t;
    t.shape.assign(shape, shape + ndim);
    t.data.assign(data, data + t.numel());
    h->tensors[key] = std::move(t);
    return 0;
}

int adec_finalize(adec_handle* h) {
    if (!h) return 1;
    if (h->finalized) return h->fail("already finalized");
    DeviceGuard dg(h->device);
    int rc = h->cfg.model_type == ADEC_MODEL_SYMAD ? build_symad(h)
           : h->cfg.model_type == ADEC_MODEL_HIFIGAN ? build_hifigan(h)
           : h->cfg.model_type == ADEC_MODEL_SYMAD_DECODER ? build_symad_decoder_only(h)
           : h->cfg.model_type == ADEC_MODEL_SYMAD_ENCODER ? build_symad_encoder_only(h)
           : h->fail("unknown model_type");
    if (rc) return rc;
    for (const auto& kv : h->tensors)   // load_state_dict(strict=True): unexpected keys are an error
        if (!h->consumed.count(kv.first)) return h->fail("unexpected key in state dict: " + kv.first);
    for (auto* ops : {&h->enc_ops, &h->dec_ops})
        for (Op& op : *ops) {
            if (finalize_op(h, &op)) return 1;
            if (alloc_state(h, &op, 1)) return 1;
        }
    h->n_streams = 1;
    h->enc_slots.bit.assign(1, 0);
    h->dec_slots.bit.assign(1, 0);
    build_state_map(h);
    h->tensors.clear();
    h->finalized = true;
    return 0;
}

int adec_n_streams(const adec_handle* h) { return h ? h->n_streams : 0; }

// Resize the per-stream causal state to n streams.  Streams that exist keep their state; new streams either copy stream 0
// (replicate: the "warm one stream, then fan out" case) or start from zero history (= reset_buffer() on them).  Buffers grow on
// demand and the replaced ones are freed.
static int resize_state(adec_handle* h, int n, bool replicate) {
    const int keep = std::min(n, h->n_streams);
    // every call in flight, on whatever stream (torch side streams do not synchronise with stream 0), has finished before the state
    // is touched; then every stream's latest state goes into st[cur]
    CK(h, cudaDeviceSynchronize());
    if (slot_fixup(h, h->enc_ops, 0) || slot_fixup(h, h->dec_ops, 0)) return 1;
    CK(h, cudaDeviceSynchronize());
    for (auto* ops : {&h->enc_ops, &h->dec_ops})
        for (Op& op : *ops) {
            // per-stream state in 4-byte words (bf16 state: st_C is a multiple of 32, so a stream's rows are whole words)
            const size_t per = (size_t)op.P * op.st_C * h->act_bytes() / 4;
            if (!per) continue;
            if (n > h->st_cap) {
                float* nb[2] = {nullptr, nullptr};
                for (int i = 0; i < 2; ++i) CK(h, cudaMalloc((void**)&nb[i], per * n * sizeof(float)));
                CK(h, cudaMemcpy(nb[0], op.st[op.cur], per * keep * sizeof(float), cudaMemcpyDeviceToDevice));
                for (int i = 0; i < 2; ++i) cudaFree(op.st[i]);
                op.st[0] = nb[0]; op.st[1] = nb[1]; op.cur = 0;
            }
            if (n > keep) {
                float* tail = op.st[op.cur] + per * keep;
                const long long tot = (long long)per * (n - keep);
                if (replicate) {
                    replicate_kernel<<<(unsigned)((tot + 255) / 256), 256>>>(tail, op.st[op.cur], (long long)per, n - keep);
                    CK(h, cudaGetLastError());
                } else {
                    CK(h, cudaMemset(tail, 0, tot * sizeof(float)));
                }
            }
        }
    CK(h, cudaDeviceSynchronize());
    if (n > h->st_cap) ++h->gen;
    h->st_cap = std::max(h->st_cap, n);
    h->n_streams = n;
    h->enc_slots.bit.assign(n, 0);
    h->dec_slots.bit.assign(n, 0);
    return 0;
}

int adec_set_streams(adec_handle* h, int n) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    if (n == h->n_streams) return 0;
    if (n < 1) return h->fail("n_streams must be >= 1");
    DeviceGuard dg(h->device);
    return resize_state(h, n, /*replicate=*/h->n_streams == 1);
}

int adec_reset(adec_handle* h, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    DeviceGuard dg(h->device);
    for (auto* ops : {&h->enc_ops, &h->dec_ops})
        for (Op& op : *ops) {
            const size_t per = (size_t)op.P * op.st_C;
            if (!per) continue;
            for (int i = 0; i < 2; ++i) CK(h, cudaMemsetAsync(op.st[i], 0, per * h->n_streams * h->act_bytes(), (cudaStream_t)stream));
        }
    for (SlotBits* sb : {&h->enc_slots, &h->dec_slots}) {     // both buffers are zero: every stream's state is in st[cur] again
        std::fill(sb->bit.begin(), sb->bit.end(), 0);
        sb->dirty = false;
    }
    return 0;
}

int adec_frames_for(const adec_handle* h, int T) {
    if (!h || (h->cfg.model_type != ADEC_MODEL_SYMAD && h->cfg.model_type != ADEC_MODEL_SYMAD_DECODER &&
               h->cfg.model_type != ADEC_MODEL_SYMAD_ENCODER))
        return -1;
    int t = T;
    for (int i = 0; i < h->cfg.n_enc; ++i) t = (t - 1) / h->cfg.enc_strides[i] + 1;
    return t;
}

int adec_hop_length(const adec_handle* h) { return h ? hop_of(h) : -1; }

// the host arguments of a varlen call: B >= 1 utterances of >= 1 samples / frames each
static int varlen_args(adec_handle* h, const char* name, const int* lengths, int B) {
    if (B < 1) return h->fail(fmt("%s: B must be >= 1, got %d", name, B));
    if (!lengths) return h->fail(fmt("%s: lengths is NULL", name));
    for (int b = 0; b < B; ++b)
        if (lengths[b] < 1) return h->fail(fmt("%s: utterance %d has length %d; every length must be >= 1", name, b, lengths[b]));
    return 0;
}

// the stream slots of a slot call: B distinct streams of the handle
static int stream_args(adec_handle* h, const char* name, const int* streams, int B) {
    if (!streams) return h->fail(fmt("%s: streams is NULL", name));
    std::vector<char> seen(h->n_streams, 0);
    for (int b = 0; b < B; ++b) {
        const int s = streams[b];
        if (s < 0 || s >= h->n_streams)
            return h->fail(fmt("%s: stream %d (entry %d) is out of range [0, %d) (call adec_set_streams)", name, s, b, h->n_streams));
        if (seen[s]) return h->fail(fmt("%s: stream %d is listed twice; each stream advances by one chunk per call", name, s));
        seen[s] = 1;
    }
    return 0;
}

// One codec entry point: the direction, the mode and the I/O dtype name it (adec_<encode|decode><mode>[_bf16]).  Only decode has bf16
// I/O, which must match the handle's activations (compute_dtype 2).  lengths / slots: HOST arrays of B entries for the varlen modes.
struct Call {
    bool decode;
    CallMode mode;
    bool bf16_io;
    const int* lengths = nullptr;
    const int* slots = nullptr;
};

static int run_call(adec_handle* h, const Call& c, const void* in, int B, int T, void* out, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    static const char* const kModeName[] = {"", "_offline", "_offline_varlen", "_streams"};
    const std::string base = std::string(c.decode ? "decode" : "encode") + kModeName[c.mode];
    const std::string name = base + (c.bf16_io ? "_bf16" : "");
    if (!c.decode && need_symad_tx(h, name)) return 1;
    if (c.decode && h->cfg.model_type == ADEC_MODEL_SYMAD_ENCODER) return fail_encoder_only(h, name);
    const char* io = c.decode ? "zq / y" : "x / z";
    if (h->act_bf16 && !c.bf16_io)
        return h->fail(fmt("%s: this handle has bf16 activations (compute_dtype 2); call adec_%s_bf16 with bf16 %s", name.c_str(),
                           base.c_str(), io));
    if (!h->act_bf16 && c.bf16_io)
        return h->fail(fmt("%s: this handle has fp32 activations (compute_dtype %d); call adec_%s with fp32 %s", name.c_str(),
                           h->cfg.compute_dtype, base.c_str(), io));
    if (c.bf16_io && (((uintptr_t)in | (uintptr_t)out) & 15))
        return h->fail(name + (c.decode ? ": zq and y must be 16-byte aligned" : ": x and z must be 16-byte aligned"));
    RunCtx rc{B, (const float*)in, (float*)out, (cudaStream_t)stream, c.mode, c.lengths, c.slots, name.c_str()};
    if (rc.varlen()) {
        if (varlen_args(h, rc.what, c.lengths, B)) return 1;
        if (c.mode == CALL_SLOTS && stream_args(h, rc.what, c.slots, B)) return 1;
        T = 1;
    } else if (B < 1 || T < 1) {
        return h->fail(name + ": empty input");
    }
    DeviceGuard dg(h->device);
    std::vector<Op>& ops = c.decode ? h->dec_ops : h->enc_ops;
    switch (c.mode) {     // the causal state the launches read
    case CALL_STREAM:     // every stream's state back in st[cur]
        if (slot_fixup(h, ops, rc.stream)) return 1;
        break;
    case CALL_OFFLINE:    // Generator.forward (codecTest.py:78-95): every causal conv starts from a zero left-pad (conv_layer.py:148-151)
        if (B != h->n_streams && resize_state(h, B, false)) return 1;
        if (adec_reset(h, stream)) return 1;
        break;
    case CALL_VARLEN:     // the state is neither read nor written; it is discarded, as the uniform offline calls discard it
        if (adec_reset(h, stream)) return 1;
        break;
    case CALL_SLOTS:      // each stream's history is where its slot bit says
        break;
    }
    if (run_ops(h, ops, rc, T, nullptr)) return 1;
    switch (c.mode) {     // where the new state went
    case CALL_STREAM:
    case CALL_OFFLINE:
        for (Op& op : ops)
            if (op.P > 0) op.cur ^= 1;
        break;
    case CALL_SLOTS: {
        SlotBits* sb = slot_bits(h, ops);
        for (int b = 0; b < B; ++b) sb->bit[c.slots[b]] ^= 1;
        sb->dirty = true;
        break;
    }
    case CALL_VARLEN:
        break;
    }
    return 0;
}

int adec_encode(adec_handle* h, const float* x, int B, int T, float* z, void* stream) {
    return run_call(h, {false, CALL_STREAM, false}, x, B, T, z, stream);
}

int adec_encode_offline(adec_handle* h, const float* x, int B, int T, float* z, void* stream) {
    return run_call(h, {false, CALL_OFFLINE, false}, x, B, T, z, stream);
}

int adec_encode_offline_varlen(adec_handle* h, const float* x, const int* lengths, int B, float* z, void* stream) {
    return run_call(h, {false, CALL_VARLEN, false, lengths}, x, B, 0, z, stream);
}

// Stream slots: advance B distinct streams of the handle by one chunk each, every chunk with its own length, in one launch sequence.
// The varlen row space with each utterance's history read from, and its new state written to, its stream's slot (ConvArgs::vl_slot).
int adec_encode_streams(adec_handle* h, const float* x, const int* lengths, const int* streams, int B, float* z, void* stream) {
    return run_call(h, {false, CALL_SLOTS, false, lengths, streams}, x, B, 0, z, stream);
}

int adec_encode_bf16(adec_handle* h, const uint16_t* x, int B, int T, uint16_t* z, void* stream) {
    return run_call(h, {false, CALL_STREAM, true}, x, B, T, z, stream);
}

int adec_encode_offline_bf16(adec_handle* h, const uint16_t* x, int B, int T, uint16_t* z, void* stream) {
    return run_call(h, {false, CALL_OFFLINE, true}, x, B, T, z, stream);
}

int adec_encode_offline_varlen_bf16(adec_handle* h, const uint16_t* x, const int* lengths, int B, uint16_t* z, void* stream) {
    return run_call(h, {false, CALL_VARLEN, true, lengths}, x, B, 0, z, stream);
}

int adec_encode_streams_bf16(adec_handle* h, const uint16_t* x, const int* lengths, const int* streams, int B, uint16_t* z, void* stream) {
    return run_call(h, {false, CALL_SLOTS, true, lengths, streams}, x, B, 0, z, stream);
}

int adec_decode(adec_handle* h, const float* zq, int B, int F, float* y, void* stream) {
    return run_call(h, {true, CALL_STREAM, false}, zq, B, F, y, stream);
}

int adec_decode_bf16(adec_handle* h, const uint16_t* zq, int B, int F, uint16_t* y, void* stream) {
    return run_call(h, {true, CALL_STREAM, true}, zq, B, F, y, stream);
}

int adec_decode_offline(adec_handle* h, const float* zq, int B, int F, float* y, void* stream) {
    return run_call(h, {true, CALL_OFFLINE, false}, zq, B, F, y, stream);
}

int adec_decode_offline_bf16(adec_handle* h, const uint16_t* zq, int B, int F, uint16_t* y, void* stream) {
    return run_call(h, {true, CALL_OFFLINE, true}, zq, B, F, y, stream);
}

int adec_decode_offline_varlen(adec_handle* h, const float* zq, const int* frames, int B, float* y, void* stream) {
    return run_call(h, {true, CALL_VARLEN, false, frames}, zq, B, 0, y, stream);
}

int adec_decode_offline_varlen_bf16(adec_handle* h, const uint16_t* zq, const int* frames, int B, uint16_t* y, void* stream) {
    return run_call(h, {true, CALL_VARLEN, true, frames}, zq, B, 0, y, stream);
}

int adec_decode_streams(adec_handle* h, const float* zq, const int* frames, const int* streams, int B, float* y, void* stream) {
    return run_call(h, {true, CALL_SLOTS, false, frames, streams}, zq, B, 0, y, stream);
}

int adec_decode_streams_bf16(adec_handle* h, const uint16_t* zq, const int* frames, const int* streams, int B, uint16_t* y, void* stream) {
    return run_call(h, {true, CALL_SLOTS, true, frames, streams}, zq, B, 0, y, stream);
}

int adec_copy_stream_state(adec_handle* h, int src, const int* dst, int n, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    if (src < 0 || src >= h->n_streams) return h->fail(fmt("copy_stream_state: src %d is out of range [0, %d)", src, h->n_streams));
    if (n < 0 || (n > 0 && !dst)) return h->fail("copy_stream_state: bad dst list");
    for (int i = 0; i < n; ++i)
        if (dst[i] < 0 || dst[i] >= h->n_streams)
            return h->fail(fmt("copy_stream_state: dst %d (entry %d) is out of range [0, %d)", dst[i], i, h->n_streams));
    DeviceGuard dg(h->device);
    for (auto* ops : {&h->enc_ops, &h->dec_ops}) {
        SlotBits* sb = slot_bits(h, *ops);
        const int sel = sb->bit[src];
        std::vector<int> pairs;
        for (int i = 0; i < n; ++i)
            if (dst[i] != src) { pairs.push_back(src); pairs.push_back(dst[i]); }
        // into the buffer src's state is in, which becomes the destination's current buffer
        if (slot_copy(h, *ops, pairs, sel, sel, (cudaStream_t)stream)) return 1;
        for (int i = 0; i < n; ++i) sb->bit[dst[i]] = (uint8_t)sel;
        if (sel) sb->dirty = true;
    }
    return 0;
}

// ---- stream state export / import: the state map (build_state_map) over the streams' current buffers
int adec_state_entries(const adec_handle* h) { return h && h->finalized ? (int)h->st_map.size() : -1; }

int adec_state_entry(const adec_handle* h, int i, const char** key, int* C, int* P) {
    if (!h || !h->finalized || i < 0 || i >= (int)h->st_map.size()) return 1;
    const auto& m = h->st_map[i];
    const StKey& k = (m.list ? h->dec_ops : h->enc_ops)[m.op].keys[m.k];
    if (key) *key = k.key.c_str();
    if (C) *C = k.C;
    if (P) *P = k.P;
    return 0;
}

int64_t adec_stream_state_elems(const adec_handle* h) { return h && h->finalized ? h->st_elems : -1; }

// One launch over every entry and every requested stream.  Each stream's state is read from / written to the buffer its slot bit names
// (st[cur ^ bit]); neither cur nor the slot bits change, so an export sees exactly what the next call of any kind would read.
static int stream_state_io(adec_handle* h, const char* name, const int* streams, int n, void* ext, bool import, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    if (n < 0) return h->fail(fmt("%s: n must be >= 0, got %d", name, n));
    if (n == 0) return 0;
    if (stream_args(h, name, streams, n)) return 1;
    if (!ext) return h->fail(fmt("%s: the state buffer is NULL", name));
    if ((uintptr_t)ext & 15) return h->fail(fmt("%s: the state buffer must be 16-byte aligned", name));
    if (h->st_map.empty()) return 0;
    std::vector<StateEntry> ents;
    for (const auto& m : h->st_map) {
        const Op& op = (m.list ? h->dec_ops : h->enc_ops)[m.op];
        const StKey& k = op.keys[m.k];
        StateEntry e{};
        e.st[0] = op.st[op.cur]; e.st[1] = op.st[op.cur ^ 1];
        e.per = (long long)op.P * op.st_C; e.off = m.off;
        e.C = k.C; e.P = k.P; e.zrows = k.zrows; e.st_C = op.st_C; e.cg = k.cg; e.col0 = k.col0; e.gstride = k.gstride;
        e.list = m.list;
        e.wc = !k.import ? 0 : k.gstride == 0 ? k.cg : k.C;
        ents.push_back(e);
    }
    std::vector<int> sv(3 * (size_t)n);
    for (int i = 0; i < n; ++i) {
        sv[3 * i] = streams[i];
        sv[3 * i + 1] = h->enc_slots.bit.empty() ? 0 : h->enc_slots.bit[streams[i]];
        sv[3 * i + 2] = h->dec_slots.bit.empty() ? 0 : h->dec_slots.bit[streams[i]];
    }
    // one upload: entries | tiles | streams (each part 16-byte aligned)
    const size_t eb = ents.size() * sizeof(StateEntry), tb = h->st_tiles.size() * sizeof(int4), sb = sv.size() * sizeof(int);
    std::vector<char> tab(eb + tb + sb);
    memcpy(tab.data(), ents.data(), eb);
    memcpy(tab.data() + eb, h->st_tiles.data(), tb);
    memcpy(tab.data() + eb + tb, sv.data(), sb);
    DeviceGuard dg(h->device);
    if (ensure(h, h->st_tab, (tab.size() + 3) / 4)) return 1;
    CK(h, cudaMemcpyAsync(h->st_tab.p, tab.data(), tab.size(), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    const char* d = reinterpret_cast<const char*>(h->st_tab.p);
    StateArgs a{};
    a.ent = reinterpret_cast<const StateEntry*>(d);
    a.tiles = reinterpret_cast<const int4*>(d + eb);
    a.streams = reinterpret_cast<const int*>(d + eb + tb);
    a.n = n; a.ext = ext; a.S = h->st_elems;
    a.err = import && h->engine == 2 && !h->bf16 ? h->d_err : nullptr;    // the fp16-split engine's range flag
    const dim3 grid((unsigned)h->st_tiles.size(), (unsigned)std::min(n, 65535));
    if (h->act_bf16) {
        if (import) stream_state_kernel<uint16_t, true><<<grid, 256, 0, (cudaStream_t)stream>>>(a);
        else stream_state_kernel<uint16_t, false><<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    } else {
        if (import) stream_state_kernel<float, true><<<grid, 256, 0, (cudaStream_t)stream>>>(a);
        else stream_state_kernel<float, false><<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    }
    CK(h, cudaGetLastError());
    ++h->launches;
    return 0;
}

int adec_get_stream_state(adec_handle* h, const int* streams, int n, void* out, void* stream) {
    return stream_state_io(h, "get_stream_state", streams, n, out, false, stream);
}

int adec_set_stream_state(adec_handle* h, const int* streams, int n, const void* in, void* stream) {
    return stream_state_io(h, "set_stream_state", streams, n, const_cast<void*>(in), true, stream);
}

static int index_bits(int n) { int b = 1; while ((1 << b) < n) ++b; return b; }

int adec_packed_frame_bytes(const adec_handle* h) {
    if (!h || (h->cfg.model_type != ADEC_MODEL_SYMAD && h->cfg.model_type != ADEC_MODEL_SYMAD_ENCODER)) return -1;
    return (h->cfg.codebook_num * index_bits(h->cfg.codebook_size) + 7) / 8;
}

// residual VQ launch: pick frames-per-pass FP and passes per block so that the grid is ONE wave with the smallest idle tail
extern "C++" template <int FP, bool FWD, bool ZB>
cudaError_t launch_rvq(const adec_handle* h, RvqArgs a, cudaStream_t s, int* cost) {
    static int per_sm[64] = {0};
    auto kern = rvq_kernel<64, 4, FP, FWD, ZB>;
    const int dev = h->device;
    const auto smem_of = [&](int n_pass) { const int FR = n_pass * FP; return (size_t)FR * (3 * 64 + 1 + 2 * (RVQ_THREADS / 32) + a.nq) * 4; };
    if (dev < 64 && !per_sm[dev]) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        int nb = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, RVQ_THREADS, smem_of(2));
        per_sm[dev] = std::max(1, nb);
    }
    const long long nfr = (long long)a.B * a.F, slots = (long long)h->n_sms * per_sm[dev < 64 ? dev : 0];
    int n_pass = (int)((nfr + slots * FP - 1) / (slots * FP));
    n_pass = std::max(1, std::min(n_pass, 96 / FP));                 // <= 96 frames of residuals (x1, x2) + zq in shared memory (79 KB)
    if (cost) { *cost = n_pass * (FP + 2) * (int)((nfr + slots * n_pass * FP - 1) / (slots * n_pass * FP)); return cudaSuccess; }
    a.n_pass = n_pass;
    const long long FR = (long long)n_pass * FP;
    kern<<<(unsigned)((nfr + FR - 1) / FR), RVQ_THREADS, smem_of(n_pass), s>>>(a);
    return cudaGetLastError();
}

extern "C++" template <bool FWD, bool ZB = false>
cudaError_t launch_rvq_best(const adec_handle* h, const RvqArgs& a, cudaStream_t s) {
    int c16 = 0, c12 = 0, c8 = 0;
    launch_rvq<16, FWD, ZB>(h, a, nullptr, &c16); launch_rvq<12, FWD, ZB>(h, a, nullptr, &c12); launch_rvq<8, FWD, ZB>(h, a, nullptr, &c8);
    return (c12 <= c16 && c12 <= c8) ? launch_rvq<12, FWD, ZB>(h, a, s, nullptr)
         : (c16 <= c8)               ? launch_rvq<16, FWD, ZB>(h, a, s, nullptr)
                                     : launch_rvq<8, FWD, ZB>(h, a, s, nullptr);
}

// fwd: zq receives ResidualVQ.forward's sum instead of lookup's (rvq_kernel's FWD).  zb: z is bf16 (rvq_kernel's ZB), which a handle
// with bf16 activations takes and every other handle refuses
static int quantize_common(adec_handle* h, const void* z, int B, int F, int64_t* idx, uint8_t* packed, float* zq, bool fwd, bool zb,
                           void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    if (need_symad_tx(h, "quantize")) return 1;
    if (h->act_bf16 && !zb)
        return h->fail("quantize: this handle has bf16 activations (compute_dtype 2); call adec_quantize_bf16 / adec_quantize_ex_bf16 with bf16 z");
    if (!h->act_bf16 && zb)
        return h->fail(fmt("quantize_bf16: this handle has fp32 activations (compute_dtype %d); call adec_quantize / adec_quantize_ex with "
                           "fp32 z", h->cfg.compute_dtype));
    if (zb && (uintptr_t)z % 16) return h->fail("quantize_bf16: z must be 16-byte aligned");
    // an encoder-only handle quantizes to indices and packed bytes; zq (the lookup) and the forward sum are the full handle's
    if (zq && h->cfg.model_type == ADEC_MODEL_SYMAD_ENCODER) return fail_encoder_only(h, fwd ? "quantize_forward" : "quantize_ex (zq)");
    if (B < 1 || F < 1) return h->fail("quantize: empty input");
    if (!idx && !packed && !zq) return h->fail("quantize: no output requested");
    DeviceGuard dg(h->device);
    RvqArgs a{};
    a.z = (const float*)z; a.B = B; a.F = F; a.nq = h->cfg.codebook_num; a.embed = h->d_embed; a.e2 = h->d_e2; a.idx = (long long*)idx;
    a.packed = packed; a.zq = zq; a.bits = index_bits(h->cfg.codebook_size); a.bpf = adec_packed_frame_bytes(h);
    const cudaError_t e = fwd ? launch_rvq_best<true>(h, a, (cudaStream_t)stream)
                        : zb  ? launch_rvq_best<false, true>(h, a, (cudaStream_t)stream)
                              : launch_rvq_best<false>(h, a, (cudaStream_t)stream);
    if (e != cudaSuccess) return h->fail(fmt("launch of rvq_kernel failed: %s", cudaGetErrorString(e)));
    ++h->launches;
    return 0;
}

int adec_quantize_ex(adec_handle* h, const float* z, int B, int F, int64_t* idx, uint8_t* packed, float* zq, void* stream) {
    return quantize_common(h, z, B, F, idx, packed, zq, false, false, stream);
}

int adec_quantize_ex_bf16(adec_handle* h, const uint16_t* z, int B, int F, int64_t* idx, uint8_t* packed, float* zq, void* stream) {
    return quantize_common(h, z, B, F, idx, packed, zq, false, true, stream);
}

int adec_quantize_bf16(adec_handle* h, const uint16_t* z, int B, int F, int64_t* idx, void* stream) {
    return quantize_common(h, z, B, F, idx, nullptr, nullptr, false, true, stream);
}

int adec_quantize_forward(adec_handle* h, const float* z, int B, int F, int64_t* idx, float* zq_fwd, void* stream) {
    if (h && !zq_fwd) return h->fail("quantize_forward: zq_fwd is NULL");
    return quantize_common(h, z, B, F, idx, nullptr, zq_fwd, true, false, stream);
}

int adec_zq_moments(adec_handle* h, const float* zq, const int* frames, int B, double* sum, double* m2, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    if (need_full_symad(h, "zq_moments")) return 1;
    if (varlen_args(h, "zq_moments", frames, B)) return 1;
    if (!zq || !sum || !m2) return h->fail("zq_moments: zq, sum and m2 must be given");
    if ((uintptr_t)zq % 16) return h->fail("zq_moments: zq must be 16-byte aligned");
    std::vector<int> off(B + 1, 0);
    long long rows = 0;
    for (int b = 0; b < B; ++b) {
        rows += frames[b];
        if (rows > INT32_MAX) return h->fail(fmt("zq_moments: the batch has more than 2^31 - 1 rows; split it"));
        off[b + 1] = (int)rows;
    }
    DeviceGuard dg(h->device);
    const cudaStream_t s = (cudaStream_t)stream;
    if (ensure(h, h->mom_tab, off.size())) return 1;
    CK(h, cudaMemcpyAsync(h->mom_tab.p, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    MomArgs a{zq, reinterpret_cast<const int*>(h->mom_tab.p), sum, m2};
    zq_moments_kernel<false><<<B, MOM_THREADS, 0, s>>>(a);
    CK(h, cudaGetLastError());
    zq_moments_kernel<true><<<B, MOM_THREADS, 0, s>>>(a);
    CK(h, cudaGetLastError());
    h->launches += 2;
    return 0;
}

int adec_quantize(adec_handle* h, const float* z, int B, int F, int64_t* idx, void* stream) {
    return adec_quantize_ex(h, z, B, F, idx, nullptr, nullptr, stream);
}

// bf16: zq is bf16 (lookup_kernel<true>), 16-byte aligned
static int lookup_common(adec_handle* h, const int64_t* idx, const uint8_t* packed, int B, int F, void* zq, bool bf16, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    const char* what = bf16 ? "lookup_bf16" : "lookup";
    if (need_full_symad(h, what)) return 1;
    if (B < 1 || F < 1) return h->fail(std::string(what) + ": empty input");
    if (bf16 && (h->cfg.code_dim % 8 || (uintptr_t)zq % 16))
        return h->fail("lookup_bf16: needs code_dim % 8 == 0 and a 16-byte aligned zq");
    DeviceGuard dg(h->device);
    LookupArgs a{};
    a.idx = (const long long*)idx; a.packed = packed; a.nfr = (long long)B * F; a.nq = h->cfg.codebook_num; a.D = h->cfg.code_dim;
    a.N = h->cfg.codebook_size; a.bits = index_bits(a.N); a.bpf = adec_packed_frame_bytes(h);
    a.codebook = h->d_codebook; a.n_rows = (long long)h->cfg.codebook_num * h->cfg.codebook_size; a.zq = (float*)zq; a.err = h->d_err;
    const long long nth = a.nfr * (a.D / 4);
    if (bf16) lookup_kernel<true><<<(unsigned)((nth + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    else lookup_kernel<false><<<(unsigned)((nth + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a);
    CK(h, cudaGetLastError());
    ++h->launches;
    return 0;
}

int adec_lookup(adec_handle* h, const int64_t* idx, int B, int F, float* zq, void* stream) {
    return lookup_common(h, idx, nullptr, B, F, zq, false, stream);
}

int adec_lookup_bf16(adec_handle* h, const int64_t* idx, int B, int F, uint16_t* zq, void* stream) {
    return lookup_common(h, idx, nullptr, B, F, zq, true, stream);
}

int adec_lookup_packed(adec_handle* h, const uint8_t* packed, int B, int F, float* zq, void* stream) {
    return lookup_common(h, nullptr, packed, B, F, zq, false, stream);
}

int adec_lookup_packed_bf16(adec_handle* h, const uint8_t* packed, int B, int F, uint16_t* zq, void* stream) {
    return lookup_common(h, nullptr, packed, B, F, zq, true, stream);
}

static_assert(sizeof(adec_conceal_row) == sizeof(ConcealRow), "adec_conceal_row and ConcealRow must share a layout");

// Every descriptor is checked here, before anything is enqueued, so that a bad one fails with the field's name instead of a fault
static int conceal_common(adec_handle* h, const uint8_t* packed, int F, const adec_conceal_row* rows, int R, float* anchors,
                          int n_anchors, void* zq, bool bf16, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    const std::string what = bf16 ? "lookup_packed_conceal_bf16" : "lookup_packed_conceal";
    if (need_full_symad(h, what)) return 1;
    if (F < 1 || R < 1) return h->fail(what + ": empty input (F and R must be >= 1)");
    if (n_anchors < 0) return h->fail(what + ": n_anchors < 0");
    if (!packed || !rows || !zq) return h->fail(what + ": packed, rows and zq must be given");
    if (n_anchors > 0 && (!anchors || (uintptr_t)anchors % 16)) return h->fail(what + ": anchors must be a 16-byte aligned device buffer");
    if (bf16 && (h->cfg.code_dim % 8 || (uintptr_t)zq % 16))
        return h->fail(what + ": needs code_dim % 8 == 0 and a 16-byte aligned zq");
    std::vector<int> reader(n_anchors, -1), writer(n_anchors, -1);     // per anchor slot: a row that reads it, a row that writes it
    for (int r = 0; r < R; ++r) {
        const adec_conceal_row& d = rows[r];
        const bool real = d.src >= 0;
        if (real && d.src >= F) return h->fail(fmt("%s: rows[%d].src = %d is out of range [0, %d)", what.c_str(), r, d.src, F));
        if (real && d.next != -1) return h->fail(fmt("%s: rows[%d].next = %d: a real row (src >= 0) has next = -1", what.c_str(), r, d.next));
        if (!real && d.src != -1) return h->fail(fmt("%s: rows[%d].src = %d is out of range: a frame in [0, %d) or -1", what.c_str(), r, d.src, F));
        if (!real && (d.next < 0 || d.next >= F))
            return h->fail(fmt("%s: rows[%d].next = %d is out of range [0, %d)", what.c_str(), r, d.next, F));
        if (!real && d.den < 2) return h->fail(fmt("%s: rows[%d].den = %d: a concealed row needs den >= 2", what.c_str(), r, d.den));
        if (!real && (d.j < 1 || d.j >= d.den))
            return h->fail(fmt("%s: rows[%d].j = %d is outside [1, den = %d)", what.c_str(), r, d.j, d.den));
        if (d.slot < -1 || d.slot >= n_anchors)
            return h->fail(fmt("%s: rows[%d].slot = %d is out of range: an anchor in [0, %d) or -1", what.c_str(), r, d.slot, n_anchors));
        if (d.slot < 0) continue;
        std::vector<int>& mine = real ? writer : reader;
        const std::vector<int>& other = real ? reader : writer;
        if (other[d.slot] >= 0)
            return h->fail(fmt("%s: rows[%d].slot = %d: anchor %d is read by row %d and written by row %d of the same call", what.c_str(), r,
                               d.slot, d.slot, real ? other[d.slot] : r, real ? r : other[d.slot]));
        if (real && mine[d.slot] >= 0)
            return h->fail(fmt("%s: rows[%d].slot = %d: anchor %d is written by rows %d and %d of the same call", what.c_str(), r, d.slot,
                               d.slot, mine[d.slot], r));
        mine[d.slot] = r;
    }
    DeviceGuard dg(h->device);
    const cudaStream_t s = (cudaStream_t)stream;
    if (ensure(h, h->conceal_tab, (size_t)R * sizeof(adec_conceal_row) / sizeof(float))) return 1;
    CK(h, cudaMemcpyAsync(h->conceal_tab.p, rows, (size_t)R * sizeof(adec_conceal_row), cudaMemcpyHostToDevice, s));
    ConcealArgs c{};
    LookupArgs& a = c.l;
    a.packed = packed; a.nfr = R; a.nq = h->cfg.codebook_num; a.D = h->cfg.code_dim;
    a.N = h->cfg.codebook_size; a.bits = index_bits(a.N); a.bpf = adec_packed_frame_bytes(h);
    a.codebook = h->d_codebook; a.n_rows = (long long)h->cfg.codebook_num * h->cfg.codebook_size; a.zq = (float*)zq; a.err = h->d_err;
    c.rows = reinterpret_cast<const ConcealRow*>(h->conceal_tab.p);
    c.anchors = anchors;
    const long long nth = a.nfr * (a.D / 4);
    if (bf16) lookup_conceal_kernel<true><<<(unsigned)((nth + 255) / 256), 256, 0, s>>>(c);
    else lookup_conceal_kernel<false><<<(unsigned)((nth + 255) / 256), 256, 0, s>>>(c);
    CK(h, cudaGetLastError());
    ++h->launches;
    return 0;
}

int adec_lookup_packed_conceal(adec_handle* h, const uint8_t* packed, int F, const adec_conceal_row* rows, int R, float* anchors,
                               int n_anchors, float* zq, void* stream) {
    return conceal_common(h, packed, F, rows, R, anchors, n_anchors, zq, false, stream);
}

int adec_lookup_packed_conceal_bf16(adec_handle* h, const uint8_t* packed, int F, const adec_conceal_row* rows, int R, float* anchors,
                                    int n_anchors, uint16_t* zq, void* stream) {
    return conceal_common(h, packed, F, rows, R, anchors, n_anchors, zq, true, stream);
}

static_assert(sizeof(adec_playout_row) == sizeof(PlayoutRow), "adec_playout_row and PlayoutRow must share a layout");

// conceal_common with the fade row kind; with timescale also between rows and frame-started fades (a real row's src with a next or
// a target).  Every descriptor is checked before anything is enqueued.
static int playout_common(adec_handle* h, const uint8_t* packed, int F, const adec_playout_row* rows, int R, float* anchors,
                          int n_anchors, const float* targets, int n_targets, void* zq, bool bf16, bool timescale, void* stream) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    const std::string what = std::string(timescale ? "lookup_packed_timescale" : "lookup_packed_playout") + (bf16 ? "_bf16" : "");
    if (need_full_symad(h, what)) return 1;
    if (F < 0 || R < 1) return h->fail(what + ": empty input (F must be >= 0 and R >= 1)");
    if (n_anchors < 0 || n_targets < 0) return h->fail(what + ": n_anchors and n_targets must be >= 0");
    if ((F > 0 && !packed) || !rows || !zq) return h->fail(what + ": packed (when F > 0), rows and zq must be given");
    if (n_anchors > 0 && (!anchors || (uintptr_t)anchors % 16)) return h->fail(what + ": anchors must be a 16-byte aligned device buffer");
    if (n_targets > 0 && (!targets || (uintptr_t)targets % 16)) return h->fail(what + ": targets must be a 16-byte aligned device buffer");
    if (bf16 && (h->cfg.code_dim % 8 || (uintptr_t)zq % 16))
        return h->fail(what + ": needs code_dim % 8 == 0 and a 16-byte aligned zq");
    std::vector<int> reader(n_anchors, -1), writer(n_anchors, -1);     // per anchor slot: a row that reads it, a row that writes it
    for (int r = 0; r < R; ++r) {
        const adec_playout_row& d = rows[r];
        const bool real = d.src >= 0, fade = d.src == -1 && d.next == -1;
        const bool between = timescale && real && d.next != -1, sfade = timescale && real && d.next == -1 && d.target != -1;
        const bool from_frame = between || sfade;   // starts from frame src: reads no anchor and stores none
        if (real && d.src >= F) return h->fail(fmt("%s: rows[%d].src = %d is out of range [0, %d)", what.c_str(), r, d.src, F));
        if (real && !timescale && d.next != -1)
            return h->fail(fmt("%s: rows[%d].next = %d: a real row (src >= 0) has next = -1", what.c_str(), r, d.next));
        if (between && (d.next < 0 || d.next >= F))
            return h->fail(fmt("%s: rows[%d].next = %d is out of range: a frame in [0, %d) or -1", what.c_str(), r, d.next, F));
        if (!real && d.src != -1) return h->fail(fmt("%s: rows[%d].src = %d is out of range: a frame in [0, %d) or -1", what.c_str(), r, d.src, F));
        if (!real && !fade && (d.next < 0 || d.next >= F))
            return h->fail(fmt("%s: rows[%d].next = %d is out of range: a frame in [0, %d) or -1", what.c_str(), r, d.next, F));
        if (!fade && !sfade && d.target != -1)
            return h->fail(fmt(timescale ? "%s: rows[%d].target = %d: only a fade row (next = -1, no src or a src to fade from) has a target"
                                         : "%s: rows[%d].target = %d: only a fade row (src = next = -1) has a target", what.c_str(), r, d.target));
        if ((fade || sfade) && (d.target < 0 || d.target >= n_targets))
            return h->fail(fmt("%s: rows[%d].target = %d is out of range [0, %d)", what.c_str(), r, d.target, n_targets));
        if (!real && !fade && d.den < 2)
            return h->fail(fmt("%s: rows[%d].den = %d: an interpolated row needs den >= 2", what.c_str(), r, d.den));
        if (between && d.den < 2) return h->fail(fmt("%s: rows[%d].den = %d: a between row needs den >= 2", what.c_str(), r, d.den));
        if (((!real && !fade) || between) && (d.j < 1 || d.j >= d.den))
            return h->fail(fmt("%s: rows[%d].j = %d is outside [1, den = %d)", what.c_str(), r, d.j, d.den));
        if ((fade || sfade) && d.den < 1) return h->fail(fmt("%s: rows[%d].den = %d: a fade row needs den >= 1", what.c_str(), r, d.den));
        if ((fade || sfade) && d.j < 1) return h->fail(fmt("%s: rows[%d].j = %d: a fade row needs j >= 1", what.c_str(), r, d.j));
        if (from_frame && d.slot != -1)
            return h->fail(fmt("%s: rows[%d].slot = %d: a %s starts from frame src and has slot = -1", what.c_str(), r, d.slot,
                               between ? "between row" : "frame-started fade"));
        if (d.slot < -1 || d.slot >= n_anchors)
            return h->fail(fmt("%s: rows[%d].slot = %d is out of range: an anchor in [0, %d) or -1", what.c_str(), r, d.slot, n_anchors));
        if (d.slot < 0) continue;
        std::vector<int>& mine = real ? writer : reader;
        const std::vector<int>& other = real ? reader : writer;
        if (other[d.slot] >= 0)
            return h->fail(fmt("%s: rows[%d].slot = %d: anchor %d is read by row %d and written by row %d of the same call", what.c_str(), r,
                               d.slot, d.slot, real ? other[d.slot] : r, real ? r : other[d.slot]));
        if (real && mine[d.slot] >= 0)
            return h->fail(fmt("%s: rows[%d].slot = %d: anchor %d is written by rows %d and %d of the same call", what.c_str(), r, d.slot,
                               d.slot, mine[d.slot], r));
        mine[d.slot] = r;
    }
    DeviceGuard dg(h->device);
    const cudaStream_t s = (cudaStream_t)stream;
    if (ensure(h, h->playout_tab, (size_t)R * sizeof(adec_playout_row) / sizeof(float))) return 1;
    // from a page-locked `rows` this copy is asynchronous: the header asks the caller to keep the buffer until the stream gets here
    CK(h, cudaMemcpyAsync(h->playout_tab.p, rows, (size_t)R * sizeof(adec_playout_row), cudaMemcpyHostToDevice, s));
    PlayoutArgs c{};
    LookupArgs& a = c.l;
    a.packed = packed; a.nfr = R; a.nq = h->cfg.codebook_num; a.D = h->cfg.code_dim;
    a.N = h->cfg.codebook_size; a.bits = index_bits(a.N); a.bpf = adec_packed_frame_bytes(h);
    a.codebook = h->d_codebook; a.n_rows = (long long)h->cfg.codebook_num * h->cfg.codebook_size; a.zq = (float*)zq; a.err = h->d_err;
    c.rows = reinterpret_cast<const PlayoutRow*>(h->playout_tab.p);
    c.anchors = anchors;
    c.targets = targets;
    const long long nth = a.nfr * (a.D / 4);
    const unsigned blocks = (unsigned)((nth + 255) / 256);
    if (timescale) {
        if (bf16) lookup_conceal_kernel<true, true, true><<<blocks, 256, 0, s>>>(c);
        else lookup_conceal_kernel<false, true, true><<<blocks, 256, 0, s>>>(c);
    } else {
        if (bf16) lookup_conceal_kernel<true, true><<<blocks, 256, 0, s>>>(c);
        else lookup_conceal_kernel<false, true><<<blocks, 256, 0, s>>>(c);
    }
    CK(h, cudaGetLastError());
    ++h->launches;
    return 0;
}

int adec_lookup_packed_playout(adec_handle* h, const uint8_t* packed, int F, const adec_playout_row* rows, int R, float* anchors,
                               int n_anchors, const float* targets, int n_targets, float* zq, void* stream) {
    return playout_common(h, packed, F, rows, R, anchors, n_anchors, targets, n_targets, zq, false, false, stream);
}

int adec_lookup_packed_playout_bf16(adec_handle* h, const uint8_t* packed, int F, const adec_playout_row* rows, int R, float* anchors,
                                    int n_anchors, const float* targets, int n_targets, uint16_t* zq, void* stream) {
    return playout_common(h, packed, F, rows, R, anchors, n_anchors, targets, n_targets, zq, true, false, stream);
}

int adec_lookup_packed_timescale(adec_handle* h, const uint8_t* packed, int F, const adec_playout_row* rows, int R, float* anchors,
                                 int n_anchors, const float* targets, int n_targets, float* zq, void* stream) {
    return playout_common(h, packed, F, rows, R, anchors, n_anchors, targets, n_targets, zq, false, true, stream);
}

int adec_lookup_packed_timescale_bf16(adec_handle* h, const uint8_t* packed, int F, const adec_playout_row* rows, int R, float* anchors,
                                      int n_anchors, const float* targets, int n_targets, uint16_t* zq, void* stream) {
    return playout_common(h, packed, F, rows, R, anchors, n_anchors, targets, n_targets, zq, true, true, stream);
}

int adec_codec_host(adec_handle* enc, adec_handle* dec, const float* x_host, int B, int T, int64_t* idx_host,
                    float* y_host, void* stream) {
    if (!enc || !dec) return 1;
    if (enc->device != dec->device) return enc->fail("codec_host: handles on different devices");
    if (dec->act_bf16) return enc->fail("codec_host: the decoder has bf16 activations (compute_dtype 2), which the host path does not carry; "
                                        "use compute_dtype 0 or 1, or adec_decode_bf16 on device buffers");
    if (need_full_symad(enc, "codec_host (enc)")) return 1;
    DeviceGuard dg(enc->device);
    cudaStream_t s = (cudaStream_t)stream;
    const int F = adec_frames_for(enc, T);
    if (F < 1) return enc->fail("codec_host: bad T or not a symAD encoder");
    const int D = enc->cfg.code_dim, nq = enc->cfg.codebook_num, hop = hop_of(dec);
    if (ensure(enc, enc->hx, (size_t)B * T) || ensure(enc, enc->hz, (size_t)B * D * F) || ensure(enc, enc->hzq, (size_t)B * F * D) ||
        ensure(enc, enc->hy, (size_t)B * F * hop))
        return 1;
    const size_t nidx = (size_t)nq * B * F;
    if (enc->hidx_cap < nidx) {
        if (enc->hidx) CK(enc, cudaFree(enc->hidx));
        CK(enc, cudaMalloc((void**)&enc->hidx, nidx * sizeof(long long)));
        enc->hidx_cap = nidx;
    }
    CK(enc, cudaMemcpyAsync(enc->hx.p, x_host, (size_t)B * T * sizeof(float), cudaMemcpyHostToDevice, s));
    if (adec_encode(enc, enc->hx.p, B, T, enc->hz.p, stream)) return 1;
    // quantize + lookup in ONE launch: the RVQ kernel also emits zq (bin/stream.py:224 hand-off without the int64 round trip)
    if (adec_quantize_ex(enc, enc->hz.p, B, F, (int64_t*)enc->hidx, nullptr, enc->hzq.p, stream)) return 1;
    if (adec_decode(dec, enc->hzq.p, B, F, enc->hy.p, stream)) { enc->err = dec->err; return 1; }
    if (idx_host) CK(enc, cudaMemcpyAsync(idx_host, enc->hidx, nidx * sizeof(long long), cudaMemcpyDeviceToHost, s));
    CK(enc, cudaMemcpyAsync(y_host, enc->hy.p, (size_t)B * F * hop * sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(enc, cudaStreamSynchronize(s));
    for (adec_handle* hh : {enc, dec}) {
        int herr = 0;
        CK(enc, cudaMemcpy(&herr, hh->d_err, sizeof(int), cudaMemcpyDeviceToHost));
        if (herr) CK(enc, cudaMemset(hh->d_err, 0, sizeof(int)));
        if (herr & 1) return enc->fail("lookup: index out of range");
        if (herr & 2) return enc->fail("an activation left the range of the fp16-split tensor-core engine (|a| >= 6e4); use ADEC_CONV_PATH=tf32");
        if (hh == dec) break;     // enc == dec
    }
    return 0;
}

static int pack_common(adec_handle* h, const char* what, int64_t* idx, int B, int F, uint8_t* packed, void* stream, bool pack) {
    if (!h || !h->finalized) return h ? h->fail("not finalized") : 1;
    if (pack ? need_symad_tx(h, what) : need_full_symad(h, what)) return 1;
    if (B < 1 || F < 1) return h->fail(std::string(what) + ": empty input");
    if (h->cfg.codebook_size < 2 || h->cfg.codebook_size > 65536) return h->fail(std::string(what) + ": codebook_size must be in [2, 65536]");
    DeviceGuard dg(h->device);
    PackArgs a{};
    a.idx = (long long*)idx; a.packed = packed; a.nfr = (long long)B * F; a.nq = h->cfg.codebook_num; a.N = h->cfg.codebook_size;
    a.bits = index_bits(a.N); a.bpf = adec_packed_frame_bytes(h); a.err = h->d_err;
    const unsigned grid = (unsigned)((a.nfr + 255) / 256);
    if (pack) pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    else unpack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(a);
    CK(h, cudaGetLastError());
    ++h->launches;
    return 0;
}

int adec_pack_indices(adec_handle* h, const int64_t* idx, int B, int F, uint8_t* packed, void* stream) {
    return pack_common(h, "pack_indices", const_cast<int64_t*>(idx), B, F, packed, stream, true);
}

int adec_unpack_indices(adec_handle* h, const uint8_t* packed, int B, int F, int64_t* idx, void* stream) {
    return pack_common(h, "unpack_indices", idx, B, F, const_cast<uint8_t*>(packed), stream, false);
}

// device flag word: bit 0 = out-of-range index (lookup / pack / unpack), bit 1 = activation outside the fp16-split range
static int read_flag(adec_handle* h, void* stream, int bit) {
    if (!h || !h->d_err) return -1;
    DeviceGuard dg(h->device);
    int herr = 0;
    if (cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess ||
        cudaMemcpy(&herr, h->d_err, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) {
        h->fail("CUDA error while reading the device flag word");
        return -1;
    }
    if (herr & bit) {
        const int rest = herr & ~bit;
        if (cudaMemcpy(h->d_err, &rest, sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) { h->fail("CUDA error while clearing the device flag word"); return -1; }
    }
    return (herr & bit) ? 1 : 0;
}

int adec_index_error(adec_handle* h, void* stream) { return read_flag(h, stream, 1); }
int adec_range_error(adec_handle* h, void* stream) { return read_flag(h, stream, 2); }

int64_t adec_launch_count(const adec_handle* h) { return h ? h->launches : 0; }

int adec_ktrace(adec_handle* h, unsigned long long* out, int max_records) {
    if (!h || !h->d_ktrace || !out) return -1;
    DeviceGuard dg(h->device);
    const int n = std::min(h->ktrace_n, max_records);
    if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(out, h->d_ktrace, (size_t)n * KT_REC * sizeof(unsigned long long), cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemset(h->d_ktrace, 0, 4096 * KT_REC * sizeof(unsigned long long)) != cudaSuccess) return -1;
    h->ktrace_n = 0;
    return n;
}

int adec_probe_mma(int device, int kind, int NT, int n_groups, double* tflops, double* ms) {
    if (!tflops || (kind != 0 && kind != 1) || (NT != 32 && NT != 64 && NT != 128 && NT != 256) || n_groups < 1) { g_create_error = "probe_mma: bad argument"; return 1; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) { g_create_error = "probe_mma: no usable CUDA device"; return 1; }
    DeviceGuard dg(device);
    int n_sms = 0;
    cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, device);
    constexpr int a_pitch_rows = 136;          // a window pitch of the engine (128 rows + halo)
    const int smem = 8 * 2 * a_pitch_rows * 16 + 8 * 2 * NT * 16;
    auto launch = [&](cudaStream_t s) {
        auto go = [&](auto kern) {
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
            kern<<<n_sms, 256, smem, s>>>(n_groups, a_pitch_rows);
        };
        if (kind == 0) {
            if (NT == 32) go(mma_probe_kernel<32, PREC_TF32>); else if (NT == 64) go(mma_probe_kernel<64, PREC_TF32>);
            else if (NT == 128) go(mma_probe_kernel<128, PREC_TF32>); else go(mma_probe_kernel<256, PREC_TF32>);
        } else {
            if (NT == 32) go(mma_probe_kernel<32, PREC_F16>); else if (NT == 64) go(mma_probe_kernel<64, PREC_F16>);
            else if (NT == 128) go(mma_probe_kernel<128, PREC_F16>); else go(mma_probe_kernel<256, PREC_F16>);
        }
    };
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch(0);                                   // warm-up: clocks, instruction cache
    cudaEventRecord(e0, 0);
    launch(0);
    cudaEventRecord(e1, 0);
    cudaError_t e = cudaEventSynchronize(e1);
    float t = 0.f;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&t, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    if (e != cudaSuccess || cudaGetLastError() != cudaSuccess) { g_create_error = fmt("probe_mma: %s", cudaGetErrorString(e)); return 1; }
    const double flops = (double)n_sms * n_groups * 12.0 * 2.0 * 128.0 * NT * (kind == 0 ? 8.0 : 16.0);
    *tflops = flops / (t * 1e-3) / 1e12;
    if (ms) *ms = t;
    return 0;
}

int adec_test_wgmma_columns(int device, const void* a, const void* b, float* d64, float* d32) {
    if (!a || !b || !d64 || !d32) { g_create_error = "test_wgmma_columns: NULL argument"; return 1; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) { g_create_error = "test_wgmma_columns: no usable CUDA device"; return 1; }
    DeviceGuard dg(device);
    const size_t na = 2 * 4 * 64 * 16, nb = 3 * 4 * 64 * 16, nd = 64 * 64 * sizeof(float);
    void* buf = nullptr;
    cudaError_t e = cudaMalloc(&buf, na + nb + 2 * nd);
    if (e == cudaSuccess) {
        char* p = static_cast<char*>(buf);
        e = cudaMemcpy(p, a, na, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(p + na, b, nb, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            wgmma_cols_kernel<<<1, 128>>>(reinterpret_cast<const uint4*>(p), reinterpret_cast<const uint4*>(p + na),
                                          reinterpret_cast<float*>(p + na + nb), reinterpret_cast<float*>(p + na + nb + nd));
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpy(d64, p + na + nb, nd, cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(d32, p + na + nb + nd, nd, cudaMemcpyDeviceToHost);
        cudaFree(buf);
    }
    if (e != cudaSuccess) { g_create_error = fmt("test_wgmma_columns: %s", cudaGetErrorString(e)); return 1; }
    return 0;
}

int adec_record_launches(adec_handle* h, int enable) {
    if (!h) return 1;
    h->launch_rec.clear();
    h->launch_log = enable ? &h->launch_rec : nullptr;
    return 0;
}

int adec_launch_records(const adec_handle* h, int* out, int max_records) {
    if (!h || (max_records > 0 && !out)) return -1;
    const int n = (int)h->launch_rec.size() / ADEC_TEST_REC;
    std::copy(h->launch_rec.begin(), h->launch_rec.begin() + (size_t)std::min(n, std::max(max_records, 0)) * ADEC_TEST_REC, out);
    return n;
}

int adec_profile(adec_handle* h, int enable) {
    if (!h) return 1;
    for (auto& ev : h->prof_events) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
    h->prof_events.clear(); h->prof_names.clear(); h->prof_bytes.clear();
    h->profiling = enable != 0;
    return 0;
}

int adec_profile_report(adec_handle* h, char* buf, int buf_len) {
    if (!h || !buf || buf_len < 2) return 1;
    DeviceGuard dg(h->device);
    std::string out;
    for (size_t i = 0; i < h->prof_events.size(); ++i) {
        if (cudaEventSynchronize(h->prof_events[i].second) != cudaSuccess) return h->fail("profile: event sync failed");
        float ms = 0.f;
        cudaEventElapsedTime(&ms, h->prof_events[i].first, h->prof_events[i].second);
        out += fmt("%s\t%.6f\t%.0f\n", h->prof_names[i].c_str(), ms, h->prof_bytes[i]);
    }
    if ((int)out.size() + 1 > buf_len) return h->fail("profile: buffer too small");
    memcpy(buf, out.c_str(), out.size() + 1);
    return 0;
}

// -------------------------------------------------------------------------------------------------
// single-layer entry points for the unit tests (HOST pointers, reference layouts)
// ---- graphed stream steps: the eager call sequence of a transmitter or receiver step, captured once per state parity
struct adec_graph {
    int kind = ADEC_GRAPH_TX;
    adec_handle* a = nullptr;     // the tx handle (ADEC_GRAPH_TX) or the rx handle (ADEC_GRAPH_RX); errors are reported on it
    adec_handle* b = nullptr;     // the decoder (ADEC_GRAPH_RX), may equal a
    int device = 0;
    int B = 0, T = 0, F = 0;      // streams, input samples (TX), frames
    bool wire = false;
    const void* in = nullptr;
    void* out = nullptr;
    void* mid = nullptr;          // TX: z (B, code_dim, F); RX: zq (B, F, code_dim); bf16 when the stateful handle has bf16 activations
    cudaStream_t cs = nullptr;    // private capture stream
    // by the parity (op.cur) of the stateful op list: both captured together, each instantiated the first time it is launched
    cudaGraph_t graph[2] = {nullptr, nullptr};
    cudaGraphExec_t exec[2] = {nullptr, nullptr};
    uint64_t gen_a = 0, gen_b = 0;                    // the handles' generations the graphs were captured at
    int64_t da = 0, db = 0;       // launches one step counts on a and on b (b != a), as the eager calls count them
    int kernels = 0, edges = 0, instantiations = 0;
};

static adec_handle* graph_state_handle(const adec_graph* g) { return g->kind == ADEC_GRAPH_TX ? g->a : g->b; }
static std::vector<Op>& graph_state_ops(adec_graph* g) { return g->kind == ADEC_GRAPH_TX ? g->a->enc_ops : g->b->dec_ops; }

// which state buffer the stateful ops of a list read next (op.cur); -1 if they disagree
static int list_parity(const std::vector<Op>& ops) {
    int p = -1;
    for (const Op& op : ops)
        if (op.P > 0) {
            if (p < 0) p = op.cur;
            else if (p != op.cur) return -1;
        }
    return p < 0 ? 0 : p;
}

// The eager sequence a step stands for: encode + quantize (TX), lookup + decode (RX), on stream s
static int graph_body(adec_graph* g, cudaStream_t s) {
    adec_handle *a = g->a, *b = g->b;
    if (g->kind == ADEC_GRAPH_TX) {
        if (run_call(a, {false, CALL_STREAM, a->act_bf16}, g->in, g->B, g->T, g->mid, s)) return 1;
        return quantize_common(a, g->mid, g->B, g->F, g->wire ? nullptr : (int64_t*)g->out, g->wire ? (uint8_t*)g->out : nullptr, nullptr,
                               false, a->act_bf16, s);
    }
    if (lookup_common(a, g->wire ? nullptr : (const int64_t*)g->in, g->wire ? (const uint8_t*)g->in : nullptr, g->B, g->F, g->mid,
                      b->act_bf16, s))
        return 1;
    if (run_call(b, {true, CALL_STREAM, b->act_bf16}, g->mid, g->B, g->F, g->out, s)) { a->err = b->err; return 1; }
    return 0;
}

// A handle's host state as a capture finds it: the capture runs the eager code, which advances it, and puts it back afterwards.
// The diagnostics (profiling events, launch records, the kernel trace) are switched off for the capture, so that none of their
// records or trace slots is baked into the graph or left behind for launches that never ran.
struct HostSnap {
    adec_handle* h;
    int64_t launches;
    SlotBits enc, dec;
    std::vector<int> cur;
    bool profiling;
    std::vector<int>* launch_log;
    unsigned long long* d_ktrace;
    int ktrace_n;
    explicit HostSnap(adec_handle* h_)
        : h(h_), launches(h_->launches), enc(h_->enc_slots), dec(h_->dec_slots), profiling(h_->profiling), launch_log(h_->launch_log),
          d_ktrace(h_->d_ktrace), ktrace_n(h_->ktrace_n) {
        for (auto* ops : {&h->enc_ops, &h->dec_ops})
            for (const Op& op : *ops) cur.push_back(op.cur);
        h->profiling = false;
        h->launch_log = nullptr;
        h->d_ktrace = nullptr;
    }
    void restore() const {
        h->launches = launches;
        h->enc_slots = enc;
        h->dec_slots = dec;
        h->profiling = profiling;
        h->launch_log = launch_log;
        h->d_ktrace = d_ktrace;
        h->ktrace_n = ktrace_n;
        size_t i = 0;
        for (auto* ops : {&h->enc_ops, &h->dec_ops})
            for (Op& op : *ops) op.cur = cur[i++];
    }
};

static void graph_drop(adec_graph* g) {
    for (int p = 0; p < 2; ++p) {
        if (g->exec[p]) { cudaGraphExecDestroy(g->exec[p]); g->exec[p] = nullptr; }
        if (g->graph[p]) { cudaGraphDestroy(g->graph[p]); g->graph[p] = nullptr; }
    }
}

// Capture the step at parity p (the stateful ops' cur set to p for the capture) into *out; counts its kernels and programmatic edges
// and the launches the eager step counts on a and on b.
static int graph_capture_one(adec_graph* g, int p, cudaGraph_t* out, int* kernels, int* edges, int64_t* da, int64_t* db) {
    adec_handle *a = g->a, *b = g->b;
    std::vector<HostSnap> snaps{HostSnap(a)};
    if (b && b != a) snaps.emplace_back(b);
    for (const HostSnap& sn : snaps) sn.h->enc_slots.dirty = sn.h->dec_slots.dirty = false;
    for (Op& op : graph_state_ops(g))
        if (op.P > 0) op.cur = p;
    cudaGraph_t graph = nullptr;
    cudaError_t ec = cudaStreamBeginCapture(g->cs, cudaStreamCaptureModeThreadLocal);
    if (ec != cudaSuccess) {
        for (const HostSnap& sn : snaps) sn.restore();
        return a->fail(fmt("graph: cudaStreamBeginCapture failed: %s", cudaGetErrorString(ec)));
    }
    const int rc = graph_body(g, g->cs);
    ec = cudaStreamEndCapture(g->cs, &graph);
    *da = a->launches - snaps[0].launches;
    *db = snaps.size() > 1 ? b->launches - snaps[1].launches : 0;
    for (const HostSnap& sn : snaps) sn.restore();
    if (rc || ec != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        return rc ? 1 : a->fail(fmt("graph: stream capture failed: %s", cudaGetErrorString(ec)));
    }
    size_t n = 0, ne = 0;
    std::vector<cudaGraphNode_t> nodes, from, to;
    std::vector<cudaGraphEdgeData> ed;
    cudaError_t e = cudaGraphGetNodes(graph, nullptr, &n);
    if (e == cudaSuccess) { nodes.resize(n); e = cudaGraphGetNodes(graph, nodes.data(), &n); }
    if (e == cudaSuccess) e = cudaGraphGetEdges_v2(graph, nullptr, nullptr, nullptr, &ne);
    if (e == cudaSuccess) { from.resize(ne); to.resize(ne); ed.resize(ne); e = cudaGraphGetEdges_v2(graph, from.data(), to.data(), ed.data(), &ne); }
    *kernels = *edges = 0;
    for (size_t i = 0; e == cudaSuccess && i < n; ++i) {
        cudaGraphNodeType t;
        e = cudaGraphNodeGetType(nodes[i], &t);
        *kernels += t == cudaGraphNodeTypeKernel;
    }
    for (size_t i = 0; i < ne; ++i) *edges += ed[i].type == cudaGraphDependencyTypeProgrammatic;
    if (e != cudaSuccess) { cudaGraphDestroy(graph); return a->fail(fmt("graph: %s", cudaGetErrorString(e))); }
    if (*kernels != *da + *db) {
        cudaGraphDestroy(graph);
        return a->fail(fmt("graph: %d kernels captured, the eager step counts %lld launches", *kernels, (long long)(*da + *db)));
    }
    *out = graph;
    return 0;
}

// Capture the step at both parities.  Every workspace is sized first, so nothing is allocated during a capture; the slot bits are
// taken as clean (adec_graph_launch copies dirty streams back eagerly before each launch).  Capturing both here keeps stream capture
// out of the launches that alternate parity: a launch only instantiates, and captures again only after a reallocation.
static int graph_capture(adec_graph* g) {
    adec_handle *a = g->a, *b = g->b, *sh = graph_state_handle(g);
    graph_drop(g);
    if (size_ws(sh, graph_state_ops(g), g->B, g->kind == ADEC_GRAPH_TX ? g->T : g->F, nullptr)) {
        if (sh != a) a->err = sh->err;
        return 1;
    }
    const uint64_t ga = a->gen, gb = b ? b->gen : 0;
    for (int p = 0; p < 2; ++p)
        if (graph_capture_one(g, p, &g->graph[p], &g->kernels, &g->edges, &g->da, &g->db)) { graph_drop(g); return 1; }
    if (a->gen != ga || (b && b->gen != gb)) {
        graph_drop(g);
        return a->fail("graph: a workspace was reallocated during the capture");
    }
    g->gen_a = ga;
    g->gen_b = gb;
    return 0;
}

static int graph_instantiate(adec_graph* g, int p) {
    const cudaError_t e = cudaGraphInstantiateWithFlags(&g->exec[p], g->graph[p], 0);
    if (e != cudaSuccess) { g->exec[p] = nullptr; return g->a->fail(fmt("graph: cudaGraphInstantiate failed: %s", cudaGetErrorString(e))); }
    ++g->instantiations;
    return 0;
}

int adec_graph_destroy(adec_graph* g) {
    if (!g) return 0;
    DeviceGuard dg(g->device);
    graph_drop(g);
    if (g->mid) cudaFree(g->mid);
    if (g->cs) cudaStreamDestroy(g->cs);
    delete g;
    return 0;
}

int adec_graph_create(int kind, adec_handle* a, adec_handle* b, int B, int T_or_F, int wire, const void* in, void* out, adec_graph** out_g) {
    if (!a || !out_g) { g_create_error = "graph_create: null argument"; return 1; }
    *out_g = nullptr;
    if (!a->finalized) return a->fail("graph_create: the handle is not finalized");
    if (kind != ADEC_GRAPH_TX && kind != ADEC_GRAPH_RX) return a->fail("graph_create: kind must be ADEC_GRAPH_TX or ADEC_GRAPH_RX");
    const bool tx = kind == ADEC_GRAPH_TX;
    if (tx && b) return a->fail("graph_create: a transmitter graph takes no decoder handle");
    if (!tx && (!b || !b->finalized)) return a->fail("graph_create: a receiver graph needs a finalized decoder handle");
    if (tx ? need_symad_tx(a, "graph_create (transmitter: encode, quantize)") : need_full_symad(a, "graph_create (receiver: lookup)"))
        return 1;
    if (!tx && b->cfg.model_type == ADEC_MODEL_SYMAD_ENCODER) return fail_encoder_only(a, "graph_create (receiver: decoder)");
    if (b && b->device != a->device)
        return a->fail(fmt("graph_create: the rx handle is on device %d, the decoder on device %d", a->device, b->device));
    if (!in || !out) return a->fail("graph_create: in and out must be device buffers");
    if (B < 1 || T_or_F < 1) return a->fail("graph_create: empty input");
    adec_handle* sh = tx ? a : b;
    if (B != sh->n_streams)
        return a->fail(fmt("graph_create: batch %d != n_streams %d of the %s handle (call adec_set_streams)", B, sh->n_streams,
                           tx ? "tx" : "decoder"));
    if (!tx) {
        const int zq_dim = b->cfg.model_type == ADEC_MODEL_HIFIGAN ? b->cfg.in_channels : b->cfg.code_dim;
        if (zq_dim != a->cfg.code_dim)
            return a->fail(fmt("graph_create: the decoder takes %d channels, the rx handle's codewords have %d", zq_dim, a->cfg.code_dim));
    }
    DeviceGuard dg(a->device);
    auto* g = new adec_graph();
    g->kind = kind; g->a = a; g->b = b; g->device = a->device; g->B = B; g->wire = wire != 0; g->in = in; g->out = out;
    g->T = tx ? T_or_F : 0;
    g->F = tx ? adec_frames_for(a, T_or_F) : T_or_F;
    const size_t mid_bytes = (size_t)B * g->F * a->cfg.code_dim * ((tx ? a : b)->act_bf16 ? 2 : 4);
    cudaError_t e = cudaStreamCreateWithFlags(&g->cs, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMalloc(&g->mid, mid_bytes);
    if (e != cudaSuccess) {
        a->fail(fmt("graph_create: %s", cudaGetErrorString(e)));
        adec_graph_destroy(g);
        return 1;
    }
    const int p = list_parity(graph_state_ops(g));
    if (p < 0) {
        a->fail("graph_create: the stateful ops of the handle disagree on which state buffer is current");
        adec_graph_destroy(g);
        return 1;
    }
    if (graph_capture(g) || graph_instantiate(g, p)) { adec_graph_destroy(g); return 1; }
    *out_g = g;
    return 0;
}

int adec_graph_launch(adec_graph* g, void* stream) {
    if (!g) return 1;
    adec_handle *a = g->a, *b = g->b, *sh = graph_state_handle(g);
    const cudaStream_t s = (cudaStream_t)stream;
    DeviceGuard dg(a->device);
    for (adec_handle* h : {a, b})     // profiling, the kernel trace and launch records see every launch: run the eager sequence
        if (h && (h->profiling || h->d_ktrace || h->launch_log)) return graph_body(g, s);
    if (sh->n_streams != g->B)
        return a->fail(fmt("graph_launch: the %s handle has %d streams, the graph was made for %d (call adec_set_streams)",
                           g->kind == ADEC_GRAPH_TX ? "tx" : "decoder", sh->n_streams, g->B));
    std::vector<Op>& ops = graph_state_ops(g);
    if (slot_fixup(sh, ops, s)) { if (sh != a) a->err = sh->err; return 1; }
    const int p = list_parity(ops);
    if (p < 0) return a->fail("graph_launch: the stateful ops of the handle disagree on which state buffer is current");
    if ((a->gen != g->gen_a || (b && b->gen != g->gen_b)) && graph_capture(g)) return 1;
    if (!g->exec[p] && graph_instantiate(g, p)) return 1;
    CK(a, cudaGraphLaunch(g->exec[p], s));
    for (Op& op : ops)
        if (op.P > 0) op.cur ^= 1;
    a->launches += g->da;
    if (b && b != a) b->launches += g->db;
    return 0;
}

int adec_graph_info(const adec_graph* g, int* kernels, int* programmatic_edges, int* instantiations) {
    if (!g) return 1;
    if (kernels) *kernels = g->kernels;
    if (programmatic_edges) *programmatic_edges = g->edges;
    if (instantiations) *instantiations = g->instantiations;
    return 0;
}

// -------------------------------------------------------------------------------------------------
// One test's op list (one op, or the two launches of a split residual unit) and its host I/O.  Elements are h->act_bytes() wide: fp32,
// or bf16 words for a compute_dtype 2 handle.  Layouts as adec_test_conv_op documents them.
struct TestIO {
    CallMode mode = CALL_STREAM;
    int n_calls = 1, B = 1, n_streams = 1;
    const int* lengths = nullptr;   // (n_calls, B)
    const int* streams = nullptr;   // (n_calls, B), CALL_SLOTS
    const void* x = nullptr;
    const void* res = nullptr;
    void* state = nullptr;
    void* y = nullptr;
    int Cin_x = 0;                  // channels of x and state
    int Cout_total = 0;             // output channels (all groups; a transposed conv's per output row)
};

// Runs `ops` (built, not finalized) as the decoder list of `h`, through run_call: the codec's own call path, slot bits and state
// buffers.  x and res go from channels-first to the channels-last row spaces the kernels read (utterance after utterance; uniform
// calls are the same rows), and y and state come back the other way.
static int run_test_ops(adec_handle* h, std::vector<Op> ops, const TestIO& io) {
    const size_t eb = h->act_bytes();
    auto put = [eb](void* dst, size_t i, const void* src, size_t j) { memcpy((char*)dst + i * eb, (const char*)src + j * eb, eb); };
    const bool vl = io.mode == CALL_VARLEN || io.mode == CALL_SLOTS;
    const bool split = ops.size() == 2;
    {   // wiring: x in EXT_IN (split unit: workspace 2, which is also its skip input), y to EXT_OUT, a conv's residual in workspace 0
        Op& f = ops.front();
        Op& l = ops.back();
        const int ldx = (f.shared_in ? 1 : f.G) * f.Cin;
        f.in_buf = split ? 2 : BUF_EXT_IN; f.ldx = ldx; f.x_goff = f.shared_in ? 0 : f.Cin;
        if (split) {
            f.out_buf = 1; f.ldy = f.Cout; f.y_goff = f.Cout;
            l.in_buf = 1; l.ldx = f.Cout; l.x_goff = l.Cin;
            l.res_buf = 2; l.ldr = ldx; l.r_goff = 0;
        }
        l.out_buf = BUF_EXT_OUT; l.ldy = l.G * l.Cout; l.y_goff = l.Cout;
        if (io.res) { l.res_buf = 0; l.ldr = l.ldy; l.r_goff = l.Cout; }
    }
    for (Op& op : ops)
        if (finalize_op(h, &op)) return 1;
    h->dec_ops = std::move(ops);        // the handle owns the state buffers from here (adec_destroy)
    for (Op& op : h->dec_ops)
        if (alloc_state(h, &op, io.n_streams)) return 1;
    h->n_streams = h->st_cap = io.n_streams;
    h->dec_slots.bit.assign(io.n_streams, 0);
    h->finalized = true;
    const Op& f = h->dec_ops.front();
    const Op& l = h->dec_ops.back();
    const int G = f.shared_in ? 1 : f.G, cin_g = io.Cin_x / G;
    const int cout_g = io.Cout_total / l.G, up = l.up;
    const size_t per = (size_t)f.P * f.st_C;
    if (per && io.state && io.mode != CALL_VARLEN) {
        std::vector<char> hs(per * io.n_streams * eb, 0);
        for (int s = 0; s < io.n_streams; ++s)
            for (int g = 0; g < G; ++g)
                for (int c = 0; c < cin_g; ++c)
                    for (int p = 0; p < f.P; ++p)
                        put(hs.data(), ((size_t)s * f.P + p) * f.st_C + g * f.Cin + c, io.state, ((size_t)s * io.Cin_x + g * cin_g + c) * f.P + p);
        CK(h, cudaMemcpy(f.st[0], hs.data(), hs.size(), cudaMemcpyHostToDevice));
    }
    size_t x_at = 0, y_at = 0;          // elements of x / y (and res) consumed by the previous calls
    for (int k = 0; k < io.n_calls; ++k) {
        const int* len = io.lengths + (size_t)k * io.B;
        std::vector<long long> in_off(io.B + 1, 0), out_off(io.B + 1, 0);
        for (int b = 0; b < io.B; ++b) {
            if (len[b] < 1 || (!vl && len[b] != len[0])) return h->fail("test_conv_op: lengths must be >= 1, and equal in modes 0 and 1");
            in_off[b + 1] = in_off[b] + len[b];
            out_off[b + 1] = out_off[b] + (len[b] - 1) / f.down + 1;
        }
        const long long rows_in = in_off[io.B], rows_out = out_off[io.B];
        std::vector<char> xl((size_t)rows_in * f.ldx * eb, 0);
        for (int b = 0; b < io.B; ++b)
            for (int g = 0; g < G; ++g)
                for (int c = 0; c < cin_g; ++c)
                    for (int t = 0; t < len[b]; ++t)
                        put(xl.data(), (size_t)(in_off[b] + t) * f.ldx + g * f.Cin + c, io.x,
                            x_at + (size_t)io.Cin_x * in_off[b] + (size_t)(g * cin_g + c) * len[b] + t);
        DevBuf& xb = split ? h->ws[2] : h->hx;
        if (ensure(h, xb, (xl.size() + 3) / 4)) return 1;
        CK(h, cudaMemcpy(xb.p, xl.data(), xl.size(), cudaMemcpyHostToDevice));
        if (io.res) {
            std::vector<char> rl((size_t)rows_out * l.ldy * eb, 0);
            for (int b = 0; b < io.B; ++b)
                for (int g = 0; g < l.G; ++g)
                    for (int c = 0; c < cout_g; ++c)
                        for (long long t = 0; t < out_off[b + 1] - out_off[b]; ++t)
                            put(rl.data(), (size_t)(out_off[b] + t) * l.ldy + g * l.Cout + c, io.res,
                                y_at + (size_t)io.Cout_total * out_off[b] + (size_t)(g * cout_g + c) * (out_off[b + 1] - out_off[b]) + t);
            if (ensure(h, h->ws[0], (rl.size() + 3) / 4)) return 1;
            CK(h, cudaMemcpy(h->ws[0].p, rl.data(), rl.size(), cudaMemcpyHostToDevice));
        }
        const size_t ybytes = (size_t)rows_out * l.ldy * eb;
        if (ensure(h, h->hy, (ybytes + 3) / 4)) return 1;
        const Call call{true, io.mode, h->act_bf16, vl ? len : nullptr, io.mode == CALL_SLOTS ? io.streams + (size_t)k * io.B : nullptr};
        if (run_call(h, call, split ? nullptr : h->hx.p, io.B, len[0], h->hy.p, nullptr)) return 1;
        CK(h, cudaDeviceSynchronize());
        std::vector<char> yl(ybytes);
        CK(h, cudaMemcpy(yl.data(), h->hy.p, yl.size(), cudaMemcpyDeviceToHost));
        for (int b = 0; b < io.B; ++b) {
            const long long to = out_off[b + 1] - out_off[b];
            const size_t yo = y_at + (size_t)io.Cout_total * up * out_off[b];
            if (up > 1) {       // (Tout, up * Cout) rows are (Tout * up, Cout)
                for (int c = 0; c < io.Cout_total; ++c)
                    for (long long j = 0; j < to; ++j)
                        for (int r = 0; r < up; ++r)
                            put(io.y, yo + (size_t)c * to * up + j * up + r, yl.data(), (size_t)(out_off[b] + j) * l.ldy + r * io.Cout_total + c);
                continue;
            }
            // out_nct: uniform calls write (B, G * Cout, Tout), varlen calls one (G * Cout, rows) over all utterances
            const long long nct_ld = vl ? rows_out : to, nct_b = vl ? out_off[b] : (long long)b * l.G * l.Cout * to;
            for (int g = 0; g < l.G; ++g)
                for (int c = 0; c < cout_g; ++c)
                    for (long long t = 0; t < to; ++t)
                        put(io.y, yo + (size_t)(g * cout_g + c) * to + t, yl.data(),
                            l.out_nct ? (size_t)(nct_b + (long long)(g * l.Cout + c) * nct_ld + t) : (size_t)(out_off[b] + t) * l.ldy + g * l.Cout + c);
        }
        x_at += (size_t)io.Cin_x * rows_in;
        y_at += (size_t)io.Cout_total * up * rows_out;
    }
    if (per && io.state && io.mode != CALL_VARLEN) {     // each stream's current state: st[cur], or the other buffer if its slot bit is set
        std::vector<char> sl[2];
        for (int i = 0; i < 2; ++i) {
            sl[i].resize(per * io.n_streams * eb);
            CK(h, cudaMemcpy(sl[i].data(), f.st[f.cur ^ i], sl[i].size(), cudaMemcpyDeviceToHost));
        }
        for (int s = 0; s < io.n_streams; ++s) {
            const char* src = sl[h->dec_slots.bit[s]].data();
            for (int g = 0; g < G; ++g)
                for (int c = 0; c < cin_g; ++c)
                    for (int p = 0; p < f.P; ++p)
                        put(io.state, ((size_t)s * io.Cin_x + g * cin_g + c) * f.P + p, src, ((size_t)s * f.P + p) * f.st_C + g * f.Cin + c);
        }
    }
    return 0;
}

// The single-layer entry points below: B uniform streams of T rows, one call.  x (B, Cin_real, T), state (B, Cin_real, P), res
// (B, Cout_real_total, Tout) or nullptr; offline: Generator.forward (zero history, first-row replication in transposed convs), state
// is neither read nor written and may be nullptr.
static int run_single(adec_handle* h, Op& op, const void* x, int B, int Cin_real, int T, int Cout_real_total, void* state, void* y,
                      const void* res = nullptr, bool offline = false) {
    TestIO io;
    io.mode = offline ? CALL_OFFLINE : CALL_STREAM;
    io.B = io.n_streams = B;
    std::vector<int> len(B, T);
    io.lengths = len.data();
    io.x = x; io.res = res; io.state = offline ? nullptr : state; io.y = y;
    io.Cin_x = Cin_real; io.Cout_total = Cout_real_total;
    return run_test_ops(h, std::vector<Op>{op}, io);
}

int adec_test_causal_conv(int device, const float* x, int B, int Cin, int T, const float* w, const float* bias, int Cout,
                          int K, int stride, int dil, int groups, int pre_act, float slope, float* state, float* y) {
    adec_config cfg{};
    adec_handle* h = nullptr;
    if (adec_create(&cfg, device, &h)) return 1;
    DeviceGuard dg(device);
    HostTensor W, Bt;
    W.shape = {Cout, Cin / groups, K};
    W.data.assign(w, w + (size_t)Cout * (Cin / groups) * K);
    if (bias) { Bt.shape = {Cout}; Bt.data.assign(bias, bias + Cout); }
    Op op;
    int rc = make_conv_op(h, &op, "test_conv", W, bias ? &Bt : nullptr, stride, dil, groups, pre_act, slope, false);
    if (!rc) rc = run_single(h, op, x, B, Cin, T, Cout, state, y);
    if (rc) g_create_error = h->err;
    adec_destroy(h);
    return rc;
}

int adec_test_residual_unit(int device, const float* x, int B, int C, int T, const float* w1, const float* w2, int K, int dil,
                            float* state, float* y) {
    adec_config cfg{};
    adec_handle* h = nullptr;
    if (adec_create(&cfg, device, &h)) return 1;
    DeviceGuard dg(device);
    HostTensor W1, W2;
    W1.shape = {C, C, K};
    W1.data.assign(w1, w1 + (size_t)C * C * K);
    W2.shape = {C, C, 1};
    W2.data.assign(w2, w2 + (size_t)C * C);
    Op op;
    int rc = make_ru_op(h, &op, "test_ru", W1, W2, dil, ACT_ELU);
    if (!rc && h->engine != 0 && op.Cout > h->tc_max_fuse) rc = h->fail("test_ru: C > 128 runs as two ops on the tensor-core path; test those separately");
    if (!rc) rc = run_single(h, op, x, B, C, T, C, state, y);
    if (rc) g_create_error = h->err;
    adec_destroy(h);
    return rc;
}

int adec_test_causal_convtr(int device, const float* x, int B, int Cin, int T, const float* w, const float* bias, int Cout,
                            int stride, float* state, float* y) {
    adec_config cfg{};
    adec_handle* h = nullptr;
    if (adec_create(&cfg, device, &h)) return 1;
    DeviceGuard dg(device);
    HostTensor W, Bt;
    W.shape = {Cin, Cout, 2 * stride};
    W.data.assign(w, w + (size_t)Cin * Cout * 2 * stride);
    if (bias) { Bt.shape = {Cout}; Bt.data.assign(bias, bias + Cout); }
    Op op;
    int rc = make_convtr_op(h, &op, "test_convtr", W, bias ? &Bt : nullptr, stride, ACT_NONE, 0.f);
    if (!rc) rc = run_single(h, op, x, B, Cin, T, Cout, state, y);
    if (rc) g_create_error = h->err;
    adec_destroy(h);
    return rc;
}

// One vocoder layer as a compute_dtype 1 / 2 HiFi-GAN handle builds and runs it (the same op builders, packer and launch path as
// build_hifigan / run_ops), so the tests can pin its rounding layer by layer.
int adec_test_vocoder_layer(int device, int compute_dtype, int kind, const void* x, int B, int Cin, int T, const float* w,
                            const float* bias, int Cout, int K, int dil, int up, int groups, int shared_in, int pre_act, float slope,
                            const float* mean, const float* scale, const void* res, int offline, void* state, void* y) {
    if (compute_dtype != 1 && compute_dtype != 2) {
        g_create_error = "adec_test_vocoder_layer: compute_dtype must be 1 or 2 (the fp32-grade engines: adec_test_causal_conv / _convtr)";
        return 1;
    }
    adec_config cfg{};
    cfg.model_type = ADEC_MODEL_HIFIGAN;
    cfg.compute_dtype = compute_dtype;
    cfg.in_channels = Cin;
    adec_handle* h = nullptr;
    if (adec_create(&cfg, device, &h)) return 1;
    DeviceGuard dg(device);
    int rc = 0;
    Op op;
    if (!x || !w || !y || B < 1 || T < 1 || (!offline && !state)) {
        rc = h->fail("adec_test_vocoder_layer: NULL x, w, y or (streaming) state, or B / T < 1");
    } else if (kind == 0 && (groups < 1 || Cin % groups || Cout % groups)) {
        rc = h->fail("adec_test_vocoder_layer: Cin and Cout must divide into groups");
    } else if (kind == 0 && pre_act == ACT_NORM && (groups != 1 || !mean || !scale)) {
        rc = h->fail("adec_test_vocoder_layer: norm needs groups = 1, mean and scale");
    } else if (kind == 0) {
        HostTensor W, Bt;
        W.shape = {Cout, Cin / groups, K};
        W.data.assign(w, w + (size_t)Cout * (Cin / groups) * K);
        if (bias) { Bt.shape = {Cout}; Bt.data.assign(bias, bias + Cout); }
        rc = make_conv_op(h, &op, "test_conv", W, bias ? &Bt : nullptr, 1, dil, groups, pre_act, slope, shared_in != 0);
        if (!rc && pre_act == ACT_NORM) {      // padded like build_hifigan's stats
            std::vector<float> mp(op.Cin, 0.f), sp(op.Cin, 1.f);
            std::copy(mean, mean + Cin, mp.begin());
            std::copy(scale, scale + Cin, sp.begin());
            if (dev_upload(h, &h->d_mean, mp) || dev_upload(h, &h->d_scale, sp)) rc = 1;
            op.mean = h->d_mean; op.scale = h->d_scale;
        }
        // shared_in: x and state hold the Cin / groups channels every group reads
        if (!rc) rc = run_single(h, op, x, B, shared_in ? Cin / groups : Cin, T, Cout, state, y, res, offline != 0);
    } else if (res) {
        rc = h->fail("adec_test_vocoder_layer: a residual is built for kind 0 only");
    } else if (kind == 1) {
        HostTensor W, Bt;
        W.shape = {Cin, Cout, 2 * up};
        W.data.assign(w, w + (size_t)Cin * Cout * 2 * up);
        if (bias) { Bt.shape = {Cout}; Bt.data.assign(bias, bias + Cout); }
        rc = make_convtr_op(h, &op, "test_convtr", W, bias ? &Bt : nullptr, up, ACT_LRELU, slope);
        if (!rc) rc = run_single(h, op, x, B, Cin, T, Cout, state, y, nullptr, offline != 0);
    } else if (kind == 2) {
        HostTensor W, Bt;      // through the state dict, as build_hifigan builds output_conv
        W.shape = {Cout, Cin, K};
        W.data.assign(w, w + (size_t)Cout * Cin * K);
        h->tensors["test_head.conv.weight"] = W;
        if (bias) { Bt.shape = {1}; Bt.data.assign(bias, bias + 1); h->tensors["test_head.conv.bias"] = Bt; }
        rc = build_head(h, &op, "test_head", ACT_LRELU, slope, true);
        if (!rc) rc = run_single(h, op, x, B, Cin, T, 1, state, y, nullptr, offline != 0);
    } else {
        rc = h->fail("adec_test_vocoder_layer: kind must be 0 (conv), 1 (transposed conv) or 2 (head)");
    }
    if (rc) g_create_error = h->err;
    adec_destroy(h);
    return rc;
}

int adec_test_conv_op(int device, const adec_test_op* d, int mode, int n_calls, int B, int n_streams, const int* lengths,
                      const int* streams, const float* x, const float* res, float* state, float* y, int* launched, int max_launched,
                      int* range_flag) {
    if (!d || !d->w || !x || !y || !lengths || mode < CALL_STREAM || mode > CALL_SLOTS || n_calls < 1 || B < 1 ||
        (mode == CALL_SLOTS && (!streams || n_streams < B)) || (launched && max_launched < 0)) {
        g_create_error = "adec_test_conv_op: bad argument";
        return 1;
    }
    // fp32: a symAD handle, the engine ADEC_CONV_PATH names; bf16: a symAD decoder-only handle with that compute_dtype (f16 engine)
    adec_config cfg{};
    cfg.model_type = d->compute_dtype ? ADEC_MODEL_SYMAD_DECODER : ADEC_MODEL_SYMAD;
    cfg.compute_dtype = d->compute_dtype;
    adec_handle* h = nullptr;
    if (adec_create(&cfg, device, &h)) return 1;
    DeviceGuard dg(device);
    if (launched) adec_record_launches(h, 1);
    auto tensor = [](std::vector<int64_t> shape, const float* p) {
        HostTensor t;
        t.shape = std::move(shape);
        if (p) t.data.assign(p, p + t.numel());
        return t;
    };
    std::vector<Op> ops(1);
    int rc = 0, cin_x = d->Cin, cout_total = d->Cout;
    const HostTensor Bt = tensor({d->kind == ADEC_TEST_CONV || d->kind == ADEC_TEST_CONVTR ? d->Cout : 0}, d->bias);   // conv biases
    switch (d->kind) {
    case ADEC_TEST_CONV:
        if (d->groups < 1 || d->Cin % d->groups || d->Cout % d->groups) { rc = h->fail("test_conv_op: Cin and Cout must divide into groups"); break; }
        if (d->pre_act == ACT_NORM && (d->groups != 1 || !d->mean || !d->scale)) { rc = h->fail("test_conv_op: norm needs groups = 1, mean and scale"); break; }
        rc = make_conv_op(h, &ops[0], "test_conv", tensor({d->Cout, d->Cin / d->groups, d->K}, d->w), d->bias ? &Bt : nullptr, d->stride,
                          d->dil, d->groups, d->pre_act, d->slope, d->shared_in != 0);
        ops[0].out_nct = d->out_nct != 0;
        if (d->shared_in) cin_x = d->Cin / d->groups;
        if (!rc && d->pre_act == ACT_NORM) {      // padded like build_hifigan's stats
            std::vector<float> mp(ops[0].Cin, 0.f), sp(ops[0].Cin, 1.f);
            std::copy(d->mean, d->mean + d->Cin, mp.begin());
            std::copy(d->scale, d->scale + d->Cin, sp.begin());
            if (dev_upload(h, &h->d_mean, mp) || dev_upload(h, &h->d_scale, sp)) rc = 1;
            ops[0].mean = h->d_mean; ops[0].scale = h->d_scale;
        }
        break;
    case ADEC_TEST_RU:
        if (!d->w2 || d->Cin != d->Cout) { rc = h->fail("test_conv_op: a residual unit needs w2 and Cin = Cout"); break; }
        rc = make_ru_op(h, &ops[0], "test_ru", tensor({d->Cout, d->Cout, d->K}, d->w), tensor({d->Cout, d->Cout, 1}, d->w2), d->dil, ACT_ELU);
        if (!rc && h->engine != 0 && ops[0].Cout > h->tc_max_fuse) {     // as push_ru builds it
            Op conv, pw;
            split_ru_op(ops[0], &conv, &pw);
            ops = {conv, pw};
        }
        break;
    case ADEC_TEST_CONVTR:
        rc = make_convtr_op(h, &ops[0], "test_convtr", tensor({d->Cin, d->Cout, 2 * d->stride}, d->w), d->bias ? &Bt : nullptr, d->stride,
                            d->pre_act, d->slope);
        break;
    case ADEC_TEST_STEM:     // through the state dict, as build_symad builds encoder.conv: fp32 weights in every compute_dtype
        h->tensors["test.conv.weight"] = tensor({32, 1, 7}, d->w);
        if (d->bias) h->tensors["test.conv.bias"] = tensor({32}, d->bias);
        rc = build_stem(h, &ops[0], "test", 32);
        cin_x = 1; cout_total = 32;
        break;
    case ADEC_TEST_HEAD:     // as build_symad / build_hifigan build decoder.conv2 / output_conv
        h->tensors["test.conv.weight"] = tensor({1, 32, 7}, d->w);
        if (d->bias) h->tensors["test.conv.bias"] = tensor({1}, d->bias);
        rc = build_head(h, &ops[0], "test", d->pre_act, d->slope, d->post_tanh != 0);
        cin_x = 32; cout_total = 1;
        break;
    default:
        rc = h->fail("test_conv_op: unknown kind");
    }
    if (!rc) {
        TestIO io;
        io.mode = (CallMode)mode;
        io.n_calls = n_calls; io.B = B;
        io.n_streams = mode == CALL_SLOTS ? n_streams : mode == CALL_VARLEN ? 1 : B;
        io.lengths = lengths; io.streams = streams;
        io.x = x; io.res = res; io.state = state; io.y = y;
        io.Cin_x = cin_x; io.Cout_total = cout_total;
        rc = run_test_ops(h, std::move(ops), io);
    }
    if (!rc && launched)
        for (int i = 0; i < max_launched * ADEC_TEST_REC; ++i) launched[i] = i < (int)h->launch_rec.size() ? h->launch_rec[i] : -1;
    if (!rc && range_flag) {
        range_flag[0] = adec_range_error(h, nullptr);
        range_flag[1] = adec_range_error(h, nullptr);
        if (range_flag[0] < 0 || range_flag[1] < 0) rc = 1;
    }
    if (rc) g_create_error = h->err;
    adec_destroy(h);
    return rc;
}

}  // extern "C"
