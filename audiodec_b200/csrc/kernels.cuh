// audiodec_b200 device kernels (sm_90a).
//
// Everything the reference does with torch.cat + nn.Conv1d / nn.ConvTranspose1d + separate
// activation / add kernels (layers/conv_layer.py:153-156,194-197; residual_unit.py:78-81) is one
// kernel family here:
//
//   conv_gemm_kernel  - stateful causal conv as an im2col-free implicit GEMM on CUDA cores
//                       (fp32 FFMA: the 1e-4 / bit-identical-index contract rules out TF32/bf16).
//                       Activations are channels-last (B,T,C) in HBM so a time window is one
//                       contiguous range and every load is a 128-bit channel vector.  The CTA keeps
//                       its input window [t0-halo, t0+TT) x C in shared memory (pre-activation and
//                       causal history applied while it is written), weight tiles are streamed
//                       L2 -> smem by a producer warp with cp.async.bulk (TMA, 1-D) through a
//                       4-stage mbarrier ring, 8x8 register micro-tiles accumulate, and the epilogue
//                       fuses bias / residual / layout.  With FUSE the whole residual unit
//                       ELU -> k7 dilated -> ELU -> 1x1 -> +x runs without leaving the SM.
//   stem_kernel       - Cin = 1 first conv (pure store bandwidth).
//   head_kernel       - Cout = 1 last conv (+ LeakyReLU / bias / tanh for the vocoder).
//   rvq_kernel        - 8-stage residual VQ: fp32 distances in the reference's rounding order,
//                       first-index arg-min by warp shuffles, int64 flat indices.
//   lookup_kernel     - codebook gather-sum (fp32 zq, or bf16 zq rounded once).
//   zq_moments_kernel - per-utterance fp64 sums and centred second moments of zq (corpus statistics).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

namespace adec {

enum PreAct { ACT_NONE = 0, ACT_ELU = 1, ACT_LRELU = 2, ACT_NORM = 3 };

// ------------------------------------------------------------------------------------------------
// small PTX helpers (mbarrier + 1-D bulk async copy)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
// try_wait with a suspend-time hint: the warp sleeps in hardware until the phase completes (or the hint expires)
// instead of spinning - polling loops were 30-40 % of all issued instructions in the first tensor-core profile.
__device__ __forceinline__ bool mbar_try_wait(uint64_t* b, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n selp.u32 %0, 1, 0, p;\n}"
        : "=r"(ok)
        : "r"(smem_u32(b)), "r"(parity), "r"(0x989680u)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug must trap (kernel error) instead of hanging the GPU.  The clock is only consulted every
// 64 failed probes so the common path stays a 2-instruction loop.  The bound is ~20 s of SM clocks: far beyond any legitimate wait
// even when the context is time-sliced with other tenants (clock64 keeps counting while descheduled); -DADEC_NO_WATCHDOG compiles
// the check out (plain try_wait loop with the hardware suspend hint).
#ifndef ADEC_WATCHDOG_CYCLES
#define ADEC_WATCHDOG_CYCLES 40000000000LL
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity, int tag = 0) {
    if (mbar_try_wait(b, parity)) return;
#ifdef ADEC_NO_WATCHDOG
    while (!mbar_try_wait(b, parity)) { }
#else
    const long long t0 = clock64();
    while (true) {
        // 64 bare probes (2 instructions each: the polling loop was 16 % of all issued instructions with the clock test inside it)
#pragma unroll 1
        for (int it = 0; it < 64; ++it) {
            if (mbar_try_wait(b, parity)) return;
#ifdef ADEC_WAIT_SLEEP
            if (tag != 200 && tag != 250 && tag != 300 && tag != 400) __nanosleep(ADEC_WAIT_SLEEP);   // not the MMA issuers: they are the critical path
#endif
        }
        if (clock64() - t0 > ADEC_WATCHDOG_CYCLES) {
#ifdef ADEC_WATCHDOG_PRINT
            printf("adec: mbarrier wait timed out: tag %d parity %u block (%d,%d,%d) thread %d\n", tag, parity, blockIdx.x, blockIdx.y,
                   blockIdx.z, threadIdx.x);
#endif
            __trap();
        }
    }
#endif
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// nn.ELU(alpha=1): x > 0 ? x : expm1(x).  expm1f() costs ~40 instructions and the elementwise work, not the tensor
// pipe, bounds the narrow layers; ex2.approx(x*log2e) - 1 is 4 instructions and within 2.4e-7 ABSOLUTE of expm1 on
// (-inf, 0] (2^-22 relative error of ex2.approx on a value <= 1) - the same order as the fp32 rounding of the O(1)
// activations it is summed with.  Parity margins: tests/test_layers_gpu.py (1e-5 on a fused unit), golden indices.
// __expf() wraps ex2.approx in a denormal-range fix-up (FSETP -126 / FMUL 0.5 / FMUL square: 8 instructions per ELU, 18 % of all
// instructions of the C = 32 unit in the round-2 ncu capture); ex2.approx.ftz is the bare MUFU.EX2 and gives the same ELU bit for bit:
// where the two differ (x log2(e) < -126) exp(x) is below 2^-126 and exp(x) - 1 rounds to -1 either way.
__device__ __forceinline__ float act_elu(float v) {
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * 1.4426950408889634f));
    e -= 1.0f;
    return v > 0.f ? v : e;
}
__device__ __forceinline__ float act_lrelu(float v, float s) { return v > 0.f ? v : v * s; }

__device__ __forceinline__ float4 apply_act(float4 v, int act, float slope) {
    if (act == ACT_ELU) {
        v.x = act_elu(v.x); v.y = act_elu(v.y); v.z = act_elu(v.z); v.w = act_elu(v.w);
    } else if (act == ACT_LRELU) {
        v.x = act_lrelu(v.x, slope); v.y = act_lrelu(v.y, slope); v.z = act_lrelu(v.z, slope); v.w = act_lrelu(v.w, slope);
    }
    return v;
}

// Activation storage in HBM (x, causal state, residual, y): fp32, or bf16 (compute_dtype 2, the vocoder's bf16-activation mode).  bf16
// values are widened to fp32 on load; arithmetic stays fp32 and every stored value is rounded to nearest once.
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t bf2_bits(float x, float y) { const __nv_bfloat162 h = __floats2bfloat162_rn(x, y); return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ float4 bf4_f4(uint2 r) { return make_float4(bf_lo(r.x), bf_hi(r.x), bf_lo(r.y), bf_hi(r.y)); }
__device__ __forceinline__ uint2 f4_bf4(float4 v) { return make_uint2(bf2_bits(v.x, v.y), bf2_bits(v.z, v.w)); }
// 8 consecutive channels: 32 B of fp32 or one 16-byte vector of bf16
__device__ __forceinline__ void ldg8(const float* p, float4& u, float4& v) {
    u = __ldg(reinterpret_cast<const float4*>(p));
    v = __ldg(reinterpret_cast<const float4*>(p) + 1);
}
__device__ __forceinline__ void ldg8(const __nv_bfloat16* p, float4& u, float4& v) {
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(p));
    u = bf4_f4(make_uint2(r.x, r.y));
    v = bf4_f4(make_uint2(r.z, r.w));
}
// 4 consecutive channels
__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ldg4(const __nv_bfloat16* p) { return bf4_f4(__ldg(reinterpret_cast<const uint2*>(p))); }
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 ld4(const __nv_bfloat16* p) { return bf4_f4(*reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__nv_bfloat16* p, float4 v) { *reinterpret_cast<uint2*>(p) = f4_bf4(v); }
// 2 consecutive channels, 1 value
__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float2 ldg2(const __nv_bfloat16* p) { const uint32_t w = __ldg(reinterpret_cast<const unsigned int*>(p)); return make_float2(bf_lo(w), bf_hi(w)); }
__device__ __forceinline__ void st2(float* p, float x, float y) { *reinterpret_cast<float2*>(p) = make_float2(x, y); }
__device__ __forceinline__ void st2(__nv_bfloat16* p, float x, float y) { *reinterpret_cast<uint32_t*>(p) = bf2_bits(x, y); }
__device__ __forceinline__ void st1(float* p, float x) { *p = x; }
__device__ __forceinline__ void st1(__nv_bfloat16* p, float x) { *p = __float2bfloat16_rn(x); }
// the value a store of type T keeps (bf16 storage: what the causal state holds, so that a window row read from the chunk matches it)
template <bool BST> __device__ __forceinline__ float4 stored4(float4 v) { return BST ? bf4_f4(f4_bf4(v)) : v; }


// ------------------------------------------------------------------------------------------------
// conv_gemm_kernel
// ------------------------------------------------------------------------------------------------
// The conv is evaluated as  Y[t][co] = sum_{piece,tap,ci} Xw[t + tap*dil][piece*CW + ci] * W[tap][ci][co]
// over an "extended" input x~ = history(P rows) || chunk(T rows) (layers/conv_layer.py:154).
//   * stride-s convs (k = 2s) use RG = s: s consecutive x~ rows are folded into one window row of
//     s*Cin channels, which turns them into 2-tap stride-1 convs (and keeps smem reads conflict-free);
//   * transposed convs (k = 2s, crop [s:-s], conv_layer.py:197) are 2-tap convs with s*Cout outputs:
//     y[j*s+r] = b + W[:,:,r]^T x[j] + W[:,:,s+r]^T x[j-1]; the (T, s*Cout) result *is* (T*s, Cout).
// ADEC_PHASES (a diagnostic build, tools/conv_phases.py): wg_conv_kernel counts SM cycles per role and phase.  A ConvArgs::dbg record
// is then {start ns, end ns, CTA 0 cycles, launch descriptor, Tout, PH_N, cycle sums [PH_N]}; the sums are over the CTAs of the
// launch, from one thread per consumer warpgroup, activation-producer thread 0 and the weight-producer lane.
enum { PH_WIN, PH_WGT, PH_MMA, PH_MID, PH_EPI,      // consumers: wait for a window piece, for a weight stage, MMA groups,
                                                    //   fused intermediate, epilogue
       PH_FREE, PH_LOAD, PH_CONV,                   // activation producers: wait for a free window buffer, global loads, convert
       PH_WFREE, PH_WISSUE,                         // weight producer: wait for a free stage, everything else
       PH_N };
#ifdef ADEC_PHASES
constexpr int KT_REC = 6 + PH_N;
#else
constexpr int KT_REC = 3;
#endif
struct ConvArgs {
    // input activations, channels-last; group g reads channels [g*x_goff, g*x_goff + Cin)
    const float* x;
    long long x_bs;
    int ldx, x_goff;
    // causal state (history rows), (B, P, st_ld); ping-pong in/out
    const float* st_in;
    float* st_out;
    int st_ld, st_goff, st_groups;   // st_groups: how many groups own distinct state channels
    int P, T, Tout;
    int Ktaps, dil, RG, lgCin, Cin;  // Cin: channels per x~ row (per group)
    int n_pieces;
    int pre_act;
    float slope;
    const float* mean;   // ACT_NORM: (v - mean[c]) / scale[c]   (HiFiGAN.py:276-279)
    const float* scale;
    // weights (packed by the host, see pack_weights in adec.cu)
    const float* w;
    const float* w2;     // FUSE: the residual unit's 1x1 conv
    const float* bias;   // [g*Cout_g + co] or nullptr
    int n_co_tiles, Cout_g;
    long long w_tile_floats;   // floats per (group, co_tile) of w
    // residual (raw), output
    const float* res;
    long long res_bs;
    int ldr, r_goff;
    float* y;
    long long y_bs;
    int ldy, y_goff, out_nct;
    int mid_act;         // FUSE: activation between the two GEMMs
    int hist_rep;        // non-streaming forward of a transposed conv: history rows = the FIRST input row (ReplicationPad1d,
                         // conv_layer.py:189-192) instead of the stored state
    // fp16-split tensor-core engine (wg_conv.cuh): each output column's weights are stored times its own power of two; the sums are
    // multiplied by cscale[g*Cout_g + co] (FUSE: the intermediate's; the 1x1 conv's are cscale[Cout_g + co]).  nullptr otherwise
    const float* cscale;
    int n_wbuf;          // window buffers in shared memory (1..4)
    // stacked rows: when a stream contributes fewer rows than a 128-row tile, the tiles run over ONE row space in which stream s owns
    // rows [s * stack_L, (s + 1) * stack_L), stack_L = Tout + (Ktaps - 1) * dil: local rows >= Tout are the receptive-field overlap into
    // the next stream and are computed but never stored.  0 = one row space per stream (blockIdx-style b dimension).
    int stack_L, n_streams;
    int* err;            // device flag word: bit 1 = an activation left the fp16-split range (|a| >= 6e4)
    unsigned long long* dbg;   // ADEC_KTRACE: {globaltimer at start, at end, SM cycles} of CTA 0, one record of KT_REC per launch
                               // (nullptr = off); ADEC_PHASES builds append the phase cycle counters of wg_conv_kernel
    // varlen (the VL kernels): vl_B utterances of different lengths, concatenated along time in x, res and y.  Utterance u's input rows
    // are [vl_in[u], vl_in[u + 1]) and its output rows [vl_out[u], vl_out[u + 1]) (B + 1 entries each); in the tiles' row space it owns
    // the stacked rows [vl_row(u), vl_row(u + 1)), vl_row(u) = vl_out[u] + u * (Ktaps - 1) * dil, as stack_L does for equal lengths.
    // Every utterance starts from zero history; T and Tout are the totals.
    const int* vl_in;
    const int* vl_out;
    int vl_B;
    // streaming varlen (stream slots): nullptr = offline (zero history, no state).  Otherwise utterance u is a chunk of stream slot
    // vl_slot[u] >> 1: its history rows come from that slot's rows of buffer (vl_slot[u] & 1 ? st_out : st_in) and its new state goes
    // to the same rows of the other buffer, so each slot keeps its own ping-pong phase and slots not in the call are not touched.
    const int* vl_slot;
};

// stream slots: the state rows of utterance u's slot that the call reads (rd = true) or writes; base = st_in / st_out of the args
template <typename T>
__device__ __forceinline__ T* slot_rows(const int* vl_slot, int u, const T* st_in, const T* st_out, long long per_slot, bool rd) {
    const int e = __ldg(vl_slot + u);
    const T* base = ((e & 1) != 0) == rd ? st_out : st_in;
    return const_cast<T*>(base) + (long long)(e >> 1) * per_slot;
}

// varlen row spaces: utterance u owns rows [off[u] + u * halo, off[u + 1] + (u + 1) * halo); off has B + 1 ascending entries
__device__ __forceinline__ int vl_row(const int* off, int halo, int u) { return __ldg(off + u) + u * halo; }
// the utterance that owns row j (the last one for rows past the end)
__device__ __forceinline__ int vl_find(const int* off, int halo, int B, int j) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (vl_row(off, halo, mid) <= j) lo = mid; else hi = mid - 1;
    }
    return lo;
}

constexpr int CONV_STAGES = 4;

template <int CW, int CO_TILE, int TT, int KC>
struct ConvCfg {
    static constexpr int NWC = (CO_TILE / 32) * (TT / 64);   // consumer warps (32 co x 64 t each)
    static constexpr int NTC = NWC * 32;
    static constexpr int NTHREADS = NTC + 32;                // + producer warp
    static constexpr int PITCH = CW + 4;                     // +4 floats: conflict-free float4 row reads
    static constexpr int CHUNK = KC * CO_TILE;               // floats per weight stage
    static constexpr size_t smem_bytes(int window_rows) {
        return 128 + sizeof(float) * ((size_t)CONV_STAGES * CHUNK + (size_t)window_rows * PITCH);
    }
};

template <int CO_TILE, int KC, int PITCH>
__device__ __forceinline__ void mma_chunk(float (&acc)[8][8], const float* __restrict__ xb, const float* __restrict__ wb) {
#pragma unroll 2
    for (int kk = 0; kk < KC; kk += 4) {
        float4 xv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) xv[j] = *reinterpret_cast<const float4*>(xb + j * 8 * PITCH + kk);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float4 wa = *reinterpret_cast<const float4*>(wb + (kk + q) * CO_TILE);
            const float4 wc = *reinterpret_cast<const float4*>(wb + (kk + q) * CO_TILE + 4);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float xq = q == 0 ? xv[j].x : q == 1 ? xv[j].y : q == 2 ? xv[j].z : xv[j].w;
                acc[j][0] = fmaf(xq, wa.x, acc[j][0]);
                acc[j][1] = fmaf(xq, wa.y, acc[j][1]);
                acc[j][2] = fmaf(xq, wa.z, acc[j][2]);
                acc[j][3] = fmaf(xq, wa.w, acc[j][3]);
                acc[j][4] = fmaf(xq, wc.x, acc[j][4]);
                acc[j][5] = fmaf(xq, wc.y, acc[j][5]);
                acc[j][6] = fmaf(xq, wc.z, acc[j][6]);
                acc[j][7] = fmaf(xq, wc.w, acc[j][7]);
            }
        }
    }
}

template <int CW, int CO_TILE, int TT, int KC, bool FUSE>
__global__ void __launch_bounds__(ConvCfg<CW, CO_TILE, TT, KC>::NTHREADS)
conv_gemm_kernel(const ConvArgs a) {
    using Cfg = ConvCfg<CW, CO_TILE, TT, KC>;
    constexpr int NWC = Cfg::NWC, NTC = Cfg::NTC, PITCH = Cfg::PITCH, CHUNK = Cfg::CHUNK;
    constexpr int CO_WARPS = CO_TILE / 32;
    static_assert(CW % KC == 0 && KC % 4 == 0, "bad KC");
    static_assert(!FUSE || CW == CO_TILE, "residual-unit fusion needs Cin == Cout == tile");

    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw);
    uint64_t* empty = full + CONV_STAGES;
    float* wst = reinterpret_cast<float*>(smem_raw + 128);
    float* xs = wst + CONV_STAGES * CHUNK;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int j0 = blockIdx.x * TT;                 // first output row of this tile
    const int g = blockIdx.y / a.n_co_tiles;
    const int co_tile = blockIdx.y - g * a.n_co_tiles;
    const int b = blockIdx.z;
    const int n1 = a.n_pieces * a.Ktaps * (CW / KC);     // weight chunks of GEMM 1
    const int ntot = n1 + (FUSE ? CO_TILE / KC : 0);

    if (tid == 0) {
        for (int s = 0; s < CONV_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], NWC);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == NWC) {
        // ------------------------------ producer warp: stream weight chunks L2 -> smem (TMA 1-D)
        if (lane == 0) {
            const float* w1 = a.w + (long long)blockIdx.y * a.w_tile_floats;
            for (int c = 0; c < ntot; ++c) {
                const int s = c % CONV_STAGES, it = c / CONV_STAGES;
                if (it > 0) mbar_wait(&empty[s], (it - 1) & 1);
                const float* src = (c < n1) ? w1 + (long long)c * CHUNK : a.w2 + (long long)(c - n1) * CHUNK;
                mbar_arrive_expect_tx(&full[s], CHUNK * 4);
                bulk_g2s(wst + s * CHUNK, src, CHUNK * 4, &full[s]);
            }
        }
        return;
    }

    // ---------------------------------- consumer warps
    const int warp_co = warp % CO_WARPS, warp_t = warp / CO_WARPS;
    const int cg = lane & 3, tg = lane >> 2;
    const int wrows = TT + (a.Ktaps - 1) * a.dil;   // window rows
    float acc[8][8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;

    const float* xg = a.x + (long long)b * a.x_bs + g * a.x_goff;
    const float* sg = a.st_in + (long long)b * a.P * a.st_ld + g * a.st_goff;
    int c = 0;
    for (int piece = 0; piece < a.n_pieces; ++piece) {
        if (piece > 0) named_bar_sync(1, NTC);
        // ---- window load: x~ rows -> smem, history from state, pre-activation applied once
        const int nvec = wrows * (CW / 4);
        for (int idx = tid; idx < nvec; idx += NTC) {
            const int m = idx / (CW / 4);
            const int c4 = idx - m * (CW / 4);
            const int q = piece * CW + c4 * 4;
            int r = 0, ci = q;
            if (a.RG > 1) { r = q >> a.lgCin; ci = q & (a.Cin - 1); }
            const long long i = (long long)(j0 + m) * a.RG + r;     // x~ row
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            long long t = i - a.P;
            if (a.hist_rep && t < 0) t = 0;
            if (t < 0) {
                v = *reinterpret_cast<const float4*>(sg + i * a.st_ld + ci);
            } else {
                if (t < a.T) {
                    v = __ldg(reinterpret_cast<const float4*>(xg + t * a.ldx + ci));
                    if (a.pre_act == ACT_NORM) {
                        const float4 mu = *reinterpret_cast<const float4*>(a.mean + ci);
                        const float4 sc = *reinterpret_cast<const float4*>(a.scale + ci);
                        v.x = __fdiv_rn(v.x - mu.x, sc.x); v.y = __fdiv_rn(v.y - mu.y, sc.y);
                        v.z = __fdiv_rn(v.z - mu.z, sc.z); v.w = __fdiv_rn(v.w - mu.w, sc.w);
                    } else {
                        v = apply_act(v, a.pre_act, a.slope);
                    }
                }
            }
            *reinterpret_cast<float4*>(xs + m * PITCH + c4 * 4) = v;
        }
        named_bar_sync(1, NTC);
        // ---- GEMM 1 over (tap, ci-chunk) of this piece
        for (int tap = 0; tap < a.Ktaps; ++tap) {
            const float* xrow = xs + (warp_t * 64 + tg + tap * a.dil) * PITCH;
            for (int kc0 = 0; kc0 < CW; kc0 += KC, ++c) {
                const int s = c % CONV_STAGES;
                mbar_wait(&full[s], (c / CONV_STAGES) & 1);
                mma_chunk<CO_TILE, KC, PITCH>(acc, xrow + kc0, wst + s * CHUNK + warp_co * 32 + cg * 8);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
            }
        }
    }

    if (FUSE) {
        // ---- residual unit: mid = act(conv_k7(act(x))) stays in smem, then the 1x1 conv
        named_bar_sync(1, NTC);     // everyone is done reading the window
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float* mrow = xs + (warp_t * 64 + tg + 8 * j) * PITCH + warp_co * 32 + cg * 8;
            float4 v0 = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
            float4 v1 = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
            *reinterpret_cast<float4*>(mrow) = apply_act(v0, a.mid_act, a.slope);
            *reinterpret_cast<float4*>(mrow + 4) = apply_act(v1, a.mid_act, a.slope);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
        }
        named_bar_sync(1, NTC);
        const float* xrow = xs + (warp_t * 64 + tg) * PITCH;
        for (int kc0 = 0; kc0 < CO_TILE; kc0 += KC, ++c) {
            const int s = c % CONV_STAGES;
            mbar_wait(&full[s], (c / CONV_STAGES) & 1);
            mma_chunk<CO_TILE, KC, PITCH>(acc, xrow + kc0, wst + s * CHUNK + warp_co * 32 + cg * 8);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
    }

    // ---------------------------------- epilogue: bias, residual, store
    {
        const int co_l = co_tile * CO_TILE + warp_co * 32 + cg * 8;   // channel within the group
        float bv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) bv[i] = a.bias ? a.bias[g * a.Cout_g + co_l + i] : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int t = j0 + warp_t * 64 + tg + 8 * j;
            if (t >= a.Tout) continue;
            float o[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = acc[j][i] + bv[i];
            if (a.res) {
                const float* rp = a.res + (long long)b * a.res_bs + (long long)t * a.ldr + g * a.r_goff + co_l;
                const float4 r0 = __ldg(reinterpret_cast<const float4*>(rp));
                const float4 r1 = __ldg(reinterpret_cast<const float4*>(rp + 4));
                // x + y  (residual_unit.py:81: `return x + y`)
                o[0] = r0.x + o[0]; o[1] = r0.y + o[1]; o[2] = r0.z + o[2]; o[3] = r0.w + o[3];
                o[4] = r1.x + o[4]; o[5] = r1.y + o[5]; o[6] = r1.z + o[6]; o[7] = r1.w + o[7];
            }
            if (a.out_nct) {
                float* yp = a.y + (long long)b * a.y_bs + (long long)(g * a.y_goff + co_l) * a.Tout + t;
#pragma unroll
                for (int i = 0; i < 8; ++i) yp[(long long)i * a.Tout] = o[i];
            } else {
                float* yp = a.y + (long long)b * a.y_bs + (long long)t * a.ldy + g * a.y_goff + co_l;
                *reinterpret_cast<float4*>(yp) = make_float4(o[0], o[1], o[2], o[3]);
                *reinterpret_cast<float4*>(yp + 4) = make_float4(o[4], o[5], o[6], o[7]);
            }
        }
    }

    // ---------------------------------- new causal state = last P rows of x~ (conv_layer.py:155)
    if (blockIdx.x == gridDim.x - 1 && co_tile == 0 && g < a.st_groups && a.P > 0) {
        float* so = a.st_out + (long long)b * a.P * a.st_ld + g * a.st_goff;
        const int nvec = a.P * (a.Cin / 4);
        for (int idx = tid; idx < nvec; idx += NTC) {
            const int r = idx / (a.Cin / 4);
            const int ci = (idx - r * (a.Cin / 4)) * 4;
            const long long i = (long long)a.T + r;      // x~ row
            float4 v;
            if (i < a.P) {
                v = *reinterpret_cast<const float4*>(sg + i * a.st_ld + ci);
            } else {
                v = __ldg(reinterpret_cast<const float4*>(xg + (i - a.P) * a.ldx + ci));
                if (a.pre_act == ACT_NORM) {
                    const float4 mu = *reinterpret_cast<const float4*>(a.mean + ci);
                    const float4 sc = *reinterpret_cast<const float4*>(a.scale + ci);
                    v.x = __fdiv_rn(v.x - mu.x, sc.x); v.y = __fdiv_rn(v.y - mu.y, sc.y);
                    v.z = __fdiv_rn(v.z - mu.z, sc.z); v.w = __fdiv_rn(v.w - mu.w, sc.w);
                } else {
                    v = apply_act(v, a.pre_act, a.slope);
                }
            }
            *reinterpret_cast<float4*>(so + (long long)r * a.st_ld + ci) = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// stem: Cin = 1 -> COUT, K taps, stride 1 (encoder.py:106-111).  x (B,T) -> y (B,T,COUT).
// ------------------------------------------------------------------------------------------------
struct StemArgs {
    const float* x; long long x_bs;
    const float* st_in; float* st_out;   // (B, K-1)
    int T;
    const float* w;                      // [K][COUT]
    const float* bias;                   // [COUT] or nullptr
    float* y; long long y_bs;
    const int* vl_off; int vl_B;         // VL: utterance u is rows [vl_off[u], vl_off[u + 1]) of x and y (B = 1, T = the total)
    const int* vl_slot;                  // VL: stream slots (ConvArgs::vl_slot), or nullptr
};

// VL: one row space of concatenated utterances, each with a zero left pad and no state written; with vl_slot, each with its slot's
// history, and the slot's new state written by the block that holds the utterance's last row.
// BST: bf16 x, state and output (the encoder-only handle's compute_dtype 2); weights, bias and the FMA chain stay fp32, each output
// is rounded once to nearest even, and the state holds the input samples as they are.
template <int COUT, int K, bool VL = false, bool BST = false>
__global__ void __launch_bounds__(256) stem_kernel(const StemArgs a) {
    using XT = typename std::conditional<BST, __nv_bfloat16, float>::type;
    constexpr int TT = 1024, P = K - 1, Q = COUT / 4;
    __shared__ float xw[TT + P];
    __shared__ __align__(16) float sw[K * COUT];
    __shared__ __align__(16) float sb[COUT];
    const int b = blockIdx.y, j0 = blockIdx.x * TT, tid = threadIdx.x;
    const XT* xg = reinterpret_cast<const XT*>(a.x) + (long long)b * a.x_bs;
    const XT* st_in = reinterpret_cast<const XT*>(a.st_in);
    XT* st_out = reinterpret_cast<XT*>(a.st_out);
    auto widen = [](XT v) -> float {
        if constexpr (BST) return __bfloat162float(v);
        else return v;
    };
    for (int i = tid; i < TT + P; i += 256) {
        const long long r = (long long)j0 + i;       // x~ row
        float v = 0.f;
        if (r < P) { if (!VL) v = widen(st_in[b * P + r]); }
        else if (r - P < a.T) v = widen(__ldg(xg + r - P));
        xw[i] = v;
    }
    for (int i = tid; i < K * COUT; i += 256) sw[i] = a.w[i];
    for (int i = tid; i < COUT; i += 256) sb[i] = a.bias ? a.bias[i] : 0.f;
    __syncthreads();
    const int q = tid % Q, tl = tid / Q;
    constexpr int TSTEP = 256 / Q;
    float* yg = a.y + (long long)b * a.y_bs;
    int u = 0, u_start = 0, u_next = 0;              // VL: the utterance of row j0 + t, its first row, the next one's first row
    if (VL && j0 + tl < a.T) {
        u = vl_find(a.vl_off, 0, a.vl_B, j0 + tl);
        u_start = __ldg(a.vl_off + u);
        u_next = __ldg(a.vl_off + u + 1);
    }
    for (int t = tl; t < TT; t += TSTEP) {
        if (j0 + t >= a.T) break;
        if (VL) while (j0 + t >= u_next) { ++u; u_start = u_next; u_next = __ldg(a.vl_off + u + 1); }
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        auto tap = [&](int k, float xv) {
            const float4 w4 = *reinterpret_cast<const float4*>(sw + k * COUT + q * 4);
            acc.x = fmaf(xv, w4.x, acc.x); acc.y = fmaf(xv, w4.y, acc.y);
            acc.z = fmaf(xv, w4.z, acc.z); acc.w = fmaf(xv, w4.w, acc.w);
        };
        if (VL && a.vl_slot && j0 + t - u_start < P) {
            // the first P rows of a stream-slot utterance: taps before it read the slot's history
            const XT* hs = slot_rows(a.vl_slot, u, st_in, st_out, P, true);
            for (int k = 0; k < K; ++k) tap(k, j0 + t + k - P < u_start ? widen(__ldg(hs + (j0 + t + k - u_start))) : xw[t + k]);
        } else {
#pragma unroll
            for (int k = 0; k < K; ++k) tap(k, (!VL || j0 + t + k - P >= u_start) ? xw[t + k] : 0.f);   // taps before the utterance: its zero pad
        }
        const float4 b4 = *reinterpret_cast<const float4*>(sb + q * 4);
        acc.x += b4.x; acc.y += b4.y; acc.z += b4.z; acc.w += b4.w;
        if constexpr (BST) st4(reinterpret_cast<__nv_bfloat16*>(a.y) + (long long)b * a.y_bs + (long long)(j0 + t) * COUT + q * 4, acc);
        else *reinterpret_cast<float4*>(yg + (long long)(j0 + t) * COUT + q * 4) = acc;
    }
    if (!VL && blockIdx.x == gridDim.x - 1) {
        for (int r = tid; r < P; r += 256) {
            const long long i = (long long)a.T + r;
            st_out[b * P + r] = (i < P) ? st_in[b * P + i] : xg[i - P];
        }
    }
    if (VL && a.vl_slot) {
        // (utterance, state row) pairs of the utterances whose last row lies in this block: rows [T_u, T_u + P) of slot history || chunk
        const int u_first = vl_find(a.vl_off, 0, a.vl_B, j0);
        for (int idx = tid;; idx += 256) {
            const int u = u_first + idx / P, r = idx % P;
            if (u >= a.vl_B || __ldg(a.vl_off + u) >= j0 + TT) break;
            const int s0 = __ldg(a.vl_off + u), s1 = __ldg(a.vl_off + u + 1);
            if (s1 - 1 < j0 || s1 - 1 >= j0 + TT) continue;
            const int i = s1 - s0 + r;
            const XT v = i < P ? __ldg(slot_rows(a.vl_slot, u, st_in, st_out, P, true) + i) : __ldg(xg + s0 + i - P);
            slot_rows(a.vl_slot, u, st_in, st_out, P, false)[r] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// head: CIN -> 1, K taps (decoder.py:133 / HiFiGAN.py:118-123, :294-296).  x (B,T,CIN) -> y (B,T).
// ------------------------------------------------------------------------------------------------
struct HeadArgs {
    const float* x; long long x_bs; int ldx;
    const float* st_in; float* st_out;   // (B, K-1, CIN)
    int T;
    const float* w;                      // [K][CIN]
    float bias; int pre_act; float slope; int post_tanh;
    float* y; long long y_bs;
    const int* vl_off; int vl_B;         // VL: utterance u is rows [vl_off[u], vl_off[u + 1]) of x and y (B = 1, T = the total)
    const int* vl_slot;                  // VL: stream slots (ConvArgs::vl_slot), or nullptr
};

// Eight lanes share one run of R = 8 consecutive outputs: lane c4 owns channels 4*c4..4*c4+3, loads the R + K - 1 window rows of its
// channel quad straight from global (a row is one coalesced 128-byte segment across the eight lanes; no shared memory, every input row
// is read 14/8 times from L1), applies the pre-activation in registers and accumulates its 4-channel share of the R dot products with
// the K x 4 weights it keeps in registers; three xor-shuffles add the eight shares and lane j stores output j.  The layer moves
// 128 B per output row and does 2*K*CIN flops on it: memory-bound once the LDS traffic of the round-1 version (112 LDS.128 per output)
// is gone.  BST: bf16 input, state and output (the vocoder's bf16-activation mode); a chunk row enters the window as the bf16 value the
// state keeps of it, so that a streamed chunk and a one-shot call see the same window.  VL: concatenated utterances, each with a zero
// left pad (a run of eight outputs may span several of them, so each output masks the taps that fall before its utterance); with
// vl_slot, those taps read the utterance's slot history instead, and the block holding its last row writes the slot's new state.
template <int CIN, int K, bool BST, bool VL = false>
__global__ void __launch_bounds__(256) head_kernel(const HeadArgs a) {
    static_assert(CIN == 32, "eight lanes x four channels");
    using XT = typename std::conditional<BST, __nv_bfloat16, float>::type;
    constexpr int R = 8, P = K - 1, TT = 256;
    const int b = blockIdx.y, tid = threadIdx.x, c4 = tid & 7;
    const int t0 = blockIdx.x * TT + (tid >> 3) * R;               // first output of this lane group
    const XT* xg = reinterpret_cast<const XT*>(a.x) + (long long)b * a.x_bs;
    const XT* sg = reinterpret_cast<const XT*>(a.st_in) + (long long)b * P * CIN;
    float4 w[K];
#pragma unroll
    for (int k = 0; k < K; ++k) w[k] = __ldg(reinterpret_cast<const float4*>(a.w + k * CIN) + c4);
    float acc[R];
#pragma unroll
    for (int j = 0; j < R; ++j) acc[j] = 0.f;
    if (t0 < a.T) {
        float4 xv[R + P];
#pragma unroll
        for (int r = 0; r < R + P; ++r) {
            const long long i = (long long)t0 + r;                  // x~ row = history(P) || chunk
            xv[r] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < P) { if (!VL) xv[r] = ldg4(sg + i * CIN + 4 * c4); }   // state rows are stored post-activation
            else if (i - P < a.T) xv[r] = stored4<BST>(apply_act(ldg4(xg + (i - P) * a.ldx + 4 * c4), a.pre_act, a.slope));
        }
        int u = 0, u_start = 0, u_next = 0;
        if (VL) {
            u = vl_find(a.vl_off, 0, a.vl_B, t0);
            u_start = __ldg(a.vl_off + u);
            u_next = __ldg(a.vl_off + u + 1);
        }
#pragma unroll
        for (int j = 0; j < R; ++j) {
            if (VL) while (u + 1 < a.vl_B && t0 + j >= u_next) { ++u; u_start = u_next; u_next = __ldg(a.vl_off + u + 1); }
#pragma unroll
            for (int k = 0; k < K; ++k) {
                float4 x = xv[j + k];
                if (VL && t0 + j + k - P < u_start)
                    x = a.vl_slot ? ldg4(slot_rows(a.vl_slot, u, reinterpret_cast<const XT*>(a.st_in), reinterpret_cast<XT*>(a.st_out), P * CIN, true) +
                                         (t0 + j + k - u_start) * CIN + 4 * c4)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
                acc[j] = fmaf(x.x, w[k].x, acc[j]); acc[j] = fmaf(x.y, w[k].y, acc[j]);
                acc[j] = fmaf(x.z, w[k].z, acc[j]); acc[j] = fmaf(x.w, w[k].w, acc[j]);
            }
        }
    }
    float mine = 0.f;
#pragma unroll
    for (int j = 0; j < R; ++j) {
        float v = acc[j];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        if (j == c4) mine = v;
    }
    if (t0 + c4 < a.T) {
        mine += a.bias;
        if (a.post_tanh) mine = tanhf(mine);
        st1(reinterpret_cast<XT*>(a.y) + (long long)b * a.y_bs + t0 + c4, mine);
    }
    if (!VL && blockIdx.x == gridDim.x - 1) {
        XT* so = reinterpret_cast<XT*>(a.st_out) + (long long)b * P * CIN;
        for (int idx = tid; idx < P * (CIN / 4); idx += 256) {
            const int r = idx / (CIN / 4), ci = (idx - r * (CIN / 4)) * 4;
            const long long i = (long long)a.T + r;
            float4 v;
            if (i < P) v = ld4(sg + i * CIN + ci);
            else v = apply_act(ldg4(xg + (i - P) * a.ldx + ci), a.pre_act, a.slope);
            st4(so + r * CIN + ci, v);
        }
    }
    if (VL && a.vl_slot) {
        // the slot state of every utterance whose last row lies in this block: rows [T_u, T_u + P) of slot history || chunk
        const int r0 = blockIdx.x * TT;
        for (int u = vl_find(a.vl_off, 0, a.vl_B, r0); u < a.vl_B && __ldg(a.vl_off + u) < r0 + TT; ++u) {
            const int s0 = __ldg(a.vl_off + u), s1 = __ldg(a.vl_off + u + 1);
            if (s1 - 1 < r0 || s1 - 1 >= r0 + TT) continue;
            const XT* so_rd = slot_rows(a.vl_slot, u, reinterpret_cast<const XT*>(a.st_in), reinterpret_cast<XT*>(a.st_out), P * CIN, true);
            XT* so_wr = slot_rows(a.vl_slot, u, reinterpret_cast<const XT*>(a.st_in), reinterpret_cast<XT*>(a.st_out), P * CIN, false);
            for (int idx = tid; idx < P * (CIN / 4); idx += 256) {
                const int r = idx / (CIN / 4), ci = (idx - r * (CIN / 4)) * 4;
                const int i = s1 - s0 + r;
                float4 v;
                if (i < P) v = ldg4(so_rd + i * CIN + ci);
                else v = apply_act(ldg4(xg + (long long)(s0 + i - P) * a.ldx + ci), a.pre_act, a.slope);
                st4(so_wr + r * CIN + ci, v);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// residual VQ (layers/vq_module.py:90-104,136-149).  Rounding order == oracle/rvq_oracle.c.
// ------------------------------------------------------------------------------------------------
struct RvqArgs {
    const float* z;        // (B, D, F) channels-first (what encode() returns)
    int B, F, nq;
    const float* embed;    // (nq, D, N) = state-dict `embed` tensors stacked
    const float* e2;       // (nq, N)   ||e||^2 in torch's summation order
    long long* idx;        // (nq, B, F) flat indices (+ N*i), or nullptr
    // fused outputs (SURVEY.md 8(f) rank 2; bin/stream.py:224 hand-off): either may be nullptr
    unsigned char* packed; // (B*F, bpf) index bitstream, same format as pack_kernel
    float* zq;             // (B*F, D) = lookup(idx) (vq_module.py:159-161), so that quantize can hand zq straight to the decoder;
                           //          with FWD the forward sum instead
    int bits, bpf, n_pass; // bits per index, bytes per packed frame, frame passes per block (frames per block = n_pass * FP)
};

constexpr int RVQ_THREADS = 256;

// One block quantises n_pass * FP frames through all nq stages.  Thread t owns codewords t, t + 256, ... (NPT of them) for FP frames
// at a time: FP * NPT independent fused-multiply-add chains over k (ascending, one chain per distance: MKL's sgemm order, which is
// what makes the indices bit-identical to torch-CPU), codeword elements streamed from L2 (the 256 KB stage table is shared by all
// blocks), residuals broadcast from shared memory.  The host picks (FP, n_pass) so that the grid is one wave with the least idle
// tail (adec_quantize), which alone took the 64 x 160-frame case from 0.58 ms (320 blocks of 32 frames = 1.08 waves) to one wave.
// FWD: zq accumulates ResidualVQ.forward's quantized_out, the sum of r + (e - r) from 0. (vq_module.py:136-143), instead of
// lookup's sum of the codewords; shared memory, grid and every other output are the same.
// ZB: z is bf16 (raw words, the encoder-only handle's compute_dtype 2), widened exactly to fp32 on load; the arithmetic after the
// load is the fp32 instantiation's, so the outputs are the spec applied to float(z).
template <int D, int NPT, int FP, bool FWD, bool ZB = false>   // codebook size N = RVQ_THREADS * NPT
__global__ void __launch_bounds__(RVQ_THREADS) rvq_kernel(const RvqArgs a) {
    constexpr int N = RVQ_THREADS * NPT, NW = RVQ_THREADS / 32;
    static_assert(D % 32 == 0 && FP % 4 == 0, "D must be a multiple of 32, FP of 4");
    extern __shared__ __align__(16) float rvq_smem[];
    const int FR = a.n_pass * FP;
    float* r = rvq_smem;                               // [FR][D] residuals
    float* zq = r + FR * D;                            // [FR][D] sum of the chosen codewords
    float* r2 = zq + FR * D;                           // [FR][D] 2 * residual (exact): the multiplicand of the distance GEMM, kept so that the
                                                       //         inner loop is FFMA + one broadcast LDS.128 per 16 of them (was + 4 FMUL)
    float* x2 = r2 + FR * D;                           // [FR]
    float* wv = x2 + FR;                               // [FR][NW]
    int* wi = reinterpret_cast<int*>(wv + FR * NW);    // [FR][NW]
    int* best = wi + FR * NW;                          // [nq][FR] local indices of every stage (for the packed frame)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long nfr = (long long)a.B * a.F;
    const long long f0 = (long long)blockIdx.x * FR;
    for (int i = tid; i < FR * D; i += RVQ_THREADS) {
        const int f = i % FR, k = i / FR;            // consecutive threads -> consecutive frames: coalesced reads of z (B,D,F)
        const long long fr = f0 + f;
        float v = 0.f;
        if (fr < nfr) {
            const long long bb = fr / a.F, ff = fr - bb * a.F;
            if constexpr (ZB) v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a.z)[(bb * D + k) * a.F + ff]);
            else v = a.z[(bb * D + k) * a.F + ff];  // quantizer.py:43 z.transpose(2,1)
        }
        r[f * D + k] = v;
        r2[f * D + k] = 2.0f * v;
        zq[f * D + k] = 0.f;
    }
    __syncthreads();
    for (int st = 0; st < a.nq; ++st) {
        const float* E = a.embed + (long long)st * D * N;
        // x2 = flatten.pow(2).sum(1): 8-lane vectors, 4 interleaved accumulators, sequential horizontal add
        for (int f = tid; f < FR; f += RVQ_THREADS) {
            float accv[4][8];
#pragma unroll
            for (int v = 0; v < 4; ++v)
#pragma unroll
                for (int l = 0; l < 8; ++l) accv[v][l] = 0.f;
#pragma unroll
            for (int v = 0; v < D / 8; ++v)
#pragma unroll
                for (int l = 0; l < 8; ++l) {
                    const float xv = r[f * D + 8 * v + l];
                    accv[v & 3][l] = __fadd_rn(accv[v & 3][l], __fmul_rn(xv, xv));
                }
            float s = 0.f;
#pragma unroll
            for (int l = 0; l < 8; ++l) {
                const float t = __fadd_rn(__fadd_rn(__fadd_rn(accv[0][l], accv[1][l]), accv[2][l]), accv[3][l]);
                s = (l == 0) ? t : __fadd_rn(s, t);
            }
            x2[f] = s;
        }
        float e2v[NPT];
#pragma unroll
        for (int m = 0; m < NPT; ++m) e2v[m] = __ldg(a.e2 + (long long)st * N + tid + m * RVQ_THREADS);
        __syncthreads();   // x2 visible
        // dot2[c] = sum_k (2 r_k) * E[k][c], k ascending, one fused multiply-add chain per output (MKL sgemm order)
#pragma unroll 1
        for (int fh = 0; fh < FR; fh += FP) {
            float acc[FP][NPT];
#pragma unroll
            for (int f = 0; f < FP; ++f)
#pragma unroll
                for (int m = 0; m < NPT; ++m) acc[f][m] = 0.f;
            float e[4][NPT], en[4][NPT];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                for (int m = 0; m < NPT; ++m) e[kk][m] = __ldg(E + (long long)kk * N + tid + m * RVQ_THREADS);
#pragma unroll 1
            for (int k = 0; k < D; k += 4) {
                const int kn = k + 4 < D ? k + 4 : k;            // prefetch the next four codeword rows while these are used
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                    for (int m = 0; m < NPT; ++m) en[kk][m] = __ldg(E + (long long)(kn + kk) * N + tid + m * RVQ_THREADS);
#pragma unroll
                for (int f = 0; f < FP; ++f) {
                    const float4 r4 = *reinterpret_cast<const float4*>(&r2[(fh + f) * D + k]);
                    const float rk[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                        for (int m = 0; m < NPT; ++m) acc[f][m] = fmaf(rk[kk], e[kk][m], acc[f][m]);
                }
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                    for (int m = 0; m < NPT; ++m) e[kk][m] = en[kk][m];
            }
#pragma unroll
            for (int f = 0; f < FP; ++f) {
                // dist = (x2 - dot2) + e2 ; index = first arg-max of -dist  (vq_module.py:93-98)
                float bv = 0.f;
                int bi = 0;
#pragma unroll
                for (int m = 0; m < NPT; ++m) {
                    const float nd = -__fadd_rn(__fsub_rn(x2[fh + f], acc[f][m]), e2v[m]);
                    if (m == 0 || nd > bv) { bv = nd; bi = tid + m * RVQ_THREADS; }
                }
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) {
                    const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
                }
                if (lane == 0) { wv[(fh + f) * NW + warp] = bv; wi[(fh + f) * NW + warp] = bi; }
            }
        }
        __syncthreads();
        for (int f = tid; f < FR; f += RVQ_THREADS) {
            float bv = wv[f * NW];
            int bi = wi[f * NW];
#pragma unroll
            for (int w = 1; w < NW; ++w) {
                const float ov = wv[f * NW + w];
                const int oi = wi[f * NW + w];
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            best[st * FR + f] = bi;
            const long long fr = f0 + f;
            if (a.idx && fr < nfr) a.idx[(long long)st * nfr + fr] = (long long)bi + (long long)N * st;   // vq_module.py:145-146
        }
        __syncthreads();
        // quantize = x + (e - x); residual -= quantize  (vq_module.py:101-102,143); zq += e in stage order (vq_module.py:159-161)
        for (int i = tid; i < FR * D; i += RVQ_THREADS) {
            const int f = i / D, k = i - f * D;
            const float rv = r[i];
            const float q = __ldg(E + (long long)k * N + best[st * FR + f]);
            const float qq = __fadd_rn(rv, __fsub_rn(q, rv));
            const float rn = __fsub_rn(rv, qq);
            r[i] = rn;
            r2[i] = 2.0f * rn;
            if (FWD) zq[i] = __fadd_rn(zq[i], qq);                 // stage 0 adds to the 0.f stored above: a -0 comes out +0
            else zq[i] = st == 0 ? q : __fadd_rn(zq[i], q);
        }
        __syncthreads();
    }
    if (a.zq) {
        for (int i = tid; i < FR * D / 4; i += RVQ_THREADS) {
            const long long fr = f0 + (i * 4) / D;
            if (fr < nfr) *reinterpret_cast<float4*>(a.zq + f0 * D + (long long)i * 4) = *reinterpret_cast<const float4*>(zq + i * 4);
        }
    }
    if (a.packed) {
        // packed frame: nq local indices of `bits` bits each, stage 0 first, little-endian bit order (same bytes as pack_kernel)
        for (int f = tid; f < FR; f += RVQ_THREADS) {
            const long long fr = f0 + f;
            if (fr >= nfr) continue;
            unsigned char* o = a.packed + fr * a.bpf;
            unsigned long long accb = 0;
            int nb = 0, ob = 0;
            for (int i = 0; i < a.nq; ++i) {
                accb |= (unsigned long long)best[i * FR + f] << nb;
                nb += a.bits;
                while (nb >= 8) { o[ob++] = (unsigned char)(accb & 0xffu); accb >>= 8; nb -= 8; }
            }
            if (nb > 0) o[ob++] = (unsigned char)(accb & 0xffu);
        }
    }
}

// codebook lookup (vq_module.py:159-161): zq[b][f][:] = sum_i codebook[idx[i][b][f]][:], i ascending.  The indices come either as the
// int64 (nq, B*F) tensor of the reference or straight from the packed bitstream (unpack fused into the lookup).
struct LookupArgs {
    const long long* idx;   // (nq, B*F) or nullptr
    const unsigned char* packed;   // (B*F, bpf) or nullptr
    long long nfr;
    int nq, D, N, bits, bpf;
    const float* codebook;  // (nq*N, D)
    long long n_rows;       // nq*N (bounds check)
    float* zq;              // (B*F, D)
    int* err;               // bit 0 set on an out-of-range index
};

// BF16: zq is bf16 words, each value the fp32 sum rounded once to nearest even, so it equals torch's .to(torch.bfloat16) of the fp32
// zq (the input of a decoder with bf16 activations); D % 8 == 0 keeps its rows 16-byte aligned.
template <bool BF16>
__global__ void __launch_bounds__(256) lookup_kernel(const LookupArgs a) {
    const int vpf = a.D / 4;    // float4 per frame
    const long long gid = (long long)blockIdx.x * 256 + threadIdx.x;
    if (gid >= a.nfr * vpf) return;
    const long long fr = gid / vpf;
    const int k4 = (int)(gid - fr * vpf) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    const unsigned char* in = a.packed ? a.packed + fr * a.bpf : nullptr;
    const unsigned long long mask = (1ull << a.bits) - 1ull;
    unsigned long long accb = 0;
    int nb = 0, ib = 0;
    for (int i = 0; i < a.nq; ++i) {
        long long row;
        if (in) {
            while (nb < a.bits) { accb |= (unsigned long long)in[ib++] << nb; nb += 8; }
            const long long v = (long long)(accb & mask);
            accb >>= a.bits; nb -= a.bits;
            row = v < a.N ? v + (long long)i * a.N : -1;
        } else {
            row = a.idx[(long long)i * a.nfr + fr];
        }
        if (row < 0 || row >= a.n_rows) { atomicOr(a.err, 1); continue; }
        const float4 v = __ldg(reinterpret_cast<const float4*>(a.codebook + row * a.D + k4));
        if (i == 0) s = v;
        else { s.x = __fadd_rn(s.x, v.x); s.y = __fadd_rn(s.y, v.y); s.z = __fadd_rn(s.z, v.z); s.w = __fadd_rn(s.w, v.w); }
    }
    if constexpr (BF16)
        *reinterpret_cast<uint2*>(reinterpret_cast<uint16_t*>(a.zq) + fr * a.D + k4) = make_uint2(bf2_bits(s.x, s.y), bf2_bits(s.z, s.w));
    else
        *reinterpret_cast<float4*>(a.zq + fr * a.D + k4) = s;
}

// Per-utterance moments of the quantizer output (codecStatistic.py:104-105 calls StandardScaler.partial_fit once per file), fp64
// throughout (fp32 values widen exactly).  Over utterance b's rows [off[b], off[b + 1]) of zq (rows, 64) channels-last:
//   CENTRED = false:  sum[b][c] = sum_f x
//   CENTRED = true:   with T = sum[b][c] / n,  m2[b][c] = sum_f (x - T)^2 - (sum_f (x - T))^2 / n   (sklearn's corrected two-pass term)
// One block per utterance.  Its rows are cut into segments of MOM_SEG rows counted from the utterance's first row; thread (j, q) adds
// rows j, j + 16, ... of a segment for channels 4q .. 4q + 3 in ascending order, the 16 row partials of a segment are added in row
// order, and the segment totals in segment order.  No atomics: an utterance's result depends on its own rows only, not on where it
// sits in the batch or what surrounds it.
constexpr int MOM_THREADS = 256, MOM_D = 64, MOM_Q = MOM_D / 4, MOM_ROWS = MOM_THREADS / MOM_Q, MOM_SEG = 256;

struct MomArgs {
    const float* zq;   // (off[B], 64), 16-byte aligned
    const int* off;    // (B + 1) row offsets
    double* sum;       // (B, 64): written by the first launch, read by the second
    double* m2;        // (B, 64)
};

template <bool CENTRED>
__global__ void __launch_bounds__(MOM_THREADS) zq_moments_kernel(const MomArgs a) {
    __shared__ double part[CENTRED ? 2 : 1][MOM_ROWS][MOM_D];
    const int b = blockIdx.x, tid = threadIdx.x, q = tid % MOM_Q, j = tid / MOM_Q;
    const int r0 = __ldg(a.off + b), n = __ldg(a.off + b + 1) - r0;
    const float* x = a.zq + (long long)r0 * MOM_D + 4 * q;
    double t[4] = {0.0, 0.0, 0.0, 0.0};
    if (CENTRED)
#pragma unroll
        for (int k = 0; k < 4; ++k) t[k] = a.sum[(long long)b * MOM_D + 4 * q + k] / (double)n;
    double tot1 = 0.0, tot2 = 0.0;            // threads c < 64: the running totals of channel c
    for (int s0 = 0; s0 < n; s0 += MOM_SEG) {
        double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int i = 0; i < MOM_SEG / MOM_ROWS; ++i) {
            const int f = s0 + j + i * MOM_ROWS;
            if (f < n) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(x + (long long)f * MOM_D));
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (CENTRED) {
                        const double d = __dsub_rn((double)vv[k], t[k]);
                        s1[k] = __dadd_rn(s1[k], d);
                        s2[k] = __dadd_rn(s2[k], __dmul_rn(d, d));     // the square rounded, then added (numpy's temp **= 2; sum)
                    } else {
                        s1[k] = __dadd_rn(s1[k], (double)vv[k]);
                    }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            part[0][j][4 * q + k] = s1[k];
            if (CENTRED) part[CENTRED ? 1 : 0][j][4 * q + k] = s2[k];
        }
        __syncthreads();
        if (tid < MOM_D) {
            double p1 = part[0][0][tid], p2 = CENTRED ? part[CENTRED ? 1 : 0][0][tid] : 0.0;
            for (int r = 1; r < MOM_ROWS; ++r) {
                p1 = __dadd_rn(p1, part[0][r][tid]);
                if (CENTRED) p2 = __dadd_rn(p2, part[CENTRED ? 1 : 0][r][tid]);
            }
            tot1 = __dadd_rn(tot1, p1);
            tot2 = __dadd_rn(tot2, p2);
        }
        __syncthreads();
    }
    if (tid < MOM_D) {
        if (CENTRED) a.m2[(long long)b * MOM_D + tid] = __dsub_rn(tot2, __ddiv_rn(__dmul_rn(tot1, tot1), (double)n));
        else a.sum[(long long)b * MOM_D + tid] = tot1;
    }
}

// Index bitstream (SURVEY.md 8(f) rank 2).  The reference has no wire format: it ships int64 (Nq,F) tensors through a queue
// (bin/stream.py:224).  Packed frame = Nq local indices (idx - i*N) of `bits` = ceil(log2 N) bits each, stage 0 first, little-endian
// bit order, zero-padded to whole bytes: 8 x 10 bit = 10 bytes per frame.  One thread per frame (a frame is 10-20 bytes).
struct PackArgs {
    long long* idx;           // (nq, nfr) flat indices (+N*i), read by pack / written by unpack
    unsigned char* packed;    // (nfr, bpf)
    long long nfr;
    int nq, N, bits, bpf;
    int* err;                 // set to 1 on an out-of-range index / code
};

__global__ void __launch_bounds__(256) pack_kernel(const PackArgs a) {
    const long long fr = (long long)blockIdx.x * 256 + threadIdx.x;
    if (fr >= a.nfr) return;
    unsigned char* o = a.packed + fr * a.bpf;
    unsigned long long acc = 0;
    int nb = 0, ob = 0;
    for (int i = 0; i < a.nq; ++i) {
        long long v = a.idx[(long long)i * a.nfr + fr] - (long long)i * a.N;
        if (v < 0 || v >= a.N) { atomicOr(a.err, 1); v = 0; }
        acc |= (unsigned long long)v << nb;
        nb += a.bits;
        while (nb >= 8) { o[ob++] = (unsigned char)(acc & 0xffu); acc >>= 8; nb -= 8; }
    }
    if (nb > 0) o[ob++] = (unsigned char)(acc & 0xffu);
}

__global__ void __launch_bounds__(256) unpack_kernel(const PackArgs a) {
    const long long fr = (long long)blockIdx.x * 256 + threadIdx.x;
    if (fr >= a.nfr) return;
    const unsigned char* in = a.packed + fr * a.bpf;
    const unsigned long long mask = (1ull << a.bits) - 1ull;
    unsigned long long acc = 0;
    int nb = 0, ib = 0;
    for (int i = 0; i < a.nq; ++i) {
        while (nb < a.bits) { acc |= (unsigned long long)in[ib++] << nb; nb += 8; }
        long long v = (long long)(acc & mask);
        acc >>= a.bits; nb -= a.bits;
        if (v >= a.N) { atomicOr(a.err, 1); v = 0; }
        a.idx[(long long)i * a.nfr + fr] = v + (long long)i * a.N;
    }
}

// per-stream state copies between stream slots (adec_copy_stream_state, and putting every stream back into the op's current buffer):
// pair j copies the `per` words of stream pairs[2j] in src to stream pairs[2j + 1] in dst
__global__ void slot_copy_kernel(float* dst, const float* src, long long per, const int* pairs, int n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= per * n) return;
    const int j = (int)(i / per);
    const long long w = i - (long long)j * per;
    dst[(long long)__ldg(pairs + 2 * j + 1) * per + w] = src[(long long)__ldg(pairs + 2 * j) * per + w];
}

// replicate stream 0's state to all streams (adec_set_streams)
__global__ void replicate_kernel(float* dst, const float* src, long long per_stream, int n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < per_stream * n) dst[i] = src[i % per_stream];
}

// ---- stream state export / import (adec_get_stream_state / adec_set_stream_state) ----------------------------------------------------
// One entry of the handle's state map as the kernels see it: a reference pad_buffer (C, P) channels-first <-> rows [zrows, zrows + P) of
// its op's (P_op, st_C) channels-last state.  Key channel c = g * cg + cc sits at column col0 + g * gstride + cc (gstride 0: the groups
// are copies of one shared input).  On import the rows [0, zrows) of the key's columns are zeroed (AD v0: they only meet zero taps).
struct alignas(16) StateEntry {      // 16-byte aligned: the tile table follows the entries in one upload
    const void* st[2];        // the op's state buffer for a stream whose slot bit is 0 (st[cur]) and 1 (st[cur ^ 1])
    long long per;            // elements per stream of the op's state (P_op * st_C)
    long long off;            // the entry's first element in a stream's exported vector
    int C, P, zrows, st_C, cg, col0, gstride;
    int list;                 // 0 = encoder ops, 1 = decoder ops: which slot bits name the stream's buffer
    int wc;                   // channels an import writes (shared input: cg, copy 0; 0: the entry is not imported)
};

struct StateArgs {
    const StateEntry* ent;
    const int4* tiles;        // {entry, c0, r0, 0}: a 32 x 32 tile of key channels [c0, +32) x handle rows [r0, +32)
    const int* streams;       // per requested stream: {stream id, encoder slot bit, decoder slot bit}
    int n;                    // requested streams
    void* ext;                // (n, S) stream-major vectors
    long long S;              // elements per stream
    int* err;                 // import on the fp16-split engine: bit 1 for a value outside its range (|v| >= 6e4 or non-finite)
};

template <typename T, bool IMPORT>
__global__ void __launch_bounds__(256) stream_state_kernel(StateArgs a) {
    __shared__ T tile[32][33];
    const int4 tl = a.tiles[blockIdx.x];
    const StateEntry& e = a.ent[tl.x];
    const int c0 = tl.y, r0 = tl.z;
    const int nc = min(32, (IMPORT ? e.wc : e.C) - c0), nr = min(32, e.zrows + e.P - r0);
    if (nc <= 0) return;
    const int tid = threadIdx.x;
    bool bad = false;
    for (int i = blockIdx.y; i < a.n; i += gridDim.y) {
        const int s = a.streams[3 * i], sel = a.streams[3 * i + 1 + e.list];
        T* st = (T*)e.st[sel] + (long long)s * e.per;
        T* ext = (T*)a.ext + (long long)i * a.S + e.off;
        if (!IMPORT) {
            // channels-last rows (consecutive threads: consecutive channels) -> tile[row][channel] -> channels-first (consecutive rows)
            for (int k = tid; k < nc * nr; k += 256) {
                const int r = k / nc, c = k - r * nc, row = r0 + r, kc = c0 + c, g = kc / e.cg;
                if (row >= e.zrows) tile[r][c] = st[(long long)row * e.st_C + e.col0 + g * e.gstride + (kc - g * e.cg)];
            }
            __syncthreads();
            for (int k = tid; k < nc * nr; k += 256) {
                const int c = k / nr, r = k - c * nr, row = r0 + r;
                if (row >= e.zrows) ext[(long long)(c0 + c) * e.P + row - e.zrows] = tile[r][c];
            }
        } else {
            for (int k = tid; k < nc * nr; k += 256) {
                const int c = k / nr, r = k - c * nr, row = r0 + r;
                T v;
                if (row >= e.zrows) {
                    v = ext[(long long)(c0 + c) * e.P + row - e.zrows];
                    if constexpr (std::is_same<T, float>::value) bad |= a.err && !(fabsf(v) < 60000.f);
                } else {
                    v = T(0);
                }
                tile[r][c] = v;
            }
            __syncthreads();
            for (int k = tid; k < nc * nr; k += 256) {
                const int r = k / nc, c = k - r * nc, row = r0 + r, kc = c0 + c, g = kc / e.cg;
                st[(long long)row * e.st_C + e.col0 + g * e.gstride + (kc - g * e.cg)] = tile[r][c];
            }
        }
        __syncthreads();
    }
    if (bad) atomicOr(a.err, 2);
}

}  // namespace adec
