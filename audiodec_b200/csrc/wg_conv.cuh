// wg_conv_kernel: the causal conv family on Hopper warpgroup tensor cores (wgmma.mma_async, sm_90a), persistent.
//
// Same ConvArgs contract as conv_gemm_kernel (kernels.cuh).  GEMM orientation: M = 128 time steps of a tile (two consumer warpgroups,
// 64 rows each), N = output-channel tile NT, K = input channels of one tap.  Both operands are K-major, no-swizzle "column blocks"
//     smem[(kb * ROWS + row) * 16 B]     (kb = 16-byte block of K, core matrices of 8 rows x 16 B: SBO = 128 B, LBO = ROWS * 16 B)
// so a conv tap is a row-shifted start address of the same window - no im2col, no copies: tap k of a dilated conv reads rows
// [k*dil, k*dil + 128).  Three precisions share the schedule:
//
//   PREC_F16 (default, fp32-grade: every layer that must stay within 1e-4 / bit-identical indices)
//       a     = A_hi + 2^-11 A_lo         A_hi = fp16(a),      A_lo = fp16((a - A_hi) * 2^11)        (producer warps)
//       w * s = W_hi + W_lo               W_hi = fp16(w * s),  W_lo = fp16(w * s - W_hi),  W_his = 2^-11 W_hi   (host, s = 2^p_c per
//                                                                    output column c: max|w| s over the column in [2^12, 2^13) keeps
//                                                                    the column's largest weights' three pieces normal)
//       a w s ~= A_lo W_his + A_hi W_lo + A_hi W_hi     three fp16 products, fp32 accumulation, result * 2^-p_c in the epilogue
//                                                       (ConvArgs::cscale).
//     fp16 and tf32 both carry 11 significand bits, so this is as accurate as 3xTF32, at half the operand bytes per MAC.
//     Range: |a| < 65504 (checked in the epilogue, ConvArgs::err).
//   PREC_TF32 (ADEC_CONV_PATH=tf32): a = A_hi + A_lo, w = W_hi + W_lo in tf32; A_lo W_hi + A_hi W_lo + A_hi W_hi.  No range limit.
//   PREC_BF16 (the bf16 modes of the HiFi-GAN vocoder and the symAD decoder-only handle): bf16 operands, one product.  In the fused
//     residual unit the intermediate operand is bf16_rne(ELU(fp32 sum of the dilated conv)), rounded once by split2.
//
// The tensor core's fp32 accumulation truncates at every step, which over the hundreds of steps of a long-K conv becomes a 1e-5-level
// systematic shrink - enough to flip nearest-codeword decisions.  So accumulation is GROUPED: one group = one 32-channel piece x up to
// TPG taps goes into a fresh register partial (scale-d = 0), and the partial is added into the fp32 accumulators with round-to-nearest
// adds.  At NT = 128 a group runs as two 64-column halves, so a consumer thread holds 64 accumulators + 32 partials.
//
// Warp roles (one CTA per SM, persistent over (time tile, channel tile, stream) tiles):
//   warps 0-7   two consumer warpgroups: wgmma issue, partial accumulation, fused residual-unit intermediate, epilogue
//   warps 8-10  activation producers (global -> pre-activation -> hi/lo split -> smem window pieces, n_wbuf buffers)
//   last warp   weight producer (1-D bulk async copies of host-packed stages)
// mbarrier rings connect them.  A parity wait cannot tell phase k from phase k-2, so every barrier has waiters that observe each
// of its phases in order: both consumer warpgroups consume every weight stage and every window piece, and a slot is refilled only
// after both released it.  The fused 1x1 conv reads only its own warpgroup's 64 rows of the intermediate, so that hand-off needs
// nothing but a warpgroup-local named barrier.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "kernels.cuh"

namespace adec {

constexpr int TC_TT = 128;             // output rows per tile
constexpr int TC_CP = 32;              // channels per activation piece
constexpr int TC_MIDP = 128;           // rows of the fused intermediate operand
constexpr float F16_LO_SCALE = 2048.f; // 2^11
enum { PREC_BF16 = 1, PREC_TF32 = 2, PREC_F16 = 3 };

// two floats from a 32-bit shared-memory address: volatile, so the compiler neither hoists it out of the tile loop nor keeps a
// generic pointer to the scales live across the kernel
__device__ __forceinline__ float2 lds_f2(uint32_t saddr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr));
    return v;
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ADEC_PHASES builds (kernels.cuh): ADEC_PH(k) adds the SM cycles since the previous mark of this thread to phase k.  The default build
// compiles none of it.
#ifdef ADEC_PHASES
#define ADEC_PH_START() (ph_t = (uint32_t)clock())
#define ADEC_PH(k) do { const uint32_t ph_now = (uint32_t)clock(); ph[k] += ph_now - ph_t; ph_t = ph_now; } while (0)
#define ADEC_PH_USE(x) (ph_sink += __float_as_uint(x))   // waits for a load: the producers' load phase ends when the data is there
#else
#define ADEC_PH_USE(x) ((void)0)
#define ADEC_PH_START() ((void)0)
#define ADEC_PH(k) ((void)0)
#endif
__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// shared-memory matrix descriptor, K-major, no swizzle: start >> 4 | LBO >> 4 << 16 | SBO (8 rows of 16 B = 128 B) >> 4 << 32
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr, uint32_t lbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)(128 >> 4) << 32);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Register fence on the accumulators: the fence / wait instructions above do not name them, so without this the compiler may move
// ordinary reads or writes of the accumulators into the asynchronous window, which ptxas then repairs by serializing the MMAs (C7514).
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x K] B[K x N], fp32 accumulators in registers; one instruction covers 32 bytes of K (k16 f16/bf16, k8 tf32)
template <int N, int PREC> struct Wgmma;
#define ADEC_WG_N32(PREC, TYPE, TAIL)                                                                                              \
    template <> struct Wgmma<32, PREC> {                                                                                           \
        __device__ __forceinline__ static void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {                     \
            asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n wgmma.mma_async.sync.aligned.m64n32" TYPE                \
                         " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1" TAIL ";\n}"                  \
                         : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),          \
                           "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])     \
                         : "l"(da), "l"(db), "r"(acc));                                                                            \
        }                                                                                                                          \
    };
#define ADEC_WG_N64(PREC, TYPE, TAIL)                                                                                              \
    template <> struct Wgmma<64, PREC> {                                                                                           \
        __device__ __forceinline__ static void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {                     \
            asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n wgmma.mma_async.sync.aligned.m64n64" TYPE                \
                         " {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27," \
                         "%28,%29,%30,%31}, %32, %33, p, 1, 1" TAIL ";\n}"                                                          \
                         : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),          \
                           "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),    \
                           "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),  \
                           "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])   \
                         : "l"(da), "l"(db), "r"(acc));                                                                            \
        }                                                                                                                          \
    };
ADEC_WG_N32(PREC_F16, "k16.f32.f16.f16", ", 0, 0")
ADEC_WG_N32(PREC_BF16, "k16.f32.bf16.bf16", ", 0, 0")
ADEC_WG_N32(PREC_TF32, "k8.f32.tf32.tf32", "")
ADEC_WG_N64(PREC_F16, "k16.f32.f16.f16", ", 0, 0")
ADEC_WG_N64(PREC_BF16, "k16.f32.bf16.bf16", ", 0, 0")
ADEC_WG_N64(PREC_TF32, "k8.f32.tf32.tf32", "")
#undef ADEC_WG_N32
#undef ADEC_WG_N64

template <int NT, int PREC> struct WgCfg {
    static constexpr int EB = PREC == PREC_TF32 ? 4 : 2;           // operand bytes
    static constexpr int KBB = TC_CP * EB / 16;                    // 16-byte K blocks per 32-channel piece and plane
    static constexpr int NPR = PREC == PREC_F16 ? 3 : PREC == PREC_TF32 ? 2 : 1;   // weight planes per tap: hi | lo (| hi * 2^-11)
    static constexpr int NPL = PREC == PREC_BF16 ? 1 : 2;          // activation planes: hi | lo
    // taps per group (= per weight stage).  The fused fp16-split unit at NT = 32 (RU(32)) takes one tap per group in every variant:
    // its paired kernel (PAIR) can only group single taps, and an output's sum must not depend on which variant computed it.
    __host__ __device__ static constexpr int tpg(bool fuse) { return PREC == PREC_TF32 || (PREC == PREC_F16 && NT == 32 && fuse) ? 1 : 2; }
    static constexpr int TAP_BYTES = NPR * KBB * NT * 16;          // one (piece, tap) of weights
    __host__ __device__ static constexpr int stage_bytes(bool fuse) { return tpg(fuse) * TAP_BYTES; }
    // the fused intermediate (all NT channels, 128 rows; PAIR: 256 rows, the two halves of the paired outputs)
    __host__ __device__ static constexpr int mid_bytes(bool pair) { return NPL * (NT * EB / 16) * TC_MIDP * (pair ? 2 : 1) * 16; }
    // weight stages: the fused tf32 unit at NT = 128 keeps a 128 KB intermediate, which leaves room for one stage and one window buffer.
    // PAIR: 9, a whole tile's weights (8 paired taps and the 1x1) in flight; 3 stages measured 3 % slower per step on an H100.
    __host__ __device__ static constexpr int stages(bool fuse, bool pair) { return pair ? 9 : PREC == PREC_TF32 && NT == 128 && fuse ? 1 : NT == 128 ? 2 : 3; }
    // PAIR: a stage holds one paired tap [W_j | W_j-1], 2 NT columns
    __host__ __device__ static constexpr int stage_alloc(bool fuse, bool pair) { return pair ? 2 * TAP_BYTES : stage_bytes(fuse); }
    static constexpr int PW = NT < 64 ? NT : 64;                   // columns per wgmma (partial width)
    // 384 threads: a multiple of 128 keeps ptxas' per-thread register budget at 168 (the consumers hold NT / 2 + PW / 2 accumulators)
    static constexpr int NPROD = 96;                               // activation-producer threads
    static constexpr int THREADS = 256 + NPROD + 32;
    __host__ __device__ static constexpr int win_pitch(int wrows) { return ((wrows + 1) & ~3) + 2; }   // rows, == 2 mod 4: conflict-free stores
    __host__ __device__ static constexpr int win_bytes(int wrows) { return NPL * KBB * win_pitch(wrows) * 16; }
    // window buffers: as many as fit (1..4): the producers run that many pieces ahead of the MMAs.  wrows: stored window rows
    // scale_bytes: the per-column weight scales at the end (PREC_F16: ConvArgs::cscale copied in at the start; 0 otherwise)
    static int n_wbuf(int wrows, bool fuse, bool pair, int scale_bytes) {
        const long long avail = 227 * 1024 - 512 - (long long)stages(fuse, pair) * stage_alloc(fuse, pair) - (fuse ? (long long)mid_bytes(pair) : 0) -
                                scale_bytes;
        const long long n = avail / win_bytes(wrows);
        return (int)(n > 4 ? 4 : n);
    }
    static size_t smem_bytes(int wrows, bool fuse, bool pair, int scale_bytes) {
        return 512 + (size_t)stages(fuse, pair) * stage_alloc(fuse, pair) + (size_t)n_wbuf(wrows, fuse, pair, scale_bytes) * win_bytes(wrows) +
               (fuse ? (size_t)mid_bytes(pair) : 0) + scale_bytes;
    }
};

// PAIR (the fused RU(32), DESIGN §4.0): one MMA row computes the outputs t and t + dil of a tile of pair_tt(dil) rows, and the window is
// stored de-interleaved by (row / dil) % 2 into an even and an odd array of pair_rows(K, dil) rows each
__host__ __device__ constexpr int pair_tt(int dil) { return 2 * dil * (TC_TT / dil); }
__host__ __device__ constexpr int pair_rows(int K, int dil) { return TC_TT + (K - 1) / 2 * dil; }

template <int ACT>
__device__ __forceinline__ float4 apply_act_t(float4 v, float slope) {
    if (ACT == ACT_ELU) { v.x = act_elu(v.x); v.y = act_elu(v.y); v.z = act_elu(v.z); v.w = act_elu(v.w); }
    if (ACT == ACT_LRELU) { v.x = act_lrelu(v.x, slope); v.y = act_lrelu(v.y, slope); v.z = act_lrelu(v.z, slope); v.w = act_lrelu(v.w, slope); }
    return v;
}

__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ uint32_t b2_bits(__nv_bfloat162 h) { return *reinterpret_cast<const uint32_t*>(&h); }
// two consecutive channels -> their hi (and lo) operand bits: one 32-bit word each for fp16 / bf16, two for tf32
template <int PREC>
__device__ __forceinline__ void split2(float x, float y, uint2& hi, uint2& lo) {
    if (PREC == PREC_F16) {
        const __half2 h = __floats2half2_rn(x, y);
        const float2 f = __half22float2(h);
        hi.x = h2_bits(h);
        lo.x = h2_bits(__floats2half2_rn((x - f.x) * F16_LO_SCALE, (y - f.y) * F16_LO_SCALE));
    } else if (PREC == PREC_TF32) {
        const float hx = tf32_rna(x), hy = tf32_rna(y);
        hi = make_uint2(__float_as_uint(hx), __float_as_uint(hy));
        lo = make_uint2(__float_as_uint(x - hx), __float_as_uint(y - hy));
    } else {
        hi.x = b2_bits(__floats2bfloat162_rn(x, y));
    }
}
// 8 consecutive channels of one window row -> 16 bytes (f16 / bf16) or 32 bytes in two K blocks `bstride` apart (tf32) per plane
template <int PREC>
__device__ __forceinline__ void split_store(unsigned char* hi, unsigned char* lo, size_t bstride, const float4 u, const float4 v) {
    uint2 h0, l0, h1, l1, h2, l2, h3, l3;
    split2<PREC>(u.x, u.y, h0, l0); split2<PREC>(u.z, u.w, h1, l1);
    split2<PREC>(v.x, v.y, h2, l2); split2<PREC>(v.z, v.w, h3, l3);
    if (PREC == PREC_TF32) {
        *reinterpret_cast<uint4*>(hi) = make_uint4(h0.x, h0.y, h1.x, h1.y);
        *reinterpret_cast<uint4*>(hi + bstride) = make_uint4(h2.x, h2.y, h3.x, h3.y);
        *reinterpret_cast<uint4*>(lo) = make_uint4(l0.x, l0.y, l1.x, l1.y);
        *reinterpret_cast<uint4*>(lo + bstride) = make_uint4(l2.x, l2.y, l3.x, l3.y);
    } else {
        *reinterpret_cast<uint4*>(hi) = make_uint4(h0.x, h1.x, h2.x, h3.x);
        if (PREC == PREC_F16) *reinterpret_cast<uint4*>(lo) = make_uint4(l0.x, l1.x, l2.x, l3.x);
    }
}

// Persistent-tile iterator: tile = xt + n_x * (y + n_y * b) advances by gridDim.x per step with carried additions instead of / and %.
struct TileIter {
    int tile, xt, y, b, sx, sy, sb, nx, ny;
    __device__ __forceinline__ TileIter(int first, int step, int n_x, int n_y) {
        nx = n_x; ny = n_y; tile = first;
        xt = first % n_x;
        const int q = first / n_x;
        y = q % n_y; b = q / n_y;
        sx = step % n_x;
        const int sq = step / n_x;
        sy = sq % n_y; sb = sq / n_y;
    }
    __device__ __forceinline__ void next(int step) {
        tile += step;
        xt += sx;
        const int cx = xt >= nx ? 1 : 0;
        xt -= cx ? nx : 0;
        y += sy + cx;
        const int cy = y >= ny ? 1 : 0;
        y -= cy ? ny : 0;
        b += sb + cy;
    }
};

__device__ __forceinline__ float4 norm4(float4 x, const float* mean, const float* scale) {
    const float4 mu = *reinterpret_cast<const float4*>(mean);
    const float4 sc = *reinterpret_cast<const float4*>(scale);
    x.x = __fdiv_rn(x.x - mu.x, sc.x); x.y = __fdiv_rn(x.y - mu.y, sc.y);
    x.z = __fdiv_rn(x.z - mu.z, sc.z); x.w = __fdiv_rn(x.w - mu.w, sc.w);
    return x;
}

// One group into a fresh partial: ntaps taps of one 32-channel piece, all three products (small terms first).  a_hi / a_lo: this
// warpgroup's first row of the piece's planes, lbo: their K-block pitch; bw: the weight stage (plus the column-half offset).
template <int NT, int PREC, int TPG>
__device__ __forceinline__ void wg_group(float (&d)[WgCfg<NT, PREC>::PW / 2], uint32_t a_hi, uint32_t a_lo, uint32_t lbo, uint32_t tap_step,
                                         int ntaps, uint32_t bw) {
    using Cfg = WgCfg<NT, PREC>;
    constexpr int NKS = Cfg::KBB / 2;
    constexpr uint32_t B_LBO = NT * 16u, B_KS = 2u * NT * 16u, B_T = Cfg::TAP_BYTES, B_PL = Cfg::KBB * NT * 16u;
    constexpr uint32_t PL_SMALL = PREC == PREC_F16 ? 2u : 0u;      // plane multiplied by A_lo: W_his (fp16) or W_hi (tf32)
    uint32_t acc = 0u;
    wg_fence_regs(d);
    wg_fence();
    if (PREC != PREC_BF16) {
#pragma unroll
        for (int t = 0; t < TPG; ++t)
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks)
                if (t < ntaps) {
                    Wgmma<Cfg::PW, PREC>::mma(d, wg_desc(a_lo + t * tap_step + ks * 2u * lbo, lbo), wg_desc(bw + t * B_T + PL_SMALL * B_PL + ks * B_KS, B_LBO), acc);
                    acc = 1u;
                }
#pragma unroll
        for (int t = 0; t < TPG; ++t)
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks)
                if (t < ntaps) Wgmma<Cfg::PW, PREC>::mma(d, wg_desc(a_hi + t * tap_step + ks * 2u * lbo, lbo), wg_desc(bw + t * B_T + B_PL + ks * B_KS, B_LBO), 1u);
    }
#pragma unroll
    for (int t = 0; t < TPG; ++t)
#pragma unroll
        for (int ks = 0; ks < NKS; ++ks)
            if (t < ntaps) {
                Wgmma<Cfg::PW, PREC>::mma(d, wg_desc(a_hi + t * tap_step + ks * 2u * lbo, lbo), wg_desc(bw + t * B_T + ks * B_KS, B_LBO), acc);
                acc = 1u;
            }
    wg_commit();
    wg_wait0();
    wg_fence_regs(d);
}

// stream slots: history row i (< P) of utterance u's slot, channel offset c within the row, in the buffer the slot is read from.  32-bit
// element offsets (the host keeps a state buffer below 2^31 elements): the window loop has no registers to spare for 64-bit math.
template <typename XT>
__device__ __forceinline__ const XT* slot_hist(const ConvArgs& a, int u, int i, int c) {
    const int e = __ldg(a.vl_slot + u);
    const XT* base = reinterpret_cast<const XT*>((e & 1) ? (const void*)a.st_out : (const void*)a.st_in);
    return base + (((e >> 1) * a.P + i) * a.st_ld + c);
}

// BST: activations, causal state, residual and output stored as bf16 in HBM (bf16 operands only; no 4-channel strided convs).  The
// fused residual unit reads its skip, its own input, as stored.
// VL: utterances of different lengths in one stacked row space (ConvArgs::vl_in / vl_out), zero history, no state written; a separate
// instantiation, so that the uniform kernels keep their code.  With ConvArgs::vl_slot set (a runtime branch, not another instantiation)
// each utterance is a chunk of one stream slot: history from the slot, new state written back to it.
// PAIR: the fused RU(32) with two output rows per MMA row (m64n64 over K + 1 paired taps [W_j | W_j-1], DESIGN §4.0); uniform rows only
// (no VL, no stacked rows), which the host guarantees.
template <int NT, bool FUSE, int PRE, int PREC, bool BST, bool VL = false, bool PAIR = false>
__global__ void __launch_bounds__(WgCfg<NT, PREC>::THREADS, 1) wg_conv_kernel(const ConvArgs a, int n_xtiles, int n_ytiles, int n_tiles) {
    static_assert(!BST || PREC == PREC_BF16, "bf16 storage is built for the bf16-operand kernels");
    static_assert(!PAIR || (NT == 32 && FUSE && PREC == PREC_F16 && !BST && !VL), "the paired kernel is built for the fused fp16-split RU(32)");
    using Cfg = WgCfg<NT, PREC>;
    using XT = typename std::conditional<BST, __nv_bfloat16, float>::type;
    constexpr int S = Cfg::stages(FUSE, PAIR), CP = TC_CP, TT = TC_TT, KBB = Cfg::KBB, EB = Cfg::EB, TPG = Cfg::tpg(FUSE), PW = Cfg::PW;
    constexpr int NPROD = Cfg::NPROD, WWARP = (256 + NPROD) / 32;         // weight producer warp
    constexpr int STAGE_BYTES = Cfg::stage_alloc(FUSE, PAIR), TAP_BYTES = Cfg::TAP_BYTES;
    constexpr int NH = NT / PW;                                  // column halves per group
    constexpr int NACC = PAIR ? NT : NT / 2;                     // accumulators per consumer thread (2 rows x NT / 4 columns; PAIR: x 2)
    constexpr int MBLK = NT * EB / 16;                           // K blocks of the fused intermediate per plane
    constexpr int MIDP = PAIR ? 2 * TC_MIDP : TC_MIDP;           // rows of the fused intermediate

    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* b_full = reinterpret_cast<uint64_t*>(smem_raw);     // [S] weights landed
    uint64_t* b_empty = b_full + S;                                // [S] weights consumed (both consumer warpgroups)
    uint64_t* w_full = b_empty + S;                                // [4] window piece written
    uint64_t* w_empty = w_full + 4;                                // [4] window piece consumed (both consumer warpgroups)
    unsigned char* bst = smem_raw + 512;
    const int ttile = PAIR ? pair_tt(a.dil) : TT;                  // output rows per tile
    const int wrows = ttile + (a.Ktaps - 1) * a.dil;               // window rows (time)
    const int prows = PAIR ? pair_rows(a.Ktaps, a.dil) : 0;        // PAIR: rows of the even array; the odd array follows it
    const int wrp = Cfg::win_pitch(PAIR ? 2 * prows : wrows);
    const int win_b = Cfg::win_bytes(PAIR ? 2 * prows : wrows);
    unsigned char* wbuf0 = bst + S * STAGE_BYTES;                  // a.n_wbuf window buffers of win_b bytes
    unsigned char* mbuf = wbuf0 + (size_t)a.n_wbuf * win_b;        // FUSE only: [plane][MBLK][MIDP rows][16 B]
    // PREC_F16: the per-column weight scales, [G * Cout_g] (FUSE: then [Cout_g] of w2), as ConvArgs::cscale, after the intermediate
    constexpr uint32_t SCALE_OFF = FUSE ? Cfg::mid_bytes(PAIR) : 0;   // bytes past mbuf
    // PAIR: window row m (time) -> its row in the de-interleaved storage
    auto srow = [&](int m) -> int {
        if constexpr (PAIR) {
            const int blk = m / a.dil;
            return (blk & 1) * prows + (blk >> 1) * a.dil + (m - blk * a.dil);
        } else {
            return m;
        }
    };

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    unsigned long long kt0 = 0;
    long long kc0 = 0;
    if (a.dbg && blockIdx.x == 0 && tid == 0) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(kt0)); kc0 = clock64(); }
#ifdef ADEC_PHASES
    uint32_t ph[PH_N] = {}, ph_t = 0, ph_sink = 0;
#endif
    if (tid == 0) {
        for (int s = 0; s < S; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], 2); }
        for (int i = 0; i < 4; ++i) { mbar_init(&w_full[i], NPROD); mbar_init(&w_empty[i], 2); }
        mbar_fence_init();
    }
    if constexpr (PREC == PREC_F16) {
        // constants, like the weights: read before griddepcontrol.wait; one shared-memory read per column pair in the tile loop
        const int n = (n_ytiles / a.n_co_tiles + (FUSE ? 1 : 0)) * a.Cout_g;
        float* sscale = reinterpret_cast<float*>(mbuf + SCALE_OFF);
        for (int i = tid; i < n; i += Cfg::THREADS) sscale[i] = __ldg(a.cscale + i);
    }
    __syncthreads();
    // programmatic dependent launch: everything above - and the weight stream, weights being constants - may overlap the previous
    // kernel's tail; the warps that read activations / state / skip tensors or write outputs wait for that grid first
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    if (warp != WWARP) asm volatile("griddepcontrol.wait;" ::: "memory");

    if (warp == WWARP) {
        // ------------------------------------------------ weight producer: one bulk copy per group (TPG taps)
        if (lane == 0) {
            int c = 0;
            ADEC_PH_START();
            auto stream = [&](const unsigned char* base, int pieces, int taps, int tap_bytes) {
                for (int p = 0; p < pieces; ++p)
                    for (int t0 = 0; t0 < taps; t0 += TPG, ++c) {
                        const int s = c % S, it = c / S;
                        const uint32_t bytes = (uint32_t)(taps - t0 >= TPG ? TPG : taps - t0) * tap_bytes;
                        ADEC_PH(PH_WISSUE);
                        if (it > 0) mbar_wait(&b_empty[s], (it - 1) & 1, 100);
                        ADEC_PH(PH_WFREE);
                        mbar_arrive_expect_tx(&b_full[s], bytes);
                        bulk_g2s(bst + s * STAGE_BYTES, base + ((long long)p * taps + t0) * tap_bytes, bytes, &b_full[s]);
                    }
            };
            const unsigned char* w1 = reinterpret_cast<const unsigned char*>(a.w);
            const unsigned char* w2 = reinterpret_cast<const unsigned char*>(a.w2);
            for (TileIter it(blockIdx.x, gridDim.x, n_xtiles, n_ytiles); it.tile < n_tiles; it.next(gridDim.x)) {
                // PAIR: K + 1 paired taps of 2 NT columns
                stream(w1 + (long long)it.y * a.w_tile_floats * 4, a.n_pieces, PAIR ? a.Ktaps + 1 : a.Ktaps, PAIR ? 2 * TAP_BYTES : TAP_BYTES);
                if (FUSE) stream(w2, NT / CP, 1, TAP_BYTES);
            }
            ADEC_PH(PH_WISSUE);
        }
    } else if (warp >= 8) {
        // ------------------------------------------------ activation producers: one item = 8 channels (32 B of fp32 / 16 B of bf16) of one
        // window row.
        // The loads of a piece are issued BEFORE the wait for a free window buffer, so global latency overlaps the MMAs that still read
        // the buffer; a.n_wbuf (2..4) buffers let the producers run several pieces ahead.
        const int pt = tid - 256;
        int wb = 0, wround = 0;                    // window piece counter wp = wround * n_wbuf + wb
        constexpr int RPP = NPROD / 4;             // window rows per pass (4 items of 8 channels per row)
        constexpr int UNR = 6;                     // rows in flight per thread (8 spilled up to 138 B and measured no faster)
        constexpr int UNR_E = VL ? 5 : 6;          // VL: the stream-slot history loads need the registers of one row
        const int c8 = pt & 3, m0 = pt >> 2;
        const size_t bstride = (size_t)wrp * 16;   // K-block pitch of a window plane
        const bool halves = a.RG > 1 && a.Cin < 8; // a 4-channel strided conv: the two halves of an item are different x~ rows
        ADEC_PH_START();
        for (TileIter it(blockIdx.x, gridDim.x, n_xtiles, n_ytiles); it.tile < n_tiles; it.next(gridDim.x)) {
            const int xt = it.xt, y = it.y, b = it.b;
            int g = 0, co_tile = y;
            if (a.n_co_tiles != n_ytiles) { g = y / a.n_co_tiles; co_tile = y - g * a.n_co_tiles; }
            const int j0 = xt * ttile;
            const XT* xg = reinterpret_cast<const XT*>(a.x) + (long long)b * a.x_bs + g * a.x_goff;
            const XT* sg = reinterpret_cast<const XT*>(a.st_in) + (long long)b * a.P * a.st_ld + g * a.st_goff;
            // VL: the utterance u0 that owns row j0, the first rows of it and of the next one, its input rows and length
            const int halo = (a.Ktaps - 1) * a.dil;
            int u0 = 0, u0_start = 0, u0_next = 0, u0_T = 0;
            const XT* xu0 = xg;
            if constexpr (VL) {
                u0 = vl_find(a.vl_out, halo, a.vl_B, j0);
                u0_start = vl_row(a.vl_out, halo, u0);
                u0_next = vl_row(a.vl_out, halo, u0 + 1);
                const int i0 = __ldg(a.vl_in + u0);
                u0_T = __ldg(a.vl_in + u0 + 1) - i0;
                xu0 = xg + (long long)i0 * a.ldx;
            }
            for (int p = 0; p < a.n_pieces; ++p) {
                const int buf = wb;
                const uint32_t wpar = (uint32_t)(wround - 1) & 1u;
                bool waited = wround == 0;
                if (++wb == a.n_wbuf) { wb = 0; ++wround; }
                unsigned char* hi = wbuf0 + (size_t)buf * win_b + (size_t)c8 * (KBB / 4) * bstride;
                unsigned char* lo = hi + (size_t)KBB * bstride;
                const int q = p * CP + c8 * 8;
                int r = 0, ci = q;
                if (a.RG > 1) { r = q >> a.lgCin; ci = q & (a.Cin - 1); }
                long long i_first = (long long)j0 * a.RG + r;
                long long i_last = (long long)(j0 + wrows - 1) * a.RG + r;
                const XT* xb = xg;
                int Tb = a.T;
                bool one_utt = true;
                if constexpr (VL) {
                    i_first = (long long)(j0 - u0_start) * a.RG + r;
                    i_last = (long long)(j0 - u0_start + wrows - 1) * a.RG + r;
                    xb = xu0;
                    Tb = u0_T;
                    one_utt = j0 + wrows <= u0_next;
                }
                if (i_first >= a.P && i_last - a.P < Tb && one_utt && PRE != ACT_NORM && !halves && !a.stack_L) {
                    // interior piece: every row comes from the chunk (VL: from one utterance)
                    const XT* xp = xb + ci + (i_first - a.P + (long long)m0 * a.RG) * a.ldx;
                    const long long xstep = (long long)RPP * a.RG * a.ldx;
                    for (int mb = m0; mb < wrows; mb += RPP * UNR, xp += xstep * UNR) {
                        float4 u[UNR], v[UNR];
#pragma unroll
                        for (int k = 0; k < UNR; ++k)
                            if (mb + k * RPP < wrows) ldg8(xp + k * xstep, u[k], v[k]);
                        ADEC_PH(PH_LOAD);
                        if (!waited) { mbar_wait(&w_empty[buf], wpar, 500); waited = true; }
                        ADEC_PH(PH_FREE);
#pragma unroll
                        for (int k = 0; k < UNR; ++k)
                            if (mb + k * RPP < wrows) { ADEC_PH_USE(u[k].x); ADEC_PH_USE(v[k].w); }
                        ADEC_PH(PH_LOAD);
#pragma unroll
                        for (int k = 0; k < UNR; ++k) {
                            const int m = mb + k * RPP;
                            if (m < wrows) split_store<PREC>(hi + srow(m) * 16, lo + srow(m) * 16, bstride, apply_act_t<PRE>(u[k], a.slope), apply_act_t<PRE>(v[k], a.slope));
                        }
                        ADEC_PH(PH_CONV);
                    }
                } else {
                    // edge piece: rows from the causal state (stored post-activation), the chunk, or beyond its end (zeros)
                    int ci2 = ci + 4;
                    // VL: this thread's rows ascend, so the utterance of each is found by stepping forward from u0
                    int vu = u0, vu_start = u0_start, vu_next = u0_next, vu_T = u0_T;
                    const XT* xvu = xu0;
                    for (int mb = m0; mb < wrows; mb += RPP * UNR_E) {
                        float4 u[UNR_E], v[UNR_E];
                        unsigned act = 0u;
#pragma unroll
                        for (int k = 0; k < UNR_E; ++k) {
                            const int m = mb + k * RPP;
                            u[k] = v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (m < wrows) {
                                // stacked rows: window row j0 + m of the stack is local row `ml` of stream `sm`
                                int ml = j0 + m;
                                const XT* xs = xg;
                                const XT* ss = sg;
                                bool live = true;
                                if constexpr (VL) {
                                    while (vu + 1 < a.vl_B && ml >= vu_next) {
                                        ++vu;
                                        vu_start = vu_next;
                                        vu_next = vl_row(a.vl_out, halo, vu + 1);
                                        const int i0 = __ldg(a.vl_in + vu);
                                        vu_T = __ldg(a.vl_in + vu + 1) - i0;
                                        xvu = xg + (long long)i0 * a.ldx;
                                    }
                                    ml -= vu_start;
                                    xs = xvu;
                                } else if (a.stack_L) {
                                    const int sm = ml / a.stack_L;
                                    ml -= sm * a.stack_L;
                                    live = sm < a.n_streams;
                                    xs = xg + (long long)sm * a.x_bs;
                                    ss = sg + (long long)sm * a.P * a.st_ld;
                                }
                                if constexpr (BST) {
                                    // both halves are one 16-byte vector of the same x~ row (bf16 storage has no 4-channel strided convs)
                                    const long long i = (long long)ml * a.RG + r;
                                    long long ti = i - a.P;
                                    if (a.hist_rep && ti < 0) ti = 0;
                                    if (live) {
                                        if (ti < 0) {       // VL: zero history, or the utterance's slot history
                                            if (!VL) ldg8(ss + i * a.st_ld + ci, u[k], v[k]);
                                            else if (a.vl_slot) ldg8(slot_hist<XT>(a, vu, (int)i, g * a.st_goff + ci), u[k], v[k]);
                                        }
                                        else if (ti < (VL ? vu_T : a.T)) { ldg8(xs + ti * a.ldx + ci, u[k], v[k]); act |= 3u << (2 * k); }
                                    }
                                } else {
#pragma unroll
                                    for (int hf = 0; hf < 2; ++hf) {
                                        int rr = r, cc = ci + 4 * hf;
                                        if (halves) { rr = (q + 4 * hf) >> a.lgCin; cc = (q + 4 * hf) & (a.Cin - 1); if (hf) ci2 = cc; }
                                        const long long i = (long long)ml * a.RG + rr;
                                        long long ti = i - a.P;
                                        if (a.hist_rep && ti < 0) ti = 0;              // non-streaming transposed conv: replicate the first input row
                                        float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f);
                                        if (live) {
                                            if (ti < 0) {
                                                if (!VL) w4 = __ldg(reinterpret_cast<const float4*>(ss + i * a.st_ld + cc));
                                                else if (a.vl_slot) w4 = ldg4(slot_hist<XT>(a, vu, (int)i, g * a.st_goff + cc));
                                            }
                                            else if (ti < (VL ? vu_T : a.T)) { w4 = __ldg(reinterpret_cast<const float4*>(xs + ti * a.ldx + cc)); act |= 1u << (2 * k + hf); }
                                        }
                                        if (hf) v[k] = w4; else u[k] = w4;
                                    }
                                }
                            }
                        }
                        ADEC_PH(PH_LOAD);
                        if (!waited) { mbar_wait(&w_empty[buf], wpar, 500); waited = true; }
                        ADEC_PH(PH_FREE);
#pragma unroll
                        for (int k = 0; k < UNR_E; ++k)
                            if (mb + k * RPP < wrows) { ADEC_PH_USE(u[k].x); ADEC_PH_USE(v[k].w); }
                        ADEC_PH(PH_LOAD);
#pragma unroll
                        for (int k = 0; k < UNR_E; ++k) {
                            const int m = mb + k * RPP;
                            if (m < wrows) {
                                float4 x0 = u[k], x1 = v[k];
                                if ((act >> (2 * k)) & 1u) x0 = PRE == ACT_NORM ? norm4(x0, a.mean + ci, a.scale + ci) : apply_act_t<PRE>(x0, a.slope);
                                if ((act >> (2 * k)) & 2u) x1 = PRE == ACT_NORM ? norm4(x1, a.mean + ci2, a.scale + ci2) : apply_act_t<PRE>(x1, a.slope);
                                split_store<PREC>(hi + srow(m) * 16, lo + srow(m) * 16, bstride, x0, x1);
                            }
                        }
                        ADEC_PH(PH_CONV);
                    }
                }
                fence_async_smem();
                mbar_arrive(&w_full[buf]);
            }
            // ---- new causal state (conv_layer.py:155): written by the CTA whose tile holds the stream's last output row
            if (!VL && co_tile == 0 && g < a.st_groups && a.P > 0) {
                int s_lo = b, s_hi = b - 1;
                if (a.stack_L) {
                    // streams whose last valid row sm * L + Tout - 1 lies in [j0, j0 + TT)
                    s_lo = (j0 - (a.Tout - 1) + a.stack_L - 1) / a.stack_L;
                    if (j0 < a.Tout - 1) s_lo = 0;
                    s_hi = (j0 + ttile - 1 - (a.Tout - 1)) / a.stack_L;
                    if (j0 + ttile - 1 < a.Tout - 1) s_hi = -1;
                    if (s_hi > a.n_streams - 1) s_hi = a.n_streams - 1;
                } else if (xt == (a.Tout - 1) / ttile) {
                    s_hi = b;
                }
                for (int sm = s_lo; sm <= s_hi; ++sm) {
                    const XT* xs = reinterpret_cast<const XT*>(a.x) + (long long)sm * a.x_bs + g * a.x_goff;
                    const XT* ss = reinterpret_cast<const XT*>(a.st_in) + (long long)sm * a.P * a.st_ld + g * a.st_goff;
                    XT* so = reinterpret_cast<XT*>(a.st_out) + (long long)sm * a.P * a.st_ld + g * a.st_goff;
                    const int nvec = a.P * (a.Cin / 4);
                    for (int idx = pt; idx < nvec; idx += NPROD) {
                        const int r = idx / (a.Cin / 4);
                        const int cc = (idx - r * (a.Cin / 4)) * 4;
                        const long long i = (long long)a.T + r;
                        float4 w4;
                        if (i < a.P) {
                            w4 = ld4(ss + i * a.st_ld + cc);
                        } else {
                            w4 = ldg4(xs + (i - a.P) * a.ldx + cc);
                            if (PRE == ACT_NORM) w4 = norm4(w4, a.mean + cc, a.scale + cc);
                            else w4 = apply_act_t<PRE>(w4, a.slope);
                        }
                        st4(so + (long long)r * a.st_ld + cc, w4);
                    }
                }
            }
        }
        // ---- stream slots: every utterance's new state (rows [T_u, T_u + P) of slot history || chunk) goes to the slot's other buffer,
        // which no CTA of this launch reads, so it is written after the tiles (the window loop keeps its registers), one (utterance,
        // group) per CTA in turn
        if (VL && a.vl_slot && a.P > 0) {
            const long long per = (long long)a.P * a.st_ld;
            const int nvec = a.P * (a.Cin / 4);
            for (int w = blockIdx.x; w < a.vl_B * a.st_groups; w += gridDim.x) {
                const int g = w / a.vl_B, u = w - g * a.vl_B;
                const int i0 = __ldg(a.vl_in + u), Tu = __ldg(a.vl_in + u + 1) - i0;
                const XT* xs = reinterpret_cast<const XT*>(a.x) + (long long)i0 * a.ldx + g * a.x_goff;
                const XT* ss = slot_rows(a.vl_slot, u, reinterpret_cast<const XT*>(a.st_in) + g * a.st_goff,
                                         reinterpret_cast<XT*>(a.st_out) + g * a.st_goff, per, true);
                XT* so = slot_rows(a.vl_slot, u, reinterpret_cast<const XT*>(a.st_in) + g * a.st_goff,
                                   reinterpret_cast<XT*>(a.st_out) + g * a.st_goff, per, false);
                for (int idx = pt; idx < nvec; idx += NPROD) {
                    const int r = idx / (a.Cin / 4);
                    const int cc = (idx - r * (a.Cin / 4)) * 4;
                    const long long i = (long long)Tu + r;
                    float4 w4;
                    if (i < a.P) {
                        w4 = ldg4(ss + i * a.st_ld + cc);
                    } else {
                        w4 = ldg4(xs + (i - a.P) * a.ldx + cc);
                        if (PRE == ACT_NORM) w4 = norm4(w4, a.mean + cc, a.scale + cc);
                        else w4 = apply_act_t<PRE>(w4, a.slope);
                    }
                    st4(so + (long long)r * a.st_ld + cc, w4);
                }
            }
        }
    } else {
        // ------------------------------------------------ consumer warpgroups: MMAs, register accumulation, fused intermediate, epilogue
        const int wg = warp >> 2;
        // accumulator fragment of wgmma m64nN: register 4j + e holds row (wrow + 8 * (e >> 1)), column 8j + col2 + (e & 1)
        const int wrow = 64 * wg + 16 * (warp & 3) + (lane >> 2), col2 = 2 * (lane & 3);
        const uint32_t row0_off = (uint32_t)(64 * wg) * 16u;            // this warpgroup's first operand row
        const uint32_t wbuf0_u = smem_u32(wbuf0), mbuf_u = smem_u32(mbuf), bst_u = smem_u32(bst);
        const uint32_t lbo1 = (uint32_t)wrp * 16u, lbo2 = (uint32_t)MIDP * 16u;
        const uint32_t tap_step = (uint32_t)a.dil * 16u;
        constexpr int NPART = PAIR ? PW : PW / 2;           // PAIR: the conv's partial is m64n64
        float racc[NACC];
        float part[NPART];
        float (&part_h)[PW / 2] = *reinterpret_cast<float (*)[PW / 2]>(part);   // an NT-wide partial
        int c = 0, wb = 0, wround = 0;
        float vmax = 0.f;                                   // largest magnitude this thread produced (fp16-split range check)
        ADEC_PH_START();
        // one group (weight stage c): partials per column half, round-to-nearest adds, stage released to the weight producer
        auto group = [&](uint32_t a_hi, uint32_t a_lo, uint32_t lbo, uint32_t row_off, int ntaps) {
            const int s = c % S;
            mbar_wait(&b_full[s], (c / S) & 1, 300);
            ADEC_PH(PH_WGT);
            const uint32_t bw = bst_u + (uint32_t)s * STAGE_BYTES;
#pragma unroll
            for (int h = 0; h < NH; ++h) {
                wg_group<NT, PREC, TPG>(part_h, a_hi + row_off, a_lo + row_off, lbo, tap_step, ntaps, bw + (uint32_t)h * PW * 16u);
#pragma unroll
                for (int i = 0; i < PW / 2; ++i) racc[h * (PW / 2) + i] = __fadd_rn(racc[h * (PW / 2) + i], part_h[i]);
            }
            ADEC_PH(PH_MMA);
            if (threadIdx.x % 128 == 0) mbar_arrive(&b_empty[s]);
            ++c;
        };
        // PAIR: one paired tap [W_j | W_j-1] as one m64n64 group (columns 0..NT-1: output t, NT..2NT-1: output t + dil)
        auto pgroup = [&](uint32_t a_hi, uint32_t a_lo, uint32_t row_off) {
            if constexpr (PAIR) {
                const int s = c % S;
                mbar_wait(&b_full[s], (c / S) & 1, 300);
                ADEC_PH(PH_WGT);
                wg_group<2 * NT, PREC, 1>(part, a_hi + row_off, a_lo + row_off, lbo1, tap_step, 1, bst_u + (uint32_t)s * STAGE_BYTES);
#pragma unroll
                for (int i = 0; i < NACC; ++i) racc[i] = __fadd_rn(racc[i], part[i]);
                ADEC_PH(PH_MMA);
                if (threadIdx.x % 128 == 0) mbar_arrive(&b_empty[s]);
                ++c;
            }
        };
        // racc index of (half h, fragment register i) -> column h * PW + 8 * (i >> 2) + col2 + (i & 1), row wrow + 8 * ((i >> 1) & 1)
        // acc_col(i), i % 4 == 0: the column of racc[i] and racc[i + 2] within the channel tile (racc[i + 1], racc[i + 3]: the next one;
        // PAIR: the outputs t + dil have the same columns)
        auto acc_col = [&](int i) {
            const int fi = PAIR ? i : i % (PW / 2);
            return ((PAIR ? 0 : i / (PW / 2) * PW) + 8 * (fi >> 2) + col2) % NT;
        };
        for (TileIter it(blockIdx.x, gridDim.x, n_xtiles, n_ytiles); it.tile < n_tiles; it.next(gridDim.x)) {
            const int xt = it.xt, y = it.y, b = it.b;
            int g = 0, co_tile = y;
            if (a.n_co_tiles != n_ytiles) { g = y / a.n_co_tiles; co_tile = y - g * a.n_co_tiles; }
            const int j0 = xt * ttile;
#pragma unroll
            for (int i = 0; i < NACC; ++i) racc[i] = 0.f;
            // the first MMA of a group ignores the partial (scale-d = 0); zeroing it here rather than once leaves its registers free
            // for the epilogue's loads
#pragma unroll
            for (int i = 0; i < NPART; ++i) part[i] = 0.f;
            for (int p = 0; p < a.n_pieces; ++p) {
                const int buf = wb;
                mbar_wait(&w_full[buf], wround & 1, 200);
                ADEC_PH(PH_WIN);
                if (++wb == a.n_wbuf) { wb = 0; ++wround; }
                const uint32_t a_hi = wbuf0_u + (uint32_t)buf * (uint32_t)win_b;
                if constexpr (PAIR) {
                    // paired tap j reads window row t + j dil of the even-block rows t: the even array (j even) or the odd one, shifted
                    for (int j = 0; j <= a.Ktaps; ++j)
                        pgroup(a_hi, a_hi + (uint32_t)KBB * lbo1, row0_off + (uint32_t)((j & 1) * prows + (j >> 1) * a.dil) * 16u);
                } else {
                    for (int t0 = 0; t0 < a.Ktaps; t0 += TPG)
                        group(a_hi, a_hi + (uint32_t)KBB * lbo1, lbo1, row0_off + (uint32_t)t0 * tap_step, a.Ktaps - t0 >= TPG ? TPG : a.Ktaps - t0);
                }
                if (threadIdx.x % 128 == 0) mbar_arrive(&w_empty[buf]);
            }
            if (FUSE) {
                // weight scale out, activation, split into the 1x1 conv's A operand: this warpgroup's 64 rows of the intermediate (PAIR:
                // its 64 MMA rows of each half, the half of output t + dil in rows TC_MIDP.. of the intermediate)
                // PAIR: MMA rows from ttile / 2 on (dil 3, 9) read window rows past the tile, computed and dropped
                const bool ok0 = !PAIR || wrow < ttile / 2, ok8 = !PAIR || wrow + 8 < ttile / 2;
#pragma unroll
                for (int i = 0; i < NACC; i += 4) {
                    float4 s4 = make_float4(racc[i], racc[i + 1], racc[i + 2], racc[i + 3]);
                    if constexpr (PREC == PREC_F16) {
                        const float2 sc = lds_f2(mbuf_u + SCALE_OFF + 4u * (uint32_t)acc_col(i));
                        s4 = make_float4(s4.x * sc.x, s4.y * sc.y, s4.z * sc.x, s4.w * sc.y);
                    }
                    const float4 m4 = apply_act_t<PRE>(s4, a.slope);
                    racc[i] = m4.x; racc[i + 1] = m4.y; racc[i + 2] = m4.z; racc[i + 3] = m4.w;
                    if (PAIR) {
                        if (ok0) vmax = fmaxf(vmax, fmaxf(fabsf(m4.x), fabsf(m4.y)));
                        if (ok8) vmax = fmaxf(vmax, fmaxf(fabsf(m4.z), fabsf(m4.w)));
                    } else {
                        vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(m4.x), fabsf(m4.y)), fmaxf(fabsf(m4.z), fabsf(m4.w))));
                    }
                }
#pragma unroll
                for (int i = 0; i < NACC; i += 2) {
                    const int h = PAIR ? 0 : i / (PW / 2), fi = PAIR ? i : i % (PW / 2);
                    int co = h * PW + 8 * (fi >> 2) + col2, row = wrow + 8 * ((fi >> 1) & 1);
                    if (PAIR) { row += (co / NT) * TC_MIDP; co %= NT; }
                    const int blk = co * EB / 16, off = (co * EB) & 15;
                    unsigned char* hp = mbuf + ((size_t)blk * MIDP + row) * 16 + off;
                    uint2 hi, lo;
                    split2<PREC>(racc[i], racc[i + 1], hi, lo);
                    if (PREC == PREC_TF32) {
                        *reinterpret_cast<uint2*>(hp) = hi;
                        *reinterpret_cast<uint2*>(hp + (size_t)MBLK * MIDP * 16) = lo;
                    } else {
                        *reinterpret_cast<uint32_t*>(hp) = hi.x;
                        if (PREC == PREC_F16) *reinterpret_cast<uint32_t*>(hp + (size_t)MBLK * MIDP * 16) = lo.x;
                    }
                }
                fence_async_smem();
                named_bar_sync(1 + wg, 128);
#pragma unroll
                for (int i = 0; i < NACC; ++i) racc[i] = 0.f;
                ADEC_PH(PH_MID);
                if constexpr (PAIR) {
                    // the 1x1 conv as two NT-wide passes over the two halves, one weight stage: the unpaired kernel's MMAs, row for row
                    const int s = c % S;
                    mbar_wait(&b_full[s], (c / S) & 1, 300);
                    ADEC_PH(PH_WGT);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const uint32_t m_hi = mbuf_u + row0_off + (uint32_t)(hh * TC_MIDP * 16);
                        wg_group<NT, PREC, 1>(part_h, m_hi, m_hi + (uint32_t)MBLK * lbo2, lbo2, tap_step, 1, bst_u + (uint32_t)s * STAGE_BYTES);
#pragma unroll
                        for (int i = 0; i < PW / 2; ++i) racc[hh * (PW / 2) + i] = __fadd_rn(racc[hh * (PW / 2) + i], part_h[i]);
                    }
                    if (threadIdx.x % 128 == 0) mbar_arrive(&b_empty[s]);
                    ++c;
                    ADEC_PH(PH_MMA);
                } else {
                    for (int p = 0; p < NT / CP; ++p) {
                        const uint32_t m_hi = mbuf_u + (uint32_t)(p * KBB) * lbo2;
                        group(m_hi, m_hi + (uint32_t)MBLK * lbo2, lbo2, row0_off, 1);
                    }
                }
                // every thread's 1x1 MMAs have completed (wgmma.wait_group) before the next tile rewrites its rows of the intermediate
            }
            // ---- epilogue: this thread's output rows (NR: wrow and wrow + 8; PAIR: those MMA rows of the outputs t and t + dil) x
            // column pairs co_tile * NT + 8 k + col2 (k < NCB), racc index 4 k + 2 (rr & 1) + (PW / 2) (rr >> 1).  The stores may alias
            // the loads for all the compiler knows, so it keeps every load after the stores before it; the epilogue therefore runs in
            // batches of KB column blocks over all NR rows, each issuing its bias and residual loads before its first store: one round
            // trip per batch instead of one per column pair (DESIGN §4.0).
            // Each output is round(round(round(racc * cscale) + bias) + residual) (PREC_F16; the other precisions have no scale), three
            // separately rounded operations, never an FMA.  The scale is applied to the accumulators first, while the batches' loads
            // have no registers yet.
            if constexpr (PREC == PREC_F16) {
                const uint32_t cs = wbuf0_u + (uint32_t)a.n_wbuf * (uint32_t)win_b + SCALE_OFF +
                                    4u * (uint32_t)((FUSE ? a.Cout_g : 0) + g * a.Cout_g + co_tile * NT);
#pragma unroll
                for (int i = 0; i < NACC; i += 4) {
                    const int co = acc_col(i);
                    const float2 sc = co_tile * NT + co < a.Cout_g ? lds_f2(cs + 4u * (uint32_t)co) : make_float2(0.f, 0.f);
                    racc[i] = __fmul_rn(racc[i], sc.x); racc[i + 1] = __fmul_rn(racc[i + 1], sc.y);
                    racc[i + 2] = __fmul_rn(racc[i + 2], sc.x); racc[i + 3] = __fmul_rn(racc[i + 3], sc.y);
                }
            }
            constexpr int PB = NT < 128 ? 16 : (PREC == PREC_TF32 && FUSE) || VL ? 4 : 8;   // residual pairs per batch: larger ones spill
            constexpr int NR = PAIR ? 4 : 2, NCB = NACC / (2 * NR), KB = NCB < PB / NR ? NCB : PB / NR;
            const int co0 = co_tile * NT + col2;     // columns from Cout_g on: the zero-padded part of a channel tile (96 outputs of 128)
            int rt[NR], rbo[NR];                     // output row and stream of row rr, rt = -1: not stored
            {
                // VL: the utterance of row j0 + wrow (then of row + 8) and where its stacked rows start and end
                const int halo = (a.Ktaps - 1) * a.dil;
                int vu = 0, vu_start = 0, vu_next = 0;
                if constexpr (VL) {
                    vu = vl_find(a.vl_out, halo, a.vl_B, j0 + wrow);
                    vu_start = vl_row(a.vl_out, halo, vu);
                    vu_next = vl_row(a.vl_out, halo, vu + 1);
                }
#pragma unroll
                for (int rr = 0; rr < NR; ++rr) {
                    int bo = b, t = j0 + wrow + 8 * rr;
                    bool ok;
                    if constexpr (PAIR) {
                        // MMA row mr holds outputs t and t + dil (rr >> 1 = 1)
                        const int mr = wrow + 8 * (rr & 1), blk = mr / a.dil;
                        t = j0 + blk * 2 * a.dil + (mr - blk * a.dil) + (rr >> 1) * a.dil;
                        ok = mr < ttile / 2 && t < a.Tout;
                    } else if constexpr (VL) {
                        // local row t - vu_start of the utterance; rows past its Tout are the receptive-field overlap, computed and dropped
                        while (vu + 1 < a.vl_B && t >= vu_next) { ++vu; vu_start = vu_next; vu_next = vl_row(a.vl_out, halo, vu + 1); }
                        const int o0 = __ldg(a.vl_out + vu), ml = t - vu_start;
                        ok = ml < __ldg(a.vl_out + vu + 1) - o0;
                        t = o0 + ml;
                    } else {
                        if (a.stack_L) { bo = t / a.stack_L; t -= bo * a.stack_L; }
                        ok = t < a.Tout && bo < a.n_streams;
                    }
                    rt[rr] = ok ? t : -1;
                    rbo[rr] = bo;
                }
            }
#pragma unroll
            for (int k0 = 0; k0 < NCB; k0 += KB) {
                float2 bb[KB], r2[NR][KB];
                if (a.bias) {
#pragma unroll
                    for (int k = 0; k < KB; ++k) {
                        const int co_l = co0 + 8 * (k0 + k);
                        bb[k] = co_l < a.Cout_g ? __ldg(reinterpret_cast<const float2*>(a.bias + g * a.Cout_g + co_l)) : make_float2(0.f, 0.f);
                    }
                }
                if (a.res) {
#pragma unroll
                    for (int rr = 0; rr < NR; ++rr)
#pragma unroll
                        for (int k = 0; k < KB; ++k) {
                            const int t = rt[rr], co_l = co0 + 8 * (k0 + k);
                            r2[rr][k] = t >= 0 && co_l < a.Cout_g
                                            ? ldg2(reinterpret_cast<const XT*>(a.res) + (long long)rbo[rr] * a.res_bs + (long long)t * a.ldr + g * a.r_goff + co_l)
                                            : make_float2(0.f, 0.f);
                        }
                }
#pragma unroll
                for (int rr = 0; rr < NR; ++rr) {
                    const int t = rt[rr], bo = rbo[rr];
                    if (t < 0) continue;
#pragma unroll
                    for (int k = 0; k < KB; ++k) {
                        const int co_l = co0 + 8 * (k0 + k), i = 4 * (k0 + k) + 2 * (rr & 1) + (PW / 2) * (rr >> 1);
                        if (co_l >= a.Cout_g) continue;
                        float v0 = racc[i], v1 = racc[i + 1];
                        if (a.bias) { v0 = __fadd_rn(v0, bb[k].x); v1 = __fadd_rn(v1, bb[k].y); }
                        if (a.res) { v0 = __fadd_rn(r2[rr][k].x, v0); v1 = __fadd_rn(r2[rr][k].y, v1); }
                        vmax = fmaxf(vmax, fmaxf(fabsf(v0), fabsf(v1)));
                        if (a.out_nct) {
                            XT* yp = reinterpret_cast<XT*>(a.y) + (long long)bo * a.y_bs + (long long)(g * a.y_goff + co_l) * a.Tout + t;
                            st1(yp, v0);
                            st1(yp + a.Tout, v1);
                        } else {
                            st2(reinterpret_cast<XT*>(a.y) + (long long)bo * a.y_bs + (long long)t * a.ldy + g * a.y_goff + co_l, v0, v1);
                        }
                    }
                }
            }
            ADEC_PH(PH_EPI);
        }
        // every activation is some launch's output: one check here bounds the operands of the next launch's fp16 split
        if (PREC == PREC_F16 && a.err && !(vmax < 60000.f)) atomicOr(a.err, 2);
    }
#ifdef ADEC_PHASES
    if (a.dbg) {
        // one reporting thread per consumer warpgroup, activation-producer thread 0 and the weight-producer lane
        if (warp < 8 ? tid % 128 == 0 : warp == WWARP ? lane == 0 : tid == 256) {
            if (ph_sink == 0x7fc00001u) ph[PH_CONV] += 1u;     // keeps the loads the load phase waits for
            for (int k = 0; k < PH_N; ++k)
                if (ph[k]) atomicAdd(a.dbg + 6 + k, (unsigned long long)ph[k]);
        }
        if (blockIdx.x == 0 && tid == 0) {
            // launch descriptor: NT | FUSE << 8 | res << 9 | PAIR << 10 | VL << 11 | BST << 12 | PREC << 13 | Ktaps << 16 | dil << 24 |
            // input channels << 32 | Cout_g << 48
            a.dbg[3] = (unsigned long long)NT | (FUSE ? 1ull << 8 : 0) | (a.res ? 1ull << 9 : 0) | (PAIR ? 1ull << 10 : 0) |
                       (VL ? 1ull << 11 : 0) | (BST ? 1ull << 12 : 0) | ((unsigned long long)PREC << 13) | ((unsigned long long)a.Ktaps << 16) |
                       ((unsigned long long)a.dil << 24) | ((unsigned long long)(a.n_pieces * CP) << 32) | ((unsigned long long)a.Cout_g << 48);
            a.dbg[4] = (unsigned long long)a.Tout;
            a.dbg[5] = PH_N;
        }
    }
#endif
    if (a.dbg && blockIdx.x == 0 && tid == 0) {
        unsigned long long kt1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(kt1));
        a.dbg[0] = kt0; a.dbg[1] = kt1; a.dbg[2] = (unsigned long long)(clock64() - kc0);
    }
}

// mma_probe_kernel: the measured compute ceiling of the conv engine (bench.py's `roofline.compute`).  Every SM runs one CTA of two
// warpgroups that stream wgmma m64 x PW (K = 32 bytes per row) from shared-memory operands in the engine's own K-major no-swizzle
// layout, in groups of 12 accumulating MMAs per column half - the issue pattern of wg_conv_kernel without producers, epilogue or
// global traffic.  NT > 64 runs as NT / 64 column slices, as in the engine.
__device__ float g_probe_sink;
template <int NT, int PREC>
__global__ void __launch_bounds__(256) mma_probe_kernel(int n_groups, int a_pitch_rows) {
    using Cfg = WgCfg<NT, PREC>;
    constexpr int PW = Cfg::PW, KSTEPS = 8;                 // resident K steps, cycled
    extern __shared__ __align__(128) unsigned char smem[];
    const int a_bytes = KSTEPS * 2 * a_pitch_rows * 16;     // [KSTEPS * 2 blocks][a_pitch_rows rows][16 B]
    for (int i = threadIdx.x; i < a_bytes / 16 + KSTEPS * 2 * NT; i += 256) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0u, 0u, 0u, 0u);
    fence_async_smem();
    __syncthreads();
    const int wg = threadIdx.x >> 7;
    const uint32_t a_u = smem_u32(smem) + (uint32_t)(64 * wg) * 16u, b_u = smem_u32(smem + a_bytes);
    const uint32_t a_lbo = (uint32_t)a_pitch_rows * 16u, b_lbo = (uint32_t)NT * 16u;
    float d[PW / 2];
#pragma unroll
    for (int i = 0; i < PW / 2; ++i) d[i] = 0.f;
    float sink = 0.f;
    for (int g = 0; g < n_groups; ++g) {
#pragma unroll 1
        for (int h = 0; h < NT / PW; ++h) {
            wg_fence_regs(d);
            wg_fence();
#pragma unroll
            for (int k = 0; k < 12; ++k) {
                const uint32_t ks = (uint32_t)((g * 12 + k) % KSTEPS);
                Wgmma<PW, PREC>::mma(d, wg_desc(a_u + ks * 2u * a_lbo, a_lbo), wg_desc(b_u + ks * 2u * b_lbo + (uint32_t)h * PW * 16u, b_lbo), k ? 1u : 0u);
            }
            wg_commit();
            wg_wait0();
            wg_fence_regs(d);
            sink += d[0];
        }
    }
    if (sink != 0.f) g_probe_sink = sink;                   // operands are zeros: only keeps the result live
}

// wgmma_cols_kernel: one warpgroup runs the fp16-split group of one 32-channel tap (wg_group) as m64n64, and as m64n32 on each
// 32-column half of the same weights.  The paired RU(32) kernel gives the same sums as the unpaired one only if the two agree column
// for column, which NVIDIA does not document.  a: [plane 2][kb 4][64 rows][8 fp16], b: [plane 3][kb 4][64 columns][8 fp16];
// d64 / d32: [64 rows][64 columns] fp32.
__global__ void __launch_bounds__(128) wgmma_cols_kernel(const uint4* a, const uint4* b, float* d64, float* d32) {
    __shared__ __align__(128) uint4 sa[2 * 4 * 64];
    __shared__ __align__(128) uint4 sb[3 * 4 * 64];
    __shared__ __align__(128) uint4 sh[2][3 * 4 * 32];      // the two column halves of sb as N = 32 images
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < 2 * 4 * 64; i += 128) sa[i] = a[i];
    for (int i = tid; i < 3 * 4 * 64; i += 128) {
        sb[i] = b[i];
        sh[(i % 64) / 32][(i / 64) * 32 + i % 32] = b[i];
    }
    fence_async_smem();
    __syncthreads();
    const uint32_t au = smem_u32(sa), lbo = 64u * 16u;
    float d[32], h[16];
    wg_group<64, PREC_F16, 1>(d, au, au + 4u * lbo, lbo, 0u, 1, smem_u32(sb));
    // fragment register i: row 16 warp + lane / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (lane & 3) + (i & 1)
    const int r0 = 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 32; ++i) d64[(r0 + 8 * ((i >> 1) & 1)) * 64 + 8 * (i >> 2) + c0 + (i & 1)] = d[i];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        wg_group<32, PREC_F16, 1>(h, au, au + 4u * lbo, lbo, 0u, 1, smem_u32(sh[hh]));
#pragma unroll
        for (int i = 0; i < 16; ++i) d32[(r0 + 8 * ((i >> 1) & 1)) * 64 + 32 * hh + 8 * (i >> 2) + c0 + (i & 1)] = h[i];
    }
}

}  // namespace adec
