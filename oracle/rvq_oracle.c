/* ORACLE - test infrastructure only; never linked into the product library.
 *
 * Plain-C restatement of the reference's residual-VQ nearest-codeword search and codebook
 * lookup (layers/vq_module.py:90-104 VectorQuantize.forward_index, :136-149
 * ResidualVQ.forward_index, :151-161 initial/lookup), written so that every fp32 rounding
 * happens where torch-CPU (2.11, oneDNN/MKL build of this image) puts it:
 *
 *   dist[c] = ( x2 - dot2[c] ) + e2[c]                       vq_module.py:93-97
 *     x2   = flatten.pow(2).sum(1)   : rounded squares, 8-lane vectors, 4 interleaved vector
 *                                      accumulators, sequential combine, sequential horizontal add
 *     dot2 = (2*flatten) @ embed     : one accumulator per output, k = 0..D-1 in order, fused
 *                                      multiply-add (what MKL sgemm does for K = 64)
 *     e2   = embed.pow(2).sum(0)     : rounded squares, cascade sum in blocks of 16 rows
 *   index = first arg-max of -dist                            vq_module.py:98
 *   quantize = x + (e[index] - x)                             vq_module.py:101-102 (kept: it rounds)
 *   residual -= quantize                                      vq_module.py:143
 *
 * The orders above were found by probing torch on the build container and are pinned by
 * tests/test_host_cpu.py::test_c_rvq_oracle_matches_torch_bitwise (bit-exact distances on random data).
 * tests/test_rvq_spec_gpu.py holds rvq_kernel / lookup_kernel to this file with no tolerance.
 *
 * build (oracle/rvq_spec.py): gcc -O2 -ffp-contract=off -shared -fPIC -o oracle/_build/librvq_oracle.so oracle/rvq_oracle.c -lm
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static float sumsq_inner(const float *x, int d)
{
    /* torch sum over the contiguous last dim; d must be a multiple of 32 (64 in AudioDec) */
    float acc[4][8];
    memset(acc, 0, sizeof acc);
    for (int v = 0; v < d / 8; ++v)
        for (int l = 0; l < 8; ++l) {
            float sq = x[8 * v + l] * x[8 * v + l];
            acc[v & 3][l] = acc[v & 3][l] + sq;
        }
    float s = 0.f;
    for (int l = 0; l < 8; ++l) {
        float t = ((acc[0][l] + acc[1][l]) + acc[2][l]) + acc[3][l];
        s = (l == 0) ? t : s + t;
    }
    return s;
}

/* e2[c] = sum_k embed[k][c]^2, embed row-major (D,N) */
void adec_oracle_codeword_norms(const float *embed, int d, int n, float *e2)
{
    for (int c = 0; c < n; ++c) {
        float total = 0.f;
        for (int b = 0; b < d; b += 16) {
            float part = 0.f;
            for (int k = b; k < b + 16 && k < d; ++k) {
                float sq = embed[(size_t)k * n + c] * embed[(size_t)k * n + c];
                part = part + sq;
            }
            total = (b == 0) ? part : total + part;
        }
        e2[c] = total;
    }
}

/* adec_oracle_rvq with the codeword norms given: e2s (nq, N).  With the norms of
 * adec_oracle_codeword_norms this is the spec; tests pass other norms to model a host that sums
 * them in another order. */
void adec_oracle_rvq_e2(const float *x, int frames, int d, const float *embeds, const float *e2s,
                        int nq, int n, int64_t *idx, float *zq, float *dist_out)
{
    float *r = (float *)malloc(sizeof(float) * d);
    float *qsum = (float *)malloc(sizeof(float) * d);
    for (int f = 0; f < frames; ++f) {
        memcpy(r, x + (size_t)f * d, sizeof(float) * d);
        for (int k = 0; k < d; ++k) qsum[k] = 0.f;
        for (int i = 0; i < nq; ++i) {
            const float *E = embeds + (size_t)i * d * n;
            const float *e2 = e2s + (size_t)i * n;
            float x2 = sumsq_inner(r, d);
            int best = 0;
            float bestv = 0.f;
            for (int c = 0; c < n; ++c) {
                float dot = 0.f;
                for (int k = 0; k < d; ++k) dot = fmaf(2.0f * r[k], E[(size_t)k * n + c], dot);
                float dist = (x2 - dot) + e2[c];
                if (dist_out) dist_out[((size_t)i * frames + f) * n + c] = dist;
                float neg = -dist;
                if (c == 0 || neg > bestv) { bestv = neg; best = c; }
            }
            idx[(size_t)i * frames + f] = (int64_t)best + (int64_t)n * i;
            for (int k = 0; k < d; ++k) {
                float q = E[(size_t)k * n + best];
                float qq = r[k] + (q - r[k]);
                r[k] = r[k] - qq;
                qsum[k] = (i == 0) ? (0.f + qq) : qsum[k] + qq;
            }
        }
        if (zq) memcpy(zq + (size_t)f * d, qsum, sizeof(float) * d);
    }
    free(r); free(qsum);
}

/* x: (frames, D) residual input (modified copy kept internally); embeds: (nq, D, N);
 * idx out: (nq, frames) int64 flat (+ N*i); zq out (frames, D) = sum of quantize; dist_out optional
 * (nq, frames, N) for tests. */
void adec_oracle_rvq(const float *x, int frames, int d, const float *embeds, int nq, int n,
                     int64_t *idx, float *zq, float *dist_out)
{
    float *e2s = (float *)malloc(sizeof(float) * (size_t)nq * n);
    for (int i = 0; i < nq; ++i) adec_oracle_codeword_norms(embeds + (size_t)i * d * n, d, n, e2s + (size_t)i * n);
    adec_oracle_rvq_e2(x, frames, d, embeds, e2s, nq, n, idx, zq, dist_out);
    free(e2s);
}

/* lookup: zq[f] = sum_i codebook[idx[i][f]], codebook (nq*N, D), summed in i order (torch.sum dim 0) */
void adec_oracle_lookup(const int64_t *idx, int nq, int frames, const float *codebook, int d, float *zq)
{
    for (int f = 0; f < frames; ++f)
        for (int k = 0; k < d; ++k) {
            float s = 0.f;
            for (int i = 0; i < nq; ++i) {
                float v = codebook[(size_t)idx[(size_t)i * frames + f] * d + k];
                s = (i == 0) ? v : s + v;
            }
            zq[(size_t)f * d + k] = s;
        }
}
