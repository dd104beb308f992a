/*
 * audiodec_b200 - C ABI of the H100-native AudioDec streaming forward path.
 *
 * This is the drop-in boundary (SURVEY.md section 8(b)).  The reference has no FFI: its
 * plug points are the two abstract hooks AudioCodec._load_encoder / _load_decoder
 * (bin/stream.py:38-45, implemented in utils/audiodec.py:32-56) whose return values are
 * duck-typed objects with encode / quantize / lookup / decode / initial_encoder /
 * initial_decoder / reset_buffer.  Every entry point below replaces one of those
 * methods; the Python shim in audiodec_b200/codec.py binds them with ctypes and
 * INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - plain C, no torch types; every function returns 0 on success, non-zero on error
 *     (adec_last_error() gives the message).  Nothing throws, nothing falls back to CPU.
 *   - all data pointers of the *_dev entry points are DEVICE pointers on the handle's GPU;
 *     `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - activations are fp32, except on HiFi-GAN handles with compute_dtype 2 (the *_bf16 decode entry points).  Layouts at
 *     the boundary are the reference's own
 *     (SURVEY.md A.3):  x (B,1,T)   z (B,64,F) channels-first   idx (Nq,B,F) int64 flat
 *     (+1024*i already added)   zq (B,F,64) channels-last   y (B,1,F*hop).
 *   - a handle owns its weights and its per-stream causal state (the reference's
 *     pad_buffer tensors, layers/conv_layer.py:144-146,185-187), for `n_streams`
 *     independent streams.  One handle is driven by one host thread at a time
 *     (bin/stream.py:343-346); different handles are independent.
 */
#ifndef AUDIODEC_B200_H
#define AUDIODEC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ADEC_MAX_STAGES 8

typedef struct adec_handle adec_handle;

enum adec_model_type {
    ADEC_MODEL_SYMAD = 0,      /* models/autoencoder/AudioDec.py:166 StreamGenerator (codec='audiodec') */
    ADEC_MODEL_HIFIGAN = 1     /* models/vocoder/HiFiGAN.py:222 StreamGenerator, MultiGroupConv1d fusion (AD v1) */
};

/* POD mirror of config.yml `generator_params` (exp/.../config.yml:102-134 resp. :102-130). */
typedef struct adec_config {
    int model_type;
    /* symAD (models/autoencoder/AudioDec.py:31-51) */
    int input_channels, output_channels, encode_channels, decode_channels;
    int code_dim, codebook_num, codebook_size;
    int n_enc;  int enc_ratios[ADEC_MAX_STAGES];  int enc_strides[ADEC_MAX_STAGES];
    int n_dec;  int dec_ratios[ADEC_MAX_STAGES];  int dec_strides[ADEC_MAX_STAGES];
    int bias;
    /* HiFi-GAN (models/vocoder/HiFiGAN.py:31-47) */
    int in_channels, out_channels, channels, kernel_size;
    int n_up;   int upsample_scales[ADEC_MAX_STAGES];  int upsample_kernel_sizes[ADEC_MAX_STAGES];
    int resblock_kernel_size;
    int n_dil;  int resblock_dilations[ADEC_MAX_STAGES];
    int groups;
    float negative_slope;
    int use_weight_norm;
    int has_stats;
    /* appended in round 1 (variants of SURVEY.md 8(f) rank 1) */
    int codec_activate;                                    /* symAAD: codec='activate_audiodec' (encoder.py:145-175, decoder.py:151-214) */
    int n_resblocks;  int resblock_kernel_sizes[ADEC_MAX_STAGES];   /* AD v0: MultiReceptiveField, one residual block per kernel size */
    /* appended in round 2 */
    int compute_dtype;                                     /* 0 = fp32-grade (default); 1 = bf16 conv operands with fp32 accumulation, HiFi-GAN vocoder
                                                              only: what `decoder.to(torch.bfloat16)` asks of the reference (BASELINE configs[2]);
                                                              2 = as 1, and every activation, the causal state and the decode input / output are
                                                              bf16 in memory (the reference's bf16 data layout and dtype contract): decode with
                                                              adec_decode_bf16 / adec_decode_offline_bf16.  1 and 2 need the f16 engine. */
} adec_config;

/* -- lifetime ---------------------------------------------------------------- */
/* replaces generator(**config['generator_params']) (utils/audiodec.py:40,54) + .eval().to(dev)
 * (bin/stream.py:60,69,75).  `device` = CUDA ordinal. */
int adec_create(const adec_config *cfg, int device, adec_handle **out);
void adec_destroy(adec_handle *h);
const char *adec_last_error(const adec_handle *h);   /* h may be NULL: error of the last failed adec_create */

/* -- weight ingest: replaces load_state_dict (utils/audiodec.py:41,55) ------- */
/* `key` is the reference state-dict key verbatim ("encoder.conv_blocks.0.conv.conv.weight",
 * "upsamples.1.deconv.weight_g", "quantizer.codebook.layers.3.embed", "mean", ...).  `data` is a HOST
 * pointer to contiguous fp32 of the given shape.  Unknown keys are an error, except the
 * training-only buffers cluster_size / embed_avg which are accepted and ignored. */
int adec_set_tensor(adec_handle *h, const char *key, const float *data, const int64_t *shape, int ndim);
/* folds weight-norm (w = g*v/||v||, HiFiGAN.py:193-203), repacks weights for the kernels, builds the
 * flat codebook + ||e||^2 (vq_module.py:151-157,96); errors if any required key is missing (strict=True). */
int adec_finalize(adec_handle *h);

/* -- per-stream causal state -------------------------------------------------- */
int adec_n_streams(const adec_handle *h);
/* n == current: no-op.  current == 1: that (warmed) stream's state is replicated n times.  current > 1: streams [0, min(n, current))
 * keep their state, streams added beyond `current` start from zero history (what reset_buffer() leaves).  Buffers are resized and
 * the replaced ones freed. */
int adec_set_streams(adec_handle *h, int n_streams);
/* reset_buffer() (AudioDec.py:250-256, HiFiGAN.py:298-305): zero all history, keep n_streams. */
int adec_reset(adec_handle *h, void *stream);

/* -- the hot path (device pointers) ------------------------------------------- */
/* StreamGenerator.encode (AudioDec.py:228-234): x (B,1,T) -> z (B,code_dim,F), F = frames_for(T). */
int adec_encode(adec_handle *h, const float *x, int B, int T, float *z, void *stream);
/* StreamGenerator.quantize (AudioDec.py:237-239): z (B,code_dim,F) -> idx (Nq,B,F) int64. Stateless. */
int adec_quantize(adec_handle *h, const float *z, int B, int F, int64_t *idx, void *stream);
/* Fused form of the quantize -> [pack] -> lookup hand-off (bin/stream.py:224 ships the int64 tensor through a queue): ONE launch
 * writes any of idx (Nq,B,F) int64, packed (B,F,adec_packed_frame_bytes) uint8 and zq (B,F,code_dim) = lookup(idx); pass NULL for
 * outputs that are not wanted (at least one must be given).  Same arithmetic, bit-identical to quantize + pack + lookup. */
int adec_quantize_ex(adec_handle *h, const float *z, int B, int F, int64_t *idx, uint8_t *packed, float *zq, void *stream);
/* StreamGenerator.lookup (AudioDec.py:242-243): idx (Nq,B,F) -> zq (B,F,code_dim). Stateless. */
int adec_lookup(adec_handle *h, const int64_t *idx, int B, int F, float *zq, void *stream);
/* StreamGenerator.decode (AudioDec.py:246-247 / HiFiGAN.py:268-273): zq (B,F,code_dim) -> y (B,1,F*hop). */
int adec_decode(adec_handle *h, const float *zq, int B, int F, float *y, void *stream);

/* Same, for a HiFi-GAN handle with compute_dtype 2: zq (B,F,in_channels) and y (B,1,F*hop) are bf16 (raw 16-bit words), both
 * 16-byte aligned.  adec_decode on such a handle fails, and so does adec_decode_bf16 on any other handle. */
int adec_decode_bf16(adec_handle *h, const uint16_t *zq, int B, int F, uint16_t *y, void *stream);

/* -- the non-streaming batch forward (SURVEY.md 8(f) rank 4; codecTest.py:78-95, codecStatistic.py:92-98) ---------- */
/* Encoder.forward + Projector.forward (models/autoencoder/modules/encoder.py:131, projector.py:49-50): every causal
 * conv zero-pads on the left (layers/conv_layer.py:148-151) = no history; any batch size.  x (B,1,T) -> z (B,code_dim,F).
 * DISCARDS the handle's streaming state (use a separate handle, or adec_reset + warm-up, before streaming again). */
int adec_encode_offline(adec_handle *h, const float *x, int B, int T, float *z, void *stream);
/* Decoder.forward (decoder.py:135-140) / HiFi-GAN Generator.forward (HiFiGAN.py:140-160): as above, and every transposed conv
 * pads with its FIRST input frame (ReplicationPad1d, conv_layer.py:189-192).  zq (B,F,code_dim) channels-last -> y (B,1,F*hop). */
int adec_decode_offline(adec_handle *h, const float *zq, int B, int F, float *y, void *stream);
/* adec_decode_offline for a compute_dtype 2 handle: bf16 zq (B,F,in_channels) channels-last -> bf16 y (B,1,F*hop), 16-byte aligned. */
int adec_decode_offline_bf16(adec_handle *h, const uint16_t *zq, int B, int F, uint16_t *y, void *stream);

/* output frames of encode for T input samples: floor((T-1)/s)+1 applied per stride (conv_layer.py:153-156) */
int adec_frames_for(const adec_handle *h, int T);
/* product of the strides (utils/audiodec.py:58-62) */
int adec_hop_length(const adec_handle *h);

/* -- whole path with HOST buffers (what demoFile.py:55-62 does around the four calls) ------- */
/* x_host (B,1,T) -> idx_host (Nq,B,F) (may be NULL) and y_host (B,1,F*hop).  Copies H2D, runs
 * enc.encode -> enc.quantize -> enc.lookup -> dec.decode on `stream`, copies D2H and synchronises.
 * `enc` must be a symAD handle; `dec` a symAD or HiFi-GAN handle (may equal enc) with fp32 activations (compute_dtype 0 or 1). */
int adec_codec_host(adec_handle *enc, adec_handle *dec, const float *x_host, int B, int T,
                    int64_t *idx_host, float *y_host, void *stream);

/* -- index bitstream (SURVEY.md 8(f) rank 2) -------------------------------------------------- */
/* The reference has no wire format: AudioCodecStreamer ships the int64 (Nq,F) index tensor through a queue
 * (bin/stream.py:224).  Packed frame = Nq local indices (idx - i*codebook_size) of ceil(log2 codebook_size) bits each,
 * stage 0 first, little-endian bit order, zero-padded to whole bytes: 8 x 10 bit = 10 bytes / frame = 12.8 kbit/s at
 * hop 300 / 48 kHz.  idx (Nq,B,F) int64 flat <-> packed (B,F,adec_packed_frame_bytes) uint8, device pointers. */
int adec_packed_frame_bytes(const adec_handle *h);       /* -1 if h is not a symAD handle */
int adec_pack_indices(adec_handle *h, const int64_t *idx, int B, int F, uint8_t *packed, void *stream);
int adec_unpack_indices(adec_handle *h, const uint8_t *packed, int B, int F, int64_t *idx, void *stream);
/* lookup straight from the packed bitstream (unpack fused into lookup): packed (B,F,bytes) -> zq (B,F,code_dim) */
int adec_lookup_packed(adec_handle *h, const uint8_t *packed, int B, int F, float *zq, void *stream);
/* synchronises `stream`, then returns and clears the handle's device-side flag: 1 if lookup / pack / unpack met an
 * out-of-range index since the last call (the reference's F.embedding would have raised, vq_module.py:160), -1 on error */
int adec_index_error(adec_handle *h, void *stream);
/* same protocol for the conv engine's range flag: 1 if an activation reached |a| >= 6e4 since the last call.  The default engine
 * multiplies fp16 pieces of the fp32 activations (wg_conv.cuh); the reference's fp32 convs (layers/conv_layer.py:55-64) have no such
 * bound, so a model that gets there must run with ADEC_CONV_PATH=tf32.  adec_codec_host checks both flags itself. */
int adec_range_error(adec_handle *h, void *stream);

/* number of kernel launches issued by this handle since creation (bench.py's gpu_launches) */
int64_t adec_launch_count(const adec_handle *h);

/* Diagnostics (handles created with ADEC_KTRACE=1 in the environment): copies up to max_records {start ns, end ns, SM cycles} records
 * of the tensor-core conv launches issued since the last call (CTA 0's globaltimer / clock64) and resets the trace; returns the
 * number of records or -1.  Used to measure the effective SM clock and the gaps between back-to-back launches. */
int adec_ktrace(adec_handle *h, unsigned long long *out, int max_records);

/* Measured compute ceiling of the conv engine for bench.py's roofline: every SM streams `n_groups` x 12 wgmma per 64-column slice
 * (M = 2 x 64, N = NT in {32, 64, 128, 256}, kind 0 = tf32 / 1 = f16) from shared-memory operands in the engine's layout, nothing else;
 * *tflops = dense TFLOP/s, *ms = duration (may be NULL).  No handle needed. */
int adec_probe_mma(int device, int kind, int NT, int n_groups, double *tflops, double *ms);

/* Per-launch CUDA-event timing on the handle's stream (bench.py's roofline leg).  adec_profile(h,1) starts
 * recording around every kernel launch, adec_profile(h,0) stops and clears.  adec_profile_report writes one line
 * per recorded launch: "<op name>\t<ms>\t<algorithmic bytes>\n" (bytes per SURVEY.md 8(d)'s per-layer model). */
int adec_profile(adec_handle *h, int enable);
int adec_profile_report(adec_handle *h, char *buf, int buf_len);

/* -- unit-test entry points for single layers (tests/test_layers_gpu.py) ------- */
/* One causal conv (layers/conv_layer.py:153-156) on device buffers, channels-first in/out like the
 * reference: x (B,Cin,T) HOST pointers, w (Cout,Cin/groups,K), state (B,Cin,(K-1)*dil) updated in place,
 * y (B,Cout,floor((T-1)/stride)+1).  bias may be NULL.  pre_act: 0 none, 1 ELU, 2 LeakyReLU(slope). */
int adec_test_causal_conv(int device, const float *x, int B, int Cin, int T, const float *w, const float *bias,
                          int Cout, int K, int stride, int dil, int groups, int pre_act, float slope,
                          float *state, float *y);
/* One causal transposed conv (layers/conv_layer.py:194-197): w (Cin,Cout,2*stride), state (B,Cin,1). */
int adec_test_causal_convtr(int device, const float *x, int B, int Cin, int T, const float *w, const float *bias,
                            int Cout, int stride, float *state, float *y);

/* One causal residual unit (models/autoencoder/modules/residual_unit.py:49-81):
 * y = x + W2 * ELU(conv_k7_dil(ELU(x))); x,y (B,C,T), w1 (C,C,K), w2 (C,C,1), state (B,C,(K-1)*dil). */
int adec_test_residual_unit(int device, const float *x, int B, int C, int T, const float *w1, const float *w2,
                            int K, int dil, float *state, float *y);

#ifdef __cplusplus
}
#endif
#endif /* AUDIODEC_B200_H */
