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
 *   - activations are fp32, except on decoder handles (HiFi-GAN, symAD decoder-only) with compute_dtype 2 (the *_bf16 decode entry
 *     points).  Layouts at
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
    ADEC_MODEL_HIFIGAN = 1,    /* models/vocoder/HiFiGAN.py:222 StreamGenerator, MultiGroupConv1d fusion (AD v1) */
    ADEC_MODEL_SYMAD_DECODER = 2,  /* the decoder of a symAD StreamGenerator alone: what the receiver's `decoder` object runs
                                      (initial_decoder / decode, utils/audiodec.py:104-106).  Same config as ADEC_MODEL_SYMAD; loads a
                                      full generator state dict (decoder.* strict, encoder.* / projector.* / quantizer.* ignored).  The
                                      decode entry points, the state calls, adec_hop_length / adec_frames_for and the diagnostics work on
                                      it; encode, quantize*, lookup*, pack / unpack and adec_zq_moments fail.  compute_dtype 1 and 2 on
                                      the f16 engine, as for HiFi-GAN. */
    ADEC_MODEL_SYMAD_ENCODER = 3   /* the transmitter of a symAD StreamGenerator alone: encoder, projector and RVQ search, what the
                                      transmitter's `tx_encoder` object runs (initial_encoder / encode / quantize, utils/audiodec.py:
                                      100-102).  Same config as ADEC_MODEL_SYMAD; loads a full generator state dict (encoder.* /
                                      projector.* / quantizer.* strict, decoder.* ignored).  adec_encode*, adec_quantize,
                                      adec_quantize_ex (idx / packed; zq must be NULL), adec_pack_indices, the state calls,
                                      adec_frames_for / adec_hop_length / adec_packed_frame_bytes, ADEC_GRAPH_TX and the diagnostics work
                                      on it; decode*, lookup*, unpack, adec_quantize_forward, adec_zq_moments and serving as `enc` of
                                      adec_codec_host fail.  compute_dtype 0 encodes and quantizes bit for bit as a full symAD handle;
                                      compute_dtype 1 (f16 engine) runs the encoder's convs on bf16 operands with fp32 activations,
                                      state, x and z, and the RVQ on that fp32 z unchanged; compute_dtype 2 also keeps x, every
                                      activation, the causal state and z in bf16 (adec_encode*_bf16, adec_quantize*_bf16).  The stem
                                      keeps fp32 weights in both. */
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
                                                              and symAD decoder-only handles: what `decoder.to(torch.bfloat16)` asks of the
                                                              reference (BASELINE configs[2]); symAD encoder-only handles: the
                                                              encoder's and projector's convs on bf16 operands (the stem keeps fp32
                                                              weights; fp32 x, activations, state and z);
                                                              2 = as 1, and every activation, the causal state and the decode input / output are
                                                              bf16 in memory (the reference's bf16 data layout and dtype contract): decode with
                                                              adec_decode_bf16 / adec_decode_offline_bf16 (decoder handles), resp. encode and
                                                              quantize with adec_encode*_bf16 / adec_quantize*_bf16 (encoder-only handle).  1 and
                                                              2 need the f16 engine. */
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
/* Quantizer.forward's zq (quantizer.py:31-34, what codecStatistic.py:92-98 fits its statistics to): ONE launch writes
 * zq_fwd (B,F,code_dim) channels-last = ResidualVQ.forward's quantized_out, the sum over stages of r + (e - r) starting from 0.
 * (vq_module.py:136-143; a -0 comes out +0), and idx (Nq,B,F) int64 unless it is NULL.  The indices are those of adec_quantize;
 * zq_fwd may differ from lookup's sum of the codewords in the last bits. */
int adec_quantize_forward(adec_handle *h, const float *z, int B, int F, int64_t *idx, float *zq_fwd, void *stream);
/* Per-utterance moments of a varlen zq (sum F_b, code_dim) channels-last fp32, 16-byte aligned, as adec_quantize_forward writes it
 * for the varlen z: utterance b's rows are [sum_{i<b} F_i, +F_b).  frames: HOST array of B frame counts (>= 1), the row count must
 * fit in 31 bits.  Writes, per utterance and channel, fp64 sum (B,code_dim) = sum_f x and m2 (B,code_dim) = sum_f (x - T)^2 -
 * (sum_f (x - T))^2 / F_b with T = sum / F_b (the corrected two-pass term StandardScaler.partial_fit computes per call).  Two
 * launches, no host synchronise; deterministic, and an utterance's result does not depend on its place in the batch. */
int adec_zq_moments(adec_handle *h, const float *zq, const int *frames, int B, double *sum, double *m2, void *stream);
/* StreamGenerator.lookup (AudioDec.py:242-243): idx (Nq,B,F) -> zq (B,F,code_dim). Stateless. */
int adec_lookup(adec_handle *h, const int64_t *idx, int B, int F, float *zq, void *stream);
/* StreamGenerator.decode (AudioDec.py:246-247 / HiFiGAN.py:268-273): zq (B,F,code_dim) -> y (B,1,F*hop). */
int adec_decode(adec_handle *h, const float *zq, int B, int F, float *y, void *stream);

/* Same, for a HiFi-GAN or symAD decoder-only handle with compute_dtype 2: zq (B,F,in_channels resp. code_dim) and y (B,1,F*hop) are
 * bf16 (raw 16-bit words), both
 * 16-byte aligned.  adec_decode on such a handle fails, and so does adec_decode_bf16 on any other handle. */
int adec_decode_bf16(adec_handle *h, const uint16_t *zq, int B, int F, uint16_t *y, void *stream);

/* The encode family and quantize for a symAD encoder-only handle with compute_dtype 2: x (B,1,T) and z (B,code_dim,F) are bf16 (raw
 * 16-bit words), 16-byte aligned; the stem reads bf16 x, every activation and the causal state are bf16, the projector stores bf16 z.
 * adec_quantize_bf16 / adec_quantize_ex_bf16 widen bf16 z exactly and then run the fp32 RVQ unchanged, so the indices and packed bytes
 * are the spec applied to float(z) (zq must be NULL on an encoder-only handle).  The fp32 entry points fail on such a handle, and these
 * fail on every other handle.  Varlen / slot layouts as adec_encode_offline_varlen / adec_encode_streams. */
int adec_encode_bf16(adec_handle *h, const uint16_t *x, int B, int T, uint16_t *z, void *stream);
int adec_encode_offline_bf16(adec_handle *h, const uint16_t *x, int B, int T, uint16_t *z, void *stream);
int adec_encode_offline_varlen_bf16(adec_handle *h, const uint16_t *x, const int *lengths, int B, uint16_t *z, void *stream);
int adec_encode_streams_bf16(adec_handle *h, const uint16_t *x, const int *lengths, const int *streams, int B, uint16_t *z, void *stream);
int adec_quantize_bf16(adec_handle *h, const uint16_t *z, int B, int F, int64_t *idx, void *stream);
int adec_quantize_ex_bf16(adec_handle *h, const uint16_t *z, int B, int F, int64_t *idx, uint8_t *packed, float *zq, void *stream);

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

/* The same forwards over B utterances of DIFFERENT lengths in one launch sequence (codecTest.py transcodes a folder of them):
 * utterance b gives exactly what a uniform offline call of its own length gives, and no padded rows are computed.
 * Encoder.forward + Projector.forward: x is the utterances' samples concatenated, (sum T_b) device floats.  lengths: HOST array of B
 * sample counts (>= 1).  z: (code_dim, sum F_b) channels-first, utterance b's frames at columns [sum_{i<b} F_i, +F_b),
 * F_b = adec_frames_for(h, T_b).  This is the uniform layout with B = 1, F = sum F_b, so adec_quantize* and adec_lookup* take it
 * unchanged.  Discards the streaming state, as adec_encode_offline does.  Every row count of the batch must fit in 31 bits. */
int adec_encode_offline_varlen(adec_handle *h, const float *x, const int *lengths, int B, float *z, void *stream);
/* Decoder.forward / HiFi-GAN Generator.forward over B utterances.  zq: (sum F_b, code_dim) channels-last.  frames: HOST array of B
 * frame counts (>= 1).  y: (sum F_b * hop) device floats, utterance b at [hop * sum_{i<b} F_i, +hop * F_b). */
int adec_decode_offline_varlen(adec_handle *h, const float *zq, const int *frames, int B, float *y, void *stream);
/* adec_decode_offline_varlen for a compute_dtype 2 handle: bf16 zq and y, 16-byte aligned. */
int adec_decode_offline_varlen_bf16(adec_handle *h, const uint16_t *zq, const int *frames, int B, uint16_t *y, void *stream);
/* The varlen entry points need a tensor-core engine (f16 or tf32); the FFMA engine (ADEC_CONV_PATH=ffma) refuses them. */

/* -- stream slots: advance any subset of the handle's streams, each by a chunk of its own length, in one launch sequence ---------- */
/* Advance streams[b] (b < B, distinct, each in [0, n_streams)) by one chunk each: x = the chunks concatenated (sum T_b device
 * floats), lengths HOST (>= 1).  z (code_dim, sum F_b), F_b = adec_frames_for(h, T_b): the B = 1 layout adec_quantize* / adec_lookup*
 * already take.  Each stream gets exactly what a B = 1 streaming adec_encode of its chunk gives it.  Streams not listed keep their
 * state untouched, and cost nothing.  Needs a tensor-core engine; every row count must fit in 31 bits. */
int adec_encode_streams(adec_handle *h, const float *x, const int *lengths, const int *streams, int B, float *z, void *stream);
/* zq (sum F_b, code_dim) channels-last, frames HOST (>= 1) -> y (sum F_b * hop), stream b at [hop * sum_{i<b} F_i, +hop * F_b). */
int adec_decode_streams(adec_handle *h, const float *zq, const int *frames, const int *streams, int B, float *y, void *stream);
/* adec_decode_streams for a compute_dtype 2 handle: bf16 zq and y, 16-byte aligned. */
int adec_decode_streams_bf16(adec_handle *h, const uint16_t *zq, const int *frames, const int *streams, int B, uint16_t *y, void *stream);
/* Copy stream src's current causal state (all layers of the handle) into each dst[i]: a joining stream starts warm. */
int adec_copy_stream_state(adec_handle *h, int src, const int *dst, int n, void *stream);

/* The uniform streaming calls, adec_set_streams and adec_reset see every stream's latest state after slot calls (a handle that made slot
 * calls copies the streams whose state sits in the other ping-pong buffer back once, before its next uniform call or resize). */

/* -- stream state out of and into a handle: save, resume, and move a stream to another handle (another server, another GPU) ---------
 * The state map lists every reference pad_buffer the handle runs (layers/conv_layer.py:146,187), with the reference's key as a state dict
 * names it and its shape (C, P); buffers of layers the handle does not run (the encoder of a decoder-only handle) are not in it.  One
 * stream's state is S = adec_stream_state_elems(h) elements: the entries in map order, each (C, P) channels-first.  A MultiGroupConv1d
 * convs1.0 buffer holds `groups` copies of its shared input: export writes every copy, import reads copy 0.  AD v0's per-block buffers are
 * the tails of the handle's longer per-group history: import zeroes the older rows (they only meet zero taps) and takes convs1.0's shared
 * input from the block with the largest kernel. */
int     adec_state_entries(const adec_handle *h);                 /* entries of the state map, -1 before adec_finalize */
/* entry i: *key (valid for the handle's life), *C, *P; any of them may be NULL.  Returns non-zero for an i out of range. */
int     adec_state_entry(const adec_handle *h, int i, const char **key, int *C, int *P);
int64_t adec_stream_state_elems(const adec_handle *h);            /* S = sum C * P, elements per stream; -1 before adec_finalize */
/* Export / import the current state of streams[0..n) (HOST array of distinct ids in [0, n_streams)) to / from a device buffer of (n, S)
 * elements, 16-byte aligned: fp32, or bf16 words on a compute_dtype 2 handle, copied as they are.  One launch on `stream`, no host
 * synchronise; neither call changes which buffer a stream's next call reads, so an export between any two calls sees what the next one
 * would read.  Streams not listed keep their state bit for bit.  On the fp16-split engine an import sets the range flag
 * (adec_range_error) for a value that is non-finite or has |v| >= 6e4. */
int adec_get_stream_state(adec_handle *h, const int *streams, int n, void *out, void *stream);
int adec_set_stream_state(adec_handle *h, const int *streams, int n, const void *in, void *stream);

/* output frames of encode for T input samples: floor((T-1)/s)+1 applied per stride (conv_layer.py:153-156) */
int adec_frames_for(const adec_handle *h, int T);
/* product of the strides (utils/audiodec.py:58-62) */
int adec_hop_length(const adec_handle *h);

/* -- whole path with HOST buffers (what demoFile.py:55-62 does around the four calls) ------- */
/* x_host (B,1,T) -> idx_host (Nq,B,F) (may be NULL) and y_host (B,1,F*hop).  Copies H2D, runs
 * enc.encode -> enc.quantize -> enc.lookup -> dec.decode on `stream`, copies D2H and synchronises.
 * `enc` must be a full symAD handle; `dec` a symAD, symAD decoder-only or HiFi-GAN handle (may equal enc) with fp32 activations
 * (compute_dtype 0 or 1). */
int adec_codec_host(adec_handle *enc, adec_handle *dec, const float *x_host, int B, int T,
                    int64_t *idx_host, float *y_host, void *stream);

/* -- index bitstream (SURVEY.md 8(f) rank 2) -------------------------------------------------- */
/* The reference has no wire format: AudioCodecStreamer ships the int64 (Nq,F) index tensor through a queue
 * (bin/stream.py:224).  Packed frame = Nq local indices (idx - i*codebook_size) of ceil(log2 codebook_size) bits each,
 * stage 0 first, little-endian bit order, zero-padded to whole bytes: 8 x 10 bit = 10 bytes / frame = 12.8 kbit/s at
 * hop 300 / 48 kHz.  idx (Nq,B,F) int64 flat <-> packed (B,F,adec_packed_frame_bytes) uint8, device pointers. */
int adec_packed_frame_bytes(const adec_handle *h);       /* -1 if h is not a full or encoder-only symAD handle */
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

/* lookup / lookup_packed with bf16 zq (what a decoder with bf16 activations, compute_dtype 2, takes): the fp32 codeword sum rounded once
 * to nearest even, equal to the fp32 zq converted to bf16.  zq 16-byte aligned; needs code_dim % 8 == 0. */
int adec_lookup_bf16(adec_handle *h, const int64_t *idx, int B, int F, uint16_t *zq, void *stream);
int adec_lookup_packed_bf16(adec_handle *h, const uint8_t *packed, int B, int F, uint16_t *zq, void *stream);

/* -- loss concealment on the packed lookup ------------------------------------------------------------------------------------------
 * One output row of adec_lookup_packed_conceal.  A real row (src >= 0) is the lookup of packed frame src, bit for bit
 * adec_lookup_packed's; with slot >= 0 its fp32 sum is also stored in anchors[slot] (a session's last real frame of the call).  A
 * concealed row (src = -1) stands for a lost frame: with s_b the fp32 sum of packed frame `next` (the first frame after the loss) and
 * a = anchors[slot] (the session's last real frame before it), zq = fl(fl(fl(j / den) * fl(s_b - a)) + a) in fp32, every operation
 * rounded to nearest on its own (no contraction); slot = -1 means no anchor and zq = s_b.  j counts the lost frames from 1 and den is
 * their number plus one. */
typedef struct adec_conceal_row {
    int32_t src;   /* real row: packed frame in [0, F); -1 for a concealed row */
    int32_t next;  /* concealed row: packed frame in [0, F) after the loss; -1 for a real row */
    int32_t slot;  /* anchor row in [0, n_anchors), or -1: written by a real row, read by a concealed one */
    int32_t j;     /* concealed row: 1 <= j < den (ignored for a real row) */
    int32_t den;   /* concealed row: >= 2 (ignored for a real row) */
} adec_conceal_row;
/* packed (F, bytes) and anchors (n_anchors, code_dim) fp32, 16-byte aligned, are device buffers; rows (R) is a HOST array, checked
 * before anything runs (an error names the field: src / next / slot out of range, den < 2, j outside [1, den), an anchor that one row
 * reads and another writes, or that two rows write) and uploaded in stream order; zq (R, code_dim).  One launch.  Full symAD handle
 * only; an out-of-range code index sets the flag adec_index_error reads.  _bf16: zq is bf16, the fp32 result rounded once to nearest
 * even (as adec_lookup_packed_bf16); the anchors stay fp32. */
int adec_lookup_packed_conceal(adec_handle *h, const uint8_t *packed, int F, const adec_conceal_row *rows, int R, float *anchors,
                               int n_anchors, float *zq, void *stream);
int adec_lookup_packed_conceal_bf16(adec_handle *h, const uint8_t *packed, int F, const adec_conceal_row *rows, int R, float *anchors,
                                    int n_anchors, uint16_t *zq, void *stream);

/* -- the packed lookup of a receiver's playout clock -------------------------------------------------------------------------------
 * One output row of adec_lookup_packed_playout.  Three kinds of row, in one launch:
 *   real row (src >= 0, next = target = -1): adec_conceal_row's real row, bit for bit (with slot >= 0 it also stores the anchor);
 *   interpolated row (src = -1, next >= 0, target = -1): adec_conceal_row's concealed row, bit for bit (1 <= j < den);
 *   fade row (src = next = -1, target in [0, n_targets)): with t = targets[target] and a = anchors[slot],
 *     zq = t when j >= den or slot = -1, and otherwise zq = fl(fl(fl(j / den) * fl(t - a)) + a) in fp32, every operation rounded to
 *     nearest on its own (no contraction).  j >= 1 and den >= 1.  No packed frame is read.
 * A receiver fades a session whose packets stopped toward the codec's silence frame (the target) over den frames. */
typedef struct adec_playout_row {
    int32_t src;     /* real row: packed frame in [0, F); -1 otherwise */
    int32_t next;    /* interpolated row: packed frame in [0, F) after the loss; -1 otherwise */
    int32_t target;  /* fade row: target row in [0, n_targets); -1 otherwise */
    int32_t slot;    /* anchor row in [0, n_anchors), or -1: written by a real row, read by an interpolated or a fade row */
    int32_t j;       /* interpolated row: 1 <= j < den; fade row: j >= 1 (ignored for a real row) */
    int32_t den;     /* interpolated row: >= 2; fade row: >= 1 (ignored for a real row) */
} adec_playout_row;
/* packed (F, bytes; F = 0 and packed = NULL are allowed when no row reads a frame), anchors (n_anchors, code_dim) fp32 and targets
 * (n_targets, code_dim) fp32, both 16-byte aligned, are device buffers; zq (R, code_dim).  rows (R) is a HOST array, checked before
 * anything runs; an error names the field: src / next / target / slot out of range, a target on a row that is not a fade row, j or den
 * outside their range for the row's kind, an anchor that one row reads and another writes, or that two rows write.  rows may be
 * page-locked: the upload is then asynchronous, and the buffer must stay unchanged until the call's work on `stream` has completed
 * (a pageable buffer may be reused as soon as the call returns).  One launch.  Full symAD handle only; an out-of-range code index sets
 * the flag adec_index_error reads.  _bf16: zq is bf16, the fp32 result rounded once to nearest even; anchors and targets stay fp32. */
int adec_lookup_packed_playout(adec_handle *h, const uint8_t *packed, int F, const adec_playout_row *rows, int R, float *anchors,
                               int n_anchors, const float *targets, int n_targets, float *zq, void *stream);
int adec_lookup_packed_playout_bf16(adec_handle *h, const uint8_t *packed, int F, const adec_playout_row *rows, int R, float *anchors,
                                    int n_anchors, const float *targets, int n_targets, uint16_t *zq, void *stream);

/* -- the packed lookup of an adaptive playout clock (time scaling in the latent domain) ---------------------------------------------
 * adec_lookup_packed_playout with two more kinds of adec_playout_row, both starting from packed frame src of the same call instead of
 * an anchor (s_x is the fp32 lookup sum of packed frame x):
 *   between row (src >= 0, next >= 0, target = -1, slot = -1, 1 <= j < den):
 *     zq = fl(fl(fl(j / den) * fl(s_next - s_src)) + s_src), every operation rounded to nearest on its own (no contraction);
 *   frame-started fade (src >= 0, next = -1, target in [0, n_targets), slot = -1, j >= 1, den >= 1):
 *     the fade row with the anchor a replaced by s_src: zq = t when j >= den, otherwise fl(fl(fl(j / den) * fl(t - s_src)) + s_src).
 * s_src is what a real row of frame src stores as its anchor, so either row equals the anchor-read row of a later call bit for bit; a
 * receiver uses them when a concealed or fade frame follows, in the same call, the real frame that is its anchor.  Every other row is
 * adec_lookup_packed_playout's, bit for bit, with the same checks and the same conditions on the arguments; an error names the field.
 * One launch.  Full symAD handle only.  _bf16: zq is bf16, the fp32 result rounded once to nearest even. */
int adec_lookup_packed_timescale(adec_handle *h, const uint8_t *packed, int F, const adec_playout_row *rows, int R, float *anchors,
                                 int n_anchors, const float *targets, int n_targets, float *zq, void *stream);
int adec_lookup_packed_timescale_bf16(adec_handle *h, const uint8_t *packed, int F, const adec_playout_row *rows, int R, float *anchors,
                                      int n_anchors, const float *targets, int n_targets, uint16_t *zq, void *stream);

/* number of kernel launches issued by this handle since creation (bench.py's gpu_launches) */
int64_t adec_launch_count(const adec_handle *h);

/* -- graphed stream steps: one CUDA graph launch for the launches of a transmitter or receiver step ------------------------------
 * ADEC_GRAPH_TX (a = full or encoder-only symAD tx handle, b = NULL, T_or_F = samples per chunk):
 *   in x (B, 1, T) fp32 (bf16 when a has bf16 activations) -> adec_encode -> adec_quantize_ex -> out idx (Nq, B, F) int64, or with `wire` packed (B, F, bytes) uint8.
 * ADEC_GRAPH_RX (a = full symAD rx handle, b = any decoder handle, may equal a; T_or_F = frames per chunk):
 *   in idx (Nq, B, F) int64, or with `wire` packed (B, F, bytes) -> adec_lookup[_packed] -> adec_decode -> out y (B, F * hop), fp32, or
 *   bf16 when b has bf16 activations (compute_dtype 2; the lookup then writes bf16 zq itself, adec_lookup_bf16).
 * in and out are the caller's device buffers, fixed for the graph's life; the intermediate z / zq belongs to the graph.  B must equal
 * n_streams of the stateful handle (a for TX, b for RX).  Creating a graph sizes the workspaces and captures the step at both parities of
 * the double-buffered causal state on a private stream (thread-local capture mode); it runs nothing and leaves the handles' state, slot
 * bits, launch counts and diagnostics as they were (profiling, launch records and the kernel trace are off during the capture).
 * adec_graph_launch(g, stream) is the eager call sequence, bit for bit: outputs, causal state, flags and launch counts.  It launches the
 * executable of the current parity, instantiated the first time that parity is launched.  A launch first copies streams that slot calls
 * left in the other buffer back (as the uniform calls do), and captures again when a workspace or the state buffers were reallocated
 * since the capture.  While profiling, the kernel trace or launch records are on, it runs the eager sequence instead.
 * Stream capture happens only in adec_graph_create and in such a re-capturing launch.  CUDA forbids synchronising the device while a
 * stream is captured, so a program whose other threads synchronise creates its graphs before those threads run.
 * Errors are reported by adec_last_error(a) (create with a == NULL: adec_last_error(NULL)).  The handles must outlive the graph. */
enum { ADEC_GRAPH_TX = 0, ADEC_GRAPH_RX = 1 };
typedef struct adec_graph adec_graph;
int adec_graph_create(int kind, adec_handle *a, adec_handle *b, int B, int T_or_F, int wire, const void *in, void *out,
                      adec_graph **g);
int adec_graph_launch(adec_graph *g, void *stream);
/* kernels per step and programmatic (PDL) edges of the last capture, and the executables instantiated since creation */
int adec_graph_info(const adec_graph *g, int *kernels, int *programmatic_edges, int *instantiations);
int adec_graph_destroy(adec_graph *g);

/* Diagnostics (handles created with ADEC_KTRACE=1 in the environment): copies up to max_records {start ns, end ns, SM cycles} records
 * of the tensor-core conv launches issued since the last call (CTA 0's globaltimer / clock64) and resets the trace; returns the
 * number of records or -1.  Used to measure the effective SM clock and the gaps between back-to-back launches.  A library built with
 * -DADEC_PHASES writes records of 16 values instead of 3: the three above, then the per-phase cycle counters of the conv engine
 * (KT_REC in csrc/kernels.cuh, read by tools/conv_phases.py). */
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

/* The fp16-split MMA group of one 32-channel tap (three products, two K steps) as wgmma m64n64 and, on each 32-column half of the
 * same weights, as m64n32.  a: 2 x 4 x 64 x 8 fp16 (activation hi | lo, K block, row), b: 3 x 4 x 64 x 8 fp16 (weight plane, K block,
 * column); d64, d32: 64 x 64 fp32, row-major.  HOST pointers.  The paired RU(32) kernel relies on the two being equal bit for bit. */
int adec_test_wgmma_columns(int device, const void *a, const void *b, float *d64, float *d32);

/* One HiFi-GAN layer as a compute_dtype 1 / 2 handle runs it.  HOST pointers, channels-first like the other test entry points;
 * x, res, state and y are fp32 for compute_dtype 1 and bf16 words for 2.
 * kind 0: causal conv, w (Cout, Cin/groups, K), dilation dil, `groups` groups; shared_in: every group reads the same Cin/groups
 *         channels (MultiGroupConv1d's repeat, convs1.0), so x and state hold those Cin/groups channels; pre_act none /
 *         LeakyReLU(slope) / norm ((x - mean) / scale, mean and scale (Cin), groups = 1), the kernels' ACT_* codes; res (B, Cout, T)
 *         added after the bias, may be NULL.
 * kind 1: causal transposed conv, w (Cin, Cout, 2*up), LeakyReLU(slope) pre-activation; y (B, Cout, T*up).
 * kind 2: output head, w (1, 32, 7), LeakyReLU(slope) pre-activation, bias, tanh; y (B, 1, T).
 * bias may be NULL.  offline != 0: zero history and first-row replication in transposed convs (Generator.forward); state is neither
 * read nor written and may be NULL.  Otherwise state (B, Cin, P) is read and updated in place, as in adec_test_causal_conv. */
int adec_test_vocoder_layer(int device, int compute_dtype, int kind, const void *x, int B, int Cin, int T,
                            const float *w, const float *bias, int Cout, int K, int dil, int up, int groups, int shared_in,
                            int pre_act, float slope, const float *mean, const float *scale, const void *res, int offline,
                            void *state, void *y);

/* One op built by the model builders and run through the codec call path in any call mode, so that tests can check every row space
 * layer by layer: fp32-grade (the engine ADEC_CONV_PATH names) or, with compute_dtype 1 / 2, bf16.  HOST pointers, channels-first per
 * utterance. */
enum { ADEC_TEST_CONV = 0, ADEC_TEST_RU = 1, ADEC_TEST_CONVTR = 2, ADEC_TEST_STEM = 3, ADEC_TEST_HEAD = 4 };
typedef struct adec_test_op {
    int kind;          /* ADEC_TEST_*                                                                                              */
    int Cin, Cout;     /* conv: w (Cout, Cin/groups, K); RU: w (C, C, K) and w2 (C, C, 1), C = Cin = Cout; transposed conv:
                        * w (Cin, Cout, 2*stride); stem: w (32, 1, 7); head: w (1, 32, 7)                                           */
    int K, stride, dil, groups, shared_in;   /* conv: stride s > 1 needs K = 2s (the encoder's strided convs)                      */
    int pre_act;       /* the kernels' ACT_* codes: 0 none, 1 ELU, 2 LeakyReLU(slope), 3 norm ((x - mean) / scale, groups = 1)   */
    float slope;
    int out_nct;       /* conv: write channels-first, as the projector writes z                                                  */
    int post_tanh;     /* head: tanh after the conv                                                                             */
    const float *w, *w2, *bias, *mean, *scale;   /* bias, mean, scale may be NULL                                             */
    int compute_dtype; /* 0: the fp32-grade engine ADEC_CONV_PATH names; 1 / 2: the op as a symAD decoder-only handle with that
                        * compute_dtype builds it (f16 engine; the stem keeps fp32 weights): x, res, state and y are fp32 for 0 and 1 and
                        * bf16 words for 2                                                                                          */
} adec_test_op;
/* launch records: 9 ints {launch kind, NT (FFMA: output tile), fuse, pre_act, prec (wg_conv.cuh PREC_*), varlen, paired, stacked,
 * bf16 storage (BST)} */
enum { ADEC_TEST_REC = 9, ADEC_TEST_LAUNCH_TC = 0, ADEC_TEST_LAUNCH_FFMA = 1, ADEC_TEST_LAUNCH_STEM = 2, ADEC_TEST_LAUNCH_HEAD = 3 };
/* mode: 0 = stream (adec_encode: B = n_streams streams advanced by equal lengths, stacked rows unless ADEC_STACK_ROWS=0), 1 = offline
 * (zero history, first-row replication in transposed convs), 2 = varlen offline, 3 = stream slots (`streams`: the B distinct streams of
 * n_streams that each call advances).  n_calls consecutive calls on one handle: lengths (n_calls, B) are input rows per utterance
 * (equal within a call in modes 0 and 1), streams (n_calls, B).  x: every call's utterances one after the other, each (Cin_x, L)
 * where Cin_x = Cin (shared_in: Cin / groups; stem: 1).  y: the same for the outputs, each (Cout, Tout * stride) for a transposed conv,
 * (Cout, (L - 1) / stride + 1) otherwise (head: 1 channel; stem: 32).  res: NULL, or a conv's residual, laid out like y, added after
 * the bias.  state (n_streams, Cin_x, P): the initial history of every stream (modes 0 and 3; may be NULL in modes 1 and 2), and on
 * return each stream's current state (not written in mode 2).  launched: NULL, or room for max_launched records; the launches of all
 * calls are written in order and the rest of the array is set to -1.  A split residual unit (C above ADEC_TC_MAXFUSE on the tensor-core
 * engines) runs as its two launches.  range_flag: NULL, or two ints: adec_range_error after the calls, then read once more (the
 * flag's report-once protocol). */
int adec_test_conv_op(int device, const adec_test_op *op, int mode, int n_calls, int B, int n_streams, const int *lengths,
                      const int *streams, const float *x, const float *res, float *state, float *y, int *launched, int max_launched,
                      int *range_flag);

/* Launch records of a model handle, in the format above: adec_record_launches(h, 1) clears the record and starts appending one
 * record per conv / stem / head launch of every later call, (h, 0) stops.  adec_launch_records copies up to max_records of them and
 * returns how many there are (-1 on error).  Tests use it to list the kernel instantiations the shipped plans select. */
int adec_record_launches(adec_handle *h, int enable);
int adec_launch_records(const adec_handle *h, int *out, int max_records);

#ifdef __cplusplus
}
#endif
#endif /* AUDIODEC_B200_H */
