/*
 * lyra_b200 — C ABI of the H100-native Lyra v1.3.2 hot path.
 *
 * This is the seam that replaces `TfLiteModelWrapper` (reference: lyra/tflite_model_wrapper.h:32-67)
 * underneath the three plugin classes bound in lyra/lyra_components.cc:42-55.  Plain pointers and
 * sizes only; the caller owns every buffer; one context per GPU; calls on one context must be
 * serialised by the caller.  Stream ids are integers in [0, max_streams): each id owns the
 * per-stream convolution state that a SoundStreamEncoder / LyraGanModel object owns in the
 * reference (TFLite resource variables, zero-initialised).
 *
 * Return value: 0 on success, a negative LYRA_B200_E* code otherwise.  A failing call maps onto the
 * reference's `std::nullopt` / `false` / `nullptr` conventions (SURVEY.md §8b); it never aborts.
 * There is NO CPU fallback: without a CUDA device lyra_b200_create fails with LYRA_B200_ENODEV.
 */
#ifndef LYRA_B200_H_
#define LYRA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LYRA_B200_OK 0
#define LYRA_B200_EINVAL (-1) /* bad argument: sample/feature count, bit count, stream id, duplicate id */
#define LYRA_B200_ENODEV (-2) /* no CUDA device or a CUDA runtime failure */
#define LYRA_B200_EMODEL (-3) /* model files missing, wrong version or unexpected graph structure */

#define LYRA_B200_HOP 320          /* samples per 20 ms hop at 16 kHz (lyra/lyra_config.h:70-73) */
#define LYRA_B200_NUM_FEATURES 64  /* lyra/lyra_config.cc:36 */
#define LYRA_B200_MAX_BITS 184     /* lyra/residual_vector_quantizer.h:50 */
#define LYRA_B200_MAX_STAGES 46

typedef struct lyra_b200_ctx lyra_b200_ctx;

/* Replaces {SoundStreamEncoder,ResidualVectorQuantizer,LyraGanModel}::Create
 * (lyra/soundstream_encoder.cc:36-46, lyra/residual_vector_quantizer.cc:36-67, lyra/lyra_gan_model.cc:36-46)
 * and the asset/version gate of AreParamsSupported (lyra/lyra_config.h:119-168): loads the three
 * .tflite files + lyra_config.binarypb from `model_dir`, uploads weights, allocates the state of
 * `max_streams` streams on CUDA device `device`.  *out is NULL on failure.
 * Every call that takes a context makes that context's device the calling thread's current CUDA device (the current
 * device is per host thread; worker threads need not set it themselves). */
int lyra_b200_create(const char* model_dir, int device, int max_streams, lyra_b200_ctx** out);
/* The same with a choice of roles.  LyraEncoder and LyraDecoder are separate objects in the reference
 * (lyra/lyra_encoder.h:112-120, lyra/lyra_decoder.h:130-160) and a full-duplex server drives them independently: an
 * encoder-only and a decoder-only context hold only their half of the streaming state and may be called concurrently
 * (one host thread / one CUDA stream each), so the uplink's encode kernels overlap the downlink's decode kernels on the
 * GPU.  Calls that need a role the context lacks return LYRA_B200_EINVAL; quantize / dequantize / logmel / noise_update /
 * cng_generate are stateless or self-contained and work in any context. */
#define LYRA_B200_ROLE_ENCODER 1
#define LYRA_B200_ROLE_DECODER 2
int lyra_b200_create_ex(const char* model_dir, int device, int max_streams, int roles, lyra_b200_ctx** out);
void lyra_b200_destroy(lyra_b200_ctx* ctx);
/* Human-readable reason of the last failure on this context (or of the last failed create when ctx is NULL). */
const char* lyra_b200_last_error(const lyra_b200_ctx* ctx);
int lyra_b200_max_streams(const lyra_b200_ctx* ctx);
int lyra_b200_tile_streams(const lyra_b200_ctx* ctx);

/* Replaces TfLiteModelWrapper::ResetVariableTensors (lyra/tflite_model_wrapper.cc:111-113) per stream:
 * encoder, decoder and log-mel state of the listed streams go back to the initial (zero) state.
 * stream_ids == NULL resets streams 0..n-1. */
int lyra_b200_reset(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n);

/* ---- fused codec calls: host buffers in, host buffers out ------------------------------------------ */

/* LyraEncoder::Encode at 16 kHz without DTX (lyra/lyra_encoder.cc:113-156) for n streams:
 * pcm[n][320] -> packets[n][ceil(num_bits/8)].  num_bits in {64,120,184} or any multiple of 4 <= 184.
 * stream_ids == NULL means streams 0..n-1. */
int lyra_b200_encode(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int16_t* pcm, int num_bits,
                     uint8_t* packets);

/* LyraDecoder::SetEncodedPacket + DecodeSamples(320) in the no-fade paths (lyra/lyra_decoder.cc:172-226,
 * 317-326): packets[n][ceil(num_bits/8)] -> pcm[n][320].  received[i] == 0 marks a lost packet: the
 * generative model is then fed 64 zero features (ZeroFeatureEstimator).  received == NULL: all received. */
int lyra_b200_decode(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const uint8_t* packets,
                     const uint8_t* received, int num_bits, int16_t* pcm);

/* ---- the plugin surface, call by call --------------------------------------------------------------- */

/* FeatureExtractorInterface::Extract as implemented by SoundStreamEncoder
 * (lyra/feature_extractor_interface.h:32-39, lyra/soundstream_encoder.cc:53-64): pcm[n][320] -> features[n][64]. */
int lyra_b200_extract_features(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int16_t* pcm, float* features);

/* VectorQuantizerInterface::Quantize + PacketInterface::PackQuantized
 * (lyra/vector_quantizer_interface.h:28-41, lyra/residual_vector_quantizer.cc:77-110, lyra/packet.h:56-60):
 * features[n][64] -> packets[n][ceil(num_bits/8)] and, if indices != NULL, indices[n][46] (-1 for unused
 * stages, the graph's output_0).  Stateless.  LYRA_B200_EINVAL for num_bits > 184 or num_bits % 4 != 0. */
int lyra_b200_quantize(lyra_b200_ctx* ctx, int n, const float* features, int num_bits, uint8_t* packets, int32_t* indices);

/* PacketInterface::UnpackPacket + VectorQuantizerInterface::DecodeToLossyFeatures
 * (lyra/packet.h:62-71, lyra/residual_vector_quantizer.cc:112-168): packets -> features[n][64].  Stateless. */
int lyra_b200_dequantize(lyra_b200_ctx* ctx, int n, const uint8_t* packets, int num_bits, float* features);

/* GenerativeModel::RunConditioning + RunModel(320) as implemented by LyraGanModel
 * (lyra/generative_model_interface.h:62-101, lyra/lyra_gan_model.cc:53-64): features[n][64] -> pcm[n][320]. */
int lyra_b200_generate(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const float* features, int16_t* pcm);

/* LogMelSpectrogramExtractorImpl::Extract for (16 kHz, hop 320, window 640)
 * (lyra/log_mel_spectrogram_extractor_impl.cc:96-126): pcm[n][320] -> out[n][num_mel_bins];
 * num_mel_bins is 160 (NoiseEstimator's extractor, lyra/lyra_config.cc:37) or 64 (integration test).
 * `bank` (0 or 1) selects which of the two independent per-stream extractor states is advanced
 * (the reference creates one extractor object per use). */
int lyra_b200_logmel(lyra_b200_ctx* ctx, int bank, const int32_t* stream_ids, int n, const int16_t* pcm,
                     int num_mel_bins, float* out);

/* NoiseEstimator::ReceiveSamples(one whole hop) + is_noise() + noise_estimate() (lyra/noise_estimator.h:44-62,
 * lyra/noise_estimator.cc:144-245; 160 features, the decoder's configuration lyra/lyra_decoder.cc:98-104), one
 * estimator per stream with its own log-mel extractor.  pcm[n][320] is the decoded hop; update_mask[n] (NULL = all
 * ones) is 1 for streams whose hop came from a received packet: only those feed the estimator
 * (LyraDecoder::DecodeSamplesInternal, lyra/lyra_decoder.cc:306-311), the others only report.  Outputs (either may
 * be NULL): is_noise[n] (1 = the last fed hop was classified as noise; 1 for a fresh estimator) and
 * noise_estimate[n][160].  State is cleared by lyra_b200_reset. */
int lyra_b200_noise_update(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int16_t* pcm,
                           const uint8_t* update_mask, uint8_t* is_noise, float* noise_estimate);

/* lyra_b200_decode followed, on the device and per sub-batch, by the noise-estimator update of every stream whose
 * packet was received — what LyraDecoder::DecodeSamplesInternal does after RunGenerativeModel
 * (lyra/lyra_decoder.cc:306-311) — without moving the decoded audio or the 160-bin spectra off the GPU.
 * is_noise[n] may be NULL; the estimate itself is read with lyra_b200_noise_update(update_mask = zeros). */
int lyra_b200_decode_track_noise(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const uint8_t* packets,
                                 const uint8_t* received, int num_bits, int16_t* pcm, uint8_t* is_noise);

/* NoiseEstimator::noise_estimate() / is_noise() of the decoder-side estimators without feeding them (read-only;
 * lyra/noise_estimator.h:55-62).  Either output may be NULL. */
int lyra_b200_noise_estimate(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, float* noise_estimate, uint8_t* is_noise);

/* ---- packet-loss concealment, comfort noise and DTX (SURVEY.md section 8 rows f2, f4) ------------------------------ */

/* LyraDecoder::SetEncodedPacket (for streams with received[i] != 0) + DecodeSamples(320) with the reference's full behaviour
 * (lyra/lyra_decoder.cc:172-315, 342-383): up to 80 ms of a lost stream are concealed by the generative model on zero
 * features, then the output cross-fades (raised cosine, 40 ms) into comfort noise synthesised from the stream's noise
 * estimate, and fades back when packets return; the noise estimator is fed by hops decoded from received packets only.
 * Per-stream control state (concealment progress, fade progress, fade direction) lives on the device; one call = one 20 ms
 * tick of every listed stream.  is_comfort_noise[n] (may be NULL) = LyraDecoder::is_comfort_noise() after the tick.
 * Requests that are not whole hops are served by the C++ adapter LyraDecoderB200 (include/lyra_b200/lyra_b200_components.h),
 * which runs the same state machine on the host over lyra_b200_generate / lyra_b200_cng_generate. */
int lyra_b200_decode_plc(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const uint8_t* packets, const uint8_t* received,
                         int num_bits, int16_t* pcm, uint8_t* is_comfort_noise);
/* The control state of the listed streams, state[n][3] = {concealment_progress, fade_progress, fade_direction (-1 = from, +1 =
 * to comfort noise)} - what the reference's test peer exposes (lyra/lyra_decoder_test.cc:56-90).  set accepts hop-aligned
 * values only. */
int lyra_b200_plc_get_state(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, int32_t* state);
int lyra_b200_plc_set_state(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int32_t* state);

/* ComfortNoiseGenerator::RunConditioning + RunModel(320) (lyra/comfort_noise_generator.cc:74-119) for n streams:
 * features[n][160] (log-mel, e.g. a noise estimate) -> pcm[n][320].  Every stream owns an overlap-add buffer and a hop
 * counter (cleared by lyra_b200_reset).  The reference draws random phases from an unseeded generator (:103); here the phase
 * of bin i of hop h of stream s is a pure function of (seed + s, h, i) - reproducible, see oracle/comfort_noise.c. */
int lyra_b200_cng_generate(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const float* features, int16_t* pcm);
int lyra_b200_set_cng_seed(lyra_b200_ctx* ctx, uint64_t seed);   /* default 0 */

/* LyraEncoder::Encode with enable_dtx (lyra/lyra_encoder.cc:113-156): every hop first updates the stream's encoder-side noise
 * estimator; a hop classified as noise is not encoded (the stream's encoder state does not advance) and yields an EMPTY packet:
 * packet_bytes[i] = 0 (its bytes in `packets` are zero), otherwise ceil(num_bits / 8). */
int lyra_b200_encode_dtx(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int16_t* pcm, int num_bits, uint8_t* packets,
                         int32_t* packet_bytes);

/* Resampler::Resample (lyra/resampler.cc:31-66, audio_dsp::QResampler with a kernel radius of 17 input samples, started fully
 * primed) for n streams: to_internal != 0 converts `external_rate_hz` (8000 / 32000 / 48000) to the codec's 16 kHz (LyraEncoder's
 * input side, lyra_encoder.cc:58-66,118-122), to_internal == 0 converts 16 kHz to the external rate (LyraDecoder's output side,
 * lyra_decoder.cc:108-114).  in[n][in_samples] -> out[n][out_stride]; out_counts[n] (may be NULL) = samples produced per stream
 * (in_samples * out / in, +-1 when down-sampling from an odd phase); at most 960 input and 960 output samples per stream and call.  Each stream owns a delay line and phase per direction,
 * cleared by lyra_b200_reset; a call at a different rate restarts that stream's filter. */
int lyra_b200_resample(lyra_b200_ctx* ctx, int to_internal, const int32_t* stream_ids, int n, int external_rate_hz, const int16_t* in,
                       int in_samples, int16_t* out, int out_stride, int32_t* out_counts);

/* ---- device-resident variants (pointers are CUDA device pointers; asynchronous on the context's
 *      stream; streams 0..n-1).  Used by bench.py for the HBM-resident `value` measurement and by
 *      callers that keep audio on the GPU. ---------------------------------------------------------- */
int lyra_b200_set_stream(lyra_b200_ctx* ctx, void* cuda_stream); /* NULL restores the context's own stream */
int lyra_b200_encode_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets);
int lyra_b200_decode_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received,
                            int num_bits, int16_t* d_pcm);
int lyra_b200_decode_track_noise_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received,
                                        int num_bits, int16_t* d_pcm, uint8_t* d_is_noise);
int lyra_b200_noise_update_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, const uint8_t* d_update_mask,
                                  uint8_t* d_is_noise, float* d_noise_estimate);
int lyra_b200_decode_plc_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                                int16_t* d_pcm, uint8_t* d_is_comfort_noise /* may be NULL */);
int lyra_b200_encode_dtx_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets,
                                uint8_t* d_is_noise /* [n], 1 = empty packet */);
int lyra_b200_synchronize(lyra_b200_ctx* ctx);
/* Dense calls (stream_ids == NULL / *_device) over many tiles are cut into `parts` (1..4, default 3) sub-batches that
 * run concurrently on internal CUDA streams so partial waves of one kernel are filled by another's blocks.
 * parts = 1 serialises the kernels (used by bench.py's per-kernel roofline pass). */
int lyra_b200_set_split(lyra_b200_ctx* ctx, int parts);
/* Arithmetic of the decoder's fp32 convolutions (decoder_1, decoder_2/simple, decoder_2, last_layer of lyragan.tflite):
 *   LYRA_B200_DECODER_EXACT  (default) every output is one fp32 fmaf chain in the canonical order: decoded PCM is
 *                            bit-identical to the CPU restatement of the reference graph;
 *   LYRA_B200_DECODER_TENSOR the same layers as split-precision TF32 tensor-core MMAs (fp32-level accuracy, different
 *                            rounding): decoded PCM stays within a few int16 LSB of the exact mode (bound stated and
 *                            tested in tests/test_gpu_parity.py), well inside the 1e-3 full-scale tolerance the
 *                            drop-in target allows.  The encoder, the quantizer and every int8 layer are exact in
 *                            both modes, so packets / RVQ indices never depend on this switch.
 * The reference has one arithmetic (TFLite's, lyra/lyra_gan_model.cc:53-64); this switch is an extension. */
#define LYRA_B200_DECODER_EXACT 0
#define LYRA_B200_DECODER_TENSOR 1
int lyra_b200_set_decoder_mode(lyra_b200_ctx* ctx, int mode);
int lyra_b200_decoder_mode(const lyra_b200_ctx* ctx);
/* How the synchronous host-buffer calls wait for the GPU: 0 (default) spins (lowest latency), 1 sleeps on a blocking-sync
 * CUDA event — for servers that run more waiting worker threads than they have cores. */
int lyra_b200_set_blocking_sync(lyra_b200_ctx* ctx, int enable);
/* CUDA priority of the context's own stream and of its sub-batch streams (0 = default, negative = higher; the device clamps).
 * A process that runs an encoder-only and a decoder-only context side by side through the asynchronous *_device calls can
 * run the encoder one step above the decoder (the uplink chain is the longer one; its blocks go first, the decoder's
 * latency-bound blocks fill what is left); with the synchronous host-buffer calls equal priorities are the better choice
 * (DESIGN.md section 6).  Waits for the context's work, re-creates the streams, drops captured
 * graphs.  A caller stream installed with lyra_b200_set_stream keeps its own priority.  Default 0, or the environment
 * variables LYRA_B200_ENC_PRIORITY / LYRA_B200_DEC_PRIORITY at creation. */
int lyra_b200_set_priority(lyra_b200_ctx* ctx, int priority);
/* CUDA graphs for the synchronous host-buffer calls lyra_b200_encode / lyra_b200_decode (no reference counterpart): with
 * enable = 1 a dense call (stream_ids == NULL) whose host buffers are page-locked is captured once - copies in, every
 * sub-batch's kernels, copies out - and later calls with the same n, num_bits and buffers replay the graph (one launch instead
 * of ~20 stream operations; matters for small batches).  Results are identical; anything that cannot be captured runs directly.
 * Default 0.  lyra_b200_graph_replays counts the calls served by a replay. */
int lyra_b200_set_graphs(lyra_b200_ctx* ctx, int enable);
uint64_t lyra_b200_graph_replays(const lyra_b200_ctx* ctx);
/* number of CUDA kernels this context has launched so far */
uint64_t lyra_b200_launch_count(const lyra_b200_ctx* ctx);

/* ---- diagnostics: per-kernel device time measured with CUDA events on the launching stream.
 *      Kernel order: 0 EncoderKernelA, 1 EncoderKernelB, 2 RvqEncodeKernel, 3 RvqDecodeKernel,
 *      4 DecoderKernelC, 5 DecoderKernelD, 6 LogMelKernel, 7 NoiseEstimatorKernel.  profile_read synchronises the stream and
 *      returns the accumulated milliseconds / launch counts since profiling was enabled. */
#define LYRA_B200_NUM_KERNELS 8
int lyra_b200_profile_enable(lyra_b200_ctx* ctx, int enable);
int lyra_b200_profile_read(lyra_b200_ctx* ctx, double* ms_sum, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LYRA_B200_H_ */
