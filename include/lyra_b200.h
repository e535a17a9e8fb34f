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
/* Streams per tile, the unit of work of one thread block in the conv-net kernels: 8 (0 when ctx is NULL). */
int lyra_b200_tile_streams(const lyra_b200_ctx* ctx);

/* Replaces TfLiteModelWrapper::ResetVariableTensors (lyra/tflite_model_wrapper.cc:111-113) per stream: every piece of
 * per-stream state of the listed streams goes back to its state at creation - the encoder and decoder networks' state,
 * both log-mel extractor banks of lyra_b200_logmel, the decoder-side and the encoder-side (DTX) noise estimators with their
 * extractors, the packet-loss control state (no concealment, fading from comfort noise), the comfort-noise generators'
 * overlap-add buffers and hop counters, both directions of lyra_b200_resample and the codec calls' own sample-rate converters
 * (lyra_b200_set_sample_rate; the next call restarts each converter fully primed).  The context's sample rate is kept.
 * stream_ids == NULL resets streams 0..n-1; an id may be listed more than once.  Ordered on the context's stream (see
 * lyra_b200_set_stream) behind the work already queued there; returns when the reset is done. */
int lyra_b200_reset(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n);

/* ---- moving streams: between ids of one context, between contexts, between GPUs and processes ----------------------
 * A stream's state is everything lyra_b200_reset restores plus lyra_b200_resample's delay lines (which reset keeps): the
 * networks' state and hop counters, the log-mel banks, both noise estimators, the packet-loss control state, the comfort-noise
 * generator (overlap-add buffer, hop counter and its phase key), both directions of lyra_b200_resample and the codec calls'
 * converters.  A moved stream continues exactly as it would have at its old id - comfort noise included, when both contexts
 * have the same lyra_b200_set_cng_seed.  Host-side state of the C++ adapters (include/lyra_b200/) is not part of it.
 *
 * Bytes of one stream's state record in this context (it depends on the context's roles); 0 when ctx is NULL. */
int lyra_b200_stream_state_bytes(const lyra_b200_ctx* ctx);
/* records[n][lyra_b200_stream_state_bytes]: the complete state of the listed streams (stream_ids == NULL: 0..n-1; an id may be
 * listed more than once).  A record holds a header (format, roles, sample rate, a fingerprint of the loaded model) and the
 * state.  Ordered on the installed stream behind the work queued there; returns when the records are in the caller's buffer. */
int lyra_b200_export_streams(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, void* records);
/* The inverse of export, into this context's streams stream_ids[k] (NULL: 0..n-1; distinct).  Every record is validated first:
 * a record of another format, roles, sample rate or model, or a damaged one, fails the whole call with LYRA_B200_EINVAL and no
 * stream changes.  Records may come from a context in the other decoder mode (the modes share their state); the stream then
 * continues in this context's mode.  Ordered on the installed stream; returns when done. */
int lyra_b200_import_streams(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const void* records);
/* Within one context: afterwards stream dst_ids[k] holds the state stream src_ids[k] had before the call; src_ids[k] == -1 is
 * the state at creation (what lyra_b200_reset gives).  Sources keep their state.  Asynchronous like the *_device calls: queued
 * on the installed stream, no host synchronisation.  LYRA_B200_EINVAL for ids out of range, a repeated id within src_ids (-1
 * excepted) or within dst_ids, or an id that is both a source and a destination.  With it a server keeps its live calls on
 * streams 0..n-1 of the *_device calls: when the call on stream h ends it copies stream n-1 into h and shrinks n. */
int lyra_b200_copy_streams(lyra_b200_ctx* ctx, const int32_t* src_ids, const int32_t* dst_ids, int n);
/* Afterwards each network hop counter of stream stream_ids[k] equals the matching counter of stream like_ids[k] (-1: counter 0,
 * the phase at creation): encoder entries in a context with the encoder role, decoder entries in one with the decoder role.
 * The stream's depthwise rings are rotated to match, so its later outputs (packets, PCM, comfort-noise flags, control state, in
 * both decoder modes) are bit-identical to what it would have produced without the call; every other piece of its state stays
 * as it is.  A hop counter only decides where each ring starts, but the conv-net kernels take their fast depthwise path only
 * on a tile whose active streams share one counter: a server aligns a moved or newly admitted stream like a live neighbour
 * of its tile, and may periodically align a whole tile to one of its lanes (streams that sit out hops, DTX or comfort noise,
 * fall behind their neighbours).  n == 0 does nothing.  LYRA_B200_EINVAL, with nothing queued or changed, for a NULL list
 * with n > 0, ids out of range, a repeated id within stream_ids, or an id in both lists; like_ids may repeat.  Asynchronous
 * like lyra_b200_copy_streams: queued on the installed stream, no host synchronisation, captured graphs stay valid. */
int lyra_b200_align_streams(lyra_b200_ctx* ctx, const int32_t* stream_ids, const int32_t* like_ids, int n);

/* ---- fused codec calls: host buffers in, host buffers out ------------------------------------------ */

/* The external sample rate of the fused codec calls (LyraEncoder::Create / LyraDecoder::Create's sample_rate_hz,
 * lyra/lyra_config.h:56): 8000, 16000 (default), 32000 or 48000; any other rate returns LYRA_B200_EINVAL and leaves the setting
 * unchanged.  The reference fixes the rate per encoder / decoder object; here it is the context's rate: it sets the row length
 * of the calls below and puts every stream at that rate.  Streams may then run at lower rates of their own
 * (lyra_b200_set_stream_sample_rates), so one context serves 8, 16, 32 and 48 kHz calls side by side.
 *   Calls that follow it: lyra_b200_encode, _encode_dtx, _decode, _decode_track_noise, _decode_plc and their *_device twins.
 *   Their PCM rows hold sample_rate_hz / 50 samples (one 20 ms hop at the external rate): input of the encoders, output of the
 *   decoders.  Packets, masks, flags and packet_bytes do not change.  Internally the codec runs at 16 kHz: the encoder role
 *   converts its input to 16 kHz (lyra/lyra_encoder.cc:58-66,118-122) before everything else, DTX included; the decoder role
 *   converts its 16 kHz output to the external rate (lyra/lyra_decoder.cc:108-114) after everything else.  Each stream owns one
 *   converter per role, separate from lyra_b200_resample's.  The encoder-side DTX estimator is built for the external rate as in
 *   the reference (NoiseEstimator::Create(sample_rate_hz, 320, 640, 160), lyra/lyra_encoder.cc:80-89: its mel bank and time
 *   constants follow the rate) and fed the 16 kHz hop; the decoder-side estimator and comfort noise stay at 16 kHz.
 *   Calls that ignore it: the plugin-level 16 kHz components extract_features, quantize, dequantize, generate, logmel,
 *   noise_update, noise_estimate, cng_generate, and resample.
 * At 16000 nothing is converted (unless a stream has a rate of its own).  Setting the current rate when no stream has a rate of
 * its own does nothing.  A change waits for the context's queued work and drops captured graphs (like lyra_b200_set_priority).
 * Every stream is at the new rate afterwards.  Streams keep their codec state (networks, estimators, packet-loss state); each
 * stream whose rate changed restarts its converters fully primed on its next call, like a fresh Resampler.  A caller that wants
 * a brand-new LyraEncoder / LyraDecoder also calls lyra_b200_reset. */
int lyra_b200_set_sample_rate(lyra_b200_ctx* ctx, int sample_rate_hz);
int lyra_b200_sample_rate(const lyra_b200_ctx* ctx);
/* Per-stream rates, one LyraEncoder / LyraDecoder pair per call at its own rate: stream stream_ids[k] (NULL: streams 0..n-1)
 * runs the fused calls at rates_hz[k], one of 8000, 16000, 32000, 48000 and at most the context's rate (its hop must fit in the
 * row).  In every fused call and *_device twin a stream at rate r uses the first r / 50 samples of its row: the encoders ignore
 * the rest, the decoders write it as 0.  The encoder-side DTX estimator follows the stream's rate; the decoder side stays at
 * 16 kHz.  An unsupported rate, a rate above the context's or a repeated id returns LYRA_B200_EINVAL and changes nothing.
 * Works in any context.  Asynchronous like lyra_b200_copy_streams: queued on the installed stream, no host synchronisation, so
 * a server admits a call with copy_streams(-1 -> slot) followed by its rate without draining.  A stream whose rate changes keeps
 * its codec state, and its converters restart fully primed on its next call; setting a stream to the rate it has changes
 * nothing.  lyra_b200_reset and copy_streams from -1 put a stream back at the context's rate; copy, export and import carry a
 * stream's rate with it (a record still holds the context's rate and import still refuses another one).
 * The rates are read on the device, so changing them does not invalidate captured graphs; the first stream given a rate of its
 * own at 16 kHz adds the converters' launches to the calls, which then capture graphs of their own (lyra_b200_set_graphs). */
int lyra_b200_set_stream_sample_rates(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int32_t* rates_hz);
/* rates_hz[k] = the rate stream stream_ids[k] (NULL: k) runs at; an id may be listed more than once.  Ordered on the installed
 * stream behind the work queued there; returns when done. */
int lyra_b200_stream_sample_rates(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, int32_t* rates_hz);
/* Per-stream bit rates: the stream's own bit count in one role, i.e. the bit rate of its LyraEncoder (LyraEncoder::set_bitrate,
 * lyra/lyra_encoder.cc:158-166) or of the packets its LyraDecoder receives (lyra/lyra_decoder.cc:172-184,
 * lyra/lyra_config.h:99-115).  role is LYRA_B200_ROLE_ENCODER or LYRA_B200_ROLE_DECODER and must be a role of the context; the
 * two words of a stream are independent.  bits[k] is 0 (follow the call's num_bits) or a bit count the calls accept: a multiple
 * of 4 in 4..184.
 *   In the fused calls and their *_device twins num_bits keeps its meaning for streams whose word is 0 and sets the packet row
 *   stride, ceil(num_bits / 8).  A stream with its own count b: the encoders write its packet at b bits into the first
 *   ceil(b / 8) bytes of its row and zeros over the rest; lyra_b200_encode_dtx reports packet_bytes 0 or ceil(b / 8); the
 *   decoders read a received packet as b bits from the first ceil(b / 8) bytes of its row and ignore the rest.  Lost packets,
 *   DTX and comfort noise behave as before.  A call returns LYRA_B200_EINVAL and queues nothing when a stream it lists has its
 *   own count above the call's num_bits; streams it does not list do not constrain it.
 *   quantize / dequantize ignore the words.
 * Changing a word between hops is LyraEncoder::set_bitrate: the next packet comes out at the new size, and the networks,
 * estimators and hop counters carry on.  A bad count, a role the context lacks (or not exactly one role), an id out of range or
 * a repeated id returns LYRA_B200_EINVAL and changes nothing.  Asynchronous like lyra_b200_set_stream_sample_rates: queued on
 * the installed stream, no host synchronisation.  lyra_b200_reset and copy_streams from -1 set both words to 0; copy, export and
 * import carry them.  A context in which no stream has its own count launches exactly what it launches without this call. */
int lyra_b200_set_stream_bits(lyra_b200_ctx* ctx, int role, const int32_t* stream_ids, int n, const int32_t* bits);
/* bits[k] = the word of stream stream_ids[k] (NULL: k) in `role` (0: it follows the call); an id may be listed more than once.
 * Ordered on the installed stream behind the work queued there; returns when done. */
int lyra_b200_stream_bits(lyra_b200_ctx* ctx, int role, const int32_t* stream_ids, int n, int32_t* bits);
/* Per-stream DTX: LyraEncoder::Create's enable_dtx (lyra/lyra_encoder.cc:79-89, 131-141) per stream, so one encoder context
 * serves DTX and non-DTX calls side by side.  enable[k] is 1 (the default, at creation) or 0 for stream stream_ids[k] (NULL:
 * streams 0..n-1).  Only a context with the encoder role accepts these calls.
 *   lyra_b200_encode_dtx and lyra_b200_encode_dtx_device treat a stream with 0 exactly like a LyraEncoder created with
 *   enable_dtx = false: its encoder-side noise estimator (and that estimator's log-mel extractor) is not fed, its hop is always
 *   encoded, its flag is 0 and its packet_bytes is ceil(b / 8), b its own bit count (lyra_b200_set_stream_bits) or the call's
 *   num_bits.  Per-stream sample rates and bit counts apply as usual.  lyra_b200_encode and lyra_b200_encode_device ignore the
 *   setting.
 *   0 -> 1 restarts the stream's encoder-side estimator and its extractor's carried samples at their creation state (a fresh
 *   NoiseEstimator::Create); 1 -> 0 leaves them as they are (they are not read while DTX is off); setting the value a stream
 *   already has does nothing.  Networks, hop counters, converters and bit counts always carry on.
 * enable == NULL, a value other than 0 or 1, an id out of range, a repeated id or a context without the encoder role returns
 * LYRA_B200_EINVAL and queues or changes nothing.  Asynchronous like lyra_b200_set_stream_bits: queued on the installed stream,
 * no host synchronisation, captured graphs stay valid.  lyra_b200_reset and copy_streams from -1 turn DTX back on; copy, export
 * and import carry the setting.  A context in which DTX was never turned off launches exactly what it launches without this call,
 * and turning it off changes no launch count. */
int lyra_b200_set_stream_dtx(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int32_t* enable);
/* enable[k] = the DTX setting of stream stream_ids[k] (NULL: k); an id may be listed more than once.  Ordered on the installed
 * stream behind the work queued there; returns when done. */
int lyra_b200_stream_dtx(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, int32_t* enable);

/* LyraEncoder::Encode without DTX (lyra/lyra_encoder.cc:113-156) for n streams:
 * pcm[n][sample_rate / 50] -> packets[n][ceil(num_bits/8)] (pcm[n][320] at the default 16 kHz; lyra_b200_set_sample_rate).
 * num_bits in {64,120,184} or any multiple of 4 <= 184.
 * stream_ids == NULL means streams 0..n-1. */
int lyra_b200_encode(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int16_t* pcm, int num_bits,
                     uint8_t* packets);

/* LyraDecoder::SetEncodedPacket + DecodeSamples(320) in the no-fade paths (lyra/lyra_decoder.cc:172-226,
 * 317-326): packets[n][ceil(num_bits/8)] -> pcm[n][sample_rate / 50].  received[i] == 0 marks a lost packet: the
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
 * of bin i of hop h of stream s is a pure function of (seed + s, h, i) - reproducible, see oracle/comfort_noise.c.  (A stream
 * moved by lyra_b200_import_streams / lyra_b200_copy_streams keeps the key of its old id.) */
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
 *      callers that keep audio on the GPU.  A call does not wait for the work it queues or for earlier
 *      work on the installed stream, reads its inputs and writes its outputs only in stream order on the installed stream, and
 *      touches no row outside [0, n) of the caller's buffers (so several contexts may work on slices of one
 *      buffer).  Role checks are those of the host-buffer twins: noise_update_device works in any context.  The codec
 *      calls' PCM rows hold sample_rate / 50 samples (lyra_b200_set_sample_rate); noise_update_device's stay 320. ---- */
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
/* The plugin surface on device memory: the twins of extract_features, quantize, dequantize, generate, logmel, noise_estimate,
 * cng_generate and resample, for a caller that keeps features, packets, spectra or audio on the GPU between its own stages (for
 * example its own model in place of one Lyra component).  Each takes the arguments, row sizes and return codes of its host-buffer
 * twin, with streams 0..n-1 and every buffer a device pointer, and has the contract above: queued on the installed stream, no
 * host wait, rows [0, n) only, LYRA_B200_EINVAL with nothing queued for a bad argument.  Role checks are the twins':
 * extract_features_device needs the encoder role, generate_device the decoder role, the others work in any context.  Like their
 * twins they run at 16 kHz on 320-sample rows (lyra_b200_set_sample_rate and the per-stream rate, bits and DTX words do not apply)
 * and advance the same state: the encoder or decoder networks and hop counters, the chosen log-mel bank, the comfort-noise
 * generators (lyra_b200_set_cng_seed and the streams' keys apply), the resampler's delay lines of that direction;
 * generate_device follows lyra_b200_set_decoder_mode.  extract_features_device and generate_device split dense calls over many
 * tiles into sub-batches like the codec calls (lyra_b200_set_split); results do not depend on the split.  None of them
 * allocates or reads the context's staging buffers. */
int lyra_b200_extract_features_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm /* [n][320] */, float* d_features /* [n][64] */);
int lyra_b200_quantize_device(lyra_b200_ctx* ctx, int n, const float* d_features, int num_bits, uint8_t* d_packets,
                              int32_t* d_indices /* [n][46] or NULL */);
int lyra_b200_dequantize_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, int num_bits, float* d_features);
int lyra_b200_generate_device(lyra_b200_ctx* ctx, int n, const float* d_features /* [n][64] */, int16_t* d_pcm /* [n][320] */);
int lyra_b200_logmel_device(lyra_b200_ctx* ctx, int bank, int n, const int16_t* d_pcm, int num_mel_bins, float* d_out);
/* either output may be NULL, not both */
int lyra_b200_noise_estimate_device(lyra_b200_ctx* ctx, int n, float* d_noise_estimate /* [n][160] or NULL */,
                                    uint8_t* d_is_noise /* [n] or NULL */);
int lyra_b200_cng_generate_device(lyra_b200_ctx* ctx, int n, const float* d_features /* [n][160] */, int16_t* d_pcm /* [n][320] */);
/* d_in[n][in_samples] -> d_out[n][out_stride]: the first d_out_counts[k] samples of row k are written, the rest of the row is
 * left as it is.  d_out_counts[n] (may be NULL) is written on the device; the host twin reads its counts back, which needs a
 * synchronisation, so this twin leaves them there. */
int lyra_b200_resample_device(lyra_b200_ctx* ctx, int to_internal, int n, int external_rate_hz, const int16_t* d_in, int in_samples,
                              int16_t* d_out, int out_stride, int32_t* d_out_counts /* [n] or NULL */);
/* Streams that sit out a hop: d_active is a device buffer the caller owns (NULL uninstalls it).  Like lyra_b200_set_stream this
 * is a host-side setting: every later encode_device, encode_dtx_device, decode_device, decode_track_noise_device and
 * decode_plc_device reads rows [0, n) of the buffer, in stream order on the installed stream, when its kernels run - so a server
 * rewrites the mask each hop (cudaMemcpyAsync or a kernel of its own) with no host synchronisation.  The library never writes
 * it; the caller keeps it valid while calls that read it are queued.
 *   A byte of 0 sits the stream out: it is exactly a LyraEncoder / LyraDecoder that is not called this hop.  None of its state
 *   changes (networks and hop counters, both noise estimators and their extractors, packet-loss control state, comfort-noise
 *   buffer and hop counter, both codec converters, its rate, bits and DTX words), and its PCM row, packet row and received byte
 *   are not read.  Its output rows: encode_device an all-zero packet; encode_dtx_device an all-zero packet and d_is_noise 1
 *   (nothing to send, as for an empty DTX packet); decode_device a zero PCM row (sample_rate / 50 samples);
 *   decode_track_noise_device a zero PCM row and its estimator's current is_noise, without feeding it; decode_plc_device a zero
 *   PCM row and is_comfort_noise of its unchanged state.  Any other byte runs the stream as usual.
 *   The host-buffer calls ignore the mask (their stream_ids say which streams run), as do noise_update_device (it has its own
 *   update mask) and the plugin-level calls and their twins: extract_features_device, quantize_device, dequantize_device,
 *   generate_device, logmel_device, noise_estimate_device, cng_generate_device and resample_device.
 * With no mask installed the calls launch exactly what they launch without it; with one they launch the same number of kernels,
 * and an all-ones mask gives bit-identical results.  A stream that sits out falls behind its tile neighbours' hop counters, as
 * after DTX or comfort-noise hops: lyra_b200_align_streams puts it back on a neighbour's phase.  LYRA_B200_EINVAL only for a
 * NULL context; works in any context. */
int lyra_b200_set_active_mask(lyra_b200_ctx* ctx, const uint8_t* d_active);
/* Per-stream call statistics on the device: audio level (RFC 6464 / RFC 6465), energy, DTX and concealment counters, per role.
 * A stream's statistics in one role are LYRA_B200_STATS_WORDS uint64 words; indices 4-6 mean different things per role:
 *   HOPS      calls in which the stream ran (the fused codec calls of the role; hops it sat out are not counted)
 *   SAT_OUT   *_device calls in which the active mask (lyra_b200_set_active_mask) sat it out
 *   ENERGY    sum over its run hops of floor(sum of squares / hop samples), in int16^2 units (WebRTC totalAudioEnergy =
 *             ENERGY * 0.02 / 2^30)
 *   LEVEL     RFC 6464 level of its last run hop, 0..127 (-dBov); 127 before any hop
 *   encoder:  EMPTY    run hops that produced an empty DTX packet (encode_dtx)
 *             BITS     sum of the bit counts of its non-empty packets (its own bits word, lyra_b200_set_stream_bits, or the
 *                      call's num_bits)
 *   decoder:  RECEIVED run hops decoded from a received packet
 *             CN_HOPS  run hops whose output contains comfort noise, fades included (decode_plc only)
 *             EVENTS   concealment events: a run hop that is not received and follows a received run hop, or is the stream's
 *                      first run hop
 * Unused words read 0.  The level and energy are taken over the stream's own hop at the external rate: the first rate / 50
 * samples of its row, the encoder's input row or the decoder's output row; DTX-empty hops are run hops.  LEVEL is the number of
 * thresholds t_k = 2^30 * 10^(-(k + 0.5) / 10), k = 0..126, computed on the host, that exceed (double)sum_of_squares / samples:
 * digital silence gives 127 and a full-scale square wave 0.
 *   lyra_b200_set_stats is a host-side setting like the active mask (no queue drain; 0 by default).  While it is 0 every call
 *   launches exactly what it launches without it and no statistic moves.  While it is 1 each of encode, encode_dtx, decode,
 *   decode_track_noise and decode_plc, host-buffer (stream_ids too) or *_device twin, launches one more kernel per sub-batch and
 *   updates the statistics of the call's role by stream id; a stream that sits out only counts SAT_OUT and its row is not read.
 *   The plugin-level calls and their twins, noise_update(_device) and resample(_device) do not count.  Captured graphs
 *   (lyra_b200_set_graphs) are kept per setting.
 *   The statistics are per-stream state: lyra_b200_reset and copy_streams from -1 restore the initial image, copy_streams,
 *   export_streams and import_streams carry them (import refuses a LEVEL above 127).
 *   lyra_b200_read_stats: stats[k][0..7] = the statistics of stream stream_ids[k] (NULL: k; an id may be listed more than once)
 *   in `role`.  Ordered on the installed stream behind the work queued there; returns when the values are in the caller's
 *   buffer.  lyra_b200_read_stats_device: the same for streams 0..n-1 into the device buffer d_stats, rows [0, n) only,
 *   asynchronous on the installed stream like the *_device calls.  clear = 1 then zeroes the counters and the energy of the
 *   listed streams, in stream order after reading; LEVEL and the event state stay, so a server can poll every hop or every
 *   second without losing a hop.
 * role is LYRA_B200_ROLE_ENCODER or LYRA_B200_ROLE_DECODER and must be a role of the context.  A bad role, n or id, or a NULL
 * buffer returns LYRA_B200_EINVAL and queues nothing. */
#define LYRA_B200_STATS_WORDS 8
#define LYRA_B200_STAT_HOPS 0
#define LYRA_B200_STAT_SAT_OUT 1
#define LYRA_B200_STAT_ENERGY 2
#define LYRA_B200_STAT_LEVEL 3
#define LYRA_B200_STAT_EMPTY 4      /* encoder */
#define LYRA_B200_STAT_BITS 5       /* encoder */
#define LYRA_B200_STAT_RECEIVED 4   /* decoder */
#define LYRA_B200_STAT_CN_HOPS 5    /* decoder */
#define LYRA_B200_STAT_EVENTS 6     /* decoder */
int lyra_b200_set_stats(lyra_b200_ctx* ctx, int enable);
int lyra_b200_read_stats(lyra_b200_ctx* ctx, int role, const int32_t* stream_ids, int n, uint64_t* stats /* [n][8] */, int clear);
int lyra_b200_read_stats_device(lyra_b200_ctx* ctx, int role, int n, uint64_t* d_stats /* [n][8] */, int clear);
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
