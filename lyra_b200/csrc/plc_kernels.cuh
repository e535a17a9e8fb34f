// Decoder packet-loss path as batched device steps (SURVEY.md section 8 rows f2, f4):
//   PlcPlanKernel        the per-stream concealment / fade bookkeeping of LyraDecoder::SetEncodedPacket +
//                        DecodeSamplesInternal for one whole hop per tick          (lyra/lyra_decoder.cc:186-196, 228-283, 303)
//   ComfortNoiseKernel   ComfortNoiseGenerator::RunConditioning + RunModel(hop)   (lyra/comfort_noise_generator.cc:74-119)
//   PlcMixKernel         LyraDecoder::MaybeOverlapAndInsert                        (lyra/lyra_decoder.cc:342-373)
// Arithmetic mirrors oracle/comfort_noise.c and oracle/lyra_decoder.c operation by operation (separately rounded f64 / f32
// operations, host-computed tables for every transcendental), so the results are bit-identical to the oracle.
#pragma once

#include "aux_kernels.cuh"

namespace lyra_b200 {

// per-stream decoder control state: {concealment_progress, fade_progress, fade_direction (-1 from / +1 to comfort noise), -}
constexpr int kPlcConcealSamples = 1280, kPlcFadeSamples = 640;

// What one tick does to one stream (whole-hop regime: one optional packet, then 320 samples):
//   received packet:  concealment_progress <- 0 (a whole fake hop has always been played out), features queued
//   then the decode step of lyra_decoder.cc:249-283 with num_samples_to_generate = 320.
// plan[slot] bits: 1 = run the generative model, 2 = run the comfort-noise generator, 4 = the hop comes from a received packet
// (feed the noise estimator); fade0[slot] = fade progress before the hop, dir[slot] = fade direction of the hop.
// A slot that sits out does so as a LyraDecoder that is not called: plan kPlanSatOut (no model, no comfort noise, no feed;
// PlcMixKernel writes zeros), its received byte is not read, its state is not written and is_comfort_noise reports the state as
// it is.
constexpr uint8_t kPlanSatOut = 8;
__global__ void __launch_bounds__(256)
PlcPlanKernel(const __grid_constant__ RowIo io, const uint8_t* __restrict__ received, int* __restrict__ state,
              uint8_t* __restrict__ plan, int* __restrict__ fade0, int* __restrict__ dir_out, uint8_t* __restrict__ skip_model,
              uint8_t* __restrict__ feed_mask, uint8_t* __restrict__ is_comfort_noise) {
  const int row = (int)(blockIdx.x * blockDim.x + threadIdx.x), slot = io.slot0 + row;
  if (row >= io.slots) return;
  int* st = state + (size_t)io.Stream(slot) * 4;
  int cp = st[0], fp = st[1], dir = st[2];
  if (io.SatOut(slot)) {
    plan[slot] = kPlanSatOut;
    skip_model[slot] = 1;
    feed_mask[slot] = 0;
    if (is_comfort_noise) is_comfort_noise[slot] = fp == kPlcFadeSamples ? 1 : 0;
    return;
  }
  const bool rec = received == nullptr || received[slot] != 0;
  if (rec && cp > 0) cp = 0;                                  // SetEncodedPacket :186-196 (nothing left of a fake hop at a hop boundary)
  const bool is_packet_received = rec && cp == 0;             // :249-251 (the model queue holds exactly this tick's packet)
  if (is_packet_received) dir = -1;                           // :253-256
  else if (cp == kPlcConcealSamples) dir = +1;                // :257-260
  else cp += 320;                                             // :261-265
  int gen = 1, cng = 1;
  int next_fp = fp + dir * 320;                               // :269-270
  if (dir == +1 && fp == kPlcFadeSamples) { next_fp = kPlcFadeSamples; gen = 0; }       // :271-276
  else if (dir == -1 && fp == 0) { next_fp = 0; cng = 0; }                               // :277-282
  plan[slot] = (uint8_t)(gen | (cng << 1) | (is_packet_received ? 4 : 0));
  fade0[slot] = fp;
  dir_out[slot] = dir;
  skip_model[slot] = gen ? 0 : 1;
  feed_mask[slot] = is_packet_received ? 1 : 0;
  st[0] = cp; st[1] = next_fp; st[2] = dir;                   // :303
  if (is_comfort_noise) is_comfort_noise[slot] = next_fp == kPlcFadeSamples ? 1 : 0;     // :381-383
}

// splitmix64 of (seed, hop, bin): the phase index (0..1023) of oracle/comfort_noise.c lo_cng_phase_index
__device__ __forceinline__ uint32_t CngPhaseIndex(unsigned long long seed, unsigned long long hop, int bin) {
  unsigned long long x = seed ^ (hop * 0xD1B54A32D192ED03ull) ^ ((unsigned long long)bin * 0x9E3779B97F4A7C15ull);
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  x ^= x >> 31;
  return (uint32_t)(x >> 54);
}

// One block of 128 threads per stream.  features: [slots][160] conditioning log-mel vectors (by slot), or nullptr = the stream's
// current noise estimate (the first 160 floats of its noise-estimator state, LyraDecoder::RunComfortNoiseGenerator,
// lyra/lyra_decoder.cc:328-340).  plan: nullptr = every slot runs; otherwise only slots with bit 2.
// work: [max_streams][1024] f64 overlap-add buffers; hops: [max_streams][2] {hop counter, key offset}: the phases of stream s are
// drawn from key seed + s + offset (offset 0 unless the stream's state was moved here by lyra_b200_import_streams / _copy_streams).
constexpr int kCngThreads = 128;
__global__ void __launch_bounds__(kCngThreads)
ComfortNoiseKernel(const uint8_t* __restrict__ blob, CngParams P, const __grid_constant__ RowIo io, const float* __restrict__ features,
                   const float* __restrict__ noise_state, int noise_units, const uint8_t* __restrict__ plan, double* __restrict__ work,
                   unsigned long long* __restrict__ hops, unsigned long long seed, int16_t* __restrict__ out) {
  unsigned char* smem = LYRA_DYN_SMEM();
  double* re = reinterpret_cast<double*>(smem);
  double* im = re + kLogMelFftPadded;
  double* xr0 = im + kLogMelFftPadded;           // spectrum in natural order: real | imag, padded like the FFT buffers
  double* xi0 = xr0 + kLogMelFftPadded;
  double* mel = xi0 + kLogMelFftPadded;          // [160]
  if ((int)blockIdx.x >= io.slots) return;
  const int slot = io.slot0 + (int)blockIdx.x;
  if (plan && !(plan[slot] & 2)) return;
  const int stream = io.Stream(slot);
  const int tid = (int)threadIdx.x;
  constexpr int NT = kCngThreads, N = kLogMelFft;
  const double* wts = BlobPtr<double>(blob, P.weights);
  const int* band = BlobPtr<int>(blob, P.band);
  const double* norm = BlobPtr<double>(blob, P.norm);
  const double* synth = BlobPtr<double>(blob, P.synth);
  const double2* tw = BlobPtr<double2>(blob, P.twiddle);
  const float* f = features ? features + (size_t)slot * P.num_mel : noise_state + (size_t)stream * noise_units;
  const unsigned long long hop_index = hops[2 * (size_t)stream];
  const unsigned long long sseed = seed + (unsigned long long)stream + hops[2 * (size_t)stream + 1];
  // mel[c] = (double)(float)exp(feature * 10)   (FftFromFeatures, .cc:87-96; exp of a float evaluated in double, rounded once)
  for (int c = tid; c < P.num_mel; c += NT) mel[c] = (double)(float)exp((double)__fmul_rn(f[c], 10.0f));
  for (int i = tid; i < N; i += NT) { xr0[FftIdx(i)] = 0.0; xi0[FftIdx(i)] = 0.0; }
  __syncthreads();
  // mel inverse -> magnitude -> unit vector at the drawn phase -> Hermitian spectrum
  for (int i = tid; i <= N / 2; i += NT) {
    double v = 0.0;
    if (i >= P.start_index && i <= P.end_index) {
      const int ch = band[i];
      if (ch >= 0) v = __dadd_rn(v, __ddiv_rn(__dmul_rn(mel[ch], wts[i]), norm[ch]));
      if (ch + 1 < P.num_mel) v = __dadd_rn(v, __ddiv_rn(__dmul_rn(mel[ch + 1], __dsub_rn(1.0, wts[i])), norm[ch + 1]));
    }
    const double mag = __dsqrt_rn(__dmul_rn(v, v));
    const uint32_t p = CngPhaseIndex(sseed, hop_index, i);
    const double2 w = tw[511 + (p & 511u)];                  // last stage's table: (cos, sin)(-2 pi k / 1024)
    double cr = w.x, ci = -w.y;
    if (p >= 512u) { cr = -cr; ci = -ci; }
    const double vr = __dmul_rn(mag, cr), vi = __dmul_rn(mag, ci);
    if (i == 0 || i == N / 2) { xr0[FftIdx(i)] = vr; }
    else { xr0[FftIdx(i)] = vr; xi0[FftIdx(i)] = vi; xr0[FftIdx(N - i)] = vr; xi0[FftIdx(N - i)] = -vi; }
  }
  __syncthreads();
  Fft1024<true>(re, im, tw, [&](int i, double& xr, double& xi) {
    xr = xr0[FftIdx(i)];
    xi = xi0[FftIdx(i)];
  });
  // 1/N, synthesis window, overlap-add; emit one hop (ClipToInt16: clamp, truncate); shift the buffer by one hop
  double* wk = work + (size_t)stream * N;
  for (int i = tid; i < N; i += NT) {
    const double v = __dadd_rn(wk[i], __dmul_rn(__ddiv_rn(re[FftIdx(i)], (double)N), synth[i]));
    xr0[FftIdx(i)] = v;                                                        // staged: the shift below crosses threads
  }
  __syncthreads();
  for (int i = tid; i < N; i += NT) wk[i] = i + P.hop < N ? xr0[FftIdx(i + P.hop)] : 0.0;
  for (int i = tid; i < P.hop; i += NT) {
    double v = xr0[FftIdx(i)];
    v = v > -32768.0 ? v : -32768.0;
    v = v < 32767.0 ? v : 32767.0;
    out[(size_t)slot * P.hop + i] = (int16_t)v;
  }
  if (tid == 0) hops[2 * (size_t)stream] = hop_index + 1;
}

// out = model hop, comfort-noise hop, or their raised-cosine cross-fade (lyra_decoder.cc:342-373); 320 threads per slot
__global__ void __launch_bounds__(320)
PlcMixKernel(const uint8_t* __restrict__ blob, CngParams P, const __grid_constant__ RowIo io, const uint8_t* __restrict__ plan,
             const int* __restrict__ fade0, const int* __restrict__ dir, const int16_t* __restrict__ model_pcm,
             const int16_t* __restrict__ cng_pcm, int16_t* __restrict__ out) {
  if ((int)blockIdx.x >= io.slots) return;
  const int slot = io.slot0 + (int)blockIdx.x, i = (int)threadIdx.x;
  const int pl = plan[slot];
  const size_t o = (size_t)slot * 320 + i;
  if (pl == kPlanSatOut) { out[o] = 0; return; }
  if (!(pl & 2)) { out[o] = model_pcm[o]; return; }
  if (!(pl & 1)) { out[o] = cng_pcm[o]; return; }
  const float* fade = BlobPtr<float>(blob, P.fade);
  const float w = fade[fade0[slot] + dir[slot] * i];
  const float v = __fadd_rn(__fmul_rn((float)model_pcm[o], w), __fmul_rn((float)cng_pcm[o], __fsub_rn(1.0f, w)));
  out[o] = (int16_t)v;
}

// read-only view of the noise estimators (NoiseEstimator::noise_estimate / is_noise, lyra/noise_estimator.h:55-62)
__global__ void __launch_bounds__(192)
NoiseReadKernel(const __grid_constant__ RowIo io, const float* __restrict__ state, int nf, float* __restrict__ estimate_out,
                uint8_t* __restrict__ is_noise_out) {
  if ((int)blockIdx.x >= io.slots) return;
  const int slot = io.slot0 + (int)blockIdx.x, i = (int)threadIdx.x;
  const float* st = state + (size_t)io.Stream(slot) * NoiseStateUnits(nf);
  if (estimate_out && i < nf) estimate_out[(size_t)slot * nf + i] = st[i];
  if (is_noise_out && i == 0) is_noise_out[slot] = reinterpret_cast<const int*>(st + 5 * nf)[2] ? 0 : 1;
}

// Resampler::Resample (lyra/resampler.cc:52-57) for n streams, `n_in` input samples each: int16 -> float, polyphase FIR over the
// 35-tap delay line, ClipToInt16.  Arithmetic and tap order are oracle/resampler.c's (one separately rounded multiply and add per
// tap, ascending input order).  Per-stream state: delay[34] (the last 34 input samples), pos = position of the next output relative
// to the next input sample, in units of 1 / den input samples; tag = the configuration the state belongs to (lyra_b200_resample:
// the external rate; the codec path: the generation of the context's rate setting).  A call with another tag starts from the
// fully-primed state, like a fresh Resampler; 0 (what lyra_b200_reset writes) never matches.  counts[slot] (may be nullptr) =
// outputs produced (they differ by at most one between streams when down-sampling from different phases).  In rows are
// `in_stride` and out rows `out_stride` samples apart.
// words.rate == nullptr (lyra_b200_resample): every stream converts n_in samples with `pair`, at most out_stride outputs.
// words.rate != nullptr (the fused codec calls, one whole hop per row): pair is 0 (to 16 kHz) or 3 (from 16 kHz) and each stream
// runs at its own rate r: pair + RateIndex(r) - 1, r / 50 samples on the external side, 320 on the 16 kHz side; a 16 kHz stream is
// copied through and its converter state is left alone.  Output rows longer than the stream's hop (a decoder row of a stream
// below the context's rate) get zeros after it.
// A slot that sits out has its input row and converter state neither read nor written; from 16 kHz (pair >= 3) its output row is
// written as zeros.
__global__ void __launch_bounds__(128)
ResampleKernel(const uint8_t* __restrict__ blob, ResamplerParams P, int pair, int tag, const __grid_constant__ RowIo io,
               const __grid_constant__ StreamWords words, const int16_t* __restrict__ in, int in_stride, int n_in,
               int16_t* __restrict__ out, int out_stride, int* __restrict__ counts, int16_t* __restrict__ delay_state,
               int* __restrict__ pos_state) {
  unsigned char* smem = LYRA_DYN_SMEM();
  float* x = reinterpret_cast<float*>(smem);              // [34 + n_in]: delay line followed by the new samples
  if ((int)blockIdx.x >= io.slots) return;
  const int slot = io.slot0 + (int)blockIdx.x;
  const int stream = io.Stream(slot);
  constexpr int T = kResamplerTaps;
  const int tid = (int)threadIdx.x, NT = (int)blockDim.x;
  const int16_t* row = in + (size_t)slot * in_stride;
  int16_t* orow = out + (size_t)slot * out_stride;
  if (io.SatOut(slot)) {
    if (pair >= 3)
      for (int j = tid; j < out_stride; j += NT) orow[j] = 0;
    return;
  }
  int n_out = out_stride;
  const bool codec = words.rate != nullptr;
  if (codec) {
    constexpr int H = 320;                                // one 16 kHz hop
    const int r = words.Rate(stream), k = RateIndex(r);
    if (k == 0) {                                         // 16 kHz: no conversion
      for (int j = tid; j < out_stride; j += NT) orow[j] = j < H ? row[j] : (int16_t)0;
      return;
    }
    n_in = pair < 3 ? r / 50 : H;
    n_out = pair < 3 ? H : r / 50;
    pair += k - 1;
  }
  int16_t* dl = delay_state + (size_t)stream * (T - 1);
  int* ps = pos_state + (size_t)stream * 2;              // {pos, tag}
  const bool fresh = ps[1] != tag;
  const int a0 = fresh ? 0 : ps[0];
  for (int i = tid; i < T - 1; i += NT) x[i] = fresh ? 0.0f : (float)dl[i];
  for (int i = tid; i < n_in; i += NT) x[T - 1 + i] = (float)row[i];
  __syncthreads();
  const int num = P.num[pair], den = P.den[pair];
  const float* coeffs = BlobPtr<float>(blob, P.coeffs[pair]);
  const int total = n_in * den;
  const int count = a0 < total ? (total - a0 + num - 1) / num : 0;
  if (codec)
    for (int j = (count < n_out ? count : n_out) + tid; j < out_stride; j += NT) orow[j] = 0;
  for (int j = tid; j < count && j < n_out; j += NT) {
    const int a = a0 + j * num, i = a / den, ph = a % den;
    const float* c = coeffs + ph * T;
    const float* xs = x + i;                              // delay-line sample 0 of the window that ends at input sample i
    float acc = 0.0f;
#pragma unroll 5
    for (int t = 0; t < T; ++t) acc = __fadd_rn(acc, __fmul_rn(c[t], xs[t]));
    float v = acc;
    v = v > -32768.0f ? v : -32768.0f;
    v = v < 32767.0f ? v : 32767.0f;
    orow[j] = (int16_t)v;
  }
  __syncthreads();
  for (int i = tid; i < T - 1; i += NT) dl[i] = (int16_t)x[n_in + i];     // the last 34 samples of [delay | in]
  if (tid == 0) {
    ps[0] = a0 + count * num - total;
    ps[1] = tag;
    if (counts) counts[slot] = count;
  }
}

// ------------------------------------------------------------------------------------------------
// Per-stream call statistics (lyra_b200_set_stats / _read_stats).  One entry per role, row-major, kStatsWords u64 per stream:
// the public words LYRA_B200_STAT_* (0..6) and word kStatPrevReceived, whether the stream's last run hop was received (decoder
// role; initially 1, so a first run hop that is not received is a concealment event).
constexpr int kStatsWords = 8;
constexpr int kStatHops = 0, kStatSatOut = 1, kStatEnergy = 2, kStatLevel = 3, kStatEmpty = 4, kStatBits = 5, kStatReceived = 4,
              kStatCnHops = 5, kStatEvents = 6, kStatPrevReceived = 7;
constexpr int kStatsLevels = 127;                 // RFC 6464 levels 1..127 (-dBov); the host's threshold table has 128 entries
constexpr int kStatsThreads = 256;                // one warp per row
constexpr int kStatsRowsPerBlock = kStatsThreads / 32;
// what the event source of CallStatsKernel is: encode (none), encode_dtx (the DTX flags, 1 = empty packet), decode /
// decode_track_noise (the received bytes, nullptr = every packet arrived), decode_plc (the plan bytes of PlcPlanKernel)
enum StatsSource { kStatsEncode = 0, kStatsEncodeDtx = 1, kStatsDecode = 2, kStatsDecodePlc = 3 };

// sum of the squares of the two int16 samples in w (each square <= 2^30, so the pair fits 32 bits)
__device__ __forceinline__ uint32_t SquarePair(uint32_t w) {
  const int lo = (int)(int16_t)(w & 0xffffu), hi = (int)(int16_t)(w >> 16);
  return (uint32_t)(lo * lo) + (uint32_t)(hi * hi);
}

// One warp per row of the call: the first rate / 50 samples of the row (rows row_stride samples apart) -> their exact sum of
// squares, with 16-byte loads over the row's 16-byte aligned middle (the ABI promises 2-byte alignment only) and a warp
// shuffle reduction; then lane 0 updates the statistics of the row's stream.  levels: the 128 host-computed thresholds
// t_k = 2^30 10^(-(k + 0.5) / 10), k < 127, and 0.  A slot that sits out counts kStatSatOut only and its row and event byte are
// not read.  bits: the call's num_bits (encoder role).
__global__ void __launch_bounds__(kStatsThreads)
CallStatsKernel(const __grid_constant__ RowIo io, const __grid_constant__ StreamWords words, const int16_t* __restrict__ pcm,
                int row_stride, int source, const uint8_t* __restrict__ events, int num_bits, const double* __restrict__ levels,
                unsigned long long* __restrict__ stats) {
  const int lane = (int)threadIdx.x % 32;
  const int row = (int)blockIdx.x * kStatsRowsPerBlock + (int)threadIdx.x / 32, slot = io.slot0 + row;
  if (row >= io.slots) return;
  const int stream = io.Stream(slot);
  unsigned long long* st = stats + (size_t)stream * kStatsWords;
  if (io.SatOut(slot)) {
    if (lane == 0) st[kStatSatOut] += 1;
    return;
  }
  const int samples = words.Rate(stream) / 50;
  const int16_t* x = pcm + (size_t)slot * row_stride;
  int head = (int)((16u - ((unsigned)(uintptr_t)x & 15u)) & 15u) / 2;
  head = head < samples ? head : samples;
  const int vecs = (samples - head) / 8;
  const uint4* xv = reinterpret_cast<const uint4*>(x + head);
  unsigned long long sq = 0;
  if (lane < head) sq += (unsigned long long)((int)x[lane] * (int)x[lane]);
  for (int i = lane; i < vecs; i += 32) {
    const uint4 v = xv[i];
    sq += (unsigned long long)SquarePair(v.x) + SquarePair(v.y) + (unsigned long long)SquarePair(v.z) + SquarePair(v.w);
  }
  for (int i = head + vecs * 8 + lane; i < samples; i += 32) sq += (unsigned long long)((int)x[i] * (int)x[i]);
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, m);
  const double msq = __ddiv_rn((double)sq, (double)samples);
  int level = 0;
  for (int k = lane; k < kStatsLevels; k += 32) level += levels[k] > msq ? 1 : 0;
#pragma unroll
  for (int m = 16; m >= 1; m >>= 1) level += __shfl_xor_sync(0xffffffffu, level, m);
  if (lane != 0) return;
  st[kStatHops] += 1;
  st[kStatEnergy] += sq / (unsigned long long)samples;
  st[kStatLevel] = (unsigned long long)level;
  if (source == kStatsEncode || source == kStatsEncodeDtx) {
    if (source == kStatsEncodeDtx && events[slot]) st[kStatEmpty] += 1;
    else st[kStatBits] += (unsigned long long)(words.Stages(stream, num_bits / kRvqBitsPerStage) * kRvqBitsPerStage);
    return;
  }
  const int e = events ? events[slot] : 1;
  const bool received = source == kStatsDecodePlc ? (e & 4) != 0 : e != 0;
  if (received) st[kStatReceived] += 1;
  if (source == kStatsDecodePlc && (e & 2)) st[kStatCnHops] += 1;
  if (!received && st[kStatPrevReceived]) st[kStatEvents] += 1;
  st[kStatPrevReceived] = received ? 1ull : 0ull;
}

// lyra_b200_read_stats(_device): out[k] (nullptr: no read) <- the public words of stream ids[k] (ids nullptr: k) in the entry
// `stats`, word kStatPrevReceived read as 0; with clear the counters and the energy are zeroed after the read (LEVEL and the
// private word stay).  A read with repeated ids and clear runs as a read launch followed by a clear launch.
__global__ void __launch_bounds__(256)
StatsReadKernel(unsigned long long* __restrict__ stats, const int* __restrict__ ids, int n, unsigned long long* __restrict__ out,
                int clear) {
  const int g = (int)(blockIdx.x * blockDim.x + threadIdx.x), k = g / kStatsWords, w = g % kStatsWords;
  if (k >= n) return;
  unsigned long long* v = stats + (size_t)(ids ? ids[k] : k) * kStatsWords + w;
  if (out) out[g] = w == kStatPrevReceived ? 0ull : *v;
  if (clear && w != kStatLevel && w != kStatPrevReceived) *v = 0ull;
}

}  // namespace lyra_b200
