// Context + launch logic + the C ABI of include/lyra_b200.h.
// Compiled by nvcc for sm_90a (product) and, for the CPU test tier only, by g++ with -DLYRA_EMU.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/lyra_b200.h"
#include "aux_kernels.cuh"
#include "model_spec.h"
#include "net_kernels.cuh"
#include "net_kernels_wgmma.cuh"
#include "plc_kernels.cuh"

using namespace lyra_b200;

namespace {

std::string g_create_error;

#define CU(call)                                                                        \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess) {                                                            \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                    \
      return LYRA_B200_ENODEV;                                                          \
    }                                                                                   \
  } while (0)

// preamble of every entry point that touches CUDA: select the context's device (the current device is per host thread),
// then refuse the call if the context lacks `role` (0: any context)
#define ENTER(role)                                                                     \
  if (!UseDevice(ctx)) return LYRA_B200_ENODEV;                                         \
  if ((role) && !RoleOk(ctx, (role))) return LYRA_B200_EINVAL;

// the per-stream words the host mirrors (lyra_b200_ctx::word_mirror); the bits words are indexed by role index (0 encoder, 1 decoder)
enum MirroredWord { kWordEncBits = 0, kWordDecBits = 1, kWordDtxOff = 2, kMirroredWords = 3 };

}  // namespace

struct lyra_b200_ctx {
  ModelSpec spec;
  int device = 0, max_streams = 0, ntiles = 0, padded = 0;
  int roles = LYRA_B200_ROLE_ENCODER | LYRA_B200_ROLE_DECODER;   // which halves of the streaming state this context holds
  std::vector<void*> allocs;         // every device allocation of the context (lyra_b200_destroy frees them)
  // Every piece of per-stream state, in one list that drives lyra_b200_reset, _export_streams, _import_streams and
  // _copy_streams: `words` 4-byte words per stream at lane stride `lanes` (layout of StateWord), initial image `init`
  // (nullptr: zero), hop counter `n18` (nullptr: none; initially 0).  `reset` = false: lyra_b200_reset leaves the entry alone
  // (lyra_b200_resample's delay lines).  `kind` (StreamStateKind) marks the words a record does not carry verbatim; `check`
  // is what import validates in a record's payload besides the hop counter.
  enum Check { kCheckNone, kCheckPlc, kCheckResamplerPos, kCheckStreamRate, kCheckStreamBits, kCheckStreamDtx, kCheckStats };
  struct StateEntry {
    StreamStateEntry e;              // e.offset is set by BuildStateTable
    bool reset;
    int check;
  };
  std::vector<StateEntry> state_list;
  StreamStateTable state_table{};    // the list as the record kernels see it (built at the end of create)
  StreamStateTable reset_table{};    // its entries that lyra_b200_reset restores
  StreamStateTable dtx_table{};      // the encoder-side DTX estimator's entries (d_noise_enc, d_logmel_prev_enc)
  uint64_t model_fingerprint = 0;    // of the loaded weights (ModelFingerprint), part of every record header
  uint32_t* d_records = nullptr;     // export / import staging: records_chunk records (allocated on first use)
  int records_chunk = 0;
  uint8_t* d_blob = nullptr;
  // streaming state, one block per kernel
  uint32_t* d_state[4] = {nullptr, nullptr, nullptr, nullptr};
  int* d_n18[4] = {nullptr, nullptr, nullptr, nullptr};
  StreamAlignTable align_table{};    // the network entries the context holds, as StreamAlignKernel sees them
  float* d_mid_enc = nullptr;
  float* d_mid_dec = nullptr;
  int16_t* d_logmel_prev[3] = {nullptr, nullptr, nullptr};   // banks 0/1: lyra_b200_logmel; bank 2: the noise estimator's extractor
  float* d_noise = nullptr;          // [max_streams][NoiseStateUnits(160)] noise-estimator state
  float* d_noise_est = nullptr;      // staging for the host-buffer API
  uint8_t* d_is_noise = nullptr;
  float* d_noise_enc = nullptr;      // the encoder side's own estimators (DTX, lyra/lyra_encoder.cc:80-89)
  int16_t* d_logmel_prev_enc = nullptr;
  NoiseParams noise_params{};
  // decoder packet-loss path (PlcPlanKernel / ComfortNoiseKernel / PlcMixKernel)
  int* d_plc = nullptr;                      // [max_streams][4] concealment_progress, fade_progress, fade_direction, -
  double* d_cng_work = nullptr;              // [max_streams][1024] overlap-add buffers of the comfort-noise generators
  unsigned long long* d_cng_hops = nullptr;  // [max_streams][2] {hop counter, comfort-noise key offset} (ComfortNoiseKernel)
  unsigned long long cng_seed = 0;
  uint8_t* d_plan = nullptr;                 // by slot
  uint8_t* d_skip = nullptr;
  uint8_t* d_feed = nullptr;
  uint8_t* d_is_cn = nullptr;
  int* d_fade0 = nullptr;
  int* d_dir = nullptr;
  int16_t* d_model_pcm = nullptr;
  int16_t* d_cng_pcm = nullptr;
  float* d_cng_feat = nullptr;
  // sample-rate converters: [direction 0 = to 16 kHz (encoder side), 1 = from 16 kHz (decoder side)][max_streams] state
  int16_t* d_rs_delay[2] = {nullptr, nullptr};   // [max_streams][34]
  int* d_rs_pos[2] = {nullptr, nullptr};         // [max_streams][2] {position, rate}
  int16_t* d_rs_in = nullptr;                    // staging [max_streams][960]
  int16_t* d_rs_out = nullptr;
  int* d_rs_counts = nullptr;
  // lyra_b200_set_sample_rate: the external rate of the fused codec calls.  Their converters are the encoder's and the decoder's
  // own (lyra/lyra_encoder.cc:58-66, lyra/lyra_decoder.cc:108-114), separate from lyra_b200_resample's: [0] external -> 16 kHz
  // (encoder role), [1] 16 kHz -> external (decoder role), same layout as d_rs_delay / d_rs_pos
  int sample_rate = 16000;
  int codec_rs_tag = 1;                          // ResampleKernel tag of the current setting (bumped by every change)
  int16_t* d_codec_rs_delay[2] = {nullptr, nullptr};
  int* d_codec_rs_pos[2] = {nullptr, nullptr};
  // lyra_b200_set_stream_sample_rates: one word per stream, 0 = sample_rate, otherwise the stream's own rate (StreamWordKernel)
  int* d_stream_rate = nullptr;
  bool rate_override = false;                    // some stream may run at another rate than sample_rate
  ByRate<NoiseParams> enc_noise_params{};        // the encoder-side estimators' constants and extractor tables, by stream rate
  ByRate<LogMelParams> enc_logmel{};
  // Per-stream words with a host mirror (MirroredWord; nullptr when the context lacks the word's role):
  //   kWordEncBits / kWordDecBits  lyra_b200_set_stream_bits: 0 = the call's num_bits, otherwise the stream's own bit count;
  //   kWordDtxOff                  lyra_b200_set_stream_dtx (encoder role), stored inverted: 0 = DTX on (the default), 1 = off.
  // Every change starts on the host (the setters, copy_streams, import_streams, reset), so word_mirror is an exact host image of
  // the words in program order, which is also stream order: the calls check their num_bits against it and the DTX setter finds
  // the streams it turns on without reading the device.  own_words[w] counts the streams whose word is not 0; while it is 0 the
  // kernels that read the word get no pointer and the calls launch exactly what they launch without the feature.
  int* d_stream_word[kMirroredWords] = {nullptr, nullptr, nullptr};
  std::vector<int> word_mirror[kMirroredWords];
  int own_words[kMirroredWords] = {0, 0, 0};
  // device staging for the host-buffer API
  int16_t* d_pcm = nullptr;
  uint8_t* d_packets = nullptr;
  uint8_t* d_received = nullptr;
  float* d_features = nullptr;
  float* d_melout = nullptr;
  int* d_indices = nullptr;
  int* d_ids = nullptr;
  // lyra_b200_set_active_mask: the caller's buffer, by row of the *_device codec calls (0 = the stream sits the call out); nullptr:
  // every stream runs and the kernels get no pointer
  const uint8_t* d_active = nullptr;
  // lyra_b200_set_stats: the fused codec calls launch CallStatsKernel once per part into d_stats[role index] (per-stream state,
  // kStatsWords u64 per stream; nullptr when the context lacks the role).  d_stats_levels: the 128 level thresholds;
  // d_stats_out: lyra_b200_read_stats's staging [max_streams][kStatsWords]
  bool stats_on = false;
  unsigned long long* d_stats[2] = {nullptr, nullptr};
  double* d_stats_levels = nullptr;
  unsigned long long* d_stats_out = nullptr;
  // tile map
  int* d_tile_list = nullptr;
  int* d_slot_of = nullptr;
  // host images of the map, pinned and double-buffered: a sparse call fills the buffer the previous call did not use and
  // copies it asynchronously (no host synchronisation on the call path); ev_map[b] marks "the copy out of buffer b is done"
  int* h_tile_list[2] = {nullptr, nullptr};
  int* h_slot_of[2] = {nullptr, nullptr};
  cudaEvent_t ev_map[2] = {nullptr, nullptr};
  bool map_pending[2] = {false, false};
  int map_buf = 0;
  std::vector<uint32_t> tile_gen;       // tile_gen[t] == map_gen: tile t is already in this call's tile list
  uint32_t map_gen = 0;
  std::vector<uint32_t> id_seen;        // id_seen[s] == id_gen: stream s is already in this call's id list (CheckIds)
  uint32_t id_gen = 0;
  std::vector<int> touched[2];          // slots of h_slot_of[b] that are not -1 (cleared lazily instead of an O(max_streams) fill)
  int map_dense_n = -1;     // >= 0: the device map currently describes streams 0..n-1
  int active_tiles = 0;
  cudaStream_t own_stream = nullptr, stream = nullptr;
  static constexpr int kMaxSplit = 4;
  cudaStream_t aux_stream[kMaxSplit - 1] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[kMaxSplit - 1] = {nullptr, nullptr, nullptr};
  int nsplit = 3;
  bool blocking_sync = false;        // host-buffer calls sleep on an event instead of spinning (lyra_b200_set_blocking_sync)
  cudaEvent_t ev_sync = nullptr;
  int decoder_mode = LYRA_B200_DECODER_EXACT;   // lyra_b200_set_decoder_mode
  int priority = 0;                  // CUDA priority of own_stream / aux_stream (lyra_b200_set_priority)
  uint64_t launches = 0;
  // lyra_b200_set_graphs: the dense host-buffer encode / decode calls replay a captured CUDA graph (copies in, kernels of every
  // sub-batch, copies out) instead of re-issuing ~20 stream operations per call; one graph per (call shape, host buffers)
  // (rates: rate_override, which adds the converters' launches at 16 kHz; bits: own_words of the call's role's bits word, which
  // hands the RVQ kernels the bits words; stats: stats_on, which adds CallStatsKernel's launches)
  struct GraphKey {
    int kind, n, num_bits, mode, nsplit;
    const void *a, *b, *c;
    bool rates, bits, stats;
    bool operator==(const GraphKey& o) const {
      return kind == o.kind && n == o.n && num_bits == o.num_bits && mode == o.mode && nsplit == o.nsplit && a == o.a && b == o.b && c == o.c &&
             rates == o.rates && bits == o.bits && stats == o.stats;
    }
  };
  struct GraphEntry { GraphKey key; void* exec; uint64_t launches; };
  bool use_graphs = false;
  std::vector<GraphEntry> graphs;
  uint64_t graph_replays = 0;
  std::string err;
  // diagnostics: CUDA-event timing of every kernel launch
  bool profiling = false;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events[LYRA_B200_NUM_KERNELS];
  size_t prof_used[LYRA_B200_NUM_KERNELS] = {};
  double prof_ms[LYRA_B200_NUM_KERNELS] = {};
  uint64_t prof_n[LYRA_B200_NUM_KERNELS] = {};
};

namespace {

int PacketBytes(int num_bits) { return (num_bits + 7) / 8; }

// index of an external rate in the resampler's filter banks (ResamplerParams pairs 0-2 to 16 kHz, 3-5 from it); -1: unsupported
int RatePair(int rate_hz) { return rate_hz == 8000 ? 0 : rate_hz == 32000 ? 1 : rate_hz == 48000 ? 2 : -1; }
bool RateOk(int rate_hz) { return rate_hz == 16000 || RatePair(rate_hz) >= 0; }

// The fused codec calls convert when the context is not at 16 kHz or some stream may have a rate of its own
bool Converts(const lyra_b200_ctx* ctx) { return ctx->sample_rate != 16000 || ctx->rate_override; }

// NoiseEstimator::Create (lyra/noise_estimator.cc:99-120) for (rate_hz, hop 320, 160 features)
NoiseParams MakeNoiseParams(int rate_hz) {
  NoiseParams p{};
  const float secs_per_hop = static_cast<float>(320) / rate_hz;
  p.nf = 160;
  p.hops_per_update = (int)std::round(1.f / secs_per_hop);
  p.max_smoothing = std::pow(0.5f, secs_per_hop / 0.7f);
  p.bound_decay = std::pow(0.5f, secs_per_hop / 1.f);
  p.log_nf = std::log((double)160);
  return p;
}

// RAII pair of events around one kernel launch (no-op unless profiling is enabled, and for kernel kNoProf)
constexpr int kNoProf = -1;
struct ProfScope {
  lyra_b200_ctx* ctx;
  int k;
  cudaEvent_t stop = nullptr;
  cudaStream_t st;
  ProfScope(lyra_b200_ctx* c, int kernel, cudaStream_t stream) : ctx(c), k(kernel), st(stream) {
    if (!ctx->profiling || k == kNoProf) return;
    auto& pool = ctx->prof_events[k];
    if (ctx->prof_used[k] == pool.size()) {
      cudaEvent_t a, b;
      cudaEventCreate(&a);
      cudaEventCreate(&b);
      pool.emplace_back(a, b);
    }
    auto& ev = pool[ctx->prof_used[k]++];
    cudaEventRecord(ev.first, st);
    stop = ev.second;
  }
  ~ProfScope() { if (stop) cudaEventRecord(stop, st); }
};

// Every kernel launch goes through LAUNCH: the profiling scope of slot `prof` (0 .. LYRA_B200_NUM_KERNELS - 1, or kNoProf), the
// launch on `st`, one more in ctx->launches (lyra_b200_launch_count) and the launch's error check.  Evaluates to the return code.
template <typename Fn>
int Launch(lyra_b200_ctx* ctx, int prof, cudaStream_t st, Fn launch) {
  {
    ProfScope ps(ctx, prof, st);
    launch();
  }
  ctx->launches += 1;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}
#define LAUNCH(prof, kernel, grid, block, smem, st, ...) \
  Launch(ctx, (prof), (st), [&]() { LYRA_LAUNCH(kernel, grid, block, smem, st, __VA_ARGS__); })

void ProfDrain(lyra_b200_ctx* ctx) {
  for (int k = 0; k < LYRA_B200_NUM_KERNELS; ++k) {
    for (size_t i = 0; i < ctx->prof_used[k]; ++i) {
      float ms = 0.0f;
      if (cudaEventElapsedTime(&ms, ctx->prof_events[k][i].first, ctx->prof_events[k][i].second) == cudaSuccess) {
        ctx->prof_ms[k] += ms;
        ctx->prof_n[k] += 1;
      }
    }
    ctx->prof_used[k] = 0;
  }
}

// End of a synchronous host-buffer call.  Spinning (cudaStreamSynchronize) has the lowest wake-up latency; when more host
// threads wait than there are cores, sleeping on a blocking-sync event keeps them from starving the launching threads.
cudaError_t SyncStream(lyra_b200_ctx* ctx) {
  if (!ctx->blocking_sync) return cudaStreamSynchronize(ctx->stream);
  cudaError_t e = cudaEventRecord(ctx->ev_sync, ctx->stream);
  return e != cudaSuccess ? e : cudaEventSynchronize(ctx->ev_sync);
}

bool UseDevice(lyra_b200_ctx* ctx) {
  if (cudaSetDevice(ctx->device) == cudaSuccess) return true;
  ctx->err = "cudaSetDevice failed";
  return false;
}

bool RoleOk(lyra_b200_ctx* ctx, int role) {
  if (ctx->roles & role) return true;
  ctx->err = role == LYRA_B200_ROLE_ENCODER ? "this context was created without the encoder role" : "this context was created without the decoder role";
  return false;
}

bool BitsOk(lyra_b200_ctx* ctx, int num_bits) {
  // lyra/residual_vector_quantizer.cc:79-89,116-126
  if (num_bits <= 0 || num_bits > LYRA_B200_MAX_BITS) { ctx->err = "the number of bits cannot exceed 184"; return false; }
  if (num_bits % ctx->spec.bits_per_stage != 0) { ctx->err = "the number of bits has to be divisible by the bits per quantizer (4)"; return false; }
  return true;
}

// a bit count lyra_b200_set_stream_bits and import accept for a stream's own word: one the calls accept
bool StreamBitsOk(const lyra_b200_ctx* ctx, int bits) {
  return bits > 0 && bits <= LYRA_B200_MAX_BITS && bits % ctx->spec.bits_per_stage == 0;
}

// mirrored word w as the kernels get it: nullptr while every stream's word is 0 (the bits words of role index r are w = r)
const int* StreamWord(const lyra_b200_ctx* ctx, int w) { return ctx->own_words[w] ? ctx->d_stream_word[w] : nullptr; }

// stream `id`'s mirrored word w in the host mirror (and own_words)
void SetMirrorWord(lyra_b200_ctx* ctx, int w, int id, int value) {
  int& v = ctx->word_mirror[w][(size_t)id];
  ctx->own_words[w] += (value != 0) - (v != 0);
  v = value;
}

// A fresh stamp for ctx->id_seen: no stream is marked with it yet
uint32_t NextIdGen(lyra_b200_ctx* ctx) {
  if (++ctx->id_gen == 0) { std::fill(ctx->id_seen.begin(), ctx->id_seen.end(), 0u); ctx->id_gen = 1; }
  return ctx->id_gen;
}

// The rows of a call: n in [1, max_streams]; ids (nullptr: streams 0..n-1) in range and, unless allow_repeats, distinct.
int CheckIds(lyra_b200_ctx* ctx, const int32_t* ids, int n, bool allow_repeats) {
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  if (!ids) return LYRA_B200_OK;
  const uint32_t gen = NextIdGen(ctx);
  for (int k = 0; k < n; ++k) {
    const int id = ids[k];
    if (id < 0 || id >= ctx->max_streams) { ctx->err = "stream id out of range"; return LYRA_B200_EINVAL; }
    if (allow_repeats) continue;
    if (ctx->id_seen[(size_t)id] == gen) { ctx->err = "duplicate stream id in one call"; return LYRA_B200_EINVAL; }
    ctx->id_seen[(size_t)id] = gen;
  }
  return LYRA_B200_OK;
}

// Stream ids of a sparse call -> ctx->d_ids on ctx->stream; *d_ids stays nullptr for dense calls.  No synchronisation: a
// host-to-device copy from pageable memory returns once `ids` has been staged.
int UploadIds(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int** d_ids) {
  *d_ids = nullptr;
  if (!ids) return LYRA_B200_OK;
  CU(cudaMemcpyAsync(ctx->d_ids, ids, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  *d_ids = ctx->d_ids;
  return LYRA_B200_OK;
}

// Check the call's ids, then build / upload the (tile list, slot-of-stream) map for this call.  The copies are stream-ordered
// behind the previous call's kernels (sub-batch streams are joined into ctx->stream at the end of every call), and the pinned
// host image is double-buffered, so a server whose active set changes every tick never waits for the GPU here.
int PrepareMap(lyra_b200_ctx* ctx, const int32_t* ids, int n) {
  int rc = CheckIds(ctx, ids, n, false);
  if (rc) return rc;
  if (ids == nullptr && ctx->map_dense_n == n) return LYRA_B200_OK;
  const int b = ctx->map_buf;
  if (ctx->map_pending[b]) { CU(cudaEventSynchronize(ctx->ev_map[b])); ctx->map_pending[b] = false; }   // two calls ago: long done
  int* slot_of = ctx->h_slot_of[b];
  int* tile_list = ctx->h_tile_list[b];
  for (int id : ctx->touched[b]) slot_of[id] = -1;
  ctx->touched[b].clear();
  int ntl = 0;
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    slot_of[id] = k;
    ctx->touched[b].push_back(id);
  }
  // tiles in order of first appearance
  if (++ctx->map_gen == 0) { std::fill(ctx->tile_gen.begin(), ctx->tile_gen.end(), 0u); ctx->map_gen = 1; }
  for (int k = 0; k < n; ++k) {
    const int t = (ids ? ids[k] : k) / kTileStreams;
    if (ctx->tile_gen[(size_t)t] != ctx->map_gen) { ctx->tile_gen[(size_t)t] = ctx->map_gen; tile_list[ntl++] = t; }
  }
  ctx->active_tiles = ntl;
  CU(cudaMemcpyAsync(ctx->d_slot_of, slot_of, sizeof(int) * (size_t)ctx->padded, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->d_tile_list, tile_list, sizeof(int) * (size_t)ntl, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaEventRecord(ctx->ev_map[b], ctx->stream));
  ctx->map_pending[b] = true;
  ctx->map_buf = b ^ 1;
  ctx->map_dense_n = ids ? -1 : n;
  return LYRA_B200_OK;
}

// A contiguous part of the current call: tiles [tile0, tile0 + ntiles) of the tile list, I/O slots
// [slot0, slot0 + nslots), launched on stream `st`.
struct Part {
  int tile0, ntiles, slot0, nslots;
  cudaStream_t st;
};
Part WholeCall(lyra_b200_ctx* ctx, int n) { return Part{0, ctx->active_tiles, 0, n, ctx->stream}; }

// The rows of part `p` as the per-row kernels see them: ids (nullptr: slot s is stream s, or no kernel reads a stream id) and
// active (lyra_b200_set_active_mask's buffer, by slot; nullptr: every slot runs)
RowIo Rows(const Part& p, const int* ids, const uint8_t* active) { return RowIo{ids, p.slot0, p.nslots, active}; }

// The per-stream words of the kernels that run every stream at 16 kHz and read no word of their own: the decoder side's noise
// estimators (they stay at 16 kHz, lyra/lyra_decoder.cc:122-132, and have no DTX switch) and lyra_b200_logmel
constexpr StreamWords kWords16k{nullptr, 16000, nullptr, nullptr};

// active: lyra_b200_set_active_mask's buffer by slot (nullptr: none), as in RowIo
int LaunchEncoderNets(lyra_b200_ctx* ctx, const Part& p, const uint8_t* skip, const int16_t* d_pcm, float* d_features,
                      const uint8_t* active) {
  const TileIo io{ctx->d_tile_list + p.tile0, ctx->d_slot_of, skip, active};
  const int rc = LAUNCH(0, EncoderKernelA, dim3((unsigned)p.ntiles), dim3(EncA::NT), (size_t)EncA::kSmemBytes, p.st,
                        ctx->d_blob, ctx->spec.enc, io, d_pcm, reinterpret_cast<float*>(ctx->d_state[0]), ctx->d_n18[0], ctx->d_mid_enc);
  return rc ? rc : LAUNCH(1, EncoderKernelB, dim3((unsigned)p.ntiles), dim3(EncB::NT), (size_t)EncB::kSmemBytes, p.st,
                          ctx->d_blob, ctx->spec.enc, io, ctx->d_mid_enc, reinterpret_cast<float*>(ctx->d_state[1]), ctx->d_n18[1], d_features);
}

int LaunchQuantize(lyra_b200_ctx* ctx, cudaStream_t st, const RowIo& io, const StreamWords& words, const float* d_features, int num_bits,
                   uint8_t* d_packets, int* d_indices, const uint8_t* d_skip) {
  const int nq = num_bits / ctx->spec.bits_per_stage, pb = PacketBytes(num_bits);
  const int blocks = (io.slots + kRvqSlotsPerBlock - 1) / kRvqSlotsPerBlock;
  return LAUNCH(2, RvqEncodeKernel, dim3((unsigned)blocks), dim3(kRvqThreads), (size_t)(2 * 1024 * 4 + kRvqSlotsPerBlock * (64 * 4 + 48 * 4)), st,
                ctx->d_blob, ctx->spec.rvq, io, words, d_features, nq, d_packets, pb, d_indices, d_skip);
}

// sat_out_pcm: the 16 kHz PCM rows by slot that the slots sitting out get as zeros (nullptr: none)
int LaunchDequantize(lyra_b200_ctx* ctx, cudaStream_t st, const RowIo& io, const StreamWords& words, const uint8_t* d_packets,
                     const uint8_t* d_received, int num_bits, float* d_features, int16_t* sat_out_pcm) {
  const int nq = num_bits / ctx->spec.bits_per_stage, pb = PacketBytes(num_bits);
  const int blocks = (io.slots * 64 + 255) / 256;
  return LAUNCH(3, RvqDecodeKernel, dim3((unsigned)blocks), dim3(256), (size_t)0, st,
                ctx->d_blob, ctx->spec.rvq, io, words, d_packets, pb, d_received, nq, d_features, sat_out_pcm);
}

// Exact mode: DecoderKernelC<false> + DecoderKernelD, fp32 FMA chains bit-exact with the oracle.  Tensor mode: DecoderKernelC<true>
// (decoder_1's 1x1 convolutions on mma.sync TF32) + DecoderKernelDW (warpgroup MMAs, A operands and accumulators in registers;
// net_kernels_wgmma.cuh).
int LaunchDecoderNets(lyra_b200_ctx* ctx, const Part& p, const uint8_t* skip, const float* d_features, int16_t* d_pcm,
                      const uint8_t* active) {
  const TileIo io{ctx->d_tile_list + p.tile0, ctx->d_slot_of, skip, active};
  const bool tc = ctx->decoder_mode == LYRA_B200_DECODER_TENSOR;
  const dim3 grid((unsigned)p.ntiles);
  float* st_c = reinterpret_cast<float*>(ctx->d_state[2]);
  float* st_d = reinterpret_cast<float*>(ctx->d_state[3]);
  const int rc = tc ? LAUNCH(4, DecoderKernelC<true>, grid, dim3(DecC<true>::NT), (size_t)DecC<true>::kSmemBytes, p.st,
                             ctx->d_blob, ctx->spec.dec, io, d_features, st_c, ctx->d_n18[2], ctx->d_mid_dec)
                    : LAUNCH(4, DecoderKernelC<false>, grid, dim3(DecC<false>::NT), (size_t)DecC<false>::kSmemBytes, p.st,
                             ctx->d_blob, ctx->spec.dec, io, d_features, st_c, ctx->d_n18[2], ctx->d_mid_dec);
  if (rc) return rc;
  return tc ? LAUNCH(5, DecoderKernelDW, grid, dim3(DecDW::NT), (size_t)DecDW::kSmemBytes, p.st,
                     ctx->d_blob, ctx->spec.dec, io, ctx->d_mid_dec, st_d, ctx->d_n18[3], d_pcm)
            : LAUNCH(5, DecoderKernelD, grid, dim3(DecD::NT), (size_t)DecD::kSmemBytes, p.st,
                     ctx->d_blob, ctx->spec.dec, io, ctx->d_mid_dec, st_d, ctx->d_n18[3], d_pcm);
}

// Dense calls over many tiles are cut into sub-batches (default 3) that run on their own CUDA streams: the block
// scheduler then fills the partial last wave of one sub-batch's kernel with blocks of another's (independent
// streams, so no ordering between them) and co-schedules blocks of different kernels on an SM, which removes most
// of the wave-quantisation loss of 512 tiles on 2-3 x 132 block slots and mixes FMA-bound with latency-bound phases.
int SplitParts(lyra_b200_ctx* ctx, int n, Part* parts) {
  int np = ctx->nsplit < 1 ? 1 : (ctx->nsplit > lyra_b200_ctx::kMaxSplit ? lyra_b200_ctx::kMaxSplit : ctx->nsplit);
  if (!(ctx->map_dense_n == n && ctx->active_tiles >= 64 * np)) np = 1;
  if (np == 1) { parts[0] = WholeCall(ctx, n); return 1; }
  for (int i = 0; i < np; ++i) {
    const int t0 = (int)((long long)ctx->active_tiles * i / np), t1 = (int)((long long)ctx->active_tiles * (i + 1) / np);
    const int s0 = t0 * kTileStreams, s1 = i + 1 == np ? n : t1 * kTileStreams;
    parts[i] = Part{t0, t1 - t0, s0, s1 - s0, i == 0 ? ctx->stream : ctx->aux_stream[i - 1]};
  }
  return np;
}
int Fork(lyra_b200_ctx* ctx, int nparts) {
  if (nparts < 2) return LYRA_B200_OK;
  CU(cudaEventRecord(ctx->ev_fork, ctx->stream));
  for (int i = 1; i < nparts; ++i) CU(cudaStreamWaitEvent(ctx->aux_stream[i - 1], ctx->ev_fork, 0));
  return LYRA_B200_OK;
}
int Join(lyra_b200_ctx* ctx, int nparts) {
  for (int i = 1; i < nparts; ++i) {
    CU(cudaEventRecord(ctx->ev_join[i - 1], ctx->aux_stream[i - 1]));
    CU(cudaStreamWaitEvent(ctx->stream, ctx->ev_join[i - 1], 0));
  }
  return LYRA_B200_OK;
}
// End of a forked region: the sub-batch streams are ALWAYS joined back, also when a copy or launch inside the region failed
// (`rc` != 0) - otherwise the next call would race leftover work on them.  After a failure the stream is drained as well and
// the caller gets the first error; per-stream state of the sub-batches that did run has advanced (the call is not atomic).
int JoinAfter(lyra_b200_ctx* ctx, int nparts, int rc) {
  if (!rc) return Join(ctx, nparts);
  const std::string first = ctx->err;
  Join(ctx, nparts);
  cudaStreamSynchronize(ctx->stream);
  ctx->err = first;
  return rc;
}

// Runs body(part) -> return code for every sub-batch of the call (SplitParts) inside a forked region; stops at the first error
template <typename Fn>
int ForEachPart(lyra_b200_ctx* ctx, int n, Fn body) {
  Part parts[lyra_b200_ctx::kMaxSplit];
  const int np = SplitParts(ctx, n, parts);
  int rc = Fork(ctx, np);
  if (rc) return rc;
  for (int i = 0; i < np && !rc; ++i) rc = body(parts[i]);
  return JoinAfter(ctx, np, rc);
}

// log-mel spectra of the rows `io` into `out` (by slot, num_mel floats per row) on stream `st`, advancing the extractor state
// `carried`.  S: the extractor's tables by rate, used per stream at its rate (one set: Uniform; the sets share their sizes)
int LaunchLogMel(lyra_b200_ctx* ctx, cudaStream_t st, const RowIo& io, const ByRate<LogMelParams>& S, const StreamWords& words,
                 const int16_t* d_pcm, int16_t* carried, const uint8_t* d_mask, float* out) {
  const LogMelParams& P = S.p[0];
  const size_t smem = sizeof(double) * (size_t)(2 * kLogMelFftPadded + P.fft / 2 + 1 + P.window_len + P.window_len / 8 + 1);
  return LAUNCH(6, LogMelKernel, dim3((unsigned)io.slots), dim3(kLogMelThreads), smem, st,
                ctx->d_blob, S, words, io, d_pcm, carried, out, d_mask);
}

// log-mel of this hop (the estimator's own extractor, bank 2) + the estimator recurrences for the rows `io` on stream `st`.
// encoder_side: the encoder side's estimators, built for each stream's rate (NoiseEstimator::Create(rate, 320, 640, 160),
// lyra/lyra_encoder.cc:80-89) and skipping the streams whose DTX is off (flag 0, state untouched), with the encoder role's words;
// otherwise the decoder side's, with kWords16k.  Streams that sit out feed neither side: the encoder side reports flag 1, the
// decoder side its current flag.
int LaunchNoiseUpdate(lyra_b200_ctx* ctx, cudaStream_t st, const RowIo& io, const StreamWords& words, bool encoder_side,
                      const int16_t* d_pcm, const uint8_t* d_mask, uint8_t* d_is_noise, float* d_estimate) {
  const int rc = LaunchLogMel(ctx, st, io, encoder_side ? ctx->enc_logmel : Uniform(ctx->spec.logmel160), words, d_pcm,
                              encoder_side ? ctx->d_logmel_prev_enc : ctx->d_logmel_prev[2], d_mask, ctx->d_melout);
  return rc ? rc : LAUNCH(7, NoiseEstimatorKernel, dim3((unsigned)io.slots), dim3(kNoiseThreads), sizeof(float) * (size_t)(2 * 160 + 2), st,
                          encoder_side ? ctx->enc_noise_params : Uniform(ctx->noise_params), words, io, ctx->d_melout, d_mask,
                          encoder_side ? ctx->d_noise_enc : ctx->d_noise, d_is_noise, d_estimate, encoder_side);
}

// comfort noise of the rows `io` into `out` (by slot, 320 samples per row) on stream `st`: from `d_features` (log-mel by slot)
// or, when that is nullptr, from the streams' noise estimates; d_plan (by slot, nullptr: every slot) selects the slots that need it
int LaunchComfortNoise(lyra_b200_ctx* ctx, cudaStream_t st, const RowIo& io, const float* d_features, const uint8_t* d_plan,
                       int16_t* out) {
  const size_t smem = sizeof(double) * (size_t)(4 * kLogMelFftPadded + 160);
  return LAUNCH(kNoProf, ComfortNoiseKernel, dim3((unsigned)io.slots), dim3(kCngThreads), smem, st,
                ctx->d_blob, ctx->spec.cng, io, d_features, ctx->d_noise, NoiseStateUnits(ctx->noise_params.nf),
                d_plan, ctx->d_cng_work, ctx->d_cng_hops, ctx->cng_seed, out);
}

// The codec path's sample-rate converter for the rows `io` on stream `st`: dir 0 converts the external-rate rows `in`
// [slot][rate / 50] to 16 kHz rows `out` [slot][320] (the encoder's input side), dir 1 the 16 kHz rows to external-rate rows (the
// decoder's output side).  Each stream converts at its own rate (words.rate; rows of a stream below the context's rate use their
// first rate / 50 samples, decoder rows get zeros after them).  Whole hops from phase 0 stay at phase 0 (the ratios are
// integers), so every row is exactly one hop.
int LaunchCodecResample(lyra_b200_ctx* ctx, cudaStream_t st, const RowIo& io, const StreamWords& words, int dir, const int16_t* in,
                        int16_t* out) {
  const int ext = ctx->sample_rate / 50;
  const int in_stride = dir ? LYRA_B200_HOP : ext, out_stride = dir ? ext : LYRA_B200_HOP;
  return LAUNCH(kNoProf, ResampleKernel, dim3((unsigned)io.slots), dim3(128), sizeof(float) * (size_t)(kResamplerTaps - 1 + in_stride), st,
                ctx->d_blob, ctx->spec.resampler, dir ? 3 : 0, ctx->codec_rs_tag, io, words, in, in_stride, in_stride, out, out_stride,
                nullptr, ctx->d_codec_rs_delay[dir], ctx->d_codec_rs_pos[dir]);
}

// The five fused codec calls; kEncode and kDecode are also GraphKey::kind
enum CallKind { kEncode, kDecode, kEncodeDtx, kDecodeTrackNoise, kDecodePlc };

// One fused codec call.  `dev` holds the buffers its kernels use: a *_device twin's own, or for a host-buffer call the context's
// staging, between which and the caller's buffers `host` (all nullptr for a twin) the call copies.  RunCodecCall fills in the
// staging, the default flag buffer, d_ids, active and words.
struct CodecCall {
  struct Io {
    const int16_t* pcm_in = nullptr;       // the encoders' rows
    int16_t* pcm_out = nullptr;            // the decoders' rows
    const uint8_t* packets_in = nullptr;   // the decoders' packets
    uint8_t* packets_out = nullptr;        // the encoders' packets
    const uint8_t* received = nullptr;     // nullptr: every packet arrived
    uint8_t* flags = nullptr;              // by slot: DTX hops (encode_dtx), noise (decode_track_noise), comfort noise (decode_plc)
  };
  CallKind kind;
  int n, num_bits;
  const int32_t* ids = nullptr;            // stream ids; nullptr: streams 0..n-1 (always for a twin)
  Io dev, host;
  int32_t* packet_bytes = nullptr;         // lyra_b200_encode_dtx: per row 0 for a DTX hop, else the packet's size
  const int* d_ids = nullptr;              // the ids on the device, for chains with kernels indexed by stream id
  const uint8_t* active = nullptr;         // a twin's lyra_b200_set_active_mask buffer, by slot (nullptr: every stream runs)
  StreamWords words{};                     // the per-stream words of the call's role
};

// lyra_b200_set_stats: CallStatsKernel over part p's rows of `pcm` (the encoders' input rows, the decoders' output rows, at the
// external rate) with the call's event source (StatsSource); nothing while statistics are off
int LaunchCallStats(lyra_b200_ctx* ctx, const Part& p, const CodecCall& c, const int16_t* pcm, const uint8_t* events) {
  if (!ctx->stats_on) return LYRA_B200_OK;
  const bool encoder = c.kind == kEncode || c.kind == kEncodeDtx;
  const int source = c.kind == kEncode ? kStatsEncode : c.kind == kEncodeDtx ? kStatsEncodeDtx : c.kind == kDecodePlc ? kStatsDecodePlc : kStatsDecode;
  return LAUNCH(kNoProf, CallStatsKernel, dim3((unsigned)((p.nslots + kStatsRowsPerBlock - 1) / kStatsRowsPerBlock)), dim3(kStatsThreads),
                (size_t)0, p.st, Rows(p, c.d_ids, c.active), c.words, pcm, ctx->sample_rate / 50, source, events, c.num_bits,
                ctx->d_stats_levels, ctx->d_stats[encoder ? 0 : 1]);
}

// encode / encode_dtx.  PCM rows hold ctx->sample_rate / 50 samples (the external rate).  At 16 kHz the encoder reads the rows
// (a host-buffer call's are copied to ctx->d_pcm first); at another rate every sub-batch first converts them into the 16 kHz scratch
// ctx->d_pcm (a host-buffer call stages its rows in ctx->d_rs_in instead).  Each part copies its own slice in on its own stream
// before its kernels and its result out right after them, so the copies of one part overlap the kernels of the others.
// encode_dtx: every sub-batch first feeds its 16 kHz hops to the encoder-side noise estimators; hops classified as noise skip the
// encoder (their streams' state does not advance) and get an empty packet (lyra/lyra_encoder.cc:131-141); flags[slot] = 1 marks
// them.  The converter runs for those hops too: the reference resamples before its DTX branch (:118-135).  A stream whose DTX is
// off (lyra_b200_set_stream_dtx) feeds no estimator and gets flag 0, so it is always encoded, as with enable_dtx = false.
// A stream that sits out (c.active) is not converted; in encode_dtx its estimator writes flag 1, which the encoder nets and the
// quantizer already skip, so only encode hands them the mask.
int RunEncode(lyra_b200_ctx* ctx, const CodecCall& c) {
  const CodecCall::Io &d = c.dev, &h = c.host;
  const bool dtx = c.kind == kEncodeDtx;
  const size_t pb = (size_t)PacketBytes(c.num_bits), hop = (size_t)ctx->sample_rate / 50;
  const bool rs = Converts(ctx);
  int16_t* stage = rs ? ctx->d_rs_in : ctx->d_pcm;      // where a host-buffer call's rows land
  const int16_t* in = h.pcm_in ? stage : d.pcm_in;
  const int16_t* pcm16 = rs ? ctx->d_pcm : in;
  const uint8_t* skip = dtx ? d.flags : nullptr;
  const uint8_t* active = dtx ? nullptr : c.active;
  return ForEachPart(ctx, c.n, [&](const Part& p) {
    int rc = LYRA_B200_OK;
    const RowIo io = Rows(p, c.d_ids, c.active);
    if (h.pcm_in)
      CU(cudaMemcpyAsync(stage + (size_t)p.slot0 * hop, h.pcm_in + (size_t)p.slot0 * hop, sizeof(int16_t) * hop * (size_t)p.nslots,
                         cudaMemcpyHostToDevice, p.st));
    if (rs && (rc = LaunchCodecResample(ctx, p.st, io, c.words, 0, in, ctx->d_pcm))) return rc;
    if (dtx) {
      if ((rc = LaunchNoiseUpdate(ctx, p.st, io, c.words, true, pcm16, nullptr, d.flags, nullptr))) return rc;
      if (h.flags) CU(cudaMemcpyAsync(h.flags + p.slot0, d.flags + p.slot0, (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
    }
    if ((rc = LaunchEncoderNets(ctx, p, skip, pcm16, ctx->d_features, active))) return rc;
    if ((rc = LaunchQuantize(ctx, p.st, Rows(p, c.d_ids, active), c.words, ctx->d_features, c.num_bits, d.packets_out, nullptr, skip)))
      return rc;
    if ((rc = LaunchCallStats(ctx, p, c, in, skip))) return rc;
    if (h.packets_out)
      CU(cudaMemcpyAsync(h.packets_out + (size_t)p.slot0 * pb, d.packets_out + (size_t)p.slot0 * pb, pb * (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
    return LYRA_B200_OK;
  });
}

// decode / decode_track_noise.  decode_track_noise: every sub-batch also feeds its decoded hops to the per-stream noise estimators
// (received streams only), as LyraDecoder::DecodeSamplesInternal does (lyra/lyra_decoder.cc:306-311).  PCM rows hold
// ctx->sample_rate / 50 samples.  At another rate than 16 kHz the decoder writes the 16 kHz scratch ctx->d_pcm, the estimator is
// fed from it (it stays at 16 kHz, lyra/lyra_decoder.cc:122-132), and one up-sampling launch per part writes the external-rate
// rows (to ctx->d_rs_out for a host-buffer call).  A stream that sits out (c.active) reads no packet, advances no state and
// gets a zero row (written by the RVQ decode at 16 kHz, which the decoder nets then skip, or by the converter); its noise flag
// reports the estimator as it is.
int RunDecode(lyra_b200_ctx* ctx, const CodecCall& c) {
  const CodecCall::Io &d = c.dev, &h = c.host;
  const size_t pb = (size_t)PacketBytes(c.num_bits), hop = (size_t)ctx->sample_rate / 50;
  const bool rs = Converts(ctx);
  int16_t* out = h.pcm_out && rs ? ctx->d_rs_out : d.pcm_out;
  int16_t* pcm16 = rs ? ctx->d_pcm : out;
  return ForEachPart(ctx, c.n, [&](const Part& p) {
    int rc = LYRA_B200_OK;
    const RowIo io = Rows(p, c.d_ids, c.active);
    if (h.packets_in)
      CU(cudaMemcpyAsync(ctx->d_packets + (size_t)p.slot0 * pb, h.packets_in + (size_t)p.slot0 * pb, pb * (size_t)p.nslots, cudaMemcpyHostToDevice, p.st));
    if (h.received)
      CU(cudaMemcpyAsync(ctx->d_received + p.slot0, h.received + p.slot0, (size_t)p.nslots, cudaMemcpyHostToDevice, p.st));
    if ((rc = LaunchDequantize(ctx, p.st, io, c.words, d.packets_in, d.received, c.num_bits, ctx->d_features, rs ? nullptr : out))) return rc;
    if ((rc = LaunchDecoderNets(ctx, p, nullptr, ctx->d_features, pcm16, c.active))) return rc;
    if (c.kind == kDecodeTrackNoise) {
      if ((rc = LaunchNoiseUpdate(ctx, p.st, io, kWords16k, false, pcm16, d.received, d.flags, nullptr))) return rc;
      if (h.flags) CU(cudaMemcpyAsync(h.flags + p.slot0, d.flags + p.slot0, (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
    }
    if (rs && (rc = LaunchCodecResample(ctx, p.st, io, c.words, 1, pcm16, out))) return rc;
    if ((rc = LaunchCallStats(ctx, p, c, out, d.received))) return rc;
    if (h.pcm_out)
      CU(cudaMemcpyAsync(h.pcm_out + (size_t)p.slot0 * hop, out + (size_t)p.slot0 * hop, sizeof(int16_t) * hop * (size_t)p.nslots,
                         cudaMemcpyDeviceToHost, p.st));
    return LYRA_B200_OK;
  });
}

// LyraDecoder::{SetEncodedPacket, DecodeSamples(320)} with the reference's concealment / comfort-noise / fade behaviour for n
// streams (lyra/lyra_decoder.cc:172-315): plan (per-stream state machine) -> RVQ decode -> LyraGAN for the streams that need
// model audio -> comfort noise from the current noise estimates for the streams that need it -> cross-fade -> noise-estimator
// update of the streams that decoded a received packet.  One whole hop per stream and call.  PCM rows and the conversion to the
// external rate as in RunDecode: the cross-fade writes the 16 kHz scratch, one up-sampling launch per part writes the rows.
// A stream that sits out (c.active) gets plan kPlanSatOut from PlcPlanKernel: the plan's skip and feed bytes keep it out of the
// decoder nets and the noise update, the comfort-noise generator skips it and the cross-fade writes zeros, so these kernels
// follow the plan and get no mask.
int RunDecodePlc(lyra_b200_ctx* ctx, const CodecCall& c) {
  const CodecCall::Io &d = c.dev, &h = c.host;
  const size_t pb = (size_t)PacketBytes(c.num_bits), hop = (size_t)ctx->sample_rate / 50;
  const bool rs = Converts(ctx);
  int16_t* out = h.pcm_out && rs ? ctx->d_rs_out : d.pcm_out;
  int16_t* pcm16 = rs ? ctx->d_pcm : out;
  if (h.received) CU(cudaMemcpyAsync(ctx->d_received, h.received, (size_t)c.n, cudaMemcpyHostToDevice, ctx->stream));
  if (int rc = LAUNCH(kNoProf, PlcPlanKernel, dim3((unsigned)((c.n + 255) / 256)), dim3(256), (size_t)0, ctx->stream,
                      Rows(WholeCall(ctx, c.n), c.d_ids, c.active), d.received, ctx->d_plc, ctx->d_plan, ctx->d_fade0, ctx->d_dir,
                      ctx->d_skip, ctx->d_feed, d.flags))
    return rc;
  return ForEachPart(ctx, c.n, [&](const Part& p) {
    int rc = LYRA_B200_OK;
    const RowIo io = Rows(p, c.d_ids, c.active), planned = Rows(p, c.d_ids, nullptr);
    if (h.packets_in)
      CU(cudaMemcpyAsync(ctx->d_packets + (size_t)p.slot0 * pb, h.packets_in + (size_t)p.slot0 * pb, pb * (size_t)p.nslots, cudaMemcpyHostToDevice, p.st));
    if ((rc = LaunchDequantize(ctx, p.st, io, c.words, d.packets_in, d.received, c.num_bits, ctx->d_features, nullptr))) return rc;
    if ((rc = LaunchDecoderNets(ctx, p, ctx->d_skip, ctx->d_features, ctx->d_model_pcm, nullptr))) return rc;
    if ((rc = LaunchComfortNoise(ctx, p.st, planned, nullptr, ctx->d_plan, ctx->d_cng_pcm))) return rc;
    if ((rc = LAUNCH(kNoProf, PlcMixKernel, dim3((unsigned)p.nslots), dim3(320), (size_t)0, p.st,
                     ctx->d_blob, ctx->spec.cng, planned, ctx->d_plan, ctx->d_fade0, ctx->d_dir, ctx->d_model_pcm, ctx->d_cng_pcm, pcm16)))
      return rc;
    if ((rc = LaunchNoiseUpdate(ctx, p.st, planned, kWords16k, false, ctx->d_model_pcm, ctx->d_feed, nullptr, nullptr))) return rc;
    if (rs && (rc = LaunchCodecResample(ctx, p.st, io, c.words, 1, pcm16, out))) return rc;
    if ((rc = LaunchCallStats(ctx, p, c, out, ctx->d_plan))) return rc;
    if (h.pcm_out)
      CU(cudaMemcpyAsync(h.pcm_out + (size_t)p.slot0 * hop, out + (size_t)p.slot0 * hop, sizeof(int16_t) * hop * (size_t)p.nslots,
                         cudaMemcpyDeviceToHost, p.st));
    if (h.flags) CU(cudaMemcpyAsync(h.flags + p.slot0, d.flags + p.slot0, (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
    return LYRA_B200_OK;
  });
}

bool SetSmemLimits() {
  return LYRA_SET_MAX_SMEM(EncoderKernelA, EncA::kSmemBytes) == 0 && LYRA_SET_MAX_SMEM(EncoderKernelB, EncB::kSmemBytes) == 0 &&
         LYRA_SET_MAX_SMEM(DecoderKernelC<false>, DecC<false>::kSmemBytes) == 0 && LYRA_SET_MAX_SMEM(DecoderKernelD, DecD::kSmemBytes) == 0 &&
         LYRA_SET_MAX_SMEM(DecoderKernelC<true>, DecC<true>::kSmemBytes) == 0 && LYRA_SET_MAX_SMEM(DecoderKernelDW, DecDW::kSmemBytes) == 0;
}

// initial value of every 4-byte state unit (all zero; int8 rings hold packed zero points)
std::vector<uint32_t> InitImage(const ModelSpec& s, int which) {
  auto pack = [](int zp) { const uint32_t b = (uint32_t)(zp & 0xff); return b | (b << 8) | (b << 16) | (b << 24); };
  std::vector<uint32_t> v;
  if (which == 0) {
    v.assign(EncStateA::kUnits, 0u);
  } else if (which == 1) {
    v.assign(EncStateB::kUnits, 0u);
    for (int i = EncStateB::kRingQ0; i < EncStateB::kRingQ1; ++i) v[(size_t)i] = pack(s.enc.zp_state[0]);
    for (int i = EncStateB::kRingQ1; i < EncStateB::kDown2; ++i) v[(size_t)i] = pack(s.enc.zp_state[1]);
    for (int i = EncStateB::kDown2; i < EncStateB::kBott; ++i) v[(size_t)i] = pack(s.enc.zp_state[2]);
    for (int i = EncStateB::kBott; i < EncStateB::kUnits; ++i) v[(size_t)i] = pack(s.enc.zp_state[3]);
  } else if (which == 2) {
    v.assign(DecStateC::kUnits, 0u);
    for (int i = DecStateC::kRingM; i < DecStateC::kRingQ0; ++i) v[(size_t)i] = pack(s.dec.zp_state[0]);
    for (int i = DecStateC::kRingQ0; i < DecStateC::kRingQ1; ++i) v[(size_t)i] = pack(s.dec.zp_state[1]);
    for (int i = DecStateC::kRingQ1; i < DecStateC::kUnits; ++i) v[(size_t)i] = pack(s.dec.zp_state[2]);
  } else {
    v.assign(DecStateD::kUnits, 0u);
  }
  return v;
}

// a zero-filled device allocation of `count` elements, recorded in ctx->allocs
template <typename T>
bool DevAlloc(lyra_b200_ctx* ctx, T** p, size_t count) {
  const size_t bytes = sizeof(T) * (count ? count : 1);
  if (cudaMalloc(reinterpret_cast<void**>(p), bytes) != cudaSuccess) return false;
  ctx->allocs.push_back(*p);
  return cudaMemset(*p, 0, bytes) == cudaSuccess;
}

// a device allocation of `per_stream` elements for each of the context's streams at lane stride `lanes` (1: row-major
// [padded][per_stream]; 8: [tile][per_stream][8]), and with n18 != nullptr a hop counter per stream in *n18, appended to
// ctx->state_list with a device copy of `init` (host image of one row; nullptr: zero).  lyra_b200_ctx::StateEntry says what
// the other arguments mean.
template <typename T>
bool DevStreamState(lyra_b200_ctx* ctx, T** p, size_t per_stream, const void* init = nullptr, int kind = kStatePlain,
                    int check = lyra_b200_ctx::kCheckNone, bool reset = true, int lanes = 1, int** n18 = nullptr) {
  const int words = (int)(sizeof(T) * per_stream / 4);
  uint32_t* d_init = nullptr;
  if (!DevAlloc(ctx, p, (size_t)ctx->padded * per_stream)) return false;
  if (n18 && !DevAlloc(ctx, n18, (size_t)ctx->padded)) return false;
  if (init && !(DevAlloc(ctx, &d_init, (size_t)words) && cudaMemcpy(d_init, init, 4 * (size_t)words, cudaMemcpyHostToDevice) == cudaSuccess))
    return false;
  ctx->state_list.push_back({{reinterpret_cast<uint32_t*>(*p), d_init, n18 ? *n18 : nullptr, words, lanes, 0, kind}, reset, check});
  return true;
}

// 64-bit FNV-1a over the weight blob, 8 bytes at a time (and its size): tells records of another model apart
uint64_t ModelFingerprint(const std::vector<uint8_t>& blob) {
  uint64_t h = 0xcbf29ce484222325ull ^ (uint64_t)blob.size();
  size_t i = 0;
  for (; i + 8 <= blob.size(); i += 8) {
    uint64_t w;
    std::memcpy(&w, blob.data() + i, 8);
    h = (h ^ w) * 0x100000001b3ull;
  }
  for (; i < blob.size(); ++i) h = (h ^ blob[i]) * 0x100000001b3ull;
  return h;
}

// ctx->state_table from ctx->state_list (payload offsets in list order) and the constant header words; ctx->reset_table and
// ctx->dtx_table
bool BuildStateTable(lyra_b200_ctx* ctx) {
  StreamStateTable& T = ctx->state_table;
  StreamStateTable& R = ctx->reset_table;
  StreamStateTable& D = ctx->dtx_table;
  if ((int)ctx->state_list.size() > kStateMaxEntries) return false;
  int off = 0;
  T.count = R.count = D.count = 0;
  for (lyra_b200_ctx::StateEntry& s : ctx->state_list) {
    s.e.offset = off;
    off += s.e.words + (s.e.n18 ? 1 : 0);
    T.e[T.count++] = s.e;
    if (s.reset) R.e[R.count++] = s.e;
    if (s.e.state == reinterpret_cast<uint32_t*>(ctx->d_noise_enc) || s.e.state == reinterpret_cast<uint32_t*>(ctx->d_logmel_prev_enc))
      D.e[D.count++] = s.e;
  }
  T.record_words = kStateHeaderWords + off;
  std::memset(T.header, 0, sizeof(T.header));
  T.header[kHdrMagic] = kStateMagic;
  T.header[kHdrVersion] = kStateVersion;
  T.header[kHdrBytes] = (uint32_t)(4 * T.record_words);
  T.header[kHdrRoles] = (uint32_t)ctx->roles;
  T.header[kHdrModelLo] = (uint32_t)ctx->model_fingerprint;
  T.header[kHdrModelHi] = (uint32_t)(ctx->model_fingerprint >> 32);
  return true;
}

#ifndef LYRA_EMU
bool PinnedHost(const void* p) {
  if (p == nullptr) return true;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeHost;
}
void DropGraphs(lyra_b200_ctx* ctx) {
  for (auto& e : ctx->graphs) cudaGraphExecDestroy(reinterpret_cast<cudaGraphExec_t>(e.exec));
  ctx->graphs.clear();
}
#endif

// Runs `enqueue` (which only issues asynchronous work on the context's streams) either directly or, for a dense call on pinned
// host buffers with graphs enabled, as a captured graph that later calls of the same shape replay.  Any capture problem turns
// graphs off for the context and the call proceeds directly: correctness never depends on the graph path.
template <typename Fn>
int RunMaybeGraphed(lyra_b200_ctx* ctx, const lyra_b200_ctx::GraphKey& key, bool eligible, Fn enqueue) {
#ifdef LYRA_EMU
  (void)key; (void)eligible;
  return enqueue();
#else
  if (!ctx->use_graphs || !eligible || ctx->profiling || !PinnedHost(key.a) || !PinnedHost(key.b) || !PinnedHost(key.c)) return enqueue();
  for (auto& e : ctx->graphs)
    if (e.key == key) {
      CU(cudaGraphLaunch(reinterpret_cast<cudaGraphExec_t>(e.exec), ctx->stream));
      ctx->launches += e.launches;
      ++ctx->graph_replays;
      return LYRA_B200_OK;
    }
  const uint64_t l0 = ctx->launches;
  if (cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
    cudaGetLastError();
    ctx->use_graphs = false;
    return enqueue();
  }
  const int rc = enqueue();
  cudaGraph_t g = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(ctx->stream, &g);
  cudaGraphExec_t exec = nullptr;
  if (rc == LYRA_B200_OK && ce == cudaSuccess && g != nullptr && cudaGraphInstantiate(&exec, g, 0) == cudaSuccess) {
    cudaGraphDestroy(g);
    if (ctx->graphs.size() >= 32) {
      cudaGraphExecDestroy(reinterpret_cast<cudaGraphExec_t>(ctx->graphs.front().exec));
      ctx->graphs.erase(ctx->graphs.begin());
    }
    ctx->graphs.push_back(lyra_b200_ctx::GraphEntry{key, exec, ctx->launches - l0});
    CU(cudaGraphLaunch(exec, ctx->stream));
    return LYRA_B200_OK;
  }
  // nothing was executed (the work was only recorded): give up on graphs and issue the call directly
  if (g) cudaGraphDestroy(g);
  cudaGetLastError();
  ctx->use_graphs = false;
  ctx->launches = l0;
  return enqueue();
#endif
}

// Every fused codec call past its own pointer checks: role, bit count (also against the listed streams' own counts, from the host
// mirror), tile map; the stream ids go to the device when the call's chain has a kernel indexed by stream id (the converters, the
// noise estimators, the PLC kernels, the RVQ kernels while some stream of the role has its own bit count, CallStatsKernel while
// statistics are on).  A host-buffer call runs on the
// context's staging buffers, a call without a flag buffer on the context's, and only the dense host-buffer encode / decode may
// replay a graph.  A host-buffer call returns when its results are in the caller's buffers; a *_device twin never waits.
int RunCodecCall(lyra_b200_ctx* ctx, CodecCall c) {
  const bool encoder = c.kind == kEncode || c.kind == kEncodeDtx;
  const int role = encoder ? LYRA_B200_ROLE_ENCODER : LYRA_B200_ROLE_DECODER;
  ENTER(role);
  if (!BitsOk(ctx, c.num_bits)) return LYRA_B200_EINVAL;
  const int r = encoder ? kWordEncBits : kWordDecBits;
  const std::vector<int>& own = ctx->word_mirror[r];
  for (int k = 0; k < c.n && ctx->own_words[r]; ++k) {
    const int id = c.ids ? c.ids[k] : k;            // an id out of range is refused by PrepareMap
    if (id >= 0 && id < ctx->max_streams && own[(size_t)id] > c.num_bits) {
      ctx->err = "a listed stream's own bit count (lyra_b200_set_stream_bits) is above the call's num_bits";
      return LYRA_B200_EINVAL;
    }
  }
  const bool by_id = Converts(ctx) || (c.kind != kEncode && c.kind != kDecode) || ctx->own_words[r] || ctx->stats_on;
  int rc = PrepareMap(ctx, c.ids, c.n);
  if (rc || (by_id && (rc = UploadIds(ctx, c.ids, c.n, &c.d_ids)))) return rc;
  const bool host = c.host.packets_in || c.host.packets_out;
  if (host) {
    c.dev.pcm_in = c.dev.pcm_out = ctx->d_pcm;
    c.dev.packets_in = c.dev.packets_out = ctx->d_packets;
    c.dev.received = c.host.received ? ctx->d_received : nullptr;
  } else {
    c.active = ctx->d_active;                       // only the *_device twins read the mask: a host call's ids say who runs
  }
  if (!c.dev.flags) c.dev.flags = c.kind == kDecodePlc ? ctx->d_is_cn : ctx->d_is_noise;
  c.words = StreamWords{ctx->d_stream_rate, ctx->sample_rate, StreamWord(ctx, r), encoder ? StreamWord(ctx, kWordDtxOff) : nullptr};
  std::vector<uint8_t> dtx_flags;
  if (c.packet_bytes) {
    dtx_flags.resize((size_t)c.n);
    c.host.flags = dtx_flags.data();
  }
  const CodecCall::Io& h = c.host;
  const lyra_b200_ctx::GraphKey key =
      encoder ? lyra_b200_ctx::GraphKey{kEncode, c.n, c.num_bits, 0, ctx->nsplit, h.pcm_in, h.packets_out, nullptr, ctx->rate_override,
                                        ctx->own_words[r] != 0, ctx->stats_on}
              : lyra_b200_ctx::GraphKey{kDecode, c.n, c.num_bits, ctx->decoder_mode, ctx->nsplit, h.packets_in, h.received, h.pcm_out,
                                        ctx->rate_override, ctx->own_words[r] != 0, ctx->stats_on};
  const bool graphed = host && (c.kind == kEncode || c.kind == kDecode) && c.ids == nullptr && ctx->map_dense_n == c.n;
  if ((rc = RunMaybeGraphed(ctx, key, graphed, [&]() {
         return encoder ? RunEncode(ctx, c) : c.kind == kDecodePlc ? RunDecodePlc(ctx, c) : RunDecode(ctx, c);
       })))
    return rc;
  if (!host) return LYRA_B200_OK;
  CU(SyncStream(ctx));
  for (int k = 0; k < c.n && c.packet_bytes; ++k) {
    const int b = own[(size_t)(c.ids ? c.ids[k] : k)];
    c.packet_bytes[k] = dtx_flags[(size_t)k] ? 0 : PacketBytes(b ? b : c.num_bits);
  }
  return LYRA_B200_OK;
}

// ---- stream-state records (lyra_b200_export_streams / _import_streams / _copy_streams) ----

size_t RecordBytes(const lyra_b200_ctx* ctx) { return 4 * (size_t)ctx->state_table.record_words; }

// the export / import staging: as many records as fit in 64 MB (at least one, at most one kernel chunk), allocated on first use
int EnsureRecordStaging(lyra_b200_ctx* ctx) {
  if (ctx->d_records) return LYRA_B200_OK;
  const size_t fit = ((size_t)64 << 20) / RecordBytes(ctx);
  const int chunk = fit < 1 ? 1 : fit > (size_t)kStateChunk ? kStateChunk : (int)fit;
  uint32_t* p = nullptr;
  CU(cudaMalloc(reinterpret_cast<void**>(&p), RecordBytes(ctx) * (size_t)chunk));
  ctx->allocs.push_back(p);
  ctx->d_records = p;
  ctx->records_chunk = chunk;
  return LYRA_B200_OK;
}

// a decoder control state lyra_b200_plc_set_state and import accept: hop-aligned concealment 0..1280, fade 0..640, direction +-1
bool PlcStateOk(int cp, int fp, int dir) {
  return cp >= 0 && cp <= kPlcConcealSamples && cp % 320 == 0 && fp >= 0 && fp <= kPlcFadeSamples && fp % 320 == 0 &&
         (dir == 1 || dir == -1);
}

// a rate lyra_b200_set_stream_sample_rates accepts: supported, and its hop fits the context's rows
bool StreamRateOk(const lyra_b200_ctx* ctx, int rate_hz) { return RateOk(rate_hz) && rate_hz <= ctx->sample_rate; }

uint32_t RecordWord(const uint8_t* rec, int i) {
  uint32_t w;
  std::memcpy(&w, rec + 4 * (size_t)i, 4);
  return w;
}

// Why record `rec` cannot be imported into this context (nullptr: it can).  Besides the header, the payload words that index
// memory are range-checked, so a damaged record cannot make a kernel read out of bounds: hop counters, the decoder control state
// (as lyra_b200_plc_set_state) and the resamplers' positions.
const char* RecordProblem(const lyra_b200_ctx* ctx, const uint8_t* rec) {
  const StreamStateTable& T = ctx->state_table;
  if (RecordWord(rec, kHdrMagic) != kStateMagic) return "not a stream-state record";
  if (RecordWord(rec, kHdrVersion) != kStateVersion) return "record format version differs";
  if (RecordWord(rec, kHdrBytes) != T.header[kHdrBytes] || RecordWord(rec, kHdrRoles) != T.header[kHdrRoles])
    return "record size / roles differ from this context's";
  if (RecordWord(rec, kHdrRate) != (uint32_t)ctx->sample_rate) return "record is from a context at another sample rate";
  if (RecordWord(rec, kHdrModelLo) != T.header[kHdrModelLo] || RecordWord(rec, kHdrModelHi) != T.header[kHdrModelHi])
    return "record is from another model";
  if (RecordWord(rec, kHdrZero5) || RecordWord(rec, kHdrLive0) > 1 || RecordWord(rec, kHdrLive1) > 1) return "malformed record header";
  for (int i = kHdrKeyHi + 1; i < kStateHeaderWords; ++i)
    if (RecordWord(rec, i)) return "malformed record header";
  for (int i = 0; i < T.count; ++i) {
    const StreamStateEntry& e = T.e[i];
    const int w0 = kStateHeaderWords + e.offset;
    if (e.n18 && RecordWord(rec, w0 + e.words) >= 18u) return "hop counter out of range";
    const int check = ctx->state_list[(size_t)i].check;
    if (check == lyra_b200_ctx::kCheckResamplerPos && (int32_t)RecordWord(rec, w0) < 0) return "resampler position out of range";
    if (check == lyra_b200_ctx::kCheckPlc &&
        !PlcStateOk((int32_t)RecordWord(rec, w0), (int32_t)RecordWord(rec, w0 + 1), (int32_t)RecordWord(rec, w0 + 2)))
      return "decoder control state out of range";
    if (check == lyra_b200_ctx::kCheckStreamRate && RecordWord(rec, w0) != 0 && !StreamRateOk(ctx, (int32_t)RecordWord(rec, w0)))
      return "stream sample rate unsupported or above the context's";
    if (check == lyra_b200_ctx::kCheckStreamBits && RecordWord(rec, w0) != 0 && !StreamBitsOk(ctx, (int32_t)RecordWord(rec, w0)))
      return "stream bit count is not a multiple of 4 in 4..184";
    if (check == lyra_b200_ctx::kCheckStreamDtx && RecordWord(rec, w0) > 1u) return "stream DTX word is not 0 or 1";
    if (check == lyra_b200_ctx::kCheckStats &&
        (RecordWord(rec, w0 + 2 * kStatLevel) > (uint32_t)kStatsLevels || RecordWord(rec, w0 + 2 * kStatLevel + 1) != 0 ||
         RecordWord(rec, w0 + 2 * kStatPrevReceived) > 1u || RecordWord(rec, w0 + 2 * kStatPrevReceived + 1) != 0))
      return "call statistics: level above 127 or event state not 0 or 1";
  }
  return nullptr;
}

// ids for lyra_b200_copy_streams: n in [1, max_streams]; src in [-1, max_streams), dst in [0, max_streams); no repeats within
// src (-1 excepted) or dst, no id in both
int CheckCopyIds(lyra_b200_ctx* ctx, const int32_t* src, const int32_t* dst, int n) {
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  const uint32_t g[2] = {NextIdGen(ctx), NextIdGen(ctx)};
  for (int k = 0; k < n; ++k) {
    const int id = src[k];
    if (id < -1 || id >= ctx->max_streams) { ctx->err = "source stream id out of range"; return LYRA_B200_EINVAL; }
    if (id < 0) continue;
    if (ctx->id_seen[(size_t)id] == g[0]) { ctx->err = "repeated source stream id"; return LYRA_B200_EINVAL; }
    ctx->id_seen[(size_t)id] = g[0];
  }
  for (int k = 0; k < n; ++k) {
    const int id = dst[k];
    if (id < 0 || id >= ctx->max_streams) { ctx->err = "destination stream id out of range"; return LYRA_B200_EINVAL; }
    if (ctx->id_seen[(size_t)id] == g[1]) { ctx->err = "repeated destination stream id"; return LYRA_B200_EINVAL; }
    if (ctx->id_seen[(size_t)id] == g[0]) { ctx->err = "a stream id is both a source and a destination"; return LYRA_B200_EINVAL; }
    ctx->id_seen[(size_t)id] = g[1];
  }
  return LYRA_B200_OK;
}

// ids for lyra_b200_align_streams: n in [1, max_streams]; ids in [0, max_streams) and distinct, like in [-1, max_streams) (repeats
// allowed), no id in both
int CheckAlignIds(lyra_b200_ctx* ctx, const int32_t* ids, const int32_t* like, int n) {
  if (int rc = CheckIds(ctx, ids, n, false)) return rc;     // marks ids with ctx->id_gen
  for (int k = 0; k < n; ++k) {
    const int id = like[k];
    if (id < -1 || id >= ctx->max_streams) { ctx->err = "like stream id out of range"; return LYRA_B200_EINVAL; }
    if (id >= 0 && ctx->id_seen[(size_t)id] == ctx->id_gen) { ctx->err = "a stream id is both aligned and a like stream"; return LYRA_B200_EINVAL; }
  }
  return LYRA_B200_OK;
}

// grid of a record kernel over `rows` rows of a call: 8 rows per block, one block row per entry of T (+ `extra`)
dim3 StateGrid(const StreamStateTable& T, int rows, int extra) {
  return dim3((unsigned)((rows + kStateRows - 1) / kStateRows), (unsigned)(T.count + extra));
}

// StreamStateCopyKernel over the entries of T on ctx->stream, one launch per kStateChunk rows: stream dst[k] (nullptr: k) <-
// stream src[k] (nullptr: -1, the state at creation).  The ids travel as kernel parameters: nothing to stage, nothing to wait for.
int CopyStreamState(lyra_b200_ctx* ctx, const StreamStateTable& T, const int32_t* src, const int32_t* dst, int n) {
  StreamIdChunk ids;
  for (int k0 = 0; k0 < n; k0 += kStateChunk) {
    ids.n = n - k0 < kStateChunk ? n - k0 : kStateChunk;
    for (int k = 0; k < ids.n; ++k) {
      ids.src[k] = src ? src[k0 + k] : -1;
      ids.dst[k] = dst ? dst[k0 + k] : k0 + k;
    }
    if (int rc = LAUNCH(kNoProf, StreamStateCopyKernel, StateGrid(T, ids.n, 0), dim3(kStateThreads), (size_t)0, ctx->stream, T, ids))
      return rc;
  }
  return LYRA_B200_OK;
}

// StreamWordKernel on ctx->stream, one launch per kStateChunk streams: word[ids[k]] (ids nullptr: k) <- values[k] (nullptr:
// ctx_value), stored as 0 when it equals ctx_value; conv0 / conv1 as in StreamWordKernel.  Ids and values travel as kernel
// parameters.  The sample rates: (ctx->sample_rate, d_stream_rate, the codec converters); the bit counts and the DTX words:
// (0, d_stream_word[w], none).
int LaunchStreamWords(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int32_t* values, int ctx_value, int* word, int* conv0,
                      int* conv1) {
  StreamWordChunk c;
  for (int k0 = 0; k0 < n; k0 += kStateChunk) {
    c.n = n - k0 < kStateChunk ? n - k0 : kStateChunk;
    for (int k = 0; k < c.n; ++k) {
      c.ids[k] = ids ? ids[k0 + k] : k0 + k;
      c.values[k] = values ? values[k0 + k] : ctx_value;
    }
    if (int rc = LAUNCH(kNoProf, StreamWordKernel, dim3((unsigned)((c.n + kStreamWordThreads - 1) / kStreamWordThreads)),
                        dim3(kStreamWordThreads), (size_t)0, ctx->stream, c, ctx_value, word, conv0, conv1))
      return rc;
  }
  return LYRA_B200_OK;
}
int LaunchStreamRates(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int32_t* rates) {
  return LaunchStreamWords(ctx, ids, n, rates, ctx->sample_rate, ctx->d_stream_rate, ctx->d_codec_rs_pos[0], ctx->d_codec_rs_pos[1]);
}

// The device words `word` of the listed streams (ids nullptr: 0 .. n-1; repeats allowed) into out[k], once the work queued on
// the context's stream has finished.  The getters of the per-stream words.
int ReadStreamWords(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int* word, int32_t* out) {
  if (int rc = CheckIds(ctx, ids, n, true)) return rc;
  CU(SyncStream(ctx));
  std::vector<int> words((size_t)ctx->max_streams);
  CU(cudaMemcpy(words.data(), word, sizeof(int) * words.size(), cudaMemcpyDeviceToHost));
  for (int k = 0; k < n; ++k) out[k] = words[(size_t)(ids ? ids[k] : k)];
  return LYRA_B200_OK;
}

// role index of a role that must be exactly one role of the context (0 encoder, 1 decoder), or -1 with ctx->err set
int BitsRole(lyra_b200_ctx* ctx, int role) {
  if (role != LYRA_B200_ROLE_ENCODER && role != LYRA_B200_ROLE_DECODER) { ctx->err = "role must be LYRA_B200_ROLE_ENCODER or _DECODER"; return -1; }
  return RoleOk(ctx, role) ? role - 1 : -1;
}

// ---- the plugin-level calls (extract_features, quantize, dequantize, generate, logmel, noise_estimate, cng_generate, resample) ----
// Each call is a Check*, which validates the call (role, arguments, stream ids) and queues nothing when it fails, and a Launch*,
// which queues the call's kernels on device pointers.  A host-buffer call copies its inputs into the context's staging between the
// two and copies its results out and synchronises after them; its *_device twin launches on the caller's buffers (rows 0..n-1)
// and returns.  The calls run every stream at 16 kHz and read no per-stream word, nor the active mask.

// the ids of a call (n in range; nullptr: streams 0..n-1) and, for a sparse host-buffer call, their device copy in *d_ids
int StageIds(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int** d_ids) {
  const int rc = CheckIds(ctx, ids, n, false);
  return rc ? rc : UploadIds(ctx, ids, n, d_ids);
}

// extract_features (encoder role) / generate (decoder role): the role and the call's tile map
int CheckNets(lyra_b200_ctx* ctx, int role, const int32_t* ids, int n) {
  ENTER(role);
  return PrepareMap(ctx, ids, n);
}

// quantize / dequantize: any context, a bit count the codec calls accept, streams 0..n-1
int CheckRvq(lyra_b200_ctx* ctx, int n, int num_bits) {
  ENTER(0);
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  return CheckIds(ctx, nullptr, n, false);
}
int LaunchQuantizeCall(lyra_b200_ctx* ctx, int n, const float* d_features, int num_bits, uint8_t* d_packets, int* d_indices) {
  return LaunchQuantize(ctx, ctx->stream, Rows(WholeCall(ctx, n), nullptr, nullptr), StreamWords{}, d_features, num_bits, d_packets,
                        d_indices, nullptr);
}
int LaunchDequantizeCall(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, int num_bits, float* d_features) {
  return LaunchDequantize(ctx, ctx->stream, Rows(WholeCall(ctx, n), nullptr, nullptr), StreamWords{}, d_packets, nullptr, num_bits,
                          d_features, nullptr);
}

// logmel: any context, bank 0 or 1, 160 or 64 bins
int CheckLogMel(lyra_b200_ctx* ctx, int bank, const int32_t* ids, int n, int num_mel_bins, const int** d_ids) {
  ENTER(0);
  if (bank < 0 || bank > 1) { ctx->err = "log-mel bank must be 0 or 1"; return LYRA_B200_EINVAL; }
  if (num_mel_bins != 160 && num_mel_bins != 64) { ctx->err = "log-mel supports 160 or 64 mel bins"; return LYRA_B200_EINVAL; }
  return StageIds(ctx, ids, n, d_ids);
}
int LaunchLogMelCall(lyra_b200_ctx* ctx, int bank, const int* d_ids, int n, const int16_t* d_pcm, int num_mel_bins, float* d_out) {
  const LogMelParams& P = num_mel_bins == 160 ? ctx->spec.logmel160 : ctx->spec.logmel64;
  return LaunchLogMel(ctx, ctx->stream, Rows(WholeCall(ctx, n), d_ids, nullptr), Uniform(P), kWords16k, d_pcm, ctx->d_logmel_prev[bank],
                      nullptr, d_out);
}

// noise_estimate / cng_generate: any context
int CheckRows(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int** d_ids) {
  ENTER(0);
  return StageIds(ctx, ids, n, d_ids);
}
int LaunchNoiseRead(lyra_b200_ctx* ctx, const int* d_ids, int n, float* d_estimate, uint8_t* d_is_noise) {
  return LAUNCH(kNoProf, NoiseReadKernel, dim3((unsigned)n), dim3(192), (size_t)0, ctx->stream,
                Rows(WholeCall(ctx, n), d_ids, nullptr), ctx->d_noise, ctx->noise_params.nf, d_estimate, d_is_noise);
}

// resample: any context, a supported rate, at most 960 samples in and out per row and room for all outputs; *pr = the filter pair
int CheckResample(lyra_b200_ctx* ctx, int to_internal, const int32_t* ids, int n, int external_rate_hz, int in_samples, int out_stride,
                  int* pr, const int** d_ids) {
  ENTER(0);
  const int pair = RatePair(external_rate_hz);
  if (pair < 0) { ctx->err = "the resampler converts between 16 kHz and 8 / 32 / 48 kHz"; return LYRA_B200_EINVAL; }
  *pr = to_internal ? pair : pair + 3;
  const int num = ctx->spec.resampler.num[*pr], den = ctx->spec.resampler.den[*pr];
  const int max_out = (in_samples * den + num - 1) / num;
  if (in_samples <= 0 || in_samples > 960 || max_out > 960 || out_stride < max_out || out_stride > 968) {
    ctx->err = "resample: at most 960 input and 960 output samples per stream and call, and room for ceil(n * out / in) outputs";
    return LYRA_B200_EINVAL;
  }
  return StageIds(ctx, ids, n, d_ids);
}
// rows of in_samples inputs -> rows of out_stride outputs, of which the first counts[slot] (counts may be nullptr) are written
int LaunchResampleCall(lyra_b200_ctx* ctx, int pr, int to_internal, int external_rate_hz, const int* d_ids, int n, const int16_t* d_in,
                       int in_samples, int16_t* d_out, int out_stride, int* d_counts) {
  const int dir = to_internal ? 0 : 1;
  return LAUNCH(kNoProf, ResampleKernel, dim3((unsigned)n), dim3(128), sizeof(float) * (size_t)(kResamplerTaps - 1 + in_samples),
                ctx->stream, ctx->d_blob, ctx->spec.resampler, pr, external_rate_hz, Rows(WholeCall(ctx, n), d_ids, nullptr),
                StreamWords{}, d_in, in_samples, in_samples, d_out, out_stride, d_counts, ctx->d_rs_delay[dir], ctx->d_rs_pos[dir]);
}

}  // namespace

extern "C" {

int lyra_b200_create(const char* model_dir, int device, int max_streams, lyra_b200_ctx** out) {
  return lyra_b200_create_ex(model_dir, device, max_streams, LYRA_B200_ROLE_ENCODER | LYRA_B200_ROLE_DECODER, out);
}

int lyra_b200_create_ex(const char* model_dir, int device, int max_streams, int roles, lyra_b200_ctx** out) {
  if (out) *out = nullptr;
  if (!out || !model_dir || max_streams <= 0 || (roles & ~3) || roles == 0) { g_create_error = "bad argument"; return LYRA_B200_EINVAL; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    g_create_error = "no CUDA device available (lyra_b200 has no CPU fallback)";
    return LYRA_B200_ENODEV;
  }
  if (device < 0 || device >= ndev) { g_create_error = "CUDA device index out of range"; return LYRA_B200_ENODEV; }
  lyra_b200_ctx* ctx = new lyra_b200_ctx();
  try {
    ctx->spec = BuildModelSpec(model_dir);
  } catch (const std::exception& e) {
    g_create_error = e.what();
    delete ctx;
    return LYRA_B200_EMODEL;
  }
  ctx->device = device;
  ctx->max_streams = max_streams;
  ctx->roles = roles;
  ctx->ntiles = (max_streams + kTileStreams - 1) / kTileStreams;
  ctx->padded = ctx->ntiles * kTileStreams;
  ctx->tile_gen.assign((size_t)ctx->ntiles, 0u);
  ctx->id_seen.assign((size_t)max_streams, 0u);
  const size_t P = (size_t)ctx->padded;
  bool ok = cudaSetDevice(device) == cudaSuccess;
  // Stream priority of the context's own and sub-batch streams: 0 unless LYRA_B200_ENC_PRIORITY / LYRA_B200_DEC_PRIORITY say
  // otherwise (encoder-only / decoder-only contexts); lyra_b200_set_priority changes it later.
  int prio = 0;
  if (const char* e = std::getenv(roles == LYRA_B200_ROLE_DECODER ? "LYRA_B200_DEC_PRIORITY" : "LYRA_B200_ENC_PRIORITY")) prio = std::atoi(e);
  ctx->priority = prio;
  ok = ok && cudaStreamCreateWithPriority(&ctx->own_stream, cudaStreamDefault, prio) == cudaSuccess;
  for (int i = 0; i < lyra_b200_ctx::kMaxSplit - 1; ++i) {
    ok = ok && cudaStreamCreateWithPriority(&ctx->aux_stream[i], cudaStreamDefault, prio) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->ev_join[i], cudaEventDisableTiming) == cudaSuccess;
  }
  ok = ok && cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming) == cudaSuccess;
  ok = ok && cudaEventCreateWithFlags(&ctx->ev_sync, cudaEventDisableTiming | cudaEventBlockingSync) == cudaSuccess;
  ctx->stream = ctx->own_stream;
  ok = ok && DevAlloc(ctx, &ctx->d_blob, ctx->spec.blob.size());
  ok = ok && cudaMemcpy(ctx->d_blob, ctx->spec.blob.data(), ctx->spec.blob.size(), cudaMemcpyHostToDevice) == cudaSuccess;
  // Device memory.  DevStreamState allocates per-stream state and lists it in ctx->state_list; DevAlloc is everything else.
  const int units[4] = {EncStateA::kUnits, EncStateB::kUnits, DecStateC::kUnits, DecStateD::kUnits};
  for (int w = 0; w < 4 && ok; ++w) {
    if (!(roles & (w < 2 ? LYRA_B200_ROLE_ENCODER : LYRA_B200_ROLE_DECODER))) continue;   // an encoder-only / decoder-only context
    ok = DevStreamState(ctx, &ctx->d_state[w], (size_t)units[w], InitImage(ctx->spec, w).data(), kStatePlain, lyra_b200_ctx::kCheckNone,
                        true, kTileStreams, &ctx->d_n18[w]);
    ctx->align_table.e[ctx->align_table.count++] = {ctx->d_state[w], ctx->d_n18[w], units[w], w};
  }
  if (roles & LYRA_B200_ROLE_ENCODER) ok = ok && DevAlloc(ctx, &ctx->d_mid_enc, P * 128 * 4);
  if (roles & LYRA_B200_ROLE_DECODER) ok = ok && DevAlloc(ctx, &ctx->d_mid_dec, P * 128 * 4);
  for (int b = 0; b < 3; ++b) ok = ok && DevStreamState(ctx, &ctx->d_logmel_prev[b], LYRA_B200_HOP);
  ctx->noise_params = MakeNoiseParams(16000);
  for (int r : {16000, 8000, 32000, 48000}) {
    ctx->enc_noise_params.p[RateIndex(r)] = MakeNoiseParams(r);
    ctx->enc_logmel.p[RateIndex(r)] = r == 16000 ? ctx->spec.logmel160 : ctx->spec.logmel160_ext[RatePair(r)];
  }
  // noise estimators: all-zero is the freshly constructed object
  ok = ok && DevStreamState(ctx, &ctx->d_noise, NoiseStateUnits(160));
  ok = ok && DevAlloc(ctx, &ctx->d_noise_est, P * 160);
  ok = ok && DevStreamState(ctx, &ctx->d_noise_enc, NoiseStateUnits(160));
  ok = ok && DevStreamState(ctx, &ctx->d_logmel_prev_enc, LYRA_B200_HOP);
  // decoder control state: (0, 0, fade from comfort noise), lyra_decoder.cc:164-166
  const int plc0[4] = {0, 0, -1, 0};
  ok = ok && DevStreamState(ctx, &ctx->d_plc, 4, plc0, kStatePlain, lyra_b200_ctx::kCheckPlc);
  ok = ok && DevStreamState(ctx, &ctx->d_cng_work, 1024);
  ok = ok && DevStreamState(ctx, &ctx->d_cng_hops, 2, nullptr, kStateCng);
  ok = ok && DevAlloc(ctx, &ctx->d_plan, P);
  ok = ok && DevAlloc(ctx, &ctx->d_skip, P);
  ok = ok && DevAlloc(ctx, &ctx->d_feed, P);
  ok = ok && DevAlloc(ctx, &ctx->d_is_cn, P);
  ok = ok && DevAlloc(ctx, &ctx->d_fade0, P);
  ok = ok && DevAlloc(ctx, &ctx->d_dir, P);
  ok = ok && DevAlloc(ctx, &ctx->d_model_pcm, P * LYRA_B200_HOP);
  ok = ok && DevAlloc(ctx, &ctx->d_cng_pcm, P * LYRA_B200_HOP);
  ok = ok && DevAlloc(ctx, &ctx->d_cng_feat, P * 160);
  for (int d = 0; d < 2; ++d) {
    // reset leaves the delay line alone: rate 0 in d_rs_pos makes the next call restart the stream fully primed (a stream
    // moved mid-phase needs it, so the records carry it)
    ok = ok && DevStreamState(ctx, &ctx->d_rs_delay[d], (size_t)(kResamplerTaps - 1), nullptr, kStatePlain, lyra_b200_ctx::kCheckNone, false);
    ok = ok && DevStreamState(ctx, &ctx->d_rs_pos[d], 2, nullptr, kStatePlain, lyra_b200_ctx::kCheckResamplerPos);
  }
  for (int d = 0; d < 2; ++d) {
    // the codec path's converters (lyra_b200_set_sample_rate): reset zeroes them, and tag 0 makes the next call restart primed
    if (!(roles & (d == 0 ? LYRA_B200_ROLE_ENCODER : LYRA_B200_ROLE_DECODER))) continue;
    ok = ok && DevStreamState(ctx, &ctx->d_codec_rs_delay[d], (size_t)(kResamplerTaps - 1));
    ok = ok && DevStreamState(ctx, &ctx->d_codec_rs_pos[d], 2, nullptr, d == 0 ? kStateCodecRs0 : kStateCodecRs1,
                              lyra_b200_ctx::kCheckResamplerPos);
  }
  // the call statistics per role (lyra_b200_set_stats): LEVEL 127 and "last run hop received" at creation and after reset
  // (registered after the network entries and before the per-stream words, which stay the last words of a record)
  unsigned long long stats0[kStatsWords] = {};
  stats0[kStatLevel] = kStatsLevels;
  stats0[kStatPrevReceived] = 1;
  for (int r = 0; r < 2; ++r)
    if (roles & (r == 0 ? LYRA_B200_ROLE_ENCODER : LYRA_B200_ROLE_DECODER))
      ok = ok && DevStreamState(ctx, &ctx->d_stats[r], (size_t)kStatsWords, stats0, kStatePlain, lyra_b200_ctx::kCheckStats);
  double levels[kStatsLevels + 1] = {};
  for (int k = 0; k < kStatsLevels; ++k) levels[k] = 1073741824.0 * std::pow(10.0, -(k + 0.5) / 10.0);
  ok = ok && DevAlloc(ctx, &ctx->d_stats_levels, (size_t)kStatsLevels + 1) &&
       cudaMemcpy(ctx->d_stats_levels, levels, sizeof(levels), cudaMemcpyHostToDevice) == cudaSuccess;
  ok = ok && DevAlloc(ctx, &ctx->d_stats_out, P * kStatsWords);
  // the stream's DTX word (lyra_b200_set_stream_dtx, encoder role): 0, DTX on, at creation and after reset; then its own bit
  // count per role (lyra_b200_set_stream_bits): 0, the call's, at creation and after reset
  // (registered before the rate word, which stays the last word of a record)
  for (int w : {kWordDtxOff, kWordEncBits, kWordDecBits}) {
    const int role = w == kWordDecBits ? LYRA_B200_ROLE_DECODER : LYRA_B200_ROLE_ENCODER;
    if (!(roles & role)) continue;
    const int check = w == kWordDtxOff ? lyra_b200_ctx::kCheckStreamDtx : lyra_b200_ctx::kCheckStreamBits;
    ok = ok && DevStreamState(ctx, &ctx->d_stream_word[w], 1, nullptr, kStatePlain, check);
    ctx->word_mirror[w].assign((size_t)max_streams, 0);
  }
  // the stream's own sample rate (lyra_b200_set_stream_sample_rates): 0, the context's, at creation and after reset
  ok = ok && DevStreamState(ctx, &ctx->d_stream_rate, 1, nullptr, kStatePlain, lyra_b200_ctx::kCheckStreamRate);
  ok = ok && DevAlloc(ctx, &ctx->d_rs_in, P * 960);
  ok = ok && DevAlloc(ctx, &ctx->d_rs_out, P * 968);
  ok = ok && DevAlloc(ctx, &ctx->d_rs_counts, P);
  ok = ok && DevAlloc(ctx, &ctx->d_is_noise, P);
  ok = ok && DevAlloc(ctx, &ctx->d_pcm, P * LYRA_B200_HOP);
  ok = ok && DevAlloc(ctx, &ctx->d_packets, P * 24);
  ok = ok && DevAlloc(ctx, &ctx->d_received, P);
  ok = ok && DevAlloc(ctx, &ctx->d_features, P * LYRA_B200_NUM_FEATURES);
  ok = ok && DevAlloc(ctx, &ctx->d_melout, P * 160);
  ok = ok && DevAlloc(ctx, &ctx->d_indices, P * LYRA_B200_MAX_STAGES);
  ok = ok && DevAlloc(ctx, &ctx->d_ids, P);
  ok = ok && DevAlloc(ctx, &ctx->d_tile_list, (size_t)ctx->ntiles);
  ok = ok && DevAlloc(ctx, &ctx->d_slot_of, P);
  for (int b = 0; b < 2 && ok; ++b) {
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&ctx->h_slot_of[b]), sizeof(int) * P) == cudaSuccess;
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&ctx->h_tile_list[b]), sizeof(int) * (size_t)ctx->ntiles) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->ev_map[b], cudaEventDisableTiming) == cudaSuccess;
    if (ok) for (size_t i = 0; i < P; ++i) ctx->h_slot_of[b][i] = -1;
  }
  if (ok) ok = SetSmemLimits();
  ctx->model_fingerprint = ModelFingerprint(ctx->spec.blob);
  ok = ok && BuildStateTable(ctx);
  if (!ok) {
    g_create_error = std::string("CUDA allocation / setup failed: ") + cudaGetErrorString(cudaGetLastError());
    lyra_b200_destroy(ctx);
    return LYRA_B200_ENODEV;
  }
  if (lyra_b200_reset(ctx, nullptr, max_streams) != LYRA_B200_OK) {
    g_create_error = ctx->err;
    lyra_b200_destroy(ctx);
    return LYRA_B200_ENODEV;
  }
  *out = ctx;
  return LYRA_B200_OK;
}

void lyra_b200_destroy(lyra_b200_ctx* ctx) {
  if (!ctx) return;
  UseDevice(ctx);
  for (void* p : ctx->allocs) cudaFree(p);
  for (int b = 0; b < 2; ++b) {
    if (ctx->h_slot_of[b]) cudaFreeHost(ctx->h_slot_of[b]);
    if (ctx->h_tile_list[b]) cudaFreeHost(ctx->h_tile_list[b]);
    if (ctx->ev_map[b]) cudaEventDestroy(ctx->ev_map[b]);
  }
  for (int k = 0; k < LYRA_B200_NUM_KERNELS; ++k)
    for (auto& ev : ctx->prof_events[k]) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
#ifndef LYRA_EMU
  DropGraphs(ctx);
#endif
  if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
  if (ctx->ev_sync) cudaEventDestroy(ctx->ev_sync);
  for (int i = 0; i < lyra_b200_ctx::kMaxSplit - 1; ++i) {
    if (ctx->ev_join[i]) cudaEventDestroy(ctx->ev_join[i]);
    if (ctx->aux_stream[i]) cudaStreamDestroy(ctx->aux_stream[i]);
  }
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

const char* lyra_b200_last_error(const lyra_b200_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }
int lyra_b200_max_streams(const lyra_b200_ctx* ctx) { return ctx ? ctx->max_streams : 0; }
int lyra_b200_tile_streams(const lyra_b200_ctx* ctx) { return ctx ? kTileStreams : 0; }
uint64_t lyra_b200_launch_count(const lyra_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int lyra_b200_profile_enable(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
  CU(SyncStream(ctx));
  ProfDrain(ctx);
  ctx->profiling = enable != 0;
  if (enable) for (int k = 0; k < LYRA_B200_NUM_KERNELS; ++k) { ctx->prof_ms[k] = 0.0; ctx->prof_n[k] = 0; }
  return LYRA_B200_OK;
}

int lyra_b200_profile_read(lyra_b200_ctx* ctx, double* ms_sum, uint64_t* launches) {
  if (!ctx || !ms_sum || !launches) return LYRA_B200_EINVAL;
  ENTER(0);
  CU(SyncStream(ctx));
  ProfDrain(ctx);
  for (int k = 0; k < LYRA_B200_NUM_KERNELS; ++k) { ms_sum[k] = ctx->prof_ms[k]; launches[k] = ctx->prof_n[k]; }
  return LYRA_B200_OK;
}

// the entries of ctx->reset_table go back to their state at creation, in order on ctx->stream.  Repeated ids are collapsed
// (first appearance kept): the copy kernel's destinations must be distinct.
int lyra_b200_reset(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
  int rc = CheckIds(ctx, stream_ids, n, true);
  if (rc) return rc;
  std::vector<int32_t> distinct;
  if (stream_ids) {
    const uint32_t gen = NextIdGen(ctx);
    for (int k = 0; k < n; ++k)
      if (ctx->id_seen[(size_t)stream_ids[k]] != gen) { ctx->id_seen[(size_t)stream_ids[k]] = gen; distinct.push_back(stream_ids[k]); }
    stream_ids = distinct.data();
    n = (int)distinct.size();
  }
  if ((rc = CopyStreamState(ctx, ctx->reset_table, nullptr, stream_ids, n))) return rc;
  for (int w = 0; w < kMirroredWords; ++w)
    for (int k = 0; k < n && ctx->own_words[w]; ++k) SetMirrorWord(ctx, w, stream_ids ? stream_ids[k] : k, 0);
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_set_stream(lyra_b200_ctx* ctx, void* cuda_stream) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
  ctx->stream = cuda_stream ? reinterpret_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
  return LYRA_B200_OK;
}

int lyra_b200_set_split(lyra_b200_ctx* ctx, int parts) {
  if (!ctx || parts < 1 || parts > lyra_b200_ctx::kMaxSplit) return LYRA_B200_EINVAL;
  ENTER(0);
  ctx->nsplit = parts;
  return LYRA_B200_OK;
}

int lyra_b200_set_blocking_sync(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
  ctx->blocking_sync = enable != 0;
  return LYRA_B200_OK;
}

int lyra_b200_set_priority(lyra_b200_ctx* ctx, int priority) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
  CU(SyncStream(ctx));
#ifndef LYRA_EMU
  DropGraphs(ctx);                   // captured graphs carry the priority of the streams they were captured on
#endif
  const bool own = ctx->stream == ctx->own_stream;
  cudaStream_t fresh[lyra_b200_ctx::kMaxSplit];
  for (int i = 0; i < lyra_b200_ctx::kMaxSplit; ++i)
    if (cudaStreamCreateWithPriority(&fresh[i], cudaStreamDefault, priority) != cudaSuccess) {      // nothing has changed yet
      while (i-- > 0) cudaStreamDestroy(fresh[i]);
      ctx->err = "cudaStreamCreateWithPriority failed";
      return LYRA_B200_ENODEV;
    }
  cudaStreamDestroy(ctx->own_stream);
  ctx->own_stream = fresh[0];
  for (int i = 0; i < lyra_b200_ctx::kMaxSplit - 1; ++i) { cudaStreamDestroy(ctx->aux_stream[i]); ctx->aux_stream[i] = fresh[i + 1]; }
  if (own) ctx->stream = ctx->own_stream;
  ctx->priority = priority;
  return LYRA_B200_OK;
}

int lyra_b200_set_decoder_mode(lyra_b200_ctx* ctx, int mode) {
  if (!ctx || (mode != LYRA_B200_DECODER_EXACT && mode != LYRA_B200_DECODER_TENSOR)) return LYRA_B200_EINVAL;
  ENTER(0);
  ctx->decoder_mode = mode;
  return LYRA_B200_OK;
}

int lyra_b200_decoder_mode(const lyra_b200_ctx* ctx) { return ctx ? ctx->decoder_mode : LYRA_B200_EINVAL; }

int lyra_b200_set_sample_rate(lyra_b200_ctx* ctx, int sample_rate_hz) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (!RateOk(sample_rate_hz)) { ctx->err = "the codec calls run at 8000, 16000, 32000 or 48000 Hz"; return LYRA_B200_EINVAL; }
  ENTER(0);
  if (sample_rate_hz == ctx->sample_rate && !ctx->rate_override) return LYRA_B200_OK;
  CU(SyncStream(ctx));
  if (sample_rate_hz == ctx->sample_rate) {
    // the same rate: the streams with a rate of their own come back to it (their converters restart), the others are untouched
    int rc = LaunchStreamRates(ctx, nullptr, ctx->max_streams, nullptr);
    if (rc) return rc;
    CU(SyncStream(ctx));
    ctx->rate_override = false;
    return LYRA_B200_OK;
  }
#ifndef LYRA_EMU
  DropGraphs(ctx);                   // captured graphs carry the converters' rate, tag and row sizes
#endif
  if (ctx->rate_override) {
    CU(cudaMemsetAsync(ctx->d_stream_rate, 0, sizeof(int) * (size_t)ctx->padded, ctx->stream));   // every stream at the new rate
    CU(SyncStream(ctx));
    ctx->rate_override = false;
  }
  ctx->sample_rate = sample_rate_hz;
  ctx->codec_rs_tag = ctx->codec_rs_tag % 1000000000 + 1;    // every stream's converters restart primed on their next call
  return LYRA_B200_OK;
}

int lyra_b200_set_stream_sample_rates(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int32_t* rates_hz) {
  if (!ctx || !rates_hz) return LYRA_B200_EINVAL;
  ENTER(0);
  int rc = CheckIds(ctx, stream_ids, n, false);
  if (rc) return rc;
  bool differs = false;
  for (int k = 0; k < n; ++k) {
    if (!StreamRateOk(ctx, rates_hz[k])) {
      ctx->err = "a stream runs at 8000, 16000, 32000 or 48000 Hz, at most the context's rate (lyra_b200_set_sample_rate)";
      return LYRA_B200_EINVAL;
    }
    differs |= rates_hz[k] != ctx->sample_rate;
  }
  if (!differs && !ctx->rate_override) return LYRA_B200_OK;     // every stream is at the context's rate already
  if ((rc = LaunchStreamRates(ctx, stream_ids, n, rates_hz))) return rc;
  ctx->rate_override = true;
  return LYRA_B200_OK;
}

int lyra_b200_stream_sample_rates(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, int32_t* rates_hz) {
  if (!ctx || !rates_hz) return LYRA_B200_EINVAL;
  ENTER(0);
  if (int rc = ReadStreamWords(ctx, stream_ids, n, ctx->d_stream_rate, rates_hz)) return rc;
  for (int k = 0; k < n; ++k) rates_hz[k] = rates_hz[k] ? rates_hz[k] : ctx->sample_rate;
  return LYRA_B200_OK;
}

int lyra_b200_sample_rate(const lyra_b200_ctx* ctx) { return ctx ? ctx->sample_rate : LYRA_B200_EINVAL; }

int lyra_b200_set_stream_bits(lyra_b200_ctx* ctx, int role, const int32_t* stream_ids, int n, const int32_t* bits) {
  if (!ctx || !bits) return LYRA_B200_EINVAL;
  ENTER(0);
  const int r = BitsRole(ctx, role);
  if (r < 0) return LYRA_B200_EINVAL;
  int rc = CheckIds(ctx, stream_ids, n, false);
  if (rc) return rc;
  bool changes = false;
  for (int k = 0; k < n; ++k) {
    if (bits[k] != 0 && !StreamBitsOk(ctx, bits[k])) {
      ctx->err = "a stream's own bit count is 0 (the call's) or a multiple of 4 in 4..184";
      return LYRA_B200_EINVAL;
    }
    changes |= ctx->word_mirror[r][(size_t)(stream_ids ? stream_ids[k] : k)] != bits[k];
  }
  if (!changes) return LYRA_B200_OK;
  if ((rc = LaunchStreamWords(ctx, stream_ids, n, bits, 0, ctx->d_stream_word[r], nullptr, nullptr))) return rc;
  for (int k = 0; k < n; ++k) SetMirrorWord(ctx, r, stream_ids ? stream_ids[k] : k, bits[k]);
  return LYRA_B200_OK;
}

int lyra_b200_stream_bits(lyra_b200_ctx* ctx, int role, const int32_t* stream_ids, int n, int32_t* bits) {
  if (!ctx || !bits) return LYRA_B200_EINVAL;
  ENTER(0);
  const int r = BitsRole(ctx, role);
  if (r < 0) return LYRA_B200_EINVAL;
  return ReadStreamWords(ctx, stream_ids, n, ctx->d_stream_word[r], bits);
}

int lyra_b200_set_stream_dtx(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const int32_t* enable) {
  if (!ctx || !enable) return LYRA_B200_EINVAL;
  ENTER(LYRA_B200_ROLE_ENCODER);
  int rc = CheckIds(ctx, stream_ids, n, false);
  if (rc) return rc;
  std::vector<int32_t> off((size_t)n), turned_on;
  bool changes = false;
  for (int k = 0; k < n; ++k) {
    if (enable[k] != 0 && enable[k] != 1) { ctx->err = "a stream's DTX setting is 0 (off) or 1 (on)"; return LYRA_B200_EINVAL; }
    const int id = stream_ids ? stream_ids[k] : k, was = ctx->word_mirror[kWordDtxOff][(size_t)id];
    off[(size_t)k] = 1 - enable[k];
    changes |= was != off[(size_t)k];
    if (was && enable[k]) turned_on.push_back(id);
  }
  if (!changes) return LYRA_B200_OK;
  // 0 -> 1: the encoder-side estimator and its extractor restart at their creation state (a fresh NoiseEstimator::Create)
  if (!turned_on.empty() && (rc = CopyStreamState(ctx, ctx->dtx_table, nullptr, turned_on.data(), (int)turned_on.size()))) return rc;
  if ((rc = LaunchStreamWords(ctx, stream_ids, n, off.data(), 0, ctx->d_stream_word[kWordDtxOff], nullptr, nullptr))) return rc;
  for (int k = 0; k < n; ++k) SetMirrorWord(ctx, kWordDtxOff, stream_ids ? stream_ids[k] : k, off[(size_t)k]);
  return LYRA_B200_OK;
}

int lyra_b200_stream_dtx(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, int32_t* enable) {
  if (!ctx || !enable) return LYRA_B200_EINVAL;
  ENTER(LYRA_B200_ROLE_ENCODER);
  if (int rc = ReadStreamWords(ctx, stream_ids, n, ctx->d_stream_word[kWordDtxOff], enable)) return rc;
  for (int k = 0; k < n; ++k) enable[k] = 1 - enable[k];
  return LYRA_B200_OK;
}

int lyra_b200_set_active_mask(lyra_b200_ctx* ctx, const uint8_t* d_active) {
  if (!ctx) return LYRA_B200_EINVAL;
  ctx->d_active = d_active;          // read by the kernels of later *_device codec calls, in stream order
  return LYRA_B200_OK;
}

int lyra_b200_set_stats(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  ctx->stats_on = enable != 0;       // read by the host when later codec calls are issued
  return LYRA_B200_OK;
}

int lyra_b200_read_stats(lyra_b200_ctx* ctx, int role, const int32_t* stream_ids, int n, uint64_t* stats, int clear) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (!stats) { ctx->err = "stats is required"; return LYRA_B200_EINVAL; }
  ENTER(0);
  const int r = BitsRole(ctx, role);
  if (r < 0) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int rc = CheckIds(ctx, stream_ids, n, true);
  if (rc || (rc = UploadIds(ctx, stream_ids, n, &d_ids))) return rc;
  const dim3 grid((unsigned)((n * kStatsWords + 255) / 256));
  // repeated ids: every read before any clear
  if ((rc = LAUNCH(kNoProf, StatsReadKernel, grid, dim3(256), (size_t)0, ctx->stream, ctx->d_stats[r], d_ids, n, ctx->d_stats_out,
                   clear && !d_ids ? 1 : 0)))
    return rc;
  if (clear && d_ids &&
      (rc = LAUNCH(kNoProf, StatsReadKernel, grid, dim3(256), (size_t)0, ctx->stream, ctx->d_stats[r], d_ids, n, nullptr, 1)))
    return rc;
  CU(cudaMemcpyAsync(stats, ctx->d_stats_out, sizeof(uint64_t) * kStatsWords * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_read_stats_device(lyra_b200_ctx* ctx, int role, int n, uint64_t* d_stats, int clear) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (!d_stats) { ctx->err = "d_stats is required"; return LYRA_B200_EINVAL; }
  ENTER(0);
  const int r = BitsRole(ctx, role);
  if (r < 0) return LYRA_B200_EINVAL;
  if (int rc = CheckIds(ctx, nullptr, n, false)) return rc;
  return LAUNCH(kNoProf, StatsReadKernel, dim3((unsigned)((n * kStatsWords + 255) / 256)), dim3(256), (size_t)0, ctx->stream,
                ctx->d_stats[r], nullptr, n, reinterpret_cast<unsigned long long*>(d_stats), clear ? 1 : 0);
}

int lyra_b200_synchronize(lyra_b200_ctx* ctx) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_encode_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets) {
  if (!ctx || !d_pcm || !d_packets) return LYRA_B200_EINVAL;
  CodecCall c{kEncode, n, num_bits};
  c.dev.pcm_in = d_pcm;
  c.dev.packets_out = d_packets;
  return RunCodecCall(ctx, c);
}

int lyra_b200_decode_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                            int16_t* d_pcm) {
  if (!ctx || !d_packets || !d_pcm) return LYRA_B200_EINVAL;
  CodecCall c{kDecode, n, num_bits};
  c.dev.packets_in = d_packets;
  c.dev.received = d_received;
  c.dev.pcm_out = d_pcm;
  return RunCodecCall(ctx, c);
}

int lyra_b200_set_graphs(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  ENTER(0);
#ifndef LYRA_EMU
  CU(SyncStream(ctx));
  if (!enable) DropGraphs(ctx);
#endif
  ctx->use_graphs = enable != 0;
  return LYRA_B200_OK;
}
uint64_t lyra_b200_graph_replays(const lyra_b200_ctx* ctx) { return ctx ? ctx->graph_replays : 0; }

int lyra_b200_encode(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, int num_bits, uint8_t* packets) {
  if (!ctx || !pcm || !packets) return LYRA_B200_EINVAL;
  CodecCall c{kEncode, n, num_bits, ids};
  c.host.pcm_in = pcm;
  c.host.packets_out = packets;
  return RunCodecCall(ctx, c);
}

int lyra_b200_decode(lyra_b200_ctx* ctx, const int32_t* ids, int n, const uint8_t* packets, const uint8_t* received,
                     int num_bits, int16_t* pcm) {
  if (!ctx || !packets || !pcm) return LYRA_B200_EINVAL;
  CodecCall c{kDecode, n, num_bits, ids};
  c.host.packets_in = packets;
  c.host.received = received;
  c.host.pcm_out = pcm;
  return RunCodecCall(ctx, c);
}

int lyra_b200_extract_features(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, float* features) {
  if (!ctx || !pcm || !features) return LYRA_B200_EINVAL;
  int rc = CheckNets(ctx, LYRA_B200_ROLE_ENCODER, ids, n);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_pcm, pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchEncoderNets(ctx, WholeCall(ctx, n), nullptr, ctx->d_pcm, ctx->d_features, nullptr))) return rc;
  CU(cudaMemcpyAsync(features, ctx->d_features, sizeof(float) * 64 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_extract_features_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, float* d_features) {
  if (!ctx || !d_pcm || !d_features) return LYRA_B200_EINVAL;
  const int rc = CheckNets(ctx, LYRA_B200_ROLE_ENCODER, nullptr, n);
  return rc ? rc : ForEachPart(ctx, n, [&](const Part& p) { return LaunchEncoderNets(ctx, p, nullptr, d_pcm, d_features, nullptr); });
}

int lyra_b200_quantize(lyra_b200_ctx* ctx, int n, const float* features, int num_bits, uint8_t* packets, int32_t* indices) {
  if (!ctx || !features || !packets) return LYRA_B200_EINVAL;
  int rc = CheckRvq(ctx, n, num_bits);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_features, features, sizeof(float) * 64 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchQuantizeCall(ctx, n, ctx->d_features, num_bits, ctx->d_packets, indices ? ctx->d_indices : nullptr))) return rc;
  CU(cudaMemcpyAsync(packets, ctx->d_packets, (size_t)PacketBytes(num_bits) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if (indices) CU(cudaMemcpyAsync(indices, ctx->d_indices, sizeof(int) * 46 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_quantize_device(lyra_b200_ctx* ctx, int n, const float* d_features, int num_bits, uint8_t* d_packets, int32_t* d_indices) {
  if (!ctx || !d_features || !d_packets) return LYRA_B200_EINVAL;
  const int rc = CheckRvq(ctx, n, num_bits);
  return rc ? rc : LaunchQuantizeCall(ctx, n, d_features, num_bits, d_packets, d_indices);
}

int lyra_b200_dequantize(lyra_b200_ctx* ctx, int n, const uint8_t* packets, int num_bits, float* features) {
  if (!ctx || !features || !packets) return LYRA_B200_EINVAL;
  int rc = CheckRvq(ctx, n, num_bits);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_packets, packets, (size_t)PacketBytes(num_bits) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchDequantizeCall(ctx, n, ctx->d_packets, num_bits, ctx->d_features))) return rc;
  CU(cudaMemcpyAsync(features, ctx->d_features, sizeof(float) * 64 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_dequantize_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, int num_bits, float* d_features) {
  if (!ctx || !d_packets || !d_features) return LYRA_B200_EINVAL;
  const int rc = CheckRvq(ctx, n, num_bits);
  return rc ? rc : LaunchDequantizeCall(ctx, n, d_packets, num_bits, d_features);
}

int lyra_b200_generate(lyra_b200_ctx* ctx, const int32_t* ids, int n, const float* features, int16_t* pcm) {
  if (!ctx || !features || !pcm) return LYRA_B200_EINVAL;
  int rc = CheckNets(ctx, LYRA_B200_ROLE_DECODER, ids, n);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_features, features, sizeof(float) * 64 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchDecoderNets(ctx, WholeCall(ctx, n), nullptr, ctx->d_features, ctx->d_pcm, nullptr))) return rc;
  CU(cudaMemcpyAsync(pcm, ctx->d_pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_generate_device(lyra_b200_ctx* ctx, int n, const float* d_features, int16_t* d_pcm) {
  if (!ctx || !d_features || !d_pcm) return LYRA_B200_EINVAL;
  const int rc = CheckNets(ctx, LYRA_B200_ROLE_DECODER, nullptr, n);
  return rc ? rc : ForEachPart(ctx, n, [&](const Part& p) { return LaunchDecoderNets(ctx, p, nullptr, d_features, d_pcm, nullptr); });
}

int lyra_b200_logmel(lyra_b200_ctx* ctx, int bank, const int32_t* ids, int n, const int16_t* pcm, int num_mel_bins, float* out) {
  if (!ctx || !pcm || !out) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int rc = CheckLogMel(ctx, bank, ids, n, num_mel_bins, &d_ids);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_pcm, pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchLogMelCall(ctx, bank, d_ids, n, ctx->d_pcm, num_mel_bins, ctx->d_melout))) return rc;
  CU(cudaMemcpyAsync(out, ctx->d_melout, sizeof(float) * (size_t)num_mel_bins * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_logmel_device(lyra_b200_ctx* ctx, int bank, int n, const int16_t* d_pcm, int num_mel_bins, float* d_out) {
  if (!ctx || !d_pcm || !d_out) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  const int rc = CheckLogMel(ctx, bank, nullptr, n, num_mel_bins, &d_ids);
  return rc ? rc : LaunchLogMelCall(ctx, bank, nullptr, n, d_pcm, num_mel_bins, d_out);
}

int lyra_b200_noise_update(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, const uint8_t* update_mask,
                           uint8_t* is_noise, float* noise_estimate) {
  if (!ctx || !pcm) return LYRA_B200_EINVAL;
  ENTER(0);
  const int* d_ids = nullptr;
  int rc = CheckIds(ctx, ids, n, false);
  if (rc || (rc = UploadIds(ctx, ids, n, &d_ids))) return rc;
  CU(cudaMemcpyAsync(ctx->d_pcm, pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if (update_mask) CU(cudaMemcpyAsync(ctx->d_received, update_mask, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  rc = LaunchNoiseUpdate(ctx, ctx->stream, Rows(WholeCall(ctx, n), d_ids, nullptr), kWords16k, false, ctx->d_pcm,
                         update_mask ? ctx->d_received : nullptr, is_noise ? ctx->d_is_noise : nullptr,
                         noise_estimate ? ctx->d_noise_est : nullptr);
  if (rc) return rc;
  if (is_noise) CU(cudaMemcpyAsync(is_noise, ctx->d_is_noise, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if (noise_estimate) CU(cudaMemcpyAsync(noise_estimate, ctx->d_noise_est, sizeof(float) * 160 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_noise_update_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, const uint8_t* d_update_mask,
                                  uint8_t* d_is_noise, float* d_noise_estimate) {
  if (!ctx || !d_pcm) return LYRA_B200_EINVAL;
  ENTER(0);
  // no role check: the estimators are self-contained and allocated in every context, as for lyra_b200_noise_update
  const int rc = CheckIds(ctx, nullptr, n, false);
  if (rc) return rc;
  return LaunchNoiseUpdate(ctx, ctx->stream, Rows(WholeCall(ctx, n), nullptr, nullptr), kWords16k, false, d_pcm, d_update_mask,
                           d_is_noise, d_noise_estimate);
}

int lyra_b200_decode_track_noise(lyra_b200_ctx* ctx, const int32_t* ids, int n, const uint8_t* packets, const uint8_t* received,
                                 int num_bits, int16_t* pcm, uint8_t* is_noise) {
  if (!ctx || !packets || !pcm) return LYRA_B200_EINVAL;
  CodecCall c{kDecodeTrackNoise, n, num_bits, ids};
  c.host.packets_in = packets;
  c.host.received = received;
  c.host.pcm_out = pcm;
  c.host.flags = is_noise;
  return RunCodecCall(ctx, c);
}

int lyra_b200_decode_track_noise_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                                        int16_t* d_pcm, uint8_t* d_is_noise) {
  if (!ctx || !d_packets || !d_pcm) return LYRA_B200_EINVAL;
  CodecCall c{kDecodeTrackNoise, n, num_bits};
  c.dev.packets_in = d_packets;
  c.dev.received = d_received;
  c.dev.pcm_out = d_pcm;
  c.dev.flags = d_is_noise;
  return RunCodecCall(ctx, c);
}

int lyra_b200_encode_dtx(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, int num_bits, uint8_t* packets,
                         int32_t* packet_bytes) {
  if (!ctx || !pcm || !packets || !packet_bytes) return LYRA_B200_EINVAL;
  CodecCall c{kEncodeDtx, n, num_bits, ids};
  c.host.pcm_in = pcm;
  c.host.packets_out = packets;
  c.packet_bytes = packet_bytes;
  return RunCodecCall(ctx, c);
}

int lyra_b200_encode_dtx_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets, uint8_t* d_is_noise) {
  if (!ctx || !d_pcm || !d_packets || !d_is_noise) return LYRA_B200_EINVAL;
  CodecCall c{kEncodeDtx, n, num_bits};
  c.dev.pcm_in = d_pcm;
  c.dev.packets_out = d_packets;
  c.dev.flags = d_is_noise;
  return RunCodecCall(ctx, c);
}

int lyra_b200_decode_plc(lyra_b200_ctx* ctx, const int32_t* ids, int n, const uint8_t* packets, const uint8_t* received, int num_bits,
                         int16_t* pcm, uint8_t* is_comfort_noise) {
  if (!ctx || !packets || !pcm) return LYRA_B200_EINVAL;
  CodecCall c{kDecodePlc, n, num_bits, ids};
  c.host.packets_in = packets;
  c.host.received = received;
  c.host.pcm_out = pcm;
  c.host.flags = is_comfort_noise;
  return RunCodecCall(ctx, c);
}

int lyra_b200_decode_plc_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                                int16_t* d_pcm, uint8_t* d_is_comfort_noise) {
  if (!ctx || !d_packets || !d_pcm) return LYRA_B200_EINVAL;
  CodecCall c{kDecodePlc, n, num_bits};
  c.dev.packets_in = d_packets;
  c.dev.received = d_received;
  c.dev.pcm_out = d_pcm;
  c.dev.flags = d_is_comfort_noise;
  return RunCodecCall(ctx, c);
}

int lyra_b200_plc_get_state(lyra_b200_ctx* ctx, const int32_t* ids, int n, int32_t* state) {
  if (!ctx || !state) return LYRA_B200_EINVAL;
  ENTER(0);
  const int rc = CheckIds(ctx, ids, n, true);
  if (rc) return rc;
  CU(SyncStream(ctx));
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    CU(cudaMemcpy(state + (size_t)k * 3, ctx->d_plc + (size_t)id * 4, sizeof(int) * 3, cudaMemcpyDeviceToHost));
  }
  return LYRA_B200_OK;
}

int lyra_b200_plc_set_state(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int32_t* state) {
  if (!ctx || !state) return LYRA_B200_EINVAL;
  ENTER(0);
  const int rc = CheckIds(ctx, ids, n, true);
  if (rc) return rc;
  CU(SyncStream(ctx));
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    const int32_t* s3 = state + (size_t)k * 3;
    if (!PlcStateOk(s3[0], s3[1], s3[2])) {
      ctx->err = "decoder control state must be hop aligned: concealment 0..1280, fade 0..640, direction +-1";
      return LYRA_B200_EINVAL;
    }
    CU(cudaMemcpy(ctx->d_plc + (size_t)id * 4, s3, sizeof(int) * 3, cudaMemcpyHostToDevice));
  }
  return LYRA_B200_OK;
}

int lyra_b200_set_cng_seed(lyra_b200_ctx* ctx, uint64_t seed) {
  if (!ctx) return LYRA_B200_EINVAL;
  ctx->cng_seed = seed;
  return LYRA_B200_OK;
}

int lyra_b200_cng_generate(lyra_b200_ctx* ctx, const int32_t* ids, int n, const float* features, int16_t* pcm) {
  if (!ctx || !features || !pcm) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int rc = CheckRows(ctx, ids, n, &d_ids);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_cng_feat, features, sizeof(float) * 160 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchComfortNoise(ctx, ctx->stream, Rows(WholeCall(ctx, n), d_ids, nullptr), ctx->d_cng_feat, nullptr, ctx->d_cng_pcm)))
    return rc;
  CU(cudaMemcpyAsync(pcm, ctx->d_cng_pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_cng_generate_device(lyra_b200_ctx* ctx, int n, const float* d_features, int16_t* d_pcm) {
  if (!ctx || !d_features || !d_pcm) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  const int rc = CheckRows(ctx, nullptr, n, &d_ids);
  return rc ? rc : LaunchComfortNoise(ctx, ctx->stream, Rows(WholeCall(ctx, n), nullptr, nullptr), d_features, nullptr, d_pcm);
}

int lyra_b200_resample(lyra_b200_ctx* ctx, int to_internal, const int32_t* ids, int n, int external_rate_hz, const int16_t* in,
                       int in_samples, int16_t* out, int out_stride, int32_t* out_counts) {
  if (!ctx || !in || !out) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int pr = 0;
  int rc = CheckResample(ctx, to_internal, ids, n, external_rate_hz, in_samples, out_stride, &pr, &d_ids);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_rs_in, in, sizeof(int16_t) * (size_t)in_samples * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchResampleCall(ctx, pr, to_internal, external_rate_hz, d_ids, n, ctx->d_rs_in, in_samples, ctx->d_rs_out, out_stride,
                               ctx->d_rs_counts)))
    return rc;
  CU(cudaMemcpyAsync(out, ctx->d_rs_out, sizeof(int16_t) * (size_t)out_stride * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<int> counts((size_t)n);
  CU(cudaMemcpyAsync(counts.data(), ctx->d_rs_counts, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  if (out_counts) for (int k = 0; k < n; ++k) out_counts[k] = counts[(size_t)k];
  return LYRA_B200_OK;
}

int lyra_b200_resample_device(lyra_b200_ctx* ctx, int to_internal, int n, int external_rate_hz, const int16_t* d_in, int in_samples,
                              int16_t* d_out, int out_stride, int32_t* d_out_counts) {
  if (!ctx || !d_in || !d_out) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int pr = 0;
  const int rc = CheckResample(ctx, to_internal, nullptr, n, external_rate_hz, in_samples, out_stride, &pr, &d_ids);
  return rc ? rc : LaunchResampleCall(ctx, pr, to_internal, external_rate_hz, nullptr, n, d_in, in_samples, d_out, out_stride, d_out_counts);
}

int lyra_b200_stream_state_bytes(const lyra_b200_ctx* ctx) { return ctx ? (int)RecordBytes(ctx) : 0; }

int lyra_b200_export_streams(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, void* records) {
  if (!ctx || !records) return LYRA_B200_EINVAL;
  ENTER(0);
  int rc = CheckIds(ctx, stream_ids, n, true);
  if (rc || (rc = EnsureRecordStaging(ctx))) return rc;
  ctx->state_table.header[kHdrRate] = (uint32_t)ctx->sample_rate;
  const size_t rb = RecordBytes(ctx);
  StreamIdChunk ids;
  for (int k0 = 0; k0 < n; k0 += ctx->records_chunk) {
    ids.n = n - k0 < ctx->records_chunk ? n - k0 : ctx->records_chunk;
    for (int k = 0; k < ids.n; ++k) ids.src[k] = stream_ids ? stream_ids[k0 + k] : k0 + k;
    if ((rc = LAUNCH(kNoProf, StreamStateGatherKernel, StateGrid(ctx->state_table, ids.n, 1), dim3(kStateThreads), (size_t)kStateSmemBytes,
                     ctx->stream, ctx->state_table, ids, ctx->d_records, ctx->codec_rs_tag)))
      return rc;
    CU(cudaMemcpyAsync(static_cast<uint8_t*>(records) + rb * (size_t)k0, ctx->d_records, rb * (size_t)ids.n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_import_streams(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n, const void* records) {
  if (!ctx || !records) return LYRA_B200_EINVAL;
  ENTER(0);
  int rc = CheckIds(ctx, stream_ids, n, false);
  if (rc) return rc;
  const size_t rb = RecordBytes(ctx);
  const uint8_t* recs = static_cast<const uint8_t*>(records);
  bool own_rate = false;
  for (int k = 0; k < n; ++k) {                    // every record first: a bad one changes nothing
    if (const char* why = RecordProblem(ctx, recs + rb * (size_t)k)) {
      ctx->err = "record " + std::to_string(k) + ": " + why;
      return LYRA_B200_EINVAL;
    }
    for (size_t i = 0; i < ctx->state_list.size(); ++i)
      if (ctx->state_list[i].check == lyra_b200_ctx::kCheckStreamRate)
        own_rate |= RecordWord(recs + rb * (size_t)k, kStateHeaderWords + ctx->state_list[i].e.offset) != 0;
  }
  if ((rc = EnsureRecordStaging(ctx))) return rc;
  if (own_rate) ctx->rate_override = true;
  for (size_t i = 0; i < ctx->state_list.size(); ++i) {      // the mirrored words' host mirror
    const StreamStateEntry& e = ctx->state_list[i].e;
    for (int w = 0; w < kMirroredWords; ++w)
      if (e.state == reinterpret_cast<uint32_t*>(ctx->d_stream_word[w]))
        for (int k = 0; k < n; ++k)
          SetMirrorWord(ctx, w, stream_ids ? stream_ids[k] : k, (int32_t)RecordWord(recs + rb * (size_t)k, kStateHeaderWords + e.offset));
  }
  StreamIdChunk ids;
  for (int k0 = 0; k0 < n; k0 += ctx->records_chunk) {
    ids.n = n - k0 < ctx->records_chunk ? n - k0 : ctx->records_chunk;
    for (int k = 0; k < ids.n; ++k) ids.dst[k] = stream_ids ? stream_ids[k0 + k] : k0 + k;
    CU(cudaMemcpyAsync(ctx->d_records, recs + rb * (size_t)k0, rb * (size_t)ids.n, cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = LAUNCH(kNoProf, StreamStateScatterKernel, StateGrid(ctx->state_table, ids.n, 0), dim3(kStateThreads), (size_t)kStateSmemBytes,
                     ctx->stream, ctx->state_table, ids, ctx->d_records, ctx->codec_rs_tag)))
      return rc;
  }
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_copy_streams(lyra_b200_ctx* ctx, const int32_t* src_ids, const int32_t* dst_ids, int n) {
  if (!ctx || !src_ids || !dst_ids) return LYRA_B200_EINVAL;
  ENTER(0);
  int rc = CheckCopyIds(ctx, src_ids, dst_ids, n);
  if (rc || (rc = CopyStreamState(ctx, ctx->state_table, src_ids, dst_ids, n))) return rc;
  for (int w = 0; w < kMirroredWords; ++w)         // sources and destinations are disjoint
    for (int k = 0; k < n && ctx->d_stream_word[w]; ++k)
      SetMirrorWord(ctx, w, dst_ids[k], src_ids[k] < 0 ? 0 : ctx->word_mirror[w][(size_t)src_ids[k]]);
  return LYRA_B200_OK;
}

int lyra_b200_align_streams(lyra_b200_ctx* ctx, const int32_t* stream_ids, const int32_t* like_ids, int n) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (n == 0) return LYRA_B200_OK;
  if (!stream_ids || !like_ids) { ctx->err = "stream_ids and like_ids are required"; return LYRA_B200_EINVAL; }
  ENTER(0);
  int rc = CheckAlignIds(ctx, stream_ids, like_ids, n);
  if (rc) return rc;
  const StreamAlignTable& T = ctx->align_table;
  StreamIdChunk ids;
  for (int k0 = 0; k0 < n; k0 += kStateChunk) {     // the ids travel as kernel parameters
    ids.n = n - k0 < kStateChunk ? n - k0 : kStateChunk;
    for (int k = 0; k < ids.n; ++k) {
      ids.src[k] = like_ids[k0 + k];
      ids.dst[k] = stream_ids[k0 + k];
    }
    if ((rc = LAUNCH(kNoProf, StreamAlignKernel, dim3((unsigned)((ids.n + kStateRows - 1) / kStateRows), (unsigned)T.count),
                     dim3(kStateThreads), (size_t)0, ctx->stream, T, ids)))
      return rc;
  }
  return LYRA_B200_OK;
}

int lyra_b200_noise_estimate(lyra_b200_ctx* ctx, const int32_t* ids, int n, float* noise_estimate, uint8_t* is_noise) {
  if (!ctx || (!noise_estimate && !is_noise)) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int rc = CheckRows(ctx, ids, n, &d_ids);
  if (rc || (rc = LaunchNoiseRead(ctx, d_ids, n, noise_estimate ? ctx->d_noise_est : nullptr, is_noise ? ctx->d_is_noise : nullptr)))
    return rc;
  if (noise_estimate) CU(cudaMemcpyAsync(noise_estimate, ctx->d_noise_est, sizeof(float) * 160 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if (is_noise) CU(cudaMemcpyAsync(is_noise, ctx->d_is_noise, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_noise_estimate_device(lyra_b200_ctx* ctx, int n, float* d_noise_estimate, uint8_t* d_is_noise) {
  if (!ctx || (!d_noise_estimate && !d_is_noise)) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  const int rc = CheckRows(ctx, nullptr, n, &d_ids);
  return rc ? rc : LaunchNoiseRead(ctx, nullptr, n, d_noise_estimate, d_is_noise);
}

}  // extern "C"
