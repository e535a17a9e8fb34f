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

// inside a loop of a forked region: record the error and leave the loop (the region is joined afterwards)
#define CUB(call)                                                                       \
  {                                                                                     \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess) {                                                            \
      ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                    \
      rc = LYRA_B200_ENODEV;                                                            \
      break;                                                                            \
    }                                                                                   \
  }

}  // namespace

struct lyra_b200_ctx {
  ModelSpec spec;
  int device = 0, max_streams = 0, ntiles = 0, padded = 0;
  int S = 8;                // streams per tile (8: two blocks per SM; 16: one)
  int roles = LYRA_B200_ROLE_ENCODER | LYRA_B200_ROLE_DECODER;   // which halves of the streaming state this context holds
  uint8_t* d_blob = nullptr;
  // streaming state, one block per kernel
  uint32_t* d_state[4] = {nullptr, nullptr, nullptr, nullptr};
  uint32_t* d_init[4] = {nullptr, nullptr, nullptr, nullptr};
  int* d_n18[4] = {nullptr, nullptr, nullptr, nullptr};
  int units[4] = {EncStateA::kUnits, EncStateB::kUnits, DecStateC::kUnits, DecStateD::kUnits};
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
  unsigned long long* d_cng_hops = nullptr;  // [max_streams]
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
  const uint8_t* cur_skip = nullptr;         // skip mask of the call in flight (TileIo::skip)
  // sample-rate converters: [direction 0 = to 16 kHz (encoder side), 1 = from 16 kHz (decoder side)][max_streams] state
  int16_t* d_rs_delay[2] = {nullptr, nullptr};   // [max_streams][34]
  int* d_rs_pos[2] = {nullptr, nullptr};         // [max_streams][2] {position, rate}
  int16_t* d_rs_in = nullptr;                    // staging [max_streams][960]
  int16_t* d_rs_out = nullptr;
  int* d_rs_counts = nullptr;
  // device staging for the host-buffer API
  int16_t* d_pcm = nullptr;
  uint8_t* d_packets = nullptr;
  uint8_t* d_received = nullptr;
  float* d_features = nullptr;
  float* d_melout = nullptr;
  int* d_indices = nullptr;
  int* d_ids = nullptr;
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
  struct GraphKey {
    int kind, n, num_bits, mode, nsplit;
    const void *a, *b, *c;
    bool operator==(const GraphKey& o) const {
      return kind == o.kind && n == o.n && num_bits == o.num_bits && mode == o.mode && nsplit == o.nsplit && a == o.a && b == o.b && c == o.c;
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

// RAII pair of events around one kernel launch (no-op unless profiling is enabled)
struct ProfScope {
  lyra_b200_ctx* ctx;
  int k;
  cudaEvent_t stop = nullptr;
  cudaStream_t st;
  ProfScope(lyra_b200_ctx* c, int kernel, cudaStream_t stream) : ctx(c), k(kernel), st(stream) {
    if (!ctx->profiling) return;
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

// Build / upload the (tile list, slot-of-stream) map for this call.  The copies are stream-ordered behind the previous call's
// kernels (sub-batch streams are joined into ctx->stream at the end of every call), and the pinned host image is
// double-buffered, so a server whose active set changes every tick never waits for the GPU here.
int PrepareMap(lyra_b200_ctx* ctx, const int32_t* ids, int n) {
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  if (ids == nullptr && ctx->map_dense_n == n) return LYRA_B200_OK;
  const int b = ctx->map_buf;
  if (ctx->map_pending[b]) { CU(cudaEventSynchronize(ctx->ev_map[b])); ctx->map_pending[b] = false; }   // two calls ago: long done
  int* slot_of = ctx->h_slot_of[b];
  int* tile_list = ctx->h_tile_list[b];
  for (int id : ctx->touched[b]) slot_of[id] = -1;
  ctx->touched[b].clear();
  int ntl = 0;
  int rc = LYRA_B200_OK;
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    if (id < 0 || id >= ctx->max_streams) { ctx->err = "stream id out of range"; rc = LYRA_B200_EINVAL; break; }
    if (slot_of[id] != -1) { ctx->err = "duplicate stream id in one call"; rc = LYRA_B200_EINVAL; break; }
    slot_of[id] = k;
    ctx->touched[b].push_back(id);
  }
  if (rc) { ctx->map_dense_n = -1; return rc; }
  // tiles in order of first appearance
  if (++ctx->map_gen == 0) { std::fill(ctx->tile_gen.begin(), ctx->tile_gen.end(), 0u); ctx->map_gen = 1; }
  for (int k = 0; k < n; ++k) {
    const int t = (ids ? ids[k] : k) / ctx->S;
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

template <int kS>
int LaunchEncoderNetsT(lyra_b200_ctx* ctx, const Part& p, const int16_t* d_pcm, float* d_features) {
  const TileIo io{ctx->d_tile_list + p.tile0, ctx->d_slot_of, ctx->cur_skip};
  { ProfScope ps(ctx, 0, p.st);
  LYRA_LAUNCH(EncoderKernelA<kS>, dim3((unsigned)p.ntiles), dim3(EncA<kS>::NT), (size_t)EncA<kS>::kSmemBytes, p.st,
              ctx->d_blob, ctx->spec.enc, io, d_pcm, reinterpret_cast<float*>(ctx->d_state[0]), ctx->d_n18[0], ctx->d_mid_enc); }
  { ProfScope ps(ctx, 1, p.st);
  LYRA_LAUNCH(EncoderKernelB<kS>, dim3((unsigned)p.ntiles), dim3(EncB<kS>::NT), (size_t)EncB<kS>::kSmemBytes, p.st,
              ctx->d_blob, ctx->spec.enc, io, ctx->d_mid_enc, reinterpret_cast<float*>(ctx->d_state[1]), ctx->d_n18[1], d_features); }
  ctx->launches += 2;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}
int LaunchEncoderNets(lyra_b200_ctx* ctx, const Part& p, const int16_t* d_pcm, float* d_features) {
  return ctx->S == 16 ? LaunchEncoderNetsT<16>(ctx, p, d_pcm, d_features) : LaunchEncoderNetsT<8>(ctx, p, d_pcm, d_features);
}

int LaunchQuantize(lyra_b200_ctx* ctx, const Part& p, const float* d_features, int num_bits, uint8_t* d_packets, int* d_indices,
                   const uint8_t* d_skip = nullptr) {
  const int nq = num_bits / ctx->spec.bits_per_stage, pb = PacketBytes(num_bits);
  const int blocks = (p.nslots + kRvqSlotsPerBlock - 1) / kRvqSlotsPerBlock;
  { ProfScope ps(ctx, 2, p.st);
  LYRA_LAUNCH(RvqEncodeKernel, dim3((unsigned)blocks), dim3(kRvqThreads), (size_t)(2 * 1024 * 4 + kRvqSlotsPerBlock * (64 * 4 + 48 * 4)), p.st,
              ctx->d_blob, ctx->spec.rvq, d_features + (size_t)p.slot0 * 64, p.nslots, nq, d_packets + (size_t)p.slot0 * pb, pb,
              d_indices ? d_indices + (size_t)p.slot0 * 46 : nullptr, d_skip ? d_skip + p.slot0 : nullptr); }
  ctx->launches += 1;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}

int LaunchDequantize(lyra_b200_ctx* ctx, const Part& p, const uint8_t* d_packets, const uint8_t* d_received, int num_bits, float* d_features) {
  const int nq = num_bits / ctx->spec.bits_per_stage, pb = PacketBytes(num_bits);
  const int blocks = (p.nslots * 64 + 255) / 256;
  { ProfScope ps(ctx, 3, p.st);
  LYRA_LAUNCH(RvqDecodeKernel, dim3((unsigned)blocks), dim3(256), (size_t)0, p.st,
              ctx->d_blob, ctx->spec.rvq, d_packets + (size_t)p.slot0 * pb, pb, d_received ? d_received + p.slot0 : nullptr, p.nslots, nq,
              d_features + (size_t)p.slot0 * 64); }
  ctx->launches += 1;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}

template <int kS, bool kTC>
int LaunchDecoderNetsT(lyra_b200_ctx* ctx, const Part& p, const float* d_features, int16_t* d_pcm) {
  const TileIo io{ctx->d_tile_list + p.tile0, ctx->d_slot_of, ctx->cur_skip};
  using LC = DecC<kS, kTC>;
  using LD = DecD<kS, kTC>;
  { ProfScope ps(ctx, 4, p.st);
  LYRA_LAUNCH((DecoderKernelC<kS, kTC>), dim3((unsigned)p.ntiles), dim3(LC::NT), (size_t)LC::kSmemBytes, p.st,
              ctx->d_blob, ctx->spec.dec, io, d_features, reinterpret_cast<float*>(ctx->d_state[2]), ctx->d_n18[2], ctx->d_mid_dec); }
  { ProfScope ps(ctx, 5, p.st);
  LYRA_LAUNCH((DecoderKernelD<kS, kTC>), dim3((unsigned)p.ntiles), dim3(LD::NT), (size_t)LD::kSmemBytes, p.st,
              ctx->d_blob, ctx->spec.dec, io, ctx->d_mid_dec, reinterpret_cast<float*>(ctx->d_state[3]), ctx->d_n18[3], d_pcm); }
  ctx->launches += 2;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}
// Tensor mode at 8-stream tiles (the default tile): kernel C with its fp32 residual units on mma.sync TF32, kernel D on warpgroup
// MMAs (wgmma, A operands and accumulators in registers; net_kernels_wgmma.cuh).
int LaunchDecoderNetsWgmma(lyra_b200_ctx* ctx, const Part& p, const float* d_features, int16_t* d_pcm) {
  const TileIo io{ctx->d_tile_list + p.tile0, ctx->d_slot_of, ctx->cur_skip};
  using LC = DecC<8, true>;
  { ProfScope ps(ctx, 4, p.st);
  LYRA_LAUNCH((DecoderKernelC<8, true>), dim3((unsigned)p.ntiles), dim3(LC::NT), (size_t)LC::kSmemBytes, p.st,
              ctx->d_blob, ctx->spec.dec, io, d_features, reinterpret_cast<float*>(ctx->d_state[2]), ctx->d_n18[2], ctx->d_mid_dec); }
  { ProfScope ps(ctx, 5, p.st);
  LYRA_LAUNCH(DecoderKernelDW, dim3((unsigned)p.ntiles), dim3(DecDW::NT), (size_t)DecDW::kSmemBytes, p.st,
              ctx->d_blob, ctx->spec.dec, io, ctx->d_mid_dec, reinterpret_cast<float*>(ctx->d_state[3]), ctx->d_n18[3], d_pcm); }
  ctx->launches += 2;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}
int LaunchDecoderNets(lyra_b200_ctx* ctx, const Part& p, const float* d_features, int16_t* d_pcm) {
  const bool tc = ctx->decoder_mode == LYRA_B200_DECODER_TENSOR;
  if (tc && ctx->S == 8) return LaunchDecoderNetsWgmma(ctx, p, d_features, d_pcm);
  if (ctx->S == 16) return tc ? LaunchDecoderNetsT<16, true>(ctx, p, d_features, d_pcm) : LaunchDecoderNetsT<16, false>(ctx, p, d_features, d_pcm);
  return tc ? LaunchDecoderNetsT<8, true>(ctx, p, d_features, d_pcm) : LaunchDecoderNetsT<8, false>(ctx, p, d_features, d_pcm);
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
    const int s0 = t0 * ctx->S, s1 = i + 1 == np ? n : t1 * ctx->S;
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

// log-mel of this hop (the estimator's own extractor, bank 2) + the estimator recurrences for slots
// [slot0, slot0 + count) on stream `st`; all arrays are indexed by slot, n = total slots of the call
int LaunchNoiseUpdate(lyra_b200_ctx* ctx, cudaStream_t st, const int* d_ids, int slot0, int count, int n, const int16_t* d_pcm,
                      const uint8_t* d_mask, uint8_t* d_is_noise, float* d_estimate, bool encoder_side = false) {
  float* noise_state = encoder_side ? ctx->d_noise_enc : ctx->d_noise;
  int16_t* carried = encoder_side ? ctx->d_logmel_prev_enc : ctx->d_logmel_prev[2];
  const LogMelParams& P = ctx->spec.logmel160;
  const size_t smem = sizeof(double) * (size_t)(2 * kLogMelFftPadded + P.fft / 2 + 1 + P.window_len + P.window_len / 8 + 1);
  { ProfScope ps(ctx, 6, st);
  LYRA_LAUNCH(LogMelKernel, dim3((unsigned)count), dim3(kLogMelThreads), smem, st,
              ctx->d_blob, P, d_ids, n, d_pcm, carried, ctx->d_melout, d_mask, slot0); }
  { ProfScope ps(ctx, 7, st);
  LYRA_LAUNCH(NoiseEstimatorKernel, dim3((unsigned)count), dim3(kNoiseThreads), sizeof(float) * (size_t)(2 * 160 + 2), st,
              ctx->noise_params, d_ids, n, ctx->d_melout, d_mask, noise_state, d_is_noise, d_estimate, slot0); }
  ctx->launches += 2;
  CU(cudaGetLastError());
  return LYRA_B200_OK;
}

// h_pcm / h_packets (host-buffer API): each part copies its own slice in on its own stream before its kernels and
// its result out right after them, so the copies of one part overlap the kernels of the others.
// dtx: every sub-batch first feeds its hops to the encoder-side noise estimators; hops classified as noise skip the encoder
// (their streams' state does not advance) and get an empty packet (lyra/lyra_encoder.cc:131-141); d_is_noise[slot] = 1 marks them
int RunEncode(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets,
              const int16_t* h_pcm = nullptr, uint8_t* h_packets = nullptr, bool dtx = false, const int* d_ids = nullptr,
              uint8_t* d_is_noise = nullptr, uint8_t* h_is_noise = nullptr) {
  Part parts[lyra_b200_ctx::kMaxSplit];
  const int np = SplitParts(ctx, n, parts);
  const size_t pb = (size_t)PacketBytes(num_bits);
  int rc = Fork(ctx, np);
  if (rc) return rc;
  for (int i = 0; i < np && !rc; ++i) {
    const Part& p = parts[i];
    if (h_pcm)
      CUB(cudaMemcpyAsync(ctx->d_pcm + (size_t)p.slot0 * 320, h_pcm + (size_t)p.slot0 * 320, sizeof(int16_t) * 320 * (size_t)p.nslots,
                          cudaMemcpyHostToDevice, p.st));
    if (dtx) {
      if ((rc = LaunchNoiseUpdate(ctx, p.st, d_ids, p.slot0, p.nslots, n, d_pcm, nullptr, d_is_noise, nullptr, true))) break;
      if (h_is_noise) CUB(cudaMemcpyAsync(h_is_noise + p.slot0, d_is_noise + p.slot0, (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
    }
    ctx->cur_skip = dtx ? d_is_noise : nullptr;
    rc = LaunchEncoderNets(ctx, p, d_pcm, ctx->d_features);
    ctx->cur_skip = nullptr;
    if (rc) break;
    if ((rc = LaunchQuantize(ctx, p, ctx->d_features, num_bits, d_packets, nullptr, dtx ? d_is_noise : nullptr))) break;
    if (h_packets)
      CUB(cudaMemcpyAsync(h_packets + (size_t)p.slot0 * pb, d_packets + (size_t)p.slot0 * pb, pb * (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
  }
  return JoinAfter(ctx, np, rc);
}

// track_noise: every sub-batch also feeds its decoded hops to the per-stream noise estimators (received streams only),
// as LyraDecoder::DecodeSamplesInternal does (lyra/lyra_decoder.cc:306-311); d_ids = the call's stream ids (sparse calls)
int RunDecode(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits, int16_t* d_pcm,
              const uint8_t* h_packets = nullptr, const uint8_t* h_received = nullptr, int16_t* h_pcm = nullptr,
              bool track_noise = false, const int* d_ids = nullptr, uint8_t* d_is_noise = nullptr, uint8_t* h_is_noise = nullptr) {
  Part parts[lyra_b200_ctx::kMaxSplit];
  const int np = SplitParts(ctx, n, parts);
  const size_t pb = (size_t)PacketBytes(num_bits);
  int rc = Fork(ctx, np);
  if (rc) return rc;
  for (int i = 0; i < np && !rc; ++i) {
    const Part& p = parts[i];
    if (h_packets)
      CUB(cudaMemcpyAsync(ctx->d_packets + (size_t)p.slot0 * pb, h_packets + (size_t)p.slot0 * pb, pb * (size_t)p.nslots, cudaMemcpyHostToDevice, p.st));
    if (h_received)
      CUB(cudaMemcpyAsync(ctx->d_received + p.slot0, h_received + p.slot0, (size_t)p.nslots, cudaMemcpyHostToDevice, p.st));
    if ((rc = LaunchDequantize(ctx, p, d_packets, d_received, num_bits, ctx->d_features))) break;
    if ((rc = LaunchDecoderNets(ctx, p, ctx->d_features, d_pcm))) break;
    if (track_noise) {
      if ((rc = LaunchNoiseUpdate(ctx, p.st, d_ids, p.slot0, p.nslots, n, d_pcm, d_received, d_is_noise, nullptr))) break;
      if (h_is_noise) CUB(cudaMemcpyAsync(h_is_noise + p.slot0, d_is_noise + p.slot0, (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
    }
    if (h_pcm)
      CUB(cudaMemcpyAsync(h_pcm + (size_t)p.slot0 * 320, d_pcm + (size_t)p.slot0 * 320, sizeof(int16_t) * 320 * (size_t)p.nslots,
                          cudaMemcpyDeviceToHost, p.st));
  }
  return JoinAfter(ctx, np, rc);
}

// LyraDecoder::{SetEncodedPacket, DecodeSamples(320)} with the reference's concealment / comfort-noise / fade behaviour for n
// streams (lyra/lyra_decoder.cc:172-315): plan (per-stream state machine) -> RVQ decode -> LyraGAN for the streams that need
// model audio -> comfort noise from the current noise estimates for the streams that need it -> cross-fade -> noise-estimator
// update of the streams that decoded a received packet.  One whole hop per stream and call.
int RunDecodePlc(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits, int16_t* d_pcm,
                 const int* d_ids, uint8_t* d_is_cn, const uint8_t* h_packets, const uint8_t* h_received, int16_t* h_pcm, uint8_t* h_is_cn) {
  const size_t pb = (size_t)PacketBytes(num_bits);
  if (h_received) CU(cudaMemcpyAsync(ctx->d_received, h_received, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  LYRA_LAUNCH(PlcPlanKernel, dim3((unsigned)((n + 255) / 256)), dim3(256), (size_t)0, ctx->stream,
              d_ids, n, d_received, ctx->d_plc, ctx->d_plan, ctx->d_fade0, ctx->d_dir, ctx->d_skip, ctx->d_feed, d_is_cn);
  ctx->launches += 1;
  CU(cudaGetLastError());
  Part parts[lyra_b200_ctx::kMaxSplit];
  const int np = SplitParts(ctx, n, parts);
  int rc = Fork(ctx, np);
  if (rc) return rc;
  const size_t cng_smem = sizeof(double) * (size_t)(4 * kLogMelFftPadded + 160);
  for (int i = 0; i < np && !rc; ++i) {
    const Part& p = parts[i];
    if (h_packets)
      CUB(cudaMemcpyAsync(ctx->d_packets + (size_t)p.slot0 * pb, h_packets + (size_t)p.slot0 * pb, pb * (size_t)p.nslots, cudaMemcpyHostToDevice, p.st));
    if ((rc = LaunchDequantize(ctx, p, d_packets, d_received, num_bits, ctx->d_features))) break;
    ctx->cur_skip = ctx->d_skip;
    rc = LaunchDecoderNets(ctx, p, ctx->d_features, ctx->d_model_pcm);
    ctx->cur_skip = nullptr;
    if (rc) break;
    LYRA_LAUNCH(ComfortNoiseKernel, dim3((unsigned)p.nslots), dim3(kCngThreads), cng_smem, p.st,
                ctx->d_blob, ctx->spec.cng, d_ids, n, (const float*)nullptr, ctx->d_noise, NoiseStateUnits(ctx->noise_params.nf),
                ctx->d_plan, ctx->d_cng_work, ctx->d_cng_hops, ctx->cng_seed, ctx->d_cng_pcm, p.slot0);
    LYRA_LAUNCH(PlcMixKernel, dim3((unsigned)p.nslots), dim3(320), (size_t)0, p.st,
                ctx->d_blob, ctx->spec.cng, p.nslots, ctx->d_plan + p.slot0, ctx->d_fade0 + p.slot0, ctx->d_dir + p.slot0,
                ctx->d_model_pcm + (size_t)p.slot0 * 320, ctx->d_cng_pcm + (size_t)p.slot0 * 320, d_pcm + (size_t)p.slot0 * 320);
    ctx->launches += 2;
    CUB(cudaGetLastError());
    if ((rc = LaunchNoiseUpdate(ctx, p.st, d_ids, p.slot0, p.nslots, n, ctx->d_model_pcm, ctx->d_feed, nullptr, nullptr))) break;
    if (h_pcm)
      CUB(cudaMemcpyAsync(h_pcm + (size_t)p.slot0 * 320, d_pcm + (size_t)p.slot0 * 320, sizeof(int16_t) * 320 * (size_t)p.nslots,
                          cudaMemcpyDeviceToHost, p.st));
    if (h_is_cn) CUB(cudaMemcpyAsync(h_is_cn + p.slot0, d_is_cn + p.slot0, (size_t)p.nslots, cudaMemcpyDeviceToHost, p.st));
  }
  return JoinAfter(ctx, np, rc);
}

// stream ids of a sparse call -> device (validated: in range, no duplicates); *d_ids stays nullptr for dense calls
int UploadIds(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int** d_ids) {
  *d_ids = nullptr;
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  if (!ids) return LYRA_B200_OK;
  std::vector<char> seen((size_t)ctx->max_streams, 0);
  for (int k = 0; k < n; ++k) {
    if (ids[k] < 0 || ids[k] >= ctx->max_streams || seen[(size_t)ids[k]]) { ctx->err = "bad or duplicate stream id"; return LYRA_B200_EINVAL; }
    seen[(size_t)ids[k]] = 1;
  }
  CU(cudaMemcpyAsync(ctx->d_ids, ids, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  CU(SyncStream(ctx));          // `ids` is the caller's (pageable) memory
  *d_ids = ctx->d_ids;
  return LYRA_B200_OK;
}

template <int kS>
bool SetSmemLimits() {
  return LYRA_SET_MAX_SMEM(EncoderKernelA<kS>, EncA<kS>::kSmemBytes) == 0 && LYRA_SET_MAX_SMEM(EncoderKernelB<kS>, EncB<kS>::kSmemBytes) == 0 &&
         LYRA_SET_MAX_SMEM((DecoderKernelC<kS, false>), (DecC<kS, false>::kSmemBytes)) == 0 &&
         LYRA_SET_MAX_SMEM((DecoderKernelD<kS, false>), (DecD<kS, false>::kSmemBytes)) == 0 &&
         LYRA_SET_MAX_SMEM((DecoderKernelC<kS, true>), (DecC<kS, true>::kSmemBytes)) == 0 &&
         LYRA_SET_MAX_SMEM((DecoderKernelD<kS, true>), (DecD<kS, true>::kSmemBytes)) == 0;
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

int ResetImpl(lyra_b200_ctx* ctx, const int32_t* ids, int n) {
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  const int* d_ids = nullptr;
  if (ids) {
    for (int k = 0; k < n; ++k)
      if (ids[k] < 0 || ids[k] >= ctx->max_streams) { ctx->err = "stream id out of range"; return LYRA_B200_EINVAL; }
    CU(cudaMemcpyAsync(ctx->d_ids, ids, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    d_ids = ctx->d_ids;
  }
  for (int w = 0; w < 4; ++w) {
    if (!ctx->d_state[w]) continue;
    LYRA_LAUNCH(ResetStateKernel, dim3((unsigned)n), dim3(256), (size_t)0, ctx->stream,
                ctx->d_state[w], ctx->d_init[w], ctx->units[w], ctx->S, d_ids, n, ctx->d_n18[w]);
    ctx->launches += 1;
  }
  CU(cudaGetLastError());
  // log-mel carried samples
  for (int b = 0; b < 3; ++b) {
    if (!ids) {
      CU(cudaMemsetAsync(ctx->d_logmel_prev[b], 0, sizeof(int16_t) * 320 * (size_t)n, ctx->stream));
    } else {
      for (int k = 0; k < n; ++k)
        CU(cudaMemsetAsync(ctx->d_logmel_prev[b] + (size_t)ids[k] * 320, 0, sizeof(int16_t) * 320, ctx->stream));
    }
  }
  // noise estimator: all-zero is the freshly constructed object
  const size_t nu = (size_t)NoiseStateUnits(ctx->noise_params.nf);
  if (!ids) {
    CU(cudaMemsetAsync(ctx->d_noise, 0, sizeof(float) * nu * (size_t)n, ctx->stream));
  } else {
    for (int k = 0; k < n; ++k) CU(cudaMemsetAsync(ctx->d_noise + (size_t)ids[k] * nu, 0, sizeof(float) * nu, ctx->stream));
  }
  // decoder control state (0, 0, fade from comfort noise: lyra_decoder.cc:164-166), comfort-noise buffers and hop counters,
  // encoder-side estimators and their carried samples
  std::vector<int> hs;
  if (ids) hs.assign(ids, ids + n); else { hs.resize((size_t)n); for (int k = 0; k < n; ++k) hs[(size_t)k] = k; }
  const int plc0[4] = {0, 0, -1, 0};
  for (int k = 0; k < n && ids; ++k) {
    const size_t id = (size_t)hs[(size_t)k];
    CU(cudaMemcpyAsync(ctx->d_plc + id * 4, plc0, sizeof(plc0), cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_cng_work + id * 1024, 0, sizeof(double) * 1024, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_cng_hops + id, 0, sizeof(unsigned long long), ctx->stream));
    CU(cudaMemsetAsync(ctx->d_noise_enc + id * nu, 0, sizeof(float) * nu, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_logmel_prev_enc + id * 320, 0, sizeof(int16_t) * 320, ctx->stream));
    for (int d = 0; d < 2; ++d) CU(cudaMemsetAsync(ctx->d_rs_pos[d] + id * 2, 0, sizeof(int) * 2, ctx->stream));   // rate 0: the next call starts fully primed
  }
  if (!ids) {
    std::vector<int> img((size_t)n * 4);
    for (int k = 0; k < n; ++k) { img[(size_t)k * 4] = 0; img[(size_t)k * 4 + 1] = 0; img[(size_t)k * 4 + 2] = -1; img[(size_t)k * 4 + 3] = 0; }
    CU(cudaMemcpy(ctx->d_plc, img.data(), sizeof(int) * img.size(), cudaMemcpyHostToDevice));
    CU(cudaMemsetAsync(ctx->d_cng_work, 0, sizeof(double) * 1024 * (size_t)n, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_cng_hops, 0, sizeof(unsigned long long) * (size_t)n, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_noise_enc, 0, sizeof(float) * nu * (size_t)n, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_logmel_prev_enc, 0, sizeof(int16_t) * 320 * (size_t)n, ctx->stream));
    for (int d = 0; d < 2; ++d) CU(cudaMemsetAsync(ctx->d_rs_pos[d], 0, sizeof(int) * 2 * (size_t)n, ctx->stream));
  }
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

template <typename T>
cudaError_t DevAlloc(T** p, size_t count) {
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), sizeof(T) * (count ? count : 1));
  if (e == cudaSuccess) e = cudaMemset(*p, 0, sizeof(T) * (count ? count : 1));
  return e;
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


}  // namespace

#if defined(LYRA_PHASE_PROF) && !defined(LYRA_EMU)
// development aid: returns clock64() stamps [4 kernels][1024 blocks][48 phases] of the most recent launches
extern "C" int lyra_b200_debug_phases(lyra_b200_ctx* ctx, long long* out) {
  static long long* d_buf = nullptr;
  const size_t n = (size_t)4 * 1024 * 48;
  if (!d_buf) {
    cudaMalloc(reinterpret_cast<void**>(&d_buf), n * sizeof(long long));
    cudaMemset(d_buf, 0, n * sizeof(long long));
    cudaMemcpyToSymbol(lyra_b200::g_phase_prof, &d_buf, sizeof(d_buf));
    return 1;
  }
  cudaStreamSynchronize(ctx->stream);
  cudaMemcpy(out, d_buf, n * sizeof(long long), cudaMemcpyDeviceToHost);
  return 0;
}
#endif

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
  {
    // streams per tile: 8 (default, two blocks per SM) or 16; LYRA_B200_TILE_STREAMS overrides for experiments
    const char* e = std::getenv("LYRA_B200_TILE_STREAMS");
    ctx->S = (e && std::atoi(e) == 16) ? 16 : 8;
  }
  const int kS = ctx->S;
  ctx->ntiles = (max_streams + kS - 1) / kS;
  ctx->padded = ctx->ntiles * kS;
  ctx->tile_gen.assign((size_t)ctx->ntiles, 0u);
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
  if (const char* e = std::getenv("LYRA_B200_BLOCKING_SYNC")) ctx->blocking_sync = std::atoi(e) != 0;
  if (const char* e = std::getenv("LYRA_B200_SPLIT")) ctx->nsplit = std::atoi(e);
  if (const char* e = std::getenv("LYRA_B200_DECODER_MODE")) ctx->decoder_mode = std::strcmp(e, "tensor") == 0 ? LYRA_B200_DECODER_TENSOR : LYRA_B200_DECODER_EXACT;
  ctx->stream = ctx->own_stream;
  ok = ok && DevAlloc(&ctx->d_blob, ctx->spec.blob.size()) == cudaSuccess;
  ok = ok && cudaMemcpy(ctx->d_blob, ctx->spec.blob.data(), ctx->spec.blob.size(), cudaMemcpyHostToDevice) == cudaSuccess;
  for (int w = 0; w < 4 && ok; ++w) {
    if (!(roles & (w < 2 ? LYRA_B200_ROLE_ENCODER : LYRA_B200_ROLE_DECODER))) continue;   // an encoder-only / decoder-only context
    const std::vector<uint32_t> img = InitImage(ctx->spec, w);
    ok = ok && DevAlloc(&ctx->d_state[w], (size_t)ctx->units[w] * P) == cudaSuccess;
    ok = ok && DevAlloc(&ctx->d_init[w], img.size()) == cudaSuccess;
    ok = ok && cudaMemcpy(ctx->d_init[w], img.data(), img.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && DevAlloc(&ctx->d_n18[w], P) == cudaSuccess;
  }
  if (roles & LYRA_B200_ROLE_ENCODER) ok = ok && DevAlloc(&ctx->d_mid_enc, (size_t)ctx->ntiles * 128 * 4 * kS) == cudaSuccess;
  if (roles & LYRA_B200_ROLE_DECODER) ok = ok && DevAlloc(&ctx->d_mid_dec, (size_t)ctx->ntiles * 128 * 4 * kS) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_logmel_prev[0], P * 320) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_logmel_prev[1], P * 320) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_logmel_prev[2], P * 320) == cudaSuccess;
  {
    // NoiseEstimator::Create (lyra/noise_estimator.cc:99-120) for (16 kHz, hop 320, 160 features)
    const float secs_per_hop = static_cast<float>(320) / 16000;
    ctx->noise_params.nf = 160;
    ctx->noise_params.hops_per_update = (int)std::round(1.f / secs_per_hop);
    ctx->noise_params.max_smoothing = std::pow(0.5f, secs_per_hop / 0.7f);
    ctx->noise_params.bound_decay = std::pow(0.5f, secs_per_hop / 1.f);
    ctx->noise_params.log_nf = std::log((double)160);
  }
  ok = ok && DevAlloc(&ctx->d_noise, P * (size_t)NoiseStateUnits(160)) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_noise_est, P * 160) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_noise_enc, P * (size_t)NoiseStateUnits(160)) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_logmel_prev_enc, P * 320) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_plc, P * 4) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_cng_work, P * 1024) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_cng_hops, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_plan, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_skip, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_feed, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_is_cn, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_fade0, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_dir, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_model_pcm, P * 320) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_cng_pcm, P * 320) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_cng_feat, P * 160) == cudaSuccess;
  for (int d = 0; d < 2; ++d) {
    ok = ok && DevAlloc(&ctx->d_rs_delay[d], P * (size_t)(kResamplerTaps - 1)) == cudaSuccess;
    ok = ok && DevAlloc(&ctx->d_rs_pos[d], P * 2) == cudaSuccess;
  }
  ok = ok && DevAlloc(&ctx->d_rs_in, P * 960) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_rs_out, P * 968) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_rs_counts, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_is_noise, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_pcm, P * 320) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_packets, P * 24) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_received, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_features, P * 64) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_melout, P * 160) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_indices, P * 46) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_ids, P) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_tile_list, (size_t)ctx->ntiles) == cudaSuccess;
  ok = ok && DevAlloc(&ctx->d_slot_of, P) == cudaSuccess;
  for (int b = 0; b < 2 && ok; ++b) {
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&ctx->h_slot_of[b]), sizeof(int) * P) == cudaSuccess;
    ok = ok && cudaMallocHost(reinterpret_cast<void**>(&ctx->h_tile_list[b]), sizeof(int) * (size_t)ctx->ntiles) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&ctx->ev_map[b], cudaEventDisableTiming) == cudaSuccess;
    if (ok) for (size_t i = 0; i < P; ++i) ctx->h_slot_of[b][i] = -1;
  }
  if (ok) ok = kS == 16 ? SetSmemLimits<16>() : SetSmemLimits<8>();
  if (ok) ok = LYRA_SET_MAX_SMEM(DecoderKernelDW, DecDW::kSmemBytes) == 0;
  if (!ok) {
    g_create_error = std::string("CUDA allocation / setup failed: ") + cudaGetErrorString(cudaGetLastError());
    lyra_b200_destroy(ctx);
    return LYRA_B200_ENODEV;
  }
  if (ResetImpl(ctx, nullptr, max_streams) != LYRA_B200_OK) {
    g_create_error = ctx->err;
    lyra_b200_destroy(ctx);
    return LYRA_B200_ENODEV;
  }
  *out = ctx;
  return LYRA_B200_OK;
}

void lyra_b200_destroy(lyra_b200_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaFree(ctx->d_blob);
  for (int w = 0; w < 4; ++w) { cudaFree(ctx->d_state[w]); cudaFree(ctx->d_init[w]); cudaFree(ctx->d_n18[w]); }
  cudaFree(ctx->d_mid_enc); cudaFree(ctx->d_mid_dec);
  cudaFree(ctx->d_logmel_prev[0]); cudaFree(ctx->d_logmel_prev[1]); cudaFree(ctx->d_logmel_prev[2]);
  cudaFree(ctx->d_noise); cudaFree(ctx->d_noise_est); cudaFree(ctx->d_is_noise);
  cudaFree(ctx->d_noise_enc); cudaFree(ctx->d_logmel_prev_enc); cudaFree(ctx->d_plc); cudaFree(ctx->d_cng_work); cudaFree(ctx->d_cng_hops);
  cudaFree(ctx->d_plan); cudaFree(ctx->d_skip); cudaFree(ctx->d_feed); cudaFree(ctx->d_is_cn); cudaFree(ctx->d_fade0); cudaFree(ctx->d_dir);
  cudaFree(ctx->d_model_pcm); cudaFree(ctx->d_cng_pcm); cudaFree(ctx->d_cng_feat);
  for (int d = 0; d < 2; ++d) { cudaFree(ctx->d_rs_delay[d]); cudaFree(ctx->d_rs_pos[d]); }
  cudaFree(ctx->d_rs_in); cudaFree(ctx->d_rs_out); cudaFree(ctx->d_rs_counts);
  cudaFree(ctx->d_pcm); cudaFree(ctx->d_packets); cudaFree(ctx->d_received); cudaFree(ctx->d_features);
  cudaFree(ctx->d_melout); cudaFree(ctx->d_indices); cudaFree(ctx->d_ids); cudaFree(ctx->d_tile_list); cudaFree(ctx->d_slot_of);
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
int lyra_b200_tile_streams(const lyra_b200_ctx* ctx) { return ctx ? ctx->S : 0; }
uint64_t lyra_b200_launch_count(const lyra_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int lyra_b200_profile_enable(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  CU(SyncStream(ctx));
  ProfDrain(ctx);
  ctx->profiling = enable != 0;
  if (enable) for (int k = 0; k < LYRA_B200_NUM_KERNELS; ++k) { ctx->prof_ms[k] = 0.0; ctx->prof_n[k] = 0; }
  return LYRA_B200_OK;
}

int lyra_b200_profile_read(lyra_b200_ctx* ctx, double* ms_sum, uint64_t* launches) {
  if (!ctx || !ms_sum || !launches) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  CU(SyncStream(ctx));
  ProfDrain(ctx);
  for (int k = 0; k < LYRA_B200_NUM_KERNELS; ++k) { ms_sum[k] = ctx->prof_ms[k]; launches[k] = ctx->prof_n[k]; }
  return LYRA_B200_OK;
}

int lyra_b200_reset(lyra_b200_ctx* ctx, const int32_t* stream_ids, int n) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  return ResetImpl(ctx, stream_ids, n);
}

int lyra_b200_set_stream(lyra_b200_ctx* ctx, void* cuda_stream) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  ctx->stream = cuda_stream ? reinterpret_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
  return LYRA_B200_OK;
}

int lyra_b200_set_split(lyra_b200_ctx* ctx, int parts) {
  if (!ctx || parts < 1 || parts > lyra_b200_ctx::kMaxSplit) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  ctx->nsplit = parts;
  return LYRA_B200_OK;
}

int lyra_b200_set_blocking_sync(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  ctx->blocking_sync = enable != 0;
  return LYRA_B200_OK;
}

int lyra_b200_set_priority(lyra_b200_ctx* ctx, int priority) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
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
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  ctx->decoder_mode = mode;
  return LYRA_B200_OK;
}

int lyra_b200_decoder_mode(const lyra_b200_ctx* ctx) { return ctx ? ctx->decoder_mode : LYRA_B200_EINVAL; }

int lyra_b200_synchronize(lyra_b200_ctx* ctx) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_encode_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets) {
  if (!ctx || !d_pcm || !d_packets) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_ENCODER)) return LYRA_B200_EINVAL;
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, nullptr, n);
  if (rc) return rc;
  return RunEncode(ctx, n, d_pcm, num_bits, d_packets);
}

int lyra_b200_decode_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                            int16_t* d_pcm) {
  if (!ctx || !d_packets || !d_pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_DECODER)) return LYRA_B200_EINVAL;
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, nullptr, n);
  if (rc) return rc;
  return RunDecode(ctx, n, d_packets, d_received, num_bits, d_pcm);
}

int lyra_b200_set_graphs(lyra_b200_ctx* ctx, int enable) {
  if (!ctx) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
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
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_ENCODER)) return LYRA_B200_EINVAL;
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, ids, n);
  if (rc) return rc;
  const lyra_b200_ctx::GraphKey key{0, n, num_bits, 0, ctx->nsplit, pcm, packets, nullptr};
  if ((rc = RunMaybeGraphed(ctx, key, ids == nullptr && ctx->map_dense_n == n,
                            [&]() { return RunEncode(ctx, n, ctx->d_pcm, num_bits, ctx->d_packets, pcm, packets); })))
    return rc;
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_decode(lyra_b200_ctx* ctx, const int32_t* ids, int n, const uint8_t* packets, const uint8_t* received,
                     int num_bits, int16_t* pcm) {
  if (!ctx || !packets || !pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_DECODER)) return LYRA_B200_EINVAL;
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, ids, n);
  if (rc) return rc;
  const lyra_b200_ctx::GraphKey key{1, n, num_bits, ctx->decoder_mode, ctx->nsplit, packets, received, pcm};
  if ((rc = RunMaybeGraphed(ctx, key, ids == nullptr && ctx->map_dense_n == n, [&]() {
         return RunDecode(ctx, n, ctx->d_packets, received ? ctx->d_received : nullptr, num_bits, ctx->d_pcm, packets, received, pcm);
       })))
    return rc;
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_extract_features(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, float* features) {
  if (!ctx || !pcm || !features) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_ENCODER)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, ids, n);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_pcm, pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchEncoderNets(ctx, WholeCall(ctx, n), ctx->d_pcm, ctx->d_features))) return rc;
  CU(cudaMemcpyAsync(features, ctx->d_features, sizeof(float) * 64 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_quantize(lyra_b200_ctx* ctx, int n, const float* features, int num_bits, uint8_t* packets, int32_t* indices) {
  if (!ctx || !features || !packets) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "count out of range"; return LYRA_B200_EINVAL; }
  CU(cudaMemcpyAsync(ctx->d_features, features, sizeof(float) * 64 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  const Part whole{0, 0, 0, n, ctx->stream};
  int rc = LaunchQuantize(ctx, whole, ctx->d_features, num_bits, ctx->d_packets, indices ? ctx->d_indices : nullptr);
  if (rc) return rc;
  CU(cudaMemcpyAsync(packets, ctx->d_packets, (size_t)PacketBytes(num_bits) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if (indices) CU(cudaMemcpyAsync(indices, ctx->d_indices, sizeof(int) * 46 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_dequantize(lyra_b200_ctx* ctx, int n, const uint8_t* packets, int num_bits, float* features) {
  if (!ctx || !features || !packets) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "count out of range"; return LYRA_B200_EINVAL; }
  CU(cudaMemcpyAsync(ctx->d_packets, packets, (size_t)PacketBytes(num_bits) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  const Part whole{0, 0, 0, n, ctx->stream};
  int rc = LaunchDequantize(ctx, whole, ctx->d_packets, nullptr, num_bits, ctx->d_features);
  if (rc) return rc;
  CU(cudaMemcpyAsync(features, ctx->d_features, sizeof(float) * 64 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_generate(lyra_b200_ctx* ctx, const int32_t* ids, int n, const float* features, int16_t* pcm) {
  if (!ctx || !features || !pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_DECODER)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, ids, n);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_features, features, sizeof(float) * 64 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = LaunchDecoderNets(ctx, WholeCall(ctx, n), ctx->d_features, ctx->d_pcm))) return rc;
  CU(cudaMemcpyAsync(pcm, ctx->d_pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_logmel(lyra_b200_ctx* ctx, int bank, const int32_t* ids, int n, const int16_t* pcm, int num_mel_bins, float* out) {
  if (!ctx || !pcm || !out) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (bank < 0 || bank > 1) { ctx->err = "log-mel bank must be 0 or 1"; return LYRA_B200_EINVAL; }
  if (num_mel_bins != 160 && num_mel_bins != 64) { ctx->err = "log-mel supports 160 or 64 mel bins"; return LYRA_B200_EINVAL; }
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  const int* d_ids = nullptr;
  if (ids) {
    std::vector<char> seen((size_t)ctx->max_streams, 0);
    for (int k = 0; k < n; ++k) {
      if (ids[k] < 0 || ids[k] >= ctx->max_streams || seen[(size_t)ids[k]]) { ctx->err = "bad or duplicate stream id"; return LYRA_B200_EINVAL; }
      seen[(size_t)ids[k]] = 1;
    }
    CU(cudaMemcpyAsync(ctx->d_ids, ids, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    d_ids = ctx->d_ids;
  }
  const LogMelParams& P = num_mel_bins == 160 ? ctx->spec.logmel160 : ctx->spec.logmel64;
  CU(cudaMemcpyAsync(ctx->d_pcm, pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  const size_t smem = sizeof(double) * (size_t)(2 * kLogMelFftPadded + P.fft / 2 + 1 + P.window_len + P.window_len / 8 + 1);
  { ProfScope ps(ctx, 6, ctx->stream);
  LYRA_LAUNCH(LogMelKernel, dim3((unsigned)n), dim3(kLogMelThreads), smem, ctx->stream,
              ctx->d_blob, P, d_ids, n, ctx->d_pcm, ctx->d_logmel_prev[bank], ctx->d_melout, (const uint8_t*)nullptr, 0); }
  ctx->launches += 1;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, ctx->d_melout, sizeof(float) * (size_t)num_mel_bins * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_noise_update(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, const uint8_t* update_mask,
                           uint8_t* is_noise, float* noise_estimate) {
  if (!ctx || !pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  const int* d_ids = nullptr;
  if (ids) {
    std::vector<char> seen((size_t)ctx->max_streams, 0);
    for (int k = 0; k < n; ++k) {
      if (ids[k] < 0 || ids[k] >= ctx->max_streams || seen[(size_t)ids[k]]) { ctx->err = "bad or duplicate stream id"; return LYRA_B200_EINVAL; }
      seen[(size_t)ids[k]] = 1;
    }
    CU(cudaMemcpyAsync(ctx->d_ids, ids, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    d_ids = ctx->d_ids;
  }
  CU(cudaMemcpyAsync(ctx->d_pcm, pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if (update_mask) CU(cudaMemcpyAsync(ctx->d_received, update_mask, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  int rc = LaunchNoiseUpdate(ctx, ctx->stream, d_ids, 0, n, n, ctx->d_pcm, update_mask ? ctx->d_received : nullptr,
                             is_noise ? ctx->d_is_noise : nullptr, noise_estimate ? ctx->d_noise_est : nullptr);
  if (rc) return rc;
  if (is_noise) CU(cudaMemcpyAsync(is_noise, ctx->d_is_noise, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if (noise_estimate) CU(cudaMemcpyAsync(noise_estimate, ctx->d_noise_est, sizeof(float) * 160 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_noise_update_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, const uint8_t* d_update_mask,
                                  uint8_t* d_is_noise, float* d_noise_estimate) {
  if (!ctx || !d_pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_DECODER)) return LYRA_B200_EINVAL;
  if (n <= 0 || n > ctx->max_streams) { ctx->err = "stream count out of range"; return LYRA_B200_EINVAL; }
  return LaunchNoiseUpdate(ctx, ctx->stream, nullptr, 0, n, n, d_pcm, d_update_mask, d_is_noise, d_noise_estimate);
}

int lyra_b200_decode_track_noise(lyra_b200_ctx* ctx, const int32_t* ids, int n, const uint8_t* packets, const uint8_t* received,
                                 int num_bits, int16_t* pcm, uint8_t* is_noise) {
  if (!ctx || !packets || !pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_DECODER)) return LYRA_B200_EINVAL;
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, ids, n);
  if (rc) return rc;
  const int* d_ids = nullptr;
  if (ids) {
    CU(cudaMemcpyAsync(ctx->d_ids, ids, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    d_ids = ctx->d_ids;
  }
  if ((rc = RunDecode(ctx, n, ctx->d_packets, received ? ctx->d_received : nullptr, num_bits, ctx->d_pcm, packets, received, pcm,
                      true, d_ids, ctx->d_is_noise, is_noise))) return rc;
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_decode_track_noise_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                                        int16_t* d_pcm, uint8_t* d_is_noise) {
  if (!ctx || !d_packets || !d_pcm) return LYRA_B200_EINVAL;
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }   // the current device is per host thread
  if (!RoleOk(ctx, LYRA_B200_ROLE_DECODER)) return LYRA_B200_EINVAL;
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, nullptr, n);
  if (rc) return rc;
  return RunDecode(ctx, n, d_packets, d_received, num_bits, d_pcm, nullptr, nullptr, nullptr, true, nullptr,
                   d_is_noise ? d_is_noise : ctx->d_is_noise, nullptr);
}

#define ENTER(role)                                                                                          \
  if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return LYRA_B200_ENODEV; }    \
  if ((role) && !RoleOk(ctx, (role))) return LYRA_B200_EINVAL;

int lyra_b200_encode_dtx(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int16_t* pcm, int num_bits, uint8_t* packets,
                         int32_t* packet_bytes) {
  if (!ctx || !pcm || !packets || !packet_bytes) return LYRA_B200_EINVAL;
  ENTER(LYRA_B200_ROLE_ENCODER);
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int rc = UploadIds(ctx, ids, n, &d_ids);
  if (rc) return rc;
  if ((rc = PrepareMap(ctx, ids, n))) return rc;
  std::vector<uint8_t> flags((size_t)n);
  if ((rc = RunEncode(ctx, n, ctx->d_pcm, num_bits, ctx->d_packets, pcm, packets, true, d_ids, ctx->d_is_noise, flags.data()))) return rc;
  CU(SyncStream(ctx));
  for (int k = 0; k < n; ++k) packet_bytes[k] = flags[(size_t)k] ? 0 : PacketBytes(num_bits);
  return LYRA_B200_OK;
}

int lyra_b200_encode_dtx_device(lyra_b200_ctx* ctx, int n, const int16_t* d_pcm, int num_bits, uint8_t* d_packets, uint8_t* d_is_noise) {
  if (!ctx || !d_pcm || !d_packets || !d_is_noise) return LYRA_B200_EINVAL;
  ENTER(LYRA_B200_ROLE_ENCODER);
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, nullptr, n);
  if (rc) return rc;
  return RunEncode(ctx, n, d_pcm, num_bits, d_packets, nullptr, nullptr, true, nullptr, d_is_noise, nullptr);
}

int lyra_b200_decode_plc(lyra_b200_ctx* ctx, const int32_t* ids, int n, const uint8_t* packets, const uint8_t* received, int num_bits,
                         int16_t* pcm, uint8_t* is_comfort_noise) {
  if (!ctx || !packets || !pcm) return LYRA_B200_EINVAL;
  ENTER(LYRA_B200_ROLE_DECODER);
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  const int* d_ids = nullptr;
  int rc = UploadIds(ctx, ids, n, &d_ids);
  if (rc) return rc;
  if ((rc = PrepareMap(ctx, ids, n))) return rc;
  if ((rc = RunDecodePlc(ctx, n, ctx->d_packets, received ? ctx->d_received : nullptr, num_bits, ctx->d_pcm, d_ids, ctx->d_is_cn, packets,
                         received, pcm, is_comfort_noise))) return rc;
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_decode_plc_device(lyra_b200_ctx* ctx, int n, const uint8_t* d_packets, const uint8_t* d_received, int num_bits,
                                int16_t* d_pcm, uint8_t* d_is_comfort_noise) {
  if (!ctx || !d_packets || !d_pcm) return LYRA_B200_EINVAL;
  ENTER(LYRA_B200_ROLE_DECODER);
  if (!BitsOk(ctx, num_bits)) return LYRA_B200_EINVAL;
  int rc = PrepareMap(ctx, nullptr, n);
  if (rc) return rc;
  return RunDecodePlc(ctx, n, d_packets, d_received, num_bits, d_pcm, nullptr, d_is_comfort_noise ? d_is_comfort_noise : ctx->d_is_cn,
                      nullptr, nullptr, nullptr, nullptr);
}

int lyra_b200_plc_get_state(lyra_b200_ctx* ctx, const int32_t* ids, int n, int32_t* state) {
  if (!ctx || !state || n <= 0 || n > ctx->max_streams) return LYRA_B200_EINVAL;
  ENTER(0);
  CU(SyncStream(ctx));
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    if (id < 0 || id >= ctx->max_streams) { ctx->err = "stream id out of range"; return LYRA_B200_EINVAL; }
    CU(cudaMemcpy(state + (size_t)k * 3, ctx->d_plc + (size_t)id * 4, sizeof(int) * 3, cudaMemcpyDeviceToHost));
  }
  return LYRA_B200_OK;
}

int lyra_b200_plc_set_state(lyra_b200_ctx* ctx, const int32_t* ids, int n, const int32_t* state) {
  if (!ctx || !state || n <= 0 || n > ctx->max_streams) return LYRA_B200_EINVAL;
  ENTER(0);
  CU(SyncStream(ctx));
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    if (id < 0 || id >= ctx->max_streams) { ctx->err = "stream id out of range"; return LYRA_B200_EINVAL; }
    const int32_t* s3 = state + (size_t)k * 3;
    if (s3[0] < 0 || s3[0] > kPlcConcealSamples || s3[0] % 320 || s3[1] < 0 || s3[1] > kPlcFadeSamples || s3[1] % 320 || (s3[2] != 1 && s3[2] != -1)) {
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
  ENTER(0);
  const int* d_ids = nullptr;
  int rc = UploadIds(ctx, ids, n, &d_ids);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_cng_feat, features, sizeof(float) * 160 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  const size_t cng_smem = sizeof(double) * (size_t)(4 * kLogMelFftPadded + 160);
  LYRA_LAUNCH(ComfortNoiseKernel, dim3((unsigned)n), dim3(kCngThreads), cng_smem, ctx->stream,
              ctx->d_blob, ctx->spec.cng, d_ids, n, ctx->d_cng_feat, ctx->d_noise, NoiseStateUnits(ctx->noise_params.nf),
              (const uint8_t*)nullptr, ctx->d_cng_work, ctx->d_cng_hops, ctx->cng_seed, ctx->d_cng_pcm, 0);
  ctx->launches += 1;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(pcm, ctx->d_cng_pcm, sizeof(int16_t) * 320 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

int lyra_b200_resample(lyra_b200_ctx* ctx, int to_internal, const int32_t* ids, int n, int external_rate_hz, const int16_t* in,
                       int in_samples, int16_t* out, int out_stride, int32_t* out_counts) {
  if (!ctx || !in || !out) return LYRA_B200_EINVAL;
  ENTER(0);
  const int pair = external_rate_hz == 8000 ? 0 : external_rate_hz == 32000 ? 1 : external_rate_hz == 48000 ? 2 : -1;
  if (pair < 0) { ctx->err = "the resampler converts between 16 kHz and 8 / 32 / 48 kHz"; return LYRA_B200_EINVAL; }
  const int pr = to_internal ? pair : pair + 3;
  const int num = ctx->spec.resampler.num[pr], den = ctx->spec.resampler.den[pr];
  const int max_out = (in_samples * den + num - 1) / num;
  if (in_samples <= 0 || in_samples > 960 || max_out > 960 || out_stride < max_out || out_stride > 968) {
    ctx->err = "resample: at most 960 input and 960 output samples per stream and call, and room for ceil(n * out / in) outputs";
    return LYRA_B200_EINVAL;
  }
  const int* d_ids = nullptr;
  int rc = UploadIds(ctx, ids, n, &d_ids);
  if (rc) return rc;
  CU(cudaMemcpyAsync(ctx->d_rs_in, in, sizeof(int16_t) * (size_t)in_samples * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  const int dir = to_internal ? 0 : 1;
  LYRA_LAUNCH(ResampleKernel, dim3((unsigned)n), dim3(128), sizeof(float) * (size_t)(kResamplerTaps - 1 + in_samples), ctx->stream,
              ctx->d_blob, ctx->spec.resampler, pr, external_rate_hz, d_ids, n, ctx->d_rs_in, in_samples, ctx->d_rs_out, out_stride,
              ctx->d_rs_counts, ctx->d_rs_delay[dir], ctx->d_rs_pos[dir]);
  ctx->launches += 1;
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(out, ctx->d_rs_out, sizeof(int16_t) * (size_t)out_stride * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<int> counts((size_t)n);
  CU(cudaMemcpyAsync(counts.data(), ctx->d_rs_counts, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  if (out_counts) for (int k = 0; k < n; ++k) out_counts[k] = counts[(size_t)k];
  return LYRA_B200_OK;
}

int lyra_b200_noise_estimate(lyra_b200_ctx* ctx, const int32_t* ids, int n, float* noise_estimate, uint8_t* is_noise) {
  if (!ctx || (!noise_estimate && !is_noise)) return LYRA_B200_EINVAL;
  ENTER(0);
  const int* d_ids = nullptr;
  int rc = UploadIds(ctx, ids, n, &d_ids);
  if (rc) return rc;
  LYRA_LAUNCH(NoiseReadKernel, dim3((unsigned)n), dim3(192), (size_t)0, ctx->stream,
              d_ids, n, ctx->d_noise, ctx->noise_params.nf, noise_estimate ? ctx->d_noise_est : nullptr, is_noise ? ctx->d_is_noise : nullptr);
  ctx->launches += 1;
  CU(cudaGetLastError());
  if (noise_estimate) CU(cudaMemcpyAsync(noise_estimate, ctx->d_noise_est, sizeof(float) * 160 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  if (is_noise) CU(cudaMemcpyAsync(is_noise, ctx->d_is_noise, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CU(SyncStream(ctx));
  return LYRA_B200_OK;
}

}  // extern "C"
