// The conv-net kernels of the per-frame hot path, one thread block per tile of S streams.
//
//   EncoderKernelA  first_layer .. encoder_0/simpleconv          (T = 20 rows, 64 ch)   -> mid [128][4][S]
//   EncoderKernelB  encoder_1 .. quant_bottleneck_1               (T = 4/2/1)            -> features f32[64]
//   DecoderKernelC  bottleneck_2 .. decoder_1                      (T = 1/2/4)            -> mid [128][4][S]
//   DecoderKernelD  decoder_2/simple .. last_layer                 (T = 20 rows, 64 ch)   -> int16 PCM
//
// Together A+B replace SoundStreamEncoder::Extract's Interpreter::Invoke (lyra/soundstream_encoder.cc:53-64)
// and C+D replace LyraGanModel::RunConditioning/RunModel (lyra/lyra_gan_model.cc:53-64) for S streams at once.
// Streaming state (TFLite resource variables in the reference) lives in HBM, tile-blocked
// [tile][unit][S]; dilated depthwise convs keep a ring of their last 2*dilation input rows.
#pragma once

#include <type_traits>

#include "kernel_prims.cuh"

// resident blocks per SM the small-M kernels (B, C) are compiled for at S = 8 (their 59-72 KB of shared memory allow 3)
#ifndef LYRA_BC_MIN_BLOCKS
#define LYRA_BC_MIN_BLOCKS 3
#endif
// output channels per fp32 thread tile in the small-M layers of kernels B / C (8 streams x LYRA_BC_TN channels)
#ifndef LYRA_B_MIN_BLOCKS
#define LYRA_B_MIN_BLOCKS LYRA_BC_MIN_BLOCKS
#endif
#ifndef LYRA_C_MIN_BLOCKS
#define LYRA_C_MIN_BLOCKS LYRA_BC_MIN_BLOCKS
#endif
#ifndef LYRA_BC_STAGES
#define LYRA_BC_STAGES 3
#endif
#ifndef LYRA_B_DEEP_RINGS
#define LYRA_B_DEEP_RINGS 0
#endif
#ifndef LYRA_BC_TN
#define LYRA_BC_TN 4
#endif

namespace lyra_b200 {

// Development aid (-DLYRA_PHASE_PROF): thread 0 of every block stamps clock64() at phase boundaries.
#if defined(LYRA_PHASE_PROF) && !defined(LYRA_EMU)
__device__ long long* g_phase_prof = nullptr;
#define LYRA_PHASE(k, ph) do { if (threadIdx.x == 0 && g_phase_prof && blockIdx.x < 1024) g_phase_prof[((size_t)(k) * 1024 + blockIdx.x) * 48 + (ph)] = clock64(); ++(ph); } while (0)
#else
#define LYRA_PHASE(k, ph) do { (void)(ph); } while (0)
#endif

// ---- per-tile state layouts, in 4-byte units (each unit is S lanes wide) ----
struct EncStateA {
  static constexpr int kFirst = 0;                               // [48]
  static constexpr int kRing0 = 48, kRing1 = kRing0 + 64 * 2, kRing2 = kRing1 + 64 * 6;   // [64][2|6|18]
  static constexpr int kDown0 = kRing2 + 64 * 18;                // [64][5]
  static constexpr int kUnits = kDown0 + 64 * 5;                 // 2032
};
struct EncStateB {
  static constexpr int kRing0 = 0, kRing1 = 128 * 2, kRing2 = kRing1 + 128 * 6;           // f32 [128][2|6|18]
  static constexpr int kDown1 = kRing2 + 128 * 18;               // f32 [128][2]
  static constexpr int kRingM = kDown1 + 128 * 2;                // f32 [256][2]
  static constexpr int kRingQ0 = kRingM + 256 * 2;               // words [64][6]
  static constexpr int kRingQ1 = kRingQ0 + 64 * 6;               // words [64][18]
  static constexpr int kDown2 = kRingQ1 + 64 * 18;               // words [64][2]
  static constexpr int kBott = kDown2 + 64 * 2;                  // words [128][2]
  static constexpr int kUnits = kBott + 128 * 2;                 // 6016
};
struct DecStateC {
  static constexpr int kBott = 0;                                // f32 [64][2]
  static constexpr int kUp0 = 128;                               // f32 [256][2]
  static constexpr int kUp1 = kUp0 + 512;                        // f32 [128][2]
  static constexpr int kRing0 = kUp1 + 256, kRing1 = kRing0 + 128 * 2, kRing2 = kRing1 + 128 * 6;  // f32 [128][2|6|18]
  static constexpr int kRingM = kRing2 + 128 * 18;               // words [64][2]
  static constexpr int kRingQ0 = kRingM + 64 * 2;                // words [64][6]
  static constexpr int kRingQ1 = kRingQ0 + 64 * 6;               // words [64][18]
  static constexpr int kUnits = kRingQ1 + 64 * 18;               // 5888
};
struct DecStateD {
  static constexpr int kUp2 = 0;                                 // f32 [64][5]
  static constexpr int kRing0 = 320, kRing1 = kRing0 + 64 * 2, kRing2 = kRing1 + 64 * 6;  // f32 [64][2|6|18]
  static constexpr int kLast = kRing2 + 64 * 18;                 // f32 [48]
  static constexpr int kUnits = kLast + 48;                      // 2032
};

struct TileIo {
  const int* tile_list;        // tiles to process, one per block
  const int* slot_of_stream;   // [max_streams] position of the stream in this call's I/O arrays, -1 = not in this call
  const uint8_t* skip;         // optional, by slot: 1 = the stream sits this call out (its state does not advance): DTX noise
                               // hops on the encoder side, pure comfort-noise hops on the decoder side
};

// Per-tile metadata in shared memory: slot[S], active[S], n18[S] and n18[S] = the frame counter shared by all
// active streams of the tile (-1 if they differ, which selects the general ring path; -2 if the tile has no active stream at
// all in this call - every stream skipped - in which case the kernels return at once: kTileIdle).
template <int S>
__device__ __forceinline__ void LoadTileMeta(const TileIo& io, const int* n18_global, int* slot, int* active, int* n18, int& tile) {
  tile = io.tile_list[blockIdx.x];
  if ((int)threadIdx.x < S) {
    const int stream = tile * S + (int)threadIdx.x;
    const int sl = io.slot_of_stream[stream];
    slot[threadIdx.x] = sl;
    active[threadIdx.x] = sl >= 0 && !(io.skip != nullptr && io.skip[sl]);
    n18[threadIdx.x] = n18_global[stream];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int u = -2;
    for (int s = 0; s < S; ++s)
      if (active[s]) u = (u == -2 || u == n18[s]) ? n18[s] : -1;
    n18[S] = u;
  }
  __syncthreads();
}
constexpr int kTileIdle = -2;

// The tile's streaming state (one contiguous block per kernel, 65-190 KB; the 262 MB working set of 4096 streams does not stay
// in the 50 MB L2 between hops) is requested into the L2 as soon as the block knows its tile: the ring / tail loads of the
// later phases then find it there instead of paying the HBM latency phase by phase.
#ifndef LYRA_PREFETCH_STATE
#define LYRA_PREFETCH_STATE 1
#endif
template <int ON>
__device__ __forceinline__ void PrefetchTileState(const void* p, int bytes) {
  if (ON && threadIdx.x == 0) lyra_prefetch_l2(p, (unsigned)bytes);
}

// One fp32 residual unit:  d = dw(lrelu(u)); h = lrelu(pw1(d)); u' = pw2(h) + u.
// u lives at row offset row0u of a [C][ldu] buffer; d is a [C][LDD] scratch.  When `last`, lrelu(u') is stored.
// TC (decoder tensor-core mode): the two 1x1 convolutions run as split-precision TF32 MMAs with warp tiles of
// WTM x WTN fragments (sized so that every warp owns at most one tile: pw1 rewrites its operand in place); the weight
// ring and its prefetch chain are not used in that mode.
template <int S, int NT, int TM, int TN1, int TN2, int WM, int KC, int C, int T, int DIL, bool TC = false, int LDD = T * S,
          int WTM = 1, int WTN = 1, int STG = kStages>
__device__ __forceinline__ void ResUnitF32(const uint8_t* blob, const ResF32& p, float* u, int ldu, int row0u, float* d,
                                           int groups2, float* ring, const int* n18,
                                           const int* active, float* wbuf, bool last, const WNext& after, int pk, int& ph,
                                           int dil_rt = DIL) {
  constexpr int ldd = LDD;
  // pw1's weight stream is started by whoever ran before this unit (previous GEMM or the kernel prologue)
  if (n18[S] >= 0) {
    auto dw = [&](auto dil) {
      DwF32RingFast<S, NT, C, T, decltype(dil)::value>(u, ldu, row0u, d, ldd, BlobPtr<float>(blob, p.dw.w), BlobPtr<float>(blob, p.dw.bias), ring, n18[S], active);
    };
    if constexpr (DIL != 0) dw(std::integral_constant<int, DIL>());
    else if (dil_rt == 1) dw(std::integral_constant<int, 1>());
    else if (dil_rt == 3) dw(std::integral_constant<int, 3>());
    else dw(std::integral_constant<int, 9>());
  } else {
    DwF32Ring<S, NT>(u, ldu, row0u, d, ldd, C, T, dil_rt, BlobPtr<float>(blob, p.dw.w), BlobPtr<float>(blob, p.dw.bias), ring, n18, active);
  }
  LYRA_PHASE(pk, ph);
  {
    const float* b1 = BlobPtr<float>(blob, p.pw1.bias);
    auto epi1 = [&](int t, int s0, int n0, auto& acc) {
      constexpr int TMx = sizeof(acc) / sizeof(acc[0]), TNx = sizeof(acc[0]) / sizeof(float);
#pragma unroll
      for (int j = 0; j < TNx; ++j) {
        const float b = b1[n0 + j];
        float* o = d + (size_t)(n0 + j) * ldd + t * S + s0;
#pragma unroll
        for (int i = 0; i < TMx; ++i) o[i] = LeakyRelu(__fadd_rn(acc[i][j], b));
      }
    };
    if constexpr (TC)
      GemmTf32Mma<S, NT, WTM, WTN, true>(d, ldd, 0, 1, 1, C, 1, T, C, BlobPtr<float2>(blob, p.pw1.wf), epi1);
    else
      GemmF32Tap<S, NT, TM, TN1, KC, WM, false, STG>(d, ldd, 0, 1, 1, C, 1, T, C, BlobPtr<float>(blob, p.pw1.w), wbuf, true,
                                                     NextF32(BlobPtr<float>(blob, p.pw2.w), KC, C, C / groups2, nullptr, STG), epi1);
  }
  LYRA_PHASE(pk, ph);
  {
    const float* b2 = BlobPtr<float>(blob, p.pw2.bias);
    auto epi2 = [&](int t, int s0, int n0, auto& acc) {
      constexpr int TMx = sizeof(acc) / sizeof(acc[0]), TNx = sizeof(acc[0]) / sizeof(float);
#pragma unroll
      for (int j = 0; j < TNx; ++j) {
        const float b = b2[n0 + j];
        float* o = u + (size_t)(n0 + j) * ldu + (row0u + t) * S + s0;
#pragma unroll
        for (int i = 0; i < TMx; ++i) {
          const float v = __fadd_rn(__fadd_rn(acc[i][j], b), o[i]);
          o[i] = last ? LeakyRelu(v) : v;
        }
      }
    };
    if constexpr (TC)
      GemmTf32Mma<S, NT, WTM, WTN, false>(d, ldd, 0, 1, 1, C / groups2, groups2, T, C, BlobPtr<float2>(blob, p.pw2.wf), epi2);
    else
      GemmF32Tap<S, NT, TM, TN2, KC, WM, false, STG>(d, ldd, 0, 1, 1, C / groups2, groups2, T, C, BlobPtr<float>(blob, p.pw2.w), wbuf, true, after, epi2);
  }
  LYRA_PHASE(pk, ph);
}

// The three residual units of one stage (dilation 1, 3, 9; ring blocks of 2, 6, 18 rows back to back) as ONE copy of the code in
// a loop that is not unrolled: the units differ only in their parameters and in the depthwise pass, and three inlined copies
// of the two GEMMs made kernels B / C overflow the instruction cache (15-20 % of their stall samples were instruction fetches).
template <int S, int NT, int TM, int TN1, int TN2, int WM, int KC, int C, int T, bool TC = false, int LDD = T * S, int WTM = 1, int WTN = 1,
          int STG = kStages>
__device__ __forceinline__ void ResUnitsF32x3(const uint8_t* blob, const ResF32* p3, float* u, int ldu, int row0u, float* d, int groups2,
                                              float* ring0, const int* n18, const int* active, float* wbuf, const WNext& after,
                                              int pk, int& ph) {
#pragma unroll 1
  for (int i = 0; i < 3; ++i) {
    const ResF32& p = p3[i];
    const int dil = i == 0 ? 1 : (i == 1 ? 3 : 9);
    float* ring = ring0 + (size_t)(i == 0 ? 0 : (i == 1 ? 2 : 8)) * C * S;       // [C][2] | [C][6] | [C][18]
    const WNext nx = i < 2 ? NextF32(BlobPtr<float>(blob, p3[i + 1].pw1.w), KC, C, C, nullptr, STG) : after;
    ResUnitF32<S, NT, TM, TN1, TN2, WM, KC, C, T, 0, TC, LDD, WTM, WTN, STG>(blob, p, u, ldu, row0u, d, groups2, ring, n18, active, wbuf, i == 2, nx,
                                                                       pk, ph, dil);
  }
}

// One int8 residual unit on packed activations (quant_encoder_2/resnet_{1,2}, quant_decoder_0/resnet_{1,2}); the two
// 1x1 convolutions run on the tensor cores.
//   aq: LeakyReLU'd input (row offset row0a of [64][lda]); resq: the pre-activation residual; both updated in place.
template <int S, int NT, int DIL, int PDI = LYRA_I8_PD>
__device__ __forceinline__ void ResUnitI8(const uint8_t* blob, const ResI8& p, uint32_t* aq, int lda, int row0a,
                                          uint32_t* resq, uint32_t* dq8, uint32_t* hq, uint32_t* ring,
                                          const int* n18, const int* active, int pk, int& ph, int dil_rt = DIL) {
  constexpr int T = 2, C = 256, LD = PadLd(T * S);
  constexpr int NTW = S >= 16 ? 8 : 4;
  if (n18[S] >= 0) {
    if constexpr (DIL != 0) DwI8RingFast<S, NT, C, T, DIL>(aq, lda, row0a, dq8, LD, blob, p.dw, ring, n18[S], active);
    else if (dil_rt == 3) DwI8RingFast<S, NT, C, T, 3>(aq, lda, row0a, dq8, LD, blob, p.dw, ring, n18[S], active);
    else DwI8RingFast<S, NT, C, T, 9>(aq, lda, row0a, dq8, LD, blob, p.dw, ring, n18[S], active);
  } else {
    DwI8Ring<S, NT>(aq, lda, row0a, dq8, LD, C, T, dil_rt, blob, p.dw, ring, n18, active);
  }
  LYRA_PHASE(pk, ph);
  {
    const int* bias = BlobPtr<int>(blob, p.pw1.bias);
    const int* mult = BlobPtr<int>(blob, p.pw1.mult);
    const int* shift = BlobPtr<int>(blob, p.pw1.shift);
    const int8_t* lut = BlobPtr<int8_t>(blob, p.lr1.lut);
    const int out_zp = p.pw1.out_zp;
    GemmI8Mma<S, NT, NTW, PDI>(dq8, LD, 0, 1, 1, C, 1, T, C, BlobPtr<uint2>(blob, p.pw1.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        int q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) q[j] = lut[RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp) + 128];
        hq[(size_t)(n0 / 4) * LD + t * S + s] = PackI8x4(q[0], q[1], q[2], q[3]);
      });
  }
  LYRA_PHASE(pk, ph);
  {
    const int* bias = BlobPtr<int>(blob, p.pw2.bias);
    const int* mult = BlobPtr<int>(blob, p.pw2.mult);
    const int* shift = BlobPtr<int>(blob, p.pw2.shift);
    const int* l1 = BlobPtr<int>(blob, p.add.lut1);
    const int* l2 = BlobPtr<int>(blob, p.add.lut2);
    const int8_t* lut = BlobPtr<int8_t>(blob, p.lr2.lut);
    const int out_zp = p.pw2.out_zp, m3 = p.add.m3, s3 = p.add.s3, add_zp = p.add.out_zp;
    GemmI8Mma<S, NT, NTW, PDI>(hq, LD, 0, 1, 1, C / 4, 4, T, C, BlobPtr<uint2>(blob, p.pw2.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        const size_t ro = (size_t)(n0 / 4) * LD + t * S + s;
        const uint32_t rw = resq[ro];
        int r[4], a[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int q = RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp);
          r[j] = ClampI8(Mbqm(l1[q + 128] + l2[UnpackI8(rw, j) + 128], m3, s3) + add_zp);
          a[j] = lut[r[j] + 128];
        }
        resq[ro] = PackI8x4(r[0], r[1], r[2], r[3]);
        aq[(size_t)(n0 / 4) * lda + (row0a + t) * S + s] = PackI8x4(a[0], a[1], a[2], a[3]);
      });
  }
  LYRA_PHASE(pk, ph);
}

// quant_{en,de}coder resnet_1 and resnet_2 (dilation 3, 9; ring blocks of 6 and 18 rows back to back) as one copy of the code
template <int S, int NT, int PDI = LYRA_I8_PD>
__device__ __forceinline__ void ResUnitsI8x2(const uint8_t* blob, const ResI8* p2, uint32_t* aq, int lda, int row0a,
                                             uint32_t* resq, uint32_t* dq8, uint32_t* hq, uint32_t* ring0,
                                             const int* n18, const int* active, int pk, int& ph) {
#pragma unroll 1
  for (int i = 0; i < 2; ++i)
    ResUnitI8<S, NT, 0, PDI>(blob, p2[i], aq, lda, row0a, resq, dq8, hq, ring0 + (size_t)(i ? 64 * 6 : 0) * S, n18, active, pk, ph, i ? 9 : 3);
}

// ================================================================================================
//                                        ENCODER  A
// ================================================================================================
#ifndef LYRA_A_TN
#define LYRA_A_TN 4
#endif
#ifndef LYRA_A_NT
#define LYRA_A_NT 320
#endif
#ifndef LYRA_A_DOWN_STAGES
#define LYRA_A_DOWN_STAGES 5
#endif
#ifndef LYRA_A_DOWN_TM
#define LYRA_A_DOWN_TM 8
#endif
#ifndef LYRA_A_DOWN_TN
#define LYRA_A_DOWN_TN 4
#endif
template <int S>
struct EncA {
  static constexpr int NT = LYRA_A_NT;
  static constexpr int TN = S >= 16 ? 8 : LYRA_A_TN;
  static constexpr int kMinBlocks = S <= 8 ? 2 : 1;       // S = 8 tiles fit two blocks per SM
  static constexpr int LDU = 25 * S, LDD = 20 * S;
  static constexpr int kStgDown = S <= 8 ? LYRA_A_DOWN_STAGES : kStages;   // ring depth of encoder_0/simpleconv (ring = the d buffer)
  static constexpr int kSmemU = 0;
  static constexpr int kSmemD = kSmemU + 64 * LDU * 4;
  static constexpr int kSmemW = kSmemD + 64 * LDD * 4;
  static constexpr int kSmemI = kSmemW + kStages * 16 * 64 * 4;   // ring of the 64-channel layers (simpleconv's ring lives in d)
  static constexpr int kSmemBytes = kSmemI + 3 * S * 4 + 16;
  static_assert(391 * S <= 64 * LDD, "first-layer input (368 rows + 23 skew rows) must fit in the d buffer");
};

template <int S>
__global__ void __launch_bounds__(EncA<S>::NT, EncA<S>::kMinBlocks)
EncoderKernelA(const uint8_t* __restrict__ blob, EncoderParams P, TileIo io, const int16_t* __restrict__ pcm,
               float* __restrict__ state, int* __restrict__ n18g, float* __restrict__ mid) {
  using L = EncA<S>;
  constexpr int NT = L::NT;
  unsigned char* smem = LYRA_DYN_SMEM();
  float* u = reinterpret_cast<float*>(smem + L::kSmemU);
  float* d = reinterpret_cast<float*>(smem + L::kSmemD);
  float* wbuf = reinterpret_cast<float*>(smem + L::kSmemW);
  int* slot = reinterpret_cast<int*>(smem + L::kSmemI);
  int* active = slot + S;
  int* n18 = active + S;
  int tile;
  InitWeightPipe<NT>();
  LoadTileMeta<S>(io, n18g, slot, active, n18, tile);
  if (n18[S] == kTileIdle) return;
  float* st = state + (size_t)tile * EncStateA::kUnits * S;
  const int tid = (int)threadIdx.x;
  PrefetchTileState<LYRA_PREFETCH_STATE>(st, EncStateA::kUnits * S * 4);
  IssuePrologue<NT>(wbuf, NextF32(BlobPtr<float>(blob, P.first.w), 16, 64, 64));
  int ph = 0;
  LYRA_PHASE(0, ph);

  // ---- input window X[368][S] (aliases d): 48 carried samples + 320 new ones as unit floats (dsp_utils.h:104-108)
  float* X = d;
  // rows are skewed by one pad row per 16 (row r lives at r + r/16) so the 4 time rows a warp reads per tap hit
  // different banks (their distance would otherwise be 16*S words = a multiple of 32 banks)
  BatchedLoop<NT, 2, float>(48 * S, [&](int i) { return st[EncStateA::kFirst * S + i]; },
                            [&](int i, float v) { const int r = i / S; X[(r + (r >> 4)) * S + i % S] = v; });
  BatchedLoop<NT, 8, float>(320 * S,
    [&](int i) { const int s = i / 320, k = i % 320; return active[s] ? (float)pcm[(size_t)slot[s] * 320 + k] * (1.0f / 32768.0f) : 0.0f; },
    [&](int i, float v) { const int s = i / 320, k = i % 320; X[(48 + k + ((48 + k) >> 4)) * S + s] = v; });
  // prefix rows 0..4 of u: the 5 carried rows of encoder_0/simpleconv
  BatchedLoop<NT, 8, float>(64 * 5 * S, [&](int i) { return st[EncStateA::kDown0 * S + i]; },
                            [&](int i, float v) { const int c = i / (5 * S), r = i % (5 * S); u[(size_t)c * L::LDU + r] = v; });
  __syncthreads();
  for (int i = tid; i < 48 * S; i += NT)
    if (active[i % S]) { const int r = 320 + i / S; st[EncStateA::kFirst * S + i] = X[(r + (r >> 4)) * S + i % S]; }
  LYRA_PHASE(0, ph);
  // ---- first_layer: K = 64, stride 16, 1 -> 64 ; u = conv + bias (pre-activation residual stream)
  {
    const float* b = BlobPtr<float>(blob, P.first.bias);
    GemmF32Tap<S, NT, 8, L::TN, 16, 4, true>(X, 0, 0, 17, 64, 1, 1, 20, 64, BlobPtr<float>(blob, P.first.w), wbuf, true,
      NextF32(BlobPtr<float>(blob, P.r0[0].pw1.w), 16, 64, 64),
      [&](int t, int s0, int n0, float (&acc)[8][L::TN]) {
#pragma unroll
        for (int j = 0; j < L::TN; ++j) {
          float* o = u + (size_t)(n0 + j) * L::LDU + (5 + t) * S + s0;
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] = __fadd_rn(acc[i][j], b[n0 + j]);
        }
      });
  }
  // ---- encoder_0: three residual units, dilation 1/3/9
  LYRA_PHASE(0, ph);
  static_assert(EncStateA::kRing1 == EncStateA::kRing0 + 64 * 2 && EncStateA::kRing2 == EncStateA::kRing1 + 64 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, 8, L::TN, L::TN, 4, 16, 64, 20>(blob, P.r0, u, L::LDU, 5, d, 1, st + (size_t)EncStateA::kRing0 * S, n18, active, wbuf,
                                                       NextF32(BlobPtr<float>(blob, P.down0.w), 16, 128, 640, d, L::kStgDown), 0, ph);
  // carried rows for the next frame: the last 5 activated rows
  for (int i = tid; i < 64 * 5 * S; i += NT) {
    const int c = i / (5 * S), r = i % (5 * S);
    if (active[r % S]) st[EncStateA::kDown0 * S + i] = u[(size_t)c * L::LDU + 20 * S + r];
  }
  // ---- encoder_0/simpleconv: K = 10, stride 5, 64 -> 128 ; pre-activation output to HBM for kernel B
  LYRA_PHASE(0, ph);
  {
    const float* b = BlobPtr<float>(blob, P.down0.bias);
    float* out = mid + (size_t)tile * 128 * 4 * S;
    // the d buffer is free from here on: it hosts this GEMM's weight ring (kStgDown x 16 x 128 floats).  With 32 GEMM rows a chunk is
    // consumed in a fraction of the L2 round trip, so the ring is as deep as d allows.
    static_assert(L::kStgDown * 16 * 128 * 4 <= 64 * L::LDD * 4, "simpleconv weight ring must fit in d");
    // 4 output rows x S streams = 32 GEMM rows only: LYRA_A_DOWN_TM x LYRA_A_DOWN_TN thread tiles decide how many of the block's
    // ten warps get a tile (8 x 4: four warps; 4 x 4 or 8 x 2: eight)
    constexpr int DTM = S >= 16 ? 8 : LYRA_A_DOWN_TM, DTN = S >= 16 ? 4 : LYRA_A_DOWN_TN;
    GemmF32Tap<S, NT, DTM, DTN, 16, 4, false, L::kStgDown>(u, L::LDU, 0, 5, 10, 64, 1, 4, 128, BlobPtr<float>(blob, P.down0.w), d, true, NoNext(),
      [&](int t, int s0, int n0, float (&acc)[DTM][DTN]) {
#pragma unroll
        for (int j = 0; j < DTN; ++j) {
          float* o = out + ((size_t)(n0 + j) * 4 + t) * S + s0;
#pragma unroll
          for (int i = 0; i < DTM; ++i) o[i] = __fadd_rn(acc[i][j], b[n0 + j]);
        }
      });
  }
  if (tid < S && active[tid]) n18g[tile * S + tid] = (n18[tid] + 1) % 18;
  LYRA_PHASE(0, ph);
}

// ================================================================================================
//                                        ENCODER  B
// ================================================================================================
template <int S>
struct EncB {
  static constexpr int NT = 256;
  static constexpr int kMinBlocks = S <= 8 ? LYRA_B_MIN_BLOCKS : 1;
  static constexpr int TM = 8;                            // streams per fp32 thread tile (8 x 4 tiles: fewer smem wavefronts per FMA)
  static constexpr int WM4 = 4 * S / TM >= 4 ? 4 : 4 * S / TM;   // m-groups per warp for T = 4 / 2 / 1 row layers
  static constexpr int WM2 = 2 * S / TM >= 4 ? 4 : 2 * S / TM;
  static constexpr int WM1 = 1 * S / TM >= 4 ? 4 : 1 * S / TM;
  static constexpr int LD1 = 6 * S;                       // u1: 2 carried rows + 4
  static constexpr int LQ2 = PadLd(2 * S), LQA = PadLd(4 * S), LQB = PadLd(3 * S);   // padded int8 word strides (MMA A operand)
  // Shared memory is reused along the layer sequence (72 KB at S = 8, so three blocks share an SM):
  //   region A: u1 f32 [128][6S]  ->  d2 f32 [256][2S]  ->  aq words [64][LQA] + bq words [128][LQB]
  //   region B: d1 f32 [128][4S]  ->  u2 f32 [256][2S]
  //   region C: hq words [64][LQ2]
  //   region W: fp32 weight ring  ->  (after the last fp32 GEMM) dq8, resq words [64][LQ2] each
  static constexpr int kMax(int a, int b) { return a > b ? a : b; }
  static constexpr int kRA = 0;
  static constexpr int kRABytes = kMax(kMax(128 * LD1 * 4, 256 * 2 * S * 4), 64 * LQA * 4 + 128 * LQB * 4);
  static constexpr int kRB = kRA + kRABytes;
  static constexpr int kRBBytes = kMax(128 * 4 * S * 4, 256 * 2 * S * 4);
  static constexpr int kRC = kRB + kRBBytes;
  static constexpr int kW = kRC + 64 * LQ2 * 4;
  static constexpr int kStg = S <= 8 ? LYRA_BC_STAGES : kStages;      // ring depth of the kernel's fp32 GEMMs
  static constexpr int kWBytes = kMax(kStg * 8 * 256 * 4, 2 * 64 * LQ2 * 4);
  static constexpr int kI8Pd = S <= 8 ? LYRA_B_I8_PD : LYRA_I8_PD;    // k-steps of int8 weight fragments in flight from L2
  // LYRA_B_DEEP_RINGS (experiment, off: slower before the H100 port - with three blocks per SM the GEMM phases are bound by
  // shared-memory operand delivery, not by the ring): the 8-32-row GEMMs' rings borrow the neighbouring regions that are dead
  // while their K loops run:
  //   encoder_1 (three units)   ring over [C | W]: hq is not written before the mixed unit      7 stages x 4 KB (8 k-rows x 128)
  //   encoder_1/simpleconv      ring over [B | C | W]: d1 is dead, u2 is written by its epilogue  5 stages x 8 KB (8 k-rows x 256)
  static constexpr bool kDeep = S <= 8 && LYRA_B_DEEP_RINGS != 0 && kStg == kStages;
  static constexpr int kStgR = kDeep ? 7 : kStg, kKcR = kDeep ? 8 : 16;
  static constexpr int kStgD = kDeep ? 5 : kStg;
  static constexpr int kI = kW + kWBytes;
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;
  static constexpr int kRingR = kDeep ? kRC : kW, kRingD = kDeep ? kRB : kW;
  static_assert(kRingR + kStgR * kKcR * 128 * 4 <= kW + kWBytes && kRingD + kStgD * 8 * 256 * 4 <= kW + kWBytes, "borrowed rings end with region W");
  static_assert(kRingR % 16 == 0 && kRingD % 16 == 0, "bulk-copy alignment");
};

template <int S>
__global__ void __launch_bounds__(EncB<S>::NT, EncB<S>::kMinBlocks)
EncoderKernelB(const uint8_t* __restrict__ blob, EncoderParams P, TileIo io, const float* __restrict__ mid,
               float* __restrict__ state, int* __restrict__ n18g, float* __restrict__ features) {
  using L = EncB<S>;
  constexpr int NT = L::NT;
  constexpr int TM = L::TM;
  unsigned char* smem = LYRA_DYN_SMEM();
  constexpr int LQ2 = L::LQ2, LQA = L::LQA, LQB = L::LQB;
  float* u1 = reinterpret_cast<float*>(smem + L::kRA);
  float* d2 = reinterpret_cast<float*>(smem + L::kRA);          // after encoder_1/simpleconv has consumed u1
  uint32_t* aq = reinterpret_cast<uint32_t*>(smem + L::kRA);    // after the mixed unit's fp32 1x1 has consumed d2
  uint32_t* bq = aq + 64 * LQA;
  float* d1 = reinterpret_cast<float*>(smem + L::kRB);
  float* u2 = reinterpret_cast<float*>(smem + L::kRB);          // d1 is dead once encoder_1's last unit is done
  uint32_t* hq = reinterpret_cast<uint32_t*>(smem + L::kRC);
  float* wbuf = reinterpret_cast<float*>(smem + L::kW);
  uint32_t* dq8 = reinterpret_cast<uint32_t*>(smem + L::kW);    // the fp32 weight ring is idle after the mixed unit's fp32 1x1
  uint32_t* resq = dq8 + 64 * LQ2;
  int* slot = reinterpret_cast<int*>(smem + L::kI);
  int* active = slot + S;
  int* n18 = active + S;
  int tile;
  InitWeightPipe<NT>();
  LoadTileMeta<S>(io, n18g, slot, active, n18, tile);
  if (n18[S] == kTileIdle) return;
  uint32_t* stw = reinterpret_cast<uint32_t*>(state) + (size_t)tile * EncStateB::kUnits * S;
  float* st = reinterpret_cast<float*>(stw);
  const int tid = (int)threadIdx.x;
  PrefetchTileState<LYRA_PREFETCH_STATE>(st, EncStateB::kUnits * S * 4);
  float* ring_r = reinterpret_cast<float*>(smem + L::kRingR);       // encoder_1's ring
  float* ring_d = reinterpret_cast<float*>(smem + L::kRingD);       // encoder_1/simpleconv's ring
  IssuePrologue<NT>(ring_r, NextF32(BlobPtr<float>(blob, P.r1[0].pw1.w), L::kKcR, 128, 128, nullptr, L::kStgR));
  int ph = 0;
  LYRA_PHASE(1, ph);

  // ---- u1 <- kernel A output (rows 2..5), carried rows of encoder_1/simpleconv (rows 0..1)
  {
    const float* in = mid + (size_t)tile * 128 * 4 * S;
    BatchedLoop<NT, 4, float4>(128 * S, [&](int i) { return reinterpret_cast<const float4*>(in)[i]; },
      [&](int i, float4 v) { const int c = i / S, r = (i % S) * 4; *reinterpret_cast<float4*>(u1 + (size_t)c * L::LD1 + 2 * S + r) = v; });
    BatchedLoop<NT, 8, float>(128 * 2 * S, [&](int i) { return st[EncStateB::kDown1 * S + i]; },
      [&](int i, float v) { const int c = i / (2 * S), r = i % (2 * S); u1[(size_t)c * L::LD1 + r] = v; });
  }
  __syncthreads();
  // ---- encoder_1: three residual units @128 (second 1x1 has 2 groups)
  LYRA_PHASE(1, ph);
  static_assert(EncStateB::kRing1 == EncStateB::kRing0 + 128 * 2 && EncStateB::kRing2 == EncStateB::kRing1 + 128 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, TM, LYRA_BC_TN, LYRA_BC_TN, L::WM4, L::kKcR, 128, 4, false, 4 * S, 1, 1, L::kStgR>(
      blob, P.r1, u1, L::LD1, 2, d1, 2, st + (size_t)EncStateB::kRing0 * S, n18, active, ring_r,
      NextF32(BlobPtr<float>(blob, P.down1.w), 8, 256, 256, ring_d, L::kStgD), 1, ph);
  for (int i = tid; i < 128 * 2 * S; i += NT) {
    const int c = i / (2 * S), r = i % (2 * S);
    if (active[r % S]) st[EncStateB::kDown1 * S + i] = u1[(size_t)c * L::LD1 + 4 * S + r];
  }
  // ---- encoder_1/simpleconv: K = 4, stride 2, 128 -> 256, 2 groups ; u2 = pre-activation
  LYRA_PHASE(1, ph);
  {
    const float* b = BlobPtr<float>(blob, P.down1.bias);
    GemmF32Tap<S, NT, TM, LYRA_BC_TN, 8, L::WM2, false, L::kStgD>(u1, L::LD1, 0, 2, 4, 64, 2, 2, 256, BlobPtr<float>(blob, P.down1.w), ring_d, true,
      NextF32(BlobPtr<float>(blob, P.m_pw1.w), 8, 256, 256, wbuf, L::kStg),
      [&](int t, int s0, int n0, float (&acc)[TM][LYRA_BC_TN]) {
#pragma unroll
        for (int j = 0; j < LYRA_BC_TN; ++j) {
          float* o = u2 + (size_t)(n0 + j) * 2 * S + t * S + s0;
#pragma unroll
          for (int i = 0; i < TM; ++i) o[i] = __fadd_rn(acc[i][j], b[n0 + j]);
        }
      });
  }
  // ---- encoder_2/resnet_0 (mixed): f32 depthwise + f32 1x1, QUANTIZE, int8 LeakyReLU, int8 1x1 (4 groups),
  //      DEQUANTIZE + f32 residual, QUANTIZE, int8 LeakyReLU
  constexpr int LD2 = 2 * S;
  LYRA_PHASE(1, ph);
  if (n18[S] >= 0)
    DwF32RingFast<S, NT, 256, 2, 1>(u2, LD2, 0, d2, LD2, BlobPtr<float>(blob, P.m_dw.w), BlobPtr<float>(blob, P.m_dw.bias),
                                    st + (size_t)EncStateB::kRingM * S, n18[S], active);
  else
    DwF32Ring<S, NT>(u2, LD2, 0, d2, LD2, 256, 2, 1, BlobPtr<float>(blob, P.m_dw.w), BlobPtr<float>(blob, P.m_dw.bias),
                     st + (size_t)EncStateB::kRingM * S, n18, active);
  {
    const float* b = BlobPtr<float>(blob, P.m_pw1.bias);
    const int8_t* lut = BlobPtr<int8_t>(blob, P.m_lr1.lut);
    const QuantP q1 = P.m_q1;
    GemmF32Tap<S, NT, TM, LYRA_BC_TN, 8, L::WM2, false, L::kStg>(d2, LD2, 0, 1, 1, 256, 1, 2, 256, BlobPtr<float>(blob, P.m_pw1.w), wbuf, true,
      NoNext(),
      [&](int t, int s0, int n0, float (&acc)[TM][LYRA_BC_TN]) {
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          int q[LYRA_BC_TN];
#pragma unroll
          for (int j = 0; j < LYRA_BC_TN; ++j) q[j] = lut[QuantizeF32(__fadd_rn(acc[i][j], b[n0 + j]), q1.scale, q1.zp) + 128];
          uint32_t* word = hq + (size_t)(n0 / 4) * LQ2 + t * S + s0 + i;       // channels 4k .. 4k+3 of one (row, stream), byte j = channel 4k + j
          if constexpr (LYRA_BC_TN == 4) *word = PackI8x4(q[0], q[1], q[2], q[3]);
          else reinterpret_cast<uint16_t*>(word)[(n0 % 4) / 2] = (uint16_t)((q[0] & 0xff) | ((q[1] & 0xff) << 8));
        }
      });
  }
  {
    const int* bias = BlobPtr<int>(blob, P.m_pw2.bias);
    const int* mult = BlobPtr<int>(blob, P.m_pw2.mult);
    const int* shift = BlobPtr<int>(blob, P.m_pw2.shift);
    const int8_t* lut = BlobPtr<int8_t>(blob, P.m_lr2.lut);
    const QuantP dq = P.m_dq, q2 = P.m_q2;
    const int out_zp = P.m_pw2.out_zp;
    GemmI8Mma<S, NT, (S >= 16 ? 8 : 4), L::kI8Pd>(hq, LQ2, 0, 1, 1, 64, 4, 2, 256, BlobPtr<uint2>(blob, P.m_pw2.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        int r[4], a[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int q = RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp);
          const float v = __fadd_rn(DequantizeI8(q, dq.scale, dq.zp), u2[(size_t)(n0 + j) * LD2 + t * S + s]);
          r[j] = QuantizeF32(v, q2.scale, q2.zp);
          a[j] = lut[r[j] + 128];
        }
        resq[(size_t)(n0 / 4) * LQ2 + t * S + s] = PackI8x4(r[0], r[1], r[2], r[3]);
        aq[(size_t)(n0 / 4) * LQA + (2 + t) * S + s] = PackI8x4(a[0], a[1], a[2], a[3]);
      });
  }
  // ---- quant_encoder_2/resnet_{1,2}
  LYRA_PHASE(1, ph);
  static_assert(EncStateB::kRingQ1 == EncStateB::kRingQ0 + 64 * 6, "ring blocks back to back");
  ResUnitsI8x2<S, NT, L::kI8Pd>(blob, P.q, aq, LQA, 2, resq, dq8, hq, stw + (size_t)EncStateB::kRingQ0 * S, n18, active, 1, ph);
  // ---- quant_encoder_2/simpleconv: K = 4, stride 2, 256 -> 512, 4 groups, then int8 LeakyReLU
  LYRA_PHASE(1, ph);
  BatchedLoop<NT, 4, uint32_t>(64 * 2 * S, [&](int i) { return stw[EncStateB::kDown2 * S + i]; },
    [&](int i, uint32_t v) { const int c = i / (2 * S), r = i % (2 * S); aq[(size_t)c * LQA + r] = v; });
  BatchedLoop<NT, 8, uint32_t>(128 * 2 * S, [&](int i) { return stw[EncStateB::kBott * S + i]; },
    [&](int i, uint32_t v) { const int c = i / (2 * S), r = i % (2 * S); bq[(size_t)c * LQB + r] = v; });
  __syncthreads();
  for (int i = tid; i < 64 * 2 * S; i += NT) {
    const int c = i / (2 * S), r = i % (2 * S);
    if (active[r % S]) stw[EncStateB::kDown2 * S + i] = aq[(size_t)c * LQA + 2 * S + r];
  }
  {
    const int* bias = BlobPtr<int>(blob, P.down2.bias);
    const int* mult = BlobPtr<int>(blob, P.down2.mult);
    const int* shift = BlobPtr<int>(blob, P.down2.shift);
    const int8_t* lut = BlobPtr<int8_t>(blob, P.down2_lr.lut);
    const int out_zp = P.down2.out_zp;
    GemmI8Mma<S, NT, 8, L::kI8Pd>(aq, LQA, 0, 2, 4, 64, 4, 1, 512, BlobPtr<uint2>(blob, P.down2.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        (void)t;
        int q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) q[j] = lut[RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp) + 128];
        bq[(size_t)(n0 / 4) * LQB + 2 * S + s] = PackI8x4(q[0], q[1], q[2], q[3]);
      });
  }
  // carried rows of quant_bottleneck_1: the two newest rows
  for (int i = tid; i < 128 * 2 * S; i += NT) {
    const int c = i / (2 * S), r = i % (2 * S);
    if (active[r % S]) stw[EncStateB::kBott * S + i] = bq[(size_t)c * LQB + S + r];
  }
  // ---- quant_bottleneck_1: K = 3, 512 -> 64, 4 groups ; DEQUANTIZE -> features
  LYRA_PHASE(1, ph);
  {
    const int* bias = BlobPtr<int>(blob, P.bott.bias);
    const int* mult = BlobPtr<int>(blob, P.bott.mult);
    const int* shift = BlobPtr<int>(blob, P.bott.shift);
    const QuantP dq = P.out_dq;
    const int out_zp = P.bott.out_zp;
    GemmI8Mma<S, NT, 1, L::kI8Pd>(bq, LQB, 0, 1, 3, 128, 4, 1, 64, BlobPtr<uint2>(blob, P.bott.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        (void)t;
        if (!active[s]) return;
        float* o = features + (size_t)slot[s] * 64 + n0;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          o[j] = DequantizeI8(RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp), dq.scale, dq.zp);
      });
  }
  if (tid < S && active[tid]) n18g[tile * S + tid] = (n18[tid] + 1) % 18;
  LYRA_PHASE(1, ph);
}

// ================================================================================================
//                                        DECODER  C
// ================================================================================================
template <int S, bool TC = false>
struct DecC {
  static constexpr int NT = 256;
  static constexpr int kMinBlocks = S <= 8 ? LYRA_C_MIN_BLOCKS : 1;
  static constexpr int kI8Pd = S <= 8 ? LYRA_C_I8_PD : LYRA_I8_PD;    // prefetch depth of the four-n-tile int8 GEMMs (the eight-n-tile upsamplers keep LYRA_I8_PD)
  static constexpr int TM = 8;                            // streams per fp32 thread tile (8 x 4 tiles: fewer smem wavefronts per FMA)
  static constexpr int WM4 = 4 * S / TM >= 4 ? 4 : 4 * S / TM;   // m-groups per warp for T = 4 / 2 / 1 row layers
  static constexpr int WM2 = 2 * S / TM >= 4 ? 4 : 2 * S / TM;
  static constexpr int WM1 = 1 * S / TM >= 4 ? 4 : 1 * S / TM;
  static constexpr int LQ2 = PadLd(2 * S), LQA = PadLd(4 * S), LQB = PadLd(3 * S);   // padded int8 word strides (MMA A operand)
  // Shared memory is reused along the layer sequence (59 KB at S = 8, so three blocks share an SM):
  //   region 1: F f32 [64][3S] + xq words [128][LQB]  ->  aq words [64][LQA]  ->  d1 f32 [128][4S]
  //   region 2: u f32 [256][2S]  ->  u1 f32 [128][4S]
  //   region W: fp32 weight ring (bottleneck_2, decoder_1)  <->  hq, dq8, resq words [64][LQ2] each (int8 phases)
  static constexpr int kMax(int a, int b) { return a > b ? a : b; }
  static constexpr int kF = 0;
  static constexpr int kXq = kF + 64 * 3 * S * 4;
  // tensor-core mode: d1 is an MMA A operand (padded stride); decoder_1 warp tiles: 2 m-tiles x RWN n-tiles
  static constexpr int LD1 = TC ? PadLd(4 * S) : 4 * S;
  static constexpr int RWM = 2, RWN = S >= 16 ? 4 : 2;
  static_assert(!TC || ((4 * S + 31) / 32) * (16 / RWN) <= NT / 32, "decoder_1: one warp tile per warp");
  static constexpr int kR1Bytes = kMax(kMax(64 * 3 * S * 4 + 128 * LQB * 4, 64 * LQA * 4), 128 * LD1 * 4);
  static constexpr int kU = kF + kR1Bytes;
  static constexpr int kW = kU + 256 * 2 * S * 4;
  static constexpr int kWBytes = kMax(kStages * 4 * 512 * 4, 3 * 64 * LQ2 * 4);
  static constexpr int kI = kW + kWBytes;
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;
};

template <int S, bool TC>
__global__ void __launch_bounds__(DecC<S, TC>::NT, DecC<S, TC>::kMinBlocks)
DecoderKernelC(const uint8_t* __restrict__ blob, DecoderParams P, TileIo io,
               const float* __restrict__ features, float* __restrict__ state, int* __restrict__ n18g,
               float* __restrict__ mid) {
  using L = DecC<S, TC>;
  constexpr int NT = L::NT;
  constexpr int TM = L::TM;
  unsigned char* smem = LYRA_DYN_SMEM();
  float* F = reinterpret_cast<float*>(smem + L::kF);
  uint32_t* xq = reinterpret_cast<uint32_t*>(smem + L::kXq);
  float* u = reinterpret_cast<float*>(smem + L::kU);
  float* u1 = u;
  constexpr int LQ2 = L::LQ2, LQA = L::LQA, LQB = L::LQB;
  uint32_t* aq = reinterpret_cast<uint32_t*>(smem + L::kF);     // F and xq are dead once the first upsampler has run
  float* d1 = reinterpret_cast<float*>(smem + L::kF);           // aq is dead once the second upsampler has run
  float* wbuf = reinterpret_cast<float*>(smem + L::kW);
  uint32_t* hq = reinterpret_cast<uint32_t*>(smem + L::kW);     // the fp32 weight ring is idle during the int8 phases
  uint32_t* dq8 = hq + 64 * LQ2;
  uint32_t* resq = dq8 + 64 * LQ2;
  int* slot = reinterpret_cast<int*>(smem + L::kI);
  int* active = slot + S;
  int* n18 = active + S;
  int tile;
  InitWeightPipe<NT>();
  LoadTileMeta<S>(io, n18g, slot, active, n18, tile);
  if (n18[S] == kTileIdle) return;
  uint32_t* stw = reinterpret_cast<uint32_t*>(state) + (size_t)tile * DecStateC::kUnits * S;
  float* st = reinterpret_cast<float*>(stw);
  const int tid = (int)threadIdx.x;
  PrefetchTileState<LYRA_PREFETCH_STATE>(st, DecStateC::kUnits * S * 4);
  constexpr int LD2 = 2 * S;
  const UpI8& up0 = P.up0;
  const UpI8& up1 = P.up1;
  IssuePrologue<NT>(wbuf, NextF32(BlobPtr<float>(blob, P.bott.w), 4, 512, 48));
  int ph = 0;
  LYRA_PHASE(2, ph);

  // ---- F: 2 carried feature rows + the new one ; overlap states into u ; padding rows of xq
  BatchedLoop<NT, 4, float>(64 * 2 * S, [&](int i) { return st[DecStateC::kBott * S + i]; },
    [&](int i, float v) { const int c = i / (2 * S), r = i % (2 * S); F[(size_t)c * 3 * S + r] = v; });
  BatchedLoop<NT, 2, float>(64 * S, [&](int i) { const int s = i / 64, c = i % 64; return active[s] ? features[(size_t)slot[s] * 64 + c] : 0.0f; },
    [&](int i, float v) { const int s = i / 64, c = i % 64; F[(size_t)c * 3 * S + 2 * S + s] = v; });
  BatchedLoop<NT, 4, float4>(256 * 2 * S / 4, [&](int i) { return reinterpret_cast<const float4*>(st + (size_t)DecStateC::kUp0 * S)[i]; },
    [&](int i, float4 v) { reinterpret_cast<float4*>(u)[i] = v; });
  {
    const uint32_t pad = PackI8x4(P.bott_q.zp, P.bott_q.zp, P.bott_q.zp, P.bott_q.zp);
    for (int i = tid; i < 128 * S; i += NT) { const int c = i / S, s = i % S; xq[(size_t)c * LQB + s] = pad; xq[(size_t)c * LQB + 2 * S + s] = pad; }
  }
  __syncthreads();
  for (int i = tid; i < 64 * 2 * S; i += NT) {
    const int c = i / (2 * S), r = i % (2 * S);
    if (active[r % S]) st[DecStateC::kBott * S + i] = F[(size_t)c * 3 * S + S + r];
  }
  // ---- bottleneck_2/simpleconv: K = 3, 64 -> 512, 4 groups ; LeakyReLU ; QUANTIZE
  LYRA_PHASE(2, ph);
  {
    const float* b = BlobPtr<float>(blob, P.bott.bias);
    const QuantP q = P.bott_q;
    GemmF32Tap<S, NT, TM, 4, 4, L::WM1, false>(F, 3 * S, 0, 1, 3, 16, 4, 1, 512, BlobPtr<float>(blob, P.bott.w), wbuf, true,
      NoNext(),
      [&](int t, int s0, int n0, float (&acc)[TM][4]) {
        (void)t;
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          int v[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) v[j] = QuantizeF32(LeakyRelu(__fadd_rn(acc[i][j], b[n0 + j])), q.scale, q.zp);
          xq[(size_t)(n0 / 4) * LQB + S + s0 + i] = PackI8x4(v[0], v[1], v[2], v[3]);
        }
      });
  }
  // ---- quant_decoder_0 upsample: 4 x TRANSPOSE_CONV (K = 4, stride 2, 128 -> 64), T 1 -> 2 (+2 tail rows)
  LYRA_PHASE(2, ph);
  {
    const int* bias = BlobPtr<int>(blob, up0.g.bias);
    const int* mult = BlobPtr<int>(blob, up0.g.mult);
    const int* shift = BlobPtr<int>(blob, up0.g.shift);
    float* tail = st + (size_t)DecStateC::kUp0 * S;
    GemmI8Mma<S, NT, 8>(xq, LQB, 0, 1, 2, 128, 4, 2, 512, BlobPtr<uint2>(blob, up0.g.w),
      [&](int q, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        const int g = n0 / 128, r = (n0 % 128) / 64;
        const float* bf = BlobPtr<float>(blob, up0.bias_f32[g]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int co = (n0 + j) % 64, ch = g * 64 + co;
          const int qv = RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], up0.out_zp[g]);
          const float f = DequantizeI8(qv, up0.dq[g].scale, up0.dq[g].zp);
          if (q == 0) {
            float* o = u + (size_t)ch * LD2 + r * S + s;
            *o = __fadd_rn(f, *o);
          } else if (active[s]) {
            tail[((size_t)ch * 2 + r) * S + s] = __fsub_rn(__fadd_rn(f, 0.0f), bf[co]);
          }
        }
      });
  }
  // ---- LeakyReLU (f32) ; QUANTIZE -> aq rows 1..2
  LYRA_PHASE(2, ph);
  {
    const QuantP q = P.up0_q;
    for (int i = tid; i < 64 * 2 * S; i += NT) {
      const int c4 = i / (2 * S), r = i % (2 * S);
      int v[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) v[b] = QuantizeF32(LeakyRelu(u[(size_t)(c4 * 4 + b) * LD2 + r]), q.scale, q.zp);
      aq[(size_t)c4 * LQA + S + r] = PackI8x4(v[0], v[1], v[2], v[3]);
    }
  }
  __syncthreads();
  // ---- quant_decoder_0/resnet_0 (int8 body, f32 residual add)
  LYRA_PHASE(2, ph);
  if (n18[S] >= 0) DwI8RingFast<S, NT, 256, 2, 1>(aq, LQA, 1, dq8, LQ2, blob, P.m_dw, stw + (size_t)DecStateC::kRingM * S, n18[S], active);
  else DwI8Ring<S, NT>(aq, LQA, 1, dq8, LQ2, 256, 2, 1, blob, P.m_dw, stw + (size_t)DecStateC::kRingM * S, n18, active);
  {
    const int* bias = BlobPtr<int>(blob, P.m_pw1.bias);
    const int* mult = BlobPtr<int>(blob, P.m_pw1.mult);
    const int* shift = BlobPtr<int>(blob, P.m_pw1.shift);
    const int8_t* lut = BlobPtr<int8_t>(blob, P.m_lr1.lut);
    const int out_zp = P.m_pw1.out_zp;
    GemmI8Mma<S, NT, (S >= 16 ? 8 : 4), L::kI8Pd>(dq8, LQ2, 0, 1, 1, 256, 1, 2, 256, BlobPtr<uint2>(blob, P.m_pw1.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        int q[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) q[j] = lut[RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp) + 128];
        hq[(size_t)(n0 / 4) * LQ2 + t * S + s] = PackI8x4(q[0], q[1], q[2], q[3]);
      });
  }
  {
    const int* bias = BlobPtr<int>(blob, P.m_pw2.bias);
    const int* mult = BlobPtr<int>(blob, P.m_pw2.mult);
    const int* shift = BlobPtr<int>(blob, P.m_pw2.shift);
    const int8_t* lut = BlobPtr<int8_t>(blob, P.m_lr2.lut);
    const QuantP dq = P.m_dq, q2 = P.m_q2;
    const int out_zp = P.m_pw2.out_zp;
    GemmI8Mma<S, NT, (S >= 16 ? 8 : 4), L::kI8Pd>(hq, LQ2, 0, 1, 1, 64, 4, 2, 256, BlobPtr<uint2>(blob, P.m_pw2.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        int r[4], a[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int q = RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp);
          const float v = __fadd_rn(DequantizeI8(q, dq.scale, dq.zp), u[(size_t)(n0 + j) * LD2 + t * S + s]);
          r[j] = QuantizeF32(v, q2.scale, q2.zp);
          a[j] = lut[r[j] + 128];
        }
        resq[(size_t)(n0 / 4) * LQ2 + t * S + s] = PackI8x4(r[0], r[1], r[2], r[3]);
        aq[(size_t)(n0 / 4) * LQA + (1 + t) * S + s] = PackI8x4(a[0], a[1], a[2], a[3]);
      });
  }
  LYRA_PHASE(2, ph);
  static_assert(DecStateC::kRingQ1 == DecStateC::kRingQ0 + 64 * 6, "ring blocks back to back");
  ResUnitsI8x2<S, NT, L::kI8Pd>(blob, P.q, aq, LQA, 1, resq, dq8, hq, stw + (size_t)DecStateC::kRingQ0 * S, n18, active, 2, ph);
  // ---- quant_decoder_1 upsample: 2 x TRANSPOSE_CONV (K = 4, stride 2, 128 -> 64), T 2 -> 4 (+2 tail rows)
  LYRA_PHASE(2, ph);
  {
    const uint32_t pad = PackI8x4(up1.g.in_zp, up1.g.in_zp, up1.g.in_zp, up1.g.in_zp);
    for (int i = tid; i < 64 * S; i += NT) { const int c = i / S, s = i % S; aq[(size_t)c * LQA + s] = pad; aq[(size_t)c * LQA + 3 * S + s] = pad; }
    // u1 [128][4S]: rows 0..1 carry the overlap, rows 2..3 start from +0 (the zeros of the reference's concat)
    BatchedLoop<NT, 8, float>(128 * 4 * S,
      [&](int i) { const int c = i / (4 * S), r = i % (4 * S); return r < 2 * S ? st[DecStateC::kUp1 * S + (size_t)c * 2 * S + r] : 0.0f; },
      [&](int i, float v) { u1[i] = v; });
  }
  __syncthreads();
  {
    const int* bias = BlobPtr<int>(blob, up1.g.bias);
    const int* mult = BlobPtr<int>(blob, up1.g.mult);
    const int* shift = BlobPtr<int>(blob, up1.g.shift);
    float* tail = st + (size_t)DecStateC::kUp1 * S;
    if (!TC) IssuePrologue<NT>(wbuf, NextF32(BlobPtr<float>(blob, P.r1[0].pw1.w), 16, 128, 128));
    GemmI8Mma<S, NT, 8>(aq, LQA, 0, 1, 2, 128, 2, 3, 256, BlobPtr<uint2>(blob, up1.g.w),
      [&](int q, int s, int n0, int (&acc)[1][4]) {
        const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
        const int g = n0 / 128, r = (n0 % 128) / 64;
        const float* bf = BlobPtr<float>(blob, up1.bias_f32[g]);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int co = (n0 + j) % 64, ch = g * 64 + co;
          const int qv = RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], up1.out_zp[g]);
          const float f = DequantizeI8(qv, up1.dq[g].scale, up1.dq[g].zp);
          if (q < 2) {
            float* o = u1 + (size_t)ch * 4 * S + (2 * q + r) * S + s;
            *o = __fadd_rn(f, *o);
          } else if (active[s]) {
            tail[((size_t)ch * 2 + r) * S + s] = __fsub_rn(__fadd_rn(f, 0.0f), bf[co]);
          }
        }
      });
  }
  // ---- decoder_1: three fp32 residual units @128
  LYRA_PHASE(2, ph);
  static_assert(DecStateC::kRing1 == DecStateC::kRing0 + 128 * 2 && DecStateC::kRing2 == DecStateC::kRing1 + 128 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, TM, LYRA_BC_TN, LYRA_BC_TN, L::WM4, 16, 128, 4, TC, L::LD1, L::RWM, L::RWN>(
      blob, P.r1, u1, 4 * S, 0, d1, 2, st + (size_t)DecStateC::kRing0 * S, n18, active, wbuf, NoNext(), 2, ph);
  {
    float* out = mid + (size_t)tile * 128 * 4 * S;
    for (int i = tid; i < 128 * 4 * S; i += NT) out[i] = u1[i];
  }
  if (tid < S && active[tid]) n18g[tile * S + tid] = (n18[tid] + 1) % 18;
  LYRA_PHASE(2, ph);
}

// ================================================================================================
//                                        DECODER  D
// ================================================================================================
template <int S, bool TC = false>
struct DecD {
  static constexpr int NT = 320;
  static constexpr int TN = S >= 16 ? 8 : 4;
  static constexpr int kMinBlocks = S <= 8 ? 2 : 1;
  static constexpr int TNU = S >= 16 ? 10 : 5;            // decoder_2/simple column tile (320 columns)
  static constexpr int TNL = S >= 16 ? 4 : 2;             // last_layer column tile (16 columns)
  static constexpr int WML = S >= 16 ? 8 : 4;
  static constexpr int WMU = S >= 16 ? 2 : 1;
  static constexpr int KCU = 8;                           // its ring starts right behind X inside d and runs into the regular ring
  // u: 3 zero rows + 20 + 3 zero rows.  Tensor-core mode pads the strides of the MMA A operands (u, d, X) and
  // needs no weight ring (weights go from L2 straight into fragments).
  static constexpr int LDU = TC ? PadLd(26 * S) : 26 * S, LDD = TC ? PadLd(20 * S) : 20 * S, LDX = TC ? PadLd(6 * S) : 6 * S;
  static constexpr int kU = 0;
  static constexpr int kD = kU + 64 * LDU * 4;              // d f32 [64][LDD]; aliases X f32 [128][LDX] and the PCM staging
  static constexpr int kW = kD + 64 * LDD * 4;
  static constexpr int kWBytes = TC ? 0 : kStages * 16 * 64 * 4 + 2048;   // regular ring (64-channel layers) + slack for the decoder_2/simple ring
  static constexpr int kSl = kW + kWBytes;                  // carried tail of last_layer [48][S]
  static_assert(TC || 128 * 6 * S * 4 + kStages * KCU * 320 * 4 <= 64 * LDD * 4 + kWBytes, "decoder_2/simple ring must fit behind X");
  static constexpr int kI = kSl + 48 * S * 4;
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;
  static_assert(128 * LDX <= 64 * LDD, "X must fit in d");
  static_assert(S * 320 * 2 <= 64 * LDD * 4, "PCM staging must fit in d");
  // tensor-core warp tiles: decoder_2 res-units RWM x RWN (one per warp), decoder_2/simple UWM x 2, last_layer 1 x 1
  static constexpr int RWM = S >= 16 ? 4 : 2, RWN = NT >= 320 ? 4 : 8;
  static constexpr int UWM = (5 * S + 15) / 16;
  static_assert(!TC || ((20 * S / 16 + RWM - 1) / RWM) * (8 / RWN) <= NT / 32, "decoder_2: one warp tile per warp");
};

template <int S, bool TC>
__global__ void __launch_bounds__(DecD<S, TC>::NT, DecD<S, TC>::kMinBlocks)
DecoderKernelD(const uint8_t* __restrict__ blob, DecoderParams P, TileIo io, const float* __restrict__ mid,
               float* __restrict__ state, int* __restrict__ n18g, int16_t* __restrict__ pcm) {
  using L = DecD<S, TC>;
  constexpr int NT = L::NT;
  unsigned char* smem = LYRA_DYN_SMEM();
  float* u = reinterpret_cast<float*>(smem + L::kU);
  float* d = reinterpret_cast<float*>(smem + L::kD);
  float* X = d;
  float* wbuf = reinterpret_cast<float*>(smem + L::kW);
  float* sl = reinterpret_cast<float*>(smem + L::kSl);
  int* slot = reinterpret_cast<int*>(smem + L::kI);
  int* active = slot + S;
  int* n18 = active + S;
  int tile;
  InitWeightPipe<NT>();
  LoadTileMeta<S>(io, n18g, slot, active, n18, tile);
  if (n18[S] == kTileIdle) return;
  float* st = state + (size_t)tile * DecStateD::kUnits * S;
  const int tid = (int)threadIdx.x;
  PrefetchTileState<LYRA_PREFETCH_STATE>(st, DecStateD::kUnits * S * 4);
  constexpr int LDX = L::LDX;
  float* wbuf_up2 = X + 128 * LDX;       // free tail of d + the regular ring
  if (!TC) IssuePrologue<NT>(wbuf_up2, NextF32(BlobPtr<float>(blob, P.up2.w), L::KCU, 320, 256));
  int ph = 0;
  LYRA_PHASE(3, ph);

  // ---- X [128][6S]: zero row, 4 rows from kernel C, zero row
  {
    const float* in = mid + (size_t)tile * 128 * 4 * S;
    BatchedLoop<NT, 4, float4>(128 * S, [&](int i) { return reinterpret_cast<const float4*>(in)[i]; },
      [&](int i, float4 v) { const int c = i / S, r = (i % S) * 4; *reinterpret_cast<float4*>(X + (size_t)c * LDX + S + r) = v; });
    for (int i = tid; i < 128 * 2 * S; i += NT) { const int c = i / (2 * S), r = i % (2 * S); X[(size_t)c * LDX + (r < S ? r : 4 * S + r)] = 0.0f; }
    // u rows: 3 zero rows | rows 0..4 carry the overlap of decoder_2/simple, rows 5..19 start from +0 | 3 zero rows
    for (int i = tid; i < 64 * 26 * S / 4; i += NT) {
      const int c = (i * 4) / (26 * S), r = (i * 4) % (26 * S);
      if (!(r >= 3 * S && r < 8 * S)) *reinterpret_cast<float4*>(u + (size_t)c * L::LDU + r) = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    BatchedLoop<NT, 8, float>(64 * 5 * S, [&](int i) { return st[DecStateD::kUp2 * S + i]; },
      [&](int i, float v) { const int c = i / (5 * S), r = i % (5 * S); u[(size_t)c * L::LDU + 3 * S + r] = v; });
    BatchedLoop<NT, 2, float>(48 * S, [&](int i) { return st[DecStateD::kLast * S + i]; }, [&](int i, float v) { sl[i] = v; });
  }
  __syncthreads();
  // ---- decoder_2/simple: TRANSPOSE_CONV K = 10, stride 5, 128 -> 64 ; T 4 -> 20 (+5 tail rows)
  LYRA_PHASE(3, ph);
  {
    const float* b = BlobPtr<float>(blob, P.up2.bias);
    float* tail = st + (size_t)DecStateD::kUp2 * S;
    auto epi_up = [&](int q, int s0, int n0, auto& acc) {
      constexpr int TMx = sizeof(acc) / sizeof(acc[0]), TNx = sizeof(acc[0]) / sizeof(float);
#pragma unroll
      for (int j = 0; j < TNx; ++j) {
        const int r = (n0 + j) / 64, co = (n0 + j) % 64;
        const float bias = b[co];
#pragma unroll
        for (int i = 0; i < TMx; ++i) {
          const float y = __fadd_rn(acc[i][j], bias);
          if (q < 4) {
            float* o = u + (size_t)co * L::LDU + (3 + 5 * q + r) * S + s0 + i;
            *o = __fadd_rn(y, *o);
          } else if (active[s0 + i]) {
            tail[((size_t)co * 5 + r) * S + s0 + i] = __fsub_rn(__fadd_rn(y, 0.0f), bias);
          }
        }
      }
    };
    if constexpr (TC)
      GemmTf32Mma<S, NT, L::UWM, 2, false>(X, LDX, 0, 1, 2, 128, 1, 5, 320, BlobPtr<float2>(blob, P.up2.wf), epi_up);
    else
      GemmF32Tap<S, NT, 8, L::TNU, L::KCU, L::WMU, false>(X, LDX, 0, 1, 2, 128, 1, 5, 320, BlobPtr<float>(blob, P.up2.w), wbuf_up2, true,
                                                          NextF32(BlobPtr<float>(blob, P.r2[0].pw1.w), 16, 64, 64, wbuf), epi_up);
  }
  // ---- decoder_2: three residual units @64, T = 20
  LYRA_PHASE(3, ph);
  static_assert(DecStateD::kRing1 == DecStateD::kRing0 + 64 * 2 && DecStateD::kRing2 == DecStateD::kRing1 + 64 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, 8, L::TN, L::TN, 4, 16, 64, 20, TC, L::LDD, L::RWM, L::RWN>(blob, P.r2, u, L::LDU, 3, d, 1, st + (size_t)DecStateD::kRing0 * S, n18, active, wbuf,
                                                       NextF32(BlobPtr<float>(blob, P.last.w), 16, 16, 256), 3, ph);
  // ---- last_layer: TRANSPOSE_CONV K = 64, stride 16, 64 -> 1 ; T 20 -> 320 (+48 tail) ; float -> int16
  LYRA_PHASE(3, ph);
  {
    const float bias = BlobPtr<float>(blob, P.last.bias)[0];
    float* tail = st + (size_t)DecStateD::kLast * S;
    int16_t* stage = reinterpret_cast<int16_t*>(d);      // [S][320]
    auto epi_last = [&](int q, int s0, int n0, auto& acc) {
      constexpr int TMx = sizeof(acc) / sizeof(acc[0]), TNx = sizeof(acc[0]) / sizeof(float);
#pragma unroll
      for (int j = 0; j < TNx; ++j) {
        const int t = 16 * q + n0 + j;
#pragma unroll
        for (int i = 0; i < TMx; ++i) {
          const float y = __fadd_rn(__fadd_rn(acc[i][j], bias), t < 48 ? sl[t * S + s0 + i] : 0.0f);
          if (t < 320) {
            // UnitToInt16Scalar (dsp_utils.h:53-60,79-88): scale, clip in float, truncate
            float v = __fmul_rn(y, 32768.0f);
            v = v > -32768.0f ? v : -32768.0f;
            v = v < 32767.0f ? v : 32767.0f;
            stage[(s0 + i) * 320 + t] = (int16_t)(int)v;
          } else if (active[s0 + i]) {
            tail[(t - 320) * S + s0 + i] = __fsub_rn(y, bias);
          }
        }
      }
    };
    if constexpr (TC)
      GemmTf32Mma<S, NT, 1, 1, false>(u, L::LDU, 0, 1, 4, 64, 1, 23, 16, BlobPtr<float2>(blob, P.last.wf), epi_last);
    else
      GemmF32Tap<S, NT, 8, L::TNL, 16, L::WML, false>(u, L::LDU, 0, 1, 4, 64, 1, 23, 16, BlobPtr<float>(blob, P.last.w), wbuf, true, NoNext(), epi_last);
    for (int i = tid; i < S * 320; i += NT) {
      const int s = i / 320;
      if (active[s]) pcm[(size_t)slot[s] * 320 + (i % 320)] = stage[i];
    }
  }
  if (tid < S && active[tid]) n18g[tile * S + tid] = (n18[tid] + 1) % 18;
  LYRA_PHASE(3, ph);
}

}  // namespace lyra_b200
