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

namespace lyra_b200 {

// Streams per tile: one thread block of every conv-net kernel processes one tile.  The kernels' shared-memory layouts (two
// resident blocks per SM for A and D, three for B and C), the tile-blocked streaming state, the host's stream -> tile map and
// DecoderKernelDW's warp-to-row mapping are all sized for it.
constexpr int kTileStreams = 8;

// ---- per-tile state layouts, in 4-byte units (each unit is S lanes wide) ----
// kT*: time rows per hop of the layers that own the rings (the T of their depthwise calls)
struct EncStateA {
  static constexpr int kFirst = 0;                               // [48]
  static constexpr int kRing0 = 48, kRing1 = kRing0 + 64 * 2, kRing2 = kRing1 + 64 * 6;   // [64][2|6|18]
  static constexpr int kDown0 = kRing2 + 64 * 18;                // [64][5]
  static constexpr int kUnits = kDown0 + 64 * 5;                 // 2032
  static constexpr int kT = 20;                                  // encoder_0
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
  static constexpr int kT1 = 4, kT2 = 2;                         // encoder_1; encoder_2 (kRingM) and quant_encoder_2 (kRingQ*)
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
  static constexpr int kT0 = 2, kT1 = 4;                         // quant_decoder_0 (kRingM, kRingQ*); decoder_1
};
struct DecStateD {
  static constexpr int kUp2 = 0;                                 // f32 [64][5]
  static constexpr int kRing0 = 320, kRing1 = kRing0 + 64 * 2, kRing2 = kRing1 + 64 * 6;  // f32 [64][2|6|18]
  static constexpr int kLast = kRing2 + 64 * 18;                 // f32 [48]
  static constexpr int kUnits = kLast + 48;                      // 2032
  static constexpr int kT = 20;                                  // decoder_2
};
// The int8 residual units (ResUnitI8) run two time rows per hop: quant_encoder_2 and quant_decoder_0
constexpr int kResI8Rows = 2;

// The dilated depthwise rings of the four layouts (w = 0 EncStateA, 1 EncStateB, 2 DecStateC, 3 DecStateD: the order of the
// network entries of a context), rings kDwRings[kDwRingFirst[w] .. kDwRingFirst[w + 1]) of layout w.  A ring is `rows`
// columns per lane (channels; int8 rings: packed words of 4 channels) of R units from unit `unit` on, [rows][R] (RingSlot);
// its layer runs T rows per hop, so a stream at hop counter n keeps relative row r in slot (n T + r) mod R.
// StreamAlignKernel (aux_kernels.cuh) rotates them.
struct DwRing { int unit, rows, R, T; };
constexpr DwRing kDwRings[] = {
    {EncStateA::kRing0, 64, 2, EncStateA::kT},  {EncStateA::kRing1, 64, 6, EncStateA::kT},  {EncStateA::kRing2, 64, 18, EncStateA::kT},
    {EncStateB::kRing0, 128, 2, EncStateB::kT1}, {EncStateB::kRing1, 128, 6, EncStateB::kT1}, {EncStateB::kRing2, 128, 18, EncStateB::kT1},
    {EncStateB::kRingM, 256, 2, EncStateB::kT2}, {EncStateB::kRingQ0, 64, 6, EncStateB::kT2}, {EncStateB::kRingQ1, 64, 18, EncStateB::kT2},
    {DecStateC::kRing0, 128, 2, DecStateC::kT1}, {DecStateC::kRing1, 128, 6, DecStateC::kT1}, {DecStateC::kRing2, 128, 18, DecStateC::kT1},
    {DecStateC::kRingM, 64, 2, DecStateC::kT0},  {DecStateC::kRingQ0, 64, 6, DecStateC::kT0}, {DecStateC::kRingQ1, 64, 18, DecStateC::kT0},
    {DecStateD::kRing0, 64, 2, DecStateD::kT},  {DecStateD::kRing1, 64, 6, DecStateD::kT},  {DecStateD::kRing2, 64, 18, DecStateD::kT},
};
constexpr int kDwRingFirst[5] = {0, 3, 9, 15, 18};
static_assert(sizeof(kDwRings) / sizeof(kDwRings[0]) == kDwRingFirst[4], "every ring belongs to one layout");
// Each ring is exactly the block its layout reserves: it ends where the next field starts.
static_assert(EncStateA::kRing1 == EncStateA::kRing0 + 64 * 2 && EncStateA::kRing2 == EncStateA::kRing1 + 64 * 6 &&
              EncStateA::kDown0 == EncStateA::kRing2 + 64 * 18, "EncStateA rings");
static_assert(EncStateB::kRing1 == EncStateB::kRing0 + 128 * 2 && EncStateB::kRing2 == EncStateB::kRing1 + 128 * 6 &&
              EncStateB::kDown1 == EncStateB::kRing2 + 128 * 18 && EncStateB::kRingQ0 == EncStateB::kRingM + 256 * 2 &&
              EncStateB::kRingQ1 == EncStateB::kRingQ0 + 64 * 6 && EncStateB::kDown2 == EncStateB::kRingQ1 + 64 * 18, "EncStateB rings");
static_assert(DecStateC::kRing1 == DecStateC::kRing0 + 128 * 2 && DecStateC::kRing2 == DecStateC::kRing1 + 128 * 6 &&
              DecStateC::kRingM == DecStateC::kRing2 + 128 * 18 && DecStateC::kRingQ0 == DecStateC::kRingM + 64 * 2 &&
              DecStateC::kRingQ1 == DecStateC::kRingQ0 + 64 * 6 && DecStateC::kUnits == DecStateC::kRingQ1 + 64 * 18, "DecStateC rings");
static_assert(DecStateD::kRing1 == DecStateD::kRing0 + 64 * 2 && DecStateD::kRing2 == DecStateD::kRing1 + 64 * 6 &&
              DecStateD::kLast == DecStateD::kRing2 + 64 * 18, "DecStateD rings");
static_assert(EncStateB::kT2 == kResI8Rows && DecStateC::kT0 == kResI8Rows, "the int8 rings' layers are ResUnitI8's");
constexpr bool DwRingsOk(int i) {
  return i == kDwRingFirst[4] ||
         ((kDwRings[i].R == 2 || kDwRings[i].R == 6 || kDwRings[i].R == 18) && kDwRings[i].T > 0 && DwRingsOk(i + 1));
}
static_assert(DwRingsOk(0), "R = 2 x dilation (1, 3, 9) divides 18, the hop counters' modulus");

struct TileIo {
  const int* tile_list;        // tiles to process, one per block
  const int* slot_of_stream;   // [max_streams] position of the stream in this call's I/O arrays, -1 = not in this call
  const uint8_t* skip;         // optional, by slot: 1 = the stream sits this call out (its state does not advance): DTX noise
                               // hops on the encoder side, pure comfort-noise hops on the decoder side
  const uint8_t* active;       // optional, by slot: 0 = the caller sits the stream out this call (lyra_b200_set_active_mask):
                               // inactive like a skipped stream
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
    active[threadIdx.x] = sl >= 0 && !(io.active != nullptr && !io.active[sl]) && !(io.skip != nullptr && io.skip[sl]);
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

// compile-time max, for the sizes of shared-memory regions that successive layers reuse
constexpr int kMax(int a, int b) { return a > b ? a : b; }

// The tile's streaming state (one contiguous block per kernel, 65-190 KB; the 262 MB working set of 4096 streams does not stay
// in the 50 MB L2 between hops) is requested into the L2 as soon as the block knows its tile: the ring / tail loads of the
// later phases then find it there instead of paying the HBM latency phase by phase.
__device__ __forceinline__ void PrefetchTileState(const void* p, int bytes) {
  if (threadIdx.x == 0) lyra_prefetch_l2(p, (unsigned)bytes);
}

// The prologue of every conv-net kernel, after its own weight-pipe or mbarrier setup: the tile's metadata into shared memory at
// meta = slot[S], active[S], n18[S + 1], then its state block (`units` 4-byte units per lane of `state`) into the L2.
// Returns false if the tile is idle.  It stays a composition of the two functions above: the same steps written inline give
// different PTX register numbering, and ptxas then allocates differently (kernels B and D spilled other amounts).
template <int S>
__device__ __forceinline__ bool BeginTile(const TileIo& io, const int* n18g, int* meta, float* state, int units, int& tile) {
  LoadTileMeta<S>(io, n18g, meta, meta + S, meta + 2 * S, tile);
  if (meta[3 * S] == kTileIdle) return false;
  PrefetchTileState(state + (size_t)tile * units * S, units * S * 4);
  return true;
}

// The epilogue of every conv-net kernel: the frame counter of each active stream of the tile advances by one hop
template <int S>
__device__ __forceinline__ void AdvanceHopCounters(int* n18g, int tile, const int* active, const int* n18) {
  const int tid = (int)threadIdx.x;
  if (tid < S && active[tid]) n18g[tile * S + tid] = (n18[tid] + 1) % 18;
}

// The newest R rows of a [C][ld] shared-memory buffer, rows row0 .. row0 + R - 1, become the carried rows [C][R] of the
// active streams: state unit `unit` onwards of the tile's state block st
template <int S, int NT, int C, int R, typename T>
__device__ __forceinline__ void StoreCarriedRows(T* st, int unit, const T* buf, int ld, int row0, const int* active) {
  for (int i = (int)threadIdx.x; i < C * R * S; i += NT) {
    const int c = i / (R * S), r = i % (R * S);
    if (active[r % S]) st[unit * S + i] = buf[(size_t)c * ld + row0 * S + r];
  }
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
                                           const int* active, float* wbuf, bool last, const WNext& after, int dil_rt = DIL) {
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
}

// The three residual units of one stage (dilation 1, 3, 9; ring blocks of 2, 6, 18 rows back to back) as ONE copy of the code in
// a loop that is not unrolled: the units differ only in their parameters and in the depthwise pass, and three inlined copies
// of the two GEMMs made kernels B / C overflow the instruction cache (15-20 % of their stall samples were instruction fetches).
template <int S, int NT, int TM, int TN1, int TN2, int WM, int KC, int C, int T, bool TC = false, int LDD = T * S, int WTM = 1, int WTN = 1,
          int STG = kStages>
__device__ __forceinline__ void ResUnitsF32x3(const uint8_t* blob, const ResF32* p3, float* u, int ldu, int row0u, float* d, int groups2,
                                              float* ring0, const int* n18, const int* active, float* wbuf, const WNext& after) {
#pragma unroll 1
  for (int i = 0; i < 3; ++i) {
    const ResF32& p = p3[i];
    const int dil = i == 0 ? 1 : (i == 1 ? 3 : 9);
    float* ring = ring0 + (size_t)(i == 0 ? 0 : (i == 1 ? 2 : 8)) * C * S;       // [C][2] | [C][6] | [C][18]
    const WNext nx = i < 2 ? NextF32(BlobPtr<float>(blob, p3[i + 1].pw1.w), KC, C, C, nullptr, STG) : after;
    ResUnitF32<S, NT, TM, TN1, TN2, WM, KC, C, T, 0, TC, LDD, WTM, WTN, STG>(blob, p, u, ldu, row0u, d, groups2, ring, n18, active, wbuf, i == 2, nx,
                                                                       dil);
  }
}

// int8 GEMM epilogue: requantise the four channels n0 .. n0 + 3 of an accumulator, int8 LeakyReLU (lut), pack them into one word
struct RequantLutPack {
  const int* bias;
  const int* mult;
  const int* shift;
  const int8_t* lut;
  int out_zp;
  __device__ __forceinline__ RequantLutPack(const uint8_t* blob, const GemmI8& g, const LReluQ& lr)
      : bias(BlobPtr<int>(blob, g.bias)), mult(BlobPtr<int>(blob, g.mult)), shift(BlobPtr<int>(blob, g.shift)),
        lut(BlobPtr<int8_t>(blob, lr.lut)), out_zp(g.out_zp) {}
  __device__ __forceinline__ uint32_t operator()(const int (&acc)[1][4], int n0) const {
    const RequantP4 rq = LoadRequant4(bias, mult, shift, n0);
    int q[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) q[j] = lut[RequantI8(acc[0][j], rq.b[j], rq.m[j], rq.s[j], out_zp) + 128];
    return PackI8x4(q[0], q[1], q[2], q[3]);
  }
};

// The int8 half of the mixed residual unit (encoder_2/resnet_0, quant_decoder_0/resnet_0): its second 1x1 convolution (4 groups)
// on hq, DEQUANTIZE + the f32 residual u [256][2S], QUANTIZE -> resq, int8 LeakyReLU -> aq rows row0a, row0a + 1.
// P: EncoderParams or DecoderParams (the same m_pw2 / m_dq / m_q2 / m_lr2 fields).
template <int S, int NT, int PDI, typename Params>
__device__ __forceinline__ void MixedUnitPw2I8(const uint8_t* blob, const Params& P, const uint32_t* hq, const float* u,
                                               uint32_t* resq, uint32_t* aq, int lda, int row0a) {
  constexpr int LQ2 = PadLd(2 * S), LD2 = 2 * S;
  const int* bias = BlobPtr<int>(blob, P.m_pw2.bias);
  const int* mult = BlobPtr<int>(blob, P.m_pw2.mult);
  const int* shift = BlobPtr<int>(blob, P.m_pw2.shift);
  const int8_t* lut = BlobPtr<int8_t>(blob, P.m_lr2.lut);
  const QuantP dq = P.m_dq, q2 = P.m_q2;
  const int out_zp = P.m_pw2.out_zp;
  GemmI8Mma<S, NT, 4, PDI>(hq, LQ2, 0, 1, 1, 64, 4, 2, 256, BlobPtr<uint2>(blob, P.m_pw2.w),
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
      aq[(size_t)(n0 / 4) * lda + (row0a + t) * S + s] = PackI8x4(a[0], a[1], a[2], a[3]);
    });
}

// One int8 residual unit on packed activations (quant_encoder_2/resnet_{1,2}, quant_decoder_0/resnet_{1,2}); the two
// 1x1 convolutions run on the tensor cores.
//   aq: LeakyReLU'd input (row offset row0a of [64][lda]); resq: the pre-activation residual; both updated in place.
template <int S, int NT, int DIL, int PDI = kI8Pd>
__device__ __forceinline__ void ResUnitI8(const uint8_t* blob, const ResI8& p, uint32_t* aq, int lda, int row0a,
                                          uint32_t* resq, uint32_t* dq8, uint32_t* hq, uint32_t* ring,
                                          const int* n18, const int* active, int dil_rt = DIL) {
  constexpr int T = kResI8Rows, C = 256, LD = PadLd(T * S);
  constexpr int NTW = 4;
  if (n18[S] >= 0) {
    if constexpr (DIL != 0) DwI8RingFast<S, NT, C, T, DIL>(aq, lda, row0a, dq8, LD, blob, p.dw, ring, n18[S], active);
    else if (dil_rt == 3) DwI8RingFast<S, NT, C, T, 3>(aq, lda, row0a, dq8, LD, blob, p.dw, ring, n18[S], active);
    else DwI8RingFast<S, NT, C, T, 9>(aq, lda, row0a, dq8, LD, blob, p.dw, ring, n18[S], active);
  } else {
    DwI8Ring<S, NT>(aq, lda, row0a, dq8, LD, C, T, dil_rt, blob, p.dw, ring, n18, active);
  }
  {
    const RequantLutPack epi(blob, p.pw1, p.lr1);
    GemmI8Mma<S, NT, NTW, PDI>(dq8, LD, 0, 1, 1, C, 1, T, C, BlobPtr<uint2>(blob, p.pw1.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) { hq[(size_t)(n0 / 4) * LD + t * S + s] = epi(acc, n0); });
  }
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
}

// quant_{en,de}coder resnet_1 and resnet_2 (dilation 3, 9; ring blocks of 6 and 18 rows back to back) as one copy of the code
template <int S, int NT, int PDI = kI8Pd>
__device__ __forceinline__ void ResUnitsI8x2(const uint8_t* blob, const ResI8* p2, uint32_t* aq, int lda, int row0a,
                                             uint32_t* resq, uint32_t* dq8, uint32_t* hq, uint32_t* ring0,
                                             const int* n18, const int* active) {
#pragma unroll 1
  for (int i = 0; i < 2; ++i)
    ResUnitI8<S, NT, 0, PDI>(blob, p2[i], aq, lda, row0a, resq, dq8, hq, ring0 + (size_t)(i ? 64 * 6 : 0) * S, n18, active, i ? 9 : 3);
}

// ================================================================================================
//                                        ENCODER  A
// ================================================================================================
struct EncA {
  static constexpr int S = kTileStreams;
  static constexpr int NT = 320;
  static constexpr int TN = 4;
  static constexpr int kMinBlocks = 2;
  static constexpr int LDU = 25 * S, LDD = 20 * S;
  static constexpr int kStgDown = 5;                      // ring depth of encoder_0/simpleconv (ring = the d buffer)
  // encoder_0/simpleconv has 4 output rows x S streams = 32 GEMM rows only: its DTM x DTN thread tiles decide how many of the
  // block's ten warps get a tile (8 x 4: four warps)
  static constexpr int DTM = 8, DTN = 4;
  static constexpr int kSmemU = 0;
  static constexpr int kSmemD = kSmemU + 64 * LDU * 4;
  static constexpr int kSmemW = kSmemD + 64 * LDD * 4;
  static constexpr int kSmemI = kSmemW + kStages * 16 * 64 * 4;   // ring of the 64-channel layers (simpleconv's ring lives in d)
  static constexpr int kSmemBytes = kSmemI + 3 * S * 4 + 16;
  static_assert(391 * S <= 64 * LDD, "first-layer input (368 rows + 23 skew rows) must fit in the d buffer");
};

__global__ void __launch_bounds__(EncA::NT, EncA::kMinBlocks)
EncoderKernelA(const uint8_t* __restrict__ blob, EncoderParams P, TileIo io, const int16_t* __restrict__ pcm,
               float* __restrict__ state, int* __restrict__ n18g, float* __restrict__ mid) {
  using L = EncA;
  constexpr int S = L::S, NT = L::NT;
  unsigned char* smem = LYRA_DYN_SMEM();
  float* u = reinterpret_cast<float*>(smem + L::kSmemU);
  float* d = reinterpret_cast<float*>(smem + L::kSmemD);
  float* wbuf = reinterpret_cast<float*>(smem + L::kSmemW);
  int* slot = reinterpret_cast<int*>(smem + L::kSmemI);
  int* active = slot + S;
  int* n18 = active + S;
  int tile;
  InitWeightPipe<NT>();
  if (!BeginTile<S>(io, n18g, slot, state, EncStateA::kUnits, tile)) return;
  float* st = state + (size_t)tile * EncStateA::kUnits * S;
  const int tid = (int)threadIdx.x;
  IssuePrologue<NT>(wbuf, NextF32(BlobPtr<float>(blob, P.first.w), 16, 64, 64));

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
  static_assert(EncStateA::kRing1 == EncStateA::kRing0 + 64 * 2 && EncStateA::kRing2 == EncStateA::kRing1 + 64 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, 8, L::TN, L::TN, 4, 16, 64, EncStateA::kT>(blob, P.r0, u, L::LDU, 5, d, 1, st + (size_t)EncStateA::kRing0 * S, n18, active, wbuf,
                                                       NextF32(BlobPtr<float>(blob, P.down0.w), 16, 128, 640, d, L::kStgDown));
  // carried rows for the next frame: the last 5 activated rows
  StoreCarriedRows<S, NT, 64, 5>(st, EncStateA::kDown0, u, L::LDU, 20, active);
  // ---- encoder_0/simpleconv: K = 10, stride 5, 64 -> 128 ; pre-activation output to HBM for kernel B
  {
    const float* b = BlobPtr<float>(blob, P.down0.bias);
    float* out = mid + (size_t)tile * 128 * 4 * S;
    // the d buffer is free from here on: it hosts this GEMM's weight ring (kStgDown x 16 x 128 floats).  With 32 GEMM rows a chunk is
    // consumed in a fraction of the L2 round trip, so the ring is as deep as d allows.
    static_assert(L::kStgDown * 16 * 128 * 4 <= 64 * L::LDD * 4, "simpleconv weight ring must fit in d");
    constexpr int DTM = L::DTM, DTN = L::DTN;
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
  AdvanceHopCounters<S>(n18g, tile, active, n18);
}

// ================================================================================================
//                                        ENCODER  B
// ================================================================================================
struct EncB {
  static constexpr int S = kTileStreams;
  static constexpr int NT = 256;
  static constexpr int kMinBlocks = 3;                    // resident blocks per SM (72 KB of shared memory each)
  static constexpr int TM = 8;                            // streams per fp32 thread tile (8 x 4 tiles: fewer smem wavefronts per FMA)
  static constexpr int TN = 4;                            // output channels per fp32 thread tile
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
  static constexpr int kRA = 0;
  static constexpr int kRABytes = kMax(kMax(128 * LD1 * 4, 256 * 2 * S * 4), 64 * LQA * 4 + 128 * LQB * 4);
  static constexpr int kRB = kRA + kRABytes;
  static constexpr int kRBBytes = kMax(128 * 4 * S * 4, 256 * 2 * S * 4);
  static constexpr int kRC = kRB + kRBBytes;
  static constexpr int kW = kRC + 64 * LQ2 * 4;
  // ring depth of the kernel's fp32 GEMMs.  Deeper rings, borrowing the regions that are dead during the K loops, were slower before
  // the H100 port: with three blocks per SM the GEMM phases are bound by shared-memory operand delivery (not re-measured on the H100).
  static constexpr int kStg = 3;
  static constexpr int kWBytes = kMax(kStg * 8 * 256 * 4, 2 * 64 * LQ2 * 4);
  static constexpr int kI8Pd = 4;                         // k-steps of int8 weight fragments in flight from L2
  static constexpr int kI = kW + kWBytes;
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;
};

__global__ void __launch_bounds__(EncB::NT, EncB::kMinBlocks)
EncoderKernelB(const uint8_t* __restrict__ blob, EncoderParams P, TileIo io, const float* __restrict__ mid,
               float* __restrict__ state, int* __restrict__ n18g, float* __restrict__ features) {
  using L = EncB;
  constexpr int S = L::S, NT = L::NT;
  constexpr int TM = L::TM, TN = L::TN;
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
  if (!BeginTile<S>(io, n18g, slot, state, EncStateB::kUnits, tile)) return;
  float* st = state + (size_t)tile * EncStateB::kUnits * S;
  uint32_t* stw = reinterpret_cast<uint32_t*>(st);
  IssuePrologue<NT>(wbuf, NextF32(BlobPtr<float>(blob, P.r1[0].pw1.w), 16, 128, 128, nullptr, L::kStg));

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
  static_assert(EncStateB::kRing1 == EncStateB::kRing0 + 128 * 2 && EncStateB::kRing2 == EncStateB::kRing1 + 128 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, TM, TN, TN, L::WM4, 16, 128, EncStateB::kT1, false, 4 * S, 1, 1, L::kStg>(
      blob, P.r1, u1, L::LD1, 2, d1, 2, st + (size_t)EncStateB::kRing0 * S, n18, active, wbuf,
      NextF32(BlobPtr<float>(blob, P.down1.w), 8, 256, 256, wbuf, L::kStg));
  StoreCarriedRows<S, NT, 128, 2>(st, EncStateB::kDown1, u1, L::LD1, 4, active);
  // ---- encoder_1/simpleconv: K = 4, stride 2, 128 -> 256, 2 groups ; u2 = pre-activation
  {
    const float* b = BlobPtr<float>(blob, P.down1.bias);
    GemmF32Tap<S, NT, TM, TN, 8, L::WM2, false, L::kStg>(u1, L::LD1, 0, 2, 4, 64, 2, 2, 256, BlobPtr<float>(blob, P.down1.w), wbuf, true,
      NextF32(BlobPtr<float>(blob, P.m_pw1.w), 8, 256, 256, wbuf, L::kStg),
      [&](int t, int s0, int n0, float (&acc)[TM][TN]) {
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          float* o = u2 + (size_t)(n0 + j) * 2 * S + t * S + s0;
#pragma unroll
          for (int i = 0; i < TM; ++i) o[i] = __fadd_rn(acc[i][j], b[n0 + j]);
        }
      });
  }
  // ---- encoder_2/resnet_0 (mixed): f32 depthwise + f32 1x1, QUANTIZE, int8 LeakyReLU, int8 1x1 (4 groups),
  //      DEQUANTIZE + f32 residual, QUANTIZE, int8 LeakyReLU
  constexpr int LD2 = 2 * S;
  if (n18[S] >= 0)
    DwF32RingFast<S, NT, 256, EncStateB::kT2, 1>(u2, LD2, 0, d2, LD2, BlobPtr<float>(blob, P.m_dw.w), BlobPtr<float>(blob, P.m_dw.bias),
                                    st + (size_t)EncStateB::kRingM * S, n18[S], active);
  else
    DwF32Ring<S, NT>(u2, LD2, 0, d2, LD2, 256, EncStateB::kT2, 1, BlobPtr<float>(blob, P.m_dw.w), BlobPtr<float>(blob, P.m_dw.bias),
                     st + (size_t)EncStateB::kRingM * S, n18, active);
  {
    const float* b = BlobPtr<float>(blob, P.m_pw1.bias);
    const int8_t* lut = BlobPtr<int8_t>(blob, P.m_lr1.lut);
    const QuantP q1 = P.m_q1;
    static_assert(TN == 4, "the epilogue packs one word of four channels per (row, stream)");
    GemmF32Tap<S, NT, TM, TN, 8, L::WM2, false, L::kStg>(d2, LD2, 0, 1, 1, 256, 1, 2, 256, BlobPtr<float>(blob, P.m_pw1.w), wbuf, true,
      NoNext(),
      [&](int t, int s0, int n0, float (&acc)[TM][TN]) {
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          int q[TN];
#pragma unroll
          for (int j = 0; j < TN; ++j) q[j] = lut[QuantizeF32(__fadd_rn(acc[i][j], b[n0 + j]), q1.scale, q1.zp) + 128];
          // channels 4k .. 4k+3 of one (row, stream), byte j = channel 4k + j
          hq[(size_t)(n0 / 4) * LQ2 + t * S + s0 + i] = PackI8x4(q[0], q[1], q[2], q[3]);
        }
      });
  }
  MixedUnitPw2I8<S, NT, L::kI8Pd>(blob, P, hq, u2, resq, aq, LQA, 2);
  // ---- quant_encoder_2/resnet_{1,2}
  static_assert(EncStateB::kRingQ1 == EncStateB::kRingQ0 + 64 * 6, "ring blocks back to back");
  ResUnitsI8x2<S, NT, L::kI8Pd>(blob, P.q, aq, LQA, 2, resq, dq8, hq, stw + (size_t)EncStateB::kRingQ0 * S, n18, active);
  // ---- quant_encoder_2/simpleconv: K = 4, stride 2, 256 -> 512, 4 groups, then int8 LeakyReLU
  BatchedLoop<NT, 4, uint32_t>(64 * 2 * S, [&](int i) { return stw[EncStateB::kDown2 * S + i]; },
    [&](int i, uint32_t v) { const int c = i / (2 * S), r = i % (2 * S); aq[(size_t)c * LQA + r] = v; });
  BatchedLoop<NT, 8, uint32_t>(128 * 2 * S, [&](int i) { return stw[EncStateB::kBott * S + i]; },
    [&](int i, uint32_t v) { const int c = i / (2 * S), r = i % (2 * S); bq[(size_t)c * LQB + r] = v; });
  __syncthreads();
  StoreCarriedRows<S, NT, 64, 2>(stw, EncStateB::kDown2, aq, LQA, 2, active);
  {
    const RequantLutPack epi(blob, P.down2, P.down2_lr);
    GemmI8Mma<S, NT, 8, L::kI8Pd>(aq, LQA, 0, 2, 4, 64, 4, 1, 512, BlobPtr<uint2>(blob, P.down2.w),
      [&](int, int s, int n0, int (&acc)[1][4]) { bq[(size_t)(n0 / 4) * LQB + 2 * S + s] = epi(acc, n0); });
  }
  // carried rows of quant_bottleneck_1: the two newest rows
  StoreCarriedRows<S, NT, 128, 2>(stw, EncStateB::kBott, bq, LQB, 1, active);
  // ---- quant_bottleneck_1: K = 3, 512 -> 64, 4 groups ; DEQUANTIZE -> features
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
  AdvanceHopCounters<S>(n18g, tile, active, n18);
}

// ================================================================================================
//                                        DECODER  C
// ================================================================================================
template <bool TC = false>
struct DecC {
  static constexpr int S = kTileStreams;
  static constexpr int NT = 256;
  static constexpr int kMinBlocks = 3;                    // resident blocks per SM (59 KB of shared memory each)
  static constexpr int kI8Pd = 2;                         // prefetch depth of the four-n-tile int8 GEMMs (the eight-n-tile upsamplers
                                                          // take GemmI8Mma's default)
  static constexpr int TM = 8;                            // streams per fp32 thread tile (8 x 4 tiles: fewer smem wavefronts per FMA)
  static constexpr int TN = 4;                            // output channels per fp32 thread tile (decoder_1)
  static constexpr int WM4 = 4 * S / TM >= 4 ? 4 : 4 * S / TM;   // m-groups per warp for T = 4 / 2 / 1 row layers
  static constexpr int WM2 = 2 * S / TM >= 4 ? 4 : 2 * S / TM;
  static constexpr int WM1 = 1 * S / TM >= 4 ? 4 : 1 * S / TM;
  static constexpr int LQ2 = PadLd(2 * S), LQA = PadLd(4 * S), LQB = PadLd(3 * S);   // padded int8 word strides (MMA A operand)
  // Shared memory is reused along the layer sequence (59 KB at S = 8, so three blocks share an SM):
  //   region 1: F f32 [64][3S] + xq words [128][LQB]  ->  aq words [64][LQA]  ->  d1 f32 [128][4S]
  //   region 2: u f32 [256][2S]  ->  u1 f32 [128][4S]
  //   region W: fp32 weight ring (bottleneck_2, decoder_1)  <->  hq, dq8, resq words [64][LQ2] each (int8 phases)
  static constexpr int kF = 0;
  static constexpr int kXq = kF + 64 * 3 * S * 4;
  // tensor-core mode: d1 is an MMA A operand (padded stride); decoder_1 warp tiles: 2 m-tiles x RWN n-tiles
  static constexpr int LD1 = TC ? PadLd(4 * S) : 4 * S;
  static constexpr int RWM = 2, RWN = 2;
  static_assert(!TC || ((4 * S + 31) / 32) * (16 / RWN) <= NT / 32, "decoder_1: one warp tile per warp");
  static constexpr int kR1Bytes = kMax(kMax(64 * 3 * S * 4 + 128 * LQB * 4, 64 * LQA * 4), 128 * LD1 * 4);
  static constexpr int kU = kF + kR1Bytes;
  static constexpr int kW = kU + 256 * 2 * S * 4;
  static constexpr int kWBytes = kMax(kStages * 4 * 512 * 4, 3 * 64 * LQ2 * 4);
  static constexpr int kI = kW + kWBytes;
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;
};

template <bool TC>
__global__ void __launch_bounds__(DecC<TC>::NT, DecC<TC>::kMinBlocks)
DecoderKernelC(const uint8_t* __restrict__ blob, DecoderParams P, TileIo io,
               const float* __restrict__ features, float* __restrict__ state, int* __restrict__ n18g,
               float* __restrict__ mid) {
  using L = DecC<TC>;
  constexpr int S = L::S, NT = L::NT;
  constexpr int TM = L::TM, TN = L::TN;
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
  if (!BeginTile<S>(io, n18g, slot, state, DecStateC::kUnits, tile)) return;
  uint32_t* stw = reinterpret_cast<uint32_t*>(state) + (size_t)tile * DecStateC::kUnits * S;
  float* st = reinterpret_cast<float*>(stw);
  const int tid = (int)threadIdx.x;
  constexpr int LD2 = 2 * S;
  const UpI8& up0 = P.up0;
  const UpI8& up1 = P.up1;
  IssuePrologue<NT>(wbuf, NextF32(BlobPtr<float>(blob, P.bott.w), 4, 512, 48));

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
  StoreCarriedRows<S, NT, 64, 2>(st, DecStateC::kBott, F, 3 * S, 1, active);
  // ---- bottleneck_2/simpleconv: K = 3, 64 -> 512, 4 groups ; LeakyReLU ; QUANTIZE
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
  if (n18[S] >= 0) DwI8RingFast<S, NT, 256, DecStateC::kT0, 1>(aq, LQA, 1, dq8, LQ2, blob, P.m_dw, stw + (size_t)DecStateC::kRingM * S, n18[S], active);
  else DwI8Ring<S, NT>(aq, LQA, 1, dq8, LQ2, 256, DecStateC::kT0, 1, blob, P.m_dw, stw + (size_t)DecStateC::kRingM * S, n18, active);
  {
    const RequantLutPack epi(blob, P.m_pw1, P.m_lr1);
    GemmI8Mma<S, NT, 4, L::kI8Pd>(dq8, LQ2, 0, 1, 1, 256, 1, 2, 256, BlobPtr<uint2>(blob, P.m_pw1.w),
      [&](int t, int s, int n0, int (&acc)[1][4]) { hq[(size_t)(n0 / 4) * LQ2 + t * S + s] = epi(acc, n0); });
  }
  MixedUnitPw2I8<S, NT, L::kI8Pd>(blob, P, hq, u, resq, aq, LQA, 1);
  static_assert(DecStateC::kRingQ1 == DecStateC::kRingQ0 + 64 * 6, "ring blocks back to back");
  ResUnitsI8x2<S, NT, L::kI8Pd>(blob, P.q, aq, LQA, 1, resq, dq8, hq, stw + (size_t)DecStateC::kRingQ0 * S, n18, active);
  // ---- quant_decoder_1 upsample: 2 x TRANSPOSE_CONV (K = 4, stride 2, 128 -> 64), T 2 -> 4 (+2 tail rows)
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
  static_assert(DecStateC::kRing1 == DecStateC::kRing0 + 128 * 2 && DecStateC::kRing2 == DecStateC::kRing1 + 128 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, TM, TN, TN, L::WM4, 16, 128, DecStateC::kT1, TC, L::LD1, L::RWM, L::RWN>(
      blob, P.r1, u1, 4 * S, 0, d1, 2, st + (size_t)DecStateC::kRing0 * S, n18, active, wbuf, NoNext());
  {
    float* out = mid + (size_t)tile * 128 * 4 * S;
    for (int i = tid; i < 128 * 4 * S; i += NT) out[i] = u1[i];
  }
  AdvanceHopCounters<S>(n18g, tile, active, n18);
}

// ================================================================================================
//                                        DECODER  D
// ================================================================================================
// The exact decoder mode's kernel D (fp32 FMA chains, bit-exact with the oracle); the tensor mode runs DecoderKernelDW
// (net_kernels_wgmma.cuh) instead.
struct DecD {
  static constexpr int S = kTileStreams;
  static constexpr int NT = 320;
  static constexpr int TN = 4;
  static constexpr int kMinBlocks = 2;
  static constexpr int TNU = 5;                           // decoder_2/simple column tile (320 columns)
  static constexpr int TNL = 2;                           // last_layer column tile (16 columns)
  static constexpr int WML = 4;
  static constexpr int WMU = 1;
  static constexpr int KCU = 8;                           // its ring starts right behind X inside d and runs into the regular ring
  static constexpr int LDU = 26 * S, LDD = 20 * S, LDX = 6 * S;   // u: 3 zero rows + 20 + 3 zero rows
  static constexpr int kU = 0;
  static constexpr int kD = kU + 64 * LDU * 4;              // d f32 [64][LDD]; aliases X f32 [128][LDX] and the PCM staging
  static constexpr int kW = kD + 64 * LDD * 4;
  static constexpr int kWBytes = kStages * 16 * 64 * 4 + 2048;   // regular ring (64-channel layers) + slack for the decoder_2/simple ring
  static constexpr int kSl = kW + kWBytes;                  // carried tail of last_layer [48][S]
  static_assert(128 * 6 * S * 4 + kStages * KCU * 320 * 4 <= 64 * LDD * 4 + kWBytes, "decoder_2/simple ring must fit behind X");
  static constexpr int kI = kSl + 48 * S * 4;
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;
  static_assert(128 * LDX <= 64 * LDD, "X must fit in d");
  static_assert(S * 320 * 2 <= 64 * LDD * 4, "PCM staging must fit in d");
};

__global__ void __launch_bounds__(DecD::NT, DecD::kMinBlocks)
DecoderKernelD(const uint8_t* __restrict__ blob, DecoderParams P, TileIo io, const float* __restrict__ mid,
               float* __restrict__ state, int* __restrict__ n18g, int16_t* __restrict__ pcm) {
  using L = DecD;
  constexpr int S = L::S, NT = L::NT;
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
  if (!BeginTile<S>(io, n18g, slot, state, DecStateD::kUnits, tile)) return;
  float* st = state + (size_t)tile * DecStateD::kUnits * S;
  const int tid = (int)threadIdx.x;
  constexpr int LDX = L::LDX;
  float* wbuf_up2 = X + 128 * LDX;       // free tail of d + the regular ring
  IssuePrologue<NT>(wbuf_up2, NextF32(BlobPtr<float>(blob, P.up2.w), L::KCU, 320, 256));

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
    GemmF32Tap<S, NT, 8, L::TNU, L::KCU, L::WMU, false>(X, LDX, 0, 1, 2, 128, 1, 5, 320, BlobPtr<float>(blob, P.up2.w), wbuf_up2, true,
                                                        NextF32(BlobPtr<float>(blob, P.r2[0].pw1.w), 16, 64, 64, wbuf), epi_up);
  }
  // ---- decoder_2: three residual units @64, T = 20
  static_assert(DecStateD::kRing1 == DecStateD::kRing0 + 64 * 2 && DecStateD::kRing2 == DecStateD::kRing1 + 64 * 6, "ring blocks back to back");
  ResUnitsF32x3<S, NT, 8, L::TN, L::TN, 4, 16, 64, DecStateD::kT>(blob, P.r2, u, L::LDU, 3, d, 1, st + (size_t)DecStateD::kRing0 * S, n18, active, wbuf,
                                                       NextF32(BlobPtr<float>(blob, P.last.w), 16, 16, 256));
  // ---- last_layer: TRANSPOSE_CONV K = 64, stride 16, 64 -> 1 ; T 20 -> 320 (+48 tail) ; float -> int16
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
    GemmF32Tap<S, NT, 8, L::TNL, 16, L::WML, false>(u, L::LDU, 0, 1, 4, 64, 1, 23, 16, BlobPtr<float>(blob, P.last.w), wbuf, true, NoNext(), epi_last);
    for (int i = tid; i < S * 320; i += NT) {
      const int s = i / 320;
      if (active[s]) pcm[(size_t)slot[s] * 320 + (i % 320)] = stage[i];
    }
  }
  AdvanceHopCounters<S>(n18g, tile, active, n18);
}

}  // namespace lyra_b200
