// Device primitives shared by the four conv-net kernels.
//
// Data layout (one thread block = one tile of S streams):
//   fp32 activations in shared memory:  act[c * ld + row * S + s]     (channel-major, stream-minor)
//   int8 activations in shared memory:  word[(c/4) * ld + row * S + s] (4 consecutive channels / word)
// so every convolution tap is a row offset, every thread owns TM consecutive streams of one output
// row and TN consecutive output channels, and both operands of the inner product are 16-byte
// shared-memory loads.  Weights stream from L2 through a cp.async double buffer.
//
// Bit-exactness contract (matches oracle/net_interp.c): each fp32 output is ONE fmaf chain over
// (tap ascending, cin ascending) starting from +0, bias added afterwards with a separate rounding;
// all other fp32 ops use the non-contracting __f*_rn intrinsics.
#pragma once

#include "device_compat.h"
#include "net_params.h"

// Weight fragments that a block reads exactly once (straight from L2 into registers).  Experiment switch LYRA_FRAG_NOALLOC: bit 0
// (int8) / bit 1 (TF32) load them without allocating an L1 line (measured slower: co-resident blocks of the same kernel find each
// other's fragments in the L1); + 4 loads them with the evict-last L1 policy instead.
#ifndef LYRA_FRAG_NOALLOC
#define LYRA_FRAG_NOALLOC 0
#endif
template <bool NOALLOC>
__device__ __forceinline__ uint2 LoadFrag(const uint2* p) {
#if defined(LYRA_EMU)
  return *p;
#else
  if (NOALLOC) {
    uint2 v;
#if LYRA_FRAG_NOALLOC >= 4
    asm volatile("ld.global.nc.L1::evict_last.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "l"(p));
#else
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "l"(p));
#endif
    return v;
  }
  return __ldg(p);
#endif
}
template <bool NOALLOC>
__device__ __forceinline__ float2 LoadFrag(const float2* p) {
#if defined(LYRA_EMU)
  return *p;
#else
  if (NOALLOC) {
    float2 v;
#if LYRA_FRAG_NOALLOC >= 4
    asm volatile("ld.global.nc.L1::evict_last.v2.f32 {%0, %1}, [%2];\n" : "=f"(v.x), "=f"(v.y) : "l"(p));
#else
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];\n" : "=f"(v.x), "=f"(v.y) : "l"(p));
#endif
    return v;
  }
  return __ldg(p);
#endif
}

// register prefetch depth (k-steps) of the int8 B fragments that GemmI8Mma takes straight from L2.  Deeper prefetch spills a few
// registers at 80 per thread; before the H100 port kernel B gained with 4 and kernel C lost (not re-measured on the H100)
#ifndef LYRA_I8_PD
#define LYRA_I8_PD 2
#endif
#ifndef LYRA_B_I8_PD
#define LYRA_B_I8_PD 4
#endif
#ifndef LYRA_C_I8_PD
#define LYRA_C_I8_PD 2
#endif

namespace lyra_b200 {

template <typename T>
__device__ __forceinline__ const T* BlobPtr(const uint8_t* blob, uint32_t off) {
  return reinterpret_cast<const T*>(blob + off);
}

// LeakyReLU(0.3): v > 0 ? v : 0.3 v.  For a slope below one that is max(v, 0.3 v) - one multiply and one FMNMX instead of a
// compare, a multiply and a select - with the same result for every input (0.3 v < v for v > 0, > v for v < 0, -0 stays -0).
__device__ __forceinline__ float LeakyRelu(float v) { return fmaxf(v, __fmul_rn(v, 0.3f)); }

// TFLite reference AffineQuantize: round-half-away(v / scale) + zp, clamped to int8
__device__ __forceinline__ int QuantizeF32(float v, float scale, int zp) {
  int q = (int)roundf(__fdiv_rn(v, scale)) + zp;
  q = q < -128 ? -128 : (q > 127 ? 127 : q);
  return q;
}
__device__ __forceinline__ float DequantizeI8(int q, float scale, int zp) { return __fmul_rn(scale, (float)(q - zp)); }

// gemmlowp MultiplyByQuantizedMultiplier (SaturatingRoundingDoublingHighMul + RoundingDivideByPOT), branch-free:
//   SRDHM   trunc((ab + (ab >= 0 ? 2^30 : 1 - 2^30)) / 2^31) == floor((ab + 2^30) / 2^31) for either sign of ab
//           (ab < 0: trunc(t / 2^31) = floor((t + 2^31 - 1) / 2^31) with t = ab + 1 - 2^30);
//   RDBPOT  (x >> e) + ((x & mask) > (mask >> 1) + (x < 0)) == (x + 2^(e-1) - (x < 0)) >> e for e >= 1, x for e = 0.
// Same integers as the oracle's literal restatement (oracle/net_interp.c) for every int32 accumulator and positive multiplier.
__device__ __forceinline__ int Mbqm(int x, int qm, int shift) {
  const int left = shift > 0 ? shift : 0, right = shift > 0 ? 0 : -shift;
  const long long ab = (long long)(int)((unsigned)x << left) * (long long)qm;
  const int hi = (int)((ab + (1ll << 30)) >> 31);
  const int half = (int)((1u << right) >> 1);
  return right ? (hi + half + (hi >> 31)) >> right : hi;
}
__device__ __forceinline__ int ClampI8(int v) { return v < -128 ? -128 : (v > 127 ? 127 : v); }
__device__ __forceinline__ int RequantI8(int acc, int bias, int mult, int shift, int out_zp) {
  return ClampI8(Mbqm(acc + bias, mult, shift) + out_zp);
}
// requantisation parameters of four consecutive output channels (n0 % 4 == 0; the blob's arrays are 16-byte aligned): three
// 16-byte loads instead of twelve scalar ones in every int8 epilogue
struct RequantP4 { int b[4], m[4], s[4]; };
__device__ __forceinline__ RequantP4 LoadRequant4(const int* __restrict__ bias, const int* __restrict__ mult, const int* __restrict__ shift, int n0) {
  const int4 b = *reinterpret_cast<const int4*>(bias + n0), m = *reinterpret_cast<const int4*>(mult + n0), s = *reinterpret_cast<const int4*>(shift + n0);
  return RequantP4{{b.x, b.y, b.z, b.w}, {m.x, m.y, m.z, m.w}, {s.x, s.y, s.z, s.w}};
}
__device__ __forceinline__ uint32_t PackI8x4(int a, int b, int c, int d) {
  return (uint32_t)(a & 0xff) | ((uint32_t)(b & 0xff) << 8) | ((uint32_t)(c & 0xff) << 16) | ((uint32_t)(d & 0xff) << 24);
}
__device__ __forceinline__ int UnpackI8(uint32_t w, int i) { return (int)(int8_t)((w >> (8 * i)) & 0xff); }

// ------------------------------------------------------------------------------------------------
// Element-wise loop whose loads are batched: every thread first issues up to U independent loads (one exposed
// memory latency instead of U), then runs the stores.  ld(i) -> T, st(i, T).
template <int NT, int U, typename T, typename LoadFn, typename StoreFn>
__device__ __forceinline__ void BatchedLoop(int n, LoadFn ld, StoreFn st) {
  for (int i0 = (int)threadIdx.x; i0 < n; i0 += NT * U) {
    T v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) { const int i = i0 + k * NT; if (i < n) v[k] = ld(i); }
#pragma unroll
    for (int k = 0; k < U; ++k) { const int i = i0 + k * NT; if (i < n) st(i, v[k]); }
  }
}

// ------------------------------------------------------------------------------------------------
// Weight pipeline of the fp32 GEMMs: a ring of kStages chunk buffers in shared memory filled by bulk asynchronous
// copies (TMA, cp.async.bulk) that one elected thread issues, with a full / empty mbarrier pair per stage.  Consumer
// warps wait on `full`, compute, and release the stage with one arrival per warp on `empty`; the producer refills a
// stage once every warp has released it.  No block-wide barrier inside the K loop: warps drift up to kStages - 1
// chunks apart instead of meeting at every chunk.
// Two barrier sets alternate between consecutive GEMMs so that the first chunks of the NEXT GEMM can be issued
// (into the other set) before the current GEMM's epilogue; each GEMM re-initialises the set its successor will use.
constexpr int kStages = 3;       // default ring depth; a GEMM may ask for more (template parameter STG, at most kMaxStages)
constexpr int kMaxStages = 8;

struct WeightPipe {
  LyraMbar full[2][kMaxStages];
  LyraMbar empty[2][kMaxStages];
  int cur;          // barrier set of the next GEMM to run (or of the prologue issued for it)
};

__device__ __forceinline__ WeightPipe* GetWeightPipe() {
  LYRA_STATIC_SMEM(WeightPipe, pipe, 1);
  return pipe;
}

__device__ __forceinline__ void InitPipeSet(WeightPipe* pipe, int set, int nwarps) {
#pragma unroll
  for (int s = 0; s < kMaxStages; ++s) { lyra_mbar_init(&pipe->full[set][s], 1); lyra_mbar_init(&pipe->empty[set][s], (unsigned)nwarps); }
  lyra_mbar_fence_init();
}

// Once per kernel, by every thread, before the first block barrier of the kernel.
template <int NT>
__device__ __forceinline__ void InitWeightPipe() {
  WeightPipe* pipe = GetWeightPipe();
  if (threadIdx.x == 0) {
    InitPipeSet(pipe, 0, NT / 32);
    InitPipeSet(pipe, 1, NT / 32);
    pipe->cur = 0;
  }
}

// Description of a GEMM's weight stream, used to issue its first kStages-1 chunks EARLY (right after the previous
// GEMM's K loop, before that GEMM's epilogue and any element-wise pass in between) so the L2 latency of the
// first chunk is never exposed.
struct WNext {
  const void* w;      // global weights (nullptr: nothing to prefetch)
  int chunk_words;    // 4-byte words per chunk (KC * N)
  int nchunks;
  void* ring;         // shared-memory ring of the next GEMM when it is not the caller's (nullptr: same ring)
  int stages;         // ring depth of the next GEMM (its STG)
};
__device__ __forceinline__ WNext NoNext() { return WNext{nullptr, 0, 0, nullptr, kStages}; }
__device__ __forceinline__ WNext NextF32(const float* w, int KC, int N, int Ktot, void* ring = nullptr, int stages = kStages) {
  return WNext{w, KC * N, Ktot / KC, ring, stages};
}

// Thread 0: chunks 0 .. stages-2 of a GEMM into barrier set `set` (whose buffers and barriers are idle).
__device__ __forceinline__ void IssuePrologueSet(WeightPipe* pipe, int set, void* wbuf, const void* w, int chunk_words, int nchunks,
                                                 int stages = kStages) {
#pragma unroll
  for (int p = 0; p < kMaxStages - 1; ++p)
    if (p < stages - 1 && p < nchunks)
      lyra_bulk_g2s(reinterpret_cast<uint32_t*>(wbuf) + (size_t)p * chunk_words,
                    reinterpret_cast<const uint32_t*>(w) + (size_t)p * chunk_words, (unsigned)chunk_words * 4u, &pipe->full[set][p]);
}

// Start the weight stream of the GEMM that runs next (kernel prologue, or after a phase without fp32 GEMMs).
// Called by every thread: the ring may alias buffers that were written with ordinary stores, so every thread fences
// its stores against the asynchronous proxy and the block synchronises before the elected thread issues the copies.
template <int NT>
__device__ __forceinline__ void IssuePrologue(void* wbuf_default, const WNext& nx) {
  if (nx.w == nullptr) return;
  lyra_fence_proxy_async();
  __syncthreads();
  if (threadIdx.x == 0) {
    WeightPipe* pipe = GetWeightPipe();
    IssuePrologueSet(pipe, pipe->cur, nx.ring ? nx.ring : wbuf_default, nx.w, nx.chunk_words, nx.nchunks, nx.stages);
  }
}

// Thread -> output tile mapping.  A warp covers WM m-groups x (32/WM) n-groups so that the A fragment is
// shared by the lanes of one m-group and the W fragment by the lanes of one n-group (shared-memory
// broadcast); warp tiles beyond NT/32 warps are handled in extra passes.
template <int WM>
struct TileMap {
  int MGB, NGB, nwt;
  __device__ __forceinline__ TileMap(int MG, int NG) {
    MGB = (MG + WM - 1) / WM;
    NGB = (NG + (32 / WM) - 1) / (32 / WM);
    nwt = MGB * NGB;
  }
  __device__ __forceinline__ bool Locate(int wt, int MG, int NG, int& mg, int& ng) const {
    const int lane = (int)threadIdx.x & 31;
    mg = (wt % MGB) * WM + lane % WM;
    ng = (wt / MGB) * (32 / WM) + lane / WM;
    return wt < nwt && mg < MG && ng < NG;
  }
};

// ------------------------------------------------------------------------------------------------
// fp32 tap-GEMM.   out[t][s][n] = sum_{tap < ntaps} sum_{ci < CinG} A[g*CinG + ci][rowA0 + t*row_stride + tap][s] * W[tap*CinG + ci][n]
//   A: shared memory [channels][ldA]; if CIN1 the K loop runs over taps only (CinG == 1, single channel).
//   W: global [ntaps*CinG][N];  wbuf: shared kStages * KC * N floats.
//   Thread tile TM (streams) x TN (channels).
//   epi(t, s0, n0, acc) is called once per tile after the K loop and a block barrier, so epilogues may
//   overwrite the A operand in place.
template <int S, int NT, int TM, int TN, int KC, int WM, bool CIN1, int STG = kStages, typename Epi>
__device__ __forceinline__ void GemmF32Tap(const float* A, int ldA, int rowA0, int row_stride, int ntaps, int CinG,
                                           int groups, int T_out, int N, const float* __restrict__ Wg, float* wbuf,
                                           bool pre, const WNext& nxt, Epi epi) {
  static_assert(S % TM == 0 && TM % 4 == 0 && 32 % WM == 0, "tile shape");
  constexpr int MGS = S / TM;
  const int MG = T_out * MGS, NG = N / TN;
  const TileMap<WM> map(MG, NG);
  const int Ktot = ntaps * CinG, nchunks = Ktot / KC;
  const int CoutG = N / groups;
  const int warp = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  WeightPipe* pipe = GetWeightPipe();
  const int set = pipe->cur;                                 // stable: written only between block barriers
  const int npass = (map.nwt + NT / 32 - 1) / (NT / 32);
  const int total = npass * nchunks;                         // chunk sequence of the whole call: every pass re-streams W
  const unsigned chunk_bytes = (unsigned)(KC * N) * 4u;
  static_assert(STG >= 2 && STG <= kMaxStages, "ring depth");
  if (nchunks < STG - 1) LYRA_TRAP();
  if (threadIdx.x == 0) {
    InitPipeSet(pipe, set ^ 1, NT / 32);                     // the set of the GEMM after this one (idle since the previous GEMM ended)
    if (!pre) IssuePrologueSet(pipe, set, wbuf, Wg, KC * N, nchunks, STG);
  }
  int cg = 0;                                                // chunk index within the call
  for (int wt0 = 0; wt0 < map.nwt; wt0 += NT / 32) {
    int mg, ng;
    const bool active = map.Locate(wt0 + warp, MG, NG, mg, ng);
    // Warps without a tile in this pass (small-M layers fill only part of the block) stay out of the K loop altogether: they
    // would only spin on the `full` barriers, taking issue slots from the warps that compute.  Warp 0 (always busy) releases
    // every stage on their behalf, so the `empty` barriers still see NT / 32 arrivals per phase.
    const int nbusy = min(NT / 32, map.nwt - wt0);
    const bool busy = warp < nbusy;
    const int t_out = active ? mg / MGS : 0, s0 = active ? (mg % MGS) * TM : 0, n0 = active ? ng * TN : 0;
    const int g = n0 / CoutG;
    const float* Abase = A + (size_t)(g * CinG) * ldA + (rowA0 + t_out * row_stride) * S + s0;
    // One IEEE round-to-nearest fma per (stream, channel) and k, in k order: the oracle's fmaf chain, bit for bit.
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

    if (!busy) cg += nchunks;
    for (int c = 0; busy && c < nchunks; ++c, ++cg) {
      if (threadIdx.x == 0) {
        // producer: chunk cg + STG - 1 goes into the stage that chunk cg - 1 occupied, once every warp has released it
        const int ci = cg + STG - 1;
        if (ci < total) {
          const int si = ci % STG;
          if (ci >= STG) lyra_mbar_wait(&pipe->empty[set][si], (unsigned)((ci / STG - 1) & 1));
          lyra_bulk_g2s(wbuf + (size_t)si * (KC * N), Wg + (size_t)(ci % nchunks) * KC * N, chunk_bytes, &pipe->full[set][si]);
        }
      }
      const int st = cg % STG;
      lyra_mbar_wait(&pipe->full[set][st], (unsigned)((cg / STG) & 1));      // chunk cg has landed
      if (active) {
        const float* wcur = wbuf + (size_t)st * (KC * N);
        const int kk0 = c * KC;
        const float* Ap;
        int astep;
        if (CIN1) { Ap = Abase + (kk0 + (kk0 >> 4)) * S; astep = S; }   // first_layer: rows skewed by one per 16 (KC == 16)
        else { const int tap = kk0 / CinG, ci0 = kk0 - tap * CinG; Ap = Abase + (size_t)ci0 * ldA + tap * S; astep = ldA; }
        const float* wp = wcur + n0;
#pragma unroll 4
        for (int kk = 0; kk < KC; ++kk) {
          float a[TM];
          float w[TN];
#pragma unroll
          for (int i = 0; i < TM; i += 4) {
            const float4 v = *reinterpret_cast<const float4*>(Ap + i);
            a[i] = v.x; a[i + 1] = v.y; a[i + 2] = v.z; a[i + 3] = v.w;
          }
          if (TN % 4 == 0) {
#pragma unroll
            for (int j = 0; j + 3 < TN; j += 4) {
              const float4 v = *reinterpret_cast<const float4*>(wp + j);
              w[j] = v.x; w[j + 1] = v.y; w[j + 2] = v.z; w[j + 3] = v.w;
            }
          } else if (TN % 2 == 0) {
#pragma unroll
            for (int j = 0; j + 1 < TN; j += 2) {
              const float2 v = *reinterpret_cast<const float2*>(wp + j);
              w[j] = v.x; w[j + 1] = v.y;
            }
          } else {
#pragma unroll
            for (int j = 0; j < TN; ++j) w[j] = wp[j];
          }
#pragma unroll
          for (int j = 0; j < TN; ++j)
#pragma unroll
            for (int i = 0; i < TM; ++i) acc[i][j] = __fmaf_rn(a[i], w[j], acc[i][j]);
          Ap += astep;
          wp += N;
        }
      }
      __syncwarp();
      if (lane == 0) {                                                           // this warp is done with the stage
        if (warp == 0 && nbusy < NT / 32) lyra_mbar_arrive_n(&pipe->empty[set][st], (unsigned)(1 + NT / 32 - nbusy));
        else lyra_mbar_arrive(&pipe->empty[set][st]);
      }
    }
    lyra_fence_proxy_async();   // this thread's earlier stores to buffers the next ring may alias, before the bulk copies below
    __syncthreads();   // every thread is past the K loop: A may be overwritten, the weight ring reused
    if (wt0 + NT / 32 >= map.nwt && threadIdx.x == 0) {
      // last pass: start the next GEMM's weight stream (other barrier set) and hand the pipe over to it
      if (nxt.w != nullptr) IssuePrologueSet(pipe, set ^ 1, nxt.ring ? nxt.ring : wbuf, nxt.w, nxt.chunk_words, nxt.nchunks, nxt.stages);
      pipe->cur = set ^ 1;
    }
    if (active) epi(t_out, s0, n0, acc);
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// int8 tap-GEMM on the tensor cores (mma.sync m16n8k32, s8 x s8 -> s32; exact integer arithmetic).
//   out[t][s][n] = sum_{tap} sum_{ci} A[g*CinG + ci][rowA0 + t*row_stride + tap][s] * W[tap*CinG + ci][n]
//   A: shared-memory words [CinTotal/4][ldA] (4 consecutive channels per word); ldA mod 32 must be 8 or 24 so
//      that the 4 k-words x 8 rows of a fragment load hit 32 different banks.
//   W: global memory in FRAGMENT ORDER [k-step][n-tile][lane] x uint2 (see model_spec.cc PackMmaB): every lane's
//      B fragment of one (k-step, n-tile) is one coalesced 8-byte load; each weight is read exactly once per
//      block, straight from L2 into registers (no shared-memory staging, no barriers in the K loop), with a
//      PD-deep register prefetch.
//   A warp owns one 16-row m-tile (rows m = t*S + s) and NTW consecutive 8-column n-tiles.
//   epi(t, s, n4, acc) is called per output row and group of 4 consecutive channels n4..n4+3 (acc is [1][4]),
//   after neighbouring lanes have exchanged their halves of the accumulator tile.
template <int S, int NT, int NTW, int PDI = LYRA_I8_PD, typename Epi>
__device__ __forceinline__ void GemmI8Mma(const uint32_t* A, int ldA, int rowA0, int row_stride, int ntaps, int CinG,
                                          int groups, int T_out, int N, const uint2* __restrict__ Wf, Epi epi) {
  constexpr int PD = PDI;             // register prefetch depth of the B fragments (k-steps)
  const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5, g = lane >> 2, t4 = lane & 3;
  const int M = T_out * S, MT = (M + 15) / 16, NTILES = N / 8, NWT = MT * (NTILES / NTW);
  const int CinG4 = CinG / 4, KS = ntaps * CinG4 / 8, CoutG = N / groups;
  for (int wt = warp; wt < NWT; wt += NT / 32) {
    const int mt = wt % MT, nt0 = (wt / MT) * NTW;
    const int m0 = mt * 16 + g, m1 = m0 + 8;
    const bool valid0 = m0 < M, valid1 = m1 < M;
    const int tr0 = valid0 ? m0 / S : T_out - 1, tr1 = valid1 ? m1 / S : T_out - 1;   // clamp: rows past M only feed discarded outputs
    const int s0 = m0 % S, s1 = m1 % S;
    const int grp = (nt0 * 8) / CoutG;
    const uint32_t* pa0 = A + (size_t)(grp * CinG4) * ldA + (rowA0 + tr0 * row_stride) * S + s0;
    const uint32_t* pa1 = A + (size_t)(grp * CinG4) * ldA + (rowA0 + tr1 * row_stride) * S + s1;
    const uint2* wp = Wf + (size_t)nt0 * 32 + lane;
    const size_t ks_stride = (size_t)NTILES * 32;
    int acc[NTW][4];
#pragma unroll
    for (int j = 0; j < NTW; ++j) { acc[j][0] = 0; acc[j][1] = 0; acc[j][2] = 0; acc[j][3] = 0; }
    uint2 bf[PD][NTW];
#pragma unroll
    for (int p = 0; p < PD; ++p)
      if (p < KS) {
#pragma unroll
        for (int j = 0; j < NTW; ++j) bf[p][j] = LoadFrag<(LYRA_FRAG_NOALLOC & 1) != 0>(wp + p * ks_stride + j * 32);
      }
    for (int ks0 = 0; ks0 < KS; ks0 += PD) {
#pragma unroll
      for (int p = 0; p < PD; ++p) {
        const int ks = ks0 + p;
        if (ks < KS) {
          const int kw = ks * 8, tap = kw / CinG4, kw0 = kw - tap * CinG4;
          const size_t off = (size_t)(kw0 + t4) * ldA + tap * S;
          uint32_t a[4];
          a[0] = pa0[off]; a[1] = pa1[off]; a[2] = pa0[off + 4 * (size_t)ldA]; a[3] = pa1[off + 4 * (size_t)ldA];
#pragma unroll
          for (int j = 0; j < NTW; ++j) {
            const uint32_t b[2] = {bf[p][j].x, bf[p][j].y};
            lyra_mma_s8_16x8x32(acc[j], a, b);
          }
          if (ks + PD < KS) {
#pragma unroll
            for (int j = 0; j < NTW; ++j) bf[p][j] = LoadFrag<(LYRA_FRAG_NOALLOC & 1) != 0>(wp + (size_t)(ks + PD) * ks_stride + j * 32);
          }
        }
      }
    }
    // lanes (2p, 2p+1) of a quad hold columns 4p..4p+1 / 4p+2..4p+3 of rows g and g+8: after one exchange the even
    // lane owns row g, the odd lane row g+8, each with 4 consecutive channels
    const bool even = (t4 & 1) == 0;
#pragma unroll
    for (int j = 0; j < NTW; ++j) {
      const int r0 = __shfl_xor_sync(0xffffffffu, even ? acc[j][2] : acc[j][0], 1);
      const int r1 = __shfl_xor_sync(0xffffffffu, even ? acc[j][3] : acc[j][1], 1);
      int out[1][4];
      if (even) { out[0][0] = acc[j][0]; out[0][1] = acc[j][1]; out[0][2] = r0; out[0][3] = r1; }
      else { out[0][0] = r0; out[0][1] = r1; out[0][2] = acc[j][2]; out[0][3] = acc[j][3]; }
      const int n4 = (nt0 + j) * 8 + (t4 >> 1) * 4;
      if (even ? valid0 : valid1) epi(even ? tr0 : tr1, even ? s0 : s1, n4, out);
    }
  }
  __syncthreads();
}

// smallest stride >= x (multiple of 4 words) whose residue mod 32 is 8 or 24: conflict-free MMA A-fragment loads
__host__ __device__ constexpr int PadLd(int x) {
  while (!(x % 4 == 0 && (x % 32 == 8 || x % 32 == 24))) ++x;
  return x;
}

// ------------------------------------------------------------------------------------------------
// fp32 tap-GEMM on the tensor cores in split precision ("3xTF32"); decoder tensor-core mode only.
//   x = hi + lo with hi = the top 19 bits of x (what a TF32 operand keeps) and lo = x - hi (exact in fp32);
//   a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, accumulated in fp32 by mma.sync m16n8k8 (small terms first).
//   The dropped a_lo*b_lo term and the TF32 truncation of lo are both below 2^-21 relative, i.e. the result
//   carries fp32-level accuracy but NOT the oracle's exact fmaf-chain rounding: outputs of this mode are
//   compared with a tolerance (DESIGN.md, tests/test_gpu_parity.py), never bit-for-bit.
//   Same operand conventions as GemmF32Tap / GemmI8Mma:
//   A: shared memory [channels][ldA] floats, rows m = t*S + s; ldA mod 32 should be 8 or 24 (PadLd) so the
//      4 k-rows x 8 m-rows of a fragment load hit 32 different banks.
//   W: global memory in FRAGMENT ORDER [Ktot/8][N/8][lane] x float2 = {W[8ks + t][8nt + g], W[8ks + t + 4][8nt + g]}
//      (model_spec.cc PackMmaBTf32), loaded straight from L2 with a PD-deep register prefetch.
//   A warp owns WTM m-tiles (16 rows each) x WTN n-tiles (8 columns each).
//   epi(t, s, n2, acc) is called per output row and pair of channels n2, n2+1 (acc is float[1][2]).
//   SYNC_EPI: the epilogue may overwrite the A operand in place: every warp owns at most one warp tile and a block
//   barrier separates the K loops from the epilogues.
__device__ __forceinline__ void SplitTf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(__fsub_rn(x, __uint_as_float(hi)));
}

#ifndef LYRA_TF32_PD
#define LYRA_TF32_PD 8
#endif
template <int S, int NT, int WTM, int WTN, bool SYNC_EPI, typename Epi>
__device__ __forceinline__ void GemmTf32Mma(const float* A, int ldA, int rowA0, int row_stride, int ntaps, int CinG,
                                            int groups, int T_out, int N, const float2* __restrict__ Wf, Epi epi) {
  constexpr int PD = LYRA_TF32_PD;      // k-steps of B fragments in flight from L2 (registers: 2 x WTN per step)
  constexpr int NW = NT / 32;
  const int lane = (int)threadIdx.x & 31, warp = (int)threadIdx.x >> 5, g = lane >> 2, t4 = lane & 3;
  const int M = T_out * S, MT = (M + 15) / 16, MTW = (MT + WTM - 1) / WTM, NTILES = N / 8, NWT = MTW * (NTILES / WTN);
  const int KS = ntaps * CinG / 8, CoutG = N / groups;
  const size_t ks_stride = (size_t)NTILES * 32;
  float acc[WTM][WTN][4];
  int tr[WTM][2], sr[WTM][2];
  bool vr[WTM][2];
  int nt0 = 0;

  auto kloop = [&](int wt) {
    const int mtb = (wt % MTW) * WTM;
    nt0 = (wt / MTW) * WTN;
    const int grp = (nt0 * 8) / CoutG;
    const float* pa[WTM][2];
#pragma unroll
    for (int i = 0; i < WTM; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = (mtb + i) * 16 + g + 8 * h;
        vr[i][h] = m < M;
        tr[i][h] = vr[i][h] ? m / S : T_out - 1;      // clamp: rows past M only feed discarded outputs
        sr[i][h] = m % S;
        pa[i][h] = A + (size_t)(grp * CinG) * ldA + (rowA0 + tr[i][h] * row_stride) * S + sr[i][h];
      }
#pragma unroll
    for (int i = 0; i < WTM; ++i)
#pragma unroll
      for (int j = 0; j < WTN; ++j) { acc[i][j][0] = 0.0f; acc[i][j][1] = 0.0f; acc[i][j][2] = 0.0f; acc[i][j][3] = 0.0f; }
    const float2* wp = Wf + (size_t)nt0 * 32 + lane;
    float2 bf[PD][WTN];
#pragma unroll
    for (int p = 0; p < PD; ++p)
      if (p < KS) {
#pragma unroll
        for (int j = 0; j < WTN; ++j) bf[p][j] = LoadFrag<(LYRA_FRAG_NOALLOC & 2) != 0>(wp + p * ks_stride + j * 32);
      }
    for (int ks0 = 0; ks0 < KS; ks0 += PD) {
#pragma unroll
      for (int p = 0; p < PD; ++p) {
        const int ks = ks0 + p;
        if (ks < KS) {
          const int k0 = ks * 8, tap = k0 / CinG, c0 = k0 - tap * CinG;
          const size_t off = (size_t)(c0 + t4) * ldA + tap * S, off4 = off + 4 * (size_t)ldA;
          uint32_t ahi[WTM][4], alo[WTM][4];
#pragma unroll
          for (int i = 0; i < WTM; ++i) {
            SplitTf32(pa[i][0][off], ahi[i][0], alo[i][0]);
            SplitTf32(pa[i][1][off], ahi[i][1], alo[i][1]);
            SplitTf32(pa[i][0][off4], ahi[i][2], alo[i][2]);
            SplitTf32(pa[i][1][off4], ahi[i][3], alo[i][3]);
          }
#pragma unroll
          for (int j = 0; j < WTN; ++j) {
            uint32_t bhi[2], blo[2];
            SplitTf32(bf[p][j].x, bhi[0], blo[0]);
            SplitTf32(bf[p][j].y, bhi[1], blo[1]);
#pragma unroll
            for (int i = 0; i < WTM; ++i) {
              lyra_mma_tf32_16x8x8(acc[i][j], alo[i], bhi);
              lyra_mma_tf32_16x8x8(acc[i][j], ahi[i], blo);
              lyra_mma_tf32_16x8x8(acc[i][j], ahi[i], bhi);
            }
          }
          if (ks + PD < KS) {
#pragma unroll
            for (int j = 0; j < WTN; ++j) bf[p][j] = LoadFrag<(LYRA_FRAG_NOALLOC & 2) != 0>(wp + (size_t)(ks + PD) * ks_stride + j * 32);
          }
        }
      }
    }
  };
  auto epilogue = [&]() {
#pragma unroll
    for (int i = 0; i < WTM; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (vr[i][h]) {
#pragma unroll
          for (int j = 0; j < WTN; ++j) {
            float o[1][2] = {{acc[i][j][2 * h], acc[i][j][2 * h + 1]}};
            epi(tr[i][h], sr[i][h], (nt0 + j) * 8 + 2 * t4, o);
          }
        }
  };
  if (SYNC_EPI) {
    if (NWT > NW) LYRA_TRAP();          // callers size the warp tile so that every warp owns at most one
    const bool has = warp < NWT;
    if (has) kloop(warp);
    __syncthreads();
    if (has) epilogue();
  } else {
    for (int wt = warp; wt < NWT; wt += NW) {
      kloop(wt);
      epilogue();
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// Ring addressing.  A dilated depthwise conv (k = 3, dilation d) needs a(i - 2d), a(i - d), a(i) for
// absolute row i; the last R = 2d rows of every stream live in a global ring [C][R][S] (slot = i mod R).
// frame counters are kept modulo 18 (every R divides 18), so base = (n18 * T) mod R.
__device__ __forceinline__ int RingSlot(int base, int t, int R) {
  int v = (base + t) % R;
  return v < 0 ? v + R : v;
}

__device__ __forceinline__ float4 LeakyRelu4(float4 v) {
  return make_float4(LeakyRelu(v.x), LeakyRelu(v.y), LeakyRelu(v.z), LeakyRelu(v.w));
}

// Fast path of DwF32Ring for tiles whose active streams share one frame counter (`n18u` >= 0): one thread
// owns (channel, 4 streams); it first issues all R ring-row loads back to back (one exposed HBM/L2 latency
// instead of one per element), then walks the T rows with compile-time indexing, and finally writes the
// newest rows of its own ring column — no block barrier is needed because nobody else touches that column.
template <int S, int NT, int C, int T, int DIL>
__device__ __forceinline__ void DwF32RingFast(const float* u, int ldu, int row0u, float* dout, int ldd,
                                              const float* __restrict__ w, const float* __restrict__ bias,
                                              float* __restrict__ ring, int n18u, const int* active) {
  constexpr int R = 2 * DIL, Q = S / 4;
  const int base = (n18u * T) % R;
  for (int item = (int)threadIdx.x; item < C * Q; item += NT) {
    const int c = item / Q, s4 = (item % Q) * 4;
    float* rc = ring + (size_t)c * R * S + s4;
    float4 rg[R];
#pragma unroll
    for (int j = 0; j < R; ++j) rg[j] = *reinterpret_cast<const float4*>(rc + ((base + j) % R) * S);
    const float w0 = w[c], w1 = w[C + c], w2 = w[2 * C + c], b = bias[c];
    const float* uc = u + (size_t)c * ldu + row0u * S + s4;
    float* dc = dout + (size_t)c * ldd + s4;
#pragma unroll
    for (int t = 0; t < T; ++t) {
      const float4 x2 = LeakyRelu4(*reinterpret_cast<const float4*>(uc + t * S));
      float4 x1, x0;
      if (t - DIL >= 0) x1 = LeakyRelu4(*reinterpret_cast<const float4*>(uc + (t - DIL) * S));
      else x1 = rg[(t - DIL + R) % R];
      if (t - 2 * DIL >= 0) x0 = LeakyRelu4(*reinterpret_cast<const float4*>(uc + (t - 2 * DIL) * S));
      else x0 = rg[(t - 2 * DIL + R) % R];
      float4 o;
      o.x = __fadd_rn(__fmaf_rn(x2.x, w2, __fmaf_rn(x1.x, w1, __fmaf_rn(x0.x, w0, 0.0f))), b);
      o.y = __fadd_rn(__fmaf_rn(x2.y, w2, __fmaf_rn(x1.y, w1, __fmaf_rn(x0.y, w0, 0.0f))), b);
      o.z = __fadd_rn(__fmaf_rn(x2.z, w2, __fmaf_rn(x1.z, w1, __fmaf_rn(x0.z, w0, 0.0f))), b);
      o.w = __fadd_rn(__fmaf_rn(x2.w, w2, __fmaf_rn(x1.w, w1, __fmaf_rn(x0.w, w0, 0.0f))), b);
      *reinterpret_cast<float4*>(dc + t * S) = o;
    }
    constexpr int TF = T > R ? T - R : 0;
    const bool all4 = active[s4] && active[s4 + 1] && active[s4 + 2] && active[s4 + 3];
#pragma unroll
    for (int t = TF; t < T; ++t) {
      const float4 a = LeakyRelu4(*reinterpret_cast<const float4*>(uc + t * S));
      float* dst = rc + ((base + t) % R) * S;
      if (all4) {
        *reinterpret_cast<float4*>(dst) = a;
      } else {
        if (active[s4]) dst[0] = a.x;
        if (active[s4 + 1]) dst[1] = a.y;
        if (active[s4 + 2]) dst[2] = a.z;
        if (active[s4 + 3]) dst[3] = a.w;
      }
    }
  }
  __syncthreads();
}

// int8 analogue on packed words: one thread owns (4 channels, 1 stream) for all T rows (C/4 * S work items, so a
// 256-channel T = 2 layer keeps every thread of the block busy with 8 requantisations each).
template <int S, int NT, int C, int T, int DIL>
__device__ __forceinline__ void DwI8RingFast(const uint32_t* aq, int lda, int row0a, uint32_t* dq, int ldd,
                                             const uint8_t* blob, const DwI8& p, uint32_t* __restrict__ ring, int n18u,
                                             const int* active) {
  constexpr int R = 2 * DIL, C4 = C / 4;
  const int base = (n18u * T) % R;
  const int* w = BlobPtr<int>(blob, p.w);
  const int* bias = BlobPtr<int>(blob, p.bias);
  const int* mult = BlobPtr<int>(blob, p.mult);
  const int* shift = BlobPtr<int>(blob, p.shift);
  for (int item = (int)threadIdx.x; item < C4 * S; item += NT) {
    const int c4 = item / S, s = item % S;
    uint32_t* rc = ring + (size_t)c4 * R * S + s;
    const uint32_t* ac = aq + (size_t)c4 * lda + row0a * S + s;
    uint32_t x0[T], x1[T], x2[T];
#pragma unroll
    for (int t = 0; t < T; ++t) {
      x2[t] = ac[t * S];
      x1[t] = t - DIL >= 0 ? ac[(t - DIL) * S] : rc[((base + t - DIL + 2 * R) % R) * S];
      x0[t] = t - 2 * DIL >= 0 ? ac[(t - 2 * DIL) * S] : rc[((base + t - 2 * DIL + 2 * R) % R) * S];
    }
    int wk[3][4], bb[4], mm[4], sh[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = c4 * 4 + b;
      wk[0][b] = w[c]; wk[1][b] = w[C + c]; wk[2][b] = w[2 * C + c];
      bb[b] = bias[c]; mm[b] = mult[c]; sh[b] = shift[c];
    }
#pragma unroll
    for (int t = 0; t < T; ++t) {
      int q[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int acc = UnpackI8(x0[t], b) * wk[0][b] + UnpackI8(x1[t], b) * wk[1][b] + UnpackI8(x2[t], b) * wk[2][b];
        q[b] = RequantI8(acc, bb[b], mm[b], sh[b], p.out_zp);
      }
      dq[(size_t)c4 * ldd + t * S + s] = PackI8x4(q[0], q[1], q[2], q[3]);
    }
    constexpr int TF = T > R ? T - R : 0;
    if (active[s]) {
#pragma unroll
      for (int t = TF; t < T; ++t) rc[((base + t) % R) * S] = x2[t];
    }
  }
  __syncthreads();
}

// fp32 depthwise conv over LeakyReLU(u).  u: shared [C][ldu] with the T new rows starting at row0u.
// dout: shared [C][ldd] rows 0..T-1.  ring: global tile block [C][R][S].  n18: shared per-stream counters.
template <int S, int NT>
__device__ __forceinline__ void DwF32Ring(const float* u, int ldu, int row0u, float* dout, int ldd, int C, int T, int dil,
                                          const float* __restrict__ w, const float* __restrict__ bias,
                                          float* __restrict__ ring, const int* n18, const int* active) {
  const int R = 2 * dil;
  const int total = C * T * S;
  for (int idx = (int)threadIdx.x; idx < total; idx += NT) {
    const int s = idx % S, t = (idx / S) % T, c = idx / (S * T);
    const int base = (n18[s] * T) % R;
    const float* uc = u + (size_t)c * ldu + row0u * S + s;
    const float x2 = LeakyRelu(uc[t * S]);
    const float x1 = t - dil >= 0 ? LeakyRelu(uc[(t - dil) * S]) : ring[((size_t)c * R + RingSlot(base, t - dil, R)) * S + s];
    const float x0 = t - 2 * dil >= 0 ? LeakyRelu(uc[(t - 2 * dil) * S]) : ring[((size_t)c * R + RingSlot(base, t - 2 * dil, R)) * S + s];
    float acc = __fmaf_rn(x0, w[c], 0.0f);
    acc = __fmaf_rn(x1, w[C + c], acc);
    acc = __fmaf_rn(x2, w[2 * C + c], acc);
    dout[(size_t)c * ldd + t * S + s] = __fadd_rn(acc, bias[c]);
  }
  __syncthreads();
  // the last min(T, R) rows become the ring's newest entries
  const int tfirst = T > R ? T - R : 0;
  const int nrows = T - tfirst;
  const int wtotal = C * nrows * S;
  for (int idx = (int)threadIdx.x; idx < wtotal; idx += NT) {
    const int s = idx % S, t = tfirst + (idx / S) % nrows, c = idx / (S * nrows);
    if (!active[s]) continue;
    const int base = (n18[s] * T) % R;
    ring[((size_t)c * R + RingSlot(base, t, R)) * S + s] = LeakyRelu(u[(size_t)c * ldu + (row0u + t) * S + s]);
  }
  __syncthreads();
}

// int8 depthwise conv on packed activations.  aq: shared words [C/4][lda], new rows at row0a.
// dq: shared words [C/4][ldd] rows 0..T-1.  ring: global words [C/4][R][S].
template <int S, int NT>
__device__ __forceinline__ void DwI8Ring(const uint32_t* aq, int lda, int row0a, uint32_t* dq, int ldd, int C, int T, int dil,
                                         const uint8_t* blob, const DwI8& p, uint32_t* __restrict__ ring, const int* n18,
                                         const int* active) {
  const int R = 2 * dil, C4 = C / 4;
  const int* w = BlobPtr<int>(blob, p.w);
  const int* bias = BlobPtr<int>(blob, p.bias);
  const int* mult = BlobPtr<int>(blob, p.mult);
  const int* shift = BlobPtr<int>(blob, p.shift);
  const int total = C4 * T * S;
  for (int idx = (int)threadIdx.x; idx < total; idx += NT) {
    const int s = idx % S, t = (idx / S) % T, c4 = idx / (S * T);
    const int base = (n18[s] * T) % R;
    const uint32_t* ac = aq + (size_t)c4 * lda + row0a * S + s;
    const uint32_t x2 = ac[t * S];
    const uint32_t x1 = t - dil >= 0 ? ac[(t - dil) * S] : ring[((size_t)c4 * R + RingSlot(base, t - dil, R)) * S + s];
    const uint32_t x0 = t - 2 * dil >= 0 ? ac[(t - 2 * dil) * S] : ring[((size_t)c4 * R + RingSlot(base, t - 2 * dil, R)) * S + s];
    int o[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = c4 * 4 + b;
      const int acc = UnpackI8(x0, b) * w[c] + UnpackI8(x1, b) * w[C + c] + UnpackI8(x2, b) * w[2 * C + c];
      o[b] = RequantI8(acc, bias[c], mult[c], shift[c], p.out_zp);
    }
    dq[(size_t)c4 * ldd + t * S + s] = PackI8x4(o[0], o[1], o[2], o[3]);
  }
  __syncthreads();
  const int tfirst = T > R ? T - R : 0;
  const int nrows = T - tfirst;
  const int wtotal = C4 * nrows * S;
  for (int idx = (int)threadIdx.x; idx < wtotal; idx += NT) {
    const int s = idx % S, t = tfirst + (idx / S) % nrows, c4 = idx / (S * nrows);
    if (!active[s]) continue;
    const int base = (n18[s] * T) % R;
    ring[((size_t)c4 * R + RingSlot(base, t, R)) * S + s] = aq[(size_t)c4 * lda + (row0a + t) * S + s];
  }
  __syncthreads();
}

}  // namespace lyra_b200
