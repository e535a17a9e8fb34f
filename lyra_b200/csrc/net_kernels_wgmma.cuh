// DecoderKernelDW: kernel D of the decoder (decoder_2/simple .. last_layer -> int16 PCM) on the Hopper tensor cores.
//
// This is the kernel that runs when the context's decoder mode is LYRA_B200_DECODER_TENSOR.  Every fp32 GEMM of the tile
// (913 k MAC per stream-frame) is issued as split-precision TF32 warpgroup MMAs (wgmma; x = hi + lo, three MMAs per product,
// fp32 accumulators in registers); the CUDA cores run the depthwise passes, the epilogues and the state I/O.
// Same inputs, outputs and streaming state as DecoderKernelD (net_kernels.cuh), so the two can alternate on one stream.
//
//   rows        a GEMM row of the T = 20 layers is (time row t, stream s) of the tile: m = t * 8 + s.  Three warpgroups own
//               64 rows each (rows 160..191 are padding: zero operands, results dropped).  A thread holds accumulator rows
//               m and m + 8 (time rows t and t + 1 of stream s = lane / 4), see device_compat.h for the fragment layout.
//   residual    A operand in REGISTERS: the depthwise conv writes the thread's A fragments directly, and each epilogue turns
//   units       its accumulators into the next GEMM's A fragments with quad shuffles, so the activations never take a round
//               trip through shared memory between the depthwise conv, the two 1x1 convolutions and last_layer.
//               B = weights from shared memory.
//   decoder_2/  computed TRANSPOSED: the 640 weight rows (tap j, phase r, cout) are the M dimension (A operand from shared
//   simple      memory, warpgroups 0 and 1 take the two 64-row halves of each 128-row chunk) and the tile's 32 (input row,
//               stream) pairs the N dimension (B operand, 16 KB per half): M = 64 blocks of a uniform tap and phase instead of
//               160-row blocks whose 32 columns would be the long side.  The two taps meet in shared memory.
//   last_layer  ONE 64 x 64 GEMM P[row][tap * 16 + n] = sum_ci lrelu(u')[row][ci] * W[(tap, ci)][n]; the four taps are summed
//               across time rows afterwards.
//   weights     pre-split on the host into hi / lo core-matrix chunks (net_params.h kDuChunkBytes), streamed by one producer
//               thread with TMA bulk copies through a 4-stage shared-memory ring; a stage is released once every row warp's
//               MMAs that read it have completed (wgmma.wait_group).
//   state       the overlap tail, the last_layer tail and the ring blocks of units 0 and 1 move by TMA bulk copies in both
//               directions (written back whole, with the lanes of inactive streams left as loaded); kernel C's tile and unit 2's
//               36 KB ring block are read from / written to global memory directly.
//   roles       warps 0..11: rows / MMAs / epilogues / state;  warp 12 lane 0: TMA producer.
// Arithmetic: products carry fp32-level accuracy (error terms below 2^-21 relative) but not the oracle's fmaf-chain rounding or
// summation order: decoded PCM is compared with a tolerance (tests/parity_cases.py TENSOR_PCM_TOL_LSB), never bit for bit.
#pragma once

#include <type_traits>

#include "net_kernels.cuh"

namespace lyra_b200 {

struct DecDW {
  static constexpr int S = kTileStreams;
  static_assert(S == 8, "the row warps map lane / 4 to the tile's stream");
  static constexpr int kRowWgs = 3, kRowThreads = kRowWgs * 128;
  static constexpr int kTmaWarp = kRowThreads / 32;
  static constexpr int NT = kRowThreads + 32;
  static constexpr int kStagesW = 4;
  static constexpr int LDU = 161;                             // u: f32 [64][LDU], element (c, row = t * 8 + s); odd stride: lanes that
                                                              // differ in c (decoder_2/simple epilogue) hit different banks
  // shared memory (bytes), 142 KB:
  //   u        the residual stream of the three units, f32 [64][LDU]
  //   region   decoder_2/simple's B operand X (hi | lo, 32 KB)  ->  once its MMAs are done: the carried overlap tail (10 KB), the ring
  //            blocks of units 0 and 1 (4 + 12 KB), PCM staging.  Unit 2's ring block (36 KB, dilation 9) stays in global memory (L2):
  //            its rows are read and replaced in place.  Kernel C's tile is read from global memory as well.
  static constexpr int kU = 0;
  static constexpr int kXc = kU + 64 * LDU * 4;               // decoder_2/simple B operand: hi | lo, each [128/4][4][8][4] f32
  static constexpr int kXPart = 32 * 4 * 32 * 4;              // 16,384
  static constexpr int kRegion = kXc, kRegionBytes = 2 * kXPart;
  static constexpr int kOv = kRegion;                         // decoder_2/simple overlap tail f32 [64][5][8]: loaded, consumed, rewritten, stored
  static constexpr int kRing0 = kOv + 64 * 5 * S * 4, kRing1 = kRing0 + 64 * 2 * S * 4;     // ring blocks [64][R][8] f32, R = 2, 6
  static constexpr int kStage = kRing1 + 64 * 6 * S * 4;      // at the end: PCM staging int16 [8][320]
  static constexpr int kSl = kRegion + kRegionBytes;          // last_layer carried tail f32 [48][8]
  static constexpr int kSlOut = kSl + 48 * S * 4;             // ... and its successor
  static constexpr int kDw4 = kSlOut + 48 * S * 4;            // depthwise parameters per channel: float4 {w0, w1, w2, bias} [3][64]
  static constexpr int kW = kDw4 + 3 * 256 * 4;               // weight ring
  static constexpr int kI = kW + kStagesW * kDuChunkBytes;    // slot[S], active[S], n18[S]
  static constexpr int kSmemBytes = kI + 3 * S * 4 + 16;      // + n18[S]
  static_assert(kStage + S * 320 * 2 <= kRegion + kRegionBytes, "overlap tail, two ring blocks and PCM staging must fit in the X region");
  static_assert(kXc % 128 == 0 && kOv % 128 == 0 && kRing0 % 128 == 0 && kRing1 % 128 == 0 && kW % 128 == 0 && kSl % 16 == 0 && kDw4 % 16 == 0,
                "bulk-copy / descriptor alignment");
  static_assert(kSmemBytes <= 227 * 1024, "shared memory of one block");
};

struct DecDWShared {
  LyraMbar w_full[DecDW::kStagesW], w_empty[DecDW::kStagesW];
  LyraMbar in_full;        // producer -> row warps: the last_layer tail has landed
  LyraMbar ov_full;        // producer -> row warps: the overlap tail has landed (in the X region, after decoder_2/simple's MMAs)
  LyraMbar ring_full[2];   // producer -> row warps: ring block u (units 0, 1) has landed
};

__device__ __forceinline__ void DwSplit(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xffffe000u;
  lo = __float_as_uint(__fsub_rn(x, __uint_as_float(hi)));
}

// Accumulator-layout values (rows m, m + 8; columns 8j + 2t, 8j + 2t + 1) -> the split A fragments of the next GEMM (columns
// 8j + t, 8j + t + 4): the four lanes of a quad hold the eight columns of a k-step between them.  Warp-collective.
__device__ __forceinline__ void DwAccToA(const float (&h)[32], uint32_t (&ah)[8][4], uint32_t (&al)[8][4]) {
  const int lane = (int)(threadIdx.x & 31), t = lane & 3;
  const int src_lo = (lane & ~3) | (t >> 1), src_hi = src_lo + 2;
  const bool odd = (t & 1) != 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float v[4];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const float e0 = __shfl_sync(0xffffffffu, h[4 * j + 2 * rr], src_lo), e1 = __shfl_sync(0xffffffffu, h[4 * j + 2 * rr + 1], src_lo);
      const float f0 = __shfl_sync(0xffffffffu, h[4 * j + 2 * rr], src_hi), f1 = __shfl_sync(0xffffffffu, h[4 * j + 2 * rr + 1], src_hi);
      v[rr] = odd ? e1 : e0;
      v[2 + rr] = odd ? f1 : f0;
    }
#pragma unroll
    for (int f = 0; f < 4; ++f) DwSplit(v[f], ah[j][f], al[j][f]);
  }
}

__global__ void __launch_bounds__(DecDW::NT, 1)
DecoderKernelDW(const uint8_t* __restrict__ blob, DecoderParams P, TileIo io, const float* __restrict__ mid,
                float* __restrict__ state, int* __restrict__ n18g, int16_t* __restrict__ pcm) {
  using L = DecDW;
  constexpr int S = L::S, LDU = L::LDU;
  unsigned char* smem = LYRA_DYN_SMEM();
  float* smf = reinterpret_cast<float*>(smem);                // every f32 buffer below is addressed as smf[float offset]
  float* u = smf + L::kU / 4;
  unsigned char* wring = smem + L::kW;
  float* ov = smf + L::kOv / 4;
  float* sl = smf + L::kSl / 4;
  float* slo = smf + L::kSlOut / 4;
  int* slot = reinterpret_cast<int*>(smem + L::kI);
  int* active = slot + S;
  int* n18 = active + S;                                      // n18[S]: tile summary (BeginTile)
  LYRA_STATIC_SMEM(DecDWShared, sh, 1);
  const int tid = (int)threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < L::kStagesW; ++i) {
      lyra_mbar_init(&sh->w_full[i], 1);
      lyra_mbar_init(&sh->w_empty[i], L::kRowThreads / 32);
    }
    lyra_mbar_init(&sh->in_full, 1);
    lyra_mbar_init(&sh->ov_full, 1);
    for (int i = 0; i < 2; ++i) lyra_mbar_init(&sh->ring_full[i], 1);
    lyra_mbar_fence_init();
  }
  // BeginTile holds two block barriers: the barrier inits above are visible after it.  Its L2 prefetch of the tile's state also
  // serves unit 2, which reads its ring block from global memory.
  int tile;
  if (!BeginTile<S>(io, n18g, slot, state, DecStateD::kUnits, tile)) return;
  float* st = state + (size_t)tile * DecStateD::kUnits * S;
  const uint8_t* chunks = blob + P.du_chunks;

  // ================================================= TMA producer =================================================
  if (warp == L::kTmaWarp) {
    if (lane == 0) {
      lyra_bulk_g2s(sl, st + (size_t)DecStateD::kLast * S, 48u * S * 4, &sh->in_full);
      for (int c = 0; c < kDuNumChunks; ++c) {
        const int stg = c % L::kStagesW;
        if (c >= L::kStagesW) lyra_mbar_wait(&sh->w_empty[stg], (unsigned)((c / L::kStagesW - 1) & 1));
        lyra_bulk_g2s(wring + (size_t)stg * kDuChunkBytes, chunks + (size_t)c * kDuChunkBytes, (unsigned)kDuChunkBytes, &sh->w_full[stg]);
        if (c == kDuUp2Chunks + L::kStagesW - 1) {
          // the wait above covered the last decoder_2/simple chunk's MMAs, the last readers of X: the overlap tail and the ring
          // blocks of units 0 and 1 may land on it
          lyra_bulk_g2s(ov, st + (size_t)DecStateD::kUp2 * S, 64u * 5 * S * 4, &sh->ov_full);
          lyra_bulk_g2s(smem + L::kRing0, st + (size_t)DecStateD::kRing0 * S, 64u * 2 * S * 4, &sh->ring_full[0]);
          lyra_bulk_g2s(smem + L::kRing1, st + (size_t)DecStateD::kRing1 * S, 64u * 6 * S * 4, &sh->ring_full[1]);
        }
      }
    }
    return;
  }

  // ================================================= row warpgroups ================================================
  const int wg = tid >> 7, wq = warp & 3, g = lane >> 2, tq = lane & 3;
  const int s = g;                                            // the thread's stream ...
  const int t0 = 8 * wg + 2 * wq;                             // ... and time rows t0, t0 + 1 (GEMM rows m0 = t0 * 8 + s, m0 + 8)
  const int m0 = t0 * S + s;
  const bool has_rows = t0 < 20;                              // warps 10 and 11 hold the padding rows 160..191
  auto row_sync = [&]() { lyra_named_bar_sync(1, L::kRowThreads); };
  int c = 0;                                                  // weight chunk counter: every row warp takes part in every chunk
  auto wait_chunk = [&]() -> const unsigned char* {
    lyra_mbar_wait(&sh->w_full[c % L::kStagesW], (unsigned)((c / L::kStagesW) & 1));
    return wring + (size_t)(c % L::kStagesW) * kDuChunkBytes;
  };
  auto release_chunk = [&]() {
    __syncwarp();
    if (lane == 0) lyra_mbar_arrive(&sh->w_empty[c % L::kStagesW]);
    ++c;
  };

  // ---- X: kernel C's tile [128 ch][4 rows][8 streams] -> B operand (split, core-matrix layout, row = (x-row, stream), k = ch)
  if (tid < 3 * 64) {                                         // depthwise parameters per channel (read after several barriers)
    const int un = tid / 64, ch = tid % 64;
    const float* w = BlobPtr<float>(blob, P.r2[un].dw.w);
    reinterpret_cast<float4*>(smf + L::kDw4 / 4)[tid] = make_float4(w[ch], w[64 + ch], w[128 + ch], BlobPtr<float>(blob, P.r2[un].dw.bias)[ch]);
  }
  {
    const float* in = mid + (size_t)tile * 128 * 4 * S;       // kernel C's tile, straight from global memory (L2)
    float* xh = smf + L::kXc / 4;
    float* xl = xh + L::kXPart / 4;
    for (int item = tid; item < 32 * 4 * 8; item += L::kRowThreads) {
      const int i = item % 8, xg = (item / 8) % 4, kg = item / 32;
      uint32_t hh[4], ll[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) DwSplit(in[((4 * kg + j) * 4 + xg) * S + i], hh[j], ll[j]);
      const int o = ((kg * 4 + xg) * 8 + i) * 4;
      *reinterpret_cast<float4*>(xh + o) = make_float4(__uint_as_float(hh[0]), __uint_as_float(hh[1]), __uint_as_float(hh[2]), __uint_as_float(hh[3]));
      *reinterpret_cast<float4*>(xl + o) = make_float4(__uint_as_float(ll[0]), __uint_as_float(ll[1]), __uint_as_float(ll[2]), __uint_as_float(ll[3]));
    }
  }
  lyra_fence_proxy_async();                                   // X is read by the tensor cores through the asynchronous proxy
  row_sync();

  // ---- decoder_2/simple, transposed: D[64 x 32] = Wt[64 x 128] * X[32 x 128]^T for the 64-row half `wg` of each of the five
  //      128-row blocks of Wt (warpgroups 0, 1; warpgroup 2 only passes the chunks on).
  float up[5][16];
  {
    const uint32_t lboW = 16u * 128u, lboX = 4u * 128u;
    const unsigned char* xh = smem + L::kXc;
    const unsigned char* xl = xh + L::kXPart;
#pragma unroll
    for (int mb = 0; mb < 5; ++mb)
#pragma unroll
      for (int kc = 0; kc < 8; ++kc) {
        const unsigned char* wst = wait_chunk();
        if (wg < 2) {
          lyra_wgmma_fence();
#pragma unroll
          for (int k2 = 0; k2 < 2; ++k2) {
            const int ks = kc * 2 + k2;
            const unsigned char* wa = wst + (size_t)k2 * 2 * lboW + (size_t)wg * 8 * 128;
            const uint64_t ah = lyra_wgmma_desc(wa, lboW, 128);
            const uint64_t al = lyra_wgmma_desc(wa + kDuChunkBytes / 2, lboW, 128);
            const uint64_t bh = lyra_wgmma_desc(xh + (size_t)ks * 2 * lboX, lboX, 128);
            const uint64_t bl = lyra_wgmma_desc(xl + (size_t)ks * 2 * lboX, lboX, 128);
            lyra_wgmma_m64n32_tf32_ss(up[mb], al, bh, ks > 0);                   // small terms first
            lyra_wgmma_m64n32_tf32_ss(up[mb], ah, bl, true);
            lyra_wgmma_m64n32_tf32_ss(up[mb], ah, bh, true);
          }
          lyra_wgmma_commit();
          lyra_wgmma_wait<0>();
        }
        release_chunk();
      }
  }

  // ---- decoder_2/simple epilogue.  Block b = 2 mb + wg of 64 weight rows has one tap j = b / 5 and phase r = b % 5; row = cout,
  //      column = (x-row, stream).  out[q][r][co] = (P[j=1][x=q] + bias + carried overlap (q = 0)) + P[j=0][x=q-1]; q = 4 is the new
  //      overlap tail.  Pass 0 stores the j = 1 terms (every element of u), pass 1 adds the j = 0 terms.
  lyra_mbar_wait(&sh->ov_full, 0);                           // the carried overlap tail (it landed on X once the MMAs above were done)
  {
    const float* b = BlobPtr<float>(blob, P.up2.bias);
    for (int pass = 0; pass < 2; ++pass) {
      if (wg < 2) {
#pragma unroll
        for (int mb = 0; mb < 5; ++mb) {
          const int blk = 2 * mb + wg, j = blk / 5, r = blk % 5;
          if (j != 1 - pass) continue;                       // warpgroup-uniform
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int x = i >> 2, ss = 2 * tq + (i & 1), co = 16 * wq + g + 8 * ((i >> 1) & 1);
            const float p = up[mb][i], bias = b[co];
            float* uc = u + co * LDU + r * S + ss;
            float* oc = ov + (co * 5 + r) * S + ss;
            if (pass == 0) {
              uc[(5 * x) * S] = __fadd_rn(__fadd_rn(p, bias), x == 0 ? *oc : 0.0f);
            } else if (x < 3) {
              float* o = uc + (5 * (x + 1)) * S;
              *o = __fadd_rn(*o, p);
            } else if (active[ss]) {
              *oc = __fsub_rn(__fadd_rn(__fadd_rn(p, bias), 0.0f), bias);
            }
          }
        }
      }
      lyra_fence_proxy_async();                              // pass 1: the rewritten overlap block, before its bulk store
      row_sync();
    }
    if (tid == 0) { lyra_bulk_s2g(st + (size_t)DecStateD::kUp2 * S, ov, 64u * 5 * S * 4); lyra_bulk_commit(); }
  }

  // One 64 x 64 GEMM of the tile on the next two weight chunks: acc = A * W, A as split fragments (hi, lo) per k-step.  The small
  // terms accumulate apart from a_hi * b_hi and join it with one round-to-nearest add (see GemmTf32Mma)
  auto gemm = [&](const uint32_t (&ah)[8][4], const uint32_t (&al)[8][4], float (&acc)[32]) {
    const uint32_t lboW = 8u * 128u;
    float accs[32];
#pragma unroll
    for (int kc = 0; kc < 2; ++kc) {
      const unsigned char* wst = wait_chunk();
      lyra_wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const int ks = kc * 4 + k4;
        const uint64_t bh = lyra_wgmma_desc(wst + (size_t)k4 * 2 * lboW, lboW, 128);
        const uint64_t bl = lyra_wgmma_desc(wst + kDuChunkBytes / 2 + (size_t)k4 * 2 * lboW, lboW, 128);
        lyra_wgmma_m64n64_tf32_rs(accs, al[ks], bh, ks > 0);
        lyra_wgmma_m64n64_tf32_rs(accs, ah[ks], bl, true);
        lyra_wgmma_m64n64_tf32_rs(acc, ah[ks], bh, ks > 0);
      }
      lyra_wgmma_commit();
      lyra_wgmma_wait<0>();
      release_chunk();
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = __fadd_rn(acc[i], accs[i]);
  };
  // accumulator element i of the thread: GEMM row m0 (+ 8 for odd pairs), column (channel) 8 (i / 4) + 2 tq + i % 2
  auto acc_row = [&](int i) { return m0 + 8 * ((i >> 1) & 1); };
  auto acc_col = [&](int i) { return 8 * (i >> 2) + 2 * tq + (i & 1); };

  // ---- decoder_2: three residual units, d = dw(lrelu(u)); h = lrelu(pw1(d)); u' = pw2(h) + u
  uint32_t ah[8][4], al[8][4];
  float acc[32];
  auto unit_body = [&](auto unit_c) {
    constexpr int unit = decltype(unit_c)::value;
    constexpr int dil = unit == 0 ? 1 : (unit == 1 ? 3 : 9), R = 2 * dil;
    // units 0, 1: ring block in shared memory (bulk-loaded, bulk-stored); unit 2 (R = 18, 36 KB): rows are read from and written
    // to the global block directly - every read precedes the row barrier that the writes follow, as for the shared-memory blocks
    constexpr bool ring_in_smem = unit < 2;
    constexpr int ring_off = (unit == 0 ? L::kRing0 : L::kRing1) / 4;                             // [64][R][S] f32 (units 0, 1)
    const ResF32& p = P.r2[unit];
    float* gring = st + (size_t)(unit == 0 ? DecStateD::kRing0 : (unit == 1 ? DecStateD::kRing1 : DecStateD::kRing2)) * S;
    float* ring = ring_in_smem ? smf + ring_off : gring;
    if (ring_in_smem) lyra_mbar_wait(&sh->ring_full[unit < 2 ? unit : 0], 0);
    // depthwise conv (k = 3, dilation dil) over LeakyReLU(u) -> A fragments of pw1.  Rows before this frame come from the ring
    // (already activated: slope 1 leaves them as they are)
    {
      const float4* w4 = reinterpret_cast<const float4*>(smf + L::kDw4 / 4) + unit * 64;      // per channel {w0, w1, w2, bias}
      static_assert(DecStateD::kT == 20, "the ring slots below are those of decoder_2's 20 rows per hop (kDwRings)");
      const int base = (n18[s] * 20) % R;                    // ring slot of this frame's row 0 for this stream
      auto dw = [&](int t, int ch) {
        if (!has_rows) return 0.0f;
        const bool r1 = t - dil < 0, r0 = t - 2 * dil < 0;
        float x2 = u[ch * LDU + t * S + s];
        float x1 = r1 ? ring[ch * (R * S) + ((base + t - dil + 2 * R) % R) * S + s] : u[ch * LDU + (t - dil) * S + s];
        float x0 = r0 ? ring[ch * (R * S) + ((base + t - 2 * dil + 2 * R) % R) * S + s] : u[ch * LDU + (t - 2 * dil) * S + s];
        const float4 wc = w4[ch];
        x2 = fmaxf(x2, __fmul_rn(x2, 0.3f));
        x1 = fmaxf(x1, __fmul_rn(x1, r1 ? 1.0f : 0.3f));
        x0 = fmaxf(x0, __fmul_rn(x0, r0 ? 1.0f : 0.3f));
        float a = __fmaf_rn(x0, wc.x, 0.0f);
        a = __fmaf_rn(x1, wc.y, a);
        a = __fmaf_rn(x2, wc.z, a);
        return __fadd_rn(a, wc.w);
      };
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) {
        const int c_lo = 8 * ks + tq, c_hi = c_lo + 4;
        DwSplit(dw(t0, c_lo), ah[ks][0], al[ks][0]);
        DwSplit(dw(t0 + 1, c_lo), ah[ks][1], al[ks][1]);
        DwSplit(dw(t0, c_hi), ah[ks][2], al[ks][2]);
        DwSplit(dw(t0 + 1, c_hi), ah[ks][3], al[ks][3]);
      }
    }
    // The newest min(20, R) rows of lrelu(u) replace the ring's oldest entries (every slot: R <= 20); one row per thread
    row_sync();                                              // all ring reads are done
    if (tid < 20 * S) {
      const int t = tid / S, ss = tid % S;
      if (t >= 20 - R && active[ss]) {
        float* wp = ring + ((((n18[ss] * 20) % R) + t) % R) * S + ss;
        const float* ip = u + tid;
#pragma unroll 16
        for (int ch = 0; ch < 64; ++ch) wp[ch * (R * S)] = LeakyRelu(ip[ch * LDU]);
      }
    }
    // pw1, then its epilogue: bias, LeakyReLU -> A fragments of pw2
    gemm(ah, al, acc);
    {
      const float* b1 = BlobPtr<float>(blob, p.pw1.bias);
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = LeakyRelu(__fadd_rn(acc[i], b1[acc_col(i)]));
      DwAccToA(acc, ah, al);
    }
    lyra_fence_proxy_async();
    row_sync();                                              // ring rows and every read of u are complete
    if (ring_in_smem && tid == 0) { lyra_bulk_s2g(gring, smf + ring_off, (unsigned)(64 * R * S * 4)); lyra_bulk_commit(); }
    // pw2, then its epilogue: bias + residual.  Units 0, 1: u' back to shared memory (the next depthwise conv reads neighbouring
    // rows); unit 2: LeakyReLU(u') as the A fragments of last_layer
    gemm(ah, al, acc);
    {
      const float* b2 = BlobPtr<float>(blob, p.pw2.bias);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        float* uc = u + acc_col(i) * LDU + acc_row(i);
        const float val = __fadd_rn(__fadd_rn(acc[i], b2[acc_col(i)]), has_rows ? *uc : 0.0f);
        if (unit == 2) acc[i] = LeakyRelu(val);
        else if (has_rows) *uc = val;
      }
      if (unit == 2) DwAccToA(acc, ah, al);
      else row_sync();                                       // u' complete before anybody reads a neighbour's rows
    }
  };
  unit_body(std::integral_constant<int, 0>());
  unit_body(std::integral_constant<int, 1>());
  unit_body(std::integral_constant<int, 2>());

  // ---- last_layer.  P[row][tap * 16 + n] from the GEMM goes to shared memory (the u buffer, same [column][row] layout; a thread
  //      only touches the elements it read itself above), then output row q (0..22) sums its four taps:
  //      out[q][n] = sum_tap P[q + tap - 3][tap][n]
  gemm(ah, al, acc);
  if (has_rows) {
#pragma unroll
    for (int i = 0; i < 32; ++i) u[acc_col(i) * LDU + acc_row(i)] = acc[i];
  }
  lyra_mbar_wait(&sh->in_full, 0);                           // the carried last_layer tail (loaded at kernel start)
  row_sync();
  int16_t* stage = reinterpret_cast<int16_t*>(smem + L::kStage);      // [S][320]
  if (tid < 23 * S) {
    const int q = tid / S, ss = tid % S;
    const float bias = BlobPtr<float>(blob, P.last.bias)[0];
#pragma unroll
    for (int n = 0; n < 16; ++n) {
      float a = 0.0f;
#pragma unroll
      for (int tap = 0; tap < 4; ++tap) {
        const int tr = q + tap - 3;
        if (tr >= 0 && tr < 20) a = __fadd_rn(a, u[(tap * 16 + n) * LDU + tr * S + ss]);
      }
      const int tt = 16 * q + n;
      const float y = __fadd_rn(__fadd_rn(a, bias), tt < 48 ? sl[tt * S + ss] : 0.0f);
      if (tt < 320) {
        // UnitToInt16Scalar (dsp_utils.h:53-60,79-88): scale, clip in float, truncate
        float x = __fmul_rn(y, 32768.0f);
        x = x > -32768.0f ? x : -32768.0f;
        x = x < 32767.0f ? x : 32767.0f;
        stage[ss * 320 + tt] = (int16_t)(int)x;
      } else {
        slo[(tt - 320) * S + ss] = active[ss] ? __fsub_rn(y, bias) : sl[(tt - 320) * S + ss];
      }
    }
  }
  lyra_fence_proxy_async();
  row_sync();
  if (tid == 0) { lyra_bulk_s2g(st + (size_t)DecStateD::kLast * S, slo, 48u * S * 4); lyra_bulk_commit(); }
  for (int i = tid; i < S * 320 / 2; i += L::kRowThreads) {         // two samples per store
    const int ss = (2 * i) / 320;
    if (active[ss]) *reinterpret_cast<uint32_t*>(pcm + (size_t)slot[ss] * 320 + (2 * i) % 320) = reinterpret_cast<const uint32_t*>(stage)[i];
  }
  AdvanceHopCounters<S>(n18g, tile, active, n18);
  if (tid == 0) lyra_bulk_wait_all();                        // every state block is in global memory before the block exits
}

}  // namespace lyra_b200
