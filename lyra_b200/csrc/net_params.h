// Plain-old-data layer descriptors shared by the host-side spec builder (model_spec.cc) and the
// kernels.  All weights live in ONE device blob; descriptors hold byte offsets into it.
//
// Layer naming follows the reference graphs (SURVEY.md App. A):
//   encoder: first_layer -> encoder_0 (3 res-units @64, T=20) -> encoder_0/simpleconv (K10 s5)
//            -> encoder_1 (3 res-units @128, T=4) -> encoder_1/simpleconv (K4 s2, g2)
//            -> encoder_2/resnet_0 (mixed f32/int8 @256, T=2) -> quant_encoder_2 (2 int8 res-units)
//            -> quant_encoder_2/simpleconv (K4 s2, g4) -> quant_bottleneck_1 (K3, g4) -> f32[64]
//   decoder: bottleneck_2 (K3, g4) -> quant_decoder_0 upsample (4 int8 transposed convs) -> 3 int8
//            res-units @256 -> quant_decoder_1 upsample (2 int8 transposed convs) -> decoder_1
//            (3 res-units @128, T=4) -> decoder_2/simple (transposed K10 s5) -> decoder_2
//            (3 res-units @64, T=20) -> last_layer (transposed K64 s16) -> f32[320]
#pragma once

#include <stdint.h>

namespace lyra_b200 {

// fp32 GEMM-shaped convolution: weights [Ktot][N] k-major (k = tap*CinG + ci), bias [N]
// wf: the same [K][N] matrix in mma.sync m16n8k8 B-fragment order [K/8][N/8][32 lanes] x float2 (decoder layers only;
// 0 = not packed) for the decoder's tensor-core mode
struct GemmF32 { uint32_t w, bias, wf; };
// int8 convolution: weights in mma.sync m16n8k32 B-fragment order [Ktot/32][N/8][32 lanes][2 words]
// (k = tap*CinG + ci), bias folded with the input zero point (bias + (-zp_in) * sum(w)), per-channel Q31
// multiplier and shift
struct GemmI8 { uint32_t w, bias, mult, shift; int32_t out_zp; int32_t in_zp; };
struct DwF32 { uint32_t w, bias; };                       // w [3][C]
struct DwI8 { uint32_t w, bias, mult, shift; int32_t out_zp; int32_t in_zp; };   // w [3][C] int32
struct LReluQ { uint32_t lut; };                          // int8[256], index = q + 128
struct AddQ { uint32_t lut1, lut2; int32_t m3, s3, out_zp; };   // int32[256] each
struct QuantP { float scale; int32_t zp; };

struct ResF32 { DwF32 dw; GemmF32 pw1, pw2; };
struct ResI8 { DwI8 dw; GemmI8 pw1; LReluQ lr1; GemmI8 pw2; AddQ add; LReluQ lr2; };

struct EncoderParams {
  // ---- kernel A: T = 20, 64 channels
  GemmF32 first;            // first_layer: K=64 s=16, 1 -> 64
  ResF32 r0[3];             // encoder_0/resnet_{0,1,2}: dilation 1/3/9
  GemmF32 down0;            // encoder_0/simpleconv: K=10 s=5, 64 -> 128
  // ---- kernel B: T = 4 / 2 / 1
  ResF32 r1[3];             // encoder_1/resnet_*: second 1x1 has groups = 2
  GemmF32 down1;            // encoder_1/simpleconv: K=4 s=2, 128 -> 256, groups = 2
  DwF32 m_dw;               // encoder_2/resnet_0 (mixed precision unit)
  GemmF32 m_pw1;
  QuantP m_q1; LReluQ m_lr1; GemmI8 m_pw2; QuantP m_dq; QuantP m_q2; LReluQ m_lr2;
  ResI8 q[2];               // quant_encoder_2/resnet_{1,2}: dilation 3/9
  GemmI8 down2; LReluQ down2_lr;   // quant_encoder_2/simpleconv: K=4 s=2, 256 -> 512, g = 4
  GemmI8 bott; QuantP out_dq;      // quant_bottleneck_1: K=3, 512 -> 64, g = 4; DEQUANTIZE
  // zero points used to initialise int8 state (real value 0): ring of q[0], q[1], down2, bott
  int32_t zp_state[4];
};

// A bank of G parallel int8 TRANSPOSE_CONVs over a channel split (quant_decoder_{0,1}/simple_g*), fused
// into one grouped tap-GEMM: B-fragment-order weights over k = (j,ci), columns g*128 + r*64 + co, per-column bias/mult/shift.
struct UpI8 {
  GemmI8 g;                 // out_zp unused (per group below); in_zp = zero point of the shared input
  QuantP dq[4];             // DEQUANTIZE of each group's int8 output
  int32_t out_zp[4];
  uint32_t bias_f32[4];     // the f32 constants subtracted from the overlap tails (SUB ops), [64] each
};

// Kernel D's GEMM weights for the tensor-core decoder (DecoderKernelDW): kDuNumChunks chunks of kDuChunkBytes.  A chunk is a
// [rows x kc] slice of one layer's weight operand, split into hi + lo (hi = the 19 bits a TF32 operand keeps, lo = x - hi) and
// stored as [hi part][lo part], each part in the K-major no-swizzle core-matrix layout [kc/4][rows/8][8 rows][4 k] that a wgmma
// shared-memory descriptor addresses with LBO = (rows/8) * 128 bytes and SBO = 128 bytes.  One chunk = one bulk copy = one
// stage of the kernel's weight ring.
//   chunks  0..39  decoder_2/simple, as the A operand (the GEMM is computed transposed: weights are the rows, the 32
//                  (input row, stream) pairs the columns): row m = (tap j, phase r, cout) = j * 320 + r * 64 + co (rows 640..
//                  are zero padding), k = cin; 128-row block major (5 blocks), 16 k per chunk
//   chunks 40..51  decoder_2/resnet_{0,1,2}: pw1 (2 chunks of 32 k), pw2 (2 chunks), B operand, row = cout
//   chunks 52..53  last_layer as ONE 64 x 64 GEMM: B row = tap * 16 + n (n = output sample within the stride), k = cin;
//                  the four taps are summed across time rows in the epilogue
constexpr int kDuChunkBytes = 16384;
constexpr int kDuNumChunks = 54;
constexpr int kDuUp2Chunks = 40, kDuUnitChunk0 = 40, kDuLastChunk0 = 52;

struct DecoderParams {
  // ---- kernel C: T = 1 / 2 / 4
  GemmF32 bott;             // bottleneck_2/simpleconv: K=3, 64 -> 512, g = 4
  QuantP bott_q;            // QUANTIZE after its LeakyReLU
  UpI8 up0;                 // quant_decoder_0/simple_g{0..3}: K=4 s=2, 128 -> 64 each
  QuantP up0_q;             // QUANTIZE of LeakyReLU(concat)
  // quant_decoder_0/resnet_0 is mixed: int8 body, f32 residual add
  DwI8 m_dw; GemmI8 m_pw1; LReluQ m_lr1; GemmI8 m_pw2; QuantP m_dq; QuantP m_q2; LReluQ m_lr2;
  ResI8 q[2];               // quant_decoder_0/resnet_{1,2}
  UpI8 up1;                 // quant_decoder_1/simple_g{0,1}: K=4 s=2, 128 -> 64 each
  ResF32 r1[3];             // decoder_1/resnet_*: 128 ch, second 1x1 groups = 2
  // ---- kernel D: T = 20
  GemmF32 up2;              // decoder_2/simple: transposed K=10 s=5, 128 -> 64; weights [(j,ci)][(r,co)], bias [64]
  ResF32 r2[3];             // decoder_2/resnet_*: 64 ch
  GemmF32 last;             // last_layer: transposed K=64 s=16, 64 -> 1; weights [(j,ci)][r], bias [1]
  uint32_t du_chunks;       // the tensor-core decoder's weight chunks (see kDuChunkBytes)
  int32_t zp_state[3];      // int8 ring zero points: m_dw ring, q[0], q[1]
};

struct RvqParams {
  uint32_t codebooks_t;     // f32 [46][64][16]  (stage, dim, code): transposed for conflict-free lanes
  uint32_t codebooks;       // f32 [46][16][64]
  int32_t num_stages;       // 46
};

struct LogMelParams {
  uint32_t window;          // f64 [640]
  uint32_t twiddle;         // f64 [1023][2] per-stage tables, stage of half-length h at entry h-1: cos, sin of -2*pi*k/(2h), k < h
  uint32_t weights;         // f64 [513]
  uint32_t band;            // i32 [513]
  uint32_t range;           // i32 [num_mel][2]: first / last spectrum bin that contributes to the channel (bands ch-1 and ch)
  int32_t start_index, end_index, num_mel, fft, window_len, hop;
};

// Comfort-noise generator (lyra/comfort_noise_generator.cc:37-119) for (16 kHz, hop 320, window 640, 160 mel bins): the mel
// tables are those of the 160-bin log-mel extractor; norm = per-channel sum of filter weights (mel inverse), synth = synthesis
// window incl. the power-preserving constant, fade = the decoder's raised-cosine cross-fade weights
// (1 + cos(p * pi / 640)) / 2 for fade progress p = 0..640 (lyra/lyra_decoder.cc:364-366), all computed on the host with the
// oracle's expressions.
struct CngParams {
  uint32_t weights, band;   // f64 [513], i32 [513]  (shared with LogMelParams of 160 bins)
  uint32_t norm;            // f64 [160]
  uint32_t synth;           // f64 [1024]
  uint32_t twiddle;         // f64 [1023][2], the FFT's per-stage tables (shared)
  uint32_t fade;            // f32 [641]
  int32_t start_index, end_index, num_mel, fft, hop;
};

// Sample-rate converters (lyra/resampler.cc:31-66): polyphase Kaiser-windowed-sinc filter banks for the six (external <-> 16 kHz)
// pairs.  Pair index: 0: 8k->16k, 1: 32k->16k, 2: 48k->16k, 3: 16k->8k, 4: 16k->32k, 5: 16k->48k.  coeffs[pair] = f32 [den][35].
struct ResamplerParams {
  uint32_t coeffs[6];
  int32_t num[6], den[6];
};
constexpr int kResamplerTaps = 35;

}  // namespace lyra_b200
