// See model_spec.h.
#include "model_spec.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <stdexcept>

#include "tflite_model.h"

namespace lyra_b200 {

// ---------------------------------------------------------------- fixed point ----

void QuantizeMultiplier(double real_multiplier, int32_t* qm, int* shift) {
  if (real_multiplier == 0.0) { *qm = 0; *shift = 0; return; }
  const double q = std::frexp(real_multiplier, shift);
  int64_t q_fixed = (int64_t)std::round(q * (double)(1ll << 31));
  if (q_fixed == (1ll << 31)) { q_fixed /= 2; ++*shift; }
  if (*shift < -31) { *shift = 0; q_fixed = 0; }
  *qm = (int32_t)q_fixed;
}

int32_t MultiplyByQuantizedMultiplier(int32_t x, int32_t qm, int shift) {
  const int left = shift > 0 ? shift : 0, right = shift > 0 ? 0 : -shift;
  const int32_t xs = x * (1 << left);
  // saturating rounding doubling high multiply
  int32_t hi;
  if (xs == qm && xs == INT32_MIN) {
    hi = INT32_MAX;
  } else {
    const int64_t ab = (int64_t)xs * (int64_t)qm;
    const int32_t nudge = ab >= 0 ? (1 << 30) : (1 - (1 << 30));
    hi = (int32_t)((ab + nudge) / (1ll << 31));
  }
  // rounding divide by power of two
  const int32_t mask = (int32_t)((1ll << right) - 1);
  const int32_t rem = hi & mask;
  const int32_t thr = (mask >> 1) + (hi < 0 ? 1 : 0);
  return (hi >> right) + (rem > thr ? 1 : 0);
}

namespace {

#define SPEC_CHECK(cond, msg) do { if (!(cond)) throw std::runtime_error(std::string("model_spec: ") + msg); } while (0)

int ClampI8(int v) { return v < -128 ? -128 : (v > 127 ? 127 : v); }

template <typename T>
uint32_t Append(std::vector<uint8_t>* blob, const std::vector<T>& v) {
  while (blob->size() % 16) blob->push_back(0);
  const size_t off = blob->size();
  const size_t nb = v.size() * sizeof(T);
  blob->resize(off + nb);
  if (nb) std::memcpy(blob->data() + off, v.data(), nb);
  SPEC_CHECK(off < 0xffffffffull, "blob too large");
  return (uint32_t)off;
}

// B operand of mma.sync.m16n8k32 (s8) in fragment order: for k-step ks (32 k-values), n-tile nt (8 columns) and
// lane L (g = L / 4, t = L % 4) two words: {B[32ks + 4t .. +3][8nt + g], B[32ks + 16 + 4t .. +3][8nt + g]}, bytes in
// ascending k.  `b` is the dense [K][N] int8 matrix (k-major).
std::vector<uint32_t> PackMmaB(const std::vector<int8_t>& b, int K, int N) {
  SPEC_CHECK(K % 32 == 0 && N % 8 == 0, "MMA operand: K must be a multiple of 32 and N of 8");
  std::vector<uint32_t> out((size_t)(K / 32) * (N / 8) * 64, 0u);
  for (int ks = 0; ks < K / 32; ++ks)
    for (int nt = 0; nt < N / 8; ++nt)
      for (int lane = 0; lane < 32; ++lane) {
        const int g = lane / 4, t = lane % 4;
        for (int half = 0; half < 2; ++half) {
          uint32_t w = 0;
          for (int byte = 0; byte < 4; ++byte) {
            const int k = 32 * ks + 16 * half + 4 * t + byte;
            w |= (uint32_t)(uint8_t)b[(size_t)k * N + 8 * nt + g] << (8 * byte);
          }
          out[(((size_t)ks * (N / 8) + nt) * 32 + lane) * 2 + half] = w;
        }
      }
  return out;
}

// fp32 GEMM B operand ([K][N], k-major) in mma.sync m16n8k8 (tf32) fragment order: for every k-step ks (8 k) and n-tile
// nt (8 n), lane L (g = L / 4, t = L % 4) holds {B[8ks + t][8nt + g], B[8ks + t + 4][8nt + g]}.
std::vector<float> PackMmaBTf32(const std::vector<float>& b, int K, int N) {
  SPEC_CHECK(K % 8 == 0 && N % 8 == 0, "TF32 MMA operand: K and N must be multiples of 8");
  std::vector<float> out((size_t)(K / 8) * (N / 8) * 64, 0.0f);
  for (int ks = 0; ks < K / 8; ++ks)
    for (int nt = 0; nt < N / 8; ++nt)
      for (int lane = 0; lane < 32; ++lane) {
        const int g = lane / 4, t = lane % 4;
        float* o = &out[(((size_t)ks * (N / 8) + nt) * 32 + lane) * 2];
        o[0] = b[(size_t)(8 * ks + t) * N + 8 * nt + g];
        o[1] = b[(size_t)(8 * ks + t + 4) * N + 8 * nt + g];
      }
  return out;
}

// One chunk of the tensor-core decoder's weight stream (net_params.h kDuChunkBytes): elem(row, k) for row < rows, k < kc as
// [hi part][lo part], each [kc/4][rows/8][8][4] floats.
template <typename Elem>
void AppendDuChunk(std::vector<uint8_t>* out, int rows, int kc, Elem elem) {
  SPEC_CHECK(kc % 8 == 0 && rows % 8 == 0 && (size_t)2 * kc * rows * 4 <= (size_t)kDuChunkBytes, "tensor-core weight chunk shape");
  std::vector<float> part((size_t)2 * kc * rows, 0.0f);
  for (int k = 0; k < kc; ++k)
    for (int n = 0; n < rows; ++n) {
      const float x = elem(n, k);
      uint32_t bits;
      std::memcpy(&bits, &x, 4);
      bits &= 0xffffe000u;
      float hi;
      std::memcpy(&hi, &bits, 4);
      const float lo = x - hi;                                   // exact in fp32
      const size_t idx = ((size_t)(k / 4) * (rows / 8) + n / 8) * 32 + (size_t)(n % 8) * 4 + k % 4;
      part[idx] = hi;
      part[(size_t)kc * rows + idx] = lo;
    }
  const size_t off = out->size();
  out->resize(off + kDuChunkBytes, 0);
  std::memcpy(out->data() + off, part.data(), part.size() * 4);
}

// k-major fp32 GEMM matrices, collected in packing order (kernel D's GEMMs: the source of the tensor-core weight chunks)
using GemmList = std::vector<std::vector<float>>;

struct Net {
  const TflModel& m;
  const TflSubgraph& g;
  std::vector<int> convs;   // CONV_2D / DEPTHWISE_CONV_2D / TRANSPOSE_CONV ops in graph order
  std::vector<uint8_t>* blob;

  Net(const TflModel& model, int sg, std::vector<uint8_t>* b) : m(model), g(model.subgraphs()[sg]), blob(b) {
    for (size_t i = 0; i < g.ops.size(); ++i) {
      const int c = g.ops[i].code;
      if (c == kConv2D || c == kDepthwiseConv2D || c == kTransposeConv) convs.push_back((int)i);
    }
  }
  const TflOp& op(int i) const { SPEC_CHECK(i >= 0 && (size_t)i < g.ops.size(), "operator index out of range"); return g.ops[(size_t)i]; }
  const TflTensor& T(int i) const { SPEC_CHECK(i >= 0 && (size_t)i < g.tensors.size(), "tensor index out of range"); return g.tensors[(size_t)i]; }
  const TflOp& conv(int i) const { return op(convs.at((size_t)i)); }
  static int In(const TflOp& o, size_t i) { SPEC_CHECK(i < o.inputs.size(), "operator has too few inputs"); return o.inputs[i]; }
  static int Out(const TflOp& o, size_t i) { SPEC_CHECK(i < o.outputs.size(), "operator has too few outputs"); return o.outputs[i]; }

  // tensor roles of a conv-like op
  int in_tensor(const TflOp& o) const { return o.code == kTransposeConv ? In(o, 2) : In(o, 0); }
  int w_tensor(const TflOp& o) const { return In(o, 1); }
  int b_tensor(const TflOp& o) const { return o.code == kTransposeConv ? In(o, 3) : In(o, 2); }

  int next(int tensor, int code) const { return g.sole_consumer(tensor, code); }
  int out0(int opi) const { return Out(op(opi), 0); }

  void expect_conv(const TflOp& o, int code, DType wt, int cout, int k, int cing, int stride, int dil = 1) const {
    const TflTensor& w = T(w_tensor(o));
    SPEC_CHECK(o.code == code, "unexpected op kind in conv sequence");
    SPEC_CHECK(w.type == wt, "unexpected weight type");
    SPEC_CHECK(w.shape.size() == 4 && w.shape[2] == 1, "unexpected filter rank");
    if (code == kDepthwiseConv2D) {
      SPEC_CHECK(w.shape[0] == 1 && w.shape[1] == k && w.shape[3] == cout, "unexpected depthwise filter shape");
      SPEC_CHECK(m.OptI32(o, 2, 1) == 1 && m.OptI32(o, 6, 1) == dil && m.OptI32(o, 3, 1) == 1, "unexpected depthwise options");
      SPEC_CHECK(m.OptI8(o, 0, 0) == 1 && m.OptI8(o, 4, 0) == 0, "depthwise padding/activation");
    } else {
      SPEC_CHECK(w.shape[0] == cout && w.shape[1] == k && w.shape[3] == cing, "unexpected filter shape");
      SPEC_CHECK(m.OptI32(o, 2, 1) == stride, "unexpected stride");
      SPEC_CHECK(m.OptI8(o, 0, 0) == 1, "padding must be VALID");
      if (code == kConv2D) SPEC_CHECK(m.OptI32(o, 5, 1) == 1 && m.OptI8(o, 3, 0) == 0, "conv dilation/activation");
    }
  }

  // ---- packers -------------------------------------------------------------------------------
  // tf32_frags: also append the mma.sync TF32 fragment-order copy (GemmF32::wf);  gemms: if given, receives the k-major matrix
  GemmF32 PackConvF32(const TflOp& o, bool tf32_frags = false, GemmList* gemms = nullptr) const {
    const TflTensor& w = T(w_tensor(o));
    const TflTensor& b = T(b_tensor(o));
    SPEC_CHECK(w.shape.size() == 4 && w.type == DType::F32 && b.type == DType::F32, "conv: filter rank / type");
    const int Cout = w.shape[0], K = w.shape[1], CinG = w.shape[3];
    SPEC_CHECK(Cout > 0 && K > 0 && CinG > 0 && w.shape[2] == 1, "conv: filter shape");
    std::vector<float> wt((size_t)K * CinG * Cout);
    const float* src = w.as<float>();
    for (int co = 0; co < Cout; ++co)
      for (int k = 0; k < K; ++k)
        for (int ci = 0; ci < CinG; ++ci)
          wt[((size_t)k * CinG + ci) * Cout + co] = src[((size_t)co * K + k) * CinG + ci];
    SPEC_CHECK((int)b.count() == Cout, "conv bias");
    std::vector<float> bias(b.as<float>((size_t)Cout), b.as<float>((size_t)Cout) + Cout);
    const uint32_t wf = tf32_frags ? Append(blob, PackMmaBTf32(wt, K * CinG, Cout)) : 0u;
    if (gemms) gemms->push_back(wt);
    return GemmF32{Append(blob, wt), Append(blob, bias), wf};
  }

  // transposed conv as a J-tap GEMM over (r, co) outputs: W'[(j,ci)][(r,co)] = W[co][r + s*(J-1-j)][ci]; both fp32 ones are kernel D
  // GEMMs, so the k-major matrix also goes to `gemms`
  GemmF32 PackTconvF32(const TflOp& o, int stride, GemmList* gemms) const {
    const TflTensor& w = T(w_tensor(o));
    const TflTensor& b = T(b_tensor(o));
    SPEC_CHECK(w.shape.size() == 4 && w.type == DType::F32 && b.type == DType::F32, "transposed conv: filter rank / type");
    const int Cout = w.shape[0], K = w.shape[1], Cin = w.shape[3];
    SPEC_CHECK(Cout > 0 && K > 0 && Cin > 0 && w.shape[2] == 1 && K % stride == 0, "transposed conv: K must be a multiple of the stride");
    const int J = K / stride, N = stride * Cout;
    std::vector<float> wt((size_t)J * Cin * N);
    const float* src = w.as<float>();
    for (int j = 0; j < J; ++j)
      for (int ci = 0; ci < Cin; ++ci)
        for (int r = 0; r < stride; ++r)
          for (int co = 0; co < Cout; ++co)
            wt[((size_t)j * Cin + ci) * N + (size_t)r * Cout + co] = src[((size_t)co * K + (r + stride * (J - 1 - j))) * Cin + ci];
    std::vector<float> bias(b.as<float>((size_t)Cout), b.as<float>((size_t)Cout) + Cout);
    gemms->push_back(wt);
    return GemmF32{Append(blob, wt), Append(blob, bias), 0u};
  }

  void RequantArrays(const TflTensor& x, const TflTensor& w, const TflTensor& y, int n, int repeat,
                     std::vector<int32_t>* mult, std::vector<int32_t>* shift) const {
    // kernel_util.cc PopulateConvolutionQuantizationParams: per-channel effective scale in double
    for (int r = 0; r < repeat; ++r)
      for (int c = 0; c < n; ++c) {
        const float fs = w.scale[w.scale.size() > 1 ? (size_t)c : 0];
        const double eff = (double)x.scale0() * (double)fs / (double)y.scale0();
        int32_t qm; int sh;
        QuantizeMultiplier(eff, &qm, &sh);
        mult->push_back(qm);
        shift->push_back(sh);
      }
  }

  GemmI8 PackConvI8(const TflOp& o) const {
    const TflTensor& w = T(w_tensor(o));
    const TflTensor& b = T(b_tensor(o));
    const TflTensor& x = T(in_tensor(o));
    const TflTensor& y = T(Out(o, 0));
    SPEC_CHECK(w.shape.size() == 4 && w.type == DType::I8 && b.type == DType::I32, "int8 conv: filter rank / type");
    const int Cout = w.shape[0], K = w.shape[1], CinG = w.shape[3];
    SPEC_CHECK(Cout > 0 && K > 0 && w.shape[2] == 1 && CinG > 0 && CinG % 32 == 0, "int8 conv: CinG must be a multiple of 32");
    std::vector<int8_t> dense((size_t)K * CinG * Cout);
    std::vector<int32_t> bias(Cout), mult, shift;
    const int8_t* src = w.as<int8_t>();
    const int32_t* bsrc = b.as<int32_t>((size_t)Cout);
    const int in_zp = x.zp0();
    SPEC_CHECK(w.scale.size() == 1 || w.scale.size() == (size_t)Cout, "int8 conv: per-channel scale count");
    for (int co = 0; co < Cout; ++co) {
      int64_t wsum = 0;
      for (int k = 0; k < K; ++k)
        for (int ci = 0; ci < CinG; ++ci) {
          const int8_t v = src[((size_t)co * K + k) * CinG + ci];
          wsum += v;
          dense[((size_t)k * CinG + ci) * Cout + co] = v;
        }
      bias[co] = (int32_t)(bsrc[co] - (int64_t)in_zp * wsum);
    }
    RequantArrays(x, w, y, Cout, 1, &mult, &shift);
    return GemmI8{Append(blob, PackMmaB(dense, K * CinG, Cout)), Append(blob, bias), Append(blob, mult), Append(blob, shift), y.zp0(), in_zp};
  }

  DwF32 PackDwF32(const TflOp& o) const {
    const TflTensor& w = T(w_tensor(o));
    const TflTensor& b = T(b_tensor(o));
    SPEC_CHECK(w.shape.size() == 4 && w.type == DType::F32 && b.type == DType::F32 && (int)b.count() == w.shape[3], "depthwise: filter rank / type / bias");
    std::vector<float> wt(w.as<float>(), w.as<float>() + w.count());
    std::vector<float> bias(b.as<float>(), b.as<float>() + b.count());
    return DwF32{Append(blob, wt), Append(blob, bias)};
  }

  DwI8 PackDwI8(const TflOp& o) const {
    const TflTensor& w = T(w_tensor(o));
    const TflTensor& b = T(b_tensor(o));
    const TflTensor& x = T(in_tensor(o));
    const TflTensor& y = T(Out(o, 0));
    SPEC_CHECK(w.shape.size() == 4 && w.type == DType::I8 && b.type == DType::I32, "int8 depthwise: filter rank / type");
    const int K = w.shape[1], C = w.shape[3];
    SPEC_CHECK(K > 0 && C > 0 && w.shape[0] == 1 && w.shape[2] == 1, "int8 depthwise: filter shape");
    SPEC_CHECK(w.scale.size() == 1 || w.scale.size() == (size_t)C, "int8 depthwise: per-channel scale count");
    std::vector<int32_t> wt((size_t)K * C), bias(C), mult, shift;
    const int in_zp = x.zp0();
    const int8_t* wsrc = w.as<int8_t>((size_t)K * C);
    const int32_t* bsrc = b.as<int32_t>((size_t)C);
    for (int c = 0; c < C; ++c) {
      int64_t wsum = 0;
      for (int k = 0; k < K; ++k) { wt[(size_t)k * C + c] = wsrc[(size_t)k * C + c]; wsum += wt[(size_t)k * C + c]; }
      bias[c] = (int32_t)(bsrc[c] - (int64_t)in_zp * wsum);
    }
    RequantArrays(x, w, y, C, 1, &mult, &shift);
    return DwI8{Append(blob, wt), Append(blob, bias), Append(blob, mult), Append(blob, shift), y.zp0(), in_zp};
  }

  QuantP QP(int tensor) const { return QuantP{T(tensor).scale0(), T(tensor).zp0()}; }

  // int8 LEAKY_RELU as a 256-entry table (kernels/activations.cc LeakyReluPrepare + QuantizeLeakyRelu)
  LReluQ PackLRelu(int opi) const {
    const TflOp& o = op(opi);
    SPEC_CHECK(o.code == kLeakyRelu, "expected LEAKY_RELU");
    const TflTensor& x = T(In(o, 0));
    const TflTensor& y = T(Out(o, 0));
    SPEC_CHECK(x.type == DType::I8 && y.type == DType::I8, "expected int8 LEAKY_RELU");
    const float alpha = m.OptF32(o, 0, 0.0f);
    const double alpha_mult = (double)(x.scale0() * alpha / y.scale0());   // float expression, widened
    const double ident_mult = (double)(x.scale0() / y.scale0());
    int32_t ma, mi; int sa, si;
    QuantizeMultiplier(alpha_mult, &ma, &sa);
    QuantizeMultiplier(ident_mult, &mi, &si);
    std::vector<int8_t> lut(256);
    for (int q = -128; q < 128; ++q) {
      const int32_t v = q - x.zp0();
      const int32_t u = y.zp0() + (v >= 0 ? MultiplyByQuantizedMultiplier(v, mi, si) : MultiplyByQuantizedMultiplier(v, ma, sa));
      lut[(size_t)(q + 128)] = (int8_t)ClampI8(u);
    }
    return LReluQ{Append(blob, lut)};
  }

  // int8 ADD: per-input scaled terms as tables, final rescale on device (kernels/add.cc + integer_ops/add.h)
  AddQ PackAdd(int opi) const {
    const TflOp& o = op(opi);
    SPEC_CHECK(o.code == kAdd && m.OptI8(o, 0, 0) == 0, "expected ADD without activation");
    const TflTensor& a = T(In(o, 0));
    const TflTensor& b = T(In(o, 1));
    const TflTensor& y = T(Out(o, 0));
    SPEC_CHECK(a.type == DType::I8 && b.type == DType::I8, "expected int8 ADD");
    const int left_shift = 20;
    const float maxs = a.scale0() > b.scale0() ? a.scale0() : b.scale0();
    const double twice_max = (double)(2 * maxs);
    const double r1 = (double)a.scale0() / twice_max, r2 = (double)b.scale0() / twice_max;
    const double ro = twice_max / (double)((float)(1 << left_shift) * y.scale0());
    int32_t m1, m2, m3; int s1, s2, s3;
    QuantizeMultiplier(r1, &m1, &s1);
    QuantizeMultiplier(r2, &m2, &s2);
    QuantizeMultiplier(ro, &m3, &s3);
    std::vector<int32_t> l1(256), l2(256);
    for (int q = -128; q < 128; ++q) {
      l1[(size_t)(q + 128)] = MultiplyByQuantizedMultiplier((q - a.zp0()) * (1 << left_shift), m1, s1);
      l2[(size_t)(q + 128)] = MultiplyByQuantizedMultiplier((q - b.zp0()) * (1 << left_shift), m2, s2);
    }
    return AddQ{Append(blob, l1), Append(blob, l2), m3, s3, y.zp0()};
  }

  ResF32 PackResF32(int first_conv, int C, int dil, int groups2, bool tf32_frags = false, GemmList* gemms = nullptr) const {
    expect_conv(conv(first_conv), kDepthwiseConv2D, DType::F32, C, 3, C, 1, dil);
    expect_conv(conv(first_conv + 1), kConv2D, DType::F32, C, 1, C, 1);
    expect_conv(conv(first_conv + 2), kConv2D, DType::F32, C, 1, C / groups2, 1);
    return ResF32{PackDwF32(conv(first_conv)), PackConvF32(conv(first_conv + 1), tf32_frags, gemms),
                  PackConvF32(conv(first_conv + 2), tf32_frags, gemms)};
  }

  ResI8 PackResI8(int first_conv, int C, int dil) const {
    expect_conv(conv(first_conv), kDepthwiseConv2D, DType::I8, C, 3, C, 1, dil);
    expect_conv(conv(first_conv + 1), kConv2D, DType::I8, C, 1, C, 1);
    expect_conv(conv(first_conv + 2), kConv2D, DType::I8, C, 1, C / 4, 1);
    ResI8 r;
    r.dw = PackDwI8(conv(first_conv));
    r.pw1 = PackConvI8(conv(first_conv + 1));
    const int lr1 = next(Out(conv(first_conv + 1), 0), kLeakyRelu);
    r.lr1 = PackLRelu(lr1);
    SPEC_CHECK(in_tensor(conv(first_conv + 2)) == out0(lr1), "res-unit wiring (pw2 input)");
    r.pw2 = PackConvI8(conv(first_conv + 2));
    const int add = next(Out(conv(first_conv + 2), 0), kAdd);
    SPEC_CHECK(In(op(add), 0) == Out(conv(first_conv + 2), 0), "res-unit ADD operand order");
    r.add = PackAdd(add);
    r.lr2 = PackLRelu(next(out0(add), kLeakyRelu));
    return r;
  }
};

EncoderParams BuildEncoder(const TflModel& m, std::vector<uint8_t>* blob) {
  int sg = m.SignatureSubgraph("serving_default");
  if (sg < 0) sg = 0;
  Net n(m, sg, blob);
  SPEC_CHECK(n.convs.size() == 32, "encoder: expected 32 convolution ops");
  EncoderParams p;
  std::memset(&p, 0, sizeof(p));
  n.expect_conv(n.conv(0), kConv2D, DType::F32, 64, 64, 1, 16);
  p.first = n.PackConvF32(n.conv(0));
  const int dil[3] = {1, 3, 9};
  for (int i = 0; i < 3; ++i) p.r0[i] = n.PackResF32(1 + 3 * i, 64, dil[i], 1);
  n.expect_conv(n.conv(10), kConv2D, DType::F32, 128, 10, 64, 5);
  p.down0 = n.PackConvF32(n.conv(10));
  for (int i = 0; i < 3; ++i) p.r1[i] = n.PackResF32(11 + 3 * i, 128, dil[i], 2);
  n.expect_conv(n.conv(20), kConv2D, DType::F32, 256, 4, 64, 2);
  p.down1 = n.PackConvF32(n.conv(20));
  // encoder_2/resnet_0: f32 dw + f32 1x1, then int8
  n.expect_conv(n.conv(21), kDepthwiseConv2D, DType::F32, 256, 3, 256, 1, 1);
  n.expect_conv(n.conv(22), kConv2D, DType::F32, 256, 1, 256, 1);
  n.expect_conv(n.conv(23), kConv2D, DType::I8, 256, 1, 64, 1);
  p.m_dw = n.PackDwF32(n.conv(21));
  p.m_pw1 = n.PackConvF32(n.conv(22));
  const int q1 = n.next(Net::Out(n.conv(22), 0), kQuantize);
  p.m_q1 = n.QP(n.out0(q1));
  const int lr1 = n.next(n.out0(q1), kLeakyRelu);
  p.m_lr1 = n.PackLRelu(lr1);
  SPEC_CHECK(n.in_tensor(n.conv(23)) == n.out0(lr1), "encoder mixed unit wiring");
  p.m_pw2 = n.PackConvI8(n.conv(23));
  const int dq = n.next(Net::Out(n.conv(23), 0), kDequantize);
  p.m_dq = n.QP(Net::Out(n.conv(23), 0));
  const int addf = n.next(n.out0(dq), kAdd);
  SPEC_CHECK(Net::In(n.op(addf), 1) == Net::Out(n.conv(20), 0), "encoder mixed unit residual");
  const int q2 = n.next(n.out0(addf), kQuantize);
  p.m_q2 = n.QP(n.out0(q2));
  // the quantised sum feeds both the next unit's ADD and a LEAKY_RELU
  p.m_lr2 = n.PackLRelu(n.next(n.out0(q2), kLeakyRelu));
  p.q[0] = n.PackResI8(24, 256, 3);
  p.q[1] = n.PackResI8(27, 256, 9);
  n.expect_conv(n.conv(30), kConv2D, DType::I8, 512, 4, 64, 2);
  p.down2 = n.PackConvI8(n.conv(30));
  p.down2_lr = n.PackLRelu(n.next(Net::Out(n.conv(30), 0), kLeakyRelu));
  n.expect_conv(n.conv(31), kConv2D, DType::I8, 64, 3, 128, 1);
  p.bott = n.PackConvI8(n.conv(31));
  p.out_dq = n.QP(Net::Out(n.conv(31), 0));
  SPEC_CHECK(!n.g.outputs.empty() && n.T(n.g.outputs[0]).count() == 64, "encoder output size");
  p.zp_state[0] = p.q[0].dw.in_zp;
  p.zp_state[1] = p.q[1].dw.in_zp;
  p.zp_state[2] = p.down2.in_zp;
  p.zp_state[3] = p.bott.in_zp;
  return p;
}

DecoderParams BuildDecoder(const TflModel& m, std::vector<uint8_t>* blob) {
  int sg = m.SignatureSubgraph("serving_default");
  if (sg < 0) sg = 0;
  Net n(m, sg, blob);
  SPEC_CHECK(n.convs.size() == 36, "decoder: expected 36 convolution ops");
  DecoderParams p;
  std::memset(&p, 0, sizeof(p));
  n.expect_conv(n.conv(0), kConv2D, DType::F32, 512, 3, 16, 1);
  p.bott = n.PackConvF32(n.conv(0));
  {
    const int lr = n.next(Net::Out(n.conv(0), 0), kLeakyRelu);
    const int q = n.next(n.out0(lr), kQuantize);
    p.bott_q = n.QP(n.out0(q));
  }
  // a bank of `G` TRANSPOSE_CONVs (convs first..first+G-1) fused into one grouped tap-GEMM
  auto pack_up = [&](int first, int G) {
    UpI8 up;
    std::memset(&up, 0, sizeof(up));
    const int stride = 2, K = 4, Cin = 128, Cout = 64, J = K / stride;
    const int NG = stride * Cout, N = G * NG;
    std::vector<int8_t> dense((size_t)J * Cin * N);
    std::vector<int32_t> bias((size_t)N), mult((size_t)N), shift((size_t)N);
    int in_zp = 0;
    for (int gi = 0; gi < G; ++gi) {
      const TflOp& o = n.conv(first + gi);
      n.expect_conv(o, kTransposeConv, DType::I8, Cout, K, Cin, stride);
      const TflTensor& w = n.T(n.w_tensor(o));
      const TflTensor& b = n.T(n.b_tensor(o));
      const TflTensor& x = n.T(n.in_tensor(o));
      const TflTensor& y = n.T(Net::Out(o, 0));
      if (gi == 0) in_zp = x.zp0();
      SPEC_CHECK(x.zp0() == in_zp, "transposed conv bank: inputs must share quantisation");
      const int8_t* src = w.as<int8_t>((size_t)Cout * K * Cin);
      const int32_t* bsrc = b.as<int32_t>((size_t)Cout);
      SPEC_CHECK(w.scale.size() == 1 || w.scale.size() == (size_t)Cout, "transposed conv bank: per-channel scale count");
      for (int r = 0; r < stride; ++r)
        for (int co = 0; co < Cout; ++co) {
          const size_t col = (size_t)gi * NG + (size_t)r * Cout + co;
          int64_t wsum = 0;
          for (int j = 0; j < J; ++j)
            for (int ci = 0; ci < Cin; ++ci) {
              const int8_t v = src[((size_t)co * K + (r + stride * (J - 1 - j))) * Cin + ci];
              wsum += v;
              dense[((size_t)j * Cin + ci) * N + col] = v;
            }
          // rows outside the input are padded with the zero point, so the fold uses all J taps
          bias[col] = (int32_t)(bsrc[co] - (int64_t)in_zp * wsum);
          const double eff = (double)x.scale0() * (double)w.scale[w.scale.size() > 1 ? (size_t)co : 0] / (double)y.scale0();
          int32_t qm; int sh;
          QuantizeMultiplier(eff, &qm, &sh);
          mult[col] = qm;
          shift[col] = sh;
        }
      const int dq = n.next(Net::Out(o, 0), kDequantize);
      up.dq[gi] = n.QP(Net::Out(o, 0));
      up.out_zp[gi] = y.zp0();
      const int add = n.next(n.out0(dq), kAdd);
      // the tail slice of the sum has the f32 bias subtracted before it becomes the next overlap state
      int sub = -1;
      for (int c : n.g.consumers(n.out0(add)))
        if (n.op(c).code == kStridedSlice)
          for (int c2 : n.g.consumers(n.out0(c)))
            if (n.op(c2).code == kSub) sub = c2;
      SPEC_CHECK(sub >= 0, "transposed conv: overlap SUB not found");
      const TflTensor& bf = n.T(Net::In(n.op(sub), 1));
      SPEC_CHECK(bf.count() == 64 && bf.type == DType::F32, "transposed conv: f32 bias constant");
      up.bias_f32[gi] = Append(blob, std::vector<float>(bf.as<float>(64), bf.as<float>(64) + 64));
    }
    up.g = GemmI8{Append(blob, PackMmaB(dense, J * Cin, N)), Append(blob, bias), Append(blob, mult), Append(blob, shift), 0, in_zp};
    return up;
  };
  p.up0 = pack_up(1, 4);
  // mixed unit quant_decoder_0/resnet_0
  n.expect_conv(n.conv(5), kDepthwiseConv2D, DType::I8, 256, 3, 256, 1, 1);
  n.expect_conv(n.conv(6), kConv2D, DType::I8, 256, 1, 256, 1);
  n.expect_conv(n.conv(7), kConv2D, DType::I8, 256, 1, 64, 1);
  p.up0_q = n.QP(n.in_tensor(n.conv(5)));
  p.m_dw = n.PackDwI8(n.conv(5));
  p.m_pw1 = n.PackConvI8(n.conv(6));
  p.m_lr1 = n.PackLRelu(n.next(Net::Out(n.conv(6), 0), kLeakyRelu));
  p.m_pw2 = n.PackConvI8(n.conv(7));
  {
    const int dq = n.next(Net::Out(n.conv(7), 0), kDequantize);
    p.m_dq = n.QP(Net::Out(n.conv(7), 0));
    const int addf = n.next(n.out0(dq), kAdd);
    const int q2 = n.next(n.out0(addf), kQuantize);
    p.m_q2 = n.QP(n.out0(q2));
    p.m_lr2 = n.PackLRelu(n.next(n.out0(q2), kLeakyRelu));
  }
  p.q[0] = n.PackResI8(8, 256, 3);
  p.q[1] = n.PackResI8(11, 256, 9);
  p.up1 = pack_up(14, 2);
  const int dil[3] = {1, 3, 9};
  // decoder_1's 1x1 convolutions also in TF32 fragment order: kernel C's tensor mode runs them on mma.sync (GemmTf32Mma)
  for (int i = 0; i < 3; ++i) p.r1[i] = n.PackResF32(16 + 3 * i, 128, dil[i], 2, true);
  n.expect_conv(n.conv(25), kTransposeConv, DType::F32, 64, 10, 128, 5);
  GemmList gemms;           // kernel D's GEMMs, in order up2, (pw1, pw2) x 3, last
  p.up2 = n.PackTconvF32(n.conv(25), 5, &gemms);
  for (int i = 0; i < 3; ++i) p.r2[i] = n.PackResF32(26 + 3 * i, 64, dil[i], 1, false, &gemms);
  n.expect_conv(n.conv(35), kTransposeConv, DType::F32, 1, 64, 64, 16);
  p.last = n.PackTconvF32(n.conv(35), 16, &gemms);
  {
    SPEC_CHECK(gemms.size() == 8 && gemms[0].size() == (size_t)256 * 320 && gemms[7].size() == (size_t)256 * 16, "tensor-core decoder: unexpected GEMM list");
    std::vector<uint8_t> chunks;
    const std::vector<float>& wu = gemms[0];                  // decoder_2/simple: [(j, ci)][(r, co)], 256 x 320
    for (int mb = 0; mb < 5; ++mb)
      for (int kc = 0; kc < 8; ++kc)
        AppendDuChunk(&chunks, 128, 16, [&](int row, int k) {
          const int m = mb * 128 + row, j = m / 320, rc = m % 320, ci = kc * 16 + k;
          return j < 2 ? wu[(size_t)(j * 128 + ci) * 320 + rc] : 0.0f;
        });
    for (int g = 1; g <= 6; ++g) {
      SPEC_CHECK(gemms[(size_t)g].size() == (size_t)64 * 64, "tensor-core decoder: residual-unit GEMM shape");
      const std::vector<float>& w = gemms[(size_t)g];          // [k = cin][n = cout]
      for (int kc = 0; kc < 2; ++kc) AppendDuChunk(&chunks, 64, 32, [&](int row, int k) { return w[(size_t)(kc * 32 + k) * 64 + row]; });
    }
    const std::vector<float>& wl = gemms[7];                  // last_layer: [(tap, ci)][n], 256 x 16
    for (int kc = 0; kc < 2; ++kc)
      AppendDuChunk(&chunks, 64, 32, [&](int row, int k) { return wl[(size_t)((row / 16) * 64 + kc * 32 + k) * 16 + row % 16]; });
    SPEC_CHECK(chunks.size() == (size_t)kDuNumChunks * kDuChunkBytes, "tensor-core decoder: chunk count");
    while (blob->size() % 128) blob->push_back(0);
    p.du_chunks = Append(blob, chunks);
  }
  p.zp_state[0] = p.m_dw.in_zp;
  p.zp_state[1] = p.q[0].dw.in_zp;
  p.zp_state[2] = p.q[1].dw.in_zp;
  return p;
}

RvqParams BuildRvq(const TflModel& m, std::vector<uint8_t>* blob, int* bits_per_stage) {
  const int se = m.SignatureSubgraph("encode"), sd = m.SignatureSubgraph("decode");
  SPEC_CHECK(se >= 0 && sd >= 0, "quantizer: missing encode/decode signatures");
  SPEC_CHECK((size_t)se < m.subgraphs().size() && (size_t)sd < m.subgraphs().size(), "quantizer: signature subgraph index");
  const TflSubgraph& ge = m.subgraphs()[(size_t)se];
  auto tensor_of = [](const TflSubgraph& g, int i) -> const TflTensor& {
    SPEC_CHECK(i >= 0 && (size_t)i < g.tensors.size(), "quantizer: tensor index out of range");
    return g.tensors[(size_t)i];
  };
  std::vector<const float*> stage_cb;
  for (const TflOp& o : ge.ops)
    if (o.code == kSquaredDifference) {
      SPEC_CHECK(o.inputs.size() >= 2, "quantizer: SQUARED_DIFFERENCE operands");
      const TflTensor& cb = tensor_of(ge, o.inputs[1]);
      SPEC_CHECK(cb.count() == 16 * 64 && cb.type == DType::F32, "quantizer: codebook shape");
      stage_cb.push_back(cb.as<float>(16 * 64));
    }
  SPEC_CHECK(stage_cb.size() == 46, "quantizer: expected 46 stages");
  *bits_per_stage = 0;
  for (int o : ge.outputs) {
    const TflTensor& t = tensor_of(ge, o);
    if (t.data && t.count() == 1 && t.type == DType::I32) *bits_per_stage = t.as<int32_t>(1)[0];
  }
  SPEC_CHECK(*bits_per_stage == 4, "quantizer: expected 4 bits per stage");
  // the decode signature must use the same codebook for the same index slot
  const TflSubgraph& gd = m.subgraphs()[(size_t)sd];
  int checked = 0;
  for (const TflOp& o : gd.ops)
    if (o.code == kGather) {
      SPEC_CHECK(o.inputs.size() >= 2, "quantizer: GATHER operands");
      const int sl = gd.producer(o.inputs[1]);
      SPEC_CHECK(sl >= 0 && gd.ops[(size_t)sl].code == kStridedSlice && gd.ops[(size_t)sl].inputs.size() >= 2, "quantizer: decode GATHER index is not a slice");
      const TflTensor& bg = tensor_of(gd, gd.ops[(size_t)sl].inputs[1]);
      SPEC_CHECK(bg.type == DType::I32 && bg.count() >= 1, "quantizer: decode slice begin");
      const int stage = bg.as<int32_t>(1)[0];
      SPEC_CHECK(stage >= 0 && stage < 46, "quantizer: decode stage index");
      const TflTensor& cb = tensor_of(gd, o.inputs[0]);
      SPEC_CHECK(cb.count() == 16 * 64 && cb.type == DType::F32 && std::memcmp(cb.as<float>(16 * 64), stage_cb[(size_t)stage], 16 * 64 * 4) == 0,
                 "quantizer: decode codebook differs from encode codebook");
      ++checked;
    }
  SPEC_CHECK(checked == 46, "quantizer: expected 46 decode GATHER ops");
  std::vector<float> cbs((size_t)46 * 16 * 64), cbt((size_t)46 * 64 * 16);
  for (int s = 0; s < 46; ++s)
    for (int c = 0; c < 16; ++c)
      for (int j = 0; j < 64; ++j) {
        cbs[((size_t)s * 16 + c) * 64 + j] = stage_cb[(size_t)s][c * 64 + j];
        cbt[((size_t)s * 64 + j) * 16 + c] = stage_cb[(size_t)s][c * 64 + j];
      }
  RvqParams p;
  p.codebooks_t = Append(blob, cbt);
  p.codebooks = Append(blob, cbs);
  p.num_stages = 46;
  return p;
}

}  // namespace

// Spectrogram + mel filterbank tables (window, FFT twiddles, triangular weights), the constants
// LogMelSpectrogramExtractorImpl::Create builds through audio_dsp
// (lyra/log_mel_spectrogram_extractor_impl.cc:53-94; limits 0 .. 0.495*fs at :39-40).
LogMelParams BuildLogMelParams(std::vector<uint8_t>* blob, int sample_rate_hz, int hop, int window, int num_mel) {
  SPEC_CHECK(window >= hop && hop > 0 && num_mel > 0, "log-mel: window must be >= hop");
  LogMelParams p;
  std::memset(&p, 0, sizeof(p));
  int fft = 1;
  while (fft < window) fft <<= 1;
  SPEC_CHECK(fft == 1024, "log-mel: the FFT kernel is specialised for 1024 points (window 513..1024)");
  const int bins = fft / 2 + 1;
  std::vector<double> win((size_t)window), tw((size_t)fft), weights((size_t)bins, 0.0);
  std::vector<int32_t> band((size_t)bins, -2);
  for (int i = 0; i < window; ++i) win[(size_t)i] = 0.5 - 0.5 * std::cos(2.0 * M_PI * i / (double)window);
  for (int k = 0; k < fft / 2; ++k) {
    const double ang = -2.0 * M_PI * (double)k / (double)fft;
    tw[(size_t)2 * k] = std::cos(ang);
    tw[(size_t)2 * k + 1] = std::sin(ang);
  }
  auto mel = [](double f) { return 1127.0 * std::log1p(f / 700.0); };
  const double lower = 0.0, upper = 0.495 * sample_rate_hz;
  const double mel_low = mel(lower), mel_hi = mel(upper);
  const double spacing = (mel_hi - mel_low) / (double)(num_mel + 1);
  std::vector<double> center((size_t)num_mel + 1);
  for (int i = 0; i <= num_mel; ++i) center[(size_t)i] = mel_low + spacing * (i + 1);
  const double hz_per_sbin = 0.5 * sample_rate_hz / (double)(bins - 1);
  p.start_index = (int)(1.5 + lower / hz_per_sbin);
  p.end_index = (int)(upper / hz_per_sbin);
  int channel = 0;
  for (int i = 0; i < bins; ++i) {
    const double melf = mel(i * hz_per_sbin);
    if (i < p.start_index || i > p.end_index) continue;
    while (channel < num_mel && center[(size_t)channel] < melf) ++channel;
    band[(size_t)i] = channel - 1;
    const int ch = channel - 1;
    if (ch >= 0) weights[(size_t)i] = (center[(size_t)ch + 1] - melf) / (center[(size_t)ch + 1] - center[(size_t)ch]);
    else weights[(size_t)i] = (center[0] - melf) / (center[0] - mel_low);
  }
  p.window = Append(blob, win);
  // per-stage copies of the same table (stage with half-length h reads tw[k * (fft/2/h)], k < h, stored contiguously
  // at entry h - 1) so that neighbouring butterflies read neighbouring twiddles
  std::vector<double> tws;
  for (int h = 1; h < fft; h <<= 1)
    for (int k = 0; k < h; ++k) {
      tws.push_back(tw[(size_t)2 * (k * (fft / 2 / h))]);
      tws.push_back(tw[(size_t)2 * (k * (fft / 2 / h)) + 1]);
    }
  p.twiddle = Append(blob, tws);
  p.weights = Append(blob, weights);
  p.band = Append(blob, band);
  // channel ch sums the bins of bands ch-1 and ch; the band index never decreases with the bin, so they are one range
  std::vector<int32_t> range((size_t)num_mel * 2);
  for (int ch = 0; ch < num_mel; ++ch) {
    int lo = bins, hi = -1;
    for (int i = p.start_index; i <= p.end_index; ++i)
      if (band[(size_t)i] == ch || band[(size_t)i] == ch - 1) { lo = std::min(lo, i); hi = std::max(hi, i); }
    range[(size_t)2 * ch] = lo;
    range[(size_t)2 * ch + 1] = hi;
  }
  p.range = Append(blob, range);
  p.num_mel = num_mel; p.fft = fft; p.window_len = window; p.hop = hop;
  return p;
}

// Tables of the comfort-noise generator; `lm` = the 160-bin log-mel tables already in the blob.  Same expressions, in the same
// order, as oracle/comfort_noise.c lo_cng_create (the sums are order-sensitive in their last bits).
CngParams BuildCngParams(std::vector<uint8_t>* blob, const LogMelParams& lm, int window) {
  CngParams p;
  std::memset(&p, 0, sizeof(p));
  const int bins = lm.fft / 2 + 1;
  const double* weights = reinterpret_cast<const double*>(blob->data() + lm.weights);
  const int32_t* band = reinterpret_cast<const int32_t*>(blob->data() + lm.band);
  std::vector<double> norm((size_t)lm.num_mel, 0.0), synth((size_t)lm.fft);
  for (int i = lm.start_index; i <= lm.end_index && i < bins; ++i) {
    const int ch = band[i];
    if (ch >= 0) norm[(size_t)ch] += weights[i];
    if (ch + 1 < lm.num_mel) norm[(size_t)ch + 1] += 1.0 - weights[i];
  }
  double swa = 0.0, sws = 0.0;
  for (int i = 0; i < window; ++i) { const double w = 0.5 - 0.5 * std::cos(2.0 * M_PI * i / (double)window); swa += w * w; }
  for (int i = 0; i < lm.fft; ++i) { synth[(size_t)i] = 0.5 - 0.5 * std::cos(2.0 * M_PI * i / (double)lm.fft); sws += synth[(size_t)i] * synth[(size_t)i]; }
  const double gain = std::sqrt((double)lm.fft * (double)lm.hop / (swa * sws));
  for (int i = 0; i < lm.fft; ++i) synth[(size_t)i] *= gain;
  std::vector<float> fade(641);
  for (int fp = 0; fp <= 640; ++fp) fade[(size_t)fp] = (float)((1.0 + std::cos((double)fp * M_PI / (double)640)) / 2.0);
  p.weights = lm.weights; p.band = lm.band; p.twiddle = lm.twiddle;
  p.norm = Append(blob, norm);
  p.synth = Append(blob, synth);
  p.fade = Append(blob, fade);
  p.start_index = lm.start_index; p.end_index = lm.end_index; p.num_mel = lm.num_mel; p.fft = lm.fft; p.hop = lm.hop;
  return p;
}

// Filter banks of the sample-rate converters; the expressions (and their order) are those of oracle/resampler.c
// lo_resampler_design, so both sides hold the same float coefficients.
namespace {
double BesselI0(double x) {
  double sum = 1.0, term = 1.0;
  const double q = x * x / 4.0;
  for (int k = 1; k < 64; ++k) {
    term *= q / ((double)k * (double)k);
    sum += term;
    if (term < 1e-17 * sum) break;
  }
  return sum;
}
}  // namespace

ResamplerParams BuildResamplerParams(std::vector<uint8_t>* blob) {
  ResamplerParams p;
  std::memset(&p, 0, sizeof(p));
  const int in_rate[6] = {8000, 32000, 48000, 16000, 16000, 16000}, out_rate[6] = {16000, 16000, 16000, 8000, 32000, 48000};
  for (int pair = 0; pair < 6; ++pair) {
    int a = in_rate[pair], b = out_rate[pair];
    while (b) { const int t = a % b; a = b; b = t; }
    const int num = in_rate[pair] / a, den = out_rate[pair] / a;
    const double factor = (double)num / (double)den;
    const double radius_factor = 17.0 * (out_rate[pair] < in_rate[pair] ? (double)((float)out_rate[pair] / (float)in_rate[pair]) : 1.0);
    const double radius = radius_factor * (factor > 1.0 ? factor : 1.0);
    const double cutoff = 0.9 * 0.5 / (factor > 1.0 ? factor : 1.0);
    const double beta = 5.658;
    const int rc = (int)std::ceil(radius - 1e-4);
    SPEC_CHECK(2 * rc + 1 == kResamplerTaps && den <= 3, "resampler: unexpected filter size");
    const double i0b = BesselI0(beta);
    std::vector<float> coeffs((size_t)den * kResamplerTaps);
    for (int ph = 0; ph < den; ++ph) {
      const double offset = (double)ph / (double)den;
      for (int j = 0; j < kResamplerTaps; ++j) {
        const double x = (double)(rc - j) + offset;
        double h = 0.0;
        if (std::fabs(x) <= radius) {
          const double z = 2.0 * cutoff * x;
          const double sinc = std::fabs(z) < 1e-12 ? 1.0 : std::sin(M_PI * z) / (M_PI * z);
          const double r = x / radius;
          h = 2.0 * cutoff * sinc * BesselI0(beta * std::sqrt(1.0 - r * r > 0.0 ? 1.0 - r * r : 0.0)) / i0b;
        }
        coeffs[(size_t)ph * kResamplerTaps + j] = (float)h;
      }
    }
    p.coeffs[pair] = Append(blob, coeffs);
    p.num[pair] = num;
    p.den[pair] = den;
  }
  return p;
}

ModelSpec BuildModelSpec(const std::string& model_dir) {
  ModelSpec s;
  {
    // lyra_config.binarypb: field 1 (identifier) varint == 3  (lyra/lyra_config.h:145-166)
    std::ifstream f(model_dir + "/lyra_config.binarypb", std::ios::binary);
    SPEC_CHECK((bool)f, "cannot open lyra_config.binarypb in " + model_dir);
    char b[2] = {0, 0};
    f.read(b, 2);
    SPEC_CHECK(f.gcount() == 2 && b[0] == 0x08 && b[1] == 0x03, "lyra_config.binarypb identifier is not 3 (weights/code version mismatch)");
  }
  const TflModel enc = TflModel::Load(model_dir + "/soundstream_encoder.tflite");
  const TflModel dec = TflModel::Load(model_dir + "/lyragan.tflite");
  const TflModel rvq = TflModel::Load(model_dir + "/quantizer.tflite");
  s.enc = BuildEncoder(enc, &s.blob);
  s.dec = BuildDecoder(dec, &s.blob);
  s.rvq = BuildRvq(rvq, &s.blob, &s.bits_per_stage);
  s.logmel160 = BuildLogMelParams(&s.blob, 16000, 320, 640, 160);
  s.logmel64 = BuildLogMelParams(&s.blob, 16000, 320, 640, 64);
  s.cng = BuildCngParams(&s.blob, s.logmel160, 640);
  s.resampler = BuildResamplerParams(&s.blob);
  const int ext_rates[3] = {8000, 32000, 48000};
  for (int r = 0; r < 3; ++r) s.logmel160_ext[r] = BuildLogMelParams(&s.blob, ext_rates[r], 320, 640, 160);
  while (s.blob.size() % 256) s.blob.push_back(0);
  return s;
}

}  // namespace lyra_b200
