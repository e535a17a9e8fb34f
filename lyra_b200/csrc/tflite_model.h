// Product-side weight/graph loader: a dependency-free reader for the three TFLite flatbuffers that
// the reference hands to tflite::FlatBufferModel::BuildFromFile (lyra/tflite_model_wrapper.cc:39-44).
// Replaces TfLiteModelWrapper::Create's model loading for the CUDA path; the graphs themselves are
// never interpreted on the product side — model_spec.cc pattern-matches them into fused layers.
#pragma once

#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

namespace lyra_b200 {

enum class DType : int { F32 = 0, I32 = 2, U8 = 3, I64 = 4, BOOL = 6, I8 = 9, RESOURCE = 13 };

enum BuiltinOp : int {
  kAdd = 0, kConcatenation = 2, kConv2D = 3, kDepthwiseConv2D = 4, kDequantize = 6, kMul = 18,
  kReshape = 22, kGather = 36, kSub = 41, kStridedSlice = 45, kSplit = 49, kCast = 53, kMaximum = 55,
  kArgMax = 56, kLess = 58, kTransposeConv = 67, kNotEqual = 72, kSum = 74, kArgMin = 79, kPack = 83,
  kOneHot = 85, kLeakyRelu = 98, kSquaredDifference = 99, kQuantize = 114, kCallOnce = 129,
  kVarHandle = 142, kReadVariable = 143, kAssignVariable = 144
};

struct TflTensor {
  std::vector<int> shape;
  DType type = DType::F32;
  std::string name;
  std::vector<float> scale;
  std::vector<int64_t> zero_point;
  const uint8_t* data = nullptr;   // constant payload (points into the file image) or nullptr
  size_t nbytes = 0;
  size_t count() const { size_t c = 1; for (int d : shape) c *= (size_t)d; return c; }
  float scale0() const { if (scale.empty()) throw std::runtime_error("tensor " + name + " has no scale"); return scale[0]; }
  int zp0() const { if (zero_point.empty()) throw std::runtime_error("tensor " + name + " has no zero point"); return (int)zero_point[0]; }
  // constant payload as `n` elements of T; throws unless the file really holds that many bytes for this tensor
  template <typename T> const T* as(size_t n) const {
    if (data == nullptr || nbytes / sizeof(T) < n) throw std::runtime_error("tensor " + name + ": constant data missing or too short");
    return reinterpret_cast<const T*>(data);
  }
  // the whole declared shape (count() elements)
  template <typename T> const T* as() const { return as<T>(count()); }
};

struct TflOp {
  int code = -1;
  std::vector<int> inputs, outputs;
  uint32_t options = 0;            // absolute offset of the builtin_options table (0 = none)
};

struct TflSubgraph {
  std::string name;
  std::vector<TflTensor> tensors;
  std::vector<TflOp> ops;
  std::vector<int> inputs, outputs;
  // graph navigation helpers
  int producer(int tensor) const;                       // op index or -1
  std::vector<int> consumers(int tensor) const;         // op indices
  int sole_consumer(int tensor, int code) const;        // op index of the only consumer with `code`, else throws
};

class TflModel {
 public:
  static TflModel Load(const std::string& path);        // throws std::runtime_error
  const std::vector<TflSubgraph>& subgraphs() const { return subgraphs_; }
  int SignatureSubgraph(const std::string& key) const;  // -1 if absent
  // builtin_options accessors (flatbuffer field ids of the op's options table)
  int32_t OptI32(const TflOp& op, int field, int32_t dflt) const;
  int OptI8(const TflOp& op, int field, int dflt) const;
  float OptF32(const TflOp& op, int field, float dflt) const;
  std::string OptString(const TflOp& op, int field) const;

 private:
  std::vector<uint8_t> image_;
  std::vector<TflSubgraph> subgraphs_;
  std::vector<std::pair<std::string, int>> signatures_;
};

}  // namespace lyra_b200
