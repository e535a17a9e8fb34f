// Host-side "graph -> fused layer" compiler: reads the three reference flatbuffers and produces the
// device weight blob + POD descriptors the kernels consume.  This replaces what
// TfLiteModelWrapper::Create + Interpreter::AllocateTensors do for the reference
// (lyra/tflite_model_wrapper.cc:36-95).  Throws std::runtime_error if a graph does not have the
// structure of the v1.3.2 models (SURVEY.md App. A).
#pragma once

#include <string>
#include <vector>

#include "net_params.h"

namespace lyra_b200 {

struct ModelSpec {
  std::vector<uint8_t> blob;      // every weight / table, 16-byte aligned entries
  EncoderParams enc;
  DecoderParams dec;
  RvqParams rvq;
  LogMelParams logmel160;         // 16 kHz, hop 320, window 640, 160 mel bins (NoiseEstimator's extractor)
  LogMelParams logmel64;          // 64 mel bins (lyra_integration_test's extractor)
  // the encoder-side (DTX) estimator's extractor at an external rate of 8 / 32 / 48 kHz: it is created for the external rate and
  // fed the 16 kHz hop (lyra/lyra_encoder.cc:80-89), so only its mel bank differs from logmel160
  LogMelParams logmel160_ext[3];
  ResamplerParams resampler;      // 8 / 32 / 48 kHz <-> 16 kHz filter banks
  CngParams cng;                  // comfort-noise generator + cross-fade tables (decoder PLC path)
  int num_features = 64;
  int bits_per_stage = 4;
};

// model_dir must contain soundstream_encoder.tflite, lyragan.tflite, quantizer.tflite and
// lyra_config.binarypb with identifier 3 (lyra/lyra_config.h:145-166, lyra/lyra_config.cc:55-58).
ModelSpec BuildModelSpec(const std::string& model_dir);

// Q31 fixed-point helpers (gemmlowp semantics used by TFLite's int8 kernels)
void QuantizeMultiplier(double real_multiplier, int32_t* quantized_multiplier, int* shift);
int32_t MultiplyByQuantizedMultiplier(int32_t x, int32_t quantized_multiplier, int shift);

// Log-mel tables for arbitrary (sample_rate, hop, window, num_mel); appended to `blob`.
LogMelParams BuildLogMelParams(std::vector<uint8_t>* blob, int sample_rate_hz, int hop, int window, int num_mel);

}  // namespace lyra_b200
