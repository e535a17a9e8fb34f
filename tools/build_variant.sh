#!/bin/bash
# usage: build_variant.sh name [-DFLAG ...]   -> devtools_build/liblyra_b200_<name>.so
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p devtools_build
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared "$@" -Ilyra_b200/csrc \
  lyra_b200/csrc/engine.cu lyra_b200/csrc/model_spec.cc lyra_b200/csrc/tflite_model.cc -o devtools_build/liblyra_b200_$name.so
