// Warpgroup MMA (wgmma) probe, built two ways from this one source:
//   * nvcc -gencode arch=compute_90a,code=sm_90a   -> runs on an H100 (the instruction sequences of device_compat.h)
//   * g++ -DLYRA_EMU -x c++ (+ tests/cuda_emu)       -> runs on the CPU tier against the emulator's wgmma model
// Case 1: D[64 x 32] = A[64 x 64] * B[32 x 64]^T, both operands from shared memory through matrix descriptors, single TF32 pass
//         (the shape and operand layout of decoder_2/simple in DecoderKernelDW).
// Case 2: OUT = LeakyReLU(A * W1^T + b1) * W2^T + b2 + U for A, U [64 x 64]: both 1x1 convolutions of a decoder_2 residual unit,
//         split precision (three MMAs per product), A in registers, the first epilogue turned into the second GEMM's A
//         fragments by DwAccToA (the data path of DecoderKernelDW's residual units).
// Exit code 0 iff both cases match their double-precision references.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "net_kernels_wgmma.cuh"

using namespace lyra_b200;

namespace {

constexpr int M = 64, K = 64, N1 = 32, N = 64;

// canonical K-major no-swizzle operand: [k/4][row/8][row%8][k%4]
__device__ inline int Canon(int row, int k, int rows) { return ((k / 4) * (rows / 8) + row / 8) * 32 + (row % 8) * 4 + k % 4; }

__global__ void __launch_bounds__(128)
WgmmaProbeKernel(int mode, const float* A, const float* W1, const float* B1, const float* W2, const float* B2, const float* U, float* OUT) {
  float* a_sm = reinterpret_cast<float*>(LYRA_DYN_SMEM());    // case 1: A [64 x 64]
  float* w_hi = a_sm + M * K;                                 // W1 (case 1: [32 x 64], single pass) or W1, W2 split (case 2)
  float* w_lo = w_hi + N * K;
  float* w2_hi = w_lo + N * K;
  float* w2_lo = w2_hi + N * K;
  const int tid = (int)threadIdx.x, lane = tid % 32, q = tid / 32, g = lane / 4, t = lane % 4;
  const int rows = mode == 0 ? N1 : N;
  for (int i = tid; i < M * K; i += 128) a_sm[Canon(i / K, i % K, M)] = A[i];
  for (int i = tid; i < rows * K; i += 128) {
    uint32_t h, l;
    DwSplit(W1[i], h, l);
    w_hi[Canon(i / K, i % K, rows)] = mode == 0 ? W1[i] : __uint_as_float(h);
    w_lo[Canon(i / K, i % K, rows)] = __uint_as_float(l);
    DwSplit(W2[i], h, l);
    w2_hi[Canon(i / K, i % K, N)] = __uint_as_float(h);
    w2_lo[Canon(i / K, i % K, N)] = __uint_as_float(l);
  }
  lyra_fence_proxy_async();                                   // operands written with ordinary stores -> visible to the tensor cores
  __syncthreads();
  if (mode == 0) {
    float d[16];
    const uint32_t lboA = (M / 8) * 128u, lboB = (N1 / 8) * 128u;
    lyra_wgmma_fence();
    for (int ks = 0; ks < K / 8; ++ks)
      lyra_wgmma_m64n32_tf32_ss(d, lyra_wgmma_desc(reinterpret_cast<char*>(a_sm) + (size_t)ks * 2 * lboA, lboA, 128),
                                lyra_wgmma_desc(reinterpret_cast<char*>(w_hi) + (size_t)ks * 2 * lboB, lboB, 128), ks > 0);
    lyra_wgmma_commit();
    lyra_wgmma_wait<0>();
    for (int i = 0; i < 16; ++i) OUT[(16 * q + g + 8 * ((i >> 1) & 1)) * N1 + 8 * (i >> 2) + 2 * t + (i & 1)] = d[i];
    return;
  }
  uint32_t ah[8][4], al[8][4];
  for (int ks = 0; ks < 8; ++ks)
    for (int f = 0; f < 4; ++f)
      DwSplit(A[(16 * q + g + 8 * (f & 1)) * K + 8 * ks + t + 4 * (f >> 1)], ah[ks][f], al[ks][f]);
  float acc[32];
  const uint32_t lboW = (N / 8) * 128u;
  for (int gemm = 0; gemm < 2; ++gemm) {
    const char* wh = reinterpret_cast<const char*>(gemm == 0 ? w_hi : w2_hi);
    const char* wl = reinterpret_cast<const char*>(gemm == 0 ? w_lo : w2_lo);
    lyra_wgmma_fence();
    for (int ks = 0; ks < 8; ++ks) {
      const uint64_t bh = lyra_wgmma_desc(wh + (size_t)ks * 2 * lboW, lboW, 128), bl = lyra_wgmma_desc(wl + (size_t)ks * 2 * lboW, lboW, 128);
      lyra_wgmma_m64n64_tf32_rs(acc, al[ks], bh, ks > 0);     // small terms first
      lyra_wgmma_m64n64_tf32_rs(acc, ah[ks], bl, true);
      lyra_wgmma_m64n64_tf32_rs(acc, ah[ks], bh, true);
    }
    lyra_wgmma_commit();
    lyra_wgmma_wait<0>();
    for (int i = 0; i < 32; ++i) {
      const int row = 16 * q + g + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * t + (i & 1);
      if (gemm == 0) acc[i] = LeakyRelu(__fadd_rn(acc[i], B1[col]));
      else OUT[row * N + col] = __fadd_rn(__fadd_rn(acc[i], B2[col]), U[row * N + col]);
    }
    if (gemm == 0) DwAccToA(acc, ah, al);
  }
}

float Tf32(float x) { uint32_t b; std::memcpy(&b, &x, 4); b &= 0xffffe000u; std::memcpy(&x, &b, 4); return x; }

template <typename T>
T* ToDevice(const std::vector<T>& v) {
  void* p = nullptr;
  if (cudaMalloc(&p, v.size() * sizeof(T)) != cudaSuccess) return nullptr;
  cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice);
  return static_cast<T*>(p);
}

}  // namespace

int main() {
  std::vector<float> A(M * K), U(M * N), W1(N * K), W2(N * K), B1(N), B2(N), OUT(M * N);
  srand(7);
  auto rnd = [] { return (float)(rand() % 20001 - 10000) / 10000.0f * 1.37f; };
  for (auto& v : A) v = rnd();
  for (auto& v : U) v = rnd();
  for (auto& v : W1) v = rnd() * 0.25f;
  for (auto& v : W2) v = rnd() * 0.25f;
  for (auto& v : B1) v = rnd() * 0.1f;
  for (auto& v : B2) v = rnd() * 0.1f;
  float *dA = ToDevice(A), *dU = ToDevice(U), *dW1 = ToDevice(W1), *dW2 = ToDevice(W2), *dB1 = ToDevice(B1), *dB2 = ToDevice(B2), *dO = ToDevice(OUT);
  if (!dA || !dU || !dW1 || !dW2 || !dB1 || !dB2 || !dO) { std::printf("allocation failed\n"); return 2; }
  const size_t smem = (size_t)(M * K + 4 * N * K) * 4;
  LYRA_SET_MAX_SMEM(WgmmaProbeKernel, smem);
  int bad = 0;
  for (int mode = 0; mode < 2; ++mode) {
    const int cols = mode == 0 ? N1 : N;
    LYRA_LAUNCH(WgmmaProbeKernel, dim3(1), dim3(128), smem, 0, mode, dA, dW1, dB1, dW2, dB2, dU, dO);
    if (cudaDeviceSynchronize() != cudaSuccess) { std::printf("case %d: kernel failed\n", mode + 1); return 1; }
    cudaMemcpy(OUT.data(), dO, OUT.size() * 4, cudaMemcpyDeviceToHost);
    double worst = 0, scale = 0;
    for (int m = 0; m < M; ++m) {
      double h[N];
      for (int n = 0; n < cols; ++n) {
        double s = 0;
        for (int k = 0; k < K; ++k)
          s += mode == 0 ? (double)Tf32(A[m * K + k]) * (double)Tf32(W1[n * K + k]) : (double)A[m * K + k] * (double)W1[n * K + k];
        if (mode == 0) { h[n] = s; continue; }
        s += B1[n];
        h[n] = (double)(float)(s > 0 ? s : s * (double)0.3f);
      }
      for (int n = 0; n < cols; ++n) {
        double ref = h[n];
        if (mode != 0) {
          ref = 0;
          for (int k = 0; k < K; ++k) ref += h[k] * (double)W2[n * K + k];
          ref += (double)B2[n] + (double)U[m * N + n];
        }
        worst = std::fmax(worst, std::fabs((double)OUT[m * cols + n] - ref));
        scale = std::fmax(scale, std::fabs(ref));
      }
    }
    const bool ok = worst / scale < 5e-6;
    std::printf("case %d: max |OUT - ref| = %.3e (scale %.2f, relative %.2e) -> %s\n", mode + 1, worst, scale, worst / scale, ok ? "MATCH" : "MISMATCH");
    bad |= !ok;
  }
  return bad;
}
