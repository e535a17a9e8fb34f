// TEST INFRASTRUCTURE ONLY — a functional simulator for CUDA thread blocks on the CPU.
//
// There is no GPU in the build container, so the kernels in lyra_b200/csrc/*.cu are also compiled
// with g++ (-DLYRA_EMU) against this header and executed one thread block at a time: every CUDA
// thread is a ucontext fiber, __syncthreads()/__syncwarp()/__shfl_*_sync() are fiber barriers.
// This validates indexing, state handling and arithmetic of the *same kernel source* against the
// oracle in the CPU test tier (-m "not gpu").  It is NOT a product path: the shipped library
// (lyra_b200/liblyra_b200.so) is built by nvcc only, never links this file, and lyra_b200/ cannot
// load the emulated build (tests/cuda_emu/_build/liblyra_b200_emu.so).
#pragma once

#include <ucontext.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__ __restrict
#define __launch_bounds__(...)
#define __shared__ static thread_local
#define __constant__ static

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint3_emu { unsigned x, y, z; };

struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) float2 { float x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
struct alignas(8) int2 { int x, y; };
struct alignas(16) double2 { double x, y; };
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
static inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }

namespace cuda_emu {

struct BlockState {
  unsigned nthreads = 0;
  std::vector<ucontext_t> ctx;
  std::vector<char*> stacks;
  ucontext_t sched;
  std::vector<int> state;          // 0 = runnable, 1 = waiting at block barrier, 2 = done, 3 = waiting at warp barrier
  unsigned cur = 0;
  unsigned arrived = 0;
  unsigned done = 0;
  std::vector<unsigned> warp_arrived;
  std::vector<unsigned> warp_live;
  uint64_t warp_xchg[64][32];
  uint32_t warp_scratch[64][32][8];
  char* smem = nullptr;
  alignas(16) char static_smem[512];   // storage for the product's function-local __shared__ objects (zeroed per block)
  std::function<void()> body;
};

extern thread_local BlockState* g_blk;
extern thread_local uint3_emu g_threadIdx, g_blockIdx;
extern thread_local dim3 g_blockDim, g_gridDim;

void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body);
void block_barrier();
void warp_barrier();
void yield();   // cooperative spin-wait: let the other fibers of the block run (used by the mbarrier emulation)
uint64_t warp_exchange(uint64_t v, int src_lane);
// every lane deposits n (<= 8) words; after the call `all` points at the warp's [32][8] table (valid until the next barrier)
const uint32_t (*warp_gather(const uint32_t* vals, int n))[8];

}  // namespace cuda_emu

#define threadIdx (cuda_emu::g_threadIdx)
#define blockIdx (cuda_emu::g_blockIdx)
#define blockDim (cuda_emu::g_blockDim)
#define gridDim (cuda_emu::g_gridDim)

static inline void __syncthreads() { cuda_emu::block_barrier(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { cuda_emu::warp_barrier(); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}

template <typename T>
static inline T __shfl_sync(unsigned, T v, int src, int width = 32) {
  static_assert(sizeof(T) <= 8, "shuffle payload");
  uint64_t raw = 0;
  std::memcpy(&raw, &v, sizeof(T));
  const int lane = (int)(threadIdx.x & 31);
  const int base = lane & ~(width - 1);
  raw = cuda_emu::warp_exchange(raw, base + (src & (width - 1)));
  T out;
  std::memcpy(&out, &raw, sizeof(T));
  return out;
}
template <typename T>
static inline T __shfl_xor_sync(unsigned m, T v, int lane_mask, int width = 32) {
  const int lane = (int)(threadIdx.x & 31);
  return __shfl_sync(m, v, (lane ^ lane_mask) & (width - 1), width);
}
template <typename T>
static inline T __shfl_down_sync(unsigned m, T v, unsigned delta, int width = 32) {
  const int lane = (int)(threadIdx.x & 31);
  const int l = lane & (width - 1);
  return __shfl_sync(m, v, (l + (int)delta < width) ? l + (int)delta : l, width);
}
static inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned r = 0;
  for (int l = 0; l < 32; ++l) r |= (unsigned)(__shfl_sync(0xffffffffu, pred ? 1 : 0, l) != 0) << l;
  return r;
}

static inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
static inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
static inline double __dsqrt_rn(double a) { return std::sqrt(a); }
static inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
static inline int __dp4a(int a, int b, int c) {
  for (int i = 0; i < 4; ++i) c += (int)(int8_t)(a >> (8 * i)) * (int)(int8_t)(b >> (8 * i));
  return c;
}
static inline int __float2int_rz(float v) { return (int)v; }
static inline unsigned __brev(unsigned v) {
  unsigned r = 0;
  for (int b = 0; b < 32; ++b) r |= ((v >> b) & 1u) << (31 - b);
  return r;
}
static inline uint32_t __float_as_uint(float v) { uint32_t b; std::memcpy(&b, &v, 4); return b; }
static inline float __uint_as_float(uint32_t b) { float v; std::memcpy(&v, &b, 4); return v; }
template <typename T>
static inline T __ldg(const T* p) { return *p; }
static inline long long __mul64hi(long long a, long long b) { return (long long)(((__int128)a * b) >> 64); }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

// ---- the subset of the CUDA runtime used by engine.cu, mapped onto host memory ----
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaGetLastError() { return 0; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return 0; }
static inline cudaError_t cudaMalloc(void** p, size_t n) { *p = std::calloc(1, n ? n : 1); return *p ? 0 : 2; }
static inline cudaError_t cudaFree(void* p) { std::free(p); return 0; }
static inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = std::calloc(1, n ? n : 1); return *p ? 0 : 2; }
static inline cudaError_t cudaFreeHost(void* p) { std::free(p); return 0; }
static inline cudaError_t cudaMemset(void* p, int v, size_t n) { std::memset(p, v, n); return 0; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { std::memset(p, v, n); return 0; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { std::memcpy(d, s, n); return 0; }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = nullptr; return 0; }
#define cudaStreamDefault 0u
static inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned, int) { *s = nullptr; return 0; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return 0; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
static inline cudaError_t cudaDeviceSynchronize() { return 0; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = nullptr; return 0; }
enum { cudaEventDisableTiming = 2, cudaEventBlockingSync = 1 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = nullptr; return 0; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return 0; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return 0; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return 0; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return 0; }
