// Build-mode shim.  The product is compiled by nvcc for sm_90a.  The same kernel sources are also
// compiled by g++ with -DLYRA_EMU against tests/cuda_emu (a test-only CPU block simulator) so the
// CPU test tier can check kernel logic against the oracle without a GPU.  Nothing in the shipped
// library depends on the emulator.
#pragma once

#ifdef LYRA_EMU
#include "cuda_emu.h"
#define LYRA_DYN_SMEM() (reinterpret_cast<unsigned char*>(cuda_emu::g_blk->smem))
#define LYRA_LAUNCH(kernel, grid, block, smem, stream, ...) \
  cuda_emu::launch((grid), (block), (smem), [&]() { kernel(__VA_ARGS__); })
#define LYRA_SET_MAX_SMEM(kernel, bytes) (0)
#define LYRA_DEVICE_CODE 1
#define LYRA_TRAP() std::abort()
#else
#include <cuda_runtime.h>
#define LYRA_DYN_SMEM() (lyra_dyn_smem_raw)
#define LYRA_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define LYRA_SET_MAX_SMEM(kernel, bytes) \
  cudaFuncSetAttribute((kernel), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))
#define LYRA_TRAP() __trap()
#ifdef __CUDACC__
extern __shared__ __align__(1024) unsigned char lyra_dyn_smem_raw[];
#endif
#endif

#include <stdint.h>

// ---- 16-byte asynchronous global->shared copies (LDGSTS); synchronous memcpy in the emulator ----
#if defined(LYRA_EMU)
static inline void lyra_cp_async16(void* smem_dst, const void* gmem_src) { std::memcpy(smem_dst, gmem_src, 16); }
static inline void lyra_cp_async_commit() {}
template <int N>
static inline void lyra_cp_async_wait() {}
#elif defined(__CUDACC__)
__device__ __forceinline__ void lyra_cp_async16(void* smem_dst, const void* gmem_src) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void lyra_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void lyra_cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
#endif

// ---- mbarrier + bulk asynchronous copy (TMA, cp.async.bulk): the weight pipeline of the fp32 GEMMs.
//      One elected thread arms a "full" barrier with the byte count and issues one bulk copy per weight chunk; consumer
//      warps wait on its phase parity, and release the stage through an "empty" barrier (one arrival per warp).
//      lyra_mbar_wait(bar, parity) returns once the phase with that parity has completed.
struct alignas(8) LyraMbar { unsigned long long v; };
#if defined(LYRA_EMU)
struct LyraMbarEmu { uint16_t expected, arrived, phase, pad; };
static inline LyraMbarEmu* lyra_mbar_emu(LyraMbar* b) { return reinterpret_cast<LyraMbarEmu*>(b); }
static inline void lyra_mbar_init(LyraMbar* b, unsigned count) { LyraMbarEmu* e = lyra_mbar_emu(b); e->expected = (uint16_t)count; e->arrived = 0; e->phase = 0; e->pad = 0; }
static inline void lyra_mbar_fence_init() {}
static inline void lyra_fence_proxy_async() {}
static inline void lyra_mbar_arrive(LyraMbar* b) {
  LyraMbarEmu* e = lyra_mbar_emu(b);
  if (++e->arrived == e->expected) { e->arrived = 0; e->phase ^= 1; }
}
// one thread arriving for `n` participants at once (mbarrier.arrive with a count operand); the count must not overshoot the phase
static inline void lyra_mbar_arrive_n(LyraMbar* b, unsigned n) {
  LyraMbarEmu* e = lyra_mbar_emu(b);
  e->arrived = (uint16_t)(e->arrived + n);
  if (e->arrived > e->expected) { std::fprintf(stderr, "cuda_emu: mbarrier arrival count overshoots the phase\n"); std::abort(); }
  if (e->arrived == e->expected) { e->arrived = 0; e->phase ^= 1; }
}
// the emulated bulk copy is synchronous and fibers are cooperative, so arming + copying is one atomic step:
// the arrival is counted after the data has been written
static inline void lyra_bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, LyraMbar* b) {
  std::memcpy(smem_dst, gmem_src, bytes);
  lyra_mbar_arrive(b);
}
static inline void lyra_mbar_wait(LyraMbar* b, unsigned parity) {
  while (lyra_mbar_emu(b)->phase == parity) cuda_emu::yield();
}
// one function-local shared object per kernel (the emulator backs them all with the same per-block scratch area)
#define LYRA_STATIC_SMEM(type, name, count) \
  static_assert(sizeof(type) * (count) <= 448, "emulated static shared memory: 448 bytes for objects + 64 for named barriers"); \
  type* name = reinterpret_cast<type*>(cuda_emu::g_blk->static_smem)
#elif defined(__CUDACC__)
__device__ __forceinline__ unsigned lyra_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void lyra_mbar_init(LyraMbar* b, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(lyra_smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void lyra_mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
// orders this thread's earlier generic-proxy accesses to shared memory before later asynchronous-proxy (bulk copy) ones
__device__ __forceinline__ void lyra_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void lyra_mbar_arrive(LyraMbar* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(lyra_smem_u32(b)) : "memory");
}
__device__ __forceinline__ void lyra_mbar_arrive_n(LyraMbar* b, unsigned n) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;\n" ::"r"(lyra_smem_u32(b)), "r"(n) : "memory");
}
// arm the barrier with the byte count and issue the bulk copy that completes it
__device__ __forceinline__ void lyra_bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, LyraMbar* b) {
  const unsigned bar = lyra_smem_u32(b);
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
               ::"r"(lyra_smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void lyra_mbar_wait(LyraMbar* b, unsigned parity) {
  const unsigned bar = lyra_smem_u32(b);
  asm volatile("{\n"
               ".reg .pred p;\n"
               "LYRA_WAIT:\n"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
               "@p bra LYRA_DONE;\n"
               "bra LYRA_WAIT;\n"
               "LYRA_DONE:\n"
               "}\n" ::"r"(bar), "r"(parity) : "memory");
}
#define LYRA_STATIC_SMEM(type, name, count) __shared__ type name##_storage[count]; type* name = name##_storage
#endif

// ---- warp-level int8 tensor-core MMA: D(16x8,s32) += A(16x32,s8,row) * B(32x8,s8,col), fragments as in the PTX ISA
//      (mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32).  Integer accumulation is exact, so results are
//      bit-identical to the dp4a / scalar formulation whatever the internal order.
#if defined(LYRA_EMU)
static inline void lyra_mma_s8_16x8x32(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  const uint32_t mine[6] = {a[0], a[1], a[2], a[3], b[0], b[1]};
  const uint32_t (*all)[8] = cuda_emu::warp_gather(mine, 6);
  const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
  auto A = [&](int row, int k) {      // row 0..15, k 0..31
    const int src = (row & 7) * 4 + (k & 15) / 4;
    const int reg = (row >> 3) + 2 * (k >> 4);
    return (int)(int8_t)((all[src][reg] >> (8 * (k & 3))) & 0xff);
  };
  auto B = [&](int k, int col) {
    const int src = col * 4 + (k & 15) / 4;
    return (int)(int8_t)((all[src][4 + (k >> 4)] >> (8 * (k & 3))) & 0xff);
  };
  int d[4] = {c[0], c[1], c[2], c[3]};
  for (int k = 0; k < 32; ++k) {
    d[0] += A(g, k) * B(k, 2 * t);
    d[1] += A(g, k) * B(k, 2 * t + 1);
    d[2] += A(g + 8, k) * B(k, 2 * t);
    d[3] += A(g + 8, k) * B(k, 2 * t + 1);
  }
  cuda_emu::warp_barrier();             // keep the table alive until every lane has read it
  c[0] = d[0]; c[1] = d[1]; c[2] = d[2]; c[3] = d[3];
}
#elif defined(__CUDACC__)
__device__ __forceinline__ void lyra_mma_s8_16x8x32(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
#endif

// ---- warp-level TF32 tensor-core MMA: D(16x8,f32) += A(16x8,tf32,row) * B(8x8,tf32,col)
//      (mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32).  Used only by the decoder's opt-in tensor-core mode
//      (split-precision "3xTF32": fp32-equivalent accuracy, not bit-identical to the fmaf chain).
//      Fragments (g = lane / 4, t = lane % 4): a0 (g, t) a1 (g+8, t) a2 (g, t+4) a3 (g+8, t+4); b0 (k=t, n=g) b1 (k=t+4, n=g);
//      c0 (g, 2t) c1 (g, 2t+1) c2 (g+8, 2t) c3 (g+8, 2t+1).
#if defined(LYRA_EMU)
static inline float lyra_emu_tf32(uint32_t bits) {          // the tensor core reads the top 19 bits of each operand
  bits &= 0xffffe000u;
  float f;
  std::memcpy(&f, &bits, 4);
  return f;
}
static inline void lyra_mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  const uint32_t mine[6] = {a[0], a[1], a[2], a[3], b[0], b[1]};
  const uint32_t (*all)[8] = cuda_emu::warp_gather(mine, 6);
  const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
  auto A = [&](int row, int k) { return (double)lyra_emu_tf32(all[(row & 7) * 4 + (k & 3)][(row >> 3) + 2 * (k >> 2)]); };
  auto B = [&](int k, int col) { return (double)lyra_emu_tf32(all[col * 4 + (k & 3)][4 + (k >> 2)]); };
  double d[4] = {c[0], c[1], c[2], c[3]};
  for (int k = 0; k < 8; ++k) {
    d[0] += A(g, k) * B(k, 2 * t);
    d[1] += A(g, k) * B(k, 2 * t + 1);
    d[2] += A(g + 8, k) * B(k, 2 * t);
    d[3] += A(g + 8, k) * B(k, 2 * t + 1);
  }
  cuda_emu::warp_barrier();
  c[0] = (float)d[0]; c[1] = (float)d[1]; c[2] = (float)d[2]; c[3] = (float)d[3];
}
#elif defined(__CUDACC__)
__device__ __forceinline__ void lyra_mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
#endif

// ---- warpgroup MMA (wgmma, sm_90a): D[64 x N] (+)= A[64 x 8] * B[N x 8]^T in TF32 with fp32 accumulators in the registers of
//      the four warps of a warpgroup (128 consecutive threads, the first a multiple of 128).  The MMA reads the top 19 bits of
//      every operand.  Shared-memory operands are K-major without swizzle, addressed by a matrix descriptor:
//        element (row, k) at start + (k / 4) * LBO + (row / 8) * SBO + (row % 8) * 16 + (k % 4) * 4   bytes
//      i.e. 8-row x 16-byte core matrices, LBO = byte distance of the two 4-element k-halves of one MMA (K = 8),
//      SBO = byte distance of consecutive 8-row groups.
//      Register fragments (warp q of the warpgroup, g = lane / 4, t = lane % 4):
//        A:  a0 (16q + g, t)   a1 (16q + g + 8, t)   a2 (16q + g, t + 4)   a3 (16q + g + 8, t + 4)
//        D:  d[4j] (16q + g, 8j + 2t)   d[4j + 1] (16q + g, 8j + 2t + 1)   d[4j + 2] (16q + g + 8, 8j + 2t)   d[4j + 3] (16q + g + 8, 8j + 2t + 1)
//      Issue order: lyra_wgmma_fence() before the first MMA that touches registers written since, the MMAs, lyra_wgmma_commit(),
//      and lyra_wgmma_wait<0>() before the accumulators are read or a shared-memory operand is overwritten.
#if defined(LYRA_EMU)
static inline uint32_t lyra_emu_smem_addr(const void* p) { return (uint32_t)(reinterpret_cast<const char*>(p) - cuda_emu::g_blk->smem); }
static inline uint64_t lyra_wgmma_desc(const void* smem, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((lyra_emu_smem_addr(smem) >> 4) & 0x3FFF) | (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16 |
         (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
}
static inline double lyra_emu_desc_elem(uint64_t d, int row, int k) {
  const uint32_t start = (uint32_t)(d & 0x3FFF) << 4, lbo = (uint32_t)((d >> 16) & 0x3FFF) << 4, sbo = (uint32_t)((d >> 32) & 0x3FFF) << 4;
  uint32_t bits;
  std::memcpy(&bits, cuda_emu::g_blk->smem + start + (uint32_t)(k / 4) * lbo + (uint32_t)(row / 8) * sbo + (uint32_t)(row % 8) * 16 + (uint32_t)(k % 4) * 4, 4);
  return (double)lyra_emu_tf32(bits);
}
// the emulated MMA completes on the spot: fence, commit and wait have nothing to order
static inline void lyra_wgmma_fence() {}
static inline void lyra_wgmma_commit() {}
template <int N>
static inline void lyra_wgmma_wait() {}
// every thread computes its own accumulator fragment from the shared-memory operands
static inline void lyra_wgmma_m64n32_tf32_ss(float (&d)[16], uint64_t desc_a, uint64_t desc_b, bool accumulate) {
  const int lane = (int)(threadIdx.x & 31), q = (int)((threadIdx.x >> 5) & 3), g = lane >> 2, t = lane & 3;
  for (int i = 0; i < 16; ++i) {
    const int row = 16 * q + g + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * t + (i & 1);
    double acc = accumulate ? (double)d[i] : 0.0;
    for (int k = 0; k < 8; ++k) acc += lyra_emu_desc_elem(desc_a, row, k) * lyra_emu_desc_elem(desc_b, col, k);
    d[i] = (float)acc;
  }
}
// A from registers: a warp's 16 rows of A are its own fragments, so the warp's lanes exchange theirs
static inline void lyra_wgmma_m64n64_tf32_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, bool accumulate) {
  const uint32_t (*all)[8] = cuda_emu::warp_gather(a, 4);
  const int lane = (int)(threadIdx.x & 31), g = lane >> 2, t = lane & 3;
  auto A = [&](int row, int k) { return (double)lyra_emu_tf32(all[(row & 7) * 4 + (k & 3)][(row >> 3) + 2 * (k >> 2)]); };
  float out[32];
  for (int i = 0; i < 32; ++i) {
    const int row = g + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * t + (i & 1);
    double acc = accumulate ? (double)d[i] : 0.0;
    for (int k = 0; k < 8; ++k) acc += A(row, k) * lyra_emu_desc_elem(desc_b, col, k);
    out[i] = (float)acc;
  }
  cuda_emu::warp_barrier();             // keep the table alive until every lane has read it
  for (int i = 0; i < 32; ++i) d[i] = out[i];
}
#elif defined(__CUDACC__)
__device__ __forceinline__ uint64_t lyra_wgmma_desc(const void* smem, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((lyra_smem_u32(smem) >> 4) & 0x3FFF) | (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16 |
         (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;                 // layout type 0: no swizzle
}
__device__ __forceinline__ void lyra_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void lyra_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void lyra_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory"); }
__device__ __forceinline__ void lyra_wgmma_m64n32_tf32_ss(float (&d)[16], uint64_t desc_a, uint64_t desc_b, bool accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(desc_a), "l"(desc_b), "r"(accumulate ? 1u : 0u));
}
__device__ __forceinline__ void lyra_wgmma_m64n64_tf32_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, bool accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
               "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
               "{%32,%33,%34,%35}, %36, p, 1, 1;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                 "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                 "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                 "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate ? 1u : 0u));
}
#endif

// ---- bulk asynchronous store shared -> global (TMA, cp.async.bulk.global.shared::cta) and named barriers for warp subsets.
//      Stores are grouped with lyra_bulk_commit(); lyra_bulk_wait_read() returns once the shared-memory source of every committed
//      group may be overwritten, lyra_bulk_wait_all() once the writes themselves are complete.  One thread issues and waits.
#if defined(LYRA_EMU)
static inline void lyra_bulk_s2g(void* gmem_dst, const void* smem_src, unsigned bytes) { std::memcpy(gmem_dst, smem_src, bytes); }
static inline void lyra_prefetch_l2(const void*, unsigned) {}
static inline void lyra_bulk_commit() {}
static inline void lyra_bulk_wait_read() {}
static inline void lyra_bulk_wait_all() {}
// barrier `id` (1..15) over `nthreads` threads (a multiple of 32): every participating thread calls it
static inline void lyra_named_bar_sync(int id, int nthreads) {
  cuda_emu::BlockState* b = cuda_emu::g_blk;
  unsigned* st = reinterpret_cast<unsigned*>(b->static_smem + 448) + 2 * (id & 7);     // {arrived, generation}; ids are used modulo 8 here
  const unsigned gen = st[1];
  if (++st[0] == (unsigned)nthreads) { st[0] = 0; st[1] = gen + 1; }
  while (st[1] == gen) cuda_emu::yield();
}
#elif defined(__CUDACC__)
// asks the L2 to fetch `bytes` (multiple of 16) starting at the 16-byte aligned global address: a hint, no completion to wait for
__device__ __forceinline__ void lyra_prefetch_l2(const void* gmem, unsigned bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;\n" ::"l"(gmem), "r"(bytes) : "memory");
}
__device__ __forceinline__ void lyra_bulk_s2g(void* gmem_dst, const void* smem_src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" ::"l"(gmem_dst), "r"(lyra_smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void lyra_bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void lyra_bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
__device__ __forceinline__ void lyra_bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }
__device__ __forceinline__ void lyra_named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(nthreads) : "memory"); }
#endif
