// TEST INFRASTRUCTURE ONLY — see cuda_emu.h.
#include "cuda_emu.h"

namespace cuda_emu {

thread_local BlockState* g_blk = nullptr;
thread_local uint3_emu g_threadIdx{0, 0, 0}, g_blockIdx{0, 0, 0};
thread_local dim3 g_blockDim, g_gridDim;

static const size_t kStack = 256 * 1024;

static void fiber_entry() {
  BlockState* b = g_blk;
  b->body();
  const unsigned me = b->cur;
  b->state[me] = 2;
  b->done++;
  b->warp_live[me / 32]--;
  swapcontext(&b->ctx[me], &b->sched);
}

static void yield_to_sched() {
  BlockState* b = g_blk;
  swapcontext(&b->ctx[b->cur], &b->sched);
}

void block_barrier() {
  BlockState* b = g_blk;
  b->state[b->cur] = 1;
  b->arrived++;
  yield_to_sched();
}

void warp_barrier() {
  BlockState* b = g_blk;
  b->state[b->cur] = 3;
  b->warp_arrived[b->cur / 32]++;
  yield_to_sched();
}

void yield() { yield_to_sched(); }

uint64_t warp_exchange(uint64_t v, int src_lane) {
  BlockState* b = g_blk;
  const unsigned w = b->cur / 32, lane = b->cur % 32;
  b->warp_xchg[w][lane] = v;
  warp_barrier();
  const uint64_t r = b->warp_xchg[w][src_lane & 31];
  warp_barrier();
  return r;
}

const uint32_t (*warp_gather(const uint32_t* vals, int n))[8] {
  BlockState* b = g_blk;
  const unsigned w = b->cur / 32, lane = b->cur % 32;
  warp_barrier();                       // previous readers of the table are done
  for (int i = 0; i < n; ++i) b->warp_scratch[w][lane][i] = vals[i];
  warp_barrier();
  return b->warp_scratch[w];
}

void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()>& body) {
  BlockState b;
  const unsigned nt = block.x * block.y * block.z;
  if (nt > 2048 || nt == 0) { std::fprintf(stderr, "cuda_emu: bad block size\n"); std::abort(); }
  b.nthreads = nt;
  b.ctx.resize(nt);
  b.stacks.resize(nt);
  b.state.assign(nt, 0);
  const unsigned nwarps = (nt + 31) / 32;
  b.warp_arrived.assign(nwarps, 0);
  b.warp_live.assign(nwarps, 0);
  for (unsigned t = 0; t < nt; ++t) b.stacks[t] = (char*)std::malloc(kStack);
  b.smem = (char*)std::aligned_alloc(1024, ((smem_bytes + 1023) / 1024 + 1) * 1024);
  b.body = body;
  g_blk = &b;
  g_blockDim = block;
  g_gridDim = grid;
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        g_blockIdx = uint3_emu{bx, by, bz};
        std::memset(b.smem, 0xCD, smem_bytes);   // poison: uninitialised shared memory shows up as garbage
        std::memset(b.static_smem, 0, sizeof(b.static_smem));
        b.arrived = 0;
        b.done = 0;
        for (unsigned w = 0; w < nwarps; ++w) {
          b.warp_arrived[w] = 0;
          b.warp_live[w] = (w + 1) * 32 <= nt ? 32 : nt - w * 32;
        }
        for (unsigned t = 0; t < nt; ++t) {
          getcontext(&b.ctx[t]);
          b.ctx[t].uc_stack.ss_sp = b.stacks[t];
          b.ctx[t].uc_stack.ss_size = kStack;
          b.ctx[t].uc_link = &b.sched;
          makecontext(&b.ctx[t], (void (*)())fiber_entry, 0);
          b.state[t] = 0;
        }
        // round-robin scheduler
        while (b.done < nt) {
          bool progressed = false;
          for (unsigned t = 0; t < nt; ++t) {
            if (b.state[t] != 0) continue;
            b.cur = t;
            g_threadIdx = uint3_emu{t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
            progressed = true;
            swapcontext(&b.sched, &b.ctx[t]);
          }
          // release warp barriers whose live lanes have all arrived
          for (unsigned w = 0; w < nwarps; ++w)
            if (b.warp_live[w] > 0 && b.warp_arrived[w] == b.warp_live[w]) {
              b.warp_arrived[w] = 0;
              for (unsigned t = w * 32; t < nt && t < (w + 1) * 32; ++t)
                if (b.state[t] == 3) b.state[t] = 0;
              progressed = true;
            }
          // release the block barrier when every live thread has arrived
          if (b.arrived > 0 && b.arrived == nt - b.done) {
            b.arrived = 0;
            for (unsigned t = 0; t < nt; ++t)
              if (b.state[t] == 1) b.state[t] = 0;
            progressed = true;
          }
          if (!progressed) {
            std::fprintf(stderr, "cuda_emu: deadlock (divergent barrier?) in block %u\n", bx);
            std::abort();
          }
        }
      }
  for (unsigned t = 0; t < nt; ++t) std::free(b.stacks[t]);
  std::free(b.smem);
  g_blk = nullptr;
}

}  // namespace cuda_emu
