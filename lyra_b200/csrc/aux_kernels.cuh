// RVQ encode/decode + bit packing, per-stream state records and the log-mel front end.
#pragma once

#include "kernel_prims.cuh"
#include "net_kernels.cuh"

namespace lyra_b200 {

constexpr int kRvqBitsPerStage = 4;

// ------------------------------------------------------------------------------------------------
// The two by-value parameters of the per-row kernels (the codec kernels that work on the rows, or slots, of a call rather than
// on tiles; the conv nets take a TileIo).  Read their fields directly: indexing an array inside a by-value parameter with a
// runtime index would copy it to local memory.  The kernels take them as `const __grid_constant__`, read in place in the
// parameter space: taken by plain value they cost LogMelKernel and ComfortNoiseKernel registers (and the latter a stack
// frame) over the scalar arguments they replace.
//
// RowIo: the rows of one part of a call, slots [slot0, slot0 + slots).  Every by-slot array of the call is indexed with
// absolute slots.  Slot s serves stream ids[s] (ids nullptr: stream s).  A sparse plain encode / decode at 16 kHz whose streams
// have no bit count of their own uploads no ids, so its ids are nullptr although slot s is not stream s: that is allowed only
// because no kernel of that chain reads anything by stream id.  active (lyra_b200_set_active_mask, by slot; nullptr: every slot
// runs): a slot whose byte is 0 sits the call out, as a reference object that is not called this hop.
struct RowIo {
  const int* ids;
  int slot0, slots;
  const uint8_t* active;
  __device__ __forceinline__ int Stream(int slot) const { return ids ? ids[slot] : slot; }
  __device__ __forceinline__ bool SatOut(int slot) const { return active != nullptr && !active[slot]; }
};

// StreamWords: the per-stream words a kernel reads, by stream id; a null pointer means every stream follows the call or the
// context.  rate (lyra_b200_set_stream_sample_rates): 0 = the context's rate ctx_rate, otherwise the stream's own.  bits
// (lyra_b200_set_stream_bits, the call's role): 0 = the call's bit count, otherwise the stream's own (at most the call's, checked
// by the host).  dtx_off (lyra_b200_set_stream_dtx): not 0 = the stream has no DTX estimator.
struct StreamWords {
  const int* rate;
  int ctx_rate;
  const int* bits;
  const int* dtx_off;
  __device__ __forceinline__ int Rate(int stream) const {
    if (!rate) return ctx_rate;
    const int w = rate[stream];
    return w ? w : ctx_rate;
  }
  // RVQ stages of the stream in a call of nq stages
  __device__ __forceinline__ int Stages(int stream, int nq) const {
    if (!bits) return nq;
    const int w = bits[stream];
    return w ? w / kRvqBitsPerStage : nq;
  }
  __device__ __forceinline__ bool DtxOff(int stream) const { return dtx_off != nullptr && dtx_off[stream] != 0; }
};

// ------------------------------------------------------------------------------------------------
// Residual vector quantizer, encode side + Packet<184>::PackQuantized (0 header bits).
// Replaces ResidualVectorQuantizer::Quantize (lyra/residual_vector_quantizer.cc:77-110; the "encode"
// subgraph of quantizer.tflite) and Packet::Pack (lyra/packet.h:91-122).
// 16 lanes per stream (one per codeword), two streams per warp.  Per stage, exactly the graph's ops:
//   d[c] = sum_j (r[j] - cb[c][j])^2 (ascending j, each op rounded), argmin with lowest-index ties,
//   q = cb[best]; t = q - r; u = r + t; r = r - u.
// Only the first `nq` stages are evaluated (a stream with a bit count of its own: StreamWords::Stages): later stages never
// influence earlier indices.
constexpr int kRvqThreads = 128;
constexpr int kRvqSlotsPerBlock = kRvqThreads / 16;

// A block runs its stage loop to the largest stage count among its slots (the codebook double buffer is shared); each slot packs
// its own stages into the first ceil(bits / 8) bytes of its row and zeros over the rest of the row.  A slot that sits out gets
// an all-zero packet, like a skipped one.
__global__ void __launch_bounds__(kRvqThreads)
RvqEncodeKernel(const uint8_t* __restrict__ blob, RvqParams P, const __grid_constant__ RowIo io, const __grid_constant__ StreamWords words,
                const float* __restrict__ features, int nq, uint8_t* __restrict__ packets, int packet_bytes, int* __restrict__ indices_out,
                const uint8_t* __restrict__ skip) {
  unsigned char* smem = LYRA_DYN_SMEM();
  float* cbs = reinterpret_cast<float*>(smem);                                  // [2][64][16] stage codebooks (double buffer, 16-byte aligned)
  float* rs = cbs + 2 * 1024;                                                   // [slots][64] residuals
  int* idxs = reinterpret_cast<int*>(rs + kRvqSlotsPerBlock * 64);              // [slots][48]
  const int tid = (int)threadIdx.x, grp = tid / 16, c = tid % 16;
  const int row = (int)blockIdx.x * kRvqSlotsPerBlock + grp, slot = io.slot0 + row;
  const bool valid = row < io.slots;
  const int my_nq = valid ? words.Stages(io.Stream(slot), nq) : 0;
  int block_nq = nq;
  if (words.bits) {
    block_nq = 0;
    for (int g = 0; g < kRvqSlotsPerBlock; ++g) {
      const int r = (int)blockIdx.x * kRvqSlotsPerBlock + g;
      if (r < io.slots) block_nq = max(block_nq, words.Stages(io.Stream(io.slot0 + r), nq));
    }
  }
  // DTX: the hop was noise, its packet is empty (bytes zeroed); the same for a slot that sits out
  const bool skipped = valid && (io.SatOut(slot) || (skip != nullptr && skip[slot]));
  float* r = rs + grp * 64;
  int* idx = idxs + grp * 48;
  const float* cbt = BlobPtr<float>(blob, P.codebooks_t);
  // per-stage codebooks (4 KB each) arrive by bulk asynchronous copy (TMA) into a double buffer; one mbarrier per buffer
  LYRA_STATIC_SMEM(LyraMbar, full, 2);
  if (tid == 0) {
    lyra_mbar_init(&full[0], 1);
    lyra_mbar_init(&full[1], 1);
    lyra_mbar_fence_init();
    lyra_bulk_g2s(cbs, cbt, 4096u, &full[0]);
  }
  for (int jj = 0; jj < 4; ++jj) r[c + 16 * jj] = valid ? features[(size_t)slot * 64 + c + 16 * jj] : 0.0f;
  for (int s = 0; s < block_nq; ++s) {
    __syncthreads();                       // everyone finished stage s-1: its buffer is free again (and the barriers are initialised)
    if (tid == 0 && s + 1 < block_nq) lyra_bulk_g2s(cbs + ((s + 1) & 1) * 1024, cbt + (size_t)(s + 1) * 1024, 4096u, &full[(s + 1) & 1]);
    lyra_mbar_wait(&full[s & 1], (unsigned)((s >> 1) & 1));     // codebook s has landed
    const float* cs = cbs + (s & 1) * 1024 + c;
    float d = 0.0f;
#pragma unroll 16
    for (int j = 0; j < 64; ++j) {
      const float df = __fsub_rn(r[j], cs[j * 16]);
      d = __fadd_rn(d, __fmul_rn(df, df));
    }
    int best = c;
#pragma unroll
    for (int m = 8; m >= 1; m >>= 1) {
      const float od = __shfl_xor_sync(0xffffffffu, d, m, 16);
      const int oi = __shfl_xor_sync(0xffffffffu, best, m, 16);
      if (od < d || (od == d && oi < best)) { d = od; best = oi; }
    }
    __syncwarp();
    const float* q = cbs + (s & 1) * 1024 + best;      // q[j] = codebook[best][j] at q[j * 16]
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = c + 16 * jj;
      const float rj = r[j];
      const float t = __fsub_rn(q[j * 16], rj);
      const float u = __fadd_rn(rj, t);
      r[j] = __fsub_rn(rj, u);
    }
    if (c == 0) idx[s] = best;
  }
  __syncthreads();
  if (valid) {
    // first quantizer in the most significant bits (residual_vector_quantizer.cc:101-109), bytes MSB-first
    for (int b = c; b < packet_bytes; b += 16) {
      const int hi = 2 * b < my_nq ? idx[2 * b] : 0, lo = 2 * b + 1 < my_nq ? idx[2 * b + 1] : 0;
      packets[(size_t)slot * packet_bytes + b] = skipped ? (uint8_t)0 : (uint8_t)((hi << 4) | lo);
    }
    if (indices_out)
      for (int s = c; s < P.num_stages; s += 16) indices_out[(size_t)slot * P.num_stages + s] = s < my_nq ? idx[s] : -1;
  }
}

// ------------------------------------------------------------------------------------------------
// RVQ decode: Packet::UnpackPacket (lyra/packet.h:62-71,126-146) + DecodeToLossyFeatures
// (lyra/residual_vector_quantizer.cc:112-168, "decode" subgraph): left-to-right sum over all 46 stages,
// unused stages contribute codebook[0] * 0.  A stream whose packet was not received gets 64 zero
// features (ZeroFeatureEstimator, lyra/lyra_decoder.cc:317-326).  A slot reads its stream's own stage count from the first
// ceil(bits / 8) bytes of its row, so a stream at b bits decodes bit for bit like a call at b bits.  A slot that sits out reads
// neither its packet nor its received byte and gets zeros; its 320-sample row of sat_out_pcm (nullptr: none) is written as zeros
// here, since the decoder nets skip it.
__global__ void __launch_bounds__(256)
RvqDecodeKernel(const uint8_t* __restrict__ blob, RvqParams P, const __grid_constant__ RowIo io, const __grid_constant__ StreamWords words,
                const uint8_t* __restrict__ packets, int packet_bytes, const uint8_t* __restrict__ received, int nq,
                float* __restrict__ features, int16_t* __restrict__ sat_out_pcm) {
  const int gid = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  const int row = gid / 64, j = gid % 64, slot = io.slot0 + row;
  if (row >= io.slots) return;
  nq = words.Stages(io.Stream(slot), nq);
  float out = 0.0f;
  const bool sat_out = io.SatOut(slot);
  if (sat_out && sat_out_pcm)
    for (int k = j; k < 320; k += 64) sat_out_pcm[(size_t)slot * 320 + k] = 0;
  if (!sat_out && (received == nullptr || received[slot])) {
    const float* cb = BlobPtr<float>(blob, P.codebooks);
    const uint8_t* pk = packets + (size_t)slot * packet_bytes;
    for (int k = 0; k < P.num_stages; ++k) {
      float t;
      if (k < nq) {
        const int byte = pk[k >> 1];
        const int idx = (k & 1) ? (byte & 15) : (byte >> 4);
        t = __fmul_rn(cb[((size_t)k * 16 + idx) * 64 + j], 1.0f);
      } else {
        t = __fmul_rn(cb[((size_t)k * 16) * 64 + j], 0.0f);
      }
      out = k == 0 ? t : __fadd_rn(out, t);
    }
  }
  features[(size_t)slot * 64 + j] = out;
}

// ------------------------------------------------------------------------------------------------
// Per-stream state records: lyra_b200_export_streams (gather), _import_streams (scatter), _copy_streams and _reset (copy).
// Every kernel is one launch over all entries of a state table (blockIdx.y = entry; reset's table leaves out the entries reset
// keeps) and 8 consecutive rows of the call per block (blockIdx.x).  A tile-blocked entry (lanes = 8) is read / written with the 8 rows of a block on 8 consecutive threads, so rows
// that are the 8 lanes of one tile move whole 32-byte tile rows; the records side goes through shared memory and moves whole
// lines.  Row-major entries (lanes = 1) are contiguous per stream on both sides.
//
// Record = kStateHeaderWords header words, then the entries' words in list order (each entry: its `words` words, then its hop
// counter if it has one).  Two kinds of words are not copied verbatim between contexts:
//   kStateCodecRs{0,1}  {position, tag} of a codec converter: the tag is a per-context counter (ResampleKernel); the record
//                       stores 0 in its place and "was live" (tag == the context's) in the header; import writes the
//                       destination's tag for a live converter and 0 (restart primed) otherwise;
//   kStateCng           {hop counter, key offset} (2 x u64) of a comfort-noise generator: the phases are drawn from
//                       seed + stream + offset; the record stores 0 for the offset and the key stream + offset in the header,
//                       import and copy set the offset so that the key travels with the stream.
enum StreamStateKind { kStatePlain = 0, kStateCodecRs0 = 1, kStateCodecRs1 = 2, kStateCng = 3 };
constexpr uint32_t kStateMagic = 0x5453594Cu;        // "LYST"
// 2: the per-stream sample rate joined the payload; 3: the per-stream bit counts.  The per-stream DTX word kept 3: it adds a word
// to encoder-role records only, whose size word (kHdrBytes) already refuses the shorter records, and decoder-only records did
// not change.  The call statistics (one entry per role) kept 3 for the same reason: every record grew, so its size word differs.
constexpr uint32_t kStateVersion = 3;
constexpr int kStateHeaderWords = 16;
// header words: magic, version, record bytes, roles, sample rate, 0, model fingerprint (lo, hi), codec converter 0 / 1 live,
// comfort-noise key (lo, hi), 0 x 4
enum { kHdrMagic = 0, kHdrVersion, kHdrBytes, kHdrRoles, kHdrRate, kHdrZero5, kHdrModelLo, kHdrModelHi, kHdrLive0, kHdrLive1,
       kHdrKeyLo, kHdrKeyHi };
constexpr int kStateMaxEntries = 27;                 // a context with both roles registers exactly 27: a new per-stream entry raises it
constexpr int kStateRows = 8;                        // rows of a call per block
constexpr int kStateChunk = 1024;                    // rows per launch (the ids travel as kernel parameters)
constexpr int kStateThreads = 256;
constexpr int kStateSmemUnits = 256;                 // units per shared-memory pass of a tile-blocked entry
constexpr int kStateSmemBytes = kStateRows * kStateSmemUnits * 4;

struct StreamStateEntry {
  uint32_t* state;
  const uint32_t* init;          // one stream's initial words (nullptr: zero)
  int* n18;                      // hop counter (nullptr: none)
  int words, lanes, offset, kind;   // offset: first word of the entry in a record
};
struct StreamStateTable {
  StreamStateEntry e[kStateMaxEntries];
  int count, record_words;
  uint32_t header[kStateHeaderWords];   // the context's constant header words (export)
};
// src: export / copy sources (-1 in a copy: the state at creation), dst: import / copy destinations
struct StreamIdChunk { int n; int src[kStateChunk]; int dst[kStateChunk]; };

__device__ __forceinline__ uint32_t* StateWord(const StreamStateEntry& e, int stream, int u) {
  return e.lanes == 1 ? e.state + (size_t)stream * e.words + u
                      : e.state + ((size_t)(stream / e.lanes) * e.words + u) * e.lanes + stream % e.lanes;
}
__device__ __forceinline__ unsigned long long StateU64(const StreamStateEntry& e, int stream, int u) {
  return (unsigned long long)*StateWord(e, stream, u) | ((unsigned long long)*StateWord(e, stream, u + 1) << 32);
}
__device__ __forceinline__ uint32_t InitWord(const StreamStateEntry& e, int u) { return e.init ? e.init[u] : 0u; }

// records[k] <- the state of stream ids.src[k]; tag = the context's codec converter tag
__global__ void __launch_bounds__(kStateThreads)
StreamStateGatherKernel(StreamStateTable T, StreamIdChunk ids, uint32_t* __restrict__ records, int tag) {
  uint32_t* sm = reinterpret_cast<uint32_t*>(LYRA_DYN_SMEM());   // [kStateRows][kStateSmemUnits] (kStateSmemBytes)
  const int r0 = (int)blockIdx.x * kStateRows, tid = (int)threadIdx.x;
  const int rows = ids.n - r0 < kStateRows ? ids.n - r0 : kStateRows;
  if (rows <= 0) return;
  const int RW = T.record_words;
  if ((int)blockIdx.y == T.count) {                  // the headers
    if (tid >= rows) return;
    const int s = ids.src[r0 + tid];
    uint32_t* h = records + (size_t)(r0 + tid) * RW;
    for (int i = 0; i < kStateHeaderWords; ++i) h[i] = T.header[i];
    for (int i = 0; i < T.count; ++i) {
      const StreamStateEntry& e = T.e[i];
      if (e.kind == kStateCodecRs0 || e.kind == kStateCodecRs1)
        h[kHdrLive0 + e.kind - kStateCodecRs0] = (int)*StateWord(e, s, 1) == tag ? 1u : 0u;
      if (e.kind == kStateCng) {
        const unsigned long long key = StateU64(e, s, 2) + (unsigned long long)s;
        h[kHdrKeyLo] = (uint32_t)key;
        h[kHdrKeyHi] = (uint32_t)(key >> 32);
      }
    }
    return;
  }
  const StreamStateEntry e = T.e[blockIdx.y];
  uint32_t* out = records + kStateHeaderWords + e.offset;
  if (e.lanes == 1) {
    for (int j = 0; j < rows; ++j) {
      const uint32_t* st = e.state + (size_t)ids.src[r0 + j] * e.words;
      uint32_t* o = out + (size_t)(r0 + j) * RW;
      for (int u = tid; u < e.words; u += kStateThreads) {
        const bool dropped = (e.kind == kStateCodecRs0 || e.kind == kStateCodecRs1) ? u == 1 : e.kind == kStateCng && u >= 2;
        o[u] = dropped ? 0u : st[u];
      }
    }
  } else {
    const int j = tid % kStateRows, uu = tid / kStateRows;
    const int s = j < rows ? ids.src[r0 + j] : 0;
    for (int u0 = 0; u0 < e.words; u0 += kStateSmemUnits) {
      const int cnt = e.words - u0 < kStateSmemUnits ? e.words - u0 : kStateSmemUnits;
      if (j < rows)
        for (int u = uu; u < cnt; u += kStateThreads / kStateRows) sm[j * kStateSmemUnits + u] = *StateWord(e, s, u0 + u);
      __syncthreads();
      for (int jj = 0; jj < rows; ++jj)
        for (int u = tid; u < cnt; u += kStateThreads) out[(size_t)(r0 + jj) * RW + u0 + u] = sm[jj * kStateSmemUnits + u];
      __syncthreads();
    }
  }
  if (e.n18 && tid < rows) out[(size_t)(r0 + tid) * RW + e.words] = (uint32_t)e.n18[ids.src[r0 + tid]];
}

// stream ids.dst[k] <- records[k] (validated by the host); tag = the context's codec converter tag
__global__ void __launch_bounds__(kStateThreads)
StreamStateScatterKernel(StreamStateTable T, StreamIdChunk ids, const uint32_t* __restrict__ records, int tag) {
  uint32_t* sm = reinterpret_cast<uint32_t*>(LYRA_DYN_SMEM());   // [kStateRows][kStateSmemUnits] (kStateSmemBytes)
  const int r0 = (int)blockIdx.x * kStateRows, tid = (int)threadIdx.x;
  const int rows = ids.n - r0 < kStateRows ? ids.n - r0 : kStateRows;
  if (rows <= 0) return;
  const int RW = T.record_words;
  const StreamStateEntry e = T.e[blockIdx.y];
  const uint32_t* in = records + kStateHeaderWords + e.offset;
  if (e.lanes == 1) {
    for (int j = 0; j < rows; ++j) {
      const int d = ids.dst[r0 + j];
      const uint32_t* h = records + (size_t)(r0 + j) * RW;
      const uint32_t* x = in + (size_t)(r0 + j) * RW;
      uint32_t* st = e.state + (size_t)d * e.words;
      const unsigned long long off = (((unsigned long long)h[kHdrKeyHi] << 32) | h[kHdrKeyLo]) - (unsigned long long)d;
      for (int u = tid; u < e.words; u += kStateThreads) {
        uint32_t v = x[u];
        if ((e.kind == kStateCodecRs0 || e.kind == kStateCodecRs1) && u == 1) v = h[kHdrLive0 + e.kind - kStateCodecRs0] ? (uint32_t)tag : 0u;
        if (e.kind == kStateCng && u >= 2) v = u == 2 ? (uint32_t)off : (uint32_t)(off >> 32);
        st[u] = v;
      }
    }
  } else {
    const int j = tid % kStateRows, uu = tid / kStateRows;
    const int d = j < rows ? ids.dst[r0 + j] : 0;
    for (int u0 = 0; u0 < e.words; u0 += kStateSmemUnits) {
      const int cnt = e.words - u0 < kStateSmemUnits ? e.words - u0 : kStateSmemUnits;
      for (int jj = 0; jj < rows; ++jj)
        for (int u = tid; u < cnt; u += kStateThreads) sm[jj * kStateSmemUnits + u] = in[(size_t)(r0 + jj) * RW + u0 + u];
      __syncthreads();
      if (j < rows)
        for (int u = uu; u < cnt; u += kStateThreads / kStateRows) *StateWord(e, d, u0 + u) = sm[j * kStateSmemUnits + u];
      __syncthreads();
    }
  }
  if (e.n18 && tid < rows) e.n18[ids.dst[r0 + tid]] = (int)in[(size_t)(r0 + tid) * RW + e.words];
}

// stream ids.dst[k] <- stream ids.src[k] within one context, lane to lane (sources and destinations are disjoint);
// ids.src[k] = -1: the entry's initial image
__global__ void __launch_bounds__(kStateThreads)
StreamStateCopyKernel(StreamStateTable T, StreamIdChunk ids) {
  const int r0 = (int)blockIdx.x * kStateRows, tid = (int)threadIdx.x;
  const int rows = ids.n - r0 < kStateRows ? ids.n - r0 : kStateRows;
  if (rows <= 0) return;
  const StreamStateEntry e = T.e[blockIdx.y];
  if (e.lanes == 1) {
    for (int j = 0; j < rows; ++j) {
      const int s = ids.src[r0 + j], d = ids.dst[r0 + j];
      // the key offset moves with the stream: seed + s + off(s) == seed + d + off(d)
      const unsigned long long off = e.kind == kStateCng && s >= 0 ? StateU64(e, s, 2) + (unsigned long long)s - (unsigned long long)d : 0ull;
      for (int u = tid; u < e.words; u += kStateThreads) {
        uint32_t v = s < 0 ? InitWord(e, u) : e.state[(size_t)s * e.words + u];
        if (e.kind == kStateCng && u >= 2) v = u == 2 ? (uint32_t)off : (uint32_t)(off >> 32);
        e.state[(size_t)d * e.words + u] = v;
      }
    }
  } else {
    const int j = tid % kStateRows, uu = tid / kStateRows;
    if (j < rows) {
      const int s = ids.src[r0 + j], d = ids.dst[r0 + j];
      for (int u = uu; u < e.words; u += kStateThreads / kStateRows) *StateWord(e, d, u) = s < 0 ? InitWord(e, u) : *StateWord(e, s, u);
    }
  }
  if (e.n18 && tid < rows) e.n18[ids.dst[r0 + tid]] = ids.src[r0 + tid] < 0 ? 0 : e.n18[ids.src[r0 + tid]];
}

// ------------------------------------------------------------------------------------------------
// lyra_b200_align_streams: stream ids.dst[k] takes the hop counter of stream ids.src[k] (-1: 0, the counter at creation) in every
// network entry of the table, and its depthwise rings are rotated so that it computes what it computed before.  A counter only
// places the rings: relative row r of a ring lives in slot (n T + r) mod R (kDwRings), so moving from n to m moves the content
// of slot p to slot p + d, d = ((m - n) T) mod R.  Same grid as the state-record kernels: blockIdx.y = entry, 8 rows of the call
// per block on 8 consecutive threads (whole 32-byte tile rows when the rows are the lanes of a tile), the other 32 threads of
// each row walk its ring columns.  A block reads and writes only its own rows' counters and rings, and no listed stream is a
// like stream, so blocks need no ordering between them.
struct StreamAlignEntry {
  uint32_t* state;               // tile-blocked [tile][units][kTileStreams]
  int* n18;
  int units, layout;             // layout: index w of the state layout (kDwRingFirst)
};
struct StreamAlignTable { StreamAlignEntry e[4]; int count; };

// entry y of the table, field by field: indexing the by-value parameter with y would copy it to local memory
__device__ __forceinline__ StreamAlignEntry PickAlignEntry(const StreamAlignTable& T, int y) {
  StreamAlignEntry e;
  e.state = y == 0 ? T.e[0].state : y == 1 ? T.e[1].state : y == 2 ? T.e[2].state : T.e[3].state;
  e.n18 = y == 0 ? T.e[0].n18 : y == 1 ? T.e[1].n18 : y == 2 ? T.e[2].n18 : T.e[3].n18;
  e.units = y == 0 ? T.e[0].units : y == 1 ? T.e[1].units : y == 2 ? T.e[2].units : T.e[3].units;
  e.layout = y == 0 ? T.e[0].layout : y == 1 ? T.e[1].layout : y == 2 ? T.e[2].layout : T.e[3].layout;
  return e;
}

// col[j] <- col[(j - d) mod R] for the R units of one ring column of one lane (unit stride kTileStreams); all R loads first
// (addresses vary, register indices do not)
template <int R>
__device__ __forceinline__ void RotateRingColumn(uint32_t* col, int d) {
  uint32_t v[R];
#pragma unroll
  for (int j = 0; j < R; ++j) v[j] = col[(j >= d ? j - d : j - d + R) * kTileStreams];
#pragma unroll
  for (int j = 0; j < R; ++j) col[j * kTileStreams] = v[j];
}

// rings I .. END - 1 of kDwRings for one lane (lane: its unit 0), counter n -> m; columns c0, c0 + step, ...
template <int I, int END>
__device__ __forceinline__ void AlignRings(uint32_t* lane, int n, int m, int c0, int step) {
  if constexpr (I < END) {
    constexpr DwRing g = kDwRings[I];
    int d = ((m - n) * g.T) % g.R;
    d += d < 0 ? g.R : 0;
    if (d)
      for (int c = c0; c < g.rows; c += step) RotateRingColumn<g.R>(lane + (size_t)(g.unit + c * g.R) * kTileStreams, d);
    AlignRings<I + 1, END>(lane, n, m, c0, step);
  }
}

__global__ void __launch_bounds__(kStateThreads)
StreamAlignKernel(StreamAlignTable T, StreamIdChunk ids) {
  const int r0 = (int)blockIdx.x * kStateRows, tid = (int)threadIdx.x;
  const int rows = ids.n - r0 < kStateRows ? ids.n - r0 : kStateRows;
  if (rows <= 0) return;
  const StreamAlignEntry e = PickAlignEntry(T, (int)blockIdx.y);
  const int j = tid % kStateRows, uu = tid / kStateRows;
  int s = 0, n = 0, m = 0;
  if (j < rows) {
    s = ids.dst[r0 + j];
    const int like = ids.src[r0 + j];
    n = e.n18[s];
    m = like < 0 ? 0 : e.n18[like];
    uint32_t* lane = e.state + (size_t)(s / kTileStreams) * e.units * kTileStreams + s % kTileStreams;
    constexpr int step = kStateThreads / kStateRows;
    if (m != n) {
      if (e.layout == 0) AlignRings<kDwRingFirst[0], kDwRingFirst[1]>(lane, n, m, uu, step);
      else if (e.layout == 1) AlignRings<kDwRingFirst[1], kDwRingFirst[2]>(lane, n, m, uu, step);
      else if (e.layout == 2) AlignRings<kDwRingFirst[2], kDwRingFirst[3]>(lane, n, m, uu, step);
      else AlignRings<kDwRingFirst[3], kDwRingFirst[4]>(lane, n, m, uu, step);
    }
  }
  __syncthreads();                                   // every thread of row j has read its counter
  if (tid < rows && m != n) e.n18[s] = m;            // thread tid < 8 is row tid
}

// ------------------------------------------------------------------------------------------------
// Per-stream sample rates of the fused codec calls (lyra_b200_set_stream_sample_rates).  Every stream has one state word: 0 =
// the context's rate (lyra_b200_set_sample_rate), otherwise the stream's own rate (8000 / 16000 / 32000 / 48000, at most the
// context's).  The converters (ResampleKernel) and the encoder-side DTX estimator (LogMelKernel, NoiseEstimatorKernel) read it.
// Index of a rate in a per-rate table (ByRate): 0 = 16 kHz, 1 = 8 kHz, 2 = 32 kHz, 3 = 48 kHz (= the resampler's pair + 1).
__host__ __device__ constexpr int RateIndex(int rate_hz) { return rate_hz == 8000 ? 1 : rate_hz == 32000 ? 2 : rate_hz == 48000 ? 3 : 0; }
// One parameter set per rate, by RateIndex.  A caller with a single set passes it at every index (Uniform).
template <typename T>
struct ByRate { T p[4]; };
template <typename T>
ByRate<T> Uniform(const T& v) { return ByRate<T>{{v, v, v, v}}; }
// the set of index k, selected field by field from the by-value kernel parameter (no dynamic indexing, so no local copy)
template <typename T>
__device__ __forceinline__ T PickByRate(const ByRate<T>& s, int k) {
  T v = s.p[0];
  if (k == 1) v = s.p[1];
  if (k == 2) v = s.p[2];
  if (k == 3) v = s.p[3];
  return v;
}

// The per-stream words' setter: stream c.ids[k] <- value c.values[k] (validated by the host), stored as 0 when it equals
// ctx_value.  The sample rates (ctx_value = the context's rate): a stream whose effective rate changes gets {position, tag} = 0
// in both codec converters (conv0 / conv1: nullptr when the context lacks that role): tag 0 never matches, so each restarts
// fully primed on its next call, as a context-level change does.  The networks, estimators and packet-loss state carry on.
// The bit counts (lyra_b200_set_stream_bits) and the DTX words (lyra_b200_set_stream_dtx): ctx_value = 0 and no converters, so
// the word is stored as given.
struct StreamWordChunk { int n; int ids[kStateChunk]; int values[kStateChunk]; };
constexpr int kStreamWordThreads = 256;

__global__ void __launch_bounds__(kStreamWordThreads)
StreamWordKernel(StreamWordChunk c, int ctx_value, int* __restrict__ word, int* __restrict__ conv0, int* __restrict__ conv1) {
  const int k = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (k >= c.n) return;
  const int s = c.ids[k], v = c.values[k], w = word[s];
  const int old = w ? w : ctx_value;
  word[s] = v == ctx_value ? 0 : v;
  if (v == old) return;
  if (conv0) { conv0[2 * (size_t)s] = 0; conv0[2 * (size_t)s + 1] = 0; }
  if (conv1) { conv1[2 * (size_t)s] = 0; conv1[2 * (size_t)s + 1] = 0; }
}

// ------------------------------------------------------------------------------------------------
// Log-mel spectrogram (LogMelSpectrogramExtractorImpl::Extract, lyra/log_mel_spectrogram_extractor_impl.cc:96-126).
// One block of 128 threads per stream: periodic-Hann window over [previous hop, current hop], zero-padded 1024-point
// radix-2 decimation-in-time FFT in double — the same butterflies, operand order and host-computed twiddles as the
// oracle, so the spectrum is bit-identical to it — |X|, triangular mel weights accumulated in bin order, float cast,
// log(max(x, 500)) / 10 with the logarithm taken in double and rounded once (equal to a correctly rounded logf).
// The ten stages run as 3 + 3 + 3 + 1: a thread keeps 8 points in registers across three consecutive stages (points
// base + j * STRIDE, the closed set of three stages whose half-lengths are STRIDE, 2 STRIDE, 4 STRIDE), so the block
// synchronises four times instead of ten.
// prev: [max_streams][window - hop] int16 carried samples (zero after reset).
constexpr int kLogMelThreads = 128;
constexpr int kLogMelFft = 1024;

// butterfly of stage `len` on (a, b = a + len/2) with twiddle w = tw[k * (fft / len)]:  x = b * w;  b = a - x;  a = a + x
__device__ __forceinline__ void FftButterfly(double& ar, double& ai, double& br, double& bi, double wr, double wi) {
  const double xr = __dsub_rn(__dmul_rn(br, wr), __dmul_rn(bi, wi));
  const double xi = __dadd_rn(__dmul_rn(br, wi), __dmul_rn(bi, wr));
  br = __dsub_rn(ar, xr); bi = __dsub_rn(ai, xi);
  ar = __dadd_rn(ar, xr); ai = __dadd_rn(ai, xi);
}

// shared-memory index of FFT point i: one pad element per 8 keeps the stride-8 and stride-64 register-blocked passes
// (nearly) free of bank conflicts
__device__ __forceinline__ int FftIdx(int i) { return i + (i >> 3); }
constexpr int kLogMelFftPadded = kLogMelFft + kLogMelFft / 8;

// three consecutive stages (half-lengths STRIDE, 2 STRIDE, 4 STRIDE) on the 8 points base + j * STRIDE; r = base mod STRIDE.
// tw: per-stage twiddle tables, the stage of half-length h starts at complex entry h - 1.  INV: the inverse transform's stages
// (conjugated twiddles).
template <int STRIDE, bool INV>
__device__ __forceinline__ void FftButterflies3(double (&xr)[8], double (&xi)[8], int r, const double2* __restrict__ tw) {
#pragma unroll
  for (int s = 0; s < 3; ++s) {
    const int half = STRIDE << s;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (!(j & (1 << s))) {
        const int k = r + (j & ((1 << s) - 1)) * STRIDE;
        const double2 w = tw[half - 1 + k];
        FftButterfly(xr[j], xi[j], xr[j + (1 << s)], xi[j + (1 << s)], w.x, INV ? -w.y : w.y);
      }
  }
}

template <int STRIDE, bool INV>
__device__ __forceinline__ void FftStages3(double* re, double* im, int base, int r, const double2* __restrict__ tw) {
  double xr[8], xi[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { xr[j] = re[FftIdx(base + j * STRIDE)]; xi[j] = im[FftIdx(base + j * STRIDE)]; }
  FftButterflies3<STRIDE, INV>(xr, xi, r, tw);
#pragma unroll
  for (int j = 0; j < 8; ++j) { re[FftIdx(base + j * STRIDE)] = xr[j]; im[FftIdx(base + j * STRIDE)] = xi[j]; }
}

// The whole 1024-point transform, run by one block of 128 threads: re / im (FftIdx layout) receive the spectrum (the signal if
// INV, unscaled) of the points that gather(i, xr, xi) reads in natural order i.  Ends with a block barrier.
template <bool INV, typename Gather>
__device__ __forceinline__ void Fft1024(double* re, double* im, const double2* __restrict__ tw, Gather gather) {
  constexpr int NT = 128;
  const int tid = (int)threadIdx.x;
  {                                                                            // stages 2, 4, 8 on points 8 tid .. 8 tid + 7
    double xr[8], xi[8];
    const int b7 = (int)(__brev((unsigned)tid) >> 25);                         // bit-reversed position 8t + j <-> natural index brev7(t) + 128 brev3(j)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int j3 = ((j & 1) << 2) | (j & 2) | ((j & 4) >> 2);
      gather(b7 + 128 * j3, xr[j], xi[j]);
    }
    FftButterflies3<1, INV>(xr, xi, 0, tw);
#pragma unroll
    for (int j = 0; j < 8; ++j) { re[FftIdx(8 * tid + j)] = xr[j]; im[FftIdx(8 * tid + j)] = xi[j]; }
  }
  __syncthreads();
  FftStages3<8, INV>(re, im, 64 * (tid / 8) + tid % 8, tid % 8, tw);           // stages 16, 32, 64
  __syncthreads();
  FftStages3<64, INV>(re, im, 512 * (tid / 64) + tid % 64, tid % 64, tw);      // stages 128, 256, 512
  __syncthreads();
#pragma unroll
  for (int m = 0; m < 4; ++m) {                                                // stage 1024
    const int a = tid + NT * m, ia = FftIdx(a), ib = FftIdx(a + 512);
    const double2 w = tw[511 + a];
    FftButterfly(re[ia], im[ia], re[ib], im[ib], w.x, INV ? -w.y : w.y);
  }
  __syncthreads();
}

// S: the extractor's tables by rate; each stream uses those of its rate (the encoder-side DTX estimator follows the stream's
// rate); the sets differ only in their tables, not in hop, window or FFT size.  A stream whose DTX is off has no DTX estimator,
// so its extractor is not fed either (no output, carried samples untouched).  A slot that sits out is not read or written at
// all, not even its update-mask byte.
__global__ void __launch_bounds__(kLogMelThreads)
LogMelKernel(const uint8_t* __restrict__ blob, ByRate<LogMelParams> S, const __grid_constant__ StreamWords words,
             const __grid_constant__ RowIo io, const int16_t* __restrict__ pcm, int16_t* __restrict__ prev, float* __restrict__ out,
             const uint8_t* __restrict__ mask) {
  unsigned char* smem = LYRA_DYN_SMEM();
  double* re = reinterpret_cast<double*>(smem);
  double* im = re + kLogMelFftPadded;
  double* mag = im + kLogMelFftPadded;       // [fft/2 + 1]
  double* xw = mag + kLogMelFft / 2 + 1;     // [window_len, padded like the FFT buffers] windowed samples in natural order
  if ((int)blockIdx.x >= io.slots) return;
  const int slot = io.slot0 + (int)blockIdx.x;
  if (io.SatOut(slot)) return;
  if (mask && !mask[slot]) return;     // this stream's extractor is not fed this hop (its carried samples stay)
  const int stream = io.Stream(slot);
  if (words.DtxOff(stream)) return;
  const LogMelParams P = PickByRate(S, RateIndex(words.Rate(stream)));
  const int tid = (int)threadIdx.x;
  constexpr int NT = kLogMelThreads;
  const int carry = P.window_len - P.hop;
  const double* win = BlobPtr<double>(blob, P.window);
  const double2* tw = BlobPtr<double2>(blob, P.twiddle);
  int16_t* pv = prev + (size_t)stream * carry;
  const int16_t* cur = pcm + (size_t)slot * P.hop;
  // windowed samples in natural order (the zero padding up to 1024 points is implicit)
  for (int i = tid; i < P.window_len; i += NT) {
    const int16_t smp = i < carry ? pv[i] : cur[i - carry];
    xw[FftIdx(i)] = __dmul_rn((double)smp, win[i]);
  }
  __syncthreads();
  // the carried samples become the tail of (previous carry, current hop); staged through `mag`
  {
    int16_t* stage = reinterpret_cast<int16_t*>(mag);
    for (int i = tid; i < carry; i += NT) {
      const int src = i + P.hop;
      stage[i] = src < carry ? pv[src] : cur[src - carry];
    }
    __syncthreads();
    for (int i = tid; i < carry; i += NT) pv[i] = stage[i];
  }
  Fft1024<false>(re, im, tw, [&](int i, double& xr, double& xi) {
    xr = i < P.window_len ? xw[FftIdx(i)] : 0.0;
    xi = 0.0;
  });
  const int bins = kLogMelFft / 2 + 1;
  for (int i = tid; i < bins; i += NT)
    mag[i] = __dsqrt_rn(__dadd_rn(__dmul_rn(re[FftIdx(i)], re[FftIdx(i)]), __dmul_rn(im[FftIdx(i)], im[FftIdx(i)])));
  __syncthreads();
  // each mel channel: bins of band ch-1 contribute (v - v*w), bins of band ch contribute v*w, in bin order
  const double* wts = BlobPtr<double>(blob, P.weights);
  const int* band = BlobPtr<int>(blob, P.band);
  const int* range = BlobPtr<int>(blob, P.range);
  for (int ch = tid; ch < P.num_mel; ch += NT) {
    double acc = 0.0;
    const int lo = range[2 * ch], hi = range[2 * ch + 1];
    for (int i = lo; i <= hi; ++i) {
      if (band[i] == ch) acc = __dadd_rn(acc, __dmul_rn(mag[i], wts[i]));
      else acc = __dadd_rn(acc, __dsub_rn(mag[i], __dmul_rn(mag[i], wts[i])));
    }
    float v = (float)acc;
    v = v > 500.0f ? v : 500.0f;
    out[(size_t)slot * P.num_mel + ch] = __fdiv_rn((float)log((double)v), 10.0f);
  }
}

// ------------------------------------------------------------------------------------------------
// Minimum-statistics noise estimator on the decoder output (SURVEY.md section 8 row f1):
// NoiseEstimator::ReceiveSamples for whole hops, after the log-mel kernel has produced this hop's
// 160-bin spectrum (lyra/noise_estimator.cc:144-245; SmoothingFactor / UpdateMinAndTemp :37-95).
// One block per stream, one thread per mel bin.  Per-stream state: est | bound | smoothed | squared-smoothed |
// tmp-min (nf floats each) followed by 4 ints {has_smoothed, hops_received, last_hop_was_not_noise, -} — all-zero
// is the reference's freshly constructed object (noise estimate and bound 0, is_noise() true).
// Arithmetic follows the C++ expression types: float ops rounded one by one, the bound in double
// (std::log of an integer is double), std::exp(float) as (float)exp((double)x) like the oracle.
// Streams whose mask byte is 0 are left untouched (LyraDecoder only feeds hops decoded from a received
// packet, lyra/lyra_decoder.cc:306-311) but still report their current is_noise / noise_estimate.
struct NoiseParams { int nf, hops_per_update; float max_smoothing, bound_decay; double log_nf; };
constexpr int kNoiseThreads = 192;
__host__ __device__ constexpr int NoiseStateUnits(int nf) { return 5 * nf + 4; }

// S: the constants by rate, selected per stream as in LogMelKernel (every set has nf = 160 bins).  A stream whose DTX is off
// reports is_noise 0 (LyraEncoder with enable_dtx = false encodes every hop) and its state is left alone - unlike a masked
// stream, which reports its current is_noise.  A slot that sits out leaves its state alone and its update-mask byte unread;
// encoder_side: it reports is_noise 1 (nothing to send, like an empty DTX packet); otherwise it reports its current is_noise /
// noise_estimate, like a masked stream.
__global__ void __launch_bounds__(kNoiseThreads)
NoiseEstimatorKernel(ByRate<NoiseParams> S, const __grid_constant__ StreamWords words, const __grid_constant__ RowIo io,
                     const float* __restrict__ mel, const uint8_t* __restrict__ mask, float* __restrict__ state,
                     uint8_t* __restrict__ is_noise_out, float* __restrict__ estimate_out, bool encoder_side) {
  if ((int)blockIdx.x >= io.slots) return;
  const int slot = io.slot0 + (int)blockIdx.x;
  const bool sat_out = io.SatOut(slot);
  if (sat_out && encoder_side) {
    if (is_noise_out && threadIdx.x == 0) is_noise_out[slot] = 1;
    return;
  }
  const int stream = io.Stream(slot);
  if (words.DtxOff(stream)) {
    if (is_noise_out && threadIdx.x == 0) is_noise_out[slot] = 0;
    return;
  }
  const NoiseParams P = PickByRate(S, RateIndex(words.Rate(stream)));
  unsigned char* smem = LYRA_DYN_SMEM();
  float* cur = reinterpret_cast<float*>(smem);       // [nf]
  float* sm = cur + P.nf;                             // [nf] smoothed power before this update
  float* red = sm + P.nf;                             // [0] smoothing correction
  int* flag = reinterpret_cast<int*>(red + 1);
  const int i = (int)threadIdx.x, nf = P.nf;
  float* st = state + (size_t)stream * NoiseStateUnits(nf);
  float* est = st;
  float* bound = st + nf;
  float* smoothed = st + 2 * nf;
  float* sq = st + 3 * nf;
  float* tmp_min = st + 4 * nf;
  int* meta = reinterpret_cast<int*>(st + 5 * nf);
  const bool feed = !sat_out && (mask == nullptr || mask[slot] != 0);
  if (!feed) {
    if (is_noise_out && i == 0) is_noise_out[slot] = meta[2] ? 0 : 1;
    if (estimate_out && i < nf) estimate_out[(size_t)slot * nf + i] = est[i];
    return;
  }
  const int has = meta[0], hops = meta[1];
  if (i == 0) *flag = 0;
  __syncthreads();
  float c = 0.0f, e = 0.0f, b = 0.0f;
  if (i < nf) {
    c = mel[(size_t)slot * nf + i];
    e = est[i];
    b = bound[i];
    cur[i] = c;
    if (fabsf(__fsub_rn(c, e)) > b) *flag = 1;       // ComputeIsNoise: any bin outside estimate +- bound
  }
  __syncthreads();
  const bool not_noise = *flag != 0;
  if (!not_noise) {
    if (i < nf) bound[i] = __fmul_rn(b, P.bound_decay);         // DecayBounds
  } else {
    float s = 0.0f, q = 0.0f, tm = 0.0f;
    if (i < nf) {
      s = has ? smoothed[i] : c;
      q = has ? sq[i] : __fmul_rn(c, c);
      tm = has ? tmp_min[i] : c;
      sm[i] = s;
    }
    __syncthreads();
    if (i == 0) {
      float a0 = 0.0f, a1 = 0.0f;                      // Average(): std::accumulate in index order, then / size
      for (int k = 0; k < nf; ++k) { a0 = __fadd_rn(a0, sm[k]); a1 = __fadd_rn(a1, cur[k]); }
      const float d = __fdiv_rn(__fsub_rn(__fdiv_rn(a0, (float)nf), __fdiv_rn(a1, (float)nf)), 0.3f);
      red[0] = (float)exp((double)(-__fmul_rn(d, d)));
    }
    __syncthreads();
    if (i < nf) {
      const float r = __fdiv_rn(__fsub_rn(s, e), 0.3f);
      const float sf = __fmul_rn(__fmul_rn(P.max_smoothing, red[0]), (float)exp((double)(-__fmul_rn(r, r))));
      const float om = __fsub_rn(1.0f, sf);
      const float ns = __fadd_rn(__fmul_rn(sf, s), __fmul_rn(om, c));
      const float nq = __fadd_rn(__fmul_rn(sf, q), __fmul_rn(om, __fmul_rn(c, c)));
      float ne, nt;
      if (hops == 0) { ne = ns < tm ? ns : tm; nt = ns; }          // UpdateMinAndTemp
      else { ne = ns < e ? ns : e; nt = ns < tm ? ns : tm; }
      const float t = __fsub_rn(nq, __fmul_rn(ns, ns));
      const float var = t > 0.0f ? t : 0.0f;
      const float nb = (float)__dmul_rn((double)0.9f, __dsqrt_rn(__dmul_rn((double)var, P.log_nf)));   // ComputeBounds
      smoothed[i] = ns; sq[i] = nq; tmp_min[i] = nt; est[i] = ne; bound[i] = nb;
      e = ne;
    }
    if (i == 0) { meta[0] = 1; meta[1] = (hops + 1) % P.hops_per_update; }
  }
  if (i == 0) {
    meta[2] = not_noise ? 1 : 0;
    if (is_noise_out) is_noise_out[slot] = not_noise ? 0 : 1;
  }
  if (estimate_out && i < nf) estimate_out[(size_t)slot * nf + i] = e;
}

}  // namespace lyra_b200
