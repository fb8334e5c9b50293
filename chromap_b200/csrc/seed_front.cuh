// chromap_b200 — tier-0 front end: one kernel from read bytes to probed minimizer records.
//   * read tiles are staged into shared memory by the copy engine (cp.async.bulk + mbarrier, double buffered) —
//     the "TMA staging of read batches" of the design; the bulk copies are 16-byte aligned, the < 16 byte head and tail
//     of a tile go through ordinary loads, so nothing outside the caller's buffers is ever touched;
//   * length filter (chromap.h:911-916), minimizers (minimizer_generator.cc:7-139) and the index probe
//     (khash.h:232-245 semantics, index.cc:237-349) run back to back on the same thread, the probes of a read issued
//     eight at a time: the random HBM reads of one warp hide behind the hashing of the others, and the hashes never
//     travel through HBM;
//   * records {table value, position | strand | kind} are written lane-interleaved (32 pairs per group), i.e. coalesced
//     here and in every kernel that reads them.
// File:line citations are into the reference's src/.
#pragma once
#include "pipeline_kernels.cuh"

// ---- mbarrier + bulk copy (PTX ISA 8.x, sm_90+) ---------------------------------------------------------------------
#ifndef CMX_HOST_EMU  // (the host emulation of a CTA supplies an mbarrier word and a copy that signals its bytes)
__device__ __forceinline__ u32 smem_u32(const void *p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64 *bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(u64 *bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(u64 *bar, u32 parity) {
  u32 ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// global -> shared bulk copy by the copy engine; completion is counted in bytes on `bar`.  16-byte aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, u32 bytes, u64 *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
#endif

// ---- the kernel ------------------------------------------------------------------------------------------------------
#define SF_TILE 64   // pairs per tile
#define SF_NT 128    // threads: warps 0-1 take mate 1 of the tile's pairs, warps 2-3 mate 2
#define SF_PROBE_BATCH 4
#define SF_KEY_ROWS 16  // minimizers per read buffered in shared memory between the scan and the probe
struct FrontShared {
  u64 bar[2];
  u32 acc[3];
};
// dynamic shared memory: 2 stages x 2 mates x tile_bytes (tile_bytes = SF_TILE * maxmm + 32, a multiple of 16), then the key
// buffer [SF_KEY_ROWS][SF_NT] u64 (one column per thread: conflict-free).  100-base reads: 41.3 KB, five CTAs per SM.
__host__ __device__ inline size_t seed_front_tile_bytes(int maxmm) { return ((size_t)SF_TILE * maxmm + 32 + 15) / 16 * 16; }
__host__ __device__ inline size_t seed_front_smem_bytes(int maxmm) { return 4 * seed_front_tile_bytes(maxmm) + (size_t)SF_KEY_ROWS * SF_NT * 8; }

// prepped = 1: prep_kernel ran before (adapter trimming): lengths and pair status are taken from the scratch.
// Pairs [slot_begin, slot_end) of the tier (a call whose reads arrive in pieces launches one grid per piece).
// FAST: k = 17, w = 7 (every preset): the packed-key scan only; otherwise the run-time scan only — one kernel per case keeps
// the other's registers and code out of the way.
template <bool FAST>
__global__ void __launch_bounds__(SF_NT, 5) seed_front_kernel(DevParams P, DevIndex ix, DevBatch B, Scratch S, Counters *ctr, int prepped, int slot_begin,
                                                           int slot_end) {
  extern __shared__ __align__(16) u8 sf_smem[];
  __shared__ FrontShared fs;
  const int tid = threadIdx.x;
  const int maxmm = S.caps.maxmm;
  const size_t tb = seed_front_tile_bytes(maxmm);
  u64 *kbuf = (u64 *)(sf_smem + 4 * tb);
  const int n_tiles = (slot_end - slot_begin + SF_TILE - 1) / SF_TILE;
  if (tid == 0) { mbar_init(&fs.bar[0], 1); mbar_init(&fs.bar[1], 1); mbar_fence_init(); }
  if (tid < 3) fs.acc[tid] = 0;
  __syncthreads();
  // stage a tile: buffer byte x of mate m mirrors global byte (g0 & ~15) + x, g0 = start of the tile's first read
  auto issue = [&](int tile, int stage) {
    const int p0 = slot_begin + tile * SF_TILE, p1 = min(slot_end, p0 + SF_TILE);
    // (tier 0 always runs on the identity pair list)
    u32 total = 0;
    u64 src[2];
    u32 dst_off[2], bytes[2];
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      bytes[m] = 0;
      if (m == 1 && P.se) continue;
      const u32 *off = m == 0 ? B.off1 : B.off2;
      const u8 *seq = m == 0 ? B.seq1 : B.seq2;
      const u64 g0 = (u64)(seq + off[p0]), g1 = (u64)(seq + off[p1]);
      const u64 base = g0 & ~15ull, a0 = (g0 + 15) & ~15ull, a1 = g1 & ~15ull;
      if (g1 - base > tb) continue;  // a read longer than the tier allows: this tile is read from global memory
      u8 *buf = sf_smem + (size_t)(stage * 2 + m) * tb;
      if (a1 > a0) { src[m] = a0; dst_off[m] = (u32)(a0 - base); bytes[m] = (u32)(a1 - a0); total += bytes[m]; }
      // head and tail (< 16 bytes each) by ordinary loads
      const u64 h1 = min(a0, g1), t0 = max(a1, h1);
      for (u64 x = g0 + tid; x < h1; x += SF_NT) buf[x - base] = *(const u8 *)x;
      for (u64 x = t0 + tid; x < g1; x += SF_NT) buf[x - base] = *(const u8 *)x;
    }
    if (tid == 0) {
      mbar_arrive_expect_tx(&fs.bar[stage], total);
#pragma unroll
      for (int m = 0; m < 2; ++m)
        if (bytes[m]) bulk_g2s(sf_smem + (size_t)(stage * 2 + m) * tb + dst_off[m], (const void *)src[m], bytes[m], &fs.bar[stage]);
    }
  };
  u32 phase[2] = {0u, 0u};
  u32 steps_total = 0, found = 0, n_mine = 0;
  if ((int)blockIdx.x < n_tiles) issue(blockIdx.x, 0);
  int it = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int st = it & 1;
    if (tile + (int)gridDim.x < n_tiles) issue(tile + gridDim.x, st ^ 1);
    while (!mbar_try_wait(&fs.bar[st], phase[st])) {}
    phase[st] ^= 1u;
    __syncthreads();  // head / tail bytes of this stage
    const int p0 = slot_begin + tile * SF_TILE;
    const int mate = tid >> 6, slot = p0 + (tid & 63);
    const bool live = slot < slot_end && !(P.se && mate == 1);
    int status = ST_OK, len = 0;
    const u8 *rd = sf_smem;  // always shared memory
    bool staged = false;
    if (slot < slot_end) {
      // lengths of both mates (length filter / tier check need them), this thread's read
      const u32 o1a = B.off1[slot], o1b = B.off1[slot + 1];
      const u32 o2a = P.se ? 0u : B.off2[slot], o2b = P.se ? 0u : B.off2[slot + 1];
      int len1 = (int)(o1b - o1a), len2 = (int)(o2b - o2a);
      if (prepped) {
        status = S.pmeta[slot].status;
        len1 = S.rmeta[2 * slot].len; len2 = S.rmeta[2 * slot + 1].len;
      } else {
        if (B.bc_ok && !B.bc_ok[slot]) status = ST_DROP;  // chromap.h:908-909
        else if (len1 < P.min_read_len || (!P.se && len2 < P.min_read_len)) status = ST_DROP;  // chromap.h:911-916, single-end :411-414
        else if (len1 > maxmm || len2 > maxmm) status = ST_OVERFLOW;  // longer than max_read_length: next tier
      }
      len = mate == 0 ? len1 : len2;
      const u32 *off = mate == 0 ? B.off1 : B.off2;
      const u8 *seq = mate == 0 ? B.seq1 : B.seq2;
      if (live) {
        const u64 g0 = (u64)(seq + off[p0]), g1 = (u64)(seq + off[min(slot_end, p0 + SF_TILE)]);
        const u64 base = g0 & ~15ull;
        staged = g1 - base <= tb;
        const u32 mine = mate == 0 ? o1a : o2a;
        u8 *buf = sf_smem + (size_t)(st * 2 + mate) * tb;
        if (staged) rd = buf + ((u64)(seq + mine) - base);
        else {  // a tile that holds a read longer than the tier allows was not staged: this thread copies its own read (clipped)
          u8 *dst = buf + (size_t)(tid & 63) * maxmm;
          for (int i = 0; i < min(len, maxmm); ++i) dst[i] = seq[mine + i];
          rd = dst;
        }
      }
      if (!prepped && mate == 0) {
        PairMeta pm;
        pm.status = status; pm.sup = 0; pm.min_sum = 0; pm.second_min_sum = 0; pm.n_best = 0; pm.n_second_best = 0; pm.n_rec = 0; pm.pad = 0;
        S.pmeta[slot] = pm;
      }
    }
    __syncthreads();  // pair status written before a mate may raise it to ST_OVERFLOW below
    int n_mm = 0;
    if (live && status == ST_OK) {
      const size_t mb = mm_base(S, slot, mate);
      u64 *mmv = S.mm_val + mb;
      u32 *mmp = S.mm_pos + mb;
      // minimizers as {hash, position | strand}: the first SF_KEY_ROWS of a read wait for their probe in shared memory
      // (column `tid` of kbuf), later ones — long reads only — are parked in the record arrays themselves
      u64 *kcol = kbuf + tid;
      const int key_rows = P.k <= 22 ? SF_KEY_ROWS : 0;  // hash << 20 | position must fit 64 bits
      auto emit = [&](u64 h, u32 p) {
        if (n_mm < key_rows) kcol[n_mm * SF_NT] = (h << 20) | p;  // p < 2^20 (reads are far shorter than 2^19), h < 2^44
        else if (n_mm < maxmm) { mmv[(size_t)n_mm * 32] = h; mmp[(size_t)n_mm * 32] = p; }
        ++n_mm;
      };
      if constexpr (FAST) minimizer_scan_packed<17, 7>([&](int i) { return rd[i]; }, len, emit);  // window in registers
      else minimizer_scan<0, 0>([&](int i) { return rd[i]; }, len, P.k, P.w, emit);
      if (n_mm > maxmm) { S.pmeta[slot].status = ST_OVERFLOW; atomicAdd(&ctr->ovf_reason[1], 1ull); }
      else {
        // probes, eight at a time: the first slots of eight chains are in flight together (one 16-byte load each; the
        // rare second step of a chain is issued when the first has come back).  One write per record, no read-back.
        for (int i0 = 0; i0 < n_mm; i0 += SF_PROBE_BATCH) {
          u64 h[SF_PROBE_BATCH], s[SF_PROBE_BATCH];
          u32 pw[SF_PROBE_BATCH];
          ulonglong2 kv[SF_PROBE_BATCH];
#pragma unroll
          for (int q = 0; q < SF_PROBE_BATCH; ++q)
            if (i0 + q < n_mm) {
              const int i = i0 + q;
              if (i < key_rows) { const u64 key = kcol[i * SF_NT]; h[q] = key >> 20; pw[q] = (u32)key & 0xFFFFFu; }
              else { h[q] = mmv[(size_t)i * 32]; pw[q] = mmp[(size_t)i * 32]; }
              s[q] = (h[q] * 0x9E3779B97F4A7C15ull) >> ix.shift;
              kv[q] = __ldg(&ix.slots[s[q]]);
            }
#pragma unroll
          for (int q = 0; q < SF_PROBE_BATCH; ++q)
            if (i0 + q < n_mm) {
              u64 val = 0;
              u32 kind = 0;
              ulonglong2 c = kv[q];
              u64 sl = s[q];
              for (;;) {
                ++steps_total;
                if (c.x == CMX_EMPTY_KEY) break;
                if ((c.x >> 1) == h[q]) { val = c.y; kind = (c.x & 1) ? 1u : 2u; break; }
                sl = (sl + 1) & ix.n_slots_mask;
                c = __ldg(&ix.slots[sl]);
              }
              mmv[(size_t)(i0 + q) * 32] = val;
              mmp[(size_t)(i0 + q) * 32] = pw[q] | (kind << 30);
              found += kind != 0;
            }
        }
        n_mine += (u32)n_mm;
      }
    }
    const int mm_done = (live && status == ST_OK && n_mm <= maxmm) ? 1 : 0;
    if (slot < slot_end && !prepped) {
      ReadMeta z;
      memset(&z, 0, sizeof(z));
      z.len = len; z.n_mm = n_mm; z.mm_done = mm_done;
      S.rmeta[2 * slot + mate] = z;
    } else if (live && status == ST_OK) {
      S.rmeta[2 * slot + mate].n_mm = n_mm;
      S.rmeta[2 * slot + mate].mm_done = mm_done;
    }
    __syncthreads();  // everyone is done with this stage before it is refilled
  }
  const u32 a = __reduce_add_sync(0xffffffffu, n_mine), b2 = __reduce_add_sync(0xffffffffu, steps_total), f = __reduce_add_sync(0xffffffffu, found);
  if ((tid & 31) == 0) { atomicAdd(&fs.acc[0], a); atomicAdd(&fs.acc[1], b2); atomicAdd(&fs.acc[2], f); }
  __syncthreads();
  if (tid == 0) { atomicAdd(&ctr->n_minimizers, (u64)fs.acc[0]); atomicAdd(&ctr->n_probe_steps, (u64)fs.acc[1]); atomicAdd(&ctr->n_found, (u64)fs.acc[2]); }
}
