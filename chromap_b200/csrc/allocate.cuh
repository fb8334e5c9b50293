// chromap_b200 — --allocate-multi-mappings on the device (cmx_allocate_multi_mappings_gpu).  Reference: AllocateMultiMappings
// (mapping_processor.h:319-440) between the in-memory dedup and the final sort (chromap.h:1322-1355 paired-end, :605-626
// single-end).  Same results as the host twin cmx_allocate_multi_mappings (std::mt19937 + std::discrete_distribution).
//
// The records arrive sorted and deduplicated (pp_device with the MAPQ filter at 0).  Then:
//   1. split: a record is multi if mapq < 4 (min_unique_mapping_mapq_, chromap.h:199), else uni; stable selects keep the order
//   2. weight of a multi record = #uni records on its sequence overlapping [qs, qe) = [start - d (clamped at 0), end + d) in
//      uint32 arithmetic: #{start < qe} - #{end <= qs} by binary search over the uni starts (sorted) and the uni ends (one radix
//      pass); when end + d wraps (qe <= qs) a scan of the uni records with qs - 65535 <= start < qe (only they can end past qs)
//   3. group by read: a stable radix sort of the multi records by read_id, run heads, per read the candidate count, the uint32
//      weight sum and whether it draws (>= 2 candidates and a non-zero sum), an exclusive scan of the draw flags
//   4. the generator: one CTA replays std::mt19937(seed) for 2 x draws outputs
//   5. the draw, one thread per read (al_draw); reads with sum 0 are dropped, a single candidate is kept without a draw
//   6. uni records + picked records are compacted; pp_device sorts them again and applies the MAPQ filter
// Bounds: n < 2^31 records per call; any number of candidates per read.
#pragma once
#include "device_common.cuh"
#include "pipeline_kernels.cuh"  // MT_N, mt_mix, mt_seed_fill
#include "postprocess.cuh"

#define AL_MIN_UNIQUE_MAPQ 4u  // chromap.h:199
#define AL_MAX_LEN 0xFFFFu     // a record's length is a uint16: its end lies at most this far past its start

// first index i in a[0, n) with a[i] >= key
__host__ __device__ __forceinline__ u32 al_lower_bound(const u64 *a, u32 n, u64 key) {
  u32 lo = 0, hi = n;
  while (lo < hi) {
    const u32 mid = lo + ((hi - lo) >> 1);
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// libstdc++ 13 std::discrete_distribution<uint32_t>(w, w + n)(mt19937) for n >= 2 and a non-zero sum, given the two generator
// outputs it consumes (random.tcc _M_initialize / operator()): probabilities w_i / sum with sum accumulated in double from
// 0.0, their partial sums with the last entry set to 1.0, p = generate_canonical<double, 53> = (g1 + g2 * 2^32) / 2^64
// (clamped below 1), the first index whose cumulative value is >= p.  Zero weights take part.  Division and addition are
// separate roundings on both sides (no contraction).
__host__ __device__ __forceinline__ u32 al_draw(const u32 *w, u32 n, u32 g1, u32 g2) {
#ifdef __CUDA_ARCH__
#define AL_ADD(a, b) __dadd_rn(a, b)
#define AL_DIV(a, b) __ddiv_rn(a, b)
#define AL_MUL(a, b) __dmul_rn(a, b)
#else
#define AL_ADD(a, b) ((a) + (b))
#define AL_DIV(a, b) ((a) / (b))
#define AL_MUL(a, b) ((a) * (b))
#endif
  double sum = 0.0;
  for (u32 i = 0; i < n; ++i) sum = AL_ADD(sum, (double)w[i]);
  double p = AL_DIV(AL_ADD((double)g1, AL_MUL((double)g2, 4294967296.0)), 18446744073709551616.0);
  if (p >= 1.0) p = 0x1.fffffffffffffp-1;  // nextafter(1, 0)
  double c = 0.0;
  for (u32 i = 0; i + 1 < n; ++i) {
    c = AL_ADD(c, AL_DIV((double)w[i], sum));
    if (c >= p) return i;
  }
  return n - 1;  // the last cumulative entry is 1.0 > p
#undef AL_ADD
#undef AL_DIV
#undef AL_MUL
}

// 1. per sorted record: uni / multi flags, start and end keys (rid << 32 | position)
__global__ void al_split_kernel(const PpRecord *recs, u64 n, u8 *uni, u8 *multi, u64 *key_start, u64 *key_end) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const PpRecord r = recs[i];
  const bool u = pe_mapq(r) >= AL_MIN_UNIQUE_MAPQ;
  uni[i] = u; multi[i] = !u;
  key_start[i] = ((u64)r.w[1] << 32) | r.w[2];
  key_end[i] = ((u64)r.w[1] << 32) | (r.w[2] + pe_len(r));
}

// 2. weight of multi record j (record midx[j]).  us: uni start keys (sorted), ue_s: uni end keys in start order, ue: uni end
// keys sorted.  rk[j] = its read_id, the key of the grouping sort.
__global__ void al_count_kernel(const PpRecord *recs, const u32 *midx, u32 m, const u64 *us, const u64 *ue_s, const u64 *ue, u32 n_uni, u32 d,
                                u32 *weight, u32 *rk) {
  const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const PpRecord r = recs[midx[j]];
  const u64 rid = (u64)r.w[1] << 32;
  const u32 start = r.w[2], end = start + pe_len(r);
  const u32 qs = start > d ? start - d : 0u, qe = end + d;  // mapping_processor.h:270-275
  const u32 lo = al_lower_bound(us, n_uni, rid), a = al_lower_bound(us, n_uni, rid | qe);  // [lo, a): uni on rid with start < qe
  u32 c = 0;
  if (qe > qs) {  // an end <= qs < qe has its start < qe too (a record's end does not wrap: it lies inside its sequence)
    const u32 b0 = al_lower_bound(ue, n_uni, rid), b = al_lower_bound(ue, n_uni, rid | (qs + 1u));  // qs < qe: qs + 1 does not wrap
    c = (a - lo) - (b - b0);
  } else {  // end + d wrapped (d close to 2^31): a uni record ends past qs only if it starts within AL_MAX_LEN of it
    const u32 i0 = max(lo, al_lower_bound(us, n_uni, rid | (qs > AL_MAX_LEN ? qs - AL_MAX_LEN : 0u)));
    for (u32 i = i0; i < a; ++i) c += (u32)ue_s[i] > qs;
  }
  weight[j] = c;
  rk[j] = r.w[0];
}

// 3. the reads: heads of the runs of equal read_id (sorted), weights in read order
__global__ void al_head_kernel(const u32 *rk_sorted, const u32 *perm, const u32 *weight, u32 m, u8 *head, u32 *w_sorted) {
  const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  head[i] = i == 0 || rk_sorted[i] != rk_sorted[i - 1];
  w_sorted[i] = weight[perm[i]];
}
// per read r (candidates w_sorted[rs[r], rs[r + 1])): whether it draws (two generator outputs) and whether it keeps a record
__global__ void al_read_kernel(const u32 *rs, u32 n_reads, u32 m, const u32 *w_sorted, u32 *draws, u8 *kept) {
  const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_reads) return;
  const u32 s = rs[r], e = r + 1 < n_reads ? rs[r + 1] : m;
  u32 sum = 0;
  for (u32 i = s; i < e; ++i) sum += w_sorted[i];  // uint32_t sum_weight (mapping_processor.h:374)
  draws[r] = sum != 0 && e - s >= 2;
  kept[r] = sum != 0;
}

// 4. std::mt19937 replayed by one CTA (>= 227 threads): the twist of mt_regen (pipeline_kernels.cuh) CTA-wide, one word per
// thread and phase; outputs [0, n_out) of the stream go to out
__global__ void __launch_bounds__(256) al_mt_kernel(const u32 *mt_init, u64 n_out, u32 *out) {
  __shared__ u32 mt[MT_N];
  const int t = threadIdx.x;
  for (int i = t; i < MT_N; i += blockDim.x) mt[i] = mt_init[i];
  __syncthreads();
  for (u64 base = 0; base < n_out; base += MT_N) {
    u32 v = 0;
    if (t < 227) v = mt_mix(mt[t], mt[t + 1], mt[t + 397]);
    __syncthreads();
    if (t < 227) mt[t] = v;
    __syncthreads();
    if (t < 227) v = mt_mix(mt[227 + t], mt[228 + t], mt[t]);
    __syncthreads();
    if (t < 227) mt[227 + t] = v;
    __syncthreads();
    if (t < 169) v = mt_mix(mt[454 + t], mt[455 + t], mt[227 + t]);
    __syncthreads();
    if (t < 169) mt[454 + t] = v;
    __syncthreads();
    if (t == 0) mt[623] = mt_mix(mt[623], mt[0], mt[396]);
    __syncthreads();
    for (int i = t; i < MT_N && base + (u64)i < n_out; i += blockDim.x) {
      u32 y = mt[i];
      y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
      out[base + (u64)i] = y;
    }
  }
}

// 5. the draw of read r: keep[] (over the sorted records, the uni flags already set) gains the picked candidate
__global__ void al_draw_kernel(const u32 *rs, u32 n_reads, u32 m, const u32 *w_sorted, const u32 *perm, const u32 *midx, const u32 *draws,
                               const u32 *draw_idx, const u8 *kept, const u32 *stream, u8 *keep) {
  const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_reads || !kept[r]) return;
  const u32 s = rs[r], e = r + 1 < n_reads ? rs[r + 1] : m;
  u32 pick = 0;
  if (draws[r]) {
    const u64 k = draw_idx[r];
    pick = al_draw(w_sorted + s, e - s, stream[2 * k], stream[2 * k + 1]);
  }
  keep[midx[perm[s + pick]]] = 1;
}

// the is_unique split of the allocated set (OutputMappingStatistics, mapping_processor.h:488-505)
__global__ void al_unique_count_kernel(const PpRecord *recs, u64 n, unsigned long long *n_unique) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const bool u = i < n && pe_uniq(recs[i]) == 1u;
  const unsigned b = __ballot_sync(0xffffffffu, u);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_unique, (unsigned long long)__popc(b));
}
