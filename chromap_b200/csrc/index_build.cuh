// chromap_b200 — device hash-table insertion and on-device index construction.
// Replaces Index::Construct (index.cc:12-89): collect reference minimizers, sort by (hash, hit), fold runs
// into {singleton: key|1 -> hit} / {multi: key -> occurrence offset<<32 | count} + occurrence table.
#pragma once
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "cuda_owners.cuh"
#include "device_common.cuh"

// Insert (key, val) pairs; keys are distinct.  slot = fib(hash) >> shift, linear probing, CAS on the key word.
__global__ void table_insert_kernel(const ulonglong2 *kv, size_t n, ulonglong2 *slots, u64 mask, int shift) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 key = kv[i].x, val = kv[i].y;
  u64 s = ((key >> 1) * 0x9E3779B97F4A7C15ull) >> shift;
  for (;;) {
    const u64 old = atomicCAS((unsigned long long *)&slots[s].x, (unsigned long long)CMX_EMPTY_KEY, (unsigned long long)key);
    if (old == CMX_EMPTY_KEY) { slots[s].y = val; return; }
    s = (s + 1) & mask;
  }
}

// khash arrays as the reference stores them (khash.h:165: 2 flag bits per bucket, 00 = occupied): count / insert the
// occupied buckets of [b0, b0 + n) without compacting them on the host first.
__global__ void khash_count_kernel(const u32 *flags, u64 n_buckets, unsigned long long *count) {
  const u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x;  // one flag word = 16 buckets
  const u64 nw = (n_buckets + 15) / 16;
  u32 c = 0;
  if (w < nw) {
    const u32 f = flags[w];
    for (u32 j = 0; j < 16; ++j) if (w * 16 + j < n_buckets && ((f >> (2 * j)) & 3u) == 0u) ++c;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}
__global__ void khash_insert_kernel(const u32 *flags, const u64 *keys, const u64 *vals, u64 b0, u64 n, ulonglong2 *slots, u64 mask, int shift) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 b = b0 + i;
  if (((flags[b >> 4] >> ((b & 0xfu) << 1)) & 3u) != 0u) return;
  const u64 key = keys[i], val = vals[i];
  u64 s = ((key >> 1) * 0x9E3779B97F4A7C15ull) >> shift;
  for (;;) {
    const u64 old = atomicCAS((unsigned long long *)&slots[s].x, (unsigned long long)CMX_EMPTY_KEY, (unsigned long long)key);
    if (old == CMX_EMPTY_KEY) { slots[s].y = val; return; }
    s = (s + 1) & mask;
  }
}

#define IB_CHUNK 2048  // reference bases per thread

// Minimizers of one chunk of one reference sequence (minimizer_generator.cc:7-139).  The emission state
// (ring of the last w seeds, rightmost-minimum, saturating run counter) is a function of the last
// w+k bases once a run is >= w+k long, so a thread warms up 2(w+k) bases before its chunk, scans w+1
// bases past it, and keeps only minimizers whose END position lies inside [c0, c1).
__global__ void ref_minimizers_kernel(const u8 *ref, const u64 *chunk_seq_off, const u32 *chunk_seq_len, const u32 *chunk_rid,
                                      const u32 *chunk_start, size_t n_chunks, int k, int w, u64 *out_hash, u64 *out_hit,
                                      unsigned long long *out_count, u64 cap) {
  const size_t ci = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (ci >= n_chunks) return;
  const u8 *seq = ref + chunk_seq_off[ci];
  const u32 len = chunk_seq_len[ci], rid = chunk_rid[ci];
  const u32 c0 = chunk_start[ci];
  const u32 c1 = (c0 + IB_CHUNK < len) ? c0 + IB_CHUNK : len;
  const u32 warm = 2u * (u32)(w + k);
  const u32 s0 = c0 > warm ? c0 - warm : 0u;
  const u32 s1 = (c1 + (u32)w + 1u < len) ? c1 + (u32)w + 1u : len;
  const u64 shift = 2 * (k - 1);
  const u64 mask = (((u64)1) << (2 * k)) - 1;
  u64 fwd = 0, rev = 0;
  u64 ring_h[CMX_W_MAX];
  u32 ring_p[CMX_W_MAX];
  for (int i = 0; i < w; ++i) { ring_h[i] = ~0ull; ring_p[i] = ~0u; }
  u64 best_h = ~0ull;
  u32 best_p = ~0u;
  int run = 0, slot = 0, best_slot = 0;
  // local staging to cut atomics: up to 64 entries then flush
  u64 lh[32];
  u32 lp[32];
  int ln = 0;
  auto flush = [&]() {
    if (!ln) return;
    const u64 base = atomicAdd(out_count, (unsigned long long)ln);
    for (int i = 0; i < ln; ++i)
      if (base + i < cap) { out_hash[base + i] = lh[i]; out_hit[base + i] = ((((u64)rid) << 32 | (lp[i] >> 1)) << 1) | (lp[i] & 1u); }
    ln = 0;
  };
#define EMIT(h, p) do { const u32 pp_ = (p) >> 1; if (pp_ >= c0 && pp_ < c1) { lh[ln] = (h); lp[ln] = (p); if (++ln == 32) flush(); } } while (0)
  for (u32 pos = s0; pos < s1; ++pos) {
    const u32 b = base_code(seq[pos]);
    u64 cur_h = ~0ull;
    u32 cur_p = ~0u;
    if (b < 4) {
      fwd = ((fwd << 2) | b) & mask;
      rev = (rev >> 2) | (((u64)(3 ^ b)) << shift);
      if (fwd == rev) continue;
      const u64 hf = mix64(fwd, mask), hr = mix64(rev, mask);
      const u32 strand = hf < hr ? 0u : 1u;
      ++run;
      if (run >= k) { cur_h = mix64(strand ? hr : hf, mask); cur_p = (pos << 1) | strand; }
    } else {
      run = 0;
    }
    ring_h[slot] = cur_h; ring_p[slot] = cur_p;
    if (run == w + k - 1 && best_h != ~0ull && best_h < cur_h) {
      for (int j = slot + 1; j < w; ++j) if (best_h == ring_h[j] && ring_p[j] != best_p) EMIT(ring_h[j], ring_p[j]);
      for (int j = 0; j < slot; ++j) if (best_h == ring_h[j] && ring_p[j] != best_p) EMIT(ring_h[j], ring_p[j]);
    }
    if (cur_h <= best_h) {
      if (run >= w + k && best_h != ~0ull) EMIT(best_h, best_p);
      best_h = cur_h; best_p = cur_p; best_slot = slot;
    } else if (slot == best_slot) {
      if (run >= w + k - 1 && best_h != ~0ull) EMIT(best_h, best_p);
      best_h = ~0ull;
      for (int j = slot + 1; j < w; ++j) if (best_h >= ring_h[j]) { best_h = ring_h[j]; best_p = ring_p[j]; best_slot = j; }
      for (int j = 0; j <= slot; ++j) if (best_h >= ring_h[j]) { best_h = ring_h[j]; best_p = ring_p[j]; best_slot = j; }
      if (run >= w + k - 1 && best_h != ~0ull) {
        for (int j = slot + 1; j < w; ++j) if (best_h == ring_h[j] && best_p != ring_p[j]) EMIT(ring_h[j], ring_p[j]);
        for (int j = 0; j <= slot; ++j) if (best_h == ring_h[j] && best_p != ring_p[j]) EMIT(ring_h[j], ring_p[j]);
      }
    }
    if (++slot == w) slot = 0;
  }
  if (s1 == len && best_h != ~0ull) EMIT(best_h, best_p);  // final flush only at the true sequence end
#undef EMIT
  flush();
}

// after sorting by (hash, hit): flags[i] = 1 if element i belongs to a run of length > 1
__global__ void multi_flag_kernel(const u64 *hash, size_t n, u32 *multi, unsigned long long *n_heads) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 h = hash[i];
  const bool eq_prev = i > 0 && hash[i - 1] == h, eq_next = i + 1 < n && hash[i + 1] == h;
  multi[i] = (eq_prev || eq_next) ? 1u : 0u;
  if (!eq_prev) atomicAdd(n_heads, 1ull);
}

__global__ void fold_runs_kernel(const u64 *hash, const u64 *hit, const u32 *multi, const u32 *occ_idx, size_t n, u64 *occ,
                                 ulonglong2 *slots, u64 mask, int shift) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 h = hash[i];
  if (multi[i]) occ[occ_idx[i]] = hit[i];
  if (i > 0 && hash[i - 1] == h) return;  // not a run head
  u64 key, val;
  if (!multi[i]) { key = (h << 1) | 1ull; val = hit[i]; }
  else {
    size_t lo = i + 1, hi = n;  // upper bound of the run
    while (lo < hi) { const size_t mid = (lo + hi) / 2; if (hash[mid] == h) lo = mid + 1; else hi = mid; }
    key = h << 1;
    val = ((u64)occ_idx[i] << 32) | (u64)(u32)(lo - i);
  }
  u64 s = (h * 0x9E3779B97F4A7C15ull) >> shift;
  for (;;) {
    const u64 old = atomicCAS((unsigned long long *)&slots[s].x, (unsigned long long)CMX_EMPTY_KEY, (unsigned long long)key);
    if (old == CMX_EMPTY_KEY) { slots[s].y = val; return; }
    s = (s + 1) & mask;
  }
}

#ifndef CMX_HOST_EMU  // (CUDA host code: the host emulation of a CTA runs the kernels above in this sequence itself)

struct IndexBuildResult {
  DevMem<ulonglong2> slots;
  u64 n_slots = 0;
  DevMem<u64> occ;
  u32 n_occ = 0;
  u64 n_keys = 0;
  u64 n_minimizers = 0;
};

// CMX_OK, or CMX_ERR_CUDA with the reason in err
static int build_index_on_device(const u8 *d_ref, const std::vector<u64> &off, const std::vector<u32> &len, int k, int w,
                                 IndexBuildResult &res, std::string &err) {
  u64 total = 0;
  std::vector<u64> c_off;
  std::vector<u32> c_len, c_rid, c_start;
  for (size_t r = 0; r < off.size(); ++r) {
    total += len[r];
    for (u64 s = 0; s < len[r]; s += IB_CHUNK) { c_off.push_back(off[r]); c_len.push_back(len[r]); c_rid.push_back((u32)r); c_start.push_back((u32)s); }
  }
  const size_t n_chunks = c_off.size();
  // minimizer density is about 2 / (w + 1) per base: 1/4 for w = 7; the buffer follows w (with 30 % slack) so that small windows fit
  const u64 cap = (u64)((double)total * std::min(1.0, 2.6 / (double)(w + 1))) + 1024 * off.size() + 4096;
  DevMem<u64> d_coff, h1, t1, h2, t2, d_occ;
  DevMem<u32> d_clen, d_crid, d_cstart, d_multi, d_occidx;
  DevMem<unsigned long long> d_cnt;
  DevMem<> d_tmp;
  DevMem<ulonglong2> d_slots;
  size_t tmp_bytes = 0, tb2 = 0;
  unsigned long long h_cnt[2] = {0, 0};
  u64 n = 0, n_keys = 0, n_slots = 1024;
  u32 n_occ = 0, last_idx = 0, last_multi = 0;
  int shift = 0;
  int hash_bits = 2 * k;
  CUE(d_coff.alloc(n_chunks * 8)); CUE(d_clen.alloc(n_chunks * 4)); CUE(d_crid.alloc(n_chunks * 4)); CUE(d_cstart.alloc(n_chunks * 4));
  CUE(cudaMemcpy(d_coff, c_off.data(), n_chunks * 8, cudaMemcpyHostToDevice)); CUE(cudaMemcpy(d_clen, c_len.data(), n_chunks * 4, cudaMemcpyHostToDevice));
  CUE(cudaMemcpy(d_crid, c_rid.data(), n_chunks * 4, cudaMemcpyHostToDevice)); CUE(cudaMemcpy(d_cstart, c_start.data(), n_chunks * 4, cudaMemcpyHostToDevice));
  CUE(h1.alloc(cap * 8)); CUE(t1.alloc(cap * 8));
  CUE(d_cnt.alloc(16)); CUE(cudaMemset(d_cnt, 0, 16));
  ref_minimizers_kernel<<<(unsigned)((n_chunks + 127) / 128), 128>>>(d_ref, d_coff, d_clen, d_crid, d_cstart, n_chunks, k, w, h1, t1, d_cnt, cap);
  CUE(cudaGetLastError());
  CUE(cudaMemcpy(h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost));
  n = h_cnt[0];
  if (n > cap) { err = "minimizer buffer too small"; return CMX_ERR_CUDA; }
  if (n == 0) { err = "reference has no minimizers"; return CMX_ERR_CUDA; }
  if (n > 0x7fffffffull) { err = "more than INT_MAX minimizers (index.cc:33)"; return CMX_ERR_CUDA; }
  // sort by (hash, hit): stable LSD — by hit first, then by hash
  CUE(h2.alloc(n * 8)); CUE(t2.alloc(n * 8));
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, t1.p, t2.p, h1.p, h2.p, (int)n, 0, 64);
  cub::DeviceRadixSort::SortPairs(nullptr, tb2, h2.p, h1.p, t2.p, t1.p, (int)n, 0, hash_bits);
  if (tb2 > tmp_bytes) tmp_bytes = tb2;
  CUE(d_tmp.alloc(tmp_bytes + 16));
  CUE(cub::DeviceRadixSort::SortPairs(d_tmp.p, tmp_bytes, t1.p, t2.p, h1.p, h2.p, (int)n, 0, 64));          // keys = hit, values = hash
  CUE(cub::DeviceRadixSort::SortPairs(d_tmp.p, tmp_bytes, h2.p, h1.p, t2.p, t1.p, (int)n, 0, hash_bits));   // keys = hash, values = hit (stable)
  h2.reset(); t2.reset();
  // runs
  CUE(d_multi.alloc(n * 4)); CUE(d_occidx.alloc(n * 4));
  CUE(cudaMemset(d_cnt, 0, 16));
  multi_flag_kernel<<<(unsigned)((n + 255) / 256), 256>>>(h1, n, d_multi, d_cnt);
  CUE(cudaGetLastError());
  CUE(cudaMemcpy(h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost));
  n_keys = h_cnt[0];
  cub::DeviceScan::ExclusiveSum(nullptr, tb2, d_multi.p, d_occidx.p, (int)n);
  if (tb2 > tmp_bytes) { tmp_bytes = tb2; CUE(d_tmp.alloc(tmp_bytes + 16)); }  // (alloc frees the smaller buffer first)
  CUE(cub::DeviceScan::ExclusiveSum(d_tmp.p, tmp_bytes, d_multi.p, d_occidx.p, (int)n));
  CUE(cudaMemcpy(&last_idx, d_occidx + (n - 1), 4, cudaMemcpyDeviceToHost));
  CUE(cudaMemcpy(&last_multi, d_multi + (n - 1), 4, cudaMemcpyDeviceToHost));
  // the sort's scratch (about the size of the keys) goes before the table is allocated: at 3 Gbp both do not fit 80 GB at once
  d_tmp.reset();
  n_occ = last_idx + last_multi;
  CUE(d_occ.alloc((size_t)(n_occ ? n_occ : 1) * 8));
  while (n_slots < 2 * n_keys) n_slots <<= 1;
  CUE(d_slots.alloc(n_slots * sizeof(ulonglong2)));
  CUE(cudaMemset(d_slots, 0xFF, n_slots * sizeof(ulonglong2)));
  while ((1ull << shift) < n_slots) ++shift;
  shift = 64 - shift;
  fold_runs_kernel<<<(unsigned)((n + 255) / 256), 256>>>(h1, t1, d_multi, d_occidx, n, d_occ, d_slots, n_slots - 1, shift);
  CUE(cudaGetLastError());
  CUE(cudaDeviceSynchronize());
  res.slots = std::move(d_slots); res.n_slots = n_slots; res.occ = std::move(d_occ); res.n_occ = n_occ; res.n_keys = n_keys; res.n_minimizers = n;
  return CMX_OK;
}
#endif
