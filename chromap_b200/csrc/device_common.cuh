// chromap_b200 — shared device types and helpers.  sm_90a only.
// File:line citations are into the reference's src/ (what each routine must reproduce bit-exactly).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

typedef unsigned long long u64;
typedef unsigned int u32;
typedef unsigned char u8;

#define CMX_W_MAX 64       // ring size bound for the minimizer window
#define CMX_MAX_BEST 8     // upper bound on max_num_best_mappings (-n)

// Parameters the kernels read (subset of cmx_params + index k/w).
struct DevParams {
  int e, min_seeds, f0, f1, max_best, max_insert, min_read_len, drop_rep, trim, k, w, lanes, split;
  int se;  // single-end: a slot holds one read (mate 0), mate 1 stays empty
};

struct Caps {  // per-read (per-strand where applicable) scratch capacities of one tier
  int maxmm, hc, cc, mc;
};

// pair status
enum { ST_OK = 0, ST_DROP = 1, ST_OVERFLOW = 2 };

struct ReadMeta {  // 64 bytes = two 32-byte sectors: what seeding / candidate pairing touch in the first, verification / pairing / emit in the second
  int len;  // after adapter trimming
  int n_mm;
  int n_cand[2];
  int n_cand_gen[2];
  u32 rep_len;
  int mm_done;  // 1: the front end left this read's probed minimizer records in the tier's scratch
  int n_map[2];
  int min_err, second_min_err, n_best, n_second_best;
  int n_aug[2];
};
static_assert(sizeof(ReadMeta) == 64, "ReadMeta: two sectors");

struct PairMeta {
  int status;
  int sup;  // SupplementCandidates result
  int min_sum, second_min_sum, n_best, n_second_best;
  int n_rec;
  int pad;
};

// Device index: open-addressing table of 16-byte slots {key = hash<<1|singleton, val}, linear probing,
// slot = fibonacci(hash) >> shift.  Layout is ours; lookups answer exactly like kh_get on the
// reference's khash (khash.h:232-245): found / key / value.
struct DevIndex {
  const ulonglong2 *slots;
  u64 n_slots_mask;  // n_slots - 1 (power of two)
  int shift;         // 64 - log2(n_slots)
  const u64 *occ;
  u32 n_occ;
  int k, w;
};
#define CMX_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

struct DevRef {
  const u8 *seq;     // concatenated ASCII, each sequence followed by >= 64 NUL bytes
  const u64 *off;    // [n_seq]
  const u32 *len;    // [n_seq]
  u32 n_seq;
};

// Where cmx_upload_reference puts n_seq sequences (lengths offsets[i + 1] - offsets[i]) in DevRef::seq: REF_PAD NUL bytes,
// then every sequence at a 64-byte aligned offset off[i] and followed by at least REF_PAD NUL bytes.  The aligners read up
// to e bytes past a sequence's end (BandedTraceback, the split aligner's drop-off): the padding is what they find there.
// Returns the size of the whole layout.
#define REF_PAD 64
inline u64 ref_layout(u32 n_seq, const u64 *offsets, u64 *off) {
  u64 cur = REF_PAD;
  for (u32 i = 0; i < n_seq; ++i) {
    off[i] = cur;
    cur = (cur + (offsets[i + 1] - offsets[i]) + REF_PAD + 63) / 64 * 64;
  }
  return cur + REF_PAD;
}

struct DevBatch {
  const u8 *seq1;
  const u32 *off1;
  const u8 *seq2;
  const u32 *off2;
  u32 n_pairs;
  u32 first_read_id;
  const u8 *bc_ok;  // scATAC: 0 = barcode not in the whitelist -> the pair is not mapped (nullptr for bulk data)
};

// One scratch tier: arrays indexed by slot (pair slot s -> read slots 2s, 2s+1).
struct Scratch {
  Caps caps;
  int n_slots;
  const int *pair_list;  // slot -> pair index in batch (nullptr = identity)
  int mm_il;             // 1: the per-read arrays mm_val .. map_split, hits excepted, lane-interleaved in groups of 32 pairs (tier 0), see il_read
  ReadMeta *rmeta;       // [2*n_slots]
  PairMeta *pmeta;       // [n_slots]
  u64 *mm_hash;          // [2n][maxmm]   (overflow tiers only)
  u64 *mm_val;           // [2n][maxmm]   lookup value
  u32 *mm_pos;           // [2n][maxmm]   (pos<<1|strand) | kind<<30   kind: 0 absent 1 singleton 2 multi
  u64 *hits;             // [2n][2][hc]   (never interleaved)
  u64 *cand_pos;         // [2n][3][2][cc]   set 0 = candidates, 1 = buffer, 2 = augment
  u8 *cand_cnt;          // same shape
  u64 *map_pos;          // [2n][2][mc]
  short *map_err;        // [2n][2][mc]   (under --split-alignment: -(matched length))
  int *map_split;        // [2n][2][mc]   split_sites word (draft_mapping_generator.cc:550-554)
};

// Layout of one tier's scratch for `slots` pair slots, its arrays in the order of Scratch's pointers (rmeta .. map_split):
// size[i] = bytes of array i, off[i] = its offset in one allocation where every array starts on a 256-byte boundary.
// Returns the size of that allocation.
#define SCRATCH_ARRAYS 11
inline size_t scratch_layout(const Caps &c, size_t slots, bool interleaved, size_t *off, size_t *size = nullptr) {
  const size_t R = 2 * slots;
  const size_t Ri = interleaved ? 2 * ((slots + 31) / 32 * 32) : R;  // interleaved arrays: whole groups of 32 pairs
  const size_t sz[SCRATCH_ARRAYS] = {R * sizeof(ReadMeta), slots * sizeof(PairMeta),
                                     interleaved ? 0 : R * c.maxmm * 8,  // hashes: tier 0 never stores them
                                     Ri * c.maxmm * 8, Ri * c.maxmm * 4, R * 2 * (size_t)c.hc * 8, Ri * 6 * (size_t)c.cc * 8, Ri * 6 * (size_t)c.cc,
                                     Ri * 2 * (size_t)c.mc * 8, Ri * 2 * (size_t)c.mc * 2, Ri * 2 * (size_t)c.mc * 4};
  size_t end = 0;
  for (int i = 0; i < SCRATCH_ARRAYS; ++i) {
    off[i] = end;
    if (size) size[i] = sz[i];
    end = (end + sz[i] + 255) / 256 * 256;
  }
  return end;
}
// Points S's arrays at a[0 .. SCRATCH_ARRAYS), in scratch_layout's order.
inline void scratch_bind(Scratch &S, char *const *a) {
  S.rmeta = (ReadMeta *)a[0]; S.pmeta = (PairMeta *)a[1];
  S.mm_hash = (u64 *)a[2]; S.mm_val = (u64 *)a[3]; S.mm_pos = (u32 *)a[4];
  S.hits = (u64 *)a[5]; S.cand_pos = (u64 *)a[6]; S.cand_cnt = (u8 *)a[7];
  S.map_pos = (u64 *)a[8]; S.map_err = (short *)a[9]; S.map_split = (int *)a[10];
}

// a[i] view of every `stride`-th element starting at base: a per-thread column of an interleaved shared-memory tile (a
// negative stride walks it backwards) or one list of a tier's per-read arrays (below).
template <typename T>
struct Strided {
  T *base;
  int stride;
  __device__ __forceinline__ T &operator[](int i) const { return base[i * stride]; }
};

// ---- where the lists of read sr = 2 * slot + mate lie in its tier's scratch: minimizer records [maxmm], candidates
// [3 sets][2 strands][cc], draft mappings [2 strands][mc].
// il = 1 (tier 0, S.mm_il): lane-interleaved in groups of 32 pairs.  Row `row` of the read's rows lies at
// (((slot >> 5) * 2 + mate) * rows + row) * 32 + (slot & 31), one row per element (stride 32): the lanes of a warp hold
// consecutive slots, so their element i is one contiguous segment instead of one sector per lane.  il = 0 (overflow tiers,
// one CTA per read or pair): [read][rows], stride 1.  The kernels that run in every tier take il from S.mm_il; the CTA-only
// kernels pass 0 and keep plain pointers.
// il_read: the read's row block (its group's mate block when interleaved); il_place: where that row block's element e lies.
__device__ __forceinline__ size_t il_read(int il, int sr) { return il ? (size_t)((sr >> 6) * 2 + (sr & 1)) : (size_t)sr; }
__device__ __forceinline__ size_t il_place(int il, int sr, size_t e) { return il ? e * 32 + ((sr >> 1) & 31) : e; }
__device__ __forceinline__ int il_stride(int il) { return il ? 32 : 1; }
__device__ __forceinline__ size_t mm_base(const Scratch &S, int slot, int mate) {  // == il_place(il, sr, il_read(il, sr) * maxmm)
  return S.mm_il ? ((size_t)((slot >> 5) * 2 + mate) * S.caps.maxmm) * 32 + (slot & 31) : (size_t)(2 * slot + mate) * S.caps.maxmm;
}
__device__ __forceinline__ int mm_stride(const Scratch &S) { return il_stride(S.mm_il); }
__device__ __forceinline__ size_t cand_base(int il, const Caps &c, int sr, int set, int strand) {
  return il_place(il, sr, ((il_read(il, sr) * 3 + set) * 2 + strand) * c.cc);
}
__device__ __forceinline__ size_t map_base(int il, const Caps &c, int sr, int strand) {
  return il_place(il, sr, (il_read(il, sr) * 2 + strand) * c.mc);
}
// the same lists as views in S's own layout
__device__ __forceinline__ Strided<u64> cand_pos_of(const Scratch &S, int sr, int set, int strand) {
  return {S.cand_pos + cand_base(S.mm_il, S.caps, sr, set, strand), il_stride(S.mm_il)};
}
__device__ __forceinline__ Strided<u8> cand_cnt_of(const Scratch &S, int sr, int set, int strand) {
  return {S.cand_cnt + cand_base(S.mm_il, S.caps, sr, set, strand), il_stride(S.mm_il)};
}
__device__ __forceinline__ Strided<u64> map_pos_of(const Scratch &S, int sr, int strand) {
  return {S.map_pos + map_base(S.mm_il, S.caps, sr, strand), il_stride(S.mm_il)};
}
__device__ __forceinline__ Strided<short> map_err_of(const Scratch &S, int sr, int strand) {
  return {S.map_err + map_base(S.mm_il, S.caps, sr, strand), il_stride(S.mm_il)};
}
__device__ __forceinline__ Strided<int> map_split_of(const Scratch &S, int sr, int strand) {
  return {S.map_split + map_base(S.mm_il, S.caps, sr, strand), il_stride(S.mm_il)};
}

__device__ __forceinline__ int slot_pair(const Scratch &S, int slot) { return S.pair_list ? S.pair_list[slot] : slot; }

// utils.h:87-104: A/a=0 C/c=1 G/g=2 T/t=3, everything else 4.  Branch-free on purpose: a chain of ternaries
// makes the compiler duplicate the caller's loop body per base and the warp then runs 4-way divergent.
__device__ __forceinline__ u32 base_code(u8 c) {
  const u32 u = (u32)c & 0xDFu;              // fold case: only {0x41,0x61}->'A', {0x43,0x63}->'C', {0x47,0x67}->'G', {0x54,0x74}->'T'
  const u32 x = (u >> 1) & 3u;               // A:0 C:1 G:3 T:2
  const u32 code = x ^ (x >> 1);             // A:0 C:1 G:2 T:3
  const u32 in_row = ((u & 0xE0u) == 0x40u) ? 1u : 0u;                      // 0x40..0x5F
  const u32 is_base = in_row & ((0x0010008Au >> (u & 31u)) & 1u);           // bits 1 (A), 3 (C), 7 (G), 20 (T)
  return is_base ? code : 4u;
}

// utils.h:76-85
__device__ __forceinline__ u64 mix64(u64 key, u64 mask) {
  key = (~key + (key << 21)) & mask;
  key = key ^ key >> 24;
  key = ((key + (key << 3)) + (key << 8)) & mask;
  key = key ^ key >> 14;
  key = ((key + (key << 2)) + (key << 4)) & mask;
  key = key ^ key >> 28;
  key = (key + (key << 31)) & mask;
  return key;
}

// Table probe.  Returns kind (0 absent, 1 singleton, 2 multi); *val = table value.  *steps counts slots read.
__device__ __forceinline__ int index_lookup(const DevIndex &ix, u64 mm_hash, u64 *val, int *steps) {
  u64 s = (mm_hash * 0x9E3779B97F4A7C15ull) >> ix.shift;
  int n = 0;
  for (;;) {
    const ulonglong2 kv = __ldg(&ix.slots[s]);
    ++n;
    if (kv.x == CMX_EMPTY_KEY) { *steps = n; return 0; }
    if ((kv.x >> 1) == mm_hash) { *val = kv.y; *steps = n; return (kv.x & 1) ? 1 : 2; }
    s = (s + 1) & ix.n_slots_mask;
  }
}

// Keyed tables of the cell barcodes (the whitelist, the --barcode-translate table): 16-byte slots {key, value}, empty
// key CMX_EMPTY_KEY, slot = fibonacci(key) >> shift, linear probing; mask = n_slots - 1.
__device__ __forceinline__ bool kv_find(const ulonglong2 *slots, u64 mask, int shift, u64 key, u64 *val) {
  u64 s = (key * 0x9E3779B97F4A7C15ull) >> shift;
  for (;;) {
    const ulonglong2 kv = __ldg(&slots[s]);
    if (kv.x == CMX_EMPTY_KEY) return false;
    if (kv.x == key) { *val = kv.y; return true; }
    s = (s + 1) & mask;
  }
}
// kv_find for the whitelist, whose keys take all 64 bits: the all-T 32-base barcode's key is CMX_EMPTY_KEY itself.  That key
// never enters the slots (wl_insert_kernel skips it); top_listed and top_count, set by cmx_upload_barcode_whitelist, answer
// for it.  The --barcode-translate table needs no such care: its FROM keys have at most 31 bases, so they stay below ~0.
__device__ __forceinline__ bool wl_lookup(const ulonglong2 *slots, u64 mask, int shift, int top_listed, u64 top_count, u64 key, u64 *count) {
  if (key == CMX_EMPTY_KEY) { *count = top_count; return top_listed != 0; }
  return kv_find(slots, mask, shift, key, count);
}
// The slot that holds `key`, claimed for it if the key is new (concurrent inserts of other keys are safe).
__device__ __forceinline__ ulonglong2 *kv_claim(ulonglong2 *slots, u64 mask, int shift, u64 key) {
  u64 s = (key * 0x9E3779B97F4A7C15ull) >> shift;
  for (;;) {
    const u64 old = atomicCAS((unsigned long long *)&slots[s].x, (unsigned long long)CMX_EMPTY_KEY, (unsigned long long)key);
    if (old == CMX_EMPTY_KEY || old == key) return &slots[s];
    s = (s + 1) & mask;
  }
}

// Bring the cache lines of [p, p + bytes) towards the SM ahead of a loop that reads them one byte at a time (the banded
// aligners consume one reference base per column: without this every column waits for its own L2 round trip).
__device__ __forceinline__ void prefetch_span(const void *p, int bytes) {
  const char *a = (const char *)((unsigned long long)p & ~127ull), *z = (const char *)p + bytes;
  for (; a < z; a += 128) asm volatile("prefetch.global.L1 [%0];" ::"l"(a));
}

// One line towards L2, long before it is read (fire and forget).
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// First index in the sorted occurrence list O[0..n) whose position (entry >> 1) is >= lo.  Four-way instead of two-way: a
// search over a list of 10^5 occurrences is a chain of dependent loads, and three independent loads per step halve the chain
// (8 round trips instead of 17); the last <= 8 entries are fetched together.  Same result as a binary lower bound.
__device__ __forceinline__ int occ_lower_bound(const u64 *O, int n, u64 lo) {
  int a = 0, z = n;
  while (z - a > 8) {
    const int q = (z - a) >> 2, m1 = a + q, m2 = m1 + q, m3 = m2 + q;
    const u64 v1 = __ldg(&O[m1]) >> 1, v2 = __ldg(&O[m2]) >> 1, v3 = __ldg(&O[m3]) >> 1;
    if (v3 < lo) a = m3 + 1;
    else if (v2 < lo) { a = m2 + 1; z = m3; }
    else if (v1 < lo) { a = m1 + 1; z = m2; }
    else z = m1;
  }
  int below = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) below += (a + i < z && (__ldg(&O[a + i]) >> 1) < lo) ? 1 : 0;
  return a + below;
}
// index.cc:443-459 replayed on (LB, E): the reference's binary search that starts at l, with every comparison against the list
// replaced by the probe's position relative to LB and LB + E.  Returns the last probe (where the reference starts emitting).
__device__ __forceinline__ int rescue_replay(int l, int n, int lb, int ue) {
  int mid = 0, r = n - 1;
  while (l <= r) {
    mid = (l + r) / 2;
    if (mid < lb) l = mid + 1;
    else if (mid >= ue) r = mid - 1;
    else break;
  }
  return mid;
}

// index.cc:491-505 (u32 wrap kept)
__device__ __forceinline__ u64 hit_to_candidate(int k, u64 ref_hit, u32 read_pos, u32 read_strand, bool *same) {
  const u32 rp = (u32)(ref_hit >> 1);
  const bool sm = ((u32)(ref_hit & 1)) == read_strand;
  const u32 start = sm ? rp - read_pos : rp + read_pos - (u32)k + 1u;
  *same = sm;
  return ((ref_hit >> 33) << 32) | start;
}

// In-place ascending sort of u64 keys by one thread: insertion for short lists, heapsort otherwise.
// A = u64* or Strided<u64>.
template <typename A>
__device__ inline void sort_u64(A a, int n) {
  if (n <= 24) {
    for (int i = 1; i < n; ++i) {
      const u64 v = a[i];
      int j = i - 1;
      while (j >= 0 && a[j] > v) { a[j + 1] = a[j]; --j; }
      a[j + 1] = v;
    }
    return;
  }
  for (int start = n / 2 - 1; start >= 0; --start) {
    int root = start;
    const u64 v = a[root];
    for (;;) {
      int child = 2 * root + 1;
      if (child >= n) break;
      if (child + 1 < n && a[child] < a[child + 1]) ++child;
      if (a[child] <= v) break;
      a[root] = a[child];
      root = child;
    }
    a[root] = v;
  }
  for (int end = n - 1; end > 0; --end) {
    const u64 v = a[end];
    a[end] = a[0];
    int root = 0;
    for (;;) {
      int child = 2 * root + 1;
      if (child >= end) break;
      if (child + 1 < end && a[child] < a[child + 1]) ++child;
      if (a[child] <= v) break;
      a[root] = a[child];
      root = child;
    }
    a[root] = v;
  }
}

// Sort (key, tag) pairs ascending by `less(ka,ta,kb,tb)` — used for candidates (count desc, pos asc) and
// draft mappings (pos asc, err asc).  Insertion for short lists, heapsort otherwise.  K / V: pointers or Strided views.
template <typename T, typename K, typename V, typename Less>
__device__ inline void sort_pairs(K k, V t, int n, Less less) {
  if (n <= 24) {
    for (int i = 1; i < n; ++i) {
      const u64 kv = k[i];
      const T tv = t[i];
      int j = i - 1;
      while (j >= 0 && less(kv, tv, k[j], t[j])) { k[j + 1] = k[j]; t[j + 1] = t[j]; --j; }
      k[j + 1] = kv; t[j + 1] = tv;
    }
    return;
  }
  auto sift = [&](int root, int end, u64 kv, T tv) {
    for (;;) {
      int child = 2 * root + 1;
      if (child >= end) break;
      if (child + 1 < end && less(k[child], t[child], k[child + 1], t[child + 1])) ++child;
      if (!less(kv, tv, k[child], t[child])) break;
      k[root] = k[child]; t[root] = t[child];
      root = child;
    }
    k[root] = kv; t[root] = tv;
  };
  for (int start = n / 2 - 1; start >= 0; --start) sift(start, n, k[start], t[start]);
  for (int end = n - 1; end > 0; --end) {
    const u64 kv = k[end];
    const T tv = t[end];
    k[end] = k[0]; t[end] = t[0];
    sift(0, end, kv, tv);
  }
}
