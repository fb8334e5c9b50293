// chromap_b200 — paired-end mapping pipeline kernels (general tier: one thread per read / per pair,
// state in global scratch).  Exact restatement of the reference's per-pair semantics; the fast
// warp-cooperative kernels for the common small case share this scratch layout.
// File:line citations are into the reference's src/.
#pragma once
#include "device_common.cuh"
#include "minimizers.cuh"

struct MapqTables {
  const double *inv_log;  // [65536]: 3 / log(alignment_length) as computed by the host libm (mapping_generator.h:956-958)
  const int *pen_thr;     // [96]: smallest n with (int)(4.343*log(n+1)+0.499) >= v   (mapping_generator.h:964-967)
};
// The two tables from the host libm, so truncations match the reference bit for bit (mapping_generator.h:920-1022).
inline void mapq_tables_fill(double *inv_log, int *pen_thr) {
  const int coef_frac = log(50);
  inv_log[0] = inv_log[1] = 0.0;
  for (int a = 2; a < 65536; ++a) inv_log[a] = coef_frac / log((unsigned short)a);
  for (int v = 0; v < 96; ++v) {  // smallest n >= 0 with (int)(4.343*log(n+1)+0.499) >= v (monotone in n)
    long long lo = 0, hi = 0x7ffffffeLL;
    auto pen = [](long long n) { return (int)(4.343 * log((double)(n + 1)) + 0.499); };
    if (pen(hi) < v) { pen_thr[v] = 0x7fffffff; continue; }
    while (lo < hi) { const long long mid = (lo + hi) / 2; if (pen(mid) >= v) hi = mid; else lo = mid + 1; }
    pen_thr[v] = (int)lo;
  }
}
// The 624-word state of std::mt19937(seed) right after seeding (an int seed is reduced mod 2^32, random.tcc seed()).
inline void mt_seed_fill(u32 *mt, u32 seed) {
  mt[0] = seed;
  for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (u32)i;
}
// select_kernel's mt_init: std::mt19937(11).
inline void mt_init_fill(u32 *mt) { mt_seed_fill(mt, 11u); }

struct Counters {  // device-side statistics (atomics)
  u64 n_minimizers, n_probe_steps, n_found, n_occ_reads, n_verified, n_candidates, n_mapped, n_unique, n_overflow;
  u64 n_bc_in_whitelist, n_bc_corrected;
  u64 ovf_reason[8];  // tier-0 escalations by cause: 0 read length, 1 #minimizers, 2 seed hits, 3 seed candidates, 4 rescue hits, 5 rescue/merge candidates, 6 draft mappings
  u64 n_bc2_listed, n_bc2_overflow;  // --bc-error-threshold 2: lengths of the correction list and of its overflow list
};

__device__ __forceinline__ const u8 *read_ptr(const DevBatch &B, int pair, int mate) {
  return mate == 0 ? B.seq1 + B.off1[pair] : B.seq2 + B.off2[pair];
}
__device__ __forceinline__ int read_raw_len(const DevBatch &B, int pair, int mate) {
  return mate == 0 ? (int)(B.off1[pair + 1] - B.off1[pair]) : (int)(B.off2[pair + 1] - B.off2[pair]);
}
// base of the reverse-complement strand string (sequence_batch.h:123-134): index i of negative read
__device__ __forceinline__ u32 neg_code(const u8 *read, int L, int i) {
  const u32 c = base_code(read[L - 1 - i]);
  return c < 4 ? 3u ^ c : 4u;
}
__device__ __forceinline__ u8 code_char(u32 c) { return c == 0 ? 'A' : c == 1 ? 'C' : c == 2 ? 'G' : c == 3 ? 'T' : 'N'; }

// Counter updates: every lane adds to the same address, and same-address atomics serialise in L2 at about one
// per clock, so the lanes that are here together add up first and one of them issues the atomic.
#ifndef CMX_HOST_EMU  // (__activemask has no host equivalent: the host emulation of a CTA supplies plain atomics)
__device__ __forceinline__ void agg_add(u64 *addr, u64 v) {
  const unsigned m = __activemask();
  const unsigned s_ = __reduce_add_sync(m, (unsigned)v);
  if ((int)(threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(addr, (u64)s_);
}
// Append to a list with one atomic per group of converged lanes; returns this lane's index.
__device__ __forceinline__ int agg_append(int *count) {
  const unsigned m = __activemask();
  const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(count, __popc(m));
  base = __shfl_sync(m, base, leader);
  return base + __popc(m & ((1u << lane) - 1u));
}
#endif

// ------------------------------------------------------------------------------------------------
// K0: per pair — length filter (chromap.h:911-916) and adapter trimming (chromap.cc:176-289).
__global__ void prep_kernel(DevParams P, DevBatch B, Scratch S) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  const int pair = slot_pair(S, slot);
  PairMeta pm;
  pm.status = ST_OK; pm.sup = 0; pm.min_sum = 0; pm.second_min_sum = 0; pm.n_best = 0; pm.n_second_best = 0; pm.n_rec = 0; pm.pad = 0;
  int len1 = read_raw_len(B, pair, 0), len2 = P.se ? 0 : read_raw_len(B, pair, 1);
  if (B.bc_ok && !B.bc_ok[pair]) pm.status = ST_DROP;  // chromap.h:908-909
  else if (len1 < P.min_read_len || (!P.se && len2 < P.min_read_len)) pm.status = ST_DROP;  // single-end: chromap.h:411-414
  else if (len1 > S.caps.maxmm || len2 > S.caps.maxmm) pm.status = ST_OVERFLOW;  // longer than max_read_length
  else if (P.trim && !P.se) {
    const u8 *raw1 = read_ptr(B, pair, 0), *raw2 = read_ptr(B, pair, 1);
    const bool swp = !(len1 <= len2);
    const u8 *r1 = swp ? raw2 : raw1;   // the shorter read
    const u8 *r2 = swp ? raw1 : raw2;   // the other one; we search in its reverse complement
    const int L1 = swp ? len2 : len1, L2 = swp ? len1 : len2;
    const int min_ovl = P.min_read_len, seed = min_ovl / 2;
    bool merged = false;
    for (int si = 0; si < 2 && !merged; ++si) {
      // std::string::find of r1[si*seed .. +seed) in neg2, scanning start positions upward
      for (int sp = 0; sp + seed <= L2 && !merged; ++sp) {
        bool hit = true;
        for (int j = 0; j < seed; ++j)
          if (code_char(neg_code(r2, L2, sp + j)) != r1[si * seed + j]) { hit = false; break; }
        if (!hit) continue;
        if (!(sp >= si * seed) || !((int)(L2 - sp + seed * si) >= min_ovl)) continue;
        bool ok = true;
        int ne = 0;
        for (int i = 0; i < seed * si; ++i) {
          if (code_char(neg_code(r2, L2, sp - si * seed + i)) != r1[i]) ++ne;
          if (ne > 1) { ok = false; break; }
        }
        if (ok)
          for (int i = seed; i + sp < L2 && si * seed + i < L1; ++i) {
            if (code_char(neg_code(r2, L2, sp + i)) != r1[si * seed + i]) ++ne;
            if (ne > 1) { ok = false; break; }
          }
        if (!ok) continue;
        int ovl = L2 - sp + si * seed, off2 = 0;
        if (ovl > L1) { off2 = ovl - L1; ovl = L1; }
        const int t1 = swp ? ovl + off2 : ovl, t2 = swp ? ovl : ovl + off2;
        if (t1 < len1) len1 = t1;
        if (t2 < len2) len2 = t2;
        merged = true;
      }
    }
  }
  S.pmeta[slot] = pm;
  ReadMeta z;
  memset(&z, 0, sizeof(z));
  z.len = len1; S.rmeta[2 * slot] = z;
  z.len = len2; S.rmeta[2 * slot + 1] = z;
}

struct RepStats { u32 len, prev; int count; };
__device__ __forceinline__ void rep_update(int k, int w, u32 read_pos, RepStats &st) {  // index.cc:507-523
  if (st.prev > read_pos) st.len += k;
  else if (read_pos < st.prev + k + w - 1) st.len += read_pos - st.prev;
  else st.len += k;
  st.prev = read_pos;
  ++st.count;
}

// candidate_processor.cc:283-342 — clustering scan over sorted hits (sentinel handled implicitly).
// A, PA, CA: pointers or Strided views.
template <typename A, typename PA, typename CA>
__device__ inline int cluster_hits(int e, int need, u32 n_mm, A hits, int nh, PA cpos, CA ccnt, int cap) {
  if (nh == 0) return 0;
  int n = 0, mcount = 1, eq = 1, best_eq = 1;
  u64 prev = hits[0], best = hits[0];
  u32 prev_rid = (u32)(prev >> 32), prev_pos = (u32)prev;
  for (int i = 1; i <= nh; ++i) {
    const u64 h = i < nh ? hits[i] : ~0ull;
    const u32 rid = (u32)(h >> 32), pos = (u32)h;
    if (rid != prev_rid || pos > prev_pos + (u32)e || ((u32)mcount >= n_mm && pos > (u32)best + (u32)e)) {
      if (mcount >= need) { if (n < cap) { cpos[n] = best; ccnt[n] = (u8)best_eq; } ++n; }
      mcount = 1; eq = 1; best_eq = 1; best = h;
    } else {
      if (h == best) { ++eq; ++best_eq; }
      else if (h == prev) { ++eq; if (eq > best_eq) { best = prev; best_eq = eq; } }
      else eq = 1;
      ++mcount;
    }
    prev = h; prev_rid = rid; prev_pos = pos;
  }
  return n;
}

// K1c: per read — hit lists from the probed values, sort, clustering (candidate_processor.cc:12-71,
// index.cc:237-349).  Tier 0 takes only "light" reads: as soon as the exact hit count (known from the table
// values before any occurrence is read) exceeds the tier's capacity the pair is escalated to the CTA tier.
// The hit lists never touch global memory: every thread owns one column of an interleaved shared-memory tile
// [hc][CLUSTER_NT] (bank-conflict free: lane t reads word i*CLUSTER_NT + t), + strand hits growing from row 0,
// - strand hits from row hc-1 downwards (their total is <= hc by the check above).
#define CLUSTER_NT 128
// Two launches: mode 0 with a `rows`-row tile (16: full occupancy) takes the reads with at most `rows` hits and
// lists the others, mode 1 runs the list with an hc-row tile.
__global__ void __launch_bounds__(CLUSTER_NT) cluster_kernel(DevParams P, DevIndex ix, Scratch S, Counters *ctr, int mode, int rows, int *list,
                                                             int *list_count) {
  extern __shared__ u64 sh_hits[];
  const int tid = blockIdx.x * CLUSTER_NT + threadIdx.x;
  int sr = tid;
  if (mode == 1) {
    if (tid >= *list_count) return;
    sr = list[tid];
  } else if (sr >= 2 * S.n_slots) return;
  const int slot = sr >> 1;
  if (S.pmeta[slot].status != ST_OK) return;
  ReadMeta &rm = S.rmeta[sr];
  const Caps c = S.caps;
  const int n_mm = rm.n_mm;
  if (n_mm == 0) return;
  const int ms = mm_stride(S);
  const u64 *mmv = S.mm_val + mm_base(S, slot, sr & 1);
  const u32 *mmp = S.mm_pos + mm_base(S, slot, sr & 1);
  long long cnt1 = 0, cnt2 = 0;
  RepStats st = {0u, 0xFFFFFFFFu, 0};
  for (int i = 0; i < n_mm; ++i) {
    const u32 kind = mmp[(size_t)i * ms] >> 30;
    if (kind == 1) { ++cnt1; ++cnt2; }
    else if (kind == 2) {
      const u64 v_ = mmv[(size_t)i * ms];
      const u32 n = (u32)v_;
      if (n < (u32)P.f1) prefetch_span(&ix.occ[(u32)(v_ >> 32)], (int)min(n, 64u) * 8);  // the expansion below reads them: request them now
      if (n < (u32)P.f0) cnt1 += n;
      if (n < (u32)P.f1) cnt2 += n;
      if (n >= (u32)P.f0) rep_update(P.k, P.w, (mmp[(size_t)i * ms] & 0x3FFFFFFFu) >> 1, st);
    }
  }
  // round 1 (f0) or, if it yields no hits at all, round 2 (f1)  (candidate_processor.cc:30-50)
  const bool round2 = cnt1 == 0;
  const long long total = round2 ? cnt2 : cnt1;
  if (total > c.hc) { S.pmeta[slot].status = ST_OVERFLOW; atomicAdd(&ctr->ovf_reason[2], 1ull); return; }  // per-strand lists can then never exceed hc
  if (total > rows) { list[agg_append(list_count)] = sr; return; }  // mode 0 only: rows == hc in mode 1
  const u32 max_freq = round2 ? (u32)P.f1 : (u32)P.f0;
  const Strided<u64> hp = {sh_hits + threadIdx.x, CLUSTER_NT};
  const Strided<u64> hn = {sh_hits + (size_t)(rows - 1) * CLUSTER_NT + threadIdx.x, -CLUSTER_NT};
  int np = 0, nn = 0;
  u32 occ_reads = 0;
  for (int i = 0; i < n_mm; ++i) {
    const u32 kind = mmp[(size_t)i * ms] >> 30;
    if (kind == 0) continue;
    const u32 rpos = (mmp[(size_t)i * ms] & 0x3FFFFFFFu) >> 1, rstrand = mmp[(size_t)i * ms] & 1u;
    const u64 val = mmv[(size_t)i * ms];
    bool same;
    if (kind == 1) {
      const u64 cp = hit_to_candidate(P.k, val, rpos, rstrand, &same);
      if (same) hp[np++] = cp; else hn[nn++] = cp;
      continue;
    }
    const u32 n = (u32)val, off = (u32)(val >> 32);
    if (n < max_freq) {
      for (u32 q = 0; q < n; ++q) {
        const u64 rh = __ldg(&ix.occ[off + q]);
        const u64 cp = hit_to_candidate(P.k, rh, rpos, rstrand, &same);
        if (same) hp[np++] = cp; else hn[nn++] = cp;
      }
      occ_reads += n;
    }
  }
  if (occ_reads) agg_add(&ctr->n_occ_reads, (u64)occ_reads);
  sort_u64(hp, np);
  sort_u64(hn, nn);
  rm.rep_len = st.len;
  int need = n_mm - st.count;
  need = need > 1 ? need : 1;
  need = need > P.min_seeds ? P.min_seeds : need;
  if (round2 && np > 0 && nn > 0) need = P.min_seeds;
  const int nc0 = cluster_hits(P.e, need, (u32)n_mm, hp, np, cand_pos_of(S, sr, 0, 0), cand_cnt_of(S, sr, 0, 0), c.cc);
  const int nc1 = cluster_hits(P.e, need, (u32)n_mm, hn, nn, cand_pos_of(S, sr, 0, 1), cand_cnt_of(S, sr, 0, 1), c.cc);
  if (nc0 > c.cc || nc1 > c.cc) { S.pmeta[slot].status = ST_OVERFLOW; atomicAdd(&ctr->ovf_reason[3], 1ull); return; }
  rm.n_cand[0] = nc0; rm.n_cand[1] = nc1;
  rm.n_cand_gen[0] = nc0; rm.n_cand_gen[1] = nc1;
}

// ------------------------------------------------------------------------------------------------
// index.cc:351-489 — mate-guided lookup on one strand for one read (by one thread).
// Returns +max count or -max count (bail-out); hits appended (sorted) into `hits`, *nh set (may exceed cap).
// PA, CA: pointers or Strided views.
template <typename PA, typename CA>
__device__ inline int rescue_hits(const DevParams &P, const DevIndex &ix, int strand, u32 range, int n_mm, const u64 *mmv,
                                  const u32 *mmp, int ms, PA mate_pos, CA mate_cnt, int n_mate, u32 *rep_len,
                                  u64 *hits, int cap, int *nh_out) {
  int max_cnt = 0, n_best = 0;
  for (int i = 0; i < n_mate; ++i) {
    const int cnt = mate_cnt[i];
    if (cnt > max_cnt) { max_cnt = cnt; n_best = 1; }
    else if (cnt == max_cnt) ++n_best;
  }
  *nh_out = 0;
  if (n_best >= 300 || n_mate > P.f0 || (max_cnt <= P.min_seeds && n_best >= 200)) return -max_cnt;
  // (raw_boundary_size == 0 cannot happen when n_mate > 0)
  int nh = 0;
  RepStats st = {0u, 0xFFFFFFFFu, 0};
  for (int mi = 0; mi < n_mm; ++mi) {
    const u32 kind = mmp[(size_t)mi * ms] >> 30;
    if (kind == 0) continue;
    const u32 rpos = (mmp[(size_t)mi * ms] & 0x3FFFFFFFu) >> 1, rstrand = mmp[(size_t)mi * ms] & 1u;
    const u64 val = mmv[(size_t)mi * ms];
    bool same;
    if (kind == 1) {
      const u64 cp = hit_to_candidate(P.k, val, rpos, rstrand, &same);
      if ((same && strand == 0) || (!same && strand == 1)) { if (nh < cap) hits[nh] = cp; ++nh; }
      continue;
    }
    const u32 off = (u32)(val >> 32), n = (u32)val;
    int prev_l = 0;
    // iterate merged windows (index.cc:383-412) generated on the fly from the sorted mate candidates
    int ci = 0;
    while (ci < n_mate) {
      while (ci < n_mate && mate_cnt[ci] != max_cnt) ++ci;
      if (ci >= n_mate) break;
      u64 lo = mate_pos[ci] < range ? 0 : mate_pos[ci] - range;
      u64 hi = mate_pos[ci] + range;
      ++ci;
      for (;;) {
        int cj = ci;
        while (cj < n_mate && mate_cnt[cj] != max_cnt) ++cj;
        if (cj >= n_mate) { ci = cj; break; }
        const u64 lo2 = mate_pos[cj] < range ? 0 : mate_pos[cj] - range;
        if (hi < lo2) { ci = cj; break; }
        hi = mate_pos[cj] + range;
        ci = cj + 1;
      }
      // the reference's search (index.cc:443-459) starts at the previous window's last probe and ends on a probe that depends on
      // its path; only the comparisons touch memory, and they only depend on where a probe lies relative to LB and LB + E: find
      // LB with the four-way search, then replay the path arithmetically (E <= 1: distinct positions, checked at index upload)
      const int lbq = occ_lower_bound(ix.occ + off, (int)n, lo);
      const int eqq = (lbq < (int)n && (__ldg(&ix.occ[off + lbq]) >> 1) == lo) ? 1 : 0;
      const int mid = rescue_replay(prev_l, (int)n, lbq, lbq + eqq);
      prev_l = mid;
      for (u32 oi = (u32)mid; oi < n; ++oi) {
        const u64 rh = __ldg(&ix.occ[off + oi]);
        if ((rh >> 1) > hi) break;
        const u64 cp = hit_to_candidate(P.k, rh, rpos, rstrand, &same);
        if ((same && strand == 0) || (!same && strand == 1)) { if (nh < cap) hits[nh] = cp; ++nh; }
      }
    }
    if (n >= (u32)P.f0) rep_update(P.k, P.w, rpos, st);
  }
  *nh_out = nh;
  if (nh <= cap) sort_u64(hits, nh);
  *rep_len = st.len;
  return max_cnt;
}

// candidate_processor.cc:345-414 — merge c2 into c1 using `out` as the buffer, result copied back to c1.
// Returns the new size of c1 (may exceed cap -> overflow).  PA, CA: pointers or Strided views.
template <typename PA, typename CA>
__device__ inline int merge_cands(int e, PA p1, CA c1, int n1, PA p2, CA c2, int n2, PA po, CA co, int cap) {
  if (n1 == 0) {
    for (int i = 0; i < n2 && i < cap; ++i) { p1[i] = p2[i]; c1[i] = c2[i]; }
    return n2;
  }
  int i = 0, j = 0, n = 0;
  u64 last = 0;
#define FAR(p) (n == 0 || (p) > last + (u64)e)
#define PUSH(p, c) do { if (n < cap) { po[n] = (p); co[n] = (c); } last = (p); ++n; } while (0)
  while (i < n1 && j < n2) {
    if (p1[i] == p2[j]) { if (FAR(p1[i])) { if (c1[i] > c2[j]) PUSH(p1[i], c1[i]); else PUSH(p2[j], c2[j]); } ++i; ++j; }
    else if (p1[i] < p2[j]) { if (FAR(p1[i])) PUSH(p1[i], c1[i]); ++i; }
    else { if (FAR(p2[j])) PUSH(p2[j], c2[j]); ++j; }
  }
  for (; i < n1; ++i) if (FAR(p1[i])) PUSH(p1[i], c1[i]);
  for (; j < n2; ++j) if (FAR(p2[j])) PUSH(p2[j], c2[j]);
#undef FAR
#undef PUSH
  for (int t = 0; t < n && t < cap; ++t) { p1[t] = po[t]; c1[t] = co[t]; }
  return n;
}

// candidate_processor.cc:416-484.  Inputs IP / IC and outputs OP / OC: pointers or Strided views.
template <typename IP, typename IC, typename OP, typename OC>
__device__ inline void pe_filter_dir(u32 dist, IP p1, IC c1, int n1, IP p2, IC c2, int n2, OP f1p, OC f1c, int *nf1, OP f2p, OC f2c, int *nf2) {
  int i1 = 0, i2 = 0, prev_end = 0, a = 0, b = 0;
  int un1 = 0, un2 = 0, max1 = 6, max2 = 6;
  while (i1 < n1 && i2 < n2) {
    if (p1[i1] > p2[i2] + dist) {
      if (i2 >= prev_end && un2 < 5 && (p1[i1] >> 32) == (p2[i2] >> 32) && c2[i2] >= max2) { f2p[b] = p2[i2]; f2c[b] = c2[i2]; ++b; ++un2; }
      ++i2;
    } else if (p2[i2] > p1[i1] + dist) {
      if (un1 < 5 && (p1[i1] >> 32) == (p2[i2] >> 32) && c1[i1] >= max1) { f1p[a] = p1[i1]; f1c[a] = c1[i1]; ++a; ++un1; }
      ++i1;
    } else {
      f1p[a] = p1[i1]; f1c[a] = c1[i1]; ++a;
      if (c1[i1] > max1) max1 = c1[i1];
      int j = i2;
      while (j < n2 && p2[j] <= p1[i1] + dist) {
        if (j >= prev_end) { f2p[b] = p2[j]; f2c[b] = c2[j]; ++b; if (c2[j] > max2) max2 = c2[j]; }
        ++j;
      }
      prev_end = j;
      ++i1;
    }
  }
  *nf1 = a; *nf2 = b;
}

// K2: per pair — SupplementCandidates (candidate_processor.cc:75-231), MoveCandidiatesToBuffer +
// ReduceCandidatesForPairedEndRead (chromap.h:1036-1052, candidate_processor.cc:233-263).
// Two launches: mode 0 handles every pair that needs no mate-guided lookup (the common case: a few loads and two short
// sweeps) and appends the others to `list`; mode 1 runs those densely packed, one thread per pair — thousands of pairs in
// flight per SM hide the dependent occurrence-list reads (a warp per pair was measured 9x slower: 32 pairs per SM in flight).
#define PC_SMALL 8          // lists of at most this many candidates take the local-memory path
#define PC_RESCUE_HEAVY 48  // more (minimizer, window) searches than this: the lookup runs in the CTA tier
__global__ void pair_candidates_kernel(DevParams P, DevIndex ix, Scratch S, Counters *ctr, int mode, int *list, int *list_count) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  int slot = tid;
  if (mode == 1) {
    if (tid >= *list_count) return;
    slot = list[tid];
  } else if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  if (pm.status != ST_OK) return;
  const Caps c = S.caps;
  ReadMeta *rm = S.rmeta + 2 * slot;
  auto CP = [&](int mate, int set, int strand) { return cand_pos_of(S, 2 * slot + mate, set, strand); };
  auto CC = [&](int mate, int set, int strand) { return cand_cnt_of(S, 2 * slot + mate, set, strand); };
  if (P.se) {  // single-end (chromap.h:449-453): a read goes on iff it has minimizers and candidates
    if (mode != 0) return;
    const int a1 = rm[0].n_cand[0] + rm[0].n_cand[1];
    if (rm[0].n_mm == 0 || a1 == 0) { pm.status = ST_DROP; return; }
    agg_add(&ctr->n_candidates, (u64)a1);
    return;
  }
  if (P.split) {  // chromap.h:1021,1036-1038: no mate supplementation and no paired-end filter under split alignment
    if (mode != 0) return;
    if (rm[0].n_mm == 0 || rm[1].n_mm == 0) { pm.status = ST_DROP; return; }
    const int a1 = rm[0].n_cand[0] + rm[0].n_cand[1], a2 = rm[1].n_cand[0] + rm[1].n_cand[1];
    if (!(a1 > 0 && a2 > 0)) { pm.status = ST_DROP; return; }
    agg_add(&ctr->n_candidates, (u64)(a1 + a2));
    return;
  }
  if (mode == 0) {
    if (rm[0].n_mm == 0 || rm[1].n_mm == 0) { pm.status = ST_DROP; return; }
    // the common case -- a handful of candidates per list -- is staged in local memory (interleaved per lane by the
    // hardware, i.e. coalesced), filtered from there straight into set 0: no round trip through the buffer set
    const int nq[4] = {rm[0].n_cand[0], rm[0].n_cand[1], rm[1].n_cand[0], rm[1].n_cand[1]};
    const bool small = nq[0] <= PC_SMALL && nq[1] <= PC_SMALL && nq[2] <= PC_SMALL && nq[3] <= PC_SMALL;
    u64 lp[4][PC_SMALL];
    u8 lc[4][PC_SMALL];
    if (small) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const Strided<u64> src = CP(q >> 1, 0, q & 1);
        const Strided<u8> srcc = CC(q >> 1, 0, q & 1);
        for (int i = 0; i < nq[q]; ++i) { lp[q][i] = src[i]; lc[q][i] = srcc[i]; }
      }
    }
    bool need = false;
    bool aug[2];
    for (int mate = 0; mate < 2; ++mate) {
      const u32 n_mm = rm[mate].n_mm;
      bool a = true;
      for (int s = 0; s < 2 && a; ++s) {
        const Strided<u8> cc = CC(mate, 0, s);
        for (int i = 0; i < nq[mate * 2 + s]; ++i) if ((small ? lc[mate * 2 + s][i] : cc[i]) >= n_mm / 2) { a = false; break; }
      }
      aug[mate] = a;
      // a rescue lookup only happens when the mate has candidates to guide it (candidate_processor.cc:163-181)
      if (a && nq[(1 - mate) * 2] + nq[(1 - mate) * 2 + 1] > 0) need = true;
    }
    if (need) {
      // one thread walks every (multi-occurrence minimizer, mate window) binary search of the lookup; when that product is
      // large the pair goes to the CTA tier, where a warp takes each minimizer and a lane each window (same results)
      u32 searches = 0;
      for (int mate = 0; mate < 2; ++mate) {
        if (!aug[mate]) continue;
        const u32 *mmp = S.mm_pos + mm_base(S, slot, mate);
        const int ms = mm_stride(S);
        u32 n_multi = 0;
        for (int i = 0; i < rm[mate].n_mm; ++i) n_multi += (mmp[(size_t)i * ms] >> 30) == 2;
        searches += n_multi * (u32)(nq[(1 - mate) * 2] + nq[(1 - mate) * 2 + 1]);
      }
      if (searches > PC_RESCUE_HEAVY) { pm.status = ST_OVERFLOW; agg_add(&ctr->ovf_reason[7], 1ull); return; }
      list[agg_append(list_count)] = slot;
      return;
    }
    // no rescue: hits are cleared in the reference but nothing reads them afterwards; ret stays 0
    if (small) {
      int nc1 = nq[0] + nq[1], nc2 = nq[2] + nq[3];
      if (nc1 > 0 && nc2 > 0) {
        int a, b;
        pe_filter_dir((u32)P.max_insert, lp[0], lc[0], nq[0], lp[3], lc[3], nq[3], CP(0, 0, 0), CC(0, 0, 0), &a, CP(1, 0, 1), CC(1, 0, 1), &b);
        rm[0].n_cand[0] = a; rm[1].n_cand[1] = b;
        nc1 = a; nc2 = b;
        pe_filter_dir((u32)P.max_insert, lp[1], lc[1], nq[1], lp[2], lc[2], nq[2], CP(0, 0, 1), CC(0, 0, 1), &a, CP(1, 0, 0), CC(1, 0, 0), &b);
        rm[0].n_cand[1] = a; rm[1].n_cand[0] = b;
        nc1 += a; nc2 += b;
      }
      if (!(nc1 > 0 && nc2 > 0)) { pm.status = ST_DROP; return; }
      agg_add(&ctr->n_candidates, (u64)(nc1 + nc2));
      return;
    }
  } else {
    int ret = 0;
    const u32 range = 2u * (u32)P.max_insert;
    bool ovf = false;
    for (int mate = 0; mate < 2; ++mate) {
      ReadMeta &me = rm[mate];
      const ReadMeta &ot = rm[1 - mate];
      const u32 n_mm = me.n_mm;
      bool a = true;
      for (int s = 0; s < 2 && a; ++s) {
        const Strided<u8> cc = CC(mate, 0, s);
        for (int i = 0; i < me.n_cand[s]; ++i) if (cc[i] >= n_mm / 2) { a = false; break; }
      }
      if (!a) continue;
      const size_t sr = 2 * slot + mate;
      const u64 *mmv = S.mm_val + mm_base(S, slot, mate);
      const u32 *mmp = S.mm_pos + mm_base(S, slot, mate);
      const int ms = mm_stride(S);
      u64 *hp = S.hits + (sr * 2 + 0) * c.hc, *hn = S.hits + (sr * 2 + 1) * c.hc;
      int pr = 0, nr = 0;
      if (ot.n_cand[0] > 0) {
        int nh;
        pr = rescue_hits(P, ix, 1, range, n_mm, mmv, mmp, ms, CP(1 - mate, 0, 0), CC(1 - mate, 0, 0), ot.n_cand[0], &me.rep_len, hn, c.hc, &nh);
        if (nh > c.hc) { ovf = true; atomicAdd(&ctr->ovf_reason[4], 1ull); break; }
        const int na = cluster_hits(P.e, 1, n_mm, hn, nh, CP(mate, 2, 1), CC(mate, 2, 1), c.cc);
        if (na > c.cc) { ovf = true; atomicAdd(&ctr->ovf_reason[5], 1ull); break; }
        me.n_aug[1] = na;
      }
      if (ot.n_cand[1] > 0) {
        int nh;
        nr = rescue_hits(P, ix, 0, range, n_mm, mmv, mmp, ms, CP(1 - mate, 0, 1), CC(1 - mate, 0, 1), ot.n_cand[1], &me.rep_len, hp, c.hc, &nh);
        if (nh > c.hc) { ovf = true; atomicAdd(&ctr->ovf_reason[4], 1ull); break; }
        const int na = cluster_hits(P.e, 1, n_mm, hp, nh, CP(mate, 2, 0), CC(mate, 2, 0), c.cc);
        if (na > c.cc) { ovf = true; atomicAdd(&ctr->ovf_reason[5], 1ull); break; }
        me.n_aug[0] = na;
      }
      if (((pr < 0 && nr > 0 && -pr >= nr) || (pr > 0 && nr < 0 && pr <= -nr)) && me.n_cand[0] + me.n_cand[1] == 0) ret = 1;
    }
    if (ovf) { pm.status = ST_OVERFLOW; return; }
    for (int mate = 0; mate < 2 && !ovf; ++mate)
      for (int s = 0; s < 2; ++s) {
        ReadMeta &me = rm[mate];
        if (me.n_aug[s] > 0) {
          const int n = merge_cands(P.e, CP(mate, 0, s), CC(mate, 0, s), me.n_cand[s], CP(mate, 2, s), CC(mate, 2, s), me.n_aug[s],
                                    CP(mate, 1, s), CC(mate, 1, s), c.cc);
          if (n > c.cc) { ovf = true; atomicAdd(&ctr->ovf_reason[5], 1ull); break; }
          me.n_cand[s] = n;
        }
      }
    if (ovf) { pm.status = ST_OVERFLOW; return; }
    pm.sup = ret;
  }
  int nc1 = rm[0].n_cand[0] + rm[0].n_cand[1], nc2 = rm[1].n_cand[0] + rm[1].n_cand[1];
  if (nc1 > 0 && nc2 > 0) {
    // move candidates to the buffer set (1), filter back into set 0
    int nbuf[2][2];
    for (int mate = 0; mate < 2; ++mate)
      for (int s = 0; s < 2; ++s) {
        const int n = rm[mate].n_cand[s];
        const Strided<u64> src = CP(mate, 0, s), dst = CP(mate, 1, s);
        const Strided<u8> srcc = CC(mate, 0, s), dstc = CC(mate, 1, s);
        for (int i = 0; i < n; ++i) { dst[i] = src[i]; dstc[i] = srcc[i]; }
        nbuf[mate][s] = n;
      }
    int a, b;
    pe_filter_dir((u32)P.max_insert, CP(0, 1, 0), CC(0, 1, 0), nbuf[0][0], CP(1, 1, 1), CC(1, 1, 1), nbuf[1][1],
                  CP(0, 0, 0), CC(0, 0, 0), &a, CP(1, 0, 1), CC(1, 0, 1), &b);
    rm[0].n_cand[0] = a; rm[1].n_cand[1] = b;
    pe_filter_dir((u32)P.max_insert, CP(0, 1, 1), CC(0, 1, 1), nbuf[0][1], CP(1, 1, 0), CC(1, 1, 0), nbuf[1][0],
                  CP(0, 0, 1), CC(0, 0, 1), &a, CP(1, 0, 0), CC(1, 0, 0), &b);
    rm[0].n_cand[1] = a; rm[1].n_cand[0] = b;
    nc1 = rm[0].n_cand[0] + rm[0].n_cand[1];
    nc2 = rm[1].n_cand[0] + rm[1].n_cand[1];
  }
  if (!(nc1 > 0 && nc2 > 0)) { pm.status = ST_DROP; return; }
  agg_add(&ctr->n_candidates, (u64)(nc1 + nc2));
}

// The pattern window of the banded aligners as three bit planes (bit i of plane b = bit b of the base code at window
// position i) instead of the reference's five Peq words: the match vector against a text base is three XORs, and a
// new pattern base costs three ORs.  Same X as `Peq[code(text)]` (code 4 matches code 4), masked to the band.
struct PatPlanes { u32 p0, p1, p2; };
__device__ __forceinline__ void planes_or(PatPlanes &w, u32 code, u32 bit) {
  w.p0 |= (0u - (code & 1u)) & bit;
  w.p1 |= (0u - ((code >> 1) & 1u)) & bit;
  w.p2 |= (0u - (code >> 2)) & bit;
}
__device__ __forceinline__ u32 planes_match(const PatPlanes &w, u32 code, u32 band_mask) {
  return ~((w.p0 ^ (0u - (code & 1u))) | (w.p1 ^ (0u - ((code >> 1) & 1u))) | (w.p2 ^ (0u - (code >> 2)))) & band_mask;
}
__device__ __forceinline__ void planes_shift(PatPlanes &w) { w.p0 >>= 1; w.p1 >>= 1; w.p2 >>= 1; }

// ------------------------------------------------------------------------------------------------
// alignment.cc:141-192 — banded Myers/Hyyro bit-vector edit distance, band 2e+1, u32 words.
// PAT(i) -> base code of the reference window at i; TXT(i) -> base code of the read at i.
template <typename PatF, typename TxtF>
__device__ __forceinline__ int banded_align(int e, int L, PatF PAT, TxtF TXT, int *end_pos) {
  PatPlanes W = {0u, 0u, 0u};
  for (int i = 0; i < 2 * e; ++i) planes_or(W, PAT(i), 1u << i);
  const u32 hi = 1u << (2 * e), band = (hi << 1) - 1u;
  u32 VP = 0, VN = 0;
  int err = 0;
  // software pipelined: the bases of column i + 1 are requested before column i is worked on, so a column never waits for
  // its own load (one reference byte and one read byte per column)
  u32 pat_n = L > 0 ? PAT(2 * e) : 0u, txt_n = L > 0 ? TXT(0) : 0u;
  for (int i = 0; i < L; ++i) {
    const u32 pat = pat_n, txt = txt_n;
    if (i + 1 < L) { pat_n = PAT(i + 1 + 2 * e); txt_n = TXT(i + 1); }
    planes_or(W, pat, hi);
    u32 X = VN | planes_match(W, txt, band);
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    VN = X & HP;
    VP = HN | ~(X | HP);
    err += 1 - (int)(D0 & 1u);
    if (err > 3 * e) return e + 1;
    planes_shift(W);
  }
  int best = err;
  *end_pos = L - 1;
  for (int i = 0; i < 2 * e; ++i) {
    err += (int)((VP >> i) & 1u);
    err -= (int)((VN >> i) & 1u);
    if (err < best || (err == best && i + 1 == e)) { best = err; *end_pos = L + i; }
  }
  return best;
}

__device__ __forceinline__ bool valid_cand(int e, u32 ref_len, u32 pos, u32 L) {  // draft_mapping_generator.cc:59-70
  return !(pos < (u32)e || pos >= ref_len || pos + L + (u32)e >= ref_len);
}

struct Tally { int min_err, second_min_err, n_best, n_second_best; };
__device__ __forceinline__ void tally(Tally &t, int err) {
  if (err < t.min_err) { t.second_min_err = t.min_err; t.n_second_best = t.n_best; t.min_err = err; t.n_best = 1; }
  else if (err == t.min_err) t.n_best++;
  else if (err == t.second_min_err) t.n_second_best++;
  else if (err < t.second_min_err) { t.n_second_best = 1; t.second_min_err = err; }
}

// K3: per read — GenerateDraftMappings (draft_mapping_generator.cc:9-57; fast path :72-157; lane-group
// driver :159-357 replayed with the scalar routine; per-candidate driver :359-557), non-split.
// Two launches: mode 0 settles the reads that take the zero-DP fast path (about 70 % at 2x50) and appends the
// others to `list`; mode 1 runs the banded alignments over the list, densely packed, so a warp is not held up by
// its few aligning lanes.
__global__ void verify_kernel(DevParams P, DevRef R, DevBatch B, Scratch S, Counters *ctr, int mode, int *list, int *list_count) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  int sr = tid;
  if (mode == 1) {
    if (tid >= *list_count) return;
    sr = list[tid];
  } else if (sr >= 2 * S.n_slots) return;
  const int slot = sr >> 1, mate = sr & 1;
  if (S.pmeta[slot].status != ST_OK || (P.se && mate == 1)) return;
  const int pair = slot_pair(S, slot);
  ReadMeta &rm = S.rmeta[sr];
  const Caps c = S.caps;
  const u8 *read = read_ptr(B, pair, mate);
  const int L = rm.len, e = P.e;
  Tally t = {e + 1, e + 1, 0, 0};
  // (views rebuilt where they are used: arrays of them would live in local memory)
  auto MP = [&](int s) { return map_pos_of(S, sr, s); };
  auto ME = [&](int s) { return map_err_of(S, sr, s); };
  int nm[2] = {0, 0};
  auto CP = [&](int s) { return cand_pos_of(S, sr, 0, s); };
  auto CC = [&](int s) { return cand_cnt_of(S, sr, 0, s); };
  const int nc[2] = {rm.n_cand[0], rm.n_cand[1]};
  bool done = false;
  if (mode == 0 && nc[0] + nc[1] == 1) {
    int n_all = 0, idx = 0, strand = 0;
    for (int i = 0; i < nc[0]; ++i) if (CC(0)[i] == rm.n_mm) { idx = i; ++n_all; }
    for (int i = 0; i < nc[1]; ++i) if (CC(1)[i] == rm.n_mm) { idx = i; strand = 1; ++n_all; }
    if (n_all == 1) {
      t.min_err = 0; t.n_best = 1; t.n_second_best = 0;
      const u64 cpos = CP(strand)[idx];
      const u32 rid = (u32)(cpos >> 32);
      const u32 pos = strand == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
      if (valid_cand(e, R.len[rid], pos, (u32)L)) {
        MP(strand)[0] = strand == 0 ? cpos + (u64)L - 1 : cpos;
        ME(strand)[0] = 0;
        nm[strand] = 1;
        done = true;
      }
    }
  }
  u64 n_verified = 0;
  if (mode == 0 && !done && nc[0] + nc[1] > 0) { list[agg_append(list_count)] = sr; return; }
  if (!done && nc[0] + nc[1] > 0) {  // (pass 0 never gets here: it has listed the read; it is launched without the code buffer)
    auto cless = [](u64 pa, u8 ca, u64 pb, u8 cb) { return ca != cb ? ca > cb : pa < pb; };  // candidate.h:23-33
    sort_pairs<u8>(CP(0), CC(0), nc[0], cless);
    sort_pairs<u8>(CP(1), CC(1), nc[1], cless);
    // the read's base codes, forward and reverse-complemented, in this thread's column of shared memory (byte i of thread t at
    // [i][t]: conflict-free): both strands then run the SAME alignment code (a warp no longer splits by strand), and a column
    // of the band costs one shared-memory byte instead of a global load + decode
    extern __shared__ u8 v_codes[];
    const int NTB = blockDim.x;
    u8 *c_fwd = v_codes + threadIdx.x, *c_neg = v_codes + (size_t)c.maxmm * NTB + threadIdx.x;
    for (int i = 0; i < L; ++i) {
      const u32 b = base_code(read[i]);
      c_fwd[(size_t)i * NTB] = (u8)b;
      c_neg[(size_t)(L - 1 - i) * NTB] = (u8)(b < 4 ? 3u ^ b : 4u);
    }
    for (int s = 0; s < 2; ++s) {
      const u8 *txt = s == 0 ? c_fwd : c_neg;
      auto run_one = [&](u64 cpos) -> bool {  // returns true if the candidate failed (> e errors)
        const u32 rid = (u32)(cpos >> 32);
        const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
        const u8 *win = R.seq + R.off[rid] + pos - e;
        prefetch_span(win, L + 2 * e);
        int endp = 0;
        const int err = banded_align(e, L, [&](int i) { return base_code(__ldg(win + i)); }, [&](int i) { return (u32)txt[(size_t)i * NTB]; }, &endp);
        ++n_verified;
        if (err > e) return true;
        tally(t, err);
        if (nm[s] < c.mc) {
          MP(s)[nm[s]] = s == 0 ? cpos - (u64)e + (u64)endp : cpos - (u64)L + 1 - (u64)e + (u64)endp;
          ME(s)[nm[s]] = (short)err;
        }
        ++nm[s];
        return false;
      };
      if (nc[s] < P.lanes) {
        for (int i = 0; i < nc[s]; ++i) {
          const u64 cpos = CP(s)[i];
          const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
          if (!valid_cand(e, R.len[(u32)(cpos >> 32)], pos, (u32)L)) continue;
          run_one(cpos);
        }
        continue;
      }
      int group[8];
      int ng = 0;
      u32 threshold = 0;
      int ci = 0;
      while (ci < nc[s]) {
        if (CC(s)[ci] < threshold) break;
        const u64 cpos = CP(s)[ci];
        const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
        if (!valid_cand(e, R.len[(u32)(cpos >> 32)], pos, (u32)L)) { ++ci; continue; }
        group[ng++] = ci; ++ci;
        if (ng < P.lanes) continue;
        for (int g = 0; g < ng; ++g) if (run_one(CP(s)[group[g]])) threshold = CC(s)[group[g]];
        ng = 0;
      }
      for (int g = 0; g < ng; ++g) run_one(CP(s)[group[g]]);
    }
  }
  if (nm[0] > c.mc || nm[1] > c.mc) { S.pmeta[slot].status = ST_OVERFLOW; atomicAdd(&ctr->ovf_reason[6], 1ull); return; }
  rm.n_map[0] = nm[0]; rm.n_map[1] = nm[1];
  rm.min_err = t.min_err; rm.second_min_err = t.second_min_err; rm.n_best = t.n_best; rm.n_second_best = t.n_second_best;
  if (n_verified) agg_add(&ctr->n_verified, n_verified);
}

// ------------------------------------------------------------------------------------------------
// mapping_generator.h:346-484 (non-split): two-pointer sweep over end positions.  VISIT(i1, j, sum) is
// called for every in-window pair in the reference's enumeration order.  PA, EA: pointers or Strided views.
template <typename PA, typename EA, typename Visit>
__device__ __forceinline__ void pair_sweep(const DevParams &P, int s1, u32 L1, u32 L2, PA p1, EA e1, int n1, PA p2, EA e2, int n2, Visit VISIT) {
  int i1 = 0, i2 = 0;
  const u64 ins = (u64)P.max_insert, ovl = (u64)(u32)P.min_read_len;
  while (i1 < n1 && i2 < n2) {
    if ((s1 == 1 && p1[i1] > p2[i2] + ins - L2) || (s1 == 0 && p1[i1] > p2[i2] + L1 - ovl)) ++i2;
    else if ((s1 == 0 && p2[i2] > p1[i1] + ins - L1) || (s1 == 1 && p2[i2] > p1[i1] + L2 - ovl)) ++i1;
    else {
      int j = i2;
      while (j < n2 && ((s1 == 0 && p2[j] <= p1[i1] + ins - L1) || (s1 == 1 && p2[j] <= p1[i1] + L2 - ovl))) {
        VISIT(i1, j, (int)e1[i1] + (int)e2[j]);
        ++j;
      }
      ++i1;
    }
  }
}
// same enumeration, VISIT returns true to stop it
template <typename PA, typename EA, typename Visit>
__device__ __forceinline__ void pair_sweep_until(const DevParams &P, int s1, u32 L1, u32 L2, PA p1, EA e1, int n1, PA p2, EA e2, int n2, Visit VISIT) {
  int i1 = 0, i2 = 0;
  const u64 ins = (u64)P.max_insert, ovl = (u64)(u32)P.min_read_len;
  while (i1 < n1 && i2 < n2) {
    if ((s1 == 1 && p1[i1] > p2[i2] + ins - L2) || (s1 == 0 && p1[i1] > p2[i2] + L1 - ovl)) ++i2;
    else if ((s1 == 0 && p2[i2] > p1[i1] + ins - L1) || (s1 == 1 && p2[i2] > p1[i1] + L2 - ovl)) ++i1;
    else {
      int j = i2;
      while (j < n2 && ((s1 == 0 && p2[j] <= p1[i1] + ins - L1) || (s1 == 1 && p2[j] <= p1[i1] + L2 - ovl))) {
        if (VISIT(i1, j, (int)e1[i1] + (int)e2[j])) return;
        ++j;
      }
      ++i1;
    }
  }
}

// K4: per pair — SortMappingsByPositions (mapping_metadata.h:70-78) + best-pair statistics
// (mapping_generator.h:160-197).  pair_nbest[pair] = #best pairs if the pair reaches sampling/emit, else 0.
__global__ void pairing_kernel(DevParams P, Scratch S, int *pair_nbest) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status != ST_OK) { if (pm.status == ST_DROP) pair_nbest[pair] = 0; return; }
  ReadMeta *rm = S.rmeta + 2 * slot;
  if (P.se) {  // single-end: the read's own best / second-best tallies; mappings stay in verification order
    if (rm[0].n_map[0] + rm[0].n_map[1] == 0) { pm.status = ST_DROP; pair_nbest[pair] = 0; return; }
    pm.min_sum = rm[0].min_err; pm.second_min_sum = rm[0].second_min_err; pm.n_best = rm[0].n_best; pm.n_second_best = rm[0].n_second_best;
    pair_nbest[pair] = rm[0].n_best;
    return;
  }
  if (rm[0].n_map[0] + rm[0].n_map[1] == 0 || rm[1].n_map[0] + rm[1].n_map[1] == 0) { pm.status = ST_DROP; pair_nbest[pair] = 0; return; }
  // equal positions are interchangeable for the output; (pos, err) makes the order canonical
  auto mless = [](u64 pa, short ea, u64 pb, short eb) { return pa != pb ? pa < pb : ea < eb; };
  // (views rebuilt where they are used: arrays of them would live in local memory)
  auto MP = [&](int m, int s) { return map_pos_of(S, 2 * slot + m, s); };
  auto ME = [&](int m, int s) { return map_err_of(S, 2 * slot + m, s); };
  for (int m = 0; m < 2; ++m)
    for (int s = 0; s < 2; ++s) sort_pairs<short>(MP(m, s), ME(m, s), rm[m].n_map[s], mless);
  int min_sum = 2 * P.e + 1, second = 2 * P.e + 1, n_best = 0, n_second = 0;
  auto visit = [&](int, int, int sum) {
    if (sum < min_sum) { second = min_sum; n_second = n_best; min_sum = sum; n_best = 1; }
    else if (sum == min_sum) n_best++;
    else if (sum == second) n_second++;
    else if (sum < second) { second = sum; n_second = 1; }
  };
  pair_sweep(P, 0, (u32)rm[0].len, (u32)rm[1].len, MP(0, 0), ME(0, 0), rm[0].n_map[0], MP(1, 1), ME(1, 1), rm[1].n_map[1], visit);
  pair_sweep(P, 1, (u32)rm[0].len, (u32)rm[1].len, MP(0, 1), ME(0, 1), rm[0].n_map[1], MP(1, 0), ME(1, 0), rm[1].n_map[0], visit);
  pm.min_sum = min_sum; pm.second_min_sum = second; pm.n_best = n_best; pm.n_second_best = n_second;
  pair_nbest[pair] = (n_best > P.drop_rep) ? 0 : n_best;
}

// ------------------------------------------------------------------------------------------------
// K5: multi-mapper sampling (mapping_generator.h:199-214).  One warp per taskloop chunk: `generator`
// (chromap.h:863) is firstprivate in each task the taskloop (chromap.h:892) generates, so every chunk
// replays std::mt19937(11) from scratch, consumed by its pairs in index order.  The generator lives in shared
// memory and is advanced by the whole warp: a twist produces 624 tempered outputs at once (three dependency
// phases), and a run of reservoir draws uniform(0, i), uniform(0, i+1), ... consumes 32 outputs per step.
#define MT_N 624
struct WarpMt {
  u32 *mt;   // [624] state
  u32 *out;  // [624] tempered outputs of the current block
  int pos;   // next unread output (warp-uniform); MT_N = block exhausted
};
__device__ __forceinline__ u32 mt_mix(u32 a, u32 b, u32 c) {  // a = mt[i], b = mt[i+1], c = mt[i+397]
  const u32 y = (a & 0x80000000u) | (b & 0x7fffffffu);
  return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
__device__ __forceinline__ void mt_regen(WarpMt &g, int lane) {
  u32 *mt = g.mt;
  // new[i] = f(old[i], old[i+1], x[(i+397) % 624]) where x is already new for i >= 227
  // phase 1: i in [0,227) reads old mt[i], mt[i+1] (mt[227] for i=226 still old) and old mt[i+397]
  u32 v[8];
  int n = 0;
  for (int i = lane; i < 227; i += 32) v[n++] = mt_mix(mt[i], mt[i + 1], mt[i + 397]);
  __syncwarp();
  n = 0;
  for (int i = lane; i < 227; i += 32) mt[i] = v[n++];
  __syncwarp();
  // phase 2: i in [227,454): old mt[i], old mt[i+1] (mt[454] old), new mt[i-227]
  n = 0;
  for (int i = 227 + lane; i < 454; i += 32) v[n++] = mt_mix(mt[i], mt[i + 1], mt[i - 227]);
  __syncwarp();
  n = 0;
  for (int i = 227 + lane; i < 454; i += 32) mt[i] = v[n++];
  __syncwarp();
  // phase 3: i in [454,623): old mt[i], old mt[i+1], new mt[i-227]; i = 623 pairs with the NEW mt[0]
  n = 0;
  for (int i = 454 + lane; i < 623; i += 32) v[n++] = mt_mix(mt[i], mt[i + 1], mt[i - 227]);
  __syncwarp();
  n = 0;
  for (int i = 454 + lane; i < 623; i += 32) mt[i] = v[n++];
  __syncwarp();
  if (lane == 0) mt[623] = mt_mix(mt[623], mt[0], mt[396]);
  __syncwarp();
  for (int i = lane; i < MT_N; i += 32) {
    u32 y = mt[i];
    y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
    g.out[i] = y;
  }
  __syncwarp();
  g.pos = 0;
}
__device__ __forceinline__ u32 mt_next(WarpMt &g, int lane) {  // warp-uniform: every lane gets the same output
  if (g.pos >= MT_N) mt_regen(g, lane);
  return g.out[g.pos++];
}
// libstdc++ 13 std::uniform_int_distribution<int>(0, hi) on a 32-bit URNG: Lemire's nearly-divisionless
// method (bits/uniform_int_dist.h, _S_nd).  hi < 2^31.  Warp-uniform.
__device__ __forceinline__ u32 uniform_0_hi(WarpMt &g, int lane, u32 hi) {
  const u32 range = hi + 1u;
  u64 product = (u64)mt_next(g, lane) * (u64)range;
  u32 low = (u32)product;
  if (low < range) {
    const u32 threshold = (0u - range) % range;
    while (low < threshold) { product = (u64)mt_next(g, lane) * (u64)range; low = (u32)product; }
  }
  return (u32)(product >> 32);
}

// one warp per chunk: all lanes scan 32 pairs at a time and write the identity selection; for the pairs with
// more best pairs than -n the warp replays the reservoir sampling, 32 draws per step.  mt_init = the state of
// std::mt19937(11) right after seeding (624 words, computed once on the host).
__global__ void __launch_bounds__(128) select_kernel(DevParams P, int n_chunks, const int *chunk_start, const int *pair_nbest, int *pair_sel,
                                                     const u32 *mt_init) {
  __shared__ u32 s_mt[4][MT_N], s_out[4][MT_N];
  const int ch = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (ch >= n_chunks) return;
  WarpMt g;
  g.mt = s_mt[wid]; g.out = s_out[wid]; g.pos = MT_N;
  bool seeded = false;
  const int mb = P.max_best;
  const int p0 = chunk_start[ch], p1 = chunk_start[ch + 1];
  for (int base = p0; base < p1; base += 32) {
    const int pair = base + lane;
    int nb = 0;
    if (pair < p1) {
      nb = pair_nbest[pair];
      int *sel = pair_sel + (size_t)pair * mb;
      for (int j = 0; j < mb; ++j) sel[j] = j;
    }
    unsigned m = __ballot_sync(0xffffffffu, nb > mb);
    __syncwarp();
    while (m) {
      const int l = __ffs(m) - 1;
      m &= m - 1;
      const int nbl = __shfl_sync(0xffffffffu, nb, l);
      if (!seeded || P.se) {  // single-end: a fresh generator per read (mapping_generator.h:128)
        __syncwarp();
        for (int i = lane; i < MT_N; i += 32) g.mt[i] = mt_init[i];
        __syncwarp();
        g.pos = MT_N;
        seeded = true;
      }
      int *sel = pair_sel + (size_t)(base + l) * mb;
      int i = mb;
      while (i < nbl) {
        if (g.pos >= MT_N) mt_regen(g, lane);
        const int cnt = min(min(32, nbl - i), MT_N - g.pos);
        // draw i + lane takes output pos + lane, unless an earlier draw of this step needs Lemire's rejection test
        u64 product = 0;
        bool slow = false;
        if (lane < cnt) {
          const u32 range = (u32)(i + lane) + 1u;
          product = (u64)g.out[g.pos + lane] * (u64)range;
          slow = (u32)product < range;
        }
        const unsigned sm_ = __ballot_sync(0xffffffffu, slow);
        const int ok = sm_ ? __ffs(sm_) - 1 : cnt;  // draws i .. i+ok-1 accept their first output
        const int j = (int)(product >> 32);
        unsigned hit = __ballot_sync(0xffffffffu, lane < ok && j < mb);
        while (hit) {  // in draw order: a later draw overwrites an earlier one in the same reservoir slot
          const int t = __ffs(hit) - 1;
          hit &= hit - 1;
          const int jt = __shfl_sync(0xffffffffu, j, t);
          if (lane == 0) sel[jt] = i + t;
        }
        i += ok; g.pos += ok;
        if (ok < cnt) {  // one draw through the full rejection loop
          const int jj = (int)uniform_0_hi(g, lane, (u32)i);
          if (jj < mb && lane == 0) sel[jj] = i;
          ++i;
        }
        __syncwarp();
      }
      if (lane == 0) {
        for (int a = 1; a < mb; ++a) {  // std::sort of <= CMX_MAX_BEST ints
          const int v = sel[a];
          int b = a - 1;
          while (b >= 0 && sel[b] > v) { sel[b + 1] = sel[b]; --b; }
          sel[b + 1] = v;
        }
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// alignment.cc:656-718 — start coordinate.  PATC(i)/TXTC(i): raw chars (the Hamming shortcut compares raw
// chars, case-sensitively, :665-669); codes via base_code().
// the bit-vector part (alignment.cc:671-717), for the mappings whose mismatch count differs from their edit distance
template <typename PatC, typename TxtC>
__device__ __forceinline__ int banded_traceback_dp(int e, int min_err, int L, PatC PATC, TxtC TXTC) {
  PatPlanes W = {0u, 0u, 0u};
  for (int i = 0; i < 2 * e; ++i) planes_or(W, base_code(PATC(L - 1 + 2 * e - i)), 1u << i);
  const u32 hi = 1u << (2 * e), band = (hi << 1) - 1u;
  u32 VP = 0, VN = 0;
  int err = 0;
  for (int i = 0; i < L; ++i) {
    planes_or(W, base_code(PATC(L - 1 - i)), hi);
    u32 X = VN | planes_match(W, base_code(TXTC(L - 1 - i)), band);
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    VN = X & HP;
    VP = HN | ~(X | HP);
    err += 1 - (int)(D0 & 1u);
    planes_shift(W);
  }
  int start = 2 * e;
  for (int i = 0; i < 2 * e; ++i) {
    err += (int)((VP >> i) & 1u);
    err -= (int)((VN >> i) & 1u);
    if (err == min_err) { start = 2 * e - (1 + i); if (i + 1 == e) return start; }
  }
  return start;
}
template <typename PatC, typename TxtC>
__device__ __forceinline__ int banded_traceback(int e, int min_err, int L, PatC PATC, TxtC TXTC) {
  if (min_err == 0) return e;
  int ham = 0;
  for (int i = 0; i < L; ++i) if (PATC(i + e) != TXTC(i)) ++ham;
  if (ham == min_err) return e;
  return banded_traceback_dp(e, min_err, L, PATC, TXTC);
}

// IEEE double ops without FMA contraction: the reference is x86-64 SSE2 scalar code (no FMA).
__device__ __forceinline__ double xmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double xadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double xsub(double a, double b) { return __dadd_rn(a, -b); }
__device__ __forceinline__ double xdiv(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ int second_best_penalty(const MapqTables &T, int n) {  // (int)(4.343*log(n+1)+0.499)
  int v = 0;
  while (v + 1 < 96 && T.pen_thr[v + 1] <= n) ++v;
  return v;
}
__device__ __forceinline__ double rep_scale(double ident, double frac) {  // the 1 - f(frac_rep) factor
  if (ident <= 0.95) return xsub(1.0, __dsqrt_rn(frac));
  if (ident <= 0.97) return xsub(1.0, frac);
  if (ident >= 0.999) return xsub(1.0, xmul(xmul(xmul(frac, frac), frac), frac));
  return xsub(1.0, xmul(frac, frac));
}
// mapping_generator.h:920-1022 (non-split)
__device__ inline u8 mapq_se(const MapqTables &T, int num_errors, unsigned short aln_len, int read_len, int max_diff, const ReadMeta &rm) {
  const int coef_len = 50;
  aln_len = (unsigned short)((int)aln_len > read_len ? (int)aln_len : read_len);
  const double ident = xsub(1.0, xdiv((double)num_errors, (double)aln_len));
  int mapq = 0;
  int second = rm.second_min_err;
  if (rm.n_best > 1) {
  } else {
    if (second > num_errors + max_diff) second = num_errors + max_diff;
    double tmp = (int)aln_len < coef_len ? 1.0 : T.inv_log[aln_len];
    tmp = xmul(tmp, xmul(ident, ident));
    // 5 * 6.02 * (second - num_errors) * tmp * tmp + 0.499, left to right
    const double v = xadd(xmul(xmul(xmul(5 * 6.02, (double)(second - num_errors)), tmp), tmp), 0.499);
    mapq = (int)v;
  }
  if (rm.n_second_best > 0) mapq -= second_best_penalty(T, rm.n_second_best);
  if (mapq > 60) mapq = 60;
  if (mapq < 0) mapq = 0;
  if (rm.rep_len > 0) {
    double frac = xdiv((double)rm.rep_len, (double)read_len);
    if (rm.rep_len >= (u32)read_len) frac = 0.999;
    mapq = (int)xadd(xmul((double)mapq, rep_scale(ident, frac)), 0.499);
  }
  return (u8)mapq;
}
// mapping_generator.h:1027-1192 (non-split)
__device__ inline u8 mapq_pe(const MapqTables &T, int e1, int e2, unsigned short al1, unsigned short al2, int L1, int L2, int force,
                             const PairMeta &pm, const ReadMeta *rm) {
  u8 pe = 0;
  const int unpaired = rm[0].min_err + rm[1].min_err + 3;
  if (pm.n_best <= 1) {
    const int adj = pm.second_min_sum < unpaired ? pm.second_min_sum : unpaired;
    pe = (u8)(int)xadd(xdiv(xmul(5 * 6.02, (double)(adj - pm.min_sum)), 1.0), .499);
    if (pm.n_second_best > 0) pe = (u8)((int)pe - second_best_penalty(T, pm.n_second_best));  // uint8 wrap (:1073)
    if (pe > 60) pe = 60;
    const int rep = (int)(rm[0].rep_len + rm[1].rep_len);
    if (rep > 0) {
      const double total = (double)(L1 + L2);
      double frac = xdiv((double)rep, total);
      if ((double)rep >= total) frac = 0.999;
      const double id1 = xsub(1.0, xdiv((double)e1, (double)(L1 > (int)al1 ? L1 : (int)al1)));
      const double id2 = xsub(1.0, xdiv((double)e2, (double)(L2 > (int)al2 ? L2 : (int)al2)));
      const double ident = id1 < id2 ? id1 : id2;
      pe = (u8)xadd(xmul((double)pe, rep_scale(ident, frac)), 0.499);
    }
  }
  u8 q1 = mapq_se(T, e1, al1, L1, 2, rm[0]);
  u8 q2 = mapq_se(T, e2, al2, L2, 2, rm[1]);
  {
    const double a = xadd((double)q1, xmul((double)pe, 0.65));
    q1 = q1 > pe ? q1 : ((double)pe < a ? pe : (u8)a);
    const double b = xadd((double)q2, xmul((double)pe, 0.65));
    q2 = q2 > pe ? q2 : ((double)pe < b ? pe : (u8)b);
  }
  q1 = (u8)xmul((double)q1, 1.2); if (q1 > 60) q1 = 60;
  q2 = (u8)xmul((double)q2, 1.2); if (q2 > 60) q2 = 60;
  u8 q = q1 < q2 ? q1 : q2;
  if (q < 60 && force >= 0 && force < q) q = (u8)force;
  return q;
}

struct OutRecord {  // == cmx_pe_record
  u32 read_id, rid, fragment_start;
  unsigned short fragment_length;
  u8 mapq, direction, is_unique, num_dups;
  unsigned short positive_alignment_length, negative_alignment_length;
};

// start / end of one mate's mapping on the reference: GetRefStartEndPositionForReadFromMapping, BED branch
// (mapping_generator.h:657-917).  r = the mate's bases as read (the reverse strand is formed on the fly).
__device__ __forceinline__ void mapping_span(const DevRef &R, int e, const u8 *r, int Lm, int s, u64 dpos, int derr, u32 *st, u32 *en) {
  const u32 rid = (u32)(dpos >> 32), rp = (u32)dpos;
  u32 vws = rp + 1u > (u32)(Lm + e) ? rp + 1u - (u32)Lm - (u32)e : 0u;
  if (rp + (u32)e >= R.len[rid]) vws = R.len[rid] - (u32)e - (u32)Lm;
  const u8 *win = R.seq + R.off[rid] + vws;
  if (derr != 0) { prefetch_span(win, Lm + 2 * e); prefetch_span(r, Lm); }
  int s0;
  if (s == 0) s0 = banded_traceback(e, derr, Lm, [&](int i) { return __ldg(win + i); }, [&](int i) { return r[i]; });
  else s0 = banded_traceback(e, derr, Lm, [&](int i) { return __ldg(win + i); }, [&](int i) { return code_char(neg_code(r, Lm, i)); });
  *st = vws + (u32)s0;
  *en = rp;
}
// one paired-end record (mapping_generator.cc:110-143) from the chosen draft mappings of the two mates; s1 = strand of mate 1
__device__ __forceinline__ OutRecord pe_record(const DevParams &P, const DevRef &R, const DevBatch &B, const MapqTables &T, const PairMeta &pm, const ReadMeta *rm,
                                               int pair, int s1, u64 pos1, int err1, u64 pos2, int err2) {
  const int L0 = rm[0].len, L1 = rm[1].len;
  u32 st1, en1, st2, en2;
  mapping_span(R, P.e, read_ptr(B, pair, 0), L0, s1, pos1, err1, &st1, &en1);
  mapping_span(R, P.e, read_ptr(B, pair, 1), L1, 1 - s1, pos2, err2, &st2, &en2);
  const unsigned short al1 = (unsigned short)(en1 - st1 + 1u), al2 = (unsigned short)(en2 - st2 + 1u);
  OutRecord o;
  o.read_id = B.first_read_id + (u32)pair;
  o.rid = (u32)(pos1 >> 32);
  o.fragment_start = s1 == 0 ? st1 : st2;
  o.fragment_length = (unsigned short)(s1 == 0 ? (int)(en2 - st1 + 1u) : (int)(en1 - st2 + 1u));
  o.mapq = mapq_pe(T, err1, err2, al1, al2, L0, L1, pm.sup != 0 ? 0 : -1, pm, rm);
  o.direction = s1 == 0 ? 1 : 0;
  o.is_unique = (pm.n_best == 1 || rm[0].n_best == 1 || rm[1].n_best == 1) ? 1 : 0;
  o.num_dups = 1;
  o.positive_alignment_length = s1 == 0 ? al1 : al2;
  o.negative_alignment_length = s1 == 1 ? al1 : al2;
  return o;
}

// K6: per pair — ProcessBestMappingsForPairedEndReadOnOneDirection (mapping_generator.h:486-654):
// the selected best pair(s), start coordinates (mapping_generator.h:657-917 BED branch), MAPQ, record.
// One thread per pair, but the warp works through the expensive parts together, in phases:
//   A  every thread walks its sweep to the selected best pair(s) and notes which mappings they are;
//   B  the Hamming shortcut of BandedTraceback (alignment.cc:665-669) for every (pair, mate) whose mapping has errors: the
//      warp takes these one at a time, 32 positions per step, window and read bytes coalesced;
//   C  the threads whose mismatch count differs from the edit distance (indels) run the bit-vector traceback side by side;
//   D  MAPQ and the record.
// (Computed inside the sweep, each thread reached its traceback at a different iteration and the warp ran them one after
// the other: 3.5 active lanes per instruction, 2 ms for 2 M pairs.)
__global__ void emit_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, const int *pair_sel, OutRecord *out,
                            int *out_n, Counters *ctr, int4 *dp_list, int *dp_count) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  const bool in_range = slot < S.n_slots;
  const int sl = in_range ? slot : 0;
  PairMeta &pm = S.pmeta[sl];
  const int pair = slot_pair(S, sl);
  const ReadMeta *rm = S.rmeta + 2 * sl;
  const int mb = P.max_best, e = P.e;
  int reported = 0;
  int ch_i1[CMX_MAX_BEST], ch_j[CMX_MAX_BEST];  // chosen mappings; bit 30 of ch_i1 = direction
  bool live = in_range && pm.status != ST_OVERFLOW;  // overflow: re-done in the large tier (or reported)
  if (live && (pm.status != ST_OK || pm.n_best > P.drop_rep || pm.n_best == 0)) { out_n[pair] = 0; live = false; }
  if (live) {  // phase A
    const int to_report = mb < pm.n_best ? mb : pm.n_best;
    const int *sel = pair_sel + (size_t)pair * mb;
    int idx = 0;
    for (int dir = 0; dir < 2 && reported != to_report; ++dir) {
      const int s1 = dir, s2 = 1 - dir;
      pair_sweep_until(P, s1, (u32)rm[0].len, (u32)rm[1].len, map_pos_of(S, 2 * slot, s1), map_err_of(S, 2 * slot, s1), rm[0].n_map[s1], map_pos_of(S, 2 * slot + 1, s2),
                       map_err_of(S, 2 * slot + 1, s2), rm[1].n_map[s2], [&](int i1, int j, int sum) -> bool {
        if (sum != pm.min_sum) return false;
        if (idx == sel[reported]) { ch_i1[reported] = i1 | (dir << 30); ch_j[reported] = j; ++reported; }
        ++idx;
        return reported == to_report;
      });
    }
  }
  const int L[2] = {live ? rm[0].len : 0, live ? rm[1].len : 0};
  const int max_rep = __reduce_max_sync(0xffffffffu, reported);
  for (int r = 0; r < max_rep; ++r) {
    const bool have = r < reported;
    int s1 = 0;
    u64 dpos[2] = {0, 0};
    int derr[2] = {0, 0};
    u32 vws[2] = {0, 0};
    const u8 *win[2] = {R.seq, R.seq};
    const u8 *rd[2] = {R.seq, R.seq};
    int s0[2] = {e, e};
    if (have) {
      s1 = ch_i1[r] >> 30;
      const int i1 = ch_i1[r] & 0x3FFFFFFF, j = ch_j[r];
      dpos[0] = map_pos_of(S, 2 * slot, s1)[i1]; derr[0] = map_err_of(S, 2 * slot, s1)[i1];
      dpos[1] = map_pos_of(S, 2 * slot + 1, 1 - s1)[j]; derr[1] = map_err_of(S, 2 * slot + 1, 1 - s1)[j];
#pragma unroll
      for (int m = 0; m < 2; ++m) {  // verification window (mapping_generator.h:696-711)
        const u32 rid = (u32)(dpos[m] >> 32), rp = (u32)dpos[m];
        u32 v = rp + 1u > (u32)(L[m] + e) ? rp + 1u - (u32)L[m] - (u32)e : 0u;
        if (rp + (u32)e >= R.len[rid]) v = R.len[rid] - (u32)e - (u32)L[m];
        vws[m] = v;
        win[m] = R.seq + R.off[rid] + v;
        rd[m] = read_ptr(B, pair, m);
      }
    }
    // phase B: mismatch counts by the whole warp, four (pair, mate) tasks per round so that their loads are in flight together
    int ham[2] = {0, 0};
#pragma unroll
    for (int m = 0; m < 2; ++m) {
      unsigned todo = __ballot_sync(0xffffffffu, have && derr[m] > 0);
      while (todo) {
        int src[4], cnt[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          src[t] = todo ? __ffs(todo) - 1 : -1;
          if (todo) todo &= todo - 1;
          cnt[t] = 0;
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          if (src[t] < 0) continue;  // warp-uniform
          const u8 *w = (const u8 *)__shfl_sync(0xffffffffu, (unsigned long long)win[m], src[t]);
          const u8 *q = (const u8 *)__shfl_sync(0xffffffffu, (unsigned long long)rd[m], src[t]);
          const int Lm = __shfl_sync(0xffffffffu, L[m], src[t]);
          const int neg = __shfl_sync(0xffffffffu, m == 0 ? s1 : 1 - s1, src[t]);
          for (int i = lane; i < Lm; i += 32) {
            const u8 a = __ldg(w + i + e);
            const u8 c0 = neg ? q[Lm - 1 - i] : q[i];
            const u32 bc = base_code(c0);
            const u8 tch = neg ? code_char(bc < 4 ? 3u ^ bc : 4u) : c0;  // the reverse strand string holds A C G T N only (sequence_batch.h:123-134)
            cnt[t] += a != tch;
          }
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          if (src[t] < 0) continue;
          const int c_ = __reduce_add_sync(0xffffffffu, cnt[t]);
          if (lane == src[t]) ham[m] = c_;
        }
      }
    }
    // phase C: mappings whose mismatch count differs from their edit distance (indels, ~5 % of reads) need the bit-vector
    // traceback: those pairs are put on a list and finished by emit_dp_kernel, one lane each, densely packed — inside this
    // kernel a warp would run a 50-column traceback for its one or two such lanes at a time
    const bool deferred = have && ((derr[0] > 0 && ham[0] != derr[0]) || (derr[1] > 0 && ham[1] != derr[1]));
    if (deferred) dp_list[agg_append(dp_count)] = make_int4(slot, r, ch_i1[r], ch_j[r]);
    if (have && !deferred) {  // phase D (mapping_generator.cc:110-143)
      const u32 st1 = vws[0] + (u32)s0[0], en1 = (u32)dpos[0], st2 = vws[1] + (u32)s0[1], en2 = (u32)dpos[1];
      const unsigned short al1 = (unsigned short)(en1 - st1 + 1u), al2 = (unsigned short)(en2 - st2 + 1u);
      OutRecord o;
      o.read_id = B.first_read_id + (u32)pair;
      o.rid = (u32)(dpos[0] >> 32);
      o.fragment_start = s1 == 0 ? st1 : st2;
      o.fragment_length = (unsigned short)(s1 == 0 ? (int)(en2 - st1 + 1u) : (int)(en1 - st2 + 1u));
      o.mapq = mapq_pe(T, derr[0], derr[1], al1, al2, L[0], L[1], pm.sup != 0 ? 0 : -1, pm, rm);
      o.direction = s1 == 0 ? 1 : 0;
      o.is_unique = (pm.n_best == 1 || rm[0].n_best == 1 || rm[1].n_best == 1) ? 1 : 0;
      o.num_dups = 1;
      o.positive_alignment_length = s1 == 0 ? al1 : al2;
      o.negative_alignment_length = s1 == 1 ? al1 : al2;
      out[(size_t)pair * mb + r] = o;
    }
  }
  if (!live) return;
  out_n[pair] = reported;
  pm.n_rec = reported;
  if (reported > 0) { agg_add(&ctr->n_mapped, 1ull); if (pm.n_best == 1) agg_add(&ctr->n_unique, 1ull); }
}

// the pairs emit_kernel left: one thread each, record computed with the full BandedTraceback
__global__ void emit_dp_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, OutRecord *out, const int4 *dp_list, const int *dp_count) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= *dp_count) return;
  const int4 q = dp_list[t];
  const int slot = q.x, r = q.y, s1 = q.z >> 30, i1 = q.z & 0x3FFFFFFF, j = q.w;
  const int pair = slot_pair(S, slot);
  out[(size_t)pair * P.max_best + r] = pe_record(P, R, B, T, S.pmeta[slot], S.rmeta + 2 * slot, pair, s1, map_pos_of(S, 2 * slot, s1)[i1], map_err_of(S, 2 * slot, s1)[i1],
                                                 map_pos_of(S, 2 * slot + 1, 1 - s1)[j], map_err_of(S, 2 * slot + 1, 1 - s1)[j]);
}

// compaction of per-pair records into read order
// Single-end emit: ProcessBestMappingsForSingleEndRead (mapping_generator.h:256-343) + EmplaceBackSingleEndMappingRecord
// (mapping_generator.cc:7-16).  + strand mappings first, then - strand, in verification order.
__global__ void emit_se_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, const int *pair_sel, OutRecord *out, int *out_n,
                               Counters *ctr) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status == ST_OVERFLOW) return;
  if (pm.status != ST_OK || pm.n_best == 0) { out_n[pair] = 0; return; }
  const ReadMeta &rm = S.rmeta[2 * slot];
  const int mb = P.max_best, e = P.e, L = rm.len;
  const int to_report = mb < rm.n_best ? mb : rm.n_best;
  const int *sel = pair_sel + (size_t)pair * mb;
  const u8 *r = read_ptr(B, pair, 0);
  int idx = 0, reported = 0;
  for (int s = 0; s < 2 && reported != to_report; ++s) {
    const Strided<u64> mp = map_pos_of(S, 2 * slot, s);
    const Strided<short> me = map_err_of(S, 2 * slot, s);
    for (int mi = 0; mi < rm.n_map[s]; ++mi) {
      if ((int)me[mi] > rm.min_err) continue;
      if (idx == sel[reported]) {
        const u64 dpos = mp[mi];
        const u32 rid = (u32)(dpos >> 32), rp = (u32)dpos;
        u32 vws = rp + 1u > (u32)(L + e) ? rp + 1u - (u32)L - (u32)e : 0u;
        if (rp + (u32)e >= R.len[rid]) vws = R.len[rid] - (u32)e - (u32)L;
        const u8 *win = R.seq + R.off[rid] + vws;
        int s0;
        if (s == 0) s0 = banded_traceback(e, (int)me[mi], L, [&](int i) { return __ldg(win + i); }, [&](int i) { return r[i]; });
        else s0 = banded_traceback(e, (int)me[mi], L, [&](int i) { return __ldg(win + i); }, [&](int i) { return code_char(neg_code(r, L, i)); });
        const u32 st = vws + (u32)s0;
        const unsigned short al = (unsigned short)(rp - st + 1u);
        OutRecord o;
        o.read_id = B.first_read_id + (u32)pair;
        o.rid = rid;
        o.fragment_start = st;
        o.fragment_length = al;
        o.mapq = mapq_se(T, (int)me[mi], al, L, e, rm);
        o.direction = s == 0 ? 1 : 0;
        o.is_unique = rm.n_best == 1 ? 1 : 0;
        o.num_dups = 1;
        o.positive_alignment_length = 0;
        o.negative_alignment_length = 0;
        out[(size_t)pair * mb + reported] = o;
        if (++reported == to_report) break;
      }
      ++idx;
    }
  }
  out_n[pair] = reported;
  pm.n_rec = reported;
  if (reported > 0) { agg_add(&ctr->n_mapped, 1ull); if (rm.n_best == 1) agg_add(&ctr->n_unique, 1ull); }
}

__global__ void compact_kernel(int n_pairs, int mb, const OutRecord *in, const int *n_rec, const u64 *offs, OutRecord *out) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= n_pairs) return;
  const int n = n_rec[pair];
  for (int j = 0; j < n; ++j) out[offs[pair] + j] = in[(size_t)pair * mb + j];
}

// collect pairs whose small-tier run overflowed
__global__ void collect_overflow_kernel(Scratch S, int *list, int *count) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  if (S.pmeta[slot].status == ST_OVERFLOW) list[agg_append(count)] = slot_pair(S, slot);
}

// =================================================================================================
// CTA-cooperative kernels for the overflow tiers (one CTA per read / per pair).  Same scratch layout and
// the same results as the general kernels; the expensive primitives — table probes, hit expansion,
// sorting, banded verification — are spread over the CTA's threads, the order-dependent scans stay on
// thread 0 and read their input through shared memory.
#define CTA_NT 128
#define CTA_SORT_SMEM_MAX 4096  // u64 entries staged in shared memory at most (32 KB); the launch picks the tier's size
#define CTA_MM_SMEM 1024    // max minimizers per read handled by the CTA kernels

// ascending bitonic sort of n keys; pads a[n..np2) with ~0 (capacity must be a power of two >= n).
// Lists that fit the shared-memory buffer are sorted there; longer ones run the sub-steps with stride >=
// sm_cap in global memory and finish every tile of sm_cap keys in shared memory (10 global passes instead of
// 136 for 65536 keys).
__device__ inline void cta_sort_keys(u64 *a, int n, u64 *sm, int sm_cap) {
  const int NT = blockDim.x;  // 32 .. CTA_NT threads
  int np2 = 1;
  while (np2 < n) np2 <<= 1;
  const int tid = threadIdx.x;
  if (n <= 1) { __syncthreads(); return; }
  if (np2 <= sm_cap) {
    for (int i = tid; i < np2; i += NT) sm[i] = i < n ? a[i] : ~0ull;
    __syncthreads();
    for (int k = 2; k <= np2; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int p = tid; p < (np2 >> 1); p += NT) {
          const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i + j;  // j is a power of two
          const u64 x = sm[i], y = sm[l];
          const bool up = (i & k) == 0;
          if ((x > y) == up) { sm[i] = y; sm[l] = x; }
        }
        __syncthreads();
      }
    for (int i = tid; i < n; i += NT) a[i] = sm[i];
    __syncthreads();
    return;
  }
  for (int i = n + tid; i < np2; i += NT) a[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    int j = k >> 1;
    for (; j >= sm_cap; j >>= 1) {  // wide strides: global memory
      for (int p = tid; p < (np2 >> 1); p += NT) {
        const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i + j;  // j is a power of two
        const u64 x = a[i], y = a[l];
        const bool up = (i & k) == 0;
        if ((x > y) == up) { a[i] = y; a[l] = x; }
      }
      __syncthreads();
    }
    // remaining strides (< sm_cap) stay inside tiles of sm_cap keys: finish each tile in shared memory.
    // (when k <= sm_cap this also covers the whole k-stage; consecutive small k stages are fused per tile)
    const bool fuse = k <= sm_cap;
    for (int base = 0; base < np2; base += sm_cap) {
      for (int i = tid; i < sm_cap; i += NT) sm[i] = a[base + i];
      __syncthreads();
      const int k_lo = fuse ? 2 : k, k_hi = fuse ? sm_cap : k;
      for (int kk = k_lo; kk <= k_hi; kk <<= 1)
        for (int jj = fuse ? (kk >> 1) : j; jj > 0; jj >>= 1) {
          for (int p = tid; p < (sm_cap >> 1); p += NT) {
            const int i = ((p & ~(jj - 1)) << 1) | (p & (jj - 1)), l = i + jj;
            const u64 x = sm[i], y = sm[l];
            const bool up = ((base + i) & kk) == 0;
            if ((x > y) == up) { sm[i] = y; sm[l] = x; }
          }
          __syncthreads();
        }
      for (int i = tid; i < sm_cap; i += NT) a[base + i] = sm[i];
      __syncthreads();
    }
    if (fuse) k = sm_cap;  // stages 2..sm_cap are done
  }
}

// same for (key, tag) pairs under `less`; pads with (pad_key, pad_tag) which must compare greatest.
template <typename T, typename Less>
__device__ inline void cta_sort_pairs(u64 *k_, T *t_, int n, u64 pad_key, T pad_tag, Less less, u64 *smk, T *smt, int sm_cap) {
  const int NT = blockDim.x;
  int np2 = 1;
  while (np2 < n) np2 <<= 1;
  const int tid = threadIdx.x;
  if (n <= 1) { __syncthreads(); return; }
  if (np2 <= sm_cap) {
    for (int i = tid; i < np2; i += NT) { smk[i] = i < n ? k_[i] : pad_key; smt[i] = i < n ? t_[i] : pad_tag; }
    __syncthreads();
    for (int k = 2; k <= np2; k <<= 1)
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int p = tid; p < (np2 >> 1); p += NT) {
          const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i + j;  // j is a power of two
          const u64 xk = smk[i], yk = smk[l];
          const T xt = smt[i], yt = smt[l];
          const bool up = (i & k) == 0;
          const bool sw = up ? less(yk, yt, xk, xt) : less(xk, xt, yk, yt);
          if (sw) { smk[i] = yk; smt[i] = yt; smk[l] = xk; smt[l] = xt; }
        }
        __syncthreads();
      }
    for (int i = tid; i < n; i += NT) { k_[i] = smk[i]; t_[i] = smt[i]; }
    __syncthreads();
    return;
  }
  for (int i = n + tid; i < np2; i += NT) { k_[i] = pad_key; t_[i] = pad_tag; }
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1) {
    int j = k >> 1;
    for (; j >= sm_cap; j >>= 1) {
      for (int p = tid; p < (np2 >> 1); p += NT) {
        const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), l = i + j;  // j is a power of two
        const u64 xk = k_[i], yk = k_[l];
        const T xt = t_[i], yt = t_[l];
        const bool up = (i & k) == 0;
        const bool sw = up ? less(yk, yt, xk, xt) : less(xk, xt, yk, yt);
        if (sw) { k_[i] = yk; t_[i] = yt; k_[l] = xk; t_[l] = xt; }
      }
      __syncthreads();
    }
    const bool fuse = k <= sm_cap;
    for (int base = 0; base < np2; base += sm_cap) {
      for (int i = tid; i < sm_cap; i += NT) { smk[i] = k_[base + i]; smt[i] = t_[base + i]; }
      __syncthreads();
      const int k_lo = fuse ? 2 : k, k_hi = fuse ? sm_cap : k;
      for (int kk = k_lo; kk <= k_hi; kk <<= 1)
        for (int jj = fuse ? (kk >> 1) : j; jj > 0; jj >>= 1) {
          for (int p = tid; p < (sm_cap >> 1); p += NT) {
            const int i = ((p & ~(jj - 1)) << 1) | (p & (jj - 1)), l = i + jj;
            const u64 xk = smk[i], yk = smk[l];
            const T xt = smt[i], yt = smt[l];
            const bool up = ((base + i) & kk) == 0;
            const bool sw = up ? less(yk, yt, xk, xt) : less(xk, xt, yk, yt);
            if (sw) { smk[i] = yk; smt[i] = yt; smk[l] = xk; smt[l] = xt; }
          }
          __syncthreads();
        }
      for (int i = tid; i < sm_cap; i += NT) { k_[base + i] = smk[i]; t_[base + i] = smt[i]; }
      __syncthreads();
    }
    if (fuse) k = sm_cap;
  }
}

// candidate_processor.cc:283-342 with the sorted hits streamed through shared memory; thread 0 scans.
// Returns the candidate count on every thread.
__device__ inline int cta_cluster(int e, int need, u32 n_mm, const u64 *hits, int nh, u64 *cpos, u8 *ccnt, int cap, u64 *sm, int sm_cap, int *s_ret) {
  const int NT = blockDim.x;  // 32 .. CTA_NT threads
  const int tid = threadIdx.x;
  int n = 0, mcount = 1, eq = 1, best_eq = 1;
  u64 prev = 0, best = 0;
  u32 prev_rid = 0, prev_pos = 0;
  for (int base = 0; base < nh; base += sm_cap) {
    const int m = min(sm_cap, nh - base);
    for (int i = tid; i < m; i += NT) sm[i] = hits[base + i];
    __syncthreads();
    if (tid == 0) {
      int i0 = 0;
      if (base == 0) { prev = sm[0]; best = prev; prev_rid = (u32)(prev >> 32); prev_pos = (u32)prev; i0 = 1; }
      for (int i = i0; i <= m; ++i) {
        if (i == m && base + m < nh) break;  // more chunks follow
        const u64 h = i < m ? sm[i] : ~0ull;  // final sentinel
        const u32 rid = (u32)(h >> 32), pos = (u32)h;
        if (rid != prev_rid || pos > prev_pos + (u32)e || ((u32)mcount >= n_mm && pos > (u32)best + (u32)e)) {
          if (mcount >= need) { if (n < cap) { cpos[n] = best; ccnt[n] = (u8)best_eq; } ++n; }
          mcount = 1; eq = 1; best_eq = 1; best = h;
        } else {
          if (h == best) { ++eq; ++best_eq; }
          else if (h == prev) { ++eq; if (eq > best_eq) { best = prev; best_eq = eq; } }
          else eq = 1;
          ++mcount;
        }
        prev = h; prev_rid = rid; prev_pos = pos;
      }
    }
    __syncthreads();
  }
  if (tid == 0) *s_ret = n;
  __syncthreads();
  const int r = *s_ret;
  __syncthreads();
  return r;
}

// Minimizer emission (minimizer_generator.cc:66-138) from per-position seeds computed in parallel, for reads
// without ambiguous bases (run length == position + 1) and odd k (no strand-symmetric k-mers).
template <int W>
__device__ __forceinline__ int emit_minimizers_from_seeds(const u64 *sh, const u32 *sp, int len, int k, u64 *out_hash, u32 *out_pos, int cap) {
  u64 rh[W];
  u32 rp[W];
#pragma unroll
  for (int i = 0; i < W; ++i) { rh[i] = ~0ull; rp[i] = ~0u; }
  u64 best_h = ~0ull;
  u32 best_p = ~0u;
  int best_age = 0, n = 0;
#define EMIT(h, p) do { if (n < cap) { out_hash[n] = (h); out_pos[n] = (p); } ++n; } while (0)
  for (int pos = 0; pos < len; ++pos) {
    const int run = pos + 1;
    const u64 cur_h = sh[pos];
    const u32 cur_p = sp[pos];
#pragma unroll
    for (int j = 0; j + 1 < W; ++j) { rh[j] = rh[j + 1]; rp[j] = rp[j + 1]; }
    rh[W - 1] = cur_h; rp[W - 1] = cur_p;
    ++best_age;
    if (run == W + k - 1 && best_h != ~0ull && best_h < cur_h) {
#pragma unroll
      for (int j = 0; j + 1 < W; ++j) if (best_h == rh[j] && rp[j] != best_p) EMIT(rh[j], rp[j]);
    }
    if (cur_h <= best_h) {
      if (run >= W + k && best_h != ~0ull) EMIT(best_h, best_p);
      best_h = cur_h; best_p = cur_p; best_age = 0;
    } else if (best_age == W) {
      if (run >= W + k - 1 && best_h != ~0ull) EMIT(best_h, best_p);
      best_h = ~0ull;
#pragma unroll
      for (int j = 0; j < W; ++j) if (best_h >= rh[j]) { best_h = rh[j]; best_p = rp[j]; best_age = W - 1 - j; }
      if (run >= W + k - 1 && best_h != ~0ull) {
#pragma unroll
        for (int j = 0; j < W; ++j) if (best_h == rh[j] && best_p != rp[j]) EMIT(rh[j], rp[j]);
      }
    }
  }
  if (best_h != ~0ull) EMIT(best_h, best_p);
#undef EMIT
  return n;
}

// CTA minimizers: every thread hashes the k-mers ending at its positions (3 x Hash64 each), thread 0 replays the
// window logic over the seeds.  Falls back to the one-thread generator for reads with ambiguous bases, even k or
// an unusual w.  `work` is scratch shared memory of at least len * 13 bytes.  Returns n_mm on thread 0 only.
__device__ inline int cta_minimizers(const u8 *seq, int len, int k, int w, u64 *out_hash, u32 *out_pos, int cap, u64 *work, int *s_flag) {
  const int tid = threadIdx.x;
  u64 *sh = work;
  u32 *sp = (u32 *)(work + len);
  u8 *sc = (u8 *)(sp + len);
  if (tid == 0) *s_flag = ((k & 1) && (w == 7 || w == 10 || w == 11)) ? 1 : 0;
  __syncthreads();
  for (int p = tid; p < len; p += CTA_NT) { const u32 c = base_code(seq[p]); sc[p] = (u8)c; if (c > 3) *s_flag = 0; }
  __syncthreads();
  const bool fast = *s_flag != 0;
  if (fast) {
    const u64 mask = (((u64)1) << (2 * k)) - 1;
    for (int p = tid; p < len; p += CTA_NT) {
      u64 h = ~0ull;
      u32 pp = ~0u;
      if (p >= k - 1) {
        u64 fwd = 0, rev = 0;
        for (int i = 0; i < k; ++i) { const u64 b = sc[p - k + 1 + i]; fwd = (fwd << 2) | b; rev |= (3ull ^ b) << (2 * i); }
        const u64 hf = mix64(fwd, mask), hr = mix64(rev, mask);
        const u32 strand = hf < hr ? 0u : 1u;
        h = mix64(strand ? hr : hf, mask);
        pp = ((u32)p << 1) | strand;
      }
      sh[p] = h; sp[p] = pp;
    }
  }
  __syncthreads();
  int n = 0;
  if (tid == 0) {
    if (!fast) minimizer_scan_any([&](int i) { return seq[i]; }, len, k, w, [&](u64 h, u32 p_) { if (n < cap) { out_hash[n] = h; out_pos[n] = p_; } ++n; });
    else if (w == 7) n = emit_minimizers_from_seeds<7>(sh, sp, len, k, out_hash, out_pos, cap);
    else if (w == 10) n = emit_minimizers_from_seeds<10>(sh, sp, len, k, out_hash, out_pos, cap);
    else n = emit_minimizers_from_seeds<11>(sh, sp, len, k, out_hash, out_pos, cap);
  }
  __syncthreads();
  return n;
}

// exclusive scan of one int per thread over the CTA; *total gets the sum.
__device__ inline int cta_excl_scan(int v, int *s_warp, int *total) {
  const int NT = blockDim.x;  // 32 .. CTA_NT threads
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  int base = 0;
  for (int i = 0; i < wid; ++i) base += s_warp[i];
  int tot = 0;
  for (int i = 0; i < (NT >> 5); ++i) tot += s_warp[i];
  __syncthreads();
  *total = tot;
  return base + x - v;
}

// candidate_processor.cc:283-342 in parallel.  A new cluster always starts where the reference id changes or
// the gap to the previous hit exceeds e — those boundaries depend only on neighbouring hits, so the list splits
// into independent segments; the third, state-dependent rule (a cluster that already holds >= n_mm hits and
// drifts more than e from its best hit) is applied by the thread that scans the segment.  Candidates are
// written in place (a segment yields at most one candidate per hit consumed) and compacted in hit order.
// Lists longer than the shared-memory tile use the streaming version above.  `aux` = 3 * sm_cap bytes.
__device__ inline int cta_cluster_par(int e, int need, u32 n_mm, const u64 *hits, int nh, u64 *cpos, u8 *ccnt, int cap, u64 *sm, int sm_cap,
                                      u8 *aux, int *s_ret) {
  const int NT = blockDim.x;  // 32 .. CTA_NT threads
  if (nh > sm_cap) return cta_cluster(e, need, n_mm, hits, nh, cpos, ccnt, cap, sm, sm_cap, s_ret);
  const int tid = threadIdx.x;
  u8 *flag = aux, *vld = aux + sm_cap, *cnt = aux + 2 * sm_cap;
  for (int i = tid; i < nh; i += NT) sm[i] = hits[i];
  __syncthreads();
  for (int i = tid; i < nh; i += NT) {
    bool b = i == 0;
    if (!b) {
      const u64 h = sm[i], q = sm[i - 1];
      b = (u32)(h >> 32) != (u32)(q >> 32) || (u32)h > (u32)q + (u32)e;
    }
    flag[i] = b; vld[i] = 0;
  }
  __syncthreads();
  const int C = (nh + NT - 1) / NT;
  const int r0 = tid * C, r1 = min(nh, r0 + C);
  for (int i = r0; i < r1; ++i) {
    if (!flag[i]) continue;
    int out = i, mcount = 1, eq = 1, best_eq = 1;
    u64 prev = sm[i], best = prev;
    int q = i + 1;
    for (; q < nh && !flag[q]; ++q) {
      const u64 h = sm[q];
      if ((u32)mcount >= n_mm && (u32)h > (u32)best + (u32)e) {
        if (mcount >= need) { sm[out] = best; cnt[out] = (u8)best_eq; vld[out] = 1; ++out; }
        mcount = 1; eq = 1; best_eq = 1; best = h;
      } else {
        if (h == best) { ++eq; ++best_eq; }
        else if (h == prev) { ++eq; if (eq > best_eq) { best = prev; best_eq = eq; } }
        else eq = 1;
        ++mcount;
      }
      prev = h;
    }
    if (mcount >= need) { sm[out] = best; cnt[out] = (u8)best_eq; vld[out] = 1; ++out; }
  }
  __syncthreads();
  int mine = 0;
  for (int i = r0; i < r1; ++i) mine += vld[i];
  __shared__ int s_warp[32];  // (up to 1024 threads)
  int total;
  int at = cta_excl_scan(mine, s_warp, &total);
  for (int i = r0; i < r1; ++i)
    if (vld[i]) { if (at < cap) { cpos[at] = sm[i]; ccnt[at] = cnt[i]; } ++at; }
  __syncthreads();
  return total;
}

// S0: tier 0's scratch.  A pair that reaches an overflow tier because of its hit / candidate / mapping counts has already been
// through the front end there: its probed minimizer records are copied instead of being computed and probed again (mm_done flag).
__global__ void __launch_bounds__(CTA_NT) seed_cta_kernel(DevParams P, DevIndex ix, DevBatch B, Scratch S, Scratch S0, Counters *ctr, int sm_cap) {
  extern __shared__ u64 sm[];  // [sm_cap] sort buffer, then per-minimizer arrays sized by the tier's maxmm
  int *s_off = (int *)(sm + sm_cap);
  u32 *s_c1 = (u32 *)(s_off + S.caps.maxmm + 1), *s_c2 = s_c1 + S.caps.maxmm;
  __shared__ int s_i[8];
  __shared__ unsigned long long s_steps;
  const int sr = blockIdx.x, tid = threadIdx.x;
  const int slot = sr >> 1, mate = sr & 1;
  // the mate's CTA may flag the pair concurrently: read the status once, uniformly
  if (tid == 0) s_i[7] = S.pmeta[slot].status;
  __syncthreads();
  if (s_i[7] != ST_OK || (P.se && mate == 1)) return;
  const int pair = slot_pair(S, slot);
  ReadMeta &rm = S.rmeta[sr];
  const Caps c = S.caps;
  u64 *mmh = S.mm_hash + (size_t)sr * c.maxmm;
  u64 *mmv = S.mm_val + (size_t)sr * c.maxmm;
  u32 *mmp = S.mm_pos + (size_t)sr * c.maxmm;
  const ReadMeta &r0 = S0.rmeta[2 * pair + mate];
  const bool reuse = r0.mm_done == 1 && r0.n_mm <= c.maxmm && r0.len == rm.len;  // uniform: global values
  if (reuse) {
    if (tid == 0) { rm.n_mm = r0.n_mm; s_i[0] = r0.n_mm; s_steps = 0; s_i[5] = 0; }
  } else {
    const int n0 = cta_minimizers(read_ptr(B, pair, mate), rm.len, P.k, P.w, mmh, mmp, c.maxmm, sm, &s_i[6]);
    if (tid == 0) {
      rm.n_mm = n0;
      s_i[0] = n0;
      s_steps = 0;
      s_i[5] = 0;  // found
    }
  }
  __syncthreads();
  const int n_mm = s_i[0];
  if (n_mm > c.maxmm) { if (tid == 0) atomicExch(&S.pmeta[slot].status, ST_OVERFLOW); return; }
  if (n_mm == 0) return;
  const size_t b0 = mm_base(S0, pair, mate);
  const int ms0 = mm_stride(S0);
  for (int i = tid; i < n_mm; i += CTA_NT) {
    u64 val = 0;
    int steps = 0, kind;
    if (reuse) {
      val = S0.mm_val[b0 + (size_t)i * ms0];
      const u32 pw = S0.mm_pos[b0 + (size_t)i * ms0];
      kind = (int)(pw >> 30);
      mmv[i] = val; mmp[i] = pw;
    } else {
      kind = index_lookup(ix, mmh[i], &val, &steps);
      mmv[i] = val;
      mmp[i] = (mmp[i] & 0x3FFFFFFFu) | ((u32)kind << 30);
      atomicAdd(&s_steps, (unsigned long long)steps);
      if (kind) atomicAdd(&s_i[5], 1);
    }
    u32 c1 = 0, c2 = 0;
    if (kind == 1) { c1 = c2 = 1; }
    else if (kind == 2) { const u32 n = (u32)val; if (n < (u32)P.f0) c1 = n; if (n < (u32)P.f1) c2 = n; }
    s_c1[i] = c1; s_c2[i] = c2;
  }
  __syncthreads();
  if (tid == 0) {
    long long cnt1 = 0;
    for (int i = 0; i < n_mm; ++i) cnt1 += s_c1[i];
    const bool round2 = cnt1 == 0;
    long long tot = 0;
    RepStats st = {0u, 0xFFFFFFFFu, 0};
    for (int i = 0; i < n_mm; ++i) {
      s_off[i] = (int)tot;
      tot += round2 ? s_c2[i] : s_c1[i];
      if ((mmp[i] >> 30) == 2 && (u32)mmv[i] >= (u32)P.f0) rep_update(P.k, P.w, (mmp[i] & 0x3FFFFFFFu) >> 1, st);
      if (tot > 2ll * c.hc) break;
    }
    s_off[n_mm] = (int)(tot > 2ll * c.hc ? 2ll * c.hc + 1 : tot);
    s_i[1] = round2;
    s_i[2] = st.count;
    rm.rep_len = st.len;
    if (!reuse) {  // (a reused read was counted by the front end)
      atomicAdd(&ctr->n_minimizers, (u64)n_mm);
      atomicAdd(&ctr->n_probe_steps, (u64)s_steps);
      atomicAdd(&ctr->n_found, (u64)s_i[5]);
    }
  }
  __syncthreads();
  const int T = s_off[n_mm];
  if (T > 2 * c.hc) { if (tid == 0) atomicExch(&S.pmeta[slot].status, ST_OVERFLOW); return; }
  u64 *hits = S.hits + (size_t)sr * 2 * c.hc;  // [2][hc] contiguous: positives first, negatives right behind them
  for (int j = tid; j < T; j += CTA_NT) {
    int lo = 0, hi = n_mm;  // last i with s_off[i] <= j
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s_off[mid] <= j) lo = mid; else hi = mid; }
    // skip empty minimizers sharing the same offset
    const int i = lo;
    const u32 rpos = (mmp[i] & 0x3FFFFFFFu) >> 1, rstrand = mmp[i] & 1u;
    const u64 val = mmv[i];
    const u64 rh = (mmp[i] >> 30) == 1 ? val : __ldg(&ix.occ[(u32)(val >> 32) + (u32)(j - s_off[i])]);
    bool same;
    const u64 cp = hit_to_candidate(P.k, rh, rpos, rstrand, &same);
    hits[j] = cp | (same ? 0ull : (1ull << 63));
  }
  if (tid == 0) { u64 occ_reads = 0; for (int i = 0; i < n_mm; ++i) if ((mmp[i] >> 30) == 2) occ_reads += s_off[i + 1] - s_off[i]; atomicAdd(&ctr->n_occ_reads, occ_reads); }
  __syncthreads();
  cta_sort_keys(hits, T, sm, sm_cap);
  if (tid == 0) {
    int lo = 0, hi = T;  // first index with the strand tag set
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (hits[mid] >> 63) hi = mid; else lo = mid + 1; }
    s_i[3] = lo;
  }
  __syncthreads();
  const int np = s_i[3], nn = T - np;
  for (int j = np + tid; j < T; j += CTA_NT) hits[j] &= ~(1ull << 63);
  __syncthreads();
  int need = n_mm - s_i[2];
  need = need > 1 ? need : 1;
  need = need > P.min_seeds ? P.min_seeds : need;
  if (s_i[1] && np > 0 && nn > 0) need = P.min_seeds;
  u64 *cp0 = S.cand_pos + cand_base(0, c, sr, 0, 0), *cp1 = cp0 + c.cc;
  u8 *cc0 = S.cand_cnt + cand_base(0, c, sr, 0, 0), *cc1 = cc0 + c.cc;
  u8 *aux = (u8 *)(s_c2 + S.caps.maxmm);
  const int nc0 = cta_cluster_par(P.e, need, (u32)n_mm, hits, np, cp0, cc0, c.cc, sm, sm_cap, aux, &s_i[4]);
  const int nc1 = cta_cluster_par(P.e, need, (u32)n_mm, hits + np, nn, cp1, cc1, c.cc, sm, sm_cap, aux, &s_i[4]);
  if (tid == 0) {
    if (nc0 > c.cc || nc1 > c.cc) atomicExch(&S.pmeta[slot].status, ST_OVERFLOW);
    else {
          rm.n_cand[0] = nc0; rm.n_cand[1] = nc1; rm.n_cand_gen[0] = nc0; rm.n_cand_gen[1] = nc1;
    }
  }
}


// =================================================================================================
// --split-alignment (Hi-C): draft_mapping_generator.cc:359-557 split branch, alignment.cc:197-376,
// mapping_generator.h:389-415 (pairing), :657-917 split branches, :920-1022 split MAPQ, mapping_generator.cc:169-210.

// alignment.cc:197-283 (from3 = false) and :285-376 (from3 = true).  PAT(i) / TXT(i): base codes at logical index i.
template <typename PatF, typename TxtF>
__device__ __forceinline__ int banded_align_dropoff(int e, int L, bool from3, PatF PAT, TxtF TXT, int *end_pos, int *read_len_out) {
  PatPlanes W = {0u, 0u, 0u};
  for (int i = 0; i < 2 * e; ++i) planes_or(W, from3 ? PAT(L + 2 * e - 1 - i) : PAT(i), 1u << i);
  const u32 hi = 1u << (2 * e), band = (hi << 1) - 1u;
  u32 VP = 0, VN = 0, pVP = 0, pVN = 0;
  int err = 0, perr = 0, i = 0, fail_beginning = 0;
  for (; i < L; ++i) {
    planes_or(W, from3 ? PAT(L - 1 - i) : PAT(i + 2 * e), hi);
    u32 X = VN | planes_match(W, from3 ? TXT(L - 1 - i) : TXT(i), band);
    const u32 D0 = ((VP + (X & VP)) ^ VP) | X;
    const u32 HN = VP & D0;
    const u32 HP = VN | ~(VP | D0);
    X = D0 >> 1;
    pVN = VN; pVP = VP;
    VN = X & HP;
    VP = HN | ~(X | HP);
    perr = err;
    err += 1 - (int)(D0 & 1u);
    if (err > 2 * e) { if (i < 4 * e && i < L / 2) fail_beginning = 1; break; }
    planes_shift(W);
  }
  if (i < L) { err = perr; VN = pVN; VP = pVP; }
  const int band_start = i - 1;
  int best = err;
  *read_len_out = i;
  int ep = band_start;
  for (int j = 0; j < 2 * e; ++j) {
    err += (int)((VP >> j) & 1u);
    err -= (int)((VN >> j) & 1u);
    if (err < best || (err == best && j + 1 == e)) { best = err; ep = band_start + 1 + j; }
  }
  if (fail_beginning || (L > 60 && ep + 1 - e - best < 30)) ep = -ep;
  *end_pos = ep;
  return best;
}

struct SplitResult { int nerr, actual, endp, gap, rml; };  // nerr = -(matched length) or e+1
// one candidate of the split driver (draft_mapping_generator.cc:410-487): drop-off alignment, retry without the first 20-e bases.
// TXT(i): base code of the strand's sequence at i (the read, or its reverse complement for s = 1) — one code path for both strands.
template <typename TxtF>
__device__ __forceinline__ SplitResult verify_split_candidate(int e, const u8 *win, TxtF TXT, int L, int s) {
  SplitResult r;
  int endp = L, gap = 0, nerr, rml = 0;
  const int allow_gap = 20 - e;
  const bool from3 = s != 0;
  nerr = banded_align_dropoff(e, L, from3, [&](int i) { return base_code(__ldg(win + i)); }, TXT, &endp, &rml);
  if (endp < 0 && allow_gap > 0) {
    const int b_err = nerr, b_end = -endp, b_rml = rml;
    const int sh = from3 ? 0 : allow_gap;  // the + strand drops the read's first bases, the - strand aligns from the 3' end anyway
    nerr = banded_align_dropoff(e, L - allow_gap, from3, [&](int i) { return base_code(__ldg(win + sh + i)); }, [&](int i) { return TXT(sh + i); }, &endp, &rml);
    if (nerr > e || endp < 0) { nerr = b_err; endp = b_end; rml = b_rml; }
    else { gap = allow_gap; endp += gap; rml += gap; }
  }
  if (endp + 1 - e - nerr - gap >= 30) { r.actual = nerr; r.nerr = -(endp - e - nerr - gap); }
  else { r.nerr = e + 1; r.actual = e + 1; }
  r.endp = endp; r.gap = gap; r.rml = rml;
  return r;
}

// K3 (split): per read, sequential driver with count-threshold pruning.
__global__ void verify_split_kernel(DevParams P, DevRef R, DevBatch B, Scratch S, Counters *ctr) {
  const int sr = blockIdx.x * blockDim.x + threadIdx.x;
  if (sr >= 2 * S.n_slots) return;
  const int slot = sr >> 1, mate = sr & 1;
  if (S.pmeta[slot].status != ST_OK || (P.se && mate == 1)) return;
  const int pair = slot_pair(S, slot);
  ReadMeta &rm = S.rmeta[sr];
  const Caps c = S.caps;
  const u8 *read = read_ptr(B, pair, mate);
  const int L = rm.len, e = P.e;
  Tally t = {e + 1, e + 1, 0, 0};
  auto cless = [](u64 pa, u8 ca, u64 pb, u8 cb) { return ca != cb ? ca > cb : pa < pb; };
  u64 n_verified = 0;
  int nm0 = 0, nm1 = 0;
  prefetch_span(read, L);
  auto CP = [&](int s) { return cand_pos_of(S, sr, 0, s); };
  auto CC = [&](int s) { return cand_cnt_of(S, sr, 0, s); };
  const int nc0 = rm.n_cand[0], nc1 = rm.n_cand[1];
  sort_pairs<u8>(CP(0), CC(0), nc0, cless);
  sort_pairs<u8>(CP(1), CC(1), nc1, cless);
  // The reference walks strand 0's candidates, then strand 1's, with a pruning threshold per strand.  Here ONE loop takes
  // "this read's next candidate" whatever its strand: the lanes of a warp (different reads) then run the alignment body
  // together even when their candidates lie on different strands — a read's true locus is on one strand only, so the
  // two-loop form left half of the lanes idle in each.  Same candidates, same order, same results.
  int s = 0, ci = 0;
  u32 threshold = 0;
  for (;;) {
    if (s >= 2) break;
    const int nc = s ? nc1 : nc0;
    const u32 cnt = ci < nc ? (u32)CC(s)[ci] : 0u;
    if (ci >= nc || cnt < threshold) { ++s; ci = 0; threshold = 0; continue; }  // strand finished or pruned (draft_mapping_generator.cc:412-414)
    const u64 cpos = CP(s)[ci];
    ++ci;
    const u32 rid = (u32)(cpos >> 32);
    const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
    if (!valid_cand(e, R.len[rid], pos, (u32)L)) continue;
    prefetch_span(R.seq + R.off[rid] + pos - e, L + 2 * e);
    const SplitResult r = verify_split_candidate(e, R.seq + R.off[rid] + pos - e, [&](int i) -> u32 {
      const u32 b = base_code(read[s ? L - 1 - i : i]);
      return s ? (b < 4 ? 3u ^ b : 4u) : b;
    }, L, s);
    ++n_verified;
    if (r.nerr <= e) {
      if (r.nerr < t.min_err) {
        t.second_min_err = t.min_err; t.n_second_best = t.n_best; t.min_err = r.nerr; t.n_best = 1;
        threshold = nc > 50 ? cnt : cnt / 2;
      } else if (r.nerr == t.min_err) t.n_best++;
      else if (r.nerr == t.second_min_err) t.n_second_best++;
      else if (r.nerr < t.second_min_err) { t.n_second_best = 1; t.second_min_err = r.nerr; }
      const int k = s ? nm1 : nm0;
      if (k < c.mc) {
        map_pos_of(S, sr, s)[k] = s == 0 ? cpos - (u64)e + (u64)r.endp : cpos - (u64)r.gap;
        map_err_of(S, sr, s)[k] = (short)r.nerr;
        map_split_of(S, sr, s)[k] = ((r.actual & 0xff) << 24) | ((r.gap & 0xff) << 16) | (r.rml & 0xffff);
      }
      if (s) ++nm1; else ++nm0;
    }
  }
  if (nm0 > c.mc || nm1 > c.mc) { S.pmeta[slot].status = ST_OVERFLOW; atomicAdd(&ctr->ovf_reason[6], 1ull); return; }
  rm.n_map[0] = nm0; rm.n_map[1] = nm1;
  rm.min_err = t.min_err; rm.second_min_err = t.second_min_err; rm.n_best = t.n_best; rm.n_second_best = t.n_second_best;
  if (n_verified) agg_add(&ctr->n_verified, n_verified);
}

// K3 (split, overflow tiers): every valid candidate verified by its own thread, thread 0 replays the pruning order.
__global__ void __launch_bounds__(CTA_NT) verify_split_cta_kernel(DevParams P, DevRef R, DevBatch B, Scratch S, Counters *ctr, int sm_cap) {
  extern __shared__ u64 smk[];
  u8 *smt = (u8 *)(smk + sm_cap);
  __shared__ int s_status;
  const int sr = blockIdx.x, tid = threadIdx.x;
  const int slot = sr >> 1, mate = sr & 1;
  if (tid == 0) s_status = S.pmeta[slot].status;
  __syncthreads();
  if (s_status != ST_OK) return;
  const int pair = slot_pair(S, slot);
  ReadMeta &rm = S.rmeta[sr];
  const Caps c = S.caps;
  const u8 *read = read_ptr(B, pair, mate);
  const int L = rm.len, e = P.e;
  auto cless = [](u64 pa, u8 ca, u64 pb, u8 cb) { return ca != cb ? ca > cb : pa < pb; };
  u64 *cp[2], *res[2];
  u8 *cc[2], *vld[2];
  for (int s = 0; s < 2; ++s) {
    cp[s] = S.cand_pos + cand_base(0, c, sr, 0, s); cc[s] = S.cand_cnt + cand_base(0, c, sr, 0, s);
    res[s] = S.cand_pos + cand_base(0, c, sr, 2, s); vld[s] = S.cand_cnt + cand_base(0, c, sr, 2, s);  // augment set is free here
  }
  const int nc[2] = {rm.n_cand[0], rm.n_cand[1]};
  cta_sort_pairs<u8>(cp[0], cc[0], nc[0], ~0ull, (u8)0, cless, smk, smt, sm_cap);
  cta_sort_pairs<u8>(cp[1], cc[1], nc[1], ~0ull, (u8)0, cless, smk, smt, sm_cap);
  u64 n_ver = 0;
  for (int s = 0; s < 2; ++s)
    for (int i = tid; i < nc[s]; i += CTA_NT) {
      const u64 cpos = cp[s][i];
      const u32 rid = (u32)(cpos >> 32);
      const u32 pos = s == 0 ? (u32)cpos : (u32)cpos - (u32)L + 1u;
      if (!valid_cand(e, R.len[rid], pos, (u32)L)) { vld[s][i] = 0; continue; }
      const SplitResult r = s == 0 ? verify_split_candidate(e, R.seq + R.off[rid] + pos - e, [&](int q) { return base_code(read[q]); }, L, 0)
                                   : verify_split_candidate(e, R.seq + R.off[rid] + pos - e, [&](int q) { return neg_code(read, L, q); }, L, 1);
      vld[s][i] = 1;
      res[s][i] = ((u64)(u32)(r.nerr + 1024) << 48) | ((u64)(r.actual & 0xff) << 40) | ((u64)(r.gap & 0xff) << 32) | ((u64)(r.rml & 0xffff) << 16) | (u64)(r.endp & 0xffff);
      ++n_ver;
    }
  if (n_ver) atomicAdd(&ctr->n_verified, n_ver);
  __syncthreads();
  if (tid != 0) return;
  Tally t = {e + 1, e + 1, 0, 0};
  int nm[2] = {0, 0};
  for (int s = 0; s < 2; ++s) {
    u64 *mp = S.map_pos + map_base(0, c, sr, s);
    short *me = S.map_err + map_base(0, c, sr, s);
    int *ms = S.map_split + map_base(0, c, sr, s);
    u32 threshold = 0;
    for (int ci = 0; ci < nc[s]; ++ci) {
      if (cc[s][ci] < threshold) break;
      if (!vld[s][ci]) continue;
      const u64 w = res[s][ci];
      const int nerr = (int)(w >> 48) - 1024, actual = (int)((w >> 40) & 0xff), gap = (int)((w >> 32) & 0xff), rml = (int)((w >> 16) & 0xffff), endp = (int)(w & 0xffff);
      if (nerr <= e) {
        if (nerr < t.min_err) {
          t.second_min_err = t.min_err; t.n_second_best = t.n_best; t.min_err = nerr; t.n_best = 1;
          threshold = nc[s] > 50 ? (u32)cc[s][ci] : (u32)cc[s][ci] / 2;
        } else if (nerr == t.min_err) t.n_best++;
        else if (nerr == t.second_min_err) t.n_second_best++;
        else if (nerr < t.second_min_err) { t.n_second_best = 1; t.second_min_err = nerr; }
        const u64 cpos = cp[s][ci];
        if (nm[s] < c.mc) {
          mp[nm[s]] = s == 0 ? cpos - (u64)e + (u64)endp : cpos - (u64)gap;
          me[nm[s]] = (short)nerr;
          ms[nm[s]] = ((actual & 0xff) << 24) | ((gap & 0xff) << 16) | (rml & 0xffff);
        }
        ++nm[s];
      }
    }
  }
  if (nm[0] > c.mc || nm[1] > c.mc) { S.pmeta[slot].status = ST_OVERFLOW; return; }
  rm.n_map[0] = nm[0]; rm.n_map[1] = nm[1];
  rm.min_err = t.min_err; rm.second_min_err = t.second_min_err; rm.n_best = t.n_best; rm.n_second_best = t.n_second_best;
}

// K4 (split): mapping_generator.h:389-415 — #best pairs = product of the mates' best-mapping counts per direction.
__global__ void pairing_split_kernel(DevParams P, Scratch S, int *pair_nbest) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status != ST_OK) { if (pm.status == ST_DROP) pair_nbest[pair] = 0; return; }
  ReadMeta *rm = S.rmeta + 2 * slot;
  if (rm[0].n_map[0] + rm[0].n_map[1] == 0 || rm[1].n_map[0] + rm[1].n_map[1] == 0) { pm.status = ST_DROP; pair_nbest[pair] = 0; return; }
  int cnt[2][2];
  for (int m = 0; m < 2; ++m)
    for (int s = 0; s < 2; ++s) {
      const Strided<short> me = map_err_of(S, 2 * slot + m, s);
      const int want = rm[m].min_err;
      int k = 0;
      for (int i = 0; i < rm[m].n_map[s]; ++i) k += me[i] == want;
      cnt[m][s] = k;
    }
  const long long nb = (long long)cnt[0][0] * cnt[1][1] + (long long)cnt[0][1] * cnt[1][0] + (long long)cnt[0][0] * cnt[1][0] + (long long)cnt[0][1] * cnt[1][1];
  const int n_best = nb > 0x7fffffffLL ? 0x7fffffff : (int)nb;
  pm.min_sum = n_best > 0 ? rm[0].min_err + rm[1].min_err : 2 * P.e + 1;
  pm.second_min_sum = 2 * P.e + 1; pm.n_best = n_best; pm.n_second_best = 0;
  pair_nbest[pair] = (n_best > P.drop_rep) ? 0 : n_best;
}

__device__ __forceinline__ int sgn_char(u8 c) { return (int)(signed char)c; }
// alignment.cc:24-83 with n_cigar == 0.  RD(i): raw read char at index i of the strand string (0 past its end).
template <typename ReadC>
__device__ __forceinline__ int adjust_gap_beginning(int strand, const u8 *ref, ReadC RD, int *gap, int read_end, int ref_start, int ref_end) {
  int i, j;
  if (strand == 0) {
    if (*gap <= 0) return ref_start;
    for (i = *gap - 1, j = ref_start - 1; i >= 0 && j >= 0; --i, --j) {
      const int a = sgn_char(RD(i)), b = sgn_char(__ldg(ref + j));
      if (a != b && a != b - 'a' + 'A') break;
    }
    *gap = i + 1;
    return j + 1;
  }
  if (*gap <= 0) return ref_end;
  for (i = read_end + 1, j = ref_end + 1; RD(i) && __ldg(ref + j); ++i, ++j) {
    const int a = sgn_char(RD(i)), b = sgn_char(__ldg(ref + j));
    if (a != b && a != b - 'a' + 'A') break;
  }
  *gap = *gap + i - (read_end + 1);
  return j - 1;
}

// mapping_generator.h:920-1022 with split_alignment.
__device__ inline u8 mapq_se_split(const MapqTables &T, const DevParams &P, int n_cand_strand, int num_errors, unsigned short aln_len, int read_len,
                                   int max_diff, const ReadMeta &rm) {
  const int coef_len = 50;
  double ident = xdiv((double)(-num_errors), (double)aln_len);
  if (ident > 1) ident = 1;
  int mapq = 0;
  int second = rm.second_min_err;
  if (rm.n_best > 1) {
  } else {
    if (second > num_errors + max_diff) second = num_errors + max_diff;
    double tmp = (int)aln_len < coef_len ? 1.0 : T.inv_log[aln_len];
    tmp = xmul(tmp, xmul(ident, ident));
    mapq = (int)xadd(xmul(xmul(xmul(5 * 6.02, (double)(second - num_errors)), tmp), tmp), 0.499);
  }
  if (rm.n_second_best > 0) mapq -= second_best_penalty(T, rm.n_second_best);
  if (mapq > 60) mapq = 60;
  if (mapq < 0) mapq = 0;
  if (rm.rep_len > 0) {
    double frac = xdiv((double)rm.rep_len, (double)read_len);
    if (rm.rep_len >= (u32)read_len) frac = 0.999;
    mapq = (int)xadd(xmul((double)mapq, rep_scale(ident, frac)), 0.499);
  }
  if ((int)aln_len < read_len - P.e && second != num_errors) {
    if (rm.rep_len >= (u32)aln_len && rm.rep_len < (u32)read_len && (int)aln_len < read_len / 3) mapq = 0;
    const int diff = second - num_errors;
    const u32 num_candidates = (u32)n_cand_strand;
    if (second - num_errors <= P.e * 3 / 4 && num_candidates >= 5) mapq -= (num_candidates / 5 / diff);  // u32 arithmetic as in the reference
    if (mapq < 0) mapq = 0;
    if (rm.n_second_best > 0 && second - num_errors <= P.e * 3 / 4) mapq /= (rm.n_second_best / diff + 1);
  }
  return (u8)mapq;
}

struct OutPairs {  // == cmx_pairs_record
  u32 read_id, rid1, rid2, pos1, pos2;
  u8 strand1, strand2, mapq, is_unique;
};

// K6 (split): the selected best pair(s) -> PairsMapping (mapping_generator.cc:169-210).
__global__ void emit_split_kernel(DevParams P, DevRef R, DevBatch B, MapqTables T, Scratch S, const int *pair_sel, OutPairs *out, int *out_n, Counters *ctr) {
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  PairMeta &pm = S.pmeta[slot];
  const int pair = slot_pair(S, slot);
  if (pm.status == ST_OVERFLOW) return;
  if (pm.status != ST_OK || pm.n_best > P.drop_rep || pm.n_best == 0) { out_n[pair] = 0; return; }
  const ReadMeta *rm = S.rmeta + 2 * slot;
  const int mb = P.max_best;
  const int to_report = mb < pm.n_best ? mb : pm.n_best;
  const int *sel = pair_sel + (size_t)pair * mb;
  const u8 uniq = (pm.n_best == 1 || rm[0].n_best == 1 || rm[1].n_best == 1) ? 1 : 0;
  const int e = P.e;
  const int L[2] = {rm[0].len, rm[1].len};
  const u8 *rd[2] = {read_ptr(B, pair, 0), read_ptr(B, pair, 1)};
  // mapping_generator.h:657-917, BED/pairs branch with split_alignment
  auto span = [&](int m, int s, u64 dpos, int split_word, u32 *st, u32 *en) {
    const u32 rid = (u32)(dpos >> 32), rp = (u32)dpos;
    const int full = L[m];
    const int split_site = split_word & 0xffff;
    int gap = (split_word >> 16) & 0xff;
    const int actual = (split_word >> 24) & 0xff;
    const int Ls = split_site - gap;
    u32 vws = rp + 1u > (u32)(Ls + e) ? rp + 1u - (u32)Ls - (u32)e : 0u;
    if (rp + (u32)e >= R.len[rid]) vws = R.len[rid] - (u32)e - (u32)Ls;
    const u8 *rseq = R.seq + R.off[rid];
    const u8 *win = rseq + vws;
    const u8 *r = rd[m];
    if (s == 0) {
      int s0 = banded_traceback(e, actual, Ls, [&](int i) { return __ldg(win + i); }, [&](int i) { return r[gap + i]; });
      if (gap > 0) s0 = adjust_gap_beginning(0, rseq, [&](int i) { return i < full ? r[i] : (u8)0; }, &gap, Ls - 1, (int)vws + s0, (int)rp) - (int)vws;
      *st = vws + (u32)s0;
      *en = rp;
      return;
    }
    const int rss = full - split_site;
    const int s0 = e;
    int en0 = (int)(rp - vws + 1u);  // kept when the aligner bails out early without writing it (mapping_generator.h:856-857)
    banded_align(e, Ls, [&](int i) { return base_code(__ldg(win + i)); }, [&](int i) { return neg_code(r, full, rss + i); }, &en0);
    en0 += 1;
    if (gap > 0)
      en0 = adjust_gap_beginning(1, rseq, [&](int i) { return (rss + i) < full ? code_char(neg_code(r, full, rss + i)) : (u8)0; }, &gap, Ls - 1, (int)vws + s0,
                                 (int)vws + en0) - (int)vws + 1;
    *st = vws + (u32)s0;
    *en = vws + (u32)en0 - 1u;
  };
  int idx = 0, reported = 0;
  const int DS1[4] = {0, 1, 0, 1}, DS2[4] = {1, 0, 0, 1};
  // phase 1: which mappings are reported (the enumeration of mapping_generator.h:389-415); phase 2: spans, MAPQ, records — all
  // threads of a warp enter phase 2 together instead of reaching their tracebacks at different loop iterations
  int ch_dir[CMX_MAX_BEST], ch_i1[CMX_MAX_BEST], ch_i2[CMX_MAX_BEST];
  for (int dir = 0; dir < 4 && reported != to_report; ++dir) {
    const int s1 = DS1[dir], s2 = DS2[dir];
    const Strided<short> e1 = map_err_of(S, 2 * slot, s1), e2 = map_err_of(S, 2 * slot + 1, s2);
    const int want1 = rm[0].min_err, want2 = rm[1].min_err;
    if (rm[0].n_map[s1] == 0 || rm[1].n_map[s2] == 0) continue;
    for (int i1 = 0; i1 < rm[0].n_map[s1] && reported != to_report; ++i1) {
      if (e1[i1] != want1) continue;
      for (int i2 = 0; i2 < rm[1].n_map[s2]; ++i2) {
        if (e2[i2] != want2) continue;
        if (idx == sel[reported]) {
          ch_dir[reported] = dir; ch_i1[reported] = i1; ch_i2[reported] = i2;
          ++reported;
          if (reported == to_report) break;
        }
        ++idx;
      }
    }
  }
  for (int r = 0; r < reported; ++r) {
    const int s1 = DS1[ch_dir[r]], s2 = DS2[ch_dir[r]], i1 = ch_i1[r], i2 = ch_i2[r];
    const Strided<u64> p1 = map_pos_of(S, 2 * slot, s1), p2 = map_pos_of(S, 2 * slot + 1, s2);
    const Strided<int> w1 = map_split_of(S, 2 * slot, s1), w2 = map_split_of(S, 2 * slot + 1, s2);
    u32 st1, en1, st2, en2;
    span(0, s1, p1[i1], w1[i1], &st1, &en1);
    span(1, s2, p2[i2], w2[i2], &st2, &en2);
    const unsigned short al1 = (unsigned short)(en1 - st1 + 1u), al2 = (unsigned short)(en2 - st2 + 1u);
    u8 q1 = mapq_se_split(T, P, rm[0].n_cand[s1], rm[0].min_err, al1, L[0], 2, rm[0]);
    u8 q2 = mapq_se_split(T, P, rm[1].n_cand[s2], rm[1].min_err, al2, L[1], 2, rm[1]);
    q1 = (u8)xmul((double)q1, 1.2); if (q1 > 60) q1 = 60;
    q2 = (u8)xmul((double)q2, 1.2); if (q2 > 60) q2 = 60;
    const u8 q = q1 < q2 ? q1 : q2;
    int rid1 = (int)(u32)(p1[i1] >> 32), rid2 = (int)(u32)(p2[i2] >> 32);
    int pos1 = (int)(s1 == 0 ? st1 : en1), pos2 = (int)(s2 == 0 ? st2 : en2);
    u8 str1 = s1 == 0 ? 1 : 0, str2 = s2 == 0 ? 1 : 0;
    const bool smaller = rid1 < rid2 || (rid1 == rid2 && pos1 < pos2);
    if (!smaller) { int tt = rid1; rid1 = rid2; rid2 = tt; tt = pos1; pos1 = pos2; pos2 = tt; const u8 ts = str1; str1 = str2; str2 = ts; }
    OutPairs o;
    o.read_id = B.first_read_id + (u32)pair; o.rid1 = (u32)rid1; o.rid2 = (u32)rid2; o.pos1 = (u32)pos1; o.pos2 = (u32)pos2;
    o.strand1 = str1; o.strand2 = str2; o.mapq = q; o.is_unique = uniq;
    out[(size_t)pair * mb + r] = o;
  }
  out_n[pair] = reported;
  pm.n_rec = reported;
  if (reported > 0) { agg_add(&ctr->n_mapped, 1ull); if (pm.n_best == 1) agg_add(&ctr->n_unique, 1ull); }
}


// =================================================================================================
// scATAC cell barcodes: CorrectBarcodeAt (chromap.cc:572-799).  barcode_kernel does --bc-error-threshold 0 and 1 whole; at 2
// it lists the barcodes that need a search and barcode_correct2_kernel searches them, one warp per barcode.
#define BC2_MAX_HITS 4560  // 3L + 9L(L-1)/2 at L = 32: the most candidates one barcode can have
#define BC2_SMEM_HITS 128  // hit list of a warp in shared memory; a barcode with more hits goes to the slab pass
#define BC2_WARPS 8        // warps per block of barcode_correct2_kernel
#define BC2_GRID_MAX 2048  // its grid: warps stride over the correction list
#define BC2_SLAB_WARPS 64  // the slab pass: warps, each with a Bc2Slab in global memory
struct Bc2Slab {  // one warp's hit list that holds any barcode's hits
  double score[BC2_MAX_HITS], sorted[BC2_MAX_HITS];
  u32 tag[BC2_MAX_HITS];
};
struct DevWhitelist {
  const ulonglong2 *slots;  // {key, count}; empty key = ~0
  u64 mask;                 // n_slots - 1
  int shift;
  int top_listed;           // the key ~0 (all-T at 32 bases) is listed, with count top_count: it cannot be in the slots
  u64 top_count;
  double num_sample;
  const double *pow_tab;    // [81]: pow(10.0, (-q) / 10.0) from the host libm (q up to 40 + 40: two changed bases)
  int err_threshold;
  double prob_threshold;
  int output_not_in_whitelist;
  int active;               // whitelist uploaded
  // --bc-error-threshold 2 only: [n] barcodes to search (Counters::n_bc2_listed), [n] those with more than BC2_SMEM_HITS hits
  // (Counters::n_bc2_overflow), and the slab pass's [BC2_SLAB_WARPS] hit lists
  u32 *c2_list, *c2_over;
  Bc2Slab *c2_slab;
};
__device__ __forceinline__ bool wl_find(const DevWhitelist &W, u64 key, u64 *count) { return wl_lookup(W.slots, W.mask, W.shift, W.top_listed, W.top_count, key, count); }
__global__ void wl_insert_kernel(const u64 *keys, const u32 *counts, u64 n, ulonglong2 *slots, u64 mask, int shift) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || keys[i] == CMX_EMPTY_KEY) return;  // DevWhitelist::top_listed holds that one
  ulonglong2 *slot = kv_claim(slots, mask, shift, keys[i]);
  slot->y = counts[i];
}
// utils.h:107-126: 2 bits per base, ambiguous base -> A
__device__ __forceinline__ u64 barcode_seed(const u8 *s, int len) {
  u64 seed = 0;
  for (int i = 0; i < len; ++i) { const u32 b = base_code(s[i]); seed = b < 4 ? (seed << 2) | b : seed << 2; }
  return seed;
}
__global__ void barcode_kernel(DevWhitelist W, const u8 *bc_seq, const u8 *bc_qual, int bc_len, int n, u64 *bc_key, u8 *bc_ok, Counters *ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u8 *bc = bc_seq + (size_t)i * bc_len, *qual = bc_qual + (size_t)i * bc_len;
  const u64 key = barcode_seed(bc, bc_len);
  if (!W.active) { bc_key[i] = key; bc_ok[i] = 1; return; }
  int n_n = 0, first_n = 0;
  for (int p = bc_len - 1; p >= 0; --p) if (bc[p] == 'N') { if (n_n == 0) first_n = bc_len - 1 - p; ++n_n; }
  u64 cnt;
  bool ok = false;
  u64 out_key = key;
  if (n_n > W.err_threshold) ok = false;
  else if (n_n == 0 && wl_find(W, key, &cnt)) { ok = true; agg_add(&ctr->n_bc_in_whitelist, 1ull); }
  else if (W.err_threshold == 2) W.c2_list[atomicAdd(&ctr->n_bc2_listed, 1ull)] = (u32)i;  // barcode_correct2_kernel decides
  else if (W.err_threshold > 0) {
    double sc[128];
    u8 ci[128], cb[128];
    int nc = 0;
    int i_start = 0, i_end = bc_len, ti_limit = 3;
    if (n_n > 0) { i_start = first_n; i_end = first_n + 1; ti_limit = 4; }
    for (int p = i_start; p < i_end; ++p) {
      const u64 keep = ~(3ull << (2 * p)) & key;
      u64 b1 = (key >> (2 * p)) & 3ull;
      for (int ti = 0; ti < ti_limit; ++ti) {
        b1 = (b1 + 1) & 3ull;
        if (wl_find(W, keep | (b1 << (2 * p)), &cnt)) {
          const double abundance = xdiv((double)cnt, W.num_sample);
          int q = (int)(signed char)qual[bc_len - 1 - p] - 33;
          q = q > 40 ? 40 : q; q = q < 3 ? 3 : q;
          if (nc < 128) { sc[nc] = xmul(W.pow_tab[q], abundance); ci[nc] = (u8)(bc_len - 1 - p); cb[nc] = (u8)b1; }
          ++nc;
        }
      }
    }
    if (nc >= 1) {
      int best = 0;
      bool accept = true;
      if (nc > 1) {
        // std::sort with std::greater<BarcodeWithQual> (utils.h:23-35): (score, index, base char) descending
        for (int a = 1; a < nc; ++a) {
          const double s_ = sc[a]; const u8 i_ = ci[a], b_ = cb[a];
          int b = a - 1;
          while (b >= 0 && (sc[b] < s_ || (sc[b] == s_ && (ci[b] < i_ || (ci[b] == i_ && cb[b] < b_))))) { sc[b + 1] = sc[b]; ci[b + 1] = ci[b]; cb[b + 1] = cb[b]; --b; }
          sc[b + 1] = s_; ci[b + 1] = i_; cb[b + 1] = b_;
        }
        double sum = 0;
        for (int a = 0; a < nc; ++a) sum = xadd(sum, sc[a]);
        accept = xdiv(sc[0], sum) > W.prob_threshold;
      }
      if (accept) {
        const int p = bc_len - 1 - (int)ci[best];  // bit position of the corrected base
        out_key = (key & ~(3ull << (2 * p))) | ((u64)cb[best] << (2 * p));
        ok = true;
        atomicAdd(&ctr->n_bc_corrected, 1ull);
      }
    }
  }
  bc_key[i] = out_key;
  bc_ok[i] = (ok || W.output_not_in_whitelist) ? 1 : 0;
}

// --bc-error-threshold 2 (chromap.cc:600-797) for one listed barcode i, by one warp.  Lanes stride over the candidates: every
// single change (i, base1), and every second change (j, base2) after it.  Ns (coded as A): only the first N is a first
// change, with all 4 bases; one N: the second change runs over the positions above it, 3 bases each; two Ns: it is the
// second N, with all 4 bases (so a key may be a candidate twice).  Hits go to hs / ht (room for cap) in enumeration order of
// the warp's ballots, the order does not matter: the choice sorts them.  Returns false, having decided nothing, when the
// barcode has more than cap hits.  pairs: the L(L-1)/2 position pairs i < j, two bytes each.
__device__ __forceinline__ int bc2_clamp_qual(u8 c) { int q = (int)(signed char)c - 33; q = q > 40 ? 40 : q; return q < 3 ? 3 : q; }
__device__ bool bc2_correct(const DevWhitelist &W, const u8 *bc_seq, const u8 *bc_qual, int L, u32 i, const u8 *pairs, double *hs, u32 *ht,
                            double *srt, int cap, u64 *bc_key, u8 *bc_ok, Counters *ctr) {
  const int lane = threadIdx.x & 31;
  const u8 *bc = bc_seq + (size_t)i * L, *qual = bc_qual + (size_t)i * L;
  const u64 key = barcode_seed(bc, L);
  const unsigned nm = __ballot_sync(0xffffffffu, lane < L && bc[L - 1 - lane] == 'N');  // bit p: an N at little-endian position p
  const int n_n = __popc(nm), n0 = __ffs(nm) - 1, n1 = __ffs(nm & (nm - 1)) - 1;
  const int m1 = L - 1 - n0;  // one N: second positions above it
  const int s1 = n_n == 0 ? 3 * L : 4, total = s1 + (n_n == 0 ? 9 * (L * (L - 1) / 2) : n_n == 1 ? 12 * m1 : 16);
  int nh = 0;  // hits so far (warp-uniform)
  for (int e0 = 0; e0 < total; e0 += 32) {
    const int e = e0 + lane;
    bool hit = false;
    double s = 0;
    u32 tag = 0;
    if (e < total) {
      int p1, t1, p2 = -1, t2 = 0;
      if (e < s1) { p1 = n_n == 0 ? e / 3 : n0; t1 = n_n == 0 ? e % 3 : e; }
      else {
        const int d = e - s1;
        if (n_n == 0) { const int pr = d / 9, r = d % 9; p1 = pairs[2 * pr]; p2 = pairs[2 * pr + 1]; t1 = r / 3; t2 = r % 3; }
        else if (n_n == 1) { const int r = d % (3 * m1); p1 = n0; t1 = d / (3 * m1); p2 = n0 + 1 + r / 3; t2 = r % 3; }
        else { p1 = n0; t1 = d >> 2; p2 = n1; t2 = d & 3; }
      }
      const u64 b1 = (((key >> (2 * p1)) & 3ull) + 1 + t1) & 3ull;
      u64 k = (key & ~(3ull << (2 * p1))) | (b1 << (2 * p1)), b2 = 0;
      if (p2 >= 0) { b2 = (((k >> (2 * p2)) & 3ull) + 1 + t2) & 3ull; k = (k & ~(3ull << (2 * p2))) | (b2 << (2 * p2)); }
      u64 cnt;
      if (wl_find(W, k, &cnt)) {
        hit = true;
        const int q = bc2_clamp_qual(qual[L - 1 - p1]) + (p2 >= 0 ? bc2_clamp_qual(qual[L - 1 - p2]) : 0);
        s = xmul(W.pow_tab[q], xdiv((double)cnt, W.num_sample));
        // (index1, base1, index2, base2) of BarcodeWithQual as one number in the same order: a single change has index2 = 0
        // and base2 = 0, below any base
        tag = (u32)(L - 1 - p1) << 11 | (u32)b1 << 9 | (p2 >= 0 ? (u32)(L - 1 - p2) << 3 | (u32)(b2 + 1) : 0u);
      }
    }
    const unsigned hm = __ballot_sync(0xffffffffu, hit);
    if (hit) {
      const int slot = nh + __popc(hm & ((1u << lane) - 1u));
      if (slot < cap) { hs[slot] = s; ht[slot] = tag; }
    }
    nh += __popc(hm);
    if (nh > cap) return false;
  }
  if (nh == 0) return true;  // not corrected: barcode_kernel's key and flag stand
  __syncwarp();
  u32 best = ht[0];
  bool accept = true;
  if (nh > 1) {
    // std::sort with std::greater<BarcodeWithQual> (utils.h:23-35), a strict order: each hit's rank is the number of hits above it
    int mine = -1;
    for (int a = lane; a < nh; a += 32) {
      const double sa = hs[a];
      const u32 ta = ht[a];
      int r = 0;
      for (int b = 0; b < nh; ++b) r += (hs[b] > sa || (hs[b] == sa && ht[b] > ta)) ? 1 : 0;
      srt[r] = sa;
      if (r == 0) mine = (int)ta;
    }
    const unsigned bm = __ballot_sync(0xffffffffu, mine >= 0);
    best = (u32)__shfl_sync(0xffffffffu, mine, __ffs(bm) - 1);
    __syncwarp();
    if (lane == 0) {  // the sum in the sorted order, as the reference adds it
      double sum = 0;
      for (int a = 0; a < nh; ++a) sum = xadd(sum, srt[a]);
      accept = xdiv(srt[0], sum) > W.prob_threshold;
    }
  }
  if (lane == 0 && accept) {
    const int p1 = L - 1 - (int)(best >> 11);
    u64 k = (key & ~(3ull << (2 * p1))) | ((u64)((best >> 9) & 3u) << (2 * p1));
    if (best & 7u) { const int p2 = L - 1 - (int)((best >> 3) & 31u); k = (k & ~(3ull << (2 * p2))) | ((u64)((best & 7u) - 1) << (2 * p2)); }
    bc_key[i] = k;
    bc_ok[i] = 1;
    atomicAdd(&ctr->n_bc_corrected, 1ull);
  }
  __syncwarp();
  return true;
}
// pass 0: the barcodes barcode_kernel listed, hit lists in shared memory; those with more hits go to the overflow list.
// pass 1: the overflow list, a Bc2Slab per warp.  Both stride over the count their list has on the device.
__global__ void __launch_bounds__(BC2_WARPS * 32) barcode_correct2_kernel(DevWhitelist W, const u8 *bc_seq, const u8 *bc_qual, int bc_len, u64 *bc_key, u8 *bc_ok,
                                                                            Counters *ctr, int pass) {
  __shared__ u8 pairs[32 * 31];
  __shared__ double hs[BC2_WARPS][BC2_SMEM_HITS], srt[BC2_WARPS][BC2_SMEM_HITS];
  __shared__ u32 ht[BC2_WARPS][BC2_SMEM_HITS];
  const int np = bc_len * (bc_len - 1) / 2;
  for (int t = threadIdx.x; t < np; t += blockDim.x) {  // pair t = (i, j), i < j, in the order j = 1, 2, ... and i < j
    int j = 1;
    while ((j + 1) * j / 2 <= t) ++j;
    pairs[2 * t] = (u8)(t - j * (j - 1) / 2); pairs[2 * t + 1] = (u8)j;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const u64 n = pass == 0 ? ctr->n_bc2_listed : ctr->n_bc2_overflow;
  const u32 *list = pass == 0 ? W.c2_list : W.c2_over;
  for (u64 w = (u64)blockIdx.x * BC2_WARPS + warp; w < n; w += (u64)gridDim.x * BC2_WARPS) {
    const u32 i = list[w];
    if (pass == 0) {
      if (!bc2_correct(W, bc_seq, bc_qual, bc_len, i, pairs, hs[warp], ht[warp], srt[warp], BC2_SMEM_HITS, bc_key, bc_ok, ctr) && lane == 0)
        W.c2_over[atomicAdd(&ctr->n_bc2_overflow, 1ull)] = i;
    } else {
      Bc2Slab &sl = W.c2_slab[(size_t)blockIdx.x * BC2_WARPS + warp];
      bc2_correct(W, bc_seq, bc_qual, bc_len, i, pairs, sl.score, sl.tag, sl.sorted, BC2_MAX_HITS, bc_key, bc_ok, ctr);
    }
  }
}

__global__ void barcode_gate_kernel(Scratch S, const u8 *bc_ok) {  // chromap.h:908-909: pairs outside the whitelist are not mapped
  const int slot = blockIdx.x * blockDim.x + threadIdx.x;
  if (slot >= S.n_slots) return;
  if (!bc_ok[slot_pair(S, slot)] && S.pmeta[slot].status == ST_OK) S.pmeta[slot].status = ST_DROP;
}

__global__ void compact_bc_kernel(int n_pairs, const int *n_rec, const u64 *offs, const u64 *bc_key, u64 *out) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= n_pairs) return;
  const int n = n_rec[pair];
  for (int j = 0; j < n; ++j) out[offs[pair] + j] = bc_key[pair];
}
