// chromap_b200 — overflow tiers, candidate supplementation / merge / paired-end filter for one pair by one CTA.
// SupplementCandidates (candidate_processor.cc:75-231), MergeCandidates (:345-414) and
// ReduceCandidatesForPairedEndReadOnOneDirection (:416-484) are sequential sweeps in the reference; here every one
// of them is restated as binary searches + prefix scans so that all CTA_NT threads work, with the lists staged in
// shared memory.  Each restatement is derived in the comment above it; results are identical element for element.
// File:line citations are into the reference's src/.
#pragma once
#include "pipeline_kernels.cuh"

// ---- CTA-wide scans (one value per thread) ---------------------------------------------------------------------
// exclusive prefix sum; *total = sum over the CTA.  s_warp: CTA_NT / 32 ints.
__device__ __forceinline__ int cta_scan_add(int v, int *s_warp, int *total) {
  const int NT = blockDim.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  int base = 0, tot = 0;
for (int i = 0; i < (NT >> 5); ++i) { const int w = s_warp[i]; if (i < wid) base += w; tot += w; }
  __syncthreads();
  *total = tot;
  return base + x - v;
}
// exclusive prefix maximum of non-negative ints (identity 0); *total = maximum over the CTA.
__device__ __forceinline__ int cta_scan_max(int v, int *s_warp, int *total) {
  const int NT = blockDim.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x = max(x, y); }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  int base = 0, tot = 0;
for (int i = 0; i < (NT >> 5); ++i) { const int w = s_warp[i]; if (i < wid) base = max(base, w); tot = max(tot, w); }
  __syncthreads();
  *total = tot;
  const int prev = __shfl_up_sync(0xffffffffu, x, 1);
  return lane == 0 ? base : max(base, prev);
}

// ---- MergeCandidates (candidate_processor.cc:345-414) ------------------------------------------------------------
// The reference merges two position-sorted lists (equal positions collapse into one entry carrying the larger count)
// and keeps an entry only if it lies more than e after the last KEPT entry.  Restated:
//   1. merged rank of list-1 entry i = i + #{p2 < p1[i]}, of list-2 entry j = j + #{p1 <= p2[j]}  (binary searches);
//      a list-1 entry with an equal twin in list 2 takes max(count) — the twin lands right behind it and can never be
//      kept (it is not more than e after anything at its own position), so it needs no special case.
//   2. an entry more than e after its predecessor is kept whatever came before ("head"), and the greedy rule restarts
//      there: the merged list splits into independent runs, each walked by the thread that owns its head.
//   3. kept entries are compacted in order (prefix sum).
// p1/c1 may alias op/oc (all reads of list 1 happen before the first barrier).  mp/mc/kf: work arrays of n1 + n2
// entries (shared or global).  Returns the merged size (the caller treats > cap as overflow, like the reference).
__device__ inline int cta_merge_cands(int e, const u64 *p1, const u8 *c1, int n1, const u64 *p2, const u8 *c2, int n2, u64 *mp, u8 *mc, u8 *kf, u64 *op,
                                      u8 *oc, int cap, int *s_warp) {
  const int NT = blockDim.x;
  const int tid = threadIdx.x;
  if (n1 == 0) {  // candidate_processor.cc:349-352: plain copy, no spacing rule
    for (int i = tid; i < n2 && i < cap; i += NT) { op[i] = p2[i]; oc[i] = c2[i]; }
    __syncthreads();
    return n2;
  }
  for (int i = tid; i < n1; i += NT) {
    const u64 p = p1[i];
    int a = 0, b = n2;
    while (a < b) { const int m = (a + b) >> 1; if (p2[m] < p) a = m + 1; else b = m; }
    u8 c = c1[i];
    if (a < n2 && p2[a] == p && c2[a] > c) c = c2[a];
    mp[i + a] = p; mc[i + a] = c;
  }
  for (int j = tid; j < n2; j += NT) {
    const u64 p = p2[j];
    int a = 0, b = n1;
    while (a < b) { const int m = (a + b) >> 1; if (p1[m] <= p) a = m + 1; else b = m; }
    mp[j + a] = p; mc[j + a] = c2[j];
  }
  __syncthreads();
  const int m = n1 + n2;
  const int C = (m + NT - 1) / NT;
  const int r0 = min(m, tid * C), r1 = min(m, r0 + C);
  int mine = 0;
  for (int i = r0; i < r1; ++i) {
    if (!(i == 0 || mp[i] > mp[i - 1] + (u64)e)) continue;  // not a head: walked by the owner of its run's head
    u64 last = mp[i];
    kf[i] = 1;
    for (int q = i + 1; q < m && !(mp[q] > mp[q - 1] + (u64)e); ++q) {
      const bool keep = mp[q] > last + (u64)e;
      kf[q] = keep;
      if (keep) last = mp[q];
    }
  }
  __syncthreads();
  for (int i = r0; i < r1; ++i) mine += kf[i];
  int total;
  int at = cta_scan_add(mine, s_warp, &total);
  for (int i = r0; i < r1; ++i)
    if (kf[i]) { if (at < cap) { op[at] = mp[i]; oc[at] = mc[i]; } ++at; }
  __syncthreads();
  return total;
}

// ---- ReduceCandidatesForPairedEndReadOnOneDirection (candidate_processor.cc:416-484) ------------------------------
// The reference sweeps both position-sorted lists with two pointers.  What it emits, restated per entry:
//   * list-1 entry i is classified while the list-2 pointer stands on lo = first j with p2[j] + dist >= p1[i]; if lo is
//     past the end the sweep has stopped and i is dropped.  i is PAIRED iff p2[lo] <= p1[i] + dist.  Symmetrically
//     list-2 entry j is PAIRED iff some p1[i] lies within dist of it; an unpaired j is skipped while the list-1 pointer
//     stands on the first i with p1[i] > p2[j] + dist (dropped if there is none).
//   * paired entries are always kept.  An unpaired entry is kept iff it lies on the same reference sequence as the
//     entry the other pointer stands on, its count is >= the running maximum (initially 6) of the counts of the PAIRED
//     entries of its own list before it, and fewer than 5 unpaired entries of its list were kept before it
//     ("j >= prev_end" in the reference is exactly "j is not paired").
//   * both outputs are in list order.
// So: two binary searches per entry, an exclusive prefix maximum over the paired counts, a prefix count of the
// qualifying unpaired entries (the first 5 survive), and a compaction.  f1 / f2: byte flags, n1 / n2 entries.
__device__ inline void cta_pe_filter(u32 dist, const u64 *p1, const u8 *c1, int n1, const u64 *p2, const u8 *c2, int n2, u64 *o1p, u8 *o1c, int *na,
                                     u64 *o2p, u8 *o2c, int *nb, u8 *f1, u8 *f2, int *s_warp) {
  const int NT = blockDim.x;
  const int tid = threadIdx.x;
  for (int i = tid; i < n1; i += NT) {
    const u64 p = p1[i];
    int a = 0, b = n2;
    while (a < b) { const int m = (a + b) >> 1; if (p > p2[m] + dist) a = m + 1; else b = m; }
    u8 f = 0;
    if (a < n2) {
      const u64 q = p2[a];
      if (!(q > p + dist)) f = 1;
      else if ((p >> 32) == (q >> 32)) f = 2;
    }
    f1[i] = f;
  }
  for (int j = tid; j < n2; j += NT) {
    const u64 q = p2[j];
    int a = 0, b = n1;
    while (a < b) { const int m = (a + b) >> 1; if (q > p1[m] + dist) a = m + 1; else b = m; }
    u8 f = 0;
    if (a < n1) {
      const u64 p = p1[a];
      if (!(p > q + dist)) f = 1;
      else if ((p >> 32) == (q >> 32)) f = 2;
    }
    f2[j] = f;
  }
  __syncthreads();
  const int C1 = (n1 + NT - 1) / NT, C2 = (n2 + NT - 1) / NT;
  const int a0 = min(n1, tid * C1), a1 = min(n1, a0 + C1), b0 = min(n2, tid * C2), b1 = min(n2, b0 + C2);
  // running maxima (one scan per list) and paired counts (both lists packed into one scan: list sizes < 2^15)
  int mx = 0, np = 0;
  for (int i = a0; i < a1; ++i) if (f1[i] == 1) { mx = max(mx, (int)c1[i]); ++np; }
  int mx2 = 0, np2 = 0;
  for (int j = b0; j < b1; ++j) if (f2[j] == 1) { mx2 = max(mx2, (int)c2[j]); ++np2; }
  int tot;
  const int pm1 = cta_scan_max(mx, s_warp, &tot);
  const int pm2 = cta_scan_max(mx2, s_warp, &tot);
  const int pp = cta_scan_add(np | (np2 << 16), s_warp, &tot);
  // qualifying unpaired entries
  int run = max(6, pm1), nq1 = 0;
  for (int i = a0; i < a1; ++i) {
    const u8 f = f1[i];
    if (f == 1) run = max(run, (int)c1[i]);
    else if (f == 2) { if ((int)c1[i] >= run) ++nq1; else f1[i] = 0; }
  }
  int run2 = max(6, pm2), nq2 = 0;
  for (int j = b0; j < b1; ++j) {
    const u8 f = f2[j];
    if (f == 1) run2 = max(run2, (int)c2[j]);
    else if (f == 2) { if ((int)c2[j] >= run2) ++nq2; else f2[j] = 0; }
  }
  int totq;
  const int pq = cta_scan_add(nq1 | (nq2 << 16), s_warp, &totq);
  int paired_before = pp & 0xffff, qual_before = pq & 0xffff;
  for (int i = a0; i < a1; ++i) {
    const u8 f = f1[i];
    if (f == 1) { const int at = paired_before + min(qual_before, 5); o1p[at] = p1[i]; o1c[at] = c1[i]; ++paired_before; }
    else if (f == 2) { if (qual_before < 5) { const int at = paired_before + qual_before; o1p[at] = p1[i]; o1c[at] = c1[i]; } ++qual_before; }
  }
  paired_before = pp >> 16; qual_before = pq >> 16;
  for (int j = b0; j < b1; ++j) {
    const u8 f = f2[j];
    if (f == 1) { const int at = paired_before + min(qual_before, 5); o2p[at] = p2[j]; o2c[at] = c2[j]; ++paired_before; }
    else if (f == 2) { if (qual_before < 5) { const int at = paired_before + qual_before; o2p[at] = p2[j]; o2c[at] = c2[j]; } ++qual_before; }
  }
  *na = (tot & 0xffff) + min(totq & 0xffff, 5);
  *nb = (tot >> 16) + min(totq >> 16, 5);
  __syncthreads();
}

// ---- mate-guided lookup (index.cc:351-489), cooperatively --------------------------------------------------------
// The windows around the mate's best candidates come from its (staged) list.  For a multi-occurrence minimizer the
// reference runs, per window, a binary search that starts at the previous window's last probe (`prev_l`) and then
// walks the occurrence list from that last probe (index.cc:443-479) — so what is emitted depends on the probe path, and
// the path of window b depends on the result of window b-1.  The dependency is thin, though:
//   * comparisons against a sorted list only depend on where the probe lies relative to LB = first entry >= window start and
//     E = number of entries equal to it; occurrence entries are distinct positions (one k-mer per reference position, Hash64
//     is a bijection on k-mers; cmx_upload_index / cmx_build_index verify it and refuse an index that breaks it), so E is 0 or 1;
//   * with E = 0 the search ends with l = LB, r = LB - 1 and its last probe is LB - 1 or LB (which one depends on the path);
//     with E = 1 it stops on LB.  So window b can only be entered with prev_l = LB(b-1) - 1 or LB(b-1).
// One WARP takes one minimizer, one LANE one window: lane b finds LB, E and UB = first entry > window end in the occurrence
// list (the only memory accesses), replays the search arithmetically for both possible entries, and the chain through
// the windows is a prefix "scan" over 2-state transition functions (5 shuffle steps).  Emission [first, max(first, UB))
// goes through a shared counter (order is irrelevant: the hits are sorted next).  No block barrier inside.
#define RESCUE_MAXWIN 300
#define PC_CTA_NT_MAX 512  // threads of pair_candidates_cta_kernel at most (the block-wide primitives size themselves from blockDim)
struct RescueShared {
  u64 win_lo[RESCUE_MAXWIN], win_hi[RESCUE_MAXWIN];
  int i[8];
  int warp[PC_CTA_NT_MAX / 32];
};
// mmv / mmp: this read's minimizer records (shared memory).  mate_pos / mate_cnt: the mate's candidates on the strand
// that guides the search.  Returns +max count or -max count (bail-out, index.cc:371-380) on every thread; *nh_out =
// number of hits appended to `hits` (global, sorted here when they fit `cap`).
__device__ inline int cta_rescue(const DevParams &P, const DevIndex &ix, int strand, u32 range, int n_mm, const u64 *mmv, const u32 *mmp,
                                 const u64 *mate_pos, const u8 *mate_cnt, int n_mate, u32 *rep_len, u64 *hits, int cap, u64 *sm, int sm_cap,
                                 RescueShared &R, int *nh_out) {
  const int NT = blockDim.x;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // best count and how many candidates carry it
  int mx = 0;
  for (int i = tid; i < n_mate; i += NT) mx = max(mx, (int)mate_cnt[i]);
  int max_cnt;
  cta_scan_max(mx, R.warp, &max_cnt);
  int nb = 0;
  for (int i = tid; i < n_mate; i += NT) nb += mate_cnt[i] == max_cnt;
  int n_best;
  cta_scan_add(nb, R.warp, &n_best);
  *nh_out = 0;
  if (n_best >= 300 || n_mate > P.f0 || (max_cnt <= P.min_seeds && n_best >= 200)) return -max_cnt;
  if (tid == 0) {  // merged windows (index.cc:383-412): at most n_best < 300 of them
    int nw = 0;
    for (int i = 0; i < n_mate; ++i) {
      if (mate_cnt[i] != max_cnt) continue;
      const u64 lo = mate_pos[i] < range ? 0 : mate_pos[i] - range, hi = mate_pos[i] + range;
      if (nw > 0 && !(R.win_hi[nw - 1] < lo)) R.win_hi[nw - 1] = hi;
      else { R.win_lo[nw] = lo; R.win_hi[nw] = hi; ++nw; }
    }
    R.i[2] = nw;
    R.i[3] = 0;  // hit counter
  }
  __syncthreads();
  const int nw = R.i[2];
  // singletons: one candidate each
  for (int mi = tid; mi < n_mm; mi += NT) {
    if ((mmp[mi] >> 30) != 1) continue;
    bool same;
    const u64 cp = hit_to_candidate(P.k, mmv[mi], (mmp[mi] & 0x3FFFFFFFu) >> 1, mmp[mi] & 1u, &same);
    if ((same && strand == 0) || (!same && strand == 1)) { const int at = atomicAdd(&R.i[3], 1); if (at < cap) hits[at] = cp; }
  }
  // multi-occurrence minimizers: one warp each
  for (int mi = wid; mi < n_mm; mi += (NT >> 5)) {
    if ((mmp[mi] >> 30) != 2) continue;
    const u64 val = mmv[mi];
    const u64 *O = ix.occ + (u32)(val >> 32);
    const int n = (int)(u32)val;
    const u32 rpos = (mmp[mi] & 0x3FFFFFFFu) >> 1, rstrand = mmp[mi] & 1u;
    int c_lb = 0, c_e = 0, c_s = 0;  // window before this chunk: LB, E and which of {LB - 1, LB} its last probe was
    for (int b0 = 0; b0 < nw; b0 += 32) {
      const int b = b0 + lane;
      const bool live = b < nw;
      int lb = 0, eq = 0, ub = 0;
      if (live) {
        const u64 lo = R.win_lo[b], hi = R.win_hi[b];
        int a = 0, z = n;  // (two-way here: with a warp's 32 searches in flight the four-way variant's extra loads cost more than its shorter chain saves)
        while (a < z) { const int m = (a + z) >> 1; if ((__ldg(&O[m]) >> 1) < lo) a = m + 1; else z = m; }
        lb = a;
        eq = (lb < n && (__ldg(&O[lb]) >> 1) == lo) ? 1 : 0;  // distinct positions (checked when the index is installed): E <= 1
        // entries inside the window are few: gallop from LB + E instead of bisecting [LB, n)
        int step = 1, lo_i = lb + eq, hi_i = lb + eq;
        while (hi_i < n && (__ldg(&O[hi_i]) >> 1) <= hi) { lo_i = hi_i + 1; hi_i += step; step <<= 1; }
        if (hi_i > n) hi_i = n;
        while (lo_i < hi_i) { const int m = (lo_i + hi_i) >> 1; if ((__ldg(&O[m]) >> 1) <= hi) lo_i = m + 1; else hi_i = m; }
        ub = lo_i;
      }
      // the window before this lane's
      int p_lb = __shfl_up_sync(0xffffffffu, lb, 1), p_e = __shfl_up_sync(0xffffffffu, eq, 1);
      if (lane == 0) { p_lb = c_lb; p_e = c_e; }
      // transition: state s = "the last probe was LB (1) or LB - 1 (0)"; f = (new state if old state 0) | (.. if old state 1) << 1
      u32 f = 2u;  // identity for lanes past the last window
      if (live) {
        int o0, o1;
        if (b == 0) o0 = o1 = rescue_replay(0, n, lb, lb + eq);  // the first window starts from 0
        else {
          o1 = rescue_replay(p_lb, n, lb, lb + eq);
          o0 = p_e ? o1 : rescue_replay(max(p_lb - 1, 0), n, lb, lb + eq);
        }
        f = (o0 == lb ? 1u : 0u) | (o1 == lb ? 2u : 0u);
      }
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const u32 g = __shfl_up_sync(0xffffffffu, f, o);  // the function of the lanes before: apply it first
        if (lane >= o) f = (((f >> (g & 1u)) & 1u)) | (((f >> ((g >> 1) & 1u)) & 1u) << 1);
      }
      const int s_out = (int)((f >> c_s) & 1u);
      if (live) {
        const int first = lb - 1 + s_out, end = max(first, ub);
        for (int oi = first; oi < end; ++oi) {
          bool same;
          const u64 cp = hit_to_candidate(P.k, __ldg(&O[oi]), rpos, rstrand, &same);
          if ((same && strand == 0) || (!same && strand == 1)) { const int at = atomicAdd(&R.i[3], 1); if (at < cap) hits[at] = cp; }
        }
      }
      c_lb = __shfl_sync(0xffffffffu, lb, 31); c_e = __shfl_sync(0xffffffffu, eq, 31); c_s = __shfl_sync(0xffffffffu, s_out, 31);
    }
  }
  __syncthreads();
  const int nh = R.i[3];
  *nh_out = nh;
  if (tid == 0) {
    RepStats st = {0u, 0xFFFFFFFFu, 0};
    for (int mi = 0; mi < n_mm; ++mi)
      if ((mmp[mi] >> 30) == 2 && (u32)mmv[mi] >= (u32)P.f0) rep_update(P.k, P.w, (mmp[mi] & 0x3FFFFFFFu) >> 1, st);
    *rep_len = st.len;
  }
  __syncthreads();
  if (nh <= cap) cta_sort_keys(hits, nh, sm, sm_cap);
  return max_cnt;
}

// ---- the kernel ------------------------------------------------------------------------------------------------------
// One CTA per pair: CTA_NT threads in the overflow tiers; ONE WARP per pair (blockDim = 32, `list` = the pairs to take) for
// the tier-0 pairs that need the mate-guided lookup — the block-wide primitives above size themselves from blockDim.  Dynamic shared memory (bytes): sort buffer sm_cap * 8 | cluster / merge flags 3 * sm_cap |
// four staged candidate lists lcap * 8 each | minimizer values maxmm * 8 | minimizer words maxmm * 4 | list counts
// 4 * lcap | filter flags 2 * fcap.  Lists longer than lcap stay in global memory (same code, other pointers).
__host__ __device__ inline size_t pair_candidates_cta_smem(int sm_cap, int lcap, int maxmm, int fcap) {
  return (size_t)sm_cap * 11 + (size_t)lcap * 4 * 9 + (size_t)maxmm * 12 + (size_t)fcap * 2 + 64;
}
__device__ inline void pair_candidates_cta_pair(const DevParams &P, const DevIndex &ix, const Scratch &S, Counters *ctr, int sm_cap, int lcap, int fcap,
                                                int slot, u64 *sm, RescueShared &RS) {
  const Caps c = S.caps;
  u8 *aux = (u8 *)(sm + sm_cap);                               // 3 * sm_cap bytes (multiple of 8: sm_cap is a power of two >= 8)
  u64 *s_lp = (u64 *)(aux + 3 * (size_t)sm_cap);               // [4][lcap]
  u64 *s_mmv = s_lp + 4 * (size_t)lcap;                        // [maxmm]
  u32 *s_mmp = (u32 *)(s_mmv + c.maxmm);                       // [maxmm]
  u8 *s_lc = (u8 *)(s_mmp + c.maxmm);                          // [4][lcap]
  u8 *fl_a = s_lc + 4 * (size_t)lcap, *fl_b = fl_a + fcap;     // [fcap] each
  const int NT = blockDim.x, tid = threadIdx.x;
  PairMeta &pm = S.pmeta[slot];
  if (pm.status != ST_OK) return;
  ReadMeta *rm = S.rmeta + 2 * slot;
  auto CP = [&](int mate, int set, int strand) { return S.cand_pos + cand_base(0, c, 2 * slot + mate, set, strand); };
  auto CC = [&](int mate, int set, int strand) { return S.cand_cnt + cand_base(0, c, 2 * slot + mate, set, strand); };
  if (P.se) {
    const int a1 = rm[0].n_cand[0] + rm[0].n_cand[1];
    __syncthreads();
    if (tid == 0) { if (rm[0].n_mm == 0 || a1 == 0) pm.status = ST_DROP; else atomicAdd(&ctr->n_candidates, (u64)a1); }
    return;
  }
  if (rm[0].n_mm == 0 || rm[1].n_mm == 0) { __syncthreads(); if (tid == 0) pm.status = ST_DROP; return; }
  if (P.split) {
    const int a1 = rm[0].n_cand[0] + rm[0].n_cand[1], a2 = rm[1].n_cand[0] + rm[1].n_cand[1];
    __syncthreads();
    if (tid == 0) { if (!(a1 > 0 && a2 > 0)) pm.status = ST_DROP; else atomicAdd(&ctr->n_candidates, (u64)(a1 + a2)); }
    return;
  }
  // list q = mate * 2 + strand; lp/lc point at the staged copy when the list fits, at set 0 in global memory otherwise
  int nq[4];
  const u64 *lp[4];
  const u8 *lc[4];
  const int n_mm2[2] = {rm[0].n_mm, rm[1].n_mm};
  auto stage = [&]() {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      nq[q] = rm[q >> 1].n_cand[q & 1];
      const u64 *gp = CP(q >> 1, 0, q & 1);
      const u8 *gc = CC(q >> 1, 0, q & 1);
      if (nq[q] <= lcap) {
        for (int i = tid; i < nq[q]; i += NT) { s_lp[q * lcap + i] = gp[i]; s_lc[q * lcap + i] = gc[i]; }
        lp[q] = s_lp + q * lcap; lc[q] = s_lc + q * lcap;
      } else { lp[q] = gp; lc[q] = gc; }
    }
    __syncthreads();
  };
  stage();
  // supplementation test (candidate_processor.cc:135-154): no candidate of the read reaches half its minimizers
  bool need[2];
#pragma unroll
  for (int mate = 0; mate < 2; ++mate) {
    const u32 half = (u32)n_mm2[mate] / 2;
    int hit = 0;
#pragma unroll
    for (int s = 0; s < 2; ++s)
      for (int i = tid; i < nq[mate * 2 + s]; i += NT) hit |= lc[mate * 2 + s][i] >= half;
    need[mate] = !__syncthreads_or(hit);
  }
  const u32 range = 2u * (u32)P.max_insert;
  int ret = 0;
  for (int mate = 0; mate < 2; ++mate) {
    if (!need[mate]) continue;
    ReadMeta &me = rm[mate];
    const int n_mm = n_mm2[mate];
    const size_t sr = 2 * slot + mate;
    {
      const size_t mb0 = mm_base(S, slot, mate);
      const int ms = mm_stride(S);
      for (int i = tid; i < n_mm; i += NT) { s_mmv[i] = S.mm_val[mb0 + (size_t)i * ms]; s_mmp[i] = S.mm_pos[mb0 + (size_t)i * ms]; }
    }
    __syncthreads();
    u64 *hp = S.hits + (sr * 2 + 0) * c.hc, *hn = S.hits + (sr * 2 + 1) * c.hc;
    int pr = 0, nr = 0;
    bool ovf = false;
    const int o0 = (1 - mate) * 2;
    if (nq[o0] > 0) {
      int nh;
      pr = cta_rescue(P, ix, 1, range, n_mm, s_mmv, s_mmp, lp[o0], lc[o0], nq[o0], &me.rep_len, hn, c.hc, sm, sm_cap, RS, &nh);
      if (nh > c.hc) ovf = true;
      else {
        const int na = cta_cluster_par(P.e, 1, (u32)n_mm, hn, nh, CP(mate, 2, 1), CC(mate, 2, 1), c.cc, sm, sm_cap, aux, &RS.i[4]);
        if (na > c.cc) ovf = true; else if (tid == 0) me.n_aug[1] = na;
      }
    }
    if (!ovf && nq[o0 + 1] > 0) {
      int nh;
      nr = cta_rescue(P, ix, 0, range, n_mm, s_mmv, s_mmp, lp[o0 + 1], lc[o0 + 1], nq[o0 + 1], &me.rep_len, hp, c.hc, sm, sm_cap, RS, &nh);
      if (nh > c.hc) ovf = true;
      else {
        const int na = cta_cluster_par(P.e, 1, (u32)n_mm, hp, nh, CP(mate, 2, 0), CC(mate, 2, 0), c.cc, sm, sm_cap, aux, &RS.i[4]);
        if (na > c.cc) ovf = true; else if (tid == 0) me.n_aug[0] = na;
      }
    }
    if (ovf) { __syncthreads(); if (tid == 0) pm.status = ST_OVERFLOW; return; }  // uniform: every thread computed the same ovf
    if (((pr < 0 && nr > 0 && -pr >= nr) || (pr > 0 && nr < 0 && pr <= -nr)) && nq[mate * 2] + nq[mate * 2 + 1] == 0) ret = 1;
    __syncthreads();  // n_aug visible to everyone
  }
  // merges: augmented candidates (set 2) into set 0, one (mate, strand) list after the other, the whole CTA on each
  bool merged = false;
  for (int q = 0; q < 4; ++q) {
    const int mate = q >> 1, s = q & 1;
    if (!need[mate]) continue;
    const int n2 = rm[mate].n_aug[s];
    if (n2 <= 0) continue;
    const int m = nq[q] + n2;
    u64 *mp;
    u8 *mc, *kf;
    if (m <= sm_cap) { mp = sm; mc = aux; kf = aux + sm_cap; }                           // sort buffer and its flag area are free here
    else { mp = CP(mate, 1, 0); mc = CC(mate, 1, 0); kf = fl_a; }                        // both strands' buffer sets: 2 * cc entries
    const int n = (m > 2 * c.cc || (m > sm_cap && m > fcap)) ? c.cc + 1
                                                             : cta_merge_cands(P.e, lp[q], lc[q], nq[q], CP(mate, 2, s), CC(mate, 2, s), n2, mp, mc, kf,
                                                                               CP(mate, 0, s), CC(mate, 0, s), c.cc, RS.warp);
    if (n > c.cc) { __syncthreads(); if (tid == 0) pm.status = ST_OVERFLOW; return; }
    if (tid == 0) rm[mate].n_cand[s] = n;
    merged = true;
  }
  if (merged) { __syncthreads(); stage(); }
  int nc1 = nq[0] + nq[1], nc2 = nq[2] + nq[3];
  if (nc1 > 0 && nc2 > 0) {
    // MoveCandidiatesToBuffer + ReduceCandidatesForPairedEndRead (chromap.h:1036-1052): the staged copies are the buffer;
    // a list too long to stage is first copied to the buffer set in global memory
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (nq[q] > lcap) {
        u64 *dst = CP(q >> 1, 1, q & 1);
        u8 *dstc = CC(q >> 1, 1, q & 1);
        for (int i = tid; i < nq[q]; i += NT) { dst[i] = lp[q][i]; dstc[i] = lc[q][i]; }
        lp[q] = dst; lc[q] = dstc;
      }
    __syncthreads();
    int a, b, a2, b2;
    cta_pe_filter((u32)P.max_insert, lp[0], lc[0], nq[0], lp[3], lc[3], nq[3], CP(0, 0, 0), CC(0, 0, 0), &a, CP(1, 0, 1), CC(1, 0, 1), &b, fl_a, fl_b, RS.warp);
    cta_pe_filter((u32)P.max_insert, lp[1], lc[1], nq[1], lp[2], lc[2], nq[2], CP(0, 0, 1), CC(0, 0, 1), &a2, CP(1, 0, 0), CC(1, 0, 0), &b2, fl_a, fl_b, RS.warp);
    if (tid == 0) {
      rm[0].n_cand[0] = a; rm[1].n_cand[1] = b; rm[0].n_cand[1] = a2; rm[1].n_cand[0] = b2;
    }
    nc1 = a + a2; nc2 = b + b2;
  }
  if (tid != 0) return;
  pm.sup = ret;
  if (!(nc1 > 0 && nc2 > 0)) { pm.status = ST_DROP; return; }
  atomicAdd(&ctr->n_candidates, (u64)(nc1 + nc2));
}

__global__ void __launch_bounds__(PC_CTA_NT_MAX) pair_candidates_cta_kernel(DevParams P, DevIndex ix, Scratch S, Counters *ctr, int sm_cap, int lcap, int fcap,
                                                                     const int *list, const int *list_count) {
  extern __shared__ u64 sm[];
  __shared__ RescueShared RS;
  if (!list) { pair_candidates_cta_pair(P, ix, S, ctr, sm_cap, lcap, fcap, (int)blockIdx.x, sm, RS); return; }
  const int n = *list_count;  // persistent: the grid strides over the listed pairs
  for (int b = blockIdx.x; b < n; b += gridDim.x) {
    pair_candidates_cta_pair(P, ix, S, ctr, sm_cap, lcap, fcap, list[b], sm, RS);
    __syncthreads();
  }
}
