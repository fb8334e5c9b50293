// chromap_b200 — minimizers of one read by one thread (minimizer_generator.cc:7-139) and the layout of the minimizer
// records in the scratch tiers.  File:line citations are into the reference's src/.
#pragma once
#include "device_common.cuh"

// ---- minimizers -----------------------------------------------------------------------------------------------------
// utils.h:76-85 (Hash64) for 2k = 34 .. 46 bit keys, on 32-bit halves.  The 64-bit formulation costs ~40 instructions:
// the compiler emulates every shift-add and cannot know that the high word only holds 2k - 32 bits.  Here
//   (~key + (key << 21)) & mask  =  (key * (2^21 - 1) + mask) & mask        one wide multiply-add + one multiply-add
//   key ^ key >> s               touches only the low word (key >> s < 2^32 and the high word's bits shift out)
//   (key + (key << a) + (key << b)) & mask = (key * (1 + 2^a + 2^b)) & mask
// 18 instructions, same value as mix64(key, mask) for every key <= mask (checked against it in tests/test_abi.py's stage test).
template <int K>
__device__ __forceinline__ u64 mix64_k(u64 key) {
  static_assert(K >= 17 && K <= 23, "mix64_k: 2k - 14 must not exceed 32");
  constexpr u64 mask = (((u64)1) << (2 * K)) - 1;
  constexpr u32 mask_hi = (u32)(mask >> 32);
  u32 lo = (u32)key, hi = (u32)(key >> 32);
  auto mul = [&](u32 c, u64 add) {  // (hi:lo) = ((hi:lo) * c + add) & mask
    const u64 p = (u64)lo * c + add;
    hi = ((u32)(p >> 32) + hi * c) & mask_hi;
    lo = (u32)p;
  };
  mul((1u << 21) - 1u, mask);
  lo ^= __funnelshift_r(lo, hi, 24);
  mul(265u, 0);
  lo ^= __funnelshift_r(lo, hi, 14);
  mul(21u, 0);
  lo ^= __funnelshift_r(lo, hi, 28);
  mul((1u << 31) + 1u, 0);
  return ((u64)hi << 32) | lo;
}

// minimizer_generator.cc:7-139 for one read by one thread.  SEQ(i) -> i-th base (ASCII); EMIT(hash, pos << 1 | strand) is
// called once per minimizer, in the reference's order.  Returns nothing: the caller counts in EMIT.
//   KS > 0: k known at compile time (must equal k); WS > 0: w known at compile time (must equal w).
// With k odd a k-mer never equals its own reverse complement, so every position advances the window: the w-entry ring is
// then addressed by (position mod w) with the position loop unrolled w times — every ring access has a static index
// and the ring lives in registers.  Hashes are only computed once k valid bases are in (before that the entry is empty
// whatever the hashes are).  Otherwise (k even or unknown w) the same body runs with a run-time slot.
template <int KS, int WS, typename SeqF, typename EmitF>
__device__ __forceinline__ void minimizer_scan(SeqF SEQ, int len, int k_rt, int w_rt, EmitF EMIT) {
  constexpr bool fast = KS > 0 && (KS & 1) && WS > 0;
  const int k = KS > 0 ? KS : k_rt, w = WS > 0 ? WS : w_rt;
  const u64 shift = 2 * (k - 1);
  const u64 mask = (((u64)1) << (2 * k)) - 1;
  u64 fwd = 0, rev = 0;
  u64 rh[WS > 0 ? WS : CMX_W_MAX];
  u32 rp[WS > 0 ? WS : CMX_W_MAX];
#pragma unroll
  for (int i = 0; i < (WS > 0 ? WS : CMX_W_MAX); ++i) { rh[i] = ~0ull; rp[i] = ~0u; }
  u64 best_h = ~0ull;
  u32 best_p = ~0u;
  int run = 0, best_slot = 0;
  auto hash = [&](u64 x) { if constexpr (KS > 0) return mix64_k<KS>(x); else return mix64(x, mask); };
  // one position; returns false if the window does not advance (strand-symmetric k-mer, minimizer_generator.cc:50-52)
  auto step = [&](int pos, int slot) -> bool {
    const u32 b = base_code(SEQ(pos));
    u64 cur_h = ~0ull;
    u32 cur_p = ~0u;
    if (b < 4) {
      fwd = ((fwd << 2) | b) & mask;
      rev = (rev >> 2) | (((u64)(3 ^ b)) << shift);
      if (!fast && fwd == rev) return false;
      ++run;
      if (run >= k) {
        const u64 hf = hash(fwd), hr = hash(rev);
        const u32 strand = hf < hr ? 0u : 1u;
        cur_h = hash(strand ? hr : hf);
        cur_p = ((u32)pos << 1) | strand;
      }
    } else {
      run = 0;
    }
    rh[slot] = cur_h; rp[slot] = cur_p;
    if (run == w + k - 1 && best_h != ~0ull && best_h < cur_h) {  // first full window: equal minima behind the current one
#pragma unroll(WS > 0 ? WS : 1)
      for (int j = 1; j < (WS > 0 ? WS : CMX_W_MAX); ++j) {
        if (WS == 0 && j >= w) break;
        int q = slot + j; if (q >= w) q -= w;
        if (best_h == rh[q] && rp[q] != best_p) EMIT(rh[q], rp[q]);
      }
    }
    if (cur_h <= best_h) {
      if (run >= w + k && best_h != ~0ull) EMIT(best_h, best_p);
      best_h = cur_h; best_p = cur_p; best_slot = slot;
    } else if (slot == best_slot) {  // the minimum leaves the window: emit it, rescan (oldest to newest, later entries win ties)
      if (run >= w + k - 1 && best_h != ~0ull) EMIT(best_h, best_p);
      best_h = ~0ull;
#pragma unroll(WS > 0 ? WS : 1)
      for (int j = 1; j <= (WS > 0 ? WS : CMX_W_MAX); ++j) {
        if (WS == 0 && j > w) break;
        int q = slot + j; if (q >= w) q -= w;
        if (best_h >= rh[q]) { best_h = rh[q]; best_p = rp[q]; best_slot = q; }
      }
      if (run >= w + k - 1 && best_h != ~0ull) {
#pragma unroll(WS > 0 ? WS : 1)
        for (int j = 1; j <= (WS > 0 ? WS : CMX_W_MAX); ++j) {
          if (WS == 0 && j > w) break;
          int q = slot + j; if (q >= w) q -= w;
          if (best_h == rh[q] && best_p != rp[q]) EMIT(rh[q], rp[q]);
        }
      }
    }
    return true;
  };
  if constexpr (fast) {
    for (int base = 0; base < len; base += WS) {
#pragma unroll
      for (int j = 0; j < WS; ++j)
        if (base + j < len) step(base + j, j);
    }
  } else {
    int slot = 0;
    for (int pos = 0; pos < len; ++pos)
      if (step(pos, slot)) { if (++slot == w) slot = 0; }
  }
  if (best_h != ~0ull) EMIT(best_h, best_p);
}
// The same algorithm for odd k <= 21 and a compile-time w, built for a warp whose 32 lanes scan 32 different reads: the
// lanes take the reference's branches at different positions, so every branch body costs the whole warp.  Restated with
// no state but the window itself:
//   * an entry is ONE 64-bit key = hash << 20 | (0xFFFFF - (pos << 1 | strand)); empty = ~0.  Smaller key = smaller hash,
//     and among equal hashes the LATER position — exactly the entry the reference's scans settle on (`<=` on insertion,
//     `>=` in the rescan, minimizer_generator.cc:95-127);
//   * therefore the reference's running minimum is, after every position, simply the minimum key of the window (w - 1
//     64-bit minima, branch-free), and its three events read off the old minimum `best`, the new key `cur` and the key `old`
//     that `cur` overwrites:   cur <= best  -> the minimum is replaced;   old == best -> it leaves the window;
//   * identical hashes inside one window (low-complexity sequence) are what the tie loops are for; a 32-bit prefix test
//     keeps them out of the common path.
// Emission order and content are those of minimizer_scan (checked against it and against the oracle in the stage tests).
// RingT: the window's storage, ring[q] for q in [0, W) — a register array (`u64[W]`) or a strided view of shared memory
// (the fused front-end kernel keeps it there: the scan then needs no more registers than the hashes do).
template <int K, int W, typename SeqF, typename EmitF, typename RingT>
__device__ __forceinline__ void minimizer_scan_packed(SeqF SEQ, int len, EmitF EMIT, RingT ring) {
  static_assert((K & 1) && K >= 17 && K <= 21 && W >= 2, "minimizer_scan_packed: odd k, 2k + 20 <= 62");
  constexpr u64 mask = (((u64)1) << (2 * K)) - 1;
  constexpr int shift = 2 * (K - 1);
  constexpr u64 NONE = ~0ull;
  constexpr u32 PM = 0xFFFFFu;
  u64 fwd = 0, rev = 0;
#pragma unroll
  for (int i = 0; i < W; ++i) ring[i] = NONE;
  u64 best = NONE;
  int run = 0, slot = 0;  // slot = pos mod W: the entry `cur` replaces is the oldest one
  auto emit_key = [&](u64 key) { EMIT(key >> 20, PM - ((u32)key & PM)); };
#pragma unroll 1
  for (int pos = 0; pos < len; ++pos) {
    const u32 b = base_code(SEQ(pos));
    u64 cur = NONE;
    if (b < 4) {
      fwd = ((fwd << 2) | b) & mask;
      rev = (rev >> 2) | (((u64)(3 ^ b)) << shift);
      ++run;
      if (run >= K) {
        const u64 hf = mix64_k<K>(fwd), hr = mix64_k<K>(rev);
        const u32 strand = hf < hr ? 0u : 1u;
        cur = (mix64_k<K>(strand ? hr : hf) << 20) | (u64)(PM - (((u32)pos << 1) | strand));
      }
    } else {
      run = 0;
    }
    // first full window: entries equal to the minimum, behind the current one, oldest first (minimizer_generator.cc:86-93)
    if (run == W + K - 1 && best != NONE && (best >> 20) < (cur >> 20)) {
      for (int j = 1; j < W; ++j) {
        int q = slot + j; if (q >= W) q -= W;
        const u64 x = ring[q];
        if ((x >> 20) == (best >> 20) && x != best) emit_key(x);
      }
    }
    const u64 old = ring[slot];
    ring[slot] = cur;
    u64 m = cur;
#pragma unroll
    for (int q = 0; q < W; ++q) m = min(m, (u64)ring[q]);
    u64 out = NONE;  // the minimizer this position retires, if any
    bool left = false;
    if (cur <= best) {  // :95-100
      if (run >= W + K && best != NONE) out = best;
    } else if (old == best) {  // the minimum leaves the window (:101-127); best != NONE here
      if (run >= W + K - 1) { out = best; left = m != NONE; }
    }
    if (out != NONE) emit_key(out);
    int same_hi = 0;  // entries sharing the 32 high bits of the new minimum's key: more than one only in low-complexity sequence
    if (left) {
#pragma unroll
      for (int q = 0; q < W; ++q) same_hi += (u32)((u64)ring[q] >> 32) == (u32)(m >> 32);
    }
    if (same_hi > 1) {  // entries sharing the new minimum's hash, oldest first
      for (int j = 1; j <= W; ++j) {
        int q = slot + j; if (q >= W) q -= W;
        const u64 x = ring[q];
        if ((x >> 20) == (m >> 20) && x != m) emit_key(x);
      }
    }
    best = m;
    if (++slot == W) slot = 0;
  }
  if (best != NONE) emit_key(best);
}
// the same with the window in registers, as a shift register (oldest entry first) so that every access has a static index
template <int K, int W, typename SeqF, typename EmitF>
__device__ __forceinline__ void minimizer_scan_packed(SeqF SEQ, int len, EmitF EMIT) {
  static_assert((K & 1) && K >= 17 && K <= 21 && W >= 2, "minimizer_scan_packed: odd k, 2k + 20 <= 62");
  constexpr u64 mask = (((u64)1) << (2 * K)) - 1;
  constexpr int shift = 2 * (K - 1);
  constexpr u64 NONE = ~0ull;
  constexpr u32 PM = 0xFFFFFu;
  u64 fwd = 0, rev = 0;
  u64 ring[W];
#pragma unroll
  for (int i = 0; i < W; ++i) ring[i] = NONE;
  u64 best = NONE;
  int run = 0;
  auto emit_key = [&](u64 key) { EMIT(key >> 20, PM - ((u32)key & PM)); };
#pragma unroll 1
  for (int pos = 0; pos < len; ++pos) {
    const u32 b = base_code(SEQ(pos));
    u64 cur = NONE;
    if (b < 4) {
      fwd = ((fwd << 2) | b) & mask;
      rev = (rev >> 2) | (((u64)(3 ^ b)) << shift);
      ++run;
      if (run >= K) {
        const u64 hf = mix64_k<K>(fwd), hr = mix64_k<K>(rev);
        const u32 strand = hf < hr ? 0u : 1u;
        cur = (mix64_k<K>(strand ? hr : hf) << 20) | (u64)(PM - (((u32)pos << 1) | strand));
      }
    } else {
      run = 0;
    }
    if (run == W + K - 1) {  // once per N-free stretch (the same position in every lane of a warp whose reads have no N)
      if (best != NONE && (best >> 20) < (cur >> 20)) {  // ring[1 .. W-1]: the entries before `cur`, oldest first
#pragma unroll
        for (int q = 1; q < W; ++q) {
          const u64 x = ring[q];
          if ((x >> 20) == (best >> 20) && x != best) emit_key(x);
        }
      }
    }
    const u64 old = ring[0];
#pragma unroll
    for (int q = 0; q + 1 < W; ++q) ring[q] = ring[q + 1];
    ring[W - 1] = cur;
    u64 m = ring[0];
#pragma unroll
    for (int q = 1; q < W; ++q) m = min(m, ring[q]);
    u64 out = NONE;
    bool left = false;
    if (cur <= best) {
      if (run >= W + K && best != NONE) out = best;
    } else if (old == best) {
      if (run >= W + K - 1) { out = best; left = m != NONE; }
    }
    if (out != NONE) emit_key(out);
    int same_hi = 0;
    if (left) {
#pragma unroll
      for (int q = 0; q < W; ++q) same_hi += (u32)(ring[q] >> 32) == (u32)(m >> 32);
    }
    if (same_hi > 1) {
#pragma unroll
      for (int q = 0; q < W; ++q) {
        const u64 x = ring[q];
        if ((x >> 20) == (m >> 20) && x != m) emit_key(x);
      }
    }
    best = m;
  }
  if (best != NONE) emit_key(best);
}

// dispatch on the (k, w) pairs the presets use; anything else takes the run-time body
template <typename SeqF, typename EmitF>
__device__ __forceinline__ void minimizer_scan_any(SeqF SEQ, int len, int k, int w, EmitF EMIT) {
  if (k == 17 && w == 7 && len < (1 << 18)) minimizer_scan_packed<17, 7>(SEQ, len, EMIT);  // default, every preset
  else minimizer_scan<0, 0>(SEQ, len, k, w, EMIT);
}

