"""Index construction of the CUDA path (chromap_b200/csrc/index_build.cuh: `ref_minimizers_kernel` — the reference's minimizers
from independent 2048-base chunks, each warmed up 2(w+k) bases early —, `multi_flag_kernel`, `fold_runs_kernel`, and the
khash upload kernels `khash_count_kernel` / `khash_insert_kernel`) run UNCHANGED on the host emulation (tests/cta_emu.h) in
`build_index_on_device`'s sequence, std::sort / a prefix sum playing CUB, against the oracle's `orc_index_build`
(Index::Construct, index.cc:12-89; shown equal to `chromap -i` by tests/test_oracle_golden.py): every key with its singleton
flag and value, occurrence offsets and counts, the occurrence table entry by entry.  References with N runs, soft-masked
bases, sequences shorter than a chunk and shorter than k, lengths off the chunk grid, tandem repeats, planted copies; three (k, w);
and a reference holding every byte 0x01-0xFF but LF and CR (`base_code` against the oracle's CharToUint8 on all of them)."""
from tests import emu

MAIN = r'''
extern "C" {
#include "%(orc_h)s"
}
int main() {
  std::mt19937 g(101);
  long bad = 0, cases = 0, keys_total = 0, occ_total = 0;
  const int KW[3][2] = {{17, 7}, {21, 10}, {16, 5}};
  for (int it = 0; it < 10; ++it) {
    const int k = KW[it %% 3][0], w = KW[it %% 3][1];
    // ---- reference
    std::vector<std::string> seqs;
    if (it == 9) {   // every byte 0x01-0xFF but '\n' and '\r', 24 times each, between 30 random bases on either side
      std::vector<int> mid;
      for (int q = 0; q < 24; ++q) for (int b = 1; b < 256; ++b) if (b != 10 && b != 13) mid.push_back(b);
      std::shuffle(mid.begin(), mid.end(), g);
      for (size_t i = 0; i < mid.size(); i += 2000) {
        std::string s;
        for (size_t q = i; q < std::min(mid.size(), i + 2000); ++q) {
          for (int x = 0; x < 30; ++x) s.push_back("ACGT"[g() %% 4]);
          s.push_back((char)mid[q]);
          for (int x = 0; x < 30; ++x) s.push_back("ACGT"[g() %% 4]);
        }
        seqs.push_back(s);
      }
    }
    const int n_seq = it == 9 ? 0 : 2 + (int)(g() %% 4);
    for (int q = 0; q < n_seq; ++q) {
      size_t L = q == 0 ? 30000 + g() %% 9000 : q == 1 ? 2048 * 3 : q == 2 ? 10 + g() %% 30 : 300 + g() %% 5000;   // off the chunk grid, on it, shorter than k + w, shorter than a chunk
      std::string s(L, 'A');
      for (auto &c : s) c = "ACGT"[g() %% 4];
      seqs.push_back(s);
    }
    std::string &big = seqs[0];
    if (it != 9) {   // planted copies, a tandem repeat, N runs and soft-masking in the first sequence
      std::string seg(700, 'A'); for (auto &c : seg) c = "ACGT"[g() %% 4];
      for (int q = 0; q < 14; ++q) big.replace(100 + g() %% (big.size() - 1000), 700, seg);                       // planted copies: multi-occurrence keys
      for (int i = 0; i < 600; ++i) big[5000 + i] = "ACG"[i %% 3];                                                // tandem repeat: ties inside a window
      big.replace(9000, 120, std::string(120, 'N'));
      big.replace(2040, 20, std::string(20, 'N'));                                                                // an N run across a chunk boundary
      for (int q = 0; q < 2000; ++q) { const size_t at = g() %% big.size(); big[at] = (char)tolower(big[at]); }
    }
    std::string concat; std::vector<uint64_t> offs{0};
    for (auto &s : seqs) { concat += s; offs.push_back(concat.size()); }
    orc_reference *oref = orc_reference_from_memory((uint32_t)seqs.size(), concat.data(), offs.data(), nullptr);
    orc_index *oix = orc_index_build(oref, k, w);
    // ---- build_index_on_device's sequence
    std::string refmem(64, '\0');
    std::vector<u64> off; std::vector<u32> len;
    for (auto &s : seqs) { off.push_back(refmem.size()); len.push_back((u32)s.size()); refmem += s; refmem.append(64 + (64 - refmem.size() %% 64) %% 64, '\0'); }
    u64 total = 0;
    std::vector<u64> c_off; std::vector<u32> c_len, c_rid, c_start;
    for (size_t r = 0; r < off.size(); ++r) { total += len[r]; for (u64 s = 0; s < len[r]; s += IB_CHUNK) { c_off.push_back(off[r]); c_len.push_back(len[r]); c_rid.push_back((u32)r); c_start.push_back((u32)s); } }
    const size_t n_chunks = c_off.size();
    const u64 cap = (u64)((double)total * std::min(1.0, 2.6 / (double)(w + 1))) + 1024 * off.size() + 4096;
    std::vector<u64> h1(cap), t1(cap);
    unsigned long long cnt = 0;
    emu_grid_serial((int)((n_chunks + 127) / 128), 128, [&]() { ref_minimizers_kernel((const u8 *)refmem.data(), c_off.data(), c_len.data(), c_rid.data(), c_start.data(), n_chunks, k, w, h1.data(), t1.data(), &cnt, cap); });
    const size_t n = (size_t)cnt;
    ++cases;
    bool ok = n > 0 && n <= cap;
    std::vector<std::pair<u64, u64>> hh(n);
    for (size_t i = 0; i < n; ++i) hh[i] = {h1[i], t1[i]};
    std::sort(hh.begin(), hh.end());                                  // by (hash, hit): CUB's two stable passes
    for (size_t i = 0; i < n; ++i) { h1[i] = hh[i].first; t1[i] = hh[i].second; }
    std::vector<u32> multi(n + 1), occidx(n + 1);
    unsigned long long n_heads = 0;
    emu_grid_serial((int)((n + 255) / 256), 256, [&]() { multi_flag_kernel(h1.data(), n, multi.data(), &n_heads); });
    u32 run = 0;
    for (size_t i = 0; i < n; ++i) { occidx[i] = run; run += multi[i]; }
    const u32 n_occ = run;
    u64 n_slots = 1024; while (n_slots < 2 * n_heads) n_slots <<= 1;
    int lg = 0; while ((1ull << lg) < n_slots) ++lg;
    std::vector<ulonglong2> slots((size_t)n_slots, ulonglong2{CMX_EMPTY_KEY, ~0ull});
    std::vector<u64> occ((size_t)n_occ + 1);
    emu_grid_serial((int)((n + 255) / 256), 256, [&]() { fold_runs_kernel(h1.data(), t1.data(), multi.data(), occidx.data(), n, occ.data(), slots.data(), n_slots - 1, 64 - lg); });
    // ---- against the oracle's index: every occupied khash bucket
    const uint32_t *kf; const uint64_t *kk, *kv, *kocc; uint32_t o_nocc = 0;
    const uint32_t nb = orc_index_arrays(oix, &kf, &kk, &kv, &kocc, &o_nocc);
    u64 o_keys = 0;
    for (uint32_t i = 0; i < nb; ++i) {
      if (((kf[i >> 4] >> ((i & 0xfU) << 1)) & 3) != 0) continue;
      ++o_keys;
      const u64 h = kk[i] >> 1;
      u64 s = (h * 0x9E3779B97F4A7C15ull) >> (64 - lg);
      bool found = false;
      for (;;) { if (slots[s].x == CMX_EMPTY_KEY) break; if ((slots[s].x >> 1) == h) { found = true; break; } s = (s + 1) & (n_slots - 1); }
      if (!found || slots[s].x != (u64)kk[i] || slots[s].y != (u64)kv[i]) { if (ok && bad < 6) printf("KEY it=%%d k=%%d w=%%d hash %%llx: found=%%d key %%llx/%%llx val %%llx/%%llx\n", it, k, w, (unsigned long long)h, found, found ? (unsigned long long)slots[s].x : 0ull, (unsigned long long)kk[i], found ? (unsigned long long)slots[s].y : 0ull, (unsigned long long)kv[i]); ok = false; }
    }
    if (o_keys != n_heads || o_nocc != n_occ) { printf("COUNTS it=%%d keys %%llu/%%llu occurrences %%u/%%u\n", it, (unsigned long long)n_heads, (unsigned long long)o_keys, n_occ, o_nocc); ok = false; }
    for (u32 i = 0; ok && i < n_occ; ++i) if (occ[i] != (u64)kocc[i]) { printf("OCC it=%%d entry %%u\n", it, i); ok = false; }
    // ---- and back up through the khash upload kernels (what cmx_upload_index does with the reference's own arrays)
    {
      unsigned long long c2 = 0;
      const u64 nfw = ((u64)nb + 15) / 16;
      emu_grid((int)((nfw + 255) / 256), 256, [&]() { khash_count_kernel(kf, nb, &c2); });
      std::vector<ulonglong2> s2((size_t)n_slots, ulonglong2{CMX_EMPTY_KEY, ~0ull});
      emu_grid_serial((int)(((u64)nb + 255) / 256), 256, [&]() { khash_insert_kernel(kf, (const u64 *)kk, (const u64 *)kv, 0, nb, s2.data(), n_slots - 1, 64 - lg); });
      if (c2 != o_keys) { printf("KHASH COUNT it=%%d %%llu/%%llu\n", it, c2, (unsigned long long)o_keys); ok = false; }
      // same key set and values as the table built on the device (slot order may differ: insertion order)
      u64 same = 0;
      for (u64 q = 0; q < n_slots; ++q) {
        if (s2[q].x == CMX_EMPTY_KEY) continue;
        u64 s = ((s2[q].x >> 1) * 0x9E3779B97F4A7C15ull) >> (64 - lg);
        while (slots[s].x != CMX_EMPTY_KEY && slots[s].x != s2[q].x) s = (s + 1) & (n_slots - 1);
        if (slots[s].x == s2[q].x && slots[s].y == s2[q].y) ++same;
      }
      if (same != o_keys) { printf("KHASH INSERT it=%%d same %%llu of %%llu\n", it, (unsigned long long)same, (unsigned long long)o_keys); ok = false; }
    }
    keys_total += (long)n_heads; occ_total += n_occ;
    if (!ok) ++bad;
    orc_index_free(oix); orc_reference_free(oref);
  }
  printf("references=%%ld keys=%%ld occurrences=%%ld bad=%%ld\n", cases, keys_total, occ_total, bad);
  return bad != 0;
}
'''


def test_index_build_kernels_equal_the_oracles_index(tmp_path):
    out = emu.run(tmp_path, ["device_common.cuh", "index_build.cuh"], MAIN % dict(orc_h=emu.ORACLE_H), timeout=1200)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["references"]) == 10 and int(f["keys"]) > 50000 and int(f["occurrences"]) > 5000, out.stdout
