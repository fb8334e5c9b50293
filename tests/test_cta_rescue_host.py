"""The mate-guided lookup (index.cc:351-489) in its two device formulations — `rescue_hits` (tier 0: one thread per pair, a
four-way lower bound + the arithmetic replay of the reference's probe path) and `cta_rescue` (overflow tiers: a warp per
minimizer, a lane per window, the chain through the windows as a prefix scan over 2-state transition functions) — run
UNCHANGED on the host (tests/cta_emu.h emulates the CTA) against the oracle's literal restatement of the reference's loop
(`orc_rescue_test`; the same code the oracle's mapper runs, pinned to the reference binary by tests/test_oracle_golden.py).
What the reference emits depends on where its binary search happens to stop, window after window; the inputs therefore put
windows before, inside, between and exactly on occurrence positions, merge neighbouring windows, and include both bail-outs."""
from tests import emu

MAIN = r'''
#include <cstdio>
#include <cstdlib>
#include <random>
extern "C" int orc_rescue_test(int k, int w, int max_seed_freq0, int min_num_seeds, int strand, u32 range, int n_mm, const u8 *kind, const u64 *val,
                               const u64 *mm_hit, const u64 *occ, const u64 *mate_pos, const u8 *mate_cnt, int n_mate, u32 *rep_len, u64 *hits, int cap,
                               int *nh);  // (u64 = unsigned long long here, uint64_t there: same size, C linkage)
int main() {
  std::mt19937 g(29);
  long bad = 0, cases = 0, total_hits = 0, bails = 0, on_boundary = 0;
  const int NTS[4] = {32, 128, 256, 512};
  for (int it = 0; it < 130; ++it) {
    const int nt = NTS[it %% 4];
    DevParams P{};
    P.k = 17; P.w = 7; P.e = 8; P.min_seeds = 2; P.f0 = (it %% 5 == 0) ? 40 : 500; P.f1 = 1000;
    // occurrence lists: sorted, distinct positions (one k-mer per reference position), random strands
    std::vector<u64> occ;
    struct L { u32 off, n; };
    std::vector<L> lists;
    const int n_lists = 1 + (int)(g() %% 6);
    for (int l = 0; l < n_lists; ++l) {
      const int n = 1 + (int)(g() %% (it %% 3 == 0 ? 3000 : 120));
      std::vector<u64> pos((size_t)n);
      for (auto &p : pos) p = ((u64)(g() %% 3) << 32) | (u64)(g() %% 200000);
      std::sort(pos.begin(), pos.end());
      pos.erase(std::unique(pos.begin(), pos.end()), pos.end());
      lists.push_back({(u32)occ.size(), (u32)pos.size()});
      for (u64 p : pos) occ.push_back((p << 1) | (g() & 1));
    }
    DevIndex ix{};
    ix.occ = occ.data(); ix.n_occ = (u32)occ.size(); ix.k = 17; ix.w = 7;
    // this read's probed minimizer records
    const int n_mm = 1 + (int)(g() %% 40);
    std::vector<u64> mmv((size_t)n_mm), mm_hit((size_t)n_mm);
    std::vector<u32> mmp((size_t)n_mm);
    std::vector<u8> kind((size_t)n_mm);
    u32 rp = 0;
    for (int i = 0; i < n_mm; ++i) {
      rp += 1 + g() %% 9;
      const u32 rs = g() & 1;
      kind[i] = (u8)(g() %% 3);
      if (kind[i] == 1) mmv[i] = (((u64)(g() %% 3) << 32 | (u64)(g() %% 200000)) << 1) | (g() & 1);
      else { const L &l = lists[g() %% lists.size()]; mmv[i] = ((u64)l.off << 32) | l.n; }
      mmp[i] = ((rp << 1) | rs) | ((u32)kind[i] << 30);
      mm_hit[i] = ((u64)rp << 1) | rs;
    }
    // the mate's candidates: near occurrence positions, some exactly range before one (window start ON an entry), clustered
    const u32 range = 50 + g() %% 4000;
    int n_mate = (int)(g() %% 60);
    if (it %% 17 == 0) n_mate = P.f0 + 1 + (int)(g() %% 10);   // index.cc:371-380 bail-out
    if (it %% 19 == 0) n_mate = 320;
    std::vector<u64> mate_pos((size_t)n_mate);
    std::vector<u8> mate_cnt((size_t)n_mate);
    for (int i = 0; i < n_mate; ++i) {
      const u64 o = occ[g() %% occ.size()] >> 1;
      const int mode = (int)(g() %% 4);
      u64 p = o;
      if (mode == 0) { p = o + range; ++on_boundary; }            // lo == an occurrence position
      else if (mode == 1) p = o + (g() %% (2 * range + 1));        // the entry somewhere inside
      else if (mode == 2) p = ((u64)(g() %% 3) << 32) | (u64)(g() %% 200000);
      else p = o > range + 1 ? o - range - 1 - g() %% 5 : o;     // the entry just past the window's end
      mate_pos[i] = p;
      mate_cnt[i] = (u8)(it %% 19 == 0 ? 3 : 1 + g() %% 4);
    }
    std::sort(mate_pos.begin(), mate_pos.end());
    for (int strand = 0; strand < 2; ++strand) {
      const int cap = 1 << 16;
      std::vector<u64> want((size_t)cap), got_t((size_t)cap), got_c((size_t)cap, ~0ull), sm(4096);
      u32 rl_w = 7, rl_t = 7, rl_c = 7;
      int nh_w = -1, nh_t = -1, nh_c = -1;
      const int r_w = orc_rescue_test(P.k, P.w, P.f0, P.min_seeds, strand, range, n_mm, kind.data(), mmv.data(), mm_hit.data(), occ.data(), mate_pos.data(),
                                      mate_cnt.data(), n_mate, &rl_w, want.data(), cap, &nh_w);
      const int r_t = rescue_hits(P, ix, strand, range, n_mm, mmv.data(), mmp.data(), 1, mate_pos.data(), mate_cnt.data(), n_mate, &rl_t, got_t.data(), cap, &nh_t);
      int r_c = 12345;
      RescueShared *R = new RescueShared;
      emu_launch(nt, [&]() {
        int nh = -1;
        const int r = cta_rescue(P, ix, strand, range, n_mm, mmv.data(), mmp.data(), mate_pos.data(), mate_cnt.data(), n_mate, &rl_c, got_c.data(), cap, sm.data(),
                                 (int)sm.size(), *R, &nh);
        if (threadIdx.x == 0) { r_c = r; nh_c = nh; }
      });
      delete R;
      ++cases;
      if (r_w < 0) ++bails;
      bool ok = r_w == r_t && r_w == r_c;
      if (ok && r_w >= 0 && n_mate > 0) {
        ok = nh_w == nh_t && nh_w == nh_c && rl_w == rl_t && rl_w == rl_c;
        for (int i = 0; ok && i < nh_w; ++i) ok = want[i] == got_t[i] && want[i] == got_c[i];
        total_hits += nh_w;
      }
      if (!ok) {
        if (bad < 6) printf("MISMATCH it=%%d nt=%%d strand=%%d n_mm=%%d n_mate=%%d range=%%u ret %%d/%%d/%%d hits %%d/%%d/%%d rep %%u/%%u/%%u\n", it, nt, strand, n_mm, n_mate, range,
                            r_w, r_t, r_c, nh_w, nh_t, nh_c, rl_w, rl_t, rl_c);
        ++bad;
      }
    }
  }
  printf("cases=%%ld hits=%%ld bails=%%ld boundary_windows=%%ld bad=%%ld\n", cases, total_hits, bails, on_boundary, bad);
  return bad != 0;
}
'''


def test_both_device_forms_of_the_mate_guided_lookup_equal_the_oracle(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN.replace("%%", "%"))
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-1500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["hits"]) > 5000 and int(f["bails"]) > 6 and int(f["boundary_windows"]) > 800, out.stdout
