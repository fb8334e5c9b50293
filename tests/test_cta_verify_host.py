"""`verify_kernel` (tier 0: every pair; the reference's drivers replayed by one thread per read, fast path in a pass of its own) and
`verify_cta_kernel` (chromap_b200/csrc/cta_verify_pairing.cuh) — GenerateDraftMappings for one read by one CTA: fast path,
cooperative candidate sort, the lane-group / threshold rule of the reference's SIMD driver restated as "one threshold value T,
one stop index", accepted mappings written in list order by prefix sums, the error tally merged by reduction — run UNCHANGED
as kernels on the host emulation of a CTA (tests/cta_emu.h) against the oracle's `verify_read` (draft_mapping_generator.cc:9-357;
the code the oracle's mapper runs, pinned to the reference binary by tests/test_oracle_golden.py).  Inputs: planted repeat
copies with 0 .. e + 3 edits so that whole groups pass, whole groups fail and groups fail in part; candidates off both ends of
the reference; single-candidate reads for the fast path; block sizes 128 and 256 as the tiers launch them; e = 4 (8 lanes) and
e = 8 (4 lanes)."""
from tests import emu

MAIN = r'''
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
extern "C" void orc_verify_test(int e, const char *ref_seq, u32 ref_len, const char *read, u32 L, int n_mm, const int *n_cand, const u64 *cand_pos,
                                const u8 *cand_cnt, int cap, int *n_map, u64 *out_pos, short *out_err, int *stats);
static char comp(char c) { return c == 'A' ? 'T' : c == 'C' ? 'G' : c == 'G' ? 'C' : c == 'T' ? 'A' : 'N'; }
int main() {
  std::mt19937 g(53);
  long bad = 0, cases = 0, fast = 0, ruled = 0, mappings = 0;
  for (int it = 0; it < 150; ++it) {
    const int e = it %% 2 ? 8 : 4, nt = it %% 3 == 0 ? 256 : 128;
    const int L = 40 + (int)(g() %% 100);
    const u32 ref_len = 30000 + g() %% 20000;
    std::string ref(ref_len, 'A');
    for (auto &c : ref) c = "ACGT"[g() %% 4];
    std::string seg((size_t)L, 'A');
    for (auto &c : seg) c = "ACGT"[g() %% 4];
    // planted copies of the segment (forward or reverse-complemented), each with its own edits
    const int n_copy = it %% 13 == 0 ? 1 : 1 + (int)(g() %% 60);
    std::vector<u64> cpos[2];
    std::vector<u8> ccnt[2];
    const int n_mm = 3 + (int)(g() %% 12);
    for (int q = 0; q < n_copy; ++q) {
      const u32 at = 200 + (u32)(g() %% (ref_len - 400 - L));
      const int strand = (int)(g() & 1);
      std::string s2 = seg;
      if (strand) { std::string r(s2.rbegin(), s2.rend()); for (auto &c : r) c = comp(c); s2 = r; }
      const int n_edit = (int)(g() %% (e + 4));
      for (int x = 0; x < n_edit; ++x) s2[g() %% L] = "ACGT"[g() %% 4];
      if (g() %% 5 == 0) s2.erase(g() %% L, 1), s2.push_back("ACGT"[g() %% 4]);     // an indel
      ref.replace(at, L, s2);
      cpos[strand].push_back(strand == 0 ? (u64)at : (u64)at + L - 1);
      ccnt[strand].push_back((u8)(1 + g() %% n_mm));
    }
    for (int q = 0; q < (int)(g() %% 8) && n_copy > 1; ++q) {      // random loci and loci off the ends of the reference
      const int strand = (int)(g() & 1);
      const int m = (int)(g() %% 4);
      const u64 p = m == 0 ? g() %% (u32)e : m == 1 ? ref_len - 1 - g() %% (L + e) : 100 + g() %% (ref_len - 200);
      cpos[strand].push_back(p); ccnt[strand].push_back((u8)(1 + g() %% n_mm));
    }
    if (n_copy == 1) { for (int s = 0; s < 2; ++s) for (auto &c : ccnt[s]) c = (u8)(it %% 26 == 0 ? n_mm : (g() %% 2 ? n_mm : 1)); }
    for (int s = 0; s < 2; ++s) {   // distinct positions per strand (candidates of one read are)
      std::vector<std::pair<u64, u8>> v;
      for (size_t i = 0; i < cpos[s].size(); ++i) v.push_back({cpos[s][i], ccnt[s][i]});
      std::sort(v.begin(), v.end());
      v.erase(std::unique(v.begin(), v.end(), [](const std::pair<u64, u8> &a, const std::pair<u64, u8> &b) { return a.first == b.first; }), v.end());
      cpos[s].clear(); ccnt[s].clear();
      for (auto &x : v) { cpos[s].push_back(x.first); ccnt[s].push_back(x.second); }
    }
    std::string read = seg;
    for (int x = 0; x < (int)(g() %% 3); ++x) read[g() %% L] = "ACGT"[g() %% 4];
    // ---- oracle
    const int cap = 1024;
    const int nc[2] = {(int)cpos[0].size(), (int)cpos[1].size()};
    std::vector<u64> flat_p; std::vector<u8> flat_c;
    for (int s = 0; s < 2; ++s) { flat_p.insert(flat_p.end(), cpos[s].begin(), cpos[s].end()); flat_c.insert(flat_c.end(), ccnt[s].begin(), ccnt[s].end()); }
    flat_p.push_back(0); flat_c.push_back(0);
    int w_n[2] = {0, 0}, w_st[4];
    std::vector<u64> w_pos((size_t)2 * cap);
    std::vector<short> w_err((size_t)2 * cap);
    orc_verify_test(e, ref.data(), ref_len, read.data(), (u32)L, n_mm, nc, flat_p.data(), flat_c.data(), cap, w_n, w_pos.data(), w_err.data(), w_st);
    // ---- the kernel on one read slot
    DevParams P{};
    P.e = e; P.lanes = e < 8 ? 8 : 4; P.k = 17; P.w = 7; P.se = 0;
    std::string refp = ref; refp.append(64, '\0');
    const u64 roff[1] = {0}; const u32 rlen[1] = {ref_len};
    DevRef R{(const u8 *)refp.data(), roff, rlen, 1};
    const u32 off1[2] = {0, (u32)L};
    DevBatch B{};
    B.seq1 = (const u8 *)read.data(); B.off1 = off1; B.seq2 = (const u8 *)read.data(); B.off2 = off1; B.n_pairs = 1;
    Scratch S{};
    S.caps = Caps{160, 1024, 1024, cap}; S.n_slots = 1;
    std::vector<ReadMeta> rmeta(2); std::vector<PairMeta> pmeta(1);
    std::vector<u64> cand_pos((size_t)2 * 3 * 2 * 1024), map_pos((size_t)2 * 2 * cap);
    std::vector<u8> cand_cnt((size_t)2 * 3 * 2 * 1024);
    std::vector<short> map_err((size_t)2 * 2 * cap);
    std::vector<int> map_split((size_t)2 * 2 * cap);
    S.rmeta = rmeta.data(); S.pmeta = pmeta.data(); S.cand_pos = cand_pos.data(); S.cand_cnt = cand_cnt.data(); S.map_pos = map_pos.data();
    S.map_err = map_err.data(); S.map_split = map_split.data();
    rmeta[0].len = L; rmeta[0].n_mm = n_mm; rmeta[0].n_cand[0] = nc[0]; rmeta[0].n_cand[1] = nc[1];
    for (int s = 0; s < 2; ++s) for (int i = 0; i < nc[s]; ++i) { cand_pos[(size_t)s * 1024 + i] = cpos[s][i]; cand_cnt[(size_t)s * 1024 + i] = ccnt[s][i]; }
    for (int form = 0; form < 2; ++form) {   // 0: verify_kernel (tier 0: fast-path pass, then the listed reads one thread each); 1: verify_cta_kernel
      std::vector<ReadMeta> rm2 = rmeta; std::vector<PairMeta> pm2 = pmeta;
      std::vector<u64> cp2 = cand_pos, mp2((size_t)2 * 2 * cap);
      std::vector<u8> cc2 = cand_cnt;
      std::vector<short> me2((size_t)2 * 2 * cap);
      Scratch S2 = S;
      S2.rmeta = rm2.data(); S2.pmeta = pm2.data(); S2.cand_pos = cp2.data(); S2.cand_cnt = cc2.data(); S2.map_pos = mp2.data(); S2.map_err = me2.data();
      Counters ctr{};
      const int sm_cap = 1024;
      std::vector<u64> dyn((size_t)sm_cap + sm_cap / 8 + 2 * 160 * 64 / 8 + 8);
      g_dyn_smem = dyn.data();
      if (form == 0) {
        int list[4] = {0, 0, 0, 0}, list_count = 0;
        emu_launch(32, [&]() { verify_kernel(P, R, B, S2, &ctr, 0, list, &list_count); });
        if (list_count) emu_launch(64, [&]() { verify_kernel(P, R, B, S2, &ctr, 1, list, &list_count); });
      } else emu_launch(nt, [&]() { verify_cta_kernel(P, R, B, S2, &ctr, sm_cap); });
      ++cases;
      bool ok = pm2[0].status == ST_OK && rm2[0].n_map[0] == w_n[0] && rm2[0].n_map[1] == w_n[1] && rm2[0].min_err == w_st[0] && rm2[0].n_best == w_st[1] &&
                rm2[0].second_min_err == w_st[2] && rm2[0].n_second_best == w_st[3];
      for (int s = 0; ok && s < 2; ++s)
        for (int i = 0; ok && i < w_n[s]; ++i) ok = mp2[(size_t)s * cap + i] == w_pos[(size_t)s * cap + i] && me2[(size_t)s * cap + i] == w_err[(size_t)s * cap + i];
      if (!ok) {
        if (bad < 6) printf("MISMATCH it=%%d form=%%d e=%%d nt=%%d L=%%d cands %%d+%%d maps %%d/%%d %%d/%%d tally %%d,%%d,%%d,%%d / %%d,%%d,%%d,%%d\n", it, form, e, nt, L, nc[0], nc[1], rm2[0].n_map[0],
                            w_n[0], rm2[0].n_map[1], w_n[1], rm2[0].min_err, rm2[0].n_best, rm2[0].second_min_err, rm2[0].n_second_best, w_st[0], w_st[1], w_st[2], w_st[3]);
        ++bad;
      }
    }
    if (nc[0] + nc[1] == 1) ++fast;
    if (nc[0] >= P.lanes || nc[1] >= P.lanes) ++ruled;
    mappings += w_n[0] + w_n[1];
  }
  printf("reads=%%ld single_candidate=%%ld group_rule=%%ld mappings=%%ld bad=%%ld\n", cases, fast, ruled, mappings, bad);
  return bad != 0;
}
'''


def test_verify_cta_kernel_equals_the_oracles_draft_mapping_generation(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN.replace("%%", "%"))
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2000:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["single_candidate"]) >= 6 and int(f["group_rule"]) > 60 and int(f["mappings"]) > 600, out.stdout
