"""Record emission of the CUDA path on the host emulation of a CTA (tests/cta_emu.h), kernels run UNCHANGED:
`pairing_kernel` -> `emit_kernel` (warp-phased: chosen best pairs, the Hamming shortcut of BandedTraceback by the whole warp,
the indel cases deferred to a list) + `emit_dp_kernel`, and `pairing_cta_kernel` -> `emit_cta_kernel` (best pairs counted per
share, located by prefix sums), with the MAPQ tables built by the library's own `mapq_tables_fill`, against the
oracle's post-verification stage (`orc_emit_test` = the tail of its mapper: mapping_generator.h:160-253, :486-1192,
mapping_generator.cc:110-143; pinned to the reference binary by tests/test_oracle_golden.py).  Draft mappings are real
alignments of mutated reads (substitutions, indels, soft-masked reference bases) at planted copies, so the spans, the alignment
lengths and with them every MAPQ branch (repetitive-seed scaling, second-best penalty, uint8 wrap, mate mixing, forced 0)
are exercised; -n 1 .. 3 with the reservoir selection computed by libstdc++ exactly as the reference does."""
from tests import emu

MAIN = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
struct orc_params { int error_threshold, min_num_seeds, max_seed_freq0, max_seed_freq1, max_num_best_mappings, max_insert_size, mapq_threshold, min_read_length,
                    drop_repetitive_reads, trim_adapters, remove_pcr_duplicates, tn5_shift, split_alignment, low_memory_mode, output_format, single_end; };
extern "C" void orc_default_params(orc_params *p);
extern "C" int orc_banded_align(int e, const char *pattern, const char *text, int read_len, int *end_pos);
extern "C" int orc_emit_test(const orc_params *p, const char *ref_seq, u32 ref_len, const char *read1, u32 L1, const char *read2, u32 L2, const int *n_map,
                             const u64 *pos, const short *err, const int *tally, const u32 *rep_len, int sup, u32 read_id, OutRecord *out, int cap);
static char comp(char c) { switch (c) { case 'A': case 'a': return 'T'; case 'C': case 'c': return 'G'; case 'G': case 'g': return 'C'; case 'T': case 't': return 'A'; default: return 'N'; } }
static std::string revc(const std::string &s) { std::string r(s.rbegin(), s.rend()); for (auto &c : r) c = comp(c); return r; }
int main() {
  std::mt19937 g(71);
  std::vector<double> il_(65536); std::vector<int> thr_(96);
  mapq_tables_fill(il_.data(), thr_.data());
  MapqTables T{il_.data(), thr_.data()};
  long bad = 0, n_pairs = 0, n_records = 0, n_deferred = 0, multi = 0, mapq_hist[4] = {0, 0, 0, 0};
  for (int it = 0; it < 220; ++it) {
    const int e = it %% 4 == 3 ? 4 : 8, mc = 256, mb = 1 + it %% 3;
    orc_params op; orc_default_params(&op);
    op.error_threshold = e; op.max_insert_size = 2000; op.max_num_best_mappings = mb;
    DevParams P{};
    P.e = e; P.max_insert = 2000; P.min_read_len = 30; P.drop_rep = 500000; P.max_best = mb; P.k = 17; P.w = 7; P.lanes = e < 8 ? 8 : 4;
    const u32 ref_len = 20000;
    std::string ref(ref_len, 'A');
    for (auto &c : ref) c = "ACGT"[g() %% 4];
    const int L[2] = {40 + (int)(g() %% 100), 40 + (int)(g() %% 100)};
    // a fragment, copied to n_copy loci (each copy with its own edits); mate 1 = its start, mate 2 = revcomp of its end
    const int frag = std::max(L[0], L[1]) + (int)(g() %% 300);
    std::string F((size_t)frag, 'A');
    for (auto &c : F) c = "ACGT"[g() %% 4];
    const int n_copy = it %% 5 == 0 ? 1 + (int)(g() %% 6) : 1;
    std::vector<u32> loci;
    for (int q = 0; q < n_copy; ++q) {
      const u32 at = 300 + (u32)(q * 2600) + g() %% 200;
      std::string c2 = F;
      if (q > 0) for (int x = 0; x < (int)(g() %% 3); ++x) c2[g() %% frag] = "ACGT"[g() %% 4];
      ref.replace(at, frag, c2);
      loci.push_back(at);
    }
    if (it %% 6 == 0) for (auto &c : ref) if (g() %% 4 == 0) c = (char)tolower(c);      // soft-masked bases: the Hamming shortcut compares raw chars
    std::string rd[2] = {F.substr(0, L[0]), revc(F.substr(frag - L[1], L[1]))};
    const bool flip = g() & 1;                                                         // half of the pairs map F2R1
    if (flip) { rd[0] = revc(F.substr(frag - L[0], L[0])); rd[1] = F.substr(0, L[1]); }
    for (int m = 0; m < 2; ++m) {
      const int n_edit = (int)(g() %% 4);
      for (int x = 0; x < n_edit; ++x) {
        const int k = (int)(g() %% 4), at = (int)(g() %% rd[m].size());
        if (k < 2) rd[m][at] = "ACGT"[g() %% 4];
        else if (k == 2) { rd[m].erase(at, 1); rd[m].push_back("ACGT"[g() %% 4]); }
        else { rd[m].insert(at, 1, "ACGT"[g() %% 4]); rd[m].pop_back(); }
      }
    }
    // draft mappings: the banded aligner at every locus, on the strand each mate lies on (what verification would have produced)
    int n_map[4] = {0, 0, 0, 0}, tal[8];
    std::vector<u64> pos; std::vector<short> err;
    bool any[2] = {false, false};
    for (int m = 0; m < 2; ++m) {
      Tally t{e + 1, e + 1, 0, 0};
      for (int st = 0; st < 2; ++st) {
        const bool on = (st == 0) == ((m == 0) != flip);       // mate 1 on + unless flipped; mate 2 the other strand
        if (!on) continue;
        const std::string text = st == 0 ? rd[m] : revc(rd[m]);
        for (u32 at : loci) {
          const u32 start = st == 0 ? (((m == 0) != flip) ? at : at) : 0;
          (void)start;
          // where the mate lies inside the fragment copy
          const u32 p0 = ((m == 0) != flip) ? at : at + (u32)(frag - L[m]);
          int endp = 0;
          const int er = orc_banded_align(e, ref.data() + p0 - e, text.data(), L[m], &endp);
          if (er > e) continue;
          pos.push_back((u64)(p0 - e + endp)); err.push_back((short)er);
          ++n_map[2 * m + st];
          tally(t, er);
          any[m] = true;
        }
      }
      tal[4 * m] = t.min_err; tal[4 * m + 1] = t.n_best; tal[4 * m + 2] = t.second_min_err; tal[4 * m + 3] = t.n_second_best;
    }
    pos.push_back(0); err.push_back(0);
    const u32 rep_len[2] = {it %% 3 == 0 ? (u32)(g() %% (L[0] + 30)) : 0u, it %% 7 == 0 ? (u32)(g() %% L[1]) : 0u};
    const int sup = it %% 9 == 0 ? 1 : 0;
    const u32 read_id = 1000 + it;
    OutRecord want[8];
    const int n_want = orc_emit_test(&op, ref.data(), ref_len, rd[0].data(), (u32)L[0], rd[1].data(), (u32)L[1], n_map, pos.data(), err.data(), tal, rep_len, sup, read_id, want, 8);
    // ---- device side: the same draft mappings in a scratch tier of one pair
    std::string refp = ref; refp.append(64, '\0');
    const u64 roff[1] = {0}; const u32 rlen[1] = {ref_len};
    DevRef R{(const u8 *)refp.data(), roff, rlen, 1};
    const u32 off1[2] = {0, (u32)L[0]}, off2[2] = {0, (u32)L[1]};
    DevBatch B{};
    B.seq1 = (const u8 *)rd[0].data(); B.off1 = off1; B.seq2 = (const u8 *)rd[1].data(); B.off2 = off2; B.n_pairs = 1; B.first_read_id = read_id;
    for (int form = 0; form < 2; ++form) {
      Scratch S{};
      S.caps = Caps{160, 64, 64, mc}; S.n_slots = 1;
      std::vector<ReadMeta> rmeta(2); std::vector<PairMeta> pmeta(1);
      std::vector<u64> map_pos((size_t)2 * 2 * mc); std::vector<short> map_err((size_t)2 * 2 * mc);
      S.rmeta = rmeta.data(); S.pmeta = pmeta.data(); S.map_pos = map_pos.data(); S.map_err = map_err.data();
      pmeta[0].sup = sup;
      size_t o = 0;
      for (int m = 0; m < 2; ++m) {
        rmeta[m].len = L[m]; rmeta[m].rep_len = rep_len[m];
        rmeta[m].min_err = tal[4 * m]; rmeta[m].n_best = tal[4 * m + 1]; rmeta[m].second_min_err = tal[4 * m + 2]; rmeta[m].n_second_best = tal[4 * m + 3];
        for (int st = 0; st < 2; ++st) {
          rmeta[m].n_map[st] = n_map[2 * m + st];
          for (int i = 0; i < n_map[2 * m + st]; ++i, ++o) { map_pos[((size_t)m * 2 + st) * mc + i] = pos[o]; map_err[((size_t)m * 2 + st) * mc + i] = err[o]; }
        }
      }
      int nbest = -1, out_n = -1;
      const int sm_cap = 1024;
      std::vector<u64> dyn((size_t)sm_cap + sm_cap / 4 + 8);
      g_dyn_smem = dyn.data();
      if (form == 0) emu_launch(32, [&]() { pairing_kernel(P, S, &nbest); });
      else emu_launch(128, [&]() { pairing_cta_kernel(P, S, &nbest, sm_cap); });
      // multi-mapper selection exactly as the reference draws it (a fresh generator here, as in orc_emit_test)
      std::vector<int> sel((size_t)mb);
      for (int j = 0; j < mb; ++j) sel[j] = j;
      if (nbest > mb) {
        std::mt19937 gen(11);
        for (int i = mb; i < nbest; ++i) { std::uniform_int_distribution<int> dist(0, i); const int j = dist(gen); if (j < mb) sel[j] = i; }
        std::sort(sel.begin(), sel.end());
      }
      OutRecord got[8];
      memset(got, 0, sizeof(got));
      Counters ctr{};
      if (form == 0) {
        std::vector<int4> dp_list(64);
        int dp_count = 0;
        emu_launch(32, [&]() { emit_kernel(P, R, B, T, S, sel.data(), got, &out_n, &ctr, dp_list.data(), &dp_count); });
        n_deferred += dp_count;
        if (dp_count) emu_launch(32, [&]() { emit_dp_kernel(P, R, B, T, S, got, dp_list.data(), &dp_count); });
      } else emu_launch(128, [&]() { emit_cta_kernel(P, R, B, T, S, sel.data(), got, &out_n, &ctr); });
      ++n_pairs;
      const bool none = !(any[0] && any[1]);
      bool ok = none ? (pmeta[0].status == ST_DROP && n_want == 0) : out_n == n_want;
      for (int i = 0; ok && !none && i < n_want; ++i) ok = memcmp(&got[i], &want[i], sizeof(OutRecord)) == 0;
      if (!none && form == 0) { n_records += n_want; if (nbest > mb) ++multi; for (int i = 0; i < n_want; ++i) ++mapq_hist[want[i].mapq == 0 ? 0 : want[i].mapq < 30 ? 1 : want[i].mapq < 60 ? 2 : 3]; }
      if (!ok) {
        if (bad < 6) {
          printf("EMIT it=%%d form=%%d e=%%d mb=%%d n %%d/%%d nbest=%%d", it, form, e, mb, out_n, n_want, nbest);
          if (n_want > 0) printf(" first: start %%u/%%u len %%u/%%u mapq %%u/%%u dir %%u/%%u uniq %%u/%%u pal %%u/%%u nal %%u/%%u", got[0].fragment_start, want[0].fragment_start, got[0].fragment_length,
                                 want[0].fragment_length, got[0].mapq, want[0].mapq, got[0].direction, want[0].direction, got[0].is_unique, want[0].is_unique,
                                 got[0].positive_alignment_length, want[0].positive_alignment_length, got[0].negative_alignment_length, want[0].negative_alignment_length);
          printf("\n");
        }
        ++bad;
      }
    }
  }
  printf("pairs=%%ld records=%%ld deferred_tracebacks=%%ld multi_best=%%ld mapq0=%%ld mapq_low=%%ld mapq_mid=%%ld mapq60=%%ld bad=%%ld\n", n_pairs, n_records, n_deferred, multi, mapq_hist[0],
         mapq_hist[1], mapq_hist[2], mapq_hist[3], bad);
  return bad != 0;
}
'''


def test_emit_kernels_equal_the_oracles_post_verification_stage(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN.replace("%%", "%"))
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["records"]) > 150 and int(f["deferred_tracebacks"]) > 20 and int(f["multi_best"]) > 3, out.stdout
