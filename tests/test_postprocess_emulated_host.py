"""Record sort / duplicate removal / MAPQ filter / Tn5 of the CUDA path (chromap_b200/csrc/postprocess.cuh: key words, run
heads, survivor rule) and the kernels of the multi-GPU duplicate removal (exchange.cuh: tuple pack, key passes, heads, survivor
rule, gather; the range shuffle's key / sample / destination / bucket-bound kernels) and the BED text kernels run UNCHANGED on the host emulation
(tests/cta_emu.h) against the oracle's post-processing (`orc_postprocess`, `_bc`, `_pairs`, `_se`; mapping_processor.h:100-202,
mapping_writer.h:166-376, pinned to the reference binary by the golden BED / pairs files).  The library drives these kernels
with CUB's stable LSD radix passes (pp_device); here std::stable_sort plays CUB, in the same pass order."""
from tests import emu

MAIN = r'''
extern "C" {
#include "%(orc_h)s"
}
template <typename F> static void launch(size_t n, F body) { emu_grid_serial((int)((n + 255) / 256), 256, body); }   // (elementwise kernels: no barriers)
// CUB SortPairs(keys, idx): stable by key
static void stable_by_key(std::vector<u64> &keys, std::vector<u32> &idx) {
  std::vector<u32> ord(keys.size());
  std::iota(ord.begin(), ord.end(), 0u);
  std::stable_sort(ord.begin(), ord.end(), [&](u32 a, u32 b) { return keys[a] < keys[b]; });
  std::vector<u32> ni(idx.size());
  for (size_t i = 0; i < ord.size(); ++i) ni[i] = idx[ord[i]];
  idx.swap(ni);
}
static std::vector<PpRecord> random_records(std::mt19937 &g, size_t n, int kind) {
  std::vector<PpRecord> r(n);
  for (size_t i = 0; i < n; ++i) {
    PpRecord &x = r[i];
    x.w[0] = (u32)i * 7u + 3u;                                   // read_id (distinct)
    if (kind == PP_PAIRS) {
      x.w[1] = g() %% 3; x.w[2] = g() %% 3; x.w[3] = g() %% 600; x.w[4] = g() %% 600;
      x.w[5] = (g() & 1) | ((g() & 1) << 8) | ((u32)(g() %% 5 * 15) << 16) | ((g() & 1) << 24);
    } else {
      x.w[1] = g() %% 3; x.w[2] = 100 + g() %% 900;               // rid, start: many collisions
      x.w[3] = (100 + g() %% 4) | ((u32)(g() %% 5 * 15) << 16) | ((g() & 1) << 24);   // length | mapq | direction
      x.w[4] = (g() & 1) | (1u << 8) | ((40 + g() %% 20) << 16);   // unique | dups | positive length
      x.w[5] = 40 + g() %% 20;
    }
  }
  for (size_t i = 0; i + 1 < n; i += 9) { r[i + 1] = r[i]; r[i + 1].w[0] += 1; if (kind == PP_PAIRS) r[i + 1].w[5] ^= (u32)(g() %% 3) << 16; else r[i + 1].w[3] ^= (u32)(g() %% 3 * 16) << 16; }
  return r;
}
int main() {
  std::mt19937 g(97);
  long bad = 0, cases = 0, kept = 0;
  g_emu_leavable = true;
  // ---- postprocess.cuh against the oracle
  for (int kind : {PP_BED, PP_BED_BC, PP_PAIRS, PP_BED_SE})
    for (int low_mem = 0; low_mem < 2; ++low_mem) for (int dedup = 0; dedup < 2; ++dedup) for (int tn5 = 0; tn5 < 2; ++tn5) for (int q : {0, 30}) {
      if (kind == PP_PAIRS && (tn5 || (dedup && !low_mem))) continue;     // pairs: no Tn5; duplicate removal only with the low-memory rule (the library refuses the other)
      const size_t n = 3000;
      std::vector<PpRecord> recs = random_records(g, n, kind);
      std::vector<u64> bcs(n);
      for (auto &b : bcs) b = (g() %% 4) * 0x1234567ull;
      const bool bc = kind == PP_BED_BC;
      PpParams P{kind, low_mem, dedup, tn5, q, kind == PP_BED_SE};
      orc_params op; orc_default_params(&op);
      op.low_memory_mode = low_mem; op.remove_pcr_duplicates = dedup; op.tn5_shift = tn5; op.mapq_threshold = q; op.single_end = kind == PP_BED_SE;
      op.output_format = kind == PP_PAIRS ? 5 : 1;
      std::vector<PpRecord> want = recs;
      std::vector<u64> wbc = bcs;
      const long nw = kind == PP_PAIRS ? (long)orc_postprocess_pairs(&op, (orc_pairs_record *)want.data(), (long)n)
                      : bc ? (long)orc_postprocess_bc(&op, (orc_pe_record *)want.data(), (uint64_t *)wbc.data(), (long)n)
                      : kind == PP_BED_SE ? (long)orc_postprocess_se(&op, (orc_pe_record *)want.data(), (long)n) : (long)orc_postprocess(&op, (orc_pe_record *)want.data(), (long)n);
      // pp_device's sequence, std::stable_sort in CUB's place
      std::vector<PpRecord> a = recs, b2(n), res(n);
      std::vector<u64> bca = bcs, bcb(n), resbc(n), keys(n);
      std::vector<u32> idx(n);
      std::vector<u8> head(n), keep(n);
      if (!low_mem && tn5 && kind != PP_PAIRS) launch(n, [&]() { pp_tn5_kernel(kind, P.se, a.data(), n); });
      launch(n, [&]() { pp_iota_kernel(idx.data(), n); });
      for (int w = pp_n_words(kind) - 1; w >= 0; --w) {
        launch(n, [&]() { pp_key_kernel(kind, w, a.data(), bc ? bca.data() : nullptr, idx.data(), n, keys.data()); });
        stable_by_key(keys, idx);
      }
      launch(n, [&]() { pp_gather_kernel(a.data(), bc ? bca.data() : nullptr, idx.data(), n, b2.data(), bcb.data()); });
      launch(n, [&]() { pp_head_kernel(kind, P.se, dedup, b2.data(), bc ? bcb.data() : nullptr, n, head.data()); });
      launch(n, [&]() { pp_resolve_kernel(P, b2.data(), bc ? bcb.data() : nullptr, head.data(), n, res.data(), bc ? resbc.data() : nullptr, keep.data()); });
      std::vector<PpRecord> got; std::vector<u64> gbc;
      for (size_t i = 0; i < n; ++i) if (keep[i]) { got.push_back(res[i]); gbc.push_back(resbc[i]); }
      ++cases; kept += nw;
      bool ok = (long)got.size() == nw;
      for (long i = 0; ok && i < nw; ++i) ok = memcmp(&got[i], &want[i], sizeof(PpRecord)) == 0 && (!bc || gbc[i] == wbc[i]);
      if (!ok) { if (bad < 6) printf("POSTPROCESS kind=%%d low_mem=%%d dedup=%%d tn5=%%d q=%%d: %%zu / %%ld records\n", kind, low_mem, dedup, tn5, q, got.size(), nw); ++bad; }
    }
  // ---- exchange.cuh, all-gather form, two "ranks" gathered by hand: survivors of each rank == its share of the low-memory result
  for (int with_bc = 0; with_bc < 2; ++with_bc) for (int dedup = 0; dedup < 2; ++dedup) {
    const size_t n0 = 1700, n1 = 1300, n_pad = std::max(n0, n1), n_all = 2 * n_pad, n_total = n0 + n1;
    std::vector<PpRecord> all = random_records(g, n_total, PP_BED);
    std::vector<u64> bcs(n_total);
    for (auto &b : bcs) b = with_bc ? (g() %% 3) * 0x9999ull : 0ull;
    const int tw = with_bc ? 3 : 2, q = 30;
    orc_params op; orc_default_params(&op);
    op.low_memory_mode = 1; op.remove_pcr_duplicates = dedup; op.tn5_shift = 0; op.mapq_threshold = q;
    std::vector<PpRecord> want = all; std::vector<u64> wbc = bcs;
    const long nw = with_bc ? (long)orc_postprocess_bc(&op, (orc_pe_record *)want.data(), (uint64_t *)wbc.data(), (long)n_total) : (long)orc_postprocess(&op, (orc_pe_record *)want.data(), (long)n_total);
    std::vector<u64> tuples(n_all * tw);
    const PpRecord *rk[2] = {all.data(), all.data() + n0}; const u64 *bk[2] = {bcs.data(), bcs.data() + n0}; const size_t nk[2] = {n0, n1};
    for (int r = 0; r < 2; ++r) launch(n_pad, [&]() { ex_pack_kernel(rk[r], with_bc ? bk[r] : nullptr, nk[r], n_pad, with_bc, tuples.data() + (size_t)r * n_pad * tw); });
    std::vector<u32> idx(n_all); std::vector<u64> keys(n_all);
    launch(n_all, [&]() { pp_iota_kernel(idx.data(), n_all); });
    const int passes_bulk[2] = {4, 3}, passes_bc[4] = {0, 1, 2, 3};
    for (int qq = 0; qq < (with_bc ? 4 : 2); ++qq) {
      const int pass = with_bc ? passes_bc[qq] : passes_bulk[qq];
      launch(n_all, [&]() { ex_key_kernel(tuples.data(), tw, pass, idx.data(), n_all, keys.data()); });
      stable_by_key(keys, idx);
    }
    std::vector<u8> head(n_all);
    launch(n_total, [&]() { ex_head_kernel(tuples.data(), tw, dedup, idx.data(), n_total, head.data()); });
    std::vector<PpRecord> merged; std::vector<u64> mbc;
    std::vector<std::pair<u64, std::pair<PpRecord, u64>>> tagged;
    for (int r = 0; r < 2; ++r) {
      std::vector<u8> keep(n_all), dups(n_all); std::vector<u32> sel(n_all);
      launch(n_total, [&]() { ex_resolve_kernel(tuples.data(), tw, idx.data(), head.data(), n_total, n_pad, r, q, keep.data(), sel.data(), dups.data()); });
      std::vector<u32> selc; std::vector<u8> dupc;
      for (size_t i = 0; i < n_total; ++i) if (keep[i]) { selc.push_back(sel[i]); dupc.push_back(dups[i]); }
      std::vector<PpRecord> out(selc.size() + 1); std::vector<u64> obc(selc.size() + 1);
      const size_t ns = selc.size();
      if (ns) launch(ns, [&]() { ex_gather_kernel(rk[r], with_bc ? bk[r] : nullptr, selc.data(), dupc.data(), dedup, ns, out.data(), with_bc ? obc.data() : nullptr); });
      // survivors come out in the reference's order: merging the two ranks' lists by sorted position restores the whole
      size_t k = 0;
      for (size_t i = 0; i < n_total; ++i) if (keep[i]) { tagged.push_back({i, {out[k], with_bc ? obc[k] : 0ull}}); ++k; }
    }
    std::sort(tagged.begin(), tagged.end(), [](auto &x, auto &y) { return x.first < y.first; });
    ++cases; kept += nw;
    bool ok = (long)tagged.size() == nw;
    for (long i = 0; ok && i < nw; ++i) ok = memcmp(&tagged[i].second.first, &want[i], sizeof(PpRecord)) == 0 && (!with_bc || tagged[i].second.second == wbc[i]);
    if (!ok) { if (bad < 6) printf("EXCHANGE bc=%%d dedup=%%d: %%zu / %%ld survivors\n", with_bc, dedup, tagged.size(), nw); ++bad; }
  }
  // ---- the range shuffle's partition kernels
  for (int it = 0; it < 6; ++it) {
    const size_t n = it == 0 ? 0 : 500 + g() %% 9000;
    const int R = 2 + (int)(g() %% 7);
    std::vector<PpRecord> recs = random_records(g, n + 1, PP_BED);
    std::vector<u64> a(n + 1), samp(SH_SAMPLE), split((size_t)R);
    launch(n + 1, [&]() { sh_key_kernel(recs.data(), n, a.data()); });
    launch(SH_SAMPLE, [&]() { sh_sample_kernel(a.data(), n, samp.data()); });
    bool ok = true;
    const size_t take = std::min<size_t>(n, SH_SAMPLE);
    for (size_t i = 0; i < SH_SAMPLE; ++i) ok = ok && samp[i] == (i < take ? a[i * n / take] : EX_PAD);
    std::vector<u64> srt(samp.begin(), samp.begin() + take);
    std::sort(srt.begin(), srt.end());
    for (int j = 1; j < R; ++j) split[(size_t)j - 1] = take ? srt[take * (size_t)j / (size_t)R] : 0;
    std::vector<u32> dest(n + 1), sd;
    launch(n + 1, [&]() { sh_dest_kernel(a.data(), n, split.data(), R - 1, dest.data()); });
    for (size_t i = 0; i < n; ++i) { u32 d = 0; for (int j = 0; j < R - 1; ++j) d += split[(size_t)j] <= a[i]; ok = ok && dest[i] == d; }
    sd.assign(dest.begin(), dest.begin() + n);
    std::sort(sd.begin(), sd.end());
    std::vector<u64> off((size_t)R + 1);
    sd.push_back(0);
    emu_grid_serial(1, 64, [&]() { sh_bounds_kernel(sd.data(), n, R, off.data()); });
    for (int d = 0; d <= R; ++d) ok = ok && off[(size_t)d] == (u64)(std::lower_bound(sd.begin(), sd.begin() + n, (u32)d) - sd.begin());
    ++cases;
    if (!ok) { if (bad < 6) printf("SHUFFLE PARTITION it=%%d n=%%zu R=%%d\n", it, n, R); ++bad; }
  }
  // ---- BED text on the device (bed_len_kernel + exclusive scan + bed_write_kernel) against the oracle's writer
  {
    const char *names[3] = {"chr1", "chrUn_long_name_7", "c"};
    const std::string concat(300, 'A');
    const uint64_t offs[4] = {0, 100, 200, 300};
    orc_reference *oref = orc_reference_from_memory(3, concat.data(), offs, names);
    std::string cat; std::vector<u32> noff{0};
    for (const char *nm : names) { cat += nm; noff.push_back((u32)cat.size()); }
    for (int with_bc = 0; with_bc < 2; ++with_bc) {
      const size_t n = 4000;
      std::vector<PpRecord> recs = random_records(g, n, PP_BED);
      const u32 starts[6] = {0u, 9u, 10u, 99999u, 4294967295u, 1000000000u};
      for (auto &r : recs) { r.w[2] = starts[g() %% 6]; r.w[4] = (r.w[4] & 0xFFFF00FFu) | ((u32)(g() %% 4 == 0 ? 255 : 1 + g() %% 12) << 8); }
      std::vector<u64> bcs(n);
      for (auto &b : bcs) b = ((u64)g() << 16) ^ g();
      const int bc_len = with_bc ? 16 : 0;
      std::vector<u32> len(n + 1, 0);
      launch(n, [&]() { bed_len_kernel(recs.data(), n, noff.data(), bc_len, len.data()); });
      std::vector<u64> off(n + 1, 0);
      for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + len[i];
      std::string text((size_t)off[n], '?');
      launch(n, [&]() { bed_write_kernel(recs.data(), with_bc ? bcs.data() : nullptr, n, cat.data(), noff.data(), bc_len, off.data(), 0, &text[0]); });
      std::string want((size_t)off[n] + 4096, '!');
      const long nb = with_bc ? (long)orc_format_bed_bc(oref, (const orc_pe_record *)recs.data(), (const uint64_t *)bcs.data(), (long)n, 16, &want[0], (long)want.size())
                              : (long)orc_format_bed(oref, (const orc_pe_record *)recs.data(), (long)n, &want[0], (long)want.size());
      ++cases;
      if (nb != (long)off[n] || memcmp(want.data(), text.data(), (size_t)nb) != 0) { if (bad < 6) printf("BED TEXT bc=%%d: %%llu / %%ld bytes\n", with_bc, (unsigned long long)off[n], nb); ++bad; }
    }
    // pairs lines (pairs_len_kernel / pairs_write_kernel) against the oracle's writer, below its header
    {
      const size_t n = 3000;
      const u32 first_read_id = 77;
      std::vector<PpRecord> recs = random_records(g, n, PP_PAIRS);
      std::string rn; std::vector<u64> roff{0}; std::vector<std::string> rnv;
      for (size_t i = 0; i < n; ++i) { rnv.push_back("read" + std::to_string(i * 13 %% 977) + (i %% 5 ? "" : "/long_name_part")); rn += rnv.back(); roff.push_back(rn.size()); }
      std::vector<const char *> rnp; for (auto &x : rnv) rnp.push_back(x.c_str());
      for (size_t i = 0; i < n; ++i) { recs[i].w[0] = first_read_id + (u32)((i * 7) %% n); recs[i].w[3] = g() %% 3 ? g() %% 100000 : 4294967294u; recs[i].w[4] = g() %% 100000; }
      std::vector<u32> len(n + 1, 0);
      launch(n, [&]() { pairs_len_kernel(recs.data(), n, noff.data(), roff.data(), first_read_id, len.data()); });
      std::vector<u64> off(n + 1, 0);
      for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + len[i];
      std::string text((size_t)off[n], '?');
      launch(n, [&]() { pairs_write_kernel(recs.data(), n, cat.data(), noff.data(), rn.data(), roff.data(), first_read_id, off.data(), &text[0]); });
      std::string want((size_t)off[n] + 65536, '!');
      const long nb = (long)orc_format_pairs(oref, (const orc_pairs_record *)recs.data(), (long)n, rnp.data(), first_read_id, &want[0], (long)want.size());
      want.resize((size_t)std::max(0l, nb));
      size_t body = 0;
      while (body < want.size() && want[body] == '#') { body = want.find('\n', body); body = body == std::string::npos ? want.size() : body + 1; }
      ++cases;
      if (want.size() - body != text.size() || memcmp(want.data() + body, text.data(), text.size()) != 0) { if (bad < 6) printf("PAIRS TEXT: %%zu / %%zu bytes\n", text.size(), want.size() - body); ++bad; }
    }
    orc_reference_free(oref);
  }
  printf("cases=%%ld records_kept=%%ld bad=%%ld\n", cases, kept, bad);
  return bad != 0;
}
'''


def test_postprocess_and_exchange_kernels_equal_the_oracle(tmp_path):
    out = emu.run(tmp_path, ["device_common.cuh", "postprocess.cuh", "exchange.cuh"], MAIN % dict(orc_h=emu.ORACLE_H), timeout=1200)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["cases"]) > 50 and int(f["records_kept"]) > 50000, out.stdout
