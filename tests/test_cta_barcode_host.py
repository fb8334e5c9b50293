"""scATAC cell-barcode correction of the CUDA path (`wl_insert_kernel` + `barcode_kernel`, chromap_b200/csrc/pipeline_kernels.cuh:
CorrectBarcodeAt, chromap.cc:572-799, for --bc-error-threshold 0 and 1) run UNCHANGED on the host emulation (tests/cta_emu.h)
against the oracle's `correct_barcode` (pinned to the reference binary by the scATAC golden files): whitelist membership, one
substitution, one N, ties broken by (score, index, base), the posterior threshold, qualities clamped to [3, 40], abundances from
a sampled count table; keys and accept flags of every barcode and both counters."""
from tests import emu

MAIN = r'''
extern "C" {
#include "%(orc_h)s"
int orc_correct_barcode_test(const orc_whitelist *wl, int err_threshold, double prob_threshold, const char *bc, const char *qual, uint32_t len, uint64_t *out_key,
                             uint64_t *n_in_whitelist, uint64_t *n_corrected);
}
int main(int argc, char **argv) {
  std::mt19937 g(83);
  long bad = 0, n_bc = 0, n_in = 0, n_cor = 0, n_rej = 0;
  for (int round = 0; round < 4; ++round) {
    const u32 bc_len = round == 3 ? 12 : 16;
    const int err_threshold = round == 2 ? 0 : 1;
    const double prob_threshold = round == 1 ? 0.6 : 0.9;
    // whitelist: random barcodes plus families of near neighbours (one substitution apart: competing corrections)
    std::vector<std::string> wl_seq;
    for (int i = 0; i < 1500; ++i) { std::string b(bc_len, 'A'); for (auto &c : b) c = "ACGT"[g() %% 4]; wl_seq.push_back(b); }
    for (int i = 0; i < 300; ++i) { std::string b = wl_seq[g() %% 1500]; b[g() %% bc_len] = "ACGT"[g() %% 4]; wl_seq.push_back(b); }
    const std::string path = std::string(argc > 1 ? argv[1] : "/tmp") + "/wl" + std::to_string(round) + ".txt";
    FILE *f = fopen(path.c_str(), "w");
    for (auto &b : wl_seq) fprintf(f, "%%s\n", b.c_str());
    fclose(f);
    orc_whitelist *wl = orc_whitelist_load(path.c_str(), bc_len);
    // observed barcodes: whitelist entries (uneven abundances), with substitutions / N's / junk
    const int n = 6000;
    std::string bcs, quals;
    for (int i = 0; i < n; ++i) {
      std::string b = wl_seq[(g() %% 7 == 0) ? g() %% wl_seq.size() : g() %% 120];
      const int m = (int)(g() %% 10);
      if (m == 0) b[g() %% bc_len] = "ACGT"[g() %% 4];
      else if (m == 1) b[g() %% bc_len] = 'N';
      else if (m == 2) { b[g() %% bc_len] = 'N'; b[g() %% bc_len] = 'N'; }
      else if (m == 3) for (auto &c : b) c = "ACGT"[g() %% 4];
      else if (m == 4) { b[g() %% bc_len] = "ACGT"[g() %% 4]; b[g() %% bc_len] = "ACGT"[g() %% 4]; }
      std::string q(bc_len, 'I');
      for (auto &c : q) c = (char)(33 + g() %% 45);       // Phred 0 .. 44: both clamps
      bcs += b; quals += q;
    }
    orc_whitelist_sample(wl, bcs.data(), (uint64_t)n, bc_len, 20000000, 500000);
    const uint64_t *keys; const uint32_t *counts; uint64_t num_sample = 0;
    const uint64_t nk = orc_whitelist_arrays(wl, &keys, &counts, &num_sample);
    // ---- device whitelist as cmx_upload_barcode_whitelist builds it
    u64 ns = 64; while (ns < 2 * nk) ns <<= 1;
    int lg = 0; while ((1ull << lg) < ns) ++lg;
    std::vector<ulonglong2> slots((size_t)ns, ulonglong2{~0ull, ~0ull});
    g_emu_leavable = true;
    emu_grid((int)((nk + 255) / 256), 256, [&]() { wl_insert_kernel((const u64 *)keys, counts, nk, slots.data(), ns - 1, 64 - lg); });
    std::vector<double> pw(41);
    for (int q = 0; q <= 40; ++q) pw[q] = pow(10.0, ((-q) / 10.0));
    DevWhitelist W{};
    W.slots = slots.data(); W.mask = ns - 1; W.shift = 64 - lg; W.num_sample = (double)num_sample; W.pow_tab = pw.data(); W.err_threshold = err_threshold;
    W.prob_threshold = prob_threshold; W.output_not_in_whitelist = 0; W.active = 1;
    std::vector<u64> bc_key((size_t)n);
    std::vector<u8> bc_ok((size_t)n);
    Counters ctr{};
    emu_grid((n + 127) / 128, 128, [&]() { barcode_kernel(W, (const u8 *)bcs.data(), (const u8 *)quals.data(), (int)bc_len, n, bc_key.data(), bc_ok.data(), &ctr); });
    g_emu_leavable = false;
    uint64_t w_in = 0, w_cor = 0;
    for (int i = 0; i < n; ++i) {
      uint64_t wk = 0;
      const int ok = orc_correct_barcode_test(wl, err_threshold, prob_threshold, bcs.data() + (size_t)i * bc_len, quals.data() + (size_t)i * bc_len, bc_len, &wk, &w_in, &w_cor);
      ++n_bc;
      if (!ok) ++n_rej;
      if ((int)bc_ok[i] != ok || (u64)wk != bc_key[i]) { if (bad < 6) printf("BARCODE round=%%d i=%%d ok %%d/%%d key %%llx/%%llx  %%.*s\n", round, i, bc_ok[i], ok, (unsigned long long)bc_key[i], (unsigned long long)wk, (int)bc_len, bcs.data() + (size_t)i * bc_len); ++bad; }
    }
    if (ctr.n_bc_in_whitelist != w_in || ctr.n_bc_corrected != w_cor) { printf("COUNTERS round=%%d in %%llu/%%llu corrected %%llu/%%llu\n", round, (unsigned long long)ctr.n_bc_in_whitelist, (unsigned long long)w_in, (unsigned long long)ctr.n_bc_corrected, (unsigned long long)w_cor); ++bad; }
    n_in += (long)w_in; n_cor += (long)w_cor;
    orc_whitelist_free(wl);
  }
  printf("barcodes=%%ld in_whitelist=%%ld corrected=%%ld rejected=%%ld bad=%%ld\n", n_bc, n_in, n_cor, n_rej, bad);
  return bad != 0;
}
'''


def test_barcode_correction_kernel_equals_the_oracle(tmp_path):
    out = emu.run(tmp_path, emu.PIPELINE, MAIN % dict(orc_h=emu.ORACLE_H), args=[str(tmp_path)], timeout=1200)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-2500:] + out.stderr[-800:]
    f = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(f["in_whitelist"]) > 5000 and int(f["corrected"]) > 1000 and int(f["rejected"]) > 2000, out.stdout
