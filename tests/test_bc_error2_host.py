"""--bc-error-threshold 2 without a GPU.

- The kernels of the barcode gate (`barcode_kernel` + `barcode_correct2_kernel`, chromap_b200/csrc/pipeline_kernels.cuh) run
  UNCHANGED on the host emulation of a CTA (tests/cta_emu.h), in the order `lane_barcodes` (lane_pipeline.cuh) gives run_lane,
  against the oracle's `correct_barcode` (CorrectBarcodeAt, chromap.cc:572-799): keys, accept flags and both counters, over
  barcode lengths 4 to 32, 0 to 3 Ns, whitelists with neighbours at distance 1 and 2, tied abundances, qualities outside
  [3, 40], probability thresholds 0 to 0.99, and barcodes whose every neighbour is in the whitelist (the hit bound, which the
  slab pass takes).  One small run is built with AddressSanitizer, which checks the shared and global hit lists' bounds.
- The oracle reproduces the synth_bc_error2 goldens written by the reference binary, counters included.
- The CLI refuses thresholds the GPU path does not take before it looks for a device."""
import gzip
import os
import subprocess

import numpy as np
import pytest

from tests import emu
from tests.bc_error2_oracle import GOLDEN, RUNS, run_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")

MAIN = r'''
extern "C" {
#include "%(orc_h)s"
int orc_correct_barcode_test(const orc_whitelist *wl, int err_threshold, double prob_threshold, const char *bc, const char *qual, uint32_t len, uint64_t *out_key,
                             uint64_t *n_in_whitelist, uint64_t *n_corrected);
}
struct EmuLaunch {  // lane_barcodes' launches on emulated CTAs
  template <typename... KA, typename... A>
  void operator()(void (*kernel)(KA...), int grid, int block, size_t, A... a) { emu_grid(grid, block, [&]() { kernel(a...); }); }
};
static void mutate(std::string &b, std::mt19937 &g, int subs, int ns) {  // subs substitutions (to another base), ns Ns, at distinct places
  std::vector<int> pos(b.size());
  std::iota(pos.begin(), pos.end(), 0);
  std::shuffle(pos.begin(), pos.end(), g);
  for (int k = 0; k < subs + ns && k < (int)b.size(); ++k) {
    char &c = b[pos[k]];
    if (k < subs) { const char o = c; while (c == o) c = "ACGT"[g() %% 4]; }
    else c = 'N';
  }
}
// every key at Hamming distance 1 or 2 from b
static void neighbours(const std::string &b, std::vector<std::string> &out) {
  for (size_t i = 0; i < b.size(); ++i)
    for (char x : std::string("ACGT")) {
      if (x == b[i]) continue;
      std::string c = b; c[i] = x; out.push_back(c);
      for (size_t j = i + 1; j < b.size(); ++j)
        for (char y : std::string("ACGT")) { if (y == b[j]) continue; std::string d = c; d[j] = y; out.push_back(d); }
    }
}
int main(int argc, char **argv) {
  const std::string dir = argv[1];
  const bool small = argc > 2 && std::string(argv[2]) == "small";
  std::mt19937 g(2027);
  const int lens[] = {4, 8, 12, 16, 24, 32, 16, 32};
  const double probs[] = {0.9, 0.4, 0.5, 0.99, 0.0, 0.9, 0.5, 0.4};
  long bad = 0, n_bc = 0, n_in = 0, n_cor = 0, n_rej = 0, n_listed = 0, n_ovf = 0;
  const int rounds = small ? 2 : 9;
  for (int round = 0; round < rounds; ++round) {
    const u32 L = small ? (round ? 8u : 32u) : round == 8 ? 16u : (u32)lens[round];
    const int err_threshold = round == 8 ? 1 : 2;  // round 8: threshold 1 through the same launch sequence
    const double prob = small ? 0.5 : probs[round %% 8];
    const int n = small ? 300 : 1500;
    // whitelist: random barcodes, neighbours two and one substitutions away from some, and a few barcodes (not listed
    // themselves) with every neighbour listed
    std::vector<std::string> wl, full;
    const int nw = L <= 4 ? 40 : L <= 8 ? 400 : 1200;
    for (int i = 0; i < nw; ++i) { std::string b(L, 'A'); for (auto &c : b) c = "ACGT"[g() %% 4]; wl.push_back(b); }
    for (int i = 0; i < nw / 3; ++i) { std::string b = wl[g() %% nw]; mutate(b, g, 2, 0); wl.push_back(b); }
    for (int i = 0; i < nw / 6; ++i) { std::string b = wl[g() %% nw]; mutate(b, g, 1, 0); wl.push_back(b); }
    if (L >= 8)
      for (int f = 0; f < 2; ++f) { std::string b(L, 'A'); for (auto &c : b) c = "ACGT"[g() %% 4]; full.push_back(b); neighbours(b, wl); }
    std::vector<std::string> in_wl(wl);
    std::set<std::string> fullset(full.begin(), full.end());
    const std::string path = dir + "/wl" + std::to_string(round) + ".txt";
    FILE *fw = fopen(path.c_str(), "w");
    for (auto &b : wl) if (!fullset.count(b)) fprintf(fw, "%%s\n", b.c_str());
    fclose(fw);
    orc_whitelist *W0 = orc_whitelist_load(path.c_str(), L);
    // abundances: a skewed sample of whitelist entries (many small equal counts: ties)
    std::string samp;
    for (int i = 0; i < 4 * nw; ++i) samp += wl[(g() %% 3 == 0) ? g() %% wl.size() : g() %% (wl.size() / 8 + 1)];
    // observed barcodes: whitelist entries with 0 to 2 substitutions and 0 to 3 Ns, the full-neighbourhood barcodes, junk
    std::string bcs, quals;
    for (int i = 0; i < n; ++i) {
      std::string b = wl[g() %% wl.size()];
      const int m = (int)(g() %% 16);
      if (m < 3) mutate(b, g, 2, 0);
      else if (m < 5) mutate(b, g, 1, 0);
      else if (m == 5) mutate(b, g, 1, 1);
      else if (m == 6) mutate(b, g, 0, 1);
      else if (m == 7) mutate(b, g, 0, 2);
      else if (m == 8) mutate(b, g, 1, 2);
      else if (m == 9) mutate(b, g, 0, 3);
      else if (m == 10) for (auto &c : b) c = "ACGT"[g() %% 4];
      else if (m == 11 && !full.empty()) { b = full[g() %% full.size()]; if (g() %% 3 == 0) mutate(b, g, 0, 1 + (int)(g() %% 2)); }
      std::string q(L, 'I');
      for (auto &c : q) c = (char)(33 + g() %% 45);  // Phred 0 .. 44: both clamps
      bcs += b; quals += q;
    }
    orc_whitelist_sample(W0, samp.data(), samp.size() / L, L, 20000000, 500000);
    const uint64_t *keys; const uint32_t *counts; uint64_t num_sample = 0;
    const uint64_t nk = orc_whitelist_arrays(W0, &keys, &counts, &num_sample);
    // ---- device whitelist as cmx_upload_barcode_whitelist builds it
    u64 ns = 64; while (ns < 2 * nk) ns <<= 1;
    int lg = 0; while ((1ull << lg) < ns) ++lg;
    std::vector<ulonglong2> slots((size_t)ns, ulonglong2{~0ull, ~0ull});
    g_emu_leavable = true;
    emu_grid((int)((nk + 255) / 256), 256, [&]() { wl_insert_kernel((const u64 *)keys, counts, nk, slots.data(), ns - 1, 64 - lg); });
    std::vector<double> pw(81);
    for (int q = 0; q <= 80; ++q) pw[q] = pow(10.0, ((-q) / 10.0));
    std::vector<u32> list((size_t)n), over((size_t)n);
    std::vector<Bc2Slab> slab(BC2_SLAB_WARPS);
    DevWhitelist W{};
    W.slots = slots.data(); W.mask = ns - 1; W.shift = 64 - lg; W.num_sample = (double)num_sample; W.pow_tab = pw.data(); W.err_threshold = err_threshold;
    W.prob_threshold = prob; W.output_not_in_whitelist = 0; W.active = 1;
    W.c2_list = list.data(); W.c2_over = over.data(); W.c2_slab = slab.data();
    std::vector<u64> bc_key((size_t)n);
    std::vector<u8> bc_ok((size_t)n);
    Counters ctr{};
    EmuLaunch x;
    lane_barcodes(x, W, (const u8 *)bcs.data(), (const u8 *)quals.data(), (int)L, n, bc_key.data(), bc_ok.data(), &ctr);
    g_emu_leavable = false;
    uint64_t w_in = 0, w_cor = 0;
    for (int i = 0; i < n; ++i) {
      uint64_t wk = 0;
      const int ok = orc_correct_barcode_test(W0, err_threshold, prob, bcs.data() + (size_t)i * L, quals.data() + (size_t)i * L, L, &wk, &w_in, &w_cor);
      ++n_bc;
      if (!ok) ++n_rej;
      if ((int)bc_ok[i] != ok || (u64)wk != bc_key[i]) { if (bad < 6) printf("BARCODE round=%%d i=%%d ok %%d/%%d key %%llx/%%llx  %%.*s\n", round, i, bc_ok[i], ok, (unsigned long long)bc_key[i], (unsigned long long)wk, (int)L, bcs.data() + (size_t)i * L); ++bad; }
    }
    if (ctr.n_bc_in_whitelist != w_in || ctr.n_bc_corrected != w_cor) { printf("COUNTERS round=%%d in %%llu/%%llu corrected %%llu/%%llu\n", round, (unsigned long long)ctr.n_bc_in_whitelist, (unsigned long long)w_in, (unsigned long long)ctr.n_bc_corrected, (unsigned long long)w_cor); ++bad; }
    printf("round=%%d L=%%u threshold=%%d prob=%%g whitelist=%%llu in=%%llu corrected=%%llu listed=%%llu slab=%%llu\n", round, L, err_threshold, prob, (unsigned long long)nk, (unsigned long long)w_in, (unsigned long long)w_cor, ctr.n_bc2_listed, ctr.n_bc2_overflow);
    n_in += (long)w_in; n_cor += (long)w_cor; n_listed += (long)ctr.n_bc2_listed; n_ovf += (long)ctr.n_bc2_overflow;
    orc_whitelist_free(W0);
  }
  printf("barcodes=%%ld in_whitelist=%%ld corrected=%%ld rejected=%%ld listed=%%ld slab=%%ld bad=%%ld\n", n_bc, n_in, n_cor, n_rej, n_listed, n_ovf, bad);
  return bad != 0;
}
'''


def _run(tmp_path, *args, flags=()):
    src = '#include <set>\n' + MAIN % dict(orc_h=emu.ORACLE_H)
    out = emu.run(tmp_path, emu.PIPELINE, src, args=[str(tmp_path)] + list(args), timeout=3000, flags=flags)
    assert out.returncode == 0 and "bad=0" in out.stdout, out.stdout[-3000:] + out.stderr[-1500:]
    return dict(kv.split("=") for kv in out.stdout.strip().splitlines()[-1].split() if "=" in kv)


def test_distance2_kernels_equal_the_oracle(tmp_path):
    f = _run(tmp_path)
    # every path taken: exact hits, corrections, refusals, the shared-memory lists and the slab pass
    assert int(f["in_whitelist"]) > 2000 and int(f["corrected"]) > 2000 and int(f["rejected"]) > 1000, f
    assert int(f["listed"]) > 4000 and int(f["slab"]) >= 20, f


def test_distance2_kernels_under_address_sanitizer(tmp_path):
    f = _run(tmp_path, "small", flags=("-fsanitize=address", "-fno-omit-frame-pointer"))
    assert int(f["slab"]) > 0 and int(f["corrected"]) > 0, f


@pytest.mark.parametrize("name", sorted(RUNS))
def test_oracle_reproduces_golden(tmp_path, name):
    text, stats = run_oracle(name)
    with gzip.open(os.path.join(GOLDEN, name + ".bed.gz"), "rb") as f:
        want = f.read()
    assert text == want, name
    with open(os.path.join(GOLDEN, "stats.txt")) as f:
        st = dict(l.split(None, 1) for l in f.read().splitlines())
    assert st[name].split() == [str(int(stats[0])), str(int(stats[1]))], (name, st[name], stats)


@pytest.mark.parametrize("thr", ["3", "-1", "7"])
def test_cli_refuses_threshold_without_a_device(tmp_path, thr):
    d = os.path.join(ROOT, "tests", "golden", "synth_sc")
    r = subprocess.run([CLI, "--preset", "atac", "-x", str(tmp_path / "none.index"), "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, "r1.fq.gz"),
                        "-2", os.path.join(d, "r2.fq.gz"), "-b", os.path.join(d, "bc.fq.gz"), "--barcode-whitelist", os.path.join(d, "whitelist.txt"),
                        "--bc-error-threshold", thr, "-o", str(tmp_path / "o.bed")], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "--bc-error-threshold " + thr in r.stderr and "0, 1 or 2" in r.stderr, r.stderr
    assert "Cannot load index" not in r.stderr and not (tmp_path / "o.bed").exists()


def test_cli_help_lists_the_threshold():
    h = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert h.returncode == 0 and "--bc-error-threshold" in h.stdout and "0, 1 or 2" in h.stdout
