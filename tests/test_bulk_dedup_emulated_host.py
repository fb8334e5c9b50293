"""Bulk-level duplicate removal: the pp_bulk_* kernels of chromap_b200/csrc/postprocess.cuh run UNCHANGED on the host emulation
(tests/cta_emu.h), in pp_device's launch order (std::stable_sort, std::partial_sum and a serial reduce-by-key stand in for CUB),
and their survivors equal the host twin cmx_postprocess_bc_bulk on seeded record sets: long groups, returning barcodes
(single-end), ties, the last-group rule, 255 saturation, Tn5, several sequences; and a barcode outside the whitelist is counted."""
import subprocess

import numpy as np

import chromap_b200 as cb
from tests import emu
from tests.test_bulk_dedup_host import random_set

MAIN = r'''
template <typename F> static void launch(size_t n, F body) { if (n) emu_grid_serial((int)((n + 255) / 256), 256, body); }
static void stable_by_key(std::vector<u64> &keys, std::vector<u32> &idx) {
  std::vector<u32> ord(keys.size());
  std::iota(ord.begin(), ord.end(), 0u);
  std::stable_sort(ord.begin(), ord.end(), [&](u32 a, u32 b) { return keys[a] < keys[b]; });
  std::vector<u32> ni(idx.size());
  for (size_t i = 0; i < ord.size(); ++i) ni[i] = idx[ord[i]];
  idx.swap(ni);
}
int main(int argc, char **argv) {  // argv[1]: case file in, argv[2]: survivors out
  FILE *f = fopen(argv[1], "rb");
  u64 h[5];  // n, n_wl, single_end, mapq threshold, Tn5
  if (fread(h, 8, 5, f) != 5) return 2;
  const size_t n = h[0], n_wl = h[1];
  std::vector<PpRecord> a(n), b(n), res(n);
  std::vector<u64> bca(n), bcb(n), resbc(n), keys(n), wk(n_wl), wc(n_wl);
  if (fread(a.data(), sizeof(PpRecord), n, f) != n || fread(bca.data(), 8, n, f) != n || fread(wk.data(), 8, n_wl, f) != n_wl || fread(wc.data(), 8, n_wl, f) != n_wl) return 2;
  fclose(f);
  u64 ns = 64;
  while (ns < 2 * n_wl) ns <<= 1;
  int shift = 64;
  for (u64 s = ns; s > 1; s >>= 1) --shift;
  std::vector<ulonglong2> slots(ns, ulonglong2{~0ull, ~0ull});
  launch(n_wl, [&]() { tr_insert_kernel(wk.data(), wc.data(), n_wl, slots.data(), ns - 1, shift); });
  PpParams P{PP_BED_BC, 1, 1, (int)h[4], (int)h[3], (int)h[2]};
  P.bulk = 1;
  std::vector<u32> idx(n);
  launch(n, [&]() { pp_iota_kernel(idx.data(), n); });
  for (int w = pp_n_words(PP_BED_BC) - 1; w >= 0; --w) {
    launch(n, [&]() { pp_key_kernel(PP_BED_BC, w, a.data(), bca.data(), idx.data(), n, keys.data()); });
    stable_by_key(keys, idx);
  }
  launch(n, [&]() { pp_gather_kernel(a.data(), bca.data(), idx.data(), n, b.data(), bcb.data()); });
  unsigned long long n_missing = 0;
  PpAbundance A{slots.data(), ns - 1, shift, &n_missing};
  std::vector<u32> head(n), gid(n), pos(n);
  launch(n, [&]() { pp_bulk_entry_kernel(P.se, b.data(), bcb.data(), n, A, head.data(), keys.data()); });
  std::partial_sum(head.begin(), head.end(), gid.begin());
  std::vector<u64> best;  // reduce-by-key (max) over runs of equal gid
  for (size_t i = 0; i < n; ++i) { if (i == 0 || gid[i] != gid[i - 1]) best.push_back(0); best.back() = std::max(best.back(), keys[i]); }
  const u32 G = (u32)best.size();
  launch(n, [&]() { pp_bulk_heads_kernel(gid.data(), n, pos.data()); });
  unsigned last_mapq = 0;
  if (G) launch(n, [&]() { pp_bulk_last_mapq_kernel(b.data(), pos.data(), G, n, &last_mapq); });
  std::vector<u8> keep(G + 1);
  launch(G, [&]() { pp_bulk_resolve_kernel(P, b.data(), bcb.data(), best.data(), pos.data(), G, n, &last_mapq, res.data(), resbc.data(), keep.data()); });
  f = fopen(argv[2], "wb");
  u64 kept = 0;
  for (u32 g = 0; g < G; ++g) kept += keep[g];
  fwrite(&n_missing, 8, 1, f); fwrite(&kept, 8, 1, f);
  for (u32 g = 0; g < G; ++g) if (keep[g]) { fwrite(&res[g], sizeof(PpRecord), 1, f); fwrite(&resbc[g], 8, 1, f); }
  fclose(f);
  return 0;
}
'''


def _cases():
    rng = np.random.default_rng(41)
    for k in range(10):
        n = [1, 2, 40, 700, 3000, 4000, 4000, 300, 2500, 1500][k]
        recs, keys, wk, wc = random_set(rng, n, n_pos=3 if k in (5, 7) else 40, dense=k % 2 == 0)
        if k == 7:  # one position, one barcode: 300 records, num_dups saturates
            recs["rid"] = 1; recs["fragment_start"] = 99; recs["fragment_length"] = 41; keys[:] = wk[2]
        for se in (0, 1):
            for q, tn5 in ((0, 0), (30, 1)):
                yield recs, keys, wk, wc, se, q, tn5


def test_bulk_kernels_equal_host_twin(tmp_path):
    exe = emu.build(tmp_path, ["device_common.cuh", "postprocess.cuh"], MAIN)
    n_cases = n_kept = 0
    for c, (recs, keys, wk, wc, se, q, tn5) in enumerate(_cases()):
        fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
        with open(fin, "wb") as f:
            f.write(np.array([len(recs), len(wk), se, q, tn5], dtype=np.uint64).tobytes())
            f.write(np.ascontiguousarray(recs).tobytes()); f.write(keys.astype(np.uint64).tobytes())
            f.write(wk.astype(np.uint64).tobytes()); f.write(wc.astype(np.uint64).tobytes())
        subprocess.check_call([str(exe), str(fin), str(fout)], timeout=600)
        raw = open(fout, "rb").read()
        n_missing, kept = np.frombuffer(raw[:16], dtype=np.uint64)
        rows = np.frombuffer(raw[16:], dtype=np.dtype([("r", cb.PE_RECORD), ("k", "<u8")]))
        p = cb.make_params("", low_memory_mode=1, remove_pcr_duplicates=1, mapq_threshold=q, single_end=se, tn5_shift=tn5)
        want_r, want_k = cb.postprocess_bc_bulk(p, wk, wc, recs, keys)
        assert n_missing == 0 and kept == len(want_r), (c, kept, len(want_r))
        for f in want_r.dtype.names:  # field by field: the two padding bytes of a record are not defined
            assert np.array_equal(rows["r"][f], want_r[f]), (c, f)
        assert np.array_equal(rows["k"], want_k), c
        n_cases += 1; n_kept += len(want_r)
    assert n_cases == 40 and n_kept > 4000


def test_bulk_entry_kernel_counts_barcodes_outside_the_whitelist(tmp_path):
    exe = emu.build(tmp_path, ["device_common.cuh", "postprocess.cuh"], MAIN)
    rng = np.random.default_rng(5)
    recs, keys, wk, wc = random_set(rng, 500)
    keys[[3, 4]] = 77777
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(fin, "wb") as f:
        f.write(np.array([len(recs), len(wk), 0, 0, 0], dtype=np.uint64).tobytes())
        f.write(np.ascontiguousarray(recs).tobytes()); f.write(keys.astype(np.uint64).tobytes())
        f.write(wk.astype(np.uint64).tobytes()); f.write(wc.astype(np.uint64).tobytes())
    subprocess.check_call([str(exe), str(fin), str(fout)], timeout=600)
    assert np.frombuffer(open(fout, "rb").read()[:8], dtype=np.uint64)[0] >= 1
