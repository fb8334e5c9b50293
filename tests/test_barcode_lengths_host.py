"""Cell barcodes of every length from 1 to 32 and at both ends of the 2L-bit key space, without a GPU.

A barcode key packs 2 bits per base, so at L = 32 the all-T barcode's key is ~0, the empty-slot marker of the device's keyed
tables.  The whitelist keeps that key out of its slots and answers for it beside them (wl_lookup, device_common.cuh).

- The barcode gate (`wl_insert_kernel`, `barcode_kernel`, `barcode_correct2_kernel` of chromap_b200/csrc/pipeline_kernels.cuh)
  runs UNCHANGED on the host emulation of a CTA (tests/cta_emu.h), in the order `lane_barcodes` gives run_lane, against the
  oracle's CorrectBarcodeAt (`orc_correct_barcode_test`) at every L from 1 to 32 and thresholds 0, 1 and 2: per barcode the
  key and the accept flag, and both counters.  Whitelists: the whole key space and the whole space but the all-T key (L <= 5);
  all-A, all-T, their keys one and two substitutions away at positions 0 and L - 1 and random keys, with and without the two
  extremes themselves.  Barcodes: the extremes and their neighbours, listed keys with 0 to 2 substitutions, an N at the first
  or the last position, both, all N, lower-case bases (they count as their base; a lower-case n counts as A in the key but
  is not an N), random ones; Phred qualities 0 to 44 (both clamps of [3, 40]).
- Bulk-level duplicate removal: the `pp_bulk_*` kernels of postprocess.cuh on the emulated CTAs equal the host twin
  cmx_postprocess_bc_bulk on records whose barcodes include the all-T 32-mer and the all-A one, in ties of entry weight, so
  their abundance decides which record a group keeps.
- The oracle's whole-file scATAC run equals the reference binary (oracle/_ref/chromap, run at test time) on a seeded set of
  20,000 pairs with barcodes of 1, 2, 17, 31 and 32 bases: the BED byte for byte and both barcode counts.  At 32 bases the
  whitelist holds both extremes and the reads carry them.  Some barcodes have lower-case bases or a lower-case n."""
import os
import re
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests import emu
from tests.bc_error2_oracle import correct_barcodes
from tests.boundary_inputs import make_reads, reference
from tests.test_bulk_dedup_host import random_set as bulk_random_set

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")
ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
ALL_T = np.uint64(0xFFFFFFFFFFFFFFFF)

MAIN = r'''
struct EmuLaunch {  // lane_barcodes' launches on emulated CTAs
  template <typename... KA, typename... A>
  void operator()(void (*kernel)(KA...), int grid, int block, size_t, A... a) { emu_grid(grid, block, [&]() { kernel(a...); }); }
};
template <typename F> static void launch(size_t n, F body) { if (n) emu_grid_serial((int)((n + 255) / 256), 256, body); }
// The whitelist table as cmx_upload_barcode_whitelist builds it.  The scan for the key ~0 restates that entry's host code, so
// this file tests the kernels' half of the table; the entry's own scan is covered by test_gpu_barcode_lengths at L = 32.
static void whitelist_table(const std::vector<u64> &wk, const std::vector<u32> &wc, std::vector<ulonglong2> &slots, u64 *mask, int *shift, int *top_listed, u64 *top_count) {
  const u64 n = wk.size();
  u64 ns = 64;
  while (ns < 2 * n) ns <<= 1;
  int lg = 0;
  while ((1ull << lg) < ns) ++lg;
  slots.assign(ns, ulonglong2{CMX_EMPTY_KEY, CMX_EMPTY_KEY});
  *mask = ns - 1; *shift = 64 - lg; *top_listed = 0; *top_count = 0;
  for (u64 i = 0; i < n; ++i) if (wk[i] == CMX_EMPTY_KEY) { *top_listed = 1; *top_count = wc[i]; }
  if (n) emu_grid((int)((n + 255) / 256), 256, [&]() { wl_insert_kernel(wk.data(), wc.data(), n, slots.data(), *mask, *shift); });
}
// in: L, threshold, n_wl, n, num_sample, output_not_in_whitelist (u64), probability threshold (double), whitelist keys (u64),
// counts (u32), barcodes, qualities.  out: keys (u64), flags (u8), in-whitelist and corrected counters (u64).
static int gate(FILE *f, FILE *o) {
  u64 h[6];
  double prob;
  if (fread(h, 8, 6, f) != 6 || fread(&prob, 8, 1, f) != 1) return 2;
  const int L = (int)h[0];
  const size_t n_wl = h[2], n = h[3];
  std::vector<u64> wk(n_wl);
  std::vector<u32> wc(n_wl);
  std::string bcs(n * L, ' '), quals(n * L, ' ');
  if (fread(wk.data(), 8, n_wl, f) != n_wl || fread(wc.data(), 4, n_wl, f) != n_wl || fread(&bcs[0], 1, n * L, f) != n * L || fread(&quals[0], 1, n * L, f) != n * L) return 2;
  std::vector<ulonglong2> slots;
  DevWhitelist W{};
  g_emu_leavable = true;
  whitelist_table(wk, wc, slots, &W.mask, &W.shift, &W.top_listed, &W.top_count);
  std::vector<double> pw(81);
  for (int q = 0; q <= 80; ++q) pw[q] = pow(10.0, ((-q) / 10.0));
  std::vector<u32> list(n + 1), over(n + 1);
  std::vector<Bc2Slab> slab(BC2_SLAB_WARPS);
  W.slots = slots.data(); W.num_sample = (double)h[4]; W.pow_tab = pw.data(); W.err_threshold = (int)h[1]; W.prob_threshold = prob;
  W.output_not_in_whitelist = (int)h[5]; W.active = 1;
  W.c2_list = list.data(); W.c2_over = over.data(); W.c2_slab = slab.data();
  std::vector<u64> key(n + 1);
  std::vector<u8> ok(n + 1);
  Counters ctr{};
  EmuLaunch x;
  lane_barcodes(x, W, (const u8 *)bcs.data(), (const u8 *)quals.data(), L, (int)n, key.data(), ok.data(), &ctr);
  g_emu_leavable = false;
  fwrite(key.data(), 8, n, o); fwrite(ok.data(), 1, n, o);
  fwrite(&ctr.n_bc_in_whitelist, 8, 1, o); fwrite(&ctr.n_bc_corrected, 8, 1, o);
  return 0;
}
static void stable_by_key(std::vector<u64> &keys, std::vector<u32> &idx) {
  std::vector<u32> ord(keys.size());
  std::iota(ord.begin(), ord.end(), 0u);
  std::stable_sort(ord.begin(), ord.end(), [&](u32 a, u32 b) { return keys[a] < keys[b]; });
  std::vector<u32> ni(idx.size());
  for (size_t i = 0; i < ord.size(); ++i) ni[i] = idx[ord[i]];
  idx.swap(ni);
}
// pp_device's launch order for bulk-level removal (std::stable_sort, std::partial_sum and a serial reduce-by-key stand in
// for CUB).  in: n, n_wl, single_end, MAPQ threshold, Tn5 (u64), records, barcode keys (u64), whitelist keys (u64), counts
// (u32).  out: missing barcodes, survivors (u64), then each survivor's record and barcode key.
static int bulk(FILE *f, FILE *o) {
  u64 h[5];
  if (fread(h, 8, 5, f) != 5) return 2;
  const size_t n = h[0], n_wl = h[1];
  std::vector<PpRecord> a(n), b(n), res(n);
  std::vector<u64> bca(n), bcb(n), resbc(n), keys(n), wk(n_wl);
  std::vector<u32> wc(n_wl);
  if (fread(a.data(), sizeof(PpRecord), n, f) != n || fread(bca.data(), 8, n, f) != n || fread(wk.data(), 8, n_wl, f) != n_wl || fread(wc.data(), 4, n_wl, f) != n_wl) return 2;
  std::vector<ulonglong2> slots;
  PpAbundance A{};
  unsigned long long n_missing = 0;
  g_emu_leavable = true;
  whitelist_table(wk, wc, slots, &A.mask, &A.shift, &A.top_listed, &A.top_count);
  g_emu_leavable = false;
  A.slots = slots.data(); A.n_missing = &n_missing;
  PpParams P{PP_BED_BC, 1, 1, (int)h[4], (int)h[3], (int)h[2]};
  P.bulk = 1;
  std::vector<u32> idx(n);
  launch(n, [&]() { pp_iota_kernel(idx.data(), n); });
  for (int w = pp_n_words(PP_BED_BC) - 1; w >= 0; --w) {
    launch(n, [&]() { pp_key_kernel(PP_BED_BC, w, a.data(), bca.data(), idx.data(), n, keys.data()); });
    stable_by_key(keys, idx);
  }
  launch(n, [&]() { pp_gather_kernel(a.data(), bca.data(), idx.data(), n, b.data(), bcb.data()); });
  std::vector<u32> head(n), gid(n), pos(n);
  launch(n, [&]() { pp_bulk_entry_kernel(P.se, b.data(), bcb.data(), n, A, head.data(), keys.data()); });
  std::partial_sum(head.begin(), head.end(), gid.begin());
  std::vector<u64> best;
  for (size_t i = 0; i < n; ++i) { if (i == 0 || gid[i] != gid[i - 1]) best.push_back(0); best.back() = std::max(best.back(), keys[i]); }
  const u32 G = (u32)best.size();
  launch(n, [&]() { pp_bulk_heads_kernel(gid.data(), n, pos.data()); });
  unsigned last_mapq = 0;
  if (G) launch(n, [&]() { pp_bulk_last_mapq_kernel(b.data(), pos.data(), G, n, &last_mapq); });
  std::vector<u8> keep(G + 1);
  launch(G, [&]() { pp_bulk_resolve_kernel(P, b.data(), bcb.data(), best.data(), pos.data(), G, n, &last_mapq, res.data(), resbc.data(), keep.data()); });
  u64 kept = 0;
  for (u32 g = 0; g < G; ++g) kept += keep[g];
  fwrite(&n_missing, 8, 1, o); fwrite(&kept, 8, 1, o);
  for (u32 g = 0; g < G; ++g) if (keep[g]) { fwrite(&res[g], sizeof(PpRecord), 1, o); fwrite(&resbc[g], 8, 1, o); }
  return 0;
}
int main(int argc, char **argv) {  // argv[1]: gate | bulk, argv[2]: case file in, argv[3]: result out
  FILE *f = fopen(argv[2], "rb"), *o = fopen(argv[3], "wb");
  const int rc = std::string(argv[1]) == "gate" ? gate(f, o) : bulk(f, o);
  fclose(f); fclose(o);
  return rc;
}
'''


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return emu.build(tmp_path_factory.mktemp("bc_lengths"), emu.PIPELINE + ["postprocess.cuh"], MAIN)


def extremes(L):
    """All-A, all-T, and their keys one and two substitutions away at positions 0 and L - 1 (rows of L bases)."""
    rows = []
    for c in b"AT":
        e = np.full(L, c, dtype=np.uint8)
        rows.append(e)
        for p in sorted({0, L - 1}):
            for x in ACGT:
                if x != c:
                    r = e.copy(); r[p] = x; rows.append(r)
        if L > 1:
            for x in ACGT:
                for y in ACGT:
                    if x != c and y != c:
                        r = e.copy(); r[0] = x; r[L - 1] = y; rows.append(r)
    return np.array(rows)


def keys_of(rows):
    """The 2-bit keys of rows of bases: either case counts as the base, anything else as A."""
    up = np.where((rows >= ord("a")) & (rows <= ord("z")), rows - 32, rows)
    code = np.where(np.isin(up, ACGT), np.searchsorted(ACGT, up), 0).astype(np.uint64)
    k = np.zeros(len(rows), dtype=np.uint64)
    for j in range(rows.shape[1]):
        k = (k << np.uint64(2)) | code[:, j]
    return k


def _substitute(rng, row, k, positions=None):
    L = len(row)
    pos = positions if positions is not None else rng.choice(L, min(k, L), replace=False)
    for p in pos:
        row[p] = ACGT[(np.searchsorted(ACGT, row[p]) + rng.integers(1, 4)) % 4]


def whitelists(L):
    """(name, rows) of the whitelists at barcode length L."""
    rng = np.random.default_rng(1000 + L)
    ext = extremes(L)
    rnd = ACGT[rng.integers(0, 4, (min(300, 4 ** L), L))]
    both = np.concatenate([ext, rnd])
    out = [("extremes", both), ("neighbours", both[~np.isin(keys_of(both), np.array([0, (1 << 2 * L) - 1], dtype=np.uint64))])]
    if L <= 5:
        every = ACGT[(np.arange(4 ** L)[:, None] >> (2 * np.arange(L - 1, -1, -1))[None, :]) & 3]
        out += [("whole space", every), ("whole space but all-T", every[:-1])]
    return out


def gate_set(L, rows, n, seed):
    """Abundance sample, barcodes and qualities for the whitelist `rows` (see the module docstring)."""
    rng = np.random.default_rng(seed)
    allA, allT = np.full(L, ord("A"), np.uint8), np.full(L, ord("T"), np.uint8)
    favT, favA = allT.copy(), allA.copy()  # one neighbour of each extreme takes a large share, so an unlisted extreme is corrected
    favT[0] = ord("G"); favA[L - 1] = ord("C")
    # abundances: all-T 25 %, all-A 10 %, the favoured neighbours 15 % and 5 %, the rest spread over the whitelist
    m = 4000
    pick = rng.random(m)
    sample = rows[rng.integers(0, len(rows), m)].copy()
    sample[pick < 0.25] = allT; sample[(pick >= 0.25) & (pick < 0.35)] = allA
    sample[(pick >= 0.35) & (pick < 0.5)] = favT; sample[(pick >= 0.5) & (pick < 0.55)] = favA
    base = rows[rng.integers(0, len(rows), n)].copy()
    which = rng.random(n)
    base[which < 0.3] = allT; base[(which >= 0.3) & (which < 0.45)] = allA
    kind = rng.integers(0, 20, n)
    for i in range(n):
        r, k = base[i], kind[i]
        if k < 6:
            continue  # as drawn
        if k < 9:
            _substitute(rng, r, 1)
        elif k == 9:
            _substitute(rng, r, 1, positions=[rng.choice([0, L - 1])])
        elif k < 12:
            _substitute(rng, r, 2)
        elif k == 12:
            _substitute(rng, r, 2, positions=sorted({0, L - 1}))
        elif k == 13:
            r[0] = ord("N")
        elif k == 14:
            r[L - 1] = ord("N")
        elif k == 15:
            r[[0, L - 1]] = ord("N")
        elif k == 16:
            r[:] = ord("N")
        elif k == 17:
            r[rng.random(L) < 0.5] += 32  # lower case: the same bases
        elif k == 18:
            r[rng.integers(0, L)] = ord("n")  # A in the key, not an N
        else:
            r[:] = ACGT[rng.integers(0, 4, L)]
    quals = (rng.integers(0, 45, (n, L)) + 33).astype(np.uint8)
    return sample.ravel(), base, quals


def _whitelist(tmp_path, L, rows, sample):
    path = tmp_path / "wl.txt"
    path.write_bytes(b"".join(bytes(r) + b"\n" for r in rows))
    wl = orc.Whitelist(str(path), L)
    wl.sample(sample)
    return wl


def _gate(exe, tmp_path, wl, L, thr, prob, bcs, quals):
    keys, counts, ns = wl.arrays()
    fin, fout = tmp_path / "gate.in", tmp_path / "gate.out"
    n = len(bcs) // L
    with open(fin, "wb") as f:
        f.write(np.array([L, thr, len(keys), n, ns, 0], dtype=np.uint64).tobytes() + np.array([prob]).tobytes())
        f.write(keys.tobytes() + counts.astype(np.uint32).tobytes() + bcs.tobytes() + quals.tobytes())
    subprocess.check_call([str(exe), "gate", str(fin), str(fout)], timeout=600)
    raw = open(fout, "rb").read()
    k = np.frombuffer(raw[:8 * n], dtype=np.uint64)
    ok = np.frombuffer(raw[8 * n:9 * n], dtype=np.uint8)
    ctr = np.frombuffer(raw[9 * n:], dtype=np.uint64)
    return k, ok, int(ctr[0]), int(ctr[1])


@pytest.mark.parametrize("L", range(1, 33))
def test_barcode_gate_equals_the_oracle_at_every_length(exe, tmp_path, L):
    prob = 0.9 if L % 2 == 0 else 0.5
    top = np.uint64((1 << 2 * L) - 1)
    floors = dict(exact_t=0, to_t=0, from_t=0)
    for c, (name, rows) in enumerate(whitelists(L)):
        sample, obs, quals = gate_set(L, rows, n=1200 if L == 32 else 500, seed=L * 10 + c)
        wl = _whitelist(tmp_path, L, rows, sample)
        listed = set(wl.arrays()[0].tolist())
        assert (int(top) in listed) == (name in ("extremes", "whole space")), name
        bcs = obs.ravel()
        pure = np.all(np.isin(obs, ACGT), axis=1)  # upper-case bases only
        for thr in (0, 1, 2):
            got = _gate(exe, tmp_path, wl, L, thr, prob, bcs, quals.ravel())
            want = correct_barcodes(wl, thr, prob, bcs, quals.ravel(), L)
            bad = np.flatnonzero((got[0] != want[0]) | (got[1] != want[1]))
            assert len(bad) == 0 and got[2:] == want[2:], (
                "L=%d whitelist=%s threshold=%d: %d barcodes differ, first %s: key %x / oracle %x, ok %d / oracle %d; counters %s / %s"
                % (L, name, thr, len(bad), bytes(obs[bad[0]]).decode() if len(bad) else "-", got[0][bad[0]] if len(bad) else 0,
                   want[0][bad[0]] if len(bad) else 0, got[1][bad[0]] if len(bad) else 0, want[1][bad[0]] if len(bad) else 0, got[2:], want[2:]))
            src = keys_of(obs)
            floors["exact_t"] += int(np.sum(pure & (src == top) & (want[1] == 1) & (want[0] == top)))
            floors["to_t"] += int(np.sum((src != top) & (want[1] == 1) & (want[0] == top)))
            floors["from_t"] += int(np.sum(pure & (src == top) & (want[1] == 1) & (want[0] != top)))
            if name.startswith("whole space"):  # every barcode without an N hits
                assert want[2] == int(np.sum(np.all(obs != ord("N"), axis=1) & ((src != top) | (name == "whole space")))), (name, thr)
    assert floors["exact_t"] > 0, floors
    if L == 32:
        assert min(floors.values()) >= 100, floors


def test_bulk_kernels_rank_the_extreme_keys_by_abundance(exe, tmp_path):
    rng = np.random.default_rng(32)
    n_cases = n_top_kept = n_top_lost = 0
    for c in range(8):
        recs, keys, wk, wc = bulk_random_set(rng, [300, 2000, 4000, 1500][c % 4], n_pos=[3, 10, 40, 2][c % 4], dense=c % 2 == 0)
        old = wk.copy()
        wk[0], wk[1] = ALL_T, 0  # the all-T and all-A 32-mers, the all-T one most or least abundant
        keys = wk[np.searchsorted(old, keys)]
        wc[:] = 7
        wc[0], wc[1] = (10, 3) if c % 2 else (3, 10)
        for se in (0, 1):
            fin, fout = tmp_path / "bulk.in", tmp_path / "bulk.out"
            with open(fin, "wb") as f:
                f.write(np.array([len(recs), len(wk), se, 0, c % 3 == 0], dtype=np.uint64).tobytes())
                f.write(np.ascontiguousarray(recs).tobytes() + keys.astype(np.uint64).tobytes() + wk.astype(np.uint64).tobytes() + wc.astype(np.uint32).tobytes())
            subprocess.check_call([str(exe), "bulk", str(fin), str(fout)], timeout=600)
            raw = open(fout, "rb").read()
            n_missing, kept = np.frombuffer(raw[:16], dtype=np.uint64)
            rows = np.frombuffer(raw[16:], dtype=np.dtype([("r", cb.PE_RECORD), ("k", "<u8")]))
            p = cb.make_params("", low_memory_mode=1, remove_pcr_duplicates=1, mapq_threshold=0, single_end=se, tn5_shift=int(c % 3 == 0))
            want_r, want_k = cb.postprocess_bc_bulk(p, wk, wc, recs, keys)
            assert n_missing == 0, (c, se, "barcodes reported missing from the whitelist", int(n_missing))
            assert kept == len(want_r), (c, se, kept, len(want_r))
            for f in want_r.dtype.names:
                assert np.array_equal(rows["r"][f], want_r[f]), (c, se, f)
            assert np.array_equal(rows["k"], want_k), (c, se)
            n_cases += 1
            top = want_k == ALL_T
            n_top_kept += int(top.sum())
            t = keys == ALL_T
            n_top_lost += len(set(zip(recs["rid"][t].tolist(), recs["fragment_start"][t].tolist(), (recs["fragment_length"][t] * (1 - se)).tolist()))) - int(top.sum())
    assert n_cases == 16 and n_top_kept > 50 and n_top_lost > 50, (n_top_kept, n_top_lost)


# ---- the oracle against the reference binary ----------------------------------------------------------------------------
N_CLI_PAIRS = 20000


def cli_barcodes(n, L, seed, path):
    """A whitelist written to `path` (distinct random keys, all-A and all-T) and n barcodes with qualities from it: 10 % all-T,
    10 % all-A, 8 % with one substitution, 4 % with two, 3 % with an N, 3 % random, 2 % with lower-case bases, 1 % with a
    lower-case n; Phred 0 to 41."""
    rng = np.random.default_rng(seed)
    wl = np.concatenate([ACGT[rng.integers(0, 4, (min(3000, 4 ** L // 2 + 1), L))], np.full((1, L), ord("A"), np.uint8), np.full((1, L), ord("T"), np.uint8)])
    wl = wl[np.sort(np.unique(keys_of(wl), return_index=True)[1])]  # the reference refuses a whitelist that lists a key twice
    with open(path, "wb") as f:
        f.write(b"".join(bytes(r) + b"\n" for r in wl))
    obs = wl[rng.integers(0, min(len(wl), 800), n)]
    kind = rng.random(n)
    obs[kind < 0.1] = ord("T")
    obs[(kind >= 0.1) & (kind < 0.2)] = ord("A")
    kind = rng.random(n)
    for i in np.flatnonzero(kind < 0.12):
        _substitute(rng, obs[i], 1 if kind[i] < 0.08 else 2)
    rows = np.flatnonzero((kind >= 0.12) & (kind < 0.15))
    obs[rows, rng.integers(0, L, len(rows))] = ord("N")
    rows = np.flatnonzero((kind >= 0.15) & (kind < 0.18))
    obs[rows] = ACGT[rng.integers(0, 4, (len(rows), L))]
    rows = np.flatnonzero((kind >= 0.18) & (kind < 0.2))  # lower case: the same bases
    obs[rows] |= (rng.random((len(rows), L)) < 0.5).astype(np.uint8) << 5
    rows = np.flatnonzero((kind >= 0.2) & (kind < 0.21))  # a lower-case n: A in the key, not an N
    obs[rows, rng.integers(0, L, len(rows))] = ord("n")
    quals = (rng.integers(0, 42, (n, L)) + 33).astype(np.uint8)
    return obs, quals


def fastq_q(seqs, quals, prefix=b"r"):
    """4-line FASTQ text of rows of bases with their qualities."""
    return b"".join(b"@%s%08d\n%s\n+\n%s\n" % (prefix, i, bytes(s), bytes(q)) for i, (s, q) in enumerate(zip(seqs, quals)))


def write_inputs(d, n_pairs=N_CLI_PAIRS):
    """The boundary_inputs reference as ref.fa and n_pairs 2x50 bp pairs as r1.fq / r2.fq in directory d."""
    seqs, _ = reference()
    with open(os.path.join(d, "ref.fa"), "wb") as f:
        for i, a in enumerate(seqs):
            f.write(b">chr%d\n" % (i + 1) + a.tobytes() + b"\n")
    s1, _, s2, _ = make_reads(n_pairs, seed=31, length=50)
    q = np.full((n_pairs, 50), ord("I"), np.uint8)
    for mate, s in (("1", s1), ("2", s2)):
        with open(os.path.join(d, "r%s.fq" % mate), "wb") as f:
            f.write(fastq_q(s.reshape(n_pairs, 50), q))


def write_barcodes(d, L, n_pairs=N_CLI_PAIRS):
    """bc<L>.fq and wl<L>.txt in directory d; returns their paths."""
    bc, wl = os.path.join(d, "bc%d.fq" % L), os.path.join(d, "wl%d.txt" % L)
    obs, quals = cli_barcodes(n_pairs, L, 500 + L, wl)
    with open(bc, "wb") as f:
        f.write(fastq_q(obs, quals, prefix=b"b"))
    return bc, wl


BC_COUNTS = re.compile(r"^Number of (barcodes in whitelist|corrected barcodes): (\d+)\.$", re.M)


def bc_counts(stderr):
    return {m.group(1): int(m.group(2)) for m in BC_COUNTS.finditer(stderr)}


@pytest.fixture(scope="module")
def cli_inputs(tmp_path_factory):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    d = str(tmp_path_factory.mktemp("bc_cli"))
    write_inputs(d)
    subprocess.check_call([REF_BIN, "-i", "-r", os.path.join(d, "ref.fa"), "-o", os.path.join(d, "ref.index")], stderr=subprocess.DEVNULL)
    return d


@pytest.mark.parametrize("L", [1, 2, 17, 31, 32])
def test_oracle_equals_the_reference_binary_at_barcode_lengths(cli_inputs, L):
    d = cli_inputs
    bc, wl = write_barcodes(d, L)
    idx, ref = os.path.join(d, "ref.index"), os.path.join(d, "ref.fa")
    want_path, got_path = os.path.join(d, "want.bed"), os.path.join(d, "got.bed")
    r = subprocess.run([REF_BIN, "--preset", "atac", "-x", idx, "-r", ref, "-1", os.path.join(d, "r1.fq"), "-2", os.path.join(d, "r2.fq"), "-b", bc,
                        "--barcode-whitelist", wl, "-t", str(os.cpu_count() or 1), "-o", want_path], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    want = open(want_path, "rb").read()
    st = orc.run_files_bc(orc.make_params("atac"), idx, ref, os.path.join(d, "r1.fq"), os.path.join(d, "r2.fq"), bc, wl, got_path, n_threads=4)
    got = open(got_path, "rb").read()
    assert got == want, (L, len(got), len(want))
    assert bc_counts(r.stderr) == {"barcodes in whitelist": int(st[0]), "corrected barcodes": int(st[1])}, (bc_counts(r.stderr), st)
    assert want.count(b"\n") > 5000 and (int(st[1]) > 0 or L == 1)  # one base: every key is listed, an N has four equal choices
    if L == 32:  # both extremes reach the output
        fields = [l.split(b"\t")[3] for l in want.splitlines()]
        assert fields.count(b"T" * 32) > 100 and fields.count(b"A" * 32) > 100
