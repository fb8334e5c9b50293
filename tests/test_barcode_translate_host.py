"""--barcode-translate without a device: the table parser against a restatement of SetTranslateTable / ProcessTranslateFileLine
(tests/translate_oracle.py), the host twin of the translated BED text against the oracle's Translate, the BED kernels with a
table on the CTA emulator, the oracle against the reference binary's translated outputs (tests/golden/synth_barcode_translate,
made by make_golden_barcode_translate.sh), and the CLI's refusals of malformed tables."""
import gzip
import hashlib
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests import emu
from tests import translate_oracle as tro
from tests.util import load_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "synth_barcode_translate")
SC = os.path.join(ROOT, "tests", "golden", "synth_sc")
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")

ACCEPTED = {
    "one": b"x,ACGT\n",
    "tab_and_comma": b"cellA\tACGT\ncellB,TTTT\n",
    "no_final_newline": b"a,AC\nb,GT",
    "empty_to": b",ACG\nb,TTT\n",
    "lower_case": b"a,acgt\nb,AcGt\n",
    "repeat_later_wins": b"first,ACGT\nother,CCCC\nsecond,ACGT\n",
    "repeat_case_folded": b"first,acgt\nsecond,ACGT\n",
    "to_with_spaces": b"cell name 1,ACGTA\n",
    "L1": b"a,A\nc,C\ng,G\nt,T\n",
    "L31": b"x," + b"ACGT" * 7 + b"ACG\n",
    "line_510": b"t" * 489 + b"," + b"A" * 20 + b"\n",
}
REFUSED = {
    "empty_file": b"",
    "empty_line": b"a,ACGT\n\nb,TTTT\n",
    "only_newline": b"\n",
    "no_separator": b"a,ACGT\nbTTTT\n",
    "empty_from": b"a,\n",
    "n_in_from": b"a,ACNT\n",
    "crlf": b"a,ACGT\r\nb,TTTT\r\n",
    "space_in_from": b"a, ACGT\n",
    "second_separator_in_from": b"a\tb,ACGT\n",
    "lengths_differ": b"a,ACGT\nb,ACG\n",
    "L32": b"x," + b"ACGT" * 8 + b"\n",
    "line_511": b"t" * 490 + b"," + b"A" * 20 + b"\n",
    "nul_in_to": b"a\0b,ACGT\n",
    "nul_in_from": b"a,AC\0T\n",
}


def _as_dict(t):
    return {int(k): v for k, v in zip(t.keys, t.to)}, t.from_len


@pytest.mark.parametrize("case", sorted(ACCEPTED))
def test_parser_accepts_what_the_reference_defines(case):
    data = ACCEPTED[case]
    assert _as_dict(cb.parse_barcode_translation(data)) == tro.load_translation(data)
    assert _as_dict(cb.parse_barcode_translation(gzip.decompress(gzip.compress(data)))) == tro.load_translation(data)


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_parser_refuses_and_names_the_line(case):
    with pytest.raises(cb.CmxError, match="line [0-9]+: "):
        cb.parse_barcode_translation(REFUSED[case])


def test_parser_keeps_first_appearance_order_and_last_value():
    t = cb.parse_barcode_translation(b"a,CCCC\nb,AAAA\nc,CCCC\n")
    assert list(t.keys) == [tro._seed(b"CCCC"), 0] and t.to == [b"c", b"b"] and t.from_len == 4


def _random_case(rng, n, bc_len, L, n_keys, drop=0.0):
    """Records over three sequences, barcodes of bc_len bases drawn so that their segments collide often, and a table of
    L-mers (with random TO names, some empty) that covers them unless `drop` removes entries."""
    recs = np.zeros(n, dtype=cb.PE_RECORD)
    recs["rid"] = rng.integers(0, 3, n)
    recs["fragment_start"] = rng.choice([0, 9, 10, 99999, 1000000000, 4294967000], n)
    recs["fragment_length"] = rng.integers(0, 700, n)
    recs["num_dups"] = rng.integers(0, 256, n)
    seg_pool = rng.integers(0, 1 << (2 * L), n_keys, dtype=np.uint64)
    nseg = bc_len // L
    bcs = rng.integers(0, 1 << 62, n, dtype=np.uint64) & np.uint64((1 << (2 * bc_len)) - 1)
    for s in range(nseg):  # segment s of every barcode from the pool
        shift = np.uint64(2 * L * (nseg - 1 - s))
        seg_mask = np.uint64((1 << (2 * L)) - 1) << shift
        bcs = (bcs & ~seg_mask) | (rng.choice(seg_pool, n) << shift)
    keys = [int(k) for k in np.unique(seg_pool) if rng.random() >= drop]
    to = [bytes(rng.choice(list(b"abcXYZ_-0123"), int(rng.integers(0, 12)))) for _ in keys]
    return recs, bcs, cb.BarcodeTranslation(keys, to, L)


NAMES = ["chr1", "chrUn_long_name_7", "c"]
SHAPES = [(16, 16), (16, 8), (16, 5), (16, 4), (16, 20), (10, 3), (32, 8), (24, 12), (32, 31), (5, 5), (1, 1)]


def _oracle_text(recs, bcs, bc_len, t):
    """mapping_writer.cc:131-137 with the oracle's Translate (t None: Seed2Sequence, barcode_translator.h:114-123)."""
    names = [n.encode() for n in NAMES]
    table = {int(k): v for k, v in zip(t.keys, t.to)} if t is not None else None
    lines = []
    for r, bc in zip(recs, bcs):
        end = (int(r["fragment_start"]) + int(r["fragment_length"])) & 0xFFFFFFFF
        field = tro.translate((table, t.from_len), bc, bc_len) if t is not None else \
            bytes(b"ACGT"[(int(bc) >> (2 * (bc_len - 1 - j))) & 3] for j in range(bc_len))
        lines.append(b"%s\t%d\t%d\t%s\t%d\n" % (names[r["rid"]], r["fragment_start"], end, field, r["num_dups"]))
    return b"".join(lines)


@pytest.mark.parametrize("bc_len,L", SHAPES)
def test_host_twin_equals_the_oracle(bc_len, L):
    rng = np.random.default_rng(bc_len * 100 + L)
    recs, bcs, t = _random_case(rng, 3000, bc_len, L, 40)
    got = cb.format_bed_bc_tr(NAMES, recs, bcs, bc_len, t)
    assert got == _oracle_text(recs, bcs, bc_len, t)
    assert cb.format_bed_bc_tr(NAMES, recs, bcs, bc_len, None) == _oracle_text(recs, bcs, bc_len, None)


@pytest.mark.parametrize("bc_len,L", [(16, 8), (16, 5), (12, 4)])
def test_host_twin_refuses_a_missing_segment(bc_len, L):
    rng = np.random.default_rng(7 + L)
    recs, bcs, t = _random_case(rng, 2000, bc_len, L, 30, drop=0.2)
    with pytest.raises(tro.BarcodeMissing):
        _oracle_text(recs, bcs, bc_len, t)
    with pytest.raises(cb.BarcodeNotTranslated):
        cb.format_bed_bc_tr(NAMES, recs, bcs, bc_len, t)


EMU_MAIN = r'''
static std::vector<char> slurp(const char *p) { FILE *f = fopen(p, "rb"); std::vector<char> v; char b[65536]; size_t n; while ((n = fread(b, 1, sizeof b, f)) > 0) v.insert(v.end(), b, b + n); fclose(f); return v; }
template <typename T> static std::vector<T> as(const std::vector<char> &v) { std::vector<T> o(v.size() / sizeof(T)); memcpy(o.data(), v.data(), o.size() * sizeof(T)); return o; }
template <typename F> static void launch(size_t n, F body) { emu_grid_serial((int)((n + 255) / 256), 256, body); }
int main(int argc, char **argv) {
  // argv: dir bc_len L with_table
  const std::string d = argv[1];
  const int bc_len = atoi(argv[2]), L = atoi(argv[3]), with_table = atoi(argv[4]);
  std::vector<PpRecord> recs = as<PpRecord>(slurp((d + "/recs").c_str()));
  std::vector<u64> bcs = as<u64>(slurp((d + "/bcs").c_str())), keys = as<u64>(slurp((d + "/keys").c_str())), vals = as<u64>(slurp((d + "/vals").c_str()));
  std::vector<char> to = slurp((d + "/to").c_str());
  to.push_back(0);
  const std::string cat = "chr1chrUn_long_name_7c";
  std::vector<u32> noff{0, 4, 21, 22};
  const size_t n = recs.size(), nk = keys.size();
  u64 ns = 64;
  while (ns < 2 * nk) ns <<= 1;
  int lg = 0; while ((1ull << lg) < ns) ++lg;
  std::vector<ulonglong2> slots(ns, ulonglong2{CMX_EMPTY_KEY, CMX_EMPTY_KEY});
  launch(nk, [&]() { tr_insert_kernel(keys.data(), vals.data(), nk, slots.data(), ns - 1, 64 - lg); });
  u64 n_missing = 0; u32 first_missing = ~0u;
  BedTranslation T{};
  if (with_table) { T.slots = slots.data(); T.mask = ns - 1; T.shift = 64 - lg; T.from_len = L; T.to = to.data(); T.n_missing = &n_missing; T.first_missing = &first_missing; }
  std::vector<u32> len(n + 1, 0);
  launch(n, [&]() { bed_len_kernel(recs.data(), n, noff.data(), bc_len, len.data(), bcs.data(), T); });
  std::vector<u64> off(n + 1, 0);
  for (size_t i = 0; i < n; ++i) off[i + 1] = off[i] + len[i];
  printf("missing=%llu first=%u bytes=%llu\n", n_missing, n_missing ? first_missing : 0u, (unsigned long long)off[n]);
  if (n_missing) return 0;
  std::string text((size_t)off[n], '?');
  launch(n, [&]() { bed_write_kernel(recs.data(), bcs.data(), n, cat.data(), noff.data(), bc_len, off.data(), 0, &text[0], T); });
  FILE *f = fopen((d + "/text").c_str(), "wb"); fwrite(text.data(), 1, text.size(), f); fclose(f);
  return 0;
}
'''


@pytest.fixture(scope="module")
def emu_exe(tmp_path_factory):
    return emu.build(tmp_path_factory.mktemp("bedtr"), ["device_common.cuh", "postprocess.cuh"], EMU_MAIN)


def _emu_run(exe, d, recs, bcs, bc_len, t, with_table=True):
    t = t if t is not None else cb.BarcodeTranslation([0], [b""], 1)
    recs.tofile(str(d / "recs")); np.asarray(bcs, dtype=np.uint64).tofile(str(d / "bcs"))
    off = np.concatenate([[0], np.cumsum([len(x) for x in t.to])]).astype(np.uint64)
    (np.asarray(off[:-1], dtype=np.uint64) << np.uint64(16) | np.array([len(x) for x in t.to], dtype=np.uint64)).tofile(str(d / "vals"))
    t.keys.tofile(str(d / "keys")); (d / "to").write_bytes(b"".join(t.to))
    r = subprocess.run([str(exe), str(d), str(bc_len), str(t.from_len), str(int(with_table))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    f = dict(kv.split("=") for kv in r.stdout.split())
    return {k: int(v) for k, v in f.items()}, ((d / "text").read_bytes() if int(f["missing"]) == 0 else None)


@pytest.mark.parametrize("bc_len,L", [(16, 16), (16, 8), (16, 5), (16, 20), (32, 8), (24, 12)])
def test_bed_kernels_translate_on_the_emulator(emu_exe, tmp_path, bc_len, L):
    rng = np.random.default_rng(bc_len * 31 + L)
    recs, bcs, t = _random_case(rng, 1500, bc_len, L, 50)
    f, text = _emu_run(emu_exe, tmp_path, recs, bcs, bc_len, t)
    assert f["missing"] == 0 and text == _oracle_text(recs, bcs, bc_len, t) == cb.format_bed_bc_tr(NAMES, recs, bcs, bc_len, t)


def test_bed_kernels_without_a_table_write_the_barcode(emu_exe, tmp_path):
    rng = np.random.default_rng(5)
    recs, bcs, t = _random_case(rng, 1500, 16, 8, 50)
    f, text = _emu_run(emu_exe, tmp_path, recs, bcs, 16, t, with_table=False)
    assert f["missing"] == 0 and text == _oracle_text(recs, bcs, 16, None)


@pytest.mark.parametrize("bc_len,L", [(16, 8), (16, 4), (15, 5)])
def test_bed_kernels_count_missing_segments(emu_exe, tmp_path, bc_len, L):
    rng = np.random.default_rng(11 * L)
    recs, bcs, t = _random_case(rng, 1500, bc_len, L, 30, drop=0.25)
    table = {int(k) for k in t.keys}
    nseg = bc_len // L
    per_rec = [sum(((int(b) >> (2 * L * (nseg - 1 - s))) & ((1 << 2 * L) - 1)) not in table for s in range(nseg)) for b in bcs]
    f, text = _emu_run(emu_exe, tmp_path, recs, bcs, bc_len, t)
    assert sum(per_rec) > 0 and text is None
    assert f["missing"] == sum(per_rec) and f["first"] == next(i for i, m in enumerate(per_rec) if m)


# ---- the oracle against the reference binary's translated outputs
def _md5s():
    return dict(line.split()[::-1] for line in open(os.path.join(GOLD, "md5.txt")))


def _barcodes(path):
    lines = gzip.open(path).read().split(b"\n")
    return np.frombuffer(b"".join(lines[1::4]), dtype=np.uint8), np.frombuffer(b"".join(lines[3::4]), dtype=np.uint8), len(lines[1])


GOLDEN_CASES = {  # output: (table, single-end, params, whitelist, --output-mappings-not-in-whitelist)
    "pe_rc16": ("rc16", False, dict(preset="atac"), True, False),
    "se_rc16": ("rc16", True, dict(preset="atac"), True, False),
    "se_inmem_rc16": ("rc16", True, dict(preset="", mapq_threshold=0, remove_pcr_duplicates=1, tn5_shift=1), True, False),
    "pe_names": ("names", False, dict(preset="atac"), True, False),
    "pe_half8": ("half8", False, dict(preset="atac"), True, False),
    "pe_all5_nowl": ("all5", False, dict(preset="atac"), False, False),
    "pe_all5_notinwl": ("all5", False, dict(preset="atac"), True, True),
    "pe_long20": ("long20", False, dict(preset="atac"), True, False),
}


@pytest.fixture(scope="module")
def sc_setup():
    ref = orc.Reference(os.path.join(SC, "ref.fa.gz"))
    idx = orc.Index(ref=ref, k=17, w=7)
    s1, o1, s2, o2 = load_pairs(SC)
    bcs, quals, bc_len = _barcodes(os.path.join(SC, "barcode.fq.gz"))
    return ref, idx, (s1, o1, s2, o2), (bcs, quals, bc_len)


def _oracle_records(sc_setup, case):
    ref, idx, (s1, o1, s2, o2), (bcs, quals, bc_len) = sc_setup
    _, se, kw, use_wl, out_nw = GOLDEN_CASES[case]
    kw = dict(kw)
    p = orc.make_params(kw.pop("preset"), single_end=int(se), **kw)
    wl = None
    if use_wl:
        wl = orc.Whitelist(os.path.join(SC, "whitelist.txt"), bc_len)
        wl.sample(bcs)
    if se:
        recs, obc, _ = orc.map_reads_se_bc(p, idx, ref, s1, o1, bcs, quals, bc_len, whitelist=wl, n_threads=2)
    else:
        recs, obc, _ = tro.map_pairs_bc(p, idx, ref, s1, o1, s2, o2, bcs, quals, bc_len, whitelist=wl, n_threads=2, output_not_in_whitelist=out_nw)
    r2, b2 = orc.postprocess_bc(p, recs, obc)
    return ref, r2, b2, bc_len


@pytest.mark.parametrize("case", sorted(GOLDEN_CASES))
def test_oracle_reproduces_reference_translated_bed(sc_setup, case):
    ref, r2, b2, bc_len = _oracle_records(sc_setup, case)
    table = tro.load_translation(gzip.open(os.path.join(GOLD, GOLDEN_CASES[case][0] + ".txt.gz")).read())
    want = gzip.open(os.path.join(GOLD, case + ".bed.gz")).read()
    assert hashlib.md5(want).hexdigest() == _md5s()[case + ".bed"]
    assert tro.format_bed_bc(ref, r2, b2, bc_len, table) == want
    t = cb.parse_barcode_translation(gzip.open(os.path.join(GOLD, GOLDEN_CASES[case][0] + ".txt.gz")).read())
    assert cb.format_bed_bc_tr(ref.names, r2, b2, bc_len, t) == want


def test_oracle_stops_where_the_reference_does(sc_setup):
    ref, r2, b2, bc_len = _oracle_records(sc_setup, "pe_rc16")
    data = gzip.open(os.path.join(GOLD, "missing_rc16.txt.gz")).read()
    with pytest.raises(tro.BarcodeMissing):
        tro.format_bed_bc(ref, r2, b2, bc_len, tro.load_translation(data))
    with pytest.raises(cb.BarcodeNotTranslated):
        cb.format_bed_bc_tr(ref.names, r2, b2, bc_len, cb.parse_barcode_translation(data))


# ---- CLI refusals: parsed before the device is touched
def _cli(*args):
    d = os.path.join(ROOT, "tests", "golden", "ref_test")
    return subprocess.run([CLI, "-x", os.path.join(d, "ref.index"), "-r", os.path.join(d, "ref.fa.gz"), "-1", os.path.join(d, "read1.fq"),
                           "-2", os.path.join(d, "read2.fq"), "-o", "/nonexistent/never.bed"] + list(args), capture_output=True, text=True)


@pytest.mark.parametrize("case", ["empty_file", "empty_line", "crlf", "n_in_from", "lengths_differ", "L32", "line_511", "no_separator"])
def test_cli_refuses_a_malformed_table_without_a_device(tmp_path, case):
    p = tmp_path / "t.txt.gz"
    p.write_bytes(gzip.compress(REFUSED[case]))
    r = _cli("--barcode-translate", str(p))
    assert r.returncode == 255 and "--barcode-translate" in r.stderr and "line " in r.stderr and "GPU path refuses it" in r.stderr, r.stderr


def test_cli_refuses_a_missing_table_file(tmp_path):
    r = _cli("--barcode-translate", str(tmp_path / "absent.txt"))
    assert r.returncode == 255 and "cannot be read" in r.stderr, r.stderr


def test_cli_accepts_a_table_and_reaches_the_device_gate(tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present: the gate is not reached")
    r = _cli("--barcode-translate", os.path.join(GOLD, "rc16.txt.gz"))
    assert r.returncode != 0 and "no CPU fallback" in r.stderr, r.stderr
    h = subprocess.run([CLI, "--help"], capture_output=True, text=True)
    assert "--barcode-translate FILE" in h.stdout
