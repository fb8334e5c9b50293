"""Cell barcodes of every length from 1 to 32 and at both ends of the key space on the GPU.  At L = 32 the all-T barcode's key
is ~0, the empty-slot marker of the device's keyed tables; the whitelist answers for it beside its slots (wl_lookup).

- cmx_stage_correct_barcodes equals the oracle's CorrectBarcodeAt on the sets of test_barcode_lengths_host at every L from 1
  to 32 and thresholds 0, 1 and 2.
- cmx_map_batch_pe, paired- and single-end, at every L from 1 to 32 on 3,000 pairs: records and barcode keys equal the
  oracle's; the keys include 0 and ~0 at L = 32.
- At L = 1, 31 and 32 the device's work on those keys equals its host twin: cell-level post-processing and BED text,
  bulk-level duplicate removal, BED text through translation tables of FROM length 1 and 31 (one with an all-T FROM), and SAM
  text with CB:Z: tags.
- `chromap-b200` against the reference binary (oracle/_ref/chromap) run at test time at L = 1, 7, 31 and 32: `--preset atac`
  and `--read-format bc:...` cutting the barcode out of a longer read with the device and the host reader; `--preset chip`
  with a whitelist (bulk level), `--SAM` and `--barcode-translate` once each.  Output files byte for byte, and the read and barcode
  counts.  Inputs come from seeds.

The whole file took 50 s on one H100 80GB HBM3 machine (8 host CPUs), 41 s of it in the CLI runs."""
import os
import re
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests.bc_error2_oracle import correct_barcodes, map_bc
from tests.boundary_inputs import make_reads, reference
from tests.test_barcode_lengths_host import ACGT, ALL_T, cli_barcodes, fastq_q, gate_set, whitelists, write_barcodes, write_inputs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")
N_MAP = 3000
N_CLI = 8000
THREADS = os.cpu_count() or 1


@pytest.fixture(scope="module")
def stage_mapper():
    m = cb.Mapper(cb.make_params("atac", max_read_length=64))
    yield m
    m.close()


@pytest.mark.parametrize("L", range(1, 33))
def test_stage_equals_the_oracle_at_every_length(stage_mapper, tmp_path, L):
    prob = 0.9 if L % 2 == 0 else 0.5
    for c, (name, rows) in enumerate(whitelists(L)):
        sample, obs, quals = gate_set(L, rows, n=1200 if L == 32 else 500, seed=L * 10 + c)
        path = tmp_path / "wl.txt"
        path.write_bytes(b"".join(bytes(r) + b"\n" for r in rows))
        wl = orc.Whitelist(str(path), L)
        wl.sample(sample)
        keys, counts, ns = wl.arrays()
        for thr in (0, 1, 2):
            stage_mapper.upload_barcode_whitelist(keys, counts, ns, L, err_threshold=thr, prob_threshold=prob)
            got = stage_mapper.stage_correct_barcodes(obs.ravel(), quals.ravel(), L)
            want = correct_barcodes(wl, thr, prob, obs.ravel(), quals.ravel(), L)
            bad = np.flatnonzero((got[0] != want[0]) | (got[1] != want[1]))
            assert len(bad) == 0 and tuple(got[2:]) == tuple(want[2:]), (L, name, thr, len(bad), bad[:5], got[2:], want[2:])


@pytest.fixture(scope="module")
def genome(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("bc_len_map"))
    write_inputs(d, n_pairs=1)
    seqs, _ = reference()
    names = ["chr%d" % (i + 1) for i in range(len(seqs))]
    oref = orc.Reference(os.path.join(d, "ref.fa"))
    oidx = orc.Index(ref=oref, k=17, w=7)
    a = oidx.arrays()
    ms = {}
    for kind in ("pe", "se", "sam"):
        m = cb.Mapper(cb.make_params("atac", max_read_length=64, single_end=int(kind == "se"), output_format=4 if kind == "sam" else 1))
        m.upload_reference(seqs, names)
        m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
        ms[kind] = m
    s1, o1, s2, o2 = make_reads(N_MAP, seed=33, length=50)
    yield dict(seqs=seqs, names=names, oref=oref, oidx=oidx, m=ms, pairs=(s1, o1, s2, o2))
    for m in ms.values():
        m.close()


def _barcode_run(g, tmp_path, L, kind):
    """The kind's mapper with the L-base whitelist uploaded, and the device's and the oracle's mapping of the pairs."""
    obs, quals = cli_barcodes(N_MAP, L, 700 + L, str(tmp_path / "wl.txt"))
    wl = orc.Whitelist(str(tmp_path / "wl.txt"), L)
    wl.sample(obs.ravel())
    keys, counts, ns = wl.arrays()
    m = g["m"][kind]
    m.upload_barcode_whitelist(keys, counts, ns, L)
    s1, o1, s2, o2 = g["pairs"]
    se = kind == "se"
    recs, st = m.map_batch(s1, o1, None if se else s2, None if se else o2, barcodes=obs.ravel(), barcode_quals=quals.ravel(), bc_len=L)
    return m, wl, obs, quals, recs, st


@pytest.mark.parametrize("se", [0, 1], ids=["pe", "se"])
@pytest.mark.parametrize("L", range(1, 33))
def test_map_batch_keys_equal_the_oracle_at_every_length(genome, tmp_path, L, se):
    m, wl, obs, quals, recs, st = _barcode_run(genome, tmp_path, L, "se" if se else "pe")
    s1, o1, s2, o2 = genome["pairs"]
    p = orc.make_params("atac", single_end=se)
    orecs, obc, ost = map_bc(p, genome["oidx"], genome["oref"], s1, o1, None if se else s2, None if se else o2, obs.ravel(), quals.ravel(), L, wl, 1, 0.9,
                             n_threads=THREADS)
    assert len(recs) == len(orecs) > N_MAP // 2
    for f in recs.dtype.names:
        assert np.array_equal(recs[f], orecs[f]), (L, f)
    assert np.array_equal(st["barcode_keys"], obc), L
    assert (st["n_barcodes_in_whitelist"], st["n_barcodes_corrected"]) == (int(ost[0]), int(ost[1]))
    if L == 32:
        assert np.sum(obc == ALL_T) > 100 and np.sum(obc == 0) > 100


def _same_records(a, b):
    assert len(a) == len(b)
    for f in a.dtype.names:
        assert np.array_equal(a[f], b[f]), f


def _translation(from_len, bcs):
    """A table with every FROM of from_len bases that the keys bcs need, the all-A and the all-T one: FROM key -> cell_<key>."""
    keys = np.union1d(np.unique(bcs & np.uint64((1 << 2 * from_len) - 1)), np.array([0, (1 << 2 * from_len) - 1], dtype=np.uint64))
    return cb.BarcodeTranslation(keys, [b"cell_%d" % int(k) for k in keys], from_len)


@pytest.mark.parametrize("L", [1, 31, 32])
def test_device_work_on_the_keys_equals_the_host_twins(genome, tmp_path, L):
    m, wl, obs, quals, recs, st = _barcode_run(genome, tmp_path, L, "pe")
    bcs = st["barcode_keys"]
    # cell level: post-processing and BED text against the oracle
    p = orc.make_params("atac")
    r2, b2 = m.postprocess_gpu(recs, bcs)
    o2, ob2 = orc.postprocess_bc(p, recs, bcs)
    _same_records(r2, o2)
    assert np.array_equal(b2, ob2)
    bed = m.format_bed_gpu(r2, b2, L)
    assert bed == orc.format_bed_bc(genome["oref"], o2, ob2, L)
    # bulk level: the whitelist's abundances rank the barcodes of a group
    keys, counts, ns = wl.arrays()
    mb = cb.Mapper(cb.make_params("chip"))
    try:
        mb.upload_reference(genome["seqs"], genome["names"])
        mb.upload_barcode_whitelist(keys, counts, ns, L)
        got = mb.postprocess_bc_bulk_gpu(recs, bcs)
        want = cb.postprocess_bc_bulk(cb.make_params("chip"), keys, counts, recs, bcs)
        _same_records(got[0], want[0])
        assert np.array_equal(got[1], want[1]) and (L != 32 or np.sum(want[1] == ALL_T) > 10)
    finally:
        mb.close()
    # translation tables: FROM of one base, and of 31 at L = 32 (the leading base plays no part)
    for from_len in ([1] + ([31] if L == 32 else [])):
        t = _translation(from_len, b2)
        m.upload_barcode_translation(t)
        try:
            assert m.format_bed_gpu(r2, b2, L) == cb.format_bed_bc_tr(genome["names"], r2, b2, L, t)
        finally:
            m.upload_barcode_translation(None)
    # SAM text with CB:Z: tags
    ms, _, _, _, cores, sst = _barcode_run(genome, tmp_path, L, "sam")
    s1, o1, s2, o2 = genome["pairs"]
    names = [b"r%08d" % i for i in range(N_MAP)]
    def reads(s, o):
        return names, [s[o[i]:o[i + 1]].tobytes() for i in range(N_MAP)], [b"I" * int(o[i + 1] - o[i]) for i in range(N_MAP)]
    r1, rr2 = reads(s1, o1), reads(s2, o2)
    got = ms.format_sam_gpu(cores, r1, rr2, sst["barcode_keys"], L)
    assert got == cb.format_sam_bc(ms.params, genome["names"], genome["seqs"], cores, sst["barcode_keys"], L, r1, rr2)
    assert got.count(b"\tCB:Z:") > N_MAP // 2
    if L == 32:
        assert b"\tCB:Z:" + b"T" * 32 + b"\n" in got or b"\tCB:Z:" + b"T" * 32 + b"\t" in got


# ---- chromap-b200 against the reference binary ------------------------------------------------------------------------
COUNT_LINES = re.compile(r"^Number of (reads|barcodes in whitelist|corrected barcodes): \d+\.$", re.M)


CLI_LENGTHS = (1, 7, 31, 32)


@pytest.fixture(scope="module")
def cli_data(tmp_path_factory):
    """The inputs of every length's runs, and the reference binary's output of each as a future: the reference binary spends
    most of a run in its single-threaded sort and output, so its runs go to a pool of one process per CPU and overlap the
    chromap-b200 runs, which wait only for the output they compare with."""
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    d = str(tmp_path_factory.mktemp("bc_len_cli"))
    write_inputs(d, n_pairs=N_CLI)
    subprocess.check_call([CLI, "-i", "-r", os.path.join(d, "ref.fa"), "-o", os.path.join(d, "ref.index")], stderr=subprocess.DEVNULL)
    common = ["-x", os.path.join(d, "ref.index"), "-r", os.path.join(d, "ref.fa")]
    runs = {L: _runs(d, L) for L in CLI_LENGTHS}

    def reference_run(L, name, args, ext):
        out = os.path.join(d, "want_%d_%s.%s" % (L, name, ext))
        r = subprocess.run([REF_BIN] + args + common + ["-t", "1", "-o", out], capture_output=True, text=True)
        return r, out

    with ThreadPoolExecutor(max_workers=THREADS) as pool:
        want = {(L, name): pool.submit(reference_run, L, name, args, ext) for L in CLI_LENGTHS for name, args, ext, _ in runs[L]}
        yield dict(d=d, common=common, runs=runs, want=want)
        for f in want.values():
            f.cancel()


def _runs(d, L):
    """(name, arguments, output extension, readers) of the runs at barcode length L; writes their inputs.  The runs that cut
    barcodes out of their records (atac, read_format) go through the device and the host reader; --SAM always reads on the
    host, and the others take the device reader."""
    bc, wl = write_barcodes(d, L, n_pairs=N_CLI)
    pe = ["-1", os.path.join(d, "r1.fq"), "-2", os.path.join(d, "r2.fq")]
    both = ([], ["--host-reader"])
    runs = [("atac", ["--preset", "atac"] + pe + ["-b", bc, "--barcode-whitelist", wl], "bed", both),
            ("chip_bulk", ["--preset", "chip"] + pe + ["-b", bc, "--barcode-whitelist", wl], "bed", ([],)),
            ("sam", ["--SAM", "--preset", "atac"] + pe + ["-b", bc, "--barcode-whitelist", wl], "sam", ([],))]
    if L >= 2:  # FROM = the last L - 1 bases: the leading base plays no part; the all-T FROM is listed
        tr = os.path.join(d, "tr%d.txt" % L)
        froms = sorted({l[1:] for l in open(wl).read().split()} | {"T" * (L - 1), "A" * (L - 1)})  # every listed barcode's
        with open(tr, "w") as f:
            f.write("".join("cell%d,%s\n" % (i, x) for i, x in enumerate(froms)))
        runs.append(("translate", ["--preset", "atac"] + pe + ["-b", bc, "--barcode-whitelist", wl, "--barcode-translate", tr], "bed", ([],)))
    if L == 32:  # the barcode cut out of a 40-base read
        obs, quals = cli_barcodes(N_CLI, 32, 500 + 32, os.path.join(d, "scratch_wl.txt"))
        rng = np.random.default_rng(40)
        pad = ACGT[rng.integers(0, 4, (len(obs), 8))]
        long_bc = os.path.join(d, "bc40.fq")
        with open(long_bc, "wb") as f:
            f.write(fastq_q(np.concatenate([pad[:, :5], obs, pad[:, 5:]], axis=1), np.concatenate([np.full((len(obs), 5), 73, np.uint8), quals,
                                                                                                    np.full((len(obs), 3), 73, np.uint8)], axis=1), prefix=b"b"))
        runs.append(("read_format", ["--preset", "atac"] + pe + ["-b", long_bc, "--barcode-whitelist", wl, "--read-format", "bc:5:36"], "bed", both))
    return runs


@pytest.mark.parametrize("L", CLI_LENGTHS)
def test_cli_equals_the_reference_binary_at_barcode_lengths(cli_data, L):
    d = cli_data["d"]
    for name, args, ext, readers in cli_data["runs"][L]:
        r, want_path = cli_data["want"][(L, name)].result()
        assert r.returncode == 0, (name, r.stderr[-2000:])
        want = open(want_path, "rb").read()
        want_counts = sorted(m.group(0) for m in COUNT_LINES.finditer(r.stderr))
        assert len(want) > 0 and any("barcodes in whitelist" in c for c in want_counts), (name, want_counts)
        for reader in readers:
            got_path = os.path.join(d, "got." + ext)
            g = subprocess.run([CLI] + args + cli_data["common"] + reader + ["-o", got_path], capture_output=True, text=True)
            assert g.returncode == 0, (name, reader, g.stderr[-2000:])
            got = open(got_path, "rb").read()
            assert got == want, (L, name, reader, len(got), len(want))
            assert sorted(m.group(0) for m in COUNT_LINES.finditer(g.stderr)) == want_counts, (L, name, reader)
            os.remove(got_path)
        os.remove(want_path)
