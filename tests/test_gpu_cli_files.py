"""`chromap-b200` with several read files per option (`-1 a,b,c`, `-1 'lane*_R1.fq'`), against the reference binary
(oracle/_ref/chromap) run at test time on the same files.

Each file starts new reference batches of 500,000 pairs, and the choice among equally good multi-mappings depends on a pair's
place in its batch, so a run on split files is not a run on their concatenation; the chip case checks that the reference's
outputs on the two differ.  The files are cut out of one seeded set of 2x50 bp pairs on a 4.5 Mbp reference with planted
repeats (tests/boundary_inputs.py): a file that ends mid-batch, an empty file, a one-pair file, a file of exactly 2,000,000
pairs (one whole device-reader call, four whole batches) and a short tail, plain and gzip mixed.  The other output formats
run on a 200,000-pair split of the same kind, and one run has a FASTA read-1 file among the FASTQ files (that file set goes
through the host reader, the next ones through the device reader again).  Output files are compared byte for byte, and so
are the read, mapped-read and uniquely-mapped-read counts (and the barcode counts of the barcoded run).  Both binaries must
also refuse files whose read or barcode counts differ per file with equal totals, and a first barcode file too small to pass
the 5 % whitelist check on its own."""
import gzip
import os
import subprocess
import time

import numpy as np
import pytest

from tests.boundary_inputs import fastq, make_barcodes, make_reads, reference
from tests.test_gpu_cli_runs import _counts, _first_diff

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")
THREADS = str(os.cpu_count() or 1)
# pairs per file, and which files are gzipped
CHIP_SPLIT, CHIP_GZ = (300_001, 0, 1, 2_000_000, 99_998), (False, False, True, False, True)
SMALL_SPLIT, SMALL_GZ = (120_001, 0, 1, 79_998), (False, True, True, False)
N_HIC = 150_000


def _write(path, data, gz):
    if gz:
        with gzip.open(path, "wb", compresslevel=1) as f:
            f.write(data)
    else:
        with open(path, "wb") as f:
            f.write(data)
    return path


def _split(d, name, text, n, sizes, gzs):
    """Files name_1.fq, name_2.fq.gz, ... holding consecutive records of `text` (n records of equal length), `sizes[i]` each."""
    rec = len(text) // n
    paths, start = [], 0
    for i, (size, gz) in enumerate(zip(sizes, gzs)):
        paths.append(_write(str(d / ("%s_%d.fq%s" % (name, i + 1, ".gz" if gz else ""))), text[start * rec:(start + size) * rec], gz))
        start += size
    return paths


def _fasta(text):
    """The records of 4-line FASTQ text as 2-line FASTA."""
    lines = text.split(b"\n")
    return b"".join(b">" + lines[i][1:] + b"\n" + lines[i + 1] + b"\n" for i in range(0, len(lines) - 3, 4))


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    if not os.path.exists(CLI):
        import __graft_entry__
        __graft_entry__.build()
    d = tmp_path_factory.mktemp("cli_files")
    seqs, _ = reference()
    ref = str(d / "ref.fa")
    with open(ref, "wb") as f:
        for i, a in enumerate(seqs):
            f.write(b">chr%d\n" % (i + 1) + a.tobytes() + b"\n")
    idx = str(d / "ref.index")
    subprocess.check_call([CLI, "-i", "-r", ref, "-o", idx], stderr=subprocess.DEVNULL)
    files = dict(d=d, ref=ref, idx=idx)
    n = sum(CHIP_SPLIT)
    s1, _, s2, _ = make_reads(n, seed=31, length=50)
    for mate, s in (("1", s1), ("2", s2)):
        text = fastq(s, 50)
        files["chip" + mate] = _split(d, "chip_R" + mate, text, n, CHIP_SPLIT, CHIP_GZ)
        files["concat" + mate] = _write(str(d / ("concat_R%s.fq" % mate)), text, False)
        small = text[:sum(SMALL_SPLIT) * (len(text) // n)]
        files["small" + mate] = _split(d, "small_R" + mate, small, sum(SMALL_SPLIT), SMALL_SPLIT, SMALL_GZ)
        files["tiny" + mate] = small[:1040 * (len(text) // n)]
    files["fasta1"] = [_write(str(d / "small_R1_1.fa"), _fasta(open(files["small1"][0], "rb").read()), False)] + files["small1"][1:]
    bcs, _, bl = make_barcodes(sum(SMALL_SPLIT), 33, str(d / "wl.txt"))
    files["wl"] = str(d / "wl.txt")
    files["bc"] = _split(d, "small_I1", fastq(bcs, bl), sum(SMALL_SPLIT), SMALL_SPLIT, SMALL_GZ)
    files["tiny_bc"] = fastq(bcs[:1040 * bl], bl)
    h1, _, h2, _ = make_reads(N_HIC, seed=32, hic=True, length=150)
    hic_split = (100_001, 0, 1, N_HIC - 100_002)
    for mate, s in (("1", h1), ("2", h2)):
        files["hic" + mate] = _split(d, "hic_R" + mate, fastq(s, 150), N_HIC, hic_split, (False, False, True, True))
    return files


def _run(binary, args, data, out, env=None, ok=True):
    cmd = [binary] + args + ["-x", data["idx"], "-r", data["ref"], "-o", out]
    if binary == REF_BIN:
        cmd += ["-t", THREADS]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    if ok:
        assert r.returncode == 0, (binary, args, r.stderr[-2000:])
    return r


def _check(data, ref_args, runs, ext="bed"):
    """The reference binary once on ref_args, then chromap-b200 on each (args, env): the same output file, the same counts.
    Returns the reference's output."""
    want_path = str(data["d"] / ("want." + ext))
    t = time.time()
    want_err = _run(REF_BIN, ref_args, data, want_path).stderr
    print("reference binary %s: %.1f s on %s threads" % (" ".join(a for a in ref_args if not a.startswith("/")), time.time() - t, THREADS))
    want = open(want_path, "rb").read()
    want_counts = _counts(want_err)
    assert len(want) > 0 and "reads" in want_counts and "mapped reads" in want_counts, want_err[-2000:]
    for args, env in runs:
        out = str(data["d"] / ("got." + ext))
        err = _run(CLI, args, data, out, env).stderr
        got = open(out, "rb").read()
        assert got == want, (args, env, len(got), len(want), _first_diff(got, want))
        assert _counts(err) == want_counts, (args, env, _counts(err), want_counts)
        os.remove(out)
    os.remove(want_path)
    return want


def _pe(r1, r2):
    return ["-1", ",".join(r1), "-2", ",".join(r2)]


def test_chip_paired_end_over_split_files(data):
    """Device reader (default lanes and one lane), host reader, and the same files as quoted glob patterns.  `-q 0` keeps
    the multi-mapped pairs (the preset's MAPQ 30 drops them), so the reference's output on the concatenated files is not
    its output on the split files: the test moves batch boundaries."""
    knobs = ["--preset", "chip", "-q", "0"]
    args = knobs + _pe(data["chip1"], data["chip2"])
    d = str(data["d"])
    glob = knobs + ["-1", os.path.join(d, "chip_R1_*"), "-2", os.path.join(d, "chip_R2_*")]
    want = _check(data, args, [(args, None), (args, {"CMX_LANES": "1"}), (args + ["--host-reader"], None), (glob, None)])
    concat = str(data["d"] / "concat.bed")
    _run(REF_BIN, knobs + ["-1", data["concat1"], "-2", data["concat2"]], data, concat)
    assert open(concat, "rb").read() != want
    os.remove(concat)


def test_barcoded_atac_over_split_files(data):
    """The barcode files split like the reads: the pre-pass batches per file, the whitelist and correction counts are totals."""
    args = ["--preset", "atac"] + _pe(data["small1"], data["small2"]) + ["-b", ",".join(data["bc"]), "--barcode-whitelist", data["wl"]]
    _check(data, args, [(args, None), (args + ["--host-reader"], None)])


def test_single_end_chip_over_split_files(data):
    args = ["--preset", "chip", "-1", ",".join(data["small1"])]
    _check(data, args, [(args, None)])


def test_sam_over_split_files(data):
    args = ["--SAM", "--preset", "chip"] + _pe(data["small1"], data["small2"])
    _check(data, args, [(args, None)], ext="sam")


def test_hic_pairs_over_split_files(data):
    args = ["--preset", "hic"] + _pe(data["hic1"], data["hic2"])
    _check(data, args, [(args, None), (args + ["--host-reader"], None)], ext="pairs")


def test_fasta_file_among_fastq_files(data):
    """Read 1 of the first set is FASTA: that set goes through the host reader, the later sets through the device reader."""
    args = ["--preset", "chip"] + _pe(data["fasta1"], data["small2"])
    _check(data, args, [(args, None)])
    r = _run(CLI, args, data, str(data["d"] / "fasta.bed"))
    assert r.stderr.count("using the host reader") == 1, r.stderr[-2000:]


def test_per_file_count_mismatch_is_refused(data):
    """Read 1 and read 2 (or barcode) files with the same totals but not the same counts per file end both runs."""
    d = data["d"]
    rec = len(data["tiny1"]) // 1040
    r1 = [_write(str(d / "mm_R1_1.fq"), data["tiny1"][:500 * rec], False), _write(str(d / "mm_R1_2.fq"), data["tiny1"][500 * rec:1000 * rec], False)]
    r2 = [_write(str(d / "mm_R2_1.fq"), data["tiny2"][:501 * rec], False), _write(str(d / "mm_R2_2.fq"), data["tiny2"][501 * rec:1000 * rec], False)]
    r2_even = [_write(str(d / "mm_R2_3.fq"), data["tiny2"][:500 * rec], False), _write(str(d / "mm_R2_4.fq"), data["tiny2"][500 * rec:1000 * rec], False)]
    brec = len(data["tiny_bc"]) // 1040
    bc = [_write(str(d / "mm_I1_1.fq"), data["tiny_bc"][:499 * brec], False), _write(str(d / "mm_I1_2.fq"), data["tiny_bc"][499 * brec:1000 * brec], False)]
    for args in (["--preset", "chip"] + _pe(r1, r2), ["--preset", "atac"] + _pe(r1, r2_even) + ["-b", ",".join(bc)]):
        for binary in (REF_BIN, CLI):
            r = _run(binary, args, data, str(d / "mm.bed"), ok=False)
            assert r.returncode != 0 and "Numbers of reads and barcodes don't match!" in r.stderr, (binary, args, r.stderr[-2000:])


def test_tiny_first_barcode_file_fails_the_whitelist_check(data):
    """The 5 % check compares the running whitelisted count with the batch just read: a first file of 40 barcodes, one in
    the whitelist, ends the run; the same barcodes in one file pass."""
    d = data["d"]
    rec, brec = len(data["tiny1"]) // 1040, len(data["tiny_bc"]) // 1040
    wl_first = open(data["wl"], "rb").readline().strip()
    rng = np.random.default_rng(34)
    head = bytearray(data["tiny_bc"][:40 * brec])
    for i in range(40):  # random barcodes (a 16-mer outside a 3,000-entry whitelist), the first one from it
        start = head.index(b"\n", i * brec) + 1  # the bases follow the name line
        head[start:start + 16] = wl_first if i == 0 else bytes(np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 16)])
    bc_text = bytes(head) + data["tiny_bc"][40 * brec:]
    split = ["-1", ",".join([_write(str(d / "wl_R1_1.fq"), data["tiny1"][:40 * rec], False), _write(str(d / "wl_R1_2.fq"), data["tiny1"][40 * rec:], False)]),
             "-2", ",".join([_write(str(d / "wl_R2_1.fq"), data["tiny2"][:40 * rec], False), _write(str(d / "wl_R2_2.fq"), data["tiny2"][40 * rec:], False)]),
             "-b", ",".join([_write(str(d / "wl_I1_1.fq"), bc_text[:40 * brec], False), _write(str(d / "wl_I1_2.fq"), bc_text[40 * brec:], False)])]
    whole = ["-1", _write(str(d / "wl_R1.fq"), data["tiny1"], False), "-2", _write(str(d / "wl_R2.fq"), data["tiny2"], False),
             "-b", _write(str(d / "wl_I1.fq"), bc_text, False)]
    for binary in (REF_BIN, CLI):
        r = _run(binary, ["--preset", "atac", "--barcode-whitelist", data["wl"]] + split, data, str(d / "wl.bed"), ok=False)
        assert r.returncode != 0 and "Less than 5% barcodes can be found or corrected" in r.stderr, (binary, r.stderr[-2000:])
        _run(binary, ["--preset", "atac", "--barcode-whitelist", data["wl"]] + whole, data, str(d / "wl.bed"))
