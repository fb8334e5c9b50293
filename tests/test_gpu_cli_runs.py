"""`chromap-b200` on runs of several library calls, against the reference binary (oracle/_ref/chromap) run at test time.

The device reader maps up to 4 x 500,000 pairs per library call and ingests the next call into the other parity's slots
while the current one is mapped; the host reader (`--SAM`, `--host-reader`) makes one call per 500,000 pairs.  The CLI sets
every call's `first_read_id` from the calls before it and gathers the records, barcode keys, SAM offsets and names across
calls; the barcode pre-pass checks its whitelist share once per 500,000 barcodes.  One seeded set of 2,200,000 pairs of
2x50 bp (two device-reader calls, five host-reader calls) on a 4.5 Mbp reference with planted repeats
(tests/boundary_inputs.py), plain and gzip, with cell barcodes against a whitelist; its first 1,100,000 pairs for `--SAM`
(three calls) and 600,000 pairs of 2x150 bp for `--preset hic --host-reader` (two calls).  Every output file is compared
byte for byte with the reference binary's, and so are the read, mapped-read and uniquely-mapped-read counts (and the
barcode counts of the barcoded run).

The reference binary's time per run on one H100 80GB HBM3 machine's host (8 CPUs, `-t 8`): `--preset chip` 58.8 s, `-n 3 -q 0`
26.0 s, barcoded atac 39.9 s, single-end chip 19.4 s, `--SAM` (1.1 M pairs) 51.8 s, Hi-C (600,000 pairs) 22.8 s.  The whole
file, inputs and the 13 `chromap-b200` runs included, takes 290 s there."""
import gzip
import os
import re
import subprocess
import time

import pytest

from tests.boundary_inputs import fastq, make_barcodes, make_reads, reference

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "chromap")
N_PAIRS, N_SAM, N_HIC = 2_200_000, 1_100_000, 600_000
THREADS = str(os.cpu_count() or 1)
COUNT_LINES = re.compile(r"^Number of (reads|mapped reads|uniquely mapped reads|barcodes in whitelist|corrected barcodes): \d+\.$", re.M)


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    if not os.path.exists(REF_BIN):
        pytest.skip("oracle/_ref/chromap not built")
    if not os.path.exists(CLI):
        import __graft_entry__
        __graft_entry__.build()
    d = tmp_path_factory.mktemp("cli_runs")
    seqs, _ = reference()
    ref = str(d / "ref.fa")
    with open(ref, "wb") as f:
        for i, a in enumerate(seqs):
            f.write(b">chr%d\n" % (i + 1) + a.tobytes() + b"\n")
    idx = str(d / "ref.index")
    subprocess.check_call([CLI, "-i", "-r", ref, "-o", idx], stderr=subprocess.DEVNULL)
    files = dict(d=d, ref=ref, idx=idx)
    s1, _, s2, _ = make_reads(N_PAIRS, seed=22, length=50)
    for mate, s in (("1", s1), ("2", s2)):
        text = fastq(s, 50)
        files["r" + mate] = str(d / ("r%s.fq" % mate))
        open(files["r" + mate], "wb").write(text)
        files["r%s_gz" % mate] = str(d / ("r%s.fq.gz" % mate))
        with gzip.open(files["r%s_gz" % mate], "wb", compresslevel=1) as f:
            f.write(text)
        files["sam_r" + mate] = str(d / ("sam_r%s.fq" % mate))
        open(files["sam_r" + mate], "wb").write(text[:N_SAM * (len(text) // N_PAIRS)])
    bcs, _, bl = make_barcodes(N_PAIRS, 23, str(d / "wl.txt"))
    files["wl"] = str(d / "wl.txt")
    files["bc"] = str(d / "bc.fq")
    open(files["bc"], "wb").write(fastq(bcs, bl))
    h1, _, h2, _ = make_reads(N_HIC, seed=24, hic=True, length=150)
    for mate, s in (("1", h1), ("2", h2)):
        files["hic_r" + mate] = str(d / ("hic_r%s.fq" % mate))
        open(files["hic_r" + mate], "wb").write(fastq(s, 150))
    return files


def _run(binary, args, data, out, env=None):
    cmd = [binary] + args + ["-x", data["idx"], "-r", data["ref"], "-o", out]
    if binary == REF_BIN:
        cmd += ["-t", THREADS]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, (binary, args, r.stderr[-2000:])
    return r.stderr


def _counts(stderr):
    """The last line of every count kind the run printed."""
    return {m.group(1): m.group(0) for m in COUNT_LINES.finditer(stderr)}


def _first_diff(a, b):
    i = next((k for k in range(min(len(a), len(b))) if a[k] != b[k]), min(len(a), len(b)))
    lo = a.rfind(b"\n", 0, i) + 1
    return a[lo:lo + 200], b[lo:lo + 200]


def _check(data, ref_args, runs, ext="bed"):
    """The reference binary once on ref_args, then chromap-b200 on each (args, env): the same output file, the same counts."""
    want_path = str(data["d"] / ("want." + ext))
    t = time.time()
    want_err = _run(REF_BIN, ref_args, data, want_path)
    print("reference binary %s: %.1f s on %s threads" % (" ".join(a for a in ref_args if not a.startswith("/")), time.time() - t, THREADS))
    want = open(want_path, "rb").read()
    want_counts = _counts(want_err)
    assert len(want) > 0 and "reads" in want_counts and "mapped reads" in want_counts, want_err[-2000:]
    for args, env in runs:
        out = str(data["d"] / ("got." + ext))
        err = _run(CLI, args, data, out, env)
        got = open(out, "rb").read()
        assert got == want, (args, env, len(got), len(want), _first_diff(got, want))
        assert _counts(err) == want_counts, (args, env, _counts(err), want_counts)
        os.remove(out)
    os.remove(want_path)


def _pe(data, gz=False):
    s = "_gz" if gz else ""
    return ["-1", data["r1" + s], "-2", data["r2" + s]]


@pytest.mark.parametrize("knobs", [["--preset", "chip"], ["-n", "3", "-q", "0"]], ids=["chip", "n3q0"])
def test_paired_end_runs_of_several_calls(data, knobs):
    """Device reader (two calls; plain and gzip; one lane and the default) and host reader (five calls)."""
    _check(data, knobs + _pe(data), [(knobs + _pe(data), None), (knobs + _pe(data, gz=True), None), (knobs + _pe(data) + ["--host-reader"], None),
                                     (knobs + _pe(data), {"CMX_LANES": "1"})])


def test_barcoded_run_of_several_calls(data):
    """`--preset atac -b --barcode-whitelist`: the barcode pre-pass over 2.2 M barcodes, keys gathered across calls, and the
    whitelist and correction counts."""
    args = ["--preset", "atac"] + _pe(data) + ["-b", data["bc"], "--barcode-whitelist", data["wl"]]
    _check(data, args, [(args, None), (args + ["--host-reader"], None)])


def test_single_end_run_of_several_calls(data):
    args = ["--preset", "chip", "-1", data["r1"]]
    _check(data, args, [(args, None)])


def test_sam_run_of_several_host_reader_calls(data):
    """--SAM reads on the host: three calls, read names and SAM offsets gathered across them."""
    args = ["--SAM", "--preset", "chip", "-1", data["sam_r1"], "-2", data["sam_r2"]]
    _check(data, args, [(args, None)], ext="sam")


def test_hic_run_of_several_host_reader_calls(data):
    args = ["--preset", "hic", "-1", data["hic_r1"], "-2", data["hic_r2"]]
    _check(data, args, [(args + ["--host-reader"], None)], ext="pairs")
