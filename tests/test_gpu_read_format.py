"""--read-format on the GPU path: the device cut (cmx_ingest_fastq_range) against the host cut (cmx_apply_read_range) on the
synthetic read files, and every case of tests/golden/synth_read_format/ through the CLI with the device reader and with the
host reader, byte-equal to the reference binary's output (make_golden_read_format.sh)."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from tests.test_gpu_parity import _d2h

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
G = os.path.join(ROOT, "tests", "golden")
RF = os.path.join(G, "synth_read_format")


def _records(text):
    lines = text.split(b"\n")
    return [(lines[i + 1], lines[i + 3]) for i in range(0, len(lines) - 3, 4)]


@pytest.mark.parametrize("path,fmt,which", [("synth_read_format/bc24.fq.gz", "bc:8:23", 2), ("synth_read_format/bc_rc.fq.gz", "bc:0:15:-", 2),
                                            ("synth_read_format/bc_split.fq.gz", "bc:0:7,bc:12:19", 2),
                                            ("synth_read_format/r1_bc.fq.gz", "bc:0:15,r1:16:-1", 0),
                                            ("synth_read_format/r1_bc.fq.gz", "bc:0:15,r1:16:-1", 2),
                                            ("synth_read_format/small_read2_rc.fq.gz", "r2:0:-1:-", 1),
                                            ("synth_small/read1.fq.gz", "r1:2:7,r1:10:12,r1:30:-1:-", 0), ("synth_hic/read2.fq.gz", "r2:20:-1", 1)])
def test_ingest_fastq_read_range_equals_the_host_cut(path, fmt, which):
    text = gzip.open(os.path.join(G, path)).read()
    r = cb.parse_read_format(fmt)[which]
    want = [cb.apply_read_range(r, s, q) for s, q in _records(text)]
    m = cb.Mapper(cb.make_params())
    for slot, want_qual in ((which, True), (3 + which, False)):
        g, _ = m.ingest_fastq(slot, text, want_qual=want_qual, read_range=r)
        n = len(want)
        assert g.n_reads == n
        off = _d2h(g.off, 4 * (n + 1)).view(np.uint32)
        assert np.array_equal(np.diff(off), [len(s) for s, _ in want])
        assert _d2h(g.seq, int(off[n])).tobytes() == b"".join(s for s, _ in want)
        if want_qual:
            assert _d2h(g.qual, int(off[n])).tobytes() == b"".join(q for _, q in want)
        assert (g.min_len, g.max_len) == (min(len(s) for s, _ in want), max(len(s) for s, _ in want))
    with pytest.raises(cb.CmxError, match="reads end before a range"):
        m.ingest_fastq(0, text, read_range=cb.parse_read_format("r1:0:%d" % (len(want[0][0]) + 200))[0])
    m.close()


@pytest.fixture(scope="module")
def index(tmp_path_factory):
    d = tmp_path_factory.mktemp("ix")
    out = {}
    for name in ("synth_sc", "synth_small", "synth_hic"):
        out[name] = str(d / (name + ".index"))
        subprocess.check_call([CLI, "-i", "-r", os.path.join(G, name, "ref.fa.gz"), "-o", out[name]], stderr=subprocess.DEVNULL)
    return out


SC = os.path.join(G, "synth_sc")
SMALL = os.path.join(G, "synth_small")
HIC = os.path.join(G, "synth_hic")
_SC_ARGS = ["--preset", "atac", "--barcode-whitelist", os.path.join(SC, "whitelist.txt")]
CASES = {  # name: (index, arguments, expected output)
    "bc24_pe": ("synth_sc", _SC_ARGS + ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", RF + "/bc24.fq.gz", "--read-format", "bc:8:23"],
                SC + "/sc_whitelist.bed.gz"),
    "bc24_se": ("synth_sc", _SC_ARGS + ["-1", SC + "/read1.fq.gz", "-b", RF + "/bc24.fq.gz", "--read-format", "bc:8:23"], SC + "/se_sc_whitelist.bed.gz"),
    "bc_rc": ("synth_sc", _SC_ARGS + ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", RF + "/bc_rc.fq.gz", "--read-format", "bc:0:15:-"],
              SC + "/sc_whitelist.bed.gz"),
    "bc_split": ("synth_sc", _SC_ARGS + ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", RF + "/bc_split.fq.gz", "--read-format", "bc:0:7,bc:12:19"],
                 SC + "/sc_whitelist.bed.gz"),
    "r1_bc": ("synth_sc", _SC_ARGS + ["-1", RF + "/r1_bc.fq.gz", "-2", SC + "/read2.fq.gz", "-b", RF + "/r1_bc.fq.gz", "--read-format", "bc:0:15,r1:16:-1"],
              SC + "/sc_whitelist.bed.gz"),
    "r2_rc": ("synth_small", ["--preset", "chip", "-1", SMALL + "/read1.fq.gz", "-2", RF + "/small_read2_rc.fq.gz", "--read-format", "r2:0:-1:-"],
              SMALL + "/chip.bed.gz"),
    "pe_chip_cut": ("synth_small", ["--preset", "chip", "-1", SMALL + "/read1.fq.gz", "-2", SMALL + "/read2.fq.gz", "--read-format", "r1:0:39,r2:5:-1"],
                    RF + "/pe_chip_r1_0_39_r2_5.bed.gz"),
    "se_cut": ("synth_small", ["-1", SMALL + "/read1.fq.gz", "--read-format", "r1:10:-1"], RF + "/se_r1_10.bed.gz"),
    "sam_rev": ("synth_small", ["--preset", "chip", "--SAM", "-1", SMALL + "/read1.fq.gz", "-2", SMALL + "/read2.fq.gz", "--read-format", "r1:2:46:-,r2:0:44:-"],
                RF + "/pe_chip_rev.sam.gz"),
    "hic_cut": ("synth_hic", ["--preset", "hic", "-1", HIC + "/read1.fq.gz", "-2", HIC + "/read2.fq.gz", "--read-format", "r1:0:99,r2:20:-1"],
                RF + "/hic_r1_0_99_r2_20.pairs.gz"),
}


@pytest.mark.parametrize("reader", ["device", "host"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_cli_read_format_equals_reference_binary_output(case, reader, index, tmp_path):
    name, args, want = CASES[case]
    out = str(tmp_path / "out")
    r = subprocess.run([CLI, "-x", index[name], "-r", os.path.join(G, name, "ref.fa.gz"), "-o", out] + args + (["--host-reader"] if reader == "host" else []),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "using the host reader" not in r.stderr   # the device reader took the files
    assert open(out, "rb").read() == gzip.open(want).read()


@pytest.mark.parametrize("reader", ["device", "host"])
def test_cli_read_format_range_past_the_read_is_refused(reader, index, tmp_path):
    for fmt in ("r1:0:59", "r1:0:9,r2:50:-1"):  # 50-base reads: an end past the read; nothing left after the cut
        r = subprocess.run([CLI, "-x", index["synth_small"], "-r", os.path.join(SMALL, "ref.fa.gz"), "-1", SMALL + "/read1.fq.gz", "-2", SMALL + "/read2.fq.gz",
                            "-o", str(tmp_path / "out.bed"), "--read-format", fmt] + (["--host-reader"] if reader == "host" else []), capture_output=True, text=True)
        assert r.returncode != 0 and "does not fit the reads" in r.stderr, r.stderr
        assert ("reads end before a range" if fmt == "r1:0:59" else "reads are empty after the cut") in r.stderr, r.stderr
