"""--SAM with cell barcodes on the GPU path: cmx_map_batch_pe's SAM cores and barcode keys against the oracle's (every whitelist
mode, paired-end and single-end, --bc-error-threshold 2); cmx_format_sam_gpu against its host twin cmx_format_sam_bc, bulk and
barcoded, with and without a translation table, across the 1 M-line text chunk; and every file of tests/golden/synth_sam_bc
through chromap-b200, byte-equal to the reference binary's output (make_golden_sam_bc.sh)."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests import sam_bc_oracle as sbo
from tests.sam_bc_device import device_cores as _device_cores, reads as _reads

pytestmark = pytest.mark.gpu

ROOT = sbo.ROOT
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
SC = sbo.SC


def _oracle_cores(name):
    ref, index, r1, r2 = sbo.setup()
    keys, ok, bc_len = sbo.barcode_gate(name)
    return sbo.cores_and_keys(sbo.params(name), index, ref, r1, None if sbo.RUNS[name][2] else r2, keys, ok)


@pytest.mark.parametrize("name", ["pe_atac", "se_atac", "pe_nowl", "pe_notinwl", "pe_n3q0", "pe_bcerr2", "se_q0dedup"])
def test_map_batch_sam_cores_and_keys_equal_the_oracle(name):
    m, _, cores, keys, _ = _device_cores(name)
    want, wkeys = _oracle_cores(name)
    m.close()
    assert len(cores) == len(want) > 1000
    for f in want.dtype.names:
        assert np.array_equal(cores[f], want[f]), f
    assert np.array_equal(keys, wkeys)


@pytest.mark.parametrize("name", sorted(sbo.RUNS))
def test_format_sam_gpu_equals_host_twin_and_golden(name):
    m, seqs, cores, keys, bc_len = _device_cores(name)
    _, _, r1, r2 = sbo.setup()
    se = sbo.RUNS[name][2]
    reads1, reads2 = _reads(r1), None if se else _reads(r2)
    tr_path = sbo.RUNS[name][7]
    t = cb.parse_barcode_translation(gzip.open(tr_path).read()) if tr_path else None
    m.upload_barcode_translation(t)
    got = m.format_sam_gpu(cores, reads1, reads2, keys, bc_len)
    host = cb.format_sam_bc(m.params, m.names, seqs, cores, keys, bc_len, reads1, reads2, translation=t)
    m.close()
    assert got == host
    assert got == gzip.open(os.path.join(sbo.OUT, name + ".sam.gz")).read()


def test_format_sam_gpu_bulk_and_untranslated_and_chunks():
    """Bulk and untranslated barcoded text, and a call of more than one 1 M-line chunk (cores replicated with new read ids)."""
    m, seqs, cores, keys, bc_len = _device_cores("pe_q0dedup")
    _, _, r1, r2 = sbo.setup()
    reads1, reads2 = _reads(r1), _reads(r2)
    for bcs in (None, keys):
        assert m.format_sam_gpu(cores, reads1, reads2, bcs, bc_len) == cb.format_sam_bc(m.params, m.names, seqs, cores, bcs, bc_len, reads1, reads2)
    n_reads = len(r1)
    reps = 1 + (1 << 20) // (2 * len(cores)) + 1
    big = np.concatenate([cores] * reps)
    big["read_id"] += np.repeat(np.arange(reps, dtype=np.uint32) * n_reads, len(cores))
    bk = np.concatenate([keys] * reps)
    bk ^= np.repeat(np.arange(reps, dtype=np.uint64), len(cores))  # other cells
    rr1 = tuple(x * reps for x in reads1)
    rr2 = tuple(x * reps for x in reads2)
    assert 2 * len(big) > (1 << 20)
    got = m.format_sam_gpu(big, rr1, rr2, bk, bc_len)
    want = cb.format_sam_bc(m.params, m.names, seqs, big, bk, bc_len, rr1, rr2)
    m.close()
    assert got.count(b"\n") > (1 << 20)
    assert got == want


def test_format_sam_gpu_missing_segment():
    m, seqs, cores, keys, bc_len = _device_cores("pe_atac")
    _, _, r1, r2 = sbo.setup()
    t = cb.parse_barcode_translation(gzip.open(os.path.join(sbo.TR, "missing_rc16.txt.gz")).read())
    m.upload_barcode_translation(t)
    with pytest.raises(cb.BarcodeNotTranslated):
        m.format_sam_gpu(cores, _reads(r1), _reads(r2), keys, bc_len)
    with pytest.raises(cb.BarcodeNotTranslated):
        cb.format_sam_bc(m.params, m.names, seqs, cores, keys, bc_len, _reads(r1), _reads(r2), translation=t)
    m.close()


@pytest.fixture(scope="module")
def index(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ix") / "sc.index")
    subprocess.check_call([CLI, "-i", "-r", os.path.join(SC, "ref.fa.gz"), "-o", out], stderr=subprocess.DEVNULL)
    return out


_WL = ["--barcode-whitelist", sbo.WL]
_PE = ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", SC + "/barcode.fq.gz"]
_SE = ["-1", SC + "/read1.fq.gz", "-b", SC + "/barcode.fq.gz"]
_ATAC = ["--preset", "atac"]
_BE = sbo.BE
CASES = {
    "pe_atac": _ATAC + _WL + _PE,
    "se_atac": _ATAC + _WL + _SE,
    "pe_q0dedup": ["-q", "0", "--remove-pcr-duplicates"] + _WL + _PE,
    "se_q0dedup": ["-q", "0", "--remove-pcr-duplicates"] + _WL + _SE,
    "pe_nowl": _ATAC + _PE,
    "pe_notinwl": _ATAC + _WL + ["--output-mappings-not-in-whitelist"] + _PE,
    "pe_n3q0": ["-n", "3", "-q", "0"] + _WL + _PE,
    "pe_bcerr2": _ATAC + ["--bc-error-threshold", "2", "--barcode-whitelist", _BE + "/dense.txt.gz", "-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz",
                          "-b", _BE + "/barcode.fq.gz"],
    "pe_rc16": _ATAC + _WL + _PE + ["--barcode-translate", sbo.TR + "/rc16.txt.gz"],
    "pe_half8": _ATAC + _WL + _PE + ["--barcode-translate", sbo.TR + "/half8.txt.gz"],
}


def _run(index, args, out):
    return subprocess.run([CLI, "--SAM", "-x", index, "-r", os.path.join(SC, "ref.fa.gz"), "-o", out] + args, capture_output=True, text=True)


@pytest.mark.parametrize("case", sorted(CASES))
def test_cli_sam_bc_equals_reference_binary_output(case, index, tmp_path):
    out = str(tmp_path / "out.sam")
    r = _run(index, CASES[case], out)
    assert r.returncode == 0, r.stderr
    assert "Number of barcodes in whitelist" in r.stderr
    assert open(out, "rb").read() == gzip.open(os.path.join(sbo.OUT, case + ".sam.gz")).read()


def test_cli_sam_bc_read_format_identity(index, tmp_path):
    out = str(tmp_path / "out.sam")
    r = _run(index, _ATAC + _WL + ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", sbo.GOLDEN + "/synth_read_format/bc24.fq.gz",
                                   "--read-format", "bc:8:23"], out)
    assert r.returncode == 0, r.stderr
    assert open(out, "rb").read() == gzip.open(os.path.join(sbo.OUT, "pe_atac.sam.gz")).read()


def test_cli_sam_missing_barcode_exits_255_and_writes_nothing(index, tmp_path):
    out = tmp_path / "out.sam"
    r = _run(index, _ATAC + _WL + _PE + ["--barcode-translate", sbo.TR + "/missing_rc16.txt.gz"], str(out))
    assert r.returncode == 255, r.stderr
    assert "Barcode does not exist in the translation table.\n" in r.stderr and "no output was written" in r.stderr
    assert not out.exists()


def test_format_sam_gpu_text_past_4_gib():
    """A call whose text passes 2^32 bytes (the offsets of the lines are 64-bit): 4,500 single-end cores at one position whose
    four reads carry 1 MB names.  Lines come in read-id order, each read's line as the host twin writes it."""
    import ctypes as C
    from tests.util import read_fasta
    names, seqs = read_fasta(os.path.join(SC, "ref.fa.gz"))
    p = cb.make_params("", output_format=4, single_end=1, mapq_threshold=0)
    n_reads, n = 4, 4500
    core = np.zeros(n_reads, dtype=cb.SAM_RECORD)
    core["rid"], core["pos"][:, 0], core["end"][:, 0], core["mapq"], core["n_cigar"][:, 0] = 0, 1000, 1049, 60, 1
    core["strand"][:, 0], core["read_id"] = 1, np.arange(n_reads)
    core["cigar"][:, 0, 0] = 50 << 4
    reads = ([b"r%d_" % i + b"x" * 1_000_000 for i in range(n_reads)], [bytes(seqs[0][1000:1050])] * n_reads, [b"I" * 50] * n_reads)
    one = cb.format_sam(p, names, seqs, core, reads)
    lines = one.split(b"\n")[len(names):-1]
    header = one[:len(one) - sum(len(x) + 1 for x in lines)]
    cores = core[np.arange(n) % n_reads]
    count = np.bincount(cores["read_id"], minlength=n_reads)
    want_len = len(header) + sum(int(count[i]) * (len(lines[i]) + 1) for i in range(n_reads))
    assert want_len > 1 << 32
    m = cb.Mapper(p)
    m.upload_reference(seqs, names)
    keep = []
    rs = cb.binding._sam_read_set(reads, keep)
    arr = (C.c_char_p * len(names))(*[s.encode() for s in names])
    lens = np.array([len(s) for s in seqs], dtype=np.uint32)
    cores = np.ascontiguousarray(cores)
    args = (m.h, arr, lens.ctypes.data, len(names), cores.ctypes.data, None, 0, n, C.byref(rs), None, 0)
    assert m.L.cmx_format_sam_gpu(*args, None, 0) == want_len
    buf = np.empty(want_len, dtype=np.uint8)
    assert m.L.cmx_format_sam_gpu(*args, buf.ctypes.data, want_len) == want_len
    m.close()
    mv = memoryview(buf)
    assert mv[:len(header)] == header
    at = len(header)
    for i in range(n_reads):
        line = lines[i] + b"\n"
        for _ in range(int(count[i])):
            assert mv[at:at + len(line)] == line, (i, at)
            at += len(line)
    assert at == want_len
