"""The host twin of the barcoded SAM writer (cmx_format_sam_bc), fed with the oracle's barcoded cores and keys, reproduces every
file of tests/golden/synth_sam_bc and refuses a table without one of the output barcodes; and the CLI refusals of barcoded
runs that need no device."""
import gzip
import os
import subprocess

import pytest

import chromap_b200 as cb
from tests import sam_bc_oracle as sbo
from tests.util import read_fasta

CLI = os.path.join(sbo.ROOT, "chromap_b200", "bin", "chromap-b200")


def _cb_params(name):
    preset, kw, se, _, _, _, _, _ = sbo.RUNS[name]
    return cb.make_params(preset, output_format=4, single_end=int(se), **kw)


def _inputs(name):
    ref, index, r1, r2 = sbo.setup()
    keys, ok, bc_len = sbo.barcode_gate(name)
    se = sbo.RUNS[name][2]
    cores, ck = sbo.cores_and_keys(sbo.params(name), index, ref, r1, None if se else r2, keys, ok)
    names, seqs = read_fasta(os.path.join(sbo.SC, "ref.fa.gz"))
    reads = lambda recs: ([r[0] for r in recs], [r[1] for r in recs], [r[2] for r in recs])
    return names, seqs, cores, ck, bc_len, reads(r1), None if se else reads(r2)


@pytest.mark.parametrize("name", sorted(sbo.RUNS))
def test_host_twin_reproduces_golden(name):
    names, seqs, cores, ck, bc_len, reads1, reads2 = _inputs(name)
    tr_path = sbo.RUNS[name][7]
    t = cb.parse_barcode_translation(gzip.open(tr_path).read()) if tr_path else None
    got = cb.format_sam_bc(_cb_params(name), names, seqs, cores, ck, bc_len, reads1, reads2, translation=t)
    assert got == gzip.open(os.path.join(sbo.OUT, name + ".sam.gz")).read()


def test_host_twin_missing_segment():
    names, seqs, cores, ck, bc_len, reads1, reads2 = _inputs("pe_atac")
    t = cb.parse_barcode_translation(gzip.open(os.path.join(sbo.TR, "missing_rc16.txt.gz")).read())
    with pytest.raises(cb.BarcodeNotTranslated):
        cb.format_sam_bc(_cb_params("pe_atac"), names, seqs, cores, ck, bc_len, reads1, reads2, translation=t)


def test_host_twin_without_keys_is_the_bulk_writer():
    names, seqs, cores, ck, bc_len, reads1, reads2 = _inputs("pe_q0dedup")
    p = _cb_params("pe_q0dedup")
    assert cb.format_sam_bc(p, names, seqs, cores, None, 0, reads1, reads2) == cb.format_sam(p, names, seqs, cores, reads1, reads2)


_BASE = ["-x", "none.index", "-r", "none.fa", "-1", "r1.fq", "-2", "r2.fq", "-b", "bc.fq", "-o", "out"]


@pytest.mark.parametrize("args,msg", [
    (["--TagAlign"], "--TagAlign / --PAF with barcodes is not on the GPU path"),
    (["--PAF"], "--TagAlign / --PAF with barcodes is not on the GPU path"),
    (["--SAM", "--low-mem", "--remove-pcr-duplicates"], "bulk-level duplicate removal of barcoded data is not on the GPU path"),
])
def test_cli_refusals_without_device(args, msg, tmp_path):
    r = subprocess.run([CLI] + _BASE + args, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 255
    assert msg in r.stderr
