"""--barcode-translate on the GPU path: cmx_format_bed_gpu with an uploaded table against the host twin (cmx_format_bed_bc_tr)
and the oracle's Translate, across the 8 M-record chunk boundary, after a re-upload and after removal; and every case of
tests/golden/synth_barcode_translate/ through the CLI with the device reader and with the host reader, byte-equal to the
reference binary's output (make_golden_barcode_translate.sh)."""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from tests.test_barcode_translate_host import NAMES, _oracle_text, _random_case

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")
G = os.path.join(ROOT, "tests", "golden")
SC = os.path.join(G, "synth_sc")
SMALL = os.path.join(G, "synth_small")
BT = os.path.join(G, "synth_barcode_translate")


@pytest.fixture(scope="module")
def mapper():
    m = cb.Mapper(cb.make_params())
    m.upload_reference([np.full(100, 65, dtype=np.uint8)] * 3, names=NAMES)
    yield m
    m.close()


@pytest.mark.parametrize("bc_len,L", [(16, 16), (16, 8), (16, 5), (16, 4), (16, 20), (10, 3), (32, 8), (32, 31), (1, 1)])
def test_format_bed_gpu_translates_like_the_host_twin_and_the_oracle(mapper, bc_len, L):
    rng = np.random.default_rng(bc_len * 1000 + L)
    recs, bcs, t = _random_case(rng, 20000, bc_len, L, 60)
    mapper.upload_barcode_translation(t)
    got = mapper.format_bed_gpu(recs, bcs, bc_len)
    assert got == cb.format_bed_bc_tr(NAMES, recs, bcs, bc_len, t) == _oracle_text(recs, bcs, bc_len, t)
    mapper.upload_barcode_translation(None)
    assert mapper.format_bed_gpu(recs, bcs, bc_len) == mapper.format_bed_bc(recs, bcs, bc_len)


def test_reupload_replaces_and_removal_restores_the_barcode(mapper):
    rng = np.random.default_rng(3)
    recs, bcs, t1 = _random_case(rng, 5000, 16, 8, 40)
    t2 = cb.BarcodeTranslation(t1.keys, [b"second_" + x for x in t1.to], 8)
    mapper.upload_barcode_translation(t1)
    assert mapper.format_bed_gpu(recs, bcs, 16) == _oracle_text(recs, bcs, 16, t1)
    mapper.upload_barcode_translation(t2)
    assert mapper.format_bed_gpu(recs, bcs, 16) == _oracle_text(recs, bcs, 16, t2)
    mapper.upload_barcode_translation(None)
    assert mapper.format_bed_gpu(recs, bcs, 16) == _oracle_text(recs, bcs, 16, None)
    assert mapper.format_bed_gpu(recs) == mapper.format_bed(recs)  # bulk text is untouched by a table either way
    mapper.upload_barcode_translation(t2)
    assert mapper.format_bed_gpu(recs) == mapper.format_bed(recs)
    mapper.upload_barcode_translation(None)


def test_missing_segments_are_counted_and_nothing_is_written(mapper):
    rng = np.random.default_rng(17)
    recs, bcs, t = _random_case(rng, 20000, 16, 4, 30, drop=0.1)
    table = {int(k) for k in t.keys}
    per_rec = [sum(((int(b) >> (8 * (3 - s))) & 0xFF) not in table for s in range(4)) for b in bcs]
    first = next(i for i, m in enumerate(per_rec) if m)
    mapper.upload_barcode_translation(t)
    with pytest.raises(cb.BarcodeNotTranslated) as e:
        mapper.format_bed_gpu(recs, bcs, 16)
    bc = "".join("ACGT"[(int(bcs[first]) >> (2 * (15 - j))) & 3] for j in range(16))
    assert "%d barcode segments" % sum(per_rec) in str(e.value) and bc in str(e.value) and "record %d" % first in str(e.value)
    with pytest.raises(cb.BarcodeNotTranslated):
        cb.format_bed_bc_tr(NAMES, recs, bcs, 16, t)
    mapper.upload_barcode_translation(None)


def test_a_call_across_the_chunk_boundary(mapper):
    n = (8 << 20) + 4321
    rng = np.random.default_rng(8)
    recs, bcs, t = _random_case(rng, n, 16, 8, 300)
    mapper.upload_barcode_translation(t)
    got = mapper.format_bed_gpu(recs, bcs, 16)
    assert got == cb.format_bed_bc_tr(NAMES, recs, bcs, 16, t)
    # a segment without an entry in the second chunk only: the call refuses before the first chunk's text reaches the buffer
    v = min(set(range(1 << 16)) - {int(k) for k in t.keys})
    bcs2 = bcs.copy()
    bcs2[n - 7] = (bcs2[n - 7] & ~np.uint64(0xFFFF)) | np.uint64(v)
    names = (C.c_char_p * 3)(*[x.encode() for x in NAMES])
    buf = C.create_string_buffer(len(got) + 1)
    rc = mapper.L.cmx_format_bed_gpu(mapper.h, names, recs.ctypes.data, bcs2.ctypes.data, n, 16, buf, len(got))
    assert rc == -8 and "record %d" % (n - 7) in mapper.L.cmx_last_error(mapper.h).decode()
    assert buf.raw[:1 << 16].count(0) == 1 << 16
    mapper.upload_barcode_translation(None)


@pytest.fixture(scope="module")
def index(tmp_path_factory):
    d = tmp_path_factory.mktemp("ix")
    out = {}
    for name in ("synth_sc", "synth_small"):
        out[name] = str(d / (name + ".index"))
        subprocess.check_call([CLI, "-i", "-r", os.path.join(G, name, "ref.fa.gz"), "-o", out[name]], stderr=subprocess.DEVNULL)
    return out


_WL = ["--barcode-whitelist", os.path.join(SC, "whitelist.txt")]
_PE = ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", SC + "/barcode.fq.gz"]
_SE = ["-1", SC + "/read1.fq.gz", "-b", SC + "/barcode.fq.gz"]
_ATAC = ["--preset", "atac"]
CASES = {  # name: (index, arguments, table, expected output)
    "pe_rc16": ("synth_sc", _ATAC + _WL + _PE, "rc16", "pe_rc16"),
    "se_rc16": ("synth_sc", _ATAC + _WL + _SE, "rc16", "se_rc16"),
    "se_inmem_rc16": ("synth_sc", ["-q", "0", "--remove-pcr-duplicates", "--Tn5-shift"] + _WL + _SE, "rc16", "se_inmem_rc16"),
    "pe_names": ("synth_sc", _ATAC + _WL + _PE, "names", "pe_names"),
    "pe_half8": ("synth_sc", _ATAC + _WL + _PE, "half8", "pe_half8"),
    "pe_all5_nowl": ("synth_sc", _ATAC + _PE, "all5", "pe_all5_nowl"),
    "pe_all5_notinwl": ("synth_sc", _ATAC + _WL + ["--output-mappings-not-in-whitelist"] + _PE, "all5", "pe_all5_notinwl"),
    "pe_long20": ("synth_sc", _ATAC + _WL + _PE, "long20", "pe_long20"),
    "bc24_read_format": ("synth_sc", _ATAC + _WL + ["-1", SC + "/read1.fq.gz", "-2", SC + "/read2.fq.gz", "-b", G + "/synth_read_format/bc24.fq.gz",
                                                    "--read-format", "bc:8:23"], "rc16", "pe_rc16"),
    "bulk_chip_ignores": ("synth_small", ["--preset", "chip", "-1", SMALL + "/read1.fq.gz", "-2", SMALL + "/read2.fq.gz"], "rc16", None),
}


def _run(index, name, args, out, reader):
    return subprocess.run([CLI, "-x", index[name], "-r", os.path.join(G, name, "ref.fa.gz"), "-o", out] + args + (["--host-reader"] if reader == "host" else []),
                          capture_output=True, text=True)


@pytest.mark.parametrize("reader", ["device", "host"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_cli_barcode_translate_equals_reference_binary_output(case, reader, index, tmp_path):
    name, args, table, want = CASES[case]
    out = str(tmp_path / "out.bed")
    r = _run(index, name, args + ["--barcode-translate", os.path.join(BT, table + ".txt.gz")], out, reader)
    assert r.returncode == 0, r.stderr
    assert "using the host reader" not in r.stderr
    want = os.path.join(BT, want + ".bed.gz") if want else os.path.join(SMALL, "chip.bed.gz")
    assert open(out, "rb").read() == gzip.open(want).read()


@pytest.mark.parametrize("reader", ["device", "host"])
def test_cli_missing_barcode_exits_255_and_writes_nothing(reader, index, tmp_path):
    out = tmp_path / "out.bed"
    r = _run(index, "synth_sc", _ATAC + _WL + _PE + ["--barcode-translate", os.path.join(BT, "missing_rc16.txt.gz")], str(out), reader)
    assert r.returncode == 255, r.stderr
    assert "Barcode does not exist in the translation table.\n" in r.stderr and "no output was written" in r.stderr
    assert not out.exists()
