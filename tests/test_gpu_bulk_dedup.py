"""Bulk-level duplicate removal of barcoded BED on the device (cmx_postprocess_bc_bulk_gpu): equal to the host twin and the
reference binary's files of tests/golden/synth_bulk_dedup, on one call of 2 M records whose largest group holds 10^6, its
refusals, and chromap-b200 with the device and the host FASTQ reader byte-identical to every golden."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from tests import bulk_dedup_oracle as bdo
from tests.test_bulk_dedup_host import BULK, _cb_params, random_set

pytestmark = pytest.mark.gpu
CLI = os.path.join(bdo.ROOT, "chromap_b200", "bin", "chromap-b200")


def _mapper(params, wk, wc, bc_len=16, output_not_in_whitelist=False):
    m = cb.Mapper(params, device=0)
    m.upload_barcode_whitelist(wk, wc, int(wc.sum()), bc_len, output_not_in_whitelist=output_not_in_whitelist)
    return m


def _same(a, b):
    assert len(a[0]) == len(b[0])
    for f in a[0].dtype.names:
        assert np.array_equal(a[0][f], b[0][f]), f
    assert np.array_equal(a[1], b[1])


@pytest.mark.parametrize("name", BULK)
def test_device_equals_host_twin_and_golden(name):
    recs, keys = bdo.records(name)
    wk, wc = bdo.whitelist()
    p = _cb_params(name)
    m = _mapper(p, wk, wc)
    got = m.postprocess_bc_bulk_gpu(recs, keys)
    _same(got, cb.postprocess_bc_bulk(p, wk, wc, recs, keys))
    tr = bdo.RUNS[name][3]
    t = cb.parse_barcode_translation(gzip.open(tr).read()) if tr else None
    assert cb.format_bed_bc_tr(bdo.ref_names(), got[0], got[1], 16, t) == bdo.golden(name)
    m.close()


@pytest.mark.parametrize("seed", range(6))
def test_device_equals_host_twin_random(seed):
    rng = np.random.default_rng(100 + seed)
    recs, keys, wk, wc = random_set(rng, [1, 3, 500, 5000, 20000, 20000][seed], n_pos=3 if seed == 5 else 40, dense=seed % 2 == 0)
    for se in (0, 1):
        for q, tn5 in ((0, 0), (30, 1)):
            p = cb.make_params("", low_memory_mode=1, remove_pcr_duplicates=1, mapq_threshold=q, single_end=se, tn5_shift=tn5)
            m = _mapper(p, wk, wc)
            _same(m.postprocess_bc_bulk_gpu(recs, keys), cb.postprocess_bc_bulk(p, wk, wc, recs, keys))
            m.close()


def test_device_two_million_records_one_group_of_a_million():
    rng = np.random.default_rng(7)
    n, hot = 2_000_000, 1_000_000
    recs, keys, wk, wc = random_set(rng, n, n_rid=25, n_pos=200000)
    wc = rng.integers(1, 1000, len(wk)).astype(np.uint32)
    hot_idx = rng.choice(n, hot, replace=False)  # a chrM-like hot spot: one position, every barcode
    recs["rid"][hot_idx] = 24; recs["fragment_start"][hot_idx] = 16000; recs["fragment_length"][hot_idx] = 300
    keys = rng.choice(wk, n)
    for se in (0, 1):
        p = cb.make_params("chip", single_end=se, tn5_shift=1)
        m = _mapper(p, wk, wc)
        got = m.postprocess_bc_bulk_gpu(recs, keys)
        _same(got, cb.postprocess_bc_bulk(p, wk, wc, recs, keys))
        m.close()


def test_refusals_leave_records_untouched():
    rng = np.random.default_rng(3)
    recs, keys, wk, wc = random_set(rng, 1000)
    def status(m, r=recs, k=keys):
        r0, k0 = r.copy(), k.copy()
        with pytest.raises(cb.BulkDedupError) as e:
            m.postprocess_bc_bulk_gpu(r, k)
        assert np.array_equal(r, r0) and np.array_equal(k, k0)
        return e.value.status
    m = cb.Mapper(cb.make_params("chip"), device=0)
    assert status(m) == -4  # no whitelist
    m.close()
    for p in (cb.make_params(""), cb.make_params("chip", remove_pcr_duplicates=0), cb.make_params("chip", output_format=4),
              cb.make_params("hic")):
        m = _mapper(p, wk, wc)
        assert status(m) == -3
        m.close()
    m = _mapper(cb.make_params("chip"), wk, wc, output_not_in_whitelist=True)
    assert status(m) == -3
    m.close()
    m = _mapper(cb.make_params("chip"), wk, wc)
    k2 = keys.copy(); k2[500] = 999
    assert status(m, recs, k2) == -3
    m.close()


@pytest.fixture(scope="module")
def index(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ix") / "sc.index")
    subprocess.check_call([CLI, "-i", "-r", os.path.join(bdo.SC, "ref.fa.gz"), "-o", out], stderr=subprocess.DEVNULL)
    return out


_ARGS = {
    "pe_chip": ["--preset", "chip"],
    "se_chip": ["--preset", "chip"],
    "pe_q0": ["--low-mem", "--remove-pcr-duplicates", "-q", "0"],
    "se_q0": ["--low-mem", "--remove-pcr-duplicates", "-q", "0"],
    "pe_atac_bulk": ["--preset", "atac", "--remove-pcr-duplicates-at-bulk-level"],
    "pe_chip_rc16": ["--preset", "chip", "--barcode-translate", bdo.RC16],
    "pe_inmem_q0": ["--remove-pcr-duplicates", "-q", "0"],
}


@pytest.mark.parametrize("reader", [[], ["--host-reader"]])
@pytest.mark.parametrize("name", sorted(bdo.RUNS))
def test_cli_equals_reference_binary_output(name, reader, index, tmp_path):
    out = str(tmp_path / "o.bed")
    reads = ["-1", os.path.join(bdo.OUT, "read1.fq.gz"), "-b", os.path.join(bdo.OUT, "barcode.fq.gz")]
    if not bdo.RUNS[name][2]:
        reads += ["-2", os.path.join(bdo.OUT, "read2.fq.gz")]
    r = subprocess.run([CLI, "-x", index, "-r", os.path.join(bdo.SC, "ref.fa.gz"), "-o", out, "--barcode-whitelist", bdo.WL] + _ARGS[name] + reads + reader,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert open(out, "rb").read() == bdo.golden(name)
    want = [l.split()[-1] for l in open(os.path.join(bdo.OUT, "stats.txt")) if l.startswith(name + ".bed ")][0]
    assert "Number of output mappings (passed filters): %s\n" % want in r.stderr
