"""--bc-error-threshold 2 on the GPU: cmx_stage_correct_barcodes (barcode_kernel + barcode_correct2_kernel, as
cmx_map_batch_pe runs them) against the oracle's CorrectBarcodeAt on random sets (barcode lengths 4 to 32, Ns, ties, full
neighbourhoods) and on 2 M barcodes against a 737,280-entry whitelist; cmx_map_batch_pe on the synth_bc_error2 fixture,
paired-end and single-end, against the oracle and the reference binary's BED; and every golden through the CLI with both
readers."""
import gzip
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from oracle import oracle_py as orc
from tests.bc_error2_oracle import GOLDEN, RUNS, SC, correct_barcodes, map_bc, random_set, read_barcodes, setup, whitelist
from tests.util import read_fasta

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")


@pytest.fixture(scope="module")
def mapper():
    m = cb.Mapper(cb.make_params("atac", max_read_length=64))
    yield m
    m.close()


def _stage_equals_oracle(m, wl, bcs, quals, bc_len, err, prob, out_nw=False):
    keys, counts, ns = wl.arrays()
    m.upload_barcode_whitelist(keys, counts, ns, bc_len, err_threshold=err, prob_threshold=prob, output_not_in_whitelist=out_nw)
    got = m.stage_correct_barcodes(bcs, quals, bc_len)
    want = correct_barcodes(wl, err, prob, bcs, quals, bc_len, out_nw)
    bad = np.flatnonzero((got[0] != want[0]) | (got[1] != want[1]))
    assert len(bad) == 0 and got[2:] == want[2:], (len(bad), bad[:5], got[2:], want[2:])
    return want


@pytest.mark.parametrize("bc_len,prob", [(4, 0.9), (8, 0.4), (12, 0.5), (16, 0.9), (16, 0.0), (24, 0.99), (32, 0.5), (32, 0.9)])
def test_stage_equals_oracle_on_random_sets(mapper, tmp_path, bc_len, prob):
    rng = np.random.default_rng(bc_len * 100 + int(prob * 100))
    path = str(tmp_path / "wl.txt")
    n_wl = 40 if bc_len == 4 else 400 if bc_len == 8 else 3000
    bcs, quals, sample = random_set(rng, bc_len, 20000, n_wl, 0 if bc_len < 8 else 3, path)
    wl = orc.Whitelist(path, bc_len)
    wl.sample(sample)
    _, _, n_in, n_cor = _stage_equals_oracle(mapper, wl, bcs, quals, bc_len, 2, prob)
    assert n_in > 0 and n_cor > 0
    _stage_equals_oracle(mapper, wl, bcs, quals, bc_len, 2, prob, out_nw=True)
    _stage_equals_oracle(mapper, wl, bcs, quals, bc_len, 1, prob)  # threshold 1 through the same entry


def test_stage_on_2m_barcodes_and_a_737k_whitelist(mapper, tmp_path):
    rng = np.random.default_rng(737280)
    A = np.frombuffer(b"ACGT", dtype=np.uint8)
    keys = np.unique(rng.integers(0, 1 << 32, 800000, dtype=np.uint64))[:737280]
    rng.shuffle(keys)
    seqs = A[((keys[:, None] >> (2 * np.arange(15, -1, -1, dtype=np.uint64))) & np.uint64(3)).astype(np.int64)]
    path = tmp_path / "wl737k.txt"
    path.write_bytes(b"".join(bytes(r) + b"\n" for r in seqs))
    n = 2_000_000
    obs = seqs[rng.integers(0, 200000, n)].copy()
    fix = rng.random(n) < 0.05  # need a search: one or two substitutions, or an N
    for i in np.flatnonzero(fix):
        for p in rng.choice(16, int(rng.integers(1, 3)), replace=False):
            obs[i, p] = ord("N") if rng.random() < 0.1 else A[(np.searchsorted(A, obs[i, p]) + rng.integers(1, 4)) % 4]
    quals = rng.integers(33, 75, (n, 16)).astype(np.uint8)
    wl = orc.Whitelist(str(path), 16)
    wl.sample(obs.ravel())
    _, _, n_in, n_cor = _stage_equals_oracle(mapper, wl, obs.ravel(), quals.ravel(), 16, 2, 0.9)
    assert n_in > 0.9 * n and n_cor > 0.03 * n


@pytest.fixture(scope="module")
def sc_mapper():
    names, seqs = read_fasta(os.path.join(SC, "ref.fa.gz"))
    ref, idx, pairs = setup()
    ms = {}
    for se in (False, True):
        m = cb.Mapper(cb.make_params("atac", max_read_length=64, single_end=int(se)))
        m.upload_reference(seqs, names)
        a = idx.arrays()
        m.upload_index(17, 7, a["n_buckets"], a["flags"], a["keys"], a["vals"], a["occ"])
        ms[se] = m
    yield ms
    for m in ms.values():
        m.close()


@pytest.mark.parametrize("name", sorted(RUNS))
def test_map_batch_equals_oracle_and_golden(sc_mapper, name):
    bc_path, _, se, prob, out_nw = RUNS[name]
    ref, idx, (s1, o1, s2, o2) = setup()
    bcs, quals, bc_len = read_barcodes(bc_path)
    wl = whitelist(name)
    m = sc_mapper[se]
    keys, counts, ns = wl.arrays()
    m.upload_barcode_whitelist(keys, counts, ns, bc_len, err_threshold=2, prob_threshold=prob, output_not_in_whitelist=out_nw)
    recs, stats = m.map_batch(s1, o1, None if se else s2, None if se else o2, barcodes=bcs, barcode_quals=quals, bc_len=bc_len)
    p = orc.make_params("atac", single_end=int(se))
    orecs, obc, ost = map_bc(p, idx, ref, s1, o1, None if se else s2, None if se else o2, bcs, quals, bc_len, wl, 2, prob, out_nw)
    assert len(recs) == len(orecs)
    for f in recs.dtype.names:
        assert np.array_equal(recs[f], orecs[f]), f
    assert np.array_equal(stats["barcode_keys"], obc)
    assert (stats["n_barcodes_in_whitelist"], stats["n_barcodes_corrected"]) == (int(ost[0]), int(ost[1]))
    r2, b2 = m.postprocess_gpu(recs, stats["barcode_keys"])
    assert m.format_bed_gpu(r2, b2, bc_len) == gzip.open(os.path.join(GOLDEN, name + ".bed.gz")).read()


@pytest.fixture(scope="module")
def index(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ix") / "sc.index")
    subprocess.check_call([CLI, "-i", "-r", os.path.join(SC, "ref.fa.gz"), "-o", out], stderr=subprocess.DEVNULL)
    return out


@pytest.mark.parametrize("reader", ["device", "host"])
@pytest.mark.parametrize("name", sorted(RUNS))
def test_cli_equals_reference_binary_output(name, reader, index, tmp_path):
    bc_path, wl_path, se, prob, out_nw = RUNS[name]
    out = str(tmp_path / "out.bed")
    args = [CLI, "--preset", "atac", "-x", index, "-r", os.path.join(SC, "ref.fa.gz"), "-1", os.path.join(SC, "read1.fq.gz")]
    args += [] if se else ["-2", os.path.join(SC, "read2.fq.gz")]
    args += ["-b", bc_path, "--barcode-whitelist", wl_path, "--bc-error-threshold", "2", "--bc-probability-threshold", str(prob), "-o", out]
    args += (["--output-mappings-not-in-whitelist"] if out_nw else []) + (["--host-reader"] if reader == "host" else [])
    r = subprocess.run(args, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert open(out, "rb").read() == gzip.open(os.path.join(GOLDEN, name + ".bed.gz")).read()
    st = dict(l.split(None, 1) for l in open(os.path.join(GOLDEN, "stats.txt")).read().splitlines())[name].split()
    assert "Number of barcodes in whitelist: %s.\nNumber of corrected barcodes: %s." % tuple(st) in r.stderr
