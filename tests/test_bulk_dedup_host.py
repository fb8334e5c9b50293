"""The host twin of bulk-level duplicate removal (cmx_postprocess_bc_bulk) reproduces every bulk-level golden of
tests/golden/synth_bulk_dedup from the oracle's records, equals the merge loop's restatement on seeded random record sets, refuses
what the reference leaves undefined; and the CLI refusals that need no device."""
import os
import subprocess

import numpy as np
import pytest

import chromap_b200 as cb
from tests import bulk_dedup_oracle as bdo

CLI = os.path.join(bdo.ROOT, "chromap_b200", "bin", "chromap-b200")
BULK = sorted(n for n in bdo.RUNS if bdo.bulk_level(n))


def _cb_params(name):
    preset, kw, se, _ = bdo.RUNS[name]
    return cb.make_params(preset, single_end=int(se), **kw)


@pytest.mark.parametrize("name", BULK)
def test_host_twin_reproduces_golden(name):
    recs, keys = bdo.records(name)
    wk, wc = bdo.whitelist()
    out_r, out_k = cb.postprocess_bc_bulk(_cb_params(name), wk, wc, recs, keys)
    tr = bdo.RUNS[name][3]
    t = cb.parse_barcode_translation(__import__("gzip").open(tr).read()) if tr else None
    got = cb.format_bed_bc_tr(bdo.ref_names(), out_r, out_k, bdo.setup()[4][2], t)
    assert got == bdo.golden(name)


def random_set(rng, n, n_rid=3, n_pos=40, n_bc=6, dense=False):
    """Records piled on few positions and barcodes: long groups, returning barcodes, mixed MAPQ, ties of abundance."""
    recs = np.zeros(n, dtype=cb.PE_RECORD)
    recs["read_id"] = rng.permutation(n) + 5
    recs["rid"] = rng.integers(0, n_rid, n)
    recs["fragment_start"] = 1000 + rng.integers(0, n_pos, n) * (1 if dense else 7)
    recs["fragment_length"] = 40 + rng.integers(0, 3, n)
    recs["mapq"] = rng.choice([0, 5, 29, 30, 31, 60], n)
    recs["direction"] = rng.integers(0, 2, n)
    recs["is_unique"] = rng.integers(0, 2, n)
    recs["num_dups"] = 1
    recs["positive_alignment_length"] = 30 + rng.integers(0, 10, n)
    recs["negative_alignment_length"] = 30 + rng.integers(0, 10, n)
    wk = np.arange(1, n_bc + 1, dtype=np.uint64) * np.uint64(0x9E37)
    wc = rng.choice([3, 3, 7, 10], n_bc).astype(np.uint32)
    return recs, wk[rng.integers(0, n_bc, n)], wk, wc


@pytest.mark.parametrize("seed", range(12))
def test_host_twin_equals_restatement(seed):
    rng = np.random.default_rng(seed)
    n = [1, 2, 50, 400, 3000, 3000][seed % 6]
    recs, keys, wk, wc = random_set(rng, n, n_pos=2 if seed % 6 == 5 else 40, dense=seed % 3 == 0)
    if seed % 6 == 5:
        keys[:] = wk[0]  # one barcode: entries of hundreds of records, num_dups saturates
        keys[::3] = wk[1]
    for se in (0, 1):
        for q in (0, 30):
            for tn5 in (0, 1):
                p = cb.make_params("", low_memory_mode=1, remove_pcr_duplicates=1, mapq_threshold=q, single_end=se, tn5_shift=tn5)
                want_r, want_k = bdo.merge(p, dict(zip(wk.tolist(), wc.tolist())), recs, keys)
                got_r, got_k = cb.postprocess_bc_bulk(p, wk, wc, recs, keys)
                assert len(got_r) == len(want_r)
                for f in got_r.dtype.names:
                    assert np.array_equal(got_r[f], want_r[f]), f
                assert np.array_equal(got_k, want_k)


def test_host_twin_saturates_and_keeps_the_last_group_rule():
    recs = np.zeros(300, dtype=cb.PE_RECORD)
    recs["rid"] = 2; recs["fragment_start"] = 500; recs["fragment_length"] = 200; recs["read_id"] = np.arange(300)
    recs["mapq"] = 10
    recs["mapq"][299] = 60  # one clean record in the last group; the best entry's own MAPQ is 10
    keys = np.full(300, 11, dtype=np.uint64); keys[299] = 12
    p = cb.make_params("chip")
    got_r, got_k = cb.postprocess_bc_bulk(p, np.array([11, 12], dtype=np.uint64), np.array([1, 50], dtype=np.uint32), recs, keys)
    assert len(got_r) == 1 and got_k[0] == 11 and got_r[0]["num_dups"] == 255 and got_r[0]["mapq"] == 10
    recs["rid"][299] = 3  # now the clean record is a group of its own, last; the big group fails its own threshold
    got_r, got_k = cb.postprocess_bc_bulk(p, np.array([11, 12], dtype=np.uint64), np.array([1, 50], dtype=np.uint32), recs, keys)
    assert len(got_r) == 1 and got_k[0] == 12 and got_r[0]["num_dups"] == 1


def test_host_twin_refusals():
    rng = np.random.default_rng(1)
    recs, keys, wk, wc = random_set(rng, 100)
    p = cb.make_params("chip")
    keys2 = keys.copy(); keys2[7] = 12345  # not in the whitelist
    for args, status in [((p, wk[:0], wc[:0], recs, keys), -4), ((p, wk, wc, recs, keys2), -3),
                         ((cb.make_params(""), wk, wc, recs, keys), -3), ((cb.make_params("chip", remove_pcr_duplicates=0), wk, wc, recs, keys), -3),
                         ((cb.make_params("chip", output_format=4), wk, wc, recs, keys), -3)]:
        with pytest.raises(cb.BulkDedupError) as e:
            cb.postprocess_bc_bulk(*args)
        assert e.value.status == status


_BASE = ["-x", "none.index", "-r", "none.fa", "-1", "r1.fq", "-2", "r2.fq", "-b", "bc.fq", "-o", "out"]


@pytest.mark.parametrize("args,msg", [
    (["--preset", "chip"], "ranks barcodes by their abundance in the whitelist; give --barcode-whitelist"),
    (["--low-mem", "--remove-pcr-duplicates", "--barcode-whitelist", "wl.txt", "--output-mappings-not-in-whitelist"],
     "does not go with --output-mappings-not-in-whitelist"),
    (["--preset", "atac", "--remove-pcr-duplicates-at-bulk-level"], "ranks barcodes by their abundance in the whitelist"),
    (["--SAM", "--preset", "chip", "--barcode-whitelist", "wl.txt"], "bulk-level duplicate removal of barcoded data is not on the GPU path"),
])
def test_cli_refusals_without_device(args, msg, tmp_path):
    r = subprocess.run([CLI] + _BASE + args, capture_output=True, text=True, cwd=tmp_path)
    assert r.returncode == 255
    assert msg in r.stderr


def test_cli_cell_level_wins_in_any_order(tmp_path):
    """--remove-pcr-duplicates-at-cell-level after or before the bulk-level option: cell level, so no bulk-level refusal."""
    for order in (["--remove-pcr-duplicates-at-cell-level", "--remove-pcr-duplicates-at-bulk-level"],
                  ["--remove-pcr-duplicates-at-bulk-level", "--remove-pcr-duplicates-at-cell-level"]):
        r = subprocess.run([CLI] + _BASE + ["--preset", "chip"] + order, capture_output=True, text=True, cwd=tmp_path)
        assert "bulk-level" not in r.stderr and "abundance" not in r.stderr
