"""Time of bulk-level duplicate removal of barcoded records: cmx_postprocess_bc_bulk_gpu against its host twin
cmx_postprocess_bc_bulk and against cell-level cmx_postprocess_gpu (the --preset atac rule) on the same seeded record set, host
buffers in and out (the host clock around calls that end in a synchronise).  The default set is 50 M paired-end records on 24
sequences of 100 Mbp under 20 000 whitelisted barcodes, with 5 % of the records at one position of a 16.5 kbp sequence (a
chrM-like hot spot: one bulk group of 2.5 M records).  Device and host-twin outputs are compared.  Prints one JSON line with the
card's name and power limit beside the times.

    python tools/bench_bulk_dedup.py [--records N] [--reps R] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import chromap_b200 as cb  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.TimeoutExpired):
        return "unknown"


def records(rng, n, n_bc=20000, n_seq=24, seq_len=100_000_000, hot_frac=0.05):
    r = np.zeros(n, dtype=cb.PE_RECORD)
    r["read_id"] = np.arange(n, dtype=np.uint32)
    r["rid"] = rng.integers(0, n_seq, n)
    r["fragment_start"] = rng.integers(0, seq_len - 1000, n)
    r["fragment_length"] = rng.integers(100, 500, n)
    dup = rng.random(n) < 0.2  # PCR duplicates: a fifth of the records copy another's position
    src = rng.integers(0, n, int(dup.sum()))
    for f in ("rid", "fragment_start", "fragment_length"):
        r[f][dup] = r[f][src]
    hot = rng.random(n) < hot_frac
    r["rid"][hot] = n_seq; r["fragment_start"][hot] = 8000; r["fragment_length"][hot] = 300
    r["mapq"] = rng.choice([0, 20, 60], n, p=[0.05, 0.05, 0.9])
    r["direction"] = rng.integers(0, 2, n)
    r["is_unique"] = 1
    r["num_dups"] = 1
    r["positive_alignment_length"] = 50
    r["negative_alignment_length"] = 50
    wk = np.unique(rng.integers(0, 1 << 32, n_bc, dtype=np.uint64))
    wc = rng.integers(1, 5000, len(wk)).astype(np.uint32)
    return r, wk[rng.integers(0, len(wk), n)], wk, wc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=50_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    rng = np.random.default_rng(2026)
    recs, keys, wk, wc = records(rng, a.records)
    p = cb.make_params("chip")
    m = cb.Mapper(p, device=0)
    m.upload_barcode_whitelist(wk, wc, int(wc.sum()), 16)
    L, h = m.L, m.h
    import ctypes as C

    def timed(fn):
        ts = []
        for i in range(a.reps + 1):  # the first call warms up
            r, k, n = recs.copy(), keys.copy(), C.c_uint64()
            t0 = time.perf_counter()
            rc = fn(r, k, n)
            ts.append(time.perf_counter() - t0)
            assert rc == 0, rc
        return sorted(ts[1:])[len(ts[1:]) // 2], r[:n.value], k[:n.value]

    pr = C.byref(p)
    t_dev, dr, dk = timed(lambda r, k, n: L.cmx_postprocess_bc_bulk_gpu(h, r.ctypes.data, k.ctypes.data, len(r), C.byref(n)))
    t_cell, cr, _ = timed(lambda r, k, n: L.cmx_postprocess_gpu(h, r.ctypes.data, k.ctypes.data, len(r), C.byref(n)))
    reps, a.reps = a.reps, 1
    t_host, hr, hk = timed(lambda r, k, n: L.cmx_postprocess_bc_bulk(pr, wk.ctypes.data, wc.ctypes.data, len(wk), r.ctypes.data, k.ctypes.data, len(r), C.byref(n)))
    same = len(dr) == len(hr) and all(np.array_equal(dr[f], hr[f]) for f in dr.dtype.names) and np.array_equal(dk, hk)
    res = dict(card=card(), records=a.records, device_bulk_s=round(t_dev, 4), host_twin_bulk_s=round(t_host, 4), device_cell_level_s=round(t_cell, 4),
               reps=reps, bulk_out=int(len(dr)), cell_out=int(len(cr)), device_equals_host_twin=bool(same))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")
    m.close()
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
