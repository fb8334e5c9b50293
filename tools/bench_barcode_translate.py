"""Time of cmx_format_bed_gpu on 20 M barcoded records (16-base barcodes, three sequences), without a translation table and
with a 16 -> 16 table of 737,280 entries (the size of the 10x Multiome ATAC whitelist), on one GPU.  Every barcode has an
entry.  Each call is host memory in and out, so the time includes the copies over PCIe; it is a host clock around calls
that return after the device is done.  Prints one JSON line with the card's name and power limit beside the times.

    python tools/bench_barcode_translate.py [--records N] [--entries M] [--reps R] [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=20_000_000)
    ap.add_argument("--entries", type=int, default=737_280)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    keys = np.unique(rng.integers(0, 1 << 32, a.entries + a.entries // 8, dtype=np.uint64))[: a.entries]
    rng.shuffle(keys)
    to = [row.tobytes() for row in np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, (len(keys), 16))]]
    table = cb.BarcodeTranslation(keys, to, 16)
    n = a.records
    recs = np.zeros(n, dtype=cb.PE_RECORD)
    recs["rid"] = rng.integers(0, 3, n)
    recs["fragment_start"] = np.sort(rng.integers(0, 250_000_000, n))
    recs["fragment_length"] = rng.integers(40, 800, n)
    recs["num_dups"] = rng.integers(1, 4, n)
    bcs = rng.choice(keys, n)
    names = ["chr1", "chr2", "chrX"]
    m = cb.Mapper(cb.make_params())
    m.upload_reference([np.full(100, 65, dtype=np.uint8)] * 3, names=names)
    res = {"records": n, "table_entries": int(len(keys)), "card": card(), "reps": a.reps}
    for label, t in (("no_table", None), ("table", table)):
        m.upload_barcode_translation(t)
        text = m.format_bed_gpu(recs, bcs, 16)  # warm-up (module load, allocations) and the size of the text
        times = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            m.format_bed_gpu(recs, bcs, 16)
            times.append(time.perf_counter() - t0)
        res[label] = {"seconds_median": float(np.median(times)), "seconds_min": float(min(times)), "bytes": len(text)}
    m.upload_barcode_translation(None)
    m.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
