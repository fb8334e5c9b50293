"""Time of barcode correction (cmx_stage_correct_barcodes: barcode_kernel, and at --bc-error-threshold 2
barcode_correct2_kernel) on 2 M 16-base barcodes against a 737,280-entry whitelist (the size of the 10x Multiome ATAC
whitelist), on one GPU, with 2 % and 10 % of the barcodes needing a search (one or two substitutions, or an N).  Thresholds 1
and 2 alternate call by call.  Reported per case: the median host time of a call (host memory in and out: includes the
copies and allocations) and the median device time of the barcode kernels per call, from torch.profiler's CUDA activity.
Prints one JSON line with the card's name and power limit beside the times.

    python tools/bench_barcode_correction.py [--barcodes N] [--entries M] [--reps R] [--out FILE]
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


def barcodes(rng, seqs, n, frac):
    A = np.frombuffer(b"ACGT", dtype=np.uint8)
    obs = seqs[rng.integers(0, len(seqs), n)].copy()
    idx = np.flatnonzero(rng.random(n) < frac)
    two = rng.random(len(idx)) < 0.5
    p1 = rng.integers(0, 16, len(idx))
    p2 = (p1 + rng.integers(1, 16, len(idx))) % 16
    for p, sel in ((p1, np.ones(len(idx), bool)), (p2, two)):
        rows, cols = idx[sel], p[sel]
        cur = np.searchsorted(A, obs[rows, cols])
        obs[rows, cols] = A[(cur + rng.integers(1, 4, len(rows))) % 4]
    nrow = idx[rng.random(len(idx)) < 0.1]
    obs[nrow, rng.integers(0, 16, len(nrow))] = ord("N")
    return obs.ravel(), rng.integers(33, 75, (n, 16)).astype(np.uint8).ravel()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--barcodes", type=int, default=2_000_000)
    ap.add_argument("--entries", type=int, default=737_280)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(1)
    keys = np.unique(rng.integers(0, 1 << 32, a.entries + a.entries // 8, dtype=np.uint64))[: a.entries]
    rng.shuffle(keys)
    A = np.frombuffer(b"ACGT", dtype=np.uint8)
    seqs = A[((keys[:, None] >> (2 * np.arange(15, -1, -1, dtype=np.uint64))) & np.uint64(3)).astype(np.int64)]
    counts = rng.integers(1, 200, len(keys)).astype(np.uint32)
    m = cb.Mapper(cb.make_params("atac"))
    res = {"barcodes": a.barcodes, "whitelist": int(len(keys)), "card": card(), "reps": a.reps}
    for frac in (0.02, 0.10):
        bcs, quals = barcodes(rng, seqs, a.barcodes, frac)
        host = {1: [], 2: []}
        dev = {1: [], 2: []}
        for thr in (1, 2):  # warm-up: module load, allocations
            m.upload_barcode_whitelist(keys, counts, int(counts.sum()), 16, err_threshold=thr)
            m.stage_correct_barcodes(bcs, quals, 16)
        for _ in range(a.reps):
            for thr in (1, 2):
                m.upload_barcode_whitelist(keys, counts, int(counts.sum()), 16, err_threshold=thr)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    t0 = time.perf_counter()
                    _, _, n_in, n_cor = m.stage_correct_barcodes(bcs, quals, 16)
                    host[thr].append(time.perf_counter() - t0)
                    torch.cuda.synchronize()
                us = sum(e.device_time_total for e in prof.events() if "barcode" in e.name and "kernel" in e.name)
                dev[thr].append(us / 1000.0)
        for thr in (1, 2):
            res["frac%g_thr%d" % (frac, thr)] = {"host_ms_median": 1000 * float(np.median(host[thr])), "kernel_ms_median": float(np.median(dev[thr])),
                                                 "kernel_ms_min": float(min(dev[thr]))}
    m.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
