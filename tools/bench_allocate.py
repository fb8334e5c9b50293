"""Time of --allocate-multi-mappings: cmx_allocate_multi_mappings_gpu against its host twin cmx_allocate_multi_mappings on the same
synthetic record set, both host buffers in and out (the host clock around calls that end in a synchronise).  The default set is
50 M paired-end records as a run at -n 4 leaves them: about 10 % multi-mappings (mapq < 4, 2 to 4 candidates per read), the rest
uni-mappings on 24 sequences of 100 Mbp.  The two outputs are compared.  One more device call runs under torch.profiler to split
its device time by kernel: the single-CTA generator (al_mt_kernel) and the other allocation kernels.  Prints one JSON line with
the card's name and power limit beside the times.

    python tools/bench_allocate.py [--records N] [--reps R] [--out FILE]
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


def records(rng, n, multi_frac=0.10, n_seq=24, seq_len=100_000_000):
    n_multi_target = int(n * multi_frac)
    cand = rng.integers(2, 5, n_multi_target // 3 + 1)
    cand = cand[:np.searchsorted(np.cumsum(cand), n_multi_target) + 1]
    n_multi = int(cand.sum())
    n_uni = n - n_multi
    r = np.zeros(n, dtype=cb.PE_RECORD)
    r["read_id"][:n_uni] = np.arange(n_uni, dtype=np.uint32) * 2
    r["read_id"][n_uni:] = np.repeat(np.arange(len(cand), dtype=np.uint32) * 2 + 1, cand)
    r["rid"] = rng.integers(0, n_seq, n)
    r["fragment_start"] = rng.integers(0, seq_len - 1000, n)
    r["fragment_length"] = rng.integers(100, 500, n)
    r["mapq"][:n_uni] = rng.integers(4, 61, n_uni)
    r["mapq"][n_uni:] = rng.integers(0, 4, n_multi)
    r["direction"] = rng.integers(0, 2, n)
    r["is_unique"][:n_uni] = 1
    r["num_dups"] = 1
    r["positive_alignment_length"] = 50
    r["negative_alignment_length"] = 50
    return rng.permutation(r), n_multi


def kernel_times(m, recs):
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
    except ImportError:
        return None
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.allocate_multi_mappings_gpu(recs, None, 0, 11)
    mt, al, total = 0.0, 0.0, 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if e.key.startswith("al_mt_kernel"):
            mt += t
        elif e.key.startswith("al_"):
            al += t
        if "kernel" in e.key.lower() or e.key.startswith(("al_", "pp_")) or "Memcpy" in e.key or "Memset" in e.key:
            total += t
    return dict(generator_ms=round(mt / 1e3, 3), other_allocation_kernels_ms=round(al / 1e3, 3), device_total_ms=round(total / 1e3, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=50_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    rng = np.random.default_rng(7)
    recs, n_multi = records(rng, a.records)
    m = cb.Mapper(cb.make_params("", max_num_best_mappings=4, mapq_threshold=0), device=0)
    m.allocate_multi_mappings_gpu(recs, None, 0, 11)  # warm-up at the timed size: module load, CUB's choices for this size
    gpu = []
    for _ in range(a.reps):
        t = time.perf_counter()
        gr, _, gs = m.allocate_multi_mappings_gpu(recs, None, 0, 11)
        gpu.append(time.perf_counter() - t)
    t = time.perf_counter()
    hr, _, hs = m.allocate_multi_mappings(recs, None, 0, 11)
    host = time.perf_counter() - t
    same = gs == hs and len(gr) == len(hr) and all(np.array_equal(gr[f], hr[f]) for f in gr.dtype.names)
    res = dict(card=card(), records=a.records, multi_records=n_multi, stats=gs, gpu_call_s=round(sorted(gpu)[len(gpu) // 2], 4),
               gpu_calls_s=[round(x, 4) for x in gpu], host_twin_s=round(host, 3), outputs_equal=bool(same), device_kernels=kernel_times(m, recs))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
