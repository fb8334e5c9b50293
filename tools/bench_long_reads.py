"""Reads longer than 160 bases on one GPU: pairs/s, device memory and the pairs each scratch tier held, for --preset chip on
bench.py's synthetic genome: 2x150 at max_read_length 160 next to 2x250 after the context has grown to 256
(cmx_set_max_read_length) and 2x300 after growing to 320, at the same pairs per call; then --SAM at 2x250 on a smaller genome.  A leg that fails records
the library's message instead of its numbers.
bench.py is imported for its genome and read synthesis only.  Prints one JSON line."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def make_batches(torch, ref, n_seq, seq_len, read_len, n_call, seed, dev):
    return [bench.gen_pairs(torch, ref, n_seq, seq_len, n_call, read_len, seed + s, dev) for s in range(2)]


def leg(torch, m, L, batches, read_len, n_call, steps, dev, rec_bytes):
    """Mean pairs/s over `steps` timed calls of n_call pairs (one untimed warm-up call first), alternating two batches."""
    import chromap_b200 as cb
    try:
        return _leg(torch, m, L, batches, read_len, n_call, steps, dev, rec_bytes)
    except cb.CmxError as e:
        free, total = torch.cuda.mem_get_info(dev)
        return {"read_len": read_len, "max_read_length": L, "pairs_per_call": n_call, "failed": str(e),
                "device_mem_in_use_gb": round((total - free) / 1e9, 2)}


def _leg(torch, m, L, batches, read_len, n_call, steps, dev, rec_bytes):
    out = torch.empty(n_call * rec_bytes, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    t = 0.0
    for s in range(steps + 1):
        r1, r2, off = batches[s % 2]
        torch.cuda.synchronize()
        t0 = time.time()
        m.map_batch(r1, off, r2, off, first_read_id=s * n_call, on_device=True, n_pairs=n_call, out=out, out_on_device=True)
        torch.cuda.synchronize()
        if s:
            t += time.time() - t0
    free, total = torch.cuda.mem_get_info(dev)
    return {"read_len": read_len, "max_read_length": L, "pairs_per_call": n_call, "calls": steps,
            "pairs_per_s": round(steps * n_call / t), "device_mem_in_use_gb": round((total - free) / 1e9, 2),
            "tier_pairs_last_call": m.timing()["tier_pairs"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-gbp", type=float, default=3.0)
    ap.add_argument("--sam-ref-gbp", type=float, default=0.2)
    ap.add_argument("--n-seq", type=int, default=24)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--pairs-per-call", type=int, default=500000, help="chromap-b200's call above 160 bases: one reference batch")
    a = ap.parse_args()
    import torch
    import chromap_b200 as cb
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_reads.py: no CUDA device")
    dev = torch.device("cuda", 0)
    res = {"gpu": bench.gpu_description(torch, dev)}
    ref, offsets, seq_len = bench.gen_reference(torch, dev, int(a.ref_gbp * 1e9), a.n_seq, a.seed)
    m = cb.Mapper(cb.make_params("chip", max_read_length=160), device=0)
    m.upload_reference_ptr(ref.data_ptr(), offsets)
    n = a.pairs_per_call
    # the reads of both legs first: the generator's copy of the genome then leaves the device before the index is built
    b150 = make_batches(torch, ref, a.n_seq, seq_len, 150, n, a.seed, dev)
    b250 = make_batches(torch, ref, a.n_seq, seq_len, 250, n, a.seed + 100, dev)
    b300 = make_batches(torch, ref, a.n_seq, seq_len, 300, n, a.seed + 200, dev)
    del ref
    torch.cuda.empty_cache()
    m.build_index(bench.K_MER, bench.WINDOW)
    free, total = torch.cuda.mem_get_info(dev)
    res["device_mem_in_use_after_index_gb"] = round((total - free) / 1e9, 2)
    res["chip_2x150_L160"] = leg(torch, m, 160, b150, 150, n, a.steps, dev, 24)
    del b150
    torch.cuda.empty_cache()
    m.set_max_read_length(256)
    res["chip_2x250_L256"] = leg(torch, m, 256, b250, 250, n, a.steps, dev, 24)
    del b250
    torch.cuda.empty_cache()
    m.set_max_read_length(320)
    res["chip_2x300_L320"] = leg(torch, m, 320, b300, 300, n, a.steps, dev, 24)
    del m, b300
    torch.cuda.empty_cache()
    ref, offsets, seq_len = bench.gen_reference(torch, dev, int(a.sam_ref_gbp * 1e9), a.n_seq, a.seed + 1)
    m = cb.Mapper(cb.make_params("", max_read_length=256, output_format=4), device=0)
    m.upload_reference_ptr(ref.data_ptr(), offsets)
    m.build_index(bench.K_MER, bench.WINDOW)
    bsam = make_batches(torch, ref, a.n_seq, seq_len, 250, n, a.seed + 300, dev)
    res["sam_2x250_L256_%.1fgbp" % a.sam_ref_gbp] = leg(torch, m, 256, bsam, 250, n, a.steps, dev, 224)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
