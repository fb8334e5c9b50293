"""Time `chromap-b200 --preset chip` on the same read pairs given as one file and as one file per lane, alternating the two.

A split run has more short calls (each file ends its last call early) and switches files while the last call of a file maps;
its `waiting for the loader` time shows whether that switch is overlapped.  Prints the card and its power limit, then the
`Mapped all reads in` and `Mapping phase` lines of every run.

    python tools/bench_cli_files.py [--lanes 4] [--pairs-per-lane 1600000] [--repeats 3] [--out DIR]
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.boundary_inputs import fastq, make_reads, reference  # noqa: E402

CLI = os.path.join(ROOT, "chromap_b200", "bin", "chromap-b200")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=4)
    ap.add_argument("--pairs-per-lane", type=int, default=1_600_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the report (default: print only)")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines = ["GPU: " + gpu]
    with tempfile.TemporaryDirectory() as d:
        seqs, _ = reference()
        ref = os.path.join(d, "ref.fa")
        with open(ref, "wb") as f:
            for i, s in enumerate(seqs):
                f.write(b">chr%d\n" % (i + 1) + s.tobytes() + b"\n")
        idx = os.path.join(d, "ref.index")
        subprocess.check_call([CLI, "-i", "-r", ref, "-o", idx], stderr=subprocess.DEVNULL)
        n = a.lanes * a.pairs_per_lane
        s1, _, s2, _ = make_reads(n, seed=41, length=50)
        one, split = {}, {}
        for mate, s in (("1", s1), ("2", s2)):
            text = fastq(s, 50)
            rec = len(text) // n
            one[mate] = os.path.join(d, "all_R%s.fq" % mate)
            open(one[mate], "wb").write(text)
            split[mate] = []
            for lane in range(a.lanes):
                p = os.path.join(d, "L%03d_R%s.fq" % (lane + 1, mate))
                open(p, "wb").write(text[lane * a.pairs_per_lane * rec:(lane + 1) * a.pairs_per_lane * rec])
                split[mate].append(p)
        del s1, s2
        lines.append("%d pairs of 2x50 bp: one file, and %d files of %d pairs" % (n, a.lanes, a.pairs_per_lane))
        runs = {"one file": ["-1", one["1"], "-2", one["2"]], "%d files" % a.lanes: ["-1", ",".join(split["1"]), "-2", ",".join(split["2"])]}
        outs = {}
        for rep in range(a.repeats):
            for name, reads in runs.items():
                out = os.path.join(d, "out.bed")
                r = subprocess.run([CLI, "--preset", "chip", "-x", idx, "-r", ref, "-o", out] + reads, capture_output=True, text=True)
                if r.returncode:
                    sys.exit(r.stderr[-2000:])
                outs[name] = os.path.getsize(out)
                keep = [l for l in r.stderr.splitlines() if re.match(r"Mapped all reads in|Mapping phase:", l)]
                lines.append("[%d] %s: %s" % (rep + 1, name, " | ".join(keep)))
        lines.append("output bytes: %s" % outs)
    text = "\n".join(lines) + "\n"
    print(text, end="")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        open(os.path.join(a.out, "bench_cli_files.txt"), "w").write(text)


if __name__ == "__main__":
    main()
