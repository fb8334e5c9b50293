"""Compare the SASS of every kernel in two builds of libchromap_b200.so, function by function:
    python tools/sass_compare.py OLD.so NEW.so
Each function's `cuobjdump -sass` text is compared with its instruction addresses removed. The SAM emit kernels and
`sam_span` became templates on the read length, so their 160-base instances (mangled `...ILi160EE...`) are matched to the
plain names of a build from before that change, with the template argument stripped from their names and from the calls
inside other functions. Prints the functions that differ, those only in OLD, those only in NEW; exits 1 if any differ or are
missing from NEW."""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def functions(lib):
    out = subprocess.run([CUOBJDUMP, "-sass", lib], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", out)
    return {name: re.sub(r"/\*[0-9a-f]{4,}\*/", "", body) for name, body in zip(parts[1::2], parts[2::2])}


def plain(name):
    """A 160-base template instance under the name its function had before it was a template."""
    name = re.sub(r"^(_Z\d+(?:emit_sam_kernel|emit_sam_se_kernel))ILi160EEv", r"\1", name)
    return re.sub(r"^(_Z8sam_span)ILi160EE", r"\1", name)


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    new_plain = {plain(n): re.sub(r"_Z8sam_spanILi160EE", "_Z8sam_span", b) for n, b in new.items()}
    differ = [n for n in old if n in new_plain and old[n] != new_plain[n]]
    missing = [n for n in old if n not in new_plain]
    added = [n for n in new if plain(n) not in old]
    print("same: %d, differ: %s, only in old: %s, only in new: %s" % (len(old) - len(differ) - len(missing), differ, missing, added))
    return 1 if differ or missing else 0


if __name__ == "__main__":
    sys.exit(main())
