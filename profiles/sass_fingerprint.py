#!/usr/bin/env python
"""Per-kernel SASS fingerprints of a built library (addresses stripped), to tell whether an edit touched a kernel's code.

    python profiles/sass_fingerprint.py [lib.so] > profiles/sass_fingerprint.txt
    python profiles/sass_fingerprint.py --diff profiles/sass_fingerprint.txt [lib.so]
"""
import hashlib
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT = os.path.join(ROOT, "mcl_3dl_b200", "libmcl3dl_b200.so")
# nvcc names a translation unit's anonymous namespace after hashes of its source path: strip them, so that the same
# code built in another directory has the same names
ANON_NS = re.compile(r"_GLOBAL__N__[0-9a-f]{8}_(\d+_\w*?)_[0-9a-f]{8}")


def _stable(text):
    return ANON_NS.sub(r"_GLOBAL__N__\1", text)


def fingerprints(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = _stable(m.group(1))
            funcs[cur] = hashlib.sha256()
            continue
        if cur:
            funcs[cur].update(_stable(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line)).encode())
    return {k: v.hexdigest()[:16] for k, v in funcs.items()}


if __name__ == "__main__":
    args = sys.argv[1:]
    if args and args[0] == "--diff":
        old = dict(line.split() for line in open(args[1]) if line.strip() and not line.startswith("#"))
        new = fingerprints(args[2] if len(args) > 2 else DEFAULT)
        for k in sorted(set(old) | set(new)):
            if old.get(k) != new.get(k):
                print(("changed " if k in old and k in new else "added   " if k in new else "removed ") + k)
        print("# %d kernels, %d identical" % (len(new), sum(1 for k in new if old.get(k) == new[k])))
    else:
        fp = fingerprints(args[0] if args else DEFAULT)
        print("# <kernel> <sha256[:16] of its SASS text (cuobjdump -sass, addresses stripped)>")
        for k in sorted(fp):
            print(k, fp[k])
