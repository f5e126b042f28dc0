#!/usr/bin/env python
"""Compare the SASS of the kernels in two object files / shared libraries instruction by instruction.

    python tools/sass_equal.py OLD.o NEW.o [--appended TYPE ...] [--tparam TYPE ...] [substring ...]

Used when a change must leave GPU-validated kernels untouched (no GPU at hand): template parameters with a `false` default are
folded away, so `kernel<3>` in OLD is matched with `kernel<3, false>` in NEW, and a kernel that only gained that parameter
(`kernel` -> `kernel<false>`) with its old self.  --appended TYPE folds away a trailing parameter of struct type TYPE that NEW's
kernels gained (`kernel(a, b)` -> `kernel(a, b, TYPE)`); such a kernel's SASS can only be identical when the instance ignores it.
--tparam TYPE folds away a trailing template argument TYPE that NEW's kernels gained as a defaulted class parameter
(`kernel<3>` -> `kernel<3, TYPE>`).
Exit code 1 if any matched kernel differs or is missing."""
import re
import subprocess
import sys


def functions(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); funcs[cur] = []; continue
        if cur and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            funcs[cur].append(re.sub(r"\s+", " ", re.sub(r"/\*.*?\*/", "", line)).strip())
    return funcs


def main():
    old, new = functions(sys.argv[1]), functions(sys.argv[2])
    rest, appended, tparams = sys.argv[3:], [], []
    for opt, into in (("--appended", appended), ("--tparam", tparams)):
        while opt in rest:
            i = rest.index(opt)
            into.append(rest[i + 1]); del rest[i:i + 2]
    want = rest
    tails = [f"{len(t)}{t}" for t in appended]

    def strip(kk):
        for t in tparams:
            kk = kk.replace(f"{len(t)}{t}E", "E")
        return kk

    def fold(kk):
        kk = re.sub(r"I(Lb0E)+Ev", "", re.sub(r"(ELb0)+EE", "EE", kk))
        for t in tails:
            if kk.endswith(t):
                kk = kk[:-len(t)]
        return kk
    bad = 0
    for k, v in sorted(old.items()):
        if want and not any(w in k for w in want):
            continue
        match = [kk for kk in new if k in (kk, fold(kk), strip(kk), fold(strip(kk)))]
        if not match:
            print(f"{k[:70]:70s} MISSING in {sys.argv[2]}"); bad += 1; continue
        same = v == new[match[0]]
        bad += 0 if same else 1
        print(f"{k[:70]:70s} {'identical' if same else 'DIFFERENT'} ({len(v)} instructions)")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
