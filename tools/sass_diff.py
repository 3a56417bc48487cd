#!/usr/bin/env python3
"""tools/sass_diff.py A.o B.o -> the kernels whose code differs between two builds of the same source (objects, cubins or
libraries; cuobjdump reads all three).

Kernels are paired by demangled name, so the per-file anonymous-namespace hash (_GLOBAL__N__<hash>_..._cu_<hash>) does
not matter.  A pair is equal when `cuobjdump -res-usage` gives the same REG / STACK / SHARED / LOCAL and the
`cuobjdump -sass` listings agree once instruction addresses, encodings and symbol names are stripped.  Prints every
kernel that differs, the kernels found in only one build, and the counts; exits 1 if anything differs."""
import re, subprocess, sys

KEYS = ("REG", "STACK", "SHARED", "LOCAL")


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def kernels(path):
    """{demangled name: (res-usage tuple, stripped SASS lines)}"""
    usage, cur = {}, None
    for line in subprocess.run(["cuobjdump", "-res-usage", path], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "REG:" in line:
            u = dict(re.findall(r"(\w+):(\d+)", line))
            usage[cur] = tuple(u.get(k) for k in KEYS)
            cur = None
    sass, cur = {}, None
    for line in subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            sass[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;?\s*/\* 0x[0-9a-f]+ \*/", line)
        if m and cur:
            sass[cur].append(re.sub(r"`\([^)]*\)", "`(sym)", m.group(1)))  # call / relocation targets
    names = demangle(sorted(set(usage) | set(sass)))
    return {names[n]: (usage.get(n), sass.get(n)) for n in names}


def main():
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    a, b = kernels(sys.argv[1]), kernels(sys.argv[2])
    both = sorted(set(a) & set(b))
    differ = 0
    for k in both:
        (ua, sa), (ub, sb) = a[k], b[k]
        if ua != ub or sa != sb:
            differ += 1
            what = f"res-usage {dict(zip(KEYS, ua or ()))} -> {dict(zip(KEYS, ub or ()))}" if ua != ub else "SASS"
            print(f"differs ({what}, {len(sa or [])} / {len(sb or [])} instructions): {k}")
    for k in sorted(set(a) - set(b)):
        print(f"only in {sys.argv[1]}: {k}")
    for k in sorted(set(b) - set(a)):
        print(f"only in {sys.argv[2]}: {k}")
    only = len(set(a) ^ set(b))
    print(f"{len(both)} kernels paired, {len(both) - differ} identical, {differ} differ, {only} unpaired")
    sys.exit(1 if differ or only else 0)


if __name__ == "__main__":
    main()
