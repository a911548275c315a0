"""Compare the SASS of two builds of libdgr_b200.so, kernel by kernel (no GPU needed: cuobjdump reads the files).

For every kernel in either library it prints whether the instruction text is identical, ignoring addresses, encodings and the
anonymous-namespace hash in mangled names, plus registers and stack before -> after; then a summary line.  This is the recipe
behind DESIGN.md's statements that a change leaves kernels instruction-for-instruction the same.

    python tools/sass_compare.py OLD/libdgr_b200.so NEW/libdgr_b200.so [--all]
"""
import argparse
import re
import shutil
import subprocess

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
ANON = re.compile(r"\d*_GLOBAL__N__[0-9a-f]+_\d+_(\w+?)_[0-9a-f]{8}")


def _run(*args):
    return subprocess.run([CUOBJDUMP, *args], stdout=subprocess.PIPE, check=True, text=True).stdout


def kernels(path):
    """{kernel: (instruction list, registers, stack bytes)}"""
    sass, name = {}, None
    for line in _run("-sass", path).splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = ANON.sub(r"_GLOBAL__N__\1", m.group(1))
            sass[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(.*?)\s*;", line)
        if m and name:
            sass[name].append(ANON.sub(r"_GLOBAL__N__\1", " ".join(m.group(1).split())))
    res, name = {}, None
    for line in _run("--dump-resource-usage", path).splitlines():
        m = re.match(r"\s*Function\s+(\S+?):?\s*$", line)
        if m:
            name = ANON.sub(r"_GLOBAL__N__\1", m.group(1))
        m = re.search(r"REG:(\d+)\s+STACK:(\d+)", line)
        if m and name:
            res[name] = (int(m.group(1)), int(m.group(2)))
    return {k: (v, *res.get(k, (-1, -1))) for k, v in sass.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--all", action="store_true", help="also list the identical kernels")
    a = ap.parse_args()
    old, new = kernels(a.old), kernels(a.new)
    same = 0
    for k in sorted(set(old) | set(new)):
        if k not in old or k not in new:
            print("%-8s %s" % ("only-new" if k in new else "only-old", k))
            continue
        (io, ro, so), (i_n, rn, sn) = old[k], new[k]
        same += io == i_n
        if io != i_n or a.all:
            d = "identical" if io == i_n else "differs %d -> %d instr" % (len(io), len(i_n))
            print("%-28s reg %3d -> %3d  stack %4d -> %4d  %s" % (d, ro, rn, so, sn, k))
    both = len(set(old) & set(new))
    print("summary: %d kernels in both, %d identical, %d differ, %d only old, %d only new"
          % (both, same, both - same, len(set(old) - set(new)), len(set(new) - set(old))))


if __name__ == "__main__":
    main()
