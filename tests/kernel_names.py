"""One normal form for the names of the library's __global__ instantiations, shared by the kernel manifest test (names from
cuobjdump, demangled by cu++filt) and the GPU coverage matrix (names from torch.profiler, demangled by the C++ ABI demangler).

The two demanglers write the same kernel differently:
    cu++filt:  void dgr::render_bwd_kernel<(int)1, (int)2, (bool)0, (bool)1>(int, int, ...)
    cxxabi:    void dgr::render_bwd_kernel<1, 2, false, true>(int, int, ...)
Both become  dgr::render_bwd_kernel<1,2,0,1>: no return type, no parameter list, no casts, bools as 0 / 1, no spaces inside the
template argument list; the anonymous namespace is written (anonymous)."""
import re

MANIFEST_SEP = " | "
EXCUSED = "excused: "


def normalize(name: str) -> str:
    s = name.strip()
    s = s.replace("(anonymous namespace)", "(anonymous)").replace("<unnamed>", "(anonymous)")
    if s.startswith("void "):
        s = s[len("void "):]
    # cut the parameter list: the first '(' outside template brackets that is not the (anonymous) namespace
    depth, cut, i = 0, len(s), 0
    while i < len(s):
        c = s[i]
        if s.startswith("(anonymous)", i):
            i += len("(anonymous)")
            continue
        if c == "<":
            depth += 1
        elif c == ">":
            depth -= 1
        elif c == "(" and depth == 0:
            cut = i
            break
        i += 1
    s = s[:cut]
    s = re.sub(r"\((?:int|bool|unsigned int|unsigned|long|char)\)", "", s)
    s = re.sub(r"\btrue\b", "1", s)
    s = re.sub(r"\bfalse\b", "0", s)
    s = re.sub(r"\s*,\s*", ",", s)
    s = re.sub(r"<\s+", "<", s)
    s = re.sub(r"\s+>", ">", s)
    return s.strip()


def is_library_kernel(name: str) -> bool:
    """A normalized name that belongs to this library (torch's own kernels, e.g. the elementwise ops of a loss, do not)."""
    return name.startswith("dgr::") or name.startswith("(anonymous)::debug_geom_kernel")


def read_manifest(path):
    """-> {name: (cells tuple, excuse or None)} from tests/kernel_manifest.txt (comments start with '#')."""
    out = {}
    with open(path) as f:
        for n, line in enumerate(f, 1):
            line = line.strip()
            if not line or line.startswith("#"):
                continue
            name, sep, rest = line.partition(MANIFEST_SEP)
            name, rest = name.strip(), rest.strip()
            if not sep or not rest:
                raise ValueError("%s:%d: expected '<kernel> | <cell ids>' or '<kernel> | excused: <reason>'" % (path, n))
            if name in out:
                raise ValueError("%s:%d: %s listed twice" % (path, n, name))
            if rest.startswith(EXCUSED):
                reason = rest[len(EXCUSED):].strip()
                if not reason:
                    raise ValueError("%s:%d: an excused kernel needs its reason" % (path, n))
                out[name] = ((), reason)
            else:
                out[name] = (tuple(rest.split()), None)
    return out
