"""Every piece of device work the engine enqueues goes through one of three routines in mcl_3dl_b200/csrc/engine.cu:
launch (a <<<>>> launch), launch_pdl (the NN-field likelihood kernels, cudaLaunchKernelEx with programmatic stream
serialization) and cub_call (one device-wide CUB call, its scratch sized by CUB's own size query).  Each returns the
error of its own launch and counts it once in mcl3dl_kernel_launches, so no call site launches, counts or sizes a CUB
scratch by hand.  These checks read the source; they need no GPU."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENGINE = os.path.join(ROOT, "mcl_3dl_b200", "csrc", "engine.cu")


def code_only(src):
    """src with comments and the contents of string and character literals blanked out (offsets kept)."""
    out, i, n = list(src), 0, len(src)

    def blank(a, b):
        for k in range(a, b):
            if out[k] != "\n":
                out[k] = " "

    while i < n:
        if src.startswith("//", i):
            j = src.find("\n", i)
            j = n if j < 0 else j
            blank(i, j)
            i = j
        elif src.startswith("/*", i):
            j = src.index("*/", i) + 2
            blank(i, j)
            i = j
        elif src[i] in "\"'":
            j = i + 1
            while src[j] != src[i]:
                j += 2 if src[j] == "\\" else 1
            blank(i + 1, j)
            i = j + 1
        else:
            i += 1
    return "".join(out)


SRC = code_only(open(ENGINE).read())


def closing(src, at):
    """Index just past the bracket that closes the one at src[at]."""
    pair = {"(": ")", "{": "}", "[": "]"}[src[at]]
    depth = 0
    for k in range(at, len(src)):
        if src[k] == src[at]:
            depth += 1
        elif src[k] == pair:
            depth -= 1
            if depth == 0:
                return k + 1
    raise AssertionError("unbalanced %r at %d" % (src[at], at))


def body(name):
    """(start, end) of the body of the helper `cudaError_t name(...)`."""
    m = re.search(r"\bcudaError_t\s+%s\s*\(" % name, SRC)
    assert m, "engine.cu defines no helper %s" % name
    start = SRC.index("{", closing(SRC, m.end() - 1))
    return start, closing(SRC, start)


def line(at):
    return SRC.count("\n", 0, at) + 1


def outside(pattern, name):
    a, b = body(name)
    return [line(m.start()) for m in re.finditer(pattern, SRC) if not a <= m.start() < b]


def test_kernels_are_launched_only_by_the_launch_helpers():
    assert re.search(r"<<<", SRC) and re.search(r"\bcudaLaunchKernelEx\b", SRC)
    assert outside(r"<<<", "launch") == [], "<<< outside launch()"
    assert outside(r"\bcudaLaunchKernelEx\b", "launch_pdl") == [], "cudaLaunchKernelEx outside launch_pdl()"


def test_the_launch_counter_is_written_only_by_the_helpers():
    writes = r"->\s*launches\s*(\+\+|--|[-+]?=(?!=))|(\+\+|--)\s*\w+\s*->\s*launches\b"
    assert re.search(writes, SRC)
    assert outside(writes, "counted") == [], "launch counter written outside counted()"
    for helper in ("launch", "launch_pdl", "cub_call"):
        a, b = body(helper)
        assert re.search(r"\bcounted\s*\(\s*eng\s*,", SRC[a:b]), helper


LAMBDA = re.compile(r"\[&\]\s*\(\s*void\s*\*\s*(\w+)\s*,\s*size_t\s*&\s*(\w+)\s*\)\s*\{")


def cub_call_spans():
    a, b = body("cub_call")
    return [(m.end() - 1, closing(SRC, m.end() - 1)) for m in re.finditer(r"\bcub_call\s*\(", SRC) if not a <= m.start() < b]


def test_every_cub_call_goes_through_cub_call():
    """Each cub::Device* call is the body of a lambda (void* t, size_t& b) that passes those two parameters on as the
    scratch and its size (so no call site makes its own size query), and the lambda is an argument of cub_call(...),
    or named and handed to cub_call by that name."""
    spans = cub_call_spans()
    calls = list(re.finditer(r"\bcub::Device\w+::\w+\s*\(", SRC))
    assert len(calls) >= 17
    for m in calls:
        where = "engine.cu:%d" % line(m.start())
        lam = [l for l in LAMBDA.finditer(SRC, 0, m.start()) if closing(SRC, l.end() - 1) > m.start()]
        assert lam, where + ": a CUB call outside a (void* t, size_t& b) lambda"
        lam = lam[-1]
        args = SRC[m.end(): closing(SRC, m.end() - 1) - 1].split(",")
        assert [a.strip() for a in args[:2]] == [lam.group(1), lam.group(2)], where + ": scratch or size not the lambda's"
        if any(a <= lam.start() < b for a, b in spans):
            continue
        named = re.search(r"\bauto\s+(\w+)\s*=\s*$", SRC[:lam.start()])
        assert named, where + ": the lambda is neither inside cub_call(...) nor named"
        assert re.search(r"\bcub_call\s*\(\s*eng\s*,[^;,]*,\s*%s\s*\)" % named.group(1), SRC), \
            where + ": %s never goes to cub_call" % named.group(1)


def test_size_queries_are_made_only_by_the_cub_helpers():
    a, b = body("cub_reserve")
    queries = [line(m.start()) for m in re.finditer(r"\(\s*nullptr\s*,\s*\w+\s*[,)]", SRC) if not a <= m.start() < b]
    assert queries == [], "size queries outside cub_reserve() at lines %s" % queries


@pytest.mark.parametrize("name", ["launch", "launch_pdl", "cub_reserve", "cub_call"])
def test_helpers_neither_allocate_nor_synchronise(name):
    """launch and launch_pdl run inside CUDA-graph captures; cub_call grows its scratch only through DevBuf::reserve."""
    a, b = body(name)
    assert not re.search(r"\bcuda(Malloc|Free|\w*Synchronize)\w*\s*\(", SRC[a:b]), name
