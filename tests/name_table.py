"""The decode kernel's name table (csrc/sse_tables.h: build_tables, name_lookup) on the host: the struct-tag names and
finish_reason values as the library declares them, a Python restatement of the perfect hash, and a small host program that runs
the header's own lookup over a list of strings."""
import os
import re
import shutil
import subprocess

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "inference_gateway_b200", "csrc")
NHASH_BITS = 7


def schema_names():
    """[(node, name)] of the schema in declaration order (csrc/sse_common.cuh c_schema)."""
    src = open(os.path.join(CSRC, "sse_common.cuh")).read()
    body = src[src.index("__constant__ Schema c_schema"):]
    body = body[:body.index("/* first */")]
    names = re.findall(r'FD\("(\w+)"', body)
    first = [int(x) for x in re.search(r"/\* first \*/ \{([^}]*)\}", src).group(1).split(",")]
    cnt = [int(x) for x in re.search(r"/\* cnt   \*/ \{([^}]*)\}", src).group(1).split(",")]
    node_of = {}
    for node, (f, c) in enumerate(zip(first, cnt)):
        for k in range(f, f + c):
            node_of[k] = node
    return [(node_of[i], n) for i, n in enumerate(names)]


def finish_names():
    src = open(os.path.join(CSRC, "sse_kernel2.cu")).read()
    return re.findall(r'"(\w+)"', re.search(r"fin_names\[\] = \{([^}]*)\}", src).group(1))


def table_names():
    """The distinct names in the order build_tables assigns their ids."""
    out = []
    for n in [n for _, n in schema_names()] + finish_names():
        if n not in out:
            out.append(n)
    return out


def fold(b: bytes) -> bytes:
    return bytes(c | 0x20 if 0x41 <= c <= 0x5A else c for c in b)


def name_hash(mul: int, body: bytes) -> int:
    w0 = int.from_bytes(fold(body[:4]).ljust(4, b"\0"), "little")
    return ((w0 * mul + len(body) * 0x9E3779B1) & 0xFFFFFFFF) >> (32 - NHASH_BITS)


def hash_mul(names) -> int:
    """The first odd multiplier under which the names fall into distinct slots (build_tables' search)."""
    mul = 0x9E3779B1
    for _ in range(100000):
        slots = {name_hash(mul, n.encode()) for n in names}
        if len(slots) == len(names):
            return mul
        mul = (mul + 0x632BE5AB * 2) & 0xFFFFFFFF
    raise AssertionError("no perfect hash")


HARNESS = r"""
#include <stdio.h>
#include <stdlib.h>
#include <initializer_list>
#include "sse_tables.h"
using namespace ssetab;
// argv: schema names, "--", finish names. stdin: one string per line. stdout: the multiplier, then "id upper" per string.
int main(int argc, char **argv) {
    static FieldSrc fs[64]; static const char *fin[16]; static uint8_t fv[16];
    int nf = 0, nfin = 0, i = 1;
    for (; i < argc && strcmp(argv[i], "--"); i++) { fs[nf].node = 1; fs[nf].name = argv[i]; fs[nf].ty = 1; nf++; }
    for (i++; i < argc; i++) { fin[nfin] = argv[i]; fv[nfin] = (uint8_t)(nfin + 1); nfin++; }
    static DfaTables T;
    if (build_tables(T, fs, nf, fin, fv, nfin) != 0) { printf("build failed\n"); return 1; }
    printf("%u\n", T.nhash_mul);
    static char line[4096];
    while (fgets(line, sizeof line, stdin)) {
        uint32_t n = (uint32_t)strlen(line);
        if (n && line[n - 1] == '\n') line[--n] = 0;
        bool upper = false;
        const uint32_t id = name_lookup(T, n, [&](uint32_t k) { uint32_t w = 0; memcpy(&w, line + k, 4); return w; }, upper);
        printf("%u %d\n", id, upper ? 1 : 0);
    }
    return 0;
}
"""


def build_harness(tmpdir) -> str:
    cxx = shutil.which("c++") or shutil.which("g++") or shutil.which("clang++")
    assert cxx, "no C++ compiler"
    src = os.path.join(tmpdir, "name_table.cpp")
    exe = os.path.join(tmpdir, "name_table")
    with open(src, "w") as f:
        f.write(HARNESS)
    subprocess.run([cxx, "-std=c++17", "-O1", "-I", CSRC, "-o", exe, src], check=True)
    return exe


def lookup(exe, strings):
    """(multiplier, [(name id or 0xFF, upper)]) of the header's name_lookup over strings (bytes without '\\n' or NUL)."""
    names = [n for _, n in schema_names()]
    inp = b"".join(s + b"\n" for s in strings)
    out = subprocess.run([exe] + names + ["--"] + finish_names(), input=inp, capture_output=True, check=True).stdout.split(b"\n")
    res = [tuple(int(x) for x in ln.split()) for ln in out[1:1 + len(strings)]]
    return int(out[0]), res
