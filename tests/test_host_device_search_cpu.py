"""last_at_most (dali_b200/csrc/host_device.h), the search that maps a flat work item to its descriptor in the batched kernels and in
tools/emul, compiled by g++ and checked against bisect_right(keys, v) - 1: prefix arrays with runs of empty samples at the start, in the
middle and at the end, one sample, sub-ranges that start past 0, uint32_t keys above 2^31 and int64_t keys above 2^32, and a key read
from a descriptor field through a lambda."""
import bisect
import ctypes as C
import os
import random
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DRIVER = r"""
#include <stdint.h>
#include "host_device.h"
using dalib200::last_at_most;
struct Desc { int32_t tag; int64_t first_item; };
extern "C" {
void search_i64(const int64_t *d, int lo, int hi, const int64_t *v, int nv, int *out) {
  for (int k = 0; k < nv; k++) out[k] = last_at_most(d, lo, hi, v[k]);
}
void search_u32(const uint32_t *d, int lo, int hi, const uint32_t *v, int nv, int *out) {
  for (int k = 0; k < nv; k++) out[k] = last_at_most(d, lo, hi, v[k]);
}
void search_desc(const int64_t *firsts, int n, const int64_t *v, int nv, int *out) {
  Desc d[64];
  for (int i = 0; i < n; i++) d[i] = Desc{-1, firsts[i]};
  for (int k = 0; k < nv; k++) out[k] = last_at_most(d, 0, n - 1, v[k], [](const Desc &s) { return s.first_item; });
}
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    tmp = tmp_path_factory.mktemp("search")
    src, out = tmp / "search.cc", str(tmp / "libsearch.so")
    src.write_text(DRIVER)
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-shared", "-fPIC",
                        "-I" + os.path.join(ROOT, "dali_b200", "csrc"), str(src), "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return C.CDLL(out)


def expect(keys, lo, hi, v):
    return max(lo, bisect.bisect_right(keys, v, lo, hi + 1) - 1)


def run(lib, fn, ctype, keys, lo, hi, vs):
    d, q, out = (ctype * len(keys))(*keys), (ctype * len(vs))(*vs), (C.c_int * len(vs))()
    getattr(lib, fn)(d, lo, hi, q, len(vs), out)
    return list(out)


def prefix(sizes):
    firsts, t = [], 0
    for s in sizes:
        firsts.append(t)
        t += s
    return firsts, t


def sizes_with_empty_runs(rng, n):
    sizes = [rng.randint(1, 9) for _ in range(n)]
    for a, b in ((0, rng.randint(1, 3)), (n // 2, n // 2 + rng.randint(1, 4)), (n - rng.randint(1, 3), n)):
        for i in range(max(a, 0), min(b, n)):
            sizes[i] = 0
    for i in rng.sample(range(n), n // 5):
        sizes[i] = 0
    assert len(sizes) == n
    return sizes


def check(lib, fn, ctype, keys, lo, hi, vs):
    got = run(lib, fn, ctype, keys, lo, hi, vs)
    want = [expect(keys, lo, hi, v) for v in vs]
    assert got == want, (fn, keys, lo, hi, [(v, g, w) for v, g, w in zip(vs, got, want) if g != w][:5])


def test_prefix_arrays_skip_empty_samples(lib):
    rng = random.Random(1)
    for n in list(range(2, 20)) + [31, 32, 33, 64]:
        for _ in range(8):
            sizes = sizes_with_empty_runs(rng, n)
            keys, total = prefix(sizes)
            vs = list(range(total + 3))
            check(lib, "search_i64", C.c_int64, keys, 0, n - 1, vs)
            got = run(lib, "search_i64", C.c_int64, keys, 0, n - 1, vs[:total])
            # every item lands in the sample that holds it, which is never an empty one
            assert all(sizes[i] > 0 and keys[i] <= v < keys[i] + sizes[i] for v, i in zip(vs, got))


def test_one_sample(lib):
    for first in (0, 5):
        check(lib, "search_i64", C.c_int64, [first], 0, 0, [0, first, first + 1, 1 << 40])
        check(lib, "search_u32", C.c_uint32, [first], 0, 0, [0, first, first + 1, 0xFFFFFFFF])


def test_sub_range_past_zero(lib):
    rng = random.Random(2)
    for _ in range(200):
        n = rng.randint(2, 40)
        keys, total = prefix(sizes_with_empty_runs(rng, n))
        lo = rng.randint(1, n - 1)
        hi = rng.randint(lo, n - 1)
        # items before keys[lo] have no match in the range and return lo
        check(lib, "search_i64", C.c_int64, keys, lo, hi, list(range(total + 2)))


def test_key_widths(lib):
    rng = random.Random(3)
    for _ in range(50):
        n = rng.randint(1, 48)
        base = rng.randint(0x80000000, 0xFFFFFFFF - 9 * n)
        keys = [base + f for f in prefix(sizes_with_empty_runs(rng, n) if n > 1 else [3])[0]]
        vs = [0, 0x7FFFFFFF, base - 1, 0xFFFFFFFF] + [rng.randint(base, keys[-1] + 9) for _ in range(64)]
        check(lib, "search_u32", C.c_uint32, keys, 0, n - 1, vs)
        keys64 = [(1 << 33) + k for k in keys]
        vs64 = [0, (1 << 33) - 1, 1 << 62] + [(1 << 33) + v for v in vs]
        check(lib, "search_i64", C.c_int64, keys64, 0, n - 1, vs64)


def test_key_from_descriptor_field(lib):
    rng = random.Random(4)
    for _ in range(100):
        n = rng.randint(1, 64)
        keys, total = prefix(sizes_with_empty_runs(rng, n) if n > 1 else [rng.randint(0, 5)])
        vs = list(range(total + 2))
        d, q, out = (C.c_int64 * n)(*keys), (C.c_int64 * len(vs))(*vs), (C.c_int * len(vs))()
        lib.search_desc(d, n, q, len(vs), out)
        assert list(out) == [expect(keys, 0, n - 1, v) for v in vs]
