"""The host build of fn.reductions.* (tools/emul/reduce_emul.cc: the planner of csrc/reduce_plan.h and the kernel bodies of
csrc/reduce_core.h compiled with g++), shared by tests/test_reduce_cpu.py and tests/test_gpu_reduce_exact.py: `build` compiles it,
`run` plans and runs one batch through it with every input, mean and output at a chosen element offset past a 16-byte boundary."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np

import reduce_ref as rr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "reduce_emul.cc")


def build(tmpdir):
    """the host build as a ctypes library in `tmpdir`, or None without g++"""
    if shutil.which("g++") is None:
        return None
    so = os.path.join(str(tmpdir), "reduce_emul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", SRC, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def placed(x, off, keep):
    """x's bytes at element offset `off` past a 16-byte boundary of a fresh buffer (kept alive in `keep`)"""
    buf = np.zeros(x.nbytes + 48, np.uint8)
    base = (-buf.ctypes.data) % 16 + off * x.itemsize
    buf[base:base + x.nbytes] = np.frombuffer(np.ascontiguousarray(x).tobytes(), np.uint8)
    keep.append(buf)
    return buf.ctypes.data + base


def run(lib, op, xs, axes=None, keep_dims=False, dtype=None, ddof=0, means=None, off=0, moff=0, ooff=0):
    """-> (outputs, kinds [sample][pass], depths) or (None, message, None).  Sample i's input sits (off + 3 i) % (16 / size) elements
    past a 16-byte boundary, its mean (moff + i) % 4 and its output (ooff + i) % (16 / size) elements past one."""
    n, nd = len(xs), xs[0].ndim
    ax = rr._axes(xs[0], axes) if nd else ()
    mask = sum(1 << a for a in ax)
    shp = (C.c_int64 * max(1, n * nd))(*[e for x in xs for e in x.shape])
    ond = nd if keep_dims else nd - len(ax)
    osh = (C.c_int64 * max(1, n * ond))()
    ot = C.c_int32()
    kinds = (C.c_int32 * (3 * n))()
    depths = (C.c_int64 * n)()
    err = C.create_string_buffer(512)
    args = (op, rr.CODE[xs[0].dtype], -1 if dtype is None else dtype, n, nd, shp, mask, int(keep_dims), ddof)
    if lib.emul_reduce(*args, None, None, None, osh, C.byref(ot), kinds, depths, err, 512):
        return None, err.value.decode(), None
    keep = []
    ip = (C.c_void_p * n)(*[placed(x, (off + 3 * i) % (16 // x.itemsize), keep) for i, x in enumerate(xs)])
    mp = None if means is None else (C.c_void_p * n)(*[placed(np.asarray(m, np.float32), (moff + i) % 4, keep) for i, m in enumerate(means)])
    ots = np.dtype(rr.TYPES[ot.value])
    outs, optrs = [], []
    for i in range(n):
        shape = tuple(osh[i * ond + a] for a in range(ond))
        nbytes = int(np.prod(shape, dtype=np.int64)) * ots.itemsize
        buf = np.full(nbytes + 64, 0xA5, np.uint8)
        base = (-buf.ctypes.data) % 16 + 16 + (ooff + i) % (16 // ots.itemsize) * ots.itemsize
        outs.append((buf, base, shape))
        optrs.append(buf.ctypes.data + base)
    assert lib.emul_reduce(*args, ip, mp, (C.c_void_p * n)(*optrs), osh, C.byref(ot), kinds, depths, err, 512) == 0
    res = []
    for buf, base, shape in outs:
        nbytes = int(np.prod(shape, dtype=np.int64)) * ots.itemsize
        assert np.all(buf[:base] == 0xA5) and np.all(buf[base + nbytes:] == 0xA5), "a write outside the output"
        res.append(np.frombuffer(buf[base:base + nbytes].tobytes(), ots).reshape(shape))
    return res, [list(kinds[3 * i:3 * i + 3]) for i in range(n)], list(depths)
