"""CPU tests of the 3-D (DHWC) resize: (1) the plain-C oracle against the committed golden vectors of the reference's
SeparableResampleCPU<.., 3> and, where oracle/_ref is built, against the compiled reference on random sweeps; (2) the PRODUCT's planner
and per-element function (dali_b200/csrc/resample3d_plan.h + resample3d_core.h -- the body of the CUDA kernel) compiled for the host by
tools/emul/resample3d_emul.cc and compared bit for bit with the oracle.  No GPU and no device code runs here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from dali_b200 import capi
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILTERS = [po.F_NN, po.F_LINEAR, po.F_TRIANGULAR, po.F_GAUSSIAN, po.F_CUBIC, po.F_LANCZOS3]


def _golden_cases(golden_dir):
    g = np.load(os.path.join(golden_dir, "resample3d_ref.npz"))
    n = len([k for k in g.files if k.startswith("in_")])
    for i in range(n):
        m = [int(v) for v in g[f"meta_{i}"]]
        out = tuple(m[0:3])
        fmin = [(m[3 + 2 * d], m[4 + 2 * d], 0.0) for d in range(3)]
        fmag = [(m[9 + 2 * d], m[10 + 2 * d], 0.0) for d in range(3)]
        order = m[15:18]
        r = g[f"roi_{i}"]
        roi = None if np.isnan(r[0]) else ([float(v) for v in r[0:3]], [float(v) for v in r[3:6]])
        yield i, g, out, fmin, fmag, roi, order


def random_case(rng, it):
    D, H, W = [int(rng.integers(1, 14)) for _ in range(3)]
    if it % 5 == 0:
        W = int(rng.integers(10, 40))
    Cn = int(rng.choice([1, 2, 3, 4]))
    out = [int(rng.integers(1, 16)) for _ in range(3)]
    if it % 7 == 0:
        out[2] = int(rng.integers(16, 50))          # wide rows: the 16-lane half-to-even groups of the u8 stores
    if it % 11 == 0:
        out = [max(1, D // 2), max(1, H // 2), max(1, W // 2)]      # exact 2x: .5 ties
    dt = np.uint8 if rng.random() < 0.6 else np.float32
    vol = rng.uniform(0, 255, (D, H, W, Cn)).astype(dt)
    odt = dt if rng.random() < 0.6 else np.float32
    def f():
        return (int(rng.choice(FILTERS)), int(rng.integers(0, 2)), 0.0)
    if rng.random() < 0.5:
        a, b = f(), f()
        fmin, fmag = [a] * 3, [b] * 3
    else:
        fmin, fmag = [f() for _ in range(3)], [f() for _ in range(3)]
    roi = None
    has_nn = any(x[0] == po.F_NN for x in fmin + fmag)
    if rng.random() < 0.4 and not has_nn:     # the reference's NN pass reads past a cropped ROI (resampling_impl_cpu.h:534-571): excluded
        lo, hi = [], []
        for s in (D, H, W):
            a, b = float(rng.uniform(0, s * 0.5)), float(rng.uniform(s * 0.5, s))
            if rng.random() < 0.2:
                a, b = b, a
            if rng.random() < 0.3:
                a = b = None
            lo.append(a)
            hi.append(b)
        roi = (lo, hi)
    return vol, tuple(out), fmin, fmag, odt, roi


def test_oracle_against_golden(golden_dir):
    for i, g, out, fmin, fmag, roi, order in _golden_cases(golden_dir):
        vol = g[f"in_{i}"]
        o8, o = po.resample3d(vol, out, fmin, fmag, np.uint8, roi, want_order=True)
        assert o == order, f"pass order, case {i}"
        assert np.array_equal(o8, g[f"out_u8_{i}"]), f"u8 case {i}"
        of = po.resample3d(vol, out, fmin, fmag, np.float32, roi)
        assert np.array_equal(of.view(np.uint32), g[f"out_f32_{i}"].view(np.uint32)), f"u8->f32 case {i}"
        volf = (vol.astype(np.float32) * 1.37 - 20).astype(np.float32)
        off = po.resample3d(volf, out, fmin, fmag, np.float32, roi)
        assert np.array_equal(off.view(np.uint32), g[f"out_f32f32_{i}"].view(np.uint32)), f"f32 case {i}"


@pytest.mark.skipif(not po.have_ref(), reason="oracle/_ref not built (no /root/reference)")
def test_oracle_against_compiled_reference():
    rng = np.random.default_rng(21)
    for it in range(250):
        vol, out, fmin, fmag, odt, roi = random_case(rng, it)
        a, oa = po.resample3d(vol, out, fmin, fmag, odt, roi, want_order=True)
        b, ob = po.ref_resample3d(vol, out, fmin, fmag, odt, roi, want_order=True)
        assert oa == ob, (it, vol.shape, out, fmin, fmag, roi)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (it, vol.shape, out, fmin, fmag, roi)


# ---- the product's planner + kernel body, compiled for the host -------------------------------------------------------------------
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emul") / "libr3emul.so")
    cmd = ["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
           os.path.join(ROOT, "tools", "emul", "resample3d_emul.cc"), "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(out)


def fill_sample(s, shape, out, fmin, fmag, roi):
    for d in range(3):
        s.in_shape[d], s.out_shape[d] = int(shape[d]), int(out[d])
        s.min_filter[d] = capi.FilterDesc(int(fmin[d][0]), int(fmin[d][1]), float(fmin[d][2]))
        s.mag_filter[d] = capi.FilterDesc(int(fmag[d][0]), int(fmag[d][1]), float(fmag[d][2]))
        if roi is not None and roi[0][d] is not None:
            s.use_roi[d], s.roi_start[d], s.roi_end[d] = 1, roi[0][d], roi[1][d]
    s.channels = int(shape[3])


def run_emul(lib, vol, out, fmin, fmag, odt, roi):
    s = capi.Resample3DSample()
    fill_sample(s, vol.shape, out, fmin, fmag, roi)
    res = np.empty(tuple(out) + (vol.shape[3],), odt)
    order = (C.c_int * 3)()
    dt = lambda t: capi.UINT8 if np.dtype(t) == np.uint8 else capi.FLOAT
    rc = lib.emul_resample3d(C.byref(s), dt(vol.dtype), dt(odt), vol.ctypes.data_as(C.c_void_p), res.ctypes.data_as(C.c_void_p), order)
    assert rc == 0, rc
    return res, list(order)


def test_kernel_body_on_host_against_golden(emul, golden_dir):
    for i, g, out, fmin, fmag, roi, order in _golden_cases(golden_dir):
        vol = np.ascontiguousarray(g[f"in_{i}"])
        o8, o = run_emul(emul, vol, out, fmin, fmag, np.uint8, roi)
        assert o == order, f"pass order, case {i}"
        assert np.array_equal(o8, g[f"out_u8_{i}"]), f"u8 case {i}"
        of, _ = run_emul(emul, vol, out, fmin, fmag, np.float32, roi)
        assert np.array_equal(of.view(np.uint32), g[f"out_f32_{i}"].view(np.uint32)), f"u8->f32 case {i}"
        volf = (vol.astype(np.float32) * 1.37 - 20).astype(np.float32)
        off, _ = run_emul(emul, volf, out, fmin, fmag, np.float32, roi)
        assert np.array_equal(off.view(np.uint32), g[f"out_f32f32_{i}"].view(np.uint32)), f"f32 case {i}"


def test_kernel_body_on_host_random_sweep(emul):
    rng = np.random.default_rng(22)
    for it in range(300):
        vol, out, fmin, fmag, odt, roi = random_case(rng, it)
        vol = np.ascontiguousarray(vol)
        a, oa = run_emul(emul, vol, out, fmin, fmag, odt, roi)
        b, ob = po.resample3d(vol, out, fmin, fmag, odt, roi, want_order=True)
        assert oa == ob, (it, vol.shape, out, fmin, fmag, roi)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (it, vol.shape, out, fmin, fmag, roi)


HOSTILE = r"""
import ctypes as C, sys
sys.path.insert(0, %r)
from dali_b200 import capi
sys.path.insert(0, %r)
from test_resample3d_cpu import fill_sample
lib = capi.lib()
plan = capi.Plan("Resample3D", 4)
s = (capi.Resample3DSample * 1)()
fill_sample(s[0], (4, 4, 4, 1), (2, 2, 2), [(1, 1, 0.0)] * 3, [(1, 0, 0.0)] * 3, None)
setup = lambda n=1, i=capi.UINT8, o=capi.UINT8: lib.dalib200Resample3DPlanSetup(plan.handle, n, s, i, o)
assert setup() == 0
order = (C.c_int32 * 3)()
assert lib.dalib200Resample3DPlanGetOrder(plan.handle, 0, order) == 0 and sorted(order) == [0, 1, 2]
assert setup(i=capi.FLOAT, o=capi.UINT8) == 1          # f32 -> u8 is not a combination the reference instantiates
assert setup(n=5) == 1                                 # over capacity
for v in (0, 17):
    s[0].channels = v
    assert setup() == 1
s[0].channels = 1
s[0].in_shape[0] = 0
assert setup() == 1
s[0].in_shape[0] = 1 << 30; s[0].in_shape[1] = 1 << 10
assert setup() == 1                                    # 2^31 elements or more
s[0].in_shape[0] = 4; s[0].in_shape[1] = 4
s[0].min_filter[1].type = 9
assert setup() == 1
s[0].min_filter[1].type = 1
s[0].use_roi[2], s[0].roi_start[2], s[0].roi_end[2] = 1, float("nan"), 3.0
assert setup() == 1
s[0].use_roi[2] = 0
s[0].out_shape[1] = 0                                  # an empty output is fine
assert setup() == 0
assert lib.dalib200Resample3DLaunch(plan.handle, (C.c_void_p * 1)(0x1000), (C.c_void_p * 1)(0x2000), None) == 0
print("hostile-ok")
"""


def test_plan_rejects_hostile_arguments(tmp_path):
    """Argument validation of the C-ABI (plan creation needs a CUDA event: the runtime is replaced by tools/fuzz/cuda_stub.c)."""
    stub = str(tmp_path / "cuda_stub.so")
    r = subprocess.run(["gcc", "-shared", "-fPIC", "-O1", "-o", stub, os.path.join(ROOT, "tools", "fuzz", "cuda_stub.c")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    env = dict(os.environ, LD_PRELOAD=stub)
    r = subprocess.run([os.sys.executable, "-c", HOSTILE % (ROOT, os.path.join(ROOT, "tests"))], capture_output=True, text=True, env=env, cwd=ROOT, timeout=300)
    assert r.returncode == 0 and "hostile-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-3000:])
