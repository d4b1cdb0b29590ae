"""The launch path of the kernels that are single host/device functions (3-D resize, progressive JPEG), executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc
is preloaded in place of the CUDA runtime -- "device" memory is host memory, copies and memsets really happen, and the launches of
resample3d_pass_kernel / prog_scan_kernel / prog_dc_kernel run on the host, block by block and thread by thread, through the same
host/device functions the device code consists of.  Everything in front of and behind the launch is the library's real code
(descriptor upload, temporaries, stage order, grid-stride loops, wave ranges, arena offsets, the operator and the executor), so the
value comparisons below are real:
  * the whole tests/test_zzy_a_gpu_resize3d.py (C-ABI and fn.resize on DHWC / FDHWC / CDHW / FCDHW) runs with its assertions intact;
  * progressive JPEG batches (alone and mixed with baseline samples, whose kernels are no-ops here) must leave the baseline twin's
    coefficients in the arena and the DC differences the shared dc_scan stage expects, and report truncated / incomplete streams."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul_env(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    stub = str(tmp_path_factory.mktemp("emul") / "cuda_emul_stub.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "cuda_emul_stub.cc"), "-o", stub, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(os.environ, DALIB200_DRYRUN="emul", LD_PRELOAD=stub, EMUL_STUB=stub)


def test_volume_resize_gpu_tests_pass_on_the_emulated_launch_path(emul_env):
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_zzy_a_gpu_resize3d.py"), "-q", "-m", "gpu",
                        "-p", "no:cacheprovider"], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    tail = r.stdout[-3000:] + r.stderr[-2000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) == 6 and "failed" not in r.stdout, tail


PROGRESSIVE = r"""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import conftest                      # DALIB200_DRYRUN=emul: "device" tensors are host memory
import gpu_helpers as g
from dali_b200 import capi
from oracle import pyoracle as po
from test_jpeg_prog_cpu import mcu_order
from test_zzy_c_gpu_jpeg_multiscan import _cases

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
cases = _cases()

def check(streams, twins, plan=None):
    outs, status, plan = g.jpeg_decode(streams, want_coefs=True, plan=plan)
    for i, (s, t) in enumerate(zip(streams, twins)):
        if t is None:
            continue                                  # a baseline sample: its kernels are not emulated
        want = mcu_order(t)
        info = po.jpeg_info(t)
        got = g.jpeg_coefs(plan, i, want.size).reshape(want.shape)
        assert np.array_equal(got[:, 1:], want[:, 1:]), ("AC", i)
        # slot 0 comes from the compact DC array, which (dc_scan not having run) holds the differences in dc_scan's order:
        # per component, MCU by MCU, the component's blocks of an MCU in ascending order
        bpm, hs, vs = sum(h * v for h, v in zip(info["hs"][:info["ncomp"]], info["vs"][:info["ncomp"]])), info["hs"], info["vs"]
        b0 = 0
        for c in range(info["ncomp"]):
            nb = hs[c] * vs[c]
            idx = (np.arange(info["mcux"] * info["mcuy"])[:, None] * bpm + b0 + np.arange(nb)[None, :]).reshape(-1)
            assert np.array_equal(np.cumsum(got[idx, 0].astype(np.int64)), want[idx, 0].astype(np.int64)), ("DC", i, c)
            b0 += nb
        assert status[i] == 0, ("status", i)
    return plan

# a batch of progressive samples only: no unit, no subsequence -- none of the baseline entropy kernels may be launched with an empty grid
plan = check([p for _, p in cases], [b for b, _ in cases])
# the same plan again (arenas reused), then mixed with baseline samples
check([p for _, p in cases[:4]], [b for b, _ in cases[:4]], plan)
check([cases[0][0], cases[3][1], cases[9][0], cases[9][1], cases[2][1], cases[4][0]], [None, cases[3][0], None, cases[9][0], cases[2][0], None])
# truncated inside the last scan / cut between two scans: decoded, with a status
base, prog = cases[3]
last = prog.rfind(b"\xff\xda")
outs, status = g.jpeg_decode([prog, prog[: (last + len(prog)) // 2], prog[: last - 3]])
assert status == [0, 1, 1], status
# sequential frames coded in several scans take the same stage (one wave); the blocks such a scan does not code stay zero
import cv2
from test_jpeg_prog_cpu import multiscan_expected, synth, to_multiscan_baseline, twins
base, _ = twins(synth(97, 61, 611), 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
multi, hblk, wblk = to_multiscan_baseline(base, 5)
outs, status, plan2 = g.jpeg_decode([multi, cases[0][1]], want_coefs=True)
want = multiscan_expected(base, hblk, wblk)
got = g.jpeg_coefs(plan2, 0, want.size).reshape(want.shape)
assert status == [0, 0] and np.array_equal(got[:, 1:], want[:, 1:])
info = po.jpeg_info(base)
b0 = 0
for c in range(3):
    nb = info["hs"][c] * info["vs"][c]
    idx = (np.arange(info["mcux"] * info["mcuy"])[:, None] * 6 + b0 + np.arange(nb)[None, :]).reshape(-1)
    assert np.array_equal(np.cumsum(got[idx, 0].astype(np.int64)), want[idx, 0].astype(np.int64)), ("DC", c)
    b0 += nb
n_scan, n_dc = stub.emul_launch_count(1), stub.emul_launch_count(2)
assert n_scan == 3 * 5 and n_dc == 5, (n_scan, n_dc)        # three waves per launch (the last batch: progressive + sequential), one DC pass
# other encoders' scripts (jpeg_extreme_streams): reordered bands, subset-interleaved DC, ten refinements, restart changes; one launch
# per wave of the batch, and the arena holds what the statement says
import jpeg_extreme_streams as xs
from test_jpeg_prog_scripts_cpu import encode, source
batch, wants = [], []
for layout, h, w, make in [("420", 33, 47, xs.reordered), ("ycck", 24, 17, xs.subset_dc), ("422", 17, 23, lambda n: xs.deep(n, 10)),
                           ("gray", 29, 1, xs.restarts), ("411", 16, 40, xs.single_coefficient)]:
    src = source(layout, h, w, 90, 40 + len(batch))
    script = make(len(src["sampling"]))
    batch.append(encode(src, h, w, script))
    wants.append((xs.expected(h, w, src["sampling"], src["planes"], script), src["sampling"], xs.waves(script)))
outs, status, plan3 = g.jpeg_decode(batch + [cases[0][0]], want_coefs=True)
assert status == [0] * len(status), status
for i, (want, sampling, _) in enumerate(wants):
    got = g.jpeg_coefs(plan3, i, want.size).reshape(want.shape)
    assert np.array_equal(got[:, 1:], want[:, 1:]), ("AC", i)
    bpm, b0 = sum(h * v for h, v in sampling), 0
    for h, v in sampling:
        idx = (np.arange(len(want) // bpm)[:, None] * bpm + b0 + np.arange(h * v)[None, :]).reshape(-1)
        assert np.array_equal(np.cumsum(got[idx, 0].astype(np.int64)), want[idx, 0].astype(np.int64)), ("DC", i)
        b0 += h * v
assert stub.emul_launch_count(1) - n_scan == max(w for *_, w in wants), (stub.emul_launch_count(1) - n_scan, [w for *_, w in wants])
print("progressive-emul-ok")
"""


def test_progressive_jpeg_launch_path_leaves_the_twin_coefficients(emul_env):
    r = subprocess.run([sys.executable, "-c", PROGRESSIVE % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "progressive-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
