"""The arithmetic-expression kernel on the H100 at its shape, broadcast, alignment and batch edges, against tests/arith_ref.py (bit for
bit; the one transcendental root within the CUDA math library's ULP bounds of a float64 evaluation).  Most of the kernel's control
flow depends on shapes rather than types: the stride table and the `linear` bit built by the planner, the index arithmetic of
broadcast operands, the vector branch (a linear operand, a full thread, an aligned address) against the element-by-element one, and
the spread of 8192-element work items over the samples of a batch.

Through the C-ABI (dalib200ArithCompile / Setup / Launch) on slices of one device allocation filled with 0xA5, whose bytes outside
the outputs must stay so:
  * arith_ref.shape_cases: ranks 0-6, lower-rank operands, two-way broadcasts, size-1 output axes, every subset of broadcast axes at
    rank 4, 16 operands filling the whole stride table, operand shapes that change from sample to sample, per-sample scalars, empty
    and 0-d samples, a batch of empty samples (no launch), volumes around the threads and work items up to 1080p x 3 for every
    output element size, both value files, the FLOAT fast path and the generic one;
  * operands and outputs at byte offsets that break the vector alignment of each element size, aligned and unaligned side by side;
  * 3000 packed samples of random volumes, each with broadcast operands of its own, every 97th empty: the grid loops;
  * one uint8 sample of more than 2^31 elements with a broadcast row and a broadcast column.
Through the pipeline: operand shapes, empty samples and CPU scalars as the front end hands them over."""
import ctypes as C
import os

import numpy as np
import pytest

import arith_ref as ar
import gpu_helpers as g

pytestmark = pytest.mark.gpu


def arith_abi(tree, types, samples, scalar=None, in_off=None, out_off=None, packed=False):
    """Evaluates the expression tree over the samples through the C-ABI.  Tensor operands are packed into one device allocation and
    the outputs into another, filled with g.SENTINEL; in_off(i, k, itemsize) / out_off(i, itemsize) give each buffer's byte offset
    past a 256-byte boundary (or packed: back to back).  Checks that the output shapes are the operands' broadcast shapes and that
    no byte outside the outputs was written.  Returns (outputs as numpy arrays, number of kernel launches)."""
    import torch
    from dali_b200 import capi
    lib = capi.lib()
    nin, n = len(types), len(samples)
    scalar = scalar or [0] * nin
    plan = capi.Plan("Arith", max(n, 1))
    ot = C.c_int32()
    capi.check(lib.dalib200ArithCompile(plan.handle, ar.tree_desc(tree).encode(), nin, (C.c_int32 * nin)(*types),
                                        (C.c_uint8 * nin)(*scalar), None, 0, None, 0, C.byref(ot)))
    arrs = [[np.ascontiguousarray(np.asarray(x, ar.NP[t])).reshape(np.shape(x)) for x, t in zip(s, types)] for s in samples]
    ndims = (C.c_int32 * nin)(*[0 if scalar[k] else arrs[0][k].ndim for k in range(nin)])
    shapes = (C.c_int64 * (n * nin * 6 or 1))()
    scal = (C.c_void_p * (n * nin or 1))()
    for i in range(n):
        for k in range(nin):
            if scalar[k]:
                scal[i * nin + k] = arrs[i][k].ctypes.data
            for a, e in enumerate(arrs[i][k].shape):
                shapes[(i * nin + k) * 6 + a] = e
    osh, ond = (C.c_int64 * (6 * n or 6))(), C.c_int32()
    capi.check(lib.dalib200ArithSetup(plan.handle, n, ndims, shapes, scal, osh, C.byref(ond)))
    out_shapes = [tuple(osh[i * 6 + a] for a in range(ond.value)) for i in range(n)]
    for i in range(n):
        want = np.broadcast_shapes(*[arrs[i][k].shape for k in range(nin) if not scalar[k]])
        assert out_shapes[i] == want, (ar.tree_desc(tree), i, out_shapes[i], want)

    tensors = [(i, k) for i in range(n) for k in range(nin) if not scalar[k]]
    din, ptrs = g.upload_slices([arrs[i][k] for i, k in tensors], [in_off(i, k, arrs[i][k].itemsize) if in_off else 0 for i, k in tensors],
                                packed)
    in_ptrs = (C.c_void_p * (n * nin or 1))()
    for (i, k), p in zip(tensors, ptrs):
        in_ptrs[i * nin + k] = p
    dt = np.dtype(ar.NP[ot.value])
    out = g.SentinelSlices([int(np.prod(s, dtype=np.int64)) * dt.itemsize for s in out_shapes], dt.itemsize,
                           [out_off(i, dt.itemsize) if out_off else 0 for i in range(n)], packed)
    n0 = capi.launch_count()
    capi.check(lib.dalib200ArithLaunch(plan.handle, in_ptrs, (C.c_void_p * (n or 1))(*out.ptrs), capi.stream_handle()))
    torch.cuda.synchronize()
    launches = capi.launch_count() - n0
    outs = [b.view(dt).reshape(s) for b, s in zip(out.read(ar.tree_desc(tree)), out_shapes)]
    return outs, launches


def _check_case(name, tree, types, samples, outs):
    for i, s in enumerate(samples):
        try:
            ar.tree_check(tree, outs[i], s, types)
        except AssertionError as e:
            raise AssertionError(f"{name}: sample {i}, operand shapes {[np.shape(x) for x in s]}: {e}") from None


def test_shape_cases():
    """Every case of arith_ref.shape_cases, the float volume cases with a 1080p x 3 sample, each buffer 256-byte aligned; exactly
    one launch, none for a batch whose samples are all empty."""
    for name, tree, types, scalar, samples in ar.shape_cases(np.random.default_rng(21), big=True):
        outs, launches = arith_abi(tree, types, samples, scalar)
        empty = all(o.size == 0 for o in outs)
        assert launches == (0 if empty else 1), (name, launches)
        _check_case(name, tree, types, samples, outs)


# element offsets that break the vector alignment (4 elements) of every element size
UNALIGNED = (1, 2, 3)


def test_unaligned_inputs_and_outputs():
    """The volume cases (two linear operands beside a broadcast one) with the linear inputs at element offsets 1-3 and the outputs
    aligned, the reverse, and both at different offsets, in one allocation each: the element-by-element branch for loads, for stores,
    and for both, next to the vector branch of the other side."""
    rng = np.random.default_rng(22)
    for name, tree, types, scalar, samples in ar.shape_cases(rng):
        if not name.startswith("volumes"):
            continue
        for mode in ("inputs", "outputs", "both"):
            in_off = (lambda i, k, sz: sz * UNALIGNED[(i + k) % 3] if k < 2 else 0) if mode != "outputs" else None
            out_off = (lambda i, sz: sz * UNALIGNED[(i + 1) % 3]) if mode != "inputs" else None
            outs, _ = arith_abi(tree, types, samples, scalar, in_off, out_off)
            _check_case(f"{name}, unaligned {mode}", tree, types, samples, outs)


def test_every_offset_of_each_element_size():
    """One sample of 97 x 85 = 8192 + 53 elements per element size with the linear input at every element offset 0-7 and the output
    at another (a multiple of the 4-element vector alignment, and each way off it), beside a broadcast row and column."""
    rng = np.random.default_rng(23)
    for t in (ar.U8, ar.F16, ar.F32, ar.I64):
        tree = ("add", ("sub", 0, 1), ("mul", 2, 0))
        samples = [[ar._rand(t, (97, 85), rng), ar._rand(t, (1, 85), rng), ar._rand(t, (97, 1), rng)]]
        for off in range(8):
            outs, _ = arith_abi(tree, [t] * 3, samples, None, lambda i, k, sz: sz * off if k == 0 else 0,
                                lambda i, sz: sz * ((off * 3 + 1) % 8))
            _check_case(f"{ar.NAMES[t]} offset {off}", tree, [t] * 3, samples, outs)


def test_batch_of_many_packed_samples():
    """3000 samples packed back to back (any alignment the element size allows), each with its own row and column operands, every
    97th empty and the first and last empty: more work items than the grid has CTAs on an H100 (132 SMs x 8), so the grid loops and
    the item -> sample search crosses many samples per CTA."""
    rng = np.random.default_rng(24)
    hs, ws = rng.integers(1, 90, 3000), rng.integers(1, 130, 3000)
    ws[::97] = 0
    hs[-1] = 0
    assert int(np.sum((hs * ws + 8191) // 8192)) > 132 * 8
    tree, types = ("add", ("mul", 0, 1), 2), [ar.U8, ar.F32, ar.F32]
    samples = [[ar._rand(ar.U8, (h, w), rng), ar._rand(ar.F32, (1, w), rng), ar._rand(ar.F32, (h, 1), rng)] for h, w in zip(hs, ws)]
    outs, launches = arith_abi(tree, types, samples, packed=True)
    assert launches == 1
    _check_case("3000 packed samples", tree, types, samples, outs)
    # the same batch, integer output: 1-byte elements packed without gaps
    tree, types = ("sub", ("add", 0, 1), 2), [ar.U8, ar.U8, ar.U8]
    samples = [[s[0], ar._rand(ar.U8, s[1].shape, rng), ar._rand(ar.U8, s[2].shape, rng)] for s in samples]
    outs, _ = arith_abi(tree, types, samples, packed=True)
    for i, (s, o) in enumerate(zip(samples, outs)):            # uint8 + - wraps: numpy's uint8 arithmetic is the statement
        assert np.array_equal(o, (s[0] + s[1]) - s[2]), i


def test_sample_of_more_than_2_pow_31_elements():
    """One uint8 sample of (32771, 65537) = 2^31 + 229379 elements: x + row - column, so that the broadcast operands' index
    divisions run on element indices above 2^31.  Checked on the rows around element 2^31, the first and the last work item and
    random rows, reading back only those."""
    import torch
    from dali_b200 import capi
    if os.environ.get("DALIB200_DRYRUN"):
        pytest.skip("4.3 GB of buffers; the host side of this launch is test_shape_cases'")
    H, W = 32771, 65537
    assert H * W > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(25)
    x = torch.randint(0, 256, (H, W), dtype=torch.uint8, device="cuda", generator=g)
    rng = np.random.default_rng(25)
    row, col = ar._rand(ar.U8, (1, W), rng), ar._rand(ar.U8, (H, 1), rng)
    drow, dcol = torch.from_numpy(row).cuda(), torch.from_numpy(col).cuda()
    out = torch.empty((H, W), dtype=torch.uint8, device="cuda")
    plan = capi.Plan("Arith", 1)
    lib = capi.lib()
    ot = C.c_int32()
    capi.check(lib.dalib200ArithCompile(plan.handle, b"sub(add(&0 &1) &2)", 3, (C.c_int32 * 3)(ar.U8, ar.U8, ar.U8), (C.c_uint8 * 3)(),
                                        None, 0, None, 0, C.byref(ot)))
    shapes = (C.c_int64 * 18)(H, W, 0, 0, 0, 0, 1, W, 0, 0, 0, 0, H, 1, 0, 0, 0, 0)
    osh, ond = (C.c_int64 * 6)(), C.c_int32()
    capi.check(lib.dalib200ArithSetup(plan.handle, 1, (C.c_int32 * 3)(2, 2, 2), shapes, None, osh, C.byref(ond)))
    assert ot.value == ar.U8 and ond.value == 2 and tuple(osh[:2]) == (H, W)
    capi.check(lib.dalib200ArithLaunch(plan.handle, capi.ptr_array([x, drow, dcol]), capi.ptr_array([out]), capi.stream_handle()))
    torch.cuda.synchronize()
    mid = 2 ** 31 // W
    rows = sorted({0, mid - 1, mid, mid + 1, H - 2, H - 1, *[int(r) for r in rng.integers(0, H, 4)]})
    idx = torch.tensor(rows, device="cuda")
    got, xs = out[idx].cpu().numpy(), x[idx].cpu().numpy()
    del x, out
    torch.cuda.empty_cache()
    for j, r in enumerate(rows):
        want = ar.evaluate("sub", [ar.evaluate("add", [xs[j], row[0]], [ar.U8, ar.U8]), col[r]], [ar.U8, ar.U8])
        assert np.array_equal(got[j], want), (r, np.flatnonzero(got[j] != want)[:8])


def _run(build, batches):
    """Outputs of a pipeline build(*external_sources) for each batch: [[numpy samples of each output]]."""
    import nvidia.dali as dali
    from nvidia.dali import fn
    nsrc = len(batches[0])
    state = {}

    @dali.pipeline_def(batch_size=max(len(b[0]) for b in batches), num_threads=1, device_id=0, prefetch_queue_depth=1, seed=11)
    def pipe():
        srcs = [fn.external_source(source=(lambda _iteration=None, k=k: state["b"][k]), device="gpu") for k in range(nsrc)]
        return build(*srcs)
    p = pipe()
    p.build()
    res = []
    for b in batches:
        state["b"] = b
        cpu = [o.as_cpu() if hasattr(o, "as_cpu") else o for o in p.run()]
        res.append([[np.asarray(o[i]) for i in range(len(b[0]))] for o in cpu])
    return res


def test_pipeline_operand_shapes_empty_samples_and_scalars():
    """Through fn.external_source and DataNode arithmetic: an operand that is (3,) in some samples and (1,) in others, empty samples
    between non-empty ones, a per-sample CPU scalar from fn.random.uniform beside the broadcast operand, and a batch whose samples
    are all empty (the output shapes still broadcast)."""
    from nvidia.dali import fn, types
    rng = np.random.default_rng(26)
    shapes = [(5, 7, 3), (0, 4, 3), (1, 1, 3), (6, 0, 3), (33, 2, 3)]
    xs = [rng.integers(0, 256, s, dtype=np.uint8) for s in shapes]
    ms = [ar._rand(ar.F32, (3,) if i % 2 else (1,), rng) for i in range(len(shapes))]
    ys = [rng.integers(0, 256, (s[0], 1, 1), dtype=np.uint8) for s in shapes]
    empty = [[np.zeros((0, 4, 3), np.uint8)] * 5, [ar._rand(ar.F32, (3,), rng)] * 5, [np.zeros((0, 1, 1), np.uint8)] * 5]

    def build(x, m, y):
        u = fn.random.uniform(range=(-2.0, 2.0))
        return (fn.cast(x, dtype=types.FLOAT) - m) * u, x - y, u
    (a, b, u), (ae, be, _) = _run(build, [[xs, ms, ys], empty])
    for i in range(len(shapes)):
        uk = np.float32(u[i])
        want = ar.evaluate("mul", [ar.evaluate("sub", [xs[i].astype(np.float32), ms[i]], [ar.F32, ar.F32]), uk], [ar.F32, ar.F32])
        assert ar.same_bits(a[i], want), i
        assert b[i].shape == shapes[i] and np.array_equal(b[i], xs[i] - ys[i]), i
    assert all(o.shape == (0, 4, 3) for o in ae + be), [o.shape for o in ae + be]
