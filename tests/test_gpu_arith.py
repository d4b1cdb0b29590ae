"""Arithmetic expressions on DataNodes, nvidia.dali.math and fn.cast on the H100, against tests/arith_ref.py:
  * every operator over every type pair of the 12 types (clamp over a set of triples), on edge values and random values, in a
    non-uniform batch: bit for bit where the result is exact (+ - * / // ** of integers, sqrt, rsqrt, floor, ceil, comparisons,
    bitwise, min / max / clamp, casts), the float transcendentals within the CUDA math library's documented ULP bounds of a float64
    evaluation;
  * broadcasting ((img - mean) / std with mean of shape (3,)), sequences with their FHWC layout, CPU per-sample scalars;
  * a fused chain bit-identical to the same chain with every step materialised, in one launch;
  * fn.cast saturation and rounding against pointwise_ref's ConvertSat;
  * the result read through DALIGenericIterator as a torch tensor, and the failing sample named in a broadcast error."""
import numpy as np
import pytest

import arith_ref as ar
import pointwise_ref as pr

pytestmark = pytest.mark.gpu

UNARY = ("plus", "minus", "abs") + tuple(f for f in ar.FLOAT_FUNCS if ar.ARITY[f] == 1)
BINARY = ("add", "sub", "mul", "fdiv", "div", "pow", "fpow", "min", "max", "atan2") + ar.CMP + ("bitand", "bitor", "bitxor")
PY = {"add": "+", "sub": "-", "mul": "*", "fdiv": "/", "div": "//", "pow": "**", "eq": "==", "neq": "!=", "lt": "<", "leq": "<=",
      "gt": ">", "geq": ">=", "bitand": "&", "bitor": "|", "bitxor": "^"}
_check = ar.check                       # bit for bit, transcendentals within the CUDA math library's ULP bounds


def _run(build, batches, **kw):
    """Builds a pipeline from build(*external_sources) and returns its outputs (lists of numpy samples) for each batch of inputs.
    batches: [[source 0 samples, source 1 samples, ...], ...]."""
    import nvidia.dali as dali
    from nvidia.dali import fn
    nsrc = len(batches[0])
    state = {}

    @dali.pipeline_def(batch_size=max(len(b[0]) for b in batches), num_threads=1, device_id=0, prefetch_queue_depth=1, seed=7)
    def pipe():
        srcs = [fn.external_source(source=(lambda _iteration=None, k=k: state["b"][k]), device="gpu", layout=kw.get("layout")) for k in range(nsrc)]
        return build(*srcs)
    p = pipe()
    p.build()
    res = []
    for b in batches:
        state["b"] = b
        outs = p.run()
        res.append([o.as_cpu() if hasattr(o, "as_cpu") else [np.asarray(o.at(i)) for i in range(len(o))] for o in outs])
    return res, p


def _grid(ta, tb, rng):
    ea, eb = ar.edge_values(ta), ar.edge_values(tb)
    a0, b0 = np.meshgrid(ea, eb, indexing="ij")
    a1, b1 = ar.random_values(ta, 97, rng), ar.random_values(tb, 97, rng)
    return [a0.ravel(), a1], [b0.ravel(), b1]


def test_unary_ops_every_type():
    from nvidia.dali import math as dmath
    rng = np.random.default_rng(1)
    for t in ar.TYPES:
        xs = [np.concatenate([ar.edge_values(t)] * 2), ar.random_values(t, 131, rng)]
        ops = [o for o in UNARY]

        def build(x):
            outs = []
            for o in ops:
                outs.append(+x if o == "plus" else -x if o == "minus" else getattr(dmath, o)(x))
            return tuple(outs)
        (outs,), _ = _run(build, [[xs]])
        for o, got in zip(ops, outs):
            for k in range(2):
                _check(o, got[k], [xs[k]], [t])


def test_binary_ops_every_type_pair():
    from nvidia.dali import math as dmath
    rng = np.random.default_rng(2)
    for ta in ar.TYPES:
        for tb in ar.TYPES:
            A, B = _grid(ta, tb, rng)
            ops = [o for o in BINARY if not (o in ar.INT_ONLY and (ta in ar.FLOATS or tb in ar.FLOATS))]

            def build(a, b):
                outs = []
                for o in ops:
                    outs.append(eval(f"a {PY[o]} b") if o in PY else getattr(dmath, o)(a, b))
                return tuple(outs)
            (outs,), _ = _run(build, [[A, B]])
            for o, got in zip(ops, outs):
                for k in range(2):
                    _check(o, got[k], [A[k], B[k]], [ta, tb])


def test_clamp_and_min_max_triples():
    from nvidia.dali import math as dmath
    rng = np.random.default_rng(3)
    for ta, tb, tc in [(ar.U8, ar.I32, ar.I32), (ar.F16, ar.F32, ar.F16), (ar.I64, ar.U8, ar.F64), (ar.BOOL, ar.U16, ar.I8),
                       (ar.F32, ar.F32, ar.F32), (ar.U64, ar.U64, ar.U32)]:
        xs = [ar.random_values(t, 300, rng) for t in (ta, tb, tc)]
        (outs,), _ = _run(lambda a, b, c: (dmath.clamp(a, b, c),), [[[x] for x in xs]])
        _check("clamp", outs[0][0], xs, [ta, tb, tc])


def test_broadcast_mean_std_sequences_and_layout():
    rng = np.random.default_rng(4)
    mean = np.array([0.485, 0.456, 0.406], np.float32) * 255
    std = np.array([0.229, 0.224, 0.225], np.float32) * 255
    imgs = [rng.integers(0, 256, s, dtype=np.uint8) for s in [(4, 30, 20, 3), (2, 7, 100, 3), (1, 1, 1, 3)]]
    from nvidia.dali import types
    from nvidia.dali import fn
    (outs,), p = _run(lambda x, m, s: ((fn.cast(x, dtype=types.FLOAT) - m) / s,), [[imgs, [mean] * 3, [std] * 3]], layout="FHWC")
    for k, img in enumerate(imgs):
        want = ar.evaluate("fdiv", [ar.evaluate("sub", [img.astype(np.float32), mean], [ar.F32, ar.F32]), std], [ar.F32, ar.F32])
        assert ar.same_bits(outs[0][k], want), k
    res, p = _run(lambda x: (x * 2,), [[imgs]], layout="FHWC")
    assert p.run()[0].layout() == "FHWC"


def test_cpu_per_sample_scalars():
    from nvidia.dali import fn
    rng = np.random.default_rng(5)
    xs = [rng.standard_normal((n, 3)).astype(np.float32) for n in (5, 17, 1, 64)]
    (outs,), _ = _run(lambda x: (lambda u: (x * u + u, u))(fn.random.uniform(range=(-2.0, 2.0))), [[xs]])
    for k, x in enumerate(xs):
        u = np.float32(outs[1][k])
        want = ar.evaluate("add", [ar.evaluate("mul", [x, u], [ar.F32, ar.F32]), u], [ar.F32, ar.F32])
        assert ar.same_bits(outs[0][k], want), k


def test_fused_chain_matches_materialised_steps_in_one_launch():
    from dali_b200 import capi
    from nvidia.dali import fn, math as dmath, types
    rng = np.random.default_rng(6)
    xs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in [(64, 48), (3, 500), (200, 1)]]

    def chain(x, m, step):
        y = step(fn.cast(x, dtype=types.FLOAT) * (1 / 255))
        y = step(y - m)
        y = step(y / 0.25)
        y = step(dmath.clamp(y, -1.5, 1.5))
        y = step(y * y + 0.5)
        return step(fn.cast(y > 0.75, dtype=types.UINT8) * 200 + dmath.sqrt(y)),
    m = [np.array([0.1, 0.5, 0.9], np.float32)] * 3
    n0 = capi.launch_count()
    (fused,), p1 = _run(lambda x, m: chain(x, m, lambda e: e), [[xs, m]])
    n1 = capi.launch_count()
    (steps,), p2 = _run(lambda x, m: chain(x, m, lambda e: e.gpu()), [[xs, m]])
    assert n1 - n0 == 1, n1 - n0
    for a, b in zip(fused[0], steps[0]):
        assert ar.same_bits(a, b)


def test_cast_saturation_and_rounding():
    from nvidia.dali import fn
    rng = np.random.default_rng(8)
    src = {ar.F32: np.concatenate([ar.edge_values(ar.F32), np.arange(-300, 300, 0.25, dtype=np.float32),
                                   rng.standard_normal(500).astype(np.float32) * 1e5]),
           ar.F64: np.concatenate([ar.edge_values(ar.F64), np.array([2.0 ** 63, -2.0 ** 63, 2.0 ** 64, 4.5e15 + 0.5])]),
           ar.I64: ar.edge_values(ar.I64), ar.U16: ar.edge_values(ar.U16), ar.F16: ar.edge_values(ar.F16)}
    for tf, x in src.items():
        (outs,), _ = _run(lambda a: tuple(fn.cast(a, dtype=t) for t in ar.TYPES), [[[x]]])
        for t, got in zip(ar.TYPES, outs):
            assert ar.same_bits(got[0], ar.convert_sat(x, tf, t)), (ar.NAMES[tf], ar.NAMES[t])
            if tf == ar.F32 and t == ar.U8:
                assert np.array_equal(got[0], pr.round_sat_u8(np.nan_to_num(x, nan=0.0)))


def test_iterator_reads_expression_output_as_torch():
    import nvidia.dali as dali
    from nvidia.dali import fn, types
    from nvidia.dali.plugin.pytorch import DALIGenericIterator
    rng = np.random.default_rng(9)
    data = [rng.integers(0, 256, (8, 6, 3), dtype=np.uint8) for _ in range(4)]

    @dali.pipeline_def(batch_size=4, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda: data, device="gpu", layout="HWC")
        return fn.cast(x, dtype=types.FLOAT) / 255 - 0.5
    it = DALIGenericIterator([pipe()], ["img"], size=8)
    batch = next(iter(it))[0]["img"]
    assert batch.is_cuda and tuple(batch.shape) == (4, 8, 6, 3)
    want = np.stack([ar.evaluate("sub", [ar.evaluate("fdiv", [d.astype(np.float32), np.float32(255)], [ar.F32, ar.F32]),
                                         np.float32(0.5)], [ar.F32, ar.F32]) for d in data])
    assert ar.same_bits(batch.cpu().numpy(), want)


def test_broadcast_error_names_the_sample():
    a = [np.zeros((4, 3), np.float32), np.zeros((5, 3), np.float32)]
    b = [np.zeros((4, 3), np.float32), np.zeros((2, 3), np.float32)]
    with pytest.raises(Exception) as e:
        _run(lambda x, y: (x + y,), [[a, b]])
    msg = str(e.value)
    assert "sample 1" in msg and "(5, 3)" in msg and "(2, 3)" in msg, msg


def test_constants_and_shared_subexpression():
    from nvidia.dali import types
    d = [np.array([1.0, 3.0, -2.5], np.float64)] * 2
    u = [np.array([1, 2 ** 63, 2 ** 64 - 1], np.uint64)] * 2

    def build(d, u):
        y = d * types.Constant(0.1, types.FLOAT64)
        for _ in range(6):
            y = y * y                                           # 7 instructions: y is evaluated once per use of the text
        return (d * types.Constant(0.1, types.FLOAT64), u & types.Constant(2 ** 64 - 1, types.UINT64),
                u + types.Constant(2 ** 63 + 5, types.UINT64), d * 0 + types.Constant(2.5, types.INT32), y)
    (outs,), _ = _run(build, [[d, u]])
    assert ar.same_bits(outs[0][0], d[0] * 0.1)
    assert np.array_equal(outs[1][0], u[0]) and np.array_equal(outs[2][1], u[0] + np.uint64(2 ** 63 + 5))
    assert list(outs[3][0]) == [3.0, 3.0, 3.0]                   # ConvertSat<int32>(2.5) = 3
    want = d[0] * 0.1
    for _ in range(6):
        want = want * want
    assert ar.same_bits(outs[4][0], want)
