"""nvidia.dali.fn for the hot-path operators: wrappers generated from the C++ schema registry, as the reference
generates them from its schemas (dali/python/nvidia/dali/fn/__init__.py:66-115, ops/_names.py:24-72:
`decoders__Image` -> fn.decoders.image, `CropMirrorNormalize` -> fn.crop_mirror_normalize).
"""
import sys
import types as _pytypes

import numpy as np

from . import arith as _arith
from . import backend
from . import types as _types
from .pipeline import DataNode, _current, _ExternalSourceGroup


def _to_snake_case(name):
    out = name[0].lower()
    for i in range(1, len(name)):
        c = name[i]
        if c.isupper():
            prev, nxt = name[i - 1], name[i + 1] if i + 1 < len(name) else ""
            if not prev.isupper() or (nxt and nxt.islower()):
                out += "_"
            out += c.lower()
        else:
            out += c
    return out


_INPUT_DEVICE = {"mixed": "cpu", "cpu": "cpu", "gpu": "gpu"}
# operators whose reference schema has a random seed argument (random_crop_attr.cc:34): unseeded ones draw from the pipeline's table
_SEEDED_SCHEMAS = ("decoders__ImageRandomCrop", "RandomResizedCrop")
# operators all of whose inputs are data: any GPU input selects the GPU operator, and a CPU input is then moved with .gpu() wherever
# it stands, not only as input 0
_GPU_DATA_SCHEMAS = ("Cat", "Stack", "MultiPaste")


def _make_wrapper(schema):
    args_info = backend.schema_args(schema)
    min_in, max_in, num_out, doc = backend.schema_info(schema)
    has_mixed = backend.operator_registered(schema, "mixed")
    has_gpu = backend.operator_registered(schema, "gpu")

    def op(*inputs, device=None, name=None, **kwargs):
        pipe = _current()
        if pipe is None:
            raise RuntimeError(f"fn.{_to_snake_case(schema.split('__')[-1])} must be called inside a pipeline definition "
                               "(@pipeline_def function or `with pipeline:` block)")
        if not (min_in <= len(inputs) <= max_in):
            raise ValueError(f"Operator {schema} expects {min_in}..{max_in} inputs, got {len(inputs)}")
        # an arithmetic expression consumed by an operator is computed by an operator of its own (dali_b200.arith)
        inputs = tuple(_arith.materialize(i) for i in inputs)
        kwargs = {k: _arith.materialize(v) for k, v in kwargs.items()}
        for i in inputs:
            if not isinstance(i, DataNode):
                raise TypeError(f"Operator inputs must be DataNodes, got {type(i).__name__}. Wrap constants with fn.external_source.")
        if device is None:
            # as in the reference: the device follows the first input (gpu input -> gpu operator)
            lead = inputs if schema in _GPU_DATA_SCHEMAS else inputs[:1]
            device = "gpu" if (any(i.device == "gpu" for i in lead) and has_gpu) else ("mixed" if has_mixed and not has_gpu else "cpu")
        if device not in ("cpu", "gpu", "mixed"):
            raise ValueError(f"Invalid device \"{device}\". Valid options are \"cpu\", \"gpu\" or \"mixed\"")
        spec = backend.OpSpec(schema)
        spec.add_arg("device", device)
        in_dev = _INPUT_DEVICE[device]
        for idx, i in enumerate(inputs):
            if i.device != in_dev:
                if i.device == "cpu" and in_dev == "gpu" and (idx == 0 or schema in _GPU_DATA_SCHEMAS):
                    i = i.gpu()
                elif i.device == "cpu" and in_dev == "gpu":
                    pass            # auxiliary inputs of GPU operators (slice anchor / shape) may stay on the CPU, as in the reference
                else:
                    raise ValueError(f"Operator {schema} on device '{device}' expects {in_dev} inputs, got a {i.device} input")
            if i.device == "cpu":
                i._consumed_cpu = True
            spec.add_input(i.name, i.device)
        for k, v in kwargs.items():
            if k not in args_info:
                raise TypeError(f"Operator {schema} got an unexpected '{k}' argument")   # same wording family as the reference
            if v is None:
                continue
            if isinstance(v, DataNode):
                if not args_info[k][0]:
                    raise TypeError(f"Argument '{k}' of operator {schema} does not accept a DataNode (per-sample tensor) input")
                if v.device != "cpu":
                    raise ValueError(f"Argument inputs must be CPU DataNodes ('{k}')")
                v._consumed_cpu = True
                spec.add_argument_input(k, v.name)
            else:
                if hasattr(v, "value") and not isinstance(v, (int, float)):
                    v = v.value
                if isinstance(v, (_types.DALIDataType, _types.DALIInterpType, _types.DALIImageType)):
                    v = int(v)
                spec.add_arg(k, v)
        inst = name or pipe._new_name(schema)
        out_dev = "cpu" if device == "cpu" else "gpu"
        outs = [DataNode(f"{inst}[{k}]" if num_out > 1 else inst, out_dev) for k in range(num_out)]
        for o in outs:
            spec.add_output(o.name, o.device)
        pipe._nodes.append((schema, inst, spec))
        # graph bookkeeping for the seed assignment (Pipeline._assign_seeds): inputs in the reference's order -- positional, then
        # argument inputs sorted by name (ops/__init__.py:400-403) -- and whether the user left the seed open
        arg_in = {k: v for k, v in kwargs.items() if isinstance(v, DataNode)}
        user_seed = kwargs.get("seed")
        pipe._op_graph[inst] = ([i.name for i in inputs] + [arg_in[k].name for k in sorted(arg_in)], [o.name for o in outs],
                                schema in _SEEDED_SCHEMAS, not (isinstance(user_seed, int) and user_seed >= 0))
        return outs[0] if num_out == 1 else tuple(outs)

    op.__name__ = _to_snake_case(schema.split("__")[-1])
    op.__doc__ = doc + "\n\nArguments: " + ", ".join(sorted(a for a in args_info if a not in ("num_threads", "max_batch_size", "seed", "preserve", "bytes_per_sample_hint")))
    op.schema_name = schema
    return op


def external_source(source=None, num_outputs=None, *, cycle=None, name=None, device="cpu", layout=None, dtype=None, ndim=None,
                    batch=True, batch_info=False, parallel=False, no_copy=None, prefetch_queue_depth=None, cuda_stream=None,
                    use_copy_kernel=None, blocking=None, repeat_last=False, **_ignored):
    """fn.external_source (dali/python/nvidia/dali/external_source.py:1002-1150), subset: callables, iterables, feed_input."""
    pipe = _current()
    if pipe is None:
        raise RuntimeError("fn.external_source must be called inside a pipeline definition")
    if device not in ("cpu", "gpu"):
        raise ValueError("external_source device must be 'cpu' or 'gpu'")
    n = num_outputs or 1
    base = name or pipe._new_name("ExternalSource")
    # no_copy=True (external_source.py `no_copy`): the caller keeps the buffers alive and unmodified until the iteration that uses
    # them has completed; page-locked encoded streams then reach the GPU decoder by DMA straight from the caller's memory
    g = _ExternalSourceGroup(source, [], batch, cycle, layout if isinstance(layout, str) or layout is None else layout[0], dtype, device,
                             batch_info, bool(no_copy))
    for k in range(n):
        node = DataNode(base if n == 1 else f"{base}[{k}]", device, source=g)
        g.outputs.append(node)
        if name:
            pipe._ext_names[name if n == 1 else f"{name}[{k}]"] = node.name
    pipe._externals.append(g)
    return g.outputs[0] if num_outputs is None else list(g.outputs)


def _install():
    this = sys.modules[__name__]
    for schema in backend.schema_names():
        parts = schema.split("__")
        mod = this
        for p in parts[:-1]:
            sub = getattr(mod, p, None)
            if sub is None:
                sub = _pytypes.ModuleType(f"{mod.__name__}.{p}")
                setattr(mod, p, sub)
                sys.modules[sub.__name__] = sub
            mod = sub
        setattr(mod, _to_snake_case(parts[-1]), _make_wrapper(schema))
    # fn.cast folds into arithmetic expressions; applied to any other node it is the Cast operator (dali_b200.arith)
    def cast(x, *, dtype, device=None, name=None):
        if device not in (None, "gpu"):
            raise ValueError("fn.cast runs on the GPU only; move the input there with .gpu()")
        return _arith.cast(x, dtype)
    cast.__doc__ = this.cast.__doc__
    cast.schema_name = "Cast"
    this.cast = cast
    # deprecated aliases kept by the reference (mixed_decoder.cc:40-50)
    if hasattr(this, "decoders"):
        this.image_decoder = this.decoders.image
        this.audio_decoder = this.decoders.audio



# ---- host-side sources in front of the hot path (SURVEY.md 8f rank 2): they feed CPU batches like an external_source callback
def _source_group(pipe, source, n, base, layout=None, device="cpu"):
    g = _ExternalSourceGroup(source, [], True, None, layout, None, device, False)
    for k in range(n):
        g.outputs.append(DataNode(base if n == 1 else f"{base}[{k}]", device, source=g))
    pipe._externals.append(g)
    return g


def _readers_file(file_root=None, file_list=None, files=None, labels=None, *, random_shuffle=False, shuffle_after_epoch=False,
                  initial_fill=1024, shard_id=0, num_shards=1, stick_to_shard=False, pad_last_batch=False, seed=-1, name=None,
                  device="cpu", shuffle_after_epoch_seed=None, file_filters=None, dir_filters=None, case_sensitive_filter=False,
                  **_ignored):
    """fn.readers.file (dali/operators/reader/file_reader_op.cc, loader/file_label_loader.h): (encoded file bytes, label)."""
    from .readers import FileReader
    pipe = _current()
    if pipe is None:
        raise RuntimeError("fn.readers.file must be called inside a pipeline definition")
    if device != "cpu":
        raise ValueError("readers.file produces CPU batches")
    reader = FileReader(pipe.max_batch_size, file_root, file_list, files, labels, random_shuffle, shuffle_after_epoch, initial_fill,
                        shard_id, num_shards, stick_to_shard, pad_last_batch, seed, shuffle_after_epoch_seed, file_filters, dir_filters,
                        case_sensitive_filter)
    inst = name or pipe._new_name("readers__File")
    g = _source_group(pipe, reader, 2, inst)
    ahead = 2                                # batches read ahead of the pipeline on the reader's own thread
    if pipe.device_id is not None:
        # GPU pipeline: page-locked reader buffers, borrowed by the decoder until the iteration completes (no_copy semantics); the
        # ring covers the batches in flight in the pipeline, the ones queued by the read-ahead thread and the one being read
        reader.enable_pinned(pipe._depth + 1 + ahead + 1, pipe.device_id)
        g.no_copy = True
    reader.enable_prefetch(ahead)
    pipe._readers[inst] = reader
    return g.outputs[0], g.outputs[1]


def _random_coin_flip(*, probability=0.5, shape=None, seed=-1, dtype=None, name=None, device="cpu", **_ignored):
    """fn.random.coin_flip (dali/operators/random/coin_flip_cpu.cc): 1 with `probability`, else 0; int32 by default."""
    from .readers import CoinFlip
    pipe = _current()
    if pipe is None:
        raise RuntimeError("fn.random.coin_flip must be called inside a pipeline definition")
    npdt = np.int32 if dtype is None else _types.to_numpy_type(int(dtype))
    return _source_group(pipe, CoinFlip(pipe.max_batch_size, probability, shape, seed, npdt), 1, name or pipe._new_name("random__CoinFlip")).outputs[0]


def _random_uniform(*, range=(-1.0, 1.0), values=None, shape=None, seed=-1, dtype=None, name=None, device="cpu", **_ignored):
    """fn.random.uniform (dali/operators/random/uniform_distribution_cpu.cc): `range` = [a, b) continuous, `values` = discrete."""
    from .readers import Uniform
    pipe = _current()
    if pipe is None:
        raise RuntimeError("fn.random.uniform must be called inside a pipeline definition")
    npdt = np.float32 if dtype is None else _types.to_numpy_type(int(dtype))
    return _source_group(pipe, Uniform(pipe.max_batch_size, range, values, shape, seed, npdt), 1, name or pipe._new_name("random__Uniform")).outputs[0]


def _install_sources():
    this = sys.modules[__name__]
    for modname, entries in (("readers", {"file": _readers_file}), ("random", {"coin_flip": _random_coin_flip, "uniform": _random_uniform})):
        sub = getattr(this, modname, None)
        if sub is None:
            sub = _pytypes.ModuleType(f"{this.__name__}.{modname}")
            setattr(this, modname, sub)
            sys.modules[sub.__name__] = sub
        for k, f in entries.items():
            f.__name__ = k
            setattr(sub, k, f)


_install()
_install_sources()
