"""``jit`` -- compile a function that contains communication ops into a CUDA graph.

The reference's ops are JAX primitives so that they run inside ``jax.jit``; XLA compiles
the surrounding program and an ordered effect token keeps the custom calls in program
order (/root/reference/mpi4jax/_src/utils.py:45-53, jax_compat.py:82-100).  The H100
design replaces the tracing compiler with **CUDA streams and graphs**: every op is a
kernel on the current stream (stream order == program order, the token is implicit), and
``jit`` records the whole function -- stencils, collectives, halo exchanges -- into one
CUDA graph that is replayed with a single launch.  All cross-GPU sequence numbers live in
device memory, so a replay is exactly as valid as the first run.

Semantics:
* call 1 runs eagerly (warm-up: allocations, staging growth, lazy communicator setup);
* call 2 captures; later calls copy the inputs into the captured input buffers and replay;
* a new graph is captured per distinct input signature (shapes, dtypes, devices, static args);
* outputs are returned as fresh clones unless ``donate_outputs=True``;
* functions of CPU tensors (and any call made while a graph is already capturing, or while
  autograd is recording) just run eagerly -- same results, no graph;
* rank-dependent Python control flow is fine: each rank captures its own graph, like each
  rank traces its own program under ``jax.jit``.
"""

from __future__ import annotations

import functools
from typing import Any, Callable

import torch


def _flatten(obj, leaves: list):
    if isinstance(obj, torch.Tensor):
        leaves.append(obj)
        return ("T", len(leaves) - 1)
    if isinstance(obj, (list, tuple)):
        kind = "L" if isinstance(obj, list) else ("N", type(obj)) if hasattr(obj, "_fields") else "U"
        return (kind, [_flatten(o, leaves) for o in obj])
    if isinstance(obj, dict):
        return ("D", {k: _flatten(v, leaves) for k, v in obj.items()})
    return ("C", obj)


def _unflatten(spec, leaves):
    kind, val = spec
    if kind == "T":
        return leaves[val]
    if kind == "L":
        return [_unflatten(s, leaves) for s in val]
    if kind == "U":
        return tuple(_unflatten(s, leaves) for s in val)
    if isinstance(kind, tuple) and kind[0] == "N":
        return kind[1](*[_unflatten(s, leaves) for s in val])
    if kind == "D":
        return {k: _unflatten(s, leaves) for k, s in val.items()}
    return val


def _spec_key(spec):
    kind, val = spec
    if kind == "T":
        return ("T",)
    if kind in ("L", "U") or (isinstance(kind, tuple) and kind[0] == "N"):
        return (str(kind), tuple(_spec_key(s) for s in val))
    if kind == "D":
        return ("D", tuple((k, _spec_key(s)) for k, s in sorted(val.items(), key=lambda kv: str(kv[0]))))
    try:
        hash(val)
        return ("C", val)
    except TypeError:
        return ("C", repr(val))


class _Captured:
    __slots__ = ("graph", "static_in", "out_spec", "static_out")


def jit(fn: Callable = None, *, donate_outputs: bool = False, static_inputs: bool = False,
        warmup: int = 1) -> Callable:
    """Decorator / wrapper: ``fast = mpi4jax_b200.jit(fn)``.

    ``donate_outputs``: return the graph's own output buffers (overwritten by the next call)
    instead of clones.  ``static_inputs``: capture the caller's tensors themselves as the graph
    inputs (no copy-in; later calls must pass the same storage, or pay one copy).
    """
    if fn is None:
        return functools.partial(jit, donate_outputs=donate_outputs, static_inputs=static_inputs,
                                 warmup=warmup)

    cache: dict = {}
    calls: dict = {}

    @functools.wraps(fn)
    def wrapped(*args, **kwargs):
        leaves: list = []
        spec = _flatten((args, kwargs), leaves)
        on_gpu = any(t.is_cuda for t in leaves) or (
            not leaves and torch.cuda.is_available() and _default_device_is_cuda()
        )
        needs_grad = torch.is_grad_enabled() and any(t.requires_grad for t in leaves)
        if (not on_gpu) or needs_grad or torch.cuda.is_current_stream_capturing() or _host_staged():
            return fn(*args, **kwargs)
        key = (_spec_key(spec), tuple((t.shape, t.dtype, t.device) for t in leaves))
        n = calls.get(key, 0)
        calls[key] = n + 1
        if n < warmup:
            return fn(*args, **kwargs)
        cap = cache.get(key)
        if cap is None:
            cap = _capture(fn, spec, leaves, static_inputs)
            cache[key] = cap
        else:
            for dst, src in zip(cap.static_in, leaves):
                if dst.data_ptr() != src.data_ptr():
                    dst.copy_(src)
            cap.graph.replay()
        outs = cap.static_out if donate_outputs else [o.clone() for o in cap.static_out]
        return _unflatten(cap.out_spec, outs)

    wrapped.__wrapped_fn__ = fn
    wrapped._cache = cache
    return wrapped


def _host_staged() -> bool:
    """Host-staged communicators block the host inside every op: nothing to capture."""
    from .backends import host_staged

    return host_staged.ACTIVE


def _default_device_is_cuda() -> bool:
    from .utils import get_default_comm

    return get_default_comm().device.type == "cuda"


def _capture(fn, spec, leaves, static_inputs: bool = False) -> _Captured:
    cap = _Captured()
    cap.static_in = [t.clone() if (t.is_cuda and not static_inputs) else t for t in leaves]
    a, k = _unflatten(spec, cap.static_in)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side, capture_error_mode="thread_local"):
            out = fn(*a, **k)
    torch.cuda.current_stream().wait_stream(side)
    out_leaves: list = []
    cap.out_spec = _flatten(out, out_leaves)
    cap.static_out = out_leaves
    cap.graph = graph
    graph.replay()          # the capture itself does not execute the work
    return cap


def linear_transpose(fn: Callable, *primals) -> Callable:
    """Transpose of a linear function, evaluated with reverse-mode AD
    (``jax.linear_transpose`` stand-in used by the reference's tests,
    tests/collective_ops/test_allreduce.py:81-138).  Returns a function mapping an output
    cotangent to a tuple of input cotangents; it is itself differentiable, so transposes
    nest (transposing ``allreduce`` twice gives ``allreduce`` again)."""
    from torch.func import vjp

    def transposed(ct):
        _, pullback = vjp(fn, *primals)
        return pullback(ct)

    return transposed
