"""The autograd rules the eager variable-count ops share (alltoallv, allgatherv, reduce_scatterv, gatherv,
scatterv), written once; each op's Function supplies only its ``forward`` and ``backward``."""

from __future__ import annotations

import torch

from ..utils import needs_autograd


class RowsvFunction(torch.autograd.Function):
    """Base of a variable-count op's Function.  ``forward(x, counts, *rest)`` returns ``(out, out_counts)``;
    ``backward`` finds ``counts, *rest`` in ``ctx.args``, the input rows in ``ctx.in_rows`` and
    ``out_counts`` in ``ctx.saved_tensors``.  ``vmap_error``: the op's message for batched counts."""

    vmap_error: str

    @classmethod
    def run(cls, x, *args):
        """The op: through ``apply`` when autograd or a ``torch.func`` transform has to see it, otherwise
        ``forward`` called directly."""
        if needs_autograd(x):
            return cls.apply(x, *args)
        return cls.forward(x, *args)

    @staticmethod
    def setup_context(ctx, inputs, output):
        x, *ctx.args = inputs
        ctx.in_rows = x.shape[0]
        ctx.mark_non_differentiable(output[1])
        ctx.save_for_backward(output[1])

    @classmethod
    def jvp(cls, ctx, x_t, *_):
        out_t, _counts = cls.apply(x_t, *ctx.args)
        return out_t, None

    @classmethod
    def vmap(cls, info, in_dims, x, *args):
        if any(d is not None for d in in_dims[1:]):
            raise ValueError(cls.vmap_error)
        if in_dims[0] is None:
            return cls.apply(x, *args), (None, None)
        # keep the row axis in front: (B, N, *S) -> (N, B, *S), moved as one message of B-times larger rows
        return cls.apply(x.movedim(in_dims[0], 1).contiguous(), *args), (1, None)
