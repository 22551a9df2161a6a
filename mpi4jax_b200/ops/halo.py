"""Fused multi-field 2-D halo exchange (CUDA tensors) -- see csrc/b2_halo.cu.

One kernel launch replaces, per field, the reference's 2 ``sendrecv`` + ``send`` + ``recv``
calls and the strided pack / unpack ops around them
(/root/reference/examples/shallow_water.py:172-264).
"""

from __future__ import annotations

from typing import Optional, Sequence

import torch

from .._src.comm import Comm
from .._src.utils import get_default_comm


def halo_exchange(fields: Sequence[torch.Tensor], kinds: Sequence[str], *, west: Optional[int],
                  east: Optional[int], south: Optional[int], north: Optional[int],
                  sw: Optional[int] = None, se: Optional[int] = None, nw: Optional[int] = None,
                  ne: Optional[int] = None, periodic_x: bool = True, at_east_wall: bool = False,
                  at_north_wall: bool = False, comm: Optional[Comm] = None) -> None:
    """Exchange the 1-cell halos of ``fields`` (contiguous float32 ``(ny, nx)`` CUDA tensors,
    updated in place) with the neighbouring ranks; ``None`` means a physical wall.  The corner
    halo cells come straight from the diagonal neighbours ``sw/se/nw/ne`` (``None`` where the
    row of processes below/above does not exist).
    ``kinds`` ("h" | "u" | "v") select the wall condition applied after the exchange.
    The receive channels of a communicator count messages per side, so every call on one
    communicator must name the same neighbours; use a ``Clone()`` per neighbour layout."""
    comm = comm or get_default_comm()
    if not fields or not all(f.is_cuda for f in fields):
        raise ValueError("halo_exchange needs CUDA tensors")
    g = lambda r: -1 if r is None else int(r)  # noqa: E731
    comm._native_comm().halo_exchange(list(fields), list(kinds), g(west), g(east), g(south), g(north),
                                      periodic_x, at_east_wall, at_north_wall,
                                      sw=g(sw), se=g(se), nw=g(nw), ne=g(ne))
