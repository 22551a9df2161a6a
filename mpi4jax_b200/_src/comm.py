"""Communicators, reduction ops, Status -- the MPI-like object model.

The reference takes ``mpi4py`` objects (``MPI.Intracomm``, ``MPI.Op``, ``MPI.Status``)
and forwards their C handles to its C++ bridge (/root/reference/mpi4jax/_src/utils.py:
60-153).  Neither mpi4py nor an MPI library exists on the target image, and the H100
transport is not MPI at all, so this module supplies the small object model user code
needs (``mpi4jax_b200.MPI``): ``COMM_WORLD``, ``Comm.Get_rank/Get_size/Clone/Split/
Free/Barrier``, the ten predefined elementwise ``Op`` constants and ``MAXLOC`` / ``MINLOC``, ``Status`` with
``Get_source/Get_tag/Get_count``, ``ANY_SOURCE``/``ANY_TAG``.

Process model (same as the reference, README.rst:83-89): one OS process per rank, one
GPU per process.  Ranks are launched by ``torchrun`` or ``python -m mpi4jax_b200.run``;
the control plane (handle exchange, CPU-tensor collectives) is a ``torch.distributed``
gloo group, the data plane for CUDA tensors is the native symmetric heap
(``_src/backends/cuda.py``).
"""

from __future__ import annotations

import atexit
import os
import threading
import weakref
from datetime import timedelta
from typing import Optional, Sequence

import torch
import torch.distributed as dist

from .native import codes

ANY_SOURCE = -1
ANY_TAG = -1
PROC_NULL = -2
UNDEFINED = -32766


class MPIError(RuntimeError):
    """Raised (or printed before aborting) when a communication call fails."""


class Op:
    """A reduction operator (stand-in for ``mpi4py.MPI.Op``): one of the ten predefined elementwise ones
    (``code`` selects the fused kernel instantiation), ``MAXLOC`` / ``MINLOC`` (which reduce
    ``(values, indices)`` pairs, collective_ops/_loc.py), or a user-defined one made with
    :meth:`Op.Create` (``code is None``, ``function`` is applied on the device)."""

    __slots__ = ("name", "code", "function", "commute")

    def __init__(self, name: str, code, function=None, commute: bool = True):
        self.name = name
        self.code = code
        self.function = function
        self.commute = commute

    @classmethod
    def Create(cls, function, commute: bool = True) -> "Op":
        """User-defined reduction (``MPI.Op.Create``).  The reference forwards any ``MPI.Op`` handle
        to the MPI library (/root/reference/mpi4jax/_src/collective_ops/allreduce.py:104), which
        calls the user's C function on the host.  Here ``function(a, b) -> Tensor`` combines two
        tensors elementwise with torch ops and runs on the device: allreduce / reduce / scan gather
        the contributions with the native all-gather / gather kernels and fold them in rank order
        (``((x_0 (+) x_1) (+) x_2) ...``, valid for non-commutative operators too)."""
        if not callable(function):
            raise TypeError("Op.Create needs a callable f(a, b) -> Tensor")
        return cls(getattr(function, "__name__", "USER_OP"), None, function, bool(commute))

    def Is_commutative(self) -> bool:
        return bool(self.commute)

    def Free(self) -> None:
        """No resources are attached to an operator (mpi4py API compatibility)."""

    def __repr__(self) -> str:
        return f"<mpi4jax_b200.MPI.{self.name}>"

    def python_function(self):
        """Binary Python function of the operator (used by the object collectives, like mpi4py's
        ``comm.allreduce(obj, op)``).  MAXLOC / MINLOC fold ``(value, index)`` pairs of Python numbers, or of
        tensors elementwise, by the rule of collective_ops/_loc.py."""
        import functools
        import operator

        if self.function is not None:
            return self.function
        if self.name in ("MAXLOC", "MINLOC"):
            from .collective_ops import _loc

            return functools.partial(_loc.fold, maxloc=self.name == "MAXLOC")

        return {
            "SUM": operator.add, "PROD": operator.mul, "MIN": min, "MAX": max,
            "LAND": lambda a, b: bool(a) and bool(b), "LOR": lambda a, b: bool(a) or bool(b),
            "LXOR": lambda a, b: bool(a) != bool(b),
            "BAND": operator.and_, "BOR": operator.or_, "BXOR": operator.xor,
        }[self.name]

    def __call__(self, a, b):
        return self.python_function()(a, b)

    def __reduce__(self):
        if self.function is not None:
            return (Op.Create, (self.function, self.commute))
        return (_op_by_name, (self.name,))


SUM = Op("SUM", codes.SUM)
PROD = Op("PROD", codes.PROD)
MIN = Op("MIN", codes.MIN)
MAX = Op("MAX", codes.MAX)
LAND = Op("LAND", codes.LAND)
LOR = Op("LOR", codes.LOR)
LXOR = Op("LXOR", codes.LXOR)
BAND = Op("BAND", codes.BAND)
BOR = Op("BOR", codes.BOR)
BXOR = Op("BXOR", codes.BXOR)
MAXLOC = Op("MAXLOC", codes.MAXLOC)
MINLOC = Op("MINLOC", codes.MINLOC)
_ALL_OPS = {o.name: o for o in (SUM, PROD, MIN, MAX, LAND, LOR, LXOR, BAND, BOR, BXOR, MAXLOC, MINLOC)}


def _op_by_name(name: str) -> Op:
    return _ALL_OPS[name]


def as_op(op) -> Op:
    """Accept our ``Op`` or (if mpi4py happens to be installed) an ``mpi4py.MPI.Op``."""
    if isinstance(op, Op):
        return op
    name = getattr(op, "name", None) or getattr(op, "Get_name", lambda: None)()
    if isinstance(name, str):
        key = name.replace("MPI_", "").upper()
        if key in _ALL_OPS:
            return _ALL_OPS[key]
    raise TypeError(f"unsupported reduction operator: {op!r}")


class Status:
    """Receive status (stand-in for ``mpi4py.MPI.Status``).

    On the GPU path the receive kernel writes (source, tag, byte count) into a
    host-mapped record; the values are read lazily, after synchronising with the
    stream the receive was enqueued on -- no host sync happens unless the user
    actually inspects the status.
    """

    def __init__(self):
        # every Status can be named by an integer (like a communicator): the traceable frontend passes
        # it through compiled graphs as a plain attribute (compile_ops.py), the counterpart of the
        # reference baking the address of the mpi4py Status object into the custom call (recv.py:100-103)
        global _status_counter
        _status_counter += 1
        self._id = _status_counter
        _status_registry[self._id] = self
        self._source = ANY_SOURCE
        self._tag = ANY_TAG
        self._count_bytes = 0
        self._error = 0
        self._native = None  # (record_ptr, event) while a GPU receive is pending
        self._itemsize = 1

    # -- filled by the backends ------------------------------------------------
    def _set(self, source: int, tag: int, count_bytes: int, itemsize: int = 1) -> None:
        self._source, self._tag, self._count_bytes = int(source), int(tag), int(count_bytes)
        self._itemsize = itemsize
        self._native = None

    def _bind_native(self, record, event, itemsize: int) -> None:
        self._native = (record, event)
        self._itemsize = itemsize

    def _set_proc_null(self) -> None:
        """MPI: a receive from PROC_NULL returns at once with source = PROC_NULL, tag = ANY_TAG, count 0."""
        self._set(PROC_NULL, ANY_TAG, 0, self._itemsize)

    def _sync(self) -> None:
        if self._native is None:
            return
        record, event = self._native
        event.synchronize()
        rec = record.contents
        self._source, self._tag = int(rec.source), int(rec.tag)
        self._count_bytes, self._error = int(rec.count_bytes), int(rec.error)
        self._native = None

    # -- mpi4py-compatible accessors --------------------------------------------
    def Get_source(self) -> int:
        self._sync()
        return self._source

    def Get_tag(self) -> int:
        self._sync()
        return self._tag

    def Get_error(self) -> int:
        self._sync()
        return self._error

    def Get_count(self, datatype=None) -> int:
        """Elements received (of the receive buffer's dtype); bytes if ``datatype`` is ``BYTE``."""
        self._sync()
        if datatype is BYTE:
            return self._count_bytes
        return self._count_bytes // max(self._itemsize, 1)

    source = property(Get_source)
    tag = property(Get_tag)


BYTE = object()
_status_registry: "weakref.WeakValueDictionary[int, Status]" = weakref.WeakValueDictionary()
_status_counter = 0

_comm_registry: "weakref.WeakSet[Comm]" = weakref.WeakSet()
_world_lock = threading.Lock()
_world: Optional["Comm"] = None
_comm_counter = 0


def _env_int(name: str, default: int) -> int:
    try:
        return int(os.environ.get(name, default))
    except ValueError:
        return default


def local_rank() -> int:
    return _env_int("LOCAL_RANK", _env_int("RANK", 0))


def select_device() -> torch.device:
    """Pin this process to its GPU (one process per GPU).  Several ranks may share a GPU
    when there are fewer devices than local ranks (correctness testing only)."""
    want = os.environ.get("MPI4JAX_B200_DEVICE", "").lower()
    if want == "cpu" or not torch.cuda.is_available():
        return torch.device("cpu")
    idx = local_rank() % torch.cuda.device_count()
    torch.cuda.set_device(idx)
    return torch.device("cuda", idx)


def _init_process_group() -> None:
    """Create the control-plane process group if the launcher has not done so."""
    if dist.is_initialized():
        return
    world = _env_int("WORLD_SIZE", 1)
    rank = _env_int("RANK", 0)
    timeout = timedelta(seconds=float(os.environ.get("MPI4JAX_B200_PG_TIMEOUT", "600")))
    if world == 1 and "MASTER_ADDR" not in os.environ:
        store = dist.HashStore()
        dist.init_process_group("gloo", store=store, rank=0, world_size=1, timeout=timeout)
        return
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timeout)


def _control_group_for_world():
    """A gloo group spanning all ranks (the default group itself when it is gloo-capable)."""
    backend = dist.get_backend()
    if "gloo" in str(backend):
        return dist.group.WORLD
    return dist.new_group(backend="gloo")


def _new_member_group(ranks: Sequence[int], gname: str):
    """A gloo group created by ITS MEMBERS ONLY, under a name they agree on.

    ``dist.new_group`` must be entered by every process of the job (its group names come from a
    job-wide counter); its ``use_local_synchronization=True`` variant hashes the member list together
    with the number of groups THIS process has created so far, so members with different histories --
    exactly the situation of a Dup / Split on a sub-communicator -- compute different names and hang
    in the rendezvous.  MPI lets any communicator be duplicated or split by its members alone, so the
    group is built one level below, with a name derived from the parent communicator (same on every
    member by construction, see ``Comm._child_name``)."""
    ranks = sorted(ranks)
    try:
        from torch.distributed import distributed_c10d as c10d

        default_pg = c10d._get_default_group()
        _, store = c10d._world.pg_map[default_pg]
        backend = c10d.Backend("gloo")
        pg, _ = c10d._new_process_group_helper(
            len(ranks), ranks.index(dist.get_rank()), ranks, backend, store, c10d.GroupName(gname),
            timeout=c10d._get_default_timeout(backend))
        c10d._world.pg_group_ranks[pg] = {g: i for i, g in enumerate(ranks)}
        return pg
    except (ImportError, AttributeError, KeyError, TypeError):   # pragma: no cover - private API moved
        return dist.new_group(ranks=ranks, backend="gloo", use_local_synchronization=True)


class Comm:
    """An intra-communicator over a subset of the job's processes."""

    def __init__(self, group, ranks: Sequence[int], name: str = "comm", gname: str = "b2w"):
        global _comm_counter
        self._gname = gname            # job-unique name of the control-plane group (same on every member)
        self._children = 0             # Clone / Split calls so far (collective, hence equal on every member)
        self._group = group
        self._ranks = list(ranks)
        self._global_rank = dist.get_rank()
        self._rank = self._ranks.index(self._global_rank)
        # torch.distributed numbers the members of a group by ascending global rank, whatever order
        # `ranks` was given in; a communicator made by Split(color, key) orders them by key.
        # _order[r] = torch's group index of the member with communicator rank r.
        by_global = sorted(self._ranks)
        self._order = [by_global.index(g) for g in self._ranks]
        self._name = name
        _comm_counter += 1
        self._id = _comm_counter
        self._native = None        # backends.cuda.NativeComm, created on first CUDA op
        self._cpu_state = None     # backends.cpu.CpuState, created on first CPU p2p op
        self._freed = False
        self.device = select_device()
        _comm_registry.add(self)
        # Communicator construction (COMM_WORLD, Clone, Split) is collective over exactly its members,
        # and so is the creation of the GPU side (symmetric heap, handle exchange).  Doing it here --
        # not on the first CUDA op -- keeps point-to-point ops point-to-point: a send / recv between
        # two ranks of a larger communicator must not wait for ranks that never communicate.
        # MPI4JAX_B200_LAZY_INIT=1 restores creation on first use (then the first CUDA op on a
        # communicator is collective).
        if self.device.type == "cuda" and os.environ.get("MPI4JAX_B200_LAZY_INIT", "0").lower() not in (
                "1", "true", "on"):
            self._native_comm()

    # -- mpi4py-style API --------------------------------------------------------
    def Get_rank(self) -> int:
        return self._rank

    def Get_size(self) -> int:
        return len(self._ranks)

    rank = property(Get_rank)
    size = property(Get_size)

    def Get_name(self) -> str:
        return self._name

    def Clone(self) -> "Comm":
        """A communicator over the same processes with private message channels
        (collective; reference default comm = ``COMM_WORLD.Clone()``, utils.py:20-27)."""
        self._check_alive()
        # only the members of THIS communicator take part (see _new_member_group), so Dup / Split work
        # on sub-communicators while the other ranks of the job do something else -- as in MPI
        gname = self._child_name("c")
        return Comm(_new_member_group(self._ranks, gname), self._ranks, name=self._name + ".clone", gname=gname)

    Dup = Clone

    def Split(self, color: int = 0, key: int = 0) -> Optional["Comm"]:
        """Partition the communicator (collective over all its ranks)."""
        self._check_alive()
        info = [None] * self.size
        dist.all_gather_object(info, (int(color), int(key), self._global_rank), group=self._group)
        info = self._in_rank_order(info)
        gname = self._child_name(f"s{color}")         # (counted on every member, UNDEFINED ones included)
        if color == UNDEFINED:
            return None
        members = sorted((k, r) for cc, k, r in info if cc == color)
        ranks = [r for _, r in members]
        # each rank creates only the group it belongs to (member-only synchronisation, see Clone)
        return Comm(_new_member_group(ranks, gname), ranks, name=f"{self._name}.split{color}", gname=gname)

    def Barrier(self) -> None:
        """Host-side barrier on the control plane (mpi4py ``comm.Barrier()``)."""
        self._check_alive()
        dist.barrier(group=self._group)

    barrier = Barrier

    def Free(self) -> None:
        if self._freed:
            return
        self._freed = True
        if self._native is not None:
            self._native.destroy()
            self._native = None

    # -- mpi4py's lower-case (pickle-based, host-synchronous) object API ----------------------
    # Scripts written for mpi4jax use mpi4py for their Python-side bookkeeping (rank-0 gathers of
    # results, parameter broadcasts, ...); there is no mpi4py here, so the communicator offers the
    # same calls over the gloo control plane.  Like in the reference (docs/sharp-bits.rst:74-135)
    # they share the tag space of the tensor ops of this communicator: do not interleave the two
    # on one communicator -- the default communicator of the tensor ops is a private clone.
    def barrier(self) -> None:
        self.Barrier()

    def bcast(self, obj=None, root: int = 0):
        self._check_alive()
        if self.size == 1:
            return obj
        box = [obj]
        dist.broadcast_object_list(box, src=self._global(root), group=self._group)
        return box[0]

    def allgather(self, obj) -> list:
        self._check_alive()
        out = [None] * self.size
        if self.size == 1:
            return [obj]
        dist.all_gather_object(out, obj, group=self._group)
        return self._in_rank_order(out)

    def gather(self, obj, root: int = 0):
        everything = self.allgather(obj)           # gloo's gather_object needs the same traffic
        return everything if self.rank == root else None

    def scatter(self, objs=None, root: int = 0):
        if self.rank == root and (objs is None or len(objs) != self.size):
            raise ValueError(f"scatter needs a sequence of {self.size} objects on the root")
        return self.bcast(list(objs) if self.rank == root else None, root)[self.rank]

    def allreduce(self, obj, op=None):
        import functools

        fn = (op or SUM).python_function()
        return functools.reduce(fn, self.allgather(obj))

    def reduce(self, obj, op=None, root: int = 0):
        total = self.allreduce(obj, op)
        return total if self.rank == root else None

    def send(self, obj, dest: int, tag: int = 0) -> None:
        from .backends import cpu as _cpu

        self._check_alive()
        _cpu.send_object(self, obj, int(dest), int(tag))

    def recv(self, buf=None, source: int = ANY_SOURCE, tag: int = ANY_TAG, status: Optional[Status] = None):
        from .backends import cpu as _cpu

        self._check_alive()
        return _cpu.recv_object(self, int(source), int(tag), status)

    def sendrecv(self, sendobj, dest: int, sendtag: int = 0, recvbuf=None, source: int = ANY_SOURCE,
                 recvtag: int = ANY_TAG, status: Optional[Status] = None):
        self.send(sendobj, dest, sendtag)          # eager: cannot deadlock against the receive
        return self.recv(None, source, recvtag, status)

    def Abort(self, errorcode: int = 1) -> None:
        """Kill the job (the launcher stops the remaining ranks when one exits non-zero)."""
        import sys

        sys.stderr.write(f"r{self.rank} | MPI_Abort called with error code {errorcode} - aborting\n")
        sys.stderr.flush()
        os._exit(errorcode if 0 < errorcode < 256 else 1)

    def py2f(self) -> int:
        return self._id

    def __repr__(self) -> str:
        return f"<mpi4jax_b200.MPI.Comm {self._name} rank={self._rank} size={self.size}>"

    def __hash__(self) -> int:
        return hash(("b200comm", self._id))

    def __eq__(self, other) -> bool:
        return isinstance(other, Comm) and other._id == self._id

    # -- internals -----------------------------------------------------------------
    def _check_alive(self) -> None:
        if self._freed:
            raise MPIError("communicator has been freed")

    def _child_name(self, kind: str) -> str:
        self._children += 1
        return f"{self._gname}/{self._children}{kind}"

    def _global(self, rank_in_comm: int) -> int:
        return self._ranks[rank_in_comm]

    def _in_rank_order(self, gathered: list) -> list:
        """Results of a torch.distributed all_gather on this group, reordered by communicator rank."""
        return [gathered[self._order[r]] for r in range(len(self._ranks))]

    def _native_comm(self):
        """The native (GPU) side of the communicator; created collectively on first use."""
        self._check_alive()
        if self._native is None:
            from .backends import transport

            self._native = transport.create(self)      # NVLink kernels, or host staging off-node
        return self._native

    @property
    def transport(self) -> str:
        """``"native"`` (NVLink kernels), ``"host"`` (host-staged fallback) or ``"cpu"``; decided
        collectively on first use."""
        if self.device.type != "cuda":
            return "cpu"
        from .backends.host_staged import HostStagedComm

        return "host" if isinstance(self._native_comm(), HostStagedComm) else "native"

    def _cpu(self):
        if self._cpu_state is None:
            from .backends.cpu import CpuState

            self._cpu_state = CpuState(self)
        return self._cpu_state


def get_world() -> Comm:
    """``MPI.COMM_WORLD`` (created lazily; initialises torch.distributed if needed)."""
    global _world
    with _world_lock:
        if _world is None:
            _init_process_group()
            group = _control_group_for_world()
            _world = Comm(group, list(range(dist.get_world_size())), name="COMM_WORLD")
        return _world


def flush() -> None:
    """Wait for every enqueued communication op to finish (reference: the atexit
    ``jax.effects_barrier()``, mpi4jax/_src/__init__.py:13-24)."""
    for comm in list(_comm_registry):
        if comm._cpu_state is not None:
            comm._cpu_state.flush()
        if comm._native is not None:
            comm._native.flush()
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        torch.cuda.synchronize()


def _shutdown() -> None:
    try:
        flush()
    except Exception:  # pragma: no cover - best effort at interpreter exit
        pass
    for comm in list(_comm_registry):
        try:
            comm.Free()
        except Exception:  # pragma: no cover
            pass
    try:
        if dist.is_initialized():
            dist.destroy_process_group()
    except Exception:  # pragma: no cover
        pass


atexit.register(_shutdown)


def _op_types() -> tuple:
    try:  # accept mpi4py operators too when mpi4py happens to be installed
        from mpi4py import MPI as _mpi4py  # type: ignore

        return (Op, _mpi4py.Op)
    except Exception:
        return (Op,)


OP_TYPES = _op_types()
