"""send, recv and sendrecv with peers, byte for byte, in every regime of the p2p kernel (csrc/b2_p2p.cu).

Regimes, by message size n and the communicator's ring slot size (``p2p_slot_bytes``):
 * flag-in-data ("LL") for 1 <= n <= 8192 (B2_P2P_LL_MAX): 4-byte words, a byte path for the last
   partial word; at 4 KiB slots an LL message of 4097..8192 bytes spans two fragments;
 * the slot path with ceil(min(n, slot) / 64 KiB) lanes, capped at 64, whose stripes are rounded to
   16 bytes (the last lanes' stripes can be empty);
 * several fragments per message (n > slot), a ring that wraps inside one message, and messages of at
   least NSLOT fragments, which are larger than the eager capacity NSLOT x slot;
 * the zero-byte message (one empty fragment).
Communicators with 4 KiB, 1 MiB and 16 MiB slots are cloned for the tests.

The oracle never goes through the library: the payload of every message is seeded random bytes of
(case, source, dest, ordinal), viewed as the test's dtype, so every rank builds it itself; bytes 0-7 of
each 16-byte word carry a 64-bit stamp of the message, so no two messages of a test share a 16-byte word
and stale or misplaced data cannot compare equal by luck (bool payloads keep the low bit of every byte
only, as a bool tensor holds 0 and 1; the other dtypes carry the guarantee).  The receiver compares raw
bytes (NaN payloads and -0.0 included) and the Status (source, tag, count); the sender checks after
``m.flush()`` that its tensor is unchanged.  Every rank records a verdict per message, and ``Checks.finish`` makes them agree.
Checks never stop a rank early: a rank that stopped would leave its peer spinning on a message that
never comes.  The schedules of test_p2p_schedules_checked_by_the_model are run on the device only when
the executable model of the matching protocol (tests/_p2p_sim.py) completes them.

In a single-process run the CUDA tests run in a two-rank job whose ranks share the GPU; the launcher at
the end runs the ANY_SOURCE test and the sendrecv ring with three ranks."""

import contextlib
import hashlib
import os
import random

import numpy as np
import pytest
import torch

import mpi4jax_b200 as m
from mpi4jax_b200 import MPI

from .._p2p_sim import ANY_TAG, NSLOT, Fatal, Pair, _oracle, _reachable, _run
from .._peer_job import Checks, expect_passed, job, needs_peers

comm = MPI.COMM_WORLD
rank = comm.Get_rank()
size = comm.Get_size()

peers = needs_peers("p2p kernel between ranks")
# (a two-rank job would report these as skipped, not passed: test_p2p_kernels_three_ranks_gpu runs them)
three_or_more = pytest.mark.skipif(size < 3, reason="needs >= 3 ranks")

LL_MAX = 8192                 # B2_P2P_LL_MAX (csrc/b2_common.h)
LANE = 65536                  # slot-path bytes per lane (lanes_for in csrc/b2_p2p.cu), at most 64 lanes
KIB4, MIB, MIB16 = 4096, 1 << 20, 16 << 20
SLOT_ENV = "MPI4JAX_B200_P2P_SLOT_BYTES"
DTYPES = (torch.uint8, torch.float16, torch.bfloat16, torch.float32, torch.int64, torch.complex128, torch.bool,
          torch.float8_e4m3fn)


def _expect(ok, message):
    assert ok, message


# ---------------------------------------------------------------------------
# messages: payloads every rank can build, posting, verdicts
# ---------------------------------------------------------------------------
class _Payloads:
    """payload(key, nbytes, dtype): the bytes of message ``key`` = (case, source, dest, ordinal)."""

    def __init__(self, chk):
        self.chk = chk
        self.stamps = {}

    def __call__(self, key, nbytes, dtype):
        h = hashlib.blake2b(repr(key).encode(), digest_size=16).digest()
        self.chk(_expect, self.stamps.setdefault(h[:8], key) == key,
                 f"messages {key} and {self.stamps[h[:8]]} have the same stamp")
        raw = np.frombuffer(np.random.default_rng(int.from_bytes(h, "little")).bytes(nbytes), dtype=np.uint8).copy()
        full = nbytes // 16 * 16
        raw[:full].view(np.uint64).reshape(-1, 2)[:, 0] = np.frombuffer(h[:8], dtype=np.uint64)[0]
        if dtype == torch.bool:
            raw &= 1                     # (the only bytes a bool tensor holds: torch copies normalise the others)
        return torch.from_numpy(raw).view(dtype) if nbytes else torch.empty(0, dtype=dtype)


class _Msg:
    """One message: where it goes, its payload (on its source and destination), what was sent and received."""

    def __init__(self, pay, label, key, src, dst, tag, nbytes, dtype):
        self.label = f"{label}: {nbytes} B {str(dtype)[6:]} {src}->{dst} tag {tag}"
        self.src, self.dst, self.tag = src, dst, tag
        self.payload = pay(key, nbytes, dtype) if rank in (src, dst) else None
        self.sent = self.got = self.status = None

    def template(self, device):
        return torch.empty(self.payload.shape, dtype=self.payload.dtype, device=device)


def _send(c, msg, device):
    msg.sent = msg.payload.to(device, copy=True)
    m.send(msg.sent, msg.dst, tag=msg.tag, comm=c)


def _recv(c, msg, device, tag=None, source=None):
    """Receive ``msg`` from its source (``source``: e.g. ANY_SOURCE) with its tag (``tag``: e.g. ANY_TAG)."""
    msg.status = MPI.Status()
    msg.got = m.recv(msg.template(device), msg.src if source is None else source,
                     tag=msg.tag if tag is None else tag, comm=c, status=msg.status)


def _sendrecv(c, out, into, device, recvtag=None):
    out.sent = out.payload.to(device, copy=True)
    into.status = MPI.Status()
    into.got = m.sendrecv(out.sent, into.template(device), source=into.src, dest=out.dst, sendtag=out.tag,
                          recvtag=into.tag if recvtag is None else recvtag, comm=c, status=into.status)


def _same_bytes(got, want, label):
    got = got.detach().cpu()
    assert got.dtype == want.dtype and got.shape == want.shape, (label, got.dtype, got.shape, want.shape)
    g, w = got.contiguous().view(torch.uint8).reshape(-1), want.view(torch.uint8).reshape(-1)
    diff = (g != w).nonzero()
    assert not len(diff), f"{label}: {len(diff)} of {w.numel()} bytes differ, the first at byte {int(diff[0])}"


def _check(msg):
    if rank == msg.dst:
        assert msg.got is not None, f"{msg.label}: never received"
        _same_bytes(msg.got, msg.payload, msg.label)
        if msg.status is not None:
            st = (msg.status.Get_source(), msg.status.Get_tag(), msg.status.Get_count())
            assert st == (msg.src, msg.tag, msg.payload.numel()), f"{msg.label}: Status (source, tag, count) {st}"
    if rank == msg.src:
        _same_bytes(msg.sent, msg.payload, f"{msg.label}: the sender's tensor changed")


def _verify(chk, msgs):
    """After m.flush(): check what this rank sent and received of ``msgs``, one verdict per message that
    every rank records (a rank that takes no part in a message records a pass)."""
    m.flush()
    for msg in msgs:
        n = len(chk.failures)
        if rank in (msg.src, msg.dst):
            chk(_check, msg)
        chk.add(msg.label, torch.tensor([len(chk.failures) == n]))


@contextlib.contextmanager
def _slot_comm(device, chk, slot_bytes):
    """(clone of the world communicator whose p2p ring slots hold ``slot_bytes``, its slot size)."""
    old = os.environ.get(SLOT_ENV)
    os.environ[SLOT_ENV] = str(slot_bytes)
    try:
        c = comm.Clone()                 # its native side is created with these slots
    finally:
        if old is None:
            del os.environ[SLOT_ENV]
        else:
            os.environ[SLOT_ENV] = old
    try:
        slot = slot_bytes
        if device.type == "cuda":
            slot = c._native_comm().get_option("p2p_slot_bytes")
            chk(_expect, slot == slot_bytes, f"{SLOT_ENV}={slot_bytes} gave {slot}-byte slots")
        yield c, slot
    finally:
        m.flush()
        c.Free()


def _anysource_scan(c, device, on):
    if device.type == "cuda":
        c._native_comm().set_option("p2p_anysource_scan", on)


def _dtypes_for(nbytes, i):
    """The dtypes whose item size divides ``nbytes``; above 128 KiB only one of them (the i-th in turn)."""
    fit = [d for d in DTYPES if nbytes % d.itemsize == 0]
    return fit if nbytes <= 2 * LANE + 1 else [fit[i % len(fit)]]


# ---------------------------------------------------------------------------
# sizes and dtypes
# ---------------------------------------------------------------------------
SIZES = (
    (MIB16, (0, 1, 2, 3, 4, 5, 15, 16, 17, 4095, 4096, 4097,
             LL_MAX - 4, LL_MAX - 3, LL_MAX - 1, LL_MAX, LL_MAX + 1, LL_MAX + 4, LL_MAX + 16,
             LANE - 1, LANE, LANE + 1, 2 * LANE + 1,
             64 * LANE - 1, 64 * LANE, 64 * LANE + 1,          # 64 lanes; the last one's stripe is 1 B or empty
             MIB16 - 1, MIB16, MIB16 + 1)),                  # the second fragment of 16 MiB + 1: 1 B over 64 lanes
    (KIB4, (4097, 8192, 8193, 7 * KIB4, NSLOT * KIB4, NSLOT * KIB4 + 1, 20 * KIB4 + 5)),
    (MIB, (MIB - 1, MIB + 1, 8 * MIB + 1)),                     # 16 lanes; 8 MiB + 1: 9 fragments
)


@peers
def test_p2p_sizes_and_dtypes(device):
    """Every size class and its edges, in every dtype whose item size divides the byte count: 0 -> 1 and
    1 -> 0 (rank 0 sends first, rank 1 receives first), and a self sendrecv on every rank."""
    chk = Checks()
    pay = _Payloads(chk)
    for slot_req, counts in SIZES:
        with _slot_comm(device, chk, slot_req) as (c, slot):
            for i, nbytes in enumerate(counts):
                for dtype in _dtypes_for(nbytes, i):
                    case = ("sizes", slot, nbytes, str(dtype))
                    label = f"slot {slot}"
                    tag = 10 + i % 7
                    a = _Msg(pay, label, (case, 0, 1, 0), 0, 1, tag, nbytes, dtype)
                    b = _Msg(pay, label, (case, 1, 0, 0), 1, 0, tag + 1, nbytes, dtype)
                    selfs = [_Msg(pay, f"{label} self", (case, q, q, 0), q, q, tag + 2, nbytes, dtype)
                             for q in range(size)]
                    if rank == 0:
                        _send(c, a, device)
                        _recv(c, b, device, tag=ANY_TAG if i % 2 else None)
                    elif rank == 1:
                        _recv(c, a, device, tag=ANY_TAG if i % 3 == 0 else None)
                        _send(c, b, device)
                    _sendrecv(c, selfs[rank], selfs[rank], device)
                    _verify(chk, [a, b, *selfs])
    chk.finish()


# ---------------------------------------------------------------------------
# sendrecv whose two directions are in different regimes
# ---------------------------------------------------------------------------
MIXED = (
    (MIB16, ((5, 64 * LANE + 1), (0, MIB16 + 1), (LL_MAX, LL_MAX + 1), (LANE + 1, MIB16), (17, 0))),
    # both directions larger than the eager capacity NSLOT x slot: they stream through the rings together
    (KIB4, ((20 * KIB4 + 5, 9 * KIB4 + 3), (8193, 4097), (0, 20 * KIB4 + 5), (3, NSLOT * KIB4))),
    (MIB, ((8 * MIB + 1, 9 * MIB + 7), (1, MIB + 1))),
)


@peers
def test_sendrecv_mixed_regimes(device):
    """A ring shift (a swap with two ranks) in which rank q sends sizes[q % 2] to q + 1: the send and the
    receive role of one kernel are in different regimes, with independent lane counts."""
    chk = Checks()
    pay = _Payloads(chk)
    for slot_req, pairs in MIXED:
        with _slot_comm(device, chk, slot_req) as (c, slot):
            for j, pair in enumerate(pairs):
                for flip in (0, 1):
                    case = ("mixed", slot, j, flip)
                    msgs = []
                    for q in range(size):
                        nbytes = pair[(q + flip) % 2]
                        fit = [d for d in DTYPES if nbytes % d.itemsize == 0]
                        msgs.append(_Msg(pay, f"sendrecv ring slot {slot}", (case, q, (q + 1) % size, 0), q,
                                         (q + 1) % size, 30 + q, nbytes, fit[(j + q) % len(fit)]))
                    _sendrecv(c, msgs[rank], msgs[(rank - 1) % size], device, recvtag=ANY_TAG if flip else None)
                    _verify(chk, msgs)
    chk.finish()


# ---------------------------------------------------------------------------
# random schedules the matching model completes
# ---------------------------------------------------------------------------
def _schedules(chk, slot, count, max_msgs, seed):
    """``count`` random (messages, receive order, oracle order) that the model completes with ``slot``-byte
    slots -- the generator of test_random_schedules_match_the_mpi_oracle with the kernel's size classes.  A
    receive of the order is (message, ANY_TAG?); the model's and the oracle's match must agree."""
    rng = random.Random(seed)
    sizes = (0, 6, 8192, 8193, slot - 1, slot, slot + 1, 3 * slot + 7, (NSLOT + 1) * slot)
    out, rejected = [], 0
    while len(out) < count:
        n = rng.randint(1, max_msgs)
        msgs = [(rng.randint(0, 3), rng.choice(sizes)) for _ in range(n)]
        nfr = [Pair(slot).nfrag(nb) for _, nb in msgs]
        received, order = set(), []
        while len(received) < n:
            oldest = min(j for j in range(n) if j not in received)
            cands = [(oldest, rng.random() < 0.3)]
            cands += [(k, False) for k in range(oldest + 1, n)
                      if k not in received and _reachable(msgs, nfr, received, k)]
            k, use_any = rng.choice(cands)
            order.append((k, use_any))
            received.add(k)
        try:
            got = _run(msgs, order, slot)
        except (Fatal, AssertionError):          # a fatal error or a deadlock on the device: not run there
            rejected += 1
            continue
        want = _oracle(msgs, [ANY_TAG if a else msgs[k][0] for k, a in order])
        chk(_expect, got == want, f"the model matches {got}, the oracle {want}: {msgs} {order}")
        if got == want:
            out.append((msgs, order, want))
    return out, rejected


@peers
def test_p2p_schedules_checked_by_the_model(device):
    """Random schedules of up to 12 tagged messages between two ranks (sizes around the LL limit and the
    slot size, up to NSLOT + 1 fragments), received in an order the model completes, with out-of-order
    tagged and ANY_TAG receives: each receive gets the oracle's message, in the model's order."""
    chk = Checks()
    pay = _Payloads(chk)
    for slot_req, count, max_msgs in ((KIB4, 100, 12), (MIB, 10, 6)):
        with _slot_comm(device, chk, slot_req) as (c, slot):
            for s, d in ((0, 1), (1, 0)):
                scheds, rejected = _schedules(chk, slot, count, max_msgs, repr(("schedules", slot, s, d)))
                chk(_expect, rejected < count, f"slot {slot}: the model rejected {rejected} schedules")
                for j, (msgs, order, want) in enumerate(scheds):
                    case = ("schedule", slot, s, d, j)
                    ms = [_Msg(pay, f"schedule {j} slot {slot} message {k}", (case, s, d, k), s, d, tag, nb,
                               torch.uint8) for k, (tag, nb) in enumerate(msgs)]
                    if rank == s:
                        for msg in ms:
                            _send(c, msg, device)
                    if rank == d:
                        for (k, use_any), w in zip(order, want):
                            _recv(c, ms[w], device, tag=ANY_TAG if use_any else msgs[k][0])
                    _verify(chk, [ms[w] for w in want])
    chk.finish()


# ---------------------------------------------------------------------------
# ANY_SOURCE with two real senders
# ---------------------------------------------------------------------------
# None: slot + 1 bytes (two fragments), received with ANY_TAG only
ANY_SOURCE_CASES = ((MIB16, (6, LL_MAX, LL_MAX + 1, LANE + 1)), (KIB4, (None,)), (MIB, (None,)))


def _receive_any(c, chk, ms, tags, nbytes, scan, any_only, device, rng):
    """Rank 0 receives every message of ``ms`` from ANY_SOURCE, choosing each tag from what is still
    pending (its own bookkeeping, updated from the Status): a tag at the head of some source's queue
    (default election) or any pending tag (scan election), or ANY_TAG.  If the bookkeeping breaks, the
    rest is drained with ANY_TAG, so no sender is left blocked."""
    pending = {s: list(range(len(tags[s]))) for s in tags}
    broken = False
    for _ in range(sum(len(q) for q in pending.values())):
        if any_only or broken:
            want = ANY_TAG
        elif scan:
            want = rng.choice(sorted({tags[s][k] for s in pending for k in pending[s]}) + [ANY_TAG])
        else:
            want = rng.choice(sorted({tags[s][q[0]] for s, q in pending.items() if q}) + [ANY_TAG])
        st = MPI.Status()
        got = m.recv(torch.empty(nbytes, dtype=torch.uint8, device=device), MPI.ANY_SOURCE, tag=want, comm=c,
                     status=st)
        src, tag = st.Get_source(), st.Get_tag()
        # the earliest pending message of that source with that tag (ANY_TAG: the head of its queue)
        ks = [k for k in pending.get(src, ()) if tags[src][k] == tag]
        if broken or not ks or (want != ANY_TAG and tag != want) or (want == ANY_TAG and ks[0] != pending[src][0]):
            chk(_expect, broken, f"ANY_SOURCE receive with tag {want}: Status names source {src} tag {tag}, "
                                 f"pending {pending}")
            broken = True
            continue
        pending[src].remove(ks[0])
        ms[src, ks[0]].got, ms[src, ks[0]].status = got, st


@three_or_more
def test_any_source_with_two_senders(device):
    """Ranks 1 and 2 send tagged messages of one size (a wrong template would be a fatal truncation, and
    the election decides the source) to rank 0, which receives them all from ANY_SOURCE in both election
    modes (communicator option p2p_anysource_scan); the multi-fragment size slot + 1 with ANY_TAG only.
    Every message is received once, as the earliest pending one of its source with its tag."""
    chk = Checks()
    pay = _Payloads(chk)
    senders = (1, 2)
    for slot_req, sizes in ANY_SOURCE_CASES:
        with _slot_comm(device, chk, slot_req) as (c, slot):
            for scan in (0, 1):
                _anysource_scan(c, device, scan)
                for nbytes in sizes:
                    any_only = nbytes is None
                    nbytes = slot + 1 if any_only else nbytes
                    # at most NSLOT fragments per sender in flight; scan mode: every tag inside the window
                    per_src = NSLOT // 2 if any_only else NSLOT - 2 if scan else NSLOT
                    case = ("any source", slot, scan, nbytes)
                    rng = random.Random(repr(case))
                    tags = {s: [rng.randint(0, 3) for _ in range(per_src)] for s in senders}
                    ms = {(s, k): _Msg(pay, f"any source slot {slot} scan {scan} message {k}", (case, s, 0, k), s, 0,
                                       tags[s][k], nbytes, torch.uint8) for s in senders for k in range(per_src)}
                    if rank in senders:
                        for k in range(per_src):
                            _send(c, ms[rank, k], device)
                    if rank == 0:
                        _receive_any(c, chk, ms, tags, nbytes, scan, any_only, device, rng)
                    _verify(chk, list(ms.values()))
                    # the next case's messages have another size: none may be sent while rank 0 still receives
                    # this case's (an ANY_SOURCE receive with a tag would rightly match one of them)
                    c.Barrier()
    chk.finish()


# ---------------------------------------------------------------------------
# a captured sequence replayed with new inputs
# ---------------------------------------------------------------------------
# (tag, bytes) sent 0 -> 1 on 1 MiB slots: LL with a byte tail, 5 lanes, zero bytes, 3 fragments x 16 lanes,
# and a small message received ahead of the streamed one; then 1 -> 0: the largest LL message, 2 lanes, 2 fragments
REPLAY = ((0, 1, ((1, 777), (2, 5 * LANE - 13), (3, 0), (4, 5 * MIB // 2 + 9), (5, 40)),
           ((0, False), (1, False), (2, True), (4, False), (3, False))),
          (1, 0, ((6, LL_MAX), (7, LANE + 1), (8, MIB + 1)), ((0, True), (1, False), (2, False))))


@peers
def test_p2p_graph_replay_with_fresh_inputs(device):
    """The REPLAY sequence as one m.jit function (a warm-up call, the capture, then replays), called 7
    times with new payloads: the device-side sequence numbers advance through slot reuse under replay,
    and stale slot contents cannot pass."""
    chk = Checks()
    pay = _Payloads(chk)
    with _slot_comm(device, chk, MIB) as (c, slot):
        plans = []
        for s, d, msgs, order in REPLAY:
            want = _oracle(msgs, [ANY_TAG if a else msgs[k][0] for k, a in order])
            assert _run(msgs, order, slot) == want         # (on every rank alike, before any message)
            plans.append((s, d, msgs, order, want))

        def step(*xs):
            outs = []
            for s, d, msgs, order, want in plans:
                if rank == s:
                    for x, (tag, _) in zip(xs, msgs):
                        m.send(x, d, tag=tag, comm=c)
                elif rank == d:
                    for (k, use_any), w in zip(order, want):
                        outs.append(m.recv(torch.empty(msgs[w][1], dtype=torch.uint8, device=device), s,
                                           tag=ANY_TAG if use_any else msgs[k][0], comm=c))
            return tuple(outs)

        f = m.jit(step)
        for call in range(7):
            ms = [[_Msg(pay, f"replay call {call}", ("replay", call, s, d, k), s, d, tag, nb, torch.uint8)
                   for k, (tag, nb) in enumerate(msgs)] for s, d, msgs, _, _ in plans]
            mine = [plan for plan in range(len(plans)) if plans[plan][0] == rank]
            if rank in (0, 1):
                xs = [msg.payload.to(device, copy=True) for p in mine for msg in ms[p]]
                outs = iter(f(*xs))
                for p, (s, d, msgs, order, want) in enumerate(plans):
                    if rank == s:
                        for msg, x in zip(ms[p], xs):
                            msg.sent = x
                    elif rank == d:
                        for w in want:
                            ms[p][w].got = next(outs)
            _verify(chk, [msg for p in ms for msg in p])
    chk.finish()


# ---------------------------------------------------------------------------
# three ranks
# ---------------------------------------------------------------------------
_inside_job = size > 1 or "MPI4JAX_B200_NESTED" in os.environ


@pytest.mark.gpu
@pytest.mark.skipif(_inside_job, reason="already inside a multi-rank job")
def test_p2p_kernels_three_ranks_gpu():
    """P = 3: two real senders for the ANY_SOURCE election, and the sendrecv ring in which every kernel
    sends and receives in different regimes."""
    code, outs = job(__file__, 3, "test_any_source_with_two_senders or test_sendrecv_mixed_regimes")
    expect_passed(code, outs, 3, ["test_any_source_with_two_senders", "test_sendrecv_mixed_regimes"])
