"""Property tests of the p2p matching protocol against an MPI-semantics oracle, on the executable
model in tests/_p2p_sim.py.  The CUDA implementation it mirrors runs schedules that this model
completes, against the same oracle, in tests/collective_ops/test_p2p_kernels.py
(test_p2p_schedules_checked_by_the_model)."""

import random

import pytest

from ._p2p_sim import ANY_TAG, FOUND, NOT_YET, NSLOT, Fatal, Inbox, Pair, _oracle, _reachable, _run


def test_the_model_has_the_kernels_ring_depth():
    """NSLOT of the model is B2_P2P_NSLOT of the library the kernels were built with."""
    from mpi4jax_b200._src import native

    if not native.HAS_CUDA_EXT:
        pytest.skip(f"the native library is not built: {native.CUDA_EXT_ERROR}")
    assert native._abi_native(native.lib)["p2p_nslot"] == NSLOT


def test_in_order_streaming_of_large_messages():
    msgs = [(1, 100), (2, 3), (3, 0), (4, 57)]              # 25 + 1 + 1 + 15 fragments of 4 bytes
    assert _run(msgs, [(0, False), (1, False), (2, True), (3, False)]) == [0, 1, 2, 3]


@pytest.mark.parametrize("order", [(2, 0, 1), (1, 2, 0), (2, 1, 0), (0, 2, 1)])
def test_three_small_messages_any_order(order):
    msgs = [(10, 4), (11, 2), (12, 0)]
    assert _run(msgs, [(k, False) for k in order]) == list(order)


def test_same_tag_never_overtaken():
    msgs = [(1, 4), (7, 4), (7, 4), (1, 4)]
    got = _run(msgs, [(1, False), (2, False), (0, False), (3, False)])
    assert got == [1, 2, 0, 3]


def test_small_message_behind_a_multi_fragment_one():
    msgs = [(3, 12), (5, 4)]                                 # 3 fragments, then 1
    assert _run(msgs, [(1, False), (0, False)]) == [1, 0]


def test_streamed_message_cannot_overtake():
    msgs = [(3, 4), (5, 12)]
    with pytest.raises(Fatal, match="cannot overtake"):
        _run(msgs, [(1, False), (0, False)])


def test_random_schedules_match_the_mpi_oracle():
    rng = random.Random(1234)
    overtakes = 0
    for _ in range(3000):
        n = rng.randint(1, 12)
        msgs = [(rng.randint(0, 3), rng.choice([0, 1, 4, 4, 4, 9, 17, 40])) for _ in range(n)]
        nfr = [Pair(4).nfrag(nb) for _, nb in msgs]
        received, order = set(), []
        while len(received) < n:
            oldest = min(j for j in range(n) if j not in received)
            cands = [(oldest, rng.random() < 0.3)]
            cands += [(k, False) for k in range(oldest + 1, n)
                      if k not in received and _reachable(msgs, nfr, received, k)]
            k, use_any = rng.choice(cands)
            overtakes += k != oldest
            order.append((k, use_any))
            received.add(k)
        recv_tags = [ANY_TAG if a else msgs[k][0] for k, a in order]
        assert _run(msgs, order) == _oracle(msgs, recv_tags), (msgs, order)
    assert overtakes > 1000          # the generator really exercises out-of-order matching


def test_unreachable_message_is_a_deadlock_not_a_wrong_match():
    """More than NSLOT - 1 messages ahead of the head: the receive keeps spinning (the device
    watchdog turns that into a timeout diagnostic), it never matches something else."""
    msgs = [(0, 4)] * NSLOT + [(9, 4)]
    pair = Pair(4)
    for tag, nb in msgs:
        pair.post_send(tag, nb)
    pair.pump_sender()
    assert pair.match(9) == (NOT_YET, None)
    assert pair.try_recv(0, 4)           # consuming the head opens the window
    pair.pump_sender()
    assert pair.match(9) == (FOUND, NSLOT)


def test_any_source_receives_respect_per_source_order():
    """ANY_SOURCE with a tag, in both election modes (the election looks at every source's window, or
    at each source's oldest pending message): whatever source is picked, the message is that source's
    earliest pending one with the tag; every message is received once."""
    for scan in (False, True):
        rng = random.Random(99)
        for _ in range(1500):
            nsrc = rng.randint(1, 5)
            inbox = Inbox(nsrc, scan)
            pending = [[] for _ in range(nsrc)]           # per source: (tag, nbytes) still to be received
            for s in range(nsrc):
                for _ in range(rng.randint(0, 6)):        # <= 6 single-fragment messages: all inside the window
                    tag, nb = rng.randint(0, 3), rng.choice([0, 1, 4])
                    inbox.pairs[s].post_send(tag, nb)
                    pending[s].append((tag, nb))
            total = sum(len(q) for q in pending)
            for _ in range(total):
                # tags the election can find: anywhere in a window when it scans, at a head when it does not
                tags = sorted({t for q in pending for t, _ in (q if scan else q[:1])})
                want = ANY_TAG if rng.random() < 0.25 else rng.choice(tags)
                got = inbox.try_recv_any(want)
                assert got is not None, (scan, pending, want)
                src, tag, nb = got
                assert want == ANY_TAG or tag == want
                if want == ANY_TAG:
                    assert pending[src][0] == (tag, nb)            # the head of that source's queue
                    pending[src].pop(0)
                else:
                    k = next(i for i, (t, _) in enumerate(pending[src]) if t == want)
                    assert pending[src][k] == (tag, nb)            # earliest with that tag from that source
                    pending[src].pop(k)
            assert all(not q for q in pending)
            assert all(p.ooo == 0 and not p.sendq for p in inbox.pairs)


def test_any_source_skips_sources_without_a_match():
    """Both election modes skip sources that hold nothing this receive may take."""
    for scan in (False, True):
        inbox = Inbox(3, scan)
        inbox.pairs[0].post_send(1, 4)
        inbox.pairs[1].post_send(2, 4)
        inbox.pairs[1].post_send(7, 4)
        inbox.pairs[2].post_send(3, 40)                    # streamed message at the head of source 2
        inbox.pairs[2].post_send(7, 40)                    # streamed, not at the head: not available yet
        if scan:
            assert inbox.try_recv_any(7) == (1, 7, 4)      # taken out of order from source 1
        else:
            assert inbox.try_recv_any(7) is None           # no source has tag 7 at its head
            assert inbox.try_recv_any(2) == (1, 2, 4)
            assert inbox.try_recv_any(7) == (1, 7, 4)      # now at the head of source 1
        assert inbox.try_recv_any(7) is None               # source 2's tag-7 message is behind a streamed one
        assert inbox.try_recv_any(3) == (2, 3, 40)
        assert inbox.try_recv_any(7) == (2, 7, 40)
