"""Executable model of the device-side point-to-point matching protocol (csrc/b2_p2p.cu):
a ring of NSLOT slots per directed pair, fragments numbered consecutively, sender credits from
per-slot acks, receiver state = (head, bitmap of slots consumed out of order).  Mirrors
``p2p_send_role`` / ``p2p_walk`` / the end-of-kernel update of ``p2p_recv_role`` line by line so
that the algorithm can be property-tested on a machine without GPUs."""

NSLOT = 8
ANY_TAG = -1
FOUND, NOT_YET, STREAMED_BEHIND = range(3)      # the three results of one pass over a window


class Fatal(Exception):
    pass


class Pair:
    """One directed (source -> dest) pair."""

    def __init__(self, slot_bytes=4):
        self.slot_bytes = slot_bytes
        # receiver-side memory written by the sender: per slot (seq+1, tag, nbytes)
        self.hdr = [(0, 0, 0)] * NSLOT
        # sender-side memory written by the receiver: per slot ack = fs + 1 of the consumed fragment
        self.ack = [0] * NSLOT
        self.send_seq = 0        # c.p2p_send_seq[dest]
        self.head = 0            # c.p2p_recv_seq[src]
        self.ooo = 0             # c.p2p_ctl[CTL_OOO + src]
        self.sendq = []          # fragments the sender still has to write: (fs, tag, nbytes)
        self.log = []            # (seq0, tag, nbytes) of every completed receive

    # ---- sender ---------------------------------------------------------------------------
    def nfrag(self, nbytes):
        return 1 if nbytes == 0 else -(-nbytes // self.slot_bytes)

    def post_send(self, tag, nbytes):
        for f in range(self.nfrag(nbytes)):
            self.sendq.append((self.send_seq + f, tag, nbytes))
        self.send_seq += self.nfrag(nbytes)

    def pump_sender(self):
        """Write every fragment whose slot credit is available (b2_wait_ge on ack[slot])."""
        progressed = False
        while self.sendq:
            fs, tag, nbytes = self.sendq[0]
            slot = fs % NSLOT
            if self.ack[slot] < fs + 1 - NSLOT:          # previous occupant not consumed yet
                break
            self.hdr[slot] = (fs + 1, tag, nbytes)
            self.sendq.pop(0)
            progressed = True
        return progressed

    # ---- receiver -------------------------------------------------------------------------
    def match(self, recv_tag, window=NSLOT):
        """p2p_walk: one pass over the `window` fragments from the head.  Returns (FOUND, seq) of
        the message to consume, (NOT_YET, None), or (STREAMED_BEHIND, seq) for a streamed message
        with the tag that is not at the head.  With a window of one only bit 0 of the bitmap is
        read, and it is never set at the head: the kernel's default election passes an empty one."""
        head, ooo = self.head, self.ooo
        i = 0
        while i < window:
            if (ooo >> i) & 1:
                i += 1
                continue
            sq = head + i
            seq1, tag, nb = self.hdr[sq % NSLOT]
            if seq1 != sq + 1:
                break
            nf = self.nfrag(nb)
            if recv_tag < 0 or tag == recv_tag:
                return (FOUND if i == 0 or nf == 1 else STREAMED_BEHIND), sq
            if nf >= window - i:
                break
            i += nf
        return NOT_YET, None

    def try_recv(self, recv_tag, recv_bytes):
        """One receive kernel; returns False if it cannot complete yet (would spin)."""
        res, seq0 = self.match(recv_tag)
        if res == STREAMED_BEHIND:
            raise Fatal("a streamed message cannot overtake")
        if res == NOT_YET:
            return False
        nfrag = self.nfrag(recv_bytes)
        for f in range(nfrag):
            fs = seq0 + f
            slot = fs % NSLOT
            while self.hdr[slot][0] != fs + 1:           # b2_wait_eq on the fragment header
                if not self.pump_sender():
                    if f == 0:
                        return False                      # nothing consumed yet: safe to retry later
                    raise Fatal("receiver stuck inside a message (sender cannot progress)")
            seq1, tag, nb = self.hdr[slot]
            if f == 0:
                if recv_tag >= 0 and tag != recv_tag:
                    raise Fatal("tag mismatch")
                if nb != recv_bytes:
                    raise Fatal("truncate")
            self.ack[slot] = fs + 1
        # end-of-kernel update by the last lane
        if seq0 == self.head:
            nh = self.head + nfrag
            ooo = 0 if nfrag >= NSLOT else (self.ooo >> nfrag)
            while ooo & 1:
                ooo >>= 1
                nh += 1
            self.head, self.ooo = nh, ooo
        else:
            self.ooo |= 1 << (seq0 - self.head)
        self.log.append((seq0, self.hdr[seq0 % NSLOT][1], recv_bytes))
        return True


class Inbox:
    """All directed pairs that end at one receiver: ANY_SOURCE receives (device-side election).
    `scan`: the communicator option p2p_anysource_scan; the election looks into every source's
    window if set, at the oldest pending message of each source (a window of one) if not.  A
    streamed message behind the head is 'not here' for the election: another source may match."""

    def __init__(self, nsources, scan, slot_bytes=4):
        self.pairs = [Pair(slot_bytes) for _ in range(nsources)]
        self.window = NSLOT if scan else 1
        self.probe = 0

    def try_recv_any(self, recv_tag):
        """One ANY_SOURCE receive; returns (source, tag, nbytes) or None if nothing matches yet."""
        n = len(self.pairs)
        for _ in range(n):
            src = self.probe
            self.probe = (self.probe + 1) % n
            pair = self.pairs[src]
            pair.pump_sender()
            res, sq = pair.match(recv_tag, self.window)
            if res != FOUND:
                continue
            _, tag, nb = pair.hdr[sq % NSLOT]
            # the followers (and lane 0 itself) now run the blocking match on the elected source
            assert pair.match(recv_tag) == (FOUND, sq)
            assert pair.try_recv(recv_tag, nb)
            return src, tag, nb
        return None


# ---- schedules: the MPI oracle, the model run and the reachability rule of a tagged receive ----
def _oracle(messages, recv_tags):
    """MPI matching: each receive takes the earliest not-yet-received message with its tag."""
    taken, order = set(), []
    for t in recv_tags:
        for k, (tag, _) in enumerate(messages):
            if k not in taken and (t == ANY_TAG or tag == t):
                taken.add(k)
                order.append(k)
                break
        else:
            raise AssertionError("test generator produced an unmatched receive")
    return order


def _run(messages, recv_order, slot_bytes=4):
    """messages: [(tag, nbytes)] sent in order; recv_order: indices in the order they are received
    (each receive uses the message's tag, or ANY_TAG when flagged)."""
    pair = Pair(slot_bytes)
    for tag, nb in messages:
        pair.post_send(tag, nb)
    starts, s = [], 0
    for tag, nb in messages:
        starts.append(s)
        s += pair.nfrag(nb)
    pending = list(recv_order)
    guard = 0
    while pending:
        pair.pump_sender()
        k, use_any = pending[0]
        tag, nb = messages[k]
        if pair.try_recv(ANY_TAG if use_any else tag, nb):
            pending.pop(0)
            guard = 0
        else:
            guard += 1
            assert guard < 4, "deadlock in the model: nothing can progress"
    pair.pump_sender()
    assert not pair.sendq, "sender still blocked after every message was received"
    assert pair.head == s and pair.ooo == 0, (pair.head, s, bin(pair.ooo))
    return [starts.index(seq0) for seq0, _, _ in pair.log]


def _reachable(msgs, nfr, received, k):
    """Can a tagged receive for message k see it?  Replays the walk of p2p_match on the send order:
    holes (already received, single-fragment) cost one slot, older unreceived messages are hopped
    over, a message whose fragments fill the rest of the window ends the scan."""
    first = min(j for j in range(len(msgs)) if j not in received)
    i = 0
    for j in range(first, len(msgs)):
        if i >= NSLOT:
            return False
        if j in received:
            i += 1
            continue
        if j == k:
            return i == 0 or nfr[k] == 1
        if msgs[j][0] == msgs[k][0]:
            return False                 # an older message with the same tag would be matched instead
        if nfr[j] >= NSLOT - i:
            return False
        i += nfr[j]
    return False
