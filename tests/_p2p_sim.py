"""Executable model of the device-side point-to-point matching protocol (csrc/b2_p2p.cu):
a ring of NSLOT slots per directed pair, fragments numbered consecutively, sender credits from
per-slot acks, receiver state = (head, bitmap of slots consumed out of order).  Mirrors
``p2p_send_role`` / ``p2p_match`` / the end-of-kernel update of ``p2p_recv_role`` line by line so
that the algorithm can be property-tested on a machine without GPUs."""

NSLOT = 8
ANY_TAG = -1


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
    def match(self, recv_tag):
        """p2p_match: sequence number of the message to consume, or None (keep spinning)."""
        head, ooo = self.head, self.ooo
        if recv_tag < 0:
            return head
        i = 0
        while i < NSLOT:
            if (ooo >> i) & 1:
                i += 1
                continue
            sq = head + i
            seq1, tag, nb = self.hdr[sq % NSLOT]
            if seq1 != sq + 1:
                break
            nf = self.nfrag(nb)
            if tag == recv_tag:
                if i != 0 and nf != 1:
                    raise Fatal("a streamed message cannot overtake")
                return sq
            if nf >= NSLOT - i:
                break
            i += nf
        return None

    def try_recv(self, recv_tag, recv_bytes):
        """One receive kernel; returns False if it cannot complete yet (would spin)."""
        seq0 = self.match(recv_tag)
        if seq0 is None:
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


    # ---- ANY_SOURCE support (communicator option p2p_anysource_scan) -----------------------
    def scan(self, recv_tag):
        """Non-blocking variant of match() used by the ANY_SOURCE election: sequence number of the
        message a receive with this tag would take from this source right now, or None.  A streamed
        message that is not at the head is simply 'not available' here (another source may match)."""
        head, ooo = self.head, self.ooo
        if recv_tag < 0:
            return head if self.hdr[head % NSLOT][0] == head + 1 else None
        i = 0
        while i < NSLOT:
            if (ooo >> i) & 1:
                i += 1
                continue
            sq = head + i
            seq1, tag, nb = self.hdr[sq % NSLOT]
            if seq1 != sq + 1:
                return None
            nf = self.nfrag(nb)
            if tag == recv_tag:
                return sq if (i == 0 or nf == 1) else None
            if nf >= NSLOT - i:
                return None
            i += nf
        return None


class Inbox:
    """All directed pairs that end at one receiver: ANY_SOURCE receives (device-side election)."""

    def __init__(self, nsources, slot_bytes=4):
        self.pairs = [Pair(slot_bytes) for _ in range(nsources)]
        self.probe = 0

    def try_recv_any(self, recv_tag):
        """One ANY_SOURCE receive; returns (source, tag, nbytes) or None if nothing matches yet."""
        n = len(self.pairs)
        for _ in range(n):
            src = self.probe
            self.probe = (self.probe + 1) % n
            pair = self.pairs[src]
            pair.pump_sender()
            sq = pair.scan(recv_tag)
            if sq is None:
                continue
            _, tag, nb = pair.hdr[sq % NSLOT]
            # the followers (and lane 0 itself) now run the blocking match on the elected source
            assert pair.match(recv_tag) == sq
            assert pair.try_recv(recv_tag, nb)
            return src, tag, nb
        return None
