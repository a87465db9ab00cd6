"""Host mirror of binder's Recursion (lib/recursion.js:285-388) for binder_b200/server.py: a miss the engine hands back
is forwarded to an upstream resolver of its datacenter, and the upstream's response becomes binder's reply on the GPU
(`resolver.relay_batch`, bb_relay_batch: lib/recursion.js:287-327 as a kernel).  Nothing here encodes a DNS answer.

It plugs into Server through options['recursion'].  The misses of one collection window, from every transport, are
forwarded together (the exchange); their upstream responses (or nothing, after the 3 s timeout of lib/recursion.js:257)
are then delivered per transport owner (the delivery):
  - resolve(packet, addr, sock): a UDP miss of a listener this object may send from.  The window's UDP misses are relayed
    as ONE batch and each reply is sent from `sock` to `addr`.  resolve(packet, None, sock) is a TCP miss of a caller that
    has not moved to submit(): it is counted in tcp_skipped and not answered.
  - submit(packet, sink, tag): a miss of a transport owner (the TCP loop, a balancer session, a TCP hub).  After the
    exchange each sink with misses in the window is called once, sink.relay(q_data, q_off, up, up_off, tags), with its
    misses in miss order; up[up_off[i]:up_off[i+1]] is miss i's upstream response, empty when the lookup failed.  A sink
    belongs to an owner, not to a connection or a session: the tag tells the owner's connections apart, so a window costs
    at most one relay launch per owner.
Sinks run on the recursion thread.  QueueSink hands a window to a single-threaded owner, which relays it with its own
engine (relay_batch, tcp=True over TCP) and frames the replies for its transport.
"""
import os
import queue
import select
import socket
import struct
import threading
import time

from .server import pack_packets

QT_PTR = 12


def _question(pkt):
    """(QNAME wire bytes, QTYPE, QCLASS, dotted name) of a query the engine accepted, or None."""
    pos = 12
    while pos < len(pkt) and pkt[pos]:
        pos += 1 + pkt[pos]
    if pos + 5 > len(pkt):
        return None
    wire = pkt[12:pos + 1]
    qtype, qclass = struct.unpack('>HH', pkt[pos + 1:pos + 5])
    labels, p = [], 0
    while wire[p]:
        labels.append(wire[p + 1:p + 1 + wire[p]].decode('latin-1'))
        p += 1 + wire[p]
    return wire, qtype, qclass, '.'.join(labels)


def split_packets(data, off):
    """(packed data, offsets[n+1]) -> [bytes]"""
    return [bytes(data[int(off[i]):int(off[i + 1])]) for i in range(len(off) - 1)]


class QueueSink(object):
    """The sink of a single-threaded transport owner.  relay() runs on the recursion thread: it queues the window's
    (q_data, q_off, up, up_off, tags) and calls wake(); the owner calls drain() on its own thread."""

    def __init__(self, wake=None):
        self._lock = threading.Lock()
        self._items = []
        self._wake = wake

    def relay(self, q_data, q_off, up, up_off, tags):
        with self._lock:
            self._items.append((q_data, q_off, up, up_off, list(tags)))
        if self._wake is not None:
            self._wake()

    def drain(self):
        """-> [(q_data, q_off, up, up_off, tags)] queued since the last drain, oldest first"""
        with self._lock:
            items, self._items = self._items, []
        return items


class UdpSink(object):
    """resolve()'s delivery: the window's UDP misses relayed as one batch on `resolver`, each reply sent from the
    listener's socket to the client; the tag is (addr, sock, when the query arrived).  A failed relay batch gets no replies and is counted."""

    def __init__(self, resolver, counters):
        self.resolver, self.counters = resolver, counters
        self.query_log = None             # binder_b200.query_log.QueryLog: a line per reply sent (the server's sink)

    def relay(self, q_data, q_off, up, up_off, tags):
        try:
            out, out_off, out_len, status = self.resolver.relay_batch(q_data, q_off, up, up_off)
        except Exception:                 # BinderError (capacity, CUDA): this window gets no replies
            self.counters['failed_batches'] += 1
            return
        for i, (addr, sock, _) in enumerate(tags):
            if status[i] == 0:
                try:
                    sock.sendto(out[out_off[i]:out_off[i] + out_len[i]].tobytes(), addr)
                    self.counters['relayed'] += 1
                except OSError:
                    pass
        if self.query_log is not None:
            self.query_log.write(self.resolver, out, out_off, out_len, status, [t[0] for t in tags], [t[2] for t in tags])


def deliver(batch, q_data, q_off, up, up_off, counters):
    """The delivery of one window: batch[i] = (packet, sink, tag), (q_data, q_off) its packets and (up, up_off) their
    upstream responses, packed in batch order.  Each sink is called once, with its own misses in batch order."""
    groups = {}
    for i, (_, sink, _) in enumerate(batch):
        groups.setdefault(id(sink), (sink, []))[1].append(i)
    for sink, idx in groups.values():
        if len(idx) == len(batch):
            q, qo, u, uo = q_data, q_off, up, up_off
        else:
            q, qo = pack_packets([bytes(q_data[int(q_off[i]):int(q_off[i + 1])]) for i in idx])
            u, uo = pack_packets([bytes(up[int(up_off[i]):int(up_off[i + 1])]) for i in idx])
        if not isinstance(sink, UdpSink):
            counters['delivered'] += len(idx)
        sink.relay(q, qo, u, uo, [batch[i][2] for i in idx])


class Recursion(object):
    """resolver   an Engine created with recursion=True that this object uses alone (or anything with the same
                  relay_batch, such as the CPU oracle in the tests)
    dns_domain    Recursion's opts.dnsDomain (the region domain)
    dcs           datacenter name -> upstream resolvers, each 'ip' (port 53) or (ip, port)   (self.dcs, :205-240)
    my_addrs      this host's own addresses: upstreams among them are skipped (:360-379)"""

    def __init__(self, resolver, dns_domain, dcs, my_addrs=(), timeout=3.0, window_s=0.002):
        self.resolver = resolver
        self.dnsDomain = dns_domain
        self.dcs = {dc: [a if isinstance(a, tuple) else (a, 53) for a in addrs] for dc, addrs in dcs.items()}
        self.my_addrs = set(my_addrs)
        self.timeout = timeout
        self.window_s = window_s
        self.counters = {'relayed': 0, 'forwarded': 0, 'upstream_answers': 0, 'tcp_skipped': 0, 'failed_batches': 0,
                         'delivered': 0}
        self._udp = UdpSink(resolver, self.counters)
        self._q = queue.Queue()
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._loop, daemon=True)
        self._thread.start()

    def upstreams(self, name, qtype):
        """The quick rejects of Recursion.prototype.resolve (:329-379): where this query would be forwarded."""
        d = self.dnsDomain
        if qtype != QT_PTR:
            if name.find(d, max(len(name) - len(d), 0)) == -1:           # indexOf(dnsDomain, length - dnsDomain.length)
                return []
            p = name[:max(len(name) - len(d) - 1, 0)]
            ups = self.dcs.get(p[p.rfind('.') + 1:], [])
        else:
            ups = [a for addrs in self.dcs.values() for a in addrs]
        return [a for a in ups if a[0] not in self.my_addrs]

    def resolve(self, packet, addr, sock, received=None):
        """options.recursion.resolve(query, cb) (lib/server.js:110-113,222-225) for one miss.  received: when the query
        arrived (time.time(); default now), the start of its query log line's latency."""
        if addr is None:
            self.counters['tcp_skipped'] += 1
            return
        self._q.put((bytes(packet), self._udp, (addr, sock, time.time() if received is None else received)))

    def set_query_log(self, query_log):
        """The server's query log sink (binder_b200.query_log.QueryLog): relayed UDP replies get their lines too."""
        self._udp.query_log = query_log

    def submit(self, packet, sink, tag):
        """One miss of a transport owner: its reply comes back through sink.relay(..., tags) with `tag`."""
        self._q.put((bytes(packet), sink, tag))

    def close(self):
        self._stop.set()
        self._thread.join(self.timeout + 2)

    # ---- one collection window at a time -----------------------------------------------------------------------------
    def _loop(self):
        while not self._stop.is_set():
            try:
                batch = [self._q.get(timeout=0.05)]
            except queue.Empty:
                continue
            deadline = time.perf_counter() + self.window_s
            while time.perf_counter() < deadline:
                try:
                    batch.append(self._q.get(timeout=max(deadline - time.perf_counter(), 1e-4)))
                except queue.Empty:
                    break
            self._relay(batch)

    def _exchange(self, batch):
        """Upstream query per miss (the client's question, RD cleared as lookup() does with msg.clearFlag('rd'),
        :253-262; a fresh ID, no OPT), sent to every upstream of its datacenter; the first response whose ID and source
        match is kept.  -> [response bytes or b'']."""
        answers = [b''] * len(batch)
        pending = {}
        s = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        try:
            s.setblocking(False)
            for i, (pkt, _, _) in enumerate(batch):
                q = _question(pkt)
                if q is None:
                    continue
                wire, qtype, qclass, name = q
                ups = self.upstreams(name, qtype)
                if not ups:
                    continue
                qid = struct.unpack('>H', os.urandom(2))[0]
                while qid in pending:
                    qid = (qid + 1) & 0xFFFF
                flags = struct.unpack('>H', pkt[2:4])[0] & 0x7800               # opcode; RD cleared
                msg = struct.pack('>HHHHHH', qid, flags, 1, 0, 0, 0) + wire + struct.pack('>HH', qtype, qclass)
                pending[qid] = (i, set(ups))
                for up in ups:
                    try:
                        s.sendto(msg, up)
                    except OSError:
                        pass
                self.counters['forwarded'] += 1
            end = time.perf_counter() + self.timeout
            while pending and time.perf_counter() < end:
                r, _, _ = select.select([s], [], [], max(end - time.perf_counter(), 0))
                if not r:
                    break
                try:
                    data, src = s.recvfrom(65535)
                except OSError:
                    continue
                if len(data) < 2:
                    continue
                hit = pending.get(struct.unpack('>H', data[:2])[0])
                if hit and src in hit[1]:
                    answers[hit[0]] = data
                    del pending[struct.unpack('>H', data[:2])[0]]
                    self.counters['upstream_answers'] += 1
        finally:
            s.close()
        return answers

    def _relay(self, batch):
        ups = self._exchange(batch)
        q_data, q_off = pack_packets([p for p, _, _ in batch])
        u_data, u_off = pack_packets(ups)
        deliver(batch, q_data, q_off, u_data, u_off, self.counters)
