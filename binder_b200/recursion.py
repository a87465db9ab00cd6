"""Host mirror of binder's Recursion (lib/recursion.js:285-388) for binder_b200/server.py: a miss the engine hands back
is forwarded to an upstream resolver of its datacenter, and the upstream's response becomes binder's reply on the GPU
(`resolver.relay_batch`, bb_relay_batch: lib/recursion.js:287-327 as a kernel).  Nothing here encodes a DNS answer.

It plugs into Server through options['recursion'], whose resolve(packet, addr, sock) the listener calls for every miss.
UDP misses are answered: the misses of one collection window are forwarded together, their upstream responses (or
nothing, after the 3 s timeout of lib/recursion.js:257) are relayed as ONE batch, and each reply is sent from `sock` to
`addr`.  TCP misses (addr None, on a socket the TCP loop owns) are not answered by this helper; a host that wants them
calls relay_batch(..., tcp=True) itself (Engine.relay_batch, bb_relay_batch with BB_BATCH_TCP).
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
        self.counters = {'relayed': 0, 'forwarded': 0, 'upstream_answers': 0, 'tcp_skipped': 0, 'failed_batches': 0}
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

    def resolve(self, packet, addr, sock):
        """options.recursion.resolve(query, cb) (lib/server.js:110-113,222-225) for one miss."""
        if addr is None:
            self.counters['tcp_skipped'] += 1
            return
        self._q.put((bytes(packet), addr, sock))

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
        try:
            out, out_off, out_len, status = self.resolver.relay_batch(q_data, q_off, u_data, u_off)
        except Exception:                 # BinderError (capacity, CUDA): this window gets no replies
            self.counters['failed_batches'] += 1
            return
        for i, (_, addr, sock) in enumerate(batch):
            if status[i] == 0:
                try:
                    sock.sendto(out[out_off[i]:out_off[i] + out_len[i]].tobytes(), addr)
                    self.counters['relayed'] += 1
                except OSError:
                    pass
