"""GpuRecursion: binder's Recursion (lib/recursion.js:253-388) for binder_b200/server.py with the upstream exchange on the
GPU.  Same interface as binder_b200.recursion.Recursion — resolve(packet, addr, sock) for a UDP miss, submit(packet,
sink, tag) for a miss of another transport owner, close() — so Server takes it through options['recursion'] unchanged.

Per collection window, the exchange (transport-blind): bb_forward_batch builds every miss's upstream query (keyed IDs,
RD cleared, no OPT) and groups them by datacenter; the host sends each datacenter's run to each of its upstreams from
one fresh socket; it receives until every forwarded miss has an accepted response or the 3 s of lib/recursion.js:257
have passed, and bb_match_upstreams picks each miss's response.  Then the delivery (recursion.deliver): the UDP misses'
replies are built by one bb_relay_batch and go out from the listener's socket; every other sink gets its misses and
their upstream responses once.  The host reads no byte of a query or a response: its per-miss work is the socket calls.
"""
import os
import queue
import select
import socket
import threading
import time

import numpy as np

from .engine import FORWARD_ROUTES, ROUTE_PTR, ip_u32
from .recursion import UdpSink, deliver
from .server import pack_packets

FORWARD_MAX = 65536


class GpuRecursion(object):
    """resolver   an Engine created with recursion=True that this object uses alone (it sets the engine's recursion
                  filter and upstream table), or anything with the same set_recursion_filter, set_recursion_upstreams,
                  forward_batch, match_upstreams and relay_batch
    dns_domain    Recursion's opts.dnsDomain (the region domain)
    dcs           datacenter name -> upstream resolvers, each 'ip' (port 53) or (ip, port), IPv4   (self.dcs, :205-240)
    my_addrs      this host's own addresses: upstreams among them are skipped (:360-379)"""

    def __init__(self, resolver, dns_domain, dcs, my_addrs=(), timeout=3.0, window_s=0.002):
        self.resolver = resolver
        self.dnsDomain = dns_domain
        mine = set(my_addrs)
        ups = {dc: [a if isinstance(a, tuple) else (a, 53) for a in addrs] for dc, addrs in dcs.items()}
        ups = {dc: [a for a in addrs if a[0] not in mine] for dc, addrs in ups.items()}
        self.dc_names = [dc for dc, addrs in ups.items() if addrs]
        if len(self.dc_names) > 16:
            raise ValueError('at most 16 datacenters with upstreams')
        # route r < 16: the upstreams of datacenter r; ROUTE_PTR: all of them
        self.route_ups = [ups[dc] for dc in self.dc_names]
        self.route_ups += [[]] * (ROUTE_PTR - len(self.route_ups)) + [[a for dc in self.dc_names for a in ups[dc]]]
        table = [(a[0], a[1], k) for k, dc in enumerate(self.dc_names) for a in ups[dc]]
        resolver.set_recursion_filter(dns_domain, self.dc_names, bool(table))
        resolver.set_recursion_upstreams(table)
        self.timeout = timeout
        self.window_s = window_s
        # misses per window: the 16-bit ID space, and no more than one forward / match / relay call of the resolver takes
        self.window_max = min(FORWARD_MAX, getattr(resolver, 'max_batch', FORWARD_MAX))
        self.counters = {'relayed': 0, 'forwarded': 0, 'upstream_answers': 0, 'tcp_skipped': 0, 'failed_batches': 0,
                         'delivered': 0}
        self._udp = UdpSink(resolver, self.counters)
        self._q = queue.Queue()
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._loop, daemon=True)
        self._thread.start()

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
        """One miss of a transport owner: its upstream response comes back through sink.relay(..., tags) with `tag`."""
        self._q.put((bytes(packet), sink, tag))

    def close(self):
        self._stop.set()
        self._thread.join(self.timeout + 2)

    def _loop(self):
        while not self._stop.is_set():
            try:
                batch = [self._q.get(timeout=0.05)]
            except queue.Empty:
                continue
            deadline = time.perf_counter() + self.window_s
            while time.perf_counter() < deadline and len(batch) < self.window_max:
                try:
                    batch.append(self._q.get(timeout=max(deadline - time.perf_counter(), 1e-4)))
                except queue.Empty:
                    break
            try:
                self._relay(batch)
            except Exception:                 # BinderError (capacity, CUDA): this window gets no replies
                self.counters['failed_batches'] += 1

    def _exchange(self, q_data, q_off):
        """forward -> sends -> receive -> match: the upstream response per miss, packed in miss order (up, up_off)."""
        key = int.from_bytes(os.urandom(8), 'little')             # fresh per call, like the socket
        uq, uq_off, _, group_off, route = self.resolver.forward_batch(q_data, q_off, key)
        n_fwd = int(group_off[FORWARD_ROUTES - 1])                  # runs before the "none" run are sent
        got, src_ip, src_port = [], [], []
        s = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        try:
            s.setblocking(False)
            for r in range(FORWARD_ROUTES - 1):
                k0, k1 = int(group_off[r]), int(group_off[r + 1])
                if k0 == k1:
                    continue
                for up in self.route_ups[r]:
                    for k in range(k0, k1):
                        try:
                            s.sendto(uq[uq_off[k]:uq_off[k + 1]].tobytes(), up)
                        except OSError:
                            pass
            self.counters['forwarded'] += n_fwd
            end = time.perf_counter() + self.timeout
            result = None
            while n_fwd and time.perf_counter() < end:
                r, _, _ = select.select([s], [], [], max(end - time.perf_counter(), 0))
                if not r:
                    break
                while True:                                          # drain what has arrived
                    try:
                        data, src = s.recvfrom(65535)
                    except OSError:
                        break
                    got.append(data)
                    src_ip.append(ip_u32(src[0]))
                    src_port.append(src[1])
                if len(got) >= n_fwd:                                # every forwarded miss may have its answer: match
                    result = self._match(got, src_ip, src_port, q_data, q_off, route, key)
                    if int(np.count_nonzero(np.diff(result[1].astype(np.int64)))) == n_fwd:
                        break
                    result = None
        finally:
            s.close()
        if result is None:
            result = self._match(got, src_ip, src_port, q_data, q_off, route, key)
        self.counters['upstream_answers'] += int(np.count_nonzero(np.diff(result[1].astype(np.int64))))
        return result

    def _match(self, got, src_ip, src_port, q_data, q_off, route, key):
        r_data, r_off = pack_packets(got)
        return self.resolver.match_upstreams(r_data, r_off, np.array(src_ip, np.uint32), np.array(src_port, np.uint16),
                                             q_data, q_off, route, key)

    def _relay(self, batch):
        q_data, q_off = pack_packets([p for p, _, _ in batch])
        try:
            up, up_off = self._exchange(q_data, q_off)
        except Exception:                 # BinderError (capacity, CUDA): the UDP misses get no replies; the other owners
            self.counters['failed_batches'] += 1      # get failed lookups (REFUSED), so what they owe is settled
            batch = [m for m in batch if m[1] is not self._udp]
            if not batch:
                return
            q_data, q_off = pack_packets([p for p, _, _ in batch])
            up, up_off = pack_packets([b''] * len(batch))
        deliver(batch, q_data, q_off, up, up_off, self.counters)
