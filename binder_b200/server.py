"""Host-side mirror of binder's server object (lib/server.js createServer / start / stop), in
Python because Node.js is not available in this image.  It keeps binder's shape — options
{host, port, dnsDomain, datacenterName, recursion, zkCache} and a UDP listener — but where mname
emits one 'query' event per packet (lib/server.js:471), packets are collected for a short window
and resolved as ONE batch by `resolver.resolve_batch` (a binder_b200.engine.Engine); the bytes it
returns are sent as they are.  Queries the engine hands back as recursion misses go to
options['recursion'].resolve(packet, addr) (lib/server.js:110-113,222-225) when one is given.

TCP (mname's listenTcp, lib/server.js:643-652): every connection is a stream of messages, each preceded
by its length as two big-endian bytes (RFC 1035 4.2.2; deps/mname-balancer/tcp_proxy.c:10-26 relays the
same framing).  TcpFramer reassembles them; messages from all connections that complete inside one
aggregation window form ONE batch, resolved with tcp=True (no UDP size limit), and each response goes
back on its connection with its own length prefix, in arrival order per connection.  A TCP miss is submitted to the
recursion (recursion.submit) with the TCP loop's queue sink, the connection as its tag, when the recursion has submit()
and the resolver has relay_batch(); the loop relays each window it drains with tcp=True and appends every reply to its
connection, length-prefixed.  Relayed replies may overtake local answers on the same connection (RFC 7766 allows it: the
ID matches them).  A connection owed a relay stays open through the idle sweep and after a half-close until the reply
is written.

Query log (lib/server.js:509-591): with options['query_log'], a writable binary stream, every batch the server answers
gets one resolver.log_batch call (bb_log_batch) and every answered query one bunyan "DNS query" line on the stream
(binder_b200/query_log.py; the request id is the DNS ID).  The same sink goes to the recursion (set_query_log), so that
relayed replies are logged on both transports when they are sent.  Without the option nothing changes.

The resolver is injected, so the CPU-only plumbing test (BASELINE config 1) drives this same code
with the CPU oracle, while production passes an Engine.
"""
import select
import selectors
import socket
import struct
import threading
import time

import numpy as np

MAX_UDP = 1500          # deps/mname-balancer/udp_proxy.c:159-170


class TcpFramer(object):
    """Reassembly of one DNS-over-TCP stream: feed() bytes as they arrive, get back the complete messages.
    A zero-length message is a protocol error (the connection is closed by the caller)."""

    def __init__(self):
        self.buf = bytearray()
        self.bad = False

    def feed(self, chunk):
        self.buf += chunk
        out = []
        while len(self.buf) >= 2:
            n = (self.buf[0] << 8) | self.buf[1]
            if n == 0:
                self.bad = True
                break
            if len(self.buf) < 2 + n:
                break
            out.append(bytes(self.buf[2:2 + n]))
            del self.buf[:2 + n]
        return out

    @staticmethod
    def frame(msg):
        return struct.pack('>H', len(msg)) + msg


def pack_packets(pkts):
    """[bytes] -> (uint8 data padded for 16-byte reads, uint32 offsets[n+1])"""
    lens = np.fromiter((len(p) for p in pkts), dtype=np.int64, count=len(pkts))
    off = np.zeros(len(pkts) + 1, dtype=np.uint32)
    np.cumsum(lens, out=off[1:])
    blob = b''.join(pkts)
    return np.frombuffer(blob + b'\0' * ((-len(blob)) % 16 + 16), dtype=np.uint8), off


class TcpConn(object):
    """One TCP connection: reassembly state, bytes still to send, queries it is owed answers (or relays) for, and
    whether it is registered with the selector (a half-closed connection that only waits for a relay is not)."""
    __slots__ = ('framer', 'outq', 'waiting', 'eof', 'last', 'reg')

    def __init__(self, now):
        self.framer, self.outq, self.waiting, self.eof, self.last, self.reg = TcpFramer(), bytearray(), 0, False, now, True


class Server(object):
    def __init__(self, options):
        for k in ('dnsDomain', 'resolver'):
            if k not in options:
                raise ValueError('options.%s is required' % k)          # assert.string(options.dnsDomain), lib/server.js:439
        self.options = options
        self.resolver = options['resolver']
        self.host = options.get('host', '127.0.0.1')
        self.port = options.get('port', 0)
        self.window_s = options.get('batch_window_us', 200) * 1e-6
        self.max_batch = options.get('max_batch', 4096)
        self.recursion = options.get('recursion')
        self.counters = {'queries': 0, 'answered': 0, 'missed': 0, 'dropped': 0, 'batches': 0,
                         'tcp_queries': 0, 'tcp_batches': 0, 'tcp_connections': 0, 'tcp_refused': 0, 'failed_batches': 0,
                         'tcp_relayed': 0}
        self._lock = threading.Lock()                # one engine, two listener threads
        self.tcp = options.get('tcp', True)
        self._sock = None
        self._tsock = None
        self._tthread = None
        self._thread = None
        self._stop = threading.Event()
        self._seed = options.get('shuffle_seed', int(time.time() * 1e6))
        self.query_log = None
        if options.get('query_log') is not None:
            from .query_log import QueryLog
            self.query_log = QueryLog(options['query_log'])
            if hasattr(self.recursion, 'set_query_log'):
                self.recursion.set_query_log(self.query_log)

    # lib/server.js:609-653: UDP and TCP on the same port (the balancer socket stays host JS)
    def start(self, callback=None):
        fam = socket.AF_INET6 if ':' in self.host else socket.AF_INET
        self._sock = socket.socket(fam, socket.SOCK_DGRAM)
        self._sock.bind((self.host, self.port))
        self.port = self._sock.getsockname()[1]
        self._sock.settimeout(0.05)
        self._thread = threading.Thread(target=self._loop, daemon=True)
        self._thread.start()
        if self.tcp:
            self._tsock = socket.socket(fam, socket.SOCK_STREAM)
            self._tsock.setsockopt(socket.SOL_SOCKET, socket.SO_REUSEADDR, 1)
            self._tsock.bind((self.host, self.port))
            self._tsock.listen(128)
            self._tsock.setblocking(False)
            self._tthread = threading.Thread(target=self._tcp_loop, daemon=True)
            self._tthread.start()
        if callback:
            callback()
        return self

    def stop(self, callback=None):
        self._stop.set()
        if self._thread:
            self._thread.join(2)
        if self._tthread:
            self._tthread.join(2)
        if self._sock:
            self._sock.close()
        if self._tsock:
            self._tsock.close()
        if callback:
            callback()

    def _loop(self):
        while not self._stop.is_set():
            try:
                pkt, addr = self._sock.recvfrom(MAX_UDP + 1)
            except socket.timeout:
                continue
            except OSError:
                break
            batch = [(pkt, addr, time.time())]
            deadline = time.perf_counter() + self.window_s
            self._sock.settimeout(max(self.window_s, 1e-4))
            while len(batch) < self.max_batch and time.perf_counter() < deadline:
                try:
                    batch.append(self._sock.recvfrom(MAX_UDP + 1) + (time.time(),))
                except (socket.timeout, BlockingIOError):
                    break
            self._sock.settimeout(0.05)
            self._resolve_and_send(batch)

    def _resolve(self, data, off, tcp=False):
        """One batch through the resolver.  The UDP and the TCP listener share ONE engine (bb_resolve_batch uses the
        engine's slot 0): calls are serialised here, and a failed batch is dropped and counted, not allowed to kill the
        listener thread.  -> (out, out_off, out_len, status, miss) or None."""
        with self._lock:
            self._seed += 1
            try:
                if tcp:
                    return self.resolver.resolve_batch(data, off, seed=self._seed, qidx_base=0, tcp=True)
                return self.resolver.resolve_batch(data, off, seed=self._seed, qidx_base=0)
            except Exception:                        # BinderError (capacity, CUDA), or a resolver bug: this batch gets no answers
                self.counters['failed_batches'] += 1
                return None

    # ---- TCP: accept, reassemble, aggregate, answer ------------------------------------------------
    # One selector (epoll) for the listening socket and every connection; writes never block: each connection has an
    # output queue drained when the socket is writable.  Connections are capped (max_tcp_conns) and closed when idle.
    def _tcp_loop(self):
        sel = selectors.DefaultSelector()
        sel.register(self._tsock, selectors.EVENT_READ)
        conns = {}                                   # socket -> TcpConn
        pending = []                                 # (message, socket) completed in the current window
        deadline = None
        max_conns = self.options.get('max_tcp_conns', 1024)
        idle_s = self.options.get('tcp_idle_s', 30.0)
        sink = wake_r = wake_w = None
        if hasattr(self.recursion, 'submit') and hasattr(self.resolver, 'relay_batch'):
            from .recursion import QueueSink
            wake_r, wake_w = socket.socketpair()
            wake_r.setblocking(False)
            wake_w.setblocking(False)

            def wake():
                try:
                    wake_w.send(b'\0')
                except OSError:                      # full: a wake-up is pending anyway
                    pass
            sink = QueueSink(wake)
            sel.register(wake_r, selectors.EVENT_READ)

        def close(s):
            c = conns.pop(s, None)
            if c is not None:
                try:
                    sel.unregister(s)
                except (KeyError, ValueError):
                    pass
                s.close()

        def want(s):                                 # (re)register for the events this connection needs
            c = conns[s]
            ev = (0 if c.eof else selectors.EVENT_READ) | (selectors.EVENT_WRITE if c.outq else 0)
            if ev:
                (sel.modify if c.reg else sel.register)(s, ev)
                c.reg = True
            elif not c.waiting:                      # peer closed its side, nothing owed, nothing left to send
                close(s)
            elif c.reg:                              # half-closed and owed a relay: nothing to select on until it comes
                sel.unregister(s)
                c.reg = False

        last_sweep = time.perf_counter()
        while not self._stop.is_set():
            timeout = 0.05 if deadline is None else max(deadline - time.perf_counter(), 0.0)
            try:
                events = sel.select(timeout)
            except OSError:
                break
            now = time.perf_counter()
            for key, ev in events:
                s = key.fileobj
                if s is wake_r:
                    try:
                        while wake_r.recv(4096):
                            pass
                    except OSError:
                        pass
                    for item in sink.drain():
                        for t in self._relay_tcp(item, conns):
                            want(t)
                    continue
                if s is self._tsock:
                    try:
                        c, _ = self._tsock.accept()
                    except OSError:
                        continue
                    if len(conns) >= max_conns:
                        c.close()
                        self.counters['tcp_refused'] += 1
                        continue
                    c.setblocking(False)
                    conns[c] = TcpConn(now)
                    sel.register(c, selectors.EVENT_READ)
                    self.counters['tcp_connections'] += 1
                    continue
                c = conns.get(s)
                if c is None:
                    continue
                if ev & selectors.EVENT_WRITE and c.outq:
                    try:
                        n = s.send(c.outq)
                        del c.outq[:n]
                        c.last = now
                    except (BlockingIOError, InterruptedError):
                        pass
                    except OSError:
                        close(s)
                        continue
                if ev & selectors.EVENT_READ and not c.eof:
                    try:
                        chunk = s.recv(65536)
                    except (BlockingIOError, InterruptedError):
                        chunk = None
                    except OSError:
                        chunk = b''
                    if chunk:
                        c.last = now
                        msgs = c.framer.feed(chunk)
                        t_recv = time.time()
                        for m in msgs:
                            pending.append((m, s, t_recv))
                        c.waiting += len(msgs)
                        if msgs and deadline is None:
                            deadline = now + self.window_s
                    if chunk == b'' or c.framer.bad:  # peer closed (its complete messages are still answered) / bad frame
                        c.eof = True
                if s in conns:
                    want(s)
            if pending and (len(pending) >= self.max_batch or time.perf_counter() >= deadline):
                self._resolve_and_send_tcp(pending, conns, sink)
                for s in set(ps for _, ps, _ in pending):
                    if s in conns:
                        want(s)
                pending, deadline = [], None
            if now - last_sweep > 1.0:                # idle connections
                last_sweep = now
                for s in [s for s, c in conns.items() if now - c.last > idle_s and not c.waiting and not c.outq]:
                    close(s)
        for s in list(conns):
            close(s)
        sel.close()
        if wake_r is not None:
            wake_r.close()
            wake_w.close()

    def _relay_tcp(self, item, conns):
        """One window of relays drained from the TCP loop's sink: replies (tcp=True) appended to their connections, which
        are owed one relay less each.  -> the connections still open"""
        q_data, q_off, up, up_off, tags = item
        with self._lock:
            try:
                res = self.resolver.relay_batch(q_data, q_off, up, up_off, tcp=True)
            except Exception:                        # BinderError (capacity, CUDA): these misses get no replies
                self.counters['failed_batches'] += 1
                res = None
        live = set()
        for i, (s, _) in enumerate(tags):
            c = conns.get(s)
            if c is None:                            # closed meanwhile
                continue
            c.waiting -= 1
            live.add(s)
            if res is not None and res[3][i] == 0:
                out, out_off, out_len, _ = res
                c.outq += TcpFramer.frame(out[out_off[i]:out_off[i] + out_len[i]].tobytes())
                self.counters['tcp_relayed'] += 1
        if res is not None and self.query_log is not None:
            self._log(res[:4], [self._peer(s) for s, _ in tags], [t for _, t in tags])
        return live

    @staticmethod
    def _peer(s):
        try:
            return s.getpeername()[:2]
        except OSError:                              # closed meanwhile: its line still names the query
            return ('', 0)

    def _log(self, res, clients, received):
        """The query log lines of one batch of sent responses (resolver calls are serialised, as in _resolve)."""
        with self._lock:
            self.query_log.write(self.resolver, *res, clients, received)

    def _resolve_and_send_tcp(self, pending, conns, sink=None):
        pkts = [m for m, _, _ in pending]
        data, off = pack_packets(pkts)
        res = self._resolve(data, off, tcp=True)
        c = self.counters
        c['tcp_batches'] += 1
        c['tcp_queries'] += len(pkts)
        for _, s, _ in pending:
            if s in conns:
                conns[s].waiting -= 1
        if res is None:
            return
        out, out_off, out_len, status, miss = res
        for i, (_, s, _) in enumerate(pending):      # per connection, in arrival order
            if status[i] == 0:
                if s in conns:
                    conns[s].outq += TcpFramer.frame(out[out_off[i]:out_off[i] + out_len[i]].tobytes())
                c['answered'] += 1
            elif status[i] == 2:
                c['dropped'] += 1
        if self.query_log is not None:
            self._log((out, out_off, out_len, status), [self._peer(s) for _, s, _ in pending], [t for _, _, t in pending])
        for i in miss:
            c['missed'] += 1
            _, s, t_recv = pending[int(i)]
            if sink is not None:
                if s in conns:
                    conns[s].waiting += 1
                    self.recursion.submit(pkts[int(i)], sink, (s, t_recv))
            elif self.recursion is not None:
                self.recursion.resolve(pkts[int(i)], None, s)

    def _resolve_and_send(self, batch):
        pkts = [p for p, _, _ in batch if len(p) <= MAX_UDP]
        addrs = [a for p, a, _ in batch if len(p) <= MAX_UDP]
        received = [t for p, _, t in batch if len(p) <= MAX_UDP]
        data, off = pack_packets(pkts)
        res = self._resolve(data, off)
        c = self.counters
        c['batches'] += 1
        c['queries'] += len(pkts)
        if res is None:
            return
        out, out_off, out_len, status, miss = res
        for i, a in enumerate(addrs):
            if status[i] == 0:
                self._sock.sendto(out[out_off[i]:out_off[i] + out_len[i]].tobytes(), a)
                c['answered'] += 1
            elif status[i] == 2:
                c['dropped'] += 1
        if self.query_log is not None:
            self._log((out, out_off, out_len, status), addrs, received)
        for i in miss:
            c['missed'] += 1
            if self.recursion is not None:
                if self.query_log is not None and hasattr(self.recursion, 'set_query_log'):
                    self.recursion.resolve(pkts[int(i)], addrs[int(i)], self._sock, received=received[int(i)])
                else:
                    self.recursion.resolve(pkts[int(i)], addrs[int(i)], self._sock)


def createServer(options):
    """core.createServer(options) (lib/server.js:435)."""
    return Server(options)
