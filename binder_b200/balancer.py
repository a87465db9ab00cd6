"""mname-balancer backend protocol adapter (SURVEY.md section 8f row 1; wire format:
deps/mname-balancer/backend.c:22-113, frame types deps/mname-balancer/bbal.h:80-87).

The balancer forwards every UDP packet to a backend over an AF_UNIX stream as an INBOUND_UDP frame
(all integers u32 little-endian):

    0   u32 frame type = 2      4   u32 source IPv4      8   u32 source port
    12  u32 packet length       16  packet bytes

and expects OUTBOUND_UDP frames (type 1002, same layout, destination instead of source) back.
Frames are already "batched raw packets + source address", i.e. exactly the engine's batch
container plus 12 bytes of addressing per packet.  This module turns a buffer of frames into a
batch for bb_resolve_batch and the results back into OUTBOUND_UDP frames; HELLO / HEARTBEAT frames
are answered in place.  numpy only: no per-packet Python on the hot path.

DNS-over-TCP clients reach a backend differently: the balancer hands each client connection over as its own AF_UNIX
session that opens with INBOUND_TCP {3, source IPv4, source port} (12 bytes), is answered INBOUND_TCP_OK (1003) and
then carries the client's raw 2-byte length-prefixed DNS stream both ways (backend.c:60-75, tcp_proxy.c:160-300).
TcpHub / NativeTcpHub hold many such sessions and resolve the messages that complete on all of them as one TCP batch.
A host routes a new AF_UNIX connection by its first frame: CLIENT_HELLO to a Backend, INBOUND_TCP to the hub.

Misses (lib/server.js:110-113,222-225) go to the recursion with the owner's sink (recursion.submit): a Backend submits
its own with the source address as the tag and relays what its sink drains into OUTBOUND_UDP frames (relay(), UDP size
limits); a hub's host submits flush()'s misses with the session id as the tag and hands what it drains to hub.relay().
"""
import ctypes
import struct

import numpy as np

from .query_log import QueryLogRecords
from .recursion import QueueSink, split_packets
from .server import TcpFramer, pack_packets

CLIENT_HELLO, INBOUND_UDP, INBOUND_TCP, CLIENT_HEARTBEAT = 1, 2, 3, 4
SERVER_HELLO, OUTBOUND_UDP, INBOUND_TCP_OK, SERVER_HEARTBEAT = 1001, 1002, 1003, 1004
MAX_UDP = 1500                      # deps/mname-balancer/udp_proxy.c:159-170, backend.c:709-716


class ProtocolError(ValueError):
    pass


def parse_frames(buf):
    """bytes-like stream of balancer->backend frames ->
    (data u8 padded, off u32[n+1], src_ip u32[n], src_port u32[n], control [frame types], consumed)
    Only whole frames are consumed; `consumed` tells the caller how much of buf to drop."""
    b = np.frombuffer(buf, dtype=np.uint8)
    pos, n = 0, len(b)
    starts, lens, ips, ports, control = [], [], [], [], []
    while pos + 4 <= n:
        ftype = int(b[pos:pos + 4].view('<u4')[0])
        if ftype in (CLIENT_HELLO, CLIENT_HEARTBEAT):
            control.append(ftype); pos += 4
        elif ftype == INBOUND_UDP:
            if pos + 16 > n:
                break
            ip, port, ln = (int(x) for x in b[pos + 4:pos + 16].view('<u4'))
            if ln > MAX_UDP:
                raise ProtocolError('INBOUND_UDP frame of %d bytes' % ln)
            if pos + 16 + ln > n:
                break
            starts.append(pos + 16); lens.append(ln); ips.append(ip); ports.append(port)
            pos += 16 + ln
        elif ftype == INBOUND_TCP:
            raise ProtocolError('INBOUND_TCP converts the session to a TCP proxy: not handled by the batch path')
        else:
            raise ProtocolError('unknown frame type %d' % ftype)
    lens_a = np.asarray(lens, dtype=np.int64)
    off = np.zeros(len(lens) + 1, dtype=np.uint32)
    np.cumsum(lens_a, out=off[1:])
    total = int(off[-1])
    data = np.zeros((total + 15) // 16 * 16 + 16, dtype=np.uint8)
    if len(lens):
        # gather the packet bytes of all frames in one indexed copy
        idx = np.repeat(np.asarray(starts, dtype=np.int64) - off[:-1].astype(np.int64), lens_a) + np.arange(total)
        data[:total] = b[idx]
    return data, off, np.asarray(ips, dtype=np.uint32), np.asarray(ports, dtype=np.uint32), control, pos


def build_frames(out, out_off, out_len, status, dst_ip, dst_port, control=()):
    """Engine results -> bytes of backend->balancer frames: SERVER_HELLO / SERVER_HEARTBEAT for each
    control frame received, then one OUTBOUND_UDP frame per answered query (status 0)."""
    ctrl = np.asarray([SERVER_HELLO if c == CLIENT_HELLO else SERVER_HEARTBEAT for c in control], dtype='<u4').tobytes()
    ans = np.nonzero(np.asarray(status) == 0)[0]
    if ans.size == 0:
        return ctrl
    ln = np.asarray(out_len)[ans].astype(np.int64)
    fstart = np.zeros(ans.size + 1, dtype=np.int64)
    np.cumsum(ln + 16, out=fstart[1:])
    buf = np.zeros(int(fstart[-1]), dtype=np.uint8)
    hdr = np.stack([np.full(ans.size, OUTBOUND_UDP, dtype='<u4'), np.asarray(dst_ip)[ans].astype('<u4'),
                    np.asarray(dst_port)[ans].astype('<u4'), ln.astype('<u4')], axis=1).view(np.uint8).reshape(ans.size, 16)
    hidx = (fstart[:-1, None] + np.arange(16)[None, :]).reshape(-1)
    buf[hidx] = hdr.reshape(-1)
    total = int(ln.sum())
    src = np.repeat(np.asarray(out_off)[:-1][ans].astype(np.int64) - (np.cumsum(ln) - ln), ln) + np.arange(total)
    dst = np.repeat(fstart[:-1] + 16 - (np.cumsum(ln) - ln), ln) + np.arange(total)
    buf[dst] = np.asarray(out)[src]
    return ctrl + buf.tobytes()


class _LogSet(object):
    """The query-log records of a Python session's last call of one kind, as the native sessions keep them (bb_log_set,
    csrc/balancer_backend.h): one resolver.log_batch per batch with an answer, a record per answer sent, in send order."""

    def __init__(self):
        self.on, self.records, self.lost = False, 0, 0
        self.clear()

    def clear(self):
        self.logs, self.rows, self.used, self.call_lost = [], [], 0, 0

    def batch(self, resolver, out, out_off, out_len, status, sent):
        """sent: [(i, ip, port, session)] of the answered responses sent, in send order."""
        if not self.on or not (np.asarray(status) == 0).any():
            return
        try:
            log, log_off, log_len, head_len = resolver.log_batch(out, out_off, out_len, status)
        except Exception:                            # BinderError: the answers are sent anyway, their records are lost
            self.call_lost += len(sent)
            self.lost += len(sent)
            return
        out = np.asarray(out)
        for i, ip, port, sid in sent:
            r = int(out_off[i])
            req_id = (int(out[r]) << 8) | int(out[r + 1]) if int(out_len[i]) >= 2 else 0
            self.rows.append((self.used + int(log_off[i]), int(log_len[i]), int(head_len[i]), req_id, ip, port, sid))
        self.logs.append(np.asarray(log, dtype=np.uint8))
        self.used += len(log)
        self.records += len(sent)

    def result(self, with_session):
        rows = self.rows
        col = lambda k, dt: np.array([r[k] for r in rows], dtype=dt)
        log = np.concatenate(self.logs) if self.logs else np.zeros(0, np.uint8)
        return QueryLogRecords(log, col(0, np.uint32), col(1, np.uint32), col(2, np.uint16), col(3, np.uint16), col(4, np.uint32),
                               col(5, np.uint32), col(6, np.uint32) if with_session else None, self.call_lost)


class _QueryLogging(object):
    """set_query_log / query_log of the Python sessions: _log = (last feed or flush, last relay)."""
    _with_session = False

    def set_query_log(self, on):
        for ls in self._log:
            ls.on = bool(on)
            ls.clear()

    def query_log(self, which):
        return self._log[which].result(self._with_session)

    def _count_log(self):
        self.counters['records'] = sum(ls.records for ls in self._log)
        self.counters['lost'] = sum(ls.lost for ls in self._log)


def _native_records(L, fn, h, which, with_session):
    """bb_query_log_backend / bb_query_log_tcp_hub -> QueryLogRecords of numpy copies"""
    from ._lib import check
    P = ctypes.POINTER

    class Records(ctypes.Structure):
        _fields_ = [('n', ctypes.c_uint32), ('log', P(ctypes.c_uint8)), ('log_off', P(ctypes.c_uint32)), ('log_len', P(ctypes.c_uint32)),
                    ('head_len', P(ctypes.c_uint16)), ('req_id', P(ctypes.c_uint16)), ('client_ip', P(ctypes.c_uint32)),
                    ('client_port', P(ctypes.c_uint32)), ('session', P(ctypes.c_uint32)), ('lost', ctypes.c_uint32)]
    if not h:
        check(-1)
    r = Records()
    check(getattr(L, fn)(h, which, ctypes.byref(r)))
    n = r.n
    arr = lambda p, dt: np.ctypeslib.as_array(p, (n,)).astype(dt) if n else np.zeros(0, dt)
    off, ln = arr(r.log_off, np.uint32), arr(r.log_len, np.uint32)
    end = int((off.astype(np.int64) + ln).max()) if n else 0
    log = np.ctypeslib.as_array(r.log, (end,)).copy() if end else np.zeros(0, np.uint8)
    return QueryLogRecords(log, off, ln, arr(r.head_len, np.uint16), arr(r.req_id, np.uint16), arr(r.client_ip, np.uint32),
                           arr(r.client_port, np.uint32), arr(r.session, np.uint32) if with_session else None, int(r.lost))


class Backend(_QueryLogging):
    """One balancer session: feed() bytes read from the AF_UNIX socket, get bytes to write back.

    With a recursion, feed() submits every miss with this session's sink (a QueueSink that calls `wake`, from the
    recursion thread, when a window arrives) and the source (ip, port) as the tag; drain() then returns the OUTBOUND_UDP
    frames of the relays that arrived.  relay(queries, upstreams, dst) builds them on `relayer` (anything with
    relay_batch; the resolver by default) in batches of max_batch, as NativeBackend.relay (bb_backend_relay) does: a
    failed batch gets no frames and is counted.  set_query_log(True): each batch's answers also get their "DNS query"
    log records (the resolver's or relayer's log_batch), read with query_log(0: last feed, 1: last relay)."""

    def __init__(self, resolver, recursion=None, shuffle_seed=1, relayer=None, max_batch=1 << 14, wake=None):
        self.resolver, self.recursion, self.seed = resolver, recursion, shuffle_seed
        self.relayer = relayer if relayer is not None else resolver
        self.max_batch = max_batch
        self.sink = QueueSink(wake)
        self.pending = b''
        self.counters = {'udp': 0, 'answered': 0, 'missed': 0, 'dropped': 0, 'relayed': 0, 'relay_failed': 0, 'records': 0, 'lost': 0}
        self._log = (_LogSet(), _LogSet())

    def feed(self, chunk):
        self._log[0].clear()
        self.pending += bytes(chunk)
        data, off, ips, ports, control, used = parse_frames(self.pending)
        self.pending = self.pending[used:]
        n = len(off) - 1
        if n == 0:
            return build_frames([], [0], [], [], [], [], control)
        self.seed += 1
        out, out_off, out_len, status, miss = self.resolver.resolve_batch(data, off, seed=self.seed, qidx_base=0)
        c = self.counters
        c['udp'] += n; c['answered'] += int((status == 0).sum()); c['missed'] += len(miss); c['dropped'] += int((status == 2).sum())
        self._log[0].batch(self.resolver, out, out_off, out_len, status,
                           [(i, int(ips[i]), int(ports[i]), 0) for i in np.flatnonzero(status == 0)])
        self._count_log()
        if self.recursion is not None:
            for i in miss:
                i = int(i)
                self.recursion.submit(bytes(data[off[i]:off[i + 1]]), self.sink, (int(ips[i]), int(ports[i])))
        return build_frames(out, out_off, out_len, status, ips, ports, control)

    def relay(self, queries, upstreams, dst):
        """Replies to misses (query i answered from upstream response i, b'' = the lookup failed) -> bytes of one
        OUTBOUND_UDP frame per answered reply, addressed to dst[i] = (ip, port)."""
        c, frames = self.counters, []
        self._log[1].clear()
        for k0 in range(0, len(queries), self.max_batch):
            qs, us, ds = queries[k0:k0 + self.max_batch], upstreams[k0:k0 + self.max_batch], dst[k0:k0 + self.max_batch]
            try:
                out, out_off, out_len, status = self.relayer.relay_batch(*(pack_packets(qs) + pack_packets(us)))
            except Exception:                        # BinderError (capacity, CUDA): this batch gets no frames
                c['relay_failed'] += len(qs)
                continue
            c['relayed'] += int((np.asarray(status) == 0).sum())
            self._log[1].batch(self.relayer, out, out_off, out_len, status,
                               [(j, ds[j][0], ds[j][1], 0) for j in np.flatnonzero(np.asarray(status) == 0)])
            self._count_log()
            frames.append(build_frames(out, out_off, out_len, status, [ip for ip, _ in ds], [p for _, p in ds]))
        return b''.join(frames)

    def drain(self):
        """Bytes of the OUTBOUND_UDP frames for the relays the recursion delivered since the last call."""
        return b''.join(self.relay(split_packets(q, qo), split_packets(u, uo), tags) for q, qo, u, uo, tags in self.sink.drain())


# ---- the same protocol, natively (csrc/balancer_frames.cpp) ---------------------------------------------
def parse_frames_native(buf, cap_n=1 << 16, cap_bytes=1 << 22, cap_ctrl=64):
    """bb_frames_parse -> (data u8, off u32[n+1], src_ip, src_port, control list, consumed, rc)"""
    import ctypes
    from ._lib import lib
    buf = bytes(buf)
    data = np.zeros(cap_bytes + 32, dtype=np.uint8); off = np.zeros(cap_n + 1, dtype=np.uint32)
    ips = np.zeros(max(cap_n, 1), dtype=np.uint32); ports = np.zeros(max(cap_n, 1), dtype=np.uint32)
    ctrl = np.zeros(max(cap_ctrl, 1), dtype=np.uint32)
    n, nc, used = ctypes.c_uint32(0), ctypes.c_uint32(0), ctypes.c_size_t(0)
    rc = lib().bb_frames_parse(buf, len(buf), data.ctypes.data, cap_bytes, off.ctypes.data, ips.ctypes.data, ports.ctypes.data,
                               cap_n, ctypes.byref(n), ctrl.ctypes.data, cap_ctrl, ctypes.byref(nc), ctypes.byref(used))
    n = n.value
    return data[:(int(off[n]) + 15) // 16 * 16 + 16], off[:n + 1], ips[:n], ports[:n], [int(x) for x in ctrl[:nc.value]], used.value, rc


def build_frames_native(out, out_off, out_len, status, dst_ip, dst_port, control=()):
    """bb_frames_build -> bytes"""
    import ctypes
    from ._lib import check, lib
    n = len(status)
    a = lambda x, dt: np.ascontiguousarray(x, dtype=dt)
    out, out_off, out_len, status = a(out, np.uint8), a(out_off, np.uint32), a(out_len, np.uint16), a(status, np.uint8)
    dst_ip, dst_port, control = a(dst_ip, np.uint32), a(dst_port, np.uint32), a(list(control), np.uint32)
    need = ctypes.c_size_t(0)
    p = lambda x: x.ctypes.data if x.size else None
    args = (p(out), p(out_off), p(out_len), p(status), p(dst_ip), p(dst_port), n, p(control), len(control))
    rc = lib().bb_frames_build(*args, None, 0, ctypes.byref(need))
    if need.value == 0:
        return b''
    buf = np.zeros(need.value, dtype=np.uint8)
    check(lib().bb_frames_build(*args, buf.ctypes.data, buf.size, ctypes.byref(need)))
    return buf.tobytes()


class NativeBackend(object):
    """bb_backend: one balancer session in the C library (frames in -> bb_resolve_batch -> frames out).
    set_query_log(True) turns on the "DNS query" log records of its answers; query_log(0: last feed, 1: last relay)
    returns them as a QueryLogRecords of numpy copies."""

    def __init__(self, engine, max_batch=1 << 14, lib=None):
        import ctypes
        from ._lib import BinderError, lib as _lib
        self._L = lib if lib is not None else _lib()
        err = ctypes.c_int(0)
        self._h = self._L.bb_backend_create(engine._h, max_batch, ctypes.byref(err))
        if not self._h:
            raise BinderError(err.value)
        self._engine, self.last_rc = engine, 0

    def feed(self, chunk, seed):
        """-> (bytes to write back, [(packet, src_ip, src_port)] handed to recursion)"""
        import ctypes
        from ._lib import check

        class Misses(ctypes.Structure):
            _fields_ = [('n', ctypes.c_uint32), ('pkts', ctypes.POINTER(ctypes.c_uint8)), ('pkt_off', ctypes.POINTER(ctypes.c_uint32)),
                        ('src_ip', ctypes.POINTER(ctypes.c_uint32)), ('src_port', ctypes.POINTER(ctypes.c_uint32))]
        chunk = bytes(chunk)
        out, out_len, m = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_size_t(0), Misses()
        check(self._L.bb_backend_feed(self._h, chunk, len(chunk), seed, ctypes.byref(out), ctypes.byref(out_len), ctypes.byref(m)))
        data = ctypes.string_at(out, out_len.value) if out_len.value else b''
        misses = [(ctypes.string_at(ctypes.addressof(m.pkts.contents) + m.pkt_off[i], m.pkt_off[i + 1] - m.pkt_off[i]),
                   int(m.src_ip[i]), int(m.src_port[i])) for i in range(m.n)]
        return data, misses

    def relay(self, queries, upstreams, dst):
        """bb_backend_relay: the same frames as Backend.relay.  A failed batch is counted (stats()['relay_failed']), not
        raised: its code is in last_rc."""
        import ctypes
        from ._lib import check
        if not self._h:
            check(-1)
        (qd, qo), (ud, uo) = pack_packets(queries), pack_packets(upstreams)
        ip = np.ascontiguousarray([a for a, _ in dst], dtype=np.uint32)
        port = np.ascontiguousarray([p for _, p in dst], dtype=np.uint32)
        out, out_len = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_size_t(0)
        rc = self._L.bb_backend_relay(self._h, qd.ctypes.data, qo.ctypes.data, ud.ctypes.data, uo.ctypes.data,
                                      ip.ctypes.data if ip.size else None, port.ctypes.data if port.size else None, len(ip),
                                      ctypes.byref(out), ctypes.byref(out_len))
        if rc == -1:
            check(rc)
        self.last_rc = rc
        return ctypes.string_at(out, out_len.value) if out_len.value else b''

    def set_query_log(self, on):
        from ._lib import check
        check(self._L.bb_query_log_backend_enable(self._h, 1 if on else 0) if self._h else -1)

    def query_log(self, which):
        return _native_records(self._L, 'bb_query_log_backend', self._h, which, False)

    def stats(self):
        keys = ('udp', 'answered', 'missed', 'dropped', 'pending_bytes', 'failed', 'relayed', 'relay_failed', 'records', 'lost')
        return {k: int(self._L.bb_backend_stat(self._h, i)) for i, k in enumerate(keys)}

    def close(self):
        if getattr(self, '_h', None):
            self._L.bb_backend_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- TCP proxy sessions: many sessions, one batch per flush ---------------------------------------------
HUB_STATS = ('sessions', 'messages', 'answered', 'missed', 'dropped', 'protocol_errors', 'failed', 'relayed', 'open', 'queued')


class _TcpSession(object):
    __slots__ = ('pre', 'framer', 'shook', 'eof', 'bad', 'queued', 'relays', 'out', 'ip', 'port')

    def __init__(self):
        self.pre, self.framer, self.out = b'', TcpFramer(), bytearray()
        self.shook = self.eof = self.bad = False
        self.queued = self.relays = self.ip = self.port = 0


class TcpHub(_QueryLogging):
    """The TCP hub (bb_tcp_hub, include/binder_b200.h) in Python, around an injected resolver (Engine or the CPU oracle)
    and relayer (anything with relay_batch(q_data, q_off, up_data, up_off, tcp=True); the resolver by default).

    open() -> session id; feed(id, bytes) -> False on a protocol error; eof(id); flush(seed) -> [(miss packet, id)];
    output(id) -> (bytes to write, closable); consume(id, n); close(id); relay(queries, upstreams, ids).  Limits as the
    native hub's: max_batch queries and max_batch_bytes query bytes per batch, out_cap answer bytes per batch (None: the
    resolver's own limit).  A batch the resolver fails, or whose answers exceed out_cap, loses its queries (counted).
    set_query_log(True) / query_log(0: last flush, 1: last relay): the answers' "DNS query" log records, as the native
    hub keeps them (the resolver's and relayer's log_batch)."""
    _with_session = True

    def __init__(self, resolver, max_batch=4096, max_batch_bytes=None, out_cap=None, relayer=None):
        self.resolver, self.relayer = resolver, relayer if relayer is not None else resolver
        self.max_batch = max_batch
        self.max_bytes = max_batch_bytes if max_batch_bytes is not None else max(64 * max_batch, 1 << 16)
        self.out_cap = out_cap
        self.sessions, self.next_id, self.queue = {}, 1, []
        self.counters = dict.fromkeys(HUB_STATS[:8] + ('records', 'lost'), 0)
        self._log = (_LogSet(), _LogSet())

    def _get(self, sid):
        s = self.sessions.get(sid)
        if s is None:
            raise KeyError('no open session %r' % (sid,))
        return s

    def open(self):
        sid, self.next_id = self.next_id, self.next_id + 1
        self.sessions[sid] = _TcpSession()
        self.counters['sessions'] += 1
        return sid

    def feed(self, sid, chunk):
        s, c = self._get(sid), self.counters
        if s.eof:
            raise KeyError('session %r is past eof' % (sid,))
        if s.bad:
            return False
        chunk = bytes(chunk)
        if not s.shook:
            s.pre += chunk
            if len(s.pre) < 4:
                return True
            if struct.unpack_from('<I', s.pre)[0] != INBOUND_TCP:     # CLIENT_HELLO, INBOUND_UDP, ...: not a TCP session
                s.bad, s.pre = True, b''
                c['protocol_errors'] += 1
                return False
            if len(s.pre) < 12:
                return True
            _, s.ip, s.port = struct.unpack_from('<III', s.pre)
            s.shook, s.out = True, s.out + struct.pack('<I', INBOUND_TCP_OK)
            chunk, s.pre = s.pre[12:], b''
        msgs = s.framer.feed(chunk)
        self.queue += [(m, sid) for m in msgs]
        s.queued += len(msgs)
        c['messages'] += len(msgs)
        if s.framer.bad:                             # zero-length message: what completed before it is still answered
            s.bad = True
            s.framer.buf.clear()
            c['protocol_errors'] += 1
            return False
        return True

    def eof(self, sid):
        s = self._get(sid)
        s.eof, s.pre = True, b''
        s.framer.buf.clear()

    def _answers(self, fn, *args):
        """resolve/relay one batch -> results, or None when it failed"""
        try:
            res = fn(*args, tcp=True)
        except Exception:                            # BinderError (capacity, CUDA), as Server._resolve
            return None
        if self.out_cap is not None and int(np.asarray(res[2], dtype=np.int64).sum()) > self.out_cap:
            return None
        return res

    def flush(self, seed):
        queue, self.queue, c = self.queue, [], self.counters
        self._log[0].clear()
        misses, qidx, i = [], 0, 0
        while i < len(queue):
            batch, nbytes = [], 0
            while i < len(queue) and len(batch) < self.max_batch:
                m, sid = queue[i]
                s = self.sessions.get(sid)
                if s is None or len(m) > self.max_bytes:
                    c['dropped'] += 1
                    if s is not None:
                        s.queued -= 1
                    i += 1
                    continue
                if nbytes + len(m) > self.max_bytes:
                    break
                batch.append((m, sid))
                nbytes += len(m)
                i += 1
            if not batch:
                continue
            data, off = pack_packets([m for m, _ in batch])
            res = self._answers(lambda d, o, tcp: self.resolver.resolve_batch(d, o, seed=seed, qidx_base=qidx, tcp=tcp), data, off)
            qidx += len(batch)
            for _, sid in batch:
                self.sessions[sid].queued -= 1
            if res is None:
                c['failed'] += len(batch)
                continue
            out, out_off, out_len, status, _ = res
            self._log[0].batch(self.resolver, out, out_off, out_len, status,
                               [(k, self.sessions[sid].ip, self.sessions[sid].port, sid) for k, (_, sid) in enumerate(batch) if status[k] == 0])
            self._count_log()
            for k, (m, sid) in enumerate(batch):
                s = self.sessions[sid]
                if status[k] == 0:
                    c['answered'] += 1
                    s.out += TcpFramer.frame(out[out_off[k]:out_off[k] + out_len[k]].tobytes())
                elif status[k] == 1:
                    c['missed'] += 1
                    s.relays += 1
                    misses.append((m, sid))
                else:
                    c['dropped'] += 1
        return misses

    def relay(self, queries, upstreams, sids):
        """Replies to misses: query i answered from upstream response i (b'' = the lookup failed), appended to sids[i]."""
        c = self.counters
        self._log[1].clear()
        for k0 in range(0, len(sids), self.max_batch):
            qs, us, ss = queries[k0:k0 + self.max_batch], upstreams[k0:k0 + self.max_batch], sids[k0:k0 + self.max_batch]
            res = self._answers(self.relayer.relay_batch, *(pack_packets(qs) + pack_packets(us)))
            if res is not None:
                live = [(j, self.sessions.get(sid), sid) for j, sid in enumerate(ss) if res[3][j] == 0]
                self._log[1].batch(self.relayer, *res, [(j, s.ip, s.port, sid) for j, s, sid in live if s is not None])
                self._count_log()
            for j, sid in enumerate(ss):
                s = self.sessions.get(sid)
                if s is not None and s.relays:
                    s.relays -= 1
                if res is None:
                    c['failed'] += 1
                elif s is None or res[3][j] != 0:
                    c['dropped'] += 1
                else:
                    out, out_off, out_len, _ = res
                    s.out += TcpFramer.frame(out[out_off[j]:out_off[j] + out_len[j]].tobytes())
                    c['relayed'] += 1

    def output(self, sid):
        s = self._get(sid)
        return bytes(s.out), (s.eof or s.bad) and not s.queued and not s.relays and not s.out

    def consume(self, sid, n):
        s = self._get(sid)
        if n > len(s.out):
            raise ValueError('consume(%d) past the %d bytes of output' % (n, len(s.out)))
        del s.out[:n]

    def close(self, sid):
        self._get(sid)
        del self.sessions[sid]

    def peer(self, sid):
        s = self._get(sid)
        return s.ip, s.port

    def stats(self):
        return dict(self.counters, open=len(self.sessions), queued=len(self.queue))


class NativeTcpHub(object):
    """bb_tcp_hub: TCP proxy sessions in the C library, their messages resolved as TCP batches on the engine.  Same
    methods as TcpHub; argument errors (unknown or closed session, a closed hub) raise BinderError.  A failed batch is
    counted, not raised: its code is in last_rc.  `lib` is the library to call (libbinder_b200.so by default).
    query_log(which) returns the records as a QueryLogRecords of numpy copies."""

    def __init__(self, engine, max_batch=4096, lib=None):
        import ctypes
        from ._lib import BinderError, lib as _lib
        self._L = lib if lib is not None else _lib()
        err = ctypes.c_int(0)
        self._h = self._L.bb_tcp_hub_create(engine._h, max_batch, ctypes.byref(err))
        if not self._h:
            raise BinderError(err.value)
        self._engine, self.last_rc = engine, 0

    def open(self):
        import ctypes
        from ._lib import check
        sid = ctypes.c_uint32(0)
        check(self._L.bb_tcp_hub_open(self._h, ctypes.byref(sid)))
        return sid.value

    def feed(self, sid, chunk):
        from ._lib import check
        chunk = bytes(chunk)
        rc = self._L.bb_tcp_hub_feed(self._h, sid, chunk, len(chunk))
        if rc == -8:
            return False
        check(rc)
        return True

    def eof(self, sid):
        from ._lib import check
        check(self._L.bb_tcp_hub_eof(self._h, sid))

    def flush(self, seed):
        import ctypes
        from ._lib import check

        class Misses(ctypes.Structure):
            _fields_ = [('n', ctypes.c_uint32), ('pkts', ctypes.POINTER(ctypes.c_uint8)), ('pkt_off', ctypes.POINTER(ctypes.c_uint32)),
                        ('session', ctypes.POINTER(ctypes.c_uint32))]
        if not self._h:
            check(-1)
        m = Misses()
        self.last_rc = self._L.bb_tcp_hub_flush(self._h, seed, ctypes.byref(m))
        if m.n == 0:
            return []
        base = ctypes.addressof(m.pkts.contents)
        return [(ctypes.string_at(base + m.pkt_off[i], m.pkt_off[i + 1] - m.pkt_off[i]), int(m.session[i])) for i in range(m.n)]

    def relay(self, queries, upstreams, sids):
        if not self._h:
            from ._lib import check
            check(-1)
        (qd, qo), (ud, uo) = pack_packets(queries), pack_packets(upstreams)
        s = np.ascontiguousarray(sids, dtype=np.uint32)
        self.last_rc = self._L.bb_tcp_hub_relay(self._h, qd.ctypes.data, qo.ctypes.data, ud.ctypes.data, uo.ctypes.data,
                                                s.ctypes.data if s.size else None, len(s))

    def output(self, sid):
        import ctypes
        from ._lib import check
        p, n, cl = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_size_t(0), ctypes.c_int(0)
        check(self._L.bb_tcp_hub_output(self._h, sid, ctypes.byref(p), ctypes.byref(n), ctypes.byref(cl)))
        return (ctypes.string_at(p, n.value) if n.value else b''), bool(cl.value)

    def consume(self, sid, n):
        from ._lib import check
        check(self._L.bb_tcp_hub_consume(self._h, sid, n))

    def close(self, sid):
        from ._lib import check
        check(self._L.bb_tcp_hub_close(self._h, sid))

    def peer(self, sid):
        import ctypes
        from ._lib import check
        ip, port = ctypes.c_uint32(0), ctypes.c_uint32(0)
        check(self._L.bb_tcp_hub_peer(self._h, sid, ctypes.byref(ip), ctypes.byref(port)))
        return ip.value, port.value

    def stats(self):
        st = {k: int(self._L.bb_tcp_hub_stat(self._h, i)) for i, k in enumerate(HUB_STATS)}
        st['answer_capacity'] = int(self._L.bb_tcp_hub_stat(self._h, len(HUB_STATS)))
        st['records'] = int(self._L.bb_tcp_hub_stat(self._h, len(HUB_STATS) + 1))
        st['lost'] = int(self._L.bb_tcp_hub_stat(self._h, len(HUB_STATS) + 2))
        return st

    def set_query_log(self, on):
        from ._lib import check
        check(self._L.bb_query_log_tcp_hub_enable(self._h, 1 if on else 0) if self._h else -1)

    def query_log(self, which):
        return _native_records(self._L, 'bb_query_log_tcp_hub', self._h, which, True)

    def destroy(self):
        if getattr(self, '_h', None):
            self._L.bb_tcp_hub_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass
