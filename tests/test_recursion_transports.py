"""Forwarded misses answered on every transport: the recursion's exchange is shared by all of them, and each transport
owner (the server's TCP loop, a balancer UDP session, a TCP hub) gets its misses back through its own sink and relays
them with its own framing.

CPU: oracle stand-ins (Oracle + RelayOracle for the dc1 server, ForwardOracle for GpuRecursion), dnspython clients over
TCP loopback, a fake balancer over socketpairs, and the native session / hub host code linked against the engine
stubs of tests/native (tcp_hub_stubs.cpp + backend_stubs.cpp), plus bb_backend_relay under ASan/UBSan
(tests/native/fuzz_backend_relay.cpp).  GPU: the same with Engines."""
import ctypes
import os
import random
import shutil
import socket
import struct
import subprocess
import threading
import time

import dns.message
import dns.query
import dns.rcode
import numpy as np
import pytest

import relay_oracle
import relaygen as G
import test_balancer_tcp as TB
from binder_b200 import _lib, balancer, synth
from binder_b200.forward import GpuRecursion
from binder_b200.recursion import QueueSink, Recursion, split_packets
from binder_b200.server import TcpFramer, createServer
from test_forward_loopback import QUESTIONS, _zone

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class WithRelay(object):
    """The dc1 server's resolver on the CPU: the resolve oracle composed with the relay oracle."""

    def __init__(self, orc):
        self.orc, self.rel = orc, relay_oracle.RelayOracle()

    def resolve_batch(self, *a, **k):
        return self.orc.resolve_batch(*a, **k)

    def relay_batch(self, *a, **k):
        return self.rel.relay_batch(*a, **k)


def makers(kind, rec_cls):
    """-> (zone resolver factory, the recursion's resolver)"""
    if kind == 'oracle':
        from forward_oracle import ForwardOracle
        from oracle_lib import Oracle
        make = lambda snap, rec: WithRelay(Oracle('foo.com', '', rec, snapshot=snap))      # noqa: E731
        return make, ForwardOracle() if rec_cls is GpuRecursion else relay_oracle.RelayOracle()
    from binder_b200.engine import Engine
    make = lambda snap, rec: Engine('foo.com', '', rec, snapshot=snap, max_batch=4096)   # noqa: E731
    return make, Engine('foo.com', '', True, max_batch=4096)


class Upstreams(object):
    """dc2 (a Server on its own zone), dc3 (silent), dc4 (this host): the upstream set of test_forward_loopback."""

    def __init__(self, make):
        self.silent = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        self.silent.bind(('127.0.0.1', 0))
        self.dc2 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc2', 20), False), 'host': '127.0.0.1', 'port': 0}).start()
        self.dcs = {'dc2': [('127.0.0.1', self.dc2.port)], 'dc3': [('127.0.0.1', self.silent.getsockname()[1])], 'dc4': ['10.99.0.1']}

    def close(self):
        self.dc2.stop()
        self.silent.close()


def tcp_exchange(port, wires, half_close=False, timeout=5.0):
    """Send the messages on one connection (pipelined), optionally half-close, read until every answer is in (or the
    server closes) -> [answer bytes] in arrival order"""
    s = socket.create_connection(('127.0.0.1', port), timeout=timeout)
    try:
        s.sendall(b''.join(TcpFramer.frame(w) for w in wires))
        if half_close:
            s.shutdown(socket.SHUT_WR)
        fr, got = TcpFramer(), []
        end = time.time() + timeout
        while len(got) < len(wires) and time.time() < end:
            chunk = s.recv(65536)
            if not chunk:
                break
            got += fr.feed(chunk)
        if half_close:                               # the server closes once everything owed is written
            s.settimeout(timeout)
            assert s.recv(1) == b''
        return got
    finally:
        s.close()


def summary(wire):
    r = dns.message.from_wire(wire)
    return r.rcode(), r.flags, sorted(rr.to_text() for rr in r.answer), r.edns


# ---- 1. DNS over TCP through server.py ---------------------------------------------------------------------------------
def tcp_answers(kind, rec_cls):
    make, rres = makers(kind, rec_cls)
    ups = Upstreams(make)
    rec = rec_cls(rres, 'foo.com', ups.dcs, my_addrs=['10.99.0.1'], timeout=0.5)
    dc1 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc1', 20), True), 'recursion': rec,
                        'host': '127.0.0.1', 'port': 0, 'tcp_idle_s': 0.2}).start()
    try:
        qs = [dns.message.make_query(n, t, use_edns=0 if e else -1) for n, t, e in QUESTIONS]
        tcp = [summary(tcp_exchange(dc1.port, [q.to_wire()])[0]) for q in qs]
        udp = [summary(dns.query.udp(q, '127.0.0.1', port=dc1.port, timeout=5).to_wire()) for q in qs]
        # a hit and a miss pipelined on one connection: both arrive (the relayed one may come second)
        hit, miss = (dns.message.make_query(n, 'A', id=i) for i, n in ((7, 'h3.dc1.foo.com'), (8, 'h4.dc2.foo.com')))
        both = {dns.message.from_wire(w).id: summary(w) for w in tcp_exchange(dc1.port, [hit.to_wire(), miss.to_wire()])}
        # half-closed right after one miss: the relayed reply is written before the server closes
        half = tcp_exchange(dc1.port, [dns.message.make_query('h5.dc2.foo.com', 'A', id=9).to_wire()], half_close=True)
        counters = dict(rec.counters)
        srv = dict(dc1.counters)
    finally:
        dc1.stop()
        ups.close()
        rec.close()
    return tcp, udp, both, [summary(w) for w in half], counters, srv


def run_tcp(kind):
    got = tcp_answers(kind, GpuRecursion)
    want = tcp_answers(kind, Recursion)
    assert got[0] == want[0] and got[2:4] == want[2:4]
    tcp, udp, both, half, counters, srv = got
    assert tcp == udp                                # every question: the TCP answer is the UDP answer
    rc = {name: g[0] for (name, _, _), g in zip(QUESTIONS, tcp)}
    assert all(rc['h%d.dc2.foo.com' % i] == dns.rcode.NOERROR for i in range(12))
    for name in ('nope.dc2.foo.com', 'h1.dc3.foo.com', 'h1.dc4.foo.com', 'h1.nodc.foo.com'):
        assert rc[name] == dns.rcode.REFUSED, name   # h1.dc3: silent upstream, after a timeout longer than tcp_idle_s
    assert both[7][2] == ['h3.dc1.foo.com. 30 IN A 10.1.0.3'] and both[8][2] == ['h4.dc2.foo.com. 30 IN A 10.2.0.4']
    assert half == [(dns.rcode.NOERROR, half[0][1], ['h5.dc2.foo.com. 30 IN A 10.2.0.5'], -1)]
    assert counters['tcp_skipped'] == 0 and counters['delivered'] >= 17 + 2
    assert srv['tcp_relayed'] >= 17 + 2


def test_tcp_misses_answered_cpu():
    run_tcp('oracle')


@pytest.mark.gpu
def test_tcp_misses_answered_gpu():
    run_tcp('gpu')


def test_submit_without_relay_batch_keeps_tcp_skipped():
    """A resolver without relay_batch: TCP misses are counted in tcp_skipped, as for a recursion without submit."""
    from oracle_lib import Oracle
    rec = Recursion(relay_oracle.RelayOracle(), 'foo.com', {'dc2': [('127.0.0.1', 9)]}, timeout=0.2)
    dc1 = createServer({'dnsDomain': 'foo.com', 'resolver': Oracle('foo.com', '', True, snapshot=_zone('dc1', 4)),
                        'recursion': rec, 'host': '127.0.0.1', 'port': 0}).start()
    try:
        s = socket.create_connection(('127.0.0.1', dc1.port), timeout=5)
        s.sendall(TcpFramer.frame(dns.message.make_query('h1.dc2.foo.com', 'A').to_wire()))
        end = time.time() + 5
        while rec.counters['tcp_skipped'] == 0 and time.time() < end:
            time.sleep(0.01)
        s.close()
        assert rec.counters['tcp_skipped'] == 1
    finally:
        dc1.stop()
        rec.close()


# ---- 2. the TCP size limit reaches the relay ---------------------------------------------------------------------------
LONG = '.'.join(['a' * 60, 'b' * 60, 'c' * 50]) + '.dc2.foo.com'


class CraftedUpstream(object):
    """A UDP upstream that answers every query with 12 CNAME RRs whose targets are compression pointers to the (long)
    question name: 370 bytes on the wire, each target 185 bytes once decompressed."""

    def __init__(self):
        self.sock = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        self.sock.bind(('127.0.0.1', 0))
        self.sock.settimeout(0.05)
        self.stop = False
        self.sent = []
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()

    def _run(self):
        while not self.stop:
            try:
                q, src = self.sock.recvfrom(4096)
            except socket.timeout:
                continue
            pos = 12
            while q[pos]:
                pos += 1 + q[pos]
            qtype = struct.unpack('>H', q[pos + 1:pos + 3])[0]
            r = G.raw_upstream(q[12:pos + 1], qtype, [(b'\xc0\x0c', 5, 1, 60 + k, b'\xc0\x0c') for k in range(12)])
            r = q[:2] + r[2:]
            self.sent.append(r)
            self.sock.sendto(r, src)

    def close(self):
        self.stop = True
        self.t.join(2)
        self.sock.close()


def size_limit(kind):
    make, rres = makers(kind, GpuRecursion)
    up = CraftedUpstream()
    rec = GpuRecursion(rres, 'foo.com', {'dc2': [('127.0.0.1', up.sock.getsockname()[1])]}, timeout=2.0)
    dc1 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc1', 4), True), 'recursion': rec,
                        'host': '127.0.0.1', 'port': 0}).start()
    try:
        q = dns.message.make_query(LONG, 'A', id=77)
        c = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        c.settimeout(5)
        c.sendto(q.to_wire(), ('127.0.0.1', dc1.port))
        u = c.recv(65535)                            # the server's bytes, not dnspython's re-encoding
        c.close()
        t = tcp_exchange(dc1.port, [q.to_wire()])[0]
    finally:
        dc1.stop()
        rec.close()
        up.close()
    assert up.sent
    data, off = synth.pack_batch([q.to_wire()])
    for wire, tcp in ((u, False), (t, True)):
        ud, uo = synth.pack_batch([up.sent[0]])
        out, ooff, olen, st = relay_oracle.relay_batch(data, off, ud, uo, tcp=tcp)
        assert st[0] == 0 and wire == bytes(out[:olen[0]])
    assert dns.message.from_wire(u).flags & 0x200 and len(u) <= 512
    assert not dns.message.from_wire(t).flags & 0x200 and len(t) > 512 and struct.unpack('>H', t[6:8])[0] == 12


def test_tcp_size_limit_reaches_relay_cpu():
    size_limit('oracle')


@pytest.mark.gpu
def test_tcp_size_limit_reaches_relay_gpu():
    size_limit('gpu')


# ---- 3. balancer UDP sessions -------------------------------------------------------------------------------------------
def udp_frame(pkt, ip, port):
    return struct.pack('<IIII', balancer.INBOUND_UDP, ip, port, len(pkt)) + pkt


def split_out(buf):
    pos, frames = 0, []
    while pos < len(buf):
        t, ip, port, ln = struct.unpack_from('<IIII', buf, pos)
        assert t == balancer.OUTBOUND_UDP
        frames.append((ip, port, bytes(buf[pos + 16:pos + 16 + ln])))
        pos += 16 + ln
    return frames


def upstream_query(pkt):
    """The upstream query the exchange sends for a client query (ID aside): flags & 0x7800, QDCOUNT 1, the question"""
    pos = 12
    while pkt[pos]:
        pos += 1 + pkt[pos]
    flags = struct.unpack('>H', pkt[2:4])[0] & 0x7800
    return struct.pack('>HHHHHH', 0x1234, flags, 1, 0, 0, 0) + pkt[12:pos + 5]


def balancer_udp(kind):
    """A fake balancer over a socketpair: INBOUND_UDP frames mixing hits and misses into a Backend whose recursion is
    GpuRecursion; the host side pumps the socket, feeds, and writes what feed() and drain() return."""
    make, rres = makers(kind, GpuRecursion)
    ups = Upstreams(make)
    rec = GpuRecursion(rres, 'foo.com', ups.dcs, my_addrs=['10.99.0.1'], timeout=0.5)
    dc1 = make(_zone('dc1', 20), True)
    bal, host = socket.socketpair()
    woke = threading.Event()
    be = balancer.Backend(dc1, rec, shuffle_seed=5, wake=woke.set)
    qs = [dns.message.make_query(n, t, use_edns=0 if e else -1, id=300 + i).to_wire() for i, (n, t, e) in enumerate(QUESTIONS)]
    addr = [(0x0A000000 + i, 2000 + i) for i in range(len(qs))]
    try:
        bal.sendall(struct.pack('<I', balancer.CLIENT_HELLO) + b''.join(udp_frame(q, *a) for q, a in zip(qs, addr)))
        host.settimeout(5)
        buf = b''
        while len(buf) < 4 + sum(16 + len(q) for q in qs):
            buf += host.recv(65536)
        first = be.feed(buf)                          # misses go to the recursion; the hits' frames come back now
        assert first[:4] == struct.pack('<I', balancer.SERVER_HELLO)
        host.sendall(first)
        n_miss = be.counters['missed']
        relayed = b''
        end = time.time() + 5
        while len(split_out(relayed)) < n_miss and time.time() < end:
            woke.wait(0.1)
            woke.clear()
            relayed += be.drain()
        host.sendall(relayed)
        host.shutdown(socket.SHUT_WR)
        got = b''
        bal.settimeout(5)
        while True:
            c = bal.recv(65536)
            if not c:
                break
            got += c
    finally:
        bal.close()
        host.close()
        ups.close()
        rec.close()
    hits = split_out(first[4:])
    frames = split_out(got[4:])
    assert frames[:len(hits)] == hits and len(frames) == len(qs) and be.counters['relayed'] == n_miss, (be.counters, rec.counters)
    by_addr = {(ip, port): w for ip, port, w in frames}
    assert sorted(by_addr) == sorted(addr)
    # each miss's payload is the oracle's relay of its query with the upstream's answer (the hit is the oracle's answer)
    from oracle_lib import Oracle
    dc2 = Oracle('foo.com', '', False, snapshot=_zone('dc2', 20))
    for (name, _, _), q, a in zip(QUESTIONS, qs, addr):
        if name == 'h3.dc1.foo.com':
            continue
        if name.endswith('.dc2.foo.com') or name.endswith('.arpa'):
            d, o = synth.pack_batch([upstream_query(q)])
            out, ooff, olen, st, _ = dc2.resolve_batch(d, o)
            upstream = bytes(out[:olen[0]])
        else:
            upstream = b''                           # silent, this host, unknown datacenter: the lookup failed
        qd, qo = synth.pack_batch([q])
        ud, uo = synth.pack_batch([upstream])
        out, ooff, olen, st = relay_oracle.relay_batch(qd, qo, ud, uo)
        assert by_addr[a] == bytes(out[:olen[0]]), name
    return by_addr


def test_balancer_udp_misses_relayed_cpu():
    balancer_udp('oracle')


@pytest.mark.gpu
def test_balancer_udp_misses_relayed_gpu():
    assert balancer_udp('gpu') == balancer_udp('oracle')


# the native session's host code on the CPU, against Backend.relay
_STUB = {}


@pytest.fixture(scope='module')
def stub_lib(tmp_path_factory):
    """csrc/balancer_frames.cpp + balancer_relay.cpp + balancer_tcp.cpp with the engine stubs, as one host-only library"""
    if 'L' not in _STUB:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        so = str(tmp_path_factory.mktemp('be') / 'libbackend_cpu.so')
        csrc = os.path.join(ROOT, 'binder_b200', 'csrc')
        subprocess.check_call([cxx, '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                               '-o', so] + [os.path.join(csrc, f) for f in ('balancer_frames.cpp', 'balancer_relay.cpp', 'balancer_tcp.cpp')] +
                              [os.path.join(ROOT, 'tests', 'native', f) for f in ('tcp_hub_stubs.cpp', 'backend_stubs.cpp')])
        L = ctypes.CDLL(so)
        for name, (res, args) in _lib.SYMBOLS.items():
            if name.startswith('bb_tcp_hub_') or name.startswith('bb_backend_'):
                getattr(L, name).restype = res
                getattr(L, name).argtypes = args
        L.bb_stub_set.argtypes = [TB.RESOLVE, TB.RELAY, ctypes.c_uint32, ctypes.c_uint32]
        _STUB['L'] = L
    return _STUB['L']


class FailingRelay(TB.CpuEngine):
    """CpuEngine whose relay calls listed in `fail_calls` (0-based) fail with BB_ERR_CUDA"""

    def __init__(self, L, oracle, fail_calls=(), **kw):
        self.fail_calls, self.n_relay = set(fail_calls), 0
        TB.CpuEngine.__init__(self, L, oracle, **kw)

    def _relay(self, *a):
        k, self.n_relay = self.n_relay, self.n_relay + 1
        if k in self.fail_calls:
            return -3
        return TB.CpuEngine._relay(self, *a)


class RelayFailAt(object):
    """relay_batch that fails on the calls listed (0-based), else the relay oracle"""

    def __init__(self, fail_calls=()):
        self.fail_calls, self.n = set(fail_calls), 0

    def relay_batch(self, q, qo, u, uo, tcp=False):
        k, self.n = self.n, self.n + 1
        if k in self.fail_calls:
            raise RuntimeError('batch failed')
        return relay_oracle.relay_batch(q, qo, u, uo, tcp)


def relay_corpus(seed, n):
    """Miss packets (fuzzed zone queries, malformed ones, EDNS), upstreams (failed, A answers, malformed bytes), sources"""
    import fuzzgen
    rng = random.Random(seed)
    snap, info = fuzzgen.gen_zone(seed + 40, n_top=20)
    pool = fuzzgen.gen_queries(seed, info, n=300) + [p for p in fuzzgen.malformed_packets() if p]
    qs = [rng.choice(pool) for _ in range(n)]
    ups = []
    for i, p in enumerate(qs):
        k = rng.randrange(6)
        if k == 0 or len(p) < 13:
            ups.append(b'')
        elif k == 5:
            ups.append(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 80))))
        else:
            ups.append(TB.upstream_for(p, i + 1) if p[12:].find(b'\0') >= 0 and len(p) >= p[12:].find(b'\0') + 17 else b'')
    dst = [(rng.getrandbits(32), rng.randrange(65536)) for _ in qs]
    return snap, info, qs, ups, dst


@pytest.mark.parametrize('seed,max_batch,fail', [(0, 4096, ()), (1, 37, ()), (2, 25, (1, 3))])
def test_native_backend_relay_on_cpu_matches_python(stub_lib, seed, max_batch, fail):
    from oracle_lib import Oracle
    snap, info, qs, ups, dst = relay_corpus(seed, 150)
    orc = Oracle(info['dns_domain'], '', True, snapshot=snap)
    eng = FailingRelay(stub_lib, orc, fail)
    nb = balancer.NativeBackend(eng, max_batch=max_batch, lib=stub_lib)
    py = balancer.Backend(orc, relayer=RelayFailAt(fail), max_batch=max_batch)
    a, b = nb.relay(qs, ups, dst), py.relay(qs, ups, dst)
    assert a == b and eng.error is None
    st = nb.stats()
    assert st['relayed'] == py.counters['relayed'] and st['relay_failed'] == py.counters['relay_failed']
    assert st['relay_failed'] == sum(len(qs[k * max_batch:(k + 1) * max_batch]) for k in fail)
    assert (nb.last_rc == -3) == bool(fail) and len(split_out(a)) == st['relayed'] > 0
    assert nb.relay([], [], []) == b''
    nb.close()


def test_native_backend_relay_argument_errors(stub_lib):
    from binder_b200._lib import BinderError
    from oracle_lib import Oracle
    nb = balancer.NativeBackend(TB.CpuEngine(stub_lib, Oracle('foo.com', '', True)), lib=stub_lib)
    p, n = ctypes.c_void_p(), ctypes.c_size_t(0)
    assert stub_lib.bb_backend_relay(None, None, None, None, None, None, None, 0, ctypes.byref(p), ctypes.byref(n)) == -1
    bad = np.array([0, 5, 3], dtype=np.uint32)
    z = np.zeros(2, np.uint32)
    assert stub_lib.bb_backend_relay(nb._h, b'x' * 8, bad.ctypes.data, b'x' * 8, bad.ctypes.data, z.ctypes.data, z.ctypes.data, 2,
                                     ctypes.byref(p), ctypes.byref(n)) == -1
    nb.close()
    with pytest.raises(BinderError):
        nb.relay([b'x'], [b''], [(1, 2)])


def test_backend_relay_sanitizer_clean(tmp_path):
    cxx = shutil.which('g++')
    if not cxx:
        pytest.skip('no g++')
    exe = str(tmp_path / 'fuzz_backend_relay')
    csrc = os.path.join(ROOT, 'binder_b200', 'csrc')
    cmd = [cxx, '-std=c++17', '-O1', '-g', '-fsanitize=address,undefined', '-fno-omit-frame-pointer', '-Wall', '-Werror',
           '-I', os.path.join(ROOT, 'include'), '-I', csrc, '-o', exe, os.path.join(ROOT, 'tests', 'native', 'fuzz_backend_relay.cpp'),
           os.path.join(csrc, 'balancer_frames.cpp'), os.path.join(csrc, 'balancer_relay.cpp')]
    b = subprocess.run(cmd, capture_output=True, text=True)
    if b.returncode != 0 and 'sanitize' in b.stderr:
        pytest.skip('toolchain without sanitizer runtimes')
    assert b.returncode == 0, b.stderr[-2000:]
    p = subprocess.run([exe, '400'], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith('OK') and 'runtime error' not in p.stderr, (p.stdout[-500:], p.stderr[-3000:])


def test_backend_relay_is_exported():
    hdr = open(os.path.join(ROOT, 'include', 'binder_b200.h')).read()
    assert 'bb_backend_relay(' in hdr and 'bb_backend_relay' in _lib.SYMBOLS
    assert hasattr(ctypes.CDLL(_lib.SO_PATH), 'bb_backend_relay')


@pytest.mark.gpu
@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_native_backend_relay_matches_python(ordered):
    from binder_b200.engine import Engine
    snap, info, qs, ups, dst = relay_corpus(7, 3000)
    eng = Engine(info['dns_domain'], recursion=True, snapshot=snap, max_batch=4096, ordered=ordered)
    for mb in (4096, 700):
        nb = balancer.NativeBackend(eng, max_batch=mb)
        py = balancer.Backend(None, relayer=relay_oracle.RelayOracle(), max_batch=mb)
        got = nb.relay(qs, ups, dst)
        assert got == py.relay(qs, ups, dst) and nb.last_rc == 0
        assert nb.stats()['relayed'] == py.counters['relayed'] > 1000 and nb.stats()['relay_failed'] == 0
        nb.close()


@pytest.mark.gpu
def test_gpu_backend_relay_capacity_failure_loses_only_its_batch():
    """2,048 EDNS relays of 1,200-byte replies do not fit a session's 1 MB of reply room: that batch is lost and counted,
    the next batch's replies arrive."""
    from binder_b200.engine import Engine
    eng = Engine('foo.com', recursion=True, max_batch=4096)
    nb = balancer.NativeBackend(eng, max_batch=2048)
    big_q = dns.message.make_query(LONG, 'A', use_edns=0, payload=1200).to_wire()
    pos = 12
    while big_q[pos]:
        pos += 1 + big_q[pos]
    big_up = G.raw_upstream(big_q[12:pos + 1], 1, [(b'\xc0\x0c', 5, 1, 60, b'\xc0\x0c')] * 12)
    small_q = [synth.make_query('h%d.dc2.foo.com' % i, 'A', qid=i) for i in range(100)]
    small_up = [TB.upstream_for(q, i + 1) for i, q in enumerate(small_q)]
    qs, ups = [big_q] * 2048 + small_q, [big_up] * 2048 + small_up
    dst = [(1, i) for i in range(len(qs))]
    got = nb.relay(qs, ups, dst)
    assert nb.last_rc == -5
    st = nb.stats()
    assert st['relay_failed'] == 2048 and st['relayed'] == 100
    assert got == balancer.Backend(None, relayer=relay_oracle.RelayOracle()).relay(small_q, small_up, dst[2048:])


# ---- 4. balancer TCP sessions --------------------------------------------------------------------------------------------
def hub_through_recursion(hub, kind, n_sess=20):
    """20 hub sessions, each with one miss and one hit, half-closed: the host submits flush()'s misses to GpuRecursion
    with its queue sink and hands what it drains to hub.relay().  Each session is closable only after its relay."""
    make, rres = makers(kind, GpuRecursion)
    ups = Upstreams(make)
    rec = GpuRecursion(rres, 'foo.com', ups.dcs, my_addrs=['10.99.0.1'], timeout=0.5)
    woke = threading.Event()
    sink = QueueSink(woke.set)
    try:
        sids = [hub.open() for _ in range(n_sess)]
        for j, s in enumerate(sids):
            miss = dns.message.make_query('h%d.dc2.foo.com' % (j % 20), 'A', id=j).to_wire()
            hit = dns.message.make_query('h%d.dc1.foo.com' % (j % 20), 'A', id=1000 + j).to_wire()
            assert hub.feed(s, TB.hello(0x0A000000 + j, 3000 + j) + TcpFramer.frame(miss) + TcpFramer.frame(hit))
            hub.eof(s)
        misses = hub.flush(11)
        assert sorted(sid for _, sid in misses) == sorted(sids)
        for p, sid in misses:
            rec.submit(p, sink, sid)
        for s in sids:                               # the hit is written, the miss still owed
            out, closable = hub.output(s)
            assert not closable and len(TcpFramer().feed(out[4:])) == 1
        done = 0
        end = time.time() + 5
        while done < len(misses) and time.time() < end:
            woke.wait(0.1)
            woke.clear()
            for q, qo, u, uo, tags in sink.drain():
                hub.relay(split_packets(q, qo), split_packets(u, uo), tags)
                done += len(tags)
        outs = []
        for j, s in enumerate(sids):
            out, closable = hub.output(s)
            got = TcpFramer().feed(out[4:])
            assert len(got) == 2 and not closable
            ans = {dns.message.from_wire(w).id: sorted(rr.to_text() for rr in dns.message.from_wire(w).answer) for w in got}
            assert ans[j] == ['h%d.dc2.foo.com. 30 IN A 10.2.0.%d' % (j % 20, j % 20)]
            hub.consume(s, len(out))
            assert hub.output(s) == (b'', True)
            outs.append(out)
        return outs, hub.stats()
    finally:
        ups.close()
        rec.close()


def test_hub_misses_through_recursion_cpu(stub_lib):
    from oracle_lib import Oracle
    orc = Oracle('foo.com', '', True, snapshot=_zone('dc1', 20))
    py, st_py = hub_through_recursion(balancer.TcpHub(orc, relayer=relay_oracle.RelayOracle()), 'oracle')
    eng = TB.CpuEngine(stub_lib, orc)
    nat, st_nat = hub_through_recursion(balancer.NativeTcpHub(eng, lib=stub_lib), 'oracle')
    assert nat == py and {k: st_nat[k] for k in st_py} == st_py and st_py['relayed'] == 20 and eng.error is None


@pytest.mark.gpu
def test_gpu_native_hub_misses_through_recursion():
    from binder_b200.engine import Engine
    from oracle_lib import Oracle
    snap = _zone('dc1', 20)
    py, st_py = hub_through_recursion(balancer.TcpHub(Oracle('foo.com', '', True, snapshot=snap),
                                                      relayer=relay_oracle.RelayOracle()), 'oracle')
    nat, st_nat = hub_through_recursion(balancer.NativeTcpHub(Engine('foo.com', '', True, snapshot=snap, max_batch=4096)), 'gpu')
    assert nat == py and {k: st_nat[k] for k in st_py} == st_py and st_py['relayed'] == 20
