"""DNS-over-TCP clients behind mname-balancer (deps/mname-balancer/backend.c:22-113, tcp_proxy.c:160-300): each client
connection arrives as its own AF_UNIX session, INBOUND_TCP {3, ip, port} -> INBOUND_TCP_OK (1003), then the raw
length-prefixed DNS stream.  The TCP hub (binder_b200.balancer.TcpHub / NativeTcpHub, csrc/balancer_tcp.cpp) resolves the
messages of all its sessions together as TCP batches.

CPU: the Python hub on the oracle against an independent model of the stream (which messages complete when, which batch
and query index each one lands on); protocol edges; misses and their relay.  The native hub's host code also runs on the
CPU, linked against stand-ins for the engine calls (tests/native/tcp_hub_stubs.cpp) that answer with the oracles.
GPU: NativeTcpHub on an Engine against the Python hub on the oracle, byte for byte and counter for counter."""
import ctypes
import os
import random
import shutil
import socket
import struct
import subprocess

import dns.message
import numpy as np
import pytest

import fuzzgen
import helpers as H
import relay_oracle
import relaygen as G
from binder_b200 import _lib, synth
from binder_b200.balancer import (CLIENT_HEARTBEAT, CLIENT_HELLO, HUB_STATS, INBOUND_TCP, INBOUND_TCP_OK, INBOUND_UDP,
                                  NativeTcpHub, TcpHub)
from binder_b200.server import TcpFramer
from test_tcp import big_zone, big_zone_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK = struct.pack('<I', INBOUND_TCP_OK)


def hello(ip=0x0A000001, port=40000):
    return struct.pack('<III', INBOUND_TCP, ip, port)


# ---- fixtures: zones, sessions, chunkings --------------------------------------------------------------------------
def workload(kind, seed, n_sess=50):
    """-> (snapshot, dns_domain, recursion, [query packets of each session])"""
    rng = random.Random(seed)
    if kind == 'fuzz':
        snap, info = fuzzgen.gen_zone(seed + 700, n_top=30)
        pool = fuzzgen.gen_queries(seed, info, n=500) + [p for p in fuzzgen.malformed_packets() if p]
        dom, rec = info['dns_domain'], True
    else:                                        # the 200- and 1,300-child services
        snap, dom, rec = big_zone(), 'foo.com', False
        pool = big_zone_batch()
    return snap, dom, rec, [[rng.choice(pool) for _ in range(rng.randint(1, 8))] for _ in range(n_sess)]


def session_stream(queries, ip, port):
    """INBOUND_TCP, then every query length-prefixed, as ONE write"""
    return hello(ip, port) + b''.join(TcpFramer.frame(q) for q in queries)


def chunk_events(streams, seed):
    """Each stream cut at random points (always inside the 12-byte frame and inside a 2-byte prefix), the sessions'
    chunks interleaved at random with each session's own order kept -> [(session index, bytes)]"""
    rng = random.Random(seed)
    per = []
    for s in streams:
        cuts = {rng.randint(1, 11), 13} | {rng.randint(1, len(s) - 1) for _ in range(rng.randint(0, 6))}
        cuts = sorted(c for c in cuts if 0 < c < len(s))
        per.append([s[a:b] for a, b in zip([0] + cuts, cuts + [len(s)])])
    order = [j for j, ch in enumerate(per) for _ in ch]
    rng.shuffle(order)
    pos = [0] * len(per)
    ev = []
    for j in order:
        ev.append((j, per[j][pos[j]]))
        pos[j] += 1
    return ev


def drive(hub, streams, events, flush_every, seed0):
    """Open a session per stream, feed the events, flush every `flush_every` events and at the end, half-close every
    other session.  -> (session ids, [(miss packet, session index)])"""
    sids = [hub.open() for _ in streams]
    index = {s: j for j, s in enumerate(sids)}
    misses = []
    for k, (j, chunk) in enumerate(events):
        assert hub.feed(sids[j], chunk)
        if (k + 1) % flush_every == 0:
            misses += [(p, index[s]) for p, s in hub.flush(seed0 + k)]
    for j in range(0, len(sids), 2):
        hub.eof(sids[j])
    misses += [(p, index[s]) for p, s in hub.flush(seed0 + len(events))]
    return sids, misses


def model(orc, sessions, events, flush_every, seed0, max_batch):
    """What each session must receive, restated from the byte positions where its messages end: INBOUND_TCP_OK, then the
    oracle's TCP answer (tcp=True) of every message, resolved in the batch and at the query index its completion gives
    it.  -> ([expected output of each session], [(miss packet, session index)])"""
    ends = [list(12 + np.cumsum([2 + len(q) for q in qs])) for qs in sessions]
    fed, done = [0] * len(sessions), [0] * len(sessions)
    want = [bytearray(OK) for _ in sessions]
    pending, misses = [], []

    def flush(seed):
        for b0 in range(0, len(pending), max_batch):
            batch = pending[b0:b0 + max_batch]
            data, off = synth.pack_batch([sessions[j][m] for j, m in batch])
            out, ooff, olen, st, _ = orc.resolve_batch(data, off, seed=seed, qidx_base=b0, tcp=True)
            for i, (j, m) in enumerate(batch):
                if st[i] == 0:
                    want[j] += TcpFramer.frame(bytes(out[ooff[i]:ooff[i] + olen[i]]))
                elif st[i] == 1:
                    misses.append((sessions[j][m], j))
        del pending[:]

    for k, (j, chunk) in enumerate(events):
        fed[j] += len(chunk)
        while done[j] < len(ends[j]) and ends[j][done[j]] <= fed[j]:
            pending.append((j, done[j]))
            done[j] += 1
        if (k + 1) % flush_every == 0:
            flush(seed0 + k)
    flush(seed0 + len(events))
    return [bytes(w) for w in want], misses


def upstream_for(pkt, i):
    """A fake upstream response to a miss (tests/relaygen.py): every third lookup failed (empty), else A answers."""
    if i % 3 == 0:
        return b''
    pos = 12
    while pkt[pos]:
        pos += 1 + pkt[pos]
    qtype = struct.unpack('>H', pkt[pos + 1:pos + 3])[0]
    return G.raw_upstream(pkt[12:pos + 1], qtype, [(b'\xc0\x0c', 1, 1, 60 + i, bytes([10, 9, i & 255, 1])) for _ in range(1 + i % 4)])


def relay_expected(misses_idx, ups):
    """relay oracle replies (TCP) of [(packet, session index)]"""
    q, qo = synth.pack_batch([p for p, _ in misses_idx])
    u, uo = synth.pack_batch(ups)
    out, ooff, olen, st = relay_oracle.relay_batch(q, qo, u, uo, tcp=True)
    return [bytes(out[ooff[i]:ooff[i] + olen[i]]) if st[i] == 0 else None for i in range(len(ups))]


def outputs(hub, sids):
    return [hub.output(s)[0] for s in sids]


# ---- the Python hub on the oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,seed', [('fuzz', 0), ('fuzz', 1), ('big', 2)])
def test_python_hub_matches_stream_model(kind, seed):
    from oracle_lib import Oracle
    snap, dom, rec, sessions = workload(kind, seed)
    orc = Oracle(dom, '', rec, snapshot=snap)
    streams = [session_stream(qs, 0x0A000000 + j, 1024 + j) for j, qs in enumerate(sessions)]
    events = chunk_events(streams, seed)
    hub = TcpHub(orc, max_batch=64, relayer=relay_oracle.RelayOracle())
    sids, misses = drive(hub, streams, events, 37, 100 * seed)
    want, want_miss = model(orc, sessions, events, 37, 100 * seed, 64)
    assert outputs(hub, sids) == want
    assert misses == want_miss and (not rec or misses)
    assert [hub.peer(s) for s in sids] == [(0x0A000000 + j, 1024 + j) for j in range(len(sids))]
    st = hub.stats()
    n = sum(len(qs) for qs in sessions)
    assert st['sessions'] == st['open'] == len(sessions) and st['messages'] == n and st['queued'] == 0
    assert st['answered'] + st['missed'] + st['dropped'] == n and st['protocol_errors'] == st['failed'] == 0
    # a session may close once it has half-closed, owes nothing and has nothing left to write
    for j, s in enumerate(sids):
        out, closable = hub.output(s)
        assert not closable
        hub.consume(s, len(out))
        owes = any(mj == j for _, mj in misses)
        assert hub.output(s)[1] == (j % 2 == 0 and not owes)
    if kind == 'big':
        # whole over TCP where UDP sets TC; the 2,600 SRV records of the 1,300-child service cut at 65,516 bytes with TC
        srv_big = synth.make_query('_http._tcp.big.foo.com', 'SRV', qid=7)
        srv_huge = synth.make_query('_http._tcp.huge.foo.com', 'SRV', qid=8)
        s = hub.open()
        hub.feed(s, hello() + TcpFramer.frame(srv_big) + TcpFramer.frame(srv_huge))
        hub.flush(5)
        got = TcpFramer().feed(hub.output(s)[0][4:])
        big, huge = (H.decode_semantic(g) for g in got)
        assert not big[4]['tc'] and len(big[1]) == 200 and len(big[3]) == 200
        u = H.resolve_list(orc, [srv_big])[0][0][1]
        assert H.decode_semantic(u)[4]['tc'] and len(u) <= 512
        assert huge[4]['tc'] and len(got[1]) == 65516 and len(huge[1]) < 2600


def test_python_hub_relays_misses_to_their_sessions():
    from oracle_lib import Oracle
    snap, dom, rec, sessions = workload('fuzz', 5)
    orc = Oracle(dom, '', True, snapshot=snap)
    streams = [session_stream(qs, 1, 2) for qs in sessions]
    events = chunk_events(streams, 5)
    hub = TcpHub(orc, max_batch=4096, relayer=relay_oracle.RelayOracle())
    sids, misses = drive(hub, streams, events, 1000, 9)
    want, _ = model(orc, sessions, events, 1000, 9, 4096)
    assert outputs(hub, sids) == want and len(misses) > 10
    # relayed out of order (RFC 7766): each reply goes to the session its miss came from, in relay order per session
    order = list(range(len(misses)))
    random.Random(1).shuffle(order)
    mix = [misses[i] for i in order]
    ups = [upstream_for(p, i) for i, (p, _) in enumerate(mix)]
    replies = relay_expected(mix, ups)
    hub.relay([p for p, _ in mix], ups, [sids[j] for _, j in mix])
    for i, (p, j) in enumerate(mix):
        if replies[i] is not None:
            want[j] += TcpFramer.frame(replies[i])
            assert replies[i][:2] == p[:2]
    assert outputs(hub, sids) == want
    st = hub.stats()
    assert st['relayed'] == sum(r is not None for r in replies) and st['relayed'] + st['dropped'] >= len(mix)
    for s in sids[::2]:                          # nothing owed any more: half-closed sessions may close once written
        hub.consume(s, len(hub.output(s)[0]))
        assert hub.output(s)[1]


# ---- protocol edges, on both hubs --------------------------------------------------------------------------------------
def edge_cases(hub, orc):
    q1, q2 = synth.make_query('hosta.foo.com', 'A', qid=1), synth.make_query('hosta.foo.com', 'A', qid=2)
    ans = lambda q: TcpFramer.frame(H.resolve_list(orc, [q])[0][0][1])      # noqa: E731
    good_a, good_b = hub.open(), hub.open()
    assert hub.feed(good_a, hello()[:5])                     # data arriving before the frame completes
    assert hub.output(good_a) == (b'', False)
    bad = {}
    for name, first in (('hello', struct.pack('<I', CLIENT_HELLO)), ('heartbeat', struct.pack('<I', CLIENT_HEARTBEAT)),
                        ('udp', struct.pack('<IIII', INBOUND_UDP, 1, 2, len(q1)) + q1), ('unknown', struct.pack('<I', 77))):
        bad[name] = hub.open()
        assert hub.feed(bad[name], first[:2])                # not yet a whole type word
        assert not hub.feed(bad[name], first[2:])
        assert not hub.feed(bad[name], hello())              # reads nothing more
    assert hub.feed(good_a, hello()[5:] + TcpFramer.frame(q1)[:1])
    assert hub.feed(good_b, hello() + TcpFramer.frame(q1) + TcpFramer.frame(q2))
    assert hub.feed(good_a, TcpFramer.frame(q1)[1:] + TcpFramer.frame(q2)[:3])
    zero = hub.open()                                        # a zero-length message: what completed before is answered
    assert not hub.feed(zero, hello() + TcpFramer.frame(q1) + b'\x00\x00' + TcpFramer.frame(q2))
    only = hub.open()                                        # only the handshake, then half-close
    assert hub.feed(only, hello(7, 8))
    half = hub.open()                                        # half-close right after the last query
    assert hub.feed(half, hello() + TcpFramer.frame(q1) + TcpFramer.frame(q2) + TcpFramer.frame(q1)[:4])
    hub.eof(half)
    hub.eof(only)
    assert hub.output(half) == (OK, False)                  # two queries still owed
    assert hub.output(only) == (OK, False)                  # one frame still to write
    assert hub.flush(3) == []
    for s in bad.values():
        assert hub.output(s) == (b'', True)
    assert hub.output(good_a) == (OK + ans(q1), False)      # q2 is incomplete
    assert hub.output(good_b) == (OK + ans(q1) + ans(q2), False)
    assert hub.output(zero) == (OK + ans(q1), False)
    assert hub.output(half) == (OK + ans(q1) + ans(q2), False)
    assert hub.peer(only) == (7, 8) and hub.peer(bad['hello']) == (0, 0)
    for s in (zero, half, only):
        out, _ = hub.output(s)
        hub.consume(s, 3)
        assert hub.output(s) == (out[3:], False)
        hub.consume(s, len(out) - 3)
        assert hub.output(s) == (b'', True)
    assert hub.feed(good_a, TcpFramer.frame(q2)[3:])
    hub.flush(4)
    assert hub.output(good_a)[0] == OK + ans(q1) + ans(q2)
    st = hub.stats()
    assert st['protocol_errors'] == 5 and st['sessions'] == 9 and st['messages'] == 7 and st['answered'] == 7
    hub.close(bad['hello'])
    assert hub.stats()['open'] == 8
    return {k: st[k] for k in HUB_STATS}


def test_protocol_edges_python():
    from oracle_lib import Oracle
    orc = Oracle('foo.com', '', False, snapshot=big_zone())
    hub = TcpHub(orc)
    edge_cases(hub, orc)
    for call in (lambda: hub.feed(99, b'x'), lambda: hub.output(99), lambda: hub.close(99)):
        with pytest.raises(KeyError):
            call()


# ---- the native hub's host code on the CPU -------------------------------------------------------------------------
RESOLVE = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p,
                           ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32)
RELAY = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32,
                         ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p)
_STUB = {}


@pytest.fixture(scope='module')
def hub_lib(tmp_path_factory):
    """csrc/balancer_tcp.cpp + tests/native/tcp_hub_stubs.cpp as one host-only library"""
    if 'L' not in _STUB:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        so = str(tmp_path_factory.mktemp('hub') / 'libtcphub_cpu.so')
        subprocess.check_call([cxx, '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                               '-o', so, os.path.join(ROOT, 'binder_b200', 'csrc', 'balancer_tcp.cpp'),
                               os.path.join(ROOT, 'tests', 'native', 'tcp_hub_stubs.cpp')])
        L = ctypes.CDLL(so)
        for name, (res, args) in _lib.SYMBOLS.items():
            if name.startswith('bb_tcp_hub_'):
                getattr(L, name).restype = res
                getattr(L, name).argtypes = args
        L.bb_stub_set.argtypes = [RESOLVE, RELAY, ctypes.c_uint32, ctypes.c_uint32]
        _STUB['L'] = L
    return _STUB['L']


def _arr(ctype, addr, n):
    return (ctype * max(n, 1)).from_address(addr)


class CpuEngine(object):
    """What the native hub's engine calls see on the CPU: the oracles' answers, packed in REVERSE query order (the
    arrival packing gives no order either) with the miss list reversed.  `fail`: query indices whose batch fails with
    BB_ERR_CUDA; `calls`: (qidx_base, n) of every resolve call."""
    _h = 1                                       # the hub only hands the handle back to the engine calls

    def __init__(self, L, oracle, max_batch=1 << 16, max_batch_bytes=1 << 22):
        self.oracle, self.fail, self.calls, self.error = oracle, set(), [], None
        self._cb = (RESOLVE(self._resolve), RELAY(self._relay))
        L.bb_stub_set(self._cb[0], self._cb[1], max_batch, max_batch_bytes)

    def _put(self, results, out, out_cap, out_off, out_len, status, n):
        o, oo, ol, st = results[:4]
        if int(ol.astype(np.int64).sum()) > out_cap:
            return -5
        offs, lens, sts, pos = _arr(ctypes.c_uint32, out_off, n + 1), _arr(ctypes.c_uint16, out_len, n), _arr(ctypes.c_uint8, status, n), 0
        for i in reversed(range(n)):
            ctypes.memmove(out + pos, o[oo[i]:oo[i] + ol[i]].tobytes(), int(ol[i]))
            offs[i], lens[i], sts[i] = pos, int(ol[i]), int(st[i])
            pos += int(ol[i])
        offs[n] = pos
        return 0

    def _resolve(self, pkts, pkt_off, n, seed, qidx, out, out_cap, out_off, out_len, status, miss, n_miss, flags):
        try:
            self.calls.append((qidx, n))
            if any(qidx <= f < qidx + n for f in self.fail):
                return -3
            off = np.array(_arr(ctypes.c_uint32, pkt_off, n + 1), dtype=np.uint32)
            data = np.frombuffer(ctypes.string_at(pkts, int(off[n])) + bytes(32), dtype=np.uint8)
            res = self.oracle.resolve_batch(data, off, seed=seed, qidx_base=qidx, tcp=bool(flags & 1))
            rc = self._put(res, out, out_cap, out_off, out_len, status, n)
            ms = [int(x) for x in res[4]][::-1]
            m = _arr(ctypes.c_uint32, miss, n)
            for k, x in enumerate(ms):
                m[k] = x
            ctypes.c_uint32.from_address(n_miss).value = len(ms)
            return rc
        except Exception as e:                   # surfaced by the test, not swallowed by ctypes
            self.error = e
            return -3

    def _relay(self, q, q_off, up, up_off, n, flags, out, out_cap, out_off, out_len, status):
        try:
            qo = np.array(_arr(ctypes.c_uint32, q_off, n + 1), dtype=np.uint32)
            uo = np.array(_arr(ctypes.c_uint32, up_off, n + 1), dtype=np.uint32)
            qd = np.frombuffer((ctypes.string_at(q, int(qo[n])) if qo[n] else b'') + bytes(32), dtype=np.uint8)
            ud = np.frombuffer((ctypes.string_at(up, int(uo[n])) if uo[n] else b'') + bytes(32), dtype=np.uint8)
            return self._put(relay_oracle.relay_batch(qd, qo, ud, uo, tcp=bool(flags & 1)), out, out_cap, out_off, out_len, status, n)
        except Exception as e:
            self.error = e
            return -3


def run_pair(native, twin, kind, seed, flush_every, relay=True):
    """The same sessions, chunking, flush seeds and relays through both hubs: outputs and counters must be identical."""
    snap, dom, rec, sessions = workload(kind, seed)
    streams = [session_stream(qs, 0x0A000000 + j, 1024 + j) for j, qs in enumerate(sessions)]
    events = chunk_events(streams, seed)
    got, want = [drive(h, streams, events, flush_every, 50 + seed) for h in (native, twin)]
    assert got[1] == want[1]
    assert outputs(native, got[0]) == outputs(twin, want[0])
    if relay and want[1]:
        mix = want[1][::-1]
        ups = [upstream_for(p, i) for i, (p, _) in enumerate(mix)]
        for h, (sids, _) in ((native, got), (twin, want)):
            h.relay([p for p, _ in mix], ups, [sids[j] for _, j in mix])
        assert outputs(native, got[0]) == outputs(twin, want[0])
    sn, st = native.stats(), twin.stats()
    assert {k: sn[k] for k in st} == st
    return sn, got[0], want[0]


@pytest.mark.parametrize('kind,seed', [('fuzz', 3), ('big', 4)])
def test_native_hub_on_cpu_matches_python(hub_lib, kind, seed):
    from oracle_lib import Oracle
    snap, dom, rec, _ = workload(kind, seed)
    orc = Oracle(dom, '', rec, snapshot=snap)
    eng = CpuEngine(hub_lib, orc)
    native = NativeTcpHub(eng, max_batch=48, lib=hub_lib)
    twin = TcpHub(orc, max_batch=48, out_cap=native.stats()['answer_capacity'], relayer=relay_oracle.RelayOracle())
    st, _, _ = run_pair(native, twin, kind, seed, 41)
    assert eng.error is None and st['messages'] > 100
    # batches split at max_batch; qidx_base runs over the batches of each flush
    assert max(n for _, n in eng.calls) == 48
    base = 0
    for q, n in eng.calls:
        assert q in (0, base)
        base = q + n


def test_native_hub_on_cpu_edges_and_failures(hub_lib):
    from oracle_lib import Oracle
    orc = Oracle('foo.com', '', False, snapshot=big_zone())
    eng = CpuEngine(hub_lib, orc)
    native = NativeTcpHub(eng, lib=hub_lib)
    assert edge_cases(native, orc) == edge_cases(TcpHub(orc), orc)
    assert eng.error is None
    # a failed batch loses its queries only: the next batch of the same flush, and the next flush, are answered
    eng2 = CpuEngine(hub_lib, orc)
    eng2.fail = {5}
    hubs = (NativeTcpHub(eng2, max_batch=4, lib=hub_lib), TcpHub(FailAt(orc, 4), max_batch=4))
    q = [synth.make_query('hosta.foo.com', 'A', qid=i) for i in range(10)]
    outs = []
    for h in hubs:
        s = h.open()
        h.feed(s, hello() + b''.join(TcpFramer.frame(x) for x in q))
        h.flush(1)
        h.feed(s, TcpFramer.frame(q[0]))
        h.flush(2)
        outs.append((h.output(s)[0], h.stats()))
    assert outs[0][0] == outs[1][0] and len(TcpFramer().feed(outs[0][0][4:])) == 7
    assert {k: outs[0][1][k] for k in outs[1][1]} == outs[1][1] and outs[1][1]['failed'] == 4
    assert hubs[0].last_rc == 0 and eng2.error is None
    assert eng2.calls == [(0, 4), (4, 4), (8, 2), (0, 1)]


class FailAt(object):
    """A resolver whose batch starting at query index `qidx` fails"""

    def __init__(self, orc, qidx):
        self.orc, self.qidx = orc, qidx

    def resolve_batch(self, data, off, seed=0, qidx_base=0, tcp=False):
        if qidx_base == self.qidx:
            raise RuntimeError('batch failed')
        return self.orc.resolve_batch(data, off, seed=seed, qidx_base=qidx_base, tcp=tcp)


def test_native_hub_argument_errors(hub_lib):
    """A null hub (the real library, no device needed), an unknown session, a closed one, a session past eof."""
    from binder_b200._lib import BinderError, lib
    L = lib()
    err = ctypes.c_int(0)
    assert not L.bb_tcp_hub_create(None, 16, ctypes.byref(err)) and err.value == -1
    sid, p, n, cl = ctypes.c_uint32(0), ctypes.c_void_p(), ctypes.c_size_t(0), ctypes.c_int(0)
    for rc in (L.bb_tcp_hub_open(None, ctypes.byref(sid)), L.bb_tcp_hub_feed(None, 1, b'x', 1), L.bb_tcp_hub_eof(None, 1),
               L.bb_tcp_hub_flush(None, 0, None), L.bb_tcp_hub_output(None, 1, ctypes.byref(p), ctypes.byref(n), ctypes.byref(cl)),
               L.bb_tcp_hub_consume(None, 1, 0), L.bb_tcp_hub_close(None, 1), L.bb_tcp_hub_relay(None, None, None, None, None, None, 0),
               L.bb_tcp_hub_peer(None, 1, ctypes.byref(sid), ctypes.byref(sid))):
        assert rc == -1
    assert L.bb_tcp_hub_stat(None, 0) == 0
    L.bb_tcp_hub_destroy(None)
    from oracle_lib import Oracle
    hub = NativeTcpHub(CpuEngine(hub_lib, Oracle('foo.com', '', False, snapshot=big_zone())), lib=hub_lib)
    s = hub.open()
    assert s != 0 and hub.feed(s, hello())
    for bad in (0, s + 1, 12345):                # never opened
        for call in (lambda: hub.feed(bad, b'x'), lambda: hub.eof(bad), lambda: hub.output(bad), lambda: hub.consume(bad, 0),
                     lambda: hub.close(bad), lambda: hub.peer(bad)):
            with pytest.raises(BinderError) as ei:
                call()
            assert ei.value.code == -1
    with pytest.raises(BinderError):
        hub.consume(s, 5)                        # more than there is to write
    hub.eof(s)
    with pytest.raises(BinderError):
        hub.feed(s, b'\x00\x05')                 # nothing arrives past eof
    hub.close(s)
    for call in (lambda: hub.feed(s, b'x'), lambda: hub.output(s), lambda: hub.close(s), lambda: hub.eof(s)):
        with pytest.raises(BinderError):
            call()
    assert hub.open() == s + 1                   # ids are not reused
    bad_off = np.array([0, 5, 3], dtype=np.uint32)
    assert hub_lib.bb_tcp_hub_relay(hub._h, b'x' * 8, bad_off.ctypes.data, b'x' * 8, bad_off.ctypes.data,
                                    np.zeros(2, np.uint32).ctypes.data, 2) == -1
    hub.destroy()
    with pytest.raises(BinderError):
        hub.open()


def test_hub_symbols_are_exported():
    hdr = open(os.path.join(ROOT, 'include', 'binder_b200.h')).read()
    names = {n for n in _lib.SYMBOLS if n.startswith('bb_tcp_hub_')}
    assert len(names) == 12 and all(n + '(' in hdr for n in names)
    L = ctypes.CDLL(_lib.SO_PATH)
    assert all(hasattr(L, n) for n in names)


# ---- a fake balancer over socketpairs --------------------------------------------------------------------------------
def loopback(hub, orc, n_sess=8):
    """8 AF_UNIX sessions as the balancer opens them: INBOUND_TCP, then dnspython-built queries; the host side feeds the
    hub, flushes, writes each session's output back.  The answers must decode and match the oracle's."""
    names = [('big.foo.com', 'A'), ('_http._tcp.big.foo.com', 'SRV'), ('hosta.foo.com', 'A'), ('nope.foo.com', 'A')]
    pairs = [socket.socketpair() for _ in range(n_sess)]
    try:
        sids, sent = [], []
        for j, (bal, host) in enumerate(pairs):
            bal.settimeout(5)
            host.setblocking(False)
            qs = [dns.message.make_query(*names[(j + k) % len(names)], id=100 * j + k).to_wire() for k in range(1 + j % 3)]
            bal.sendall(hello(0x7F000001, 5000 + j) + b''.join(TcpFramer.frame(q) for q in qs))
            bal.shutdown(socket.SHUT_WR)
            sids.append(hub.open())
            sent.append(qs)
        open_ = set(range(n_sess))
        for _ in range(100):
            if not open_:
                break
            for j in list(open_):
                host = pairs[j][1]
                try:
                    chunk = host.recv(7)                 # small reads: frames and prefixes arrive split
                except BlockingIOError:
                    chunk = None
                if chunk:
                    hub.feed(sids[j], chunk)
                elif chunk == b'':
                    hub.eof(sids[j])
            hub.flush(77)
            for j in list(open_):
                out, closable = hub.output(sids[j])
                if out:
                    pairs[j][1].setblocking(True)
                    pairs[j][1].sendall(out)
                    pairs[j][1].setblocking(False)
                    hub.consume(sids[j], len(out))
                if hub.output(sids[j])[1]:
                    pairs[j][1].close()
                    hub.close(sids[j])
                    open_.discard(j)
        assert not open_
        for j, (bal, _) in enumerate(pairs):
            buf = b''
            while True:
                c = bal.recv(1 << 16)
                if not c:
                    break
                buf += c
            assert buf[:4] == OK
            got = TcpFramer().feed(buf[4:])
            assert len(got) == len(sent[j])
            for q, a in zip(sent[j], got):
                assert dns.message.from_wire(a).id == dns.message.from_wire(q).id
                data, off = synth.pack_batch([q])
                out, ooff, olen, _, _ = orc.resolve_batch(data, off, tcp=True)
                got_s, want_s = H.decode_semantic(a), H.decode_semantic(bytes(out[:olen[0]]))
                # the service shuffle keys on the position in the batch: the same records, maybe in another order
                assert got_s[0] == want_s[0] and got_s[4] == want_s[4] and not got_s[4]['tc']
                assert [sorted(x) for x in got_s[1:4]] == [sorted(x) for x in want_s[1:4]]
    finally:
        for a, b in pairs:
            a.close()
            b.close()


def test_loopback_python_hub():
    from oracle_lib import Oracle
    orc = Oracle('foo.com', '', False, snapshot=big_zone())
    loopback(TcpHub(orc), orc)


# ---- GPU: the native hub on an Engine against the Python hub on the oracle -------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('ordered', [False, True])
@pytest.mark.parametrize('kind,seed', [('fuzz', 10), ('fuzz', 11), ('big', 12)])
def test_gpu_hub_matches_python(ordered, kind, seed):
    from binder_b200.engine import Engine
    from oracle_lib import Oracle
    snap, dom, rec, _ = workload(kind, seed)
    eng = Engine(dom, '', rec, snapshot=snap, max_batch=1 << 14, ordered=ordered)
    orc = Oracle(dom, '', rec, snapshot=snap)
    for max_batch, every in ((4096, 1000), (40, 29)):           # one flush; many flushes of several batches each
        native = NativeTcpHub(eng, max_batch=max_batch)
        twin = TcpHub(orc, max_batch=max_batch, out_cap=native.stats()['answer_capacity'], relayer=relay_oracle.RelayOracle())
        st, _, _ = run_pair(native, twin, kind, seed, every)
        assert st['failed'] == 0 and native.last_rc == 0 and (st['relayed'] > 0) == rec
        native.destroy()


@pytest.mark.gpu
def test_gpu_hub_capacity_failure_loses_only_its_batch():
    """64 answers of the 1,300-child service (65,516 bytes each) do not fit a batch's 1 MB of answer room: that batch is
    lost and counted; the short answers of the next batch and of the next flush arrive."""
    from binder_b200.engine import Engine
    from oracle_lib import Oracle
    snap = big_zone()
    eng = Engine('foo.com', snapshot=snap, max_batch=256)
    native = NativeTcpHub(eng, max_batch=64)
    cap = native.stats()['answer_capacity']
    assert cap == 1 << 20
    twin = TcpHub(Oracle('foo.com', '', False, snapshot=snap), max_batch=64, out_cap=cap)
    huge = [synth.make_query('_http._tcp.huge.foo.com', 'SRV', qid=i) for i in range(64)]
    small = [synth.make_query('hosta.foo.com', 'A', qid=1000 + i) for i in range(30)]
    for h in (native, twin):
        a, b = h.open(), h.open()
        h.feed(a, hello() + b''.join(TcpFramer.frame(q) for q in huge))
        h.feed(b, hello() + b''.join(TcpFramer.frame(q) for q in small))
        h.flush(3)
        h.feed(a, TcpFramer.frame(huge[0]))
        h.flush(4)
    assert native.last_rc == 0
    assert native.output(1) == twin.output(1) and native.output(2) == twin.output(2)
    assert len(TcpFramer().feed(native.output(2)[0][4:])) == 30 and len(TcpFramer().feed(native.output(1)[0][4:])) == 1
    sn, st = native.stats(), twin.stats()
    assert {k: sn[k] for k in st} == st and st['failed'] == 64 and st['answered'] == 31


@pytest.mark.gpu
def test_gpu_loopback():
    from binder_b200.engine import Engine
    from oracle_lib import Oracle
    snap = big_zone()
    loopback(NativeTcpHub(Engine('foo.com', snapshot=snap, max_batch=4096)), Oracle('foo.com', '', False, snapshot=snap))
