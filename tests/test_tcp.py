"""DNS over TCP (SURVEY.md section 8f row 4; mname listenTcp, lib/server.js:643-652): two-byte length framing
and the aggregation window on the host side (binder_b200/server.py), BB_BATCH_TCP on the resolve side (no UDP
size limit: a response is truncated only beyond 65,535 bytes)."""
import random
import socket
import struct

import dns.message
import dns.query
import dns.rdatatype
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth
from binder_b200.server import TcpFramer, createServer


def big_zone(n_big=200, n_huge=1300):
    ent = [('/com/foo', None),
           ('/com/foo/hosta', {'type': 'host', 'host': {'address': '192.168.0.1'}}),
           ('/com/foo/big', {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80}}),
           ('/com/foo/huge', {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80, 'ttl': 9}})]
    for i in range(n_big):
        ent.append(('/com/foo/big/lb%03d' % i, {'type': 'load_balancer', 'load_balancer': {'address': '10.2.%d.%d' % (i >> 8, i & 255)}}))
    for i in range(n_huge):
        ent.append(('/com/foo/huge/backend-%04d' % i, {'type': 'rr_host', 'rr_host': {'address': '10.3.%d.%d' % (i >> 8, i & 255), 'ports': [8080, 8081]}}))
    return H.snapshot(ent)


def test_framer_reassembles_any_chunking():
    msgs = [bytes([i]) * n for i, n in enumerate([1, 17, 512, 513, 4000, 65535, 2])]
    stream = b''.join(TcpFramer.frame(m) for m in msgs)
    rng = random.Random(3)
    for trial in range(20):
        fr, got, pos = TcpFramer(), [], 0
        while pos < len(stream):
            step = rng.choice([1, 2, 3, 7, 100, 1000, 70000])
            got += fr.feed(stream[pos:pos + step]); pos += step
        assert got == msgs and not fr.bad and len(fr.buf) == 0
    fr = TcpFramer()
    assert fr.feed(b'\x00\x00rest') == [] and fr.bad


def test_oracle_tcp_lifts_the_size_limit():
    orc = H.make_impl('oracle', 'foo.com', big_zone())
    opts = H.ref_options(big_zone(), 'foo.com')
    pk = [synth.make_query('_http._tcp.big.foo.com', 'SRV'), synth.make_query('big.foo.com', 'A'),
          synth.make_query('_http._tcp.huge.foo.com', 'SRV'), synth.make_query('hosta.foo.com', 'A', edns=4096)]
    data, off = synth.pack_batch(pk)
    out, ooff, olen, st, miss = orc.resolve_batch(data, off, seed=3, tcp=True)
    u_out, u_off, u_len, _, _ = orc.resolve_batch(data, off, seed=3)
    wires = [bytes(out[ooff[i]:ooff[i] + olen[i]]) for i in range(4)]
    # 200 SRV + 200 additional A: everything fits over TCP, next to nothing over UDP
    rcode, ans, auth, add, f = H.decode_semantic(wires[0])
    ref = H.ref_semantic(opts, pk[0], seed=3, qidx=0)
    assert not f['tc'] and (ans, auth, add) == ref[2:] and len(ans) == 200 and len(add) == 200
    assert H.decode_semantic(bytes(u_out[u_off[0]:u_off[0] + u_len[0]]))[4]['tc'] and u_len[0] <= 512
    assert len(H.decode_semantic(wires[1])[1]) == 200 and not H.decode_semantic(wires[1])[4]['tc']
    # 2,600 SRV records do not fit 65,535 bytes: truncated even on TCP, longest prefix kept
    rcode, ans, auth, add, f = H.decode_semantic(wires[2])
    ref = H.ref_semantic(opts, pk[2], seed=3, qidx=2)
    assert f['tc'] and 60000 < olen[2] <= 65535 and ans == ref[2][:len(ans)] and not add
    assert wires[3] == bytes(u_out[u_off[3]:u_off[3] + u_len[3]])          # small answers are the same bytes


def _tcp_exchange(port, queries):
    """All queries framed in ONE write on one connection; responses read back in order."""
    s = socket.create_connection(('127.0.0.1', port), timeout=5)
    s.sendall(b''.join(TcpFramer.frame(q) for q in queries))
    fr, got = TcpFramer(), []
    while len(got) < len(queries):
        chunk = s.recv(1 << 20)
        assert chunk, 'connection closed early'
        got += fr.feed(chunk)
    s.close()
    return got


def _serve_and_check(kind):
    snap = big_zone()
    impl = H.make_impl(kind, 'foo.com', snap)
    direct = H.make_impl('oracle', 'foo.com', snap)
    srv = createServer({'dnsDomain': 'foo.com', 'resolver': impl, 'host': '127.0.0.1', 'port': 0, 'shuffle_seed': 40}).start()
    try:
        # dnspython over TCP: the large answer arrives whole
        r = dns.query.tcp(dns.message.make_query('big.foo.com', 'A'), '127.0.0.1', port=srv.port, timeout=5)
        assert r.rcode() == 0 and sum(len(x) for x in r.answer) == 200
        u = socket.socket(socket.AF_INET, socket.SOCK_DGRAM); u.settimeout(5)
        u.sendto(synth.make_query('big.foo.com', 'A'), ('127.0.0.1', srv.port))
        ur = u.recv(4096); u.close()
        assert ur[2] & 0x02 and len(ur) <= 512                             # over UDP: truncated
        # 60 pipelined queries in one write: answered in order, one aggregated batch or a few
        qs = [synth.make_query('hosta.foo.com' if i % 3 else '_http._tcp.big.foo.com', 'A' if i % 3 else 'SRV', qid=1000 + i) for i in range(60)]
        b0 = srv.counters['tcp_batches']
        got = _tcp_exchange(srv.port, qs)
        assert [struct.unpack('>H', g[:2])[0] for g in got] == list(range(1000, 1060))
        assert srv.counters['tcp_batches'] - b0 <= 10 and srv.counters['tcp_queries'] >= 61
        for q, g in zip(qs, got):
            if q[-4:-2] == b'\x00\x01':                               # A hosta: deterministic bytes
                data, off = synth.pack_batch([q])
                out, ooff, olen, _, _ = direct.resolve_batch(data, off, tcp=True)
                assert g == bytes(out[:olen[0]])
            else:
                assert len(g) > 10000 and not (g[2] & 0x02)
        # several connections at once, closed by the client after writing
        socks = [socket.create_connection(('127.0.0.1', srv.port), timeout=5) for _ in range(8)]
        for i, s in enumerate(socks):
            s.sendall(TcpFramer.frame(synth.make_query('hosta.foo.com', 'A', qid=i)))
            s.shutdown(socket.SHUT_WR)
        for i, s in enumerate(socks):
            buf = b''
            while True:
                c = s.recv(65536)
                if not c:
                    break
                buf += c
            (m,) = TcpFramer().feed(buf)
            assert struct.unpack('>H', m[:2])[0] == i and m[3] & 0xF == 0
            s.close()
    finally:
        srv.stop()


def test_tcp_server_cpu_oracle():
    _serve_and_check('oracle')


@pytest.mark.gpu
def test_tcp_server_gpu():
    _serve_and_check('gpu')


def big_zone_batch():
    """700 queries on big_zone(): the 200- and 1,300-child services (answers of up to 65,535 bytes over TCP) among
    short answers, misses and NOTIMP."""
    rng = random.Random(8)
    pk = []
    for i in range(700):
        r = rng.random()
        if r < 0.25:
            pk.append(synth.make_query('_http._tcp.big.foo.com', 'SRV', qid=i, edns=rng.choice([None, 4096])))
        elif r < 0.4:
            pk.append(synth.make_query('big.foo.com', 'A', qid=i))
        elif r < 0.42:
            pk.append(synth.make_query('_http._tcp.huge.foo.com', 'SRV', qid=i))
        elif r < 0.45:
            pk.append(synth.make_query('huge.foo.com', 'A', qid=i))
        else:
            pk.append(synth.make_query(rng.choice(['hosta.foo.com', 'nope.foo.com', 'lb007.big.foo.com']), rng.choice(['A', 'SRV', 'AAAA']), qid=i))
    return pk


@pytest.mark.gpu
@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_tcp_batches_are_bit_exact(ordered):
    from test_gpu_parity import assert_same
    snap = big_zone()
    gpu = H.make_impl('gpu', 'foo.com', snap, ordered=ordered)
    orc = H.make_impl('oracle', 'foo.com', snap)
    data, off = synth.pack_batch(big_zone_batch())
    assert_same(gpu, orc, data, off, seed=77, tcp=True)
    assert_same(gpu, orc, data, off, seed=77)                   # and the same engine still applies the UDP limits


@pytest.mark.gpu
@pytest.mark.parametrize('seed', range(4))
def test_gpu_tcp_fuzz(seed):
    from test_gpu_parity import assert_same
    snap, info = fuzzgen.gen_zone(seed + 400, n_top=40)
    gpu = H.make_impl('gpu', info['dns_domain'], snap, recursion=seed % 2 == 0, ordered=seed % 2 == 1)
    orc = H.make_impl('oracle', info['dns_domain'], snap, recursion=seed % 2 == 0)
    data, off = synth.pack_batch(fuzzgen.gen_queries(seed, info, n=2500))
    assert_same(gpu, orc, data, off, seed=seed, tcp=True)
