"""Forwarded misses end to end over UDP loopback through binder_b200.forward.GpuRecursion: a dc1 Server whose misses go
to GpuRecursion, which forwards them to a second Server (the dc2 upstream), matches the responses and relays them;
dnspython is the client.  The same questions asked through binder_b200.recursion.Recursion give the same answers, and a
silent upstream gives REFUSED after the timeout.  The CPU variant uses oracle stand-ins (resolve, forward, match,
relay), the GPU variant Engines."""
import socket

import dns.message
import dns.query
import dns.rcode
import pytest

import helpers as H
from binder_b200.forward import GpuRecursion
from binder_b200.recursion import Recursion
from binder_b200.server import createServer


def _zone(dc, n):
    ent = [('/com/foo/%s' % dc, None)]
    ent += [('/com/foo/%s/h%d' % (dc, i), {'type': 'host', 'host': {'address': '10.%d.0.%d' % (2 if dc == 'dc2' else 1, i)}})
            for i in range(n)]
    return H.snapshot(ent)


QUESTIONS = [('h%d.dc2.foo.com' % i, 'A', i % 2) for i in range(12)] + [
    ('h3.dc1.foo.com', 'A', 0),            # a hit never leaves dc1
    ('nope.dc2.foo.com', 'A', 1),          # dc2 refuses its own miss: REFUSED
    ('_http._tcp.h1.dc2.foo.com', 'SRV', 0),
    ('5.0.2.10.in-addr.arpa', 'PTR', 1),   # PTR asks every datacenter
    ('h1.dc3.foo.com', 'A', 0),            # silent upstream: REFUSED after the timeout
    ('h1.dc4.foo.com', 'A', 0),            # its only upstream is this host
    ('h1.nodc.foo.com', 'A', 1),           # unknown datacenter
]


def _answers(kind, rec_cls):
    if kind == 'oracle':
        from oracle_lib import Oracle
        from forward_oracle import ForwardOracle
        from relay_oracle import RelayOracle
        make = lambda snap, rec: Oracle('foo.com', '', rec, snapshot=snap)      # noqa: E731
        resolver = ForwardOracle() if rec_cls is GpuRecursion else RelayOracle()
    else:
        from binder_b200.engine import Engine
        make = lambda snap, rec: Engine('foo.com', '', rec, snapshot=snap, max_batch=4096)   # noqa: E731
        resolver = Engine('foo.com', '', True, max_batch=4096)
    silent = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    silent.bind(('127.0.0.1', 0))
    dc2 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc2', 20), False), 'host': '127.0.0.1', 'port': 0}).start()
    rec = rec_cls(resolver, 'foo.com', {'dc2': [('127.0.0.1', dc2.port)], 'dc3': [('127.0.0.1', silent.getsockname()[1])],
                                        'dc4': ['10.99.0.1']}, my_addrs=['10.99.0.1'], timeout=0.5)
    dc1 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc1', 20), True), 'recursion': rec,
                        'host': '127.0.0.1', 'port': 0}).start()
    out = []
    try:
        for name, t, edns in QUESTIONS:
            q = dns.message.make_query(name, t, use_edns=0 if edns else -1)
            r = dns.query.udp(q, '127.0.0.1', port=dc1.port, timeout=5)
            out.append((r.rcode(), r.flags, sorted(rr.to_text() for rr in r.answer), r.edns))
        counters = dict(rec.counters)
    finally:
        dc1.stop()
        dc2.stop()
        rec.close()
        silent.close()
    return out, counters


def _run(kind):
    got, counters = _answers(kind, GpuRecursion)
    want, _ = _answers(kind, Recursion)
    assert got == want
    rc = {name: g[0] for (name, _, _), g in zip(QUESTIONS, got)}
    assert all(rc['h%d.dc2.foo.com' % i] == dns.rcode.NOERROR for i in range(12))
    assert got[0][2] == ['h0.dc2.foo.com. 30 IN A 10.2.0.0']
    assert got[15][2] == ['5.0.2.10.in-addr.arpa. 30 IN PTR h5.dc2.foo.com.']
    for name in ('nope.dc2.foo.com', 'h1.dc3.foo.com', 'h1.dc4.foo.com', 'h1.nodc.foo.com'):
        assert rc[name] == dns.rcode.REFUSED, name
    assert counters['upstream_answers'] >= 14 and counters['relayed'] >= 17


def test_gpu_recursion_loopback_cpu():
    _run('oracle')


@pytest.mark.gpu
def test_gpu_recursion_loopback_gpu():
    _run('gpu')
