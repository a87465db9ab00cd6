"""Forwarded misses answered end to end over UDP loopback: a dc1 Server whose misses go to binder_b200.recursion.Recursion,
which asks a second Server (the dc2 upstream) and relays its responses into dc1's replies; dnspython is the client.
The CPU variant injects the oracle (resolve and relay), the GPU variant Engines."""
import socket

import dns.message
import dns.query
import dns.rcode
import dns.rdatatype
import pytest

import helpers as H
from binder_b200.recursion import Recursion
from binder_b200.server import createServer


def _zone(dc, n):
    ent = [('/com/foo/%s' % dc, None)]
    ent += [('/com/foo/%s/h%d' % (dc, i), {'type': 'host', 'host': {'address': '10.%d.0.%d' % (2 if dc == 'dc2' else 1, i)}})
            for i in range(n)]
    return H.snapshot(ent)


def _run(kind):
    if kind == 'oracle':
        from oracle_lib import Oracle
        from relay_oracle import RelayOracle
        make = lambda snap, rec: Oracle('foo.com', '', rec, snapshot=snap)      # noqa: E731
        relayer = RelayOracle()
    else:
        from binder_b200.engine import Engine
        make = lambda snap, rec: Engine('foo.com', '', rec, snapshot=snap, max_batch=4096)   # noqa: E731
        relayer = Engine('foo.com', '', True, max_batch=4096)
    silent = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)          # an upstream that never answers
    silent.bind(('127.0.0.1', 0))
    dc2 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc2', 20), False), 'host': '127.0.0.1', 'port': 0}).start()
    rec = Recursion(relayer, 'foo.com', {'dc2': [('127.0.0.1', dc2.port)], 'dc3': [('127.0.0.1', silent.getsockname()[1])],
                                         'dc4': ['10.99.0.1']}, my_addrs=['10.99.0.1'], timeout=0.5)
    dc1 = createServer({'dnsDomain': 'foo.com', 'resolver': make(_zone('dc1', 20), True), 'recursion': rec,
                        'host': '127.0.0.1', 'port': 0}).start()
    try:
        def ask(name, edns=-1, rd=True):
            q = dns.message.make_query(name, 'A', use_edns=edns)
            if not rd:
                q.flags &= ~dns.flags.RD
            return dns.query.udp(q, '127.0.0.1', port=dc1.port, timeout=5)
        for i in range(20):                                   # dc2's names, relayed through dc1
            r = ask('h%d.dc2.foo.com' % i, edns=0 if i % 2 else -1)
            assert r.rcode() == dns.rcode.NOERROR and not r.flags & dns.flags.RA and r.flags & dns.flags.AA
            assert [(rr.name.to_text(), rr.rdtype, rr[0].address) for rr in r.answer] == \
                [('h%d.dc2.foo.com.' % i, dns.rdatatype.A, '10.2.0.%d' % i)]
            assert (r.edns >= 0) == bool(i % 2)
        r = ask('h3.dc1.foo.com')                             # a hit never leaves dc1
        assert r.rcode() == dns.rcode.NOERROR and r.answer[0][0].address == '10.1.0.3'
        r = ask('nope.dc2.foo.com')                           # dc2 refuses its own miss: no answers upstream -> REFUSED
        assert r.rcode() == dns.rcode.REFUSED and not r.answer
        for name in ('h1.dc3.foo.com', 'h1.dc4.foo.com', 'h1.nodc.foo.com'):   # silent upstream (timeout), own address, unknown dc
            r = ask(name)
            assert r.rcode() == dns.rcode.REFUSED and not r.answer, name
        assert rec.counters['relayed'] >= 24 and rec.counters['upstream_answers'] >= 21
    finally:
        dc1.stop()
        dc2.stop()
        rec.close()
        silent.close()


def test_loopback_relay_cpu():
    _run('oracle')


@pytest.mark.gpu
def test_loopback_relay_gpu():
    _run('gpu')
