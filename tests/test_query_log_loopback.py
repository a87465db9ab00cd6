"""The query log end to end over loopback: a Server with options['query_log'] answers a client over UDP and TCP, and a
miss over UDP is forwarded by Recursion to a second Server and relayed back.  Every line the server writes is one JSON
object with bunyan's fields in bunyan's order, and its query, edns, rcode, answers and additional equal the
restatement's (tests/query_log_ref.py) for the response bytes the client received.  The CPU variant uses oracle
stand-ins, with log_batch run by the device source on the CPU (tests/native/emu_log.cpp); the GPU variant Engines, and
its lines equal the CPU variant's but for latency, level, time and the client's port."""
import io
import json
import socket
import struct

import dns.message
import numpy as np
import pytest

import helpers as H
import query_log_ref as L
from binder_b200.recursion import Recursion
from binder_b200.server import createServer
from test_query_log import emu_exe, emu_log

FIELDS = ['name', 'hostname', 'pid', 'req_id', 'client', 'port', 'query', 'edns', 'level', 'rcode', 'answers', 'additional',
          'latency', 'timers', 'msg', 'time', 'v']
DOM = 'foo.com'


def _zone(dc, n):
    ent = [('/com/foo/%s' % dc, None)]
    ent += [('/com/foo/%s/h%d' % (dc, i), {'type': 'host', 'host': {'address': '10.%d.0.%d' % (2 if dc == 'dc2' else 1, i)}})
            for i in range(n)]
    ent += [('/com/foo/%s/svc' % dc, {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80}}),
            ('/com/foo/%s/svc/i1' % dc, {'type': 'load_balancer', 'load_balancer': {'address': '10.9.0.1', 'ports': [8080]}})]
    return H.snapshot(ent)


class EmuLog(object):
    """A CPU resolver stand-in with log_batch: `inner` answers, the device source on the CPU renders the records."""

    def __init__(self, inner, exe, tmp_path):
        self.inner, self.exe, self.tmp = inner, exe, tmp_path

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def log_batch(self, out, out_off, out_len, status):
        n = len(status)
        recs = emu_log(self.exe, (np.asarray(out, np.uint8), np.asarray(out_off, np.uint32)[:n], np.asarray(out_len, np.uint16)[:n],
                                  np.asarray(status, np.uint8)), DOM, self.tmp)
        lens = np.array([len(h) + len(b) for h, b, _ in recs], np.uint32)
        off = np.zeros(n + 1, np.uint32)
        np.cumsum(lens, out=off[1:])
        return (np.frombuffer(b''.join(h + b for h, b, _ in recs), np.uint8), off, lens,
                np.array([len(h) for h, _, _ in recs], np.uint16))


def _tcp_ask(port, wire):
    with socket.create_connection(('127.0.0.1', port), timeout=5) as s:
        s.sendall(struct.pack('>H', len(wire)) + wire)
        buf = b''
        while len(buf) < 2 or len(buf) < 2 + struct.unpack('>H', buf[:2])[0]:
            chunk = s.recv(65536)
            assert chunk
            buf += chunk
        return buf[2:]


def run_loopback(kind, tmp_path_factory=None, tmp_path=None):
    """-> ([(transport, response bytes)], [log line dicts])"""
    if kind == 'oracle':
        from oracle_lib import Oracle
        from relay_oracle import RelayOracle
        exe = emu_exe(tmp_path_factory)
        make = lambda snap, rec: EmuLog(Oracle(DOM, '', rec, snapshot=snap), exe, tmp_path)      # noqa: E731
        relay = EmuLog(RelayOracle(), exe, tmp_path)
    else:
        from binder_b200.engine import Engine
        make = lambda snap, rec: Engine(DOM, '', rec, snapshot=snap, max_batch=4096)                # noqa: E731
        relay = Engine(DOM, '', True, max_batch=4096)
    sink = io.BytesIO()
    dc2 = createServer({'dnsDomain': DOM, 'resolver': make(_zone('dc2', 10), False), 'host': '127.0.0.1', 'port': 0}).start()
    rec = Recursion(relay, DOM, {'dc2': [('127.0.0.1', dc2.port)]}, timeout=2.0)
    dc1 = createServer({'dnsDomain': DOM, 'resolver': make(_zone('dc1', 10), True), 'recursion': rec, 'host': '127.0.0.1',
                        'port': 0, 'query_log': sink}).start()
    got = []
    try:
        qid = 100
        for transport, name, t, edns in [('udp', 'h1.dc1.foo.com', 'A', -1), ('udp', '_http._tcp.svc.dc1.foo.com', 'SRV', 0),
                                         ('tcp', 'h2.dc1.foo.com', 'A', 0), ('tcp', 'svc.dc1.foo.com', 'A', -1),
                                         ('udp', 'h3.dc2.foo.com', 'A', 0), ('udp', 'h4.dc2.foo.com', 'A', -1),
                                         ('udp', 'nope.dc1.foo.com', 'A', -1)]:
            q = dns.message.make_query(name, t, use_edns=edns)
            q.id = qid
            qid += 1
            wire = q.to_wire()
            if transport == 'udp':
                with socket.socket(socket.AF_INET, socket.SOCK_DGRAM) as s:
                    s.settimeout(5)
                    s.sendto(wire, ('127.0.0.1', dc1.port))
                    got.append(('udp', s.recv(65536)))
            else:
                got.append(('tcp', _tcp_ask(dc1.port, wire)))
    finally:
        dc1.stop()
        dc2.stop()
        rec.close()
    lines = sink.getvalue().splitlines()
    return got, [json.loads(x, object_pairs_hook=lambda kv: kv) for x in lines], lines


def check_lines(got, lines):
    by_id = {}
    for pairs in lines:
        assert [k for k, _ in pairs] == FIELDS
        d = dict(pairs)
        assert d['name'] == 'binder' and d['msg'] == 'DNS query' and d['v'] == 0 and d['timers'] == []
        assert d['client'] == '127.0.0.1' and d['port'].endswith('/ipv4') and d['level'] in (30, 40)
        assert isinstance(d['latency'], int) and d['time'].endswith('Z')
        by_id[d['req_id']] = d
    assert len(by_id) == len(got) == len(lines)
    for _, wire in got:
        d = by_id[struct.unpack('>H', wire[:2])[0]]
        head, body, _ = L.record(wire, DOM)
        want = dict(json.loads('{' + head.decode() + ',' + body.decode() + '}'))
        for k in ('query', 'edns', 'rcode', 'answers', 'additional'):
            got_v = d[k]
            if k == 'query':
                got_v = dict(got_v)
            assert json.dumps(got_v) == json.dumps(want[k]), (k, got_v, want[k])


def normalised(lines):
    """Lines without what differs between runs: latency, level, time and the client's ephemeral port."""
    return sorted(json.dumps([(k, v.split('/')[1] if k == 'port' else v) for k, v in p if k not in ('latency', 'level', 'time')])
                  for p in lines)


def test_query_log_loopback_cpu(tmp_path_factory, tmp_path):
    got, lines, _ = run_loopback('oracle', tmp_path_factory, tmp_path)
    check_lines(got, lines)
    recs = [dict(p) for p in lines]
    assert any(a.startswith('SRV ') for d in recs for a in d['answers'])
    assert any(dict(d['query'])['name'] == 'h3.dc2.foo.com' and d['answers'] == ['A 10.2.0.3'] for d in recs)     # relayed


@pytest.mark.gpu
def test_query_log_loopback_gpu(tmp_path_factory, tmp_path):
    got, lines, _ = run_loopback('gpu')
    check_lines(got, lines)
    _, cpu_lines, _ = run_loopback('oracle', tmp_path_factory, tmp_path)
    assert normalised(lines) == normalised(cpu_lines)
