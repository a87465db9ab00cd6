"""Query log of the balancer sessions on the GPU (DESIGN.md section 15): NativeBackend and NativeTcpHub on an Engine in
both packings, with logging on.  Every record is checked against the restatement (tests/query_log_ref.py) of the answer
at its position and against the Python session on the same engine; frames and outputs are byte-identical with logging
off; a fake balancer over socketpairs writes the lines through QueryLog."""
import io
import json
import socket
import struct

import pytest

import test_balancer_tcp as TB
from binder_b200 import balancer, synth
from binder_b200.query_log import QueryLog
from test_balancer_frames import frame
from test_balancer_query_log import expect, fuzz_stream, hub_answers, relay_pairs, rows, udp_answers

pytestmark = pytest.mark.gpu
BUNYAN = ['name', 'hostname', 'pid', 'req_id', 'client', 'port', 'query', 'edns', 'level', 'rcode', 'answers', 'additional',
          'latency', 'timers', 'msg', 'time', 'v']


def engine(dom, snap, ordered, recursion=True, max_batch=1 << 14):
    from binder_b200.engine import Engine
    return Engine(dom, '', recursion, snapshot=snap, max_batch=max_batch, ordered=ordered)


def feed_all(nb, stream, step, seed):
    outs, recs = [], []
    for k, pos in enumerate(range(0, len(stream), step)):
        outs.append(nb.feed(stream[pos:pos + step], seed=seed + k)[0])
        recs.append(rows(nb.query_log(0)))
    return outs, recs


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_backend_feed_and_relay_records(ordered):
    snap, dom, stream = fuzz_stream(21, n=3000)
    eng = engine(dom, snap, ordered)
    on, off = balancer.NativeBackend(eng, max_batch=500), balancer.NativeBackend(eng, max_batch=500)
    on.set_query_log(True)
    got, want = feed_all(on, stream, 7001, 30), feed_all(off, stream, 7001, 30)
    assert got[0] == want[0] and all(r == [] for r in want[1])            # logging off: the same frames, no records
    for out, rec in zip(*got):
        assert rec == expect(udp_answers(out), dom)
    st = on.stats()
    assert st['records'] == st['answered'] > 2000 and st['lost'] == 0 and st['failed'] == 0
    # the Python session on the same engine gives the same answer frames and records (the native session parses at most
    # 64 control frames per batch, so its HELLO / HEARTBEAT replies may sit between batches)
    one, py = balancer.NativeBackend(eng, max_batch=1 << 14), balancer.Backend(eng, shuffle_seed=40)
    for s in (one, py):
        s.set_query_log(True)
    out = one.feed(stream, seed=41)[0]
    assert udp_answers(out) == udp_answers(py.feed(stream))
    assert rows(one.query_log(0)) == rows(py.query_log(0)) == expect(udp_answers(out), dom)
    # relays, split into batches, through the native session and the Python one
    qs, us, dst = relay_pairs(22, n=2000)
    for mb in (300, 4096):
        nb, py = balancer.NativeBackend(eng, max_batch=mb), balancer.Backend(eng, max_batch=mb)
        for s in (nb, py):
            s.set_query_log(True)
        r_out = nb.relay(qs, us, dst)
        assert r_out == py.relay(qs, us, dst) and nb.last_rc == 0
        assert rows(nb.query_log(1)) == rows(py.query_log(1)) == expect(udp_answers(r_out), dom)
        assert len(nb.query_log(1).log_len) == nb.stats()['relayed'] > 1500
        nb.close()


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_backend_records_outgrow_the_log_buffer(ordered):
    """16,384 frames in one feed of 4,096-query batches: the records pass the session's first 1 MB of log buffer."""
    snap = TB.big_zone()
    eng = engine('foo.com', snap, ordered, recursion=False)
    pool = [q for q in TB.big_zone_batch() if len(q) < 200]
    stream = b''.join(frame(pool[i % len(pool)], 0x0A000000 + i, 1024 + i % 50000) for i in range(16384))
    on, off = balancer.NativeBackend(eng, max_batch=4096), balancer.NativeBackend(eng, max_batch=4096)
    on.set_query_log(True)
    out = on.feed(stream, seed=3)[0]
    assert out == off.feed(stream, seed=3)[0]
    rec = on.query_log(0)
    assert int(rec.log_len.sum()) > 1 << 20 and rows(rec) == expect(udp_answers(out), 'foo.com')
    assert on.stats()['records'] == len(udp_answers(out)) and rec.lost == 0


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_hub_records(ordered):
    """Fuzzed sessions and the big services (answers up to 65,516 bytes, records around 80 KB), flushed in batches, one
    session closed before the relay; the Python hub on the same engine gives the same records."""
    for kind, seed, rec_on in (('fuzz', 31, True), ('big', 32, False)):
        snap, dom, rec, sessions = TB.workload(kind, seed, n_sess=40)
        eng = engine(dom, snap, ordered, recursion=rec)
        streams = [TB.session_stream(q, 0x0A000100 + j, 7000 + j) for j, q in enumerate(sessions)]
        events = TB.chunk_events(streams, seed)
        native, quiet = balancer.NativeTcpHub(eng, max_batch=12), balancer.NativeTcpHub(eng, max_batch=12)
        twin = balancer.TcpHub(eng, max_batch=12, out_cap=native.stats()['answer_capacity'])
        got = {}
        for h in (native, quiet, twin):
            h.set_query_log(h is not quiet)
            sids = [h.open() for _ in streams]
            recs, misses = [], []
            for k, (j, chunk) in enumerate(events):
                h.feed(sids[j], chunk)
                if (k + 1) % 23 == 0:
                    misses += h.flush(60 + k)
                    recs.append(rows(h.query_log(0)))
            misses += h.flush(9)
            recs.append(rows(h.query_log(0)))
            if misses:
                h.close(misses[0][1])
                h.relay([p for p, _ in misses], [TB.upstream_for(p, i) for i, (p, _) in enumerate(misses)], [s for _, s in misses])
                recs.append(rows(h.query_log(1)))
            got[h] = (recs, [h.output(s)[0] if s != (misses[0][1] if misses else 0) else b'' for s in sids])
        assert got[native] == got[twin] and got[native][1] == got[quiet][1]
        assert all(r == [] for r in got[quiet][0])
        flat = [r for batch in got[native][0] for r in batch]
        for j, (s, out) in enumerate(zip(sids, got[native][1])):
            if out:
                assert [r for r in flat if r[5] == s] == expect(hub_answers(out, s, 0x0A000100 + j, 7000 + j), dom)
        st = native.stats()
        assert st['records'] == len(flat) == st['answered'] + st['relayed'] > 50 and st['lost'] == 0 and (st['relayed'] > 0) == rec_on
        if kind == 'big':
            assert max(len(r[1]) for r in flat) > 40000


def test_gpu_fake_balancer_writes_lines():
    """A balancer over a socketpair sends INBOUND_UDP frames; the backend answers them and writes one line per answer."""
    snap = TB.big_zone()
    eng = engine('foo.com', snap, True, recursion=False)
    nb = balancer.NativeBackend(eng, max_batch=256)
    nb.set_query_log(True)
    sink = io.BytesIO()
    qlog = QueryLog(sink, hostname='test', pid=42)
    bal, be = socket.socketpair()
    try:
        qs = [synth.make_query('hosta.foo.com', 'A', qid=i) for i in range(600)]
        clients = [(0xC0A80001 + i, 30000 + i) for i in range(600)]
        bal.sendall(struct.pack('<I', balancer.CLIENT_HELLO) + b''.join(frame(q, *c) for q, c in zip(qs, clients)))
        bal.shutdown(socket.SHUT_WR)
        got = b''
        while True:
            chunk = be.recv(65536)
            if not chunk:
                break
            t = 1000.0
            out, _ = nb.feed(chunk, seed=1)
            be.sendall(out)
            qlog.write_records(nb.query_log(0), t, sent=t + 0.0025)
        be.shutdown(socket.SHUT_WR)
        while True:
            chunk = bal.recv(65536)
            if not chunk:
                break
            got += chunk
    finally:
        bal.close()
        be.close()
    answers = udp_answers(got[4:])
    lines = sink.getvalue().split(b'\n')[:-1]
    assert len(lines) == len(answers) == 600 == qlog.lines
    for ln, (ip, port, _, resp) in zip(lines, answers):
        d = json.loads(ln)
        assert list(d) == BUNYAN and d['req_id'] == struct.unpack('>H', resp[:2])[0] and d['latency'] == 2
        assert d['client'] == '%d.%d.%d.%d' % (ip >> 24, (ip >> 16) & 255, (ip >> 8) & 255, ip & 255) and d['port'] == '%d/ipv4' % port
        assert d['query'] == {'name': 'hosta.foo.com', 'type': 'A'} and d['rcode'] == 0
