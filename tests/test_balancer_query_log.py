"""Query log of the balancer sessions on the CPU (DESIGN.md section 15): bb_backend and bb_tcp_hub (csrc/balancer_frames.cpp,
balancer_relay.cpp, balancer_tcp.cpp, balancer_query_log.cpp) linked against the engine stand-ins of tests/native, whose
bb_log_batch (query_log_stubs.cpp) calls back into this file and renders the records with the restatement
(tests/query_log_ref.py), packed in reverse index order as the arrival packing may.  Every record is checked against the frame or answer at its position, against the Python sessions
(balancer.Backend / TcpHub over the same restatement) and through QueryLog.write_records; log failures, capacity retries,
logging off, and the host code under AddressSanitizer and UndefinedBehaviorSanitizer (tests/native/fuzz_query_log.cpp)."""
import ctypes
import io
import json
import os
import random
import shutil
import struct
import subprocess

import numpy as np
import pytest

import fuzzgen
import query_log_ref as R
import relay_oracle
import relaygen as G
import test_balancer_tcp as TB
from binder_b200 import _lib, balancer, synth
from binder_b200.query_log import QueryLog
from binder_b200.server import TcpFramer
from test_balancer_frames import frame, split_out

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32,
                       ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p)
_STUB = {}


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    """the session sources with the engine stand-ins (tcp_hub_stubs.cpp, backend_stubs.cpp, query_log_stubs.cpp), as one
    host-only library"""
    if 'L' not in _STUB:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        so = str(tmp_path_factory.mktemp('qlog') / 'libsessions_cpu.so')
        csrc = os.path.join(ROOT, 'binder_b200', 'csrc')
        subprocess.check_call([cxx, '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'),
                               '-o', so] + [os.path.join(csrc, f) for f in ('balancer_frames.cpp', 'balancer_relay.cpp', 'balancer_tcp.cpp',
                                                               'balancer_query_log.cpp')] +
                              [os.path.join(ROOT, 'tests', 'native', f) for f in ('tcp_hub_stubs.cpp', 'backend_stubs.cpp', 'query_log_stubs.cpp')])
        L = ctypes.CDLL(so)
        for name, (res, args) in _lib.SYMBOLS.items():
            if name.startswith(('bb_tcp_hub_', 'bb_backend_', 'bb_query_log_')):
                getattr(L, name).restype = res
                getattr(L, name).argtypes = args
        L.bb_stub_set.argtypes = [TB.RESOLVE, TB.RELAY, ctypes.c_uint32, ctypes.c_uint32]
        L.bb_stub_set_log.argtypes = [LOG]
        _STUB['L'] = L
    return _STUB['L']


def _restated(out, out_off, out_len, status, dom):
    """A result set's records by the restatement -> [(head, body)] (b'', b'' without a record)"""
    return [(h, b) for h, b, _ in R.log_set(out, out_off, out_len, status, dom)]


class LogEngine(TB.CpuEngine):
    """CpuEngine with bb_log_batch: the restatement's records, packed in reverse index order.  log_calls counts the calls;
    fail_calls (0-based) fail with BB_ERR_CUDA; capacity_calls report BB_ERR_CAPACITY (with the bytes needed at
    log_off[n], as the kernel leaves them) whatever the room."""

    def __init__(self, L, oracle, dom, fail_calls=(), capacity_calls=(), **kw):
        TB.CpuEngine.__init__(self, L, oracle, **kw)
        self.dom, self.fail_calls, self.capacity_calls, self.log_calls, self.caps = dom, set(fail_calls), set(capacity_calls), 0, []
        self._log_cb = LOG(self._log)
        L.bb_stub_set_log(self._log_cb)

    def _log(self, resp, resp_bytes, out_off, out_len, status, n, log, log_cap, log_off, log_len, head_len):
        try:
            k, self.log_calls = self.log_calls, self.log_calls + 1
            self.caps.append(log_cap)
            if k in self.fail_calls:
                return -3
            oo = np.array(TB._arr(ctypes.c_uint32, out_off, n), dtype=np.uint32)
            ol = np.array(TB._arr(ctypes.c_uint16, out_len, n), dtype=np.uint16)
            st = np.array(TB._arr(ctypes.c_uint8, status, n), dtype=np.uint8)
            out = ctypes.string_at(resp, resp_bytes) if resp_bytes else b''
            recs = _restated(out, oo, ol, st, self.dom)
            lo, ll, hl = TB._arr(ctypes.c_uint32, log_off, n + 1), TB._arr(ctypes.c_uint32, log_len, n), TB._arr(ctypes.c_uint16, head_len, n)
            total = sum(len(h) + len(b) for h, b in recs)
            lo[n] = total
            if total > log_cap or k in self.capacity_calls:
                return -5
            pos = 0
            for i in reversed(range(n)):
                rec = recs[i][0] + recs[i][1]
                ctypes.memmove(log + pos, rec, len(rec))
                lo[i], ll[i], hl[i] = pos, len(rec), len(recs[i][0]) if rec else 0
                pos += len(rec)
            return 0
        except Exception as e:
            self.error = e
            return -3


class RefLog(object):
    """A Python session's resolver and relayer: the oracles' answers, the restatement's records (packed in order)."""

    def __init__(self, oracle, dom):
        self.oracle, self.dom = oracle, dom

    def resolve_batch(self, *a, **kw):
        return self.oracle.resolve_batch(*a, **kw)

    def relay_batch(self, *a, **kw):
        return relay_oracle.relay_batch(*a, **kw)

    def log_batch(self, out, out_off, out_len, status):
        recs = _restated(out, out_off, out_len, status, self.dom)
        ll = np.array([len(h) + len(b) for h, b in recs], dtype=np.uint32)
        off = np.zeros(len(recs) + 1, dtype=np.uint32)
        np.cumsum(ll, out=off[1:])
        log = np.frombuffer(b''.join(h + b for h, b in recs), dtype=np.uint8)
        return log, off, ll, np.array([len(h) if b else 0 for h, b in recs], dtype=np.uint16)


def rows(rec):
    """QueryLogRecords -> [(head, body, req_id, ip, port, session)]"""
    log = rec.log.tobytes()
    res = []
    for i in range(len(rec.log_len)):
        o, ll, hl = int(rec.log_off[i]), int(rec.log_len[i]), int(rec.head_len[i])
        res.append((log[o:o + hl], log[o + hl:o + ll], int(rec.req_id[i]), int(rec.client_ip[i]), int(rec.client_port[i]),
                    None if rec.session is None else int(rec.session[i])))
    return res


def expect(answers, dom):
    """[(ip, port, session, response bytes)] of the answers sent, in order -> rows() they must have"""
    res = []
    for ip, port, sid, r in answers:
        x = R.record(r, dom)
        h, b = (x[0], x[1]) if x else (b'', b'')
        res.append((h, b, struct.unpack('>H', r[:2])[0], ip, port, sid))
    return res


def udp_answers(out):
    return [(ip, port, None, p) for ip, port, p in split_out(out)[1]]


def fuzz_stream(seed, n=700):
    """fuzzgen queries (misses, malformed drops) as INBOUND_UDP frames from distinct clients, HELLO / HEARTBEAT between"""
    snap, info = fuzzgen.gen_zone(seed, n_top=30)
    pkts = fuzzgen.gen_queries(seed, info, n=n) + fuzzgen.malformed_packets()[:8]
    random.Random(seed).shuffle(pkts)
    rng = random.Random(seed + 1)
    parts = [struct.pack('<I', balancer.CLIENT_HELLO)]
    for i, p in enumerate(pkts):
        parts.append(frame(p, 0x0A000000 + i, 1024 + (i * 7) % 60000))
        if rng.random() < 0.03:
            parts.append(struct.pack('<I', rng.choice((balancer.CLIENT_HEARTBEAT, balancer.CLIENT_HELLO))))
    return snap, info['dns_domain'], b''.join(parts)


def chunks(stream, seed):
    rng = random.Random(seed)
    pos = 0
    while pos < len(stream):
        step = rng.choice((1, 3, 17, 200, 1500, 9000))
        yield stream[pos:pos + step]
        pos += step


# ---- UDP backend -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('seed,max_batch', [(1, 7), (2, 40), (3, 4096)])
def test_backend_feed_records_match_frames(lib, seed, max_batch):
    from oracle_lib import Oracle
    snap, dom, stream = fuzz_stream(seed)
    orc = Oracle(dom, '', True, snapshot=snap)
    eng = LogEngine(lib, orc, dom)
    nb = balancer.NativeBackend(eng, max_batch=max_batch, lib=lib)
    nb.set_query_log(True)
    n_rec = n_ans = 0
    for k, c in enumerate(chunks(stream, seed)):
        out, misses = nb.feed(c, seed=50 + k)
        rec = nb.query_log(0)
        assert rows(rec) == expect(udp_answers(out), dom) and rec.lost == 0 and rec.session is None
        n_rec += len(rec.log_len)
        n_ans += len(udp_answers(out))
    st = nb.stats()
    assert eng.error is None and n_rec == n_ans == st['answered'] == st['records'] > 300 and st['lost'] == 0 and st['missed'] > 0
    assert nb.query_log(1).log_len.size == 0                 # no relay yet
    nb.close()


def relay_pairs(seed, n=300):
    """relaygen relays plus misses whose lookup failed (empty upstream: REFUSED)"""
    rng = random.Random(seed)
    pairs = G.gen_relays(seed, n) + [(G.relay_case(rng, 'empty')[0], b'') for _ in range(20)]
    rng.shuffle(pairs)
    return [q for q, _ in pairs], [u for _, u in pairs], [(0x7F000001 + i, 2000 + i) for i in range(len(pairs))]


@pytest.mark.parametrize('max_batch', [9, 4096])
def test_backend_relay_records_and_python_model(lib, max_batch):
    from oracle_lib import Oracle
    dom = 'example.com'
    orc = Oracle(dom, '', True, snapshot=fuzzgen.gen_zone(4, n_top=10)[0])
    eng = LogEngine(lib, orc, dom)
    nb = balancer.NativeBackend(eng, max_batch=max_batch, lib=lib)
    py = balancer.Backend(RefLog(orc, dom), max_batch=max_batch)
    qs, us, dst = relay_pairs(max_batch)
    for s in (nb, py):
        s.set_query_log(True)
    out = nb.relay(qs, us, dst)
    assert out == py.relay(qs, us, dst) and nb.last_rc == 0
    rec = nb.query_log(1)
    assert rows(rec) == expect(udp_answers(out), dom) == rows(py.query_log(1))
    assert len(rec.log_len) == nb.stats()['relayed'] == nb.stats()['records'] > 200
    assert {k: v for k, v in nb.stats().items() if k in py.counters} == py.counters
    # a feed leaves the relay's records alone
    _, _, stream = fuzz_stream(5, n=50)
    fo = nb.feed(stream, seed=100)[0]
    assert rows(nb.query_log(0)) == expect(udp_answers(fo), dom) and len(udp_answers(fo)) > 0
    assert rows(nb.query_log(1)) == rows(rec)
    assert eng.error is None


def test_feed_records_outgrow_the_buffer_and_python_lines(lib):
    """A feed of 6,000 frames, records well past the session's first 1 MB of log buffer, in small batches; the Python
    session gives the same records, and QueryLog the same lines."""
    from oracle_lib import Oracle
    snap, dom, rec = TB.big_zone(), 'foo.com', False
    orc = Oracle(dom, '', rec, snapshot=snap)
    pool = [q for q in TB.big_zone_batch() if len(q) < 200][:40]
    frames = b''.join(frame(pool[i % len(pool)], 0xC0A80000 + i, 5000 + i % 1000) for i in range(6000))
    eng = LogEngine(lib, orc, dom)
    nb = balancer.NativeBackend(eng, max_batch=6000, lib=lib)
    py = balancer.Backend(RefLog(orc, dom), shuffle_seed=6)
    for s in (nb, py):
        s.set_query_log(True)
    out = nb.feed(frames, seed=7)[0]
    assert out == py.feed(frames)
    a, b = nb.query_log(0), py.query_log(0)
    assert rows(a) == rows(b) == expect(udp_answers(out), dom)
    assert int(a.log_len.sum()) > 1 << 20 and eng.log_calls == 2 and eng.caps[1] > eng.caps[0]      # grown once, then all there
    lines = []
    for r in (a, b):
        s = io.BytesIO()
        QueryLog(s, hostname='h', pid=7).write_records(r, 1000.0 + np.arange(len(r.log_len)) * 1e-3, sent=1003.5)
        lines.append(s.getvalue())
    assert lines[0] == lines[1]
    first = json.loads(lines[0].split(b'\n')[0])
    assert list(first)[:6] == ['name', 'hostname', 'pid', 'req_id', 'client', 'port'] and first['client'] == '192.168.0.0'
    assert first['port'] == '5000/ipv4' and first['latency'] == 3500 and first['level'] == 40 and first['time'] == '1970-01-01T00:16:43.500Z'


def test_log_failures_keep_frames(lib):
    """Capacity once: the batch is grown into and all records are there.  A hard failure: that batch's answers still go
    out, and count as lost; the return code and the frames are those of a session with logging off."""
    from oracle_lib import Oracle
    snap, dom, stream = fuzz_stream(8, n=400)
    orc = Oracle(dom, '', True, snapshot=snap)
    runs = {}
    for key, fail, cap in (('off', (), ()), ('cap', (), (1,)), ('fail', (2,), ())):
        eng = LogEngine(lib, orc, dom, fail_calls=fail, capacity_calls=cap)
        nb = balancer.NativeBackend(eng, max_batch=50, lib=lib)
        nb.set_query_log(key != 'off')
        out, misses = nb.feed(stream, seed=3)
        runs[key] = (out, misses, nb.stats(), nb.query_log(0), eng.log_calls, nb.last_rc)
        assert eng.error is None
    off, cap, fail = runs['off'], runs['cap'], runs['fail']
    assert off[4] == 0 and off[3].log_len.size == 0 and off[2]['records'] == 0
    assert cap[0] == fail[0] == off[0] and cap[1] == fail[1] == off[1]
    strip = lambda st: {k: v for k, v in st.items() if k not in ('records', 'lost')}
    assert strip(cap[2]) == strip(fail[2]) == strip(off[2])
    answered = udp_answers(off[0])
    assert rows(cap[3]) == expect(answered, dom) and cap[3].lost == 0 and cap[2]['lost'] == 0
    assert fail[3].lost == fail[2]['lost'] > 0 and len(fail[3].log_len) + fail[3].lost == len(answered) == fail[2]['records'] + fail[2]['lost']
    # the lost batch is the third with an answer: the others' records are those of the frames around it
    got = rows(fail[3])
    want = expect(answered, dom)
    assert got == [w for w in want if w in got] and len(set(map(tuple, got))) > 0


# ---- TCP hub -----------------------------------------------------------------------------------------------------------
def hub_answers(out, sid, ip, port):
    return [(ip, port, sid, a) for a in TcpFramer().feed(out[4:])]


@pytest.mark.parametrize('kind,seed,max_batch', [('fuzz', 1, 13), ('fuzz', 2, 4096), ('big', 3, 24)])
def test_hub_records_match_answers_and_python(lib, kind, seed, max_batch):
    from oracle_lib import Oracle
    snap, dom, rec, sessions = TB.workload(kind, seed, n_sess=30)
    orc = Oracle(dom, '', rec, snapshot=snap)
    eng = LogEngine(lib, orc, dom)
    native = balancer.NativeTcpHub(eng, max_batch=max_batch, lib=lib)
    twin = balancer.TcpHub(RefLog(orc, dom), max_batch=max_batch, out_cap=native.stats()['answer_capacity'])
    streams = [TB.session_stream(q, 0x0A000100 + j, 7000 + j) for j, q in enumerate(sessions)]
    events = TB.chunk_events(streams, seed)
    recs = ([], [])
    for h, acc in ((native, recs[0]), (twin, recs[1])):
        h.set_query_log(True)
        sids = [h.open() for _ in streams]
        bad = [h.open(), h.open()]                           # a session that is no TCP session, one that breaks later
        assert not h.feed(bad[0], struct.pack('<I', balancer.CLIENT_HELLO))
        assert not h.feed(bad[1], TB.hello(0x0B000001, 9) + TcpFramer.frame(sessions[0][0]) + b'\x00\x00')
        for k, (j, chunk) in enumerate(events):
            h.feed(sids[j], chunk)
            if (k + 1) % 17 == 0:
                misses = h.flush(40 + k)
                acc.append(rows(h.query_log(0)))
        misses = h.flush(999)
        acc.append(rows(h.query_log(0)))
    assert recs[0] == recs[1]
    flat = [r for batch in recs[0] for r in batch]
    # per session, in order, the answers written to it (INBOUND_TCP_OK first)
    for j, s in enumerate(sids):
        assert [r for r in flat if r[5] == s] == expect(hub_answers(native.output(s)[0], s, 0x0A000100 + j, 7000 + j), dom)
    assert [r for r in flat if r[5] == bad[1]] == expect(hub_answers(native.output(bad[1])[0], bad[1], 0x0B000001, 9), dom)
    st = native.stats()
    assert len(flat) == st['answered'] == st['records'] > 20 and st['lost'] == 0 and eng.error is None
    if misses:
        # a session closed between the flush and the relay: its replies are not sent and have no record
        gone = misses[0][1]
        ups = [TB.upstream_for(p, i) for i, (p, _) in enumerate(misses)]
        for h in (native, twin):
            h.close(gone)
            h.relay([p for p, _ in misses], ups, [s for _, s in misses])
        a, b = rows(native.query_log(1)), rows(twin.query_log(1))
        assert a == b and all(r[5] != gone for r in a) and len(a) == native.stats()['relayed']
        assert rows(native.query_log(0)) == recs[0][-1]          # the flush's records stay
        assert {k: v for k, v in native.stats().items() if k in twin.stats()} == twin.stats()


def test_hub_relay_records_and_lines(lib):
    from oracle_lib import Oracle
    dom = 'example.com'
    orc = Oracle(dom, '', True, snapshot=fuzzgen.gen_zone(4, n_top=10)[0])
    qs, us, _ = relay_pairs(11, n=120)
    hubs = []
    for h in (balancer.NativeTcpHub(LogEngine(lib, orc, dom), max_batch=16, lib=lib), balancer.TcpHub(RefLog(orc, dom), max_batch=16)):
        h.set_query_log(True)
        sids = [h.open() for _ in range(5)]
        for j, s in enumerate(sids):
            h.feed(s, TB.hello(0x7F000001, 40000 + j))
        h.flush(1)
        h.relay(qs, us, [sids[i % 5] for i in range(len(qs))])
        hubs.append(h)
    a, b = hubs[0].query_log(1), hubs[1].query_log(1)
    assert rows(a) == rows(b) and len(a.log_len) > 100
    outs = [io.BytesIO(), io.BytesIO()]
    for o, r in zip(outs, (a, b)):
        QueryLog(o, hostname='h', pid=1).write_records(r, 5.0, sent=5.25)
    assert outs[0].getvalue() == outs[1].getvalue()
    lines = outs[0].getvalue().split(b'\n')[:-1]
    assert len(lines) == int((a.log_len > 0).sum())
    for ln, r in zip(lines, [r for r in rows(a) if r[0] or r[1]]):
        d = json.loads(ln)
        assert d['client'] == '127.0.0.1' and d['port'] == '%d/ipv4' % r[4] and d['req_id'] == r[2] and d['latency'] == 250


def test_hub_log_failure_counts_lost(lib):
    from oracle_lib import Oracle
    snap = TB.big_zone()
    orc = Oracle('foo.com', '', False, snapshot=snap)
    q = [synth.make_query('hosta.foo.com', 'A', qid=i) for i in range(30)]
    res = []
    for fail in ((), (1,)):
        eng = LogEngine(lib, orc, 'foo.com', fail_calls=fail)
        h = balancer.NativeTcpHub(eng, max_batch=10, lib=lib)
        h.set_query_log(bool(fail))
        s = h.open()
        h.feed(s, TB.hello() + b''.join(TcpFramer.frame(x) for x in q))
        h.flush(2)
        res.append((h.output(s)[0], h.stats(), h.query_log(0), h.last_rc))
    assert res[0][0] == res[1][0] and res[0][3] == res[1][3] == 0
    assert res[1][2].lost == 10 == res[1][1]['lost'] and len(res[1][2].log_len) == 20 == res[1][1]['records']
    assert [int(x) for x in res[1][2].req_id] == list(range(10)) + list(range(20, 30))


def test_query_log_switch_and_args(lib):
    from oracle_lib import Oracle
    orc = Oracle('foo.com', '', False, snapshot=TB.big_zone())
    eng = LogEngine(lib, orc, 'foo.com')
    nb = balancer.NativeBackend(eng, lib=lib)
    pkt = synth.make_query('hosta.foo.com', 'A', qid=5)
    nb.set_query_log(True)
    nb.feed(frame(pkt, 1, 2), seed=1)
    assert len(nb.query_log(0).log_len) == 1
    nb.set_query_log(False)                                  # off: no records, no calls
    calls = eng.log_calls
    nb.feed(frame(pkt, 1, 2), seed=1)
    assert len(nb.query_log(0).log_len) == 0 and eng.log_calls == calls
    r = ctypes.create_string_buffer(128)
    assert lib.bb_query_log_backend(nb._h, 2, r) == -1 and lib.bb_query_log_backend(None, 0, r) == -1
    assert lib.bb_query_log_backend_enable(None, 1) == -1 and lib.bb_query_log_tcp_hub_enable(None, 1) == -1
    assert lib.bb_query_log_tcp_hub(None, 0, r) == -1


def test_sanitizer_clean(tmp_path):
    cxx = shutil.which('g++')
    if not cxx:
        pytest.skip('no g++')
    exe = str(tmp_path / 'fuzz_query_log')
    csrc = os.path.join(ROOT, 'binder_b200', 'csrc')
    cmd = [cxx, '-std=c++17', '-O1', '-g', '-fsanitize=address,undefined', '-fno-omit-frame-pointer', '-Wall', '-Werror',
           '-I', os.path.join(ROOT, 'include'), '-I', csrc, '-o', exe, os.path.join(ROOT, 'tests', 'native', 'fuzz_query_log.cpp')] + \
          [os.path.join(csrc, f) for f in ('balancer_frames.cpp', 'balancer_relay.cpp', 'balancer_tcp.cpp', 'balancer_query_log.cpp')]
    b = subprocess.run(cmd, capture_output=True, text=True)
    if b.returncode != 0 and 'sanitize' in b.stderr:
        pytest.skip('toolchain without sanitizer runtimes')
    assert b.returncode == 0, b.stderr[-2000:]
    p = subprocess.run([exe, '300'], capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and p.stdout.strip().endswith('OK') and 'runtime error' not in p.stderr, (p.stdout[-500:], p.stderr[-3000:])
