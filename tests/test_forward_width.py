"""The recursion forward and match at the full width of their ABI (DESIGN.md section 14), on the CPU: the device source
(binder_b200/csrc/forward_device.cuh through tests/native/emu_forward.cpp) bit-exact against the forward oracle with
16 datacenters and 64 upstreams, contended answers, and QNAME labels that contain a '.' (routed on the dotted name, as
lib/recursion.js routes them); GpuRecursion's collection windows cut at the resolver's batch limit.  The generators here
also feed tests/test_gpu_forward_width.py."""
import random
import socket
import struct
import subprocess
import threading
import time

import numpy as np
import pytest

import forward_oracle as O
import forward_ref as R
import forwardgen as G
from binder_b200 import synth
from binder_b200.engine import ip_u32
from binder_b200.forward import GpuRecursion
from test_forward_emu import emu, emu_exe

REGION = 'foo.com'
# 16 datacenters, the filter's limit: names of 1 and 63 bytes, a prefix / suffix family (w, we, web, eb), case twins
WIDE_DCS = ['w', 'we', 'web', 'eb', 'WEB', 'Web', 'x' * 63, 'b', 'db', 'c', 'h1', 'a-b', 'x_y', 'dc13', 'nope', 'z' * 62 + 'q']
# datacenters without an upstream: 7, and 14 next to 15 that has some (14 & 7 = 6 has upstreams, 15 & 7 = 7 has none)
HOLES = (7, 14)


def wide_upstreams(holes=HOLES, seed=0):
    """64 upstreams (the table's limit) round-robin over the datacenters outside `holes`: ports 0, 53 and 65535,
    0.0.0.0 and 255.255.255.255, and one IP on several ports in different datacenters (10.1.2.3:53 in two of them)."""
    rng = random.Random(seed)
    dcs = [k for k in range(len(WIDE_DCS)) if k not in holes]
    special = [('0.0.0.0', 0), ('255.255.255.255', 65535), ('10.1.2.3', 53), ('10.1.2.3', 5353), ('10.1.2.3', 0),
               ('10.1.2.3', 65535), ('0.0.0.0', 53), ('255.255.255.255', 0)]
    ups = []
    for i in range(64):
        if i < len(special):
            ip, port = special[i]
        elif i == 63:
            ip, port = '10.1.2.3', 53
        else:
            ip = '%d.%d.%d.%d' % (rng.randrange(1, 255), rng.randrange(256), rng.randrange(256), rng.randrange(1, 255))
            port = rng.choice([53, 5353, rng.randrange(1, 65535)])
        ups.append((ip, port, dcs[i % len(dcs)]))
    return ups


def wide_misses(seed=0, n_random=600):
    """Misses for the wide filter: every datacenter name and near names (prefixes, suffixes, case variants), SRV
    prefixes, 255-byte names ending in a datacenter label, PTR and undecodable packets."""
    rng = random.Random(seed)
    tops = WIDE_DCS + ['WEb', 'wE', 'weeb', 'xweb', 'e', 'x' * 62, 'zz', 'nopE', 'dc1', 'z' * 62 + 'Q']
    pkts = []
    for i, top in enumerate(tops):
        for pre in ('h%d.' % i, '', '_http._tcp.h%d.' % i, 'a.b.c.'):
            t = 'SRV' if pre.startswith('_') else 'A'
            pkts.append(synth.make_query(pre + top + '.' + REGION, t, qid=i, edns=1200 if i % 2 else None))
    for i in range(n_random):
        top = rng.choice(tops)
        pkts.append(synth.make_query('h%d.%s.%s' % (i, top, REGION), rng.choice(['A', 'SRV', 'AAAA']), qid=rng.randrange(65536),
                                     rd=rng.random() < 0.9, edns=rng.choice([None, 512, 4096]), opcode=rng.choice([0, 0, 0, 2])))
    for i, top in enumerate(WIDE_DCS):                      # 255-byte names
        tail = [top.encode(), b'foo', b'com']
        used = sum(1 + len(l) for l in tail) + 1
        head = []
        while used + 64 <= 255:
            head.append(b'a' * 63)
            used += 64
        if used < 255:
            head.append(b'b' * (255 - used - 1))
        pkts.append(synth.make_query(None, 'A', qid=i, labels=head + tail))
    pkts += [synth.make_query('%d.%d.0.10.in-addr.arpa' % (i, i), 'PTR', qid=i) for i in range(16)]
    good = synth.make_query('h1.web.foo.com', 'A', qid=3)
    pkts += [good[:11], b'', good[:2] + b'\x81\x00' + good[4:], synth.make_query('h1.web.foo.com', 'A', qclass=3)]
    rng.shuffle(pkts)
    return pkts


def route_pool(ups, seed=1):
    """route -> [packets with that route] under the wide filter and `ups`, for the route distributions."""
    rng = random.Random(seed)
    cand = wide_misses(seed, n_random=400)
    for k, dc in enumerate(WIDE_DCS):
        cand += [synth.make_query('q%d.%s.%s' % (i, dc, REGION), rng.choice(['A', 'SRV']), qid=i) for i in range(8)]
    cand += [synth.make_query('%d.1.0.10.in-addr.arpa' % i, 'PTR', qid=i, edns=512) for i in range(8)]
    routes, _ = R.forward(REGION, WIDE_DCS, ups, cand, 1)
    pool = {}
    for p, r in zip(cand, routes):
        pool.setdefault(r, []).append(p)
    return pool


DISTRIBUTIONS = ('route15', 'all_routes_per_tile', 'blocks', 'round_robin')


def route_batch(pool, kind, n, seed):
    """n misses whose routes follow `kind`: all on route 15 (one run); every route present in every 128-miss tile;
    single-route blocks of 100-1,000 misses that cross tile boundaries; routes round-robin."""
    rng = random.Random(seed)
    routes = sorted(pool)
    if kind == 'route15':
        seq = [15] * n
    elif kind == 'all_routes_per_tile':
        seq = []
        while len(seq) < n:
            tile = routes + [rng.choice(routes) for _ in range(128 - len(routes))]
            rng.shuffle(tile)
            seq += tile
        seq = seq[:n]
    elif kind == 'blocks':
        seq = []
        while len(seq) < n:
            seq += [rng.choice(routes)] * rng.randint(100, 1000)
        seq = seq[:n]
    else:
        seq = [routes[j % len(routes)] for j in range(n)]
    return [rng.choice(pool[r]) for r in seq]


KEYS = [0, 2 ** 64 - 1, 1 << 32, 0xFFFFFFFF, 0x8F1BBCDCCA62C1D6]


def answer(upq, i):
    """A response to upstream query upq (its ID, opcode and question) with one A record whose address is i: answers
    with different i are different datagrams."""
    hdr = upq[:2] + bytes([0x84 | (upq[2] & 0x78), 0x00]) + b'\x00\x01\x00\x01\x00\x00\x00\x00'
    return hdr + upq[12:] + b'\xc0\x0c\x00\x01\x00\x01\x00\x00\x00\x3c\x00\x04' + struct.pack('>I', i)


NEAR = 0xFFFF0000                       # A-record addresses of the near-misses: never a winner


def contended(ups, routes, msgs, key, rng, most=64, near=True):
    """The datagrams of one exchange in arrival order: every forwarded miss gets 1..most valid answers from upstreams of
    its route (a PTR miss one from each of the 64), shuffled together; with `near`, before a miss's first valid answer
    come the datagrams that must lose: its ID from a wrong port, its question re-cased, QR = 0, the ID a foreign key
    gives it, and an ID that decodes to a miss >= n."""
    n = len(msgs)
    ev = []
    for j, (rt, m) in enumerate(zip(routes, msgs)):
        if not m or rt == R.R_NONE:
            continue
        valid = [(a, p) for a, p, d in ups if rt == R.R_PTR or d == rt]
        srcs = valid if rt == R.R_PTR else [rng.choice(valid) for _ in range(rng.randint(1, most))]
        ts = [rng.random() for _ in srcs]
        ev += [(t, answer(m, i), s) for i, (t, s) in enumerate(zip(ts, srcs))]
        if not near:
            continue
        first, s = min(ts), rng.choice(valid)
        a = answer(m, NEAR)
        taken = {(x, p) for x, p, _ in ups}
        port = next(p for p in range(s[1] + 1, s[1] + 70000) if (s[0], p & 0xFFFF) not in taken) & 0xFFFF
        bad = [(a, (s[0], port)), (a[:2] + bytes([a[2] & 0x7F]) + a[3:], s)]
        k = next((i for i in range(13, 12 + len(m) - 16) if 65 <= (a[i] | 0x20) <= 122), None)
        if k is not None:
            bad.append((a[:k] + bytes([a[k] ^ 0x20]) + a[k + 1:], s))
        fid = O.fwd_id(key ^ 0x5DEECE66D, j)
        if O.fwd_id(key, fid, inverse=True) >= n:
            bad.append((struct.pack('>H', fid) + a[2:], s))
        if n < 65536:
            bad.append((struct.pack('>H', O.fwd_id(key, rng.randrange(n, 65536))) + a[2:], s))
        ev += [(rng.uniform(0, first), b, src) for b, src in bad]
    ev.sort(key=lambda e: e[0])
    return [(b, s) for _, b, s in ev]


def responses(ups, routes, msgs, rng, key):
    """forwardgen.responses with its wrong-port answers kept to 16 bits (the wide table has an upstream on port 65535)."""
    return [(b, (a, p & 0xFFFF)) for b, (a, p) in G.responses(ups, routes, msgs, rng, key)]


def msgs_by_miss(fwd, n):
    """Upstream query of each miss from a forward call's (uq, uq_off, order)."""
    uq, uq_off, order = fwd[0], fwd[1], fwd[2]
    out = [b''] * n
    for k, j in enumerate(order):
        out[int(j)] = bytes(uq[uq_off[k]:uq_off[k + 1]])
    return out


def check_winners(up, up_off, routes, msgs):
    """Every forwarded miss has a winner, and it is a valid answer (the oracle rejected every near-miss)."""
    for j, (rt, m) in enumerate(zip(routes, msgs)):
        w = bytes(up[up_off[j]:up_off[j + 1]])
        if m and rt != R.R_NONE:
            assert w and w[:2] == m[:2] and struct.unpack('>I', w[-4:])[0] != NEAR, j
        else:
            assert not w, j


def check_emu(exe, region, dcs, ups, pkts, items, key, tmp_path):
    """The device source against the C++ oracle and the Python restatement: routes, upstream queries and winners."""
    data, off = synth.pack_batch(pkts)
    tb = O.Table(region, dcs, ups)
    fwd = O.forward_batch(tb, data, off, key)
    e_route, e_msgs, e_win = emu(exe, region, dcs, ups, pkts, items, key, tmp_path)
    assert e_route == fwd[4].tolist()
    assert e_msgs == msgs_by_miss(fwd, len(pkts))
    routes, msgs = R.forward(region, dcs, ups, pkts, key)
    assert routes == e_route and msgs == e_msgs
    order, group_off = R.grouped(routes)
    assert fwd[2].tolist() == order and fwd[3].tolist() == group_off
    up, up_off = O.match_upstreams(tb, *G.pack(items), data, off, fwd[4], key)
    assert [items[w][0] if w is not None else b'' for w in e_win] == [bytes(up[up_off[j]:up_off[j + 1]]) for j in range(len(pkts))]
    assert [items[w][0] if w is not None else b'' for w in e_win] == R.match(ups, items, pkts, routes, key)
    return routes, msgs, (up, up_off)


# ---- 16 datacenters, 64 upstreams -----------------------------------------------------------------------------------
@pytest.mark.parametrize('key', KEYS)
def test_wide_table_emulated_is_bit_exact(key, tmp_path_factory, tmp_path):
    exe = emu_exe(tmp_path_factory)
    ups = wide_upstreams()
    pkts = wide_misses()
    routes, msgs = R.forward(REGION, WIDE_DCS, ups, pkts, key)
    assert set(routes) == set(range(18)) - set(HOLES)
    for p, r in zip(pkts, routes):                          # a datacenter without upstreams is no route, its neighbour is
        q = R.parse_query(p)
        if q and q[1] != R.QT_PTR and q[2].endswith('.%s.%s' % (WIDE_DCS[14], REGION)):
            assert r == R.R_NONE
        if q and q[1] != R.QT_PTR and q[2].endswith('.%s.%s' % (WIDE_DCS[15], REGION)):
            assert r == 15
    sets = {'contended': contended(ups, routes, msgs, key, random.Random(key & 0xFFFF)),
            'generated': responses(ups, routes, msgs, random.Random(3), key)}
    sets.update(G.hand_written(ups, pkts, routes, msgs, key)[1])
    for name, items in sets.items():
        _, _, (up, up_off) = check_emu(exe, REGION, WIDE_DCS, ups, pkts, items, key, tmp_path)
        if name == 'contended':
            check_winners(up, up_off, routes, msgs)


@pytest.mark.parametrize('kind', DISTRIBUTIONS)
def test_wide_routes_at_full_batch_emulated(kind, tmp_path_factory, tmp_path):
    """65,536 misses under a table where all 16 datacenters have upstreams: routes and upstream queries of the device
    source equal the oracle's, and every ID decodes to its own miss."""
    ups = wide_upstreams(holes=())
    pool = route_pool(ups)
    assert sorted(pool) == list(range(18))
    pkts = route_batch(pool, kind, 65536, DISTRIBUTIONS.index(kind))
    key = KEYS[DISTRIBUTIONS.index(kind)]
    data, off = synth.pack_batch(pkts)
    fwd = O.forward_batch(O.Table(REGION, WIDE_DCS, ups), data, off, key)
    e_route, e_msgs, _ = emu(emu_exe(tmp_path_factory), REGION, WIDE_DCS, ups, pkts, [], key, tmp_path)
    assert e_route == fwd[4].tolist()
    assert e_msgs == msgs_by_miss(fwd, len(pkts))
    ids = [struct.unpack('>H', m[:2])[0] for m in e_msgs if m]
    assert len(set(ids)) == len(ids)
    assert all(O.fwd_id(key, struct.unpack('>H', m[:2])[0], inverse=True) == j for j, m in enumerate(e_msgs) if m)


def test_width_limits_are_argument_errors(tmp_path_factory, tmp_path):
    """17 datacenters and 65 upstreams are rejected by the table builder the kernels share; GpuRecursion refuses 17
    datacenters with upstreams before it touches the resolver."""
    exe = emu_exe(tmp_path_factory)
    pkts = wide_misses()[:20]
    for dcs, ups in ((WIDE_DCS + ['one-more'], wide_upstreams()[:10]), (WIDE_DCS, wide_upstreams() + [('10.0.0.9', 53, 0)])):
        data, off = synth.pack_batch(pkts)
        buf = struct.pack('<I', len(dcs)) + b''.join(struct.pack('<I', len(d)) + d.encode() for d in dcs)
        buf += struct.pack('<I', len(REGION)) + REGION.encode() + struct.pack('<I', len(ups))
        buf += np.array([ip_u32(a) for a, _, _ in ups], np.uint32).tobytes() + np.array([p for _, p, _ in ups], np.uint16).tobytes()
        buf += np.array([d for _, _, d in ups], np.uint8).tobytes() + struct.pack('<QI', 1, len(pkts)) + off.tobytes()
        buf += data[:off[-1]].tobytes() + struct.pack('<II', 0, 0)
        src = tmp_path / 'in.bin'
        src.write_bytes(buf)
        p = subprocess.run([exe, str(src), str(tmp_path / 'out.bin')], capture_output=True, text=True)
        assert p.returncode == 2 and 'bad table' in p.stderr
    # sixteen with upstreams is the limit; a seventeenth is refused whatever the resolver
    ok = GpuRecursion(O.ForwardOracle(), REGION, {d: ['10.0.0.%d' % k] for k, d in enumerate(WIDE_DCS)}, timeout=0.1)
    ok.close()
    with pytest.raises(ValueError):
        GpuRecursion(O.ForwardOracle(), REGION, {d: ['10.0.0.%d' % k] for k, d in enumerate(WIDE_DCS + ['one-more'])})


# ---- QNAME labels with a '.' inside ---------------------------------------------------------------------------------
# (region, datacenters, QNAME labels, route of lib/recursion.js on the dotted name)
DOT_CASES = [
    ('foo.com', ['web', 'b'], [b'h1', b'x.web', b'foo', b'com'], 0),
    ('foo.com', ['web', 'b'], [b'h1', b'web', b'foo.com'], 0),
    ('foo.com', ['web', 'b'], [b'h1', b'a.b', b'foo', b'com'], 1),
    ('foo.com', ['x.web', 'b'], [b'h1', b'x.web', b'foo', b'com'], R.R_NONE),     # a dc name the dotted string never yields
    ('com', ['foo'], [b'h1', b'web.foo', b'com'], 0),
]


def dot_ups(dcs):
    return [('10.0.%d.1' % k, 53, k) for k in range(len(dcs))]


@pytest.mark.parametrize('ci', range(len(DOT_CASES)))
def test_in_label_dot_routes_like_the_dotted_name(ci, tmp_path_factory, tmp_path):
    region, dcs, labels, want = DOT_CASES[ci]
    ups = dot_ups(dcs)
    pkts = [synth.make_query(None, 'A', qid=7, labels=labels), synth.make_query(None, 'SRV', qid=8, edns=1200, labels=labels)]
    items = [(answer(m, 1), (ups[k][0], 53)) for m in R.forward(region, dcs, ups, pkts, 5)[1] for k in range(len(dcs))]
    routes, _, (up, up_off) = check_emu(emu_exe(tmp_path_factory), region, dcs, ups, pkts, items, 5, tmp_path)
    assert routes == [want, want]
    assert (up_off[-1] > 0) == (want != R.R_NONE)          # the datacenter's upstream is the one whose answer is taken


DOT_REGIONS = ['', '.', '.foo.com', 'foo.com', 'oo.com', 'FOO.com', 'Foo.Com', 'com', 'o.com', 'a.b.foo.com', 'x.web.foo.com',
               'web.foo.com', 'foo.c']
DOT_DCS = ['web', 'Web', 'WEB', 'w', 'b', 'eb', 'x.web', 'a.b', 'web.foo', 'foo', 'com', 'h1', 'x' * 63, 'c.d.e', '.', 'db',
           'a-b', 'o', 'Foo', 'oo', 'b.foo', '.web']


def dotted_name(rng, region, dcs):
    """QNAME labels: a prefix, a datacenter-like label and the region (or something near it), with random neighbouring
    pieces joined into one label around a '.' — inside the datacenter label, inside the region's labels, or both."""
    tail = rng.choice([region, region, region.upper(), 'foo.org', region[1:], 'x' + region])
    parts = [rng.choice(['h1', 'a', 'Q', 'x.y', '']), rng.choice(dcs + ['zz', 'web.zz', 'eb'])] + [tail]
    pieces = [p for p in '.'.join(parts).split('.') if p] or ['a']
    labels = [pieces[0]]
    for p in pieces[1:]:
        if rng.random() < 0.35 and len(labels[-1]) + 1 + len(p) <= 63:
            labels[-1] += '.' + p
        else:
            labels.append(p)
    return [l.encode() for l in labels]


def dot_filters(count=200, seed=4242):
    """(region, datacenters, upstreams, misses) of the differential fuzz: 1-16 datacenters, some without upstreams."""
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        region = rng.choice(DOT_REGIONS)
        dcs = rng.sample(DOT_DCS, rng.randint(1, 16))
        ups = [('10.%d.0.1' % k, 53, k) for k in range(len(dcs)) if rng.random() < 0.85] or [('10.0.0.1', 53, 0)]
        pkts = [synth.make_query(None, rng.choice(['A', 'A', 'SRV']), qid=i, labels=dotted_name(rng, region, dcs)) for i in range(40)]
        pkts += [synth.make_query('1.0.0.10.in-addr.arpa', 'PTR', qid=99)]
        out.append((region, dcs, ups, pkts))
    return out


def test_in_label_dot_fuzz_emulated_matches_both_oracles(tmp_path_factory, tmp_path):
    exe = emu_exe(tmp_path_factory)
    dotted_routes = 0
    for fi, (region, dcs, ups, pkts) in enumerate(dot_filters()):
        routes, msgs = R.forward(region, dcs, ups, pkts, fi)
        items = [(answer(m, 2), (ups[0][0], ups[0][1])) for m in msgs if m]
        check_emu(exe, region, dcs, ups, pkts, items, fi, tmp_path)
        dotted_routes += sum(1 for p, r in zip(pkts, routes) if r < R.R_PTR and b'.' in p[12:])
    assert dotted_routes > 200                              # the corpus does route names with in-label dots


# ---- GpuRecursion windows no larger than the resolver takes ----------------------------------------------------------
class FakeUpstream(object):
    """A UDP resolver on loopback answering every query with one A record, paced so that no socket buffer overflows."""

    def __init__(self):
        self.sock = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
        self.sock.setsockopt(socket.SOL_SOCKET, socket.SO_RCVBUF, 1 << 20)
        self.sock.bind(('127.0.0.1', 0))
        self.sock.settimeout(0.05)
        self.addr = self.sock.getsockname()
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()

    def _run(self):
        sent = 0
        while not self._stop.is_set():
            try:
                data, src = self.sock.recvfrom(65535)
            except socket.timeout:
                continue
            self.sock.sendto(answer(data, len(data)), src)
            sent += 1
            if sent % 16 == 0:
                time.sleep(0.0005)

    def close(self):
        self._stop.set()
        self._thread.join(2)
        self.sock.close()


class ListSink(object):
    """A transport owner's sink that keeps each tag's (client query, upstream response)."""

    def __init__(self):
        self.got, self.windows = {}, []
        self.lock = threading.Lock()

    def relay(self, q_data, q_off, up, up_off, tags):
        with self.lock:
            self.windows.append(len(tags))
            for i, t in enumerate(tags):
                self.got[t] = (bytes(q_data[q_off[i]:q_off[i + 1]]), bytes(up[up_off[i]:up_off[i + 1]]))


class CappedOracle(O.ForwardOracle):
    """The CPU stand-in for an Engine(max_batch=256): more misses in one call is an error, as bb_forward_batch,
    bb_match_upstreams and bb_relay_batch make it."""
    max_batch = 256

    def _check(self, off):
        if len(off) - 1 > self.max_batch:
            raise ValueError('%d misses > max_batch %d' % (len(off) - 1, self.max_batch))

    def forward_batch(self, data, off, id_key):
        self._check(off)
        return super(CappedOracle, self).forward_batch(data, off, id_key)

    def match_upstreams(self, resp, resp_off, src_ip, src_port, q_data, q_off, route, id_key):
        self._check(q_off)
        return super(CappedOracle, self).match_upstreams(resp, resp_off, src_ip, src_port, q_data, q_off, route, id_key)

    def relay_batch(self, q_data, q_off, up_data, up_off, tcp=False):
        self._check(q_off)
        return super(CappedOracle, self).relay_batch(q_data, q_off, up_data, up_off, tcp)


def run_window_cap(resolver, n=1000):
    """n misses submitted at once to a GpuRecursion with a long collection window: each comes back with its upstream's
    answer, through windows of at most resolver.max_batch misses."""
    up = FakeUpstream()
    rec = GpuRecursion(resolver, REGION, {'dc2': [up.addr]}, timeout=3.0, window_s=1.0)
    sink = ListSink()
    pkts = [synth.make_query('h%d.dc2.%s' % (i, REGION), 'A', qid=i) for i in range(n)]
    try:
        for i, p in enumerate(pkts):
            rec.submit(p, sink, i)
        end = time.time() + 60
        while len(sink.got) < n and time.time() < end:
            time.sleep(0.05)
        counters = dict(rec.counters)
    finally:
        rec.close()
        up.close()
    assert counters['failed_batches'] == 0
    assert len(sink.got) == n and max(sink.windows) <= resolver.max_batch
    for i, p in enumerate(pkts):
        q, u = sink.got[i]
        assert q == p
        assert len(u) > 12 and u[2] & 0x80 and u[12:12 + len(p) - 12] == p[12:], i
    assert counters['upstream_answers'] == n


def test_window_cap_cpu():
    run_window_cap(CappedOracle())
