"""Recursion relay on the CPU (DESIGN.md section 13, lib/recursion.js:287-327): the C++ oracle against the independent
Python restatement on fuzzed upstreams built with dnspython, every reply decoded by dnspython; hand-written malformed
upstreams; the NOTIMP quirk; the failed-lookup reply against the pre-filter's REFUSED; and the device source
(binder_b200/csrc/relay_device.cuh, through tests/native/emu_relay.cpp) bit-exact against the oracle, also under
AddressSanitizer and UndefinedBehaviorSanitizer."""
import os
import random
import shutil
import struct
import subprocess

import dns.flags
import dns.ipv4
import dns.ipv6
import dns.message
import dns.rdatatype
import numpy as np
import pytest

import fuzzgen
from oracle_lib import Oracle
import relay_oracle
import relaygen as G
from binder_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def relay_list(pairs, tcp=False):
    """[(query, upstream)] through the oracle -> [(status, reply bytes)]."""
    out, off, lens, st = relay_oracle.relay_batch(*G.pack_pairs(pairs), tcp=tcp)
    return [(int(st[i]), bytes(out[off[i]:off[i] + lens[i]])) for i in range(len(pairs))]


def _labels(name):
    return tuple(l for l in name.labels if l)


def decode_reply(wire):
    """dnspython's view of a reply -> (message, [(owner, ttl, type, data)]) shaped like relay_ref.relay's answers."""
    m = dns.message.from_wire(wire, one_rr_per_rrset=True, raise_on_truncation=False)
    ans = []
    for rrset in m.answer:
        owner = '.'.join(l.decode('latin-1') for l in _labels(rrset.name))
        for rd in rrset:
            t = dns.rdatatype.to_text(rrset.rdtype)
            if t == 'A':
                data = dns.ipv4.inet_aton(rd.address)
            elif t == 'AAAA':
                data = dns.ipv6.inet_aton(rd.address)
            elif t == 'TXT':
                data = b''.join(bytes([len(s)]) + s for s in rd.strings)
            elif t in ('CNAME', 'PTR'):
                data = _labels(rd.target)
            elif t == 'SRV':
                data = (rd.priority, rd.weight, rd.port, _labels(rd.target))
            else:
                raise AssertionError('unexpected type %s' % t)
            ans.append((owner, rrset.ttl, t, data))
    return m, ans


def size_limit(q, tcp):
    if tcp:
        return 65535
    if struct.unpack('>H', q[10:12])[0]:
        qn = 12
        while q[qn]:
            qn += 1 + q[qn]
        adv = struct.unpack('>H', q[qn + 8:qn + 10])[0]
        return min(max(adv, 512), 1200)
    return 512


def check_semantic(pair, status, wire, tcp):
    """One oracle reply against relay_ref.relay, through dnspython."""
    q = pair[0]
    rcode, answers = G.semantic(pair)
    # dnspython reads a TTL with the top bit set as 0 (RFC 2181 8); the reply carries the upstream's 32 bits
    answers = tuple((o, t if t < 2 ** 31 else 0) + tuple(rest) for o, t, *rest in answers)
    assert status == 0
    m, ans = decode_reply(wire)
    assert m.rcode() == rcode
    assert tuple(ans) == answers[:len(ans)]
    assert bool(m.flags & dns.flags.TC) == (len(ans) < len(answers))
    assert m.id == struct.unpack('>H', q[:2])[0] and m.flags & dns.flags.QR and m.flags & dns.flags.AA
    assert not m.flags & dns.flags.RA and bool(m.flags & dns.flags.RD) == bool(q[2] & 1)
    assert wire[12:12 + len(q) - 12 - (11 if q[11] else 0)] == q[12:len(q) - (11 if q[11] else 0)]   # question verbatim
    assert (m.edns >= 0) == bool(q[11])
    assert len(wire) <= size_limit(q, tcp)
    return rcode, len(ans) < len(answers)


@pytest.mark.parametrize('tcp', [False, True])
def test_oracles_agree_on_fuzzed_relays(tcp):
    pairs = G.gen_relays(7 + tcp, 3000)
    seen = set()
    for pair, (st, wire) in zip(pairs, relay_list(pairs, tcp)):
        seen.add(check_semantic(pair, st, wire, tcp))
    assert {(0, False), (4, False), (5, False), (0, True)} <= seen, seen


def test_truncation_over_udp_and_tcp():
    rng = random.Random(3)
    pairs = [G.relay_case(rng, 'expand') for _ in range(6)] + [G.relay_case(rng, 'many') for _ in range(20)]
    udp, tcp = relay_list(pairs), relay_list(pairs, tcp=True)
    for pair, (_, w) in zip(pairs, udp):
        assert len(w) <= size_limit(pair[0], False)
    for pair, (_, wu), (_, wt) in zip(pairs[:6], udp, tcp):
        mu, _ = decode_reply(wu)
        mt, at = decode_reply(wt)
        assert mu.flags & dns.flags.TC and mt.flags & dns.flags.TC     # > 65,535 bytes once the pointers are expanded
        assert 65535 - 300 < len(wt) <= 65535 and len(at) < struct.unpack('>H', pair[1][6:8])[0]


def test_malformed_upstreams_are_refused():
    q = synth.make_query('h1.dc2.example.com', 'A', qid=7, edns=1200)
    empty = relay_list([(q, b'')])[0]
    bad = G.malformed_upstreams()
    res = relay_list([(q, u) for u in bad.values()])
    for name, (st, wire) in zip(bad, res):
        assert st == 0 and wire == empty[1], name
        m, ans = decode_reply(wire)
        assert m.rcode() == 5 and not ans, name


def test_only_dropped_types_give_notimp():
    rng = random.Random(5)
    for _ in range(20):
        pair = G.relay_case(rng, 'only_mx')
        st, wire = relay_list([pair])[0]
        m, ans = decode_reply(wire)
        assert st == 0 and m.rcode() == 4 and not ans and not m.flags & dns.flags.TC


def test_failed_lookup_equals_prefilter_refusal():
    """A relay whose lookup failed sends exactly the REFUSED the pre-filter answers on the device for the same query."""
    snap, info = fuzzgen.gen_zone(901, n_top=10)
    dom = info['dns_domain']
    orc = Oracle(dom, '', True, snapshot=snap)
    rng = random.Random(11)
    pkts = [synth.make_query('zz%d.nodc.%s' % (i, dom), 'A', qid=rng.randrange(65536),
                             rd=True, edns=rng.choice([None, 512, 1200, 4096])) for i in range(200)]
    pkts = [p if i % 3 else synth.make_query('_x._tcp.zz%d.nodc.%s' % (i, dom), 'SRV', qid=i, edns=1200) for i, p in enumerate(pkts)]
    data, off = synth.pack_batch(pkts)
    _, _, _, st0, _ = orc.resolve_batch(data, off)
    assert (st0 == 1).all()                                        # misses handed to recursion without the filter
    orc.set_recursion_filter(dom, [], False)
    out, ooff, olen, st, miss = orc.resolve_batch(data, off)
    assert (st == 0).all() and len(miss) == 0
    relayed = relay_list([(p, b'') for p in pkts])
    for i, (s, w) in enumerate(relayed):
        assert s == 0 and w == bytes(out[ooff[i]:ooff[i] + olen[i]]), i


# ---- the device source on the CPU ----------------------------------------------------------------------------------
_EXE = {}


def emu_exe(tmp_factory, sanitize=False):
    if sanitize not in _EXE:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        exe = str(tmp_factory.mktemp('emu_relay') / 'emu_relay')
        san = ['-g', '-fsanitize=address,undefined', '-fno-sanitize-recover=undefined', '-fno-omit-frame-pointer'] if sanitize else []
        b = subprocess.run([cxx, '-std=c++17', '-O1', '-Wno-unknown-pragmas'] + san + ['-I', os.path.join(ROOT, 'include'),
                            '-I', os.path.join(ROOT, 'binder_b200', 'csrc'), '-o', exe, os.path.join(ROOT, 'tests', 'native', 'emu_relay.cpp')],
                           capture_output=True, text=True)
        if sanitize and b.returncode != 0 and 'sanitize' in b.stderr:
            pytest.skip('toolchain without sanitizer runtimes')
        assert b.returncode == 0, b.stderr[-3000:]
        _EXE[sanitize] = exe
    return _EXE[sanitize]


def emu_relay(exe, pairs, tcp, tmp_path):
    """The device source on the CPU -> ((out, out_off, out_len, status), stderr)."""
    q_data, q_off, up_data, up_off = G.pack_pairs(pairs)
    n = len(pairs)
    src, dst = str(tmp_path / 'in.bin'), str(tmp_path / 'out.bin')
    with open(src, 'wb') as f:
        f.write(struct.pack('<II', n, 1 if tcp else 0) + q_off.tobytes() + up_off.tobytes() +
                q_data[:q_off[n]].tobytes() + up_data[:up_off[n]].tobytes())
    p = subprocess.run([exe, src, dst], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0:abort_on_error=1'))
    assert p.returncode == 0 and p.stdout.startswith('OK') and 'runtime error' not in p.stderr, p.stderr[-3000:]
    raw = open(dst, 'rb').read()
    out_off = np.frombuffer(raw[:4 * (n + 1)], dtype=np.uint32)
    status = np.frombuffer(raw[4 * (n + 1):4 * (n + 1) + n], dtype=np.uint8)
    out = np.frombuffer(raw[4 * (n + 1) + n:], dtype=np.uint8)
    return (out, out_off, np.diff(out_off.astype(np.int64)).astype(np.uint16), status)


def bad_queries(rng, n):
    """Queries decode() rejects (the relay drops them) and queries it accepts that no resolver path would answer."""
    good = synth.make_query('x.dc2.example.com', 'A', qid=9)
    out = [good[:11], b'', good[:2] + b'\x81\x00' + good[4:], good[:4] + b'\x00\x02' + good[6:], good + b'trailing',
           synth.make_query('x.dc2.example.com', 'A', qclass=3), synth.make_query('x.y', 'A', opcode=2),
           synth.make_query('x.y', 99), good[:-3]]
    return [(out[i % len(out)], G.relay_case(rng, 'a')[1]) for i in range(n)]


def corpus(seed, n):
    rng = random.Random(seed)
    pairs = G.gen_relays(seed, n)
    pairs += [(synth.make_query('h1.dc2.example.com', 'A', qid=i, edns=rng.choice([None, 1200])), u)
              for i, u in enumerate(G.malformed_upstreams().values())]
    pairs += [(q, G.mutate(rng, u)) for q, u in G.gen_relays(seed + 1, n // 2)]
    return pairs + bad_queries(rng, 40)


def assert_same_relays(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize('tcp', [False, True])
def test_emulated_relay_is_bit_exact(tcp, tmp_path_factory, tmp_path):
    pairs = corpus(21 + tcp, 3000)
    got = emu_relay(emu_exe(tmp_path_factory), pairs, tcp, tmp_path)
    want = relay_oracle.relay_batch(*G.pack_pairs(pairs), tcp=tcp)
    assert_same_relays(got, want)
    st = want[3]
    assert (st == 2).sum() >= 20 and (st == 0).sum() > 4000


def test_emulated_relay_is_sanitizer_clean(tmp_path_factory, tmp_path):
    """The malformed corpus and a few thousand randomly damaged upstreams under ASan/UBSan (any finding aborts)."""
    rng = random.Random(99)
    valid = G.gen_relays(31, 1500)
    pairs = [(q, G.mutate(rng, u)) for q, u in valid for _ in range(2)]
    pairs += [(synth.make_query('h1.dc2.example.com', 'A', qid=i), u) for i, u in enumerate(G.malformed_upstreams().values())]
    pairs += bad_queries(rng, 40)
    exe = emu_exe(tmp_path_factory, sanitize=True)
    for tcp in (False, True):
        got = emu_relay(exe, pairs, tcp, tmp_path)
        assert_same_relays(got, relay_oracle.relay_batch(*G.pack_pairs(pairs), tcp=tcp))
