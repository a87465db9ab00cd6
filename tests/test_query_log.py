"""Query log on the CPU (DESIGN.md section 15, lib/server.js:509-591): the device source (binder_b200/csrc/log_device.cuh,
through tests/native/emu_log.cpp) byte for byte against the independent restatement (tests/query_log_ref.py), per record
and per fragment, on result sets of the C++ oracles (fuzzgen and namegen zones, relaygen relays, the reference's golden
cases; UDP and TCP) and on hand-written responses: every escaped byte class, names at their length limits, suffix
stripping at its edges, RFC 5952 addresses, and malformed responses, which get an empty record and the bad bit.  The
malformed set and randomly damaged responses also run under AddressSanitizer and UndefinedBehaviorSanitizer."""
import json
import os
import random
import shutil
import struct
import subprocess

import numpy as np
import pytest

import fuzzgen
import helpers as H
import namegen as N
import query_log_ref as L
import relay_oracle
import relaygen as G
from binder_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'reference_cases.json')))
DOM = 'example.com'


# ---- result sets -------------------------------------------------------------------------------------------------
def pack_set(resps, status=None):
    """[response bytes] -> (out, out_off uint32[n+1], out_len uint16[n], status uint8[n]), packed in order."""
    out, off = synth.pack_batch(resps) if resps else (np.zeros(16, np.uint8), np.zeros(1, np.uint32))
    n = len(resps)
    st = np.zeros(n, np.uint8) if status is None else np.asarray(status, np.uint8)
    return out, off, np.diff(off.astype(np.int64)).astype(np.uint16), st


def fuzz_set(seed, tcp=False, n=400):
    """A fuzzgen zone's queries (plus malformed ones, dropped) through the oracle with recursion (misses) -> (result set, dnsDomain)."""
    snap, info = fuzzgen.gen_zone(seed)
    dom = info['dns_domain']
    orc = H.make_impl('oracle', dom, snap, recursion=True)
    pkts = fuzzgen.gen_queries(seed, info, n) + fuzzgen.malformed_packets()
    out, off, lens, st, _ = orc.resolve_batch(*synth.pack_batch(pkts), seed=seed, tcp=tcp)
    return (out, off, lens, st), dom


def name_sets(tcp=False):
    """Every namegen dnsDomain's boundary zone: A queries of its hosts, SRV queries of its services."""
    for key in N.DOMAINS:
        z = N.BoundaryZone(key)
        orc = H.make_impl('oracle', z.dom, z.snap)
        pkts = [synth.make_query(h, 'A', qid=i, edns=1200 if i % 2 else None) for i, (h, _) in enumerate(z.hosts)]
        pkts += [synth.make_query('%s.%s.%s' % (sv, pr, s), 'SRV', qid=i, edns=4096 if i % 3 else None)
                 for i, (s, sv, pr) in enumerate(z.services)]
        pkts += [synth.make_query(s, 'A', qid=i) for i, (s, _, _) in enumerate(z.services)]
        out, off, lens, st, _ = orc.resolve_batch(*synth.pack_batch(pkts), seed=5, tcp=tcp)
        yield key, (out, off, lens, st), z.dom


def relay_set(seed, tcp=False, n=1500):
    """relaygen relays (AAAA, TXT, CNAME, PTR, upstream SRV, NOTIMP, REFUSED misses, truncations) through the oracle."""
    rng = random.Random(seed)
    pairs = G.gen_relays(seed, n) + [G.relay_case(rng, k) for k in ('expand', 'many', 'srv3', 'empty', 'only_mx') for _ in range(4)]
    out, off, lens, st = relay_oracle.relay_batch(*G.pack_pairs(pairs), tcp=tcp)
    return out, off[:len(pairs) + 1], lens, st


def golden_set():
    """The reference's 13 golden cases, without and with EDNS, one oracle per suite -> [(result set, dnsDomain)]."""
    sets = []
    for suite in GOLD['suites']:
        orc = H.make_impl('oracle', GOLD['dns_domain'], H.snapshot(suite['snapshot']))
        pkts = [synth.make_query(c['name'], c['type'], qid=0xBEEF, edns=e) for c in suite['cases'] for e in (None, 4096)]
        out, off, lens, st, _ = orc.resolve_batch(*synth.pack_batch(pkts), seed=7)
        sets.append(((out, off, lens, st), GOLD['dns_domain']))
    return sets


# ---- hand-written responses --------------------------------------------------------------------------------------
def wire(labels):
    return b''.join(bytes([len(l)]) + l for l in labels) + b'\x00'


def response(qlabels, qtype, an=(), ns=(), ar=(), edns=False, rcode=0, tc=False):
    """Raw response: RRs are (owner wire, type, rdata); b'\\xc0\\x0c' names the question."""
    flags = 0x8400 | (0x200 if tc else 0) | rcode
    ar = list(ar) + ([(b'\x00', 41, b'')] if edns else [])
    pkt = struct.pack('>HHHHHH', 0x4242, flags, 1, len(an), len(ns), len(ar)) + wire(qlabels) + struct.pack('>HH', qtype, 1)
    for owner, t, rd in list(an) + list(ns) + ar:
        pkt += owner + struct.pack('>HHIH', t, 4096 if t == 41 else 1, 0 if t == 41 else 30, len(rd)) + rd
    return pkt


def srv(target, port=8080):
    return struct.pack('>HHH', 0, 10, port) + target


ODD = [b'a"b\\c/d', bytes(range(0, 32)), b'\x7f~ ', bytes(range(0x80, 0xBF)), bytes(range(0xBF, 0xFE)), b'\xfe\xff']
V6 = [bytes(16), bytes(15) + b'\x01', b'\x00\x01' + bytes(14), b'\x00\x01\x00\x00\x00\x00\x00\x02\x00\x00\x00\x00\x00\x03\x00\x04',
      bytes(10) + b'\xff\xff\x01\x02\x03\x04', b'\x20\x01\x0d\xb8\x00\x00\x00\x01\x00\x02\x00\x03\x00\x04\x00\x05',
      b'\x00\x01\x00\x00\x00\x02\x00\x03\x00\x04\x00\x05\x00\x06\x00\x07', b'\xfe\x80' + bytes(6) + b'\xab\xcd' * 4]
D = [b'example', b'com']


def hand_responses():
    long4 = [b'a' * 63, b'b' * 63, b'c' * 63, b'd' * 61]                               # 255 wire bytes
    names = [[b'x'] + D, D, [b'x', b'EXAMPLE', b'com'], [b'xexample', b'com'], [b'a.b', b'dc2'] + D,
             [b'x', b'foo.example', b'com'], [b'.example.com'], [b'q.example.com'], ODD + D, long4, [b'z' * 63] + D, []]
    out = []
    for i, nm in enumerate(names):                                                       # SRV targets and additional owners
        out.append(response([b'_s', b'_tcp'] + D, 33, an=[(b'\xc0\x0c', 33, srv(wire(nm), i))],
                            ar=[(wire(nm), 1, bytes([10, 0, 0, i]))], edns=i % 2 == 0))
        out.append(response(nm, 12, an=[(b'\xc0\x0c', 12, wire(nm))], ar=[(wire(nm), 28, V6[i % len(V6)])]))
    for lab in ODD + [b'q' * 63]:                                                         # odd bytes in names and text
        out.append(response([lab] + D, 16, an=[(b'\xc0\x0c', 16, bytes([len(lab)]) + lab + b'\x03end')]))
        out.append(response([lab, lab[:10] or b'x'], 5, an=[(b'\xc0\x0c', 5, wire([lab] + D))]))
    out.append(response(long4, 1, an=[(b'\xc0\x0c', 1, b'\x01\x02\x03\x04')]))
    out.append(response([b'h'] + D, 28, an=[(b'\xc0\x0c', 28, v) for v in V6]))
    soa = wire(D) + wire([b'hostmaster'] + D) + struct.pack('>IIIII', 0, 10, 10, 10, 60)
    out.append(response([b'nodata'] + D, 28, ns=[(b'\xc0\x0c', 6, soa)], edns=True))                # NODATA, authority not logged
    out.append(response([b'nx'] + D, 1, ns=[(wire(D), 6, soa)], rcode=3))
    out.append(response([b'r'] + D, 1, rcode=5, edns=True))                                           # REFUSED
    out.append(response([b'ni'] + D, 15, rcode=4))                                                    # NOTIMP
    out.append(response([b't'] + D, 1, an=[(b'\xc0\x0c', 1, bytes([1, 2, 3, i])) for i in range(3)], tc=True))
    out.append(response([], 2, an=[(b'\x00', 99, b'\x01\x02'), (b'\x00', 15, b'\x00\x0a' + wire(D)), (b'\x00', 2, wire(D))],
                        ar=[(b'\xc0\x0c', 12, wire(ODD)), (b'\xc0\x0c', 16, b'\x02hi'), (b'\xc0\x0c', 33, srv(wire(D))),
                            (b'\xc0\x0c', 65280, b'')]))
    for t in (1, 2, 5, 6, 12, 15, 16, 28, 33, 41, 252, 255, 0, 99, 65535):                            # type mnemonics
        out.append(response([b'ty'] + D, t))
    return out


def malformed_responses():
    good = response([b'h1'] + D, 1, an=[(b'\xc0\x0c', 1, b'\x01\x02\x03\x04')])
    q = good[:good.index(b'\x00\x01\x00\x01') + 4]
    body = lambda *rrs: q[:6] + struct.pack('>H', len(rrs)) + q[8:] + b''.join(rrs)        # noqa: E731
    rr = lambda owner, t, rd: owner + struct.pack('>HHIH', t, 1, 60, len(rd)) + rd          # noqa: E731
    return {
        'forward_pointer': body(rr(b'\xc0\x30', 1, b'\x01\x02\x03\x04')) + b'\x02xx\x00',
        'pointer_loop': body(rr(b'\x01a\xc0\x1f', 1, b'\x01\x02\x03\x04')),
        'self_pointer': body(rr(b'\xc0\x1f', 1, b'\x01\x02\x03\x04')),
        'rdlen_past_end': body(b'\xc0\x0c' + struct.pack('>HHIH', 1, 1, 60, 40) + b'\x01\x02\x03\x04'),
        'a_rdlen_5': body(rr(b'\xc0\x0c', 1, b'\x01\x02\x03\x04\x05')),
        'aaaa_rdlen_4': body(rr(b'\xc0\x0c', 28, b'\x01\x02\x03\x04')),
        'srv_rdlen_6': body(rr(b'\xc0\x0c', 33, b'\x00\x01\x00\x02\x00\x03')),
        'ptr_name_past_rdlen': body(rr(b'\xc0\x0c', 12, b'\x03abc')) + b'\x00',
        'txt_string_past_rdlen': body(rr(b'\xc0\x0c', 16, b'\x05ab')),
        'txt_empty': body(rr(b'\xc0\x0c', 16, b'')),
        'count_too_high': body(rr(b'\xc0\x0c', 1, b'\x01\x02\x03\x04'), b''),
        'label_over_63': body(rr(b'\x40' + b'a' * 64 + b'\x00', 1, b'\x01\x02\x03\x04')),
        'name_over_255': body(rr((b'\x3f' + b'a' * 63) * 4 + b'\x00', 1, b'\x01\x02\x03\x04')),
        'question_pointer': good[:12] + b'\x01x\xc0\x0c' + good[12 + len(wire([b'h1'] + D)):],
        'question_cut': good[:20],
        'qr_zero': good[:2] + bytes([good[2] & 0x7F]) + good[3:],
        'qdcount_2': good[:4] + b'\x00\x02' + good[6:],
        'header_only_11': good[:11],
    }


# ---- the device source on the CPU --------------------------------------------------------------------------------
_EXE = {}


def emu_exe(tmp_factory, sanitize=False):
    if sanitize not in _EXE:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        exe = str(tmp_factory.mktemp('emu_log') / 'emu_log')
        san = ['-g', '-fsanitize=address,undefined', '-fno-sanitize-recover=undefined', '-fno-omit-frame-pointer'] if sanitize else []
        b = subprocess.run([cxx, '-std=c++17', '-O1', '-Wno-unknown-pragmas'] + san + ['-I', os.path.join(ROOT, 'include'),
                            '-o', exe, os.path.join(ROOT, 'tests', 'native', 'emu_log.cpp')], capture_output=True, text=True)
        if sanitize and b.returncode != 0 and 'sanitize' in b.stderr:
            pytest.skip('toolchain without sanitizer runtimes')
        assert b.returncode == 0, b.stderr[-3000:]
        _EXE[sanitize] = exe
    return _EXE[sanitize]


def emu_log(exe, rs, dom, tmp_path, resp_bytes=None):
    """The device source on the CPU over a result set -> [(head, body, summary)] as query_log_ref.log_set gives."""
    out, off, lens, st = rs
    n = len(st)
    rb = len(out) if resp_bytes is None else resp_bytes
    sfx = ('.' + dom).encode('latin-1') if dom else b''
    src, dst = str(tmp_path / 'in.bin'), str(tmp_path / 'out.bin')
    with open(src, 'wb') as f:
        f.write(struct.pack('<III', n, rb, len(sfx)) + sfx + np.asarray(off[:n], np.uint32).tobytes() +
                np.asarray(lens, np.uint16).tobytes() + np.asarray(st, np.uint8).tobytes() + bytes(out[:rb]))
    p = subprocess.run([exe, src, dst], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0:abort_on_error=1'))
    assert p.returncode == 0 and p.stdout.startswith('OK') and 'runtime error' not in p.stderr, p.stderr[-3000:]
    raw = open(dst, 'rb').read()
    ll, hl, sm = (np.frombuffer(raw[4 * n * k:4 * n * (k + 1)], np.uint32) for k in range(3))
    text, at, res = raw[12 * n:], 0, []
    for i in range(n):
        rec = text[at:at + ll[i]]
        at += int(ll[i])
        res.append((rec[:hl[i]], rec[hl[i]:], int(sm[i])))
    assert at == len(text)
    return res


def assert_same_log(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, g, w)


def check_set(exe, rs, dom, tmp_path):
    want = L.log_set(*rs, dom)
    assert_same_log(emu_log(exe, rs, dom, tmp_path), want)
    return want


@pytest.mark.parametrize('tcp', [False, True])
def test_fuzzed_zones(tcp, tmp_path_factory, tmp_path):
    exe = emu_exe(tmp_path_factory)
    for seed in (3, 4):
        rs, dom = fuzz_set(seed + 10 * tcp, tcp)
        want = check_set(exe, rs, dom, tmp_path)
        assert sum(1 for h, _, _ in want if h) > 200 and any(s == 2 for s in rs[3]) and any(s == 1 for s in rs[3])


@pytest.mark.parametrize('tcp', [False, True])
def test_names_at_length_limits(tcp, tmp_path_factory, tmp_path):
    exe = emu_exe(tmp_path_factory)
    stripped = 0
    for key, rs, dom in name_sets(tcp):
        want = check_set(exe, rs, dom, tmp_path)
        assert sum(1 for h, _, _ in want if h) > 10, key
        stripped += sum(b.count(b'...') for _, b, _ in want)
    assert stripped > 100


@pytest.mark.parametrize('tcp', [False, True])
def test_relayed_replies(tcp, tmp_path_factory, tmp_path):
    want = check_set(emu_exe(tmp_path_factory), relay_set(40 + tcp, tcp), 'dc2.example.com', tmp_path)
    body = b''.join(b for _, b, _ in want)
    for needle in (b'"AAAA ', b'"type":"TXT"', b'"type":"CNAME"', b'"type":"PTR"', b'"SRV ', b'...:', b'"rcode":4', b'"rcode":5'):
        assert needle in body, needle
    assert any(s >> 21 & 1 for _, _, s in want)                                       # truncated replies


def test_golden_reference_cases(tmp_path_factory, tmp_path):
    exe = emu_exe(tmp_path_factory)
    for rs, dom in golden_set():
        want = check_set(exe, rs, dom, tmp_path)
        assert all(h for h, _, _ in want)


@pytest.mark.parametrize('dom', [DOM, '', 'com'])
def test_hand_written_responses(dom, tmp_path_factory, tmp_path):
    resps = hand_responses()
    want = check_set(emu_exe(tmp_path_factory), pack_set(resps), dom, tmp_path)
    assert all(s & L.BAD == 0 for _, _, s in want)
    if dom == DOM:
        text = b'\n'.join(h + b'|' + b for h, b, _ in want)
        for needle in ('"SRV x...:0"', '"SRV example.com:1"', '"SRV x.EXAMPLE.com:2"', '"SRV xexample.com:3"',
                       '"SRV a.b.dc2...:4"', '"SRV x.foo...:5"', '"SRV ...:6"', '"SRV q...:7"', '"x... A 10.0.0.0"',
                       '"AAAA ::"', '"AAAA ::1"', '"AAAA 1::"', '"AAAA 1::2:0:0:3:4"', '"AAAA ::ffff:102:304"',
                       '"AAAA 2001:db8:0:1:2:3:4:5"', '"AAAA 1:0:2:3:4:5:6:7"', '"AAAA fe80::abcd:abcd:abcd:abcd"',
                       '\\u0000\\u0001', '\\b\\t\\n\\u000b\\f\\r', '\\u001f', 'a\\"b\\\\c/d', '\x7f~ ', '\u0080\u0081',
                       'ÿ', '"type":"TYPE99"', '{"type":"MX"}', '{"type":"TYPE65280"}', '{"type":"SRV"}',
                       '"type":"TYPE0"', '"type":"ANY"', '"name":""', '"rcode":3', '"edns":true'):
            assert needle.encode('utf-8') in text, needle
        assert b'hostmaster' not in text and b'OPT' not in text.replace(b'"type":"OPT"', b'')


def test_malformed_responses_get_the_bad_bit(tmp_path_factory, tmp_path):
    exe = emu_exe(tmp_path_factory)
    bad = malformed_responses()
    rs = pack_set(list(bad.values()))
    got = emu_log(exe, rs, DOM, tmp_path)
    assert_same_log(got, L.log_set(*rs, DOM))
    for name, (h, b, s) in zip(bad, got):
        assert h == b == b'' and s == L.BAD, name
    # offsets or lengths outside the response bytes
    good = pack_set([response([b'h'] + D, 1, an=[(b'\xc0\x0c', 1, b'\x01\x02\x03\x04')])] * 4)
    out, off, lens, st = good
    total = int(off[4])
    off = off.copy(); lens = lens.copy()
    off[1], off[2], lens[3] = total + 1, 0xFFFFFFF0, 0xFFFF
    got = emu_log(exe, (out, off, lens, st), DOM, tmp_path, resp_bytes=total)
    assert got[0][0] and [g[2] for g in got[1:]] == [L.BAD] * 3


def test_sanitizer_clean(tmp_path_factory, tmp_path):
    """The malformed set and a few thousand randomly damaged responses under ASan/UBSan (any finding aborts)."""
    exe = emu_exe(tmp_path_factory, sanitize=True)
    rng = random.Random(17)
    (rout, roff, rlens, rst), dom = fuzz_set(5)
    valid = [bytes(rout[roff[i]:roff[i] + rlens[i]]) for i in range(len(rst)) if rst[i] == 0]
    rel = relay_set(6, n=600)
    valid += [bytes(rel[0][rel[1][i]:rel[1][i] + rel[2][i]]) for i in range(len(rel[3])) if rel[3][i] == 0]
    valid += hand_responses()
    resps = [G.mutate(rng, v) for v in valid for _ in range(3)] + list(malformed_responses().values())
    rs = pack_set(resps)
    got = emu_log(exe, rs, dom, tmp_path)
    assert sum(1 for _, _, s in got if s & L.BAD) > 500 and sum(1 for h, _, _ in got if h) > 500
    # where both sides accept a damaged response they render the same record.  dnspython checks the RDATA of types the
    # record never reads (MX, SOA, ...) and the device does not, so only the device may accept where it refuses.
    want = L.log_set(*rs, dom)
    both = [i for i, (g, w) in enumerate(zip(got, want)) if g[0] and w[0]]
    assert len(both) > 500 and all(got[i] == want[i] for i in both)
    assert not [i for i, (g, w) in enumerate(zip(got, want)) if w[0] and not g[0]]          # the restatement accepts only what the device does
    assert_same_log(emu_log(exe, pack_set(valid), dom, tmp_path), L.log_set(*pack_set(valid), dom))
