"""Forward / match corpora (DESIGN.md section 14): misses at every filter shape of test_recursion_filter.py, upstream
tables for them, and response sets — hand-written cases plus generated answers for random misses."""
import random
import struct

import forward_ref as R
import fuzzgen
from binder_b200 import synth
from test_recursion_filter import FILTERS, filter_queries

UP_IPS = ['127.0.0.1', '10.0.0.2', '10.0.0.3', '192.168.7.9']


def upstream_table(dcs, rng):
    """Upstreams for every datacenter but (when there are several) one, some with two resolvers."""
    ups = []
    for k in range(len(dcs)):
        if len(dcs) > 1 and k == len(dcs) - 1:
            continue
        for _ in range(rng.choice([1, 1, 2])):
            ups.append((rng.choice(UP_IPS), rng.choice([53, 5353, 40000 + k]), k))
    return ups


def misses(fi, seed=0):
    """The filter's queries plus EDNS, non-QUERY opcodes, 255-byte names, PTR and undecodable packets."""
    region, dcs, _ = FILTERS[fi]
    rng = random.Random(1000 * fi + seed)
    _, info = fuzzgen.gen_zone(900 + fi, n_top=25)
    pkts = [p for p in filter_queries(fi, info)]
    dom = region.lstrip('.')
    tops = list(dcs) + ['zz', 'Web']
    for i in range(300):
        top = rng.choice(tops)
        name = 'h%d.%s.%s' % (i, top, dom) if top else dom
        pkts.append(synth.make_query(name, rng.choice(['A', 'SRV', 'A']), qid=rng.randrange(65536), rd=rng.random() < 0.9,
                                     edns=rng.choice([None, 512, 1200, 4096]), opcode=rng.choice([0, 0, 0, 1, 2, 4])))
    for i in range(20):                                     # 255-byte names ending in a datacenter label
        top = (dcs[i % len(dcs)] if dcs else 'web').encode()
        tail = [top] + [l.encode() for l in dom.split('.') if l]
        used = sum(1 + len(l) for l in tail) + 1
        head = []
        while used + 64 <= 255:
            head.append(b'a' * 63)
            used += 64
        if used < 255:
            head.append(b'b' * (255 - used - 1))
        pkts.append(synth.make_query(None, 'A', qid=i, labels=head + tail))
    pkts += [synth.make_query('%d.%d.0.10.in-addr.arpa' % (i, i), 'PTR', qid=i, edns=1200) for i in range(20)]
    good = synth.make_query('x.web.foo.com', 'A', qid=3)
    pkts += [good[:11], b'', good[:2] + b'\x81\x00' + good[4:], synth.make_query('x.web.foo.com', 'A', qclass=3)]
    return pkts


def answer_for(upq, rng):
    """A response to the upstream query upq (same ID, opcode and question), with one A record or none."""
    an = rng.random() < 0.8
    hdr = struct.pack('>HHHHHH', struct.unpack('>H', upq[:2])[0], 0x8400 | (upq[2] & 0x78) << 8, 1, 1 if an else 0, 0, 0)
    rr = b'\xc0\x0c' + struct.pack('>HHIH', 1, 1, 60, 4) + bytes(rng.randrange(256) for _ in range(4)) if an else b''
    return hdr + upq[12:] + rr


def responses(ups, routes, msgs, rng, key):
    """Answers from the right upstream for most forwarded misses, some duplicated or from the wrong place, plus noise."""
    out = []
    for j, (rt, m) in enumerate(zip(routes, msgs)):
        if not m or rng.random() < 0.15:
            continue
        cand = [(a, p) for a, p, d in ups if rt == R.R_PTR or d == rt] or [(UP_IPS[0], 53)]
        src = rng.choice(cand)
        if rng.random() < 0.1:
            src = (src[0], src[1] + 1)                      # wrong port
        data = answer_for(m, rng)
        out.append((data, src))
        if rng.random() < 0.1:
            out.append((data[:2] + b'\x84\x05' + data[4:], rng.choice(cand)))   # a second answer: loses to the first
    rng.shuffle(out)
    out += [(bytes(rng.randrange(256) for _ in range(rng.randrange(40))), (UP_IPS[0], 53)) for _ in range(30)]
    return out


def hand_written(ups, pkts, routes, msgs, key):
    """Named response sets for the first forwarded miss of each kind; -> {name: [(bytes, (ip, port))]}."""
    j = next(i for i, (rt, m) in enumerate(zip(routes, msgs)) if m and rt < R.R_PTR)
    m = msgs[j]
    src = next((a, p) for a, p, d in ups if d == routes[j])
    ans = answer_for(m, random.Random(1))
    qn_end = 12 + len(m) - 16
    cases = {
        'duplicate': [(ans, src), (ans[:3] + b'\x05' + ans[4:], src)],
        'wrong_ip': [(ans, ('10.77.0.1', src[1]))],
        'wrong_port': [(ans, (src[0], (src[1] + 7) & 0xFFFF))],
        'foreign_id': [(struct.pack('>H', R.fid(key ^ 1, j)) + ans[2:], src)],
        'id_past_n': [(struct.pack('>H', R.fid(key, len(pkts) + 5)) + ans[2:], src)] if len(pkts) + 5 < 65536 else [],
        'qr0': [(ans[:2] + bytes([ans[2] & 0x7F]) + ans[3:], src)],
        'short': [(ans[:11], src)],
        'case': [(ans[:13] + bytes([ans[13] ^ 0x20]) + ans[14:], src)] if 65 <= (ans[13] | 0x20) <= 122 and ans[12] else [],
        'type': [(ans[:qn_end] + b'\x00\x63' + ans[qn_end + 2:], src)],
        'class': [(ans[:qn_end + 2] + b'\x00\x03' + ans[qn_end + 4:], src)],
        'compressed': [(ans[:12] + b'\xc0\x0c' + ans[qn_end:], src)],
        'no_question': [(ans[:4] + b'\x00\x00' + ans[6:], src)],
    }
    two = [(a, p) for a, p, d in ups if d == routes[j]]
    if len(two) > 1:
        cases['two_upstreams'] = [(ans, two[1]), (ans[:3] + b'\x05' + ans[4:], two[0])]
    none = [i for i, (rt, mm) in enumerate(zip(routes, msgs)) if rt == R.R_NONE and mm]
    if none:
        mm = msgs[none[0]]
        cases['none_route'] = [(answer_for(mm, random.Random(2)), (a, p)) for a, p, _ in ups]
    return j, cases


def pack(items):
    """[(bytes, (ip, port))] -> (data, off, ip u32, port u16) as the match calls take them."""
    import numpy as np
    from binder_b200.engine import ip_u32
    data, off = synth.pack_batch([b for b, _ in items]) if items else (np.zeros(16, np.uint8), np.zeros(1, np.uint32))
    return (data, off, np.array([ip_u32(a) for _, (a, _) in items], dtype=np.uint32),
            np.array([p for _, (_, p) in items], dtype=np.uint16))
