"""Relay corpora (DESIGN.md section 13): client queries paired with upstream responses.  Upstreams are built with
dnspython, an independent DNS codec, except where it cannot express the case (compressed SRV targets, non-IN classes,
answers that expand past 65,535 bytes once decompressed), which a small raw packer writes; malformed upstreams are
written by hand, and `mutate` derives random damage from valid ones."""
import random
import struct

import dns.flags
import dns.message
import dns.name
import dns.rdata
import dns.rdataclass
import dns.rdatatype
import dns.rrset

import relay_ref
from binder_b200 import synth

IN = dns.rdataclass.IN


def rrset(owner, ttl, rdtype, text, rdclass=IN):
    rd = dns.rdata.from_text(rdclass, rdtype, text, origin=dns.name.root, relativize=False)
    return dns.rrset.from_rdata(dns.name.from_text(owner or '.'), ttl, rd)


def dnspython_upstream(qname, qtype, answers, rcode=0, authority=(), qid=0):
    """A response packet from dnspython; each answer RR is its own RRset, so order and TTLs stay as given."""
    m = dns.message.Message(id=qid)
    m.flags = dns.flags.QR | dns.flags.AA
    m.set_rcode(rcode)
    m.question = [dns.rrset.RRset(dns.name.from_text(qname or '.'), IN, qtype)]
    m.answer = list(answers)
    m.authority = list(authority)
    return m.to_wire()


def raw_upstream(qwire, qtype, rrs, flags=0x8400, qd=1):
    """Packer for what dnspython will not write: rrs = [(owner wire, type, class, ttl, rdata bytes)]; the question
    (qwire) starts at offset 12, so b'\\xc0\\x0c' names it."""
    pkt = struct.pack('>HHHHHH', 0x4242, flags, qd, len(rrs), 0, 0)
    if qd:
        pkt += qwire + struct.pack('>HH', qtype, 1)
    for owner, t, k, ttl, rd in rrs:
        pkt += owner + struct.pack('>HHIH', t, k, ttl, len(rd)) + rd
    return pkt


def _label(rng, n=None):
    n = n or rng.randint(1, 12)
    return ''.join(rng.choice('abcdefghijklmnopqrstuvwxyzABCDEF0123456789-') for _ in range(n))


def _name(rng, parts=None):
    return '.'.join(_label(rng) for _ in range(parts or rng.randint(1, 4))) + '.dc2.example.com'


def _ip4(rng):
    return '.'.join(str(rng.randrange(256)) for _ in range(4))


def _ip6(rng):
    return ':'.join('%x' % rng.randrange(65536) for _ in range(8))


def _query(rng, name, qtype, edns=None, labels=None):
    if edns is None:
        edns = rng.choice([None, None, 512, 1000, 1200, 4096, 100])
    return synth.make_query(name, int(dns.rdatatype.from_text(qtype)), qid=rng.randrange(65536), rd=rng.random() < 0.9, edns=edns, labels=labels)


KINDS = ('a', 'cname_a', 'srv3', 'srv_dns', 'aaaa', 'txt', 'ptr', 'dropped_mix', 'only_mx', 'non_in', 'nxdomain',
         'empty', 'many', 'expand')


def relay_case(rng, kind, tcp=False):
    """(query packet, upstream packet) of one kind."""
    name = _name(rng)
    ttl = lambda: rng.choice([0, 1, 30, 3600, 86400, 2 ** 31 - 1, 2 ** 32 - 1])       # noqa: E731
    if kind == 'a':
        q = _query(rng, name, 'A')
        return q, dnspython_upstream(name, 1, [rrset(name, ttl(), 'A', _ip4(rng))], qid=rng.randrange(65536))
    if kind == 'cname_a':                     # a chain whose owners are not the query's name
        a1, a2 = 'alias.' + _name(rng), 'real.' + _name(rng)
        ans = [rrset(name, ttl(), 'CNAME', a1), rrset(a1, ttl(), 'CNAME', a2), rrset(a2, ttl(), 'A', _ip4(rng))]
        return _query(rng, name, 'A'), dnspython_upstream(name, 1, ans)
    if kind == 'srv3':                        # compressed targets: a label + a pointer to the question's name
        sname = '_http._tcp.' + name
        q = _query(rng, sname, 'SRV')
        qwire = synth.encode_name(sname)
        rrs = []
        for i in range(3):
            lab = _label(rng).encode()
            rd = struct.pack('>HHH', rng.randrange(65536), rng.randrange(65536), rng.randrange(65536)) + \
                bytes([len(lab)]) + lab + b'\xc0\x0c'
            rrs.append((b'\xc0\x0c', 33, 1, ttl(), rd))
        return q, raw_upstream(qwire, 33, rrs)
    if kind == 'srv_dns':
        sname = '_ldap._udp.' + name
        ans = [rrset(sname, ttl(), 'SRV', '%d %d %d %s' % (rng.randrange(65536), rng.randrange(65536), rng.randrange(65536),
                                                             _name(rng) + '.')) for _ in range(rng.randint(1, 4))]
        return _query(rng, sname, 'SRV'), dnspython_upstream(sname, 33, ans)
    if kind == 'aaaa':
        ans = [rrset(name, ttl(), 'AAAA', _ip6(rng)) for _ in range(rng.randint(1, 3))]
        return _query(rng, name, 'AAAA'), dnspython_upstream(name, 28, ans)
    if kind == 'txt':
        ans = [rrset(name, ttl(), 'TXT', ' '.join('"%s"' % _label(rng, rng.randint(1, 60)) for _ in range(rng.randint(1, 4))))
               for _ in range(rng.randint(1, 3))]
        return _query(rng, name, 'TXT'), dnspython_upstream(name, 16, ans)
    if kind == 'ptr':
        pname = '%d.%d.0.10.in-addr.arpa' % (rng.randrange(256), rng.randrange(256))
        ans = [rrset(pname, ttl(), 'PTR', _name(rng) + '.')]
        return _query(rng, pname, 'PTR'), dnspython_upstream(pname, 12, ans)
    if kind == 'dropped_mix':                 # MX, NS, SOA in the answer section between kept records
        ans = [rrset(name, ttl(), 'MX', '10 mail.' + name + '.'), rrset(name, ttl(), 'A', _ip4(rng)),
               rrset(name, ttl(), 'NS', 'ns1.' + name + '.'),
               rrset(name, ttl(), 'SOA', 'ns1.%s. host.%s. 1 2 3 4 5' % (name, name)), rrset(name, ttl(), 'A', _ip4(rng))]
        rng.shuffle(ans)
        return _query(rng, name, 'A'), dnspython_upstream(name, 1, ans)
    if kind == 'only_mx':                     # every answer dropped: no error set, nothing added -> NOTIMP
        ans = [rrset(name, ttl(), 'MX', '%d mx%d.%s.' % (i, i, name)) for i in range(rng.randint(1, 3))]
        return _query(rng, name, 'MX'), dnspython_upstream(name, 15, ans)
    if kind == 'non_in':                      # CH / HS / class 254 answers are dropped, IN ones kept
        qwire = synth.encode_name(name)
        rrs = [(b'\xc0\x0c', rng.choice([1, 16]), rng.choice([3, 4, 254]), ttl(), b'\x01\x02\x03\x04')]
        if rng.random() < 0.5:
            rrs.append((b'\xc0\x0c', 1, 1, ttl(), bytes(rng.randrange(256) for _ in range(4))))
        rng.shuffle(rrs)
        return _query(rng, name, 'A'), raw_upstream(qwire, 1, rrs)
    if kind == 'nxdomain':
        auth = [rrset('example.com', 300, 'SOA', 'ns.example.com. h.example.com. 1 2 3 4 5')]
        return _query(rng, name, 'A'), dnspython_upstream(name, 1, [], rcode=3, authority=auth)
    if kind == 'empty':
        return _query(rng, name, rng.choice(['A', 'SRV', 'PTR'])), b''
    if kind == 'many':                        # past 512 and 1,200 bytes over UDP
        ans = [rrset(name, ttl(), 'A', _ip4(rng)) if rng.random() < 0.5 else rrset(name, ttl(), 'TXT', '"%s"' % _label(rng, 40))
               for _ in range(rng.randint(20, 120))]
        return _query(rng, name, 'A'), dnspython_upstream(name, 1, ans)
    if kind == 'expand':                      # 2-byte pointers expand to ~200-byte names: past 65,535 bytes over TCP
        long_name = '.'.join(_label(rng, 60) for _ in range(3))
        qwire = synth.encode_name(long_name)
        rrs = [(b'\xc0\x0c', 5, 1, ttl(), b'\xc0\x0c') for _ in range(rng.randint(400, 600))]
        return _query(rng, long_name, 'A', edns=rng.choice([None, 1200])), raw_upstream(qwire, 1, rrs)
    raise ValueError(kind)


def gen_relays(seed, n):
    """n (query, upstream) pairs over every kind, a few with a root or in-label-dot QNAME."""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        q, u = relay_case(rng, KINDS[i % len(KINDS)])
        if rng.random() < 0.02:               # root QNAME: the owner is the root name itself
            q = _query(rng, '', 'A')
        elif rng.random() < 0.02:             # a '.' inside a label: the owner is still the QNAME (a pointer)
            q = _query(rng, None, 'A', labels=[b'a.b', b'dc2', b'example', b'com'])
        out.append((q, u))
    return out


def malformed_upstreams(rng=None):
    """Hand-written damage; every one of these must be treated as a failed lookup (REFUSED)."""
    qwire = synth.encode_name('h1.dc2.example.com')
    q = struct.pack('>HHHHHH', 7, 0x8400, 1, 1, 0, 0) + qwire + struct.pack('>HH', 1, 1)
    rr = lambda owner, t, rd, k=1: owner + struct.pack('>HHIH', t, k, 60, len(rd)) + rd       # noqa: E731
    a_ok = rr(b'\xc0\x0c', 1, b'\x01\x02\x03\x04')
    return {
        'forward_pointer': q + rr(b'\xc0\x34', 1, b'\x01\x02\x03\x04') + b'\x02xx\x00',
        'pointer_loop': q + rr(b'\x01a\xc0\x24', 1, b'\x01\x02\x03\x04'),
        'self_pointer': q + rr(b'\xc0\x24', 1, b'\x01\x02\x03\x04'),
        'pointer_past_end': q + rr(b'\xc0\x0c', 5, b'\x01a\xc0'),
        'cut_pointer_owner': q + b'\xc0',
        'label_over_63': q + rr(b'\x40' + b'a' * 64 + b'\x00', 1, b'\x01\x02\x03\x04'),
        'label_type_0x80': q + rr(b'\x80\x00', 1, b'\x01\x02\x03\x04'),
        'name_over_255': q + rr((b'\x3f' + b'a' * 63) * 4 + b'\x00', 1, b'\x01\x02\x03\x04'),
        'name_over_255_via_pointers': q[:6] + b'\x00\x02' + q[8:] + rr(b'\x3fa' + b'b' * 62 + b'\xc0\x0c', 16, b'\x01x') +
            rr(b'\x3fc' + b'd' * 62 + b'\x3fe' + b'f' * 62 + b'\x3fg' + b'h' * 62 + b'\xc0\x24', 1, b'\x01\x02\x03\x04'),
        'rdlen_past_end': q + b'\xc0\x0c' + struct.pack('>HHIH', 1, 1, 60, 40) + b'\x01\x02\x03\x04',
        'a_rdlen_5': q + rr(b'\xc0\x0c', 1, b'\x01\x02\x03\x04\x05'),
        'aaaa_rdlen_4': q + rr(b'\xc0\x0c', 28, b'\x01\x02\x03\x04'),
        'srv_rdlen_6': q + rr(b'\xc0\x0c', 33, b'\x00\x01\x00\x02\x00\x03'),
        'srv_name_past_rdlen': q + rr(b'\xc0\x0c', 33, b'\x00\x01\x00\x02\x00\x03\x05ab') + b'cde\x00',
        'cname_name_past_rdlen': q + rr(b'\xc0\x0c', 5, b'\x03abc') + b'\x00',
        'bad_after_good': q[:6] + b'\x00\x02' + q[8:] + a_ok + rr(b'\xc0\x0c', 1, b'\x01\x02\x03'),
        'answer_count_too_high': q[:6] + b'\x00\x02' + q[8:] + a_ok,
        'question_cut': struct.pack('>HHHHHH', 7, 0x8400, 1, 1, 0, 0) + qwire[:5],
        'truncated_header': q[:11],
        'qr_zero': q[:2] + b'\x04\x00' + q[4:] + a_ok,
        'over_65535': q + a_ok + b'\x00' * (65536 - len(q) - len(a_ok)),
    }


def mutate(rng, pkt):
    """Random damage to a valid packet: flipped bytes, a cut, or a byte run inserted."""
    b = bytearray(pkt)
    if not b:
        return bytes(rng.randrange(256) for _ in range(rng.randint(0, 40)))
    for _ in range(rng.randint(1, 4)):
        op = rng.random()
        if op < 0.6 and b:
            b[rng.randrange(len(b))] = rng.choice([0, 0xC0, 0x3F, 0x40, 0xFF, rng.randrange(256)])
        elif op < 0.8:
            del b[rng.randrange(len(b) + 1):]
        else:
            i = rng.randrange(len(b) + 1)
            b[i:i] = bytes(rng.randrange(256) for _ in range(rng.randint(1, 8)))
    return bytes(b)


def pack_pairs(pairs):
    """[(query, upstream)] -> (q_data, q_off, up_data, up_off), each byte array padded for 16-byte reads."""
    q_data, q_off = synth.pack_batch([q for q, _ in pairs])
    up_data, up_off = synth.pack_batch([u for _, u in pairs])
    return q_data, q_off, up_data, up_off


def semantic(pair):
    """relay_ref's restatement for one pair -> (rcode, answers)."""
    labels = []
    q = pair[0]
    pos = 12
    while q[pos]:
        labels.append(bytes(q[pos + 1:pos + 1 + q[pos]]))
        pos += 1 + q[pos]
    return relay_ref.relay(labels, pair[1])
