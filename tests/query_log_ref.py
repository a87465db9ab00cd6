"""Independent restatement of binder's per-query "DNS query" record (lib/server.js:509-591, DESIGN.md section 15): the
response decoded with dnspython, stripSuffix applied to the dotted strings, the record rendered with json.dumps as
bunyan's JSON.stringify writes it.  Test infrastructure, not product: tests compare the device source (log_device.cuh,
through tests/native/emu_log.cpp) and the log kernel against it."""
import json
import struct

import dns.exception
import dns.ipv6
import dns.message
import dns.rdatatype

MNEMONIC = {1: 'A', 2: 'NS', 5: 'CNAME', 6: 'SOA', 12: 'PTR', 15: 'MX', 16: 'TXT', 28: 'AAAA', 33: 'SRV', 41: 'OPT',
            252: 'AXFR', 255: 'ANY'}
BAD = 1 << 22


def type_name(t):
    return MNEMONIC.get(t, 'TYPE%d' % t)


def dotted(name):
    """query.name(): the raw labels joined by '.', latin-1, no escaping; the root is ''."""
    return '.'.join(l.decode('latin-1') for l in name.labels if l)


def strip_suffix(suffix, s):
    idx = s.rfind(suffix)
    return s[:len(s) - len(suffix)] + '...' if idx >= 0 and idx + len(suffix) == len(s) else s


def ipv6_text(b):
    """RFC 5952: lower-case hex, the first longest run of two or more zero groups as '::', no embedded IPv4."""
    g = struct.unpack('>8H', b)
    best, run = (8, 0), 0
    for i in range(8):
        run = run + 1 if g[i] == 0 else 0
        if run > best[1]:
            best = (i - run + 1, run)
    if best[1] < 2:
        return ':'.join('%x' % x for x in g)
    z0, zn = best
    return ':'.join('%x' % x for x in g[:z0]) + '::' + ':'.join('%x' % x for x in g[z0 + zn:])


def dumps(v):
    return json.dumps(v, ensure_ascii=False, separators=(',', ':'))


def _address(rd):
    if rd.rdtype == dns.rdatatype.A:
        return rd.address
    return ipv6_text(dns.ipv6.inet_aton(rd.address))


def _obj(rd):
    if rd.rdtype in (dns.rdatatype.PTR, dns.rdatatype.CNAME):
        return {'target': dotted(rd.target), 'type': type_name(rd.rdtype)}
    if rd.rdtype == dns.rdatatype.TXT:
        return {'target': b''.join(rd.strings).decode('latin-1'), 'type': 'TXT'}
    return {'type': type_name(rd.rdtype)}


def _pointer_free_question(wire):
    pos = 12
    while pos < len(wire):
        c = wire[pos]
        if c == 0:
            return True
        if c > 63:
            return False
        pos += 1 + c
    return False


def record(wire, dns_domain):
    """One answered response -> (head bytes, body bytes, summary), or None when it breaks a decode rule."""
    wire = bytes(wire)
    if len(wire) < 12 or not wire[2] & 0x80 or struct.unpack('>H', wire[4:6])[0] != 1 or not _pointer_free_question(wire):
        return None
    try:                  # the opcode does not enter the record; dnspython would parse an UPDATE's sections differently
        m = dns.message.from_wire(wire[:2] + bytes([wire[2] & 0x87]) + wire[3:], one_rr_per_rrset=True, raise_on_truncation=False, ignore_trailing=True)
    except (dns.exception.DNSException, ValueError, struct.error):
        return None
    # a record read as a type other than the one the log renders (a non-IN class) is beyond what this restatement covers
    if any(rrset.rdtype in (1, 5, 12, 16, 28, 33) and not hasattr(rd, 'target' if rrset.rdtype in (5, 12, 33) else
                                                                    'strings' if rrset.rdtype == 16 else 'address')
           for rrset in m.answer + m.additional for rd in rrset):
        return None
    suffix = '.' + dns_domain if dns_domain else None
    strip = (lambda s: strip_suffix(suffix, s)) if suffix else (lambda s: s)
    q = m.question[0]
    edns = m.edns >= 0
    answers = []
    for rrset in m.answer:
        for rd in rrset:
            t = type_name(rd.rdtype)
            if t == 'SRV':
                answers.append('SRV %s:%d' % (strip(dotted(rd.target)), rd.port))
            elif t in ('A', 'AAAA'):
                answers.append('%s %s' % (t, _address(rd)))
            else:
                answers.append(_obj(rd))
    additional = []
    for rrset in m.additional:
        for rd in rrset:
            t = type_name(rd.rdtype)
            if t in ('A', 'AAAA'):
                additional.append('%s %s %s' % (strip(dotted(rrset.name)), t, _address(rd)))
            else:
                additional.append(_obj(rd))
    rcode = wire[3] & 15
    head = '"query":%s,"edns":%s' % (dumps({'name': dotted(q.name), 'type': type_name(q.rdtype)}), 'true' if edns else 'false')
    body = '"rcode":%d,"answers":%s,"additional":%s' % (rcode, dumps(answers), dumps(additional))
    summary = q.rdtype | rcode << 16 | edns << 20 | ((wire[2] >> 1) & 1) << 21
    return head.encode(), body.encode(), summary


def log_set(out, out_off, out_len, status, dns_domain):
    """A result set -> [(head, body, summary)]: b'' fragments for a response without a record (a miss, a dropped query)
    and for one that breaks a decode rule (summary = the bad bit)."""
    out = bytes(out)
    res = []
    for i in range(len(status)):
        o, l = int(out_off[i]), int(out_len[i])
        if status[i] != 0:
            res.append((b'', b'', 0))
            continue
        r = record(out[o:o + l], dns_domain) if o + l <= len(out) else None
        res.append(r if r else (b'', b'', BAD))
    return res
