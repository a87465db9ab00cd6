"""TEST INFRASTRUCTURE — the recursion relay restated at the semantic level (rcode + answer tuples), independently of
tests/native/relay_oracle.cpp, so that the two can be cross-checked (DESIGN.md section 13, lib/recursion.js:287-327)."""
from binder_ref import NOTIMP_DEFAULT, RCODE

# what recursion.js re-wraps (:299-315), by type number
RELAY_TYPES = {1: 'A', 28: 'AAAA', 16: 'TXT', 12: 'PTR', 5: 'CNAME', 33: 'SRV'}


class _Malformed(Exception):
    pass


def _up_name(pkt, pos, budget=255):
    """(labels, position after the name's own bytes) of the possibly compressed name at pos."""
    labels, wire, after = [], 1, None
    while True:
        if pos >= len(pkt):
            raise _Malformed('name runs off the packet')
        c = pkt[pos]
        if c >= 0xC0:
            if pos + 1 >= len(pkt):
                raise _Malformed('cut pointer')
            target = ((c & 0x3F) << 8) | pkt[pos + 1]
            if target >= pos:
                raise _Malformed('pointer not strictly backwards')
            if after is None:
                after = pos + 2
            pos = target
        elif c >= 0x40:
            raise _Malformed('label type')
        elif c == 0:
            return tuple(labels), (pos + 1 if after is None else after)
        else:
            if pos + 1 + c > len(pkt):
                raise _Malformed('label runs off the packet')
            labels.append(bytes(pkt[pos + 1:pos + 1 + c]))
            wire += 1 + c
            if wire > budget:
                raise _Malformed('name over 255 bytes')
            pos += 1 + c


def upstream_answers(pkt):
    """The upstream response's answer records as (type number, class, ttl, data), or None when the
    response is empty or malformed (the lookup failed: recursion.js keeps answers = [])."""
    pkt = bytes(pkt)
    if len(pkt) < 12 or len(pkt) > 65535 or not pkt[2] & 0x80:
        return None
    qd, an = int.from_bytes(pkt[4:6], 'big'), int.from_bytes(pkt[6:8], 'big')
    try:
        pos = 12
        for _ in range(qd):
            _, pos = _up_name(pkt, pos)
            if pos + 4 > len(pkt):
                raise _Malformed('question')
            pos += 4
        recs = []
        for _ in range(an):
            _, pos = _up_name(pkt, pos)
            if pos + 10 > len(pkt):
                raise _Malformed('rr header')
            t, k, ttl, rdlen = int.from_bytes(pkt[pos:pos + 2], 'big'), int.from_bytes(pkt[pos + 2:pos + 4], 'big'), \
                int.from_bytes(pkt[pos + 4:pos + 8], 'big'), int.from_bytes(pkt[pos + 8:pos + 10], 'big')
            rd, end = pos + 10, pos + 10 + rdlen
            if end > len(pkt):
                raise _Malformed('rdata')
            data = bytes(pkt[rd:end])
            if t in (1, 28) and rdlen != (4 if t == 1 else 16):
                raise _Malformed('address length')
            if t in (5, 12):
                data, after = _up_name(pkt, rd)
                if after > end:
                    raise _Malformed('name past rdata')
            elif t == 33:
                if rdlen < 7:
                    raise _Malformed('srv length')
                target, after = _up_name(pkt, rd + 6)
                if after > end:
                    raise _Malformed('name past rdata')
                data = (int.from_bytes(pkt[rd:rd + 2], 'big'), int.from_bytes(pkt[rd + 2:rd + 4], 'big'),
                        int.from_bytes(pkt[rd + 4:rd + 6], 'big'), target)
            recs.append((t, k, ttl, data))
            pos = end
        return recs
    except _Malformed:
        return None


def relay(labels, upstream):
    """Recursion.prototype.resolve's respond() for a query with these QNAME labels and this upstream
    response -> (rcode, answers), answers = [(owner, ttl, type name, data)] in upstream order (the reply
    keeps the longest prefix that fits, DESIGN.md section 3)."""
    name = '.'.join(l.decode('latin-1') for l in labels)
    recs = upstream_answers(upstream) or []
    if not recs:
        return RCODE['refused'], ()
    answers = tuple((name, ttl, RELAY_TYPES[t], data) for t, k, ttl, data in recs if k == 1 and t in RELAY_TYPES)
    return (0 if answers else NOTIMP_DEFAULT), answers
