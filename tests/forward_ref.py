"""TEST INFRASTRUCTURE — an independent Python restatement of the recursion forward and match (DESIGN.md section 14).

Written from recursion.py's _exchange and the match rules of include/binder_b200.h, not from either native
implementation: the question is parsed here, the datacenter is found with the same string operations as Recursion's
quick rejects (recursion.py's upstreams()), the IDs come from a separately written Feistel network."""
import struct

QT_PTR = 12
R_PTR, R_NONE, N_ROUTES = 16, 17, 18
M32 = 0xFFFFFFFF


def fmix32(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def round_keys(key):
    lo, hi = key & M32, (key >> 32) & M32
    return [fmix32(lo ^ fmix32((hi + 0x9E3779B9 * (i + 1)) & M32)) for i in range(4)]


def fid(key, j):
    k = round_keys(key)
    left, right = j >> 8, j & 0xFF
    for i in range(4):
        left, right = right, left ^ (fmix32(right ^ k[i]) & 0xFF)
    return left << 8 | right


def fid_inv(key, x):
    k = round_keys(key)
    left, right = x >> 8, x & 0xFF
    for i in reversed(range(4)):
        left, right = right ^ (fmix32(left ^ k[i]) & 0xFF), left
    return left << 8 | right


def parse_query(pkt):
    """The resolve path's decode() acceptance -> (question bytes, qtype, dotted name) or None."""
    if len(pkt) < 12 or len(pkt) > 65535 or pkt[2] & 0x80:
        return None
    qd, an, ns, ar = struct.unpack('>HHHH', pkt[4:12])
    if qd != 1 or an or ns or ar > 1:
        return None
    pos, labels = 12, []
    while True:
        if pos >= len(pkt):
            return None
        c = pkt[pos]
        if c == 0:
            pos += 1
            break
        if c > 63 or pos + 1 + c > len(pkt):
            return None
        labels.append(pkt[pos + 1:pos + 1 + c].decode('latin-1'))
        pos += 1 + c
        if pos - 12 + 1 > 255:
            return None
    if pos + 4 > len(pkt):
        return None
    qtype, qclass = struct.unpack('>HH', pkt[pos:pos + 4])
    if qclass != 1:
        return None
    end = pos + 4
    if ar:
        if end + 11 > len(pkt) or pkt[end] != 0 or struct.unpack('>H', pkt[end + 1:end + 3])[0] != 41:
            return None
        if end + 11 + struct.unpack('>H', pkt[end + 9:end + 11])[0] > len(pkt):
            return None
    return pkt[12:end], qtype, '.'.join(labels)


def route_of(region, dcs, upstreams, qtype, name):
    if qtype == QT_PTR:
        return R_PTR if upstreams else R_NONE
    if name.find(region, max(len(name) - len(region), 0)) == -1:
        return R_NONE
    p = name[:max(len(name) - len(region) - 1, 0)]
    dc = p[p.rfind('.') + 1:]
    if dc not in dcs:
        return R_NONE
    k = dcs.index(dc)
    return k if any(d == k for _, _, d in upstreams) else R_NONE


def forward(region, dcs, upstreams, pkts, key):
    """-> (route per miss, upstream query per miss)."""
    routes, msgs = [], []
    for j, pkt in enumerate(pkts):
        q = parse_query(pkt)
        if q is None:
            routes.append(R_NONE)
            msgs.append(b'')
            continue
        question, qtype, name = q
        routes.append(route_of(region, dcs, upstreams, qtype, name))
        flags = struct.unpack('>H', pkt[2:4])[0] & 0x7800
        msgs.append(struct.pack('>HHHHHH', fid(key, j), flags, 1, 0, 0, 0) + question)
    return routes, msgs


def grouped(routes):
    """Stable grouping by route -> (order, group_off)."""
    order, group_off = [], []
    for r in range(N_ROUTES):
        group_off.append(len(order))
        order += [j for j, x in enumerate(routes) if x == r]
    group_off.append(len(order))
    return order, group_off


def match(upstreams, responses, pkts, routes, key):
    """responses: [(bytes, (ip, port))] in arrival order -> the accepted response per miss (b'' when none)."""
    out = [None] * len(pkts)
    for data, (ip, port) in responses:
        if len(data) < 12 or not data[2] & 0x80:
            continue
        j = fid_inv(key, struct.unpack('>H', data[:2])[0])
        if j >= len(pkts) or out[j] is not None or routes[j] == R_NONE:
            continue
        if not any(a == ip and p == port and (routes[j] == R_PTR or d == routes[j]) for a, p, d in upstreams):
            continue
        if struct.unpack('>H', data[4:6])[0] == 0:
            continue
        q = parse_query(pkts[j])
        if q is None or data[12:12 + len(q[0])] != q[0]:
            continue
        out[j] = data
    return [x or b'' for x in out]
