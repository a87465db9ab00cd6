"""Seeded zones and queries at the DNS length limits, under dnsDomains of many shapes (tests/test_name_limits.py).

The rest of the suite serves foo.com, dc1.example.com and example.com, whose '.' + dnsDomain lengths (8, 16, 12) are all
multiples of four, with short names inside.  The zones here put names on both sides of every length the builder and the
kernel branch on:
  - the word-wise suffix gate of lean_query compares '.' + dnsDomain (as wire labels) one 32-bit word at a time and masks
    the last, partial word: DOMAINS cover every length mod 4, one label, many labels, a 63-byte label, and the longest
    dnsDomain whose SOA rname (hostmaster.<dnsDomain>) still fits 255 bytes;
  - lean_query takes names of at most 64 wire bytes (63 before the terminator) whose key part is at most 48 bytes; keys
    over 20 bytes live in the arena;
  - a name is at most 255 wire bytes: hosts sit at 254 and 255, and one at 256 that only its PTR can reach;
  - "_srvce._proto" fits the service header up to 11 wire bytes and lives in the arena beyond (SVC_SP_EXT);
  - a service child is a znode path component and may contain dots: its wire name runs up to 255 - dom_wl bytes
    (dom_wl: the service's own fqdn as wire labels + terminator), its additional RR to 268 bytes.
"""
import json
import random

from binder_b200 import synth

ALNUM = 'abcdefghijklmnopqrstuvwxyz0123456789'


def _word(rng, n):
    """n characters of [a-z0-9-], not starting or ending with '-'."""
    s = [rng.choice(ALNUM + '-') for _ in range(n)]
    s[0] = rng.choice(ALNUM)
    s[-1] = rng.choice(ALNUM)
    return ''.join(s)


def _longest_domain():
    rng = random.Random(242)
    return '.'.join(_word(rng, n) for n in (63, 63, 63, 50))


LONGEST_DOMAIN = _longest_domain()            # 242 characters: hostmaster. + it is 253 wire bytes + terminator
TOO_LONG_DOMAIN = LONGEST_DOMAIN + 'x'       # 243: its SOA rname no longer fits 255 bytes
assert len(LONGEST_DOMAIN) == 242

# name -> dnsDomain; '.' + dnsDomain is as many bytes as dnsDomain's wire labels without the terminator
DOMAINS = {
    'corp': 'corp',                                                          # 5 = 1 mod 4, one label
    'foo.co': 'foo.co',                                                      # 7 = 3 mod 4
    'five': 'x.y.z.w.v',                                                     # 10 = 2 mod 4, five one-letter labels
    'abc.example': 'abc.example',                                            # 12 = 0 mod 4
    'label63': 'q' * 31 + '-' + 'r' * 31 + '.ex',                            # 67: a 63-byte label
    'lean-edge': 'lab-1.us-west-2a.compute.example-corporation.internal.net',  # 58: keys of 2..5 bytes stay on the lean path
    'longest': LONGEST_DOMAIN,                                               # 243
    'not-lean': 'f+o.com',                                                   # '+' is outside [a-z0-9_.-]: lean_ok = 0
}
for _d in DOMAINS.values():
    assert all(1 <= len(l) <= 63 for l in _d.split('.')) and len(_d) <= 242


def wire_len(name):
    """Wire bytes of a dotted name without the terminator ('' -> 0)."""
    return len(name) + 1 if name else 0


def labels_of_len(rng, n):
    """Labels of [a-z0-9-] whose wire form (length byte + bytes each, no terminator) is n >= 2 bytes."""
    assert n >= 2
    out = []
    while n:
        choices = [l for l in range(1, min(63, n - 1) + 1) if n - 1 - l != 1]
        l = rng.choice(choices)
        out.append(_word(rng, l))
        n -= 1 + l
    return out


def dotted(rng, n):
    return '.'.join(labels_of_len(rng, n))


def root_path(dom):
    return '/' + '/'.join(reversed(dom.split('.')))


# "_srvce._proto" of the services: wire lengths 10, 11 (fills the header), 12, 17 and 128 (two 63-byte labels)
SP = [('_http', '_tc'), ('_http', '_tcp'), ('_https', '_tcp'), ('_xmpp-clien', '_tcp'), ('_' + 'p' * 62, '_' + 'q' * 62)]
assert [2 + len(a) + len(b) for a, b in SP] == [10, 11, 12, 17, 128]


class BoundaryZone(object):
    """One dnsDomain's boundary zone.

    snap     the whole zone (JSON lines)
    base     the zone without the `late` znodes
    late     [(what, delta)]: each long child (and each long "_srvce._proto" change) as a watch event on `base`
    hosts    [(fqdn, address)]; services [(fqdn, srvce, proto)]; kids [fqdn of every service child]
    kw       wire lengths of the service children it holds
    """

    def __init__(self, key, seed=0):
        self.key, self.dom = key, DOMAINS[key]
        dom = self.dom
        self.sl = sl = wire_len(dom)
        rng = random.Random('%s/%d' % (key, seed))
        root = root_path(dom)
        d_ix = sorted(DOMAINS).index(key)
        ent = {root: None}
        order = [root]
        self.hosts, self.services, self.kids, self.kw = [], [], [], []
        self.late = []
        late_lines = []
        n_addr = [0]

        def addr():
            n_addr[0] += 1
            return '10.%d.%d.%d' % (d_ix, n_addr[0] >> 8, n_addr[0] & 255)

        def put(labels, data):
            """labels: the key part, outermost last (as in the name); parents get null data."""
            for j in range(len(labels) - 1, 0, -1):
                p = root + '/' + '/'.join(reversed(labels[j:]))
                if p not in ent:
                    ent[p] = None
                    order.append(p)
            p = root + '/' + '/'.join(reversed(labels))
            if p not in ent:
                order.append(p)
            ent[p] = data
            return p

        # ---- hosts: key parts on both sides of every limit -----------------------------------------------------------
        pls = set([2, 3, 4, 5, 20, 21, 48, 49])
        for q in (63, 64, 65):                      # A names of 63/64/65 wire bytes with the terminator
            pls.add(q - 1 - sl)
            pls.add(q - 1 - sl - 11)                # the same totals for SRV names with an 11-byte prefix
        for total in (254, 255, 256):               # fqdns near and past 255 (256: only its PTR reaches it)
            pls.add(total - 1 - sl)
        for i, pl in enumerate(sorted(p for p in pls if 2 <= p)):
            labels = labels_of_len(rng, pl)
            a = addr()
            rec = {'type': 'host', 'host': {'address': a}}
            if i % 3 == 1:
                rec['ttl'] = 30 + i
            put(labels, rec)
            self.hosts.append(('.'.join(labels) + '.' + dom, a))

        # ---- services ----------------------------------------------------------------------------------------------
        def service(name, sp, kids, ttl=None, late_kids=()):
            s = {'srvce': sp[0], 'proto': sp[1], 'port': 80 + len(self.services)}
            if ttl is not None:
                s['ttl'] = ttl
            fq = name + '.' + dom
            if wire_len(fq) + 1 > 255:
                return
            p = put(name.split('.'), {'type': 'service', 'service': s})
            self.services.append((fq, sp[0], sp[1]))
            dom_wl = wire_len(fq) + 1
            for late, (kn, rec) in [(False, k) for k in kids] + [(True, k) for k in late_kids]:
                if isinstance(kn, int):                       # a wire length: a dotted name of that many bytes
                    if kn > 256 - dom_wl or kn < 2:
                        continue
                    kn = dotted(rng, kn)
                self.kw.append(wire_len(kn))
                line = (p + '/' + kn, rec)
                self.kids.append(kn + '.' + fq)
                if late:
                    late_lines.append(('child of %d wire bytes under %s' % (wire_len(kn), fq), line))
                else:
                    ent[line[0]] = rec
                    order.append(line[0])

        def lb(ttl=None, ports=None):
            a = addr()
            if ports:
                rec = {'type': 'rr_host', 'rr_host': {'address': a, 'ports': ports}}
            else:
                rec = {'type': 'load_balancer', 'load_balancer': {'address': a}}
            if ttl is not None:
                rec[rec['type']]['ttl'] = ttl
            return rec

        for i, sp in enumerate(SP):
            # children of 2 (one letter), 63 (one label) and 64 (two labels) wire bytes, several ports, their own ttl
            service('s%d' % i, sp, [('a', lb()), ('c' * 62, lb(ttl=7 + i)), (_word(rng, 31) + '.' + _word(rng, 31), lb(ports=[8000 + i, 9000 + i])),
                                    ('m%d' % i, lb(ports=[1, 2, 3]))], ttl=60 + i if i % 2 else None)
        # the long-child services all have 5-character names: one dom_wl for all of them
        svc_dom_wl = wire_len('l0.lk.' + dom) + 1
        long_kw = sorted(set(k for k in (224, 225, 240, 241, 255 - svc_dom_wl) if 2 <= k <= 255 - svc_dom_wl))
        for j, k in enumerate(long_kw):
            # a short child, and a long one that arrives later as a watch event
            service('l%d.lk' % j, SP[1], [('lb0', lb())], late_kids=[(k, lb(ttl=5 if j % 2 else None))])
        # all the long children in one service: strides of 272 bytes, runs of SRV RRs of 250+ bytes
        service('mn.lk', SP[1], [(k, lb(ports=[7000 + k, 7100 + k] if k % 2 else None)) for k in long_kw] + [('lb0', lb())])
        # a child whose name cannot be spelled under its service: "bad zk info" for SRV
        service('bd.lk', SP[1], [('lb0', lb()), (256 - svc_dom_wl, lb())])
        self.long_kw = long_kw
        # a service's "_srvce._proto" changed from 11 wire bytes (in the header) to 128 (in the arena)
        if root + '/s1' in ent:
            late_lines.append(('s1 prefix -> 128 bytes', (root + '/s1', {'type': 'service', 'service': {
                'srvce': SP[4][0], 'proto': SP[4][1], 'port': 81}})))
        self.base = _jsonl([(p, ent[p]) for p in order])
        for what, (p, rec) in late_lines:
            if p not in ent:
                order.append(p)
            ent[p] = rec
            self.late.append((what, _jsonl([(p, rec)])))
        self.snap = _jsonl([(p, ent[p]) for p in order])       # base with every late change
        self.info = {'dns_domain': dom, 'names': [h for h, _ in self.hosts] + [s[0] for s in self.services] + self.kids,
                     'addrs': [a for _, a in self.hosts], 'services': [s[0] for s in self.services]}

    # ---- queries ---------------------------------------------------------------------------------------------------
    def queries(self, seed=0, n=3000):
        """At least n queries: every name exact, re-cased in front of the domain, with an upper-case letter inside the
        domain, off a label boundary ('x' + dnsDomain); the bare domain and SRV names with an empty key part; matching and
        non-matching SRV prefixes; PTR of every address; EDNS absent, 512, 700, 1200 and 4096 in turn."""
        dom = self.dom
        rng = random.Random('%s/q/%d' % (self.key, seed))
        up = dom.replace(next(c for c in dom if c.isalpha()), next(c for c in dom if c.isalpha()).upper(), 1)
        shapes = []
        for fq in [h for h, _ in self.hosts] + self.kids + [s[0] for s in self.services]:
            pre = fq[:-len(dom) - 1]
            for name in (fq, pre.upper() + '.' + dom, _mixed(pre) + '.' + dom, pre + '.' + up, pre + '.x' + dom):
                shapes.append((name, 'A'))
            shapes.append(('_http._tcp.' + fq, 'SRV'))
        for fq, srvce, proto in self.services:
            pre = fq[:-len(dom) - 1]
            shapes += [('%s.%s.%s' % (srvce, proto, fq), 'SRV'), ('%s.%s.%s.%s' % (srvce, proto, _mixed(pre), dom), 'SRV'),
                       ('%s.%s.%s' % (srvce, proto[:-1] + 'x', fq), 'SRV'), ('%s.%s.%s' % (srvce.upper(), proto, fq), 'SRV'),
                       ('%s.%s.%s.%s' % (srvce, proto, pre, up), 'SRV'), ('_x._y.' + fq, 'SRV')]
        shapes += [(dom, 'A'), (dom, 'SRV'), ('_http._tcp.' + dom, 'SRV'), ('_a._b.' + dom, 'SRV'), ('x' + dom, 'A'),
                   (up, 'A'), ('nope.' + dom, 'A'), ('_http._tcp.nope.' + dom, 'SRV')]
        shapes += [(h, 'AAAA') for h, _ in self.hosts[:3]] + [(h, 'TXT') for h, _ in self.hosts[-3:]]
        ptrs = ['.'.join(reversed(a.split('.'))) + '.in-addr.arpa' for a in self.info['addrs']]
        ptrs += ['.'.join(reversed(a.split('.'))) + '.in-addr.arpa' for a in self.kid_addrs()]
        shapes += [(p, 'PTR') for p in ptrs] + [('7.7.7.7.in-addr.arpa', 'PTR')]
        shapes = [s for s in shapes if _encodable(s[0])]
        out = []
        edns = (None, 512, 700, 1200, 4096)
        k = 0
        while len(out) < n:
            for name, t in shapes:
                out.append(synth.make_query(name, t, qid=rng.randrange(65536), rd=rng.random() < 0.8, edns=edns[k % 5]))
                k += 1
            k += 1                               # every shape under another EDNS size on the next pass
        return out

    def kid_addrs(self):
        out = []
        for line in self.snap.decode().split('\n'):
            if line:
                d = json.loads(line)['data']
                if isinstance(d, dict) and d.get('type') in ('load_balancer', 'rr_host'):
                    out.append(d[d['type']]['address'])
        return out

    def growth(self, n=3000):
        """A delta of n new hosts: more than the table holds at its load limit, so it is laid out again."""
        root = root_path(self.dom)
        return _jsonl([('%s/g%05d' % (root, i), {'type': 'host', 'host': {'address': '198.51.%d.%d' % (i >> 8, i & 255)}})
                       for i in range(n)])


def _jsonl(entries):
    return ('\n'.join(json.dumps({'path': p, 'data': d}) for p, d in entries) + '\n').encode()


def _mixed(s):
    return ''.join(c.upper() if k % 2 else c for k, c in enumerate(s))


def _encodable(name):
    labels = name.split('.') if name else []
    return all(1 <= len(l) <= 63 for l in labels) and sum(len(l) + 1 for l in labels) + 1 <= 255
