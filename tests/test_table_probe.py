"""Key lookups in the cuckoo table (zone_image.h) at the inputs their comparison code exists for, against the oracle.

A wrong lookup still sends a well-formed answer, only for another name, and random names almost never reach the cases
that tell keys apart.  So this module crafts them, proves each crafted state holds in the built image, and compares whole
batches with the oracle:
  collisions    pairs of keys of one length with the same 32-bit hash h (so the same first slot under any mask), forward
                keys inline (3-20 bytes), in the arena on the lean path (21-48) and on the general path (49-120), reverse
                keys over 20 bytes; one member present and the other absent, and both present (one then lives in its
                second slot).  Keys of 3 and 4 bytes have too few spellings for a 32-bit collision: their pairs share the
                low 16 bits of h, which still puts them in one first slot.
  windows       collisions between keys that differ only inside one window: each word of an inline key, the first, a
                middle and the last arena word, at lengths with every len % 4, so each term of lean_query's comparison is
                the only thing that tells the two keys apart.
  displacement  keys forced into one first slot, the slot2_of case h2 & mask == h & mask (second slot = first ^ 1), and a
                delta sequence: the resident of a flagged position deleted, re-inserted, the displaced key deleted, new
                keys that are displaced on insert or start a kick chain, all through the incremental path.
The CPU half runs the device source through tests/native/emu_resolve.cpp; the GPU half runs the same zones through
Engine (both packings, both kernel profiles, UDP and TCP, host and device-resident entry points), the delta sequence
through Engine.apply_update (the slot patch), and the collision zone through the one-GPU sharded cluster at W = 3.
"""
import ctypes
import json

import numpy as np
import pytest

import helpers as H
from binder_b200 import synth
from binder_b200.shard import fmix32, hash_keys, owner_of
from test_gpu_parity import MODES, assert_same
from test_host_emulation import EmuEngine, _path_counts, emu_lib

DOM = 'foo.com'
ALPHA = np.frombuffer(b'abcdefghijklmnopqrstuvwxyz0123456789', dtype=np.uint8)
NONE = 0xFFFFFFFF
LEAN_MAX_KEY = 48                # lean_query hashes and compares keys up to this many bytes ...
LEAN_MAX_NAME = 63               # ... of names up to this many wire bytes before the terminator


# ---- 1. hashes, collision search, table states ---------------------------------------------------------------------
def _mulfold(x, k):
    p = x * np.uint64(k)
    return (p ^ (p >> np.uint64(32))) & np.uint64(0xFFFFFFFF)


def hash_key2(keys, ns=0):
    """bb::hash_key2 (zone_image.h) over an (n, L) uint8 array of canonical keys (or a list of equal-length byte strings)
    -> (h, h2), uint64 arrays."""
    arr = keys if isinstance(keys, np.ndarray) else np.frombuffer(b''.join(keys), dtype=np.uint8).reshape(len(keys), -1)
    n, L = arr.shape
    if L % 4:
        arr = np.concatenate([arr, np.zeros((n, 4 - L % 4), np.uint8)], axis=1)
    w = np.ascontiguousarray(arr).view('<u4').astype(np.uint64)
    h = np.full(n, 0x52455631 if ns else 0x42494E44, dtype=np.uint64)
    g = np.full(n, 0x7F4A7C15 if ns else 0x2545F491, dtype=np.uint64)
    for i in range(w.shape[1]):
        h = _mulfold(h ^ w[:, i], 0x9E3779B1)
        g = _mulfold(g ^ w[:, i], 0x85EBCA77)
    h = fmix32(h ^ np.uint64(L))
    g = fmix32((g + np.uint64(L * 0xC2B2AE3D)) & np.uint64(0xFFFFFFFF))
    return h, g


def slot2_of(h, h2, mask):
    a, b = int(h) & mask, int(h2) & mask
    return b if b != a else (a ^ 1) & mask


def template(ns, length):
    """A key shape of `length` bytes: (bytes with the fixed characters in place, bool mask of the free positions).
    Forward: wire labels of at most 63 bytes (length bytes fixed); reverse: '10.' + labels of at most 60 + '.7'."""
    base = np.zeros(length, np.uint8)
    free = np.zeros(length, bool)
    if ns == 0:
        pos, rem = 0, length
        while rem:
            lab = min(63, rem - 1) if rem != 65 else 62
            assert lab >= 1
            base[pos] = lab
            free[pos + 1:pos + 1 + lab] = True
            pos += 1 + lab
            rem -= 1 + lab
    else:
        assert length >= 6
        base[:3] = np.frombuffer(b'10.', np.uint8)
        base[-2:] = np.frombuffer(b'.7', np.uint8)
        pos, end = 3, length - 2
        while pos < end:
            lab = min(60, end - pos)
            if end - pos - lab == 1:
                lab -= 1
            free[pos:pos + lab] = True
            if pos + lab < end:
                base[pos + lab] = ord('.')
            pos += lab + 1
    return base, free


def find_pair(ns, length, window=None, seed=0, n=1 << 18):
    """Seeded search for two keys of one shape with the same hash h that differ only at free positions inside `window`
    (a (lo, hi) byte range; None = the whole key).  Shapes with under 2**20 spellings cannot hold a 32-bit collision:
    their pairs share the low 16 bits of h.  -> (a, b, bits)"""
    base, free = template(ns, length)
    var = np.nonzero(free & (np.arange(length) >= (window[0] if window else 0)) &
                     (np.arange(length) < (window[1] if window else length)))[0]
    bits = 32 if len(ALPHA) ** len(var) >= 1 << 20 else 16
    keep = np.uint64((1 << bits) - 1)
    rng = np.random.default_rng([seed, ns, length] + list(window or ()))
    for _ in range(16):
        b0 = base.copy()
        b0[free] = ALPHA[rng.integers(0, len(ALPHA), int(free.sum()))]
        cand = np.repeat(b0[None], n, axis=0)
        cand[:, var] = ALPHA[rng.integers(0, len(ALPHA), (n, len(var)))]
        h, h2 = hash_key2(cand, ns)
        k = h & keep
        order = np.argsort(k, kind='stable')
        ks = k[order]
        for i in np.nonzero(ks[1:] == ks[:-1])[0]:
            x, y = order[i], order[i + 1]
            if (h2[x] ^ h2[y]) & np.uint64(0xFFFF) and not np.array_equal(cand[x], cand[y]):
                return bytes(cand[x]), bytes(cand[y]), bits
    raise AssertionError(('no collision found', ns, length, window))


def labels_of(key):
    """Canonical forward key (wire labels) -> list of label bytes."""
    out, p = [], 0
    while p < len(key):
        out.append(key[p + 1:p + 1 + key[p]])
        p += 1 + key[p]
    assert p == len(key)
    return out


def name_of(key):
    return '.'.join(l.decode() for l in labels_of(key)) + '.' + DOM


def path_of(labels):
    return '/com/foo/' + '/'.join(l.decode() for l in reversed(labels))


def mixed_case(s):
    return ''.join(c.upper() if k % 2 else c for k, c in enumerate(s))


def ptr_query(addr, **kw):
    return synth.make_query(None, 'PTR', labels=[l.encode() for l in reversed(addr.split('.'))] + [b'in-addr', b'arpa'], **kw)


def forward_queries(key, qid):
    """A and SRV spellings of a forward key's name: lower case, upper case and mixed case (the `anyup` re-spelling;
    only what precedes dnsDomain varies, the suffix gate is case-sensitive), with and without EDNS."""
    nm = name_of(key)[:-len(DOM) - 1]
    q = lambda name, t, **kw: synth.make_query(name + '.' + DOM, t, qid & 0xFFFF, **kw)
    return [q(nm, 'A'), q(nm.upper(), 'A', edns=1232), q(mixed_case(nm), 'A', rd=False), q(nm, 'A', edns=700),
            q('_http._tcp.' + nm, 'SRV'), q('_http._tcp.' + mixed_case(nm), 'SRV', edns=4096),
            q('_http._tcp.' + nm.upper(), 'SRV', edns=1232)]


def reverse_queries(addr, qid):
    return [ptr_query(addr, qid=qid & 0xFFFF), ptr_query(addr, qid=(qid + 1) & 0xFFFF, edns=1232),
            ptr_query(addr, qid=(qid + 2) & 0xFFFF, rd=False)]


# The crafted pairs: (namespace, key length, window).  Full-hash collisions first, then the window collisions.
FULL = [(0, L, None) for L in range(3, 21)] + [(0, L, None) for L in (21, 24, 25, 48, 49, 64, 120)] + \
       [(1, L, None) for L in (21, 24, 37, 90)]


def _last_window(L):
    return (L - 4, L) if L % 4 == 0 else (L - L % 4 - 4, L)   # a partial last word alone has under four free bytes


WINDOWS = []
for _L in (17, 18, 19, 20):                                   # inline: every word of the slot's key, every len % 4
    WINDOWS += [(0, _L, (0, 8)), (0, _L, (4, 8)), (0, _L, (8, 12)), (0, _L, (12, 16)), (0, _L, _last_window(_L))]
for _L in (24, 25, 26, 27):                                   # lean arena path: first, a middle and the last word
    WINDOWS += [(0, _L, (0, 8)), (0, _L, (12, 16)), (0, _L, _last_window(_L))]
WINDOWS += [(0, 48, (20, 24)), (0, 48, (44, 48)), (0, 64, (32, 36)), (0, 120, (116, 120)), (1, 37, (20, 24))]


class Pair(object):
    def __init__(self, i, ns, length, window):
        self.i, self.ns, self.length, self.window = i, ns, length, window
        self.a, self.b, self.bits = find_pair(ns, length, window, seed=i)

    def addr(self, k):
        return (self.a, self.b)[k].decode()


def collision_snapshot(pairs, both):
    """Forward pairs: member a a service (with one load_balancer child), member b a host; reverse pairs: hosts whose
    address strings are the keys.  both=False: only member a is in the zone."""
    ent = {'/com/foo': None}
    for p in pairs:
        members = (0, 1) if both else (0,)
        if p.ns == 0:
            for k in members:
                labels = labels_of((p.a, p.b)[k])
                for j in range(len(labels) - 1, 0, -1):
                    ent.setdefault(path_of(labels[j:]), None)
                if k == 0:
                    ent[path_of(labels)] = {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80 + p.i % 50}}
                    ent[path_of(labels) + '/lb'] = {'type': 'load_balancer', 'load_balancer': {'address': '10.200.%d.%d' % (p.i >> 8, p.i & 255)}}
                else:
                    ent[path_of(labels)] = {'type': 'host', 'host': {'address': '10.100.%d.%d' % (p.i >> 8, p.i & 255)}, 'ttl': 60 + p.i}
        else:
            for k in members:
                ent['/com/foo/rv%03d%s' % (p.i, 'ab'[k])] = {'type': 'host', 'host': {'address': p.addr(k)}, 'ttl': 90 + k}
    return H.snapshot(sorted(ent.items(), key=lambda e: e[0].count('/')))


def pair_queries(pairs):
    pk = []
    for p in pairs:
        for k, key in enumerate((p.a, p.b)):
            if p.ns == 0:
                pk += forward_queries(key, 16 * p.i + k)
            else:
                pk += reverse_queries(key.decode(), 16 * p.i + 4 * k)
                pk.append(synth.make_query('rv%03d%s.%s' % (p.i, 'ab'[k], DOM), 'A'))
    return pk


def bind_emu(L):
    L.bb_emu_slot_of.restype = ctypes.c_int
    L.bb_emu_slot_of.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32] + [ctypes.c_void_p] * 5
    L.bb_zone_stat.restype = ctypes.c_uint64
    L.bb_zone_stat.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.bb_zone_mark_synced.argtypes = [ctypes.c_void_p]
    return L


class Where(object):
    """bb_emu_slot_of: where a canonical key lives in a zone's table."""

    def __init__(self, L, zone, ns, key):
        m, s, d, h, h2 = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_int(), ctypes.c_uint32(), ctypes.c_uint32()
        rc = L.bb_emu_slot_of(zone, ns, key, len(key), ctypes.byref(m), ctypes.byref(s), ctypes.byref(d), ctypes.byref(h),
                              ctypes.byref(h2))
        assert rc in (0, 1), rc
        self.present, self.mask, self.slot, self.flag, self.h, self.h2 = rc == 1, m.value, s.value, bool(d.value), h.value, h2.value
        self.first, self.second = self.h & self.mask, slot2_of(self.h, self.h2, self.mask)

    @property
    def displaced(self):
        return self.present and self.slot == self.second


@pytest.fixture(scope='module')
def L(tmp_path_factory):
    return bind_emu(emu_lib(tmp_path_factory.mktemp('emu')))


@pytest.fixture(scope='module')
def pairs():
    return [Pair(i, ns, length, w) for i, (ns, length, w) in enumerate(FULL + WINDOWS)]


@pytest.fixture(scope='module')
def snaps(pairs):
    return {'one': collision_snapshot(pairs, False), 'both': collision_snapshot(pairs, True)}


def test_python_hashes_match_the_table_builder(L):
    """hash_key2 here (h and h2) == bb::hash_key2 as compiled into the emulation, on 4,000 random keys of 1..130 bytes of
    both namespaces; h also == binder_b200.shard.hash_keys; and a present key lives in one of the two slots the hashes
    name."""
    rng = np.random.default_rng(5)
    snap = H.snapshot([('/com/foo', None), ('/com/foo/x', {'type': 'host', 'host': {'address': '10.0.0.1'}})])
    z = EmuEngine(L, DOM, snap).zone
    for ns in (0, 1):
        for length in (1, 2, 3, 4, 5, 7, 8, 13, 20, 21, 24, 33, 48, 49, 64, 77, 120, 130):
            keys = rng.integers(0, 256, (4000 // 36 + 1, length), dtype=np.uint8)
            h, h2 = hash_key2(keys, ns)
            assert np.array_equal(h, hash_keys([bytes(k) for k in keys], ns=ns))
            for k, a, b in zip(keys, h, h2):
                w = Where(L, z, ns, bytes(k))
                assert (w.h, w.h2) == (int(a), int(b)), (ns, length, bytes(k))
    for ns, key in ((0, b'\x01x'), (1, b'10.0.0.1'), (0, b'')):
        w = Where(L, z, ns, key)
        assert w.present and w.slot in (w.first, w.second), (ns, key)


def test_crafted_pairs_hold_what_they_claim(L, pairs, snaps):
    """Every pair: equal h (or equal low 16 bits for the 3- and 4-byte keys), different h2, equal length, differing only
    inside its window.  In the one-member zone a is present and b absent at a's first slot; in the both-members zone
    both are present, they share a first slot, one of them lives in its second slot and that position carries
    SLOT_DISPLACED."""
    zs = {k: EmuEngine(L, DOM, s).zone for k, s in snaps.items()}
    mask = Where(L, zs['both'], 0, b'').mask
    assert mask < 1 << 16
    displaced = 0
    for p in pairs:
        h, h2 = hash_key2([p.a, p.b], p.ns)
        assert len(p.a) == len(p.b) == p.length and p.a != p.b
        keep = (1 << p.bits) - 1
        assert int(h[0]) & keep == int(h[1]) & keep and h2[0] != h2[1], p.i
        assert p.bits == 32 or p.length <= 4, p.i
        diff = [j for j in range(p.length) if p.a[j] != p.b[j]]
        lo, hi = p.window or (0, p.length)
        assert diff and lo <= min(diff) and max(diff) < hi, (p.i, diff)
        wa, wb = Where(L, zs['one'], p.ns, p.a), Where(L, zs['one'], p.ns, p.b)
        assert wa.present and not wb.present and wb.first == wa.first, p.i
        wa, wb = Where(L, zs['both'], p.ns, p.a), Where(L, zs['both'], p.ns, p.b)
        assert wa.present and wb.present and wa.first == wb.first, p.i
        assert (wa.displaced or wb.displaced) and wa.flag and wb.flag, p.i
        displaced += 1
    assert L.bb_zone_stat(zs['both'], 8) >= displaced
    # the lean arena comparison is the only term that can tell a window pair apart: same length, same stored hash
    assert any(p.window and 20 < p.length <= LEAN_MAX_KEY and p.window[0] >= 20 for p in pairs)


@pytest.mark.parametrize('zone,recursion', [('one', False), ('one', True), ('both', False), ('both', True)])
def test_collisions_match_oracle_on_cpu(L, pairs, snaps, zone, recursion):
    """Every crafted name as A, SRV (upper, mixed case, EDNS) or PTR against the oracle, UDP and TCP."""
    emu = EmuEngine(L, DOM, snaps[zone], recursion)
    orc = H.make_impl('oracle', DOM, snaps[zone], recursion=recursion)
    data, off = synth.pack_batch(pair_queries(pairs))
    assert_same(emu, orc, data, off, seed=3, qidx_base=77)
    assert_same(emu, orc, data, off, seed=4, tcp=True)


def _front_end(L, emu, pkts):
    data, off = synth.pack_batch(pkts)
    _path_counts(L)
    emu.resolve_batch(data, off, seed=1)
    return _path_counts(L)


def test_each_length_class_takes_its_front_end(L, pairs, snaps):
    """A queries on keys up to 48 bytes (names up to 63 wire bytes) are settled by lean_query, longer ones by the
    general path (probe<KG>); SRV the same with its 11-byte prefix; PTR always by the general path."""
    emu = EmuEngine(L, DOM, snaps['both'])
    suffix = len(DOM) + 1
    for p in pairs:
        for key in (p.a, p.b):
            if p.ns == 1:
                lean, general = _front_end(L, emu, reverse_queries(key.decode(), p.i))
                assert (lean, general) == (0, 3), (p.i, lean, general)
                continue
            fq = forward_queries(key, p.i)
            a_q, srv_q = fq[:4], fq[4:]
            lean_a = p.length <= LEAN_MAX_KEY and p.length + suffix <= LEAN_MAX_NAME
            lean_srv = p.length <= LEAN_MAX_KEY and 11 + p.length + suffix <= LEAN_MAX_NAME
            assert _front_end(L, emu, a_q) == ((4, 0) if lean_a else (0, 4)), (p.i, p.length)
            assert _front_end(L, emu, srv_q) == ((3, 0) if lean_srv else (0, 3)), (p.i, p.length)
    assert any(p.length > LEAN_MAX_KEY for p in pairs) and any(20 < p.length <= LEAN_MAX_KEY for p in pairs)


@pytest.mark.parametrize('world', [2, 3, 8])
def test_route_mode_owner_of_crafted_keys(L, pairs, world):
    """Route mode (both front ends) sends every crafted query to owner_of(hash_keys(canonical key))."""
    pk, want = [], []
    for p in pairs:
        for key in (p.a, p.b):
            own = int(owner_of(hash_keys([key], ns=p.ns), world)[0])
            q = forward_queries(key, p.i) if p.ns == 0 else reverse_queries(key.decode(), p.i)
            pk += q
            want += [own] * len(q)
    data, off = synth.pack_batch(pk)
    owner = np.zeros(len(pk), dtype=np.uint8)
    assert L.bb_emu_route_batch(DOM.encode(), 0, data.ctypes.data, off.ctypes.data, len(pk), world, world - 1, owner.ctypes.data) == 0
    bad = np.nonzero(owner != np.array(want))[0]
    assert bad.size == 0, (bad[:5], [pk[i] for i in bad[:3]])
    assert len(set(want)) == world


# ---- displacement and the delta sequence ---------------------------------------------------------------------------
N_FILL = 60


def _db(i):
    return {'type': 'database', 'database': {'primary': 'tcp://10.9.%d.%d:5432/db' % (i >> 8, i & 255)}}


def _fill_key(i):
    return b'\x04f%03d' % i


def _random_keys(rng, length, n=1 << 16):
    return np.concatenate([np.full((n, 1), length - 1, np.uint8), ALPHA[rng.integers(0, len(ALPHA), (n, length - 1))]], axis=1)


def _pick(rng, length, cond, mask, taken):
    """A random single-label key of `length` bytes with cond(first, h & mask, h2 & mask) true, not among `taken`."""
    for _ in range(64):
        keys = _random_keys(rng, length)
        h, h2 = hash_key2(keys)
        a, b = (h & np.uint64(mask)).astype(np.int64), (h2 & np.uint64(mask)).astype(np.int64)
        second = np.where(b != a, b, (a ^ 1) & mask)
        for j in np.nonzero(cond(a, b, second))[0]:
            k = bytes(keys[j])
            if k not in taken:
                taken.add(k)
                return k, int(a[j]), int(second[j])
    raise AssertionError('no key found')


class Displacement(object):
    """A zone of N_FILL single-label database records (no reverse keys: nothing is inserted after the crafted forward keys)
    plus crafted keys, and the delta sequence run on it.  Groups (resident r, displaced d, absent near miss m):
      inline  8-byte keys sharing a first slot
      arena   24-byte keys sharing a first slot (the lean arena comparison)
      xor1    12-byte keys; d's h2 & mask == h & mask, so its second slot is first ^ 1
      general 56-byte keys sharing a first slot (names over 63 wire bytes: the general path)
    Step 4 adds n_disp (its first slot held by a filler that stays, its second free: displaced on insert, the flag set on
    a slot nothing else touches), every group's d again, and kick (both of its slots held: it evicts a filler)."""
    GROUPS = (('inline', 8, False), ('arena', 24, False), ('xor1', 12, True), ('general', 56, False))

    def __init__(self, L):
        self.L = L
        base = [('/com/foo', None)] + [('/com/foo/f%03d' % i, _db(i)) for i in range(N_FILL)]
        z0 = EmuEngine(L, DOM, H.snapshot(base)).zone
        fills = [Where(L, z0, 0, _fill_key(i)) for i in range(N_FILL)] + [Where(L, z0, 0, b'')]
        self.mask = mask = fills[0].mask
        used = set(w.slot for w in fills)
        assert len(used) == N_FILL + 1
        rng = np.random.default_rng(2024)
        taken = set()
        free = lambda s: ~np.isin(s, list(used))
        self.g = {}
        for name, length, xor1 in self.GROUPS:
            r, p, _ = _pick(rng, length, lambda a, b, s: free(a) & free(a ^ 1) if xor1 else free(a), mask, taken)
            used.add(p)
            if xor1:
                d, _, q = _pick(rng, length, lambda a, b, s: (a == p) & (b == p), mask, taken)
                assert q == p ^ 1
            else:
                d, _, q = _pick(rng, length, lambda a, b, s: (a == p) & free(s) & (s != p), mask, taken)
            used.add(q)
            m, _, _ = _pick(rng, length, lambda a, b, s: a == p, mask, taken)
            self.g[name] = dict(r=r, d=d, m=m, p=p, q=q, i=len(self.g))
        fill_slots = [w.slot for w in fills[:N_FILL]]
        self.n_disp, f, q = _pick(rng, 10, lambda a, b, s: np.isin(a, fill_slots) & free(s), mask, taken)
        used.add(q)
        self.n_disp_first, self.n_disp_second = f, q
        # the evicted filler's other slot is free: the chain ends there and disturbs no crafted key
        movable = [w.slot for w in fills[:N_FILL] if (w.second if w.slot == w.first else w.first) not in used and w.slot != f]
        self.kick, self.kick_first, _ = _pick(rng, 16, lambda a, b, s: np.isin(a, movable) & np.isin(s, fill_slots) & (a != s),
                                              mask, taken)
        self.kicked = [i for i in range(N_FILL) if fill_slots[i] == self.kick_first]
        self.fills = fills
        ent = list(base)
        for name, _, _ in self.GROUPS:
            for k in ('r', 'd'):
                ent.append((self.path(self.g[name][k]), self.record(name, k)))
        self.snap = H.snapshot(ent)

    @staticmethod
    def path(key):
        return path_of(labels_of(key))

    def record(self, name, k):
        return _db(1000 + 10 * self.g[name]['i'] + 'rdm'.index(k))

    def line(self, key, data=None, rec=None):
        return json.dumps({'path': self.path(key), 'deleted': True} if data is None else {'path': self.path(key), 'data': rec})

    def steps(self):
        """[(what, delta bytes)]"""
        G = [self.g[n] for n, _, _ in self.GROUPS]
        names = [n for n, _, _ in self.GROUPS]
        dele = lambda k: '\n'.join(self.line(g[k]) for g in G).encode()
        put = lambda k: '\n'.join(self.line(g[k], True, self.record(n, k)) for n, g in zip(names, G)).encode()
        add = '\n'.join([self.line(self.n_disp, True, _db(2000)), put('d').decode(), self.line(self.kick, True, _db(2001))]).encode()
        return [('delete residents', dele('r')), ('re-insert residents', put('r')), ('delete displaced', dele('d')),
                ('displace and kick', add)]

    def queries(self):
        pk = [synth.make_query('f%03d.%s' % (i, DOM), 'A', i) for i in range(N_FILL)]
        keys = [self.n_disp, self.kick] + [g[k] for g in self.g.values() for k in 'rdm']
        for j, key in enumerate(keys):
            pk += forward_queries(key, 100 + j)[:4]
        return pk

    def check_state(self, z, step):
        """The table state each step claims, read from the image with bb_emu_slot_of."""
        L = self.L
        assert Where(L, z, 0, b'').mask == self.mask
        for name, g in self.g.items():
            r, d, m = (Where(L, z, 0, g[k]) for k in 'rdm')
            assert r.first == d.first == m.first == g['p'] and d.second == g['q'] and not m.present, (step, name)
            if name == 'xor1':
                assert d.h2 & self.mask == d.h & self.mask and d.second == d.first ^ 1, step
            r_in = step in (0, 2, 3, 4)
            d_in = step in (0, 1, 2, 4)
            assert r.present == r_in and (not r_in or r.slot == g['p']), (step, name)
            assert d.present == d_in and (not d_in or d.slot == g['q']), (step, name)
            assert r.flag == d_in, (step, name, 'SLOT_DISPLACED at the shared first slot')
        if step == 4:
            n = Where(L, z, 0, self.n_disp)
            assert n.displaced and n.slot == self.n_disp_second and n.flag, step
            k = Where(L, z, 0, self.kick)
            assert k.present and k.slot == self.kick_first, step
            assert self.kicked and all(Where(L, z, 0, _fill_key(i)).slot != self.kick_first for i in self.kicked), step
        else:
            assert not Where(L, z, 0, self.n_disp).present and not Where(L, z, 0, self.kick).present
            assert all(Where(L, z, 0, _fill_key(i)).slot == self.fills[i].slot for i in range(N_FILL)), step
        assert L.bb_zone_stat(z, 8) == sum(1 for i in range(N_FILL) if Where(L, z, 0, _fill_key(i)).displaced) + \
            sum(1 for g in self.g.values() if Where(L, z, 0, g['d']).present) + (step == 4)


@pytest.fixture(scope='module')
def disp(L):
    return Displacement(L)


@pytest.mark.parametrize('recursion', [False, True])
def test_displacement_deltas_on_cpu(L, disp, recursion):
    """The delta sequence through bb_zone_apply: after every step each key and the near misses equal the oracle, the
    step went through the incremental path (changed slots, no new layout) and the table holds the claimed state."""
    emu = EmuEngine(L, DOM, disp.snap, recursion)
    orc = H.make_impl('oracle', DOM, disp.snap, recursion=recursion)
    L.bb_zone_mark_synced(emu.zone)
    data, off = synth.pack_batch(disp.queries())
    disp.check_state(emu.zone, 0)
    assert_same(emu, orc, data, off, seed=1)
    for step, (what, delta) in enumerate(disp.steps(), 1):
        emu.apply(delta)
        orc.apply_delta(delta)
        assert L.bb_zone_stat(emu.zone, 6) > 0 and L.bb_zone_stat(emu.zone, 7) == 0, what
        L.bb_zone_mark_synced(emu.zone)
        disp.check_state(emu.zone, step)
        assert_same(emu, orc, data, off, seed=step, qidx_base=step * 1000)
        assert_same(emu, orc, data, off, seed=step, tcp=True)


# ---- 3. the GPU half -----------------------------------------------------------------------------------------------
ENTRIES = [pytest.param(False, id='host'), pytest.param(True, id='device')]


def _device_check(eng, orc, data, off, seed, ordered, tcp):
    """bb_resolve_batch_device_ex on device buffers, exact against the oracle with the totals contract."""
    import torch
    from test_gpu_tcp_paths import TDevBatch
    from binder_b200._lib import check
    data = np.concatenate([data, np.zeros((-data.size) % 16, np.uint8)])
    b = TDevBatch(data, off, out_cap=max(8192, (len(off) - 1) * (16384 if tcp else 1232)))
    torch.cuda.synchronize()
    rc, ep = b.launch_ex(eng, seed, 1 if tcp else 0, qidx_base=seed * 3)
    check(rc)
    torch.cuda.synchronize()
    b.check(orc, seed, ep, ordered, qidx_base=seed * 3, tcp=tcp)


@pytest.mark.gpu
@pytest.mark.parametrize('device', ENTRIES)
@pytest.mark.parametrize('profile', ['small', 'service'])
@pytest.mark.parametrize('ordered', MODES)
def test_gpu_collisions_match_oracle(pairs, snaps, ordered, profile, device):
    data, off = synth.pack_batch(pair_queries(pairs))
    for zone, recursion in (('one', False), ('both', True)):
        gpu = H.make_impl('gpu', DOM, snaps[zone], recursion=recursion, ordered=ordered)
        orc = H.make_impl('oracle', DOM, snaps[zone], recursion=recursion)
        try:
            gpu.set_kernel_profile(profile)
            for tcp in (False, True):
                if device:
                    _device_check(gpu, orc, data, off, 5 + tcp, ordered, tcp)
                else:
                    assert_same(gpu, orc, data, off, seed=5 + tcp, qidx_base=99, tcp=tcp)
        finally:
            gpu.close()


@pytest.mark.gpu
@pytest.mark.parametrize('ordered', MODES)
def test_gpu_displacement_deltas_through_slot_patch(L, disp, ordered):
    """The delta sequence through Engine.apply_update, which ships only the touched slots (patch_slots_kernel): a
    SLOT_DISPLACED change on a first slot that is not shipped leaves the device with a stale flag.  Checked after every
    step, with an emulated twin of the zone proving the table state."""
    from binder_b200.engine import Engine, Zone
    zone = Zone(disp.snap, DOM)
    twin = EmuEngine(L, DOM, disp.snap)
    gpu = Engine(DOM, recursion=True, ordered=ordered)
    orc = H.make_impl('oracle', DOM, disp.snap, recursion=True)
    try:
        gpu.swap_zone(zone)
        assert zone.stat()['slots'] == disp.mask + 1
        data, off = synth.pack_batch(disp.queries())
        assert_same(gpu, orc, data, off, seed=1)
        for step, (what, delta) in enumerate(disp.steps(), 1):
            zone.apply(delta)
            twin.apply(delta)
            orc.apply_delta(delta)
            n_dirty, relaid = zone.pending()
            assert n_dirty > 0 and not relaid, what
            gpu.apply_update(zone)
            assert zone.pending() == (0, False)
            disp.check_state(twin.zone, step)
            for tcp in (False, True):
                assert_same(gpu, orc, data, off, seed=step, qidx_base=step * 1000, tcp=tcp)
    finally:
        gpu.close()
        zone.close()


@pytest.mark.gpu
@pytest.mark.parametrize('ordered', MODES)
def test_gpu_sharded_collisions(L, pairs, snaps, ordered):
    """The both-members collision zone at W = 3 through the one-GPU sharded cluster (route_push_kernel + the
    multi-region resolve_kernel), every region against the oracle and the CPU router."""
    from test_gpu_shard_paths import Batch, Cluster
    world = 3
    snap = snaps['both']
    orc = H.make_impl('oracle', DOM, snap, recursion=True)

    def route(dom, recursion, data, off, world, rank):
        owner = np.zeros(max(len(off) - 1, 1), dtype=np.uint8)
        assert L.bb_emu_route_batch(dom.encode(), int(recursion), data.ctypes.data, off.ctypes.data, len(off) - 1, world, rank,
                                    owner.ctypes.data) == 0
        return owner[:len(off) - 1].astype(np.int64)

    pk = pair_queries(pairs)
    cl = Cluster(DOM, snap, world, 4096, ordered=ordered, host=(1,))
    try:
        for k in range(2):
            seed = 31 + k
            batches = [Batch(pk[r::world] if k == 0 else pk, r, world, r * 4096, seed, orc, route, DOM, True)
                       for r in range(world)]
            cl.step(batches, seed, exact=k == 0)
            cl.check(batches, what=('step', k))
    finally:
        cl.close()
