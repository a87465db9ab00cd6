"""Names at their length limits under dnsDomains of many shapes (tests/namegen.py), against the oracle.

The rest of the suite serves three dnsDomains whose '.' + dnsDomain lengths are multiples of four, with short names
inside.  Here every dnsDomain of namegen.DOMAINS gets a boundary zone: hosts whose names sit on both sides of the lean
front end's limits (64 wire bytes, a 48-byte key part) and of the 20-byte inline key, fqdns of 254-256 bytes,
"_srvce._proto" prefixes of 10-128 wire bytes, and service children whose dotted names run up to 255 - dom_wl wire bytes.

CPU half: every zone builds and takes its long children as watch events; the dnsDomain length limit; the oracle against
the independent restatement (oracle/binder_ref.py); the device source (tests/native/emu_resolve.cpp) against the oracle,
with the front-end thresholds and the copy-job paths shown to be crossed; the emulated sharded pipeline.
GPU half: Engine in both packings, both kernel profiles, UDP and TCP; pinned results; the long-child and long-prefix
deltas through the slot patch and a re-layout; the recursion pre-filter on the zone's own dnsDomain; the one-GPU sharded
cluster at W = 2 and 3.
"""
import ctypes
import random

import numpy as np
import pytest

import helpers as H
import namegen as N
from binder_b200 import synth
from test_gpu_parity import MODES, assert_same
from test_host_emulation import EmuEngine, _path_counts, emu_lib
from test_oracle_cross import check_against_ref

ERR_DOMAIN = -7
KEYS = list(N.DOMAINS)
LEAN_MAX_NAME = 63               # lean_query: wire bytes of the QNAME before its terminator ...
LEAN_MAX_KEY = 48                # ... and of the key part in front of dnsDomain
PROFILES = ['small', 'service']
_ZONES = {}


def zone(key):
    if key not in _ZONES:
        _ZONES[key] = N.BoundaryZone(key)
    return _ZONES[key]


def batch(key, seed=0):
    return synth.pack_batch(zone(key).queries(seed))


@pytest.fixture(scope='module')
def L(tmp_path_factory):
    L = emu_lib(tmp_path_factory.mktemp('emu'))
    L.bb_zone_stat.restype = ctypes.c_uint64
    L.bb_zone_stat.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.bb_zone_probe.restype = ctypes.c_int
    L.bb_zone_probe.argtypes = [ctypes.c_void_p, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint32] + [ctypes.c_void_p] * 4 + \
        [ctypes.c_uint32, ctypes.c_void_p]
    L.bb_zone_mark_synced.argtypes = [ctypes.c_void_p]
    return L


def build(L, snap, dom):
    err = ctypes.c_int(0)
    z = L.bb_zone_build(snap, len(snap), dom.encode(), ctypes.byref(err))
    return z, err.value


def probe(L, z, fqdn):
    """(kind, ttl, payload) the image holds for a forward name (bb_zone_probe: a service's payload is its header, its
    "_srvce._proto" when that lives in the arena, and its record with every section)."""
    k = fqdn.encode()
    kind, ttl, rl = ctypes.c_uint8(0), ctypes.c_uint32(0), ctypes.c_uint32(0)
    buf = ctypes.create_string_buffer(1 << 20)
    if not L.bb_zone_probe(z, 0, k, len(k), ctypes.byref(kind), ctypes.byref(ttl), None, buf, len(buf), ctypes.byref(rl)):
        return None
    return kind.value, ttl.value, buf.raw[:rl.value]


# ---- 1. acceptance -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('key', KEYS)
def test_boundary_zones_build_and_take_long_children(L, key):
    """The whole zone builds; its long children and the long-prefix change, applied one by one as watch events to the
    zone without them, are accepted, and every service then holds what a fresh build of the result holds.  A child of
    225..255 - dom_wl wire bytes needs an additional-section stride of 17 units of 16, which the header stores as 0."""
    b = zone(key)
    whole, err = build(L, b.snap, b.dom)
    assert whole, err
    z, err = build(L, b.base, b.dom)
    assert z, err
    try:
        kind, _, rec = probe(L, whole, 'mn.lk.' + b.dom)
        add = max(b.long_kw) + 16                    # the longest additional RR
        assert kind == 4 and int.from_bytes(rec[4:6], 'little') == len(b.long_kw) + 1
        assert rec[16] >> 4 == (0 if add > 240 else (add + 15) // 16), rec[16]
        for what, delta in b.late:
            assert L.bb_zone_apply(z, delta, len(delta)) == 0, what
        fresh, err = build(L, b.snap, b.dom)
        for fq, _, _ in b.services:
            assert probe(L, z, fq) == probe(L, fresh, fq) != None, fq
        L.bb_zone_free(fresh)
    finally:
        L.bb_zone_free(z)
        L.bb_zone_free(whole)
    if b.sl <= 12:                                   # short dnsDomains reach the window above 224 bytes
        assert any(k >= 225 for k in b.long_kw) and max(b.long_kw) + 16 > 240


def test_issue_shape_two_children(L):
    """svc.foo.com with two load_balancer children, one named by a dotted path component of kw wire bytes: every kw up
    to 255 - dom_wl builds, as a snapshot and as a delta, and answers as the oracle does; 243 bytes cannot be spelled
    under the service (SRV: SERVFAIL)."""
    rng = random.Random(5)
    dom = 'foo.com'
    head = [('/com/foo', None), ('/com/foo/svc', {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80}}),
            ('/com/foo/svc/lb0', {'type': 'load_balancer', 'load_balancer': {'address': '10.0.0.1'}})]
    for kw in (223, 224, 225, 230, 241, 242, 243):
        kid = ('/com/foo/svc/' + N.dotted(rng, kw), {'type': 'load_balancer', 'load_balancer': {'address': '10.0.0.2'}})
        snap = H.snapshot(head + [kid])
        z, err = build(L, snap, dom)
        assert z, (kw, err)
        L.bb_zone_free(z)
        z, err = build(L, H.snapshot(head), dom)
        assert L.bb_zone_apply(z, H.snapshot([kid]), len(H.snapshot([kid]))) == 0, kw
        L.bb_zone_free(z)
        emu = EmuEngine(L, dom, snap)
        orc = H.make_impl('oracle', dom, snap)
        pk = [synth.make_query('_http._tcp.svc.foo.com', 'SRV', edns=e) for e in (None, 1200, 4096)] + [synth.make_query('svc.foo.com', 'A')]
        data, off = synth.pack_batch(pk * 40)
        for tcp in (False, True):
            g = assert_same(emu, orc, data, off, seed=kw, tcp=tcp)
            assert (g[3] == 0).all()
        # what the answers hold: both SRV answers up to 242 bytes, SERVFAIL for the child that cannot be spelled
        rcode, an, _, _, f = H.decode_semantic(bytes(g[0][g[1][2]:g[1][3]]))
        assert rcode == 2 if kw == 243 else (rcode, len(an), f['tc']) == (0, 2, False), (kw, rcode, an)


def test_dns_domain_length_limit(L):
    """A dnsDomain of 242 characters is served; one of 243 is refused (BB_ERR_DOMAIN): the SOA's rname,
    hostmaster.<dnsDomain>, would not fit 255 bytes."""
    from binder_b200._lib import BinderError
    from binder_b200.engine import Zone
    snap = H.snapshot([('/' + '/'.join(reversed(N.LONGEST_DOMAIN.split('.'))), None)])
    z, err = build(L, snap, N.LONGEST_DOMAIN)
    assert z and err == 0
    L.bb_zone_free(z)
    Zone(snap, N.LONGEST_DOMAIN).close()
    snap = H.snapshot([('/' + '/'.join(reversed(N.TOO_LONG_DOMAIN.split('.'))), None)])
    z, err = build(L, snap, N.TOO_LONG_DOMAIN)
    assert not z and err == ERR_DOMAIN
    with pytest.raises(BinderError) as ei:
        Zone(snap, N.TOO_LONG_DOMAIN)
    assert ei.value.code == ERR_DOMAIN
    data, off = synth.pack_batch([synth.make_query('x.' + N.TOO_LONG_DOMAIN[:200], 'A')])
    with pytest.raises(AssertionError, match=str(ERR_DOMAIN)):
        EmuEngine(L, N.TOO_LONG_DOMAIN, None).resolve_batch(data, off)        # the per-engine constants refuse it too


# ---- 2. the oracle at these lengths --------------------------------------------------------------------------------
@pytest.mark.parametrize('key', KEYS)
def test_oracle_matches_restatement(key):
    """The GPU is only ever compared with the oracle: at these lengths the oracle must first agree with the independent
    restatement (binder_ref.py through dnspython), for every query shape once."""
    b = zone(key)
    recursion = KEYS.index(key) % 2 == 1
    pkts = b.queries(seed=1, n=1)
    for snap in (b.snap, b.base):
        orc = H.make_impl('oracle', b.dom, snap, recursion=recursion)
        check_against_ref(orc, snap, b.info, pkts, recursion, seed=KEYS.index(key) + 17)


# ---- 3. the device source on the CPU -------------------------------------------------------------------------------
@pytest.mark.parametrize('key', KEYS)
def test_emulated_device_code_matches_oracle(L, key):
    """Before and after the long-child and long-prefix watch events, UDP and TCP; then a fresh build of the whole zone."""
    b = zone(key)
    recursion = KEYS.index(key) % 2 == 0
    data, off = batch(key)
    emu = EmuEngine(L, b.dom, b.base, recursion)
    orc = H.make_impl('oracle', b.dom, b.base, recursion=recursion)
    assert_same(emu, orc, data, off, seed=1, qidx_base=3)
    assert_same(emu, orc, data, off, seed=2, tcp=True)
    L.bb_zone_mark_synced(emu.zone)
    for what, delta in b.late:
        emu.apply(delta)
        orc.apply_delta(delta)
        assert L.bb_zone_stat(emu.zone, 6) > 0 and L.bb_zone_stat(emu.zone, 7) == 0, what     # changed slots, no new layout
        L.bb_zone_mark_synced(emu.zone)
    assert_same(emu, orc, data, off, seed=3, qidx_base=1 << 31)
    assert_same(emu, orc, data, off, seed=4, tcp=True)
    emu = EmuEngine(L, b.dom, b.snap, recursion)
    orc = H.make_impl('oracle', b.dom, b.snap, recursion=recursion)
    assert_same(emu, orc, data, off, seed=5)
    assert_same(emu, orc, data, off, seed=6, tcp=True)


def _front_end(L, emu, pkt):
    data, off = synth.pack_batch([pkt])
    _path_counts(L)
    emu.resolve_batch(data, off, seed=1)
    return _path_counts(L)


@pytest.mark.parametrize('key', KEYS)
def test_front_end_thresholds(L, key):
    """A and SRV names of at most 63 wire bytes before the terminator whose key part is at most 48 bytes are settled by
    lean_query, every other name by the general path; under a dnsDomain with a byte outside [a-z0-9_.-] all of them."""
    b = zone(key)
    emu = EmuEngine(L, b.dom, b.snap)
    lean_ok = all(c.isalnum() and c.islower() or c.isdigit() or c in '_.-' for c in b.dom)
    assert lean_ok == (key != 'not-lean')
    seen = []                                        # (lean, d_end, pl) of every name asked
    for fq, _ in b.hosts:
        if not N._encodable(fq):
            continue
        pl = N.wire_len(fq) - b.sl
        pre = fq[:-len(b.dom) - 1]
        for name, t, d_end in ((fq, 'A', N.wire_len(fq)), (pre.upper() + '.' + b.dom, 'A', N.wire_len(fq)),
                               ('_http._tcp.' + fq, 'SRV', 11 + N.wire_len(fq))):
            if not N._encodable(name):
                continue
            lean = lean_ok and d_end <= LEAN_MAX_NAME and pl <= LEAN_MAX_KEY
            assert _front_end(L, emu, synth.make_query(name, t, edns=1232 if t == 'SRV' else None)) == ((1, 0) if lean else (0, 1)), \
                (name, t, d_end, pl)
            seen.append((lean, d_end, pl))
    for a in b.info['addrs'][:4]:
        assert _front_end(L, emu, synth.make_query('.'.join(reversed(a.split('.'))) + '.in-addr.arpa', 'PTR')) == (0, 1)
    # each limit was crossed where the dnsDomain leaves room for it: a name of 63 wire bytes lean, one of 64 not ...
    if b.sl <= LEAN_MAX_NAME - 2:
        assert any(d == 63 and p <= LEAN_MAX_KEY and l == lean_ok for l, d, p in seen), seen
        assert any(d == 64 and p <= LEAN_MAX_KEY and not l for l, d, p in seen), seen
    # ... a key part of 48 bytes lean, one of 49 in a name short enough not
    if b.sl <= LEAN_MAX_NAME - LEAN_MAX_KEY - 1:
        assert any(p == 48 and d <= 63 and l == lean_ok for l, d, p in seen), seen
        assert any(p == 49 and d <= 63 and not l for l, d, p in seen), seen
    if not lean_ok:
        assert not any(l for l, _, _ in seen)


@pytest.mark.parametrize('key', [k for k in KEYS if N.wire_len(N.DOMAINS[k]) <= 12 and k != 'not-lean'])
def test_copy_jobs_on_long_children(L, key):
    """SRV answers of the long-child services in big tiles: answered as copy jobs, and runs of SRV RRs cut short by
    truncation (jobs with a masked tail).  Over TCP a tile holding an answer over 1,232 bytes is written response by
    response, so the TCP batch asks the two-child services only."""
    b = zone(key)
    emu = EmuEngine(L, b.dom, b.snap)
    orc = H.make_impl('oracle', b.dom, b.snap)
    st = (ctypes.c_ulonglong * 5)()
    for tcp in (False, True):
        svcs = [fq for fq, _, _ in b.services if '.lk.' in fq and (not tcp or fq.startswith('l'))]
        pk = []
        for i in range(1500):
            fq = svcs[i % len(svcs)]
            pk.append(synth.make_query('_http._tcp.' + fq, 'SRV', i, edns=(None, 700, 1200, 4096)[i % 4]) if i % 5 else
                      synth.make_query(fq, 'A', i, edns=1200))
        data, off = synth.pack_batch(pk)
        L.bb_emu_job_stats(st, 1)
        assert_same(emu, orc, data, off, seed=9, tcp=tcp)
        L.bb_emu_job_stats(st, 1)
        big, job_resp, unfit, masked, rounds = [int(x) for x in st]
        assert big > 0 and job_resp > 500 and rounds > big, (tcp, list(st))
        if not tcp:
            assert masked > 0, list(st)


def emulated_sharded(L, b, pkts, world):
    """Route mode of the device source picks each query's owner; the owner's shard answers it with its ingress index:
    every answer equals the unsharded oracle's."""
    dom = b.dom
    orc = H.make_impl('oracle', dom, b.snap, recursion=True)
    shards = [EmuEngine(L, dom, b.snap, recursion=True, nranks=world, rank=r) for r in range(world)]
    data, off = synth.pack_batch(pkts)
    n = len(pkts)
    owner = np.zeros(n, dtype=np.uint8)
    assert L.bb_emu_route_batch(dom.encode(), 1, data.ctypes.data, off.ctypes.data, n, world, 0, owner.ctypes.data) == 0
    o_out, o_off, o_len, o_st, o_miss = orc.resolve_batch(data, off, seed=77, qidx_base=4000)
    assert len(set(owner.tolist())) == world
    for r in range(world):
        idx = np.nonzero(owner == r)[0]
        d, o = synth.pack_batch([pkts[i] for i in idx])
        out, ooff, olen, st, miss = shards[r].resolve_batch(d, o, seed=77, qidx_map=(4000 + idx).astype(np.uint32))
        assert np.array_equal(st, o_st[idx]) and np.array_equal(olen, o_len[idx]), (r, 'status/lengths')
        for k, i in enumerate(idx):
            assert bytes(out[ooff[k]:ooff[k] + olen[k]]) == bytes(o_out[o_off[i]:o_off[i + 1]]), (r, int(i), pkts[i])
        assert sorted(int(idx[m]) for m in miss) == [int(i) for i in o_miss if owner[i] == r]


@pytest.mark.parametrize('key,world', [('five', 2), ('label63', 3), ('longest', 3), ('not-lean', 5)])
def test_emulated_sharded_pipeline(L, key, world):
    emulated_sharded(L, zone(key), zone(key).queries(seed=2), world)


# ---- 4. the GPU ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('key', KEYS)
def test_gpu_matches_oracle(key, ordered):
    b = zone(key)
    recursion = KEYS.index(key) % 2 == 0
    data, off = batch(key)
    gpu = H.make_impl('gpu', b.dom, b.snap, recursion=recursion, ordered=ordered)
    orc = H.make_impl('oracle', b.dom, b.snap, recursion=recursion)
    try:
        for profile in PROFILES:
            gpu.set_kernel_profile(profile)
            for tcp in (False, True):
                assert_same(gpu, orc, data, off, seed=11 + tcp, qidx_base=5, tcp=tcp)
    finally:
        gpu.close()


@pytest.mark.gpu
@pytest.mark.parametrize('profile', PROFILES)
def test_gpu_pinned_results(profile):
    """The kernel writing straight into pinned host memory (zero-copy results) on the 'corp' zone, UDP and TCP."""
    from test_gpu_kernel_paths import Outputs, run_slot
    from test_gpu_parity import compare
    b = zone('corp')
    data, off = batch('corp', seed=3)
    gpu = H.make_impl('gpu', b.dom, b.snap, ordered=profile == 'service')
    orc = H.make_impl('oracle', b.dom, b.snap)
    gpu.set_kernel_profile(profile)
    outs = []
    try:
        for tcp in (False, True):
            o_res = orc.resolve_batch(data, off, seed=21, qidx_base=9, tcp=tcp)
            outs.append(Outputs(len(off) - 1, len(o_res[0]) + 4096))
            compare(run_slot(gpu, 1, data, off, outs[-1], 21, qidx_base=9, tcp=tcp), o_res, data, off, gpu.ordered)
    finally:
        gpu.close()
        for o in outs:
            o.release()


@pytest.mark.gpu
@pytest.mark.parametrize('key', ['corp', 'five', 'not-lean', 'longest'])
def test_gpu_long_child_deltas(key):
    """The long children and the long "_srvce._proto" as watch events through Engine.apply_update (only the touched
    slots and the arena tail are shipped), checked after each; then a growth that lays the table out again."""
    from binder_b200.engine import Engine, Zone
    b = zone(key)
    data, off = batch(key, seed=4)
    z = Zone(b.base, b.dom)
    gpu = Engine(b.dom, recursion=True, ordered=KEYS.index(key) % 2 == 1)
    orc = H.make_impl('oracle', b.dom, b.base, recursion=True)
    try:
        gpu.swap_zone(z)
        assert_same(gpu, orc, data, off, seed=1)
        for step, (what, delta) in enumerate(b.late, 1):
            z.apply(delta)
            orc.apply_delta(delta)
            n_dirty, relaid = z.pending()
            assert n_dirty > 0 and not relaid, what
            gpu.apply_update(z)
            assert z.pending() == (0, False)
            gpu.set_kernel_profile(PROFILES[step % 2])
            assert_same(gpu, orc, data, off, seed=step, qidx_base=step * 1000, tcp=step % 2 == 1)
        grow = b.growth()
        slots0 = z.stat()['slots']
        z.apply(grow)
        orc.apply_delta(grow)
        assert z.stat()['slots'] > slots0 and z.pending()[1]
        gpu.apply_update(z)
        for profile in PROFILES:
            gpu.set_kernel_profile(profile)
            for tcp in (False, True):
                assert_same(gpu, orc, data, off, seed=40 + tcp, tcp=tcp)
    finally:
        gpu.close()
        z.close()


@pytest.mark.gpu
@pytest.mark.parametrize('key', ['five', 'lean-edge'])
def test_gpu_recursion_filter_on_own_domain(key):
    """The recursion pre-filter with region = the zone's own dnsDomain (binder's configuration), then without it."""
    b = zone(key)
    data, off = batch(key, seed=5)
    gpu = H.make_impl('gpu', b.dom, b.snap, recursion=True, ordered=key == 'five')
    orc = H.make_impl('oracle', b.dom, b.snap, recursion=True)
    dcs = ['s1', 'lk', 'nope', b.hosts[0][0].split('.')[-len(b.dom.split('.')) - 1]]
    try:
        for region in (b.dom, None):
            gpu.set_recursion_filter(region, dcs, True)
            orc.set_recursion_filter(region, dcs, True)
            g = assert_same(gpu, orc, data, off, seed=5)
            assert region is not None or len(g[4]) > 0
    finally:
        gpu.close()


@pytest.mark.gpu
@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('key,world', [('foo.co', 2), ('foo.co', 3), ('longest', 2), ('longest', 3)])
def test_gpu_sharded_cluster(L, key, world, ordered):
    """route_push_kernel and the multi-region resolve kernel on one GPU (test_gpu_shard_paths.Cluster)."""
    from test_gpu_shard_paths import Batch, Cluster, run_steps
    b = zone(key)
    orc = H.make_impl('oracle', b.dom, b.snap, recursion=True)

    def route(dom, recursion, data, off, world, rank):
        owner = np.zeros(max(len(off) - 1, 1), dtype=np.uint8)
        assert L.bb_emu_route_batch(dom.encode(), int(recursion), data.ctypes.data, off.ctypes.data, len(off) - 1, world, rank,
                                    owner.ctypes.data) == 0
        return owner[:len(off) - 1].astype(np.int64)

    def make(k, seed):
        return [Batch(b.queries(seed=100 * k + r), r, world, r * 8192 + k, seed, orc, route, b.dom, True) for r in range(world)]

    cl = Cluster(b.dom, b.snap, world, 8192, ordered=ordered, host=(1,))
    try:
        run_steps(cl, make, 2, 0x11A + world)
    finally:
        cl.close()
