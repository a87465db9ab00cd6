"""The per-query device code (binder_b200/csrc/resolve_device.cuh) compiled for the host and run on the CPU by
tests/native/emu_resolve.cpp, against the oracle: the same source the GPU runs, checked without a GPU.  What this
does NOT cover is the CUDA kernel body itself (cooperative staging, scan, claims, flush) — the `-m gpu` tests do."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth
from test_gpu_parity import assert_same

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_EMU = {}


def emu_lib(tmp):
    if 'lib' not in _EMU:
        cxx = shutil.which('g++')
        if not cxx:
            pytest.skip('no g++')
        so = os.path.join(str(tmp), 'libbbemu.so')
        srcs = [os.path.join(ROOT, 'tests', 'native', 'emu_resolve.cpp'), os.path.join(ROOT, 'binder_b200', 'csrc', 'zone_build.cpp')]
        san = ['-g', '-fsanitize=address,undefined', '-fno-omit-frame-pointer'] if os.environ.get('BB_EMU_SANITIZE') else []   # run under LD_PRELOAD=libasan
        subprocess.check_call([cxx, '-std=c++17', '-O1', '-fPIC', '-shared', '-Wno-unknown-pragmas'] + san + ['-I', os.path.join(ROOT, 'include'),
                               '-I', os.path.join(ROOT, 'binder_b200', 'csrc'), '-o', so] + srcs)
        L = ctypes.CDLL(so)
        L.bb_zone_build.restype = ctypes.c_void_p
        L.bb_zone_build.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int)]
        L.bb_zone_free.argtypes = [ctypes.c_void_p]
        L.bb_zone_apply.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_size_t]
        L.bb_emu_resolve_batch.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_uint32,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32,
                                           ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        L.bb_zone_build_shard.restype = ctypes.c_void_p
        L.bb_zone_build_shard.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.POINTER(ctypes.c_int)]
        L.bb_emu_route_batch.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32,
                                         ctypes.c_uint32, ctypes.c_void_p]
        _EMU['lib'] = L
    return _EMU['lib']


class EmuEngine(object):
    """Engine look-alike over bb_emu_resolve_batch (query-order packing, like ordered_output=1)."""
    ordered = True

    def __init__(self, L, dns_domain, snap, recursion=False, nranks=1, rank=0):
        self.L, self.dom, self.recursion, self.rf = L, dns_domain.encode(), recursion, None
        self.zone = None
        if snap is not None:
            err = ctypes.c_int(0)
            self.zone = L.bb_zone_build_shard(snap, len(snap), self.dom, nranks, rank, ctypes.byref(err))
            assert self.zone, err.value

    def apply(self, delta):
        assert self.L.bb_zone_apply(self.zone, delta, len(delta)) == 0

    def set_recursion_filter(self, region, dcs=(), ptr=False):
        self.rf = None if region is None else (region.encode('latin-1'), [d.encode('latin-1') for d in dcs], ptr)

    def resolve_batch(self, data, off, seed=0, qidx_base=0, tcp=False, qidx_map=None):
        data = np.ascontiguousarray(data, dtype=np.uint8); off = np.ascontiguousarray(off, dtype=np.uint32)
        n = len(off) - 1
        cap = max(4096, min(n * (65536 if tcp else 1232), 0xFFFFFF00))
        out = np.zeros(cap, dtype=np.uint8); ooff = np.zeros(n + 1, dtype=np.uint32); olen = np.zeros(max(n, 1), dtype=np.uint16)
        st = np.zeros(max(n, 1), dtype=np.uint8); miss = np.zeros(max(n, 1), dtype=np.uint32); nm = ctypes.c_uint32(0)
        region, arr, ndc, ptr = None, None, 0, 0
        if self.rf:
            region, dcs, ptr = self.rf
            arr = (ctypes.c_char_p * max(len(dcs), 1))(*dcs); ndc = len(dcs)
        rc = self.L.bb_emu_resolve_batch(self.zone, self.dom, int(self.recursion), region, arr, ndc, int(ptr), data.ctypes.data, off.ctypes.data, n,
                                         seed, qidx_base, 1, int(tcp), out.ctypes.data, cap, ooff.ctypes.data, olen.ctypes.data,
                                         st.ctypes.data, miss.ctypes.data, ctypes.byref(nm),
                                         None if qidx_map is None else np.ascontiguousarray(qidx_map, dtype=np.uint32).ctypes.data)
        assert rc == 0, rc
        return out[:ooff[n]].copy(), ooff, olen[:n], st[:n], miss[:nm.value].copy()


@pytest.fixture(scope='module')
def L(tmp_path_factory):
    return emu_lib(tmp_path_factory.mktemp('emu'))


@pytest.mark.parametrize('seed', range(12))
def test_device_source_on_cpu_matches_oracle(L, seed):
    snap, info = fuzzgen.gen_zone(seed, n_top=40)
    recursion = seed % 3 == 0
    emu = EmuEngine(L, info['dns_domain'], snap, recursion)
    orc = H.make_impl('oracle', info['dns_domain'], snap, recursion=recursion)
    pkts = fuzzgen.gen_queries(seed, info, n=3000) + fuzzgen.malformed_packets() + fuzzgen.tolerated_packets()
    data, off = synth.pack_batch(pkts)
    assert_same(emu, orc, data, off, seed=seed * 1315423911 + 3, qidx_base=seed * 1000)
    assert_same(emu, orc, data, off, seed=seed + 1, tcp=True)


def test_emulated_not_ready_and_edges(L):
    emu = EmuEngine(L, 'foo.com', None)
    orc = H.make_impl('oracle', 'foo.com', None)
    pkts = fuzzgen.malformed_packets() + fuzzgen.tolerated_packets() + [
        synth.make_query('hosta.foo.com', 'A'), synth.make_query('1.0.0.10.in-addr.arpa', 'PTR'),
        synth.make_query('hosta.bar.org', 'A'), synth.make_query('_http._tcp.s.foo.com', 'SRV'), synth.make_query('x.foo.com', 'TXT')]
    data, off = synth.pack_batch(pkts)
    assert_same(emu, orc, data, off)
    for n in (0, 1, 127, 128, 129):
        d, o = synth.pack_batch(pkts[:n] if n <= len(pkts) else (pkts * 8)[:n])
        assert_same(emu, orc, d, o, seed=n)


@pytest.mark.parametrize('seed', range(4))
def test_emulated_updates_filter(L, seed):
    """Deltas (bb_zone_apply) and the recursion pre-filter through the emulated device code."""
    snap, info = fuzzgen.gen_zone(seed + 300, n_top=30)
    emu = EmuEngine(L, info['dns_domain'], snap, recursion=True)
    orc = H.make_impl('oracle', info['dns_domain'], snap, recursion=True)
    paths = fuzzgen.snapshot_paths(snap)
    for rnd in range(3):
        delta, paths = fuzzgen.gen_delta(seed * 100 + rnd, paths, info, n_ops=50)
        emu.apply(delta); orc.apply_delta(delta)
        data, off = synth.pack_batch(fuzzgen.gen_queries(seed * 17 + rnd, info, n=1500))
        assert_same(emu, orc, data, off, seed=rnd)
    for region, dcs, ptr in (('foo.com', ['web', 'h1', 'nope', 'c'], True), ('oo.com', ['web'], False), ('com', ['foo'], True)):
        emu.set_recursion_filter(region, dcs, ptr); orc.set_recursion_filter(region, dcs, ptr)
        assert_same(emu, orc, data, off, seed=9)


def test_emulated_large_answers_over_tcp(L):
    from test_tcp import big_zone
    snap = big_zone()
    emu = EmuEngine(L, 'foo.com', snap)
    orc = H.make_impl('oracle', 'foo.com', snap)
    pk = [synth.make_query('_http._tcp.big.foo.com', 'SRV'), synth.make_query('big.foo.com', 'A'), synth.make_query('_http._tcp.huge.foo.com', 'SRV'),
          synth.make_query('huge.foo.com', 'A'), synth.make_query('hosta.foo.com', 'A', edns=4096)] * 30
    data, off = synth.pack_batch(pk)
    assert_same(emu, orc, data, off, seed=3, tcp=True)
    assert_same(emu, orc, data, off, seed=3)


@pytest.mark.parametrize('seed,world', [(0, 2), (1, 3), (2, 8), (3, 5)])
def test_emulated_sharded_pipeline(L, seed, world):
    """The whole sharded path on the CPU: route mode of the device code picks each query's owner, the owner's shard
    (bb_zone_build_shard) resolves it with the query's ingress index — every answer must equal the unsharded oracle's."""
    snap, info = fuzzgen.gen_zone(seed + 600, n_top=35)
    dom = info['dns_domain']
    orc = H.make_impl('oracle', dom, snap, recursion=True)
    shards = [EmuEngine(L, dom, snap, recursion=True, nranks=world, rank=r) for r in range(world)]
    pkts = fuzzgen.gen_queries(seed, info, n=2500) + fuzzgen.malformed_packets()
    data, off = synth.pack_batch(pkts)
    n = len(pkts)
    ingress = 1 % world                                        # the rank these queries arrive at
    owner = np.zeros(n, dtype=np.uint8)
    assert L.bb_emu_route_batch(dom.encode(), 1, data.ctypes.data, off.ctypes.data, n, world, ingress, owner.ctypes.data) == 0
    o_out, o_off, o_len, o_st, o_miss = orc.resolve_batch(data, off, seed=77, qidx_base=4000)
    assert len(set(owner.tolist())) > 1 or world == 1
    seen = 0
    for r in range(world):
        idx = np.nonzero(owner == r)[0]
        if idx.size == 0:
            continue
        sub = [pkts[i] for i in idx]
        d, o = synth.pack_batch(sub)
        out, ooff, olen, st, miss = shards[r].resolve_batch(d, o, seed=77, qidx_map=(4000 + idx).astype(np.uint32))
        assert np.array_equal(st, o_st[idx]) and np.array_equal(olen, o_len[idx]), (r, 'status/lengths')
        for k, i in enumerate(idx):
            assert bytes(out[ooff[k]:ooff[k] + olen[k]]) == bytes(o_out[o_off[i]:o_off[i + 1]]), (r, int(i), pkts[i])
        assert sorted(int(idx[m]) for m in miss) == [int(i) for i in o_miss if owner[i] == r]
        seen += idx.size
    assert seen == n


def padded_queries(lengths):
    """A valid query padded with trailing bytes to each length (and a short query after each): a DNS message is at
    most 65,535 bytes, so the padded ones up to that are answered and the longer ones are dropped."""
    pk = []
    for i, ln in enumerate(lengths):
        q = synth.make_query('hosta.foo.com' if i % 2 == 0 else '_http._tcp.svc.foo.com', 'A' if i % 2 == 0 else 'SRV', qid=i)
        pk += [q + bytes([0x41 + i % 7]) * (ln - len(q)), synth.make_query('hostb.foo.com', 'A', qid=1000 + i)]
    return pk


def size_zone():
    return H.snapshot([('/com/foo', None), ('/com/foo/hosta', {'type': 'host', 'host': {'address': '10.0.0.1'}}),
                       ('/com/foo/hostb', {'type': 'host', 'host': {'address': '10.0.0.2'}}),
                       ('/com/foo/svc', {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80}}),
                       ('/com/foo/svc/lb0', {'type': 'load_balancer', 'load_balancer': {'address': '10.1.0.1'}})])


@pytest.mark.parametrize('tcp', [False, True], ids=['udp', 'tcp'])
def test_emulated_packet_length_limit(L, tcp):
    """Packets of 65,534 and 65,535 bytes are queries (trailing bytes ignored); 65,536 and 70,000 bytes are dropped,
    by the device code and the oracle alike."""
    snap = size_zone()
    emu = EmuEngine(L, 'foo.com', snap)
    orc = H.make_impl('oracle', 'foo.com', snap)
    lengths = [65534, 65535, 65536, 70000, 65535, 70000]
    data, off = synth.pack_batch(padded_queries(lengths))
    g = assert_same(emu, orc, data, off, seed=5, tcp=tcp)
    assert list(g[3][0::2]) == [0, 0, 2, 2, 0, 2] and (g[3][1::2] == 0).all()


def _path_counts(L, reset=True):
    c = (ctypes.c_ulonglong * 2)()
    L.bb_emu_path_counts(c, int(reset))
    return int(c[0]), int(c[1])


@pytest.mark.parametrize('workload', ['config2', 'config3', 'config4', 'config5'])
def test_workloads_take_the_lean_front_end(L, workload):
    """Every query shape of the BASELINE.json configs is settled by lean_query (the word-wise front end): the general
    path (complete decoder + byte-serial resolve) is for unusual packets only.  Also bit-exact against the oracle,
    hits, misses, services, NOTIMP and EDNS included."""
    desc, service_frac, mix, miss_frac, recursion = synth.WORKLOADS[workload]
    z = synth.gen_zone(30000, service_frac=service_frac)
    emu = EmuEngine(L, z.dns_domain, z.jsonl, recursion)
    orc = H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=recursion)
    data, off, meta = synth.gen_batch(z, 6000, 5, mix, miss_frac)
    _path_counts(L)
    assert_same(emu, orc, data, off, seed=11)
    lean, general = _path_counts(L)
    assert general == 0 and lean == 6000, (lean, general)
    # the same names with an OPT, upper-case letters, RD=0: still the lean path
    pk = []
    for i in range(0, 6000, 7):
        k, ix = int(meta['kind'][i]), int(meta['idx'][i])
        name = synth.host_name(ix) if k <= synth.K_HOST_AAAA else synth.svc_name(ix)
        cut = len(name) - len(z.dns_domain)                 # the suffix gate is case-sensitive: only what precedes dnsDomain varies
        name = (name[:cut].upper() if i % 3 == 0 else name[:3].upper() + name[3:cut]) + name[cut:]
        if k == synth.K_SVC_SRV:
            name = '_http._tcp.' + name
        pk.append(synth.make_query(name, {0: 1, 1: 28, 2: 1, 3: 33}[k], i & 0xFFFF, rd=bool(i & 1), edns=(4096 if i % 2 else 600)))
    d2, o2 = synth.pack_batch(pk)
    assert_same(emu, orc, d2, o2, seed=12)
    lean, general = _path_counts(L)
    assert general == 0, (lean, general)


def test_fuzz_queries_mostly_lean(L):
    snap, info = fuzzgen.gen_zone(5, n_top=40)
    emu = EmuEngine(L, info['dns_domain'], snap, True)
    data, off = synth.pack_batch(fuzzgen.gen_queries(5, info, n=3000))
    _path_counts(L)
    emu.resolve_batch(data, off, seed=1)
    lean, general = _path_counts(L)
    assert lean > general, (lean, general)


def job_zone():
    """Services whose answers exercise the copy-job machinery of big tiles: 3..14 children, some with several ports
    (a truncated answer then cuts a run of SRV RRs short), a null-address child, a child with its own ttl."""
    ent = [('/com/foo', None)]
    for s in range(24):
        ent.append(('/com/foo/svc%02d' % s, {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80 + s, 'ttl': 30 + s}}))
        for k in range(3 + s % 12):
            if (s + k) % 5 == 0:
                rec = {'type': 'rr_host', 'rr_host': {'address': '10.%d.%d.1' % (s, k), 'ports': [8000 + k, 8100 + k, 8200 + k]}}
            elif (s + k) % 7 == 3:
                rec = {'type': 'load_balancer', 'load_balancer': {'address': None}}
            elif (s + k) % 4 == 1:
                rec = {'type': 'load_balancer', 'load_balancer': {'address': '10.%d.%d.2' % (s, k), 'ttl': 7 + k}}
            else:
                rec = {'type': 'load_balancer', 'load_balancer': {'address': '10.%d.%d.3' % (s, k)}}
            ent.append(('/com/foo/svc%02d/%s%d' % (s, 'backend-number-' if k % 3 == 0 else 'lb', k), rec))
    return H.snapshot(ent)


@pytest.mark.parametrize('edns', [0, 1200, 700])
def test_emulated_copy_jobs_edges(L, edns):
    """Big tiles of service answers: more jobs than the list holds (the threads behind the first that does not fit write
    their own answers), answers truncated in the middle of a multi-port child's SRV run (a job whose source does not
    end in padding), the OPT as a job, several emit rounds per tile, upper-case names (not job mode) mixed in."""
    snap = job_zone()
    emu = EmuEngine(L, 'foo.com', snap)
    orc = H.make_impl('oracle', 'foo.com', snap)
    pk = []
    for i in range(700):
        s = (i * 7) % 24
        name = 'svc%02d.foo.com' % s
        if i % 11 == 0:
            name = name.upper()[:5] + name[5:]
        if i % 3 == 2:
            pk.append(synth.make_query(name, 'A', i, edns=edns))
        else:
            pk.append(synth.make_query('_http._tcp.' + name, 'SRV', i, edns=edns))
    data, off = synth.pack_batch(pk)
    st = (ctypes.c_ulonglong * 5)()
    L.bb_emu_job_stats(st, 1)
    for seed in (1, 2):
        assert_same(emu, orc, data, off, seed=seed)
    L.bb_emu_job_stats(st, 1)
    big, job_resp, unfit, masked, rounds = [int(x) for x in st]
    assert big >= 10 and job_resp > 500 and rounds > 2 * big, list(st)
    if edns == 1200:
        assert unfit > 0, list(st)          # whole answers: more jobs than the list holds
    else:
        assert masked > 0, list(st)         # truncated answers: SRV runs cut short
