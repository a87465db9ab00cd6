"""Parity tests proper: the CUDA path, called through the C ABI, must be byte-identical to the
CPU oracle (oracle/liboracle.so) — responses, offsets, status and the miss list."""
import numpy as np
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth

pytestmark = pytest.mark.gpu


from binder_b200.engine import repack


def assert_same(gpu, orc, data, off, seed=0, qidx_base=0, **kw):
    """GPU result == oracle result: status, every response's bytes, the miss set — and in
    ordered mode also the exact layout (offsets, packed bytes, ascending miss list)."""
    return compare(gpu.resolve_batch(data, off, seed=seed, qidx_base=qidx_base, **kw),
                   orc.resolve_batch(data, off, seed=seed, qidx_base=qidx_base, **kw), data, off, gpu.ordered)


def compare(res, oracle_res, data, off, ordered):
    """The checks of assert_same on results already computed: res = (out, out_off, out_len, status, miss) from the
    engine, oracle_res the same from the oracle; ordered = the engine's packing."""
    out, ooff, olen, status, miss = res
    o_out, o_off, o_len, o_status, o_miss = oracle_res
    n = len(off) - 1
    bad = np.nonzero(status != o_status)[0]
    assert bad.size == 0, ('status differs at', bad[:5], status[bad[:5]], o_status[bad[:5]])
    assert ooff[n] == o_off[n] == len(out), 'total bytes differ'
    packed, poff = repack(out, ooff, olen)
    if not np.array_equal(olen, o_len) or not np.array_equal(packed, o_out):
        for i in range(n):
            a = bytes(out[ooff[i]:ooff[i] + olen[i]]); b = bytes(o_out[o_off[i]:o_off[i + 1]])
            if a != b:
                q = bytes(data[off[i]:off[i + 1]])
                raise AssertionError('query %d %r\n gpu    %s\n oracle %s' % (i, q, a.hex(), b.hex()))
        raise AssertionError('length arrays differ')
    if ordered:
        assert np.array_equal(ooff, o_off) and np.array_equal(out, o_out) and np.array_equal(miss, o_miss)
    else:
        # arrival packing: a permutation of whole responses, no gaps, no overlap
        nz = np.nonzero(olen)[0]
        if nz.size:
            nz = nz[np.argsort(ooff[:n][nz], kind='stable')]
            st = ooff[:n][nz].astype(np.int64)
            assert st[0] == 0 and np.array_equal(st[1:], (st + olen[nz])[:-1]) and st[-1] + olen[nz][-1] == len(out)
        assert np.array_equal(np.sort(miss), o_miss)
    return packed, poff, olen, status, np.sort(miss)


MODES = [pytest.param(False, id='arrival'), pytest.param(True, id='ordered')]


def pair(dns_domain, snap, recursion=False, ordered=False, **kw):
    return (H.make_impl('gpu', dns_domain, snap, recursion=recursion, ordered=ordered),
            H.make_impl('oracle', dns_domain, snap, recursion=recursion))


@pytest.mark.parametrize('seed', range(12))
def test_fuzz_zone_parity(seed):
    snap, info = fuzzgen.gen_zone(seed, n_top=40)
    recursion = seed % 3 == 0
    gpu, orc = pair(info['dns_domain'], snap, recursion, ordered=seed % 2 == 1)
    pkts = fuzzgen.gen_queries(seed, info, n=3000) + fuzzgen.malformed_packets() + fuzzgen.tolerated_packets()
    data, off = synth.pack_batch(pkts)
    assert_same(gpu, orc, data, off, seed=seed * 1315423911 + 3, qidx_base=seed * 1000)


def test_malformed_and_not_ready():
    gpu, orc = pair('foo.com', None)
    pkts = fuzzgen.malformed_packets() + fuzzgen.tolerated_packets() + [
        synth.make_query('hosta.foo.com', 'A'), synth.make_query('1.0.0.10.in-addr.arpa', 'PTR'),
        synth.make_query('hosta.bar.org', 'A'), synth.make_query('_http._tcp.s.foo.com', 'SRV'),
        synth.make_query('x.foo.com', 'TXT')]
    data, off = synth.pack_batch(pkts)
    g = assert_same(gpu, orc, data, off)
    assert list(g[3][:len(fuzzgen.malformed_packets())]) == [2] * len(fuzzgen.malformed_packets())
    assert not gpu.is_ready()


@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('n', [0, 1, 31, 127, 128, 129, 1000])
def test_batch_size_edges(n, ordered):
    z = synth.gen_zone(3000, service_frac=0.3)
    gpu, orc = pair(z.dns_domain, z.jsonl, ordered=ordered)
    data, off = synth.pack_batch(synth.batch_mixed(z, n, seed=n))
    assert_same(gpu, orc, data, off, seed=99)


def staging_case():
    """(snapshot, packets): tiles whose packets (> 8 KB) or responses (> 12 KB) exceed the shared-memory staging."""
    kids = [('/com/foo/svc/lb%02d' % i, {'type': 'load_balancer', 'load_balancer': {'address': '10.0.0.%d' % i}})
            for i in range(30)]
    snap = H.snapshot([('/com/foo', None), ('/com/foo/svc', {'type': 'service', 'service': {
        'srvce': '_http', 'proto': '_tcp', 'port': 80}})] + kids +
        [('/com/foo/' + 'h' * 60, {'type': 'host', 'host': {'address': '10.9.9.9'}})])
    big = synth.make_query('_http._tcp.svc.foo.com', 'SRV', edns=4096) + b'\x55' * 200
    long_a = synth.make_query('H' * 60 + '.foo.com', 'A', edns=1232)
    pkts = []
    for i in range(700):
        pkts.append(big if i % 3 else long_a)
        if i % 7 == 0:
            pkts.append(synth.make_query('svc.foo.com', 'A'))
        if i % 11 == 0:
            pkts.append(b'\x00' * 5)
    return snap, pkts


@pytest.mark.parametrize('ordered', MODES)
def test_tiles_larger_than_staging(ordered):
    """Tiles whose packets (> 8 KB) or responses (> 12 KB) exceed the shared-memory staging."""
    snap, pkts = staging_case()
    gpu, orc = pair('foo.com', snap, ordered=ordered)
    data, off = synth.pack_batch(pkts)
    assert_same(gpu, orc, data, off, seed=4242)


@pytest.mark.parametrize('ordered', MODES)
def test_config2_full_size(ordered):
    """BASELINE config 2: 1M-record host zone, 65,536 uniform-hit A lookups."""
    z = synth.gen_zone(1000000)
    gpu = H.make_impl('gpu', z.dns_domain, None, ordered=ordered)
    st = gpu.load_snapshot(z.jsonl)
    assert st['nodes'] == z.n_records + 1 - 0 or st['nodes'] == z.n_records
    orc = H.make_impl('oracle', z.dns_domain, z.jsonl)
    data, off = synth.pack_batch(synth.batch_host_a(z, 65536, seed=2))
    g = assert_same(gpu, orc, data, off)
    assert (g[3] == 0).all() and len(g[0]) == 65536 * 64       # 48 B query -> 64 B answer
    # size-independent property at full size: every answer carries the address the generator
    # assigned to that host (10.x.y.z from the index in the name)
    out = g[0].reshape(65536, 64)
    names = out[:, 14:21].astype(np.int64)      # \x08 'h' then 7 digits
    idx = np.zeros(65536, dtype=np.int64)
    for k in range(7):
        idx = idx * 10 + (names[:, k] - 48)
    want = np.stack([np.full(65536, 10), (idx >> 16) & 255, (idx >> 8) & 255, idx & 255], axis=1)
    assert np.array_equal(out[:, 60:64], want)


@pytest.mark.parametrize('ordered', MODES)
def test_config3_services_and_misses(ordered):
    """Configs 3/5 in miniature plus the recursion split: services (SRV + A), 40 % absent names."""
    z = synth.gen_zone(300000, service_frac=0.15)
    gpu, orc = pair(z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    pk = synth.batch_service(z, 40000, seed=5) + synth.batch_mixed(z, 25536, seed=6, miss_frac=0.4)
    data, off = synth.pack_batch(pk)
    g = assert_same(gpu, orc, data, off, seed=0xB1DDE5)
    assert 1000 < len(g[4]) < 20000
    # same batch, different seed: only the service answers' order may change
    r2 = gpu.resolve_batch(data, off, seed=7)
    p2, o2 = repack(r2[0], r2[1], r2[2])
    assert np.array_equal(g[1], o2) and not np.array_equal(g[0], p2)


def test_pipelined_submit_wait():
    import ctypes
    from binder_b200._lib import lib, check
    z = synth.gen_zone(50000, service_frac=0.1)
    gpu, orc = pair(z.dns_domain, z.jsonl, recursion=True, ordered=True)
    L = lib()
    nslots = L.bb_engine_slots(gpu._h)
    jobs = []
    for s in range(nslots * 2):
        data, off = synth.pack_batch(synth.batch_mixed(z, 5000 + 13 * s, seed=100 + s, miss_frac=0.2))
        n = len(off) - 1
        bufs = dict(data=data, off=off, out=np.empty(n * 600, np.uint8), out_off=np.zeros(n + 1, np.uint32),
                    out_len=np.zeros(n, np.uint16), status=np.zeros(n, np.uint8), miss=np.zeros(n, np.uint32), n_miss=ctypes.c_uint32(0), n=n)
        jobs.append(bufs)
    for rnd in range(2):
        batch = jobs[rnd * nslots:(rnd + 1) * nslots]
        for s, b in enumerate(batch):
            check(L.bb_resolve_submit(gpu._h, s, b['data'].ctypes.data, b['off'].ctypes.data, b['n'], 77, 1000 * s,
                                      b['out'].ctypes.data, b['out'].size, b['out_off'].ctypes.data,
                                      b['out_len'].ctypes.data, b['status'].ctypes.data, b['miss'].ctypes.data, ctypes.byref(b['n_miss'])))
        for s, b in enumerate(batch):
            check(L.bb_resolve_wait(gpu._h, s))
            o = orc.resolve_batch(b['data'], b['off'], seed=77, qidx_base=1000 * s)
            assert np.array_equal(b['out_off'], o[1]) and np.array_equal(b['status'], o[3])
            assert np.array_equal(b['out_len'], o[2]) and np.array_equal(b['out'][:o[1][-1]], o[0])
            assert np.array_equal(b['miss'][:b['n_miss'].value], o[4])


def test_capacity_error_is_reported():
    from binder_b200._lib import BinderError
    z = synth.gen_zone(3000)
    gpu, _ = pair(z.dns_domain, z.jsonl)
    data, off = synth.pack_batch(synth.batch_host_a(z, 1000, seed=1))
    with pytest.raises(BinderError) as ei:
        gpu.resolve_batch(data, off, out_cap=4096)
    assert ei.value.code == -5


def test_device_resident_api():
    import torch
    z = synth.gen_zone(20000, service_frac=0.1)
    gpu, orc = pair(z.dns_domain, z.jsonl, ordered=True)
    data, off = synth.pack_batch(synth.batch_mixed(z, 20000, seed=3))
    n = len(off) - 1
    dev = torch.device('cuda:0')
    d_pk = torch.from_numpy(data).to(dev); d_off = torch.from_numpy(off.view(np.int32)).to(dev)
    d_out = torch.empty(n * 600, dtype=torch.uint8, device=dev); d_oo = torch.empty(n + 1, dtype=torch.int32, device=dev)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev); d_ms = torch.empty(n, dtype=torch.int32, device=dev)
    d_ol = torch.empty(n, dtype=torch.int16, device=dev)
    d_tot = torch.zeros(4, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream()
    before = gpu.launch_count()
    gpu.resolve_device(d_pk.data_ptr(), d_off.data_ptr(), n, 5, 0, d_out.data_ptr(), d_out.numel(), d_oo.data_ptr(),
                       d_ol.data_ptr(), d_st.data_ptr(), d_ms.data_ptr(), d_tot.data_ptr(), st.cuda_stream)
    st.synchronize()
    assert gpu.launch_count() == before + 1
    o = orc.resolve_batch(data, off, seed=5)
    tot = d_tot.cpu().numpy()
    assert tot[0] == o[1][-1] and tot[2] == 0 and tot[3] != 0
    assert np.array_equal(d_oo.cpu().numpy().view(np.uint32), o[1])
    assert np.array_equal(d_out.cpu().numpy()[:tot[0]], o[0])
    assert np.array_equal(d_st.cpu().numpy(), o[3]) and np.array_equal(d_ol.cpu().numpy().view(np.uint16), o[2])
