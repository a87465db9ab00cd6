"""The recursion forward and match on the GPU at the full width of their ABI (DESIGN.md section 14), bit-exact against
the forward oracle: 16 datacenters and 64 upstreams, route distributions that stress the counting sort at 65,536 misses
and at 128 k +- 1, in-label dots, contended answers racing for one miss (host and device form, both packings of the
feeding resolve), BB_MATCH_MAX_RESPONSES datagrams, repeated matches on one engine as GpuRecursion makes them, and
device-form chains resolve -> forward -> match -> relay on several streams at once."""
import random

import numpy as np
import pytest

import forward_oracle as O
import forward_ref as R
import forwardgen as G
import relay_oracle
from binder_b200 import synth
from binder_b200._lib import BinderError, lib
from binder_b200.engine import Engine, ip_u32, repack
from binder_b200.forward import GpuRecursion
from test_forward_width import (DISTRIBUTIONS, DOT_CASES, KEYS, REGION, WIDE_DCS, check_winners,
                                contended, dot_filters, dot_ups, msgs_by_miss, responses, route_batch, route_pool, run_window_cap,
                                wide_misses, wide_upstreams)
from test_gpu_forward import _zone, same

pytestmark = pytest.mark.gpu


def engine(dcs=WIDE_DCS, ups=None, region=REGION, **kw):
    e = Engine('foo.com', 'dc1', recursion=True, **kw)
    e.set_recursion_filter(region, dcs, True)
    e.set_recursion_upstreams(wide_upstreams() if ups is None else ups)
    return e


def match_both(e, tb, items, data, off, route, key):
    """Engine.match_upstreams equals the oracle; -> the oracle's (up, up_off)."""
    args = G.pack(items) + (data, off, route, key)
    want = O.match_upstreams(tb, *args)
    same(e.match_upstreams(*args), want)
    return want


# ---- 16 datacenters, 64 upstreams -----------------------------------------------------------------------------------
def test_gpu_wide_table_matches_oracle():
    ups = wide_upstreams()
    tb = O.Table(REGION, WIDE_DCS, ups)
    e = engine()
    pkts = wide_misses()
    data, off = synth.pack_batch(pkts)
    for key in KEYS:
        want = O.forward_batch(tb, data, off, key)
        same(e.forward_batch(data, off, key), want)
        routes, msgs = R.forward(REGION, WIDE_DCS, ups, pkts, key)
        assert routes == want[4].tolist() and msgs == msgs_by_miss(want, len(pkts))
        sets = {'contended': contended(ups, routes, msgs, key, random.Random(key & 0xFFF)),
                'generated': responses(ups, routes, msgs, random.Random(4), key)}
        sets.update(G.hand_written(ups, pkts, routes, msgs, key)[1])
        for name, items in sets.items():
            up, up_off = match_both(e, tb, items, data, off, want[4], key)
            if name == 'contended':
                check_winners(up, up_off, routes, msgs)


@pytest.mark.parametrize('n', [127, 129, 257, 639, 65535, 65536])
@pytest.mark.parametrize('kind', DISTRIBUTIONS)
def test_gpu_route_distributions(kind, n):
    """Every output of forward_batch (uq, uq_off, order, group_off, route) under a table where every datacenter has
    upstreams; at 65,536 misses every ID decodes to its own miss."""
    ups = wide_upstreams(holes=())
    tb = O.Table(REGION, WIDE_DCS, ups)
    pool = route_pool(ups)
    pkts = route_batch(pool, kind, n, n + DISTRIBUTIONS.index(kind))
    data, off = synth.pack_batch(pkts)
    key = KEYS[(n + DISTRIBUTIONS.index(kind)) % len(KEYS)]
    e = engine(ups=ups)
    want = O.forward_batch(tb, data, off, key)
    same(e.forward_batch(data, off, key), want)
    uq, uq_off, order, goff, route = want
    if kind == 'route15':
        assert goff[15] == 0 and goff[16] == n
    if n == 65536:
        sent = np.nonzero(uq_off[1:] > uq_off[:-1])[0]
        ids = (uq[uq_off[sent]].astype(np.uint32) << 8) | uq[uq_off[sent] + 1]
        assert len(sent) > 60000 and all(O.fwd_id(key, int(i), inverse=True) == int(order[k]) for i, k in zip(ids, sent))
    msgs = msgs_by_miss(want, n)
    items = responses(ups, route.tolist(), msgs, random.Random(n), key)
    match_both(e, tb, items, data, off, route, key)


def test_gpu_forward_uq_cap_exact():
    """bb_forward_batch with uq_cap exactly the upstream-query bytes, then one byte less (BB_ERR_CAPACITY)."""
    e = engine()
    pkts = wide_misses()
    data, off = synth.pack_batch(pkts)
    n, key = len(pkts), 0xABCDEF
    want = O.forward_batch(O.Table(REGION, WIDE_DCS, wide_upstreams()), data, off, key)
    total = int(want[1][n])
    for cap in (total, total - 1):
        uq, uq_off, order = np.zeros(cap, np.uint8), np.zeros(n + 1, np.uint32), np.zeros(n, np.uint32)
        goff, route = np.zeros(19, np.uint32), np.zeros(n, np.uint8)
        rc = lib().bb_forward_batch(e._h, data.ctypes.data, off.ctypes.data, n, key, uq.ctypes.data, cap, uq_off.ctypes.data,
                                    order.ctypes.data, goff.ctypes.data, route.ctypes.data)
        if cap == total:
            assert rc == 0
            same((uq, uq_off, order, goff, route), want)
        else:
            assert rc == -5


def test_gpu_width_limits_are_argument_errors():
    e = Engine('foo.com', 'dc1', recursion=True)
    with pytest.raises(BinderError) as ei:                 # 17 datacenters
        e.set_recursion_filter(REGION, WIDE_DCS + ['one-more'], True)
    assert ei.value.code == -1
    e.set_recursion_filter(REGION, WIDE_DCS, True)
    with pytest.raises(BinderError) as ei:                 # 65 upstreams
        e.set_recursion_upstreams(wide_upstreams() + [('10.0.0.9', 53, 0)])
    assert ei.value.code == -1
    e.set_recursion_upstreams(wide_upstreams())
    with pytest.raises(ValueError):
        GpuRecursion(e, REGION, {d: ['10.0.0.%d' % k] for k, d in enumerate(WIDE_DCS + ['one-more'])})
    e.close()


def test_gpu_in_label_dots_match_oracle():
    e = Engine('foo.com', 'dc1', recursion=True)
    cases = [(region, dcs, dot_ups(dcs), [synth.make_query(None, 'A', qid=1, labels=labels)]) for region, dcs, labels, _ in DOT_CASES]
    for fi, (region, dcs, ups, pkts) in enumerate(cases + dot_filters()):
        e.set_recursion_filter(region, dcs, True)
        e.set_recursion_upstreams(ups)
        data, off = synth.pack_batch(pkts)
        want = O.forward_batch(O.Table(region, dcs, ups), data, off, fi)
        same(e.forward_batch(data, off, fi), want)
        assert want[4].tolist() == R.forward(region, dcs, ups, pkts, fi)[0]
        if fi < len(DOT_CASES):
            assert want[4][0] == DOT_CASES[fi][3]


# ---- contended matches ----------------------------------------------------------------------------------------------
def forwarded_batch(n, seed, ups):
    """n misses of the wide filter, most of them forwarded."""
    pool = route_pool(ups)
    return route_batch(pool, 'all_routes_per_tile', n, seed)


def test_gpu_contended_matches_host_form():
    ups = wide_upstreams()
    tb = O.Table(REGION, WIDE_DCS, ups)
    e = engine()
    pkts = forwarded_batch(4096, 5, ups)
    data, off = synth.pack_batch(pkts)
    key = 0x243F6A8885A308D3
    want = O.forward_batch(tb, data, off, key)
    same(e.forward_batch(data, off, key), want)
    routes, msgs = want[4].tolist(), msgs_by_miss(want, len(pkts))
    items = contended(ups, routes, msgs, key, random.Random(6))
    up, up_off = match_both(e, tb, items, data, off, want[4], key)
    check_winners(up, up_off, routes, msgs)


class Dev(object):
    """Device copies of host arrays and zeroed device buffers (torch, cuda:0)."""

    def __init__(self):
        import torch
        self.torch, self.dev = torch, torch.device('cuda:0')

    def put(self, a, pad=0):
        a = np.ascontiguousarray(a)
        if pad:
            a = np.concatenate([a.view(np.uint8), np.zeros(pad, np.uint8)])
        return self.torch.from_numpy(a.view(np.uint8).copy()).to(self.dev)

    def zeros(self, nbytes):
        return self.torch.zeros(max(nbytes, 16), dtype=self.torch.uint8, device=self.dev)


def u32(t, k=None):
    a = t.cpu().numpy().view(np.uint32)
    return a if k is None else a[:k]


def zone_engine(ordered, ups=None):
    e = Engine('foo.com', 'dc1', recursion=True, snapshot=_zone('dc1', 200), ordered=ordered)
    e.set_recursion_filter(REGION, WIDE_DCS, True)
    e.set_recursion_upstreams(wide_upstreams() if ups is None else ups)
    return e


@pytest.mark.parametrize('ordered', [False, True])
def test_gpu_contended_matches_device_form(ordered):
    """resolve_device -> forward_device -> match_device on contended answers; the winners equal the oracle's over the
    resolve launch's own miss list (any order with arrival packing)."""
    ups = wide_upstreams()
    tb = O.Table(REGION, WIDE_DCS, ups)
    e = zone_engine(ordered)
    d = Dev()
    pkts = forwarded_batch(6000, 7 + ordered, ups)
    n = len(pkts)
    data, off = synth.pack_batch(pkts)
    d_pk, d_off = d.put(data, 16), d.put(off)
    r_out, r_off, r_len, r_st, r_miss, r_tot = d.zeros(n * 1232), d.zeros(4 * n + 4), d.zeros(2 * n), d.zeros(n), d.zeros(4 * n), d.zeros(16)
    e.resolve_device(d_pk.data_ptr(), d_off.data_ptr(), n, 3, 0, r_out.data_ptr(), n * 1232, r_off.data_ptr(), r_len.data_ptr(),
                     r_st.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr())
    d.torch.cuda.synchronize()
    m = int(u32(r_tot)[1])
    miss = u32(r_miss, m).copy()
    assert m > n // 4 and (not ordered or np.all(np.diff(miss.astype(np.int64)) > 0))
    mq, moff = synth.pack_batch([pkts[i] for i in miss])
    key = 0x13198A2E03707344 + ordered
    fwd = O.forward_batch(tb, mq, moff, key)
    routes, msgs = fwd[4].tolist(), msgs_by_miss(fwd, m)
    items = contended(ups, routes, msgs, key, random.Random(8 + ordered))
    up, up_off = O.match_upstreams(tb, *G.pack(items), mq, moff, fwd[4], key)
    check_winners(up, up_off, routes, msgs)
    cap = len(data) + 64
    f = [d.zeros(cap), d.zeros(4 * 65537), d.zeros(4 * 65536), d.zeros(4 * 19), d.zeros(65536), d.zeros(cap), d.zeros(4 * 65537), d.zeros(32)]
    e.forward_device(d_pk.data_ptr(), d_off.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr(), n, key, f[0].data_ptr(), cap,
                     f[1].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), f[4].data_ptr(), f[5].data_ptr(), cap, f[6].data_ptr(), f[7].data_ptr())
    rd, ro, rip, rport = G.pack(items)
    dr = [d.put(rd, 16), d.put(ro), d.put(rip), d.put(rport)]
    mu, muo, mt = d.zeros(len(rd) + 64), d.zeros(4 * 65537), d.zeros(16)
    e.match_device(dr[0].data_ptr(), dr[1].data_ptr(), dr[2].data_ptr(), dr[3].data_ptr(), len(items), f[5].data_ptr(),
                   f[6].data_ptr(), f[4].data_ptr(), f[7].data_ptr(), n, key, mu.data_ptr(), len(rd) + 64, muo.data_ptr(), mt.data_ptr())
    d.torch.cuda.synchronize()
    ftot = u32(f[7])
    assert ftot[1] == m and ftot[0] == fwd[1][m]
    same((f[0].cpu().numpy()[:ftot[0]], u32(f[1], m + 1), u32(f[2], m), u32(f[3]), f[4].cpu().numpy()[:m]), fwd)
    tot = u32(mt)
    assert tot[0] == up_off[m] and tot[1] == int((np.diff(up_off.astype(np.int64)) > 0).sum())
    assert np.array_equal(mu.cpu().numpy()[:tot[0]], up) and np.array_equal(u32(muo, m + 1), up_off)


def test_gpu_match_max_responses():
    """65,536 forwarded misses x 16 answers = BB_MATCH_MAX_RESPONSES datagrams, shuffled: equal to the oracle; one
    datagram more is BB_ERR_ARG."""
    ups = wide_upstreams(holes=())
    tb = O.Table(REGION, WIDE_DCS, ups)
    pool = route_pool(ups)
    del pool[R.R_NONE]
    pkts = route_batch(pool, 'blocks', 65536, 11)
    data, off = synth.pack_batch(pkts)
    key = 0xA4093822299F31D0
    e = engine(ups=ups)
    fwd = O.forward_batch(tb, data, off, key)
    same(e.forward_batch(data, off, key), fwd)
    route = fwd[4]
    assert int(fwd[3][R.R_NONE]) == 65536                 # every miss is forwarded
    rng = np.random.default_rng(12)
    by_route = [np.array([i for i, (_, _, d) in enumerate(ups) if r == R.R_PTR or d == r]) for r in range(17)]
    ip = np.array([ip_u32(a) for a, _, _ in ups], np.uint32)
    port = np.array([p for _, p, _ in ups], np.uint16)
    tails = [b'\xc0\x0c\x00\x01\x00\x01\x00\x00\x00\x3c\x00\x04' + bytes([10, 9, 0, i]) for i in range(16)]
    dgrams, src = [], np.empty(65536 * 16, np.int64)
    for k in range(65536):
        m = bytes(fwd[0][fwd[1][k]:fwd[1][k + 1]])
        head = m[:2] + bytes([0x84 | (m[2] & 0x78), 0]) + b'\x00\x01\x00\x01\x00\x00\x00\x00' + m[12:]
        dgrams += [head + t for t in tails]
        cand = by_route[route[fwd[2][k]]]
        src[16 * k:16 * k + 16] = cand[rng.integers(0, len(cand), 16)]
    perm = rng.permutation(len(dgrams))
    dgrams = [dgrams[i] for i in perm]
    src = src[perm]
    rd, ro = synth.pack_batch(dgrams)
    args = (rd, ro, ip[src], port[src], data, off, route, key)
    want = O.match_upstreams(tb, *args)
    assert int((np.diff(want[1].astype(np.int64)) > 0).sum()) == 65536
    same(e.match_upstreams(*args), want)
    rd1, ro1 = synth.pack_batch(dgrams + [dgrams[0]])
    with pytest.raises(BinderError) as ei:
        e.match_upstreams(rd1, ro1, ip[np.append(src, src[0])], port[np.append(src, src[0])], data, off, route, key)
    assert ei.value.code == -1


# ---- repeated and concurrent calls ----------------------------------------------------------------------------------
def test_gpu_repeated_prefix_matches():
    """GpuRecursion._exchange's pattern: one response list matched at growing prefixes with one key on one engine, each
    equal to the oracle on its prefix; in between, a host-form call one byte short (BB_ERR_CAPACITY) and a device-form
    call one byte short (overflow marker), each followed by an exact call; then a second window with a fresh key."""
    ups = wide_upstreams()
    tb = O.Table(REGION, WIDE_DCS, ups)
    e = engine()
    d = Dev()
    for window, key in enumerate((0x6A09E667F3BCC908, 0xBB67AE8584CAA73B)):
        pkts = forwarded_batch(3000, 20 + window, ups)
        data, off = synth.pack_batch(pkts)
        n = len(pkts)
        fwd = O.forward_batch(tb, data, off, key)
        same(e.forward_batch(data, off, key), fwd)
        routes, msgs = fwd[4].tolist(), msgs_by_miss(fwd, n)
        items = contended(ups, routes, msgs, key, random.Random(30 + window), most=8)
        L = len(items)
        d_q, d_qoff, d_route, d_ftot = d.put(data, 16), d.put(off), d.put(fwd[4], 16), d.put(np.array([0, n, 0, 0, 0], np.uint32))
        for step, k in enumerate((0, 1, 7, L // 16, L // 4, L // 2, 3 * L // 4, L - 1, L)):
            pre = items[:k]
            args = G.pack(pre) + (data, off, fwd[4], key)
            up, up_off = O.match_upstreams(tb, *args)
            if step == 4 and len(up):                       # host form, one byte short: BB_ERR_CAPACITY
                rd, ro, rip, rport = args[:4]
                buf, boff = np.zeros(len(up) - 1 + 16, np.uint8), np.zeros(n + 1, np.uint32)
                rc = lib().bb_match_upstreams(e._h, rd.ctypes.data, ro.ctypes.data, rip.ctypes.data, rport.ctypes.data, k,
                                              data.ctypes.data, off.ctypes.data, np.ascontiguousarray(fwd[4]).ctypes.data, n,
                                              key, buf.ctypes.data, len(up) - 1, boff.ctypes.data)
                assert rc == -5
            same(e.match_upstreams(*args), (up, up_off))
            if step in (5, 8):                              # device form: one byte short, then exact
                rd, ro, rip, rport = args[:4]
                dr = [d.put(rd, 16), d.put(ro), d.put(rip), d.put(rport)]
                mu, muo, mt = d.zeros(len(rd) + 64), d.zeros(4 * (n + 1)), d.zeros(16)
                for cap in (len(up) - 1, len(up)):
                    e.match_device(dr[0].data_ptr(), dr[1].data_ptr(), dr[2].data_ptr(), dr[3].data_ptr(), k, d_q.data_ptr(),
                                   d_qoff.data_ptr(), d_route.data_ptr(), d_ftot.data_ptr(), n, key, mu.data_ptr(), cap,
                                   muo.data_ptr(), mt.data_ptr())
                    d.torch.cuda.synchronize()
                    ep = lib().bb_engine_launch_epoch(e._h)
                    tot = u32(mt)
                    assert tot[3] == ep and tot[0] == len(up)
                    if cap < len(up):
                        assert tot[2] == ep
                    else:
                        assert tot[2] != ep
                        assert np.array_equal(mu.cpu().numpy()[:len(up)], up) and np.array_equal(u32(muo, n + 1), up_off)
        check_winners(up, up_off, routes, msgs)


def test_gpu_device_chains_on_streams():
    """Three chains resolve_device -> forward_device -> match_device -> relay_device on each of four streams and the
    default stream, all enqueued before any synchronisation, distinct batches and keys; each equals the oracle chain."""
    import torch
    from oracle_lib import Oracle
    ups = wide_upstreams()
    tb = O.Table(REGION, WIDE_DCS, ups)
    e = zone_engine(True)
    orc = Oracle('foo.com', 'dc1', True, snapshot=_zone('dc1', 200))
    orc.set_recursion_filter(REGION, WIDE_DCS, True)
    d = Dev()
    pool = route_pool(ups)
    hits = [synth.make_query('h%d.dc1.foo.com' % i, 'A', qid=i) for i in range(200)]
    streams = [torch.cuda.Stream() for _ in range(4)]
    chains = []
    for s in range(5):
        for c in range(3):
            seed = 100 + 3 * s + c
            rng = random.Random(seed)
            pkts = route_batch(pool, DISTRIBUTIONS[seed % 4], 2000 + 700 * c + 300 * s, seed)
            pkts = [rng.choice(hits) if rng.random() < 0.1 else p for p in pkts]
            n = len(pkts)
            data, off = synth.pack_batch(pkts)
            miss = orc.resolve_batch(data, off, seed=5)[4]
            mq, moff = synth.pack_batch([pkts[i] for i in miss])
            key = KEYS[seed % len(KEYS)] ^ seed
            fwd = O.forward_batch(tb, mq, moff, key)
            routes, msgs = fwd[4].tolist(), msgs_by_miss(fwd, len(miss))
            items = contended(ups, routes, msgs, key, rng, most=4)
            up, up_off = O.match_upstreams(tb, *G.pack(items), mq, moff, fwd[4], key)
            rel = relay_oracle.relay_batch(mq, moff, up, up_off)
            rd, ro, rip, rport = G.pack(items)
            m, cap = len(miss), len(data) + 64
            b = dict(pk=d.put(data, 16), off=d.put(off), r=[d.zeros(n * 1232), d.zeros(4 * n + 4), d.zeros(2 * n), d.zeros(n),
                                                            d.zeros(4 * n), d.zeros(16)],
                     f=[d.zeros(cap), d.zeros(4 * 65537), d.zeros(4 * 65536), d.zeros(4 * 19), d.zeros(65536), d.zeros(cap),
                        d.zeros(4 * 65537), d.zeros(32)],
                     resp=[d.put(rd, 16), d.put(ro), d.put(rip), d.put(rport)],
                     mt=[d.zeros(len(rd) + 64), d.zeros(4 * 65537), d.zeros(16)],
                     o=[d.zeros(m * 1200), d.zeros(4 * m + 4), d.zeros(2 * m), d.zeros(m), d.zeros(16)])
            chains.append((s, n, m, key, len(items), cap, fwd, (up, up_off), rel, b))
    torch.cuda.synchronize()
    for s, n, m, key, n_resp, cap, _, _, _, b in chains:
        st = streams[s].cuda_stream if s < 4 else 0
        r, f, resp, mt, o = b['r'], b['f'], b['resp'], b['mt'], b['o']
        e.resolve_device(b['pk'].data_ptr(), b['off'].data_ptr(), n, 5, 0, r[0].data_ptr(), n * 1232, r[1].data_ptr(),
                         r[2].data_ptr(), r[3].data_ptr(), r[4].data_ptr(), r[5].data_ptr(), stream=st)
        e.forward_device(b['pk'].data_ptr(), b['off'].data_ptr(), r[4].data_ptr(), r[5].data_ptr(), n, key, f[0].data_ptr(), cap,
                         f[1].data_ptr(), f[2].data_ptr(), f[3].data_ptr(), f[4].data_ptr(), f[5].data_ptr(), cap, f[6].data_ptr(),
                         f[7].data_ptr(), stream=st)
        e.match_device(resp[0].data_ptr(), resp[1].data_ptr(), resp[2].data_ptr(), resp[3].data_ptr(), n_resp, f[5].data_ptr(),
                       f[6].data_ptr(), f[4].data_ptr(), f[7].data_ptr(), n, key, mt[0].data_ptr(), mt[0].numel(), mt[1].data_ptr(),
                       mt[2].data_ptr(), stream=st)
        e.relay_device(f[5].data_ptr(), f[6].data_ptr(), mt[0].data_ptr(), mt[1].data_ptr(), m, o[0].data_ptr(), m * 1200,
                       o[1].data_ptr(), o[2].data_ptr(), o[3].data_ptr(), o[4].data_ptr(), stream=st)
    torch.cuda.synchronize()
    for i, (s, n, m, key, n_resp, cap, fwd, (up, up_off), rel, b) in enumerate(chains):
        r, f, mt, o = b['r'], b['f'], b['mt'], b['o']
        assert u32(r[5])[1] == m, i
        ftot = u32(f[7])
        assert ftot[1] == m and ftot[0] == fwd[1][m], i
        same((f[0].cpu().numpy()[:ftot[0]], u32(f[1], m + 1), u32(f[2], m), u32(f[3]), f[4].cpu().numpy()[:m]), fwd)
        tot = u32(mt[2])
        assert tot[0] == up_off[m] and np.array_equal(mt[0].cpu().numpy()[:tot[0]], up) and np.array_equal(u32(mt[1], m + 1), up_off), i
        ot = u32(o[4])
        got = (o[0].cpu().numpy()[:ot[0]], u32(o[1], m + 1), o[2].cpu().numpy().view(np.uint16)[:m], o[3].cpu().numpy()[:m])
        packed, poff = repack(*got[:3])
        assert np.array_equal(packed, rel[0]) and np.array_equal(poff, rel[1]) and np.array_equal(got[3], rel[3]), i


# ---- GpuRecursion window cap ----------------------------------------------------------------------------------------
def test_gpu_window_cap():
    e = Engine('foo.com', '', True, max_batch=256)
    run_window_cap(e)
    e.close()
