"""Recursion forward and match on the GPU (DESIGN.md section 14): Engine.forward_batch and Engine.match_upstreams
bit-exact against the CPU oracle at every filter shape, at batch-size edges, with their error cases; the device-resident
forms straight from a resolve launch; and one device-resident chain resolve -> forward -> (a dc2 oracle answers) ->
match -> relay equal to the oracle's chain."""
import random

import numpy as np
import pytest

import forward_oracle as O
import forward_ref as R
import forwardgen as G
import helpers as H
import relay_oracle
from binder_b200 import synth
from binder_b200._lib import BinderError, lib
from binder_b200.engine import Engine, ip_u32
from test_recursion_filter import FILTERS

pytestmark = pytest.mark.gpu


def engine(region, dcs, ups, snapshot=None, max_batch=1 << 16, dom='example.com'):
    e = Engine(dom, 'dc1', recursion=True, snapshot=snapshot, max_batch=max_batch)
    e.set_recursion_filter(region, dcs, True)
    e.set_recursion_upstreams(ups)
    return e


def same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


@pytest.mark.parametrize('fi', range(len(FILTERS)))
def test_gpu_forward_and_match_match_oracle(fi):
    region, dcs, _ = FILTERS[fi]
    ups = G.upstream_table(dcs, random.Random(fi))
    if not ups:
        pytest.skip('a filter without datacenters has no upstream table')
    pkts = G.misses(fi)
    key = 0x5151 * (fi + 3) << 17
    tb = O.Table(region, dcs, ups)
    e = engine(region, dcs, ups)
    data, off = synth.pack_batch(pkts)
    got = e.forward_batch(data, off, key)
    want = O.forward_batch(tb, data, off, key)
    same(got, want)
    routes, msgs = R.forward(region, dcs, ups, pkts, key)
    sets = {'generated': G.responses(ups, routes, msgs, random.Random(70 + fi), key)}
    if any(m and r < R.R_PTR for r, m in zip(routes, msgs)):
        sets.update(G.hand_written(ups, pkts, routes, msgs, key)[1])
    for name, items in sets.items():
        args = G.pack(items) + (data, off, want[4], key)
        same(e.match_upstreams(*args), O.match_upstreams(tb, *args))


@pytest.mark.parametrize('n', [0, 1, 127, 128, 129, 65536])
def test_gpu_forward_batch_sizes(n):
    region, dcs, _ = FILTERS[0]
    ups = G.upstream_table(dcs, random.Random(1))
    base = [p for p in G.misses(0)]
    pkts = [base[i % len(base)] for i in range(n)]
    data, off = synth.pack_batch(pkts) if n else (np.zeros(16, np.uint8), np.zeros(1, np.uint32))
    e = engine(region, dcs, ups)
    tb = O.Table(region, dcs, ups)
    key = 0x77 + n
    want = O.forward_batch(tb, data, off, key)
    same(e.forward_batch(data, off, key), want)
    if n == 65536:
        uq, uq_off = want[0], want[1]
        ids = (uq[uq_off[:-1]].astype(np.uint32) << 8) | uq[uq_off[:-1] + 1]
        nonempty = uq_off[1:] > uq_off[:-1]
        assert len(np.unique(ids[nonempty])) == int(nonempty.sum())
    routes, msgs = R.forward(region, dcs, ups, pkts, key)
    items = G.responses(ups, routes, msgs, random.Random(n), key)
    args = G.pack(items) + (data, off, want[4], key)
    same(e.match_upstreams(*args), O.match_upstreams(tb, *args))


def test_gpu_forward_errors():
    region, dcs, _ = FILTERS[0]
    ups = G.upstream_table(dcs, random.Random(2))
    pkts = G.misses(0)[:50]
    data, off = synth.pack_batch(pkts)
    e = Engine('example.com', 'dc1', recursion=True, max_batch=1 << 17)
    with pytest.raises(BinderError) as ei:                  # no filter
        e.forward_batch(data, off, 1)
    assert ei.value.code == -1
    with pytest.raises(BinderError) as ei:                  # upstreams need a filter
        e.set_recursion_upstreams(ups)
    assert ei.value.code == -1
    e.set_recursion_filter(region, dcs, True)
    with pytest.raises(BinderError) as ei:                  # no upstream table
        e.forward_batch(data, off, 1)
    assert ei.value.code == -1
    with pytest.raises(BinderError) as ei:                  # a datacenter index the filter does not have
        e.set_recursion_upstreams([('10.0.0.1', 53, len(dcs))])
    assert ei.value.code == -1
    e.set_recursion_upstreams(ups)
    big = [pkts[i % len(pkts)] for i in range(65537)]
    bd, bo = synth.pack_batch(big)
    with pytest.raises(BinderError) as ei:                  # n > 65,536
        e.forward_batch(bd, bo, 1)
    assert ei.value.code == -1
    want = O.forward_batch(O.Table(region, dcs, ups), data, off, 5)
    routes, msgs = R.forward(region, dcs, ups, pkts, 5)
    items = [(G.answer_for(m, random.Random(j)), (ups[0][0], ups[0][1])) for j, m in enumerate(msgs) if m]
    resp = G.pack(items)
    full = O.match_upstreams(O.Table(region, dcs, ups), *resp, data, off, want[4], 5)
    assert len(full[0]) > 0
    up = np.zeros(len(full[0]) - 1 if len(full[0]) else 0, np.uint8)
    up_off = np.zeros(len(pkts) + 1, np.uint32)
    rc = lib().bb_match_upstreams(e._h, resp[0].ctypes.data, resp[1].ctypes.data, resp[2].ctypes.data, resp[3].ctypes.data,
                                  len(items), data.ctypes.data, off.ctypes.data, np.ascontiguousarray(want[4]).ctypes.data,
                                  len(pkts), 5, up.ctypes.data, len(up), up_off.ctypes.data)
    assert rc == -5                                          # BB_ERR_CAPACITY
    uq = np.zeros(8, np.uint8)
    rc = lib().bb_forward_batch(e._h, data.ctypes.data, off.ctypes.data, len(pkts), 5, uq.ctypes.data, 8,
                                np.zeros(len(pkts) + 1, np.uint32).ctypes.data, np.zeros(len(pkts), np.uint32).ctypes.data,
                                np.zeros(19, np.uint32).ctypes.data, np.zeros(len(pkts), np.uint8).ctypes.data)
    assert rc == -5
    # setting the filter again clears the upstream table: its datacenter indices referred to the old list
    e.set_recursion_filter(region, list(reversed(dcs)), True)
    with pytest.raises(BinderError) as ei:
        e.forward_batch(data, off, 1)
    assert ei.value.code == -1
    e.set_recursion_upstreams(ups)
    e.forward_batch(data, off, 1)
    e.set_recursion_filter(None)
    with pytest.raises(BinderError) as ei:
        e.forward_batch(data, off, 1)
    assert ei.value.code == -1


def _zone(dc, n):
    ent = [('/com/foo/%s' % dc, None)]
    ent += [('/com/foo/%s/h%d' % (dc, i), {'type': 'host', 'host': {'address': '10.%d.0.%d' % (2 if dc == 'dc2' else 1, i % 250)}})
            for i in range(n)]
    return H.snapshot(ent)


def chain_batch(n, seed):
    """A config-5-shaped batch at dc1: 10 % hits, the rest misses for dc2 (answered there), dc3 (silent), PTR, nowhere."""
    rng = random.Random(seed)
    pkts = []
    for i in range(n):
        x = rng.random()
        if x < 0.1:
            name, t = 'h%d.dc1.foo.com' % rng.randrange(200), 'A'
        elif x < 0.8:
            name, t = 'h%d.dc2.foo.com' % rng.randrange(300), 'A'
        elif x < 0.88:
            name, t = 'h%d.dc3.foo.com' % rng.randrange(300), 'A'
        elif x < 0.93:
            name, t = '%d.0.2.10.in-addr.arpa' % rng.randrange(200), 'PTR'
        else:
            name, t = 'h%d.nodc.foo.com' % rng.randrange(300), 'A'
        pkts.append(synth.make_query(name, t, qid=rng.randrange(65536), edns=rng.choice([None, 1200])))
    return pkts


def test_gpu_device_chain_equals_oracle_chain():
    import torch
    from oracle_lib import Oracle
    dev = torch.device('cuda:0')
    region, dcs = 'foo.com', ['dc2', 'dc3']
    ups = [('127.0.0.1', 5302, 0), ('10.0.0.2', 53, 0), ('127.0.0.1', 5303, 1)]
    tb = O.Table(region, dcs, ups)
    e = engine(region, dcs, ups, snapshot=_zone('dc1', 200), dom='foo.com')
    dc1 = Oracle('foo.com', '', True, snapshot=_zone('dc1', 200))
    dc1.set_recursion_filter(region, dcs, True)
    dc2 = Oracle('foo.com', '', False, snapshot=_zone('dc2', 300))
    n = 60000
    pkts = chain_batch(n, 9)
    data, off = synth.pack_batch(pkts)
    key = 0xC0FFEE1234567
    # device resolve
    t = lambda a, dt=torch.uint8: torch.from_numpy(np.ascontiguousarray(a)).to(dev)      # noqa: E731
    d_pk = t(np.concatenate([data, np.zeros(16, np.uint8)]))
    d_off = t(off.view(np.int32))
    cap = len(data) + 64
    z = lambda k, dt=torch.int32: torch.zeros(k, dtype=dt, device=dev)                    # noqa: E731
    r_out, r_off, r_len, r_st, r_miss, r_tot = z(n * 1232, torch.uint8), z(n + 1), z(n, torch.int16), z(n, torch.uint8), z(n), z(4)
    e.resolve_device(d_pk.data_ptr(), d_off.data_ptr(), n, 3, 0, r_out.data_ptr(), n * 1232, r_off.data_ptr(), r_len.data_ptr(),
                     r_st.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr())
    torch.cuda.synchronize()
    # the forward runs on the resolve launch's own miss list, in the order that launch wrote it (arrival packing: any
    # order); the oracle's chain is taken over the same misses in the same order
    miss = r_miss.cpu().numpy()[:int(r_tot.cpu().numpy()[1])].view(np.uint32).copy()
    _, _, _, _, omiss = dc1.resolve_batch(data, off, seed=3)
    assert np.array_equal(np.sort(miss), np.sort(omiss))
    # oracle chain
    mq, moff = synth.pack_batch([pkts[i] for i in miss])
    f = O.forward_batch(tb, mq, moff, key)
    uq, uq_off, order, goff, route = f

    def upstream_answers(uq, uq_off, goff):
        """dc2 answers the queries of route 0 (and the PTR run) from its first upstream; dc3 never answers."""
        sel = [k for k in range(int(goff[0]), int(goff[1]))] + [k for k in range(int(goff[16]), int(goff[17]))]
        qs = [bytes(uq[uq_off[k]:uq_off[k + 1]]) for k in sel]
        d, o = synth.pack_batch(qs)
        out, ooff, olen, st2, _ = dc2.resolve_batch(d, o, seed=1)
        return [(bytes(out[ooff[i]:ooff[i] + olen[i]]), ('127.0.0.1', 5302)) for i in range(len(qs)) if st2[i] == 0]

    items = upstream_answers(uq, uq_off, goff)
    up, up_off = O.match_upstreams(tb, *G.pack(items), mq, moff, route, key)
    want = relay_oracle.relay_batch(mq, moff, up, up_off)

    # device chain
    f_uq, f_uqoff, f_order, f_goff, f_route = z(cap, torch.uint8), z(65537), z(65536), z(19), z(65536, torch.uint8)
    f_q, f_qoff, f_tot = z(cap, torch.uint8), z(65537), z(8)
    e.forward_device(d_pk.data_ptr(), d_off.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr(), n, key, f_uq.data_ptr(), cap,
                     f_uqoff.data_ptr(), f_order.data_ptr(), f_goff.data_ptr(), f_route.data_ptr(), f_q.data_ptr(), cap,
                     f_qoff.data_ptr(), f_tot.data_ptr())
    torch.cuda.synchronize()
    ftot = f_tot.cpu().numpy().view(np.uint32)
    ep = lib().bb_engine_launch_epoch(e._h)
    m = len(miss)
    assert ftot[1] == m and ftot[2] != ep and ftot[3] == ep and ftot[0] == uq_off[m] and ftot[4] == moff[m]
    ftot = ftot.copy()
    g_uqoff = f_uqoff.cpu().numpy().view(np.uint32)[:m + 1]
    g = (f_uq.cpu().numpy()[:ftot[0]], g_uqoff, f_order.cpu().numpy().view(np.uint32)[:m],
         f_goff.cpu().numpy().view(np.uint32), f_route.cpu().numpy()[:m])
    same(g, f)
    assert np.array_equal(f_q.cpu().numpy()[:ftot[4]], mq[:moff[m]])
    assert np.array_equal(f_qoff.cpu().numpy().view(np.uint32)[:m + 1], moff)
    rd, ro, rip, rport = G.pack(items)
    d_rd, d_ro, d_rip, d_rport = t(np.concatenate([rd, np.zeros(16, np.uint8)])), t(ro.view(np.int32)), t(rip.view(np.int32)), \
        t(rport.view(np.int16))
    m_up, m_upoff, m_tot = z(len(rd) + 64, torch.uint8), z(65537), z(4)
    e.match_device(d_rd.data_ptr(), d_ro.data_ptr(), d_rip.data_ptr(), d_rport.data_ptr(), len(items), f_q.data_ptr(),
                   f_qoff.data_ptr(), f_route.data_ptr(), f_tot.data_ptr(), n, key, m_up.data_ptr(), len(rd) + 64,
                   m_upoff.data_ptr(), m_tot.data_ptr())
    out_cap = m * 1200
    o_out, o_off, o_len, o_st, o_tot = z(out_cap, torch.uint8), z(m + 1), z(m, torch.int16), z(m, torch.uint8), z(4)
    e.relay_device(f_q.data_ptr(), f_qoff.data_ptr(), m_up.data_ptr(), m_upoff.data_ptr(), m, o_out.data_ptr(), out_cap,
                   o_off.data_ptr(), o_len.data_ptr(), o_st.data_ptr(), o_tot.data_ptr())
    torch.cuda.synchronize()
    mt = m_tot.cpu().numpy().view(np.uint32)
    assert mt[0] == up_off[m] and mt[1] == int((np.diff(up_off.astype(np.int64)) > 0).sum()) and mt[1] > m // 2
    assert np.array_equal(m_up.cpu().numpy()[:mt[0]], up) and np.array_equal(m_upoff.cpu().numpy().view(np.uint32)[:m + 1], up_off)
    from binder_b200.engine import repack
    ot = o_tot.cpu().numpy().view(np.uint32)
    got = (o_out.cpu().numpy()[:ot[0]], o_off.cpu().numpy().view(np.uint32), o_len.cpu().numpy().view(np.uint16), o_st.cpu().numpy())
    packed, poff = repack(*got[:3])
    assert np.array_equal(packed, want[0]) and np.array_equal(poff, want[1]) and np.array_equal(got[3], want[3])
    # device-form capacity: the responses one byte over up_cap, the upstream queries over uq_cap, the client queries over
    # q_cap, the miss count over n_cap — each sets the call's error marker in its totals
    e.match_device(d_rd.data_ptr(), d_ro.data_ptr(), d_rip.data_ptr(), d_rport.data_ptr(), len(items), f_q.data_ptr(),
                   f_qoff.data_ptr(), f_route.data_ptr(), f_tot.data_ptr(), n, key, m_up.data_ptr(), int(mt[0]) - 1,
                   m_upoff.data_ptr(), m_tot.data_ptr())
    torch.cuda.synchronize()
    ep = lib().bb_engine_launch_epoch(e._h)
    mt2 = m_tot.cpu().numpy().view(np.uint32)
    assert mt2[2] == ep and mt2[3] == ep
    for uq_cap, q_cap in ((int(ftot[0]) - 1, cap), (cap, int(ftot[4]) - 1)):
        e.forward_device(d_pk.data_ptr(), d_off.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr(), n, key, f_uq.data_ptr(), uq_cap,
                         f_uqoff.data_ptr(), f_order.data_ptr(), f_goff.data_ptr(), f_route.data_ptr(), f_q.data_ptr(), q_cap,
                         f_qoff.data_ptr(), f_tot.data_ptr())
        torch.cuda.synchronize()
        ep = lib().bb_engine_launch_epoch(e._h)
        assert f_tot.cpu().numpy().view(np.uint32)[2] == ep, (uq_cap, q_cap)
    e.forward_device(d_pk.data_ptr(), d_off.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr(), m - 1, key, f_uq.data_ptr(), cap,
                     f_uqoff.data_ptr(), f_order.data_ptr(), f_goff.data_ptr(), f_route.data_ptr(), f_q.data_ptr(), cap,
                     f_qoff.data_ptr(), f_tot.data_ptr())
    torch.cuda.synchronize()
    ep = lib().bb_engine_launch_epoch(e._h)
    ftot = f_tot.cpu().numpy().view(np.uint32)
    assert ftot[2] == ep and ftot[1] == 0
    assert ip_u32('127.0.0.1') == 0x7F000001
