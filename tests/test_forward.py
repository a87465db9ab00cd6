"""Recursion forward and match on the CPU (DESIGN.md section 14): the C++ oracle against the independent Python
restatement on miss corpora at every filter shape and on hand-written and generated response sets; the ID bijection;
the upstream query bytes against what recursion.py's _exchange sends."""
import random
import struct

import numpy as np
import pytest

import forward_oracle as O
import forward_ref as R
import forwardgen as G
from binder_b200 import synth
from test_recursion_filter import FILTERS

KEYS = [0, 1, 0xFFFFFFFFFFFFFFFF, 0x0123456789ABCDEF, 0xDEADBEEF00000000]


def test_ids_are_a_keyed_bijection():
    for key in KEYS:
        ids = [R.fid(key, j) for j in range(65536)]
        assert sorted(ids) == list(range(65536))
        assert all(R.fid_inv(key, x) == j for j, x in enumerate(ids))
        sample = random.Random(key & 0xFFFF).sample(range(65536), 500)
        assert all(O.fwd_id(key, j) == ids[j] and O.fwd_id(key, ids[j], True) == j for j in sample)
    a, b = [R.fid(1, j) for j in range(64)], [R.fid(2, j) for j in range(64)]
    assert a != b and a != list(range(64)) and sum(x == y - 1 for x, y in zip(a, a[1:])) < 4     # not sequential


def oracle_forward(fi, pkts, key, rng):
    region, dcs, _ = FILTERS[fi]
    ups = G.upstream_table(dcs, rng)
    tb = O.Table(region, dcs, ups)
    data, off = synth.pack_batch(pkts)
    return tb, ups, O.forward_batch(tb, data, off, key)


@pytest.mark.parametrize('fi', range(len(FILTERS)))
def test_oracles_agree_on_forward(fi):
    region, dcs, _ = FILTERS[fi]
    pkts = G.misses(fi)
    key = 0x1111 * (fi + 1) << 20
    tb, ups, (uq, uq_off, order, group_off, route) = oracle_forward(fi, pkts, key, random.Random(fi))
    routes, msgs = R.forward(region, dcs, ups, pkts, key)
    assert route.tolist() == routes
    ref_order, ref_goff = R.grouped(routes)
    assert order.tolist() == ref_order and group_off.tolist() == ref_goff
    for k, j in enumerate(ref_order):
        assert bytes(uq[uq_off[k]:uq_off[k + 1]]) == msgs[j], (k, j)
    if dcs:
        assert len(set(routes)) >= 2
    # responses: oracle and Python agree on generated and hand-written sets
    rng = random.Random(50 + fi)
    q_data, q_off = synth.pack_batch(pkts)
    sets = {'generated': G.responses(ups, routes, msgs, rng, key)}
    if any(m and r < R.R_PTR for r, m in zip(routes, msgs)):
        sets.update(G.hand_written(ups, pkts, routes, msgs, key)[1])
    for name, items in sets.items():
        up, up_off = O.match_upstreams(tb, *G.pack(items), q_data, q_off, route, key)
        want = R.match(ups, items, pkts, routes, key)
        got = [bytes(up[up_off[j]:up_off[j + 1]]) for j in range(len(pkts))]
        assert got == want, name


def test_hand_written_responses():
    region, dcs, _ = FILTERS[0]
    pkts = G.misses(0)
    key = 0xA5A5A5A5A5A5A5A5
    tb, ups, (_, _, _, _, route) = oracle_forward(0, pkts, key, random.Random(3))
    routes, msgs = R.forward(region, dcs, ups, pkts, key)
    j, cases = G.hand_written(ups, pkts, routes, msgs, key)
    q_data, q_off = synth.pack_batch(pkts)
    accepted = {}
    for name, items in cases.items():
        up, up_off = O.match_upstreams(tb, *G.pack(items), q_data, q_off, route, key)
        accepted[name] = [i for i in range(len(pkts)) if up_off[i + 1] > up_off[i]]
        if name in ('duplicate', 'two_upstreams'):      # the first arrival wins
            assert accepted[name] == [j] and bytes(up[up_off[j]:up_off[j + 1]]) == items[0][0]
        else:
            assert accepted[name] == [], name
    assert {'duplicate', 'two_upstreams', 'wrong_ip', 'wrong_port', 'foreign_id', 'qr0', 'short', 'type', 'class',
            'compressed', 'none_route'} <= set(cases)


def test_upstream_query_equals_exchange(monkeypatch):
    """The upstream query with its ID masked out is the message recursion.py's _exchange sends for the same packet."""
    from binder_b200 import recursion as rmod
    sent = []

    class FakeSocket(object):
        def __init__(self, *a):
            pass

        def setblocking(self, _):
            pass

        def sendto(self, msg, addr):
            sent.append(msg)

        def close(self):
            pass

    monkeypatch.setattr(rmod.socket, 'socket', FakeSocket)
    monkeypatch.setattr(rmod.select, 'select', lambda *a: ([], [], []))
    region, dcs, _ = FILTERS[0]
    pkts = [p for p in G.misses(0) if R.parse_query(p)]
    ups = [('10.0.0.2', 53, k) for k in range(len(dcs))]
    routes, msgs = R.forward(region, dcs, ups, pkts, 7)
    rec = rmod.Recursion(None, region, {d: [('10.0.0.2', 53)] for d in dcs}, timeout=0)
    try:
        for p, rt, m in zip(pkts, routes, msgs):
            del sent[:]
            rec._exchange([(p, None, None)])
            if rt == R.R_NONE:
                assert sent == []
                continue
            assert len(sent) == (len(dcs) if rt == R.R_PTR else 1)
            assert sent[0][2:] == m[2:]
    finally:
        rec.close()
    data, off = synth.pack_batch(pkts)
    uq, uq_off, order, _, _ = O.forward_batch(O.Table(region, dcs, ups), data, off, 7)
    for k, j in enumerate(order):
        assert bytes(uq[uq_off[k] + 2:uq_off[k + 1]]) == msgs[j][2:]
        assert struct.unpack('>H', bytes(uq[uq_off[k]:uq_off[k] + 2]))[0] == R.fid(7, int(j))
    assert np.count_nonzero(np.array(routes) < R.R_NONE) > 100
