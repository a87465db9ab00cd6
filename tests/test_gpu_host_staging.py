"""The synchronous host-buffer calls of one recursion engine share one device staging block (DESIGN.md section 13):
resolve_batch, relay_batch (pageable and pinned results), forward_batch, match_upstreams and log_batch (pageable, and
pinned with and without a summary), interleaved, bit-exact against the CPU oracles and the query log restatement.
Batch sizes go small, large, small, large, so each call cuts its pieces out of a block that an earlier call of another
kind grew and left full of its own bytes.  Device-form relay and forward calls on two other
streams run alongside, on their own placement and forward scratch.  A relay that overflows its capacity is followed by an
exact one on the same engine."""
import random

import numpy as np
import pytest

import forward_oracle as O
import forwardgen as G
import query_log_ref as L
import relay_oracle
import relaygen as RG
from binder_b200 import synth
from binder_b200._lib import BinderError, lib
from binder_b200.engine import Engine
from oracle_lib import Oracle
from test_gpu_forward import _zone, chain_batch, same
from test_gpu_parity import compare
from test_gpu_query_log import records
from test_gpu_relay import check, pinned
from test_relay import corpus

pytestmark = pytest.mark.gpu

REGION, DCS = 'foo.com', ['dc2', 'dc3']
UPS = [('127.0.0.1', 5302, 0), ('10.0.0.2', 53, 0), ('127.0.0.1', 5303, 1)]


def misses(orc, n, seed):
    """A config-5-shaped batch, the oracle's resolve of it, and its misses packed in miss order."""
    pkts = chain_batch(n, seed)
    data, off = synth.pack_batch(pkts)
    want = orc.resolve_batch(data, off, seed=seed)
    mq, moff = synth.pack_batch([pkts[i] for i in want[4]])
    return data, off, want, mq, moff


def answers(fwd, key, seed):
    """Upstream responses to a forward call's queries (some missing, duplicated or from the wrong port, plus noise)."""
    uq, uq_off, order, _, route = fwd
    msgs = [b''] * len(route)
    for k, j in enumerate(order):
        msgs[j] = bytes(uq[uq_off[k]:uq_off[k + 1]])
    return G.pack(G.responses(UPS, list(route), msgs, random.Random(seed), key))


class DeviceCalls(object):
    """A device-form relay on one stream and a device-form forward on another, enqueued and checked once per round."""

    def __init__(self, e, orc, tb):
        import torch
        self.torch, self.e = torch, e
        dev = torch.device('cuda:0')
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                      # noqa: E731
        z = lambda k, dt=torch.int32: torch.zeros(k, dtype=dt, device=dev)                   # noqa: E731
        q_data, q_off, up_data, up_off = packed = RG.pack_pairs(corpus(80, 1500))
        self.r_want = relay_oracle.relay_batch(*packed, nthreads=8)
        self.rn = len(q_off) - 1
        self.r_in = [t(np.concatenate([q_data, np.zeros(16, np.uint8)])), t(q_off.view(np.int32)),
                     t(np.concatenate([up_data, np.zeros(16, np.uint8)])), t(up_off.view(np.int32))]
        self.r_out = [z(len(self.r_want[0]) + 64, torch.uint8), z(self.rn + 1), z(self.rn, torch.int16), z(self.rn, torch.uint8),
                      z(4)]
        _, _, _, mq, moff = misses(orc, 3000, 77)
        self.m, self.key = len(moff) - 1, 0xFEED5
        self.f_want = O.forward_batch(tb, mq, moff, self.key)
        self.f_in = [t(np.concatenate([mq, np.zeros(16, np.uint8)])), t(moff.view(np.int32)),
                     t(np.arange(self.m, dtype=np.int32)), t(np.array([0, self.m, 0, 0], np.int32))]
        self.cap = len(mq) + 64
        self.f_out = [z(self.cap, torch.uint8), z(self.m + 1), z(self.m), z(19), z(self.m, torch.uint8), z(self.cap, torch.uint8),
                      z(self.m + 1), z(8)]
        self.streams = (torch.cuda.Stream(), torch.cuda.Stream())
        torch.cuda.synchronize()

    def enqueue(self):
        ptrs = lambda xs: [x.data_ptr() for x in xs]                                          # noqa: E731
        s_r, s_f = self.streams
        with self.torch.cuda.stream(s_r):
            for x in self.r_out:
                x.zero_()
        q, qo, u, uo = ptrs(self.r_in)
        out, off, ln, st, tot = ptrs(self.r_out)
        self.e.relay_device(q, qo, u, uo, self.rn, out, len(self.r_want[0]), off, ln, st, tot, stream=s_r.cuda_stream)
        self.r_epoch = lib().bb_engine_launch_epoch(self.e._h)
        with self.torch.cuda.stream(s_f):
            for x in self.f_out:
                x.zero_()
        pk, po, mi, rt = ptrs(self.f_in)
        uq, uqo, order, goff, route, fq, fqo, ftot = ptrs(self.f_out)
        self.e.forward_device(pk, po, mi, rt, self.m, self.key, uq, self.cap, uqo, order, goff, route, fq, self.cap, fqo, ftot,
                              stream=s_f.cuda_stream)
        self.f_epoch = lib().bb_engine_launch_epoch(self.e._h)

    def check(self):
        self.torch.cuda.synchronize()
        h = [x.cpu().numpy() for x in self.r_out]
        tot = h[4].view(np.uint32)
        assert tot[0] == len(self.r_want[0]) and tot[2] != self.r_epoch and tot[3] == self.r_epoch
        check((h[0][:tot[0]], h[1].view(np.uint32), h[2].view(np.uint16), h[3]), self.r_want, True)
        h = [x.cpu().numpy() for x in self.f_out]
        ftot, m = h[7].view(np.uint32), self.m
        assert ftot[1] == m and ftot[2] != self.f_epoch and ftot[3] == self.f_epoch and ftot[0] == self.f_want[1][m]
        same((h[0][:ftot[0]], h[1].view(np.uint32), h[2].view(np.uint32), h[3].view(np.uint32), h[4]), self.f_want)


def relay_pinned(e, mq, moff, up, up_off, want):
    n = len(moff) - 1
    bufs = [pinned(len(want[0]) + 64, np.uint8), pinned(n + 1, np.uint32), pinned(n, np.uint16), pinned(n, np.uint8)]
    try:
        check(e.relay_batch(mq, moff, up, up_off, out=tuple(b for b, _ in bufs)), want, True)
    finally:
        for _, p in bufs:
            lib().bb_host_free(p)


def log_pageable(e, rs):
    """The query log of result set rs, with summaries, against the restatement."""
    assert records(e.log_batch(*rs, summary=True)) == L.log_set(*rs, 'foo.com')


def log_pinned(e, rs):
    """The query log of result set rs into pinned buffers, without and with a summary, against the restatement."""
    want = L.log_set(*rs, 'foo.com')
    n, total = len(rs[3]), sum(len(h) + len(b) for h, b, _ in want)
    for summary in (False, True):
        bufs = [pinned(total + 64, np.uint8), pinned(n + 1, np.uint32), pinned(n, np.uint32), pinned(n, np.uint16),
                pinned(n, np.uint32)]
        try:
            arrs = [b for b, _ in bufs]
            if not summary:
                arrs[4] = None
            res = e.log_batch(*rs, summary=summary, buffers=tuple(arrs))
            assert records(res if summary else res + (np.array([w[2] for w in want], np.uint32),)) == want
        finally:
            for _, p in bufs:
                lib().bb_host_free(p)


def test_gpu_host_staging_shared_across_calls():
    orc = Oracle('foo.com', 'dc1', True, snapshot=_zone('dc1', 200))
    orc.set_recursion_filter(REGION, DCS, True)
    tb = O.Table(REGION, DCS, UPS)
    e = Engine('foo.com', 'dc1', recursion=True, snapshot=_zone('dc1', 200), max_batch=1 << 16, ordered=True)
    e.set_recursion_filter(REGION, DCS, True)
    e.set_recursion_upstreams(UPS)
    dev = DeviceCalls(e, orc, tb)
    for r, n in enumerate((300, 60000, 40, 45000)):
        dev.enqueue()
        data, off, want, mq, moff = misses(orc, n, 10 + r)
        res = e.resolve_batch(data, off, seed=10 + r)
        compare(res, want, data, off, True)
        log_pageable(e, res[:4])
        key = 0xC0FFEE12345 * (r + 1)
        fwd = O.forward_batch(tb, mq, moff, key)
        same(e.forward_batch(mq, moff, key), fwd)
        args = answers(fwd, key, r) + (mq, moff, fwd[4], key)
        up, up_off = O.match_upstreams(tb, *args)
        same(e.match_upstreams(*args), (up, up_off))
        relayed = relay_oracle.relay_batch(mq, moff, up, up_off, nthreads=8)
        rel = e.relay_batch(mq, moff, up, up_off)
        check(rel, relayed, True)
        relay_pinned(e, mq, moff, up, up_off, relayed)
        log_pinned(e, rel)
        dev.check()
    # one byte short of the replies: BB_ERR_CAPACITY, then the exact capacity on the same engine
    m = len(moff) - 1
    total = len(relayed[0])
    for cap in (total - 1, total):
        out = (np.zeros(cap, np.uint8), np.zeros(m + 1, np.uint32), np.zeros(m, np.uint16), np.zeros(m, np.uint8))
        if cap < total:
            with pytest.raises(BinderError) as ei:
                e.relay_batch(mq, moff, up, up_off, out=out)
            assert ei.value.code == -5
        else:
            check(e.relay_batch(mq, moff, up, up_off, out=out), relayed, True)
    e.close()
