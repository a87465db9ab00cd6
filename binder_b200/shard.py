"""Multi-GPU face of the engine: one process per GPU, zone sharded by key hash, queries routed
to their owner with one exchange over NVLink peer memory (include/binder_b200.h, bb_shard_*).

torch.distributed is plumbing only: it carries the opaque CUDA IPC handles between the
processes once, and provides the cross-rank barrier between "everyone has pushed" and "owners
resolve" (a 1-element all-reduce on the compute stream).
"""
import ctypes

import numpy as np

from . import _lib
from ._lib import check, lib
from .engine import Engine


def fmix32(h):
    h = h.astype(np.uint64)
    h ^= h >> np.uint64(16); h = (h * np.uint64(0x85EBCA6B)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(13); h = (h * np.uint64(0xC2B2AE35)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(16)
    return h


def canon_forward(key, dns_domain):
    """The form the table stores a forward key in (TableBuilder::canon, zone_build.cpp): the lower-cased fqdn minus
    '.' + dnsDomain, as DNS wire labels; b'' for the root domain itself; None for a name no query can spell."""
    if isinstance(key, str):
        key = key.encode('latin-1')
    dom = dns_domain.encode('latin-1') if isinstance(dns_domain, str) else dns_domain
    if key == dom:
        return b''
    if len(key) <= len(dom) + 1 or key[-len(dom) - 1:] != b'.' + dom:
        return None
    out = bytearray()
    for lab in key[:-len(dom) - 1].split(b'.'):
        if not 1 <= len(lab) <= 63:
            return None
        out.append(len(lab))
        out += lab
    return bytes(out)


def _mulfold(x, k):
    p = x * np.uint64(k)
    return (p ^ (p >> np.uint64(32))) & np.uint64(0xFFFFFFFF)


def hash_keys(keys, ns=0, dns_domain=None):
    """bb::hash_key (zone_image.h) for a list of equal-length byte keys, vectorised.  Forward keys (ns 0) are given
    as lower-cased fqdns together with dns_domain and hashed in their canonical form (all must be reachable)."""
    if ns == 0 and dns_domain is not None:
        keys = [canon_forward(k, dns_domain) for k in keys]
    arr = np.frombuffer(b''.join(keys), dtype=np.uint8).reshape(len(keys), -1)
    n, L = arr.shape
    pad = (-L) % 4
    if pad:
        arr = np.concatenate([arr, np.zeros((n, pad), np.uint8)], axis=1)
    words = arr.reshape(n, -1, 4).astype(np.uint64)
    w = words[:, :, 0] | words[:, :, 1] << np.uint64(8) | words[:, :, 2] << np.uint64(16) | words[:, :, 3] << np.uint64(24)
    h = np.full(n, 0x52455631 if ns else 0x42494E44, dtype=np.uint64)
    for i in range(w.shape[1]):
        h = _mulfold(h ^ w[:, i], 0x9E3779B1)
    return fmix32(h ^ np.uint64(L))


def owner_of(key_hash, nranks):
    """bb::owner_of (zone_image.h)."""
    h = (key_hash * np.uint64(0x9E3779B1) + np.uint64(0x7F4A7C15)) & np.uint64(0xFFFFFFFF)
    return ((fmix32(h) * np.uint64(nranks)) >> np.uint64(32)).astype(np.int64)


class ShardedEngine(object):
    """One rank of the sharded resolver.  `lanes` independent exchange contexts (each with its own
    double-buffered receive regions) let several steps be in flight on different streams."""

    def __init__(self, dns_domain, datacenter, snapshot, rank, world, device, max_batch, recursion=False,
                 ordered=False, bytes_per_query=64, dist=None, lanes=1, sync='flags', host_results=False):
        self.rank, self.world, self.sync, self.host_results = rank, world, sync, host_results
        self.engine = Engine(dns_domain, datacenter, recursion=recursion, device=device, max_batch=max_batch,
                             max_batch_bytes=max_batch * bytes_per_query, ordered=ordered)
        self.zone_stat = self.engine.load_snapshot(snapshot, world, rank)
        self.dist = dist
        self._flag = None
        self._lanes = []
        self._fetch_bufs = {}
        for _ in range(lanes):
            err = ctypes.c_int(0)
            h = lib().bb_shard_create(self.engine._h, world, rank, max_batch, bytes_per_query, ctypes.byref(err))
            if not h:
                raise _lib.BinderError(err.value)
            self._lanes.append(h)
            if host_results:            # results land in the shard's pinned host mirrors (zero-copy)
                check(lib().bb_shard_host_results(h, 1))
        self._h = self._lanes[0]
        self.cap_q = lib().bb_shard_region_capacity(self._h)
        self._xch = []
        if sync == 'nccl_a2a':
            # the collective baseline: per lane a local send buffer and a receive buffer (torch tensors), exchanged with
            # grouped ncclSend/ncclRecv (torch.distributed.batch_isend_irecv) instead of peer stores
            import torch
            lay = (ctypes.c_uint64 * 5)()
            lib().bb_shard_region_layout(self._h, lay)
            self._lay = [int(x) for x in lay]
            nb = int(lib().bb_shard_exchange_bytes(self._h))
            for h in self._lanes:
                snd = torch.zeros(nb, dtype=torch.uint8, device='cuda')
                rcv = torch.zeros(nb, dtype=torch.uint8, device='cuda')
                check(lib().bb_shard_use_exchange_buffers(h, snd.data_ptr(), rcv.data_ptr()))
                self._xch.append((snd, rcv, torch.empty((world, 4), dtype=torch.int32).pin_memory(), torch.empty((world, 4), dtype=torch.int32).pin_memory()))
        if world > 1 and sync != 'nccl_a2a':
            hs = lib().bb_shard_ipc_handle_size()
            for h in self._lanes:
                mine = (ctypes.c_uint8 * hs)()
                check(lib().bb_shard_get_ipc_handle(h, mine))
                gathered = [None] * world
                dist.all_gather_object(gathered, bytes(mine))
                check(lib().bb_shard_open_peers(h, b''.join(gathered)))
            dist.barrier()

    def set_host_results(self, on):
        """Switch every lane between device result buffers (+ fetch copies) and pinned host mirrors
        the resolve kernel writes directly (bb_shard_host_results).  Synchronises the device."""
        for h in self._lanes:
            check(lib().bb_shard_host_results(h, 1 if on else 0))
        self.host_results = bool(on)

    def route_push(self, d_pkts, d_off, n, qidx_base, stream, lane=0, tcp=False):
        """bb_shard_route_push_ex.  tcp: the batch arrived over TCP; its owners answer it without the UDP size limit."""
        check(lib().bb_shard_route_push_ex(self._lanes[lane], d_pkts, d_off, n, qidx_base, 1 if tcp else 0, stream))

    def barrier(self):
        """sync='nccl': cross-rank barrier in stream order (1-element all-reduce)."""
        if self.world > 1:
            import torch
            if self._flag is None:
                self._flag = torch.zeros(1, dtype=torch.int32, device='cuda')
            self.dist.all_reduce(self._flag)

    def resolve(self, seed, stream, lane=0):
        wait = 1 if (self.sync == 'flags' and self.world > 1) else 0
        check(lib().bb_shard_resolve(self._lanes[lane], seed, wait, stream))

    def exchange(self, lane=0):
        """sync='nccl_a2a': move every send region to its destination's receive region with ONE grouped exchange of
        ncclSend/ncclRecv (headers first — their counts size the rest, which costs a host round trip per step: that is
        what a collective on data-dependent sizes needs).  Runs on the current torch stream."""
        import torch
        dist = self.dist
        W, R = self.world, self.rank
        snd, rcv, h_s, h_r = self._xch[lane]
        reg, cap, o_off, o_qi, o_by = self._lay
        st = int(lib().bb_shard_exchange_set(self._lanes[lane]))
        sreg = lambda d: snd[(st * W + d) * reg:(st * W + d + 1) * reg]
        rreg = lambda s_: rcv[(st * W + s_) * reg:(st * W + s_ + 1) * reg]
        hs = torch.stack([sreg(d)[:16].view(torch.int32) for d in range(W)])         # what this rank sends to each rank
        hr = torch.empty_like(hs)
        if W > 1:
            dist.all_to_all_single(hr, hs)
        else:
            hr.copy_(hs)
        h_s.copy_(hs, non_blocking=True); h_r.copy_(hr, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        ops = []
        for p in range(W):
            cs, bs = int(h_s[p, 0]), int(h_s[p, 1])
            cr, br = int(h_r[p, 0]), int(h_r[p, 1])
            rreg(p)[:16].view(torch.int32).copy_(hr[p])
            if p == R:                               # own region: device copies
                for o, n in ((o_off, 4 * (cs + 1)), (o_qi, 4 * cs), (o_by, (bs + 15) // 16 * 16)):
                    if n:
                        rreg(p)[o:o + n].copy_(sreg(p)[o:o + n])
                continue
            for o, n in ((o_off, 4 * (cs + 1)), (o_qi, 4 * cs), (o_by, (bs + 15) // 16 * 16)):
                if n:
                    ops.append(dist.P2POp(dist.isend, sreg(p)[o:o + n], p))
            for o, n in ((o_off, 4 * (cr + 1)), (o_qi, 4 * cr), (o_by, (br + 15) // 16 * 16)):
                if n:
                    ops.append(dist.P2POp(dist.irecv, rreg(p)[o:o + n], p))
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()

    def step(self, d_pkts, d_off, n, qidx_base, seed, stream, lane=0, tcp=False):
        self.route_push(d_pkts, d_off, n, qidx_base, stream, lane, tcp)
        if self.sync == 'nccl':
            self.barrier()
        elif self.sync == 'nccl_a2a':
            self.exchange(lane)
        self.resolve(seed, stream, lane)

    def _bufs(self, lane, src):
        """Pinned host buffers for one region's results, allocated once (a fresh pageable array per
        call costs page faults on every copy)."""
        key = (lane, src)
        if key not in self._fetch_bufs:
            import torch
            cap = self.cap_q
            pin = torch.cuda.is_available()
            mk = lambda n, dt: torch.empty(n, dtype=dt, pin_memory=pin).numpy()
            self._fetch_bufs[key] = dict(out=mk(cap * 256, torch.uint8), out_off=mk(cap + 1, torch.int32).view(np.uint32),
                                         out_len=mk(cap, torch.int16).view(np.uint16), status=mk(cap, torch.uint8),
                                         qidx=mk(cap, torch.int32).view(np.uint32), miss=mk(cap, torch.int32).view(np.uint32))
        return self._fetch_bufs[key]

    def fetch(self, src, lane=0, copy=True):
        """Region `src` -> dict(out, out_off, out_len, status, qidx, miss) as numpy arrays (views of
        reused pinned buffers unless copy=True).  With host_results the arrays are views of the
        shard's own mirrors: the caller must have waited for the resolve's stream."""
        if self.host_results:
            return self._results(src, lane, copy)
        b = self._bufs(lane, src)
        n, nm, tot = ctypes.c_uint32(0), ctypes.c_uint32(0), ctypes.c_uint32(0)
        check(lib().bb_shard_fetch(self._lanes[lane], src, b['out'].ctypes.data, b['out'].size, b['out_off'].ctypes.data,
                                   b['out_len'].ctypes.data, b['status'].ctypes.data, b['qidx'].ctypes.data,
                                   b['miss'].ctypes.data, ctypes.byref(n), ctypes.byref(nm), ctypes.byref(tot)))
        n = n.value
        f = (lambda a: a.copy()) if copy else (lambda a: a)
        return dict(n=n, out=f(b['out'][:tot.value]), out_off=f(b['out_off'][:n + 1]), out_len=f(b['out_len'][:n]),
                    status=f(b['status'][:n]), qidx=f(b['qidx'][:n]), miss=f(b['miss'][:nm.value]))

    def _results(self, src, lane, copy):
        P = ctypes.POINTER
        out, status = P(ctypes.c_uint8)(), P(ctypes.c_uint8)()
        out_off, qidx, miss = P(ctypes.c_uint32)(), P(ctypes.c_uint32)(), P(ctypes.c_uint32)()
        out_len = P(ctypes.c_uint16)()
        n, nm, tot = ctypes.c_uint32(0), ctypes.c_uint32(0), ctypes.c_uint32(0)
        check(lib().bb_shard_results(self._lanes[lane], src, ctypes.byref(out), ctypes.byref(out_off), ctypes.byref(out_len),
                                     ctypes.byref(status), ctypes.byref(qidx), ctypes.byref(miss),
                                     ctypes.byref(n), ctypes.byref(nm), ctypes.byref(tot)))
        n = n.value

        def view(ptr, count):
            if count == 0:
                return np.zeros(0, dtype=np.dtype(ptr._type_))
            a = np.ctypeslib.as_array(ptr, shape=(count,))
            return a.copy() if copy else a
        return dict(n=n, out=view(out, tot.value), out_off=view(out_off, n + 1), out_len=view(out_len, n),
                    status=view(status, n), qidx=view(qidx, n), miss=view(miss, nm.value))

    def totals(self, src, lane=0):
        """(queries, misses, response bytes) of region `src` after a finished resolve (host_results only)."""
        r = self._results(src, lane, False)
        return r['n'], len(r['miss']), len(r['out'])

    def close(self):
        for h in self._lanes:
            lib().bb_shard_destroy(h)
        self._lanes = []
        self.engine.close()
