"""DNS-over-TCP batches (BB_BATCH_TCP) on the sharded path and through the device-resident resolve API, against the oracle.

Sharded (one GPU, the in-process cluster of tests/test_gpu_shard_paths.py): bb_shard_route_push_ex marks every query of a
push as TCP, the flag travels in word 3 of each region header of the step, and the multi-region resolve_kernel sizes
each region under its own source's limit.  Every region of every step is checked with check_region against the oracle
run with tcp=True for a TCP source and tcp=False for a UDP one.  The peer-store arm (W = 2 processes on cuda:0) shows the
flag is visible once the epoch flag is.

Device-resident: bb_resolve_batch_device_ex with BB_BATCH_TCP on several streams, next to UDP launches of the same batch,
flags = 0 against bb_resolve_batch_device, and its argument errors.
"""
import ctypes
import os
import traceback

import numpy as np
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth
from binder_b200._lib import BinderError, check, lib
from test_gpu_kernel_paths import DevBatch, gen
from test_gpu_parity import MODES
from test_gpu_shard_paths import Cluster, check_region, fuzz_zones, route, svc_zone  # noqa: F401  (fixtures)
from test_tcp import big_zone, big_zone_batch

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAPACITY, BATCH_TCP = -1, -5, 1
UDP_MAX = 1232                   # the largest response a UDP query can get (EDNS payload size, capped)
SRV_CUT = 65516                  # the 1,300-child service's 2,600 SRV RRs, truncated over TCP


# ---- expected results ----------------------------------------------------------------------------------------------
class TBatch(object):
    """One rank's ingress batch of one step, pushed with `flags` (BB_BATCH_TCP or 0, unknown bits allowed): the oracle's
    results for its own mode at (seed, qidx_base), and the router's owner of every packet."""

    def __init__(self, pkts, rank, world, qidx_base, seed, orc, route, dom, recursion, flags, data=None, off=None):
        if data is None:
            data, off = synth.pack_batch(pkts)
        self.flags, self.tcp = flags, bool(flags & BATCH_TCP)
        self.data, self.off, self.n, self.base = data, off, len(off) - 1, qidx_base
        self.res = orc.resolve_batch(data, off, seed=seed, qidx_base=qidx_base, nthreads=os.cpu_count(), tcp=self.tcp)
        self.owner = route(dom, recursion, data, off, world, rank)


class TcpCluster(Cluster):
    """Cluster whose pushes carry each batch's flags: ShardedEngine.route_push(tcp=...) for flags 0 / BB_BATCH_TCP, the
    C call for any other bits."""

    def push(self, batches, lane, st):
        keep = []
        for r, se in enumerate(self.ranks):
            b = batches[r]
            d_pk, d_off = self.upload(b, st.device)
            keep += [d_pk, d_off]
            if b.flags in (0, BATCH_TCP):
                se.route_push(d_pk.data_ptr(), d_off.data_ptr(), b.n, b.base, st.cuda_stream, lane, tcp=b.tcp)
            else:
                check(lib().bb_shard_route_push_ex(se._lanes[lane], d_pk.data_ptr(), d_off.data_ptr(), b.n, b.base, b.flags,
                                                   st.cuda_stream))
        return keep

    def finish(self, seed, lane, exact, st):
        self.exchange(lane, exact)
        for se in self.ranks:
            se.resolve(seed, st.cuda_stream, lane)

    def enqueue(self, batches, seed, lane=0, exact=True, stream=None):
        import torch
        st = stream if stream is not None else torch.cuda.current_stream()
        with torch.cuda.stream(st):
            keep = self.push(batches, lane, st)
            self.finish(seed, lane, exact, st)
        return keep

    def step(self, batches, seed, lane=0, exact=True):
        """One step, with the headers every push published checked before anything reads them (check_headers)."""
        import torch
        st = torch.cuda.current_stream()
        keep = self.push(batches, lane, st)
        torch.cuda.synchronize()
        self.check_headers(batches, lane)
        self.finish(seed, lane, exact, st)
        torch.cuda.synchronize()
        del keep

    def headers(self, lane=0):
        """[src][owner][4] the 16-byte headers the last push of every rank published (its send regions, current set)."""
        import torch
        W = self.world
        reg = self.lay[0]
        out = np.zeros((W, W, 4), dtype=np.int64)
        for s, se in enumerate(self.ranks):
            st = int(lib().bb_shard_exchange_set(se._lanes[lane]))
            snd = se._xch[lane][0]
            for d in range(W):
                out[s, d] = snd[(st * W + d) * reg:(st * W + d) * reg + 16].view(torch.int32).cpu().numpy().view(np.uint32)
        return out

    def check_headers(self, batches, lane=0):
        """Word 0 = the queries the router sends that owner, word 1 = their packet bytes (both what the exchange sizes its
        copies from), word 3 = 2 for a TCP push and 0 for a UDP one, in every region of the step, empty ones included."""
        hdr = self.headers(lane)
        for s, b in enumerate(batches):
            lens = np.diff(b.off.astype(np.int64))
            lens[lens > 65535] = 0                     # such packets stay home, dropped: no bytes pushed
            for d in range(self.world):
                own = b.owner == d
                want = (int(own.sum()), int(lens[own].sum()), 2 if b.tcp else 0)
                assert (hdr[s, d, 0], hdr[s, d, 1], hdr[s, d, 3]) == want, (s, d, hdr[s, d], want)



@pytest.fixture(scope='module')
def big():
    """foo.com with a 200-child service and a 1,300-child service (rr_hosts with two ports each)."""
    snap = big_zone()
    return snap, H.make_impl('oracle', 'foo.com', snap)


def big_pkts(k, n=350):
    pk = big_zone_batch()
    s = (97 * k) % len(pk)
    return (pk[s:] + pk[:s])[:n]


def fuzz_make(world, info, orc, route, flags_of, size=900):
    dom = info['dns_domain']

    def make(k, seed):
        return [TBatch(fuzzgen.gen_queries(1000 * k + 10 * world + r, info, n=size) + fuzzgen.malformed_packets(), r, world,
                       (r * 100003 + k * 7) & 0xFFFFFFFF, seed, orc, route, dom, True, flags_of(k, r)) for r in range(world)]
    return make


def big_make(world, orc, route, flags_of, size=350):
    def make(k, seed):
        return [TBatch(big_pkts(3 * k + r, size), r, world, r * 4000 + k, seed, orc, route, 'foo.com', False, flags_of(k, r))
                for r in range(world)]
    return make


def run(cl, make, steps, seed0):
    """`steps` steps (headers checked by TcpCluster.step), every region against the oracle; step k exchanges exactly on
    k % 4 in (0, 3) and whole regions otherwise."""
    for k in range(steps):
        seed = seed0 + 7919 * k
        batches = make(k, seed)
        cl.step(batches, seed, exact=k % 4 in (0, 3))
        cl.check(batches, what=('step', k, [b.flags for b in batches]))
    return batches


def results_of(world, ordered):
    """Host mirrors on the odd ranks (device fetch on the even ones); W = 1: mirrors in ordered packing only."""
    return tuple(range(1, world, 2)) if world > 1 else ((0,) if ordered else ())


# ---- zones and sizes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('world', [1, 2, 3, 5, 8])
def test_fuzz_zone_tcp_shards_match_oracle(fuzz_zones, route, world, ordered):
    """Every rank pushes TCP: fuzz zones, 3 steps, exact and whole-region exchange, device fetch and host mirrors."""
    snap, info, orc = fuzz_zones(world)
    cl = TcpCluster(info['dns_domain'], snap, world, 8192, ordered=ordered, host=results_of(world, ordered))
    try:
        run(cl, fuzz_make(world, info, orc, route, lambda k, r: BATCH_TCP), 4, 0x7C9 + world)
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('world', [1, 2, 3, 5, 8])
def test_large_answers_over_tcp_shards(big, route, world, ordered):
    """The 200- and 1,300-child services over TCP: SRV and A answers whole (far beyond 1,232 bytes), the 2,600 SRV RRs
    cut at 65,516 bytes with TC set; every region byte-exact."""
    snap, orc = big
    cl = TcpCluster('foo.com', snap, world, 16384, recursion=False, ordered=ordered, host=results_of(world, ordered))
    try:
        batches = run(cl, big_make(world, orc, route, lambda k, r: BATCH_TCP), 3, 0x51E + world)
        lens = np.concatenate([b.res[2] for b in batches]).astype(np.int64)
        assert lens.max() == SRV_CUT and (lens > UDP_MAX).sum() > 50
        for b in batches:
            for i in np.nonzero(b.res[2] == SRV_CUT)[0]:
                assert b.res[0][b.res[1][i] + 2] & 0x02                # TC
    finally:
        cl.close()


# ---- TCP and UDP sources in one step, on one region set, on two lanes -----------------------------------------------
@pytest.mark.parametrize('ordered', MODES)
def test_mixed_step_each_region_under_its_source_limit(big, route, ordered):
    """Even ranks push TCP and odd ranks UDP in the same step (then the other way round): each owner answers each region
    under its own source's limit."""
    snap, orc = big
    world = 4
    cl = TcpCluster('foo.com', snap, world, 16384, recursion=False, ordered=ordered, host=(2, 3))
    try:
        batches = run(cl, big_make(world, orc, route, lambda k, r: BATCH_TCP if (r + k) % 2 == 0 else 0), 4, 0xA11)
        for b in batches:
            assert (b.res[2].max() > UDP_MAX) == b.tcp
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
def test_mixed_step_fuzz_zone(fuzz_zones, route, ordered):
    world = 5
    snap, info, orc = fuzz_zones(world)
    cl = TcpCluster(info['dns_domain'], snap, world, 8192, ordered=ordered, host=(1, 4))
    try:
        run(cl, fuzz_make(world, info, orc, route, lambda k, r: BATCH_TCP if (r + k) % 2 == 0 else 0), 4, 0xF22)
    finally:
        cl.close()


@pytest.mark.parametrize('host', [pytest.param(False, id='device'), pytest.param(True, id='host')])
@pytest.mark.parametrize('ordered', MODES)
def test_alternating_lane_carries_no_flag_over(big, route, ordered, host):
    """One lane runs TCP, UDP, UDP, TCP, UDP, TCP: region set 0 (even steps) sees T, U, U and set 1 sees U, T, T, so each
    set is reused after a step of the other kind; no flag carries over."""
    snap, orc = big
    world = 3
    seq = [1, 0, 0, 1, 0, 1]
    cl = TcpCluster('foo.com', snap, world, 16384, recursion=False, ordered=ordered, host=range(world) if host else ())
    try:
        run(cl, big_make(world, orc, route, lambda k, r: BATCH_TCP if seq[k] else 0), len(seq), 0xA17)
    finally:
        cl.close()


def test_unknown_flag_bits_are_ignored(big, route):
    """flags with bits other than BB_BATCH_TCP: 0x101 pushes TCP, 0x100 and 0xFFFFFFFE push UDP."""
    snap, orc = big
    world = 2
    seq = [0x101, 0x100, 0xFFFFFFFE, 0xFFFFFFFF]
    cl = TcpCluster('foo.com', snap, world, 16384, recursion=False)
    try:
        run(cl, big_make(world, orc, route, lambda k, r: seq[k]), len(seq), 0xB17)
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
def test_two_lanes_tcp_and_udp_on_two_streams(big, route, ordered):
    """Lane 0 pushes TCP and lane 1 UDP (swapped every round), on two streams, both enqueued before any
    synchronisation; each lane holds its own step's answers under its own limit."""
    import torch
    snap, orc = big
    world = 3
    cl = TcpCluster('foo.com', snap, world, 16384, recursion=False, ordered=ordered, host=(1,), lanes=2)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    try:
        for rnd in range(3):
            tcp_lane = rnd % 2
            work = [big_make(world, orc, route, lambda k, r, lane=lane: BATCH_TCP if lane == tcp_lane else 0)(2 * rnd + lane, 40 + lane)
                    for lane in range(2)]
            keep = [cl.enqueue(work[lane], 40 + lane, lane=lane, exact=False, stream=streams[lane]) for lane in range(2)]
            torch.cuda.synchronize()
            del keep
            for lane in range(2):
                cl.check(work[lane], lane=lane, what=('lanes', rnd, lane))
                assert (max(int(b.res[2].max()) for b in work[lane]) > UDP_MAX) == (lane == tcp_lane)
    finally:
        cl.close()


# ---- capacity and edges ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('host', [pytest.param(False, id='device'), pytest.param(True, id='host')])
def test_tcp_answers_over_out_cap_fail_only_their_step(big, route, host):
    """out_cap = cap_q x 256 bytes: four 1,300-child SRV answers over TCP (4 x 65,516 bytes) do not fit a region of a
    512-query shard.  That region is BB_ERR_CAPACITY for the step; the other regions are answered, the same queries over
    UDP fit, and the next TCP step of small answers is answered — through bb_shard_fetch and bb_shard_results alike."""
    snap, orc = big
    world, B = 2, 512
    cl = TcpCluster('foo.com', snap, world, B, recursion=False, host=range(world) if host else ())
    mk = lambda pk, r, seed, flags: TBatch(pk, r, world, r * B, seed, orc, route, 'foo.com', False, flags)
    huge = [synth.make_query('_http._tcp.huge.foo.com', 'SRV', i) for i in range(4)]
    small = lambda k: [synth.make_query(['hosta.foo.com', 'lb%03d.big.foo.com' % k, 'nope.foo.com'][i % 3], 'A', i) for i in range(60)]
    try:
        for k, flags in enumerate([BATCH_TCP, BATCH_TCP, 0, BATCH_TCP]):
            seed = 70 + k
            batches = [mk(huge + small(k) if k in (1, 2) else small(k), 0, seed, flags), mk(small(k + 9), 1, seed, BATCH_TCP)]
            cl.step(batches, seed, exact=k != 2)
            if k != 1:
                cl.check(batches, what=('tcp capacity', k))
                continue
            hot = int(batches[0].owner[0])
            owned = batches[0].res[2][batches[0].owner == hot].astype(np.int64).sum()
            assert owned > B * 256, owned
            with pytest.raises(BinderError) as ei:
                cl.ranks[hot].fetch(0)
            assert ei.value.code == ERR_CAPACITY
            check_region(cl.ranks[1 - hot].fetch(0), batches[0], 1 - hot, False, 'other owner')
            for d, se in enumerate(cl.ranks):
                check_region(se.fetch(1), batches[1], d, False, ('other sender', d))
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
def test_empty_and_tiny_tcp_pushes(fuzz_zones, route, ordered):
    """n = 0 TCP pushes on every rank, n = 1 at W = 8 (seven empty regions per source, each still carrying the flag), a
    silent rank among TCP senders, and a UDP step between them."""
    world = 8
    snap, info, orc = fuzz_zones(world)
    dom = info['dns_domain']
    cl = TcpCluster(dom, snap, world, 8192, ordered=ordered, host=(0, 5))
    mk = lambda pk, r, seed, flags: TBatch(pk, r, world, r * 1000, seed, orc, route, dom, True, flags)
    try:
        one = fuzzgen.gen_queries(6, info, n=64)[:world]
        full = fuzz_make(world, info, orc, route, lambda k, r: BATCH_TCP, size=600)
        for k, shape in enumerate(['empty', 'one', 'full', 'one_udp', 'silent', 'one']):
            seed = 131 + k
            flags = 0 if shape == 'one_udp' else BATCH_TCP
            if shape == 'empty':
                batches = [mk([], r, seed, flags) for r in range(world)]
            elif shape in ('one', 'one_udp'):
                batches = [mk(one[r:r + 1], r, seed, flags) for r in range(world)]
            else:
                batches = full(k, seed)
                if shape == 'silent':
                    batches[3] = mk([], 3, seed, flags)
            cl.step(batches, seed, exact=k % 2 == 0)
            cl.check(batches, what=shape)
    finally:
        cl.close()


def test_route_push_ex_argument_errors(big, route):
    """bb_shard_route_push_ex: NULL shard, n > max_batch, a misaligned d_pkts, and a shard without peers or exchange
    buffers are BB_ERR_ARG whatever the flags; nothing is launched, and the next step is exact."""
    import torch
    snap, orc = big
    world, B = 2, 16384
    cl = TcpCluster('foo.com', snap, world, B, recursion=False)
    L = lib()
    try:
        mk = lambda k, r: TBatch(big_pkts(k, 300), r, world, r * B, 9, orc, route, 'foo.com', False, BATCH_TCP)
        batches = [mk(0, 0), mk(1, 1)]
        d_pk, d_off = Cluster.upload(batches[0], torch.device('cuda:0'))
        stream = torch.cuda.current_stream().cuda_stream
        h = cl.ranks[0]._h
        for flags in (0, BATCH_TCP, 0xFFFFFFFF):
            assert L.bb_shard_route_push_ex(None, d_pk.data_ptr(), d_off.data_ptr(), batches[0].n, 0, flags, stream) == ERR_ARG
            assert L.bb_shard_route_push_ex(h, d_pk.data_ptr(), d_off.data_ptr(), B + 1, 0, flags, stream) == ERR_ARG
            for k in (1, 4, 8):
                assert L.bb_shard_route_push_ex(h, d_pk.data_ptr() + k, d_off.data_ptr(), batches[0].n, 0, flags, stream) == ERR_ARG
        err = ctypes.c_int(0)
        lone = L.bb_shard_create(cl.ranks[0].engine._h, 2, 0, 512, 64, ctypes.byref(err))       # peers never opened
        assert lone and err.value == 0
        try:
            assert L.bb_shard_route_push_ex(lone, d_pk.data_ptr(), d_off.data_ptr(), 10, 0, BATCH_TCP, stream) == ERR_ARG
        finally:
            L.bb_shard_destroy(lone)
        cl.step(batches, 9)
        cl.check(batches, what='after refusals')
    finally:
        cl.close()


def test_sharded_engine_step_tcp(big, route):
    """ShardedEngine.step(..., tcp=...) on one rank (collective arm, nothing to exchange with): TCP, UDP, TCP."""
    import torch
    snap, orc = big
    cl = TcpCluster('foo.com', snap, 1, 16384, recursion=False)
    se = cl.ranks[0]
    try:
        for k, tcp in enumerate([True, False, True]):
            b = TBatch(big_pkts(k), 0, 1, 77 * k, 5 + k, orc, route, 'foo.com', False, BATCH_TCP if tcp else 0)
            d_pk, d_off = Cluster.upload(b, torch.device('cuda:0'))
            se.step(d_pk.data_ptr(), d_off.data_ptr(), b.n, b.base, 5 + k, torch.cuda.current_stream().cuda_stream, tcp=tcp)
            torch.cuda.synchronize()
            assert check_region(se.fetch(0), b, 0, False, ('step', k)) == b.n
            assert (b.res[2].max() > UDP_MAX) == tcp
    finally:
        cl.close()


# ---- peer stores across processes on one GPU ------------------------------------------------------------------------
def _tcp_peer_worker(rank, world, port, ordered, snap, work, q):
    """One rank in its own process on cuda:0 (sync='flags'): pushes with each batch's TCP flag into the other process's
    receive buffer through CUDA IPC, publishes the epoch flags, resolves after the wait kernel has seen them."""
    from binder_b200.shard import ShardedEngine
    se = None
    try:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(0)
        dist.init_process_group('gloo', rank=rank, world_size=world)
        se = ShardedEngine('foo.com', '', snap, rank, world, 0, 16384, recursion=False, ordered=ordered, dist=dist, sync='flags')
        st = torch.cuda.current_stream()
        for k, (seed, batches) in enumerate(work):
            b = batches[rank]
            d_pk, d_off = Cluster.upload(b, torch.device('cuda:0'))
            se.route_push(d_pk.data_ptr(), d_off.data_ptr(), b.n, b.base, st.cuda_stream, tcp=b.tcp)
            torch.cuda.synchronize()
            dist.barrier()
            se.resolve(seed, st.cuda_stream)
            torch.cuda.synchronize()
            for src, sb in enumerate(batches):
                check_region(se.fetch(src), sb, rank, ordered, ('peer', k, src, rank))
            dist.barrier()
        q.put((rank, 'ok'))
    except BaseException:
        q.put((rank, traceback.format_exc()))
    finally:
        if se is not None:
            se.close()
        try:
            import torch.distributed as dist
            dist.destroy_process_group()
        except Exception:
            pass


@pytest.mark.parametrize('ordered', MODES)
def test_tcp_pushes_through_peer_stores(big, route, ordered):
    """W = 2 processes sharing cuda:0: steps where both ranks push TCP, one does, and none does."""
    import torch.multiprocessing as mp
    snap, orc = big
    world = 2
    flags = [(1, 1), (1, 0), (0, 1), (0, 0), (1, 1)]
    work = []
    for k, fl in enumerate(flags):
        seed = 4321 + k
        work.append((seed, big_make(world, orc, route, lambda kk, r, fl=fl: fl[r])(k, seed)))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 33000 + (os.getpid() + ordered) % 2000
    procs = [ctx.Process(target=_tcp_peer_worker, args=(r, world, port, ordered, snap, work, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=300) for _ in procs)
        for p in procs:
            p.join(60)
        assert res == {r: 'ok' for r in range(world)}, '\n'.join(str(v) for v in res.values())
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
            p.join(10)


# ---- device-resident: bb_resolve_batch_device_ex ---------------------------------------------------------------------
class TDevBatch(DevBatch):
    def launch_ex(self, eng, seed, flags, qidx_base=0, stream=0, out_cap=None, n=None, d_pkts=None, d_out=None):
        """-> (return code, bb_engine_launch_epoch() right after the call)"""
        rc = lib().bb_resolve_batch_device_ex(eng._h, self.d_pk.data_ptr() if d_pkts is None else d_pkts, self.d_off.data_ptr(),
                                              self.n if n is None else n, seed, qidx_base,
                                              self.d_out.data_ptr() if d_out is None else d_out,
                                              self.cap if out_cap is None else out_cap, self.d_oo.data_ptr(), self.d_ol.data_ptr(),
                                              self.d_st.data_ptr(), self.d_ms.data_ptr(), self.d_tot.data_ptr(), stream, flags)
        return rc, int(lib().bb_engine_launch_epoch(eng._h))


def padded(pkts):
    data, off = synth.pack_batch(pkts)
    return np.concatenate([data, np.zeros((-data.size) % 16, np.uint8)]), off


@pytest.fixture(scope='module')
def big_recursion():
    snap = big_zone()
    return snap, H.make_impl('oracle', 'foo.com', snap, recursion=True)


@pytest.mark.parametrize('profile', ['small', 'service'])
@pytest.mark.parametrize('ordered', MODES)
def test_device_tcp_launches_on_five_streams(svc_zone, big_recursion, ordered, profile):
    """Four torch streams and the default stream, three TCP launches each, enqueued before anything synchronises: service
    zones (configs 2-5) and the 200- / 1,300-child services; each exact against the oracle with tcp=True, with the totals
    contract (bytes, misses, no overflow marker, done marker = the launch's epoch)."""
    import torch
    z, zorc = svc_zone
    bsnap, borc = big_recursion
    engs = [H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered),
            H.make_impl('gpu', 'foo.com', bsnap, recursion=True, ordered=ordered)]
    WORK = ['config2', 'config3', 'config4', 'config5']
    try:
        for e in engs:
            e.set_kernel_profile(profile)
        streams = [torch.cuda.Stream() for _ in range(4)]
        ptrs = [s.cuda_stream for s in streams] + [0]
        sizes = [1, 129, 3000, 20000]
        jobs = []
        for k in range(3):
            for j in range(5):
                i = k * 5 + j
                if (i + k) % 2 == 1:
                    b = TDevBatch(*padded(big_pkts(i, 200 + 50 * k)), out_cap=4 << 20)
                    jobs.append((b, 1, borc, ptrs[j], i))
                else:
                    data, off = gen(z, sizes[i % 4], 700 + i, WORK[(i + k) % 4])
                    jobs.append((TDevBatch(data, off, out_cap=max(8192, sizes[i % 4] * 4000)), 0, zorc, ptrs[j], i))
        torch.cuda.synchronize()
        epochs = []
        for b, e, _, st, i in jobs:
            rc, ep = b.launch_ex(engs[e], 900 + i, BATCH_TCP, qidx_base=i << 20, stream=st)
            check(rc)
            epochs.append(ep)
        torch.cuda.synchronize()
        saw_big = 0
        for (b, _, orc, _, i), ep in zip(jobs, epochs):
            b.check(orc, 900 + i, ep, ordered, qidx_base=i << 20, tcp=True)
            saw_big += int(b.results()[2].max(initial=0)) > UDP_MAX
        assert saw_big >= 6
    finally:
        for e in engs:
            e.close()


@pytest.mark.parametrize('ordered', MODES)
def test_device_udp_and_tcp_of_one_batch_on_two_streams(big_recursion, ordered):
    """The same batch launched as UDP on one stream and as TCP on another, back to back, three rounds: each result matches
    the oracle for its own mode (the flag is per launch, never per engine or per stream)."""
    import torch
    snap, orc = big_recursion
    eng = H.make_impl('gpu', 'foo.com', snap, recursion=True, ordered=ordered)
    try:
        data, off = padded(big_zone_batch())
        sts = [torch.cuda.Stream(), torch.cuda.Stream()]
        for rnd in range(3):
            bs = [TDevBatch(data, off, out_cap=8 << 20) for _ in range(2)]
            eps = {}
            for mode in (0, 1) if rnd % 2 == 0 else (1, 0):           # mode = flags: 0 UDP, 1 TCP
                rc, eps[mode] = bs[mode].launch_ex(eng, 17 + rnd, mode, stream=sts[mode].cuda_stream)
                check(rc)
            torch.cuda.synchronize()
            for mode, ep in eps.items():
                bs[mode].check(orc, 17 + rnd, ep, ordered, tcp=bool(mode))
            assert int(bs[1].totals()[0]) > 5 * int(bs[0].totals()[0])
    finally:
        eng.close()


@pytest.mark.parametrize('ordered', MODES)
def test_device_ex_flags_zero_is_the_plain_call(svc_zone, ordered):
    """flags = 0 (and bits other than BB_BATCH_TCP) give the bytes, offsets, lengths, statuses, misses and totals of
    bb_resolve_batch_device."""
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=ordered)
    try:
        data, off = gen(z, 5000, 31, 'config3')
        ref = TDevBatch(data, off)
        rc, ep0 = ref.launch(eng, 8, qidx_base=99)
        check(rc)
        torch.cuda.synchronize()
        ref.check(orc, 8, ep0, ordered, qidx_base=99)
        want = ref.results()
        for flags in (0, 0x100, 0xFFFFFFFE):
            b = TDevBatch(data, off)
            rc, ep = b.launch_ex(eng, 8, flags, qidx_base=99)
            check(rc)
            torch.cuda.synchronize()
            got = b.results()
            if ordered:
                for a, w in zip(got, want):
                    assert np.array_equal(a, w), flags
            else:                                  # arrival packing: the same responses, placed wherever the claims fell
                b.check(orc, 8, ep, ordered, qidx_base=99)
                assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3])
            tot = b.totals()
            assert tot[0] == ref.totals()[0] and tot[1] == ref.totals()[1] and tot[3] == ep
    finally:
        eng.close()


def test_device_ex_argument_errors(svc_zone):
    """The BB_ERR_ARG cases of bb_resolve_batch_device, with either flag: misaligned d_pkts or d_out, n > max_batch, a
    17th distinct stream; the first 16 streams keep working."""
    import torch
    z, orc = svc_zone
    eng = H.make_impl('gpu', z.dns_domain, z.jsonl, recursion=True, ordered=True, max_batch=4096)
    try:
        b = TDevBatch(*gen(z, 300, 1, 'config4'))
        for flags in (0, BATCH_TCP):
            for k in (1, 4, 8):
                assert b.launch_ex(eng, 1, flags, d_pkts=b.d_pk.data_ptr() + k)[0] == ERR_ARG
                assert b.launch_ex(eng, 1, flags, d_out=b.d_out.data_ptr() + k)[0] == ERR_ARG
            assert b.launch_ex(eng, 1, flags, n=4097)[0] == ERR_ARG
        assert lib().bb_resolve_batch_device_ex(None, b.d_pk.data_ptr(), b.d_off.data_ptr(), b.n, 1, 0, b.d_out.data_ptr(), b.cap,
                                                b.d_oo.data_ptr(), b.d_ol.data_ptr(), b.d_st.data_ptr(), b.d_ms.data_ptr(),
                                                b.d_tot.data_ptr(), 0, BATCH_TCP) == ERR_ARG
        streams = [torch.cuda.Stream() for _ in range(17)]
        outs = [TDevBatch(b.data, b.off, out_cap=300 * 4000) for _ in range(16)]
        for i, (s, o) in enumerate(zip(streams, outs)):
            check(o.launch_ex(eng, 1, i % 2, stream=s.cuda_stream)[0])
        assert b.launch_ex(eng, 1, BATCH_TCP, stream=streams[16].cuda_stream)[0] == ERR_ARG
        torch.cuda.synchronize()
        eps = []
        for i, (s, o) in enumerate(zip(streams, outs)):
            rc, ep = o.launch_ex(eng, 10, (i + 1) % 2, stream=s.cuda_stream)
            check(rc)
            eps.append(ep)
        torch.cuda.synchronize()
        for i, (o, ep) in enumerate(zip(outs, eps)):
            o.check(orc, 10, ep, True, tcp=bool((i + 1) % 2))
    finally:
        eng.close()
