"""The sharded path — route_push_kernel and the multi-region (MULTI) resolve_kernel — on ONE GPU, against the oracle.

A sharded run needs one device, not W of them.  In the collective arm (bb_shard_use_exchange_buffers) route_push fills
LOCAL send regions and bb_shard_resolve(wait_for_peers = 0) reads a receive buffer its caller fills.  So one process holds
W engines (Zone(snapshot, domain, W, r)) and their W shards on cuda:0 and does the all-to-all as device-to-device copies:
the kernels a W-GPU run launches, with no torchrun, NCCL or peer access.  Section 4 runs the peer-store arm as well
(CUDA IPC mappings, epoch flags, wait_regions_kernel) with W processes sharing cuda:0.

Every region (src -> owner) of every step is checked against the oracle's answers for src's whole batch and against the
CPU router (bb_emu_route_batch: the device source's route mode compiled for the host):
  membership  the region's ingress indices are exactly the positions of src's batch the router gives this owner, once;
  answers     statuses, lengths and bytes equal the oracle's at those positions;
  miss list   the region's misses, mapped to ingress positions, are the oracle's misses inside the region;
  layout      ordered packing: responses in region order, out_off the prefix sum of out_len, misses ascending;
              arrival packing: whole responses, no gaps, no overlap;
  totals      n, the miss count and the byte total agree with the arrays.
Receive and send buffers start as a poison pattern, so a kernel reading bytes nobody sent answers wrongly.
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
from binder_b200.engine import Zone, repack
from binder_b200.shard import ShardedEngine
from test_gpu_parity import MODES
from test_host_emulation import emu_lib, padded_queries, size_zone

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAPACITY = -1, -5
POISON = 0xA5
S_IN = 8192                      # staged packet bytes per tile (route_push_kernel, resolve_kernel)
RESULTS = [pytest.param(False, id='device'), pytest.param(True, id='host')]


# ---- expected results ----------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def route(tmp_path_factory):
    """The CPU router: owner rank of every packet of a batch arriving at `rank`."""
    L = emu_lib(tmp_path_factory.mktemp('emu'))

    def fn(dom, recursion, data, off, world, rank):
        data = np.ascontiguousarray(data, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.uint32)
        n = len(off) - 1
        owner = np.zeros(max(n, 1), dtype=np.uint8)
        assert L.bb_emu_route_batch(dom.encode(), int(recursion), data.ctypes.data, off.ctypes.data, n, world, rank,
                                    owner.ctypes.data) == 0
        return owner[:n].astype(np.int64)
    return fn


class Batch(object):
    """One rank's ingress batch of one step with what it should produce: the oracle's results at (seed, qidx_base) and
    the router's owner of every packet."""

    def __init__(self, pkts, rank, world, qidx_base, seed, orc, route, dom, recursion, data=None, off=None):
        if data is None:
            data, off = synth.pack_batch(pkts)
        self.data, self.off, self.n, self.base = data, off, len(off) - 1, qidx_base
        self.res = orc.resolve_batch(data, off, seed=seed, qidx_base=qidx_base, nthreads=os.cpu_count())
        self.owner = route(dom, recursion, data, off, world, rank)


def check_region(reg, b, owner, ordered, what):
    """Region (src -> owner) `reg` (ShardedEngine.fetch) against src's Batch b."""
    o_out, o_off, o_len, o_st, o_miss = b.res
    n = reg['n']
    assert len(reg['qidx']) == len(reg['status']) == len(reg['out_len']) == n and len(reg['out_off']) == n + 1, what
    local = (reg['qidx'].astype(np.int64) - b.base) % (1 << 32)
    want = np.nonzero(b.owner == owner)[0]
    assert np.array_equal(np.sort(local), want), (what, 'membership', n, len(want))
    if n == 0:                          # (bb_shard_fetch copies no offsets for an empty region)
        assert len(reg['out']) == 0 and len(reg['miss']) == 0, what
        return 0
    bad = np.nonzero(reg['status'] != o_st[local])[0]
    assert bad.size == 0, (what, 'status', local[bad[:5]], reg['status'][bad[:5]], o_st[local[bad[:5]]])
    assert np.array_equal(reg['out_len'], o_len[local]), (what, 'lengths')
    lens = reg['out_len'].astype(np.int64)
    assert len(reg['out']) == int(lens.sum()) == int(reg['out_off'][n]), (what, 'total bytes')
    packed, _ = repack(reg['out'], reg['out_off'], reg['out_len'])
    want_bytes, _ = repack(o_out, o_off[:-1][local], o_len[local])
    if not np.array_equal(packed, want_bytes):
        for i in range(n):
            a = bytes(reg['out'][reg['out_off'][i]:reg['out_off'][i] + reg['out_len'][i]])
            q = int(local[i])
            e = bytes(o_out[o_off[q]:o_off[q + 1]])
            assert a == e, (what, 'query %d' % q, bytes(b.data[b.off[q]:b.off[q + 1]]), a.hex(), e.hex())
    miss = reg['miss'].astype(np.int64)
    assert miss.size == 0 or miss.max() < n, (what, 'miss index out of range')
    assert len(miss) == int((reg['status'] == 1).sum()), (what, 'miss count')
    assert np.array_equal(np.sort(local[miss]), o_miss[np.isin(o_miss, want)]), (what, 'miss list')
    if ordered:
        starts = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(lens, out=starts[1:])
        assert np.array_equal(reg['out_off'].astype(np.int64), starts), (what, 'ordered offsets')
        assert np.all(np.diff(miss) > 0), (what, 'miss list not ascending')
    else:
        nz = np.nonzero(lens)[0]
        if nz.size:
            st = reg['out_off'][:n][nz].astype(np.int64)
            order = np.argsort(st, kind='stable')
            st, ln = st[order], lens[nz][order]
            assert st[0] == 0 and np.array_equal(st[1:], (st + ln)[:-1]) and st[-1] + ln[-1] == len(reg['out']), \
                (what, 'gaps or overlap')
        assert len(np.unique(miss)) == len(miss), (what, 'miss listed twice')
    return n


# ---- the in-process cluster ----------------------------------------------------------------------------------------
class Cluster(object):
    """W ranks of one sharded resolver on cuda:0: ShardedEngine in the collective arm (dist=None: its constructor does not
    touch dist in that mode), `lanes` exchange contexts per rank, every exchange buffer poisoned."""

    def __init__(self, dom, snap, world, max_batch, recursion=True, ordered=False, bytes_per_query=64, host=(), lanes=1,
                 dc='', zones=None):
        import torch
        self.world, self.ordered, self.lanes = world, ordered, lanes
        self.ranks = []
        for r in range(world):
            se = ShardedEngine(dom, dc, snap, r, world, 0, max_batch, recursion=recursion, ordered=ordered,
                               bytes_per_query=bytes_per_query, lanes=lanes, sync='nccl_a2a', host_results=r in host)
            self.ranks.append(se)
            if zones is not None:             # the caller keeps these Zone handles to apply deltas to
                se.engine.swap_zone(zones[r])
            for snd, rcv, _, _ in se._xch:
                snd.fill_(POISON)
                rcv.fill_(POISON)
        torch.cuda.synchronize()
        self.lay = self.ranks[0]._lay

    def close(self):
        for se in self.ranks:
            se.close()

    @staticmethod
    def upload(b, dev):
        import torch
        data = b.data if len(b.data) else np.zeros(16, dtype=np.uint8)
        return torch.from_numpy(data).to(dev), torch.from_numpy(b.off.view(np.int32)).to(dev)

    def exchange(self, lane, exact):
        """Send region d of every rank s -> receive region s of rank d, on the current stream.  exact: what
        ShardedEngine.exchange moves (header, 4(c+1) offset bytes, 4c index bytes, the packet bytes rounded up to 16; the
        counts come to the host first); else the whole region, in stream order with no host round trip."""
        import torch
        W = self.world
        reg, _, o_off, o_qi, o_by = self.lay
        sets = set(int(lib().bb_shard_exchange_set(se._lanes[lane])) for se in self.ranks)
        assert len(sets) == 1
        st = sets.pop()
        cut = lambda buf, k: buf[(st * W + k) * reg:(st * W + k + 1) * reg]
        if exact:
            hdr = torch.stack([torch.stack([cut(se._xch[lane][0], d)[:16].view(torch.int32) for d in range(W)])
                               for se in self.ranks]).cpu().numpy()
        for s, se in enumerate(self.ranks):
            for d, de in enumerate(self.ranks):
                sreg, rreg = cut(se._xch[lane][0], d), cut(de._xch[lane][1], s)
                if not exact:
                    rreg.copy_(sreg)
                    continue
                c, nb = int(hdr[s, d, 0]), int(hdr[s, d, 1])
                for o, k in ((0, 16), (o_off, 4 * (c + 1)), (o_qi, 4 * c), (o_by, (nb + 15) // 16 * 16)):
                    if k:
                        rreg[o:o + k].copy_(sreg[o:o + k])

    def enqueue(self, batches, seed, lane=0, exact=True, stream=None):
        """One step on `stream` (default: the current one): route_push of every rank's batch, the exchange, every rank's
        resolve.  Returns the device copies of the batches (keep them until the step has run)."""
        import torch
        st = stream if stream is not None else torch.cuda.current_stream()
        keep = []
        with torch.cuda.stream(st):
            for r, se in enumerate(self.ranks):
                d_pk, d_off = self.upload(batches[r], st.device)
                keep += [d_pk, d_off]
                se.route_push(d_pk.data_ptr(), d_off.data_ptr(), batches[r].n, batches[r].base, st.cuda_stream, lane)
            self.exchange(lane, exact)
            for se in self.ranks:
                se.resolve(seed, st.cuda_stream, lane)
        return keep

    def step(self, batches, seed, lane=0, exact=True):
        import torch
        keep = self.enqueue(batches, seed, lane, exact)
        torch.cuda.synchronize()
        del keep

    def check(self, batches, lane=0, what=''):
        """Every region of the last step on `lane` against its source's Batch: each ingress query answered exactly once."""
        for src, b in enumerate(batches):
            seen = 0
            for d, se in enumerate(self.ranks):
                seen += check_region(se.fetch(src, lane), b, d, self.ordered, (what, 'lane', lane, 'src', src, 'owner', d))
            assert seen == b.n, (what, src, 'coverage', seen, b.n)


def run_steps(cl, make_batches, steps, seed0):
    """`steps` checked steps; step k exchanges exactly on k % 4 in (0, 3) and whole regions otherwise (each of the two
    region sets sees both forms in four steps)."""
    for k in range(steps):
        seed = seed0 + 7919 * k
        batches = make_batches(k, seed)
        cl.step(batches, seed, exact=k % 4 in (0, 3))
        cl.check(batches, what=('step', k))


# ---- workloads -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def fuzz_zones():
    cache = {}

    def get(world):
        if world not in cache:
            snap, info = fuzzgen.gen_zone(900 + world, n_top=40)
            cache[world] = (snap, info, H.make_impl('oracle', info['dns_domain'], snap, recursion=True))
        return cache[world]
    return get


@pytest.fixture(scope='module')
def svc_zone():
    z = synth.gen_zone(30000, service_frac=0.15)
    return z, H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=True)


def fuzz_batches(world, info, orc, route, size=1500):
    dom = info['dns_domain']

    def make(k, seed):
        out = []
        for r in range(world):
            pk = fuzzgen.gen_queries(1000 * k + 10 * world + r, info, n=size) + fuzzgen.malformed_packets() + \
                fuzzgen.tolerated_packets()
            out.append(Batch(pk, r, world, (r * 100003 + k * 7) & 0xFFFFFFFF, seed, orc, route, dom, True))
        return out
    return make


def svc_batches(world, z, orc, route, size=2000):
    def make(k, seed):
        out = []
        for r in range(world):
            pk = synth.batch_mixed(z, size - size * 3 // 10, seed=100 * k + r, miss_frac=0.3) + \
                synth.batch_service(z, size * 3 // 10, seed=77 * k + r)
            out.append(Batch(pk, r, world, r * size, seed, orc, route, z.dns_domain, True))
        return out
    return make


# ---- 2. parity matrix ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('host', RESULTS)
@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('world', [2, 3, 5, 8])
def test_fuzz_zone_shards_match_oracle(fuzz_zones, route, world, ordered, host):
    snap, info, orc = fuzz_zones(world)
    cl = Cluster(info['dns_domain'], snap, world, 2048, ordered=ordered, host=range(world) if host else ())
    try:
        run_steps(cl, fuzz_batches(world, info, orc, route), 4, 0x5EED + world)
    finally:
        cl.close()


@pytest.mark.parametrize('host', RESULTS)
@pytest.mark.parametrize('ordered', MODES)
@pytest.mark.parametrize('world', [2, 8])
def test_service_zone_shards_match_oracle(svc_zone, route, world, ordered, host):
    z, orc = svc_zone
    cl = Cluster(z.dns_domain, z.jsonl, world, 4096, ordered=ordered, host=range(world) if host else (), dc=z.datacenter)
    try:
        make = svc_batches(world, z, orc, route)
        run_steps(cl, make, 3, 0xB1DDE5)
        b = make(0, 1)[0]
        assert len(b.res[4]) > 0.08 * b.n                    # recursion misses in every region
    finally:
        cl.close()


# ---- 3. edges --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('host', RESULTS)
@pytest.mark.parametrize('ordered', MODES)
def test_empty_and_tiny_batches(fuzz_zones, route, ordered, host):
    """n = 0 on every rank (headers still published, every region n = 0, the results accept the epoch); n = 1 on every
    rank of 8 (seven empty regions per source); one rank sending nothing while the others send."""
    world = 8
    snap, info, orc = fuzz_zones(world)
    dom = info['dns_domain']
    cl = Cluster(dom, snap, world, 2048, ordered=ordered, host=range(world) if host else ())
    mk = lambda pk, r, seed: Batch(pk, r, world, r * 1000, seed, orc, route, dom, True)
    try:
        one = fuzzgen.gen_queries(5, info, n=64)[:world]
        assert len(one) == world
        full = fuzz_batches(world, info, orc, route, size=800)
        for k, shape in enumerate(['empty', 'one', 'full', 'empty', 'one_silent', 'one']):
            seed = 31 + k
            if shape == 'empty':
                batches = [mk([], r, seed) for r in range(world)]
            elif shape == 'one':
                batches = [mk(one[r:r + 1], r, seed) for r in range(world)]
            elif shape == 'full':
                batches = full(k, seed)
            else:
                batches = full(k, seed)
                batches[3] = mk([], 3, seed)
            cl.step(batches, seed, exact=k % 2 == 0)
            cl.check(batches, what=shape)
            if shape == 'one':
                for b in batches:
                    assert b.n == 1
                    for d, se in enumerate(cl.ranks):
                        assert se.fetch(0)['n'] == int(batches[0].owner[0] == d)
    finally:
        cl.close()


def owned_names(route, z, world, owner, count, dom):
    """`count` A queries for hosts of zone z that rank `owner` owns."""
    pk = synth.batch_host_a(z, count * world * 2, seed=owner + 17)
    data, off = synth.pack_batch(pk)
    own = route(dom, True, data, off, world, 0)
    idx = np.nonzero(own == owner)[0]
    assert idx.size >= count
    return [pk[i] for i in idx[:count]]


@pytest.mark.parametrize('host', RESULTS)
@pytest.mark.parametrize('ordered', MODES)
def test_hot_owner_fills_a_region(svc_zone, route, ordered, host):
    """A whole max_batch of names rank 2 owns: region (0 -> 2) holds exactly cap_q queries, every other region of
    rank 0 is empty."""
    z, orc = svc_zone
    world, B = 4, 1024
    cl = Cluster(z.dns_domain, z.jsonl, world, B, ordered=ordered, host=range(world) if host else (), dc=z.datacenter)
    try:
        assert cl.ranks[0].cap_q == B
        hot = owned_names(route, z, world, 2, B, z.dns_domain)
        normal = svc_batches(world, z, orc, route, size=B)
        for k in range(3):
            seed = 90 + k
            batches = normal(k, seed)
            batches[0] = Batch(hot, 0, world, 0, seed, orc, route, z.dns_domain, True)
            cl.step(batches, seed, exact=k != 1)
            cl.check(batches, what=('hot', k))
            assert [cl.ranks[d].fetch(0)['n'] for d in range(world)] == [0, 0, B, 0]
    finally:
        cl.close()


def padded_to(pkts, total):
    """The packets with trailing bytes added so that their lengths sum to exactly `total`."""
    base, extra = divmod(total, len(pkts))
    out = []
    for i, p in enumerate(pkts):
        ln = base + (1 if i < extra else 0)
        assert ln >= len(p)
        out.append(p + bytes([0x30 + i % 10]) * (ln - len(p)))
    assert sum(len(p) for p in out) == total
    return out


@pytest.mark.parametrize('host', RESULTS)
@pytest.mark.parametrize('ordered', MODES)
def test_byte_capacity_overflow_fails_only_its_step(svc_zone, route, ordered, host):
    """Exactly cap_b packet bytes to one owner fit; one byte more is BB_ERR_CAPACITY for every region of the sender in
    that step (the other sender's regions are answered); the next step is exact again on every region."""
    z, orc = svc_zone
    world, B, bpq = 2, 512, 64
    cl = Cluster(z.dns_domain, z.jsonl, world, B, ordered=ordered, bytes_per_query=bpq, host=range(world) if host else (),
                 dc=z.datacenter)
    cap_b = B * bpq
    hot = owned_names(route, z, world, 1, 400, z.dns_domain)
    exact = padded_to(hot, cap_b)
    over = exact[:-1] + [exact[-1] + b'!']
    normal = svc_batches(world, z, orc, route, size=400)
    mk = lambda pk, seed: Batch(pk, 0, world, 0, seed, orc, route, z.dns_domain, True)
    try:
        for k, pk in enumerate([exact, over, exact, None, over, None]):
            seed = 50 + k
            batches = normal(k, seed)
            if pk is not None:
                batches[0] = mk(pk, seed)
            cl.step(batches, seed, exact=k % 2 == 0)
            if pk is over:
                for d, se in enumerate(cl.ranks):
                    with pytest.raises(BinderError) as ei:
                        se.fetch(0)
                    assert ei.value.code == ERR_CAPACITY, (k, d)
                    check_region(se.fetch(1), batches[1], d, ordered, ('other sender', k, d))
            else:
                cl.check(batches, what=('byte capacity', k))
                if pk is exact:
                    assert cl.ranks[1].fetch(0)['n'] == len(exact)
    finally:
        cl.close()


def wide_service_zone():
    """foo.com: 200 short host names, 40 hosts with 63-byte labels, and a service of 30 load balancers."""
    ent = [('/com/foo', None), ('/com/foo/svc', {'type': 'service', 'service': {'srvce': '_http', 'proto': '_tcp', 'port': 80}})]
    ent += [('/com/foo/svc/lb%02d' % i, {'type': 'load_balancer', 'load_balancer': {'address': '10.0.0.%d' % i}}) for i in range(30)]
    ent += [('/com/foo/h%03d' % i, {'type': 'host', 'host': {'address': '10.1.%d.%d' % (i >> 8, i & 255)}}) for i in range(200)]
    ent += [('/com/foo/' + long_label(i), {'type': 'host', 'host': {'address': '10.2.0.%d' % i}}) for i in range(40)]
    return H.snapshot(ent)


def long_label(i):
    return 'n%03d' % i + 'q' * 59


@pytest.mark.parametrize('host', RESULTS)
def test_output_capacity_fails_only_its_step(route, host):
    """A region whose answers exceed out_cap = cap_q x 256 (every query an SRV of a 30-child service, EDNS 1232) is
    BB_ERR_CAPACITY through bb_shard_fetch / bb_shard_results; the other regions are answered, and the next step
    recovers."""
    snap = wide_service_zone()
    world, B = 2, 256
    orc = H.make_impl('oracle', 'foo.com', snap)
    cl = Cluster('foo.com', snap, world, B, recursion=False, host=range(world) if host else ())
    mk = lambda pk, r, seed: Batch(pk, r, world, r * B, seed, orc, route, 'foo.com', False)
    wide = [synth.make_query('_http._tcp.svc.foo.com', 'SRV', i, edns=1232) for i in range(B)]
    small = lambda k: [synth.make_query('h%03d.foo.com' % ((7 * i + k) % 200), 'A', i) for i in range(B)]
    try:
        for k in range(3):
            seed = 60 + k
            batches = [mk(wide if k == 1 else small(k), 0, seed), mk(small(k + 5), 1, seed)]
            cl.step(batches, seed, exact=True)
            if k != 1:
                cl.check(batches, what=('output capacity', k))
                continue
            hot = int(batches[0].owner[0])
            assert (batches[0].owner == hot).all() and int(batches[0].res[1][-1]) > B * 256
            with pytest.raises(BinderError) as ei:
                cl.ranks[hot].fetch(0)
            assert ei.value.code == ERR_CAPACITY
            check_region(cl.ranks[1 - hot].fetch(0), batches[0], 1 - hot, False, 'empty region')
            for d, se in enumerate(cl.ranks):
                check_region(se.fetch(1), batches[1], d, False, ('other sender', d))
    finally:
        cl.close()


def big_tile_packets(k):
    """Tiles of 128 packets of 100 bytes (a 63-byte label and an OPT: > S_IN bytes per tile), tiles of short queries,
    and tiles mixing both; present and absent names, so every tile has several owners.  The long packets end in the
    OPT's RDLENGTH: a byte short and the answer changes."""
    longq = lambda i: synth.make_query(long_label((i + k) % 60) + '.foo.com', 'A', i, edns=1232)   # 20 of 60 are absent
    short = lambda i: synth.make_query('h%03d.foo.com' % ((i * 7 + k) % 230), 'A' if i % 5 else 'AAAA', i) \
        if i % 9 else synth.make_query('_http._tcp.svc.foo.com', 'SRV', i)
    pk = [longq(i) for i in range(256)] + [short(i) for i in range(256)]
    pk += [longq(i) if i % 2 else short(i) for i in range(384)] + [longq(i) if i % 4 == 0 else short(i) for i in range(300)]
    return pk


@pytest.mark.parametrize('host', RESULTS)
@pytest.mark.parametrize('ordered', MODES)
def test_tiles_over_the_staging_buffer(route, ordered, host):
    """Tiles of more than S_IN packet bytes take route_push_kernel's unstaged branch (byte-wise stores) and the owners'
    unstaged tiles, next to staged tiles in the same batch."""
    snap = wide_service_zone()
    world = 3
    orc = H.make_impl('oracle', 'foo.com', snap, recursion=True)
    cl = Cluster('foo.com', snap, world, 2048, ordered=ordered, host=range(world) if host else ())
    try:
        def make(k, seed):
            return [Batch(big_tile_packets(3 * k + r), r, world, r * 5000, seed, orc, route, 'foo.com', True) for r in range(world)]
        b = make(0, 0)[0]
        tiles = [int(b.off[min(t + 128, b.n)]) - (int(b.off[t]) & ~15) for t in range(0, b.n, 128)]
        assert max(tiles) > S_IN >= min(tiles) and sum(t > S_IN for t in tiles) >= 4
        assert all(len(set(b.owner[t:t + 128].tolist())) == world for t in range(0, 256, 128))
        run_steps(cl, make, 4, 0xB16)
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
def test_packet_length_limit(route, ordered):
    """Packets of 65,534 and 65,535 bytes are routed and answered; 65,536 and 70,000 bytes stay on the ingress rank,
    dropped (status 2)."""
    snap = size_zone()
    world = 2
    orc = H.make_impl('oracle', 'foo.com', snap)
    cl = Cluster('foo.com', snap, world, 64, recursion=False, ordered=ordered, bytes_per_query=8192)
    try:
        lengths = [65534, 65535, 65536, 70000, 65535, 70000]
        for k in range(3):
            seed = 5 + k
            batches = [Batch(padded_queries(lengths[k:] + lengths[:k]) if r == k % 2 else padded_queries([100, 200]),
                             r, world, r * 64, seed, orc, route, 'foo.com', False) for r in range(world)]
            cl.step(batches, seed, exact=k != 1)
            cl.check(batches, what=('length', k))
            b, r = batches[k % 2], k % 2
            lens = np.diff(b.off.astype(np.int64))
            assert list(b.res[3][0::2]) == [0 if ln <= 65535 else 2 for ln in lens[0::2]]
            assert (b.owner[0::2][lens[0::2] > 65535] == r).all()
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
def test_zero_length_and_malformed_stay_home(fuzz_zones, route, ordered):
    """Zero-length and malformed packets need no lookup: they stay in region (r -> r), with the oracle's statuses."""
    world = 3
    snap, info, orc = fuzz_zones(world)
    dom = info['dns_domain']
    cl = Cluster(dom, snap, world, 2048, ordered=ordered)
    try:
        for k in range(3):
            seed = 70 + k
            batches = []
            for r in range(world):
                pk = fuzzgen.gen_queries(300 * k + r, info, n=600)
                pk = pk[:50] + [b''] * 3 + pk[50:300] + [b''] * 128 + fuzzgen.malformed_packets() + pk[300:]
                batches.append(Batch(pk, r, world, r * 4000, seed, orc, route, dom, True))
            cl.step(batches, seed, exact=k != 1)
            cl.check(batches, what=('zero-length', k))
            for r, b in enumerate(batches):
                lens = np.diff(b.off.astype(np.int64))
                assert (b.owner[lens == 0] == r).all() and (b.res[3][lens == 0] == 2).all()
                assert (lens == 0).sum() >= 131
    finally:
        cl.close()


def test_offsets_from_byte_five_and_misaligned_pointer(svc_zone, route):
    """A batch whose offsets start at byte 5 of a 16-byte aligned buffer is routed and answered; a d_pkts that is not
    16-byte aligned is BB_ERR_ARG."""
    import torch
    z, orc = svc_zone
    world = 3
    cl = Cluster(z.dns_domain, z.jsonl, world, 2048, dc=z.datacenter)
    try:
        batches = []
        for r in range(world):
            data, off = synth.pack_batch(synth.batch_mixed(z, 1000, seed=14 + r, miss_frac=0.2))
            d5 = np.concatenate([np.full(5, 0xEE, np.uint8), data, np.zeros(11, np.uint8)])
            batches.append(Batch(None, r, world, r * 1000, 22, orc, route, z.dns_domain, True, data=d5, off=off + np.uint32(5)))
        cl.step(batches, 22)
        cl.check(batches, what='offset 5')
        d_pk, d_off = Cluster.upload(batches[0], torch.device('cuda:0'))
        for k in (1, 4, 8):
            assert lib().bb_shard_route_push(cl.ranks[0]._h, d_pk.data_ptr() + k, d_off.data_ptr(), batches[0].n, 0,
                                             torch.cuda.current_stream().cuda_stream) == ERR_ARG
        cl.step(batches, 22)                       # nothing was launched by the refused calls
        cl.check(batches, what='after refusals')
    finally:
        cl.close()


@pytest.mark.parametrize('host', RESULTS)
def test_ingress_index_wraps(svc_zone, route, host):
    """qidx_base = 2^32 - 200 on every rank: the returned indices wrap to 0, and the shuffle (keyed by the ingress
    index) matches the oracle's at the same base."""
    z, orc = svc_zone
    world = 3
    cl = Cluster(z.dns_domain, z.jsonl, world, 2048, ordered=True, host=range(world) if host else (), dc=z.datacenter)
    try:
        for k in range(3):
            batches = [Batch(synth.batch_service(z, 1000, seed=12 + 3 * k + r, srv_frac=0.6), r, world, 2 ** 32 - 200, 21 + k,
                             orc, route, z.dns_domain, True) for r in range(world)]
            cl.step(batches, 21 + k, exact=k != 1)
            cl.check(batches, what=('wrap', k))
            q = np.concatenate([se.fetch(0)['qidx'] for se in cl.ranks]).astype(np.int64)
            assert (q < 800).sum() == 800 and (q >= 2 ** 32 - 200).sum() == 200
    finally:
        cl.close()


def _err(fn):
    try:
        fn()
    except BinderError as e:
        return e.code
    return 0


def test_argument_errors(svc_zone):
    """bb_shard_create with nranks 0 or 9, rank >= nranks, max_batch over the engine's; route_push with n > max_batch;
    fetch / results with src >= nranks; bb_shard_fetch while host mirrors are on; bb_shard_results before any resolve."""
    import torch
    z, orc = svc_zone
    L = lib()
    se = ShardedEngine(z.dns_domain, z.datacenter, z.jsonl, 0, 2, 0, 1024, recursion=True, sync='nccl_a2a')
    try:
        h = se.engine._h
        err = ctypes.c_int(0)
        for nranks, rank, mb in ((0, 0, 512), (9, 0, 512), (2, 2, 512), (3, 5, 512), (2, 1, 1025), (2, 0, 0)):
            assert not L.bb_shard_create(h, nranks, rank, mb, 64, ctypes.byref(err)), (nranks, rank, mb)
            assert err.value == ERR_ARG
        s8 = L.bb_shard_create(h, 8, 7, 1024, 64, ctypes.byref(err))
        assert s8 and err.value == 0
        L.bb_shard_destroy(s8)
        data, off = synth.pack_batch(synth.batch_mixed(z, 1025, seed=3))
        d_pk, d_off = torch.from_numpy(data).cuda(), torch.from_numpy(off.view(np.int32)).cuda()
        stream = torch.cuda.current_stream().cuda_stream
        assert L.bb_shard_route_push(se._h, d_pk.data_ptr(), d_off.data_ptr(), 1025, 0, stream) == ERR_ARG
        P = ctypes.POINTER
        ptrs = [P(ctypes.c_uint8)() for _ in range(6)]
        cnt = [ctypes.c_uint32(0) for _ in range(3)]
        results = lambda src: L.bb_shard_results(se._h, src, *[ctypes.byref(p) for p in ptrs], *[ctypes.byref(c) for c in cnt])
        se.set_host_results(True)
        assert results(0) == ERR_ARG                          # no resolve yet
        se.set_host_results(False)
        check(L.bb_shard_route_push(se._h, d_pk.data_ptr(), d_off.data_ptr(), 1000, 0, stream))
        se._xch[0][1].zero_()                                 # every receive region empty: a valid, empty exchange
        check(L.bb_shard_resolve(se._h, 1, 0, stream))
        torch.cuda.synchronize()
        assert _err(lambda: se.fetch(2)) == ERR_ARG and _err(lambda: se.fetch(7)) == ERR_ARG
        assert se.fetch(0)['n'] == 0 and se.fetch(1)['n'] == 0
        se.set_host_results(True)
        b = se._bufs(0, 0)
        n, nm, tot = ctypes.c_uint32(0), ctypes.c_uint32(0), ctypes.c_uint32(0)
        assert L.bb_shard_fetch(se._h, 0, b['out'].ctypes.data, b['out'].size, b['out_off'].ctypes.data, b['out_len'].ctypes.data,
                                b['status'].ctypes.data, b['qidx'].ctypes.data, b['miss'].ctypes.data, ctypes.byref(n),
                                ctypes.byref(nm), ctypes.byref(tot)) == ERR_ARG
        assert results(0) == ERR_ARG                          # mirrors switched on after that resolve: its epoch is not theirs
        check(L.bb_shard_resolve(se._h, 2, 0, stream))
        torch.cuda.synchronize()
        assert results(0) == 0 and cnt[0].value == 0
        assert results(2) == ERR_ARG and results(9) == ERR_ARG
    finally:
        se.close()


def test_several_waves_per_region(route):
    """W = 2, 262,144 config-3 queries per rank, ordered packing: 2,048 tiles x 2 regions in one launch, the look-back
    running inside each region.  Rank 0 takes its results through host mirrors, rank 1 through device buffers."""
    z = synth.gen_zone(100000, service_frac=0.15)
    orc = H.make_impl('oracle', z.dns_domain, z.jsonl, recursion=True)
    world, B = 2, 262144
    _, _, mix, miss_frac, _ = synth.WORKLOADS['config3']
    cl = Cluster(z.dns_domain, z.jsonl, world, B, ordered=True, host=(0,), dc=z.datacenter)
    try:
        def make(k, seed):
            out = []
            for r in range(world):
                data, off, _ = synth.gen_batch(z, B, 11 * k + r, mix, miss_frac)
                out.append(Batch(None, r, world, r * B, seed, orc, route, z.dns_domain, True, data=data, off=off))
            return out
        for k in range(2):
            seed = 0x5EED + k
            batches = make(k, seed)
            cl.step(batches, seed, exact=k == 0)
            cl.check(batches, what=('waves', k))
            assert min(se.fetch(s)['n'] for se in cl.ranks for s in range(world)) > 3 * B // 8
    finally:
        cl.close()


@pytest.mark.parametrize('ordered', MODES)
def test_two_lanes_on_two_streams(fuzz_zones, route, ordered):
    """Two shard lanes per rank: both lanes' steps (route_push, whole-region exchange, resolve) are enqueued on two
    streams before anything synchronises; each lane then holds its own step's answers."""
    import torch
    world = 3
    snap, info, orc = fuzz_zones(world)
    cl = Cluster(info['dns_domain'], snap, world, 2048, ordered=ordered, host=(1,), lanes=2)
    make = fuzz_batches(world, info, orc, route, size=1200)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    try:
        for rnd in range(3):
            work = [make(10 + 2 * rnd + lane, 300 + 2 * rnd + lane) for lane in range(2)]
            keep = [cl.enqueue(work[lane], 300 + 2 * rnd + lane, lane=lane, exact=False, stream=streams[lane]) for lane in range(2)]
            torch.cuda.synchronize()
            del keep
            for lane in range(2):
                cl.check(work[lane], lane=lane, what=('lanes', rnd))
    finally:
        cl.close()


def test_zone_deltas_on_every_shard(route):
    """W = 3: each of 4 rounds of watch events is applied to every rank's Zone(..., 3, r) and uploaded
    (apply_update); every step matches an oracle that applied the same events (DESIGN.md section 9)."""
    world = 3
    snap, info = fuzzgen.gen_zone(1300, n_top=30)
    dom = info['dns_domain']
    orc = H.make_impl('oracle', dom, snap, recursion=True)
    zones = [Zone(snap, dom, world, r) for r in range(world)]
    cl = Cluster(dom, snap, world, 2048, zones=zones)
    paths = fuzzgen.snapshot_paths(snap)
    try:
        for rnd in range(4):
            delta, paths = fuzzgen.gen_delta(4242 + rnd, paths, info, n_ops=60)
            for se, zone in zip(cl.ranks, zones):
                zone.apply(delta)
                se.engine.apply_update(zone)
                assert zone.pending() == (0, False)
            orc.apply_delta(delta)
            seed = 800 + rnd
            batches = [Batch(fuzzgen.gen_queries(50 * rnd + r, info, n=1500), r, world, r * 2000, seed, orc, route, dom, True)
                       for r in range(world)]
            cl.step(batches, seed, exact=rnd % 2 == 0)
            cl.check(batches, what=('delta', rnd))
    finally:
        cl.close()
        for zone in zones:
            zone.close()


# ---- 4. peer stores across processes on one GPU ----------------------------------------------------------------------
def _peer_worker(rank, world, port, ordered, host, dom, snap, work, q):
    """One rank in its own process on cuda:0: ShardedEngine(sync='flags') pushes into the other processes' receive
    buffers through CUDA IPC mappings and publishes the epoch flags; resolve waits for them (already published here)."""
    se = None
    try:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(0)
        dist.init_process_group('gloo', rank=rank, world_size=world)
        se = ShardedEngine(dom, '', snap, rank, world, 0, 2048, recursion=True, ordered=ordered, dist=dist,
                           sync='flags', host_results=host)
        st = torch.cuda.current_stream()
        for k, (seed, batches) in enumerate(work):
            b = batches[rank]
            d_pk, d_off = Cluster.upload(b, torch.device('cuda:0'))
            se.route_push(d_pk.data_ptr(), d_off.data_ptr(), b.n, b.base, st.cuda_stream)
            torch.cuda.synchronize()
            dist.barrier()                               # every rank's flags are published: the wait kernel returns at once
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


@pytest.mark.parametrize('world,ordered,host', [(2, False, False), (2, True, False), (3, False, True)],
                         ids=['w2-arrival', 'w2-ordered', 'w3-host'])
def test_peer_stores_across_processes(fuzz_zones, route, world, ordered, host):
    import torch.multiprocessing as mp
    snap, info, orc = fuzz_zones(world)
    dom = info['dns_domain']
    make = fuzz_batches(world, info, orc, route, size=1000)
    work = []
    for k in range(3):
        seed = 1234 + k
        work.append((seed, make(20 + k, seed)))
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 31000 + (os.getpid() + world * 7 + ordered) % 2000
    procs = [ctx.Process(target=_peer_worker, args=(r, world, port, ordered, host, dom, snap, work, q)) for r in range(world)]
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
