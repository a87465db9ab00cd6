"""The sharded pipeline for TCP batches on the CPU: route mode of the device source (bb_emu_route_batch) picks each
query's owner, the owner's shard resolves its region at the queries' ingress indices with the TCP flag set — the flag a
region header carries to the multi-region kernel — and every answer must equal the unsharded oracle's TCP answer."""
import numpy as np
import pytest

import fuzzgen
import helpers as H
from binder_b200 import synth
from test_host_emulation import EmuEngine, emu_lib
from test_tcp import big_zone, big_zone_batch


@pytest.fixture(scope='module')
def L(tmp_path_factory):
    return emu_lib(tmp_path_factory.mktemp('emu'))


def sharded_tcp_matches_oracle(L, dom, snap, pkts, world, recursion, seed, qidx_base):
    orc = H.make_impl('oracle', dom, snap, recursion=recursion)
    shards = [EmuEngine(L, dom, snap, recursion=recursion, nranks=world, rank=r) for r in range(world)]
    data, off = synth.pack_batch(pkts)
    n = len(pkts)
    ingress = (world - 1) // 2
    owner = np.zeros(n, dtype=np.uint8)
    assert L.bb_emu_route_batch(dom.encode(), int(recursion), data.ctypes.data, off.ctypes.data, n, world, ingress,
                                owner.ctypes.data) == 0
    o_out, o_off, o_len, o_st, o_miss = orc.resolve_batch(data, off, seed=seed, qidx_base=qidx_base, tcp=True)
    assert len(set(owner.tolist())) > 1
    seen = 0
    for r in range(world):
        idx = np.nonzero(owner == r)[0]
        if idx.size == 0:
            continue
        d, o = synth.pack_batch([pkts[i] for i in idx])
        out, ooff, olen, st, miss = shards[r].resolve_batch(d, o, seed=seed, tcp=True, qidx_map=(qidx_base + idx).astype(np.uint32))
        assert np.array_equal(st, o_st[idx]) and np.array_equal(olen, o_len[idx]), (r, 'status/lengths')
        for k, i in enumerate(idx):
            assert bytes(out[ooff[k]:ooff[k] + olen[k]]) == bytes(o_out[o_off[i]:o_off[i + 1]]), (r, int(i), pkts[i])
        assert sorted(int(idx[m]) for m in miss) == [int(i) for i in o_miss if owner[i] == r]
        seen += idx.size
    assert seen == n
    return o_len


@pytest.mark.parametrize('seed,world', [(0, 2), (1, 3), (2, 5), (3, 8)])
def test_emulated_sharded_pipeline_tcp(L, seed, world):
    """Fuzz zones: every region answered at its ingress indices under TCP limits equals the oracle with tcp=True."""
    snap, info = fuzzgen.gen_zone(seed + 640, n_top=35)
    pkts = fuzzgen.gen_queries(seed + 40, info, n=2500) + fuzzgen.malformed_packets()
    sharded_tcp_matches_oracle(L, info['dns_domain'], snap, pkts, world, True, 91 + seed, 7000 * seed)


@pytest.mark.parametrize('world', [2, 3, 5, 8])
def test_emulated_sharded_large_answers_tcp(L, world):
    """The 200- and 1,300-child services: SRV and A answers whole over TCP, the 2,600 SRV RRs cut at 65,516 bytes."""
    lens = sharded_tcp_matches_oracle(L, 'foo.com', big_zone(), big_zone_batch(), world, False, 5 + world, 2 ** 32 - 300)
    assert lens.max() == 65516 and (lens > 1232).sum() > 100
