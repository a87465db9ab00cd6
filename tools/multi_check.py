"""Sharded multi-GPU parity check (run under torchrun, one rank per GPU):
every query of every rank's ingress batch must be answered exactly once, by the rank that owns
its key, with the bytes the single-engine CPU oracle produces for (seed, ingress index).
--tcp: every rank pushes its batches as TCP queries (bb_shard_route_push_ex, BB_BATCH_TCP), checked against the oracle's
TCP answers (no UDP size limit)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'oracle')]
import numpy as np
import torch
import torch.distributed as dist
from binder_b200 import synth, build
from binder_b200.shard import ShardedEngine
from oracle_lib import Oracle


def main():
    rank = int(os.environ['RANK']); world = int(os.environ['WORLD_SIZE']); lr = int(os.environ.get('LOCAL_RANK', rank))
    torch.cuda.set_device(lr)
    dist.init_process_group('nccl', device_id=torch.device('cuda', lr))
    if rank == 0:
        build.build()
    dist.barrier()
    tcp = '--tcp' in sys.argv[1:]
    B = int(os.environ.get('BB_BATCH', '20000'))
    zone = synth.gen_zone(int(os.environ.get('BB_ZONE', '200000')), service_frac=0.15)
    se = ShardedEngine(zone.dns_domain, zone.datacenter, zone.jsonl, rank, world, lr, max_batch=B, recursion=True,
                       ordered=bool(int(os.environ.get('BB_ORDERED', '0'))), dist=dist, sync=os.environ.get('BB_SYNC', 'flags'),
                       host_results=bool(int(os.environ.get('BB_HOST_RESULTS', '0'))))
    orc = Oracle(zone.dns_domain, zone.datacenter, True, snapshot=zone.jsonl)

    def ingress(r, rnd):      # rank r's batch in round rnd (any rank can regenerate it)
        pk = synth.batch_mixed(zone, B - 7000, seed=1000 * rnd + r, miss_frac=0.3) + synth.batch_service(zone, 6000, seed=77 * rnd + r)
        pk += [b'\x00' * 5] * 500 + [synth.make_query('1.0.0.10.in-addr.arpa', 'PTR')] * 500
        return synth.pack_batch(pk)

    dev = torch.device('cuda', lr)
    st = torch.cuda.current_stream()
    for rnd in range(3):
        data, off = ingress(rank, rnd)
        n = len(off) - 1
        d_pk = torch.from_numpy(data).to(dev); d_off = torch.from_numpy(off.view(np.int32)).to(dev)
        seed = 0xB1DDE5 + rnd
        se.step(d_pk.data_ptr(), d_off.data_ptr(), n, rank * B, seed, st.cuda_stream, tcp=tcp)
        torch.cuda.synchronize()
        got = torch.zeros(world, dtype=torch.int64, device=dev)
        nonlocal_bytes = 0
        for src in range(world):
            reg = se.fetch(src)
            sdata, soff = ingress(src, rnd)
            o_out, o_off, o_len, o_st, o_miss = orc.resolve_batch(sdata, soff, seed=seed, qidx_base=src * B, tcp=tcp)
            local = reg['qidx'].astype(np.int64) - src * B
            assert local.min(initial=0) >= 0 and local.max(initial=0) < len(soff) - 1
            assert len(np.unique(local)) == len(local), 'a query was delivered twice'
            assert np.array_equal(reg['status'], o_st[local]), (rank, src, 'status')
            assert np.array_equal(reg['out_len'], o_len[local]), (rank, src, 'lengths')
            for i in np.random.default_rng(rnd).permutation(reg['n'])[:4000]:
                a = bytes(reg['out'][reg['out_off'][i]:reg['out_off'][i] + reg['out_len'][i]])
                q = local[i]
                b = bytes(o_out[o_off[q]:o_off[q + 1]])
                assert a == b, (rank, src, int(q), a.hex(), b.hex())
            # vectorised full compare
            from binder_b200.engine import repack
            packed, _ = repack(reg['out'], reg['out_off'], reg['out_len'])
            want, _ = repack(o_out, o_off[:-1][local].astype(np.uint32) if len(local) else np.zeros(0, np.uint32), o_len[local])
            assert np.array_equal(packed, want), (rank, src, 'bytes')
            # the region's miss list (region positions) names exactly the oracle's misses among its queries; the totals
            # (query count, miss count, response bytes) agree with the arrays and with the oracle
            miss = reg['miss'].astype(np.int64)
            assert miss.size == 0 or miss.max() < reg['n'], (rank, src, 'miss index out of range')
            assert np.array_equal(np.sort(local[miss]), o_miss[np.isin(o_miss, local)]), (rank, src, 'miss list')
            assert len(miss) == int((reg['status'] == 1).sum()), (rank, src, 'miss count')
            assert len(reg['out']) == int(reg['out_len'].astype(np.int64).sum()) == int(o_len[local].astype(np.int64).sum()), (rank, src, 'total bytes')
            if se.engine.ordered and reg['n']:
                assert np.array_equal(reg['out_off'][:reg['n']].astype(np.int64), np.cumsum(reg['out_len'].astype(np.int64)) - reg['out_len']), (rank, src, 'ordered offsets')
                assert np.all(np.diff(miss) > 0), (rank, src, 'miss list not ascending')
            got[src] += reg['n']
            if src != rank:
                nonlocal_bytes += int(reg['out_len'].sum())
        dist.all_reduce(got)
        assert all(int(g) == B for g in got), ('coverage', got.tolist())
        if rank == 0:
            print('round %d ok: %s queries/rank routed over %d ranks (rank 0 owned %d from peers)' % (rnd, B, world, int(se.fetch(1 % world)['n'])), flush=True)
    dist.barrier()
    if rank == 0:
        print('MULTI_CHECK_OK world=%d%s' % (world, ' tcp' if tcp else ''), flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
