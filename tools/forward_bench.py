"""Recursion forward and match throughput (bb_forward_batch_device / bb_match_upstreams_device, DESIGN.md section 14) on
a config-5-shaped step: a 65,536-query resolve batch of which 90 % miss (dc2, dc3 and PTR misses, a few with nowhere to
go), i.e. one forward call of ~59,000 misses, the largest a call takes (16-bit IDs).

Everything stays in HBM.  The upstream responses are the forwarded queries themselves with QR set, arriving from the
first upstream of their route (the match accepts them: same ID, same question), built once on the host from the first
forward's output.  Reports, as one JSON line (CUDA events over --steps launches after --warmup, each timed separately):
  forward  forwarded misses per second (bb_forward_batch_device straight from the resolve launch's miss list)
  match    received responses per second (bb_match_upstreams_device)
  chain    ms per step of resolve -> forward -> match -> relay, all device-resident, on one stream
  gpu      card name, power limit and max SM clock, read in the same run

    python tools/forward_bench.py [--steps 50] [--warmup 10]
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                      # noqa: BLE001
        return 'unknown (%s)' % ex


def batch(n, seed):
    from binder_b200 import synth
    rng = random.Random(seed)
    pkts = []
    for _ in range(n):
        x = rng.random()
        if x < 0.1:
            name, t = 'h%d.dc1.foo.com' % rng.randrange(200), 'A'
        elif x < 0.75:
            name, t = 'h%d.dc2.foo.com' % rng.randrange(100000), 'A'
        elif x < 0.88:
            name, t = '_http._tcp.s%d.dc3.foo.com' % rng.randrange(100000), 'SRV'
        elif x < 0.95:
            name, t = '%d.%d.2.10.in-addr.arpa' % (rng.randrange(256), rng.randrange(256)), 'PTR'
        else:
            name, t = 'h%d.nodc.foo.com' % rng.randrange(1000), 'A'
        pkts.append(synth.make_query(name, t, qid=rng.randrange(65536), edns=rng.choice([None, 1200])))
    return synth.pack_batch(pkts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    args = ap.parse_args()
    import torch
    from binder_b200 import synth
    from binder_b200.engine import Engine, ip_u32
    import helpers as H
    if not torch.cuda.is_available():
        raise SystemExit('forward_bench: no CUDA device (nothing is measured on the CPU)')
    dev = torch.device('cuda:0')
    ent = [('/com/foo/dc1', None)] + [('/com/foo/dc1/h%d' % i, {'type': 'host', 'host': {'address': '10.1.0.%d' % (i % 250)}})
                                      for i in range(200)]
    n = 65536
    # ordered packing: every resolve launch lists the misses in the same order, so the responses built once from the first
    # forward's queries answer the same misses in every timed step (arrival packing may list them in another order)
    e = Engine('foo.com', '', True, snapshot=H.snapshot(ent), max_batch=n, ordered=True)
    dcs = ['dc2', 'dc3']
    ups = [('10.0.0.2', 53, 0), ('10.0.0.3', 53, 0), ('10.0.1.2', 53, 1)]
    e.set_recursion_filter('foo.com', dcs, True)
    e.set_recursion_upstreams(ups)
    data, off = batch(n, 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                       # noqa: E731
    z = lambda k, dt=torch.int32: torch.zeros(k, dtype=dt, device=dev)                    # noqa: E731
    d_pk, d_off = t(np.concatenate([data, np.zeros(16, np.uint8)])), t(off.view(np.int32))
    cap = len(data) + 64
    r_out, r_off, r_len, r_st, r_miss, r_tot = z(n * 1232, torch.uint8), z(n + 1), z(n, torch.int16), z(n, torch.uint8), z(n), z(4)
    f_uq, f_uqoff, f_order, f_goff, f_route = z(cap, torch.uint8), z(n + 1), z(n), z(19), z(n, torch.uint8)
    f_q, f_qoff, f_tot = z(cap, torch.uint8), z(n + 1), z(8)
    key = 0x5EED

    def resolve():
        e.resolve_device(d_pk.data_ptr(), d_off.data_ptr(), n, 3, 0, r_out.data_ptr(), n * 1232, r_off.data_ptr(), r_len.data_ptr(),
                         r_st.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr())

    def forward():
        e.forward_device(d_pk.data_ptr(), d_off.data_ptr(), r_miss.data_ptr(), r_tot.data_ptr(), n, key, f_uq.data_ptr(), cap,
                         f_uqoff.data_ptr(), f_order.data_ptr(), f_goff.data_ptr(), f_route.data_ptr(), f_q.data_ptr(), cap,
                         f_qoff.data_ptr(), f_tot.data_ptr())

    resolve()
    forward()
    torch.cuda.synchronize()
    ft = f_tot.cpu().numpy().view(np.uint32)
    m = int(ft[1])
    goff = f_goff.cpu().numpy().view(np.uint32)
    uq = f_uq.cpu().numpy()[:ft[0]]
    uq_off = f_uqoff.cpu().numpy().view(np.uint32)[:m + 1]
    # responses: every sent query echoed with QR set, from the first upstream of its route
    first = {0: ups[0][:2], 1: ups[2][:2], 16: ups[0][:2]}
    resp, src = [], []
    for r in (0, 1, 16):
        for k in range(int(goff[r]), int(goff[r + 1])):
            q = bytearray(uq[uq_off[k]:uq_off[k + 1]].tobytes())
            q[2] |= 0x80
            resp.append(bytes(q))
            src.append(first[r])
    rd, ro = synth.pack_batch(resp)
    d_rd, d_ro = t(np.concatenate([rd, np.zeros(16, np.uint8)])), t(ro.view(np.int32))
    d_ip = t(np.array([ip_u32(a) for a, _ in src], np.uint32).view(np.int32))
    d_port = t(np.array([p for _, p in src], np.uint16).view(np.int16))
    m_up, m_upoff, m_tot = z(len(rd) + 64, torch.uint8), z(n + 1), z(4)
    o_cap = m * 1200
    o_out, o_ooff, o_len, o_st, o_tot = z(o_cap, torch.uint8), z(m + 1), z(m, torch.int16), z(m, torch.uint8), z(4)

    def match():
        e.match_device(d_rd.data_ptr(), d_ro.data_ptr(), d_ip.data_ptr(), d_port.data_ptr(), len(resp), f_q.data_ptr(),
                       f_qoff.data_ptr(), f_route.data_ptr(), f_tot.data_ptr(), n, key, m_up.data_ptr(), len(rd) + 64,
                       m_upoff.data_ptr(), m_tot.data_ptr())

    def relay():
        e.relay_device(f_q.data_ptr(), f_qoff.data_ptr(), m_up.data_ptr(), m_upoff.data_ptr(), m, o_out.data_ptr(), o_cap,
                       o_ooff.data_ptr(), o_len.data_ptr(), o_st.data_ptr(), o_tot.data_ptr())

    def chain():
        resolve(); forward(); match(); relay()       # noqa: E702

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()             # noqa: E702
            ts.append((a, b))
        torch.cuda.synchronize()
        return float(np.median([a.elapsed_time(b) for a, b in ts]))

    chain()
    torch.cuda.synchronize()
    mt = m_tot.cpu().numpy().view(np.uint32)
    assert int(mt[1]) == int(goff[17]), (int(mt[1]), int(goff[17]))
    assert int(o_tot.cpu().numpy().view(np.uint32)[3]) == lib_epoch(e)
    f_ms, m_ms, c_ms = timed(forward), timed(match), timed(chain)
    print(json.dumps({
        'metric': 'forward_misses_per_sec', 'value': m / (f_ms * 1e-3), 'unit': 'misses/s',
        'forward': {'misses': m, 'forwarded': int(goff[17]), 'ms': f_ms},
        'match': {'responses': len(resp), 'responses_per_sec': len(resp) / (m_ms * 1e-3), 'ms': m_ms, 'answered': int(mt[1])},
        'chain': {'ms_per_step': c_ms, 'queries': n, 'what': 'resolve -> forward -> match -> relay, device-resident, one stream'},
        'timing': 'CUDA events, median of %d launches after %d warm-up' % (args.steps, args.warmup),
        'gpu': gpu_info(),
    }))


def lib_epoch(e):
    from binder_b200._lib import lib
    return int(lib().bb_engine_launch_epoch(e._h))


if __name__ == '__main__':
    main()
