"""Recursion relay throughput (bb_relay_batch_device / bb_relay_batch, DESIGN.md section 13) on a config-5-shaped step:
the 90 % misses of a 1,048,576-query batch, 943,718 relays, each a client query plus its upstream response.

Upstream mix: one A; CNAME + A; three SRV with compressed targets; NXDOMAIN; empty (failed lookup) — a few hundred
distinct templates built with dnspython (tests/relaygen.py), tiled with numpy.  Reports, as one JSON line:
  device   relays/s with inputs and outputs in HBM (CUDA events, after warm-up, over a ring of batches larger than the
           50 MB L2), and the algorithmic bytes per relay (query + upstream + reply + offsets, lengths, status) over the
           kernel time as a fraction of the H100 SXM data-sheet HBM bandwidth (3.35 TB/s)
  e2e      relays/s through bb_relay_batch with pinned host buffers (H2D of the inputs, results written into host memory)
  oracle   the relay oracle (tests/native/relay_oracle.cpp) on the host's threads, for context
  parity   every reply of the last timed device step against the oracle
  gpu      card name, power limit and max SM clock, read in the same run

    python tools/relay_bench.py [--steps 50] [--warmup 10] [--n 943718]
"""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM = 3.35e12
MIX = ('a', 'cname_a', 'srv3', 'nxdomain', 'empty')


def templates(n_each=80, seed=1):
    import relaygen as G
    rng = random.Random(seed)
    return [G.relay_case(rng, k) for k in MIX for _ in range(n_each)]


def tile(tpl, n, seed):
    """n (query, upstream) pairs drawn from the templates, packed with numpy: (q_data, q_off, up_data, up_off)."""
    idx = np.random.default_rng(seed).integers(len(tpl), size=n)
    out = []
    for which in (0, 1):
        blob = np.frombuffer(b''.join(t[which] for t in tpl), dtype=np.uint8)
        lens = np.array([len(t[which]) for t in tpl], dtype=np.int64)
        starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
        l = lens[idx]
        off = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(l, out=off[1:])
        total = int(off[-1])
        src = np.repeat(starts[idx] - off[:-1], l) + np.arange(total)
        data = np.zeros(total + 16 + (-total) % 16, dtype=np.uint8)
        data[:total] = blob[src]
        out += [data, off.astype(np.uint32)]
    return tuple(out)


def gpu_info():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:                      # noqa: BLE001
        return 'unknown (%s)' % ex


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--n', type=int, default=943718)
    ap.add_argument('--e2e-steps', type=int, default=10)
    args = ap.parse_args()
    import torch
    import relay_oracle
    from binder_b200._lib import lib
    from binder_b200.engine import Engine, repack
    if not torch.cuda.is_available():
        raise SystemExit('relay_bench: no CUDA device (there is no CPU path to measure)')
    dev = torch.device('cuda:0')
    n = args.n
    tpl = templates()
    eng = Engine('example.com', 'dc1', recursion=True, max_batch=1 << 20)
    # ring of batches: inputs + outputs of the ring exceed the 50 MB L2
    ring, host = [], []
    while True:
        b = tile(tpl, n, seed=len(ring))
        host.append(b)
        q, qo, u, uo = b
        cap = n * 1200
        t = dict(q=torch.from_numpy(q).to(dev), qo=torch.from_numpy(qo.view(np.int32)).to(dev), u=torch.from_numpy(u).to(dev),
                 uo=torch.from_numpy(uo.view(np.int32)).to(dev), out=torch.empty(cap, dtype=torch.uint8, device=dev),
                 off=torch.empty(n + 1, dtype=torch.int32, device=dev), ln=torch.empty(n, dtype=torch.int16, device=dev),
                 st=torch.empty(n, dtype=torch.uint8, device=dev), tot=torch.zeros(4, dtype=torch.int32, device=dev), cap=cap)
        ring.append(t)
        ring_bytes = sum(int(x['q'].numel() + x['u'].numel()) + 8 * n for x in ring)
        if ring_bytes > 2 * 50e6 and len(ring) >= 2:
            break
    stream = torch.cuda.Stream()

    def launch(t):
        eng.relay_device(t['q'].data_ptr(), t['qo'].data_ptr(), t['u'].data_ptr(), t['uo'].data_ptr(), n, t['out'].data_ptr(),
                         t['cap'], t['off'].data_ptr(), t['ln'].data_ptr(), t['st'].data_ptr(), t['tot'].data_ptr(),
                         stream=stream.cuda_stream)
    with torch.cuda.stream(stream):
        for i in range(args.warmup):
            launch(ring[i % len(ring)])
        stream.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream)
        for i in range(args.steps):
            launch(ring[i % len(ring)])
        ev1.record(stream)
        ev1.synchronize()
    ms = ev0.elapsed_time(ev1) / args.steps
    last = (args.steps - 1) % len(ring)
    t = ring[last]
    tot = t['tot'].cpu().numpy().view(np.uint32)
    q, qo, u, uo = host[last]
    want = relay_oracle.relay_batch(q, qo, u, uo, nthreads=os.cpu_count() or 1)
    got = (t['out'][:int(tot[0])].cpu().numpy(), t['off'].cpu().numpy().view(np.uint32), t['ln'].cpu().numpy().view(np.uint16),
           t['st'].cpu().numpy())
    packed, poff = repack(got[0], got[1], got[2])
    parity = bool(np.array_equal(got[3], want[3]) and np.array_equal(got[2], want[2]) and np.array_equal(poff, want[1]) and
                  np.array_equal(packed, want[0]))
    alg = int(qo[-1]) + int(uo[-1]) + int(tot[0]) + n * (4 + 4 + 4 + 2 + 1)
    # e2e: pinned host buffers, one synchronous call per step
    bufs, ptrs = [], []
    for cnt, dt in ((n * 1200, np.uint8), (n + 1, np.uint32), (n, np.uint16), (n, np.uint8)):
        nb = cnt * np.dtype(dt).itemsize
        p = lib().bb_host_alloc(nb)
        ptrs.append(p)
        bufs.append(np.frombuffer((ctypes.c_uint8 * nb).from_address(p), dtype=dt, count=cnt))
    pq, pqo, pu, puo = [], [], [], []
    for arr, lst in ((q, pq), (qo, pqo), (u, pu), (uo, puo)):
        p = lib().bb_host_alloc(arr.nbytes)
        ptrs.append(p)
        v = np.frombuffer((ctypes.c_uint8 * arr.nbytes).from_address(p), dtype=arr.dtype, count=arr.size)
        v[:] = arr
        lst.append(v)
    eng.relay_batch(pq[0], pqo[0], pu[0], puo[0], out=tuple(bufs))
    t0 = time.perf_counter()
    for _ in range(args.e2e_steps):
        eng.relay_batch(pq[0], pqo[0], pu[0], puo[0], out=tuple(bufs))
    e2e_s = (time.perf_counter() - t0) / args.e2e_steps
    for p in ptrs:
        lib().bb_host_free(p)
    t0 = time.perf_counter()
    relay_oracle.relay_batch(q, qo, u, uo, nthreads=os.cpu_count() or 1)
    orc_s = time.perf_counter() - t0
    print(json.dumps({
        'metric': 'relays_per_s', 'value': n / (ms * 1e-3), 'unit': 'relays/s', 'relays_per_step': n,
        'device': {'step_ms': ms, 'steps': args.steps, 'ring_batches': len(ring), 'bytes_per_relay': alg / n,
                   'hbm_frac_of_3.35TBps': alg / (ms * 1e-3) / HBM},
        'e2e': {'relays_per_s': n / e2e_s, 'step_ms': e2e_s * 1e3},
        'oracle_host_threads': {'threads': os.cpu_count(), 'relays_per_s': n / orc_s},
        'parity': 'bit-exact vs oracle, %d relays' % n if parity else 'MISMATCH',
        'mix': MIX, 'gpu': gpu_info()}))
    if not parity:
        sys.exit(1)


if __name__ == '__main__':
    main()
